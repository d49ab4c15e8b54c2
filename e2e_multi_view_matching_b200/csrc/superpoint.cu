// SuperPoint front-end (SURVEY.md §8 f-3): the step before the matcher in both eval entry points
// (models/models/superpoint.py:147-229 -- shared VGG encoder, detector head, descriptor head, NMS, descriptor
// sampling), so that eval_pairs / eval_multi_view go image-in -> pose-out on the device.
//
// Layout: activations NHWC fp32 (channels innermost: a warp's 32 pixels x one channel chunk are contiguous loads,
// the 1x1 convolutions are plain row-major GEMMs on the tensor-core kernel).  Weights are repacked on the host to
// [tap][Cin][Cout].
//   sp_conv3x3_kernel     3x3 / pad 1 convolution + bias + ReLU, fp32 CUDA cores: a CTA computes 16 x 16 pixels x 32
//                         output channels, input patch and weights staged in shared memory per 16-channel slice,
//                         2 pixels x 32 channels of accumulators per thread.  (First cut of this row: an implicit-GEMM
//                         tensor-core version is the next step; the 1x1 heads already run on the tensor cores.)
//   sp_maxpool2_kernel    2x2 / stride 2 max pooling; odd sizes floor like nn.MaxPool2d(2, 2) (the last row / column
//                         is dropped), so after three pools the coarse map is h = floor(H/8) x w = floor(W/8)
//   sp_scores_kernel      convPb (1x1, 256 -> 65) + softmax over the 65 bins + depth-to-space into the [8h, 8w] score map
//                         (rows / columns of the image past 8h / 8w have no score, as in the reference)
//   sp_maxpool_rows/cols  separable (2r+1)^2 max filter used by simple_nms (superpoint.py:47-63)
//   sp_nms_step kernels   the reference's three-round suppression, statement for statement
//   sp_l2norm_kernel      per-pixel L2 normalisation of the dense descriptors (:216)
//   sp_sample_kernel      bilinear sampling (grid_sample, align_corners=True) at the keypoints + L2 normalisation (:86-100)
//   sp_sample_batch_kernel  the same sampling for [B, K] keypoints into [B, 256, K] descriptors
//   sp_select_kernel      threshold + border mask + exact top-k of every image of a batch in one launch (radix select)
#include "../../include/mvm_b200.h"
#include "common.cuh"
#include "kernels.cuh"

namespace {

constexpr int TP = 16;                 // tile: 16 x 16 pixels
constexpr int OCB = 32;                // output channels per CTA
constexpr int ICS = 16;                // input channels per shared-memory slice
constexpr int PATCH = TP + 2;          // 18
constexpr int SP_SMEM_IN = ICS * PATCH * PATCH;     // [c][y][x]
constexpr int SP_SMEM_W = 9 * ICS * OCB;            // [tap][c][oc]

// in [B,H,W,Cin] -> out [B,H,W,Cout], w [9][Cin][Cout], bias [Cout]; blockIdx.x = tile, blockIdx.y = Cout / 32, z = image
__global__ void __launch_bounds__(128) sp_conv3x3_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                                         const float* __restrict__ bias, float* __restrict__ out,
                                                         int H, int W, int Cin, int Cout, int relu) {
  __shared__ float s_in[SP_SMEM_IN];
  __shared__ __align__(16) float s_w[SP_SMEM_W];
  const int tiles_x = (W + TP - 1) / TP;
  const int ty0 = (blockIdx.x / tiles_x) * TP, tx0 = (blockIdx.x % tiles_x) * TP;
  const int oc0 = blockIdx.y * OCB;
  const int b = blockIdx.z;
  const int tid = threadIdx.x;
  const int px = tid & 15, py = tid >> 4;            // pixels (py, px) and (py + 8, px) of the tile
  float acc0[OCB], acc1[OCB];
#pragma unroll
  for (int o = 0; o < OCB; ++o) { acc0[o] = 0.f; acc1[o] = 0.f; }
  const float* inb = in + (long long)b * H * W * Cin;
  for (int c0 = 0; c0 < Cin; c0 += ICS) {
    const int nc = min(ICS, Cin - c0);
    __syncthreads();
    // input patch [c][y][x] with zero padding
    for (int e = tid; e < ICS * PATCH * PATCH; e += 128) {
      const int c = e % ICS, p = e / ICS;              // channel fastest in GLOBAL memory -> coalesced reads
      const int yy = p / PATCH, xx = p % PATCH;
      const int gy = ty0 + yy - 1, gx = tx0 + xx - 1;
      float v = 0.f;
      if (c < nc && gy >= 0 && gy < H && gx >= 0 && gx < W) v = inb[((long long)gy * W + gx) * Cin + c0 + c];
      s_in[(c * PATCH + yy) * PATCH + xx] = v;
    }
    for (int e = tid; e < 9 * ICS * OCB; e += 128) {
      const int o = e % OCB, c = (e / OCB) % ICS, t = e / (OCB * ICS);
      float v = 0.f;
      if (c < nc && oc0 + o < Cout) v = w[((long long)t * Cin + c0 + c) * Cout + oc0 + o];
      s_w[e] = v;
    }
    __syncthreads();
#pragma unroll 1
    for (int t = 0; t < 9; ++t) {
      const int dy = t / 3, dx = t % 3;
#pragma unroll 4
      for (int c = 0; c < ICS; ++c) {
        const float a0 = s_in[(c * PATCH + py + dy) * PATCH + px + dx];
        const float a1 = s_in[(c * PATCH + py + 8 + dy) * PATCH + px + dx];
        const float4* wp = reinterpret_cast<const float4*>(s_w + (t * ICS + c) * OCB);
#pragma unroll
        for (int q = 0; q < OCB / 4; ++q) {
          const float4 w4 = wp[q];
          acc0[4 * q] = fmaf(a0, w4.x, acc0[4 * q]); acc0[4 * q + 1] = fmaf(a0, w4.y, acc0[4 * q + 1]);
          acc0[4 * q + 2] = fmaf(a0, w4.z, acc0[4 * q + 2]); acc0[4 * q + 3] = fmaf(a0, w4.w, acc0[4 * q + 3]);
          acc1[4 * q] = fmaf(a1, w4.x, acc1[4 * q]); acc1[4 * q + 1] = fmaf(a1, w4.y, acc1[4 * q + 1]);
          acc1[4 * q + 2] = fmaf(a1, w4.z, acc1[4 * q + 2]); acc1[4 * q + 3] = fmaf(a1, w4.w, acc1[4 * q + 3]);
        }
      }
    }
  }
  float* outb = out + (long long)b * H * W * Cout;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int gy = ty0 + py + half * 8, gx = tx0 + px;
    if (gy < H && gx < W) {
      float* o = outb + ((long long)gy * W + gx) * Cout + oc0;
#pragma unroll
      for (int q = 0; q < OCB; ++q) {
        if (oc0 + q < Cout) {
          float v = (half ? acc1[q] : acc0[q]) + bias[oc0 + q];
          o[q] = relu ? fmaxf(v, 0.f) : v;
        }
      }
    }
  }
}

__global__ void sp_maxpool2_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  const long long n = (long long)B * Ho * Wo * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = i % C;
    const long long p = i / C;
    const int x = p % Wo, y = (p / Wo) % Ho, b = p / ((long long)Wo * Ho);
    const float* s = in + (((long long)b * H + 2 * y) * W + 2 * x) * C + c;
    out[i] = fmaxf(fmaxf(s[0], s[C]), fmaxf(s[(long long)W * C], s[(long long)W * C + C]));
  }
}

// convPb (1x1, 256 -> 65) + softmax over the 65 channels, dustbin dropped, depth-to-space:
// scores[b, 8y + i, 8x + j] = softmax(...)[8 i + j]  (superpoint.py:164-169).  One warp per coarse pixel.
__global__ void __launch_bounds__(256) sp_scores_kernel(const float* __restrict__ feat, const float* __restrict__ w,
                                                        const float* __restrict__ bias, float* __restrict__ scores,
                                                        int B, int h, int w8) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * h * w8) return;
  const int x = warp % w8, y = (warp / w8) % h, b = warp / (w8 * h);
  const float* f = feat + (long long)warp * 256;
  float fr[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) fr[k] = f[lane + 32 * k];
  // lane computes channels lane, lane + 32 and (lane == 0) channel 64; the dot products are warp reductions
  float logit[3] = {0.f, 0.f, 0.f};
  for (int oc = 0; oc < 65; ++oc) {
    const float* wr = w + (long long)oc * 256;
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s = fmaf(fr[k], wr[lane + 32 * k], s);
    s = warp_sum(s) + bias[oc];
    if (oc < 32) { if (lane == oc) logit[0] = s; }
    else if (oc < 64) { if (lane == oc - 32) logit[1] = s; }
    else if (lane == 0) logit[2] = s;
  }
  float mx = fmaxf(logit[0], logit[1]);
  if (lane == 0) mx = fmaxf(mx, logit[2]);
  mx = warp_max(mx);
  const float e0 = expf(logit[0] - mx), e1 = expf(logit[1] - mx), e2 = lane == 0 ? expf(logit[2] - mx) : 0.f;
  const float den = warp_sum(e0 + e1 + e2);
  const int W = w8 * 8;
  float* sb = scores + (long long)b * h * 8 * W;
  {
    const int c = lane, i = c >> 3, j = c & 7;
    sb[(long long)(8 * y + i) * W + 8 * x + j] = e0 / den;
  }
  {
    const int c = lane + 32, i = c >> 3, j = c & 7;
    sb[(long long)(8 * y + i) * W + 8 * x + j] = e1 / den;
  }
}

// separable max filter of radius r with -inf padding (torch max_pool2d pads with -inf)
__global__ void sp_maxrow_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W, int r) {
  const long long n = (long long)B * H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int x = i % W;
    const float* row = in + (i - x);
    float m = -INFINITY;
    for (int d = -r; d <= r; ++d) {
      const int xx = x + d;
      if (xx >= 0 && xx < W) m = fmaxf(m, row[xx]);
    }
    out[i] = m;
  }
}
__global__ void sp_maxcol_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W, int r) {
  const long long n = (long long)B * H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int x = i % W, y = (i / W) % H;
    const float* col = in + (i - (long long)y * W - x) + x;
    float m = -INFINITY;
    for (int d = -r; d <= r; ++d) {
      const int yy = y + d;
      if (yy >= 0 && yy < H) m = fmaxf(m, col[(long long)yy * W]);
    }
    out[i] = m;
  }
}
// simple_nms element-wise steps (superpoint.py:55-63)
__global__ void sp_nms_init_kernel(const float* __restrict__ scores, const float* __restrict__ pooled,
                                   float* __restrict__ mask, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    mask[i] = scores[i] == pooled[i] ? 1.f : 0.f;                               // max_mask = scores == max_pool(scores)
}
__global__ void sp_nms_supp_kernel(const float* __restrict__ scores, const float* __restrict__ pooled_mask,
                                   float* __restrict__ supp_scores, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    supp_scores[i] = pooled_mask[i] > 0.f ? 0.f : scores[i];                    // supp_scores = where(supp_mask, 0, scores)
}
__global__ void sp_nms_update_kernel(const float* __restrict__ supp_scores, const float* __restrict__ pooled_supp,
                                     const float* __restrict__ pooled_mask, float* __restrict__ mask, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const bool new_max = supp_scores[i] == pooled_supp[i];
    if (new_max && !(pooled_mask[i] > 0.f)) mask[i] = 1.f;                      // max_mask |= new_max & ~supp_mask
  }
}
__global__ void sp_nms_final_kernel(const float* __restrict__ scores, const float* __restrict__ mask,
                                    float* __restrict__ out, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = mask[i] > 0.f ? scores[i] : 0.f;
}

// in-place per-pixel L2 normalisation over C = 256 channels (F.normalize, eps 1e-12); one warp per pixel
__global__ void __launch_bounds__(256) sp_l2norm_kernel(float* __restrict__ d, long long n_pix) {
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= n_pix) return;
  float* p = d + warp * 256;
  float v[8], s = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) { v[k] = p[lane + 32 * k]; s = fmaf(v[k], v[k], s); }
  s = warp_sum(s);
  const float inv = 1.f / fmaxf(sqrtf(s), 1e-12f);
#pragma unroll
  for (int k = 0; k < 8; ++k) p[lane + 32 * k] = v[k] * inv;
}

// sample_descriptors (superpoint.py:86-100) for one keypoint, one warp: keypoint (x, y) in pixels of the s = 8 times
// larger image, bilinear grid_sample with align_corners=True on the dense [h, w, 256] map, L2 normalisation; channel c
// goes to out[c * stride].  Both sampling kernels run this code, so their descriptors are the same bits.
__device__ __forceinline__ void sp_sample_point(const float* __restrict__ dense, const float* __restrict__ kp, int h,
                                                int w, int lane, float* __restrict__ out, long long stride) {
  const float s = 8.f;
  float kx = kp[0] - s / 2 + 0.5f, ky = kp[1] - s / 2 + 0.5f;
  kx /= (w * s - s / 2 - 0.5f);
  ky /= (h * s - s / 2 - 0.5f);
  kx = kx * 2 - 1;
  ky = ky * 2 - 1;
  // align_corners=True: pixel = (g + 1) / 2 * (size - 1)
  const float fx = (kx + 1.f) * 0.5f * (w - 1), fy = (ky + 1.f) * 0.5f * (h - 1);
  const float x0f = floorf(fx), y0f = floorf(fy);
  const int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
  const float wx1 = fx - x0f, wx0 = 1.f - wx1, wy1 = fy - y0f, wy0 = 1.f - wy1;
  auto at = [&](int yy, int xx, int c) -> float {
    return (yy >= 0 && yy < h && xx >= 0 && xx < w) ? dense[((long long)yy * w + xx) * 256 + c] : 0.f;   // zeros padding
  };
  float v[8], ss = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int c = lane + 32 * k;
    // same association as grid_sample: nw*w_nw + ne*w_ne + sw*w_sw + se*w_se
    v[k] = at(y0, x0, c) * (wx0 * wy0) + at(y0, x1, c) * (wx1 * wy0) + at(y1, x0, c) * (wx0 * wy1) + at(y1, x1, c) * (wx1 * wy1);
    ss = fmaf(v[k], v[k], ss);
  }
  ss = warp_sum(ss);
  const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
#pragma unroll
  for (int k = 0; k < 8; ++k) out[(lane + 32 * k) * stride] = v[k] * inv;
}

// one image: keypoints [n, 2] -> out [256, n]
__global__ void __launch_bounds__(256) sp_sample_kernel(const float* __restrict__ dense, const float* __restrict__ kpts,
                                                        float* __restrict__ out, int n, int h, int w) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n) return;
  sp_sample_point(dense, kpts + 2 * warp, h, w, lane, out + warp, n);
}

// a batch: dense [B, h, w, 256], keypoints [B, K, 2], counts [B] -> out [B, 256, K]; columns at or past counts[b] are
// zero
__global__ void __launch_bounds__(256) sp_sample_batch_kernel(const float* __restrict__ dense,
                                                              const float* __restrict__ kpts,
                                                              const int* __restrict__ counts, float* __restrict__ out,
                                                              int B, int K, int h, int w) {
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= (long long)B * K) return;
  const int b = (int)(warp / K), i = (int)(warp % K);
  float* o = out + (long long)b * 256 * K + i;
  if (i >= counts[b]) {
#pragma unroll
    for (int k = 0; k < 8; ++k) o[(long long)(lane + 32 * k) * K] = 0.f;
    return;
  }
  sp_sample_point(dense + (long long)b * h * w * 256, kpts + 2 * warp, h, w, lane, o, K);
}

// ---- batched keypoint selection (superpoint.py:181-189 without the host round trips) ----------------------------------
// One CTA per image scans its score map [Hs, Ws] (Hs, Ws multiples of 8, so a float4 never crosses a row).  Candidates
// are the pixels with score > threshold inside the border (remove_borders).  With at most K candidates they are written
// in raster order, which is what torch.nonzero + top_k_keypoints gives when k >= len.  With more, an MSB-first radix
// select over the order-preserving 32-bit keys of the scores (four 8-bit digits, one pass over the map each) finds the
// K-th largest key T and how many keys equal to T are taken; those are the first ones in raster order (the tie rule:
// lower y * Ws + x first).  The K chosen (key, index) pairs are bitonic-sorted in shared memory: descending score,
// ties by raster index.  Candidates are sparse after NMS, so the shared-memory atomics of the histograms are few; the
// cost is the five reads of the map, spread over B CTAs.
constexpr int SEL_THREADS = 1024;
constexpr int SEL_WARPS = SEL_THREADS / 32;

__device__ __forceinline__ unsigned sp_order_key(float s) {   // a > b as floats <=> key(a) > key(b) as unsigned
  const unsigned u = __float_as_uint(s);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// exclusive block-wide prefix sum of v; *total = sum over the block.  Every thread of the block must call it.
__device__ __forceinline__ int sp_block_scan(int v, int* s_warp, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_warp[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int t = s_warp[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += y;
    }
    s_warp[lane] = t;
  }
  __syncthreads();
  const int excl = x - v + (wid ? s_warp[wid - 1] : 0);
  *total = s_warp[SEL_WARPS - 1];
  __syncthreads();                                     // s_warp is reused by the next call
  return excl;
}

// grid = B, block = SEL_THREADS, dynamic shared memory = P * 8 bytes, P = the power of two >= K
__global__ void __launch_bounds__(SEL_THREADS) sp_select_kernel(const float* __restrict__ scores, int Hs, int Ws,
                                                                float thr, int border, int K, float* __restrict__ kpts,
                                                                float* __restrict__ out_scores, int* __restrict__ counts) {
  extern __shared__ unsigned long long s_sel[];        // (key << 32) | ~index: descending order = the output order
  __shared__ int s_hist[256];
  __shared__ int s_warp[SEL_WARPS];
  __shared__ unsigned s_prefix;
  __shared__ int s_krem;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int n = Hs * Ws, n4 = n / 4;
  const float* map = scores + (long long)b * n;
  const float4* map4 = reinterpret_cast<const float4*>(map);
  float* kp_out = kpts + (long long)b * K * 2;
  float* sc_out = out_scores + (long long)b * K;
  auto candidate = [&](int idx, float s) {
    const int y = idx / Ws, x = idx - y * Ws;
    return s > thr && y >= border && y < Hs - border && x >= border && x < Ws - border;
  };

  // radix select: after pass p, prefix holds the top 8 (p + 1) bits of T and krem the rank of T among the keys that
  // share them
  unsigned prefix = 0;
  int krem = K, total = 0;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    for (int i = tid; i < 256; i += SEL_THREADS) s_hist[i] = 0;
    __syncthreads();
    for (int i4 = tid; i4 < n4; i4 += SEL_THREADS) {
      const float4 v4 = map4[i4];
      const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (!candidate(4 * i4 + j, v[j])) continue;
        const unsigned key = sp_order_key(v[j]);
        if (pass == 0 || (key ^ prefix) >> (shift + 8) == 0) atomicAdd(&s_hist[(key >> shift) & 255], 1);
      }
    }
    __syncthreads();
    const int c = tid < 256 ? s_hist[255 - tid] : 0;   // bins from the largest digit down
    int sum;
    const int above = sp_block_scan(c, s_warp, &sum);
    if (pass == 0) {
      total = sum;
      if (total <= K) break;                           // uniform: every thread has the same sum
    }
    if (tid < 256 && above < krem && above + c >= krem) {
      s_prefix = prefix | ((unsigned)(255 - tid) << shift);
      s_krem = krem - above;
    }
    __syncthreads();
    prefix = s_prefix;
    krem = s_krem;
    __syncthreads();
  }
  if (tid == 0) counts[b] = total;

  if (total <= K) {
    // every candidate, raster order, straight to the outputs; zeros past the count
    int base = 0;
    for (int t0 = 0; t0 < n4; t0 += SEL_THREADS) {
      const int i4 = t0 + tid;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      bool take[4] = {false, false, false, false};
      int mine = 0;
      if (i4 < n4) {
        const float4 v4 = map4[i4];
        v[0] = v4.x; v[1] = v4.y; v[2] = v4.z; v[3] = v4.w;
#pragma unroll
        for (int j = 0; j < 4; ++j) { take[j] = candidate(4 * i4 + j, v[j]); mine += take[j]; }
      }
      int tile;
      int pos = base + sp_block_scan(mine, s_warp, &tile);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (!take[j]) continue;
        const int idx = 4 * i4 + j, y = idx / Ws;
        kp_out[2 * pos] = (float)(idx - y * Ws);
        kp_out[2 * pos + 1] = (float)y;
        sc_out[pos] = v[j];
        ++pos;
      }
      base += tile;
    }
    for (int i = total + tid; i < K; i += SEL_THREADS) {
      kp_out[2 * i] = 0.f;
      kp_out[2 * i + 1] = 0.f;
      sc_out[i] = 0.f;
    }
    return;
  }

  // more than K candidates: the keys above T, and the first krem keys equal to T in raster order
  const unsigned T = prefix;
  int base = 0, eq_base = 0;
  for (int t0 = 0; t0 < n4; t0 += SEL_THREADS) {
    const int i4 = t0 + tid;
    unsigned key[4] = {0u, 0u, 0u, 0u};
    bool cand[4] = {false, false, false, false};
    int n_eq = 0;
    if (i4 < n4) {
      const float4 v4 = map4[i4];
      const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        cand[j] = candidate(4 * i4 + j, v[j]);
        key[j] = sp_order_key(v[j]);
        n_eq += cand[j] && key[j] == T;
      }
    }
    int eq_tile;
    int eq_rank = eq_base + sp_block_scan(n_eq, s_warp, &eq_tile);
    bool take[4];
    int mine = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      take[j] = cand[j] && (key[j] > T || (key[j] == T && eq_rank < krem));
      eq_rank += cand[j] && key[j] == T;
      mine += take[j];
    }
    int tile;
    int pos = base + sp_block_scan(mine, s_warp, &tile);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (take[j]) s_sel[pos++] = ((unsigned long long)key[j] << 32) | (unsigned)~(unsigned)(4 * i4 + j);
    base += tile;
    eq_base += eq_tile;
  }
  int P = 1;
  while (P < K) P <<= 1;
  for (int i = K + tid; i < P; i += SEL_THREADS) s_sel[i] = 0ull;   // below every real entry: no finite score has key 0
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P; i += SEL_THREADS) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long a = s_sel[i], c = s_sel[l];
          if ((i & k) == 0 ? a < c : a > c) { s_sel[i] = c; s_sel[l] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (int i = tid; i < K; i += SEL_THREADS) {
    const int idx = (int)~(unsigned)(s_sel[i] & 0xffffffffull), y = idx / Ws;
    kp_out[2 * i] = (float)(idx - y * Ws);
    kp_out[2 * i + 1] = (float)y;
    sc_out[i] = map[idx];
  }
}

int conv3x3(const float* in, const float* w, const float* b, float* out, int B, int H, int W, int Cin, int Cout, int relu,
            cudaStream_t s) {
  dim3 grid(((H + TP - 1) / TP) * ((W + TP - 1) / TP), (Cout + OCB - 1) / OCB, B);
  sp_conv3x3_kernel<<<grid, 128, 0, s>>>(in, w, b, out, H, W, Cin, Cout, relu);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}
int maxpool2(const float* in, float* out, int B, int H, int W, int C, cudaStream_t s) {
  sp_maxpool2_kernel<<<mvm_dev_info().n_sm * 8, 256, 0, s>>>(in, out, B, H, W, C);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}
int maxfilter(const float* in, float* tmp, float* out, int B, int H, int W, int r, cudaStream_t s) {
  sp_maxrow_kernel<<<mvm_dev_info().n_sm * 4, 256, 0, s>>>(in, tmp, B, H, W, r);
  MVM_CHECK_LAUNCH();
  sp_maxcol_kernel<<<mvm_dev_info().n_sm * 4, 256, 0, s>>>(tmp, out, B, H, W, r);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

#define SP_TRY(x)                     \
  do {                                \
    int rc__ = (x);                   \
    if (rc__ != MVM_OK) return rc__;  \
  } while (0)

}  // namespace

extern "C" {

size_t mvm_superpoint_workspace_bytes(int batch, int height, int width) {
  const size_t px = (size_t)batch * height * width;
  // two ping-pong activation buffers at full resolution x 64 channels + 5 score-map planes
  return (2 * px * 64 + 5 * px) * sizeof(float) + 1024;
}

int mvm_superpoint_dense(const mvm_superpoint_weights* wt, const float* image, int batch, int height, int width,
                         int nms_radius, float* scores_nms, float* dense_desc, void* workspace, size_t workspace_bytes,
                         void* stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MVM_REQUIRE(wt && image && scores_nms && dense_desc && workspace);
  MVM_REQUIRE(batch >= 1 && height >= 16 && width >= 16 && nms_radius >= 0);
  if (workspace_bytes < mvm_superpoint_workspace_bytes(batch, height, width)) return MVM_ERR_WORKSPACE;
  MvmProfScope prof__(MVM_TAG_MISC, s);
  const size_t px = (size_t)batch * height * width;
  float* A = reinterpret_cast<float*>(workspace);
  float* Bf = A + px * 64;
  float* P0 = Bf + px * 64;          // score-map planes
  float* P1 = P0 + px; float* P2 = P1 + px; float* P3 = P2 + px; float* P4 = P3 + px;
  int H = height, W = width;
  // shared encoder (superpoint.py:150-161); image [B,H,W] == NHWC with C = 1
  SP_TRY(conv3x3(image, wt->w[0], wt->b[0], A, batch, H, W, 1, 64, 1, s));
  SP_TRY(conv3x3(A, wt->w[1], wt->b[1], Bf, batch, H, W, 64, 64, 1, s));
  SP_TRY(maxpool2(Bf, A, batch, H, W, 64, s)); H /= 2; W /= 2;
  SP_TRY(conv3x3(A, wt->w[2], wt->b[2], Bf, batch, H, W, 64, 64, 1, s));
  SP_TRY(conv3x3(Bf, wt->w[3], wt->b[3], A, batch, H, W, 64, 64, 1, s));
  SP_TRY(maxpool2(A, Bf, batch, H, W, 64, s)); H /= 2; W /= 2;
  SP_TRY(conv3x3(Bf, wt->w[4], wt->b[4], A, batch, H, W, 64, 128, 1, s));
  SP_TRY(conv3x3(A, wt->w[5], wt->b[5], Bf, batch, H, W, 128, 128, 1, s));
  SP_TRY(maxpool2(Bf, A, batch, H, W, 128, s)); H /= 2; W /= 2;
  SP_TRY(conv3x3(A, wt->w[6], wt->b[6], Bf, batch, H, W, 128, 128, 1, s));
  SP_TRY(conv3x3(Bf, wt->w[7], wt->b[7], A, batch, H, W, 128, 128, 1, s));      // x = A  [B, H/8, W/8, 128]
  const long long cpx = (long long)batch * H * W;
  // detector head (:163-170)
  SP_TRY(conv3x3(A, wt->w[8], wt->b[8], Bf, batch, H, W, 128, 256, 1, s));       // cPa
  sp_scores_kernel<<<(int)((cpx * 32 + 255) / 256), 256, 0, s>>>(Bf, wt->w_pb, wt->b_pb, P0, batch, H, W);
  MVM_CHECK_LAUNCH();
  // simple_nms (:47-63) on the [8h, 8w] score map
  const int hs = 8 * H, ws = 8 * W;
  {
    const long long n = (long long)batch * hs * ws;
    const int blocks = mvm_dev_info().n_sm * 4;
    SP_TRY(maxfilter(P0, P4, P1, batch, hs, ws, nms_radius, s));                  // P1 = max_pool(scores)
    sp_nms_init_kernel<<<blocks, 256, 0, s>>>(P0, P1, P2, n);                    // P2 = max_mask
    MVM_CHECK_LAUNCH();
    for (int it = 0; it < 2; ++it) {
      SP_TRY(maxfilter(P2, P4, P1, batch, hs, ws, nms_radius, s));                // P1 = max_pool(max_mask)  (> 0 = supp_mask)
      sp_nms_supp_kernel<<<blocks, 256, 0, s>>>(P0, P1, P3, n);                  // P3 = supp_scores
      MVM_CHECK_LAUNCH();
      float* pooled_supp = scores_nms;                                           // scratch until the final write
      SP_TRY(maxfilter(P3, P4, pooled_supp, batch, hs, ws, nms_radius, s));
      sp_nms_update_kernel<<<blocks, 256, 0, s>>>(P3, pooled_supp, P1, P2, n);
      MVM_CHECK_LAUNCH();
    }
    sp_nms_final_kernel<<<blocks, 256, 0, s>>>(P0, P2, scores_nms, n);
    MVM_CHECK_LAUNCH();
  }
  // descriptor head (:213-216): convDa (3x3) on the CUDA cores, convDb (1x1) on the tensor cores (3xTF32)
  SP_TRY(conv3x3(A, wt->w[9], wt->b[9], Bf, batch, H, W, 128, 256, 1, s));       // cDa
  {
    GemmDesc g;
    g.A = Bf; g.lda = 256; g.A2 = nullptr; g.lda2 = 0; g.K1 = 256;
    g.W = wt->w_db; g.ldw = 256; g.Whi = nullptr; g.Wlo = nullptr; g.Whi16 = nullptr; g.Wlo16 = nullptr; g.wscale = 0.f;
    g.bias = wt->b_db; g.R = nullptr; g.ldr = 0;
    g.C = dense_desc; g.ldc = 256; g.M = (int)cpx; g.N = 256; g.K = 256; g.alpha = 1.f; g.relu = 0;
    g.batch = 1; g.sA = g.sA2 = g.sW = g.sR = g.sC = 0;
    SP_TRY(launch_gemm_tc(g, 3, nullptr, 0, 0, s, nullptr, nullptr, 128, 0));
  }
  sp_l2norm_kernel<<<(int)((cpx * 32 + 255) / 256), 256, 0, s>>>(dense_desc, cpx);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

int mvm_superpoint_sample(const float* dense_desc, const float* keypoints, int n, int h, int w, float* descriptors,
                          void* stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MVM_REQUIRE(dense_desc && descriptors && n >= 0 && h >= 1 && w >= 1 && (n == 0 || keypoints));
  if (n == 0) return MVM_OK;
  MvmProfScope prof__(MVM_TAG_MISC, s);
  sp_sample_kernel<<<(n * 32 + 255) / 256, 256, 0, s>>>(dense_desc, keypoints, descriptors, n, h, w);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

int mvm_superpoint_select(const float* scores_nms, int batch, int height, int width, float keypoint_threshold,
                          int remove_borders, int max_keypoints, float* keypoints, float* scores, int* counts,
                          void* stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MVM_REQUIRE(scores_nms && keypoints && scores && counts);
  MVM_REQUIRE(((uintptr_t)scores_nms & 15) == 0);                                     // read as float4
  MVM_REQUIRE(batch >= 1 && height >= 8 && width >= 8 && height % 8 == 0 && width % 8 == 0);
  MVM_REQUIRE((long long)height * width <= 0x7fffffffLL && batch <= 65535);
  MVM_REQUIRE(remove_borders >= 0 && keypoint_threshold == keypoint_threshold);        // not NaN
  MVM_REQUIRE(max_keypoints >= 1 && max_keypoints <= MVM_SUPERPOINT_MAX_SELECT &&
              (long long)max_keypoints <= (long long)height * width);
  MvmProfScope prof__(MVM_TAG_MISC, s);
  int P = 1;
  while (P < max_keypoints) P <<= 1;
  const int smem = P * (int)sizeof(unsigned long long);
  mvm_once_per_device(MVM_ONCE_SP_SELECT, [&] {
    cudaFuncSetAttribute(sp_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         MVM_SUPERPOINT_MAX_SELECT * (int)sizeof(unsigned long long));
  });
  sp_select_kernel<<<batch, SEL_THREADS, smem, s>>>(scores_nms, height, width, keypoint_threshold, remove_borders,
                                                    max_keypoints, keypoints, scores, counts);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

int mvm_superpoint_sample_batch(const float* dense_desc, const float* keypoints, const int* counts, int batch,
                                int max_keypoints, int h, int w, float* descriptors, void* stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MVM_REQUIRE(dense_desc && keypoints && counts && descriptors);
  MVM_REQUIRE(batch >= 1 && max_keypoints >= 1 && h >= 1 && w >= 1);
  const long long warps = (long long)batch * max_keypoints;
  MVM_REQUIRE(warps * 32 / 256 < 0x7fffffffLL);
  MvmProfScope prof__(MVM_TAG_MISC, s);
  sp_sample_batch_kernel<<<(int)((warps * 32 + 255) / 256), 256, 0, s>>>(dense_desc, keypoints, counts, descriptors,
                                                                         batch, max_keypoints, h, w);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

}  // extern "C"
