// Training-image preparation (datasets/matching_dataset.py:182-211) for a batch of decoded uint8 RGB images:
// ToTensor, square crop, zero-row pad, bilinear resize, ColorJitter in the drawn order, rgb_to_grayscale.
//
// Every step reproduces the float32 torch / torchvision op sequence of the reference, one rounding per torch op:
// the arithmetic below is written with __fmul_rn / __fadd_rn / __fdiv_rn, which nvcc never contracts.  The two
// fused multiply-adds of the resize are the ones torch's CPU bilinear kernel (generic N-d path, AVX2 build) performs.
//
// Launches: without jitter one pass (prep_kernel<false, 2>).  With jitter, adjust_contrast needs the mean of the
// grayscale image as it stands when contrast comes up in the order: pass 1 applies the ops before contrast and
// writes per-CTA fp64 partial sums of the grayscale image (fixed assignment of pixels to threads, fixed reduction
// tree: deterministic, independent of the batch size); pass 2 finishes the mean, recomputes the ops before contrast
// and applies the rest and the grayscale conversion.  Recomputing re-reads the uint8 source, a quarter of the size
// of a float RGB intermediate; the intermediate-buffer variant has not been timed against it.
#include "common.cuh"
#include "../../include/mvm_b200.h"

namespace {

constexpr int IP_THREADS = 256;
constexpr int IP_MAX_BLOCKS_PER_IMAGE = 256;

struct Geom {
  int top, left, ch, cw, pad_top, pad_bottom;
};

__device__ __forceinline__ float clamp01(float x) { return fminf(fmaxf(x, 0.f), 1.f); }

// _blend(img1, img2, ratio) = (ratio * img1 + (1.0 - ratio) * img2).clamp(0, 1), ratio and 1.0 - ratio rounded to
// float32 from the Python doubles.
__device__ __forceinline__ float blend(float x, float y, float f, float fc) {
  return clamp01(__fadd_rn(__fmul_rn(x, f), __fmul_rn(y, fc)));
}

// rgb_to_grayscale: (0.2989 * r + 0.587 * g + 0.114 * b), left to right.
__device__ __forceinline__ float gray(float r, float g, float b) {
  return __fadd_rn(__fadd_rn(__fmul_rn(r, 0.2989f), __fmul_rn(g, 0.587f)), __fmul_rn(b, 0.114f));
}

// adjust_hue: _rgb2hsv, (h + hue) % 1.0, _hsv2rgb, as torchvision's tensor code writes them.
__device__ __forceinline__ void hue_shift(float& r, float& g, float& b, float hue) {
  const float maxc = fmaxf(fmaxf(r, g), b);
  const float minc = fminf(fminf(r, g), b);
  const bool eqc = maxc == minc;
  const float cr = __fsub_rn(maxc, minc);
  const float s = __fdiv_rn(cr, eqc ? 1.f : maxc);
  const float crd = eqc ? 1.f : cr;
  const float rc = __fdiv_rn(__fsub_rn(maxc, r), crd);
  const float gc = __fdiv_rn(__fsub_rn(maxc, g), crd);
  const float bc = __fdiv_rn(__fsub_rn(maxc, b), crd);
  // bool * float: the mask is 0.0 or 1.0 and the product keeps the sign of zero
  const float hr = __fmul_rn(maxc == r ? 1.f : 0.f, __fsub_rn(bc, gc));
  const float hg = __fmul_rn((maxc == g && maxc != r) ? 1.f : 0.f, __fsub_rn(__fadd_rn(rc, 2.f), bc));
  const float hb = __fmul_rn((maxc != g && maxc != r) ? 1.f : 0.f, __fsub_rn(__fadd_rn(gc, 4.f), rc));
  float h = __fadd_rn(__fadd_rn(hr, hg), hb);
  h = fmodf(__fadd_rn(__fdiv_rn(h, 6.f), 1.f), 1.f);
  // torch.remainder for floats: fmod, then + divisor when the result is non-zero and of the other sign
  h = fmodf(__fadd_rn(h, hue), 1.f);
  if (h != 0.f && h < 0.f) h = __fadd_rn(h, 1.f);
  const float v = maxc;
  const float h6 = __fmul_rn(h, 6.f);
  const float fi = floorf(h6);
  const float f = __fsub_rn(h6, fi);
  int i = (int)fi;
  const float p = clamp01(__fmul_rn(v, __fsub_rn(1.f, s)));
  const float q = clamp01(__fmul_rn(v, __fsub_rn(1.f, __fmul_rn(s, f))));
  const float t = clamp01(__fmul_rn(v, __fsub_rn(1.f, __fmul_rn(s, __fsub_rn(1.f, f)))));
  i = ((i % 6) + 6) % 6;
  switch (i) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
}

struct Jitter {
  int order[4];
  float f[4], fc[4];   // float32(factor), float32(1.0 - factor); f[3] = float32(hue)
  int contrast_pos;    // index of op 1 in order
};

// op 0 brightness, 1 contrast (needs the mean), 2 saturation, 3 hue
__device__ __forceinline__ void apply_op(int op, const Jitter& j, float mean, float& r, float& g, float& b) {
  if (op == 0) {
    r = blend(r, 0.f, j.f[0], j.fc[0]); g = blend(g, 0.f, j.f[0], j.fc[0]); b = blend(b, 0.f, j.f[0], j.fc[0]);
  } else if (op == 1) {
    r = blend(r, mean, j.f[1], j.fc[1]); g = blend(g, mean, j.f[1], j.fc[1]); b = blend(b, mean, j.f[1], j.fc[1]);
  } else if (op == 2) {
    const float l = gray(r, g, b);
    r = blend(r, l, j.f[2], j.fc[2]); g = blend(g, l, j.f[2], j.fc[2]); b = blend(b, l, j.f[2], j.fc[2]);
  } else {
    hue_shift(r, g, b, j.f[3]);
  }
}

// ToTensor of one source pixel of the cropped, padded image (row y counts the pad rows above the crop).
__device__ __forceinline__ void load_px(const unsigned char* img, int src_w, const Geom& gm, int y, int x, float& r,
                                        float& g, float& b) {
  const int yy = y - gm.pad_top;
  if (yy < 0 || yy >= gm.ch) { r = g = b = 0.f; return; }
  const unsigned char* p = img + ((size_t)(gm.top + yy) * src_w + (gm.left + x)) * 3;
  r = __fdiv_rn((float)p[0], 255.f);
  g = __fdiv_rn((float)p[1], 255.f);
  b = __fdiv_rn((float)p[2], 255.f);
}

// upsample_bilinear2d, align_corners=False, no antialiasing, scale = in / out: source index, lambdas and the
// index clamp of torch's compute_source_index_and_lambda.
__device__ __forceinline__ void lin_coef(int o, int in, int out, int& i0, int& i1, float& l0, float& l1) {
  const float scale = __fdiv_rn((float)in, (float)out);
  float s = __fmaf_rn(scale, __fadd_rn((float)o, 0.5f), -0.5f);
  s = s < 0.f ? 0.f : s;
  i0 = min((int)floorf(s), in - 1);
  l1 = fminf(fmaxf(__fsub_rn(s, (float)i0), 0.f), 1.f);
  l0 = __fsub_rn(1.f, l1);
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
}

__device__ __forceinline__ float lerp2(float a, float b, float wa, float wb) { return __fmaf_rn(a, wa, __fmul_rn(b, wb)); }

// The RGB of output pixel (oy, ox) before jitter.
__device__ __forceinline__ void source_rgb(const unsigned char* img, int src_w, const Geom& gm, int out_h, int out_w,
                                           int oy, int ox, float& r, float& g, float& b) {
  const int in_h = gm.ch + gm.pad_top + gm.pad_bottom, in_w = gm.cw;
  if (in_h == out_h && in_w == out_w) { load_px(img, src_w, gm, oy, ox, r, g, b); return; }
  int y0, y1, x0, x1;
  float ly0, ly1, lx0, lx1;
  lin_coef(oy, in_h, out_h, y0, y1, ly0, ly1);
  lin_coef(ox, in_w, out_w, x0, x1, lx0, lx1);
  float r00, g00, b00, r01, g01, b01, r10, g10, b10, r11, g11, b11;
  load_px(img, src_w, gm, y0, x0, r00, g00, b00);
  load_px(img, src_w, gm, y0, x1, r01, g01, b01);
  load_px(img, src_w, gm, y1, x0, r10, g10, b10);
  load_px(img, src_w, gm, y1, x1, r11, g11, b11);
  r = lerp2(lerp2(r00, r01, lx0, lx1), lerp2(r10, r11, lx0, lx1), ly0, ly1);
  g = lerp2(lerp2(g00, g01, lx0, lx1), lerp2(g10, g11, lx0, lx1), ly0, ly1);
  b = lerp2(lerp2(b00, b01, lx0, lx1), lerp2(b10, b11, lx0, lx1), ly0, ly1);
}

__device__ __forceinline__ bool load_params(const int* geometry, const int* jitter_order, const double* jitter_factors,
                                            int img, int src_h, int src_w, int out_h, int out_w, bool jitter, Geom& gm,
                                            Jitter& j) {
  const int* gp = geometry + (size_t)img * 6;
  gm = Geom{gp[0], gp[1], gp[2], gp[3], gp[4], gp[5]};
  // the host refuses these before any launch; device-resident values are re-checked so that no load leaves the image
  bool ok = gm.top >= 0 && gm.left >= 0 && gm.ch >= 1 && gm.cw >= 1 && gm.top + gm.ch <= src_h &&
            gm.left + gm.cw <= src_w && gm.pad_top >= 0 && gm.pad_bottom >= 0;
  if (!jitter) return ok;
  unsigned seen = 0;
  j.contrast_pos = -1;
  for (int k = 0; k < 4; ++k) {
    const int op = jitter_order[(size_t)img * 4 + k];
    j.order[k] = op;
    if (op < 0 || op > 3) return false;
    seen |= 1u << op;
    if (op == 1) j.contrast_pos = k;
  }
  for (int k = 0; k < 4; ++k) {
    const double v = jitter_factors[(size_t)img * 4 + k];
    j.f[k] = __double2float_rn(v);
    j.fc[k] = __double2float_rn(1.0 - v);
  }
  return ok && seen == 0xfu;
}

// PASS 1: ops before contrast, fp64 partial sums of the grayscale image per CTA.
// PASS 2: mean from the partial sums (with jitter), all ops, grayscale out.
template <bool JITTER, int PASS>
__global__ void __launch_bounds__(IP_THREADS) prep_kernel(const unsigned char* __restrict__ rgb, int src_h, int src_w,
                                                          const int* __restrict__ geometry,
                                                          const int* __restrict__ jitter_order,
                                                          const double* __restrict__ jitter_factors, int out_h,
                                                          int out_w, float* __restrict__ out,
                                                          double* __restrict__ partial) {
  const int img = blockIdx.y;
  const int nblk = gridDim.x;
  const long long npix = (long long)out_h * out_w;
  Geom gm;
  Jitter j;
  const bool ok = load_params(geometry, jitter_order, jitter_factors, img, src_h, src_w, out_h, out_w, JITTER, gm, j);
  const unsigned char* src = rgb + (size_t)img * src_h * src_w * 3;
  __shared__ double red[IP_THREADS / 32];
  __shared__ float s_mean;

  if (PASS == 2 && JITTER) {
    if (threadIdx.x < 32) {
      double acc = 0.0;
      for (int k = threadIdx.x; k < nblk; k += 32) acc += partial[(size_t)img * nblk + k];
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (threadIdx.x == 0) s_mean = (float)(acc / (double)npix);
    }
    __syncthreads();
  }
  const float mean = (PASS == 2 && JITTER) ? s_mean : 0.f;
  float* dst = out + (size_t)img * npix;
  double acc = 0.0;
  for (long long p = (long long)blockIdx.x * IP_THREADS + threadIdx.x; p < npix; p += (long long)nblk * IP_THREADS) {
    const int oy = (int)(p / out_w), ox = (int)(p % out_w);
    if (!ok) {
      if (PASS == 2) dst[p] = __int_as_float(0x7fc00000);
      continue;
    }
    float r, g, b;
    source_rgb(src, src_w, gm, out_h, out_w, oy, ox, r, g, b);
    if (JITTER) {
      const int stop = PASS == 1 ? j.contrast_pos : 4;
#pragma unroll
      for (int k = 0; k < 4; ++k)   // unrolled so that the parameters stay in registers
        if (k < stop) apply_op(j.order[k], j, mean, r, g, b);
    }
    if (PASS == 1) acc += (double)gray(r, g, b);
    else dst[p] = gray(r, g, b);
  }
  if (PASS == 1) {
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int w = 0; w < IP_THREADS / 32; ++w) s += red[w];
      partial[(size_t)img * nblk + blockIdx.x] = s;
    }
  }
}

int blocks_per_image(int out_h, int out_w) {
  const long long npix = (long long)out_h * out_w;
  const long long b = (npix + IP_THREADS * 4 - 1) / (IP_THREADS * 4);
  return (int)(b < IP_MAX_BLOCKS_PER_IMAGE ? b : IP_MAX_BLOCKS_PER_IMAGE);
}

}  // namespace

extern "C" {

size_t mvm_image_prep_workspace_bytes(int n, int out_h, int out_w) {
  if (n < 1 || out_h < 1 || out_w < 1) return 0;
  return (size_t)n * blocks_per_image(out_h, out_w) * sizeof(double);
}

int mvm_image_prep(const unsigned char* rgb, int n, int src_h, int src_w, const int* geometry, const int* jitter_order,
                   const double* jitter_factors, int out_h, int out_w, float* out, void* workspace,
                   size_t workspace_bytes, void* stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MVM_REQUIRE(rgb && geometry && out);
  MVM_REQUIRE((jitter_order == nullptr) == (jitter_factors == nullptr));
  MVM_REQUIRE(n >= 1 && n <= 65535 && src_h >= 1 && src_w >= 1 && out_h >= 1 && out_w >= 1);
  MVM_REQUIRE((long long)src_h * src_w * 3 <= 0x7fffffffLL && (long long)out_h * out_w <= 0x7fffffffLL);
  const int nblk = blocks_per_image(out_h, out_w);
  const dim3 grid(nblk, n);
  MvmProfScope prof__(MVM_TAG_MISC, s);
  if (jitter_order) {
    MVM_REQUIRE(workspace && workspace_bytes >= mvm_image_prep_workspace_bytes(n, out_h, out_w));
    double* partial = (double*)workspace;
    prep_kernel<true, 1><<<grid, IP_THREADS, 0, s>>>(rgb, src_h, src_w, geometry, jitter_order, jitter_factors, out_h,
                                                     out_w, out, partial);
    MVM_CHECK_LAUNCH();
    prep_kernel<true, 2><<<grid, IP_THREADS, 0, s>>>(rgb, src_h, src_w, geometry, jitter_order, jitter_factors, out_h,
                                                     out_w, out, partial);
    MVM_CHECK_LAUNCH();
  } else {
    prep_kernel<false, 2><<<grid, IP_THREADS, 0, s>>>(rgb, src_h, src_w, geometry, nullptr, nullptr, out_h, out_w,
                                                      out, nullptr);
    MVM_CHECK_LAUNCH();
  }
  return MVM_OK;
}

}  // extern "C"
