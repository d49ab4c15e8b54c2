// Keypoint encoder front (3->32->64->128 with folded BN + ReLU) and the channel-first ->
// point-major descriptor transpose.  Keypoints are normalised by the image size of their own view slot (a pair may
// mix portrait and landscape images).  Reference: normalize_keypoints superglue.py:65-72,
// KeypointEncoder multi_view_matcher.py:24-37.  The 128->256->256 tail runs as GEMMs.
#include "../../include/mvm_b200.h"
#include "common.cuh"
#include "kernels.cuh"

namespace {

constexpr int PTS = 64;  // points per block

// normalize_keypoints (superglue.py:65-72) per view slot: x_n = (x - cx) / scale, y_n = (y - cy) / scale
struct KencViews {
  float cx[MVM_MAX_VIEWS], cy[MVM_MAX_VIEWS], scale[MVM_MAX_VIEWS];
  int n_views, n_pad;
};

// Shared-memory layout (floats).  Weights are staged k-major ([k][c]) and activations point-minor ([k][p]) so
// that a thread's register tile (4 points x 4 or 8 channels) is fed by float4 loads that are broadcast across
// the warp: 12 shared loads per 32 FMAs in the dominant 64 -> 128 layer.
constexpr int OFF_W1 = 0;                      // [32][64]
constexpr int OFF_W2 = OFF_W1 + 32 * 64;       // [64][128]
constexpr int OFF_H1 = OFF_W2 + 64 * 128;      // [32][PTS]
constexpr int OFF_H2 = OFF_H1 + 32 * PTS;      // [64][PTS]
constexpr int OFF_IN = OFF_H2 + 64 * PTS;      // [3][PTS]
constexpr int KENC_SMEM = (OFF_IN + 3 * PTS) * 4;

__global__ void __launch_bounds__(256) kenc_front_kernel(const float* __restrict__ kpts,
                                                         const float* __restrict__ kscores,
                                                         const float* w0, const float* b0,
                                                         const float* w1, const float* b1,
                                                         const float* w2, const float* b2,
                                                         float* __restrict__ h3, int n_points,
                                                         const KencViews vt) {
  extern __shared__ float sm[];
  float* s_w1 = sm + OFF_W1; float* s_w2 = sm + OFF_W2;
  float* s_h1 = sm + OFF_H1; float* s_h2 = sm + OFF_H2; float* s_in = sm + OFF_IN;
  const int tid = threadIdx.x;
  const int p0 = blockIdx.x * PTS;
  // stage the two larger weight matrices transposed: w1 [64][32] -> [k][c], w2 [128][64] -> [k][c]
  // (consecutive threads -> consecutive c: conflict-free shared stores; the strided global reads hit L1/L2)
  for (int i = tid; i < 64 * 32; i += 256) { const int k = i / 64, c = i % 64; s_w1[i] = __ldg(w1 + c * 32 + k); }
  for (int i = tid; i < 128 * 64; i += 256) { const int k = i / 128, c = i % 128; s_w2[i] = __ldg(w2 + c * 64 + k); }
  if (tid < PTS) {
    const int p = p0 + tid;
    float x = 0.f, y = 0.f, sc = 0.f;
    if (p < n_points) {
      // the slot's entry by compare-and-select: a dynamic index into the parameter table would go through local memory
      const int v = (p / vt.n_pad) % vt.n_views;
      float cx = vt.cx[0], cy = vt.cy[0], scale = vt.scale[0];
#pragma unroll
      for (int i = 1; i < MVM_MAX_VIEWS; ++i)
        if (i == v) { cx = vt.cx[i]; cy = vt.cy[i]; scale = vt.scale[i]; }
      x = (kpts[2 * p] - cx) / scale;
      y = (kpts[2 * p + 1] - cy) / scale;
      sc = kscores[p];
    }
    s_in[tid] = x; s_in[PTS + tid] = y; s_in[2 * PTS + tid] = sc;
  }
  __syncthreads();
  // layer 0: 3 -> 32 (weights straight from L1; 8 outputs per thread)
  for (int o = tid; o < PTS * 32; o += 256) {
    const int c = o / PTS, p = o % PTS;
    float acc = __ldg(b0 + c);
    acc = fmaf(__ldg(w0 + c * 3 + 0), s_in[p], acc);
    acc = fmaf(__ldg(w0 + c * 3 + 1), s_in[PTS + p], acc);
    acc = fmaf(__ldg(w0 + c * 3 + 2), s_in[2 * PTS + p], acc);
    s_h1[c * PTS + p] = fmaxf(acc, 0.f);
  }
  __syncthreads();
  const int tx = tid & 15, ty = tid >> 4;      // channel group, point group (4 points each)
  // layer 1: 32 -> 64, thread tile 4 points x 4 channels
  {
    float acc[4][4];
    const float4 bb = __ldg(reinterpret_cast<const float4*>(b1) + tx);
#pragma unroll
    for (int i = 0; i < 4; ++i) { acc[i][0] = bb.x; acc[i][1] = bb.y; acc[i][2] = bb.z; acc[i][3] = bb.w; }
#pragma unroll 8
    for (int k = 0; k < 32; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(s_h1 + k * PTS + ty * 4);
      const float4 w = *reinterpret_cast<const float4*>(s_w1 + k * 64 + tx * 4);
      const float av[4] = {a.x, a.y, a.z, a.w}, wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(wv[j], av[i], acc[i][j]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<float4*>(s_h2 + (tx * 4 + j) * PTS + ty * 4) =
          make_float4(fmaxf(acc[0][j], 0.f), fmaxf(acc[1][j], 0.f), fmaxf(acc[2][j], 0.f), fmaxf(acc[3][j], 0.f));
  }
  __syncthreads();
  // layer 2: 64 -> 128, thread tile 4 points x (channels 4tx..4tx+3 and 64+4tx..64+4tx+3: both shared loads
  // contiguous across the 16 lanes of a point group), straight to global
  {
    float acc[4][8];
    const float4 ba = __ldg(reinterpret_cast<const float4*>(b2) + tx), bc = __ldg(reinterpret_cast<const float4*>(b2) + 16 + tx);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      acc[i][0] = ba.x; acc[i][1] = ba.y; acc[i][2] = ba.z; acc[i][3] = ba.w;
      acc[i][4] = bc.x; acc[i][5] = bc.y; acc[i][6] = bc.z; acc[i][7] = bc.w;
    }
#pragma unroll 8
    for (int k = 0; k < 64; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(s_h2 + k * PTS + ty * 4);
      const float4 wa = *reinterpret_cast<const float4*>(s_w2 + k * 128 + tx * 4);
      const float4 wb = *reinterpret_cast<const float4*>(s_w2 + k * 128 + 64 + tx * 4);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float wv[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(wv[j], av[i], acc[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int p = p0 + ty * 4 + i;
      if (p >= n_points) continue;
      float4* o = reinterpret_cast<float4*>(h3 + (long long)p * 128 + tx * 4);
      o[0] = make_float4(fmaxf(acc[i][0], 0.f), fmaxf(acc[i][1], 0.f), fmaxf(acc[i][2], 0.f), fmaxf(acc[i][3], 0.f));
      o[16] = make_float4(fmaxf(acc[i][4], 0.f), fmaxf(acc[i][5], 0.f), fmaxf(acc[i][6], 0.f), fmaxf(acc[i][7], 0.f));
    }
  }
}

// [V, C, n_pad] -> [V, n_pad, C]
__global__ void transpose_cn_kernel(const float* __restrict__ in, float* __restrict__ out, int C,
                                    int n_pad) {
  __shared__ float tile[32][33];
  const int v = blockIdx.z;
  const float* src = in + (long long)v * C * n_pad;
  float* dst = out + (long long)v * C * n_pad;
  const int n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y)
    tile[r][threadIdx.x] = src[(long long)(c0 + r) * n_pad + n0 + threadIdx.x];
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y)
    dst[(long long)(n0 + r) * C + c0 + threadIdx.x] = tile[threadIdx.x][r];
}

}  // namespace

int launch_kenc_front(const float* kpts, const float* kscores, const float* const* w,
                      const float* const* b, float* h3, int n_points, const float* view_wh, int n_views,
                      int n_pad, cudaStream_t stream) {
  MVM_REQUIRE(view_wh && n_views >= 1 && n_views <= MVM_MAX_VIEWS && n_pad >= 1);
  MvmProfScope prof__(MVM_TAG_KENC, stream);
  KencViews vt = {};
  vt.n_views = n_views;
  vt.n_pad = n_pad;
  for (int t = 0; t < n_views; ++t) {
    const float img_w = view_wh[2 * t], img_h = view_wh[2 * t + 1];
    vt.cx[t] = img_w * 0.5f;
    vt.cy[t] = img_h * 0.5f;
    vt.scale[t] = 0.7f * fmaxf(img_w, img_h);
  }
  mvm_once_per_device(MVM_ONCE_KENC, [&] {
    cudaFuncSetAttribute(kenc_front_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, KENC_SMEM);
  });
  kenc_front_kernel<<<mvm_div_up(n_points, PTS), 256, KENC_SMEM, stream>>>(
      kpts, kscores, w[0], b[0], w[1], b[1], w[2], b[2], h3, n_points, vt);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

int launch_transpose_cn(const float* in, float* out, int n_views_total, int C, int n_pad,
                        cudaStream_t stream) {
  MVM_REQUIRE(C % 32 == 0 && n_pad % 32 == 0);
  dim3 grid(n_pad / 32, C / 32, n_views_total), block(32, 8);
  transpose_cn_kernel<<<grid, block, 0, stream>>>(in, out, C, n_pad);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}
