// fp32 CUDA-core GEMM with fused epilogue (bias, ReLU, residual, concat-by-K-split).
// Exact-fp32 path used for (a) small/odd shapes (score matrix with ldc = n+1, keypoint
// encoder) and (b) as the on-device cross-check of the tensor-core path.
// Replaces the reference's nn.Conv1d(k=1)+BatchNorm1d(eval)+ReLU chains
// (superglue.py:51-62,101-121; multi_view_matcher.py:8-53) on point-major activations.
#include "common.cuh"
#include "kernels.cuh"

namespace {

constexpr int BM = 128, BN = 128, BK = 16, PAD = 4;

__device__ __forceinline__ void gemm_body(const GemmDesc& g, const float* __restrict__ A,
                                          const float* __restrict__ A2,
                                          const float* __restrict__ W,
                                          const float* __restrict__ R, float* __restrict__ C,
                                          int m0, int n0) {
  __shared__ float As[2][BK][BM + PAD];
  __shared__ float Bs[2][BK][BN + PAD];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;

  // global->smem load mapping: 128 rows x 4 float4 (BK=16) = 512 float4, 2 per thread
  const int lrow = tid >> 2;          // 0..63 (+64 for the second)
  const int lk4 = (tid & 3) * 4;      // 0,4,8,12

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 ra[2], rb[2];
  const int nk = g.K / BK;

  auto load_tile = [&](int kt) {
    const int k = kt * BK + lk4;
    const float* Ap;
    int ld, kk;
    if (k < g.K1) { Ap = A; ld = g.lda; kk = k; } else { Ap = A2; ld = g.lda2; kk = k - g.K1; }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + lrow + h * 64;
      ra[h] = (m < g.M) ? *reinterpret_cast<const float4*>(Ap + (long long)m * ld + kk)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
      const int n = n0 + lrow + h * 64;
      rb[h] = (n < g.N) ? *reinterpret_cast<const float4*>(W + (long long)n * g.ldw + k)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store_tile = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = lrow + h * 64;
      As[buf][lk4 + 0][r] = ra[h].x; As[buf][lk4 + 1][r] = ra[h].y;
      As[buf][lk4 + 2][r] = ra[h].z; As[buf][lk4 + 3][r] = ra[h].w;
      Bs[buf][lk4 + 0][r] = rb[h].x; Bs[buf][lk4 + 1][r] = rb[h].y;
      Bs[buf][lk4 + 2][r] = rb[h].z; Bs[buf][lk4 + 3][r] = rb[h].w;
    }
  };

  load_tile(0);
  store_tile(0);
  __syncthreads();

  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tile(kt + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_tile(buf ^ 1);
      __syncthreads();
    }
  }

  // epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (n >= g.N) continue;
      float v = g.alpha * acc[i][j];
      if (g.bias) v += g.bias[n];
      if (g.relu) v = fmaxf(v, 0.f);
      if (R) v += R[(long long)m * g.ldr + n];
      C[(long long)m * g.ldc + n] = v;
    }
  }
}

__global__ void __launch_bounds__(256, 2) gemm_simt_kernel(GemmDesc g) {
  const int bz = blockIdx.z;
  gemm_body(g, g.A + bz * g.sA, g.A2 ? g.A2 + bz * g.sA2 : nullptr, g.W + bz * g.sW,
            g.R ? g.R + bz * g.sR : nullptr, g.C + bz * g.sC, blockIdx.y * BM, blockIdx.x * BN);
}

// One launch for every (pair, batch) score matrix: scores = mdesc_a . mdesc_b^T * alpha into
// the inner [m,n] block of the [m+1,n+1] coupling buffer (multi_view_matcher.py:278-280).
__global__ void __launch_bounds__(256, 2) score_gemm_simt_kernel(const float* __restrict__ mdesc,
                                                                 int n_pad, PairTable tab,
                                                                 int batch, float alpha) {
  const int prob = blockIdx.z;
  const int p = prob / batch, bi = prob % batch;
  const int m = tab.m[p], n = tab.n[p];
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  if (m0 >= m || n0 >= n) return;
  GemmDesc g;
  g.lda = 256; g.A2 = nullptr; g.lda2 = 0; g.K1 = 256; g.ldw = 256; g.bias = nullptr;
  g.R = nullptr; g.ldr = 0; g.ldc = n + 1; g.M = m; g.N = n; g.K = 256; g.alpha = alpha;
  g.relu = 0;
  const float* A = mdesc + (long long)(bi * tab.n_views + tab.a[p]) * n_pad * 256;
  const float* W = mdesc + (long long)(bi * tab.n_views + tab.b[p]) * n_pad * 256;
  float* C = tab.scores[p] + (long long)bi * (m + 1) * (n + 1);
  gemm_body(g, A, nullptr, W, nullptr, C, m0, n0);
}

}  // namespace

int launch_score_gemm_simt(const float* mdesc, int n_pad, const PairTable& tab, int batch,
                           float alpha, cudaStream_t stream) {
  MvmProfScope prof__(MVM_TAG_SCORE, stream);
  int max_m = 0, max_n = 0;
  for (int p = 0; p < tab.n_pairs; ++p) {
    max_m = tab.m[p] > max_m ? tab.m[p] : max_m;
    max_n = tab.n[p] > max_n ? tab.n[p] : max_n;
  }
  dim3 grid(mvm_div_up(max_n, BN), mvm_div_up(max_m, BM), tab.n_pairs * batch);
  score_gemm_simt_kernel<<<grid, 256, 0, stream>>>(mdesc, n_pad, tab, batch, alpha);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

int launch_gemm_simt(const GemmDesc& g, cudaStream_t stream) {
  static_assert(BK == 16, "gemm_desc_valid(GEMM_SIMT) states K in k-blocks of 16");
  MVM_REQUIRE(gemm_desc_valid(g, GEMM_SIMT));
  MvmProfScope prof__(MVM_TAG_GEMM, stream);
  dim3 grid(mvm_div_up(g.N, BN), mvm_div_up(g.M, BM), g.batch);
  gemm_simt_kernel<<<grid, 256, 0, stream>>>(g);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}
