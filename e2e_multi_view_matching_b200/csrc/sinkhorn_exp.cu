// Production Sinkhorn: stabilised scaling-domain iteration with the kernel matrix resident in
// shared memory.  Same fixed point and the same 100 iterations as log_optimal_transport /
// log_sinkhorn_iterations (superglue.py:143-172), reformulated so that the inner loops are pure FMA:
//
//   K~_ij = exp(Z_ij + u~_i + v~_j)            (absorbed potentials u~, v~; stored in shared memory)
//   row:  a_i = mu_i / sum_j K~_ij b_j         <=>  u_i = log_mu_i - LSE_j(Z_ij + v_j),  u = u~ + log a
//   col:  b_j = nu_j / sum_i K~_ij a_i         <=>  v_j = log_nu_j - LSE_i(Z_ij + u_i),  v = v~ + log b
//
// The reference evaluates 2.1e8 exp per 1024^2 pair (SURVEY.md §8d); here exp is evaluated once per
// element plus once per re-absorption (when a scaling leaves [e^-8, e^8], which happens a handful of
// times in the first iterations), so the 100 iterations cost 2 FMA per element each.  A group of G
// co-resident CTAs owns one problem, CTA c keeps rows [c*R, (c+1)*R) of K~; column sums are exchanged
// through L2 with two software group barriers per iteration and merged in a fixed order
// (deterministic).  Dustbin row/column are rank-1 and never stored.  The raw scores stay in the
// output buffer (L2) until the final pass rewrites them as Z + u + v - norm.
#include "common.cuh"
#include "kernels.cuh"

namespace {

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void group_barrier(unsigned* ctr, unsigned target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    red_release_add(ctr, 1u);
    while (ld_acquire_u32(ctr) < target) {}
  }
  __syncthreads();
}

struct SinkCfg {
  int G, NG, batch, iters;
  float alpha;
  int xch_stride;
  long long* timing;   // optional [8] cycle counters of CTA 0 (debug/profiling), or null
};

constexpr float ABSORB_HI = 2980.958f;     // e^8
constexpr float ABSORB_LO = 3.3546263e-4f; // e^-8

__global__ void __launch_bounds__(1024, 1) sinkhorn_exp_kernel(PairTable tab, SinkCfg cfg,
                                                               float* __restrict__ xch,
                                                               unsigned* __restrict__ ctrs) {
  extern __shared__ float smem[];
  __shared__ float s_red[32];
  __shared__ int s_flag[2];
  const int G = cfg.G;
  const int group = blockIdx.x / G, c = blockIdx.x % G;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = 32;
  unsigned* ctr = ctrs + group;
  unsigned bar_count = 0;
  const float alpha = cfg.alpha;
  const int n_prob = tab.n_pairs * cfg.batch;

  for (int prob = group; prob < n_prob; prob += cfg.NG) {
    const int p = prob / cfg.batch, bi = prob % cfg.batch;
    // this problem's counts; the buffer keeps the capacity shape [m_cap + 1, n_cap + 1] (PairTable::slot)
    const int m = slot_count(tab.slot, bi, tab.n_views, tab.a[p], tab.m[p]);
    const int n = slot_count(tab.slot, bi, tab.n_views, tab.b[p], tab.n[p]);
    const int ld = tab.n[p] + 1;
    float* Zg = tab.scores[p] + (long long)bi * (tab.m[p] + 1) * ld;
    const int R = (m + G - 1) / G;
    const int r0 = min(m, c * R), r1 = min(m, r0 + R);
    const int nrows = r1 - r0;
    const int CS = (n + 1 + G - 1) / G;
    const int c0 = min(n + 1, c * CS), c1 = min(n + 1, c0 + CS);

    float* Ks = smem;                         // [R][n]   K~ of the inner block
    float* b_s = Ks + (size_t)R * n;          // [n+1]    column scalings b_j
    float* vt_s = b_s + (n + 1);              // [n+1]    absorbed column potentials v~_j
    float* kb_s = vt_s + (n + 1);             // [n+1]    exp(v~_j): dustbin row of K~ (u~_m = -alpha)
    float* ut_s = kb_s + (n + 1);             // [R]      absorbed row potentials u~_i
    float* a_s = ut_s + R;                    // [R+1]    row scalings a_i, a_s[R] = a_m (dustbin row)
    float* e_s = a_s + (R + 1);               // [R]      exp(alpha + u~_i): dustbin column of K~ / kb_n
    float* cpart = xch + (size_t)group * cfg.xch_stride;   // [G][n+1] partial column sums
    float* bx = cpart + (size_t)G * (n + 1);               // [n+1]    merged b

    const float norm = -logf((float)(m + n));
    const float mu = 1.0f / (float)(m + n), mu_bin = (float)n / (float)(m + n);
    const float nu = mu, nu_bin = (float)m / (float)(m + n);

    // ---- init: u~_i = -max(rowmax_i, alpha), v~ = 0, b = 1; K~ = exp(Z + u~) <= 1 ----
    for (int r = warp; r < nrows; r += NW) {
      const float* zr = Zg + (long long)(r0 + r) * ld;
      float mx = alpha;
      for (int j = lane; j < n; j += 32) mx = fmaxf(mx, zr[j]);
      mx = warp_max(mx);
      float* kr = Ks + (size_t)r * n;
      for (int j = lane; j < n; j += 32) kr[j] = __expf(zr[j] - mx);
      if (lane == 0) { ut_s[r] = -mx; e_s[r] = __expf(alpha - mx); }
    }
    for (int j = tid; j <= n; j += blockDim.x) { b_s[j] = 1.f; vt_s[j] = 0.f; kb_s[j] = 1.f; }
    __syncthreads();

    long long tacc[6] = {0, 0, 0, 0, 0, 0};
    for (int it = 0; it < cfg.iters; ++it) {
      long long t0 = clock64();
      // ---- row pass: a_i = mu / (sum_j K~_ij b_j + e_i kb_n b_n) ----
      const float bin_col = kb_s[n] * b_s[n];
      bool row_bad = false;
      for (int r = warp; r < nrows; r += NW) {
        const float* kr = Ks + (size_t)r * n;
        float s = 0.f;
        for (int j = lane; j < n; j += 32) s = fmaf(kr[j], b_s[j], s);
        s = warp_sum(s);
        const float a = mu / (s + e_s[r] * bin_col);
        if (lane == 0) a_s[r] = a;
        row_bad |= (a > ABSORB_HI) | (a < ABSORB_LO);
      }
      if (warp == NW - 1) {   // dustbin row (replicated in every CTA): a_m = mu_bin / sum_j kb_j b_j
        float s = 0.f;
        for (int j = lane; j <= n; j += 32) s = fmaf(kb_s[j], b_s[j], s);
        s = warp_sum(s);
        if (lane == 0) a_s[R] = mu_bin / s;
      }
      // row re-absorption (local decision): u~_i += log a_i, K~ row rescaled, a_i = 1
      const int any_row_bad = __syncthreads_or(row_bad ? 1 : 0);
      if (any_row_bad) {
        for (int r = warp; r < nrows; r += NW) {
          const float a = a_s[r];
          if (a > ABSORB_HI || a < ABSORB_LO) {
            float* kr = Ks + (size_t)r * n;
            for (int j = lane; j < n; j += 32) kr[j] *= a;
            __syncwarp();        // every lane has read a_s[r] before lane 0 resets it (racecheck)
            if (lane == 0) { ut_s[r] += logf(a); e_s[r] *= a; a_s[r] = 1.f; }
          }
        }
        __syncthreads();
      }
      { long long t1 = clock64(); tacc[0] += t1 - t0; t0 = t1; }
      // ---- column pass: partial c_j = sum_{own rows} K~_ij a_i ; dustbin column: kb_n sum e_i a_i ----
      for (int j = tid; j < n; j += blockDim.x) {
        float s = 0.f;
        int r = 0;
        // the row scalings are a broadcast read: fetch four per shared-memory instruction (same summation order)
        if ((reinterpret_cast<uintptr_t>(a_s) & 15) == 0) {
          for (; r + 4 <= nrows; r += 4) {
            const float4 a4 = *reinterpret_cast<const float4*>(a_s + r);
            s = fmaf(Ks[(size_t)r * n + j], a4.x, s);
            s = fmaf(Ks[(size_t)(r + 1) * n + j], a4.y, s);
            s = fmaf(Ks[(size_t)(r + 2) * n + j], a4.z, s);
            s = fmaf(Ks[(size_t)(r + 3) * n + j], a4.w, s);
          }
        }
        for (; r < nrows; ++r) s = fmaf(Ks[(size_t)r * n + j], a_s[r], s);
        __stcg(cpart + (size_t)c * (n + 1) + j, s);
      }
      if (warp == NW - 1) {
        float s = 0.f;
        for (int r = lane; r < nrows; r += 32) s = fmaf(e_s[r], a_s[r], s);
        s = warp_sum(s);
        if (lane == 0) __stcg(cpart + (size_t)c * (n + 1) + n, s * kb_s[n]);
      }
      { long long t1 = clock64(); tacc[1] += t1 - t0; t0 = t1; }
      bar_count += G;
      group_barrier(ctr, bar_count);
      { long long t1 = clock64(); tacc[2] += t1 - t0; t0 = t1; }
      // ---- merge this CTA's column slice in a fixed order: b_j = nu_j / (sum_g c_j^g + kb_j a_m) ----
      {
        const float am = a_s[R];
        for (int j = c0 + warp; j < c1; j += NW) {
          float s = 0.f;
          for (int g = lane; g < G; g += 32) s += __ldcg(cpart + (size_t)g * (n + 1) + j);
          s = warp_sum(s);
          if (lane == 0) __stcg(bx + j, (j < n ? nu : nu_bin) / (s + kb_s[j] * am));
        }
      }
      { long long t1 = clock64(); tacc[3] += t1 - t0; t0 = t1; }
      bar_count += G;
      group_barrier(ctr, bar_count);
      { long long t1 = clock64(); tacc[4] += t1 - t0; t0 = t1; }
      // ---- reload b; column re-absorption decided identically by every CTA of the group ----
      float bmx = 0.f, bmn = 3.0e38f;
      for (int j = tid; j <= n; j += blockDim.x) {
        const float bv = __ldcg(bx + j);
        b_s[j] = bv;
        bmx = fmaxf(bmx, bv);
        bmn = fminf(bmn, bv);
      }
      const int col_bad = __syncthreads_or((bmx > ABSORB_HI || bmn < ABSORB_LO) ? 1 : 0);
      if (col_bad) {
        // v~_j += log b_j, K~_ij *= b_j, kb_j *= b_j, b_j = 1   (all columns)
        for (int e = tid; e < nrows * n; e += blockDim.x) Ks[e] *= b_s[e % n];
        __syncthreads();
        for (int j = tid; j <= n; j += blockDim.x) {
          const float bv = b_s[j];
          vt_s[j] += logf(bv);
          kb_s[j] *= bv;
          b_s[j] = 1.f;
        }
        __syncthreads();
      }
    }

    if (cfg.timing && blockIdx.x == 0 && tid == 0 && prob == 0)
      for (int i = 0; i < 5; ++i) cfg.timing[i] = tacc[i];
    // ---- output: Z + u + v - norm with u = u~ + log a, v = v~ + log b ----
    for (int j = tid; j <= n; j += blockDim.x) vt_s[j] += logf(b_s[j]);
    __syncthreads();
    for (int r = warp; r < nrows; r += NW) {
      const float u = ut_s[r] + logf(a_s[r]);
      float* zr = Zg + (long long)(r0 + r) * ld;
      for (int j = lane; j < n; j += 32) zr[j] = zr[j] + u + vt_s[j] - norm;
      if (lane == 0) zr[n] = alpha + u + vt_s[n] - norm;
    }
    if (c == G - 1) {
      const float um = -alpha + logf(a_s[R]);     // u~_m = -alpha
      for (int j = tid; j <= n; j += blockDim.x) Zg[(long long)m * ld + j] = alpha + um + vt_s[j] - norm;
    }
    bar_count += G;
    group_barrier(ctr, bar_count);
  }
}

}  // namespace

long long* g_sink_timing = nullptr;
extern "C" void mvm_debug_set_sinkhorn_timing(long long* p) { g_sink_timing = p; }

// Production dispatch: problems of up to 1024 x 1024 run on one hardware cluster each (sinkhorn_cl.cu);
// larger ones (cfg4: 2048 keypoints, 16.8 MB per matrix) on the multi-CTA kernel below.
// variant: 0 = automatic (cluster kernel, two row groups per warp), 1 = force the multi-CTA kernel, 2 / 3 = cluster kernel
// with one row group per warp (1024 threads; 8 / 6 register rows), 4 = cluster kernel with two row groups per warp.
int launch_sinkhorn(const SinkhornTable& tab, int batch, float bin_score, int iters, float* ws,
                    cudaStream_t stream, int variant) {
  MVM_REQUIRE(tab.n_pairs >= 1 && tab.n_pairs <= MVM_MAX_PAIRS && batch >= 1 && iters >= 1);
  int mm = 0, mn = 0;
  for (int p = 0; p < tab.n_pairs; ++p) {
    mm = tab.m[p] > mm ? tab.m[p] : mm;
    mn = tab.n[p] > mn ? tab.n[p] : mn;
  }
  if (variant != 1) {
    const int C = sinkhorn_cluster_size(mm, mn);
    if (C > 0 && sinkhorn_cluster_max_active(C, mn) > 0)
      return launch_sinkhorn_cluster(tab, batch, bin_score, iters, C, stream, variant == 3 ? 6 : variant == 2 ? 8 : variant == 4 ? 16 : 0);
    MVM_REQUIRE(variant == 0);
  }
  return launch_sinkhorn_multicta(tab, batch, bin_score, iters, ws, stream);
}

int launch_sinkhorn_multicta(const SinkhornTable& tab, int batch, float bin_score, int iters, float* ws,
                             cudaStream_t stream) {
  MVM_REQUIRE(tab.n_pairs >= 1 && tab.n_pairs <= MVM_MAX_PAIRS && batch >= 1 && iters >= 1);
  MvmProfScope prof__(MVM_TAG_SINKHORN, stream);
  const int n_sm = mvm_dev_info().n_sm;
  const size_t max_smem = mvm_dev_info().max_smem;
  MVM_REQUIRE(n_sm <= 192);   // sinkhorn_ws_floats sizes the exchange buffer for at most 192 SMs
  mvm_once_per_device(MVM_ONCE_SINKHORN_EXP, [&] {
    cudaFuncSetAttribute(sinkhorn_exp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_smem);
  });
  int max_m = 0, max_n = 0;
  for (int p = 0; p < tab.n_pairs; ++p) {
    max_m = tab.m[p] > max_m ? tab.m[p] : max_m;
    max_n = tab.n[p] > max_n ? tab.n[p] : max_n;
  }
  const int n_prob = tab.n_pairs * batch;
  auto smem_need = [&](int G) {
    size_t need = 0;
    for (int p = 0; p < tab.n_pairs; ++p) {
      const size_t R = (tab.m[p] + G - 1) / G;
      const size_t b = (R * tab.n[p] + 3 * (size_t)(tab.n[p] + 1) + 3 * R + 1) * sizeof(float);
      need = b > need ? b : need;
    }
    return need;
  };
  int g_min = 1;
  while (g_min <= n_sm && smem_need(g_min) > max_smem - 2048) ++g_min;
  MVM_REQUIRE(g_min <= n_sm);
  // the iteration is barrier-latency bound, not compute bound: throughput = concurrent groups, so
  // use the smallest group that fits and as many groups as there are problems / SMs
  int NG = n_sm / g_min;
  if (NG > n_prob) NG = n_prob;
  int G = g_min;
  if (NG * (G + 1) <= n_sm && n_prob <= NG) G = n_sm / NG;   // few problems: spread over all SMs
  if (G > max_m) G = max_m;
  if (G < g_min) G = g_min;
  SinkCfg cfg;
  cfg.G = G; cfg.NG = NG; cfg.batch = batch; cfg.iters = iters; cfg.alpha = bin_score;
  cfg.xch_stride = (G + 1) * (max_n + 1);
  cfg.timing = g_sink_timing;
  unsigned* ctrs = reinterpret_cast<unsigned*>(ws);
  float* xch = ws + 256;
  cudaMemsetAsync(ctrs, 0, 256 * sizeof(float), stream);
  const size_t smem = smem_need(G);
  {
    // software group barriers inside: cooperative launch = co-residency guaranteed or an error, never a hang
    void* kargs[] = {(void*)const_cast<SinkhornTable*>(&tab), (void*)&cfg, (void*)&xch, (void*)&ctrs};
    cudaLaunchCooperativeKernel((const void*)sinkhorn_exp_kernel, dim3(G * NG), dim3(1024), kargs, smem, stream);
  }
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}
