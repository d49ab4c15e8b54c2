// log-domain optimal transport (Sinkhorn), reference: log_optimal_transport and
// log_sinkhorn_iterations, superglue.py:143-172 (SURVEY.md appendix A.3).
//
// v1 ("ref" kernel): one CTA per problem, coupling matrix resident in L2/HBM, warp-shuffle
// row LSE + column-strided column LSE.  Exact op order of the reference per element:
//   u_i = log_mu_i - LSE_j(Z_ij + v_j);  v_j = log_nu_j - LSE_i(Z_ij + u_i);  out = Z+u+v-norm.
#include "common.cuh"
#include "kernels.cuh"

namespace {

__global__ void __launch_bounds__(1024) sinkhorn_ref_kernel(SinkhornTable tab, int batch,
                                                            float alpha, int iters,
                                                            float* __restrict__ ws) {
  const int prob = blockIdx.x;
  const int p = prob / batch, bi = prob % batch;
  const int m = tab.m[p], n = tab.n[p];
  const int ld = n + 1;
  float* Z = tab.scores[p] + (long long)bi * (m + 1) * ld;
  float* u = ws + tab.ws_off[p] + (long long)bi * (m + n + 2);
  float* v = u + (m + 1);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;

  // dustbin augmentation (superglue.py:159-164)
  for (int i = tid; i < m; i += blockDim.x) Z[(long long)i * ld + n] = alpha;
  for (int j = tid; j <= n; j += blockDim.x) Z[(long long)m * ld + j] = alpha;
  for (int i = tid; i <= m; i += blockDim.x) u[i] = 0.f;
  for (int j = tid; j <= n; j += blockDim.x) v[j] = 0.f;
  const float norm = -logf((float)(m + n));
  const float log_mu_bin = logf((float)n) + norm;
  const float log_nu_bin = logf((float)m) + norm;
  __syncthreads();

  for (int it = 0; it < iters; ++it) {
    // rows: one warp per row
    for (int i = warp; i <= m; i += nwarps) {
      const float* zr = Z + (long long)i * ld;
      float mx = -INFINITY;
      for (int j = lane; j <= n; j += 32) mx = fmaxf(mx, zr[j] + v[j]);
      mx = warp_max(mx);
      float s = 0.f;
      for (int j = lane; j <= n; j += 32) s += expf(zr[j] + v[j] - mx);
      s = warp_sum(s);
      if (lane == 0) u[i] = (i < m ? norm : log_mu_bin) - (logf(s) + mx);
    }
    __syncthreads();
    // columns: one thread per column, coalesced across the warp
    for (int j = tid; j <= n; j += blockDim.x) {
      float mx = -INFINITY;
      for (int i = 0; i <= m; ++i) mx = fmaxf(mx, Z[(long long)i * ld + j] + u[i]);
      float s = 0.f;
      for (int i = 0; i <= m; ++i) s += expf(Z[(long long)i * ld + j] + u[i] - mx);
      v[j] = (j < n ? norm : log_nu_bin) - (logf(s) + mx);
    }
    __syncthreads();
  }
  for (long long e = tid; e < (long long)(m + 1) * ld; e += blockDim.x) {
    const int i = (int)(e / ld), j = (int)(e % ld);
    Z[e] = Z[e] + u[i] + v[j] - norm;
  }
}

}  // namespace

int launch_sinkhorn_ref(const SinkhornTable& tab, int batch, float bin_score, int iters,
                        float* ws, cudaStream_t stream) {
  MVM_REQUIRE(tab.n_pairs >= 1 && tab.n_pairs <= MVM_MAX_PAIRS && batch >= 1 && iters >= 1);
  sinkhorn_ref_kernel<<<tab.n_pairs * batch, 1024, 0, stream>>>(tab, batch, bin_score, iters, ws);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

// =======================================================================================
// v2 (log domain, kept as the second on-device cross-check): shared-memory-resident Sinkhorn.  A group of G co-resident CTAs owns one problem; CTA c
// keeps rows [c*R, (c+1)*R) of the inner m x n score block in shared memory for all
// iterations, so the coupling matrix is read from HBM/L2 exactly once and written once
// (the reference makes 200 full passes, SURVEY.md §8 a10).  Per iteration:
//   row pass   (local)  u_i = log_mu_i - LSE_j(Z_ij + v_j)            warp per row, shuffles
//   col pass   (local)  per-column partial (max, sum exp) over the CTA's rows
//   exchange            partials -> global (L2), group barrier, CTA c merges the partials of
//                       its column slice in fixed order (deterministic), writes v slice,
//                       group barrier, every CTA reloads v.
// Dustbin row/column are the constant alpha (superglue.py:159-164): they are never stored,
// their LSE terms are added analytically.
// =======================================================================================
namespace {

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void group_barrier(unsigned* ctr, unsigned target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(ctr, 1u);
    while (ld_acquire_u32(ctr) < target) { __nanosleep(20); }
    __threadfence();
  }
  __syncthreads();
}

struct SinkCfg {
  int G;        // CTAs per group
  int NG;       // groups
  int batch;
  int iters;
  float alpha;
  int xch_stride;   // floats per group in the exchange buffer
};

__global__ void __launch_bounds__(1024, 1) sinkhorn_smem_kernel(PairTable tab, SinkCfg cfg,
                                                                float* __restrict__ xch,
                                                                unsigned* __restrict__ ctrs) {
  extern __shared__ float smem[];
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
    const int m = tab.m[p], n = tab.n[p];
    const int ld = n + 1;
    float* Zg = tab.scores[p] + (long long)bi * (m + 1) * ld;
    const int R = (m + G - 1) / G;
    const int r0 = min(m, c * R), r1 = min(m, r0 + R);
    const int nrows = r1 - r0;
    const int CS = (n + 1 + G - 1) / G;                 // column slice width
    const int c0 = min(n + 1, c * CS), c1 = min(n + 1, c0 + CS);

    float* Zs = smem;                       // [R][n]
    float* v_s = Zs + (size_t)R * n;        // [n+1]
    float* u_s = v_s + (n + 1);             // [R] own rows, u_s[R] = u_m (dustbin row)
    // exchange: pm[G][n+1], ps[G][n+1], vx[n+1]
    float* pm_g = xch + (size_t)group * cfg.xch_stride;
    float* ps_g = pm_g + (size_t)G * (n + 1);
    float* vx_g = ps_g + (size_t)G * (n + 1);

    const float norm = -logf((float)(m + n));
    const float log_mu_bin = logf((float)n) + norm;
    const float log_nu_bin = logf((float)m) + norm;

    // load own rows of the inner block
    for (int e = tid; e < nrows * n; e += blockDim.x) {
      const int r = e / n, j = e % n;
      Zs[(size_t)r * n + j] = Zg[(long long)(r0 + r) * ld + j];
    }
    for (int j = tid; j <= n; j += blockDim.x) v_s[j] = 0.f;
    __syncthreads();

    for (int it = 0; it < cfg.iters; ++it) {
      // ---- row pass: u for own rows (warps 0..), dustbin row u_m (last warp) ----
      for (int r = warp; r < nrows; r += NW) {
        const float* zr = Zs + (size_t)r * n;
        float mx = alpha + v_s[n];
        for (int j = lane; j < n; j += 32) mx = fmaxf(mx, zr[j] + v_s[j]);
        mx = warp_max(mx);
        float s = 0.f;
        for (int j = lane; j < n; j += 32) s += expf(zr[j] + v_s[j] - mx);
        s = warp_sum(s);
        s += expf(alpha + v_s[n] - mx);
        if (lane == 0) u_s[r] = norm - (logf(s) + mx);
      }
      if (warp == NW - 1) {
        float mx = -INFINITY;
        for (int j = lane; j <= n; j += 32) mx = fmaxf(mx, alpha + v_s[j]);
        mx = warp_max(mx);
        float s = 0.f;
        for (int j = lane; j <= n; j += 32) s += expf(alpha + v_s[j] - mx);
        s = warp_sum(s);
        if (lane == 0) u_s[R] = log_mu_bin - (logf(s) + mx);
      }
      __syncthreads();
      // ---- column pass: partial (max, sumexp) over own rows ----
      for (int j = tid; j < n; j += blockDim.x) {
        float mx = -INFINITY;
        for (int r = 0; r < nrows; ++r) mx = fmaxf(mx, Zs[(size_t)r * n + j] + u_s[r]);
        float s = 0.f;
        for (int r = 0; r < nrows; ++r) s += expf(Zs[(size_t)r * n + j] + u_s[r] - mx);
        __stcg(pm_g + (size_t)c * (n + 1) + j, mx);
        __stcg(ps_g + (size_t)c * (n + 1) + j, s);
      }
      if (warp == NW - 1) {   // dustbin column: elements alpha + u_i over own rows
        float mx = -INFINITY;
        for (int r = lane; r < nrows; r += 32) mx = fmaxf(mx, alpha + u_s[r]);
        mx = warp_max(mx);
        float s = 0.f;
        for (int r = lane; r < nrows; r += 32) s += expf(alpha + u_s[r] - mx);
        s = warp_sum(s);
        if (lane == 0) {
          __stcg(pm_g + (size_t)c * (n + 1) + n, mx);
          __stcg(ps_g + (size_t)c * (n + 1) + n, nrows > 0 ? s : 0.f);
        }
      }
      bar_count += G;
      group_barrier(ctr, bar_count);
      // ---- merge the partials of this CTA's column slice (warp per column) ----
      const float d = alpha + u_s[R];      // dustbin-row term, identical in every CTA
      for (int j = c0 + warp; j < c1; j += NW) {
        float mx = d;
        for (int g = lane; g < G; g += 32) mx = fmaxf(mx, __ldcg(pm_g + (size_t)g * (n + 1) + j));
        mx = warp_max(mx);
        float s = 0.f;
        for (int g = lane; g < G; g += 32) {
          const float pmv = __ldcg(pm_g + (size_t)g * (n + 1) + j);
          const float psv = __ldcg(ps_g + (size_t)g * (n + 1) + j);
          s += psv * expf(pmv - mx);       // ps == 0 (empty CTA) -> contributes 0
        }
        s = warp_sum(s);
        s += expf(d - mx);
        if (lane == 0) __stcg(vx_g + j, (j < n ? norm : log_nu_bin) - (logf(s) + mx));
      }
      bar_count += G;
      group_barrier(ctr, bar_count);
      for (int j = tid; j <= n; j += blockDim.x) v_s[j] = __ldcg(vx_g + j);
      __syncthreads();
    }

    // ---- output: Z + u + v - norm (superglue.py:148,170) ----
    for (int e = tid; e < nrows * ld; e += blockDim.x) {
      const int r = e / ld, j = e % ld;
      const float z = j < n ? Zs[(size_t)r * n + j] : alpha;
      Zg[(long long)(r0 + r) * ld + j] = z + u_s[r] + v_s[j] - norm;
    }
    if (c == G - 1)
      for (int j = tid; j <= n; j += blockDim.x)
        Zg[(long long)m * ld + j] = alpha + u_s[R] + v_s[j] - norm;
    // the next problem reuses the exchange buffers: make sure every CTA of the group is done
    // reading vx before anyone overwrites it
    bar_count += G;
    group_barrier(ctr, bar_count);
  }
}

}  // namespace

int launch_sinkhorn_log(const SinkhornTable& tab, int batch, float bin_score, int iters, float* ws,
                        cudaStream_t stream) {
  MvmProfScope prof__(MVM_TAG_SINKHORN, stream);
  MVM_REQUIRE(tab.n_pairs >= 1 && tab.n_pairs <= MVM_MAX_PAIRS && batch >= 1 && iters >= 1);
  const int n_sm = mvm_dev_info().n_sm;
  const size_t max_smem = mvm_dev_info().max_smem;
  mvm_once_per_device(MVM_ONCE_SINKHORN_LOG, [&] {
    cudaFuncSetAttribute(sinkhorn_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_smem);
  });
  int max_m = 0, max_n = 0;
  size_t max_mn = 0;
  for (int p = 0; p < tab.n_pairs; ++p) {
    max_m = tab.m[p] > max_m ? tab.m[p] : max_m;
    max_n = tab.n[p] > max_n ? tab.n[p] : max_n;
    const size_t mn = (size_t)tab.m[p] * tab.n[p];
    max_mn = mn > max_mn ? mn : max_mn;
  }
  const int n_prob = tab.n_pairs * batch;
  // smallest group that fits the largest problem in shared memory
  auto smem_need = [&](int G) {
    size_t need = 0;
    for (int p = 0; p < tab.n_pairs; ++p) {
      const size_t R = (tab.m[p] + G - 1) / G;
      const size_t b = (R * tab.n[p] + (tab.n[p] + 1) + (R + 1)) * sizeof(float);
      need = b > need ? b : need;
    }
    return need;
  };
  int g_min = 1;
  while (g_min <= n_sm && smem_need(g_min) > max_smem - 1024) ++g_min;
  MVM_REQUIRE(g_min <= n_sm && n_sm <= 192);
  int NG = n_sm / g_min;
  if (NG > n_prob) NG = n_prob;
  const int rounds = (n_prob + NG - 1) / NG;
  NG = (n_prob + rounds - 1) / rounds;
  int G = n_sm / NG;
  if (G > max_m) G = max_m;        // at least one row per CTA
  if (G < g_min) G = g_min;
  SinkCfg cfg;
  cfg.G = G; cfg.NG = NG; cfg.batch = batch; cfg.iters = iters; cfg.alpha = bin_score;
  cfg.xch_stride = (2 * G + 1) * (max_n + 1);
  // ws layout: [NG] counters (as 64 floats) | exchange
  unsigned* ctrs = reinterpret_cast<unsigned*>(ws);
  float* xch = ws + 256;
  cudaMemsetAsync(ctrs, 0, 256 * sizeof(float), stream);
  const size_t smem = smem_need(G);
  {
    // software group barriers inside: cooperative launch = co-residency guaranteed or an error, never a hang
    void* kargs[] = {(void*)const_cast<SinkhornTable*>(&tab), (void*)&cfg, (void*)&xch, (void*)&ctrs};
    cudaLaunchCooperativeKernel((const void*)sinkhorn_smem_kernel, dim3(G * NG), dim3(1024), kargs, smem, stream);
  }
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

size_t sinkhorn_ws_floats(int n_pairs, int batch, int n_pad) {
  // counters + worst-case exchange ((2G+1)(n+1) per group, G*NG <= the SM count) and the v1 (u,v) scratch
  // (sized for up to 192 SMs; the launchers check the real SM count against this bound)
  const size_t xch = 256 + (size_t)(2 * 192 + 192) * (n_pad + 1) * 2;   // log-domain partials / 8-byte LL words
  const size_t uv = (size_t)n_pairs * batch * (2 * (size_t)n_pad + 2);
  return xch > uv ? xch : uv;
}
