// Production Sinkhorn for problems up to 1024 x 1024: one thread-block CLUSTER per assignment problem.
//
// Same fixed point and the same 100 iterations as log_optimal_transport / log_sinkhorn_iterations
// (superglue.py:143-172) in the stabilised scaling domain of sinkhorn_exp.cu:
//
//   K~_ij = exp(Z_ij + u~_i + v~_j)        evaluated once (and on the rare re-absorptions)
//   row:  a_i = mu_i / sum_j K~_ij b_j     <=>  u_i = log_mu_i - LSE_j(Z_ij + v_j),  u = u~ + log a
//   col:  b_j = nu_j / sum_i K~_ij a_i     <=>  v_j = log_nu_j - LSE_i(Z_ij + u_i),  v = v~ + log b
//
// What is different from sinkhorn_exp.cu (software group barrier through L2, 11 us per iteration):
//   * the C CTAs of a problem are a hardware cluster (C = 16 for 513..1024 rows: non-portable size,
//     gang-scheduled by the hardware, so there is no co-residency assumption and nothing to deadlock);
//   * CTA c keeps rows [c*R, (c+1)*R), R <= 64, of K~ ON CHIP: every warp owns a 16 x 128 tile, RR rows of
//     it in REGISTERS (float4 per lane) and 16 - RR rows in shared memory, so an iteration streams only
//     (16-RR)/16 of the slab from shared memory, with 128-bit conflict-free accesses;
//   * row sums: transposed 16-value warp reduction (16 shuffles) + 8 strip partials per row in shared memory;
//     column sums: 4 row-group partials per column in shared memory, then the CTA's partial of column j is
//     PUSHED into the shared memory of the CTA that owns column j (st.shared::cluster), one
//     barrier.cluster, the owner adds the C partials in rank order (deterministic), divides, and pushes
//     b_j into every CTA's copy of b, second barrier.cluster.  4 KB of DSMEM traffic per CTA and iteration.
//   * dustbin row / column are rank-1 and never stored (as before).
// The raw scores stay in the output buffer (L2) until the final pass rewrites them as Z + u + v - norm.
// TMA is not applicable to the staging: the reference's [m+1, n+1] fp32 layout has a 4*(n+1)-byte row pitch,
// which is not a multiple of 16 bytes for n = 1024 (tensor maps and bulk copies need 16-byte pitch/alignment).
#include "common.cuh"
#include "kernels.cuh"

extern long long* g_sink_timing;   // sinkhorn_exp.cu (mvm_debug_set_sinkhorn_timing)

namespace {

constexpr float ABSORB_HI = 2980.958f;     // e^8
constexpr float ABSORB_LO = 3.3546263e-4f; // e^-8
constexpr int CL_ROWS = 64;                // rows of K~ per CTA
constexpr int CL_MAXN = 1024;              // columns
constexpr int CL_CRECV = CL_MAXN + 4 + 16; // floats of the crecv region: C * CS <= 1040 for every C
constexpr int CL_MERGE_COLS = 3;           // columns of its slice one thread of the owner merges: 3 x 512 >= 1025 (C = 1)

__device__ __forceinline__ unsigned cluster_ctarank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned mapa_u32(unsigned saddr, unsigned rank) {
  unsigned r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank));
  return r;
}

// remote shared-memory store that reports its 4 bytes to an mbarrier of the destination CTA
__device__ __forceinline__ void st_async_f32(unsigned addr, float v, unsigned mbar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(addr),
               "r"(__float_as_uint(v)), "r"(mbar)
               : "memory");
}
__device__ __forceinline__ void mbar_init(unsigned mbar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned mbar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned mbar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(mbar),
      "r"(parity)
      : "memory");
}

struct OpSum { __device__ __forceinline__ float operator()(float a, float b) const { return a + b; } };
struct OpMax { __device__ __forceinline__ float operator()(float a, float b) const { return fmaxf(a, b); } };

// Transposed warp reduction: at the level with lane distance S, value k of lane l (k < H) becomes the sum of values
// k and k + H over the lane pair (l, l ^ S), the lane with bit S clear keeping the lower half.  The levels
// S = 16, 8, ... run while H >= 1.  Template recursion with a compile-time H at every level: a loop over the levels
// with a runtime-halving bound is not unrolled by nvcc, and the partials then live in a local-memory array.
template <int S, int H, int N, class Op>
__device__ __forceinline__ void xreduce(float (&p)[N], int lane, Op op) {
  if constexpr (H >= 1) {
    const bool hi = lane & S;
#pragma unroll
    for (int k = 0; k < H; ++k) {
      const float send = hi ? p[k] : p[k + H], keep = hi ? p[k + H] : p[k];
      p[k] = op(keep, __shfl_xor_sync(0xffffffffu, send, S));
    }
    xreduce<S / 2, H / 2>(p, lane, op);
  }
}

// 8 values per lane, reduced over the 32 lanes in 9 shuffles; afterwards every lane holds the total of value index
// row8(lane) (the four lanes that differ in bits 0-1 hold the same value).
template <class Op>
__device__ __forceinline__ float reduce8(float (&p)[8], int lane, Op op) {
  xreduce<16, 4>(p, lane, op);
  p[0] = op(p[0], __shfl_xor_sync(0xffffffffu, p[0], 2));
  return op(p[0], __shfl_xor_sync(0xffffffffu, p[0], 1));
}
__device__ __forceinline__ int row8(int lane) { return ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1); }

// 16 values per lane, reduced over the 32 lanes in 16 shuffles; afterwards every lane holds the total of
// value index row16(lane) (lanes 2k and 2k+1 hold the same value).
template <class Op>
__device__ __forceinline__ float reduce16(float (&p)[16], int lane, Op op) {
  xreduce<16, 8>(p, lane, op);
  return op(p[0], __shfl_xor_sync(0xffffffffu, p[0], 1));
}
__device__ __forceinline__ int row16(int lane) {
  return ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
}

// b_j of the thread's four columns; 1 beyond the last column (K~ is 0 there)
__device__ __forceinline__ float4 load_b4(const float* b_s, int col0, int n) {
  float4 b4 = *reinterpret_cast<const float4*>(b_s + col0);
  if (col0 + 0 >= n) b4.x = 1.f;
  if (col0 + 1 >= n) b4.y = 1.f;
  if (col0 + 2 >= n) b4.z = 1.f;
  if (col0 + 3 >= n) b4.w = 1.f;
  return b4;
}

struct SinkClCfg {
  int C, batch, iters;
  float alpha;
  long long* timing;   // optional [6] cycle counters of thread 0 of CTA 0 (TIMING instance only), or null
};

// shared-memory carve (floats): fixed-size vectors at compile-time offsets (no registers spent on pointers),
// the K~ rows last with the per-problem row stride LD = round_up(n, 128); identical in every CTA of a cluster
constexpr int CL_VEC = CL_MAXN + 4;
constexpr int OFF_B = 0;                              // [n+1]  column scalings b_j
constexpr int OFF_KB = OFF_B + CL_VEC;                // [n+1]  exp(v~_j): dustbin row of K~ (u~_m = -alpha)
constexpr int OFF_VT = OFF_KB + CL_VEC;               // [n+1]  absorbed column potentials v~_j
constexpr int OFF_COLPART = OFF_VT + CL_VEC;          // [4][1024] column partials of the 4 row groups
constexpr int OFF_CRECV = OFF_COLPART + 4 * CL_MAXN;  // [C][CS] partials pushed by the peers for my column slice
constexpr int OFF_ROWPART = OFF_CRECV + CL_CRECV;     // [8][64] row partials of the 8 column strips
constexpr int OFF_A = OFF_ROWPART + 8 * CL_ROWS;      // [64] row scalings a_i, a[64] = dustbin row
constexpr int OFF_UT = OFF_A + CL_ROWS + 4;           // [64] absorbed row potentials u~_i
constexpr int OFF_E = OFF_UT + CL_ROWS;               // [64] exp(alpha + u~_i): dustbin column of K~ / kb_n
constexpr int OFF_EA = OFF_E + CL_ROWS;               // [64] e_i a_i (dustbin column terms; 0 beyond the CTA's rows)
constexpr int OFF_AW = OFF_EA + CL_ROWS;              // [32][16] per-warp copy of the row scalings of its row group
constexpr int OFF_DUST = OFF_AW + 32 * 16;            // [8] strip partials of the dustbin row sum
constexpr int OFF_MBAR = OFF_DUST + 8;                // 2 x 8-byte mbarriers (A: partials landed, B: b landed)
constexpr int OFF_KS = OFF_MBAR + 4;                  // [4][16-RR][1024]  (compile-time row stride: immediate offsets)
static_assert(OFF_KS % 4 == 0 && OFF_A % 4 == 0 && OFF_COLPART % 4 == 0 && OFF_AW % 4 == 0 && OFF_KB % 4 == 0,
              "16-byte alignment of the float4 regions");
static_assert(OFF_MBAR % 2 == 0, "8-byte alignment of the mbarriers");
inline size_t cl_smem_bytes(int n, int RS) { (void)n; return (size_t)(OFF_KS + 4 * RS * CL_MAXN) * sizeof(float); }

// RG = 16-row groups per warp: 1 (1024 threads, 64 registers each) or 2 (512 threads, 128 registers each: the same
// K~ tile per SM, but the per-warp overhead of an iteration -- operand addresses the 64-register build keeps
// rematerialising, b_j loads and masks, absorb checks, the a_i pass -- is paid once per 32 rows instead of once per
// 16; the phase trace of r02 showed both passes issue-bound with 22 % of the instructions being the FMAs)
template <int RR, int RG, bool TIMING>
__global__ void __launch_bounds__(1024 / RG, 1) sinkhorn_cl_kernel(PairTable tab, SinkClCfg cfg) {
  extern __shared__ __align__(16) float smem[];
  constexpr int RS = 16 - RR;
  constexpr int NW = 32 / RG;                       // warps per CTA
  constexpr int NT = 32 * NW;                       // threads per CTA
  const int C = cfg.C;
  const unsigned c = cluster_ctarank();
  const int prob = blockIdx.x / C;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rp = warp >> 3, cw = warp & 7;         // row groups rp * RG ... rp * RG + RG - 1, column strip cw
#define RGI(g) (rp * RG + (g))
  const float alpha = cfg.alpha;

  const int p = prob / cfg.batch, bi = prob % cfg.batch;
  // this problem's counts; the buffer keeps the capacity shape [m_cap + 1, n_cap + 1] (PairTable::slot)
  const int m = slot_count(tab.slot, bi, tab.n_views, tab.a[p], tab.m[p]);
  const int n = slot_count(tab.slot, bi, tab.n_views, tab.b[p], tab.n[p]);
  const int ld = tab.n[p] + 1;
  float* Zg = tab.scores[p] + (long long)bi * (tab.m[p] + 1) * ld;
  const int R = (m + C - 1) / C;
  const int r0 = min(m, (int)c * R), nrows = min(m, r0 + R) - r0;
  constexpr int LD = CL_MAXN;
  const int CS = (n + 1 + C - 1) / C;
  const bool active = cw * 128 < n;
  const int col0 = cw * 128 + lane * 4;

  float* const b_s = smem + OFF_B;
  float* const kb_s = smem + OFF_KB;
  float* const vt_s = smem + OFF_VT;
  float* const colpart = smem + OFF_COLPART;
  float* const crecv = smem + OFF_CRECV;
  float* const rowpart = smem + OFF_ROWPART;
  float* const a_s = smem + OFF_A;
  float* const ut_s = smem + OFF_UT;
  float* const e_s = smem + OFF_E;
  float* const ea_s = smem + OFF_EA;
  float* const aw_s = smem + OFF_AW;
  float* const dust_s = smem + OFF_DUST;
  float* const ksm = smem + OFF_KS + (size_t)(rp * RG) * RS * LD + col0;   // this thread's shared-memory rows (i >= RR)

  const float mu = 1.0f / (float)(m + n), mu_bin = (float)n / (float)(m + n);
  const float nu = mu, nu_bin = (float)m / (float)(m + n);
  const float norm = -logf((float)(m + n));

  float4 kreg[RG][RR];
#define K_GET(g, i) ((i) < RR ? kreg[g][(i) < RR ? (i) : 0] : *reinterpret_cast<const float4*>(ksm + ((g) * RS + (i) - RR) * LD))
#define K_PUT(g, i, v)                                                           \
  do {                                                                           \
    if ((i) < RR) kreg[g][(i) < RR ? (i) : 0] = (v);                             \
    else *reinterpret_cast<float4*>(ksm + ((g) * RS + (i) - RR) * LD) = (v);     \
  } while (0)

  // ---- init: u~_i = -max(rowmax_i, alpha), v~ = 0, b = 1; K~ = exp(Z + u~) <= 1 ----
#pragma unroll
  for (int g = 0; g < RG; ++g) {
    const int rg = RGI(g);
    float part[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int row = rg * 16 + i;
      float mx = -3.0e38f;
      if (active && row < nrows) {
        const float* zr = Zg + (long long)(r0 + row) * ld + col0;
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (col0 + k < n) mx = fmaxf(mx, zr[k]);
      }
      part[i] = mx;
    }
    const float v = reduce16(part, lane, OpMax());
    if (!(lane & 1)) rowpart[cw * CL_ROWS + rg * 16 + row16(lane)] = v;
  }
  for (int j = tid; j < CL_VEC; j += blockDim.x) { b_s[j] = 1.f; vt_s[j] = 0.f; kb_s[j] = 1.f; }
  __syncthreads();
  if (tid < CL_ROWS) {
    float mx = alpha;
#pragma unroll
    for (int s = 0; s < 8; ++s) mx = fmaxf(mx, rowpart[s * CL_ROWS + tid]);
    ut_s[tid] = -mx;
    e_s[tid] = tid < nrows ? __expf(alpha - mx) : 0.f;
    a_s[tid] = tid < nrows ? 1.f : 0.f;
    ea_s[tid] = 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int g = 0; g < RG; ++g)
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int row = RGI(g) * 16 + i;
    float4 k4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (active && row < nrows) {
      const float* zr = Zg + (long long)(r0 + row) * ld + col0;
      const float ut = ut_s[row];
      if (col0 + 0 < n) k4.x = __expf(zr[0] + ut);
      if (col0 + 1 < n) k4.y = __expf(zr[1] + ut);
      if (col0 + 2 < n) k4.z = __expf(zr[2] + ut);
      if (col0 + 3 < n) k4.w = __expf(zr[3] + ut);
    }
    if (active) K_PUT(g, i, k4);
  }
  // ---- exchange machinery: two transaction mbarriers per CTA.  mbar A completes when the C partials of every
  // column this CTA owns have landed in crecv; mbar B when all n+1 merged b_j have landed in b_s.  The values
  // travel by st.async (remote shared-memory store that reports its bytes to the destination's mbarrier), so an
  // iteration has no cluster-wide barrier: a CTA only ever waits for the data it needs. ----
  const unsigned mbarA = smem_u32(smem + OFF_MBAR), mbarB = mbarA + 8;
  const int owned = max(0, min(n + 1, ((int)c + 1) * CS) - (int)c * CS);
  if (tid == 0) {
    mbar_init(mbarA, 1);
    mbar_init(mbarB, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (tid < 8) dust_s[tid] = 0.f;
  // the row-max scratch of the strips beyond the last column becomes the (never written) zero partial of those strips
  for (int j = tid; j < 8 * CL_ROWS; j += blockDim.x)
    if ((j / CL_ROWS) * 128 >= n) rowpart[j] = 0.f;
  // peers' shared memory is about to be written: every CTA of the cluster must have started
  cluster_sync_all();

  const unsigned crecv_addr = smem_u32(crecv), b_addr = smem_u32(b_s);
  // column j = tid of this CTA's partial sums goes to slot (c, j - owner CS) of its owner (n <= 1024: one column per
  // thread; the dustbin column n is pushed by warp 31)
  unsigned push_addr[RG], push_mbar[RG];
#pragma unroll
  for (int q = 0; q < RG; ++q) {
    const int j = tid + q * (1024 / RG);
    push_addr[q] = 0; push_mbar[q] = 0;
    if (j < n) {
      const int owner = j / CS, slot = j - owner * CS;
      push_addr[q] = mapa_u32(crecv_addr + (unsigned)(((int)c * CS + slot) * 4), (unsigned)owner);
      push_mbar[q] = mapa_u32(mbarA, (unsigned)owner);
    }
  }
  unsigned tacc[6] = {0u, 0u, 0u, 0u, 0u, 0u};
  unsigned tprev = 0;
  if (TIMING) tprev = (unsigned)clock();
#define T_MARK(k)                                   \
  do {                                              \
    if (TIMING) {                                   \
      const unsigned tn__ = (unsigned)clock();      \
      tacc[k] += tn__ - tprev;                      \
      tprev = tn__;                                 \
    }                                               \
  } while (0)

  for (int it = 0; it < cfg.iters; ++it) {
    const unsigned ph = (unsigned)it & 1u;
    if (tid == 0) {   // arm this iteration's phase (transactions that arrive earlier are accounted for)
      mbar_expect_tx(mbarA, (unsigned)(owned * C * 4));
      mbar_expect_tx(mbarB, (unsigned)((n + 1) * 4));
    }
    // ---- row pass: partial sums of sum_j K~_ij b_j over this warp's 128-column strip ----
    const float bin_col = kb_s[n] * b_s[n];
    int cbad = 0;
    if (active) {
      const float4 b4 = load_b4(b_s, col0, n);
      // column re-absorption is decided on the freshly merged b (identical in every CTA of the cluster)
      cbad = (fmaxf(fmaxf(b4.x, b4.y), fmaxf(b4.z, b4.w)) > ABSORB_HI) | (fminf(fminf(b4.x, b4.y), fminf(b4.z, b4.w)) < ABSORB_LO);
      if constexpr (RG == 2) {
        // all 32 row partials of the warp in one transposed reduction (levels 16, 8, 4, 2, 1): lane l ends up with
        // the strip total of row l.  The first level pairs row i of the two row groups, so it runs as soon as both
        // dot products exist: 16 partials live instead of 32, next to the 64 K~ registers
        float part[16];
        const bool hi16 = lane & 16;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const float4 k0 = K_GET(0, i), k1 = K_GET(1, i);
          const float p0 = fmaf(k0.w, b4.w, fmaf(k0.z, b4.z, fmaf(k0.y, b4.y, k0.x * b4.x)));
          const float p1 = fmaf(k1.w, b4.w, fmaf(k1.z, b4.z, fmaf(k1.y, b4.y, k1.x * b4.x)));
          part[i] = (hi16 ? p1 : p0) + __shfl_xor_sync(0xffffffffu, hi16 ? p0 : p1, 16);
        }
        xreduce<8, 8>(part, lane, OpSum());
        rowpart[cw * CL_ROWS + rp * 32 + lane] = part[0];
      } else {
#pragma unroll
      for (int h8 = 0; h8 < 2; ++h8) {           // groups of 8 rows: 8 partials live instead of 16
        float part[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 k = K_GET(0, h8 * 8 + i);
          part[i] = fmaf(k.w, b4.w, fmaf(k.z, b4.z, fmaf(k.y, b4.y, k.x * b4.x)));
        }
        const float v = reduce8(part, lane, OpSum());
        if (!(lane & 3)) rowpart[cw * CL_ROWS + RGI(0) * 16 + h8 * 8 + row8(lane)] = v;
      }
      }
      if (rp == 0) {   // dustbin row (replicated in every CTA): strip partial of sum_{j<n} kb_j b_j
        const float4 kb4 = *reinterpret_cast<const float4*>(kb_s + col0);
        float d = 0.f;
        if (col0 + 0 < n) d = kb4.x * b4.x;
        if (col0 + 1 < n) d = fmaf(kb4.y, b4.y, d);
        if (col0 + 2 < n) d = fmaf(kb4.z, b4.z, d);
        if (col0 + 3 < n) d = fmaf(kb4.w, b4.w, d);
        d = warp_sum(d);
        if (lane == 0) dust_s[cw] = d;
      }
    }
    if (tid == 0) {
      const float bn = b_s[n];
      cbad |= (bn > ABSORB_HI) | (bn < ABSORB_LO);
    }
    T_MARK(0);
    if (__syncthreads_or(cbad)) {
      // v~_j += log b_j, K~_ij *= b_j, kb_j *= b_j, b_j = 1 (all columns); the row sums above are unchanged
      if (active) {
        const float4 b4 = load_b4(b_s, col0, n);
#pragma unroll
        for (int g = 0; g < RG; ++g)
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          float4 k = K_GET(g, i);
          k.x *= b4.x; k.y *= b4.y; k.z *= b4.z; k.w *= b4.w;
          K_PUT(g, i, k);
        }
      }
      for (int j = tid; j <= n; j += blockDim.x) {
        const float bv = b_s[j];
        vt_s[j] += logf(bv);
        kb_s[j] *= bv;
      }
      __syncthreads();     // every b_s read of this iteration is done (bin_col, dustbin row, b4)
      for (int j = tid; j <= n; j += blockDim.x) b_s[j] = 1.f;
    }
    T_MARK(1);
    if (tid == 0) {      // a_m = mu_bin / sum_{j<=n} kb_j b_j  (strip partials in a fixed order + the corner term)
      float sd = 0.f;
#pragma unroll
      for (int q = 0; q < 8; ++q) sd += dust_s[q];
      a_s[CL_ROWS] = mu_bin / (sd + bin_col);
    }
    // ---- every warp: a_i = mu / (sum_j K~_ij b_j + e_i kb_n b_n) for the 16 rows of its row group ----
    float a_abs = 1.f;         // scaling absorbed into u~ this iteration (book-keeping by the strip-0 warp)
    if (active) {
      // RG = 1: lanes 16-31 mirror lanes 0-15; RG = 2: lanes 0-15 take the warp's first row group, 16-31 the second
      const int rl = lane & 15, row = RGI(RG == 2 ? (lane >> 4) : 0) * 16 + rl;
      float a_mine = 0.f, ea = 0.f;
      {
        float s = 0.f;
#pragma unroll
        for (int q = 0; q < 8; ++q) s += rowpart[q * CL_ROWS + row];      // strips beyond n hold 0
        const float e = e_s[row];
        if (row < nrows) {
          a_mine = mu / (s + e * bin_col);
          ea = e * a_mine;
        }
      }
      const bool bad = row < nrows && (a_mine > ABSORB_HI || a_mine < ABSORB_LO);
      if (__any_sync(0xffffffffu, bad)) {
        // row re-absorption (every strip warp of the row group takes the same decision): K~ row *= a_i, a_i = 1
#pragma unroll
        for (int g = 0; g < RG; ++g)
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const float ai = __shfl_sync(0xffffffffu, a_mine, g * 16 + i);
          if (__shfl_sync(0xffffffffu, (int)bad, g * 16 + i)) {
            float4 k = K_GET(g, i);
            k.x *= ai; k.y *= ai; k.z *= ai; k.w *= ai;
            K_PUT(g, i, k);
          }
        }
        if (bad) { a_abs = a_mine; a_mine = 1.f; }
      }
      float* aw = aw_s + warp * (16 * RG);
      if (lane < 16 * RG) {
        aw[lane] = a_mine;
        if (cw == 0) { a_s[row] = a_mine; ea_s[row] = ea; }
      }
      __syncwarp();
      // ---- column pass: partial c_j over this warp's 16 RG rows ----
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int g = 0; g < RG; ++g)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 a4 = *reinterpret_cast<const float4*>(aw + g * 16 + q * 4);
        const float av[4] = {a4.x, a4.y, a4.z, a4.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float4 k = K_GET(g, q * 4 + t);
          acc.x = fmaf(k.x, av[t], acc.x);
          acc.y = fmaf(k.y, av[t], acc.y);
          acc.z = fmaf(k.z, av[t], acc.z);
          acc.w = fmaf(k.w, av[t], acc.w);
        }
      }
      *reinterpret_cast<float4*>(colpart + rp * CL_MAXN + col0) = acc;
    }
    T_MARK(2);
    __syncthreads();
    if (cw == 0 && lane < 16 * RG && a_abs != 1.f) {     // deferred: nobody reads e_s / ut_s before the next barrier
      const int row = RGI(RG == 2 ? (lane >> 4) : 0) * 16 + (lane & 15);
      ut_s[row] += logf(a_abs);
      e_s[row] *= a_abs;
    }
    // ---- this CTA's partial of column j goes to the CTA that owns column j ----
#pragma unroll
    for (int q = 0; q < RG; ++q) {
      const int j = tid + q * (1024 / RG);
      if (j < n) {
        const float s = RG == 1 ? ((colpart[j] + colpart[CL_MAXN + j]) + colpart[2 * CL_MAXN + j]) + colpart[3 * CL_MAXN + j]
                                : colpart[j] + colpart[CL_MAXN + j];
        st_async_f32(push_addr[q], s, push_mbar[q]);
      }
    }
    if (warp == NW - 1) {   // dustbin column: kb_n sum_i e_i a_i
      float s = ea_s[lane] + ea_s[lane + 32];
      s = warp_sum(s);
      if (lane == 0) {
        const int owner = n / CS, slot = n - owner * CS;
        st_async_f32(mapa_u32(crecv_addr + (unsigned)(((int)c * CS + slot) * 4), (unsigned)owner), s * kb_s[n],
                     mapa_u32(mbarA, (unsigned)owner));
      }
    }
    T_MARK(3);
    // ---- the owner of column j adds the C partials in rank order: b_j = nu_j / (sum_g c_j^g + kb_j a_m).  A slice
    // can be wider than the CTA (CS = n + 1 for C = 1): thread tid merges columns tid, tid + NT, ... of it.  The loop
    // bound is what cl_partition_ok checks before the launch: change the two together ----
    if (tid < owned) {
      mbar_wait(mbarA, ph);
      const float am = a_s[CL_ROWS];
#pragma unroll 1
      for (int k = 0; k < CL_MERGE_COLS; ++k) {
        const int t = tid + k * NT, j = (int)c * CS + t;
        if (t >= owned) break;
        float s = 0.f;
        for (int g = 0; g < C; ++g) s += crecv[g * CS + t];
        const float bj = (j < n ? nu : nu_bin) / (s + kb_s[j] * am);
        for (int g = 0; g < C; ++g)
          st_async_f32(mapa_u32(b_addr + (unsigned)(j * 4), (unsigned)g), bj, mapa_u32(mbarB, (unsigned)g));
      }
    }
    T_MARK(4);
    // all n+1 scalings of this iteration have landed in b_s.  One warp polls, the others sleep in the barrier: 32
    // polling warps cost 34 instruction issues per warp and iteration (ncu source view, r02)
    if (warp == 0) mbar_wait(mbarB, ph);
    __syncthreads();
    T_MARK(5);
  }
  if (TIMING && cfg.timing && blockIdx.x == 0 && tid == 0)
    for (int i = 0; i < 6; ++i) cfg.timing[i] = (long long)tacc[i];
#undef T_MARK
  cluster_sync_all();          // nobody leaves while a peer may still have traffic in flight

  // ---- output: Z + u + v - norm with u = u~ + log a, v = v~ + log b ----
  __syncthreads();
  for (int j = tid; j <= n; j += blockDim.x) vt_s[j] += logf(b_s[j]);
  __syncthreads();
  if (active) {
#pragma unroll
    for (int g = 0; g < RG; ++g)
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int row = RGI(g) * 16 + i;
      if (row < nrows) {
        const float u = ut_s[row] + logf(a_s[row]) - norm;
        float* zr = Zg + (long long)(r0 + row) * ld + col0;
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (col0 + k < n) zr[k] = zr[k] + u + vt_s[col0 + k];
      }
    }
  }
  if (tid < nrows) Zg[(long long)(r0 + tid) * ld + n] = alpha + ut_s[tid] + logf(a_s[tid]) + vt_s[n] - norm;
  if (c == (unsigned)(C - 1)) {
    const float um = -alpha + logf(a_s[CL_ROWS]);     // u~_m = -alpha
    for (int j = tid; j <= n; j += blockDim.x) Zg[(long long)m * ld + j] = alpha + um + vt_s[j] - norm;
  }
#undef K_GET
#undef K_PUT
#undef RGI
}

constexpr int CL_RR = 8;   // rows of every 16-row warp tile held in registers (default)
int g_cl_default = 16;     // launch_sinkhorn_cluster's rr when the caller passes 0: 16 = two row groups per warp
#define CL_DEFAULT g_cl_default

void cl_set_attrs() {
  mvm_once_per_device(MVM_ONCE_SINKHORN_CL, [&] {
    const int smem = (int)mvm_dev_info().max_smem;
    auto set = [&](const void* k) {
      cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
      cudaFuncSetAttribute(k, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    };
    set((const void*)sinkhorn_cl_kernel<8, 1, false>);
    set((const void*)sinkhorn_cl_kernel<6, 1, false>);
    set((const void*)sinkhorn_cl_kernel<6, 1, true>);
    set((const void*)sinkhorn_cl_kernel<8, 2, false>);
    set((const void*)sinkhorn_cl_kernel<8, 2, true>);
  });
}

}  // namespace

// Smallest cluster size whose CTAs hold <= 64 rows each; 0 when the problem does not fit a cluster
// (more than 1024 rows or columns): the caller then uses the multi-CTA kernel of sinkhorn_exp.cu.
int sinkhorn_cluster_size(int max_m, int max_n) {
  if (max_n > CL_MAXN || max_m > 16 * CL_ROWS) return 0;
  int C = 1;
  while (C * CL_ROWS < max_m) C *= 2;
  return C;
}

// The column partition sinkhorn_cl_kernel relies on for an n-column problem on C CTAs of 1024 / rg threads.  Each
// iteration waits for the partials and the b_j of every column, so a column that no thread pushes or merges would
// leave the kernel waiting forever: such a shape is refused before the launch.
static bool cl_partition_ok(int n, int C, int rg) {
  const int nt = 1024 / rg, CS = (n + 1 + C - 1) / C;
  return n <= rg * nt                      // the push loop j = tid + q * nt, q < rg, reaches every column j < n
         && CS <= CL_MERGE_COLS * nt       // the owner merge has a thread for every column of its slice
         && C * CS <= CL_CRECV;            // the C partials of a slice fit crecv
}

int launch_sinkhorn_cluster(const SinkhornTable& tab, int batch, float bin_score, int iters, int C,
                            cudaStream_t stream, int rr) {
  MVM_REQUIRE(tab.n_pairs >= 1 && tab.n_pairs <= MVM_MAX_PAIRS && batch >= 1 && iters >= 1);
  MVM_REQUIRE(C == 1 || C == 2 || C == 4 || C == 8 || C == 16);
  if (rr == 0) rr = CL_DEFAULT;
  MVM_REQUIRE(rr == 6 || rr == 8 || rr == 16);      // 16 = two row groups per warp (512 threads), 8 register rows each
  const int rg = rr == 16 ? 2 : 1;
  int max_n = 0;
  for (int p = 0; p < tab.n_pairs; ++p) {
    MVM_REQUIRE(tab.m[p] >= 1 && tab.n[p] >= 1 && tab.n[p] <= CL_MAXN && tab.m[p] <= C * CL_ROWS);
    MVM_REQUIRE(cl_partition_ok(tab.n[p], C, rg));
    max_n = tab.n[p] > max_n ? tab.n[p] : max_n;
  }
  const size_t smem = cl_smem_bytes(max_n, 16 - (rr == 16 ? 8 : rr));
  auto kern = rr == 16 ? (g_sink_timing ? sinkhorn_cl_kernel<8, 2, true> : sinkhorn_cl_kernel<8, 2, false>)
              : rr == 8 ? sinkhorn_cl_kernel<8, 1, false>
                        : (g_sink_timing ? sinkhorn_cl_kernel<6, 1, true> : sinkhorn_cl_kernel<6, 1, false>);
  cl_set_attrs();
  MVM_REQUIRE(smem <= mvm_dev_info().max_smem);
  SinkClCfg cfg;
  cfg.C = C; cfg.batch = batch; cfg.iters = iters; cfg.alpha = bin_score; cfg.timing = g_sink_timing;
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3((unsigned)(tab.n_pairs * batch * C));
  lc.blockDim = dim3(1024 / rg);
  lc.dynamicSmemBytes = smem;
  lc.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = (unsigned)C;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  lc.attrs = at;
  lc.numAttrs = 1;
  MvmProfScope prof__(MVM_TAG_SINKHORN, stream);
  cudaLaunchKernelEx(&lc, kern, tab, cfg);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

// Clusters of size C that can be co-resident on the current device with this kernel's footprint
// (0: the size is not launchable here).  Used to pick the kernel and reported by bench.py.
int sinkhorn_cluster_max_active(int C, int n) {
  auto kern = CL_DEFAULT == 16 ? sinkhorn_cl_kernel<CL_RR, 2, false> : sinkhorn_cl_kernel<CL_RR, 1, false>;
  cl_set_attrs();
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3((unsigned)(C * 64));
  lc.blockDim = dim3(CL_DEFAULT == 16 ? 512 : 1024);
  lc.dynamicSmemBytes = cl_smem_bytes(n, 16 - CL_RR);
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = (unsigned)C;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  lc.attrs = at;
  lc.numAttrs = 1;
  int num = 0;
  if (cudaOccupancyMaxActiveClusters(&num, kern, &lc) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return num;
}
