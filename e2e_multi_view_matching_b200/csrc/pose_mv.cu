// Multi-view stage on the GPU: match compaction, spanning-tree initialisation and the global
// bundle adjustment that replaces the reference's Ceres `bundle_adjuster` binary.
//
// Reference:
//   * gather/compaction of valid matches  pose_optimization/multi_view/bundle_adjust_io.py:66-98
//     (and eval_pairs.py:215-222)
//   * maximum-spanning-tree initial poses  bundle_adjust_io.py:135-172
//   * problem construction (one 3-D point per pairwise match, DLT triangulation, confidence
//     normalisation c / (0.5 (sum c + 1e-3)))  bundle_adjust_io.py:193-259
//   * residual / parameterisation  problem/include/ba_problem.h:60-151, camera 0 fixed
//     (ba_problem.cpp:129-147); solver = Ceres 2.0 trust-region LM with DENSE_SCHUR and default
//     options (ba_problem.cpp:150-155), restated in oracle/mvba.py.
//
// Mapping: one CTA per (tuple, pair).  A pair's points only touch that pair's two cameras, so a
// CTA eliminates its 3x3 point blocks in registers and contributes a 12x12 block to the reduced
// camera system; the CTAs of a tuple exchange their partial blocks through L2 with a group
// barrier (two per LM iteration) and every CTA then solves the <= 42x42 reduced system redundantly
// (warp-cooperative Cholesky), so the step decision is replicated, not communicated.  fp64.
#include "../../include/mvm_b200.h"
#include "common.cuh"
#include "kernels.cuh"
#include <cstring>
#include "linalg_small.cuh"

namespace {

constexpr int NT = 256;
constexpr int NW = NT / 32;
constexpr int MAXC = 7;                 // free cameras (views - 1)
constexpr int NPART = 128;              // doubles per CTA partial record

// ---------------------------------------------------------------------------------------------
// order-preserving compaction of the valid matches of every (tuple, pair)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT) gather_matches_kernel(const float* __restrict__ kpts,
                                                            PairTable tab, int batch, int n_pad,
                                                            float conf_thresh,
                                                            float* __restrict__ mk0,
                                                            float* __restrict__ mk1,
                                                            float* __restrict__ mconf,
                                                            int* __restrict__ n_valid) {
  __shared__ int s_warp[NW];
  __shared__ int s_base;
  const int prob = blockIdx.x;                  // = bi * n_pairs + p
  const int bi = prob / tab.n_pairs, p = prob % tab.n_pairs;
  const int m = slot_count(tab.slot, bi, tab.n_views, tab.a[p], tab.m[p]);
  const int64_t* ma = tab.matches_a[p] + (long long)bi * tab.m[p];      // capacity strides
  const float* cf = tab.conf[p] + (long long)bi * tab.m[p];
  const float* ka = kpts + (long long)(bi * tab.n_views + tab.a[p]) * n_pad * 2;
  const float* kb = kpts + (long long)(bi * tab.n_views + tab.b[p]) * n_pad * 2;
  float* o0 = mk0 + (long long)prob * n_pad * 2;
  float* o1 = mk1 + (long long)prob * n_pad * 2;
  float* oc = mconf + (long long)prob * n_pad;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_base = 0;
  __syncthreads();
  for (int i0 = 0; i0 < m; i0 += NT) {
    const int i = i0 + tid;
    long long j = -1;
    float c = 0.f;
    bool valid = false;
    if (i < m) {
      j = ma[i];
      c = cf[i];
      valid = (j >= 0) && (c > conf_thresh);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, valid);
    const int wpre = __popc(bal & ((1u << lane) - 1));
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int woff = 0;
    for (int w = 0; w < warp; ++w) woff += s_warp[w];
    int total = 0;
    for (int w = 0; w < NW; ++w) total += s_warp[w];
    const int base = s_base;
    if (valid) {
      const int o = base + woff + wpre;
      o0[2 * o] = ka[2 * i]; o0[2 * o + 1] = ka[2 * i + 1];
      o1[2 * o] = kb[2 * j]; o1[2 * o + 1] = kb[2 * j + 1];
      oc[o] = c;
    }
    __syncthreads();
    if (tid == 0) s_base = base + total;
    __syncthreads();
  }
  const int cnt = s_base;
  for (int i = cnt + tid; i < n_pad; i += NT) {
    o0[2 * i] = 0.f; o0[2 * i + 1] = 0.f; o1[2 * i] = 0.f; o1[2 * i + 1] = 0.f; oc[i] = 0.f;
  }
  if (tid == 0) n_valid[prob] = cnt;
}

// ---------------------------------------------------------------------------------------------
// spanning-tree initial extrinsics (one thread per tuple; <= 8 views)
// ---------------------------------------------------------------------------------------------
__device__ void mat4_mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double s = 0;
      for (int k = 0; k < 4; ++k) s += A[i * 4 + k] * B[k * 4 + j];
      C[i * 4 + j] = s;
    }
}
__device__ void rigid_inv(const double* T, double* I) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) I[i * 4 + j] = T[j * 4 + i];
    I[i * 4 + 3] = -(T[0 * 4 + i] * T[3] + T[1 * 4 + i] * T[7] + T[2 * 4 + i] * T[11]);
  }
  I[12] = 0; I[13] = 0; I[14] = 0; I[15] = 1;
}

struct TreeArgs {
  int n_views, n_pairs, batch;
  int a[MVM_MAX_PAIRS], b[MVM_MAX_PAIRS];
  const float* T_rel;            // [B,P,16] relative poses a->b
  const int* weight;             // [B,P] edge weight (number of matches), 0 = no edge
  const unsigned char* success;  // [B,P]
  double* extr;                  // [B,T,16] world->cam
  unsigned char* on_tree;        // [B,P] or null
};

__global__ void spanning_tree_kernel(const __grid_constant__ TreeArgs t) {
  const int bi = blockIdx.x * blockDim.x + threadIdx.x;
  if (bi >= t.batch) return;
  const int T = t.n_views, P = t.n_pairs;
  // Kruskal on (max - w + 1) with a stable sort in row-major edge order == scipy's
  // minimum_spanning_tree on the transformed graph (bundle_adjust_io.py:135-140)
  int order[MVM_MAX_PAIRS], key[MVM_MAX_PAIRS], ne = 0, wmax = 0;
  int rm[MVM_MAX_PAIRS];   // pair ids sorted row-major by (a, b)
  for (int p = 0; p < P; ++p) rm[p] = p;
  for (int i = 1; i < P; ++i) {
    const int x = rm[i];
    int j = i - 1;
    while (j >= 0 && (t.a[rm[j]] * 64 + t.b[rm[j]] > t.a[x] * 64 + t.b[x])) { rm[j + 1] = rm[j]; --j; }
    rm[j + 1] = x;
  }
  for (int p = 0; p < P; ++p) {
    const int w = t.success[bi * P + p] ? t.weight[bi * P + p] : 0;
    wmax = w > wmax ? w : wmax;
  }
  for (int q = 0; q < P; ++q) {
    const int p = rm[q];
    const int w = t.success[bi * P + p] ? t.weight[bi * P + p] : 0;
    if (w > 0) { order[ne] = p; key[ne] = wmax - w + 1; ++ne; }
  }
  for (int i = 1; i < ne; ++i) {   // stable insertion sort by key
    const int kx = key[i], ox = order[i];
    int j = i - 1;
    while (j >= 0 && key[j] > kx) { key[j + 1] = key[j]; order[j + 1] = order[j]; --j; }
    key[j + 1] = kx; order[j + 1] = ox;
  }
  int comp[MVM_MAX_VIEWS];
  for (int v = 0; v < T; ++v) comp[v] = v;
  bool tree[MVM_MAX_PAIRS];
  for (int p = 0; p < P; ++p) tree[p] = false;
  for (int e = 0; e < ne; ++e) {
    const int p = order[e], ca = comp[t.a[p]], cb = comp[t.b[p]];
    if (ca != cb) {
      tree[p] = true;
      for (int v = 0; v < T; ++v)
        if (comp[v] == cb) comp[v] = ca;
    }
  }
  if (t.on_tree)
    for (int p = 0; p < P; ++p) t.on_tree[bi * P + p] = tree[p] ? 1 : 0;
  // chain absolute poses from view 0 (bundle_adjust_io.py:141-172): extr_b = T_ab extr_a
  double E[MVM_MAX_VIEWS][16];
  bool have[MVM_MAX_VIEWS];
  for (int v = 0; v < T; ++v) {
    have[v] = v == 0;
    for (int i = 0; i < 16; ++i) E[v][i] = (i % 5 == 0) ? 1.0 : 0.0;
  }
  for (int round = 0; round < T; ++round)
    for (int p = 0; p < P; ++p) {
      if (!tree[p]) continue;
      const int a = t.a[p], b = t.b[p];
      double R[16];
      for (int i = 0; i < 16; ++i) R[i] = (double)t.T_rel[((long long)bi * P + p) * 16 + i];
      if (have[a] && !have[b]) { mat4_mul(R, E[a], E[b]); have[b] = true; }
      else if (have[b] && !have[a]) { double Ri[16]; rigid_inv(R, Ri); mat4_mul(Ri, E[b], E[a]); have[a] = true; }
    }
  for (int v = 0; v < T; ++v)
    for (int i = 0; i < 16; ++i) t.extr[((long long)bi * T + v) * 16 + i] = E[v][i];
}

// ---------------------------------------------------------------------------------------------
// global bundle adjustment
// ---------------------------------------------------------------------------------------------
struct MvbaArgs {
  int n_views, n_pairs, batch, n_pad, n_groups;
  int a[MVM_MAX_PAIRS], b[MVM_MAX_PAIRS];
  const float* xa; const float* xb;     // [B,P,n_pad,2] normalised observations in views a, b
  const float* conf;                    // [B,P,n_pad] weight of a match (both observations), or of its view-a observation
  const float* conf_b;                  // [B,P,n_pad] weight of the view-b observation (per-observation weights), or null
  const int* n_valid;                   // [B,P]
  const double* extr_init;              // [B,T,16]
  const double* pts_init;               // [B,P,n_pad,3] given initial points, or null: DLT from extr_init
  int prenorm;                          // 1: conf already holds the normalised weights of ba_in.csv
  float* extr_out;                      // [B,T,16]
  double* extr_out64;                   // [B,T,16] optional fp64 copy of the result
  double* pts;                          // [B,P,2,n_pad,3] current / candidate points
  double* pscale;                       // [B,P,n_pad,3] Jacobi column scale of the points
  double* xch;                          // [groups, P, NPART] exchange
  unsigned* ctrs;                       // [groups]
  int max_iter;
  int* iters_out;                       // [B] or null
  double* cost_out;                     // [B,2] initial / final cost or null
  long long* timing;                    // optional [8] phase cycle counters of CTA 0 (tools/debug_mvba.py), or null
};
long long* g_mvba_timing = nullptr;

__device__ __forceinline__ unsigned ld_acq(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void group_barrier(unsigned* ctr, unsigned target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(ctr, 1u);
    while (ld_acq(ctr) < target) { __nanosleep(20); }
    __threadfence();
  }
  __syncthreads();
}

// d(R(w) p)/dw = -R [p]x (w w^T + (R^T - I)[w]x) / |w|^2   (-[p]x at w = 0)
__device__ void dRp_dw(const double* w, const double* R, const double* p, double* D) {
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  const double px[9] = {0, -p[2], p[1], p[2], 0, -p[0], -p[1], p[0], 0};
  if (th2 < 1e-16) {
    for (int i = 0; i < 9; ++i) D[i] = -px[i];
    return;
  }
  const double wx[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
  double A[9];   // w w^T + (R^T - I) [w]x
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = w[i] * w[j];
      for (int k = 0; k < 3; ++k) s += (R[k * 3 + i] - (i == k ? 1.0 : 0.0)) * wx[k * 3 + j];
      A[i * 3 + j] = s;
    }
  double B[9];   // [p]x A
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0;
      for (int k = 0; k < 3; ++k) s += px[i * 3 + k] * A[k * 3 + j];
      B[i * 3 + j] = s;
    }
  const double inv = -1.0 / th2;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0;
      for (int k = 0; k < 3; ++k) s += R[i * 3 + k] * B[k * 3 + j];
      D[i * 3 + j] = s * inv;
    }
}

// general two-view DLT (cv2.triangulatePoints, bundle_adjust_io.py:222)
__device__ void triangulate_general(const double* P0, const double* P1, double x0, double y0,
                                    double x1, double y1, double* X) {
  double A[4][4];
  for (int i = 0; i < 4; ++i) {
    A[0][i] = x0 * P0[8 + i] - P0[i];
    A[1][i] = y0 * P0[8 + i] - P0[4 + i];
    A[2][i] = x1 * P1[8 + i] - P1[i];
    A[3][i] = y1 * P1[8 + i] - P1[4 + i];
  }
  double M[4][4], V[4][4];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double s = 0;
      for (int k = 0; k < 4; ++k) s += A[k][i] * A[k][j];
      M[i][j] = s;
    }
  jacobi_eig_reg<4, 8>(M, V);
  const int m = argmin_diag<4>(M);
  double h[4];
  for (int i = 0; i < 4; ++i) {
    h[i] = V[i][0];
    if (m == 1) h[i] = V[i][1];
    if (m == 2) h[i] = V[i][2];
    if (m == 3) h[i] = V[i][3];
  }
  X[0] = h[0] / h[3]; X[1] = h[1] / h[3]; X[2] = h[2] / h[3];
}

// One observation: residual, weighted projection Jacobian blocks (already column-scaled).
struct Obs {
  double r[2];
  double Jc[2][6];   // zero for the fixed camera
  double Jp[2][3];
};

__device__ __forceinline__ void eval_obs(bool fixed, const double* cam, const double* R,
                                         const double* sc, const double* p, const double* sp,
                                         double x, double y, double w, bool want_J, Obs& o) {
  double q[3];
  if (fixed) { q[0] = p[0]; q[1] = p[1]; q[2] = p[2]; }
  else
    for (int i = 0; i < 3; ++i) q[i] = R[i * 3] * p[0] + R[i * 3 + 1] * p[1] + R[i * 3 + 2] * p[2] + cam[3 + i];
  const double iz = 1.0 / q[2];
  o.r[0] = w * (q[0] * iz - x);
  o.r[1] = w * (q[1] * iz - y);
  if (!want_J) return;
  const double Jpi[2][3] = {{w * iz, 0.0, -w * q[0] * iz * iz}, {0.0, w * iz, -w * q[1] * iz * iz}};
  for (int r = 0; r < 2; ++r)
    for (int c = 0; c < 3; ++c) {
      const double v = fixed ? Jpi[r][c] : Jpi[r][0] * R[c] + Jpi[r][1] * R[3 + c] + Jpi[r][2] * R[6 + c];
      o.Jp[r][c] = v * sp[c];
    }
  if (fixed) {
    for (int r = 0; r < 2; ++r)
      for (int c = 0; c < 6; ++c) o.Jc[r][c] = 0.0;
  } else {
    double D[9];
    dRp_dw(cam, R, p, D);
    for (int r = 0; r < 2; ++r) {
      for (int c = 0; c < 3; ++c)
        o.Jc[r][c] = (Jpi[r][0] * D[c] + Jpi[r][1] * D[3 + c] + Jpi[r][2] * D[6 + c]) * sc[c];
      for (int c = 0; c < 3; ++c) o.Jc[r][3 + c] = Jpi[r][c] * sc[3 + c];
    }
  }
}

// Sum 32 per-lane quantities across the warp with 31 shuffle steps (instead of 32 x 5): after the
// call q[0] of lane l holds the warp total of quantity l.  Fixed order => deterministic.
__device__ __forceinline__ void warp_reduce_transpose32(double (&q)[32], int lane) {
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const bool up = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < off; ++i) {
      const double send = up ? q[i] : q[i + off];
      const double keep = up ? q[i + off] : q[i];
      q[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
}

__device__ constexpr int kSymR[21] = {0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 4, 4, 5};
__device__ constexpr int kSymC[21] = {0, 1, 2, 3, 4, 5, 1, 2, 3, 4, 5, 2, 3, 4, 5, 3, 4, 5, 4, 5, 5};

// flat record layout of pass A: S_aa (21) | S_bb (21) | S_ab (36) | rhs_a (6) | rhs_b (6) | hdiag_a (6) |
// hdiag_b (6) | cost | (gmax, handled separately) | gc_a (6) | gc_b (6)
__device__ __forceinline__ double passA_quantity(int idx, const Obs& oa, const Obs& ob, const double (&Ua)[2][6],
                                                 const double (&Ub)[2][6], const double (&Uab)[2][6],
                                                 const double (&ra)[2], const double (&rb)[2], double cost) {
  if (idx < 21) { const int r = kSymR[idx], c = kSymC[idx]; return oa.Jc[0][r] * Ua[0][c] + oa.Jc[1][r] * Ua[1][c]; }
  if (idx < 42) { const int r = kSymR[idx - 21], c = kSymC[idx - 21]; return ob.Jc[0][r] * Ub[0][c] + ob.Jc[1][r] * Ub[1][c]; }
  if (idx < 78) { const int r = (idx - 42) / 6, c = (idx - 42) % 6; return oa.Jc[0][r] * Uab[0][c] + oa.Jc[1][r] * Uab[1][c]; }
  if (idx < 84) { const int c = idx - 78; return oa.Jc[0][c] * ra[0] + oa.Jc[1][c] * ra[1]; }
  if (idx < 90) { const int c = idx - 84; return ob.Jc[0][c] * rb[0] + ob.Jc[1][c] * rb[1]; }
  if (idx < 96) { const int c = idx - 90; return oa.Jc[0][c] * oa.Jc[0][c] + oa.Jc[1][c] * oa.Jc[1][c]; }
  if (idx < 102) { const int c = idx - 96; return ob.Jc[0][c] * ob.Jc[0][c] + ob.Jc[1][c] * ob.Jc[1][c]; }
  if (idx == 102) return cost;
  if (idx >= 104 && idx < 110) { const int c = idx - 104; return oa.Jc[0][c] * oa.r[0] + oa.Jc[1][c] * oa.r[1]; }
  if (idx >= 110 && idx < 116) { const int c = idx - 110; return ob.Jc[0][c] * ob.r[0] + ob.Jc[1][c] * ob.r[1]; }
  return 0.0;
}

// accumulate v (per lane) into dst: warp reduce, lane 0 adds
__device__ __forceinline__ void wacc(double* dst, double v, int lane) {
  v = warp_sum_d(v);
  if (lane == 0) *dst += v;
}

__global__ void __launch_bounds__(NT) mvba_kernel(const __grid_constant__ MvbaArgs g) {
  extern __shared__ double s_rec[];   // [P][NPART] all partial records of the tuple, staged once per exchange
  __shared__ double s_acc[NW][NPART];
  __shared__ double s_tot[NPART];
  __shared__ double s_H[MAXU * MAXU];
  __shared__ double s_rhs[MAXU], s_hd[MAXU], s_gc[MAXU];
  __shared__ double s_pc[MVM_MAX_PAIRS], s_pg[MVM_MAX_PAIRS], s_dec[4 * MVM_MAX_PAIRS];
  __shared__ double s_cam[MVM_MAX_VIEWS][6], s_camn[MVM_MAX_VIEWS][6];
  __shared__ double s_Ra[9], s_Rb[9], s_sc[MVM_MAX_VIEWS][6];
  __shared__ double s_ctl[8];   // radius, decrease, cost, flags
  __shared__ int s_flag[4];

  const int P = g.n_pairs, T = g.n_views;
  const int p = blockIdx.x % P;
  const int group = blockIdx.x / P;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int va = g.a[p], vb = g.b[p];
  const bool fix_a = va == 0, fix_b = vb == 0;
  unsigned* ctr = g.ctrs + group;
  unsigned bar = 0;
  double* xch_base = g.xch + (long long)group * 2 * P * NPART;   // two buffers, used alternately
  unsigned xk = 0;
  const int nu = 6 * (T - 1);

  auto zero_acc = [&]() {
    for (int e = tid; e < NW * NPART; e += NT) (&s_acc[0][0])[e] = 0.0;
    __syncthreads();
  };
  // publish this CTA's partial record, barrier, then every CTA sums all P records
  auto exchange = [&](int n) {
    // ping-pong exchange buffers: a CTA can only reach exchange k+2 (which reuses buffer k) after the
    // barrier of exchange k+1, which every CTA passes after it has staged the records of exchange k
    double* xch = xch_base + (long long)(xk & 1u) * P * NPART;
    ++xk;
    __syncthreads();
    for (int e = tid; e < n; e += NT) {
      double s = 0.0;
      for (int w = 0; w < NW; ++w) s += s_acc[w][e];
      __stcg(xch + (long long)p * NPART + e, s);
    }
    bar += P;
    group_barrier(ctr, bar);
    for (int e = tid; e < P * n; e += NT) s_rec[(e / n) * NPART + (e % n)] = __ldcg(xch + (long long)(e / n) * NPART + (e % n));
    __syncthreads();
  };

  for (int bi = group; bi < g.batch; bi += g.n_groups) {
    const long long prob = (long long)bi * P + p;
    const int n = g.n_valid[prob];
    const float* xa = g.xa + prob * g.n_pad * 2;
    const float* xb = g.xb + prob * g.n_pad * 2;
    const float* cf = g.conf + prob * g.n_pad;
    const float* cfb = g.conf_b ? g.conf_b + prob * g.n_pad : cf;     // BaProblem weights are per OBSERVATION (ba_problem.h:60-151)
    double* pcur = g.pts + prob * 2 * g.n_pad * 3;
    double* pnew = pcur + (long long)g.n_pad * 3;
    double* psc = g.pscale + prob * g.n_pad * 3;

    // ---- cameras: world->cam extrinsics -> (angle axis | t) ----
    if (tid < T) {
      const double* E = g.extr_init + ((long long)bi * T + tid) * 16;
      const double R[9] = {E[0], E[1], E[2], E[4], E[5], E[6], E[8], E[9], E[10]};
      double w[3];
      R_to_aa(R, w);
      s_cam[tid][0] = w[0]; s_cam[tid][1] = w[1]; s_cam[tid][2] = w[2];
      s_cam[tid][3] = E[3]; s_cam[tid][4] = E[7]; s_cam[tid][5] = E[11];
    }
    zero_acc();
    // ---- confidence normalisation over all observations of the tuple (:56-60) ----
    {
      double c = 0.0;
      for (int i = tid; i < n; i += NT) c += (double)cf[i] + (double)cfb[i];
      wacc(&s_acc[warp][0], c, lane);
      exchange(1);
    }
    double csum = 0.0;
    for (int q = 0; q < P; ++q) csum += s_rec[q * NPART];
    const double wscale = g.prenorm ? 1.0 : 1.0 / (0.5 * (csum + 1e-3));

    // ---- initial points: DLT with the initial extrinsics ----
    {
      const double* Ea = g.extr_init + ((long long)bi * T + va) * 16;
      const double* Eb = g.extr_init + ((long long)bi * T + vb) * 16;
      const double* pin = g.pts_init ? g.pts_init + prob * g.n_pad * 3 : nullptr;
      for (int i = tid; i < n; i += NT) {
        double X[3];
        if (pin) { X[0] = pin[3 * i]; X[1] = pin[3 * i + 1]; X[2] = pin[3 * i + 2]; }
        else triangulate_general(Ea, Eb, xa[2 * i], xa[2 * i + 1], xb[2 * i], xb[2 * i + 1], X);
        pcur[3 * i] = X[0]; pcur[3 * i + 1] = X[1]; pcur[3 * i + 2] = X[2];
      }
    }
    __syncthreads();

    // ---- Jacobi column scaling, fixed at the first linearisation ----
    if (tid == 0) { aa_to_R(s_cam[va], s_Ra); aa_to_R(s_cam[vb], s_Rb); }
    zero_acc();
    {
      const double one6[6] = {1, 1, 1, 1, 1, 1}, one3[3] = {1, 1, 1};
      for (int i0 = 0; i0 < n; i0 += NT) {
        const int i = i0 + tid;
        double na[6] = {0, 0, 0, 0, 0, 0}, nb[6] = {0, 0, 0, 0, 0, 0};
        if (i < n) {
          const double pt[3] = {pcur[3 * i], pcur[3 * i + 1], pcur[3 * i + 2]};
          const double w = (double)cf[i] * wscale, wB = (double)cfb[i] * wscale;
          Obs oa, ob;
          eval_obs(fix_a, s_cam[va], s_Ra, one6, pt, one3, xa[2 * i], xa[2 * i + 1], w, true, oa);
          eval_obs(fix_b, s_cam[vb], s_Rb, one6, pt, one3, xb[2 * i], xb[2 * i + 1], wB, true, ob);
          for (int c = 0; c < 3; ++c) {
            const double s = oa.Jp[0][c] * oa.Jp[0][c] + oa.Jp[1][c] * oa.Jp[1][c] +
                             ob.Jp[0][c] * ob.Jp[0][c] + ob.Jp[1][c] * ob.Jp[1][c];
            psc[3 * i + c] = 1.0 / (1.0 + sqrt(s));
          }
          for (int c = 0; c < 6; ++c) {
            na[c] = oa.Jc[0][c] * oa.Jc[0][c] + oa.Jc[1][c] * oa.Jc[1][c];
            nb[c] = ob.Jc[0][c] * ob.Jc[0][c] + ob.Jc[1][c] * ob.Jc[1][c];
          }
        }
        for (int c = 0; c < 6; ++c) { wacc(&s_acc[warp][c], na[c], lane); wacc(&s_acc[warp][6 + c], nb[c], lane); }
      }
      exchange(12);
    }
    if (tid < 6 * T) {
      const int v = tid / 6, c = tid % 6;
      double s = 0.0;
      for (int q = 0; q < P; ++q) {
        if (g.a[q] == v) s += s_rec[q * NPART + c];
        if (g.b[q] == v) s += s_rec[q * NPART + 6 + c];
      }
      s_sc[v][c] = 1.0 / (1.0 + sqrt(s));
    }
    if (tid == 0) { s_ctl[0] = 1e4; s_ctl[1] = 2.0; s_ctl[2] = -1.0; s_flag[0] = 0; }
    __syncthreads();

    int it = 0;
    bool need_cost0 = true;
    long long tacc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (; it < g.max_iter; ++it) {
      long long tph = clock64();
      auto phase = [&](int k) { const long long t1 = clock64(); tacc[k] += t1 - tph; tph = t1; };
      // ================= pass A: reduced camera system at the current point =================
      if (tid == 0) { aa_to_R(s_cam[va], s_Ra); aa_to_R(s_cam[vb], s_Rb); }
      zero_acc();
      const double radius = s_ctl[0];
      for (int i0 = 0; i0 < n; i0 += NT) {
        const int i = i0 + tid;
        const bool act = i < n;
        Obs oa, ob;
        double Ua[2][6], Ub[2][6], Uab[2][6], ra[2], rb[2], cost = 0.0, gmax = 0.0;
        if (act) {
          const double pt[3] = {pcur[3 * i], pcur[3 * i + 1], pcur[3 * i + 2]};
          const double sp[3] = {psc[3 * i], psc[3 * i + 1], psc[3 * i + 2]};
          const double w = (double)cf[i] * wscale, wB = (double)cfb[i] * wscale;
          eval_obs(fix_a, s_cam[va], s_Ra, s_sc[va], pt, sp, xa[2 * i], xa[2 * i + 1], w, true, oa);
          eval_obs(fix_b, s_cam[vb], s_Rb, s_sc[vb], pt, sp, xb[2 * i], xb[2 * i + 1], wB, true, ob);
          cost = 0.5 * (oa.r[0] * oa.r[0] + oa.r[1] * oa.r[1] + ob.r[0] * ob.r[0] + ob.r[1] * ob.r[1]);
          // point block M = Hpp + clamp(diag)/radius
          double H[6];
          int e = 0;
          for (int r = 0; r < 3; ++r)
            for (int c = r; c < 3; ++c)
              H[e++] = oa.Jp[0][r] * oa.Jp[0][c] + oa.Jp[1][r] * oa.Jp[1][c] + ob.Jp[0][r] * ob.Jp[0][c] + ob.Jp[1][r] * ob.Jp[1][c];
          H[0] += fmin(fmax(H[0], 1e-6), 1e32) / radius;
          H[3] += fmin(fmax(H[3], 1e-6), 1e32) / radius;
          H[5] += fmin(fmax(H[5], 1e-6), 1e32) / radius;
          double Mi[6];
          inv3_sym(H, Mi);
          // Z_x = Jp_x Mi (2x3);  W_xy = Z_x Jp_y^T (2x2)
          double Za[2][3], Zb[2][3];
          for (int r = 0; r < 2; ++r) {
            Za[r][0] = oa.Jp[r][0] * Mi[0] + oa.Jp[r][1] * Mi[1] + oa.Jp[r][2] * Mi[2];
            Za[r][1] = oa.Jp[r][0] * Mi[1] + oa.Jp[r][1] * Mi[3] + oa.Jp[r][2] * Mi[4];
            Za[r][2] = oa.Jp[r][0] * Mi[2] + oa.Jp[r][1] * Mi[4] + oa.Jp[r][2] * Mi[5];
            Zb[r][0] = ob.Jp[r][0] * Mi[0] + ob.Jp[r][1] * Mi[1] + ob.Jp[r][2] * Mi[2];
            Zb[r][1] = ob.Jp[r][0] * Mi[1] + ob.Jp[r][1] * Mi[3] + ob.Jp[r][2] * Mi[4];
            Zb[r][2] = ob.Jp[r][0] * Mi[2] + ob.Jp[r][1] * Mi[4] + ob.Jp[r][2] * Mi[5];
          }
          double Waa[2][2], Wab[2][2], Wbb[2][2];
          for (int r = 0; r < 2; ++r)
            for (int c = 0; c < 2; ++c) {
              Waa[r][c] = Za[r][0] * oa.Jp[c][0] + Za[r][1] * oa.Jp[c][1] + Za[r][2] * oa.Jp[c][2];
              Wab[r][c] = Za[r][0] * ob.Jp[c][0] + Za[r][1] * ob.Jp[c][1] + Za[r][2] * ob.Jp[c][2];
              Wbb[r][c] = Zb[r][0] * ob.Jp[c][0] + Zb[r][1] * ob.Jp[c][1] + Zb[r][2] * ob.Jp[c][2];
            }
          // U_a = (I - Waa) Jc_a, U_b = (I - Wbb) Jc_b, U_ab = -Wab Jc_b
          for (int c = 0; c < 6; ++c) {
            Ua[0][c] = (1.0 - Waa[0][0]) * oa.Jc[0][c] - Waa[0][1] * oa.Jc[1][c];
            Ua[1][c] = -Waa[1][0] * oa.Jc[0][c] + (1.0 - Waa[1][1]) * oa.Jc[1][c];
            Ub[0][c] = (1.0 - Wbb[0][0]) * ob.Jc[0][c] - Wbb[0][1] * ob.Jc[1][c];
            Ub[1][c] = -Wbb[1][0] * ob.Jc[0][c] + (1.0 - Wbb[1][1]) * ob.Jc[1][c];
            Uab[0][c] = -(Wab[0][0] * ob.Jc[0][c] + Wab[0][1] * ob.Jc[1][c]);
            Uab[1][c] = -(Wab[1][0] * ob.Jc[0][c] + Wab[1][1] * ob.Jc[1][c]);
          }
          // reduced rhs pieces: -(I - Waa) r_a + Wab r_b etc.  gp = Jpa^T ra + Jpb^T rb
          double gp[3];
          for (int c = 0; c < 3; ++c) {
            gp[c] = oa.Jp[0][c] * oa.r[0] + oa.Jp[1][c] * oa.r[1] + ob.Jp[0][c] * ob.r[0] + ob.Jp[1][c] * ob.r[1];
            gmax = fmax(gmax, fabs(gp[c] / sp[c]));
          }
          for (int r = 0; r < 2; ++r) {
            ra[r] = -oa.r[r] + Za[r][0] * gp[0] + Za[r][1] * gp[1] + Za[r][2] * gp[2];
            rb[r] = -ob.r[r] + Zb[r][0] * gp[0] + Zb[r][1] * gp[1] + Zb[r][2] * gp[2];
          }
        } else {
          for (int r = 0; r < 2; ++r) {
            ra[r] = rb[r] = oa.r[r] = ob.r[r] = 0.0;
            for (int c = 0; c < 6; ++c) { Ua[r][c] = Ub[r][c] = Uab[r][c] = oa.Jc[r][c] = ob.Jc[r][c] = 0.0; }
          }
        }
        // accumulate the 116 sums of this 32-point batch: four transposed warp reductions of 32 quantities
        double* acc = s_acc[warp];
#pragma unroll
        for (int grp = 0; grp < 4; ++grp) {
          double q[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) q[i] = passA_quantity(grp * 32 + i, oa, ob, Ua, Ub, Uab, ra, rb, cost);
          warp_reduce_transpose32(q, lane);
          if (grp * 32 + lane != 103) acc[grp * 32 + lane] += q[0];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) gmax = fmax(gmax, __shfl_xor_sync(0xffffffffu, gmax, o));
        if (lane == 0) acc[103] = fmax(acc[103], gmax);
      }
      // gmax is a max, not a sum: fold the per-warp maxima before publishing
      __syncthreads();
      if (tid == 0) {
        double m = 0.0;
        for (int w = 0; w < NW; ++w) { m = fmax(m, s_acc[w][103]); s_acc[w][103] = 0.0; }
        s_acc[0][103] = m;
      }
      phase(0);
      exchange(116);
      phase(1);

      // ---- assemble the reduced system from all partial records.  Every output element is owned
      // by one thread and summed over the pairs in a fixed order, so all CTAs of the tuple build
      // bit-identical systems (their replicated accept/reject decisions must never diverge). ----
      for (int e = tid; e < nu * nu; e += NT) {
        const int u = e / nu, v = e % nu;
        const int cu = u / 6 + 1, r = u % 6, cv = v / 6 + 1, c = v % 6;
        double s = 0.0;
        for (int q = 0; q < P; ++q) {
          const double* rec = s_rec + q * NPART;
          const int lo = r < c ? r : c, hi = r < c ? c : r;
          const int sym = lo * 6 - lo * (lo - 1) / 2 + (hi - lo);
          if (g.a[q] == cu && g.a[q] == cv) s += *(rec + sym);
          if (g.b[q] == cu && g.b[q] == cv) s += *(rec + 21 + sym);
          if (g.a[q] == cu && g.b[q] == cv) s += *(rec + 42 + r * 6 + c);
          if (g.b[q] == cu && g.a[q] == cv) s += *(rec + 42 + c * 6 + r);
        }
        s_H[u * MAXU + v] = s;
      }
      if (tid < nu) {
        const int cu = tid / 6 + 1, c = tid % 6;
        double rs = 0.0, hd = 0.0, gc = 0.0;
        for (int q = 0; q < P; ++q) {
          const double* rec = s_rec + q * NPART;
          if (g.a[q] == cu) { rs += *(rec + 78 + c); hd += *(rec + 90 + c); gc += *(rec + 104 + c); }
          if (g.b[q] == cu) { rs += *(rec + 84 + c); hd += *(rec + 96 + c); gc += *(rec + 110 + c); }
        }
        s_rhs[tid] = rs;
        s_hd[tid] = hd;
        s_gc[tid] = fabs(gc / s_sc[cu][c]);   // camera part of the unscaled gradient (Ceres tests max |J^T r|)
      }
      if (tid >= 64 && tid < 64 + P) {        // per-pair cost / point-gradient records, one load per thread
        const double* rec = s_rec + (tid - 64) * NPART;
        s_pc[tid - 64] = *(rec + 102);
        s_pg[tid - 64] = *(rec + 103);
      }
      __syncthreads();
      if (tid == 0) {
        double cost = 0.0, gmax = 0.0;
        for (int q = 0; q < P; ++q) { cost += s_pc[q]; gmax = fmax(gmax, s_pg[q]); }   // fixed order
        for (int u = 0; u < nu; ++u) gmax = fmax(gmax, s_gc[u]);
        for (int u = 0; u < nu; ++u) s_H[u * MAXU + u] += fmin(fmax(s_hd[u], 1e-6), 1e32) / radius;
        if (need_cost0) { s_ctl[2] = cost; if (g.cost_out && p == 0) g.cost_out[bi * 2] = cost; }
        s_ctl[3] = gmax;
      }
      __syncthreads();
      need_cost0 = false;
      phase(2);
      if (warp == 0) {
        const bool ok = nu < 32 ? chol_solve_warp_rows(s_H, s_rhs, nu, lane) : chol_solve_warp(s_H, s_rhs, nu, lane);
        if (lane == 0) s_flag[1] = ok ? 1 : 0;
      }
      __syncthreads();
      phase(3);
      const bool solved = s_flag[1] != 0;
      const double cost_cur = s_ctl[2];
      if (s_ctl[3] <= 1e-10) { if (tid == 0) s_flag[0] = 1; __syncthreads(); break; }   // gradient tolerance

      // ================= pass B: candidate step, model and true cost change =================
      if (tid < T) {
        for (int c = 0; c < 6; ++c) {
          const double d = (tid == 0 || !solved) ? 0.0 : s_rhs[(tid - 1) * 6 + c] * s_sc[tid][c];
          s_camn[tid][c] = s_cam[tid][c] + d;
        }
      }
      __syncthreads();
      if (tid == 0) { aa_to_R(s_camn[va], s_Ra); aa_to_R(s_camn[vb], s_Rb); }
      zero_acc();
      {
        double Rca[9], Rcb[9];
        aa_to_R(s_cam[va], Rca);
        aa_to_R(s_cam[vb], Rcb);
        double dca[6], dcb[6];
        for (int c = 0; c < 6; ++c) {
          dca[c] = (fix_a || !solved) ? 0.0 : s_rhs[(va - 1) * 6 + c];
          dcb[c] = (fix_b || !solved) ? 0.0 : s_rhs[(vb - 1) * 6 + c];
        }
        for (int i0 = 0; i0 < n; i0 += NT) {
          const int i = i0 + tid;
          double cnew = 0.0, mod = 0.0, dn2 = 0.0, xn2 = 0.0;
          if (i < n && solved) {
            const double pt[3] = {pcur[3 * i], pcur[3 * i + 1], pcur[3 * i + 2]};
            const double sp[3] = {psc[3 * i], psc[3 * i + 1], psc[3 * i + 2]};
            const double w = (double)cf[i] * wscale, wB = (double)cfb[i] * wscale;
            Obs oa, ob;
            eval_obs(fix_a, s_cam[va], Rca, s_sc[va], pt, sp, xa[2 * i], xa[2 * i + 1], w, true, oa);
            eval_obs(fix_b, s_cam[vb], Rcb, s_sc[vb], pt, sp, xb[2 * i], xb[2 * i + 1], wB, true, ob);
            double H[6];
            int e = 0;
            for (int r = 0; r < 3; ++r)
              for (int c = r; c < 3; ++c)
                H[e++] = oa.Jp[0][r] * oa.Jp[0][c] + oa.Jp[1][r] * oa.Jp[1][c] + ob.Jp[0][r] * ob.Jp[0][c] + ob.Jp[1][r] * ob.Jp[1][c];
            H[0] += fmin(fmax(H[0], 1e-6), 1e32) / radius;
            H[3] += fmin(fmax(H[3], 1e-6), 1e32) / radius;
            H[5] += fmin(fmax(H[5], 1e-6), 1e32) / radius;
            double Mi[6];
            inv3_sym(H, Mi);
            // camera-induced residual change  ja = Jc_a dca, jb = Jc_b dcb
            double ja[2] = {0, 0}, jb[2] = {0, 0};
            for (int c = 0; c < 6; ++c) {
              ja[0] += oa.Jc[0][c] * dca[c]; ja[1] += oa.Jc[1][c] * dca[c];
              jb[0] += ob.Jc[0][c] * dcb[c]; jb[1] += ob.Jc[1][c] * dcb[c];
            }
            double rhs[3], dp[3];
            for (int c = 0; c < 3; ++c)
              rhs[c] = -(oa.Jp[0][c] * (oa.r[0] + ja[0]) + oa.Jp[1][c] * (oa.r[1] + ja[1]) +
                         ob.Jp[0][c] * (ob.r[0] + jb[0]) + ob.Jp[1][c] * (ob.r[1] + jb[1]));
            dp[0] = Mi[0] * rhs[0] + Mi[1] * rhs[1] + Mi[2] * rhs[2];
            dp[1] = Mi[1] * rhs[0] + Mi[3] * rhs[1] + Mi[4] * rhs[2];
            dp[2] = Mi[2] * rhs[0] + Mi[4] * rhs[1] + Mi[5] * rhs[2];
            for (int r = 0; r < 2; ++r) {
              const double ma = oa.r[r] + ja[r] + oa.Jp[r][0] * dp[0] + oa.Jp[r][1] * dp[1] + oa.Jp[r][2] * dp[2];
              const double mb = ob.r[r] + jb[r] + ob.Jp[r][0] * dp[0] + ob.Jp[r][1] * dp[1] + ob.Jp[r][2] * dp[2];
              mod += 0.5 * (ma * ma + mb * mb);
            }
            double pn[3];
            for (int c = 0; c < 3; ++c) {
              const double d = dp[c] * sp[c];
              pn[c] = pt[c] + d;
              dn2 += d * d;
              xn2 += pt[c] * pt[c];
              pnew[3 * i + c] = pn[c];
            }
            Obs na, nb;
            const double one6[6] = {1, 1, 1, 1, 1, 1}, one3[3] = {1, 1, 1};
            eval_obs(fix_a, s_camn[va], s_Ra, one6, pn, one3, xa[2 * i], xa[2 * i + 1], w, false, na);
            eval_obs(fix_b, s_camn[vb], s_Rb, one6, pn, one3, xb[2 * i], xb[2 * i + 1], wB, false, nb);
            cnew = 0.5 * (na.r[0] * na.r[0] + na.r[1] * na.r[1] + nb.r[0] * nb.r[0] + nb.r[1] * nb.r[1]);
          }
          wacc(&s_acc[warp][0], cnew, lane);
          wacc(&s_acc[warp][1], mod, lane);
          wacc(&s_acc[warp][2], dn2, lane);
          wacc(&s_acc[warp][3], xn2, lane);
        }
      }
      phase(4);
      exchange(4);
      phase(5);
      if (tid < 4 * P) s_dec[tid] = s_rec[(tid >> 2) * NPART + (tid & 3)];
      __syncthreads();
      if (tid == 0) {
        double cnew = 0.0, mod = 0.0, dn2 = 0.0, xn2 = 0.0;
        for (int q = 0; q < P; ++q) {     // fixed order: identical on every CTA of the tuple
          cnew += s_dec[4 * q]; mod += s_dec[4 * q + 1]; dn2 += s_dec[4 * q + 2]; xn2 += s_dec[4 * q + 3];
        }
        for (int v = 1; v < T; ++v)
          for (int c = 0; c < 6; ++c) {
            const double d = s_camn[v][c] - s_cam[v][c];
            dn2 += d * d;
            xn2 += s_cam[v][c] * s_cam[v][c];
          }
        int stop = 0, accept = 0;
        double radius_n = s_ctl[0], dec = s_ctl[1];
        if (!solved) {
          radius_n /= dec; dec *= 2.0;
        } else if (sqrt(dn2) <= 1e-8 * (sqrt(xn2) + 1e-8)) {
          stop = 1;                                            // parameter tolerance
        } else {
          const double model_change = cost_cur - mod;
          const double rho = model_change > 0.0 ? (cost_cur - cnew) / model_change : -1.0;
          if (rho > 1e-3) {
            accept = 1;
            const double t = 2.0 * rho - 1.0;
            radius_n = fmin(radius_n / fmax(1.0 / 3.0, 1.0 - t * t * t), 1e16);
            dec = 2.0;
            if (fabs(cost_cur - cnew) <= 1e-6 * cost_cur) stop = 1;   // function tolerance
            s_ctl[2] = cnew;
          } else {
            radius_n /= dec; dec *= 2.0;
          }
        }
        s_ctl[0] = radius_n; s_ctl[1] = dec;
        s_flag[2] = accept; s_flag[3] = stop;
      }
      __syncthreads();
      if (s_flag[2]) {
        if (tid < T)
          for (int c = 0; c < 6; ++c) s_cam[tid][c] = s_camn[tid][c];
        double* t = pcur; pcur = pnew; pnew = t;
      }
      __syncthreads();
      phase(6);
      if (s_flag[3]) { ++it; break; }
    }
    if (g.timing && blockIdx.x == 0 && tid == 0 && bi == group) {
      for (int k = 0; k < 7; ++k) g.timing[k] = tacc[k];
      g.timing[7] = it;
    }

    // ---- result: extrinsics of every view (camera 0 untouched) ----
    if (p == 0 && tid < T) {
      double R[9];
      aa_to_R(s_cam[tid], R);
      float* E = g.extr_out + ((long long)bi * T + tid) * 16;
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) E[i * 4 + j] = (float)R[i * 3 + j];
        E[i * 4 + 3] = (float)s_cam[tid][3 + i];
      }
      E[12] = 0.f; E[13] = 0.f; E[14] = 0.f; E[15] = 1.f;
      if (g.extr_out64) {
        double* D = g.extr_out64 + ((long long)bi * T + tid) * 16;
        for (int i = 0; i < 3; ++i) {
          for (int j = 0; j < 3; ++j) D[i * 4 + j] = R[i * 3 + j];
          D[i * 4 + 3] = s_cam[tid][3 + i];
        }
        D[12] = 0.0; D[13] = 0.0; D[14] = 0.0; D[15] = 1.0;
      }
      if (tid == 0) {
        if (g.iters_out) g.iters_out[bi] = it;
        if (g.cost_out) g.cost_out[bi * 2 + 1] = s_ctl[2];
      }
    }
    bar += P;
    group_barrier(ctr, bar);
  }
}

// cv2.triangulatePoints of every match of every (tuple, pair) with given extrinsics
// (write_bundle_adjust_problem, bundle_adjust_io.py:219-225)
__global__ void __launch_bounds__(NT) triangulate_pairs_kernel(const __grid_constant__ MvbaArgs g, double* __restrict__ out) {
  const int P = g.n_pairs, T = g.n_views;
  const long long prob = blockIdx.x;
  const int bi = (int)(prob / P), p = (int)(prob % P);
  const int n = g.n_valid[prob];
  const double* Ea = g.extr_init + ((long long)bi * T + g.a[p]) * 16;
  const double* Eb = g.extr_init + ((long long)bi * T + g.b[p]) * 16;
  const float* xa = g.xa + prob * g.n_pad * 2;
  const float* xb = g.xb + prob * g.n_pad * 2;
  double* o = out + prob * g.n_pad * 3;
  for (int i = threadIdx.x; i < g.n_pad; i += NT) {
    double X[3] = {0.0, 0.0, 0.0};
    if (i < n) triangulate_general(Ea, Eb, xa[2 * i], xa[2 * i + 1], xb[2 * i], xb[2 * i + 1], X);
    o[3 * i] = X[0]; o[3 * i + 1] = X[1]; o[3 * i + 2] = X[2];
  }
}

}  // namespace

extern "C" {

int mvm_gather_matches(const float* kpts, int n_views, int n_pad, const int* counts,
                       const mvm_pair_io* pairs, int n_pairs, int batch, float conf_thresh,
                       float* mkpts_a, float* mkpts_b, float* mconf, int* n_valid, void* stream) {
  return mvm_gather_matches_ragged(kpts, n_views, n_pad, counts, nullptr, pairs, n_pairs, batch, conf_thresh, mkpts_a,
                                   mkpts_b, mconf, n_valid, stream);
}

int mvm_gather_matches_ragged(const float* kpts, int n_views, int n_pad, const int* counts, const int* slot_counts,
                              const mvm_pair_io* pairs, int n_pairs, int batch, float conf_thresh,
                              float* mkpts_a, float* mkpts_b, float* mconf, int* n_valid, void* stream) {
  MVM_REQUIRE(kpts && counts && pairs && mkpts_a && mkpts_b && mconf && n_valid);
  MVM_REQUIRE(n_pairs >= 1 && n_pairs <= MVM_MAX_PAIRS && batch >= 1);
  MvmProfScope prof__(MVM_TAG_MISC, (cudaStream_t)stream);
  PairTable tab;
  tab.n_pairs = n_pairs; tab.n_views = n_views; tab.slot = slot_counts;
  for (int p = 0; p < n_pairs; ++p) {
    // a view id indexes counts (host), the views of kpts and, with slot_counts, the slots
    MVM_REQUIRE(pairs[p].view_a >= 0 && pairs[p].view_a < n_views && pairs[p].view_b >= 0 &&
                pairs[p].view_b < n_views);
    tab.a[p] = pairs[p].view_a; tab.b[p] = pairs[p].view_b;
    tab.m[p] = counts[pairs[p].view_a]; tab.n[p] = counts[pairs[p].view_b];
    tab.matches_a[p] = pairs[p].matches_a; tab.conf[p] = pairs[p].conf;
    MVM_REQUIRE(pairs[p].matches_a && pairs[p].conf);
  }
  gather_matches_kernel<<<batch * n_pairs, NT, 0, (cudaStream_t)stream>>>(
      kpts, tab, batch, n_pad, conf_thresh, mkpts_a, mkpts_b, mconf, n_valid);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

int mvm_spanning_tree_init(const int* pair_a, const int* pair_b, int n_views, int n_pairs, int batch,
                           const float* T_rel, const int* weight, const unsigned char* success,
                           double* extr, unsigned char* on_tree, void* stream) {
  MVM_REQUIRE(pair_a && pair_b && T_rel && weight && success && extr);
  MVM_REQUIRE(n_views >= 2 && n_views <= MVM_MAX_VIEWS && n_pairs >= 1 && n_pairs <= MVM_MAX_PAIRS);
  MvmProfScope prof__(MVM_TAG_MISC, (cudaStream_t)stream);
  TreeArgs t;
  t.n_views = n_views; t.n_pairs = n_pairs; t.batch = batch;
  for (int p = 0; p < n_pairs; ++p) { t.a[p] = pair_a[p]; t.b[p] = pair_b[p]; MVM_REQUIRE(0 <= pair_a[p] && pair_a[p] < pair_b[p] && pair_b[p] < n_views); }
  t.T_rel = T_rel; t.weight = weight; t.success = success; t.extr = extr; t.on_tree = on_tree;
  spanning_tree_kernel<<<mvm_div_up(batch, 64), 64, 0, (cudaStream_t)stream>>>(t);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

size_t mvm_mvba_workspace_bytes(int n_views, int n_pairs, int batch, int n_pad) {
  const size_t pts = (size_t)batch * n_pairs * 2 * n_pad * 3 * sizeof(double);
  const size_t psc = (size_t)batch * n_pairs * n_pad * 3 * sizeof(double);
  const size_t xch = (size_t)2 * 160 * n_pairs * NPART * sizeof(double);
  return pts + psc + xch + 1024;
}

void mvm_debug_set_mvba_timing(long long* p) { g_mvba_timing = p; }

int mvm_multi_view_ba_ex(const int* pair_a, const int* pair_b, int n_views, int n_pairs, int batch,
                         int n_pad, const float* xn_a, const float* xn_b, const float* conf,
                         const int* n_valid, const double* extr_init, const double* points_init,
                         int weights_prenormalized, float* extr_out, double* extr_out_f64, int max_iterations,
                         int* iterations_out, double* cost_out, void* workspace, size_t workspace_bytes,
                         void* stream_) {
  return mvm_multi_view_ba_obs(pair_a, pair_b, n_views, n_pairs, batch, n_pad, xn_a, xn_b, conf, nullptr, n_valid, extr_init,
                               points_init, weights_prenormalized, extr_out, extr_out_f64, max_iterations, iterations_out,
                               cost_out, workspace, workspace_bytes, stream_);
}

int mvm_multi_view_ba_obs(const int* pair_a, const int* pair_b, int n_views, int n_pairs, int batch,
                         int n_pad, const float* xn_a, const float* xn_b, const float* conf, const float* conf_b,
                         const int* n_valid, const double* extr_init, const double* points_init,
                         int weights_prenormalized, float* extr_out, double* extr_out_f64, int max_iterations,
                         int* iterations_out, double* cost_out, void* workspace, size_t workspace_bytes,
                         void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  MVM_REQUIRE(pair_a && pair_b && xn_a && xn_b && conf && n_valid && extr_init && extr_out && workspace);
  MVM_REQUIRE(n_views >= 2 && n_views <= MVM_MAX_VIEWS && n_pairs >= 1 && n_pairs <= MVM_MAX_PAIRS);
  if (workspace_bytes < mvm_mvba_workspace_bytes(n_views, n_pairs, batch, n_pad)) return MVM_ERR_WORKSPACE;
  MvmProfScope prof__(MVM_TAG_MVBA, stream);
  const int n_sm = mvm_dev_info().n_sm;
  MvbaArgs g;
  g.n_views = n_views; g.n_pairs = n_pairs; g.batch = batch; g.n_pad = n_pad;
  for (int p = 0; p < n_pairs; ++p) { g.a[p] = pair_a[p]; g.b[p] = pair_b[p]; MVM_REQUIRE(0 <= pair_a[p] && pair_a[p] < pair_b[p] && pair_b[p] < n_views); }
  int groups = n_sm / n_pairs;          // one CTA per SM keeps every group co-resident
  if (groups < 1) return MVM_ERR_INVALID;
  if (groups > batch) groups = batch;
  g.n_groups = groups;
  g.xa = xn_a; g.xb = xn_b; g.conf = conf; g.conf_b = conf_b; g.n_valid = n_valid; g.extr_init = extr_init;
  g.pts_init = points_init; g.prenorm = weights_prenormalized ? 1 : 0; g.extr_out64 = extr_out_f64;
  g.extr_out = extr_out; g.max_iter = max_iterations; g.iters_out = iterations_out; g.cost_out = cost_out;
  g.timing = g_mvba_timing;
  char* w = (char*)workspace;
  g.ctrs = (unsigned*)w; w += 1024;
  g.pts = (double*)w; w += (size_t)batch * n_pairs * 2 * n_pad * 3 * sizeof(double);
  g.pscale = (double*)w; w += (size_t)batch * n_pairs * n_pad * 3 * sizeof(double);
  g.xch = (double*)w;
  cudaMemsetAsync(g.ctrs, 0, 1024, stream);
  // s_rec holds the records of every pair of the tuple: at 8 views (28 pairs, 28 KB) it takes the CTA past the
  // 48 KB of shared memory a kernel gets without opting in, and the cooperative launch would find no room at all
  mvm_once_per_device(MVM_ONCE_MVBA, [] {
    cudaFuncSetAttribute(mvba_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)(MVM_MAX_PAIRS * NPART * sizeof(double)));
  });
  // the CTAs of a group spin on a software barrier: launch cooperatively so that co-residency of the whole
  // grid is guaranteed by the driver (fails with an error instead of deadlocking when it cannot be)
  {
    void* kargs[] = {(void*)&g};
    cudaLaunchCooperativeKernel((const void*)mvba_kernel, dim3(groups * n_pairs), dim3(NT), kargs,
                                (size_t)n_pairs * NPART * sizeof(double), stream);
  }
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

int mvm_multi_view_ba(const int* pair_a, const int* pair_b, int n_views, int n_pairs, int batch,
                      int n_pad, const float* xn_a, const float* xn_b, const float* conf,
                      const int* n_valid, const double* extr_init, float* extr_out, int max_iterations,
                      int* iterations_out, double* cost_out, void* workspace, size_t workspace_bytes,
                      void* stream_) {
  return mvm_multi_view_ba_ex(pair_a, pair_b, n_views, n_pairs, batch, n_pad, xn_a, xn_b, conf, n_valid, extr_init,
                              nullptr, 0, extr_out, nullptr, max_iterations, iterations_out, cost_out, workspace,
                              workspace_bytes, stream_);
}

int mvm_triangulate_pairs(const int* pair_a, const int* pair_b, int n_views, int n_pairs, int batch, int n_pad,
                          const float* xn_a, const float* xn_b, const int* n_valid, const double* extr,
                          double* points_out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  MVM_REQUIRE(pair_a && pair_b && xn_a && xn_b && n_valid && extr && points_out);
  MVM_REQUIRE(n_views >= 2 && n_views <= MVM_MAX_VIEWS && n_pairs >= 1 && n_pairs <= MVM_MAX_PAIRS && batch >= 1);
  MvmProfScope prof__(MVM_TAG_MISC, stream);
  MvbaArgs g;
  memset(&g, 0, sizeof(g));
  g.n_views = n_views; g.n_pairs = n_pairs; g.batch = batch; g.n_pad = n_pad;
  for (int p = 0; p < n_pairs; ++p) { g.a[p] = pair_a[p]; g.b[p] = pair_b[p]; MVM_REQUIRE(0 <= pair_a[p] && pair_a[p] < pair_b[p] && pair_b[p] < n_views); }
  g.xa = xn_a; g.xb = xn_b; g.n_valid = n_valid; g.extr_init = extr;
  triangulate_pairs_kernel<<<batch * n_pairs, NT, 0, stream>>>(g, points_out);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}

}  // extern "C"
