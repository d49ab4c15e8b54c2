// GPU replacement of the reference's `ba_initializer` binary (ba_init.cpp:77-91 -> Theia
// RobustRotationEstimator + LeastUnsquaredDeviationPositionEstimator, default options), restated in
// oracle/ba_init.py.  One warp per tuple, fp64, everything in shared memory (<= 8 views, <= 28 pairs).
//
//   rotation averaging  residual_e = log(R_j^T R_ij R_i), A = (-I at view i, +I at view j), view 0 fixed
//       L1 phase   <= 5 x { ADMM for min |A d - r|_1 (rho = alpha = 1, 5 iterations doubling every pass,
//                           abs 1e-4 / rel 1e-2 stopping rule); R_v <- R_v exp(d_v); mean step <= 1e-3 stops }
//       IRLS phase <= 100 x { w_e = sigma / (|r_e|^2 + sigma^2)^2, sigma = 5 deg; (A^T W A) d = A^T W r }
//       A^T A is the graph Laplacian (x) I_3, so both phases only ever factor (views-1)^2 systems.
//   positions (LUD)     min sum_e |c_j - c_i - s_e d_e|  s.t. s_e >= 1, c_0 = 0, d_e = R_i^T position_2
//       IRLS (<= 40 reweightings, w_e = 1 / max(|res_e|, 1e-6)); each bounded weighted LS problem solved
//       exactly by an active set on s_e >= 1 with the free scales eliminated analytically
//       (3(views-1) unknowns, warp-cooperative Cholesky).
// Edge set = pairs the reference writes to ba_init_in.csv (bundle_adjust_io.py:181-190): successful
// pairs with >= 20 inliers or on the spanning tree.  If that graph does not reach every view the
// spanning-tree poses are returned unchanged.
#include "../../include/mvm_b200.h"
#include "common.cuh"
#include "kernels.cuh"
#include "linalg_small.cuh"

namespace {

constexpr int MV = MVM_MAX_VIEWS;      // 8
constexpr int ME = MVM_MAX_PAIRS;      // 28
constexpr int NR = 3 * ME;             // residual rows
constexpr int NU = 3 * (MV - 1);       // unknowns

struct BaInitArgs {
  int n_views, n_pairs, batch, n_pad, min_inliers;
  int a[ME], b[ME];
  const double* extr0;            // [B,T,16]
  const float* T_rel;             // [B,P,16]
  const unsigned char* success;   // [B,P]
  const unsigned char* on_tree;   // [B,P]
  const unsigned char* inliers;   // [B,P,n_pad]
  double* extr;                   // [B,T,16]
  int* n_edges;                   // [B] or null (debug)
};

__device__ inline void aa_mul(const double* a, const double* b, double* out) {
  double Ra[9], Rb[9], R[9];
  aa_to_R(a, Ra);
  aa_to_R(b, Rb);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) R[i * 3 + j] = Ra[i * 3] * Rb[j] + Ra[i * 3 + 1] * Rb[3 + j] + Ra[i * 3 + 2] * Rb[6 + j];
  R_to_aa(R, out);
}

__device__ inline double wsum(double v) { return warp_sum_d(v); }

__global__ void __launch_bounds__(32) ba_init_kernel(const __grid_constant__ BaInitArgs g) {
  __shared__ double rot[MV][3], prot[ME][3], ppos[ME][3], dirs[ME][3], cpos[MV][3], cprev[MV][3];
  __shared__ int ei[ME], ej[ME];
  __shared__ double GJ[(MV - 1) * 2 * (MV - 1)], Linv[(MV - 1) * (MV - 1)];
  __shared__ double r[NR], z[NR], u[NR], zold[NR], ax[NR];
  __shared__ double x[NU], y[NU];
  __shared__ double wgt[ME], sc[ME];
  __shared__ unsigned char act[ME];
  __shared__ double H[MAXU * MAXU], gv[MAXU];
  __shared__ int s_E, s_conn, s_flag;

  const int bi = blockIdx.x, lane = threadIdx.x;
  const int T = g.n_views, P = g.n_pairs, nf = T - 1;

  // ---- edges: successful pairs with >= min_inliers inliers or on the spanning tree ----
  if (lane == 0) s_E = 0;
  __syncwarp();
  for (int p = 0; p < P; ++p) {
    int cnt = 0;
    if (g.inliers) {   // null: the caller already decided the edge set (success && on_tree)
      const unsigned char* m = g.inliers + ((long long)bi * P + p) * g.n_pad;
      for (int i = lane; i < g.n_pad; i += 32) cnt += m[i];
    }
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0 && g.success[bi * P + p] && (cnt >= g.min_inliers || g.on_tree[bi * P + p])) {
      const int e = s_E++;
      ei[e] = g.a[p]; ej[e] = g.b[p];
      const float* Tr = g.T_rel + ((long long)bi * P + p) * 16;
      const double R[9] = {Tr[0], Tr[1], Tr[2], Tr[4], Tr[5], Tr[6], Tr[8], Tr[9], Tr[10]};
      R_to_aa(R, prot[e]);
      // position of camera b in camera a's frame: -R^T t   (bundle_adjust_io.py:186-187)
      for (int c = 0; c < 3; ++c) ppos[e][c] = -(R[c] * (double)Tr[3] + R[3 + c] * (double)Tr[7] + R[6 + c] * (double)Tr[11]);
    }
    __syncwarp();
  }
  const int E = s_E;
  if (lane < T) {
    const double* X = g.extr0 + ((long long)bi * T + lane) * 16;
    const double R[9] = {X[0], X[1], X[2], X[4], X[5], X[6], X[8], X[9], X[10]};
    R_to_aa(R, rot[lane]);
  }
  // connectivity from view 0
  if (lane == 0) {
    bool seen[MV];
    for (int v = 0; v < T; ++v) seen[v] = v == 0;
    for (int it = 0; it < T; ++it)
      for (int e = 0; e < E; ++e) {
        if (seen[ei[e]] && !seen[ej[e]]) seen[ej[e]] = true;
        if (seen[ej[e]] && !seen[ei[e]]) seen[ei[e]] = true;
      }
    int ok = 1;
    for (int v = 0; v < T; ++v) ok &= seen[v] ? 1 : 0;
    s_conn = ok;
    if (g.n_edges) g.n_edges[bi] = E;
  }
  __syncwarp();
  double* out = g.extr + (long long)bi * T * 16;
  if (!s_conn) {
    for (int i = lane; i < T * 16; i += 32) out[i] = g.extr0[(long long)bi * T * 16 + i];
    return;
  }
  const int m3 = 3 * E, n3 = 3 * nf;

  // weighted Laplacian of the free views -> inverse Linv (warp-cooperative Gauss-Jordan in shared memory;
  // the Laplacian of a connected graph with view 0 removed is SPD, so no pivoting is needed)
  auto build_laplacian_inverse = [&](const double* w) {
    const int nc2 = 2 * nf;
    for (int k = lane; k < nf * nc2; k += 32) GJ[k] = (k % nc2 == nf + k / nc2) ? 1.0 : 0.0;
    __syncwarp();
    for (int k = lane; k < nf * nf; k += 32) {
      const int a = k / nf + 1, b = k % nf + 1;
      double s = 0.0;
      for (int e = 0; e < E; ++e) {
        const double we = w ? w[e] : 1.0;
        if (a == b) { if (ei[e] == a || ej[e] == a) s += we; }
        else if ((ei[e] == a && ej[e] == b) || (ei[e] == b && ej[e] == a)) s -= we;
      }
      GJ[(a - 1) * nc2 + (b - 1)] = s;
    }
    __syncwarp();
    for (int k = 0; k < nf; ++k) {
      const double inv = 1.0 / GJ[k * nc2 + k];
      __syncwarp();
      for (int j = lane; j < nc2; j += 32) GJ[k * nc2 + j] *= inv;
      __syncwarp();
      for (int idx = lane; idx < nf * nc2; idx += 32) {
        const int i = idx / nc2, j = idx % nc2;
        if (i != k && j != k) GJ[idx] -= GJ[i * nc2 + k] * GJ[k * nc2 + j];
      }
      __syncwarp();
      for (int i = lane; i < nf; i += 32)
        if (i != k) GJ[i * nc2 + k] = 0.0;
      __syncwarp();
    }
    for (int k = lane; k < nf * nf; k += 32) Linv[k] = GJ[(k / nf) * nc2 + nf + k % nf];
    __syncwarp();
  };
  // y = A^T (w .* v)  (n3),  lanes over unknowns
  auto At_mul = [&](const double* v, const double* w, double* dst) {
    for (int k = lane; k < n3; k += 32) {
      const int view = k / 3 + 1, c = k % 3;
      double s = 0.0;
      for (int e = 0; e < E; ++e) {
        const double we = w ? w[e] : 1.0;
        if (ej[e] == view) s += we * v[3 * e + c];
        if (ei[e] == view) s -= we * v[3 * e + c];
      }
      dst[k] = s;
    }
    __syncwarp();
  };
  // x = (Linv (x) I3) y
  auto solve_normal = [&](const double* rhs, double* dst) {
    for (int k = lane; k < n3; k += 32) {
      const int vi = k / 3, c = k % 3;
      double s = 0.0;
      for (int l = 0; l < nf; ++l) s += Linv[vi * nf + l] * rhs[3 * l + c];
      dst[k] = s;
    }
    __syncwarp();
  };
  auto A_mul = [&](const double* xx, double* dst) {
    for (int k = lane; k < m3; k += 32) {
      const int e = k / 3, c = k % 3;
      double s = 0.0;
      if (ej[e] > 0) s += xx[3 * (ej[e] - 1) + c];
      if (ei[e] > 0) s -= xx[3 * (ei[e] - 1) + c];
      dst[k] = s;
    }
    __syncwarp();
  };
  auto residuals = [&]() {
    for (int e = lane; e < E; e += 32) {
      double t1[3], nr[3] = {-rot[ej[e]][0], -rot[ej[e]][1], -rot[ej[e]][2]};
      aa_mul(prot[e], rot[ei[e]], t1);
      aa_mul(nr, t1, &r[3 * e]);
    }
    __syncwarp();
  };
  // R_v <- R_v exp(step_v); returns the mean step norm
  auto update = [&](const double* step) {
    double sn = 0.0;
    if (lane >= 1 && lane < T) {
      const double* d = step + 3 * (lane - 1);
      double nr[3];
      aa_mul(rot[lane], d, nr);
      rot[lane][0] = nr[0]; rot[lane][1] = nr[1]; rot[lane][2] = nr[2];
      sn = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    }
    sn = wsum(sn) / nf;
    __syncwarp();
    return sn;
  };

  // ================= rotation averaging: L1 phase =================
  build_laplacian_inverse(nullptr);
  int admm_iters = 5;   // 5 ADMM iterations in the first pass, doubled in every following one
  for (int outer = 0; outer < 5; ++outer, admm_iters *= 2) {
    residuals();
    for (int k = lane; k < m3; k += 32) { z[k] = 0.0; u[k] = 0.0; }
    __syncwarp();
    for (int it = 0; it < admm_iters; ++it) {
      for (int k = lane; k < m3; k += 32) ax[k] = r[k] + z[k] - u[k];
      __syncwarp();
      At_mul(ax, nullptr, y);
      solve_normal(y, x);
      A_mul(x, ax);
      double n_ax = 0, n_z = 0, n_b = 0, n_r = 0;
      for (int k = lane; k < m3; k += 32) {
        zold[k] = z[k];
        const double v = ax[k] - r[k] + u[k];
        const double zn = (v > 1.0 ? v - 1.0 : (v < -1.0 ? v + 1.0 : 0.0));   // shrinkage, 1/rho = 1
        z[k] = zn;
        u[k] += ax[k] - zn - r[k];
        const double pr = ax[k] - zn - r[k];
        n_r += pr * pr; n_ax += ax[k] * ax[k]; n_z += zn * zn; n_b += r[k] * r[k];
      }
      __syncwarp();
      n_r = sqrt(wsum(n_r)); n_ax = sqrt(wsum(n_ax)); n_z = sqrt(wsum(n_z)); n_b = sqrt(wsum(n_b));
      // dual residual |A^T (z - zold)| and |A^T u|
      for (int k = lane; k < m3; k += 32) zold[k] = z[k] - zold[k];
      __syncwarp();
      At_mul(zold, nullptr, y);
      double n_s = 0;
      for (int k = lane; k < n3; k += 32) n_s += y[k] * y[k];
      n_s = sqrt(wsum(n_s));
      At_mul(u, nullptr, y);
      double n_u = 0;
      for (int k = lane; k < n3; k += 32) n_u += y[k] * y[k];
      n_u = sqrt(wsum(n_u));
      const double eps_pri = sqrt((double)m3) * 1e-4 + 1e-2 * fmax(n_ax, fmax(n_z, n_b));
      const double eps_dual = sqrt((double)n3) * 1e-4 + 1e-2 * n_u;
      if (n_r < eps_pri && n_s < eps_dual) break;
    }
    if (update(x) <= 1e-3) break;
  }
  // ================= rotation averaging: IRLS phase =================
  const double sigma = 5.0 * 3.14159265358979323846 / 180.0;
  for (int it = 0; it < 100; ++it) {
    residuals();
    for (int e = lane; e < E; e += 32) {
      const double e2 = r[3 * e] * r[3 * e] + r[3 * e + 1] * r[3 * e + 1] + r[3 * e + 2] * r[3 * e + 2];
      const double t = e2 + sigma * sigma;
      wgt[e] = sigma / (t * t);
    }
    __syncwarp();
    build_laplacian_inverse(wgt);
    At_mul(r, wgt, y);
    solve_normal(y, x);
    if (update(x) <= 1e-3) break;
  }

  // ================= positions: least unsquared deviations =================
  for (int e = lane; e < E; e += 32) {
    double R[9];
    aa_to_R(rot[ei[e]], R);
    for (int c = 0; c < 3; ++c) dirs[e][c] = R[c] * ppos[e][0] + R[3 + c] * ppos[e][1] + R[6 + c] * ppos[e][2];   // R^T p
    wgt[e] = 1.0;
  }
  for (int k = lane; k < 3 * MV; k += 32) { (&cpos[0][0])[k] = 0.0; (&cprev[0][0])[k] = 0.0; }
  __syncwarp();
  // active set of s_e >= 1: all active at the start, warm-started across the reweightings
  for (int e = lane; e < E; e += 32) { act[e] = 1; sc[e] = 1.0; }
  __syncwarp();
  for (int rw = 0; rw < 40; ++rw) {
    for (int as = 0; as < 2 * E + 2; ++as) {
      // H = sum_e w_e B_e^T Q_e B_e,  g = sum_active w_e B_e^T Q_e d_e
      for (int k = lane; k < n3 * n3; k += 32) {
        const int rr = k / n3, cc = k % n3;
        const int va = rr / 3 + 1, ca = rr % 3, vb = cc / 3 + 1, cb = cc % 3;
        double s = 0.0;
        for (int e = 0; e < E; ++e) {
          double sa = 0.0, sb = 0.0;
          if (ej[e] == va) sa = 1.0; else if (ei[e] == va) sa = -1.0;
          if (ej[e] == vb) sb = 1.0; else if (ei[e] == vb) sb = -1.0;
          if (sa == 0.0 || sb == 0.0) continue;
          const double dd = dirs[e][0] * dirs[e][0] + dirs[e][1] * dirs[e][1] + dirs[e][2] * dirs[e][2];
          const double q = (ca == cb ? 1.0 : 0.0) - (act[e] ? 0.0 : dirs[e][ca] * dirs[e][cb] / dd);
          s += sa * sb * wgt[e] * q;
        }
        H[rr * MAXU + cc] = s + (rr == cc ? 1e-12 : 0.0);
      }
      for (int k = lane; k < n3; k += 32) {
        const int va = k / 3 + 1, ca = k % 3;
        double s = 0.0;
        for (int e = 0; e < E; ++e) {
          if (!act[e]) continue;
          if (ej[e] == va) s += wgt[e] * dirs[e][ca];
          else if (ei[e] == va) s -= wgt[e] * dirs[e][ca];
        }
        gv[k] = s;
      }
      __syncwarp();
      chol_solve_warp(H, gv, n3, lane);
      for (int k = lane; k < n3; k += 32) cpos[k / 3 + 1][k % 3] = gv[k];
      __syncwarp();
      int changed = 0;
      for (int e = lane; e < E; e += 32) {
        const double dd = dirs[e][0] * dirs[e][0] + dirs[e][1] * dirs[e][1] + dirs[e][2] * dirs[e][2];
        double proj = 0.0;
        for (int c = 0; c < 3; ++c) proj += dirs[e][c] * (cpos[ej[e]][c] - cpos[ei[e]][c]);
        proj /= dd;
        if (!act[e]) {
          sc[e] = proj;
          if (proj < 1.0 - 1e-12) { act[e] = 1; sc[e] = 1.0; changed = 1; }
        } else {
          sc[e] = 1.0;
          if (proj > 1.0 + 1e-12) { act[e] = 0; changed = 1; }
        }
      }
      changed = __any_sync(0xffffffffu, changed);
      __syncwarp();
      if (!changed) break;
    }
    // reweight and test convergence
    double dmax = 0.0;
    for (int e = lane; e < E; e += 32) {
      double rs = 0.0;
      for (int c = 0; c < 3; ++c) {
        const double d = cpos[ej[e]][c] - cpos[ei[e]][c] - sc[e] * dirs[e][c];
        rs += d * d;
      }
      wgt[e] = 1.0 / fmax(sqrt(rs), 1e-6);
    }
    for (int k = lane; k < 3 * T; k += 32) {
      dmax = fmax(dmax, fabs((&cpos[0][0])[k] - (&cprev[0][0])[k]));
      (&cprev[0][0])[k] = (&cpos[0][0])[k];
    }
    for (int o = 16; o > 0; o >>= 1) dmax = fmax(dmax, __shfl_xor_sync(0xffffffffu, dmax, o));
    __syncwarp();
    if (rw > 0 && dmax < 1e-9) break;
  }

  // ---- world->cam extrinsics: R_v, t_v = -R_v c_v  (ba_init.cpp:58-75) ----
  if (lane < T) {
    double R[9];
    aa_to_R(rot[lane], R);
    double* X = out + lane * 16;
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) X[i * 4 + j] = R[i * 3 + j];
      X[i * 4 + 3] = -(R[i * 3] * cpos[lane][0] + R[i * 3 + 1] * cpos[lane][1] + R[i * 3 + 2] * cpos[lane][2]);
    }
    X[12] = 0; X[13] = 0; X[14] = 0; X[15] = 1;
  }
}

}  // namespace

extern "C" int mvm_ba_initialize(const int* pair_a, const int* pair_b, int n_views, int n_pairs, int batch,
                                 int n_pad, const double* extr_tree, const float* T_rel,
                                 const unsigned char* success, const unsigned char* on_tree,
                                 const unsigned char* inliers, int min_inliers, double* extr_out,
                                 int* n_edges_out, void* stream) {
  MVM_REQUIRE(pair_a && pair_b && extr_tree && T_rel && success && on_tree && extr_out);
  MVM_REQUIRE(n_views >= 2 && n_views <= MVM_MAX_VIEWS && n_pairs >= 1 && n_pairs <= MVM_MAX_PAIRS && batch >= 1);
  MvmProfScope prof__(MVM_TAG_MISC, (cudaStream_t)stream);
  BaInitArgs g;
  g.n_views = n_views; g.n_pairs = n_pairs; g.batch = batch; g.n_pad = n_pad; g.min_inliers = min_inliers;
  for (int p = 0; p < n_pairs; ++p) { g.a[p] = pair_a[p]; g.b[p] = pair_b[p]; MVM_REQUIRE(0 <= pair_a[p] && pair_a[p] < pair_b[p] && pair_b[p] < n_views); }
  g.extr0 = extr_tree; g.T_rel = T_rel; g.success = success; g.on_tree = on_tree; g.inliers = inliers;
  g.extr = extr_out; g.n_edges = n_edges_out;
  ba_init_kernel<<<batch, 32, 0, (cudaStream_t)stream>>>(g);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}
