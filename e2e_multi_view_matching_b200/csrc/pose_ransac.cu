// Two-view RANSAC on essential matrices with cheirality pose recovery, one CTA per pair problem, fp64 on chip.
// Semantics: the reference's estimate_pose (models/models/utils.py:288-312), i.e. OpenCV's
// findEssentialMat(method=RANSAC) followed by recoverPose, restated in tests/ransac_oracle.py:
//  * hypotheses come from a counter-based sampler (splitmix64 of seed, hypothesis, draw, attempt; never of the batch
//    item, so item i of a batch equals a batch-of-one launch) and the five-point solver (null space by Householder QR,
//    the ten cubic constraints of an essential matrix, Gauss-Jordan on the 10 x 20 system, real roots of the degree-10
//    determinant found by isolating them between the roots of its derivatives);
//  * hypotheses are generated and scored in rounds of ROUND (a warp per minimal problem, the whole CTA scores every
//    model of the round), then one thread walks the round in hypothesis order exactly like OpenCV's sequential loop:
//    strictly-greater-than-max(best, 4) replacement, RANSACUpdateNumIters after each improvement, stop when the
//    hypothesis index reaches the iteration bound.  The result is the sequential algorithm's; at most one round of
//    work past the stopping point is wasted;
//  * recoverPose (distanceThresh 50, see DIST) on the chosen E and the RANSAC mask, which it rewrites in place (the
//    Python binding's behaviour); with exactly five points every solution is tried in turn, each seeing the mask the
//    previous call left, the strictly largest count wins.
#include <cfloat>

#include "../../include/mvm_b200.h"
#include "common.cuh"
#include "linalg_small.cuh"

namespace {

constexpr int NT = 256;
constexpr int NW = NT / 32;
constexpr int ROUND = 32;            // hypotheses per round
constexpr int MAXSOL = 10;           // real solutions of the five-point problem
constexpr int MAX_N = 2048;          // points held in shared memory (32 bytes each)
constexpr int MAX_ATTEMPTS = 64;     // redraws of one sample index (tests/ransac_oracle.py: MAX_ATTEMPTS)
constexpr double DIST = 50.0;        // recoverPose's distanceThresh as estimate_pose gets it: its positional 1e9
                                     // lands in the R slot of the (E, p1, p2, K[, R[, t[, mask]]]) overload, whose
                                     // threshold is OpenCV's fixed 50

// products of monomials x^a y^b z^c: linear [x, y, z, 1] x linear -> quadratic
// [x2, y2, z2, xy, xz, yz, x, y, z, 1]; quadratic x linear -> cubic in the order of Nister's elimination
// [x3, y3, x2y, xy2, x2z, x2, y2z, y2, xyz, xy | xz2, xz, x, yz2, yz, y, z3, z2, z, 1]
__constant__ unsigned char c_mul11[4][4] = {{0, 3, 4, 6}, {3, 1, 5, 7}, {4, 5, 2, 8}, {6, 7, 8, 9}};
__constant__ unsigned char c_mul21[10][4] = {{0, 2, 4, 5},     {3, 1, 6, 7},     {10, 13, 16, 17}, {2, 3, 8, 9},
                                             {4, 8, 10, 11},   {8, 6, 13, 14},   {5, 9, 11, 12},   {9, 7, 14, 15},
                                             {11, 14, 17, 18}, {12, 15, 18, 19}};

struct WarpScratch {
  double basis[36];     // X, Y, Z, W (E = x X + y Y + z Z + W), 9 entries each, row-major E
  double eet[90];       // E E^T: 9 quadratic polynomials
  double M[200];        // 10 x 20 constraint system (first 45 entries double as the QR workspace)
  double hv[45];        // Householder vectors
  double bz[39];        // B(z): 3 rows of x-coef [4] | y-coef [4] | constant [5], ascending powers
  double poly[11];      // det B(z)
  double q[11];         // current derivative of poly
  double crit[12];      // real roots of the previous derivative, ascending
  int flags;
  int idx[5];
};

struct RansacArgs {
  const float* kpts0; const float* kpts1; const float* intr0; const float* intr1;
  const int* n_valid;
  int N;
  float thresh_px; double prob; int max_iters;
  unsigned long long seed_key;
  float* T021; float* k0n; float* k1n;
  unsigned char* inliers; int* n_inliers;
  double* E_out; int* n_models; int* iterations; unsigned char* success;
};

__host__ __device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
  unsigned long long z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// five distinct indices in [0, n) for hypothesis hyp; false when MAX_ATTEMPTS redraws find no new index
__device__ bool sample5(unsigned long long seed_key, unsigned long long hyp, int n, int* idx) {
  const unsigned long long k0 = splitmix64(seed_key ^ hyp);
  for (int d = 0; d < 5; ++d) {
    bool found = false;
    for (int a = 0; a < MAX_ATTEMPTS && !found; ++a) {
      const int i = (int)(splitmix64(k0 ^ (((unsigned long long)d << 32) | (unsigned)a)) % (unsigned long long)n);
      bool dup = false;
      for (int e = 0; e < d; ++e) dup |= idx[e] == i;
      if (!dup) { idx[d] = i; found = true; }
    }
    if (!found) return false;
  }
  return true;
}

__device__ __forceinline__ void m11_acc(const double* a, const double* b, double s, double* out) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) out[c_mul11[i][j]] += s * a[i] * b[j];
}
__device__ __forceinline__ void m21_acc(const double* a, const double* b, double s, double* out) {
#pragma unroll
  for (int i = 0; i < 10; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) out[c_mul21[i][j]] += s * a[i] * b[j];
}
__device__ __forceinline__ void ebasis(const double* basis, int e, double* p) {
  p[0] = basis[e]; p[1] = basis[9 + e]; p[2] = basis[18 + e]; p[3] = basis[27 + e];
}

// c += s * a * b for ascending coefficient arrays
__device__ __forceinline__ void pmul_acc(const double* a, int na, const double* b, int nb, double s, double* c) {
  for (int i = 0; i < na; ++i)
    for (int j = 0; j < nb; ++j) c[i + j] += s * a[i] * b[j];
}

__device__ __forceinline__ double horner(const double* c, int deg, double x) {
  double s = c[deg];
  for (int i = deg - 1; i >= 0; --i) s = s * x + c[i];
  return s;
}

// the root of the polynomial q (degree deg, monotone on [lo, hi], sign change inside): Newton steps safeguarded by the
// shrinking bracket, bisection whenever a step would leave it or would not at least halve the previous step (a far
// start on a steep high-degree polynomial otherwise creeps in by 1/deg per step)
__device__ double bracketed_root(const double* q, int deg, double lo, double hi, double flo) {
  double x = 0.5 * (lo + hi), dxold = hi - lo, dx = dxold;
  for (int it = 0; it < 200; ++it) {
    double f = q[deg], df = 0.0;
    for (int i = deg - 1; i >= 0; --i) { df = df * x + f; f = f * x + q[i]; }
    if (f == 0.0) break;
    if ((f < 0.0) == (flo < 0.0)) lo = x; else hi = x;
    const double xn = x - f / df;
    if (!(xn > lo && xn < hi) || fabs(2.0 * f) > fabs(dxold * df)) {
      dxold = dx;
      dx = 0.5 * (hi - lo);
      x = lo + dx;
      if (!(x > lo && x < hi)) break;             // bracket down to adjacent doubles
    } else {
      dxold = dx;
      dx = x - xn;
      x = xn;
      if (fabs(dx) <= 1e-16 * fabs(x)) break;
    }
  }
  return x;
}

// the ten cubic constraints of an essential matrix at E (2 E E' E - tr(E E') E row-major, det E) or, with D, their
// derivative along D (tests/ransac_oracle.py: essential_constraints)
__device__ void essential_constraints(const double* E, const double* D, double* r) {
  double EEt[9], EtE[9], trEEt = 0.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double a = 0.0, b = 0.0;
      for (int k = 0; k < 3; ++k) { a += E[i * 3 + k] * E[j * 3 + k]; b += E[k * 3 + i] * E[k * 3 + j]; }
      EEt[i * 3 + j] = a; EtE[i * 3 + j] = b;
    }
  trEEt = EEt[0] + EEt[4] + EEt[8];
  const double cof[9] = {E[4] * E[8] - E[5] * E[7], E[5] * E[6] - E[3] * E[8], E[3] * E[7] - E[4] * E[6],
                         E[2] * E[7] - E[1] * E[8], E[0] * E[8] - E[2] * E[6], E[1] * E[6] - E[0] * E[7],
                         E[1] * E[5] - E[2] * E[4], E[2] * E[3] - E[0] * E[5], E[0] * E[4] - E[1] * E[3]};
  if (!D) {
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        double s = 0.0;
        for (int k = 0; k < 3; ++k) s += EEt[i * 3 + k] * E[k * 3 + j];
        r[i * 3 + j] = 2.0 * s - trEEt * E[i * 3 + j];
      }
    r[9] = E[0] * cof[0] + E[1] * cof[1] + E[2] * cof[2];
    return;
  }
  // d(2 E E' E - tr(E E') E) = 2 (D E'E + E D' E + E E' D) - 2 tr(D E') E - tr(E E') D;  d det = sum cof . D
  double trDEt = 0.0, EDt[9];
  for (int e = 0; e < 9; ++e) trDEt += D[e] * E[e];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double a = 0.0;
      for (int k = 0; k < 3; ++k) a += E[i * 3 + k] * D[j * 3 + k];
      EDt[i * 3 + j] = a;
    }
  double dd = 0.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0.0;
      for (int k = 0; k < 3; ++k)
        s += D[i * 3 + k] * EtE[k * 3 + j] + EDt[i * 3 + k] * E[k * 3 + j] + EEt[i * 3 + k] * D[k * 3 + j];
      r[i * 3 + j] = 2.0 * s - 2.0 * trDEt * E[i * 3 + j] - trEEt * D[i * 3 + j];
      dd += cof[i * 3 + j] * D[i * 3 + j];
    }
  r[9] = dd;
}

constexpr int REFINE_STEPS = 3;   // tests/ransac_oracle.py: REFINE_STEPS

// Gauss-Newton steps on the ten constraints in (x, y, z), each kept only when it lowers the squared residual: the
// elimination loses digits on sets with close roots, the constraints themselves do not
__device__ __noinline__ void refine_xyz(const double* basis, double* p) {
  double E[9], r[10], rr = 0.0;
  for (int e = 0; e < 9; ++e) E[e] = p[0] * basis[e] + p[1] * basis[9 + e] + p[2] * basis[18 + e] + basis[27 + e];
  essential_constraints(E, nullptr, r);
  for (int i = 0; i < 10; ++i) rr += r[i] * r[i];
  for (int it = 0; it < REFINE_STEPS; ++it) {
    double J[3][10];
    for (int c = 0; c < 3; ++c) essential_constraints(E, basis + 9 * c, J[c]);
    double A[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
    for (int i = 0; i < 10; ++i) {
      A[0] += J[0][i] * J[0][i]; A[1] += J[0][i] * J[1][i]; A[2] += J[0][i] * J[2][i];
      A[3] += J[1][i] * J[1][i]; A[4] += J[1][i] * J[2][i]; A[5] += J[2][i] * J[2][i];
      for (int c = 0; c < 3; ++c) g[c] += J[c][i] * r[i];
    }
    double inv[6];
    if (!inv3_sym(A, inv)) break;
    const double pn[3] = {p[0] - (inv[0] * g[0] + inv[1] * g[1] + inv[2] * g[2]),
                          p[1] - (inv[1] * g[0] + inv[3] * g[1] + inv[4] * g[2]),
                          p[2] - (inv[2] * g[0] + inv[4] * g[1] + inv[5] * g[2])};
    double En[9], rn[10], rrn = 0.0;
    for (int e = 0; e < 9; ++e) En[e] = pn[0] * basis[e] + pn[1] * basis[9 + e] + pn[2] * basis[18 + e] + basis[27 + e];
    essential_constraints(En, nullptr, rn);
    for (int i = 0; i < 10; ++i) rrn += rn[i] * rn[i];
    if (!(rrn < rr)) break;
    for (int c = 0; c < 3; ++c) p[c] = pn[c];
    for (int e = 0; e < 9; ++e) E[e] = En[e];
    for (int i = 0; i < 10; ++i) r[i] = rn[i];
    rr = rrn;
  }
}

// All real essential matrices through the five correspondences ws.idx of pts ([n][4] = x1, y1, x2, y2), written to
// models (unit Frobenius norm, largest entry positive, ascending hidden variable z).  All 32 lanes call; returns the
// number of solutions (uniform).
__device__ int five_point_warp(WarpScratch& ws, const double* pts, double* models, int lane) {
  // 1. null space of the 5 x 9 epipolar system: Householder QR of its transpose (9 x 5), last four columns of Q
  if (lane == 0) {
    double* A = ws.M;   // A[r * 5 + c] = coefficient r of point c
    for (int c = 0; c < 5; ++c) {
      const double* p = pts + 4 * ws.idx[c];
      const double u1 = p[0], v1 = p[1], u2 = p[2], v2 = p[3];
      const double row[9] = {u2 * u1, u2 * v1, u2, v2 * u1, v2 * v1, v2, u1, v1, 1.0};
      for (int r = 0; r < 9; ++r) A[r * 5 + c] = row[r];
    }
    for (int k = 0; k < 5; ++k) {
      double nrm = 0.0;
      for (int r = k; r < 9; ++r) nrm += A[r * 5 + k] * A[r * 5 + k];
      nrm = sqrt(nrm);
      const double alpha = A[k * 5 + k] > 0.0 ? -nrm : nrm;
      double* v = ws.hv + k * 9;
      for (int r = 0; r < 9; ++r) v[r] = r < k ? 0.0 : A[r * 5 + k];
      v[k] -= alpha;
      double vv = 0.0;
      for (int r = k; r < 9; ++r) vv += v[r] * v[r];
      const double inv = vv > 0.0 ? 2.0 / vv : 0.0;
      for (int r = 0; r < 9; ++r) v[r] *= sqrt(inv);   // H_k = I - v v^T
      for (int c = k; c < 5; ++c) {
        double s = 0.0;
        for (int r = k; r < 9; ++r) s += v[r] * A[r * 5 + c];
        for (int r = k; r < 9; ++r) A[r * 5 + c] -= s * v[r];
      }
    }
    for (int j = 0; j < 4; ++j) {
      double y[9];
      for (int r = 0; r < 9; ++r) y[r] = r == 5 + j ? 1.0 : 0.0;
      for (int k = 4; k >= 0; --k) {
        const double* v = ws.hv + k * 9;
        double s = 0.0;
        for (int r = 0; r < 9; ++r) s += v[r] * y[r];
        for (int r = 0; r < 9; ++r) y[r] -= s * v[r];
      }
      for (int r = 0; r < 9; ++r) ws.basis[j * 9 + r] = y[r];
    }
  }
  __syncwarp();
  // 2. E E^T as quadratic polynomials (lane l < 9: entry (l / 3, l % 3))
  if (lane < 9) {
    const int i = lane / 3, j = lane % 3;
    double acc[10];
#pragma unroll
    for (int e = 0; e < 10; ++e) acc[e] = 0.0;
    for (int k = 0; k < 3; ++k) {
      double a[4], b[4];
      ebasis(ws.basis, i * 3 + k, a);
      ebasis(ws.basis, j * 3 + k, b);
      m11_acc(a, b, 1.0, acc);
    }
    for (int e = 0; e < 10; ++e) ws.eet[lane * 10 + e] = acc[e];
  }
  __syncwarp();
  // 3. the ten cubic constraints (lane r < 9: entry r of 2 E E^T E - tr(E E^T) E; lane 9: det E)
  if (lane < 10) {
    double acc[20];
#pragma unroll
    for (int e = 0; e < 20; ++e) acc[e] = 0.0;
    if (lane < 9) {
      const int i = lane / 3, j = lane % 3;
      double tr[10], b[4];
      for (int e = 0; e < 10; ++e) tr[e] = ws.eet[e] + ws.eet[40 + e] + ws.eet[80 + e];
      ebasis(ws.basis, i * 3 + j, b);
      m21_acc(tr, b, -1.0, acc);
      for (int k = 0; k < 3; ++k) {
        ebasis(ws.basis, k * 3 + j, b);
        m21_acc(ws.eet + (i * 3 + k) * 10, b, 2.0, acc);
      }
    } else {
      double e[9][4];
      for (int k = 0; k < 9; ++k) ebasis(ws.basis, k, e[k]);
      const int cof[3][4] = {{4, 8, 5, 7}, {3, 8, 5, 6}, {3, 7, 4, 6}};   // minors of row 0
      const double sg[3] = {1.0, -1.0, 1.0};
      for (int c = 0; c < 3; ++c) {
        double m[10];
        for (int t = 0; t < 10; ++t) m[t] = 0.0;
        m11_acc(e[cof[c][0]], e[cof[c][1]], 1.0, m);
        m11_acc(e[cof[c][2]], e[cof[c][3]], -1.0, m);
        m21_acc(m, e[c], sg[c], acc);
      }
    }
    for (int e = 0; e < 20; ++e) ws.M[lane * 20 + e] = acc[e];
  }
  __syncwarp();
  // 4. Gauss-Jordan with partial pivoting, lane c < 20 owns column c
  bool ok = true;
  for (int k = 0; k < 10; ++k) {
    int p = k;
    double best = fabs(ws.M[k * 20 + k]);
    for (int r = k + 1; r < 10; ++r)
      if (fabs(ws.M[r * 20 + k]) > best) { best = fabs(ws.M[r * 20 + k]); p = r; }
    if (!(best > 0.0) || !isfinite(best)) { ok = false; break; }
    double colk[10];
#pragma unroll
    for (int r = 0; r < 10; ++r) colk[r] = ws.M[r * 20 + k];
    __syncwarp();
    {
      const double t = colk[k]; colk[k] = colk[p]; colk[p] = t;   // p >= k: the swap is a select
    }
    if (lane < 20) {
      double* col = ws.M + lane;
      if (p != k) { const double t = col[k * 20]; col[k * 20] = col[p * 20]; col[p * 20] = t; }
      const double rk = col[k * 20] / colk[k];
      col[k * 20] = rk;
#pragma unroll
      for (int r = 0; r < 10; ++r)
        if (r != k) col[r * 20] -= colk[r] * rk;
    }
    __syncwarp();
  }
  if (!ok) return 0;
  // 5. B(z) and its determinant
  if (lane == 0) {
    for (int a = 0; a < 3; ++a) {
      const double* ga = ws.M + (4 + 2 * a) * 20 + 10;
      const double* gb = ga + 20;
      double* b = ws.bz + a * 13;
      b[0] = ga[2]; b[1] = ga[1] - gb[2]; b[2] = ga[0] - gb[1]; b[3] = -gb[0];
      b[4] = ga[5]; b[5] = ga[4] - gb[5]; b[6] = ga[3] - gb[4]; b[7] = -gb[3];
      b[8] = ga[9]; b[9] = ga[8] - gb[9]; b[10] = ga[7] - gb[8]; b[11] = ga[6] - gb[7]; b[12] = -gb[6];
    }
    const double *bx0 = ws.bz, *by0 = ws.bz + 4, *bc0 = ws.bz + 8;
    const double *bx1 = ws.bz + 13, *by1 = ws.bz + 17, *bc1 = ws.bz + 21;
    const double *bx2 = ws.bz + 26, *by2 = ws.bz + 30, *bc2 = ws.bz + 34;
    double m1[8], m2[8], m3[7];
    for (int i = 0; i < 8; ++i) { m1[i] = 0.0; m2[i] = 0.0; }
    for (int i = 0; i < 7; ++i) m3[i] = 0.0;
    pmul_acc(by1, 4, bc2, 5, 1.0, m1); pmul_acc(bc1, 5, by2, 4, -1.0, m1);
    pmul_acc(bx1, 4, bc2, 5, 1.0, m2); pmul_acc(bc1, 5, bx2, 4, -1.0, m2);
    pmul_acc(bx1, 4, by2, 4, 1.0, m3); pmul_acc(by1, 4, bx2, 4, -1.0, m3);
    double* d = ws.poly;
    for (int i = 0; i < 11; ++i) d[i] = 0.0;
    pmul_acc(bx0, 4, m1, 8, 1.0, d);
    pmul_acc(by0, 4, m2, 8, -1.0, d);
    pmul_acc(bc0, 5, m3, 7, 1.0, d);
    int deg = -1;
    bool fin = true;
    for (int i = 0; i < 11; ++i) { fin &= isfinite(d[i]); if (d[i] != 0.0) deg = i; }
    double bound = 0.0;
    if (fin && deg >= 1) {
      for (int i = 0; i < deg; ++i) bound = fmax(bound, fabs(d[i] / d[deg]));
      bound += 1.0;
    }
    ws.flags = (fin && deg >= 1 && isfinite(bound)) ? deg : 0;
    ws.crit[0] = bound;   // passed to the lanes below
  }
  __syncwarp();
  const int deg = ws.flags;
  if (deg == 0) return 0;
  const double bound = ws.crit[0];
  // 6. real roots: the roots of the k-th derivative split [-bound, bound] into intervals on which the (k-1)-th is
  //    monotone; one lane per interval, from the linear derivative down to the polynomial itself
  int ncrit = 0;
  for (int k = deg - 1; k >= 0; --k) {
    const int dk = deg - k;
    if (lane <= dk) {
      double ff = 1.0;
      for (int j = lane + 1; j <= lane + k; ++j) ff *= (double)j;
      ws.q[lane] = ws.poly[lane + k] * ff;
    }
    __syncwarp();
    const int nint = ncrit + 1;
    bool has = false;
    double root = 0.0;
    if (lane < nint) {
      const double a = lane == 0 ? -bound : ws.crit[lane - 1];
      const double b = lane == ncrit ? bound : ws.crit[lane];
      const double qa = horner(ws.q, dk, a), qb = horner(ws.q, dk, b);
      has = (qa < 0.0 && qb >= 0.0) || (qa > 0.0 && qb <= 0.0);
      if (has) root = qb == 0.0 ? b : (dk == 1 ? fmin(fmax(-ws.q[0] / ws.q[1], a), b) : bracketed_root(ws.q, dk, a, b, qa));
      if (has && k == 0) {
        // polish on the polynomial itself: Newton steps kept while they reduce |p|
        for (int it = 0; it < 3; ++it) {
          double f = ws.q[dk], df = 0.0;
          for (int i = dk - 1; i >= 0; --i) { df = df * root + f; f = f * root + ws.q[i]; }
          if (f == 0.0 || df == 0.0) break;
          const double xn = root - f / df;
          if (!(fabs(horner(ws.q, dk, xn)) < fabs(f))) break;
          root = xn;
        }
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, has);
    __syncwarp();
    if (has) ws.crit[__popc(bal & ((1u << lane) - 1u))] = root;
    ncrit = __popc(bal);
    __syncwarp();
  }
  // 7. x, y from the null vector of B(z), (x, y, z) refined on the constraints; E = x X + y Y + z Z + W
  bool valid = false;
  double E[9];
  if (lane < ncrit) {
    const double z = ws.crit[lane];
    double B[3][3];
    for (int a = 0; a < 3; ++a) {
      const double* b = ws.bz + a * 13;
      B[a][0] = horner(b, 3, z); B[a][1] = horner(b + 4, 3, z); B[a][2] = horner(b + 8, 4, z);
    }
    const int pr[3][2] = {{0, 1}, {0, 2}, {1, 2}};
    double c[3] = {0.0, 0.0, 0.0};
    for (int s = 0; s < 3; ++s) {
      const double* r0 = B[pr[s][0]];
      const double* r1 = B[pr[s][1]];
      const double cc[3] = {r0[1] * r1[2] - r0[2] * r1[1], r0[2] * r1[0] - r0[0] * r1[2], r0[0] * r1[1] - r0[1] * r1[0]};
      if (fabs(cc[2]) > fabs(c[2])) { c[0] = cc[0]; c[1] = cc[1]; c[2] = cc[2]; }
    }
    if (c[2] != 0.0) {
      double p[3] = {c[0] / c[2], c[1] / c[2], z};
      refine_xyz(ws.basis, p);
      double nrm = 0.0;
      for (int e = 0; e < 9; ++e) {
        E[e] = p[0] * ws.basis[e] + p[1] * ws.basis[9 + e] + p[2] * ws.basis[18 + e] + ws.basis[27 + e];
        nrm += E[e] * E[e];
      }
      nrm = sqrt(nrm);
      if (nrm > 0.0 && isfinite(nrm)) {
        int kmax = 0;
        for (int e = 1; e < 9; ++e)
          if (fabs(E[e]) > fabs(E[kmax])) kmax = e;
        const double s = (E[kmax] > 0.0 ? 1.0 : -1.0) / nrm;
        for (int e = 0; e < 9; ++e) E[e] *= s;
        valid = true;
      }
    }
  }
  const unsigned vb = __ballot_sync(0xffffffffu, valid);
  if (valid) {
    double* out = models + 9 * __popc(vb & ((1u << lane) - 1u));
    for (int e = 0; e < 9; ++e) out[e] = E[e];
  }
  __syncwarp();
  return __popc(vb);
}

__device__ __forceinline__ bool is_inlier(const double* E, const double* p, float thr2) {
  const double u1 = p[0], v1 = p[1], u2 = p[2], v2 = p[3];
  const double a0 = E[0] * u1 + E[1] * v1 + E[2];
  const double a1 = E[3] * u1 + E[4] * v1 + E[5];
  const double a2 = E[6] * u1 + E[7] * v1 + E[8];
  const double b0 = E[0] * u2 + E[3] * v2 + E[6];
  const double b1 = E[1] * u2 + E[4] * v2 + E[7];
  const double num = u2 * a0 + v2 * a1 + a2;
  const float err = (float)(num * num / (a0 * a0 + a1 * a1 + b0 * b0 + b1 * b1));
  return err <= thr2;
}

// RANSACUpdateNumIters
__device__ int update_num_iters(double p, double ep, int model_points, int max_iters) {
  p = fmin(fmax(p, 0.0), 1.0);
  ep = fmin(fmax(ep, 0.0), 1.0);
  double num = fmax(1.0 - p, DBL_MIN);
  double denom = 1.0 - pow(1.0 - ep, (double)model_points);
  if (denom < DBL_MIN) return 0;
  num = log(num);
  denom = log(denom);
  return (denom >= 0.0 || -num >= max_iters * (-denom)) ? max_iters : __double2int_rn(num / denom);
}

// cv::decomposeEssentialMat: R1 = U W Vt, R2 = U W^T Vt, t = U[:, 2], W = [[0,1,0],[-1,0,0],[0,0,1]], with
// det U = det Vt = +1
__device__ void decompose_essential(const double* E, double* R1, double* R2, double* t) {
  double a[3][3], v[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0.0;
      for (int k = 0; k < 3; ++k) s += E[k * 3 + i] * E[k * 3 + j];
      a[i][j] = s;
    }
  jacobi_eig_reg<3, 10>(a, v);
  int o[3] = {0, 1, 2};
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2 - i; ++j)
      if (a[o[j]][o[j]] < a[o[j + 1]][o[j + 1]]) { const int tt = o[j]; o[j] = o[j + 1]; o[j + 1] = tt; }
  double vc[3][3], u[3][3];
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) vc[c][r] = v[r][o[c]];
  // v0, v1 with their largest entry positive, v2 = v0 x v1 (det Vt = +1)
  for (int c = 0; c < 2; ++c) {
    int m = 0;
    for (int r = 1; r < 3; ++r)
      if (fabs(vc[c][r]) > fabs(vc[c][m])) m = r;
    if (vc[c][m] < 0.0)
      for (int r = 0; r < 3; ++r) vc[c][r] = -vc[c][r];
  }
  vc[2][0] = vc[0][1] * vc[1][2] - vc[0][2] * vc[1][1];
  vc[2][1] = vc[0][2] * vc[1][0] - vc[0][0] * vc[1][2];
  vc[2][2] = vc[0][0] * vc[1][1] - vc[0][1] * vc[1][0];
  for (int c = 0; c < 2; ++c) {
    double n = 0.0;
    for (int r = 0; r < 3; ++r) {
      u[c][r] = E[r * 3] * vc[c][0] + E[r * 3 + 1] * vc[c][1] + E[r * 3 + 2] * vc[c][2];
    }
    if (c == 1) {
      const double d = u[0][0] * u[1][0] + u[0][1] * u[1][1] + u[0][2] * u[1][2];
      for (int r = 0; r < 3; ++r) u[1][r] -= d * u[0][r];
    }
    for (int r = 0; r < 3; ++r) n += u[c][r] * u[c][r];
    n = sqrt(n);
    for (int r = 0; r < 3; ++r) u[c][r] /= n;
  }
  u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
  u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
  u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      R1[i * 3 + j] = -u[1][i] * vc[0][j] + u[0][i] * vc[1][j] + u[2][i] * vc[2][j];
      R2[i * 3 + j] = u[1][i] * vc[0][j] - u[0][i] * vc[1][j] + u[2][i] * vc[2][j];
    }
  // E's two equal singular values leave the orientation of (v0, v1), hence the sign of t and the R1 / R2 labels, to
  // rounding: fix them (t with its largest entry positive, R1 the one of larger trace), as the oracle does
  int m = 0;
  for (int r = 1; r < 3; ++r)
    if (fabs(u[2][r]) > fabs(u[2][m])) m = r;
  const double st = u[2][m] < 0.0 ? -1.0 : 1.0;
  for (int r = 0; r < 3; ++r) t[r] = st * u[2][r];
  if (R1[0] + R1[4] + R1[8] < R2[0] + R2[4] + R2[8])
    for (int e = 0; e < 9; ++e) { const double tmp = R1[e]; R1[e] = R2[e]; R2[e] = tmp; }
}

// cv::triangulatePoints with P0 = [I|0], P1 = [R|t] (smallest eigenvector of the 4 x 4 DLT normal matrix, not
// de-homogenised) and recoverPose's test: positive depth below DIST in both cameras
__device__ bool cheirality_ok(const double* R, const double* t, const double* p) {
  const double x1 = p[0], y1 = p[1], x2 = p[2], y2 = p[3];
  double A[4][4];
  A[0][0] = -1.0; A[0][1] = 0.0;  A[0][2] = x1; A[0][3] = 0.0;
  A[1][0] = 0.0;  A[1][1] = -1.0; A[1][2] = y1; A[1][3] = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    A[2][i] = x2 * R[6 + i] - R[i];
    A[3][i] = y2 * R[6 + i] - R[3 + i];
  }
  A[2][3] = x2 * t[2] - t[0];
  A[3][3] = y2 * t[2] - t[1];
  double M[4][4], V[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double s = 0.0;
#pragma unroll
      for (int k = 0; k < 4; ++k) s += A[k][i] * A[k][j];
      M[i][j] = s;
    }
  jacobi_eig_reg<4, 8>(M, V);
  const int m = argmin_diag<4>(M);
  double h[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    h[i] = V[i][0];
    if (m == 1) h[i] = V[i][1];
    if (m == 2) h[i] = V[i][2];
    if (m == 3) h[i] = V[i][3];
  }
  if (!(h[2] * h[3] > 0.0)) return false;
  const double X0 = h[0] / h[3], X1 = h[1] / h[3], X2 = h[2] / h[3];
  if (!(X2 < DIST)) return false;
  const double z1 = R[6] * X0 + R[7] * X1 + R[8] * X2 + t[2];
  return z1 > 0.0 && z1 < DIST;
}

struct PoseShared {
  double R[2][9], t[3];
  int cnt[4];
  int choice;
};

// recoverPose(E, x1, x2, I, DIST, mask): mask [n] (global, written by this block) is read and rewritten in place.
// Every thread returns the count of the chosen candidate; ps.R / ps.t / ps.choice describe it.
__device__ int recover_pose_block(const double* E, const double* pts, int n, unsigned char* mask, PoseShared& ps) {
  const int tid = threadIdx.x, lane = tid & 31;
  if (tid == 0) {
    decompose_essential(E, ps.R[0], ps.R[1], ps.t);
    for (int c = 0; c < 4; ++c) ps.cnt[c] = 0;
  }
  __syncthreads();
  unsigned bits = 0;    // 4 candidate bits per point of this thread (n <= 8 NT)
  int cnt[4] = {0, 0, 0, 0};
  for (int j = 0, i = tid; i < n; ++j, i += NT) {
    if (!mask[i]) continue;
#pragma unroll 1
    for (int c = 0; c < 4; ++c) {
      const double sg = c < 2 ? 1.0 : -1.0;     // R1,t / R2,t / R1,-t / R2,-t
      const double t[3] = {sg * ps.t[0], sg * ps.t[1], sg * ps.t[2]};
      if (cheirality_ok(ps.R[c & 1], t, pts + 4 * i)) { bits |= 1u << (4 * j + c); cnt[c]++; }
    }
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    int v = cnt[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0 && v) atomicAdd(&ps.cnt[c], v);
  }
  __syncthreads();
  if (tid == 0) {
    int bc = 0;
    for (int c = 1; c < 4; ++c)
      if (ps.cnt[c] > ps.cnt[bc]) bc = c;
    ps.choice = bc;
  }
  __syncthreads();
  const int c = ps.choice;
  for (int j = 0, i = tid; i < n; ++j, i += NT) mask[i] = (bits >> (4 * j + c)) & 1u;
  const int good = ps.cnt[c];
  __syncthreads();
  return good;
}

__global__ void __launch_bounds__(NT, 1) ransac_kernel(RansacArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  WarpScratch* wss = reinterpret_cast<WarpScratch*>(smem);
  double* s_models = reinterpret_cast<double*>(smem + NW * sizeof(WarpScratch));   // [ROUND][MAXSOL][9]
  double* s_pts = s_models + ROUND * MAXSOL * 9;                                      // [n][4]
  __shared__ int s_cnt[ROUND * MAXSOL];
  __shared__ int s_nmod[ROUND];
  __shared__ double s_bestE[9], s_R[9], s_t[3];
  __shared__ int s_best, s_niters, s_iter, s_done, s_good;
  __shared__ unsigned char s_m5[5];
  __shared__ PoseShared ps;

  const int b = blockIdx.x, NS = a.N, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = a.n_valid ? min(max(a.n_valid[b], 0), NS) : NS;
  WarpScratch& ws = wss[warp];
  const float fx0 = a.intr0[b * 4 + 0], fy0 = a.intr0[b * 4 + 1], cx0 = a.intr0[b * 4 + 2], cy0 = a.intr0[b * 4 + 3];
  const float fx1 = a.intr1[b * 4 + 0], fy1 = a.intr1[b * 4 + 1], cx1 = a.intr1[b * 4 + 2], cy1 = a.intr1[b * 4 + 3];
  const float* k0 = a.kpts0 + (long long)b * NS * 2;
  const float* k1 = a.kpts1 + (long long)b * NS * 2;
  float* k0n = a.k0n + (long long)b * NS * 2;
  float* k1n = a.k1n + (long long)b * NS * 2;
  unsigned char* mask = a.inliers + (long long)b * NS;
  double* E_out = a.E_out + (long long)b * MAXSOL * 9;

  // normalised points (fp64, (k - c) / f), padded outputs zero
  for (int i = tid; i < NS; i += NT) {
    if (i < n) {
      const double x1 = ((double)k0[2 * i] - (double)cx0) / (double)fx0, y1 = ((double)k0[2 * i + 1] - (double)cy0) / (double)fy0;
      const double x2 = ((double)k1[2 * i] - (double)cx1) / (double)fx1, y2 = ((double)k1[2 * i + 1] - (double)cy1) / (double)fy1;
      s_pts[4 * i] = x1; s_pts[4 * i + 1] = y1; s_pts[4 * i + 2] = x2; s_pts[4 * i + 3] = y2;
      k0n[2 * i] = (float)x1; k0n[2 * i + 1] = (float)y1; k1n[2 * i] = (float)x2; k1n[2 * i + 1] = (float)y2;
    } else {
      k0n[2 * i] = 0.f; k0n[2 * i + 1] = 0.f; k1n[2 * i] = 0.f; k1n[2 * i + 1] = 0.f;
    }
    mask[i] = 0;
  }
  for (int e = tid; e < MAXSOL * 9; e += NT) E_out[e] = 0.0;
  if (tid == 0) {
    s_best = 0; s_niters = a.max_iters; s_iter = 0; s_done = 0; s_good = 0;
  }
  __syncthreads();

  const double thr = (double)a.thresh_px / (((double)fx0 + (double)fy1 + (double)fx0 + (double)fy1) / 4.0);
  const float thr2 = (float)(thr * thr);
  int n_models = 0;

  if (n == 5) {
    // findEssentialMat returns every solution; estimate_pose tries them in turn
    if (warp == 0) {
      if (lane < 5) ws.idx[lane] = lane;
      __syncwarp();
      const int k = five_point_warp(ws, s_pts, s_models, lane);
      if (lane == 0) s_nmod[0] = k;
    }
    if (tid < 5) mask[tid] = 1;
    __syncthreads();
    n_models = s_nmod[0];
    for (int e = tid; e < n_models * 9; e += NT) E_out[e] = s_models[e];
    for (int s = 0; s < n_models; ++s) {
      const int good = recover_pose_block(s_models + 9 * s, s_pts, n, mask, ps);
      if (good > s_good) {
        __syncthreads();
        if (tid == 0) {
          s_good = good;
          for (int e = 0; e < 9; ++e) s_R[e] = ps.R[ps.choice & 1][e];
          const double sg = ps.choice < 2 ? 1.0 : -1.0;
          for (int e = 0; e < 3; ++e) s_t[e] = sg * ps.t[e];
        }
        if (tid < 5) s_m5[tid] = mask[tid];
      }
      __syncthreads();
    }
    if (tid < 5) mask[tid] = s_good > 0 ? s_m5[tid] : 0;
  } else if (n > 5) {
    for (int base = 0; !s_done; base += ROUND) {
      const int niters0 = s_niters;
      for (int e = tid; e < ROUND * MAXSOL; e += NT) s_cnt[e] = 0;
      for (int hl = warp; hl < ROUND; hl += NW) {
        const int h = base + hl;
        int k = 0;
        if (h < niters0) {      // the bound only decreases: hypotheses past it are never consumed
          bool ok = false;
          if (lane == 0) ok = sample5(a.seed_key, (unsigned long long)h, n, ws.idx);
          ok = __shfl_sync(0xffffffffu, ok, 0);
          __syncwarp();
          if (ok) k = five_point_warp(ws, s_pts, s_models + hl * MAXSOL * 9, lane);
        }
        if (lane == 0) s_nmod[hl] = k;
        __syncwarp();
      }
      __syncthreads();
      // inlier counts of every model of the round
      for (int sl = 0; sl < ROUND * MAXSOL; ++sl) {
        if (sl % MAXSOL >= s_nmod[sl / MAXSOL]) continue;
        const double* E = s_models + sl * 9;
        double e[9];
#pragma unroll
        for (int q = 0; q < 9; ++q) e[q] = E[q];
        int c = 0;
        for (int i = tid; i < n; i += NT) c += is_inlier(e, s_pts + 4 * i, thr2);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0 && c) atomicAdd(&s_cnt[sl], c);
      }
      __syncthreads();
      // OpenCV's sequential loop over this round's hypotheses
      if (tid == 0) {
        int niters = s_niters, best = s_best, it = s_iter;
        for (int hl = 0; hl < ROUND; ++hl) {
          const int h = base + hl;
          if (h >= niters) break;
          for (int m = 0; m < s_nmod[hl]; ++m) {
            const int g = s_cnt[hl * MAXSOL + m];
            if (g > max(best, 4)) {
              best = g;
              for (int q = 0; q < 9; ++q) s_bestE[q] = s_models[(hl * MAXSOL + m) * 9 + q];
              niters = update_num_iters(a.prob, (double)(n - g) / n, 5, niters);
            }
          }
          it = h + 1;
        }
        s_niters = niters; s_best = best; s_iter = it;
        s_done = it >= niters;
      }
      __syncthreads();
    }
    if (s_best > 0) {
      n_models = 1;
      for (int i = tid; i < n; i += NT) mask[i] = is_inlier(s_bestE, s_pts + 4 * i, thr2) ? 1 : 0;
      if (tid < 9) E_out[tid] = s_bestE[tid];
      __syncthreads();
      const int good = recover_pose_block(s_bestE, s_pts, n, mask, ps);
      if (tid == 0) {
        s_good = good;
        for (int e = 0; e < 9; ++e) s_R[e] = ps.R[ps.choice & 1][e];
        const double sg = ps.choice < 2 ? 1.0 : -1.0;
        for (int e = 0; e < 3; ++e) s_t[e] = sg * ps.t[e];
      }
    }
  }
  __syncthreads();
  const bool success = s_good > 0;
  if (tid < 16) {
    const int r = tid / 4, c = tid % 4;
    float v = (r == c) ? 1.f : 0.f;
    if (success && r < 3) v = c < 3 ? (float)s_R[r * 3 + c] : (float)s_t[r];
    a.T021[b * 16 + tid] = v;
  }
  if (!success)
    for (int i = tid; i < n; i += NT) mask[i] = 0;
  if (tid == 0) {
    a.success[b] = success ? 1 : 0;
    a.n_inliers[b] = success ? s_good : 0;
    a.n_models[b] = n_models;
    a.iterations[b] = s_iter;
  }
}

}  // namespace

extern "C" int mvm_ransac_essential(const float* kpts0, const float* kpts1, const float* intr0, const float* intr1,
                                    int batch, int n, const int* n_valid, float thresh_px, double prob, int max_iters,
                                    unsigned long long seed, float* T021, float* kpts0_norm, float* kpts1_norm,
                                    unsigned char* inliers, int* n_inliers, double* E_out, int* n_models,
                                    int* iterations, unsigned char* success, void* stream) {
  MvmProfScope prof__(MVM_TAG_MISC, (cudaStream_t)stream);
  MVM_REQUIRE(kpts0 && kpts1 && intr0 && intr1 && T021 && kpts0_norm && kpts1_norm && inliers && n_inliers && E_out &&
              n_models && iterations && success);
  MVM_REQUIRE(batch >= 1 && n >= 1);
  if (n > MAX_N) {
    fprintf(stderr, "[mvm_b200] mvm_ransac_essential: n = %d matches per pair exceeds the %d held on chip\n", n, MAX_N);
    return MVM_ERR_INVALID;
  }
  MVM_REQUIRE(thresh_px > 0.f && prob >= 0.0 && prob <= 1.0 && max_iters >= 1);
  RansacArgs a;
  a.kpts0 = kpts0; a.kpts1 = kpts1; a.intr0 = intr0; a.intr1 = intr1; a.n_valid = n_valid; a.N = n;
  a.thresh_px = thresh_px; a.prob = prob; a.max_iters = max_iters; a.seed_key = splitmix64(seed);
  a.T021 = T021; a.k0n = kpts0_norm; a.k1n = kpts1_norm; a.inliers = inliers; a.n_inliers = n_inliers;
  a.E_out = E_out; a.n_models = n_models; a.iterations = iterations; a.success = success;
  const size_t smem = NW * sizeof(WarpScratch) + sizeof(double) * (ROUND * MAXSOL * 9 + 4 * (size_t)n);
  if (cudaFuncSetAttribute(ransac_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return MVM_ERR_LAUNCH;
  ransac_kernel<<<batch, NT, smem, (cudaStream_t)stream>>>(a);
  MVM_CHECK_LAUNCH();
  return MVM_OK;
}
