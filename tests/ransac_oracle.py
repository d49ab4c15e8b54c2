"""float64 numpy restatement of the two-view RANSAC path: OpenCV's findEssentialMat(method=RANSAC) followed by
recoverPose, driven the way the reference's ``estimate_pose`` drives them (models/models/utils.py:288-312).  TEST
INFRASTRUCTURE ONLY: tests/test_ransac_oracle_opencv.py pins it to OpenCV 4.13, tests/test_ransac_gpu.py pins
csrc/pose_ransac.cu to it.

What is OpenCV's, restated:
  * the RANSAC loop of RANSACPointSetRegistrator::run: each model of a sample scored on its own, a model replaces the
    best only when its inlier count is strictly greater than max(best, 4), RANSACUpdateNumIters after every
    improvement (the iteration bound only decreases); with exactly 5 points no loop: every solution, mask all ones;
  * EMEstimatorCallback::computeError: (x2' E x1)^2 / (Ex1_0^2 + Ex1_1^2 + E'x2_0^2 + E'x2_1^2) rounded to float and
    compared with (float)(thr^2);
  * recoverPose: decomposeEssentialMat (W = [[0,1,0],[-1,0,0],[0,0,1]], det U = det Vt = +1), DLT triangulation,
    depth in (0, 50) in both cameras -- estimate_pose's positional 1e9 lands in the R output slot of the
    (E, p1, p2, K[, R[, t[, mask]]]) overload, so OpenCV's fixed distance threshold of 50 applies -- candidates R1,t / R2,t / R1,-t / R2,-t with the
    first maximum winning, and the mask argument rewritten in place.

What is this project's (shared with the CUDA kernel, so that the two agree draw for draw):
  * the sampler: splitmix64 of (seed, hypothesis, draw, attempt) mod n, duplicates redrawn (sample_indices);
  * the five-point solver: null space of the 5 x 9 epipolar system, the ten cubic constraints of an essential matrix
    (det E = 0, 2 E E' E - tr(E E') E = 0) in the monomials of Nister's elimination, Gauss-Jordan on the 10 x 20
    system, the degree-10 determinant of the 3 x 3 polynomial matrix in z, its real roots in ascending order,
    x and y from the null vector of that matrix; every E scaled to unit Frobenius norm, largest entry positive.
"""
import math

import numpy as np

from oracle import pose as P

M64 = (1 << 64) - 1
MAX_ATTEMPTS = 64          # redraws of one sample index before the hypothesis is given up (yields no model)
DBL_MIN = np.finfo(np.float64).tiny


# ----------------------------------------------------------------------------------------------------------------
# sampler
# ----------------------------------------------------------------------------------------------------------------
def splitmix64(x):
    z = (x + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def sample_indices(seed, hyp, n):
    """Five distinct indices in [0, n) for hypothesis `hyp`: index d is splitmix64(splitmix64(splitmix64(seed) ^ hyp)
    ^ (d << 32 | attempt)) mod n, attempt = 0, 1, ... until it differs from the earlier draws.  None when
    MAX_ATTEMPTS redraws do not give a new index."""
    k0 = splitmix64(splitmix64(seed & M64) ^ hyp)
    idx = []
    for d in range(5):
        for a in range(MAX_ATTEMPTS):
            i = splitmix64(k0 ^ ((d << 32) | a)) % n
            if i not in idx:
                idx.append(i)
                break
        else:
            return None
    return idx


# ----------------------------------------------------------------------------------------------------------------
# five-point solver
# ----------------------------------------------------------------------------------------------------------------
# monomials x^a y^b z^c.  Degree 3 in the order of Nister's elimination: the first ten are eliminated, rows 4..9 of
# the reduced system lead with x^2 z, x^2, y^2 z, y^2, xyz, xy.
MONO1 = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0)]
MONO2 = [(2, 0, 0), (0, 2, 0), (0, 0, 2), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0)]
MONO3 = [(3, 0, 0), (0, 3, 0), (2, 1, 0), (1, 2, 0), (2, 0, 1), (2, 0, 0), (0, 2, 1), (0, 2, 0), (1, 1, 1), (1, 1, 0),
         (1, 0, 2), (1, 0, 1), (1, 0, 0), (0, 1, 2), (0, 1, 1), (0, 1, 0), (0, 0, 3), (0, 0, 2), (0, 0, 1), (0, 0, 0)]


def _mul_table(ma, mb, mc):
    T = np.zeros((len(ma), len(mb), len(mc)))
    for i, a in enumerate(ma):
        for j, b in enumerate(mb):
            T[i, j, mc.index(tuple(p + q for p, q in zip(a, b)))] = 1.0
    return T


MUL11 = _mul_table(MONO1, MONO1, MONO2)       # linear x linear -> quadratic
MUL21 = _mul_table(MONO2, MONO1, MONO3)       # quadratic x linear -> cubic


def _m11(a, b):
    return np.einsum('i,j,ijk->k', a, b, MUL11)


def _m21(a, b):
    return np.einsum('i,j,ijk->k', a, b, MUL21)


def epipolar_rows(x1, x2):
    """[n, 9]: x2' E x1 = row . vec(E) (row-major E)."""
    u1, v1 = x1[:, 0], x1[:, 1]
    u2, v2 = x2[:, 0], x2[:, 1]
    one = np.ones_like(u1)
    return np.stack([u2 * u1, u2 * v1, u2, v2 * u1, v2 * v1, v2, u1, v1, one], 1)


def constraint_matrix(basis):
    """basis [4, 9] = X, Y, Z, W (E = x X + y Y + z Z + W) -> the 10 x 20 coefficient matrix of the cubic constraints
    2 E E' E - tr(E E') E = 0 (nine rows, row-major) and det E = 0 (last row)."""
    Eb = basis.T.reshape(3, 3, 4)                  # Eb[i, j] = linear polynomial of E_ij in MONO1
    EEt = [[sum(_m11(Eb[i, k], Eb[j, k]) for k in range(3)) for j in range(3)] for i in range(3)]
    tr = EEt[0][0] + EEt[1][1] + EEt[2][2]
    rows = []
    for i in range(3):
        for j in range(3):
            r = -_m21(tr, Eb[i, j])
            for k in range(3):
                r = r + 2.0 * _m21(EEt[i][k], Eb[k, j])
            rows.append(r)
    det = (_m21(_m11(Eb[1, 1], Eb[2, 2]) - _m11(Eb[1, 2], Eb[2, 1]), Eb[0, 0])
           - _m21(_m11(Eb[1, 0], Eb[2, 2]) - _m11(Eb[1, 2], Eb[2, 0]), Eb[0, 1])
           + _m21(_m11(Eb[1, 0], Eb[2, 1]) - _m11(Eb[1, 1], Eb[2, 0]), Eb[0, 2]))
    rows.append(det)
    return np.array(rows)


def _pmul(a, b):
    return np.convolve(a, b)


def hidden_variable_matrix(G):
    """G [10, 10] = right half of the reduced 10 x 20 system -> B(z) as three rows of (x coefficient [4], y
    coefficient [4], constant [5]), ascending powers of z: row (a, b) - z row (a + 1) for a = 4, 6, 8."""
    out = []
    for a in (4, 6, 8):
        ga, gb = G[a], G[a + 1]
        bx = np.array([ga[2], ga[1] - gb[2], ga[0] - gb[1], -gb[0]])
        by = np.array([ga[5], ga[4] - gb[5], ga[3] - gb[4], -gb[3]])
        b1 = np.array([ga[9], ga[8] - gb[9], ga[7] - gb[8], ga[6] - gb[7], -gb[6]])
        out.append((bx, by, b1))
    return out


def det_polynomial(Bz):
    """Degree-10 determinant of B(z), ascending coefficients [11]."""
    (bx0, by0, b10), (bx1, by1, b11), (bx2, by2, b12) = Bz
    d = (_pmul(bx0, _pmul(by1, b12) - _pmul(b11, by2))
         - _pmul(by0, _pmul(bx1, b12) - _pmul(b11, bx2))
         + _pmul(b10, _pmul(bx1, by2) - _pmul(by1, bx2)))
    return d


def _polyval(c, z):
    s = 0.0
    for a in c[::-1]:
        s = s * z + a
    return s


def real_roots(c, imag_tol=1e-8):
    """Real roots of the polynomial with ascending coefficients c, ascending, Newton-polished."""
    c = np.asarray(c, np.float64)
    nz = np.nonzero(c)[0]
    if len(nz) == 0:
        return []
    c = c[:nz[-1] + 1]
    if len(c) < 2:
        return []
    r = np.roots(c[::-1])
    dc = c[1:] * np.arange(1, len(c))
    out = []
    for z in r:
        if abs(z.imag) > imag_tol * max(1.0, abs(z.real)):
            continue
        z = float(z.real)
        for _ in range(3):
            d = _polyval(dc, z)
            if d == 0.0:
                break
            z = z - _polyval(c, z) / d
        out.append(z)
    return sorted(out)


def normalize_E(E):
    E = E / np.linalg.norm(E)
    k = int(np.argmax(np.abs(E)))
    return E if E.flat[k] > 0 else -E


def null_space_householder(Q):
    """Last four columns of the Householder QR of Q' (9 x 5), with the kernel's reflector signs, so that the two
    parametrise the solutions identically even where the problem is ill-conditioned."""
    A = Q.T.copy()
    V = np.zeros((5, 9))
    for k in range(5):
        nrm = math.sqrt(float((A[k:, k] ** 2).sum()))
        alpha = -nrm if A[k, k] > 0 else nrm
        v = np.zeros(9)
        v[k:] = A[k:, k]
        v[k] -= alpha
        vv = float((v[k:] ** 2).sum())
        v *= math.sqrt(2.0 / vv if vv > 0 else 0.0)            # H_k = I - v v'
        for c in range(k, 5):
            A[k:, c] -= (v[k:] @ A[k:, c]) * v[k:]
        V[k] = v
    basis = np.zeros((4, 9))
    for j in range(4):
        y = np.zeros(9)
        y[5 + j] = 1.0
        for k in range(4, -1, -1):
            y -= (V[k] @ y) * V[k]
        basis[j] = y
    return basis


def gauss_jordan(M):
    """[I | G] = reduced row echelon form of the 10 x 20 system (partial pivoting, first maximum) -> G, or None."""
    M = M.copy()
    for k in range(10):
        p = k + int(np.argmax(np.abs(M[k:, k])))
        if not (abs(M[p, k]) > 0) or not np.isfinite(M[p, k]):
            return None
        M[[k, p]] = M[[p, k]]
        col = M[:, k].copy()
        M[k] = M[k] / col[k]
        for r in range(10):
            if r != k:
                M[r] -= col[r] * M[k]
    return M[:, 10:]


def essential_constraints(E, D=None):
    """The ten cubic constraints of an essential matrix at E (2 E E' E - tr(E E') E row-major, det E), or with D their
    derivative along D."""
    if D is None:
        return np.append((2 * E @ E.T @ E - np.trace(E @ E.T) * E).reshape(9), np.linalg.det(E))
    cof = np.array([[E[1, 1] * E[2, 2] - E[1, 2] * E[2, 1], E[1, 2] * E[2, 0] - E[1, 0] * E[2, 2], E[1, 0] * E[2, 1] - E[1, 1] * E[2, 0]],
                    [E[0, 2] * E[2, 1] - E[0, 1] * E[2, 2], E[0, 0] * E[2, 2] - E[0, 2] * E[2, 0], E[0, 1] * E[2, 0] - E[0, 0] * E[2, 1]],
                    [E[0, 1] * E[1, 2] - E[0, 2] * E[1, 1], E[0, 2] * E[1, 0] - E[0, 0] * E[1, 2], E[0, 0] * E[1, 1] - E[0, 1] * E[1, 0]]])
    dT = 2 * (D @ E.T @ E + E @ D.T @ E + E @ E.T @ D) - 2 * np.trace(D @ E.T) * E - np.trace(E @ E.T) * D
    return np.append(dT.reshape(9), (cof * D).sum())


REFINE_STEPS = 3


def refine_xyz(basis, x, y, z):
    """Gauss-Newton steps on the ten constraints in (x, y, z), each kept only when it lowers the squared residual:
    the elimination loses digits on sets with close roots, the constraints themselves do not."""
    X, Y, Z, W = (basis[k].reshape(3, 3) for k in range(4))
    p = np.array([x, y, z])
    E = p[0] * X + p[1] * Y + p[2] * Z + W
    r = essential_constraints(E)
    rr = float(r @ r)
    for _ in range(REFINE_STEPS):
        J = np.stack([essential_constraints(E, D) for D in (X, Y, Z)], 1)
        try:
            d = np.linalg.solve(J.T @ J, -(J.T @ r))
        except np.linalg.LinAlgError:
            break
        pn = p + d
        En = pn[0] * X + pn[1] * Y + pn[2] * Z + W
        rn = essential_constraints(En)
        if not (float(rn @ rn) < rr):
            break
        p, E, r, rr = pn, En, rn, float(rn @ rn)
    return p[0], p[1], p[2]


def five_point(x1, x2):
    """All real essential matrices through five correspondences (normalised coordinates [5, 2] each), as a list of
    unit-norm 3 x 3 arrays in ascending order of the hidden variable z."""
    Q = epipolar_rows(np.asarray(x1, np.float64), np.asarray(x2, np.float64))
    basis = null_space_householder(Q)                          # X, Y, Z, W
    G = gauss_jordan(constraint_matrix(basis))
    if G is None or not np.isfinite(G).all():
        return []
    Bz = hidden_variable_matrix(G)
    sols = []
    for z in real_roots(det_polynomial(Bz)):
        B = np.array([[_polyval(bx, z), _polyval(by, z), _polyval(b1, z)] for bx, by, b1 in Bz])
        cands = [np.cross(B[0], B[1]), np.cross(B[0], B[2]), np.cross(B[1], B[2])]
        c = max(cands, key=lambda v: abs(v[2]))
        if c[2] == 0.0:
            continue
        x, y, z = refine_xyz(basis, c[0] / c[2], c[1] / c[2], z)
        E = (x * basis[0] + y * basis[1] + z * basis[2] + basis[3]).reshape(3, 3)
        if np.isfinite(E).all() and np.linalg.norm(E) > 0:
            sols.append(normalize_E(E))
    return sols


# ----------------------------------------------------------------------------------------------------------------
# scoring and the RANSAC loop
# ----------------------------------------------------------------------------------------------------------------
def sampson_errors(E, x1, x2):
    """EMEstimatorCallback::computeError, computed in double and rounded to float."""
    u1, v1 = x1[:, 0], x1[:, 1]
    u2, v2 = x2[:, 0], x2[:, 1]
    e = E.reshape(9)
    a0 = e[0] * u1 + e[1] * v1 + e[2]
    a1 = e[3] * u1 + e[4] * v1 + e[5]
    a2 = e[6] * u1 + e[7] * v1 + e[8]
    b0 = e[0] * u2 + e[3] * v2 + e[6]
    b1 = e[1] * u2 + e[4] * v2 + e[7]
    num = u2 * a0 + v2 * a1 + a2
    return (num * num / (a0 * a0 + a1 * a1 + b0 * b0 + b1 * b1)).astype(np.float32)


def inlier_mask(E, x1, x2, threshold):
    with np.errstate(divide='ignore', invalid='ignore'):
        return sampson_errors(E, x1, x2) <= np.float32(threshold * threshold)


def update_num_iters(p, ep, model_points, max_iters):
    """RANSACUpdateNumIters."""
    p = min(max(p, 0.0), 1.0)
    ep = min(max(ep, 0.0), 1.0)
    num = max(1.0 - p, DBL_MIN)
    denom = 1.0 - math.pow(1.0 - ep, model_points)
    if denom < DBL_MIN:
        return 0
    num = math.log(num)
    denom = math.log(denom)
    if denom >= 0 or -num >= max_iters * (-denom):
        return max_iters
    return int(np.rint(num / denom))


def find_essential_ransac(x1, x2, threshold, prob=0.99999, max_iters=1000, seed=0):
    """-> (E [3k, 3] or None, mask [n] bool or None, iterations, index of the chosen model as (hypothesis, solution)
    or None).  x1, x2 [n, 2] normalised float64; threshold in normalised units."""
    x1 = np.asarray(x1, np.float64)
    x2 = np.asarray(x2, np.float64)
    n = len(x1)
    if n < 5:
        return None, None, 0, None
    if n == 5:
        Es = five_point(x1, x2)
        if not Es:
            return None, None, 0, None
        return np.concatenate(Es, 0), np.ones(5, bool), 0, None
    niters, best, best_E, best_mask, chosen = max_iters, 0, None, None, None
    it = 0
    while it < niters:
        idx = sample_indices(seed, it, n)
        if idx is not None:
            for s, E in enumerate(five_point(x1[idx], x2[idx])):
                m = inlier_mask(E, x1, x2, threshold)
                g = int(m.sum())
                if g > max(best, 4):
                    best, best_E, best_mask, chosen = g, E, m, (it, s)
                    niters = update_num_iters(prob, (n - g) / n, 5, niters)
        it += 1
    if best_E is None:
        return None, None, it, None
    return best_E, best_mask, it, chosen


# ----------------------------------------------------------------------------------------------------------------
# recoverPose
# ----------------------------------------------------------------------------------------------------------------
def _canonical_sign(v):
    return v if v[int(np.argmax(np.abs(v)))] > 0 else -v


def decompose_essential_cv(E):
    """cv::decomposeEssentialMat -> R1 = U W Vt, R2 = U W' Vt, t = U[:, 2], W = [[0,1,0],[-1,0,0],[0,0,1]], det U =
    det Vt = +1.  The signs of the singular vectors, which OpenCV leaves to its SVD (they only decide which of two
    tied recoverPose candidates comes first), are fixed as in the kernel: v0, v1 with their largest entry positive,
    v2 = v0 x v1, u_i = E v_i / s_i, u2 = u0 x u1."""
    _, S, Vt = np.linalg.svd(E)
    v0, v1 = _canonical_sign(Vt[0]), _canonical_sign(Vt[1])
    v2 = np.cross(v0, v1)
    u0 = E @ v0
    u0 = u0 / np.linalg.norm(u0)
    u1 = E @ v1
    u1 = u1 - (u0 @ u1) * u0
    u1 = u1 / np.linalg.norm(u1)
    u2 = np.cross(u0, u1)
    R1 = -np.outer(u1, v0) + np.outer(u0, v1) + np.outer(u2, v2)
    R2 = np.outer(u1, v0) - np.outer(u0, v1) + np.outer(u2, v2)
    # E's two equal singular values leave the orientation of (v0, v1), hence the sign of t and the R1 / R2 labels, to
    # rounding: fix them (t with its largest entry positive, R1 the one of larger trace), as the kernel does
    t = _canonical_sign(u2)
    if np.trace(R1) < np.trace(R2):
        R1, R2 = R2, R1
    return R1, R2, t


def triangulate_homogeneous(R, t, x1, x2):
    """cv::triangulatePoints with P0 = [I|0], P1 = [R|t]: last right-singular vector of the 4 x 4 DLT system, not
    de-homogenised.  [n, 4]."""
    P0 = np.hstack([np.eye(3), np.zeros((3, 1))])
    P1 = np.hstack([R, t[:, None]])
    A = np.stack([x1[:, 0:1] * P0[2] - P0[0], x1[:, 1:2] * P0[2] - P0[1],
                  x2[:, 0:1] * P1[2] - P1[0], x2[:, 1:2] * P1[2] - P1[1]], 1)
    _, _, Vt = np.linalg.svd(A)
    return Vt[:, -1, :]


def recover_pose(E, x1, x2, mask=None, dist=50.0, return_counts=False):
    """cv::recoverPose(E, x1, x2, I, dist, mask) -> (n, R, t, mask after the call) [, counts of the four candidates]."""
    x1 = np.asarray(x1, np.float64)
    x2 = np.asarray(x2, np.float64)
    R1, R2, t = decompose_essential_cv(E)
    masks, cands = [], [(R1, t), (R2, t), (R1, -t), (R2, -t)]
    with np.errstate(divide='ignore', invalid='ignore'):
        for R, tt in cands:
            Q = triangulate_homogeneous(R, tt, x1, x2)
            m = Q[:, 2] * Q[:, 3] > 0
            X = Q[:, :3] / Q[:, 3:4]
            m &= X[:, 2] < dist
            z1 = X @ R[2] + tt[2]
            m &= (z1 > 0) & (z1 < dist)
            if mask is not None:
                m &= np.asarray(mask, bool)
            masks.append(m)
    good = [int(m.sum()) for m in masks]
    c = int(np.argmax(good))                      # first maximum, OpenCV's >= chain
    R, tt = cands[c]
    if return_counts:
        return good[c], R, tt, masks[c], good
    return good[c], R, tt, masks[c]


def recover_pose_loop(E_stack, x1, x2, mask):
    """The loop of estimate_pose over the stacked solutions: each recoverPose call sees the mask the previous one left,
    the strictly largest count wins.  -> (R, t, mask) or None."""
    best, ret = 0, None
    mask = np.asarray(mask, bool).copy()
    for k in range(len(E_stack) // 3):
        n, R, t, mask = recover_pose(E_stack[3 * k:3 * k + 3], x1, x2, mask)
        if n > best:
            best, ret = n, (R, t, mask.copy())
    return ret


# ----------------------------------------------------------------------------------------------------------------
# estimate_pose
# ----------------------------------------------------------------------------------------------------------------
def normalize_kpts(kpts, K):
    K = np.asarray(K, np.float64)
    k = np.asarray(kpts, np.float32).astype(np.float64)
    return np.stack([(k[:, 0] - K[0, 2]) / K[0, 0], (k[:, 1] - K[1, 2]) / K[1, 1]], 1)


def norm_threshold(K0, K1, thresh):
    K0 = np.asarray(K0, np.float32).astype(np.float64)
    K1 = np.asarray(K1, np.float32).astype(np.float64)
    return thresh / ((K0[0, 0] + K1[1, 1] + K0[0, 0] + K1[1, 1]) / 4.0)


def estimate_pose(kpts0, kpts1, K0, K1, thresh, conf=0.99999, max_iters=1000, seed=0, return_info=False):
    """models/models/utils.py:288-312 on this oracle: (R, t, mask) or None.  Keypoints are float32 pixels, normalised
    in float64; K0 / K1 as float32 like the kernel's intrinsics."""
    info = {'iterations': 0, 'E': None, 'chosen': None}
    ret = None
    if len(kpts0) >= 5:
        K0 = np.asarray(K0, np.float32).astype(np.float64)
        K1 = np.asarray(K1, np.float32).astype(np.float64)
        x1, x2 = normalize_kpts(kpts0, K0), normalize_kpts(kpts1, K1)
        E, mask, it, chosen = find_essential_ransac(x1, x2, norm_threshold(K0, K1, thresh), conf, max_iters, seed)
        info.update(iterations=it, E=E, chosen=chosen, ransac_mask=mask)
        if E is not None:
            ret = recover_pose_loop(E, x1, x2, mask)
    return (ret, info) if return_info else ret


def pose_errors_deg(T_gt, R, t):
    return P.compute_pose_error(T_gt, R, t)
