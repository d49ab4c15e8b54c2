"""fp64 CPU restatement of the reference's `ba_initializer` binary.  TEST INFRASTRUCTURE.

The reference delegates to Theia 0.7.0 with default options (ba_init.cpp:77-91):
``RobustRotationEstimator`` (Chatterjee & Govindu, ICCV'13: L1 averaging then IRLS in the tangent
space of SO(3)) initialised from the spanning-tree rotations, followed by
``LeastUnsquaredDeviationPositionEstimator`` (Ozyesil & Singer, CVPR'15).  Theia is a third-party
dependency that is absent from /root/reference and from this image; its published algorithms are
restated here (PARITY UNPINNED against Theia's exact iterates) and pinned on the reference's own
known-answer tests (ba_init/test/test_ba_init.cpp:93-274: same four-camera scene, same glibc rand()
noise stream, same tolerances) by tests/test_ba_init_oracle.py.

Conventions (ba_init.cpp:10-52, test_ba_init.cpp:16-36): global rotation i = angle-axis of the
world->cam rotation R_i; view pair (i, j), i < j: rotation_2 = angle-axis of R_ij = R_j R_i^T,
position_2 = position of camera j in camera i's frame (= -R_ij^T t_ij).  Output translation is
t_i = -R_i c_i (ba_init.cpp:58-75).

Rotation averaging (robust_rotation_estimator.cc):
  residual_e = log(R_j^T R_ij R_i);  A has -I at view i and +I at view j (view 0 fixed);
  L1 phase: <= 5 times { min |A d - r|_1 by ADMM (rho = 1, alpha = 1, abs tol 1e-4, rel tol 1e-2) with
  5 ADMM iterations in the first pass and twice as many in every following one; R_v <- R_v exp(d_v);
  stop when the mean step <= 1e-3 };
  IRLS phase: <= 100 times { w_e = sigma / (|r_e|^2 + sigma^2)^2, sigma = 5 deg; solve
  (A^T W A) d = A^T W r; update; stop when the mean step <= 1e-3 }.
Position estimation (least_unsquared_deviation_position_estimator.cc):
  min sum_e | c_j - c_i - s_e d_e |   s.t. s_e >= 1,  c_0 = 0,   d_e = R_i^T position_2
  by iteratively reweighted least squares (<= 40 reweightings, weights 1 / max(|res_e|, 1e-6)), each
  weighted bound-constrained least-squares problem solved exactly (active set on s_e >= 1).  The
  objective is convex, so any convergent solver reaches the same minimiser Theia's ADMM-QP does.
"""
import numpy as np

from .mvba import angle_axis_to_R, R_to_angle_axis, _GlibcRand

SIGMA = np.deg2rad(5.0)


def _mul(aa1, aa2):
    """theia::MultiplyRotations: angle-axis of R(aa1) R(aa2)."""
    return R_to_angle_axis(angle_axis_to_R(np.asarray(aa1, float)) @ angle_axis_to_R(np.asarray(aa2, float)))


def _build_A(n_views, edges):
    m, n = 3 * len(edges), 3 * (n_views - 1)
    A = np.zeros((m, n))
    for e, (i, j) in enumerate(edges):
        if i != 0:
            A[3 * e:3 * e + 3, 3 * (i - 1):3 * i] = -np.eye(3)
        if j != 0:
            A[3 * e:3 * e + 3, 3 * (j - 1):3 * j] = np.eye(3)
    return A


def l1_admm(A, b, max_iter=1000, rho=1.0, alpha=1.0, abs_tol=1e-4, rel_tol=1e-2):
    """theia::L1Solver (ADMM for least absolute deviations, Boyd et al. §6.1)."""
    m, n = A.shape
    AtA_inv = np.linalg.inv(A.T @ A)
    x = np.zeros(n)
    z = np.zeros(m)
    u = np.zeros(m)
    for _ in range(max_iter):
        x = AtA_inv @ (A.T @ (b + z - u))
        Ax = A @ x
        ax_hat = alpha * Ax + (1 - alpha) * (z + b)
        z_old = z
        v = ax_hat - b + u
        z = np.sign(v) * np.maximum(np.abs(v) - 1.0 / rho, 0.0)
        u = u + ax_hat - z - b
        r_norm = np.linalg.norm(Ax - z - b)
        s_norm = np.linalg.norm(-rho * A.T @ (z - z_old))
        eps_pri = np.sqrt(m) * abs_tol + rel_tol * max(np.linalg.norm(Ax), np.linalg.norm(z), np.linalg.norm(b))
        eps_dual = np.sqrt(n) * abs_tol + rel_tol * np.linalg.norm(rho * A.T @ u)
        if r_norm < eps_pri and s_norm < eps_dual:
            break
    return x


def robust_rotation_averaging(n_views, pair_rot, init_rot, max_l1=5, max_irls=100, step_tol=1e-3):
    """pair_rot[(i,j)] = angle-axis of R_ij; init_rot [n,3] angle-axis.  View 0 stays fixed."""
    edges = sorted(pair_rot.keys())
    rot = np.array(init_rot, float).copy()
    if not edges:
        return rot
    A = _build_A(n_views, edges)

    def residuals():
        return np.concatenate([_mul(-rot[j], _mul(pair_rot[(i, j)], rot[i])) for (i, j) in edges])

    def update(step):
        for v in range(1, n_views):
            rot[v] = _mul(rot[v], step[3 * (v - 1):3 * v])
        return np.mean([np.linalg.norm(step[3 * (v - 1):3 * v]) for v in range(1, n_views)])

    admm_iters = 5                       # robust_rotation_estimator.cc: 5 ADMM iterations, doubled every outer pass
    for _ in range(max_l1):
        if update(l1_admm(A, residuals(), max_iter=admm_iters)) <= step_tol:
            break
        admm_iters *= 2
    for _ in range(max_irls):
        r = residuals()
        w = np.repeat([SIGMA / (r[3 * e:3 * e + 3] @ r[3 * e:3 * e + 3] + SIGMA ** 2) ** 2 for e in range(len(edges))], 3)
        AtW = A.T * w
        step = np.linalg.solve(AtW @ A, AtW @ r)
        if update(step) <= step_tol:
            break
    return rot


def _bounded_wls(n_views, edges, dirs, w, active):
    """min sum_e w_e |c_j - c_i - s_e d_e|^2  s.t. s_e >= 1, c_0 = 0.  For a given active set the free
    scales are eliminated analytically (s_e = d_e.(c_j - c_i) / |d_e|^2), leaving a 3(n-1) system in the
    positions: H = sum_e w_e B_e^T Q_e B_e, Q_e = I - d d^T/|d|^2 (free) or I (active, s_e = 1)."""
    nc, E = 3 * (n_views - 1), len(edges)
    c = np.zeros((n_views, 3))
    s = np.ones(E)
    for _ in range(2 * E + 2):
        H = np.zeros((nc, nc))
        g = np.zeros(nc)
        for e, (i, j) in enumerate(edges):
            d = dirs[e]
            Q = np.eye(3) if active[e] else np.eye(3) - np.outer(d, d) / (d @ d)
            Q = w[e] * Q
            for (a, sa) in ((i, -1.0), (j, 1.0)):
                if a == 0:
                    continue
                if active[e]:
                    g[3 * (a - 1):3 * a] += sa * (Q @ d)
                for (b, sb) in ((i, -1.0), (j, 1.0)):
                    if b == 0:
                        continue
                    H[3 * (a - 1):3 * a, 3 * (b - 1):3 * b] += sa * sb * Q
        H += 1e-12 * np.eye(nc)
        c[1:] = np.linalg.solve(H, g).reshape(-1, 3)
        changed = False
        for e, (i, j) in enumerate(edges):
            d = dirs[e]
            proj = d @ (c[j] - c[i]) / (d @ d)
            if not active[e]:
                s[e] = proj
                if proj < 1.0 - 1e-12:
                    active[e] = True
                    s[e] = 1.0
                    changed = True
            else:
                s[e] = 1.0
                if proj > 1.0 + 1e-12:       # the bound's multiplier has the wrong sign: release
                    active[e] = False
                    changed = True
        if not changed:
            break
    return c[1:].copy(), s


def lud_positions(n_views, pair_pos, rot, max_reweight=40, tol=1e-9):
    """pair_pos[(i,j)] = position of camera j in camera i's frame; rot [n,3] global rotations."""
    edges = sorted(pair_pos.keys())
    if not edges:
        return np.zeros((n_views, 3))
    dirs = [angle_axis_to_R(rot[i]).T @ np.asarray(pair_pos[(i, j)], float) for (i, j) in edges]
    w = np.ones(len(edges))
    c_prev = None
    # active set of the bounds s_e >= 1: starts from s_e = 1 everywhere (the all-free problem is
    # scale-degenerate) and is carried over from one reweighting to the next (warm start)
    active = np.ones(len(edges), bool)
    for _ in range(max_reweight):
        c, s = _bounded_wls(n_views, edges, dirs, w, active)
        call = np.vstack([np.zeros(3), c])
        res = np.array([np.linalg.norm(call[j] - call[i] - s[e] * dirs[e]) for e, (i, j) in enumerate(edges)])
        w = 1.0 / np.maximum(res, 1e-6)
        if c_prev is not None and np.abs(c - c_prev).max() < tol:
            break
        c_prev = c
    return np.vstack([np.zeros(3), c])


def ba_initialize(n_views, extr_init, rel_pose):
    """The whole `ba_initializer`: extr_init [n,4,4] world->cam (spanning tree), rel_pose[(i,j)] = T_i->j 4x4
    (as written by initialize_bundle_adjust, bundle_adjust_io.py:175-190).  Returns world->cam extrinsics."""
    init_rot = np.array([R_to_angle_axis(e[:3, :3]) for e in extr_init])
    pair_rot = {k: R_to_angle_axis(T[:3, :3]) for k, T in rel_pose.items()}
    pair_pos = {k: -T[:3, :3].T @ T[:3, 3] for k, T in rel_pose.items()}
    rot = robust_rotation_averaging(n_views, pair_rot, init_rot)
    pos = lud_positions(n_views, pair_pos, rot)
    out = []
    for v in range(n_views):
        T = np.eye(4)
        T[:3, :3] = angle_axis_to_R(rot[v])
        T[:3, 3] = -T[:3, :3] @ pos[v]
        out.append(T)
    return np.array(out)


def ba_initialize_edges(n_views, pairs, extr_tree, T_rel, success, on_tree, inliers, min_inliers=20):
    """``mvm_ba_initialize`` for one tuple, edge selection included.  The pairs written to ba_init_in.csv
    (bundle_adjust_io.py, initialize_bundle_adjust) are the edges: pair p = (a, b) is one when
    success[p] and (its inlier count >= min_inliers or on_tree[p]).  inliers [P, n_pad] is the 0/1 inlier
    mask of every pair, counted over all n_pad entries (None: no pair has inliers, only the tree counts).
    If those edges do not connect every view to view 0, extr_tree is returned unchanged; otherwise
    ba_initialize runs on them, with T_rel [P,4,4] taken as given (float32 inputs are widened to float64).
    Returns (extrinsics [n_views,4,4], number of edges)."""
    keep, connected = ba_init_edge_set(n_views, pairs, T_rel, success, on_tree, inliers, min_inliers)
    if not connected:
        return np.array(extr_tree, np.float64).copy(), len(keep)
    return ba_initialize(n_views, np.asarray(extr_tree, np.float64), keep), len(keep)


def ba_init_edge_set(n_views, pairs, T_rel, success, on_tree, inliers, min_inliers=20):
    """The edge rule of ba_initialize_edges alone: ({(a, b): T_rel float64}, whether the edges reach every
    view from view 0)."""
    keep = {}
    for p, (a, b) in enumerate(pairs):
        cnt = 0 if inliers is None else int(np.asarray(inliers[p], np.int64).sum())
        if success[p] and (cnt >= min_inliers or on_tree[p]):
            keep[(int(a), int(b))] = np.asarray(T_rel[p], np.float64)
    seen = {0}
    for _ in range(n_views):
        for a, b in keep:
            if a in seen or b in seen:
                seen |= {a, b}
    return keep, len(seen) == n_views


def make_pose_graph(seed, n_views, rot_deg=(3, 12), baseline=(0.2, 0.6), collinear=0.0, corrupt=None):
    """Ground-truth world->cam extrinsics [n_views,4,4] (view 0 = identity) and the exact relative poses
    T_a->b = E_b E_a^-1 of every pair a < b, as a dict.
      rot_deg      every view v > 0 is rotated by U(rot_deg) degrees about a random axis; (130, 179) gives
                   relative rotations past 120 deg (trace of R < 0);
      collinear    > 0: camera centres on the x axis at 0, 1, 2, ... m, each moved off the line by at most
                   `collinear` m (near-collinear centres); 0: centres at U(baseline) m in random directions;
      corrupt      a pair (a, b) whose relative pose is replaced by one rotated a further 40 deg and with a
                   translation direction turned by 90 deg (an outlier edge)."""
    from .pose import rodrigues
    rng = np.random.default_rng(seed)
    extr = [np.eye(4)]
    for v in range(1, n_views):
        ax = rng.standard_normal(3)
        R = rodrigues(ax / np.linalg.norm(ax) * np.deg2rad(rng.uniform(*rot_deg)))
        if collinear > 0:
            c = np.array([float(v), 0.0, 0.0]) + collinear * rng.uniform(-1, 1, 3)
        else:
            d = rng.standard_normal(3)
            c = d / np.linalg.norm(d) * rng.uniform(*baseline)
        E = np.eye(4)
        E[:3, :3] = R
        E[:3, 3] = -R @ c
        extr.append(E)
    extr = np.array(extr)
    rel = {(a, b): extr[b] @ np.linalg.inv(extr[a]) for b in range(n_views) for a in range(b)}
    if corrupt is not None:
        ax = rng.standard_normal(3)
        T = rel[corrupt].copy()
        T[:3, :3] = rodrigues(ax / np.linalg.norm(ax) * np.deg2rad(40.0)) @ T[:3, :3]
        t = T[:3, 3]
        perp = np.cross(t, rng.standard_normal(3))
        T[:3, 3] = perp / np.linalg.norm(perp) * np.linalg.norm(t)
        rel[corrupt] = T
    return extr, rel


# ---------------------------------------------------------------------------------------------
# the reference's known-answer scene (test_ba_init.cpp:84-91) and noise helpers (:10-49)
# ---------------------------------------------------------------------------------------------
def gtest_extrinsics():
    out = []
    for pos, yaw in (((0., 0., 0.), 0.0), ((1., 0., 0.), np.pi / 4), ((1., 1., 0.), np.pi / 2), ((0., 1., 0.), -3 * np.pi / 4)):
        T = np.eye(4)
        T[:3, :3] = angle_axis_to_R(np.array([0, 0, yaw]))
        T[:3, 3] = pos
        out.append(np.linalg.inv(T))
    return out


class GtestNoise:
    """std::rand() based Err() of the gtest; the draw ORDER of each helper follows the C++ source."""

    def __init__(self):
        self.rnd = _GlibcRand.__new__(_GlibcRand)
        import ctypes
        self.rnd.libc = ctypes.CDLL('libc.so.6')
        self.rnd.RAND_MAX = 2147483647

    def view_pairs(self, extr, max_err=0.0):
        rot, pos = {}, {}
        for j in range(len(extr)):
            for i in range(j):
                T = extr[j] @ np.linalg.inv(extr[i])
                r = R_to_angle_axis(T[:3, :3])
                r = r + np.array([self.rnd.err(max_err) for _ in range(3)])
                p = np.linalg.inv(T)[:3, 3] + np.array([self.rnd.err(max_err) for _ in range(3)])
                rot[(i, j)], pos[(i, j)] = r, p
        return rot, pos

    def global_rotations(self, extr, max_err=0.0):
        return np.array([R_to_angle_axis(e[:3, :3]) + np.array([self.rnd.err(max_err) for _ in range(3)]) for e in extr])
