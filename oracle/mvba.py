"""fp64 CPU restatement of the reference's multi-view bundle adjustment.  TEST INFRASTRUCTURE.

What it restates
  * the residual model and parameterisation of the reference's own code:
    ``ReprojectionError`` / ``ReprojectionErrorFixedCamera`` (ba_problem.h:60-151): residual
    w * (f * pi(R(angle_axis) p + t) + c - x), camera 0 fixed by omitting its parameter block
    (ba_problem.cpp:129-147), no robust loss, ``DENSE_SCHUR`` (:150-152);
  * the problem construction of ``write_bundle_adjust_problem`` (bundle_adjust_io.py:193-259):
    one 3-D point per pairwise match, triangulated from the initial extrinsics, confidences
    normalised by c / (0.5 * sum c + 1e-3);
  * the spanning-tree initialisation of ``initialize_bundle_adjust`` (bundle_adjust_io.py:135-172).
  * the solver the reference delegates to -- Ceres 2.0.0 trust-region Levenberg-Marquardt with its
    default options (README.md:82; SURVEY.md A.7).  Ceres is a third-party dependency that is
    absent from /root/reference and from this image: its published algorithm is restated
    (Jacobi column scaling 1/(1+|J_j|) fixed at the first iteration, LM diagonal
    clamp(diag, 1e-6, 1e32)/radius, radius0 = 1e4, accept when rho > 1e-3, radius update
    r/max(1/3, 1-(2 rho-1)^3), reject: r /= k, k *= 2, <= 50 iterations, function tolerance 1e-6,
    gradient tolerance 1e-10, parameter tolerance 1e-8).  PARITY UNPINNED against Ceres' exact
    iterates; pinned on the reference's own known-answer scenes (test_ba_problem.cpp:165-184) by
    tests/test_mvba_oracle.py.
"""
import ctypes

import numpy as np


# ---------------------------------------------------------------------------------------------
# rotations (ceres/rotation.h semantics)
# ---------------------------------------------------------------------------------------------
def hat(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]], float)


def angle_axis_to_R(w):
    """ceres::AngleAxisToRotationMatrix."""
    th2 = float(w @ w)
    if th2 > np.finfo(float).eps:
        th = np.sqrt(th2)
        k = w / th
        K = hat(k)
        return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)
    return np.eye(3) + hat(w)


def R_to_angle_axis(R):
    """ceres::RotationMatrixToAngleAxis (via quaternion)."""
    tr = np.trace(R)
    if tr >= 0:
        t = np.sqrt(tr + 1.0)
        q0 = 0.5 * t
        t = 0.5 / t
        q = np.array([q0, (R[2, 1] - R[1, 2]) * t, (R[0, 2] - R[2, 0]) * t, (R[1, 0] - R[0, 1]) * t])
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        t = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
        q = np.zeros(4)
        q[i + 1] = 0.5 * t
        t = 0.5 / t
        q[0] = (R[k, j] - R[j, k]) * t
        q[j + 1] = (R[j, i] + R[i, j]) * t
        q[k + 1] = (R[k, i] + R[i, k]) * t
    s2 = q[1:] @ q[1:]
    if s2 > 0:
        s = np.sqrt(s2)
        th = 2 * np.arctan2(-s, -q[0]) if q[0] < 0 else 2 * np.arctan2(s, q[0])
        return q[1:] * th / s
    return q[1:] * 2.0


def d_rotated_point_d_angle_axis(w, p):
    """d(R(w) p)/dw (Gallego & Yezzi 2015): -R [p]x (w w^T + (R^T - I)[w]x) / |w|^2; -[p]x at 0."""
    th2 = float(w @ w)
    if th2 < 1e-16:
        return -hat(p)
    R = angle_axis_to_R(w)
    return -R @ hat(p) @ (np.outer(w, w) + (R.T - np.eye(3)) @ hat(w)) / th2


# ---------------------------------------------------------------------------------------------
# problem container
# ---------------------------------------------------------------------------------------------
class BaProblem:
    """Arrays of the CSV problem (ba_problem.cpp:8-90): cameras [C,6] (angle-axis | t), points
    [P,3], observations (cam, pt, xy, w)."""

    def __init__(self, cams, points, obs_cam, obs_pt, obs_xy, obs_w, fixed_cam=0,
                 intr=(1.0, 1.0, 0.0, 0.0)):
        self.cams = np.array(cams, float).reshape(-1, 6)
        self.points = np.array(points, float).reshape(-1, 3)
        self.obs_cam = np.array(obs_cam, int)
        self.obs_pt = np.array(obs_pt, int)
        self.obs_xy = np.array(obs_xy, float).reshape(-1, 2)
        w = np.array(obs_w, float)
        self.obs_w = np.stack([w, w], 1) if w.ndim == 1 else w.reshape(-1, 2)
        self.fixed = fixed_cam
        self.intr = intr


def _residuals_and_jacobian(pb, cams, points, want_J=True):
    fx, fy, cx, cy = pb.intr
    n_obs = len(pb.obs_cam)
    C, P = cams.shape[0], points.shape[0]
    free = [c for c in range(C) if c != pb.fixed]
    col_of = {c: 6 * i for i, c in enumerate(free)}
    ncam = 6 * len(free)
    r = np.zeros(2 * n_obs)
    J = np.zeros((2 * n_obs, ncam + 3 * P)) if want_J else None
    for o in range(n_obs):
        c, k = pb.obs_cam[o], pb.obs_pt[o]
        w = pb.obs_w[o]
        p = points[k]
        if c == pb.fixed:
            q = p.copy()      # ReprojectionErrorFixedCamera: the point is used as is (ba_problem.h:64-76)
            R = np.eye(3)
        else:
            R = angle_axis_to_R(cams[c, :3])
            q = R @ p + cams[c, 3:]
        r[2 * o] = w[0] * (fx * q[0] / q[2] + cx - pb.obs_xy[o, 0])
        r[2 * o + 1] = w[1] * (fy * q[1] / q[2] + cy - pb.obs_xy[o, 1])
        if want_J:
            Jpi = np.array([[w[0] * fx / q[2], 0, -w[0] * fx * q[0] / q[2] ** 2],
                            [0, w[1] * fy / q[2], -w[1] * fy * q[1] / q[2] ** 2]])
            J[2 * o:2 * o + 2, ncam + 3 * k:ncam + 3 * k + 3] = Jpi @ R
            if c != pb.fixed:
                col = col_of[c]
                J[2 * o:2 * o + 2, col:col + 3] = Jpi @ d_rotated_point_d_angle_axis(cams[c, :3], p)
                J[2 * o:2 * o + 2, col + 3:col + 6] = Jpi
    return r, J, free, ncam


def solve(pb, max_iterations=50, function_tolerance=1e-6, gradient_tolerance=1e-10,
          parameter_tolerance=1e-8, verbose=False):
    """Ceres-style trust-region LM (see module docstring).  Returns (cams [C,6], points, info)."""
    cams, points = pb.cams.copy(), pb.points.copy()
    r, J, free, ncam = _residuals_and_jacobian(pb, cams, points)
    cost = 0.5 * r @ r
    scale = 1.0 / (1.0 + np.sqrt((J ** 2).sum(0)))          # jacobi_scaling, fixed after iteration 0
    radius, decrease = 1e4, 2.0
    info = {'iterations': 0, 'initial_cost': cost, 'termination': 'max_iterations'}

    def pack(cams, points):
        return np.concatenate([cams[free].reshape(-1), points.reshape(-1)])

    x = pack(cams, points)
    g = J.T @ r
    if np.abs(g).max() <= gradient_tolerance:
        info['termination'] = 'gradient'
        info['final_cost'] = cost
        return cams, points, info
    for it in range(max_iterations):
        info['iterations'] = it + 1
        Js = J * scale
        gs = Js.T @ r
        H = Js.T @ Js
        D2 = np.clip(np.diag(H), 1e-6, 1e32) / radius
        # Schur complement on the point blocks == dense solve of (H + D2) d = -g
        try:
            ds = np.linalg.solve(H + np.diag(D2), -gs)
        except np.linalg.LinAlgError:
            radius /= decrease
            decrease *= 2
            continue
        d = ds * scale
        model = Js @ ds + r
        model_change = cost - 0.5 * model @ model
        x_new = x + d
        cams_n, points_n = cams.copy(), points.copy()
        cams_n[free] = x_new[:ncam].reshape(-1, 6)
        points_n[:] = x_new[ncam:].reshape(-1, 3)
        r_n, _, _, _ = _residuals_and_jacobian(pb, cams_n, points_n, want_J=False)
        cost_n = 0.5 * r_n @ r_n
        step_norm, x_norm = np.linalg.norm(d), np.linalg.norm(x)
        if step_norm <= parameter_tolerance * (x_norm + parameter_tolerance):
            info['termination'] = 'parameter'
            break
        rho = (cost - cost_n) / model_change if model_change > 0 else -1.0
        if verbose:
            print(it, cost, cost_n, rho, radius)
        if rho > 1e-3:
            cost_change = cost - cost_n
            cams, points, x = cams_n, points_n, x_new
            radius = min(radius / max(1.0 / 3.0, 1.0 - (2 * rho - 1) ** 3), 1e16)
            decrease = 2.0
            converged = abs(cost_change) <= function_tolerance * cost
            cost = cost_n
            r, J, _, _ = _residuals_and_jacobian(pb, cams, points)
            g = J.T @ r
            if converged:
                info['termination'] = 'function'
                break
            if np.abs(g).max() <= gradient_tolerance:
                info['termination'] = 'gradient'
                break
        else:
            radius /= decrease
            decrease *= 2
    info['final_cost'] = cost
    return cams, points, info


# ---------------------------------------------------------------------------------------------
# the same solver with the point blocks eliminated by a Schur complement (what DENSE_SCHUR does,
# ba_problem.cpp:150-152): identical iterates to `solve` up to rounding, O(P) instead of O(P^3)
# ---------------------------------------------------------------------------------------------
def _blocks(pb, cams, points, want_J=True):
    """Vectorised residuals and per-observation Jacobian blocks: r [O,2], Jc [O,2,6] (zero for the
    fixed camera), Jp [O,2,3]."""
    fx, fy, cx, cy = pb.intr
    oc, ok, w = pb.obs_cam, pb.obs_pt, pb.obs_w
    C = cams.shape[0]
    Rs = np.stack([np.eye(3) if c == pb.fixed else angle_axis_to_R(cams[c, :3]) for c in range(C)])
    ts = np.stack([np.zeros(3) if c == pb.fixed else cams[c, 3:] for c in range(C)])
    p = points[ok]
    q = np.einsum('oij,oj->oi', Rs[oc], p) + ts[oc]
    r = np.stack([w[:, 0] * (fx * q[:, 0] / q[:, 2] + cx - pb.obs_xy[:, 0]),
                  w[:, 1] * (fy * q[:, 1] / q[:, 2] + cy - pb.obs_xy[:, 1])], 1)
    if not want_J:
        return r, None, None
    O = len(oc)
    Jpi = np.zeros((O, 2, 3))
    Jpi[:, 0, 0] = w[:, 0] * fx / q[:, 2]
    Jpi[:, 0, 2] = -w[:, 0] * fx * q[:, 0] / q[:, 2] ** 2
    Jpi[:, 1, 1] = w[:, 1] * fy / q[:, 2]
    Jpi[:, 1, 2] = -w[:, 1] * fy * q[:, 1] / q[:, 2] ** 2
    Jp = Jpi @ Rs[oc]
    Jc = np.zeros((O, 2, 6))
    free_obs = oc != pb.fixed
    Jc[free_obs, :, 3:] = Jpi[free_obs]
    # d(R(w) p)/dw = -R [p]x (w w^T + (R^T - I)[w]x) / |w|^2   (-[p]x at w = 0), per camera
    px = np.zeros((O, 3, 3))
    px[:, 0, 1], px[:, 0, 2] = -p[:, 2], p[:, 1]
    px[:, 1, 0], px[:, 1, 2] = p[:, 2], -p[:, 0]
    px[:, 2, 0], px[:, 2, 1] = -p[:, 1], p[:, 0]
    for c in range(C):
        if c == pb.fixed:
            continue
        sel = oc == c
        if not sel.any():
            continue
        wv = cams[c, :3]
        th2 = float(wv @ wv)
        if th2 < 1e-16:
            dR = -px[sel]
        else:
            R = Rs[c]
            M_ = (np.outer(wv, wv) + (R.T - np.eye(3)) @ hat(wv)) / th2
            dR = -(R @ px[sel]) @ M_
        Jc[sel, :, :3] = Jpi[sel] @ dR
    return r, Jc, Jp


def solve_schur(pb, max_iterations=50, function_tolerance=1e-6, gradient_tolerance=1e-10,
                parameter_tolerance=1e-8):
    """`solve` with (H + D) d = -g solved through the reduced camera system.  Same returns."""
    cams, points = pb.cams.copy(), pb.points.copy()
    C, P = cams.shape[0], points.shape[0]
    free = [c for c in range(C) if c != pb.fixed]
    slot = np.full(C, -1)
    slot[free] = np.arange(len(free))
    nf = len(free)
    oc, ok = pb.obs_cam, pb.obs_pt
    os_ = slot[oc]
    fo = os_ >= 0

    def evaluate(cams, points, want_J=True):
        r, Jc, Jp = _blocks(pb, cams, points, want_J)
        return r, Jc, Jp

    r, Jc, Jp = evaluate(cams, points)
    cost = 0.5 * (r * r).sum()
    # jacobi_scaling, fixed after iteration 0
    nc = np.zeros((nf, 6))
    np.add.at(nc, os_[fo], (Jc[fo] ** 2).sum(1))
    npt = np.zeros((P, 3))
    np.add.at(npt, ok, (Jp ** 2).sum(1))
    sc, sp = 1.0 / (1.0 + np.sqrt(nc)), 1.0 / (1.0 + np.sqrt(npt))
    radius, decrease = 1e4, 2.0
    info = {'iterations': 0, 'initial_cost': cost, 'termination': 'max_iterations'}

    def gradient_max(r, Jc, Jp):
        gc = np.zeros((nf, 6))
        np.add.at(gc, os_[fo], np.einsum('oij,oi->oj', Jc[fo], r[fo]))
        gp = np.zeros((P, 3))
        np.add.at(gp, ok, np.einsum('oij,oi->oj', Jp, r))
        return max(np.abs(gc).max() if nf else 0.0, np.abs(gp).max())

    if gradient_max(r, Jc, Jp) <= gradient_tolerance:
        info['termination'] = 'gradient'
        info['final_cost'] = cost
        return cams, points, info
    for it in range(max_iterations):
        info['iterations'] = it + 1
        Jcs = Jc * sc[np.maximum(os_, 0)][:, None, :] * fo[:, None, None]
        Jps = Jp * sp[ok][:, None, :]
        gc = np.zeros((nf, 6))
        np.add.at(gc, os_[fo], np.einsum('oij,oi->oj', Jcs[fo], r[fo]))
        gp = np.zeros((P, 3))
        np.add.at(gp, ok, np.einsum('oij,oi->oj', Jps, r))
        B = np.zeros((nf, 6, 6))
        np.add.at(B, os_[fo], np.einsum('oij,oik->ojk', Jcs[fo], Jcs[fo]))
        Cb = np.zeros((P, 3, 3))
        np.add.at(Cb, ok, np.einsum('oij,oik->ojk', Jps, Jps))
        E = np.zeros((nf, P, 6, 3))
        np.add.at(E, (os_[fo], ok[fo]), np.einsum('oij,oik->ojk', Jcs[fo], Jps[fo]))
        i6, i3 = np.arange(6), np.arange(3)
        B[:, i6, i6] += np.clip(B[:, i6, i6], 1e-6, 1e32) / radius
        Cb[:, i3, i3] += np.clip(Cb[:, i3, i3], 1e-6, 1e32) / radius
        try:
            Ci = np.linalg.inv(Cb)
            ECi = np.einsum('apij,pjk->apik', E, Ci)                       # [nf,P,6,3]
            S = np.zeros((nf * 6, nf * 6))
            for a in range(nf):
                S[6 * a:6 * a + 6, 6 * a:6 * a + 6] = B[a]
            S -= np.einsum('apij,bpkj->aibk', ECi, E).reshape(nf * 6, nf * 6)
            rhs = -gc.reshape(-1) + np.einsum('apij,pj->ai', ECi, gp).reshape(-1)
            dc = np.linalg.solve(S, rhs).reshape(nf, 6)
            dp = np.einsum('pij,pj->pi', Ci, -gp - np.einsum('apij,ai->pj', E, dc))
        except np.linalg.LinAlgError:
            radius /= decrease
            decrease *= 2
            continue
        model = r + np.einsum('oij,oj->oi', Jcs, dc[np.maximum(os_, 0)]) + np.einsum('oij,oj->oi', Jps, dp[ok])
        model_change = cost - 0.5 * (model * model).sum()
        d_c, d_p = dc * sc, dp * sp
        cams_n, points_n = cams.copy(), points.copy()
        cams_n[free] += d_c
        points_n += d_p
        r_n, _, _ = evaluate(cams_n, points_n, want_J=False)
        cost_n = 0.5 * (r_n * r_n).sum()
        step_norm = np.sqrt((d_c ** 2).sum() + (d_p ** 2).sum())
        x_norm = np.sqrt((cams[free] ** 2).sum() + (points ** 2).sum())
        if step_norm <= parameter_tolerance * (x_norm + parameter_tolerance):
            info['termination'] = 'parameter'
            break
        rho = (cost - cost_n) / model_change if model_change > 0 else -1.0
        if rho > 1e-3:
            cost_change = cost - cost_n
            cams, points = cams_n, points_n
            radius = min(radius / max(1.0 / 3.0, 1.0 - (2 * rho - 1) ** 3), 1e16)
            decrease = 2.0
            converged = abs(cost_change) <= function_tolerance * cost
            cost = cost_n
            r, Jc, Jp = evaluate(cams, points)
            if converged:
                info['termination'] = 'function'
                break
            if gradient_max(r, Jc, Jp) <= gradient_tolerance:
                info['termination'] = 'gradient'
                break
        else:
            radius /= decrease
            decrease *= 2
    info['final_cost'] = cost
    return cams, points, info


# ---------------------------------------------------------------------------------------------
# reference known-answer scenes (test_ba_problem.cpp:30-184)
# ---------------------------------------------------------------------------------------------
class _GlibcRand:
    """std::rand() after std::srand(seed) of the gtest (glibc)."""

    def __init__(self, seed):
        self.libc = ctypes.CDLL('libc.so.6')
        self.libc.srand(seed)
        self.RAND_MAX = 2147483647

    def err(self, max_err):
        return self.libc.rand() / self.RAND_MAX * 2.0 * max_err - max_err


def gtest_problem(extr_1, err_cam=0.0, err_2d=0.0, err_3d=0.0):
    """DefineProblem(...) of test_ba_problem.cpp:40-115 (same draw order of the noise)."""
    rnd = _GlibcRand(0)
    err_2d = err_2d / 575.0
    pts = np.array([[-2., 1., 1.], [-1., 0., 1.5], [0., 2., 1.], [1., 0.5, 1.5], [2., -1., 1.]])
    extr_0 = np.zeros(6)
    obs_cam, obs_pt, obs_xy, obs_w = [], [], [], []
    for ci, e in enumerate((extr_0, np.array(extr_1, float))):
        R = angle_axis_to_R(e[:3])
        for k, p in enumerate(pts):
            q = R @ p + e[3:]
            x = q[0] / q[2] + rnd.err(err_2d)
            y = q[1] / q[2] + rnd.err(err_2d)
            obs_cam.append(ci); obs_pt.append(k); obs_xy.append([x, y]); obs_w.append(q[2])  # weight = depth (:66-67)
    e1 = np.array([extr_1[i] + rnd.err(err_cam) for i in range(6)])
    # the file stores R (column major) and ceres::RotationMatrixToAngleAxis reads it back
    e1[:3] = R_to_angle_axis(angle_axis_to_R(e1[:3]))
    cams = np.stack([np.zeros(6), e1])
    pts_init = np.array([[p[0] + rnd.err(err_3d), p[1] + rnd.err(err_3d), p[2] + rnd.err(err_3d)] for p in pts])
    return BaProblem(cams, pts_init, obs_cam, obs_pt, obs_xy, obs_w)


# ---------------------------------------------------------------------------------------------
# bundle_adjust_io.py restatement: spanning tree + problem construction
# ---------------------------------------------------------------------------------------------
def spanning_tree_extrinsics(n_images, rel_pose, weight):
    """initialize_bundle_adjust, bundle_adjust_io.py:135-172.  rel_pose[(i,j)] = T_i->j (4x4),
    weight[(i,j)] > 0 edge weight (number of matches / inliers).  Maximum spanning tree by
    Kruskal on max - w + 1 (scipy's minimum_spanning_tree semantics), absolute poses chained from
    view 0, unreachable views stay identity.  Returns world->cam extrinsics [n,4,4]."""
    from scipy.sparse.csgraph import minimum_spanning_tree
    g = np.zeros((n_images, n_images), dtype=int)
    for (i, j), w in weight.items():
        g[i, j] = int(w)
    mx = g.max()
    nz = g != 0
    g[nz] = mx - g[nz] + 1
    mst = minimum_spanning_tree(g).toarray().astype(int)
    row, col = np.nonzero(mst)
    absp = {0: np.eye(4)}
    for _ in range(n_images):
        for r, c in zip(row, col):
            i, j = (r, c) if r < c else (c, r)
            if j not in absp and i in absp:
                absp[j] = absp[i] @ np.linalg.inv(rel_pose[(i, j)])
            elif i not in absp and j in absp:
                absp[i] = absp[j] @ rel_pose[(i, j)]
        if len(absp) == n_images:
            break
    ext = [np.linalg.inv(absp[i]) if i in absp else np.eye(4) for i in range(n_images)]
    return np.array(ext), [(min(r, c), max(r, c)) for r, c in zip(row, col)]


def triangulate_dlt(P0, P1, x0, x1):
    """cv2.triangulatePoints (bundle_adjust_io.py:222): DLT, smallest right-singular vector."""
    if x0.shape[0] == 0:
        return np.zeros((0, 3))
    A = np.stack([x0[:, 0:1] * P0[2] - P0[0], x0[:, 1:2] * P0[2] - P0[1],
                  x1[:, 0:1] * P1[2] - P1[0], x1[:, 1:2] * P1[2] - P1[1]], 1)       # [n,4,4]
    v = np.linalg.svd(A)[2][:, -1]
    return v[:, :3] / v[:, 3:4]


def build_problem(n_images, pair_matches, extrinsics):
    """write_bundle_adjust_problem, bundle_adjust_io.py:193-259.  pair_matches[(i,j)] =
    (x_i [n,2], x_j [n,2], conf [n]) in NORMALISED image coordinates."""
    obs_cam, obs_pt, obs_xy, obs_c, pts = [], [], [], [], []
    n_pts = 0
    for j in range(n_images):
        for i in range(j):
            if (i, j) not in pair_matches:
                continue
            xi, xj, c = pair_matches[(i, j)]
            n = xi.shape[0]
            p3 = triangulate_dlt(extrinsics[i, :3], extrinsics[j, :3], xi, xj) if n else np.zeros((0, 3))
            for cam, x in ((i, xi), (j, xj)):
                obs_cam += [cam] * n
                obs_pt += list(range(n_pts, n_pts + n))
                obs_xy += list(x)
                obs_c += list(c)
            n_pts += n
            pts.append(p3)
    c = np.array(obs_c, float)
    w = c / (0.5 * (c.sum() + 1e-3))                     # normalize_confidences (:56-60)
    cams = np.array([np.concatenate([R_to_angle_axis(e[:3, :3]), e[:3, 3]]) for e in extrinsics])
    return BaProblem(cams, np.concatenate(pts, 0), obs_cam, obs_pt, obs_xy, w)


def cams_to_extrinsics(cams):
    out = []
    for c in cams:
        T = np.eye(4)
        T[:3, :3] = angle_axis_to_R(c[:3])
        T[:3, 3] = c[3:]
        out.append(T)
    return np.array(out)


# ---------------------------------------------------------------------------------------------
# synthetic multi-view scenes + the whole eval_bundle_adjust flow on the CPU
# ---------------------------------------------------------------------------------------------
def make_multi_view_scene(seed, n_views, n_kpts, outlier_frac=0.1, noise_px=0.5, width=640, height=480,
                          f=577.87, view_counts=None, empty_pairs=()):
    """Landmarks in front of every camera, view 0 = identity, other views rotated <= 12 deg with a
    <= 0.6 m baseline.  Returns pixel keypoints per view, K, GT world->cam poses, and for every pair
    a<b the matcher-style outputs matches_a [n_a] (index into view b or -1) and conf [n_a].
    view_counts: keypoints per view (ragged views, each <= n_kpts; None = n_kpts for every view);
    empty_pairs: pairs (a, b) whose matches are all -1.  With the defaults the scene, random draws
    included, is the one this function has always produced."""
    from .pose import rodrigues
    counts = [n_kpts] * n_views if view_counts is None else [int(c) for c in view_counts]
    assert len(counts) == n_views and max(counts) <= n_kpts
    rng = np.random.default_rng(seed)
    K = np.array([[f, 0, (width - 1) / 2], [0, f, (height - 1) / 2], [0, 0, 1.0]])
    poses = [np.eye(4)]
    for _ in range(1, n_views):
        ax = rng.standard_normal(3)
        ax /= np.linalg.norm(ax)
        T = np.eye(4)
        T[:3, :3] = rodrigues(ax * np.deg2rad(rng.uniform(3, 12)))
        d = rng.standard_normal(3)
        T[:3, 3] = d / np.linalg.norm(d) * rng.uniform(0.2, 0.6)
        poses.append(T)
    land = []
    while len(land) < int(1.3 * n_kpts):
        z = rng.uniform(2, 6)
        uv = rng.uniform([40, 40], [width - 40, height - 40])
        X = np.linalg.inv(K) @ np.array([uv[0], uv[1], 1.0]) * z
        ok = True
        for T in poses:
            q = T[:3, :3] @ X + T[:3, 3]
            px = (K @ q)[:2] / q[2]
            ok &= q[2] > 0.5 and 0 <= px[0] < width and 0 <= px[1] < height
        if ok:
            land.append(X)
    land = np.array(land)
    kpts, ids = [], []
    for T, n_v in zip(poses, counts):
        sel = rng.permutation(len(land))[:n_v]
        q = land[sel] @ T[:3, :3].T + T[:3, 3]
        px = (q @ K.T)[:, :2] / q[:, 2:3] + noise_px * rng.standard_normal((n_v, 2))
        kpts.append(px.astype(np.float32))
        ids.append(sel)
    matches, conf = {}, {}
    for b in range(n_views):
        for a in range(b):
            lut = {l: j for j, l in enumerate(ids[b])}
            m = np.array([lut.get(l, -1) for l in ids[a]], dtype=np.int64)
            c = rng.uniform(0.5, 1.0, counts[a])
            bad = (rng.uniform(size=counts[a]) < outlier_frac) & (m >= 0)
            m[bad] = rng.integers(0, counts[b], int(bad.sum()))
            c[bad] = rng.uniform(0.05, 0.3, int(bad.sum()))
            if (a, b) in empty_pairs:
                m[:] = -1
            matches[(a, b)] = m
            conf[(a, b)] = c.astype(np.float32)
    return {'kpts': kpts, 'K': K.astype(np.float32), 'poses': np.array(poses), 'matches': matches, 'conf': conf}


def multi_view_pipeline(scene, conf_thresh=0.0, n_it2=10, max_iterations=50, use_ba_init=True, min_inliers=20):
    """eval_bundle_adjust (eval_multi_view.py:21-68) without the Theia averaging step (the engine
    does not build it yet): per pair compaction -> w8pt -> two-view BA -> spanning tree -> global BA.
    fp64 throughout."""
    from . import pose as Pz
    T = len(scene['kpts'])
    K = scene['K'].astype(np.float64)[None]
    rel, weight, pm, info_all = {}, {}, {}, {}
    for b in range(T):
        for a in range(b):
            m, c = scene['matches'][(a, b)], scene['conf'][(a, b)].astype(np.float64)
            valid = (m >= 0) & (c > conf_thresh)
            k0 = scene['kpts'][a][valid].astype(np.float64)[None]
            k1 = scene['kpts'][b][m[valid]].astype(np.float64)[None]
            cc = c[valid][None, :, None]
            Tw, info = Pz.estimate_relative_pose_w8pt(k0, k1, K, K, cc, determine_inliers=True)
            if Tw is None:
                pm[(a, b)] = (Pz.normalize(k0, K)[0], Pz.normalize(k1, K)[0], c[valid])
                continue
            cn = info['confidence'].copy()
            cn[~info['pos_depth_mask']] = 0
            ext, vb = Pz.run_bundle_adjust_2_view(info['kpts0_norm'], info['kpts1_norm'], cn, Tw, n_it2)
            Tp = Tw.copy()
            if vb[0]:
                Tp[0] = ext[0]
            rel[(a, b)] = Tp[0]
            weight[(a, b)] = int(valid.sum())
            pm[(a, b)] = (info['kpts0_norm'][0], info['kpts1_norm'][0], c[valid])
            info_all[(a, b)] = {'T_w8pt': Tw[0], 'inliers': info['inliers'][0], 'vote_counts': info['vote_counts'][0]}
    extr0, tree = spanning_tree_extrinsics(T, rel, weight)
    extr_tree = extr0
    if use_ba_init:     # ba_initializer: pairs written to ba_init_in.csv (bundle_adjust_io.py:181-190)
        from .ba_init import ba_initialize
        keep = {k: v for k, v in rel.items() if int(info_all[k]['inliers'].sum()) >= min_inliers or k in tree}
        extr0 = ba_initialize(T, extr_tree, keep)
    pb = build_problem(T, pm, extr0)
    cams, pts, info = solve_schur(pb, max_iterations=max_iterations)
    return {'rel': rel, 'extr_tree': extr_tree, 'extr_init': extr0, 'extr': cams_to_extrinsics(cams), 'info': info, 'pairs': info_all,
            'weight': weight, 'problem': pb}
