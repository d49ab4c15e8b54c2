"""numpy restatement of the reference's two-view pose path.  TEST INFRASTRUCTURE ONLY.

PINNED on the reference's own code since round 2: ``oracle/ref_shim.py`` imports ``estimate_relative_pose.py`` and
``bundle_adjust_gauss_newton_2_view.py`` from /root/reference UNMODIFIED (stub modules provide only the nine third-party
leaf functions they call) and ``oracle/make_pose_golden.py`` asserts this restatement == the reference (w8pt <= 1e-15 in
fp64, two-view BA <= 6e-10) and writes tests/golden/pose_*.npz, which tests/test_pose_ref_golden.py re-checks without
/root/reference.

PARITY UNPINNED only for those nine leaves: kornia==0.7.0 (requirements.txt:20) and pytorch3d==0.7.5 (requirements.txt:36)
are pip-pinned dependencies absent from /root/reference and from this image.  Their published algorithms are restated
below (function docstrings name the upstream function) and cross-checked against OpenCV 4.13 / SciPy
(tests/test_pose_oracle_opencv.py, tests/test_pose_oracle_scipy.py; cv2.triangulatePoints is also what the reference calls).

fp32 everywhere the reference is fp32 (``dtype=np.float32``); set ``dtype=np.float64`` to get
the same algorithm in double (used to judge which of two fp32 answers is closer to the truth).
"""
import numpy as np


# ----------------------------------------------------------------------------------------
# kornia.geometry restatements
# ----------------------------------------------------------------------------------------
def normalize_points(points, eps=1e-8):
    """kornia.geometry.epipolar.normalize_points: mean-centre, scale so the mean distance to
    the centre is sqrt(2).  points [B,N,2] -> (points_norm [B,N,2], transform [B,3,3])."""
    dt = points.dtype
    x_mean = points.mean(axis=1, keepdims=True)
    scale = np.linalg.norm(points - x_mean, axis=-1).mean(axis=-1)
    scale = (np.sqrt(dt.type(2.0)) / (scale + dt.type(eps))).astype(dt)
    B = points.shape[0]
    T = np.zeros((B, 3, 3), dt)
    T[:, 0, 0] = scale
    T[:, 0, 2] = -scale * x_mean[:, 0, 0]
    T[:, 1, 1] = scale
    T[:, 1, 2] = -scale * x_mean[:, 0, 1]
    T[:, 2, 2] = 1
    ph = np.concatenate([points, np.ones_like(points[..., :1])], -1)
    pn = np.einsum('bij,bnj->bni', T, ph)
    return convert_points_from_homogeneous(pn), T


def convert_points_from_homogeneous(p, eps=1e-8):
    """kornia.geometry.conversions.convert_points_from_homogeneous."""
    dt = p.dtype
    z = p[..., -1:]
    scale = np.where(np.abs(z) > eps, dt.type(1.0) / (z + dt.type(eps)), np.ones_like(z))
    return (scale * p[..., :-1]).astype(dt)


def normalize_transformation(M, eps=1e-8):
    """kornia.geometry.epipolar.normalize_transformation: divide by M[2,2] when |.| > eps."""
    nv = M[..., -1:, -1:]
    return np.where(np.abs(nv) > eps, M / (nv + M.dtype.type(eps)), M).astype(M.dtype)


def _svd(A):
    """torch.svd convention: A = U diag(S) V^T, returns (U, S, V)."""
    U, S, Vh = np.linalg.svd(A, full_matrices=False)
    return U, S, np.swapaxes(Vh, -1, -2)


def decompose_essential_matrix(E):
    """kornia.geometry.epipolar.decompose_essential_matrix."""
    dt = E.dtype
    U, _, V = _svd(E)
    Vt = np.swapaxes(V, -1, -2)
    mask = np.ones_like(E)
    mask[..., -1:] *= -1            # last column negative
    maskt = np.swapaxes(mask, -1, -2)
    U = np.where((np.linalg.det(U) < 0)[..., None, None], U * mask, U)
    Vt = np.where((np.linalg.det(Vt) < 0)[..., None, None], Vt * maskt, Vt)
    W = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1]], dt)
    R1 = U @ W @ Vt
    R2 = U @ W.T @ Vt
    t = U[..., -1:]
    return R1.astype(dt), R2.astype(dt), t.astype(dt)


def motion_from_essential(E):
    """kornia.geometry.epipolar.motion_from_essential -> Rs [B,4,3,3], ts [B,4,3,1] in the order
    (R1,t), (R1,-t), (R2,t), (R2,-t)."""
    R1, R2, t = decompose_essential_matrix(E)
    return np.stack([R1, R1, R2, R2], 1), np.stack([t, -t, t, -t], 1)


def triangulate_points(P1, P2, x1, x2):
    """kornia.geometry.epipolar.triangulate_points (DLT, last right-singular vector of the 4x4).
    P1,P2 [...,3,4]; x1,x2 [...,N,2] -> [...,N,3]."""
    dt = x1.dtype
    lead = np.broadcast_shapes(x1.shape[:-2], P1.shape[:-2], P2.shape[:-2])
    X = np.zeros(lead + (x1.shape[-2], 4, 4), dt)
    for i in range(4):
        X[..., 0, i] = x1[..., 0] * P1[..., 2:3, i] - P1[..., 0:1, i]
        X[..., 1, i] = x1[..., 1] * P1[..., 2:3, i] - P1[..., 1:2, i]
        X[..., 2, i] = x2[..., 0] * P2[..., 2:3, i] - P2[..., 0:1, i]
        X[..., 3, i] = x2[..., 1] * P2[..., 2:3, i] - P2[..., 1:2, i]
    _, _, V = _svd(X)
    return convert_points_from_homogeneous(V[..., -1])


def depth_from_point(R, t, X):
    """kornia.geometry.epipolar.projection.depth_from_point: (R X)_z + t_z."""
    Xt = R @ np.swapaxes(X, -1, -2)
    return Xt[..., 2, :] + t[..., 2, :]


def motion_from_essential_choose_solution(E, x1, x2):
    """kornia.geometry.epipolar.motion_from_essential_choose_solution with K1=K2=I, mask=None.
    Per batch element (the 0.7.0 indexing quirk only matters for B>1, which the reference never
    uses on this branch -- SURVEY.md A.5): candidate with the most points of positive depth in
    both cameras, first maximum wins."""
    dt = E.dtype
    Rs, ts = motion_from_essential(E)
    B = E.shape[0]
    P1 = np.zeros((B, 4, 3, 4), dt)
    P1[..., :3, :3] = np.eye(3, dtype=dt)
    P2 = np.concatenate([Rs, ts], -1)
    X = triangulate_points(P1, P2, x1[:, None], x2[:, None])       # [B,4,N,3]
    R1 = np.broadcast_to(np.eye(3, dtype=dt), (B, 4, 3, 3))
    t1 = np.zeros((B, 4, 3, 1), dt)
    d1 = depth_from_point(R1, t1, X)
    d2 = depth_from_point(Rs, ts, X)
    cnt = ((d1 > 0) & (d2 > 0)).sum(-1)                            # [B,4]
    idx = cnt.argmax(-1)
    bi = np.arange(B)
    return Rs[bi, idx], ts[bi, idx], X[bi, idx], cnt


def symmetrical_epipolar_distance(p1, p2, F):
    """kornia.geometry.epipolar.symmetrical_epipolar_distance (squared=True)."""
    p1h = np.concatenate([p1, np.ones_like(p1[..., :1])], -1)
    p2h = np.concatenate([p2, np.ones_like(p2[..., :1])], -1)
    l1in2 = p1h @ np.swapaxes(F, -1, -2)
    l2in1 = p2h @ F
    num = (p2h * l1in2).sum(-1) ** 2
    den_inv = 1.0 / (np.linalg.norm(l1in2[..., :2], axis=-1) ** 2) + \
        1.0 / (np.linalg.norm(l2in1[..., :2], axis=-1) ** 2)
    return (num * den_inv).astype(p1.dtype)


# ----------------------------------------------------------------------------------------
# pytorch3d restatements
# ----------------------------------------------------------------------------------------
def hat(v):
    """pytorch3d.transforms.so3.hat."""
    x, y, z = v[..., 0], v[..., 1], v[..., 2]
    o = np.zeros_like(x)
    return np.stack([np.stack([o, -z, y], -1), np.stack([z, o, -x], -1), np.stack([-y, x, o], -1)], -2)


def se3_exp_map_T(log_transform, eps=1e-4):
    """pytorch3d.transforms.se3_exp_map followed by the reference's ``.permute(0,2,1)``
    (bundle_adjust_gauss_newton_2_view.py:194): returns [[R, V t],[0,1]] with
    theta = sqrt(clamp(|w|^2, eps))."""
    dt = log_transform.dtype
    v, w = log_transform[..., :3], log_transform[..., 3:]
    nrms = (w * w).sum(-1)
    th = np.sqrt(np.maximum(nrms, dt.type(eps)))
    K = hat(w)
    K2 = K @ K
    I = np.eye(3, dtype=dt)
    fac1 = np.sin(th) / th
    fac2 = (1 - np.cos(th)) / (th * th)
    R = fac1[..., None, None] * K + fac2[..., None, None] * K2 + I
    V = I + K * ((1 - np.cos(th)) / th ** 2)[..., None, None] + \
        K2 * ((th - np.sin(th)) / th ** 3)[..., None, None]
    T = np.zeros(log_transform.shape[:-1] + (4, 4), dt)
    T[..., :3, :3] = R
    T[..., :3, 3] = (V @ v[..., None])[..., 0]
    T[..., 3, 3] = 1
    return T.astype(dt)


# ----------------------------------------------------------------------------------------
# the reference's own code: pose_optimization/two_view/*.py
# ----------------------------------------------------------------------------------------
def normalize(kpts, intr):
    """estimate_relative_pose.py:9-14 (intr 3x3 or 4x4)."""
    out = np.zeros_like(kpts)
    fx, fy, cx, cy = intr[..., 0, 0], intr[..., 1, 1], intr[..., 0, 2], intr[..., 1, 2]
    out[..., 0] = (kpts[..., 0] - cx[..., None]) / fx[..., None]
    out[..., 1] = (kpts[..., 1] - cy[..., None]) / fy[..., None]
    return out


def find_fundamental(points1, points2, weights):
    """estimate_relative_pose.py:34-82 (weighted DLT; weights enter linearly in X)."""
    dt = points1.dtype
    p1n, T1 = normalize_points(points1)
    p2n, T2 = normalize_points(points2)
    x1, y1 = p1n[..., 0:1], p1n[..., 1:2]
    x2, y2 = p2n[..., 0:1], p2n[..., 1:2]
    ones = np.ones_like(x1)
    X = np.concatenate([x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, ones], -1)  # :65
    X = weights[..., None] * X                                                          # :68-69
    _, _, V = _svd(X)                                                                   # :72
    Fm = V[..., -1].reshape(-1, 3, 3)
    U, S, V = _svd(Fm)                                                                  # :76
    S = S * np.array([1, 1, 0], dt)
    Fp = U @ (S[..., None] * np.swapaxes(V, -1, -2))
    Fe = np.swapaxes(T2, -1, -2) @ (Fp @ T1)                                            # :80
    return normalize_transformation(Fe.astype(dt))                                      # :82


def compute_rotation_error(T0, T1):
    """compute_pose_error.py:3-12 (reduce=False)."""
    tr = np.trace(np.swapaxes(T0[..., :3, :3], -1, -2) @ T1[..., :3, :3], axis1=-2, axis2=-1)
    return np.abs(np.arccos(np.clip((tr - 1) / 2, -1, 1)))


def compute_translation_error_as_angle(T0, T1):
    """compute_pose_error.py:14-21 (reduce=False; pairs with |t0||t1| <= 1e-6 are dropped by the
    reference -- here they yield 0 so the shape is kept)."""
    n = np.linalg.norm(T0[..., :3, 3], axis=-1) * np.linalg.norm(T1[..., :3, 3], axis=-1)
    dot = (T0[..., :3, 3] * T1[..., :3, 3]).sum(-1)
    safe = np.where(n > 1e-6, n, 1)
    return np.where(n > 1e-6, np.abs(np.arccos(np.clip(dot / safe, -1, 1))), 0).astype(T0.dtype)


def estimate_relative_pose_w8pt(kpts0, kpts1, intr0, intr1, confidence, choose_closest=False,
                                T_021=None, determine_inliers=False):
    """estimate_relative_pose.py:84-128.  confidence [B,N,1]."""
    if kpts0.shape[1] < 8:
        return None, None
    dt = kpts0.dtype
    sum_conf = confidence.sum(axis=1, keepdims=True) + dt.type(1e-6)
    confidence = (confidence / sum_conf).astype(dt)
    k0n = normalize(kpts0, intr0)
    k1n = normalize(kpts1, intr1)
    B = intr0.shape[0]
    vote_counts = None
    Fs = find_fundamental(k0n, k1n, confidence[..., 0])
    T = np.tile(np.eye(4, dtype=dt), (B, 1, 1))
    if choose_closest:
        Rs, ts = motion_from_essential(Fs)
        min_err = np.full(B, 1e6, dt)
        for c in range(4):
            P = np.tile(np.eye(4, dtype=dt), (B, 1, 1))
            P[:, :3, :3] = Rs[:, c]
            P[:, :3, 3] = ts[:, c, :, 0]
            err = compute_rotation_error(P, T_021) + compute_translation_error_as_angle(P, T_021)
            upd = err < min_err
            min_err[upd] = err[upd]
            T[upd] = P[upd]
    else:
        R, t, _, vote_counts = motion_from_essential_choose_solution(Fs, k0n, k1n)
        T[:, :3, :3] = R
        T[:, :3, 3] = t[..., 0]
    P0 = np.tile(np.eye(4, dtype=dt)[:3], (B, 1, 1))
    pts = triangulate_points(P0, T[:, :3, :], k0n, k1n)
    depth0 = pts[..., -1]
    depth1 = depth_from_point(T[:, :3, :3], T[:, :3, 3:], pts)
    pos = (depth0 > 0) & (depth1 > 0)
    inliers = None
    if determine_inliers:
        epi = np.sqrt(symmetrical_epipolar_distance(k0n, k1n, Fs))
        thresh = 3.0 / ((intr0[:, 0, 0] + intr0[:, 1, 1] + intr1[:, 0, 0] + intr1[:, 1, 1]) / 4.0)
        inliers = pos & (epi <= thresh[:, None])
    info = {'kpts0_norm': k0n, 'kpts1_norm': k1n, 'confidence': confidence, 'inliers': inliers,
            'pos_depth_mask': pos, 'F': Fs, 'vote_counts': vote_counts}
    return T, info


def _ba_residual_jacobian(T1, pts3d, x0, x1, w):
    """fill_J / compute_A_b for one batch element (bundle_adjust_gauss_newton_2_view.py:50-99).
    Observation order follows Observations.add_matches (:24-33): all cam-0 observations, then all
    cam-1 observations.  Unknown order: 6 camera DoF [v | omega], then 3 per point."""
    dt = pts3d.dtype
    n = pts3d.shape[0]
    J = np.zeros((4 * n, 6 + 3 * n), dt)
    r = np.zeros((4 * n,), dt)
    I3 = np.eye(3, dtype=dt)
    for cam, (obs, Tm) in enumerate(((x0, np.eye(4, dtype=dt)), (x1, T1))):
        Ap = pts3d @ Tm[:3, :3].T + Tm[:3, 3]
        pi = Ap[:, :2] / Ap[:, 2:3]
        Jp = np.zeros((n, 2, 3), dt)
        Jp[:, 0, 0] = 1 / Ap[:, 2]
        Jp[:, 0, 2] = -Ap[:, 0] / Ap[:, 2] ** 2
        Jp[:, 1, 1] = 1 / Ap[:, 2]
        Jp[:, 1, 2] = -Ap[:, 1] / Ap[:, 2] ** 2
        Jpt = w[:, None, None] * (Jp @ Tm[:3, :3])
        rows = (cam * n + np.arange(n)) * 2
        for k in range(n):
            J[rows[k]:rows[k] + 2, 6 + 3 * k:9 + 3 * k] = Jpt[k]
        if cam == 1:
            IA = np.concatenate([np.broadcast_to(I3, (n, 3, 3)), -hat(Ap)], 2)
            Jc = w[:, None, None] * (Jp @ IA)
            for k in range(n):
                J[rows[k]:rows[k] + 2, 0:6] = Jc[k]
        rr = w[:, None] * (pi - obs)
        r[cam * 2 * n:(cam + 1) * 2 * n] = rr.reshape(-1)
    return J, r


def run_bundle_adjust_2_view(kpts0_norm, kpts1_norm, confidence, init_T021, n_iterations=10,
                             lm_increase=1.5, lm_decrease=3.5, return_trace=False, jacobi_precond=True):
    """run_bundle_adjust_2_view (estimate_relative_pose.py:138-143) ->
    BundleAdjustGaussNewton2View.run (bundle_adjust_gauss_newton_2_view.py:127-201) with the
    defaults jacobi_precond=True, vary_lm_fact=True, non-strict checks.  Dense (6+3n)^2 solve
    like the reference: keep n small.  Returns (extrinsics of valid batches [nv,4,4], valid [B])."""
    dt = kpts0_norm.dtype
    B = kpts0_norm.shape[0]
    conf = confidence[..., 0] if confidence.ndim == 3 else confidence
    valid = conf > 0
    n_matches = valid.sum(-1)
    valid_batch = n_matches > 6
    out = []
    trace = []
    for b in range(B):
        if not valid_batch[b]:
            continue
        mk = valid[b]
        x0, x1, c = kpts0_norm[b][mk], kpts1_norm[b][mk], conf[b][mk]
        # normalize_confidences (:44-48): obs conf / (0.5 * sum over the 2n observations)
        c2 = np.concatenate([c, c])
        w = (c / (dt.type(0.5) * max(c2.sum(), dt.type(1e-6)))).astype(dt)
        T1 = init_T021[b].astype(dt).copy()
        P0 = np.eye(4, dtype=dt)[:3]
        pts = triangulate_points(P0[None], T1[None, :3], x0[None], x1[None])[0]     # :115-125
        best_T, best_r = T1.copy(), None
        lam = dt.type(0.1)
        tr = []
        for i in range(n_iterations + 1):
            J, r = _ba_residual_jacobian(T1, pts, x0, x1, w)
            A = J.T @ J
            bvec = -J.T @ r
            rn = (r ** 2).sum()
            tr.append(float(rn))
            if i == 0:
                best_r = rn
                best_T = T1.copy()
            else:
                if rn < best_r:                       # :160-165
                    best_r = rn
                    best_T = T1.copy()
                    lam = lam / dt.type(lm_decrease)
                else:
                    lam = lam * dt.type(lm_increase)
            if i == n_iterations:
                break
            dA = np.diagonal(A)
            if jacobi_precond and (dA > 0).all():     # :171-177 Jacobi scaling
                inv = 1.0 / np.maximum(dA, dt.type(1e-12))
                A = inv[:, None] * A
                bvec = inv * bvec
            A = A + np.eye(A.shape[0], dtype=dt) * lam
            try:
                dx = np.linalg.solve(A, bvec)         # LU with partial pivoting (:184-188)
            except np.linalg.LinAlgError:
                continue
            dT = se3_exp_map_T(dx[None, :6].astype(dt))[0]
            T1 = (dT @ T1).astype(dt)                 # :195
            pts = (pts + dx[6:].reshape(-1, 3)).astype(dt)
        out.append(best_T)
        trace.append(tr)
    ext = np.stack(out, 0) if out else np.zeros((0, 4, 4), dt)
    if return_trace:
        return ext, valid_batch, trace
    return ext, valid_batch


def _inv3_sym(M):
    """Inverse of symmetric 3x3 blocks [n,3,3] by cofactors; ok [n] is False where the determinant is
    not a non-zero number (the block is singular to float64)."""
    a00, a01, a02 = M[:, 0, 0], M[:, 0, 1], M[:, 0, 2]
    a11, a12, a22 = M[:, 1, 1], M[:, 1, 2], M[:, 2, 2]
    c00 = a11 * a22 - a12 * a12
    c01 = a02 * a12 - a01 * a22
    c02 = a01 * a12 - a02 * a11
    det = a00 * c00 + a01 * c01 + a02 * c02
    ok = np.abs(det) > 0.0
    with np.errstate(divide='ignore', invalid='ignore'):
        idet = 1.0 / det
        c11 = a00 * a22 - a02 * a02
        c12 = a01 * a02 - a00 * a12
        c22 = a00 * a11 - a01 * a01
        inv = np.stack([np.stack([c00, c01, c02], -1), np.stack([c01, c11, c12], -1),
                        np.stack([c02, c12, c22], -1)], -2) * idet[:, None, None]
    return inv, ok


def _ba_point_blocks(T1, pts, x0, x1, w):
    """Per-point blocks of the normal equations of _ba_residual_jacobian's problem, without forming J:
    App [n,3,3] (point), Acp [n,6,3] (camera x point), bp [n,3], and the sums Acc [6,6], bc [6] and
    the squared residual norm."""
    R, t = T1[:3, :3], T1[:3, 3]

    def proj_jac(q):
        iz = 1.0 / q[:, 2]
        J = np.zeros((q.shape[0], 2, 3))
        J[:, 0, 0] = iz
        J[:, 1, 1] = iz
        J[:, 0, 2] = -q[:, 0] * iz * iz
        J[:, 1, 2] = -q[:, 1] * iz * iz
        return w[:, None, None] * J, w[:, None] * (q[:, :2] * iz[:, None])

    J0, pr0 = proj_jac(pts)
    r0 = pr0 - w[:, None] * x0
    q = pts @ R.T + t
    Jpi, pr1 = proj_jac(q)
    r1 = pr1 - w[:, None] * x1
    J1 = Jpi @ R
    IA = np.concatenate([np.broadcast_to(np.eye(3), (q.shape[0], 3, 3)), -hat(q)], 2)
    Jc = Jpi @ IA                                                               # [n,2,6]
    tr = lambda X: np.swapaxes(X, -1, -2)
    App = tr(J0) @ J0 + tr(J1) @ J1
    Acp = tr(Jc) @ J1
    bp = -((tr(J0) @ r0[..., None]) + (tr(J1) @ r1[..., None]))[..., 0]
    Acc = (tr(Jc) @ Jc).sum(0)
    bc = -(tr(Jc) @ r1[..., None])[..., 0].sum(0)
    rho = float((r0 ** 2).sum() + (r1 ** 2).sum())
    return App, Acp, bp, Acc, bc, rho


def triangulate_points_first_view_identity(T1, x0, x1, dlt='svd'):
    """triangulate_points with P0 = [I|0], P1 = T1[:3] and one rule for a degenerate match: when the match sits
    at the principal point of camera 0 and camera 1 observes it where camera 0's optical axis and camera 0's centre
    both project (x0 = 0 and columns z and w of the 4x4 DLT matrix are exactly zero), the null space of the DLT
    matrix is span(e_z, e_w) and the point is not unique.  The SVD then returns e_w, camera 0's centre, whose zero
    depth makes the BA's Jacobians infinite; here the point is e_z, (0, 0, 1), which is what the smallest
    eigenvector of A^T A by cyclic Jacobi gives (no rotation touches the zero rows and columns, and the first
    smallest diagonal entry wins).  x0, x1 [n,2] -> [n,3] float64.

    dlt='normal' takes the smallest eigenvector of A^T A instead of the smallest right-singular vector of A: the
    same point in exact arithmetic, but its rounding error grows with cond(A)^2 instead of cond(A), which is what a
    solver working on A^T A (as the CUDA kernels do) carries on near-parallel rays."""
    R, t = T1[:3, :3], T1[:3, 3]
    if dlt == 'svd':
        X = triangulate_points(np.eye(4)[:3][None], T1[None, :3], x0[None], x1[None])[0]
    else:
        assert dlt == 'normal', dlt
        A = np.zeros((x0.shape[0], 4, 4))
        A[:, 0, 0] = A[:, 1, 1] = -1.0
        A[:, 0, 2], A[:, 1, 2] = x0[:, 0], x0[:, 1]
        A[:, 2, :3] = x1[:, 0:1] * R[2] - R[0]
        A[:, 3, :3] = x1[:, 1:2] * R[2] - R[1]
        A[:, 2, 3], A[:, 3, 3] = x1[:, 0] * t[2] - t[0], x1[:, 1] * t[2] - t[1]
        h = np.linalg.eigh(np.swapaxes(A, 1, 2) @ A)[1][:, :, 0]
        X = convert_points_from_homogeneous(h)
    colz = np.stack([x0[:, 0], x0[:, 1], x1[:, 0] * R[2, 2] - R[0, 2], x1[:, 1] * R[2, 2] - R[1, 2]], 1)
    colw = np.stack([x1[:, 0] * t[2] - t[0], x1[:, 1] * t[2] - t[1]], 1)
    tie = ~colz.any(1) & ~colw.any(1)
    X[tie] = [0.0, 0.0, 1.0]
    return X


def run_bundle_adjust_2_view_schur(kpts0_norm, kpts1_norm, confidence, init_T021, n_iterations=10,
                                   lm_increase=1.5, lm_decrease=3.5, jacobi_precond=True, dlt='svd'):
    """run_bundle_adjust_2_view in float64 with the 3x3 point blocks eliminated (Schur complement)
    instead of the dense (6+3n)^2 solve: the same LM iteration at any n.

    For every item: valid matches conf > 0, excluded (T_init returned) with <= 6 of them; weights
    conf / (0.5 * max(sum over the 2n observations, 1e-6)); points triangulated with T_init; n_iterations+1
    evaluations of the squared residual norm (the trace), lambda0 = 0.1, lambda / lm_decrease on a new
    best residual and * lm_increase otherwise; each step solves (A + lambda D) delta = b with D = max(diag A,
    1e-12) when every diagonal entry is positive (Jacobi scaling) and D = I otherwise, and is applied
    unconditionally; the best evaluated pose is returned.  The points are triangulated by
    triangulate_points_first_view_identity (a match on both optical axes of a forward motion becomes (0, 0, 1);
    dlt selects its solver).  A step is skipped (nothing moves) when a damped
    point block has a zero determinant, when the 6x6 camera system is singular, or when its solution is
    not finite.

    Returns (T_out [B,4,4] with T_init for excluded items, valid [B], trace: a list with an
    [n_iterations+1] array per item, None for excluded ones)."""
    B = kpts0_norm.shape[0]
    conf = confidence[..., 0] if confidence.ndim == 3 else confidence
    T_out = np.array(init_T021, np.float64).copy()
    valid_batch = np.zeros(B, bool)
    traces = []
    for b in range(B):
        mk = conf[b] > 0
        if mk.sum() <= 6:
            traces.append(None)
            continue
        valid_batch[b] = True
        x0 = np.asarray(kpts0_norm[b][mk], np.float64)
        x1 = np.asarray(kpts1_norm[b][mk], np.float64)
        c = np.asarray(conf[b][mk], np.float64)
        w = c / (0.5 * max(2.0 * c.sum(), 1e-6))
        T1 = np.array(init_T021[b], np.float64).copy()
        T1[3] = [0, 0, 0, 1]
        pts = triangulate_points_first_view_identity(T1, x0, x1, dlt)
        best_T, best_r, lam = T1.copy(), None, 0.1
        tr = []
        for i in range(n_iterations + 1):
            App, Acp, bp, Acc, bc, rn = _ba_point_blocks(T1, pts, x0, x1, w)
            tr.append(rn)
            if i == 0:
                best_r, best_T = rn, T1.copy()
            elif rn < best_r:
                best_r, best_T = rn, T1.copy()
                lam = lam / lm_decrease
            else:
                lam = lam * lm_increase
            if i == n_iterations:
                break
            dP = np.diagonal(App, axis1=1, axis2=2)
            dC = np.diagonal(Acc)
            if jacobi_precond and (dP > 0).all() and (dC > 0).all():
                Dp, Dc = np.maximum(dP, 1e-12), np.maximum(dC, 1e-12)
            else:
                Dp, Dc = np.ones_like(dP), np.ones(6)
            Mi, ok = _inv3_sym(App + lam * Dp[:, :, None] * np.eye(3))
            if not ok.all():
                continue
            Y = Acp @ Mi                                                    # [n,6,3]
            S = Acc - (Y @ np.swapaxes(Acp, 1, 2)).sum(0) + lam * np.diag(Dc)
            g = bc - (Y @ bp[..., None])[..., 0].sum(0)
            try:
                dc = np.linalg.solve(S, g)
            except np.linalg.LinAlgError:
                continue
            if not np.isfinite(dc).all():
                continue
            dp = (Mi @ (bp - (np.swapaxes(Acp, 1, 2) @ dc))[..., None])[..., 0]
            T1 = se3_exp_map_T(dc[None])[0] @ T1
            pts = pts + dp
        T_out[b] = best_T
        traces.append(np.array(tr))
    return T_out, valid_batch, traces


# ----------------------------------------------------------------------------------------
# metrics (models/models/utils.py:377-409), numpy fp64 like the reference
# ----------------------------------------------------------------------------------------
def angle_error_mat(R1, R2):
    cos = (np.trace(np.dot(R1.T, R2)) - 1) / 2
    return np.rad2deg(np.abs(np.arccos(np.clip(cos, -1., 1.))))


def angle_error_vec(v1, v2):
    n = np.linalg.norm(v1) * np.linalg.norm(v2)
    return np.rad2deg(np.arccos(np.clip(np.dot(v1, v2) / n, -1.0, 1.0)))


def compute_pose_error(T_0to1, R, t):
    """models/models/utils.py:388-395."""
    et = angle_error_vec(t, T_0to1[:3, 3])
    et = np.minimum(et, 180 - et)
    return et, angle_error_mat(R, T_0to1[:3, :3])


def pose_auc(errors, thresholds):
    """models/models/utils.py:397-409."""
    sort_idx = np.argsort(errors)
    errors = np.array(errors.copy())[sort_idx]
    recall = (np.arange(len(errors)) + 1) / len(errors)
    errors = np.r_[0., errors]
    recall = np.r_[0., recall]
    aucs = []
    for t in thresholds:
        last_index = np.searchsorted(errors, t)
        r = np.r_[recall[:last_index], recall[last_index - 1]]
        e = np.r_[errors[:last_index], t]
        aucs.append(np.trapezoid(r, x=e) / t)
    return aucs


# ----------------------------------------------------------------------------------------
# synthetic two-view scenes (SURVEY.md §8d)
# ----------------------------------------------------------------------------------------
def rodrigues(w):
    th = np.linalg.norm(w)
    if th < 1e-12:
        return np.eye(3)
    K = hat(w / th)
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)


def make_two_view_scene(seed, n, outlier_frac=0.3, noise_px=1.0, width=640, height=480,
                        f=577.87, dtype=np.float32, motion='random', rot_deg=(5, 30)):
    """3-D points in the frustum of camera 0 (depth 1..5 m), K = [[f,0,319.5],[0,f,239.5],[0,0,1]],
    1 px noise, 30 % outlier matches, confidences U(0.5,1) inliers / U(0,0.3) outliers.  Camera 1:
      motion='random'  rotated by U(rot_deg) degrees (default 5..30) about a random axis, 0.1..1 m
                       baseline in a random direction (the defaults give the scenes this function
                       has always produced);
      motion='forward' rotated by U(rot_deg) degrees, centre 0.1..0.5 m straight ahead of camera 0
                       (rot_deg=(0, 0): pure forward motion, the epipole at the principal point);
      motion='orbit'   rotated by U(rot_deg) degrees about an axis in camera 0's image plane and
                       looking at the point 3 m ahead of camera 0 from 3 m away: relative rotations
                       past 90 deg (e.g. rot_deg=(130, 179)) with every point in front of both."""
    rng = np.random.default_rng(seed)
    K = np.array([[f, 0, (width - 1) / 2], [0, f, (height - 1) / 2], [0, 0, 1]], np.float64)
    axis = rng.standard_normal(3)
    if motion == 'orbit':
        axis[2] = 0.0
    axis /= np.linalg.norm(axis)
    R = rodrigues(axis * np.deg2rad(rng.uniform(*rot_deg)))
    tdir = rng.standard_normal(3)
    tdir /= np.linalg.norm(tdir)
    t = tdir * rng.uniform(0.1, 1.0)
    if motion == 'forward':
        t = -R @ np.array([0.0, 0.0, rng.uniform(0.1, 0.5)])
    elif motion == 'orbit':
        t = np.array([0.0, 0.0, 3.0]) - R @ np.array([0.0, 0.0, 3.0])
    else:
        assert motion == 'random', motion
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    pts0, pts1 = [], []
    while len(pts0) < n:
        z = rng.uniform(1, 5)
        uv = rng.uniform([0, 0], [width, height])
        X = np.linalg.inv(K) @ np.array([uv[0], uv[1], 1.0]) * z
        X1 = R @ X + t
        if X1[2] <= 0.1:
            continue
        uv1 = (K @ X1)[:2] / X1[2]
        if not (0 <= uv1[0] < width and 0 <= uv1[1] < height):
            continue
        pts0.append(uv)
        pts1.append(uv1)
    k0 = np.array(pts0) + noise_px * rng.standard_normal((n, 2))
    k1 = np.array(pts1) + noise_px * rng.standard_normal((n, 2))
    out = rng.uniform(size=n) < outlier_frac
    k1[out] = rng.uniform([0, 0], [width, height], size=(int(out.sum()), 2))
    conf = np.where(out, rng.uniform(0, 0.3, n), rng.uniform(0.5, 1.0, n))
    return {'kpts0': k0.astype(dtype)[None], 'kpts1': k1.astype(dtype)[None],
            'intr': K.astype(dtype)[None], 'conf': conf.astype(dtype)[None, :, None],
            'T_021': T.astype(dtype)[None], 'outlier': out[None]}
