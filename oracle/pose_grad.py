"""float64 numpy restatement of the weighted eight-point's gradient with respect to the confidences.  TEST
INFRASTRUCTURE ONLY.

The closed-form backward that csrc/pose_w8pt.cu's w8pt_backward_kernel computes, built on the forward restatement in
``oracle/pose.py``.  PINNED on the reference's own autograd: ``oracle/make_w8pt_grad_golden.py`` runs the unmodified
``estimate_relative_pose_w8pt`` through ``oracle/ref_shim.py`` in fp64, calls ``.backward()`` and asserts that
``w8pt_conf_grad`` reproduces the gradient to 1e-8 of each item's scale; tests/test_w8pt_grad_oracle.py re-checks it
against the stored fixtures without /root/reference.
"""
import numpy as np

from oracle.pose import (compute_rotation_error, compute_translation_error_as_angle,
                         motion_from_essential_choose_solution, normalize, normalize_points, normalize_transformation)


def _eigvec_grad_coeffs(V, lam, j, gv):
    """Gradient through the eigenvector v_j of a symmetric matrix with eigenvectors V (columns) and
    eigenvalues lam: c_k = (v_k . g_v) / (lam_k - lam_j), k != j, so that g_A = -sum_k c_k sym(v_k v_j^T)."""
    c = (V.T @ gv) / np.where(np.arange(len(lam)) == j, 1.0, lam - lam[j])
    c[j] = 0.0
    return c


def w8pt_conf_grad(kpts0, kpts1, intr0, intr1, confidence, grad_T, grad_conf_norm=None, choose_closest=False,
                   T_021=None):
    """float64 gradient of estimate_relative_pose_w8pt's (T021, info["confidence"]) with respect to `confidence`,
    in closed form -- the analytic backward that csrc/pose_w8pt.cu's w8pt_backward_kernel computes.  It
    differentiates the reference's steps: w = c / (sum c + 1e-6); f = last right-singular vector of the weighted
    design matrix X (the smallest-eigenvalue eigenvector of X^T X); the rank-2 projection of F = f.view(3, 3);
    T2^T Fp T1; normalize_transformation; decompose_essential_matrix; the chosen candidate.  Keypoints,
    intrinsics and the target are constants.  Items with fewer than 8 non-zero weights get NaN (their f is not
    unique).  grad_T [B,4,4], grad_conf_norm [B,N] or None -> [B,N]."""
    kpts0, kpts1, intr0, intr1 = (np.asarray(x, np.float64) for x in (kpts0, kpts1, intr0, intr1))
    conf = np.asarray(confidence, np.float64).reshape(kpts0.shape[:2])
    B, N = conf.shape
    out = np.zeros((B, N))
    W0 = np.array([[0., -1, 0], [1, 0, 0], [0, 0, 1]])
    for b in range(B):
        c = conf[b]
        S = c.sum() + 1e-6
        w = c / S
        k0n = normalize(kpts0[b:b + 1], intr0[b:b + 1])
        k1n = normalize(kpts1[b:b + 1], intr1[b:b + 1])
        p1n, T1 = normalize_points(k0n)
        p2n, T2 = normalize_points(k1n)
        x1, y1 = p1n[0, :, 0], p1n[0, :, 1]
        x2, y2 = p2n[0, :, 0], p2n[0, :, 1]
        Xu = np.stack([x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, np.ones_like(x1)], -1)   # [N,9]
        _, sv, Vh = np.linalg.svd(w[:, None] * Xu, full_matrices=True)
        Vx = Vh.T
        lam = np.zeros(9)
        lam[:len(sv)] = sv ** 2
        j = 8 if N > 8 else 7          # the reduced svd's last column (see the N == 8 note in the kernel)
        f = Vx[:, j]
        F = f.reshape(3, 3)
        _, sf, Vft = np.linalg.svd(F)
        v3 = Vft[2]
        Fp = F - np.outer(F @ v3, v3)
        Epre = T2[0].T @ Fp @ T1[0]
        E = normalize_transformation(Epre)
        # decompose_essential_matrix with kornia's det fixes; candidates (R1, t), (R1, -t), (R2, t), (R2, -t)
        U, se, Vt = np.linalg.svd(E)
        if np.linalg.det(U) < 0:
            U[:, 2] *= -1
        if np.linalg.det(Vt) < 0:
            Vt[2] *= -1
        V = Vt.T
        Rs = [U @ W0 @ Vt, U @ W0.T @ Vt]
        if choose_closest:
            ch, best = -1, 1e6
            for k in range(4):
                P = np.eye(4)
                P[:3, :3], P[:3, 3] = Rs[k >> 1], (-1.0 if k & 1 else 1.0) * U[:, 2]
                err = compute_rotation_error(P, T_021[b]) + compute_translation_error_as_angle(P, T_021[b])
                if err < best:
                    ch, best = k, err
        else:
            _, _, _, cnt = motion_from_essential_choose_solution(E[None], k0n, k1n)
            ch = int(cnt[0].argmax())
        gE = np.zeros((3, 3))
        if ch >= 0:
            sg = -1.0 if ch & 1 else 1.0
            Wm = W0 if ch >> 1 == 0 else W0.T
            Gb = U.T @ grad_T[b, :3, :3] @ V
            h = U.T @ (sg * grad_T[b, :3, 3])
            A, Bm = Gb @ Wm.T, Wm.T @ Gb
            al01 = A[0, 1] - A[1, 0]
            al02, al12 = A[0, 2] - A[2, 0] + h[0], A[1, 2] - A[2, 1] + h[1]
            be02, be12 = -(Bm[0, 2] - Bm[2, 0]), -(Bm[1, 2] - Bm[2, 1])
            Q = np.zeros((3, 3))
            Q[0, 1], Q[1, 0] = al01 / (se[0] + se[1]), -al01 / (se[0] + se[1])
            Q[0, 2], Q[2, 0] = -be02 / se[0], -al02 / se[0]
            Q[1, 2], Q[2, 1] = -be12 / se[1], -al12 / se[1]
            gE = U @ Q @ Vt
        if abs(Epre[2, 2]) > 1e-8:
            d = Epre[2, 2] + 1e-8
            dot = (gE * Epre).sum()
            gE = gE / d
            gE[2, 2] -= dot / (d * d)
        G = T2[0] @ gE @ T1[0].T
        gv3 = -(F.T @ G @ v3 + G.T @ F @ v3)
        ck = _eigvec_grad_coeffs(Vft.T, sf ** 2, 2, gv3)
        gA2 = -sum(ck[k] * (np.outer(Vft[k], v3) + np.outer(v3, Vft[k])) for k in range(2))
        gf = (G - np.outer(G @ v3, v3) + F @ gA2).reshape(9)
        cm = _eigvec_grad_coeffs(Vx, lam, j, gf)
        proj = Xu @ Vx                                           # [N,9]: x_i . v_k
        gw = -2.0 * w * proj[:, j] * (proj @ cm)
        if grad_conf_norm is not None:
            gw = gw + np.asarray(grad_conf_norm, np.float64).reshape(B, N)[b]
        g = gw / S - (gw * c).sum() / (S * S)
        out[b] = np.nan if (w != 0).sum() < 8 else g
    return out
