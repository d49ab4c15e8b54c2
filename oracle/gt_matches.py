"""float64 restatement of the ground-truth matching of an image pair (helpers.py:115-213), the rules of
csrc/gt_matches.cu where the reference leaves the result undefined, and the intermediates a test needs to tell a
stable decision from one float32 rounding can flip.

TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.  Pinned on the reference's own outputs by
tests/test_gt_matches_oracle.py.

What is computed, per batch item and with n keypoints per view:
  - the keypoint pixel is the coordinate truncated toward zero (`.long()`); the depth is read there.  The reference
    indexes the depth map with that pixel and fails on one outside the image; the kernel clamps the pixel to the border
    for the depth look-up and the back-projection, and this module does the same.  The reprojection error below uses
    the truncated pixel without the clamp, as the reference does;
  - view s is reprojected into view o = 1 - s with M = K_o . T_so . inv(K_s) (T_01 = T0to1, T_10 = inv(T0to1)) applied
    to (x d, y d, d, 1); z is the third row, the projection (row 0, row 1) / z;
  - the error of keypoint i of view 0 and j of view 1 is (|p10_j - k0_i| + |p01_i - k1_j|) / 2;
  - row and column arg-min, the first index on ties (torch.argmin);
  - keypoint i of view 0 matches i1 = rowmin_i when colmin_i1 == i, err <= max_matched, d0_i > 1e-6, d1_i1 > 1e-6,
    |z01_i - d1_i1| / d1_i1 < 0.1 and |z10_i1 - d0_i| / d0_i < 0.1;
  - an unmatched keypoint is dropped (weight 0) when a depth of it or of its arg-min partner is not valid, or its
    arg-min error is <= min_unmatched;
  - class balancing in float32 from the integer counts: w_match = 2 M / (2 n - D), w_unmatch = 0.5 / (1 - w_match),
    w_match = 0.5 / w_match; both are 0 when either is not finite (no match, every keypoint matched, every keypoint
    dropped).  Dustbin entries (index n) never match and carry w_unmatch.
Inputs with NaN or infinite coordinates are outside this definition (and outside the kernel's).
"""
import numpy as np

F32 = np.float32
EPS32 = float(np.finfo(np.float32).eps)


def _pixels(kpts, H, W):
    """(truncated pixel [n, 2] int64, the same clamped into the image)."""
    t = np.trunc(np.asarray(kpts, np.float64)).astype(np.int64)
    c = t.copy()
    c[:, 0] = np.clip(c[:, 0], 0, W - 1)
    c[:, 1] = np.clip(c[:, 1], 0, H - 1)
    return t, c


def _project(pix_c, d, M):
    """M [4, 4] float64 applied to (x d, y d, d, 1): (projection [n, 2], depth [n], noise [n]).  noise is a bound on
    the float32 rounding of the projection: ~ulp-level error of each product, scaled by the size of the terms over |z|
    (it grows without limit as z -> 0)."""
    v = np.stack([pix_c[:, 0] * d, pix_c[:, 1] * d, d, np.ones_like(d)], 1)
    p = v @ M[:3].T
    mag = np.abs(v) @ np.abs(M[:3]).T                      # [n, 3] sum of |terms| per row
    with np.errstate(divide='ignore', invalid='ignore'):
        proj = p[:, :2] / p[:, 2:3]
        az = np.abs(p[:, 2])
        noise = 8 * EPS32 * (mag[:, :2].max(1) + mag[:, 2] * np.abs(proj).max(1)) / az + 4 * EPS32 * np.abs(proj).max(1)
    noise = np.where(np.isfinite(noise), noise, np.inf)
    return proj, p[:, 2], noise


def _argmin_first(e):
    """Arg-min along axis 1 with the first index on ties, and the minimum.  A NaN error wins, like torch.argmin's."""
    nan = np.isnan(e)
    a = np.where(nan.any(1), nan.argmax(1), np.argmin(np.where(nan, np.inf, e), 1))
    return a, e[np.arange(e.shape[0]), a]


def _margin(e, amin, groups):
    """Distance from the minimum to the smallest error of a candidate in another pixel group, and that candidate.
    Candidates that share the arg-min's truncated pixel get the same error in any precision, so they never make a
    decision unstable (the first index wins among them in float32 and float64 alike)."""
    same = groups[None, :] == groups[amin][:, None]
    other = np.where(same | np.isnan(e), np.inf, e)
    runner = other.argmin(1)
    return other[np.arange(e.shape[0]), runner] - e[np.arange(e.shape[0]), amin], runner


def _weights(n, n_match, n_drop):
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        mw = (F32(2) * F32(n_match)) / (F32(2) * F32(n) - F32(n_drop))
        uw = F32(0.5) / (F32(1) - mw)
        mw = F32(0.5) / mw
    if not (np.isfinite(mw) and np.isfinite(uw)):
        return F32(0), F32(0)
    return F32(mw), F32(uw)


def gt_matches_pair(kpts0, kpts1, K0, K1, T0to1, depth0, depth1, max_matched, min_unmatched, tau=1e-3):
    """Batched: kpts [bs, n, 2], K / T [bs, 4, 4], depth [bs, H, W].  Returns a dict with
    indices [bs, 2, n+1] int64, weights [bs, 2, n+1] float32 (the outputs), and the intermediates:
    proj [bs, 2, n, 2], zproj [bs, 2, n], depth [bs, 2, n], amin [bs, 2, n], emin [bs, 2, n], margin [bs, 2, n],
    proj_noise [bs, 2, n], and `stable` [bs, 2, n]: the decision about that keypoint (matched to which index, dropped
    or not) is the same for every evaluation whose errors, projected depths and depth ratios are within their float32
    noise (tau px of absolute slack on top of the projection noise)."""
    kp = [np.asarray(kpts0, np.float64), np.asarray(kpts1, np.float64)]
    Ks = [np.asarray(K0, np.float64), np.asarray(K1, np.float64)]
    T = np.asarray(T0to1, np.float64)
    D = [np.asarray(depth0, np.float64), np.asarray(depth1, np.float64)]
    bs, n, _ = kp[0].shape
    H, W = D[0].shape[1:]
    thr_m, thr_u = float(F32(max_matched)), float(F32(min_unmatched))
    out = {k: [] for k in ('indices', 'weights', 'proj', 'zproj', 'depth', 'amin', 'emin', 'margin', 'proj_noise',
                           'stable')}
    for b in range(bs):
        Tb = [T[b], np.linalg.inv(T[b])]
        pix_t, pix_c, d, proj, z, noise = [], [], [], [], [], []
        for s in range(2):
            t, c = _pixels(kp[s][b], H, W)
            ds = D[s][b][c[:, 1], c[:, 0]]
            M = Ks[1 - s][b] @ Tb[s] @ np.linalg.inv(Ks[s][b])
            p, zz, nz = _project(c, ds, M)
            pix_t.append(t); pix_c.append(c); d.append(ds); proj.append(p); z.append(zz); noise.append(nz)
        # err[i, j]: keypoint i of view 0 against keypoint j of view 1
        k0, k1 = pix_t[0].astype(np.float64), pix_t[1].astype(np.float64)
        with np.errstate(invalid='ignore'):
            e10 = np.sqrt(((proj[1][None, :, :] - k0[:, None, :]) ** 2).sum(2))
            e01 = np.sqrt(((proj[0][:, None, :] - k1[None, :, :]) ** 2).sum(2))
        err = (e10 + e01) / 2
        rmin, rerr = _argmin_first(err)
        cmin, cerr = _argmin_first(err.T)
        # pixel groups: keypoints with the same truncated pixel are indistinguishable to the error
        g = [np.unique(pix_t[s], axis=0, return_inverse=True)[1].reshape(-1) for s in range(2)]
        rmar, rrun = _margin(err, rmin, g[1])
        cmar, crun = _margin(err.T, cmin, g[0])
        # float32 noise of one error: both projections involved plus tau; the margin also carries the runner-up's
        rtau = tau + 2 * (noise[0] + noise[1][rmin])
        ctau = tau + 2 * (noise[1] + noise[0][cmin])
        rtau_m = rtau + 2 * noise[1][rrun]
        ctau_m = ctau + 2 * noise[0][crun]
        ar = np.arange(n)
        valid0, valid1 = d[0] > float(F32(1e-6)), d[1] > float(F32(1e-6))
        md1 = d[1][rmin]
        with np.errstate(divide='ignore', invalid='ignore'):
            rel01 = np.abs(z[0] - md1) / md1
            rel10 = np.abs(z[1][rmin] - d[0]) / d[0]
        both = cmin[rmin] == ar
        small = rerr <= thr_m
        match = both & small & valid0 & valid1[rmin] & (rel01 < 0.1) & (rel10 < 0.1)
        drop0 = ~match & (~valid0 | ~valid1[rmin] | (rerr <= thr_u))
        idx0 = np.full(n + 1, -1, np.int64)
        idx1 = np.full(n + 1, -1, np.int64)
        idx0[:n][match] = rmin[match]
        idx1[rmin[match]] = ar[match]
        unmatched1 = idx1[:n] == -1
        drop1 = unmatched1 & (~valid0[cmin] | ~valid1 | (cerr <= thr_u))
        n_match, n_drop = int(match.sum()), int(drop0.sum() + drop1.sum())
        mw, uw = _weights(n, n_match, n_drop)
        w = np.zeros((2, n + 1), np.float32)
        for s, (idx, drop) in enumerate(((idx0, drop0), (idx1, drop1))):
            w[s] = np.where(idx == -1, uw, mw)
            w[s, :n][drop] = 0
        # stability: every comparison the decision reads is away from its threshold by more than its noise
        rel_tau = 1e-5 + 4 * (noise[0] + noise[1][rmin]) / np.maximum(np.abs(md1), 1e-30)
        rel_ok = (~(valid0 & valid1[rmin])) | ((np.abs(rel01 - 0.1) > rel_tau) & (np.abs(rel10 - 0.1) > rel_tau))
        row_ok = (rmar > rtau_m) & (np.abs(rerr - thr_m) > rtau) & (np.abs(rerr - thr_u) > rtau)
        col_ok = (cmar > ctau_m)
        stable0 = row_ok & col_ok[rmin] & rel_ok & np.isfinite(rerr)
        stable1 = col_ok & stable0[cmin] & (np.abs(cerr - thr_u) > ctau) & np.isfinite(cerr)
        out['indices'].append(np.stack([idx0, idx1]))
        out['weights'].append(w)
        out['proj'].append(np.stack(proj))
        out['zproj'].append(np.stack(z))
        out['depth'].append(np.stack(d))
        out['amin'].append(np.stack([rmin, cmin]))
        out['emin'].append(np.stack([rerr, cerr]))
        out['margin'].append(np.stack([rmar, cmar]))
        out['proj_noise'].append(np.stack(noise))
        out['stable'].append(np.stack([stable0, stable1]))
    return {k: np.stack(v) for k, v in out.items()}
