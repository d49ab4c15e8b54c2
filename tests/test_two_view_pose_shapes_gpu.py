"""GPU: the fp64 pose kernels every evaluation pair runs -- the weighted eight-point (mvm_w8pt), the two-view BA
(mvm_ba2view) and the BA initialiser (mvm_ba_initialize) -- each through its C ABI on its own, against float64
oracles fed the same fp32 inputs the kernel reads, at the match counts, masks, solver branches and edge sets where
the kernels take their own paths.

  a. mvm_w8pt vs oracle.pose.estimate_relative_pose_w8pt: n from 8 to 2048 (around the 256-thread CTA), a different
     n_valid per item (0, 7, 8, n) with garbage and NaN past it, choose_closest x determine_inliers, confidences
     scaled by 1e-9 / 1 / 1e6 with zero and negative weights.  The oracle is given the kernel's fp32 normalised
     coordinates and fp32 normalised weights (both checked on their own), so what is compared is the solve.
  b. mvm_ba2view vs oracle.pose.run_bundle_adjust_2_view_schur: n from 7 to 2048, n_valid and mask together,
     items of exactly 6 (excluded) and 7 valid matches, 0 / 1 / 10 / 25 iterations; the residual trace of every
     evaluation (which pins each accept / reject and lambda update), valid_batch and the best pose.  Three items per
     shape go to the oracle: all n rows with a mask, a ragged n_valid with a mask, zero weights and garbage rows past
     n_valid, and the 7-match item.  Branch case (i), the step without Jacobi scaling, has its own test.
  c. mvm_ba_initialize vs oracle.ba_init.ba_initialize_edges: 2, 3, 5 and 8 views, random edge subsets with 19 / 20
     / 21 inliers counted over n_pad = 64 / 100 / 1024, failed pairs, an edge kept only because it is on the tree,
     disconnected graphs (the tree extrinsics come back bit for bit), an outlier edge, relative rotations past
     120 deg (the tr < 0 branch of R_to_aa) and near-collinear centres; n_edges_out exactly.
  d. batch invariance: every item of a 140- and a 300-item launch bit for bit what a batch-of-one launch gives, and
     repeated launches bit for bit equal.
  e. host refusals of pair tables with ids outside [0, n_views), in the four entries that take pair_a / pair_b
     and in mvm_gather_matches.

Bounds come from each case's own conditioning and every case prints its largest error as a share of its bound:
  T021 (a)   4 x max(|oracle in float32 - oracle in float64| on the same inputs, 2^-23): the gap measures how far
             input rounding moves this item's pose; 2^-23 covers the rounding of the kernel's fp32 output.
  trace (b)  relative to the trace's first entry: 2^-21 x max(trace) / trace[0] (the fp32 trace output) + 100 x
             the change of the oracle's trace when its inputs move by 1e-12 relative (the problem's sensitivity to
             float64 rounding, with room for the different summation order) + 4 x the change of the oracle's trace
             when its initial points come from the smallest eigenvector of A^T A, as the kernel's triangulate_dlt
             computes them, instead of the SVD of A.  That solver's rounding error grows with cond(A)^2: on
             near-parallel rays (a point 590 m away on a 0.2..1 m baseline) it moves the point by 1e-5 relative, and
             a later overshooting step carries that into the trace at 1e-6 of its first entry.  The pose: 2^-22 +
             the same two changes of the oracle's pose.
  extr (c)   1e-9 + 100 x the change of the oracle's extrinsics when T_rel moves by 1e-12 relative.

Branch cases of the two-view BA.  (i) precond = 0 is built from finite inputs: a match at the principal point of
both images under pure forward motion triangulates onto both optical axes, where its point's z diagonal App[5] is
exactly 0 (test_ba2view_branch_i_no_jacobi_scaling).  The DLT point of such a match is not unique; the kernel's
eigen-solver takes (0, 0, 1), the reference's SVD the camera centre, whose zero depth makes the reference's BA NaN;
the oracle states the kernel's choice (oracle.pose.triangulate_points_first_view_identity).  (ii) and (iii) cannot be
built from finite inputs and are left out: a singular damped point block needs det(App + lambda D) = 0 with App
positive semi-definite and D = max(diag, 1e-12) or I, so the determinant stays above (lambda min D)^3 > 0; a failed
6x6 solve needs an exactly zero pivot column of a positive-definite Schur complement.

Measured on an H100 80GB HBM3 (700 W power limit): the file runs in about 25 s (the oracles included).  Largest
error as a share of its bound: T021 0.074 (every case is at the fp32 rounding of the output, 1.2e-8 to 3.5e-8),
two-view BA trace 0.34 (the ragged item at n = 1024) and pose 0.27, branch case (i) 0.12, BA initialiser 0.001
(6e-13 against a 1e-9 floor).  One trajectory is determined only in part: the ragged item at n = 1024 overshoots to
30 x its first residual at evaluation 11 of 25, where the float64 variants part by 1e-3; its first 11 evaluations
and its best pose are compared.  No kernel was found wrong; the host-side view-id checks were (section e).
"""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

F32_EPS = 2.0 ** -23


def _L():
    from e2e_multi_view_matching_b200 import _lib
    return _lib


def _dev(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype=dt).cuda().contiguous()


def _bits(x):
    a = x.cpu().numpy() if torch.is_tensor(x) else np.asarray(x)
    return np.ascontiguousarray(a).view(np.uint8)


def _cint(v):
    return (C.c_int * len(v))(*[int(x) for x in v])


def _pairs(T):
    return [(a, b) for b in range(T) for a in range(b)]      # the engine's pair order


def _report(what, err, bound):
    print('%-48s err %.3e  bound %.3e  share %.3f' % (what, err, bound, err / bound))
    assert err <= bound, (what, err, bound)


# ---------------------------------------------------------------------------------------------------------------
# a. mvm_w8pt
# ---------------------------------------------------------------------------------------------------------------
def _w8pt(k0, k1, i0, i1, conf, nv, cc, di, T_gt):
    L = _L()
    lib = L.lib()
    B, N = conf.shape
    d = [_dev(x, torch.float32) for x in (k0, k1, i0, i1, conf)]
    d_gt = _dev(T_gt, torch.float32)
    d_nv = None if nv is None else _dev(nv, torch.int32)
    f32 = lambda *s: torch.full(s, -7.0, device='cuda')
    u8 = lambda *s: torch.full(s, 7, dtype=torch.uint8, device='cuda')
    o = {'T': f32(B, 4, 4), 'k0n': f32(B, N, 2), 'k1n': f32(B, N, 2), 'cn': f32(B, N), 'pos': u8(B, N),
         'inl': u8(B, N), 'F': f32(B, 3, 3), 'succ': u8(B)}
    rc = lib.mvm_w8pt(*[L.ptr(x) for x in d], B, N, L.ptr(d_gt) if cc else None, cc, di, L.ptr(o['T']),
                      L.ptr(o['k0n']), L.ptr(o['k1n']), L.ptr(o['cn']), L.ptr(o['pos']),
                      L.ptr(o['inl']) if di else None, L.ptr(o['F']), L.ptr(d_nv), L.ptr(o['succ']), L.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


def _w8pt_item(seed, n, motion):
    """A two-view scene of n matches whose float64 cheirality vote has a clear winner (seeds are tried in turn)."""
    from oracle import pose as P
    kw = {'random': {}, 'forward': {'motion': 'forward', 'rot_deg': (0, 0)},
          'orbit': {'motion': 'orbit', 'rot_deg': (130, 179)}}[motion]
    for s in range(seed, seed + 50):
        sc = P.make_two_view_scene(s, n, outlier_frac=0.3 if n >= 40 else 0.0, **kw)
        f = {k: v.astype(np.float64) for k, v in sc.items() if k != 'outlier'}
        _, info = P.estimate_relative_pose_w8pt(f['kpts0'], f['kpts1'], f['intr'], f['intr'], f['conf'])
        v = np.sort(info['vote_counts'][0])
        if v[-1] != v[-2]:
            return sc
    raise AssertionError('no scene without a tied cheirality vote')


def _w8pt_oracle(k0n, k1n, cn, T_gt, cc, intr_sum, T_kernel):
    """The float64 (and float32) oracle on the kernel's normalised inputs (identity intrinsics); the depth mask
    and inliers are evaluated with the kernel's own fp32 pose, as the kernel does, together with the distance of
    each decision from its threshold."""
    from oracle import pose as P
    out = {}
    for dt in (np.float64, np.float32):
        I = np.eye(3, dtype=dt)[None]
        Tr, info = P.estimate_relative_pose_w8pt(k0n[None].astype(dt), k1n[None].astype(dt), I, I,
                                                 cn[None, :, None].astype(dt), choose_closest=bool(cc),
                                                 T_021=T_gt[None].astype(dt))
        out[dt] = (Tr[0], info)
    T64, info = out[np.float64]
    if not cc:
        v = np.sort(info['vote_counts'][0])
        assert v[-1] != v[-2], ('tied cheirality vote', info['vote_counts'])
    x0, x1 = k0n.astype(np.float64)[None], k1n.astype(np.float64)[None]
    Tk = T_kernel.astype(np.float64)
    X = P.triangulate_points(np.eye(4)[:3][None], Tk[None, :3], x0, x1)[0]
    d0, d1 = X[:, 2], X @ Tk[2, :3] + Tk[2, 3]
    pos = (d0 > 0) & (d1 > 0)
    scale = np.linalg.norm(X, axis=1) + 1.0
    pos_margin = np.minimum(np.abs(d0), np.abs(d1)) / scale
    epi = np.sqrt(P.symmetrical_epipolar_distance(x0, x1, info['F'])[0])
    thresh = 3.0 / (intr_sum / 4.0)
    inl = pos & (epi <= thresh)
    inl_margin = np.minimum(np.abs(epi - thresh) / thresh, np.where(pos_margin > 0, pos_margin, np.inf))
    gap = float(np.abs(out[np.float32][0] - T64).max())
    return T64, gap, pos, pos_margin, inl, inl_margin


W8PT_N = [8, 9, 255, 256, 257, 513, 1024, 2048]


@pytest.mark.parametrize('n', W8PT_N)
def test_w8pt_vs_float64(n):
    from oracle import pose as P
    rng = np.random.default_rng(n)
    motion = {8: 'random', 9: 'forward', 255: 'orbit', 256: 'random', 257: 'forward', 513: 'orbit',
              1024: 'random', 2048: 'orbit'}[n]
    nvs = [n, max(8, n // 2 + 1), 7, 0, 8]
    B = len(nvs)
    k0 = rng.uniform(-100, 700, (B, n, 2)).astype(np.float32)          # finite garbage past n_valid ...
    k1 = rng.uniform(-100, 700, (B, n, 2)).astype(np.float32)
    conf = rng.uniform(-1, 2, (B, n)).astype(np.float32)
    k0[:, n - 1], conf[:, n - 1] = np.nan, np.nan                      # ... and NaN in the last row
    i0 = np.tile(np.array([577.87, 580.5, 319.5, 239.5], np.float32), (B, 1))
    i1 = np.tile(np.array([560.25, 561.0, 330.0, 250.0], np.float32), (B, 1))
    T_gt = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    for b, m in enumerate(nvs):
        if m == 0:
            continue
        if m < 8:
            sc = P.make_two_view_scene(100 * n + 10 * b, m)
        else:
            sc = _w8pt_item(100 * n + 10 * b, m, motion if b < 2 else 'random')
        K = sc['intr'][0]
        i0[b] = i1[b] = [K[0, 0], K[1, 1], K[0, 2], K[1, 2]]
        k0[b, :m], k1[b, :m], conf[b, :m], T_gt[b] = sc['kpts0'][0], sc['kpts1'][0], sc['conf'][0, :, 0], sc['T_021'][0]
    # weights: item 1 has two zero and one negative weight (far more than 8 non-zero ones remain)
    if nvs[1] >= 12:
        conf[1, [1, 4]] = 0.0
        conf[1, 6] = -0.25
    nv = np.array(nvs, np.int32)
    combos = [(0, 0), (0, 1), (1, 0), (1, 1)]
    scales = (1e-9, 1.0, 1e6)
    for ci, (cc, di) in enumerate(combos):
        c = conf.copy()
        for b in range(B):
            c[b, :nvs[b]] *= np.float32(scales[(ci + b) % 3])
        o = _w8pt(k0, k1, i0, i1, c, nv, cc, di, T_gt)
        for b, m in enumerate(nvs):
            tag = 'n=%d item %d n_valid=%d cc=%d di=%d' % (n, b, m, cc, di)
            k0n_ref = (k0[b, :m] - i0[b, 2:]) / i0[b, :2]
            k1n_ref = (k1[b, :m] - i1[b, 2:]) / i1[b, :2]
            assert np.array_equal(_bits(o['k0n'][b, :m]), _bits(k0n_ref)), tag
            assert np.array_equal(_bits(o['k1n'][b, :m]), _bits(k1n_ref)), tag
            for k in ('k0n', 'k1n', 'cn', 'pos', 'inl'):               # padding rows: exactly zero
                if k == 'inl' and not di:
                    continue
                assert not o[k][b, m:].any(), (tag, k)
            assert o['succ'][b] == (m >= 8), tag
            if m < 8:
                np.testing.assert_array_equal(o['T'][b], np.eye(4))
                continue
            # conf_norm = conf / (sum + 1e-6) in fp32 (the sum is accumulated in double, then rounded)
            cd = c[b, :m].astype(np.float64)
            cn_ref = cd / (np.float64(np.float32(cd.sum())) + np.float64(np.float32(1e-6)))
            cerr = np.abs(o['cn'][b, :m] - cn_ref) / np.abs(cn_ref).max()
            assert cerr.max() <= 4 * F32_EPS, (tag, cerr.max())
            if b not in (0, 1):
                continue                                               # at most two items per shape to the oracle
            T64, gap, pos, pm, inl, im = _w8pt_oracle(o['k0n'][b, :m], o['k1n'][b, :m], o['cn'][b, :m], T_gt[b],
                                                      cc, float(np.float64(i0[b, 0]) + i0[b, 1] + i1[b, 0] + i1[b, 1]),
                                                      o['T'][b])
            _report('w8pt T021 ' + tag, float(np.abs(o['T'][b] - T64).max()), 4 * max(gap, F32_EPS))
            away = pm > 1e-9
            assert (o['pos'][b, :m].astype(bool) == pos)[away].all(), (tag, 'pos_depth_mask')
            assert away.mean() > 0.99, tag
            if di:
                away = im > 1e-9
                assert (o['inl'][b, :m].astype(bool) == inl)[away].all(), (tag, 'inliers')
                assert away.mean() > 0.99, tag


# ---------------------------------------------------------------------------------------------------------------
# b. mvm_ba2view
# ---------------------------------------------------------------------------------------------------------------
def _fast_pair(rng, n, noise=2e-3):
    """n matches in normalised coordinates of a random two-view scene (depth 1..5 m, <= 20 deg, 0.2..1 m
    baseline), float32, and an initial pose 1 deg / 2 cm off the true one."""
    from oracle.pose import rodrigues
    ax = rng.standard_normal(3)
    R = rodrigues(ax / np.linalg.norm(ax) * np.deg2rad(rng.uniform(3, 20)))
    d = rng.standard_normal(3)
    t = d / np.linalg.norm(d) * rng.uniform(0.2, 1.0)
    z = rng.uniform(1, 5, n)
    X = np.stack([rng.uniform(-0.5, 0.5, n) * z, rng.uniform(-0.4, 0.4, n) * z, z], 1)
    q = X @ R.T + t
    q[:, 2] = np.maximum(q[:, 2], 0.3)
    x0 = X[:, :2] / X[:, 2:] + noise * rng.standard_normal((n, 2))
    x1 = q[:, :2] / q[:, 2:] + noise * rng.standard_normal((n, 2))
    ax = rng.standard_normal(3)
    T0 = np.eye(4)
    T0[:3, :3] = rodrigues(ax / np.linalg.norm(ax) * np.deg2rad(1.0)) @ R
    T0[:3, 3] = t + 0.02 * rng.standard_normal(3)
    return x0.astype(np.float32), x1.astype(np.float32), T0.astype(np.float32)


def _ba2(k0, k1, conf, T0, nv, mask, n_iter):
    L = _L()
    lib = L.lib()
    B, N = conf.shape
    d = [_dev(x, torch.float32) for x in (k0, k1, conf, T0)]
    d_nv = None if nv is None else _dev(nv, torch.int32)
    d_mk = None if mask is None else _dev(mask, torch.uint8)
    T = torch.full((B, 4, 4), -7.0, device='cuda')
    vb = torch.full((B,), 7, dtype=torch.uint8, device='cuda')
    ws = torch.empty(B, N, 3, dtype=torch.float64, device='cuda')
    tr = torch.full((B, n_iter + 1), -7.0, device='cuda')
    rc = lib.mvm_ba2view(L.ptr(d[0]), L.ptr(d[1]), L.ptr(d[2]), L.ptr(d[3]), B, N, n_iter, L.ptr(T), L.ptr(vb),
                         L.ptr(ws), L.ptr(tr), L.ptr(d_nv), L.ptr(d_mk), L.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    return T.cpu().numpy(), vb.cpu().numpy(), tr.cpu().numpy()


def _ba2_inputs(n, seed):
    """Four items: 0 all n rows (a 10 % mask), 1 ragged n_valid with a mask and a few zero weights, 2 exactly 6 valid
    matches (excluded), 3 exactly 7 valid (kept).  Rows past n_valid hold garbage."""
    rng = np.random.default_rng(seed)
    B = 4
    k0 = rng.uniform(-1, 1, (B, n, 2)).astype(np.float32)
    k1 = rng.uniform(-1, 1, (B, n, 2)).astype(np.float32)
    conf = rng.uniform(0.5, 3.0, (B, n)).astype(np.float32)
    T0 = np.zeros((B, 4, 4), np.float32)
    nv = np.array([n, max(7, (2 * n) // 3), n, n], np.int32)
    mask = (rng.uniform(size=(B, n)) > 0.1).astype(np.uint8)
    for b in range(B):
        x0, x1, T = _fast_pair(rng, n)
        k0[b], k1[b], T0[b] = x0, x1, T
        conf[b] /= np.float32(n)
    conf[1, : nv[1]: 17] = 0.0
    k0[1, nv[1]:], k1[1, nv[1]:] = 50.0, -50.0
    for b, want in ((2, 6), (3, 7)):
        valid = np.nonzero(conf[b] > 0)[0]
        mask[b] = 0
        mask[b, valid[:want]] = 1
    if n <= 8:
        mask[0] = 1
    return k0, k1, conf, T0, nv, mask


def _eff_conf(conf, nv, mask):
    c = conf.astype(np.float64) * (mask > 0)
    c[np.arange(conf.shape[1])[None] >= nv[:, None]] = 0.0
    return c


def _check_ba2_item(tag, T, tr, Tr, trr, x0, x1, ce, T0, it, rng):
    """One item: the kernel's pose T [4,4] and trace tr against the oracle's Tr / trr, under bounds from the oracle's
    change when its inputs x0, x1 [1,n,2] (float64) move by 1e-12 relative, and when its initial points come from
    the eigenvector of A^T A (the kernel's DLT formulation) instead of the SVD of A."""
    from oracle import pose as P
    pert = lambda a: a * (1 + 1e-12 * rng.uniform(-1, 1, a.shape))
    Tp, _, trp = P.run_bundle_adjust_2_view_schur(pert(x0), pert(x1), ce, T0, it)
    Tn, _, trn = P.run_bundle_adjust_2_view_schur(x0, x1, ce, T0, it, dlt='normal')
    # the trajectory is determined by the inputs only as long as these float64 variants follow it: past the first
    # evaluation where one of them leaves it by 1e-3 of trace[0], a rounding-level difference has grown into a
    # different LM path (an overshooting step on an ill-conditioned item), and nothing later can be compared
    dev = np.maximum(np.abs(trp[0] - trr), np.abs(trn[0] - trr)) / trr[0]
    k = int(np.argmax(dev > 1e-3)) if (dev > 1e-3).any() else it + 1
    dtr = 100 * float(np.abs(trp[0] - trr)[:k].max() / trr[0]) + 4 * float(np.abs(trn[0] - trr)[:k].max() / trr[0])
    _report(tag + ' trace[:%d]' % k, float(np.abs(tr - trr)[:k].max() / trr[0]),
            4 * F32_EPS * float(trr[:k].max() / trr[0]) + dtr)
    assert np.isfinite(tr).all() and (T[3] == [0, 0, 0, 1]).all()
    # the best pose: the same bound terms, over the whole run (they grow where the variants' paths part)
    dT = 100 * float(np.abs(Tp[0] - Tr).max()) + 4 * float(np.abs(Tn[0] - Tr).max())
    _report(tag + ' pose', float(np.abs(T - Tr).max()), 2 * F32_EPS + dT)
    return k == it + 1


@pytest.mark.parametrize('n', [7, 8, 255, 256, 257, 1024, 2048])
def test_ba2view_trace_vs_float64_schur(n):
    from oracle import pose as P
    k0, k1, conf, T0, nv, mask = _ba2_inputs(n, 7 + n)
    ce = _eff_conf(conf, nv, mask)
    n_valid_matches = (ce > 0).sum(1)
    assert n_valid_matches[2] == 6 and n_valid_matches[3] == 7
    x0, x1, T0d = k0.astype(np.float64), k1.astype(np.float64), T0.astype(np.float64)
    rng = np.random.default_rng(n)
    for it in (0, 1, 10, 25):
        T, vb, tr = _ba2(k0, k1, conf, T0, nv, mask, it)
        Tr, vr, trr = P.run_bundle_adjust_2_view_schur(x0, x1, ce, T0d, it)
        assert vb.tolist() == vr.astype(np.uint8).tolist(), (n, it, vb, vr)
        assert vb[2] == 0
        assert np.array_equal(_bits(T[2]), _bits(T0[2])), 'excluded item: T_init'
        for b in (0, 1, 3):
            if not vr[b]:
                continue
            s = slice(b, b + 1)
            full = _check_ba2_item('ba2 n=%d item %d it=%d' % (n, b, it), T[b], tr[b], Tr[b], trr[b], x0[s], x1[s], ce[s],
                            T0d[s], it, rng)
            assert full or it > 10, ('trajectory not determined within 10 iterations', n, b, it)


@pytest.mark.parametrize('n', [8, 300])
def test_ba2view_branch_i_no_jacobi_scaling(n):
    """Branch case (i): the fallback without Jacobi scaling (precond = 0), built from finite inputs.  Pure forward
    motion, T_init = [I | (0, 0, -b)], and one match at the principal point of both images.  Its DLT matrix has zero
    z and w columns, the point is taken as (0, 0, 1) (see oracle.pose.triangulate_points_first_view_identity), and it
    lies on both optical axes: its z row of J is zero, so App[5] = 0 and the first step is the undamped-Jacobi one,
    (A + lambda I) delta = b.  Later steps move the point off the axes and scale again.  Item 0 has the match in row
    0, item 1 in row n - 1 (past the 256-thread chunk at n = 300)."""
    from oracle import pose as P
    B = 2
    k0 = np.zeros((B, n, 2), np.float32)
    k1 = np.zeros_like(k0)
    conf = np.zeros((B, n), np.float32)
    T0 = np.zeros((B, 4, 4), np.float32)
    for b in range(B):
        sc = P.make_two_view_scene(40 + b, n, outlier_frac=0.0, motion='forward', rot_deg=(0, 0))
        K = sc['intr'][0]
        k0[b] = (sc['kpts0'][0] - K[:2, 2]) / K[[0, 1], [0, 1]]
        k1[b] = (sc['kpts1'][0] - K[:2, 2]) / K[[0, 1], [0, 1]]
        conf[b] = sc['conf'][0, :, 0] / np.float32(n)
        T0[b] = sc['T_021'][0]
        assert (T0[b, :3, :3] == np.eye(3)).all() and (T0[b, :2, 3] == 0).all()
    row = [0, n - 1]
    for b in range(B):
        k0[b, row[b]] = 0.0
        k1[b, row[b]] = 0.0
    x0, x1, ce, T0d = k0.astype(np.float64), k1.astype(np.float64), conf.astype(np.float64), T0.astype(np.float64)
    for b in range(B):                                   # the branch is taken: a zero point diagonal at the start
        pts = P.triangulate_points_first_view_identity(T0d[b], x0[b], x1[b])
        np.testing.assert_array_equal(pts[row[b]], [0.0, 0.0, 1.0])
        App = P._ba_point_blocks(T0d[b], pts, x0[b], x1[b], ce[b] / ce[b].sum())[0]
        assert App[row[b], 2, 2] == 0.0 and (np.diagonal(App, axis1=1, axis2=2) > 0).sum() == 3 * n - 1
    rng = np.random.default_rng(n)
    for it in (1, 10, 25):
        T, vb, tr = _ba2(k0, k1, conf, T0, None, None, it)
        Tr, vr, trr = P.run_bundle_adjust_2_view_schur(x0, x1, ce, T0d, it)
        assert vb.tolist() == [1, 1] and vr.tolist() == [True, True]
        for b in range(B):
            s = slice(b, b + 1)
            assert np.isfinite(tr[b]).all()
            _check_ba2_item('ba2 (i) n=%d item %d it=%d' % (n, b, it), T[b], tr[b], Tr[b], trr[b], x0[s], x1[s],
                            ce[s], T0d[s], it, rng)


def test_ba2view_mask_and_n_valid_are_the_same_as_zero_weights():
    """n_valid and mask drop matches exactly as conf = 0 does: the three ways of excluding rows give bitwise the
    same output."""
    k0, k1, conf, T0, nv, mask = _ba2_inputs(1024, 3)
    a = _ba2(k0, k1, conf, T0, nv, mask, 10)
    c = (_eff_conf(conf, nv, mask)).astype(np.float32)
    b = _ba2(k0, k1, c, T0, None, None, 10)
    for x, y in zip(a, b):
        assert np.array_equal(_bits(x), _bits(y))


# ---------------------------------------------------------------------------------------------------------------
# c. mvm_ba_initialize
# ---------------------------------------------------------------------------------------------------------------
def _ba_init(pids, T, extr_tree, T_rel, succ, on_tree, inl, min_inliers=20):
    L = _L()
    lib = L.lib()
    B = extr_tree.shape[0]
    n_pad = inl.shape[2]
    d_e, d_T = _dev(extr_tree, torch.float64), _dev(T_rel, torch.float32)
    d_s, d_o, d_i = _dev(succ, torch.uint8), _dev(on_tree, torch.uint8), _dev(inl, torch.uint8)
    out = torch.full((B, T, 4, 4), -7.0, dtype=torch.float64, device='cuda')
    ne = torch.full((B,), -1, dtype=torch.int32, device='cuda')
    rc = lib.mvm_ba_initialize(_cint([a for a, _ in pids]), _cint([b for _, b in pids]), T, len(pids), B, n_pad,
                               L.ptr(d_e), L.ptr(d_T), L.ptr(d_s), L.ptr(d_o), L.ptr(d_i), min_inliers, L.ptr(out),
                               L.ptr(ne), L.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    return out.cpu().numpy(), ne.cpu().numpy()


def _noisy(rng, T, rot_deg, trans):
    from oracle.pose import rodrigues
    ax = rng.standard_normal(3)
    out = T.copy()
    out[:3, :3] = rodrigues(ax / np.linalg.norm(ax) * np.deg2rad(rot_deg)) @ T[:3, :3]
    out[:3, 3] = T[:3, 3] + trans * np.linalg.norm(T[:3, 3]) * rng.standard_normal(3)
    return out


def _inlier_mask(rng, n_pad, cnt):
    m = np.zeros(n_pad, np.uint8)
    m[rng.choice(n_pad, cnt, replace=False)] = 1
    return m


# per T: n_pad and the two oracle tuples' scenes (kwargs of make_pose_graph)
_BAI = {2: (64, [{}, {'rot_deg': (130, 179)}]),
        3: (100, [{'rot_deg': (130, 179)}, {'collinear': 0.02}]),
        5: (1024, [{'collinear': 0.02, 'corrupt': (1, 3)}, {}]),
        8: (100, [{'rot_deg': (130, 179), 'corrupt': (2, 6)}, {}])}


def _ba_init_batch(T, seed, B):
    """B tuples: 0 and 1 the oracle scenes of _BAI (every pair succeeded with 0 / 19 / 20 / 21 / n_pad inliers placed
    anywhere in n_pad, and a chain of tree edges (v-1, v) keeps them connected),
    2 a tuple whose only link to view T-1 is a tree edge with 19 inliers, 3 a disconnected graph (every pair touching
    view T-1 failed or below min_inliers and off the tree), 4 nothing succeeded, the rest random edge subsets."""
    from oracle import ba_init as BI
    n_pad, kinds = _BAI[T]
    rng = np.random.default_rng(seed)
    pids = _pairs(T)
    P = len(pids)
    extr_tree = np.zeros((B, T, 4, 4))
    T_rel = np.zeros((B, P, 4, 4), np.float32)
    succ = np.ones((B, P), np.uint8)
    on = np.zeros((B, P), np.uint8)
    inl = np.zeros((B, P, n_pad), np.uint8)
    chain = [pids.index((v - 1, v)) for v in range(1, T)]
    for b in range(B):
        kw = kinds[b] if b < 2 else ({'rot_deg': (10, 60)} if b % 2 else {})
        gt, rel = BI.make_pose_graph(seed * 100 + b, T, **kw)
        extr_tree[b] = [gt[0]] + [_noisy(rng, E, 2.0, 0.05) for E in gt[1:]]
        for p, pq in enumerate(pids):
            T_rel[b, p] = _noisy(rng, rel[pq], 0.3, 0.01) if pq != kw.get('corrupt') else rel[pq]
            cnt = int(rng.choice([19, 20, 21, n_pad, 0]))
            inl[b, p] = _inlier_mask(rng, n_pad, cnt)
        on[b, chain] = 1
        if 'corrupt' in kw:                                         # the outlier edge is an edge
            inl[b, pids.index(kw['corrupt'])] = _inlier_mask(rng, n_pad, 21)
        if b >= 5:
            succ[b] = rng.uniform(size=P) < 0.7
            on[b] = rng.uniform(size=P) < 0.3
    touch = [p for p, (x, y) in enumerate(pids) if y == T - 1 or x == T - 1]
    if B > 2:                                                       # kept only because it is on the tree
        for p in touch:
            inl[2, p] = _inlier_mask(rng, n_pad, 19)
            on[2, p] = 0
        on[2, touch[0]] = 1
    if B > 3:                                                       # disconnected
        for k, p in enumerate(touch):
            inl[3, p] = _inlier_mask(rng, n_pad, 19)
            on[3, p] = 0
            if k % 2:
                succ[3, p] = 0
                inl[3, p] = 1
                on[3, p] = 1
    if B > 4:
        succ[4] = 0
    return pids, extr_tree, T_rel, succ, on, inl


@pytest.mark.parametrize('T', [2, 3, 5, 8])
def test_ba_initialize_vs_float64(T):
    from oracle import ba_init as BI
    B = 9
    pids, extr_tree, T_rel, succ, on, inl = _ba_init_batch(T, 50 + T, B)
    out, ne = _ba_init(pids, T, extr_tree, T_rel, succ, on, inl)
    rng = np.random.default_rng(T)
    seen = set()
    for b in range(B):
        keep, connected = BI.ba_init_edge_set(T, pids, T_rel[b], succ[b], on[b], inl[b])
        assert ne[b] == len(keep), (T, b, ne[b], len(keep))
        if not connected:
            seen.add('disconnected')
            assert np.array_equal(_bits(out[b]), _bits(extr_tree[b])), (T, b, 'tree extrinsics unchanged')
            continue
        assert np.isfinite(out[b]).all() and (out[b, 0] == np.eye(4)).all()
        if b == 2:
            seen.add('tree-only edge')
        if b >= 2:
            continue
        ref, n_ref = BI.ba_initialize_edges(T, pids, extr_tree[b], T_rel[b], succ[b], on[b], inl[b])
        Tp = T_rel[b].astype(np.float64) * (1 + 1e-12 * rng.uniform(-1, 1, T_rel[b].shape))
        refp, _ = BI.ba_initialize_edges(T, pids, extr_tree[b], Tp, succ[b], on[b], inl[b])
        _report('ba_init T=%d item %d %s' % (T, b, _BAI[T][1][b]), float(np.abs(out[b] - ref).max()),
                1e-9 + 100 * float(np.abs(refp - ref).max()))
    assert 'disconnected' in seen or T == 2
    if T > 2:
        assert 'tree-only edge' in seen


# ---------------------------------------------------------------------------------------------------------------
# d. batch invariance and repeatability
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,n', [(140, 1024), (300, 256)])
def test_batch_invariance_w8pt_ba2view(B, n):
    rng = np.random.default_rng(B)
    k0n = np.zeros((B, n, 2), np.float32)
    k1n = np.zeros_like(k0n)
    T0 = np.zeros((B, 4, 4), np.float32)
    for b in range(B):
        k0n[b], k1n[b], T0[b] = _fast_pair(rng, n)
    intr = np.tile(np.array([577.87, 577.87, 319.5, 239.5], np.float32), (B, 1))
    k0 = (k0n * intr[:, None, :2] + intr[:, None, 2:]).astype(np.float32)
    k1 = (k1n * intr[:, None, :2] + intr[:, None, 2:]).astype(np.float32)
    conf = rng.uniform(0.0, 1.0, (B, n)).astype(np.float32)
    nv = rng.integers(0, n + 1, B).astype(np.int32)
    nv[:4] = [0, 7, 8, n]
    mask = (rng.uniform(size=(B, n)) > 0.2).astype(np.uint8)
    for cc, di in ((0, 1), (1, 0)):
        o = _w8pt(k0, k1, intr, intr, conf, nv, cc, di, T0)
        o2 = _w8pt(k0, k1, intr, intr, conf, nv, cc, di, T0)
        for k in o:
            assert np.array_equal(_bits(o[k]), _bits(o2[k])), ('w8pt repeat', k)
        for b in range(B):
            s = slice(b, b + 1)
            one = _w8pt(k0[s], k1[s], intr[s], intr[s], conf[s], nv[s], cc, di, T0[s])
            for k in o:
                if k == 'inl' and not di:
                    continue
                assert np.array_equal(_bits(one[k][0]), _bits(o[k][b])), ('w8pt', b, k)
    a = _ba2(k0n, k1n, conf, T0, nv, mask, 10)
    for x, y in zip(a, _ba2(k0n, k1n, conf, T0, nv, mask, 10)):          # pose, valid_batch and trace
        assert np.array_equal(_bits(x), _bits(y)), 'ba2 repeat'
    for b in range(B):
        s = slice(b, b + 1)
        one = _ba2(k0n[s], k1n[s], conf[s], T0[s], nv[s], mask[s], 10)
        for x, y in zip(one, a):
            assert np.array_equal(_bits(x[0]), _bits(y[b])), ('ba2', b)


def test_batch_invariance_ba_initialize():
    T, B = 5, 150
    pids, extr_tree, T_rel, succ, on, inl = _ba_init_batch(T, 7, B)
    out, ne = _ba_init(pids, T, extr_tree, T_rel, succ, on, inl)
    out2, ne2 = _ba_init(pids, T, extr_tree, T_rel, succ, on, inl)
    assert np.array_equal(_bits(out), _bits(out2)) and np.array_equal(ne, ne2)
    for b in range(B):
        s = slice(b, b + 1)
        o1, n1 = _ba_init(pids, T, extr_tree[s], T_rel[s], succ[s], on[s], inl[s])
        assert np.array_equal(_bits(o1[0]), _bits(out[b])) and n1[0] == ne[b], b


# ---------------------------------------------------------------------------------------------------------------
# e. refusals of out-of-range pair ids: host-side, nothing is launched
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('bad', [(0, 3), (-1, 1), (3, 4), (0, 1 << 20)], ids=['b_eq_T', 'a_negative', 'a_b_past_T',
                                                                         'b_large'])
def test_pair_ids_outside_the_views_are_refused(bad):
    L = _L()
    lib = L.lib()
    T, n_pad, B = 3, 64, 1
    pids = [(0, 1), bad, (1, 2)]
    pa, pb = _cint([a for a, _ in pids]), _cint([b for _, b in pids])
    P = len(pids)
    buf = torch.zeros(1 << 20, dtype=torch.float64, device='cuda')
    p = L.ptr(buf)
    sp = L.stream_ptr()
    u8 = L.ptr(torch.zeros(1 << 16, dtype=torch.uint8, device='cuda'))
    nb = lib.mvm_mvba_workspace_bytes(T, P, B, n_pad)
    ws = torch.zeros(nb, dtype=torch.uint8, device='cuda')
    torch.cuda.synchronize()
    assert lib.mvm_ba_initialize(pa, pb, T, P, B, n_pad, p, p, u8, u8, u8, 20, p, p, sp) == 1
    assert lib.mvm_spanning_tree_init(pa, pb, T, P, B, p, p, u8, p, u8, sp) == 1
    assert lib.mvm_multi_view_ba(pa, pb, T, P, B, n_pad, p, p, p, p, p, p, 50, p, p, L.ptr(ws), nb, sp) == 1
    assert lib.mvm_multi_view_ba_ex(pa, pb, T, P, B, n_pad, p, p, p, p, p, None, 0, p, None, 50, p, p, L.ptr(ws), nb,
                                    sp) == 1
    assert lib.mvm_multi_view_ba_obs(pa, pb, T, P, B, n_pad, p, p, p, None, p, p, None, 0, p, None, 50, p, p,
                                     L.ptr(ws), nb, sp) == 1
    assert lib.mvm_triangulate_pairs(pa, pb, T, P, B, n_pad, p, p, p, p, p, sp) == 1
    io = (L.PairIO * P)()                                           # view ids of the match gather, without slot counts
    for k, (a, b) in enumerate(pids):
        io[k].view_a, io[k].view_b = a, b
        io[k].matches_a, io[k].conf = buf.data_ptr(), buf.data_ptr()
    assert lib.mvm_gather_matches(p, T, n_pad, _cint([n_pad] * T), io, P, B, 0.0, p, p, p, p, sp) == 1
    torch.cuda.synchronize()
    assert not buf.any() and not ws.any()                           # nothing ran
