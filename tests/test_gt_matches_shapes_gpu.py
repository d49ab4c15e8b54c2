"""Ground-truth matches (csrc/gt_matches.cu: gt_project / gt_argmin / gt_assign) against the float64 oracle
(oracle/gt_matches.py) across keypoint counts around the 128-wide arg-min tile, batches of different scenes, exact ties,
pixels on and past the border, depth holes / negative depth / depth steps, large rotations and translations, non-square
pixels, and pairs that are all matched, none matched or all dropped.

On every decision the oracle calls stable, the kernel's index must be the oracle's; unstable decisions are counted and
printed.  When every decision agrees, the class weights must be the same float32 numbers."""
import numpy as np
import pytest
import torch

from oracle.gt_matches import gt_matches_pair

pytestmark = pytest.mark.gpu

E_MATCH, E_UNMATCH = 5.0, 15.0
H, W = 120, 160


def _K(rng, square=True):
    f = rng.uniform(80, 200)
    K = np.eye(4)
    K[0, 0], K[1, 1] = f, (f if square else f * rng.uniform(0.6, 1.6))
    K[0, 2], K[1, 2] = W / 2 + rng.uniform(-5, 5), H / 2 + rng.uniform(-5, 5)
    return K


def _rot(axis, deg):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    t = np.deg2rad(deg)
    X = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(t) * X + (1 - np.cos(t)) * X @ X


def make_scene(rng, n, kind):
    """One batch item: (kpts0, kpts1, K0, K1, T0to1, depth0, depth1), float32.
    kind: 'orbit' (rotation past 90 deg about the scene centre), 'forward' (translation 1e3 along z, where the second
    relative-depth test fails while the first passes), 'identity' (all matched), 'none' (every relative-depth test
    fails), 'dropped' (no valid depth)."""
    K0, K1 = _K(rng, square=kind != 'orbit'), _K(rng, square=kind == 'identity')
    if kind == 'identity':
        K1 = K0.copy()
    T = np.eye(4)
    D0 = 20.0
    if kind == 'orbit':
        R = _rot(rng.standard_normal(3) * [0.2, 1, 0.2], rng.uniform(95, 150))
        c = np.array([0, 0, D0])
        T[:3, :3], T[:3, 3] = R, c - R @ c
    elif kind == 'forward':
        # view 1 sits 1e3 behind view 0 with a focal length that keeps the image scale
        D0 = 100.0
        T[:3, :3], T[:3, 3] = _rot([0, 0, 1], rng.uniform(-30, 30)), [rng.uniform(-5, 5), rng.uniform(-5, 5), 1e3]
        K1[0, 0] *= (D0 + 1e3) / D0
        K1[1, 1] *= (D0 + 1e3) / D0
    elif kind in ('none', 'dropped'):
        T[:3, :3], T[:3, 3] = _rot([1, 1, 0], 10), [1, 0, 0.5]
    # depth0: a slanted plane plus texture, with holes (0) and negative patches
    yy, xx = np.mgrid[0:H, 0:W]
    d0 = D0 * (1 + 0.002 * (xx - W / 2) + 0.001 * (yy - H / 2)) + 0.3 * np.sin(xx * 0.7) * np.cos(yy * 0.5)
    if kind != 'identity':
        d0[rng.random((H, W)) < 0.04] = 0.0
        d0[rng.random((H, W)) < 0.02] *= -1
    if kind == 'dropped':
        d0[:] = 0.0
    # keypoints of view 0: distinct pixels for 'identity', otherwise any pixel plus border cases
    if kind == 'identity':
        pix = rng.choice(H * W, n, replace=False)
        k0 = np.stack([pix % W, pix // W], 1).astype(np.float64) + rng.uniform(0, 0.99, (n, 2))
    else:
        k0 = rng.uniform(0, [W, H], (n, 2))
        sel = rng.random(n)
        k0[sel < 0.03, 0] = W - 1 + rng.uniform(0, 0.999, (sel < 0.03).sum())      # on the last column
        k0[(sel >= 0.03) & (sel < 0.05), 0] = rng.uniform(-0.99, 0, ((sel >= 0.03) & (sel < 0.05)).sum())  # -> 0
        k0[(sel >= 0.05) & (sel < 0.06), 1] = H + rng.uniform(0, 8, ((sel >= 0.05) & (sel < 0.06)).sum())  # past
        k0[(sel >= 0.06) & (sel < 0.07), 1] = rng.uniform(-0.99, 0, ((sel >= 0.06) & (sel < 0.07)).sum())
    k0 = k0.astype(np.float32).astype(np.float64)
    # project into view 1 (float64) from the clamped truncated pixel
    p = np.trunc(k0).astype(np.int64)
    px, py = np.clip(p[:, 0], 0, W - 1), np.clip(p[:, 1], 0, H - 1)
    d = d0[py, px]
    M = K1 @ T @ np.linalg.inv(K0)
    X = np.stack([px * d, py * d, d, np.ones(n)], 1) @ M.T
    with np.errstate(divide='ignore', invalid='ignore'):
        q = X[:, :2] / X[:, 2:3]
    ok = (d > 0) & (X[:, 2] > 0) & np.isfinite(q).all(1) & (q[:, 0] >= 0) & (q[:, 0] < W) & (q[:, 1] >= 0) & (q[:, 1] < H)
    k1 = rng.uniform(0, [W, H], (n, 2))
    noise = 0 if kind == 'identity' else rng.normal(0, 1.0, (n, 2))
    k1[ok] = np.clip(q[ok] + (noise[ok] if kind != 'identity' else 0), 0, [W - 1e-3, H - 1e-3])
    d1 = np.full((H, W), D0 * 1.3)
    q1 = np.trunc(k1).astype(np.int64)
    # depth1 at the partner pixels: the projected depth, with a relative step on some of them
    step = rng.choice([0.0, 0.0, 0.0, 0.03, -0.05, 0.05, 0.2], n)
    if kind == 'identity':
        step[:] = 0
    d1[q1[ok, 1], q1[ok, 0]] = X[ok, 2] * (1 + step[ok])
    if kind != 'identity':
        d1[rng.random((H, W)) < 0.03] = 0.0
        d1[rng.random((H, W)) < 0.01] = -3.0
    if kind == 'dropped':
        d1[:] = 0.0
    if kind == 'none':
        d1[:] = 1e4                                       # every relative-depth test fails: no match
    if kind == 'identity':
        k1 = k0.copy()
        d1 = d0.copy()
    perm = rng.permutation(n)
    k1 = k1[perm]
    # exact duplicates in both views (ties the first index must win)
    if n >= 8 and kind != 'identity':
        dup = rng.choice(n, max(2, n // 16), replace=False)
        k0[dup[1::2]] = k0[dup[0::2]][:len(dup[1::2])]
        k1[dup[0::2][:len(dup[1::2])]] = k1[dup[1::2]]
    f = lambda a: np.asarray(a, np.float32)
    return f(k0), f(k1), f(K0), f(K1), f(T), f(d0), f(d1)


def make_batch(seed, n, bs, kinds):
    rng = np.random.default_rng(seed)
    items = [make_scene(rng, n, kinds[b % len(kinds)]) for b in range(bs)]
    return [np.stack([it[k] for it in items]) for k in range(7)]


def check(batch, label):
    from e2e_multi_view_matching_b200.training import compute_gt_matches_of_image_pair
    t = [torch.from_numpy(x).cuda() for x in batch]
    idx, w = compute_gt_matches_of_image_pair(*t, E_MATCH, E_UNMATCH)
    idx, w = idx.cpu().numpy(), w.cpu().numpy()
    o = gt_matches_pair(*batch, E_MATCH, E_UNMATCH)
    assert np.isfinite(o['emin']).all()                   # the scenes keep every projection finite
    assert idx.dtype == np.int64 and w.dtype == np.float32 and idx.shape == o['indices'].shape
    st = o['stable']
    mism = idx[:, :, :-1] != o['indices'][:, :, :-1]
    print('%s: unstable %d of %d, index mismatches %d (on stable %d), matches %s' % (
        label, int((~st).sum()), st.size, int(mism.sum()), int((mism & st).sum()),
        [int((o['indices'][b, 0] >= 0).sum()) for b in range(idx.shape[0])]))
    assert not (mism & st).any(), np.argwhere(mism & st)[:8]
    assert (idx[:, :, -1] == -1).all()
    if not mism.any():
        assert np.array_equal(w, o['weights']), (w[w != o['weights']][:8], o['weights'][w != o['weights']][:8])
    return idx, w, o


NS = [1, 2, 127, 128, 129, 255, 256, 257, 1000, 2048]


@pytest.mark.parametrize('bs', [1, 3])
@pytest.mark.parametrize('n', NS)
def test_gt_matches_vs_oracle(n, bs):
    kinds = ['orbit', 'forward', 'identity'] if bs == 3 else [['orbit', 'forward', 'identity'][n % 3]]
    batch = make_batch(1000 * n + bs, n, bs, kinds)
    idx, w, o = check(batch, 'n=%d bs=%d %s' % (n, bs, kinds))
    for b, kind in enumerate(kinds):
        if kind == 'identity':
            assert (idx[b, :, :n] >= 0).all() and (w[b] == 0).all()                # all matched: weights 0


@pytest.mark.parametrize('n', [1, 129, 1000])
def test_gt_matches_none_matched_and_all_dropped(n):
    batch = make_batch(7 + n, n, 3, ['none', 'dropped', 'forward'])
    idx, w, o = check(batch, 'n=%d none/dropped/forward' % n)
    for b in (0, 1):
        assert (idx[b] == -1).all() and (w[b] == 0).all()   # non-finite class weights -> 0
    assert (o['weights'][1] == 0).all() and (o['indices'][1] == -1).all()


def test_gt_matches_workspace_intermediates():
    """The kernel's own projections, depths and arg-min errors, read from the workspace of mvm_gt_matches_pair.  Its
    layout is fixed there: per view v in (0, 1) proj [bs, n, 2], zproj [bs, n], d [bs, n], aerr [bs, n] (float32),
    then amin [bs, n] (int32) for views 0 and 1."""
    from e2e_multi_view_matching_b200 import _lib
    lib = _lib.lib()
    n, bs = 257, 3
    batch = make_batch(42, n, bs, ['orbit', 'forward', 'identity'])
    t = [torch.from_numpy(x).cuda().contiguous() for x in batch]
    idx = torch.empty(bs, 2, n + 1, dtype=torch.int64, device='cuda')
    w = torch.empty(bs, 2, n + 1, dtype=torch.float32, device='cuda')
    nbytes = lib.mvm_gt_matches_workspace_bytes(bs, n)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device='cuda')
    rc = lib.mvm_gt_matches_pair(*[_lib.ptr(x) for x in t], bs, n, H, W, E_MATCH, E_UNMATCH, _lib.ptr(idx), _lib.ptr(w),
                                 _lib.ptr(ws), nbytes, _lib.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    f = ws[:bs * n * 10 * 4].view(torch.float32).cpu().numpy()
    am = ws[bs * n * 10 * 4:bs * n * 12 * 4].view(torch.int32).cpu().numpy().reshape(2, bs, n)
    o = gt_matches_pair(*batch, E_MATCH, E_UNMATCH)
    bn, off = bs * n, 0
    for v in range(2):
        proj = f[off:off + 2 * bn].reshape(bs, n, 2); off += 2 * bn
        zp = f[off:off + bn].reshape(bs, n); off += bn
        dd = f[off:off + bn].reshape(bs, n); off += bn
        aerr = f[off:off + bn].reshape(bs, n); off += bn
        np.testing.assert_array_equal(dd, o['depth'][:, v])             # the depth at the truncated, clamped pixel
        err = np.abs(proj - o['proj'][:, v]).max(-1)
        lim = 2 * o['proj_noise'][:, v] + 1e-4
        print('view %d: projection error / bound max %.3f' % (v, float((err / lim).max())))
        assert (err <= lim).all()
        np.testing.assert_allclose(zp, o['zproj'][:, v], rtol=1e-5, atol=1e-5 * np.abs(o['zproj']).max())
        st = o['stable'][:, v]
        assert (am[v][st] == o['amin'][:, v][st]).all()
        np.testing.assert_allclose(aerr[st], o['emin'][:, v][st], rtol=1e-4, atol=1e-3)
    from e2e_multi_view_matching_b200.training import compute_gt_matches_of_image_pair
    idx2, w2 = compute_gt_matches_of_image_pair(*t, E_MATCH, E_UNMATCH)
    assert torch.equal(idx, idx2) and torch.equal(w, w2)


def test_gt_matches_refusals():
    """n < 1 and a workspace one byte short are refused before any launch."""
    from e2e_multi_view_matching_b200 import _lib
    lib = _lib.lib()
    x = torch.zeros(1, 8, 2, device='cuda')
    K = torch.eye(4, device='cuda')[None].contiguous()
    d = torch.ones(1, 4, 4, device='cuda')
    idx = torch.full((1, 2, 9), 7, dtype=torch.int64, device='cuda')
    w = torch.full((1, 2, 9), 7.0, device='cuda')
    nbytes = lib.mvm_gt_matches_workspace_bytes(1, 8)
    ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
    P = _lib.ptr
    args = (P(x), P(x), P(K), P(K), P(K), P(d), P(d))
    for n, nb in ((0, nbytes), (-1, nbytes), (8, nbytes - 1)):
        rc = lib.mvm_gt_matches_pair(*args, 1, n, 4, 4, 5.0, 15.0, P(idx), P(w), P(ws), nb, _lib.stream_ptr())
        assert rc != 0, (n, nb)
    torch.cuda.synchronize()
    assert (idx == 7).all() and (w == 7).all()          # nothing was launched
    assert lib.mvm_gt_matches_pair(*args, 1, 8, 4, 4, 5.0, 15.0, P(idx), P(w), P(ws), nbytes, _lib.stream_ptr()) == 0
