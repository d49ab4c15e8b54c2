"""The two ends of the matcher against float64: the keypoint encoder (csrc/kenc.cu), match extraction (csrc/match.cu)
and the confidence head (csrc/conf.cu).

With zero GNN layers the matcher computes  md = final_proj(desc + kenc(kpts, scores)) -> md_a . md_b^T / 16 -> Sinkhorn.
Every Sinkhorn kernel writes Z_ij = S_ij + u_i + v_j - norm, and the dustbin entries of S are alpha = bin_score, so for
the inner block of one tuple (counts m, n)
    S_ij = Z_ij - Z_in - Z_mj + Z_mn + alpha
for any number of iterations.  This recovers the encoder's output, through the score GEMM, from the couplings alone,
up to the float32 rounding of four Z entries; the recovered S is compared with float64 S.

Every bound is (a multiple of) the float32-vs-float64 deviation of the same oracle chain plus a few ulp, derived per
case and printed as the share of it that the kernel used.

Match extraction is compared bit for bit with the float64 extraction on the kernel's own couplings, both through
mvm_extract_matches and through the matcher's multi-pair path with per-slot counts.  The confidence head is compared
with the float64 head (oracle/matcher_torch.confidence_head) fed with the kernel's couplings and matches, so that match
flips cannot hide an error."""
import numpy as np
import pytest
import torch

from oracle.matcher_torch import _mlp, confidence_head, _log_optimal_transport

pytestmark = pytest.mark.gpu

EPS32 = float(np.finfo(np.float32).eps)


@pytest.fixture(autouse=True)
def _no_tf32():
    """The float32 oracle chain is the yardstick of every bound: keep TF32 out of its convolutions and products."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


# ---------------------------------------------------------------------------------------------------------------------
# zero-layer matcher runs
# ---------------------------------------------------------------------------------------------------------------------

def _state_dict(seed, conf_head):
    from e2e_multi_view_matching_b200.synthetic import make_state_dict
    sd = make_state_dict(0, seed=seed, final_proj_gain=3.0, conf_head=conf_head)
    if conf_head == 'random':
        # a non-zero output bias, and logits of order one: the sigmoid stays away from saturation
        sd['conf_mlp.layers.0.weight'] = sd['conf_mlp.layers.0.weight'] * np.float32(0.5)
        sd['conf_mlp.layers.0.bias'] = np.array([0.3], np.float32)
    return sd


def _inputs(seed, caps, wh, B):
    """Per view slot: keypoints [B, cap, 2] (some outside the image), scores [B, cap] (with exact 0, 1 and 10),
    descriptors [B, 256, cap] drawn around shared landmarks so that the views have real mutual matches."""
    rng = np.random.default_rng(seed)
    land = rng.standard_normal((B, max(caps) * 2, 256))
    views = []
    for cap, (w, h) in zip(caps, wh):
        kp = rng.uniform(0, 1, (B, cap, 2)) * [w, h]
        sel = rng.random((B, cap))
        s = 0.7 * max(w, h)
        kp[sel < 0.05, 0] = w / 2 + s * rng.choice([-1.3, 1.2], (sel < 0.05).sum())        # normalised |x| > 1
        kp[(sel >= 0.05) & (sel < 0.08), 1] = h / 2 - 1.1 * s
        sc = rng.uniform(0, 1, (B, cap))
        sc[(sel >= 0.1) & (sel < 0.15)] = 0.0
        sc[(sel >= 0.15) & (sel < 0.2)] = 1.0
        sc[(sel >= 0.2) & (sel < 0.23)] = 10.0
        ids = np.stack([rng.permutation(land.shape[1])[:cap] for _ in range(B)])
        de = np.take_along_axis(land, ids[..., None], 1) + 0.4 * rng.standard_normal((B, cap, 256))
        de = de / np.linalg.norm(de, axis=2, keepdims=True)
        views.append(tuple(torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()
                           for x in (kp, sc, de.transpose(0, 2, 1))))
    return views


def _run_kernel(sd, views, wh, pair_ids, slot_counts, math_mode):
    import e2e_multi_view_matching_b200 as pkg
    from e2e_multi_view_matching_b200.models.multi_view_matcher import MatcherEngine
    from e2e_multi_view_matching_b200.packing import PackedMatcher
    packed = PackedMatcher({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, [], conf_mlp=True,
                           device='cuda')
    if math_mode != 3:
        pkg.set_math_mode(math_mode)
    try:
        outs = MatcherEngine().run(packed, views, wh, pair_ids, 100, 0.0, slot_counts)
    finally:
        pkg.set_math_mode(3)
    torch.cuda.synchronize()
    return outs


def _md_chain(sd, views, wh, dtype):
    """final_proj(desc + kenc(normalised keypoints, scores)) per view slot, in `dtype` on the GPU: [B, 256, cap]."""
    t = {k: torch.from_numpy(np.asarray(v)).cuda().to(dtype) for k, v in sd.items() if np.asarray(v).dtype == np.float32}
    out = []
    for (kp, sc, de), (w, h) in zip(views, wh):
        kp = kp.to(dtype)
        size = torch.tensor([w, h], dtype=dtype, device='cuda')
        k = (kp - size / 2) / (size.max() * 0.7)
        x = torch.cat([k.transpose(1, 2), sc.to(dtype).unsqueeze(1)], 1)
        d = de.to(dtype) + _mlp(t, 'kenc.encoder', [3, 32, 64, 128, 256, 256], x)
        out.append(torch.nn.functional.conv1d(d, t['final_proj.weight'], t['final_proj.bias']))
    return out, t


def _extract64(Z, thr, ms0_kernel=None):
    """The reference's extraction (multi_view_matcher.py:288-300) on Z [B, m+1, n+1] in float64.  With the kernel's
    own ms0 the validity test `ms > thr` reads the kernel's numbers (expf rounding cannot flip it).
    Returns (matches0, matches1, mutual0, exp(max0) in float64 where mutual, matching_scores1 from ms0)."""
    Z = np.asarray(Z, np.float64)
    inner = Z[:, :-1, :-1]
    idx0, idx1 = inner.argmax(2), inner.argmax(1)
    max0 = inner.max(2)
    mutual0 = np.arange(idx0.shape[1])[None] == np.take_along_axis(idx1, idx0, 1)
    mutual1 = np.arange(idx1.shape[1])[None] == np.take_along_axis(idx0, idx1, 1)
    e0 = np.where(mutual0, np.exp(max0), 0.0)
    ms0 = e0.astype(np.float32) if ms0_kernel is None else ms0_kernel
    valid0 = mutual0 & (ms0 > np.float32(thr))
    valid1 = mutual1 & np.take_along_axis(valid0, idx1, 1)
    ms1 = np.where(mutual1, np.take_along_axis(ms0, idx1, 1), np.float32(0))
    return (np.where(valid0, idx0, -1), np.where(valid1, idx1, -1), mutual0, e0, ms1)


def _check_ms(ms, e0):
    """ms (float32, kernel expf) against float64 exp(max): expf is within 2 ulp; the float64 -> float32 rounding adds
    half an ulp."""
    lim = 3 * np.spacing(e0.astype(np.float32)).astype(np.float64)
    err = np.abs(ms.astype(np.float64) - e0)
    assert (err <= lim).all(), float((err - lim).max())


CASES = {
    # name: (views (w, h) per slot, capacities, batch, ragged device counts, math mode, conf head)
    '2v_b1_portrait_landscape': ([(480, 640), (640, 480)], [133, 70], 1, False, 3, 'random'),
    '3v_b2_odd_16x16_count1': ([(133, 201), (16, 16), (640, 480)], [64, 17, 1], 2, False, 3, 'score'),
    '5v_b3_ragged': ([(133, 201), (640, 480), (480, 640), (16, 16), (1600, 1066)], [256, 200, 130, 256, 64], 3, True,
                     3, 'random'),
    '8v_b2_ragged': ([(64 + 37 * i, 480 - 41 * i) for i in range(8)], [128] * 8, 2, True, 3, 'score'),
    '3v_b4_ragged_512': ([(640, 480), (201, 133), (480, 640)], [512, 400, 512], 4, True, 3, 'score'),
    '2v_b1_2048': ([(1600, 1066), (1066, 1600)], [2048, 1999], 1, False, 3, 'random'),
    '4v_b2_mode0': ([(640, 480), (133, 201), (16, 16), (480, 640)], [300, 257, 64, 31], 2, False, 0, 'random'),
}


@pytest.mark.parametrize('name', list(CASES))
def test_zero_layer_matcher_vs_float64(name):
    wh, caps, B, ragged, mode, head = CASES[name]
    seed = sum(map(ord, name))
    T = len(wh)
    sd = _state_dict(seed, head)
    views = _inputs(seed, caps, wh, B)
    rng = np.random.default_rng(seed + 1)
    if ragged:
        cnt = np.stack([rng.integers(1, c + 1, B) for c in caps], 1)
        cnt[0, 0], cnt[-1, -1] = caps[0], 1                   # a full slot and a one-keypoint slot
        cnt[B // 2, 1] = 1
        slot_counts = torch.from_numpy(cnt.astype(np.int32)).cuda()
    else:
        cnt = np.tile(np.asarray(caps), (B, 1))
        slot_counts = None
    pair_ids = [(a, b) for b in range(T) for a in range(b)]
    outs = _run_kernel(sd, views, wh, pair_ids, slot_counts, mode)
    md64, sd64 = _md_chain(sd, views, wh, torch.float64)
    md32, sd32 = _md_chain(sd, views, wh, torch.float32)
    alpha = float(np.float32(sd['bin_score']))
    share = {'S': 0.0, 'Z': 0.0, 'conf': 0.0}
    for (a, b) in pair_ids:
        o = outs[(a, b)]
        Zk_all = o['scores'].double()
        for bi in range(B):
            m, n = int(cnt[bi, a]), int(cnt[bi, b])
            Zk = Zk_all[bi, :m + 1, :n + 1]
            # ---- part 1: recover S by double centring, compare with float64 S ----
            Srec = Zk[:m, :n] - Zk[:m, n:n + 1] - Zk[m:m + 1, :n] + Zk[m, n] + alpha
            S64 = md64[a][bi, :, :m].T @ md64[b][bi, :, :n] / 16
            S32 = (md32[a][bi, :, :m].T @ md32[b][bi, :, :n] / 16).double()
            dev_S = float((S32 - S64).abs().max())
            zmax = float(Zk.abs().max())
            # the kernel's GEMMs are fp32-faithful split-operand products, not fp32 with the oracle's summation order
            lim_S = 32 * dev_S + 16 * EPS32 * zmax
            err_S = float((Srec - S64).abs().max())
            share['S'] = max(share['S'], err_S / lim_S)
            assert err_S <= lim_S, (a, b, bi, err_S, lim_S)
            # ---- and Z itself against the float64 chain ----
            Z64 = _log_optimal_transport(S64[None], torch.tensor(alpha, dtype=torch.float64, device='cuda'), 100)[0]
            Z32 = _log_optimal_transport(S32.float()[None], torch.tensor(alpha, device='cuda'), 100)[0].double()
            lim_Z = 16 * float((Z32 - Z64).abs().max()) + 16 * EPS32 * zmax
            err_Z = float((Zk - Z64).abs().max())
            share['Z'] = max(share['Z'], err_Z / lim_Z)
            assert err_Z <= lim_Z, (a, b, bi, err_Z, lim_Z)
            # ---- part 2: matches on the kernel's own couplings, float64 extraction ----
            ms0 = o['mscores_a'][bi].cpu().numpy()
            ms1 = o['mscores_b'][bi].cpu().numpy()
            i0k = o['matches_a'][bi].cpu().numpy()
            i1k = o['matches_b'][bi].cpu().numpy()
            e_i0, e_i1, mutual0, e0, e_ms1 = _extract64(Zk.cpu().numpy()[None], 0.0, ms0[None, :m])
            assert np.array_equal(i0k[:m], e_i0[0]) and np.array_equal(i1k[:n], e_i1[0]), (a, b, bi)
            _check_ms(ms0[:m], e0[0])
            assert np.array_equal(ms1[:n], e_ms1[0])
            assert (i0k[m:] == -1).all() and (ms0[m:] == 0).all() and (i1k[n:] == -1).all() and (ms1[n:] == 0).all()
            # ---- part 3: the confidence head on the kernel's couplings and matches ----
            conf = o['conf'][bi, :, 0].double()
            assert (conf[m:] == 0).all()                        # rows past this tuple's count
            idx = torch.from_numpy(i0k[None, :m]).cuda()
            c64 = confidence_head(sd64, md64[a][bi:bi + 1, :, :m], md64[b][bi:bi + 1, :, :n], Zk[None], idx)[0, :, 0]
            c32 = confidence_head(sd32, md32[a][bi:bi + 1, :, :m], md32[b][bi:bi + 1, :, :n], Zk.float()[None],
                                  idx)[0, :, 0].double()
            lim_c = 16 * float((c32 - c64).abs().max()) + 8 * EPS32
            err_c = float((conf[:m] - c64).abs().max())
            share['conf'] = max(share['conf'], err_c / lim_c)
            assert err_c <= lim_c, (a, b, bi, err_c, lim_c)
    unmatched = sum(int((outs[p]['matches_a'] == -1).sum()) for p in pair_ids)
    conf_all = torch.cat([outs[p]['conf'].flatten() for p in pair_ids])
    print('%s: largest share of bound S %.3f Z %.3f conf %.3f; unmatched rows %d; conf in [%.3f, %.3f]' % (
        name, share['S'], share['Z'], share['conf'], unmatched, float(conf_all[conf_all > 0].min()),
        float(conf_all.max())))


# ---------------------------------------------------------------------------------------------------------------------
# mvm_extract_matches on built couplings
# ---------------------------------------------------------------------------------------------------------------------

SIZES = [1, 7, 8, 9, 31, 32, 33, 255, 256, 257, 1024, 2047, 2048]


def _couplings(rng, B, m, n):
    """[B, m+1, n+1] float32, one style per batch item: peaked mutual matches, quantised values (ties everywhere),
    all-equal / -inf / signed-zero rows and columns, a dustbin larger than every inner entry, scores around log 0.2
    and deep underflow."""
    Z = np.empty((B, m + 1, n + 1), np.float32)
    for b in range(B):
        style = b % 5
        x = rng.standard_normal((m + 1, n + 1)) * 3 - 5
        if style == 0:
            k = min(m, n)
            x[rng.permutation(m)[:k], rng.permutation(n)[:k]] += 12
        elif style == 1:
            x = np.round(rng.standard_normal((m + 1, n + 1)))      # -2..2: exact ties in rows and columns
        elif style == 2:
            x[:m:3, :] = 0.5                                       # all-equal rows
            x[1:m:5, :] = -np.inf                                  # -inf rows
            x[:, 2:n:7] = -np.inf                                  # -inf columns
            z = rng.random((m + 1, n + 1)) < 0.5
            x[2:m:4, :] = np.where(z[2:m:4], 0.0, -0.0)            # +0.0 against -0.0
        elif style == 3:
            x[:, n] = 100.0                                        # dustbin column / row above every inner entry
            x[m, :] = 100.0
        elif m % 2:
            x = np.log(0.2) + rng.standard_normal((m + 1, n + 1)) * 1e-3
            x[::2] -= 200.0                                        # exp underflows to 0
        else:
            x = rng.standard_normal((m + 1, n + 1)) - 200.0        # every mutual pair scores exp(max) == 0
        Z[b] = x
    return Z


@pytest.mark.parametrize('m', SIZES)
def test_extract_matches_vs_float64(m):
    from e2e_multi_view_matching_b200 import ops
    rng = np.random.default_rng(m)
    for n in SIZES:
        B = 1 + (m + n) % 5
        Z = _couplings(rng, B, m, n)
        Zd = torch.from_numpy(Z).cuda()
        for thr in (0.0, 0.2):
            i0, i1, s0, s1 = [x.cpu().numpy() for x in ops.extract_matches(Zd, thr)]
            e_i0, e_i1, mutual0, e0, e_ms1 = _extract64(Z, thr, s0)
            assert np.array_equal(i0, e_i0), (m, n, thr, np.argwhere(i0 != e_i0)[:4])
            assert np.array_equal(i1, e_i1), (m, n, thr, np.argwhere(i1 != e_i1)[:4])
            _check_ms(s0, e0)
            assert np.array_equal(s1, e_ms1)
            # valid == mutual & (ms > thr) on the kernel's own ms
            assert np.array_equal(i0 >= 0, mutual0 & (s0 > np.float32(thr)))
            # a -inf row: index 0, score 0, no match
            inf_rows = np.isneginf(Z[:, :m, :n]).all(2)
            assert (s0[inf_rows] == 0).all() and (i0[inf_rows] == -1).all()
            # the dustbin is never chosen
            assert (i0 < n).all() and (i1 < m).all()


def test_extract_matches_refuses_empty_views():
    """m or n == 0 is refused before any launch."""
    from e2e_multi_view_matching_b200 import _lib
    lib = _lib.lib()
    Z = torch.zeros(1, 9, 9, device='cuda')
    m0 = torch.full((1, 8), 7, dtype=torch.int64, device='cuda')
    m1 = torch.full((1, 8), 7, dtype=torch.int64, device='cuda')
    s0 = torch.full((1, 8), 7.0, device='cuda')
    s1 = torch.full((1, 8), 7.0, device='cuda')
    ws = torch.zeros(3 * 64, dtype=torch.int32, device='cuda')
    P = _lib.ptr
    for m, n in ((0, 8), (8, 0), (0, 0)):
        rc = lib.mvm_extract_matches(P(Z), 1, m, n, 0.0, P(m0), P(m1), P(s0), P(s1), P(ws), _lib.stream_ptr())
        assert rc != 0, (m, n)
    torch.cuda.synchronize()
    assert (m0 == 7).all() and (m1 == 7).all() and (s0 == 7).all() and (s1 == 7).all()
    assert lib.mvm_extract_matches(P(Z), 1, 8, 8, 0.0, P(m0), P(m1), P(s0), P(s1), P(ws), _lib.stream_ptr()) == 0
