"""Images at their native sizes (sides that are not multiples of 8; pairs of one portrait and one landscape image, as the
MegaDepth / YFCC100M pair evaluation makes them) against fixtures of the UNMODIFIED reference
(oracle/make_native_sizes_golden.py): SuperPoint on any size, the pairwise matcher and SuperGlue normalising each view by
its own image in eval and train mode, the per-view C entry point, the image-in chain, and PairPipeline in all four
modes on mixed-size synthetic pairs."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import pose as P
from oracle import make_native_sizes_golden as G
from tests import ransac_oracle as RO
from tests.util import GOLDEN, compare_matcher_outputs, stable_rows

pytestmark = pytest.mark.gpu

REPORT = json.load(open(os.path.join(GOLDEN, 'native_report.json')))


def _load(name):
    z = np.load(os.path.join(GOLDEN, 'native_%s.npz' % name))
    return json.loads(str(z['meta'])), {k: z[k] for k in z.files if k != 'meta'}


def _cuda(data):
    return {k: (torch.from_numpy(v).cuda() if isinstance(v, np.ndarray) else v) for k, v in data.items()}


def _matcher(layers, sd, multi=False, **cfg):
    from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher
    m = MultiViewMatcher({'multi_frame_matching': multi, 'GNN_layers': layers, 'conf_mlp': True, **cfg})
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
    return m.cuda()


def _superpoint(config, wseed):
    from e2e_multi_view_matching_b200.models.superpoint import SuperPoint
    from e2e_multi_view_matching_b200.synthetic import make_superpoint_state_dict
    sp = SuperPoint(config).eval()
    sp.load_state_dict({k: torch.from_numpy(v) for k, v in make_superpoint_state_dict(wseed).items()}, strict=True)
    return sp.cuda()


@pytest.mark.parametrize('name', [c['name'] for c in G.SP_CASES])
def test_superpoint_native_size_vs_reference(name):
    """Keypoints exact (as sets under top-k), scores rtol 2e-5, descriptors within 1e-4 (test_superpoint_gpu.py)."""
    from e2e_multi_view_matching_b200.synthetic import make_image
    meta, ref = _load(name)
    sp = _superpoint({'max_keypoints': meta['max_keypoints']}, meta['wseed'])
    img = torch.from_numpy(make_image(meta['seed'], meta['height'], meta['width'])).cuda()
    scores_map, dense = sp.dense(img)
    h, w = meta['height'] // 8, meta['width'] // 8
    assert scores_map.shape == (1, 8 * h, 8 * w) and dense.shape == (1, h, w, 256)
    out = sp({'image': [img]})
    kp = out['keypoints'][0].cpu().numpy()
    kp_ref = ref['keypoints'].astype(np.int64)                        # (x, y)
    assert kp.dtype == np.float32 and kp.shape == kp_ref.shape, (kp.shape, kp_ref.shape)
    assert kp[:, 0].max() < 8 * w and kp[:, 1].max() < 8 * h
    if meta['max_keypoints'] < 0:
        assert np.array_equal(kp.astype(np.int64), kp_ref)           # nonzero order = row-major, exact
        order = order_ref = np.arange(kp.shape[0])
    else:
        key = lambda a: a[:, 1] * 100000 + a[:, 0]
        order, order_ref = np.argsort(key(kp.astype(np.int64))), np.argsort(key(kp_ref))
        assert np.array_equal(kp.astype(np.int64)[order], kp_ref[order_ref])
    sc = out['scores'][0].cpu().numpy()
    np.testing.assert_allclose(sc[order], ref['scores'][order_ref], rtol=2e-5, atol=1e-7)
    # stored descriptor columns -> the same keypoints of ours
    inv = np.empty_like(order)
    inv[order_ref] = order                                            # reference index -> our index
    d = out['descriptors'][0].cpu().numpy()[:, inv[ref['desc_columns']]]
    assert d.shape == ref['descriptors'].shape
    err = np.abs(d - ref['descriptors']).max()
    assert err < 1e-4, err
    np.testing.assert_allclose(np.linalg.norm(out['descriptors'][0].cpu().numpy(), axis=0), 1.0, atol=1e-5)


@pytest.mark.parametrize('mode', [3, 0])
@pytest.mark.parametrize('name', [c['name'] for c in G.EVAL_CASES])
def test_eval_matcher_mixed_sizes_vs_reference(name, mode):
    """Each view normalised by its own image; the margin rule of the matcher fixtures (tests/test_matcher_gpu.py)."""
    import e2e_multi_view_matching_b200 as pkg
    meta, ref = _load(name)
    sd, data = G.eval_inputs(meta)
    noise = REPORT[name]['max_abs_ref32_vs_ref64']
    pkg.set_math_mode(mode)
    try:
        with torch.no_grad():
            got = _matcher(meta['layers'], sd).eval()(_cuda(data))
        torch.cuda.synchronize()
    finally:
        pkg.set_math_mode(3)
    got = {k: v.cpu().numpy() for k, v in got.items() if v is not None}
    assert set(got) == set(ref)
    tol = dict(tau=2e-4, score_tol=(max(2e-4, 2.5 * noise), 1e-5)) if mode == 0 else \
        dict(tau=2e-3, score_tol=(max(3e-4, 4.0 * noise), 3e-5))
    print(name, mode, compare_matcher_outputs(ref, got, min_stable=0.9, **tol))


def test_eval_matcher_uses_each_views_own_size():
    """Normalising both views by image0 (what the engine did before per-view sizes) moves the couplings far beyond the
    tolerance of the fixture: the per-view sizes are what the comparison above pins."""
    meta, ref = _load(G.EVAL_CASES[0]['name'])
    sd, data = G.eval_inputs(meta)
    data['image1'] = data['image0']
    with torch.no_grad():
        got = _matcher(meta['layers'], sd).eval()(_cuda(data))
    assert np.abs(got['scores_0_1'].cpu().numpy() - ref['scores_0_1']).max() > 1e-2


def test_superglue_mixed_sizes_vs_reference():
    """SuperGlue (no confidence head, match_threshold 0.2) on the portrait / landscape pair: its matches are the
    reference's with every match whose score is not above 0.2 dropped (superglue.py:275-279)."""
    from e2e_multi_view_matching_b200.models.superglue import SuperGlue
    name = G.EVAL_CASES[0]['name']
    meta, ref = _load(name)
    sd, data = G.eval_inputs(meta)
    model = SuperGlue({'GNN_layers': meta['layers']}).eval()
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items() if not k.startswith('conf_mlp')},
                          strict=True)
    with torch.no_grad():
        out = model.cuda()(_cuda(data))
    tau = 2e-3
    st0, st1 = stable_rows(ref['scores_0_1'], tau)
    for side, st in ((0, st0), (1, st1)):
        ms_ref = ref['matching_scores%d_0_1' % side]
        m_ref = np.where(ms_ref > 0.2, ref['matches%d_0_1' % side], -1)
        keep = st & (np.abs(ms_ref - 0.2) > 1e-3)
        got = out['matches%d' % side].cpu().numpy()
        assert got.dtype == np.int64 and got.shape == m_ref.shape
        assert np.array_equal(got[keep], m_ref[keep]), int((got[keep] != m_ref[keep]).sum())
        assert keep.mean() > 0.9 and (m_ref[keep] >= 0).sum() > 10


def test_train_pair_mixed_sizes_vs_reference():
    """Train mode (batch-statistics BatchNorm, full_output) on the portrait / landscape pair, with the tolerances of
    tests/test_train_forward_gpu.py: couplings within 6x the reference's fp32-vs-fp64 noise, matches exact on rows
    whose margins exceed 10x that noise, running statistics within 4x their noise."""
    meta, z = _load(G.TRAIN_CASE['name'])
    sd, data = G.train_inputs(meta)
    model = _matcher(meta['layers'], sd, full_output=True).train()
    with torch.no_grad():
        res = model(_cuda(data))
    keys = [k[5:] for k in z if k.startswith('f64__') and '__stat__' not in k]
    assert sorted(k for k, v in res.items() if v is not None) == sorted(keys)
    fails = []
    for k in sorted(keys):
        r32, r64 = z['f32__' + k], z['f64__' + k]
        got = res[k].cpu().numpy()
        assert got.shape == r64.shape, (k, got.shape, r64.shape)
        if k.startswith('matches'):
            pair = k.split('_', 1)[1]
            first = k[len('matches'):].split('_')[0] == pair.split('_')[0]
            Z64, Z32 = z['f64__scores_' + pair], z['f32__scores_' + pair]
            st0, st1 = stable_rows(Z64, 10.0 * float(np.abs(Z32.astype(np.float64) - Z64).max()))
            stable = st0 if first else st1
            bad = int(((got != r64) & stable).sum())
            if bad > max(1, int(0.02 * stable.sum())):
                fails.append((k, bad, int(stable.sum())))
            continue
        noise = float(np.abs(r32.astype(np.float64) - r64).max())
        d = np.abs(got.astype(np.float64) - r64)
        if k.startswith('matching_scores') or k.startswith('conf_scores'):
            mk = 'matches' + k.split('scores', 1)[1].lstrip('_') if k.startswith('matching') else \
                'matches%s_%s' % (k.split('_')[2], k.split('_', 2)[2])
            same = res[mk].cpu().numpy() == z['f64__' + mk]
            d = d.reshape(same.shape)[same]
        err = float(d.max()) if d.size else 0.0
        print(k, 'max err %.3g  reference fp32-vs-fp64 %.3g' % (err, noise))
        if err > max(6.0 * noise, 2e-4):
            fails.append((k, err, noise))
    assert not fails, fails
    st = model.state_dict()
    for k in G.TRAIN_STATS:
        got, r32, r64 = st[k].cpu().numpy(), z['f32__stat__' + k], z['f64__stat__' + k]
        if k.endswith('num_batches_tracked'):
            assert int(got) == int(r64)
            continue
        noise = float(np.abs(r32.astype(np.float64) - r64).max())
        assert np.abs(got.astype(np.float64) - r64).max() <= max(4.0 * noise, 1e-5 * max(1.0, np.abs(r64).max())), k


@pytest.mark.parametrize('math_mode', [3, 0])
def test_views_entry_with_uniform_table_is_bitwise_ex(math_mode):
    """mvm_matcher_forward_views with every entry (w, h) gives exactly what mvm_matcher_forward_ex gives."""
    import ctypes as C
    from e2e_multi_view_matching_b200 import _lib, ops
    from oracle.weights import make_state_dict, make_correlated_view_inputs
    layers = ['self', 'cross'] * 2
    model = _matcher(layers, make_state_dict(len(layers), seed=3, final_proj_gain=12.0)).eval()
    data = _cuda(make_correlated_view_inputs(4, 3, 150, batch=2, width=1066, height=1600))
    lib = _lib.lib()
    dev = torch.device('cuda')
    packed = model._pack(dev)
    B, T, n_pad, counts = 2, 3, 192, [150] * 3
    kp, sc, de = ops.pack_views([model._view(data, i) for i in range(T)], n_pad)
    opt = _lib.MatcherOptions()
    lib.mvm_matcher_options_default(opt)
    opt.math_mode = math_mode
    pair_ids = [(0, 1), (0, 2), (1, 2)]
    nbytes = lib.mvm_matcher_workspace_bytes(B, T, n_pad, len(pair_ids), 1)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)

    def run(views_entry):
        pairs = (_lib.PairIO * len(pair_ids))()
        outs = []
        for p, (a, b) in enumerate(pair_ids):
            o = [torch.empty(B, 150, dtype=torch.int64, device=dev), torch.empty(B, 150, dtype=torch.int64, device=dev),
                 torch.empty(B, 150, device=dev), torch.empty(B, 150, device=dev), torch.empty(B, 151, 151, device=dev),
                 torch.empty(B, 150, 1, device=dev)]
            pairs[p].view_a, pairs[p].view_b = a, b
            (pairs[p].matches_a, pairs[p].matches_b, pairs[p].mscores_a, pairs[p].mscores_b, pairs[p].scores,
             pairs[p].conf) = [x.data_ptr() for x in o]
            outs += o
        args = (C.byref(packed.struct), B, T, n_pad, (C.c_int * T)(*counts), _lib.ptr(kp), _lib.ptr(sc), _lib.ptr(de))
        tail = (100, 0.0, pairs, len(pair_ids), _lib.ptr(ws), nbytes, C.byref(opt), _lib.stream_ptr())
        if views_entry:
            rc = lib.mvm_matcher_forward_views(*args, (C.c_float * (2 * T))(*([1066.0, 1600.0] * T)), *tail)
        else:
            rc = lib.mvm_matcher_forward_ex(*args, 1066.0, 1600.0, *tail)
        _lib.check(rc, 'forward')
        torch.cuda.synchronize()
        return outs

    for a, b in zip(run(False), run(True)):
        assert torch.equal(a, b)


def test_image_in_chain_vs_reference():
    """Two seeded images of different sizes, neither a multiple of 8 -> SuperPoint one image per call (merge=False) ->
    pairwise matcher, against the same chain of the reference."""
    meta, ref = _load(G.CHAIN_CASE['name'])
    imgs = G.chain_images(meta)
    sp = _superpoint(meta['sp_config'], meta['sp_wseed'])
    data = {'ids': [0, 1]}
    for i, img in enumerate(imgs):
        img = torch.from_numpy(img).cuda()
        p = sp({'image': [img]})
        assert np.array_equal(p['keypoints'][0].cpu().numpy().astype(np.int64), ref['keypoints%d' % i].astype(np.int64))
        data.update({'keypoints%d' % i: p['keypoints'][0][None], 'scores%d' % i: p['scores'][0][None],
                     'descriptors%d' % i: p['descriptors'][0][None], 'image%d' % i: img})
    with torch.no_grad():
        got = _matcher(meta['layers'], G.chain_matcher_state_dict(meta)).eval()(data)
    got = {k: v.cpu().numpy() for k, v in got.items() if v is not None}
    rref = {k[5:]: v for k, v in ref.items() if k.startswith('ref__')}
    # SuperPoint's descriptors carry up to 1e-4 of their own error into the matcher: looser couplings, same margin rule
    print(compare_matcher_outputs(rref, got, tau=5e-3, score_tol=(1e-2, 1e-3), min_stable=0.3, conf_tol=1e-2))


def _mixed_pair(seed=0):
    from e2e_multi_view_matching_b200.synthetic import make_state_dict, make_scene_tuple_inputs
    layers = ['self', 'cross'] * 2
    m = _matcher(layers, make_state_dict(len(layers), seed=seed, final_proj_gain=12.0, conf_head='score')).eval()
    data = make_scene_tuple_inputs(78, 2, 256, batch=2, f=500.0, sizes=[(640, 480), (480, 640)])
    data = {k: (torch.from_numpy(v).cuda() if isinstance(v, np.ndarray) and not k.startswith('image')
                else (torch.empty(v.shape, device='meta') if isinstance(v, np.ndarray) else v)) for k, v in data.items()}
    return m, data


@pytest.mark.parametrize('mode', ['w8pt', 'w8pt_ba', 'ransac', 'ransac_ba'])
def test_pair_pipeline_mixed_sizes_matches_oracle(mode):
    """PairPipeline on portrait / landscape synthetic pairs; the pose of the engine's own matches against oracle/pose.py
    (eight-point, two-view BA) and tests/ransac_oracle.py (RANSAC), as test_ransac_gpu.py does for one size."""
    from e2e_multi_view_matching_b200.pipeline import PairPipeline
    matcher, data = _mixed_pair()
    thresh = 0.02
    with torch.no_grad():
        res, pose = PairPipeline(matcher, eval_mode=mode, match_threshold=thresh)(data)
    torch.cuda.synchronize()
    for b in range(2):
        K0, K1 = data['intr0'][b].cpu().numpy(), data['intr1'][b].cpu().numpy()
        if mode.startswith('ransac'):
            n = int(pose['n_matches'][b, 0])
            mk0, mk1 = pose['kpts_a'][b, 0, :n].cpu().numpy(), pose['kpts_b'][b, 0, :n].cpu().numpy()
            mconf = pose['mconf'][b, 0, :n].cpu().numpy()
            ret = RO.estimate_pose(mk0, mk1, K0, K1, 1.0)
            assert bool(pose['success'][b]) == (ret is not None)
            if ret is None:
                continue
            R, t, m = ret
            np.testing.assert_array_equal(pose['inliers'][b, :n].cpu().numpy() > 0, m)
            T = np.eye(4)
            T[:3, :3], T[:3, 3] = R, t
            if mode == 'ransac_ba':
                x0 = P.normalize(mk0[m][None].astype(np.float32), K0[None].astype(np.float32))
                x1 = P.normalize(mk1[m][None].astype(np.float32), K1[None].astype(np.float32))
                ext, valid = P.run_bundle_adjust_2_view(x0.astype(np.float64), x1.astype(np.float64),
                                                        mconf[m][None].astype(np.float64), T[None], n_iterations=10)
                assert bool(pose['valid_ba'][b, 0]) == bool(valid[0])
                if valid[0]:
                    T = ext[0]
            np.testing.assert_allclose(pose['T_021'][b].double().cpu().numpy(), T, atol=1e-4)
            continue
        m0 = res['matches0_0_1'][b].cpu().numpy()
        c = res['conf_scores_0_1'][b, :, 0].cpu().numpy()
        valid = (m0 >= 0) & (c > thresh)
        assert int(pose['n_matches'][b, 0]) == int(valid.sum()) >= 8
        k0 = data['keypoints0'][b].cpu().numpy()[valid].astype(np.float64)[None]
        k1 = data['keypoints1'][b].cpu().numpy()[m0[valid]].astype(np.float64)[None]
        Tw, info = P.estimate_relative_pose_w8pt(k0, k1, K0[None].astype(np.float64), K1[None].astype(np.float64),
                                                 c[valid].astype(np.float64)[None, :, None], determine_inliers=True)
        T = Tw[0]
        if mode == 'w8pt_ba':
            cn = info['confidence'].copy()
            cn[~info['pos_depth_mask']] = 0
            ext, vb = P.run_bundle_adjust_2_view(info['kpts0_norm'], info['kpts1_norm'], cn, Tw, 10)
            T = ext[0] if vb[0] else Tw[0]
        np.testing.assert_allclose(pose['T_021'][b].double().cpu().numpy(), T, atol=1e-3)
