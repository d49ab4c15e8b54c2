"""Batched SuperPoint keypoint selection and descriptor sampling (mvm_superpoint_select / mvm_superpoint_sample_batch,
SuperPoint.forward_batch) on the GPU:
  - the selection against a float64 NumPy restatement of threshold, border mask and top-k (tie rule included) on
    planted score maps of every size class;
  - forward_batch against forward, bitwise, at the cfg5 training shape, with and without fill_with_random_keypoints;
  - forward_batch against the reference fixtures, with the criteria of tests/test_superpoint_gpu.py;
  - no host synchronisation without fill;
  - train_step / validation_step / MultiViewPipeline from images against the same calls after run_super_point by hand."""
import json
import os
import types
import zlib

import numpy as np
import pytest
import torch

from tests.util import GOLDEN

pytestmark = pytest.mark.gpu


# ---- selection against a float64 restatement ---------------------------------------------------------------------------
def select_ref(smap, thr, border, k):
    """superpoint.py:181-189 restated in float64 on one map [Hs, Ws]: candidates in raster order; with more than k of them
    the k largest, descending, equal scores by raster index.  -> (count, indices)."""
    s = smap.astype(np.float64)
    Hs, Ws = s.shape
    yy, xx = np.mgrid[0:Hs, 0:Ws]
    cand = (s > np.float64(np.float32(thr))) & (yy >= border) & (yy < Hs - border) & (xx >= border) & (xx < Ws - border)
    idx = np.flatnonzero(cand)
    if len(idx) <= k:
        return len(idx), idx
    vals = s.reshape(-1)[idx]
    order = np.lexsort((idx, -vals))
    return len(idx), idx[order[:k]]


def run_select(maps, thr, border, k):
    from e2e_multi_view_matching_b200 import _lib
    B, Hs, Ws = maps.shape
    kp = torch.full((B, k, 2), -1.0, device='cuda')
    sc = torch.full((B, k), -1.0, device='cuda')
    cnt = torch.full((B,), -1, dtype=torch.int32, device='cuda')
    _lib.check(_lib.lib().mvm_superpoint_select(_lib.ptr(maps), B, Hs, Ws, float(thr), border, k, _lib.ptr(kp),
                                                _lib.ptr(sc), _lib.ptr(cnt), _lib.stream_ptr()), 'select')
    torch.cuda.synchronize()
    return kp.cpu().numpy(), sc.cpu().numpy(), cnt.cpu().numpy()


SIZES = {(16, 16): (40, 20, 0.5), (133, 201): (7, 400, 0.06), (480, 640): (5, 400, 0.04), (1066, 1600): (2, 2048, 0.03)}


def planted_maps(H, W, B, density, seed):
    """Post-NMS-like score maps [B, 8*(H//8), 8*(W//8)]: a sparse set of pixels with scores in (0, 1), zeros elsewhere."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    Hs, Ws = H // 8 * 8, W // 8 * 8
    vals = torch.rand(B, Hs, Ws, generator=g, device='cuda') * 0.999 + 0.0005
    keep = torch.rand(B, Hs, Ws, generator=g, device='cuda') < density
    return (vals * keep).contiguous()


def valid_values(smap, border):
    Hs, Ws = smap.shape
    v = smap[border:Hs - border, border:Ws - border].reshape(-1) if border else smap.reshape(-1)
    return np.sort(v[v > 0])[::-1]


@pytest.mark.parametrize('border', [0, 4, 12])
@pytest.mark.parametrize('mode', ['none', 'fewer', 'exact', 'many', 'ties'])
@pytest.mark.parametrize('size', list(SIZES), ids=lambda s: '%dx%d' % s)
def test_select_vs_float64(size, mode, border):
    B, k, density = SIZES[size]
    maps = planted_maps(*size, B, density, seed=zlib.crc32(repr((size, mode, border)).encode()))
    m = maps.cpu().numpy()
    thr = [0.0] * B
    for b in range(B):
        v = valid_values(m[b], border)
        if mode == 'none':
            thr[b] = 0.9995
        elif mode == 'fewer' and len(v) > 1:
            thr[b] = float(v[min(k // 2, len(v) - 1)])
        elif mode == 'exact' and len(v) > k and v[k - 1] > v[k]:
            thr[b] = float(v[k])
        elif mode == 'ties' and len(v) > k + 4:
            # the k-th score repeated on both sides of the cut: the lower raster indices must win
            Hs, Ws = m[b].shape
            ys, xs = np.nonzero(m[b] > 0)
            inside = (ys >= border) & (ys < Hs - border) & (xs >= border) & (xs < Ws - border)
            ys, xs = ys[inside], xs[inside]
            below = m[b][ys, xs] < v[k - 1]
            pick = np.random.default_rng(b).permutation(np.flatnonzero(below))[:max(3, k // 4)]
            m[b][ys[pick], xs[pick]] = v[k - 1]
    # the selection reads one threshold per call: 'fewer' / 'exact' run image by image
    per_image = mode in ('fewer', 'exact')
    maps = torch.from_numpy(m).cuda().contiguous()
    groups = [[b] for b in range(B)] if per_image else [list(range(B))]
    for grp in groups:
        t = thr[grp[0]]
        kp, sc, cnt = run_select(maps[grp].contiguous(), t, border, k)
        for j, b in enumerate(grp):
            n, idx = select_ref(m[b], t, border, k)
            if mode == 'exact' and thr[b] > 0:
                assert n == k
            assert cnt[j] == n, (b, cnt[j], n)
            got = len(idx)
            Ws = m[b].shape[1]
            assert np.array_equal(kp[j, :got, 0], (idx % Ws).astype(np.float32))
            assert np.array_equal(kp[j, :got, 1], (idx // Ws).astype(np.float32))
            assert np.array_equal(sc[j, :got], m[b].reshape(-1)[idx])
            if n > k:
                assert np.all(np.diff(sc[j].astype(np.float64)) <= 0)                  # descending
            assert not kp[j, got:].any() and not sc[j, got:].any()                     # zeros past the count
    if mode == 'none':
        assert cnt.max() == 0
    if mode == 'many' and not (size == (16, 16) and border == 12):                 # (no pixel is 12 inside a 16 x 16 map)
        assert cnt.min() > k


@pytest.mark.parametrize('B', [1, 40])
def test_select_batch_extremes(B):
    """B = 1 and B = 40 maps of 480 x 640 in one launch, every image with its own count above and below k."""
    maps = planted_maps(480, 640, B, 0.002, seed=B)
    m = maps.cpu().numpy()
    k = 600
    kp, sc, cnt = run_select(maps, 0.3, 4, k)
    for b in range(B):
        n, idx = select_ref(m[b], 0.3, 4, k)
        assert cnt[b] == n
        assert np.array_equal(kp[b, :len(idx), 0], (idx % 640).astype(np.float32))
        assert np.array_equal(kp[b, :len(idx), 1], (idx // 640).astype(np.float32))
        assert np.array_equal(sc[b, :len(idx)], m[b].reshape(-1)[idx])


# ---- forward_batch against forward ----------------------------------------------------------------------------------
def _superpoint(config, wseed=1):
    from e2e_multi_view_matching_b200.models.superpoint import SuperPoint
    from e2e_multi_view_matching_b200.synthetic import make_superpoint_state_dict
    sp = SuperPoint(config).eval()
    sp.load_state_dict({k: torch.from_numpy(v) for k, v in make_superpoint_state_dict(wseed).items()}, strict=True)
    return sp.cuda()


def _cfg5_images(n=40, seed=11):
    from e2e_multi_view_matching_b200.synthetic import make_image
    return torch.from_numpy(make_image(seed, 480, 640, batch=n)).cuda()


CFG5 = {'nms_radius': 4, 'keypoint_threshold': 0.001, 'max_keypoints': 400, 'remove_borders': 12}


def _aligned(kp, sc, de, W):
    """forward's output of one image in the selection's order: descending score, equal scores by raster index (torch.topk
    leaves that order open)."""
    order = np.lexsort((kp[:, 1] * W + kp[:, 0], -sc.astype(np.float64)))
    return kp[order], sc[order], de[:, order]


@pytest.mark.parametrize('fill', [False, True])
@pytest.mark.parametrize('k', ['cfg5', 'median'])
def test_forward_batch_equals_forward(fill, k):
    imgs = _cfg5_images()
    cfg = dict(CFG5, fill_with_random_keypoints=fill)
    sp = _superpoint(cfg)
    if k == 'median':
        # max_keypoints at the median candidate count: half of the images are short of it, half are cut
        smap, _ = sp.dense(imgs)
        s = smap[:, 12:-12, 12:-12]
        cfg['max_keypoints'] = int(torch.median((s > cfg['keypoint_threshold']).sum((1, 2))).item())
        sp.config.update(cfg)
        torch.cuda.synchronize()
    K = cfg['max_keypoints']
    smap, _ = sp.dense(imgs)
    n_cand = (smap[:, 12:-12, 12:-12] > cfg['keypoint_threshold']).sum((1, 2)).cpu().numpy()
    torch.manual_seed(123)
    ref = sp({'image': [imgs]})
    torch.manual_seed(123)
    out = sp.forward_batch(imgs)
    torch.cuda.synchronize()
    assert out['keypoints'].shape == (40, K, 2) and out['scores'].shape == (40, K)
    assert out['descriptors'].shape == (40, 256, K) and out['counts'].dtype == torch.int32
    counts = out['counts'].cpu().numpy()
    assert np.array_equal(counts, np.full(40, K) if fill else np.minimum(n_cand, K))
    for b in range(40):
        kp_r = ref['keypoints'][b].cpu().numpy()
        sc_r = ref['scores'][b].cpu().numpy()
        de_r = ref['descriptors'][b].cpu().numpy()
        if n_cand[b] > K:                                                    # cut by torch.topk
            kp_r, sc_r, de_r = _aligned(kp_r, sc_r, de_r, 640)
        kp, sc, de = (out['keypoints'][b].cpu().numpy(), out['scores'][b].cpu().numpy(),
                      out['descriptors'][b].cpu().numpy())
        n = kp_r.shape[0]
        assert np.array_equal(kp[:n], kp_r) and np.array_equal(sc[:n], sc_r), b
        assert np.array_equal(de[:, :n], de_r), b                               # bitwise: the same sampling code
        assert not kp[n:].any() and not sc[n:].any() and not de[:, n:].any()
    if k == 'median':
        assert 0 < (n_cand < K).sum() < 40
    else:
        assert (n_cand > K).all()


def test_forward_batch_has_no_host_sync():
    imgs = _cfg5_images(8)
    sp = _superpoint(dict(CFG5, fill_with_random_keypoints=False))
    sp.forward_batch(imgs)                                  # weights packed, workspace allocated
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = sp.forward_batch(imgs)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert out['descriptors'].shape == (8, 256, 400)


SP_GOLDEN = ['superpoint_240x320_top200_b2', 'superpoint_480x640_top1024', 'superpoint_120x160_all',
             'native_sp_1066x1600_top2048', 'native_sp_1600x1066_top2048', 'native_sp_133x201_all']


@pytest.mark.parametrize('name', SP_GOLDEN)
def test_forward_batch_vs_reference_golden(name):
    """The fixtures of the unmodified reference: keypoints exact (raster order when all are kept, as sets under top-k),
    scores rtol 2e-5, descriptors within 1e-4, unit norm.  A fixture that keeps every keypoint (max_keypoints -1) runs
    with max_keypoints = its keypoint count."""
    from e2e_multi_view_matching_b200.synthetic import make_image
    z = np.load(os.path.join(GOLDEN, name + '.npz'))
    meta = json.loads(str(z['meta']))
    batch = meta.get('batch', 1)
    refs = [{'keypoints': z['keypoints%d' % b], 'scores': z['scores%d' % b], 'descriptors': z['descriptors%d' % b]}
            for b in range(batch)] if 'keypoints0' in z.files else [{k: z[k] for k in ('keypoints', 'scores',
                                                                                        'descriptors', 'desc_columns')}]
    K = meta['max_keypoints'] if meta['max_keypoints'] > 0 else max(r['keypoints'].shape[0] for r in refs)
    sp = _superpoint({'max_keypoints': K}, meta['wseed'])
    img = torch.from_numpy(make_image(meta['seed'], meta['height'], meta['width'], batch)).cuda()
    out = sp.forward_batch(img)
    for b, r in enumerate(refs):
        n = int(out['counts'][b])
        kp_ref = r['keypoints'].astype(np.int64)
        kp = out['keypoints'][b, :n].cpu().numpy()
        assert kp.shape == kp_ref.shape
        if meta['max_keypoints'] < 0:
            assert np.array_equal(kp.astype(np.int64), kp_ref)
            order = order_ref = np.arange(n)
        else:
            key = lambda a: a[:, 1] * 100000 + a[:, 0]
            order, order_ref = np.argsort(key(kp.astype(np.int64))), np.argsort(key(kp_ref))
            assert np.array_equal(kp.astype(np.int64)[order], kp_ref[order_ref])
        np.testing.assert_allclose(out['scores'][b, :n].cpu().numpy()[order], r['scores'][order_ref], rtol=2e-5, atol=1e-7)
        d = out['descriptors'][b, :, :n].cpu().numpy()
        if 'desc_columns' in r:
            inv = np.empty_like(order)
            inv[order_ref] = order
            err = np.abs(d[:, inv[r['desc_columns']]] - r['descriptors']).max()
        else:
            err = np.abs(d[:, order] - r['descriptors'][:, order_ref]).max()
        assert err < 1e-4, err
        np.testing.assert_allclose(np.linalg.norm(d, axis=0), 1.0, atol=1e-5)


# ---- end to end from images -----------------------------------------------------------------------------------------
def _image_batch(T=3, B=2, H=240, W=320, seed=3):
    """A rendered tuple batch with images, depth maps, 4x4 intrinsics and cam->world poses, and no keypoints."""
    from e2e_multi_view_matching_b200.synthetic import make_scene_tuple_inputs, render_tuple_images
    d = render_tuple_images(make_scene_tuple_inputs(seed, T, 300, batch=B, width=W, height=H, noise_px=0.0), seed=seed)
    data = {'ids': list(range(T))}
    for i in range(T):
        K4 = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
        K4[:, :3, :3] = d['intr%d' % i]
        data['image%d' % i] = torch.from_numpy(d['image%d' % i]).cuda()
        data['depth%d' % i] = torch.full((B, H, W), 4.0, device='cuda')
        data['intr%d' % i] = torch.from_numpy(K4).cuda()
        data['pose%d' % i] = torch.from_numpy(d['pose%d' % i]).cuda()
    return data


def _train_matcher(T, seed=5):
    from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher
    from e2e_multi_view_matching_b200.synthetic import make_state_dict
    layers = ['self', 'cross'] * 2
    m = MultiViewMatcher({'multi_frame_matching': T > 2, 'GNN_layers': layers, 'conf_mlp': False, 'full_output': False})
    sd = make_state_dict(len(layers), seed=seed, final_proj_gain=8.0)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items() if not k.startswith('conf_mlp')})
    return m.cuda()


TRAIN_SP = {'nms_radius': 4, 'keypoint_threshold': 0.001, 'max_keypoints': 128, 'remove_borders': 12,
            'fill_with_random_keypoints': True}
OPT = types.SimpleNamespace(pose_loss=False, batch_size=2, match_reproj_err=5.0, unmatch_reproj_err=15.0,
                            rot_weight=0.0, trans_weight=0.0)


def test_train_step_from_images_is_bitwise_the_step_after_run_super_point():
    from e2e_multi_view_matching_b200 import training
    sp = _superpoint(TRAIN_SP)
    data = _image_batch()
    model_a = _train_matcher(3).train()
    model_b = _train_matcher(3).train()
    opt_a = torch.optim.Adam(model_a.parameters(), lr=1e-4)
    opt_b = torch.optim.Adam(model_b.parameters(), lr=1e-4)
    torch.manual_seed(7)
    loss_a, _ = training.train_step(OPT, dict(data), model_a, opt_a, 3, super_point=sp)
    by_hand = dict(data)
    torch.manual_seed(7)
    training.run_super_point(OPT, by_hand, sp)
    assert by_hand['keypoints0'].shape == (2, 128, 2) and by_hand['descriptors2'].shape == (2, 256, 128)
    loss_b, _ = training.train_step(OPT, by_hand, model_b, opt_b, 3)
    assert torch.isfinite(loss_a) and torch.equal(loss_a, loss_b)
    for (n, pa), pb in zip(model_a.named_parameters(), model_b.parameters()):
        assert (pa.grad is None) == (pb.grad is None), n
        if pa.grad is not None:
            assert torch.equal(pa.grad, pb.grad), n
        assert torch.equal(pa, pb), n


def test_validation_step_from_images_is_bitwise_the_step_after_run_super_point():
    from e2e_multi_view_matching_b200 import training
    sp = _superpoint(TRAIN_SP)
    data = _image_batch(seed=4)
    model = _train_matcher(3).eval()
    torch.manual_seed(8)
    val_a, parts_a = training.validation_step(OPT, dict(data), model, 3, 0.0, super_point=sp)
    by_hand = dict(data)
    torch.manual_seed(8)
    training.run_super_point(OPT, by_hand, sp)
    val_b, parts_b = training.validation_step(OPT, by_hand, model, 3, 0.0)
    assert torch.isfinite(val_a).all() and torch.equal(val_a, val_b)
    assert all(torch.equal(parts_a[k], parts_b[k]) for k in parts_a)


def test_multi_view_pipeline_from_images_matches_keypoint_in():
    from e2e_multi_view_matching_b200 import training
    from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher
    from e2e_multi_view_matching_b200.pipeline import MultiViewPipeline
    from e2e_multi_view_matching_b200.synthetic import make_state_dict
    layers = (['self'] + ['cross'] * 3) * 2
    m = MultiViewMatcher({'multi_frame_matching': True, 'GNN_layers': layers}).eval()
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in
                       make_state_dict(len(layers), seed=2, final_proj_gain=12.0, conf_head='score').items()})
    m = m.cuda()
    sp = _superpoint({'max_keypoints': 256, 'keypoint_threshold': 0.005, 'remove_borders': 4})
    data = _image_batch(T=4, B=1, H=480, W=640, seed=9)
    for i in range(4):
        data.pop('depth%d' % i)
        data['intr%d' % i] = data['intr%d' % i][:, :3, :3].contiguous()
    with torch.no_grad():
        res_a, pose_a = MultiViewPipeline(m, superpoint=sp)(data)
        by_hand = dict(data)
        training.run_super_point(types.SimpleNamespace(batch_size=1), by_hand, sp)
        res_b, pose_b = MultiViewPipeline(m)(by_hand)
    assert 'keypoints0' not in data and pose_a is not None
    for k, v in res_b.items():
        assert torch.equal(res_a[k], v), k
    for i in range(4):
        assert torch.equal(res_a['keypoints%d' % i], by_hand['keypoints%d' % i])
    assert torch.equal(pose_a['extrinsics'], pose_b['extrinsics'])


def test_run_super_point_short_images_take_one_dense_pass():
    """Without fill, a merged batch with images short of max_keypoints: run_super_point makes one SuperPoint.dense call
    and hands each image forward's keypoints / scores / descriptors (bitwise; equal scores at the cut by the tie rule)."""
    from e2e_multi_view_matching_b200 import training
    imgs = _cfg5_images(3, seed=21)
    sp = _superpoint(dict(CFG5, fill_with_random_keypoints=False))
    smap, _ = sp.dense(imgs)
    n_cand = (smap[:, 12:-12, 12:-12] > CFG5['keypoint_threshold']).sum((1, 2)).cpu().numpy()
    K = int(np.sort(n_cand)[1])                                       # one image short, one exact, one cut
    sp.config['max_keypoints'] = K
    dense_calls = []
    real_dense = sp.dense
    sp.dense = lambda images: dense_calls.append(images.shape) or real_dense(images)
    data = {'ids': [0, 1, 2], **{'image%d' % m: imgs[m:m + 1] for m in range(3)}}
    training.run_super_point(types.SimpleNamespace(batch_size=1), data, sp)
    assert len(dense_calls) == 1
    ref = sp({'image': [imgs]})
    for m in range(3):
        kp_r, sc_r, de_r = (ref[k][m].cpu().numpy() for k in ('keypoints', 'scores', 'descriptors'))
        if n_cand[m] > K:
            kp_r, sc_r, de_r = _aligned(kp_r, sc_r, de_r, 640)
        assert data['keypoints%d' % m].shape == (1, min(n_cand[m], K), 2)
        assert np.array_equal(data['keypoints%d' % m][0].cpu().numpy(), kp_r)
        assert np.array_equal(data['scores%d' % m][0].cpu().numpy(), sc_r)
        assert np.array_equal(data['descriptors%d' % m][0].cpu().numpy(), de_r)


def test_eval_multi_view_images_mode(tmp_path):
    """eval_multi_view --images end to end on one rendered tuple: SuperPoint, matcher, bundle adjustment, AUC file."""
    from e2e_multi_view_matching_b200 import eval_multi_view
    out = tmp_path / 'mv.json'
    metrics = eval_multi_view.main(['--images', '--n_tuples', '1', '--tuple_size', '3', '--max_keypoints', '256',
                                    '--out', str(out)])
    assert json.load(open(out)) == metrics
    assert sorted(metrics) == sorted('%s_AUC@%ddeg' % (n, t) for n in ('pose', 'transl', 'rot') for t in (5, 10, 20))
    assert all(np.isfinite(v) and 0.0 <= v <= 100.0 for v in metrics.values())
