"""GPU: mvm_image_prep / image_prep.prepare_tuple_batch against the reference's transform sequence written with
torchvision functional ops on the CPU in float32 (oracle/image_prep.py).

Tiers: chains without contrast and resize are bitwise (every order of brightness, saturation and hue; contrast at
factor 1.0 is the identity in any position); the resize reproduces the arithmetic of torch's generic CPU bilinear
kernel: bitwise at the ScanNet shape and at ratios like 2 or 0.96, a few ulps off at odd ratios such as 37 -> 20,
where torch's vectorised loop rounds differently (and its single-thread three-channel path differs throughout), so
it is held to 2^-22 with the differing pixels counted; contrast's mean is an fp64 reduction on the GPU and a float32
cascade sum in torch (at most one ulp apart, printed), and _rgb2hsv's divisions by small chroma amplify that ulp when
hue follows contrast, so contrast chains are held to 2^-20."""
import itertools

import numpy as np
import pytest
import torch

from e2e_multi_view_matching_b200 import image_prep as IP
from oracle import image_prep as R

pytestmark = pytest.mark.gpu

SCANNET = (968, 1296)


def _special_image(h, w, seed):
    """Random colours plus, in the first rows: black, white, greys (maxc == minc), channel ties (maxc == r == g and
    the others), pure and near-pure primaries whose hue wraps past 0 and 1 under a shift."""
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    special = [(0, 0, 0), (255, 255, 255), (128, 128, 128), (1, 1, 1), (254, 254, 254), (200, 200, 50),
               (50, 200, 200), (200, 50, 200), (50, 50, 200), (200, 50, 50), (50, 200, 50), (255, 0, 10),
               (255, 10, 0), (255, 0, 0), (0, 255, 0), (0, 0, 255), (255, 0, 255), (10, 0, 255), (255, 255, 0),
               (0, 255, 255), (255, 1, 0), (255, 0, 1), (3, 2, 2), (2, 3, 3), (100, 100, 101), (101, 100, 100)]
    flat = img.reshape(-1, 3)
    k = min(len(special), len(flat))
    flat[:k] = special[:k]
    k = min(len(special), max(0, len(flat) - w))
    flat[w:w + k] = np.array(special)[::-1][:k]
    return img


def _run(imgs, geoms, out_size, params=None):
    """imgs list of [H, W, 3] uint8 of one size -> kernel output [n, 1, oh, ow] on the CPU."""
    rgb = torch.from_numpy(np.stack(imgs))
    order = factors = None
    if params is not None:
        order = np.stack([np.asarray(p[0], np.int64) for p in params])
        factors = np.array([p[1:] for p in params], np.float64)
    out = IP.prepare_images(rgb, geoms, out_size, order, factors)
    torch.cuda.synchronize()
    return out.cpu()


def _oracle(img, depth_shape, crop=None, params=None):
    jp = None if params is None else (torch.as_tensor(params[0]),) + tuple(params[1:])
    gray, _, _ = R.prepare_image(img, np.zeros(depth_shape, np.float32), np.eye(3, dtype=np.float32), crop, jp)
    return gray


def _full(img):
    h, w = img.shape[:2]
    return [0, 0, h, w, 0, 0]


EDGE_FACTORS = [(0.8, 1.0, 0.8, -0.2), (1.2, 1.0, 1.2, 0.2), (0.8, 1.0, 1.2, 0.5), (1.2, 1.0, 0.8, -0.5),
                (1.0, 1.0, 1.0, 0.0), (0.0, 1.0, 0.0, 0.5), (1.2, 1.0, 1.2, -0.5)]


def test_chains_without_contrast_or_resize_are_bitwise():
    """All 24 orders x edge factors (contrast 1.0: the identity wherever it sits in the order), on pixels that take
    every branch of _rgb2hsv / _hsv2rgb."""
    imgs, params, geoms = [], [], []
    for k, (order, fac) in enumerate(itertools.product(itertools.permutations(range(4)), EDGE_FACTORS)):
        img = _special_image(12, 40, k % 5)
        imgs.append(img)
        params.append((list(order),) + fac)
        geoms.append(_full(img))
    out = _run(imgs, geoms, (12, 40), params)
    bad = 0
    for k, img in enumerate(imgs):
        ref = _oracle(img, (12, 40), None, params[k])
        if not torch.equal(out[k], ref):
            bad += 1
            d = (out[k] - ref).abs()
            print('order %s factors %s: %d pixels differ, max %.3e' % (params[k][0], params[k][1:], int((d > 0).sum()),
                                                                       float(d.max())))
    assert bad == 0


def test_hue_wraps_and_hue_only_chains_are_bitwise():
    img = _special_image(30, 64, 9)
    hues = [-0.5, -0.4999, -0.3, -0.2, -1e-7, 0.0, 1e-7, 0.2, 0.3, 0.4999, 0.5]
    params = [([3, 0, 1, 2], 1.0, 1.0, 1.0, h) for h in hues]
    out = _run([img] * len(hues), [_full(img)] * len(hues), (30, 64), params)
    for k, p in enumerate(params):
        assert torch.equal(out[k], _oracle(img, (30, 64), None, p)), p


@pytest.mark.parametrize('src,dst', [(SCANNET, (480, 640)), ((480, 640), (240, 320)), ((37, 53), (20, 31)),
                                     ((20, 31), (37, 53)), ((500, 500), (480, 640)), ((97, 101), (50, 60))])
def test_resize_against_torch_cpu(src, dst):
    imgs = [_special_image(src[0], src[1], s) for s in range(2)]
    geoms = [_full(imgs[0]) for _ in imgs]
    if src == SCANNET:
        geoms = [[0, 0, src[0], src[1], 2, 2] for _ in imgs]
    out = _run(imgs, geoms, dst)
    n_diff, worst = 0, 0.0
    for k, img in enumerate(imgs):
        d = (out[k] - _oracle(img, dst)).abs()
        n_diff += int((d > 0).sum())
        worst = max(worst, float(d.max()))
    print('resize %s -> %s (torch threads %d): %d of %d pixels differ, max %.3e'
          % (src, dst, torch.get_num_threads(), n_diff, out.numel(), worst))
    assert worst <= 2.0 ** -22


def test_contrast_all_orders():
    rng = np.random.default_rng(3)
    imgs, params = [], []
    for k, order in enumerate(itertools.permutations(range(4))):
        imgs.append(_special_image(40, 56, k))
        params.append((list(order),) + tuple(float(np.float32(v)) for v in
                                             (rng.uniform(0.8, 1.2), rng.uniform(0.8, 1.2), rng.uniform(0.8, 1.2),
                                              rng.uniform(-0.2, 0.2))))
    out = _run(imgs, [_full(imgs[0])] * len(imgs), (40, 56), params)
    worst = 0.0
    for k, img in enumerate(imgs):
        worst = max(worst, float((out[k] - _oracle(img, (40, 56), None, params[k])).abs().max()))
    # the means themselves: contrast factor 0 turns the image into its mean, gray(mean, mean, mean) for both sides
    mean_params = [(p[0], p[1], 0.0, p[3], p[4]) for p in params]
    out_m = _run(imgs, [_full(imgs[0])] * len(imgs), (40, 56), mean_params)
    mdiff = [float((out_m[k, 0, 0, 0].double() - _oracle(img, (40, 56), None, mean_params[k])[0, 0, 0].double()).abs())
             for k, img in enumerate(imgs)]
    print('contrast: max |kernel - oracle| %.3e; contrast-mean difference (through gray) max %.3e, mean %.3e'
          % (worst, max(mdiff), float(np.mean(mdiff))))
    assert worst <= 2.0 ** -20 and max(mdiff) <= 2.0 ** -22


def test_contrast_with_resize_at_the_scannet_shape():
    img = _special_image(*SCANNET, 4)
    p = ([2, 1, 3, 0], 1.1, 0.9, 1.15, 0.13)
    out = _run([img], [[0, 0, 968, 1296, 2, 2]], (480, 640), [p])
    d = (out[0] - _oracle(img, (480, 640), None, p)).abs()
    print('scannet + jitter: %d pixels differ, max %.3e' % (int((d > 0).sum()), float(d.max())))
    assert float(d.max()) <= 2.0 ** -20


@pytest.mark.parametrize('h,w,offset', [(1064, 1600, None), (1064, 1600, 0), (1064, 1600, 536), (1064, 1600, 211),
                                        (1600, 1063, 377), (63, 64, None), (77, 45, 5)])
def test_megadepth_square_crops(h, w, offset):
    img = _special_image(h, w, 7)
    top, left, s, _ = IP.square_crop_window(h, w, offset)
    out = _run([img], [[top, left, s, s, 0, 0]], (s, s))
    assert torch.equal(out[0], _oracle(img, (h, w), (top, top + s, left, left + s)))


@pytest.mark.parametrize('h,w', [(480, 640), (7, 5), (1, 1), (33, 17)])
def test_unchanged_sizes_without_jitter_are_bitwise(h, w):
    img = _special_image(h, w, 1)
    out = _run([img], [_full(img)], (h, w))
    assert out.shape == (1, 1, h, w) and torch.equal(out[0], _oracle(img, (h, w)))


def test_repeat_launches_and_batch_of_40_against_batch_of_1_are_bitwise():
    rng = np.random.default_rng(0)
    imgs = [_special_image(*SCANNET, s) for s in range(40)]
    torch.manual_seed(1)
    params = [IP.color_jitter_params(0.2) for _ in range(40)]
    params = [(p[0].tolist(),) + p[1:] for p in params]
    geoms = [[0, 0, 968, 1296, 2, 2]] * 40
    a = _run(imgs, geoms, (480, 640), params)
    b = _run(imgs, geoms, (480, 640), params)
    assert torch.equal(a, b)
    for k in rng.choice(40, 6, replace=False):
        assert torch.equal(_run([imgs[k]], geoms[:1], (480, 640), [params[k]])[0], a[k])
    # and the batch against the oracle, at the contrast tier
    worst = max(float((a[k] - _oracle(imgs[k], (480, 640), None, params[k])).abs().max()) for k in range(0, 40, 13))
    print('cfg5 scannet batch, max |kernel - oracle| %.3e' % worst)
    assert worst <= 2.0 ** -20


def test_graph_capture_replays_the_eager_result():
    img = _special_image(64, 96, 2)
    rgb = torch.from_numpy(np.stack([img] * 3)).cuda()
    g = torch.tensor([[0, 0, 64, 96, 1, 1]] * 3, dtype=torch.int32, device='cuda')
    order = torch.tensor([[1, 0, 2, 3], [3, 2, 1, 0], [0, 3, 1, 2]], dtype=torch.int32, device='cuda')
    fac = torch.tensor([[1.1, 0.9, 1.2, 0.1]] * 3, dtype=torch.float64, device='cuda')
    from e2e_multi_view_matching_b200 import _lib
    L = _lib.lib()
    out = torch.empty(3, 1, 48, 80, device='cuda')
    ws = torch.empty(L.mvm_image_prep_workspace_bytes(3, 48, 80), dtype=torch.uint8, device='cuda')

    def launch():
        _lib.check(L.mvm_image_prep(_lib.ptr(rgb), 3, 64, 96, _lib.ptr(g), _lib.ptr(order), _lib.ptr(fac), 48, 80,
                                    _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), 'mvm_image_prep')
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        launch()
    torch.cuda.synchronize()
    eager = out.clone()
    out.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        launch()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


def test_library_refuses_null_pointers_and_empty_outputs():
    from e2e_multi_view_matching_b200 import _lib
    L = _lib.lib()
    rgb = torch.zeros(1, 8, 8, 3, dtype=torch.uint8, device='cuda')
    g = torch.tensor([[0, 0, 8, 8, 0, 0]], dtype=torch.int32, device='cuda')
    out = torch.empty(1, 1, 8, 8, device='cuda')
    o = torch.tensor([[0, 1, 2, 3]], dtype=torch.int32, device='cuda')
    f = torch.ones(1, 4, dtype=torch.float64, device='cuda')
    p = _lib.ptr
    assert L.mvm_image_prep(p(None), 1, 8, 8, p(g), None, None, 8, 8, p(out), None, 0, _lib.stream_ptr()) == 1
    assert L.mvm_image_prep(p(rgb), 1, 8, 8, p(None), None, None, 8, 8, p(out), None, 0, _lib.stream_ptr()) == 1
    assert L.mvm_image_prep(p(rgb), 1, 8, 8, p(g), None, None, 8, 8, p(None), None, 0, _lib.stream_ptr()) == 1
    assert L.mvm_image_prep(p(rgb), 1, 8, 8, p(g), None, None, 0, 8, p(out), None, 0, _lib.stream_ptr()) == 1
    assert L.mvm_image_prep(p(rgb), 1, 8, 8, p(g), p(o), None, 8, 8, p(out), None, 0, _lib.stream_ptr()) == 1
    assert L.mvm_image_prep(p(rgb), 1, 8, 8, p(g), p(o), p(f), 8, 8, p(out), None, 0, _lib.stream_ptr()) == 1


# ---- end to end -------------------------------------------------------------------------------------------------------
def _u8_tuple_batch(T=3, B=2, H=240, W=320, seed=3):
    """A rendered tuple batch handed over as the dataset would after the change: decoded uint8 RGB, depth, 4x4
    intrinsics, poses, and the tuple's jitter parameters (contrast 1.0: the bitwise tier)."""
    from e2e_multi_view_matching_b200.synthetic import make_scene_tuple_inputs, render_tuple_images
    d = render_tuple_images(make_scene_tuple_inputs(seed, T, 300, batch=B, width=W, height=H, noise_px=0.0), seed=seed)
    data = {'ids': list(range(T))}
    tint = np.array([1.0, 0.85, 0.7], np.float32)
    for i in range(T):
        K4 = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
        K4[:, :3, :3] = d['intr%d' % i]
        data['rgb%d' % i] = torch.from_numpy(np.round(d['image%d' % i][:, 0, :, :, None] * tint * 255).astype(np.uint8))
        data['depth%d' % i] = torch.full((B, H, W), 4.0)
        data['intr%d' % i] = torch.from_numpy(K4)
        data['pose%d' % i] = torch.from_numpy(d['pose%d' % i])
    g = torch.Generator().manual_seed(seed)
    params = [IP.color_jitter_params(0.2, g) for _ in range(B)]
    data['jitter_order'] = torch.stack([p[0] for p in params])
    data['jitter_factors'] = torch.tensor([(p[1], 1.0, p[3], p[4]) for p in params], dtype=torch.float64)
    return data


def _oracle_batch(data):
    T = len(data['ids'])
    out = {'ids': data['ids']}
    B = data['rgb0'].shape[0]
    for i in range(T):
        imgs, intrs = [], []
        for b in range(B):
            jp = (data['jitter_order'][b],) + tuple(float(v) for v in data['jitter_factors'][b])
            gray, _, K = R.prepare_image(data['rgb%d' % i][b].numpy(), data['depth%d' % i][b].numpy(),
                                         data['intr%d' % i][b].numpy(), None, jp)
            imgs.append(gray)
            intrs.append(torch.from_numpy(K))
        out['image%d' % i] = torch.stack(imgs)
        out['intr%d' % i] = torch.stack(intrs)
        out['depth%d' % i] = data['depth%d' % i].clone()
        out['pose%d' % i] = data['pose%d' % i].clone()
    return out


def _cuda(data):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in data.items()}


def test_prepare_tuple_batch_then_train_step_is_bitwise_the_oracle_batch():
    from e2e_multi_view_matching_b200 import training
    from tests.test_superpoint_batch_gpu import OPT, TRAIN_SP, _superpoint, _train_matcher
    raw = _u8_tuple_batch()
    ref = _cuda(_oracle_batch(raw))
    ours = IP.prepare_tuple_batch(dict(raw))
    assert not any(k.startswith(('rgb', 'jitter')) for k in ours)
    ours = _cuda(ours)
    assert ours.keys() == ref.keys()
    for k in ref:
        if isinstance(ref[k], torch.Tensor):
            assert ours[k].shape == ref[k].shape and torch.equal(ours[k], ref[k]), k
    sp = _superpoint(TRAIN_SP)
    model_a, model_b = _train_matcher(3).train(), _train_matcher(3).train()
    opt_a = torch.optim.Adam(model_a.parameters(), lr=1e-4)
    opt_b = torch.optim.Adam(model_b.parameters(), lr=1e-4)
    torch.manual_seed(7)
    loss_a, _ = training.train_step(OPT, ours, model_a, opt_a, 3, super_point=sp)
    torch.manual_seed(7)
    loss_b, _ = training.train_step(OPT, ref, model_b, opt_b, 3, super_point=sp)
    assert torch.isfinite(loss_a) and torch.equal(loss_a, loss_b)
    for (n, pa), pb in zip(model_a.named_parameters(), model_b.parameters()):
        assert (pa.grad is None) == (pb.grad is None), n
        if pa.grad is not None:
            assert torch.equal(pa.grad, pb.grad), n


def test_prepare_tuple_batch_scannet_and_megadepth_match_getitem():
    """Intrinsics, depth crops and images of prepare_tuple_batch against __getitem__ view by view: a ScanNet-sized
    view (pad + resize, jitter 0.2) and a MegaDepth-like view (random square crop offsets, no jitter)."""
    rng = np.random.default_rng(5)
    B = 2
    Ks = np.tile(np.array([[1160., 0, 648.5], [0, 1165., 484.25], [0, 0, 1]], np.float32), (B, 1, 1))
    torch.manual_seed(2)
    params = [IP.color_jitter_params(0.2) for _ in range(B)]
    sc = {'ids': [0], 'rgb0': torch.from_numpy(rng.integers(0, 256, (B, 968, 1296, 3), dtype=np.uint8)),
          'depth0': torch.from_numpy(rng.uniform(0, 5, (B, 480, 640)).astype(np.float32)), 'intr0': torch.from_numpy(Ks),
          'jitter_order': torch.stack([p[0] for p in params]),
          'jitter_factors': torch.tensor([p[1:] for p in params], dtype=torch.float64)}
    offs = [17, 120]
    md = {'ids': [0], 'rgb0': torch.from_numpy(rng.integers(0, 256, (B, 300, 420, 3), dtype=np.uint8)),
          'depth0': torch.from_numpy(rng.uniform(0, 5, (B, 300, 420)).astype(np.float32)),
          'intr0': torch.from_numpy(Ks.copy()), 'crop0': torch.tensor(offs)}
    for data, jit, crops in ((sc, True, None), (md, False, offs)):
        raw = {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in data.items()}
        out = IP.prepare_tuple_batch(data)
        for b in range(B):
            jp = (raw['jitter_order'][b],) + tuple(float(v) for v in raw['jitter_factors'][b]) if jit else None
            crop = None
            if crops is not None:
                t, lf, s, _ = IP.square_crop_window(300, 420, crops[b])
                crop = (t, t + s, lf, lf + s)
            gray, depth, K = R.prepare_image(raw['rgb0'][b].numpy(), raw['depth0'][b].numpy(), raw['intr0'][b].numpy(),
                                             crop, jp)
            assert np.array_equal(out['intr0'][b].numpy(), K)
            assert np.array_equal(out['depth0'][b].numpy(), depth)
            d = float((out['image0'][b].cpu() - gray).abs().max())
            assert d <= (2.0 ** -20 if jit else 0.0), d
