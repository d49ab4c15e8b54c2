"""CPU: the host side of the training-image preparation (e2e_multi_view_matching_b200/image_prep.py) against the
reference's formulas (oracle/image_prep.py): the jitter draw, the crop window rule, the intrinsics bookkeeping, and
the refusals that come before any launch."""
import numpy as np
import pytest
import torch

from e2e_multi_view_matching_b200 import image_prep as IP
from oracle import image_prep as R


@pytest.mark.parametrize('jitter', [0.2, 0.4])
def test_color_jitter_params_is_colorjitter_get_params(jitter):
    torch.manual_seed(123)
    ref = [R.get_color_jitter_params(jitter) for _ in range(300)]
    torch.manual_seed(123)
    ours = [IP.color_jitter_params(jitter) for _ in range(300)]
    g = torch.Generator().manual_seed(123)
    with_gen = [IP.color_jitter_params(jitter, generator=g) for _ in range(300)]
    for a, b, c in zip(ref, ours, with_gen):
        assert torch.equal(a[0], b[0]) and torch.equal(a[0], c[0])
        assert a[1:] == b[1:] == c[1:]
        assert all(isinstance(v, float) for v in b[1:])
    assert len({tuple(p[0].tolist()) for p in ours}) > 12          # the orders vary


def test_color_jitter_params_does_not_import_torchvision():
    import os
    import re
    src = open(os.path.join(os.path.dirname(IP.__file__), 'image_prep.py')).read()
    assert not re.search(r'^\s*(from|import)\s+torchvision\b', src, flags=re.M)


@pytest.mark.parametrize('h,w', [(480, 640), (640, 480), (1064, 1600), (1600, 1063), (500, 500), (3, 8)])
def test_square_crop_window_matches_crop(h, w):
    top, bottom, left, right = R.crop_window(h, w, center=True)
    assert IP.square_crop_window(h, w) == (top, left, bottom - top, right - left)
    rng = np.random.RandomState(5)
    for _ in range(20):
        top, bottom, left, right = R.crop_window(h, w, center=False, rng=rng)
        off = left if w > h else top
        assert IP.square_crop_window(h, w, off) == (top, left, bottom - top, right - left)
    with pytest.raises(ValueError):
        IP.square_crop_window(h, w, abs(w - h) + 1)
    with pytest.raises(ValueError):
        IP.square_crop_window(h, w, -1)


def _intr(rng, n=None):
    K = np.eye(3, dtype=np.float32) if n is None else np.tile(np.eye(3, dtype=np.float32), (n, 1, 1))
    K[..., 0, 0] = rng.uniform(300, 1500, () if n is None else n)
    K[..., 1, 1] = rng.uniform(300, 1500, () if n is None else n)
    K[..., 0, 2] = rng.uniform(200, 900, () if n is None else n)
    K[..., 1, 2] = rng.uniform(200, 700, () if n is None else n)
    return K.astype(np.float32)


@pytest.mark.parametrize('kind', ['numpy', 'torch'])
def test_intrinsics_bookkeeping_is_bitwise_the_reference(kind):
    rng = np.random.RandomState(0)
    for _ in range(50):
        K = _intr(rng)
        cx, cy = int(rng.randint(0, 600)), int(rng.randint(0, 600))
        fx, fy = 480 / float(rng.randint(200, 2000)), 640 / float(rng.randint(200, 2000))
        ref = R.resize_intrinsics(R.crop_intrinsics(K.copy(), cx, cy), fx, fy)
        ref_pad = K.copy()
        ref_pad[1, 2] = ref_pad[1, 2] + 2
        ref_pad = R.resize_intrinsics(ref_pad, 640 / 1296, 480 / 972)
        k = K.copy() if kind == 'numpy' else torch.from_numpy(K.copy())
        ours = IP.resize_intrinsics(IP.crop_intrinsics(k, cx, cy), fx, fy)
        k = K.copy() if kind == 'numpy' else torch.from_numpy(K.copy())
        ours_pad = IP.resize_intrinsics(IP.pad_intrinsics(k), 640 / 1296, 480 / 972)
        assert np.array_equal(np.asarray(ours), ref) and np.asarray(ours).dtype == np.float32
        assert np.array_equal(np.asarray(ours_pad), ref_pad)


def test_batched_crop_intrinsics_per_sample_offsets():
    rng = np.random.RandomState(1)
    K = _intr(rng, 6)
    lefts, tops = rng.randint(0, 500, 6), rng.randint(0, 500, 6)
    ref = np.stack([R.crop_intrinsics(K[b].copy(), int(lefts[b]), int(tops[b])) for b in range(6)])
    t = torch.from_numpy(K.copy())
    IP.crop_intrinsics(t, torch.from_numpy(lefts), torch.from_numpy(tops))
    assert np.array_equal(t.numpy(), ref)
    n = K.copy()
    IP.crop_intrinsics(n, lefts, tops)
    assert np.array_equal(n, ref) and n.dtype == np.float32


GEOM = [[0, 0, 968, 1296, 2, 2]]
ORDER = [[3, 1, 0, 2]]


@pytest.mark.parametrize('geometry,src,out,order,factors', [
    ([[0, 1, 968, 1296, 2, 2]], (968, 1296), (480, 640), None, None),        # crop past the right edge
    ([[-1, 0, 10, 10, 0, 0]], (968, 1296), (480, 640), None, None),          # negative top
    ([[0, 0, 0, 10, 0, 0]], (968, 1296), (480, 640), None, None),            # empty crop
    ([[0, 0, 10, 10, -1, 0]], (968, 1296), (480, 640), None, None),          # negative pad
    (GEOM, (968, 1296), (0, 640), None, None),                               # output size below 1
    (GEOM, (968, 1296), (480, 0), None, None),
    (GEOM, (968, 1296), (480, 640), [[0, 1, 2, 2]], [[1., 1., 1., 0.]]),     # not a permutation
    (GEOM, (968, 1296), (480, 640), [[0, 1, 2, 4]], [[1., 1., 1., 0.]]),
    (GEOM, (968, 1296), (480, 640), ORDER, [[-0.1, 1., 1., 0.]]),            # negative brightness
    (GEOM, (968, 1296), (480, 640), ORDER, [[1., -1e-9, 1., 0.]]),           # negative contrast
    (GEOM, (968, 1296), (480, 640), ORDER, [[1., 1., -2., 0.]]),             # negative saturation
    (GEOM, (968, 1296), (480, 640), ORDER, [[1., 1., 1., 0.5000001]]),       # hue outside [-0.5, 0.5]
    (GEOM, (968, 1296), (480, 640), ORDER, [[1., 1., 1., -0.51]]),
    (GEOM, (968, 1296), (480, 640), ORDER, [[1., 1., 1., float('nan')]]),
    (GEOM, (968, 1296), (480, 640), ORDER, None),                            # order without factors
])
def test_check_params_refuses(geometry, src, out, order, factors):
    with pytest.raises(ValueError):
        IP.check_params(src, geometry, out, order, factors)


def test_check_params_accepts_the_range_edges():
    g, o, f = IP.check_params((968, 1296), GEOM * 2, (480, 640), ORDER * 2, [[0., 0., 0., -0.5], [1.2, 0.8, 1.2, 0.5]])
    assert g.dtype == np.int32 and o.dtype == np.int32 and f.dtype == np.float64


def test_prepare_images_refuses_before_any_launch():
    """The refusals come from the host checks: they hold without a GPU and without the library."""
    rgb = torch.zeros(1, 8, 8, 3, dtype=torch.uint8)
    with pytest.raises(ValueError):
        IP.prepare_images(rgb, [[0, 0, 9, 8, 0, 0]], (8, 8))
    with pytest.raises(ValueError):
        IP.prepare_images(rgb.float(), [[0, 0, 8, 8, 0, 0]], (8, 8))
    with pytest.raises(ValueError):
        IP.prepare_images(rgb, [[0, 0, 8, 8, 0, 0]] * 2, (8, 8))
    with pytest.raises(ValueError):
        IP.prepare_images(rgb, [[0, 0, 8, 8, 0, 0]], (8, 8), [[0, 1, 2, 3]], [[1., 1., 1., 0.7]])


def test_prepare_tuple_batch_leaves_image_batches_alone():
    data = {'image0': torch.zeros(2, 1, 4, 4), 'depth0': torch.zeros(2, 4, 4), 'intr0': torch.eye(3).expand(2, 3, 3)}
    before = dict(data)
    assert IP.prepare_tuple_batch(data) is data
    assert data.keys() == before.keys() and all(data[k] is before[k] for k in data)
