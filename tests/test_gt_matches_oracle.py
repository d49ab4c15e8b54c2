"""CPU: the float64 ground-truth matching of oracle/gt_matches.py against the reference's own outputs
(tests/golden/gt_matches_*.npz, written by oracle/make_gt_matches_golden.py), and its rules where the reference is
undefined (out-of-image pixels, non-finite class weights)."""
import glob
import os

import numpy as np
import pytest

from oracle.gt_matches import gt_matches_pair

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CASES = sorted(glob.glob(os.path.join(GOLDEN, 'gt_matches_*.npz')))


def test_fixtures_exist():
    assert len(CASES) >= 4


@pytest.mark.parametrize('path', CASES, ids=[os.path.basename(p)[11:-4] for p in CASES])
def test_oracle_vs_reference_golden(path):
    z = np.load(path)
    e_match, e_unmatch = [float(x) for x in z['thresholds']]
    o = gt_matches_pair(z['kpts0'], z['kpts1'], z['K0'], z['K1'], z['T'], z['depth0'], z['depth1'], e_match, e_unmatch)
    ref_i, ref_w = z['indices'], z['weights']
    assert o['indices'].shape == ref_i.shape and o['weights'].shape == ref_w.shape and o['weights'].dtype == np.float32
    # the same stable-decision rule as the GPU tests: equal indices wherever the oracle calls the decision stable
    stable = o['stable']
    mism = o['indices'][:, :, :-1] != ref_i[:, :, :-1]
    print(os.path.basename(path), 'unstable decisions:', int((~stable).sum()), 'of', stable.size,
          'index mismatches:', int(mism.sum()))
    assert not (mism & stable).any(), int((mism & stable).sum())
    assert (o['indices'][:, :, -1] == -1).all()
    # the fixtures' own arg-min statistics (reference float32) agree with the oracle's to float32 noise
    for s, key in ((0, 'row_min'), (1, 'col_min')):
        np.testing.assert_allclose(o['emin'][:, s], z[key], rtol=1e-4, atol=1e-3)
    if not mism.any():
        # same decisions => same integer counts => the same float32 class weights
        assert np.array_equal(o['weights'], ref_w)


def _grid_scene(n, H=48, W=64, depth=5.0):
    """n keypoints on distinct integer pixels of a constant-depth plane, identity K and pose: every keypoint is its own
    partner at error 0."""
    ys, xs = np.divmod(np.arange(n) * 7 % (H * W), W)
    k = np.stack([xs, ys], 1).astype(np.float32)[None]
    K = np.diag([50.0, 50.0, 1.0, 1.0]).astype(np.float32)
    K[0, 2], K[1, 2] = W / 2, H / 2
    d = np.full((1, H, W), depth, np.float32)
    return k, K[None], np.eye(4, dtype=np.float32)[None], d


def test_non_finite_weights_are_zero():
    k, K, T, d = _grid_scene(40)
    # every keypoint matched: w_unmatch = 0.5 / 0
    o = gt_matches_pair(k, k, K, K, T, d, d, 5.0, 15.0)
    assert (o['indices'][0, 0, :-1] == np.arange(40)).all() and (o['weights'] == 0).all()
    # every keypoint dropped (no valid depth): 0 / 0
    o = gt_matches_pair(k, k, K, K, T, d * 0, d * 0, 5.0, 15.0)
    assert (o['indices'] == -1).all() and (o['weights'] == 0).all()
    # no match and no drop: w_match = 0.5 / 0
    far = k.copy()
    far[..., 0] = (far[..., 0] + 32) % 64
    far[..., 1] = (far[..., 1] + 24) % 48
    o = gt_matches_pair(k, far, K, K, T, d, d, 0.5, 0.6)
    assert (o['indices'] == -1).all() and (o['weights'] == 0).all()
    # one keypoint less matched than all: finite weights
    o = gt_matches_pair(k, np.concatenate([k[:, :-1], far[:, -1:]], 1), K, K, T, d, d, 0.5, 0.6)
    w = o['weights'][0]
    assert (o['indices'][0, 0, :39] == np.arange(39)).all() and np.isfinite(w).all() and (w > 0).sum() > 0


def test_out_of_image_pixels_clamp_to_the_border():
    k, K, T, d = _grid_scene(4)
    d = d.copy()
    d[0, :, -1] = 9.0                     # right border column
    d[0, 0, :] = 3.0                      # top row
    k = np.array([[[70.5, 10.0], [-0.9, 20.2], [10.0, -0.5], [63.99, 47.99]]], np.float32)
    o = gt_matches_pair(k, k, K, K, T, d, d, 5.0, 15.0)
    # depth look-up at the clamped pixel; -0.9 and -0.5 truncate to 0
    np.testing.assert_array_equal(o['depth'][0, 0], [9.0, 5.0, 3.0, 9.0])
    # the error uses the unclamped truncated pixel: keypoint 0 reprojects from the clamped column 63 but sits at 70
    assert o['emin'][0, 0, 0] == pytest.approx(7.0, abs=1e-9)
    assert o['emin'][0, 0, 1] == pytest.approx(0.0, abs=1e-9)


def test_ties_go_to_the_first_index():
    k, K, T, d = _grid_scene(6)
    k1 = k.copy()
    k1[0, 4] = k1[0, 2]                   # duplicate in view 1: rows tie between 2 and 4
    k1[0, 5] = k1[0, 2] + 0.5             # same truncated pixel
    o = gt_matches_pair(k, k1, K, K, T, d, d, 5.0, 15.0)
    assert o['amin'][0, 0, 2] == 2 and o['indices'][0, 0, 2] == 2
    assert o['stable'][0, 0, 2]           # an exact tie between copies of one pixel is not a rounding question
