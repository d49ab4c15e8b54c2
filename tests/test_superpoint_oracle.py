"""CPU: the SuperPoint restatement of oracle/superpoint.py, run in float64 on the seeded weights and images of the
reference fixtures (oracle/make_superpoint_golden.py, oracle/make_native_sizes_golden.py), reproduces what the
unmodified reference computed in float32: the same keypoints after the threshold, remove_borders and top-k rules,
and the scores and descriptors at them within the reference's float32 noise.  That pins the restatement before
tests/test_superpoint_shapes_gpu.py uses it as the float64 yardstick of the kernels.

Keypoint sets may differ only at near-ties, decisions that float32 noise can flip: a score within the noise of the
threshold, of the k-th score, or of another score in its NMS window.  They are counted and printed (none on these
fixtures)."""
import json
import os

import numpy as np
import pytest
import torch

from tests.util import GOLDEN

NMS_RADIUS, THRESHOLD, BORDER = 4, 0.005, 4        # the SuperPoint defaults the fixtures were made with
EPS32 = 2.0 ** -24


def _case(name):
    z = np.load(os.path.join(GOLDEN, name + '.npz'))
    meta = json.loads(str(z['meta']))
    B = meta.get('batch', 1)
    per = []
    for b in range(B):
        sfx = str(b) if 'keypoints0' in z.files else ''
        kp = z['keypoints' + sfx].astype(np.int64)
        cols = z['desc_columns'] if 'desc_columns' in z.files else np.arange(len(kp))
        per.append(dict(kp=kp, scores=z['scores' + sfx], desc=z['descriptors' + sfx], cols=cols))
    return meta, per


def _near_ties(raw, kp, tol, k_score):
    """Of the keypoints kp (x, y), those whose selection float32 noise could flip."""
    out = []
    for x, y in kp:
        s = raw[y, x]
        win = raw[max(0, y - NMS_RADIUS):y + NMS_RADIUS + 1, max(0, x - NMS_RADIUS):x + NMS_RADIUS + 1]
        others = np.sort(np.abs(win.ravel() - s))[1:]               # drop the pixel itself
        if abs(s - THRESHOLD) <= tol or (k_score is not None and abs(s - k_score) <= tol) or \
                (others.size and others[0] <= tol):
            out.append((x, y))
    return out


@pytest.mark.parametrize('name', ['superpoint_120x160_all', 'superpoint_240x320_top200_b2', 'native_sp_133x201_all'])
def test_restatement_reproduces_reference_fixture(name):
    from oracle import superpoint as O
    from e2e_multi_view_matching_b200.synthetic import make_superpoint_state_dict, make_image
    meta, per = _case(name)
    sd = make_superpoint_state_dict(meta['wseed'])
    img = make_image(meta['seed'], meta['height'], meta['width'], meta.get('batch', 1))
    raw64, nms64, d64 = O.dense(img, sd, NMS_RADIUS, torch.float64)
    raw32, _, d32 = O.dense(img, sd, NMS_RADIUS, torch.float32)
    h, w = meta['height'] // 8, meta['width'] // 8
    assert raw64.shape == (len(per), 8 * h, 8 * w) and d64.shape == (len(per), h, w, 256)
    # the yardstick: how far a float32 run of the same operations lands from float64, over the whole case
    dev_s = float((raw32.double() - raw64).abs().max())
    for b, ref in enumerate(per):
        kp, sc = O.select(nms64[b], THRESHOLD, BORDER, meta['max_keypoints'])
        kp = kp.numpy()
        ours, theirs = set(map(tuple, kp.tolist())), set(map(tuple, ref['kp'].tolist()))
        diff = sorted(ours ^ theirs)
        tol = 3 * dev_s
        k_score = float(sc.min()) if meta['max_keypoints'] >= 0 and len(sc) == meta['max_keypoints'] else None
        ties = _near_ties(raw64[b].numpy(), diff, tol, k_score)
        print('%s[%d]: %d keypoints, %d differ from the fixture, %d of them near-ties' %
              (name, b, len(theirs), len(diff), len(ties)))
        assert len(ties) == len(diff), [p for p in diff if p not in ties]
        assert len(diff) <= max(2, len(theirs) // 100)
        # scores at the fixture's keypoints: within 3 x the float32 deviation + 4 ulp of the map's maximum
        kg = ref['kp']
        s64 = raw64[b].numpy()[kg[:, 1], kg[:, 0]]
        bound_s = 3 * dev_s + 4 * EPS32 * float(raw64[b].max())
        err_s = float(np.abs(ref['scores'] - s64).max())
        # descriptors at the fixture's keypoints: the float64 dense map sampled there, against the same yardstick
        kc = torch.from_numpy(kg[ref['cols']])
        D64 = O.sample(d64[b], kc.double()).numpy()
        D32 = O.sample(d32[b], kc.float()).double().numpy()
        bound_d = 3 * float(np.abs(D32 - D64).max()) + 4 * EPS32
        err_d = float(np.abs(ref['desc'] - D64).max())
        print('  scores %.2e (%.2f of bound), descriptors %.2e (%.2f of bound)' %
              (err_s, err_s / bound_s, err_d, err_d / bound_d))
        assert err_s <= bound_s and err_d <= bound_d


def test_simple_nms_rules():
    """The suppression on hand-made maps: a plateau keeps every pixel of it that no kept neighbour suppresses; the
    second and third rounds revive maxima that were only hidden by suppressed pixels; radius 0 is the identity."""
    from oracle.superpoint import simple_nms
    s = torch.zeros(1, 1, 12)
    s[0, 0, [0, 3, 6, 9]] = torch.tensor([0.5, 0.6, 0.7, 0.8])
    # r = 2: every peak's larger neighbour is 3 away, outside its window, so all four are window maxima
    assert torch.equal(simple_nms(s, 2), s)
    # r = 3: only 0.8 is a window max; 0.7 is suppressed by it; 0.6 becomes a max of what is left in round one;
    # 0.5 is suppressed by 0.6 (3 away)
    out = simple_nms(s, 3)
    assert out[0, 0].tolist() == [0, 0, 0, pytest.approx(0.6), 0, 0, 0, 0, 0, pytest.approx(0.8), 0, 0]
    p = torch.full((1, 5, 5), 0.25)
    assert torch.equal(simple_nms(p, 1), p)                       # a plateau: every pixel equals its window max
    r = torch.rand(2, 9, 11, dtype=torch.float64)
    assert torch.equal(simple_nms(r, 0), r)
