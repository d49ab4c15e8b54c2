"""The float64 numpy restatement of the weighted eight-point's confidence gradient (oracle.pose_grad.w8pt_conf_grad, the
closed forms the CUDA backward computes) against the reference's own float64 autograd, stored in
tests/golden/w8pt_grad_*.npz by oracle/make_w8pt_grad_golden.py.  CPU only."""
import glob
import json
import os

import numpy as np
import pytest

from oracle import pose as P
from oracle import pose_grad as PG
from tests.util import GOLDEN

CASES = sorted(glob.glob(os.path.join(GOLDEN, 'w8pt_grad_*.npz')))
LOSSES = ('rot', 'transl', 'both', 'conf')


def test_goldens_present():
    assert len(CASES) >= 9


@pytest.mark.parametrize('branch', ['closest', 'vote'])
@pytest.mark.parametrize('path', CASES, ids=[os.path.basename(p)[10:-4] for p in CASES])
def test_oracle_vs_reference_fp64_autograd(path, branch):
    z = np.load(path)
    name = json.loads(str(z['meta']))['name']
    nz = (z['conf'][..., 0] != 0).sum(-1)
    worst = 0.0
    for loss in LOSSES:
        key = '%s_%s' % (branch, loss)
        g = PG.w8pt_conf_grad(z['kpts0'], z['kpts1'], z['intr'], z['intr'], z['conf'], z['gT64_' + key],
                              z['gcn_' + key], choose_closest=branch == 'closest', T_021=z['T_gt'].astype(np.float64))
        ref = z['g64_' + key]
        for b in range(len(nz)):
            if nz[b] < 8:
                # rank-deficient: the eigenvector is not unique; the reference's float64 autograd returns huge values
                assert np.isnan(g[b]).all(), (name, key, b)
                continue
            scale = np.abs(ref[b]).max()
            err = np.abs(g[b] - ref[b]).max()
            assert err <= 1e-8 * scale + 1e-12, (name, key, b, err, scale)
            if scale > 1e-9:
                worst = max(worst, err / scale)
    print('%s %s: worst |oracle - ref64| / max|ref64| = %.2e' % (name, branch, worst))


def test_oracle_matches_finite_differences():
    """The closed forms against central differences of the numpy forward, on a scene with outliers and zeroed rows."""
    sc = P.make_two_view_scene(7, 60, outlier_frac=0.3)
    k0, k1, K, c, Tg = (sc[k].astype(np.float64) for k in ('kpts0', 'kpts1', 'intr', 'conf', 'T_021'))
    c[0, :5, 0] = 0.0
    rng = np.random.default_rng(0)
    gT = np.zeros((1, 4, 4))
    gT[0, :3, :4] = rng.standard_normal((3, 4))
    gcn = rng.standard_normal((1, 60))
    for cc in (True, False):
        g = PG.w8pt_conf_grad(k0, k1, K, K, c, gT, gcn, choose_closest=cc, T_021=Tg)

        def L(cv):
            T, info = P.estimate_relative_pose_w8pt(k0, k1, K, K, cv, choose_closest=cc, T_021=Tg)
            return (gT * T).sum() + (gcn * info['confidence'][..., 0]).sum()
        for i in (0, 7, 31, 59):
            d = np.zeros_like(c)
            d[0, i, 0] = 1e-6
            fd = (L(c + d) - L(c - d)) / 2e-6
            assert abs(fd - g[0, i]) <= 1e-6 * max(1.0, abs(fd)), (cc, i, fd, g[0, i])
