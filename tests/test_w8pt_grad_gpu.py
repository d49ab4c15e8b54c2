"""The CUDA backward of the weighted eight-point (mvm_w8pt_backward behind estimate_relative_pose_w8pt's autograd):
against the reference's own autograd (tests/golden/w8pt_grad_*.npz, oracle/make_w8pt_grad_golden.py), against the
float64 numpy oracle (oracle.pose_grad.w8pt_conf_grad) on seeded batches up to the cfg5 and cfg2 shapes, NaN on
rank-deficient items only, determinism, no change to the forward, and one use: learning to down-weight outliers."""
import ctypes
import glob
import json
import os

import numpy as np
import pytest
import torch

from oracle import pose as P
from oracle import pose_grad as PG
from tests.util import GOLDEN

pytestmark = pytest.mark.gpu

CASES = sorted(glob.glob(os.path.join(GOLDEN, 'w8pt_grad_*.npz')))
LOSSES = ('rot', 'transl', 'both', 'conf')


def _erp():
    from e2e_multi_view_matching_b200.pose_optimization.two_view.estimate_relative_pose import estimate_relative_pose_w8pt
    return estimate_relative_pose_w8pt


def _grad(k0, k1, K, conf, gT, gcn, choose_closest, Tg):
    """conf [B,N,1] float32 CUDA -> d<gT, T021> + <gcn, conf_norm> / d conf, [B,N] numpy."""
    c = conf.detach().clone().requires_grad_()
    T, info = _erp()(k0, k1, K, K, c, choose_closest=choose_closest, T_021=Tg)
    torch.autograd.backward([T, info['confidence']], [gT, gcn.reshape(info['confidence'].shape)])
    return c.grad[..., 0].cpu().numpy().astype(np.float64)


def _batch(seeds, n, outl=0.3, zero=0.0):
    rng = np.random.default_rng(seeds[0])
    scs = [P.make_two_view_scene(s, n, outlier_frac=outl) for s in seeds]
    z = {k: np.concatenate([s[k] for s in scs]).astype(np.float32) for k in ('kpts0', 'kpts1', 'intr', 'conf', 'T_021')}
    drop = rng.uniform(size=z['conf'].shape[:2]) < zero
    z['conf'][drop] = 0.0
    z['kpts1'][drop] = z['kpts1'][:, -1:].repeat(n, 1)[drop]
    return z


def _cuda(z, *keys):
    return [torch.from_numpy(np.ascontiguousarray(z[k])).cuda() for k in keys]


@pytest.mark.parametrize('branch', ['closest', 'vote'])
@pytest.mark.parametrize('path', CASES, ids=[os.path.basename(p)[10:-4] for p in CASES])
def test_grad_vs_reference_golden(path, branch):
    z = np.load(path)
    name = json.loads(str(z['meta']))['name']
    k0, k1, K, c, Tg = _cuda(z, 'kpts0', 'kpts1', 'intr', 'conf', 'T_gt')
    nz = (z['conf'][..., 0] != 0).sum(-1)
    ratios = []
    for loss in LOSSES:
        key = '%s_%s' % (branch, loss)
        gT = torch.from_numpy(z['gT64_' + key]).float().cuda()
        gcn = torch.from_numpy(z['gcn_' + key]).float().cuda()
        g = _grad(k0, k1, K, c, gT, gcn, branch == 'closest', Tg)
        g64, g32 = z['g64_' + key], z['g32_' + key]
        for b in range(len(nz)):
            if nz[b] < 8:
                assert np.isnan(g[b]).all(), (name, key, b)
                continue
            scale = np.abs(g64[b]).max()
            tol = max(3.0 * np.abs(g32[b] - g64[b]).max(), 1e-5 * scale)
            err = np.abs(g[b] - g64[b]).max()
            ratios.append(err / tol)
            assert err <= tol, (name, key, b, err, tol, scale)
    print('%s %s: |cuda - ref64| / tol: max %.3f median %.3f' % (name, branch, max(ratios), float(np.median(ratios))))


@pytest.mark.parametrize('B,n', [(2, 40), (8, 400), (32, 1024)])
@pytest.mark.parametrize('choose_closest', [True, False])
def test_grad_vs_numpy_oracle(B, n, choose_closest):
    z = _batch(list(range(500 + B, 500 + 2 * B)), n, outl=0.3, zero=0.05)
    rng = np.random.default_rng(B * n)
    gT = np.zeros((B, 4, 4), np.float32)
    gT[:, :3, :] = rng.standard_normal((B, 3, 4))
    gcn = (rng.standard_normal((B, n)) / n).astype(np.float32)
    k0, k1, K, c, Tg = _cuda(z, 'kpts0', 'kpts1', 'intr', 'conf', 'T_021')
    g = _grad(k0, k1, K, c, torch.from_numpy(gT).cuda(), torch.from_numpy(gcn).cuda(), choose_closest, Tg)
    go = PG.w8pt_conf_grad(z['kpts0'], z['kpts1'], z['intr'], z['intr'], z['conf'], gT.astype(np.float64),
                           gcn.astype(np.float64), choose_closest=choose_closest, T_021=z['T_021'].astype(np.float64))
    rel = np.abs(g - go).max(-1) / np.abs(go).max(-1)
    print('B=%d n=%d closest=%s: |cuda - oracle| / max|oracle| per item: max %.2e median %.2e'
          % (B, n, choose_closest, rel.max(), np.median(rel)))
    assert np.isfinite(g).all()
    assert rel.max() < 1e-5, rel


def test_rank_deficient_items_are_nan_and_only_those():
    B, n = 6, 30
    z = _batch(list(range(600, 600 + B)), n, outl=0.0)
    keep = [30, 8, 7, 3, 0, 9]          # non-zero weights per item
    for b, k in enumerate(keep):
        z['conf'][b, k:] = 0.0
    k0, k1, K, c, Tg = _cuda(z, 'kpts0', 'kpts1', 'intr', 'conf', 'T_021')
    for cc in (True, False):
        gT = torch.randn(B, 4, 4, device='cuda')
        g = _grad(k0, k1, K, c, gT, torch.zeros(B, n, device='cuda'), cc, Tg)
        for b, k in enumerate(keep):
            if k < 8:
                assert np.isnan(g[b]).all(), (cc, b)
            else:
                assert np.isfinite(g[b]).all(), (cc, b)


def test_backward_deterministic_and_batch_independent():
    B, n = 8, 400
    z = _batch(list(range(700, 700 + B)), n, zero=0.05)
    k0, k1, K, c, Tg = _cuda(z, 'kpts0', 'kpts1', 'intr', 'conf', 'T_021')
    gT = torch.randn(B, 4, 4, device='cuda', generator=torch.Generator('cuda').manual_seed(0))
    gcn = torch.randn(B, n, device='cuda', generator=torch.Generator('cuda').manual_seed(1))
    for cc in (True, False):
        g0 = _grad(k0, k1, K, c, gT, gcn, cc, Tg)
        for _ in range(3):
            assert np.array_equal(_grad(k0, k1, K, c, gT, gcn, cc, Tg), g0, equal_nan=True)
        for b in (0, 3, 7):
            s = slice(b, b + 1)
            gb = _grad(k0[s], k1[s], K[s], c[s], gT[s], gcn[s], cc, Tg[s])
            assert np.array_equal(gb[0], g0[b], equal_nan=True), (cc, b)


def test_forward_unchanged_by_requires_grad():
    from e2e_multi_view_matching_b200 import _lib
    B, n = 4, 200
    z = _batch(list(range(800, 800 + B)), n, zero=0.1)
    k0, k1, K, c, Tg = _cuda(z, 'kpts0', 'kpts1', 'intr', 'conf', 'T_021')
    L = _lib.lib()
    for cc in (True, False):
        n0 = L.mvm_launch_count()
        T, info = _erp()(k0, k1, K, K, c, choose_closest=cc, T_021=Tg, determine_inliers=True)
        torch.cuda.synchronize()
        assert L.mvm_launch_count() - n0 == 1
        assert not T.requires_grad and T.grad_fn is None
        cg = c.clone().requires_grad_()
        Tr, infor = _erp()(k0, k1, K, K, cg, choose_closest=cc, T_021=Tg, determine_inliers=True)
        assert Tr.requires_grad and infor['confidence'].requires_grad
        assert torch.equal(T, Tr.detach())
        for k in ('kpts0_norm', 'kpts1_norm', 'confidence', 'inliers', 'pos_depth_mask', 'F'):
            assert torch.equal(info[k], infor[k].detach()), k
            if k != 'confidence':
                assert not infor[k].requires_grad, k
        with torch.no_grad():
            n0 = L.mvm_launch_count()
            Tn, _ = _erp()(k0, k1, K, K, cg, choose_closest=cc, T_021=Tg)
            assert L.mvm_launch_count() - n0 == 1 and Tn.grad_fn is None
            assert torch.equal(T, Tn)


def test_backward_refuses_invalid_arguments_like_forward():
    from e2e_multi_view_matching_b200 import _lib
    L = _lib.lib()
    x = torch.zeros(64, device='cuda')
    p = _lib.ptr(x)
    null = ctypes.c_void_p(0)
    s = _lib.stream_ptr()
    fwd_null = L.mvm_w8pt(null, p, p, p, p, 1, 8, null, 0, 0, p, p, p, p, p, null, null, null, null, s)
    fwd_batch = L.mvm_w8pt(p, p, p, p, p, 0, 8, null, 0, 0, p, p, p, p, p, null, null, null, null, s)
    fwd_tgt = L.mvm_w8pt(p, p, p, p, p, 1, 8, null, 1, 0, p, p, p, p, p, null, null, null, null, s)
    assert fwd_null != 0 and fwd_batch != 0 and fwd_tgt != 0
    assert L.mvm_w8pt_backward(null, p, p, p, p, 1, 8, null, 0, p, p, null, p, s) == fwd_null
    assert L.mvm_w8pt_backward(p, p, p, p, p, 1, 8, null, 0, p, p, null, null, s) == fwd_null
    assert L.mvm_w8pt_backward(p, p, p, p, p, 0, 8, null, 0, p, p, null, p, s) == fwd_batch
    assert L.mvm_w8pt_backward(p, p, p, p, p, 1, 0, null, 0, p, p, null, p, s) == fwd_batch
    assert L.mvm_w8pt_backward(p, p, p, p, p, 1, 8, null, 1, p, p, null, p, s) == fwd_tgt


def test_learning_confidences_downweights_outliers():
    """Adam on per-match confidence logits through the pose losses (rotation + translation angle, choose_closest
    against the true pose, as the reference's stage-2 training): the loss falls and the outliers end below the
    inliers."""
    from e2e_multi_view_matching_b200.pose_optimization.two_view.compute_pose_error import (
        compute_rotation_error, compute_translation_error_as_angle)
    sc = P.make_two_view_scene(900, 200, outlier_frac=0.4, noise_px=1.0)
    k0, k1, K, Tg = _cuda(sc, 'kpts0', 'kpts1', 'intr', 'T_021')
    out = torch.from_numpy(sc['outlier'][0]).cuda()
    logits = torch.zeros(1, 200, 1, device='cuda', requires_grad=True)
    opt = torch.optim.Adam([logits], lr=0.1)
    losses = []
    for _ in range(40):
        T, _ = _erp()(k0, k1, K, K, torch.sigmoid(logits), choose_closest=True, T_021=Tg)
        loss = compute_rotation_error(T, Tg) + compute_translation_error_as_angle(T, Tg)
        opt.zero_grad()
        loss.backward()
        assert torch.isfinite(logits.grad).all()
        opt.step()
        losses.append(loss.item())
    conf = torch.sigmoid(logits.detach())[0, :, 0]
    print('loss %.4f -> %.4f (min %.4f); mean conf inliers %.3f outliers %.3f'
          % (losses[0], losses[-1], min(losses), float(conf[~out].mean()), float(conf[out].mean())))
    assert losses[-1] < 0.8 * losses[0]
    assert float(conf[out].mean()) < float(conf[~out].mean())
