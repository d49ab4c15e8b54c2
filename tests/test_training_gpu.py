"""Training consumers (SURVEY.md §8 a20 / f-2): compute_match_loss kernels (forward + backward) and the
exact unrolled-iteration gradient of log_optimal_transport, against autograd through the CPU restatement of the
reference's functions (helpers.py:228-241, superglue.py:143-172) in double precision."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref_match_loss(log_p, gt_indices, gt_weights):
    """helpers.py:228-241, statement for statement (torch, any device / dtype)."""
    bs, ft, _ = log_p.shape
    mi0, mi1 = gt_indices.narrow(1, 0, 1), gt_indices.narrow(1, 1, 1)
    mw0, mw1 = gt_weights.narrow(1, 0, 1), gt_weights.narrow(1, 1, 1)
    l0 = -log_p.reshape(bs * ft, ft)[range(bs * ft), mi0.reshape(bs * ft)]
    l1 = -log_p.transpose(1, 2).reshape(bs * ft, ft)[range(bs * ft), mi1.reshape(bs * ft)]
    return (torch.dot(l0, mw0.reshape(bs * ft)) + torch.dot(l1, mw1.reshape(bs * ft))) / bs


@pytest.mark.parametrize('bs,ft', [(1, 9), (3, 65), (2, 257), (1, 2), (2, 401), (80, 401), (1, 1025), (1, 2049)])
def test_match_loss_forward_backward(bs, ft):
    from e2e_multi_view_matching_b200.training import compute_match_loss
    g = torch.Generator().manual_seed(ft)
    log_p = -torch.rand(bs, ft, ft, generator=g) * 5
    idx = torch.randint(-1, ft - 1, (bs, 2, ft), generator=g)            # -1 = dustbin (last index)
    w = torch.rand(bs, 2, ft, generator=g)
    w[idx == -1] *= 0.3
    ref_in = log_p.double().requires_grad_(True)
    ref = _ref_match_loss(ref_in, idx, w.double())
    ref.backward()
    x = log_p.cuda().requires_grad_(True)
    loss = compute_match_loss(x, idx.cuda(), w.cuda())
    (2.5 * loss).backward()
    assert abs(loss.item() - ref.item()) < 1e-5 * max(1.0, abs(ref.item()))
    np.testing.assert_allclose(x.grad.cpu().numpy(), 2.5 * ref_in.grad.numpy(), rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize('shape,spread', [((2, 40, 33), 1.0), ((1, 128, 128), 6.0), ((1, 300, 257), 3.0)])
def test_log_optimal_transport_gradient(shape, spread):
    from e2e_multi_view_matching_b200.training import log_optimal_transport
    from oracle.matcher_torch import _log_optimal_transport as ref_lot
    b, m, n = shape
    g = torch.Generator().manual_seed(m + n)
    s = torch.randn(b, m, n, generator=g) * spread
    G = torch.randn(b, m + 1, n + 1, generator=g)
    sr = s.double().requires_grad_(True)
    ar = torch.tensor(1.0, dtype=torch.float64, requires_grad=True)
    Zr = ref_lot(sr, ar, 100)
    (Zr * G.double()).sum().backward()
    sc = s.cuda().requires_grad_(True)
    ac = torch.tensor(1.0, device='cuda', requires_grad=True)
    Z = log_optimal_transport(sc, ac, 100)
    assert (Z.detach().cpu().double() - Zr.detach()).abs().max().item() < 1e-4 + 1e-5 * Zr.abs().max().item()
    (Z * G.cuda()).sum().backward()
    scale = sr.grad.abs().max().item()
    assert (sc.grad.cpu().double() - sr.grad).abs().max().item() < 1e-5 * scale + 1e-7
    assert abs(ac.grad.item() - ar.grad.item()) < 1e-4 * max(1.0, abs(ar.grad.item()))


def test_combine_losses():
    from e2e_multi_view_matching_b200.training import combine_losses
    losses = {'match_loss': torch.tensor(6.0), 'rot_loss': torch.tensor(3.0), 'transl_loss': torch.tensor(9.0)}
    total, per = combine_losses(losses, 3, 0.25, 2.0, 0.5)
    assert abs(per['match_loss'].item() - 2.0) < 1e-7
    assert abs(total.item() - (0.75 * 2.0 + 0.25 * (2.0 * 1.0 + 0.5 * 3.0))) < 1e-6


@pytest.mark.parametrize('name', ['mv3_128', 'pair_192'])
def test_run_matcher_vs_reference_golden(name):
    """helpers.run_matcher (helpers.py:243-260) in eval mode -- the reference's validation pass -- against the losses the
    unmodified reference produced on the same seeded inputs (oracle/make_validation_golden.py, fp32 and fp64 runs)."""
    import json
    import types
    from oracle.make_validation_golden import build
    from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher
    from e2e_multi_view_matching_b200.training import run_matcher, validation_step
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'validation_%s.npz' % name))
    case = json.loads(str(z['meta']))
    data_np, sd = build(case)
    model = MultiViewMatcher({'multi_frame_matching': case['views'] > 2, 'GNN_layers': case['layers'], 'conf_mlp': True}).eval()
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    model = model.cuda()
    data = {k: (torch.from_numpy(v).cuda() if isinstance(v, np.ndarray) else v) for k, v in data_np.items()}
    opt = types.SimpleNamespace(pose_loss=True, rot_weight=1.0, trans_weight=0.5)
    with torch.no_grad():
        losses, result = run_matcher(opt, data, model)
    for k in ('match_loss', 'rot_loss', 'transl_loss'):
        ours, r32, r64 = float(losses[k]), float(z[k + '_f32']), float(z[k + '_f64'])
        tol = max(4.0 * abs(r32 - r64), 2e-4 * abs(r64))          # the reference's own fp32 noise is the yardstick
        print(name, k, 'ours %.8g  ref fp32 %.8g  ref fp64 %.8g  tol %.3g' % (ours, r32, r64, tol))
        assert abs(ours - r64) <= tol, (k, ours, r32, r64)
    n_pairs = case['views'] * (case['views'] - 1) // 2
    val, parts = validation_step(opt, data, model, n_pairs, 0.25)
    expect = 0.75 * float(losses['match_loss']) / n_pairs + 0.25 * (float(losses['rot_loss']) + 0.5 * float(losses['transl_loss'])) / n_pairs
    assert abs(float(val) - expect) <= 1e-5 * abs(expect)
