"""Stage 2 of the training step (the pose loss) on the CPU: the product's host-side orchestration -- training.train_step
with opt.pose_loss, run_matcher with `conf_grad`, MatcherTrainFn's differentiable conf_scores and the confidence head's
backward (models/train_forward.py) -- with the stage kernels replaced by float64 stand-ins: oracle/train_ops.py for the
matcher, oracle/conf_grad.py for the two confidence-head kernels (csrc/conf_train.cu), oracle/pose.py and
oracle/pose_grad.w8pt_conf_grad for the weighted eight-point and its backward.  Against the unmodified reference
(tests/golden/train_pose_*.npz, oracle/make_train_pose_golden.py): losses, every parameter's gradient (conf_mlp.*
included), the gradient at conf_scores_*, the matches and the head's running statistics.  Also: the head's forward
over every pair at once, the optimiser helpers, the ratio ramp, the skipped step on a non-finite gradient, and the code
generation of the new kernels."""
import argparse
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tests import emul_ops
from tests.test_train_host_logic import PATCHED, check_gradients, match_loss

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ['mv3_r05', 'mv3_r10', 'mv5_r05', 'mv5_r10', 'pair_r05', 'pair_r10']


class _W8ptStandIn(torch.autograd.Function):
    """estimate_relative_pose_w8pt(choose_closest=True) -> T021 on oracle/pose.py (float64), its backward by
    oracle/pose_grad.w8pt_conf_grad (the closed form mvm_w8pt_backward computes)."""

    @staticmethod
    def forward(ctx, conf, kpts0, kpts1, intr0, intr1, T_021):
        from oracle import pose as P
        a = [t.detach().double().numpy() for t in (kpts0, kpts1, intr0, intr1, conf, T_021)]
        T, _ = P.estimate_relative_pose_w8pt(*a[:5], choose_closest=True, T_021=a[5])
        ctx.args, ctx.shape = a, conf.shape
        return torch.from_numpy(T).float()

    @staticmethod
    def backward(ctx, gT):
        from oracle.pose_grad import w8pt_conf_grad
        k0, k1, i0, i1, c, Tt = ctx.args
        g = w8pt_conf_grad(k0, k1, i0, i1, c, gT.double().numpy(), None, choose_closest=True, T_021=Tt)
        return torch.from_numpy(g).float().reshape(ctx.shape), None, None, None, None, None


def _w8pt_stand_in(kpts0, kpts1, intr0, intr1, confidence, choose_closest=False, T_021=None, determine_inliers=False):
    assert choose_closest and not determine_inliers
    return _W8ptStandIn.apply(confidence, kpts0, kpts1, intr0, intr1, T_021), {}


def _patch(monkeypatch):
    from e2e_multi_view_matching_b200 import ops, _lib, training
    from e2e_multi_view_matching_b200.pose_optimization.two_view import estimate_relative_pose as erp
    from oracle import conf_grad
    for f in PATCHED + ['extract_matches']:
        monkeypatch.setattr(ops, f, getattr(emul_ops, f))
    for f in ('conf_tail_backward', 'conf_gather_backward'):
        monkeypatch.setattr(ops, f, getattr(conf_grad, f))
    monkeypatch.setattr(_lib, 'require_cuda', lambda device, what: None)
    monkeypatch.setattr(erp, 'estimate_relative_pose_w8pt', _w8pt_stand_in)
    monkeypatch.setattr(training, 'compute_match_loss', match_loss)


def _setup(name):
    from oracle.make_train_pose_golden import build
    from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher
    z = np.load(os.path.join(GOLDEN, 'train_pose_%s.npz' % name))
    case = json.loads(str(z['meta']))
    data_np, sd = build(case)
    model = MultiViewMatcher({'multi_frame_matching': case['multi'], 'GNN_layers': case['layers'], 'conf_mlp': True})
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    model.train()
    data = {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in data_np.items()}
    opt = argparse.Namespace(pose_loss=True, rot_weight=case['rot_weight'], trans_weight=case['trans_weight'])
    return z, case, model, data, opt


def _optimizer(model, lr=0.0):
    from e2e_multi_view_matching_b200.training import get_parameters
    opt = torch.optim.Adam(get_parameters(model, blacklist_key='conf_mlp'), lr=lr)
    opt.add_param_group({'params': get_parameters(model, whitelist_key='conf_mlp'), 'lr': lr})
    return opt


def _spy_run_matcher(monkeypatch, seen):
    """run_matcher as train_step calls it, keeping its result with the gradients of conf_scores_*."""
    from e2e_multi_view_matching_b200 import training
    orig = training.run_matcher

    def spy(opt, data, matcher):
        losses, result = orig(opt, data, matcher)
        for k, v in result.items():
            if k.startswith('conf_scores_'):
                v.retain_grad()
        seen.update(result)
        return losses, result
    monkeypatch.setattr(training, 'run_matcher', spy)


@pytest.mark.parametrize('name', CASES)
def test_stage2_train_step_vs_reference(name, monkeypatch):
    from e2e_multi_view_matching_b200 import training
    _patch(monkeypatch)
    z, case, model, data, opt = _setup(name)
    seen = {}
    _spy_run_matcher(monkeypatch, seen)
    n_pairs = case['views'] * (case['views'] - 1) // 2
    loss, parts = training.train_step(opt, data, model, _optimizer(model), n_pairs, pose_match_ratio=case['ratio'])
    assert bool(parts.pop('finite_gradients'))
    assert abs(float(loss) - float(z['loss_f64'])) <= 4 * abs(float(z['loss_f32']) - float(z['loss_f64'])) + 1e-5 * abs(float(z['loss_f64']))
    for k, v in parts.items():
        r64, r32 = float(z['part__%s_f64' % k]), float(z['part__%s_f32' % k])
        assert abs(float(v) - r64) <= 4 * abs(r32 - r64) + 1e-5 * abs(r64) + 1e-7, (k, float(v), r64, r32)
    for k in [k for k in z.files if k.startswith('match__')]:
        assert np.array_equal(seen[k[len('match__'):]].numpy(), z[k]), k
    for k in [k for k in z.files if k.startswith('gconf__')]:
        pair = k[len('gconf__'):]
        got = seen['conf_scores_' + pair].grad.double().numpy()
        err = float(np.abs(got - z[k]).max())
        assert err <= 3 * float(z['gconf_noise__' + pair]) + 1e-5 * float(np.abs(z[k]).max()), (pair, err)
    state = model.state_dict()
    for k in [k for k in z.files if k.startswith('stat_f64__')]:
        s = k[len('stat_f64__'):]
        assert np.abs(state[s].double().numpy() - z[k]).max() <= 3 * float(z['stat_noise__' + s]) + 1e-6, s
    worst = check_gradients(model, z, tol_noise=3.0, tol_rel=2e-5, what=name)
    assert all(p.grad is not None for n, p in model.named_parameters() if n.startswith('conf_mlp'))
    print(name, 'worst gradient error / tolerance: %.3f at %s' % worst)


def test_conf_grad_off_keeps_conf_scores_without_graph(monkeypatch):
    """A bare model(data) with full_output keeps today's behaviour; conf_grad=True makes conf_scores differentiable."""
    _patch(monkeypatch)
    z, case, model, data, opt = _setup('mv3_r05')
    model.config['full_output'] = True
    res = model(data)
    assert not res['conf_scores_0_1'].requires_grad
    model.config['conf_grad'] = True
    res = model(data)
    assert res['conf_scores_0_1'].requires_grad and not res['matching_scores0_0_1'].requires_grad


def test_stage2_forward_runs_the_head_once_over_every_pair(monkeypatch):
    """The stage-2 forward of a 3-view tuple extracts the matches of its 3 pairs in one call and runs each of the
    confidence head's 4 BatchNorms once over the rows of every pair."""
    from e2e_multi_view_matching_b200 import ops
    _patch(monkeypatch)
    z, case, model, data, opt = _setup('mv3_r05')
    model.config.update(full_output=True, conf_grad=True)
    head_stats = {id(m.running_mean) for m in model.conf_mlp.modules() if isinstance(m, torch.nn.BatchNorm1d)}
    calls = {'extract_matches': 0, 'head_batchnorm_train': 0}
    extract, bn = ops.extract_matches, ops.batchnorm_train

    def counted_extract(*a, **k):
        calls['extract_matches'] += 1
        return extract(*a, **k)

    def counted_bn(x, weight, bias, running_mean, *a, **k):
        calls['head_batchnorm_train'] += id(running_mean) in head_stats
        return bn(x, weight, bias, running_mean, *a, **k)
    monkeypatch.setattr(ops, 'extract_matches', counted_extract)
    monkeypatch.setattr(ops, 'batchnorm_train', counted_bn)
    res = model(data)
    assert all(res['conf_scores_' + k].requires_grad for k in ('0_1', '0_2', '1_2'))
    assert calls == {'extract_matches': 1, 'head_batchnorm_train': 4}


def test_loss_without_conf_scores_gives_stage1_gradients(monkeypatch):
    """conf_grad on, a loss on the couplings only: the confidence head's backward does not run, every gradient equals
    the conf_grad-off one bit for bit and conf_mlp.* get none."""
    _patch(monkeypatch)
    grads = []
    for cg in (False, True):
        z, case, model, data, opt = _setup('mv3_r05')
        model.config.update(full_output=True, conf_grad=cg)
        res = model(data)
        sum((res['scores_%s' % k] * (1 + torch.arange(res['scores_%s' % k].numel()).view_as(res['scores_%s' % k]) % 7)).sum()
            for k in ('0_1', '0_2', '1_2')).backward()
        grads.append({n: (p.grad.clone() if p.grad is not None else None) for n, p in model.named_parameters()})
    for n, g in grads[0].items():
        if g is None:
            assert grads[1][n] is None and n.startswith('conf_mlp'), n
        else:
            assert torch.equal(g, grads[1][n]), n


def test_get_parameters_and_optimiser_groups():
    from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher
    from e2e_multi_view_matching_b200.training import get_parameters
    m = MultiViewMatcher({'GNN_layers': ['self', 'cross']})
    names = [n for n, _ in m.named_parameters()]
    ids = {id(p): n for n, p in m.named_parameters()}
    assert [ids[id(p)] for p in get_parameters(m)] == names
    assert [ids[id(p)] for p in get_parameters(m, whitelist_key='conf_mlp')] == [n for n in names if 'conf_mlp' in n]
    assert [ids[id(p)] for p in get_parameters(m, blacklist_key='conf_mlp')] == [n for n in names if 'conf_mlp' not in n]
    assert get_parameters(m, whitelist_key='conf_mlp', blacklist_key='layers_c') == \
        [p for n, p in m.named_parameters() if 'conf_mlp' in n and 'layers_c' not in n]
    wrapped = torch.nn.DataParallel(m)              # the reference calls it on the wrapped matcher: 'module.' names
    assert len(get_parameters(wrapped, whitelist_key='conf_mlp')) == sum('conf_mlp' in n for n in names)


def test_has_finite_gradients():
    from e2e_multi_view_matching_b200.training import has_finite_gradients
    m = torch.nn.Sequential(torch.nn.Linear(3, 4), torch.nn.Linear(4, 2))
    assert has_finite_gradients(m)                  # no gradients at all
    m(torch.ones(1, 3)).sum().backward()
    assert has_finite_gradients(m)
    m[1].bias.grad = None                           # a parameter without a gradient is skipped
    assert has_finite_gradients(m)
    for bad in (float('nan'), float('inf'), -float('inf')):
        m[0].weight.grad[1, 2] = bad
        assert not has_finite_gradients(m)
        m[0].weight.grad[1, 2] = 0.0


def test_pose_match_ratio_ramp():
    """train.py:414-416 step by step: +2.5e-5 while below the final ratio, capped at 1."""
    from e2e_multi_view_matching_b200.training import next_pose_match_ratio
    r, ref = 0.0, 0.0
    for _ in range(5000):
        r = next_pose_match_ratio(r, 0.1)
        if ref < 0.1:
            ref += 2.5e-5
            ref = min(ref, 1.)
        assert r == ref
    assert abs(r - 0.1) < 3e-5 and next_pose_match_ratio(r, 0.1) == r
    assert next_pose_match_ratio(1.0 - 1e-6, 2.0) == 1.0 and next_pose_match_ratio(1.0, 2.0) == 1.0
    assert next_pose_match_ratio(0.3, 0.2) == 0.3


def test_nonfinite_gradient_skips_the_step(monkeypatch):
    """A NaN in one pair's conf_scores gradient: train_step reports finite_gradients False and leaves the parameters
    and the Adam state as they were; without it the step is applied."""
    from e2e_multi_view_matching_b200 import training
    _patch(monkeypatch)
    z, case, model, data, opt = _setup('mv3_r05')
    orig = training.run_matcher

    def poisoned(opt_, data_, matcher):
        losses, result = orig(opt_, data_, matcher)
        result['conf_scores_0_2'].register_hook(lambda g: g.index_fill(1, torch.tensor([3]), float('nan')))
        return losses, result
    optimizer = _optimizer(model, lr=1e-3)
    before = {n: p.detach().clone() for n, p in model.named_parameters()}
    monkeypatch.setattr(training, 'run_matcher', poisoned)
    _, parts = training.train_step(opt, dict(data), model, optimizer, 3, pose_match_ratio=0.5)
    assert not bool(parts['finite_gradients'])
    assert all(torch.equal(p, before[n]) for n, p in model.named_parameters())
    assert len(optimizer.state) == 0
    monkeypatch.setattr(training, 'run_matcher', orig)
    _, parts = training.train_step(opt, dict(data), model, optimizer, 3, pose_match_ratio=0.5)
    assert bool(parts['finite_gradients'])
    assert any(not torch.equal(p, before[n]) for n, p in model.named_parameters())
    assert len(optimizer.state) == len(before)


def _nan_rank_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from e2e_multi_view_matching_b200 import training
    torch.manual_seed(0)
    model = torch.nn.Linear(3, 2)

    class Opt:
        pose_loss = True
        rot_weight = trans_weight = 1.0

    def fake_run_matcher(opt, data, matcher):
        y = matcher(torch.ones(1, 3)).sum()
        if rank == 1:
            y = y * torch.tensor(float('nan'))        # this rank's gradient holds NaNs
        z = torch.zeros(1)
        return {'match_loss': y.reshape(1), 'rot_loss': z, 'transl_loss': z}, {}
    training.run_matcher = fake_run_matcher
    optimizer = torch.optim.Adam(model.parameters(), lr=1e-2)
    before = [p.detach().clone() for p in model.parameters()]
    _, parts = training.train_step(Opt(), {}, model, optimizer, 1, pose_match_ratio=0.0)
    skipped = not bool(parts['finite_gradients']) and all(torch.equal(p, b) for p, b in zip(model.parameters(), before))
    flags = [None] * world
    dist.all_gather_object(flags, skipped)
    if rank == 0:
        open(out, 'w').write(json.dumps(flags))
    dist.barrier()
    dist.destroy_process_group()


def test_nan_on_one_rank_skips_the_step_on_every_rank(tmp_path):
    import torch.multiprocessing as mp
    out = str(tmp_path / 'flags.json')
    mp.spawn(_nan_rank_worker, args=(2, 29547, out), nprocs=2, join=True)
    assert json.load(open(out)) == [True, True]


def test_conf_kernels_compile_without_spills():
    """csrc/conf_train.cu for sm_90a: every kernel without a stack frame or spills."""
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    nvcc = nvcc if os.path.exists(nvcc) else shutil.which('nvcc')
    if not nvcc:
        pytest.skip('nvcc not available')
    src = os.path.join(ROOT, 'e2e_multi_view_matching_b200', 'csrc', 'conf_train.cu')
    r = subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xptxas', '-v',
                        '-c', src, '-o', os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', r.stderr)
    assert len(props) >= 5, r.stderr
    assert all(p == ('0', '0', '0') for p in props), r.stderr
