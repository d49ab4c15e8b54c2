"""Golden losses and gradients for STAGE 2 of the training step (BASELINE cfg5, train.py:405-426 with --pose_loss): the
unmodified reference MultiViewMatcher in .train() with conf_mlp and full_output, wrapped in torch.nn.DataParallel
(on a host without CUDA it calls the module directly) so that the reference's OWN helpers.run_matcher (helpers.py:243-260,
pose_loss=True: match loss, run_weighted_8_point with choose_closest, rotation / translation errors) finds `.module`;
combine_losses (train.py:36-40, restated as e2e_multi_view_matching_b200.training.combine_losses) and loss.backward(),
in fp32 and (yardstick) fp64 -> tests/golden/train_pose_*.npz:
  * the loss parts (match / rot / transl, after combine_losses, and the total);
  * per parameter, conf_mlp.* included, the gradient in the layout of make_train_backward_golden (fp64 run stored as
    float32 in full up to 1024 elements, else 1024 seeded samples; its L2 norm; the largest deviation of the fp32 run
    from the fp64 run over the whole gradient = `noise`);
  * the gradient at every conf_scores_* (retain_grad), the matches, the confidence head's running statistics;
  * per pair and item, the choose_closest candidate errors of the fp64 run and the margin between the best and the
    second best.
The generator asserts that the fp32 and fp64 runs agree on every match and every chosen candidate.
The two-view pose files run through oracle/ref_shim.py.  TEST INFRASTRUCTURE ONLY (needs the reference sources); the
tests rebuild inputs and weights from the seeds."""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402
from oracle.make_train_backward_golden import sample_index  # noqa: E402
from oracle.make_validation_golden import gt_from_landmarks  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden')
# ScanNet rot / trans weights of train.py:218-225: 1597 / 270 for pairs, 726 / 244 for 5-tuples (the reference defines
# none for 3 views: the 3-view case takes the 5-tuple weights).  The seeds and final-projection gains are chosen so that
# the fp32 and fp64 runs agree on every match and every choose_closest candidate (a larger gain saturates the couplings:
# two rows then share a column at exactly log(1/2) and its argmax is a tie)
CASES = []
for ratio in (0.5, 1.0):
    tag = '%02d' % int(round(ratio * 10))
    CASES += [dict(name='mv3_r' + tag, multi=True, views=3, kpts=64, batch=2, layers=['self', 'cross'] * 2, wseed=81,
                   iseed=91, gain=1.0, ratio=ratio, rot_weight=726.0, trans_weight=244.0),
              dict(name='mv5_r' + tag, multi=True, views=5, kpts=40, batch=2, layers=['self', 'cross'], wseed=82,
                   iseed=92, gain=2.0, ratio=ratio, rot_weight=726.0, trans_weight=244.0),
              dict(name='pair_r' + tag, multi=False, views=2, kpts=80, batch=2, layers=['self', 'cross'] * 2, wseed=83,
                   iseed=93, gain=1.0, ratio=ratio, rot_weight=1597.0, trans_weight=270.0)]
CONF_STATS = ['conf_mlp.layers_f.1.running_mean', 'conf_mlp.layers_f.1.running_var', 'conf_mlp.layers_f.4.running_mean',
              'conf_mlp.layers_f.4.running_var', 'conf_mlp.layers_c.1.running_mean', 'conf_mlp.layers_c.1.running_var',
              'conf_mlp.layers_c.4.running_mean', 'conf_mlp.layers_c.4.running_var']


def build(case):
    """-> (data dict of numpy arrays with ground-truth matches, state dict)."""
    from e2e_multi_view_matching_b200.synthetic import make_scene_tuple_inputs, make_state_dict
    data = make_scene_tuple_inputs(case['iseed'], n_views=case['views'], n_kpts=case['kpts'], batch=case['batch'])
    for b_ in range(case['views']):
        for a_ in range(b_):
            pairs = [gt_from_landmarks(data['landmark%d' % a_][b], data['landmark%d' % b_][b]) for b in range(case['batch'])]
            data['gt_indices_%d_%d' % (a_, b_)] = np.stack([p[0] for p in pairs])
            data['gt_weights_%d_%d' % (a_, b_)] = np.stack([p[1] for p in pairs])
    sd = make_state_dict(len(case['layers']), seed=case['wseed'], final_proj_gain=case['gain'], conf_head='score')
    return data, sd


def opt_of(case):
    return argparse.Namespace(pose_loss=True, rot_weight=case['rot_weight'], trans_weight=case['trans_weight'])


def n_pairs(case):
    return case['views'] * (case['views'] - 1) // 2


def candidate_errors(erp, cpe, data, result, id0, id1):
    """The four choose_closest candidates' rot + transl errors [B, 4] of the pair, by the reference's own steps
    (estimate_relative_pose.py:84-106)."""
    k0, k1, i0, i1, conf = erp.get_kpts(data, result, id0, id1)
    conf = conf.detach()
    w = conf / (conf.sum(dim=1, keepdim=True) + 1e-6)
    Fs = erp.find_fundamental(erp.normalize(k0, i0), erp.normalize(k1, i1), w.squeeze(-1))
    Rs, ts = erp.motion_from_essential(Fs)
    target = torch.linalg.inv(data['pose%d' % id1]) @ data['pose%d' % id0]
    errs = []
    for R, t in zip(Rs.permute(1, 0, 2, 3), ts.permute(1, 0, 2, 3)):
        P = torch.eye(4, dtype=R.dtype).unsqueeze(0).repeat(R.shape[0], 1, 1)
        P[:, :3, :3], P[:, :3, 3] = R, t.squeeze(-1)
        errs.append(cpe.compute_rotation_error(P, target, reduce=False) + cpe.compute_translation_error_as_angle(P, target, reduce=False))
    return torch.stack(errs, 1).detach().numpy().astype(np.float64)


def run_reference(case, dtype):
    # the reference's pose files build their identity transforms and zero losses in the default dtype: the fp64 run
    # sets it, as oracle/make_w8pt_grad_golden.py does
    old = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        return _run_reference(case, dtype)
    finally:
        torch.set_default_dtype(old)


def _run_reference(case, dtype):
    import helpers
    import importlib
    from models.models.multi_view_matcher import MultiViewMatcher
    from e2e_multi_view_matching_b200.training import combine_losses
    erp, _ = ref_shim.load()
    cpe = importlib.import_module('pose_optimization.two_view.compute_pose_error')
    data_np, sd = build(case)
    torch.manual_seed(0)
    model = MultiViewMatcher({'multi_frame_matching': case['multi'], 'GNN_layers': case['layers'], 'conf_mlp': True,
                              'full_output': True})
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
    model = model.to(dtype).train()
    matcher = torch.nn.DataParallel(model)
    data = {k: (torch.from_numpy(v).to(dtype) if isinstance(v, np.ndarray) and v.dtype.kind == 'f' else
                (torch.from_numpy(v) if isinstance(v, np.ndarray) else v)) for k, v in data_np.items()}
    losses, result = helpers.run_matcher(opt_of(case), data, matcher)
    conf_keys = sorted(k for k in result if k.startswith('conf_scores_'))
    for k in conf_keys:
        result[k].retain_grad()
    loss, parts = combine_losses(losses, n_pairs(case), case['ratio'], case['rot_weight'], case['trans_weight'])
    loss.backward()
    out = {'loss': float(loss.item())}
    for k, v in parts.items():
        out['part__' + k] = float(v.item())
    for k in conf_keys:
        out['gconf__' + k[len('conf_scores_'):]] = result[k].grad.detach().numpy().astype(np.float64)
    for k in result:
        if k.startswith('matches'):
            out['match__' + k] = result[k].numpy().copy()
    for n, p in model.named_parameters():
        if p.grad is not None:
            out['grad__' + n] = p.grad.detach().numpy().reshape(-1).astype(np.float64)
    st = model.state_dict()
    for k in CONF_STATS:
        out['stat__' + k] = st[k].detach().numpy().astype(np.float64)
    with torch.no_grad():
        for b_ in range(case['views']):
            for a_ in range(b_):
                out['cand__%d_%d' % (a_, b_)] = candidate_errors(erp, cpe, data, result, a_, b_)
    return out


def main():
    ref_shim.load()
    import helpers
    assert helpers.__file__.startswith(ref_shim.REF)
    torch.set_num_threads(8)
    report = {}
    for case in CASES:
        r32, r64 = run_reference(case, torch.float32), run_reference(case, torch.float64)
        small = {'meta': json.dumps(case), 'loss_f64': np.float64(r64['loss']), 'loss_f32': np.float64(r32['loss'])}
        for k in [k for k in r64 if k.startswith('part__')]:
            small[k + '_f64'], small[k + '_f32'] = np.float64(r64[k]), np.float64(r32[k])
        for k in [k for k in r64 if k.startswith('match__')]:
            assert np.array_equal(r32[k], r64[k]), (case['name'], k, int((r32[k] != r64[k]).sum()))
            small[k] = r64[k]
        margins = []
        for k in [k for k in r64 if k.startswith('cand__')]:
            c32, c64 = r32[k], r64[k]
            assert np.array_equal(c32.argmin(1), c64.argmin(1)), (case['name'], k)
            srt = np.sort(c64, 1)
            small['margin__' + k[len('cand__'):]] = srt[:, 1] - srt[:, 0]
            margins.append(float((srt[:, 1] - srt[:, 0]).min()))
            small[k] = c64
        for k in [k for k in r64 if k.startswith('gconf__')]:
            small[k] = r64[k].astype(np.float32)
            small['gconf_noise__' + k[len('gconf__'):]] = np.float64(np.abs(r32[k] - r64[k]).max())
        for k in [k for k in r64 if k.startswith('stat__')]:
            small['stat_f64__' + k[len('stat__'):]] = r64[k].astype(np.float32)
            small['stat_noise__' + k[len('stat__'):]] = np.float64(np.abs(r32[k] - r64[k]).max())
        rel = {}
        names = [k[len('grad__'):] for k in r64 if k.startswith('grad__')]
        for k in names:
            g64, g32 = r64['grad__' + k], r32['grad__' + k]
            assert np.isfinite(g64).all() and np.isfinite(g32).all(), (case['name'], k)
            small['grad__' + k] = g64[sample_index(k, g64.size)].astype(np.float32)
            small['noise__' + k] = np.float64(np.abs(g32 - g64).max())
            small['norm__' + k] = np.float64(np.linalg.norm(g64))
            rel[k] = float(small['noise__' + k] / max(np.abs(g64).max(), 1e-30))
        worst = max(rel, key=rel.get)
        n_match = {k[len('match__'):]: [int(x) for x in (r64[k] >= 0).sum(1)] for k in r64 if k.startswith('match__')}
        report[case['name']] = {'loss_f64': r64['loss'], 'loss_f32': r32['loss'],
                                'parts_f64': {k[6:]: r64[k] for k in r64 if k.startswith('part__')},
                                'n_params_with_grad': len(names),
                                'conf_params_with_grad': sum(1 for k in names if k.startswith('conf_mlp')),
                                'max_rel_ref32_vs_ref64': rel[worst], 'at': worst,
                                'median_rel_ref32_vs_ref64': float(np.median(list(rel.values()))),
                                'min_candidate_margin_rad': min(margins), 'matches_per_item': n_match}
        print(case['name'], json.dumps(report[case['name']]))
        np.savez_compressed(os.path.join(OUT, 'train_pose_%s.npz' % case['name']), **small)
    json.dump(report, open(os.path.join(OUT, 'train_pose_report.json'), 'w'), indent=1)


if __name__ == '__main__':
    main()
