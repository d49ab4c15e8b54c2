"""Step time of training stage 1 (match loss) and stage 2 (--pose_loss) at the cfg5 shape: 8 five-view tuples x 400
keypoints, 28 GNN layers, synthetic scenes (synthetic.make_scene_tuple_inputs, ground truth from the landmark ids).
The two steps alternate in one process.  The stage-2 step is split into
  * the confidence head's backward (models/train_forward._conf_backward),
  * the weighted eight-point's forward and backward (mvm_w8pt / mvm_w8pt_backward, all 10 pairs),
  * the extra forward work of full_output (match extraction and the confidence head's forward: a train-mode forward
    with full_output minus one without, timed on their own),
  * the rest,
each by CUDA events around the calls, and each step into run_matcher (forward and losses), the finite-gradient check
(stage 2) and the rest (backward, all-reduce, optimiser step).  Each repetition also times a stage-2 step with the read-back of the match
indices' range in mvm_conf_gather_backward switched off (mvm_debug_set_conf_i0_check(0)).  Writes
profiles/pose_train_h100.json (or --out) with the card name and its power limit.

    python tools/pose_train_timing.py [--reps 8] [--out profiles/pose_train_h100.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class _Timer:
    def __init__(self):
        self.pairs = {}

    def wrap(self, name, fn):
        def inner(*a, **k):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out = fn(*a, **k)
            e.record()
            self.pairs.setdefault(name, []).append((s, e))
            return out
        return inner

    def collect(self):
        torch.cuda.synchronize()
        out = {k: sum(s.elapsed_time(e) for s, e in v) for k, v in self.pairs.items()}
        self.pairs = {}
        return out


def _power_limit():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:      # noqa: BLE001
        return 'unknown (%s)' % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=8)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'pose_train_h100.json'))
    args = ap.parse_args()
    from e2e_multi_view_matching_b200 import training, _lib
    from e2e_multi_view_matching_b200.models import train_forward as TF
    from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher
    from e2e_multi_view_matching_b200.pose_optimization.two_view import estimate_relative_pose as erp
    from e2e_multi_view_matching_b200.synthetic import landmark_gt_matches, make_scene_tuple_inputs, make_state_dict
    T, N, B, L = 5, 400, 8, 28
    d = make_scene_tuple_inputs(11, n_views=T, n_kpts=N, batch=B)
    for b in range(T):
        for a in range(b):
            idx, w = landmark_gt_matches(d['landmark%d' % a], d['landmark%d' % b])
            d['gt_indices_%d_%d' % (a, b)], d['gt_weights_%d_%d' % (a, b)] = idx, w
    data = {k: (torch.from_numpy(v).cuda() if isinstance(v, np.ndarray) else v) for k, v in d.items()}
    sd = make_state_dict(L, seed=3, final_proj_gain=2.0, conf_head='score')
    model = MultiViewMatcher({'GNN_layers': ['self', 'cross'] * (L // 2), 'conf_mlp': True})
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    model = model.cuda().train()
    optimizer = torch.optim.Adam(training.get_parameters(model, blacklist_key='conf_mlp'), lr=1e-6)
    optimizer.add_param_group({'params': training.get_parameters(model, whitelist_key='conf_mlp'), 'lr': 1e-6})
    opt1 = argparse.Namespace(pose_loss=False)
    opt2 = argparse.Namespace(pose_loss=True, rot_weight=726.0, trans_weight=244.0)
    n_pairs = T * (T - 1) // 2
    lib = _lib.lib()
    tm = _Timer()
    TF._conf_backward = tm.wrap('conf_head_backward', TF._conf_backward)
    erp._run_w8pt = tm.wrap('w8pt_forward', erp._run_w8pt)
    erp._W8ptFunction.backward = staticmethod(tm.wrap('w8pt_backward', erp._W8ptFunction.backward))
    training.run_matcher = tm.wrap('run_matcher', training.run_matcher)
    training._all_finite = tm.wrap('finite_check', training._all_finite)

    def step(opt):
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        _, parts = training.train_step(opt, dict(data), model, optimizer, n_pairs, pose_match_ratio=0.5)
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e), parts

    def fwd(full):
        model.config.update(full_output=full, conf_grad=False)
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        with torch.no_grad():
            model(dict(data))
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e)

    rows = []
    for r in range(args.warmup + args.reps):
        t1, _ = step(opt1)
        split1 = tm.collect()
        t2, parts = step(opt2)
        split = tm.collect()
        f_full, f_plain = fwd(True), fwd(False)
        # the same stage-2 step without the read-back of the match indices' range in mvm_conf_gather_backward (the
        # indices come from mvm_extract_matches, so they are in range): what that stream synchronisation costs
        lib.mvm_debug_set_conf_i0_check(0)
        t2_nocheck, _ = step(opt2)
        lib.mvm_debug_set_conf_i0_check(1)
        tm.collect()
        if r >= args.warmup:
            rows.append(dict(stage1_ms=t1, stage2_ms=t2, stage2_without_i0_readback_ms=t2_nocheck,
                             finite=bool(parts['finite_gradients']),
                             stage1_forward_and_losses_ms=split1['run_matcher'],
                             stage2_forward_and_losses_ms=split['run_matcher'],
                             stage2_finite_check_ms=split['finite_check'],
                             conf_head_backward_ms=split.get('conf_head_backward', 0.0),
                             w8pt_forward_ms=split.get('w8pt_forward', 0.0), w8pt_backward_ms=split.get('w8pt_backward', 0.0),
                             full_output_forward_extra_ms=f_full - f_plain))
    med = {k: float(np.median([r_[k] for r_ in rows])) for k in rows[0] if k != 'finite'}
    med['stage2_rest_ms'] = med['stage2_ms'] - med['conf_head_backward_ms'] - med['w8pt_forward_ms'] - \
        med['w8pt_backward_ms'] - med['full_output_forward_extra_ms']
    # backward + all-reduce + optimiser step: the step minus run_matcher (forward and losses) and the finite check
    med['stage1_backward_and_step_ms'] = med['stage1_ms'] - med['stage1_forward_and_losses_ms']
    med['stage2_backward_and_step_ms'] = med['stage2_ms'] - med['stage2_forward_and_losses_ms'] - med['stage2_finite_check_ms']
    rep = {'what': 'train_step at the cfg5 shape (%d tuples x %d views x %d keypoints, %d layers), stage 1 and stage 2 '
                   '(pose_match_ratio 0.5) alternated in one process; medians over %d repetitions' % (B, T, N, L, args.reps),
           'device': torch.cuda.get_device_name(0), 'power_limit': _power_limit(),
           'date': time.strftime('%Y-%m-%d'), 'median': med, 'runs': rows}
    print(json.dumps(rep['median'], indent=1))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump(rep, open(args.out, 'w'), indent=1)


if __name__ == '__main__':
    main()
