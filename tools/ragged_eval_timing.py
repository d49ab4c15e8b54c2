"""Image-in multi-view evaluation throughput: a loop of batch-of-one MultiViewPipeline calls (the reference's test
loader, batch_size=1) against ragged batches of 4 and 14 tuples (each view keeps its own SuperPoint count per tuple).
Rendered synthetic 5-view tuples (synthetic.render_tuple_images), SuperPoint with seeded weights at max_keypoints 1024
and 2048 (the MegaDepth setting, whose 2048-wide pairs take the multi-CTA Sinkhorn), the scannet-depth matcher with the
score-driven confidence head, w8pt + two-view BA + global BA.  Reports tuples/s (host clock around synchronised
batches), the library's per-stage device time (CUDA events, a separate pass) and the card name and power limit read in
the same run.

    python tools/ragged_eval_timing.py [--out profiles/ragged_eval_h100.json] [--n_tuples 56] [--warmup 1]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from e2e_multi_view_matching_b200 import _lib  # noqa: E402
from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher  # noqa: E402
from e2e_multi_view_matching_b200.models.superpoint import SuperPoint  # noqa: E402
from e2e_multi_view_matching_b200.pipeline import MultiViewPipeline  # noqa: E402
from e2e_multi_view_matching_b200.synthetic import (make_scene_tuple_inputs, make_state_dict,  # noqa: E402
                                                   make_superpoint_state_dict, render_tuple_images)

T = 5
LAYERS = (['self'] + ['cross'] * 3) * 7


def tuples(n, k_max):
    out = []
    for i in range(n):
        d = render_tuple_images(make_scene_tuple_inputs(1000 + i, T, k_max, batch=1, noise_px=0.0), seed=1000 + i)
        out.append({k: v for k, v in d.items() if not k.startswith(('keypoints', 'scores', 'descriptors'))})
    return out


def batch_of(parts):
    return {k: (torch.from_numpy(np.concatenate([p[k] for p in parts])).cuda() if isinstance(v, np.ndarray) else v)
            for k, v in parts[0].items()}


def run_all(pipe, batches):
    for d in batches:
        pipe.run_tuples(d)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default='profiles/ragged_eval_h100.json')
    ap.add_argument('--n_tuples', type=int, default=56)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    rec = {'device': torch.cuda.get_device_name(0), 'nvidia_smi_name_power_limit_max_sm_clock': q.stdout.strip(),
           'views': T, 'tuples': args.n_tuples, 'matcher_layers': len(LAYERS), 'reps': args.reps,
           'timing': 'host clock around each pass over all tuples, torch.cuda.synchronize at both ends; best of reps',
           'runs': []}
    sd = make_state_dict(len(LAYERS), seed=0, final_proj_gain=12.0, conf_head='score')
    matcher = MultiViewMatcher({'multi_frame_matching': True, 'GNN_layers': LAYERS}).eval()
    matcher.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    matcher = matcher.cuda()
    # With these seeded weights nearly every NMS survivor of a rendered image clears the usual 0.005 threshold (4000-5000
    # per image), which fills every view to max_keypoints.  These thresholds leave 800-1200 (1024) and 1700-2300 (2048)
    # keypoints per image, so the counts differ from view to view and tuple to tuple as they do on real images.
    for k_max, thresh in ((1024, 0.55), (2048, 0.42)):
        sp = SuperPoint({'max_keypoints': k_max, 'keypoint_threshold': thresh, 'nms_radius': 4,
                         'remove_borders': 4}).eval()
        sp.load_state_dict({k: torch.from_numpy(v) for k, v in make_superpoint_state_dict(0).items()})
        pipe = MultiViewPipeline(matcher, superpoint=sp.cuda())
        parts = tuples(args.n_tuples, k_max)
        for bs in (1, 4, 14):
            batches = [batch_of(parts[s:s + bs]) for s in range(0, args.n_tuples, bs)]
            with torch.no_grad():
                for _ in range(args.warmup):
                    run_all(pipe, batches)
                torch.cuda.synchronize()
                best = float('inf')
                for _ in range(args.reps):
                    t0 = time.perf_counter()
                    run_all(pipe, batches)
                    torch.cuda.synchronize()
                    best = min(best, time.perf_counter() - t0)
                _lib.lib().mvm_profile_enable(1)
                _lib.profile_collect()
                run_all(pipe, batches)
                torch.cuda.synchronize()
                stages = {k: round(v[0], 3) for k, v in _lib.profile_collect().items() if v[1]}
                _lib.lib().mvm_profile_enable(0)
                counts = sp.forward_batch(batches[0]['image0'])['counts'].tolist()
            run = {'max_keypoints': k_max, 'keypoint_threshold': thresh, 'batch': bs, 'seconds': round(best, 4),
                   'tuples_per_s': round(args.n_tuples / best, 2), 'stage_ms_per_pass': stages,
                   'superpoint_counts_view0_first_batch': counts}
            rec['runs'].append(run)
            print(json.dumps(run), flush=True)
        base = [r for r in rec['runs'] if r['max_keypoints'] == k_max and r['batch'] == 1][0]
        for r in rec['runs']:
            if r['max_keypoints'] == k_max:
                r['speedup_vs_batch_1'] = round(base['seconds'] / r['seconds'], 2)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == '__main__':
    main()
