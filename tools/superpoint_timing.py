"""GPU time of SuperPoint at the MegaDepth / YFCC100M pair-evaluation sizes (longer side 1600, aspect kept: eval_pairs.py
resizes that way) and of the whole pair chain, with CUDA events after warm-up:
  - SuperPoint per image (dense network + NMS, and the full forward with top-2048 keypoints) at 1600 x 1066 and
    1600 x 1200 (width x height);
  - the pair chain: SuperPoint on a landscape 1600 x 1066 and a portrait 1066 x 1600 image, the 18-layer pairwise
    matcher at 2048 keypoints per view and the two-view pose (`w8pt_ba`), with each stage timed on its own as well.
Seeded weights and images (synthetic.make_superpoint_state_dict / make_image / make_state_dict).  Writes a JSON record
with the card name and power limit read in the same run.

    python tools/superpoint_timing.py [--out profiles/superpoint_h100.json] [--reps 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher  # noqa: E402
from e2e_multi_view_matching_b200.models.superpoint import SuperPoint  # noqa: E402
from e2e_multi_view_matching_b200.pipeline import PairPipeline  # noqa: E402
from e2e_multi_view_matching_b200.synthetic import make_image, make_state_dict, make_superpoint_state_dict  # noqa: E402


def _time(fn, reps, warmup):
    """-> (median ms, min ms) of fn() over `reps` event-timed calls after `warmup` untimed ones."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms)), float(np.min(ms))


def _superpoint(max_keypoints):
    sp = SuperPoint({'max_keypoints': max_keypoints}).eval()
    sp.load_state_dict({k: torch.from_numpy(v) for k, v in make_superpoint_state_dict(1).items()}, strict=True)
    return sp.cuda()


def _K(w, h, f):
    K = torch.tensor([[f, 0, (w - 1) / 2], [0, f, (h - 1) / 2], [0, 0, 1.0]], dtype=torch.float32)
    return K[None].cuda()


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'superpoint_h100.json'))
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit('superpoint_timing needs a CUDA device')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    rec = {'device': torch.cuda.get_device_name(0), 'nvidia_smi_name_power_limit_max_sm_clock': q.stdout.strip(),
           'reps': args.reps, 'warmup': args.warmup, 'superpoint': [], 'pair_chain': {}}
    sp = _superpoint(2048)
    with torch.no_grad():
        for w, h in ((1600, 1066), (1600, 1200)):
            img = torch.from_numpy(make_image(11, h, w)).cuda()
            dense = _time(lambda: sp.dense(img), args.reps, args.warmup)
            full = _time(lambda: sp({'image': [img]}), args.reps, args.warmup)
            n = int(sp({'image': [img]})['keypoints'][0].shape[0])
            # multiply-adds of the convolutions (3x3 at full / half / quarter / eighth resolution, 1x1 heads)
            macs = (h * w * 9 * (1 * 64 + 64 * 64) + (h // 2) * (w // 2) * 9 * 2 * 64 * 64
                    + (h // 4) * (w // 4) * 9 * (64 * 128 + 128 * 128)
                    + (h // 8) * (w // 8) * (9 * (2 * 128 * 128 + 2 * 128 * 256) + 256 * 65 + 256 * 256))
            rec['superpoint'].append({'width': w, 'height': h, 'keypoints': n, 'dense_ms_median': dense[0],
                                      'dense_ms_min': dense[1], 'forward_top2048_ms_median': full[0],
                                      'forward_top2048_ms_min': full[1], 'conv_gflop': 2 * macs / 1e9,
                                      'dense_fp32_tflops_achieved': 2 * macs / (dense[0] * 1e-3) / 1e12})
            print(rec['superpoint'][-1])

        layers = ['self', 'cross'] * 9
        matcher = MultiViewMatcher({'multi_frame_matching': False, 'GNN_layers': layers}).eval()
        matcher.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in
                                 make_state_dict(len(layers), seed=0, final_proj_gain=12.0).items()})
        pipe = PairPipeline(matcher.cuda(), 'w8pt_ba')
        sizes = [(1600, 1066), (1066, 1600)]
        imgs = [torch.from_numpy(make_image(12 + i, h, w)).cuda() for i, (w, h) in enumerate(sizes)]
        intr = {'intr%d' % i: _K(w, h, 1200.0) for i, (w, h) in enumerate(sizes)}

        def features():
            data = {'ids': [0, 1], **intr}
            for i, img in enumerate(imgs):          # one image per call (merge=False): the two sizes differ
                p = sp({'image': [img]})
                data.update({'keypoints%d' % i: p['keypoints'][0][None], 'scores%d' % i: p['scores'][0][None],
                             'descriptors%d' % i: p['descriptors'][0][None], 'image%d' % i: img})
            return data

        data = features()
        counts = [int(data['keypoints%d' % i].shape[1]) for i in range(2)]
        chain = _time(lambda: pipe(features()), args.reps, args.warmup)
        sp_only = _time(features, args.reps, args.warmup)
        match_pose = _time(lambda: pipe(data), args.reps, args.warmup)
        rec['pair_chain'] = {'sizes_wh': sizes, 'keypoints': counts, 'matcher_layers': len(layers), 'pose': 'w8pt_ba',
                             'chain_ms_median': chain[0], 'chain_ms_min': chain[1],
                             'two_superpoints_ms_median': sp_only[0], 'matcher_and_pose_ms_median': match_pose[0]}
        print(rec['pair_chain'])
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(rec, f, indent=2)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
