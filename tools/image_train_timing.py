"""GPU time of the image-in training step at the cfg5 shape (train.py with --dataset scannet: 8 tuples x 5 views of
480 x 640, SuperPoint with max_keypoints 400, keypoint_threshold 0.001, nms_radius 4, remove_borders 12,
fill_with_random_keypoints; 28-layer multi-view matcher, stage 1 match loss, Adam), with CUDA events after warm-up:
  - training.train_step from images (run_super_point inside the step) against the same step from precomputed keypoints,
    alternated call by call;
  - SuperPoint on the 40 images through forward (per-image selection on the host side) against forward_batch;
  - mvm_superpoint_select alone on 40 maps of 480 x 640 and on 1 and 40 maps of 1064 x 1600.
Seeded weights, rendered synthetic tuples (synthetic.render_tuple_images) with constant-depth maps for the ground
truth.  Writes a JSON record with the card name and power limit read in the same run.

    python tools/image_train_timing.py [--out profiles/image_train_h100.json] [--reps 10] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from e2e_multi_view_matching_b200 import training  # noqa: E402
from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher  # noqa: E402
from e2e_multi_view_matching_b200.models.superpoint import SuperPoint  # noqa: E402
from e2e_multi_view_matching_b200.synthetic import (make_scene_tuple_inputs, make_state_dict,  # noqa: E402
                                                    make_superpoint_state_dict, render_tuple_images)

T, B, H, W = 5, 8, 480, 640
SP_CFG = {'max_keypoints': 400, 'keypoint_threshold': 0.001, 'nms_radius': 4, 'remove_borders': 12,
          'fill_with_random_keypoints': True}
LAYERS = (['self'] + ['cross'] * 3) * 7


def _event_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def _alternate(fns, reps, warmup):
    """-> per fn (median ms, min ms), the fns called in turn so that both see the same machine state."""
    for _ in range(warmup):
        for fn in fns:
            fn()
    torch.cuda.synchronize()
    ms = [[] for _ in fns]
    for _ in range(reps):
        for i, fn in enumerate(fns):
            ms[i].append(_event_ms(fn))
    return [(float(np.median(m)), float(np.min(m))) for m in ms]


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'image_train_h100.json'))
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit('image_train_timing needs a CUDA device')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    rec = {'device': torch.cuda.get_device_name(0), 'nvidia_smi_name_power_limit_max_sm_clock': q.stdout.strip(),
           'reps': args.reps, 'warmup': args.warmup, 'tuples': B, 'views': T, 'height': H, 'width': W,
           'superpoint_config': SP_CFG, 'matcher_layers': len(LAYERS)}

    sp = SuperPoint(SP_CFG).eval()
    sp.load_state_dict({k: torch.from_numpy(v) for k, v in make_superpoint_state_dict(1).items()})
    sp = sp.cuda()
    model = MultiViewMatcher({'GNN_layers': LAYERS, 'multi_frame_matching': True, 'conf_mlp': False, 'full_output': False})
    sd = make_state_dict(len(LAYERS), seed=0, final_proj_gain=12.0)
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items() if not k.startswith('conf_mlp')})
    model = model.cuda().train()
    optimizer = torch.optim.Adam(model.parameters(), lr=1e-4)
    opt = types.SimpleNamespace(pose_loss=False, batch_size=B, match_reproj_err=5.0, unmatch_reproj_err=15.0,
                                rot_weight=0.0, trans_weight=0.0)

    d = render_tuple_images(make_scene_tuple_inputs(5000, T, 400, batch=B, width=W, height=H, noise_px=0.0), seed=5000)
    images = {'ids': list(range(T))}
    for i in range(T):
        K4 = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
        K4[:, :3, :3] = d['intr%d' % i]
        images['image%d' % i] = torch.from_numpy(d['image%d' % i]).cuda()
        images['depth%d' % i] = torch.full((B, H, W), 4.0, device='cuda')
        images['intr%d' % i] = torch.from_numpy(K4).cuda()
        images['pose%d' % i] = torch.from_numpy(d['pose%d' % i]).cuda()
    keypoints = dict(images)
    training.run_super_point(opt, keypoints, sp)
    n_pairs = T * (T - 1) // 2

    def step_images():
        return training.train_step(opt, dict(images), model, optimizer, n_pairs, super_point=sp)

    def step_keypoints():
        return training.train_step(opt, dict(keypoints), model, optimizer, n_pairs)

    (img_med, img_min), (kp_med, kp_min) = _alternate([step_images, step_keypoints], args.reps, args.warmup)
    rec['train_step'] = {'from_images_ms_median': img_med, 'from_images_ms_min': img_min,
                         'from_keypoints_ms_median': kp_med, 'from_keypoints_ms_min': kp_min,
                         'superpoint_share_of_image_step': (img_med - kp_med) / img_med}
    print(rec['train_step'])

    merged = torch.cat([images['image%d' % i] for i in range(T)], 0)
    with torch.no_grad():
        (f_med, f_min), (b_med, b_min), (d_med, d_min) = _alternate(
            [lambda: sp({'image': [merged]}), lambda: sp.forward_batch(merged), lambda: sp.dense(merged)],
            args.reps, args.warmup)
    rec['superpoint_40_images'] = {'forward_ms_median': f_med, 'forward_ms_min': f_min,
                                   'forward_batch_ms_median': b_med, 'forward_batch_ms_min': b_min,
                                   'dense_only_ms_median': d_med, 'dense_only_ms_min': d_min}
    print(rec['superpoint_40_images'])

    # the selection kernel alone (one CTA per image) on SuperPoint score maps: the cfg5 batch, and 1600-px maps at B = 1
    # and B = 40, where a single image's five passes over its map run on one SM
    from e2e_multi_view_matching_b200 import _lib
    from e2e_multi_view_matching_b200.synthetic import make_image
    lib = _lib.lib()
    rec['select_only'] = []
    with torch.no_grad():
        big = sp.dense(torch.from_numpy(make_image(7, 1066, 1600)).cuda())[0]
        small = sp.dense(merged)[0]
        for name, smap, k in (('40 x 480x640', small, 400), ('1 x 1064x1600', big, 2048),
                              ('40 x 1064x1600', big.expand(40, -1, -1).contiguous(), 2048)):
            Bm, Hs, Ws = smap.shape
            kp = torch.empty(Bm, k, 2, device='cuda')
            sc = torch.empty(Bm, k, device='cuda')
            cnt = torch.empty(Bm, dtype=torch.int32, device='cuda')

            def select():
                _lib.check(lib.mvm_superpoint_select(_lib.ptr(smap), Bm, Hs, Ws, SP_CFG['keypoint_threshold'],
                                                     SP_CFG['remove_borders'], k, _lib.ptr(kp), _lib.ptr(sc),
                                                     _lib.ptr(cnt), _lib.stream_ptr()), 'mvm_superpoint_select')
            (med, mn), = _alternate([select], max(args.reps, 20), args.warmup)
            rec['select_only'].append({'maps': name, 'max_keypoints': k, 'candidates_max': int(cnt.max()),
                                       'map_mb_per_image': Hs * Ws * 4 / 1e6, 'ms_median': med, 'ms_min': mn})
            print(rec['select_only'][-1])
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(rec, f, indent=2)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
