"""Multi-view benchmark driver with the reference's flow (eval_multi_view.py:89-165): matcher on
fixed 5-tuples, then eval_bundle_adjust, then pose / translation / rotation AUC@5/10/20 written as
JSON (eval_multi_view.py:70-87).  The reference reads ScanNet/Matterport/MegaDepth tuples and a
trained checkpoint; neither exists offline, so tuples are synthetic scenes
(synthetic.make_scene_tuple_inputs) and weights are either a reference checkpoint given with --ckpt
(helpers.load_ckpt format: {'model': state_dict with 'module.' prefix}) or seeded random weights.

With --images the tuples are image-in, as in the reference: the scene is rendered into every view
(synthetic.render_tuple_images) and SuperPoint (seeded weights, or a superpoint_v1.pth-style state dict given with
--superpoint_weights; max_keypoints, keypoint_threshold, nms_radius and remove_borders as eval_multi_view.py:125-141)
finds the keypoints on the device before the matcher (run_super_point, eval_multi_view.py:157), one tuple per batch as
the reference's test loader (batch_size=1), so every view keeps its own keypoint count.  --image_batch N runs N tuples
per batch instead: their views keep their own counts as a ragged batch (MultiViewPipeline.run_tuples).  Without --images, the
matcher gets the synthetic keypoints directly.

    python -m e2e_multi_view_matching_b200.eval_multi_view --n_tuples 16 --out result.json
    python -m e2e_multi_view_matching_b200.eval_multi_view --images --n_tuples 16 --out result.json
"""
import argparse
import json

import numpy as np
import torch

from .models.multi_view_matcher import MultiViewMatcher
from .models.superpoint import SuperPoint
from .pipeline import MultiViewPipeline, pose_auc
from .synthetic import make_state_dict, make_scene_tuple_inputs, make_superpoint_state_dict, render_tuple_images


def write_result(pose_errors, file):
    thresholds = [5, 10, 20]
    metrics = dict()
    for name, errs in (('pose', pose_errors[0]), ('transl', pose_errors[1]), ('rot', pose_errors[2])):
        for thresh, auc in zip(thresholds, pose_auc(errs, thresholds)):
            metrics["{}_AUC@{}deg".format(name, thresh)] = auc * 100.0
    if file:
        with open(file, 'w') as tf:
            json.dump(metrics, tf, indent=4)
    return metrics


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--n_tuples', type=int, default=8)
    ap.add_argument('--tuple_size', type=int, default=5)
    ap.add_argument('--max_keypoints', type=int, default=1024)
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--dataset', default='scannet', choices=['scannet', 'matterport', 'megadepth'])
    ap.add_argument('--ckpt', default=None)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--math_mode', type=int, default=3)
    ap.add_argument('--out', default=None)
    ap.add_argument('--images', action='store_true', help='render the tuples and run SuperPoint on them')
    ap.add_argument('--image_batch', type=int, default=1,
                    help='tuples per batch with --images (1: the reference test loader; more: ragged batches)')
    ap.add_argument('--superpoint_weights', default=None)
    ap.add_argument('--keypoint_threshold', type=float, default=0.005)
    ap.add_argument('--nms_radius', type=int, default=4)
    ap.add_argument('--remove_borders', type=int, default=4)
    opt = ap.parse_args(argv)
    import e2e_multi_view_matching_b200 as pkg
    pkg.set_math_mode(opt.math_mode)
    # GNN depth per dataset (train.py:262-268)
    layers = ['self', 'cross'] * 9 if opt.dataset == 'megadepth' else (['self'] + ['cross'] * 3) * 7
    matcher = MultiViewMatcher({'multi_frame_matching': True, 'GNN_layers': layers}).eval()
    if opt.ckpt:
        sd = torch.load(opt.ckpt, map_location='cpu')
        sd = sd.get('model', sd)
        # the reference loads with strict=False (helpers.py:48), which hides key mismatches: load the same way,
        # but say what did not line up
        missing, unexpected = matcher.load_state_dict({k[7:] if k.startswith('module.') else k: v for k, v in sd.items()},
                                                      strict=False)
        if missing or unexpected:
            import logging
            logging.warning('checkpoint keys: %d missing (%s...), %d unexpected (%s...)', len(missing),
                            ', '.join(missing[:3]), len(unexpected), ', '.join(unexpected[:3]))
    else:
        sd = make_state_dict(len(layers), seed=opt.seed, final_proj_gain=12.0, conf_head='score')
        matcher.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    matcher = matcher.cuda()
    superpoint = None
    if opt.images:
        superpoint = SuperPoint({'max_keypoints': opt.max_keypoints, 'keypoint_threshold': opt.keypoint_threshold,
                                 'nms_radius': opt.nms_radius, 'remove_borders': opt.remove_borders,
                                 'weights': opt.superpoint_weights}).eval()
        if not opt.superpoint_weights:
            superpoint.load_state_dict({k: torch.from_numpy(v) for k, v in make_superpoint_state_dict(opt.seed).items()})
        superpoint = superpoint.cuda()
        opt.batch = opt.image_batch
    pipe = MultiViewPipeline(matcher, superpoint=superpoint)
    pose_errors = [[], [], []]
    with torch.no_grad():
        for start in range(0, opt.n_tuples, opt.batch):
            b = min(opt.batch, opt.n_tuples - start)
            if opt.images:
                # tuple i is rendered from seed 1000 + i whatever the batch size, so --image_batch changes the batching
                # and nothing else
                parts = [render_tuple_images(make_scene_tuple_inputs(1000 + i, opt.tuple_size, opt.max_keypoints,
                                                                     batch=1, noise_px=0.0), seed=1000 + i)
                         for i in range(start, start + b)]
                data = {k: (torch.from_numpy(np.concatenate([p[k] for p in parts])).cuda() if isinstance(v, np.ndarray)
                            else v) for k, v in parts[0].items()
                        if not k.startswith(('keypoints', 'scores', 'descriptors'))}
            else:
                data = make_scene_tuple_inputs(1000 + start, opt.tuple_size, opt.max_keypoints, batch=b)
                data = {k: (torch.from_numpy(v).cuda() if isinstance(v, np.ndarray) and not k.startswith('image')
                            else (torch.empty(v.shape, device='meta') if isinstance(v, np.ndarray) else v))
                        for k, v in data.items()}
            if opt.images:
                # one (result, pose) per tuple: the SuperPoint counts of a batch may differ between tuples
                errs = MultiViewPipeline.tuple_errors(data, [p for _, p in pipe.run_tuples(data)], opt.tuple_size)
            else:
                errs = MultiViewPipeline.pair_errors(data, pipe(data)[1], opt.tuple_size)
            for e in errs:
                for i in range(3):
                    pose_errors[i].append(e[i])
    metrics = write_result(pose_errors, opt.out)
    print(json.dumps(metrics))
    return metrics


if __name__ == '__main__':
    main()
