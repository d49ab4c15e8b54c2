"""Two-view benchmark driver with the reference's flow (eval_pairs.py:130-278) for its four modes: pairwise matcher
(multi_frame_matching=False, 18 layers, confidence head), then weighted eight-point (`w8pt`) or RANSAC + recoverPose on
the matches above match_threshold 0.02 (`ransac`, eval_pairs.py:152), each optionally followed by the two-view bundle
adjustment (`w8pt_ba`, `ransac_ba`), AUC@5/10/20 as JSON.  Data are synthetic two-view
scenes (no datasets offline): 1024 keypoints @ 640x480 ("scannet") or 2048 @ 1600x1200 ("megadepth").

    python -m e2e_multi_view_matching_b200.eval_pairs --eval_mode w8pt_ba --n_pairs 64
"""
import argparse
import json

import numpy as np
import torch

from .models.multi_view_matcher import MultiViewMatcher
from .pipeline import PairPipeline, compute_pose_error_np, pose_auc
from .synthetic import make_state_dict, make_scene_tuple_inputs


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--eval_mode', default='w8pt_ba', choices=['ransac', 'ransac_ba', 'w8pt', 'w8pt_ba'])
    ap.add_argument('--dataset', default='scannet', choices=['scannet', 'megadepth', 'yfcc100m'])
    ap.add_argument('--n_pairs', type=int, default=32)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--ckpt', default=None)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--math_mode', type=int, default=3)
    ap.add_argument('--out', default=None)
    opt = ap.parse_args(argv)
    import e2e_multi_view_matching_b200 as pkg
    pkg.set_math_mode(opt.math_mode)
    n_kpts, (w, h) = (1024, (640, 480)) if opt.dataset == 'scannet' else (2048, (1600, 1200))   # eval_pairs.py:157-180
    layers = ['self', 'cross'] * 9
    matcher = MultiViewMatcher({'multi_frame_matching': False, 'GNN_layers': layers, 'conf_mlp': True}).eval()
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
    match_threshold = 0.02 if 'ransac' in opt.eval_mode else 0.0        # eval_pairs.py:152
    pipe = PairPipeline(matcher, eval_mode=opt.eval_mode, match_threshold=match_threshold)
    errors, failed = [], 0
    with torch.no_grad():
        for start in range(0, opt.n_pairs, opt.batch):
            b = min(opt.batch, opt.n_pairs - start)
            data = make_scene_tuple_inputs(5000 + start, 2, n_kpts, batch=b, width=w, height=h,
                                           f=577.87 * w / 640.0)
            gt = [np.linalg.inv(data['pose1'][i].astype(np.float64)) @ data['pose0'][i].astype(np.float64)
                  for i in range(b)]
            data = {k: (torch.from_numpy(v).cuda() if isinstance(v, np.ndarray) and not k.startswith('image')
                        else (torch.empty(v.shape, device='meta') if isinstance(v, np.ndarray) else v))
                    for k, v in data.items()}
            _, pose = pipe(data)
            T = pose['T_021'].double().cpu().numpy()
            ok = pose['success'].cpu().numpy()
            for i in range(b):
                if not ok[i]:
                    errors.append(np.inf)       # eval_pairs.py:258-260
                    failed += 1
                    continue
                et, er = compute_pose_error_np(gt[i], T[i, :3, :3], T[i, :3, 3])
                errors.append(max(et, er))
    aucs = pose_auc(errors, [5, 10, 20])
    result = {"AUC@5deg": 100. * aucs[0], "AUC@10deg": 100. * aucs[1], "AUC@20deg": 100. * aucs[2],
              "cannot_compute_pose": failed, "n_pairs": len(errors)}
    if opt.out:
        with open(opt.out, 'w') as tf:
            json.dump(result, tf, indent=4)
    print(json.dumps(result))
    return result


if __name__ == '__main__':
    main()
