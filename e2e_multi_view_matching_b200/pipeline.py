"""Public end-to-end API: the loop bodies of the reference's eval entry points, device resident.

  MultiViewPipeline.__call__  ==  eval_multi_view.py:152-162 (matcher on a tuple, then
                                  eval_bundle_adjust, eval_multi_view.py:21-68)
  PairPipeline.__call__       ==  eval_pairs.py:208-267 for the w8pt / w8pt_ba / ransac / ransac_ba modes

Inputs are the reference's `data` dicts (keypoints{i}, scores{i}, descriptors{i}, image{i}, intr{i},
ids; MultiViewPipeline with a SuperPoint front-end also takes image{i} without keypoints); there is no numpy hop
between matcher and pose, no subprocess and no CSV file.
"""
import types

import numpy as np
import torch

from .models.multi_view_matcher import MultiViewMatcher
from .pose_optimization.multi_view.pose_engine import MultiViewPoseEngine


def compute_pose_error_np(T_0to1, R, t):
    """models/models/utils.py:388-395 (numpy fp64, evaluation only)."""
    t_gt = T_0to1[:3, 3]
    n = np.linalg.norm(t) * np.linalg.norm(t_gt)
    et = np.rad2deg(np.arccos(np.clip(np.dot(t, t_gt) / n, -1.0, 1.0))) if n > 0 else 180.0
    et = np.minimum(et, 180 - et)
    cos = np.clip((np.trace(np.dot(R.T, T_0to1[:3, :3])) - 1) / 2, -1., 1.)
    return et, np.rad2deg(np.abs(np.arccos(cos)))


def pose_auc(errors, thresholds):
    """models/models/utils.py:397-409."""
    sort_idx = np.argsort(errors)
    errors = np.array(errors.copy())[sort_idx]
    recall = (np.arange(len(errors)) + 1) / len(errors)
    errors = np.r_[0., errors]
    recall = np.r_[0., recall]
    aucs = []
    for t in thresholds:
        last_index = np.searchsorted(errors, t)
        r = np.r_[recall[:last_index], recall[last_index - 1]]
        e = np.r_[errors[:last_index], t]
        aucs.append(np.trapezoid(r, x=e) / t)
    return aucs


class MultiViewPipeline:
    """[SuperPoint +] matcher (multi_frame_matching=True) + multi-view pose stage for batches of tuples."""

    def __init__(self, matcher: MultiViewMatcher, conf_thresh=0.0, superpoint=None):
        assert matcher.config['multi_frame_matching'] and matcher.config['conf_mlp']
        self.matcher = matcher
        self.superpoint = superpoint
        self.pose = MultiViewPoseEngine(conf_thresh=conf_thresh)

    def __call__(self, data, global_ba=True):
        """-> (matcher result, pose).  When `data` has no keypoints0, the `superpoint` front-end runs on image{i} first
        (run_super_point, as eval_multi_view.py:157 does; views of one image size run as one batch) and the result
        also carries its keypoints{i} / scores{i} / descriptors{i}; the caller's dict is left as it is.  Views without
        keypoints are skipped by the matcher (multi_view_matcher.py:155-162), so the pose stage works on view SLOTS:
        pose['view_ids'][s] is the id (in `data`) of slot s, the extrinsics / pair tensors are indexed by slot.  pose
        is None when fewer than two views have keypoints (nothing to estimate: the reference's "cannot compute pose"
        case)."""
        features = {}
        if 'keypoints0' not in data:
            if self.superpoint is None:
                raise ValueError('keypoints0 missing and no SuperPoint front-end given')
            from .training import run_super_point
            views = ['image%d' % i for i in range(len(data['ids']))]
            batch = data['image0'].shape[0]
            data = dict(data)
            before = set(data)
            run_super_point(types.SimpleNamespace(batch_size=batch), data, self.superpoint,
                            merge=len({tuple(data[k].shape) for k in views}) == 1)
            features = {k: data[k] for k in set(data) - before}
        result = self.matcher(data)
        result.update(features)
        state = self.matcher._engine.last
        if state is None:
            return result, None
        view_ids = state['view_ids']
        intr = [data['intr%d' % i] for i in view_ids]
        pose = self.pose.run(state, intr, global_ba=global_ba)
        pose['view_ids'] = list(view_ids)
        return result, pose

    @staticmethod
    def pair_errors(data, pose, tuple_size):
        """Pose errors of every pair id0 < id1 from the absolute extrinsics (eval_multi_view.py:53-66); pairs with
        a view that has no keypoints (or pose None) count as failures (inf), like eval_pairs.py:258-260."""
        n_batch = data['pose0'].shape[0]
        if pose is None:
            return [(np.inf, np.inf, np.inf)] * (n_batch * tuple_size * (tuple_size - 1) // 2)
        extr = pose['extrinsics'].double().cpu().numpy()
        slot = {v: s for s, v in enumerate(pose.get('view_ids', range(tuple_size)))}
        errs = []
        for b in range(extr.shape[0]):
            for id1 in range(tuple_size):
                for id0 in range(id1):
                    if id0 not in slot or id1 not in slot:
                        errs.append((np.inf, np.inf, np.inf))
                        continue
                    p0 = data['pose%d' % id0][b].double().cpu().numpy()
                    p1 = data['pose%d' % id1][b].double().cpu().numpy()
                    T_gt = np.linalg.inv(p1) @ p0            # cam->world poses, as the reference (eval_multi_view.py:59)
                    T_pr = extr[b, slot[id1]] @ np.linalg.inv(extr[b, slot[id0]])
                    et, er = compute_pose_error_np(T_gt, T_pr[:3, :3], T_pr[:3, 3])
                    errs.append((max(et, er), et, er))
        return errs


class PairPipeline:
    """matcher (pairwise) + w8pt or RANSAC [+ two-view BA] (eval_pairs.py modes `w8pt`, `w8pt_ba`, `ransac`,
    `ransac_ba`)."""

    def __init__(self, matcher: MultiViewMatcher, eval_mode='w8pt_ba', match_threshold=0.0):
        assert eval_mode in ('w8pt', 'w8pt_ba', 'ransac', 'ransac_ba')
        self.matcher = matcher
        self.eval_mode = eval_mode
        self.pose = MultiViewPoseEngine(conf_thresh=match_threshold)

    def __call__(self, data):
        result = self.matcher(data)
        state = self.matcher._engine.last
        if state is None:            # a view without keypoints: "cannot compute pose" (eval_pairs.py:258-260)
            return result, None
        intr = [data['intr0'], data['intr1']]
        if self.eval_mode.startswith('ransac'):
            pose = self.pose.run(state, intr, global_ba=False, rel_pose_method=self.eval_mode)
            return result, {'T_021': pose['T_pair'][:, 0], 'success': pose['success'][:, 0],
                            'inliers': pose['inliers'][:, 0], 'n_inliers': pose['n_inliers'][:, 0],
                            'ransac_iterations': pose['ransac_iterations'][:, 0], **{k: v for k, v in pose.items()
                                                                                    if k not in ('inliers', 'n_inliers')}}
        pose = self.pose.run(state, intr, global_ba=False)
        T = pose['T_pair'] if self.eval_mode == 'w8pt_ba' else pose['T_w8pt']
        return result, {'T_021': T[:, 0], 'success': pose['success'][:, 0], **pose}
