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

from . import _lib
from .models.multi_view_matcher import MultiViewMatcher, split_ragged_result
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
        case).  A batch of tuples has one tensor per output, so an image batch (B > 1) whose SuperPoint counts differ
        between tuples is refused here: run_tuples matches it as a ragged batch."""
        out = self._run(data, global_ba)
        if isinstance(out, list):
            raise ValueError('the SuperPoint counts of this image batch differ between tuples: use '
                             'MultiViewPipeline.run_tuples, which returns one (result, pose) per tuple')
        return out

    def run_tuples(self, data, global_ba=True):
        """-> a list with one (result, pose) per tuple of the batch, each as __call__ returns it for that tuple alone
        (batch dimension 1, tensors cut to the tuple's keypoint counts).  Any batch: keypoints given (counts{i} for a
        ragged one), or images, whose SuperPoint counts may differ between tuples (a ragged batch, see _run_ragged)."""
        out = self._run(data, global_ba)
        if isinstance(out, list):
            return out
        result, pose = out
        B = result['keypoints0'].shape[0] if 'keypoints0' in result else data['keypoints0'].shape[0]
        if B == 1:
            return [out]
        src = result if 'keypoints0' in result else data      # the front end's features, or the caller's
        T = len(data['ids'])
        counts = [data['counts%d' % i] if 'counts%d' % i in data else [src['keypoints%d' % i].shape[1]] * B
                  for i in range(T)]
        results = split_ragged_result(result, counts)
        return [(results[b], None if pose is None else
                 {k: (v[b:b + 1] if torch.is_tensor(v) else v) for k, v in pose.items()}) for b in range(B)]

    def _run(self, data, global_ba):
        """__call__'s work; a list of per-tuple (result, pose) for a ragged image batch."""
        features = {}
        if 'keypoints0' not in data:
            if self.superpoint is None:
                raise ValueError('keypoints0 missing and no SuperPoint front-end given')
            from .training import run_super_point
            views = ['image%d' % i for i in range(len(data['ids']))]
            batch = data['image0'].shape[0]
            data = dict(data)
            before = set(data)
            merge = len({tuple(data[k].shape) for k in views}) == 1
            if batch > 1 and merge and self._batched_front_end(data):
                ragged = self._super_point_batch(data)
                if ragged is not None:
                    return self._run_ragged(data, ragged, global_ba)
            else:
                run_super_point(types.SimpleNamespace(batch_size=batch), data, self.superpoint, merge=merge)
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

    def _batched_front_end(self, data):
        """True when SuperPoint.forward_batch serves this image batch (run_super_point's condition for it)."""
        k_max = self.superpoint.config['max_keypoints']
        h, w = data['image0'].shape[-2:]
        return 0 < k_max <= min(_lib.MVM_SUPERPOINT_MAX_SELECT, (h // 8 * 8) * (w // 8 * 8))

    def _super_point_batch(self, data):
        """SuperPoint on every image of the batch in one forward_batch.  Every image at max_keypoints (always so with
        fill_with_random_keypoints): data gets keypoints{i} / scores{i} / descriptors{i} as run_super_point gives them,
        returns None.  Otherwise returns the [T, B] host counts and the padded [T, B, ...] device tensors."""
        T, B = len(data['ids']), data['image0'].shape[0]
        K = self.superpoint.config['max_keypoints']
        out = self.superpoint.forward_batch(torch.cat([data['image%d' % i].cuda() for i in range(T)], 0))
        counts = out['counts'].view(T, B)
        host = counts.tolist()               # the one read of the counts per batch: routing and splitting need it
        feats = {k: out[k].view(T, B, *out[k].shape[1:]) for k in ('keypoints', 'scores', 'descriptors')}
        if all(n == K for row in host for n in row):
            for k, v in feats.items():
                for m in range(T):
                    data[k + str(m)] = v[m]
            return None
        return host, counts, feats

    def _run_ragged(self, data, ragged, global_ba):
        """An image batch whose views have different keypoint counts per tuple.  The tuples with keypoints in every
        view run as one ragged batch (counts{i} on the device, capacities = the largest count of each view); a tuple
        with an empty view runs alone through the batch-of-one call, which drops that view as the reference does, so it
        cannot touch another tuple's results.  Returns one (result, pose) per tuple, each shaped as a batch-of-one call
        returns it."""
        host, counts, feats = ragged
        T, B = len(host), len(host[0])
        full = [b for b in range(B) if all(host[m][b] > 0 for m in range(T))]
        alone = [b for b in range(B) if b not in full]
        results, poses = [None] * B, [None] * B
        if len(full) < 2:
            alone, full = sorted(alone + full), []

        def tuples(idx, caps):
            sel = torch.tensor(idx, device=counts.device)
            d = {k: (v.index_select(0, sel.to(v.device)) if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == B else v)
                 for k, v in data.items()}
            for m in range(T):
                d['keypoints%d' % m] = feats['keypoints'][m].index_select(0, sel)[:, :caps[m]]
                d['scores%d' % m] = feats['scores'][m].index_select(0, sel)[:, :caps[m]]
                d['descriptors%d' % m] = feats['descriptors'][m].index_select(0, sel)[:, :, :caps[m]]
            return d

        for b in alone:
            d = tuples([b], [host[m][b] for m in range(T)])
            results[b], poses[b] = self._run(d, global_ba)
            results[b].update({k: d[k] for k in d if k.startswith(('keypoints', 'scores', 'descriptors'))})
        if full:
            d = tuples(full, [max(host[m][b] for b in full) for m in range(T)])
            sel = torch.tensor(full, device=counts.device)
            for m in range(T):
                d['counts%d' % m] = counts[m].index_select(0, sel)
            result = self.matcher(d)
            result.update({k: d[k] for k in d if k.startswith(('keypoints', 'scores', 'descriptors'))})
            state = self.matcher._engine.last
            pose = self.pose.run(state, [d['intr%d' % i] for i in state['view_ids']], global_ba=global_ba)
            pose['view_ids'] = list(state['view_ids'])
            split = split_ragged_result(result, [[host[m][b] for b in full] for m in range(T)])
            for i, b in enumerate(full):
                results[b] = split[i]
                poses[b] = {k: (v[i:i + 1] if torch.is_tensor(v) else v) for k, v in pose.items()}
        return list(zip(results, poses))

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

    @staticmethod
    def tuple_errors(data, poses, tuple_size):
        """pair_errors of run_tuples' output: poses = the pose of every tuple of `data`, in order."""
        return [e for b, p in enumerate(poses)
                for e in MultiViewPipeline.pair_errors({'pose%d' % i: data['pose%d' % i][b:b + 1]
                                                        for i in range(tuple_size)}, p, tuple_size)]


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
