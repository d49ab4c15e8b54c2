"""Training-side consumers of the matcher output -- SURVEY.md §8 f-2 / a20 (BASELINE cfg5).

Built:
  * run_super_point (helpers.py:83-96): SuperPoint on the images of a tuple batch, merged batches through
    SuperPoint.forward_batch (keypoint selection and descriptor sampling on the device, one launch each, one dense pass
    whether or not every image reaches max_keypoints);
    train_step / validation_step call it when the batch has images and no keypoints;
  * compute_match_loss (helpers.py:228-241) as an autograd.Function on CUDA kernels (csrc/train_loss.cu), forward
    and backward;
  * combine_losses (train.py:36-40);
  * compute_gt_matches_of_image_pair / compute_gt_matches (helpers.py:121-226): ground-truth assignments from depth
    maps and poses on CUDA kernels (csrc/gt_matches.cu; the [bs, N, N] error matrix is never materialised);
  * run_matcher (helpers.py:243-260) and validation_step (the loop body of Trainer.validate, train.py:89-106): matcher
    forward, match loss, weighted eight-point with choose_closest against the ground-truth pose, rotation / translation
    losses, combine_losses and the validation-loss all-reduce;
  * the TRAINING step of stage 1 (train.py:405-426 without --pose_loss: match loss only): train_step = compute_gt_matches,
    run_matcher with the matcher in train() mode (models/train_forward.py: batch-statistics BatchNorm, and
    MatcherTrainFn's backward on the kernels: attention backward, BatchNorm backward, the exact gradient of the
    unrolled Sinkhorn iterations, 3xTF32 GEMMs), combine_losses, backward, the data-parallel gradient all-reduce
    (sharding.all_reduce_gradients, what DistributedDataParallel does for the reference) and the optimiser step;
  * LogOptimalTransport: autograd.Function over mvm_sinkhorn_train_{forward,backward} -- the exact gradient of the 100
    unrolled iterations (what autograd computes for the reference, superglue.py:143-172), with respect to the scores
    and to bin_score.
The weighted eight-point is differentiable with respect to the match confidences
(pose_optimization/two_view/estimate_relative_pose.py, mvm_w8pt_backward), so the pose losses of run_matcher carry a
graph as far as conf_scores.  Not built (stated, not hidden): the rest of stage 2 of cfg5 (--pose_loss): the backward of
the ConfidenceMLP, the graph through the train-mode full_output, and train_step with opt.pose_loss (it raises).
"""
import torch

from . import _lib
from . import ops


class _MatchLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, log_p, gt_indices, gt_weights):
        if log_p.device.type != 'cuda':
            raise _lib.MvmError('compute_match_loss needs CUDA tensors (no CPU fallback)')
        lib = _lib.lib()
        bs, ft, ft2 = log_p.shape
        assert ft == ft2 and gt_indices.shape == (bs, 2, ft) and gt_weights.shape == (bs, 2, ft)
        lp = log_p.detach().float().contiguous()
        idx = gt_indices.long().contiguous()
        w = gt_weights.float().contiguous()
        part = torch.empty(bs, dtype=torch.float64, device=lp.device)
        loss = torch.empty(1, dtype=torch.float32, device=lp.device)
        with torch.cuda.device(lp.device):
            _lib.check(lib.mvm_match_loss_forward(_lib.ptr(lp), _lib.ptr(idx), _lib.ptr(w), bs, ft, _lib.ptr(part),
                                                  _lib.ptr(loss), _lib.stream_ptr()), 'mvm_match_loss_forward')
        ctx.save_for_backward(idx, w)
        ctx.shape = (bs, ft)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, grad):
        lib = _lib.lib()
        idx, w = ctx.saved_tensors
        bs, ft = ctx.shape
        g = grad.detach().float().reshape(1).contiguous()
        out = torch.empty(bs, ft, ft, dtype=torch.float32, device=idx.device)
        with torch.cuda.device(idx.device):
            _lib.check(lib.mvm_match_loss_backward(_lib.ptr(idx), _lib.ptr(w), _lib.ptr(g), bs, ft, _lib.ptr(out),
                                                   _lib.stream_ptr()), 'mvm_match_loss_backward')
        return out, None, None


def compute_match_loss(log_p, gt_indices_0_1, gt_weights_0_1):
    """helpers.py:228-241."""
    return _MatchLoss.apply(log_p, gt_indices_0_1, gt_weights_0_1)


def combine_losses(losses, n_pairs, pose_match_ratio, rot_weight, trans_weight):
    """train.py:36-40."""
    losses = {k: v / float(n_pairs) for k, v in losses.items()}
    pose_loss = rot_weight * losses["rot_loss"] + trans_weight * losses["transl_loss"]
    total_loss = (1. - pose_match_ratio) * losses["match_loss"] + pose_match_ratio * pose_loss
    return total_loss, losses


class LogOptimalTransport(torch.autograd.Function):
    """log_optimal_transport(scores, alpha, iters) (superglue.py:152-172) with gradients w.r.t. scores and alpha:
    mvm_sinkhorn_train_forward keeps the potentials of every iteration, mvm_sinkhorn_train_backward runs the exact
    reverse recursion of the unrolled iterations (csrc/sinkhorn_train.cu)."""

    @staticmethod
    def forward(ctx, scores, alpha, iters):
        _lib.require_cuda(scores.device, 'LogOptimalTransport')
        s = scores.detach().float().contiguous()
        a = alpha.detach().float().reshape(1).to(s.device).contiguous()
        with _lib.device_ctx(s.device):
            Z, pot = ops.sinkhorn_train_forward(s, a, int(iters))
        ctx.save_for_backward(s, a, pot)
        ctx.iters = int(iters)
        ctx.alpha_shape = alpha.shape
        return Z

    @staticmethod
    def backward(ctx, G):
        s, a, pot = ctx.saved_tensors
        _, m, n = s.shape
        with _lib.device_ctx(s.device):
            dZ, d_alpha = ops.sinkhorn_train_backward(s, a, pot, ctx.iters, G)
        return dZ[:, :m, :n].contiguous(), d_alpha.float().reshape(ctx.alpha_shape), None


def log_optimal_transport(scores, alpha, iters):
    return LogOptimalTransport.apply(scores, alpha if torch.is_tensor(alpha) else torch.tensor(float(alpha)), iters)


def compute_gt_matches_of_image_pair(kpts0, kpts1, K0, K1, T0to1, depth0, depth1, max_matched_reproj_err,
                                     min_unmatched_reproj_err):
    """helpers.py:121-203 -> (indices [bs,2,N+1] int64, weights [bs,2,N+1] float32)."""
    if kpts0.device.type != 'cuda':
        raise _lib.MvmError('compute_gt_matches_of_image_pair needs CUDA tensors (no CPU fallback)')
    lib = _lib.lib()
    bs, n, _ = kpts0.shape
    assert kpts1.shape == (bs, n, 2) and depth0.shape == depth1.shape and depth0.dim() == 3
    H, W = depth0.shape[1:]
    dev = kpts0.device
    f = lambda t: t.detach().float().contiguous()
    k0, k1, K0_, K1_, T_, d0, d1 = f(kpts0), f(kpts1), f(K0), f(K1), f(T0to1), f(depth0), f(depth1)
    assert K0_.shape == (bs, 4, 4) and K1_.shape == (bs, 4, 4) and T_.shape == (bs, 4, 4)
    indices = torch.empty(bs, 2, n + 1, dtype=torch.int64, device=dev)
    weights = torch.empty(bs, 2, n + 1, dtype=torch.float32, device=dev)
    nbytes = lib.mvm_gt_matches_workspace_bytes(bs, n)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.mvm_gt_matches_pair(_lib.ptr(k0), _lib.ptr(k1), _lib.ptr(K0_), _lib.ptr(K1_), _lib.ptr(T_),
                                           _lib.ptr(d0), _lib.ptr(d1), bs, n, H, W, float(max_matched_reproj_err),
                                           float(min_unmatched_reproj_err), _lib.ptr(indices), _lib.ptr(weights),
                                           _lib.ptr(ws), nbytes, _lib.stream_ptr()), 'mvm_gt_matches_pair')
    return indices, weights


def run_super_point(opt, data, super_point, merge=True):
    """helpers.py:83-96: SuperPoint on image{m} of every view m of the tuple, results as data['keypoints' + m],
    data['scores' + m], data['descriptors' + m] ([B,N,2], [B,N], [B,256,N]).  With merge the T views' [B,1,H,W] batches
    run as one through SuperPoint.forward_batch (when 0 < max_keypoints <= MVM_SUPERPOINT_MAX_SELECT and max_keypoints
    is at most the score map's pixel count).  When every image ends with max_keypoints keypoints (always so with
    fill_with_random_keypoints) its [T*B, ...] tensors are viewed as [T, B, ...]; otherwise each image's valid entries
    become the per-image lists forward would give (bitwise; among equal scores at the cut, the selection's tie rule)
    without a second dense pass.  merge=False and the other configurations go through SuperPoint.forward.  The lists
    are stacked as the reference does (batch size 1: each image's tensors with a leading 1)."""
    curr_tuple_size = len(data["ids"])
    images = [data["image" + str(i)].cuda() for i in range(curr_tuple_size)]
    if merge:
        images = [torch.cat(images, 0)]
    k_max = super_point.config['max_keypoints']
    map_px = (images[0].shape[-2] // 8 * 8) * (images[0].shape[-1] // 8 * 8)
    with torch.no_grad():
        if merge and 0 < k_max <= min(_lib.MVM_SUPERPOINT_MAX_SELECT, map_px):
            out = super_point.forward_batch(images[0])
            counts = out['counts'].tolist() if not super_point.config['fill_with_random_keypoints'] else None
            if counts is None or all(n == k_max for n in counts):
                for k in ('keypoints', 'scores', 'descriptors'):
                    res = out[k].view(curr_tuple_size, opt.batch_size, *out[k].shape[1:])
                    for m in range(curr_tuple_size):
                        data[k + str(m)] = res[m]
                return
            pred = {'keypoints': [out['keypoints'][b, :n] for b, n in enumerate(counts)],
                    'scores': [out['scores'][b, :n] for b, n in enumerate(counts)],
                    'descriptors': [out['descriptors'][b, :, :n].contiguous() for b, n in enumerate(counts)]}
        else:
            pred = super_point({"image": images})
        for k, v in pred.items():
            if len(v) != curr_tuple_size:  # batch size > 1
                res = torch.stack(v)
                res = res.view(curr_tuple_size, opt.batch_size, *res.shape[1:])
            else:  # batch size 1
                res = [v_i.unsqueeze(0) for v_i in v]
            for m in range(curr_tuple_size):
                data[k + str(m)] = res[m]


def _images_in(data, super_point):
    """True when the batch carries images and no keypoints yet: SuperPoint runs first (train.py:409)."""
    if "image0" not in data or "keypoints0" in data:
        return False
    if super_point is None:
        raise ValueError('the batch has images and no keypoints: pass super_point= to run SuperPoint on them')
    return True


def compute_gt_matches(opt, data):
    """helpers.py:215-226: gt_indices_k_m / gt_weights_k_m for every pair k < m of the tuple; pops the depth maps."""
    curr_tuple_size = len(data["ids"])
    for m in range(curr_tuple_size):
        for k in range(m):
            T_k2m = torch.linalg.inv(data["pose" + str(m)]) @ data["pose" + str(k)]
            data["gt_indices_{}_{}".format(k, m)], data["gt_weights_{}_{}".format(k, m)] = \
                compute_gt_matches_of_image_pair(data["keypoints" + str(k)], data["keypoints" + str(m)],
                                                 data["intr" + str(k)], data["intr" + str(m)], T_k2m,
                                                 data["depth" + str(k)], data["depth" + str(m)],
                                                 opt.match_reproj_err, opt.unmatch_reproj_err)
    for m in range(curr_tuple_size):
        data.pop("depth" + str(m))


def run_matcher(opt, data, matcher):
    """helpers.py:243-260.  Eval mode = the validation pass (train.py:66-68); train mode = the training step, where the
    match loss carries MatcherTrainFn's graph.  The pose losses carry a graph through the weighted eight-point as far
    as conf_scores when those require grad; the train-mode conf_scores have none yet (the confidence head's backward
    is not built), so in train mode the pose losses still reach no parameter."""
    from .pose_optimization.two_view.estimate_relative_pose import run_weighted_8_point
    from .pose_optimization.two_view.compute_pose_error import compute_rotation_error, compute_translation_error_as_angle
    curr_tuple_size = len(data["ids"])
    getattr(matcher, 'module', matcher).config["full_output"] = opt.pose_loss        # DataParallel / DDP wrapped or bare
    result = matcher(data)
    match_loss = torch.zeros(1, device=data["pose0"].device)
    rot_loss = torch.zeros(1, device=match_loss.device)
    transl_loss = torch.zeros(1, device=match_loss.device)
    for id1 in range(curr_tuple_size):
        for id0 in range(id1):
            match_loss = match_loss + compute_match_loss(result["scores_{}_{}".format(id0, id1)],
                                                         data["gt_indices_{}_{}".format(id0, id1)],
                                                         data["gt_weights_{}_{}".format(id0, id1)])
            if opt.pose_loss:
                target = torch.linalg.inv(data["pose{}".format(id1)]) @ data["pose{}".format(id0)]
                pred, _ = run_weighted_8_point(data, result, id0, id1, choose_closest=True, target_T_021=target)
                rot_loss = rot_loss + compute_rotation_error(pred, target)
                transl_loss = transl_loss + compute_translation_error_as_angle(pred, target)
    losses = {"match_loss": match_loss, "rot_loss": rot_loss, "transl_loss": transl_loss}
    return losses, result


def validation_step(opt, data, matcher, n_pairs, pose_match_ratio, process_group=None, super_point=None):
    """One batch of Trainer.validate (train.py:89-106): run_super_point when the batch carries images and no keypoints
    (then `super_point` is required), ground-truth matches when it still carries depth maps, run_matcher,
    combine_losses; the scalar validation loss is all-reduced over the ranks (mean) when torch.distributed is
    initialised.  -> (val_loss tensor [1], losses dict)."""
    with torch.no_grad():
        if _images_in(data, super_point):
            run_super_point(opt, data, super_point)
        if "depth0" in data:
            compute_gt_matches(opt, data)
        losses, _ = run_matcher(opt, data, matcher)
        val_loss, losses = combine_losses(losses, n_pairs, pose_match_ratio, opt.rot_weight, opt.trans_weight)
        val_loss = val_loss.reshape(1).clone()
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            torch.distributed.all_reduce(val_loss, group=process_group)
            val_loss /= torch.distributed.get_world_size(process_group)
    return val_loss, losses


def train_step(opt, data, matcher, optimizer, n_pairs, pose_match_ratio=0.0, grad_clip=-1.0, super_point=None):
    """One iteration of the training loop (train.py:409-426), stage 1 (match loss): run_super_point when the batch
    carries images and no keypoints (then `super_point` is required), ground-truth matches when it still carries depth
    maps, run_matcher in train mode, combine_losses, backward through the kernels, gradient averaging over the ranks
    when torch.distributed is initialised (DistributedDataParallel's all-reduce in the reference), optional value
    clipping, optimiser step.  -> (train_loss tensor, losses dict)."""
    if getattr(opt, 'pose_loss', False):
        raise NotImplementedError('stage 2 (--pose_loss) needs the gradients of the pose stage, which are not built')
    from . import sharding
    if _images_in(data, super_point):
        run_super_point(opt, data, super_point)
    if "depth0" in data:
        with torch.no_grad():
            compute_gt_matches(opt, data)
    losses, _ = run_matcher(opt, data, matcher)
    train_loss, losses = combine_losses(losses, n_pairs, pose_match_ratio, getattr(opt, 'rot_weight', 0.0),
                                        getattr(opt, 'trans_weight', 0.0))
    optimizer.zero_grad(set_to_none=True)
    train_loss.backward()
    params = [p for group in optimizer.param_groups for p in group['params']]
    sharding.all_reduce_gradients(params)
    if grad_clip > 0.0:
        torch.nn.utils.clip_grad_value_(params, grad_clip)
    optimizer.step()
    return train_loss.detach(), {k: v.detach() for k, v in losses.items()}
