"""Two-view relative pose with the reference's call signatures
(pose_optimization/two_view/estimate_relative_pose.py:9-143), computing in libmvm_b200.so:
mvm_w8pt (weighted eight-point + cheirality / choose-closest + inlier test, one CTA per pair) and
mvm_ba2view (LM bundle adjustment with a Schur-complement step).  Errors are values, like the
reference: (None, None) for fewer than 8 keypoints or a missing key, a valid_batch mask for items
with <= 6 matches."""
import logging

import torch

from ... import _lib
from .bundle_adjust_gauss_newton_2_view import BundleAdjustGaussNewton2View


def _intr4(intr):
    """[B,3,3] or [B,4,4] K -> [B,4] (fx, fy, cx, cy)."""
    return torch.stack([intr[..., 0, 0], intr[..., 1, 1], intr[..., 0, 2], intr[..., 1, 2]], -1).float().contiguous()


def normalize(kpts, intr):
    """Pixel -> normalised camera coordinates with (fx, fy, cx, cy) of a 3x3 or 4x4 K; same result as the reference's
    normalize (estimate_relative_pose.py:9-14).  (The kernels fuse this; the function serves callers of the API.)"""
    focal = torch.stack((intr[..., 0, 0], intr[..., 1, 1]), -1).unsqueeze(-2)       # [..., 1, 2]
    centre = torch.stack((intr[..., 0, 2], intr[..., 1, 2]), -1).unsqueeze(-2)
    return (kpts - centre) / focal


def get_kpts(data, result, id0, id1):
    """Matched keypoints of pair (id0, id1) and their confidences, contract of estimate_relative_pose.py:16-31:
    view-1 keypoints gathered by matches0 (an unmatched keypoint, index -1, picks up the LAST keypoint like the
    reference's negative index does -- its confidence is zeroed), confidence = conf_scores masked by matches >= 0."""
    pair = "{}_{}".format(id0, id1)
    per_view = "keypoints" + str(id0) in data
    k0 = data["keypoints" + str(id0)] if per_view else data["keypoints{}_{}".format(id0, pair)]
    k1 = data["keypoints" + str(id1)] if per_view else data["keypoints{}_{}".format(id1, pair)]
    m0 = result["matches{}_{}".format(id0, pair)]
    wrapped = torch.where(m0 < 0, m0 + k1.shape[1], m0).long()
    k1_matched = torch.gather(k1, 1, wrapped.unsqueeze(-1).expand(-1, -1, k1.shape[-1]))
    conf = result["conf_scores_" + pair] * (m0 >= 0).unsqueeze(-1).to(result["conf_scores_" + pair].dtype)
    return k0, k1_matched, data["intr" + str(id0)], data["intr" + str(id1)], conf


def _run_w8pt(kpts0, kpts1, intr0, intr1, conf, choose_closest, T_021, determine_inliers, n_valid=None,
              success=None):
    lib = _lib.lib()
    dev = kpts0.device
    if dev.type != 'cuda':
        raise _lib.MvmError('estimate_relative_pose_w8pt needs CUDA tensors (no CPU fallback)')
    B, N, _ = kpts0.shape
    k0 = kpts0.float().contiguous()
    k1 = kpts1.float().contiguous()
    c = conf.reshape(B, N).float().contiguous()
    i0, i1 = _intr4(intr0.to(dev)), _intr4(intr1.to(dev))
    T = torch.empty(B, 4, 4, dtype=torch.float32, device=dev)
    k0n = torch.empty(B, N, 2, dtype=torch.float32, device=dev)
    k1n = torch.empty(B, N, 2, dtype=torch.float32, device=dev)
    cn = torch.empty(B, N, dtype=torch.float32, device=dev)
    pos = torch.empty(B, N, dtype=torch.uint8, device=dev)
    inl = torch.empty(B, N, dtype=torch.uint8, device=dev) if determine_inliers else None
    F = torch.empty(B, 3, 3, dtype=torch.float32, device=dev)
    Tg = T_021.float().contiguous() if choose_closest else None
    with torch.cuda.device(dev):
        rc = lib.mvm_w8pt(_lib.ptr(k0), _lib.ptr(k1), _lib.ptr(i0), _lib.ptr(i1), _lib.ptr(c), B, N,
                          _lib.ptr(Tg), int(bool(choose_closest)), int(bool(determine_inliers)),
                          _lib.ptr(T), _lib.ptr(k0n), _lib.ptr(k1n), _lib.ptr(cn), _lib.ptr(pos),
                          _lib.ptr(inl), _lib.ptr(F), _lib.ptr(n_valid), _lib.ptr(success), _lib.stream_ptr())
    _lib.check(rc, 'mvm_w8pt')
    return T, k0n, k1n, cn, pos.bool(), (inl.bool() if inl is not None else None), F


class _W8ptFunction(torch.autograd.Function):
    """_run_w8pt with a gradient for `conf` (mvm_w8pt_backward).  Differentiable outputs: T021 and conf_norm; the
    normalised keypoints, the masks and F are not.  Keypoints, intrinsics and the target are constants."""

    @staticmethod
    def forward(ctx, conf, kpts0, kpts1, intr0, intr1, choose_closest, T_021, determine_inliers):
        T, k0n, k1n, cn, pos, inl, F = _run_w8pt(kpts0, kpts1, intr0, intr1, conf, choose_closest, T_021,
                                                 determine_inliers)
        ctx.mark_non_differentiable(k0n, k1n, pos, F, *([inl] if inl is not None else []))
        B, N, _ = kpts0.shape
        ctx.choose_closest = bool(choose_closest)
        ctx.conf_shape, ctx.conf_dtype = conf.shape, conf.dtype
        Tg = T_021.float().contiguous() if choose_closest else None
        ctx.save_for_backward(kpts0.float().contiguous(), kpts1.float().contiguous(), _intr4(intr0.to(kpts0.device)),
                              _intr4(intr1.to(kpts0.device)), conf.reshape(B, N).float().contiguous(), Tg, T)
        return T, cn, k0n, k1n, pos, inl, F

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gT, gcn, *unused):
        k0, k1, i0, i1, c, Tg, T = ctx.saved_tensors
        B, N = c.shape
        gT = torch.zeros_like(T) if gT is None else gT.float().contiguous()
        gcn = None if gcn is None else gcn.reshape(B, N).float().contiguous()
        gc = torch.empty(B, N, dtype=torch.float32, device=c.device)
        lib = _lib.lib()
        with torch.cuda.device(c.device):
            rc = lib.mvm_w8pt_backward(_lib.ptr(k0), _lib.ptr(k1), _lib.ptr(i0), _lib.ptr(i1), _lib.ptr(c), B, N,
                                       _lib.ptr(Tg), int(ctx.choose_closest), _lib.ptr(T), _lib.ptr(gT), _lib.ptr(gcn),
                                       _lib.ptr(gc), _lib.stream_ptr())
        _lib.check(rc, 'mvm_w8pt_backward')
        return gc.reshape(ctx.conf_shape).to(ctx.conf_dtype), None, None, None, None, None, None, None


def find_fundamental(points1, points2, weights):
    """Weighted DLT fundamental matrix (estimate_relative_pose.py:34-82) -> [B,3,3]."""
    B = points1.shape[0]
    eye = torch.eye(3, device=points1.device).unsqueeze(0).repeat(B, 1, 1)
    return _run_w8pt(points1, points2, eye, eye, weights, False, None, False)[6]


def estimate_relative_pose_w8pt(kpts0, kpts1, intr0, intr1, confidence, choose_closest=False, T_021=None, determine_inliers=False):
    """estimate_relative_pose.py:84-128.  Returns (T021 [B,4,4], info) or (None, None).

    Differentiable with respect to `confidence`, in both branches, like the reference: T021 and info["confidence"]
    carry a graph (the backward is mvm_w8pt_backward); the normalised keypoints, the masks and F do not.  The
    keypoints, the intrinsics and T_021 are treated as constants -- in the reference's training they are data.  An
    item with fewer than 8 non-zero confidences gets a NaN gradient: its eight-point solution is not unique.  The
    default branch selects the cheirality candidate per item (kornia 0.7.0 applies item 0's vote to the whole
    batch; the reference only calls it with one pair).  When `confidence` does not require grad (or grad mode is
    off) this is the plain forward launch, and nothing is saved."""
    if kpts0.shape[1] < 8:
        return None, None
    if torch.is_grad_enabled() and confidence.requires_grad:
        T, cn, k0n, k1n, pos, inl, F = _W8ptFunction.apply(confidence, kpts0, kpts1, intr0, intr1, choose_closest,
                                                           T_021, determine_inliers)
    else:
        T, k0n, k1n, cn, pos, inl, F = _run_w8pt(kpts0, kpts1, intr0, intr1, confidence, choose_closest,
                                                 T_021, determine_inliers)
    info = {"kpts0_norm": k0n, "kpts1_norm": k1n, "confidence": cn.unsqueeze(-1), "inliers": inl,
            "pos_depth_mask": pos, "F": F}
    return T, info


def run_weighted_8_point(data, result, id0, id1, choose_closest=False, target_T_021=None):
    """estimate_relative_pose.py:130-136."""
    match_key = "matches{}_{}_{}".format(id0, id0, id1)
    if match_key in result and result[match_key].shape[1] != 0:
        kpts0, kpts1, intr0, intr1, confidence = get_kpts(data, result, id0, id1)
        return estimate_relative_pose_w8pt(kpts0, kpts1, intr0, intr1, confidence, choose_closest=choose_closest, T_021=target_T_021)
    else:
        return None, None


def run_bundle_adjust_2_view(kpts0_norm, kpts1_norm, confidence, init_T021, n_iterations, check_lu_info_strict=False,
                             check_precond_strict=False):
    """estimate_relative_pose.py:138-143 -> (extrinsics of the valid items [nv,4,4], valid_batch [B])."""
    bs = kpts0_norm.shape[0]
    ba = BundleAdjustGaussNewton2View(batch_size=bs, n_iterations=n_iterations, check_lu_info_strict=check_lu_info_strict,
                                      check_precond_strict=check_precond_strict)
    extrinsics, valid_batch = ba.run(kpts0_norm, kpts1_norm, confidence.squeeze(-1), init_T021)
    return extrinsics[:, 1], valid_batch
