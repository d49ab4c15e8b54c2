"""The geometry helper of the reference's models/models/utils.py that its RANSAC eval modes call, computing in
libmvm_b200.so (mvm_ransac_essential, csrc/pose_ransac.cu).  numpy in, numpy out, like the reference; there is no
CPU fallback."""
import numpy as np
import torch

from .. import _lib

RANSAC_MAX_ITERS = 1000      # OpenCV's findEssentialMat default
RANSAC_SEED = 0


def estimate_pose(kpts0, kpts1, K0, K1, thresh, conf=0.99999):
    """models/models/utils.py:288-312: essential matrix by RANSAC on the matches kpts0 <-> kpts1 ([n, 2] pixels),
    pose by recoverPose.  Returns (R [3,3], t [3] unit, mask [n] bool: the inliers in front of both cameras) or None
    (fewer than 5 matches, or no pose found)."""
    kpts0 = np.ascontiguousarray(kpts0, np.float32).reshape(-1, 2)
    kpts1 = np.ascontiguousarray(kpts1, np.float32).reshape(-1, 2)
    n = len(kpts0)
    if n < 5:
        return None
    dev = torch.device('cuda', torch.cuda.current_device()) if torch.cuda.is_available() else torch.device('cpu')
    _lib.require_cuda(dev, 'estimate_pose')
    lib = _lib.lib()
    f32 = dict(dtype=torch.float32, device=dev)
    k0 = torch.from_numpy(kpts0).to(dev)[None]
    k1 = torch.from_numpy(kpts1).to(dev)[None]
    intr = [torch.tensor([[K[0, 0], K[1, 1], K[0, 2], K[1, 2]]], **f32) for K in (np.asarray(K0), np.asarray(K1))]
    T = torch.empty(1, 16, **f32)
    k0n = torch.empty(1, n, 2, **f32)
    k1n = torch.empty(1, n, 2, **f32)
    inl = torch.empty(1, n, dtype=torch.uint8, device=dev)
    n_inl = torch.empty(1, dtype=torch.int32, device=dev)
    E = torch.empty(1, 10, 9, dtype=torch.float64, device=dev)
    n_mod = torch.empty(1, dtype=torch.int32, device=dev)
    iters = torch.empty(1, dtype=torch.int32, device=dev)
    succ = torch.empty(1, dtype=torch.uint8, device=dev)
    with _lib.device_ctx(dev):
        _lib.check(lib.mvm_ransac_essential(_lib.ptr(k0), _lib.ptr(k1), _lib.ptr(intr[0]), _lib.ptr(intr[1]), 1, n, None,
                                            float(thresh), float(conf), RANSAC_MAX_ITERS, RANSAC_SEED, _lib.ptr(T),
                                            _lib.ptr(k0n), _lib.ptr(k1n), _lib.ptr(inl), _lib.ptr(n_inl), _lib.ptr(E),
                                            _lib.ptr(n_mod), _lib.ptr(iters), _lib.ptr(succ), _lib.stream_ptr()),
                   'mvm_ransac_essential')
    if not bool(succ[0]):
        return None
    T = T.view(4, 4).double().cpu().numpy()
    return T[:3, :3], T[:3, 3], inl[0].cpu().numpy() > 0
