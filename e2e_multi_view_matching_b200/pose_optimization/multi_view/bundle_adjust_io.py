"""The reference's multi-view glue (pose_optimization/multi_view/bundle_adjust_io.py) with the same
function names, arguments, `pair_wise_data` keys and CSV file formats, computing in libmvm_b200.so.

  initialize_bundle_adjust      bundle_adjust_io.py:62-191  (valid matches, w8pt + two-view BA per pair,
                                maximum spanning tree, `ba_init_in.csv`)
  write_bundle_adjust_problem   bundle_adjust_io.py:193-259 (triangulation, weights, `ba_in.csv`)
  read_bundle_adjust_result     bundle_adjust_io.py:261-273
  normalize_confidences         bundle_adjust_io.py:56-60
  estimate_relative_pose_w8pt_ba  bundle_adjust_io.py:12-23

Together with the two binaries in `e2e_multi_view_matching_b200/bin/` (`ba_initializer`, `bundle_adjuster`:
same names, same `<dir>` argument, same files -- build.py::build_cli) the unmodified
`eval_multi_view.eval_bundle_adjust` (eval_multi_view.py:21-68) runs against the GPU solvers by pointing its
`build_dir` at `BUNDLE_ADJUSTMENT_BUILD_DIR`.  `solve()` is the in-process route (no files, no subprocess);
the batched, device-resident route of the hot path is `pose_engine.MultiViewPoseEngine`.

The RANSAC relative-pose modes (`rel_pose_method="ransac"/"ransac_ba"`) are not wired into the multi-view flow:
they raise NotImplementedError here.  Their two-view form (estimate_pose, eval_pairs.py's `ransac` / `ransac_ba`) runs
on the GPU through `models.utils.estimate_pose` and `MultiViewPoseEngine.run(..., rel_pose_method='ransac'|'ransac_ba',
global_ba=False)`.
"""
import ctypes as C
import logging
import os

import numpy as np
import torch

from ... import _lib
from ..two_view.estimate_relative_pose import run_bundle_adjust_2_view, estimate_relative_pose_w8pt

BUNDLE_ADJUSTMENT_BUILD_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), 'bin')
MIN_INLIERS = 20     # bundle_adjust_io.py:63


def _cuda(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.cuda()


def estimate_relative_pose_w8pt_ba(intr0, intr1, mkpts0, mkpts1, conf):
    """numpy in, numpy out, batch of one (bundle_adjust_io.py:12-23): weighted eight-point with the inlier
    test, matches behind a camera dropped, ten LM iterations of two-view bundle adjustment."""
    args = [_cuda(a).unsqueeze(0) for a in (mkpts0, mkpts1, intr0, intr1, conf)]
    T, info = estimate_relative_pose_w8pt(*args, determine_inliers=True)
    if T is None:                                   # fewer than 8 matches
        return False, None, None, None
    weights = info["confidence"].masked_fill(~info["pos_depth_mask"].unsqueeze(-1), 0.)
    refined, ok = run_bundle_adjust_2_view(info["kpts0_norm"], info["kpts1_norm"], weights, T, n_iterations=10)
    if bool(ok[0]):
        T = refined
    T = T[0].cpu().numpy()
    return True, T[:3, :3], T[:3, 3], info["inliers"][0].cpu().numpy()


def normalize_confidences(obs_xyc):
    """Third column onwards = confidences of the observations; scaled in place so that they sum to 2 per unit of
    total match confidence (every match contributes two observations; bundle_adjust_io.py:56-60)."""
    obs_xyc[:, 2:] *= 2.0 / (obs_xyc[:, 2:].sum(axis=0, keepdims=True) + 1e-3)
    return obs_xyc


def _all_pairs(n_images):
    return [(id0, id1) for id1 in range(n_images) for id0 in range(id1)]


def _spanning_tree(n_images, pair_wise_data):
    """Maximum spanning tree of the match graph + chained absolute poses on the device
    (mvm_spanning_tree_init; bundle_adjust_io.py:135-172).  Returns (extr [n,4,4] world->cam, on_tree pairs)."""
    lib = _lib.lib()
    pairs = _all_pairs(n_images)
    P = len(pairs)
    T_rel = np.zeros((1, P, 4, 4), np.float32)
    weight = np.zeros((1, P), np.int32)
    success = np.zeros((1, P), np.uint8)
    for p, (id0, id1) in enumerate(pairs):
        key = "rel_pose{}_{}".format(id0, id1)
        if key in pair_wise_data:
            T_rel[0, p] = pair_wise_data[key]
            weight[0, p] = pair_wise_data["mkpts{}_{}_{}".format(id0, id0, id1)].shape[0]
            success[0, p] = 1
    pa = (C.c_int * P)(*[a for a, _ in pairs])
    pb = (C.c_int * P)(*[b for _, b in pairs])
    d_T, d_w, d_s = _cuda(T_rel), _cuda(weight), _cuda(success)
    extr = torch.empty(1, n_images, 4, 4, dtype=torch.float64, device='cuda')
    on_tree = torch.empty(1, P, dtype=torch.uint8, device='cuda')
    _lib.check(lib.mvm_spanning_tree_init(pa, pb, n_images, P, 1, _lib.ptr(d_T), _lib.ptr(d_w), _lib.ptr(d_s),
                                          _lib.ptr(extr), _lib.ptr(on_tree), _lib.stream_ptr()), 'mvm_spanning_tree_init')
    on = on_tree[0].cpu().numpy().astype(bool)
    return extr[0].cpu().numpy(), [pairs[p] for p in range(P) if on[p]]


def initialize_bundle_adjust(n_images, data, result, file_path, conf_thresh=0., rel_pose_method="w8pt_ba"):
    """Same contract as the reference (bundle_adjust_io.py:62-191); `file_path=None` skips the file."""
    if rel_pose_method != "w8pt_ba":
        if rel_pose_method in ("ransac", "ransac_ba"):
            raise NotImplementedError("rel_pose_method '{}' is an OpenCV CPU baseline of the reference; only 'w8pt_ba' "
                                      "runs on the GPU path".format(rel_pose_method))
        logging.error("Relative pose estimation method {} is not defined".format(rel_pose_method))
    pair_wise_data = dict()
    for id0, id1 in _all_pairs(n_images):
        matches_key = "matches{}_{}_{}".format(id0, id0, id1)
        if matches_key not in result:
            continue
        if "keypoints" + str(id0) in data:
            kpts0, kpts1 = data["keypoints" + str(id0)][0].cpu().numpy(), data["keypoints" + str(id1)][0].cpu().numpy()
        else:
            kpts0 = data["keypoints{}_{}_{}".format(id0, id0, id1)][0].cpu().numpy()
            kpts1 = data["keypoints{}_{}_{}".format(id1, id0, id1)][0].cpu().numpy()
        matches = result[matches_key][0].cpu().numpy()
        intr0, intr1 = data["intr" + str(id0)][0].cpu().numpy(), data["intr" + str(id1)][0].cpu().numpy()
        confidence = result["conf_scores_{}_{}".format(id0, id1)][0].cpu().numpy()
        valid = (matches >= 0) & np.all(confidence > conf_thresh, -1)
        pair_wise_data["mkpts{}_{}_{}".format(id0, id0, id1)] = kpts0[valid]
        pair_wise_data["mkpts{}_{}_{}".format(id1, id0, id1)] = kpts1[matches[valid]]
        confidence = confidence[valid]
        pair_wise_data["conf{}_{}_{}".format(id0, id0, id1)] = confidence
        pair_wise_data["conf{}_{}_{}".format(id1, id0, id1)] = confidence
        pair_wise_data["intr{}".format(id0)] = intr0
        pair_wise_data["intr{}".format(id1)] = intr1

    for id0, id1 in _all_pairs(n_images):
        k0, k1 = "mkpts{}_{}_{}".format(id0, id0, id1), "mkpts{}_{}_{}".format(id1, id0, id1)
        if k0 not in pair_wise_data:
            continue
        success, R, t, inliers = estimate_relative_pose_w8pt_ba(pair_wise_data["intr{}".format(id0)],
                                                                pair_wise_data["intr{}".format(id1)],
                                                                pair_wise_data[k0], pair_wise_data[k1],
                                                                pair_wise_data["conf{}_{}_{}".format(id0, id0, id1)])
        # the w8pt_ba mode counts the inliers but keeps every match (bundle_adjust_io.py:114-117)
        pair_wise_data["inlier_count{}_{}".format(id0, id1)] = inliers.sum() if success else 0
        if success:
            rel_pose = np.eye(4)
            rel_pose[:3, :3] = R
            rel_pose[:3, 3] = t
            pair_wise_data["rel_pose{}_{}".format(id0, id1)] = rel_pose

    extr, pairs_on_spanning_tree = _spanning_tree(n_images, pair_wise_data)
    reached = {0}
    for _ in range(n_images):
        for a, b in pairs_on_spanning_tree:
            if a in reached or b in reached:
                reached.update((a, b))
    for v in sorted(reached):
        pair_wise_data["abs_init_pose{}".format(v)] = np.linalg.inv(extr[v])

    if file_path is not None:
        with open(file_path, 'w') as f:
            for id in range(n_images):
                R = extr[id, :3, :3]
                f.write(",".join([str(id)] + [repr(float(R[r, c])) for c in range(3) for r in range(3)]) + "\n")
            for id0, id1 in _all_pairs(n_images):
                rel_pose_key = "rel_pose{}_{}".format(id0, id1)
                if rel_pose_key not in pair_wise_data:
                    continue
                if pair_wise_data["inlier_count{}_{}".format(id0, id1)] >= MIN_INLIERS or (id0, id1) in pairs_on_spanning_tree:
                    T_021 = pair_wise_data[rel_pose_key]
                    R_021 = T_021[:3, :3]
                    t_021 = -R_021.transpose() @ T_021[:3, 3]      # position of camera id1 in camera id0's frame
                    f.write(",".join([str(id0), str(id1)] + [repr(float(R_021[r, c])) for c in range(3) for r in range(3)] +
                                     [repr(float(x)) for x in t_021]) + "\n")
    pair_wise_data["pairs_on_spanning_tree"] = pairs_on_spanning_tree
    return pair_wise_data


def _pairwise_arrays(n_images, pair_wise_data):
    """Padded per-pair arrays of the pairwise problem: normalised observations, raw confidences, counts."""
    pairs = _all_pairs(n_images)
    P = len(pairs)
    n_max = max([1] + [pair_wise_data["mkpts{}_{}_{}".format(a, a, b)].shape[0] for a, b in pairs
                       if "mkpts{}_{}_{}".format(a, a, b) in pair_wise_data])
    n_pad = (n_max + 63) // 64 * 64
    xa = np.zeros((1, P, n_pad, 2), np.float32)
    xb = np.zeros((1, P, n_pad, 2), np.float32)
    cf = np.zeros((1, P, n_pad), np.float32)
    nv = np.zeros((1, P), np.int32)
    norm = {}
    for p, (id0, id1) in enumerate(pairs):
        k0 = "mkpts{}_{}_{}".format(id0, id0, id1)
        if k0 not in pair_wise_data:
            continue
        mkpts0, mkpts1 = pair_wise_data[k0], pair_wise_data["mkpts{}_{}_{}".format(id1, id0, id1)]
        intr0, intr1 = pair_wise_data["intr{}".format(id0)], pair_wise_data["intr{}".format(id1)]
        mkpts0 = (mkpts0 - intr0[[0, 1], [2, 2]][None]) / intr0[[0, 1], [0, 1]][None]
        mkpts1 = (mkpts1 - intr1[[0, 1], [2, 2]][None]) / intr1[[0, 1], [0, 1]][None]
        n = mkpts0.shape[0]
        xa[0, p, :n], xb[0, p, :n] = mkpts0, mkpts1
        cf[0, p, :n] = pair_wise_data["conf{}_{}_{}".format(id0, id0, id1)].reshape(n)
        nv[0, p] = n
        norm[(id0, id1)] = (mkpts0, mkpts1)
    return pairs, n_pad, xa, xb, cf, nv, norm


def _triangulate(n_images, pairs, n_pad, xa, xb, nv, extrinsics):
    lib = _lib.lib()
    P = len(pairs)
    pa = (C.c_int * P)(*[a for a, _ in pairs])
    pb = (C.c_int * P)(*[b for _, b in pairs])
    d_xa, d_xb, d_nv = _cuda(xa), _cuda(xb), _cuda(nv)
    d_e = _cuda(np.asarray(extrinsics, np.float64).reshape(1, n_images, 4, 4))
    pts = torch.empty(1, P, n_pad, 3, dtype=torch.float64, device='cuda')
    _lib.check(lib.mvm_triangulate_pairs(pa, pb, n_images, P, 1, n_pad, _lib.ptr(d_xa), _lib.ptr(d_xb), _lib.ptr(d_nv),
                                         _lib.ptr(d_e), _lib.ptr(pts), _lib.stream_ptr()), 'mvm_triangulate_pairs')
    return pts[0].cpu().numpy()


def write_bundle_adjust_problem(n_images, pair_wise_data, extrinsics, file_path):
    """`ba_in.csv` exactly as the reference lays it out (bundle_adjust_io.py:193-259): header, two observations
    per match (first all of id0, then all of id1, pair by pair), cameras, points."""
    extrinsics = np.asarray(extrinsics)
    if extrinsics.ndim != 3:
        extrinsics = np.array([np.eye(4) for _ in range(n_images)])
    pairs, n_pad, xa, xb, cf, nv, norm = _pairwise_arrays(n_images, pair_wise_data)
    pts = _triangulate(n_images, pairs, n_pad, xa, xb, nv, extrinsics)
    observations_img_id, observations_pt_id, observations_xyc, points_in_3d = [], [], [], []
    n_3d_pts = 0
    for p, (id0, id1) in enumerate(pairs):
        if (id0, id1) not in norm:
            continue
        n = int(nv[0, p])
        conf = pair_wise_data["conf{}_{}_{}".format(id0, id0, id1)]
        for id, mkpts in zip((id0, id1), norm[(id0, id1)]):
            observations_img_id.append(np.full(n, id, dtype=int))
            observations_pt_id.append(np.arange(n_3d_pts, n_3d_pts + n, dtype=int))
            observations_xyc.append(np.concatenate((mkpts, conf), -1))
        n_3d_pts += n
        points_in_3d.append(pts[p, :n])
    observations_img_id = np.concatenate(observations_img_id, 0)
    observations_pt_id = np.concatenate(observations_pt_id, 0)
    observations_xyc = normalize_confidences(np.concatenate(observations_xyc, 0))
    points_in_3d = np.concatenate(points_in_3d, 0)
    with open(file_path, 'w') as f:
        f.write("{},{},{},{},{},{},{},{}\n".format(n_images, 0, n_3d_pts, 2 * n_3d_pts, 1., 1., 0., 0.))
        for id, pt_id, kpt in zip(observations_img_id, observations_pt_id, observations_xyc):
            f.write(",".join([str(id), str(pt_id)] + [repr(float(x)) for x in kpt]) + "\n")
        for id in range(n_images):
            R, t = extrinsics[id, :3, :3], extrinsics[id, :3, 3]
            f.write(",".join([repr(float(R[r, c])) for c in range(3) for r in range(3)] + [repr(float(x)) for x in t]) + "\n")
        for pt_3d in points_in_3d:
            f.write("{},{},{}\n".format(repr(float(pt_3d[0])), repr(float(pt_3d[1])), repr(float(pt_3d[2]))))


def read_bundle_adjust_result(file_path):
    """12 fields per camera: rotation column-major, translation; world->cam (bundle_adjust_io.py:261-273)."""
    extrinsics = []
    with open(file_path, "r") as f:
        for line in f:
            w = [float(x) for x in line.split(',')]
            T = np.eye(4)
            T[:3, :3] = np.array(w[:9]).reshape(3, 3).T
            T[:3, 3] = w[9:12]
            extrinsics.append(T)
    return extrinsics


def ba_initialize(n_images, pair_wise_data):
    """In-process `ba_initializer` (ba_init.cpp:77-91) on the pairs `initialize_bundle_adjust` would write."""
    lib = _lib.lib()
    pairs = _all_pairs(n_images)
    P = len(pairs)
    T_rel = np.zeros((1, P, 4, 4), np.float32)
    edge = np.zeros((1, P), np.uint8)
    on_tree = pair_wise_data.get("pairs_on_spanning_tree", [])
    for p, (id0, id1) in enumerate(pairs):
        key = "rel_pose{}_{}".format(id0, id1)
        if key in pair_wise_data and (pair_wise_data["inlier_count{}_{}".format(id0, id1)] >= MIN_INLIERS or (id0, id1) in on_tree):
            T_rel[0, p] = pair_wise_data[key]
            edge[0, p] = 1
    extr_tree = np.array([np.linalg.inv(pair_wise_data["abs_init_pose{}".format(v)]) if "abs_init_pose{}".format(v) in pair_wise_data
                          else np.eye(4) for v in range(n_images)])[None]
    pa = (C.c_int * P)(*[a for a, _ in pairs])
    pb = (C.c_int * P)(*[b for _, b in pairs])
    d_T, d_e, d_x = _cuda(T_rel), _cuda(edge), _cuda(extr_tree, torch.float64)
    out = torch.empty(1, n_images, 4, 4, dtype=torch.float64, device='cuda')
    _lib.check(lib.mvm_ba_initialize(pa, pb, n_images, P, 1, 64, _lib.ptr(d_x), _lib.ptr(d_T), _lib.ptr(d_e), _lib.ptr(d_e),
                                     None, 0, _lib.ptr(out), None, _lib.stream_ptr()), 'mvm_ba_initialize')
    return out[0].cpu().numpy()


def solve_bundle_adjust(n_images, pair_wise_data, extrinsics, max_iterations=50):
    """In-process `bundle_adjuster` on the problem `write_bundle_adjust_problem` would write.  Returns the list
    of world->cam 4x4 extrinsics `read_bundle_adjust_result` would return."""
    lib = _lib.lib()
    extrinsics = np.asarray(extrinsics)
    if extrinsics.ndim != 3:
        extrinsics = np.array([np.eye(4) for _ in range(n_images)])
    pairs, n_pad, xa, xb, cf, nv, _ = _pairwise_arrays(n_images, pair_wise_data)
    P = len(pairs)
    pa = (C.c_int * P)(*[a for a, _ in pairs])
    pb = (C.c_int * P)(*[b for _, b in pairs])
    d_xa, d_xb, d_cf, d_nv = _cuda(xa), _cuda(xb), _cuda(cf), _cuda(nv)
    d_e = _cuda(extrinsics.reshape(1, n_images, 4, 4), torch.float64)
    out32 = torch.empty(1, n_images, 4, 4, dtype=torch.float32, device='cuda')
    out64 = torch.empty(1, n_images, 4, 4, dtype=torch.float64, device='cuda')
    nbytes = lib.mvm_mvba_workspace_bytes(n_images, P, 1, n_pad)
    ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
    _lib.check(lib.mvm_multi_view_ba_ex(pa, pb, n_images, P, 1, n_pad, _lib.ptr(d_xa), _lib.ptr(d_xb), _lib.ptr(d_cf),
                                        _lib.ptr(d_nv), _lib.ptr(d_e), None, 0, _lib.ptr(out32), _lib.ptr(out64),
                                        int(max_iterations), None, None, _lib.ptr(ws), nbytes, _lib.stream_ptr()),
               'mvm_multi_view_ba_ex')
    return [T for T in out64[0].cpu().numpy()]


def solve(n_images, data, result, conf_thresh=0.):
    """eval_bundle_adjust (eval_multi_view.py:21-51) without files or subprocesses: pairwise poses, spanning
    tree, rotation averaging + LUD positions, global bundle adjustment.  Returns [n_images] 4x4 extrinsics."""
    pair_wise_data = initialize_bundle_adjust(n_images, data, result, None, conf_thresh=conf_thresh)
    extrinsics = ba_initialize(n_images, pair_wise_data)
    return solve_bundle_adjust(n_images, pair_wise_data, extrinsics)
