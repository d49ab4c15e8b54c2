"""GPU time of mvm_ransac_essential (CUDA events, after warm-up) at the cfg2 (32 pairs x 1024 matches) and cfg4
(8 pairs x 2048 matches) shapes on synthetic scenes with 30 % and 60 % outliers and 1 px noise, the iterations the
RANSAC loop used, and OpenCV's findEssentialMat + recoverPose per pair on the CPU on the same scenes for context (when
cv2 is installed).  Writes profiles/ransac_h100.json with the card name and power limit.

    python tools/ransac_timing.py [--out profiles/ransac_h100.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from e2e_multi_view_matching_b200 import _lib  # noqa: E402
from oracle import pose as P  # noqa: E402


def _scenes(B, n, outlier, seed0):
    k0 = np.zeros((B, n, 2), np.float32)
    k1 = np.zeros((B, n, 2), np.float32)
    intr = np.zeros((B, 4), np.float32)
    for b in range(B):
        sc = P.make_two_view_scene(seed0 + b, n, outlier_frac=outlier, noise_px=1.0)
        k0[b], k1[b] = sc['kpts0'][0], sc['kpts1'][0]
        K = sc['intr'][0]
        intr[b] = [K[0, 0], K[1, 1], K[0, 2], K[1, 2]]
    return k0, k1, intr


def _gpu(k0, k1, intr, reps=20):
    dev = torch.device('cuda')
    B, n = k0.shape[:2]
    a = [torch.from_numpy(x).to(dev) for x in (k0, k1, intr)]
    outs = [torch.empty(B, 16, device=dev), torch.empty(B, n, 2, device=dev), torch.empty(B, n, 2, device=dev),
            torch.empty(B, n, dtype=torch.uint8, device=dev), torch.empty(B, dtype=torch.int32, device=dev),
            torch.empty(B, 10, 9, dtype=torch.float64, device=dev), torch.empty(B, dtype=torch.int32, device=dev),
            torch.empty(B, dtype=torch.int32, device=dev), torch.empty(B, dtype=torch.uint8, device=dev)]
    L = _lib.lib()

    def launch():
        _lib.check(L.mvm_ransac_essential(_lib.ptr(a[0]), _lib.ptr(a[1]), _lib.ptr(a[2]), _lib.ptr(a[2]), B, n, None, 1.0,
                                          0.99999, 1000, 0, *[_lib.ptr(o) for o in outs], _lib.stream_ptr()),
                   'mvm_ransac_essential')
    for _ in range(3):
        launch()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        launch()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    it = outs[7].cpu().numpy()
    return {'ms_median': float(np.median(ms)), 'ms_min': float(np.min(ms)),
            'iterations_mean': float(it.mean()), 'iterations_max': int(it.max()),
            'success': int(outs[8].sum())}


def _cv2(k0, k1, intr):
    try:
        import cv2
    except ImportError:
        return None
    ts = []
    for b in range(len(k0)):
        fx, fy, cx, cy = intr[b].astype(np.float64)
        x0 = (k0[b] - [cx, cy]) / [fx, fy]
        x1 = (k1[b] - [cx, cy]) / [fx, fy]
        t0 = time.perf_counter()
        E, m = cv2.findEssentialMat(x0, x1, np.eye(3), threshold=1.0 / fx, prob=0.99999, method=cv2.RANSAC)
        if E is not None:
            cv2.recoverPose(E[:3], x0, x1, np.eye(3), 1e9, mask=m)
        ts.append(time.perf_counter() - t0)
    return {'ms_per_pair_median': 1e3 * float(np.median(ts)), 'cpu_threads': cv2.getNumThreads()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'ransac_h100.json'))
    opt = ap.parse_args()
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res = {'device': torch.cuda.get_device_name(0), 'nvidia_smi_name_power_limit': q[0] if q else None, 'runs': []}
    for name, B, n in (('cfg2', 32, 1024), ('cfg4', 8, 2048)):
        for outlier in (0.3, 0.6):
            k0, k1, intr = _scenes(B, n, outlier, 1000)
            r = {'shape': name, 'pairs': B, 'matches': n, 'outlier_frac': outlier, 'noise_px': 1.0,
                 'gpu': _gpu(k0, k1, intr), 'opencv_cpu': _cv2(k0, k1, intr)}
            res['runs'].append(r)
            print(json.dumps(r))
    os.makedirs(os.path.dirname(opt.out), exist_ok=True)
    with open(opt.out, 'w') as f:
        json.dump(res, f, indent=2)
    print(json.dumps({'device': res['device'], 'power': res['nvidia_smi_name_power_limit']}))


if __name__ == '__main__':
    main()
