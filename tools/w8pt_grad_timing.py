"""GPU time of the weighted eight-point forward (mvm_w8pt) and its backward with respect to the confidences
(mvm_w8pt_backward), CUDA events after warm-up, at the cfg5 shape (8 pairs x 400 matches, choose_closest as in the
stage-2 training) and at 32 pairs x 1024 matches, on synthetic scenes with 30 % outliers.  Writes
profiles/w8pt_grad_h100.json with the card name and power limit.

    python tools/w8pt_grad_timing.py [--out profiles/w8pt_grad_h100.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from e2e_multi_view_matching_b200 import _lib  # noqa: E402
from oracle import pose as P  # noqa: E402


def _time(fn, reps=50):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return {'ms_median': float(np.median(ms)), 'ms_min': float(np.min(ms))}


def _run(B, n, choose_closest):
    dev = torch.device('cuda')
    scs = [P.make_two_view_scene(2000 + b, n, outlier_frac=0.3) for b in range(B)]
    k0, k1, K, c, Tg = (torch.from_numpy(np.concatenate([s[k] for s in scs]).astype(np.float32)).to(dev)
                        for k in ('kpts0', 'kpts1', 'intr', 'conf', 'T_021'))
    i4 = torch.stack([K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2]], -1).contiguous()
    c = c.reshape(B, n).contiguous()
    T = torch.empty(B, 16, device=dev)
    k0n, k1n = torch.empty(B, n, 2, device=dev), torch.empty(B, n, 2, device=dev)
    cn = torch.empty(B, n, device=dev)
    pos = torch.empty(B, n, dtype=torch.uint8, device=dev)
    F = torch.empty(B, 9, device=dev)
    gT = torch.randn(B, 16, device=dev)
    gcn = torch.randn(B, n, device=dev)
    gc = torch.empty(B, n, device=dev)
    tg = Tg.reshape(B, 16).contiguous() if choose_closest else None
    L = _lib.lib()
    p = _lib.ptr

    def fwd():
        _lib.check(L.mvm_w8pt(p(k0), p(k1), p(i4), p(i4), p(c), B, n, p(tg), int(choose_closest), 0, p(T), p(k0n), p(k1n),
                              p(cn), p(pos), None, p(F), None, None, _lib.stream_ptr()), 'mvm_w8pt')

    def bwd():
        _lib.check(L.mvm_w8pt_backward(p(k0), p(k1), p(i4), p(i4), p(c), B, n, p(tg), int(choose_closest), p(T), p(gT),
                                       p(gcn), p(gc), _lib.stream_ptr()), 'mvm_w8pt_backward')
    fwd()
    return {'forward': _time(fwd), 'backward': _time(bwd), 'grad_finite': bool(torch.isfinite(gc).all())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'w8pt_grad_h100.json'))
    opt = ap.parse_args()
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res = {'device': torch.cuda.get_device_name(0), 'nvidia_smi_name_power_limit': q[0] if q else None, 'runs': []}
    for name, B, n in (('cfg5', 8, 400), ('b32_n1024', 32, 1024)):
        for cc in (True, False):
            r = {'shape': name, 'pairs': B, 'matches': n, 'choose_closest': cc, 'outlier_frac': 0.3, **_run(B, n, cc)}
            res['runs'].append(r)
            print(json.dumps(r))
    os.makedirs(os.path.dirname(opt.out), exist_ok=True)
    with open(opt.out, 'w') as f:
        json.dump(res, f, indent=2)
    print(json.dumps({'device': res['device'], 'power': res['nvidia_smi_name_power_limit']}))


if __name__ == '__main__':
    main()
