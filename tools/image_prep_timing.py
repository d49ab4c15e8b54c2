"""Time the GPU training-image preparation (mvm_image_prep, csrc/image_prep.cu) against the reference's CPU transform
chain (MatchingDataset.__getitem__ :182-211 as oracle/image_prep.py restates it with torchvision), on two batches:
  - ScanNet, cfg5-shaped: 40 images of 968 x 1296 -> 2-row pad -> 480 x 640, ColorJitter 0.2 (two launches);
  - MegaDepth-like: 8 images of 1064 x 1600, random square crops (1064 x 1064), no resize, no jitter (one launch).
Records the CUDA-event time of the preparation alone (parameters already on the device), of prepare_images from a
pinned host batch (parameter checks + host->device copies + launch), of the pinned host->device copy of the uint8
batch alone, and the CPU chain per image at 1 thread and at all threads, with the card name and power limit read in the
same run.

    python tools/image_prep_timing.py [--out profiles/image_prep_h100.json] [--reps 20] [--cpu_images 3]
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

from e2e_multi_view_matching_b200 import _lib, image_prep as IP  # noqa: E402
from oracle import image_prep as R  # noqa: E402


def _event_ms(fn, reps, warmup):
    for _ in range(warmup):
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
    return float(np.median(ms)), float(np.min(ms))


def _workload(name, rng):
    if name == 'scannet_cfg5':
        n, H, W, out = 40, 968, 1296, (480, 640)
        geom = np.tile([0, 0, H, W, 2, 2], (n, 1))
        torch.manual_seed(0)
        params = [IP.color_jitter_params(0.2) for _ in range(n)]
        order = np.stack([p[0].numpy() for p in params])
        factors = np.array([p[1:] for p in params], np.float64)
        crops = [None] * n
    else:
        n, H, W = 8, 1064, 1600
        offs = rng.integers(0, W - H + 1, n)
        geom = np.stack([[0, o, H, H, 0, 0] for o in offs])
        out, order, factors, params = (H, H), None, None, [None] * n
        crops = [(0, H, int(o), int(o) + H) for o in offs]
    rgb = torch.from_numpy(rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8))
    return rgb, geom, out, order, factors, params, crops


def _cpu_chain_ms(rgb, out, params, crops, k):
    """The reference's per-image chain (ToTensor .. rgb_to_grayscale) on the CPU, ms per image over k images."""
    t0 = time.perf_counter()
    for i in range(k):
        jp = None if params[i] is None else (params[i][0],) + tuple(params[i][1:])
        depth_shape = out if crops[i] is None else (rgb.shape[1], rgb.shape[2])
        R.prepare_image(rgb[i].numpy(), np.zeros(depth_shape, np.float32), np.eye(3, dtype=np.float32), crops[i], jp)
    return (time.perf_counter() - t0) * 1e3 / k


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'image_prep_h100.json'))
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--cpu_images', type=int, default=3)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit('image_prep_timing needs a CUDA device')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    rec = {'device': torch.cuda.get_device_name(0), 'nvidia_smi_name_power_limit_max_sm_clock': q.stdout.strip(),
           'torch': torch.__version__, 'host_cpus': os.cpu_count(), 'reps': args.reps, 'warmup': args.warmup,
           'workloads': []}
    rng = np.random.default_rng(0)
    L = _lib.lib()
    n_threads = torch.get_num_threads()
    for name in ('scannet_cfg5', 'megadepth_crop'):
        rgb, geom, out_size, order, factors, params, crops = _workload(name, rng)
        n, H, W = rgb.shape[:3]
        oh, ow = out_size
        pinned = rgb.pin_memory()
        dev = torch.empty_like(rgb, device='cuda')
        g_d = torch.from_numpy(geom.astype(np.int32)).cuda()
        o_d = None if order is None else torch.from_numpy(order.astype(np.int32)).cuda()
        f_d = None if factors is None else torch.from_numpy(factors).cuda()
        out = torch.empty(n, 1, oh, ow, device='cuda')
        ws = torch.empty(max(1, L.mvm_image_prep_workspace_bytes(n, oh, ow)), dtype=torch.uint8, device='cuda')
        dev.copy_(pinned)

        def kernel():
            _lib.check(L.mvm_image_prep(_lib.ptr(dev), n, H, W, _lib.ptr(g_d), _lib.ptr(o_d), _lib.ptr(f_d), oh, ow,
                                        _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), 'mvm_image_prep')

        k_med, k_min = _event_ms(kernel, args.reps, args.warmup)
        c_med, c_min = _event_ms(lambda: dev.copy_(pinned, non_blocking=True), args.reps, args.warmup)
        p_med, p_min = _event_ms(lambda: IP.prepare_images(pinned, geom, out_size, order, factors), args.reps,
                                 args.warmup)
        src_bytes = n * H * W * 3
        cpu = {}
        for threads in (1, n_threads):
            torch.set_num_threads(threads)
            cpu['threads_%d_ms_per_image' % threads] = _cpu_chain_ms(rgb, out_size, params, crops,
                                                                    min(args.cpu_images, n))
        torch.set_num_threads(n_threads)
        w = {'workload': name, 'images': n, 'source': [H, W], 'output': [oh, ow], 'jitter': order is not None,
             'launches': 2 if order is not None else 1,
             'prep_kernel_ms_median': k_med, 'prep_kernel_ms_min': k_min,
             'prepare_images_from_pinned_ms_median': p_med, 'prepare_images_from_pinned_ms_min': p_min,
             'h2d_uint8_pinned_ms_median': c_med, 'h2d_uint8_pinned_ms_min': c_min,
             'h2d_uint8_mb': src_bytes / 1e6, 'h2d_float_chw_mb_the_workers_shipped': src_bytes * 4 / 1e6,
             'h2d_gb_per_s': src_bytes / (c_med * 1e-3) / 1e9,
             'cpu_reference_chain': cpu,
             'cpu_reference_chain_batch_s_at_1_thread': cpu['threads_1_ms_per_image'] * n / 1e3}
        rec['workloads'].append(w)
        print(json.dumps(w))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(rec, f, indent=2)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
