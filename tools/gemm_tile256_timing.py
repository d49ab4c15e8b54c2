"""Timing of the 256-column tensor-core GEMM instances (gemm_wg_kernel<256, 1, W_RAW> and <256, 3, W_TF32>), which serve
the non-default paths: single-pass TF32 (math mode 1, mvm_linear_tc with n_pass 1) and the one-tile-per-CTA 3xTF32
schedule (gemm_kernel 0, gemm_tile 256).  Shapes are the matcher's layer GEMMs at one cfg3 step (71680 rows).

CUDA events around `--reps` back-to-back launches after a warm-up; the median of `--rounds` such windows is printed per
shape as microseconds per launch, one JSON line, with the GPU's name and power limit.

    python tools/gemm_tile256_timing.py [--reps 50] [--rounds 5]
"""
import argparse, json, os, subprocess, sys
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from e2e_multi_view_matching_b200 import _lib, ops  # noqa: E402

M = 14 * 5 * 1024
SHAPES = [('qkv', 256, 768), ('mlp.0', 512, 512), ('mlp.2', 512, 256)]      # name, K, N


def time_us(fn, reps, rounds):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) * 1e3 / reps)
    return sorted(out)[len(out) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    lib = _lib.lib()
    g = torch.Generator(device='cuda').manual_seed(0)
    res = {}
    for name, K, N in SHAPES:
        a = torch.randn(M, K, device='cuda', generator=g)
        w = torch.randn(N, K, device='cuda', generator=g) / 16
        b = torch.randn(N, device='cuda', generator=g)
        res[name + ' tf32 <256,1>'] = time_us(lambda: ops.linear(a, w, bias=b, tc_passes=1), args.reps, args.rounds)
        try:
            lib.mvm_debug_set_gemm_kernel(0)
            lib.mvm_debug_set_gemm_tile(256)
            res[name + ' 3xtf32 <256,3> one tile/CTA'] = time_us(
                lambda: ops.linear(a, w, bias=b, tc_passes=3, presplit=True), args.reps, args.rounds)
        finally:
            lib.mvm_debug_set_gemm_kernel(1)
            lib.mvm_debug_set_gemm_tile(256)
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                          str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    print(json.dumps({'gpu': smi, 'rows': M, 'us_per_launch': {k: round(v, 1) for k, v in res.items()}}))


if __name__ == '__main__':
    main()
