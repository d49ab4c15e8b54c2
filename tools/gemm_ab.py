"""Per-shape timing of the fp16x3 layer GEMM (gemm_wg_kernel<128, 3, W_F16>) at the shapes of one cfg3 step
(14 tuples x 5 views x 1024 keypoints = 71680 rows; the confidence head runs on twice as many rows).  'qkv' is the
projection as a plain fp32 [M, 768] output; 'qkv.planes' is the matcher's own launch (ops.qkv_projection, planes='fp16'):
Q in fp32, K and V as the fp16 hi / lo planes of the attention.

Kernel durations come from CUPTI (torch.profiler, CUDA activities) with the L2 flushed before every launch.  For each
shape the script prints the median duration, the algorithmic rate (2 M N K per launch; fp16x3 issues three tensor-core
passes over it) and its share of the fp16x3 ceiling: SMs x 4096 f16 FLOP/clk x the SM clock sampled during the run / 3.

    python tools/gemm_ab.py [--reps 20] [--json out.json]
"""
import argparse, json, os, subprocess, sys, tempfile, threading
import numpy as np
import torch
from torch.profiler import profile, ProfilerActivity

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from e2e_multi_view_matching_b200 import ops  # noqa: E402

M = 14 * 5 * 1024
# name, rows, K1, K2 (K-split concat), N, epilogue
SHAPES = [('qkv', M, 256, 0, 768, 'bias'),
          ('mlp.0', M, 256, 256, 512, 'concat+bias+relu'),
          ('mlp.2', M, 512, 0, 256, 'bias+residual'),
          ('conf.0', 2 * M, 512, 0, 512, 'bias+relu'),
          ('conf.1', 2 * M, 512, 0, 256, 'bias'),
          ('qkv.planes', M, 256, 0, 768, 'bias+fp16 planes')]


def smi(query):
    r = subprocess.run(['nvidia-smi', '--query-gpu=' + query, '--format=csv,noheader,nounits', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return r.stdout.strip()


class ClockSampler(threading.Thread):
    def __init__(self):
        super().__init__(daemon=True)
        self.samples, self.stop = [], threading.Event()

    def run(self):
        while not self.stop.wait(0.1):
            try:
                self.samples.append(float(smi('clocks.sm')))
            except ValueError:
                pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--json', default='')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'gemm_ab.py times the GPU kernel: no CUDA device'
    dev = torch.cuda.get_device_properties(0)
    card, power = smi('name'), smi('power.limit')
    g = torch.Generator().manual_seed(0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    cases = []
    for name, rows, K1, K2, N, epi in SHAPES:
        a = torch.randn(rows, K1, generator=g).cuda()
        a2 = torch.randn(rows, K2, generator=g).cuda() if K2 else None
        w = (torch.randn(N, K1 + K2, generator=g) / 16).cuda()
        b = torch.randn(N, generator=g).cuda()
        r = torch.randn(rows, N, generator=g).cuda() if 'residual' in epi else None
        cases.append((name, rows, K1 + K2, N, epi, dict(a=a, w=w, bias=b, a2=a2, residual=r, relu='relu' in epi)))
    qkv_out = torch.empty(M, 768, device='cuda')

    def run(name, kw):
        if name == 'qkv.planes':
            ops.qkv_projection(kw['a'], kw['w'], kw['bias'], 1024, planes='fp16', out=qkv_out)
        else:
            ops.linear(tc_passes='h16', **kw)
    for name, *_, kw in cases:                  # warm-up: module load, tensor maps
        for _ in range(3):
            run(name, kw)
    torch.cuda.synchronize()
    sampler = ClockSampler()
    sampler.start()
    durs = {}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, *_, kw in cases:
            for _ in range(args.reps):
                flush.zero_()
                run(name, kw)
        torch.cuda.synchronize()
    sampler.stop.set()
    sampler.join()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, 'trace.json')
        prof.export_chrome_trace(path)
        ev = [e for e in json.load(open(path))['traceEvents'] if e.get('cat') == 'kernel' and 'gemm_wg_kernel' in e['name']]
    ev.sort(key=lambda e: e['ts'])
    assert len(ev) == args.reps * len(cases), 'expected %d gemm_wg_kernel launches, found %d' % (args.reps * len(cases), len(ev))
    clock_mhz = float(np.median(sampler.samples)) if sampler.samples else float(smi('clocks.sm'))
    ceiling = dev.multi_processor_count * 4096 * clock_mhz * 1e6 / 3
    print('%s, power limit %s W, %d SMs, SM clock sampled %.0f MHz: fp16x3 ceiling %.0f TFLOP/s algorithmic'
          % (card, power, dev.multi_processor_count, clock_mhz, ceiling / 1e12))
    print('%-8s %-22s %-18s %10s %10s %8s' % ('gemm', 'M x N x K', 'epilogue', 'median us', 'TFLOP/s', 'ceiling'))
    rows = []
    for i, (name, m, K, N, epi, _) in enumerate(cases):
        d = np.array([e['dur'] for e in ev[i * args.reps:(i + 1) * args.reps]])
        us = float(np.median(d))
        tflops = 2.0 * m * N * K / us / 1e6
        rows.append(dict(gemm=name, M=m, N=N, K=K, epilogue=epi, median_us=round(us, 1), min_us=round(float(d.min()), 1),
                         max_us=round(float(d.max()), 1), tflops=round(tflops, 1), share_of_ceiling=round(tflops * 1e12 / ceiling, 3)))
        print('%-8s %-22s %-18s %10.1f %10.1f %8.3f' % (name, '%d x %d x %d' % (m, N, K), epi, us, tflops, tflops * 1e12 / ceiling))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(dict(card=card, power_limit_w=power, sms=dev.multi_processor_count, sm_clock_mhz=clock_mhz,
                           reps=args.reps, shapes=rows), f, indent=1)


if __name__ == '__main__':
    main()
