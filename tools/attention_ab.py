"""Per-launch timing of the attention kernel (attention_wg_kernel) at the shapes of one cfg3 layer: 14 tuples x 5 views
= 70 view slots of 1024 keypoints; a self layer attends 1024 queries to the 1024 keys of their own view, a cross layer
to the 4096 keys of the other four views.

The operand planes (fp16 hi / lo of K and V for fp16x3; V^T and the tf32 lo planes for 3xTF32) are built once, outside
the timed region, so only the kernel is timed: mvm_attention_h3 (fp16x3, the default) and mvm_attention_tc with one and
three tf32 passes.  Kernel durations come from CUPTI (torch.profiler, CUDA activities) with the L2 flushed before every
launch.  For each case the script prints the median duration, the algorithmic rate (4 N M 256 FLOP per view: Q K^T and
P V over four heads of 64) and its share of the fp16x3 ceiling: SMs x 4096 f16 FLOP/clk x the SM clock sampled during
the run / 3 (three tensor-core passes per product).

    python tools/attention_ab.py [--reps 20] [--json out.json]
"""
import argparse, ctypes, json, os, sys, tempfile
import numpy as np
import torch
from torch.profiler import profile, ProfilerActivity

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from e2e_multi_view_matching_b200 import _lib  # noqa: E402
from gemm_ab import smi, ClockSampler  # noqa: E402

B, T, N = 14, 5, 1024


def rn_tf32(x):
    """round to nearest (ties away) on the 13 mantissa bits tf32 drops: what the QKV GEMM epilogue writes"""
    return ((x.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--json', default='')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'attention_ab.py times the GPU kernel: no CUDA device'
    L = _lib.lib()
    dev = torch.cuda.get_device_properties(0)
    card, power = smi('name'), smi('power.limit')
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(B * T, N, 768, generator=g).cuda()
    out = torch.empty(B * T, N, 256, device='cuda')
    cnt = (ctypes.c_int * T)(*([N] * T))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')

    k, v = qkv[:, :, 256:512], qkv[:, :, 512:]
    kh, vh = k.half(), v.half()
    h3 = [t.reshape(-1, 256).contiguous() for t in (kh, (k - kh.float()).half(), vh, (v - vh.float()).half())]
    vt = v.transpose(1, 2).contiguous()                          # [views, 256, keys]
    qkv3 = qkv.clone()
    khi = rn_tf32(k.contiguous())
    qkv3[:, :, 256:512] = khi
    klo = rn_tf32(k - khi).reshape(-1, 256).contiguous()
    vthi = rn_tf32(vt)
    vtlo = rn_tf32(vt - vthi).contiguous()
    P = _lib.ptr

    def run_h3(cross):
        _lib.check(L.mvm_attention_h3(P(qkv), *[P(t) for t in h3], P(out), B, T, N, cnt, cross, _lib.stream_ptr()),
                   'mvm_attention_h3')

    def run_tc1(cross):
        _lib.check(L.mvm_attention_tc(P(qkv), P(vt), P(out), B, T, N, cnt, cross, 1, P(None), P(None),
                                      _lib.stream_ptr()), 'mvm_attention_tc')

    def run_tc3(cross):
        _lib.check(L.mvm_attention_tc(P(qkv3), P(vthi), P(out), B, T, N, cnt, cross, 3, P(klo), P(vtlo),
                                      _lib.stream_ptr()), 'mvm_attention_tc')

    cases = [('fp16x3', run_h3), ('tf32', run_tc1), ('3xtf32', run_tc3)]
    cases = [(mode, layer, fn, cross) for mode, fn in cases for layer, cross in (('self', 0), ('cross', 1))]
    for *_, fn, cross in cases:                 # warm-up: module load, tensor maps
        for _ in range(3):
            fn(cross)
    torch.cuda.synchronize()
    sampler = ClockSampler()
    sampler.start()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for *_, fn, cross in cases:
            for _ in range(args.reps):
                flush.zero_()
                fn(cross)
        torch.cuda.synchronize()
    sampler.stop.set()
    sampler.join()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, 'trace.json')
        prof.export_chrome_trace(path)
        ev = [e for e in json.load(open(path))['traceEvents']
              if e.get('cat') == 'kernel' and 'attention_wg_kernel' in e['name']]
    ev.sort(key=lambda e: e['ts'])
    assert len(ev) == args.reps * len(cases), \
        'expected %d attention_wg_kernel launches, found %d' % (args.reps * len(cases), len(ev))
    clock_mhz = float(np.median(sampler.samples)) if sampler.samples else float(smi('clocks.sm'))
    ceiling = dev.multi_processor_count * 4096 * clock_mhz * 1e6 / 3
    print('%s, power limit %s W, %d SMs, SM clock sampled %.0f MHz: fp16x3 ceiling %.0f TFLOP/s algorithmic'
          % (card, power, dev.multi_processor_count, clock_mhz, ceiling / 1e12))
    print('%-8s %-6s %-20s %10s %10s %8s' % ('mode', 'layer', 'views x N x keys', 'median ms', 'TFLOP/s', 'fp16x3'))
    rows = []
    for i, (mode, layer, _, cross) in enumerate(cases):
        keys = N * (T - 1) if cross else N
        d = np.array([e['dur'] for e in ev[i * args.reps:(i + 1) * args.reps]]) / 1e3
        ms = float(np.median(d))
        tflops = 4.0 * N * keys * 256 * B * T / ms / 1e9
        rows.append(dict(mode=mode, layer=layer, views=B * T, queries=N, keys=keys, median_ms=round(ms, 4),
                         min_ms=round(float(d.min()), 4), max_ms=round(float(d.max()), 4), tflops=round(tflops, 1),
                         share_of_fp16x3_ceiling=round(tflops * 1e12 / ceiling, 3)))
        print('%-8s %-6s %-20s %10.3f %10.1f %8.3f' % (mode, layer, '%d x %d x %d' % (B * T, N, keys), ms, tflops,
                                                       tflops * 1e12 / ceiling))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(dict(card=card, power_limit_w=power, sms=dev.multi_processor_count, sm_clock_mhz=clock_mhz,
                           reps=args.reps, cases=rows), f, indent=1)


if __name__ == '__main__':
    main()
