"""Magnitudes of the operands of every tensor-core GEMM of the matcher, measured on the CPU (DESIGN.md section 3, the
fp16x3 operand range).  Authoring container only: the SuperPoint -> matcher chain runs the reference's SuperPoint.

The GEMMs are the 1x1 convolutions of oracle/matcher_torch (F.conv1d, recorded by wrapping it): the keypoint encoder's
128 -> 256 and 256 -> 256 convolutions (the three before them run in kenc.cu), Q / K / V, the merge (folded into mlp.0 by
packing.py: its input is mlp.0's message half) and mlp.0 / mlp.3 of every GNN layer, final_proj, and the confidence
head's GEMMs.  A is the convolution's input, W its weight;
the packed fp16 planes hold 64 W.  Sources:
  goldens  every tests/golden/matcher_*.npz fixture but the full-size ones (the fixtures' seeded synthetic weights)
  chain    tests/golden/native_chain_landscape_portrait.npz: the reference SuperPoint on the fixture's two crops, whose
           descriptors are L2-normalised, into the pairwise matcher
Per (source, GEMM): median and max of |a|, the shares of elements that are exactly zero (post-ReLU inputs: split exactly),
below 2^-3 (lo = fp16(a - hi) subnormal) and below 2^-8 (where the fp16x3 GEMM left its bound in
tests/test_gemm_shapes_gpu.py), and the median of 64 |W| with its share below 2^-3.  Trained weights are not measured.

    python oracle/measure_gemm_operands.py [--json out.json]
"""
import argparse
import collections
import glob
import json
import os
import re
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
REF = '/root/reference'

GROUPS = [(r'kenc\.encoder\.9\.', 'kenc 128->256'), (r'kenc\.encoder\.12\.', 'kenc 256->256'),
          (r'attn\.proj\.', 'qkv'), (r'attn\.merge\.', 'merge'), (r'mlp\.0\.', 'mlp.0'), (r'mlp\.3\.', 'mlp.3'),
          (r'final_proj\.', 'final_proj'), (r'conf_mlp\.', 'confidence head')]


def record(sd, run):
    """Run `run()` with F.conv1d wrapped; -> {GEMM group: ([|a| arrays], [|W| arrays])} for the convolutions whose weight
    is one of sd's (matched by value)."""
    import oracle.matcher_torch as MT
    by_shape = collections.defaultdict(list)
    for k, v in sd.items():
        if k.endswith('.weight') and np.ndim(v) == 3:
            by_shape[tuple(np.shape(v))].append(k)
    out = collections.defaultdict(lambda: ([], []))
    orig = MT.F

    class Shim:
        def __getattr__(self, name):
            return getattr(F, name)

        @staticmethod
        def conv1d(x, w, b=None, *a, **kw):
            wn = w.detach().cpu().numpy()
            key = next((k for k in by_shape.get(tuple(wn.shape), []) if np.array_equal(np.asarray(sd[k]), wn)), None)
            group = next((g for p, g in GROUPS if key and re.search(p, key)), None)
            if group:
                out[group][0].append(x.detach().abs().double().numpy().ravel())
                out[group][1].append(w.detach().abs().double().numpy().ravel())
            return F.conv1d(x, w, b, *a, **kw)
    MT.F = Shim()
    try:
        run()
    finally:
        MT.F = orig
    return out


def stats(rec):
    res = {}
    for g, (xs, ws) in rec.items():
        a, w = np.concatenate(xs), 64.0 * np.concatenate(ws)
        res[g] = dict(a_median=float(np.median(a)), a_max=float(a.max()), a_zero=float((a == 0).mean()),
                      a_below_2m3=float((a < 2.0 ** -3).mean()), a_below_2m8=float((a < 2.0 ** -8).mean()),
                      w64_median=float(np.median(w)), w64_below_2m3=float((w < 2.0 ** -3).mean()))
    return res


def merge(recs):
    out = collections.defaultdict(lambda: ([], []))
    for r in recs:
        for g, (xs, ws) in r.items():
            out[g][0].extend(xs)
            out[g][1].extend(ws)
    return out


def goldens():
    from oracle.matcher_torch import matcher_forward
    from tests.util import load_case, case_inputs
    recs = []
    for p in sorted(glob.glob(os.path.join(ROOT, 'tests', 'golden', 'matcher_*.npz'))):
        name = os.path.basename(p)[len('matcher_'):-4]
        if name.startswith('full'):
            continue
        meta, _ = load_case(name)
        sd, data = case_inputs(meta)
        cfg = {'GNN_layers': meta['layers'], 'multi_frame_matching': meta['multi']}
        recs.append(record(sd, lambda: matcher_forward(sd, cfg, data)))
    return merge(recs)


def chain():
    from oracle import make_native_sizes_golden as G
    from oracle.matcher_torch import matcher_forward
    if REF not in sys.path:
        sys.path.insert(0, REF)
    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'native_chain_landscape_portrait.npz'), allow_pickle=True)
    meta = json.loads(str(z['meta']))
    sp = G._ref_superpoint(meta['sp_config'], meta['sp_wseed'])
    data = {'ids': [0, 1]}
    for i, img in enumerate(G.chain_images(meta)):
        with torch.no_grad():
            p = sp({'image': [torch.from_numpy(img)]})
        data.update({'keypoints%d' % i: p['keypoints'][0][None].numpy(), 'scores%d' % i: p['scores'][0][None].numpy(),
                     'descriptors%d' % i: p['descriptors'][0][None].numpy(), 'image%d' % i: img})
    d = np.abs(np.concatenate([data['descriptors0'].ravel(), data['descriptors1'].ravel()]))
    desc = dict(median=float(np.median(d)), max=float(d.max()), below_2m3=float((d < 2.0 ** -3).mean()),
                below_2m8=float((d < 2.0 ** -8).mean()))
    sd = G.chain_matcher_state_dict(meta)
    cfg = {'GNN_layers': meta['layers'], 'multi_frame_matching': False}
    return record(sd, lambda: matcher_forward(sd, cfg, data)), desc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--json', default='')
    args = ap.parse_args()
    rec_c, desc = chain()
    res = {'goldens': stats(goldens()), 'chain': stats(rec_c), 'chain_descriptors': desc}
    for src in ('goldens', 'chain'):
        for g, s in res[src].items():
            print('%-8s %-18s |a| median %.3g max %.3g zero %.2f <2^-3 %.2f <2^-8 %.3f   64|W| median %.3g <2^-3 %.3f'
                  % (src, g, s['a_median'], s['a_max'], s['a_zero'], s['a_below_2m3'], s['a_below_2m8'],
                     s['w64_median'], s['w64_below_2m3']))
    print('chain descriptors', {k: round(v, 4) for k, v in desc.items()})
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
