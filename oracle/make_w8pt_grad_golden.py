"""Generate tests/golden/w8pt_grad_*.npz: the gradient of the REFERENCE's estimate_relative_pose_w8pt with respect to
the confidences, by the reference's own autograd.

Run in the authoring container only (needs /root/reference):
    python -m oracle.make_w8pt_grad_golden
``oracle/ref_shim.py`` imports ``pose_optimization/two_view/estimate_relative_pose.py`` unmodified.  For each seeded
batch this script runs it in fp32 (what the reference ships) and in fp64 (``torch.set_default_dtype(float64)``), for
both branches (choose_closest against the true pose, and the cheirality vote), with four losses built from the
reference's ``compute_pose_error``: rotation, translation angle, both, and a random linear functional of
info["confidence"].  It calls ``.backward()`` and stores the inputs, the gradient reaching T021, the gradient of the
loss with respect to info["confidence"] as an output, and the gradient of the confidences.  It asserts that the numpy
restatement ``oracle.pose_grad.w8pt_conf_grad`` reproduces the fp64 gradients (this is what pins the oracle) and writes
``tests/golden/w8pt_grad_report.json`` with the fp32-vs-fp64 deviation of every item.

The cheirality branch is run one pair at a time: kornia 0.7.0 applies batch item 0's vote to every item of a batch
(``oracle/ref_shim.py``), the reference only calls that branch with one pair, and this engine selects per item.
"""
import importlib
import json
import os
import sys
import warnings

import numpy as np
import torch

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')

CASES = [
    # name, seeds (batch), matches, outlier fraction, zeroed (unmatched) rows per item, non-zero weights kept per item
    dict(name='n8_b2', seeds=[201, 202], n=8, outl=0.0),
    dict(name='n12_nz8_b2', seeds=[203, 204], n=12, outl=0.0, keep=[8, 8]),
    dict(name='n12_nz7_b2', seeds=[205, 206], n=12, outl=0.0, keep=[7, None]),
    dict(name='n40_b4', seeds=[207, 208, 209, 210], n=40, outl=0.3),
    dict(name='n150_b3', seeds=[211, 212, 213], n=150, outl=0.3, zero=0.1),
    dict(name='n400_b4', seeds=[214, 215, 216, 217], n=400, outl=0.3, zero=0.05),
    dict(name='n1024_b2', seeds=[218, 219], n=1024, outl=0.3),
    dict(name='n2048_b1', seeds=[220], n=2048, outl=0.3),
    dict(name='small_baseline_b2', seeds=[221, 222], n=150, outl=0.3, baseline=0.01),
]
LOSSES = ('rot', 'transl', 'both', 'conf')
BRANCHES = ('closest', 'vote')


def _scene(seed, n, outl, baseline=None):
    from oracle import pose as P
    if baseline is None:
        return P.make_two_view_scene(seed, n, outlier_frac=outl)
    # small baseline, small rotation: an ill-conditioned eight-point problem
    rng = np.random.default_rng(seed)
    f, w, h = 577.87, 640, 480
    K = np.array([[f, 0, (w - 1) / 2], [0, f, (h - 1) / 2], [0, 0, 1]])
    axis = rng.standard_normal(3)
    R = P.rodrigues(axis / np.linalg.norm(axis) * np.deg2rad(2.0))
    t = rng.standard_normal(3)
    t *= baseline / np.linalg.norm(t)
    uv = rng.uniform([0, 0], [w, h], (n, 2))
    X = np.linalg.solve(K, np.concatenate([uv, np.ones((n, 1))], 1).T).T * rng.uniform(2, 6, (n, 1))
    X1 = X @ R.T + t
    uv1 = (X1 @ K.T)[:, :2] / X1[:, 2:]
    k0 = uv + 0.5 * rng.standard_normal((n, 2))
    k1 = uv1 + 0.5 * rng.standard_normal((n, 2))
    out = rng.uniform(size=n) < outl
    k1[out] = rng.uniform([0, 0], [w, h], (int(out.sum()), 2))
    conf = np.where(out, rng.uniform(0, 0.3, n), rng.uniform(0.5, 1.0, n))
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return {'kpts0': k0[None], 'kpts1': k1[None], 'intr': K[None], 'conf': conf[None, :, None], 'T_021': T[None]}


def _batch(case):
    rng = np.random.default_rng(case['seeds'][0] + 17)
    items = []
    for bi, s in enumerate(case['seeds']):
        sc = _scene(s, case['n'], case['outl'], case.get('baseline'))
        k1, c = sc['kpts1'][0].copy(), sc['conf'][0, :, 0].copy()
        n = case['n']
        # unmatched keypoints as get_kpts produces them: the gather picks up the last view-1 keypoint, weight 0
        drop = rng.uniform(size=n) < case.get('zero', 0.0)
        keep = case.get('keep', [None] * len(case['seeds']))[bi]
        if keep is not None:
            drop = np.ones(n, bool)
            drop[rng.permutation(n)[:keep]] = False
        k1[drop] = k1[-1]
        c[drop] = 0.0
        items.append(dict(kpts0=sc['kpts0'][0], kpts1=k1, intr=sc['intr'][0], conf=c[:, None], T_gt=sc['T_021'][0]))
    # fp32 inputs: both reference runs and the tests see the same numbers
    return {k: np.stack([it[k] for it in items]).astype(np.float32) for k in items[0]}


def _reference_grads(erp, cpe, z, branch, loss, tdt, r):
    """-> (grad_conf [B,N], grad_T [B,4,4], grad_conf_norm [B,N], T [B,4,4]) of the reference in dtype tdt."""
    old = torch.get_default_dtype()
    torch.set_default_dtype(tdt)
    try:
        k0, k1, K, Tg = (torch.from_numpy(z[k]).to(tdt) for k in ('kpts0', 'kpts1', 'intr', 'T_gt'))
        c = torch.from_numpy(z['conf']).to(tdt).requires_grad_()
        if branch == 'closest':
            T, info = erp.estimate_relative_pose_w8pt(k0, k1, K, K, c, choose_closest=True, T_021=Tg)
            cn = info['confidence']
        else:
            outs = [erp.estimate_relative_pose_w8pt(k0[b:b + 1], k1[b:b + 1], K[b:b + 1], K[b:b + 1], c[b:b + 1])
                    for b in range(k0.shape[0])]
            T = torch.cat([o[0] for o in outs])
            cn = torch.cat([o[1]['confidence'] for o in outs])
        T.retain_grad()
        rt = torch.from_numpy(r).to(tdt)
        terms = {'rot': lambda: cpe.compute_rotation_error(T, Tg),
                 'transl': lambda: cpe.compute_translation_error_as_angle(T, Tg),
                 'conf': lambda: (cn[..., 0] * rt).sum()}
        L = terms['rot']() + terms['transl']() if loss == 'both' else terms[loss]()
        L.backward()
        gT = T.grad if T.grad is not None else torch.zeros_like(T)
        gcn = rt if loss == 'conf' else torch.zeros_like(rt)
        return (c.grad[..., 0].detach().numpy().astype(np.float64), gT.numpy().astype(np.float64),
                gcn.numpy().astype(np.float64), T.detach().numpy().astype(np.float64))
    finally:
        torch.set_default_dtype(old)


def main():
    warnings.filterwarnings('ignore')
    from oracle import ref_shim
    from oracle import pose as P
    from oracle import pose_grad as PG
    erp, _ = ref_shim.load()
    cpe = importlib.import_module('pose_optimization.two_view.compute_pose_error')
    assert cpe.__file__.startswith(ref_shim.REF), cpe.__file__
    torch.set_num_threads(8)
    os.makedirs(OUT, exist_ok=True)
    report = {}
    for case in CASES:
        z = _batch(case)
        B, N = z['conf'].shape[:2]
        nz = (z['conf'][..., 0] != 0).sum(-1)
        out = {}
        rep = {'nonzero_weights': nz.tolist()}
        for branch in BRANCHES:
            Tv, info = P.estimate_relative_pose_w8pt(*(z[k].astype(np.float64) for k in ('kpts0', 'kpts1', 'intr', 'intr', 'conf')))
            if branch == 'vote':
                rep['vote_choice'] = info['vote_counts'].argmax(-1).tolist()
            for li, loss in enumerate(LOSSES):
                r = np.random.default_rng([case['seeds'][0], li]).standard_normal((B, N))
                g64, gT64, gcn, T64 = _reference_grads(erp, cpe, z, branch, loss, torch.float64, r)
                g32, _, _, _ = _reference_grads(erp, cpe, z, branch, loss, torch.float32, r)
                go = PG.w8pt_conf_grad(z['kpts0'], z['kpts1'], z['intr'], z['intr'], z['conf'], gT64, gcn,
                                       choose_closest=branch == 'closest', T_021=z['T_gt'].astype(np.float64))
                key = '%s_%s' % (branch, loss)
                items = []
                for b in range(B):
                    scale = float(np.abs(g64[b]).max()) if np.isfinite(g64[b]).all() else float('nan')
                    it = {'scale': scale, 'ref32_vs_ref64': float(np.abs(g32[b] - g64[b]).max()),
                          'ref64_finite': bool(np.isfinite(g64[b]).all())}
                    if nz[b] >= 8:
                        err = float(np.abs(go[b] - g64[b]).max())
                        it['oracle_vs_ref64_rel'] = err / scale
                        assert err <= 1e-8 * scale + 1e-12, (case['name'], key, b, err, scale)
                    else:
                        assert np.isnan(go[b]).all()
                        it['ref64_max_abs'] = float(np.nanmax(np.abs(g64[b]))) if np.isfinite(g64[b]).any() else None
                    items.append(it)
                rep[key] = items
                out['g64_' + key], out['g32_' + key], out['gT64_' + key], out['gcn_' + key] = g64, g32, gT64, gcn
                out['T64_' + branch] = T64
        report[case['name']] = rep
        np.savez_compressed(os.path.join(OUT, 'w8pt_grad_%s.npz' % case['name']), meta=json.dumps(case), **z, **out)
        worst = max(it.get('oracle_vs_ref64_rel', 0.0) for k, v in rep.items() if isinstance(v, list) and v and isinstance(v[0], dict) for it in v)
        print(case['name'], 'ok; vote choice', rep['vote_choice'], 'worst oracle/ref64 rel %.2e' % worst)
    with open(os.path.join(OUT, 'w8pt_grad_report.json'), 'w') as f:
        json.dump(report, f, indent=1)


if __name__ == '__main__':
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    main()
