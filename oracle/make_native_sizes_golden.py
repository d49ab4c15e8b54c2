"""Fixtures for images at their native sizes -- sides that are not multiples of 8, and pairs of one portrait and one
landscape image, as eval_pairs.py makes them for MegaDepth / YFCC100M (longer side resized to 1600, aspect kept) -- from
the UNMODIFIED reference with seeded weights and inputs.  Authoring container only (needs /root/reference):
    python -m oracle.make_native_sizes_golden
Writes tests/golden/native_*.npz and tests/golden/native_report.json:
  - native_sp_*:     SuperPoint (models/models/superpoint.py) on odd and MegaDepth-scale sizes.  Every keypoint and score
                     is stored; the large cases store the descriptors of every `desc_every`-th keypoint (in (y, x) order)
                     only, to keep the files small.
  - native_eval_*:   MultiViewMatcher(multi_frame_matching=False) in eval mode on pairs whose images differ in size (each
                     view normalised by its own image, multi_view_matcher.py:165-166), with the fp32-vs-fp64 noise and
                     the top-2 margins the tests compare with.
  - native_train_*:  the same model in .train() with full_output on a portrait / landscape pair (fp32 and fp64 runs,
                     BatchNorm running statistics after the call), in the layout of make_train_forward_golden.py.
  - native_chain_*:  two seeded images of different sizes (neither a multiple of 8) -> reference SuperPoint, one image
                     per call (merge=False, eval_pairs.py:210) -> reference pairwise matcher.
The GPU tests rebuild every input from the seeds stored in the metadata."""
import contextlib
import io
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
REF = '/root/reference'
OUT = os.path.join(ROOT, 'tests', 'golden')

SP_CASES = [
    dict(name='sp_133x201_all', seed=4, height=133, width=201, max_keypoints=-1, wseed=0, desc_every=1),
    dict(name='sp_1600x1066_top2048', seed=5, height=1600, width=1066, max_keypoints=2048, wseed=1, desc_every=16),
    dict(name='sp_1066x1600_top2048', seed=6, height=1066, width=1600, max_keypoints=2048, wseed=1, desc_every=16),
]
# sizes: one (width, height) per view; keypoints of the seeded 640 x 480 inputs are scaled to each view's image
EVAL_CASES = [
    dict(name='eval_portrait_landscape_18l_b2', layers=['self', 'cross'] * 9, counts=[256, 256], batch=2,
         sizes=[(1600, 1066), (1066, 1600)], wseed=8, iseed=18, corr=True, gain=12.0),
    dict(name='eval_pair3_ragged', layers=['self', 'cross'] * 2, counts=[70, 50, 90], batch=1,
         sizes=[(201, 133), (1066, 1600), (1600, 1066)], wseed=9, iseed=19, corr=False, gain=16.0),
]
TRAIN_CASE = dict(name='train_portrait_landscape_128', multi=False, views=2, kpts=128, batch=2, layers=['self', 'cross'] * 2,
                  sizes=[(1600, 1066), (1066, 1600)], wseed=43, iseed=53, gain=10.0)
TRAIN_STATS = ['kenc.encoder.1.running_mean', 'kenc.encoder.10.running_var', 'gnn.layers.0.mlp.1.running_mean',
               'gnn.layers.3.mlp.1.running_var', 'conf_mlp.layers_f.1.running_mean', 'conf_mlp.layers_c.4.running_var',
               'conf_mlp.layers_f.4.num_batches_tracked']
# two crops (y0, x0, height, width) of one seeded image: a landscape and a portrait view of shared content
CHAIN_CASE = dict(name='chain_landscape_portrait', base_seed=7, base_hw=[240, 320], crops=[[0, 0, 155, 229], [8, 64, 187, 131]],
                  sp_wseed=0, sp_config={'max_keypoints': -1, 'remove_borders': 0}, layers=['self', 'cross'] * 3,
                  wseed=10, gain=12.0)


def sp_desc_columns(kp_yx, every):
    """Indices of the keypoints whose descriptors a fixture stores: every `every`-th in (y, x) order (independent of
    the order top-k returns them in)."""
    order = np.lexsort((kp_yx[:, 1], kp_yx[:, 0]))
    return np.sort(order[::every])


def scale_inputs(data, sizes, batch):
    """Seeded matcher inputs made for 640 x 480 -> keypoints scaled into each view's own (width, height), image{i}
    of that shape."""
    for i, (w, h) in enumerate(sizes):
        data['keypoints%d' % i] = (data['keypoints%d' % i] * np.array([w / 640.0, h / 480.0])).astype(np.float32)
        data['image%d' % i] = np.zeros((batch, 1, h, w), np.float32)
    return data


def eval_inputs(case):
    from oracle.weights import make_state_dict, make_view_inputs, make_correlated_view_inputs
    sd = make_state_dict(len(case['layers']), seed=case['wseed'], final_proj_gain=case['gain'])
    if case['corr']:
        data = make_correlated_view_inputs(case['iseed'], len(case['counts']), case['counts'][0], batch=case['batch'])
    else:
        data = make_view_inputs(case['iseed'], case['counts'], batch=case['batch'])
    return sd, scale_inputs(data, case['sizes'], case['batch'])


def train_inputs(case):
    from oracle.weights import make_state_dict, make_correlated_view_inputs
    sd = make_state_dict(len(case['layers']), seed=case['wseed'], final_proj_gain=case['gain'])
    data = make_correlated_view_inputs(case['iseed'], case['views'], case['kpts'], batch=case['batch'])
    return sd, scale_inputs(data, case['sizes'], case['batch'])


def chain_images(case):
    from e2e_multi_view_matching_b200.synthetic import make_image
    base = make_image(case['base_seed'], *case['base_hw'])
    return [np.ascontiguousarray(base[:, :, y0:y0 + h, x0:x0 + w]) for y0, x0, h, w in case['crops']]


def chain_matcher_state_dict(case):
    from oracle.weights import make_state_dict
    return make_state_dict(len(case['layers']), seed=case['wseed'], final_proj_gain=case['gain'])


def _ref_superpoint(config, wseed):
    from models.models.superpoint import SuperPoint          # the unmodified reference
    from e2e_multi_view_matching_b200.synthetic import make_superpoint_state_dict
    with contextlib.redirect_stdout(io.StringIO()):
        sp = SuperPoint(config).eval()
    sp.load_state_dict({k: torch.from_numpy(v) for k, v in make_superpoint_state_dict(wseed).items()}, strict=True)
    return sp


def _noise_and_margins(ref, ref64):
    from tests.util import stable_rows
    margins, st, tot, noise = [], 0, 0, 0.0
    for k, v in ref.items():
        if k.startswith('scores_'):
            inner = np.sort(v[:, :-1, :-1], axis=2)
            margins.append(float((inner[..., -1] - inner[..., -2]).min()))
            s0, s1 = stable_rows(v, 2e-3)
            st += int(s0.sum() + s1.sum())
            tot += int(s0.size + s1.size)
            noise = max(noise, float(np.abs(v.astype(np.float64) - ref64[k]).max()))
    return {'min_top2_margin': min(margins), 'stable_frac_tau_2e-3': st / tot, 'max_abs_ref32_vs_ref64': noise}


def make_superpoint(report):
    from e2e_multi_view_matching_b200.synthetic import make_image
    for case in SP_CASES:
        img = torch.from_numpy(make_image(case['seed'], case['height'], case['width']))
        with torch.no_grad():
            out = _ref_superpoint({'max_keypoints': case['max_keypoints']}, case['wseed'])({'image': [img]})
            everything = _ref_superpoint({'max_keypoints': -1}, case['wseed'])({'image': [img]})
        kp = out['keypoints'][0].numpy().astype(np.int16)
        sc = out['scores'][0].numpy()
        cols = sp_desc_columns(kp[:, ::-1], case['desc_every'])
        meta = dict(case)
        meta['n_keypoints'] = int(kp.shape[0])
        all_sc = np.sort(everything['scores'][0].numpy())[::-1]
        meta['min_threshold_margin'] = float(np.abs(all_sc - 0.005).min())
        if 0 < case['max_keypoints'] < all_sc.size:
            # the top-k boundary: a gap far above fp32 noise keeps the selected set well defined
            meta['topk_margin'] = float(all_sc[case['max_keypoints'] - 1] - all_sc[case['max_keypoints']])
        report[case['name']] = {k: meta[k] for k in ('n_keypoints', 'min_threshold_margin', 'topk_margin') if k in meta}
        np.savez_compressed(os.path.join(OUT, 'native_%s.npz' % case['name']), meta=json.dumps(meta), keypoints=kp,
                            scores=sc, desc_columns=cols.astype(np.int32),
                            descriptors=out['descriptors'][0].numpy()[:, cols].astype(np.float32))
        print(case['name'], report[case['name']])


def make_eval(report):
    from oracle.make_golden import run_reference
    for case in EVAL_CASES:
        sd, data = eval_inputs(case)
        rcase = dict(multi=False, layers=case['layers'])
        ref = run_reference(rcase, sd, data)
        stats = _noise_and_margins(ref, run_reference(rcase, sd, data, double=True))
        assert stats['stable_frac_tau_2e-3'] >= 0.9, (case['name'], stats)
        report[case['name']] = stats
        np.savez_compressed(os.path.join(OUT, 'native_%s.npz' % case['name']), meta=json.dumps(case), **ref)
        print(case['name'], stats)


def make_train(report):
    from models.models.multi_view_matcher import MultiViewMatcher
    case = TRAIN_CASE
    sd, data_np = train_inputs(case)
    out = {}
    for dtype, tag in ((torch.float32, 'f32'), (torch.float64, 'f64')):
        torch.manual_seed(0)
        model = MultiViewMatcher({'multi_frame_matching': False, 'GNN_layers': case['layers'], 'conf_mlp': True,
                                  'full_output': True})
        model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
        model = model.to(dtype).train()
        data = {k: (torch.from_numpy(v).to(dtype) if isinstance(v, np.ndarray) and v.dtype.kind == 'f' else v)
                for k, v in data_np.items()}
        res = model(data)
        st = model.state_dict()
        for k, v in res.items():
            if v is not None:
                out['%s__%s' % (tag, k)] = v.detach().numpy()
        for k in TRAIN_STATS:
            out['%s__stat__%s' % (tag, k)] = st[k].detach().numpy()
    noise = max(float(np.abs(out['f32__' + k[5:]].astype(np.float64) - v).max()) for k, v in out.items()
                if k.startswith('f64__scores_'))
    report[case['name']] = {'max_abs_ref32_vs_ref64_scores': noise}
    np.savez_compressed(os.path.join(OUT, 'native_%s.npz' % case['name']), meta=json.dumps(case), **out)
    print(case['name'], report[case['name']])


def make_chain(report):
    from oracle.make_golden import run_reference
    case = CHAIN_CASE
    imgs = chain_images(case)
    sp = _ref_superpoint(case['sp_config'], case['sp_wseed'])
    data = {'ids': [0, 1]}
    with torch.no_grad():
        for i, img in enumerate(imgs):          # one image per call: merge=False
            p = sp({'image': [torch.from_numpy(img)]})
            data['keypoints%d' % i] = p['keypoints'][0][None].numpy()
            data['scores%d' % i] = p['scores'][0][None].numpy()
            data['descriptors%d' % i] = p['descriptors'][0][None].numpy()
            data['image%d' % i] = img
    sd = chain_matcher_state_dict(case)
    rcase = dict(multi=False, layers=case['layers'])
    ref = run_reference(rcase, sd, data)
    stats = _noise_and_margins(ref, run_reference(rcase, sd, data, double=True))
    stats['n_keypoints'] = [int(data['keypoints%d' % i].shape[1]) for i in range(2)]
    report[case['name']] = stats
    store = {'keypoints%d' % i: data['keypoints%d' % i][0].astype(np.int16) for i in range(2)}
    store.update({'ref__' + k: v for k, v in ref.items()})
    np.savez_compressed(os.path.join(OUT, 'native_%s.npz' % case['name']), meta=json.dumps(case), **store)
    print(case['name'], stats)


def main():
    if REF not in sys.path:
        sys.path.insert(0, REF)
    torch.set_num_threads(os.cpu_count())
    os.makedirs(OUT, exist_ok=True)
    report = {}
    make_superpoint(report)
    make_eval(report)
    make_train(report)
    make_chain(report)
    with open(os.path.join(OUT, 'native_report.json'), 'w') as f:
        json.dump(report, f, indent=1)


if __name__ == '__main__':
    main()
