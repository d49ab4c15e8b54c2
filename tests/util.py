"""Shared helpers for the parity tests (oracle side is test infrastructure)."""
import json
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')

MATCHER_CASES = ['pair_small_ragged', 'pair_18l_128', 'mv3_ragged', 'mv5_28l_96', 'pair3_mv_false', 'pair_flat',
                 'pair_18l_128_sharp', 'mv5_28l_96_sharp', 'mv4_ragged_sharp']


def load_case(name):
    z = np.load(os.path.join(GOLDEN, 'matcher_%s.npz' % name))
    meta = json.loads(str(z['meta']))
    ref = {k: z[k] for k in z.files if k != 'meta'}
    return meta, ref


def case_inputs(meta):
    from oracle.weights import make_state_dict, make_view_inputs, make_correlated_view_inputs
    sd = make_state_dict(len(meta['layers']), seed=meta['wseed'], final_proj_gain=meta.get('gain', 1.0))
    if meta['corr']:
        data = make_correlated_view_inputs(meta['iseed'], len(meta['counts']), meta['counts'][0])
    else:
        data = make_view_inputs(meta['iseed'], meta['counts'])
    return sd, data


def score_tol_for(name):
    """(abs, rel) tolerance on the log-couplings of a golden case in the default fp32-faithful tensor-core mode.  The
    reference's own fp32 run sits `noise` away from its double-precision run (matcher_report.json, measured by the
    generator).  The split-operand arithmetic (22-bit operands, lo.lo term dropped) is measured at up to 3.6x that noise
    in absolute terms on top of a 3e-5 relative term (tools/score_ab.py; the fp32 CUDA-core
    mode sits AT the noise): 4x noise, never below 3e-4."""
    noise = json.load(open(os.path.join(GOLDEN, 'matcher_report.json')))[name]['max_abs_ref32_vs_ref64']
    return (max(3e-4, 4.0 * noise), 3e-5)


def stable_rows(Z, tau):
    """Rows/cols of the reference coupling matrix whose arg-max decision has a top-2 margin > tau
    in both directions (SURVEY.md A.4: ties are not part of the contract)."""
    inner = Z[:, :-1, :-1]
    srt = np.sort(inner, axis=2)
    row_margin = srt[..., -1] - srt[..., -2] if inner.shape[2] > 1 else np.full(inner.shape[:2], np.inf)
    srt = np.sort(inner, axis=1)
    col_margin = srt[:, -1, :] - srt[:, -2, :] if inner.shape[1] > 1 else np.full((inner.shape[0], inner.shape[2]), np.inf)
    j = inner.argmax(2)
    i = inner.argmax(1)
    st0 = (row_margin > tau) & (np.take_along_axis(col_margin, j, 1) > tau)
    st1 = (col_margin > tau) & (np.take_along_axis(row_margin, i, 1) > tau)
    return st0, st1


def compare_matcher_outputs(ref, got, tau=2e-4, score_tol=(2e-4, 1e-5), min_stable=0.0, conf_tol=2e-4):
    """ref: dict of numpy arrays (reference outputs), got: dict of numpy arrays (ours).
    - coupling matrices / confidences: allclose with abs + rel tolerance
    - matches: bit-exact on every keypoint whose decision margin exceeds tau
    Returns a small report dict."""
    report = {'n_pairs': 0, 'unstable': 0, 'rows': 0, 'max_score_err': 0.0, 'max_conf_err': 0.0,
              'mismatch_at_margin_0': 0}
    for k in ref:
        if not k.startswith('scores_'):
            continue
        a, b = k.split('_')[1:]
        Z, Zg = ref[k], got[k]
        assert Z.shape == Zg.shape, (k, Z.shape, Zg.shape)
        err = np.abs(Z - Zg)
        lim = score_tol[0] + score_tol[1] * np.abs(Z)
        assert (err <= lim).all(), (k, float(err.max()), float((err - lim).max()))
        report['max_score_err'] = max(report['max_score_err'], float(err.max()))
        st0, st1 = stable_rows(Z, tau)
        for side, st, vid in ((0, st0, a), (1, st1, b)):
            mk = 'matches%s_%s_%s' % (vid, a, b)
            sk = 'matching_scores%s_%s_%s' % (vid, a, b)
            assert got[mk].dtype == np.int64 and got[mk].shape == ref[mk].shape
            assert np.array_equal(ref[mk][st], got[mk][st]), (mk, int((ref[mk][st] != got[mk][st]).sum()))
            same = ref[mk] == got[mk]
            report['mismatch_at_margin_0'] += int((~same).sum())    # measured, incl. the near-ties (informational)
            np.testing.assert_allclose(got[sk][same], ref[sk][same], rtol=max(2e-3, 2 * score_tol[0]), atol=1e-6)
            report['unstable'] += int((~st).sum())
            report['rows'] += int(st.size)
        ck = 'conf_scores_%s_%s' % (a, b)
        if ck in ref:
            same = (ref['matches%s_%s_%s' % (a, a, b)] == got['matches%s_%s_%s' % (a, a, b)])
            cerr = np.abs(ref[ck][..., 0] - got[ck][..., 0])[same]
            assert (cerr < conf_tol).all(), (ck, float(cerr.max()))
            report['max_conf_err'] = max(report['max_conf_err'], float(cerr.max()) if cerr.size else 0.0)
        report['n_pairs'] += 1
    assert report['n_pairs'] > 0
    assert report['unstable'] <= (1 - min_stable) * report['rows'] or tau == 0, report
    return report
