"""The production Sinkhorn against the reference iteration in float64, at the shapes where its work split changes.

The cluster kernel (csrc/sinkhorn_cl.cu) picks its cluster size C from the largest m (1, 2, 4, 8 or 16 CTAs of at most
64 rows), gives each CTA a slice of ceil((n+1)/C) columns to merge, activates its 128-column strips while
strip * 128 < n, and re-absorbs scalings that leave [e^-8, e^8]; above 1024 rows or columns the multi-CTA kernel
(csrc/sinkhorn_exp.cu) takes over.  The cases below sit on both sides of every one of those edges, include the
short-view-against-long-view shapes whose column slices are wider than the CTA, and vary the bin score, the iteration
count (odd counts flip the mbarrier phase parity) and the score spread.

Yardstick: oracle.matcher_torch._log_optimal_transport (the reference's iteration, superglue.py:143-172) in float64
on the CPU.  The same function in float32 gives the reference's own fp32 noise for each case, and every kernel must
stay within max(1e-4, 3 x that noise) + 1e-5 |Z| on the whole [B, m+1, n+1] matrix, dustbins included.
"""
import functools
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from tests.util import GOLDEN, compare_matcher_outputs

pytestmark = pytest.mark.gpu

CLUSTER = ('cluster2', 'cluster', 'cluster6')      # the 512-thread default instance and the two 1024-thread ones
PREFIX_HASHES = os.path.join(GOLDEN, 'sinkhorn_prefix_sha256.json')

# Known defect of the scaling-domain kernels (cluster and multi-CTA; the log-domain 'log' and 'ref' kernels are not
# affected).  They keep the dustbin column of K~ as the product e_i * kb_n with e_i = exp(bin_score + u~_i) and
# kb_n = exp(v~_n).  u~_i starts at -(row max), so e_i underflows to 0 in fp32 for every row whose best score exceeds the
# bin score by more than ~88, while v~_n later grows by as much: the entry itself is O(1) but its two factors are out of
# range, and multiplying 0 by absorbed scalings never brings it back.  That matters when most rows must go to the
# dustbin (m well above n) and the spread is large: at 700 x 64 the inner columns end up off by up to 104 in log space,
# at 1500 x 300 the output is NaN.  A numpy emulation of the iteration that keeps each dustbin-column entry whole,
# exp(bin_score + u~_i + v~_n) recomputed from the potentials on every absorption, stays within 5e-5 of float64 on both.
TALL_SPREAD_40 = [(1, 700, 64, 2.3, 100, 40.0, 'randn'), (1, 1500, 300, -0.5, 100, 40.0, 'randn')]
SCALING_DOMAIN = (None, 'multicta') + ('cluster2', 'cluster', 'cluster6')

# (B, m, n, bin_score, iters, spread, kind)
CASES = [
    (1, 1, 1, 1.0, 100, 1.0, 'randn'),
    (3, 1, 1024, 1.0, 100, 12.0, 'randn'),         # C = 1: a slice of 1025 columns, twice the 512 threads
    (1, 1, 3, 2.3, 7, 12.0, 'randn'),
    (1, 64, 3, -0.5, 100, 12.0, 'randn'),
    (1, 64, 512, 1.0, 100, 12.0, 'randn'),         # C = 1: first n whose slice exceeds 512 columns
    (1, 64, 700, 2.3, 7, 40.0, 'randn'),
    (3, 40, 1024, 1.0, 100, 12.0, 'randn'),
    (1, 65, 127, 1.0, 1, 12.0, 'randn'),           # C = 2
    (1, 100, 1024, -0.5, 100, 40.0, 'randn'),      # C = 2 with a 513-column slice
    (1, 128, 1024, 1.0, 2, 12.0, 'randn'),
    (1, 128, 128, 2.3, 100, 1.0, 'flat'),
    (1, 129, 129, 1.0, 100, 40.0, 'randn'),        # C = 4
    (3, 256, 511, 1.0, 7, 12.0, 'randn'),
    (1, 257, 513, 2.3, 100, 1.0, 'low'),           # C = 8, the dustbins carry most of the mass
    (1, 512, 1023, 1.0, 100, 40.0, 'randn'),
    (1, 513, 512, -0.5, 100, 12.0, 'randn'),       # C = 16
    (1, 1024, 40, 1.0, 100, 12.0, 'randn'),
    (1, 700, 64, 2.3, 100, 40.0, 'randn'),         # most rows go to the dustbin
    (1, 1024, 1, 1.0, 100, 12.0, 'randn'),
    (1, 1024, 1023, 1.0, 7, 12.0, 'randn'),
    (1, 1024, 1024, 2.3, 100, 12.0, 'randn'),
    (1, 1025, 1025, 1.0, 100, 12.0, 'randn'),      # multi-CTA from here on
    (1, 1500, 300, -0.5, 100, 40.0, 'randn'),
    (1, 64, 2048, 1.0, 100, 12.0, 'randn'),
    (1, 2048, 2048, 1.0, 100, 12.0, 'randn'),      # cfg4 size
]

# shapes every build of the cluster kernel could run: their outputs must not change by a bit
PREFIX_CASES = [
    (3, 60, 500, 1.0, 100, 12.0, 'randn'),         # C = 1, 501-column slice
    (1, 65, 1023, 2.3, 7, 40.0, 'randn'),          # C = 2, 512-column slice
    (1, 129, 255, -0.5, 100, 12.0, 'randn'),
    (1, 300, 257, 1.0, 100, 40.0, 'randn'),
    (1, 1024, 1024, 1.0, 100, 12.0, 'randn'),      # the benchmark's shape
]


def case_id(c):
    return 'B%d_%dx%d_bin%g_it%d_%s%g' % (c[0], c[1], c[2], c[3], c[4], c[6], c[5])


def kernels_for(case):
    """Every kernel a case runs on; the cluster variants also where they must refuse the shape."""
    _, m, n = case[:3]
    ks = [None, 'multicta'] + list(CLUSTER)
    if m <= 1024 and n <= 1024:
        ks.append('log')
    if (m + 1) * (n + 1) <= 140000:     # the one-CTA cross-check walks the whole matrix from L2 every iteration
        ks.append('ref')
    return ks


def refuses(case, k):
    return k in CLUSTER and (case[1] > 1024 or case[2] > 1024)


KERNEL_CASES = [pytest.param(c, k, id='%s-%s' % (case_id(c), k),
                             marks=[pytest.mark.xfail(strict=True, reason='scaling-domain dustbin column leaves the fp32 range')]
                             if c in TALL_SPREAD_40 and k in SCALING_DOMAIN and not refuses(c, k) else [])
                for c in CASES for k in kernels_for(c)]


def make_scores(case):
    B, m, n, _, _, spread, kind = case
    rng = np.random.default_rng(m * 7919 + n * 31 + B)
    if kind == 'flat':       # every score equal up to tiny noise
        s = 0.5 + 1e-3 * rng.standard_normal((B, m, n))
    elif kind == 'low':      # scores well below the bin score
        s = -6.0 + spread * rng.standard_normal((B, m, n))
    else:
        s = spread * rng.standard_normal((B, m, n))
    return torch.from_numpy(s.astype(np.float32))


@functools.lru_cache(maxsize=1)         # the kernels of a case run one after the other
def reference(case):
    """(float64 couplings, max |fp32 run - float64 run|) of the reference iteration."""
    from oracle.matcher_torch import _log_optimal_transport
    s, alpha, iters = make_scores(case), case[3], case[4]
    z64 = _log_optimal_transport(s.double(), torch.tensor(alpha, dtype=torch.float64), iters)
    z32 = _log_optimal_transport(s.float(), torch.tensor(alpha, dtype=torch.float32), iters)
    return z64, float((z32.double() - z64).abs().max())


def run(s, alpha, iters, kernel):
    from e2e_multi_view_matching_b200 import ops
    Z = ops.log_optimal_transport(s.cuda(), alpha, iters, kernel=kernel)
    torch.cuda.synchronize()
    return Z.cpu()


def marginals(Z):
    """Row and column sums of exp(Z) (couplings times m + n), dustbins included."""
    P = torch.exp(Z.double())
    return P.sum(2), P.sum(1)


@pytest.mark.parametrize('case,k', KERNEL_CASES)
def test_sinkhorn_vs_float64(case, k):
    from e2e_multi_view_matching_b200._lib import MvmError
    B, m, n, alpha, iters, _, _ = case
    s = make_scores(case)
    if refuses(case, k):
        with pytest.raises(MvmError):       # more than 1024 rows or columns do not fit a cluster
            run(s, alpha, iters, k)
        return
    z64, noise = reference(case)
    tol = max(1e-4, 3.0 * noise)
    lim = tol + 1e-5 * z64.abs()
    r64, c64 = marginals(z64)
    Z = run(s, alpha, iters, k)
    assert Z.shape == (B, m + 1, n + 1)
    err = (Z.double() - z64).abs()
    r, c = marginals(Z)
    merr = max(float(((r - r64).abs() / r64).max()), float(((c - c64).abs() / c64).max()))
    print('%s %-8s max err %.2e (bound %.2e, fp32 noise %.2e), marginals rel err %.2e'
          % (case_id(case), k, float(err.max()), tol, noise, merr))
    assert (err <= lim).all(), (k, float(err.max()), float((err - lim).max()))
    assert merr <= 2 * tol + 1e-4, (k, merr)
    # a fixed summation order: the same input gives the same bits
    assert torch.equal(run(s, alpha, iters, k), Z), k
    # the cluster kernels and the one-CTA kernel treat every problem alike whatever the batch (the multi-CTA
    # kernels size their groups from the number of problems, so their summation order depends on B)
    if B > 1 and (k in CLUSTER or k == 'ref' or (k is None and m <= 1024 and n <= 1024)):
        for b in range(B):
            assert torch.equal(run(s[b:b + 1], alpha, iters, k)[0], Z[b]), (k, b)


def output_hash(Z):
    return hashlib.sha256(Z.contiguous().numpy().tobytes()).hexdigest()


def prefix_hashes():
    return {case_id(c): {str(k): output_hash(run(make_scores(c), c[3], c[4], k)) for k in (None,) + CLUSTER}
            for c in PREFIX_CASES}


def test_sinkhorn_outputs_unchanged_on_shapes_that_always_ran():
    """Bitwise equal to the outputs of the build before the owner merge walked slices wider than the CTA.  The hashes
    were written by this module's __main__ on that build (commit c823a42) on an H100 SXM.  They cover the cluster
    kernels only: the cluster size follows m alone, while the multi-CTA kernel sizes its groups from the SM count."""
    want = json.load(open(PREFIX_HASHES))
    got = prefix_hashes()
    assert got == want, [(c, k) for c in want for k in want[c] if got[c][k] != want[c][k]]


@pytest.mark.parametrize('iters', [0, -1])
def test_sinkhorn_refuses_fewer_than_one_iteration(iters):
    from e2e_multi_view_matching_b200._lib import MvmError
    from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher
    from e2e_multi_view_matching_b200.models.superglue import SuperGlue
    from oracle.weights import make_state_dict, make_view_inputs
    s = make_scores((1, 40, 50, 1.0, 1, 12.0, 'randn'))
    for k in (None, 'multicta', 'ref', 'log') + CLUSTER:
        with pytest.raises(MvmError):
            run(s, 1.0, iters, k)
    layers = ['self', 'cross']
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in make_state_dict(len(layers), seed=3).items()}
    data = {k: (torch.from_numpy(v).cuda() if isinstance(v, np.ndarray) else v)
            for k, v in make_view_inputs(3, [40, 50]).items()}
    mv = MultiViewMatcher({'GNN_layers': layers, 'sinkhorn_iterations': iters}).eval()
    mv.load_state_dict(sd)
    with pytest.raises(MvmError):
        mv.cuda()(data)
    sg = SuperGlue({'GNN_layers': layers, 'sinkhorn_iterations': iters}).eval()
    sg.load_state_dict({k: v for k, v in sd.items() if not k.startswith('conf_mlp')})
    with pytest.raises(MvmError):
        sg.cuda()(data)


# Ragged pair tables through the matcher: one Sinkhorn launch runs every pair with its own (m, n), and the cluster
# size comes from the largest m of the table.  (counts, multi_frame_matching, GNN layers)
RAGGED = [
    ([40, 30, 700], True, 2),        # C = 1 with long columns
    ([90, 1024, 300], True, 2),      # C = 2 with n = 1024
    ([1024, 513, 65, 1], True, 2),   # C = 16 with pairs of every width
    ([1100, 40, 600], True, 2),      # m = 1100: the whole table goes to the multi-CTA kernel
    ([50, 800], False, 4),           # pair mode
]


def run_matcher(multi, layers, sd, data, variant=None, monkeypatch=None):
    """MultiViewMatcher.forward on the GPU; with `variant`, through mvm_matcher_forward_ex with that Sinkhorn variant."""
    from e2e_multi_view_matching_b200 import _lib
    from e2e_multi_view_matching_b200.models.multi_view_matcher import MultiViewMatcher
    if variant is not None:
        lib = _lib.lib()
        opt = _lib.MatcherOptions()
        lib.mvm_matcher_options_default(opt)
        opt.sinkhorn_variant = variant
        fwd_ex = lib.mvm_matcher_forward_ex
        monkeypatch.setattr(lib, 'mvm_matcher_forward', lambda *a: fwd_ex(*a[:-1], opt, a[-1]))
    model = MultiViewMatcher({'multi_frame_matching': multi, 'GNN_layers': layers, 'conf_mlp': True}).eval()
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
    out = model.cuda()({k: (torch.from_numpy(v).cuda() if isinstance(v, np.ndarray) else v) for k, v in data.items()})
    torch.cuda.synchronize()
    if variant is not None:
        monkeypatch.undo()
    return {k: v.cpu().numpy() for k, v in out.items() if v is not None}


@pytest.mark.parametrize('counts,multi,n_layers', RAGGED, ids=lambda v: '-'.join(map(str, v)) if isinstance(v, list) else str(v))
def test_matcher_ragged_pair_table(counts, multi, n_layers, monkeypatch):
    import e2e_multi_view_matching_b200 as pkg
    from oracle.matcher import matcher_forward
    from oracle.matcher_torch import matcher_forward as matcher_forward_torch
    from oracle.weights import make_state_dict, make_view_inputs
    layers = ['self', 'cross'] * (n_layers // 2)
    sd = make_state_dict(n_layers, seed=31, final_proj_gain=16.0)
    data = make_view_inputs(41, counts)
    cfg = {'multi_frame_matching': multi, 'GNN_layers': layers}
    ref = matcher_forward(sd, cfg, data)
    # the reference's own fp32 noise: its fp32 run against a float64 run of the same ops
    ref64 = matcher_forward_torch({k: np.asarray(v, dtype=np.float64) for k, v in sd.items()}, cfg,
                                  {k: (v.astype(np.float64) if isinstance(v, np.ndarray) else v) for k, v in data.items()})
    noise = max(float(np.abs(ref[k].astype(np.float64) - ref64[k]).max()) for k in ref if k.startswith('scores_'))
    pkg.set_math_mode(0)
    try:
        got0 = run_matcher(multi, layers, sd, data)
    finally:
        pkg.set_math_mode(3)
    rep0 = compare_matcher_outputs(ref, got0, tau=2e-4, score_tol=(max(2e-4, 2.5 * noise), 1e-5))
    got = run_matcher(multi, layers, sd, data)
    rep = compare_matcher_outputs(ref, got, tau=2e-3, score_tol=(max(3e-4, 4.0 * noise), 3e-5))
    # variant 1 forces the multi-CTA Sinkhorn; every stage before it is deterministic, so the two runs differ in
    # the Sinkhorn kernel alone
    got_cl = run_matcher(multi, layers, sd, data, variant=0, monkeypatch=monkeypatch)
    got_mc = run_matcher(multi, layers, sd, data, variant=1, monkeypatch=monkeypatch)
    assert all(np.array_equal(got_cl[k], got[k]) for k in got)
    rep_v = compare_matcher_outputs(got_cl, got_mc, tau=2e-4, score_tol=(max(2e-4, 2.0 * noise), 1e-5))
    print(counts, 'reference fp32 noise %.2e' % noise, 'mode 0', rep0, 'default', rep, 'multi-CTA vs cluster', rep_v)


if __name__ == '__main__':
    # writes the output hashes of the library as built: run on the build the hashes should pin
    with open(PREFIX_HASHES, 'w') as f:
        json.dump(prefix_hashes(), f, indent=1, sort_keys=True)
