"""The attention kernels against float64, at the shapes, segment layouts and operand magnitudes where they go wrong.

Four forward kernels run every case: the fp32 CUDA-core kernel (csrc/attention_simt.cu, ops.attention mode 0), and
attn_wg::attention_wg_kernel in single-pass TF32, 3xTF32 (csrc/attention_tc.cu) and fp16x3 (csrc/attention_h3.cu, the
default of the matcher and of training).  The tensor-core kernels walk a query view's source segments in 64-key tiles
with 128-query tiles, issue S(j+1) while P(j) V(j) is on the tensor cores, and keep a lazy online softmax: a row's
reference maximum is raised (and O, l rescaled by fo = 2^(m_old - m_new)) only when the tile maximum outgrows it by more
than 2^8, and P is taken relative to 2^-7 of it, so P <= 2^15.  The cases sit on the tile edges (n_pad % 128 == 64,
counts of 1, 63, 65, 127, 129, 191), at the production shapes (cfg3 5 x 1024 with 4096 cross keys, cfg4 2 x 2048,
cfg5 5 x 400 in n_pad 448), at the 8-view maximum, and use inputs that aim at the softmax's branches:

  late_max  one-dimensional Q and K, so each head gets designed logits (log2 units, all |q|, |k| < 2^12):
            head 0  the maximum rises by 7.9 once: P reaches ~2^15 with no rescale;
            head 1  the maximum rises by >= 8.1 on every tile: the row rescales on every tile;
            head 2  the only large logit (+140) is the last key of the last source segment (a partial tile wherever
                    the count is not a multiple of 64): fo flushes to zero;
            head 3  the maximum sits in the first tile and every later tile is 60 lower.
  flat      identical K rows: the output is the exact mean of V over the source keys.
  range     V at 2^e for e in -12 .. 12, Q and K at 2^-8, 1 and 2^4.

Yardstick: oracle.train_ops._attend in float64 on the CPU.  Every (view, head) block must stay, on its valid query
rows, within 3 x noise + f max|V| (1 + sabs), where noise is the same function's float32 error on that block, max|V|
is taken over the block's source keys (the output is a convex combination of V rows), sabs = max_ij sum_d |q_id k_jd| / 8
is the block's logit magnitude, and f = 2^-20, or 2^-9 for single-pass TF32.  The sabs term is there because the
split-operand kernels hold Q and K to 22 bits (TF32 to 11), so their logit error follows sum |q k|, not the fp32
noise: with Q and K at 2^4 (logits in the thousands) the 3xTF32 kernel sat at 6 x the noise bound alone.
Largest error as a share of the bound over every case on an H100 80GB HBM3 (700 W): SIMT 0.06, 3xTF32 0.20,
fp16x3 0.51 (0.12 outside the range cases), single-pass TF32 0.39.

fp16x3 has a lower edge in |V|: lo = fp16(v - hi) is exact to 2^-24 absolute only, an fp16 subnormal once |v| < 2^-3,
so hi + lo keeps fewer than 22 bits the smaller V gets.  On the H100 the fp16x3 kernel passes with V at 2^-8 (max|V|
~2^-6; at most 0.51 of the bound) and leaves the bound with V at 2^-12 (max|V| ~2^-10) unless Q and K are large:
1.3-1.9 x the bound with Q, K at 1, 5.5-7.9 x with Q, K at 2^-8, where the output averages many V rows.  Those cases
are strict xfails.  Per-layer |V| of the matcher on the golden fixtures' synthetic weights: median 0.05-0.2, max
0.3-1.1; trained weights are not measured.

The backward (csrc/attention_bwd.cu, both variants) is checked against torch autograd through the same function in
float64: relative error (to max |reference|) below 2e-5 (the bound of tests/test_train_backward_gpu.py) + 3 x the fp32
autograd's own relative error, plus for dq and dk a term for the cancellation in dP - D.  The kernel takes
D = rowsum(dO * O) from the given O, so where a row's P is one-hot (the late_max logits) dP - D keeps the rounding of two
64-term dot products, times |k| / 8 (up to 97 there) in dq and times |q| / 8 and the key's attention mass in dk.  On an
H100 dq reached 1.5e-4 (TF32x3) and 3.7e-5 (fp32) there, and at cfg5 with 1600 cross keys the TF32x3 variant reached
2.4e-5 on dq and 2.7e-5 on dk; the largest error over all backward cases was 0.67 of its bound.
"""
import functools
import zlib

import numpy as np
import pytest
import torch

from tests import emul_ops

pytestmark = pytest.mark.gpu

KERNELS = {'simt': 0, 'tf32': 1, 'tf32x3': 3, 'fp16x3': 'h3'}
C_L2E = 0.125 * 1.4426950408889634          # a logit q.k / sqrt(64) in log2 units, per unit of q.k
BIG = 3.0e4                                  # padding garbage: finite, inside the fp16 range

# (B, T, n_pad, counts, is_cross)
SHAPES = [
    (1, 1, 64, (1,), 0),                                        # a single key: the output is its V row
    (1, 2, 64, (1, 1), 1),
]
for _c in [(63, 65, 192), (1, 129, 191), (64, 128, 127)]:      # n_pad % 128 == 64: the second query tile is half outside
    SHAPES += [(2, 3, 192, _c, 0), (2, 3, 192, _c, 1)]
for _c in [(400,) * 5, (400, 1, 399, 257, 64)]:                # cfg5
    SHAPES += [(2, 5, 448, _c, 0), (2, 5, 448, _c, 1)]
SHAPES += [(2, 5, 1024, (1024,) * 5, 0), (2, 5, 1024, (1024,) * 5, 1)]   # cfg3: 64 key tiles per query view in cross
for _c in [(2048, 2048), (2048, 1)]:                           # cfg4
    SHAPES += [(1, 2, 2048, _c, 0), (1, 2, 2048, _c, 1)]
SHAPES += [(2, 8, 128, (128, 1, 65, 64, 127, 3, 100, 128), 0), (2, 8, 128, (128, 1, 65, 64, 127, 3, 100, 128), 1)]
SHAPES += [(1, 3, 64, (0, 64, 5), 0), (1, 3, 64, (0, 64, 5), 1), (1, 3, 64, (0, 0, 5), 0)]   # views without keypoints

V_EXPS = (-12, -8, -6, -4, 0, 8, 12)
QK_EXPS = (-8, 0, 4)
RANGE_SHAPES = [(2, 3, 192, (63, 65, 192), 0), (2, 3, 192, (1, 129, 191), 1)]
# (V, Q/K) scale exponents at which fp16x3 leaves the bound on an H100: lo = fp16(v - hi) is ~2^-11 |v|, an fp16
# subnormal once |v| < 2^-3, so hi + lo keeps fewer bits the smaller V gets.  With Q and K at 2^4 the logit term of the
# bound is large enough to cover it.
FP16X3_RANGE_EDGE = ((-12, -8), (-12, 0))

CASES = [s + (r,) for s in SHAPES for r in ('randn1', 'randn6', 'late_max', 'flat')]
CASES += [s + ('range_v%d_qk%d' % (ev, eq),) for s in RANGE_SHAPES for ev in V_EXPS for eq in QK_EXPS]


def case_id(c):
    B, T, n_pad, counts, is_cross, regime = c
    return 'B%d_T%d_n%d_%s_%s_%s' % (B, T, n_pad, '-'.join(map(str, counts)), 'cross' if is_cross else 'self', regime)


def range_exps(regime):
    return tuple(int(p[1:] if p[0] == 'v' else p[2:]) for p in regime.split('_')[1:])


def marks_for(c, k):
    if k == 'fp16x3' and c[5].startswith('range') and range_exps(c[5]) in FP16X3_RANGE_EDGE:
        return [pytest.mark.xfail(strict=True, reason='|V| below the fp16x3 edge: the lo plane is an fp16 subnormal')]
    return []


KERNEL_CASES = [pytest.param(c, k, id='%s-%s' % (case_id(c), k), marks=marks_for(c, k)) for c in CASES for k in KERNELS]


def sources(T, t, is_cross):
    return [s for s in range(T) if (s != t if is_cross else s == t)]


def make_qkv(case):
    """Seeded [B*T, n_pad, 768] float32 input of a case, zero beyond each view's count."""
    B, T, n_pad, counts, is_cross, regime = case
    rng = np.random.default_rng(zlib.crc32(case_id(case).encode()))
    x = np.zeros((B, T, n_pad, 768))
    if regime.startswith('randn'):
        x[:] = float(regime[5:]) * rng.standard_normal(x.shape)
    elif regime == 'flat':
        x[..., :256] = rng.standard_normal((B, T, n_pad, 256))
        x[..., 256:512] = rng.standard_normal(256)                  # one K row for every key
        x[..., 512:] = rng.standard_normal((B, T, n_pad, 256))
    elif regime.startswith('range'):
        ev, eq = range_exps(regime)
        x[..., :512] = 2.0 ** eq * rng.standard_normal((B, T, n_pad, 512))
        x[..., 512:] = 2.0 ** ev * rng.standard_normal((B, T, n_pad, 256))
    else:
        assert regime == 'late_max'
        x[..., 512:] = rng.standard_normal((B, T, n_pad, 256))
        x[..., 0:256:64] = 1.0 - 0.01 * rng.random((B, T, n_pad, 4))   # q in [0.99, 1]: the designed rises hold
        tiles = [(c + 63) // 64 for c in counts]
        for t in range(T):
            r = np.arange(counts[t])
            g = sum(tiles[:t]) + r // 64                             # tile index in the order the views are walked
            jitter = np.where(r % 64 == 0, 0.0, -3.0 * rng.random(counts[t]))  # each tile's first key holds its max
            # the walk of a query view starts at view 0 (view 1 for view 0 in cross attention)
            lead = (r < 64) & ((t <= 1) if is_cross else True)
            L = np.stack([np.where(r < 64, 0.0, 7.9) + jitter,
                          8.1 * g + jitter,
                          jitter.copy(),
                          np.where(lead, 0.0, -60.0) + jitter], 1)
            if counts[t] and (not is_cross or t >= T - 2):
                L[-1, 2] = 140.0
            x[:, t, :counts[t], 256:512:64] = L / C_L2E
    for t in range(T):
        x[:, t, counts[t]:] = 0.0
    return torch.from_numpy(x.reshape(B * T, n_pad, 768).astype(np.float32))


@functools.lru_cache(maxsize=1)         # the kernels of a case run one after the other
def reference(case):
    """Per case: the float64 output, and per (view, head) block [V, 4] the fp32 noise, max |V| over the source keys and
    the logit magnitude max_ij sum_d |q_id k_jd| / 8."""
    B, T, n_pad, counts, is_cross, _ = case
    qkv = make_qkv(case)
    r64 = emul_ops._attend(qkv.double(), B, T, list(counts), is_cross)
    r32 = emul_ops._attend(qkv.float(), B, T, list(counts), is_cross).double()
    noise, vmax, sabs = (torch.zeros(B * T, 4, dtype=torch.float64) for _ in range(3))
    for v in range(B * T):
        b, t = divmod(v, T)
        c = counts[t]
        src = [b * T + s for s in sources(T, t, is_cross) if counts[s]]
        if not c or not src:
            continue
        for h in range(4):
            hs = slice(h * 64, (h + 1) * 64)
            noise[v, h] = (r32[v, :c, hs] - r64[v, :c, hs]).abs().max()
            vmax[v, h] = max(float(qkv[s, :counts[s % T], 512:][:, hs].abs().max()) for s in src)
            k = torch.cat([qkv[s, :counts[s % T], 256:512][:, hs] for s in src]).abs()
            sabs[v, h] = float((qkv[v, :c, hs].abs() @ k.t()).max()) / 8.0
    return r64, noise, vmax, sabs


def run(qkv, B, T, counts, is_cross, k):
    from e2e_multi_view_matching_b200 import ops
    out = ops.attention(qkv.cuda(), B, T, list(counts), is_cross, tc_passes=KERNELS[k])
    torch.cuda.synchronize()
    return out.cpu()


def bound(k, noise, vmax, sabs):
    """3 x the fp32 noise + 2^-20 (2^-9 for single-pass TF32) max|V| (1 + sabs).  The split-operand kernels carry 22
    bits of Q and K (TF32 11), so a logit is off by up to ~2^-21 (2^-10) sum_d |q_d k_d| / 8 = sabs: that moves P by the
    same relative amount and the output by at most twice it times max|V|, on top of the rounding of P and V."""
    return 3.0 * noise + (2.0 ** -9 if k == 'tf32' else 2.0 ** -20) * vmax * (1.0 + sabs)


@pytest.mark.parametrize('case,k', KERNEL_CASES)
def test_attention_vs_float64(case, k):
    B, T, n_pad, counts, is_cross, regime = case
    qkv = make_qkv(case)
    r64, noise, vmax, sabs = reference(case)
    out = run(qkv, B, T, counts, is_cross, k)
    assert torch.isfinite(out).all()
    worst, bad = 0.0, []
    for v in range(B * T):
        c = counts[v % T]
        for h in range(4):
            if not c:
                continue
            hs = slice(h * 64, (h + 1) * 64)
            err = float((out[v, :c, hs].double() - r64[v, :c, hs]).abs().max())
            lim = bound(k, float(noise[v, h]), float(vmax[v, h]), float(sabs[v, h]))
            worst = max(worst, err / lim)
            if err > lim:
                bad.append((v, h, err, lim))
    print('%s %-6s max err / bound %.3f' % (case_id(case), k, worst))
    assert not bad, bad[:8]
    if counts == (1,) * T and k == 'simt':      # a single source key: its V row, bit for bit
        for v in range(B * T):
            src = sources(T, v % T, is_cross)[0] + (v // T) * T
            assert torch.equal(out[v, :1], qkv[src, :1, 512:]), v
    # a fixed summation order: the same input gives the same bits
    assert torch.equal(run(qkv, B, T, counts, is_cross, k), out), k


INVARIANCE_CASES = [(2, 3, 192, (63, 65, 192), 0, 'randn1'), (2, 3, 192, (1, 129, 191), 1, 'randn1'),
                    (2, 5, 448, (400, 1, 399, 257, 64), 1, 'randn1'),
                    (2, 8, 128, (128, 1, 65, 64, 127, 3, 100, 128), 1, 'randn1')]


def valid_rows(out, T, counts):
    return [out[v, :counts[v % T]] for v in range(out.shape[0])]


@pytest.mark.parametrize('k', list(KERNELS))
@pytest.mark.parametrize('case', INVARIANCE_CASES, ids=case_id)
def test_attention_padding_rows_do_not_leak(case, k):
    """Rows of qkv at and beyond a view's count (and so of the K / V planes) may hold any finite value: the kernels mask
    those keys to P = 0 and multiply their V rows by it, so the valid rows come out bitwise as with zero padding."""
    B, T, n_pad, counts, is_cross, _ = case
    qkv = make_qkv(case)
    dirty = qkv.clone()
    rng = np.random.default_rng(7)
    for v in range(B * T):
        c = counts[v % T]
        junk = rng.uniform(1e4, BIG, (n_pad - c, 768)) * rng.choice([-1.0, 1.0], (n_pad - c, 768))
        dirty[v, c:] = torch.from_numpy(junk.astype(np.float32))
    a = run(qkv, B, T, counts, is_cross, k)
    d = run(dirty, B, T, counts, is_cross, k)
    for v, (x, y) in enumerate(zip(valid_rows(a, T, counts), valid_rows(d, T, counts))):
        assert torch.equal(x, y), (k, v)


@pytest.mark.parametrize('k', list(KERNELS))
@pytest.mark.parametrize('case', INVARIANCE_CASES[1:3], ids=case_id)
def test_attention_batch_invariance(case, k):
    """Each item of a B = 3 launch is bitwise equal to a B = 1 launch of that item."""
    _, T, n_pad, counts, is_cross, regime = case
    qkv = make_qkv((3, T, n_pad, counts, is_cross, regime))
    whole = run(qkv, 3, T, counts, is_cross, k)
    for b in range(3):
        one = run(qkv[b * T:(b + 1) * T], 1, T, counts, is_cross, k)
        for t in range(T):
            assert torch.equal(one[t, :counts[t]], whole[b * T + t, :counts[t]]), (k, b, t)


# Calls every forward launch must refuse before touching the GPU.  Each one stays inside its buffers even if its check
# went missing: an oversized count sits on view 0, whose keys and queries then run into view 1's rows of the same buffer.
# (T, n_pad, counts, is_cross)
REFUSED = {
    'count_above_n_pad_self': (2, 64, (128, 64), 0),
    'count_above_n_pad_cross': (2, 64, (128, 64), 1),
    'negative_count': (2, 64, (64, -1), 0),
    'query_view_without_keys': (2, 64, (64, 0), 1),
    'nine_views': (9, 64, (64,) * 9, 0),
    'cross_with_one_view': (1, 64, (64,), 1),
}


@pytest.mark.parametrize('k', list(KERNELS))
@pytest.mark.parametrize('what', list(REFUSED))
def test_attention_refuses(what, k):
    from e2e_multi_view_matching_b200 import ops
    from e2e_multi_view_matching_b200._lib import MvmError
    T, n_pad, counts, is_cross = REFUSED[what]
    qkv = torch.randn(T, n_pad, 768, generator=torch.Generator().manual_seed(3)).cuda()
    with pytest.raises(MvmError, match='invalid argument'):
        ops.attention(qkv, 1, T, list(counts), is_cross, tc_passes=KERNELS[k])
    torch.cuda.synchronize()


# ---- backward: mvm_attention_backward against torch autograd through _attend in float64

RAGGED8 = (128, 1, 65, 0, 127, 3, 100, 128)      # a view without keypoints, which the backward accepts
BWD_CASES = [(2, 5, 448, (400,) * 5, 0, 'randn1'), (2, 5, 448, (400,) * 5, 1, 'randn1'),
             (2, 5, 448, (400, 1, 399, 257, 64), 0, 'randn1'), (2, 5, 448, (400, 1, 399, 257, 64), 1, 'randn1'),
             (2, 8, 128, RAGGED8, 0, 'randn1'), (2, 8, 128, RAGGED8, 1, 'randn1'),
             (2, 3, 192, (63, 65, 192), 0, 'late_max'), (2, 3, 192, (63, 65, 192), 1, 'late_max'),
             (2, 3, 192, (63, 65, 192), 0, 'flat'), (2, 3, 192, (63, 65, 192), 1, 'flat')]


def column_mass(qkv, B, T, counts, is_cross):
    """max over keys of sum_i P_ij: the weight with which a key's dk collects the rounding of its query rows' dP - D."""
    x = qkv.double()
    worst = 0.0
    for b in range(B):
        for s in range(T):
            if counts[s] == 0:
                continue
            for h in range(4):
                hs = slice(h * 64, (h + 1) * 64)
                k = x[b * T + s, :counts[s], 256:512][:, hs]
                mass = torch.zeros(counts[s], dtype=torch.float64)
                for t in range(T):
                    src = sources(T, t, is_cross)
                    if s not in src or counts[t] == 0:
                        continue
                    allk = torch.cat([x[b * T + u, :counts[u], 256:512][:, hs] for u in src])
                    lse = torch.logsumexp(x[b * T + t, :counts[t], hs] @ allk.t() / 8.0, 1, keepdim=True)
                    mass += torch.exp(x[b * T + t, :counts[t], hs] @ k.t() / 8.0 - lse).sum(0)
                worst = max(worst, float(mass.max()))
    return worst


def dq_gross(qkv, dout, B, T, counts, is_cross):
    """The size dq has without cancellation, max over rows of 1/8 sum_j P_ij |dP_ij - D_i| max|k_j|: with identical K
    rows the exact dq is 0, and its error is measured against this."""
    x = qkv.double()
    worst = 0.0
    for b in range(B):
        for t in range(T):
            src = sources(T, t, is_cross)
            if counts[t] == 0:
                continue
            for h in range(4):
                hs = slice(h * 64, (h + 1) * 64)
                q = x[b * T + t, :counts[t], hs]
                k = torch.cat([x[b * T + s, :counts[s], 256:512][:, hs] for s in src])
                v = torch.cat([x[b * T + s, :counts[s], 512:][:, hs] for s in src])
                P = torch.softmax(q @ k.t() / 8.0, 1)
                dP = dout[b * T + t, :counts[t], hs].double() @ v.t()
                D = (P * dP).sum(1, keepdim=True)
                worst = max(worst, float(((P * (dP - D).abs()) @ k.abs().max(1).values[:, None]).max()) / 8.0)
    return worst


def fp32_backward(qkv, out, dout, B, T, counts, is_cross):
    """The reference's float32 gradient: its distance from float64 measures how the case amplifies fp32 rounding."""
    with torch.enable_grad():
        x = qkv.float().clone().requires_grad_(True)
        (g,) = torch.autograd.grad(emul_ops._attend(x, B, T, list(counts), is_cross), x, dout.float())
    return g.double()


@pytest.mark.parametrize('variant', [1, 0])       # 1 = mma.sync TF32x3 (default), 0 = fp32 CUDA cores
@pytest.mark.parametrize('case', BWD_CASES, ids=case_id)
def test_attention_backward_vs_float64(case, variant):
    from e2e_multi_view_matching_b200 import ops, _lib
    B, T, n_pad, counts, is_cross, regime = case
    qkv = make_qkv(case)
    g = torch.Generator().manual_seed(zlib.crc32(case_id(case).encode()))
    dout = torch.randn(B * T, n_pad, 256, generator=g)
    for v in range(B * T):
        dout[v, counts[v % T]:] = 0          # the gradient of padding rows is zero by construction
    out = emul_ops.attention(qkv, B, T, counts, is_cross)
    ref = emul_ops.attention_backward(qkv, out, dout, B, T, counts, is_cross).double()
    ref32 = fp32_backward(qkv, out, dout, B, T, counts, is_cross)
    _lib.lib().mvm_debug_set_attention_backward_variant(variant)
    try:
        got = ops.attention_backward(qkv.cuda(), out.cuda(), dout.cuda(), B, T, list(counts), is_cross)
        torch.cuda.synchronize()
    finally:
        _lib.lib().mvm_debug_set_attention_backward_variant(1)
    got = got.cpu().double()
    # dS = P (dP - D) with D = rowsum(dO * O) from the given O, not from the kernel's own P dP: where they nearly cancel,
    # the rounding of the two 64-term dot products is left, times |k| / 8 in dq, and times |q| / 8 and the key's
    # attention mass sum_i P_ij in dk
    dpd = 2.0 ** -24 * 64 * float(dout.abs().max()) * float(qkv[..., 512:].abs().max()) / 8
    cancel = {'dq': dpd * float(qkv[..., 256:512].abs().max()),
              'dk': dpd * float(qkv[..., :256].abs().max()) * column_mass(qkv, B, T, counts, is_cross), 'dv': 0.0}
    for name, lo in (('dq', 0), ('dk', 256), ('dv', 512)):
        cols = slice(lo, lo + 256)
        scale = float(ref[:, :, cols].abs().max())
        if name == 'dq' and regime == 'flat':
            scale = dq_gross(qkv, dout, B, T, counts, is_cross)
        e = float((got[:, :, cols] - ref[:, :, cols]).abs().max()) / scale
        noise = float((ref32[:, :, cols] - ref[:, :, cols]).abs().max()) / scale
        lim = 2e-5 + 3.0 * noise + 0.5 * cancel[name] / scale
        print('%s variant %d %s rel err %.2e (bound %.2e, fp32 noise %.2e)'
              % (case_id(case), variant, name, e, lim, noise))
        assert e < lim, (name, e, lim)
    for v in range(B * T):
        assert (got[v, counts[v % T]:] == 0).all(), v
