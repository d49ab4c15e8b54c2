"""The tensor-core GEMM (csrc/gemm_tc.cu) against float64, at the shapes, epilogues and operand magnitudes where it goes
wrong.

Kernels, one test per (case, kernel), each reached through its C entry:
  fp16x3          gemm_wg_kernel<128, 3, W_F16>, persistent       mvm_linear_tc_h16 (W as fp16 planes of 64 W)
  tf32x3          gemm_wg_kernel<128, 3, W_TF32>, persistent      mvm_linear_tc_presplit, gemm_kernel 1
  tf32x3_tile128  the same instance, one tile per CTA             gemm_kernel 0, gemm_tile 128
  tf32x3_tile256  gemm_wg_kernel<256, 3, W_TF32>, one tile / CTA  gemm_kernel 0, gemm_tile 256 (N % 256 == 0)
  tf32x3_rawW     gemm_wg_kernel<128, 3, W_RAW>                   mvm_linear_tc, n_pass 3
  tf32            gemm_wg_kernel<256, 1> (N % 256 == 0) or <128, 1>   mvm_linear_tc, n_pass 1
  simt            the fp32 CUDA-core kernel, as the control       mvm_linear
plus split-K (mvm_linear_tc_presplit_splitk) and the score mode (mvm_pair_scores), tested on their own below.

Cases: M on the 64 / 128-row tile edges, at cfg3 (14 x 5 x 1024 rows) and cfg3 - 37, and at n_sm - 1, n_sm, n_sm + 1
and 2 n_sm + 1 tiles of the persistent schedule; 1, 2, 3 and 8 k-blocks (BK is 32 for tf32, 64 for fp16x3, so odd
counts end the two-k-block trip of the pipelined mainloop half way); concat splits K1 / K2 at 32 and 64; N from 128 to
768; leading dimensions wider than the logical widths; alpha 1/16 and 3, bias, relu, residual separate or aliased to C.
Regimes: randn at scales 1 and 6, A at 2^e (|a| in [2^e, 2^(e+1))) for e in -16 .. 14 against W at 2^-10, 1/16 and 2^6,
rows that mix one column at 2^10 with the rest at 2^-10, cancellation rows (A and W in orthogonal subspaces: the exact
result is the rounding residue of the operands, near zero), and L2-normalised rows (SuperPoint descriptors).

Yardstick: the same operation in float64 on the GPU.  Every element must stay within
    3 x noise + f |alpha| sum_k |a_k| |w_k| + 2^-23 (|bias| + |r|)
where noise is that element's error in float32 (torch, TF32 disabled), and f = 2^-19 for the split modes (3xTF32,
fp16x3, split-K, score mode), 2^-20 for the fp32 control and 2^-9 for single-pass TF32.  The split modes hold both
operands to 22 bits, so their error follows sum |a||w| rather than the fp32 noise (the cancellation rows show it: noise
is tiny there).  f = 2^-20 was the first choice; 3xTF32 reached 1.4 x that bound on randn at cfg3 and 1.2 x at K = 512,
hence 2^-19.  Two terms cover the fp32 accumulation where the blocked float32 reference rounds less than a sequential
sum: rows dominated by one product (the mixed regime) add K 2^-24 max|a| max|w|, which the fp32 control needed too
(1.6 x without it), and split-K adds 4 sqrt(n) 2^-24 sum |a||w| for its chain of n = K / (8 ksplit) + ksplit roundings
(one K = 17920 case reached 3.2 x without it).  Split-K is also pinned exactly: its output is bitwise the fixed-order
fp32 sum of the persistent kernel's products over the K slices, so it carries that kernel's precision.

Largest error as a share of the bound on an H100 80GB HBM3 (400 W and 700 W power limits, the same to the digits
given): 3xTF32 0.70 (every schedule and W form, cfg3 randn), single-pass TF32 0.48, fp32 control 0.31, fp16x3 0.43
outside the magnitude edge (0.20-0.34 with A from 2^-7 to 2^14 on every W scale, 0.57 at 2^-8), split-K 0.35, score
mode 0.59.  The range cases run without a bias: far below |bias| its 2^-23 term would set the bound and the rounding
of the output the error, hiding the GEMM's own.

fp16x3 leaves the bound once A is small: lo = fp16(a - hi) is an fp16 subnormal for |a| < 2^-3, exact to 2^-24 absolute
only.  On the H100, with |a| in [2^e, 2^(e+1)), the share against all three W scales is at most 0.57 for e >= -8,
0.92-1.10 at e = -9, 2.0-2.1 at e = -10, and doubles with each further halving of A, to 124-136 at e = -16.  e <= -10
are strict xfails, as is |a| >= 2^16, where hi = fp16(a) is inf; e = -9 is not run for fp16x3.
"""
import ctypes as C
import functools
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N_SM = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
CFG3 = 14 * 5 * 1024

KERNELS = ('fp16x3', 'tf32x3', 'tf32x3_tile128', 'tf32x3_tile256', 'tf32x3_rawW', 'tf32', 'simt')
BK = {'fp16x3': 64, 'simt': 16}                 # k-block; 32 for the tf32 kernels
F_SPLIT, F_FP32, F_TF32 = 2.0 ** -19, 2.0 ** -20, 2.0 ** -9

# fp16x3 against A at 2^e: lo = fp16(a - hi) is an fp16 subnormal once |a| < 2^-3, exact to 2^-24 absolute only, and
# the share of the bound doubles with each halving of A.  e >= -8 stays inside, e <= FP16X3_LOW_EXP leaves it (strict
# xfails), and e = -9, the crossing itself (0.9-1.1 of the bound), is not run for fp16x3: neither outcome has a margin.
# hi = fp16(a) overflows at |a| >= 65520 (e = FP16X3_OVERFLOW_EXP).
FP16X3_LOW_EXP, FP16X3_EDGE_EXP = -10, -9
FP16X3_OVERFLOW_EXP = 16


def case(M=129, N=256, K1=256, K2=0, pa=0, pw=0, pc=0, pr=0, alpha=1.0, bias=True, relu=False, res=None,
         regime='randn1'):
    return (M, N, K1, K2, pa, pw, pc, pr, alpha, bias, relu, res, regime)


def case_id(c):
    M, N, K1, K2, pa, pw, pc, pr, alpha, bias, relu, res, regime = c
    s = 'M%d_N%d_K%d' % (M, N, K1) + ('+%d' % K2 if K2 else '')
    if pa or pw or pc or pr:
        s += '_ld+%d+%d+%d+%d' % (pa, pw, pc, pr)
    if alpha != 1.0:
        s += '_a%g' % alpha
    s += ('_bias' if bias else '_nobias') + ('_relu' if relu else '') + ('_r' + res if res else '')
    return s + '_' + regime


CASES = []
for _m in (1, 63, 64, 65, 127, 128, 129, 191):
    CASES.append(case(M=_m))
for _m in (CFG3, CFG3 - 37):
    CASES.append(case(M=_m, N=768))
for _t in (N_SM - 1, N_SM, N_SM + 1, 2 * N_SM + 1):          # tiles of the persistent schedule at N = 128
    CASES.append(case(M=128 * _t - 5, N=128, res='sep'))
for _k in (32, 64, 96, 128, 192, 256, 512):                  # 1, 2, 3, 4, 6, 8 (fp16: 1, 2, 3, 4, 8) k-blocks
    CASES.append(case(M=129, N=128, K1=_k))
for _k1, _k2 in ((32, 224), (64, 192), (128, 128), (192, 64), (224, 32)):
    CASES.append(case(M=191, N=256, K1=_k1, K2=_k2, relu=True))
for _n in (128, 256, 384, 512, 768):
    CASES.append(case(M=191, N=_n))
CASES += [case(M=191, N=256, pa=4, pw=8, pc=4, pr=12, res='sep'), case(M=191, N=384, pa=32, pw=64, pc=128, pr=4, res='sep'),
          case(M=191, N=512, K1=256, K2=256, pa=8, pw=16, pc=4, relu=True), case(M=191, N=256, pc=4, res='alias')]
for _alpha in (1.0 / 16.0, 3.0):
    for _bias in (False, True):
        for _relu in (False, True):
            for _res in (None, 'sep', 'alias'):
                CASES.append(case(M=191, N=256, alpha=_alpha, bias=_bias, relu=_relu, res=_res))
CASES += [case(M=191, N=384, regime='randn6'), case(M=191, N=256, K1=256, K2=256, relu=True, res='sep', regime='randn6'),
          case(M=191, N=256, regime='mixed'), case(M=191, N=384, regime='cancel'), case(M=191, N=768, regime='l2rows'),
          case(M=CFG3 - 37, N=768, regime='l2rows')]
A_EXPS = tuple(range(-16, 15)) + (FP16X3_OVERFLOW_EXP,)
W_EXPS = (-10, -4, 6)
for _ea in A_EXPS:
    for _ew in W_EXPS:
        # no bias: far below |bias| its 2^-23 term would set the bound and the output's rounding the error
        CASES.append(case(M=129, N=256, bias=False, regime='range_a%d_w%d' % (_ea, _ew)))


def range_exps(regime):
    a, w = regime.split('_')[1:]
    return int(a[1:]), int(w[1:])


def supports(c, k):
    M, N, K1, K2 = c[:4]
    bk = BK.get(k, 32)
    if K1 % bk or K2 % bk:
        return False
    if k == 'tf32x3_tile256' and N % 256:
        return False                                      # would run the 128-column instance again
    if k == 'simt' and c[12].startswith('range') and range_exps(c[12])[0] not in (-16, 0, 14):
        return False                                      # the fp32 control once per W scale and edge
    if k == 'fp16x3' and c[12].startswith('range') and range_exps(c[12])[0] == FP16X3_EDGE_EXP:
        return False
    return True


def marks_for(c, k):
    regime = c[12]
    if k == 'fp16x3' and regime.startswith('range'):
        ea, ew = range_exps(regime)
        if ea >= FP16X3_OVERFLOW_EXP:
            return [pytest.mark.xfail(strict=True, reason='|a| >= 65520: hi = fp16(a) is inf')]
        if ea <= FP16X3_LOW_EXP:
            return [pytest.mark.xfail(strict=True, reason='|a| below the fp16x3 edge: the lo plane of A is an fp16 '
                                                          'subnormal')]
    return []


KERNEL_CASES = [pytest.param(c, k, id='%s-%s' % (case_id(c), k), marks=marks_for(c, k))
                for c in CASES for k in KERNELS if supports(c, k)]


def make_operands(c):
    """Seeded float32 CPU operands of a case: A [M, K], W [N, K], bias [N] or None, r [M, N] or None."""
    M, N, K1, K2, pa, pw, pc, pr, alpha, bias, relu, res, regime = c
    K = K1 + K2
    g = torch.Generator().manual_seed(zlib.crc32(case_id(c).encode()))
    A = torch.randn(M, K, generator=g, dtype=torch.float64)
    W = torch.randn(N, K, generator=g, dtype=torch.float64) / 16
    if regime.startswith('randn'):
        A *= float(regime[5:])
    elif regime.startswith('range'):
        ea, ew = range_exps(regime)
        A = torch.sign(A) * 2.0 ** ea * (1 + torch.rand(M, K, generator=g, dtype=torch.float64))
        W = torch.randn(N, K, generator=g, dtype=torch.float64) * 2.0 ** ew
    elif regime == 'mixed':                               # one large column per row, the rest tiny
        A = A * 2.0 ** -10
        A[torch.arange(M), torch.randint(0, K, (M,), generator=g)] = 2.0 ** 10
    elif regime == 'cancel':                              # rows of A orthogonal to rows of W
        Q, _ = torch.linalg.qr(torch.randn(K, K, generator=g, dtype=torch.float64))
        A = torch.randn(M, K // 2, generator=g, dtype=torch.float64) @ Q[:, :K // 2].T
        W = torch.randn(N, K // 2, generator=g, dtype=torch.float64) @ Q[:, K // 2:].T / 16
    elif regime == 'l2rows':                              # SuperPoint descriptors: unit rows
        A = A / A.norm(dim=1, keepdim=True)
    else:
        raise AssertionError(regime)
    b = torch.randn(N, generator=g, dtype=torch.float64) if bias else None
    r = torch.randn(M, N, generator=g, dtype=torch.float64) if res else None
    f = (lambda t: None if t is None else t.float())
    return f(A), f(W), f(b), f(r)


def epilogue(x, alpha, b, relu, r):
    x = alpha * x
    if b is not None:
        x = x + b
    if relu:
        x = torch.relu(x)
    if r is not None:
        x = x + r
    return x


@functools.lru_cache(maxsize=1)            # the kernels of a case run one after the other
def reference(c):
    """float64 result, and the per-element bound without its f term and the f term's sum_k |a_k||w_k| (on the GPU)."""
    alpha, relu = c[8], c[10]
    A, W, b, r = (t.cuda() if t is not None else None for t in make_operands(c))
    d = (lambda t: None if t is None else t.double())
    ref = epilogue(d(A) @ d(W).T, alpha, d(b), relu, d(r))
    prev = torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cuda.matmul.allow_tf32 = False
        r32 = epilogue(A @ W.T, alpha, b, relu, r).double()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    noise = (r32 - ref).abs()
    sabs = abs(alpha) * (d(A).abs() @ d(W).abs().T)
    base = 3.0 * noise
    if c[12] == 'mixed':
        # one product dominates each row: every later fp32 addition rounds at its magnitude, whatever order the
        # reference's float32 sum took (K additions of at most 2^-24 max_k |a_k| |w_k|)
        K = c[2] + c[3]
        base = base + K * 2.0 ** -24 * abs(alpha) * (A.abs().max(1).values.double()[:, None] *
                                                     W.abs().max(1).values.double()[None, :])
    extra = torch.zeros_like(ref)
    if b is not None:
        extra = extra + d(b).abs()
    if r is not None:
        extra = extra + d(r).abs()
    return ref, base + 2.0 ** -23 * extra, sabs


def vp(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def padded(t, pad, dtype=None):
    """A GPU copy of the 2-D tensor t as a column slice of a buffer `pad` columns wider (filled with junk)."""
    rows, cols = t.shape
    buf = torch.full((rows, cols + pad), 7.0e3, dtype=dtype or t.dtype, device='cuda')
    buf[:, :cols] = t.to(buf.dtype).cuda()
    return buf[:, :cols]


SETTERS = {'tf32x3': (1, 256), 'tf32x3_tile128': (0, 128), 'tf32x3_tile256': (0, 256)}


def run_gemm(k, A, W, b, r, c):
    """One launch of kernel k on the case's layout -> C [M, N] (a column slice of a wider buffer when pc > 0)."""
    from e2e_multi_view_matching_b200 import _lib, ops
    M, N, K1, K2, pa, pw, pc, pr, alpha, bias, relu, res, _ = c
    K = K1 + K2
    lib = _lib.lib()
    a1 = padded(A[:, :K1], pa)
    a2 = padded(A[:, K1:], pa) if K2 else None
    out = padded(torch.zeros(M, N), pc)
    if res == 'alias':
        out[:] = r.cuda()
        rr = out
    else:
        rr = padded(r, pr) if r is not None else None
    bb = b.cuda() if b is not None else None
    ld = (lambda t: 0 if t is None else t.stride(0))
    common = (vp(a1), ld(a1), vp(a2), ld(a2), K1)
    tail = (vp(bb), vp(rr), ld(rr), vp(out), ld(out), M, N, K, float(alpha), int(relu))
    s = _lib.stream_ptr()
    if k == 'fp16x3':
        wb = torch.full((N, K + pw), 700.0, dtype=torch.float64)       # junk inside the fp16 range of 64 W
        wb[:, :K] = W.double()
        hi, lo = ops.h16_planes(wb.cuda())
        rc = lib.mvm_linear_tc_h16(*common, vp(hi), vp(lo), ops.H16_SCALE, hi.stride(0), *tail, s)
    elif k in SETTERS:
        hi = padded(ops.rn_tf32(W.cuda()), pw)
        lo = padded(ops.rn_tf32(W.cuda() - ops.rn_tf32(W.cuda())), pw)
        persist, tile = SETTERS[k]
        try:
            lib.mvm_debug_set_gemm_kernel(persist)
            lib.mvm_debug_set_gemm_tile(tile)
            rc = lib.mvm_linear_tc_presplit(*common, vp(hi), vp(lo), hi.stride(0), *tail, s)
        finally:
            lib.mvm_debug_set_gemm_kernel(1)
            lib.mvm_debug_set_gemm_tile(256)
    elif k in ('tf32x3_rawW', 'tf32'):
        wf = padded(W, pw)
        rc = lib.mvm_linear_tc(*common, vp(wf), wf.stride(0), *tail, 3 if k == 'tf32x3_rawW' else 1, s)
    else:
        wf = padded(W, pw)
        rc = lib.mvm_linear(*common, vp(wf), wf.stride(0), *tail, s)
    _lib.check(rc, k)
    torch.cuda.synchronize()
    return out


def f_of(k):
    return {'tf32': F_TF32, 'simt': F_FP32}.get(k, F_SPLIT)


@pytest.mark.parametrize('c,k', KERNEL_CASES)
def test_gemm_vs_float64(c, k):
    A, W, b, r = make_operands(c)
    ref, base, sabs = reference(c)
    out = run_gemm(k, A, W, b, r, c)
    assert torch.isfinite(out).all()
    lim = base + f_of(k) * sabs
    err = (out.double() - ref).abs()
    share = float((err / lim).max())
    print('%s %-14s max err / bound %.4f' % (case_id(c), k, share))
    bad = int((err > lim).sum())
    assert bad == 0, (bad, share)
    # a fixed summation order: the same input gives the same bits
    assert torch.equal(run_gemm(k, A, W, b, r, c), out), k
    if k in ('tf32x3_tile128', 'tf32x3_tile256'):
        # the persistent and one-tile schedules issue the same instructions per tile
        assert torch.equal(run_gemm('tf32x3', A, W, b, r, c), out), k


@pytest.mark.parametrize('k', ['fp16x3', 'tf32x3', 'tf32x3_tile128', 'tf32x3_tile256', 'tf32x3_rawW', 'tf32', 'simt'])
@pytest.mark.parametrize('relu', [False, True])
def test_residual_in_place_is_bitwise(k, relu):
    """R == C (every GNN layer's mlp.1) gives the bits of a separate residual buffer, in both epilogues."""
    c_sep = case(M=191, N=256, relu=relu, res='sep', pr=0)
    c_alias = case(M=191, N=256, relu=relu, res='alias')
    A, W, b, r = make_operands(c_sep)
    sep = run_gemm(k, A, W, b, r, c_sep)
    alias = run_gemm(k, A, W, b, r, c_alias)
    assert torch.equal(sep, alias), k


@pytest.mark.parametrize('k', ['tf32x3', 'fp16x3'])
@pytest.mark.parametrize('M', [CFG3, CFG3 - 37])
def test_persistent_rows_match_one_tile_launch(k, M):
    """Rows of a launch in which every CTA walks many tiles equal the same rows of a launch with one tile per CTA."""
    c = case(M=M, N=768, res='sep', relu=True)
    A, W, b, r = make_operands(c)
    full = run_gemm(k, A, W, b, r, c)
    for r0, r1 in ((0, 256), (M // 2 - 77, M // 2 + 179), (M - 200, M)):
        cs = case(M=r1 - r0, N=768, res='sep', relu=True)
        small = run_gemm(k, A[r0:r1], W, b, r[r0:r1], cs)
        assert torch.equal(small, full[r0:r1]), (k, M, r0, r1)


# ---- split-K: mvm_linear_tc_presplit_splitk (the weight gradients of training)

SPLITK = []
for _ks in (2, 3, 7, 64):
    for _kb, (_m, _n) in zip((1, 2, 3), ((128, 768), (768, 128), (768, 768))):
        SPLITK.append((_m, _n, 32 * _ks * _kb, _ks))
SPLITK += [(128, 128, 17920, 2), (768, 768, 17920, 7), (128, 768, 17920, 35)]


def run_splitk(A, W, ksplit, alpha=1.0):
    from e2e_multi_view_matching_b200 import ops
    out = ops.linear_presplit_splitk(A.cuda(), ops.rn_tf32(W.cuda()), ops.rn_tf32(W.cuda() - ops.rn_tf32(W.cuda())),
                                     ksplit, alpha=alpha)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize('M,N,K,ksplit', SPLITK, ids=['M%d_N%d_K%d_s%d' % s for s in SPLITK])
def test_splitk_vs_float64(M, N, K, ksplit):
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K + ksplit)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / 16
    alpha = 0.5
    out = run_splitk(A, W, ksplit, alpha)
    A64, W64 = A.double().cuda(), W.double().cuda()
    ref = alpha * (A64 @ W64.T)
    prev = torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cuda.matmul.allow_tf32 = False
        noise = (alpha * (A.cuda() @ W.cuda().T)).double() - ref
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    sabs = alpha * (A64.abs() @ W64.abs().T)
    # + the fp32 accumulation chain of an element, n = K / (8 ksplit) wgmma k-steps per slice and then the ksplit slice
    # results: a long contraction's sequential sum outgrows the blocked float32 sum the noise is measured on.  Its n
    # roundings of at most 2^-24 sum |a||w| each add up as a random walk: 4 sqrt(n) of them.
    lim = 3.0 * noise.abs() + (F_SPLIT + 4.0 * (K // (8 * ksplit) + ksplit) ** 0.5 * 2.0 ** -24) * sabs
    err = (out.double() - ref).abs()
    print('splitk M%d N%d K%d s%d max err / bound %.4f' % (M, N, K, ksplit, float((err / lim).max())))
    assert int((err > lim).sum()) == 0
    assert torch.equal(run_splitk(A, W, ksplit, alpha), out)          # deterministic
    # rows of the many-tile launch equal the same rows computed by a launch over only them
    part = run_splitk(A[M - 128:], W, ksplit, alpha)
    assert torch.equal(part, out[M - 128:])
    # exactly the sum, slice by slice in fixed order, of the persistent kernel's product over each K slice: split-K
    # inherits that kernel's precision, which the float64 cases above pin at K <= 512
    assert torch.equal(out, splitk_by_slices(A, W, ksplit, alpha))


def splitk_by_slices(A, W, ksplit, alpha):
    from e2e_multi_view_matching_b200 import _lib, ops
    M, K = A.shape
    N, ks = W.shape[0], K // ksplit
    a, whi = A.cuda(), ops.rn_tf32(W.cuda())
    wlo = ops.rn_tf32(W.cuda() - whi)
    total = None
    for s in range(ksplit):
        part = torch.empty(M, N, device='cuda')
        cols = slice(s * ks, (s + 1) * ks)           # column slices: lda = ldw = K
        try:
            _lib.lib().mvm_debug_set_gemm_kernel(1)
            _lib.check(_lib.lib().mvm_linear_tc_presplit(vp(a[:, cols]), K, C.c_void_p(0), 0, ks, vp(whi[:, cols]),
                                                         vp(wlo[:, cols]), K, C.c_void_p(0), C.c_void_p(0), 0, vp(part),
                                                         N, M, N, ks, float(alpha), 0, _lib.stream_ptr()),
                       'mvm_linear_tc_presplit')
        finally:
            _lib.lib().mvm_debug_set_gemm_kernel(1)
        total = part if total is None else total + part
    torch.cuda.synchronize()
    return total


@pytest.mark.parametrize('what,M,N,K,ksplit', [('M_not_128', 100, 128, 256, 2), ('N_not_128', 128, 100, 256, 2),
                                               ('K_not_sliced', 128, 128, 96, 2), ('ksplit_1', 128, 128, 256, 1),
                                               ('ksplit_0', 128, 128, 256, 0)])
def test_splitk_refuses(what, M, N, K, ksplit):
    from e2e_multi_view_matching_b200 import _lib
    lib = _lib.lib()
    A = torch.zeros(128, 256, device='cuda')
    W = torch.zeros(128, 256, device='cuda')
    out = torch.zeros(128, 128, device='cuda')
    ws = torch.zeros(4 * 128 * 128, device='cuda')
    rc = lib.mvm_linear_tc_presplit_splitk(vp(A), 256, vp(W), vp(W), 256, vp(out), 128, M, N, K, 1.0, ksplit, vp(ws),
                                           _lib.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 1, what


# Refusals on the GPU, limited to calls that stay harmless even if their check went missing: on the tensor cores M = 0
# and K = 0 fail the tensor-map encode on the host, N = 100 holds no whole 128-column tile (no CTA would run), and
# K = 48 (40 on the CUDA cores) reads only k-blocks inside the buffers.  K = 0 is not launched on the CUDA-core kernel:
# without its check that kernel would load its first k-block from A2 = NULL.  That refusal, and misaligned pointers, are
# checked on the CPU only (tests/test_gemm_args.py).
REFUSED = {'M0': dict(M=0), 'K0': dict(K=0), 'N_not_128': dict(N=100), 'K_not_kblock': dict(K=48)}


@pytest.mark.parametrize('k', ['fp16x3', 'tf32x3', 'tf32x3_rawW', 'tf32', 'simt'])
@pytest.mark.parametrize('what', list(REFUSED))
def test_gemm_refuses(what, k):
    from e2e_multi_view_matching_b200 import _lib, ops
    lib = _lib.lib()
    d = dict(M=128, N=128, K=128)
    d.update(REFUSED[what])
    if k == 'simt' and what == 'N_not_128':
        pytest.skip('the CUDA-core kernel takes any N')
    if k == 'simt' and what == 'K0':
        pytest.skip('would fault if the check regressed: checked on the CPU (tests/test_gemm_args.py)')
    if k == 'simt' and what == 'K_not_kblock':
        d['K'] = 40
    M, N, K = d['M'], d['N'], d['K']
    A = torch.zeros(128, 128, device='cuda')
    W = torch.zeros(128, 128, device='cuda')
    out = torch.zeros(128, 128, device='cuda')
    hi, lo = ops.h16_planes(W)
    s = _lib.stream_ptr()
    common = (vp(A), 128, C.c_void_p(0), 0, K)
    tail = (C.c_void_p(0), C.c_void_p(0), 0, vp(out), 128, M, N, K, 1.0, 0)
    if k == 'fp16x3':
        rc = lib.mvm_linear_tc_h16(*common, vp(hi), vp(lo), 64.0, 128, *tail, s)
    elif k == 'tf32x3':
        rc = lib.mvm_linear_tc_presplit(*common, vp(W), vp(W), 128, *tail, s)
    elif k in ('tf32x3_rawW', 'tf32'):
        rc = lib.mvm_linear_tc(*common, vp(W), 128, *tail, 3 if k == 'tf32x3_rawW' else 1, s)
    else:
        rc = lib.mvm_linear(*common, vp(W), 128, *tail, s)
    torch.cuda.synchronize()
    assert rc == 1, (what, k, rc)
    assert (out == 0).all()


# ---- score mode: mvm_pair_scores with a per-pair (m, n) table

SENTINEL = -1234.5
GAP = 67                                       # floats between two pairs' buffers, checked to stay untouched


def score_cases():
    vals = (1, 63, 64, 65, 127, 128, 129, 1023, 1024)
    out = []
    for n_pad, T in ((64, 3), (192, 4), (448, 3), (1024, 3)):
        v = [x for x in vals if x <= n_pad] + [n_pad]
        pairs = []
        i = 0
        for a in range(T):
            for b in range(T):
                if a != b:                                    # both (a, b) and (b, a); the last slot included
                    pairs.append((a, b, v[i % len(v)], v[(i * 5 + 3) % len(v)]))
                    i += 1
        for j in range(max(0, min(28, 2 * len(v)) - len(pairs))):
            a, b = (T - 1, 0) if j % 2 else (0, T - 1)
            pairs.append((a, b, v[i % len(v)], v[(i * 7 + 1) % len(v)]))
            i += 1
        out.append((3, T, n_pad, tuple(pairs)))
    return out


SCORE_CASES = score_cases()


@pytest.mark.parametrize('sc', SCORE_CASES, ids=['B%d_T%d_npad%d' % s[:3] for s in SCORE_CASES])
def test_pair_scores_vs_float64(sc):
    from e2e_multi_view_matching_b200 import _lib
    B, T, n_pad, pairs = sc
    lib = _lib.lib()
    g = torch.Generator().manual_seed(n_pad * 31 + T)
    md = torch.randn(B, T, n_pad, 256, generator=g).cuda()
    alpha = 1.0 / 16.0
    sizes = [B * (m + 1) * (n + 1) for _, _, m, n in pairs]
    offs = np.concatenate([[0], np.cumsum([(s + GAP + 3) // 4 * 4 for s in sizes])]).astype(int)
    flat = torch.full((int(offs[-1]) + GAP,), SENTINEL, device='cuda')
    hi, lo = torch.empty_like(md), torch.empty_like(md)
    P = len(pairs)
    I = C.c_int * P
    ptrs = (C.c_void_p * P)(*[flat[int(o):].data_ptr() for o in offs[:-1]])
    rc = lib.mvm_pair_scores(vp(md), vp(hi), vp(lo), B, T, n_pad, P, I(*[p[0] for p in pairs]), I(*[p[1] for p in pairs]),
                             I(*[p[2] for p in pairs]), I(*[p[3] for p in pairs]), ptrs, alpha, _lib.stream_ptr())
    _lib.check(rc, 'mvm_pair_scores')
    torch.cuda.synchronize()
    touched = torch.zeros_like(flat, dtype=torch.bool)
    md64 = md.double()
    worst = 0.0
    for p, (a, b, m, n) in enumerate(pairs):
        o = int(offs[p])
        buf = flat[o:o + sizes[p]].view(B, m + 1, n + 1)
        for bi in range(B):
            A, W = md64[bi, a, :m], md64[bi, b, :n]
            ref = alpha * (A @ W.T)
            prev = torch.backends.cuda.matmul.allow_tf32
            try:
                torch.backends.cuda.matmul.allow_tf32 = False
                noise = (alpha * (md[bi, a, :m] @ md[bi, b, :n].T)).double() - ref
            finally:
                torch.backends.cuda.matmul.allow_tf32 = prev
            lim = 3.0 * noise.abs() + F_SPLIT * alpha * (A.abs() @ W.abs().T)
            err = (buf[bi, :m, :n].double() - ref).abs()
            worst = max(worst, float((err / lim).max()))
            assert int((err > lim).sum()) == 0, (a, b, m, n, bi)
        inner = touched[o:o + sizes[p]].view(B, m + 1, n + 1)
        inner[:, :m, :n] = True
    # the dustbin row and column of every buffer, and the gaps between buffers, keep their bits
    assert (flat[~touched] == SENTINEL).all()
    print('scores B%d T%d n_pad %d max err / bound %.4f' % (B, T, n_pad, worst))


# ---- the QKV projection's operand planes (mvm_qkv_projection), bitwise against a plain launch of the same kernel

QKV_SHAPES = [(2, 3, 192), (1, 5, 448), (2, 2, 64)]      # (B, T, n_pad): rows = B T n_pad, several slabs


def qkv_operands(B, T, n_pad, scale=1.0):
    g = torch.Generator().manual_seed(B * 100 + T * 10 + n_pad)
    x = (torch.randn(B * T * n_pad, 256, generator=g) * scale).cuda()
    w = (torch.randn(768, 256, generator=g) / 16).cuda()
    b = torch.randn(768, generator=g).cuda()
    return x, w, b


@pytest.mark.parametrize('w16', [True, False], ids=['fp16_gemm', 'tf32_gemm'])
@pytest.mark.parametrize('shape', QKV_SHAPES, ids=['B%d_T%d_npad%d' % s for s in QKV_SHAPES])
def test_qkv_fp16_planes_bitwise(shape, w16):
    from e2e_multi_view_matching_b200 import ops
    B, T, n_pad = shape
    x, w, b = qkv_operands(B, T, n_pad)
    fill = torch.full((x.shape[0], 768), 3.0e4, device='cuda')
    qkv, (kh, kl, vh, vl) = ops.qkv_projection(x, w, b, n_pad, planes='fp16', w16=w16, out=fill.clone())
    plain = ops.linear(x, w, bias=b, tc_passes='h16') if w16 else ops.linear(x, w, bias=b, tc_passes=3, presplit=True)
    torch.cuda.synchronize()
    assert torch.equal(qkv[:, :256], plain[:, :256])
    assert torch.equal(qkv[:, 256:], fill[:, 256:])            # K and V leave as planes only
    for hi, lo, cols in ((kh, kl, slice(256, 512)), (vh, vl, slice(512, 768))):
        x_ = plain[:, cols].contiguous()
        assert torch.equal(hi, x_.half())
        assert torch.equal(lo, (x_ - x_.half().float()).half())
    # the planes feed the fp16x3 attention exactly as ops.attention builds them from the fp32 projection
    counts = [n_pad - 5 * t for t in range(T)]
    for is_cross in (0, 1):
        from e2e_multi_view_matching_b200 import _lib
        out = torch.zeros(B * T, n_pad, 256, device='cuda')
        cnt = (C.c_int * T)(*counts)
        _lib.check(_lib.lib().mvm_attention_h3(vp(qkv), vp(kh), vp(kl), vp(vh), vp(vl), vp(out), B, T, n_pad, cnt,
                                               is_cross, _lib.stream_ptr()), 'mvm_attention_h3')
        want = ops.attention(plain.view(B * T, n_pad, 768), B, T, counts, is_cross, tc_passes='h3')
        torch.cuda.synchronize()
        for v in range(B * T):
            assert torch.equal(out[v, :counts[v % T]], want[v, :counts[v % T]]), (is_cross, v)


@pytest.mark.parametrize('kernel', [(1, 256), (0, 128), (0, 256)], ids=['persistent', 'tile128', 'tile256'])
@pytest.mark.parametrize('shape', QKV_SHAPES, ids=['B%d_T%d_npad%d' % s for s in QKV_SHAPES])
def test_qkv_tf32_planes_bitwise(shape, kernel):
    from e2e_multi_view_matching_b200 import _lib, ops
    B, T, n_pad = shape
    x, w, b = qkv_operands(B, T, n_pad)
    lib = _lib.lib()
    fill = torch.full((x.shape[0], 768), 3.0e4, device='cuda')
    try:
        lib.mvm_debug_set_gemm_kernel(kernel[0])
        lib.mvm_debug_set_gemm_tile(kernel[1])
        qkv, (klo, vt, vtlo) = ops.qkv_projection(x, w, b, n_pad, planes='tf32', out=fill.clone())
        plain = ops.linear(x, w, bias=b, tc_passes=3, presplit=True)
        torch.cuda.synchronize()
    finally:
        lib.mvm_debug_set_gemm_kernel(1)
        lib.mvm_debug_set_gemm_tile(256)
    assert torch.equal(qkv[:, :256], plain[:, :256])
    k = plain[:, 256:512].contiguous()
    assert torch.equal(qkv[:, 256:512], ops.rn_tf32(k))
    assert torch.equal(klo, ops.rn_tf32(k - ops.rn_tf32(k)))
    assert torch.equal(qkv[:, 512:], fill[:, 512:])              # V leaves as V^T only
    v_t = plain[:, 512:].reshape(B * T, n_pad, 256).transpose(1, 2).contiguous()
    assert torch.equal(vt, ops.rn_tf32(v_t))
    assert torch.equal(vtlo, ops.rn_tf32(v_t - ops.rn_tf32(v_t)))
