"""The kernels every training step runs, against float64, at the shapes and inputs where their work split changes.

Training Sinkhorn (csrc/sinkhorn_train.cu, ops.sinkhorn_train_forward / _backward).  One 1024-thread CTA per problem:
  - column registers: `if (n + 1 <= 13 * 32)` picks KC = 13, else 33 (mvm_sinkhorn_train_forward / _backward):
      n = 415 (31x415) and n = 416 (32x416);
  - column-merge rounds: `for (int c0 = 0; c0 <= n; c0 += CH)` with CH = 416 (forward column pass and merge_columns):
      one round n <= 415; n = 416, the second round holds one column (32x416); n = 831, two full rounds (64x831);
      n = 832, the third round holds one column (100x832); n = 1055 = SK_MAX_N, 33 columns per lane (1x1055, 1055x1055);
  - rows over 32 warps: `for (int i = warp; i <= m; i += 32)`: m = 1, 30 warps keep -inf partials and take lse_merge's
      early exit (1x1, 1x1055); m + 1 = 32 (31x415); m = 32, warp 0 takes two rows (32x416); m = 1055 (1055x1, 1055x1055);
  - shape mix: tall 1000x8, wide 1x1055 and 8x1000, n = 1 (1x1, 1055x1);
  - iterations: iters = 1 leaves the backward's `t > 1 ? ... : 0.f` at v^0 = 0 (100x832), 2 (64x831), 7 (31x415,
      8x1000), 100 (the rest);
  - bin score from -3 (32x416, 50x60) to 5 (1000x8, 100x832 with scores well below it: the dustbins take most mass);
  - score spread 1 (1x1, 200x300), 12, 40 (32x416, 1000x8, 80x400x400) and 300, the untrained network (64x831, 50x60);
  - batch: B = 80 at 400x400 (a cfg5 step's launch) and B = 1;
  - layouts: packed [B, m, n]; the [B, m+1, n+1] buffers of pair_scores with the dustbin row and column NaN; rows of
      stride scores_ld > n with NaN in the padding and between problems (the library called directly).
Couplings [B, m+1, n+1] (dustbins included) against oracle.train_ops._ot in float64 with the yardstick of
tests/test_sinkhorn_shapes_gpu.py: max(1e-4, 3 x the same function's float32 deviation) + 1e-5 |Z|.  The potentials
(pot [B, iters, m+n+2] = u^t | v^t, the layout the backward reads) at t = 1, iters/2 and iters with the same yardstick.
The gradient with respect to the whole augmented matrix (dustbin row and column included) against float64 autograd
with the augmented matrix as one leaf, checkpointed per iteration (sk_grad below): max(1e-5 max|dZ|, 3 x the float32
deviation of either way to compute it), the float32 autograd or the reverse recursion the kernel runs (sk_recursion,
equal to autograd in float64).  The recursion rounds more: at spread 300 (50x60, max|dZ| 22) it is 3.5e-2 off in
float32 where autograd is 1.9e-3 off, and the kernel's own error (1.7e-2) followed it, 3.0 x the autograd-only
bound; at 80x400x400 spread 40 1.9e-2 against 4.3e-3 for autograd and 1.7e-2 for the recursion.  d_alpha, the sum of
the dustbin entries, within max(1e-5 sum|dustbin dZ|, 3 x the larger float32 deviation).  At B = 80 three problems are
compared with float64, and every problem run alone must give the bits it gets in the batch.

BatchNorm in training mode (csrc/bn_train.cu, ops.batchnorm_train / _backward; the library directly for ld > C):
  - channels: one thread per channel in `((C + 31) / 32) * 32` threads: C = 1, 31, 33, 96, 256, 512, 1024; 1025 refused;
  - row split: `blocks = rows < max_blocks ? rows : max_blocks` with max_blocks = 4 SMs (528 on an H100 SXM) forward and
      592 backward: 300 rows (one row per block in both), 560 rows (two rows per forward block with a remainder, one per
      backward block), 17920 rows = 40 x 448 with 400 valid (cfg5), 32000 rows = 10 groups of 3200 unpadded rows (the
      confidence head);
  - masks `r % n_pad >= n_valid || (r / n_pad) % slot_mod != slot_rem`: n_valid = 1 (count 2, 10 slots in 5 groups),
      n_valid = n_pad, two valid rows in one slot (count 2: the unbiased factor is 2); slot_mod 1, 2, 3, 5, 10, every
      slot_rem;
  - shifted double sums (`shift = sums[2 * C + c]`, the first row of the group's first slot): 'edge' inputs hold, by
      channel, normal values, |mean| / std = 1e3 of both signs, a constant channel (invstd = 1 / sqrt(eps)) and an
      outlier in the shift row;
  - momentum 0.1 / 0.01, eps 1e-5 / 1e-3, ReLU on and off.
y per channel within max(1e-5 max(1, |y|), 3 x the deviation of fp32 torch.nn.functional.batch_norm on the same rows);
saved mean within 2^-22 |mean| + 1e-6 std; invstd within 1e-6 relative; running statistics within 1e-6 relative
+ momentum 1e-6 of the statistic's scale, or 3 x fp32 torch's deviation.  The backward on the kernel's saved statistics
and y: dx per channel within max(1e-5 max|dx|, 3 x the same formula's fp32 deviation)
+ 2^-21 |gamma invstd| (|g| + |mean g| + |xhat mean(g xhat)|) per element (dx cancels in groups of two rows), dgamma and dbeta within
(groups + 2) 2^-23 sum |terms| (double sums rounded once per group).  NaN in padding rows and in other groups' rows
reaches nothing; padding rows of an out-of-place y and of dy keep their contents; in-place equals out-of-place.
These cases found that bn_apply_kernel computed y = x scale + (beta - mean scale), which loses ~ulp(mean scale): on the
constant channels (scale = gamma / sqrt(eps)) y was 6e-5 off beta, up to 4.8 x the bound (c256_cfg5, c1024_g3,
head_10x3200), and with |mean| / std ~ 1e4 over two rows 1.7e-3 off (c96_two_rows, 5.1 x), where fp32 torch is exact
or nearly so.  It now subtracts the float mean first and folds the mean's low part into the bias.

mvm_colsum: `blockIdx.y` covers 256 channels, `blocks = rows < 296 ? rows : 296`: C = 1, 255, 256, 257, 768 against
rows = 1, 295, 296, 297, 17920; ld > C, accumulate = 1 and cancelling columns.  The kernel sums in double and rounds once:
within 1 ulp of the float64 sum rounded to float32, + rows max|x| 2^-52.
mvm_transpose_split: 32 x 32 tiles, `(r < R && c < C)` and `if (c >= C || r >= R) continue`: R, C in {1, 31, 32, 33,
100, 1000}, ld > C, and ldo > R through two calls into the halves of one plane (and the concat-by-rows staging of
ops.gemm_dw); raw only, planes only, both.  hi and lo bitwise equal to tf32_rna below, on ties, 0x0fff, all-ones
mantissas, negatives, subnormals and zeros; output entries outside the block keep their sentinels.

Match loss (csrc/train_loss.cu): ft = 2, 401, 1025, 2049 and bs = 80 at ft 401 go through the parametrisation of
tests/test_training_gpu.py; test_match_loss_edges covers dustbin rows and columns, mutual matches (two atomics on one
element), the dustbin corner's two contributions, zero weights, a gradient buffer full of garbage and a reused partial
workspace.

Every case prints its error and its bound.  The tests not marked gpu check the reference helpers on the CPU.
"""
import ctypes as C
import functools
import zlib

import numpy as np
import pytest
import torch
from torch.utils.checkpoint import checkpoint

gpu = pytest.mark.gpu
D, F = torch.float64, torch.float32
EPS32 = 2.0 ** -23


def vp(t):
    """Raw device pointer of any (strided) tensor."""
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def _stream():
    from e2e_multi_view_matching_b200 import _lib
    return _lib.stream_ptr()


def _check(status, what):
    from e2e_multi_view_matching_b200 import _lib
    _lib.check(status, what)


# ---------------------------------------------------------------------------------------------------------------------
# Training Sinkhorn
# ---------------------------------------------------------------------------------------------------------------------

def _augment(s, alpha):
    b, m, n = s.shape
    a = torch.as_tensor(alpha, dtype=s.dtype)
    return torch.cat([torch.cat([s, a.expand(b, m, 1)], 2), a.expand(b, 1, n + 1)], 1)


def _marginals(m, n, dtype):
    norm = -torch.log(torch.tensor(float(m + n), dtype=dtype))
    log_mu = torch.cat([norm.expand(m), (torch.log(torch.tensor(float(n), dtype=dtype)) + norm)[None]])[None]
    log_nu = torch.cat([norm.expand(n), (torch.log(torch.tensor(float(m), dtype=dtype)) + norm)[None]])[None]
    return norm, log_mu, log_nu


def sk_iterate(Za, iters, keep=(), checkpointed=False):
    """The iteration of oracle.train_ops._ot on an augmented matrix Za [b, m+1, n+1] (any dtype) -> (couplings,
    {t: (u^t, v^t)} for t in keep).  checkpointed: recompute each iteration in the backward instead of keeping its
    log-sum-exp inputs (plain autograd through 100 iterations at 1055^2 keeps several GB)."""
    b, m1, n1 = Za.shape
    norm, log_mu, log_nu = _marginals(m1 - 1, n1 - 1, Za.dtype)

    def step(Z, v):
        u = log_mu - torch.logsumexp(Z + v.unsqueeze(1), dim=2)
        return u, log_nu - torch.logsumexp(Z + u.unsqueeze(2), dim=1)

    v = torch.zeros(b, n1, dtype=Za.dtype)
    pots = {}
    for t in range(1, iters + 1):
        u, v = checkpoint(step, Za, v, use_reentrant=False) if checkpointed else step(Za, v)
        if t in keep:
            pots[t] = (u.detach(), v.detach())
    return Za + u.unsqueeze(2) + v.unsqueeze(1) - norm, pots


def sk_grad(s, alpha, iters, G, keep=(), checkpointed=True):
    """(couplings, potentials, gradient w.r.t. the augmented matrix as one leaf) in the dtype of s."""
    with torch.enable_grad():
        Za = _augment(s, alpha).detach().requires_grad_(True)
        Z, pots = sk_iterate(Za, iters, keep, checkpointed)
        (dZ,) = torch.autograd.grad(Z, Za, G.to(s.dtype))
    return Z.detach(), pots, dZ


def sk_recursion(s, alpha, iters, G):
    """The reverse recursion the kernel runs (the header of csrc/sinkhorn_train.cu), restated in the dtype of s [m, n]
    on the potentials of the forward in that dtype -> the gradient w.r.t. the augmented matrix [m+1, n+1]."""
    m, n = s.shape
    Z = _augment(s[None], alpha)[0]
    _, pots = sk_iterate(Z[None], iters, keep=range(1, iters + 1))
    _, log_mu, log_nu = _marginals(m, n, s.dtype)
    log_mu, log_nu = log_mu[0], log_nu[0]
    dZ = G.to(s.dtype).clone()
    gu, gv = dZ.sum(1), dZ.sum(0)
    for t in range(iters, 0, -1):
        u, v = pots[t][0][0], pots[t][1][0]
        vp = pots[t - 1][1][0] if t > 1 else torch.zeros_like(v)
        W = torch.exp(Z + u[:, None] + v[None] - log_nu[None]) * gv[None]
        dZ -= W
        gu = gu - W.sum(1)
        W = torch.exp(Z + u[:, None] - log_mu[:, None] + vp[None]) * gu[:, None]
        dZ -= W
        gv, gu = -W.sum(0), torch.zeros_like(gu)
    return dZ


def dustbin_sum(dZ):
    """[b, m+1, n+1] -> [b]: the dustbin row and column (the corner once), i.e. d alpha per problem."""
    return dZ[:, -1, :].sum(1) + dZ[:, :-1, -1].sum(1)


# (B, m, n, bin score, iters, spread, kind)
SK_CASES = [
    (1, 1, 1, 1.0, 100, 1.0, 'randn'),
    (1, 1, 1055, 1.0, 100, 12.0, 'randn'),
    (1, 31, 415, 2.0, 7, 12.0, 'randn'),
    (1, 32, 416, -3.0, 100, 40.0, 'randn'),
    (2, 64, 831, 1.0, 2, 300.0, 'randn'),
    (1, 100, 832, 5.0, 1, 12.0, 'low'),
    (1, 1000, 8, 5.0, 100, 40.0, 'randn'),
    (1, 8, 1000, 0.5, 7, 12.0, 'randn'),
    (1, 1055, 1, -1.0, 100, 12.0, 'randn'),
    (1, 1055, 1055, 1.0, 100, 12.0, 'randn'),
    (3, 200, 300, 4.0, 100, 1.0, 'randn'),
    (2, 50, 60, -3.0, 100, 300.0, 'randn'),
    (80, 400, 400, 1.0, 100, 40.0, 'randn'),
]


def sk_id(c):
    return 'B%d_%dx%d_bin%g_it%d_%s%g' % (c[0], c[1], c[2], c[3], c[4], c[6], c[5])


def sk_sampled(case):
    B = case[0]
    return sorted({0, B // 2, B - 1})


def pot_iters(iters):
    return sorted({1, max(1, iters // 2), iters})


@functools.lru_cache(maxsize=None)
def sk_inputs(case):
    B, m, n, _, _, spread, kind = case
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    s = spread * rng.standard_normal((B, m, n))
    if kind == 'low':             # scores well below the bin score: the dustbins take most of the mass
        s -= 6.0
    G = rng.standard_normal((B, m + 1, n + 1))
    return torch.from_numpy(s.astype(np.float32)), torch.from_numpy(G.astype(np.float32))


@functools.lru_cache(maxsize=None)
def sk_reference(case, b):
    """Problem b of a case in float64 and float32 (the yardstick's noise): couplings, potentials at pot_iters, dZ by
    autograd and, in float32, dZ by the kernel's recursion."""
    s, G = sk_inputs(case)
    alpha, iters = case[3], case[4]
    keep = pot_iters(iters)
    ref = {}
    for dt in (D, F):
        Z, pots, dZ = sk_grad(s[b:b + 1].to(dt), alpha, iters, G[b:b + 1], keep)
        ref[dt] = (Z[0], {t: (u[0], v[0]) for t, (u, v) in pots.items()}, dZ[0])
    ref['recursion32'] = sk_recursion(s[b], alpha, iters, G[b])
    return ref


def _sk_layouts(s):
    """(name, buffer, scores_ld, scores_stride) of the three layouts holding the scores s [B, m, n]."""
    B, m, n = s.shape
    aug = torch.full((B, m + 1, n + 1), float('nan'))
    aug[:, :m, :n] = s
    strided = torch.full((B, m + 2, n + 3), float('nan'))        # NaN in each row's padding and in two rows per problem
    strided[:, :m, :n] = s
    return [('packed', s.contiguous(), n, m * n), ('augmented', aug, n + 1, (m + 1) * (n + 1)),
            ('strided', strided, n + 3, (m + 2) * (n + 3))]


def sk_launch(buf, ld, stride, alpha, B, m, n, iters, G=None):
    """mvm_sinkhorn_train_forward (and _backward with G) on any layout -> Z, pot (, dZ, d_alpha)."""
    from e2e_multi_view_matching_b200 import _lib
    lib = _lib.lib()
    buf = buf.cuda()
    a = torch.tensor([alpha], dtype=F, device='cuda')
    Z = torch.empty(B, m + 1, n + 1, dtype=F, device='cuda')
    pot = torch.empty(lib.mvm_sinkhorn_train_pot_floats(B, m, n, iters), dtype=F, device='cuda')
    _check(lib.mvm_sinkhorn_train_forward(vp(buf), ld, stride, vp(a), B, m, n, iters, vp(Z), vp(pot), _stream()),
           'mvm_sinkhorn_train_forward')
    if G is None:
        torch.cuda.synchronize()
        return Z.cpu(), pot.cpu().view(B, iters, m + n + 2)
    dZ = G.cuda().contiguous().clone()
    da = torch.zeros(1, dtype=D, device='cuda')
    _check(lib.mvm_sinkhorn_train_backward(vp(buf), ld, stride, vp(a), vp(pot), B, m, n, iters, vp(dZ), vp(da),
                                           _stream()), 'mvm_sinkhorn_train_backward')
    torch.cuda.synchronize()
    return Z.cpu(), pot.cpu().view(B, iters, m + n + 2), dZ.cpu(), float(da)


def sk_run_ops(s, alpha, iters, G, augmented=False):
    """The package's entry points (packed scores, or the augmented buffers of pair_scores)."""
    from e2e_multi_view_matching_b200 import ops
    B, m, n = s.shape
    if augmented:
        buf = torch.full((B, m + 1, n + 1), float('nan'))
        buf[:, :m, :n] = s
    else:
        buf = s
    buf = buf.cuda()
    a = torch.tensor([alpha], dtype=F, device='cuda')
    Z, pot = ops.sinkhorn_train_forward(buf, a, iters, augmented=augmented)
    dZ, da = ops.sinkhorn_train_backward(buf, a, pot, iters, G.cuda(), augmented=augmented)
    torch.cuda.synchronize()
    return Z.cpu(), pot.cpu().view(B, iters, m + n + 2), dZ.cpu(), float(da)


@functools.lru_cache(maxsize=None)
def sk_gpu(case):
    """Packed run through ops -> (Z, pot, dZ, d_alpha), {run: (Z, pot and dZ bitwise equal to it, its d_alpha)} for the
    augmented buffers through ops, a repeat launch and the three layouts through the library."""
    s, G = sk_inputs(case)
    B, m, n, alpha, iters = case[:5]
    out = sk_run_ops(s, alpha, iters, G)
    runs = [('augmented (ops)', lambda: sk_run_ops(s, alpha, iters, G, augmented=True)),
            ('repeat', lambda: sk_run_ops(s, alpha, iters, G))]
    runs += [(name, functools.partial(sk_launch, buf, ld, stride, alpha, B, m, n, iters, G))
             for name, buf, ld, stride in _sk_layouts(s)]
    same = {}
    for name, run in runs:
        Z2, pot2, dZ2, da2 = run()
        same[name] = (torch.equal(Z2, out[0]), torch.equal(pot2, out[1]), torch.equal(dZ2, out[2]), da2)
    return out, same


def _pot_split(pot, m):
    return pot[:m + 1], pot[m + 1:]


@gpu
@pytest.mark.parametrize('case', SK_CASES, ids=sk_id)
def test_sinkhorn_train_forward_vs_float64(case):
    B, m, n, alpha, iters = case[:5]
    (Z, pot, _, _), same = sk_gpu(case)
    assert Z.shape == (B, m + 1, n + 1) and pot.shape == (B, iters, m + n + 2)
    for b in sk_sampled(case):
        ref = sk_reference(case, b)
        z64, p64, _ = ref[D]
        z32, p32, _ = ref[F]
        noise = float((z32.double() - z64).abs().max())
        tol = max(1e-4, 3.0 * noise)
        err = (Z[b].double() - z64).abs()
        ratio = float((err / (tol + 1e-5 * z64.abs())).max())
        print('%s b=%d couplings: max err %.2e, bound %.2e (fp32 noise %.2e), worst err / bound %.3f'
              % (sk_id(case), b, float(err.max()), tol, noise, ratio))
        assert torch.isfinite(Z[b]).all() and ratio <= 1.0, (b, ratio)
        for t in pot_iters(iters):
            u, v = _pot_split(pot[b, t - 1], m)
            for name, got, r64, r32 in (('u', u, p64[t][0], p32[t][0]), ('v', v, p64[t][1], p32[t][1])):
                noise_p = float((r32.double() - r64).abs().max())
                tol_p = max(1e-4, 3.0 * noise_p)
                err_p = (got.double() - r64).abs()
                ratio_p = float((err_p / (tol_p + 1e-5 * r64.abs())).max())
                print('  t=%d %s^t: max err %.2e, bound %.2e, err / bound %.3f' % (t, name, float(err_p.max()), tol_p, ratio_p))
                assert ratio_p <= 1.0, (b, t, name, ratio_p)
    for name, (z_eq, pot_eq, _, _) in same.items():
        assert z_eq and pot_eq, name


@gpu
@pytest.mark.parametrize('case', SK_CASES, ids=sk_id)
def test_sinkhorn_train_backward_vs_float64(case):
    B, m, n = case[:3]
    (_, _, dZ, da), same = sk_gpu(case)
    assert dZ.shape == (B, m + 1, n + 1) and torch.isfinite(dZ).all()
    da64 = noise_a = dust_abs = 0.0
    for b in sk_sampled(case):
        ref = sk_reference(case, b)
        g64, g32, r32 = ref[D][2], ref[F][2], ref['recursion32']
        noise_ag = float((g32.double() - g64).abs().max())
        noise_rec = float((r32.double() - g64).abs().max())
        tol = max(1e-5 * float(g64.abs().max()), 3.0 * noise_ag, 3.0 * noise_rec)
        err = float((dZ[b].double() - g64).abs().max())
        err_bins = max(float((dZ[b, -1].double() - g64[-1]).abs().max()), float((dZ[b, :, -1].double() - g64[:, -1]).abs().max()))
        print('%s b=%d dZ: max err %.2e (dustbins %.2e), bound %.2e (fp32 noise: autograd %.2e, recursion %.2e, '
              'max|dZ| %.3g), err / bound %.3f' % (sk_id(case), b, err, err_bins, tol, noise_ag, noise_rec,
                                                   float(g64.abs().max()), err / tol))
        assert err <= tol, (b, err, tol)
        a64 = float(dustbin_sum(g64[None]))
        da64 += a64
        noise_a += max(abs(float(dustbin_sum(g[None].double())) - a64) for g in (g32, r32))
        dust_abs += float(dustbin_sum(g64.abs()[None]))
    if len(sk_sampled(case)) == B:
        tol_a = max(1e-5 * dust_abs, 3.0 * noise_a)
        print('%s d_alpha: %.9g vs float64 %.9g, err %.2e, bound %.2e' % (sk_id(case), da, da64, abs(da - da64), tol_a))
        assert abs(da - da64) <= tol_a
    if B == 1:      # d_alpha is the (double) sum of the kernel's own dustbin entries
        own = float(dustbin_sum(dZ.double()))
        assert abs(da - own) <= 1e-12 * float(dustbin_sum(dZ.double().abs())), (da, own)
    for name, (_, _, dz_eq, da2) in same.items():
        assert dz_eq, name
        # one problem adds one double to zero: fixed bits; several add in no fixed order
        assert da2 == da if B == 1 else abs(da2 - da) <= 1e-12 * abs(da), (name, da2, da)


@gpu
def test_sinkhorn_train_batch_invariance():
    """Problem b alone gives the bits it gets inside the cfg5 launch of 80 problems; d_alpha (double atomics in no fixed
    order) is the sum of the 80 single-problem values."""
    case = SK_CASES[-1]
    B, m, n, alpha, iters = case[:5]
    s, G = sk_inputs(case)
    (Z, pot, dZ, da), _ = sk_gpu(case)
    total = 0.0
    for b in range(B):
        Zb, potb, dZb, dab = sk_run_ops(s[b:b + 1], alpha, iters, G[b:b + 1])
        assert torch.equal(Zb[0], Z[b]) and torch.equal(potb[0], pot[b]) and torch.equal(dZb[0], dZ[b]), b
        total += dab
    print('B=80 d_alpha %.15g, sum of singles %.15g, rel diff %.2e' % (da, total, abs(da - total) / abs(total)))
    assert abs(da - total) <= 1e-12 * abs(total)


@gpu
@pytest.mark.parametrize('m,n,iters,ld', [(0, 5, 3, 5), (5, 0, 3, 5), (1056, 5, 3, 5), (5, 1056, 3, 1056), (5, 5, 0, 5),
                                          (5, 6, 3, 5)])
def test_sinkhorn_train_refusals(m, n, iters, ld):
    from e2e_multi_view_matching_b200 import _lib
    lib = _lib.lib()
    big = 1060 * 1060
    buf = torch.zeros(big, device='cuda')
    a = torch.ones(1, device='cuda')
    Z, dZ, pot = torch.zeros(big, device='cuda'), torch.zeros(big, device='cuda'), torch.zeros(8 * big, device='cuda')
    da = torch.zeros(1, dtype=D, device='cuda')
    with pytest.raises(_lib.MvmError, match='invalid argument'):
        _check(lib.mvm_sinkhorn_train_forward(vp(buf), ld, max(m, 1) * ld, vp(a), 1, m, n, iters, vp(Z), vp(pot), _stream()),
               'mvm_sinkhorn_train_forward')
    with pytest.raises(_lib.MvmError, match='invalid argument'):
        _check(lib.mvm_sinkhorn_train_backward(vp(buf), ld, max(m, 1) * ld, vp(a), vp(pot), 1, m, n, iters, vp(dZ), vp(da),
                                               _stream()), 'mvm_sinkhorn_train_backward')
    torch.cuda.synchronize()


def test_sinkhorn_reference_checkpointed_equals_plain_autograd():
    g = torch.Generator().manual_seed(3)
    s = torch.randn(2, 30, 41, generator=g, dtype=D) * 12
    G = torch.randn(2, 31, 42, generator=g, dtype=D)
    Zc, pc, dc = sk_grad(s, 1.3, 20, G, keep=(1, 10, 20), checkpointed=True)
    Zp, pp, dp = sk_grad(s, 1.3, 20, G, keep=(1, 10, 20), checkpointed=False)
    assert torch.equal(Zc, Zp) and torch.equal(dc, dp)
    assert all(torch.equal(pc[t][0], pp[t][0]) and torch.equal(pc[t][1], pp[t][1]) for t in pc)


def test_sinkhorn_reference_matches_oracle():
    """sk_grad's couplings are oracle.train_ops._ot's, its inner block is the oracle's d scores and its dustbin entries
    sum to the oracle's d_alpha."""
    from oracle import train_ops
    g = torch.Generator().manual_seed(4)
    s = torch.randn(2, 17, 23, generator=g) * 5
    G = torch.randn(2, 18, 24, generator=g)
    alpha = torch.tensor([0.7])
    Z, _, dZ = sk_grad(s.double(), float(alpha), 15, G, checkpointed=True)
    Zo = train_ops._ot(s.double(), alpha.double().reshape(()), 15)
    dZo, dao = train_ops.sinkhorn_train_backward(s, alpha, None, 15, G)
    assert float((Z - Zo).abs().max()) <= 1e-12
    assert float((dZ[:, :-1, :-1].float() - dZo[:, :-1, :-1]).abs().max()) <= 1e-6 * float(dZo.abs().max())
    da = float(dustbin_sum(dZ).sum())
    assert abs(da - float(dao)) <= 1e-10 * max(1.0, abs(float(dao))), (da, float(dao))
    # the kernel's reverse recursion, restated in float64, is the same gradient (dustbins included)
    for b in range(2):
        r = sk_recursion(s[b].double(), float(alpha), 15, G[b])
        assert float((r - dZ[b]).abs().max()) <= 1e-10 * float(dZ[b].abs().max())


# ---------------------------------------------------------------------------------------------------------------------
# BatchNorm in training mode
# ---------------------------------------------------------------------------------------------------------------------

# (name, slots, n_pad, n_valid, groups, C, relu, momentum, eps, kind)
BN_CASES = [
    ('c1_300rows', 3, 100, 100, 1, 1, True, 0.1, 1e-5, 'randn'),
    ('c31_560rows', 4, 140, 131, 2, 31, False, 0.01, 1e-3, 'edge'),
    ('c33_g3', 6, 128, 100, 3, 33, True, 0.1, 1e-5, 'edge'),
    ('c96_nvalid1', 10, 64, 1, 5, 96, True, 0.1, 1e-5, 'randn'),
    ('c96_two_rows', 2, 50, 2, 2, 96, False, 0.1, 1e-3, 'edge'),
    ('c256_cfg5', 40, 448, 400, 1, 256, True, 0.1, 1e-5, 'edge'),
    ('c512_cfg5_g2', 40, 448, 400, 2, 512, True, 0.01, 1e-3, 'randn'),
    ('c1024_g3', 12, 100, 77, 3, 1024, False, 0.1, 1e-5, 'edge'),
    ('head_10x3200', 10, 3200, 3200, 10, 256, True, 0.1, 1e-5, 'edge'),
]


def bn_mask(rows, n_pad, n_valid, groups, g):
    r = torch.arange(rows)
    return (r % n_pad < n_valid) & ((r // n_pad) % groups == g)


def bn_inputs(case):
    name, slots, n_pad, n_valid, groups, Cc, relu, momentum, eps, kind = case
    rows = slots * n_pad
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = rng.standard_normal((rows, Cc)) * 3 + 1
    if kind == 'edge':
        c = np.arange(Cc)
        big = c % 4 == 1                                 # |mean| / std = 1e3, both signs
        x[:, big] = np.where(c[big] % 8 == 1, 1e3, -1e3) + rng.standard_normal((rows, int(big.sum())))
        x[:, c % 4 == 2] = 2.5                           # constant: var = 0
        out = c % 4 == 3                                 # an outlier in the shift row of every group
        for g in range(groups):
            x[g * n_pad, out] = 5e3
    x = torch.from_numpy(x.astype(np.float32))
    valid = torch.arange(rows) % n_pad < n_valid
    x[~valid] = float('nan')                             # padding rows: must not reach any output
    w = torch.from_numpy((rng.random(Cc) + 0.5).astype(np.float32))
    b = torch.from_numpy(rng.standard_normal(Cc).astype(np.float32))
    rm = torch.from_numpy(rng.standard_normal(Cc).astype(np.float32))
    rv = torch.from_numpy((rng.random(Cc) + 0.5).astype(np.float32))
    dy = torch.from_numpy(rng.standard_normal((rows, Cc)).astype(np.float32))
    dy[~valid] = float('nan')
    return x, w, b, rm, rv, dy, valid


def bn_backward(x, y, dy, w, stats, n_pad, n_valid, relu, dtype):
    """The backward formula of oracle.train_ops.batchnorm_train_backward in `dtype` on given saved statistics ->
    (dx on the valid rows [rows, C] (others 0), dgamma, dbeta, sum |g xhat|, sum |g|, and per element
    |gamma invstd| (|g| + |mean g| + |xhat mean(g xhat)|), the size of the terms whose rounding dx keeps)."""
    rows, Cc = x.shape
    groups = stats.shape[0]
    dx = torch.zeros(rows, Cc, dtype=dtype)
    terms = torch.zeros(rows, Cc, dtype=D)
    dg, db, ag, ab = (torch.zeros(Cc, dtype=dtype) for _ in range(4))
    for g in range(groups):
        m = bn_mask(rows, n_pad, n_valid, groups, g)
        mean, invstd = stats[g, :Cc].to(dtype), stats[g, Cc:].to(dtype)
        gq = dy[m].to(dtype)
        if relu:
            gq = gq * (y[m] > 0)
        xh = (x[m].to(dtype) - mean) * invstd
        sg, sgx = gq.sum(0), (gq * xh).sum(0)
        n = gq.shape[0]
        dx[m] = w.to(dtype) * invstd * (gq - sg / n - xh * sgx / n)
        terms[m] = ((w.to(dtype) * invstd).abs() * (gq.abs() + (sg / n).abs() + (xh * sgx / n).abs())).double()
        dg, db = dg + sgx, db + sg
        ag, ab = ag + (gq * xh).abs().sum(0), ab + gq.abs().sum(0)
    return dx, dg, db, ag, ab, terms


def bn_reference(case):
    """oracle.train_ops.batchnorm_train (float64 inside; y and the saved statistics rounded to float32, the running
    statistics kept in float64) and fp32 torch.nn.functional.batch_norm on the same rows (the yardstick's noise)
    -> y64, stats64, running mean / var 64, y32, running mean / var 32, per-group std in float64."""
    from oracle import train_ops
    name, slots, n_pad, n_valid, groups, Cc, relu, momentum, eps, kind = case
    x, w, b, rm, rv, _, _ = bn_inputs(case)
    rows = x.shape[0]
    rm64, rv64 = rm.double(), rv.double()
    y64, st64 = train_ops.batchnorm_train(x, w, b, rm64, rv64, momentum, eps, n_pad, n_valid, relu=relu, groups=groups,
                                          out=torch.zeros(rows, Cc), save=True)
    y32 = torch.zeros(rows, Cc)
    rm32, rv32 = rm.clone(), rv.clone()
    std64 = torch.zeros(groups, Cc, dtype=D)
    for g in range(groups):
        msk = bn_mask(rows, n_pad, n_valid, groups, g)
        o = torch.nn.functional.batch_norm(x[msk], rm32, rv32, w, b, training=True, momentum=momentum, eps=eps)
        y32[msk] = o.clamp_min(0) if relu else o
        std64[g] = x[msk].double().std(0, unbiased=False)
    return y64, st64, rm64, rv64, y32, rm32, rv32, std64


def _bn_ratio(err, tol):
    return float((err / tol).max())


@gpu
@pytest.mark.parametrize('case', BN_CASES, ids=lambda c: c[0])
def test_batchnorm_train_vs_float64(case):
    from e2e_multi_view_matching_b200 import ops
    name, slots, n_pad, n_valid, groups, Cc, relu, momentum, eps, kind = case
    x, w, b, rm, rv, dy, valid = bn_inputs(case)
    y64, st64, rm64, rv64, y32, rm32, rv32, std64 = bn_reference(case)
    # kernel: out of place into a sentinel buffer, and in place
    sentinel = -777.25
    xc = x.cuda()
    rmc, rvc = rm.cuda(), rv.cuda()
    yc, st = ops.batchnorm_train(xc, w.cuda(), b.cuda(), rmc, rvc, momentum, eps, n_pad, n_valid, relu=relu,
                                 groups=groups, out=torch.full_like(xc, sentinel), save=True)
    xi = x.cuda()
    yi, st_i = ops.batchnorm_train(xi, w.cuda(), b.cuda(), rm.cuda(), rv.cuda(), momentum, eps, n_pad, n_valid,
                                   relu=relu, groups=groups, save=True)
    torch.cuda.synchronize()
    y, st, yi, st_i = yc.cpu(), st.cpu(), yi.cpu(), st_i.cpu()
    assert torch.equal(xc.cpu()[valid], x[valid]) and torch.isnan(xc.cpu()[~valid]).all()     # x untouched
    assert (y[~valid] == sentinel).all() and torch.isnan(yi[~valid]).all()                    # padding untouched
    assert torch.equal(yi[valid], y[valid]) and torch.equal(st_i, st)                          # in place = out of place
    # y, per channel
    noise = (y32[valid].double() - y64[valid]).abs().amax(0)
    tol = torch.maximum(1e-5 * y64[valid].abs().amax(0).clamp_min(1.0), 3.0 * noise)
    err = (y[valid].double() - y64[valid]).abs().amax(0)
    print('%s y: max err %.2e, worst err / bound %.3f (channel %d, bound %.2e)'
          % (name, float(err.max()), _bn_ratio(err, tol), int((err / tol).argmax()), float(tol[(err / tol).argmax()])))
    assert torch.isfinite(y[valid]).all() and (err <= tol).all()
    # saved statistics
    mean, invstd = st[:, :Cc].double(), st[:, Cc:].double()
    mean64, invstd64 = st64[:, :Cc].double(), st64[:, Cc:].double()
    # (st64 holds the float64 statistics rounded to float32: half an ulp of them is part of every bound)
    tol_m = 2.0 ** -22 * mean64.abs() + 1e-6 * std64
    tol_i = 1e-6 * invstd64
    print('%s mean: worst err / bound %.3f; invstd: %.3f' % (name, _bn_ratio((mean - mean64).abs(), tol_m + 1e-30),
                                                             _bn_ratio((invstd - invstd64).abs(), tol_i)))
    assert ((mean - mean64).abs() <= tol_m).all() and ((invstd - invstd64).abs() <= tol_i).all()
    # running statistics (updated once per group, in group order)
    scale = std64.amax(0)
    for what, got, r64, r32, s in (('running_mean', rmc.cpu(), rm64, rm32, scale), ('running_var', rvc.cpu(), rv64, rv32, scale ** 2)):
        tol_r = torch.maximum(1e-6 * r64.abs() + 1e-6 * momentum * s, 3.0 * (r32.double() - r64).abs())
        e = (got.double() - r64).abs()
        print('%s %s: max err %.2e, worst err / bound %.3f' % (name, what, float(e.max()), _bn_ratio(e, tol_r + 1e-30)))
        assert (e <= tol_r).all(), what

    # backward on the kernel's y and saved statistics; dy's padding rows hold NaN and must stay as they are
    dyc = dy.cuda()
    dg, db = ops.batchnorm_train_backward(xc, yc, dyc, w.cuda(), st.cuda(), n_pad, n_valid, relu=relu)
    torch.cuda.synchronize()
    dx, dg, db = dyc.cpu(), dg.cpu(), db.cpu()
    assert torch.isnan(dx[~valid]).all()
    dx64, dg64, db64, ag, ab, terms = bn_backward(x, y, dy, w, st, n_pad, n_valid, relu, D)
    dx32 = bn_backward(x, y, dy, w, st, n_pad, n_valid, relu, F)[0]
    noise = (dx32[valid].double() - dx64[valid]).abs().amax(0)
    # (where dx cancels, as in a group of two rows, the rounding of its terms is the floor)
    tol = torch.maximum(1e-5 * dx64[valid].abs().amax(0), 3.0 * noise) + 4 * EPS32 * terms[valid] + 1e-30
    err = (dx[valid].double() - dx64[valid]).abs()
    print('%s dx: max err %.2e, worst err / bound %.3f' % (name, float(err.max()), _bn_ratio(err, tol)))
    assert torch.isfinite(dx[valid]).all() and (err <= tol).all()
    k = (groups + 2) * EPS32
    for what, got, r64, a in (('dgamma', dg, dg64, ag), ('dbeta', db, db64, ab)):
        e = (got.double() - r64).abs()
        t = k * a + 1e-30
        print('%s %s: max err %.2e, worst err / bound %.3f' % (name, what, float(e.max()), _bn_ratio(e, t)))
        assert torch.isfinite(got).all() and (e <= t).all(), what


def _bn_lib(x, y, rows, Cc, ld, n_pad, n_valid, slot_mod, slot_rem, w, b, rm, rv, stats, ws, eps=1e-5, relu=1, mom=0.1):
    from e2e_multi_view_matching_b200 import _lib
    return _lib.lib().mvm_batchnorm_train(vp(x), vp(y), rows, Cc, ld, n_pad, n_valid, slot_mod, slot_rem, vp(w), vp(b),
                                          eps, relu, vp(rm), vp(rv), mom, vp(stats), vp(ws), _stream())


def _bn_bwd_lib(x, y, dy, rows, Cc, ld, n_pad, n_valid, slot_mod, slot_rem, w, stats, dg, db, ws, relu=1, acc=0):
    from e2e_multi_view_matching_b200 import _lib
    return _lib.lib().mvm_batchnorm_train_backward(vp(x), vp(y), vp(dy), rows, Cc, ld, n_pad, n_valid, slot_mod, slot_rem,
                                                   vp(w), vp(stats), relu, vp(dg), vp(db), acc, vp(ws), _stream())


@gpu
def test_batchnorm_train_row_stride_and_other_groups():
    """ld > C through the library: the extra columns keep their contents, the results equal the contiguous call bit for
    bit, and the rows of the other groups (NaN here) are neither read nor written."""
    Cc, ld, n_pad, n_valid, slot_mod, slot_rem, slots = 70, 77, 96, 90, 3, 1, 9
    rows = slots * n_pad
    g = torch.Generator().manual_seed(21)
    x = torch.randn(rows, Cc, generator=g) * 2 - 0.5
    other = ((torch.arange(rows) // n_pad) % slot_mod != slot_rem) | (torch.arange(rows) % n_pad >= n_valid)
    x[other] = float('nan')
    w, b = torch.rand(Cc, generator=g) + 0.5, torch.randn(Cc, generator=g)
    dy = torch.randn(rows, Cc, generator=g)
    dy[other] = float('nan')
    dev = lambda t: t.cuda().contiguous()
    xs = torch.full((rows, ld), 31.5)
    xs[:, :Cc] = x
    xs = xs.cuda()
    ys = torch.full((rows, ld), -5.0, device='cuda')
    dys = torch.full((rows, ld), 9.0)
    dys[:, :Cc] = dy
    dys = dys.cuda()
    xc, yc, dyc = dev(x), torch.full((rows, Cc), -5.0, device='cuda'), dev(dy)
    out = {}
    for name, (X, Y, DY, L) in {'strided': (xs, ys, dys, ld), 'contiguous': (xc, yc, dyc, Cc)}.items():
        rm, rv = torch.zeros(Cc, device='cuda'), torch.ones(Cc, device='cuda')
        st = torch.empty(2 * Cc, device='cuda')
        ws = torch.empty(3 * Cc, dtype=D, device='cuda')
        _check(_bn_lib(X, Y, rows, Cc, L, n_pad, n_valid, slot_mod, slot_rem, dev(w), dev(b), rm, rv, st, ws), 'bn')
        dg, db = torch.full((Cc,), 2.0, device='cuda'), torch.full((Cc,), 3.0, device='cuda')
        _check(_bn_bwd_lib(X, Y, DY, rows, Cc, L, n_pad, n_valid, slot_mod, slot_rem, dev(w), st, dg, db, ws, acc=1), 'bn bwd')
        torch.cuda.synchronize()
        out[name] = [t.cpu() for t in (Y[:, :Cc], DY[:, :Cc], st, rm, rv, dg, db)]
    for a, c in zip(out['strided'], out['contiguous']):
        assert torch.equal(torch.nan_to_num(a, nan=1e30), torch.nan_to_num(c, nan=1e30))
    y, dx = out['contiguous'][:2]
    assert (y[other] == -5.0).all() and torch.isfinite(y[~other]).all()
    assert torch.isnan(dx[other]).all() and torch.isfinite(dx[~other]).all()
    assert all(torch.isfinite(t).all() for t in out['contiguous'][2:])
    assert (xs.cpu()[:, Cc:] == 31.5).all() and (ys.cpu()[:, Cc:] == -5.0).all() and (dys.cpu()[:, Cc:] == 9.0).all()
    # accumulate = 1 added this group's sums to 2 and 3
    msk = ~other
    st = out['contiguous'][2]
    gq = dy[msk].double() * (y[msk] > 0)
    xh = (x[msk].double() - st[:Cc].double()) * st[Cc:].double()
    assert ((out['contiguous'][5].double() - (2.0 + (gq * xh).sum(0))).abs() <= 4 * EPS32 * (2.0 + (gq * xh).abs().sum(0))).all()
    assert ((out['contiguous'][6].double() - (3.0 + gq.sum(0))).abs() <= 4 * EPS32 * (3.0 + gq.abs().sum(0))).all()


BN_BAD = [  # (rows, C, ld, n_pad, n_valid, slot_mod, slot_rem, running buffers given)
    ('C0', 64, 0, 8, 8, 8, 1, 0, 2),
    ('C1025', 64, 1025, 1025, 8, 8, 1, 0, 2),
    ('ld_lt_C', 64, 8, 7, 8, 8, 1, 0, 2),
    ('n_valid_gt_n_pad', 64, 8, 8, 8, 9, 1, 0, 2),
    ('n_valid0', 64, 8, 8, 8, 0, 1, 0, 2),
    ('rows_mod_n_pad', 60, 8, 8, 8, 8, 1, 0, 2),
    ('slots_mod_slot_mod', 64, 8, 8, 8, 8, 3, 0, 2),
    ('slot_rem_ge_slot_mod', 64, 8, 8, 8, 8, 2, 2, 2),
    ('slot_mod0', 64, 8, 8, 8, 8, 0, 0, 2),
    ('one_running_buffer', 64, 8, 8, 8, 8, 1, 0, 1),
]


@gpu
@pytest.mark.parametrize('bad', BN_BAD, ids=lambda c: c[0])
def test_batchnorm_train_refusals(bad):
    from e2e_multi_view_matching_b200 import _lib
    name, rows, Cc, ld, n_pad, n_valid, slot_mod, slot_rem, nrun = bad
    buf = lambda k: torch.zeros(k, device='cuda')
    x, y, dy = buf(rows * 1100), buf(rows * 1100), buf(rows * 1100)
    w, b, rm, rv, st = buf(1100), buf(1100), buf(1100), buf(1100), buf(2200)
    ws = torch.zeros(3300, dtype=D, device='cuda')
    with pytest.raises(_lib.MvmError, match='invalid argument'):
        _check(_bn_lib(x, y, rows, Cc, ld, n_pad, n_valid, slot_mod, slot_rem, w, b, rm, rv if nrun == 2 else None, st, ws),
               'mvm_batchnorm_train')
    if name != 'one_running_buffer':         # the backward takes no running buffers
        with pytest.raises(_lib.MvmError, match='invalid argument'):
            _check(_bn_bwd_lib(x, y, dy, rows, Cc, ld, n_pad, n_valid, slot_mod, slot_rem, w, st, buf(1100), buf(1100), ws),
                   'mvm_batchnorm_train_backward')
    torch.cuda.synchronize()


def test_batchnorm_backward_reference_matches_oracle():
    from oracle import train_ops
    g = torch.Generator().manual_seed(8)
    rows, Cc, n_pad, n_valid, groups = 6 * 20, 7, 20, 17, 3
    x, dy = torch.randn(rows, Cc, generator=g), torch.randn(rows, Cc, generator=g)
    w, b = torch.rand(Cc, generator=g) + 0.5, torch.randn(Cc, generator=g)
    y, st = train_ops.batchnorm_train(x, w, b, None, None, 0.1, 1e-5, n_pad, n_valid, groups=groups,
                                      out=torch.zeros_like(x), save=True)
    dxo = dy.clone()
    dgo, dbo = train_ops.batchnorm_train_backward(x, y, dxo, w, st, n_pad, n_valid)
    dx, dg, db = bn_backward(x, y, dy, w, st, n_pad, n_valid, True, D)[:3]
    valid = torch.arange(rows) % n_pad < n_valid
    assert torch.equal(dx[valid].float(), dxo[valid]) and torch.equal(dg.float(), dgo) and torch.equal(db.float(), dbo)


# ---------------------------------------------------------------------------------------------------------------------
# mvm_colsum and mvm_transpose_split
# ---------------------------------------------------------------------------------------------------------------------

def _ulp32(a):
    """ulp of float32 values (as float64), a float64 array."""
    a = np.abs(np.asarray(a, dtype=np.float32))
    return (np.nextafter(a, np.float32(np.inf)) - a).astype(np.float64)


def _colsum_lib(x, rows, Cc, ld, out, accumulate):
    from e2e_multi_view_matching_b200 import _lib
    ws = torch.empty(Cc, dtype=D, device='cuda')
    _check(_lib.lib().mvm_colsum(vp(x), rows, Cc, ld, vp(out), accumulate, vp(ws), _stream()), 'mvm_colsum')
    torch.cuda.synchronize()
    return out.cpu()


def _colsum_bound(x64, expect):
    rows = x64.shape[0]
    return _ulp32(expect) + rows * np.abs(x64).max() * 2.0 ** -52


@gpu
@pytest.mark.parametrize('rows', [1, 295, 296, 297, 17920])
@pytest.mark.parametrize('Cc', [1, 255, 256, 257, 768])
def test_colsum_vs_float64(Cc, rows):
    from e2e_multi_view_matching_b200 import ops
    rng = np.random.default_rng(rows * 1000 + Cc)
    x = rng.standard_normal((rows, Cc)).astype(np.float32) * np.float32(3.0)
    got = ops.colsum(torch.from_numpy(x).cuda()).cpu().numpy().astype(np.float64)
    s64 = x.astype(np.float64).sum(0)
    expect = s64.astype(np.float32).astype(np.float64)
    err, tol = np.abs(got - expect), _colsum_bound(x.astype(np.float64), expect)
    print('colsum %dx%d: max err %.2e, worst err / bound %.3f' % (rows, Cc, err.max(), (err / tol).max()))
    assert (err <= tol).all()


@gpu
@pytest.mark.parametrize('rows,Cc,ld', [(297, 257, 300), (17920, 768, 777), (1, 1, 5)])
def test_colsum_stride_accumulate_cancellation(rows, Cc, ld):
    """ld > C (the other columns hold NaN), accumulate = 1, and columns of +-1e4 pairs plus small values."""
    rng = np.random.default_rng(rows + Cc)
    x = rng.standard_normal((rows, Cc)) * 1e-3
    big = rng.choice([-1e4, 1e4], size=((rows + 1) // 2, Cc))
    x[0::2] += big
    x[1::2] -= big[:rows // 2]                   # +-1e4 cancels in pairs (the last row of an odd count does not)
    x = x.astype(np.float32)
    buf = np.full((rows, ld), np.nan, dtype=np.float32)
    buf[:, :Cc] = x
    prev = rng.standard_normal(Cc).astype(np.float32)
    out = torch.from_numpy(prev.copy()).cuda()
    got = _colsum_lib(torch.from_numpy(buf).cuda(), rows, Cc, ld, out, 1).numpy().astype(np.float64)
    s = x.astype(np.float64).sum(0).astype(np.float32)
    expect = (prev + s).astype(np.float64)       # the kernel adds the rounded sum to out in float32
    tol = _colsum_bound(x.astype(np.float64), s) + _ulp32(expect)
    err = np.abs(got - expect)
    print('colsum accumulate %dx%d ld %d: max err %.2e, worst err / bound %.3f' % (rows, Cc, ld, err.max(), (err / tol).max()))
    assert np.isfinite(got).all() and (err <= tol).all()
    out0 = torch.full((Cc,), float('nan'), device='cuda')
    got0 = _colsum_lib(torch.from_numpy(buf).cuda(), rows, Cc, ld, out0, 0).numpy().astype(np.float64)
    err0 = np.abs(got0 - s.astype(np.float64))
    assert (err0 <= _colsum_bound(x.astype(np.float64), s)).all()


def tf32_rna(a):
    """cvt.rna.tf32.f32 restated on float32 bits: round the magnitude to nearest on the 13 dropped mantissa bits, ties
    away from zero, keep the sign."""
    bits = np.asarray(a, dtype=np.float32).view(np.uint32)
    mag = bits & np.uint32(0x7fffffff)
    r = ((mag + np.uint32(0x1000)) & np.uint32(0xffffe000)) | (bits & np.uint32(0x80000000))
    return r.view(np.float32)


def tf32_bits(n, rng):
    """float32 values of mixed exponents, with the dropped-bit patterns where rounding goes wrong."""
    sign = rng.integers(0, 2, n, dtype=np.uint32) << np.uint32(31)
    expo = rng.integers(60, 190, n, dtype=np.uint32) << np.uint32(23)
    mant = rng.integers(0, 1 << 23, n, dtype=np.uint32)
    kind = rng.integers(0, 8, n)
    low = np.array([0x1000, 0x0fff, 0x1fff, 0x0000, 0x1001], dtype=np.uint32)[rng.integers(0, 5, n)]
    mant = np.where(kind == 1, (mant & np.uint32(0x7fe000)) | low, mant)           # ties, just below, just above
    mant = np.where(kind == 2, np.uint32(0x7fffff), mant)                           # carries into the exponent
    expo = np.where(kind == 3, np.uint32(0), expo)                                  # subnormals
    mant = np.where(kind == 4, np.uint32(0), mant)
    expo = np.where(kind == 4, np.uint32(0), expo)                                  # +-0
    return (sign | expo | mant).view(np.float32)


@gpu
@pytest.mark.parametrize('mode', ['raw', 'planes', 'both'])
@pytest.mark.parametrize('R,Cc', [(1, 1), (1, 1000), (1000, 1), (31, 33), (32, 32), (33, 31), (100, 1000), (1000, 100),
                                  (33, 100)])
def test_transpose_split_bitwise(R, Cc, mode):
    from e2e_multi_view_matching_b200 import _lib
    lib = _lib.lib()
    rng = np.random.default_rng(R * 7 + Cc)
    x = tf32_bits(R * Cc, rng).reshape(R, Cc)
    ld, pad = Cc + 3, 5
    buf = np.full((R, ld), np.nan, dtype=np.float32)
    buf[:, :Cc] = x
    xd = torch.from_numpy(buf).cuda()
    sent = np.float32(-1234.5)
    hi_ref = tf32_rna(x.T)
    lo_ref = tf32_rna(x.T - hi_ref)                              # (x - hi is exact in float32)
    want_raw, want_planes = mode in ('raw', 'both'), mode in ('planes', 'both')
    # one [C, 2R + pad] plane: the transposed block written twice, into columns [0, R) and [R, 2R), with ldo > R
    ldo = 2 * R + pad
    planes = [torch.full((Cc, ldo), float(sent), device='cuda') if w else None
              for w in (want_raw, want_planes, want_planes)]
    for off in (0, R):
        r, h, l = [p.view(-1)[off:] if p is not None else None for p in planes]
        _check(lib.mvm_transpose_split(vp(xd), R, Cc, ld, vp(r), vp(h), vp(l), ldo, _stream()), 'mvm_transpose_split')
    torch.cuda.synchronize()
    for p, want in zip(planes, (x.T, hi_ref, lo_ref)):
        if p is None:
            continue
        got = p.cpu().numpy()
        for off in (0, R):
            assert np.array_equal(got[:, off:off + R].view(np.uint32), np.ascontiguousarray(want).view(np.uint32))
        assert (got[:, 2 * R:] == sent).all()
    # the concat-by-rows staging of ops.gemm_dw: x^T into rows [0, C) of a [C + 7, R] plane, ldo = R
    if want_planes:
        from e2e_multi_view_matching_b200 import ops
        hi = torch.full((Cc + 7, R), float(sent), device='cuda')
        lo = torch.full((Cc + 7, R), float(sent), device='cuda')
        ops.transpose_split(xd[:, :Cc].contiguous(), out=(None, hi[:Cc], lo[:Cc]))
        torch.cuda.synchronize()
        assert np.array_equal(hi.cpu().numpy()[:Cc].view(np.uint32), hi_ref.view(np.uint32))
        assert np.array_equal(lo.cpu().numpy()[:Cc].view(np.uint32), lo_ref.view(np.uint32))
        assert (hi.cpu().numpy()[Cc:] == sent).all() and (lo.cpu().numpy()[Cc:] == sent).all()
    print('transpose_split %dx%d %s: bitwise equal' % (R, Cc, mode))


def test_tf32_rna_restatement():
    cases = {                    # input bits -> cvt.rna.tf32.f32 bits
        0x3f800000: 0x3f800000,  # 1.0: nothing dropped
        0x3f801000: 0x3f802000,  # a tie rounds away from zero
        0x3f803000: 0x3f804000,  # a tie above an odd kept bit
        0x3f800fff: 0x3f800000,  # just below the tie
        0x3f801001: 0x3f802000,  # just above
        0x3fffffff: 0x40000000,  # all-ones mantissa carries into the exponent
        0xbf801000: 0xbf802000,  # negative tie: away from zero
        0xbf800fff: 0xbf800000,
        0x00001000: 0x00002000,  # subnormal tie
        0x00000fff: 0x00000000,  # subnormal rounds to +0
        0x807fffff: 0x80800000,  # negative subnormal carries into the smallest normal
        0x00000000: 0x00000000,
        0x80000000: 0x80000000,  # -0 keeps its sign
    }
    src = np.array(list(cases), dtype=np.uint32).view(np.float32)
    got = tf32_rna(src).view(np.uint32)
    assert [hex(v) for v in got] == [hex(v) for v in cases.values()]
    # and the package's own restatement (ops.rn_tf32) agrees on random patterns
    from e2e_multi_view_matching_b200 import ops
    x = tf32_bits(4096, np.random.default_rng(1))
    assert np.array_equal(ops.rn_tf32(torch.from_numpy(x)).numpy().view(np.uint32), tf32_rna(x).view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------
# Match loss
# ---------------------------------------------------------------------------------------------------------------------

def _ml_forward(log_p, idx, w, part, bs, ft):
    from e2e_multi_view_matching_b200 import _lib
    loss = torch.empty(1, device='cuda')
    _check(_lib.lib().mvm_match_loss_forward(vp(log_p), vp(idx), vp(w), bs, ft, vp(part), vp(loss), _stream()),
           'mvm_match_loss_forward')
    torch.cuda.synchronize()
    return float(loss)


@gpu
def test_match_loss_edges():
    """Dustbin rows and columns, mutual matches, the dustbin corner's two contributions, zero weights, a garbage-filled
    gradient buffer and one partial workspace for calls of different batch sizes."""
    from e2e_multi_view_matching_b200 import _lib
    from tests.test_training_gpu import _ref_match_loss
    bs, ft = 4, 301
    g = torch.Generator().manual_seed(17)
    log_p = -torch.rand(bs, ft, ft, generator=g) * 8
    idx = torch.randint(-1, ft - 1, (bs, 2, ft), generator=g)
    w = torch.rand(bs, 2, ft, generator=g)
    idx[0] = -1                                        # problem 0: every row and column to the dustbin (as -1) ...
    idx[0, 0, ::2] = ft - 1                            # ... or as its index; the corner (ft-1, ft-1) gets two terms
    perm = torch.randperm(ft - 1, generator=g)         # problem 1: mutual matches, both terms on one element
    idx[1, 0, :ft - 1] = perm
    idx[1, 1, perm] = torch.arange(ft - 1)
    idx[1, :, ft - 1] = -1
    w[2, :, ::3] = 0.0                                  # problem 2: zero weights
    w[3] = 0.0                                          # problem 3: all weights zero
    ref_in = log_p.double().requires_grad_(True)
    ref = _ref_match_loss(ref_in, idx, w.double())
    ref.backward()
    lp, ix, wc = log_p.cuda(), idx.cuda(), w.cuda()
    part = torch.full((bs + 3,), float('nan'), dtype=D, device='cuda')
    loss = _ml_forward(lp, ix, wc, part, bs, ft)
    print('match loss edges: %.9g vs float64 %.9g' % (loss, float(ref)))
    assert abs(loss - float(ref)) < 1e-5 * max(1.0, abs(float(ref)))
    # the same workspace for one problem and again for all: the stale partials are not read
    ref1 = _ref_match_loss(log_p[1:2].double(), idx[1:2], w[1:2].double())
    assert abs(_ml_forward(lp[1:2].contiguous(), ix[1:2].contiguous(), wc[1:2].contiguous(), part, 1, ft) - float(ref1)) \
        < 1e-5 * max(1.0, abs(float(ref1)))
    assert _ml_forward(lp, ix, wc, part, bs, ft) == loss
    grad = torch.tensor([2.5], device='cuda')
    out = torch.full((bs, ft, ft), float('nan'), device='cuda')
    out.view(-1)[::7] = 3.0e38
    _check(_lib.lib().mvm_match_loss_backward(vp(ix), vp(wc), vp(grad), bs, ft, vp(out), _stream()), 'mvm_match_loss_backward')
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    want = 2.5 * ref_in.grad.numpy()
    assert want[0, ft - 1, ft - 1] != 0 and (want[3] == 0).all()
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-9)
