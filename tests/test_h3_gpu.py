"""fp16x3 attention (attention_h3.cu): hi = fp16(x), lo = fp16(x - hi) operand planes, three f16 MMAs per product.
Stage parity against the fp32 CUDA-core attention, and the whole matcher with this variant against the reference
goldens at the same tolerances as the tf32x3 default."""
import json
import os

import numpy as np
import pytest
import torch

from tests.util import GOLDEN, MATCHER_CASES, load_case, case_inputs, compare_matcher_outputs, score_tol_for

pytestmark = pytest.mark.gpu


@pytest.fixture(params=[1, 0], ids=['two_ctas_per_sm', 'two_groups_one_cta'])
def h3_variant(request):
    """Both fp16-plane kernels of attention_h3.cu: one softmax group with two CTAs per SM (default), and the
    two-group one-CTA-per-SM kernel kept for A/B."""
    from e2e_multi_view_matching_b200 import _lib
    lib = _lib.lib()
    lib.mvm_debug_set_attention_h3_variant(request.param)
    yield request.param
    lib.mvm_debug_set_attention_h3_variant(1)


@pytest.mark.parametrize('cfg', [(1, 2, 128, [128, 128]), (2, 3, 192, [100, 192, 77]), (1, 5, 256, [256] * 5),
                                 (3, 4, 1024, [1024, 1000, 1024, 65])])
@pytest.mark.parametrize('scale', [1.0, 6.0])
def test_attention_h3_vs_fp32(cfg, scale, h3_variant):
    from e2e_multi_view_matching_b200 import ops
    B, T, n_pad, counts = cfg
    g = torch.Generator().manual_seed(n_pad + T)
    qkv = (torch.randn(B * T, n_pad, 768, generator=g) * scale).cuda()
    for is_cross in (0, 1):
        ref = ops.attention(qkv, B, T, counts, is_cross)                     # fp32 CUDA cores
        out = ops.attention(qkv, B, T, counts, is_cross, tc_passes='h3')
        tc3 = ops.attention(qkv, B, T, counts, is_cross, tc_passes=3)        # tf32x3
        for b in range(B):
            for t in range(T):
                v = b * T + t
                e_h = (out[v, :counts[t]] - ref[v, :counts[t]]).abs().max().item()
                e_t = (tc3[v, :counts[t]] - ref[v, :counts[t]]).abs().max().item()
                assert e_h < max(3e-5 * scale, 2.0 * e_t + 1e-6), (cfg, scale, is_cross, e_h, e_t)


@pytest.mark.parametrize('name', MATCHER_CASES)
def test_matcher_h3_vs_reference_golden(name, h3_variant):
    import e2e_multi_view_matching_b200 as pkg
    from e2e_multi_view_matching_b200 import _lib
    from tests.test_matcher_gpu import run_ours
    lib = _lib.lib()
    meta, ref = load_case(name)
    sd, data = case_inputs(meta)
    pkg.set_math_mode(3)
    try:
        lib.mvm_debug_set_attention_split(1)
        got = run_ours(meta, sd, data)
        lib.mvm_debug_set_attention_split(0)
        base = run_ours(meta, sd, data)
    finally:
        lib.mvm_debug_set_attention_split(1)
    rep = compare_matcher_outputs(ref, got, tau=2e-3, score_tol=score_tol_for(name), min_stable=0.0 if name == 'pair_flat' else 0.9)
    rep0 = compare_matcher_outputs(ref, base, tau=2e-3, score_tol=score_tol_for(name))
    print(name, 'fp16x3', rep, 'tf32x3 max_score_err', rep0['max_score_err'])


@pytest.mark.parametrize('shape', [(300, 256, 128, 0), (1024, 768, 256, 0), (130, 512, 256, 256), (4096, 256, 512, 0)])
def test_linear_h16_vs_fp64(shape):
    """fp16x3 GEMM (persistent kernel, half-precision W planes pre-scaled by 64, A split on chip) against fp64, and
    against the tf32x3 kernel on the same operands."""
    from e2e_multi_view_matching_b200 import ops
    M, N, K1, K2 = shape
    g = torch.Generator().manual_seed(M + N)
    a = (torch.randn(M, K1, generator=g) * 3).cuda()
    a2 = (torch.randn(M, K2, generator=g) * 3).cuda() if K2 else None
    w = (torch.randn(N, K1 + K2, generator=g) / 16).cuda()
    b = torch.randn(N, generator=g).cuda()
    r = torch.randn(M, N, generator=g).cuda()
    A = torch.cat([a, a2], 1) if a2 is not None else a
    ref = torch.relu(A.double() @ w.double().T + b.double()) + r.double()
    out = ops.linear(a, w, bias=b, a2=a2, residual=r, relu=True, tc_passes='h16')
    t32 = ops.linear(a, w, bias=b, a2=a2, residual=r, relu=True, tc_passes=3, presplit=True)
    e_h, e_t = (out.double() - ref).abs().max().item(), (t32.double() - ref).abs().max().item()
    assert e_h < max(1e-4, 2.0 * e_t), (shape, e_h, e_t)


@pytest.mark.parametrize('name', ['pair_18l_128', 'mv5_28l_96_sharp', 'mv4_ragged_sharp'])
def test_matcher_gemm_split_ab(name):
    """Whole matcher with the GEMMs in fp16x3 (default) and in tf32x3: both within the golden tolerance, and close to
    each other."""
    import e2e_multi_view_matching_b200 as pkg
    from e2e_multi_view_matching_b200 import _lib
    from tests.test_matcher_gpu import run_ours
    lib = _lib.lib()
    meta, ref = load_case(name)
    sd, data = case_inputs(meta)
    pkg.set_math_mode(3)
    try:
        lib.mvm_debug_set_gemm_split(1)
        got = run_ours(meta, sd, data)
        lib.mvm_debug_set_gemm_split(0)
        base = run_ours(meta, sd, data)
    finally:
        lib.mvm_debug_set_gemm_split(1)
    rep = compare_matcher_outputs(ref, got, tau=2e-3, score_tol=score_tol_for(name), min_stable=0.9)
    rep0 = compare_matcher_outputs(ref, base, tau=2e-3, score_tol=score_tol_for(name), min_stable=0.9)
    print(name, 'gemm fp16x3', rep['max_score_err'], 'gemm tf32x3', rep0['max_score_err'])
