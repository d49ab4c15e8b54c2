"""GPU: tensor-core (wgmma) kernels against fp64 math and the fp32 CUDA-core kernels."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('shape', [(128, 128, 32, 0), (256, 256, 128, 0), (1024, 768, 256, 0), (320, 512, 256, 256),
                                   (5120, 256, 512, 0), (192, 256, 256, 0)])
@pytest.mark.parametrize('passes', [3, 1])
def test_gemm_tc_vs_fp64(shape, passes):
    from e2e_multi_view_matching_b200 import ops
    M, N, K1, K2 = shape
    g = torch.Generator().manual_seed(M + N + K1)
    a = torch.randn(M, K1, generator=g).cuda()
    a2 = torch.randn(M, K2, generator=g).cuda() if K2 else None
    w = (torch.randn(N, K1 + K2, generator=g) / 16).cuda()
    b = torch.randn(N, generator=g).cuda()
    r = torch.randn(M, N, generator=g).cuda()
    out = ops.linear(a, w, bias=b, a2=a2, residual=r, relu=True, tc_passes=passes)
    torch.cuda.synchronize()
    A = torch.cat([a, a2], 1) if a2 is not None else a
    ref = torch.relu(A.double() @ w.double().T + b.double()) + r.double()
    err = (out.double() - ref).abs().max().item()
    tol = 1e-4 if passes == 3 else 2e-2
    assert err < tol, (shape, passes, err)
    if passes == 3:
        simt = ops.linear(a, w, bias=b, a2=a2, residual=r, relu=True)
        assert (simt - out).abs().max().item() < 1e-4


@pytest.mark.parametrize('name', ['pair_small_ragged', 'pair_18l_128_sharp', 'mv5_28l_96_sharp', 'mv4_ragged_sharp'])
@pytest.mark.parametrize('mode', [3, 1])
def test_matcher_tensor_core_modes(name, mode):
    """Whole matcher with the GEMMs (and attention) on the tensor cores: 3xTF32 keeps the fp32
    parity contract; single-pass TF32 (torch 1.10's Ampere default) is compared at TF32 accuracy."""
    import e2e_multi_view_matching_b200 as pkg
    from tests.util import load_case, case_inputs, compare_matcher_outputs, score_tol_for
    from tests.test_matcher_gpu import run_ours
    meta, ref = load_case(name)
    sd, data = case_inputs(meta)
    pkg.set_math_mode(mode)
    got = run_ours(meta, sd, data)
    if mode == 3:
        # 'sharp' cases scale the raw scores by gain^2 = 256: the ~1e-5 relative 3xTF32 error of the raw
        # score shows up as an absolute error of the (O(1)) log-coupling entries
        rep = compare_matcher_outputs(ref, got, tau=2e-3, score_tol=score_tol_for(name))
    else:
        rep = compare_matcher_outputs(ref, got, tau=0.3, score_tol=(0.3, 3e-2), conf_tol=5e-2)   # single-pass TF32: ~1e-3 relative per GEMM
    print(name, mode, rep)


@pytest.mark.parametrize('passes', [3, 1])
@pytest.mark.parametrize('cfg', [(1, 2, 128, [128, 128]), (2, 3, 192, [100, 192, 77]), (1, 5, 256, [256] * 5)])
def test_attention_tc_vs_simt(cfg, passes):
    from e2e_multi_view_matching_b200 import ops
    B, T, n_pad, counts = cfg
    g = torch.Generator().manual_seed(n_pad + T)
    qkv = torch.randn(B * T, n_pad, 768, generator=g).cuda()
    for is_cross in (0, 1):
        ref = ops.attention(qkv, B, T, counts, is_cross)
        got = ops.attention(qkv, B, T, counts, is_cross, tc_passes=passes)
        torch.cuda.synchronize()
        tol = 2e-5 if passes == 3 else 5e-3
        for v in range(B * T):
            n = counts[v % T]
            err = (ref[v, :n] - got[v, :n]).abs().max().item()
            assert err < tol, (cfg, passes, is_cross, v, err)


def test_gemm_kernel_variants_bit_identical():
    """The persistent kernel (A operand split into tensor memory, 128-column tiles, TMA-store epilogue) and the
    one-tile-per-CTA kernel with 128- or 256-column tiles accumulate over K in the same order with the same three
    passes, so the whole matcher must produce bit-identical outputs with any of them (operand split 0 = tf32 hi/lo
    in all three; the persistent kernel's default fp16 hi/lo planes are a different rounding, covered by
    tests/test_h3_gpu.py::test_matcher_gemm_split_ab)."""
    import e2e_multi_view_matching_b200 as pkg
    from e2e_multi_view_matching_b200 import _lib
    from tests.test_matcher_gpu import run_ours
    from tests.util import load_case, case_inputs
    meta, ref = load_case('mv4_ragged_sharp')
    sd, data = case_inputs(meta)
    lib = _lib.lib()
    outs = []
    try:
        lib.mvm_debug_set_score_kernel(0)       # same (fp32 CUDA-core) score GEMM for every variant
        lib.mvm_debug_set_gemm_split(0)
        for persist, tile in ((1, 256), (0, 128), (0, 256)):
            lib.mvm_debug_set_gemm_kernel(persist)
            lib.mvm_debug_set_gemm_tile(tile)
            pkg.set_math_mode(3)
            outs.append(run_ours(meta, sd, data))
    finally:
        lib.mvm_debug_set_gemm_kernel(1)
        lib.mvm_debug_set_gemm_tile(256)
        lib.mvm_debug_set_score_kernel(1)
        lib.mvm_debug_set_gemm_split(1)
    for other in outs[1:]:
        for k in outs[0]:
            assert np.array_equal(outs[0][k], other[k]), k


@pytest.mark.parametrize('shape', [(128, 128, 32, 0), (256, 256, 256, 0), (1024, 768, 256, 0), (320, 512, 256, 256),
                                   (5120, 256, 512, 0), (192, 256, 256, 0), (40960, 256, 256, 0)])
def test_gemm_persistent_presplit(shape):
    """mvm_linear_tc_presplit (the production 3xTF32 path) against fp64 and, bit for bit, against the
    one-tile-per-CTA kernel; ragged M (192, 320: not multiples of the 128-row tile), K-split concat, residual."""
    from e2e_multi_view_matching_b200 import ops, _lib
    M, N, K1, K2 = shape
    g = torch.Generator().manual_seed(M + N + K1 + 1)
    a = torch.randn(M, K1, generator=g).cuda()
    a2 = torch.randn(M, K2, generator=g).cuda() if K2 else None
    w = (torch.randn(N, K1 + K2, generator=g) / 16).cuda()
    b = torch.randn(N, generator=g).cuda()
    r = torch.randn(M, N, generator=g).cuda()
    lib = _lib.lib()
    try:
        lib.mvm_debug_set_gemm_kernel(1)
        out = ops.linear(a, w, bias=b, a2=a2, residual=r, relu=True, tc_passes=3, presplit=True)
        plain = ops.linear(a, w, tc_passes=3, presplit=True)            # no bias / residual / activation
        lib.mvm_debug_set_gemm_kernel(0)
        old = ops.linear(a, w, bias=b, a2=a2, residual=r, relu=True, tc_passes=3, presplit=True)
    finally:
        lib.mvm_debug_set_gemm_kernel(1)
    torch.cuda.synchronize()
    A = torch.cat([a, a2], 1) if a2 is not None else a
    ref = torch.relu(A.double() @ w.double().T + b.double()) + r.double()
    assert (out.double() - ref).abs().max().item() < 1e-4
    assert torch.equal(out, old)
    if a2 is None:
        assert (plain.double() - a.double() @ w.double().T).abs().max().item() < 1e-4


def test_score_gemm_tensor_cores_vs_cuda_cores():
    """Score matrices of every pair from the persistent 3xTF32 kernel (SCORE mode, ragged views) against the fp32
    CUDA-core kernel: the raw scores feed Sinkhorn, so compare the coupling matrices and the matches."""
    import e2e_multi_view_matching_b200 as pkg
    from e2e_multi_view_matching_b200 import _lib
    from tests.test_matcher_gpu import run_ours
    from tests.util import load_case, case_inputs, compare_matcher_outputs, score_tol_for
    lib = _lib.lib()
    for name in ('mv4_ragged_sharp', 'pair_small_ragged', 'mv5_28l_96'):
        meta, ref = load_case(name)
        sd, data = case_inputs(meta)
        pkg.set_math_mode(3)
        try:
            lib.mvm_debug_set_score_kernel(0)
            simt = run_ours(meta, sd, data)
            lib.mvm_debug_set_score_kernel(1)
            tcs = run_ours(meta, sd, data)
        finally:
            lib.mvm_debug_set_score_kernel(1)
        rep = compare_matcher_outputs(simt, tcs, tau=2e-3, score_tol=score_tol_for(name))
        print(name, rep)
