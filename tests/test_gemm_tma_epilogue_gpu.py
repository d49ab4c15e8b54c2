"""What the staged epilogue of the persistent tensor-core GEMM (csrc/gemm_tc.cu) adds: output tiles leave through
shared memory by TMA stores, which write whole boxes clipped only at the tensor map's bounds.

- C as a column slice of a wider buffer pre-filled with a sentinel, with M off the tile edge and more rows allocated
  than M: rows >= M and the columns N .. ldc keep the sentinel's bits, for fp16x3 and tf32x3, with and without a residual.
- C and R at an 8-byte offset (accepted by gemm_desc_valid, but not a TMA base, so those launches keep the direct
  stores) give the bits of the 16-byte aligned launch, with a separate and with an aliased residual.
"""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

KERNELS = ('fp16x3', 'tf32x3')
SENTINEL = -7.25e3


def vp(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def operands(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g).cuda()
    W = (torch.randn(N, K, generator=g) / 16).cuda()
    b = torch.randn(N, generator=g).cuda()
    r = torch.randn(M, N, generator=g).cuda()
    return A, W, b, r


def launch(k, A, W, b, R, out, relu=True):
    """One persistent launch of kernel k writing out [M, N] (any row stride), residual R (None, a tensor, or out)."""
    from e2e_multi_view_matching_b200 import _lib, ops
    lib = _lib.lib()
    M, K = A.shape
    N = W.shape[0]
    common = (vp(A), A.stride(0), C.c_void_p(0), 0, K)
    tail = (vp(b), vp(R), R.stride(0) if R is not None else 0, vp(out), out.stride(0), M, N, K, 1.0, int(relu))
    s = _lib.stream_ptr()
    if k == 'fp16x3':
        hi, lo = ops.h16_planes(W)
        rc = lib.mvm_linear_tc_h16(*common, vp(hi), vp(lo), ops.H16_SCALE, hi.stride(0), *tail, s)
    else:
        hi = ops.rn_tf32(W)
        lo = ops.rn_tf32(W - hi)
        rc = lib.mvm_linear_tc_presplit(*common, vp(hi), vp(lo), hi.stride(0), *tail, s)
    _lib.check(rc, k)
    torch.cuda.synchronize()


@pytest.mark.parametrize('res', [None, 'sep', 'alias'])
@pytest.mark.parametrize('M', [191, 128 * 133 - 37])
@pytest.mark.parametrize('k', KERNELS)
def test_stores_stay_inside_M_and_N(k, M, res):
    N, K, ldc = 256, 256, 256 + 12
    A, W, b, r = operands(M, N, K, M + N)
    buf = torch.full((M + 70, ldc), SENTINEL, device='cuda')
    out = buf[:M, :N]
    R = None if res is None else r if res == 'sep' else out
    if res == 'alias':
        out.copy_(r)
    launch(k, A, W, b, R, out)
    assert torch.equal(buf[M:], torch.full_like(buf[M:], SENTINEL)), 'rows >= M written'
    assert torch.equal(buf[:M, N:], torch.full_like(buf[:M, N:], SENTINEL)), 'columns N .. ldc written'
    want = torch.empty(M, N, device='cuda')
    if res == 'alias':
        want.copy_(r)
    launch(k, A, W, b, None if res is None else r if res == 'sep' else want, want)
    assert torch.equal(out, want)


@pytest.mark.parametrize('res', ['sep', 'alias'])
@pytest.mark.parametrize('k', KERNELS)
def test_8_byte_aligned_C_and_R_give_the_aligned_bits(k, res):
    M, N, K = 128 * 133 + 61, 384, 256
    A, W, b, r = operands(M, N, K, 17)

    def run(off):
        # C (and a separate R) as [M, N] views starting `off` floats into their buffers, rows N + 4 floats apart
        cb = torch.full((M * (N + 4) + 8,), SENTINEL, device='cuda')
        out = cb[off:off + M * (N + 4)].view(M, N + 4)[:, :N]
        if res == 'alias':
            out.copy_(r)
            R = out
        else:
            rb = torch.zeros(M * (N + 4) + 8, device='cuda')
            R = rb[off:off + M * (N + 4)].view(M, N + 4)[:, :N]
            R.copy_(r)
        assert (out.data_ptr() % 16 == 0) == (off == 0)
        launch(k, A, W, b, R, out)
        return out.clone(), cb

    aligned, _ = run(0)
    shifted, cb = run(2)
    assert torch.equal(shifted, aligned)
    assert torch.equal(cb[:2], torch.full_like(cb[:2], SENTINEL))
