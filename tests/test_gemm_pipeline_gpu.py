"""The fp16x3 layer GEMM at the size of a cfg3 step (14 tuples x 5 views x 1024 keypoints = 71680 rows), where every CTA
of the persistent launch walks many output tiles, some CTAs an odd number of them, so the ring stages and barrier phases
carry over from tile to tile.  Rows taken from that launch must be bit-identical to the same rows computed by a small
launch in which each CTA has a single tile: the sum order of an output element does not depend on where its tile falls
in a CTA's walk."""
import pytest
import torch

pytestmark = pytest.mark.gpu

M_FULL = 14 * 5 * 1024


@pytest.mark.parametrize('M', [M_FULL, M_FULL - 37])            # the second one ends in a partial tile of 91 rows
@pytest.mark.parametrize('shape', [(768, 256, 0, 'bias'), (512, 256, 256, 'relu'), (256, 512, 0, 'residual')],
                         ids=['qkv', 'mlp0_concat_relu', 'mlp2_residual'])
def test_h16_gemm_many_tiles_per_cta(M, shape):
    from e2e_multi_view_matching_b200 import ops
    N, K1, K2, epi = shape
    g = torch.Generator().manual_seed(M + N)
    a = (torch.randn(M, K1, generator=g) * 3).cuda()
    a2 = (torch.randn(M, K2, generator=g) * 3).cuda() if K2 else None
    w = (torch.randn(N, K1 + K2, generator=g) / 16).cuda()
    b = torch.randn(N, generator=g).cuda()
    r = torch.randn(M, N, generator=g).cuda() if epi == 'residual' else None
    relu = epi == 'relu'
    out = ops.linear(a, w, bias=b, a2=a2, residual=r, relu=relu, tc_passes='h16')
    t32 = ops.linear(a, w, bias=b, a2=a2, residual=r, relu=relu, tc_passes=3, presplit=True)

    A = torch.cat([a, a2], 1) if a2 is not None else a
    ref = A.double() @ w.double().T + b.double()
    if relu:
        ref = torch.relu(ref)
    if r is not None:
        ref = ref + r.double()
    e_h, e_t = (out.double() - ref).abs().max().item(), (t32.double() - ref).abs().max().item()
    assert e_h < max(1e-4, 2.0 * e_t), (M, shape, e_h, e_t)

    # row blocks: the first tiles, the middle of the walk (not tile-aligned), the last (possibly partial) tile
    for r0, r1 in ((0, 256), (M // 2 - 77, M // 2 + 179), (M - 200, M)):
        small = ops.linear(a[r0:r1].contiguous(), w, bias=b, a2=a2[r0:r1].contiguous() if a2 is not None else None,
                           residual=r[r0:r1].contiguous() if r is not None else None, relu=relu, tc_passes='h16')
        assert torch.equal(small, out[r0:r1]), (M, shape, r0, r1)
