"""Tensor-core attention on views of at most 64 keys: every key segment is one tile, so the pipelined kernel runs only its
first and last stages, and with n_pad = 64 the second consumer warpgroup of each CTA holds no query row of the view."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('cfg', [(1, 2, 64, [64, 64]), (2, 3, 64, [1, 40, 64]), (1, 4, 128, [64, 17, 128, 3])])
@pytest.mark.parametrize('passes', ['h3', 1, 3])
def test_attention_single_key_tile_vs_fp32(cfg, passes):
    from e2e_multi_view_matching_b200 import ops
    B, T, n_pad, counts = cfg
    g = torch.Generator().manual_seed(7 * n_pad + T)
    qkv = torch.randn(B * T, n_pad, 768, generator=g).cuda()
    for is_cross in (0, 1):
        ref = ops.attention(qkv, B, T, counts, is_cross)                     # fp32 CUDA cores
        out = ops.attention(qkv, B, T, counts, is_cross, tc_passes=passes)
        tol = 2e-2 if passes == 1 else 1e-4                                 # single-pass tf32: 10-bit mantissa
        for b in range(B):
            for t in range(T):
                v = b * T + t
                err = (out[v, :counts[t]] - ref[v, :counts[t]]).abs().max().item()
                assert err < tol, (cfg, passes, is_cross, t, err)
