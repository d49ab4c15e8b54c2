"""CPU restatement (torch, float64 inside) of the two confidence-head backward ops of the training path, with the
signatures of e2e_multi_view_matching_b200.ops -- TEST INFRASTRUCTURE ONLY (never imported by the package).

  conf_tail_backward    sigmoid' and the 256 -> 1 Conv1d of ConfidenceMLP.layers (multi_view_matcher.py:39-53)
  conf_gather_backward  the transposes of the head's input gathers (multi_view_matcher.py:302-306):
                        m0 = mdesc0, m1g = mdesc1[b, i0] (-1 -> keypoint N-1), add = scores[b, i, i0] (-1 -> dustbin
                        column N), and the score-input Conv1d (K = 1)

These are what torch autograd computes for the reference's indexing and layers; the GPU tests
(tests/test_train_pose_gpu.py) check csrc/conf_train.cu against them."""
import torch

D = torch.float64


def conf_tail_backward(conf, g_conf, h, w_last):
    c = conf.to(D).reshape(-1)
    gl = g_conf.to(D).reshape(-1) * c * (1.0 - c)
    g_h = gl[:, None] * w_last.to(D).reshape(1, -1)
    return g_h.float(), (gl[:, None] * h.to(D)).sum(0).float(), gl.sum().reshape(1).float()


def conf_gather_backward(g_x, g_pre_c0, add, w_c0, i0, pairs, g_md, g_scores):
    P, B, N = i0.shape
    g_x = g_x.to(D).view(P, B, N, 512)
    gp = g_pre_c0.to(D).view(P, B, N, 256)
    acc = torch.zeros(g_md.shape, dtype=D)
    touched = torch.zeros(g_md.shape[:3], dtype=torch.bool)
    bi = torch.arange(B)[:, None].expand(B, N)
    ii = torch.arange(N)[None].expand(B, N)
    for p, (a, b_) in enumerate(pairs):
        acc[:, a, :N] += g_x[p, :, :, :256]
        touched[:, a, :N] = True
        j = torch.where(i0[p] < 0, i0[p] + N, i0[p])
        acc[:, b_].index_put_((bi, j), g_x[p, :, :, 256:], accumulate=True)
        touched[:, b_][bi, j] = True
        g_add = (gp[p] * w_c0.to(D).reshape(1, 1, 256)).sum(-1)                      # [B, N]
        col = torch.where(i0[p] < 0, torch.full_like(i0[p], N), i0[p])
        sl = g_scores[p * B:(p + 1) * B]
        sl[bi, ii, col] = (sl[bi, ii, col].to(D) + g_add).float()
    upd = (g_md.to(D) + acc).float()
    g_md.copy_(torch.where(touched[..., None], upd, g_md))
    return (gp * add.to(D).view(P, B, N, 1)).sum((0, 1, 2)).float()
