"""TRAIN-MODE forward AND backward of the matcher (SURVEY.md 8 a8 / a13 / f-2): the `self.training` branches of
models/models/multi_view_matcher.py -- stacked views (:219-226), KeypointEncoder / AttentionalPropagation /
ConfidenceMLP with BatchNorm1d in training mode, i.e. BATCH statistics over all B*T*N points of the call and
running-statistics updates (:8-22), combined cross attention over the other views (:65-86), `full_output` gating
(:187,287,316-319) -- and the gradient of the `scores_*` outputs w.r.t. every parameter on that path, which is what
`loss.backward()` computes for the reference when it trains on the match loss (train.py stage 1, helpers.py:228-260).

The eval forward runs as one fused C call on packed weights with the BatchNorms folded into the convolutions; batch
statistics cannot be folded, so the train branch sequences the stage kernels from Python: tensor-core GEMMs (fp16x3 forward,
3xTF32 backward -- gradients need the fp32 exponent range), the fp16x3 attention forward, `mvm_attention_backward`,
`mvm_batchnorm_train[_backward]`, `mvm_sinkhorn_train_{forward,backward}` (exact gradient of the unrolled iterations).
The whole matcher is ONE autograd.Function (`MatcherTrainFn`): its inputs are the module's parameters, its outputs the
coupling matrices, so `loss.backward()`, torch optimisers and DistributedDataParallel's gradient hooks work unchanged.

The confidence head's graph is opt-in, through the matcher config key `conf_grad` (default False; training.run_matcher
sets it to opt.pose_loss, like `full_output`).  With `full_output` and `conf_grad` in train mode under autograd, the
forward keeps the head's state of every pair (its inputs m0, m1g and the score input, the pre- and post-BatchNorm
activations and statistics, h = out_f + out_c, the sigmoid output, the matches) and `conf_scores_*` are differentiable
outputs beside `scores_*`.  Their gradient runs back through the head (`mvm_conf_tail_backward`, the 3xTF32 GEMMs, the
BatchNorm backward with one group per pair, `mvm_conf_gather_backward`) into the couplings, before the Sinkhorn
backward, and into the matching descriptors, before the final projection's backward: stage 2 of training (the pose
loss).  The forward's outputs and running statistics are bitwise those of `conf_grad=False`, and when no loss reaches
`conf_scores` the head's backward does not run.  Without `conf_grad` the `conf_scores_*` of `full_output` carry no
graph.  `matching_scores*` never do (the reference computes them under torch.no_grad())."""
import torch

from .. import _lib
from .. import ops
from .multi_view_matcher import image_wh


def _round_up(x, m):
    return (x + m - 1) // m * m


def _head_perm(device):
    """new channel h*64 + d  <-  reference channel d*4 + h (superglue.py:106: .view(B, 64, 4, N))."""
    return torch.arange(256, device=device).view(64, 4).t().reshape(-1)


def _lin(x, w, b, relu=False, a2=None, residual=None, alpha=1.0):
    """Conv1d(k=1) on point-major rows: tensor-core fp16x3 when the shape allows, fp32 CUDA cores otherwise."""
    w = w.detach().float().contiguous()
    b = None if b is None else b.detach().float().contiguous()
    K = x.shape[1] + (a2.shape[1] if a2 is not None else 0)
    N = w.shape[0]
    if K % 64 == 0 and N % 128 == 0 and x.shape[1] % 64 == 0:
        return ops.linear(x, w, bias=b, a2=a2, residual=residual, relu=relu, alpha=alpha, tc_passes='h16')
    if K % 16:                                   # first encoder layer (3 inputs), confidence score branch (1 input)
        assert a2 is None
        pad = _round_up(K, 16) - K
        x = torch.nn.functional.pad(x, (0, pad)).contiguous()
        w = torch.nn.functional.pad(w, (0, pad)).contiguous()
    return ops.linear(x, w, bias=b, a2=a2, residual=residual, relu=relu, alpha=alpha, tc_passes=0)


def _bn(x, bn, n_pad, n_valid, relu=True, groups=1, save=False):
    """nn.BatchNorm1d in training mode on x [rows, C]; updates the module's running statistics.  groups > 1: the view
    slots s = g (mod groups) are normalised one group after the other (one BatchNorm call per view, as the pairwise
    train path makes them).  save: out of place (padding rows of y = 0: the weight-gradient GEMMs contract over them), ->
    (y, saved statistics) for the backward; else in place -> y."""
    assert bn.weight is not None and bn.track_running_stats
    momentum = 0.1 if bn.momentum is None else bn.momentum
    with _lib.device_ctx(x.device):
        y, stats = ops.batchnorm_train(x, bn.weight.detach().float().contiguous(), bn.bias.detach().float().contiguous(),
                                       bn.running_mean, bn.running_var, momentum, bn.eps, n_pad, n_valid, relu=relu,
                                       groups=groups, out=torch.zeros_like(x) if save else None, save=save)
    bn.num_batches_tracked += groups
    return (y, stats) if save else y


def _conv(seq, i):
    return seq[i].weight[:, :, 0], seq[i].bias


class _Saved:
    pass


def _forward(model, data, view_ids=None, save=False, debug=None):
    """-> (result dict of MultiViewMatcher.multi_match / .match in training mode for the views `view_ids` (default: all;
    a pair = the pairwise mode, where the keypoint encoder and every GNN layer see one view per BatchNorm call), saved
    state for `_backward` or None)."""
    cfg = model.config
    g_bn = 1 if view_ids is None else len(view_ids)
    ids = list(range(len(data['ids']))) if view_ids is None else list(view_ids)
    T = len(ids)
    views = [model._view(data, i) for i in ids]
    dev = views[0][0].device
    _lib.require_cuda(dev, 'MultiViewMatcher')
    B, N = views[0][0].shape[:2]
    assert N > 0 and all(v[0].shape[:2] == (B, N) for v in views), 'training uses a fixed number of keypoints per view'
    n_pad = max(64, _round_up(N, 64))
    rows = B * T * n_pad
    S = _Saved() if save else None
    # ---- gather the views (one launch) -> point-major rows, slot = b * T + t
    with _lib.device_ctx(dev):
        kp, sc, de = ops.pack_views([tuple(x.detach().float().contiguous() for x in v) for v in views], n_pad)
    x_desc = de.permute(0, 1, 3, 2).reshape(rows, 256).contiguous()
    # ---- normalize_keypoints (superglue.py:65-72) + KeypointEncoder (multi_view_matcher.py:24-37): the multi-frame
    # branch normalises every view by image0 ("assume all images have the same size", :264), the pairwise one each view
    # by its own image (:165-166)
    wh = [image_wh(data, 0)] * T if view_ids is None else [image_wh(data, i) for i in ids]
    inp = torch.zeros(rows, 16, dtype=torch.float32, device=dev)
    inp_slots = inp.view(B, T, n_pad, 16)
    for t, (w_img, h_img) in enumerate(wh):
        center = torch.tensor([w_img / 2.0, h_img / 2.0], dtype=torch.float32, device=dev)
        scaling = 0.7 * float(max(w_img, h_img))
        inp_slots[:, t, :, 0:2] = (kp[:, t] - center) / scaling
    inp[:, 2] = sc.reshape(rows)
    enc = model.kenc.encoder
    h = inp
    kenc_saved = []
    for i in (0, 3, 6, 9):
        w, b = _conv(enc, i)
        if i == 0:
            w = torch.nn.functional.pad(w, (0, 13))
        pre = _lin(h, w, b)
        if save:
            y, st = _bn(pre, enc[i + 1], n_pad, N, groups=g_bn, save=True)
            kenc_saved.append((h, pre, y, st))
            h = y
        else:
            h = _bn(pre, enc[i + 1], n_pad, N, groups=g_bn)
    x = _lin(h, *_conv(enc, 12), residual=x_desc)                            # desc + kenc(kpts, scores)
    if debug is not None:
        debug['kenc'] = (x - x_desc).view(B, T, n_pad, 256)[:, :, :N].clone()
    # ---- MultiFrameAttentionalGNN, train branch (multi_view_matcher.py:65-86)
    perm = _head_perm(dev)
    counts = [N] * T
    layers_saved = []
    for layer, name in zip(model.gnn.layers, model.gnn.names):
        attn = layer.attn
        wqkv = torch.cat([attn.proj[i].weight[:, :, 0][perm] for i in range(3)], 0)
        bqkv = torch.cat([attn.proj[i].bias[perm] for i in range(3)], 0)
        qkv = _lin(x, wqkv, bqkv)
        msg = ops.attention(qkv.view(B * T, n_pad, 768), B, T, counts, 1 if name == 'cross' else 0, tc_passes='h3')
        merged = _lin(msg.view(rows, 256), attn.merge.weight[:, :, 0][:, perm], attn.merge.bias)
        hid_pre = _lin(x, *_conv(layer.mlp, 0), a2=merged)
        if save:
            hid, st = _bn(hid_pre, layer.mlp[1], n_pad, N, groups=g_bn, save=True)
            layers_saved.append((x, qkv, msg, merged, hid_pre, hid, st, name))
        else:
            hid = _bn(hid_pre, layer.mlp[1], n_pad, N, groups=g_bn)
        x_new = _lin(hid, *_conv(layer.mlp, 3), residual=x)                  # desc + delta (multi_view_matcher.py:80,83)
        if debug is not None and 'layer0_delta' not in debug:
            debug['layer0_delta'] = (x_new - x).view(B, T, n_pad, 256)[:, :, :N].clone()
        x = x_new
        if debug is not None:
            debug.setdefault('x_layers', []).append(x.clone())
    # ---- final projection, scores, optimal transport (multi_view_matcher.py:275-285)
    if debug is not None:
        debug['gnn'] = x.view(B, T, n_pad, 256)[:, :, :N].clone()
    md = _lin(x, model.final_proj.weight[:, :, 0], model.final_proj.bias).view(B, T, n_pad, 256)
    result = {}
    full = bool(cfg['full_output'])
    slot = {v: s for s, v in enumerate(ids)}
    alpha = model.bin_score.detach().float().reshape(1).contiguous()
    iters = int(cfg['sinkhorn_iterations'])
    # score matrices of every pair in one launch (score mode of the persistent GEMM, as the eval path), then ONE
    # optimal-transport launch over all (pair, tuple) problems.  The log-domain
    # training kernel keeps the potentials of every iteration; couplings of an untrained / early-training network span
    # thousands of nats, beyond the range of the scaling-domain kernels of the eval path.
    pair_list = [(id0, id1) for id1 in ids for id0 in ids if id0 < id1]
    with _lib.device_ctx(dev):
        raw_all = ops.pair_scores(md, [(slot[id0], slot[id1]) for id0, id1 in pair_list], N)          # [P * B, N+1, N+1]
        Z_all, pot_all = ops.sinkhorn_train_forward(raw_all, alpha, iters, augmented=True)
    pairs_saved = []
    # conf_grad (train mode, autograd on): keep the confidence head's state of every pair for its backward
    conf_grad = save and full and bool(cfg['conf_mlp']) and bool(cfg.get('conf_grad', False))
    conf_saved = {}

    def keep(name, t, p_):
        # the head's state goes straight into pair-major buffers (rows (p B + b) N + i; statistics one row per pair)
        if name not in conf_saved:
            conf_saved[name] = torch.empty((len(pair_list) * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        conf_saved[name][p_ * t.shape[0]:(p_ + 1) * t.shape[0]].copy_(t)
    for p_, (id0, id1) in enumerate(pair_list):
            a, b_ = slot[id0], slot[id1]
            m0 = md[:, a, :N].contiguous()
            m1 = md[:, b_, :N].contiguous()
            Z = Z_all[p_ * B:(p_ + 1) * B]
            key = '{}_{}'.format(id0, id1)
            result['scores_' + key] = Z
            if save:
                pairs_saved.append((key, a, b_))
            if not full:
                continue
            i0, i1, s0, s1 = ops.extract_matches(Z, model.match_threshold)
            conf = None
            if cfg['conf_mlp']:
                # inputs of ConfidenceMLP (multi_view_matcher.py:302-306): -1 wraps to the last keypoint / dustbin column
                bi = torch.arange(B, device=dev).unsqueeze(-1).expand(B, N)
                m1g = m1[bi, i0]                                               # [B, N, 256]
                add = Z[bi, torch.arange(N, device=dev).unsqueeze(0).expand(B, N), i0].reshape(B * N, 1)
                cm = model.conf_mlp

                def head_bn(x, mod):
                    # conf_grad: out of place with the statistics kept (same kernel, same values); else in place
                    return _bn(x, mod, N, N, save=True) if conf_grad else (_bn(x, mod, N, N), None)
                x0, x1 = m0.reshape(B * N, 256), m1g.reshape(B * N, 256).contiguous()
                pre_f0 = _lin(x0, *_conv(cm.layers_f, 0), a2=x1)
                y_f1, st_f1 = head_bn(pre_f0, cm.layers_f[1])
                pre_f3 = _lin(y_f1, *_conv(cm.layers_f, 3))
                f, st_f4 = head_bn(pre_f3, cm.layers_f[4])
                add = add.contiguous()
                pre_c0 = _lin(add, *_conv(cm.layers_c, 0))
                y_c1, st_c1 = head_bn(pre_c0, cm.layers_c[1])
                pre_c3 = _lin(y_c1, *_conv(cm.layers_c, 3))
                c, st_c4 = head_bn(pre_c3, cm.layers_c[4])
                w_last, b_last = _conv(cm.layers, 0)
                h_sum = (f + c).contiguous()
                logit = _lin(h_sum, torch.nn.functional.pad(w_last, (0, 0, 0, 15)), torch.nn.functional.pad(b_last, (0, 15)))
                conf = torch.sigmoid(logit[:, :1]).reshape(B, N, 1)
                if conf_grad:
                    for name, t in dict(m0=x0, m1g=x1, add=add, pre_f0=pre_f0, y_f1=y_f1, st_f1=st_f1, pre_f3=pre_f3,
                                        y_f4=f, st_f4=st_f4, pre_c0=pre_c0, y_c1=y_c1, st_c1=st_c1, pre_c3=pre_c3, y_c4=c,
                                        st_c4=st_c4, h=h_sum, conf=conf.reshape(B * N), i0=i0.reshape(B * N)).items():
                        keep(name, t, p_)
            result['matches{}_{}'.format(id0, key)] = i0
            result['matches{}_{}'.format(id1, key)] = i1
            result['matching_scores{}_{}'.format(id0, key)] = s0
            result['matching_scores{}_{}'.format(id1, key)] = s1
            result['conf_scores_' + key] = conf
    if save:
        S.dims = (B, T, N, n_pad, rows, g_bn)
        S.inp, S.kenc, S.kenc_last_in, S.layers, S.x_final, S.md = inp, kenc_saved, h, layers_saved, x, md
        S.pairs, S.alpha, S.iters, S.perm, S.dev = pairs_saved, alpha, iters, perm, dev
        S.raw_all, S.pot_all = raw_all, pot_all
        S.conf = conf_saved if conf_grad else None
    return result, S


def _backward(model, S, grads):
    """grads: {'scores_a_b': gradient w.r.t. that coupling matrix [B, N+1, N+1] or None} -> {parameter: gradient}."""
    B, T, N, n_pad, rows, g_bn = S.dims
    dev, perm = S.dev, S.perm
    G = {}

    def acc(p, g):
        g = g.reshape(p.shape).to(p.dtype)
        G[p] = g if p not in G else G[p] + g

    # the confidence head's backward runs when it kept its state (conf_grad) and some conf_scores got a gradient
    conf_g = [grads.get('conf_scores_' + key) for key, _, _ in S.pairs] if S.conf is not None else []
    head = any(g is not None for g in conf_g)
    with _lib.device_ctx(dev):
        # ---- optimal transport and the score products (multi_view_matcher.py:275-285)
        g_md = torch.zeros(B, T, n_pad, 256, dtype=torch.float32, device=dev)
        G_all = torch.zeros(len(S.pairs) * B, N + 1, N + 1, dtype=torch.float32, device=dev)
        for p_, (key, a, b_) in enumerate(S.pairs):
            go = grads.get('scores_' + key)
            if go is not None:
                G_all[p_ * B:(p_ + 1) * B] = go
        if head:        # its gradients w.r.t. the couplings and the matching descriptors go in first
            _conf_backward(model, S, conf_g, g_md, G_all, acc)
        dZ_all, d_alpha = ops.sinkhorn_train_backward(S.raw_all, S.alpha, S.pot_all, S.iters, G_all, augmented=True)      # ONE launch
        for p_, (key, a, b_) in enumerate(S.pairs):
            if grads.get('scores_' + key) is None and not (head and conf_g[p_] is not None):
                continue
            dS = torch.zeros(B, n_pad, n_pad, dtype=torch.float32, device=dev)
            dS[:, :N, :N] = dZ_all[p_ * B:(p_ + 1) * B, :N, :N]
            for i in range(B):
                # scores = m0 m1^T / 16:  d m0 = dS m1 / 16,  d m1 = dS^T m0 / 16
                _, hi, lo = ops.transpose_split(S.md[i, b_])
                g_md[i, a] = ops.linear_presplit(dS[i], hi, lo, residual=g_md[i, a], alpha=1.0 / 16.0)
                dSt, _, _ = ops.transpose_split(dS[i], raw=True, planes=False)
                _, hi, lo = ops.transpose_split(S.md[i, a])
                g_md[i, b_] = ops.linear_presplit(dSt, hi, lo, residual=g_md[i, b_], alpha=1.0 / 16.0)
        acc(model.bin_score, d_alpha.float())
        g_md = g_md.view(rows, 256)
        dbg = getattr(model, '_train_debug', None)      # tests: gradients at the stage boundaries, [B, T, N, 256]
        if dbg is not None:
            dbg['g_mdesc'] = g_md.view(B, T, n_pad, 256)[:, :, :N].clone()
        # ---- final projection
        wf = model.final_proj.weight[:, :, 0]
        acc(model.final_proj.weight, ops.gemm_dw(g_md, S.x_final))
        acc(model.final_proj.bias, ops.colsum(g_md))
        gx = ops.gemm_dx(g_md, wf)
        if dbg is not None:
            dbg['g_gnn'] = gx.view(B, T, n_pad, 256)[:, :, :N].clone()
        # ---- GNN layers, last to first (superglue.py:94-121, multi_view_matcher.py:65-86)
        inv = torch.empty_like(perm)
        inv[perm] = torch.arange(256, device=dev)
        for layer, (x_in, qkv, msg, merged, hid_pre, hid, st, name) in zip(reversed(list(model.gnn.layers)), reversed(S.layers)):
            attn = layer.attn
            w0, w3 = layer.mlp[0].weight[:, :, 0], layer.mlp[3].weight[:, :, 0]
            acc(layer.mlp[3].weight, ops.gemm_dw(gx, hid))
            acc(layer.mlp[3].bias, ops.colsum(gx))
            g_hid = ops.gemm_dx(gx, w3)
            dg, db = ops.batchnorm_train_backward(hid_pre, hid, g_hid, layer.mlp[1].weight.detach().float().contiguous(), st,
                                                  n_pad, N)
            acc(layer.mlp[1].weight, dg)
            acc(layer.mlp[1].bias, db)
            acc(layer.mlp[0].weight, ops.gemm_dw(g_hid, x_in, merged))
            acc(layer.mlp[0].bias, ops.colsum(g_hid))
            gx = ops.gemm_dx(g_hid, w0[:, :256], residual=gx)          # residual path + the x half of the concat
            g_merged = ops.gemm_dx(g_hid, w0[:, 256:])
            wm = attn.merge.weight[:, :, 0][:, perm]                    # as the forward used it (message head-contiguous)
            acc(attn.merge.weight, ops.gemm_dw(g_merged, msg.view(rows, 256))[:, inv])
            acc(attn.merge.bias, ops.colsum(g_merged))
            g_msg = ops.gemm_dx(g_merged, wm)
            g_qkv = ops.attention_backward(qkv.view(B * T, n_pad, 768), msg, g_msg.view(B * T, n_pad, 256), B, T, [N] * T,
                                           1 if name == 'cross' else 0).view(rows, 768)
            if dbg is not None:
                dbg.setdefault('layers', []).append({'g_hid': g_hid.clone(), 'g_merged': g_merged.clone(), 'g_msg': g_msg.clone(),
                                                     'g_qkv': g_qkv.clone()})
            g_wqkv = ops.gemm_dw(g_qkv, x_in)                           # [768, 256], rows head-contiguous per projection
            g_bqkv = ops.colsum(g_qkv)
            for i in range(3):
                acc(attn.proj[i].weight, g_wqkv[i * 256:(i + 1) * 256][inv])
                acc(attn.proj[i].bias, g_bqkv[i * 256:(i + 1) * 256][inv])
            wqkv = torch.cat([attn.proj[i].weight[:, :, 0][perm] for i in range(3)], 0)
            gx = ops.gemm_dx(g_qkv, wqkv, residual=gx)
            if dbg is not None:
                dbg['layers'][-1]['gx'] = gx.clone()
        # ---- keypoint encoder (x = kenc(kpts, scores) + descriptors)
        enc = model.kenc.encoder
        if dbg is not None:
            dbg['g_kenc'] = gx.view(B, T, n_pad, 256)[:, :, :N].clone()
        acc(enc[12].weight, ops.gemm_dw(gx, S.kenc_last_in))
        acc(enc[12].bias, ops.colsum(gx))
        g_h = ops.gemm_dx(gx, enc[12].weight[:, :, 0])
        for i, (h_in, pre, y, st) in zip((9, 6, 3, 0), reversed(S.kenc)):
            dg, db = ops.batchnorm_train_backward(pre, y, g_h, enc[i + 1].weight.detach().float().contiguous(), st, n_pad, N)
            acc(enc[i + 1].weight, dg)
            acc(enc[i + 1].bias, db)
            g_w = ops.gemm_dw(g_h, h_in)
            acc(enc[i].weight, g_w[:, :3] if i == 0 else g_w)
            acc(enc[i].bias, ops.colsum(g_h))
            if i:
                g_h = ops.gemm_dx(g_h, enc[i].weight[:, :, 0])
    return G


def _conf_backward(model, S, conf_g, g_md, G_all, acc):
    """Backward of ConfidenceMLP (multi_view_matcher.py:39-53, 302-306) over every pair at once, on the pair-major
    buffers the forward filled (rows r = (p B + b) N + i).  conf_g: per pair the gradient w.r.t. conf_scores
    [B, N, 1] or None (zero).  Adds the gradients w.r.t. the gathered inputs to g_md [B, T, n_pad, 256] (m0, m1g) and
    G_all [P B, N+1, N+1] (add), and the parameter gradients through acc.  Each pair's BatchNorms took their statistics over its own B N rows: one group
    per pair (slot size B N)."""
    B, T, N, n_pad, rows, g_bn = S.dims
    cm = model.conf_mlp
    P = len(S.pairs)
    sv = S.conf
    dbg = getattr(model, '_train_debug', None)      # tests: the head's gradients at its stage boundaries
    g_conf = torch.cat([(g.detach().float() if g is not None else torch.zeros(B, N, 1, device=S.dev)).reshape(-1)
                        for g in conf_g])
    # sigmoid' and the 256 -> 1 layer (csrc/conf_train.cu)
    g_h, dw_last, db_last = ops.conf_tail_backward(sv['conf'], g_conf, sv['h'], cm.layers[0].weight[:, :, 0])
    acc(cm.layers[0].weight, dw_last)
    acc(cm.layers[0].bias, db_last)
    bn_rows = B * N
    g_x = g_pre_c0 = None
    for br, mods in (('f', cm.layers_f), ('c', cm.layers_c)):
        g = g_h.clone() if br == 'f' else g_h         # the BatchNorm backward runs in place
        if dbg is not None:
            dbg.setdefault('conf', {})['g_h'] = g_h.clone()
        dg, db = ops.batchnorm_train_backward(sv['pre_%s3' % br], sv['y_%s4' % br], g,
                                              mods[4].weight.detach().float().contiguous(), sv['st_%s4' % br],
                                              bn_rows, bn_rows)
        acc(mods[4].weight, dg)
        acc(mods[4].bias, db)
        acc(mods[3].weight, ops.gemm_dw(g, sv['y_%s1' % br]))
        acc(mods[3].bias, ops.colsum(g))
        g1 = ops.gemm_dx(g, mods[3].weight[:, :, 0])
        if dbg is not None:
            dbg['conf'].update({'g_pre_%s3' % br: g.clone(), 'g_y_%s1' % br: g1.clone()})
        dg, db = ops.batchnorm_train_backward(sv['pre_%s0' % br], sv['y_%s1' % br], g1,
                                              mods[1].weight.detach().float().contiguous(), sv['st_%s1' % br],
                                              bn_rows, bn_rows)
        acc(mods[1].weight, dg)
        acc(mods[1].bias, db)
        if dbg is not None:
            dbg['conf'].update({'g_pre_%s0' % br: g1.clone(), 'dgamma_%s1' % br: dg.clone()})
        acc(mods[0].bias, ops.colsum(g1))
        if br == 'f':
            acc(mods[0].weight, ops.gemm_dw(g1, sv['m0'], sv['m1g']))
            g_x = ops.gemm_dx(g1, mods[0].weight[:, :, 0])                  # [rows, 512]: m0 | m1g
        else:
            g_pre_c0 = g1
    # the gathers' transposes and the score-input layer (K = 1) (csrc/conf_train.cu)
    i0 = sv['i0'].view(P, B, N)
    dw_c0 = ops.conf_gather_backward(g_x, g_pre_c0, sv['add'], cm.layers_c[0].weight[:, 0, 0], i0,
                                     [(a, b_) for _, a, b_ in S.pairs], g_md, G_all)
    acc(cm.layers_c[0].weight, dw_c0)


class MatcherTrainFn(torch.autograd.Function):
    """(model, data, view_ids, holder, *parameters) -> the coupling matrices of every pair; the non-differentiable
    outputs of `full_output` are left in `holder`."""

    @staticmethod
    def forward(ctx, model, data, view_ids, holder, *params):
        result, S = _forward(model, data, view_ids, save=True)
        keys = [k for k in result if k.startswith('scores_')]
        if S.conf is not None:          # conf_grad: the confidences are differentiable outputs too
            keys += [k for k in result if k.startswith('conf_scores_')]
            # an output without a gradient arrives as None, not zeros: the confidence head's backward runs only when a
            # loss reaches conf_scores
            ctx.set_materialize_grads(False)
        holder.update({k: v for k, v in result.items() if k not in keys})
        holder['__keys__'] = keys
        ctx.model, ctx.S, ctx.keys, ctx.params = model, S, keys, params
        return tuple(result[k] for k in keys)

    @staticmethod
    def backward(ctx, *grads):
        G = _backward(ctx.model, ctx.S, {k: g for k, g in zip(ctx.keys, grads)})
        ctx.S = None
        return (None, None, None, None) + tuple(G.get(p) for p in ctx.params)


def train_forward(model, data, view_ids=None, debug=None):
    """Result dict of the train branch.  With autograd enabled (and parameters that require grad) the `scores_*` tensors
    carry the graph of MatcherTrainFn; under torch.no_grad() this is a plain forward."""
    params = [p for p in model.parameters() if p.requires_grad]
    with _lib.device_ctx(data['keypoints0'].device):      # every launch of the call on the device of the inputs
        if debug is None and torch.is_grad_enabled() and params:
            holder = {}
            outs = MatcherTrainFn.apply(model, data, view_ids, holder, *params)
            result = dict(zip(holder.pop('__keys__'), outs))
            result.update(holder)
            return result
        with torch.no_grad():
            return _forward(model, data, view_ids, save=False, debug=debug)[0]
