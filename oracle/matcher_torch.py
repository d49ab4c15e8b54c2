"""torch restatement of the reference matcher forward (eval mode), op for op (CPU by default; `device=` runs the
same stock-PyTorch ops on a GPU for bench.py's informational "torch_gpu_port" line).

TEST INFRASTRUCTURE ONLY.  Same functions as oracle/matcher.py (numpy) but written with the torch
ops the reference itself calls (F.conv1d, einsum, softmax, logsumexp), so that the CPU baseline of
bench.py is timed on the same library path the reference runs on a CPU (multi-threaded MKL/oneDNN)
rather than on a slower numpy rewrite.  Checked against tests/golden/ by tests/test_oracle_matcher.py.
Citations: see oracle/matcher.py (identical structure).
"""
import numpy as np
import torch
import torch.nn.functional as F

from e2e_multi_view_matching_b200.synthetic import BN_EPS


def _t(sd):
    return {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}


def _mlp(sd, prefix, channels, x, last_layer=True):
    n = len(channels)
    for i in range(1, n):
        k = '%s.%d' % (prefix, 3 * (i - 1))
        x = F.conv1d(x, sd[k + '.weight'], sd[k + '.bias'])
        if i < (n - 1 if last_layer else n):
            b = '%s.%d' % (prefix, 3 * (i - 1) + 1)
            x = F.batch_norm(x, sd[b + '.running_mean'], sd[b + '.running_var'], sd[b + '.weight'], sd[b + '.bias'],
                             False, 0.1, BN_EPS)
            x = F.relu(x)
    return x


def _normalize_keypoints(kpts, image_shape):
    _, _, height, width = image_shape
    one = kpts.new_tensor(1)
    size = torch.stack([one * width, one * height])[None]
    center = size / 2
    scaling = size.max(1, keepdim=True).values * 0.7
    return (kpts - center[:, None, :]) / scaling[:, None, :]


def _attn_prop(sd, p, x, source):
    b = x.size(0)
    q = F.conv1d(x, sd[p + '.attn.proj.0.weight'], sd[p + '.attn.proj.0.bias']).view(b, 64, 4, -1)
    k = F.conv1d(source, sd[p + '.attn.proj.1.weight'], sd[p + '.attn.proj.1.bias']).view(b, 64, 4, -1)
    v = F.conv1d(source, sd[p + '.attn.proj.2.weight'], sd[p + '.attn.proj.2.bias']).view(b, 64, 4, -1)
    scores = torch.einsum('bdhn,bdhm->bhnm', q, k) / 64 ** .5
    prob = torch.softmax(scores, dim=-1)
    msg = torch.einsum('bhnm,bdhm->bdhn', prob, v).contiguous().view(b, 256, -1)
    msg = F.conv1d(msg, sd[p + '.attn.merge.weight'], sd[p + '.attn.merge.bias'])
    return _mlp(sd, p + '.mlp', [512, 512, 256], torch.cat([x, msg], dim=1))


def _log_optimal_transport(scores, alpha, iters):
    b, m, n = scores.shape
    one = scores.new_tensor(1)
    ms, ns = (m * one).to(scores), (n * one).to(scores)
    bins0 = alpha.expand(b, m, 1)
    bins1 = alpha.expand(b, 1, n)
    alpha = alpha.expand(b, 1, 1)
    Z = torch.cat([torch.cat([scores, bins0], -1), torch.cat([bins1, alpha], -1)], 1)
    norm = -(ms + ns).log()
    log_mu = torch.cat([norm.expand(m), ns.log()[None] + norm])[None].expand(b, -1)
    log_nu = torch.cat([norm.expand(n), ms.log()[None] + norm])[None].expand(b, -1)
    u, v = torch.zeros_like(log_mu), torch.zeros_like(log_nu)
    for _ in range(iters):
        u = log_mu - torch.logsumexp(Z + v.unsqueeze(1), dim=2)
        v = log_nu - torch.logsumexp(Z + u.unsqueeze(2), dim=1)
    return Z + u.unsqueeze(2) + v.unsqueeze(1) - norm


def confidence_head(sd, mdesc0, mdesc1, scores, indices0):
    """ConfidenceMLP and its call site (multi_view_matcher.py:39-53, :302-306) in the dtype of mdesc0: the conf_mlp
    weights of `sd` (torch tensors) are cast to it.  mdesc0 [B, 256, m], mdesc1 [B, 256, n], scores [B, m+1, n+1],
    indices0 [B, m] (int64, -1 = no match: gathers the last keypoint of view 1 and the dustbin column).
    Returns [B, m, 1]."""
    dt, dev = mdesc0.dtype, mdesc0.device
    sd = {k: (v.to(dev, dt) if v.is_floating_point() else v) for k, v in sd.items() if k.startswith('conf_mlp.')}
    bi = torch.arange(indices0.shape[0], device=dev).unsqueeze(-1).repeat(1, indices0.shape[-1])
    add = scores.to(dt)[bi, torch.arange(indices0.shape[-1], device=dev), indices0].unsqueeze(-2)
    g1 = mdesc1.transpose(-2, -1)[bi, indices0].transpose(-2, -1)
    of = _mlp(sd, 'conf_mlp.layers_f', [512, 512, 256], torch.cat([mdesc0, g1], -2), last_layer=False)
    oc = _mlp(sd, 'conf_mlp.layers_c', [1, 256, 256], add, last_layer=False)
    return torch.sigmoid(_mlp(sd, 'conf_mlp.layers', [256, 1], of + oc)).transpose(-2, -1)


def matcher_forward(sd_np, config, data_np, device=None, to_numpy=True):
    """MultiViewMatcher.forward (eval, multi_frame_matching=True branch or pairwise) -> numpy dict."""
    dev = torch.device(device) if device is not None else torch.device('cpu')
    sd = {k: v.to(dev) for k, v in _t(sd_np).items()}
    out = (lambda t: t.cpu().numpy()) if to_numpy else (lambda t: t)
    names = config['GNN_layers']
    multi = config.get('multi_frame_matching', True)
    iters = config.get('sinkhorn_iterations', 100)
    data = {k: (torch.from_numpy(v).to(dev) if isinstance(v, np.ndarray) else (v.to(dev) if torch.is_tensor(v) and not v.is_meta else v))
            for k, v in data_np.items()}
    T = len(data['ids'])
    res = {}
    with torch.no_grad():
        def kenc(i, img):
            k = _normalize_keypoints(data['keypoints%d' % i], data[img].shape)
            inp = torch.cat([k.transpose(1, 2), data['scores%d' % i].unsqueeze(1)], 1)
            return data['descriptors%d' % i] + _mlp(sd, 'kenc.encoder', [3, 32, 64, 128, 256, 256], inp)

        def head(d0, d1, a, b):
            m0 = F.conv1d(d0, sd['final_proj.weight'], sd['final_proj.bias'])
            m1 = F.conv1d(d1, sd['final_proj.weight'], sd['final_proj.bias'])
            sc = torch.einsum('bdn,bdm->bnm', m0, m1) / 256 ** .5
            sc = _log_optimal_transport(sc, sd['bin_score'], iters)
            max0, max1 = sc[:, :-1, :-1].max(2), sc[:, :-1, :-1].max(1)
            i0, i1 = max0.indices, max1.indices
            ar0 = torch.arange(i0.shape[1], device=dev)[None]
            ar1 = torch.arange(i1.shape[1], device=dev)[None]
            mut0 = ar0 == i1.gather(1, i0)
            mut1 = ar1 == i0.gather(1, i1)
            zero = sc.new_tensor(0)
            ms0 = torch.where(mut0, max0.values.exp(), zero)
            ms1 = torch.where(mut1, ms0.gather(1, i1), zero)
            v0 = mut0 & (ms0 > 0.)
            v1 = mut1 & v0.gather(1, i1)
            i0 = torch.where(v0, i0, i0.new_tensor(-1))
            i1 = torch.where(v1, i1, i1.new_tensor(-1))
            conf = confidence_head(sd, m0, m1, sc, i0)
            res['matches%d_%d_%d' % (a, a, b)] = out(i0)
            res['matches%d_%d_%d' % (b, a, b)] = out(i1)
            res['matching_scores%d_%d_%d' % (a, a, b)] = out(ms0)
            res['matching_scores%d_%d_%d' % (b, a, b)] = out(ms1)
            res['scores_%d_%d' % (a, b)] = out(sc)
            res['conf_scores_%d_%d' % (a, b)] = out(conf)

        if multi:
            desc = [kenc(i, 'image0') for i in range(T)]
            for l, name in enumerate(names):
                p = 'gnn.layers.%d' % l
                if name == 'cross':
                    delta = [_attn_prop(sd, p, desc[i], torch.cat([desc[j] for j in range(T) if j != i], -1))
                             for i in range(T)]
                    desc = [d + dl for d, dl in zip(desc, delta)]
                else:
                    desc = [d + _attn_prop(sd, p, d, d) for d in desc]
            for b in range(T):
                for a in range(b):
                    head(desc[a], desc[b], a, b)
        else:
            for b in range(T):
                for a in range(b):
                    d0, d1 = kenc(a, 'image%d' % a), kenc(b, 'image%d' % b)
                    for l, name in enumerate(names):
                        p = 'gnn.layers.%d' % l
                        s0, s1 = (d1, d0) if name == 'cross' else (d0, d1)
                        n0, n1 = _attn_prop(sd, p, d0, s0), _attn_prop(sd, p, d1, s1)
                        d0, d1 = d0 + n0, d1 + n1
                    head(d0, d1, a, b)
    return res
