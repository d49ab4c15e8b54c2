"""Repack a reference state dict for the H100 kernels.

* eval-mode BatchNorm1d folded into the preceding 1x1 conv:
    W' = W * g / sqrt(var + eps),  b' = (b - mean) * g / sqrt(var + eps) + beta
  (MLP factories superglue.py:51-62, multi_view_matcher.py:8-22; eps = 1e-5)
* q/k/v output rows and merge input columns permuted from the reference's
  ``.view(B, 64, 4, N)`` interleave (channel = d*4 + h, superglue.py:106,109) to
  head-contiguous (h*64 + d); q,k,v stacked into one [768,256] matrix
* everything concatenated in one device buffer (256-byte aligned sub-tensors) so the
  whole model is a single allocation that stays L2-resident (19 M params = 76 MB).
Keys may carry the DataParallel/DDP ``module.`` prefix (helpers.py:27-33).
"""
import torch

from . import _lib

BN_EPS = 1e-5


def _strip(sd):
    out = {}
    for k, v in sd.items():
        out[k[7:] if k.startswith('module.') else k] = v
    return out


def _conv(sd, key):
    w = sd[key + '.weight'].detach().double().cpu()
    b = sd[key + '.bias'].detach().double().cpu()
    return w.reshape(w.shape[0], w.shape[1]), b


def _fold(sd, conv_key, bn_key):
    w, b = _conv(sd, conv_key)
    g = sd[bn_key + '.weight'].detach().double().cpu()
    beta = sd[bn_key + '.bias'].detach().double().cpu()
    mean = sd[bn_key + '.running_mean'].detach().double().cpu()
    var = sd[bn_key + '.running_var'].detach().double().cpu()
    s = g / torch.sqrt(var + BN_EPS)
    return w * s[:, None], (b - mean) * s + beta


def head_permutation(d_model=256, heads=4):
    """src[c'] = reference channel feeding head-contiguous channel c' = h*64 + d."""
    dim = d_model // heads
    cp = torch.arange(d_model)
    return (cp % dim) * heads + (cp // dim)


class PackedMatcher:
    """Flat device buffer + the mvm_matcher_weights struct pointing into it."""

    def __init__(self, state_dict, layer_names, conf_mlp=True, device='cuda', fold_merge=True):
        sd = _strip(state_dict)
        tensors = []   # (name, cpu double tensor)

        def add(name, t):
            tensors.append((name, t.contiguous()))

        n_kenc = 5
        for i in range(n_kenc):
            ck = 'kenc.encoder.%d' % (3 * i)
            if i < n_kenc - 1:
                w, b = _fold(sd, ck, 'kenc.encoder.%d' % (3 * i + 1))
            else:
                w, b = _conv(sd, ck)
            add('kenc_w%d' % i, w)
            add('kenc_b%d' % i, b)
        src = head_permutation()
        for l, _ in enumerate(layer_names):
            p = 'gnn.layers.%d.' % l
            ws, bs = [], []
            for j in range(3):
                w, b = _conv(sd, p + 'attn.proj.%d' % j)
                ws.append(w[src])
                bs.append(b[src])
            add('l%d_w_qkv' % l, torch.cat(ws, 0))
            add('l%d_b_qkv' % l, torch.cat(bs, 0))
            wm, bm = _conv(sd, p + 'attn.merge')
            wm = wm[:, src]
            w, b = _fold(sd, p + 'mlp.0', p + 'mlp.1')
            if fold_merge:
                # mlp.0(cat[x, merge(a)]) = W0x x + (W0m Wm) a + (b0 + W0m bm): merge is linear and has no other
                # consumer (superglue.py:109,121), so it is folded offline in fp64: -10 % GEMM FLOPs, one launch
                # and one [rows,256] round trip less per layer
                d = wm.shape[0]
                b = b + w[:, d:] @ bm
                w = torch.cat([w[:, :d], w[:, d:] @ wm], 1)
            else:
                add('l%d_w_merge' % l, wm)
                add('l%d_b_merge' % l, bm)
            add('l%d_w_mlp0' % l, w)
            add('l%d_b_mlp0' % l, b)
            w, b = _conv(sd, p + 'mlp.3')
            add('l%d_w_mlp1' % l, w)
            add('l%d_b_mlp1' % l, b)
        w, b = _conv(sd, 'final_proj')
        add('w_final', w)
        add('b_final', b)
        conf_bl = 0.0
        if conf_mlp:
            w, b = _fold(sd, 'conf_mlp.layers_f.0', 'conf_mlp.layers_f.1')
            add('conf_wf0', w); add('conf_bf0', b)
            w, b = _fold(sd, 'conf_mlp.layers_f.3', 'conf_mlp.layers_f.4')
            add('conf_wf1', w); add('conf_bf1', b)
            w, b = _fold(sd, 'conf_mlp.layers_c.0', 'conf_mlp.layers_c.1')
            add('conf_wc0', w.reshape(-1)); add('conf_bc0', b)
            w, b = _fold(sd, 'conf_mlp.layers_c.3', 'conf_mlp.layers_c.4')
            add('conf_wc1', w); add('conf_bc1', b)
            w, b = _conv(sd, 'conf_mlp.layers.0')
            add('conf_wl', w.reshape(-1))
            conf_bl = float(b.reshape(-1)[0])

        offsets, off = {}, 0
        for name, t in tensors:
            offsets[name] = off
            off += (t.numel() + 63) // 64 * 64
        flat = torch.zeros(off, dtype=torch.float32)
        for name, t in tensors:
            flat[offsets[name]:offsets[name] + t.numel()] = t.reshape(-1).float()
        # three planes in one allocation: raw fp32 | rn_tf32(w) | rn_tf32(w - rn_tf32(w))
        def rn_tf32(x):     # cvt.rna.tf32.f32: round to nearest, ties away, on the 13 dropped bits
            return ((x.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)
        hi = rn_tf32(flat)
        lo = rn_tf32(flat - hi)
        self.flat = torch.cat([flat, hi, lo]).to(device)
        # half-precision planes for the fp16x3 GEMMs: hi = fp16(S w), lo = fp16(S w - hi); the power-of-two scale S lifts
        # the lo plane out of the fp16 subnormals (|w| ~ 0.06 -> |lo| ~ 2e-5 unscaled) and is divided out in the epilogue
        self.w16_scale = 64.0
        assert float(flat.abs().max()) * self.w16_scale < 6.0e4, 'weight magnitude exceeds the fp16 range of the fp16x3 GEMM planes'
        scaled = flat.double() * self.w16_scale
        h16 = scaled.to(torch.float16)
        l16 = (scaled - h16.double()).to(torch.float16)
        self.flat16 = torch.cat([h16, l16]).to(device)
        self.offsets = offsets
        base = self.flat.data_ptr()

        def P(name):
            return base + 4 * offsets[name]

        W = _lib.MatcherWeights()
        W.n_layers = len(layer_names)
        W.hi_offset = off
        W.lo_offset = 2 * off
        for i in range(n_kenc):
            W.kenc_w[i] = P('kenc_w%d' % i)
            W.kenc_b[i] = P('kenc_b%d' % i)
        for l, name in enumerate(layer_names):
            L = W.layers[l]
            for f in ('w_qkv', 'b_qkv', 'w_merge', 'b_merge', 'w_mlp0', 'b_mlp0', 'w_mlp1', 'b_mlp1'):
                setattr(L, f, P('l%d_%s' % (l, f)) if 'l%d_%s' % (l, f) in offsets else None)
            L.is_cross = 1 if name == 'cross' else 0
        W.w_final = P('w_final')
        W.b_final = P('b_final')
        W.bin_score = float(sd['bin_score'])
        W.has_conf = 1 if conf_mlp else 0
        if conf_mlp:
            for f in ('conf_wf0', 'conf_bf0', 'conf_wf1', 'conf_bf1', 'conf_wc0', 'conf_bc0',
                      'conf_wc1', 'conf_bc1', 'conf_wl'):
                setattr(W, f, P(f))
            W.conf_bl = conf_bl
        W.flat_base = base
        W.w16_hi = self.flat16.data_ptr()
        W.w16_lo = self.flat16.data_ptr() + 2 * off
        W.w16_scale = self.w16_scale
        self.struct = W
        self.n_layers = len(layer_names)
        self.has_conf = bool(conf_mlp)
        self.fold_merge = bool(fold_merge)
