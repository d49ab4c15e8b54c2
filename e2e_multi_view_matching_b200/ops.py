"""Stage-level entry points (torch tensors in/out) over the C ABI.  Names follow the reference
functions they replace (superglue.py:87-172, multi_view_matcher.py:288-300)."""
import ctypes as C

import torch

from . import _lib


def rn_tf32(x):
    """cvt.rna.tf32.f32 on a tensor: round to nearest (ties away) on the 13 dropped mantissa bits."""
    return ((x.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


H16_SCALE = 64.0     # the fp16 planes hold H16_SCALE * W, as packing.py stores them


def h16_planes(w):
    """(hi, lo) fp16 planes of H16_SCALE * w: hi = fp16(s w), lo = fp16(s w - hi)."""
    ws = w.double() * H16_SCALE
    w_hi = ws.to(torch.float16)
    return w_hi.contiguous(), (ws - w_hi.double()).to(torch.float16).contiguous()


def linear(a, w, bias=None, a2=None, residual=None, relu=False, alpha=1.0, tc_passes=0, presplit=False):
    """act(alpha * [a|a2] @ w.T + bias) + residual on point-major activations (Conv1d k=1).
    tc_passes: 0 = fp32 CUDA cores, 3 = 3xTF32 on the tensor cores, 1 = single-pass TF32.
    presplit (with tc_passes=3): hand W over as its tf32 hi/lo planes, like the packed matcher weights do --
    this is the production path (persistent kernel)."""
    lib = _lib.lib()
    if tc_passes == 'h16':      # fp16x3 on the persistent kernel (what the packed matcher weights use by default)
        M, K1 = a.shape
        K = K1 + (a2.shape[1] if a2 is not None else 0)
        N = w.shape[0]
        out = torch.empty(M, N, dtype=torch.float32, device=a.device)
        scale = H16_SCALE
        w_hi, w_lo = h16_planes(w)
        rc = lib.mvm_linear_tc_h16(_lib.ptr(a), a.stride(0), _lib.ptr(a2), a2.stride(0) if a2 is not None else 0, K1,
                                   _lib.ptr(w_hi), _lib.ptr(w_lo), scale, w_hi.stride(0), _lib.ptr(bias), _lib.ptr(residual),
                                   residual.stride(0) if residual is not None else 0, _lib.ptr(out), N, M, N, K,
                                   float(alpha), int(relu), _lib.stream_ptr())
        _lib.check(rc, 'mvm_linear_tc_h16')
        return out
    if tc_passes:
        M, K1 = a.shape
        K = K1 + (a2.shape[1] if a2 is not None else 0)
        N = w.shape[0]
        out = torch.empty(M, N, dtype=torch.float32, device=a.device)
        if presplit:
            assert tc_passes == 3
            w_hi = rn_tf32(w)
            w_lo = rn_tf32(w - w_hi)
            rc = lib.mvm_linear_tc_presplit(_lib.ptr(a), a.stride(0), _lib.ptr(a2), a2.stride(0) if a2 is not None else 0,
                                            K1, _lib.ptr(w_hi), _lib.ptr(w_lo), w_hi.stride(0), _lib.ptr(bias),
                                            _lib.ptr(residual), residual.stride(0) if residual is not None else 0,
                                            _lib.ptr(out), N, M, N, K, float(alpha), int(relu), _lib.stream_ptr())
            _lib.check(rc, 'mvm_linear_tc_presplit')
            return out
        rc = lib.mvm_linear_tc(_lib.ptr(a), a.stride(0), _lib.ptr(a2), a2.stride(0) if a2 is not None else 0,
                               K1, _lib.ptr(w), w.stride(0), _lib.ptr(bias), _lib.ptr(residual),
                               residual.stride(0) if residual is not None else 0, _lib.ptr(out), N, M, N, K,
                               float(alpha), int(relu), int(tc_passes), _lib.stream_ptr())
        _lib.check(rc, 'mvm_linear_tc')
        return out
    M, K1 = a.shape
    K = K1 + (a2.shape[1] if a2 is not None else 0)
    N = w.shape[0]
    out = torch.empty(M, N, dtype=torch.float32, device=a.device)
    rc = lib.mvm_linear(_lib.ptr(a), a.stride(0), _lib.ptr(a2), a2.stride(0) if a2 is not None else 0,
                        K1, _lib.ptr(w), w.stride(0), _lib.ptr(bias), _lib.ptr(residual),
                        residual.stride(0) if residual is not None else 0, _lib.ptr(out), N, M, N, K,
                        float(alpha), int(relu), _lib.stream_ptr())
    _lib.check(rc, 'mvm_linear')
    return out


def qkv_projection(x, w, bias, n_pad, planes='fp16', w16=True, out=None):
    """The QKV projection of one GNN layer as the matcher launches it (mvm_qkv_projection): x [rows, 256], w [768, 256],
    bias [768] -> (qkv [rows, 768] with Q in columns 0..255, planes).
    planes 'fp16': (kh, kl, vh, vl), half [rows, 256], for the fp16x3 attention; W enters as the fp16 planes of
    H16_SCALE * w (w16) or as its tf32 planes.  planes 'tf32': (klo [rows, 256], vt, vtlo [rows / n_pad, 256, n_pad]),
    with rn_tf32(K) in columns 256..511 of qkv.  Columns of qkv that go to planes are left as `out` had them."""
    lib = _lib.lib()
    rows = x.shape[0]
    dev = x.device
    qkv = torch.empty(rows, 768, dtype=torch.float32, device=dev) if out is None else out
    w_hi = rn_tf32(w)
    w_lo = rn_tf32(w - w_hi)
    h_hi, h_lo = h16_planes(w) if (planes == 'fp16' and w16) else (None, None)
    if planes == 'fp16':
        p = tuple(torch.empty(rows, 256, dtype=torch.float16, device=dev) for _ in range(4))
        ptrs = p
    else:
        p = (torch.empty(rows, 256, dtype=torch.float32, device=dev),
             torch.empty(rows // n_pad, 256, n_pad, dtype=torch.float32, device=dev),
             torch.empty(rows // n_pad, 256, n_pad, dtype=torch.float32, device=dev))
        ptrs = (None,) + p
    _lib.check(lib.mvm_qkv_projection(_lib.ptr(x), _lib.ptr(w_hi), _lib.ptr(w_lo), _lib.ptr(h_hi), _lib.ptr(h_lo),
                                      H16_SCALE, _lib.ptr(bias), _lib.ptr(qkv), rows, n_pad, int(planes == 'fp16'),
                                      *[_lib.ptr(t) for t in ptrs], _lib.stream_ptr()), 'mvm_qkv_projection')
    return qkv, p


def attention(qkv, batch, n_views, counts, is_cross, tc_passes=0):
    """qkv [batch*n_views, n_pad, 768] (q|k|v, head-contiguous) -> [batch*n_views, n_pad, 256]."""
    lib = _lib.lib()
    V, n_pad, _ = qkv.shape
    out = torch.zeros(V, n_pad, 256, dtype=torch.float32, device=qkv.device)
    cnt = (C.c_int * n_views)(*counts)
    if tc_passes == 'h3':     # fp16x3: the planes the QKV GEMM epilogue writes in the matcher
        k = qkv[:, :, 256:512].contiguous()
        kh = k.half()
        kl = (k - kh.float()).half().reshape(-1, 256).contiguous()
        kh = kh.reshape(-1, 256).contiguous()
        v = qkv[:, :, 512:].contiguous()                      # V stays key-major [rows, 256] (MN-major B operand)
        vh = v.half()
        vl = (v - vh.float()).half().reshape(-1, 256).contiguous()
        vh = vh.reshape(-1, 256).contiguous()
        rc = lib.mvm_attention_h3(_lib.ptr(qkv), _lib.ptr(kh), _lib.ptr(kl), _lib.ptr(vh), _lib.ptr(vl),
                                  _lib.ptr(out), batch, n_views, n_pad, cnt, int(is_cross), _lib.stream_ptr())
        _lib.check(rc, 'mvm_attention_h3')
        return out
    if tc_passes:
        vt = qkv[:, :, 512:].transpose(1, 2).contiguous()      # [V, 256, n_pad]
        klo = vtlo = None
        if tc_passes == 3:      # what the QKV GEMM epilogue does in 3xTF32 mode: rn_tf32 planes + remainders
            def rn(x):          # round to nearest (ties away) on the 13 dropped mantissa bits
                return ((x.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)
            qkv = qkv.clone()
            k = qkv[:, :, 256:512].contiguous()
            khi = rn(k)
            klo = rn(k - khi).reshape(-1, 256).contiguous()
            qkv[:, :, 256:512] = khi
            vhi = rn(vt)
            vtlo = rn(vt - vhi).contiguous()
            vt = vhi
        rc = lib.mvm_attention_tc(_lib.ptr(qkv), _lib.ptr(vt), _lib.ptr(out), batch, n_views, n_pad, cnt,
                                  int(is_cross), int(tc_passes), _lib.ptr(klo), _lib.ptr(vtlo), _lib.stream_ptr())
        _lib.check(rc, 'mvm_attention_tc')
        return out
    rc = lib.mvm_attention(_lib.ptr(qkv), _lib.ptr(out), batch, n_views, n_pad, cnt, int(is_cross),
                           _lib.stream_ptr())
    _lib.check(rc, 'mvm_attention')
    return out


def log_optimal_transport(scores, alpha, iters, ref_kernel=False, kernel=None):
    """superglue.py:152-172: scores [B,m,n] -> couplings [B,m+1,n+1]."""
    lib = _lib.lib()
    B, m, n = scores.shape
    Z = torch.empty(B, m + 1, n + 1, dtype=torch.float32, device=scores.device)
    Z[:, :m, :n] = scores
    nws = lib.mvm_sinkhorn_workspace_floats(1, B, max(m, n))
    ws = torch.empty(nws, dtype=torch.float32, device=scores.device)
    variants = {'multicta': 1, 'cluster': 2, 'cluster6': 3, 'cluster2': 4}
    if kernel in variants:
        rc = lib.mvm_log_optimal_transport_ex(_lib.ptr(Z), B, m, n, float(alpha), int(iters), _lib.ptr(ws),
                                              variants[kernel], _lib.stream_ptr())
        _lib.check(rc, 'mvm_log_optimal_transport_ex')
        return Z
    fn = {None: lib.mvm_log_optimal_transport, 'ref': lib.mvm_log_optimal_transport_ref,
          'log': lib.mvm_log_optimal_transport_logdomain}['ref' if ref_kernel else kernel]
    rc = fn(_lib.ptr(Z), B, m, n, float(alpha), int(iters), _lib.ptr(ws), _lib.stream_ptr())
    _lib.check(rc, 'mvm_log_optimal_transport')
    return Z


def extract_matches(Z, match_threshold=0.0):
    """multi_view_matcher.py:288-300 on couplings [B,m+1,n+1]."""
    lib = _lib.lib()
    B, m1, n1 = Z.shape
    m, n = m1 - 1, n1 - 1
    dev = Z.device
    m0 = torch.empty(B, m, dtype=torch.int64, device=dev)
    m1_ = torch.empty(B, n, dtype=torch.int64, device=dev)
    s0 = torch.empty(B, m, dtype=torch.float32, device=dev)
    s1 = torch.empty(B, n, dtype=torch.float32, device=dev)
    n_pad = (max(m, n) + 63) // 64 * 64
    ws = torch.empty(3 * B * n_pad, dtype=torch.int32, device=dev)
    rc = lib.mvm_extract_matches(_lib.ptr(Z.contiguous()), B, m, n, float(match_threshold), _lib.ptr(m0),
                                 _lib.ptr(m1_), _lib.ptr(s0), _lib.ptr(s1), _lib.ptr(ws), _lib.stream_ptr())
    _lib.check(rc, 'mvm_extract_matches')
    return m0, m1_, s0, s1


# ---- training-path stage ops (SURVEY.md 8 f-2): operand staging + backward GEMMs, BatchNorm, attention, Sinkhorn -------

def pack_views(views, n_pad):
    """views: [(keypoints [B, N, 2], scores [B, N], descriptors [B, 256, N])] per view -> the zero-padded view-slot-major
    buffers kpts [B, T, n_pad, 2], scores [B, T, n_pad], desc [B, T, 256, n_pad] (mvm_pack_views, one launch)."""
    lib = _lib.lib()
    T = len(views)
    B = views[0][0].shape[0]
    dev = views[0][0].device
    kp = torch.empty(B, T, n_pad, 2, dtype=torch.float32, device=dev)
    sc = torch.empty(B, T, n_pad, dtype=torch.float32, device=dev)
    de = torch.empty(B, T, 256, n_pad, dtype=torch.float32, device=dev)
    ptrs = [(C.c_void_p * T)(*[v[i].data_ptr() for v in views]) for i in range(3)]
    counts = (C.c_int * T)(*[v[0].shape[1] for v in views])
    _lib.check(lib.mvm_pack_views(ptrs[0], ptrs[1], ptrs[2], counts, B, T, n_pad, _lib.ptr(kp), _lib.ptr(sc), _lib.ptr(de),
                                  _lib.stream_ptr()), 'mvm_pack_views')
    return kp, sc, de


def transpose_split(x, raw=False, planes=True, out=None):
    """x [R, C] -> ([C, R] raw copy or None, tf32 hi plane or None, lo plane or None) of x^T (mvm_transpose_split).
    out: optional (raw, hi, lo) destination views with row stride `ldo` = out[..].stride(0) (concat-by-rows staging)."""
    lib = _lib.lib()
    R, Cc = x.shape
    assert x.stride(1) == 1
    if out is None:
        r = torch.empty(Cc, R, dtype=torch.float32, device=x.device) if raw else None
        h = torch.empty(Cc, R, dtype=torch.float32, device=x.device) if planes else None
        l = torch.empty(Cc, R, dtype=torch.float32, device=x.device) if planes else None
    else:
        r, h, l = out
    ldo = (r if r is not None else h).stride(0)
    _lib.check(lib.mvm_transpose_split(_lib.ptr(x), R, Cc, x.stride(0), _lib.ptr(r), _lib.ptr(h), _lib.ptr(l), ldo,
                                       _lib.stream_ptr()), 'mvm_transpose_split')
    return r, h, l


def linear_presplit(a, w_hi, w_lo, residual=None, alpha=1.0):
    """alpha * a [M, K] @ w^T + residual with w [N, K] given as its tf32 planes: the 3xTF32 tensor-core GEMM (fp32 range --
    the half-precision planes of the inference path would flush small gradients)."""
    lib = _lib.lib()
    M, K = a.shape
    N = w_hi.shape[0]
    out = torch.empty(M, N, dtype=torch.float32, device=a.device)
    rc = lib.mvm_linear_tc_presplit(_lib.ptr(a), a.stride(0), None, 0, K, _lib.ptr(w_hi), _lib.ptr(w_lo), w_hi.stride(0),
                                    None, _lib.ptr(residual), residual.stride(0) if residual is not None else 0,
                                    _lib.ptr(out), N, M, N, K, float(alpha), 0, _lib.stream_ptr())
    _lib.check(rc, 'mvm_linear_tc_presplit')
    return out


def linear_presplit_splitk(a, w_hi, w_lo, ksplit, alpha=1.0):
    """linear_presplit for few output tiles and a very long contraction: K cut into `ksplit` slices computed by different
    CTAs of the persistent kernel and summed in fixed order (mvm_linear_tc_presplit_splitk)."""
    lib = _lib.lib()
    M, K = a.shape
    N = w_hi.shape[0]
    out = torch.empty(M, N, dtype=torch.float32, device=a.device)
    ws = torch.empty(ksplit * M * N, dtype=torch.float32, device=a.device)
    _lib.check(lib.mvm_linear_tc_presplit_splitk(_lib.ptr(a), a.stride(0), _lib.ptr(w_hi), _lib.ptr(w_lo), w_hi.stride(0),
                                                 _lib.ptr(out), N, M, N, K, float(alpha), int(ksplit), _lib.ptr(ws),
                                                 _lib.stream_ptr()), 'mvm_linear_tc_presplit_splitk')
    return out


def gemm_dx(dy, w, residual=None, alpha=1.0):
    """Gradient w.r.t. the input of y = x @ w^T: dy [M, N_out] @ w [N_out, K_in] (+ residual) -> [M, K_in]."""
    n_out, k_in = w.shape
    w = w.detach().float().contiguous()
    if k_in % 128 == 0 and n_out % 32 == 0:
        _, hi, lo = transpose_split(w)
        return linear_presplit(dy, hi, lo, residual=residual, alpha=alpha)
    wt, _, _ = transpose_split(w, raw=True, planes=False)
    return linear(dy, wt, residual=residual, alpha=alpha, tc_passes=0)


def gemm_dw(dy, x, x2=None, alpha=1.0):
    """Gradient w.r.t. the weight of y = [x | x2] @ w^T: dy^T [N_out, rows] @ [x | x2] [rows, K_in] -> [N_out, K_in]."""
    rows, n_out = dy.shape
    k1 = x.shape[1]
    k_in = k1 + (x2.shape[1] if x2 is not None else 0)
    dyt, _, _ = transpose_split(dy, raw=True, planes=False)
    tc = k_in % 128 == 0 and rows % 32 == 0
    dev = dy.device
    if tc:
        hi = torch.empty(k_in, rows, dtype=torch.float32, device=dev)
        lo = torch.empty(k_in, rows, dtype=torch.float32, device=dev)
        transpose_split(x, out=(None, hi[:k1], lo[:k1]))
        if x2 is not None:
            transpose_split(x2, out=(None, hi[k1:], lo[k1:]))
        # few output tiles, a very long contraction: cut K = rows into slices for different CTAs (split-K)
        tiles = (n_out // 128) * (k_in // 128) if n_out % 128 == 0 else 0
        kb = rows // 32
        # (the CPU stand-ins of the tests take the split of the GPU they run beside; 132 = H100 SXM without one)
        n_sm = torch.cuda.get_device_properties(dev if dev.type == 'cuda' else torch.cuda.current_device()).multi_processor_count \
            if torch.cuda.is_available() else 132
        ks = max([s_ for s_ in range(1, 65) if kb % s_ == 0 and kb // s_ >= 8 and tiles * s_ <= n_sm] or [1]) if tiles else 1
        if ks >= 2:
            return linear_presplit_splitk(dyt, hi, lo, ks, alpha=alpha)
        return linear_presplit(dyt, hi, lo, alpha=alpha)
    xt = torch.empty(k_in, rows, dtype=torch.float32, device=dev)
    transpose_split(x, out=(xt[:k1], None, None))
    if x2 is not None:
        transpose_split(x2, out=(xt[k1:], None, None))
    return linear(dyt, xt, alpha=alpha, tc_passes=0)


def colsum(x):
    """x [rows, C] -> [C] column sums (bias gradient)."""
    lib = _lib.lib()
    rows, Cc = x.shape
    out = torch.empty(Cc, dtype=torch.float32, device=x.device)
    ws = torch.empty(Cc, dtype=torch.float64, device=x.device)
    _lib.check(lib.mvm_colsum(_lib.ptr(x), rows, Cc, x.stride(0), _lib.ptr(out), 0, _lib.ptr(ws), _lib.stream_ptr()),
               'mvm_colsum')
    return out


def batchnorm_train(x, weight, bias, running_mean, running_var, momentum, eps, n_pad, n_valid, relu=True, groups=1,
                    out=None, save=False):
    """BatchNorm1d (+ReLU) in training mode on x [rows, C] -> (out (default: in place), stats [groups, 2C] or None)."""
    lib = _lib.lib()
    rows, Cc = x.shape
    assert x.is_contiguous()
    y = x if out is None else out
    stats = torch.empty(groups, 2 * Cc, dtype=torch.float32, device=x.device) if save else None
    ws = torch.empty(3 * Cc, dtype=torch.float64, device=x.device)
    for g in range(groups):
        _lib.check(lib.mvm_batchnorm_train(_lib.ptr(x), _lib.ptr(y), rows, Cc, x.stride(0), n_pad, n_valid, groups, g,
                                           _lib.ptr(weight), _lib.ptr(bias), float(eps), int(relu), _lib.ptr(running_mean),
                                           _lib.ptr(running_var), float(momentum),
                                           _lib.ptr(stats[g]) if save else None, _lib.ptr(ws), _lib.stream_ptr()),
                   'mvm_batchnorm_train')
    return y, stats


def batchnorm_train_backward(x, y, dy, weight, stats, n_pad, n_valid, relu=True):
    """In place on dy (gradient w.r.t. y -> gradient w.r.t. x); -> (dgamma, dbeta)."""
    lib = _lib.lib()
    rows, Cc = x.shape
    groups = stats.shape[0]
    dg = torch.empty(Cc, dtype=torch.float32, device=x.device)
    db = torch.empty(Cc, dtype=torch.float32, device=x.device)
    ws = torch.empty(2 * Cc, dtype=torch.float64, device=x.device)
    assert x.is_contiguous() and dy.is_contiguous() and y.is_contiguous()
    for g in range(groups):
        _lib.check(lib.mvm_batchnorm_train_backward(_lib.ptr(x), _lib.ptr(y), _lib.ptr(dy), rows, Cc, x.stride(0), n_pad,
                                                    n_valid, groups, g, _lib.ptr(weight), _lib.ptr(stats[g]), int(relu),
                                                    _lib.ptr(dg), _lib.ptr(db), int(g > 0), _lib.ptr(ws),
                                                    _lib.stream_ptr()), 'mvm_batchnorm_train_backward')
    return dg, db


def attention_backward(qkv, out, dout, batch, n_views, counts, is_cross):
    """qkv [V, n_pad, 768], out / dout [V, n_pad, 256] -> dqkv [V, n_pad, 768] (mvm_attention_backward)."""
    lib = _lib.lib()
    V, n_pad, _ = qkv.shape
    dqkv = torch.empty_like(qkv)
    ws = torch.empty(2 * V * 4 * n_pad, dtype=torch.float32, device=qkv.device)
    cnt = (C.c_int * n_views)(*counts)
    assert qkv.is_contiguous() and out.is_contiguous() and dout.is_contiguous()
    _lib.check(lib.mvm_attention_backward(_lib.ptr(qkv), _lib.ptr(out), _lib.ptr(dout), _lib.ptr(dqkv), _lib.ptr(ws), batch,
                                          n_views, n_pad, cnt, int(is_cross), _lib.stream_ptr()), 'mvm_attention_backward')
    return dqkv


def pair_scores(md, pairs, N, alpha=1.0 / 16.0):
    """md [B, T, n_pad, 256] matching descriptors, pairs [(slot a, slot b)] -> score buffers [P * B, N + 1, N + 1] whose
    inner blocks hold md_a md_b^T * alpha (pair-major; the dustbin row / column are left unset): one launch of the
    tensor-core GEMM's score mode (mvm_pair_scores)."""
    lib = _lib.lib()
    B, T, n_pad, _ = md.shape
    P = len(pairs)
    assert md.is_contiguous()
    out = torch.empty(P * B, N + 1, N + 1, dtype=torch.float32, device=md.device)
    hi, lo = torch.empty_like(md), torch.empty_like(md)
    I = C.c_int * P
    ptrs = (C.c_void_p * P)(*[out[p * B].data_ptr() for p in range(P)])
    _lib.check(lib.mvm_pair_scores(_lib.ptr(md), _lib.ptr(hi), _lib.ptr(lo), B, T, n_pad, P, I(*[a for a, _ in pairs]),
                                   I(*[b for _, b in pairs]), I(*([N] * P)), I(*([N] * P)), ptrs, float(alpha),
                                   _lib.stream_ptr()), 'mvm_pair_scores')
    return out


def _sk_layout(scores, augmented):
    B, r, c = scores.shape
    m, n = (r - 1, c - 1) if augmented else (r, c)
    return B, m, n, c, r * c


def sinkhorn_train_forward(scores, alpha, iters, augmented=False):
    """scores [B, m, n] (or, augmented, the [B, m+1, n+1] buffers of pair_scores whose inner blocks hold the scores),
    alpha: device scalar tensor -> (couplings [B, m+1, n+1], potentials of every iteration)."""
    lib = _lib.lib()
    B, m, n, ld, stride = _sk_layout(scores, augmented)
    assert scores.is_contiguous() and alpha.dtype == torch.float32 and alpha.device == scores.device
    Z = torch.empty(B, m + 1, n + 1, dtype=torch.float32, device=scores.device)
    pot = torch.empty(lib.mvm_sinkhorn_train_pot_floats(B, m, n, iters), dtype=torch.float32, device=scores.device)
    _lib.check(lib.mvm_sinkhorn_train_forward(_lib.ptr(scores), ld, stride, _lib.ptr(alpha), B, m, n, int(iters), _lib.ptr(Z),
                                              _lib.ptr(pot), _lib.stream_ptr()), 'mvm_sinkhorn_train_forward')
    return Z, pot


def sinkhorn_train_backward(scores, alpha, pot, iters, grad_out, augmented=False):
    """-> (dZ [B, m+1, n+1]: gradient w.r.t. the augmented score matrix, d_alpha: [1] float64)."""
    lib = _lib.lib()
    B, m, n, ld, stride = _sk_layout(scores, augmented)
    dZ = grad_out.detach().float().contiguous().clone()
    d_alpha = torch.zeros(1, dtype=torch.float64, device=scores.device)
    _lib.check(lib.mvm_sinkhorn_train_backward(_lib.ptr(scores), ld, stride, _lib.ptr(alpha), _lib.ptr(pot), B, m, n,
                                               int(iters), _lib.ptr(dZ), _lib.ptr(d_alpha), _lib.stream_ptr()),
               'mvm_sinkhorn_train_backward')
    return dZ, d_alpha
