"""The SuperPoint front end (csrc/superpoint.cu: mvm_superpoint_dense / _sample / _sample_batch) against the float64
restatement of oracle/superpoint.py, over the whole dense maps, at the shapes and inputs where its kernels have edges.

Sizes, as H x W with the four resolutions H, H/2, H/4, H/8 (floored) that the convolutions run at:
  - sp_conv3x3_kernel tiles 16 x 16 pixels (TP) per CTA, partial tiles where a side is not a multiple of 16, with a
      zero halo at the image edge; 32 output channels per CTA (OCB); input channels in slices of 16 (ICS), one
      partial slice for conv1a (Cin = 1); one image per blockIdx.z:
      16x16 (16, 8, 4, 2: one full tile, then below one tile; the smallest image the API takes),
      17x23 / 23x17 (17, 8, 4, 2 and 23, 11, 5, 2: one pixel past a tile, then odd pool inputs),
      31x33 / 33x31 (31, 15, 7, 3 and 33, 16, 8, 4: one short of two tiles, one past; 16 exactly at H/2),
      129x255 / 255x129 (129, 64, 32, 16 and 255, 127, 63, 31: a one-pixel tile row, then whole tiles; one short),
      135x271 / 271x135 (135, 67, 33, 16 and 271, 135, 67, 33: odd at three levels),
      71x101 (71, 35, 17, 8 and 101, 50, 25, 12), 256x256, and the production 480x640 at B = 40 (the cfg5 training
      batch: 40 x 60 x 80 = 192000 convDb GEMM rows) and 1066x1600 at B = 1 (133 x 200 cells);
  - sp_maxpool2_kernel floors odd sides (the last row / column is dropped) with the input's W as the row stride: every
      odd entry above;
  - the last H % 8 rows and W % 8 columns get no score but feed conv1a / conv1b through the halo before the first pool:
      the 'tail' content is zero except there (17x23, 23x17, 31x33, 33x31, 129x255, 135x271, 271x135, 71x101);
  - sp_scores_kernel: 65-way softmax over lanes (bins lane and lane + 32, bin 64 on lane 0), dustbin dropped,
      depth-to-space; weights with logit gain 3 (the fixtures' default), 30 (the softmax saturates: exact-zero
      scores) and 0.1 (every score near 1/65, a map of near-ties);
  - sp_maxrow / sp_maxcol + sp_nms_*: separable (2r+1)^2 max filter with -inf padding, three-round suppression, exact
      `==`: r = 0 (the identity), 1, 2, 4, 8 on every case but the production ones (r = 4 there), and on the maps of at
      most 64 x 64 a radius larger than the map; constant images (0, 0.5, 1 at 256x256, so that interior cells lie
      outside the zero padding's receptive field) give plateaus of identical bits;
  - sp_l2norm_kernel and convDb on the 3xTF32 GEMM: M = B h w rows, from 4 to 192000;
  - sp_sample_point: grid_sample with align_corners=True and zero padding, keypoints within 4 pixels of an edge mix in
      a zero neighbour; h != w on every non-square map; sp_sample_batch_kernel zeroes the columns past counts[b].
Batches of 3 or 5 hold different images (make_image, constants, a texture with a constant block, a 0/1 checkerboard,
iid noise, the tail content), so that a halo or pool read that crosses into the next image shows.

Checks:
  1. the raw score map (nms_radius = 0: the suppression keeps every pixel, in the kernels as in the restatement) over
     the whole map against float64, within 3 x the float32 restatement's own deviation on the case + 4 ulp of the map
     maximum;
  2. for r > 0, the NMS'd map bit for bit against the restatement's simple_nms run in float32 on the kernel's own raw
     map (max and == are exact, so any difference is a kernel error; a float64 map would not have the kernel's
     plateaus), every kept value the raw value's bits, and the dense descriptors the bits of the r = 0 call;
  3. the dense descriptors [B, h, w, 256] against float64 with the bound of check 1 (4 ulp of 1 as the floor), and unit
     norm per pixel within 2^-20;
  4. mvm_superpoint_sample and _sample_batch on the kernel's own dense map against the restatement's sample in float64
     at every integer position of maps of 2x2 to 4x4 cells, and elsewhere at the corners, the first and last four rows
     and columns, random interior points, the random fill range [12, 8h - 12) and fractional positions.  The bound per
     channel is derived from the kernel's float32 arithmetic: 16 ulp of 1 for the rounding of the bilinear sum and the
     normalisation, plus the grid coordinate's rounding (8 ulp of w, resp. h, in cell units) times the bilinear slope
     of the channel, both carried through the normalisation.  _sample_batch equals _sample bit for bit; counts 0, 1,
     K - 1, K with K = 37 leave exact zeros past the count;
  5. forward_batch at the cfg5 config (nms_radius 4, threshold 0.001, K = 400, border 12, with and without fill) on the
     480x640 batch: descriptors at the keypoints it selected against the float64 pipeline sampled there, within 3 x the
     float32 restatement's deviation + the sampling bound of check 4; scores the raw map's bits;
  6. every image of a B = 5 batch gives the bits it gets alone: raw map, NMS map, descriptors (each pixel's arithmetic
     does not depend on the batch; convDb runs on 128-row tiles without split-K, so a row's sum does not depend on M).

Every case prints its largest error and its bound.  On an H100 80GB HBM3 at a 700 W power limit the largest share of
bound was, per check: 1. raw scores 0.59 (const256; 0.50 at 255x129, where the softmax saturates); 2. NMS bit for
bit at every radius, no pixel differs; 3. dense descriptors 0.42 (23x17); 4. sampling 0.11 (1066x1600, where the
coordinate term of the 200-cell rows dominates; 0.02 on the maps of 2x2 to 4x4 cells); 5. forward_batch 0.13;
6. bit for bit.  The file runs in about 40 s there, most of it the float64 restatement on the CPU.
"""
import functools

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
D, F32 = torch.float64, torch.float32
U = 2.0 ** -24


class Case:
    def __init__(self, name, H, W, content, gain=3.0, wseed=0, radii=(1, 2, 4, 8), f64=None):
        self.name, self.H, self.W, self.content, self.gain, self.wseed = name, H, W, content, gain, wseed
        self.B = len(content)
        self.h, self.w = H // 8, W // 8
        big = max(8 * self.h, 8 * self.w) + 1
        self.radii = tuple(radii) + ((big,) if max(8 * self.h, 8 * self.w) <= 64 and radii else ())
        self.f64 = tuple(range(self.B)) if f64 is None else f64      # the images compared with float64

    def __repr__(self):
        return self.name


CASES = [
    Case('16x16', 16, 16, ['make', 'noise', 'checker']),
    Case('17x23', 17, 23, ['make', 'tail', 'noise']),
    Case('23x17', 23, 17, ['tail', 'make', 'checker'], gain=30.0),
    Case('31x33_b5', 31, 33, ['make', 'noise', 'block', 'checker', 'tail'], gain=30.0),
    Case('33x31', 33, 31, ['make', 'tail', 'noise'], gain=0.1),
    Case('129x255', 129, 255, ['make', 'block', 'tail']),
    Case('255x129', 255, 129, ['make', 'noise', 'checker'], gain=30.0),
    Case('135x271', 135, 271, ['make', 'tail', 'block'], gain=0.1),
    Case('271x135', 271, 135, ['noise', 'make', 'tail'], wseed=1),
    Case('71x101_b5', 71, 101, ['block', 'checker', 'noise', 'tail', 'make'], wseed=1),
    Case('const256', 256, 256, ['const0', 'const0.5', 'const1']),
    Case('const256_g01', 256, 256, ['const0.5', 'const1', 'make'], gain=0.1),
    Case('480x640_b40', 480, 640, ['make'] * 40, wseed=1, radii=(4,), f64=(0, 39)),
    Case('1066x1600', 1066, 1600, ['make'], radii=(4,)),
]
BY_NAME = {c.name: c for c in CASES}
BATCH5 = [c for c in CASES if c.B == 5]


def _content(kind, seed, H, W):
    from e2e_multi_view_matching_b200.synthetic import make_image
    rng = np.random.default_rng(1000 + seed)
    if kind == 'make':
        return make_image(seed, H, W)[0, 0]
    if kind.startswith('const'):
        return np.full((H, W), float(kind[5:]), np.float32)
    if kind == 'block':                          # texture with a constant block
        img = make_image(seed, H, W)[0, 0].copy()
        img[H // 4:(3 * H) // 4, W // 5:W // 2] = 0.3
        return img
    if kind == 'checker':
        yy, xx = np.mgrid[0:H, 0:W]
        return ((yy + xx) % 2).astype(np.float32)
    if kind == 'noise':
        return rng.random((H, W), dtype=np.float32)
    if kind == 'tail':                           # content only in the rows and columns that get no score
        img = np.zeros((H, W), np.float32)
        img[H - H % 8:, :] = rng.random((H % 8, W), dtype=np.float32)
        img[:, W - W % 8:] = rng.random((H, W % 8), dtype=np.float32)
        return img
    raise ValueError(kind)


@functools.lru_cache(None)
def _images(name):
    c = BY_NAME[name]
    return np.stack([_content(k, i, c.H, c.W) for i, k in enumerate(c.content)])[:, None]     # [B, 1, H, W]


@functools.lru_cache(None)
def _state_dict(wseed, gain):
    from e2e_multi_view_matching_b200.synthetic import make_superpoint_state_dict
    return make_superpoint_state_dict(wseed, logit_gain=gain)


def _model(c, **cfg):
    from e2e_multi_view_matching_b200.models.superpoint import SuperPoint
    sp = SuperPoint(cfg).eval()
    sp.load_state_dict({k: torch.from_numpy(v) for k, v in _state_dict(c.wseed, c.gain).items()}, strict=True)
    return sp.cuda()


@functools.lru_cache(8)
def _kernel(name, r):
    """(scores after NMS of radius r [B, 8h, 8w], dense descriptors [B, h, w, 256]) from the kernels."""
    c = BY_NAME[name]
    out = _model(c, nms_radius=r).dense(torch.from_numpy(_images(name)).cuda())
    torch.cuda.synchronize()
    return out


@functools.lru_cache(None)
def _oracle(name, dtype):
    """(raw scores, dense descriptors) of the restatement in dtype, on the CPU, for the images c.f64."""
    from oracle.superpoint import dense
    c = BY_NAME[name]
    raw, _, desc = dense(_images(name)[list(c.f64)], _state_dict(c.wseed, c.gain), 0, dtype)
    return raw.double(), desc.double()


def _bits(t):
    return t.contiguous().view(torch.int32)


def _report(what, c, err, bound):
    print('%-10s %-14s err %.3e  bound %.3e  share %.3f' % (what, c.name, err, bound, err / bound))


@pytest.mark.parametrize('c', CASES, ids=repr)
def test_raw_scores_vs_float64(c):
    raw_k, dense_k = _kernel(c.name, 0)
    assert raw_k.shape == (c.B, 8 * c.h, 8 * c.w) and dense_k.shape == (c.B, c.h, c.w, 256)
    raw64, _ = _oracle(c.name, D)
    raw32, _ = _oracle(c.name, F32)
    got = raw_k[list(c.f64)].cpu().double()
    bound = 3 * float((raw32 - raw64).abs().max()) + 4 * U * float(raw64.abs().max())
    err = float((got - raw64).abs().max())
    _report('scores', c, err, bound)
    assert err <= bound
    if c.name == '255x129':                              # gain 30: the softmax underflows to exact zeros
        assert int((raw_k == 0).sum()) > 0


@pytest.mark.parametrize('c', CASES, ids=repr)
def test_nms_bitwise(c):
    from oracle.superpoint import simple_nms
    raw_k, dense_k = _kernel(c.name, 0)
    for r in c.radii:
        nms_k, dense_r = _kernel(c.name, r)
        ref = simple_nms(raw_k, r)                      # float32, on the kernel's own map: max and == are exact
        bad = int((_bits(nms_k) != _bits(ref)).sum())
        kept = nms_k != 0
        print('nms        %-14s r = %4d: %d of %d kept, %d differ' % (c.name, r, int(kept.sum()), nms_k.numel(), bad))
        assert bad == 0
        assert torch.equal(_bits(nms_k[kept]), _bits(raw_k[kept]))
        assert torch.equal(_bits(dense_r), _bits(dense_k))


@pytest.mark.parametrize('c', CASES, ids=repr)
def test_dense_descriptors_vs_float64(c):
    _, dense_k = _kernel(c.name, 0)
    _, d64 = _oracle(c.name, D)
    _, d32 = _oracle(c.name, F32)
    got = dense_k[list(c.f64)].cpu().double()
    bound = 3 * float((d32 - d64).abs().max()) + 4 * U
    err = float((got - d64).abs().max())
    _report('dense', c, err, bound)
    assert err <= bound
    norm_err = float((dense_k.double().norm(dim=-1) - 1).abs().max())
    assert norm_err <= 2.0 ** -20, norm_err


# ---- sampling -------------------------------------------------------------------------------------------------------

def _sample_kernel(dense_b, kp):
    from e2e_multi_view_matching_b200 import _lib
    n = kp.shape[0]
    out = torch.full((256, n), float('nan'), device='cuda')
    rc = _lib.lib().mvm_superpoint_sample(_lib.ptr(dense_b.contiguous()), _lib.ptr(kp), n, dense_b.shape[0],
                                          dense_b.shape[1], _lib.ptr(out), _lib.stream_ptr())
    _lib.check(rc, 'mvm_superpoint_sample')
    return out


def _sample_batch_kernel(dense, kp, counts):
    from e2e_multi_view_matching_b200 import _lib
    B, K, _ = kp.shape
    out = torch.full((B, 256, K), float('nan'), device='cuda')
    cnt = torch.tensor(counts, dtype=torch.int32, device='cuda')
    rc = _lib.lib().mvm_superpoint_sample_batch(_lib.ptr(dense), _lib.ptr(kp.contiguous()), _lib.ptr(cnt), B, K,
                                                dense.shape[1], dense.shape[2], _lib.ptr(out), _lib.stream_ptr())
    _lib.check(rc, 'mvm_superpoint_sample_batch')
    return out


def _keypoints(h, w, seed):
    """[n, 2] float32 (x, y) pixel positions of the [8h, 8w] map: every integer one on maps of at most 4 x 4 cells;
    else the corners, the first and last four rows and columns, random interior points and random points of the
    fill range [12, 8h - 12); and fractional positions."""
    rng = np.random.default_rng(seed)
    Hs, Ws = 8 * h, 8 * w
    if h * w <= 16:
        ys, xs = np.mgrid[0:Hs, 0:Ws]
        pts = [np.stack([xs.ravel(), ys.ravel()], 1)]
    else:
        ex, ey = np.r_[0:4, Ws - 4:Ws], np.r_[0:4, Hs - 4:Hs]
        xs = np.unique(np.r_[ex, rng.integers(0, Ws, 64)])
        ys = np.unique(np.r_[ey, rng.integers(0, Hs, 64)])
        pts = [np.stack(np.meshgrid(xs, ey), -1).reshape(-1, 2), np.stack(np.meshgrid(ex, ys), -1).reshape(-1, 2),
               np.stack([rng.integers(4, Ws - 4, 256), rng.integers(4, Hs - 4, 256)], 1)]
        if Hs > 24 and Ws > 24:
            pts.append(np.stack([rng.integers(12, Ws - 12, 256), rng.integers(12, Hs - 12, 256)], 1))
    pts.append(np.stack([rng.uniform(0, Ws - 1, 32), rng.uniform(0, Hs - 1, 32)], 1))
    pts.append(np.array([[0.5, 0.25], [Ws - 1.25, Hs - 1.5], [3.75, Hs / 2 + 0.125], [Ws / 2 - 0.0625, 2.5]]))
    return torch.from_numpy(np.concatenate(pts).astype(np.float32))


def _sample_bound(dmap, kp):
    """Per-channel bound [256, n] of the kernel's sampling error on the float64 copy dmap [h, w, 256] of its own
    dense map, derived from sp_sample_point's float32 arithmetic: the grid coordinate fx = ((k - 3.5) / (8w - 4.5)
    * 2 - 1 + 1) / 2 * (w - 1) is rounded at most 8 ulp of w away (in cells) from its exact value, which moves the
    sample by that times the bilinear slope (the steepest of the cell and its two neighbours along the axis, zero
    padding included); the four weighted products and their sum round within 8 ulp of the sum of their magnitudes;
    the normalisation adds 16 ulp of 1."""
    h, w, C = dmap.shape
    P = torch.zeros(h + 4, w + 4, C, dtype=D)
    P[2:h + 2, 2:w + 2] = dmap
    k = kp.double()
    fx = (((k[:, 0] - 3.5) / (8 * w - 4.5)) * 2 - 1 + 1) / 2 * (w - 1)
    fy = (((k[:, 1] - 3.5) / (8 * h - 4.5)) * 2 - 1 + 1) / 2 * (h - 1)
    x0, y0 = torch.floor(fx).long(), torch.floor(fy).long()
    ax, ay = (fx - x0)[:, None], (fy - y0)[:, None]

    def at(yy, xx):
        return P[(yy + 2).clamp(0, h + 3), (xx + 2).clamp(0, w + 3)]                  # [n, C], zeros outside

    c00, c01, c10, c11 = at(y0, x0), at(y0, x0 + 1), at(y0 + 1, x0), at(y0 + 1, x0 + 1)
    v = c00 * (1 - ax) * (1 - ay) + c01 * ax * (1 - ay) + c10 * (1 - ax) * ay + c11 * ax * ay
    mag = (c00.abs() * (1 - ax) * (1 - ay) + c01.abs() * ax * (1 - ay) + c10.abs() * (1 - ax) * ay
           + c11.abs() * ax * ay)
    gx = torch.stack([((1 - ay) * (at(y0, x0 + d + 1) - at(y0, x0 + d)) + ay * (at(y0 + 1, x0 + d + 1)
                       - at(y0 + 1, x0 + d))).abs() for d in (-1, 0, 1)]).amax(0)
    gy = torch.stack([((1 - ax) * (at(y0 + d + 1, x0) - at(y0 + d, x0)) + ax * (at(y0 + d + 1, x0 + 1)
                       - at(y0 + d, x0 + 1))).abs() for d in (-1, 0, 1)]).amax(0)
    e = 8 * U * w * gx + 8 * U * h * gy + 8 * U * mag                              # [n, C]
    nv = v.norm(dim=1, keepdim=True)
    return (16 * U + e / nv + v.abs() / nv * e.norm(dim=1, keepdim=True) / nv).t()


SAMPLE_CASES = [c for c in CASES if c.B < 40]


@pytest.mark.parametrize('c', SAMPLE_CASES, ids=repr)
def test_sample_vs_float64(c):
    from oracle.superpoint import sample
    _, dense_k = _kernel(c.name, 0)
    worst = 0.0
    for b in range(c.B):
        kp = _keypoints(c.h, c.w, b)
        got = _sample_kernel(dense_k[b], kp.cuda())
        dmap = dense_k[b].cpu().double()
        ref = sample(dmap, kp.double())
        bound = _sample_bound(dmap, kp)
        err = (got.cpu().double() - ref).abs()
        share = float((err / bound).max())
        worst = max(worst, share)
        assert share <= 1, (b, float(err.max()))
        # the batch kernel: same bits where counted, exact zeros past the count
        K = 37
        sel = kp[torch.from_numpy(np.random.default_rng(b).choice(kp.shape[0], K * c.B))].reshape(c.B, K, 2)
        counts = [(0, 1, K - 1, K, K // 2)[(i + b) % 5] for i in range(c.B)]
        out = _sample_batch_kernel(dense_k, sel.cuda(), counts)
        full = _sample_batch_kernel(dense_k, sel.cuda(), [K] * c.B)
        for i in range(c.B):
            alone = _sample_kernel(dense_k[i], sel[i].cuda())
            assert torch.equal(_bits(full[i]), _bits(alone))
            n = counts[i]
            assert torch.equal(_bits(out[i, :, :n]), _bits(alone[:, :n]))
            assert bool((out[i, :, n:] == 0).all())
    print('sample     %-14s worst share of bound %.3f' % (c.name, worst))


# ---- end to end and batch invariance ----------------------------------------------------------------------------------

@pytest.mark.parametrize('fill', [False, True])
def test_forward_batch_cfg5_vs_float64(fill):
    from oracle.superpoint import sample
    c = BY_NAME['480x640_b40']
    cfg = dict(nms_radius=4, keypoint_threshold=0.001, max_keypoints=400, remove_borders=12,
               fill_with_random_keypoints=fill)
    torch.manual_seed(0)
    out = _model(c, **cfg).forward_batch(torch.from_numpy(_images(c.name)).cuda())
    raw_k, _ = _kernel(c.name, 0)
    _, d64 = _oracle(c.name, D)
    _, d32 = _oracle(c.name, F32)
    counts = out['counts'].cpu().tolist()
    if fill:
        assert counts == [400] * c.B
    worst = 0.0
    for j, b in enumerate(c.f64):
        n = counts[b]
        kp = out['keypoints'][b, :n].cpu()
        assert n > 0
        assert bool(((kp >= 12) & (kp < torch.tensor([8 * c.w - 12, 8 * c.h - 12]))).all())
        got = out['descriptors'][b, :, :n].cpu().double()
        ref = sample(d64[j], kp.double())
        dev32 = float((sample(d32[j], kp.float()).double() - ref).abs().max())
        bound = 3 * dev32 + _sample_bound(d64[j], kp)
        share = float(((got - ref).abs() / bound).max())
        worst = max(worst, share)
        assert share <= 1, (b, share)
        if not fill:
            sc = out['scores'][b, :n]
            xi, yi = kp[:, 0].long().cuda(), kp[:, 1].long().cuda()
            assert torch.equal(_bits(sc), _bits(raw_k[b, yi, xi].contiguous()))
    print('e2e        fill=%d worst share of bound %.3f' % (fill, worst))


@pytest.mark.parametrize('c', BATCH5, ids=repr)
def test_batch_invariance(c):
    imgs = torch.from_numpy(_images(c.name)).cuda()
    for r in (0, 4):
        nms_k, dense_k = _kernel(c.name, r)
        model = _model(c, nms_radius=r)
        for b in range(c.B):
            s1, d1 = model.dense(imgs[b:b + 1])
            assert torch.equal(_bits(s1[0]), _bits(nms_k[b])), (r, b)
            assert torch.equal(_bits(d1[0]), _bits(dense_k[b])), (r, b)
