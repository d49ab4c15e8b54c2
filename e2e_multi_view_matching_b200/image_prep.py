"""Training-image preparation on the GPU: the per-image transforms of MatchingDataset.__getitem__
(datasets/matching_dataset.py:156-213) moved out of the DataLoader workers.

The workers then only decode the JPEG (uint8 RGB, HWC) and read the depth map, and hand over the tuple's crop offsets
and jitter parameters; prepare_tuple_batch turns the collated batch into exactly the dict __getitem__ + collate would
have produced: image{i} [B, 1, H, W] float32 on the device (mvm_image_prep, csrc/image_prep.cu), intr{i} adjusted
for the crop, the ScanNet pad and the resize, depth{i} cropped.

  * color_jitter_params: get_color_jitter_params (:125-130) -> ColorJitter.get_params, the same torch RNG calls in the
    same order, so a seeded generator gives the reference's parameters;
  * square_crop_window: the window rule of crop() (:132-154), centred or at an offset the caller drew;
  * crop_intrinsics / pad_intrinsics / resize_intrinsics: the bookkeeping of :14-23, :151, :192-201 in float32;
  * prepare_images: the kernel's Python face for a batch of one source size;
  * prepare_tuple_batch: the collated-batch entry point.
"""
import numpy as np
import torch

from . import _lib

# fn_idx values of ColorJitter.get_params
BRIGHTNESS, CONTRAST, SATURATION, HUE = 0, 1, 2, 3
# ScanNet colour images of this size get two zero rows above and below before the resize (:192-195)
SCANNET_PADDED_SIZE = (968, 1296)
SCANNET_PAD_ROWS = 2


def color_jitter_params(jitter, generator=None):
    """-> (fn_idx int64 [4], brightness, contrast, saturation, hue) as MatchingDataset.get_color_jitter_params draws
    them: torch.randperm(4), then one uniform_ per factor over (1 - jitter, 1 + jitter) and, for hue, (-jitter, jitter).
    With generator=None the global torch RNG is used, as the reference does."""
    lo, hi = 1. - jitter, 1. + jitter
    fn_idx = torch.randperm(4, generator=generator)

    def draw(a, b):
        return float(torch.empty(1).uniform_(a, b, generator=generator))

    b = draw(lo, hi)
    c = draw(lo, hi)
    s = draw(lo, hi)
    h = draw(-jitter, jitter)
    return fn_idx, b, c, s, h


def square_crop_window(height, width, offset=None):
    """crop() (:132-154) on a depth map of height x width: the largest square, centred along the longer side when
    offset is None (the test split), else starting at `offset` (the reference draws np.random.randint(0, |w - h| + 1)).
    -> (top, left, size, size)."""
    height, width = int(height), int(width)
    span = abs(width - height)
    if offset is None:
        offset = int(span / 2.)
    elif not 0 <= int(offset) <= span:
        raise ValueError('crop offset %s outside [0, %d]' % (offset, span))
    offset = int(offset)
    if width > height:
        return 0, offset, height, height
    return offset, 0, width, width


def crop_intrinsics(K, crop_x, crop_y):
    """crop_intrinsics (:21-24) in place on K [..., 3|4, 3|4] (numpy or torch, float32); crop_x, crop_y scalars or
    per-batch arrays."""
    K[..., 0, 2] -= crop_x
    K[..., 1, 2] -= crop_y
    return K


def pad_intrinsics(K, rows=SCANNET_PAD_ROWS):
    """The ScanNet pad's principal-point shift (:195): cy + rows."""
    K[..., 1, 2] += rows
    return K


def resize_intrinsics(K, fact_x, fact_y):
    """resize_intrinsics (:14-19) in place; fact_x, fact_y Python floats (out / in), rounded to float32 by the
    multiply as numpy does for a float32 K."""
    K[..., 0, 0] *= fact_x
    K[..., 1, 1] *= fact_y
    K[..., 0, 2] *= fact_x
    K[..., 1, 2] *= fact_y
    return K


def _host(x, dtype):
    if isinstance(x, torch.Tensor):
        if x.is_cuda:
            raise ValueError('image preparation parameters are checked on the host: pass CPU tensors or arrays')
        x = x.numpy()
    return np.ascontiguousarray(np.asarray(x), dtype=dtype)


def check_params(src_size, geometry, out_size, jitter_order=None, jitter_factors=None):
    """Refuse what torchvision or the shapes would refuse, before any launch.  -> (geometry int32 [n, 6],
    order int32 [n, 4] | None, factors float64 [n, 4] | None) as host arrays."""
    src_h, src_w = (int(v) for v in src_size)
    out_h, out_w = (int(v) for v in out_size)
    if out_h < 1 or out_w < 1:
        raise ValueError('output size %s below 1' % ((out_h, out_w),))
    g = _host(geometry, np.int64).reshape(-1, 6)
    top, left, ch, cw, pt, pb = g.T
    bad = (top < 0) | (left < 0) | (ch < 1) | (cw < 1) | (top + ch > src_h) | (left + cw > src_w) | (pt < 0) | (pb < 0)
    if bad.any():
        raise ValueError('crop window %s outside the %d x %d source (or a negative pad)'
                         % (g[np.argmax(bad)].tolist(), src_h, src_w))
    if (jitter_order is None) != (jitter_factors is None):
        raise ValueError('jitter needs both the order and the factors')
    if jitter_order is None:
        return g.astype(np.int32), None, None
    order = _host(jitter_order, np.int64).reshape(-1, 4)
    fac = _host(jitter_factors, np.float64).reshape(-1, 4)
    if len(order) != len(g) or len(fac) != len(g):
        raise ValueError('one jitter order and one set of factors per image')
    if not (np.sort(order, axis=1) == np.arange(4)).all():
        raise ValueError('jitter order is not a permutation of 0-3')
    for k, name in ((BRIGHTNESS, 'brightness'), (CONTRAST, 'contrast'), (SATURATION, 'saturation')):
        if (fac[:, k] < 0).any():
            raise ValueError('%s_factor (%s) is not non-negative.' % (name, fac[np.argmax(fac[:, k] < 0), k]))
    h = fac[:, HUE]
    if not ((-0.5 <= h) & (h <= 0.5)).all():
        raise ValueError('hue_factor (%s) is not in [-0.5, 0.5].' % h[np.argmax(~((-0.5 <= h) & (h <= 0.5)))])
    return g.astype(np.int32), order.astype(np.int32), fac


def prepare_images(rgb, geometry, out_size, jitter_order=None, jitter_factors=None, device=None):
    """rgb [n, H, W, 3] uint8 (CPU, ideally pinned, or CUDA) -> [n, 1, out_h, out_w] float32 on the device: ToTensor,
    crop, zero-row pad, bilinear resize when the size changes, ColorJitter in the given order, rgb_to_grayscale.
    geometry [n, 6]: crop top, left, height, width, pad rows above, below; jitter_order [n, 4] a permutation of
    0-3 (BRIGHTNESS, CONTRAST, SATURATION, HUE) and jitter_factors [n, 4] (in that order), or both None."""
    if not isinstance(rgb, torch.Tensor):
        rgb = torch.from_numpy(np.asarray(rgb))
    if rgb.dtype != torch.uint8 or rgb.dim() != 4 or rgb.shape[3] != 3:
        raise ValueError('rgb must be uint8 [n, H, W, 3], got %s %s' % (rgb.dtype, tuple(rgb.shape)))
    n, src_h, src_w = rgb.shape[:3]
    g, order, fac = check_params((src_h, src_w), geometry, out_size, jitter_order, jitter_factors)
    if len(g) != n:
        raise ValueError('one geometry row per image: %d rows for %d images' % (len(g), n))
    device = torch.device(device) if device is not None else (rgb.device if rgb.is_cuda else torch.device('cuda'))
    _lib.require_cuda(device, 'prepare_images')
    out_h, out_w = (int(v) for v in out_size)
    L = _lib.lib()
    with _lib.device_ctx(device):
        src = rgb.to(device, non_blocking=True).contiguous()
        up = lambda a: torch.from_numpy(a).to(device, non_blocking=True)   # noqa: E731
        g_d = up(g)
        o_d = up(order) if order is not None else None
        f_d = up(fac) if fac is not None else None
        out = torch.empty(n, 1, out_h, out_w, dtype=torch.float32, device=device)
        ws = None
        if o_d is not None:
            ws = torch.empty(L.mvm_image_prep_workspace_bytes(n, out_h, out_w), dtype=torch.uint8, device=device)
        _lib.check(L.mvm_image_prep(_lib.ptr(src), n, src_h, src_w, _lib.ptr(g_d), _lib.ptr(o_d), _lib.ptr(f_d),
                                    out_h, out_w, _lib.ptr(out), _lib.ptr(ws), 0 if ws is None else ws.numel(),
                                    _lib.stream_ptr()), 'mvm_image_prep')
    return out


def _view_ids(data):
    return sorted(int(k[3:]) for k in data if k.startswith('rgb') and k[3:].isdigit())


def prepare_tuple_batch(data, device=None):
    """A collated batch whose dataset returned, per view i, decoded rgb{i} ([B, H, W, 3] uint8), depth{i} [B, h, w],
    intr{i} [B, 3|4, 3|4] float32 and, for MegaDepth, crop{i} [B] (the square crop's offset along the longer side,
    square_crop_window), plus once per tuple jitter_order [B, 4] and jitter_factors [B, 4] (brightness, contrast,
    saturation, hue; both absent without jitter) -> the same dict with image{i} [B, 1, h', w'] float32 on the device,
    intr{i} adjusted and depth{i} cropped, as MatchingDataset.__getitem__ + collate would have produced it.  The
    rgb / crop / jitter keys are consumed.  A batch without rgb{i} (it already carries image{i}) is returned as is.
    All views of one source size and output size go through one mvm_image_prep call."""
    views = _view_ids(data)
    if not views:
        return data
    device = torch.device(device) if device is not None else torch.device('cuda')
    order = data.pop('jitter_order', None)
    factors = data.pop('jitter_factors', None)
    groups = {}
    for i in views:
        rgb = data.pop('rgb%d' % i)
        if not isinstance(rgb, torch.Tensor):
            rgb = torch.as_tensor(np.asarray(rgb))
        B, H, W = rgb.shape[:3]
        depth = data['depth%d' % i]
        K = data['intr%d' % i]
        crop = data.pop('crop%d' % i, None)
        h, w = depth.shape[-2:]
        if crop is not None:
            wins = [square_crop_window(h, w, int(c)) for c in np.asarray(crop).reshape(-1)]
            if len(wins) != B:
                raise ValueError('crop%d holds %d offsets for a batch of %d' % (i, len(wins), B))
            tops = np.array([t for t, _, _, _ in wins])
            lefts = np.array([lf for _, lf, _, _ in wins])
            s = wins[0][2]
            crop_intrinsics(K, _like(K, lefts), _like(K, tops))
            data['depth%d' % i] = _stack([depth[b, t:t + s, lf:lf + s] for b, (t, lf, _, _) in enumerate(wins)],
                                         depth)
            ch = cw = s
        else:
            tops = lefts = np.zeros(B, np.int64)
            ch, cw = H, W
        pad = SCANNET_PAD_ROWS if (ch, cw) == SCANNET_PADDED_SIZE else 0
        if pad:
            pad_intrinsics(K, pad)
        out_h, out_w = data['depth%d' % i].shape[-2:]
        in_h = ch + 2 * pad
        if (out_h, out_w) != (in_h, cw):
            resize_intrinsics(K, out_w / cw, out_h / in_h)
        geom = np.stack([tops, lefts, np.full(B, ch), np.full(B, cw), np.full(B, pad), np.full(B, pad)], 1)
        groups.setdefault((H, W, out_h, out_w), []).append((i, rgb, geom))
    for (H, W, out_h, out_w), members in groups.items():
        rgb = torch.cat([m[1] for m in members], 0)
        if rgb.device.type == 'cpu' and torch.cuda.is_available() and not rgb.is_pinned():
            rgb = rgb.pin_memory()
        geom = np.concatenate([m[2] for m in members], 0)
        jo = jf = None
        if order is not None:
            jo = _host(order, np.int64).reshape(-1, 4)
            jf = _host(factors, np.float64).reshape(-1, 4)
            jo, jf = np.tile(jo, (len(members), 1)), np.tile(jf, (len(members), 1))
        out = prepare_images(rgb, geom, (out_h, out_w), jo, jf, device=device)
        B = members[0][1].shape[0]
        for k, (i, _, _) in enumerate(members):
            data['image%d' % i] = out[k * B:(k + 1) * B]
    return data


def _like(K, a):
    return torch.as_tensor(a, device=K.device) if isinstance(K, torch.Tensor) else a


def _stack(parts, like):
    return torch.stack(parts) if isinstance(like, torch.Tensor) else np.stack(parts)
