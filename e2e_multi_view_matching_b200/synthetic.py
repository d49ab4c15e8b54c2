"""Seeded synthetic weights + inputs (SURVEY.md §8d) shared by bench.py, the tests and the
oracle.  Pure numpy so that the exact same tensors can be regenerated on the GPU box, where
/root/reference does not exist (there are no datasets or checkpoints offline).

State-dict keys and shapes follow the reference model
(models/models/multi_view_matcher.py:117-148, SURVEY.md appendix A.1):
  kenc.encoder.{0,3,6,9,12}  Conv1d 3->32->64->128->256->256, BN at {1,4,7,10}
  gnn.layers.{l}.attn.{proj.0,proj.1,proj.2,merge}  Conv1d 256->256
  gnn.layers.{l}.mlp.{0 (512->512), 1 (BN512), 3 (512->256, bias 0)}
  final_proj, bin_score, conf_mlp.{layers_f,layers_c,layers}
"""
import numpy as np

BN_EPS = 1e-5


def _conv(rng, out_c, in_c, zero_bias=False):
    bound = 1.0 / np.sqrt(in_c)
    w = rng.uniform(-bound, bound, size=(out_c, in_c, 1)).astype(np.float32)
    b = (np.zeros(out_c, np.float32) if zero_bias
         else rng.uniform(-bound, bound, size=(out_c,)).astype(np.float32))
    return w, b


def _bn(rng, c):
    return {
        'weight': rng.uniform(0.5, 1.5, size=(c,)).astype(np.float32),
        'bias': rng.uniform(-0.2, 0.2, size=(c,)).astype(np.float32),
        'running_mean': (0.1 * rng.standard_normal(c)).astype(np.float32),
        'running_var': rng.uniform(0.5, 1.5, size=(c,)).astype(np.float32),
        'num_batches_tracked': np.array(0, dtype=np.int64),
    }


def _put_conv(sd, key, w, b):
    sd[key + '.weight'] = w
    sd[key + '.bias'] = b


def _put_bn(sd, key, bn):
    for k, v in bn.items():
        sd[key + '.' + k] = v


def make_state_dict(n_layers, seed=0, conf_mlp=True, desc_dim=256,
                    kenc_layers=(32, 64, 128, 256), bin_score=1.0, final_proj_gain=1.0, residual_gain=1.0,
                    conf_head='random'):
    """Deterministic random state dict (numpy arrays) with the reference's keys.
    conf_head='score': instead of a random confidence head (whose output is noise, so the weighted eight-point
    sees every wrong match at full weight and the pose AUC is ~0), a 'trained-like' one: channel 0 of the
    layers_c path carries relu(s + 4) of the assignment log-score s of the match (multi_view_matcher.py:303-305)
    to the output, conf ~ sigmoid(2 relu(s + 4) - 6) -- 0.88 for a certain match, 0.5 at s = -1, ~0 below -3 --
    on top of a small random contribution of every other weight (all kernels stay exercised)."""
    rng = np.random.default_rng(seed)
    sd = {}
    sd['bin_score'] = np.array(bin_score, dtype=np.float32)
    ch = [3] + list(kenc_layers) + [desc_dim]
    for i in range(1, len(ch)):
        last = i == len(ch) - 1
        w, b = _conv(rng, ch[i], ch[i - 1], zero_bias=last)
        _put_conv(sd, 'kenc.encoder.%d' % (3 * (i - 1)), w, b)
        if not last:
            _put_bn(sd, 'kenc.encoder.%d' % (3 * (i - 1) + 1), _bn(rng, ch[i]))
    d = desc_dim
    for l in range(n_layers):
        p = 'gnn.layers.%d.' % l
        for name in ('attn.proj.0', 'attn.proj.1', 'attn.proj.2', 'attn.merge'):
            w, b = _conv(rng, d, d)
            _put_conv(sd, p + name, w, b)
        w, b = _conv(rng, 2 * d, 2 * d)
        _put_conv(sd, p + 'mlp.0', w, b)
        _put_bn(sd, p + 'mlp.1', _bn(rng, 2 * d))
        w, b = _conv(rng, d, 2 * d, zero_bias=True)
        # residual_gain < 1 shrinks the (random) update every GNN layer adds to the descriptors, so that the
        # landmark structure of the synthetic descriptors survives 18-28 random layers
        _put_conv(sd, p + 'mlp.3', w * np.float32(residual_gain), b)
    w, b = _conv(rng, d, d)
    # gain > 1 sharpens the (otherwise nearly flat, random-weight) assignment so
    # that match margins sit well above fp32 noise and Sinkhorn sees a wide range
    _put_conv(sd, 'final_proj', (w * np.float32(final_proj_gain)), (b * np.float32(final_proj_gain)))
    if conf_mlp:
        w, b = _conv(rng, 2 * d, 2 * d)
        _put_conv(sd, 'conf_mlp.layers_f.0', w, b)
        _put_bn(sd, 'conf_mlp.layers_f.1', _bn(rng, 2 * d))
        w, b = _conv(rng, d, 2 * d)
        _put_conv(sd, 'conf_mlp.layers_f.3', w, b)
        _put_bn(sd, 'conf_mlp.layers_f.4', _bn(rng, d))
        w, b = _conv(rng, d, 1)
        _put_conv(sd, 'conf_mlp.layers_c.0', w, b)
        _put_bn(sd, 'conf_mlp.layers_c.1', _bn(rng, d))
        w, b = _conv(rng, d, d)
        _put_conv(sd, 'conf_mlp.layers_c.3', w, b)
        _put_bn(sd, 'conf_mlp.layers_c.4', _bn(rng, d))
        w, b = _conv(rng, 1, d, zero_bias=True)
        _put_conv(sd, 'conf_mlp.layers.0', w, b)
        if conf_head == 'score':
            ident = {'weight': np.ones, 'bias': np.zeros, 'running_mean': np.zeros, 'running_var': np.ones}
            for key in ('layers_f.1', 'layers_f.4', 'layers_c.1', 'layers_c.4'):
                c = sd['conf_mlp.%s.weight' % key].shape[0]
                for name, fn in ident.items():
                    sd['conf_mlp.%s.%s' % (key, name)] = fn(c, np.float32)
            for key in ('layers_f.0', 'layers_f.3', 'layers_c.0', 'layers_c.3', 'layers.0'):
                sd['conf_mlp.%s.weight' % key] = sd['conf_mlp.%s.weight' % key] * np.float32(0.02)
                sd['conf_mlp.%s.bias' % key] = sd['conf_mlp.%s.bias' % key] * np.float32(0.02)
            sd['conf_mlp.layers_c.0.weight'][0, 0, 0] = 1.0
            sd['conf_mlp.layers_c.0.bias'][0] = 4.0
            sd['conf_mlp.layers_c.3.weight'][0, :, 0] = 0.0
            sd['conf_mlp.layers_c.3.weight'][0, 0, 0] = 1.0
            sd['conf_mlp.layers_c.3.bias'][0] = 0.0
            sd['conf_mlp.layers_f.3.weight'][0, :, 0] = 0.0
            sd['conf_mlp.layers_f.3.bias'][0] = 0.0
            sd['conf_mlp.layers.0.weight'][0, 0, 0] = 2.0
            sd['conf_mlp.layers.0.bias'][0] = -6.0
    return sd


def make_view_inputs(seed, counts, batch=1, width=640, height=480, desc_dim=256):
    """Synthetic matcher inputs (SURVEY.md §8d): per view keypoints ~ U(image),
    scores ~ U(0,1), descriptors ~ N(0,1) L2-normalised over channels
    (SuperPoint contract, superpoint.py:91-92), image{i} zeros (shape only)."""
    rng = np.random.default_rng(seed)
    data = {}
    for i, n in enumerate(counts):
        kp = rng.uniform(0.0, 1.0, size=(batch, n, 2)) * np.array([width, height])
        sc = rng.uniform(0.0, 1.0, size=(batch, n))
        de = rng.standard_normal((batch, desc_dim, n))
        de = de / np.maximum(np.linalg.norm(de, axis=1, keepdims=True), 1e-12)
        data['keypoints%d' % i] = kp.astype(np.float32)
        data['scores%d' % i] = sc.astype(np.float32)
        data['descriptors%d' % i] = de.astype(np.float32)
        data['image%d' % i] = np.zeros((batch, 1, height, width), np.float32)
    data['ids'] = list(range(len(counts)))
    return data


def make_correlated_view_inputs(seed, n_views, n_kpts, batch=1, width=640, height=480,
                                desc_dim=256, shared_frac=0.6, desc_noise=0.25):
    """Like make_view_inputs, but views share a pool of 'landmarks' so that the
    assignment has real structure (descriptor of the same landmark is similar in
    every view that sees it).  Keeps match margins away from fp32 noise."""
    rng = np.random.default_rng(seed)
    n_land = int(n_kpts / shared_frac)
    data = {}
    for b in range(batch):
        land_desc = rng.standard_normal((n_land, desc_dim))
        land_xy = rng.uniform(0.0, 1.0, size=(n_land, 2))
        for i in range(n_views):
            ids = rng.permutation(n_land)[:n_kpts]
            de = land_desc[ids] + desc_noise * rng.standard_normal((n_kpts, desc_dim))
            de = de / np.linalg.norm(de, axis=1, keepdims=True)
            xy = land_xy[ids] + 0.02 * rng.standard_normal((n_kpts, 2))
            xy = np.clip(xy, 0.0, 0.999) * np.array([width, height])
            sc = rng.uniform(0.0, 1.0, size=(n_kpts,))
            for key, val in (('keypoints%d' % i, xy), ('scores%d' % i, sc),
                             ('descriptors%d' % i, de.T)):
                data.setdefault(key, []).append(val.astype(np.float32))
    for k in list(data.keys()):
        data[k] = np.stack(data[k], 0)
    for i in range(n_views):
        data['image%d' % i] = np.zeros((batch, 1, height, width), np.float32)
    data['ids'] = list(range(n_views))
    return data


def make_scene_tuple_inputs(seed, n_views=5, n_kpts=1024, batch=1, width=640, height=480, f=577.87,
                            desc_dim=256, desc_noise=0.25, noise_px=1.0, sizes=None):
    """Geometrically consistent synthetic tuples for the end-to-end bench: 3-D landmarks (depth
    2..6 m) seen by `n_views` cameras (view 0 identity, others rotated <= 12 deg, baseline <= 0.6 m),
    pixel keypoints with `noise_px` noise, descriptors = landmark descriptor + noise (unit norm),
    scores U(0,1), K = [[f,0,(w-1)/2],[0,f,(h-1)/2],[0,0,1]].  `sizes`: optional list of one (width, height)
    per view (e.g. a portrait and a landscape image of a pair); each view then has its own K and image{i} shape, and
    the landmarks are the ones that project inside every view's image.  Default: (width, height) for every view.
    Returns the matcher `data` dict (numpy) with intr{i} [B,3,3], pose{i} [B,4,4] (cam->world ground truth, the
    reference's convention) and extr{i} (its inverse, world->cam)."""
    rng = np.random.default_rng(seed)
    sizes = [(width, height)] * n_views if sizes is None else [tuple(s) for s in sizes]
    assert len(sizes) == n_views
    Ks = [np.array([[f, 0, (w - 1) / 2], [0, f, (h - 1) / 2], [0, 0, 1.0]]) for w, h in sizes]
    Kinv = np.linalg.inv(Ks[0])
    out = {}

    def rod(w):
        th = np.linalg.norm(w)
        k = w / th
        Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * (Kx @ Kx)

    for b in range(batch):
        poses = [np.eye(4)]
        for _ in range(1, n_views):
            ax = rng.standard_normal(3)
            ax /= np.linalg.norm(ax)
            T = np.eye(4)
            T[:3, :3] = rod(ax * np.deg2rad(rng.uniform(3, 12)))
            d = rng.standard_normal(3)
            T[:3, 3] = d / np.linalg.norm(d) * rng.uniform(0.2, 0.6)
            poses.append(T)
        n_land = int(1.4 * n_kpts)
        # landmarks visible in every view (rejection sampling, vectorised)
        land = np.zeros((0, 3))
        while land.shape[0] < n_land:
            m = 4 * n_land
            z = rng.uniform(2, 6, m)
            uv = rng.uniform([30, 30], [sizes[0][0] - 30, sizes[0][1] - 30], size=(m, 2))
            X = (Kinv @ np.concatenate([uv, np.ones((m, 1))], 1).T).T * z[:, None]
            ok = np.ones(m, bool)
            for T, K, (w, h) in zip(poses, Ks, sizes):
                q = X @ T[:3, :3].T + T[:3, 3]
                px = (q @ K.T)[:, :2] / q[:, 2:3]
                ok &= (q[:, 2] > 0.5) & (px[:, 0] >= 0) & (px[:, 0] < w) & (px[:, 1] >= 0) & (px[:, 1] < h)
            land = np.concatenate([land, X[ok]], 0)
        land = land[:n_land]
        land_desc = rng.standard_normal((n_land, desc_dim))
        for i, (T, K) in enumerate(zip(poses, Ks)):
            sel = rng.permutation(n_land)[:n_kpts]
            q = land[sel] @ T[:3, :3].T + T[:3, 3]
            px = (q @ K.T)[:, :2] / q[:, 2:3] + noise_px * rng.standard_normal((n_kpts, 2))
            de = land_desc[sel] + desc_noise * rng.standard_normal((n_kpts, desc_dim))
            de /= np.linalg.norm(de, axis=1, keepdims=True)
            sc = rng.uniform(0, 1, n_kpts)
            # pose{i} follows the reference's data dicts: CAMERA-TO-WORLD (T_021 = inv(pose1) @ pose0,
            # eval_multi_view.py:58-59, helpers.py:255); extr{i} is the world-to-camera matrix used above
            for key, val in (('keypoints%d' % i, px), ('scores%d' % i, sc), ('descriptors%d' % i, de.T),
                             ('intr%d' % i, K), ('pose%d' % i, np.linalg.inv(T)), ('extr%d' % i, T)):
                out.setdefault(key, []).append(val.astype(np.float32))
            out.setdefault('landmark%d' % i, []).append(sel.astype(np.int64))
    for k in list(out.keys()):
        out[k] = np.stack(out[k], 0)
    for i, (w, h) in enumerate(sizes):
        out['image%d' % i] = np.zeros((batch, 1, h, w), np.float32)
    out['ids'] = list(range(n_views))
    return out


def render_tuple_images(data, seed=0, blob_sigma=2.0):
    """Render image{i} [B,1,H,W] in [0,1] for a make_scene_tuple_inputs tuple (best made with noise_px=0): every
    landmark a view sees is drawn as a Gaussian blob of radius ~blob_sigma px at its projection keypoints{i}, with a
    contrast of its own (bright or dark) on a mid-grey background, so that all views show the same scene points.  The
    image-in input of the multi-view evaluation; replaces the zero images in `data` in place and returns it."""
    rng = np.random.default_rng(seed)
    n_land = max(int(data['landmark%d' % i].max()) for i in data['ids']) + 1
    contrast = rng.uniform(0.4, 1.0, n_land) * rng.choice([-1.0, 1.0], n_land)
    r = int(np.ceil(3 * blob_sigma))
    g = np.exp(-np.arange(-r, r + 1) ** 2 / (2 * blob_sigma ** 2))         # peak 1: a lone blob reaches its contrast
    for i in data['ids']:
        B, _, H, W = data['image%d' % i].shape
        out = np.zeros((B, 1, H, W), np.float32)
        for b in range(B):
            acc = np.zeros((H, W))
            kp = data['keypoints%d' % i][b]
            x = np.clip(np.rint(kp[:, 0]).astype(np.int64), 0, W - 1)
            y = np.clip(np.rint(kp[:, 1]).astype(np.int64), 0, H - 1)
            np.add.at(acc, (y, x), contrast[data['landmark%d' % i][b]])
            acc = np.apply_along_axis(lambda row: np.convolve(row, g, mode='same'), 1, acc)
            acc = np.apply_along_axis(lambda col: np.convolve(col, g, mode='same'), 0, acc)
            out[b, 0] = np.clip(0.5 + 0.5 * acc, 0.0, 1.0)
        data['image%d' % i] = out
    return data


def make_superpoint_state_dict(seed=0, logit_gain=3.0):
    """Seeded SuperPoint weights with the reference's keys/shapes (models/models/superpoint.py:120-137): He-uniform
    convolutions; the detector logits are scaled by `logit_gain` so that the 65-way softmax has peaks."""
    rng = np.random.default_rng(seed)
    shapes = [('conv1a', 1, 64, 3), ('conv1b', 64, 64, 3), ('conv2a', 64, 64, 3), ('conv2b', 64, 64, 3),
              ('conv3a', 64, 128, 3), ('conv3b', 128, 128, 3), ('conv4a', 128, 128, 3), ('conv4b', 128, 128, 3),
              ('convPa', 128, 256, 3), ('convPb', 256, 65, 1), ('convDa', 128, 256, 3), ('convDb', 256, 256, 1)]
    sd = {}
    for name, cin, cout, k in shapes:
        bound = np.sqrt(6.0 / (cin * k * k))
        g = logit_gain if name == 'convPb' else 1.0
        sd[name + '.weight'] = (rng.uniform(-bound, bound, size=(cout, cin, k, k)) * g).astype(np.float32)
        sd[name + '.bias'] = (rng.uniform(-0.1, 0.1, size=(cout,)) * g).astype(np.float32)
    return sd


def make_image(seed, height, width, batch=1):
    """Seeded grayscale test image in [0,1]: smooth blobs + oriented edges + fine texture.  [batch,1,H,W] float32."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:height, 0:width].astype(np.float64)
    out = []
    for _ in range(batch):
        img = np.zeros((height, width))
        for _ in range(24):
            cx, cy = rng.uniform(0, width), rng.uniform(0, height)
            s = rng.uniform(4, 30)
            img += rng.uniform(-1, 1) * np.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / (2 * s * s))
        for _ in range(8):
            th = rng.uniform(0, np.pi)
            img += 0.3 * np.sign(np.sin((xx * np.cos(th) + yy * np.sin(th)) / rng.uniform(6, 25) + rng.uniform(0, 6)))
        img += 0.15 * rng.standard_normal((height, width))
        img = (img - img.min()) / (img.max() - img.min())
        out.append(img[None])
    return np.stack(out, 0).astype(np.float32)


def landmark_gt_matches(la, lb):
    """Ground-truth assignments of one pair from the scene's landmark ids (two keypoints match iff they observe the same
    landmark), in the layout and with the class-balancing weights of compute_gt_matches_of_image_pair
    (helpers.py:190-213): la, lb [B, n] -> (indices [B, 2, n+1] int64, weights [B, 2, n+1] float32).  For the training
    bench / tests, whose synthetic scenes carry landmark ids instead of depth maps."""
    la, lb = np.asarray(la), np.asarray(lb)
    B, n = la.shape
    idx = np.full((B, 2, n + 1), -1, np.int64)
    w = np.zeros((B, 2, n + 1), np.float32)
    for b in range(B):
        order = np.argsort(lb[b], kind='stable')
        pos = np.searchsorted(lb[b][order], la[b])
        pos = np.clip(pos, 0, n - 1)
        hit = lb[b][order][pos] == la[b]
        i0 = np.where(hit, order[pos], -1)
        idx[b, 0, :n] = i0
        i1 = np.full(n, -1, np.int64)
        i1[i0[hit]] = np.nonzero(hit)[0]
        idx[b, 1, :n] = i1
        m = int(hit.sum())
        mw = np.float32(2.0 * m) / np.float32(2.0 * n)
        uw = np.float32(0.5) / (np.float32(1.0) - mw)
        mw = np.float32(0.5) / mw if m else np.float32(0.0)
        w[b, 0] = np.where(idx[b, 0] >= 0, mw, uw)
        w[b, 1] = np.where(idx[b, 1] >= 0, mw, uw)
    return idx, w
