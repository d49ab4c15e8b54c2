"""SuperPoint with the reference's constructor, config keys, state-dict keys and forward(data) -> dict contract
(models/models/superpoint.py:102-229), computing in libmvm_b200.so: the VGG encoder, both heads, the three-round
non-maximum suppression and the descriptor sampling are CUDA kernels (csrc/superpoint.cu); the nn.Conv2d modules below
only own the parameters under the reference's key names.  In forward, what stays in torch is index book-keeping on the
NMS output (nonzero / border mask / top-k), as in the reference; forward_batch does that selection on the device too,
for a whole batch in one launch.  No CPU fallback.

`weights`: path of a `superpoint_v1.pth`-style state dict, or None to keep the random initialisation (then load one with
load_state_dict); the reference hard-codes the path next to its source file, which does not exist here."""
import ctypes as C

import torch
from torch import nn

from .. import _lib

CONV3 = ['conv1a', 'conv1b', 'conv2a', 'conv2b', 'conv3a', 'conv3b', 'conv4a', 'conv4b', 'convPa', 'convDa']


def remove_borders(keypoints, scores, border, height, width):
    """superpoint.py:66-71."""
    mask_h = (keypoints[:, 0] >= border) & (keypoints[:, 0] < (height - border))
    mask_w = (keypoints[:, 1] >= border) & (keypoints[:, 1] < (width - border))
    mask = mask_h & mask_w
    return keypoints[mask], scores[mask]


def top_k_keypoints(keypoints, scores, k):
    """superpoint.py:74-78."""
    if k >= len(keypoints):
        return keypoints, scores
    scores, indices = torch.topk(scores, k, dim=0)
    return keypoints[indices], scores


class SuperPoint(nn.Module):
    default_config = {
        'descriptor_dim': 256,
        'nms_radius': 4,
        'keypoint_threshold': 0.005,
        'max_keypoints': -1,
        'remove_borders': 4,
        'fill_with_random_keypoints': False,
        'weights': None,
    }

    def __init__(self, config):
        super().__init__()
        self.config = {**self.default_config, **config}
        assert self.config['descriptor_dim'] == 256, 'the kernels are specialised for 256-d descriptors'
        c1, c2, c3, c4, c5 = 64, 64, 128, 128, 256
        self.conv1a = nn.Conv2d(1, c1, kernel_size=3, stride=1, padding=1)
        self.conv1b = nn.Conv2d(c1, c1, kernel_size=3, stride=1, padding=1)
        self.conv2a = nn.Conv2d(c1, c2, kernel_size=3, stride=1, padding=1)
        self.conv2b = nn.Conv2d(c2, c2, kernel_size=3, stride=1, padding=1)
        self.conv3a = nn.Conv2d(c2, c3, kernel_size=3, stride=1, padding=1)
        self.conv3b = nn.Conv2d(c3, c3, kernel_size=3, stride=1, padding=1)
        self.conv4a = nn.Conv2d(c3, c4, kernel_size=3, stride=1, padding=1)
        self.conv4b = nn.Conv2d(c4, c4, kernel_size=3, stride=1, padding=1)
        self.convPa = nn.Conv2d(c4, c5, kernel_size=3, stride=1, padding=1)
        self.convPb = nn.Conv2d(c5, 65, kernel_size=1, stride=1, padding=0)
        self.convDa = nn.Conv2d(c4, c5, kernel_size=3, stride=1, padding=1)
        self.convDb = nn.Conv2d(c5, 256, kernel_size=1, stride=1, padding=0)
        if self.config['weights']:
            self.load_state_dict(torch.load(str(self.config['weights']), map_location='cpu'))
        mk = self.config['max_keypoints']
        if mk == 0 or mk < -1:
            raise ValueError('"max_keypoints" must be positive or "-1"')
        self._packed = None
        self._packed_key = None
        self._ws = None

    def _pack(self, device):
        key = (str(device),) + tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._packed is not None and key == self._packed_key:
            return self._packed
        keep = []
        W = _lib.SuperPointWeights()
        for i, name in enumerate(CONV3):
            conv = getattr(self, name)
            w = conv.weight.detach().float().permute(2, 3, 1, 0).contiguous().reshape(9, conv.in_channels, conv.out_channels)
            w = w.to(device).contiguous()
            b = conv.bias.detach().float().to(device).contiguous()
            keep += [w, b]
            W.w[i], W.b[i] = w.data_ptr(), b.data_ptr()
        for tag, name in (('pb', 'convPb'), ('db', 'convDb')):
            conv = getattr(self, name)
            w = conv.weight.detach().float().reshape(conv.out_channels, conv.in_channels).to(device).contiguous()
            b = conv.bias.detach().float().to(device).contiguous()
            keep += [w, b]
            setattr(W, 'w_' + tag, w.data_ptr())
            setattr(W, 'b_' + tag, b.data_ptr())
        self._packed, self._packed_key = (W, keep), key
        return self._packed

    def dense(self, images):
        """images [B,1,H,W], any H, W >= 16 -> (scores after NMS [B,8*(H//8),8*(W//8)], dense descriptors
        [B,H//8,W//8,256]): the three 2x2 pools floor odd sizes, so the last H % 8 rows and W % 8 columns get no score,
        as in the reference."""
        lib = _lib.lib()
        if images.device.type != 'cuda':
            raise _lib.MvmError('SuperPoint needs CUDA tensors (no CPU fallback)')
        B, c, H, Wd = images.shape
        assert c == 1
        dev = images.device
        W, _ = self._pack(dev)
        img = images.float().reshape(B, H, Wd).contiguous()
        scores = torch.empty(B, H // 8 * 8, Wd // 8 * 8, dtype=torch.float32, device=dev)
        dense = torch.empty(B, H // 8, Wd // 8, 256, dtype=torch.float32, device=dev)
        nbytes = lib.mvm_superpoint_workspace_bytes(B, H, Wd)
        if self._ws is None or self._ws.numel() < nbytes or self._ws.device != dev:
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            rc = lib.mvm_superpoint_dense(C.byref(W), _lib.ptr(img), B, H, Wd, int(self.config['nms_radius']), _lib.ptr(scores),
                                          _lib.ptr(dense), _lib.ptr(self._ws), nbytes, _lib.stream_ptr())
        _lib.check(rc, 'mvm_superpoint_dense')
        return scores, dense

    def forward(self, data):
        """Compute keypoints, scores, descriptors for the images (superpoint.py:143-229): data['image'] is an iterable of
        [B,1,H,W] batches (batches may differ in size, as with merge=False in eval_pairs.py); returns lists over all
        images."""
        lib = _lib.lib()
        all_keypoints, all_scores, all_descriptors = [], [], []
        with torch.no_grad():
            for images in data['image']:
                scores_map, dense = self.dense(images)
                B, H, Wd = scores_map.shape
                h, w = H // 8, Wd // 8
                for bi in range(B):
                    s = scores_map[bi]
                    kp = torch.nonzero(s > self.config['keypoint_threshold'])
                    sc = s[tuple(kp.t())]
                    if self.config['remove_borders'] > 0:
                        kp, sc = remove_borders(kp, sc, self.config['remove_borders'], h * 8, w * 8)
                    if self.config['max_keypoints'] >= 0:
                        kp, sc = top_k_keypoints(kp, sc, self.config['max_keypoints'])
                        if self.config['fill_with_random_keypoints'] and kp.shape[0] < self.config['max_keypoints']:
                            add_n = self.config['max_keypoints'] - kp.shape[0]
                            border = self.config['remove_borders']
                            add_k = torch.cat((torch.randint(border, h * 8 - border, (add_n, 1), device=kp.device),
                                               torch.randint(border, w * 8 - border, (add_n, 1), device=kp.device)), 1)
                            kp = torch.cat((kp, add_k), 0)
                            sc = torch.cat((sc, torch.zeros(add_n, device=sc.device)), 0)
                    kxy = torch.flip(kp, [1]).float().contiguous()          # (h, w) -> (x, y)
                    n = kxy.shape[0]
                    desc = torch.empty(256, n, dtype=torch.float32, device=kxy.device)
                    with torch.cuda.device(kxy.device):
                        rc = lib.mvm_superpoint_sample(_lib.ptr(dense[bi].contiguous()), _lib.ptr(kxy) if n else None, n, h, w,
                                                       _lib.ptr(desc) if n else None, _lib.stream_ptr())
                    _lib.check(rc, 'mvm_superpoint_sample')
                    all_keypoints.append(kxy)
                    all_scores.append(sc)
                    all_descriptors.append(desc)
        return {'keypoints': all_keypoints, 'scores': all_scores, 'descriptors': all_descriptors}

    def forward_batch(self, images):
        """forward for one batch of images [B,1,H,W] whose results are used as stacked tensors (run_super_point): needs
        max_keypoints = K > 0 and returns {'keypoints' [B,K,2] (x, y), 'scores' [B,K], 'descriptors' [B,256,K],
        'counts' [B] int32 = valid entries per image}.  Selection and sampling are one launch each for the batch
        (mvm_superpoint_select / mvm_superpoint_sample_batch) and do not synchronise with the host.  Entries at or past
        an image's count are zero.  Per image the result is forward's, bit for bit, except for the order among equal
        scores: torch.topk leaves it open, here the lower raster index comes first (also at the K-th score).

        With fill_with_random_keypoints the [B] counts are read once (one synchronisation per batch) and every short
        image is filled with the same torch.randint calls, in the same order, as forward makes, so the fill draws the
        same keypoints from the same generator state; counts are then K."""
        K = self.config['max_keypoints']
        if K < 0:
            raise ValueError('forward_batch needs "max_keypoints" > 0 (fixed-size outputs); use forward')
        lib = _lib.lib()
        with torch.no_grad():
            scores_map, dense = self.dense(images)
            B, H, Wd = scores_map.shape
            h, w = H // 8, Wd // 8
            dev = scores_map.device
            kxy = torch.empty(B, K, 2, dtype=torch.float32, device=dev)
            sc = torch.empty(B, K, dtype=torch.float32, device=dev)
            counts = torch.empty(B, dtype=torch.int32, device=dev)
            with torch.cuda.device(dev):
                rc = lib.mvm_superpoint_select(_lib.ptr(scores_map), B, H, Wd, float(self.config['keypoint_threshold']),
                                               int(self.config['remove_borders']), K, _lib.ptr(kxy), _lib.ptr(sc),
                                               _lib.ptr(counts), _lib.stream_ptr())
            _lib.check(rc, 'mvm_superpoint_select')
            counts.clamp_(max=K)
            if self.config['fill_with_random_keypoints']:
                border = self.config['remove_borders']
                for bi, n in enumerate(counts.tolist()):
                    if n < K:
                        add_n = K - n
                        add_k = torch.cat((torch.randint(border, h * 8 - border, (add_n, 1), device=dev),
                                           torch.randint(border, w * 8 - border, (add_n, 1), device=dev)), 1)
                        kxy[bi, n:] = torch.flip(add_k, [1]).float()
                counts.fill_(K)
            desc = torch.empty(B, 256, K, dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                rc = lib.mvm_superpoint_sample_batch(_lib.ptr(dense), _lib.ptr(kxy), _lib.ptr(counts), B, K, h, w,
                                                     _lib.ptr(desc), _lib.stream_ptr())
            _lib.check(rc, 'mvm_superpoint_sample_batch')
        return {'keypoints': kxy, 'scores': sc, 'descriptors': desc, 'counts': counts}
