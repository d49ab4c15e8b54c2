"""SuperPoint restated in plain torch.nn.functional, parameterised by dtype: float64 is the reference the kernels of
csrc/superpoint.cu are tested against, float32 the yardstick of how far a correct float32 computation strays from it.

The operations are the ones models/superpoint.py describes: a VGG encoder (conv1a .. conv4b, 3x3 / pad 1, each with
ReLU, a 2x2 / stride 2 max pool after conv1b, conv2b and conv3b that floors odd sides), the detector head (convPa +
ReLU, convPb, softmax over 65 bins with the last, the dustbin, dropped, then depth-to-space), the three-round
non-maximum suppression, the descriptor head (convDa + ReLU, convDb, L2 normalisation over channels) and bilinear
descriptor sampling at keypoints in the coordinates of the 8 times larger score map.
"""
import torch
import torch.nn.functional as F

ENCODER = [('conv1a', 'conv1b'), ('conv2a', 'conv2b'), ('conv3a', 'conv3b'), ('conv4a', 'conv4b')]


def _params(state_dict, dtype, device):
    return {k: torch.as_tensor(v).to(device=device, dtype=dtype) for k, v in state_dict.items()}


def _conv(x, p, name, relu=True):
    wt = p[name + '.weight']
    y = F.conv2d(x, wt, p[name + '.bias'], padding=wt.shape[-1] // 2)
    return F.relu(y) if relu else y


def simple_nms(scores, nms_radius):
    """[B, H, W] -> [B, H, W]: keep a score where it is the maximum of its (2r+1)^2 window (-inf outside the map), then
    twice: suppress the windows around the kept points and keep the new window maxima among what is left."""
    r = int(nms_radius)

    def max_pool(x):
        return F.max_pool2d(x[:, None], kernel_size=2 * r + 1, stride=1, padding=r)[:, 0]

    zeros = torch.zeros_like(scores)
    max_mask = scores == max_pool(scores)
    for _ in range(2):
        supp_mask = max_pool(max_mask.to(scores.dtype)) > 0
        supp_scores = torch.where(supp_mask, zeros, scores)
        new_max_mask = supp_scores == max_pool(supp_scores)
        max_mask = max_mask | (new_max_mask & ~supp_mask)
    return torch.where(max_mask, scores, zeros)


def dense(images, state_dict, nms_radius, dtype=torch.float64, device='cpu'):
    """images [B, 1, H, W] -> (raw scores [B, 8h, 8w], scores after NMS [B, 8h, 8w], unit dense descriptors
    [B, h, w, 256]) with h = H // 8, w = W // 8, computed in `dtype` on `device`."""
    p = _params(state_dict, dtype, device)
    x = torch.as_tensor(images).to(device=device, dtype=dtype)
    for i, (a, b) in enumerate(ENCODER):
        x = _conv(_conv(x, p, a), p, b)
        if i < 3:
            x = F.max_pool2d(x, 2, 2)
    B, _, h, w = x.shape
    logits = _conv(_conv(x, p, 'convPa'), p, 'convPb', relu=False)                  # [B, 65, h, w]
    prob = F.softmax(logits, dim=1)[:, :-1]                                         # dustbin dropped
    # depth-to-space: scores[b, 8y + i, 8x + j] = prob[b, 8i + j, y, x]
    raw = prob.reshape(B, 8, 8, h, w).permute(0, 3, 1, 4, 2).reshape(B, 8 * h, 8 * w)
    desc = _conv(_conv(x, p, 'convDa'), p, 'convDb', relu=False)                    # [B, 256, h, w]
    desc = F.normalize(desc, p=2, dim=1, eps=1e-12).permute(0, 2, 3, 1).contiguous()
    return raw, simple_nms(raw, nms_radius), desc


def sample(dense_map, keypoints, normalize=True):
    """dense_map [h, w, 256], keypoints [n, 2] as (x, y) pixels of the [8h, 8w] score map -> [256, n]: each keypoint
    mapped to grid coordinates by (k - s/2 + 0.5) / (size s - s/2 - 0.5) * 2 - 1 with s = 8, bilinear grid_sample with
    align_corners=True and zero padding, then (unless normalize is False) L2 normalisation over the channels."""
    h, w, c = dense_map.shape
    s = 8
    k = torch.as_tensor(keypoints).to(device=dense_map.device, dtype=dense_map.dtype).reshape(-1, 2)
    size = torch.tensor([w * s - s / 2 - 0.5, h * s - s / 2 - 0.5], dtype=dense_map.dtype, device=dense_map.device)
    grid = ((k - s / 2 + 0.5) / size) * 2 - 1
    d = F.grid_sample(dense_map.permute(2, 0, 1)[None], grid.view(1, 1, -1, 2), mode='bilinear',
                      padding_mode='zeros', align_corners=True).reshape(c, -1)
    return F.normalize(d, p=2, dim=0) if normalize else d


def select(scores_nms, threshold, border, max_keypoints):
    """One image's keypoint rule of models/superpoint.py on a [8h, 8w] NMS'd map: scores above the threshold, at least
    `border` pixels inside every edge, then the max_keypoints largest (all when -1).  Returns (keypoints [n, 2] as
    (x, y), scores [n])."""
    from e2e_multi_view_matching_b200.models.superpoint import remove_borders, top_k_keypoints
    H, W = scores_nms.shape
    kp = torch.nonzero(scores_nms > threshold)
    sc = scores_nms[tuple(kp.t())]
    if border > 0:
        kp, sc = remove_borders(kp, sc, border, H, W)
    if max_keypoints >= 0:
        kp, sc = top_k_keypoints(kp, sc, max_keypoints)
    return torch.flip(kp, [1]), sc
