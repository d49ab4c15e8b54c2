"""Reference restatement of MatchingDataset.__getitem__'s per-image transforms (datasets/matching_dataset.py:14-24,
:110-154, :182-211) for the image-preparation tests: float32 torch / torchvision functional ops on the CPU, and the
intrinsics bookkeeping in float32 numpy, line for line.

The resize passes antialias=False: the reference pins torchvision 0.11.2, whose tensor resize does not antialias;
torchvision >= 0.17 does by default."""
import numpy as np
import torch
import torchvision
from torchvision.transforms import functional as TF


def resize_intrinsics(K, fact_x, fact_y):
    K[0, 0] *= fact_x
    K[1, 1] *= fact_y
    K[0, 2] *= fact_x
    K[1, 2] *= fact_y
    return K


def crop_intrinsics(K, crop_x, crop_y):
    K[0, 2] -= crop_x
    K[1, 2] -= crop_y
    return K


def crop_window(h, w, center=True, rng=np.random):
    """crop() (:132-154): -> (top, bottom, left, right)."""
    if w > h:
        left = int((w - h) / 2.) if center else rng.randint(0, w - h + 1)
        right = left + h
        top, bottom = 0, h
    else:
        top = int((h - w) / 2.) if center else rng.randint(0, h - w + 1)
        bottom = top + w
        left, right = 0, w
    return top, bottom, left, right


def get_color_jitter_params(jitter):
    centered_at_1 = (1. - jitter, 1. + jitter)
    centered_at_0 = (-jitter, jitter)
    return torchvision.transforms.ColorJitter.get_params(brightness=centered_at_1, contrast=centered_at_1,
                                                         saturation=centered_at_1, hue=centered_at_0)


def apply_color_jitter(rgb, jitter_params):
    fn_idx, brightness, contrast, saturation, hue = jitter_params
    for fn_id in fn_idx:
        if fn_id == 0 and brightness is not None:
            rgb = TF.adjust_brightness(rgb, brightness)
        elif fn_id == 1 and contrast is not None:
            rgb = TF.adjust_contrast(rgb, contrast)
        elif fn_id == 2 and saturation is not None:
            rgb = TF.adjust_saturation(rgb, saturation)
        elif fn_id == 3 and hue is not None:
            rgb = TF.adjust_hue(rgb, hue)
    return rgb


def prepare_image(rgb_u8, depth, intr, crop=None, jitter_params=None):
    """One view of __getitem__ (:182-211): rgb_u8 [H, W, 3] uint8, depth [h, w], intr float32 (copied), crop None or
    (top, bottom, left, right) of crop_window -> (gray [1, h', w'] float32, depth, intr)."""
    intr = intr.copy().astype(np.float32)
    rgb = torchvision.transforms.ToTensor()(rgb_u8)
    if crop is not None:
        top, bottom, left, right = crop
        intr = crop_intrinsics(intr, left, top)
        rgb = rgb[:, top:bottom, left:right]
        depth = depth[top:bottom, left:right]
    if rgb.shape[2] == 1296 and rgb.shape[1] == 968:
        rgb = torch.nn.functional.pad(rgb, (0, 0, 2, 2), "constant", 0)
        intr[1, 2] = intr[1, 2] + 2
    resize_size = depth.shape
    if resize_size[1] != rgb.shape[2] or resize_size[0] != rgb.shape[1]:
        fact_x, fact_y = resize_size[1] / rgb.shape[2], resize_size[0] / rgb.shape[1]
        intr = resize_intrinsics(intr, fact_x, fact_y)
        rgb = TF.resize(rgb, size=list(resize_size), antialias=False)
    if jitter_params is not None:
        rgb = apply_color_jitter(rgb, jitter_params)
    return TF.rgb_to_grayscale(rgb), depth, intr


def grayscale_mean_before_contrast(rgb_u8, jitter_params, size=None):
    """The mean adjust_contrast takes, for printing the oracle-vs-kernel difference: the grayscale mean of the image
    after the ops that precede contrast in the order (after the resize to `size`, if given)."""
    rgb = torchvision.transforms.ToTensor()(rgb_u8)
    if size is not None and tuple(size) != tuple(rgb.shape[1:]):
        rgb = TF.resize(rgb, size=list(size), antialias=False)
    fn_idx = [int(v) for v in jitter_params[0]]
    pos = fn_idx.index(1)
    rgb = apply_color_jitter(rgb, (fn_idx[:pos],) + tuple(jitter_params[1:]))
    return torch.mean(TF.rgb_to_grayscale(rgb).to(torch.float32), dim=(-3, -2, -1))
