"""Seeded inputs of the improved precision and recall tests: VGG16 weights with He scaling (activations stay O(1)
through the 13 convolutions), top-down-render-like images (coloured rectangles on white) and clustered features."""
import numpy as np
import torch

from oracle.vgg16_ref import CHANNELS, CONV_IDX

MEAN = np.array([0.485, 0.456, 0.406], np.float32)[:, None, None]
STD = np.array([0.229, 0.224, 0.225], np.float32)[:, None, None]


def he_state_dict(seed=0):
    """A torchvision-vgg16-shaped state dict (classifier.6 included) with He-scaled normal weights."""
    g = torch.Generator().manual_seed(seed)
    sd, cin = {}, 3
    for i, cout in zip(CONV_IDX, CHANNELS):
        sd["features.%d.weight" % i] = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (9 * cin)) ** 0.5
        sd["features.%d.bias" % i] = torch.randn(cout, generator=g) * 0.05
        cin = cout
    for i, (n, k) in zip((0, 3, 6), ((4096, 25088), (4096, 4096), (1000, 4096))):
        sd["classifier.%d.weight" % i] = torch.randn(n, k, generator=g) * (2.0 / k) ** 0.5
        sd["classifier.%d.bias" % i] = torch.randn(n, generator=g) * 0.05
    return sd


def render_like(n, size=224, seed=0):
    """uint8 [n, size, size, 3]: white floor with 2..8 coloured axis-aligned rectangles."""
    rng = np.random.default_rng(seed)
    img = np.full((n, size, size, 3), 255, np.uint8)
    for b in range(n):
        for _ in range(rng.integers(2, 9)):
            y0, x0 = rng.integers(0, size - 8, 2)
            h, w = rng.integers(8, size // 3, 2)
            img[b, y0:y0 + h, x0:x0 + w] = rng.integers(0, 256, 3)
    return img


def normalise(img_u8):
    """ToTensor + ImageNet Normalize in fp32: uint8 [n, H, W, 3] -> float32 [n, 3, H, W]."""
    x = img_u8.astype(np.float32).transpose(0, 3, 1, 2) / np.float32(255)
    return torch.from_numpy(np.ascontiguousarray((x - MEAN) / STD))


def clustered(n, d, clusters=8, spread=0.3, seed=0, dtype=np.float32, centre_seed=None):
    """Points around `clusters` centres (drawn from centre_seed, default seed), so two sets can share them."""
    centres = np.random.default_rng(seed if centre_seed is None else centre_seed).normal(0, 1, (clusters, d)) * 3
    rng = np.random.default_rng(seed + 7919)
    lab = rng.integers(0, clusters, n)
    return (centres[lab] + rng.normal(0, spread, (n, d))).astype(dtype)
