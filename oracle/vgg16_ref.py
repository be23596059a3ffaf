"""ORACLE: torchvision `vgg16` feature path as improved_precision_recall.py:159-163 runs it,
classifier[:4](features(x).view(-1, 7 * 7 * 512)), written with torch.nn.functional so that it runs in any dtype
(fp64 for the tests) without torchvision.  `sd` is a torchvision vgg16 state dict (classifier.6 unused)."""
import torch
import torch.nn.functional as F

CONV_IDX = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
POOL_AFTER = (2, 4, 7, 10, 13)       # 1-based conv layers followed by the 2 x 2 max-pool
CHANNELS = (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)


def conv_layer(x, w, b, pool):
    y = F.relu(F.conv2d(x, w, b, padding=1))
    return F.max_pool2d(y, 2, 2) if pool else y


def features(sd, x, dtype=torch.float64):
    """x [B, 3, 224, 224] normalised -> fc2 output before its ReLU [B, 4096]."""
    g = lambda n: sd[n].to(dtype)
    x = x.to(dtype)
    for l, i in enumerate(CONV_IDX):
        x = conv_layer(x, g("features.%d.weight" % i), g("features.%d.bias" % i), (l + 1) in POOL_AFTER)
    x = x.reshape(-1, 7 * 7 * 512)
    x = F.relu(F.linear(x, g("classifier.0.weight"), g("classifier.0.bias")))
    return F.linear(x, g("classifier.3.weight"), g("classifier.3.bias"))


def resize_nearest(x, size=224):
    """extract_features' resize of tensors that are not 224 x 224: F.interpolate's default (nearest) mode."""
    return x if tuple(x.shape[-2:]) == (size, size) else F.interpolate(x, size=(size, size))
