"""Shared inputs of the FID / KID tests: the distinct convolution geometries of the FID Inception-v3, render-like
images and random weights (oracle.inception_ref.random_state_dict)."""
import numpy as np
import torch
from PIL import Image, ImageDraw


def conv_geometries():
    """Distinct (cin, cout, kh, kw, stride, pad_h, pad_w, H, W) of the 94 convolutions at a 299 x 299 input, in
    network order (torchvision's Inception3 shapes, found with forward hooks)."""
    from torchvision.models import inception_v3
    net = inception_v3(weights=None, aux_logits=False, init_weights=False, num_classes=1008).eval()
    seen = []

    def hook(mod, inp, out):
        x = inp[0]
        g = (mod.in_channels, mod.out_channels, mod.kernel_size[0], mod.kernel_size[1], mod.stride[0],
             mod.padding[0], mod.padding[1], x.shape[2], x.shape[3])
        seen.append(g)

    hs = [m.register_forward_hook(hook) for m in net.modules() if isinstance(m, torch.nn.Conv2d)]
    with torch.no_grad():
        net(torch.zeros(1, 3, 299, 299))
    for h in hs:
        h.remove()
    out = []
    for g in seen:
        if g not in out:
            out.append(g)
    return seen, out


def render_like(seed, size=256, mode="RGB"):
    """A top-down-render-like image: a light floor with a few solid boxes, RGB or RGBA."""
    rng = np.random.default_rng(seed)
    bg = tuple(int(v) for v in rng.integers(200, 256, 3)) + ((255,) if mode == "RGBA" else ())
    im = Image.new(mode, (size, size), bg)
    d = ImageDraw.Draw(im)
    for _ in range(int(rng.integers(3, 8))):
        x0, y0 = (int(v) for v in rng.integers(0, size - 40, 2))
        w, h = (int(v) for v in rng.integers(15, 90, 2))
        col = tuple(int(v) for v in rng.integers(0, 256, 3)) + ((int(rng.integers(128, 256)),) if mode == "RGBA" else ())
        d.rectangle([x0, y0, min(size - 1, x0 + w), min(size - 1, y0 + h)], fill=col)
    return im


def write_folder(path, seeds, mode="RGB"):
    path.mkdir(parents=True, exist_ok=True)
    for s in seeds:
        render_like(s, mode=mode).save(str(path / ("%05d.png" % s)))
    return path
