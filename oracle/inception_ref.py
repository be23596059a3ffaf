"""fp64 functional restatement of the FID Inception-v3 (torchvision `Inception3` layout, aux_logits off) up to the
pool3 output [B, 2048], for tests.  `fid=True` applies the FID blocks (pytorch-fid's FIDInceptionA / C / E_1 / E_2):
branch_pool average pools without the padding in the count, and Mixed_7c's branch_pool as a 3 x 3 / stride 1 / pad 1
max pool; `fid=False` is torchvision's network.  Runs on any device in the dtype of its input."""
import torch
import torch.nn.functional as F

BN_EPS = 1e-3


def basic_conv(sd, name, x, stride=1, padding=0):
    w = sd[name + ".conv.weight"].to(x)
    y = F.conv2d(x, w, stride=stride, padding=padding)
    g, b = sd[name + ".bn.weight"].to(x), sd[name + ".bn.bias"].to(x)
    rm, rv = sd[name + ".bn.running_mean"].to(x), sd[name + ".bn.running_var"].to(x)
    y = F.batch_norm(y, rm, rv, g, b, training=False, eps=BN_EPS)
    return F.relu(y)


def _avg(x, fid):
    return F.avg_pool2d(x, 3, stride=1, padding=1, count_include_pad=not fid)


def block_a(sd, p, x, fid):
    b1 = basic_conv(sd, p + ".branch1x1", x)
    b5 = basic_conv(sd, p + ".branch5x5_2", basic_conv(sd, p + ".branch5x5_1", x), padding=2)
    b3 = basic_conv(sd, p + ".branch3x3dbl_1", x)
    b3 = basic_conv(sd, p + ".branch3x3dbl_3", basic_conv(sd, p + ".branch3x3dbl_2", b3, padding=1), padding=1)
    bp = basic_conv(sd, p + ".branch_pool", _avg(x, fid))
    return torch.cat([b1, b5, b3, bp], 1)


def block_b(sd, p, x):
    b3 = basic_conv(sd, p + ".branch3x3", x, stride=2)
    bd = basic_conv(sd, p + ".branch3x3dbl_1", x)
    bd = basic_conv(sd, p + ".branch3x3dbl_3", basic_conv(sd, p + ".branch3x3dbl_2", bd, padding=1), stride=2)
    return torch.cat([b3, bd, F.max_pool2d(x, 3, stride=2)], 1)


def block_c(sd, p, x, fid):
    b1 = basic_conv(sd, p + ".branch1x1", x)
    b7 = basic_conv(sd, p + ".branch7x7_1", x)
    b7 = basic_conv(sd, p + ".branch7x7_2", b7, padding=(0, 3))
    b7 = basic_conv(sd, p + ".branch7x7_3", b7, padding=(3, 0))
    bd = basic_conv(sd, p + ".branch7x7dbl_1", x)
    bd = basic_conv(sd, p + ".branch7x7dbl_2", bd, padding=(3, 0))
    bd = basic_conv(sd, p + ".branch7x7dbl_3", bd, padding=(0, 3))
    bd = basic_conv(sd, p + ".branch7x7dbl_4", bd, padding=(3, 0))
    bd = basic_conv(sd, p + ".branch7x7dbl_5", bd, padding=(0, 3))
    bp = basic_conv(sd, p + ".branch_pool", _avg(x, fid))
    return torch.cat([b1, b7, bd, bp], 1)


def block_d(sd, p, x):
    b3 = basic_conv(sd, p + ".branch3x3_2", basic_conv(sd, p + ".branch3x3_1", x), stride=2)
    b7 = basic_conv(sd, p + ".branch7x7x3_1", x)
    b7 = basic_conv(sd, p + ".branch7x7x3_2", b7, padding=(0, 3))
    b7 = basic_conv(sd, p + ".branch7x7x3_3", b7, padding=(3, 0))
    b7 = basic_conv(sd, p + ".branch7x7x3_4", b7, stride=2)
    return torch.cat([b3, b7, F.max_pool2d(x, 3, stride=2)], 1)


def block_e(sd, p, x, pool):
    b1 = basic_conv(sd, p + ".branch1x1", x)
    b3 = basic_conv(sd, p + ".branch3x3_1", x)
    b3 = torch.cat([basic_conv(sd, p + ".branch3x3_2a", b3, padding=(0, 1)),
                    basic_conv(sd, p + ".branch3x3_2b", b3, padding=(1, 0))], 1)
    bd = basic_conv(sd, p + ".branch3x3dbl_2", basic_conv(sd, p + ".branch3x3dbl_1", x), padding=1)
    bd = torch.cat([basic_conv(sd, p + ".branch3x3dbl_3a", bd, padding=(0, 1)),
                    basic_conv(sd, p + ".branch3x3dbl_3b", bd, padding=(1, 0))], 1)
    bp = basic_conv(sd, p + ".branch_pool", pool(x))
    return torch.cat([b1, b3, bd, bp], 1)


def inception_features(sd, x, fid=True):
    """x: the detector's input [B, 3, 299, 299] (already (v - 128) / 128 for clean-fid) -> [B, 2048]."""
    x = basic_conv(sd, "Conv2d_1a_3x3", x, stride=2)
    x = basic_conv(sd, "Conv2d_2a_3x3", x)
    x = basic_conv(sd, "Conv2d_2b_3x3", x, padding=1)
    x = F.max_pool2d(x, 3, stride=2)
    x = basic_conv(sd, "Conv2d_3b_1x1", x)
    x = basic_conv(sd, "Conv2d_4a_3x3", x)
    x = F.max_pool2d(x, 3, stride=2)
    for name in ("Mixed_5b", "Mixed_5c", "Mixed_5d"):
        x = block_a(sd, name, x, fid)
    x = block_b(sd, "Mixed_6a", x)
    for name in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
        x = block_c(sd, name, x, fid)
    x = block_d(sd, "Mixed_7a", x)
    x = block_e(sd, "Mixed_7b", x, lambda t: _avg(t, fid))
    x = block_e(sd, "Mixed_7c", x, (lambda t: F.max_pool2d(t, 3, stride=1, padding=1)) if fid else
                (lambda t: _avg(t, False)))
    return x.mean((2, 3))


def detector_input(images):
    """clean-fid's normalisation of [0, 255] images: x1 = x - 128, x2 = x1 / 128."""
    return (images - 128) / 128


def random_state_dict(seed=0, dtype=torch.float32):
    """He-scaled random conv weights and non-trivial BatchNorm statistics under torchvision's Inception3 key names
    (aux_logits off, without fc.* and num_batches_tracked)."""
    from torchvision.models import inception_v3
    net = inception_v3(weights=None, aux_logits=False, init_weights=False, num_classes=1008)
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, v in net.state_dict().items():
        if k.startswith("fc.") or k.endswith("num_batches_tracked"):
            continue
        if k.endswith("conv.weight"):
            fan_in = v[0].numel()
            t = torch.randn(v.shape, generator=g, dtype=torch.float64) * (2.0 / fan_in) ** 0.5
        elif k.endswith("bn.weight"):
            t = 0.5 + torch.rand(v.shape, generator=g, dtype=torch.float64)
        elif k.endswith("bn.bias"):
            t = 0.2 * torch.randn(v.shape, generator=g, dtype=torch.float64)
        elif k.endswith("running_mean"):
            t = 0.2 * torch.randn(v.shape, generator=g, dtype=torch.float64)
        else:
            t = 0.5 + torch.rand(v.shape, generator=g, dtype=torch.float64)
        sd[k] = t.to(dtype)
    return sd
