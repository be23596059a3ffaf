"""GPU: each bf16 VGG16 convolution alone (ds_vgg_test_conv, the kernel ds_vgg_features runs) against fp64
F.conv2d + ReLU (+ max_pool2d) of the same bf16-rounded input and weights, at every VGG16 channel width and
spatial size, with and without the fused pool, plus partial tiles; near-duplicate realism; the library defaults."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from diffuscene_b200 import capi
from diffuscene_b200 import ipr as I
from tests.cases_ipr import clustered, he_state_dict

pytestmark = pytest.mark.gpu

# (cin, cout, H, W, pool): the 13 layers of VGG16 as the network runs them, then partial 8 x 16 tiles for both output
# widths, with and without the pool, and non-square images
LAYERS = [(3, 64, 224, 224, 0), (64, 64, 224, 224, 1), (64, 128, 112, 112, 0), (128, 128, 112, 112, 1),
          (128, 256, 56, 56, 0), (256, 256, 56, 56, 0), (256, 256, 56, 56, 1), (256, 512, 28, 28, 0),
          (512, 512, 28, 28, 0), (512, 512, 28, 28, 1), (512, 512, 14, 14, 0), (512, 512, 14, 14, 1),
          (3, 64, 14, 14, 0), (64, 64, 14, 14, 1), (64, 64, 28, 28, 0), (128, 128, 14, 14, 0), (64, 128, 56, 56, 1),
          (512, 512, 7, 7, 0), (128, 256, 20, 36, 1), (64, 64, 18, 50, 0)]
# |got - want| <= 2^-8 |want| (the output's bf16 rounding) + BOUND_RMS x RMS(want) (fp32 accumulation over up to
# 4608 products).  The worst ratio of error to bound measured on one H100 80GB HBM3 was 0.92 (64 -> 64 channels,
# 28 x 28); the test prints each layer's ratio
BOUND_RMS = 2.0 ** -10


def bf16_round(t):
    return t.to(torch.bfloat16).to(torch.float64)


@pytest.mark.parametrize("cin,cout,H,W,pool", LAYERS)
def test_conv_layer_against_fp64(cin, cout, H, W, pool):
    g = torch.Generator().manual_seed(cin * 7 + cout + H * 3 + W + pool)
    B = 2
    x = torch.randn(B, H, W, cin, generator=g).abs() if cin > 3 else torch.randn(B, H, W, cin, generator=g)
    w = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (9 * cin)) ** 0.5
    b = torch.randn(cout, generator=g) * 0.05
    Ho, Wo = (H // 2, W // 2) if pool else (H, W)
    out = torch.full((B, Ho, Wo, cout), float("nan"), device="cuda")
    xd, wd, bd = x.cuda().contiguous(), w.cuda().contiguous(), b.cuda()
    lib = capi.load()
    capi.check(lib.ds_vgg_test_conv(C.c_void_p(xd.data_ptr()), B, H, W, cin, cout, pool, C.c_void_p(wd.data_ptr()),
                                    C.c_void_p(bd.data_ptr()), C.c_void_p(out.data_ptr()), None))
    want = F.relu(F.conv2d(bf16_round(x).permute(0, 3, 1, 2), bf16_round(w), b.double(), padding=1))
    if pool:
        want = F.max_pool2d(want, 2, 2)
    want = want.permute(0, 2, 3, 1)
    got = out.cpu().double()
    assert torch.isfinite(got).all()                                  # every output written
    bound = 2.0 ** -8 * want.abs() + BOUND_RMS * want.pow(2).mean().sqrt()
    ratio = ((got - want).abs() / bound).max().item()
    print("conv %d->%d %dx%d pool=%d: max error / bound %.3f" % (cin, cout, H, W, pool, ratio))
    assert ratio <= 1.0


def test_test_conv_rejects_bad_geometry():
    lib = capi.load()
    t = torch.zeros(64, device="cuda")
    p = C.c_void_p(t.data_ptr())
    assert lib.ds_vgg_test_conv(p, 1, 8, 8, 32, 64, 0, p, p, p, None) == -1      # cin not 3 / multiple of 64
    assert lib.ds_vgg_test_conv(p, 1, 8, 8, 64, 96, 0, p, p, p, None) == -1      # cout not 64 / multiple of 128
    assert lib.ds_vgg_test_conv(p, 1, 7, 8, 64, 64, 1, p, p, p, None) == -1      # odd pooled side
    assert lib.ds_vgg_test_conv(None, 1, 8, 8, 64, 64, 0, p, p, p, None) == -1


def test_realism_of_near_duplicates_uses_the_difference():
    """A subject equal (or within 1e-9) to a real feature: the reference's norm(real_i - f) is ~0, so realism is
    about radius / 1e-6; the expansion |x|^2 - 2 x.y + |y|^2 alone would leave sqrt(rounding) ~ 1e-6 .. 1e-5."""
    real = clustered(300, 4096, seed=8, centre_seed=0).astype(np.float64) * 4      # |x|^2 ~ 1e5
    radii = I.manifold_radii(real, 3)
    rng = np.random.default_rng(9)
    subj = np.concatenate([real[:5], real[5:10] + rng.normal(0, 1e-9, (5, 4096)), clustered(5, 4096, seed=10) * 4])
    _, _, got = I.manifold_cover(I.Manifold(real, radii), subj, want_realism=True)
    d = np.linalg.norm(real[None, :, :] - subj[:, None, :], axis=2)               # [subjects, real], direct
    want = (radii[None, :] / (d + 1e-6)).max(axis=1)
    np.testing.assert_allclose(got, want, rtol=1e-6)
    assert (got[:5] > 1e6 * radii[:5] * 0.5).all()


def test_defaults_are_fp32_and_accept_a_module():
    sd = he_state_dict(seed=2)
    m = torch.nn.Module()
    for n, v in sd.items():                                   # a module whose state_dict() is the vgg16 one
        m.register_buffer(n.replace(".", "_"), v)
    m.state_dict = lambda: sd
    net = I.VGG16Features(m)
    assert net.precision == "fp32"
    with pytest.raises(TypeError):
        I.VGG16Features(3.0)
    ipr = I.IPR(model=net)
    assert ipr.vgg16.precision == "fp32"
    net.close()
