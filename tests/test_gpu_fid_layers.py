"""GPU: each of the 43 distinct convolution geometries of the FID Inception-v3 alone (ds_inception_test_conv, the
kernels ds_inception_features runs) against fp64 F.conv2d + ReLU of the same operands, in bf16 and fp32; a write into
a concatenation slice whose neighbouring channels hold sentinels; and the C ABI's error cases."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from diffuscene_b200 import capi
from tests.cases_fid import conv_geometries

pytestmark = pytest.mark.gpu
GEOMS = conv_geometries()[1]
# bf16: |got - want| <= 2^-8 |want| (the output's rounding) + 2^-10 RMS(want) (fp32 accumulation), as the VGG16 layer
# test; fp32: 1e-5 |want| + 1e-5 RMS(want)
BOUNDS = {"bf16": (2.0 ** -8, 2.0 ** -10), "fp32": (1e-5, 1e-5)}


def run_conv(prec, x, w, b, stride, ph, pw, out, pitch, off):
    lib = capi.load()
    B, H, W, cin = x.shape
    cout, _, kh, kw = w.shape
    s = torch.cuda.current_stream()
    return lib.ds_inception_test_conv(prec, C.c_void_p(x.data_ptr()), B, H, W, cin, cout, kh, kw, stride, ph, pw,
                                      C.c_void_p(w.data_ptr()), C.c_void_p(b.data_ptr()), C.c_void_p(out.data_ptr()),
                                      pitch, off, C.c_void_p(s.cuda_stream))


def operands(g, seed):
    cin, cout, kh, kw, st, ph, pw, H, W = g
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(2, H, W, cin, generator=gen).abs()
    w = torch.randn(cout, cin, kh, kw, generator=gen) * (2.0 / (kh * kw * cin)) ** 0.5
    b = torch.randn(cout, generator=gen) * 0.05
    return x.cuda(), w.cuda(), b.cuda()


def reference(x, w, b, st, ph, pw, bf16):
    r = (lambda t: t.to(torch.bfloat16).double()) if bf16 else (lambda t: t.double())
    y = TF.conv2d(r(x).permute(0, 3, 1, 2), r(w), b.double(), stride=st, padding=(ph, pw))
    return TF.relu(y).permute(0, 2, 3, 1)


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("g", GEOMS, ids=["x".join(map(str, g)) for g in GEOMS])
def test_conv_geometry_against_fp64(g, prec):
    cin, cout, kh, kw, st, ph, pw, H, W = g
    x, w, b = operands(g, sum(g))
    want = reference(x, w, b, st, ph, pw, prec == "bf16")
    out = torch.zeros(want.shape, device="cuda", dtype=torch.float32)
    assert run_conv(capi.DS_PREC_BF16 if prec == "bf16" else capi.DS_PREC_FP32, x, w, b, st, ph, pw, out, cout, 0) == 0
    rel, rms = BOUNDS[prec]
    bound = rel * want.abs() + rms * want.pow(2).mean().sqrt()
    ratio = ((out.double() - want).abs() / bound).max().item()
    print("%s %s: err / bound = %.3f" % (prec, g, ratio))
    assert ratio <= 1.0


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("cout,off,pitch,g", [(64, 224, 288, (288, 64, 1, 1, 1, 0, 0, 35, 35)),
                                               (48, 64, 288, (48, 48, 5, 5, 1, 2, 2, 35, 35)),
                                               (96, 384, 768, (288, 96, 3, 3, 2, 0, 0, 35, 35)),
                                               (192, 1856, 2048, (1280, 192, 1, 1, 1, 0, 0, 8, 8))])
def test_concat_slice_keeps_neighbours(cout, off, pitch, g, prec):
    cin, _, kh, kw, st, ph, pw, H, W = g
    x, w, b = operands((cin, cout, kh, kw, st, ph, pw, H, W), cout + off)
    want = reference(x, w, b, st, ph, pw, prec == "bf16")
    out = torch.full(want.shape[:3] + (pitch,), -3.5, device="cuda")
    assert run_conv(capi.DS_PREC_BF16 if prec == "bf16" else capi.DS_PREC_FP32, x, w, b, st, ph, pw, out, pitch,
                    off) == 0
    assert (out[..., :off] == -3.5).all() and (out[..., off + cout:] == -3.5).all()
    rel, rms = BOUNDS[prec]
    bound = rel * want.abs() + rms * want.pow(2).mean().sqrt()
    assert ((out[..., off:off + cout].double() - want).abs() <= bound).all()


def test_abi_errors():
    lib = capi.load()
    null = None
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    cfg = capi.DsInceptionConfig()
    h = C.c_void_p()
    cfg.precision, cfg.capacity = 7, 1
    assert lib.ds_inception_create(C.byref(cfg), C.byref(h)) == -1
    cfg.precision, cfg.capacity = capi.DS_PREC_FP32, 0
    assert lib.ds_inception_create(C.byref(cfg), C.byref(h)) == -1
    cfg.capacity = 2
    assert lib.ds_inception_create(null, C.byref(h)) == -1
    assert lib.ds_inception_create(C.byref(cfg), C.byref(h)) == 0
    try:
        img = torch.zeros(1, 3, 299, 299, device="cuda")
        feat = torch.zeros(1, 2048, device="cuda")
        p = lambda t: C.c_void_p(t.data_ptr())      # noqa: E731
        assert lib.ds_inception_features(h, p(img), 1, 299, 299, p(feat), s) == -4       # before set_weights
        flat = torch.zeros(10, device="cuda")
        assert lib.ds_inception_set_weights(h, p(flat), 10, s) == -1                     # count mismatch
        assert lib.ds_inception_set_weights(h, null, 10, s) == -1
        total = sum(capi_numel(lib, h))
        flat = torch.ones(total, device="cuda")
        assert lib.ds_inception_set_weights(h, p(flat), total, s) == 0
        img298 = torch.zeros(1, 3, 298, 298, device="cuda")
        assert lib.ds_inception_features(h, p(img298), 1, 298, 298, p(feat), s) == -1
        assert lib.ds_inception_features(h, p(img), -1, 299, 299, p(feat), s) == -1
        assert lib.ds_inception_features(h, null, 1, 299, 299, p(feat), s) == -1
        assert lib.ds_inception_features(h, p(img), 1, 299, 299, p(feat), s) == 0
        name, numel = C.c_char_p(), C.c_int64()
        assert lib.ds_inception_expected_weight(h, 470, C.byref(name), C.byref(numel)) == -1
        assert lib.ds_inception_expected_weight(h, 0, null, C.byref(numel)) == -1
    finally:
        lib.ds_inception_destroy(h)
    f = torch.zeros(4, 8, device="cuda")
    mu = torch.zeros(8, device="cuda", dtype=torch.float64)
    cov = torch.zeros(8, 8, device="cuda", dtype=torch.float64)
    p = lambda t: C.c_void_p(t.data_ptr())      # noqa: E731
    assert lib.ds_feature_stats(p(f), 1, 8, p(mu), p(cov), s) == -1
    assert lib.ds_feature_stats(null, 4, 8, p(mu), p(cov), s) == -1
    assert lib.ds_feature_stats(p(f), 4, 8, p(mu), p(cov), s) == 0
    idx = torch.tensor([[0, 1, 2]], device="cuda", dtype=torch.int64)
    bad = torch.tensor([[0, 1, 4]], device="cuda", dtype=torch.int64)
    neg = torch.tensor([[0, -1, 2]], device="cuda", dtype=torch.int64)
    t = torch.zeros(1, device="cuda", dtype=torch.float64)
    assert lib.ds_kid_terms(p(f), 4, p(f), 4, 8, p(idx), p(idx), 1, 3, p(t), s) == 0
    assert lib.ds_kid_terms(p(f), 4, p(f), 4, 8, p(bad), p(idx), 1, 3, p(t), s) == -1
    assert lib.ds_kid_terms(p(f), 4, p(f), 4, 8, p(idx), p(neg), 1, 3, p(t), s) == -1
    assert lib.ds_kid_terms(p(f), 4, p(f), 4, 8, p(idx), p(idx), 1, 1, p(t), s) == -1
    assert lib.ds_kid_terms(p(f), 4, p(f), 2, 8, p(idx), p(idx), 1, 3, p(t), s) == -1
    assert lib.ds_kid_terms(p(f), 4, p(f), 4, 8, null, p(idx), 1, 3, p(t), s) == -1
    x = torch.zeros(1, 8, 8, 16, device="cuda")
    w = torch.zeros(8, 16, 3, 3, device="cuda")
    b = torch.zeros(8, device="cuda")
    o = torch.zeros(1, 8, 8, 8, device="cuda")
    assert run_conv(capi.DS_PREC_BF16, x, w, b, 1, 1, 1, o, 8, 0) == 0
    assert run_conv(capi.DS_PREC_BF16, x, w, b, 1, 1, 1, o, 8, 4) == -1      # slice past the pitch
    assert run_conv(9, x, w, b, 1, 1, 1, o, 8, 0) == -1


def capi_numel(lib, h):
    out = []
    for i in range(lib.ds_inception_expected_weight_count(h)):
        name, numel = C.c_char_p(), C.c_int64()
        assert lib.ds_inception_expected_weight(h, i, C.byref(name), C.byref(numel)) == 0
        out.append(numel.value)
    return out
