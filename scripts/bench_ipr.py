#!/usr/bin/env python3
"""Improved precision and recall timings on one GPU: VGG16 feature extraction (native bf16 / fp32 against a plain
torch.nn VGG16 in fp32 and in bf16 channels-last), the manifold metrics (native fp64 against the reference's numpy
fp64 computation where its N x N matrices fit), and host PNG decode + resize on its own.  Prints one JSON line per
measurement and a summary; the card's name and power limit are part of the output.

    python scripts/bench_ipr.py [--batch 64] [--sizes 5000,20000,50000] [--numpy_max 5000] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C  # noqa: E402

from diffuscene_b200 import capi  # noqa: E402
from diffuscene_b200 import ipr as I  # noqa: E402
from oracle.vgg16_ref import CHANNELS, CONV_IDX, POOL_AFTER  # noqa: E402
from tests.cases_ipr import clustered, he_state_dict, normalise, render_like  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:      # the numbers still carry the torch device name
        return "%s (power limit unknown: %s)" % (torch.cuda.get_device_name(), e)


def vgg_flops_per_image():
    f, hw, cin = [], 224, 3
    for l, cout in enumerate(CHANNELS):
        f.append(2.0 * hw * hw * cout * cin * 9)
        cin = cout
        if l + 1 in POOL_AFTER:
            hw //= 2
    return f + [2.0 * 25088 * 4096, 2.0 * 4096 * 4096]


def torch_vgg(sd):
    layers, cin = [], 3
    for l, (i, cout) in enumerate(zip(CONV_IDX, CHANNELS)):
        layers += [nn.Conv2d(cin, cout, 3, padding=1), nn.ReLU(inplace=True)]
        if l + 1 in POOL_AFTER:
            layers.append(nn.MaxPool2d(2, 2))
        cin = cout
    features = nn.Sequential(*layers)
    fc = nn.Sequential(nn.Linear(25088, 4096), nn.ReLU(inplace=True), nn.Linear(4096, 4096))
    convs = [m for m in features if isinstance(m, nn.Conv2d)]
    for m, i in zip(convs, CONV_IDX):
        m.weight.data.copy_(sd["features.%d.weight" % i])
        m.bias.data.copy_(sd["features.%d.bias" % i])
    for m, i in zip((fc[0], fc[2]), (0, 3)):
        m.weight.data.copy_(sd["classifier.%d.weight" % i])
        m.bias.data.copy_(sd["classifier.%d.bias" % i])
    return features.cuda().eval(), fc.cuda().eval()


def cuda_ms(fn, iters, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernel_share(fn, names):
    """Share of device time spent in kernels whose name contains one of `names` (torch.profiler, separate run)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = part = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        if getattr(e, "device_type", None) is not None and "CUDA" not in str(e.device_type):
            continue
        tot += t
        if any(n in e.key for n in names):
            part += t
    return part / tot if tot else float("nan")


def reference_numpy(real, fake, k):
    """The reference's computation: three dense fp64 N x N matrices, argpartition per row, a loop per subject."""
    def dist(X, Y=None):
        X = X.astype(np.float64)
        xx = np.sum(X ** 2, axis=1, keepdims=True)
        yy = xx if Y is None else np.sum(Y ** 2, axis=1, keepdims=True)
        Y = X if Y is None else Y
        d2 = np.repeat(xx, Y.shape[0], 1) - 2 * np.dot(X, Y.T) + np.repeat(yy.T, X.shape[0], 0)
        d2[d2 < 0] = 0
        return np.sqrt(d2)

    def radii(d):
        return np.array([row[np.argpartition(row, k + 1)[:k + 1]].max() for row in d])

    def metric(ref, rr, subj):
        d = dist(ref, subj)
        return sum((d[:, i] < rr).any() for i in range(subj.shape[0])) / subj.shape[0]

    r_real, r_fake = radii(dist(real)), radii(dist(fake))
    return metric(real, r_real, fake), metric(fake, r_fake, real)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--sizes", default="5000,20000,50000")
    ap.add_argument("--numpy_max", type=int, default=5000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--decode_images", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ipr.py measures on a GPU"
    torch.backends.cudnn.benchmark = True
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    rows = []

    def emit(**kw):
        kw["card"] = CARD
        rows.append(kw)
        print(json.dumps(kw), flush=True)

    CARD = card()
    sd = he_state_dict(seed=1)
    x = normalise(render_like(a.batch, 224, seed=3)).cuda()
    flops = vgg_flops_per_image()
    fl_img = sum(flops)
    with torch.no_grad():
        for prec in ("bf16", "fp32"):
            net = I.VGG16Features(sd, precision=prec, capacity=a.batch)
            ms = cuda_ms(lambda: net(x), a.iters, warmup=1)
            share = kernel_share(lambda: net(x), ["k_vgg_conv<64, false>", "k_vgg_conv<(int)64, (bool)0>",
                                                  "k_re_im2col"]) if prec == "bf16" else None
            emit(what="vgg16 features", impl="native " + prec, batch=a.batch, ms=ms, images_per_s=a.batch / ms * 1e3,
                 tflops=fl_img * a.batch / ms / 1e9, first_layer_share=share)
            net.close()
            del net
        features, fc = torch_vgg(sd)
        fwd = lambda xx: fc(features(xx).reshape(-1, 25088))
        ms = cuda_ms(lambda: fwd(x), 2, warmup=1)
        emit(what="vgg16 features", impl="torch.nn fp32", batch=a.batch, ms=ms, images_per_s=a.batch / ms * 1e3,
             tflops=fl_img * a.batch / ms / 1e9)
        features, fc = features.to(memory_format=torch.channels_last).bfloat16(), fc.bfloat16()
        xb = x.to(memory_format=torch.channels_last).bfloat16()
        ms = cuda_ms(lambda: fwd(xb), a.iters, warmup=2)
        emit(what="vgg16 features", impl="torch.nn bf16 channels-last", batch=a.batch, ms=ms,
             images_per_s=a.batch / ms * 1e3, tflops=fl_img * a.batch / ms / 1e9)
        del features, fc

    for n in [int(s) for s in a.sizes.split(",")]:
        real = clustered(n, 4096, clusters=64, seed=1, centre_seed=0)
        fake = clustered(n, 4096, clusters=64, seed=2, centre_seed=0)
        rd, fd = torch.from_numpy(real).cuda().double(), torch.from_numpy(fake).cuda().double()
        torch.cuda.synchronize()

        lib = capi.load()
        rr, rf = (torch.empty(n, device="cuda", dtype=torch.float64) for _ in range(2))
        pf, rcf = (torch.empty(n, device="cuda", dtype=torch.uint8) for _ in range(2))
        P = lambda t: C.c_void_p(t.data_ptr())

        def native():
            capi.check(lib.ds_manifold_radii(P(rd), n, 4096, 3, P(rr), None, None))
            capi.check(lib.ds_manifold_radii(P(fd), n, 4096, 3, P(rf), None, None))
            capi.check(lib.ds_manifold_cover(P(rd), P(rr), n, P(fd), P(rf), n, 4096, P(pf), P(rcf), None, None, None))

        times = sorted(cuda_ms(native, 1, warmup=1 if r == 0 else 0) for r in range(a.repeats))
        ms = times[len(times) // 2]
        emit(what="manifold metrics", impl="native fp64", n=n, d=4096, ms=ms, ms_min=times[0], ms_max=times[-1],
             repeats=a.repeats, precision=pf.float().mean().item(), recall=rcf.float().mean().item(),
             dmma_tflops=3 * 2.0 * n * n * 4096 / ms / 1e9, timing="CUDA events around the three calls, outputs on the device")
        if n <= a.numpy_max:
            t0 = time.perf_counter()
            p_ref = reference_numpy(real, fake, 3)
            emit(what="manifold metrics", impl="reference numpy fp64", n=n, d=4096,
                 ms=(time.perf_counter() - t0) * 1e3, precision=float(p_ref[0]), recall=float(p_ref[1]))
        else:
            emit(what="manifold metrics", impl="reference numpy fp64", n=n, d=4096, ms="not measured",
                 note="three %.1f GB matrices" % (n * n * 8 / 1e9))
        del rd, fd

    from PIL import Image
    with tempfile.TemporaryDirectory() as tmp:
        imgs = render_like(a.decode_images, 256, seed=9)
        files = []
        for i, im in enumerate(imgs):
            files.append(os.path.join(tmp, "%05d.png" % i))
            Image.fromarray(im).save(files[-1])
        from concurrent.futures import ThreadPoolExecutor
        for workers in (1, 4):
            with ThreadPoolExecutor(workers) as pool:
                list(pool.map(I.load_image, files[:8]))
                t0 = time.perf_counter()
                list(pool.map(I.load_image, files))
                s = time.perf_counter() - t0
            emit(what="host decode + resize", impl="PIL, %d threads" % workers, images=len(files),
                 images_per_s=len(files) / s)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
