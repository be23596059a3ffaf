#!/usr/bin/env python3
"""Times the native FID / KID pieces on one GPU and prints one JSON line (GPU name and power limit included):

  - Inception pool3 features, native bf16 and fp32: images/s and TFLOP/s from the per-layer multiply-adds (computed
    from the shapes below), against torchvision's inception_v3 in fp32 (TF32 off) and in bf16 channels-last;
  - ds_feature_stats at n = 5000 and 50000 (d = 2048);
  - KID, 100 subsets of m = 1000: ds_kid_terms against clean-fid's float32 numpy expression on the host;
  - the host trace term: scipy.linalg.sqrtm of the product against the eigen form (n = 1000 features);
  - host decode + clean resize of 256 x 256 PNGs, images/s per thread count.

Random weights and synthetic inputs: nothing is read from outside the repository.

    python scripts/bench_fid.py [--batch 64] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from diffuscene_b200 import fid as F  # noqa: E402
from oracle import fid_ref as R  # noqa: E402
from oracle import inception_ref as IR  # noqa: E402
from tests.cases_fid import conv_geometries, render_like  # noqa: E402


def macs_per_image():
    """Multiply-adds of the 94 convolutions at 299 x 299 (pools and the global average left out)."""
    total = 0
    for cin, cout, kh, kw, st, ph, pw, H, W in conv_geometries()[0]:
        Ho, Wo = (H + 2 * ph - kh) // st + 1, (W + 2 * pw - kw) // st + 1
        total += Ho * Wo * cout * cin * kh * kw
    return total


def cuda_time(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / iters


def host_time(fn, warmup=True):
    """Seconds of one call (after one untimed call when `warmup`)."""
    if warmup:
        fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--batch", type=int, default=64)
    p.add_argument("--out", type=str, default=None)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fid.py needs a GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res = {"gpu": q[0] if q else "unknown", "batch": a.batch}
    macs = macs_per_image()
    res["gmacs_per_image"] = macs / 1e9
    sd = IR.random_state_dict(seed=0)
    B = a.batch
    imgs = torch.rand(B, 3, 299, 299, device="cuda") * 255
    for prec in ("bf16", "fp32"):
        m = F.InceptionFeatures(sd, precision=prec, capacity=B if prec == "bf16" else 8)
        t = cuda_time(lambda: m(imgs), 5 if prec == "bf16" else 2)
        res["native_%s" % prec] = {"images_per_s": B / t, "tflops": 2 * macs * B / t / 1e12}
        m.close()

    from torchvision.models import inception_v3
    net = inception_v3(weights=None, aux_logits=False, init_weights=False, num_classes=1008).cuda().eval()
    net.fc = torch.nn.Identity()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    with torch.no_grad():
        x = (imgs - 128) / 128
        t = cuda_time(lambda: net(x), 3)
        res["torchvision_fp32"] = {"images_per_s": B / t, "tflops": 2 * macs * B / t / 1e12}
        net16 = net.to(torch.bfloat16).to(memory_format=torch.channels_last)
        x16 = x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        t = cuda_time(lambda: net16(x16), 5)
        res["torchvision_bf16_cl"] = {"images_per_s": B / t, "tflops": 2 * macs * B / t / 1e12}
    del net, net16

    for n in (5000, 50000):
        f = torch.rand(n, 2048, device="cuda")
        t = cuda_time(lambda: F.feature_stats(f), 2)
        res["feature_stats_n%d_s" % n] = t

    rng = np.random.default_rng(0)
    real = rng.random((5000, 2048), dtype=np.float32)
    fake = rng.random((5000, 2048), dtype=np.float32)
    np.random.seed(0)
    ix, iy = F.kid_subsets(5000, 5000, 100, 1000)
    rd, fd = torch.from_numpy(real).cuda(), torch.from_numpy(fake).cuda()
    res["kid_native_s"] = host_time(lambda: F.kid_terms(rd, fd, ix, iy))
    res["kid_host_f32_s"] = host_time(lambda: R.kid_terms_f32(real, fake, ix, iy))

    from scipy import linalg
    fr = rng.standard_normal((1000, 2048))
    ff = rng.standard_normal((1000, 2048)) * 1.1
    s1, s2 = np.cov(fr, rowvar=False), np.cov(ff, rowvar=False)
    res["trace_sqrtm_s"] = host_time(lambda: linalg.sqrtm(s1.dot(s2)), False)
    res["trace_eigen_s"] = host_time(lambda: F.trace_sqrt_product(s1, s2), False)

    with tempfile.TemporaryDirectory() as d:
        files = []
        for i in range(128):
            files.append(os.path.join(d, "%d.png" % i))
            render_like(i).save(files[-1])
        dec = {}
        for th in (1, 4, 8):
            with ThreadPoolExecutor(th) as pool:
                t = host_time(lambda: list(pool.map(F.clean_resize, files)), False)
            dec[str(th)] = len(files) / t
        res["decode_resize_images_per_s"] = dec

    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
