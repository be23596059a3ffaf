"""Throughput of the variational bound (`diffusion.all_kl`) against sampling on the same engine and batch.

    python scripts/bench_vlb.py [--batch 4096] [--windows 3] [--precision bf16]

Workload: the shipped bedroom config (config/uncond/diffusion_bedrooms_instancond_lat32_v.yaml: N = 12, d = 62,
T = 1000, v-prediction, fixedsmall), random-init weights, synthetic clean scenes.  One all_kl window is one full
calc_bpd_loop (T denoiser forwards plus the VLB terms of every scene at every t, Philox q_sample draws); one sampling
window is one full 1000-step `DenoiserEngine.sample` of the same batch on the same engine, the natural ceiling since
each VLB step also runs one forward.  Windows of the two alternate after one warm-up call of each, and are bracketed
by CUDA events after a device synchronise.  Prints one JSON line; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_identity():
    name = torch.cuda.get_device_name(torch.cuda.current_device())
    try:
        idx = str(torch.cuda.current_device())
        out = subprocess.run(["nvidia-smi", "-i", idx, "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = None
    return name, out or None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--windows", type=int, default=3, help="timed windows per path (alternating)")
    ap.add_argument("--precision", default="bf16", choices=["bf16", "fp32"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vlb.py measures on a CUDA device; none is available")
    import yaml
    from scene_synthesis.networks import build_network

    B, N, d = args.batch, 12, 62
    cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "uncond", "diffusion_bedrooms_instancond_lat32_v.yaml")))
    cfg["network"]["diffusion_kwargs"]["loss_iou"] = False       # training-only; no stats file needed
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    net, _, _ = build_network(30, 23, cfg, None, device=dev, precision=args.precision)
    net.eval()
    T = net.time_num

    g = torch.Generator().manual_seed(1)
    cls = torch.randint(0, 22, (B, N), generator=g)
    x0 = torch.cat([torch.rand(B, N, 6, generator=g) * 2 - 1,
                    torch.nn.functional.normalize(torch.randn(B, N, 2, generator=g), dim=-1),
                    torch.nn.functional.one_hot(cls, 22).float() * 2 - 1,
                    torch.rand(B, N, 32, generator=g) * 2 - 1], dim=-1).to(dev)
    assert x0.shape == (B, N, d)
    with torch.no_grad():
        cond, shared = net._condition(B, dev)
    assert shared and cond.shape[0] == N
    eng = net.engine()
    last = {}

    def run(kind, k):
        if kind == "all_kl":
            last[kind] = net.diffusion.all_kl(x0, cond, None, clip_denoised=True, seed=100 + k)
        else:
            last[kind] = eng.sample(B, clip_denoised=True, seed=200 + k)

    def window(kind, k):
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run(kind, k)
        e1.record()
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1)

    kinds = ("all_kl", "sample")
    for kind in kinds:
        window(kind, -1)
    ms = {k: [] for k in kinds}
    for w in range(args.windows):
        for kind in kinds:
            ms[kind].append(window(kind, w))
    vals = {k: float(v) for k, v in last["all_kl"].items()}
    assert all(torch.isfinite(torch.tensor(v)) for v in vals.values()), vals
    gpu, power = gpu_identity()
    med = {k: statistics.median(v) for k, v in ms.items()}
    print(json.dumps({
        "metric": "variational bound (all_kl) scenes/s, median of windows", "unit": "scenes/s",
        "all_kl_scenes_per_s": B / (med["all_kl"] / 1000.0), "all_kl_ms_per_timestep": med["all_kl"] / T,
        "sample_scenes_per_s": B / (med["sample"] / 1000.0), "sample_ms_per_timestep": med["sample"] / T,
        "all_kl_over_sample": med["sample"] / med["all_kl"],
        "all_kl_windows_ms": ms["all_kl"], "sample_windows_ms": ms["sample"], "last_all_kl": vals,
        "config": {"workload": "bedroom N=12 d=62, T=%d, v-prediction, fixedsmall, random-init weights, synthetic "
                               "scenes, clip_denoised" % T, "precision": args.precision, "scenes": B,
                   "windows": args.windows, "warmup": "one call of each"},
        "gpu": gpu, "power_limit": power}))


if __name__ == "__main__":
    main()
