"""Object shape auto-encoder: native training step and encoding against the autograd twin.

    python scripts/bench_shape_ae.py [--batches 16 128] [--steps 5] [--warmup 2] [--windows 3] [--encode 4096]

Workload: config/obj_autoencoder/bedrooms_lat32.yaml (F = 32, P = 2048 points per object, the reference's dataset
size), random-init weights, seeded synthetic shapes (SyntheticShapes, drawn with replacement).  Measures, with CUDA
events around device-synchronised windows:
  - train_on_batch objects/s of the native model (`native_backward = True`: ds_shape_ae_train_step and NativeAdam)
    against the autograd twin (`native_backward = False`: torch topk kNN, cuDNN / cuBLAS convolutions in fp32 (TF32
    off), the torch Chamfer restatement, torch Adam), in alternating windows, at each --batches size (16 is the reference's);
  - eval-mode encoding of --encode objects (objects/s), native against the twin;
  - per-phase device milliseconds of one native training step at the first batch size, from torch.profiler kernel
    times grouped by kernel name (kNN, GEMMs, BatchNorm, Chamfer, the rest).
Prints one JSON line with the card's name and power limit.  Writes nothing into the repository.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_train_text import gpu_identity  # noqa: E402

PHASES = (("knn", ("k_sae_knn",)), ("gemm", ("k_gemm_simt", "k_gemm_nn", "k_gemm_tn", "k_colsum")),
          ("batchnorm", ("k_bn_",)), ("chamfer", ("k_chamfer",)), ("local_max", ("k_sae_nbr_max", "k_csr_")))


def timed(fn, reps, dev):
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize(dev)
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[16, 128])
    ap.add_argument("--steps", type=int, default=5, help="optimizer iterations per timed window")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--windows", type=int, default=3, help="timed windows per path (alternating)")
    ap.add_argument("--encode", type=int, default=4096)
    ap.add_argument("--encode-chunk", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_shape_ae.py measures on a CUDA device; none is available")
    from diffuscene_b200.optim import NativeAdam
    from diffuscene_b200.shape_ae import KLAutoEncoder
    from diffuscene_b200.synthetic import SyntheticShapes
    from scene_synthesis.networks.foldingnet_autoencoder import train_on_batch

    dev = torch.device("cuda", 0)
    # the twin is timed in fp32 like the native path (torch would otherwise run cuDNN convolutions in TF32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    P, F = 2048, 32
    config = {"training": {"max_grad_norm": 10.0}}
    torch.manual_seed(0)
    proto = KLAutoEncoder(latent_dim=F, num_points=P)
    result = {"metric": "shape_ae", "gpu": gpu_identity(), "P": P, "F": F, "train": {}}
    ds = SyntheticShapes(max(args.batches + [args.encode_chunk]), P, seed=1)
    pool = torch.stack([ds[i]["points"] for i in range(len(ds))]).to(dev)

    def make(native):
        m = KLAutoEncoder(latent_dim=F, num_points=P)
        m.load_state_dict(proto.state_dict())
        m.native_backward = native
        m.to(dev).train()
        opt = NativeAdam(m.parameters(), lr=1e-4) if native else torch.optim.Adam(m.parameters(), lr=1e-4)
        return m, opt

    for B in args.batches:
        pts = pool[:B].contiguous()
        paths = {name: make(native) for name, native in (("native", True), ("twin", False))}
        step = {name: (lambda m=m, o=o: train_on_batch(m, o, {"points": pts}, config)) for name, (m, o) in paths.items()}
        for name in paths:
            timed(step[name], args.warmup, dev)
        ms = {name: [] for name in paths}
        for _ in range(args.windows):
            for name in paths:
                ms[name].append(timed(step[name], args.steps, dev))
        result["train"][str(B)] = {name: {"ms_per_step": round(statistics.median(v), 3),
                                          "objects_per_s": round(B * 1000.0 / statistics.median(v), 1),
                                          "windows_ms": [round(x, 3) for x in v]} for name, v in ms.items()}
        del paths, step
        torch.cuda.empty_cache()

    # eval-mode encoding
    enc = {}
    for name, native in (("native", True), ("twin", False)):
        m, _ = make(native)
        m.eval()
        chunk = pool[:args.encode_chunk].contiguous()
        n_chunks = (args.encode + args.encode_chunk - 1) // args.encode_chunk

        def encode_all(m=m):
            with torch.no_grad():
                for _ in range(n_chunks):
                    m.encode(chunk.permute(0, 2, 1))
        timed(encode_all, 1, dev)
        t = statistics.median(timed(encode_all, 1, dev) for _ in range(args.windows))
        enc[name] = {"ms": round(t, 2), "objects_per_s": round(n_chunks * args.encode_chunk * 1000.0 / t, 1)}
        del m
        torch.cuda.empty_cache()
    result["encode"] = dict(enc, objects=n_chunks * args.encode_chunk)

    # per-phase device time of one native training step (a profiled run of its own)
    B = args.batches[0]
    m, opt = make(True)
    pts = pool[:B].contiguous()
    for _ in range(2):
        train_on_batch(m, opt, {"points": pts}, config)
    torch.cuda.synchronize(dev)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        train_on_batch(m, opt, {"points": pts}, config)
        torch.cuda.synchronize(dev)
    phases = {k: 0.0 for k, _ in PHASES}
    phases["other"] = 0.0
    for ev in prof.key_averages():
        us = getattr(ev, "device_time_total", None)
        if us is None:
            us = getattr(ev, "cuda_time_total", 0.0)
        if not us:
            continue
        for k, keys in PHASES:
            if any(s in ev.key for s in keys):
                phases[k] += us / 1000.0
                break
        else:
            phases["other"] += us / 1000.0
    result["phases_ms_B%d" % B] = {k: round(v, 3) for k, v in phases.items()}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
