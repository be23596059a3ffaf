"""Cost of batched scene evaluation (`diffuscene_b200.evaluate.evaluate_samples`) against sampling the same batch.

    python scripts/bench_scene_eval.py [--batch 4096] [--reps 20] [--oracle_scenes 4096]

Workloads: the shipped bedroom (N = 12, d = 62) and living-room (N = 21, d = 65) configs with random-init weights
in bf16.  Per config, one full 1000-step `sample()` of the batch is timed after one warm-up call; then the whole
evaluation chain on those samples (keep mask, post_process_batch, argmax, objfeats retrieval from a synthetic
catalogue of 2000 models with xz-hull footprints, boxes and statistics) and the two evaluation kernels alone
(ds_scene_boxes + ds_scene_stats), each as the median of `--reps` calls bracketed by CUDA events after a warm-up.
The CPU arm is the numpy oracle's per-scene loop over the same placed bounds (oracle/scene_eval_ref.py: the
statistics only; mesh loading, which dominates the reference's own cost, is not measured).  Prints one JSON line per
config; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_vlb import gpu_identity  # noqa: E402


def timed(fn, reps, dev):
    fn()
    ms = []
    for _ in range(reps):
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize(dev)
        ms.append(e0.elapsed_time(e1))
    return statistics.median(ms), ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--oracle_scenes", type=int, default=4096)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_scene_eval.py measures on a CUDA device; none is available")
    import yaml
    from scene_synthesis.networks import build_network
    from diffuscene_b200 import evaluate as E
    from diffuscene_b200.postprocess import ObjectCatalog, post_process_batch
    from diffuscene_b200.synthetic import DEFAULT_BOUNDS
    from oracle import scene_eval_ref as R
    from tests.cases_scene_eval import random_mesh

    dev = torch.device("cuda", torch.cuda.current_device())
    B = args.batch
    bounds = dict(DEFAULT_BOUNDS, objfeats=DEFAULT_BOUNDS["objfeats_32"])
    gpu, power = gpu_identity()
    for name in ("diffusion_bedrooms_instancond_lat32_v", "diffusion_livingrooms_instancond_lat32_v"):
        cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "uncond", name + ".yaml")))
        cfg["network"]["diffusion_kwargs"]["loss_iou"] = False
        N, d = cfg["network"]["sample_num_points"], cfg["network"]["point_dim"]
        torch.manual_seed(0)
        net, _, _ = build_network(30, cfg["network"]["class_dim"] + 1, cfg, None, device=dev, precision="bf16")
        net.eval()
        room = torch.zeros(B, 1, 64, 64, device=dev)
        out = {}
        sample_ms, _ = timed(lambda: out.__setitem__("x", net.sample(room, N, d, batch_size=B, clip_denoised=True,
                                                                      seed=7)), 1, dev)
        x = out["x"]
        rng = np.random.default_rng(0)
        M, n_cls = 2000, net.class_dim - 1
        meshes = [random_mesh(rng, 200) for _ in range(64)]
        fps = [E.model_footprint(*meshes[m % 64]) for m in range(M)]
        sizes = np.array([R.raw_half_sizes(meshes[m % 64][1]) for m in range(M)], np.float32)
        cat = ObjectCatalog(np.arange(M) % n_cls, rng.normal(size=(M, 32)).astype(np.float32), sizes,
                            n_classes=n_cls, footprints=E.footprint_table(fps))
        chain_ms, chain_all = timed(lambda: out.__setitem__("ev", E.evaluate_samples(net, x, bounds, cat, "objfeats")),
                                    args.reps, dev)
        ev = out["ev"]
        kp = ev["keep"]
        mid = cat.model_ids[ev["model_index"].clamp(min=0)]
        bb = net.bbox_dim
        w = post_process_batch({"translations": x[:, :, :3], "sizes": x[:, :, 3:6], "angles": x[:, :, 6:bb]}, bounds)
        kern_ms, _ = timed(lambda: E.scene_stats(E.scene_boxes(w["translations"], w["sizes"], w["angles"],
                                                               ev["model_index"], cat), ev["class_index"], kp, mid),
                           args.reps, dev)
        bh, kh, ch, mh = (t.cpu().numpy() for t in (ev["bounds"], kp, ev["class_index"], mid))
        S = min(args.oracle_scenes, B)
        t0 = time.perf_counter()
        for b in range(S):
            k = kh[b]
            R.evaluate_scene(bh[b][k], ch[b][k], mh[b][k])
        oracle_ms = (time.perf_counter() - t0) * 1000.0 * B / S
        print(json.dumps({
            "metric": "scene evaluation of one sampled batch, median CUDA-event time", "unit": "ms",
            "config": name, "scenes": B, "objects_per_scene": N, "kept_objects": int(kh.sum()),
            "sample_ms": sample_ms, "evaluate_samples_ms": chain_ms, "evaluate_samples_share_of_sample":
                chain_ms / sample_ms, "boxes_and_stats_kernels_ms": kern_ms,
            "numpy_oracle_stats_loop_ms": oracle_ms, "oracle_scenes_timed": S,
            "speedup_chain_vs_oracle_stats": oracle_ms / chain_ms, "evaluate_samples_windows_ms": chain_all,
            "precision": "bf16", "reps": args.reps, "gpu": gpu, "power_limit": power}))


if __name__ == "__main__":
    main()
