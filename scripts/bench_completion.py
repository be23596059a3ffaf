#!/usr/bin/env python3
"""Times scene completion and rearrangement of B real-layout scenes on one GPU (the steps of
scripts/completion_rearrange.py) and prints one JSON line, GPU name and power limit included:

  - sampling: network.sample(partial_boxes=...) (uncond config, 3 partial objects) or sample(input_boxes=...)
    (rearrange config, noised inputs), full 1000-step DDPM, bf16, random weights;
  - retrieval + placement: evaluate.place_samples of the results against a 512-model catalogue;
  - renders: ds_render_scenes of the placed results, 512^2 perspective (REFERENCE_PERSPECTIVE) and 256^2 top-down;
  - the reference's loop: one scene per call (sample, place, perspective render), timed over --loop_scenes scenes and
    given per scene.

Scenes are seeded synthetic rooms (diffuscene_b200.synthetic_meshes); nothing is read from outside the tree.

    python scripts/bench_completion.py [--batches 512,4096] [--loop_scenes 4] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from completion_rearrange import encode_scenes  # noqa: E402
from training_utils import load_config  # noqa: E402

from scene_synthesis.networks import build_network  # noqa: E402
from diffuscene_b200 import render as R, synthetic_meshes as SM  # noqa: E402
from diffuscene_b200.evaluate import place_samples  # noqa: E402
from diffuscene_b200.postprocess import ObjectCatalog  # noqa: E402
from diffuscene_b200.synthetic import DEFAULT_BOUNDS, SyntheticScenes  # noqa: E402

CFG = {"complete": os.path.join(os.path.dirname(HERE), "config", "uncond", "diffusion_bedrooms_instancond_lat32_v.yaml"),
       "arrange": os.path.join(os.path.dirname(HERE), "config", "rearrange",
                               "diffusion_bedrooms_instancond_lat32_v_rearrange.yaml")}


def sync_time(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def rooms(B, M, seed):
    sc = SM.scenes(B, 8, M, seed=seed, empty=0.0)
    out = []
    for b in range(B):
        n = 4 + b % 5
        cl = np.zeros((n, 23), np.float32)
        cl[np.arange(n), sc["class_index"][b, :n]] = 1
        out.append({"class_labels": cl, "translations": sc["translations"][b, :n], "sizes": sc["sizes"][b, :n],
                    "angles": sc["angles"][b, :n]})
    return out, sc["floors"]


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("--batches", default="512,4096")
    p.add_argument("--loop_scenes", type=int, default=4)
    p.add_argument("--models", type=int, default=512)
    p.add_argument("--out", default=None)
    a = p.parse_args(argv)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res = {"gpu": q[0] if q else "unknown"}
    dev = torch.device("cuda:0")
    M = a.models
    meshes = R.MeshCatalog(SM.catalogue(seed=0, num_models=M, detail=2, texture_size=64))
    rng = np.random.default_rng(0)
    cat = ObjectCatalog(np.arange(M) % 21, rng.normal(size=(M, 32)).astype(np.float32),
                        rng.uniform(0.2, 0.8, (M, 3)).astype(np.float32), n_classes=21)
    for task in ("complete", "arrange"):
        config = load_config(CFG[task])
        config["network"]["diffusion_kwargs"]["loss_iou"] = False
        ds = SyntheticScenes(config["network"], 1)
        torch.manual_seed(0)
        net, _, _ = build_network(ds.feature_size, ds.n_classes, config, None, device=dev, precision="bf16")
        net.eval()
        N, d = config["network"]["sample_num_points"], config["network"]["point_dim"]

        def sample(x, bs, seed):
            mask = torch.zeros(bs, 1, 64, 64, device=dev)
            if task == "arrange":
                return net.sample(mask, N, d, batch_size=bs, input_boxes=x, seed=seed)
            return net.sample(mask, N, d, batch_size=bs, partial_boxes=x[:, :3].contiguous(), seed=seed)

        for B in (int(v) for v in a.batches.split(",")):
            raw, floors = rooms(B, M, seed=B)
            x = encode_scenes(raw, N, DEFAULT_BOUNDS, 32).to(dev)
            if task == "arrange":
                x[..., :3] += torch.randn(B, N, 3, device=dev)
            fl = R.floor_triangles(floors)
            sample(x[:1], 1, 0)                                         # warm-up
            t_s, s = sync_time(lambda: sample(x, B, 1))
            t_p, placed = sync_time(lambda: place_samples(net, s, DEFAULT_BOUNDS, cat, "objfeats"))
            world, keep, cls, mi = placed
            mi = torch.where(keep, mi, -1)
            draw = lambda cam: R.render_scenes(meshes, world["translations"], world["sizes"], world["angles"], mi,
                                               cls, floors=fl, white_background=True, camera=cam)
            draw(R.REFERENCE_PERSPECTIVE); draw(R.Camera())             # warm-up
            t_rp, _ = sync_time(lambda: draw(R.REFERENCE_PERSPECTIVE))
            t_rt, _ = sync_time(lambda: draw(R.Camera()))
            key = "%s_%d" % (task, B)
            res[key] = {"sample_s": t_s, "retrieve_place_s": t_p, "render_perspective_512_s": t_rp,
                        "render_top2down_256_s": t_rt, "scenes_per_s": B / (t_s + t_p + t_rp)}
        # the reference's loop: one scene per call
        L = a.loop_scenes
        raw, floors = rooms(L, M, seed=7)
        x = encode_scenes(raw, N, DEFAULT_BOUNDS, 32).to(dev)

        def loop():
            for i in range(L):
                s = sample(x[i:i + 1], 1, i)
                world, keep, cls, mi = place_samples(net, s, DEFAULT_BOUNDS, cat, "objfeats")
                R.render_scenes(meshes, world["translations"], world["sizes"], world["angles"],
                                torch.where(keep, mi, -1), cls, floors=R.floor_triangles(floors[i:i + 1]),
                                white_background=True, camera=R.REFERENCE_PERSPECTIVE)
        loop()
        t_l, _ = sync_time(loop)
        res["%s_one_scene_per_call" % task] = {"scenes": L, "s_per_scene": t_l / L, "scenes_per_s": L / t_l}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
