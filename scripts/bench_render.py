#!/usr/bin/env python3
"""Times the native top-down rendering paths on one GPU and prints one JSON line (GPU name and power limit included):

  - render only: ds_render_scenes of B seeded scenes (8 slots, a quarter empty, a floor each) from a synthetic
    catalogue of subdivided boxes, cylinders, wedges and tables (diffuscene_b200.synthetic_meshes, ~20 k faces per
    model at --detail 20): scenes/s and placed triangles/s (the triangles of every non-empty slot and floor);
  - perspective render only: the same scenes through the completion driver's 512^2 perspective camera
    (render.REFERENCE_PERSPECTIVE), scenes/s and placed triangles/s;
  - render + device resize + features: the same batch through render.inception_features and render.vgg16_features
    (bf16 extractors, random weights), scenes/s;
  - render -> PNG -> the existing folder path: --png_scenes renders written as PNG, then read back through
    fid.folder_features and the IPR file path (host decode and PIL resize), scenes/s.

Everything is generated from seeds in the tree.

    python scripts/bench_render.py [--batch 4096] [--detail 20] [--out result.json]
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

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from diffuscene_b200 import fid as F, ipr as I, render as R, synthetic_meshes as SM  # noqa: E402
from oracle import inception_ref as IR  # noqa: E402
from tests.cases_ipr import he_state_dict  # noqa: E402


def timed(fn, reps):
    """Mean seconds of fn() over reps calls after one warm-up, with a device synchronise around the window."""
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / reps


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("--batch", type=int, default=4096)
    p.add_argument("--objects", type=int, default=8)
    p.add_argument("--models", type=int, default=64)
    p.add_argument("--detail", type=int, default=20)
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--png_scenes", type=int, default=512)
    p.add_argument("--out", default=None)
    a = p.parse_args(argv)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res = {"gpu": q[0] if q else "unknown", "batch": a.batch, "objects": a.objects}
    cat_np = SM.catalogue(seed=0, num_models=a.models, detail=a.detail, texture_size=256)
    cat = R.MeshCatalog(cat_np)
    sc = SM.scenes(a.batch, a.objects, a.models, seed=1)
    floors = R.floor_triangles(sc["floors"])
    dev = torch.device("cuda")
    args = [torch.as_tensor(sc[k]).to(dev) for k in ("translations", "sizes", "angles", "model_index")]
    res["faces_per_model"] = float(np.diff(cat_np["face_offsets"]).mean())
    mi = sc["model_index"]
    tris = int(cat.face_counts[mi[mi >= 0]].sum() + len(floors[1]))
    res["triangles_per_batch"] = tris

    render = lambda: R.render_scenes(cat, *args, floors=floors)
    t = timed(render, a.reps)
    res["render_ms"] = t * 1e3
    res["render_scenes_per_s"] = a.batch / t
    res["render_triangles_per_s"] = tris / t
    persp = lambda: R.render_scenes(cat, *args, floors=floors, camera=R.REFERENCE_PERSPECTIVE)
    t = timed(persp, a.reps)
    res["perspective_512_render_ms"] = t * 1e3
    res["perspective_512_scenes_per_s"] = a.batch / t
    res["perspective_512_triangles_per_s"] = tris / t

    inc = F.InceptionFeatures(IR.random_state_dict(seed=5), precision="bf16", capacity=64)
    vgg = I.VGG16Features(he_state_dict(0), precision="bf16", capacity=64)
    def full():
        imgs = render()
        return R.inception_features(inc, imgs), R.vgg16_features(vgg, imgs)
    t = timed(full, 1)
    res["render_resize_features_s"] = t
    res["render_resize_features_scenes_per_s"] = a.batch / t

    n = min(a.png_scenes, a.batch)
    with tempfile.TemporaryDirectory() as tmp:
        from PIL import Image
        imgs = render()[:n]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host = imgs.cpu().numpy()
        files = []
        for i, im in enumerate(host):
            files.append(os.path.join(tmp, "scene_%05d_render.png" % i))
            Image.fromarray(im).save(files[-1])
        F.folder_features(files, inc, batch_size=64, num_workers=8)
        ipr = I.IPR(batch_size=64, num_samples=n, model=vgg)
        ipr.extract_features_from_files(files)
        torch.cuda.synchronize()
        t = time.perf_counter() - t0 + res["render_ms"] / 1e3 * n / a.batch
        res["png_path_scenes"] = n
        res["png_path_scenes_per_s"] = n / t
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
