#!/usr/bin/env python3
"""Times the device-resident training data (diffuscene_b200.scene_data) on one GPU and prints one JSON line, GPU
name and power limit included.

A seeded store of 4096 rooms is written in the reference's preprocessed format to a temporary directory, for N = 12
and N = 21 objects (objfeat 32, 256^2 room masks resized to 64 x 64, fixed rotations + jitter, permutation):

  - kernel: ds_scene_batch alone, us per batch, at B = 128, 1024 and 8192 (CUDA events over --iters launches);
  - loader: one SceneLoader batch, its draws included, us per batch;
  - step: one native bf16 training step (train_on_batch) at the same B, floor-plan network (N = 12 only; random
    weights), ms per step;
  - epoch: scripts/train_diffusion.py's inner loop over the 4096 rooms at B = 128, in scenes/s, with the real-format
    loader and with the synthetic DataLoader;
  - numpy: the reference's per-scene chain (np.load of the npz per item, PIL resize, augment, scale, permute, pad;
    tests/scene_data_ref.py) through a DataLoader with 0 and 8 workers, scenes/s, no training step.

    python scripts/bench_scene_data.py [--iters 200] [--out result.json]
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

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from training_utils import load_config  # noqa: E402

from scene_synthesis.networks import build_network, optimizer_factory, train_on_batch  # noqa: E402
from diffuscene_b200 import scene_data as SD  # noqa: E402
from diffuscene_b200.synthetic import SyntheticScenes, write_reference_rooms  # noqa: E402
from tests import scene_data_ref as ref  # noqa: E402

CFG = os.path.join(ROOT, "config", "floorplan", "diffusion_bedrooms_instancond_lat32_v_floorplan.yaml")
AUGS = ["fixed_rotations", "jitter"]
BATCHES = (128, 1024, 8192)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def event_us(fn, iters):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


class NumpyChain(torch.utils.data.Dataset):
    """The reference's per-item path: np.load the room, resize its layout, draw and apply the chain."""

    def __init__(self, store, ds):
        self.store, self.ds = store, ds

    def __len__(self):
        return len(self.store)

    def __getitem__(self, i):
        s = self.store
        D = np.load(os.path.join(self.ds, s.tags[i], "boxes.npz"))
        room = {"room_layout": SD.room_layout(D, (64, 64))[None], "class_labels": D["class_labels"],
                "translations": D["translations"], "sizes": D["sizes"], "angles": D["angles"],
                "objfeats": D["objfeats"], "objfeats_32": D["objfeats_32"]}
        r = np.random.rand()
        theta = np.pi * 1.5 if r < 0.25 else np.pi if np.random.rand() < 0.5 else \
            np.pi * 0.5 if np.random.rand() < 0.75 else 0.0
        jit = [np.random.normal(0, 0.01) for _ in range(3)]
        order = np.random.permutation(len(D["class_labels"]))
        out = ref.sample(room, s.encoding_type, AUGS, s.bounds, s.N, theta=theta, jitter=jit, ordering=order)
        return {k: torch.as_tensor(np.asarray(v)) for k, v in out.items()}


def epoch_rate(loader, step, to_device=False):
    torch.cuda.synchronize()
    t = time.perf_counter()
    n = 0
    for sample in loader:
        if to_device:
            sample = {k: v.cuda(non_blocking=True) for k, v in sample.items()}
        step(sample)
        n += int(sample["length"].shape[0])
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t)


def main():
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--iters", type=int, default=200)
    p.add_argument("--out", default=None)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_scene_data.py needs a CUDA device")
    res = {"gpu": gpu_info(), "scenes": 4096, "augmentations": AUGS}
    config = load_config(CFG)
    with tempfile.TemporaryDirectory() as tmp:
        stores = {}
        for N in (12, 21):
            ds, csv = os.path.join(tmp, "ds%d" % N), os.path.join(tmp, "splits%d.csv" % N)
            write_reference_rooms(ds, csv, 4096, max_objects=N, seed=N, splits=("train",))
            net = dict(config["network"], sample_num_points=N)
            t = time.perf_counter()
            stores[N] = (SD.SceneStore(ds, csv, ["train"], net, device="cuda"), ds)
            res["store_load_s_N%d" % N] = round(time.perf_counter() - t, 3)
        for N, (store, _) in stores.items():
            for B in BATCHES:
                loader = SD.SceneLoader(store, B, augmentations=AUGS, seed=B)
                idx = torch.randint(0, len(store), (B,), device="cuda")
                draws = loader.draws(B)
                res["kernel_us_N%d_B%d" % (N, B)] = round(event_us(
                    lambda: store._launch(idx, loader.augs, True, *draws), args.iters), 2)
                res["loader_us_N%d_B%d" % (N, B)] = round(event_us(
                    lambda: store._launch(idx, loader.augs, True, *loader.draws(B)), args.iters), 2)

        store, ds = stores[12]
        config["network"]["diffusion_kwargs"]["train_stats_file"] = store.stats_path
        torch.manual_seed(0)
        network, _, _ = build_network(store.feature_size, store.n_classes, config, None, device=torch.device("cuda"),
                                      precision="bf16")
        network.train()
        optimizer = optimizer_factory(config["training"], [q for q in network.parameters() if q.requires_grad])
        step = lambda s: train_on_batch(network, optimizer, s, config)
        for B in BATCHES:
            try:
                loader = SD.SceneLoader(store, B, augmentations=AUGS, seed=B)
                idx = torch.randint(0, len(store), (B,), device="cuda")
                batch = store._launch(idx, loader.augs, True, *loader.draws(B))
                res["step_ms_N12_B%d" % B] = round(event_us(lambda: step(batch), 10) / 1e3, 3)
            except torch.cuda.OutOfMemoryError:
                res["step_ms_N12_B%d" % B] = "not measured (out of memory)"
                torch.cuda.empty_cache()
        B = config["training"]["batch_size"]
        loader = SD.SceneLoader(store, B, augmentations=AUGS, seed=1)
        epoch_rate(loader, step)
        res["epoch_scenes_per_s_native_loader"] = round(epoch_rate(loader, step), 1)
        syn = torch.utils.data.DataLoader(SyntheticScenes(config["network"], 4096, seed=0), batch_size=B, shuffle=True)
        res["epoch_scenes_per_s_synthetic_dataloader"] = round(epoch_rate(syn, step, to_device=True), 1)
        nothing = lambda s: None
        for w in (0, 8):
            dl = torch.utils.data.DataLoader(NumpyChain(store, ds), batch_size=B, shuffle=True, num_workers=w)
            res["numpy_chain_scenes_per_s_workers%d" % w] = round(epoch_rate(dl, nothing), 1)
        res["native_loader_scenes_per_s_B%d" % B] = round(B / (res["loader_us_N12_B%d" % B] * 1e-6), 1)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
