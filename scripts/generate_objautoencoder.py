#!/usr/bin/env python
"""Encode objects with a trained shape auto-encoder (reference scripts/generate_objautoencoder.py): one latent per
object, the std-based scale factor the reference prints, and a catalogue file for retrieval.

Writes into `output_directory`: `objfeats/<index>.npz` (key `latent`, [F]) per object, as the reference stores them,
and `catalogue.npz` with `latents` [M, F], `labels` [M] and `sizes` [M, 3], the arrays
`diffuscene_b200.postprocess.ObjectCatalog` takes.  The latent is the posterior sample, as in the reference.
`--synthetic` (the default) encodes diffuscene_b200.synthetic.SyntheticShapes.
"""
import argparse
import os
import sys

import numpy as np
import torch
from torch.utils.data import DataLoader

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from training_utils import load_config  # noqa: E402

from scene_synthesis.networks.foldingnet_autoencoder import KLAutoEncoder  # noqa: E402
from diffuscene_b200.synthetic import SyntheticShapes  # noqa: E402


def main(argv):
    p = argparse.ArgumentParser(description="Encode objects with a trained shape auto-encoder")
    p.add_argument("config_file")
    p.add_argument("output_directory")
    p.add_argument("--weight_file", default=None)
    p.add_argument("--seed", type=int, default=27)
    p.add_argument("--batch_size", type=int, default=64)
    p.add_argument("--synthetic", action=argparse.BooleanOptionalAction, default=True)
    p.add_argument("--synthetic_objects", type=int, default=1024)
    p.add_argument("--num_points", type=int, default=None, help="points per object (config data.num_points, 2048)")
    args = p.parse_args(argv)

    np.random.seed(args.seed)
    torch.manual_seed(np.random.randint(np.iinfo(np.int32).max))
    if not torch.cuda.is_available():
        raise RuntimeError("generate_objautoencoder.py needs a CUDA device (H100); there is no CPU path")
    device = torch.device("cuda:0")
    config = load_config(args.config_file)
    if not args.synthetic:
        raise RuntimeError("the 3D-FUTURE data layer (scene_synthesis.datasets) is outside this repository's scope")
    P = args.num_points or config.get("data", {}).get("num_points", 2048)
    ds = SyntheticShapes(args.synthetic_objects, P, seed=args.seed)
    net = KLAutoEncoder(latent_dim=config["network"].get("objfeat_dim", 64),
                        kl_weight=config["network"].get("kl_weight", 0.001), num_points=P)
    if args.weight_file is not None:
        net.load_state_dict(torch.load(args.weight_file, map_location="cpu"), strict=True)
    net.to(device).eval()
    lats, labels, sizes = [], [], []
    with torch.no_grad():
        for sample in DataLoader(ds, batch_size=args.batch_size):
            _, lat = net.encode(sample["points"].to(device).permute(0, 2, 1))
            lats.append(lat.cpu().numpy())
            labels.append(sample["label"].numpy())
            sizes.append(sample["size"].numpy())
    lat_all, labels, sizes = np.concatenate(lats), np.concatenate(labels), np.concatenate(sizes)
    out_dir = os.path.join(args.output_directory, "objfeats")
    os.makedirs(out_dir, exist_ok=True)
    for i, lat in enumerate(lat_all):
        np.savez(os.path.join(out_dir, "%05d.npz" % i), latent=lat)
    print("before: std {}, min {}, max {}".format(lat_all.flatten().std(), lat_all.min(), lat_all.max()))
    scale_factor = 1.0 / lat_all.flatten().std()
    print("scale factor:", scale_factor)
    lat_scaled = lat_all * scale_factor
    print("after: std {}, min {}, max {}".format(lat_scaled.flatten().std(), lat_scaled.min(), lat_scaled.max()))
    np.savez(os.path.join(args.output_directory, "catalogue.npz"), latents=lat_all.astype(np.float32),
             labels=labels.astype(np.int64), sizes=sizes.astype(np.float32))
    print("Saved %d latents to %s" % (len(lat_all), args.output_directory))


if __name__ == "__main__":
    main(sys.argv[1:])
