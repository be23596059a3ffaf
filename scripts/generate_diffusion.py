#!/usr/bin/env python
"""Generation entry point (reference scripts/generate_diffusion.py:47-468, hot call :314-323).

Builds the network from the same YAML, loads a reference-format checkpoint, and samples scenes.  Rendering,
CAD retrieval and mesh export are outside the hot path (their dependencies are absent here); results are written
as `.npz` dictionaries after the reference's `post_process` (descale + atan2).  Unlike the reference loop
(one scene per call), `--batch_size` scenes are sampled per call and emptiness is decided per scene.

`--compute_intersec` scores every sampled batch on the device (diffuscene_b200.evaluate) and appends the
reference's per-scene lines to `iou_states.txt` (:394-430): box IoU, intersecting pairs, overlap ratio and symmetric
pairs of the objects placed with their retrieved models.  `--catalogue` is the `catalogue.npz` that
generate_objautoencoder.py writes (latents, labels, sizes), optionally with the footprint table of
`evaluate.footprint_table` (hull_offsets, hull_xz, raw_half, raw_aabb) and `model_ids`; without it every object is
its own box.  With a retrieval mode other than "box" a second line per scene scores the size-retrieved models, as the
reference's "retrive only size" line does.
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from training_utils import load_config  # noqa: E402

from scene_synthesis.networks import build_network  # noqa: E402
from diffuscene_b200.evaluate import PlausibilityAggregator, evaluate_samples  # noqa: E402
from diffuscene_b200.postprocess import ObjectCatalog  # noqa: E402
from diffuscene_b200.synthetic import SyntheticScenes  # noqa: E402


def _catalogue(path, network, mode):
    """(ObjectCatalog or None, retrieval mode) for --compute_intersec."""
    if path is None:
        return None, "box"
    cat = np.load(path)
    has_fp = all(k in cat for k in ObjectCatalog.FOOTPRINT_KEYS)
    catalog = ObjectCatalog(cat["labels"], cat["latents"] if "latents" in cat else None, cat["sizes"],
                            n_classes=network.class_dim - 1, footprints=cat if has_fp else None,
                            model_ids=cat["model_ids"] if "model_ids" in cat else None)
    if mode is None:
        mode = "objfeats" if network.objfeat_dim > 0 and catalog.feats is not None else "box"
    return catalog, mode


def main(argv):
    p = argparse.ArgumentParser(description="Generate scenes using a previously trained model")
    p.add_argument("config_file")
    p.add_argument("output_directory")
    p.add_argument("--weight_file", default=None)
    p.add_argument("--n_sequences", default=10, type=int)
    p.add_argument("--batch_size", default=1, type=int)
    p.add_argument("--clip_denoised", action="store_true")
    p.add_argument("--ddim", action="store_true")
    p.add_argument("--ddim_steps", type=int, default=50)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--precision", default="bf16", choices=["bf16", "fp32"])
    p.add_argument("--compute_intersec", action="store_true", help="append scene statistics to iou_states.txt")
    p.add_argument("--catalogue", default=None, help="catalogue.npz of the models to place (default: boxes)")
    p.add_argument("--retrieve_mode", default=None, choices=["objfeats", "objfeats_and_size", "box"],
                   help="retrieval for --compute_intersec (default: objfeats when the network and catalogue have them)")
    args = p.parse_args(argv)
    if not torch.cuda.is_available():
        raise RuntimeError("generate_diffusion.py needs a CUDA device (H100); there is no CPU path")
    device = torch.device("cuda:0")
    os.makedirs(args.output_directory, exist_ok=True)
    torch.manual_seed(args.seed)
    config = load_config(args.config_file)
    config["network"]["diffusion_kwargs"]["loss_iou"] = False        # no dataset stats needed to sample
    ds = SyntheticScenes(config["network"], 1)
    network, _, _ = build_network(ds.feature_size, ds.n_classes, config, args.weight_file, device=device,
                                  precision=args.precision)
    network.eval()
    N, d = config["network"]["sample_num_points"], config["network"]["point_dim"]
    if args.compute_intersec:
        catalog, mode = _catalogue(args.catalogue, network, args.retrieve_mode)
        aggs = [PlausibilityAggregator(PlausibilityAggregator.SUFFIX_OBJFEATS)]
        modes = [mode]
        if catalog is not None and mode != "box":
            aggs.append(PlausibilityAggregator(PlausibilityAggregator.SUFFIX_ONLYSIZE))
            modes.append("box")
    done = 0
    while done < args.n_sequences:
        bs = min(args.batch_size, args.n_sequences - done)
        if network.room_mask_condition:      # floor-plan configs: the synthetic floor plans of these scenes
            sds = SyntheticScenes(config["network"], args.n_sequences, seed=args.seed)
            room_mask = torch.stack([sds[done + i]["room_layout"] for i in range(bs)]).to(device)
        else:
            room_mask = torch.zeros(bs, 1, 64, 64, device=device)
        samples = network.sample(room_mask, N, d, batch_size=bs, clip_denoised=args.clip_denoised, ddim=args.ddim,
                                 ddim_steps=args.ddim_steps, seed=args.seed * 100003 + done)
        for i, scene in enumerate(network.delete_empty_batched(samples)):
            boxes = {k: v[None].numpy() for k, v in scene.items() if k != "class_index"}
            out = ds.post_process(boxes)
            out["class_index"] = scene["class_index"].numpy()
            np.savez(os.path.join(args.output_directory, "scene_{:05d}.npz".format(done + i)), **out)
        if args.compute_intersec:
            lines = [agg.update(evaluate_samples(network, samples, ds.bounds, catalog, m)) for agg, m in zip(aggs, modes)]
            with open(os.path.join(args.output_directory, "iou_states.txt"), "a") as f:
                for per_scene in zip(*lines):
                    f.write("".join(line + "\n" for line in per_scene))
            print(lines[0][-1])
        done += bs
    print("generated {} scenes in {}".format(done, args.output_directory))


if __name__ == "__main__":
    main(sys.argv[1:])
