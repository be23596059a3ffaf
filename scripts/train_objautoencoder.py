#!/usr/bin/env python
"""Train the object shape auto-encoder (reference scripts/train_objautoencoder.py) on the H100-native KLAutoEncoder.

The 3D-FUTURE object meshes are absent here, so `--synthetic` (the default) trains on seeded boxes and ellipsoids
(diffuscene_b200.synthetic.SyntheticShapes) with the dataset's point-cloud contract.  Checkpoints are
`model_XXXXX` / `opt_XXXXX` in the experiment directory, as for the denoiser.
"""
import argparse
import os
import sys

import numpy as np
import torch
from torch.utils.data import DataLoader

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from training_utils import id_generator, load_checkpoints, load_config, save_checkpoints, save_experiment_params  # noqa: E402

from scene_synthesis.networks import adjust_learning_rate, optimizer_factory, schedule_factory  # noqa: E402
from scene_synthesis.networks.foldingnet_autoencoder import KLAutoEncoder, train_on_batch, validate_on_batch  # noqa: E402
from scene_synthesis.stats_logger import StatsLogger  # noqa: E402
from diffuscene_b200.synthetic import SyntheticShapes  # noqa: E402


def main(argv):
    p = argparse.ArgumentParser(description="Train the object shape auto-encoder")
    p.add_argument("config_file")
    p.add_argument("output_directory")
    p.add_argument("--weight_file", default=None)
    p.add_argument("--continue_from_epoch", default=0, type=int)
    p.add_argument("--n_processes", type=int, default=0)
    p.add_argument("--seed", type=int, default=27)
    p.add_argument("--experiment_tag", default=None)
    p.add_argument("--synthetic", action=argparse.BooleanOptionalAction, default=True)
    p.add_argument("--synthetic_objects", type=int, default=1024)
    p.add_argument("--num_points", type=int, default=None, help="points per object (config data.num_points, 2048)")
    p.add_argument("--max_epochs", type=int, default=None, help="cap on config training.epochs")
    args = p.parse_args(argv)

    np.random.seed(args.seed)
    torch.manual_seed(np.random.randint(np.iinfo(np.int32).max))
    if not torch.cuda.is_available():
        raise RuntimeError("train_objautoencoder.py needs a CUDA device (H100); there is no CPU path")
    device = torch.device("cuda:0")
    os.makedirs(args.output_directory, exist_ok=True)
    tag = args.experiment_tag or id_generator(9)
    exp_dir = os.path.join(args.output_directory, tag)
    os.makedirs(exp_dir, exist_ok=True)
    save_experiment_params(args, tag, exp_dir)
    config = load_config(args.config_file)
    if not args.synthetic:
        raise RuntimeError("the 3D-FUTURE data layer (scene_synthesis.datasets) is outside this repository's scope")
    P = args.num_points or config.get("data", {}).get("num_points", 2048)
    train_ds = SyntheticShapes(args.synthetic_objects, P, seed=args.seed)
    val_ds = SyntheticShapes(max(args.synthetic_objects // 8, 8), P, seed=args.seed + 1)
    tr, va = config["training"], config.get("validation", {})
    train_loader = DataLoader(train_ds, batch_size=tr.get("batch_size", 16), shuffle=True, drop_last=True,
                              num_workers=args.n_processes)
    val_loader = DataLoader(val_ds, batch_size=va.get("batch_size", 16), num_workers=args.n_processes)

    net = KLAutoEncoder(latent_dim=config["network"].get("objfeat_dim", 64),
                        kl_weight=config["network"].get("kl_weight", 0.001), num_points=P)
    if args.weight_file is not None:
        net.load_state_dict(torch.load(args.weight_file, map_location="cpu"), strict=True)
    net.to(device)
    optimizer = optimizer_factory(tr, filter(lambda q: q.requires_grad, net.parameters()))
    load_checkpoints(net, optimizer, exp_dir, args, device)
    lr_scheduler = schedule_factory(tr)
    epochs = tr.get("epochs", 150) if args.max_epochs is None else min(args.max_epochs, tr.get("epochs", 150))
    steps_per_epoch = tr.get("steps_per_epoch", 500)
    for i in range(args.continue_from_epoch, epochs):
        adjust_learning_rate(lr_scheduler, optimizer, i)
        net.train()
        for b, sample in zip(range(steps_per_epoch), train_loader):
            train_on_batch(net, optimizer, {"points": sample["points"].to(device)}, config)
            StatsLogger.instance().print_progress(i + 1, b + 1, 0.0)
        if (i % tr.get("save_frequency", 10)) == 0 or i == epochs - 1:
            save_checkpoints(i, net, optimizer, exp_dir)
        StatsLogger.instance().clear()
        if i % va.get("frequency", 10) == 0 or i == epochs - 1:
            net.eval()
            for b, sample in enumerate(val_loader):
                validate_on_batch(net, {"points": sample["points"].to(device)}, config)
                StatsLogger.instance().print_progress(-1, b + 1, 0.0)
            StatsLogger.instance().clear()
    print("Saved to", exp_dir)


if __name__ == "__main__":
    main(sys.argv[1:])
