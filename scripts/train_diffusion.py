#!/usr/bin/env python
"""Training entry point (reference scripts/train_diffusion.py:27-255) on the H100-native network.

Same positional arguments, flags, experiment-directory layout and checkpoint files.  `--synthetic` (the default)
feeds scenes from diffuscene_b200.synthetic with the same `sample_params` contract.  `--no-synthetic` trains on the
reference's preprocessed 3D-FRONT rooms (<dataset_directory>/<room>/boxes.npz and dataset_stats.txt), held on the
device by diffuscene_b200.scene_data and batched by one CUDA kernel per batch:

    python scripts/train_diffusion.py CONFIG OUT --no-synthetic --dataset_directory DIR --annotation_file SPLITS.csv

Data settings come from the flags, else from the config's `data` section, else the reference's shipped defaults.
"""
import argparse
import os
import sys

import numpy as np
import torch
from torch.utils.data import DataLoader

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from training_utils import id_generator, load_checkpoints, load_config, save_checkpoints, save_experiment_params  # noqa: E402

from scene_synthesis.networks import adjust_learning_rate, build_network, optimizer_factory, schedule_factory  # noqa: E402
from scene_synthesis.stats_logger import StatsLogger  # noqa: E402
from diffuscene_b200.synthetic import SyntheticScenes, write_stats_file  # noqa: E402
from diffuscene_b200 import scene_data  # noqa: E402


def main(argv):
    p = argparse.ArgumentParser(description="Train a generative model on bounding boxes")
    p.add_argument("config_file")
    p.add_argument("output_directory")
    p.add_argument("--weight_file", default=None)
    p.add_argument("--continue_from_epoch", default=0, type=int)
    p.add_argument("--n_processes", type=int, default=0,
                   help="DataLoader workers of the synthetic scenes; no effect with --no-synthetic (batches are built "
                        "on the device)")
    p.add_argument("--seed", type=int, default=27)
    p.add_argument("--experiment_tag", default=None)
    p.add_argument("--with_wandb_logger", action="store_true")
    p.add_argument("--synthetic", action=argparse.BooleanOptionalAction, default=True)
    p.add_argument("--synthetic_scenes", type=int, default=2048)
    p.add_argument("--max_epochs", type=int, default=None, help="cap on config training.epochs")
    p.add_argument("--precision", default="bf16", choices=["bf16", "fp32"])
    p.add_argument("--dataset_directory", default=None, help="--no-synthetic: the preprocessed rooms (or data."
                   "dataset_directory)")
    p.add_argument("--annotation_file", default=None, help="--no-synthetic: the splits CSV (or data.annotation_file)")
    p.add_argument("--encoding_type", default=None,
                   help="--no-synthetic: or data.encoding_type, default %s" % scene_data.DEFAULT_ENCODING)
    p.add_argument("--augmentations", default=None, help="--no-synthetic: comma-separated, or data.augmentations, "
                   "default %s" % ",".join(scene_data.DEFAULT_AUGMENTATIONS))
    p.add_argument("--train_stats", default=None,
                   help="--no-synthetic: stats file in the dataset directory (or data.train_stats, default %s)"
                        % scene_data.DEFAULT_STATS)
    args = p.parse_args(argv)
    config = load_config(args.config_file)
    data = None
    if not args.synthetic:
        data = dict(config.get("data") or {})
        for k in ("dataset_directory", "annotation_file", "encoding_type", "train_stats"):
            if getattr(args, k) is not None:
                data[k] = getattr(args, k)
        if args.augmentations is not None:
            data["augmentations"] = [a for a in args.augmentations.split(",") if a]
        for k in ("dataset_directory", "annotation_file"):
            if not data.get(k):
                p.error("--no-synthetic needs --%s (or data.%s in the config)" % (k, k))
        if not os.path.isdir(data["dataset_directory"]):
            p.error("no dataset directory %s" % data["dataset_directory"])
        if not os.path.isfile(data["annotation_file"]):
            p.error("no annotation file %s" % data["annotation_file"])

    np.random.seed(args.seed)
    torch.manual_seed(np.random.randint(np.iinfo(np.int32).max))
    if not torch.cuda.is_available():
        raise RuntimeError("train_diffusion.py needs a CUDA device (H100); there is no CPU path")
    torch.cuda.manual_seed_all(np.random.randint(np.iinfo(np.int32).max))
    device = torch.device("cuda:0")

    os.makedirs(args.output_directory, exist_ok=True)
    tag = args.experiment_tag or id_generator(9)
    exp_dir = os.path.join(args.output_directory, tag)
    os.makedirs(exp_dir, exist_ok=True)
    save_experiment_params(args, tag, exp_dir)

    net_cfg = config["network"]
    if args.synthetic:
        train_ds = SyntheticScenes(net_cfg, args.synthetic_scenes, seed=args.seed)
        val_ds = SyntheticScenes(net_cfg, max(args.synthetic_scenes // 8, 8), seed=args.seed + 1)
        np.savez(os.path.join(exp_dir, "bounds.npz"), translations=np.stack(train_ds.bounds["translations"]),
                 sizes=np.stack(train_ds.bounds["sizes"]), angles=np.stack(train_ds.bounds["angles"]))
        if net_cfg["diffusion_kwargs"].get("loss_iou", False):
            net_cfg["diffusion_kwargs"]["train_stats_file"] = write_stats_file(os.path.join(exp_dir,
                                                                                            "dataset_stats.txt"))
        train_loader = DataLoader(train_ds, batch_size=config["training"].get("batch_size", 128),
                                  num_workers=args.n_processes, shuffle=True)
        val_loader = DataLoader(val_ds, batch_size=config["validation"].get("batch_size", 1),
                                num_workers=args.n_processes)
    else:
        store_kw = dict(encoding_type=data.get("encoding_type", scene_data.DEFAULT_ENCODING),
                        train_stats=data.get("train_stats", scene_data.DEFAULT_STATS),
                        room_layout_size=data.get("room_layout_size", "64,64"), max_length=data.get("max_length"),
                        device=device)
        train_ds = scene_data.SceneStore(data["dataset_directory"], data["annotation_file"],
                                         config["training"].get("splits", ["train", "val"]), net_cfg, **store_kw)
        val_ds = scene_data.SceneStore(data["dataset_directory"], data["annotation_file"],
                                       config["validation"].get("splits", ["test"]), net_cfg, **store_kw)
        b = train_ds.bounds      # the reference's bounds.npz (train_diffusion.py:126-135)
        np.savez(os.path.join(exp_dir, "bounds.npz"), sizes=b["sizes"], translations=b["translations"],
                 angles=b["angles"], objfeats=b["objfeats"])
        net_cfg["diffusion_kwargs"]["train_stats_file"] = train_ds.stats_path
        train_loader = scene_data.SceneLoader(train_ds, config["training"].get("batch_size", 128), shuffle=True,
                                              augmentations=data.get("augmentations",
                                                                     list(scene_data.DEFAULT_AUGMENTATIONS)),
                                              seed=args.seed)
        val_loader = scene_data.SceneLoader(val_ds, config["validation"].get("batch_size", 1), shuffle=False,
                                            augmentations=[], seed=args.seed + 1)

    network, train_on_batch, validate_on_batch = build_network(train_ds.feature_size, train_ds.n_classes, config,
                                                               args.weight_file, device=device,
                                                               precision=args.precision)
    optimizer = optimizer_factory(config["training"], filter(lambda q: q.requires_grad, network.parameters()))
    load_checkpoints(network, optimizer, exp_dir, args, device)
    lr_scheduler = schedule_factory(config["training"])
    StatsLogger.instance().add_output_file(open(os.path.join(exp_dir, "stats.txt"), "w"))

    epochs = config["training"].get("epochs", 150)
    if args.max_epochs is not None:
        epochs = min(epochs, args.continue_from_epoch + args.max_epochs)
    save_every = config["training"].get("save_frequency", 10)
    val_every = config["validation"].get("frequency", 100)
    for i in range(args.continue_from_epoch, epochs):
        adjust_learning_rate(lr_scheduler, optimizer, i)
        network.train()
        for b, sample in enumerate(train_loader):
            sample = {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in sample.items()}
            batch_loss = train_on_batch(network, optimizer, sample, config)
            StatsLogger.instance().print_progress(i + 1, b + 1, batch_loss)
        if (i % save_every) == 0 or i == epochs - 1:
            save_checkpoints(i, network, optimizer, exp_dir)
        StatsLogger.instance().clear()
        if i % val_every == 0 and i > 0:
            network.eval()
            for b, sample in enumerate(val_loader):
                sample = {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in sample.items()}
                batch_loss = validate_on_batch(network, sample, config)
                StatsLogger.instance().print_progress(-1, b + 1, batch_loss)
            StatsLogger.instance().clear()


if __name__ == "__main__":
    main(sys.argv[1:])
