"""Drop-in for `scene_synthesis.networks` (reference scene_synthesis/networks/__init__.py:15-169):
build_network(), optimizer_factory(), schedule_factory(), adjust_learning_rate() with the reference's
signatures, config keys and error behaviour; the network they build runs on the CUDA engine."""
from __future__ import annotations

import math

import torch

from .diffusion_scene_layout_ddpm import DiffusionSceneLayout_DDPM, train_on_batch as _train_on_batch, \
    validate_on_batch as _validate_on_batch


def optimizer_factory(config, parameters):
    """Reference :15-34: SGD / Adam / RAdam, weight decay pinned to 0."""
    optimizer = config.get("optimizer", "Adam")
    lr = config.get("lr", 1e-3)
    momentum = config.get("momentum", 0.9)
    weight_decay = 0.0
    if optimizer == "SGD":
        return torch.optim.SGD(parameters, lr=lr, momentum=momentum, weight_decay=weight_decay)
    if optimizer == "Adam":      # a torch.optim.Adam whose step() is one fused kernel on the native training path
        from ..optim import NativeAdam
        return NativeAdam(parameters, lr=lr, weight_decay=weight_decay)
    if optimizer == "RAdam":
        return torch.optim.RAdam(parameters, lr=lr, weight_decay=weight_decay)
    raise NotImplementedError()


def build_network(input_dims, n_classes, config, weight_file=None, device="cpu", precision="bf16",
                  gemm_backend="auto"):
    """Reference :37-68.  The `feature_extractor` section configures the floor-plan encoder of networks with
    room_mask_condition (ignored otherwise)."""
    network_type = config["network"]["type"]
    if network_type == "diffusion_scene_layout_ddpm":
        network = DiffusionSceneLayout_DDPM(n_classes, config.get("feature_extractor"), config["network"],
                                            precision=precision, gemm_backend=gemm_backend)
    else:
        raise NotImplementedError()
    if weight_file is not None:
        print("Loading weight file from {}".format(weight_file))
        network.load_state_dict(torch.load(weight_file, map_location=device))
    network.to(device)
    return network, _train_on_batch, _validate_on_batch


class LearningRateSchedule:
    def get_learning_rate(self, epoch):
        pass


class StepLearningRateSchedule(LearningRateSchedule):
    def __init__(self, specs):
        self.initial, self.interval, self.factor = specs["initial"], specs["interval"], specs["factor"]

    def get_learning_rate(self, epoch):
        return self.initial * (self.factor ** (epoch // self.interval))


class LambdaLearningRateSchedule(LearningRateSchedule):
    def __init__(self, specs):
        self.start_epoch, self.end_epoch = specs["start_epoch"], specs["end_epoch"]
        self.start_lr, self.end_lr = specs["start_lr"], specs["end_lr"]

    def lr_func(self, epoch):
        if epoch <= self.start_epoch:
            return 1.0
        if epoch <= self.end_epoch:
            frac = (epoch - self.start_epoch) / (self.end_epoch - self.start_epoch)
            return (1 - frac) * 1.0 + frac * (self.end_lr / self.start_lr)
        return self.end_lr / self.start_lr

    def get_learning_rate(self, epoch):
        return self.start_lr * self.lr_func(epoch)


class WarmupCosineLearningRateSchedule(LearningRateSchedule):
    def __init__(self, specs):
        self.warmup_epochs, self.total_epochs = specs["warmup_epochs"], specs["total_epochs"]
        self.lr, self.min_lr = specs["lr"], specs["min_lr"]

    def get_learning_rate(self, epoch):
        if epoch <= self.warmup_epochs:
            return self.lr
        return self.min_lr + (self.lr - self.min_lr) * 0.5 * (
            1.0 + math.cos(math.pi * (epoch - self.warmup_epochs) / (self.total_epochs - self.warmup_epochs)))


def adjust_learning_rate(lr_schedules, optimizer, epoch):
    for i, param_group in enumerate(optimizer.param_groups):
        sched = lr_schedules[i] if isinstance(lr_schedules, list) else lr_schedules
        param_group["lr"] = sched.get_learning_rate(epoch)


def schedule_factory(config):
    """Reference :135-169."""
    schedule = config.get("schedule", "lambda")
    if schedule in ("step", "Step"):
        return StepLearningRateSchedule({"type": "step", "initial": config.get("lr", 1e-3),
                                         "interval": config.get("lr_step", 100), "factor": config.get("lr_decay", 0.1)})
    if schedule in ("lambda", "Lambda"):
        return LambdaLearningRateSchedule({"type": "lambda", "start_epoch": config.get("start_epoch", 1000),
                                           "end_epoch": config.get("end_epoch", 1000),
                                           "start_lr": config.get("start_lr", 0.002),
                                           "end_lr": config.get("end_lr", 0.002)})
    if schedule in ("warmupcosine", "WarmupCosine"):
        return WarmupCosineLearningRateSchedule({"type": "warmupcosine", "warmup_epochs": config.get("warmup_epochs", 10),
                                                 "total_epochs": config.get("total_epochs", 2000),
                                                 "lr": config.get("lr", 2e-4), "min_lr": config.get("min_lr", 1e-6)})
    raise NotImplementedError()
