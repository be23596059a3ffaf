"""Floor-plan-conditioned training and the native room-mask encoder.

    python scripts/bench_floorplan.py [--batch 1024] [--steps 5] [--warmup 2] [--windows 3] [--sample-batch 4096]

Workload: config/floorplan/diffusion_bedrooms_instancond_lat32_v_floorplan.yaml (bedroom N = 12, d = 62, the
ResNet-18 encoder on 64 x 64 masks), bf16, random-init weights, seeded synthetic floor plans.  Measures, with CUDA
events around device-synchronised windows:
  - training scenes/s (train_on_batch) of the native model (`native_backward = True`: encoder and denoiser forward and
    backward in the CUDA library) against its autograd twin (`native_backward = False`), in alternating windows;
  - the encoder's forward and backward milliseconds at that batch (ds_room_enc_forward / _backward);
  - the encoder's forward at --sample-batch scenes as a share of one full sample() call (T = 1000) at that batch.
Prints one JSON line with the card's name and power limit.  Writes nothing into the repository.
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_train_text import STATS, gpu_identity  # noqa: E402


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
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=5, help="optimizer iterations per timed window")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--windows", type=int, default=3, help="timed windows per path (alternating)")
    ap.add_argument("--sample-batch", type=int, default=4096)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_floorplan.py measures on a CUDA device; none is available")
    import yaml
    from diffuscene_b200.synthetic import SyntheticScenes
    from scene_synthesis.networks import build_network, optimizer_factory

    B, N = args.batch, 12
    tmp = tempfile.mkdtemp(prefix="ds_bench_fp_")
    stats = os.path.join(tmp, "stats.json")
    with open(stats, "w") as f:
        json.dump(STATS, f)
    cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "floorplan",
                                           "diffusion_bedrooms_instancond_lat32_v_floorplan.yaml")))
    cfg["network"]["diffusion_kwargs"]["train_stats_file"] = stats
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    nets, opts = {}, {}
    nets["native"], train_on_batch, _ = build_network(30, 23, cfg, None, device=dev, precision="bf16")
    nets["autograd"], _, _ = build_network(30, 23, cfg, None, device=dev, precision="bf16")
    nets["autograd"].load_state_dict(copy.deepcopy(nets["native"].state_dict()))
    nets["autograd"].native_backward = False
    for k, net in nets.items():
        opts[k] = optimizer_factory(cfg["training"], net.parameters())

    ds = SyntheticScenes(cfg["network"], max(B, args.sample_batch), seed=1)
    items = [ds[i] for i in range(B)]
    sp = {k: torch.stack([it[k] for it in items]).to(dev) for k in items[0] if torch.is_tensor(items[0][k])}
    last = {}

    def window(k, steps):
        def step():
            last[k] = train_on_batch(nets[k], opts[k], sp, cfg)
        return timed(step, steps, dev) * steps

    for k in nets:
        window(k, args.warmup)
    rates = {k: [] for k in nets}
    for _ in range(args.windows):
        for k in nets:
            rates[k].append(B * args.steps / (window(k, args.steps) / 1000.0))

    net = nets["native"]
    enc = net._ensure_room_flat(64, 64)
    mask = sp["room_layout"]
    dfeat = torch.randn(B, 512, device=dev)
    with torch.no_grad():
        fwd_ms = timed(lambda: enc.forward(net._room_flat, mask, keep=True), 10, dev)
        bwd_ms = timed(lambda: enc.backward(dfeat, net._room_grads), 10, dev)
        SB = args.sample_batch
        big = torch.stack([ds[i]["room_layout"] for i in range(SB)]).to(dev)
        fwd_big_ms = timed(lambda: enc.forward(net._room_flat, big), 5, dev)
        net.sample(big, N, 62, batch_size=SB, seed=1)      # warm-up: graph capture, buffers
        sample_ms = timed(lambda: net.sample(big, N, 62, batch_size=SB, seed=1), 1, dev)
    gpu, power = gpu_identity()
    nat, ag = statistics.median(rates["native"]), statistics.median(rates["autograd"])
    print(json.dumps({
        "metric": "floor-plan training scenes/s (train_on_batch, median of windows)", "unit": "scenes/s",
        "native": nat, "autograd": ag, "speedup": nat / ag,
        "native_windows": rates["native"], "autograd_windows": rates["autograd"],
        "encoder_forward_ms": fwd_ms, "encoder_backward_ms": bwd_ms, "encoder_batch": B,
        "encoder_forward_ms_at_sample_batch": fwd_big_ms, "sample_ms": sample_ms, "sample_batch": SB,
        "encoder_share_of_sample": fwd_big_ms / sample_ms,
        "last_loss": {"native": last["native"], "autograd": last["autograd"]},
        "config": {"workload": "floor-plan bedroom N=12 d=62, ResNet-18 encoder on 64x64 masks, Adam, clip 10, "
                               "random-init weights, synthetic floor plans", "precision": "bf16", "scenes": B,
                   "steps_per_window": args.steps, "windows": args.windows, "warmup": args.warmup, "T": 1000},
        "gpu": gpu, "power_limit": power}))


if __name__ == "__main__":
    main()
