"""Training throughput of the text-conditioned bedroom network: native training step against the torch autograd path.

    python scripts/bench_train_text.py [--batch 1024] [--text-len 64] [--steps 5] [--warmup 2] [--windows 3]

Workload: the shipped text config (config/text/diffusion_bedrooms_instancond_lat32_v_bert.yaml: bedroom N = 12,
d = 62, 9 LinearAttentionCross layers on a 512-d text projection), loss_separate + loss_iou, gradient clip 10, Adam,
random-init weights, synthetic BERT hidden states [B, L, 768] (BERT itself is frozen and outside the timed step;
L = 64 tokens is an assumption about description length, stated in the output).  One step = one `train_on_batch`.

Two models with the same weights run in one process: `native_backward = True` (ds_train_step_cross: forward and
backward of the denoiser in the CUDA library, fused Adam) and `native_backward = False` (torch autograd over
functional.DenoiserFn, torch Adam).  Timed windows of the two alternate, each bracketed by CUDA events after a
device synchronise.  Prints one JSON line.  Writes nothing into the repository (the stats file goes to a temporary
directory).
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STATS = {"bounds_translations": [-2.7, 0.04, -2.75, 2.8, 3.6, 2.9], "bounds_sizes": [0.04, 0.02, 0.01, 2.9, 1.8, 2.6],
         "bounds_angles": [-3.14159, 3.14159]}


def gpu_identity():
    name = torch.cuda.get_device_name(torch.cuda.current_device())
    try:
        idx = str(torch.cuda.current_device())
        out = subprocess.run(["nvidia-smi", "-i", idx, "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = None
    return name, out or None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--text-len", type=int, default=64)
    ap.add_argument("--steps", type=int, default=5, help="optimizer iterations per timed window")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--windows", type=int, default=3, help="timed windows per path (alternating)")
    ap.add_argument("--precision", default="bf16", choices=["bf16", "fp32"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_text.py measures on a CUDA device; none is available")
    import yaml
    from scene_synthesis.networks import build_network, optimizer_factory

    B, L, N = args.batch, args.text_len, 12
    tmp = tempfile.mkdtemp(prefix="ds_bench_text_")
    stats = os.path.join(tmp, "stats.json")
    with open(stats, "w") as f:
        json.dump(STATS, f)
    cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "text", "diffusion_bedrooms_instancond_lat32_v_bert.yaml")))
    cfg["network"]["diffusion_kwargs"]["train_stats_file"] = stats
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    nets, opts = {}, {}
    nets["native"], train_on_batch, _ = build_network(30, 23, cfg, None, device=dev, precision=args.precision)
    nets["autograd"], _, _ = build_network(30, 23, cfg, None, device=dev, precision=args.precision)
    nets["autograd"].load_state_dict(copy.deepcopy(nets["native"].state_dict()))
    nets["autograd"].native_backward = False
    for k, net in nets.items():
        opts[k] = optimizer_factory(cfg["training"], net.parameters())

    g = torch.Generator().manual_seed(1)
    cls = torch.randint(0, 22, (B, N), generator=g)
    sp = dict(translations=torch.rand(B, N, 3, generator=g) * 2 - 1, sizes=torch.rand(B, N, 3, generator=g) * 2 - 1,
              angles=torch.nn.functional.normalize(torch.randn(B, N, 2, generator=g), dim=-1),
              class_labels=torch.nn.functional.one_hot(cls, 22).float() * 2 - 1,
              objfeats_32=torch.rand(B, N, 32, generator=g) * 2 - 1, room_layout=torch.zeros(B, 1, 64, 64),
              description=torch.randn(B, L, 768, generator=g))
    sp = {k: v.to(dev) for k, v in sp.items()}

    last = {}

    def window(k, steps):
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            last[k] = train_on_batch(nets[k], opts[k], sp, cfg)
        e1.record()
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1)

    for k in nets:
        window(k, args.warmup)
    rates = {k: [] for k in nets}
    for _ in range(args.windows):
        for k in nets:
            rates[k].append(B * args.steps / (window(k, args.steps) / 1000.0))
    assert nets["native"]._native_grads_ready, "the native path did not run the native backward pass"
    phases = nets["native"].engine(commit=False).train_phase_ms()
    gpu, power = gpu_identity()
    nat, ag = statistics.median(rates["native"]), statistics.median(rates["autograd"])
    print(json.dumps({
        "metric": "training scenes/s (train_on_batch, median of windows)", "unit": "scenes/s",
        "native": nat, "autograd": ag, "speedup": nat / ag,
        "native_windows": rates["native"], "autograd_windows": rates["autograd"],
        "native_phases_ms": phases, "last_loss": {"native": last["native"], "autograd": last["autograd"]},
        "config": {"workload": "text-conditioned bedroom N=12 d=62 (text_dim 512, 9 cross-attention layers), Adam, "
                               "loss_separate + loss_iou, clip 10, random-init weights", "precision": args.precision,
                   "scenes": B, "steps_per_window": args.steps, "windows": args.windows, "warmup": args.warmup,
                   "text": "synthetic BERT hidden states [B, %d, 768]; %d tokens per description is an assumption" % (L, L)},
        "gpu": gpu, "power_limit": power}))


if __name__ == "__main__":
    main()
