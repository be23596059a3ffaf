"""Per-launch time and rate of the tensor-core GEMM (`k_gemm_wg`) in one diffusion step, grouped by epilogue.

    python scripts/profile_gemm_ops.py [--config bed_d97] [--batch 0] [--runs 5] [--plan-only]

Builds the engine of a `bench.py` config (same network, weights, schedule and context, the config's batch unless
`--batch` is given), runs `DenoiserEngine.profile_ops` (CUDA events around every op of an eager pass of the step
program, 5 timed passes after a warm-up pass) `--runs` times and takes each op's median.  The GEMM ops of the
exported step program are grouped into

  plain K=<K> N=<N>   bias / activation / residual epilogue, by shape
  gn time FiLM        conv + GroupNorm + time FiLM + SiLU, K = 512 (FiLM row looked up by the scene's t)
  gn context FiLM     ... context FiLM, K = 512 (per-object row, or per-token row for per-scene contexts)
  gn residual         ... no FiLM, + residual (the second Block of each ResnetBlock), K = 512
  gn K=<K>            every GroupNorm launch of another K (the skip-concatenated up-path inputs)

For each group: launches, microseconds per launch and TFLOP/s from 2 M N K.  `gn_over_plain_k512` compares the 512 x
512 GroupNorm launches with the plain launches of the same shape, the like-for-like cost of the GroupNorm epilogue.
Prints one JSON line with the card's name and power limit; writes nothing.  `--plan-only` prints the grouping of the
exported plan without a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CONFIGS, OP_GEMM, OP_GEMM_GN  # noqa: E402

FILM_TIME, FILM_CONTEXT = 1, 2      # Op::film of csrc/plan.h


def gpu_identity():
    import torch
    name = torch.cuda.get_device_name(torch.cuda.current_device())
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = None
    return name, out or None


def group_of(op) -> str:
    K = op["in0"]["k"] + op["in1"]["k"]
    if op["kind"] == OP_GEMM:
        return "plain K=%d N=%d" % (K, op["N"])
    if K != 512:
        return "gn K=%d" % K
    if op["film"] == FILM_TIME:
        return "gn time FiLM"
    if op["film"] == FILM_CONTEXT:
        return "gn context FiLM"
    if op["res"] >= 0:
        return "gn residual"
    return "gn other"


def gemm_groups(plan):
    """{group: [op, ...]} over the GEMM ops of an exported plan, in plan order."""
    groups = {}
    for op in plan["ops"]:
        if op["kind"] in (OP_GEMM, OP_GEMM_GN):
            groups.setdefault(group_of(op), []).append(op)
    return groups


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--config", default="bed_d97", choices=sorted(CONFIGS))
    ap.add_argument("--batch", type=int, default=0, help="scenes (0: the config's batch)")
    ap.add_argument("--runs", type=int, default=5, help="profile_ops calls; each op's median is kept")
    ap.add_argument("--plan-only", action="store_true", help="print the grouping of the exported plan (no GPU)")
    args = ap.parse_args()

    from diffuscene_b200 import capi
    from diffuscene_b200.weights import NetSpec, seeded_state_dict, unet1d_param_specs

    kw, N_OBJ, _, T, scenes, prec, _, label = CONFIGS[args.config]
    B = args.batch or scenes
    spec = NetSpec.from_net_kwargs(kw)
    if args.plan_only:
        cfg = capi.make_config(spec, N_OBJ, T, capi.DS_PREC_BF16, capi.DS_GEMM_AUTO, 0, 5)
        groups = gemm_groups(capi.plan_export(cfg))
        print(json.dumps({"config": args.config, "groups": {g: [o["name"] for o in ops] for g, ops in groups.items()},
                          "launches": {g: len(ops) for g, ops in groups.items()}}))
        return

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("profile_gemm_ops.py measures on a CUDA device; none is available")
    from diffuscene_b200.engine import DenoiserEngine
    from diffuscene_b200.schedule import get_betas, make_tables

    assert prec == "bf16", "k_gemm_wg runs in bf16 mode only"
    dev = torch.device("cuda", 0)
    eng = DenoiserEngine(spec, N_OBJ, T, precision=prec)
    eng.load_state_dict(seeded_state_dict(unet1d_param_specs(spec), seed=0))
    eng.set_schedule(make_tables(get_betas("linear", 1e-4, 0.02, T), "v", "fixedsmall"))
    g = torch.Generator().manual_seed(1)
    eng.set_context(torch.randn(N_OBJ, 128, generator=g).to(dev), shared=True)
    if spec.text_condition:
        eng.set_context_cross(torch.randn(B, 32, 512, generator=g).to(dev))

    runs = [dict(eng.profile_ops(B)) for _ in range(args.runs)]
    us = {name: statistics.median(r[name] for r in runs) for name in runs[0]}
    groups = gemm_groups(capi.plan_export(eng.cfg))
    M = B * N_OBJ

    def summary(ops):
        t = sum(us[o["name"]] for o in ops)
        flop = sum(2.0 * M * o["N"] * (o["in0"]["k"] + o["in1"]["k"]) for o in ops)
        return {"launches": len(ops), "us_total": round(t, 1), "us_per_launch": round(t / len(ops), 2),
                "tflops": round(flop / (t * 1e-6) / 1e12, 1)}

    table = {name: summary(ops) for name, ops in groups.items()}
    gn = [o for name, ops in groups.items() if name.startswith("gn") for o in ops]
    plain = [o for name, ops in groups.items() if name.startswith("plain") for o in ops]
    gn512 = [o for o in gn if o["in0"]["k"] + o["in1"]["k"] == 512 and o["N"] == 512]
    res = {
        "metric": "k_gemm_wg per-launch device time by epilogue, median of %d profile_ops runs" % args.runs,
        "config": {"name": args.config, "workload": label, "scenes": B, "tokens": M, "T": T},
        "groups": table, "gn_all": summary(gn), "plain_all": summary(plain),
        "step_us": round(sum(us.values()), 1),
        "gpu": None, "power_limit": None,
    }
    if gn512 and "plain K=512 N=512" in groups:
        res["gn_k512"] = summary(gn512)
        res["gn_over_plain_k512"] = round(res["gn_k512"]["tflops"] / table["plain K=512 N=512"]["tflops"], 3)
    res["gpu"], res["power_limit"] = gpu_identity()
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
