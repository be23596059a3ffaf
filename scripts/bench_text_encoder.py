"""Throughput of the frozen BERT text encoder: the native encoder (ds_text_enc_*) against Hugging Face `BertModel`.

    python scripts/bench_text_encoder.py [--batches 128,1024] [--text-len 64] [--steps 5] [--warmup 2] [--windows 3]

Workload: random-init `bert-base-cased` geometry (12 layers, hidden 768, 12 heads, intermediate 3072, vocab 28996),
built offline.  Each batch holds descriptions of 16 .. 64 tokens right-padded to L = 64, the same assumed description
length as scripts/bench_train_text.py (an assumption, stated in the output).  128 is the text config's batch_size.

1. Encoder alone: native bf16, native fp32, HF fp32 (as the reference runs it: torch's default fp32 matmul, TF32 off)
   and HF under bf16 autocast.  ms per batch, sequences/s and achieved TFLOP/s from the FLOP count of `bert_flops`
   (the nominal count over all L keys; the native kernels skip key tiles past a sequence's length).
2. Text training step: text encoder + `train_on_batch` of the shipped text config (native denoiser step, fused Adam),
   with the native bf16 encoder against HF fp32 BERT.  The batch is tokenized once outside the timed windows; the
   tokenizer runs on the host and is the same for both paths.

Timed windows of the compared paths alternate, each bracketed by CUDA events after a device synchronise, after a
warm-up of every shape.  Prints one JSON line.  Writes nothing into the repository.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.bench_train_text import STATS, gpu_identity  # noqa: E402

BERT_BASE = dict(vocab_size=28996, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                 intermediate_size=3072, max_position_embeddings=512)


def bert_flops(B: int, L: int, layers: int = 12, H: int = 768, I: int = 3072) -> float:
    """Multiply-adds x 2 of the encoder: the four linear layers (2 H (3H + H + 2 I) per token) and the two attention
    products over all L keys (4 L H per token), per layer."""
    return float(B) * L * layers * (2.0 * H * (4 * H + 2 * I) + 4.0 * L * H)


def make_batch(B, L, vocab, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(16, L + 1, (B,), generator=g)
    lengths[0] = L
    mask = (torch.arange(L)[None] < lengths[:, None]).long()
    ids = torch.randint(1000, vocab, (B, L), generator=g) * mask
    return dict(input_ids=ids, attention_mask=mask, token_type_ids=torch.zeros_like(ids))


def timed(fns, steps, windows, warmup, dev):
    """Median ms per call of each fn over alternating windows of `steps` calls."""
    def window(fn, n):
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1) / n
    for fn in fns.values():
        window(fn, warmup)
    ms = {k: [] for k in fns}
    for _ in range(windows):
        for k, fn in fns.items():
            ms[k].append(window(fn, steps))
    return {k: statistics.median(v) for k, v in ms.items()}, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="128,1024")
    ap.add_argument("--text-len", type=int, default=64)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--no-train", action="store_true", help="skip the training-step comparison")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_text_encoder.py measures on a CUDA device; none is available")
    import transformers
    from diffuscene_b200.text_encoder import BertTextEncoder
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    bert = transformers.BertModel(transformers.BertConfig(**BERT_BASE)).eval()
    native = {p: BertTextEncoder(bert, precision=p, device=dev.index) for p in ("bf16", "fp32")}
    hf = bert.to(dev)
    L = args.text_len
    batches = [int(b) for b in args.batches.split(",")]
    enc_res = {}
    for B in batches:
        tok = make_batch(B, L, BERT_BASE["vocab_size"], B)
        tok_d = {k: v.to(dev) for k, v in tok.items()}

        def hf_fp32():
            with torch.no_grad():
                return hf(**tok_d).last_hidden_state

        def hf_autocast():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                return hf(**tok_d).last_hidden_state

        fns = {"native_bf16": lambda: native["bf16"](**tok), "native_fp32": lambda: native["fp32"](**tok),
               "hf_fp32": hf_fp32, "hf_bf16_autocast": hf_autocast}
        med, wins = timed(fns, args.steps, args.windows, args.warmup, dev)
        fl = bert_flops(B, L)
        enc_res[str(B)] = {k: {"ms": med[k], "sequences_per_s": B / (med[k] / 1e3), "tflops": fl / (med[k] / 1e3) / 1e12,
                               "windows_ms": wins[k]} for k in fns}

    train_res = None
    if not args.no_train:
        train_res = train_step_bench(args, bert, hf, native["bf16"], batches, dev)
    gpu, power = gpu_identity()
    print(json.dumps({
        "metric": "frozen BERT encoder: ms per batch (median of alternating windows)", "unit": "ms",
        "encoder": enc_res, "train_step": train_res,
        "config": {"geometry": "bert-base-cased, random init", "text_len": L,
                   "text": "descriptions of 16..%d tokens right-padded to L = %d; %d tokens per description is an "
                           "assumption" % (L, L, L),
                   "flops_per_batch": {str(B): bert_flops(B, L) for B in batches},
                   "steps_per_window": args.steps, "windows": args.windows, "warmup": args.warmup},
        "gpu": gpu, "power_limit": power}))


def train_step_bench(args, bert, hf, enc, batches, dev):
    import yaml
    from scene_synthesis.networks import build_network, optimizer_factory
    tmp = tempfile.mkdtemp(prefix="ds_bench_text_enc_")
    stats = os.path.join(tmp, "stats.json")
    with open(stats, "w") as f:
        json.dump(STATS, f)
    cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "text", "diffusion_bedrooms_instancond_lat32_v_bert.yaml")))
    cfg["network"]["diffusion_kwargs"]["train_stats_file"] = stats
    torch.manual_seed(0)
    net, train_on_batch, _ = build_network(30, 23, cfg, None, device=dev, precision="bf16")
    opt = optimizer_factory(cfg["training"], net.parameters())
    N, L = 12, args.text_len
    out = {}
    for B in batches:
        g = torch.Generator().manual_seed(1)
        cls = torch.randint(0, 22, (B, N), generator=g)
        sp = dict(translations=torch.rand(B, N, 3, generator=g) * 2 - 1, sizes=torch.rand(B, N, 3, generator=g) * 2 - 1,
                  angles=torch.nn.functional.normalize(torch.randn(B, N, 2, generator=g), dim=-1),
                  class_labels=torch.nn.functional.one_hot(cls, 22).float() * 2 - 1,
                  objfeats_32=torch.rand(B, N, 32, generator=g) * 2 - 1, room_layout=torch.zeros(B, 1, 64, 64))
        sp = {k: v.to(dev) for k, v in sp.items()}
        tok = make_batch(B, L, BERT_BASE["vocab_size"], B)
        tok_d = {k: v.to(dev) for k, v in tok.items()}

        def step_native():
            train_on_batch(net, opt, dict(sp, description=enc(**tok)), cfg)

        def step_hf():
            with torch.no_grad():
                hid = hf(**tok_d).last_hidden_state
            train_on_batch(net, opt, dict(sp, description=hid), cfg)

        med, wins = timed({"native_encoder": step_native, "hf_fp32_encoder": step_hf}, args.steps, args.windows,
                          args.warmup, dev)
        assert net._native_grads_ready, "the native denoiser step did not run"
        out[str(B)] = {k: {"ms": med[k], "scenes_per_s": B / (med[k] / 1e3), "windows_ms": wins[k]} for k in med}
        out[str(B)]["speedup"] = med["hf_fp32_encoder"] / med["native_encoder"]
    out["workload"] = ("text encoder + train_on_batch of the shipped text config (bf16 native denoiser step, fused Adam, "
                       "N = 12, 9 cross-attention layers); tokenization outside the timed step")
    return out


if __name__ == "__main__":
    main()
