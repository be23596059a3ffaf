"""Run under torchrun with 2 ranks on a machine with two GPUs (python -m torch.distributed.run --nproc-per-node 2):
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tests/gpu_dp_train_check.py
Data-parallel native training on NCCL: every rank takes its shard through model.get_loss().backward() (native backward,
bucketed all-reduce overlapped with it) and the averaged gradient must equal the gradient of the full batch computed
by one rank alone; then two optimizer iterations keep the replicas bit-identical."""
import json
import os
import sys

import torch
import torch.distributed as dist
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.cases import STATS  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    from scene_synthesis.networks import build_network, optimizer_factory
    cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "uncond/diffusion_bedrooms_instancond_lat32_v.yaml")).read().replace("\r", ""))
    stats = "/tmp/ds_dp_stats_%d.json" % rank
    json.dump(STATS, open(stats, "w"))
    cfg["network"]["diffusion_kwargs"]["train_stats_file"] = stats
    torch.manual_seed(5)                                   # same initial weights on every rank
    net, train_on_batch, _ = build_network(0, 23, cfg, None, device=dev, precision="fp32")
    Bs = 6
    g = torch.Generator().manual_seed(1)
    B = Bs * world
    cls = torch.randint(0, 22, (B, 12), generator=g)
    full = dict(translations=torch.rand(B, 12, 3, generator=g) * 2 - 1, sizes=torch.rand(B, 12, 3, generator=g) * 2 - 1,
                angles=torch.nn.functional.normalize(torch.randn(B, 12, 2, generator=g), dim=-1),
                class_labels=torch.nn.functional.one_hot(cls, 22).float() * 2 - 1,
                objfeats_32=torch.rand(B, 12, 32, generator=g) * 2 - 1, room_layout=torch.zeros(B, 1, 64, 64))
    t = torch.randint(0, 1000, (B,), generator=g)
    noise = torch.randn(B, 12, 62, generator=g)
    sl = slice(rank * Bs, (rank + 1) * Bs)
    shard = {k: v[sl].to(dev) for k, v in full.items()}
    # ---- data-parallel gradient (native backward + overlapped bucketed all-reduce)
    loss, _ = net.get_loss(shard, t=t[sl], noise=noise[sl])
    loss.backward()
    assert net._overlap is not None and len(net._overlap.events) >= 4
    from diffuscene_b200.parallel import allreduce_flat
    allreduce_flat(None, [p for p in net.parameters() if p.grad is not None and not hasattr(p, "_ds_flat_owner")])
    torch.cuda.synchronize()
    dp_flat = net._flat_grads.clone()
    dp_pos = net.positional_embedding.grad.clone()
    # ---- the same gradient from the full batch on this rank alone (engine call, no collective)
    eng = net.engine(commit=False)
    target = net._pack_target({k: v.to(dev) for k, v in full.items()}).float()
    gfull = torch.zeros_like(dp_flat)
    _, _, dctx = eng.train_step(net._flat, target, t.to(dev), noise.to(dev), net.positional_embedding.detach(), True,
                                net.loss_separate, net.loss_iou, net.bounds, flat_grads=gfull, grad_scale=1.0)
    torch.cuda.synchronize()
    err = (dp_flat - gfull).abs().max().item() / gfull.abs().max().item()
    err_pos = (dp_pos - dctx).abs().max().item() / dctx.abs().max().item()
    # ---- two optimizer iterations: replicas stay identical
    opt = optimizer_factory(cfg["training"], net.parameters())
    for it in range(2):
        torch.manual_seed(50 + it + 1000 * rank)
        train_on_batch(net, opt, shard, cfg)
    torch.cuda.synchronize()
    chk = net._flat.double().sum().reshape(1)
    both = [torch.zeros_like(chk) for _ in range(world)]
    dist.all_gather(both, chk)
    same = all(torch.equal(both[0], b) for b in both)
    if rank == 0:
        print(json.dumps({"dp_grad_rel_err": err, "dp_pos_emb_rel_err": err_pos, "replicas_identical_after_2_iters": same,
                          "buckets": len(net._overlap.events)}))
        assert err < 1e-4 and err_pos < 1e-4 and same
        print("DP TRAIN CHECK OK")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
