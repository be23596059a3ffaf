"""Shape auto-encoder golden cases: seeded weights and point clouds shared by the golden maker
(tests/golden/make_golden_shape_ae.py) and the tests."""
import math

import numpy as np
import torch

from diffuscene_b200.synthetic import SyntheticShapes

SAE_CASES = {
    # F = 32, the lat32 configs' latent; train mode; the dataset's 2048 points drawn with replacement (duplicates)
    "sae_a": dict(latent_dim=32, B=4, P=2048, train=True, seed=11, kl_weight=0.001),
    # F = 64, eval mode with non-trivial running statistics
    "sae_b": dict(latent_dim=64, B=3, P=1000, train=False, seed=12, kl_weight=0.001),
}
FULL_GRAD_MAX = 70000
# Biases whose exact gradient is zero: each feeds a BatchNorm (directly, or as a per-channel constant through fc into
# both folding layers, or through fold1's output into fold2's first conv), which removes any per-channel shift.  Their
# computed gradients are rounding noise, so tests bound them instead of matching them.
ZERO_GRAD = {"encoder.conv1.bias", "encoder.conv2.bias", "encoder.conv3.bias", "encoder.conv4.bias",
             "encoder.graph_layer1.conv.bias", "encoder.graph_layer2.conv.bias", "fc.bias",
             "decoder.fold1.layers.0.bias", "decoder.fold1.layers.3.bias", "decoder.fold1.layers.6.bias",
             "decoder.fold2.layers.0.bias", "decoder.fold2.layers.3.bias"}
ZERO_GRAD_BOUND = 1e-4      # gradients of tensors below this many elements are stored in full


def sae_points(case) -> torch.Tensor:
    ds = SyntheticShapes(length=case["B"], num_points=case["P"], seed=case["seed"])
    return torch.stack([ds[i]["points"] for i in range(case["B"])])


def sae_state_dict(ref_sd, case):
    """Seeded values for every tensor of a reference-format state dict: conv / linear weights and biases uniform in
    +-1/sqrt(fan_in) (torch's default range), BatchNorm affine near (1, 0), and in eval cases running statistics away
    from (0, 1)."""
    g = torch.Generator().manual_seed(case["seed"])
    out = {}
    fan_in = None
    for k, v in ref_sd.items():
        if k.endswith("num_batches_tracked"):
            out[k] = v.clone()
            continue
        if v.dim() >= 2:
            fan_in = int(math.prod(v.shape[1:]))
        bound = 1.0 / math.sqrt(fan_in)
        u = lambda: (torch.rand(v.shape, generator=g) * 2 - 1) * bound
        is_bn = v.dim() == 1 and (k.replace(".weight", ".running_mean").replace(".bias", ".running_mean")
                                  .replace(".running_var", ".running_mean") in ref_sd) and \
            (k.rsplit(".", 1)[0] + ".running_mean") in ref_sd
        if is_bn:
            leaf = k.rsplit(".", 1)[1]
            if leaf == "weight":
                out[k] = 1.0 + 0.1 * torch.randn(v.shape, generator=g)
            elif leaf == "bias":
                out[k] = 0.1 * torch.randn(v.shape, generator=g)
            elif leaf == "running_mean":
                out[k] = 0.1 * torch.randn(v.shape, generator=g) if not case["train"] else torch.zeros(v.shape)
            else:
                out[k] = 0.5 + torch.rand(v.shape, generator=g) if not case["train"] else torch.ones(v.shape)
        elif v.dim() >= 2:
            out[k] = u()
        else:
            out[k] = u()
    return out


def probe(name, shape) -> torch.Tensor:
    g = torch.Generator().manual_seed(sum(ord(c) for c in name))
    return torch.randn(tuple(shape), generator=g)


def check_knn(x, idx, k=16, rtol=1e-6):
    """fp64 check of kNN indices: x [B, P, C], idx [B, P, k].  Each row must hold k distinct indices in ascending
    fp64 distance, the k nearest points; a neighbour may differ from the exact order or set only where its fp64
    distance ties the one it swaps with (or the 16th) within `rtol` relative.  Returns the number of such swaps."""
    x = torch.as_tensor(x, dtype=torch.float64)
    idx = torch.as_tensor(idx, dtype=torch.int64)
    B, P, _ = x.shape
    assert tuple(idx.shape) == (B, P, k)
    assert int(idx.min()) >= 0 and int(idx.max()) < P
    swaps = 0
    for b in range(B):
        d = torch.cdist(x[b], x[b]) ** 2 if x.shape[-1] > 3 else ((x[b][:, None] - x[b][None]) ** 2).sum(-1)
        got = torch.gather(d, 1, idx[b])
        srt = d.sort(dim=1).values
        kth = srt[:, k - 1:k]
        tol = rtol * kth.abs() + 1e-12
        assert bool((idx[b].sort(dim=1).values.diff(dim=1) > 0).all()), "repeated neighbour"
        assert bool((got <= kth + tol).all()), "a neighbour beyond the 16th nearest"
        assert bool((got.diff(dim=1) >= -tol).all()), "neighbours out of order"
        swaps += int(((got - srt[:, :k]).abs() > 0).sum())
    return swaps
