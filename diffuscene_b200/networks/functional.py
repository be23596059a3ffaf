"""Differentiable (torch autograd) forward of the denoiser used ONLY for training on the GPU.

The native CUDA engine implements the forward of every op (sampling, validation loss); backward kernels are
not written yet, so `train_on_batch` differentiates this functional form with torch autograd on the same
parameters (a library path, stated as such in DESIGN.md).  Semantics: reference
scene_synthesis/networks/denoise_net.py:507-593 in token-major layout.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def _w(p):
    return p.reshape(p.shape[0], -1)


def _ws(w):
    w = _w(w)
    mean = w.mean(dim=1, keepdim=True)
    var = w.var(dim=1, unbiased=False, keepdim=True)
    return (w - mean) * torch.rsqrt(var + 1e-5)


def _ln(x, g):
    mean = x.mean(dim=-1, keepdim=True)
    var = x.var(dim=-1, unbiased=False, keepdim=True)
    return (x - mean) * torch.rsqrt(var + 1e-5) * g.reshape(1, 1, -1)


def _gn(x, gamma, beta, groups=8):
    B, N, C = x.shape
    xg = x.reshape(B, N, groups, C // groups)
    mean = xg.mean(dim=(1, 3), keepdim=True)
    var = xg.var(dim=(1, 3), unbiased=False, keepdim=True)
    return ((xg - mean) * torch.rsqrt(var + 1e-5)).reshape(B, N, C) * gamma + beta


class DenoiserFn:
    """Callable closure over a name -> parameter mapping (names without the 'diffusion.model.' prefix)."""

    def __init__(self, params, spec):
        self.p = params
        self.s = spec

    def block(self, n, x, ss=None):
        p = self.p
        h = F.linear(x, _ws(p[n + ".proj.weight"]), p[n + ".proj.bias"])
        h = _gn(h, p[n + ".norm.weight"], p[n + ".norm.bias"])
        if ss is not None:
            h = h * (ss[0] + 1) + ss[1]
        return F.silu(h)

    def res(self, n, x, cond):
        p = self.p
        e = F.linear(F.silu(cond), p[n + ".mlp.1.weight"], p[n + ".mlp.1.bias"])
        if e.dim() == 2:
            e = e[:, None, :]
        h = self.block(n + ".block2", self.block(n + ".block1", x, e.chunk(2, dim=-1)))
        if (n + ".res_conv.weight") in p:
            return h + F.linear(x, _w(p[n + ".res_conv.weight"]), p[n + ".res_conv.bias"])
        return h + x

    def _heads(self, t):
        B, N, HC = t.shape
        return t.reshape(B, N, 4, HC // 4)

    def linattn(self, n, x):
        p = self.p
        qkv = F.linear(_ln(x, p[n + ".fn.norm.g"]), _w(p[n + ".fn.fn.to_qkv.weight"]))
        q, k, v = (self._heads(t) for t in qkv.chunk(3, dim=-1))
        q = q.softmax(dim=-1) * (32 ** -0.5)
        k = k.softmax(dim=1)
        ctx = torch.einsum("bnhd,bnhe->bhde", k, v)
        o = torch.einsum("bhde,bnhd->bnhe", ctx, q).reshape(x.shape[0], x.shape[1], -1)
        y = F.linear(o, _w(p[n + ".fn.fn.to_out.0.weight"]), p[n + ".fn.fn.to_out.0.bias"])
        return _ln(y, p[n + ".fn.fn.to_out.1.g"]) + x

    def attn(self, n, x):
        p = self.p
        qkv = F.linear(_ln(x, p[n + ".fn.norm.g"]), _w(p[n + ".fn.fn.to_qkv.weight"]))
        q, k, v = (self._heads(t) for t in qkv.chunk(3, dim=-1))
        sim = torch.einsum("bihd,bjhd->bhij", q * (32 ** -0.5), k)
        o = torch.einsum("bhij,bjhd->bihd", sim.softmax(dim=-1), v).reshape(x.shape[0], x.shape[1], -1)
        return F.linear(o, _w(p[n + ".fn.fn.to_out.weight"]), p[n + ".fn.fn.to_out.bias"]) + x

    def xattn(self, n, x, text):
        p = self.p
        q = self._heads(F.linear(_ln(x, p[n + ".fn.norm.g"]), _w(p[n + ".fn.fn.to_q.weight"])))
        kv = F.linear(text, _w(p[n + ".fn.fn.to_kv.weight"]))
        k, v = (t.reshape(t.shape[0], t.shape[1], 4, 32) for t in kv.chunk(2, dim=-1))
        q = q.softmax(dim=-1) * (32 ** -0.5)
        k = k.softmax(dim=1)
        ctx = torch.einsum("blhd,blhe->bhde", k, v)
        o = torch.einsum("bhde,bnhd->bnhe", ctx, q).reshape(x.shape[0], x.shape[1], -1)
        y = F.linear(o, _w(p[n + ".fn.fn.to_out.0.weight"]), p[n + ".fn.fn.to_out.0.bias"])
        return _ln(y, p[n + ".fn.fn.to_out.1.g"]) + x

    def mlp3(self, n, x):
        p = self.p
        h = F.gelu(F.linear(x, _w(p[n + ".0.weight"]), p[n + ".0.bias"]))
        h = F.gelu(F.linear(h, _w(p[n + ".2.weight"]), p[n + ".2.bias"]))
        return F.linear(h, _w(p[n + ".4.weight"]), p[n + ".4.bias"])

    def __call__(self, x, t, context, context_cross=None):
        p, s = self.p, self.s
        b0 = s.bbox_dim
        if s.seperate_all:
            c0 = b0 + s.class_dim
            h = self.mlp3("class_embedf", x[..., b0:c0]) + self.mlp3("bbox_embedf", x[..., :b0])
            if s.objectness_dim > 0:
                h = h + self.mlp3("objectness_embedf", x[..., c0:c0 + s.objectness_dim])
            if s.objfeat_dim > 0:
                o0 = c0 + s.objectness_dim
                h = h + self.mlp3("objfeat_embedf", x[..., o0:o0 + s.objfeat_dim])
        else:
            h = x
        h = F.linear(h, _w(p["init_conv.weight"]), p["init_conv.bias"])
        r = h
        half = s.dim // 2
        freq = torch.exp(torch.arange(half, device=x.device, dtype=torch.float32) * -(math.log(10000) / (half - 1)))
        ang = t.to(torch.float32)[:, None] * freq[None, :]
        e = torch.cat([ang.sin(), ang.cos()], dim=-1)
        e = F.gelu(F.linear(e, p["time_mlp.1.weight"], p["time_mlp.1.bias"]))
        temb = F.linear(e, p["time_mlp.3.weight"], p["time_mlp.3.bias"])
        text = context_cross if s.text_condition else None
        skips = []
        for i in range(s.n_stages):
            d = "downs.%d" % i
            h = self.res(d + ".0", h, context)
            h = self.res(d + ".1", h, temb)
            skips.append(h)
            if text is not None:
                h = self.xattn(d + ".2", h, text)
            h = self.res(d + ".3", h, temb)
            h = self.linattn(d + ".4", h)
            skips.append(h)
            if i == s.n_stages - 1:
                h = F.linear(h, _w(p[d + ".5.weight"]), p[d + ".5.bias"])
        h = self.res("mid_block0", h, context)
        h = self.res("mid_block1", h, temb)
        if text is not None:
            h = self.xattn("mid_attn_cross", h, text)
        h = self.attn("mid_attn", h)
        h = self.res("mid_block2", h, temb)
        for i in range(s.n_stages):
            u = "ups.%d" % i
            h = self.res(u + ".0", h, context)
            h = self.res(u + ".1", torch.cat([h, skips.pop()], dim=-1), temb)
            if text is not None:
                h = self.xattn(u + ".2", h, text)
            h = self.res(u + ".3", torch.cat([h, skips.pop()], dim=-1), temb)
            h = self.linattn(u + ".4", h)
            if i == s.n_stages - 1:
                h = F.linear(h, _w(p[u + ".5.weight"]), p[u + ".5.bias"])
        h = self.res("final_res_block", torch.cat([h, r], dim=-1), temb)
        if s.seperate_all:
            outs = [self.mlp3("bbox_hidden2output", h), self.mlp3("class_hidden2output", h)]
            if s.objectness_dim > 0:
                outs.append(self.mlp3("objectness_hidden2output", h))
            if s.objfeat_dim > 0:
                outs.append(self.mlp3("objfeat_hidden2output", h))
            return torch.cat(outs, dim=-1)
        return F.linear(h, _w(p["final_conv.weight"]), p["final_conv.bias"])


def _frozen_bn(x, t, name):
    """FrozenBatchNorm2d (reference frozen_batchnorm.py): no eps, it was folded into running_var when frozen."""
    scale = t[name + ".weight"] * t[name + ".running_var"].rsqrt()
    bias = t[name + ".bias"] - t[name + ".running_mean"] * scale
    return x * scale.reshape(1, -1, 1, 1) + bias.reshape(1, -1, 1, 1)


def room_trunk(t, x):
    """The ResNet-18 trunk of the floor-plan encoder (torchvision resnet18 with the reference's conv1 and frozen
    BatchNorm, feature_extractors.py:19-47) up to the global average pool: mask [B, C, H, W] -> [B, 512].  `t` maps the
    names relative to `feature_extractor._feature_extractor.` to tensors.  The autograd twin of the CUDA encoder."""
    x = F.relu(_frozen_bn(F.conv2d(x, t["conv1.weight"], stride=2, padding=3), t, "bn1"))
    x = F.max_pool2d(x, 3, 2, 1)
    for L in range(1, 5):
        for j in range(2):
            pre = "layer%d.%d." % (L, j)
            stride = 2 if (L > 1 and j == 0) else 1
            out = F.relu(_frozen_bn(F.conv2d(x, t[pre + "conv1.weight"], stride=stride, padding=1), t, pre + "bn1"))
            out = _frozen_bn(F.conv2d(out, t[pre + "conv2.weight"], padding=1), t, pre + "bn2")
            idn = x
            if pre + "downsample.0.weight" in t:
                idn = _frozen_bn(F.conv2d(x, t[pre + "downsample.0.weight"], stride=stride), t, pre + "downsample.1")
            x = F.relu(out + idn)
    return F.adaptive_avg_pool2d(x, 1).flatten(1)


# ---- object shape auto-encoder (reference foldingnet_autoencoder.py:131-390) --------------------------------------------
def shape_ae_grid(device=None) -> torch.Tensor:
    """The decoder's fixed 2 x 2025 grid: np.meshgrid(linspace(-0.3, 0.3, 45) x 2), flattened (:253-258)."""
    import numpy as np
    xx = np.linspace(-0.3, 0.3, 45, dtype=np.float32)
    return torch.from_numpy(np.stack(np.meshgrid(xx, xx)).reshape(2, -1)).to(device)


def knn_reference(x, k: int = 16):
    """The reference's kNN (:59-76): x [B, C, N] -> [B, N, k], topk of the negated squared distance in its expanded
    form.  The order of equal distances is torch's; the CUDA kernel breaks ties by the lower index."""
    inner = -2 * torch.matmul(x.transpose(2, 1), x)
    xx = torch.sum(x ** 2, dim=1, keepdim=True)
    return (-xx - inner - xx.transpose(2, 1)).topk(k=k, dim=-1)[1]


def _gather_points(x, idx):
    """x [B, C, N], idx [B, N, k] -> [B, N, k, C] (index_points of :39-56)."""
    B, N, k = idx.shape
    pts = x.permute(0, 2, 1)
    return torch.gather(pts, 1, idx.reshape(B, -1, 1).expand(-1, -1, pts.shape[-1])).reshape(B, N, k, -1)


def _bn1d(x, t, name, train):
    return F.batch_norm(x, t[name + ".running_mean"], t[name + ".running_var"], t[name + ".weight"], t[name + ".bias"],
                        training=train, momentum=0.1, eps=1e-5)


def _conv1d(x, t, name):
    return F.conv1d(x, t[name + ".weight"], t[name + ".bias"])


def shape_ae_forward(t, points, eps, knn=None, train: bool = True):
    """The autograd twin of the CUDA shape auto-encoder: points [B, P, 3], eps [B, F] -> dict of kl [B], latent [B, F],
    recon [B, 2025, 3], the three stages' kNN indices (`knn`) and the features they searched (`knn_inputs`, [B, P, C]).  `t` maps the reference's state-dict names to tensors; in
    train mode BatchNorm uses batch statistics and updates the running statistics in `t` in place.  `knn` (three
    [B, P, 16] index tensors) replaces the kNN searches."""
    x = points.permute(0, 2, 1)
    b, _, n = x.shape
    used, inputs = [], []

    def nbrs(feat, stage):
        idx = knn_reference(feat) if knn is None else knn[stage].to(feat.device, torch.long)
        used.append(idx)
        inputs.append(feat.detach().permute(0, 2, 1))
        return _gather_points(feat, idx)

    knn_x = nbrs(x, 0)
    knn_x = knn_x - knn_x.mean(dim=2, keepdim=True)
    cov = torch.matmul(knn_x.permute(0, 1, 3, 2), knn_x).view(b, n, -1).permute(0, 2, 1)
    h = torch.cat([x, cov], dim=1)
    for i in (1, 2, 3):
        h = F.relu(_bn1d(_conv1d(h, t, "encoder.conv%d" % i), t, "encoder.bn%d" % i, train))
    for g in (1, 2):
        h = torch.max(nbrs(h, g), dim=2)[0].permute(0, 2, 1)
        pre = "encoder.graph_layer%d" % g
        h = F.relu(_bn1d(_conv1d(h, t, pre + ".conv"), t, pre + ".bn", train))
    code = torch.max(_bn1d(_conv1d(h, t, "encoder.conv4"), t, "encoder.bn4", train), dim=-1)[0]
    mean = F.linear(code, t["mean_fc.weight"], t["mean_fc.bias"])
    logvar = torch.clamp(F.linear(code, t["logvar_fc.weight"], t["logvar_fc.bias"]), -30.0, 20.0)
    lat = mean + torch.exp(0.5 * logvar) * eps
    kl = 0.5 * torch.mean(torch.pow(mean, 2) + torch.exp(logvar) - 1.0 - logvar, dim=[1])
    code = F.linear(lat, t["fc.weight"], t["fc.bias"])[:, :, None].repeat(1, 1, 2025)
    rec = shape_ae_grid(points.device)[None].repeat(b, 1, 1)
    for f in ("fold1", "fold2"):
        pre = "decoder.%s.layers." % f
        z = torch.cat([rec, code], dim=1)
        z = F.relu(_bn1d(_conv1d(z, t, pre + "0"), t, pre + "1", train))
        z = F.relu(_bn1d(_conv1d(z, t, pre + "3"), t, pre + "4", train))
        rec = _conv1d(z, t, pre + "6")
    return {"kl": kl, "latent": lat, "recon": rec.permute(0, 2, 1), "knn": used, "knn_inputs": inputs}


def chamfer_torch(a, b):
    """chamfer_3DDist restated with torch ops: a [B, n, 3], b [B, m, 3] -> dist1 [B, n], dist2 [B, m], idx1, idx2
    (int32), squared distances in the difference form."""
    d = ((a[:, :, None, :] - b[:, None, :, :]) ** 2).sum(-1)
    d1, i1 = d.min(dim=2)
    d2, i2 = d.min(dim=1)
    return d1, d2, i1.int(), i2.int()


def shape_ae_loss(out, points, kl_weight):
    """get_loss (:374-390) on the twin's outputs: (loss, loss_cd, loss_kl)."""
    d1, d2, _, _ = chamfer_torch(points, out["recon"])
    loss_kl = torch.sum(out["kl"]) / out["kl"].shape[0]
    loss_cd = (d1.mean(dim=1) + d2.mean(dim=1)).mean()
    return loss_cd + loss_kl * kl_weight, loss_cd, loss_kl
