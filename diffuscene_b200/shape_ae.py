"""Object shape auto-encoder: the reference's `KLAutoEncoder` (scene_synthesis/networks/foldingnet_autoencoder.py:131-390)
on the CUDA library (ds_shape_ae_*).  It produces the per-object `objfeats_32` / `objfeats` latents that the lat32
denoiser configs and the retrieval catalogue consume.

`KLAutoEncoder` has the reference's submodule names, so its state dict has the reference's keys and reference
checkpoints load with `strict=True`.  The submodules only hold parameters and BatchNorm statistics: on the GPU every
parameter and running statistic is a view into one flat fp32 buffer (`_flat`) that the library reads, and the training
step writes the gradients into a second flat buffer (`_flat_grads`).  `native_backward = False` differentiates the
autograd twin (`networks.functional.shape_ae_forward`) instead, on any device.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from . import capi
from .networks import functional as Fn

GRID_POINTS = 2025


def _bn_modules(module: nn.Module) -> List[nn.BatchNorm1d]:
    return [m for m in module.modules() if isinstance(m, nn.BatchNorm1d)]


class _GraphLayer(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.conv = nn.Conv1d(cin, cout, 1)
        self.bn = nn.BatchNorm1d(cout)


class _Encoder(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv1d(12, 64, 1)
        self.conv2 = nn.Conv1d(64, 64, 1)
        self.conv3 = nn.Conv1d(64, 64, 1)
        self.bn1 = nn.BatchNorm1d(64)
        self.bn2 = nn.BatchNorm1d(64)
        self.bn3 = nn.BatchNorm1d(64)
        self.graph_layer1 = _GraphLayer(64, 128)
        self.graph_layer2 = _GraphLayer(128, 1024)
        self.conv4 = nn.Conv1d(1024, 512, 1)
        self.bn4 = nn.BatchNorm1d(512)


class _FoldingLayer(nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.layers = nn.Sequential(nn.Conv1d(cin, 512, 1), nn.BatchNorm1d(512), nn.ReLU(inplace=True),
                                    nn.Conv1d(512, 512, 1), nn.BatchNorm1d(512), nn.ReLU(inplace=True),
                                    nn.Conv1d(512, 3, 1))


class _Decoder(nn.Module):
    def __init__(self):
        super().__init__()
        self.fold1 = _FoldingLayer(512 + 2)
        self.fold2 = _FoldingLayer(512 + 3)


class ShapeAE:
    """One ds_shape_ae handle for objects of `num_points` points and a `latent_dim`-wide latent."""

    def __init__(self, latent_dim: int, num_points: int, device: int = 0):
        self.lib = capi.load()
        cfg = capi.DsShapeAeConfig()
        cfg.latent_dim, cfg.num_points, cfg.device = latent_dim, num_points, device
        self.cfg = cfg
        self.device = torch.device("cuda", device)
        self.h = C.c_void_p()
        capi.check(self.lib.ds_shape_ae_create(C.byref(cfg), C.byref(self.h)))
        self._inject = None

    def expected_weights(self) -> List[Tuple[str, int]]:
        return capi.expected_weights(self.lib, "ds_shape_ae", self.h)

    def _points(self, points):
        points = points.to(self.device, torch.float32).contiguous()
        if points.dim() != 3 or points.shape[1] != self.cfg.num_points or points.shape[2] != 3:
            raise ValueError("points must be [B, %d, 3], got %s" % (self.cfg.num_points, tuple(points.shape)))
        return points

    def forward(self, flat, points, eps, train: bool, keep: bool = False):
        points = self._points(points)
        B, F = points.shape[0], self.cfg.latent_dim
        eps = eps.to(self.device, torch.float32).contiguous()
        lat = torch.empty(B, F, device=self.device)
        kl = torch.empty(B, device=self.device)
        rec = torch.empty(B, GRID_POINTS, 3, device=self.device)
        capi.check(self.lib.ds_shape_ae_forward(self.h, capi.ptr(flat), capi.ptr(points), B, capi.ptr(eps), int(train),
                                                int(keep), capi.ptr(lat), capi.ptr(kl), capi.ptr(rec), capi.stream(self.device)))
        return kl, lat, rec

    def train_step(self, flat, grads, points, eps, kl_weight: float) -> torch.Tensor:
        """losses [3] = (loss, loss.cd, loss.kl) on the device; gradients into `grads`."""
        points = self._points(points)
        eps = eps.to(self.device, torch.float32).contiguous()
        losses = torch.empty(3, device=self.device)
        capi.check(self.lib.ds_shape_ae_train_step(self.h, capi.ptr(flat), capi.ptr(points), points.shape[0],
                                                   capi.ptr(eps), float(kl_weight), capi.ptr(grads), capi.ptr(losses),
                                                   capi.stream(self.device)))
        return losses

    def set_knn(self, idx: Optional[torch.Tensor]):
        """Replace the kNN searches by `idx` [3, B, P, 16] (None: search again)."""
        self._inject = None if idx is None else idx.to(self.device, torch.int32).contiguous()
        capi.check(self.lib.ds_shape_ae_set_knn(self.h, None if self._inject is None else
                                                C.c_void_p(self._inject.data_ptr())))

    def get_knn(self, batch: int) -> torch.Tensor:
        out = torch.empty(3, batch, self.cfg.num_points, 16, dtype=torch.int32, device=self.device)
        capi.check(self.lib.ds_shape_ae_get_knn(self.h, C.c_void_p(out.data_ptr()), capi.stream(self.device)))
        return out

    def close(self):
        if self.h:
            self.lib.ds_shape_ae_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _NativeLoss(torch.autograd.Function):
    """The training loss computed by ds_shape_ae_train_step; its backward exposes the flat gradient buffer (already
    computed) as the parameters' .grad."""

    @staticmethod
    def forward(ctx, model, anchor, loss):
        ctx.model = model
        return loss.clone()

    @staticmethod
    def backward(ctx, g):
        ctx.model._assign_native_grads(g)
        return None, None, None


class KLAutoEncoder(nn.Module):
    def __init__(self, latent_dim: int = 64, kl_weight: float = 0.001, num_points: int = 2048):
        super().__init__()
        self.latent_dim = latent_dim
        self.kl_weight = kl_weight
        self.num_points = num_points
        self.encoder = _Encoder()
        self.mean_fc = nn.Linear(512, latent_dim)
        self.logvar_fc = nn.Linear(512, latent_dim)
        self.fc = nn.Linear(latent_dim, 512)
        self.decoder = _Decoder()
        self.native_backward = True      # False: differentiate functional.shape_ae_forward with torch autograd
        self._ae: Optional[ShapeAE] = None
        self._flat = None
        self._flat_grads = None
        self._flat_names = None
        self._native_grads_ready = False
        self._overlap = None             # the denoiser's train_on_batch checks for an all-reduce in flight

    # ---- state ----------------------------------------------------------------------------------------------------
    def _tensors(self) -> Dict[str, torch.Tensor]:
        """Parameters and running statistics by reference name (the flat layout's order)."""
        return {k: v for k, v in self.state_dict(keep_vars=True).items() if not k.endswith("num_batches_tracked")}

    def mark_weights_dirty(self):
        pass      # the library reads the flat parameter buffer at every call: nothing to re-upload

    def _handle(self) -> ShapeAE:
        dev = self.fc.weight.device
        if dev.type != "cuda":
            raise RuntimeError("KLAutoEncoder runs on a CUDA device only (no CPU fallback); call .to('cuda') or set "
                               "native_backward = False for the autograd twin")
        if self._ae is None or self._ae.device != dev:
            self._ae = ShapeAE(self.latent_dim, self.num_points, dev.index or 0)
        return self._ae

    def _ensure_flat(self) -> ShapeAE:
        """Every parameter and running statistic as a view into ONE flat fp32 device buffer (ds_shape_ae order)."""
        ae = self._handle()
        named = self._tensors()
        if self._flat is not None:
            base = self._flat.data_ptr()
            if all(named[n].data_ptr() == base + 4 * off for n, off, _ in self._flat_names):
                return ae
        layout, off = [], 0
        for name, numel in ae.expected_weights():
            if name not in named or named[name].numel() != numel:
                raise RuntimeError("shape auto-encoder layout mismatch at %r" % name)
            layout.append((name, off, numel))
            off += numel
        flat = torch.empty(off, device=self.fc.weight.device, dtype=torch.float32)
        for name, o, n in layout:
            t = named[name]
            flat[o:o + n].copy_(t.detach().reshape(-1))
            t.data = flat[o:o + n].view(t.shape)
            if isinstance(t, nn.Parameter):
                t._ds_flat_owner = self
        self._flat, self._flat_names = flat, layout
        self._flat_grads = torch.zeros(off, device=flat.device, dtype=torch.float32)
        self._native_grads_ready = False
        return ae

    def _assign_native_grads(self, g):
        if not (torch.is_tensor(g) and g.numel() == 1 and float(g) == 1.0):
            self._flat_grads.mul_(g)
        named = dict(self.named_parameters())
        for name, off, n in self._flat_names:
            p = named.get(name)
            if p is None:
                continue
            view = self._flat_grads[off:off + n].view(p.shape)
            if p.grad is None or p.grad.data_ptr() == view.data_ptr():
                p.grad = view
            else:
                p.grad = p.grad + view
        self._native_grads_ready = True

    def _count_batch(self):
        for m in _bn_modules(self):
            m.num_batches_tracked += 1

    def _eps(self, batch: int) -> torch.Tensor:
        # the reference draws torch.randn(mean.shape) on the CPU generator and copies it over (:308-310)
        return torch.randn((batch, self.latent_dim)).to(self.fc.weight.device)

    # ---- reference interface ---------------------------------------------------------------------------------------
    def forward(self, pc):
        """pc [B, P, 3] -> (kl [B], latent [B, F], recon [B, 2025, 3]).  The native pass is not differentiable;
        get_loss is the training entry point."""
        eps = self._eps(pc.shape[0])
        if not self.native_backward:
            if self.training:
                self._count_batch()
            out = Fn.shape_ae_forward(self._tensors(), pc, eps, train=self.training)
            return out["kl"], out["latent"], out["recon"]
        ae = self._ensure_flat()
        if self.training:
            self._count_batch()
        with torch.no_grad():
            return ae.forward(self._flat, pc, eps, train=self.training, keep=True)

    def encode(self, x):
        """x [B, 3, P] -> (kl, latent)."""
        kl, lat, _ = self.forward(x.permute(0, 2, 1))
        return kl, lat

    def decode(self, lat):
        """latent [B, F] -> [B, 2025, 3], the decoder alone.  It runs the autograd twin's folding layers (torch ops) on
        the same parameters: the library decodes only inside `forward` / `get_loss`, which is where training and
        encoding spend their time."""
        t = self._tensors()
        code = torch.nn.functional.linear(lat, t["fc.weight"], t["fc.bias"])[:, :, None].repeat(1, 1, GRID_POINTS)
        rec = Fn.shape_ae_grid(lat.device)[None].repeat(lat.shape[0], 1, 1)
        for f in ("fold1", "fold2"):
            pre = "decoder.%s.layers." % f
            z = torch.cat([rec, code], dim=1)
            z = torch.relu(Fn._bn1d(Fn._conv1d(z, t, pre + "0"), t, pre + "1", self.training))
            z = torch.relu(Fn._bn1d(Fn._conv1d(z, t, pre + "3"), t, pre + "4", self.training))
            rec = Fn._conv1d(z, t, pre + "6")
        return rec.permute(0, 2, 1)

    def get_loss(self, samples):
        pc = samples["points"]
        if self.native_backward and self.training and torch.is_grad_enabled():
            ae = self._ensure_flat()
            self._count_batch()
            eps = self._eps(pc.shape[0])
            losses = ae.train_step(self._flat, self._flat_grads, pc, eps, self.kl_weight)
            self._native_grads_ready = False
            loss = _NativeLoss.apply(self, self.fc.weight, losses[0])
            return loss, {"loss.cd": losses[1], "loss.kl": losses[2]}
        if self.native_backward:
            kl, lat, rec = self.forward(pc)
            d1, d2, _, _ = chamfer_3d(pc.to(rec.device, torch.float32), rec)
        else:
            kl, lat, rec = self.forward(pc)
            d1, d2, _, _ = Fn.chamfer_torch(pc.to(rec.device, torch.float32), rec)
        loss_kl = torch.sum(kl) / kl.shape[0]
        loss_cd = (d1.mean(dim=1) + d2.mean(dim=1)).mean()
        return loss_cd + loss_kl * self.kl_weight, {"loss.cd": loss_cd, "loss.kl": loss_kl}


# ---- Chamfer distance -----------------------------------------------------------------------------------------------
def chamfer_3d(a, b):
    """dist1 [B, n], dist2 [B, m], idx1, idx2 (int32) of ds_chamfer_forward; no gradient."""
    lib = capi.load()
    a = a.to(torch.float32).contiguous()
    b = b.to(a.device, torch.float32).contiguous()
    B, n, m = a.shape[0], a.shape[1], b.shape[1]
    d1 = torch.empty(B, n, device=a.device)
    d2 = torch.empty(B, m, device=a.device)
    i1 = torch.empty(B, n, device=a.device, dtype=torch.int32)
    i2 = torch.empty(B, m, device=a.device, dtype=torch.int32)
    capi.check(lib.ds_chamfer_forward(capi.ptr(a), n, capi.ptr(b), m, B, capi.ptr(d1), capi.ptr(d2), capi.ptr(i1),
                                      capi.ptr(i2), capi.stream(a.device)))
    return d1, d2, i1, i2


class ChamferFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        a = a.to(torch.float32).contiguous()
        b = b.to(torch.float32).contiguous()
        d1, d2, i1, i2 = chamfer_3d(a, b)
        ctx.save_for_backward(a, b, i1, i2)
        ctx.mark_non_differentiable(i1, i2)
        return d1, d2, i1, i2

    @staticmethod
    def backward(ctx, g1, g2, _gi1, _gi2):
        a, b, i1, i2 = ctx.saved_tensors
        g1 = torch.zeros_like(a[..., 0]) if g1 is None else g1.contiguous()
        g2 = torch.zeros_like(b[..., 0]) if g2 is None else g2.contiguous()
        ga = torch.empty_like(a) if ctx.needs_input_grad[0] else None
        gb = torch.empty_like(b) if ctx.needs_input_grad[1] else None
        if ga is not None or gb is not None:
            capi.check(capi.load().ds_chamfer_backward(
                capi.ptr(a), a.shape[1], capi.ptr(b), b.shape[1], a.shape[0], capi.ptr(i1), capi.ptr(i2), capi.ptr(g1),
                capi.ptr(g2), capi.ptr(ga), capi.ptr(gb), capi.stream(a.device)))
        return ga, gb


class chamfer_3DDist(nn.Module):
    """The reference's ChamferDistancePytorch.chamfer3D.dist_chamfer_3D.chamfer_3DDist on ds_chamfer_*."""

    def forward(self, input1, input2):
        return ChamferFunction.apply(input1, input2)
