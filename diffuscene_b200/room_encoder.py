"""Floor-plan encoder: the ResNet-18 trunk of the reference's room-mask feature extractor
(scene_synthesis/networks/feature_extractors.py:19-47, FrozenBatchNorm2d) on the CUDA library (ds_room_enc_*).

`RoomMaskEncoder` wraps one encoder handle: mask [B, C, H, W] fp32 -> trunk features [B, 512] fp32 (the input of the
reference's fc head), and the backward pass into a flat gradient buffer.  `RoomEncoderFn` is the autograd node that
lets the trunk's parameters receive their gradients as `.grad`.  The fc head and `fc_room_f` stay torch modules.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Tuple

import torch

from . import capi

BN_KEYS = ("weight", "bias", "running_mean", "running_var")


def trunk_specs(input_channels: int = 1) -> List[Tuple[str, tuple, bool]]:
    """(name, shape, is_buffer) of every trunk tensor in the reference's state-dict order (names relative to
    `feature_extractor._feature_extractor.`); the order is the flat layout of ds_room_enc_expected_weight."""
    out = []

    def conv(name, cin, cout, k):
        out.append((name + ".weight", (cout, cin, k, k), False))

    def bn(name, c):
        for key in BN_KEYS:
            out.append(("%s.%s" % (name, key), (c,), key.startswith("running")))

    conv("conv1", input_channels, 64, 7)
    bn("bn1", 64)
    cin = 64
    for L in range(4):
        cout = 64 << L
        for j in range(2):
            pre = "layer%d.%d." % (L + 1, j)
            conv(pre + "conv1", cin, cout, 3)
            bn(pre + "bn1", cout)
            conv(pre + "conv2", cout, cout, 3)
            bn(pre + "bn2", cout)
            if L > 0 and j == 0:
                conv(pre + "downsample.0", cin, cout, 1)
                bn(pre + "downsample.1", cout)
            cin = cout
    return out


class RoomMaskEncoder:
    """One ds_room_enc handle.  Parameters travel as one flat fp32 device buffer in `trunk_specs` order (running
    statistics included); gradients land in a buffer of the same layout."""

    def __init__(self, input_channels: int = 1, height: int = 64, width: int = 64, precision: str = "bf16",
                 device: int = 0):
        self.lib = capi.load()
        cfg = capi.DsRoomEncConfig()
        cfg.precision = {"fp32": capi.DS_PREC_FP32, "bf16": capi.DS_PREC_BF16}[precision]
        cfg.input_channels, cfg.height, cfg.width, cfg.device = input_channels, height, width, device
        self.cfg = cfg
        self.device = torch.device("cuda", device)
        self.h = C.c_void_p()
        capi.check(self.lib.ds_room_enc_create(C.byref(cfg), C.byref(self.h)))
        self.generation = 0      # bumped by every forward that keeps its activations

    def expected_weights(self) -> List[Tuple[str, int]]:
        return capi.expected_weights(self.lib, "ds_room_enc", self.h)

    def forward(self, flat: torch.Tensor, mask: torch.Tensor, keep: bool = False) -> torch.Tensor:
        cfg = self.cfg
        mask = mask.to(self.device, torch.float32).contiguous()
        if mask.dim() != 4 or tuple(mask.shape[1:]) != (cfg.input_channels, cfg.height, cfg.width):
            raise ValueError("room mask must be [B, %d, %d, %d], got %s" % (cfg.input_channels, cfg.height, cfg.width,
                                                                            tuple(mask.shape)))
        feat = torch.empty(mask.shape[0], 512, device=self.device, dtype=torch.float32)
        capi.check(self.lib.ds_room_enc_forward(self.h, C.c_void_p(flat.data_ptr()), C.c_void_p(mask.data_ptr()),
                                                mask.shape[0], C.c_void_p(feat.data_ptr()), int(keep), capi.stream(self.device)))
        if keep:
            self.generation += 1
        return feat

    def backward(self, dfeat: torch.Tensor, grads: torch.Tensor):
        dfeat = dfeat.to(self.device, torch.float32).contiguous()
        capi.check(self.lib.ds_room_enc_backward(self.h, C.c_void_p(dfeat.data_ptr()), C.c_void_p(grads.data_ptr()),
                                                 capi.stream(self.device)))

    def read(self, kind, index: int = 0) -> torch.Tensor:
        """One array of the encoder's state (ds_room_enc_read), fp32 [rows, width] on the device: kind is a name of
        capi.ROOM_ENC_STATE (or its DS_RE_* value), index a block (0 .. 7) or a conv in expected-weight order."""
        if isinstance(kind, str):
            kind = capi.ROOM_ENC_STATE[kind]
        r, w = C.c_int32(), C.c_int32()
        capi.check(self.lib.ds_room_enc_read(self.h, kind, int(index), None, 0, C.byref(r), C.byref(w),
                                             capi.stream(self.device)))
        out = torch.empty(r.value, w.value, device=self.device, dtype=torch.float32)
        capi.check(self.lib.ds_room_enc_read(self.h, kind, int(index), C.c_void_p(out.data_ptr()), out.numel(),
                                             C.byref(r), C.byref(w), capi.stream(self.device)))
        return out

    def close(self):
        if self.h:
            self.lib.ds_room_enc_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class RoomEncoderFn(torch.autograd.Function):
    """feat = trunk(mask) with the forward and backward pass in the CUDA library.  `params` are the trainable trunk
    tensors (views into `flat`, in `trunk_specs` order); their gradients come back as a copy of `grads`."""

    @staticmethod
    def forward(ctx, mask, enc, flat, grads, slices, *params):
        feat = enc.forward(flat, mask, keep=True)
        ctx.enc, ctx.grads, ctx.slices, ctx.gen = enc, grads, slices, enc.generation
        return feat

    @staticmethod
    def backward(ctx, g):
        if ctx.enc.generation != ctx.gen:
            raise RuntimeError("the room encoder ran another forward pass before this backward pass")
        ctx.enc.backward(g, ctx.grads)
        # a copy: autograd may keep a returned gradient as the parameter's .grad, and the flat buffer is rewritten by
        # the next backward pass
        grads = ctx.grads.clone()
        return (None, None, None, None, None) + tuple(grads[o:o + n].view(shape) for o, n, shape in ctx.slices)
