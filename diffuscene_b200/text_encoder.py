"""Frozen BERT text encoder on the CUDA library (ds_text_enc_*): the forward pass of Hugging Face `BertModel` up to
`last_hidden_state`, which the text-conditioned networks run on each tokenized description (the reference keeps
`bert-base-cased` frozen, scene_synthesis/networks/diffusion_scene_layout_ddpm.py:217-218, 285-287).

`BertTextEncoder` is built from a `BertModel` (or its config and state dict) and a precision and is called like the
model on the tokenizer's output: `enc(input_ids=..., attention_mask=..., token_type_ids=...)` returns the fp32
`last_hidden_state` [B, L, hidden] on the device, padded positions included.  Tokenization stays in Hugging Face.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Tuple

import torch

from . import capi

LN_EPS = 1e-12


def weight_inventory(layers: int, hidden: int, intermediate: int, vocab: int, max_positions: int,
                     type_vocab: int) -> List[Tuple[str, tuple]]:
    """(name, shape) of every `BertModel` state-dict tensor the encoder reads, in state-dict order, `pooler.*` left
    out; the order is the flat layout of ds_text_enc_expected_weight."""
    H, I = hidden, intermediate
    out = [("embeddings.word_embeddings.weight", (vocab, H)),
           ("embeddings.position_embeddings.weight", (max_positions, H)),
           ("embeddings.token_type_embeddings.weight", (type_vocab, H)),
           ("embeddings.LayerNorm.weight", (H,)), ("embeddings.LayerNorm.bias", (H,))]
    for l in range(layers):
        pre = "encoder.layer.%d." % l
        for n in ("query", "key", "value"):
            out += [(pre + "attention.self.%s.weight" % n, (H, H)), (pre + "attention.self.%s.bias" % n, (H,))]
        out += [(pre + "attention.output.dense.weight", (H, H)), (pre + "attention.output.dense.bias", (H,)),
                (pre + "attention.output.LayerNorm.weight", (H,)), (pre + "attention.output.LayerNorm.bias", (H,)),
                (pre + "intermediate.dense.weight", (I, H)), (pre + "intermediate.dense.bias", (I,)),
                (pre + "output.dense.weight", (H, I)), (pre + "output.dense.bias", (H,)),
                (pre + "output.LayerNorm.weight", (H,)), (pre + "output.LayerNorm.bias", (H,))]
    return out


def config_geometry(config) -> dict:
    """The encoder geometry of a `BertConfig`; ValueError for the semantics the kernels do not implement."""
    act = getattr(config, "hidden_act", "gelu")
    if act != "gelu":
        raise ValueError("text encoder implements hidden_act 'gelu' (erf form), not %r" % (act,))
    eps = getattr(config, "layer_norm_eps", LN_EPS)
    if eps != LN_EPS:
        raise ValueError("text encoder implements layer_norm_eps %g, not %g" % (LN_EPS, eps))
    pet = getattr(config, "position_embedding_type", "absolute")
    if pet not in (None, "absolute"):
        raise ValueError("text encoder implements absolute position embeddings, not %r" % (pet,))
    if getattr(config, "is_decoder", False):
        raise ValueError("text encoder implements the bidirectional encoder, not a decoder")
    return dict(layers=config.num_hidden_layers, hidden=config.hidden_size, intermediate=config.intermediate_size,
                vocab=config.vocab_size, max_positions=config.max_position_embeddings,
                type_vocab=config.type_vocab_size, heads=config.num_attention_heads)


def input_lengths(input_ids, attention_mask=None, token_type_ids=None, vocab: Optional[int] = None,
                  max_positions: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Host-side checks of a right-padded tokenizer batch; returns (ids int32 [B, L], lengths int32 [B]) on the CPU.
    ValueError for ids outside [0, vocab), a mask that is not a prefix mask with at least one token, non-zero token
    types, or a length above max_positions."""
    ids = torch.as_tensor(input_ids).cpu()
    if ids.dim() != 2 or ids.shape[0] < 1 or ids.shape[1] < 1 or ids.dtype.is_floating_point or ids.dtype == torch.bool:
        raise ValueError("input_ids must be a non-empty integer [B, L] tensor, got %s %s" % (ids.dtype, tuple(ids.shape)))
    B, L = ids.shape
    if max_positions is not None and L > max_positions:
        raise ValueError("sequence length %d exceeds max_position_embeddings %d" % (L, max_positions))
    if vocab is not None and (int(ids.min()) < 0 or int(ids.max()) >= vocab):
        raise ValueError("token ids must lie in [0, %d), got [%d, %d]" % (vocab, int(ids.min()), int(ids.max())))
    if attention_mask is None:
        lengths = torch.full((B,), L, dtype=torch.int64)
    else:
        mask = torch.as_tensor(attention_mask).cpu()
        if tuple(mask.shape) != (B, L):
            raise ValueError("attention_mask must be [%d, %d], got %s" % (B, L, tuple(mask.shape)))
        lengths = (mask != 0).sum(dim=1)
        prefix = torch.arange(L)[None] < lengths[:, None]
        if not bool(((mask == 1) == prefix).all()) or not bool(((mask == 0) == ~prefix).all()):
            raise ValueError("attention_mask must be a right-padding prefix mask of ones and zeros")
        if int(lengths.min()) < 1:
            raise ValueError("every sequence needs at least one token (an all-zero attention_mask row)")
    if token_type_ids is not None and bool((torch.as_tensor(token_type_ids).cpu() != 0).any()):
        raise ValueError("token_type_ids must be all zero (single-segment text)")
    return ids.to(torch.int32).contiguous(), lengths.to(torch.int32).contiguous()


class BertTextEncoder:
    """One ds_text_enc handle with the weights of a `BertModel` packed in `precision` ("fp32" parity mode or "bf16"
    tensor-core mode).  The handle is recreated with a larger token capacity when a batch needs it."""

    def __init__(self, model=None, precision: str = "bf16", config=None, state_dict=None, device: Optional[int] = None,
                 capacity: int = 4096):
        if model is not None:
            config, state_dict = model.config, model.state_dict()
        if config is None or state_dict is None:
            raise ValueError("BertTextEncoder needs a BertModel, or its config and state dict")
        self.geometry = config_geometry(config)
        self.precision = {"fp32": capi.DS_PREC_FP32, "bf16": capi.DS_PREC_BF16}[precision]
        g = self.geometry
        inv = weight_inventory(g["layers"], g["hidden"], g["intermediate"], g["vocab"], g["max_positions"],
                               g["type_vocab"])
        parts = []
        for name, shape in inv:
            if name not in state_dict:
                raise ValueError("state dict lacks %s" % name)
            t = state_dict[name]
            if tuple(t.shape) != shape:
                raise ValueError("%s has shape %s, expected %s" % (name, tuple(t.shape), shape))
            parts.append(t.detach().reshape(-1).to("cpu", torch.float32))
        self._flat_host = torch.cat(parts)      # kept to repack the weights when the handle grows
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.lib = capi.load()
        self.h = C.c_void_p()
        self.capacity = 0
        self.tap_layer = -1
        self._create(capacity)

    def _create(self, capacity: int):
        self.close()
        g = self.geometry
        cfg = capi.DsTextEncConfig()
        for k in ("layers", "hidden", "heads", "intermediate", "vocab", "max_positions", "type_vocab"):
            setattr(cfg, k, g[k])
        cfg.precision, cfg.capacity, cfg.device = self.precision, capacity, self.device.index
        h = C.c_void_p()
        capi.check(self.lib.ds_text_enc_create(C.byref(cfg), C.byref(h)))
        self.h, self.capacity = h, capacity
        flat = self._flat_host.to(self.device)
        capi.check(self.lib.ds_text_enc_set_weights(self.h, C.c_void_p(flat.data_ptr()), capi.stream(self.device)))
        if self.tap_layer >= 0:
            capi.check(self.lib.ds_text_enc_set_tap(self.h, self.tap_layer))

    def expected_weights(self) -> List[Tuple[str, int]]:
        return capi.expected_weights(self.lib, "ds_text_enc", self.h)

    def __call__(self, input_ids, attention_mask=None, token_type_ids=None, **unused) -> torch.Tensor:
        g = self.geometry
        ids, lengths = input_lengths(input_ids, attention_mask, token_type_ids, g["vocab"], g["max_positions"])
        B, L = ids.shape
        if B * L > self.capacity:
            self._create(B * L)
        ids_d, len_d = ids.to(self.device), lengths.to(self.device)
        out = torch.empty(B, L, g["hidden"], device=self.device, dtype=torch.float32)
        capi.check(self.lib.ds_text_enc_forward(self.h, C.c_void_p(ids_d.data_ptr()), C.c_void_p(len_d.data_ptr()),
                                                B, L, C.c_void_p(out.data_ptr()), capi.stream(self.device)))
        return out

    def set_tap(self, layer: int):
        """Tap encoder layer `layer` on the following forwards (ds_text_enc_set_tap); -1 turns the tap off."""
        capi.check(self.lib.ds_text_enc_set_tap(self.h, int(layer)))
        self.tap_layer = int(layer)

    def read(self, kind) -> torch.Tensor:
        """One array of the tapped layer of the last forward (ds_text_enc_read), fp32 [B * L, width] on the device:
        kind is a name of capi.TEXT_ENC_TAP (or its DS_TE_* value)."""
        if isinstance(kind, str):
            kind = capi.TEXT_ENC_TAP[kind]
        r, w = C.c_int32(), C.c_int32()
        capi.check(self.lib.ds_text_enc_read(self.h, kind, None, 0, C.byref(r), C.byref(w), capi.stream(self.device)))
        out = torch.empty(r.value, w.value, device=self.device, dtype=torch.float32)
        capi.check(self.lib.ds_text_enc_read(self.h, kind, C.c_void_p(out.data_ptr()), out.numel(), C.byref(r),
                                             C.byref(w), capi.stream(self.device)))
        return out

    def close(self):
        if self.h:
            self.lib.ds_text_enc_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
