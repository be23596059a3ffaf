"""Python host wrapper over the C ABI: owns one `ds_handle`, feeds it torch-allocated device memory.

PyTorch is plumbing here (device allocations, streams); every FLOP of the denoiser and of the
diffusion step runs in the CUDA library.  If the library or the GPU is missing, construction raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import capi
from .schedule import DiffusionTables
from .weights import NetSpec

_PREC = {"fp32": capi.DS_PREC_FP32, "bf16": capi.DS_PREC_BF16}
_BACKEND = {"auto": capi.DS_GEMM_AUTO, "simt": capi.DS_GEMM_SIMT, "tcgen05": capi.DS_GEMM_TCGEN05}
LOSS_KEYS = ["loss.bbox", "loss.trans", "loss.size", "loss.angle", "loss.class", "loss.object", "loss.objfeat",
             "loss.liou", "loss.bbox_iou"]


class DenoiserEngine:
    """One Unet1D + diffusion schedule on one GPU (reference: DiffusionPoint, diffusion_ddpm.py:721-803)."""

    def __init__(self, spec: NetSpec, num_objects: int, num_timesteps: int, precision: str = "bf16",
                 gemm_backend: str = "auto", device: int = 0, fuse_level: Optional[int] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("diffuscene_b200 needs a CUDA device (H100, sm_90a); there is no CPU path")
        self.lib = capi.load()
        self.spec = spec
        self.num_objects = num_objects
        self.num_timesteps = num_timesteps
        self.precision = precision
        self.device = torch.device("cuda", device)
        if fuse_level is None:      # fused GEMM epilogues exist for the tensor-core path only
            # 1: every conv + GroupNorm + FiLM + SiLU Block is one GEMM with the GroupNorm epilogue (k_gemm_wg)
            # 4: ... and to_out + LayerNorm + residual of the attention wrappers as one kernel (k_gemm_ln)
            # 5: ... and LayerNorm + to_qkv + linear-attention core as one kernel (k_ln_qkv_attn, N = 12 or 21)
            fuse_level = 5 if (precision == "bf16" and gemm_backend != "simt") else 0
        # levels 2 and 3 named the channels-on-tensor-memory-lanes GEMM of the sm_100a build; the library runs the
        # level-1 program for them, and this attribute reports the level that runs
        self.fuse_level = 1 if fuse_level in (2, 3) else fuse_level
        self.cfg = capi.make_config(spec, num_objects, num_timesteps, _PREC[precision], _BACKEND[gemm_backend],
                                    device, fuse_level)
        h = C.c_void_p()
        capi.check(self.lib.ds_create(C.byref(self.cfg), C.byref(h)))
        self.h = h
        self.d = spec.point_dim
        self.tables: Optional[DiffusionTables] = None
        self._keep: List[torch.Tensor] = []

    def close(self):
        if getattr(self, "h", None):
            self.lib.ds_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return capi.stream(self.device)

    # ---- weights --------------------------------------------------------------------------------
    def expected_weights(self) -> List[tuple]:
        return capi.expected_weights(self.lib, "ds", self.h)

    def load_state_dict(self, sd: Dict[str, torch.Tensor], prefix: str = "diffusion.model."):
        """Load reference-format weights (keys as in the reference checkpoints) and commit them."""
        for name, numel in self.expected_weights():
            key = prefix + name
            if key not in sd:
                raise KeyError("state dict is missing '%s'" % key)
            w = sd[key].detach().to(device="cpu", dtype=torch.float32).contiguous()
            if w.numel() != numel:
                raise ValueError("'%s' has %d elements, expected %d" % (key, w.numel(), numel))
            capi.check(self.lib.ds_load_weight(self.h, name.encode(), C.c_void_p(w.data_ptr()), numel))
        capi.check(self.lib.ds_commit_weights(self.h))

    # ---- schedule / conditioning ----------------------------------------------------------------
    def set_schedule(self, tables: DiffusionTables):
        s = capi.DsSchedule()
        s.T = tables.T
        s.mean_type = capi.MEAN_TYPES[tables.mean_type]
        keep = []
        for f in ("sqrt_ac", "sqrt_1mac", "sqrt_recip_ac", "sqrt_recipm1_ac", "coef1", "coef2", "sigma",
                  "alphas_cumprod", "loss_weight"):
            a = tables[f].detach().to(dtype=torch.float32, device="cpu").contiguous()
            keep.append(a)
            setattr(s, f, C.cast(C.c_void_p(a.data_ptr()), C.POINTER(C.c_float)))
        capi.check(self.lib.ds_set_schedule(self.h, C.byref(s)))
        vt = [tables[f].detach().to(dtype=torch.float32, device="cpu").contiguous()
              for f in ("posterior_log_variance_clipped", "model_log_variance", "log_one_minus_alphas_cumprod")]
        capi.check(self.lib.ds_set_vlb_schedule(self.h, tables.T, *[capi.ptr(a) for a in vt]))
        self.tables = tables

    def set_context(self, context: torch.Tensor, shared: Optional[bool] = None):
        """context: [B, N, cond_dim] or [N, cond_dim] (shared over the batch), fp32."""
        if context.dim() == 2:
            shared, batch = True, 0
        else:
            batch = context.shape[0]
            if shared is None:
                shared = False
            if shared:
                context = context[0]
        ctx = context.detach().to(device=self.device, dtype=torch.float32).contiguous()
        # with torch on its default stream the library works on its own non-blocking stream, which does not wait for
        # the kernels that produced `context`: let them finish first
        torch.cuda.current_stream(self.device).synchronize()
        capi.check(self.lib.ds_set_context(self.h, capi.ptr(ctx), batch, int(bool(shared)), self._stream()))
        torch.cuda.current_stream(self.device).synchronize()

    def set_context_cross(self, cross: Optional[torch.Tensor]):
        if cross is None:
            capi.check(self.lib.ds_set_context_cross(self.h, None, 0, 0, self._stream()))
            return
        c = cross.detach().to(device=self.device, dtype=torch.float32).contiguous()
        torch.cuda.current_stream(self.device).synchronize()      # as in set_context
        capi.check(self.lib.ds_set_context_cross(self.h, capi.ptr(c), c.shape[0], c.shape[1], self._stream()))
        torch.cuda.current_stream(self.device).synchronize()

    # ---- denoiser -------------------------------------------------------------------------------
    def forward(self, x_t: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """Unet1D.forward on device tensors: x_t [B, N, d] fp32, t [B] int64 -> [B, N, d] fp32."""
        assert x_t.is_cuda and x_t.dtype == torch.float32 and t.dtype == torch.int64
        x_t, t = x_t.contiguous(), t.to(self.device).contiguous()
        out = torch.empty_like(x_t)
        capi.check(self.lib.ds_denoise_forward(self.h, capi.ptr(x_t), capi.ptr(t), capi.ptr(out), x_t.shape[0],
                                               self._stream()))
        return out

    def forward_host(self, x_t: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """Same through HOST buffers (H2D + D2H inside the call)."""
        x_t = x_t.detach().to("cpu", torch.float32).contiguous()
        t = t.detach().to("cpu", torch.int64).contiguous()
        out = torch.empty_like(x_t)
        capi.check(self.lib.ds_denoise_forward_host(self.h, capi.ptr(x_t), capi.ptr(t), capi.ptr(out), x_t.shape[0]))
        return out

    # ---- sampling -------------------------------------------------------------------------------
    def _sample_args(self, batch, clip_denoised, num_steps, ddim, ddim_eta, seed, scene_offset, x_init, noise,
                     partial, partial_noise, traj_freq, traj, use_graph, ddim_times, chunk_scenes=0):
        a = capi.DsSampleArgs()
        a.chunk_scenes = int(chunk_scenes)
        a.batch, a.clip_denoised, a.num_steps = batch, int(clip_denoised), num_steps
        a.ddim, a.ddim_eta, a.seed, a.scene_offset = int(ddim), float(ddim_eta), seed, scene_offset
        a.x_init_dev = None if x_init is None else x_init.data_ptr()
        a.noise_dev = None if noise is None else noise.data_ptr()
        a.partial_dev = None if partial is None else partial.data_ptr()
        a.num_partial = 0 if partial is None else partial.shape[1]
        a.partial_noise_dev = None if partial_noise is None else partial_noise.data_ptr()
        a.traj_freq = traj_freq
        a.traj_dev = None if traj is None else traj.data_ptr()
        a.use_graph = int(use_graph)
        if ddim_times is not None:
            arr = (C.c_int32 * len(ddim_times))(*ddim_times)
            self._keep = [arr]
            a.ddim_times = C.cast(arr, C.POINTER(C.c_int32))
        return a

    def sample(self, batch: int, clip_denoised: bool = True, num_steps: int = 0, ddim: bool = False,
               ddim_eta: float = 0.0, seed: int = 0, scene_offset: int = 0, x_init: Optional[torch.Tensor] = None,
               noise: Optional[torch.Tensor] = None, partial: Optional[torch.Tensor] = None,
               partial_noise: Optional[torch.Tensor] = None, traj_freq: int = 0, use_graph: bool = True,
               ddim_times: Optional[Sequence[int]] = None, host_output: bool = False, chunk_scenes: int = 0):
        """p_sample_loop (diffusion_ddpm.py:355-371) and its trajectory / completion / DDIM variants.

        noise: optional [steps, B, N, d] injected step noise (loop order T-1 .. 0); x_init: optional x_T.
        Returns x_0 [B, N, d] (device, or host when host_output), or (x_0, trajectory) when traj_freq > 0."""
        dev = self.device
        f = lambda z: None if z is None else z.detach().to(device=dev, dtype=torch.float32).contiguous()
        x_init, noise, partial, partial_noise = f(x_init), f(noise), f(partial), f(partial_noise)
        if ddim and ddim_times is None:
            # the reference's grid expression, evaluated by torch itself (fp32 linspace, then .int()):
            # diffusion_ddpm.py:407-408 -- identical truncation when S does not divide T
            S = num_steps if num_steps > 0 else 50
            ddim_times = list(reversed(torch.linspace(-1, self.num_timesteps - 1, steps=S + 1).int().tolist()))
        traj = None
        if traj_freq > 0:
            if ddim:      # snapshots follow the timestep VALUES the loop visits (engine.cu: ts[i] % freq == 0 or i == 0)
                n_snap = sum(1 for i, tt in enumerate(ddim_times[:-1]) if tt % traj_freq == 0 or i == 0)
            else:
                n_snap = self.lib.ds_traj_count(num_steps if num_steps > 0 else self.num_timesteps, traj_freq)
            traj = torch.zeros((n_snap, batch, self.num_objects, self.d), device=dev, dtype=torch.float32)
        a = self._sample_args(batch, clip_denoised, num_steps, ddim, ddim_eta, seed, scene_offset, x_init, noise,
                              partial, partial_noise, traj_freq, traj, use_graph, ddim_times, chunk_scenes)
        torch.cuda.current_stream(dev).synchronize()
        if host_output:
            out = torch.empty((batch, self.num_objects, self.d), dtype=torch.float32).pin_memory()
            capi.check(self.lib.ds_sample_loop_host(self.h, C.byref(a), capi.ptr(out)))
        else:
            out = torch.empty((batch, self.num_objects, self.d), device=dev, dtype=torch.float32)
            capi.check(self.lib.ds_sample_loop(self.h, C.byref(a), capi.ptr(out), None))
        return (out, traj) if traj is not None else out

    def p_sample_step(self, x_t: torch.Tensor, t: torch.Tensor, noise: torch.Tensor, clip_denoised: bool):
        x_t, t, noise = x_t.contiguous(), t.to(self.device).contiguous(), noise.to(self.device).contiguous()
        out = torch.empty_like(x_t)
        capi.check(self.lib.ds_p_sample_step(self.h, capi.ptr(x_t), capi.ptr(t), capi.ptr(noise), int(clip_denoised),
                                             capi.ptr(out), x_t.shape[0], self._stream()))
        return out

    def q_sample(self, x0: torch.Tensor, t: torch.Tensor, noise: torch.Tensor):
        x0, t, noise = x0.contiguous(), t.to(self.device).contiguous(), noise.contiguous()
        out = torch.empty_like(x0)
        capi.check(self.lib.ds_q_sample(self.h, capi.ptr(x0), capi.ptr(t), capi.ptr(noise), capi.ptr(out), x0.shape[0],
                                        self._stream()))
        return out

    def p_losses(self, x0: torch.Tensor, t: torch.Tensor, noise: torch.Tensor, loss_separate: bool, loss_iou: bool,
                 bounds: Optional[Sequence[float]] = None):
        """Forward value of p_losses (diffusion_ddpm.py:520-652): (losses [B], dict of 9 scalar means)."""
        x0, t, noise = x0.contiguous(), t.to(self.device).contiguous(), noise.contiguous()
        B = x0.shape[0]
        losses = torch.empty(B, device=self.device, dtype=torch.float32)
        ld = torch.empty(9, device=self.device, dtype=torch.float32)
        barr = None
        if bounds is not None:
            barr = (C.c_float * 12)(*[float(v) for v in bounds])
        capi.check(self.lib.ds_p_losses(self.h, capi.ptr(x0), capi.ptr(t), capi.ptr(noise), int(loss_separate),
                                        int(loss_iou), barr, capi.ptr(losses), capi.ptr(ld), B, self._stream()))
        return losses, {k: ld[i] for i, k in enumerate(LOSS_KEYS)}

    # ---- variational bound ----------------------------------------------------------------------
    def vlb(self, x0: torch.Tensor, clip_denoised: bool = True, seed: int = 0, scene_offset: int = 0,
            noise: Optional[torch.Tensor] = None, use_graph: bool = True, prior_only: bool = False):
        """calc_bpd_loop (diffusion_ddpm.py:690-717) per scene: (vb [B, T], mse [B, T], prior [B]), fp32 device
        tensors, vb / prior in bits per dimension.  The q_sample draws come from Philox (seed, scene_offset + b) or from
        `noise` [T, B, N, d] in loop order T-1 .. 0.  prior_only: just _prior_bpd (:679-688), no denoiser pass; vb and
        mse are then None.  Conditioning is what set_context / set_context_cross last set."""
        dev = self.device
        x0 = x0.detach().to(device=dev, dtype=torch.float32).contiguous()
        B = x0.shape[0]
        noise = None if noise is None else noise.detach().to(device=dev, dtype=torch.float32).contiguous()
        a = capi.DsVlbArgs()
        a.batch, a.clip_denoised, a.x0_dev = B, int(bool(clip_denoised)), x0.data_ptr()
        a.seed, a.scene_offset = int(seed), int(scene_offset)
        a.noise_dev = None if noise is None else noise.data_ptr()
        a.use_graph = int(use_graph)
        T = self.num_timesteps
        vb = None if prior_only else torch.empty((B, T), device=dev, dtype=torch.float32)
        mse = None if prior_only else torch.empty((B, T), device=dev, dtype=torch.float32)
        prior = torch.empty(B, device=dev, dtype=torch.float32)
        torch.cuda.current_stream(dev).synchronize()
        capi.check(self.lib.ds_vlb_loop(self.h, C.byref(a), capi.ptr(vb), capi.ptr(mse), capi.ptr(prior), None))
        return vb, mse, prior

    # ---- native training ------------------------------------------------------------------------
    def flat_layout(self, prefix: str = "diffusion.model.") -> Dict[str, tuple]:
        """name -> (offset, numel) of every denoiser parameter inside the flat fp32 parameter / gradient buffers."""
        out, off = {}, 0
        for name, numel in self.expected_weights():
            out[prefix + name] = (off, numel)
            off += numel
        return out

    def train_step(self, flat_params: torch.Tensor, x0: torch.Tensor, t: torch.Tensor, noise: torch.Tensor,
                   context: torch.Tensor, shared: bool, loss_separate: bool, loss_iou: bool,
                   bounds: Optional[Sequence[float]] = None, flat_grads: Optional[torch.Tensor] = None,
                   want_dcontext: bool = True, grad_scale: float = 1.0, cross: Optional[torch.Tensor] = None,
                   want_dcross: bool = True):
        """Forward of p_losses + the native backward pass: (losses [B], loss dict, d(context) or None).
        Gradients of every denoiser parameter land in `flat_grads` (flat_layout order).
        Text-conditioned networks pass `cross` (context_cross [B, L, text_dim]); the result then has a fourth entry,
        d(cross) or None (ds_train_step_cross)."""
        assert flat_params.is_cuda and flat_params.dtype == torch.float32 and flat_params.is_contiguous()
        x0, t, noise = x0.contiguous(), t.to(self.device).contiguous(), noise.contiguous()
        ctx = context.detach().to(self.device, torch.float32).contiguous()
        B = x0.shape[0]
        losses = torch.empty(B, device=self.device, dtype=torch.float32)
        ld = torch.empty(9, device=self.device, dtype=torch.float32)
        dctx = torch.empty_like(ctx) if (want_dcontext and flat_grads is not None) else None
        barr = None if bounds is None else (C.c_float * 12)(*[float(v) for v in bounds])
        args = (self.h, capi.ptr(flat_params), capi.ptr(x0), capi.ptr(t), capi.ptr(noise), capi.ptr(ctx),
                0 if shared else B, int(bool(shared)), int(loss_separate), int(loss_iou), barr, float(grad_scale),
                capi.ptr(losses), capi.ptr(ld), capi.ptr(flat_grads), capi.ptr(dctx))
        if cross is None:
            capi.check(self.lib.ds_train_step(*args, B, self._stream()))
            return losses, {k: ld[i] for i, k in enumerate(LOSS_KEYS)}, dctx
        xc = cross.detach().to(self.device, torch.float32).contiguous()
        dxc = torch.empty_like(xc) if (want_dcross and flat_grads is not None) else None
        capi.check(self.lib.ds_train_step_cross(*args, capi.ptr(xc), xc.shape[1], capi.ptr(dxc), B, self._stream()))
        return losses, {k: ld[i] for i, k in enumerate(LOSS_KEYS)}, dctx, dxc

    def train_set_buckets(self, bounds: Sequence[int], events: Sequence["torch.cuda.Event"]):
        """Gradient buckets for the overlapped all-reduce (see ds_train_set_buckets); `events` are torch.cuda.Event
        objects (recorded once so that their cudaEvent_t exists), kept alive by this object."""
        n = len(events)
        self._bucket_events = list(events)
        arr_b = (C.c_int64 * (n + 1))(*[int(b) for b in bounds]) if n else None
        arr_e = (C.c_void_p * n)(*[C.c_void_p(e.cuda_event) for e in events]) if n else None
        capi.check(self.lib.ds_train_set_buckets(self.h, arr_b, n, arr_e))

    def train_phase_ms(self):
        out = (C.c_float * 6)()
        capi.check(self.lib.ds_train_phase_ms(self.h, out))
        return dict(zip(("pack", "forward", "loss", "backward", "cond_paths", "unpack"), [float(v) for v in out]))

    def train_read(self, kind: int, index) -> torch.Tensor:
        """One array of the training state after the last train_step with gradients (ds_train_read), fp32 on the
        device: kind is capi.DS_TRAIN_*, index a buffer / weight matrix / vector id of the train plan, or for
        DS_TRAIN_COND a name of capi.TRAIN_COND."""
        if kind == capi.DS_TRAIN_COND and isinstance(index, str):
            index = capi.TRAIN_COND[index]
        r, w = C.c_int32(), C.c_int32()
        capi.check(self.lib.ds_train_read(self.h, kind, int(index), None, 0, C.byref(r), C.byref(w), self._stream()))
        out = torch.empty(r.value * w.value, device=self.device, dtype=torch.float32)
        capi.check(self.lib.ds_train_read(self.h, kind, int(index), capi.ptr(out), out.numel(), C.byref(r), C.byref(w),
                                          self._stream()))
        return out[: r.value * w.value].view(r.value, w.value)

    # ---- debugging ------------------------------------------------------------------------------
    def enable_taps(self, on: bool = True):
        capi.check(self.lib.ds_enable_taps(self.h, int(on)))

    def read_tap(self, name: str, rows: int) -> torch.Tensor:
        cap = 1 << 26
        buf = torch.empty(cap, dtype=torch.float32)
        r, w = C.c_int32(), C.c_int32()
        capi.check(self.lib.ds_read_tap(self.h, name.encode(), capi.ptr(buf), cap, C.byref(r), C.byref(w)))
        return buf[: r.value * w.value].reshape(r.value, w.value)[:rows].clone()

    def launch_count(self) -> int:
        return int(self.lib.ds_launch_count(self.h))

    def graph_build_count(self) -> int:
        return int(self.lib.ds_graph_build_count(self.h))

    def profile_ops(self, batch: int):
        names = C.create_string_buffer(1 << 16)
        us = (C.c_float * 1024)()
        n = capi.check(self.lib.ds_profile_ops(self.h, batch, names, len(names), us, 1024))
        nm = names.value.decode().strip().split("\n")
        return [(nm[i], us[i]) for i in range(min(n, len(nm)))]
