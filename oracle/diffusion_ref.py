"""ORACLE (test infrastructure, not product code): CPU restatement of the DDPM process.

Restates the arithmetic of `GaussianDiffusion` (reference scene_synthesis/networks/diffusion_ddpm.py)
as plain functions over a `Schedule` of fp32 tables: q_sample (:276-286), v / eps / x0
conversions (:217-240), one reverse step (:305-352), the sampling loops (:355-398, :447-506), a
working DDIM loop following the formula at :401-444 (the reference's own is dead code), and
p_losses with the IoU regulariser (:520-665, loss.py:7-102).

Pinned against the live reference by tests/golden/make_golden.py.  Only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import torch

Tensor = torch.Tensor
DenoiseFn = Callable[[Tensor, Tensor], Tensor]       # (x_t [B,N,d], t [B] int64) -> model output


def make_betas(schedule_type: str, b_start: float, b_end: float, T: int) -> np.ndarray:
    """diffusion_ddpm.py:45-91 (the `cosine` branch of the reference is broken and not restated)."""
    if schedule_type == "linear":
        return np.linspace(b_start, b_end, T)
    if schedule_type.startswith("warm"):
        frac = float(schedule_type[4:])
        betas = b_end * np.ones(T, dtype=np.float64)
        w = int(T * frac)
        betas[:w] = np.linspace(b_start, b_end, w, dtype=np.float64)
        return betas
    raise NotImplementedError(schedule_type)


@dataclass
class Schedule:
    """fp32 tables of diffusion_ddpm.py:168-203 (fp64 cumprod -> fp32, everything else in fp32)."""
    T: int
    betas: Tensor
    alphas_cumprod: Tensor
    alphas_cumprod_prev: Tensor
    sqrt_ac: Tensor
    sqrt_1mac: Tensor
    sqrt_recip_ac: Tensor
    sqrt_recipm1_ac: Tensor
    post_var: Tensor
    post_logvar_clipped: Tensor
    coef1: Tensor
    coef2: Tensor
    loss_weight: Tensor
    mean_type: str
    var_type: str


def make_schedule(betas64: np.ndarray, mean_type: str = "v", var_type: str = "fixedsmall") -> Schedule:
    betas64 = betas64.astype(np.float64)
    alphas64 = 1.0 - betas64
    ac = torch.from_numpy(np.cumprod(alphas64, axis=0)).float()
    ac_prev = torch.from_numpy(np.append(1.0, ac[:-1].numpy())).float()
    betas = torch.from_numpy(betas64).float()
    alphas = torch.from_numpy(alphas64).float()
    post_var = betas * (1.0 - ac_prev) / (1.0 - ac)
    snr = ac / (1 - ac)
    lw = {"eps": torch.ones_like(snr), "x0": snr, "v": snr / (snr + 1)}[mean_type]
    return Schedule(
        T=len(betas64), betas=betas, alphas_cumprod=ac, alphas_cumprod_prev=ac_prev,
        sqrt_ac=torch.sqrt(ac), sqrt_1mac=torch.sqrt(1.0 - ac),
        sqrt_recip_ac=torch.sqrt(1.0 / ac), sqrt_recipm1_ac=torch.sqrt(1.0 / ac - 1),
        post_var=post_var,
        post_logvar_clipped=torch.log(torch.max(post_var, 1e-20 * torch.ones_like(post_var))),
        coef1=betas * torch.sqrt(ac_prev) / (1.0 - ac),
        coef2=(1.0 - ac_prev) * torch.sqrt(alphas) / (1.0 - ac),
        loss_weight=lw, mean_type=mean_type, var_type=var_type)


def _ex(tab: Tensor, t: Tensor, ndim: int) -> Tensor:
    return tab[t].reshape([-1] + [1] * (ndim - 1))


def q_sample(s: Schedule, x0: Tensor, t: Tensor, noise: Tensor) -> Tensor:
    return _ex(s.sqrt_ac, t, x0.dim()) * x0 + _ex(s.sqrt_1mac, t, x0.dim()) * noise


def v_target(s: Schedule, x0: Tensor, t: Tensor, noise: Tensor) -> Tensor:
    return _ex(s.sqrt_ac, t, x0.dim()) * noise - _ex(s.sqrt_1mac, t, x0.dim()) * x0


def x0_from_output(s: Schedule, x_t: Tensor, t: Tensor, out: Tensor) -> Tensor:
    """model_predictions (:242-264) without the dead pred_noise leg."""
    if s.mean_type == "v":
        return _ex(s.sqrt_ac, t, x_t.dim()) * x_t - _ex(s.sqrt_1mac, t, x_t.dim()) * out
    if s.mean_type == "eps":
        return _ex(s.sqrt_recip_ac, t, x_t.dim()) * x_t - _ex(s.sqrt_recipm1_ac, t, x_t.dim()) * out
    if s.mean_type == "x0":
        return out
    raise NotImplementedError(s.mean_type)


def eps_from_x0(s: Schedule, x_t: Tensor, t: Tensor, x0: Tensor) -> Tensor:
    return (_ex(s.sqrt_recip_ac, t, x_t.dim()) * x_t - x0) / _ex(s.sqrt_recipm1_ac, t, x_t.dim())


def step_logvar(s: Schedule) -> Tensor:
    if s.var_type == "fixedsmall":
        return s.post_logvar_clipped
    if s.var_type == "fixedlarge":
        return torch.log(torch.cat([s.post_var[1:2], s.betas[1:]]))
    raise NotImplementedError(s.var_type)


def p_sample_step(s: Schedule, denoise: DenoiseFn, x_t: Tensor, t: Tensor, noise: Tensor,
                  clip_denoised: bool) -> Tuple[Tensor, Tensor]:
    """One reverse step (:305-352). Returns (x_{t-1}, clamped x0 estimate)."""
    out = denoise(x_t, t)
    x0 = x0_from_output(s, x_t, t, out)
    if clip_denoised:
        x0 = x0.clamp(-1.0, 1.0)
    mean = _ex(s.coef1, t, x_t.dim()) * x0 + _ex(s.coef2, t, x_t.dim()) * x_t
    logvar = _ex(step_logvar(s), t, x_t.dim())
    nonzero = (1 - (t == 0).float()).reshape([-1] + [1] * (x_t.dim() - 1))
    return mean + nonzero * torch.exp(0.5 * logvar) * noise, x0


def p_sample_loop(s: Schedule, denoise: DenoiseFn, shape, noise_fn, clip_denoised: bool = True,
                  freq: Optional[int] = None, num_steps: Optional[int] = None):
    """:355-398. noise_fn(shape) -> tensor; first call yields x_T. With `freq` returns the trajectory list."""
    x = noise_fn(tuple(shape))
    traj = [x]
    T = s.T if num_steps is None else num_steps
    for step in reversed(range(T)):
        t = torch.full((shape[0],), step, dtype=torch.int64)
        x, _ = p_sample_step(s, denoise, x, t, noise_fn(tuple(shape)), clip_denoised)
        if freq is not None and (step % freq == 0 or step == T - 1):
            traj.append(x)
    return traj if freq is not None else x


def p_sample_loop_complete(s: Schedule, denoise: DenoiseFn, shape, noise_fn, partial: Tensor,
                           clip_denoised: bool = True) -> Tensor:
    """:447-476: first P objects re-noised from `partial` every step, pasted clean at t == 0."""
    x = noise_fn(tuple(shape))
    P_ = partial.shape[1]
    for step in reversed(range(s.T)):
        t = torch.full((shape[0],), step, dtype=torch.int64)
        part_t = q_sample(s, partial, t, noise_fn(tuple(partial.shape)))
        x = torch.cat([part_t, x[:, P_:, :]], dim=1)
        x, _ = p_sample_step(s, denoise, x, t, noise_fn(tuple(shape)), clip_denoised)
        if step == 0:
            x = torch.cat([partial, x[:, P_:, :]], dim=1)
    return x


def p_sample_loop_arrange(s: Schedule, denoise: DenoiseFn, shape, noise_fn, boxes: Tensor,
                          trans_dim: int, size_dim: int, angle_dim: int, clip_denoised: bool = True) -> Tensor:
    """:478-506: diffuse (translation, angle) only; interleave with the given size / class / feats at the end."""
    small = (shape[0], shape[1], trans_dim + angle_dim)
    x = noise_fn(small)
    for step in reversed(range(s.T)):
        t = torch.full((shape[0],), step, dtype=torch.int64)
        x, _ = p_sample_step(s, denoise, x, t, noise_fn(small), clip_denoised)
    bbox = trans_dim + size_dim + angle_dim
    return torch.cat([x[..., :trans_dim], boxes[..., trans_dim:trans_dim + size_dim],
                      x[..., trans_dim:], boxes[..., bbox:]], dim=-1)


def ddim_times(T: int, S: int) -> List[Tuple[int, int]]:
    times = torch.linspace(-1, T - 1, steps=S + 1)
    times = list(reversed(times.int().tolist()))
    return list(zip(times[:-1], times[1:]))


def ddim_sample_loop(s: Schedule, denoise: DenoiseFn, shape, noise_fn, steps: int = 50, eta: float = 0.0) -> Tensor:
    """Working DDIM per the formula at :401-444 (x0 clamped, eps re-derived from the clamped x0)."""
    x = noise_fn(tuple(shape))
    for time, time_next in ddim_times(s.T, steps):
        t = torch.full((shape[0],), time, dtype=torch.int64)
        out = denoise(x, t)
        x0 = x0_from_output(s, x, t, out).clamp(-1.0, 1.0)
        eps = eps_from_x0(s, x, t, x0)
        if time_next < 0:
            x = x0
            continue
        a, an = s.alphas_cumprod[time], s.alphas_cumprod[time_next]
        sigma = eta * ((1 - a / an) * (1 - an) / (1 - a)).sqrt()
        c = (1 - an - sigma ** 2).sqrt()
        x = x0 * an.sqrt() + c * eps + sigma * noise_fn(tuple(shape))
    return x


def iou3d_pairwise(boxes: Tensor, eps: float = 1e-6) -> Tensor:
    """loss.py:7-102, mode='iou', is_aligned=False, boxes [B, N, 6] = (min xyz, max xyz) against itself."""
    lo, hi = boxes[..., :3], boxes[..., 3:]
    vol = (hi - lo).prod(dim=-1)
    ilo = torch.max(lo[:, :, None, :], lo[:, None, :, :])
    ihi = torch.min(hi[:, :, None, :], hi[:, None, :, :])
    inter = (ihi - ilo).clamp(min=0).prod(dim=-1)
    union = torch.max(vol[:, :, None] + vol[:, None, :] - inter, torch.tensor([eps], dtype=vol.dtype, device=vol.device))
    return inter / union


@dataclass
class LossSpec:
    translation_dim: int = 3
    size_dim: int = 3
    angle_dim: int = 2
    class_dim: int = 22
    objectness_dim: int = 0
    objfeat_dim: int = 32
    loss_separate: bool = True
    loss_iou: bool = False
    bounds_translations: Optional[List[float]] = None    # 6 numbers: min xyz, max xyz
    bounds_sizes: Optional[List[float]] = None
    room_arrange_condition: bool = False


def p_losses(s: Schedule, ls: LossSpec, denoise: DenoiseFn, x0: Tensor, t: Tensor, noise: Tensor,
             x_t: Optional[Tensor] = None):
    """:520-652, loss_type 'mse'. Returns (losses [B], dict of scalar means).  The schedule tables may live on the
    device of x0; x_t, when given, replaces q_sample(x0, t, noise) (the noisy input as a caller computed it)."""
    if x_t is None:
        x_t = q_sample(s, x0, t, noise)
    target = {"eps": noise, "x0": x0, "v": v_target(s, x0, t, noise)}[s.mean_type]
    out = denoise(x_t, t)
    sq = (target - out) ** 2

    def m(a, b):
        return sq[:, :, a:b].mean(dim=(1, 2))

    td, sd_, ad = ls.translation_dim, ls.size_dim, ls.angle_dim
    if ls.room_arrange_condition:
        l_tr, l_an = m(0, td), m(td, td + ad)
        losses = l_tr + l_an if ls.loss_separate else sq.mean(dim=(1, 2))
        return losses * s.loss_weight[t], {"loss.trans": l_tr.mean(), "loss.angle": l_an.mean()}
    bb = td + sd_ + ad
    cd = ls.class_dim
    l_tr, l_sz, l_an, l_bb, l_cl = m(0, td), m(td, td + sd_), m(td + sd_, bb), m(0, bb), m(bb, bb + cd)
    if ls.objectness_dim == 0:
        l_ob = m(bb + cd - 1, bb + cd)
    else:
        l_ob = m(bb + cd, bb + cd + ls.objectness_dim)
    l_of = m(bb + cd + ls.objectness_dim, sq.shape[-1]) if ls.objfeat_dim > 0 else x0.new_zeros(x0.shape[0])
    if ls.loss_separate:
        losses = l_bb + l_cl
        if ls.objectness_dim > 0:
            losses = losses + l_ob
        if ls.objfeat_dim > 0:
            losses = losses + l_of
    else:
        losses = sq.mean(dim=(1, 2))
    losses = losses * s.loss_weight[t]
    B = x0.shape[0]
    if ls.loss_iou:
        xr = x0_from_output(s, x_t, t, out).clamp(-1.0, 1.0)
        if ls.objectness_dim > 0:
            valid = (xr[:, :, bb + cd] >= 0).float()
        else:
            valid = (xr[:, :, bb + cd - 1] <= 0).float()
        bt = lambda v: torch.tensor(v, device=x0.device)
        tmin, tmax = bt(ls.bounds_translations[:3]), bt(ls.bounds_translations[3:])
        smin, smax = bt(ls.bounds_sizes[:3]), bt(ls.bounds_sizes[3:])
        tr = (xr[:, :, :td] + 1) / 2 * (tmax - tmin) + tmin
        sz = (xr[:, :, td:td + sd_] + 1) / 2 * (smax - smin) + smin
        iou = iou3d_pairwise(torch.cat([tr - sz, tr + sz], dim=-1))
        mask = valid[:, :, None] * valid[:, None, :]
        iou_valid = iou * mask
        denom = mask.sum(dim=(1, 2)) + 1e-6
        iou_avg = iou_valid.sum(dim=(1, 2)) / denom
        w = s.alphas_cumprod[t].reshape(B, 1, 1)
        l_iou = (w * 0.1 * iou_valid).sum(dim=(1, 2)) / denom
        losses = losses + l_iou
    else:
        l_iou = x0.new_zeros(B)
        iou_avg = x0.new_zeros(B)
    return losses, {
        "loss.bbox": l_bb.mean(), "loss.trans": l_tr.mean(), "loss.size": l_sz.mean(),
        "loss.angle": l_an.mean(), "loss.class": l_cl.mean(), "loss.object": l_ob.mean(),
        "loss.objfeat": l_of.mean(), "loss.liou": l_iou.mean(), "loss.bbox_iou": iou_avg.mean()}
