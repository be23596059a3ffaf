"""CPU restatement of the reference's variational bound (test infrastructure, not product code).

normal_kl (diffusion_ddpm.py:96-101), _vb_terms_bpd (:511-518), _prior_bpd (:679-688) and calc_bpd_loop (:690-717)
as plain functions over the oracle's `Schedule`, returning the per-(scene, t) arrays as well as the reference's four
means.  Pinned against the unmodified reference by tests/golden/make_golden_vlb.py.
"""
from __future__ import annotations

from typing import Callable, Dict

import numpy as np
import torch

from oracle import diffusion_ref as D

Tensor = torch.Tensor


def normal_kl(mean1: Tensor, logvar1: Tensor, mean2: Tensor, logvar2: Tensor) -> Tensor:
    return 0.5 * (-1.0 + logvar2 - logvar1 + torch.exp(logvar1 - logvar2) + (mean1 - mean2) ** 2 * torch.exp(-logvar2))


def log_one_minus_ac(s: D.Schedule) -> Tensor:
    """q_mean_variance's log-variance table (:179)."""
    return torch.log(1.0 - s.alphas_cumprod)


def vb_terms_bpd(s: D.Schedule, denoise: D.DenoiseFn, x0: Tensor, x_t: Tensor, t: Tensor, clip_denoised: bool):
    """(KL [B] in bits per dim, x0 estimate) at per-scene t (:511-518 with p_mean_variance :305-335)."""
    n = x0.dim()
    xh = D.x0_from_output(s, x_t, t, denoise(x_t, t))
    if clip_denoised:
        xh = xh.clamp(-1.0, 1.0)
    true_mean = D._ex(s.coef1, t, n) * x0 + D._ex(s.coef2, t, n) * x_t
    model_mean = D._ex(s.coef1, t, n) * xh + D._ex(s.coef2, t, n) * x_t
    model_logvar = D._ex(D.step_logvar(s), t, n) * torch.ones_like(x_t)
    kl = normal_kl(true_mean, D._ex(s.post_logvar_clipped, t, n), model_mean, model_logvar)
    return kl.mean(dim=list(range(1, n))) / np.log(2.0), xh


def prior_bpd(s: D.Schedule, x0: Tensor) -> Tensor:
    t = torch.full((x0.shape[0],), s.T - 1, dtype=torch.int64)
    mean = D._ex(s.sqrt_ac, t, x0.dim()) * x0
    logvar = D._ex(log_one_minus_ac(s), t, x0.dim())
    kl = normal_kl(mean, logvar, torch.tensor([0.0]), torch.tensor([0.0]))
    return kl.mean(dim=list(range(1, x0.dim()))) / np.log(2.0)


def calc_bpd_loop(s: D.Schedule, denoise: D.DenoiseFn, x0: Tensor, noise_fn: Callable, clip_denoised: bool = True
                  ) -> Dict[str, Tensor]:
    """noise_fn(shape) gives the q_sample draw of each iteration, t = T-1 .. 0.  Returns vb [B, T], mse [B, T],
    prior [B] and the four means of all_kl (:717, :737-745)."""
    B, T = x0.shape[0], s.T
    vb, mse = torch.zeros(B, T), torch.zeros(B, T)
    for t in reversed(range(T)):
        tb = torch.full((B,), t, dtype=torch.int64)
        x_t = D.q_sample(s, x0, tb, noise_fn(tuple(x0.shape)))
        v, xh = vb_terms_bpd(s, denoise, x0, x_t, tb, clip_denoised)
        vb[:, t] = v
        mse[:, t] = ((xh - x0) ** 2).mean(dim=list(range(1, x0.dim())))
    prior = prior_bpd(s, x0)
    return {"vb": vb, "mse": mse, "prior": prior, "total_bpd_b": (vb.sum(dim=1) + prior).mean(),
            "terms_bpd": vb.mean(), "prior_bpd_b": prior.mean(), "mse_bt": mse.mean()}
