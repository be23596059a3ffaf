"""Diffusion schedule tables (host side), built with the same torch expressions and precision path as
the reference `GaussianDiffusion.__init__` (scene_synthesis/networks/diffusion_ddpm.py:45-91, 168-203):
betas in float64, cumprod in float64 cast to float32, every derived table computed in float32.
The tables are handed to the CUDA engine unchanged (ds_set_schedule)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict

import numpy as np
import torch


def get_betas(schedule_type: str, b_start: float, b_end: float, time_num: int) -> np.ndarray:
    """Same schedule names as the reference (diffusion_ddpm.py:45-91).  The reference's `cosine`
    branch never returns a value (SURVEY.md A.6.2); it raises NotImplementedError here."""
    if schedule_type == "linear":
        return np.linspace(b_start, b_end, time_num)
    if schedule_type in ("warm0.1", "warm0.2", "warm0.5"):
        betas = b_end * np.ones(time_num, dtype=np.float64)
        warm = int(time_num * float(schedule_type[4:]))
        betas[:warm] = np.linspace(b_start, b_end, warm, dtype=np.float64)
        return betas
    raise NotImplementedError(schedule_type)


@dataclass
class DiffusionTables:
    T: int
    mean_type: str
    var_type: str
    tables: Dict[str, torch.Tensor]     # float32 CPU tensors of length T

    def __getitem__(self, k: str) -> torch.Tensor:
        return self.tables[k]


def make_tables(betas: np.ndarray, mean_type: str = "eps", var_type: str = "fixedsmall") -> DiffusionTables:
    assert isinstance(betas, np.ndarray)
    betas64 = betas.astype(np.float64)
    assert (betas64 > 0).all() and (betas64 <= 1).all()
    alphas64 = 1.0 - betas64
    ac = torch.from_numpy(np.cumprod(alphas64, axis=0)).float()
    ac_prev = torch.from_numpy(np.append(1.0, ac[:-1].numpy())).float()
    b = torch.from_numpy(betas64).float()
    a = torch.from_numpy(alphas64).float()
    post_var = b * (1.0 - ac_prev) / (1.0 - ac)
    post_logvar = torch.log(torch.max(post_var, 1e-20 * torch.ones_like(post_var)))
    if var_type == "fixedsmall":
        logvar = post_logvar
    elif var_type == "fixedlarge":
        logvar = torch.log(torch.cat([post_var[1:2], b[1:]]))
    else:
        raise NotImplementedError(var_type)
    sigma = torch.exp(0.5 * logvar)
    sigma[0] = 0.0          # nonzero_mask of p_sample (diffusion_ddpm.py:348)
    snr = ac / (1 - ac)
    if mean_type == "eps":
        lw = torch.ones_like(snr)
    elif mean_type == "x0":
        lw = snr
    elif mean_type == "v":
        lw = snr / (snr + 1)
    else:
        raise NotImplementedError(mean_type)
    t = {
        "betas": b, "alphas_cumprod": ac, "alphas_cumprod_prev": ac_prev,
        "sqrt_ac": torch.sqrt(ac), "sqrt_1mac": torch.sqrt(1.0 - ac),
        "sqrt_recip_ac": torch.sqrt(1.0 / ac), "sqrt_recipm1_ac": torch.sqrt(1.0 / ac - 1),
        "posterior_variance": post_var, "posterior_log_variance_clipped": post_logvar,
        "coef1": b * torch.sqrt(ac_prev) / (1.0 - ac), "coef2": (1.0 - ac_prev) * torch.sqrt(a) / (1.0 - ac),
        "sigma": sigma, "loss_weight": lw,
        # variational bound (ds_set_vlb_schedule): q_mean_variance's log-variance (:179) and p_mean_variance's model
        # log-variance (:314-323), whose t = 0 entry `sigma` does not keep
        "log_one_minus_alphas_cumprod": torch.log(1.0 - ac), "model_log_variance": logvar,
    }
    return DiffusionTables(T=len(betas64), mean_type=mean_type, var_type=var_type,
                           tables={k: v.float().contiguous() for k, v in t.items()})
