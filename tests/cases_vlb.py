"""Cases of the variational-bound (all_kl / prior_kl) parity tests.

They reuse the networks of tests/cases.py with short schedules, so that the reference's loop of T denoiser forwards
stays cheap on the CPU.  Kept apart from CASES on purpose: every existing parametrised test iterates over CASES.
"""
from __future__ import annotations

from tests.cases import CASES


def _short(base: str, seed: int, T: int, **dk):
    c = dict(CASES[base])
    c["seed"] = seed
    c["diffusion_kwargs"] = dict(c["diffusion_kwargs"], time_num=T, loss_iou=False, **dk)
    c["base"] = base
    return c


VLB_CASES = {
    # shipped bedroom network, v-prediction, fixedsmall
    "vlb_bed62": _short("bed62", 41, 8),
    # d = 97, eps-prediction
    "vlb_bed97": _short("bed97", 42, 6),
    # living room (N = 21), x0-prediction, fixedlarge variance
    "vlb_liv65": _short("liv65", 43, 6),
    # text-conditioned network (cross-attention on a synthetic [B, L, 512] prefix)
    "vlb_text62": _short("text62", 44, 5),
    # re-arrangement network: 5 diffused channels, per-scene condition
    "vlb_arr5": _short("arr5", 45, 6),
}
