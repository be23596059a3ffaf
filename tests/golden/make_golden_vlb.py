"""Variational-bound golden vectors: the UNMODIFIED reference DiffusionPoint.all_kl / prior_kl
(scene_synthesis/networks/diffusion_ddpm.py:679-745) on CPU / fp32, for every case of tests/cases_vlb.py.

Run in the authoring container only (needs the reference checkout, like make_golden.py):
    python tests/golden/make_golden_vlb.py
Writes tests/golden/vlb_*.npz:
  noise                  [T, B, N, d] the q_sample draws of calc_bpd_loop in loop order (recorded, see below)
  prior                  [B] _prior_bpd
  vb_clip{0,1}           [B, T] _vb_terms_bpd per timestep, clip_denoised False / True
  mse_clip{0,1}          [B, T] the matching x0-prediction MSE
  <key>_clip{0,1}        the four scalars of all_kl: total_bpd_b, terms_bpd, prior_bpd_b, mse_bt
Randomness: calc_bpd_loop's q_sample calls torch.randn; the `Recorder` of make_golden_class.py replaces it by a seeded,
recorded stream while all_kl runs.  The per-timestep arrays are then the reference's own _vb_terms_bpd evaluated on
the recorded draws (all_kl returns means only), and their means are checked against all_kl's.
Weights and inputs: as make_golden.py (seeded by the case).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import build_reference      # noqa: E402  (also puts the reference on sys.path)
from make_golden_class import Recorder       # noqa: E402

from tests.cases import make_inputs          # noqa: E402
from tests.cases_vlb import VLB_CASES        # noqa: E402


def main():
    torch.manual_seed(0)
    torch.set_grad_enabled(False)
    for name, case in VLB_CASES.items():
        dp, spec = build_reference(case)
        gd = dp.diffusion
        inp = make_inputs(case, spec)
        x0, ctx, cross = inp["x0"], inp["context"], inp["context_cross"]
        B, T = x0.shape[0], case["diffusion_kwargs"]["time_num"]
        out = {"prior": dp.prior_kl(x0).numpy()}
        draws = None
        for clip in (False, True):
            with Recorder(case["seed"] + 500) as r:
                res = dp.all_kl(x0, ctx, cross, clip_denoised=clip)
            assert len(r.randn_draws) == T
            noise = torch.stack(r.randn_draws)
            if draws is None:
                draws = noise
            assert torch.equal(draws, noise)
            vb, mse = torch.zeros(B, T), torch.zeros(B, T)
            for k, t in enumerate(reversed(range(T))):
                tb = torch.full((B,), t, dtype=torch.int64)
                x_t = gd.q_sample(x0, tb, noise=noise[k])
                v, xh = gd._vb_terms_bpd(dp._denoise, x0, x_t, tb, ctx, cross, clip_denoised=clip,
                                         return_pred_xstart=True)
                vb[:, t] = v
                mse[:, t] = ((xh - x0) ** 2).mean(dim=(1, 2))
            # the replay is the loop all_kl ran: its means agree
            np.testing.assert_allclose(float(vb.mean()), float(res["terms_bpd"]), rtol=1e-6)
            np.testing.assert_allclose(float(mse.mean()), float(res["mse_bt"]), rtol=1e-6)
            out["vb_clip%d" % clip] = vb.numpy()
            out["mse_clip%d" % clip] = mse.numpy()
            for k, v in res.items():
                out["%s_clip%d" % (k, clip)] = np.asarray(v.numpy())
        out["noise"] = draws.numpy()
        np.savez(os.path.join(HERE, name + ".npz"), **out)
        print(name, {k: v.shape for k, v in out.items()}, "total_bpd_b(clip)", float(out["total_bpd_b_clip1"]))


if __name__ == "__main__":
    main()
