"""CPU: the variational-bound restatement (tests/vlb_oracle.py) against the golden vectors of the unmodified reference
(tests/golden/make_golden_vlb.py), the schedule tables the CUDA loop reads, and the host side of the drop-in
`diffusion.all_kl` / `prior_kl` surface."""
import copy
import os

import numpy as np
import pytest
import torch
import yaml

from diffuscene_b200.schedule import get_betas, make_tables
from diffuscene_b200.weights import NetSpec, seeded_state_dict, unet1d_param_specs
from oracle import diffusion_ref as D
from oracle.unet1d_ref import unet1d_forward
from tests import vlb_oracle as V
from tests.cases import make_inputs
from tests.cases_vlb import VLB_CASES

TOL = dict(rtol=2e-4, atol=2e-5)      # test_oracle_vs_golden.py
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _replay(draws):
    it = iter(draws)
    return lambda shape: next(it)


@pytest.mark.parametrize("name", list(VLB_CASES))
def test_oracle_matches_reference_goldens(name, golden_dir):
    torch.set_grad_enabled(False)
    case = VLB_CASES[name]
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    spec = NetSpec.from_net_kwargs(case["net_kwargs"])
    sd = seeded_state_dict(unet1d_param_specs(spec), seed=case["seed"])
    inp = make_inputs(case, spec)
    dk = case["diffusion_kwargs"]
    s = D.make_schedule(D.make_betas(dk["schedule_type"], dk["beta_start"], dk["beta_end"], dk["time_num"]),
                        dk["model_mean_type"], dk["model_var_type"])
    den = lambda x, t: unet1d_forward(sd, spec, x, t, inp["context"], inp["context_cross"])
    noise = torch.from_numpy(g["noise"])
    np.testing.assert_allclose(V.prior_bpd(s, inp["x0"]).numpy(), g["prior"], **TOL)
    for clip in (0, 1):
        r = V.calc_bpd_loop(s, den, inp["x0"], _replay(noise), clip_denoised=bool(clip))
        np.testing.assert_allclose(r["vb"].numpy(), g["vb_clip%d" % clip], **TOL)
        np.testing.assert_allclose(r["mse"].numpy(), g["mse_clip%d" % clip], **TOL)
        for k in ("total_bpd_b", "terms_bpd", "prior_bpd_b", "mse_bt"):
            np.testing.assert_allclose(float(r[k]), float(g["%s_clip%d" % (k, clip)]), **TOL)


@pytest.mark.parametrize("mean,var", [("v", "fixedsmall"), ("eps", "fixedlarge"), ("x0", "fixedsmall"),
                                      ("x0", "fixedlarge")])
def test_vlb_schedule_tables_are_the_oracle_expressions(mean, var):
    for T in (1000, 6):
        t = make_tables(get_betas("linear", 1e-4, 0.02, T), mean, var)
        o = D.make_schedule(D.make_betas("linear", 1e-4, 0.02, T), mean, var)
        assert torch.equal(t["log_one_minus_alphas_cumprod"], V.log_one_minus_ac(o))
        assert torch.equal(t["model_log_variance"], D.step_logvar(o))
        assert torch.equal(t["posterior_log_variance_clipped"], o.post_logvar_clipped)
        assert t["log_one_minus_alphas_cumprod"].dtype == torch.float32
        # sigma keeps its meaning: exp(0.5 * model_log_variance) with the t = 0 entry forced to 0
        sig = torch.exp(0.5 * t["model_log_variance"])
        sig[0] = 0
        assert torch.equal(t["sigma"], sig)


def test_t0_term_is_finite_in_fp32():
    """The reference's t = 0 quirk: the posterior variance clipped to 1e-20 puts exp(-logvar2) ~ 1e20 on the squared
    mean error.  Its worst case over a whole scene, (2^2) * 1e20 * N * d, stays far below the fp32 range."""
    o = D.make_schedule(D.make_betas("linear", 1e-4, 0.02, 1000), "v", "fixedsmall")
    lv = o.post_logvar_clipped[0:1]
    e = torch.exp(-lv)
    assert 0.9e20 < float(e) < 1.1e20
    worst = torch.tensor([4.0]) * e * (21 * 105)
    assert torch.isfinite(worst).all() and float(worst) < 1e25
    kl = V.normal_kl(torch.tensor([1.0]), lv, torch.tensor([-1.0]), lv)
    assert torch.isfinite(kl).all() and 1e20 < float(kl) < 3e20


def _model():
    from scene_synthesis.networks import build_network
    cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "uncond", "diffusion_bedrooms_instancond_lat32_v.yaml")))
    cfg["network"]["diffusion_kwargs"]["loss_iou"] = False
    net, _, _ = build_network(30, 23, cfg, None, "cpu")
    return net


def test_diffusion_container_adds_no_state_and_owns_no_parent():
    net = _model()
    diff = net.diffusion
    assert callable(diff.all_kl) and callable(diff.prior_kl)
    assert diff._model() is net
    assert list(diff._modules) == ["model"]                # the owner is a weak reference, not a child
    assert not list(diff.buffers()) and all(n.startswith("model.") for n, _ in diff.named_parameters())
    keys = set(net.state_dict())
    assert all(k == "positional_embedding" or k.startswith("diffusion.model.") for k in keys)
    # a copy carries its own owner
    cp = copy.deepcopy(net)
    assert cp.diffusion._model() is cp and set(cp.state_dict()) == keys


def test_all_kl_has_no_cpu_path():
    net = _model()
    x0 = torch.zeros(1, 12, 62)
    with pytest.raises(RuntimeError, match="CUDA"):
        net.diffusion.all_kl(x0, torch.zeros(12, 128), None)
    with pytest.raises(RuntimeError, match="CUDA"):
        net.diffusion.prior_kl(x0)
