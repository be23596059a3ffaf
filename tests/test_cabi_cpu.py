"""CPU: the C-ABI shared library builds, loads, exports every symbol declared in include/diffuscene_b200.h,
and its host-side plan agrees with the Python parameter inventory.  No compute calls (no GPU here)."""
import ctypes as C
import math
import os
import re

import pytest
import torch

from diffuscene_b200 import capi
from diffuscene_b200.weights import NetSpec, count_params, unet1d_param_specs
from tests.cases import CASES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    lib = capi.load()
    hdr = open(os.path.join(ROOT, "include", "diffuscene_b200.h")).read()
    declared = re.findall(r"^DS_API [a-z0-9_ \*]+?(ds_[a-z0-9_]+)\(", hdr, flags=re.M)
    assert len(declared) >= 25
    for name in declared:
        assert hasattr(lib, name), name
    assert sorted(declared) == sorted(capi.EXPORTED)
    assert b"sm_90a" in lib.ds_version()


@pytest.mark.parametrize("name", list(CASES))
def test_plan_inventory_matches_python_inventory(name):
    case = CASES[name]
    spec = NetSpec.from_net_kwargs(case["net_kwargs"])
    cfg = capi.make_config(spec, case["N"], case["diffusion_kwargs"]["time_num"])
    got = dict(capi.plan_expected_weights(cfg))
    want = {n[len("diffusion.model."):]: int(math.prod(shp)) for (n, shp, _) in unet1d_param_specs(spec)}
    assert got == want
    txt = capi.plan_describe(cfg)
    assert "GEMM encoder" in txt or "GEMM init_conv" in txt
    assert txt.count(" GN ") == 2 * (3 * spec.n_stages * 2 + 3 + 1)    # two Blocks per ResnetBlock


def test_bedroom_param_count():
    spec = NetSpec.from_net_kwargs(CASES["bed62"]["net_kwargs"])
    assert count_params(unet1d_param_specs(spec)) == 77676094        # SURVEY.md A.1


def test_invalid_config_is_rejected():
    spec = NetSpec.from_net_kwargs(CASES["bed62"]["net_kwargs"])
    cfg = capi.make_config(spec, 12, 1000)
    cfg.dim = 500
    with pytest.raises(capi.DsError):
        capi.plan_describe(cfg)
    with pytest.raises(NotImplementedError):
        NetSpec.from_net_kwargs(dict(CASES["bed62"]["net_kwargs"], dim_mults=[1, 2, 4, 8]))


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    lib = capi.load()
    spec = NetSpec.from_net_kwargs(CASES["bed62"]["net_kwargs"])
    cfg = capi.make_config(spec, 12, 1000)
    h = C.c_void_p()
    rc = lib.ds_create(C.byref(cfg), C.byref(h))
    assert rc == -2 and not h.value                      # DS_ERR_NO_DEVICE
    assert b"no CPU fallback" in lib.ds_last_error()
    from diffuscene_b200.engine import DenoiserEngine
    with pytest.raises(RuntimeError):
        DenoiserEngine(spec, 12, 1000)

