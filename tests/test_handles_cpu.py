"""CPU: the scaffold every model handle shares.  The null-handle checks of the weight inventory, the device check of
every create function, the Python inventory helper and the symbol table run without a GPU."""
import ctypes as C
import os
import re

import pytest
import torch

from diffuscene_b200 import capi
from diffuscene_b200.weights import NetSpec
from tests.cases import CASES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAMILIES = ("ds_room_enc", "ds_shape_ae", "ds_text_enc", "ds_vgg", "ds_inception")


def _configs():
    re_cfg = capi.DsRoomEncConfig()
    re_cfg.precision, re_cfg.input_channels, re_cfg.height, re_cfg.width = capi.DS_PREC_FP32, 1, 64, 64
    sae = capi.DsShapeAeConfig()
    sae.latent_dim, sae.num_points = 32, 2048
    te = capi.DsTextEncConfig()
    te.layers, te.hidden, te.heads, te.intermediate, te.vocab, te.max_positions, te.type_vocab = 1, 128, 2, 512, 30, 8, 2
    te.precision, te.capacity = capi.DS_PREC_FP32, 16
    vgg, inc = capi.DsVggConfig(), capi.DsInceptionConfig()
    vgg.capacity = inc.capacity = 1
    den = capi.make_config(NetSpec.from_net_kwargs(CASES["bed62"]["net_kwargs"]), 12, 1000)
    return {"ds_room_enc": re_cfg, "ds_shape_ae": sae, "ds_text_enc": te, "ds_vgg": vgg, "ds_inception": inc,
            "ds": den}


@pytest.mark.parametrize("prefix", FAMILIES)
def test_weight_inventory_refuses_a_null_handle(prefix):
    lib = capi.load()
    assert getattr(lib, prefix + "_expected_weight_count")(None) == -1      # DS_ERR_INVALID
    assert lib.ds_last_error() == b"null handle"
    name, numel = C.c_char_p(), C.c_int64()
    assert getattr(lib, prefix + "_expected_weight")(None, 0, C.byref(name), C.byref(numel)) == -1
    assert lib.ds_last_error() == b"null argument"


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
@pytest.mark.parametrize("prefix", FAMILIES + ("ds",))
def test_create_has_no_cpu_fallback(prefix):
    lib = capi.load()
    h = C.c_void_p()
    rc = getattr(lib, prefix + "_create")(C.byref(_configs()[prefix]), C.byref(h))
    assert rc == -2 and not h.value                      # DS_ERR_NO_DEVICE
    assert b"no CPU fallback" in lib.ds_last_error()


def test_expected_weights_checks_the_count():
    class Lib:
        def ds_x_expected_weight_count(self, h):
            return -1

        def ds_x_expected_weight(self, h, i, name, numel):
            raise AssertionError("no index is read after a failed count")

        def ds_last_error(self):
            return b"null handle"

    real = capi._lib
    capi._lib = Lib()      # check() reads the message through load()
    try:
        with pytest.raises(capi.DsError, match="null handle"):
            capi.expected_weights(capi._lib, "ds_x", None)
    finally:
        capi._lib = real


def test_exported_is_the_prototype_table():
    assert capi.EXPORTED == list(capi.sig)
    hdr = open(os.path.join(ROOT, "include", "diffuscene_b200.h")).read()
    declared = re.findall(r"^DS_API [a-z0-9_ \*]+?(ds_[a-z0-9_]+)\(", hdr, flags=re.M)
    assert sorted(declared) == sorted(capi.EXPORTED)
