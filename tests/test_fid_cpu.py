"""CPU: the fp64 Inception oracle against torchvision, the weight inventory, clean-fid's resize, the eigen form of the
Frechet trace term against sqrtm, the KID draw order, the evaluation script's file lists, input checks and the
absence of a CPU fallback."""
import os
import sys

import numpy as np
import pytest
import torch

from diffuscene_b200 import capi
from diffuscene_b200 import fid as F
from diffuscene_b200.renders import real_renders
from oracle import fid_ref as R
from oracle import inception_ref as IR
from tests.cases_fid import conv_geometries, render_like

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_matches_torchvision_inception():
    from torchvision.models import inception_v3
    sd = IR.random_state_dict(seed=1, dtype=torch.float64)
    net = inception_v3(weights=None, aux_logits=False, init_weights=False, num_classes=1008).double().eval()
    missing, _ = net.load_state_dict(sd, strict=False)
    assert all(k.startswith("fc.") for k in missing)
    net.fc = torch.nn.Identity()
    net.dropout = torch.nn.Identity()
    x = torch.randn(1, 3, 299, 299, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    with torch.no_grad():
        want = net(x)
        got = IR.inception_features(sd, x, fid=False)
        fid = IR.inception_features(sd, x, fid=True)
    assert ((got - want).norm() / want.norm()).item() <= 1e-10
    assert ((fid - want).norm() / want.norm()).item() > 1e-6      # the FID blocks change the features


def test_weight_inventory_and_geometries():
    sd = IR.random_state_dict()
    assert len(sd) == 470
    assert sum(v.numel() for v in sd.values()) == 21_820_000
    assert sum(k.endswith("conv.weight") for k in sd) == 94
    seen, distinct = conv_geometries()
    assert len(seen) == 94 and len(distinct) == 43


def test_clean_resize_is_bit_exact(tmp_path):
    for mode in ("RGB", "RGBA"):
        p = str(tmp_path / ("x_%s.png" % mode))
        render_like(3, mode=mode).save(p)
        got = F.clean_resize(p)
        want = R.clean_resize_ref(p)
        assert got.dtype == np.float32 and got.shape == (3, 299, 299)
        assert np.array_equal(got, want)


@pytest.mark.parametrize("D", [256, 512])
@pytest.mark.parametrize("n", ["deficient", "full"])
def test_trace_term_matches_sqrtm(D, n):
    from scipy import linalg
    rng = np.random.default_rng(D)
    rows = D // 2 if n == "deficient" else 3 * D
    a = rng.standard_normal((rows, D))
    b = rng.standard_normal((rows, D)) * 1.3 + 0.2
    s1, s2 = np.cov(a, rowvar=False), np.cov(b, rowvar=False)
    want = np.trace(linalg.sqrtm(s1.dot(s2))).real
    got = F.trace_sqrt_product(s1, s2)
    assert abs(got - want) <= 1e-7 * abs(want)
    mu1, mu2 = a.mean(0), b.mean(0)
    assert abs(F.frechet_distance(mu1, s1, mu2, s2) - R.frechet_distance_sqrtm(mu1, s1, mu2, s2)) <= 1e-7 * abs(want)


def test_frechet_rejects_non_finite():
    s = np.eye(4)
    with pytest.raises(ValueError):
        F.frechet_distance(np.array([np.nan, 0, 0, 0]), s, np.zeros(4), s)
    with pytest.raises(ValueError):
        F.frechet_distance(np.zeros(3), s, np.zeros(4), s)


def test_kid_draw_order():
    np.random.seed(7)
    ix, iy = F.kid_subsets(50, 40, num_subsets=3, max_subset_size=30)
    np.random.seed(7)
    for s in range(3):
        assert np.array_equal(ix[s], np.random.choice(40, 30, replace=False))      # fake first
        assert np.array_equal(iy[s], np.random.choice(50, 30, replace=False))
    ix, _ = F.kid_subsets(5, 8, num_subsets=1)
    assert ix.shape == (1, 5)


def _scenes(tmp_path, name="rendered_scene_256.png"):
    base = tmp_path / "real"
    rows = [("a1", "train"), ("b2", "val"), ("c3", "test"), ("d4", "train")]
    for sid, _ in rows:
        d = base / ("Bedroom_%s" % sid)
        d.mkdir(parents=True)
        (d / name).write_bytes(b"")
    csv = tmp_path / "splits.csv"
    csv.write_text("".join("%s,%s\n" % r for r in rows))
    return str(base), str(csv)


def test_script_file_lists(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import compute_fid_scores as S
    base, csv = _scenes(tmp_path)
    got = real_renders(base, csv)
    assert [os.path.basename(os.path.dirname(p)) for p in got] == ["Bedroom_a1", "Bedroom_b2", "Bedroom_d4"]
    got = real_renders(base, csv, ("train", "val", "test"))
    assert len(got) == 4 and os.path.basename(got[0]) == "rendered_scene_256.png"
    fake = tmp_path / "fake"
    fake.mkdir()
    for n in ("b.png", "a.png", "c.jpg"):
        (fake / n).write_bytes(b"")
    assert S.fake_renders(str(fake)) == [os.path.join(str(fake), f) for f in os.listdir(str(fake)) if f.endswith(".png")]


def test_input_checks():
    with pytest.raises(ValueError):
        F.InceptionFeatures({}, precision="fp16")
    with pytest.raises(TypeError):
        F.InceptionFeatures(3)
    with pytest.raises(FileNotFoundError):
        F.find_weights("/nonexistent/pt_inception.pth")
    with pytest.raises(FileNotFoundError):
        F.folder_features("/nonexistent_dir", None)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the behaviour without a device")
def test_no_cpu_fallback():
    with pytest.raises(RuntimeError):
        F.InceptionFeatures(IR.random_state_dict())
    lib = capi.load()
    import ctypes as C
    cfg = capi.DsInceptionConfig()
    cfg.capacity = 1
    h = C.c_void_p()
    assert lib.ds_inception_create(C.byref(cfg), C.byref(h)) == -2        # DS_ERR_NO_DEVICE
    assert lib.ds_feature_stats(C.c_void_p(8), 4, 4, C.c_void_p(8), C.c_void_p(8), None) == -2
