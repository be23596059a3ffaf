"""GPU: improved precision and recall (ds_vgg_*, ds_manifold_*, diffuscene_b200.ipr) against the fp64 oracles
(oracle/vgg16_ref.py, oracle/ipr_ref.py) and the reference's own functions (tests/golden/ipr_*.npz)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from diffuscene_b200 import capi
from diffuscene_b200 import ipr as I
from oracle import ipr_ref as R
from oracle import vgg16_ref as V
from tests.cases_ipr import clustered, he_state_dict, normalise, render_like

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# relative L2 error of a feature vector against fp64, measured on one H100 over the He-scaled cases below: at most
# 0.0072 in bf16 mode and 3.1e-6 in fp32 mode
BF16_REL_L2 = 0.03
FP32_REL_L2 = 2e-5

_SD = {}
_NETS = {}


def sd():
    if "sd" not in _SD:
        _SD["sd"] = he_state_dict(seed=1)
    return _SD["sd"]


def net(precision, capacity=None):
    key = (precision, capacity)
    if key not in _NETS:
        _NETS[key] = I.VGG16Features(sd(), precision=precision, capacity=capacity)
    return _NETS[key]


def rel_l2(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return np.linalg.norm(got - want, axis=1) / np.linalg.norm(want, axis=1)


def oracle_features(x):
    with torch.no_grad():
        return V.features(sd(), V.resize_nearest(x)).numpy()


# ---- features ---------------------------------------------------------------------------------------------------

def test_weight_inventory_matches_torchvision_order():
    names = [n for n, _ in I.expected_weights()]
    assert names == [n for n in sd() if not n.startswith("classifier.6")]
    assert [numel for _, numel in I.expected_weights()] == [sd()[n].numel() for n in names]


@pytest.mark.parametrize("precision,bound", [("fp32", FP32_REL_L2), ("bf16", BF16_REL_L2)])
@pytest.mark.parametrize("size,n", [(224, 5), (256, 3)])
def test_features_match_fp64(precision, bound, size, n):
    x = normalise(render_like(n, size, seed=size + n))
    got = net(precision)(x).cpu().numpy()
    err = rel_l2(got, oracle_features(x))
    print("%s %dx%d: max relative L2 %.3g" % (precision, size, size, err.max()))
    assert err.max() < bound, err


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_batch_split_gives_identical_features(precision):
    """Passes of `capacity` images, a ragged last pass and single images all give the same bits."""
    x = normalise(render_like(11, 224, seed=7))
    small = net(precision, capacity=4)
    whole = small(x).cpu()
    assert torch.equal(whole[:3], small(x[:3]).cpu())
    assert torch.equal(whole[9:10], small(x[9:10]).cpu())
    assert torch.equal(whole, net(precision)(x).cpu())


def test_golden_features():
    path = os.path.join(GOLDEN, "ipr_features.npz")
    g = np.load(path)
    x = normalise(g["images_u8"])
    for precision, bound in (("fp32", FP32_REL_L2), ("bf16", BF16_REL_L2)):
        err = rel_l2(net(precision)(x).cpu().numpy(), g["features"])
        print("%s vs torchvision: max relative L2 %.3g" % (precision, err.max()))
        assert err.max() < bound


# ---- manifold metrics -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,m,d", [(1, 1, 1), (70, 33, 5), (300, 129, 4096)])
def test_distances(n, m, d):
    x, y = clustered(n, d, seed=1, dtype=np.float64), clustered(m, d, seed=2, dtype=np.float64)
    want, _ = R.pairwise_distances(x, y)
    got = I.compute_pairwise_distances(x, y)
    assert got.shape == (n, m)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-9)


@pytest.mark.parametrize("k", [1, 3, 16])
@pytest.mark.parametrize("n,d", [(17, 3), (200, 37), (1000, 4096)])
def test_radii(k, n, d):
    if n <= k:
        pytest.skip("needs n > k")
    x = clustered(n, d, seed=n + k).astype(np.float64)
    np.testing.assert_allclose(I.manifold_radii(x, k), R.radii(x, k), rtol=1e-12, atol=0)


@pytest.mark.parametrize("k", [1, 2, 3])
def test_radii_with_duplicate_features(k):
    """Integer-valued features: every dot product is exact, duplicates are at distance exactly 0."""
    rng = np.random.default_rng(3)
    base = rng.integers(-4, 5, (40, 19)).astype(np.float64)
    x = np.concatenate([base, base[:25], base[:10]])
    rng.shuffle(x)
    assert np.array_equal(I.manifold_radii(x, k), R.radii(x, k))


def test_precision_recall_flags_identical_to_oracle():
    real = clustered(700, 4096, seed=4, centre_seed=0)
    fake = clustered(500, 4096, clusters=10, seed=5, spread=0.3, centre_seed=0)
    r_real, r_fake = I.manifold_radii(real, 3), I.manifold_radii(fake, 3)
    p, r, real_ism = I.manifold_cover(I.Manifold(real, r_real), fake, r_fake, want_realism=True)
    assert np.array_equal(p, R.cover(real, r_real, fake))
    assert np.array_equal(r, R.cover(fake, r_fake, real))
    np.testing.assert_allclose(real_ism, R.realism(real, r_real, fake), rtol=1e-6)
    assert 0 < p.mean() < 1 and 0 < r.mean() < 1


def test_precision_recall_against_reference_goldens():
    """The reference's own compute_pairwise_distances / distances2radii / compute_metric / realism.  Its subject
    norms |y|^2 are summed in fp32, so a subject whose margin |d - r| is within the error that implies may differ."""
    g = np.load(os.path.join(GOLDEN, "ipr_metrics.npz"))
    real, fake, k = g["real"], g["fake"], int(g["k"])
    r_real, r_fake = I.manifold_radii(real, k), I.manifold_radii(fake, k)
    np.testing.assert_allclose(r_real, g["radii_real"], rtol=1e-12)
    np.testing.assert_allclose(r_fake, g["radii_fake"], rtol=1e-12)
    p, r, real_ism = I.manifold_cover(I.Manifold(real, r_real), fake, r_fake, want_realism=True)
    for flags, want, ref, subj, radii in ((p, g["precision_flags"], real, fake, r_real),
                                          (r, g["recall_flags"], fake, real, r_fake)):
        d, _ = R.pairwise_distances(ref, subj)
        yy = (subj.astype(np.float64) ** 2).sum(1)
        # |fl32(sum y^2) - sum y^2| <= D u32 sum y^2; d changes by at most that / (2 d)
        tol = subj.shape[1] * 2.0 ** -24 * yy[None, :] / np.maximum(2 * d, 1e-300)
        margin = np.min(np.where(np.abs(d - radii[:, None]) <= tol, 0, 1), axis=0)
        differ = flags != want
        assert not (differ & (margin == 1)).any()
    assert p.mean() == pytest.approx(float(g["precision"]), abs=2.0 / len(fake))
    np.testing.assert_allclose(real_ism[:len(g["realism"])], g["realism"], rtol=1e-5)


def test_scale_50k():
    """N = 50 000 x D = 4096 in fp64: 1.6 GB of features, while the distance matrix would be 20 GB."""
    n, d, k = 50000, 4096, 3
    x = torch.randn(n, d, device="cuda", dtype=torch.float64, generator=torch.Generator("cuda").manual_seed(0))
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    lib = capi.load()
    radii = torch.empty(n, device="cuda", dtype=torch.float64)
    capi.check(lib.ds_manifold_radii(C.c_void_p(x.data_ptr()), n, d, k, C.c_void_p(radii.data_ptr()), None, None))
    free_during = torch.cuda.mem_get_info()[0]       # the call returned before the kernels end; scratch still held
    torch.cuda.synchronize()
    assert free0 - free_during < n * n * 8 // 100
    rows = torch.arange(0, n, 997, device="cuda")
    dd = torch.cdist(x[rows], x)
    want = torch.kthvalue(dd, k + 1, dim=1).values
    torch.testing.assert_close(radii[rows], want, rtol=1e-9, atol=0)


def test_invalid_input_is_an_error_not_a_fault():
    lib = capi.load()
    x = torch.zeros(8, 4, device="cuda", dtype=torch.float64)
    r = torch.zeros(8, device="cuda", dtype=torch.float64)
    px, pr = C.c_void_p(x.data_ptr()), C.c_void_p(r.data_ptr())
    assert lib.ds_manifold_radii(px, 8, 4, 17, pr, None, None) == -1          # k > DS_MANIFOLD_MAX_K
    assert lib.ds_manifold_radii(px, 8, 4, 0, pr, None, None) == -1
    assert lib.ds_manifold_radii(px, 3, 4, 3, pr, None, None) == -1           # N <= k
    assert lib.ds_manifold_radii(None, 8, 4, 3, pr, None, None) == -1
    assert lib.ds_manifold_radii(px, 8, 4, 3, None, None, None) == -1
    assert lib.ds_manifold_cover(px, None, 8, px, None, 8, 4, None, None, None, None, None) == -1
    f = torch.zeros(8, device="cuda", dtype=torch.uint8)
    assert lib.ds_manifold_cover(px, pr, 8, px, None, 8, 4, None, C.c_void_p(f.data_ptr()), None, None, None) == -1
    assert lib.ds_manifold_distances(px, 8, None, 8, 4, px, None, None) == -1
    cfg = capi.DsVggConfig()
    cfg.precision, cfg.capacity = capi.DS_PREC_FP32, 1
    h = C.c_void_p()
    capi.check(lib.ds_vgg_create(C.byref(cfg), C.byref(h)))
    try:
        w = torch.zeros(16, device="cuda")
        assert lib.ds_vgg_set_weights(h, C.c_void_p(w.data_ptr()), 16, None) == -1      # wrong weight count
        assert lib.ds_vgg_set_weights(h, None, 16, None) == -1
        out = torch.zeros(1, 4096, device="cuda")
        img = torch.zeros(1, 3, 224, 224, device="cuda")
        assert lib.ds_vgg_features(h, C.c_void_p(img.data_ptr()), 1, 224, 224, C.c_void_p(out.data_ptr()), None) == -4
        assert lib.ds_vgg_features(h, None, 1, 224, 224, C.c_void_p(out.data_ptr()), None) == -1
    finally:
        lib.ds_vgg_destroy(h)
    cfg.capacity = 0
    assert lib.ds_vgg_create(C.byref(cfg), C.byref(h)) == -1
    torch.cuda.synchronize()


def test_script_end_to_end(tmp_path, capsys):
    """The command line on PNG folders with an explicit weight file, and its --fname_precalc manifold."""
    import importlib.util
    from PIL import Image
    for name, seed in (("real", 30), ("fake", 31)):
        (tmp_path / name).mkdir()
        for i, im in enumerate(render_like(7, 256, seed=seed)):
            Image.fromarray(im).save(str(tmp_path / name / ("%02d.png" % i)))
    w = str(tmp_path / "vgg16.pth")
    torch.save(sd(), w)
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts",
                        "improved_precision_recall.py")
    spec = importlib.util.spec_from_file_location("ipr_script", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    args = [str(tmp_path / "real"), str(tmp_path / "fake"), "--vgg16_weights", w, "--num_samples", "6", "--k", "2",
            "--precision", "fp32"]
    mod.main(args)
    out = capsys.readouterr().out
    vals = {l.split(":")[0]: float(l.split(":")[1]) for l in out.splitlines() if l.split(":")[0] in
            ("precision", "recall", "fscore")}
    assert set(vals) == {"precision", "recall", "fscore"}
    real = [str(tmp_path / "real" / f) for f in sorted(os.listdir(tmp_path / "real"))]
    fake = [str(tmp_path / "fake" / f) for f in sorted(os.listdir(tmp_path / "fake"))]
    feats = lambda files: oracle_features(torch.from_numpy(np.stack([I.load_image(f) for f in I.subsample(files, 6)])))
    p, r = R.precision_recall(feats(real), feats(fake), 2)
    assert (vals["precision"], vals["recall"]) == (p, r)
    mod.main(args + ["--fname_precalc", str(tmp_path / "m.npz")])
    with np.load(str(tmp_path / "m.npz")) as z:
        assert z["feature"].shape == (6, 4096) and z["radii"].shape == (6,)
