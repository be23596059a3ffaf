"""GPU: whole-network FID Inception features against the fp64 oracle (oracle.inception_ref) in fp32 and bf16, batch
independence, the fp64 feature statistics and KID terms against numpy, and compute_fid / compute_kid and the script
end to end against the oracle pipeline (clean resize, fp64 Inception, np.cov, sqrtm)."""
import importlib.util
import io
import os
import contextlib

import numpy as np
import pytest
import torch

from diffuscene_b200 import fid as F
from oracle import fid_ref as R
from oracle import inception_ref as IR
from tests.cases_fid import render_like, write_folder

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# relative L2 per image against fp64, 4x or more above the worst measured on one H100 80GB HBM3 (fp32 6.4e-7, bf16
# 5.95e-3 over B = 1, 7 and 64); the test prints each value
FEAT_TOL = {"fp32": 3e-6, "bf16": 2.5e-2}


@pytest.fixture(scope="module")
def sd():
    return IR.random_state_dict(seed=5)


@pytest.fixture(scope="module")
def images():
    return torch.from_numpy(np.stack([F.clean_resize(render_like(100 + i)) for i in range(64)]))


def oracle_feats(sd, imgs):
    sd64 = {k: v.double().cuda() for k, v in sd.items()}
    with torch.no_grad():
        return torch.cat([IR.inception_features(sd64, IR.detector_input(imgs[i:i + 16].double().cuda()))
                          for i in range(0, len(imgs), 16)])


def test_weight_inventory(sd):
    names = F.expected_weights()
    assert [n for n, _ in names] == list(sd.keys())
    assert [k for _, k in names] == [v.numel() for v in sd.values()]
    assert len(names) == 470 and sum(k for _, k in names) == 21_820_000


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_features_against_fp64(sd, images, prec):
    want = oracle_feats(sd, images)
    worst = 0.0
    for B, cap in ((1, None), (7, 5), (64, None)):
        m = F.InceptionFeatures(sd, precision=prec, capacity=cap)
        got = m(images[:B]).double()
        rel = ((got - want[:B]).norm(dim=1) / want[:B].norm(dim=1)).max().item()
        worst = max(worst, rel)
        print("%s B=%d capacity=%s: max relative L2 %.3g" % (prec, B, m.capacity, rel))
        m.close()
    assert worst <= FEAT_TOL[prec]


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_batch_independence(sd, images, prec):
    m = F.InceptionFeatures(sd, precision=prec, capacity=64)
    alone = m(images[3:4])
    b37 = m(images[:37])
    b64 = m(images)
    assert torch.equal(alone[0], b37[3]) and torch.equal(alone[0], b64[3])
    m2 = F.InceptionFeatures(sd, precision=prec, capacity=16)
    assert torch.equal(m2(images)[3], alone[0])


@pytest.mark.parametrize("n", [2, 3, 1000, 2049, 5000])
def test_feature_stats(n):
    rng = np.random.default_rng(n)
    f = (np.abs(rng.standard_normal((n, 2048))) * rng.random(2048) + 0.3).astype(np.float32)
    mu, sigma = F.feature_stats(f)
    f64 = f.astype(np.float64)
    mw, sw = np.mean(f64, 0), np.cov(f64, rowvar=False)
    assert np.linalg.norm(mu - mw) <= 1e-12 * np.linalg.norm(mw)
    assert np.linalg.norm(sigma - sw) <= 1e-12 * np.linalg.norm(sw)
    assert np.array_equal(sigma, sigma.T)


def _feats(n, seed):
    rng = np.random.default_rng(seed)
    return (np.abs(rng.standard_normal((n, 2048))) * 0.4).astype(np.float32)


@pytest.mark.parametrize("m,n_real,n_fake", [(2, 5, 5), (17, 40, 23), (1000, 1500, 1200)])
def test_kid_terms(m, n_real, n_fake):
    real, fake = _feats(n_real, 1), _feats(n_fake, 2)
    np.random.seed(m)
    ix, iy = F.kid_subsets(n_real, n_fake, num_subsets=4, max_subset_size=m)
    got = F.kid_terms(real, fake, ix, iy)
    want = R.kid_terms_f64(real, fake, ix, iy)
    d = 2048.0
    for s in range(4):
        x, y = fake[ix[s]].astype(np.float64), real[iy[s]].astype(np.float64)
        a = (x @ x.T / d + 1) ** 3 + (y @ y.T / d + 1) ** 3
        b = (x @ y.T / d + 1) ** 3
        scale = abs(a.sum() - np.trace(a)) / (m - 1) + 2 * abs(b.sum()) / m
        assert abs(got[s] - want[s]) <= 1e-12 * scale
        # float32 reference: each of its m x m sums carries a relative rounding of at most ~m^2 * 2^-24 (pairwise
        # summation keeps it far smaller); the bound uses 8 m 2^-24 of the summed magnitudes
        f32 = R.kid_terms_f32(real, fake, ix[s:s + 1], iy[s:s + 1])[0]
        assert abs(f32 - got[s]) <= 8 * m * 2.0 ** -24 * scale
    one_by_one = np.concatenate([F.kid_terms(real, fake, ix[s:s + 1], iy[s:s + 1]) for s in range(4)])
    assert np.array_equal(one_by_one, got)


def test_compute_fid_kid_end_to_end(sd, tmp_path):
    real = write_folder(tmp_path / "real", range(12), mode="RGBA")
    fake = write_folder(tmp_path / "fake", range(50, 60))
    model = F.InceptionFeatures(sd, precision="fp32")
    fid = F.compute_fid(str(real), str(fake), model=model, num_workers=4)
    np.random.seed(3)
    kid = F.compute_kid(str(real), str(fake), model=model, num_workers=4)

    def ofeats(folder):
        files = sorted(str(p) for p in folder.glob("*.png"))
        imgs = torch.from_numpy(np.stack([R.clean_resize_ref(p) for p in files]))
        return oracle_feats(sd, imgs).cpu().numpy()
    fr, ff = ofeats(real), ofeats(fake)
    want = R.frechet_distance_sqrtm(fr.mean(0), np.cov(fr, rowvar=False), ff.mean(0), np.cov(ff, rowvar=False))
    assert abs(fid - want) <= 1e-4 * abs(want), (fid, want)
    np.random.seed(3)
    ix, iy = F.kid_subsets(len(fr), len(ff), 100, 1000)
    kw = R.kid_terms_f32(fr.astype(np.float32), ff.astype(np.float32), ix, iy).sum() / 100 / ix.shape[1]
    assert abs(kid - kw) <= 1e-3 * abs(kw), (kid, kw)
    fid16 = F.compute_fid(str(real), str(fake), model=F.InceptionFeatures(sd, precision="bf16"), num_workers=4)
    print("FID fp32 %.6g, bf16 %.6g (difference %.3g); KID %.6g" % (fid, fid16, fid16 - fid, kid))


def test_script_prints_api_values(sd, tmp_path):
    base = tmp_path / "scenes"
    rows = []
    for i in range(6):
        d = base / ("Bedroom_s%d" % i)
        d.mkdir(parents=True)
        render_like(200 + i, mode="RGBA").save(str(d / "rendered_scene_256.png"))
        rows.append("s%d,%s\n" % (i, ("train", "val", "test")[i % 3]))
    csv = tmp_path / "splits.csv"
    csv.write_text("".join(rows))
    fake = write_folder(tmp_path / "fake", range(300, 305))
    wfile = str(tmp_path / "w.pth")
    torch.save(sd, wfile)
    spec = importlib.util.spec_from_file_location("cfs", os.path.join(ROOT, "scripts", "compute_fid_scores.py"))
    S = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(S)
    buf = io.StringIO()
    np.random.seed(11)
    with contextlib.redirect_stdout(buf):
        S.main([str(base), str(fake), str(csv), "--inception_weights", wfile, "--num_workers", "2"])
    lines = dict(l.split(":", 1) for l in buf.getvalue().splitlines() if "score:" in l)
    model = F.InceptionFeatures(sd)
    real_files = [str(base / ("Bedroom_s%d" % i) / "rendered_scene_256.png") for i in (0, 1, 3, 4)]
    fr = F.folder_features(real_files, model)
    ff = F.folder_features(S.fake_renders(str(fake)), model)
    np.random.seed(11)
    assert float(lines["fid score"]) == F.fid_from_features(fr, ff)
    assert float(lines["kid score"]) == F.kernel_distance(fr, ff)
    assert buf.getvalue().count("number of synthesized images :") == 2
