"""CPU: the improved precision and recall oracles against the reference's own functions (tests/golden/ipr_*.npz),
the VGG16 weight inventory, the fc1 column permutation, the manifold file format, the file listing and subsampling,
and the weight lookup."""
import os
import random
import sys

import numpy as np
import pytest
import torch

from diffuscene_b200 import capi
from diffuscene_b200 import ipr as I
from oracle import ipr_ref as R
from oracle import vgg16_ref as V
from tests.cases_ipr import he_state_dict, normalise

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_metric_oracle_matches_reference_goldens():
    g = np.load(os.path.join(GOLDEN, "ipr_metrics.npz"))
    k = int(g["k"])
    np.testing.assert_allclose(R.radii(g["real"], k), g["radii_real"], rtol=1e-12)
    np.testing.assert_allclose(R.radii(g["fake"], k), g["radii_fake"], rtol=1e-12)
    p = R.cover(g["real"], g["radii_real"], g["fake"])
    r = R.cover(g["fake"], g["radii_fake"], g["real"])
    assert np.array_equal(p, g["precision_flags"]) and np.array_equal(r, g["recall_flags"])
    assert p.mean() == float(g["precision"]) and r.mean() == float(g["recall"])
    assert 0 < p.mean() < 1 and 0 < r.mean() < 1
    np.testing.assert_allclose(R.realism(g["real"], g["radii_real"], g["fake"][:20]), g["realism"], rtol=1e-5)


def test_distances2radii_is_the_references_order_statistic():
    rng = np.random.default_rng(0)
    d = rng.random((30, 30))
    d[:, 5] = d[:, 6]                                    # ties
    for k in (1, 3, 16):
        want = np.array([np.partition(row, k + 1)[:k + 1].max() for row in d])      # get_kth_value
        assert np.array_equal(I.distances2radii(d, k), want)


def test_vgg_oracle_matches_torchvision_golden():
    g = np.load(os.path.join(GOLDEN, "ipr_features.npz"))
    with torch.no_grad():
        got = V.features(he_state_dict(seed=1), normalise(g["images_u8"])).numpy()
    err = np.linalg.norm(got - g["features"], axis=1) / np.linalg.norm(got, axis=1)
    assert err.max() < 1e-5, err


def test_weight_names_follow_torchvision_state_dict():
    tv = pytest.importorskip("torchvision")
    sd = tv.models.vgg16().state_dict()
    ours = he_state_dict(seed=0)
    assert list(ours) == list(sd)
    assert all(ours[n].shape == sd[n].shape for n in sd)


def test_fc1_column_permutation():
    """NHWC (y, x, c) flatten with permuted fc1 columns == the reference's NCHW (c, y, x) flatten."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 512, 7, 7, generator=g, dtype=torch.float64)
    w = torch.randn(5, 25088, generator=g, dtype=torch.float64)
    j = torch.arange(25088)
    src = (j % 512) * 49 + j // 512                      # k_vgg_pack_fc with permute = 1
    got = x.permute(0, 2, 3, 1).reshape(2, -1) @ w[:, src].T
    assert torch.allclose(got, x.reshape(2, -1) @ w.T, rtol=1e-12, atol=1e-12)


def test_cabi_symbols_exported():
    lib = capi.load()
    for name in ("ds_vgg_create", "ds_vgg_destroy", "ds_vgg_expected_weight_count", "ds_vgg_expected_weight",
                 "ds_vgg_set_weights", "ds_vgg_features", "ds_manifold_distances", "ds_manifold_radii",
                 "ds_manifold_cover"):
        assert hasattr(lib, name) and name in capi.EXPORTED


def test_manifold_file_interchanges_with_reference(tmp_path):
    m = I.Manifold(np.random.default_rng(0).random((7, 4096), dtype=np.float32), np.arange(7.0))
    f = str(tmp_path / "m.npz")
    I.save_manifold(f, m)
    with np.load(f) as z:                                  # the reference's compute_manifold reads these keys
        assert sorted(z.files) == ["feature", "radii"]
        assert np.array_equal(z["feature"], m.features) and np.array_equal(z["radii"], m.radii)
    np.savez_compressed(f, feature=m.features, radii=m.radii)      # the reference's save_ref
    back = I.load_manifold(f)
    assert np.array_equal(back.features, m.features) and np.array_equal(back.radii, m.radii)


def test_file_listing_and_subsampling_match_reference(tmp_path):
    from glob import glob
    for rel in ("a/1.png", "b/2.jpg", "3.png", "c/d/4.jpg", "5.txt"):
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(b"")
    root = str(tmp_path)
    want = glob(os.path.join(root, "**", "*.jpg"), recursive=True) + glob(os.path.join(root, "**", "*.png"),
                                                                          recursive=True)
    assert I.image_files(root) == want and len(want) == 4
    files = ["%05d.png" % i for i in range(50)]
    ref = list(files)
    random.Random(100).shuffle(ref)
    assert I.subsample(files, 20) == ref[:20]
    assert I.subsample(files, 0) == ref


def test_image_transform_matches_torchvision(tmp_path):
    tv = pytest.importorskip("torchvision")
    from PIL import Image
    from torchvision import transforms
    rng = np.random.default_rng(1)
    p = str(tmp_path / "x.png")
    Image.fromarray(rng.integers(0, 256, (256, 256, 4), dtype=np.uint8), "RGBA").save(p)
    t = transforms.Compose([transforms.Resize([224, 224]), transforms.ToTensor(),
                            transforms.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])])
    want = t(Image.open(p).convert("RGB")).numpy()
    assert np.array_equal(I.load_image(p), want)


def test_weight_lookup_raises_without_a_file(tmp_path, monkeypatch):
    monkeypatch.setenv("TORCH_HOME", str(tmp_path))
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url",
                        lambda *a, **k: pytest.fail("the weight lookup must not download"))
    with pytest.raises(FileNotFoundError, match="vgg16-397923af.pth"):
        I.find_weights()
    with pytest.raises(FileNotFoundError):
        I.find_weights(str(tmp_path / "nope.pth"))
    ck = tmp_path / "hub" / "checkpoints"
    ck.mkdir(parents=True)
    (ck / I.VGG16_WEIGHTS).write_bytes(b"")
    assert I.find_weights() == str(ck / I.VGG16_WEIGHTS)
