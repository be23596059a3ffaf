"""CPU: the training-data layer (diffuscene_b200.scene_data) without a GPU.

* tests/scene_data_ref.py reproduces the unmodified reference's samples (tests/golden/scene_data.npz) from the
  recorded draws;
* store loading in the reference's format: split selection, sorted order, class indices, the objfeat key and the
  layout resize; every refusal;
* the rotation draws (the fixed cascade and the continuous range), epoch coverage and the right-angle layout rotation;
* train_diffusion.py --no-synthetic needs a dataset directory.
"""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from diffuscene_b200 import scene_data as SD
from diffuscene_b200.synthetic import write_reference_rooms
from tests import scene_data_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "scene_data.npz")
NET = dict(sample_num_points=12, class_dim=22, angle_dim=2, objfeat_dim=32, objectness_dim=0,
           room_mask_condition=True)


def golden():
    return np.load(GOLDEN)


def golden_bounds(z, d):
    stats = json.loads(str(z[d + "/stats"]))
    t, s, a = (np.array(stats["bounds_" + k]) for k in ("translations", "sizes", "angles"))
    return {"translations": (t[:3], t[3:]), "sizes": (s[:3], s[3:]), "angles": (np.array(a[0]), np.array(a[1])),
            "objfeats": tuple(np.array([v]) for v in stats["bounds_objfeats"]),
            "objfeats_32": tuple(np.array([v]) for v in stats["bounds_objfeats_32"])}


def golden_cases(z):
    return [k[:-len("/meta")] for k in z.files if k.endswith("/meta")]


def test_oracle_reproduces_reference_golden():
    z = golden()
    assert sorted(golden_cases(z)) == ["jit_crot", "living", "no_prm", "rot_jit", "scale"]
    for c in golden_cases(z):
        meta = json.loads(str(z[c + "/meta"]))
        layout = c + "/out/room_layout_u8" in z.files        # only the right-angle cases keep their layouts
        rooms = ref.golden_rooms(z, meta["dataset"], (64, 64) if layout else None)
        bounds = golden_bounds(z, meta["dataset"])
        assert len(rooms) == len(z[c + "/out/length"]) == 24
        for i, room in enumerate(rooms):
            theta, jitter, ordering = ref.golden_draws(z, c, i)
            got = ref.sample(room, meta["encoding"], meta["augmentations"], bounds, meta["N"], theta=theta,
                             jitter=jitter, ordering=ordering)
            want = ref.golden_out(z, c, i)
            assert sorted(got) == sorted(want), (c, sorted(got), sorted(want))
            for k, v in got.items():
                assert np.asarray(v).shape == want[k].shape, (c, i, k)
                tol = 1e-6 if k == "room_layout" else 1e-7
                np.testing.assert_allclose(np.asarray(v, np.float64), want[k], rtol=0, atol=tol, err_msg=(c, i, k))


def test_fixed_rotation_cascade():
    pi = math.pi
    u = torch.tensor([[0.1, 0.9, 0.9], [0.25, 0.49, 0.0], [0.3, 0.5, 0.74], [0.9, 0.9, 0.75], [0.0, 0.0, 0.0]],
                     dtype=torch.float64)
    assert SD.fixed_rotation_angles(u).tolist() == [pi * 1.5, pi, pi * 0.5, 0.0, pi * 1.5]
    # the reference's cascade draws a new uniform per test; its angle from the recorded draws
    z = golden()
    n = 0
    for c in golden_cases(z):
        meta = json.loads(str(z[c + "/meta"]))
        if "fixed_rotations" not in meta["augmentations"]:
            continue
        for i in range(len(z[meta["dataset"] + "/tags"])):
            r = z[c + "/rand"][i]
            u = torch.from_numpy(np.where(np.isnan(r), 0.5, r))[None]      # draws the cascade did not make
            assert SD.fixed_rotation_angles(u).item() == z[c + "/theta"][i]
            n += 1
    assert n >= 72
    # probabilities 0.25, 0.375, 0.28125, 0.09375 on a fine grid of the three uniforms
    g = (torch.arange(16, dtype=torch.float64) + 0.5) / 16
    u = torch.cartesian_prod(g, g, g)
    th = SD.fixed_rotation_angles(u)
    frac = [float((th == v).double().mean()) for v in (pi * 1.5, pi, pi * 0.5, 0.0)]
    assert frac == [0.25, 0.375, 0.28125, 0.09375]


def test_continuous_rotation_draws():
    u = torch.tensor([[0.2, 0.0], [0.2, 1.0], [0.5, 0.3], [0.49, 0.5]], dtype=torch.float64)
    got = SD.continuous_rotation_angles(u).tolist()
    assert got[0] == 0.174533 and got[1] == pytest.approx(5.06145, abs=1e-15) and got[2] == 0.0
    assert got[3] == 0.5 * (5.06145 - 0.174533) + 0.174533
    z = golden()
    for i in range(24):     # np.random.uniform(lo, hi) = lo + (hi - lo) * u: the recorded angle lies in range
        th = z["jit_crot/theta"][i]
        assert th == 0.0 or 0.174533 <= th <= 5.06145


@pytest.mark.parametrize("k", [1, 2, 3])
def test_right_angle_rotation_is_rot90(k):
    from scipy.ndimage import rotate
    g = torch.Generator().manual_seed(k)
    from diffuscene_b200.synthetic import floor_plan_mask
    m = floor_plan_mask(g, 64)[0].numpy().astype(np.float32) * np.float32(0.75)
    m[3, 5] = 0.3
    theta = [0.0, np.pi * 0.5, np.pi, np.pi * 1.5][k]
    r = rotate(m[:, :, None], theta * 180 / np.pi, reshape=False)[:, :, 0]
    assert np.abs(r - np.rot90(m, k)).max() < 1e-6
    sp = {"room_layout": m[None]}
    ref._rotate(sp, theta, 0.0)
    np.testing.assert_array_equal(sp["room_layout"][0], np.rot90(m, k))


def _write(tmp_path, n=12, **kw):
    ds, csv = str(tmp_path / "ds"), str(tmp_path / "splits.csv")
    tags = write_reference_rooms(ds, csv, n, seed=3, **kw)
    return ds, csv, tags


def test_store_selects_splits_in_sorted_order(tmp_path):
    ds, csv, tags = _write(tmp_path, 12)
    rows = [l.strip().split(",") for l in open(csv)]
    open(os.path.join(ds, "README"), "w").close()                  # no "_": the reference would fail here
    os.makedirs(os.path.join(ds, "x_" + rows[0][0] + "_empty"))     # no boxes.npz
    store = SD.SceneStore(ds, csv, ["train", "val"], NET, device="cpu")
    want = sorted(t for t in tags if t.split("_")[1] in {r[0] for r in rows if r[1] in ("train", "val")})
    assert store.tags == want and len(store) == 8
    test = SD.SceneStore(ds, csv, ["test"], NET, device="cpu")
    assert len(test) == 4 and not set(test.tags) & set(store.tags)
    assert store.n_classes == 23 and store.feature_size == 30 and store.objfeat_key == "objfeats_32"
    off = store.offsets.numpy()
    for s, tag in enumerate(store.tags):
        D = np.load(os.path.join(ds, tag, "boxes.npz"))
        L = len(D["class_labels"])
        assert store.lengths[s] == L
        sl = slice(off[s], off[s] + L)
        np.testing.assert_array_equal(store.class_index[sl].numpy(), D["class_labels"].argmax(1))
        np.testing.assert_array_equal(store.translations[sl].numpy(), D["translations"])
        np.testing.assert_array_equal(store.angles[sl].numpy(), D["angles"][:, 0])
        np.testing.assert_array_equal(store.objfeats[sl].numpy(), D["objfeats_32"])
        pil = Image.fromarray(D["room_layout"][:, :, 0]).resize((64, 64), resample=Image.BILINEAR)
        np.testing.assert_array_equal(store.layouts[s, 0].numpy(), np.asarray(pil).astype(np.float32) / np.float32(255))
    s64 = SD.SceneStore(ds, csv, ["train"], dict(NET, objfeat_dim=64, room_mask_condition=False), device="cpu",
                        room_layout_size="32,32")
    assert s64.objfeat_key == "objfeats" and s64.objfeats.shape[1] == 64 and s64.layouts is None
    assert SD.SceneStore(ds, csv, ["train"], dict(NET, objfeat_dim=0), device="cpu").objfeats is None
    assert s64.bounds["objfeats"][1][0] == -5.0 and s64.bounds["translations"][0].dtype == np.float64


def test_store_refusals(tmp_path):
    ds, csv, tags = _write(tmp_path, 6, max_objects=12)
    with pytest.raises(ValueError, match="more than sample_num_points"):
        SD.SceneStore(ds, csv, ["train", "val", "test"], dict(NET, sample_num_points=3), device="cpu")
    with pytest.raises(ValueError, match="sample_num_points 33"):
        SD.SceneStore(ds, csv, ["train"], dict(NET, sample_num_points=33), device="cpu")
    with pytest.raises(ValueError, match="max_length"):
        SD.SceneStore(ds, csv, ["train"], NET, max_length=21, device="cpu")
    with pytest.raises(ValueError, match="class_dim"):
        SD.SceneStore(ds, csv, ["train"], dict(NET, class_dim=21), device="cpu")
    with pytest.raises(ValueError, match="angle_dim"):
        SD.SceneStore(ds, csv, ["train"], dict(NET, angle_dim=1), device="cpu")
    with pytest.raises(ValueError, match="text"):
        SD.SceneStore(ds, csv, ["train"], NET, encoding_type="cached_diffusion_cosin_angle_text_wocm", device="cpu")
    with pytest.raises(ValueError, match="objectness"):
        SD.SceneStore(ds, csv, ["train"], dict(NET, objectness_dim=1), device="cpu")
    with pytest.raises(ValueError, match="no room"):
        SD.SceneStore(ds, csv, ["overfit"], NET, device="cpu")
    tag = sorted(tags)[0]
    split = [l.split(",")[1].strip() for l in open(csv) if l.startswith(tag.split("_")[1] + ",")][0]
    path = os.path.join(ds, tag, "boxes.npz")
    D = dict(np.load(path))
    np.savez(path, **{k: v for k, v in D.items() if k != "objfeats_32"})
    with pytest.raises(ValueError, match="%s has no objfeats_32" % tag):
        SD.SceneStore(ds, csv, [split], NET, device="cpu")
    cl = D["class_labels"].copy()
    cl[0, -1] = 1
    np.savez(path, **dict(D, class_labels=cl))
    with pytest.raises(ValueError, match="%s: a class_labels row is not one-hot" % tag):
        SD.SceneStore(ds, csv, [split], NET, device="cpu")
    for bad, msg in ((["jitter", "jitter"], "twice"), (["flip"], "unknown"), (["rotations"], "continuous"),
                     (["rotations", "fixed_rotations"], "together")):
        with pytest.raises(ValueError, match=msg):
            SD.parse_augmentations(bad, layouts=True)
    assert SD.parse_augmentations(["jitter", "rotations"], layouts=False) == [3, 2]
    assert SD.parse_encoding("cached_diffusion_cosin_angle_wocm_no_prm", 2) == (1, False)
    assert SD.parse_encoding("cached_diffusion_objfeats_lat32_wocm", 1) == (0, True)


def test_epoch_coverage_and_reproducibility(tmp_path):
    ds, csv, _ = _write(tmp_path, 23)
    store = SD.SceneStore(ds, csv, ["train", "val", "test"], NET, device="cpu")
    loader = SD.SceneLoader(store, 5, shuffle=True, seed=4)
    assert len(loader) == 5
    e1, e2 = loader.epoch_indices(), loader.epoch_indices()
    assert [len(b) for b in e1] == [5, 5, 5, 5, 3]
    assert sorted(torch.cat(e1).tolist()) == list(range(23)) == sorted(torch.cat(e2).tolist())
    assert torch.cat(e1).tolist() != torch.cat(e2).tolist()
    again = SD.SceneLoader(store, 5, shuffle=True, seed=4)
    assert [b.tolist() for b in again.epoch_indices()] == [b.tolist() for b in e1]
    d1 = loader.draws(7)
    assert d1[0].shape == (7,) and d1[1] is None and d1[2].shape == (7, 12) and d1[2].dtype == torch.float32
    assert [b.tolist() for b in SD.SceneLoader(store, 10, shuffle=False).epoch_indices()] == \
        [list(range(10)), list(range(10, 20)), [20, 21, 22]]
    val = SD.SceneLoader(store, 4, shuffle=False, augmentations=[])
    rot, jit, key = val.draws(4)
    assert rot is None and jit is None and key.shape == (4, 12)
    with pytest.raises(IndexError):
        store.batch([0, 23])


def test_no_synthetic_needs_a_dataset_directory(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import train_diffusion
    cfg = os.path.join(ROOT, "config", "uncond", "diffusion_bedrooms_instancond_lat32_v.yaml")
    with pytest.raises(SystemExit):
        train_diffusion.main([cfg, str(tmp_path / "out"), "--no-synthetic"])
    with pytest.raises(SystemExit):
        train_diffusion.main([cfg, str(tmp_path / "out"), "--no-synthetic", "--dataset_directory", str(tmp_path)])
