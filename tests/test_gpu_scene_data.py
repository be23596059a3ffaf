"""GPU: ds_scene_batch and the device-resident training data of diffuscene_b200.scene_data.

* the kernel on the reference's golden rooms with its recorded draws: class labels, lengths and padding identical,
  floats within 2 ulp of fp32, layouts within 1e-6; the living-room encoding differs only in the documented objfeat
  permutation;
* the kernel against tests/scene_data_ref.py on seeded stores of 4096 rooms over object counts, objfeat widths,
  angle encodings, augmentation orders, permutation, the four layout rotations and batch sizes;
* repeat launches are bit-identical and permutation only reorders a scene's rows; ABI errors;
* a native loss on a kernel-built batch equals get_loss on the oracle-built batch;
* train_diffusion.py --no-synthetic end to end.
"""
import json
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from diffuscene_b200 import capi
from diffuscene_b200 import scene_data as SD
from diffuscene_b200.synthetic import write_reference_rooms
from tests import scene_data_ref as ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "scene_data.npz")
DS_ERR_INVALID = -1      # include/diffuscene_b200.h ds_status
FLOAT_KEYS = ("translations", "sizes", "angles", "objfeats_32", "objfeats")


def assert_ulp(got, want, n=2, what=""):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    tol = n * np.spacing(np.maximum(np.abs(got), np.abs(want)))
    bad = np.abs(got.astype(np.float64) - want.astype(np.float64)) > tol
    assert not bad.any(), (what, int(bad.sum()), got[bad][:4], want[bad][:4])


def _net(N, class_dim, angle_dim, objfeat_dim, layouts):
    return dict(sample_num_points=N, class_dim=class_dim, angle_dim=angle_dim, objfeat_dim=objfeat_dim,
                objectness_dim=0, room_mask_condition=layouts)


def golden_batch(tmp_path, z, c):
    meta = json.loads(str(z[c + "/meta"]))
    d, N = meta["dataset"], meta["N"]
    layouts = c + "/out/room_layout_u8" in z.files
    cosin = "cosin_angle" in meta["encoding"] or "objfeatsnorm" in meta["encoding"]
    class_dim = z[d + "/class_labels"].shape[1] - 1
    ds, csv = tmp_path / d, tmp_path / (d + ".csv")
    tags = [str(t) for t in z[d + "/tags"]]
    ds.mkdir()
    for r, (tag, room) in enumerate(zip(tags, ref.golden_rooms(z, d))):
        (ds / tag).mkdir()
        np.savez(str(ds / tag / "boxes.npz"), room_layout=z[d + "/room_layout"][r], **room)
    (ds / "dataset_stats.txt").write_text(str(z[d + "/stats"]))
    csv.write_text("".join("%s,train\n" % t.split("_")[1] for t in tags))
    store = SD.SceneStore(str(ds), str(csv), ["train"], _net(N, class_dim, 2 if cosin else 1, 32, layouts),
                          encoding_type=meta["encoding"], device="cuda")
    S = len(store)
    assert store.tags == tags
    draws = [ref.golden_draws(z, c, i) for i in range(S)]
    theta = torch.tensor([t for t, _, _ in draws], dtype=torch.float64)
    jitter = torch.tensor(np.stack([j for _, j, _ in draws]), dtype=torch.float64)
    keys = None
    if store.permute:
        keys = torch.from_numpy(np.stack([ref.keys_from_ordering(o, N) for _, _, o in draws]))
    out = store.batch(torch.arange(S), rot_angle=theta, jitter=jitter, perm_key=keys,
                      augmentations=meta["augmentations"])
    return meta, store, {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("case", ["rot_jit", "jit_crot", "scale", "no_prm", "living"])
def test_kernel_matches_reference_golden(tmp_path, case):
    z = np.load(GOLDEN)
    meta, store, got = golden_batch(tmp_path, z, case)
    assert len(store) == 24
    for i in range(len(store)):
        want = ref.golden_out(z, case, i)
        assert got["length"][i] == want["length"]
        np.testing.assert_array_equal(got["class_labels"][i], want["class_labels"])
        L = int(want["length"])
        for k in FLOAT_KEYS:
            if k not in got:
                continue
            if case == "living" and k == "objfeats_32":
                # the documented difference: the reference leaves the shape latents in file order, here they move
                # with their boxes
                perm = ref.golden_draws(z, case, i)[2]
                assert_ulp(got[k][i][:L], want[k][:L][perm], what=(case, i, k))
                assert_ulp(got[k][i][L:], want[k][L:], what=(case, i, k))
                if L > 1 and (perm != np.arange(L)).any():
                    assert (got[k][i][:L] != want[k][:L]).any()
                continue
            assert_ulp(got[k][i], want[k], what=(case, i, k))
            assert (got[k][i][L:] == 0).all()
        assert ("room_layout" in want) == ("room_layout" in got)
        if "room_layout" in want:
            np.testing.assert_allclose(got["room_layout"][i], want["room_layout"], rtol=0, atol=1e-6)


@pytest.fixture(scope="module")
def big_datasets(tmp_path_factory):
    out = {}
    for N in (12, 21):
        d = tmp_path_factory.mktemp("rooms%d" % N)
        write_reference_rooms(str(d / "ds"), str(d / "splits.csv"), 4096, max_objects=N, n_object_classes=21,
                              layout_size=64, seed=N, splits=("train",))
        out[N] = (str(d / "ds"), str(d / "splits.csv"))
    return out


def oracle_batch(store, idx, augs, rot, jit, keys, permute=True):
    """tests/scene_data_ref.py on the store's own rooms (get_room_params' dicts rebuilt from the packed arrays)."""
    enc = store.encoding_type
    b = store.bounds
    names = [n for n in augs]
    out = []
    off, lens = store.offsets.cpu().numpy(), store.lengths.cpu().numpy()
    cls, tr, sz = store.class_index.cpu().numpy(), store.translations.cpu().numpy(), store.sizes.cpu().numpy()
    an = store.angles.cpu().numpy()
    of = store.objfeats.cpu().numpy() if store.objfeats is not None else None
    lay = store.layouts.cpu().numpy() if store.layouts is not None else None
    for r, s in enumerate(idx.tolist()):
        sl = slice(off[s], off[s] + lens[s])
        L = int(lens[s])
        room = {}
        if lay is not None:
            room["room_layout"] = lay[s]
        room.update(class_labels=np.eye(store.n_classes, dtype=np.float32)[cls[sl]], translations=tr[sl],
                    sizes=sz[sl], angles=an[sl][:, None])
        if of is not None:
            room[store.objfeat_key] = of[sl]
        ordering = ref.ordering_from_keys(keys[r], L) if permute else None
        out.append(ref.sample(room, enc if permute else enc + "_no_prm", names, b, store.N,
                              theta=float(rot[r]) if rot is not None else 0.0,
                              jitter=jit[r] if jit is not None else (0.0, 0.0, 0.0), ordering=ordering,
                              permute_objfeats=True))
    return {k: np.stack([o[k] for o in out]) for k in out[0]}


ORACLE_CASES = [
    # N, objfeat, angle_dim, augmentations, permute, layouts, B
    (12, 32, 2, ["fixed_rotations", "jitter"], True, True, 4096),
    (21, 64, 2, ["jitter", "fixed_rotations"], True, True, 128),
    (12, 0, 1, ["fixed_rotations", "jitter"], True, False, 37),
    (21, 32, 1, ["jitter", "rotations"], False, False, 1),
    (12, 64, 2, ["rotations", "jitter"], True, False, 4096),
    (21, 0, 2, ["fixed_rotations"], False, True, 37),
    (12, 32, 2, [], True, False, 128),
    (21, 32, 2, ["jitter", "rotations"], True, False, 4096),
]


@pytest.mark.parametrize("N,F,angle_dim,augs,permute,layouts,B", ORACLE_CASES)
def test_kernel_matches_oracle(big_datasets, N, F, angle_dim, augs, permute, layouts, B):
    ds, csv = big_datasets[N]
    enc = ("cached_diffusion_cosin_angle_objfeatsnorm_lat32_wocm" if angle_dim == 2 else
           "cached_diffusion_objfeats_lat32_wocm") + ("" if permute else "_no_prm")
    store = SD.SceneStore(ds, csv, ["train"], _net(N, 22, angle_dim, F, layouts), encoding_type=enc,
                          room_layout_size="32,32", device="cuda")
    assert len(store) == 4096 and int(store.lengths.max()) == N
    loader = SD.SceneLoader(store, B, augmentations=augs, seed=B + N)
    idx = loader.epoch_indices()[0]
    rot, jit, keys = loader.draws(B)
    if permute:      # ties, broken by index
        keys[:, 1] = keys[:, 0]
    got = {k: v.cpu().numpy() for k, v in store._launch(idx, loader.augs, permute, rot, jit, keys).items()}
    c = lambda t: None if t is None else t.cpu().numpy()
    want = oracle_batch(store, idx.cpu(), augs, c(rot), c(jit), c(keys), permute)
    np.testing.assert_array_equal(got["length"], want["length"])
    np.testing.assert_array_equal(got["class_labels"], want["class_labels"])
    for k in FLOAT_KEYS:
        if k in want:
            assert_ulp(got[k], want[k], what=k)
    assert ("objfeats" in got or "objfeats_32" in got) == (F > 0)
    if layouts:
        np.testing.assert_allclose(got["room_layout"], want["room_layout"], rtol=0, atol=1e-6)
        if "fixed_rotations" in augs and B == 4096:
            assert sorted(set(np.round(c(rot) / (math.pi / 2)).astype(int).tolist())) == [0, 1, 2, 3]


def test_repeatable_and_permutation_only_reorders(big_datasets):
    ds, csv = big_datasets[21]
    store = SD.SceneStore(ds, csv, ["train"], _net(21, 22, 2, 32, True), device="cuda")
    loader = SD.SceneLoader(store, 4096, augmentations=["fixed_rotations", "jitter"], seed=1)
    idx = loader.epoch_indices()[0]
    rot, jit, keys = loader.draws(4096)
    a = store._launch(idx, loader.augs, True, rot, jit, keys)
    b = store._launch(idx, loader.augs, True, rot, jit, keys)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    plain = store._launch(idx, loader.augs, False, rot, jit, None)
    rows = lambda o: torch.cat([o["class_labels"], o["translations"], o["sizes"], o["angles"], o["objfeats_32"]], -1)
    ra, rp = rows(a).cpu().numpy(), rows(plain).cpu().numpy()
    for s in range(0, 4096, 97):
        assert sorted(map(tuple, ra[s])) == sorted(map(tuple, rp[s]))
    assert not np.array_equal(ra, rp)
    assert torch.equal(a["room_layout"], plain["room_layout"])


def test_abi_errors(big_datasets):
    ds, csv = big_datasets[12]
    store = SD.SceneStore(ds, csv, ["train"], _net(12, 22, 2, 32, True), device="cuda")
    idx = torch.arange(4, device="cuda")
    rot = torch.zeros(4, dtype=torch.float64, device="cuda")
    keys = torch.rand(4, 12, device="cuda")
    lib = capi.load()

    def call(**over):
        a = capi.DsSceneBatchArgs()
        out = store._launch(idx, [capi.DS_SCENE_AUG_FIXED_ROTATION], True, rot, None, keys)
        assert out["length"].shape == (4,)
        import ctypes
        # rebuild the same arguments and break one field
        s = store
        a.num_scenes, a.num_class_columns, a.objfeat_dim, a.layout_h, a.layout_w = len(s), s.n_classes, 32, 32, 32
        a.layout_h = a.layout_w = int(s.layouts.shape[-1])
        a.scaling, a.angle_dim, a.permute, a.num_augmentations = 1, 2, 1, 1
        a.augmentations[0] = capi.DS_SCENE_AUG_FIXED_ROTATION
        a.batch, a.num_slots = 4, 12
        a.offsets_dev, a.lengths_dev, a.class_dev = s.offsets.data_ptr(), s.lengths.data_ptr(), s.class_index.data_ptr()
        a.translations_dev, a.sizes_dev, a.angles_dev = (s.translations.data_ptr(), s.sizes.data_ptr(),
                                                         s.angles.data_ptr())
        a.objfeats_dev, a.layouts_dev = s.objfeats.data_ptr(), s.layouts.data_ptr()
        a.scene_index_dev, a.rot_angle_dev, a.perm_key_dev = idx.data_ptr(), rot.data_ptr(), keys.data_ptr()
        for k in ("class_labels", "translations", "sizes", "angles", "objfeats_32", "length", "room_layout"):
            name = {"objfeats_32": "objfeats_out_dev", "length": "length_out_dev",
                    "room_layout": "room_layout_out_dev"}.get(k, k + "_out_dev")
            setattr(a, name, out[k].data_ptr())
        for k, v in over.items():
            if k == "augs":
                a.num_augmentations = len(v)
                for i, op in enumerate(v):
                    a.augmentations[i] = op
            else:
                setattr(a, k, v)
        return lib.ds_scene_batch(ctypes.byref(a), None)

    assert call() == 0
    torch.cuda.synchronize()
    assert lib.ds_scene_batch(None, None) == DS_ERR_INVALID
    bad = [dict(num_slots=33), dict(num_slots=0), dict(batch=-1), dict(angle_dim=1), dict(scaling=7),
           dict(objfeat_dim=30), dict(offsets_dev=None), dict(objfeats_out_dev=None), dict(perm_key_dev=None),
           dict(rot_angle_dev=None), dict(room_layout_out_dev=None), dict(augs=[capi.DS_SCENE_AUG_ROTATION]),
           dict(augs=[capi.DS_SCENE_AUG_JITTER, capi.DS_SCENE_AUG_JITTER]), dict(augs=[9]),
           dict(augs=[capi.DS_SCENE_AUG_FIXED_ROTATION, capi.DS_SCENE_AUG_FIXED_ROTATION]),
           dict(layout_h=16), dict(num_scenes=0), dict(num_class_columns=1)]
    for over in bad:
        assert call(**over) == DS_ERR_INVALID, over
    assert call(augs=[capi.DS_SCENE_AUG_JITTER]) == DS_ERR_INVALID        # jitter without draws
    with pytest.raises(IndexError):
        store.batch([0, 4096], rot_angle=[0.0, 0.0], perm_key=torch.zeros(2, 12))
    with pytest.raises(ValueError, match="shape"):
        store.batch([0, 1], rot_angle=[0.0], perm_key=torch.zeros(2, 12), augmentations=["fixed_rotations"])


def test_native_loss_on_kernel_batch_equals_oracle_batch(big_datasets):
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    from training_utils import load_config
    from scene_synthesis.networks import build_network
    ds, csv = big_datasets[12]
    config = load_config(os.path.join(ROOT, "config", "uncond", "diffusion_bedrooms_instancond_lat32_v.yaml"))
    config["network"]["diffusion_kwargs"]["loss_iou"] = False
    store = SD.SceneStore(ds, csv, ["train"], config["network"], device="cuda")
    loader = SD.SceneLoader(store, 128, augmentations=["fixed_rotations", "jitter"], seed=3)
    idx = loader.epoch_indices()[0]
    rot, jit, keys = loader.draws(128)
    got = store._launch(idx, loader.augs, True, rot, jit, keys)
    c = lambda t: t.cpu().numpy()
    want = oracle_batch(store, idx.cpu(), ["fixed_rotations", "jitter"], c(rot), c(jit), c(keys))
    want = {k: torch.from_numpy(np.asarray(v)).cuda() for k, v in want.items()}
    torch.manual_seed(0)
    network, _, _ = build_network(store.feature_size, store.n_classes, config, None, device=torch.device("cuda"),
                                  precision="fp32")
    network.eval()
    g = torch.Generator(device="cuda").manual_seed(5)
    t = torch.randint(0, 1000, (128,), device="cuda", generator=g)
    noise = torch.randn(128, 12, config["network"]["point_dim"], device="cuda", generator=g)
    with torch.no_grad():
        la, _ = network.get_loss(got, t=t, noise=noise)
        lb, _ = network.get_loss(want, t=t, noise=noise)
    assert torch.isfinite(la)
    assert abs(la.item() - lb.item()) <= 1e-5 * abs(lb.item()), (la.item(), lb.item())


@pytest.mark.parametrize("config", ["uncond/diffusion_bedrooms_instancond_lat32_v.yaml",
                                    "floorplan/diffusion_bedrooms_instancond_lat32_v_floorplan.yaml",
                                    "rearrange/diffusion_bedrooms_instancond_lat32_v_rearrange.yaml"])
def test_train_script_on_real_format_rooms(tmp_path, config):
    ds, csv = tmp_path / "ds", tmp_path / "splits.csv"
    write_reference_rooms(str(ds), str(csv), 200, max_objects=12, seed=2)      # 134 train + val: 128 + 6
    out = tmp_path / "out"
    cmd = [sys.executable, os.path.join(ROOT, "scripts", "train_diffusion.py"), os.path.join(ROOT, "config", config),
           str(out), "--no-synthetic", "--dataset_directory", str(ds), "--annotation_file", str(csv),
           "--max_epochs", "2", "--experiment_tag", "run", "--augmentations", "fixed_rotations,jitter"]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    exp = out / "run"
    assert (exp / "bounds.npz").exists()
    b = np.load(str(exp / "bounds.npz"))
    assert b["translations"].shape == (2, 3) and b["objfeats"].shape == (3, 1)
    assert sorted(p.name for p in exp.iterdir() if p.name.startswith("model_")) == ["model_00000", "model_00001"]
    lines = (exp / "stats.txt").read_text().splitlines()
    losses = [float(m.group(1)) for m in (re.search(r"loss: ([-\d.eE+naif]+)", l) for l in lines) if m]
    assert len(losses) >= 2 and all(math.isfinite(v) for v in losses), lines[-4:]
    batches = {int(re.search(r"batch: (\d+)", l).group(1)) for l in lines if l.startswith("epoch: 1 ")}
    assert batches == {1, 2}
