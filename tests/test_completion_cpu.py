"""CPU: the completion / rearrangement driver's host side (scripts/completion_rearrange.py): scene choice and
arrangement noise against the reference's lines, the encode -> post_process round trip of real boxes.npz scenes,
the dataset_stats.txt loader and flag checks that run before any device work."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

from diffuscene_b200 import synthetic_meshes as SM
from diffuscene_b200.postprocess import load_dataset_stats, post_process_batch
from diffuscene_b200.synthetic import DEFAULT_BOUNDS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REARRANGE = os.path.join(ROOT, "config", "rearrange", "diffusion_bedrooms_instancond_lat32_v_rearrange.yaml")
UNCOND = os.path.join(ROOT, "config", "uncond", "diffusion_bedrooms_instancond_lat32_v.yaml")


def _load():
    spec = importlib.util.spec_from_file_location("completion_rearrange",
                                                  os.path.join(ROOT, "scripts", "completion_rearrange.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


CR = _load()


def _reference_draws(n_sequences, n_rooms, arrange, given, seed, N=12, angle_dim=2):
    # scripts/completion_rearrange.py:290-324 of the reference, restated (given is a nonzero room index or None)
    np.random.seed(seed)
    out = []
    for i in range(n_sequences):
        if arrange:
            if i < n_rooms:
                scene_idx = given or i
            else:
                scene_idx = given or (i % n_rooms)
        else:
            scene_idx = given or np.random.choice(n_rooms)
        nt = na = None
        if arrange:
            if given:
                nt = 0.4 * np.random.randn(N, 3).astype(np.float32)
            else:
                np.random.seed(scene_idx); nt = np.random.randn(N, 3).astype(np.float32)
            np.random.seed(scene_idx + n_rooms); na = np.random.randn(N, angle_dim).astype(np.float32)
        out.append((int(scene_idx), nt, na))
    return out


@pytest.mark.parametrize("arrange", [False, True])
@pytest.mark.parametrize("given", [None, 3])
def test_scene_choice_and_noise_match_reference(arrange, given):
    n_rooms, n = 7, 20
    want = _reference_draws(n, n_rooms, arrange, given, seed=5)
    order = CR.choose_scenes(n, n_rooms, arrange, given, seed=5)
    assert order == [w[0] for w in want]
    if arrange:
        noise = CR.arrangement_noise(order, n_rooms, 12, 2, given is not None)
        for (nt, replace, na), (_, wt, wa) in zip(noise, want):
            assert replace == (given is not None)
            assert np.array_equal(nt, wt) and np.array_equal(na, wa)


def _rooms(tmp_path, n=4, layout=False):
    sc = SM.scenes(n, 7, 10, seed=30, empty=0.0)
    rng = np.random.default_rng(2)
    for b in range(n):
        k = 3 + b
        cl = np.zeros((k, 23), np.float32)
        cl[np.arange(k), sc["class_index"][b, :k]] = 1
        fv, ff = sc["floors"][b]
        d = tmp_path / ("Bedroom_s%d" % b)
        d.mkdir(parents=True)
        extra = {"room_layout": rng.integers(0, 2, (256, 256, 1)).astype(np.uint8) * 255} if layout else {}
        np.savez_compressed(str(d / "boxes.npz"), jids=np.array(["m%d" % j for j in range(k)]), class_labels=cl,
                            translations=sc["translations"][b, :k], sizes=sc["sizes"][b, :k],
                            angles=sc["angles"][b, :k], floor_plan_vertices=fv, floor_plan_faces=ff,
                            floor_plan_centroid=np.zeros(3, np.float32), **extra)
    return sc


def test_round_trip_of_real_scenes(tmp_path):
    _rooms(tmp_path)
    spec = importlib.util.spec_from_file_location("render_scenes", os.path.join(ROOT, "scripts", "render_scenes.py"))
    rs = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(rs)
    rooms, raw = rs.load_rooms(str(tmp_path))
    assert rooms == ["Bedroom_s%d" % b for b in range(4)]
    x = CR.encode_scenes(raw, 12, DEFAULT_BOUNDS, objfeat_dim=32)
    assert x.shape == (4, 12, 62)
    world = post_process_batch({"translations": x[..., :3], "sizes": x[..., 3:6], "angles": x[..., 6:8]},
                               DEFAULT_BOUNDS)
    for b, s in enumerate(raw):
        k = len(s["class_labels"])
        np.testing.assert_allclose(world["translations"][b, :k].numpy(), s["translations"], atol=2e-6)
        np.testing.assert_allclose(world["sizes"][b, :k].numpy(), s["sizes"], atol=2e-6)
        ang = world["angles"][b, :k, 0].numpy()
        np.testing.assert_allclose(np.cos(ang), np.cos(s["angles"][:, 0]), atol=2e-6)
        np.testing.assert_allclose(np.sin(ang), np.sin(s["angles"][:, 0]), atol=2e-6)
        cls = x[b, :, 8:30]
        assert torch.equal(cls[:k].argmax(-1), torch.as_tensor(s["class_labels"].argmax(-1)))
        assert (cls[k:, -1] == 1).all() and (cls[k:, :-1] == -1).all()         # padding rows: the empty class
        assert (x[b, k:, :8] == 0).all()


def test_room_layout_resize(tmp_path):
    from PIL import Image
    _rooms(tmp_path, n=1, layout=True)
    s = dict(np.load(str(tmp_path / "Bedroom_s0" / "boxes.npz")))
    m = CR.room_layout(s, (64, 64))
    want = np.asarray(Image.fromarray(s["room_layout"][:, :, 0]).resize((64, 64), resample=Image.BILINEAR))
    assert m.dtype == np.float32 and np.array_equal(m, want.astype(np.float32) / np.float32(255))


def test_dataset_stats_loader(tmp_path):
    stats = {"bounds_translations": [-2.7, 0.04, -2.75, 2.8, 3.6, 2.9], "bounds_sizes": [0.04, 0.02, 0.01, 2.9, 1.8, 2.6],
             "bounds_angles": [-3.14159, 3.14159], "bounds_objfeats_32": [1.0, -4.0, 4.0],
             "class_labels": ["bed", "chair", "end"], "object_types": ["bed", "chair"]}
    p = tmp_path / "dataset_stats.txt"
    p.write_text(json.dumps(stats))
    b = load_dataset_stats(str(p))
    for k in ("translations", "sizes", "angles", "objfeats_32"):
        assert len(b[k]) == len(DEFAULT_BOUNDS[k])
        for got, want in zip(b[k], DEFAULT_BOUNDS[k]):
            assert np.array_equal(got, want), k
    del stats["bounds_sizes"]
    p.write_text(json.dumps(stats))
    with pytest.raises(ValueError, match="bounds_sizes"):
        load_dataset_stats(str(p))


@pytest.mark.parametrize("argv,msg", [
    (["--arrange_objects"], "room_arrange_condition"),
    (["--num_partial", "13"], "num_partial"),
    (["--num_partial", "0"], "num_partial"),
    (["--n_sequences", "0"], "n_sequences"),
    (["--batch_size", "0"], "batch_size"),
    (["--mesh_catalogue", "m.npz"], "catalogue"),
    (["--window_size", "512"], "window_size"),
    (["--camera_position", "1,2"], "camera_position"),
])
def test_bad_flags_rejected_before_device_work(tmp_path, capsys, argv, msg):
    _rooms(tmp_path)
    with pytest.raises(SystemExit):
        CR.main([UNCOND, str(tmp_path / "out"), str(tmp_path)] + argv)
    assert msg in capsys.readouterr().err
    assert not (tmp_path / "out").exists()


def test_unknown_scene_id_and_missing_rooms(tmp_path):
    _rooms(tmp_path)
    with pytest.raises(SystemExit, match="not a room"):
        CR.main([REARRANGE, str(tmp_path / "out"), str(tmp_path), "--arrange_objects", "--scene_id", "Kitchen_x"])
    with pytest.raises(SystemExit):
        CR.main([UNCOND, str(tmp_path / "out"), str(tmp_path / "nowhere")])
    assert not (tmp_path / "out").exists()
