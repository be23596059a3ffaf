"""GPU: scripts/completion_rearrange.py end to end on synthetic rooms -- completion keeps the partial scene,
arrangement keeps classes and sizes and resamples translations and angles, every render is written, iou_states.txt
lines, a floor-plan config with real room_layout, and render_scenes.py scoring the results."""
import contextlib
import importlib.util
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image

from diffuscene_b200 import synthetic_meshes as SM
from oracle import inception_ref as IR
from tests.cases_ipr import he_state_dict

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = {k: os.path.join(ROOT, "config", k, n) for k, n in (
    ("uncond", "diffusion_bedrooms_instancond_lat32_v.yaml"),
    ("rearrange", "diffusion_bedrooms_instancond_lat32_v_rearrange.yaml"),
    ("floorplan", "diffusion_bedrooms_instancond_lat32_v_floorplan.yaml"))}


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "scripts", name + ".py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("cr")
    M = 42
    big = SM.catalogue(seed=6, num_models=M, detail=2, texture_size=32)
    np.savez(str(tmp / "mesh_catalogue.npz"), **big)
    rng = np.random.default_rng(8)
    np.savez(str(tmp / "catalogue.npz"), latents=rng.normal(size=(M, 32)).astype(np.float32),
             labels=np.arange(M) % 21, sizes=rng.uniform(0.2, 0.8, (M, 3)).astype(np.float32))
    rooms = tmp / "rooms"
    sc = SM.scenes(6, 7, M, seed=30, empty=0.0)
    for b in range(6):
        n = 4 + b % 3
        cl = np.zeros((n, 23), np.float32)
        cl[np.arange(n), sc["class_index"][b, :n]] = 1
        fv, ff = sc["floors"][b]
        centroid = np.array([0.3, 0.0, -0.2], np.float32)
        layout = np.zeros((256, 256, 1), np.uint8)
        layout[30 + 10 * b:200, 40:220] = 255
        d = rooms / ("Bedroom_s%d" % b)
        d.mkdir(parents=True)
        np.savez_compressed(str(d / "boxes.npz"), jids=big["jids"][sc["model_index"][b, :n]], class_labels=cl,
                            translations=sc["translations"][b, :n], sizes=sc["sizes"][b, :n],
                            angles=sc["angles"][b, :n], floor_plan_vertices=fv + centroid, floor_plan_faces=ff,
                            floor_plan_centroid=centroid, room_layout=layout)
    return tmp


def _run(data, cfg, out, *extra):
    args = [CFG[cfg], str(out), str(data / "rooms"), "--n_sequences", "5", "--batch_size", "2", "--ddim",
            "--ddim_steps", "5", "--catalogue", str(data / "catalogue.npz"), "--mesh_catalogue",
            str(data / "mesh_catalogue.npz"), "--compute_intersec", "--gen_gt"] + list(extra)
    with contextlib.redirect_stdout(io.StringIO()):
        _load("completion_rearrange").main(args)
    return [dict(np.load(str(out / ("scene_%05d.npz" % i)))) for i in range(5)]


def _pngs(out, folder, shape):
    names = []
    for i in range(5):
        npz = np.load(str(out / ("scene_%05d.npz" % i)))
        name = "%s_%d_%03d" % (str(npz["room"]), int(npz["scene_idx"]), i)
        for p in (out / folder / (name + "_render.png"), out / (name + ".png"),
                  out / "groundtruth" / (name + "_render.png")):
            img = np.asarray(Image.open(str(p)))
            assert img.shape == shape, (p, img.shape)
            assert (img != 255).any(), p                                # something was drawn on the white background
        names.append(name)
    return names


def _lines(out):
    return (out / "iou_states.txt").read_text().strip().split("\n")


def test_completion(data):
    out = data / "complete"
    res = _run(data, "uncond", out)
    np.random.seed(0)
    order = [int(np.random.choice(6)) for _ in range(5)]
    for i, r in enumerate(res):
        assert int(r["scene_idx"]) == order[i] and str(r["room"]) == "Bedroom_s%d" % order[i]
        s = np.load(str(data / "rooms" / str(r["room"]) / "boxes.npz"))
        assert r["translations"].shape[1] >= 3
        np.testing.assert_allclose(r["translations"][0, :3], s["translations"][:3], atol=1e-4)
        np.testing.assert_allclose(r["sizes"][0, :3], s["sizes"][:3], atol=1e-4)
        np.testing.assert_allclose(np.cos(r["angles"][0, :3]), np.cos(s["angles"][:3]), atol=1e-4)
        assert np.array_equal(r["class_index"][:3], s["class_labels"][:3].argmax(-1))
        assert r["model_index"].shape == r["class_index"].shape
    _pngs(out, "partial", (512, 512, 3))
    assert len(_lines(out)) == 2 * 5                                    # objfeat retrieval: plus an "only size" line


def test_arrangement(data):
    out = data / "arrange"
    res = _run(data, "rearrange", out, "--arrange_objects", "--retrieve_mode", "box")
    for i, r in enumerate(res):
        assert int(r["scene_idx"]) == i % 6
        s = np.load(str(data / "rooms" / str(r["room"]) / "boxes.npz"))
        n = len(s["class_labels"])
        assert np.array_equal(r["class_index"][:n], s["class_labels"].argmax(-1))
        np.testing.assert_allclose(r["sizes"][0, :n], s["sizes"], atol=1e-4)
        assert np.abs(r["translations"][0, :n] - s["translations"]).max() > 1e-2
        assert np.abs(np.cos(r["angles"][0, :n]) - np.cos(s["angles"])).max() > 1e-3
    _pngs(out, "noisy", (512, 512, 3))
    assert len(_lines(out)) == 5                                        # box retrieval: one line per sequence


def test_top2down_floorplan_and_scoring(data):
    out = data / "floorplan"
    _run(data, "floorplan", out, "--render_top2down", "--num_partial", "2")
    _pngs(out, "partial", (256, 256, 3))
    wi, wv = str(data / "inc.pth"), str(data / "vgg.pth")
    torch.save(IR.random_state_dict(seed=5), wi)
    torch.save(he_state_dict(1), wv)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        _load("render_scenes").main([str(data / "rooms"), "--mesh_catalogue", str(data / "mesh_catalogue.npz"),
                                     "--generated", str(out), "--fid", "--ipr", "--inception_weights", wi,
                                     "--vgg16_weights", wv])
    text = buf.getvalue()
    for key in ("fid: ", "kid: ", "precision: ", "recall: "):
        assert key in text, text
