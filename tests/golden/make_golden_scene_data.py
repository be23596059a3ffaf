"""Training-data golden vectors: the UNMODIFIED reference data layer (scene_synthesis.datasets.get_encoded_dataset
with CachedThreedFront) on seeded rooms written in its preprocessed format, with every random draw recorded.

Run in the authoring container only (needs the reference checkout):
    python tests/golden/make_golden_scene_data.py
The reference's datasets package imports text and rendering modules at module level (torchtext, num2words, nltk,
trimesh, simple_3dviz, tkinter); the cached training chain uses none of them, so empty stand-ins are registered first
(nltk.corpus.cmudict needs a dict()).  The splits CSV lives outside the dataset directory, because the reference lists
every entry of that directory as a room.

np.random.rand / uniform / normal / permutation are wrapped to log each call, and
RotationAugmentation.rotation_matrix_around_y to log the angle it was given.  Writes tests/golden/scene_data.npz,
arrays stacked so the file holds few of them:
  * per dataset d: `d/tags` [R], `d/stats` (the dataset_stats.txt text), `d/lengths` [R] and the rooms' objects packed
    back to back in tag order: `d/class_labels` [T, C + 2], `d/translations`, `d/sizes` [T, 3], `d/angles` [T, 1],
    `d/objfeats_32` [T, 32]; `d/room_layout` [R, 256, 256, 1] uint8;
  * per case c: `c/meta` (JSON: dataset, encoding, augmentations, N, seed), `c/out/<key>` [R, ...] (the reference's
    samples after Diffusion, item i = room i), and the draws of each item: `c/rand` [R, 3] (the np.random.rand values
    in call order), `c/uniform` [R], `c/normal` [R, 3], `c/theta` [R] (NaN where not drawn) and `c/perm` [R, N]
    (-1 past the room's length).

To keep the file small, three things are left out or packed; none changes what the tests compare:
  * the 64-wide `objfeats`: the rooms hold them and the reference carries them through, but every case's network
    reads `objfeats_32`;
  * the output room_layout of all but LAYOUT_CASES;
  * the output room_layout of LAYOUT_CASES is stored as `out/room_layout_u8` = round(255 * layout) in uint8.  The
    reference's layout is a PIL-resized uint8 mask / 255, rotated by a right angle with scipy's spline (which adds
    roundoff of about 1e-25), so u8 / 255 is it to within 1e-6; the script asserts that.
"""
import json
import os
import shutil
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("DS_REFERENCE_ROOT", "/root/reference")
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from diffuscene_b200.synthetic import write_reference_rooms  # noqa: E402

DATASETS = {"bed": dict(n_rooms=24, max_objects=12, n_object_classes=21, seed=5),
            "liv": dict(n_rooms=24, max_objects=21, n_object_classes=24, seed=6)}
CASES = {
    "rot_jit": ("bed", "cached_diffusion_cosin_angle_objfeatsnorm_lat32_wocm", ["fixed_rotations", "jitter"], 12, 11),
    "jit_crot": ("bed", "cached_diffusion_cosin_angle_objfeatsnorm_lat32_wocm", ["jitter", "rotations"], 12, 12),
    "scale": ("bed", "cached_diffusion_objfeats_lat32_wocm", ["fixed_rotations", "jitter"], 12, 13),
    "no_prm": ("bed", "cached_diffusion_cosin_angle_objfeatsnorm_lat32_wocm_no_prm", ["fixed_rotations", "jitter"],
               12, 14),
    "living": ("liv", "cached_diffusion_cosin_angle_wocm", ["fixed_rotations"], 21, 15),
}
LAYOUT_CASES = ("rot_jit", "living")


def _stub_modules():
    for name in ("torchtext", "num2words", "nltk", "nltk.tokenize", "nltk.corpus", "trimesh", "simple_3dviz",
                 "simple_3dviz.renderables", "simple_3dviz.renderables.textured_mesh", "simple_3dviz.behaviours",
                 "simple_3dviz.behaviours.keyboard", "simple_3dviz.behaviours.misc", "simple_3dviz.utils",
                 "simple_3dviz.window", "tkinter"):
        sys.modules[name] = types.ModuleType(name)
    sys.modules["num2words"].num2words = None
    sys.modules["nltk.tokenize"].word_tokenize = None
    sys.modules["nltk.corpus"].cmudict = types.SimpleNamespace(dict=lambda: {})
    sys.modules["tkinter"].E = None
    for attr in ("Lines", "Mesh", "Spherecloud", "Scene"):
        setattr(sys.modules["simple_3dviz"], attr, None)
    sys.modules["simple_3dviz.renderables.textured_mesh"].Material = None
    sys.modules["simple_3dviz.renderables.textured_mesh"].TexturedMesh = None
    sys.modules["simple_3dviz.behaviours.keyboard"].SnapshotOnKey = lambda *a, **k: None
    sys.modules["simple_3dviz.behaviours.misc"].LightToCamera = lambda *a, **k: None


def _load_reference():
    _stub_modules()
    sys.path.insert(0, REF)
    for k in [k for k in sys.modules if k == "scene_synthesis" or k.startswith("scene_synthesis.")]:
        del sys.modules[k]
    import scene_synthesis.datasets as D
    import scene_synthesis.datasets.threed_front_dataset as TD
    assert os.path.realpath(D.__file__).startswith(os.path.realpath(REF)), D.__file__
    return D, TD


class Recorder:
    def __init__(self, TD):
        self.log = None
        for name in ("rand", "uniform", "normal", "permutation"):
            orig = getattr(np.random, name)
            setattr(np.random, name, self._wrap(name, orig))
        rot = TD.RotationAugmentation.rotation_matrix_around_y

        def rec_rot(theta):
            self.log.append(("theta", float(theta)))
            return rot(theta)
        TD.RotationAugmentation.rotation_matrix_around_y = staticmethod(rec_rot)

    def _wrap(self, name, orig):
        def f(*a, **k):
            v = orig(*a, **k)
            if self.log is not None:
                self.log.append((name, np.asarray(v).copy()))
            return v
        return f


def main():
    D, TD = _load_reference()
    rec = Recorder(TD)
    tmp = tempfile.mkdtemp()
    out = {}
    try:
        for d, kw in DATASETS.items():
            ds_dir, csv_path = os.path.join(tmp, d), os.path.join(tmp, d + "_splits.csv")
            tags = write_reference_rooms(ds_dir, csv_path, splits=("train",), **kw)
            rooms = [np.load(os.path.join(ds_dir, tag, "boxes.npz")) for tag in tags]
            out[d + "/tags"] = np.array(tags)
            out[d + "/lengths"] = np.array([len(z["class_labels"]) for z in rooms])
            for k in ("class_labels", "translations", "sizes", "angles", "objfeats_32"):
                out["%s/%s" % (d, k)] = np.concatenate([z[k] for z in rooms])
            out[d + "/room_layout"] = np.stack([z["room_layout"] for z in rooms])
            with open(os.path.join(ds_dir, "dataset_stats.txt")) as f:
                out[d + "/stats"] = np.array(f.read())
        for c, (d, enc, augs, N, seed) in CASES.items():
            cfg = {"dataset_type": "cached_threedfront", "encoding_type": enc,
                   "dataset_directory": os.path.join(tmp, d), "annotation_file": os.path.join(tmp, d + "_splits.csv"),
                   "augmentations": augs, "train_stats": "dataset_stats.txt", "room_layout_size": "64,64",
                   "max_length": N}
            ds = D.get_encoded_dataset(cfg, lambda s: s, path_to_bounds=None, augmentations=augs, split=["train"])
            np.random.seed(seed)
            out[c + "/meta"] = np.array(json.dumps(dict(dataset=d, encoding=enc, augmentations=augs, N=N, seed=seed)))
            R = len(ds)
            samples = []
            draws = {"rand": np.full((R, 3), np.nan), "uniform": np.full(R, np.nan), "normal": np.full((R, 3), np.nan),
                     "theta": np.full(R, np.nan), "perm": np.full((R, N), -1, np.int64)}
            for i in range(R):
                rec.log = []
                samples.append(ds[i])
                log, rec.log = rec.log, None
                for name in ("rand", "uniform", "normal", "permutation", "theta"):
                    vals = [np.asarray(v).reshape(-1) for n, v in log if n == name]
                    if vals:
                        v = np.concatenate(vals)
                        key = "perm" if name == "permutation" else name
                        if draws[key].ndim == 1:
                            assert len(v) == 1, (name, v)
                            draws[key][i] = v[0]
                        else:
                            draws[key][i, :len(v)] = v
            for k, v in draws.items():
                out["%s/%s" % (c, k)] = v
            for k in samples[0]:
                if k == "objfeats":
                    continue
                v = np.stack([np.asarray(s[k]) for s in samples])
                if k == "room_layout":
                    if c in LAYOUT_CASES:
                        u8 = np.round(v.astype(np.float64) * 255).astype(np.uint8)
                        assert np.abs(u8.astype(np.float32) / np.float32(255) - v).max() < 1e-6
                        out[c + "/out/room_layout_u8"] = u8
                    continue
                out["%s/out/%s" % (c, k)] = v
    finally:
        shutil.rmtree(tmp)
    path = os.path.join(HERE, "scene_data.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays,", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
