"""Scene-evaluation golden vectors: the UNMODIFIED reference `computer_intersection` and `computer_symmetry`
(scripts/utils.py:560-745) on hand-made and seeded scenes.

Run in the authoring container only (needs the reference checkout):
    python tests/golden/make_golden_scene_eval.py
scripts/utils.py imports rendering and mesh libraries (turtle, pyrr, simple_3dviz, trimesh, open3d, pyvista) and
scene_synthesis.utils at module level; the two functions use none of them, so empty stand-in modules are registered
before the import.  `scene_synthesis` itself stays the reference's package; only its `utils` submodule (which needs
seaborn and simple_3dviz) is replaced.  The functions receive stub meshes exposing `.bounding_box.bounds`,
`.vertices` and `.faces` (the 8 corners and 12 triangles of the box).

Writes tests/golden/scene_eval.npz: `names`, and per case k `k/bounds` [n, 6] float64, `k/classes` [n],
`k/jids` [n], `k/iou` [n, n] float32 (the reference's pair-IoU matrix; empty for n <= 1), `k/inter` [5] float64
(the five computer_intersection outputs) and `k/sym` [2] (computer_symmetry with the jids, and without them).
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("DS_REFERENCE_ROOT", "/root/reference")
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests.cases_scene_eval import golden_cases  # noqa: E402


def _load_reference_utils():
    for name in ("turtle", "pyrr", "simple_3dviz", "simple_3dviz.renderables", "simple_3dviz.renderables.textured_mesh",
                 "simple_3dviz.utils", "simple_3dviz.behaviours", "simple_3dviz.behaviours.misc",
                 "simple_3dviz.behaviours.io", "trimesh", "open3d", "pyvista"):
        sys.modules[name] = types.ModuleType(name)
    sys.modules["turtle"].color = None
    sys.modules["pyrr"].Matrix44 = None
    sys.modules["simple_3dviz"].Mesh = sys.modules["simple_3dviz"].Scene = None
    sys.modules["simple_3dviz.renderables.textured_mesh"].Material = None
    sys.modules["simple_3dviz.renderables.textured_mesh"].TexturedMesh = None
    sys.modules["simple_3dviz.utils"].save_frame = sys.modules["simple_3dviz.utils"].render = None
    sys.modules["simple_3dviz.behaviours.misc"].LightToCamera = None
    sys.modules["simple_3dviz.behaviours.io"].SaveFrames = None
    sys.path.insert(0, REF)
    import scene_synthesis
    assert os.path.realpath(scene_synthesis.__file__).startswith(os.path.realpath(REF)), scene_synthesis.__file__
    su = types.ModuleType("scene_synthesis.utils")
    su.get_textured_objects = su.get_textured_objects_based_on_objfeats = None
    sys.modules["scene_synthesis.utils"] = su
    spec = importlib.util.spec_from_file_location("reference_scripts_utils", os.path.join(REF, "scripts", "utils.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class _BBox:
    def __init__(self, b):
        self.bounds = np.asarray(b, np.float64).reshape(2, 3)


class StubMesh:
    FACES = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6],
                      [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]])

    def __init__(self, b):
        self.bounding_box = _BBox(b)
        lo, hi = self.bounding_box.bounds
        self.vertices = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])])
        self.faces = self.FACES


def main():
    U = _load_reference_utils()
    out = {}
    names = []
    for name, (bounds, classes, jids) in golden_cases().items():
        names.append(name)
        meshes = [StubMesh(b) for b in bounds]
        n_cls = int(classes.max()) + 2 if len(classes) else 2
        onehot = np.eye(n_cls, dtype=np.float32)[classes]
        inter = U.computer_intersection(meshes)
        if len(meshes) > 1:
            box = torch.from_numpy(np.stack([m.bounding_box.bounds.reshape(-1) for m in meshes]).astype(np.float32)[None])
            iou = U.axis_aligned_bbox_overlaps_3d(box, box)[0][0].numpy()
        else:
            iou = np.zeros((0, 0), np.float32)
        out[name + "/bounds"] = np.asarray(bounds, np.float64).reshape(-1, 6)
        out[name + "/classes"] = classes.astype(np.int64)
        out[name + "/jids"] = jids.astype(np.int64)
        out[name + "/iou"] = iou
        out[name + "/inter"] = np.array([float(v) for v in inter], np.float64)
        out[name + "/sym"] = np.array([U.computer_symmetry(meshes, onehot, [int(j) for j in jids]),
                                       U.computer_symmetry(meshes, onehot)], np.int64)
        print("%-16s n=%2d  %s  sym %s" % (name, len(meshes), inter, out[name + "/sym"]))
    out["names"] = np.array(names)
    np.savez_compressed(os.path.join(HERE, "scene_eval.npz"), **out)


if __name__ == "__main__":
    main()
