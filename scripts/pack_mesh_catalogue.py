#!/usr/bin/env python
"""Pack 3D-FUTURE models into one mesh_catalogue.npz for the native top-down renderer (diffuscene_b200.render).

    python scripts/pack_mesh_catalogue.py MODEL_ROOT JIDS OUT.npz [--texture_size 256]

JIDS lists the models in catalogue order, the order of the catalogue.npz that generate_objautoencoder.py writes and
ObjectCatalog indexes: a text file with one jid per line, or an .npz with a `jids` array.  Each model is
MODEL_ROOT/<jid>/ with raw_model.obj (+ its .mtl for Kd), texture.png and bbox_vertices.npy.  The file holds the raw
vertices, triangles (polygons fanned), per-corner UVs, per-model offsets, raw_half / raw_aabb as
evaluate.model_footprint computes them, Kd, one texture per model resized to texture_size^2 with PIL bilinear, and
the jids.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from diffuscene_b200.render import TEXTURE_SIZE, pack_catalogue  # noqa: E402


def read_jids(path):
    if path.endswith(".npz"):
        with np.load(path) as f:
            return [str(j) for j in f["jids"]]
    with open(path) as f:
        return [l.strip() for l in f if l.strip()]


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("model_root", help="3D-FUTURE-model directory")
    p.add_argument("jids", help="jids in catalogue order: a text file (one per line) or an .npz with `jids`")
    p.add_argument("output", help="mesh_catalogue.npz to write")
    p.add_argument("--texture_size", type=int, default=TEXTURE_SIZE, help="side of the packed textures")
    a = p.parse_args(argv)
    jids = read_jids(a.jids)
    cat = pack_catalogue([os.path.join(a.model_root, j) for j in jids], jids, a.texture_size)
    np.savez(a.output, **cat)
    print("packed %d models, %d triangles into %s" % (len(jids), len(cat["faces"]), a.output))


if __name__ == "__main__":
    main()
