#!/usr/bin/env python
"""Native top-down renders of the real scenes, and FID / KID / precision-recall of generated scenes against them.

    python scripts/render_scenes.py ROOM_DIR OUT --mesh_catalogue mesh_catalogue.npz [--no_texture] [--without_floor]
    python scripts/render_scenes.py ROOM_DIR --mesh_catalogue F --generated GEN_DIR --fid --inception_weights W \
        [--ipr --vgg16_weights V]

ROOM_DIR holds the reference's preprocessed scenes (<room>/boxes.npz: jids, class_labels, translations, sizes,
angles, floor_plan_vertices / faces / centroid).  Each scene is written to OUT/<room>/rendered_scene_256.png
(rendered_scene_notexture_256.png with --no_texture), the layout the metric scripts read.  Models are matched by jid
and placed by the size-ratio rule the generated scenes use (scale = size / raw_half); the reference's own real renders
scale by the dataset's furniture.scale instead.

With --fid / --ipr nothing is written: the real scenes and the generated ones (GEN_DIR/scene_*.npz from
generate_diffusion.py with --render_top2down's retrieval, holding `model_index`) are rendered on the device and
scored without leaving it.  The shading is this project's, not simple-3dviz's: native renders compare only with
native renders, never with images the reference rendered.
"""
import argparse
import glob
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from diffuscene_b200 import render as R  # noqa: E402

NOTE = ("Native renders use this project's shading: their FID / KID / precision-recall compare only with native "
        "renders of the real scenes (this script), never with the reference's simple-3dviz images.")


def load_rooms(room_dir):
    rooms = sorted(d for d in os.listdir(room_dir) if os.path.isfile(os.path.join(room_dir, d, "boxes.npz")))
    if not rooms:
        raise SystemExit("no <room>/boxes.npz under %s" % room_dir)
    return rooms, [dict(np.load(os.path.join(room_dir, d, "boxes.npz"), allow_pickle=True)) for d in rooms]


def stack(scenes, key, width, fill, dtype):
    """[B, N, width] (or [B, N] for width 0) of per-scene arrays padded with `fill`."""
    N = max(1, max(len(s[key]) for s in scenes))
    out = np.full((len(scenes), N) + ((width,) if width else ()), fill, dtype)
    for b, s in enumerate(scenes):
        v = np.asarray(s[key], dtype)
        out[b, :len(v)] = v.reshape((len(v),) + ((width,) if width else ()))
    return out


def render_batch(cat, scenes, args, palette, floor_tex=None, seed=0):
    """uint8 [B, 256, 256, 3] device renders of scene dicts with translations / sizes / angles / class_index /
    model_index and optional floor_plan_* arrays."""
    floors = None
    if not args.without_floor:
        floors = R.floor_triangles([(s["floor_plan_vertices"] - s["floor_plan_centroid"], s["floor_plan_faces"])
                                    if "floor_plan_vertices" in s else None for s in scenes])
    fti = None
    if floor_tex is not None and floors is not None:
        fti = R.choose_floor_textures(len(scenes), len(floor_tex), seed)
    return R.render_scenes(cat, stack(scenes, "translations", 3, 0, np.float32), stack(scenes, "sizes", 3, 0, np.float32),
                           stack(scenes, "angles", 0, 0, np.float32), stack(scenes, "model_index", 0, -1, np.int64),
                           stack(scenes, "class_index", 0, 0, np.int64), floors=floors, no_texture=args.no_texture,
                           white_background=args.without_floor, palette=palette, floor_textures=floor_tex,
                           floor_texture_index=fti)


def real_scene(cat, s):
    out = {k: s[k] for k in ("translations", "sizes", "angles", "floor_plan_vertices", "floor_plan_faces",
                             "floor_plan_centroid") if k in s}
    out["class_index"] = np.asarray(s["class_labels"]).argmax(-1)
    out["model_index"] = cat.index_of(s["jids"])
    missing = int((out["model_index"] < 0).sum())
    if missing:
        print("WARNING: %d jids are not in the mesh catalogue; those objects are not drawn" % missing)
    return out


def render_all(cat, scenes, args, palette, floor_tex):
    out = []
    for b0 in range(0, len(scenes), args.batch_size):
        out.append(render_batch(cat, scenes[b0:b0 + args.batch_size], args, palette, floor_tex, args.seed + b0))
    return torch.cat(out)


def main(argv=None):
    p = argparse.ArgumentParser(description="Render real scenes top-down on the device. " + NOTE)
    p.add_argument("room_dir", help="directory of <room>/boxes.npz (the reference's preprocessed scenes)")
    p.add_argument("output_directory", nargs="?", default=None, help="where to write <room>/rendered_scene_256.png")
    p.add_argument("--mesh_catalogue", required=True, help="mesh_catalogue.npz (scripts/pack_mesh_catalogue.py)")
    p.add_argument("--no_texture", action="store_true", help="flat per-class colours (seaborn 'hls' palette)")
    p.add_argument("--without_floor", action="store_true", help="no floor, white background")
    p.add_argument("--floor_textures", default=None, help="folder of floor textures (default: a white floor)")
    p.add_argument("--seed", type=int, default=0, help="seed of the floor-texture choice")
    p.add_argument("--batch_size", type=int, default=512, help="scenes per render call")
    p.add_argument("--generated", default=None, help="scene_*.npz of generate_diffusion.py --render_top2down")
    p.add_argument("--fid", action="store_true", help="print FID and KID of --generated against the real scenes")
    p.add_argument("--ipr", action="store_true", help="print improved precision and recall likewise")
    p.add_argument("--inception_weights", default=None, help="pytorch-fid Inception state dict")
    p.add_argument("--vgg16_weights", default=None, help="torchvision vgg16 state dict")
    p.add_argument("--precision", choices=("fp32", "bf16"), default="fp32", help="feature-extractor precision")
    a = p.parse_args(argv)
    if not torch.cuda.is_available():
        raise RuntimeError("render_scenes.py needs a CUDA device; there is no CPU path")
    metrics = a.fid or a.ipr
    if metrics and not a.generated:
        p.error("--fid / --ipr need --generated")
    if not metrics and not a.output_directory:
        p.error("the output directory is required unless --fid / --ipr is given")
    cat = R.MeshCatalog(a.mesh_catalogue)
    rooms, raw = load_rooms(a.room_dir)
    palette = R.hls_palette(np.asarray(raw[0]["class_labels"]).shape[1] - 2)
    floor_tex = R.load_floor_textures(a.floor_textures) if a.floor_textures else None
    real = render_all(cat, [real_scene(cat, s) for s in raw], a, palette, floor_tex)
    if not metrics:
        from PIL import Image
        name = "rendered_scene_notexture_256.png" if a.no_texture else "rendered_scene_256.png"
        host = real.cpu().numpy()
        for room, img in zip(rooms, host):
            os.makedirs(os.path.join(a.output_directory, room), exist_ok=True)
            Image.fromarray(img).save(os.path.join(a.output_directory, room, name))
        print("rendered %d scenes into %s" % (len(rooms), a.output_directory))
        return
    gen = []
    for f in sorted(glob.glob(os.path.join(a.generated, "scene_*.npz"))):
        s = dict(np.load(f))
        gen.append({"translations": s["translations"][0], "sizes": s["sizes"][0], "angles": s["angles"][0],
                    "class_index": s["class_index"], "model_index": s["model_index"]})
    fake = render_all(cat, gen, a, palette, floor_tex)
    from diffuscene_b200 import fid as F, ipr as I
    inc = F.InceptionFeatures(F.find_weights(a.inception_weights), precision=a.precision) if a.fid else None
    vgg = I.VGG16Features(I.find_weights(a.vgg16_weights), precision=a.precision) if a.ipr else None
    for k, v in R.evaluate_renders(real, fake, inception=inc, vgg16=vgg).items():
        print("%s: %r" % (k, v))


if __name__ == "__main__":
    main()
