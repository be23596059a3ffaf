"""The real renderings of a splits CSV, in CachedThreedFront order, shared by the image-space evaluation scripts
(scripts/improved_precision_recall.py, scripts/compute_fid_scores.py)."""
from __future__ import annotations

import csv
import os
from typing import List, Sequence

RENDER_NAMES = ("rendered_scene_256.png", "rendered_scene_256_no_lamps.png", "rendered_scene_notexture_256.png")


def real_renders(base_dir: str, splits_csv: str, splits: Sequence[str] = ("train", "val")) -> List[str]:
    """CachedThreedFront's renders of the scenes of `splits`: directories `<x>_<scene id>` sorted, one file name
    chosen from the first directory."""
    with open(splits_csv) as f:
        ids = {r[0] for r in csv.reader(f) if len(r) > 1 and r[1] in splits}
    tags = sorted(d for d in os.listdir(base_dir) if len(d.split("_")) > 1 and d.split("_")[1] in ids)
    if not tags:
        raise SystemExit("no scene of %s in %s" % (splits_csv, base_dir))
    name = next((n for n in RENDER_NAMES[:2] if os.path.isfile(os.path.join(base_dir, tags[0], n))), RENDER_NAMES[2])
    print("rendered_scene is :", name)
    return sorted(os.path.join(base_dir, t, name) for t in tags)
