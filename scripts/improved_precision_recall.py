#!/usr/bin/env python3
"""Improved precision and recall of synthesized top-down renderings against real ones, natively (the reference's
scripts/improved_precision_recall.py command line).

    python scripts/improved_precision_recall.py REAL_DIR FAKE_DIR [SPLITS_CSV] --vgg16_weights vgg16-397923af.pth

Without SPLITS_CSV the real set is every *.jpg / *.png under REAL_DIR; with it, `<scene>/rendered_scene_256.png`
(or the reference's two fallback names) of every train / val scene of the CSV.  Both lists are sorted, shuffled with
random.Random(100) and cut to --num_samples, as the reference does with its temporary copies (none are made here).
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from diffuscene_b200 import ipr as I  # noqa: E402
from diffuscene_b200.renders import real_renders  # noqa: E402


def toy():
    offset = 2
    real = np.random.rand(10).reshape(-1, 1)
    fake = np.random.rand(10).reshape(-1, 1) + offset
    real[0], fake[0] = offset, 1
    print("real:", real)
    print("fake:", fake)
    m_real = I.Manifold(real, I.manifold_radii(real))
    m_fake = I.Manifold(fake, I.manifold_radii(fake))
    print("precision:", I.compute_metric(m_real, fake))
    print("recall:", I.compute_metric(m_fake, real))


def main(argv=None):
    p = argparse.ArgumentParser(formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument("path_to_real_renderings", nargs="?", help="Folder of the real renderings")
    p.add_argument("path_to_synthesized_renderings", nargs="?", help="Folder of the synthesized renderings")
    p.add_argument("path_to_annotations", nargs="?", default=None, help="Optional train/val/test splits CSV")
    p.add_argument("--batch_size", type=int, default=50, help="Images per feature-extraction batch")
    p.add_argument("--k", type=int, default=3, help="k of the k-NN radii")
    p.add_argument("--num_samples", type=int, default=5000, help="Images of each set to use")
    p.add_argument("--toy", action="store_true")
    p.add_argument("--fname_precalc", type=str, default="", help="Save the real manifold here and stop")
    p.add_argument("--vgg16_weights", type=str, default=None,
                   help="torchvision vgg16 state dict (default: $TORCH_HOME/hub/checkpoints/%s)" % I.VGG16_WEIGHTS)
    p.add_argument("--precision", choices=("fp32", "bf16"), default="fp32",
                   help="Feature-extractor precision: fp32 reproduces the reference's features; bf16 is faster, and its "
                        "features (about 0.7%% relative L2 from fp64) can move ball memberships near their boundary")
    a = p.parse_args(argv)
    if a.toy:
        print("running toy example...")
        toy()
        return
    if not a.path_to_real_renderings or not a.path_to_synthesized_renderings:
        p.error("the real and synthesized renderings are required")

    if a.path_to_annotations:
        real = real_renders(a.path_to_real_renderings, a.path_to_annotations)
    elif a.path_to_real_renderings.endswith(".npz"):
        real = a.path_to_real_renderings
    else:
        real = sorted(I.image_files(a.path_to_real_renderings))
    fake = sorted(os.path.join(a.path_to_synthesized_renderings, f)
                  for f in os.listdir(a.path_to_synthesized_renderings) if f.endswith(".png"))
    print("number of real images :", 1 if isinstance(real, str) else len(real))
    print("number of synthesized images :", len(fake))

    ipr = I.IPR(a.batch_size, a.k, a.num_samples, model=I.find_weights(a.vgg16_weights), precision=a.precision)
    ipr.compute_manifold_ref(real if isinstance(real, str) else I.subsample(real, a.num_samples))
    if a.fname_precalc:
        ipr.save_ref(a.fname_precalc)
        print("path_fake (%s) is ignored for precalc" % a.path_to_synthesized_renderings)
        return
    precision, recall = ipr.precision_and_recall(I.subsample(fake, a.num_samples))
    print("precision:", precision)
    print("recall:", recall)
    print("fscore:", (precision * recall) / (precision + recall))


if __name__ == "__main__":
    main()
