#!/usr/bin/env python3
"""FID and KID between the real and the synthesized top-down renderings, natively (the reference's
scripts/compute_fid_scores.py command line, clean-fid's `clean` mode).

    python scripts/compute_fid_scores.py REAL_DIR FAKE_DIR SPLITS_CSV [--compare_all] \
        --inception_weights pt_inception-2015-12-05-6726825d.pth

The real set is `<scene>/rendered_scene_256.png` (or the reference's two fallback names) of every train / val scene of
the CSV (train / val / test with --compare_all), in CachedThreedFront order; the fake set is every *.png of FAKE_DIR in
os.listdir order.  Features are extracted once for both metrics and no temporary copies are made.  Seed: KID draws
its subsets from the global np.random, unseeded as in the reference.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from diffuscene_b200 import fid as F  # noqa: E402
from diffuscene_b200.renders import real_renders  # noqa: E402


def fake_renders(fake_dir):
    return [os.path.join(fake_dir, f) for f in os.listdir(fake_dir) if f.endswith(".png")]


def main(argv=None):
    p = argparse.ArgumentParser(description="Compute the FID scores between the real and the synthetic images",
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument("path_to_real_renderings", help="Path to the folder containing the real renderings")
    p.add_argument("path_to_synthesized_renderings", help="Path to the folder containing the synthesized")
    p.add_argument("path_to_annotations", help="Path to the train/val/test splits CSV")
    p.add_argument("--compare_all", action="store_true", help="Include the test scenes in the real set")
    p.add_argument("--inception_weights", type=str, default=None,
                   help="pytorch-fid Inception state dict (default: $TORCH_HOME/hub/checkpoints/%s)" % F.INCEPTION_WEIGHTS)
    p.add_argument("--precision", choices=("fp32", "bf16"), default="fp32",
                   help="Feature-extractor precision: fp32 reproduces the detector's features; bf16 is faster")
    p.add_argument("--batch_size", type=int, default=32, help="Images per feature-extraction batch")
    p.add_argument("--num_workers", type=int, default=8, help="Host threads decoding and resizing images")
    a = p.parse_args(argv)

    splits = ("train", "val", "test") if a.compare_all else ("train", "val")
    real = real_renders(a.path_to_real_renderings, a.path_to_annotations, splits)
    print("number of synthesized images :", len(real))
    fake = fake_renders(a.path_to_synthesized_renderings)
    print("number of synthesized images :", len(fake))

    model = F.InceptionFeatures(F.find_weights(a.inception_weights), precision=a.precision)
    feats_real = F.folder_features(real, model, a.batch_size, a.num_workers)
    feats_fake = F.folder_features(fake, model, a.batch_size, a.num_workers)
    print("fid score:", F.fid_from_features(feats_real, feats_fake))
    print("kid score:", F.kernel_distance(feats_real, feats_fake))


if __name__ == "__main__":
    main()
