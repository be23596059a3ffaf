"""Writes tests/golden/ipr_features.npz and tests/golden/ipr_metrics.npz from the UNMODIFIED reference module
scripts/improved_precision_recall.py (its dataset imports stubbed) and torchvision's vgg16.  Needs a reference
checkout ($DS_REFERENCE_ROOT) and torchvision; the tests only read the .npz files.

    python tests/golden/make_golden_ipr.py
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from tests.cases_ipr import clustered, he_state_dict, normalise, render_like  # noqa: E402

REF = os.environ.get("DS_REFERENCE_ROOT", "/root/reference")


def reference_module():
    for name, attrs in (("scene_synthesis", {}), ("scene_synthesis.datasets", {}),
                        ("scene_synthesis.datasets.splits_builder", {"CSVSplitsBuilder": object}),
                        ("scene_synthesis.datasets.threed_front", {"CachedThreedFront": object})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
    spec = importlib.util.spec_from_file_location("ref_ipr", os.path.join(REF, "scripts", "improved_precision_recall.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    import torchvision
    ref = reference_module()
    torch.manual_seed(0)
    vgg = torchvision.models.vgg16()
    vgg.load_state_dict(he_state_dict(seed=1))
    vgg.eval()
    img = render_like(2, 224, seed=11)
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda t, *a, **kw: t          # the reference moves each batch with .cuda(); stay on the host
    try:
        with torch.no_grad():
            ipr = ref.IPR(batch_size=50, k=3, num_samples=10, model=vgg)
            feats = ipr.extract_features(normalise(img))
    finally:
        torch.Tensor.cuda = cuda
    np.savez_compressed(os.path.join(HERE, "ipr_features.npz"), images_u8=img, features=feats)

    k = 3
    real = clustered(300, 96, seed=21, centre_seed=0)
    fake = clustered(240, 96, clusters=10, seed=22, spread=0.35, centre_seed=0)
    r_real = ref.distances2radii(ref.compute_pairwise_distances(real), k=k)
    r_fake = ref.distances2radii(ref.compute_pairwise_distances(fake), k=k)
    m_real, m_fake = ref.Manifold(real, r_real), ref.Manifold(fake, r_fake)
    d_rf = ref.compute_pairwise_distances(real, fake)
    d_fr = ref.compute_pairwise_distances(fake, real)
    np.savez_compressed(
        os.path.join(HERE, "ipr_metrics.npz"), real=real, fake=fake, k=k, radii_real=r_real, radii_fake=r_fake,
        precision_flags=(d_rf < r_real[:, None]).any(axis=0), recall_flags=(d_fr < r_fake[:, None]).any(axis=0),
        precision=ref.compute_metric(m_real, fake), recall=ref.compute_metric(m_fake, real),
        realism=np.array([ref.realism(m_real, fake[j]) for j in range(20)]))


if __name__ == "__main__":
    main()
