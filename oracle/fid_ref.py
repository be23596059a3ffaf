"""Restatements of clean-fid's `clean` mode, for tests: the image resize, the Frechet distance through
scipy.linalg.sqrtm with its two fallbacks, and the KID float32 expression (clean-fid 0.1.x as restated; see DESIGN.md
for what could not be checked against its source)."""
import numpy as np
from PIL import Image
from scipy import linalg


def clean_resize_ref(path):
    img = np.array(Image.open(path).convert("RGB")).astype(np.uint8)
    out = []
    for i in range(3):
        ch = Image.fromarray(img[:, :, i].astype(np.float32), mode="F").resize((299, 299), resample=Image.BICUBIC)
        out.append(np.asarray(ch).clip(0, 255).reshape(299, 299, 1))
    return np.concatenate(out, axis=2).transpose(2, 0, 1).astype(np.float32)


def frechet_distance_sqrtm(mu1, sigma1, mu2, sigma2, eps=1e-6):
    mu1, mu2 = np.atleast_1d(mu1), np.atleast_1d(mu2)
    sigma1, sigma2 = np.atleast_2d(sigma1), np.atleast_2d(sigma2)
    diff = mu1 - mu2
    covmean = linalg.sqrtm(sigma1.dot(sigma2))
    if not np.isfinite(covmean).all():
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = linalg.sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            raise ValueError("Imaginary component {}".format(np.max(np.abs(covmean.imag))))
        covmean = covmean.real
    return diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean)


def kid_terms_f32(feats1, feats2, idx_fake, idx_real):
    """Per-subset terms of clean-fid's kernel_distance in its float32 arithmetic (feats1 = real, feats2 = fake)."""
    n = feats1.shape[1]
    m = idx_fake.shape[1]
    out = []
    for s in range(idx_fake.shape[0]):
        x = feats2[idx_fake[s]]
        y = feats1[idx_real[s]]
        a = (x @ x.T / n + 1) ** 3 + (y @ y.T / n + 1) ** 3
        b = (x @ y.T / n + 1) ** 3
        out.append((a.sum() - np.diag(a).sum()) / (m - 1) - b.sum() * 2 / m)
    return np.asarray(out)


def kid_terms_f64(feats1, feats2, idx_fake, idx_real):
    return kid_terms_f32(np.asarray(feats1, np.float64), np.asarray(feats2, np.float64), idx_fake, idx_real)
