"""FID and KID of rendered scenes (reference scripts/compute_fid_scores.py, clean-fid's `clean` mode), native.

Features are the 2048-d pool3 output of the FID Inception-v3, extracted by the library's own kernels
(`InceptionFeatures`, ds_inception_*) from images resized as clean-fid does (`clean_resize`).  The feature mean and
covariance are fp64 on the device (ds_feature_stats); the trace term of the Frechet distance runs on the host in fp64
through two symmetric eigen-decompositions (`frechet_distance`); the KID subset terms run in fp64 on the device
(ds_kid_terms) over subsets drawn with the global `np.random` in clean-fid's order.

The Inception weights are never downloaded: pass pytorch-fid's state dict (torchvision key names) as a file, dict or
module, or put `pt_inception-2015-12-05-6726825d.pth` under `$TORCH_HOME/hub/checkpoints`.
"""
from __future__ import annotations

import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor
from glob import glob
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import capi

INCEPTION_WEIGHTS = "pt_inception-2015-12-05-6726825d.pth"      # pytorch-fid's FID Inception state dict
IMAGE_SIZE = 299
FEATURES = 2048                                                  # DS_INCEPTION_FEATURES
IMAGE_EXTENSIONS = ("bmp", "jpg", "jpeg", "pgm", "png", "ppm", "tif", "tiff", "webp")


def default_weights_path() -> str:
    """$TORCH_HOME/hub/checkpoints (torch.hub.get_dir(), no network)."""
    return os.path.join(torch.hub.get_dir(), "checkpoints", INCEPTION_WEIGHTS)


def find_weights(path: Optional[str] = None) -> str:
    """The Inception state-dict file to use: `path` if given, else the torch hub cache location.  Raises
    FileNotFoundError naming where to put the file; nothing is downloaded."""
    cand = path if path is not None else default_weights_path()
    if not os.path.isfile(cand):
        raise FileNotFoundError(
            "FID Inception weights not found at %s. Put pytorch-fid's %s there (or under $TORCH_HOME/hub/checkpoints) "
            "or pass its path explicitly; it is never downloaded." % (cand, INCEPTION_WEIGHTS))
    return cand


# ---- images -----------------------------------------------------------------------------------------------------

def clean_resize(image) -> np.ndarray:
    """clean-fid's `clean` preprocessing of one image (a path or a PIL image): RGB, then each channel resized alone as a
    float32 'F' image to 299 x 299 with PIL's bicubic filter and clipped to [0, 255] -> float32 [3, 299, 299]."""
    from PIL import Image
    if isinstance(image, (str, os.PathLike)):
        with Image.open(image) as im:
            arr = np.asarray(im.convert("RGB"), dtype=np.uint8)
    else:
        arr = np.asarray(image.convert("RGB"), dtype=np.uint8)
    chans = []
    for c in range(3):
        ch = Image.fromarray(arr[:, :, c].astype(np.float32), mode="F")
        ch = ch.resize((IMAGE_SIZE, IMAGE_SIZE), resample=Image.BICUBIC)
        chans.append(np.asarray(ch).clip(0, 255))
    return np.stack(chans, 0).astype(np.float32)


def image_files(root: str) -> List[str]:
    """clean-fid's folder listing: every file with an image extension under `root`, recursively, sorted."""
    return sorted(f for ext in IMAGE_EXTENSIONS for f in glob(os.path.join(root, "**", "*." + ext), recursive=True))


def _files(src: Union[str, Sequence[str]]) -> List[str]:
    if isinstance(src, (str, os.PathLike)):
        if not os.path.isdir(src):
            raise FileNotFoundError("%s is not a directory" % src)
        return image_files(str(src))
    out: List[str] = []
    for s in src:
        out.extend(image_files(s) if os.path.isdir(s) else [s])
    return out


# ---- features ---------------------------------------------------------------------------------------------------

class InceptionFeatures:
    """pool3 features of the FID Inception-v3 on the device.

    precision "fp32" (default): im2col + exact SIMT GEMMs, the detector's fp32 features up to summation order;
    "bf16": wgmma implicit-GEMM convolutions, an opt-in for throughput.  `state_dict_or_path` is pytorch-fid's
    Inception state dict (torchvision `Inception3` key names), a file holding one, or the module itself.
    Call with fp32 [B, 3, 299, 299] in [0, 255] (any device, already clean-resized); returns fp32 [B, 2048] on the
    device."""

    def __init__(self, state_dict_or_path: Union[str, dict, torch.nn.Module], precision: str = "fp32",
                 capacity: Optional[int] = None, device: int = 0):
        if precision not in ("bf16", "fp32"):
            raise ValueError("precision must be 'bf16' or 'fp32', not %r" % (precision,))
        sd = state_dict_or_path
        if isinstance(sd, (str, os.PathLike)):
            sd = torch.load(sd, map_location="cpu", weights_only=True)
        elif isinstance(sd, torch.nn.Module):
            sd = sd.state_dict()
        if not isinstance(sd, dict):
            raise TypeError("Inception weights must be a state dict, a state-dict file or a module, not %s"
                            % type(state_dict_or_path).__name__)
        if not torch.cuda.is_available():
            raise RuntimeError("InceptionFeatures needs a CUDA device: diffuscene_b200 has no CPU fallback")
        self.lib = capi.load()
        self.device = torch.device("cuda", device)
        cfg = capi.DsInceptionConfig()
        cfg.precision = capi.DS_PREC_BF16 if precision == "bf16" else capi.DS_PREC_FP32
        cfg.capacity = capacity or (64 if precision == "bf16" else 8)
        cfg.device = device
        self.capacity = cfg.capacity
        self.precision = precision
        self._h = C.c_void_p()
        capi.check(self.lib.ds_inception_create(C.byref(cfg), C.byref(self._h)))
        names = expected_weights(self.lib, self._h)
        missing = [n for n, _ in names if n not in sd]
        if missing:
            self.close()
            raise KeyError("Inception state dict lacks %s" % ", ".join(missing))
        for n, numel in names:
            if sd[n].numel() != numel:
                self.close()
                raise ValueError("%s has %d elements, expected %d" % (n, sd[n].numel(), numel))
        flat = torch.cat([sd[n].reshape(-1).float() for n, _ in names]).to(self.device)
        stream = torch.cuda.current_stream(self.device)
        capi.check(self.lib.ds_inception_set_weights(self._h, C.c_void_p(flat.data_ptr()), flat.numel(),
                                                     C.c_void_p(stream.cuda_stream)))
        stream.synchronize()

    def __call__(self, images: torch.Tensor) -> torch.Tensor:
        if images.dim() != 4 or images.shape[1] != 3:
            raise ValueError("images must be [B, 3, 299, 299], got %s" % (tuple(images.shape),))
        x = images.to(self.device, torch.float32).contiguous()
        out = torch.empty(x.shape[0], FEATURES, device=self.device, dtype=torch.float32)
        if x.shape[0] == 0:
            return out
        stream = torch.cuda.current_stream(self.device)
        capi.check(self.lib.ds_inception_features(self._h, C.c_void_p(x.data_ptr()), x.shape[0], x.shape[2],
                                                  x.shape[3], C.c_void_p(out.data_ptr()),
                                                  C.c_void_p(stream.cuda_stream)))
        return out

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self.lib.ds_inception_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def expected_weights(lib=None, h=None) -> List[tuple]:
    """(name, numel) of the flat parameter buffer, torchvision state-dict order (needs a device for the handle)."""
    lib = lib or capi.load()
    own = h is None
    if own:
        cfg = capi.DsInceptionConfig()
        cfg.precision, cfg.capacity = capi.DS_PREC_FP32, 1
        h = C.c_void_p()
        capi.check(lib.ds_inception_create(C.byref(cfg), C.byref(h)))
    try:
        out = []
        for i in range(capi.check(lib.ds_inception_expected_weight_count(h))):
            name, numel = C.c_char_p(), C.c_int64()
            capi.check(lib.ds_inception_expected_weight(h, i, C.byref(name), C.byref(numel)))
            out.append((name.value.decode(), numel.value))
        return out
    finally:
        if own:
            lib.ds_inception_destroy(h)


def folder_features(files: Union[str, Sequence[str]], model: InceptionFeatures, batch_size: int = 32,
                    num_workers: int = 8) -> np.ndarray:
    """float32 [N, 2048] features of image files (or of every image under a directory), decoded and clean-resized on
    a thread pool (PIL releases the GIL), in file order."""
    files = _files(files)
    out = np.empty((len(files), FEATURES), np.float32)
    with ThreadPoolExecutor(max(1, num_workers)) as pool:
        for b0 in range(0, len(files), batch_size):
            imgs = np.stack(list(pool.map(clean_resize, files[b0:b0 + batch_size])))
            out[b0:b0 + len(imgs)] = model(torch.from_numpy(imgs)).cpu().numpy()
    return out


# ---- statistics and distances -----------------------------------------------------------------------------------

def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev32(x) -> torch.Tensor:
    t = x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x, np.float32))
    return t.to("cuda", torch.float32).contiguous()


def feature_stats(feats) -> Tuple[np.ndarray, np.ndarray]:
    """(mu [d], sigma [d, d]) in fp64 of features [n, d], n >= 2: np.mean and np.cov(rowvar=False) of the
    float64-promoted features, computed on the device."""
    f = _dev32(feats)
    if f.dim() != 2 or f.shape[0] < 2:
        raise ValueError("features must be [n >= 2, d], got %s" % (tuple(f.shape),))
    n, d = f.shape
    mu = torch.empty(d, device=f.device, dtype=torch.float64)
    sigma = torch.empty(d, d, device=f.device, dtype=torch.float64)
    capi.check(capi.load().ds_feature_stats(C.c_void_p(f.data_ptr()), n, d, C.c_void_p(mu.data_ptr()),
                                            C.c_void_p(sigma.data_ptr()), _stream()))
    return mu.cpu().numpy(), sigma.cpu().numpy()


def trace_sqrt_product(sigma1, sigma2) -> float:
    """tr sqrtm(sigma1 sigma2) of two covariance matrices: with sigma1 = V diag(w) V^T and S = V diag(sqrt(max(w, 0)))
    V^T, sigma1 sigma2 is similar to the symmetric S sigma2 S, so the trace is the sum of sqrt(max(lambda, 0)) over
    its eigenvalues.  fp64; never complex or non-finite for finite input."""
    from scipy import linalg
    w, v = linalg.eigh(np.asarray(sigma1, np.float64))
    s = (v * np.sqrt(np.maximum(w, 0.0))) @ v.T
    m = s @ np.asarray(sigma2, np.float64) @ s
    lam = linalg.eigvalsh((m + m.T) / 2)
    return float(np.sqrt(np.maximum(lam, 0.0)).sum())


def frechet_distance(mu1, sigma1, mu2, sigma2) -> float:
    """|mu1 - mu2|^2 + tr sigma1 + tr sigma2 - 2 tr sqrtm(sigma1 sigma2), fp64 on the host, the trace term from
    `trace_sqrt_product`.  Raises ValueError for non-finite statistics."""
    mu1, mu2 = np.atleast_1d(np.asarray(mu1, np.float64)), np.atleast_1d(np.asarray(mu2, np.float64))
    sigma1, sigma2 = np.atleast_2d(np.asarray(sigma1, np.float64)), np.atleast_2d(np.asarray(sigma2, np.float64))
    if mu1.shape != mu2.shape or sigma1.shape != sigma2.shape or sigma1.shape != (mu1.size, mu1.size):
        raise ValueError("mean / covariance shapes differ: %s %s %s %s" % (mu1.shape, sigma1.shape, mu2.shape,
                                                                         sigma2.shape))
    for a in (mu1, sigma1, mu2, sigma2):
        if not np.isfinite(a).all():
            raise ValueError("feature statistics are not finite")
    diff = mu1 - mu2
    return float(diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2.0 * trace_sqrt_product(sigma1, sigma2))


def kid_subsets(n_real: int, n_fake: int, num_subsets: int = 100, max_subset_size: int = 1000):
    """The subsets clean-fid's kernel_distance draws from the global np.random: per subset, the fake rows first, then
    the real rows, each np.random.choice(n, m, replace=False) with m = min(n_real, n_fake, max_subset_size)."""
    m = min(n_real, n_fake, max_subset_size)
    idx_fake = np.empty((num_subsets, m), np.int64)
    idx_real = np.empty((num_subsets, m), np.int64)
    for s in range(num_subsets):
        idx_fake[s] = np.random.choice(n_fake, m, replace=False)
        idx_real[s] = np.random.choice(n_real, m, replace=False)
    return idx_fake, idx_real


def kid_terms(feats_real, feats_fake, idx_fake, idx_real) -> np.ndarray:
    """fp64 per-subset terms t_s = (sum a - sum diag a) / (m - 1) - 2 sum b / m (ds_kid_terms)."""
    r, f = _dev32(feats_real), _dev32(feats_fake)
    if r.dim() != 2 or f.dim() != 2 or r.shape[1] != f.shape[1]:
        raise ValueError("features must be [n, d] with the same d, got %s and %s" % (tuple(r.shape), tuple(f.shape)))
    ix = torch.as_tensor(np.asarray(idx_fake, np.int64)).cuda().contiguous()
    iy = torch.as_tensor(np.asarray(idx_real, np.int64)).cuda().contiguous()
    if ix.dim() != 2 or ix.shape != iy.shape:
        raise ValueError("index arrays must be [subsets, m] of one shape")
    subsets, m = ix.shape
    terms = torch.empty(subsets, device="cuda", dtype=torch.float64)
    capi.check(capi.load().ds_kid_terms(C.c_void_p(r.data_ptr()), r.shape[0], C.c_void_p(f.data_ptr()), f.shape[0],
                                        r.shape[1], C.c_void_p(ix.data_ptr()), C.c_void_p(iy.data_ptr()), subsets, m,
                                        C.c_void_p(terms.data_ptr()), _stream()))
    return terms.cpu().numpy()


def kernel_distance(feats1, feats2, num_subsets: int = 100, max_subset_size: int = 1000) -> float:
    """clean-fid's kernel_distance(feats1 = real, feats2 = fake): the mean over subsets of the unbiased MMD^2 with the
    cubic polynomial kernel (x.y / d + 1)^3, the subsets drawn as `kid_subsets`, the terms in fp64 on the device."""
    feats1, feats2 = np.asarray(feats1, np.float32), np.asarray(feats2, np.float32)
    if not (np.isfinite(feats1).all() and np.isfinite(feats2).all()):
        raise ValueError("features are not finite")
    idx_fake, idx_real = kid_subsets(len(feats1), len(feats2), num_subsets, max_subset_size)
    m = idx_fake.shape[1]
    return float(kid_terms(feats1, feats2, idx_fake, idx_real).sum() / num_subsets / m)


def fid_from_features(feats_real, feats_fake) -> float:
    for f in (feats_real, feats_fake):
        if not np.isfinite(np.asarray(f)).all():
            raise ValueError("features are not finite")
    mu1, s1 = feature_stats(feats_real)
    mu2, s2 = feature_stats(feats_fake)
    return frechet_distance(mu1, s1, mu2, s2)


def _model(model, weights, precision):
    if model is not None:
        return model
    return InceptionFeatures(find_weights(weights), precision=precision)


def compute_fid(real, fake, model: Optional[InceptionFeatures] = None, weights: Optional[str] = None,
                precision: str = "fp32", batch_size: int = 32, num_workers: int = 8) -> float:
    """FID between two image sets, each a directory or a list of files / directories (clean-fid's compute_fid in
    `clean` mode)."""
    model = _model(model, weights, precision)
    return fid_from_features(folder_features(real, model, batch_size, num_workers),
                             folder_features(fake, model, batch_size, num_workers))


def compute_kid(real, fake, model: Optional[InceptionFeatures] = None, weights: Optional[str] = None,
                precision: str = "fp32", batch_size: int = 32, num_workers: int = 8, num_subsets: int = 100,
                max_subset_size: int = 1000) -> float:
    """KID between two image sets (clean-fid's compute_kid in `clean` mode); seed np.random for reproducible subsets."""
    model = _model(model, weights, precision)
    return kernel_distance(folder_features(real, model, batch_size, num_workers),
                           folder_features(fake, model, batch_size, num_workers), num_subsets, max_subset_size)
