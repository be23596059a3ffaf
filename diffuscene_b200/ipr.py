"""Improved precision and recall of rendered scenes (reference scripts/improved_precision_recall.py), native.

Features are the fc2 output of torchvision's `vgg16` before its ReLU, extracted by the library's own kernels
(`VGG16Features`, ds_vgg_*); the k-NN manifold metrics run in fp64 on the device without an N x N matrix
(ds_manifold_radii / ds_manifold_cover).  The surface mirrors the reference: `IPR`, `Manifold`,
`PrecisionAndRecall`, `compute_pairwise_distances`, `distances2radii`, `compute_metric`, `realism`, and `.npz`
manifold files with the keys `feature` and `radii` that interchange with the reference's `save_ref`.

The VGG16 weights are never downloaded: pass a torchvision state-dict file or dict, or put
`vgg16-397923af.pth` under `$TORCH_HOME/hub/checkpoints`.
"""
from __future__ import annotations

import ctypes as C
import os
import random
from collections import namedtuple
from concurrent.futures import ThreadPoolExecutor
from glob import glob
from typing import List, Optional, Sequence, Union

import numpy as np
import torch

from . import capi

Manifold = namedtuple("Manifold", ["features", "radii"])
PrecisionAndRecall = namedtuple("PrecisionAndRecall", ["precision", "recall"])

VGG16_WEIGHTS = "vgg16-397923af.pth"          # torchvision's ImageNet checkpoint name
IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)
IMAGE_SIZE = 224
MAX_K = 16                                     # DS_MANIFOLD_MAX_K


def default_weights_path() -> str:
    """Where torchvision keeps the checkpoint: $TORCH_HOME/hub/checkpoints (torch.hub.get_dir(), no network)."""
    return os.path.join(torch.hub.get_dir(), "checkpoints", VGG16_WEIGHTS)


def find_weights(path: Optional[str] = None) -> str:
    """The VGG16 state-dict file to use: `path` if given, else the torchvision cache location.  Raises
    FileNotFoundError naming where to put the file; nothing is downloaded."""
    cand = path if path is not None else default_weights_path()
    if not os.path.isfile(cand):
        raise FileNotFoundError(
            "VGG16 weights not found at %s. Put torchvision's ImageNet checkpoint %s there (or under "
            "$TORCH_HOME/hub/checkpoints) or pass its path explicitly; it is never downloaded." % (cand, VGG16_WEIGHTS))
    return cand


# ---- features ---------------------------------------------------------------------------------------------------

class VGG16Features:
    """classifier[:4](features(x).view(-1, 25088)) of torchvision vgg16 on the device.

    precision "fp32" (default): im2col + exact SIMT GEMMs, the reference's fp32 features up to summation order;
    "bf16": wgmma implicit-GEMM convolutions (about 0.7 % relative L2 from fp64 on the tests' inputs), an opt-in for
    throughput whose features can move k-NN ball memberships near their boundary.  `state_dict_or_path` is a
    torchvision vgg16 state dict, a file holding one, or the vgg16 nn.Module itself.
    Call with a normalised fp32 tensor [B, 3, H, W] (any device); returns fp32 [B, 4096] on the device.  Inputs other
    than 224 x 224 are resized with F.interpolate's nearest pixel choice, as the reference's extract_features."""

    def __init__(self, state_dict_or_path: Union[str, dict, torch.nn.Module], precision: str = "fp32",
                 capacity: Optional[int] = None,
                 device: int = 0):
        if precision not in ("bf16", "fp32"):
            raise ValueError("precision must be 'bf16' or 'fp32', not %r" % (precision,))
        sd = state_dict_or_path
        if isinstance(sd, str):
            sd = torch.load(sd, map_location="cpu", weights_only=True)
        elif isinstance(sd, torch.nn.Module):
            sd = sd.state_dict()
        if not isinstance(sd, dict):
            raise TypeError("VGG16 weights must be a state dict, a state-dict file or a vgg16 module, not %s"
                            % type(state_dict_or_path).__name__)
        self.lib = capi.load()
        self.device = torch.device("cuda", device)
        cfg = capi.DsVggConfig()
        cfg.precision = capi.DS_PREC_BF16 if precision == "bf16" else capi.DS_PREC_FP32
        cfg.capacity = capacity or (64 if precision == "bf16" else 8)
        cfg.device = device
        self.capacity = cfg.capacity
        self.precision = precision
        self._h = C.c_void_p()
        capi.check(self.lib.ds_vgg_create(C.byref(cfg), C.byref(self._h)))
        names = expected_weights(self.lib, self._h)
        missing = [n for n, _ in names if n not in sd]
        if missing:
            self.close()
            raise KeyError("VGG16 state dict lacks %s" % ", ".join(missing))
        for n, numel in names:
            if sd[n].numel() != numel:
                self.close()
                raise ValueError("%s has %d elements, expected %d" % (n, sd[n].numel(), numel))
        flat = torch.cat([sd[n].reshape(-1).float() for n, _ in names]).to(self.device)
        stream = torch.cuda.current_stream(self.device)
        capi.check(self.lib.ds_vgg_set_weights(self._h, C.c_void_p(flat.data_ptr()), flat.numel(),
                                               C.c_void_p(stream.cuda_stream)))
        stream.synchronize()

    def __call__(self, images: torch.Tensor) -> torch.Tensor:
        if images.dim() != 4 or images.shape[1] != 3:
            raise ValueError("images must be [B, 3, H, W], got %s" % (tuple(images.shape),))
        x = images.to(self.device, torch.float32).contiguous()
        out = torch.empty(x.shape[0], 4096, device=self.device, dtype=torch.float32)
        if x.shape[0] == 0:
            return out
        stream = torch.cuda.current_stream(self.device)
        capi.check(self.lib.ds_vgg_features(self._h, C.c_void_p(x.data_ptr()), x.shape[0], x.shape[2], x.shape[3],
                                            C.c_void_p(out.data_ptr()), C.c_void_p(stream.cuda_stream)))
        return out

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self.lib.ds_vgg_destroy(self._h)
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
        cfg = capi.DsVggConfig()
        cfg.precision, cfg.capacity = capi.DS_PREC_FP32, 1
        h = C.c_void_p()
        capi.check(lib.ds_vgg_create(C.byref(cfg), C.byref(h)))
    try:
        out = []
        for i in range(capi.check(lib.ds_vgg_expected_weight_count(h))):
            name, numel = C.c_char_p(), C.c_int64()
            capi.check(lib.ds_vgg_expected_weight(h, i, C.byref(name), C.byref(numel)))
            out.append((name.value.decode(), numel.value))
        return out
    finally:
        if own:
            lib.ds_vgg_destroy(h)


def load_image(path: str) -> np.ndarray:
    """The reference's file transform: PIL RGB, Resize([224, 224]) (PIL bilinear), ToTensor, ImageNet Normalize,
    in the same fp32 operations -> [3, 224, 224]."""
    from PIL import Image
    with Image.open(path) as im:
        im = im.convert("RGB").resize((IMAGE_SIZE, IMAGE_SIZE), Image.BILINEAR)
        x = np.asarray(im, dtype=np.uint8).astype(np.float32) / np.float32(255)
    x = x.transpose(2, 0, 1)
    mean = np.asarray(IMAGENET_MEAN, np.float32)[:, None, None]
    std = np.asarray(IMAGENET_STD, np.float32)[:, None, None]
    return np.ascontiguousarray((x - mean) / std)


def image_files(root: str) -> List[str]:
    """The reference's ImageFolder listing: every *.jpg, then every *.png, recursively, in glob order."""
    return glob(os.path.join(root, "**", "*.jpg"), recursive=True) + glob(os.path.join(root, "**", "*.png"),
                                                                          recursive=True)


def subsample(files: Sequence[str], num_samples: int, seed: int = 100) -> List[str]:
    """The script's subsampling: random.Random(seed).shuffle, then the first num_samples (all when <= 0)."""
    files = list(files)
    random.Random(seed).shuffle(files)
    return files[:num_samples] if num_samples > 0 else files


# ---- manifold metrics -------------------------------------------------------------------------------------------

def _dev64(x) -> torch.Tensor:
    t = torch.as_tensor(np.asarray(x) if not isinstance(x, torch.Tensor) else x)
    if t.dim() == 1:
        t = t[:, None]
    return t.to("cuda", torch.float64).contiguous()


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _warn_clamped(clamped: torch.Tensor):
    n = int(clamped.item())
    if n:
        print("WARNING: %d negative diff_squares found and set to zero" % n)


def compute_pairwise_distances(X, Y=None) -> np.ndarray:
    """N x M fp64 distance matrix (small inputs and tests only; the metrics below never form it)."""
    lib = capi.load()
    x = _dev64(X)
    y = x if Y is None else _dev64(Y)
    if x.shape[1] != y.shape[1]:
        raise ValueError("feature sizes differ: %d and %d" % (x.shape[1], y.shape[1]))
    out = torch.empty(x.shape[0], y.shape[0], device="cuda", dtype=torch.float64)
    clamped = torch.zeros(1, device="cuda", dtype=torch.int64)
    capi.check(lib.ds_manifold_distances(_ptr(x), x.shape[0], _ptr(y), y.shape[0], x.shape[1], _ptr(out),
                                         _ptr(clamped), _stream()))
    _warn_clamped(clamped)
    return out.cpu().numpy()


def distances2radii(distances, k: int = 3) -> np.ndarray:
    """(k+1)-th smallest entry of each row of a given distance matrix (the ~0 self distance counted).

    This selects on a matrix the caller already holds, on the host.  The native path, which never forms the matrix,
    is manifold_radii(features, k) (ds_manifold_radii); IPR.compute_manifold uses it."""
    d = np.asarray(distances, dtype=np.float64)
    return np.partition(d, k, axis=1)[:, k].copy()


def manifold_radii(features, k: int = 3) -> np.ndarray:
    """distances2radii(compute_pairwise_distances(features), k) on the device, without the N x N matrix."""
    lib = capi.load()
    x = _dev64(features)
    radii = torch.empty(x.shape[0], device="cuda", dtype=torch.float64)
    clamped = torch.zeros(1, device="cuda", dtype=torch.int64)
    capi.check(lib.ds_manifold_radii(_ptr(x), x.shape[0], x.shape[1], int(k), _ptr(radii), _ptr(clamped), _stream()))
    _warn_clamped(clamped)
    return radii.cpu().numpy()


def manifold_cover(manifold_ref: Manifold, feats_subject, radii_subject=None, want_realism: bool = False):
    """One pass over reference x subject pairs -> (subject flags, reference flags or None, realism or None)."""
    lib = capi.load()
    ref, subj = _dev64(manifold_ref.features), _dev64(feats_subject)
    if ref.shape[1] != subj.shape[1]:
        raise ValueError("feature sizes differ: %d and %d" % (ref.shape[1], subj.shape[1]))
    r_ref = torch.as_tensor(np.asarray(manifold_ref.radii, dtype=np.float64)).cuda()
    r_subj = None if radii_subject is None else torch.as_tensor(np.asarray(radii_subject, np.float64)).cuda()
    if r_ref.numel() != ref.shape[0] or (r_subj is not None and r_subj.numel() != subj.shape[0]):
        raise ValueError("one radius per feature vector is required")
    s_cov = torch.empty(subj.shape[0], device="cuda", dtype=torch.uint8)
    r_cov = torch.empty(ref.shape[0], device="cuda", dtype=torch.uint8) if r_subj is not None else None
    real = torch.empty(subj.shape[0], device="cuda", dtype=torch.float64) if want_realism else None
    clamped = torch.zeros(1, device="cuda", dtype=torch.int64)
    capi.check(lib.ds_manifold_cover(_ptr(ref), _ptr(r_ref), ref.shape[0], _ptr(subj), _ptr(r_subj), subj.shape[0],
                                     ref.shape[1], _ptr(s_cov), _ptr(r_cov), _ptr(real), _ptr(clamped), _stream()))
    _warn_clamped(clamped)
    return (s_cov.cpu().numpy().astype(bool), None if r_cov is None else r_cov.cpu().numpy().astype(bool),
            None if real is None else real.cpu().numpy())


def compute_metric(manifold_ref: Manifold, feats_subject, desc: str = "") -> float:
    """Fraction of subjects inside some reference ball (strict <)."""
    flags, _, _ = manifold_cover(manifold_ref, feats_subject)
    return float(flags.mean())


def realism(manifold_real: Manifold, feat_subject):
    """max_i radius_i / (|real_i - f| + 1e-6): a float for one feature vector, an array for several."""
    f = np.asarray(feat_subject.cpu() if isinstance(feat_subject, torch.Tensor) else feat_subject)
    single = f.ndim == 1 or f.shape[0] == 1
    _, _, r = manifold_cover(manifold_real, f.reshape(-1, np.asarray(manifold_real.features).shape[1]),
                             want_realism=True)
    return float(r[0]) if single else r


def save_manifold(fname: str, manifold: Manifold):
    np.savez_compressed(fname, feature=manifold.features, radii=manifold.radii)


def load_manifold(fname: str) -> Manifold:
    with np.load(fname) as f:
        return Manifold(f["feature"], f["radii"])


# ---- the reference's IPR class ------------------------------------------------------------------------------------

class IPR:
    def __init__(self, batch_size: int = 50, k: int = 3, num_samples: int = 10000, model=None,
                 precision: str = "fp32", num_workers: int = 4):
        """model: a VGG16Features, a torchvision vgg16 module or state dict, a state-dict file, or None for the
        torchvision cache.  precision "fp32" reproduces the reference's features; "bf16" is a faster opt-in."""
        if not 1 <= k <= MAX_K:
            raise ValueError("k must be in [1, %d]" % MAX_K)
        self.manifold_ref = None
        self.batch_size = batch_size
        self.k = k
        self.num_samples = num_samples
        self.num_workers = num_workers
        self.vgg16 = model if isinstance(model, VGG16Features) else VGG16Features(
            find_weights() if model is None else model, precision=precision)

    def __call__(self, subject):
        return self.precision_and_recall(subject)

    def precision_and_recall(self, subject) -> PrecisionAndRecall:
        assert self.manifold_ref is not None, "call IPR.compute_manifold_ref() first"
        subj = self.compute_manifold(subject)
        prec, rec, _ = manifold_cover(self.manifold_ref, subj.features, subj.radii)
        return PrecisionAndRecall(float(prec.mean()), float(rec.mean()))

    def compute_manifold_ref(self, path):
        self.manifold_ref = self.compute_manifold(path)

    def realism(self, image):
        return realism(self.manifold_ref, self.extract_features(image))

    def compute_manifold(self, input) -> Manifold:
        if isinstance(input, str):
            if input.endswith(".npz"):
                return load_manifold(input)
            feats = self.extract_features_from_files(input)
        elif isinstance(input, torch.Tensor):
            feats = self.extract_features(input)
        elif isinstance(input, np.ndarray):
            feats = self.extract_features(torch.as_tensor(input, dtype=torch.float32))
        elif isinstance(input, list) and input:
            if isinstance(input[0], torch.Tensor):
                feats = self.extract_features(torch.cat(input, dim=0))
            elif isinstance(input[0], np.ndarray):
                feats = self.extract_features(torch.as_tensor(np.concatenate(input, axis=0), dtype=torch.float32))
            elif isinstance(input[0], str):
                feats = self.extract_features_from_files(input)
            else:
                raise TypeError(type(input[0]))
        else:
            raise TypeError(type(input))
        return Manifold(feats, manifold_radii(feats, self.k))

    def extract_features(self, images: torch.Tensor) -> np.ndarray:
        """fp32 [N, 4096] features of normalised images [N, 3, H, W] (nearest-resized to 224 x 224 if needed)."""
        out = [self.vgg16(images[s:s + self.batch_size]).cpu() for s in range(0, images.shape[0], self.batch_size)]
        return torch.cat(out).numpy() if out else np.zeros((0, 4096), np.float32)

    def extract_features_from_files(self, path_or_fnames) -> np.ndarray:
        files = image_files(path_or_fnames) if isinstance(path_or_fnames, str) else list(path_or_fnames)
        if self.num_samples > 0:
            files = files[:self.num_samples]
        if len(files) < self.num_samples:
            print("WARNING: num_found_images(%d) < num_samples(%d)" % (len(files), self.num_samples))
        feats = []
        with ThreadPoolExecutor(max(1, self.num_workers)) as pool:      # PIL decodes and resizes without the GIL
            for s in range(0, len(files), self.batch_size):
                batch = np.stack(list(pool.map(load_image, files[s:s + self.batch_size])))
                feats.append(self.vgg16(torch.from_numpy(batch)).cpu())
        return torch.cat(feats).numpy() if feats else np.zeros((0, 4096), np.float32)

    def save_ref(self, fname: str):
        print("saving manifold to", fname, "...")
        save_manifold(fname, self.manifold_ref)
