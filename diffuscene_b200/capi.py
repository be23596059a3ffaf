"""ctypes binding of include/diffuscene_b200.h (the C ABI of the CUDA engine).

This is exactly the stub a reference maintainer would add (INTEGRATION.md): load the shared library,
declare argtypes, pass raw device pointers (`tensor.data_ptr()`) and the CUDA stream handle.
There is no fallback: if the library is missing it is built with nvcc; if that fails, import fails.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Optional, Tuple

import torch

from . import build as _build

DS_PREC_FP32, DS_PREC_BF16 = 0, 1
DS_GEMM_AUTO, DS_GEMM_SIMT, DS_GEMM_TCGEN05 = 0, 1, 2
DS_MEAN_EPS, DS_MEAN_X0, DS_MEAN_V = 0, 1, 2
MEAN_TYPES = {"eps": DS_MEAN_EPS, "x0": DS_MEAN_X0, "v": DS_MEAN_V}
DS_TRAIN_ACT, DS_TRAIN_GRAD, DS_TRAIN_DW, DS_TRAIN_DVEC, DS_TRAIN_COND = range(5)
TRAIN_COND = {n: i for i, n in enumerate((
    "emb", "z1", "h1", "temb", "st", "film", "dfilm", "dtemb", "dh1", "dst", "ctx_act", "ctx_film", "dctx_film",
    "dctx_act", "xkv", "xctx", "x_t"))}      # DS_TRAIN_COND indices (include/diffuscene_b200.h)
ROOM_ENC_STATE = {n: i for i, n in enumerate((
    "x0", "a1", "p", "h", "o", "wp", "bias", "dwp", "dbias", "dz", "dh", "dp", "da1"))}      # DS_RE_* kinds
TEXT_ENC_TAP = {n: i for i, n in enumerate(("x", "qkv", "ctx", "y1", "h1", "inter", "y2", "out"))}      # DS_TE_* kinds


class DsConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "dim", "channels", "seperate_all", "objectness_dim", "class_dim", "translation_dim", "size_dim",
        "angle_dim", "objfeat_dim", "cond_dim", "text_condition", "text_dim", "n_stages", "num_objects",
        "num_timesteps", "precision", "gemm_backend", "device", "fuse_level", "train")] + [("reserved", C.c_int32 * 6)]


class DsSchedule(C.Structure):
    _fields_ = [("T", C.c_int32), ("mean_type", C.c_int32)] + [(n, C.POINTER(C.c_float)) for n in (
        "sqrt_ac", "sqrt_1mac", "sqrt_recip_ac", "sqrt_recipm1_ac", "coef1", "coef2", "sigma", "alphas_cumprod",
        "loss_weight")]


class DsSampleArgs(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("clip_denoised", C.c_int32), ("num_steps", C.c_int32), ("ddim", C.c_int32),
        ("ddim_eta", C.c_float), ("seed", C.c_uint64), ("scene_offset", C.c_uint64),
        ("x_init_dev", C.c_void_p), ("noise_dev", C.c_void_p), ("partial_dev", C.c_void_p),
        ("num_partial", C.c_int32), ("partial_noise_dev", C.c_void_p), ("traj_freq", C.c_int32),
        ("traj_dev", C.c_void_p), ("use_graph", C.c_int32), ("ddim_times", C.POINTER(C.c_int32)),
        ("chunk_scenes", C.c_int32), ("reserved", C.c_int32 * 5)]


class DsRoomEncConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("precision", "input_channels", "height", "width", "device")] + \
        [("reserved", C.c_int32 * 3)]


class DsShapeAeConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("latent_dim", "num_points", "device")] + [("reserved", C.c_int32 * 5)]


class DsTextEncConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("layers", "hidden", "heads", "intermediate", "vocab", "max_positions",
                                         "type_vocab", "precision", "capacity", "device")] + [("reserved", C.c_int32 * 6)]


class DsVggConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("precision", "capacity", "device")] + [("reserved", C.c_int32 * 5)]


class DsInceptionConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("precision", "capacity", "device")] + [("reserved", C.c_int32 * 5)]


class DsRenderCamera(C.Structure):
    _fields_ = [("eye", C.c_float * 3), ("target", C.c_float * 3), ("up", C.c_float * 3)] + \
        [(n, C.c_float) for n in ("left", "right", "bottom", "top", "near_plane", "far_plane")] + \
        [("width", C.c_int32), ("height", C.c_int32), ("projection", C.c_int32), ("reserved", C.c_int32 * 3)]


class DsRenderArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("num_objects", C.c_int32)] + \
        [(n, C.c_void_p) for n in ("translation_dev", "size_dev", "angle_dev", "model_index_dev", "class_index_dev",
                                   "floor_offsets_dev", "floor_tris_dev")] + \
        [("num_floor_tris", C.c_int32), ("num_colors", C.c_int32), ("palette_dev", C.c_void_p),
         ("floor_textures_dev", C.c_void_p), ("num_floor_textures", C.c_int32), ("floor_texture_size", C.c_int32),
         ("floor_texture_index_dev", C.c_void_p), ("flags", C.c_int32), ("reserved0", C.c_int32),
         ("image_dev", C.c_void_p), ("id_dev", C.c_void_p), ("reserved", C.c_int32 * 8)]


DS_RENDER_NO_TEXTURE, DS_RENDER_WHITE_BACKGROUND = 1, 2
DS_RENDER_ORTHOGRAPHIC, DS_RENDER_PERSPECTIVE = 0, 1


class DsSceneBatchArgs(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("num_scenes", "num_class_columns", "objfeat_dim", "layout_h", "layout_w",
                                         "scaling", "angle_dim", "permute", "num_augmentations")] + \
        [("augmentations", C.c_int32 * 2), ("batch", C.c_int32), ("num_slots", C.c_int32)] + \
        [(n, C.c_void_p) for n in ("offsets_dev", "lengths_dev", "class_dev", "translations_dev", "sizes_dev",
                                   "angles_dev", "objfeats_dev", "layouts_dev")] + \
        [("bounds_translations", C.c_double * 6), ("bounds_sizes", C.c_double * 6), ("bounds_angles", C.c_double * 2),
         ("bounds_objfeats", C.c_double * 2)] + \
        [(n, C.c_void_p) for n in ("scene_index_dev", "rot_angle_dev", "jitter_dev", "perm_key_dev",
                                   "class_labels_out_dev", "translations_out_dev", "sizes_out_dev", "angles_out_dev",
                                   "objfeats_out_dev", "length_out_dev", "room_layout_out_dev")]


DS_SCENE_AUG_FIXED_ROTATION, DS_SCENE_AUG_ROTATION, DS_SCENE_AUG_JITTER = 1, 2, 3
DS_SCENE_SCALE, DS_SCENE_SCALE_COSIN_OBJFEATSNORM = 0, 1


class DsVlbArgs(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("clip_denoised", C.c_int32), ("x0_dev", C.c_void_p), ("seed", C.c_uint64),
        ("scene_offset", C.c_uint64), ("noise_dev", C.c_void_p), ("use_graph", C.c_int32),
        ("reserved", C.c_int32 * 7)]


# prototype of every symbol of include/diffuscene_b200.h: name -> (restype, argtypes)
_H = C.c_void_p
_p = C.c_void_p
sig = {
    "ds_create": (C.c_int, [C.POINTER(DsConfig), C.POINTER(_H)]),
    "ds_destroy": (C.c_int, [_H]),
    "ds_last_error": (C.c_char_p, []),
    "ds_version": (C.c_char_p, []),
    "ds_load_weight": (C.c_int, [_H, C.c_char_p, _p, C.c_int64]),
    "ds_commit_weights": (C.c_int, [_H]),
    "ds_expected_weight_count": (C.c_int, [_H]),
    "ds_expected_weight": (C.c_int, [_H, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64)]),
    "ds_set_schedule": (C.c_int, [_H, C.POINTER(DsSchedule)]),
    "ds_set_vlb_schedule": (C.c_int, [_H, C.c_int32, _p, _p, _p]),
    "ds_vlb_loop": (C.c_int, [_H, C.POINTER(DsVlbArgs), _p, _p, _p, _p]),
    "ds_set_context": (C.c_int, [_H, _p, C.c_int32, C.c_int32, _p]),
    "ds_set_context_cross": (C.c_int, [_H, _p, C.c_int32, C.c_int32, _p]),
    "ds_denoise_forward": (C.c_int, [_H, _p, _p, _p, C.c_int32, _p]),
    "ds_denoise_forward_host": (C.c_int, [_H, _p, _p, _p, C.c_int32]),
    "ds_sample_loop": (C.c_int, [_H, C.POINTER(DsSampleArgs), _p, _p]),
    "ds_sample_loop_host": (C.c_int, [_H, C.POINTER(DsSampleArgs), _p]),
    "ds_traj_count": (C.c_int, [C.c_int32, C.c_int32]),
    "ds_p_sample_step": (C.c_int, [_H, _p, _p, _p, C.c_int32, _p, C.c_int32, _p]),
    "ds_q_sample": (C.c_int, [_H, _p, _p, _p, _p, C.c_int32, _p]),
    "ds_p_losses": (C.c_int, [_H, _p, _p, _p, C.c_int32, C.c_int32, _p, _p, _p, C.c_int32, _p]),
    "ds_train_param_count": (C.c_int64, [_H]),
    "ds_train_step": (C.c_int, [_H, _p, _p, _p, _p, _p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _p, C.c_float, _p, _p, _p, _p,
                                C.c_int32, _p]),
    "ds_train_step_cross": (C.c_int, [_H, _p, _p, _p, _p, _p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _p, C.c_float, _p, _p,
                                      _p, _p, _p, C.c_int32, _p, C.c_int32, _p]),
    "ds_train_set_buckets": (C.c_int, [_H, _p, C.c_int32, _p]),
    "ds_train_phase_ms": (C.c_int, [_H, _p]),
    "ds_train_read": (C.c_int, [_H, C.c_int32, C.c_int32, _p, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int32), _p]),
    "ds_sumsq": (C.c_int, [_p, C.c_int64, _p, _p]),
    "ds_adam_step": (C.c_int, [_p, _p, _p, _p, C.c_int64, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int32, _p,
                               C.c_float, _p]),
    "ds_retrieve_objects": (C.c_int, [_p, C.c_int32, _p, _p, C.c_int32, C.c_int32, _p, _p, _p, C.c_int32, C.c_int32, _p, _p]),
    "ds_scene_boxes": (C.c_int, [_p, _p, _p, _p, C.c_int32, _p, _p, C.c_int32, _p, _p, C.c_int32, _p, _p]),
    "ds_scene_stats": (C.c_int, [_p, _p, _p, _p, C.c_int32, C.c_int32, _p, _p, _p, _p, _p, _p, _p, _p]),
    "ds_plan_describe": (C.c_int, [C.POINTER(DsConfig), C.c_char_p, C.c_int64]),
    "ds_plan_export_json": (C.c_int, [C.POINTER(DsConfig), C.c_int32, C.c_char_p, C.c_int64]),
    "ds_enable_taps": (C.c_int, [_H, C.c_int32]),
    "ds_read_tap": (C.c_int, [_H, C.c_char_p, _p, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "ds_launch_count": (C.c_int64, [_H]),
    "ds_graph_build_count": (C.c_int64, [_H]),
    "ds_profile_ops": (C.c_int, [_H, C.c_int32, C.c_char_p, C.c_int64, _p, C.c_int32]),
    "ds_test_gemm_bf16": (C.c_int, [C.c_int, _p, _p, _p, _p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _p]),
    "ds_room_enc_create": (C.c_int, [C.POINTER(DsRoomEncConfig), C.POINTER(_H)]),
    "ds_room_enc_destroy": (C.c_int, [_H]),
    "ds_room_enc_expected_weight_count": (C.c_int, [_H]),
    "ds_room_enc_expected_weight": (C.c_int, [_H, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64)]),
    "ds_room_enc_forward": (C.c_int, [_H, _p, _p, C.c_int32, _p, C.c_int32, _p]),
    "ds_room_enc_backward": (C.c_int, [_H, _p, _p, _p]),
    "ds_room_enc_read": (C.c_int, [_H, C.c_int32, C.c_int32, _p, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int32), _p]),
    "ds_shape_ae_create": (C.c_int, [C.POINTER(DsShapeAeConfig), C.POINTER(_H)]),
    "ds_shape_ae_destroy": (C.c_int, [_H]),
    "ds_shape_ae_expected_weight_count": (C.c_int, [_H]),
    "ds_shape_ae_expected_weight": (C.c_int, [_H, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64)]),
    "ds_shape_ae_forward": (C.c_int, [_H, _p, _p, C.c_int32, _p, C.c_int32, C.c_int32, _p, _p, _p, _p]),
    "ds_shape_ae_train_step": (C.c_int, [_H, _p, _p, C.c_int32, _p, C.c_float, _p, _p, _p]),
    "ds_shape_ae_set_knn": (C.c_int, [_H, _p]),
    "ds_shape_ae_get_knn": (C.c_int, [_H, _p, _p]),
    "ds_knn": (C.c_int, [_p, C.c_int32, C.c_int32, C.c_int32, _p, _p]),
    "ds_chamfer_forward": (C.c_int, [_p, C.c_int32, _p, C.c_int32, C.c_int32, _p, _p, _p, _p, _p]),
    "ds_chamfer_backward": (C.c_int, [_p, C.c_int32, _p, C.c_int32, C.c_int32, _p, _p, _p, _p, _p, _p, _p]),
    "ds_text_enc_create": (C.c_int, [C.POINTER(DsTextEncConfig), C.POINTER(_H)]),
    "ds_text_enc_destroy": (C.c_int, [_H]),
    "ds_text_enc_expected_weight_count": (C.c_int, [_H]),
    "ds_text_enc_expected_weight": (C.c_int, [_H, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64)]),
    "ds_text_enc_set_weights": (C.c_int, [_H, _p, _p]),
    "ds_text_enc_forward": (C.c_int, [_H, _p, _p, C.c_int32, C.c_int32, _p, _p]),
    "ds_text_enc_set_tap": (C.c_int, [_H, C.c_int32]),
    "ds_text_enc_read": (C.c_int, [_H, C.c_int32, _p, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int32), _p]),
    "ds_vgg_create": (C.c_int, [C.POINTER(DsVggConfig), C.POINTER(_H)]),
    "ds_vgg_destroy": (C.c_int, [_H]),
    "ds_vgg_expected_weight_count": (C.c_int, [_H]),
    "ds_vgg_expected_weight": (C.c_int, [_H, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64)]),
    "ds_vgg_set_weights": (C.c_int, [_H, _p, C.c_int64, _p]),
    "ds_vgg_features": (C.c_int, [_H, _p, C.c_int32, C.c_int32, C.c_int32, _p, _p]),
    "ds_vgg_test_conv": (C.c_int, [_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _p, _p, _p, _p]),
    "ds_manifold_distances": (C.c_int, [_p, C.c_int32, _p, C.c_int32, C.c_int32, _p, _p, _p]),
    "ds_manifold_radii": (C.c_int, [_p, C.c_int32, C.c_int32, C.c_int32, _p, _p, _p]),
    "ds_manifold_cover": (C.c_int, [_p, _p, C.c_int32, _p, _p, C.c_int32, C.c_int32, _p, _p, _p, _p, _p]),
    "ds_inception_create": (C.c_int, [C.POINTER(DsInceptionConfig), C.POINTER(_H)]),
    "ds_inception_destroy": (C.c_int, [_H]),
    "ds_inception_expected_weight_count": (C.c_int, [_H]),
    "ds_inception_expected_weight": (C.c_int, [_H, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64)]),
    "ds_inception_set_weights": (C.c_int, [_H, _p, C.c_int64, _p]),
    "ds_inception_features": (C.c_int, [_H, _p, C.c_int32, C.c_int32, C.c_int32, _p, _p]),
    "ds_inception_test_conv": (C.c_int, [C.c_int32, _p] + [C.c_int32] * 10 + [_p, _p, _p, C.c_int32, C.c_int32, _p]),
    "ds_feature_stats": (C.c_int, [_p, C.c_int32, C.c_int32, _p, _p, _p]),
    "ds_kid_terms": (C.c_int, [_p, C.c_int32, _p, C.c_int32, C.c_int32, _p, _p, C.c_int32, C.c_int32, _p, _p]),
    "ds_mesh_catalog_create": (C.c_int, [C.c_int32, _p, _p, _p, _p, _p, _p, _p, _p, _p, C.c_int32, C.c_int32, C.POINTER(_H)]),
    "ds_mesh_catalog_destroy": (C.c_int, [_H]),
    "ds_render_scenes": (C.c_int, [_H, C.POINTER(DsRenderCamera), C.POINTER(DsRenderArgs), _p]),
    "ds_resize_f32": (C.c_int, [_p] + [C.c_int32] * 5 + [_p, _p, C.c_int32, _p, _p, C.c_int32, _p, _p]),
    "ds_resize_u8": (C.c_int, [_p] + [C.c_int32] * 5 + [_p, _p, C.c_int32, _p, _p, C.c_int32, _p, _p, _p]),
    "ds_scene_batch": (C.c_int, [C.POINTER(DsSceneBatchArgs), _p]),
}


_lib = None


def lib_path() -> str:
    return _build.LIB_PATH


def load(rebuild: bool = False):
    """Load (building first if needed) the shared library and declare its prototypes."""
    global _lib
    if _lib is not None and not rebuild:
        return _lib
    path = _build.build(force=rebuild)
    lib = C.CDLL(path)
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)      # AttributeError here == a symbol of the header is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


EXPORTED = list(sig)


class DsError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__("diffuscene_b200 error %d: %s" % (code, msg))
        self.code = code


def check(rc: int):
    if rc < 0:
        raise DsError(rc, load().ds_last_error().decode(errors="replace"))
    return rc


def ptr(t: Optional[torch.Tensor]):
    """The device pointer argument of a tensor (None: NULL)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream(device=None):
    """The stream argument: torch's current stream on `device` (None: the current device)."""
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def expected_weights(lib, prefix: str, h) -> List[Tuple[str, int]]:
    """(name, numel) of handle `h`'s flat parameter buffer, in order: <prefix>_expected_weight over
    <prefix>_expected_weight_count, e.g. prefix "ds_vgg" (the denoiser's is "ds")."""
    get = getattr(lib, prefix + "_expected_weight")
    out = []
    for i in range(check(getattr(lib, prefix + "_expected_weight_count")(h))):
        name, numel = C.c_char_p(), C.c_int64()
        check(get(h, i, C.byref(name), C.byref(numel)))
        out.append((name.value.decode(), numel.value))
    return out


class FeatureNet:
    """An image feature network on the device: one <prefix>_* handle (create, expected_weight, set_weights, features,
    destroy) whose weights come from a torchvision-style state dict, uploaded once as one flat fp32 buffer.

    precision "fp32" (default) or "bf16"; `state_dict_or_path` is a state dict, a file holding one, or the module
    itself.  Calling it with fp32 images [B, 3, H, W] (any device) returns fp32 [B, features] on the device.
    Subclasses set the symbol prefix, config struct, feature width and the names their messages use."""
    prefix = ""              # "ds_vgg", "ds_inception"
    config = None            # DsVggConfig, DsInceptionConfig
    features = 0
    name = ""                # the network in messages
    module = "a module"      # what else a state dict may come from, in the TypeError
    image_shape = "[B, 3, H, W]"
    cuda_guard = False       # raise RuntimeError before any library call when torch sees no CUDA device

    def __init__(self, state_dict_or_path, precision: str = "fp32", capacity: Optional[int] = None, device: int = 0):
        if precision not in ("bf16", "fp32"):
            raise ValueError("precision must be 'bf16' or 'fp32', not %r" % (precision,))
        sd = state_dict_or_path
        if isinstance(sd, (str, os.PathLike)):
            sd = torch.load(sd, map_location="cpu", weights_only=True)
        elif isinstance(sd, torch.nn.Module):
            sd = sd.state_dict()
        if not isinstance(sd, dict):
            raise TypeError("%s weights must be a state dict, a state-dict file or %s, not %s"
                            % (self.name, self.module, type(state_dict_or_path).__name__))
        if self.cuda_guard and not torch.cuda.is_available():
            raise RuntimeError("%s needs a CUDA device: diffuscene_b200 has no CPU fallback" % type(self).__name__)
        self.lib = load()
        self.device = torch.device("cuda", device)
        cfg = self.config()
        cfg.precision = DS_PREC_BF16 if precision == "bf16" else DS_PREC_FP32
        cfg.capacity = capacity or (64 if precision == "bf16" else 8)
        cfg.device = device
        self.capacity = cfg.capacity
        self.precision = precision
        self._h = C.c_void_p()
        check(self._fn("create")(C.byref(cfg), C.byref(self._h)))
        names = expected_weights(self.lib, self.prefix, self._h)
        missing = [n for n, _ in names if n not in sd]
        if missing:
            self.close()
            raise KeyError("%s state dict lacks %s" % (self.name, ", ".join(missing)))
        for n, numel in names:
            if sd[n].numel() != numel:
                self.close()
                raise ValueError("%s has %d elements, expected %d" % (n, sd[n].numel(), numel))
        flat = torch.cat([sd[n].reshape(-1).float() for n, _ in names]).to(self.device)
        check(self._fn("set_weights")(self._h, ptr(flat), flat.numel(), stream(self.device)))
        torch.cuda.current_stream(self.device).synchronize()

    def _fn(self, suffix: str):
        return getattr(self.lib, self.prefix + "_" + suffix)

    @classmethod
    def inventory(cls, lib=None, h=None) -> List[Tuple[str, int]]:
        """(name, numel) of the flat parameter buffer, state-dict order; without `h`, of a temporary fp32 handle of
        capacity 1 (which needs a device)."""
        lib = lib or load()
        if h is not None:
            return expected_weights(lib, cls.prefix, h)
        cfg = cls.config()
        cfg.precision, cfg.capacity = DS_PREC_FP32, 1
        h = C.c_void_p()
        check(getattr(lib, cls.prefix + "_create")(C.byref(cfg), C.byref(h)))
        try:
            return expected_weights(lib, cls.prefix, h)
        finally:
            getattr(lib, cls.prefix + "_destroy")(h)

    def __call__(self, images: torch.Tensor) -> torch.Tensor:
        if images.dim() != 4 or images.shape[1] != 3:
            raise ValueError("images must be %s, got %s" % (self.image_shape, tuple(images.shape)))
        x = images.to(self.device, torch.float32).contiguous()
        out = torch.empty(x.shape[0], self.features, device=self.device, dtype=torch.float32)
        if x.shape[0] == 0:
            return out
        check(self._fn("features")(self._h, ptr(x), x.shape[0], x.shape[2], x.shape[3], ptr(out), stream(self.device)))
        return out

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._fn("destroy")(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def make_config(spec, num_objects: int, num_timesteps: int, precision: int = DS_PREC_BF16,
                gemm_backend: int = DS_GEMM_AUTO, device: int = 0, fuse_level: int = 0, train: int = 0) -> DsConfig:
    """DsConfig from a diffuscene_b200.weights.NetSpec."""
    c = DsConfig()
    c.dim, c.channels, c.seperate_all = spec.dim, spec.channels, int(spec.seperate_all)
    c.objectness_dim, c.class_dim = spec.objectness_dim, spec.class_dim
    c.translation_dim, c.size_dim, c.angle_dim = spec.translation_dim, spec.size_dim, spec.angle_dim
    c.objfeat_dim, c.cond_dim = spec.objfeat_dim, spec.cond_dim
    c.text_condition, c.text_dim = int(spec.text_condition), spec.text_dim
    c.n_stages, c.num_objects, c.num_timesteps = spec.n_stages, num_objects, num_timesteps
    c.precision, c.gemm_backend, c.device, c.fuse_level = precision, gemm_backend, device, fuse_level
    c.train = int(train)
    return c


def plan_describe(cfg: DsConfig) -> str:
    lib = load()
    buf = C.create_string_buffer(1 << 20)
    check(lib.ds_plan_describe(C.byref(cfg), buf, len(buf)))
    return buf.value.decode()


def plan_export(cfg: DsConfig, no_reuse: bool = False) -> dict:
    import json
    lib = load()
    buf = C.create_string_buffer(1 << 22)
    check(lib.ds_plan_export_json(C.byref(cfg), int(no_reuse), buf, len(buf)))
    return json.loads(buf.value.decode())


def plan_expected_weights(cfg: DsConfig) -> List[Tuple[str, int]]:
    txt = plan_describe(cfg)
    lines = txt.split("weights:\n", 1)[1].strip().split("\n")
    return [(l.rsplit(" ", 1)[0], int(l.rsplit(" ", 1)[1])) for l in lines]
