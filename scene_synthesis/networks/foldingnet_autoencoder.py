"""Drop-in for the reference's scene_synthesis/networks/foldingnet_autoencoder.py: the KL shape auto-encoder that
produces the per-object latents, on the CUDA library (diffuscene_b200/shape_ae.py)."""
from diffuscene_b200.networks.diffusion_scene_layout_ddpm import train_on_batch, validate_on_batch  # noqa: F401
from diffuscene_b200.shape_ae import KLAutoEncoder, chamfer_3DDist  # noqa: F401


class AutoEncoder:
    """The reference's plain (non-variational) FoldingNet auto-encoder; no shipped config trains it."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError("the plain AutoEncoder is not ported; use KLAutoEncoder")
