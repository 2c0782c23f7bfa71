"""Opt-in stand-in for the `diffusers` names the reference's inference scripts import (SURVEY.md §8b "Import surface of
the callers"): put `imagdressing_b200/compat` on PYTHONPATH *instead of* a diffusers install and

    from diffusers import UNet2DConditionModel, AutoencoderKL, DDIMScheduler, ControlNetModel

resolves to the H100 host models of this repo: the denoising / garment UNet, the ControlNet, the DDIM scheduler and (round 2,
SURVEY.md §8f row 1) the VAE, all executing on the sm_90a kernels.
Never shadow a real diffusers install with this package by accident: it is not on the path unless you add it.
"""
from imagdressing_b200.modeling import ControlNetModel, UNet2DConditionModel  # noqa: F401
from imagdressing_b200.scheduler import DDIMScheduler  # noqa: F401
from imagdressing_b200.vae import AutoencoderKL  # noqa: F401

__version__ = "0.24.0+imagd_b200_compat"


from . import utils, pipelines, schedulers  # noqa: E402,F401
