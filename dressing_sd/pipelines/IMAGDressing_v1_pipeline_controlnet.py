"""Drop-in for the reference's dressing_sd/pipelines/IMAGDressing_v1_pipeline_controlnet.py: same import path and class name
(`IMAGDressing_v1`), constructor and `__call__` keyword arguments; implemented by
imagdressing_b200.pipelines.IMAGDressing_v1_ControlNet on the sm_90a kernels."""
from imagdressing_b200.pipelines import IMAGDressing_v1_ControlNet as _Impl
from imagdressing_b200.pipelines import StableDiffusionPipelineOutput  # noqa: F401


class IMAGDressing_v1(_Impl):
    __doc__ = _Impl.__doc__


__all__ = ["IMAGDressing_v1"]
