"""Scheduler names the reference pipelines use in type annotations. DDIM, DPM-Solver++, Euler / Euler-ancestral and
UniPC are implemented; PNDM and LMS are not."""
from imagdressing_b200.samplers import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,  # noqa: F401
                                        EulerDiscreteScheduler, UniPCMultistepScheduler)
from imagdressing_b200.scheduler import DDIMScheduler  # noqa: F401


class _NotBuilt:
    def __init__(self, *a, **k):
        raise NotImplementedError(f"{type(self).__name__} is not built; available: DDIMScheduler, "
                                  "DPMSolverMultistepScheduler, EulerDiscreteScheduler, "
                                  "EulerAncestralDiscreteScheduler, UniPCMultistepScheduler")


class LMSDiscreteScheduler(_NotBuilt):
    pass


class PNDMScheduler(_NotBuilt):
    pass
