"""diffusers.pipelines.controlnet.multicontrolnet (SURVEY.md §8b): the multi-ControlNet container the reference's
ControlNet pipelines import."""
from imagdressing_b200.modeling import MultiControlNetModel  # noqa: F401
