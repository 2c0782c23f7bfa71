from .multicontrolnet import MultiControlNetModel  # noqa: F401
