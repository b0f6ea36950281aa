"""H100 renderer modules served under the reference import name ``training.volumetric_rendering``."""
