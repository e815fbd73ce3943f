"""Alias of lvdm/modules/encoders/resampler.py (reference :96): the image-context Resampler on the H100 kernels."""
from tooncrafter_b200.modules import Resampler  # noqa: F401
