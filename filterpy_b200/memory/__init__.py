"""The fading-memory polynomial filter on the GPU: a mirror of filterpy.memory."""
from .fading_memory import FadingMemoryFilter  # noqa: F401
