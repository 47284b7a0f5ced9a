"""The expanding-memory least-squares filter on the GPU: a mirror of filterpy.leastsq."""
from .least_squares import LeastSquaresFilter  # noqa: F401
