"""g-h filters on the GPU: mirrors of filterpy.gh (GHFilter, GHKFilter, GHFilterOrder) and its gain helpers."""
from .gh_filter import (GHFilter, GHKFilter, GHFilterOrder, optimal_noise_smoothing,  # noqa: F401
                        least_squares_parameters, critical_damping_parameters, benedict_bornder_constants)
