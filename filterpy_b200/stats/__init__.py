"""filterpy.stats's evaluators on the GPU: single calls and banks of tracks against candidates."""
from .stats import mahalanobis, log_likelihood, likelihood, logpdf, NEES, score_measurements  # noqa: F401
