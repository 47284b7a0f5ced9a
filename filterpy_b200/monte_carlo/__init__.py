"""GPU mirrors of ``filterpy.monte_carlo`` for the hot path."""
from .resampling import (systematic_resample, stratified_resample, multinomial_resample, residual_resample,  # noqa: F401
                         residual_resample_with_uniforms,
                         gather_particles, exact_cumsum, ResamplePlan, normalize_weights,
                         systematic_resample_bank, stratified_resample_bank, gather_particles_bank,
                         BankResamplePlan, multinomial_resample_bank, residual_resample_bank,
                         systematic_resample_bank_if_degenerate, stratified_resample_bank_if_degenerate)
