"""GPU mirrors of ``filterpy.kalman`` for the hot path (see DESIGN.md for the scope)."""
from .kalman_filter import KalmanFilter, predict, update, batch_filter, rts_smoother  # noqa: F401
from .sigma_points import MerweScaledSigmaPoints, JulierSigmaPoints  # noqa: F401
from .UKF import (UnscentedKalmanFilter, LinearFx, ConstVelFx, LinearHx, RangeAzElHx,  # noqa: F401
                  RangeBearingHx, DeviceFx, DeviceHx)
from .CubatureKalmanFilter import CubatureKalmanFilter  # noqa: F401
from .square_root import SquareRootKalmanFilter  # noqa: F401
from .unscented_transform import unscented_transform  # noqa: F401
from .IMM import IMMEstimator  # noqa: F401
from .mmae import MMAEFilterBank  # noqa: F401
