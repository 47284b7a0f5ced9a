// ukf_rts_launch.cuh — parameter block of the UKF RTS smoother kernel (shared by ukf_rts.cu and ukf_rtc.cu)
#pragma once
#include "ukf_rts_kernel.cuh"

namespace bke {

template <typename T>
inline void ukf_rts_fill_params(const bke_ukf_rts_args &a, UrP<T> &p)
{
    const int n = a.dim_x;
    p.N = a.n_filters; p.Tn = a.n_steps; p.n = n; p.fx = a.fx_model;
    if (a.flags & BKE_UKF_SIMPLEX) {                                        // sigma_points.py:516-522
        p.scale = T(1);
        p.wm0 = p.wc0 = p.wi = (T)(1. / (n + 1));
    } else {
        const double lambda_ = a.alpha * a.alpha * (n + a.kappa) - n;      // sigma_points.py:167
        p.scale = (T)(lambda_ + n);
        p.wm0 = (T)(lambda_ / (n + lambda_));
        p.wc0 = (T)(lambda_ / (n + lambda_) + (1 - a.alpha * a.alpha + a.beta));
        p.wi = (T)(.5 / (n + lambda_));
    }
    p.dt = (T)a.dt;
    p.Xs = (const T *)a.Xs; p.Ps = (const T *)a.Ps; p.Q = (const T *)a.Q; p.F = (const T *)a.F;
    p.sQ = a.Q_stride; p.sF = a.F_stride; p.dts = a.dts;
    p.x_out = (T *)a.x_out; p.P_out = (T *)a.P_out; p.K = (T *)a.K; p.status = a.status;
    p.fx_args = nullptr; p.s_fx_args = 0;
}

}  // namespace bke
