"""Seeded synthetic inputs for the benchmark configurations (BASELINE.json ``configs``).

Pure NumPy, setup-time only (never on the timed path).  The model builders follow the
definitions the reference uses to build its kinematic examples — constant-velocity /
constant-acceleration transition blocks (``filterpy/common/kinematic.py:41-44``) and the
piecewise-white-noise Q (``filterpy/common/discretization.py:130-136``) — written out per
filter so that every filter of a bank has its own dt / q / r (F, Q, R traffic is real).
"""
import numpy as np

__all__ = ["q_white_noise_block", "kf_bank_cv2d", "kf_bank_ca3d", "kf_single_cv2d",
           "ukf_bank_cv3d", "resample_weights"]


def q_white_noise_block(dim, dt, var):
    """Discrete white-noise Q block for one axis; dt/var broadcast over a leading N axis.

    dim=2: [[dt^4/4, dt^3/2],[dt^3/2, dt^2]] * var;  dim=3 adds the acceleration row
    (discretization.py:130-136)."""
    dt = np.asarray(dt, float)
    var = np.asarray(var, float)
    if dim == 2:
        rows = [[.25 * dt ** 4, .5 * dt ** 3],
                [.5 * dt ** 3, dt ** 2]]
    elif dim == 3:
        one = np.ones_like(dt)
        rows = [[.25 * dt ** 4, .5 * dt ** 3, .5 * dt ** 2],
                [.5 * dt ** 3, dt ** 2, dt],
                [.5 * dt ** 2, dt, one]]
    else:
        raise ValueError("dim must be 2 or 3")
    q = np.stack([np.stack(r, axis=-1) for r in rows], axis=-2)
    return q * var[..., None, None]


def _block_diag(blocks):
    """blocks: list of [..., k, k] -> [..., K, K]."""
    lead = blocks[0].shape[:-2]
    K = sum(b.shape[-1] for b in blocks)
    out = np.zeros(lead + (K, K))
    o = 0
    for b in blocks:
        k = b.shape[-1]
        out[..., o:o + k, o:o + k] = b
        o += k
    return out


def kf_single_cv2d(T=1000, seed=0):
    """Config C1: one KalmanFilter(4, 2), constant velocity, dt=1."""
    dt = 1.0
    F = np.array([[1, dt, 0, 0], [0, 1, 0, 0], [0, 0, 1, dt], [0, 0, 0, 1]], float)
    H = np.array([[1, 0, 0, 0], [0, 0, 1, 0]], float)
    q = q_white_noise_block(2, dt, 0.01)
    Q = _block_diag([q, q])
    R = 0.25 * np.eye(2)
    P0 = 10.0 * np.eye(4)
    x0 = np.zeros(4)
    rs = np.random.RandomState(seed)
    xt = np.array([0.0, 1.0, 0.0, 0.5])
    zs = np.zeros((T, 2))
    for t in range(T):
        xt = F @ xt
        zs[t] = H @ xt + 0.5 * rs.randn(2)
    return dict(x=x0, P=P0, F=F, H=H, Q=Q, R=R, zs=zs)


def kf_bank_cv2d(N, seed=1234, steps=1, dtype=np.float64):
    """Config C2: N filters, dim_x=4 (x, vx, y, vy), dim_z=2, per-filter dt/q/r."""
    rng = np.random.default_rng(seed)
    dt = rng.uniform(0.05, 0.2, N)
    q = np.exp(rng.uniform(np.log(1e-3), np.log(1e-1), N))
    r = rng.uniform(0.1, 1.0, N)
    F1 = np.zeros((N, 2, 2)); F1[:, 0, 0] = 1; F1[:, 0, 1] = dt; F1[:, 1, 1] = 1
    F = _block_diag([F1, F1])
    H = np.zeros((N, 2, 4)); H[:, 0, 0] = 1; H[:, 1, 2] = 1
    qb = q_white_noise_block(2, dt, q)
    Q = _block_diag([qb, qb])
    R = r[:, None, None] * np.eye(2)
    P0 = np.zeros((N, 4, 4))
    P0[:, np.arange(4), np.arange(4)] = rng.uniform(1.0, 10.0, (N, 4))
    x0 = rng.standard_normal((N, 4))
    xt = x0 + rng.standard_normal((N, 4))
    zs = np.zeros((steps, N, 2))
    for t in range(steps):
        xt = np.einsum("nij,nj->ni", F, xt)
        zs[t] = np.einsum("nij,nj->ni", H, xt) + np.sqrt(r)[:, None] * rng.standard_normal((N, 2))
    out = dict(x=x0, P=P0, F=F, H=H, Q=Q, R=R, zs=zs)
    return {k: np.ascontiguousarray(v, dtype=dtype) for k, v in out.items()}


def kf_bank_ca3d(N, seed=4321, steps=1, dtype=np.float64):
    """Config C3: N filters, dim_x=9 (x,x',x'',y,...), dim_z=3 position sensor."""
    rng = np.random.default_rng(seed)
    dt = rng.uniform(0.05, 0.2, N)
    q = np.exp(rng.uniform(np.log(1e-3), np.log(1e-1), N))
    r = rng.uniform(0.1, 1.0, N)
    F2 = np.zeros((N, 3, 3))
    F2[:, 0, 0] = 1; F2[:, 0, 1] = dt; F2[:, 0, 2] = .5 * dt * dt
    F2[:, 1, 1] = 1; F2[:, 1, 2] = dt; F2[:, 2, 2] = 1
    F = _block_diag([F2, F2, F2])
    H = np.zeros((N, 3, 9))
    for i in range(3):
        H[:, i, 3 * i] = 1
    qb = q_white_noise_block(3, dt, q)
    Q = _block_diag([qb, qb, qb])
    R = r[:, None, None] * np.eye(3)
    P0 = np.zeros((N, 9, 9))
    P0[:, np.arange(9), np.arange(9)] = rng.uniform(1.0, 10.0, (N, 9))
    x0 = rng.standard_normal((N, 9))
    xt = x0 + rng.standard_normal((N, 9))
    zs = np.zeros((steps, N, 3))
    for t in range(steps):
        xt = np.einsum("nij,nj->ni", F, xt)
        zs[t] = np.einsum("nij,nj->ni", H, xt) + np.sqrt(r)[:, None] * rng.standard_normal((N, 3))
    out = dict(x=x0, P=P0, F=F, H=H, Q=Q, R=R, zs=zs)
    return {k: np.ascontiguousarray(v, dtype=dtype) for k, v in out.items()}


def ukf_bank_cv3d(N, seed=2468, steps=1, dt=0.1, dtype=np.float64, linear_hx=False):
    """Config C4: N UKFs, state (x,vx,y,vy,z,vz), measurement (range, azimuth, elevation)
    — or the position triple when ``linear_hx`` — targets >= 100 m out and away from the
    +-pi azimuth cut."""
    rng = np.random.default_rng(seed)
    pos = np.stack([rng.uniform(100, 500, N), rng.uniform(-300, 300, N), rng.uniform(20, 200, N)], 1)
    vel = rng.uniform(-10, 10, (N, 3))
    xt = np.zeros((N, 6))
    xt[:, 0::2] = pos; xt[:, 1::2] = vel
    x0 = xt + rng.standard_normal((N, 6)) * np.array([2, .5, 2, .5, 2, .5])
    P0 = np.zeros((N, 6, 6))
    P0[:, np.arange(6), np.arange(6)] = rng.uniform(1.0, 9.0, (N, 6))
    q = np.exp(rng.uniform(np.log(1e-3), np.log(1e-1), N))
    qb = q_white_noise_block(2, np.full(N, dt), q)
    Q = _block_diag([qb, qb, qb])
    if linear_hx:
        sig = np.array([1.0, 1.0, 1.0])
    else:
        sig = np.array([1.0, 0.005, 0.005])
    R = np.broadcast_to(np.diag(sig ** 2), (N, 3, 3)).copy()
    zs = np.zeros((steps, N, 3))
    for t in range(steps):
        xt = xt.copy()
        xt[:, 0::2] += dt * xt[:, 1::2]
        px, py, pz = xt[:, 0], xt[:, 2], xt[:, 4]
        if linear_hx:
            h = np.stack([px, py, pz], 1)
        else:
            h = np.stack([np.sqrt(px * px + py * py + pz * pz), np.arctan2(py, px),
                          np.arctan2(pz, np.sqrt(px * px + py * py))], 1)
        zs[t] = h + sig * rng.standard_normal((N, 3))
    F = np.eye(6)
    for i in range(3):
        F[2 * i, 2 * i + 1] = dt
    Hlin = np.zeros((3, 6)); Hlin[0, 0] = Hlin[1, 2] = Hlin[2, 4] = 1
    out = dict(x=x0, P=P0, Q=Q, R=R, zs=zs, F=F, H=Hlin)
    return {k: np.ascontiguousarray(v, dtype=dtype) for k, v in out.items()}


# ----------------------------------------------------------------------------- user-supplied UKF models
# A process / measurement pair outside the built-in set, once as CUDA source text (DeviceFx / DeviceHx)
# and once as the Python callables the reference takes (tests/golden/make_golden.py runs those).
CT_FX_SOURCE = """
// coordinated turn, state (px, vx, py, vy); args[0] = turn rate omega [rad/s]
__device__ void fx(const real *x, real *out, real dt, const real *args)
{
    const real w = args[0], s = sin(w * dt), c = cos(w * dt);
    out[0] = x[0] + (s / w) * x[1] - ((1 - c) / w) * x[3];
    out[1] = c * x[1] - s * x[3];
    out[2] = x[2] + ((1 - c) / w) * x[1] + (s / w) * x[3];
    out[3] = s * x[1] + c * x[3];
}
"""
OFFSET_RB_HX_SOURCE = """
// range and bearing from a sensor at (args[0], args[1])
__device__ void hx(const real *x, real *z, const real *args)
{
    const real dx = x[0] - args[0], dy = x[2] - args[1];
    z[0] = sqrt(dx * dx + dy * dy);
    z[1] = atan2(dy, dx);
}
"""


def ct_fx(x, dt, omega):
    s, c = np.sin(omega * dt), np.cos(omega * dt)
    return np.array([x[0] + (s / omega) * x[1] - ((1 - c) / omega) * x[3],
                     c * x[1] - s * x[3],
                     x[2] + ((1 - c) / omega) * x[1] + (s / omega) * x[3],
                     s * x[1] + c * x[3]])


def offset_rb_hx(x, sx, sy):
    dx, dy = x[0] - sx, x[2] - sy
    return np.array([np.sqrt(dx * dx + dy * dy), np.arctan2(dy, dx)])


def ukf_bank_ct2d(N, seed=9753, steps=1, dt=0.5, dtype=np.float64, linear_hx=False):
    """N coordinated-turn targets (per-filter turn rate ``omega``) seen by a range / bearing sensor at
    ``sensor`` (or, ``linear_hx``, by a position sensor); targets stay right of the sensor, away from
    the +-pi bearing cut (the default residual does not wrap, UKF.py:327-335)."""
    rng = np.random.default_rng(seed)
    sensor = np.array([-50.0, 20.0])
    omega = rng.uniform(0.02, 0.12, N) * rng.choice([-1.0, 1.0], N)
    xt = np.stack([rng.uniform(200, 600, N), rng.uniform(-8, 8, N), rng.uniform(-200, 200, N), rng.uniform(-8, 8, N)], 1)
    x0 = xt + rng.standard_normal((N, 4)) * np.array([3, .5, 3, .5])
    P0 = np.zeros((N, 4, 4))
    P0[:, np.arange(4), np.arange(4)] = rng.uniform(1.0, 16.0, (N, 4))
    q = np.exp(rng.uniform(np.log(1e-3), np.log(1e-1), N))
    qb = q_white_noise_block(2, np.full(N, dt), q)
    Q = _block_diag([qb, qb])
    sig = np.array([2.5, 2.5]) if linear_hx else np.array([1.5, 0.004])
    R = np.broadcast_to(np.diag(sig ** 2), (N, 2, 2)).copy()
    zs = np.zeros((steps, N, 2))
    for t in range(steps):
        xt = np.stack([ct_fx(xt[f], dt, omega[f]) for f in range(N)])
        h = xt[:, [0, 2]] if linear_hx else np.stack([offset_rb_hx(xt[f], *sensor) for f in range(N)])
        zs[t] = h + sig * rng.standard_normal((N, 2))
    Hlin = np.zeros((2, 4)); Hlin[0, 0] = Hlin[1, 2] = 1
    out = dict(x=x0, P=P0, Q=Q, R=R, zs=zs, H=Hlin, omega=omega, sensor=sensor)
    return {k: np.ascontiguousarray(v, dtype=dtype) for k, v in out.items()}


def resample_weights(N, kind="heavy", seed=97):
    """Config C5 weights (fp64, normalised on the host with ``w /= w.sum()``)."""
    rng = np.random.default_rng(seed)
    if kind == "heavy":
        w = rng.random(N) ** 4
    elif kind == "uniform":
        w = np.full(N, 1.0)
    elif kind == "random":
        w = rng.random(N)
    elif kind == "zeros":          # 1 % exact zeros
        w = rng.random(N)
        w[rng.random(N) < 0.01] = 0.0
    elif kind == "degenerate":     # one particle holds 0.999
        w = rng.random(N)
        w *= 0.001 / w.sum()
        w[N // 3] = 0.999
    elif kind == "dyadic":         # multiples of 2^-52: every summation order is exact
        w = rng.random(N)
        w /= w.sum()
        w = np.floor(w * 2.0 ** 52) * 2.0 ** -52
        return w
    else:
        raise ValueError(kind)
    w /= w.sum()
    return w


# ----------------------------------------------------------------------------- angle hooks (UKF.py:97-140)
# Trackers whose angles cross +-pi: the reference's recipe passes residual / mean / state-add callables that
# wrap the angle and take circular means.  Each function is given as CUDA source text (DeviceFn, DeviceFx,
# DeviceHx) and as the Python callable the reference takes (tests/golden/make_golden_ukf_hooks.py).
RB_HOOKS_SOURCE = """
// (range, bearing) measurements: the bearing difference wrapped into (-pi, pi], the circular mean of the bearing
__device__ real rb_wrap(real a)
{
    const real pi = 3.14159265358979323846;
    if (a > pi) a -= 2 * pi; else if (a <= -pi) a += 2 * pi;
    return a;
}
__device__ void residual_z(const real *a, const real *b, real *out) { out[0] = a[0] - b[0]; out[1] = rb_wrap(a[1] - b[1]); }
__device__ void z_mean_fn(const real *sigmas, const real *Wm, real *out)
{
    real r = 0, s = 0, c = 0;
    for (int i = 0; i < BKE_N_SIGMAS; i++) {
        r += Wm[i] * sigmas[2 * i];
        s += Wm[i] * sin(sigmas[2 * i + 1]);
        c += Wm[i] * cos(sigmas[2 * i + 1]);
    }
    out[0] = r;
    out[1] = atan2(s, c);
}
"""
CTRV_FX_SOURCE = """
// constant turn rate and velocity, state (px, py, heading, speed, yaw rate); the heading stays in (-pi, pi]
__device__ void fx(const real *x, real *out, real dt, const real *args)
{
    const real pi = 3.14159265358979323846;
    const real psi = x[2], v = x[3], w = x[4];
    if (fabs(w) > real(1e-4)) {
        out[0] = x[0] + v / w * (sin(psi + w * dt) - sin(psi));
        out[1] = x[1] + v / w * (cos(psi) - cos(psi + w * dt));
    } else {
        out[0] = x[0] + v * cos(psi) * dt;
        out[1] = x[1] + v * sin(psi) * dt;
    }
    real h = psi + w * dt;
    if (h > pi) h -= 2 * pi; else if (h <= -pi) h += 2 * pi;
    out[2] = h; out[3] = v; out[4] = w;
}
"""
CTRV_RB_HX_SOURCE = """
// range and bearing of (px, py) from a sensor at (args[0], args[1])
__device__ void hx(const real *x, real *z, const real *args)
{
    const real dx = x[0] - args[0], dy = x[1] - args[1];
    z[0] = sqrt(dx * dx + dy * dy);
    z[1] = atan2(dy, dx);
}
"""
CTRV_X_HOOKS_SOURCE = """
// CTRV state: the heading (x[2]) is an angle
__device__ real ctrv_wrap(real a)
{
    const real pi = 3.14159265358979323846;
    if (a > pi) a -= 2 * pi; else if (a <= -pi) a += 2 * pi;
    return a;
}
__device__ void residual_x(const real *a, const real *b, real *out)
{
    for (int i = 0; i < BKE_DIM_X; i++) out[i] = a[i] - b[i];
    out[2] = ctrv_wrap(out[2]);
}
__device__ void state_add(const real *a, const real *b, real *out)
{
    for (int i = 0; i < BKE_DIM_X; i++) out[i] = a[i] + b[i];
    out[2] = ctrv_wrap(out[2]);
}
__device__ void x_mean_fn(const real *sigmas, const real *Wm, real *out)
{
    real s = 0, c = 0;
    for (int i = 0; i < BKE_DIM_X; i++) out[i] = 0;
    for (int k = 0; k < BKE_N_SIGMAS; k++) {
        for (int i = 0; i < BKE_DIM_X; i++) if (i != 2) out[i] += Wm[k] * sigmas[k * BKE_DIM_X + i];
        s += Wm[k] * sin(sigmas[k * BKE_DIM_X + 2]);
        c += Wm[k] * cos(sigmas[k * BKE_DIM_X + 2]);
    }
    out[2] = atan2(s, c);
}
"""


def wrap_angle(a):
    """Into (-pi, pi] for differences of two angles in (-pi, pi] (the CUDA text's rb_wrap / ctrv_wrap)."""
    a = np.asarray(a, float)
    return np.where(a > np.pi, a - 2 * np.pi, np.where(a <= -np.pi, a + 2 * np.pi, a))


def rb_residual_z(a, b):
    d = np.array(a - b, float)          # 1-D, or the CKF's (2, 1) columns: row 1 is the bearing either way
    d[1] = wrap_angle(d[1])
    return d


def rb_z_mean(sigmas, Wm):
    return np.array([np.dot(Wm, sigmas[:, 0]), np.arctan2(np.dot(Wm, np.sin(sigmas[:, 1])), np.dot(Wm, np.cos(sigmas[:, 1])))])


def ctrv_fx(x, dt):
    psi, v, w = x[2], x[3], x[4]
    if abs(w) > 1e-4:
        px = x[0] + v / w * (np.sin(psi + w * dt) - np.sin(psi))
        py = x[1] + v / w * (np.cos(psi) - np.cos(psi + w * dt))
    else:
        px = x[0] + v * np.cos(psi) * dt
        py = x[1] + v * np.sin(psi) * dt
    return np.array([px, py, float(wrap_angle(psi + w * dt)), v, w])


def ctrv_rb_hx(x, sx, sy):
    dx, dy = x[0] - sx, x[1] - sy
    return np.array([np.sqrt(dx * dx + dy * dy), np.arctan2(dy, dx)])


def ctrv_residual_x(a, b):
    d = np.array(a - b, float)
    d[2] = wrap_angle(d[2])
    return d


def ctrv_state_add(a, b):
    s = np.array(a + b, float)
    s[2] = wrap_angle(s[2])
    return s


def ctrv_x_mean(sigmas, Wm):
    x = np.dot(Wm, sigmas)
    x[2] = np.arctan2(np.dot(Wm, np.sin(sigmas[:, 2])), np.dot(Wm, np.cos(sigmas[:, 2])))
    return x


def ukf_bank_rb_behind(N, seed=8080, steps=1, dt=1.0, dtype=np.float64):
    """(a) N constant-velocity targets (x, vx, y, vy) BEHIND a range / bearing sensor at the origin, each
    crossing the x axis (bearing +-pi) within ten steps."""
    rng = np.random.default_rng(seed)
    py = rng.uniform(-60, 60, N)
    vy = -np.sign(py) * rng.uniform(6, 14, N)
    xt = np.stack([rng.uniform(-400, -150, N), rng.uniform(-3, 3, N), py, vy], 1)
    x0 = xt + rng.standard_normal((N, 4)) * np.array([2, .5, 2, .5])
    P0 = np.zeros((N, 4, 4))
    P0[:, np.arange(4), np.arange(4)] = rng.uniform(1.0, 9.0, (N, 4))
    q = np.exp(rng.uniform(np.log(1e-3), np.log(1e-1), N))
    qb = q_white_noise_block(2, np.full(N, dt), q)
    Q = _block_diag([qb, qb])
    sig = np.array([1.0, 0.01])
    R = np.broadcast_to(np.diag(sig ** 2), (N, 2, 2)).copy()
    zs = np.zeros((steps, N, 2))
    for t in range(steps):
        xt = xt.copy()
        xt[:, 0::2] += dt * xt[:, 1::2]
        px, pyt = xt[:, 0], xt[:, 2]
        h = np.stack([np.sqrt(px * px + pyt * pyt), np.arctan2(pyt, px)], 1) + sig * rng.standard_normal((N, 2))
        h[:, 1] = wrap_angle(h[:, 1])
        zs[t] = h
    out = dict(x=x0, P=P0, Q=Q, R=R, zs=zs)
    return {k: np.ascontiguousarray(v, dtype=dtype) for k, v in out.items()}


def ukf_bank_ctrv(N, seed=6060, steps=1, dt=0.5, dtype=np.float64):
    """(b) N CTRV targets (px, py, heading, speed, yaw rate) whose heading crosses +-pi, seen by a range /
    bearing sensor at ``sensor``."""
    rng = np.random.default_rng(seed)
    sensor = np.array([-50.0, 20.0])
    xt = np.stack([rng.uniform(200, 600, N), rng.uniform(-200, 200, N), wrap_angle(np.pi + rng.uniform(-0.4, 0.4, N)),
                   rng.uniform(5, 15, N), rng.uniform(0.15, 0.35, N) * rng.choice([-1.0, 1.0], N)], 1)
    x0 = xt + rng.standard_normal((N, 5)) * np.array([2, 2, .05, .5, .02])
    x0[:, 2] = wrap_angle(x0[:, 2])
    P0 = np.zeros((N, 5, 5))
    P0[:, np.arange(5), np.arange(5)] = np.array([4, 4, .01, .25, .001]) * rng.uniform(1.0, 2.0, (N, 5))
    q = rng.uniform(0.5, 2.0, N)
    Q = np.zeros((N, 5, 5))
    Q[:, np.arange(5), np.arange(5)] = q[:, None] * np.array([.01, .01, 1e-4, .01, 1e-4]) * dt
    sig = np.array([1.5, 0.004])
    R = np.broadcast_to(np.diag(sig ** 2), (N, 2, 2)).copy()
    zs = np.zeros((steps, N, 2))
    for t in range(steps):
        xt = np.stack([ctrv_fx(xt[f], dt) for f in range(N)])
        zs[t] = np.stack([ctrv_rb_hx(xt[f], *sensor) for f in range(N)]) + sig * rng.standard_normal((N, 2))
    out = dict(x=x0, P=P0, Q=Q, R=R, zs=zs, sensor=sensor)
    return {k: np.ascontiguousarray(v, dtype=dtype) for k, v in out.items()}
