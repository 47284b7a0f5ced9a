"""fp64 NumPy restatement of the polynomial trackers (filterpy/gh/gh_filter.py, filterpy/leastsq/least_squares.py,
filterpy/memory/fading_memory.py), vectorised over a bank: every filter is one element of the arrays, and every
expression keeps the reference's operation order, so each element reproduces the reference object bit for bit
(NumPy's element-wise + - * / round each operation, as Python's float operations do).

``run(case)`` takes a golden case (tests/golden/make_golden_poly.py) and returns its outputs in the same layout.
The constants the reference derives from Python scalars (dt**2, h / dt, the beta powers) are evaluated the same way,
per filter, on Python floats (``consts``)."""
import numpy as np


def _py(fn, *arrs):
    return np.array([fn(*[float(v) for v in vals]) for vals in zip(*arrs)], np.float64)


def gh_update(x, dx, z, g, h, dt):
    """GHFilter.update, gh_filter.py:369-375"""
    dx_prediction = dx
    x_prediction = x + (dx * dt)
    y = z - x_prediction
    dx = dx_prediction + h * y / dt
    x = x_prediction + g * y
    return x, dx, y, x_prediction, dx_prediction


def gh_batch_step(x, dx, z, g, h_dt, dt):
    """GHFilter.batch_filter's loop body, gh_filter.py:437-442 (GHKFilter's :733-738 is the same)"""
    x_est = x + (dx * dt)
    residual = z - x_est
    dx = dx + h_dt * residual
    x = x_est + g * residual
    return x, dx, x_est


def ghk_update(x, dx, ddx, z, g, h, k, dt, dt_sqr):
    """GHKFilter.update, gh_filter.py:666-678"""
    ddx_prediction = ddx
    dx_prediction = dx + ddx * dt
    x_prediction = x + dx * dt + .5 * ddx * (dt_sqr)
    y = z - x_prediction
    ddx = ddx_prediction + 2 * k * y / dt_sqr
    dx = dx_prediction + h * y / dt
    x = x_prediction + g * y
    return x, dx, ddx, y, x_prediction, dx_prediction, ddx_prediction


def gho_update(order, X, z, g, h, k, dt, T2):
    """GHFilterOrder.update, gh_filter.py:142-181 (X[N, order+1]); returns (X, y)"""
    X = X.copy()
    if order == 0:
        y = z - X[:, 0]
        X[:, 0] = X[:, 0] + g * y
    elif order == 1:
        x, dx = X[:, 0], X[:, 1]
        dxdt = dx * dt
        y = z - (x + dxdt)
        X[:, 0], X[:, 1] = x + dxdt + g * y, dx + h * y / dt
    else:
        x, dx, ddx = X[:, 0], X[:, 1], X[:, 2]
        dxdt = dx * dt
        y = z - (x + dxdt + 0.5 * ddx * T2)
        X[:, 0] = x + dxdt + 0.5 * ddx * T2 + g * y
        X[:, 1] = dx + ddx * dt + h * y / dt
        X[:, 2] = ddx + 2 * k * y / T2          # / (self.dt**2): the same value as T2 = self.dt**2.
    return X, y


def lsq_update(order, X, n, z, dt, dt2, hdt2):
    """LeastSquaresFilter.update, least_squares.py:122-154 (X[N, order+1], n[N] int64 before the call); returns
    (X, n, K).  The int products stay int64 and meet the floats the way Python's int and float do."""
    X, n = X.copy(), n + 1
    K = np.zeros_like(X)
    if order == 0:
        K[:, 0] = 1. / n
        y = z - X[:, 0]
        X[:, 0] = X[:, 0] + K[:, 0] * y
    elif order == 1:
        K[:, 0] = 2. * (2 * n - 1) / (n * (n + 1)).astype(np.float64)
        K[:, 1] = 6. / ((n * (n + 1)).astype(np.float64) * dt)
        x0, x1 = X[:, 0], X[:, 1]
        y = z - x0 - (dt * x1)
        X[:, 0] = x0 + ((K[:, 0] * y) + (dt * x1))
        X[:, 1] = x1 + (K[:, 1] * y)
    else:
        den = (n * (n + 1) * (n + 2)).astype(np.float64)
        K[:, 0] = 3. * (3 * n**2 - 3 * n + 2) / den
        K[:, 1] = 18. * (2 * n - 1) / (den * dt)
        K[:, 2] = 60. / (den * dt2)
        x0, x1, x2 = X[:, 0], X[:, 1], X[:, 2]
        y = z - x0 - (dt * x1) - (hdt2 * x2)
        X[:, 0] = x0 + ((K[:, 0] * y) + (x1 * dt) + (hdt2 * x2))
        X[:, 1] = x1 + ((K[:, 1] * y) + (x2 * dt))
        X[:, 2] = x2 + (K[:, 2] * y)
    return X, n, K


def fm_update(order, X, z, G, H_dt, K2_dt2, dt, T2):
    """FadingMemoryFilter.update, fading_memory.py:164-194, with G, H / dt and 2*K / dt**2 per order"""
    X = X.copy()
    if order == 0:
        X[:, 0] = X[:, 0] + G * (z - X[:, 0])
    elif order == 1:
        x, dx = X[:, 0], X[:, 1]
        dxdt = dx * dt
        residual = z - (x + dxdt)
        X[:, 0], X[:, 1] = x + dxdt + G * residual, dx + H_dt * residual
    else:
        x, dx, ddx = X[:, 0], X[:, 1], X[:, 2]
        dxdt = dx * dt
        residual = z - (x + dxdt + 0.5 * ddx * T2)
        X[:, 0] = x + dxdt + 0.5 * ddx * T2 + G * residual
        X[:, 1] = dx + ddx * dt + H_dt * residual
        X[:, 2] = ddx + K2_dt2 * residual
    return X


def consts(c):
    """the constants of case c, each from Python floats with the reference's expression"""
    fam, order = str(c["family"]), int(c["order"])
    dt, h, beta = c["dt"], c["h"], c["beta"]
    out = dict(dt2=_py(lambda d: d**2, dt))                                    # gh_filter.py:667, :175 (dt**2.)
    if fam in ("gh", "ghk"):
        out["h_dt"] = _py(lambda a, d: a / d, h, dt)                            # :433, :729
    if fam == "lsq":
        out["hdt2"] = _py(lambda d: 0.5 * d**2, dt)                             # least_squares.py:150
    if fam == "fm":
        G = {0: lambda b: 1 - b, 1: lambda b: 1 - b**2, 2: lambda b: 1 - b**3}[order]
        out["G"] = _py(G, beta)                                                 # fading_memory.py:165, 169, 180
        if order == 1:
            out["H_dt"] = _py(lambda b, d: (1 - b)**2 / d, beta, dt)            # :170, :177
        if order == 2:
            out["H_dt"] = _py(lambda b, d: 1.5 * (1 + b) * (1 - b)**2 / d, beta, dt)       # :181, :193
            out["K2_dt2"] = _py(lambda b, d: 2 * (0.5 * (1 - b)**3) / (d**2), beta, dt)    # :182, :194
    return out


def run(c):
    """every output the golden case c stores, from its inputs"""
    fam, order = str(c["family"]), int(c["order"])
    zs, x0 = c["zs"], c["x0"]
    T, N = zs.shape
    k = consts(c)
    g, h, kk, dt = c["g"], c["h"], c["k"], c["dt"]
    st = [x0.copy()]
    y, xp, dxp, ddxp, zz, K = [], [], [], [], [], []
    X = x0.copy()
    n = np.zeros(N, np.int64)
    for t in range(T):
        z = zs[t]
        if fam == "gh":
            x, dx, yy, a, b = gh_update(X[:, 0], X[:, 1], z, g, h, dt)
            X = np.stack([x, dx], 1)
            y.append(yy); xp.append(a); dxp.append(b)
        elif fam == "ghk":
            x, dx, ddx, yy, a, b, cc = ghk_update(X[:, 0], X[:, 1], X[:, 2], z, g, h, kk, dt, k["dt2"])
            X = np.stack([x, dx, ddx], 1)
            y.append(yy); xp.append(a); dxp.append(b); ddxp.append(cc)
        elif fam == "gho":
            X, yy = gho_update(order, X, z, g, h, kk, dt, k["dt2"])
            y.append(yy)
            zz.append(z if order == 1 else np.zeros(N))                          # gh_filter.py:161
        elif fam == "lsq":
            X, n, KK = lsq_update(order, X, n, z, dt, k["dt2"], k.get("hdt2"))
            K.append(KK)
        else:
            X = fm_update(order, X, z, k["G"], k.get("H_dt"), k.get("K2_dt2"), dt, k["dt2"])
        st.append(X.copy())
    snap = c["snap"]
    ep = snap[1:] - 1
    out = dict(upd_state=np.array(st)[snap])
    for name, v in (("upd_y", y), ("upd_xp", xp), ("upd_dxp", dxp), ("upd_ddxp", ddxp), ("upd_z", zz), ("upd_K", K)):
        if v:
            out[name] = np.array(v)[ep]
    if fam in ("gh", "ghk"):
        x, dx = x0[:, 0], x0[:, 1]
        res, pred = [np.stack([x, dx], 1)], []
        for t in range(T):
            x, dx, x_est = gh_batch_step(x, dx, zs[t], g, k["h_dt"], dt)
            res.append(np.stack([x, dx], 1))
            pred.append(x_est)
        out["bat_res"], out["bat_pred"] = np.array(res)[snap], np.array(pred)[ep]
    return out

