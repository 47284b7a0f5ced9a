"""fp64 NumPy restatement of the polynomial trackers (filterpy/gh/gh_filter.py, filterpy/leastsq/least_squares.py,
filterpy/memory/fading_memory.py), vectorised over a bank: every filter is one element of the arrays, and every
expression keeps the reference's operation order, so each element reproduces the reference object bit for bit
(NumPy's element-wise + - * / round each operation, as Python's float operations do).

``run(case)`` takes a golden case (tests/golden/make_golden_poly.py) and returns its outputs in the same layout.
The constants the reference derives from Python scalars (dt**2, h / dt, the beta powers) are evaluated the same way,
per filter, on Python floats (``consts``).

The update functions take a ``dtype``.  float64 (the default) is the reference.  float32 is the twin of the kernel's
fp32 instances (csrc/poly.cu), which run the same sequence of explicitly rounded operations in fp32: the caller passes
float32 arrays, every constant is a float32 and every operation rounds to float32, so the twin matches the kernel
bit for bit.  The LSQ gains convert the exact int64 products with ``astype(dtype)``, one rounding as __ll2float_rn
(going through a Python float would round twice).  ``bank`` runs n_steps epochs of one bke_poly_filter call."""
import numpy as np


def _py(fn, *arrs):
    return np.array([fn(*[float(v) for v in vals]) for vals in zip(*arrs)], np.float64)


def gh_update(x, dx, z, g, h, dt, dtype=np.float64):
    """GHFilter.update, gh_filter.py:369-375 (no constant: dtype is the arrays')"""
    dx_prediction = dx
    x_prediction = x + (dx * dt)
    y = z - x_prediction
    dx = dx_prediction + h * y / dt
    x = x_prediction + g * y
    return x, dx, y, x_prediction, dx_prediction


def gh_batch_step(x, dx, z, g, h_dt, dt, dtype=np.float64):
    """GHFilter.batch_filter's loop body, gh_filter.py:437-442 (GHKFilter's :733-738 is the same; no constant:
    dtype is the arrays')"""
    x_est = x + (dx * dt)
    residual = z - x_est
    dx = dx + h_dt * residual
    x = x_est + g * residual
    return x, dx, x_est


def ghk_update(x, dx, ddx, z, g, h, k, dt, dt_sqr, dtype=np.float64):
    """GHKFilter.update, gh_filter.py:666-678"""
    T = dtype
    ddx_prediction = ddx
    dx_prediction = dx + ddx * dt
    x_prediction = x + dx * dt + T(.5) * ddx * (dt_sqr)
    y = z - x_prediction
    ddx = ddx_prediction + T(2) * k * y / dt_sqr
    dx = dx_prediction + h * y / dt
    x = x_prediction + g * y
    return x, dx, ddx, y, x_prediction, dx_prediction, ddx_prediction


def gho_update(order, X, z, g, h, k, dt, T2, dtype=np.float64):
    """GHFilterOrder.update, gh_filter.py:142-181 (X[N, order+1]); returns (X, y)"""
    T = dtype
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
        y = z - (x + dxdt + T(0.5) * ddx * T2)
        X[:, 0] = x + dxdt + T(0.5) * ddx * T2 + g * y
        X[:, 1] = dx + ddx * dt + h * y / dt
        X[:, 2] = ddx + T(2) * k * y / T2       # / (self.dt**2): the same value as T2 = self.dt**2.
    return X, y


def lsq_update(order, X, n, z, dt, dt2, hdt2, dtype=np.float64):
    """LeastSquaresFilter.update, least_squares.py:122-154 (X[N, order+1], n[N] int64 before the call); returns
    (X, n, K).  The int products stay int64 and meet the floats the way Python's int and float do: one
    round-to-nearest conversion each (``astype``)."""
    T = dtype
    X, n = X.copy(), n + 1
    K = np.zeros_like(X)
    if order == 0:
        K[:, 0] = T(1.) / n.astype(T)
        y = z - X[:, 0]
        X[:, 0] = X[:, 0] + K[:, 0] * y
    elif order == 1:
        K[:, 0] = T(2.) * (2 * n - 1).astype(T) / (n * (n + 1)).astype(T)
        K[:, 1] = T(6.) / ((n * (n + 1)).astype(T) * dt)
        x0, x1 = X[:, 0], X[:, 1]
        y = z - x0 - (dt * x1)
        X[:, 0] = x0 + ((K[:, 0] * y) + (dt * x1))
        X[:, 1] = x1 + (K[:, 1] * y)
    else:
        den = (n * (n + 1) * (n + 2)).astype(T)
        K[:, 0] = T(3.) * (3 * n**2 - 3 * n + 2).astype(T) / den
        K[:, 1] = T(18.) * (2 * n - 1).astype(T) / (den * dt)
        K[:, 2] = T(60.) / (den * dt2)
        x0, x1, x2 = X[:, 0], X[:, 1], X[:, 2]
        y = z - x0 - (dt * x1) - (hdt2 * x2)
        X[:, 0] = x0 + ((K[:, 0] * y) + (x1 * dt) + (hdt2 * x2))
        X[:, 1] = x1 + ((K[:, 1] * y) + (x2 * dt))
        X[:, 2] = x2 + (K[:, 2] * y)
    return X, n, K


def fm_update(order, X, z, G, H_dt, K2_dt2, dt, T2, dtype=np.float64):
    """FadingMemoryFilter.update, fading_memory.py:164-194, with G, H / dt and 2*K / dt**2 per order"""
    T = dtype
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
        residual = z - (x + dxdt + T(0.5) * ddx * T2)
        X[:, 0] = x + dxdt + T(0.5) * ddx * T2 + G * residual
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



# ---------------------------------------------------------------------------------------------- one kernel call
FAMILY = {0: "gh", 1: "ghk", 2: "gho", 3: "lsq", 4: "fm"}       # include/bke.h BKE_POLY_GH .. BKE_POLY_FADING


def bank(family, order, batch, X, zs, p, n=None, dtype=np.float64):
    """One bke_poly_filter call in ``dtype``: family a BKE_POLY_* value, batch its mode BKE_POLY_BATCH, X[N, S] the
    state (x, dx for GH; x, dx, ddx for GHK; order + 1 columns otherwise), zs[T, N], p the kernel's parameters by name
    (g, h, k, dt, dt2, hdt2: [N] arrays or None for one the instance does not read; for GH and GHK batch h is h / dt,
    for FADING g, h and k are G, H / dt and 2*K / dt**2), n[N] the int64 LSQ counters.  Returns results[T+1, N, W]
    and the last epoch's state ``X`` (and LSQ ``n``), y, x/dx/ddx_prediction and K, and for GH / GHK batch
    predictions[T, N]."""
    fam = FAMILY[family]
    T = dtype
    g, h, k, dt, dt2, hdt2 = (p.get(name) for name in ("g", "h", "k", "dt", "dt2", "hdt2"))
    gh_like = fam in ("gh", "ghk")
    X = X.copy()
    W = 2 if gh_like else X.shape[1]
    res, out = [X[:, :W].copy()], {}
    if gh_like and batch:                            # GHKFilter.batch_filter is GHFilter's recursion
        x, dx, pred = X[:, 0], X[:, 1], []
        for z in zs:
            x, dx, x_est = gh_batch_step(x, dx, z, g, h, dt, T)
            res.append(np.stack([x, dx], 1))
            pred.append(x_est)
        out.update(results=np.array(res), predictions=np.array(pred), X=X)
        return out
    for z in zs:
        if fam == "gh":
            x, dx, out["y"], out["x_prediction"], out["dx_prediction"] = gh_update(X[:, 0], X[:, 1], z, g, h, dt, T)
            X = np.stack([x, dx], 1)
        elif fam == "ghk":
            x, dx, ddx, out["y"], out["x_prediction"], out["dx_prediction"], out["ddx_prediction"] = ghk_update(
                X[:, 0], X[:, 1], X[:, 2], z, g, h, k, dt, dt2, T)
            X = np.stack([x, dx, ddx], 1)
        elif fam == "gho":
            X, out["y"] = gho_update(order, X, z, g, h, k, dt, dt2, T)
        elif fam == "lsq":
            X, n, out["K"] = lsq_update(order, X, n, z, dt, dt2, hdt2, T)
        else:
            X = fm_update(order, X, z, g, h, k, dt, dt2, T)
        res.append(X[:, :W].copy())
    out.update(results=np.array(res), X=X)
    if fam == "lsq":
        out["n"] = n
    return out
