"""Every kernel instance behind bke_enkf_step and bke_enkf_initialize against the fp64 oracle (oracle/enkf.py), through
the C-ABI, with a table that names the kernel each case launches.

bke_enkf_step (csrc/enkf.cu) runs enkf_kernel<T, N, M, FX, HX, EXTRAS> for every (N, M, FX, HX) row of
BKE_SIGMA_INSTANCES (sigma_launch.cuh), EXTRAS = false when x_prior, P_prior, K, S and SI are all NULL.  One warp per
filter, EW filters per CTA; a CTA's ensembles sit in dynamic shared memory when EW * members * (N | 1) elements fit in
ENKF_SMEM_MAX bytes (above 48 KB near the limit), otherwise the passes run over sigmas_out in global memory, after a
copy-in when sigmas_out is not sigmas.  bke_enkf_initialize runs enkf_init_kernel<T, N> for N = 1..16.  CASES runs
every one of them, each step instance at the largest on-chip member count and one above it.

Each launch is compared with the oracle started from that launch's inputs: the first from inputs rounded to the
kernel's dtype, the next two from the outputs of the launch before as they were read back, so no error carries over.
The oracle draws with Stream(seed, filter, dtype): the fp32 kernel forms its uniforms from 24 bits of one word, which
the fp64 stream does not reproduce in the tails.  Every output starts as a finite sentinel inside NaN guards, so a
write outside an array, a missing write, or one to an output that must be left alone shows up.

Error measure, per filter:
- members, x and x_prior: against the member scale sx (the largest |entry| of the filter's members in and out);
- P: against the prior P an update subtracted K S K' from (at 2 members most of it cancels), else its own;
  P and P_prior through _cov_scale, max(|P|, sx sqrt|P|): centring members of size sx rounds at eps sx, which a
  spread far below the members' size (2 members after an update) multiplies;
- K, S and SI in measurement units of one standard deviation sqrt(S_aa) each (K D, D^-1 S D^-1, D SI D), so a range
  in metres and angles in radians are measured on one scale; S through _cov_scale with the size of z in those units;
- everything that solves with S (members and x after an update, P, K, SI) divided by cond(D^-1 S D^-1) of the
  filter's update, the condition of the solve rather than of the units; 1 where the filter does not update.

Worst cases measured on an H100 80GB HBM3 (700 W power limit) with BKE_TEST_ERRLOG over every case, output and launch
of the family, and the bound set from each (pair_gain: K and SI at 2 members, where the gain is formed from a spread
that the previous update collapsed; every other output at 2 members is "pair"):

    family                                   fp64 worst  bound     fp32 worst  bound
    onchip     5+ members, shared memory       2.9e-15    1.2e-14   2.5e-6     1e-5
    global     5+ members, global memory       7.8e-15    3e-14     9.2e-7     4e-6
    pair       2 members (on chip)             1.7e-15    7e-15     5.8e-6     2.5e-5
    pair_gain  K and SI at 2 members           1.1e-13    4.5e-13   2.6e-4     1e-3
    init       enkf_init_kernel                3.9e-16    1.5e-15   1.1e-7     5e-7
"""
import ctypes
import re

import numpy as np
import pytest

from gpu_harness import (F32, F64, SIGMA_DT, SIGMA_FX, SIGMA_HX, TNAME, Bufs, b, body, call, check_launch_order, close,
                         mag, profiled_names, ptr, rd, sigma_problem, spd, src)

EW = 4                                           # enkf_kernel.cuh: warps (= filters) per CTA
SMEM_MAX = 64 * 1024                             # sigma_launch.cuh ENKF_SMEM_MAX
DT, FX, HX = SIGMA_DT, SIGMA_FX, SIGMA_HX        # the models of gpu_harness.sigma_problem (include/bke.h ids)
OK, SINGULAR_S, NOT_PD = 0, 1, 2
EXTRAS = ("x_prior", "P_prior", "K", "S", "SI")
# the pre-built (dim_x, dim_z, fx, hx) rows of BKE_SIGMA_INSTANCES, in dispatch order
INSTANCES = [
    (6, 3, "CONST_VEL", "RANGE_AZ_EL"), (6, 3, "CONST_VEL", "LINEAR"), (6, 3, "LINEAR", "LINEAR"),
    (6, 3, "LINEAR", "RANGE_AZ_EL"), (4, 2, "CONST_VEL", "RANGE_BEARING"), (4, 2, "LINEAR", "RANGE_BEARING"),
    (4, 2, "CONST_VEL", "LINEAR"), (4, 2, "LINEAR", "LINEAR"), (1, 1, "LINEAR", "LINEAR"), (2, 1, "LINEAR", "LINEAR"),
    (2, 1, "CONST_VEL", "LINEAR"), (2, 2, "LINEAR", "LINEAR"), (3, 1, "LINEAR", "LINEAR"), (3, 3, "LINEAR", "LINEAR"),
    (4, 4, "LINEAR", "LINEAR"),
]

TOL = {
    "onchip": {F64: 1.2e-14, F32: 1e-5},
    "global": {F64: 3e-14, F32: 4e-6},
    "pair": {F64: 7e-15, F32: 2.5e-5},
    "pair_gain": {F64: 4.5e-13, F32: 1e-3},
    "init": {F64: 1.5e-15, F32: 5e-7},
}


def smem_bytes(n, members, dt):
    """sigma_launch.cuh enkf_smem_bytes before the cap: the CTA's EW ensembles at the odd member stride n | 1."""
    return EW * members * (n | 1) * np.dtype(dt).itemsize


def max_onchip(n, dt):
    """The largest member count whose ensembles a CTA stages in shared memory."""
    return SMEM_MAX // (EW * (n | 1) * np.dtype(dt).itemsize)


def k_step(dt, n, m, fx, hx, extras):
    return "enkf_kernel<%s, %d, %d, %d, %d, %s>" % (TNAME[dt], n, m, FX[fx], HX[hx], b(extras))


def k_init(dt, n):
    return "enkf_init_kernel<%s, %d>" % (TNAME[dt], n)


# ------------------------------------------------------------------------------------------ the instance table
class Cfg:
    """One run of a step case: N filters of `members`, models per filter or shared (stride 0), one flag set per
    launch ("p", "u", "pu"), the first launch's draw counter and the seed; `outs` the optional outputs passed
    (status too unless no_status); `alias` sigmas_out = sigmas, `alias_xp` x_out = x and P_out = P; `mis` every
    array one element past a 16-byte boundary; `mask` ~20 % of z_valid 0 (else z_valid NULL); `fails` a filter
    with each failure (indefinite Q, indefinite R, singular S) and with rank-deficient Q and R, and Q = 0.
    For an init case: N filters, `members`, the seed and counter, status passed or not."""

    def __init__(self, N, members, shared=False, flags=("pu", "p", "u"), counter=0, seed=0, outs=(), alias=False,
                 alias_xp=False, mis=False, mask=True, fails=False, no_status=False):
        self.N, self.members, self.shared, self.flags, self.counter, self.seed = N, members, shared, flags, counter, seed
        self.outs, self.alias, self.alias_xp, self.mis, self.mask, self.fails = tuple(outs), alias, alias_xp, mis, mask, fails
        self.no_status = no_status

    def __repr__(self):
        return "N=%d members=%d%s flags=%s counter=%#x seed=%#x outs=%s%s%s%s%s%s" % (
            self.N, self.members, " shared" if self.shared else "", "/".join(self.flags), self.counter, self.seed,
            ",".join(self.outs) or "-", " alias" if self.alias else "", " alias_xp" if self.alias_xp else "",
            " mis" if self.mis else "", " fails" if self.fails else "", " no_status" if self.no_status else "")


class Case:
    """A step instance (kind "step": inst = (n, m, fx, hx), extras) or an init instance (kind "init": n)."""

    def __init__(self, kind, dt, inst, extras, cfgs):
        self.kind, self.dt, self.inst, self.extras, self.cfgs = kind, dt, inst, extras, list(cfgs)

    @property
    def n(self):
        return self.inst[0] if self.kind == "step" else self.inst

    @property
    def id(self):
        d = "f32" if self.dt == F32 else "f64"
        if self.kind == "init":
            return "init-%s-%d" % (d, self.inst)
        n, m, fx, hx = self.inst
        return "step-%s-%d_%d_%s_%s-%s" % (d, n, m, fx.lower(), hx.lower(), "extras" if self.extras else "plain")

    def kernels(self):
        if self.kind == "init":
            return [k_init(self.dt, self.inst)]
        return [k_step(self.dt, *self.inst, self.extras)]

    def onchip(self, g):
        return smem_bytes(self.n, g.members, self.dt) <= SMEM_MAX


ARB = 0x9E3779B9                                 # an arbitrary counter
TOP = 0xFFFFFFFF


def _step_cfgs(i, dt, n, extras):
    """Case i's runs: 2 members (rank-one covariances) in a bank of 37 (the last CTA holds one filter) with every
    failure; 5, 32 or 33 members per filter with counter 0xFFFFFFFF (the fused update draws with call 0) and in a
    bank of 5 with shared models; the largest on-chip member count (> 48 KB of shared memory) in a bank of 4; one
    more member (the global path) in banks of 1 and 5.  The optional outputs rotate over all five, each alone and
    none; sigmas_out is sigmas and separate on both paths."""
    mx = max_onchip(n, dt)
    one = lambda k: (EXTRAS[k % 5],) if extras else ()                                       # noqa: E731
    every = EXTRAS if extras else ()
    small = (5, 32, 33)
    return [
        Cfg(37, 2, flags=("pu", "p", "u"), counter=ARB, seed=0, outs=every, fails=True),
        Cfg(37, small[i % 3], flags=("pu", "u", "p"), counter=TOP, seed=TOP, outs=one(i), alias=True, alias_xp=True,
            fails=True, no_status=True),
        Cfg(5, small[(i + 1) % 3], shared=True, flags=("p", "pu", "u"), counter=0, seed=TOP, outs=one(i + 1),
            mis=(i % 4 == 0), mask=False),
        Cfg(4, mx, flags=("pu", "u", "pu"), counter=ARB, seed=0, outs=every, alias=(i % 2 == 1)),
        Cfg(1, mx + 1, shared=True, flags=("pu", "p", "u"), counter=TOP, seed=TOP, outs=one(i + 3)),
        Cfg(5, mx + 1, flags=("u", "pu", "pu"), counter=0, seed=0, outs=every, alias=True, alias_xp=True,
            mis=(i % 4 == 2)),
    ]


def _init_cfgs(n):
    return [Cfg(7, 33, counter=ARB, seed=0), Cfg(5, 2, counter=TOP, seed=TOP, no_status=True),
            Cfg(3, 1000 + n, counter=0, seed=TOP), Cfg(1, 33, counter=1, seed=0, mis=True)]


def _cases():
    out, i = [], 0
    for dt in (F64, F32):
        for inst in INSTANCES:
            for extras in (True, False):
                out.append(Case("step", dt, inst, extras, _step_cfgs(i, dt, inst[0], extras)))
                i += 1
    for dt in (F64, F32):
        for n in range(1, 17):
            out.append(Case("init", dt, n, False, _init_cfgs(n)))
    return out


CASES = _cases()
STEPS = [c for c in CASES if c.kind == "step"]
INITS = [c for c in CASES if c.kind == "init"]


# ------------------------------------------------------------------------------------------ the table vs the source
def _source_table():
    """BKE_SIGMA_INSTANCES, EW and ENKF_SMEM_MAX as the sources define them."""
    text = src("sigma_launch.cuh")
    table = re.search(r"#define BKE_SIGMA_INSTANCES\(X\)((?:.*\\\n)*.*)", text).group(1)
    rows = [(int(n), int(m), fx, hx) for n, m, fx, hx in
            re.findall(r"\w+\(\s*(\d+)\s*,\s*(\d+)\s*,\s*BKE_FX_(\w+)\s*,\s*BKE_HX_(\w+)\s*\)", table)]
    smem = re.search(r"constexpr size_t ENKF_SMEM_MAX = ([\d\s*]+);", text).group(1)
    smem_max = int(np.prod([int(v) for v in smem.split("*")]))
    ew = int(re.search(r"constexpr int EW = (\d+);", src("enkf_kernel.cuh")).group(1))
    assert "const size_t b = (size_t)enkfk::EW * (size_t)n_members * (size_t)(n | 1) * elem;" in text
    assert "return b <= ENKF_SMEM_MAX ? b : 0;" in text
    assert "return a.x_prior || a.P_prior || a.K || a.S || a.SI;" in body(text, "inline bool enkf_has_extras(")
    enkf = src("enkf.cu")
    assert ("enkf_has_extras(a) ? enkf_kernel<T, N, M, FX, HX, true> : enkf_kernel<T, N, M, FX, HX, false>"
            in body(enkf, "int launch_inst(const bke_enkf_args &a, cudaStream_t s)"))
    assert re.search(r"^\s*BKE_SIGMA_INSTANCES\(BKE_SIGMA_DISPATCH_ROW\)", enkf, re.M)
    inits = [int(v) for v in re.findall(r"BKE_ENKF_INIT\((\d+)\)\s", body(enkf, "int init_dispatch("))]
    return rows, ew, smem_max, inits


def test_cases_cover_every_instance_on_both_sides_of_the_onchip_limit():
    """CASES runs every enkf_kernel instance (each BKE_SIGMA_INSTANCES row x dtype x EXTRAS) at the largest member
    count whose ensembles fit in ENKF_SMEM_MAX and at one more, plus 2, 5, 32 and 33 members, banks of 1, 4, 5 and
    37, each flag set, counters 0 / arbitrary / 0xFFFFFFFF and seeds 0 / 0xFFFFFFFF, shared and per-filter models,
    each optional output alone, all and none, both sigmas_out layouts on both paths; and enkf_init_kernel for every
    dim_x 1..16 the dispatch builds.  A row added to the table, or a moved shared-memory limit, fails here on a
    machine without a GPU."""
    rows, ew, smem_max, inits = _source_table()
    assert rows == INSTANCES and ew == EW and smem_max == SMEM_MAX
    lim = lambda n, dt: smem_max // (ew * (n | 1) * np.dtype(dt).itemsize)                   # noqa: E731
    assert lim(1, F32) == 4096 and lim(6, F64) == 292
    on = lambda n, k, dt: ew * k * (n | 1) * np.dtype(dt).itemsize <= smem_max              # noqa: E731
    want = {(dt, r, ex) for dt in (F32, F64) for r in rows for ex in (True, False)}
    assert {(c.dt, c.inst, c.extras) for c in STEPS} == want and len(STEPS) == len(want)
    for c in STEPS:
        n, mx = c.n, lim(c.n, c.dt)
        counts = {g.members for g in c.cfgs}
        assert {2, mx, mx + 1} <= counts, c.id
        assert on(n, mx, c.dt) and not on(n, mx + 1, c.dt), c.id
        assert smem_bytes(n, mx, c.dt) > 48 * 1024, c.id
        for alias in (False, True):
            assert any(g.alias == alias and on(n, g.members, c.dt) for g in c.cfgs), c.id
            assert any(g.alias == alias and not on(n, g.members, c.dt) for g in c.cfgs), c.id
        assert {1, 4, 5, 37} == {g.N for g in c.cfgs}
        assert {"p", "u", "pu"} == {f for g in c.cfgs for f in g.flags}
        assert {0, ARB, TOP} == {g.counter for g in c.cfgs} and {0, TOP} == {g.seed for g in c.cfgs}
        assert any(g.counter == TOP and g.flags[0] == "pu" for g in c.cfgs)
        assert {True, False} == {g.shared for g in c.cfgs} == {g.no_status for g in c.cfgs}
        assert any(g.alias_xp for g in c.cfgs) and any(g.fails for g in c.cfgs) and any(g.mask for g in c.cfgs)
        outs = {g.outs for g in c.cfgs}
        assert (EXTRAS in outs and any(len(k) == 1 for k in outs)) if c.extras else outs == {()}, c.id
    for r in rows:
        assert {5, 32, 33} <= {g.members for c in STEPS if c.inst == r for g in c.cfgs}, r
    singles = {g.outs for c in STEPS for g in c.cfgs if len(g.outs) == 1}
    assert singles == {(k,) for k in EXTRAS}
    assert any(g.mis for c in STEPS for g in c.cfgs)
    assert inits == list(range(1, 17))
    assert {(c.dt, c.n) for c in INITS} == {(dt, n) for dt in (F32, F64) for n in inits} and len(INITS) == 32
    for c in INITS:
        assert {2, 33} <= {g.members for g in c.cfgs} and max(g.members for g in c.cfgs) >= 1000
        assert any(g.N % EW for g in c.cfgs) and any(g.no_status for g in c.cfgs)


# ------------------------------------------------------------------------------------------ inputs
def _fail_rows(g, c):
    """Filter -> failure of a cfg with fails: indefinite Q, indefinite R, singular S, rank-deficient Q, rank-deficient
    R, Q = 0; one in the part-empty last CTA.  Singular S: H = 0 and R = 0 at a linear hx; at a range hx a collapsed
    ensemble (every member at x, Q = 0) with R = 0, which only at 2 members keeps the mean of its hx values exactly
    equal to them.  A rank-deficient R measures some direction perfectly: the update leaves no spread there, and an
    update that follows it without a predict in between has a singular S (in exact arithmetic; in rounding, any
    status), so that filter is planted only in runs where a predict comes between two updates."""
    if not g.fails:
        return {}
    rows = {5: "q_indef", 10: "r_indef", 22: "q_rank", 36: "q_zero"}
    if c.inst[3] == "LINEAR" or g.members == 2:
        rows[17] = "singular"
    if not any(g.flags[t] == "u" and "u" in g.flags[t - 1] for t in range(1, len(g.flags))):
        rows[29] = "r_rank"
    return rows


def _rank_one_blocks(rng, k):
    """A k x k PSD matrix of rank k // 2: rank-one 2 x 2 blocks u u' on the diagonal (as Q_discrete_white_noise
    builds them), 0 in the last row and column of an odd k.  Rounding leaves each block's second pivot within a
    few eps of max diag, far inside psd_factor's 16 k eps."""
    C = np.zeros((k, k))
    for i in range(0, k - 1, 2):
        u = rng.uniform(0.5, 1.5, 2) * rng.choice([-1.0, 1.0], 2)
        C[i:i + 2, i:i + 2] = np.outer(u, u)
    return C


def step_inputs(c, g, seed):
    """x, P, members, models (per filter or shared), z per launch and the masks, rounded to the kernel's dtype."""
    n, m, fx, hx = c.inst
    pr = sigma_problem(*c.inst, N=g.N, T=3, seed=seed)
    rng = np.random.default_rng(seed + 1)
    mats = {k: (None if v is None else v.copy()) for k, v in pr["shared" if g.shared else "per"].items()}
    x, P = pr["x"], pr["P"]
    sig = x[:, None, :] + rng.standard_normal((g.N, g.members, n)) @ np.swapaxes(np.linalg.cholesky(P), 1, 2)
    valid = pr["valid"] if g.mask else np.ones((3, g.N), bool)
    fails = _fail_rows(g, c)
    for f, kind in fails.items():
        if kind == "q_indef":
            mats["Q"][f] = -mats["Q"][f]
        elif kind == "r_indef":
            mats["R"][f] = -mats["R"][f]
        elif kind == "singular":
            mats["R"][f] = 0
            if hx == "LINEAR":
                mats["H"][f] = 0
            else:
                sig[f] = x[f]
                mats["Q"][f] = 0
        elif kind == "q_rank":
            mats["Q"][f] = 0.1 * _rank_one_blocks(rng, n)
        elif kind == "r_rank":                      # rank m - 1: at 2 members S = (rank one) + R is regular
            mats["R"][f] = 0.5 * _rank_one_blocks(rng, m)
            mats["R"][f][2:, 2:] += np.diag(rng.uniform(0.5, 1.5, max(m - 2, 0)))
        elif kind == "q_zero":
            mats["Q"][f] = 0
        valid[:, f] = True
    d = dict(x=x, P=P, sig=sig, zs=pr["zs"], **{k: v for k, v in mats.items() if v is not None})
    d = {k: rd(v, c.dt) for k, v in d.items()}
    d["valid"] = valid.astype(np.uint8)
    return d, fails


# ------------------------------------------------------------------------------------------ the C-ABI call
def run_step(c, g, d, state, t):
    """One bke_enkf_step launch (flags g.flags[t], counter of launch t) from state = (x, P, members): (outputs
    host-side, Bufs)."""
    from filterpy_b200 import _lib
    n, m, fx, hx = c.inst
    N, Nm, dt = g.N, g.members, c.dt
    flags = g.flags[t]
    bf = Bufs(dt)
    a = _lib.EnkfArgs()
    a.n_filters, a.dim_x, a.dim_z, a.n_members = N, n, m, Nm
    a.dtype = _lib.BKE_F32 if dt == F32 else _lib.BKE_F64
    a.flags = (_lib.BKE_DO_PREDICT if "p" in flags else 0) | (_lib.BKE_DO_UPDATE if "u" in flags else 0)
    a.fx_model, a.hx_model = FX[fx], HX[hx]
    a.seed, a.counter, a.dt = g.seed, launch_counter(g, t), DT
    x, P, sig = state
    if g.alias_xp:
        xb, Pb = bf.put(x, g.mis, out=True), bf.put(P, g.mis, out=True)
        xo, Po = xb, Pb
    else:
        xb, Pb = bf.put(x, g.mis), bf.put(P, g.mis)
        xo, Po = bf.out((N, n), g.mis), bf.out((N, n, n), g.mis)
    a.x, a.P, a.x_out, a.P_out = ptr(xb), ptr(Pb), ptr(xo), ptr(Po)
    if g.alias:
        sb = bf.put(sig, g.mis, out=True)
        so = sb
    else:
        sb, so = bf.put(sig, g.mis), bf.out((N, Nm, n), g.mis)
    a.sigmas, a.sigmas_out = ptr(sb), ptr(so)
    for name, k in (("Q", n), ("R", m), ("F", n), ("H", n)):
        if name in d:
            arr = d[name]
            setattr(a, name, ptr(bf.put(arr, g.mis)))
            setattr(a, name + "_stride", 0 if arr.ndim == 2 else arr.shape[-1] * arr.shape[-2])
    a.z = ptr(bf.put(d["zs"][t], g.mis))
    if g.mask:
        a.z_valid = ptr(bf.put(d["valid"][t], g.mis, dtype=np.uint8))
    shapes = dict(x_prior=(N, n), P_prior=(N, n, n), K=(N, n, m), S=(N, m, m), SI=(N, m, m))
    outs = {k: bf.out(shapes[k], g.mis) for k in g.outs}
    for k, v in outs.items():
        setattr(a, k, ptr(v))
    st = None if g.no_status else bf.out((N,), g.mis, dtype=np.int32, fill=-7)
    a.status = ptr(st)
    rc, err = call("bke_enkf_step", ctypes.byref(a))
    assert rc == 0, err
    got = dict(x=xo.cpu().numpy().reshape(N, n), P=Po.cpu().numpy().reshape(N, n, n),
               sig=so.cpu().numpy().reshape(N, Nm, n), sig_in=sb.cpu().numpy().reshape(N, Nm, n))
    for k, v in outs.items():
        got[k] = v.cpu().numpy().reshape(shapes[k])
    if st is not None:
        got["status"] = st.cpu().numpy()
    return got, bf


def launch_counter(g, t):
    """The draw counter of launch t: the launches before it drew once per half they ran."""
    return (g.counter + sum(len(f) for f in g.flags[:t])) & 0xffffffff


# ------------------------------------------------------------------------------------------ the oracle
def step_oracle(c, g, d, state, t):
    """oracle.enkf.EnKF per filter on the launch's inputs, with the kernel's failure rules: an indefinite Q fails the
    predict (NOT_PD), a singular S or an indefinite R the update (SINGULAR_S, then NOT_PD), and the filter keeps the
    state it had before the failing half."""
    from oracle import enkf as oe
    from oracle import ukf as oukf
    n, m, fx, hx = c.inst
    x, P, sig = state
    flags = g.flags[t]
    counter = launch_counter(g, t)
    dt = float(rd(DT, c.dt))
    N = g.N
    w = dict(x=x.copy(), P=P.copy(), sig=sig.copy(), status=np.zeros(N, np.int32), pred=np.zeros(N, bool),
             upd=np.zeros(N, bool), cond=np.ones(N), P_upd=np.zeros((N, n, n)), x_prior=np.zeros((N, n)),
             P_prior=np.zeros((N, n, n)), K=np.zeros((N, n, m)), S=np.zeros((N, m, m)), SI=np.zeros((N, m, m)))
    per = lambda k, f: None if k not in d else (d[k] if d[k].ndim == 2 else d[k][f])           # noqa: E731
    for f in range(N):
        Ff, Hf = per("F", f), per("H", f)
        e = oe.EnKF(x[f], np.zeros((n, n)), m, dt, g.members, lambda s, Hf=Hf: oukf.hx_apply(HX[hx], s, Hf),
                    lambda s, dt, Ff=Ff: oukf.fx_apply(FX[fx], s, dt, Ff), oe.Stream(g.seed, f, c.dt))
        e.sigmas, e.x, e.P, e.Q, e.R = sig[f].copy(), x[f].copy(), P[f].copy(), per("Q", f), per("R", f)
        st = OK
        if "p" in flags:
            e.counter = counter
            keep = (e.sigmas, e.x, e.P)
            try:
                e.predict()
                w["pred"][f] = True
                w["x_prior"][f], w["P_prior"][f] = e.x_prior, e.P_prior
            except np.linalg.LinAlgError:
                e.sigmas, e.x, e.P = keep
                st = NOT_PD
        if "u" in flags and st == OK and d["valid"][t, f]:
            e.counter = (counter + (1 if "p" in flags else 0)) & 0xffffffff
            keep = (e.sigmas, e.x, e.P)
            try:
                e.update(d["zs"][t, f], R=e.R)
                w["upd"][f] = True
                w["cond"][f] = np.linalg.cond(_equilibrated(e.S))
                w["P_upd"][f] = keep[2]
                w["K"][f], w["S"][f], w["SI"][f] = e.K, e.S, e.SI
            except np.linalg.LinAlgError as err:
                e.sigmas, e.x, e.P = keep
                st = SINGULAR_S if "ingular" in str(err) else NOT_PD
        w["x"][f], w["P"][f], w["sig"][f], w["status"][f] = e.x, e.P, e.sigmas, st
    w["zs"] = d["zs"][t]
    return w


def _family(c, g, out=None):
    """init; pair (2 members, on chip), pair_gain (K and SI at 2 members); onchip or global (5 or more members)."""
    if c.kind == "init":
        return "init"
    if g.members == 2:
        return "pair_gain" if out in ("K", "SI") else "pair"
    return "onchip" if c.onchip(g) else "global"


def _bound(c, g, out=None):
    fam = _family(c, g, out)
    return TOL[fam][c.dt], "test_gpu_enkf_instances %s %s" % (fam, np.dtype(c.dt).name)


def _equilibrated(S):
    """D^-1/2 S D^-1/2, D = diag S: S in measurement units of one standard deviation each, so its condition number
    says how hard the solve is, not how the units (metres, radians) compare."""
    d = np.sqrt(np.abs(np.diagonal(S, axis1=-2, axis2=-1)))
    d = np.where(d > 0, d, 1.0)
    return S / (d[..., :, None] * d[..., None, :])


def _cov_scale(sP, sx):
    """The scale of a covariance summed from members of scale sx: its own, or sx sqrt(sP) where the spread is small
    against the members (centring a member of size sx rounds at eps sx, and the spread multiplies that)."""
    return np.maximum(sP, sx * np.sqrt(sP))


def check_step(c, g, t, state, got, want, fails, what):
    tol, label = _bound(c, g)
    flags = g.flags[t]
    x, P, sig = state
    N = g.N
    if "status" in got:
        assert np.array_equal(got["status"], want["status"]), (what, got["status"], want["status"])
    # a filter that neither predicted nor updated comes back bit for bit
    same = ~want["pred"] & ~want["upd"]
    assert np.array_equal(got["sig"][same], sig[same]), what + " members of a filter that did not step"
    assert np.array_equal(got["x"][same], x[same]) and np.array_equal(got["P"][same], P[same]), what
    if not g.alias:
        assert np.array_equal(got["sig_in"], sig), what + " sigmas changed"
    cond = want["cond"]
    sx = mag(sig, want["sig"])
    close(got["sig"], want["sig"], sx, cond, tol, what + " members", label)
    close(got["x"], want["x"], sx, cond, tol, what + " x", label)
    sP = _cov_scale(np.where(want["upd"], mag(want["P_upd"], want["P"]), mag(want["P"])), sx)
    close(got["P"], want["P"], sP, cond, tol, what + " P", label)
    pred, upd = want["pred"], want["upd"]
    # K, S and SI in measurement units of one standard deviation sqrt(S_aa) of the filter's S: every entry of the
    # same kind, so that one filter-wide scale measures them all (a range in metres next to angles in radians)
    sd = np.sqrt(np.abs(np.diagonal(want["S"], axis1=1, axis2=2)))
    sd = np.where(sd > 0, sd, 1.0)
    unit = dict(K=sd[:, None, :], S=1.0 / (sd[:, :, None] * sd[:, None, :]), SI=sd[:, :, None] * sd[:, None, :])
    sz = mag(np.asarray(want["zs"]) / sd)
    for k in g.outs:
        on = pred if k in ("x_prior", "P_prior") else upd
        assert np.all(got[k][~on] == Bufs.SENT), "%s %s written where the filter did not %s" % (
            what, k, "predict" if k in ("x_prior", "P_prior") else "update")
        if not on.any():
            continue
        gk, wk = got[k] * unit.get(k, 1.0), want[k] * unit.get(k, 1.0)
        if k == "x_prior":
            scale, kc = sx, 1.0
        elif k == "P_prior":
            scale, kc = _cov_scale(mag(wk), sx), 1.0
        elif k == "S":                      # a centred sum of hx values of the size of z, plus R: no solve in it
            scale, kc = _cov_scale(mag(wk), sz), 1.0
        else:
            scale, kc = mag(wk), cond
        ktol, klabel = _bound(c, g, k)
        close(gk, wk, scale, kc, ktol, what + " " + k, klabel, rows=on)
    # the oracle meets each planted failure where the launch reaches it
    for f, kind in fails.items():
        if kind in ("q_rank", "r_rank", "q_zero"):
            assert want["status"][f] == OK and want["pred"][f] == ("p" in flags), (what, kind)
        elif kind == "q_indef" and "p" in flags:
            assert want["status"][f] == NOT_PD and not want["pred"][f] and not want["upd"][f], (what, kind)
        elif kind == "r_indef" and "u" in flags:
            assert want["status"][f] == NOT_PD and want["pred"][f] == ("p" in flags) and not want["upd"][f], (what, kind)
        elif kind == "singular" and "u" in flags:
            assert want["status"][f] == SINGULAR_S and not want["upd"][f], (what, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("case", STEPS, ids=[c.id for c in STEPS])
def test_step_vs_oracle(case):
    """Three launches of each run, each against the oracle from its own inputs: members, x, P, every optional output
    passed and status; outputs a filter must not write stay at the sentinel, nothing is written outside an array,
    and sigmas is left alone when sigmas_out is separate."""
    for j, g in enumerate(case.cfgs):
        d, fails = step_inputs(case, g, seed=1000 * j + case.n)
        state = (d["x"], d["P"], d["sig"])
        for t in range(len(g.flags)):
            got, bf = run_step(case, g, d, state, t)
            bf.check_guards()
            want = step_oracle(case, g, d, state, t)
            check_step(case, g, t, state, got, want, fails, "%s %r launch %d" % (case.id, g, t))
            state = (got["x"].astype(np.float64), got["P"].astype(np.float64), got["sig"].astype(np.float64))


# ------------------------------------------------------------------------------------------ initialize
def init_inputs(c, g, seed):
    """x and P per filter: SPD, rank-deficient PSD (rank n // 2: _rank_one_blocks) and indefinite in turn."""
    rng = np.random.default_rng(seed)
    n = c.n
    x = rng.normal(0.0, 5.0, (g.N, n))
    P = spd(rng, (g.N,), n, 2.0)
    kinds = ["spd", "rank_def", "indef"]
    for f in range(g.N):
        k = kinds[(f + seed) % 3] if g.N > 1 else "spd"
        if k == "rank_def":
            P[f] = 2.0 * _rank_one_blocks(rng, n)
        elif k == "indef":
            P[f][n - 1, n - 1] = -1.0 - P[f][n - 1, n - 1]
    return rd(x, c.dt), rd(P, c.dt)


def run_init(c, g, x, P):
    from filterpy_b200 import _lib
    n, N, Nm = c.n, g.N, g.members
    bf = Bufs(c.dt)
    xb, Pb = bf.put(x, g.mis), bf.put(P, g.mis)
    so = bf.out((N, Nm, n), g.mis)
    st = None if g.no_status else bf.out((N,), g.mis, dtype=np.int32, fill=-7)
    rc, err = call("bke_enkf_initialize", ctypes.c_int64(N), n, Nm, _lib.BKE_F32 if c.dt == F32 else _lib.BKE_F64,
                   ctypes.c_uint32(g.seed), ctypes.c_uint32(g.counter), ptr(xb), ptr(Pb), ptr(so), ptr(st))
    assert rc == 0, err
    got = dict(sig=so.cpu().numpy().reshape(N, Nm, n))
    if st is not None:
        got["status"] = st.cpu().numpy()
    return got, bf


@pytest.mark.gpu
@pytest.mark.parametrize("case", INITS, ids=[c.id for c in INITS])
def test_initialize_vs_oracle(case):
    """members = x + L_P xi for SPD and rank-deficient P; an indefinite P sets NOT_PD and every member is x."""
    from oracle import enkf as oe
    for j, g in enumerate(case.cfgs):
        x, P = init_inputs(case, g, seed=100 * j + case.n)
        got, bf = run_init(case, g, x, P)
        bf.check_guards()
        want = np.empty_like(got["sig"], dtype=np.float64)
        status = np.zeros(g.N, np.int32)
        for f in range(g.N):
            try:
                want[f] = oe.Stream(g.seed, f, case.dt).draw(g.counter, x[f], P[f], g.members)
            except np.linalg.LinAlgError:
                want[f] = x[f]
                status[f] = NOT_PD
        what = "%s %r" % (case.id, g)
        if "status" in got:
            assert np.array_equal(got["status"], status), (what, got["status"], status)
        bad = status != OK
        assert np.array_equal(got["sig"][bad], np.broadcast_to(x[bad][:, None, :], got["sig"][bad].shape)), what
        tol, label = _bound(case, g)
        close(got["sig"], want, mag(want), 1.0, tol, what + " members", label)


# ------------------------------------------------------------------------------------------ which kernel runs
def _run_cases():
    for c in CASES:
        g = c.cfgs[0]
        if c.kind == "init":
            x, P = init_inputs(c, g, seed=1)
            run_init(c, g, x, P)
        else:
            d, _ = step_inputs(c, g, seed=1)
            run_step(c, g, d, (d["x"], d["P"], d["sig"]), 0)


def _profiled_names():
    return profiled_names(_run_cases, r"enkf_\w*kernel")


@pytest.mark.gpu
def test_dispatch_runs_the_kernels_of_the_table():
    """Each CASES entry, run once at its first configuration, launches the kernel the table names: the 60 step
    instances and the 32 initialize instances.  The profile is taken in a process of its own."""
    check_launch_order("test_gpu_enkf_instances", [(c.id, c.kernels()) for c in CASES])
