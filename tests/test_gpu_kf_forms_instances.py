"""Every kernel instance behind bke_kf_step_correlated and bke_kf_update_rows against the fp64 oracle
(tests/kf_forms_oracle.py), through the C-ABI, with a table that names the kernel(s) each case launches.

Both calls run on bke_kf_step's kernels with the update form a template parameter (FORM_CORRELATED = 1,
FORM_ROWS = 2).  bke_kf_step_correlated tries the register tile kf_direct_kernel<T, N, M, EX, 1> (dispatch_correlated
in csrc/kf_direct.cu: EX = false when no optional output is passed) and falls back to the catch-all
kf_generic_kernel<T, 1> (csrc/kf_generic.cu) for any other shape, a control input, or x, P, a model, an output or M
off a 16-byte boundary.  bke_kf_update_rows runs a block of L rows on kf_direct_kernel<T, N, L, true, 2>
(dispatch_rows) or on kf_generic_kernel<T, 2>.  The catch-all's shared-memory slice per warp is kf_generic.cu's
per_warp, 2·n·m words larger for the correlated form; blocks of 4, 2 or 1 warps, a refusal above 200 KB per warp.

Inputs are rounded to the kernel's dtype before the oracle sees them.  Each error is taken relative to the filter's
own scale and divided by the condition of its solve: cond(S_i) for a block of L > 1 rows, 1 for L = 1 and where
nothing is inverted.  The correlated S = H P H' + H M + M' H' + R sums terms of either sign, so there the condition
is ||S^-1|| ||T|| with T = |H P H'| + |H M| + |M' H'| + |R| (cond(S) when nothing cancels), and S itself is measured
against T.  The correlated P is P - K (H P + M'), neither Joseph nor symmetrised: its scale includes
max |K (H P + M')|, the term that cancels; K = (P H' + M) SI is measured against (|P H'| + |M|) |SI|.

Every output starts as a finite sentinel between NaN guards, so a write outside an array, a missing write or one to
an entry a filter must leave alone shows up.  Edge filters (an exactly singular S or S_i, an indefinite S from a
large M, an ill-conditioned S, and L = 1 with S_i = 0, whose inf / NaN pattern is compared with the oracle's entry by
entry) sit inside otherwise healthy blocks, and every other filter must equal a clean run bit for bit.

Worst cases measured on an H100 80GB HBM3 (700 W power limit) with BKE_TEST_ERRLOG, as error / (scale * cond) over
every case, output and bank size of the family, and the bound set from each (about 4x):

    family                                   fp64 worst  bound     fp32 worst  bound
    corr-direct   kf_direct_kernel<.., 1>     1.1e-15    5e-15     5.8e-7      2.5e-6
    corr-generic  kf_generic_kernel<T, 1>     9.6e-16    4e-15     7.6e-7      3e-6
    rows-direct   kf_direct_kernel<.., 2>     9.1e-16    4e-15     4.5e-7      2e-6
    rows-generic  kf_generic_kernel<T, 2>     9.9e-16    4e-15     1.1e-6      4.5e-6    (dim_x 111, the largest)
"""
import ctypes
import re

import numpy as np
import pytest

from gpu_harness import (BUDGET, F32, F64, Bufs, body, call, check_launch_order, close, k_direct, k_gen, mag,
                         profiled_names, ptr, rd, spd, src)

import kf_forms_oracle as kfo

ALPHA_SQ = 1.01 ** 2
SENT = Bufs.SENT
STATUS_FILL = 5                                  # a status word no call writes: BKE_STATUS_STICKY must keep it
CORR, ROWS = 1, 2                                # kf_direct.cu / kf_generic.cu FORM_CORRELATED, FORM_ROWS

TOL = {
    "corr-direct": {F64: 5e-15, F32: 2.5e-6},
    "corr-generic": {F64: 4e-15, F32: 3e-6},
    "rows-direct": {F64: 4e-15, F32: 2e-6},
    "rows-generic": {F64: 4e-15, F32: 4.5e-6},
}

# the register tiles: dispatch_correlated's (dim_x, dim_z) and dispatch_rows's (dim_x, L), fp32 extras included
CORR_TILES = {F64: [(4, 2), (2, 1), (1, 1), (2, 2), (3, 1), (4, 1), (4, 4)],
              F32: [(4, 2), (2, 1), (1, 1), (2, 2), (3, 1), (4, 1), (4, 4), (6, 3), (6, 2)]}
ROW_TILES = {F64: [(1, 1), (2, 1), (2, 2), (3, 1), (4, 1), (4, 2), (4, 3), (4, 4)],
             F32: [(1, 1), (2, 1), (2, 2), (3, 1), (4, 1), (4, 2), (4, 3), (4, 4), (6, 1), (6, 2), (6, 3)]}
CORR_OUTS = ("x_prior", "P_prior", "K", "y", "S", "SI", "log_likelihood")
ROWS_OUTS = ("x_prior", "P_prior", "K", "y", "z_record")
SHARED = {"per": "", "shared": "FQHRM", "FQ": "FQ", "HRM": "HRM"}     # the models a bank shares (stride 0)
EDGE_OK, SINGULAR, INDEFINITE, ILLCOND, ZERO_S = 0, 1, 2, 3, 4
ILLCOND_COND = {F32: 1e3, F64: 1e9}


# ------------------------------------------------------------------------------------------ the catch-all's limits
def per_warp(n, m, form):
    """kf_generic.cu launch_t: the words of one warp's slice (m: the block's L for the rows form)."""
    w = 2 * n + 4 * (n * n) + 3 * (n * m) + 4 * (m * m) + 2 * m + (2 * n * m if form == CORR else 0)
    return (w + 3) & ~3


def warps_per_block(n, m, form, dt):
    """api.cu warp_shape: 4 warps per block, halved until the block's slices fit the budget; 0 = refused."""
    bw = per_warp(n, m, form) * np.dtype(dt).itemsize
    w = 4
    while w > 1 and bw * w > BUDGET:
        w >>= 1
    return w if bw * w <= BUDGET else 0


def warp_shapes(dt, form, m):
    """At dim_z (or L) = m: (the first n of 4 warps per block above 48 KB, the first n with 2 warps per block, the first
    with 1, the largest accepted n, the first refused n)."""
    es = np.dtype(dt).itemsize
    big = next(n for n in range(1, 400) if per_warp(n, m, form) * es * 4 > 48 * 1024)
    two = next(n for n in range(1, 400) if warps_per_block(n, m, form, dt) == 2)
    one = next(n for n in range(1, 400) if warps_per_block(n, m, form, dt) == 1)
    refused = next(n for n in range(1, 400) if warps_per_block(n, m, form, dt) == 0)
    assert warps_per_block(big, m, form, dt) == 4
    return big, two, one, refused - 1, refused


# ------------------------------------------------------------------------------------------ the instance table
class Case:
    """One call of bke_kf_step_correlated (form CORR) or bke_kf_update_rows (ROWS) and the kernels it launches.
      n, m       dim_x and the bank's dim_z; L, start: the block of rows (ROWS)
      mode       BKE_DO_UPDATE (2) or BKE_DO_PREDICT | BKE_DO_UPDATE (3)
      models     SHARED key: which of F, Q, H, R, M (and H_i / R_i with H / R) are one matrix for the bank
      outs       the optional outputs passed (CORR_OUTS / ROWS_OUTS names)
      Hi, Ri     (ROWS) H_i / R_i passed, else read in place from the bank's H / R (R with row pitch m)
      inplace    x_out / P_out are x / P;  mask: a z_valid mask (else NULL);  sticky: BKE_STATUS_STICKY
      mis        None, "bank" (x, P and every output one element past a 16-byte boundary), "M" (M so)
      ctrl       B u;  grid: one more bank, of sm_count * 16 * warps-per-block + 37 filters (the grid-stride loop)
      refused    the catch-all refuses the shape: BKE_ERR_UNSUPPORTED, nothing launched"""

    def __init__(self, form, family, dt, n, m, kernels, Ns, L=None, start=0, mode=3, models="per", outs=(),
                 Hi=False, Ri=False, inplace=False, mask=True, sticky=False, mis=None, ctrl=False, grid=False,
                 refused=False, tag=""):
        self.form, self.family, self.dt, self.n, self.m = form, family, dt, n, m
        self.L = m if form == CORR else L
        self.start, self.kernels, self.Ns, self.mode, self.models = start, list(kernels), tuple(Ns), mode, models
        self.outs, self.Hi, self.Ri, self.inplace, self.mask = tuple(outs), Hi, Ri, inplace, mask
        self.sticky, self.mis, self.ctrl, self.grid, self.refused, self.tag = sticky, mis, ctrl, grid, refused, tag

    @property
    def fam(self):
        return ("corr-" if self.form == CORR else "rows-") + self.family

    @property
    def id(self):
        s = "%s-%s-%d_%d" % (self.fam, "f32" if self.dt == F32 else "f64", self.n, self.m)
        if self.form == ROWS:
            s += "-L%d_s%d%s%s" % (self.L, self.start, "-Hi" if self.Hi else "", "-Ri" if self.Ri else "")
        s += "-mode%d-%s" % (self.mode, self.models)
        allo = CORR_OUTS if self.form == CORR else ROWS_OUTS
        s += "-all" if set(self.outs) == set(allo) else ("-none" if not self.outs else
                                                          "-" + "+".join(k for k in allo if k in self.outs))
        for flag, name in ((self.inplace, "inplace"), (not self.mask, "nomask"), (self.sticky, "sticky"),
                           (self.mis, "mis" + str(self.mis)), (self.ctrl, "ctrl"), (self.grid, "grid"),
                           (self.refused, "refused"), (self.tag, self.tag)):
            if flag:
                s += "-" + name
        return s


TILE_NS = (1, 127, 129, 1037)
GEN_NS = (1, 3, 5, 1037)
BIG_NS = (1, 3, 5, 67)


def _cases():
    out = []
    # correlated register tiles: every shape x dtype x EX x mode, the models, outputs and options spread over them
    i = 0
    single = [k for k in CORR_OUTS]
    for dt in (F64, F32):
        for n, m in CORR_TILES[dt]:
            for ex in (True, False):
                for mode in (2, 3):
                    outs = (CORR_OUTS if i % 3 == 0 else (single[(i // 3) % len(single)],)) if ex else ()
                    out.append(Case(CORR, "direct", dt, n, m, [k_direct(dt, n, m, ex, CORR)], TILE_NS, mode=mode,
                                    models=("per", "shared", "FQ", "HRM")[i % 4], outs=outs, inplace=(i % 3 == 1),
                                    mask=(i % 5 != 4), sticky=(i % 2 == 1)))
                    i += 1
    # row-block register tiles: every (n, L) x dtype in a bank of dim_z L + 2 at start 0, 1 (the middle) and 2
    # (m - L), and once with L = m; R read in place (row pitch m) at starts 1 and m - L
    i = 0
    for dt in (F64, F32):
        for n, L in ROW_TILES[dt]:
            for m, start in ((L + 2, 0), (L + 2, 1), (L + 2, 2), (L, 0)):
                Ri = (start == 0 and m > L) or (m == L and i % 2 == 0)
                outs = [ROWS_OUTS, ("K", "y", "z_record"), ("x_prior", "K", "z_record"), ("P_prior", "y", "z_record"),
                        ("x_prior", "P_prior", "y", "K"), ()][i % 6]
                out.append(Case(ROWS, "direct", dt, n, m, [k_direct(dt, n, L, True, ROWS)], TILE_NS, L=L, start=start,
                                mode=(2, 3)[i % 2], models=("per", "shared", "FQ", "HRM")[(i // 2) % 4], outs=outs,
                                Hi=(i % 3 != 1), Ri=Ri, inplace=(i % 4 == 1), mask=(i % 5 != 3),
                                sticky=(i % 2 == 0)))
                i += 1
    # the catch-all, each form x dtype through each route
    for dt in (F64, F32):
        gc = [k_gen(dt, CORR)]
        gr = [k_gen(dt, ROWS)]
        AC, AR = CORR_OUTS, ROWS_OUTS
        out += [
            # shapes without a tile
            Case(CORR, "generic", dt, 5, 3, gc, GEN_NS, outs=AC, grid=True),
            Case(CORR, "generic", dt, 9, 3, gc, GEN_NS, mode=2, models="shared", sticky=True),
            Case(CORR, "generic", dt, 12, 5, gc, GEN_NS, models="FQ", outs=("y", "S"), inplace=True),
            Case(ROWS, "generic", dt, 5, 4, gr, GEN_NS, L=3, start=1, outs=AR, grid=True),
            Case(ROWS, "generic", dt, 9, 3, gr, GEN_NS, L=3, mode=2, models="shared", Hi=True, Ri=True, sticky=True),
            Case(ROWS, "generic", dt, 12, 7, gr, GEN_NS, L=5, start=2, models="HRM", outs=("K", "y"), Hi=True),
            # B u at a tile shape
            Case(CORR, "generic", dt, 4, 2, gc, GEN_NS, outs=AC, ctrl=True),
            Case(CORR, "generic", dt, 2, 1, gc, GEN_NS, models="shared", ctrl=True, mask=False),
            Case(ROWS, "generic", dt, 4, 3, gr, GEN_NS, L=2, start=1, outs=AR, ctrl=True, sticky=True),
            Case(ROWS, "generic", dt, 2, 2, gr, GEN_NS, L=1, start=1, models="shared", ctrl=True, Ri=True),
            # x, P and their outputs one element off a 16-byte boundary at a tile shape
            Case(CORR, "generic", dt, 4, 2, gc, GEN_NS, outs=AC, mis="bank", sticky=True),
            Case(CORR, "generic", dt, 4, 4, gc, GEN_NS, mode=2, mis="bank", inplace=True),
            Case(ROWS, "generic", dt, 4, 4, gr, GEN_NS, L=2, start=2, outs=AR, mis="bank"),
            Case(ROWS, "generic", dt, 4, 3, gr, GEN_NS, L=3, mode=2, mis="bank", inplace=True, Hi=True),
            # a misaligned M at a tile shape: per filter, and shared
            Case(CORR, "generic", dt, 4, 2, gc, GEN_NS, outs=AC, mis="M"),
            Case(CORR, "generic", dt, 2, 2, gc, GEN_NS, mode=2, models="HRM", outs=("K",), mis="M", sticky=True),
        ]
        if dt == F64:                              # 6 x 6 fp64 has no register tile
            out += [Case(CORR, "generic", dt, 6, 3, gc, GEN_NS, outs=AC),
                    Case(CORR, "generic", dt, 6, 2, gc, GEN_NS, mode=2, models="shared", outs=("log_likelihood",))]
            out += [Case(ROWS, "generic", dt, 6, 3, gr, GEN_NS, L=L, start=s, outs=AR, Hi=(L == 2), sticky=(L == 1))
                    for L, s in ((1, 2), (2, 1), (3, 0))]
        # 4 warps per block above 48 KB, 2 and 1 warps per block, the largest accepted shape and the first refused one
        for form, ks in ((CORR, gc), (ROWS, gr)):
            big, two, one, top, refused = warp_shapes(dt, form, 3)
            kw = dict(L=3, start=1) if form == ROWS else {}
            mm = 4 if form == ROWS else 3
            out += [
                Case(form, "generic", dt, big, mm, ks, BIG_NS, outs=CORR_OUTS if form == CORR else ROWS_OUTS,
                     tag="over48k", **kw),
                Case(form, "generic", dt, two, mm, ks, BIG_NS, mode=2, models="shared", tag="wpb2", **kw),
                Case(form, "generic", dt, one, mm, ks, BIG_NS, outs=("y",), tag="wpb1", **kw),
                Case(form, "generic", dt, top, mm, ks, BIG_NS, outs=("K", "y"), sticky=True, tag="top", **kw),
                Case(form, "generic", dt, refused, mm, [], (3,), refused=True, **kw),
            ]
    return out


CASES = _cases()
RUN_CASES = [c for c in CASES if not c.refused]


def _dispatched():
    """Every kernel instance the two entry points can launch, parsed from the source."""
    d = src("kf_direct.cu")
    inst = set()
    li = body(d, "int launch_inst(const bke_kf_args &a, cudaStream_t s, const DirP<T> *form")
    assert re.search(r"if \(FORM == FORM_ROWS \|\| ex\) kf_direct_kernel<T, N, M, true, FORM><<<", li), li
    assert re.search(r"else kf_direct_kernel<T, N, M, false, FORM><<<", li), li
    shapes = {}
    for fn, macro, form in (("int dispatch_correlated(", "BKE_CORR", CORR), ("int dispatch_rows(", "BKE_ROWS", ROWS)):
        bd = body(d, fn)
        both, f32only = bd.split("if constexpr (sizeof(T) == 4)")
        got = {F64: [], F32: []}
        for part, dts in ((both, (F64, F32)), (f32only, (F32,))):
            for a, e in re.findall(r"\b%s\((\d+), (\d+)\)" % macro, part):
                for dt in dts:
                    got[dt].append((int(a), int(e)))
        shapes[form] = got
        for dt, sh in got.items():
            for n, m in sh:
                for ex in ((True, False) if form == CORR else (True,)):
                    inst.add(k_direct(dt, n, m, ex, form))
            inst.add(k_gen(dt, form))
    return inst, shapes


def test_instance_table_matches_dispatch():
    """CASES launches every instance the two entry points can reach (and no other), through every route of the
    catch-all: a new tile shape, an EX rule, a moved shared-memory formula or another launch order fails here, on a
    machine without a GPU too."""
    inst, shapes = _dispatched()
    assert shapes[CORR] == CORR_TILES and shapes[ROWS] == ROW_TILES
    table = {k for c in CASES for k in c.kernels}
    assert table == inst, (sorted(inst - table), sorted(table - inst))
    # every correlated tile x dtype x EX x mode; every rows tile x dtype at start 0, the middle and m - L, and L = m
    got = {(c.dt, c.n, c.m, bool(c.outs), c.mode) for c in CASES if c.fam == "corr-direct"}
    assert got == {(dt, n, m, ex, mode) for dt in (F32, F64) for n, m in CORR_TILES[dt] for ex in (True, False)
                   for mode in (2, 3)}
    for dt in (F32, F64):
        for n, L in ROW_TILES[dt]:
            rc = [c for c in CASES if c.fam == "rows-direct" and (c.dt, c.n, c.L) == (dt, n, L)]
            assert {c.start for c in rc if c.m > L} >= {0, 1, rc[0].m - L} and any(c.m == L for c in rc)
            assert any(not c.Ri and c.start > 0 and c.m > L for c in rc)
    # the catch-all's routes, each form x dtype
    for form in (CORR, ROWS):
        tiles = CORR_TILES if form == CORR else ROW_TILES
        for dt in (F32, F64):
            g = [c for c in CASES if c.form == form and c.family == "generic" and c.dt == dt]
            assert any((c.n, c.L) not in tiles[dt] and not (c.ctrl or c.mis) for c in g)
            assert any(c.ctrl and (c.n, c.L) in tiles[dt] for c in g)
            assert any(c.mis == "bank" and (c.n, c.L) in tiles[dt] for c in g)
            if form == CORR:
                assert any(c.mis == "M" and (c.n, c.L) in tiles[dt] for c in g)
            wpbs = {warps_per_block(c.n, c.L, form, dt) for c in g}
            assert wpbs == {0, 1, 2, 4}
            assert any(per_warp(c.n, c.L, form) * np.dtype(dt).itemsize * 4 > 48 * 1024
                       and warps_per_block(c.n, c.L, form, dt) == 4 for c in g)
            top = max(c.n for c in g if not c.refused and c.L == 3)
            assert warps_per_block(top + 1, 3, form, dt) == 0 and any(c.refused and c.n == top + 1 for c in g)
            assert any(c.grid for c in g)
    # kf_generic.cu's slice and refusal, and the direct-then-generic order of both entry points
    lt = body(src("kf_generic.cu"), "int launch_t(const bke_kf_args &a, cudaStream_t s, const KfP<T> *form")
    assert ("int per_warp = 2 * n + 4 * (n * n) + 3 * (n * m) + 4 * (m * m) + 2 * m + (FORM == FORM_CORRELATED ? "
            "2 * n * m : 0);" in lt and "per_warp = (per_warp + 3) & ~3;" in lt and "budget = 200 * 1024" in lt)
    api = src("api.cu")
    corr = body(api, "int bke_kf_step_correlated(")
    assert re.search(r"int rc = launch_kf_direct_correlated\(a, M, M_stride, s\);\s*return rc == BKE_ERR_UNSUPPORTED "
                     r"\? launch_kf_generic_correlated\(a, M, M_stride, s\) : rc;", corr), corr
    rows = body(api, "static int launch_rows(")
    assert re.search(r"int rc = launch_kf_direct_rows\(b, [^;]*\);\s*if \(rc == BKE_ERR_UNSUPPORTED\) rc = "
                     r"launch_kf_generic_rows\(b, [^;]*\);\s*return rc;", rows), rows
    kd = src("kf_direct.cu")
    for fn in ("int launch_kf_direct_correlated(", "int launch_kf_direct_rows("):
        assert "if (a.B != nullptr && a.u != nullptr) return BKE_ERR_UNSUPPORTED;" in body(kd, fn)


# ------------------------------------------------------------------------------------------ inputs
def _edge_kinds(c):
    if c.form == CORR:
        return (SINGULAR, INDEFINITE) + ((ILLCOND,) if c.m > 1 else ())
    return (ZERO_S,) if c.L == 1 else (SINGULAR,)


def _inputs(c, N, seed, edges, models):
    """The arrays of one call, rounded to the case's dtype (a shared model is one matrix), and the edge kind of each
    filter.  The edges are placed at filters 30, 91, 152, ... (inside healthy blocks and warps): their F is 0 and
    Q = P, so the update starts from P (x = B u or 0) whether or not a predict runs, and the rest of their models
    make S singular, indefinite or ill-conditioned.  Nothing else differs from the run without edges."""
    rng = np.random.default_rng(seed)
    n, m, L, dt = c.n, c.m, c.L, c.dt
    sh = SHARED[models]
    cnt = lambda k: () if k in sh else (N,)
    d = dict(x=rng.normal(size=(N, n)) * 3, P=spd(rng, (N,), n, 2.0),
             F=np.eye(n) + 0.1 * rng.normal(size=cnt("F") + (n, n)), Q=spd(rng, cnt("Q"), n, 0.05),
             H=rng.normal(size=cnt("H") + (m, n)), R=spd(rng, cnt("R"), m, 0.5))
    if c.form == CORR:
        d["M"] = 0.3 * rng.normal(size=cnt("M") + (n, m))
    if c.Hi:
        d["Hi"] = rng.normal(size=cnt("H") + (L, n))
    if c.Ri:
        d["Ri"] = spd(rng, cnt("R"), L, 0.5)
    d["z"] = rng.normal(size=(N, L)) * 3
    if c.ctrl:
        d["B"] = rng.normal(size=cnt("F") + (n, 2))
        d["u"] = rng.normal(size=(N, 2))
    d = {k: rd(v, dt) for k, v in d.items()}
    kind = np.zeros(N, int)
    if not edges:
        return d, kind
    assert models == "per"
    er = np.random.default_rng(seed + 99)
    kinds = _edge_kinds(c)
    s, e = c.start, c.start + L
    for f in range(30, N, 61):
        k = kinds[(f // 61) % len(kinds)]
        kind[f] = k
        d["F"][f] = 0
        if k == ZERO_S:                        # H_i = e0, P00 = 2, R_i = -2: S_i = 0 and P H' nonzero
            d["P"][f] *= 2.0 / d["P"][f, 0, 0]
            d["P"][f, 0, 0] = 2.0
        d["Q"][f] = d["P"][f]
        P = d["P"][f]
        if c.form == CORR:
            H, R, M = d["H"][f], d["R"][f], d["M"][f]
            if k == SINGULAR:                  # a zero last row of H, R and M': S has a zero row and column
                H[-1] = 0; R[-1] = 0; R[:, -1] = 0; M[:, -1] = 0
            elif k == INDEFINITE:              # M[:, 0] = -c (P H')[:, 0]: S_00 = -(H P H')_00 - R_00 < 0
                PH = P @ H.T
                M[:, 0] = -(1 + R[0, 0] / (H[0] @ PH[:, 0])) * PH[:, 0]
            else:                              # R such that S = U diag(1 .. 1 / cond) U' * 4
                U = np.linalg.qr(er.normal(size=(m, m)))[0]
                St = 4 * (U * np.logspace(0, -np.log10(ILLCOND_COND[dt]), m)) @ U.T
                d["M"][f] = rd(M, dt)
                HM = H @ d["M"][f]
                R[:] = St - (H @ P @ H.T + HM + HM.T)
        else:
            Hb = d["Hi"][f] if c.Hi else d["H"][f, s:e]
            if c.Ri:
                Rb = d["Ri"][f]
            else:
                Rb = d["R"][f, s:e, s:e]
            if k == ZERO_S:
                Hb[:] = 0; Hb[0, 0] = 1.0
                Rb[:] = -2.0
            else:                              # a zero last row of H_i and R_i (and R_i's column)
                Hb[-1] = 0; Rb[-1] = 0; Rb[:, -1] = 0
            if not c.Hi:
                d["H"][f, s:e] = Hb
            if not c.Ri:
                d["R"][f, s:e, s:e] = Rb
    return {k: rd(v, dt) for k, v in d.items()}, kind


def _full(a, N):
    return np.broadcast_to(a, (N,) + a.shape[-2:]) if a.ndim == 2 else a


def _shapes(c, N):
    n, m = c.n, c.m
    return dict(x_prior=(N, n), P_prior=(N, n, n), K=(N, n, m), y=(N, m), S=(N, m, m), SI=(N, m, m),
                log_likelihood=(N,), z_record=(N, m))


# ------------------------------------------------------------------------------------------ one call
def run(c, N, seed=0, edges=False, models=None):
    """One call of case c on N filters: (rc, error text, got, inputs, valid, edge kinds)."""
    from filterpy_b200 import _lib
    models = models or c.models
    dt, n, m, L = c.dt, c.n, c.m, c.L
    d, kind = _inputs(c, N, seed, edges, models)
    valid = None
    if c.mask:
        valid = np.random.default_rng(seed + 1).random(N) > 0.2
        valid[kind != EDGE_OK] = True
        if N > 1:
            valid[1] = False
    bf = Bufs(dt)
    r = _lib.KfRowsArgs()
    a = _lib.KfArgs() if c.form == CORR else r.step
    a.n_filters, a.dim_x, a.dim_z = N, n, m
    a.dtype = _lib.BKE_F32 if dt == F32 else _lib.BKE_F64
    a.flags = c.mode | (_lib.BKE_STATUS_STICKY if c.sticky else 0)
    a.alpha_sq = ALPHA_SQ
    mis = c.mis == "bank"
    xv = bf.put(d["x"], mis, out=c.inplace); Pv = bf.put(d["P"], mis, out=c.inplace)
    a.x, a.P = ptr(xv), ptr(Pv)
    xo, Po = (xv, Pv) if c.inplace else (bf.out((N, n), mis), bf.out((N, n, n), mis))
    a.x_out, a.P_out = ptr(xo), ptr(Po)
    for k in "FQHR":
        setattr(a, k, ptr(bf.put(d[k])))
        setattr(a, k + "_stride", 0 if d[k].ndim == 2 else d[k].shape[-1] * d[k].shape[-2])
    if c.ctrl:
        a.dim_u = 2
        a.B = ptr(bf.put(d["B"])); a.B_stride = 0 if d["B"].ndim == 2 else 2 * n
        a.u = ptr(bf.put(d["u"])); a.u_stride = 2
    a.z = ptr(bf.put(d["z"]))
    if valid is not None:
        a.z_valid = ptr(bf.put(valid.astype(np.uint8), dtype=np.uint8))
    outs = {}
    shp = _shapes(c, N)
    for k in c.outs:
        outs[k] = bf.out(shp[k], mis)
        setattr(r if k == "z_record" else a, k, ptr(outs[k]))
    st = bf.out((N,), dtype=np.int32, fill=STATUS_FILL)
    a.status = ptr(st)
    if c.form == CORR:
        Mv = bf.put(d["M"], c.mis == "M")
        rc, err = call("bke_kf_step_correlated", ctypes.byref(a), ptr(Mv), 0 if d["M"].ndim == 2 else n * m)
    else:
        r.start, r.rows = c.start, L
        if c.Hi:
            r.H_i = ptr(bf.put(d["Hi"])); r.H_i_stride = 0 if d["Hi"].ndim == 2 else L * n
        if c.Ri:
            r.R_i = ptr(bf.put(d["Ri"])); r.R_i_stride = 0 if d["Ri"].ndim == 2 else L * L
        rc, err = call("bke_kf_update_rows", ctypes.byref(r))
    if rc:
        return rc, err, None, d, valid, kind
    bf.check_guards()
    got = dict(x=xo.cpu().numpy().reshape(N, n), P=Po.cpu().numpy().reshape(N, n, n), status=st.cpu().numpy())
    for k, v in outs.items():
        got[k] = v.cpu().numpy().reshape(shp[k])
    return rc, err, got, d, valid, kind


# ------------------------------------------------------------------------------------------ the oracle and the checks
def oracle(c, d, N, valid):
    """(x and P entering the update, the oracle's update dict) in fp64."""
    from oracle import kf as okf
    F, Q, H, R = (_full(d[k], N) for k in "FQHR")
    if c.mode & 1:
        B = _full(d["B"], N) if "B" in d else None
        xu, Pu = okf.kf_predict_bank(d["x"], d["P"], F, Q, ALPHA_SQ, B, d.get("u"))
    else:
        xu, Pu = d["x"], d["P"]
    st0 = np.full(N, STATUS_FILL, np.int32)
    if c.form == CORR:
        o = kfo.kf_update_correlated_bank(xu, Pu, d["z"], H, R, _full(d["M"], N), valid, st0, c.sticky)
    else:
        y0, K0 = np.full((N, c.m), SENT), np.full((N, c.n, c.m), SENT)
        o = kfo.kf_update_sequential_bank(xu, Pu, c.start, d["z"], H, R, y0, K0, y0.copy(),
                                          R_i=_full(d["Ri"], N) if c.Ri else None,
                                          H_i=_full(d["Hi"], N) if c.Hi else None, valid=valid, status=st0,
                                          sticky=c.sticky)
    return xu, Pu, o


def nclose(got, want, scale, cond, tol, what, label, rows=None):
    """close() for outputs that may hold inf / NaN (a one-row block with S_i = 0): got has NaN exactly where want
    does and the same infinities, and the finite entries are compared as close() does."""
    got = np.asarray(got, np.float64); want = np.asarray(want, np.float64)
    if rows is not None:
        got, want = got[rows], want[rows]
        scale = np.asarray(scale)[rows]
        cond = np.broadcast_to(np.asarray(cond, np.float64), rows.shape)[rows]
    assert np.array_equal(np.isnan(got), np.isnan(want)), "%s: the NaN pattern differs" % what
    if got.size:
        nan = np.isnan(want)
        close(np.where(nan, 0.0, got), np.where(nan, 0.0, want), scale, cond, tol, what, label, match_inf=True)


def _untouched(got, want_mask, what):
    assert np.all(got[~want_mask] == SENT), what + " written where it must be left alone"


def check(c, N, seed, edges=False, models=None):
    """One call of c against the oracle; returns what the call wrote."""
    rc, err, got, d, valid, kind = run(c, N, seed, edges, models)
    assert rc == 0, err
    n, m, L = c.n, c.m, c.L
    what = "%s N=%d seed=%d%s" % (c.id, N, seed, " edges" if edges else "")
    tol, label = TOL[c.fam][c.dt], "test_gpu_kf_forms_instances %s %s" % (c.fam, np.dtype(c.dt).name)
    xu, Pu, o = oracle(c, d, N, valid)
    v = np.ones(N, bool) if valid is None else valid
    sing = o["status"] == 1
    upd = v & ~sing
    assert np.array_equal(got["status"], o["status"]), what + " status"
    assert not sing[kind == EDGE_OK].any() and np.all(sing[(kind == SINGULAR)] == v[kind == SINGULAR]), what
    H = _full(d["H"], N)
    cond = np.ones(N)
    if c.form == CORR:
        S = o["S"]
        Mf = _full(d["M"], N)
        # S = H P H' + H M + M' H' + R sums terms of either sign: a solve with it is conditioned by
        # ||S^-1|| || |H P H'| + |H M| + |M' H'| + |R| || (cond(S) when nothing cancels), and S's own
        # rounding is relative to the terms, not to the sum
        HM = np.matmul(H, Mf)
        terms = (np.abs(np.matmul(np.matmul(H, Pu), np.swapaxes(H, 1, 2))) + np.abs(HM) + np.abs(np.swapaxes(HM, 1, 2))
                 + np.abs(_full(d["R"], N)))
        if upd.any():
            cond[upd] = np.linalg.norm(o["SI"][upd], 2, axis=(1, 2)) * np.linalg.norm(terms[upd], 2, axis=(1, 2))
        G = np.matmul(H, Pu) + np.swapaxes(Mf, 1, 2)
        KG = np.where(upd[:, None, None], np.matmul(np.nan_to_num(o["K"]), G), 0.0)
        sx = mag(d["x"], xu, o["x"]); sP = mag(Pu, o["P"], KG)
        close(got["x"], o["x"], sx, cond, tol, what + " x", label)
        close(got["P"], o["P"], sP, cond, tol, what + " P", label)
        Hb, zb = H, d["z"]
    else:
        s, e = c.start, c.start + L
        Hb = _full(d["Hi"], N) if c.Hi else H[:, s:e]
        Rb = _full(d["Ri"], N) if c.Ri else _full(d["R"], N)[:, s:e, s:e]
        Si = np.matmul(np.matmul(Hb, Pu), np.swapaxes(Hb, 1, 2)) + Rb
        if L > 1 and upd.any():
            cond[upd] = np.linalg.cond(Si[upd])
        zs = kind == ZERO_S
        assert np.all(Si[zs] == 0), what + " the S_i = 0 edge is not exactly zero"
        sx = mag(d["x"], xu, np.nan_to_num(o["x"], posinf=0, neginf=0))
        sP = mag(Pu, np.nan_to_num(o["P"], posinf=0, neginf=0))
        nclose(got["x"], o["x"], sx, cond, tol, what + " x", label)
        nclose(got["P"], o["P"], sP, cond, tol, what + " P", label)
        zb = d["z"]
    # a filter whose S is singular keeps the prior exactly: the predicted one, or the input without a predict
    for k in ("x", "P"):
        prior = got.get(k + "_prior") if c.mode & 1 else d[k]
        if prior is not None and sing.any():
            assert np.array_equal(got[k][sing], prior[sing]), what + " %s of a singular S is not the prior" % k
    for k, sc in (("x_prior", sx), ("P_prior", sP)):
        if k in got:
            if c.mode & 1:
                close(got[k], xu if k == "x_prior" else Pu, sc, 1.0, tol, what + " " + k, label)
            else:
                assert np.all(got[k] == SENT), what + " %s written without a predict" % k
    sy = np.abs(Hb).max(axis=(1, 2)) * np.abs(xu).sum(axis=1) + np.abs(zb).max(axis=1)
    if c.form == CORR:
        if "y" in got:
            close(got["y"], o["y"], sy, cond, tol, what + " y", label, upd)
            assert np.all(got["y"][~v] == 0), what + " y of a missed measurement"
            assert np.all(got["y"][sing] == SENT), what + " y of a singular S"
        # K = (P H' + M) SI: P H' and M cancel, so K is measured against (|P H'| + |M|) |SI|
        kscale = dict(K=mag(np.matmul(np.abs(np.matmul(Pu, np.swapaxes(H, 1, 2))) + np.abs(Mf),
                                      np.abs(np.nan_to_num(o["SI"])))), SI=mag(np.nan_to_num(o["SI"])))
        for k in ("K", "SI"):
            if k in got:
                close(got[k], o[k], kscale[k], cond, tol, what + " " + k, label, upd)
                assert np.all(got[k][~upd] == SENT), what + " %s written without an update" % k
        if "S" in got:
            close(got["S"], o["S"], mag(terms), 1.0, tol, what + " S", label, v)
            assert np.all(got["S"][~v] == SENT), what + " S written for a missed measurement"
        if "log_likelihood" in got:
            ll = np.full(N, np.nan)
            if upd.any():
                y, SI = o["y"][upd], o["SI"][upd]
                ll[upd] = -0.5 * (np.einsum("ni,nij,nj->n", y, SI, y) + np.linalg.slogdet(S[upd])[1]
                                  + m * np.log(2 * np.pi))
            close(got["log_likelihood"], ll, np.maximum(np.abs(np.nan_to_num(ll)), 1.0), cond, tol,
                  what + " log_likelihood", label, upd)
            assert np.all(got["log_likelihood"][~upd] == SENT), what + " log_likelihood written without an update"
    else:
        blk = np.zeros((N, m), bool)
        blk[upd, s:e] = True
        if "y" in got:
            nclose(got["y"][:, s:e], o["y"][:, s:e], sy, cond, tol, what + " y", label, upd)
            _untouched(got["y"], blk, what + " y")
        if "K" in got:
            Kb = o["K"][:, :, s:e]
            nclose(got["K"][:, :, s:e], Kb, mag(np.nan_to_num(Kb, posinf=0, neginf=0)), cond, tol, what + " K",
                   label, upd)
            _untouched(got["K"], np.broadcast_to(blk[:, None, :], got["K"].shape), what + " K")
        if "z_record" in got:
            assert np.array_equal(got["z_record"][upd, s:e], d["z"][upd]), what + " z_record"
            _untouched(got["z_record"], blk, what + " z_record")
    return got, kind, o


def _grid_N(c):
    import torch
    return 16 * torch.cuda.get_device_properties(0).multi_processor_count * warps_per_block(c.n, c.L, c.form, c.dt) + 37


def check_edges(c, N, seed):
    """The edge filters against the oracle, and every other filter bit-equal to the same bank without them."""
    clean, _, _ = check(c, N, seed, models="per")
    got, kind, o = check(c, N, seed, edges=True, models="per")
    ok = kind == EDGE_OK
    assert (~ok).sum() >= 1
    for k in clean:
        assert np.array_equal(clean[k][ok], got[k][ok]), "%s: %s of a healthy filter changed next to an edge" % (c.id, k)
    if c.form == CORR:
        S = o["S"]
        ind = kind == INDEFINITE
        if ind.any():
            assert np.all(np.linalg.eigvalsh(S[ind])[:, 0] < 0), "the indefinite edge is not indefinite"
        ill = kind == ILLCOND
        if ill.any():
            cd = np.linalg.cond(S[ill])
            assert np.all((cd > ILLCOND_COND[c.dt] / 10) & (cd < ILLCOND_COND[c.dt] * 10)), cd


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_instance_vs_oracle(case):
    """Every output and the status of one call against the fp64 oracle over the family's bank sizes (and a bank past
    the grid-stride threshold), then the edge filters inside a healthy bank; a shape the catch-all refuses returns
    BKE_ERR_UNSUPPORTED with the entry point's text."""
    from filterpy_b200 import _lib
    c = case
    if c.refused:
        rc, err, *_ = run(c, 3, seed=1)
        per = per_warp(c.n, c.L, c.form) * np.dtype(c.dt).itemsize
        assert rc == _lib.BKE_ERR_UNSUPPORTED, rc
        name = "bke_kf_step_correlated" if c.form == CORR else "bke_kf_update_rows"
        assert err == ("%s: dim_x=%d %s=%d needs %d B of shared memory per filter (> %d)"
                       % (name, c.n, "dim_z" if c.form == CORR else "rows", c.L, per, BUDGET)), err
        return
    Ns = c.Ns + ((_grid_N(c),) if c.grid else ())
    for i, N in enumerate(Ns):
        check(c, N, seed=N + 7 * i)
    check_edges(c, c.Ns[-1], seed=3)


# ------------------------------------------------------------------------------------------ refusals
def _rows_args(N=4, n=4, m=3, start=0, rows=1):
    from filterpy_b200 import _lib
    keep = [np.zeros((N, n)), np.zeros((N, n, n)), np.zeros((m, n)), np.eye(m), np.zeros((N, rows)), np.zeros(256)]
    r = _lib.KfRowsArgs()
    a = r.step
    a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags, a.alpha_sq = N, n, m, _lib.BKE_F64, _lib.BKE_DO_UPDATE, 1.0
    a.x = a.x_out = keep[0].ctypes.data; a.P = a.P_out = keep[1].ctypes.data
    a.H = keep[2].ctypes.data; a.R = keep[3].ctypes.data; a.z = keep[4].ctypes.data
    r.start, r.rows = start, rows
    return r, keep


def _refused(fn, *args):
    from filterpy_b200 import _lib
    lib = _lib.load()
    rc = getattr(lib, fn)(*args, None)
    return rc, lib.bke_last_error().decode()


STRIDE_TEXT = "model strides must be 0 (shared) or the dense per-filter size"


def test_refusals():
    """Each argument the two entry points refuse returns BKE_ERR_BAD_ARG with its text (before any device is
    needed)."""
    from filterpy_b200 import _lib
    BAD = _lib.BKE_ERR_BAD_ARG
    for start, rows in ((-1, 1), (0, 0), (2, 2), (3, 1), (0, 4)):
        r, keep = _rows_args(start=start, rows=rows)
        assert _refused("bke_kf_update_rows", ctypes.byref(r)) == (
            BAD, "the block of rows %d .. %d is not within the 3 rows of z" % (start, start + rows - 1))
    for field, stride in (("H_i", 5), ("R_i", 2)):
        r, keep = _rows_args(rows=2)
        setattr(r, field, keep[5].ctypes.data)
        setattr(r, field + "_stride", stride)
        assert _refused("bke_kf_update_rows", ctypes.byref(r)) == (BAD, STRIDE_TEXT)
    for field in ("S", "SI", "log_likelihood"):
        r, keep = _rows_args()
        setattr(r.step, field, keep[5].ctypes.data)
        assert _refused("bke_kf_update_rows", ctypes.byref(r)) == (
            BAD, "update_rows does not write S, SI or log_likelihood: they must be NULL")
    r, keep = _rows_args()
    r.step.flags = _lib.BKE_DO_PREDICT
    r.step.F = r.step.Q = keep[5].ctypes.data
    assert _refused("bke_kf_update_rows", ctypes.byref(r)) == (BAD, "flags must hold BKE_DO_UPDATE")
    # bke_kf_step_correlated
    r, keep = _rows_args()
    a = r.step
    M = keep[5].ctypes.data
    assert _refused("bke_kf_step_correlated", ctypes.byref(a), None, 0) == (BAD, "M is NULL")
    for stride in (7, 4 * 3 + 1, -12):
        assert _refused("bke_kf_step_correlated", ctypes.byref(a), M, stride) == (BAD, STRIDE_TEXT)
    a.flags = _lib.BKE_DO_PREDICT
    a.F = a.Q = M
    assert _refused("bke_kf_step_correlated", ctypes.byref(a), M, 0) == (BAD, "flags must hold BKE_DO_UPDATE")


@pytest.mark.gpu
@pytest.mark.parametrize("form", [CORR, ROWS], ids=["corr", "rows"])
def test_empty_bank_writes_nothing(form):
    """N = 0 returns BKE_OK and writes nothing."""
    from filterpy_b200 import _lib
    c = Case(form, "direct", F64, 4, 2, [], (1,), L=1, start=1, outs=CORR_OUTS if form == CORR else ROWS_OUTS)
    d, _ = _inputs(c, 1, 0, False, "per")
    bf = Bufs(F64)
    r = _lib.KfRowsArgs()
    a = _lib.KfArgs() if form == CORR else r.step
    a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags, a.alpha_sq = 0, 4, 2, _lib.BKE_F64, 3, 1.0
    a.x, a.P = ptr(bf.put(d["x"])), ptr(bf.put(d["P"]))
    a.x_out, a.P_out = ptr(bf.out((1, 4))), ptr(bf.out((1, 4, 4)))
    for k in "FQHR":
        setattr(a, k, ptr(bf.put(d[k])))
    a.z = ptr(bf.put(d["z"]))
    shp = _shapes(c, 1)
    for k in c.outs:
        setattr(r if k == "z_record" else a, k, ptr(bf.out(shp[k])))
    a.status = ptr(bf.out((1,), dtype=np.int32, fill=STATUS_FILL))
    if form == CORR:
        rc, err = call("bke_kf_step_correlated", ctypes.byref(a), ptr(bf.put(d["M"])), 8)
    else:
        r.start, r.rows = 1, 1
        rc, err = call("bke_kf_update_rows", ctypes.byref(r))
    assert rc == _lib.BKE_OK, err
    bf.check_guards()
    for buf, off, cnt, _ in bf.outs:
        h = buf.cpu().numpy()[off:off + cnt]
        assert np.all(h == (STATUS_FILL if h.dtype.kind == "i" else SENT))


# ------------------------------------------------------------------------------------------ which kernel runs
def _profiled_names():
    """The kernel names of every CASES entry run once, in launch order."""
    def go():
        for c in CASES:
            run(c, c.Ns[min(1, len(c.Ns) - 1)], seed=1)
    return profiled_names(go, r"kf_direct_kernel|kf_generic_kernel")


@pytest.mark.gpu
def test_dispatch_runs_the_kernels_of_the_table():
    """Each CASES entry, run once, launches the kernels the table names, template arguments included (a refused shape
    none), through every fall-through route to the catch-all."""
    check_launch_order("test_gpu_kf_forms_instances", [(c.id, c.kernels) for c in CASES])
