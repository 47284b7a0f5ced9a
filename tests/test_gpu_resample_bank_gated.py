"""GPU parity of the gated bank resampler (csrc/resample_bank.cu: k_gated_stats, k_resample_bank<., RowList>,
k_gather_reset): every row is normalised, gated, resampled and gathered as the per-set loop of a particle
filter does it, bit for bit."""
import numpy as np
import pytest

from oracle import resample as ors
import resample_bank_gated_oracle as rgo
from test_gpu_resample_bank import _special_rows

pytestmark = pytest.mark.gpu

KINDS = ["heavy", "uniform", "random", "zeros", "degenerate", "dyadic"]
PARTICLES = [(np.float32, (4,)), (np.float64, (6,)), (np.float32, (3,)), (np.int8, ())]


def _bank(B, M, seed):
    from filterpy_b200.common import workloads as wl
    w = np.stack([wl.resample_weights(M, KINDS[b % len(KINDS)], seed=seed + b) for b in range(B)])
    w[1::7] *= 3.0                               # unnormalised rows
    w[2::11] *= 1e-200
    return w


def _particles(B, M, dtype, tail, seed):
    rng = np.random.default_rng(seed)
    if dtype == np.int8:
        return rng.integers(-128, 128, size=(B, M) + tail).astype(np.int8)
    return (rng.standard_normal((B, M) + tail) * 100).astype(dtype)


def _same_bits(a, b):
    """Equal as floats bit for bit, NaN compared as NaN (x86's 0/0 sets the sign bit, the GPU's does not)."""
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint64), b[~nb].view(np.uint64))


def _gpu(w, p, u=None, U=None, threshold=None):
    import torch
    from filterpy_b200.monte_carlo import BankResamplePlan
    B, M = w.shape
    plan = BankResamplePlan(B, M)
    wd = torch.from_numpy(np.ascontiguousarray(w)).cuda()
    pd = torch.from_numpy(np.ascontiguousarray(p)).cuda()
    ud = torch.from_numpy(u).cuda() if u is not None else None
    Ud = torch.from_numpy(U).cuda() if U is not None else None
    res, neff = plan.resample_if_degenerate(wd, pd, u=ud, uniforms=Ud, threshold=threshold)
    return dict(weights=wd.cpu().numpy(), particles=pd.cpu().numpy(), resampled=res.cpu().numpy(),
                neff=neff.cpu().numpy(), indexes=plan.indexes.cpu().numpy(), status=plan.status.cpu().numpy())


def _oracle(w, u=None, U=None, threshold=None):
    """The loop, given the bank's per-row draws: the k-th resampled set takes its own row's draw."""
    B, M = w.shape
    thr = M / 2 if threshold is None else threshold
    with np.errstate(all="ignore"):
        mask = np.array([1. / np.sum(np.square(w[b] / np.sum(w[b]))) < thr for b in range(B)], bool)
    if U is None:
        return rgo.resample_if_degenerate_loop(w, np.zeros((B, M), np.int8), u[mask], threshold,
                                               "systematic", ors.systematic_resample_c)
    return rgo.resample_if_degenerate_loop(w, np.zeros((B, M), np.int8), U[mask], threshold,
                                           "stratified", ors.stratified_resample_c)


def _check(w, p, u=None, U=None, threshold=None, o=None):
    o = _oracle(w, u, U, threshold) if o is None else o
    g = _gpu(w, p, u, U, threshold)
    assert np.array_equal(g["resampled"], o["resampled"])
    assert _same_bits(g["neff"], o["neff"])
    assert _same_bits(g["weights"], o["weights"])
    failed = np.zeros(w.shape[0], bool)
    failed[o["failed"]] = True
    assert np.array_equal(g["status"] == 1, failed)
    ok = o["resampled"] & ~failed
    assert np.array_equal(g["indexes"][ok], o["indexes"][ok])
    want = p.copy()
    for b in np.flatnonzero(ok):
        want[b] = p[b][o["indexes"][b]]
    assert g["particles"].tobytes() == want.tobytes()        # untouched rows byte for byte
    return o, g


@pytest.mark.parametrize("B,M", [(1, 1), (3, 7), (1000, 1), (130, 1001), (257, 4099), (4096, 1024), (1 << 16, 64)])
def test_bank_equals_the_loop_per_row(B, M):
    rng = np.random.default_rng(B * 5 + M)
    w = _bank(B, M, seed=B + M)
    u, U = rng.random(B), rng.random((B, M))
    types = PARTICLES if B * M <= 1 << 20 else PARTICLES[::3]
    o_s, o_t = _oracle(w, u=u), _oracle(w, U=U)
    assert M < 8 or (0 < o_s["resampled"].sum() < B)      # M = 1: neff = 1 is never below 1 / 2
    for i, (dtype, tail) in enumerate(types):
        p = _particles(B, M, dtype, tail, seed=i)
        _check(w, p, u=u, o=o_s)
        _check(w, p, U=U, o=o_t)


@pytest.mark.parametrize("M", [5, 37, 130, 4099])
def test_special_rows(M):
    rng = np.random.default_rng(M)
    w = _special_rows(M, rng)
    w = np.concatenate([w, np.zeros((1, M)), np.full((1, M), 1e-300)])
    B = w.shape[0]
    p = _particles(B, M, np.float32, (3,), seed=M)
    _check(w, p, u=rng.random(B))
    _check(w, p, U=rng.random((B, M)))
    _check(w, p, u=np.zeros(B))


def test_golden_through_the_plan_and_the_module_functions(golden):
    import torch
    from filterpy_b200.monte_carlo import (systematic_resample_bank_if_degenerate,
                                           stratified_resample_bank_if_degenerate)
    g = golden("resample_bank_gated")
    for (k, B, M, seed, sys_fail, str_fail) in g["meta"]:
        w, p = g["w%d" % k], g["p%d" % k]
        for kind, fail, fn in (("sys", sys_fail, systematic_resample_bank_if_degenerate),
                               ("str", str_fail, stratified_resample_bank_if_degenerate)):
            mask = g["%s_mask%d" % (kind, k)]
            ok = mask.copy()
            if fail >= 0:
                ok[fail] = False
            # the plan, with the draws the seeded loop takes
            np.random.seed(seed)
            n_res = int(mask.sum())
            if kind == "sys":
                u = np.zeros(B)
                u[mask] = np.random.random(n_res)
                r = _gpu(w, p, u=u)
            else:
                U = np.zeros((B, M))
                U[mask] = np.random.random((n_res, M))
                r = _gpu(w, p, U=U)
            assert np.array_equal(r["resampled"], mask) and _same_bits(r["neff"], g["%s_neff%d" % (kind, k)])
            assert _same_bits(r["weights"], g["%s_w%d" % (kind, k)]), (kind, k)
            assert np.array_equal(r["particles"], g["%s_p%d" % (kind, k)]), (kind, k)
            assert np.array_equal(r["indexes"][ok], g["%s_idx%d" % (kind, k)][ok]), (kind, k)
            assert np.array_equal(np.flatnonzero(r["status"]), [] if fail < 0 else [fail])
            # the seeded module functions, on arrays and on tensors, in place
            for as_tensor in (False, True):
                wa, pa = w.copy(), p.copy()
                if as_tensor:
                    wa, pa = torch.from_numpy(wa).cuda(), torch.from_numpy(pa).cuda()
                np.random.seed(seed)
                if fail >= 0:
                    with pytest.raises(IndexError, match="set %d:" % fail):
                        fn(wa, pa)
                    res = None
                else:
                    res, neff = fn(wa, pa)
                    assert np.random.random() == g["%s_next%d" % (kind, k)], (kind, k)
                if as_tensor:
                    wa, pa = wa.cpu().numpy(), pa.cpu().numpy()
                    res = res.cpu().numpy() if res is not None else None
                if res is not None:
                    assert res.dtype == np.bool_ and np.array_equal(res, mask)
                    assert _same_bits(np.asarray(neff.cpu() if hasattr(neff, "cpu") else neff),
                                      g["%s_neff%d" % (kind, k)])
                assert _same_bits(wa, g["%s_w%d" % (kind, k)]), (kind, k, as_tensor)
                assert np.array_equal(pa, g["%s_p%d" % (kind, k)]), (kind, k, as_tensor)


def test_threshold_zero_and_infinity():
    import torch
    from filterpy_b200.monte_carlo import BankResamplePlan, gather_particles_bank
    B, M = 300, 257
    rng = np.random.default_rng(3)
    w = _bank(B, M, seed=4)
    p = _particles(B, M, np.float32, (4,), seed=5)
    u, U = rng.random(B), rng.random((B, M))
    normalised = np.stack([w[b] / np.sum(w[b]) for b in range(B)])
    r = _gpu(w, p, u=u, threshold=0.0)
    assert not r["resampled"].any() and r["particles"].tobytes() == p.tobytes()
    assert _same_bits(r["weights"], normalised)
    nd = torch.from_numpy(normalised).cuda()
    for kw in (dict(u=u), dict(U=U)):
        r = _gpu(w, p, threshold=np.inf, **kw)
        assert r["resampled"].all() and not r["status"].any()
        plan = BankResamplePlan(B, M)
        idx = plan.systematic(nd, torch.from_numpy(u).cuda()) if "u" in kw else \
            plan.stratified(nd, torch.from_numpy(U).cuda())
        gathered = gather_particles_bank(torch.from_numpy(p).cuda(), idx).cpu().numpy()
        assert np.array_equal(r["indexes"], idx.cpu().numpy())
        assert r["particles"].tobytes() == gathered.tobytes()
        assert (r["weights"] == 1. / M).all()


def test_failing_row_keeps_its_particles(golden):
    from filterpy_b200.monte_carlo import systematic_resample_bank_if_degenerate
    g = golden("resample_bank_gated")
    k = int(np.flatnonzero(g["meta"][:, 4] >= 0)[0])
    bad = g["w%d" % k][int(g["meta"][k][4])]
    B, M = 12, bad.shape[0]
    w = _bank(B, M, seed=7)
    rows = [3, 10]
    w[rows] = bad
    p = _particles(B, M, np.float64, (6,), seed=1)
    o, r = _check(w, p, u=np.random.default_rng(2).random(B))
    assert o["failed"] == rows and np.flatnonzero(r["status"]).tolist() == rows
    for b in rows:
        assert r["resampled"][b] and r["particles"][b].tobytes() == p[b].tobytes()
        assert _same_bits(r["weights"][b], bad / np.sum(bad))
    wa, pa = w.copy(), p.copy()
    with pytest.raises(IndexError, match="set 3:"):
        systematic_resample_bank_if_degenerate(wa, pa)
    assert _same_bits(wa[3], bad / np.sum(bad)) and pa[3].tobytes() == p[3].tobytes()


def test_graph_capture_equals_eager_calls():
    import torch
    from filterpy_b200._dev import StepGraph
    from filterpy_b200.monte_carlo import BankResamplePlan
    B, M = 500, 200
    rng = np.random.default_rng(8)
    inputs = []
    for s in range(2):
        inputs.append((_bank(B, M, seed=20 + s), _particles(B, M, np.float32, (4,), seed=s), rng.random(B)))
    eager = []
    plan = BankResamplePlan(B, M)
    for w, p, u in inputs:
        wd, pd, ud = (torch.from_numpy(x.copy()).cuda() for x in (w, p, u))
        res, neff = plan.resample_if_degenerate(wd, pd, u=ud)
        eager.append((wd.clone(), pd.clone(), res.clone(), neff.clone(), plan.status.clone()))
    W = torch.empty((B, M), dtype=torch.float64, device="cuda")
    P = torch.empty((B, M, 4), dtype=torch.float32, device="cuda")
    Uu = torch.empty(B, dtype=torch.float64, device="cuda")
    gplan = BankResamplePlan(B, M)

    def load(i):
        w, p, u = inputs[i]
        W.copy_(torch.from_numpy(w)); P.copy_(torch.from_numpy(p)); Uu.copy_(torch.from_numpy(u))

    load(0)
    graph = StepGraph(lambda: gplan.resample_if_degenerate(W, P, u=Uu), torch.device("cuda", torch.cuda.current_device()))
    for i in range(2):
        load(i)
        graph.replay()
        torch.cuda.synchronize()
        wd, pd, res, neff, status = eager[i]
        assert torch.equal(W.isnan(), wd.isnan()) and torch.equal(W.nan_to_num(), wd.nan_to_num())
        assert torch.equal(P, pd) and torch.equal(gplan._resampled, res) and torch.equal(gplan.status, status)
        assert torch.equal(gplan._neff.nan_to_num(), neff.nan_to_num())


def test_torch_ops_equal_the_plan():
    import torch
    from filterpy_b200 import torch_ops
    ops = torch_ops.load()
    B, M = 70, 513
    rng = np.random.default_rng(6)
    w = _bank(B, M, seed=2)
    p = _particles(B, M, np.float32, (3,), seed=3)
    u, U = rng.random(B), rng.random((B, M))
    for name, kw, arg in (("systematic_resample_bank_if_degenerate", dict(u=u), u),
                          ("stratified_resample_bank_if_degenerate", dict(U=U), U)):
        ref = _gpu(w, p, threshold=200.0, **kw)
        wd, pd = torch.from_numpy(w.copy()).cuda(), torch.from_numpy(p.copy()).cuda()
        res, neff = getattr(ops, name)(wd, pd, torch.from_numpy(arg).cuda(), 200.0)
        assert res.dtype == torch.bool and np.array_equal(res.cpu().numpy(), ref["resampled"])
        assert _same_bits(neff.cpu().numpy(), ref["neff"]) and _same_bits(wd.cpu().numpy(), ref["weights"])
        assert pd.cpu().numpy().tobytes() == ref["particles"].tobytes()


def test_particle_row_over_the_cap_and_argument_checks():
    import torch
    from filterpy_b200.monte_carlo import BankResamplePlan
    cap = 227 * 1024                                  # the H100's opt-in shared memory per block
    for M, pb in ((4096, cap // 4096), (cap, 1)):      # rows of 224 KB and of exactly the cap: one particle
        w = torch.zeros((2, M), dtype=torch.float64, device="cuda")
        w[:, M // 2] = 1.0                            # neff = 1: both sets resample
        p = torch.arange(2 * M * pb, device="cuda").to(torch.uint8).view(2, M, pb)
        want = p[:, M // 2:M // 2 + 1].expand(2, M, pb).clone()
        plan = BankResamplePlan(2, M)
        res, _ = plan.resample_if_degenerate(w, p, u=torch.full((2,), 0.5, dtype=torch.float64, device="cuda"))
        assert bool(res.all()) and torch.equal(p, want) and bool((w == 1. / M).all())
    M = cap + 1                                       # one byte over
    plan = BankResamplePlan(2, M)
    w = torch.ones((2, M), dtype=torch.float64, device="cuda")
    p = torch.zeros((2, M), dtype=torch.int8, device="cuda")
    u = torch.full((2,), 0.5, dtype=torch.float64, device="cuda")
    with pytest.raises(ValueError, match="%d bytes.*gather_particles_bank" % cap):
        plan.resample_if_degenerate(w, p, u=u)
    assert bool((w == 1.0).all())                     # refused before the weights were touched
    with pytest.raises(ValueError):
        plan.resample_if_degenerate(w, p, u=u, uniforms=torch.zeros((2, M), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        plan.resample_if_degenerate(w, p[:, :M - 1].contiguous(), u=u)
    with pytest.raises(ValueError):
        plan.resample_if_degenerate(w.float(), p, u=u)
