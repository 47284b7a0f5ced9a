"""GPU parity of the bank resamplers (csrc/resample_bank.cu): every row equals the reference's
systematic / stratified resample of that row bit for bit, for any weights and uniforms."""
import numpy as np
import pytest

from oracle import resample as ors

pytestmark = pytest.mark.gpu

KINDS = ["heavy", "uniform", "zeros", "degenerate", "dyadic", "random"]


def _bank(B, M, seed):
    from filterpy_b200.common import workloads as wl
    return np.stack([wl.resample_weights(M, KINDS[b % len(KINDS)], seed=seed + b) for b in range(B)]) if B else \
        np.zeros((0, M))


def _run(w, u=None, U=None):
    import torch
    from filterpy_b200.monte_carlo import BankResamplePlan
    B, M = w.shape
    plan = BankResamplePlan(B, M)
    wd = torch.from_numpy(np.ascontiguousarray(w)).cuda()
    if U is None:
        idx = plan.systematic(wd, torch.from_numpy(np.ascontiguousarray(u, dtype=np.float64)).cuda())
    else:
        idx = plan.stratified(wd, torch.from_numpy(np.ascontiguousarray(U, dtype=np.float64)).cuda())
    return idx.cpu().numpy(), plan.status.cpu().numpy()


def _check(w, u=None, U=None, loop=False):
    """Every row against the C oracle (and the pure-Python literal loop for small banks); a row the
    reference fails on must be flagged, and only that row."""
    idx, status = _run(w, u, U)
    assert idx.dtype == np.int32 and idx.shape == w.shape
    for b in range(w.shape[0]):
        try:
            ref = ors.systematic_resample_c(w[b], u[b]) if U is None else ors.stratified_resample_c(w[b], U[b])
        except IndexError:
            assert status[b] == 1, b
            continue
        assert status[b] == 0, b
        assert np.array_equal(idx[b], ref), (b, np.flatnonzero(idx[b] != ref)[:5])
        if loop:
            pos = ors.positions_systematic(w.shape[1], u[b]) if U is None else ors.positions_stratified(w.shape[1], U[b])
            assert np.array_equal(idx[b], ors.resample_loop(w[b], pos)), b
    return idx, status


@pytest.mark.parametrize("B,M", [(1, 1), (3, 7), (1000, 1), (257, 4099), (4096, 1024), (16, 65536), (2, 1 << 20),
                                 (130, 1001)])
def test_bank_equals_reference_per_row(B, M):
    rng = np.random.default_rng(B * 7 + M)
    w = _bank(B, M, seed=B + M)
    _check(w, u=rng.random(B), loop=B * M <= 64)
    _check(w, U=rng.random((B, M)), loop=B * M <= 64)


def _special_rows(M, rng):
    rows = []
    r = rng.random(M); r[::5] *= -1; rows.append(r / np.abs(r).sum())                    # negative weights
    r = rng.random(M) / M; r[M // 2] = np.nan; rows.append(r)                            # NaN
    r = rng.random(M) / M; r[3] = np.inf; rows.append(r)                                 # +inf
    r = rng.random(M) / M; r[1] = -np.inf; r[2] = np.inf; rows.append(r)                 # -inf then +inf (NaN sum)
    r = np.full(M, -0.0); r[-1] = 1.0; rows.append(r)                                    # signed zeros
    r = np.full(M, 5e-324); r[M // 3] = 1.0; rows.append(r)                              # subnormals
    rows.append(np.full(M, 1.0 / M))                                                     # ties with u = 0
    r = np.zeros(M); r[0] = 1.0; rows.append(r)
    r = rng.random(M); rows.append(2.0 * r / r.sum())                                    # unnormalised, sum 2
    r = rng.random(M); rows.append(0.5 * r / r.sum())                                    # sum 0.5: IndexError
    return np.stack(rows)


@pytest.mark.parametrize("M", [5, 37, 96, 4099])
def test_special_values_and_ties(M):
    rng = np.random.default_rng(M)
    w = _special_rows(M, rng)
    B = w.shape[0]
    _check(w, u=np.zeros(B), loop=M <= 96)
    _check(w, u=rng.random(B), loop=M <= 96)
    # u outside [0, 1): the reference accepts any float
    _check(w, u=np.array([-0.5, 1.5, -3.0, 0.999, 7.25, -0.0, 1e-300, 0.5, 2.0, -1e9][:B]), loop=M <= 96)
    U = rng.random((B, M))
    U[0] = -U[0]                      # below 0
    U[1] = U[1] + 1.5                 # above 1
    U[2] = np.sort(U[2])[::-1] * 3    # decreasing, large
    U[3, ::2] = np.nan
    U[4] = -np.arange(M, dtype=float)  # positions all at or below 0
    U[6] = 0.0                        # ties with w = 1/M
    _check(w, U=U, loop=M <= 96)


def test_overflow_marks_only_its_rows():
    rng = np.random.default_rng(5)
    w = _bank(40, 333, seed=9)
    bad = [3, 17, 39]
    w[bad] *= 0.75
    idx, status = _check(w, u=rng.random(40))
    assert np.flatnonzero(status).tolist() == bad


def test_b1_equals_single_set_path():
    import torch
    from filterpy_b200.monte_carlo import ResamplePlan
    for M, kind in ((1, "heavy"), (4096, "heavy"), (100003, "zeros"), (65536, "dyadic")):
        w = _bank(1, M, seed=M)
        if kind != "heavy":
            from filterpy_b200.common import workloads as wl
            w = wl.resample_weights(M, kind, seed=M)[None]
        for u in (0.0, 0.31337, 0.999999):
            idx, status = _run(w, u=np.array([u]))
            one = ResamplePlan(M).systematic(torch.from_numpy(w[0]).cuda(), u).cpu().numpy()
            assert status[0] == 0 and np.array_equal(idx[0], one), (M, u)


def test_seeded_mirrors_reproduce_golden(golden):
    from filterpy_b200.monte_carlo import systematic_resample_bank, stratified_resample_bank
    g = golden("resample_bank")
    for (k, B, M, seed, sys_fail, str_fail) in g["meta"]:
        w = g["w%d" % k]
        for kind, fail, fn in (("sys", sys_fail, systematic_resample_bank), ("str", str_fail, stratified_resample_bank)):
            np.random.seed(seed)
            if fail >= 0:
                with pytest.raises(IndexError, match="set %d:" % fail):
                    fn(w)
                continue
            idx = fn(w)
            assert isinstance(idx, np.ndarray) and idx.dtype == np.int32
            assert np.array_equal(idx, g["%s%d" % (kind, k)]), (kind, k)
            assert np.random.random() == g["%s_next%d" % (kind, k)], (kind, k)


def test_mirrors_take_tensors_and_empty_banks():
    import torch
    from filterpy_b200.monte_carlo import systematic_resample_bank, stratified_resample_bank
    w = _bank(9, 50, seed=3)
    np.random.seed(1)
    a = systematic_resample_bank(torch.from_numpy(w).cuda())
    np.random.seed(1)
    b = systematic_resample_bank(w)
    assert a.is_cuda and a.dtype == torch.int32 and np.array_equal(a.cpu().numpy(), b)
    for shape in ((0, 5), (4, 0), (0, 0)):
        for fn, drawn in ((systematic_resample_bank, shape[0]), (stratified_resample_bank, shape)):
            np.random.seed(2)
            out = fn(np.zeros(shape))
            after = np.random.random()
            np.random.seed(2)
            np.random.random(drawn)                       # the loop of the reference draws these for its rows
            assert out.shape == shape and out.dtype == np.int32
            assert after == np.random.random()
    with pytest.raises(ValueError):
        systematic_resample_bank(np.full(8, 0.125))        # 1-D input is not a bank


@pytest.mark.parametrize("dtype,tail", [(np.float32, (4,)), (np.float64, (2,)), (np.uint8, (3,)), (np.float32, ())])
@pytest.mark.parametrize("index_dtype", [np.int32, np.int64])
def test_gather_bank(dtype, tail, index_dtype):
    import torch
    from filterpy_b200.monte_carlo import gather_particles_bank
    rng = np.random.default_rng(11)
    B, M = 37, 129
    p = (rng.random((B, M) + tail) * 200).astype(dtype)
    idx = rng.integers(0, M, size=(B, M)).astype(index_dtype)
    ref = np.stack([p[b][idx[b]] for b in range(B)])
    assert np.array_equal(gather_particles_bank(p, idx), ref)
    out = gather_particles_bank(torch.from_numpy(p).cuda(), torch.from_numpy(idx).cuda())
    assert out.is_cuda and np.array_equal(out.cpu().numpy(), ref)
    for v in (M, -1):
        bad = idx.copy()
        bad[5, 7] = v
        with pytest.raises(IndexError):
            gather_particles_bank(p, bad)


def test_plan_gather_and_graph_capture():
    import torch
    from filterpy_b200._dev import StepGraph
    from filterpy_b200.monte_carlo import BankResamplePlan
    B, M = 300, 257
    rng = np.random.default_rng(4)
    w = torch.from_numpy(_bank(B, M, seed=8)).cuda()
    u = torch.from_numpy(rng.random(B)).cuda()
    U = torch.from_numpy(rng.random((B, M))).cuda()
    parts = torch.from_numpy(rng.random((B, M, 4)).astype(np.float32)).cuda()
    plan = BankResamplePlan(B, M)
    idx_s = torch.empty((B, M), dtype=torch.int32, device="cuda")
    gathered = torch.empty_like(parts)

    def step():
        plan.systematic(w, u, out=idx_s)
        plan.stratified(w, U)
        plan.gather(parts, out=gathered)

    step()
    torch.cuda.synchronize()
    want_s, want_t, want_g = idx_s.clone(), plan.indexes.clone(), gathered.clone()
    ref_g = torch.stack([parts[b][want_t[b].long()] for b in range(B)])
    assert torch.equal(want_g, ref_g)
    plan.raise_if_overflow()
    plan.raise_if_bad_index()
    g = StepGraph(step, torch.device("cuda", torch.cuda.current_device()))
    for t in (idx_s, plan.indexes, gathered):
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(idx_s, want_s) and torch.equal(plan.indexes, want_t) and torch.equal(gathered, want_g)
    # a new offset in the same buffer is picked up by the replay
    u.copy_(torch.from_numpy(rng.random(B)))
    g.replay()
    torch.cuda.synchronize()
    wn = w.cpu().numpy()
    un = u.cpu().numpy()
    for b in range(0, B, 37):
        assert np.array_equal(idx_s[b].cpu().numpy(), ors.systematic_resample_c(wn[b], un[b]))


def test_torch_ops_equal_mirror():
    import torch
    from filterpy_b200 import torch_ops
    from filterpy_b200.monte_carlo import BankResamplePlan
    ops = torch_ops.load()
    B, M = 70, 513
    rng = np.random.default_rng(6)
    w = torch.from_numpy(_bank(B, M, seed=2)).cuda()
    u = torch.from_numpy(rng.random(B)).cuda()
    U = torch.from_numpy(rng.random((B, M))).cuda()
    plan = BankResamplePlan(B, M)
    assert torch.equal(ops.systematic_resample_bank(w, u), plan.systematic(w, u).clone())
    assert torch.equal(ops.stratified_resample_bank(w, U), plan.stratified(w, U).clone())
    w2 = w.clone()
    w2[11] *= 0.5
    with pytest.raises(IndexError, match="set 11"):
        ops.systematic_resample_bank(w2, u)


def test_plan_gather_reports_bad_indexes_and_checks_its_arguments():
    import torch
    from filterpy_b200.monte_carlo import BankResamplePlan
    B, M = 20, 65
    rng = np.random.default_rng(12)
    plan = BankResamplePlan(B, M)
    parts = torch.from_numpy(rng.random((B, M, 3))).cuda()
    idx = torch.from_numpy(rng.integers(0, M, size=(B, M)).astype(np.int32)).cuda()
    out = plan.gather(parts, idx)
    plan.raise_if_bad_index()
    assert torch.equal(out, torch.stack([parts[b][idx[b].long()] for b in range(B)]))
    idx[4, 9] = M
    plan.gather(parts, idx)
    with pytest.raises(IndexError):
        plan.raise_if_bad_index()
    plan.raise_if_bad_index()                        # the flag was cleared by the report
    idx[4, 9] = 0
    big = torch.zeros((B, M, 8), dtype=torch.float64, device="cuda")
    for bad_parts, bad_idx in ((big[:, :, :3], idx), (parts.cpu(), idx), (parts[:, :M - 1], idx),
                               (parts, idx.to(torch.int16)), (parts, idx.t().contiguous().t()), (parts, idx[:, :M - 1])):
        with pytest.raises(ValueError):
            plan.gather(bad_parts, bad_idx)
    w = torch.full((B, M), 1.0 / M, dtype=torch.float64, device="cuda")
    u = torch.full((B,), 0.5, dtype=torch.float64, device="cuda")
    for args in ((w.cpu(), u), (w, u.cpu()), (w[:, :M - 1], u), (w.float(), u)):
        with pytest.raises(ValueError):
            plan.systematic(*args)
    with pytest.raises(ValueError):
        plan.systematic(w, u, out=torch.empty((B, M), dtype=torch.int64, device="cuda"))
