"""GPU parity of the multinomial / residual bank resamplers (csrc/resample_bank.cu): every row equals the
reference's multinomial_resample / residual_resample of that row bit for bit, for any weights and uniforms."""
import numpy as np
import pytest

from oracle import resample as ors
import resample_bank_mr_oracle as mro

pytestmark = pytest.mark.gpu

KINDS = ["heavy", "uniform", "zeros", "degenerate", "dyadic", "random"]


def _bank(B, M, seed):
    from filterpy_b200.common import workloads as wl
    return np.stack([wl.resample_weights(M, KINDS[b % len(KINDS)], seed=seed + b) for b in range(B)])


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype=a.dtype)).cuda()


def _mul(w, U):
    from filterpy_b200.monte_carlo import BankResamplePlan
    plan = BankResamplePlan(*w.shape)
    idx = plan.multinomial(_cuda(w), _cuda(U)).cpu().numpy()
    return idx, plan.status.cpu().numpy()


def _res(w, U):
    from filterpy_b200.monte_carlo import BankResamplePlan
    plan = BankResamplePlan(*w.shape)
    idx = plan.residual(_cuda(w), _cuda(U)).cpu().numpy()
    return idx, plan.n_copies.cpu().numpy(), plan.status.cpu().numpy()


def _check(w, U, literal=False):
    """Both resamplers against the NumPy oracle (and binsearch_left when ``literal``); returns the statuses."""
    M = w.shape[1]
    idx, st_m = _mul(w, U)
    assert idx.dtype == np.int64 and (st_m & 1).sum() == 0
    assert np.array_equal(idx, mro.multinomial_bank(w, U))
    ridx, k, st_r = _res(w, U)
    ref, kr, bad = mro.residual_bank(w, U)
    assert ridx.dtype == np.int32
    assert np.array_equal(np.flatnonzero(st_r & 1), bad)
    ok = k <= M
    assert np.array_equal(k[ok], kr[ok]) and (kr[~ok] > M).all()
    assert np.array_equal(ridx[ok], ref[ok])
    if literal:
        with np.errstate(all="ignore"):
            for b in range(w.shape[0]):
                c = np.cumsum(w[b]); c[-1] = 1.
                assert np.array_equal(idx[b], ors.binsearch_left(c, U[b])), b
                if ok[b]:
                    assert np.array_equal(ridx[b], ors.residual_resample_vec(w[b], U[b, :M - k[b]])), b
    return st_m, st_r


@pytest.mark.parametrize("B,M", [(1, 1), (3, 7), (1000, 1), (257, 4099), (4096, 1024), (16, 65536), (2, 1 << 20)])
def test_bank_equals_reference_per_row(B, M):
    rng = np.random.default_rng(B * 5 + M)
    w = _bank(B, M, seed=B + M)
    _check(w, rng.random((B, M)), literal=B * M <= 64)


def _special_rows(M, rng):
    rows = []
    r = rng.random(M); r[::5] *= -1; rows.append(r / np.abs(r).sum())                    # negative weights
    r = rng.random(M) / M; r[M // 2] = np.nan; rows.append(r)                            # NaN
    r = rng.random(M) / M; r[3] = np.inf; rows.append(r)                                 # +inf
    r = rng.random(M) / M; r[1] = -np.inf; rows.append(r)                                # -inf
    r = rng.random(M) / M; r[1] = -np.inf; r[2] = np.inf; rows.append(r)                 # NaN sum
    r = np.full(M, -0.0); r[-1] = 1.0; rows.append(r)                                    # signed zeros
    r = np.full(M, 5e-324); r[M // 3] = 1.0; rows.append(r)                              # subnormals
    rows.append(np.full(M, 1.0 / M))                                                     # ties
    r = rng.random(M); rows.append(2.0 * r / r.sum())                                    # c[M-2] > 1
    r = rng.random(M) ** 4; rows.append(1.5 * r / r.sum())                               # k > M (residual)
    r = rng.random(M); rows.append(1e300 * r)                                            # M w beyond int64
    return np.stack(rows)


@pytest.mark.parametrize("M", [5, 37, 96, 4099])
def test_special_values(M):
    rng = np.random.default_rng(M)
    w = _special_rows(M, rng)
    B = w.shape[0]
    _, st_r = _check(w, rng.random((B, M)), literal=M <= 96)
    assert st_r[9] & 1                                     # the 1.5-scaled row fails in residual


@pytest.mark.parametrize("M", [7, 64, 1000])
def test_keys_outside_unit_interval_and_out_of_order(M):
    """Sorted cumulative sums with keys outside [0, 1), NaN or in reverse order: the per-key search and the
    carried-bracket search both give NumPy's answer; a row whose c[M-2] > 1 is routed to the exact path."""
    rng = np.random.default_rng(M + 1)
    w = _bank(8, M, seed=M)
    w[7] *= 2.0
    U = rng.random((8, M))
    U[0] = -U[0]
    U[1] = U[1] + 1.5
    U[2] = np.sort(U[2])[::-1]
    U[3] = np.sort(U[3])[::-1] * 3
    U[4, ::2] = np.nan
    U[5] = np.linspace(2, -1, M)
    U[7] = np.linspace(0, 2.5, M)
    st_m, _ = _check(w, U, literal=True)
    assert st_m[7] == 2 and (st_m[:7] == 0).all()


def test_seeded_mirrors_reproduce_golden(golden):
    from filterpy_b200.monte_carlo import multinomial_resample_bank, residual_resample_bank
    g = golden("resample_bank_mr")
    for (k, B, M, seed, mul_fail, res_fail) in g["meta"]:
        w = g["w%d" % k]
        np.random.seed(seed)
        idx = multinomial_resample_bank(w)
        assert isinstance(idx, np.ndarray) and idx.dtype == np.int64
        assert np.array_equal(idx, g["mul%d" % k]) and np.random.random() == g["mul_next%d" % k], k
        np.random.seed(seed)
        if res_fail >= 0:
            with pytest.raises(IndexError, match="set %d:" % res_fail):
                residual_resample_bank(w)
            # the loop drew random(M - k_b) for the rows before the failing one, and nothing more
            _, kk, _ = mro.residual_prepare_bank(w)
            nxt = np.random.random()
            np.random.seed(seed)
            np.random.random(int((M - kk[:res_fail]).sum()))
            assert nxt == np.random.random(), k
            continue
        idx = residual_resample_bank(w)
        assert isinstance(idx, np.ndarray) and idx.dtype == np.int32
        assert np.array_equal(idx, g["res%d" % k]) and np.random.random() == g["res_next%d" % k], k


def test_b1_equals_single_set_mirrors():
    from filterpy_b200.monte_carlo import (multinomial_resample, residual_resample, multinomial_resample_bank,
                                           residual_resample_bank)
    for M, kind in ((1, "heavy"), (1000, "heavy"), (4099, "zeros"), (65536, "dyadic"), (5000, "uniform")):
        w = _bank(1, M, seed=M) if kind == "heavy" else __import__(
            "filterpy_b200.common.workloads", fromlist=["x"]).resample_weights(M, kind, seed=M)[None]
        np.random.seed(M)
        one = residual_resample(w[0])
        np.random.seed(M)
        assert np.array_equal(residual_resample_bank(w)[0], one), (M, kind)
        np.random.seed(M)
        one = multinomial_resample(w[0])
        np.random.seed(M)
        assert np.array_equal(multinomial_resample_bank(w)[0], one), (M, kind)


def test_mirrors_take_tensors_and_empty_banks():
    import torch
    from filterpy_b200.monte_carlo import multinomial_resample_bank, residual_resample_bank
    w = _bank(9, 50, seed=3)
    for fn, dt in ((multinomial_resample_bank, torch.int64), (residual_resample_bank, torch.int32)):
        np.random.seed(1)
        a = fn(torch.from_numpy(w).cuda())
        np.random.seed(1)
        b = fn(w)
        assert a.is_cuda and a.dtype == dt and np.array_equal(a.cpu().numpy(), b)
        np.random.seed(2)
        out = fn(np.zeros((0, 5)))
        assert out.shape == (0, 5)
        after = np.random.random()
        np.random.seed(2)
        assert after == np.random.random()
        np.random.seed(2)
        with pytest.raises(IndexError, match="set 0"):
            fn(np.zeros((3, 0)))
        after = np.random.random()
        np.random.seed(2)
        assert after == np.random.random()                  # the reference fails before drawing
        with pytest.raises(ValueError):
            fn(np.full(8, 0.125))


def test_plan_graph_capture():
    import torch
    from filterpy_b200._dev import StepGraph
    from filterpy_b200.monte_carlo import BankResamplePlan
    B, M = 300, 257
    rng = np.random.default_rng(4)
    w = torch.from_numpy(_bank(B, M, seed=8)).cuda()
    U = torch.from_numpy(rng.random((B, M))).cuda()
    plan = BankResamplePlan(B, M)
    mul = torch.empty((B, M), dtype=torch.int64, device="cuda")

    def step():
        plan.multinomial(w, U, out=mul)
        plan.residual(w, U)

    step()
    torch.cuda.synchronize()
    want_m, want_r = mul.clone(), plan.indexes.clone()
    g = StepGraph(step, torch.device("cuda", torch.cuda.current_device()))
    mul.zero_()
    plan.indexes.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(mul, want_m) and torch.equal(plan.indexes, want_r)
    U.copy_(torch.from_numpy(rng.random((B, M))))
    g.replay()
    torch.cuda.synchronize()
    wn, Un = w.cpu().numpy(), U.cpu().numpy()
    assert np.array_equal(mul.cpu().numpy(), mro.multinomial_bank(wn, Un))
    assert np.array_equal(plan.indexes.cpu().numpy(), mro.residual_bank(wn, Un)[0])


def test_torch_ops_equal_mirror():
    import torch
    from filterpy_b200 import torch_ops
    from filterpy_b200.monte_carlo import BankResamplePlan
    ops = torch_ops.load()
    B, M = 70, 513
    rng = np.random.default_rng(6)
    w = torch.from_numpy(_bank(B, M, seed=2)).cuda()
    U = torch.from_numpy(rng.random((B, M))).cuda()
    plan = BankResamplePlan(B, M)
    assert torch.equal(ops.multinomial_resample_bank(w, U), plan.multinomial(w, U).clone())
    assert torch.equal(ops.residual_resample_bank(w, U), plan.residual(w, U).clone())
    w2 = w.clone()
    w2[11] *= 1.5
    w2[11, 0] += 1.0
    with pytest.raises(IndexError, match="set 11"):
        ops.residual_resample_bank(w2, U)
    with pytest.raises(RuntimeError):
        ops.multinomial_resample_bank(w, U[:, :-1].contiguous())
