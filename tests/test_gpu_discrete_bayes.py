"""GPU parity of the discrete Bayes filter banks (csrc/discrete_bayes.cu, filterpy_b200.discrete_bayes): every row
against the reference's goldens and the fp64 oracle, on the single-pass path (a row staged in one CTA) and the
multi-pass path (rows too long to stage), through the C-ABI, the Python bank forms, the drop-ins and the torch
operator.  Wrap mode, update and normalize are bit for bit; constant mode is bit for bit against the oracle's exact
shift and within the reference's spline roundoff against the reference."""
import ctypes

import numpy as np
import pytest

from gpu_harness import Bufs, call, ptr
from oracle import discrete_bayes as odb
from test_oracle_discrete_bayes import CASES, const_close

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
LONG = {F32: 28929, F64: 14465}           # one bin past the rows one CTA stages


def _torch():
    import torch
    return torch


def _cuda(a):
    return _torch().from_numpy(np.ascontiguousarray(a)).cuda()


# ------------------------------------------------------------------------------------------- goldens
@pytest.mark.parametrize("name", CASES)
def test_bank_forms_match_the_reference(golden, name):
    from filterpy_b200.discrete_bayes import normalize_bank, predict_bank, update_bank, predict_update_bank
    g = golden(name)
    mode = "wrap" if int(g["wrap"]) else "constant"
    cval = float(g["cval"])
    prior = predict_bank(g["pdf"], g["offsets"], g["kernel"], mode=mode, cval=cval)
    assert isinstance(prior, np.ndarray) and prior.dtype == g["pdf"].dtype
    if mode == "wrap":
        np.testing.assert_array_equal(prior, g["prior"])
    else:
        const_close(prior, g["prior"])
        np.testing.assert_array_equal(prior, odb.step_bank(g["pdf"], g["kernel"], g["offsets"], mode=mode, cval=cval)[0])
    np.testing.assert_array_equal(update_bank(g["lik"], g["prior"]), g["post"])
    p = g["pdf"].copy()
    assert normalize_bank(p) is p
    np.testing.assert_array_equal(p, g["norm"])
    fused = predict_update_bank(_cuda(g["pdf"]), _cuda(g["offsets"]), _cuda(g["kernel"]), _cuda(g["lik"]), mode, cval)
    want, _ = odb.step_bank(g["pdf"], g["kernel"], g["offsets"], g["lik"], mode, cval, normalize=True)
    np.testing.assert_array_equal(fused.cpu().numpy(), want)
    if mode == "wrap":
        np.testing.assert_array_equal(fused.cpu().numpy(), g["post"])


@pytest.mark.parametrize("name", CASES)
def test_drop_ins_return_what_the_reference_returns(golden, name):
    from filterpy_b200.discrete_bayes import normalize, predict, update
    g = golden(name)
    mode = "wrap" if int(g["wrap"]) else "constant"
    for b in range(g["pdf"].shape[0]):
        pr = predict(g["pdf"][b], int(g["offsets"][b]), g["kernel"][b], mode=mode, cval=float(g["cval"]))
        assert isinstance(pr, np.ndarray) and pr.shape == g["pdf"][b].shape
        if mode == "wrap":
            np.testing.assert_array_equal(pr, g["prior"][b])
        else:
            const_close(pr, g["prior"][b])
        np.testing.assert_array_equal(update(g["lik"][b], g["prior"][b]), g["post"][b])
        p = g["pdf"][b].copy()
        assert normalize(p) is p
        np.testing.assert_array_equal(p, g["norm"][b])
        t = _cuda(g["pdf"][b])
        assert normalize(t) is t
        np.testing.assert_array_equal(t.cpu().numpy(), g["norm"][b])
        tu = update(_cuda(g["lik"][b]), _cuda(g["prior"][b]))
        np.testing.assert_array_equal(tu.cpu().numpy(), g["post"][b])


def test_drop_in_update_promotes_like_numpy():
    from filterpy_b200.discrete_bayes import update
    rng = np.random.default_rng(7)
    prior, lik = rng.random(40).astype(F32), rng.random(40)
    got = update(lik, prior)
    want = odb.update_row(lik, prior)
    assert got.dtype == want.dtype == F64
    np.testing.assert_array_equal(got, want)


# ------------------------------------------------------------------------------------------- C-ABI, both paths
def db_call(dt, pdf, kernel, offsets, offset, lik, flags, cval=0.0, in_place=False, with_sums=True):
    """bke_db_step on guarded buffers -> (out, sums)."""
    torch = _torch()
    bf = Bufs(dt)
    B, M = pdf.shape
    p = bf.put(pdf, out=in_place)
    out = p if in_place else bf.out(pdf.shape)
    lk = bf.put(lik) if lik is not None else None
    kr = bf.put(kernel, dtype=F64) if kernel is not None else None
    sums = bf.out((B,), dtype=F64) if with_sums and (flags & 1) else None
    offs = torch.from_numpy(np.asarray(offsets, np.int64)).cuda() if offsets is not None else None
    a = _lib().DbArgs()
    a.n_rows, a.n_bins, a.dtype, a.flags = B, M, 0 if dt == F32 else 1, flags
    if kernel is not None:
        a.kernel, a.kernel_len, a.kernel_stride = ptr(kr), kernel.shape[-1], 0 if kernel.ndim == 1 else kernel.shape[-1]
        a.offsets, a.offset, a.cval = ptr(offs), offset, cval
    a.pdf, a.likelihood, a.out, a.sums = ptr(p), ptr(lk), ptr(out), ptr(sums)
    wsb = _lib().load().bke_db_workspace_bytes(M, a.dtype)
    if wsb:
        ws = torch.empty(wsb + 256, dtype=torch.uint8, device="cuda")
        a.workspace, a.workspace_bytes = ws.data_ptr() + (-ws.data_ptr()) % 256, wsb
    rc, err = call("bke_db_step", ctypes.byref(a))
    assert rc == 0, err
    bf.check_guards()
    return out.cpu().numpy().reshape(B, M), (sums.cpu().numpy() if sums is not None else None)


def _lib():
    from filterpy_b200 import _lib as lib
    return lib


def bank_inputs(dt, B, M, K, seed, per_row):
    rng = np.random.default_rng(seed)
    pdf = rng.random((B, M)).astype(dt)
    lik = (rng.random((B, M)) + 0.01).astype(dt)
    kernel = rng.random((B, K) if per_row else K)
    kernel[..., K // 2] = 0.0 if K > 2 else kernel[..., K // 2]            # a zero weight in every kernel
    offsets = rng.integers(-3 * M, 3 * M, B) if per_row else None
    return pdf, lik, kernel, offsets


# (dtype, M, K, B, per-row kernel and offsets, mode, in place)
SHAPES = [(F64, 1024, 3, 37, True, "wrap", False), (F32, 1024, 15, 37, False, "wrap", True),
          (F32, 1000, 4, 20, True, "constant", False), (F64, 777, 15, 9, False, "constant", True),
          (F64, 5, 12, 7, True, "wrap", True), (F32, 1, 3, 5, True, "constant", False),
          (F64, 14464, 3, 3, True, "wrap", False), (F32, 28928, 3, 2, False, "wrap", True),
          (F64, LONG[F64], 5, 2, True, "wrap", False), (F32, LONG[F32], 4, 2, False, "wrap", True),
          (F64, LONG[F64] + 1000, 15, 2, True, "constant", True), (F32, LONG[F32], 3, 2, True, "constant", False)]


@pytest.mark.parametrize("dt, M, K, B, per_row, mode, in_place", SHAPES,
                         ids=["%s-M%d-K%d-%s-%s%s" % (np.dtype(s[0]).name, s[1], s[2], "rows" if s[4] else "shared",
                                                       s[5], "-inplace" if s[6] else "") for s in SHAPES])
def test_fused_epoch_matches_the_oracle(dt, M, K, B, per_row, mode, in_place):
    pdf, lik, kernel, offsets = bank_inputs(dt, B, M, K, M * 31 + K, per_row)
    offset = 0 if per_row else -2 * M - 5
    flags = 1 | (2 if mode != "wrap" else 0)
    got, sums = db_call(dt, pdf, kernel, offsets, offset, lik, flags, cval=0.01, in_place=in_place)
    want, wsums = odb.step_bank(pdf, kernel, offsets if per_row else offset, lik, mode, 0.01, normalize=True)
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(sums, wsums)


@pytest.mark.parametrize("dt, M", [(F64, 512), (F32, 512), (F64, LONG[F64]), (F32, LONG[F32])])
@pytest.mark.parametrize("what", ["predict", "update", "normalize", "predict+update", "update+normalize"])
def test_each_subset_matches_the_oracle(dt, M, what):
    pdf, lik, kernel, offsets = bank_inputs(dt, 3, M, 5, 11, True)
    pdf[1] = 0                                                               # 0 / 0 = NaN, as NumPy gives
    k = kernel if "predict" in what else None
    lk = lik if "update" in what else None
    norm = what in ("normalize", "update+normalize")
    got, sums = db_call(dt, pdf, k, offsets, 0, lk, 1 if norm else 0)
    want, wsums = odb.step_bank(pdf, k, offsets, lk, "wrap", 0.0, normalize=norm)
    np.testing.assert_array_equal(got, want)
    if norm:
        np.testing.assert_array_equal(sums, wsums)
        assert np.isnan(got[1]).all()


def test_one_long_row_with_negative_and_infinite_terms():
    """The multi-pass sum falls back to the scan's sequential walk for terms the parity maps do not take (negative
    or infinite): the result is still the reference's."""
    rng = np.random.default_rng(5)
    M = 40000
    pdf = rng.random((1, M))
    pdf[0, 10] = -0.25
    got, sums = db_call(F64, pdf, None, None, 0, None, 1)
    want, wsums = odb.step_bank(pdf, normalize=True)
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(sums, wsums)


def test_a_captured_graph_replays_both_paths():
    """The call allocates nothing and synchronises nothing: both paths capture into a CUDA graph."""
    torch = _torch()
    from filterpy_b200.discrete_bayes.discrete_bayes import _step
    for M in (1024, LONG[F32]):
        pdf, lik, kernel, offsets = bank_inputs(F32, 3, M, 3, 2, True)
        tp, tl, tk, to = _cuda(pdf), _cuda(lik), _cuda(kernel), _cuda(offsets)
        out = torch.empty_like(tp)
        args = dict(kernel=tk, offset=to, likelihood=tl, normalize=True)
        _step(tp, out, **args)                                               # warm: function attributes
        torch.cuda.synchronize()
        from filterpy_b200 import _lib as lib
        a, wsb = lib.DbArgs(), lib.load().bke_db_workspace_bytes(M, lib.BKE_F32)
        ws = torch.empty(wsb + 256, dtype=torch.uint8, device="cuda")
        a.n_rows, a.n_bins, a.dtype, a.flags = 3, M, lib.BKE_F32, lib.BKE_DB_NORMALIZE
        a.kernel, a.kernel_len, a.kernel_stride, a.offsets = tk.data_ptr(), 3, 3, to.data_ptr()
        a.pdf, a.likelihood, a.out = tp.data_ptr(), tl.data_ptr(), out.data_ptr()
        if wsb:
            a.workspace, a.workspace_bytes = ws.data_ptr() + (-ws.data_ptr()) % 256, wsb
        out.zero_()
        s = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            lib.check(lib.load().bke_db_step(ctypes.byref(a), s.cuda_stream))
        g.replay()
        torch.cuda.synchronize()
        want, _ = odb.step_bank(pdf, kernel, offsets, lik, normalize=True)
        np.testing.assert_array_equal(out.cpu().numpy(), want)


# ------------------------------------------------------------------------------------------- Python surface
def test_python_argument_errors_raise_before_any_launch():
    torch = _torch()
    from filterpy_b200.discrete_bayes import predict, predict_bank, predict_update_bank, normalize, update_bank
    pdf = np.full((2, 8), 0.125)
    keep = pdf.copy()
    with pytest.raises(NotImplementedError):
        predict(pdf[0], 1.5, [0.1, 0.8, 0.1])
    with pytest.raises(NotImplementedError):
        predict(pdf[0], 1.5, [0.1, 0.8, 0.1], mode="constant")
    with pytest.raises(NotImplementedError):
        predict_bank(pdf, np.array([1.0, 0.5]), [0.1, 0.8, 0.1])
    with pytest.raises(ValueError):
        predict_bank(pdf, [1, 2, 3], [0.1, 0.8, 0.1])                        # one offset per row
    with pytest.raises(ValueError):
        predict_bank(pdf, 1, np.ones((3, 3)))                               # kernel rows != pdf rows
    with pytest.raises(ValueError):
        predict_bank(pdf, 1, [])
    with pytest.raises(ValueError):
        predict_update_bank(pdf, 1, [1.0], np.ones((2, 7)))
    with pytest.raises(ValueError):
        normalize(pdf)                                                       # 2-D: the reference means column sums
    with pytest.raises(TypeError):
        normalize(np.arange(4))
    with pytest.raises(ValueError):
        update_bank(np.ones(8), np.ones(8))
    np.testing.assert_array_equal(pdf, keep)
    assert predict(pdf[0], 2.0, [0.1, 0.8, 0.1]).shape == (8,)              # an integral float is the integer
    t = torch.ones(2, 8, dtype=torch.float32, device="cuda")
    with pytest.raises(ValueError):
        predict_update_bank(t, 0, [1.0], torch.ones(2, 8, dtype=torch.float32, device="cuda"),
                            out=torch.empty(2, 8, dtype=torch.float32, device="cuda")[:, :7])


def test_in_place_epoch_and_torch_op_equal_the_python_path():
    torch = _torch()
    from filterpy_b200.discrete_bayes import predict_update_bank
    from filterpy_b200 import torch_ops
    ops = torch_ops.load()
    for dt, M in ((F32, 1024), (F64, 1024), (F32, LONG[F32])):
        pdf, lik, kernel, offsets = bank_inputs(dt, 4, M, 15, 3, True)
        tp, tl, tk, to = _cuda(pdf), _cuda(lik), _cuda(kernel), _cuda(offsets)
        py = predict_update_bank(tp, to, tk, tl)
        op = ops.discrete_bayes_step(tp, tk, to, 0, tl, True)
        torch.testing.assert_close(op, py, rtol=0, atol=0, equal_nan=True)
        inplace = tp.clone()
        assert predict_update_bank(inplace, to, tk, tl, out=inplace) is inplace
        torch.testing.assert_close(inplace, py, rtol=0, atol=0, equal_nan=True)
        opc = ops.discrete_bayes_step(tp, tk[0].contiguous(), None, -7, None, False, True, 0.5)
        want, _ = odb.step_bank(pdf, kernel[0], -7, mode="constant", cval=0.5)
        np.testing.assert_array_equal(opc.cpu().numpy(), want)
