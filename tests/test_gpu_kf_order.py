"""The reversed tile order of the 4/2 fp32 step (BKE_REVERSE_TILES): a scheduling hint that no result
depends on.  Every kernel instance gives the same bits in either order; a reversed step reads what the
previous step wrote; the mirror alternates the order on every launch, eagerly and in captured graphs;
every other kernel ignores the bit."""
import os

import numpy as np
import pytest

from test_gpu_kf_sym import MODES, _args, _dev, _outputs, _pack, _sym_bank

REV = 16                         # BKE_REVERSE_TILES (test_reverse_tiles_flag_matches_the_header checks it)

# N = 1 (a single, odd filter), 127 and 129 (one ragged tile, two tiles), 2^13 + 1 (odd, a ragged tile of
# one filter), 40 000 (313 tiles: fewer than the grid), 2^20 + 3 (8193 tiles: about 20 per CTA).
# A bank stepped in place whose state fits L2 (N * 80 B <= 38 MiB) keeps the forward order, so the
# instance test steps out of place, where every size takes the order it is given.
NS = [1, 127, 129, (1 << 13) + 1, 40000, (1 << 20) + 3]
MODELS = ["dense", "sym", "packed", "shared_dev", "shared_host"]

_cache = {}


def _bank(N):
    if N not in _cache:
        _cache.clear()
        w = _sym_bank(N, 91)
        _cache[N] = (w, _dev(w))
    return _cache[N]


def _scan_and_pack(d, N):
    from test_gpu_kf_packed import _scan_and_pack as scan
    return scan(d, N)


@pytest.mark.gpu
@pytest.mark.parametrize("extras", [False, True], ids=["plain", "extras"])
@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("N", NS)
def test_every_instance_is_bitwise_the_same_in_reverse(N, mode, model, extras):
    """One launch of each kf42_f32_kernel instance the dispatcher reaches, with and without
    BKE_REVERSE_TILES, out of place into separate outputs: x, P and every optional output equal bit for bit."""
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    w, d = _bank(N)
    z = d["zs"][0]
    rec = hmap = None
    if model == "sym":
        rec, asym = _pack(d, N)
        assert asym == 0
    elif model == "packed":
        rec, hmap = _scan_and_pack(d, N)
        assert hmap.asymmetric == 0
    host = {k: np.ascontiguousarray(w[k][0]) for k in "FQHR"}
    shared = {k: d[k][0].contiguous() for k in "FQHR"}
    outs = []
    for flags in (MODES[mode], MODES[mode] | REV):
        o = _outputs(d, N, extras)
        a = _args(d, o, N, flags, extras, z)
        a.x, a.P = d["x"].data_ptr(), d["P"].data_ptr()     # out of place: o["x"], o["P"] receive the posterior
        if model.startswith("shared"):
            a.F, a.Q, a.H, a.R = (shared[k].data_ptr() for k in "FQHR")
            a.F_stride = a.Q_stride = a.H_stride = a.R_stride = 0
            if model == "shared_host":
                a.F_host, a.Q_host, a.H_host, a.R_host = (host[k].ctypes.data for k in "FQHR")
        s = torch.cuda.current_stream().cuda_stream
        if model == "sym":
            _lib.check(lib.bke_kf_step_sym(a, rec.data_ptr(), s))
        elif model == "packed":
            _lib.check(lib.bke_kf_step_packed(a, rec.data_ptr(), hmap, s))
        else:
            _lib.check(lib.bke_kf_step(a, s))
        torch.cuda.synchronize()
        outs.append({k: v.cpu().numpy().view(np.uint32) for k, v in o.items()})
    for k in outs[0]:
        np.testing.assert_array_equal(outs[1][k], outs[0][k], err_msg=k)


def _chain(d, N, flags_seq, graphed, valid=None):
    """Steps of the dense 4/2 fp32 bank through bke_kf_step, one per entry of flags_seq, the
    measurements taken in turn from the two of the bank; -> (x, P) as bits."""
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    o = _outputs(d, N, False)
    args = []
    for i, fl in enumerate(flags_seq):
        a = _args(d, o, N, fl, False, d["zs"][i % 2])
        if valid is not None:
            a.z_valid = valid.data_ptr()
        args.append(a)

    def run():
        s = torch.cuda.current_stream().cuda_stream
        for a in args:
            _lib.check(lib.bke_kf_step(a, s))
    if graphed:
        x0, P0 = o["x"].clone(), o["P"].clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            run()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            run()
        o["x"].copy_(x0); o["P"].copy_(P0)
        g.replay()
    else:
        run()
    torch.cuda.synchronize()
    return o["x"].cpu().numpy().view(np.uint32), o["P"].cpu().numpy().view(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("graphed", [False, True], ids=["eager", "graph"])
def test_each_reversed_step_reads_what_the_previous_step_wrote(graphed):
    """Eight fused steps of a 2^20-filter bank, alternating the order (each launch starts on the tiles
    the previous one wrote last, while that launch may still be draining), equal eight forward steps."""
    N = 1 << 20
    _, d = _bank(N)
    fwd = _chain(d, N, [3] * 8, graphed)
    alt = _chain(d, N, [3 | (REV if i % 2 else 0) for i in range(8)], graphed)
    np.testing.assert_array_equal(alt[0], fwd[0])
    np.testing.assert_array_equal(alt[1], fwd[1])


@pytest.mark.gpu
def test_reversed_update_without_measurements_leaves_the_state_untouched():
    """An update-only launch in which no filter has a measurement, in reverse order, eight times: the
    whole state stays bit-identical (the stage ring must not be refilled under a tile still being read)."""
    import torch
    N = 1 << 20
    w, d = _bank(N)
    valid = torch.zeros(N, dtype=torch.uint8, device="cuda")
    x, P = _chain(d, N, [2 | REV] * 8, False, valid)
    np.testing.assert_array_equal(x, w["x"].view(np.uint32))
    np.testing.assert_array_equal(P, w["P"].view(np.uint32))


def _mirror(w, N):
    from filterpy_b200.kalman import KalmanFilter
    kf = KalmanFilter(4, 2, n_filters=N, dtype=np.float32, device="cuda", diagnostics=False)
    for k in "xPFHQR":
        setattr(kf, k, w[k])
    return kf


def _record_flags(kf):
    """Log the flags of every launch the mirror makes."""
    log, step = [], kf._step

    def logged(a, rec):
        log.append(a.flags)
        return step(a, rec)
    kf._step = logged
    return log


@pytest.mark.gpu
def test_mirror_alternates_and_matches_forward_stepping():
    """Fused steps, a split predict / update, z=None and a valid mask through the mirror, which
    alternates the order on every launch, equal the same launches through the C-ABI in forward order."""
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    N = (1 << 19) + 1                                   # 40 MiB of state: above the bound, so the order applies
    w, d = _bank(N)
    valid = np.arange(N) % 3 != 0
    kf = _mirror(w, N)
    log = _record_flags(kf)
    zs = [d["zs"][i % 2] for i in range(4)]
    kf.predict(); kf.update(zs[0])                      # fused
    kf.predict(); kf.update(zs[1])                      # fused (the mirror now steps from the packed words)
    kf.predict(); kf.x                                  # predict alone
    kf.update(zs[2])                                    # update alone
    kf.predict(); kf.update(None)                       # z=None: predict alone
    kf.predict(); kf.update(zs[3], valid=valid)         # fused, with a mask
    x, P = kf.x.clone(), kf.P.clone()
    torch.cuda.synchronize()
    assert [f & REV for f in log] == [0, REV, 0, REV, 0, REV]
    assert [f & ~REV for f in log] == [3, 3, 1, 2, 1, 3]

    o = _outputs(d, N, False)
    vt = torch.from_numpy(valid.astype(np.uint8)).cuda()
    s = torch.cuda.current_stream().cuda_stream
    for flags, z, v in ((3, zs[0], None), (3, zs[1], None), (1, zs[0], None), (2, zs[2], None), (1, zs[0], None),
                        (3, zs[3], vt)):
        a = _args(d, o, N, flags, False, z)
        if v is not None:
            a.z_valid = v.data_ptr()
        _lib.check(lib.bke_kf_step(a, s))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(x.cpu().numpy().view(np.uint32), o["x"].cpu().numpy().view(np.uint32))
    np.testing.assert_array_equal(P.cpu().numpy().view(np.uint32), o["P"].cpu().numpy().view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("ring", [3, 4])
def test_graph_replays_equal_eager_stepping(ring):
    """A ring of fused steps captured from the mirror: each captured launch keeps the order it was
    captured with (alternating inside the ring; across replays too when the ring is even), and three
    replays equal 3 * ring eager steps bit for bit."""
    import torch
    N = (1 << 20) + 3
    w, d = _bank(N)
    zs = [d["zs"][i % 2] for i in range(ring)]
    kf = _mirror(w, N)
    log = _record_flags(kf)

    def steps():
        for z in zs:
            kf.predict(); kf.update(z)
    graph = kf.capture(steps)
    captured = [f & REV for f in log[-ring:]]
    assert all(captured[i] != captured[i + 1] for i in range(ring - 1))
    assert (captured[0] != captured[-1]) == (ring % 2 == 0)
    kf.x.copy_(d["x"]); kf.P.copy_(d["P"])             # in place: the graph reads these buffers
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()

    ref = _mirror(w, N)
    for _ in range(3):
        for z in zs:
            ref.predict(); ref.update(z)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(kf.x.cpu().numpy().view(np.uint32), ref.x.cpu().numpy().view(np.uint32))
    np.testing.assert_array_equal(kf.P.cpu().numpy().view(np.uint32), ref.P.cpu().numpy().view(np.uint32))


def _generic_bank(n, m, N, dtype, shared_fq=False, seed=3):
    """A random stable bank of N filters of dim_x n, dim_z m; F and Q shared when shared_fq."""
    rng = np.random.default_rng(seed)
    F = (np.eye(n) + 0.01 * rng.standard_normal((N, n, n))).astype(dtype)
    A = rng.standard_normal((N, n, n))
    P = (A @ np.swapaxes(A, 1, 2) / n + np.eye(n)).astype(dtype)
    Q = (0.01 * np.eye(n) * np.ones((N, 1, 1))).astype(dtype)
    H = rng.standard_normal((N, m, n)).astype(dtype)
    R = (np.eye(m) * np.ones((N, 1, 1))).astype(dtype)
    if shared_fq:
        F, Q = np.ascontiguousarray(F[0]), np.ascontiguousarray(Q[0])
        H, R = np.ascontiguousarray(H[0]), np.ascontiguousarray(R[0])
    return dict(x=rng.standard_normal((N, n)).astype(dtype), P=P, F=F, Q=Q, H=H, R=R,
                z=rng.standard_normal((N, m)).astype(dtype))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(4, 2, np.float64, False), (9, 3, np.float64, False), (7, 2, np.float32, False),
                                   (16, 2, np.float32, True)],
                         ids=["kf42_f64_direct", "kf93_f64_rowblock", "kf72_f32_generic", "kf16_2_f32_wgmma"])
def test_other_kernels_ignore_the_bit(shape):
    """Banks that other kernels step give the same bits with BKE_REVERSE_TILES set and without."""
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    n, m, dtype, shared = shape
    N = 5000
    w = _generic_bank(n, m, N, dtype, shared)
    d = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in w.items()}
    outs = []
    for flags in (3, 3 | REV):
        x, P = d["x"].clone(), d["P"].clone()
        K = torch.zeros(N, n, m, dtype=x.dtype, device="cuda")
        st = torch.full((N,), 9, dtype=torch.int32, device="cuda")
        a = _lib.KfArgs()
        a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags, a.alpha_sq = N, n, m, \
            (_lib.BKE_F32 if dtype == np.float32 else _lib.BKE_F64), flags, 1.0
        a.x = a.x_out = x.data_ptr(); a.P = a.P_out = P.data_ptr()
        a.F, a.F_stride = d["F"].data_ptr(), 0 if shared else n * n
        a.Q, a.Q_stride = d["Q"].data_ptr(), 0 if shared else n * n
        a.H, a.H_stride = d["H"].data_ptr(), 0 if shared else m * n
        a.R, a.R_stride = d["R"].data_ptr(), 0 if shared else m * m
        a.z = d["z"].data_ptr()
        a.K, a.status = K.data_ptr(), st.data_ptr()
        _lib.check(lib.bke_kf_step(a, torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        outs.append([t.cpu().numpy() for t in (x, P, K, st)])
    for got, want in zip(outs[1], outs[0]):
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8))
    assert np.isfinite(outs[0][1]).all()


def test_reverse_tiles_flag_matches_the_header():
    from filterpy_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "bke.h")).read()
    line = [ln for ln in hdr.splitlines() if ln.startswith("#define BKE_REVERSE_TILES")][0]
    assert int(line.split()[2].rstrip("u")) == _lib.BKE_REVERSE_TILES == REV
