"""The packed symmetric Q / R record of the 4/2 fp32 step (bke_kf_pack_sym_models, bke_kf_step_sym):
bit-identical to the dense step in every mode, eagerly and in a captured graph; only built for
exactly symmetric banks; never used once Q or R may have changed under it."""
import numpy as np
import pytest

from gpu_harness import rel_close

pytestmark = pytest.mark.gpu

NS = [(1 << 18) + 1, 1 << 20]     # a ragged last tile (odd: half a 16-byte granule of z) and the bench size
MODES = {"fused": 3, "predict": 1, "update": 2}


def _sym_bank(N, seed):
    """kf_bank_cv2d with a symmetric random perturbation of Q and R, so every word of the upper
    triangles carries distinct bits; float32, exactly symmetric."""
    from filterpy_b200.common import workloads as wl
    w = wl.kf_bank_cv2d(N, seed=seed, steps=2, dtype=np.float32)
    rng = np.random.default_rng(seed)
    for k, n in (("Q", 4), ("R", 2)):
        a = w[k] + np.float32(1e-3) * rng.standard_normal((N, n, n)).astype(np.float32)
        up = np.triu(a)
        w[k] = np.ascontiguousarray(up + np.swapaxes(np.triu(a, 1), 1, 2))
    return w


def _dev(w):
    import torch
    return {k: torch.from_numpy(v).cuda() for k, v in w.items()}


def _pack(d, N):
    """-> (record, asymmetric flag as int)"""
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    rec = torch.empty(lib.bke_kf_sym_models_bytes(N) // 4, dtype=torch.float32, device="cuda")
    flag = torch.full((1,), 7, dtype=torch.int32, device="cuda")
    _lib.check(lib.bke_kf_pack_sym_models(N, 4, 2, _lib.BKE_F32, d["Q"].data_ptr(), d["R"].data_ptr(), rec.data_ptr(),
                                          flag.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return rec, int(flag.item())


def _outputs(d, N, extras):
    import torch
    kw = dict(dtype=torch.float32, device="cuda")
    o = {"x": d["x"].clone(), "P": d["P"].clone()}
    if extras:
        o.update(x_prior=torch.zeros(N, 4, **kw), P_prior=torch.zeros(N, 4, 4, **kw), K=torch.zeros(N, 4, 2, **kw),
                 y=torch.zeros(N, 2, **kw), S=torch.zeros(N, 2, 2, **kw), SI=torch.zeros(N, 2, 2, **kw),
                 ll=torch.zeros(N, **kw), status=torch.full((N,), 9, dtype=torch.int32, device="cuda"))
    return o


def _args(d, o, N, flags, extras, z):
    from filterpy_b200 import _lib
    a = _lib.KfArgs()
    a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags, a.alpha_sq = N, 4, 2, _lib.BKE_F32, flags, 1.0
    a.x = a.x_out = o["x"].data_ptr()
    a.P = a.P_out = o["P"].data_ptr()
    a.F, a.F_stride, a.Q, a.Q_stride = d["F"].data_ptr(), 16, d["Q"].data_ptr(), 16
    a.H, a.H_stride, a.R, a.R_stride = d["H"].data_ptr(), 8, d["R"].data_ptr(), 4
    a.z = z.data_ptr()
    if extras:
        a.x_prior, a.P_prior = o["x_prior"].data_ptr(), o["P_prior"].data_ptr()
        a.K, a.y, a.S, a.SI = o["K"].data_ptr(), o["y"].data_ptr(), o["S"].data_ptr(), o["SI"].data_ptr()
        a.log_likelihood, a.status = o["ll"].data_ptr(), o["status"].data_ptr()
    return a


@pytest.mark.parametrize("graphed", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("extras", [False, True], ids=["plain", "extras"])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("N", NS)
def test_packed_step_is_bitwise_the_dense_step(N, mode, extras, graphed):
    """Two chained steps through the C-ABI, dense (bke_kf_step) and packed (bke_kf_step_sym), on
    separate copies of the state: every output equal bit for bit."""
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    w = _sym_bank(N, 77)
    d = _dev(w)
    zs = [torch.from_numpy(w["zs"][t]).cuda() for t in range(2)]
    rec, asym = _pack(d, N)
    assert asym == 0
    flags = MODES[mode]
    outs = {}
    for kind in ("dense", "sym"):
        o = _outputs(d, N, extras)
        args = [_args(d, o, N, flags, extras, z) for z in zs]

        def run():
            s = torch.cuda.current_stream().cuda_stream
            for a in args:
                _lib.check(lib.bke_kf_step(a, s) if kind == "dense" else lib.bke_kf_step_sym(a, rec.data_ptr(), s))
        if graphed:
            x0, P0 = o["x"].clone(), o["P"].clone()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                run()                                     # warm-up: module load, function attributes
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
        outs[kind] = {k: v.cpu().numpy().view(np.uint32) for k, v in o.items()}       # compare bits
    for k in outs["dense"]:
        np.testing.assert_array_equal(outs["sym"][k], outs["dense"][k], err_msg=k)


def test_record_layout():
    """Plane k of tile t holds word k of the upper triangles of that tile's filters; the padding of the
    last tile is zero."""
    N = 300
    w = _sym_bank(N, 5)
    rec, asym = _pack(_dev(w), N)
    assert asym == 0
    r = rec.cpu().numpy().reshape(3, 13, 128)
    iu = np.triu_indices(4)
    want = np.concatenate([w["Q"][:, iu[0], iu[1]], w["R"][:, [0, 0, 1], [0, 1, 1]]], axis=1)     # (N, 13)
    got = r.transpose(0, 2, 1).reshape(-1, 13)
    np.testing.assert_array_equal(got[:N], want)
    assert not got[N:].any()


def _mirror(w):
    from filterpy_b200.kalman import KalmanFilter
    N = w["x"].shape[0]
    kf = KalmanFilter(4, 2, n_filters=N, dtype=np.float32, device="cuda", diagnostics=False)
    for k in "xPFHQR":
        setattr(kf, k, w[k])
    return kf


def _oracle_step(w, z, Q=None):
    from oracle import kf as okf
    return okf.kf_step_bank(w["x"], w["P"], z, w["F"], w["H"], w["Q"] if Q is None else Q, w["R"])


def _uses_record(kf):
    return kf._sym_state is not None and kf._sym_state[1] and kf._sym_buf is not None


@pytest.mark.parametrize("flip", ["value", "signed_zero"])
def test_asymmetric_bank_falls_back_to_the_dense_models(flip):
    """One filter whose Q differs from its transpose (by value, or only as -0.0 against +0.0): the pack
    reports it, no record is used, and the steps match the oracle."""
    import torch
    N = (1 << 12) + 3
    w = _sym_bank(N, 21)
    f = 1000
    if flip == "value":
        w["Q"][f, 0, 1] += np.float32(1e-3)
    else:
        w["Q"][f, 0, 3] = np.float32(0.0); w["Q"][f, 3, 0] = np.float32(-0.0)
    assert _pack(_dev(w), N)[1] == 1
    kf = _mirror(w)
    zs = [torch.from_numpy(w["zs"][t]).cuda() for t in range(2)]
    st = dict(w)
    for t in range(2):
        kf.predict(); kf.update(zs[t])
        o = _oracle_step(st, w["zs"][t])
        st["x"], st["P"] = o["x"], o["P"]
    assert kf._sym_state is not None and not kf._sym_state[1]
    rel_close(kf.x.cpu().numpy(), st["x"], 1e-3, "x"); rel_close(kf.P.cpu().numpy(), st["P"], 1e-3, "P")


def test_graph_captured_by_the_mirror_uses_the_record():
    """The flow of bench.py: the record is packed during the capture's warm-up and the graph reads it."""
    import torch
    N = (1 << 18) + 1
    w = _sym_bank(N, 31)
    kf = _mirror(w)
    z = torch.from_numpy(w["zs"][0]).cuda()
    g = kf.capture(lambda: (kf.predict(), kf.update(z)))
    assert _uses_record(kf)
    kf.x.copy_(torch.from_numpy(w["x"])); kf.P.copy_(torch.from_numpy(w["P"]))
    g.replay()
    torch.cuda.synchronize()
    o = _oracle_step(w, w["zs"][0])
    rel_close(kf.x.cpu().numpy(), o["x"], 1e-3, "x"); rel_close(kf.P.cpu().numpy(), o["P"], 1e-3, "P")


def test_in_place_edit_through_the_getter_takes_effect():
    """kf.Q hands out the live tensor: an edit of it must reach the next step, even though a record
    of the old Q exists."""
    import torch
    N = (1 << 12) + 1
    w = _sym_bank(N, 41)
    kf = _mirror(w)
    z = torch.from_numpy(w["zs"][0]).cuda()
    for _ in range(3):
        kf.predict(); kf.update(z)
    assert _uses_record(kf)
    kf.x = w["x"]; kf.P = w["P"]
    kf.Q.mul_(4.0)
    kf.predict(); kf.update(z)
    o = _oracle_step(w, w["zs"][0], Q=w["Q"] * np.float32(4.0))
    rel_close(kf.x.cpu().numpy(), o["x"], 1e-3, "x"); rel_close(kf.P.cpu().numpy(), o["P"], 1e-3, "P")


def test_aliased_tensor_edited_in_place_takes_effect():
    """kf.Q = t with t already a contiguous float32 CUDA tensor aliases t: an in-place edit of t after a
    record was built (its version counter moves) must reach the next step."""
    import torch
    N = (1 << 12) + 1
    w = _sym_bank(N, 51)
    kf = _mirror(w)
    tq = torch.from_numpy(w["Q"]).cuda()
    tr = torch.from_numpy(w["R"]).cuda()
    kf.Q = tq; kf.R = tr
    z = torch.from_numpy(w["zs"][0]).cuda()
    for _ in range(3):
        kf.predict(); kf.update(z)
    assert _uses_record(kf)
    kf.x = w["x"]; kf.P = w["P"]
    tq.mul_(4.0); tr.add_(0.5)
    kf.predict(); kf.update(z)
    w2 = dict(w, R=w["R"] + np.float32(0.5))
    o = _oracle_step(w2, w["zs"][0], Q=w["Q"] * np.float32(4.0))
    rel_close(kf.x.cpu().numpy(), o["x"], 1e-3, "x"); rel_close(kf.P.cpu().numpy(), o["P"], 1e-3, "P")
    for _ in range(2):
        kf.predict(); kf.update(z)
    assert _uses_record(kf)                              # re-packed once Q and R stood still again


def test_assigning_q_every_step_never_packs():
    import torch
    N = (1 << 12) + 1
    w = _sym_bank(N, 61)
    kf = _mirror(w)
    z = torch.from_numpy(w["zs"][0]).cuda()
    for _ in range(6):
        kf.Q = w["Q"]
        kf.predict(); kf.update(z)
    assert kf._sym_buf is None and kf._sym_state is None


@pytest.mark.parametrize("q2", ["asymmetric", "symmetric"])
def test_graph_keeps_the_q_and_r_of_its_capture(q2):
    """Q and R are frozen into a graph captured with the record.  After an in-place edit of Q (to an
    asymmetric or to another symmetric matrix) and two eager steps (the second one packs the new Q,
    into a new record), the eager steps use the new Q and the replay still uses the Q of the capture."""
    import torch
    N = (1 << 14) + 1
    w = _sym_bank(N, 71)
    kf = _mirror(w)
    z = torch.from_numpy(w["zs"][0]).cuda()
    g = kf.capture(lambda: (kf.predict(), kf.update(z)))
    assert _uses_record(kf) and kf._sym_pinned
    captured = kf._sym_buf
    Q2 = w["Q"] * np.float32(3.0)
    if q2 == "asymmetric":
        Q2[7, 1, 2] += np.float32(1e-3)
    kf.Q.copy_(torch.from_numpy(Q2))

    def reset():
        kf.x.copy_(torch.from_numpy(w["x"])); kf.P.copy_(torch.from_numpy(w["P"]))
    reset()
    for _ in range(2):
        kf.predict(); kf.update(z)
    st = dict(w)
    for _ in range(2):
        o = _oracle_step(st, w["zs"][0], Q=Q2)
        st["x"], st["P"] = o["x"], o["P"]
    rel_close(kf.x.cpu().numpy(), st["x"], 1e-3, "eager x"); rel_close(kf.P.cpu().numpy(), st["P"], 1e-3, "eager P")
    assert kf._sym_state[1] == (q2 == "symmetric")
    assert kf._sym_buf is not captured and any(b is captured for b in kf._sym_held)
    reset()
    g.replay()
    torch.cuda.synchronize()
    o = _oracle_step(w, w["zs"][0])
    rel_close(kf.x.cpu().numpy(), o["x"], 1e-3, "replay x"); rel_close(kf.P.cpu().numpy(), o["P"], 1e-3, "replay P")


def test_missing_or_shared_models_never_pack():
    """A predict-only loop on a bank without R, and a bank whose F is shared while Q and R are per
    filter (the packed kernel takes no mixture), run on the dense models and never pack."""
    import torch
    N = (1 << 12) + 1
    w = _sym_bank(N, 81)
    kf = _mirror(w)
    kf.R = None
    for _ in range(3):
        kf.predict()
        x = kf.x
    assert kf._sym_buf is None
    want = w["x"].astype(np.float64)
    for _ in range(3):
        want = np.einsum("nij,nj->ni", w["F"].astype(np.float64), want)
    rel_close(x.cpu().numpy(), want, 1e-5, "x")
    kf2 = _mirror(w)
    kf2.F = w["F"][0]
    z = torch.from_numpy(w["zs"][0]).cuda()
    for _ in range(3):
        kf2.predict(); kf2.update(z)
    assert kf2._sym_ok and kf2._sym_buf is None and kf2._sym_state is None
    o = _oracle_step(dict(w, F=np.broadcast_to(w["F"][0], w["F"].shape)), w["zs"][0])
    st = o
    for _ in range(2):
        st = _oracle_step(dict(w, x=st["x"], P=st["P"], F=np.broadcast_to(w["F"][0], w["F"].shape)), w["zs"][0])
    rel_close(kf2.x.cpu().numpy(), st["x"], 1e-3, "x"); rel_close(kf2.P.cpu().numpy(), st["P"], 1e-3, "P")


def test_successful_packed_step_leaves_no_error_text():
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    N = 1000
    w = _sym_bank(N, 91)
    d = _dev(w)
    rec, asym = _pack(d, N)
    assert asym == 0
    o = _outputs(d, N, False)
    z = torch.from_numpy(w["zs"][0]).cuda()
    _lib.check(lib.bke_kf_step_sym(_args(d, o, N, 3, False, z), rec.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert lib.bke_last_error() == b""
