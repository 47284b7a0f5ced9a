"""The packed model words of the 4/2 fp32 step (bke_kf_scan_models, bke_kf_pack_models,
bke_kf_step_packed): the scan and the record match NumPy, the step is bit-identical to the dense step
in every mode, eagerly and in a captured graph, and the mirror never steps from a stale record."""
import ctypes

import numpy as np
import pytest

from gpu_harness import rel_close
from test_gpu_kf_sym import MODES, NS, _args, _mirror, _oracle_step, _outputs, _uses_record

pytestmark = pytest.mark.gpu

IU = np.triu_indices(4)


def _words(w):
    """(N, 37) float32: F row-major | Q upper triangle | H row-major | R00 R01 R11."""
    N = w["F"].shape[0]
    return np.concatenate([w["F"].reshape(N, 16), w["Q"][:, IU[0], IU[1]], w["H"].reshape(N, 8),
                           w["R"][:, [0, 0, 1], [0, 1, 1]]], axis=1)


def _varying(w):
    bits = _words(w).view(np.uint32)
    return sum(1 << e for e in range(37) if (bits[:, e] != bits[0, e]).any())


def _bench_bank(N, seed):
    from filterpy_b200.common import workloads as wl
    return wl.kf_bank_cv2d(N, seed=seed, steps=2, dtype=np.float32)


def _all_words_bank(N, seed):
    """kf_bank_cv2d with a random perturbation of every model word; Q and R stay exactly symmetric."""
    w = _bench_bank(N, seed)
    rng = np.random.default_rng(seed)
    for k, shape in (("F", (4, 4)), ("H", (2, 4))):
        w[k] = np.ascontiguousarray(w[k] + np.float32(1e-3) * rng.standard_normal((N,) + shape).astype(np.float32))
    for k, n in (("Q", 4), ("R", 2)):
        a = w[k] + np.float32(1e-3) * rng.standard_normal((N, n, n)).astype(np.float32)
        w[k] = np.ascontiguousarray(np.triu(a) + np.swapaxes(np.triu(a, 1), 1, 2))
    return w


def _last_filter_bank(N, seed):
    """kf_bank_cv2d whose last filter (in the ragged last tile) alone differs in one word of each of F,
    Q, H and R that every other filter has equal (F02, Q02 = Q20, H01, R01 = R10)."""
    w = _bench_bank(N, seed)
    f = N - 1
    w["F"][f, 0, 2] = np.float32(1e-3)
    w["Q"][f, 0, 2] = w["Q"][f, 2, 0] = np.float32(1e-5)
    w["H"][f, 0, 1] = np.float32(0.25)
    w["R"][f, 0, 1] = w["R"][f, 1, 0] = np.float32(1e-3)
    return w


def _signed_zero_bank(N, seed):
    """kf_bank_cv2d where one filter has -0.0 in F02 and every other filter +0.0."""
    w = _bench_bank(N, seed)
    w["F"][N // 3, 0, 2] = np.float32(-0.0)
    return w


BANKS = {"bench": _bench_bank, "all_words": _all_words_bank, "last_filter": _last_filter_bank,
         "signed_zero": _signed_zero_bank}
K = {"bench": 10, "all_words": 37, "last_filter": 14, "signed_zero": 11}

_cache = {}


def _bank(kind, N):
    if (kind, N) not in _cache:
        _cache.clear()                                   # one bank of 2^20 filters at a time
        _cache[(kind, N)] = BANKS[kind](N, 7)
    return _cache[(kind, N)]


def _dev(w):
    import torch
    return {k: torch.from_numpy(v).cuda() for k, v in w.items()}


def _scan_and_pack(d, N):
    """-> (record, host map)"""
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    s = torch.cuda.current_stream().cuda_stream
    dmap = torch.full((ctypes.sizeof(_lib.KfModelMap),), 0x5a, dtype=torch.uint8, device="cuda")
    _lib.check(lib.bke_kf_scan_models(N, 4, 2, _lib.BKE_F32, d["F"].data_ptr(), d["Q"].data_ptr(), d["H"].data_ptr(),
                                      d["R"].data_ptr(), dmap.data_ptr(), s))
    hmap = _lib.KfModelMap.from_buffer_copy(dmap.cpu().numpy().tobytes())
    nb = lib.bke_kf_packed_models_bytes(N, hmap.varying)
    rec = torch.full((max(nb, 4) // 4,), float("nan"), dtype=torch.float32, device="cuda")
    _lib.check(lib.bke_kf_pack_models(N, 4, 2, _lib.BKE_F32, d["F"].data_ptr(), d["Q"].data_ptr(), d["H"].data_ptr(),
                                      d["R"].data_ptr(), hmap.varying, rec.data_ptr(), s))
    return rec, hmap


@pytest.mark.parametrize("kind", list(BANKS))
def test_scan_and_record_match_numpy(kind):
    """The map holds the varying mask, filter 0's words and the symmetry flag; plane s of tile t holds
    the s-th varying word of that tile's filters, and the padding of the last tile is zero."""
    N = 1000
    w = BANKS[kind](N, 3)
    rec, hmap = _scan_and_pack(_dev(w), N)
    assert hmap.asymmetric == 0
    assert hmap.varying == _varying(w) and bin(hmap.varying).count("1") == K[kind]
    words = _words(w)
    np.testing.assert_array_equal(np.array(hmap.words, dtype=np.float32).view(np.uint32), words[0].view(np.uint32))
    sel = [e for e in range(37) if hmap.varying >> e & 1]
    tiles = (N + 127) // 128
    got = rec.cpu().numpy().reshape(tiles, len(sel), 128).transpose(0, 2, 1).reshape(-1, len(sel))
    np.testing.assert_array_equal(got[:N].view(np.uint32), words[:, sel].view(np.uint32))
    assert not got[N:].any()


def test_scan_reports_an_asymmetric_bank_and_the_step_refuses_it():
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    N = 3000
    w = _bench_bank(N, 11)
    w["Q"][2500, 1, 3] = np.float32(1e-4)                # Q13 set, Q31 left at 0
    d = _dev(w)
    rec, hmap = _scan_and_pack(d, N)
    assert hmap.asymmetric == 1
    o = _outputs(d, N, False)
    z = torch.from_numpy(w["zs"][0]).cuda()
    rc = lib.bke_kf_step_packed(_args(d, o, N, 3, False, z), rec.data_ptr(), hmap, torch.cuda.current_stream().cuda_stream)
    assert rc == _lib.BKE_ERR_UNSUPPORTED


@pytest.mark.parametrize("graphed", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("extras", [False, True], ids=["plain", "extras"])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("kind", list(BANKS))
def test_packed_step_is_bitwise_the_dense_step(kind, N, mode, extras, graphed):
    """Two chained steps through the C-ABI, dense (bke_kf_step) and packed (bke_kf_step_packed), on
    separate copies of the state: every output equal bit for bit."""
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    w = _bank(kind, N)
    d = _dev(w)
    zs = [torch.from_numpy(w["zs"][t]).cuda() for t in range(2)]
    rec, hmap = _scan_and_pack(d, N)
    assert hmap.asymmetric == 0 and bin(hmap.varying).count("1") == K[kind]
    flags = MODES[mode]
    outs = {}
    for arm in ("dense", "packed"):
        o = _outputs(d, N, extras)
        args = [_args(d, o, N, flags, extras, z) for z in zs]

        def run():
            s = torch.cuda.current_stream().cuda_stream
            for a in args:
                _lib.check(lib.bke_kf_step(a, s) if arm == "dense" else lib.bke_kf_step_packed(a, rec.data_ptr(), hmap, s))
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
        outs[arm] = {k: v.cpu().numpy().view(np.uint32) for k, v in o.items()}
    for k in outs["dense"]:
        np.testing.assert_array_equal(outs["packed"][k], outs["dense"][k], err_msg=k)


def test_mirror_steps_from_the_packed_words():
    """The mirror's record of the bench bank holds the 10 varying words, 40 B per filter."""
    import torch
    N = (1 << 14) + 1
    w = _bench_bank(N, 13)
    kf = _mirror(w)
    z = torch.from_numpy(w["zs"][0]).cuda()
    for _ in range(3):
        kf.predict(); kf.update(z)
    assert _uses_record(kf)
    assert kf._sym_buf.numel() == (N + 127) // 128 * 128 * 10
    assert kf._sym_host_map.varying == _varying(w)


@pytest.mark.parametrize("name", ["F", "H"])
def test_graph_keeps_the_f_and_h_of_its_capture(name):
    """F and H are frozen into a graph captured with the record, like Q and R: after an in-place edit
    of F (or H) and two eager steps (the second packs the new model into a new record), the eager
    steps use the new model and the replay still uses the one of the capture."""
    import torch
    N = (1 << 14) + 1
    w = _bench_bank(N, 17)
    kf = _mirror(w)
    z = torch.from_numpy(w["zs"][0]).cuda()
    g = kf.capture(lambda: (kf.predict(), kf.update(z)))
    assert _uses_record(kf) and kf._sym_pinned
    captured = kf._sym_buf
    new = w[name].copy()
    if name == "F":
        new[:, 0, 1] *= np.float32(2.0)
    else:
        new[:, 1, 2] = np.float32(0.5)
    getattr(kf, name).copy_(torch.from_numpy(new))
    w2 = dict(w, **{name: new})

    def reset():
        kf.x.copy_(torch.from_numpy(w["x"])); kf.P.copy_(torch.from_numpy(w["P"]))
    reset()
    for _ in range(2):
        kf.predict(); kf.update(z)
    st = dict(w2)
    for _ in range(2):
        o = _oracle_step(st, w["zs"][0])
        st["x"], st["P"] = o["x"], o["P"]
    rel_close(kf.x.cpu().numpy(), st["x"], 1e-3, "eager x"); rel_close(kf.P.cpu().numpy(), st["P"], 1e-3, "eager P")
    assert _uses_record(kf) and kf._sym_buf is not captured and any(b is captured for b in kf._sym_held)
    reset()
    g.replay()
    torch.cuda.synchronize()
    o = _oracle_step(w, w["zs"][0])
    rel_close(kf.x.cpu().numpy(), o["x"], 1e-3, "replay x"); rel_close(kf.P.cpu().numpy(), o["P"], 1e-3, "replay P")


@pytest.mark.parametrize("how", ["getter", "aliased"])
@pytest.mark.parametrize("name", ["F", "H"])
def test_in_place_edit_of_f_or_h_takes_effect(name, how):
    """An in-place edit of F or H, through the getter or of a tensor the bank aliases, after a record
    was built, reaches the next step."""
    import torch
    N = (1 << 12) + 1
    w = _bench_bank(N, 19)
    kf = _mirror(w)
    t = torch.from_numpy(w[name]).cuda()
    if how == "aliased":
        setattr(kf, name, t)
    z = torch.from_numpy(w["zs"][0]).cuda()
    for _ in range(3):
        kf.predict(); kf.update(z)
    assert _uses_record(kf)
    kf.x = w["x"]; kf.P = w["P"]
    target = getattr(kf, name) if how == "getter" else t
    if name == "F":
        target[:, 2, 3].mul_(3.0)                        # a varying word
        target[:, 1, 0].add_(0.01)                       # and a shared one
    else:
        target[:, 0, 0].mul_(2.0)
    new = w[name].copy()
    if name == "F":
        new[:, 2, 3] *= np.float32(3.0); new[:, 1, 0] += np.float32(0.01)
    else:
        new[:, 0, 0] *= np.float32(2.0)
    kf.predict(); kf.update(z)
    o = _oracle_step(dict(w, **{name: new}), w["zs"][0])
    rel_close(kf.x.cpu().numpy(), o["x"], 1e-3, "x"); rel_close(kf.P.cpu().numpy(), o["P"], 1e-3, "P")


def test_assigning_f_every_step_never_packs():
    import torch
    N = (1 << 12) + 1
    w = _bench_bank(N, 23)
    kf = _mirror(w)
    z = torch.from_numpy(w["zs"][0]).cuda()
    for _ in range(6):
        kf.F = w["F"]
        kf.predict(); kf.update(z)
    assert kf._sym_buf is None and kf._sym_state is None
