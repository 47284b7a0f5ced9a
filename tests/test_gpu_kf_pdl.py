"""Consecutive launches of the 4/2 fp32 step overlap at their edges (programmatic dependent launch):
the next launch's CTAs start while the previous kernel drains and must not touch memory before it
has completed.  These chains put a producer of what the step reads, or a consumer of what it writes,
right next to a step on the stream, eagerly and inside a captured graph, and compare 8 chained
steps with the oracle."""
import numpy as np
import pytest

from gpu_harness import rel_close

pytestmark = pytest.mark.gpu

STEPS = 8
RING = 4                     # measurement buffers; a captured graph holds RING steps and is replayed STEPS // RING times
NA = (1 << 18) + 1           # odd: a ragged last tile that ends in half a 16-byte granule of z
GRAPHED = pytest.mark.parametrize("graphed", [False, True], ids=["eager", "graph"])


def _bank(N, seed):
    from filterpy_b200.kalman import KalmanFilter
    from filterpy_b200.common import workloads as wl
    w = wl.kf_bank_cv2d(N, seed=seed, steps=STEPS)
    kf = KalmanFilter(4, 2, n_filters=N, dtype=np.float32, device="cuda", diagnostics=False)
    for k in "xPFHQR":
        setattr(kf, k, w[k])
    return kf, w


def _ring(w):
    """RING device buffers and fill(r): load the measurements of steps r*RING .. r*RING+RING-1."""
    import torch
    zbuf = [torch.empty(w["zs"].shape[1:], dtype=torch.float32, device="cuda") for _ in range(RING)]

    def fill(r):
        for t in range(RING):
            zbuf[t].copy_(torch.from_numpy(w["zs"][r * RING + t].astype(np.float32)))
    return zbuf, fill


def _chain(kfs, step, fill, graphed, after=None):
    """STEPS steps: for every block r of RING steps, fill(r), then step(0..RING-1) eagerly or as one
    replay of a graph of them, then after(r).  When graphed, the banks' state is put back in place
    (the graph holds the buffers) after the capture's warm-up runs."""
    import torch
    g = None
    if graphed:
        init = [(kf.x.clone(), kf.P.clone()) for kf in kfs]
        fill(0)
        g = kfs[0].capture(lambda: [step(t) for t in range(RING)])
        for kf, (x0, P0) in zip(kfs, init):
            kf.x.copy_(x0); kf.P.copy_(P0)
    for r in range(STEPS // RING):
        fill(r)
        if g is not None:
            g.replay()
        else:
            for t in range(RING):
                step(t)
        if after is not None:
            after(r)
    torch.cuda.synchronize()


def _oracle(w, zs):
    """The oracle's chain of steps on the bank w with measurements zs[t]; yields the state per step."""
    from oracle import kf as okf
    x, P = w["x"], w["P"]
    for z in zs:
        o = okf.kf_step_bank(x, P, z, w["F"], w["H"], w["Q"], w["R"])
        x, P = o["x"], o["P"]
        yield x, P


@GRAPHED
def test_step_reads_what_the_previous_step_wrote(graphed):
    """Bank B (2 NA filters) steps with z = A.x viewed as (2 NA, 2) right after bank A's step: one
    launch of the kernel reads what the launch before it wrote."""
    a, wa = _bank(NA, 11)
    b, wb = _bank(2 * NA, 12)
    zbuf, fill = _ring(wa)

    def step(t):
        a.predict(); a.update(zbuf[t])
        b.predict(); b.update(a.x.view(-1, 2))

    _chain([a, b], step, fill, graphed)
    sa = list(_oracle(wa, [z.astype(np.float32) for z in wa["zs"]]))
    xa, Pa = sa[-1]
    xb, Pb = list(_oracle(wb, [x.astype(np.float32).reshape(-1, 2) for x, _ in sa]))[-1]
    rel_close(a.x.cpu().numpy(), xa, 1e-3, "A.x"); rel_close(a.P.cpu().numpy(), Pa, 1e-3, "A.P")
    rel_close(b.x.cpu().numpy(), xb, 1e-3, "B.x"); rel_close(b.P.cpu().numpy(), Pb, 1e-3, "B.P")


@GRAPHED
def test_step_reads_z_a_torch_kernel_just_wrote(graphed):
    """z of every step is written by a torch kernel immediately before the update that reads it."""
    import torch
    kf, w = _bank(NA, 13)
    zbuf, fill = _ring(w)
    z = torch.empty_like(zbuf[0])

    def step(t):
        kf.predict()
        torch.mul(zbuf[t], 2.0, out=z)
        kf.update(z)

    _chain([kf], step, fill, graphed)
    x, P = list(_oracle(w, [2.0 * z.astype(np.float32) for z in w["zs"]]))[-1]
    rel_close(kf.x.cpu().numpy(), x, 1e-3, "x"); rel_close(kf.P.cpu().numpy(), P, 1e-3, "P")


@GRAPHED
def test_torch_kernel_reads_x_right_after_the_step(graphed):
    """kf.x is copied by a torch kernel right after every step, and the next step overwrites it."""
    import torch
    kf, w = _bank(NA, 14)
    zbuf, fill = _ring(w)
    seen = [torch.empty_like(kf.x) for _ in range(RING)]
    got = []

    def step(t):
        kf.predict(); kf.update(zbuf[t])
        seen[t].copy_(kf.x)

    _chain([kf], step, fill, graphed, after=lambda r: got.extend(s.cpu().numpy() for s in seen))
    want = list(_oracle(w, [z.astype(np.float32) for z in w["zs"]]))
    assert len(got) == STEPS
    for t in range(STEPS):
        rel_close(got[t], want[t][0], 1e-3, "x after step %d" % t)
    rel_close(kf.P.cpu().numpy(), want[-1][1], 1e-3, "P")
