"""GPU: the PointPillars training step through its C ABI (bevb200_pillar_forward_train / _backward_train) at every
P, F, chunk, segment and canvas boundary, against the float64 oracle (pillars_train_oracle.train_step) on the cases
of pillars_train_cases, whose every ReLU and max decision has a margin built in.

State and workspace are exactly their queried sizes inside canary-filled buffers, and so is the zeroed canvas;
every backward output starts as NaN.  Bounds are those of test_pillars_train_gpu: canvas and running-statistics
moves <= 1e-5, gradients <= 1e-4 (max-abs error over the float64 value's max); the one-slot case, the dead channels
and the contracts are exact.  Each group's worst error / bound ratio is printed."""
import numpy as np
import pytest
import torch

import pillars_train_cases as C
from bevfusion_b200 import _C
from bevfusion_b200.encoder_plan import _BNDesc
from test_encoder_train_edges_gpu import CANARY, _guard_intact, _guarded
from test_pillars_train_gpu import rel_err

pytestmark = pytest.mark.gpu

EWORKSPACE, FEW_ROWS = -3, 2
CANVAS_BOUND, STATS_BOUND, GRAD_BOUND = 1e-5, 1e-5, 1e-4
GRADS = ["dW1", "dW2", "dg1", "db1", "dg2", "db2"]
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for group, (ratio, what) in sorted(WORST.items()):
        print("pillar train edges  %-10s worst error / bound %.3f  (%s)" % (group, ratio, what))


class Run:
    """one case on the device: its row source, parameters, guarded state / workspace / canvas"""

    def __init__(self, case, dev, nbt=True):
        self.case, self.dev, self.L = case, dev, _C.lib()

        def t(a, dt=np.float32):
            return torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)
        p = case.params
        self.vox, self.num, self.c4 = t(case.voxels), t(case.num_points, np.int32), t(case.coords4, np.int32)
        self.n_dev = None if case.n_dev is None else t(case.n_dev, np.int32)
        self.w1, self.w2 = t(p["W1"]), t(p["W2"])
        self.g, self.b = [t(p["g1"]), t(p["g2"])], [t(p["b1"]), t(p["b2"])]
        self.rm, self.rv = [t(p["rm1"]), t(p["rm2"])], [t(p["rv1"]), t(p["rv2"])]
        self.nbt = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in range(2)] if nbt else None
        self.sb = self.L.bevb200_pillar_train_state_bytes(case.R, case.P)
        self.wb = self.L.bevb200_pillar_train_workspace_bytes(case.R, case.P)
        assert self.sb > 0 and self.wb > 0
        self.state_buf, self.state = _guarded(self.sb, dev)
        self.ws_buf, self.ws = _guarded(self.wb, dev)
        B, nx, ny = case.canvas
        self.cb = B * 64 * nx * ny * 4
        self.canvas_buf, cv = _guarded(self.cb, dev)
        cv.zero_()
        self.canvas = cv.view(torch.float32).view(B, 64, nx, ny)
        self.gcan = t(case.grad_canvas)
        self.status = torch.full((1,), -1, dtype=torch.int32, device=dev)

    def _rows(self):
        c = self.case
        return (_C.ptr(self.vox), _C.ptr(self.num), _C.ptr(self.c4), c.R, c.segments, _C.ptr(self.n_dev), c.P, c.F,
                *c.geom)

    def _bn(self):
        descs = (_BNDesc * 2)()
        for i, d in enumerate(descs):
            d.weight, d.bias = _C.ptr(self.g[i]), _C.ptr(self.b[i])
            d.running_mean, d.running_var = _C.ptr(self.rm[i]), _C.ptr(self.rv[i])
            d.num_batches_tracked = _C.ptr(self.nbt[i]) if self.nbt else None
            d.eps, d.momentum = C.EPS, C.MOMENTUM
        return descs

    def forward(self, sb=None, wb=None):
        B, nx, ny = self.case.canvas
        rc = self.L.bevb200_pillar_forward_train(
            *self._rows(), _C.ptr(self.w1), _C.ptr(self.w2), self._bn(), _C.ptr(self.canvas), B, nx, ny,
            _C.ptr(self.status), _C.ptr(self.state), self.sb if sb is None else sb, _C.ptr(self.ws),
            self.wb if wb is None else wb, _C.current_stream(self.dev))
        torch.cuda.synchronize()
        return rc

    def backward(self, sb=None, wb=None, fill=float("nan")):
        """-> (return code, {name: gradient on the host}), every output prefilled with `fill`"""
        B, nx, ny = self.case.canvas
        like = (self.w1, self.w2, self.g[0], self.b[0], self.g[1], self.b[1])
        outs = [torch.full_like(t, fill) for t in like]
        rc = self.L.bevb200_pillar_backward_train(
            *self._rows(), _C.ptr(self.gcan), B, nx, ny, _C.ptr(self.state), self.sb if sb is None else sb,
            *[_C.ptr(o) for o in outs], _C.ptr(self.ws), self.wb if wb is None else wb, _C.current_stream(self.dev))
        torch.cuda.synchronize()
        return rc, dict(zip(GRADS, [o.cpu() for o in outs]))

    def guards_intact(self):
        return all(_guard_intact(b, n) for b, n in ((self.state_buf, self.sb), (self.ws_buf, self.wb),
                                                  (self.canvas_buf, self.cb)))

    def stats(self):
        return {"rm1": self.rm[0], "rv1": self.rv[0], "rm2": self.rm[1], "rv2": self.rv[1]}


def _record(group, ratio, what):
    if ratio >= WORST.get(group, (-1.0, ""))[0]:
        WORST[group] = (ratio, what)


def check(case, dev, group):
    """one full step against float64 -> (run, gradients)"""
    run = Run(case, dev)
    assert run.forward() == 0, run.L.bevb200_last_error()
    rc, got = run.backward()
    assert rc == 0, run.L.bevb200_last_error()
    gold, p = case.gold(), case.params
    assert int(run.status[0]) == 0
    canvas = run.canvas.cpu().numpy()
    errs = {"canvas": rel_err(canvas, gold["canvas"]) / CANVAS_BOUND}
    for k, v in run.stats().items():
        errs[k] = rel_err(v.cpu().double().numpy() - p[k], gold[k] - p[k]) / STATS_BOUND
    errs.update({k: rel_err(got[k].numpy(), gold[k]) / GRAD_BOUND for k in GRADS})
    worst = max(errs, key=errs.get)
    _record(group, errs[worst], "%s, %s" % (case.name, worst))
    print("%-24s worst error / bound %.3f (%s)" % (case.name, errs[worst], worst))
    assert errs[worst] <= 1.0, (case.name, errs)
    assert not canvas[gold["canvas"] == 0].any(), "%s: a cell without a positive max is not 0" % case.name
    assert [int(n) for n in run.nbt] == [1, 1]
    assert run.guards_intact(), "%s: a byte outside the state, the workspace or the canvas changed" % case.name
    return run, got


# ---------------------------------------------------------------------------------------------------- P x F
@pytest.mark.parametrize("F", range(3, C.MAX_F + 1))
@pytest.mark.parametrize("P", [1, 2, 3, C.MAX_P - 1, C.MAX_P])
def test_p_by_f(cuda, P, F):
    """every pad kind P allows: no padding row, kind A alone, kind B once and many times (n >= 1)"""
    check(C.pf_case(P, F, seed=P * 10 + F), cuda, "P x F")


# ---------------------------------------------------------------------------------------------------- few rows
def test_one_slot_sets_the_flag(cuda):
    """N = P * pillars = 1: the flag, untouched statistics and canvas, every gradient exactly 0 (over NaN)"""
    case = C.few_rows_case("N1")
    assert case.slots() == 1
    run = Run(case, cuda)
    before = {k: v.clone() for k, v in run.stats().items()}
    assert run.forward() == 0
    rc, got = run.backward()
    assert rc == 0
    assert int(run.status[0]) == FEW_ROWS
    for k, v in run.stats().items():
        assert torch.equal(v, before[k]), k
    assert [int(n) for n in run.nbt] == [0, 0]
    assert not run.canvas.any()
    for k in GRADS:
        assert not got[k].isnan().any() and not got[k].any(), k
    assert run.guards_intact()
    _record("few rows", 0.0, "N1 exact")


@pytest.mark.parametrize("name", ["N2-P1", "N2-P2"])
def test_two_slots_proceed(cuda, name):
    """N = 2 (two 1-point pillars at P = 1, or one 1-point pillar and its padding row at P = 2): the step runs and
    running_var takes the unbiased factor N / (N - 1) = 2"""
    case = C.few_rows_case(name)
    assert case.slots() == 2
    check(case, cuda, "few rows")


# ---------------------------------------------------------------------------------------------------- chunks
@pytest.mark.parametrize("R", C.chunk_rows())
def test_chunk_rows(cuda, R):
    check(C.rows_case(R, seed=R), cuda, "chunks")


@pytest.mark.parametrize("chunks", C.grid_chunks())
def test_grid_stride_chunks(cuda, chunks):
    """chunk counts around kNumSMs * 2 (the B2 / B3 grid) and kNumSMs * 4 (the P1-P3 / B1 grid)"""
    check(C.grid_case(chunks, seed=chunks), cuda, "grids")


# ---------------------------------------------------------------------------------------------------- segments
@pytest.mark.parametrize("name", list(C.SEGMENTS))
def test_segments(cuda, name):
    """n_dev of -1, 0, 1, cap, cap + 1 and INT32_MAX, or null; rows past each count are NaN with garbage counts and
    coordinates"""
    check(C.segment_case(name, seed=len(name)), cuda, "segments")


# ---------------------------------------------------------------------------------------------------- canvas
@pytest.mark.parametrize("nx, ny", [(37, 53), (53, 37)])
def test_canvas(cuda, nx, ny):
    """nx != ny both ways, pillars on the last batch, row and column, and pillars just off the canvas (counted in
    both BNs, no write, no gradient; the canvas guard catches a write past its end)"""
    check(C.canvas_case(nx, ny, seed=nx), cuda, "canvas")


# ---------------------------------------------------------------------------------------------------- ties
@pytest.mark.parametrize("kind", ["a", "b", "c"])
def test_ties_and_dead_channels(cuda, kind):
    """(a) two real rows tied in one layer-1 channel, (b) a real row tied with the padding row in both layers: the
    lowest slot takes the gradient (test_pillars_train_edges_cpu shows the other choice moves dW1 far past the
    bound); (c) layer-2 channels below 0 everywhere or exactly 0 take no gradient at all"""
    case = C.tie_case(kind)
    run, got = check(case, cuda, "ties")
    if kind == "c":
        for ch in (5, 17, 40):
            assert got["dg2"][ch] == 0 and got["db2"][ch] == 0 and not got["dW2"][ch].any(), ch
            assert not run.canvas[:, ch].any(), ch


# ---------------------------------------------------------------------------------------------------- contracts
def test_backward_reads_state_only_and_steps_repeat(cuda):
    """two backwards on one state (over NaN, then over 1e30) are bit-equal and leave the state alone; a second full
    step on fresh buffers from the same starting statistics is bit-equal to the first"""
    case = C.pf_case(C.MAX_P, 5, seed=99)
    runs = []
    for _ in range(2):
        run, got = check(case, cuda, "contracts")
        state = run.state_buf.clone()
        rc, again = run.backward(fill=1e30)
        assert rc == 0 and torch.equal(run.state_buf, state)
        for k in GRADS:
            assert torch.equal(got[k], again[k]), k
        runs.append((run, got))
    (a, ga), (b, gb) = runs
    assert torch.equal(a.canvas, b.canvas)
    for k in GRADS:
        assert torch.equal(ga[k], gb[k]), k
    for k, v in a.stats().items():
        assert torch.equal(v, b.stats()[k]), k


@pytest.mark.parametrize("which", ["forward state", "forward workspace", "backward state", "backward workspace"])
def test_one_byte_short(cuda, which):
    """a state or workspace one byte short of its query: BEVB200_EWORKSPACE before any write"""
    case = C.pf_case(3, 4, seed=7)
    run = Run(case, cuda)
    short = dict(sb=run.sb - 1) if which.endswith("state") else dict(wb=run.wb - 1)
    stats = {k: v.clone() for k, v in run.stats().items()}
    if which.startswith("forward"):
        assert run.forward(**short) == EWORKSPACE
        assert int(run.status[0]) == -1 and not run.canvas.any()
        assert bool((run.state_buf == CANARY).all())
        assert [int(n) for n in run.nbt] == [0, 0]
        assert bool((run.ws_buf == CANARY).all())
    else:
        assert run.forward() == 0
        stats = {k: v.clone() for k, v in run.stats().items()}
        state, ws = run.state_buf.clone(), run.ws_buf.clone()   # the forward used the workspace too
        rc, got = run.backward(fill=3.5, **short)
        assert rc == EWORKSPACE
        assert torch.equal(run.state_buf, state) and torch.equal(run.ws_buf, ws)
        for k in GRADS:
            assert bool((got[k] == 3.5).all()), k
    for k, v in run.stats().items():
        assert torch.equal(v, stats[k]), k
    assert run.guards_intact()


def test_num_batches_tracked_nullable(cuda):
    """a null num_batches_tracked changes nothing else; a non-null one counts the step"""
    case = C.pf_case(2, 6, seed=5)
    a, ga = check(case, cuda, "contracts")
    b = Run(case, cuda, nbt=False)
    assert b.forward() == 0
    rc, gb = b.backward()
    assert rc == 0
    assert torch.equal(a.canvas, b.canvas)
    for k in GRADS:
        assert torch.equal(ga[k], gb[k]), k
    for k, v in a.stats().items():
        assert torch.equal(v, b.stats()[k]), k
