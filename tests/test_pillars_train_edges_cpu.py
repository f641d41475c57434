"""CPU: the boundary cases of the PointPillars training step (pillars_train_cases) land on their boundaries and meet
their margins, and the float64 oracle's collapsed padding (kind A / kind B rows) equals an uncollapsed float64
autograd restatement in plain torch on every P x F, few-row, canvas and tie case."""
import numpy as np
import pytest
import torch
from torch.nn import functional as Fn

import pillars_train_cases as C
from pillars_train_oracle import inside_canvas

KEYS = ["canvas", "dW1", "dW2", "dg1", "db1", "dg2", "db2", "rm1", "rv1", "rm2", "rv2"]
PS = [1, 2, 3, C.MAX_P - 1, C.MAX_P]
FS = list(range(3, C.MAX_F + 1))


def torch_step(case, rule="first"):
    """one training step over every slot of the kept rows: decorate, mask, linear, batch_norm(training=True) over
    all M * P slots, ReLU, the max as a gather at an explicit argmax (the first slot attaining it, or the last),
    concat, layer 2, the scatter to the canvas -> the oracle's dict"""
    k = case.keep()
    x = torch.from_numpy(case.voxels[k])
    n = torch.from_numpy(case.num_points[k].astype(np.int64))
    c = torch.from_numpy(case.coords4[k].astype(np.int64))
    p = {key: torch.from_numpy(v.copy()) for key, v in case.params.items()}
    for key in ("W1", "W2", "g1", "b1", "g2", "b2"):
        p[key].requires_grad_(True)
    M, P, _ = x.shape
    vx, vy, xo, yo = case.geom
    mean = x[:, :, :3].sum(dim=1, keepdim=True) / n.double()[:, None, None]
    xc, yc = c[:, 1].double() * vx + xo, c[:, 2].double() * vy + yo
    h = torch.cat([x, x[:, :, :3] - mean, (x[:, :, 0] - xc[:, None])[..., None], (x[:, :, 1] - yc[:, None])[..., None]],
                  dim=2)
    h = h * (torch.arange(P)[None, :] < n[:, None]).double()[..., None]

    def bn_relu(z, layer):
        y = Fn.batch_norm(z.reshape(M * P, -1), p["rm" + layer], p["rv" + layer], p["g" + layer], p["b" + layer],
                          training=True, momentum=C.MOMENTUM, eps=C.EPS)
        return torch.relu(y).reshape(M, P, -1)

    def pick(y):
        v = y.detach().numpy()
        idx = v.argmax(axis=1) if rule == "first" else P - 1 - v[:, ::-1].argmax(axis=1)  # numpy: first occurrence
        return y.gather(1, torch.from_numpy(idx)[:, None, :]).squeeze(1)

    y1 = bn_relu(Fn.linear(h, p["W1"]), "1")
    m1 = pick(y1)
    y2 = bn_relu(Fn.linear(torch.cat([y1, m1[:, None, :].expand(M, P, 32)], dim=2), p["W2"]), "2")
    out = pick(y2)
    B, _, nx, ny = case.canvas_shape
    ins = torch.from_numpy(inside_canvas(case.coords4[k], case.canvas_shape))
    ci = c[ins]
    canvas = torch.zeros(B, nx, ny, 64, dtype=torch.float64).index_put((ci[:, 0], ci[:, 1], ci[:, 2]), out[ins])
    canvas = canvas.permute(0, 3, 1, 2)
    (canvas * torch.from_numpy(case.grad_canvas)).sum().backward()
    got = dict(canvas=canvas.detach().numpy(), dW1=p["W1"].grad, dW2=p["W2"].grad, dg1=p["g1"].grad,
               db1=p["b1"].grad, dg2=p["g2"].grad, db2=p["b2"].grad)
    got.update({key: p[key] for key in ("rm1", "rv1", "rm2", "rv2")})
    return {key: np.asarray(v.detach() if torch.is_tensor(v) else v) for key, v in got.items()}


def rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def assert_matches_oracle(case):
    got, gold = torch_step(case), case.gold()
    errs = {key: rel(got[key], gold[key]) for key in KEYS}
    assert max(errs.values()) <= 1e-12, (case.name, errs)


def assert_settled(case):
    relu, gap, found, undeclared = C.margins(case)
    assert relu >= 1.0 and gap >= 1.0, (case.name, relu, gap)
    assert not undeclared, (case.name, undeclared)
    assert C.landed(case, found), (case.name, case.ties, found)


# ---------------------------------------------------------------------------------------------------- constants
def test_boundaries_come_from_the_source():
    assert C.CHUNK % C.WARPS == 0 and C.CHUNK > C.WARPS
    assert (C.MAX_P, C.MAX_F) == (C.cu_int("kPfnMaxP"), C.cu_int("kPfnMaxF")) and C.MAX_P <= 32   # one warp lane each
    assert C.GRID_B23 < C.GRID_P13
    assert C.grid_chunks() == [C.NUM_SMS * C.GRID_B23 + d for d in (-1, 0, 1)] + \
        [C.NUM_SMS * C.GRID_P13 + d for d in (-1, 0, 1)]


# ---------------------------------------------------------------------------------------------------- builders
@pytest.mark.parametrize("F", FS)
@pytest.mark.parametrize("P", PS)
def test_pf_case_lands_and_matches_autograd(P, F):
    case = C.pf_case(P, F, seed=P * 10 + F)
    assert (case.P, case.F) == (P, F)
    pads = set((P - case.num_points).tolist())
    assert pads == set(C.pad_kinds(P)) and (case.num_points >= 1).all()
    assert {0, 1, 2} & set(range(P)) <= pads and (P < 4 or max(pads) > 2)
    assert_settled(case)
    assert_matches_oracle(case)


@pytest.mark.parametrize("name", list(C.FEW_ROWS))
def test_few_rows_cases(name):
    case = C.few_rows_case(name)
    assert case.slots() == (1 if name == "N1" else 2)
    if name != "N1":
        assert_settled(case)
        assert_matches_oracle(case)
        gold = case.gold()
        for layer in "12":                     # the unbiased factor N / (N - 1) = 2
            want = (1 - C.MOMENTUM) * case.params["rv" + layer] + C.MOMENTUM * 2.0 * gold["var" + layer]
            assert np.allclose(gold["rv" + layer], want, rtol=1e-14, atol=0)


@pytest.mark.parametrize("R", C.chunk_rows())
def test_chunk_rows_case(R):
    case = C.rows_case(R, seed=R)
    assert case.R == R and R % C.CHUNK in (C.CHUNK - 1, 0, 1)
    assert_settled(case)


@pytest.mark.parametrize("chunks", C.grid_chunks())
def test_grid_case(chunks):
    case = C.grid_case(chunks, seed=chunks)
    assert -(-case.R // C.CHUNK) == chunks and case.R % C.CHUNK != 0
    assert_settled(case)


@pytest.mark.parametrize("name", list(C.SEGMENTS))
def test_segment_case(name):
    case = C.segment_case(name, seed=len(name))
    S, cap, n_dev = C.SEGMENTS[name]
    assert (case.segments, case.cap) == (S, cap)
    if n_dev is not None:
        assert len(case.keep()) == sum(min(max(n, 0), cap) for n in n_dev)
        assert {-1, cap + 1, C.INT32_MAX} & set(n_dev) or name == "S1 null"
    drop = np.setdiff1d(np.arange(case.R), case.keep())
    assert np.isnan(case.voxels[drop]).all()
    assert_settled(case)


def test_segment_counts_cover_every_clamp():
    counts = set(C.SEGMENTS["S64 every count"][2])
    assert {-1, 0, 1, 4, 5, C.INT32_MAX} <= counts


@pytest.mark.parametrize("nx, ny", [(37, 53), (53, 37)])
def test_canvas_case_lands_and_matches_autograd(nx, ny):
    case = C.canvas_case(nx, ny, seed=nx)
    B = case.canvas[0]
    cells = {tuple(r[:3]) for r in case.coords4.tolist()}
    assert {(B - 1, nx - 1, ny - 1), (0, nx, 3), (1, 2, ny), (0, 4, -1), (B, 1, 1)} <= cells
    assert_settled(case)
    assert_matches_oracle(case)
    off = ~inside_canvas(case.coords4, case.canvas_shape)
    gold = case.gold()
    assert gold["canvas"].any() and off.sum() == 5


@pytest.mark.parametrize("kind", ["a", "b", "c"])
def test_tie_case_lands_and_matches_autograd(kind):
    case = C.tie_case(kind)
    assert_settled(case)
    assert_matches_oracle(case)
    gold = case.gold()
    if kind == "c":
        for ch in (5, 17, 40):
            assert gold["dg2"][ch] == 0 and gold["db2"][ch] == 0 and not gold["dW2"][ch].any()
            assert not gold["canvas"][:, ch].any()


@pytest.mark.parametrize("kind", ["a", "b"])
def test_tie_routing_shows_in_dw1(kind):
    """the last instead of the first tied slot moves dW1 by far more than the GPU bound (1e-4): a kernel that routed
    a built tie's gradient to the wrong row would fail"""
    case = C.tie_case(kind)
    first, last = torch_step(case), torch_step(case, rule="last")
    assert rel(last["dW1"], first["dW1"]) >= 1e-2
