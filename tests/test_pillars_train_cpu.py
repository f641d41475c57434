"""CPU: the float64 training-step oracle of the pillar net against the reference's own autograd step, the fixture's
coverage, and host-side refusals of the pillar training C ABI.  No compute calls."""
import ctypes
import os

import numpy as np
import pytest

from pillars_train_oracle import params_from_state_dict, train_step

FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pillars_train_tiny.npz")
CASES = ["A", "beta", "zero"]
KEYS = ["canvas", "dW1", "dW2", "dg1", "db1", "dg2", "db2", "rm1", "rv1", "rm2", "rv2"]


def fixture_case(d, name):
    sd = {str(k): d["%s__sd__%s" % (name, k)] for k in d[name + "__sd_keys"]}
    vs, pcr = d["voxel_size"], d["point_cloud_range"]
    geom = (vs[0], vs[1], vs[0] / 2 + pcr[0], vs[1] / 2 + pcr[1])
    shape = (int(d["batch"]), 64, int(d["nx"]), int(d["ny"]))
    return params_from_state_dict(sd, "pts_voxel_encoder."), geom, shape


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_step(name):
    d = np.load(FIX)
    params, geom, shape = fixture_case(d, name)
    got = train_step(d["features"], d["num_voxels"], d["coors"], params, geom, shape, d["grad_canvas"])
    for k in KEYS:
        gold = d["%s__%s" % (name, k)]
        err = np.abs(got[k] - gold).max() / max(np.abs(gold).max(), 1e-30)
        assert err <= 1e-12, (k, err)
    assert int(d[name + "__nbt1"]) == int(d[name + "__nbt2"]) == 1


def test_fixture_covers_the_traps():
    d = np.load(FIX)
    num, P = d["num_voxels"], int(d["P"])
    assert set(num.tolist()) == set(range(1, P + 1)) and (num == P).sum() >= 4
    assert (d["A__sd__pts_voxel_encoder.pfn_layers.0.norm.weight"] < 0).any()
    # beta: a large shift makes the padded row (relu(shift1)) win the layer-1 max for some channels
    params, geom, shape = fixture_case(d, "beta")
    assert (params["b1"] > 1.0).all()
    # zero: layer-1 channel 3 is zero after ReLU on every slot, so its max ties at 0 and it gets no gradient
    params, geom, shape = fixture_case(d, "zero")
    assert params["b1"][3] < -10 and d["zero__dg1"][3] == 0.0 and d["zero__db1"][3] == 0.0


def test_symbols_exported():
    from bevfusion_b200 import _C
    L = _C.lib()
    for name in ("bevb200_pillar_train_state_bytes", "bevb200_pillar_train_workspace_bytes",
                 "bevb200_pillar_forward_train", "bevb200_pillar_backward_train"):
        assert name in _C.declared_symbols() and hasattr(L, name)


def test_sizes_fit_one_point_tensor():
    from bevfusion_b200 import _C
    L = _C.lib()
    for R in (1, 127, 128, 129, 30000, 120000):
        total = L.bevb200_pillar_train_state_bytes(R, 20) + L.bevb200_pillar_train_workspace_bytes(R, 20)
        assert 0 < total <= R * 640 + (1 << 20), R
    assert L.bevb200_pillar_train_state_bytes(10, 33) == 0 and L.bevb200_pillar_train_workspace_bytes(10, 0) == 0


def _fwd(L, R=10, S=1, P=20, F=5, vox=1, w=1, bn=True, canvas=1, status=1, state=1, sb=None, ws=1, wb=None,
         batch=1, nx=8, ny=8):
    from bevfusion_b200.encoder_plan import _BNDesc
    descs = (_BNDesc * 2)()
    for dd in descs:
        dd.weight = dd.bias = dd.running_mean = dd.running_var = 16
        dd.eps, dd.momentum = 1e-3, 0.01
    sb = L.bevb200_pillar_train_state_bytes(R, P) if sb is None else sb
    wb = L.bevb200_pillar_train_workspace_bytes(R, P) if wb is None else wb
    return L.bevb200_pillar_forward_train(vox and 16, vox and 16, vox and 16, R, S, None, P, F, 0.2, 0.2, 0.1, 0.1,
                                          w and 16, w and 16, descs if bn else None, canvas and 16, batch, nx, ny,
                                          status and 16, state and 16, sb, ws and 16, wb, None)


def _bwd(L, R=10, S=1, P=20, F=5, vox=1, grad=1, out=1, sb=None, wb=None, batch=1):
    sb = L.bevb200_pillar_train_state_bytes(R, P) if sb is None else sb
    wb = L.bevb200_pillar_train_workspace_bytes(R, P) if wb is None else wb
    o = out and 16
    return L.bevb200_pillar_backward_train(vox and 16, vox and 16, vox and 16, R, S, None, P, F, 0.2, 0.2, 0.1, 0.1,
                                           grad and 16, batch, 8, 8, 16, sb, o, o, o, o, o, o, 16, wb, None)


def test_abi_refusals_before_any_launch():
    """Every refusal returns before the first launch: the pointers here are not device memory."""
    from bevfusion_b200 import _C
    L = _C.lib()
    _C.reset_launch_count()
    for kw in (dict(P=33), dict(P=0), dict(F=9), dict(F=2)):
        assert _fwd(L, **kw) == -4 and _bwd(L, **kw) == -4, kw
    for kw in (dict(R=-1), dict(S=0), dict(R=10, S=3), dict(batch=0), dict(nx=0)):
        assert _fwd(L, **kw) == -1, kw
    for kw in (dict(vox=0), dict(w=0), dict(bn=False), dict(canvas=0), dict(status=0), dict(state=0), dict(ws=0)):
        assert _fwd(L, **kw) == -1, kw
    for kw in (dict(R=-1), dict(S=0), dict(vox=0), dict(grad=0), dict(out=0)):
        assert _bwd(L, **kw) == -1, kw
    need_s, need_w = L.bevb200_pillar_train_state_bytes(10, 20), L.bevb200_pillar_train_workspace_bytes(10, 20)
    assert _fwd(L, sb=need_s - 1) == -3 and _fwd(L, wb=need_w - 1) == -3
    assert _bwd(L, sb=need_s - 1) == -3 and _bwd(L, wb=need_w - 1) == -3
    assert _C.launch_count() == 0
