"""Host side of the native SparseEncoder training path: the C declarations and their ctypes signatures, the size
of the state a training forward keeps, and the float64 oracle's BatchNorm against torch's.  No device is touched."""
import ctypes
import re

import pytest
import torch

from bevfusion_b200 import _C
from bevfusion_b200.encoder_plan import EncoderPlan, _BNDesc
from bevfusion_b200.sparse_encoder import voxelnet_0p075_encoder
from encoder_train_oracle import bn_train

NEW = ["bevb200_encoder_train_state_bytes", "bevb200_encoder_train_saved", "bevb200_encoder_forward_train",
       "bevb200_encoder_backward_workspace_bytes", "bevb200_encoder_backward"]


def _declaration(name):
    with open(_C.HEADER_PATH) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    m = re.search(r"BEVB200_API\s+([^;]*?)\b%s\s*\(([^)]*)\)\s*;" % name, text, flags=re.S)
    assert m, name
    return m.group(1).strip(), [a.strip() for a in m.group(2).split(",")]


@pytest.mark.parametrize("name", NEW)
def test_declared_with_matching_signature(name):
    assert name in _C.declared_symbols()
    ret, args = _declaration(name)
    res, argtypes = _C._SIGNATURES[name]
    assert len(args) == len(argtypes), (name, args)
    assert (res is _C.c_size_t) == (ret == "size_t") and (res is _C.c_int) == (ret == "int")
    for a, t in zip(args, argtypes):
        if "*" in a:
            assert t is _C._P, (name, a)
        elif a.startswith("long long"):
            assert t is ctypes.c_longlong, (name, a)
        elif a.startswith("size_t"):
            assert t is _C.c_size_t, (name, a)
        else:
            assert t is _C.c_int, (name, a)


def test_bn_struct_mirrors_the_header():
    with open(_C.HEADER_PATH) as f:
        text = f.read()
    body = re.search(r"typedef struct \{([^}]*)\} bevb200_encoder_bn_t;", text, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = re.findall(r"\**(\w+)\s*[,;]", body)
    assert names == [f[0] for f in _BNDesc._fields_]


def test_train_state_bytes_scales_with_rows_batch_and_caps():
    plan = EncoderPlan(voxelnet_0p075_encoder())
    a = plan.train_state_bytes(60000, 1)
    b = plan.train_state_bytes(120000, 1)
    c = plan.train_state_bytes(120000, 4)
    caps = plan.level_caps(120000, 1)
    tight = plan.train_state_bytes(120000, 1, [0] + [v // 2 for v in caps[1:]])
    assert 0 < a < b < c and tight < b
    assert plan.backward_workspace_bytes(60000, 1) < plan.backward_workspace_bytes(120000, 1)
    print("voxelnet 0.075, 120000 voxels, B = 1: train state %.2f GB, backward workspace %.2f GB" % (
        b / 1e9, plan.backward_workspace_bytes(120000, 1) / 1e9))


@pytest.mark.parametrize("n", [2, 7, 1000])
def test_oracle_bn_matches_torch_batchnorm(n):
    torch.manual_seed(n)
    bn = torch.nn.BatchNorm1d(16, eps=1e-3, momentum=0.01).double().train()
    bn.running_mean.normal_(0, 0.1)
    bn.running_var.uniform_(0.5, 1.5)
    bn.weight.data.uniform_(0.8, 1.2)
    bn.bias.data.normal_(0, 0.1)
    x = torch.randn(n, 16, dtype=torch.float64) * 2 + 0.5
    rm, rv = bn.running_mean.clone(), bn.running_var.clone()
    y = bn_train(x, bn.weight.detach(), bn.bias.detach(), rm, rv, bn.eps, bn.momentum)
    want = bn(x)
    assert torch.allclose(y, want.detach(), rtol=1e-12, atol=1e-12)
    assert torch.allclose(rm, bn.running_mean, rtol=1e-12, atol=1e-14)
    assert torch.allclose(rv, bn.running_var, rtol=1e-12, atol=1e-14)
