"""CPU: the C ABI of the sync-free BEV pooling / fused-lift twins (*_dev) -- workspace queries against their layouts,
refusal of zero and negative capacities before any device work, and the ctypes signatures against the header."""
import re

import pytest

INT_MAX = 2**31 - 1
TUNED = (16, 32, 64, 80, 96, 128, 160, 256)


def align(nbytes):
    return (nbytes + 255) // 256 * 256


def test_dev_workspace_queries_match_their_layouts():
    from bevfusion_b200 import _C
    L = _C.lib()
    for n in (1, 7040, 1993728, 13516800):
        for c in (16, 24, 80, 256):
            ranges = max((n + 127) // 128, 132 * 8)          # two partial rows per TMA warp range, one cell per interval
            want = align(2 * ranges * c * 4) + align(n * 4)
            assert L.bevb200_bev_pool_dev_workspace_bytes(n, c) == want == L.bevb200_bev_pool_workspace_bytes(n, c)
        for cap in (1, n // 3 + 1, n):
            assert L.bevb200_bev_pool_lift_prepare_dev_workspace_bytes(n, cap) == \
                L.bevb200_bev_pool_lift_prepare_workspace_bytes(n) > 16 * n
            for c in TUNED:
                # one partial row per segment under the cap + the cell of every interval; one int per segment
                assert L.bevb200_bev_pool_lift_columns_dev_workspace_bytes(cap, n, c) == \
                    align(cap * c * 4) + align(n * 4) + 256
                assert L.bevb200_bev_pool_lift_columns_backward_dev_workspace_bytes(cap, c) == align(cap * 4) + 256
        for c in TUNED:
            assert L.bevb200_bev_pool_lift_backward_dev_workspace_bytes(n, c) == align(n * 4) + 256
    assert L.bevb200_bev_pool_lift_columns_backward_dev_workspace_bytes(100, 24) == 0      # no tuned kernel
    assert L.bevb200_bev_pool_lift_backward_dev_workspace_bytes(100, 24) == 0
    assert L.bevb200_bev_pool_lift_prepare_dev_workspace_bytes(100, 101) == 0               # cap above capacity


@pytest.mark.parametrize("bad", [0, -1, -INT_MAX])
def test_zero_and_negative_capacities_are_refused(bad):
    from bevfusion_b200 import _C
    L = _C.lib()
    assert L.bevb200_bev_pool_dev_workspace_bytes(bad, 80) == 0
    assert L.bevb200_bev_pool_lift_prepare_dev_workspace_bytes(bad, 10) == 0
    assert L.bevb200_bev_pool_lift_prepare_dev_workspace_bytes(1000, bad) == 0
    assert L.bevb200_bev_pool_lift_columns_dev_workspace_bytes(bad, 1000, 80) == 0
    assert L.bevb200_bev_pool_lift_columns_dev_workspace_bytes(10, bad, 80) == 0
    assert L.bevb200_bev_pool_lift_columns_dev_workspace_bytes(10, 1000, bad) == 0
    assert L.bevb200_bev_pool_lift_columns_backward_dev_workspace_bytes(bad, 80) == 0
    assert L.bevb200_bev_pool_lift_backward_dev_workspace_bytes(bad, 80) == 0
    # the calls refuse before touching a pointer or the device (all pointers here are NULL, the stream is 0)
    einval = -1
    P = [None] * 12
    assert L.bevb200_bev_pool_perm_dev(1, 1, 4, 4, bad, 80, *P[:8], 0, None) == einval
    assert L.bevb200_bev_pool_grad_perm_dev(1, 1, 4, 4, bad, 80, *P[:8]) == einval
    assert L.bevb200_bev_pool_lift_dev(1, 1, 4, 4, bad, 80, None, None, 2, 4, *P[:8], 0, None) == einval
    assert L.bevb200_bev_pool_lift_prepare_dev(None, None, None, bad, 1, 1, 2, 2, 2, *P[:8], 0, None) == einval
    assert L.bevb200_bev_pool_lift_prepare_dev(None, None, None, 16, bad, 1, 2, 2, 2, *P[:8], 0, None) == einval
    assert L.bevb200_bev_pool_lift_columns_dev(1, 1, 4, 4, bad, 80, None, None, 1, 2, 2, 2, *P[:7], 8, *P[:4], 0,
                                               None) == einval
    assert L.bevb200_bev_pool_lift_columns_dev(1, 1, 4, 4, 16, 80, None, None, 1, 2, 2, 2, *P[:7], bad, *P[:4], 0,
                                               None) == einval
    assert L.bevb200_bev_pool_lift_columns_backward_dev(1, 1, 4, 4, bad, 80, None, None, None, 1, 2, 2, 2, *P[:5], 8,
                                                        *P[:6], 0, None) == einval
    assert L.bevb200_bev_pool_lift_backward_dev(1, 1, 4, 4, bad, 80, None, None, None, 2, 4, *P[:9], 0, None) == einval
    assert b"capacit" in L.bevb200_last_error()


def test_prepare_dev_refuses_a_cap_above_capacity_and_a_missing_status_word():
    from bevfusion_b200 import _C
    L = _C.lib()
    A = [0x100] * 8                       # placeholder addresses: the checks come before any access
    assert L.bevb200_bev_pool_lift_prepare_dev(*A[:3], 16, 17, 1, 2, 2, 2, *A, 0, None) == -1
    assert b"max_segments" in L.bevb200_last_error()
    assert L.bevb200_bev_pool_lift_prepare_dev(*A[:3], 16, 8, 1, 2, 2, 2, *A[:6], None, 0x100, 0, None) == -1
    assert b"lift_form" in L.bevb200_last_error()
    assert L.bevb200_bev_pool_lift_columns_dev(1, 1, 4, 4, 16, 80, None, None, 1, 2, 2, 2, *[None] * 7, 8,
                                               None, None, None, None, 0, None) == -1
    assert b"lift_form" in L.bevb200_last_error()


_CTYPE = {"int": "c_int", "size_t": "c_size_t", "float": "c_float", "double": "c_double", "long long": "c_longlong"}


def _header_signature(text, name):
    m = re.search(r"BEVB200_API\s+([\w\s\*]+?)\s*\b" + name + r"\s*\(([^)]*)\)\s*;", text, re.S)
    assert m, name
    ret, params = m.group(1).strip(), m.group(2)

    def kind(decl):
        decl = " ".join(decl.replace("const ", "").split())
        if "*" in decl:
            return "c_void_p"
        return _CTYPE[decl.rsplit(" ", 1)[0]]

    args = [kind(p) for p in params.split(",") if p.strip() and p.strip() != "void"]
    return kind(ret + " x"), args


def test_dev_signatures_match_the_header():
    import ctypes
    from bevfusion_b200 import _C
    with open(_C.HEADER_PATH) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    names = [n for n in _C.declared_symbols() if n.startswith("bevb200_bev_pool") and "_dev" in n]
    assert len(names) == 12
    for name in names:
        res, args = _C._SIGNATURES[name]
        want_res, want_args = _header_signature(text, name)
        assert res is getattr(ctypes, want_res), name
        assert list(args) == [getattr(ctypes, a) for a in want_args], name
    order = list(_C._SIGNATURES)
    assert [n for n in order if n in names] == sorted(names, key=lambda n: text.index(n + "("))
    assert ctypes.sizeof(ctypes.c_void_p) == 8
