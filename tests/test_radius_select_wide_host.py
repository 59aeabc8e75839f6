"""CPU checks of the wide cell-grid radius select (k up to 256): the C-ABI entries and header agree, their host checks
return the documented codes, `radius_neighbors_wide` rejects misuse before anything launches, and a layer descriptor grows
by exactly the cell scratch when EGNN_FLAG_CELL_SELECT_WIDE makes a k > 32 layer eligible, and not otherwise."""
import ctypes as C
import os
import re

import pytest
import torch

from test_radius_select_host import _layer_descs, cell_bytes
from util import nat  # noqa: F401  (module-scoped fixture)

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDE = ("egnn_radius_select_wide_workspace_bytes", "egnn_radius_select_wide", "egnn_radius_select_wide_triclinic")


def test_symbols_match_the_header(nat):
    header = open(os.path.join(REPO, "include", "egnn_b200.h")).read()
    assert re.search(r"#define EGNN_FLAG_CELL_SELECT_WIDE \(1u << 11\)", header)
    assert nat.FLAG_CELL_SELECT_WIDE == 1 << 11
    for name in WIDE:
        assert name in nat.SYMBOLS
        m = re.search(r"\bint " + name + r"\(([^)]*)\);", header)
        assert m, name
        assert len(m.group(1).split(",")) == len(nat.SYMBOLS[name][1]), name
    # the wide entries take the arguments of the k <= 32 ones
    for name in WIDE:
        assert nat.SYMBOLS[name] == nat.SYMBOLS[name.replace("_wide", "")], name


def test_workspace_is_the_cell_scratch_and_the_checks(nat):
    lib = nat.load()
    nb = C.c_size_t()
    for B, N, Cd, k in ((1, 1, 1, 1), (2, 1000, 3, 33), (3, 4096, 2, 256), (1, 300, 3, 128)):
        assert lib.egnn_radius_select_wide_workspace_bytes(B, N, Cd, k, C.byref(nb)) == 0
        assert nb.value == cell_bytes(B, N, Cd, 8)
        if k <= 32:
            nb2 = C.c_size_t()
            assert lib.egnn_radius_select_workspace_bytes(B, N, Cd, k, C.byref(nb2)) == 0 and nb2.value == nb.value
    for args, code in (((1, 1000, 3, 257), -3), ((1, 1000, 4, 64), -3), ((1, 100, 3, 101), -2), ((1, 100, 3, 0), -2),
                       ((0, 100, 3, 40), -2), ((1, 100, 0, 40), -2)):
        assert lib.egnn_radius_select_wide_workspace_bytes(*args, C.byref(nb)) == code, args
    assert lib.egnn_radius_select_wide_workspace_bytes(1, 100, 3, 40, None) == -1
    # the k <= 32 entries keep rejecting k = 33
    assert lib.egnn_radius_select_workspace_bytes(1, 100, 3, 33, C.byref(nb)) == -3

    # the select itself: every check runs before a launch, so host pointers are enough for the failing calls
    B, N, Cd, k = 1, 100, 3, 64
    assert lib.egnn_radius_select_wide_workspace_bytes(B, N, Cd, k, C.byref(nb)) == 0
    ws = (C.c_uint8 * (nb.value + 512))()
    base = (C.addressof(ws) + 255) // 256 * 256
    dummy = C.c_void_p(base)
    ptr = C.c_void_p(base)

    def call(entry=lib.egnn_radius_select_wide, dtype=nat.DTYPE_F32, b=B, n=N, c=Cd, kk=k, coors=dummy, lat=None,
             out=dummy, w=ptr, nbytes=nb.value):
        return entry(dtype, b, n, c, kk, coors, None, lat, 1.0, out, None, w, nbytes, None)

    assert call(kk=257, n=300) == nat.ERR_UNSUPPORTED
    assert call(c=4) == nat.ERR_UNSUPPORTED
    assert call(kk=N + 1) == -2
    assert call(w=None) == -1
    assert call(coors=None) == -1
    assert call(out=None) == -1
    assert call(w=C.c_void_p(base + 16)) == -4
    assert call(nbytes=nb.value - 1) < 0 and call(nbytes=nb.value - 1) not in (-1, -2, -3, -4)
    assert call(dtype=nat.DTYPE_BF16) == nat.ERR_UNSUPPORTED
    tri = lib.egnn_radius_select_wide_triclinic
    assert call(tri) == -1                                 # no cell
    assert call(tri, c=1, lat=dummy) == -2 and call(tri, c=4, lat=dummy) == -2
    assert call(tri, kk=257, n=300, lat=dummy) == nat.ERR_UNSUPPORTED


def test_radius_neighbors_wide_rejects_misuse_before_launching():
    from egnn_pytorch_b200 import radius_neighbors_wide
    x = torch.zeros(2, 300, 3)
    for kw, msg in (
        (dict(k=0), r"k must be an int in \[1, min\(256, N\)\] = \[1, 256\]"),
        (dict(k=257), "k must be"),
        (dict(coors=torch.zeros(2, 10, 3), k=11), r"\[1, 10\]"),
        (dict(k=64.0), "k must be"),
        (dict(k=True), "k must be"),
        (dict(coors=torch.zeros(2, 300, 4)), "radius_neighbors_wide supports C <= 3"),
        (dict(coors=torch.zeros(2, 300, 3, dtype=torch.float16)), "float32 or float64"),
        (dict(cutoff=0.0), "cutoff must be"),
        (dict(cutoff=float("inf")), "cutoff must be"),
        (dict(mask=torch.ones(2, 299)), "mask must be a"),
        (dict(box=torch.ones(3), cell=torch.eye(3)), "either box= or cell="),
        (dict(box=torch.tensor([1.0, -1.0, 1.0])), "box lengths"),
        (dict(cell=torch.ones(3, 3)), "lower-triangular"),
    ):
        args = dict(coors=x, cutoff=1.0, k=40)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            radius_neighbors_wide(args.pop("coors"), args.pop("cutoff"), args.pop("k"), **args)


def test_flagged_layer_workspace_grows_by_the_cell_scratch_only_when_eligible(nat):
    """Every layer descriptor of the case table with k set to 40 and 256 (clipped at N): with EGNN_FLAG_CELL_SELECT_WIDE
    an eligible one grows by exactly the cell scratch over the same descriptor without the flag, which is not eligible
    (k > 32) and keeps its size; with an infinite radius the flag changes nothing."""
    lib = nat.load()
    seen = {True: 0, False: 0}
    for name, d0 in _layer_descs(nat):
        for k in (40, 256):
            if d0.k == 0 or k > d0.N:
                continue
            sizes = {}
            for flag in (0, nat.FLAG_CELL_SELECT_WIDE):
                for inf_r in (False, True):
                    d = nat.LayerDesc()
                    C.memmove(C.byref(d), C.byref(d0), C.sizeof(nat.LayerDesc))
                    d.k, d.flags = k, d0.flags | flag
                    d.valid_radius = float("inf") if inf_r else d0.valid_radius
                    nb = C.c_size_t()
                    rc = lib.egnn_layer_workspace_bytes(C.byref(d), C.byref(nb))
                    sizes[flag, inf_r] = (rc, nb.value)
            rc = {v[0] for v in sizes.values()}
            assert len(rc) == 1, (name, sizes)
            if rc != {0}:
                assert rc == {nat.ERR_UNSUPPORTED} and d0.dtype == nat.DTYPE_BF16, (name, sizes)
                continue
            base = sizes[0, False][1]
            assert sizes[0, True][1] == base and sizes[nat.FLAG_CELL_SELECT_WIDE, True][1] == base, (name, sizes)
            vr = d0.valid_radius if d0.dtype == nat.DTYPE_F64 else float(torch.tensor(d0.valid_radius, dtype=torch.float32))
            bad = nat.FLAG_ONLY_SPARSE | nat.FLAG_ADJ_BATCHED | nat.FLAG_EDGES_PER_SLOT
            el = 1 <= d0.C <= 3 and not (d0.flags & bad) and 0.0 < vr < 1e5
            seen[el] += 1
            grow = cell_bytes(d0.B, d0.N, d0.C, 8 if d0.dtype == nat.DTYPE_F64 else 4) if el else 0
            assert sizes[nat.FLAG_CELL_SELECT_WIDE, False][1] == base + grow, (name, k, sizes, grow)
    assert seen[True] > 10 and seen[False] > 10, seen


def test_flagged_backward_workspace_accepts_the_flag(nat):
    lib = nat.load()
    kw = dict(abi_version=nat.ABI_VERSION, dtype=nat.DTYPE_F32, B=1, N=5000, C=3, dim=16, edge_dim=0, label_dim=0,
              num_labels=0, m_dim=16, fourier=0, k=64, row_begin=0, row_end=0, reserved=0, clamp=0.0, valid_radius=1.0)
    fl = nat.FLAG_UPDATE_FEATS | nat.FLAG_UPDATE_COORS
    a, b = C.c_size_t(), C.c_size_t()
    assert lib.egnn_layer_backward_workspace_bytes(C.byref(nat.LayerDesc(flags=fl, **kw)), C.byref(a)) == 0
    assert lib.egnn_layer_backward_workspace_bytes(
        C.byref(nat.LayerDesc(flags=fl | nat.FLAG_CELL_SELECT_WIDE, **kw)), C.byref(b)) == 0
