"""Packed batches on the cell grids, without a GPU: the C entries' workspace formulas and argument checks, and the
Python routing between egnn_knn_select_packed and the grid entries."""
import ctypes as C
import math
import os
import re

import pytest
import torch

from util import nat  # noqa: F401  (module-scoped fixture)

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRIDS = ("radius", "knn_grid")


def _r(x):
    return (x + 255) // 256 * 256


def expected_ws(grid, G, T, Cd):
    """tile0 [G+1] and the validity flag, then the grid's scratch for T nodes in 4 T buckets (float64 coordinates):
    bucket counts and ends, coordinates in cell order, node indices; the kNN grid adds G KGrids (176 bytes), its
    full-scan rows and their count."""
    head = _r(4 * (G + 2))
    cell = _r(16 * T) * 2 + _r(8 * Cd * T) + _r(4 * T)
    return head + cell + (_r(176 * G) + _r(4 * T) + _r(4) if grid == "knn_grid" else 0)


def test_symbols_match_the_header(nat):
    header = open(os.path.join(REPO, "include", "egnn_b200.h")).read()
    for g in GRIDS:
        for name in (f"egnn_{g}_select_packed", f"egnn_{g}_select_packed_triclinic",
                     f"egnn_{g}_select_packed_workspace_bytes"):
            assert name in nat.SYMBOLS
            m = re.search(r"\bint " + name + r"\(([^)]*)\);", header)
            assert m, name
            assert len(m.group(1).split(",")) == len(nat.SYMBOLS[name][1]), name


@pytest.mark.parametrize("grid", GRIDS)
def test_workspace_formula_and_host_checks(nat, grid):
    lib = nat.load()
    ws_fn = getattr(lib, f"egnn_{grid}_select_packed_workspace_bytes")
    nb = C.c_size_t()
    for G, T, Cd, k in ((1, 1, 1, 1), (2, 1000, 3, 33), (64, 4096, 3, 32), (1000, 20000, 2, 256)):
        assert ws_fn(G, T, Cd, k, C.byref(nb)) == 0
        assert nb.value == expected_ws(grid, G, T, Cd), (G, T, Cd, k)
    # C > 3 runs the segmented select alone: its scratch only
    assert ws_fn(3, 100, 5, 8, C.byref(nb)) == 0 and nb.value == _r(4 * 5)
    for args, code in (((1, 100, 3, 257), -3), ((1, 100, 9, 8), -2), ((1, 100, 0, 8), -2), ((1, 100, 3, 0), -2),
                       ((0, 100, 3, 8), -2), ((1, 0, 3, 8), -2), ((1, 1 << 29, 3, 8), -2)):
        assert ws_fn(*args, C.byref(nb)) == code, args      # 4 T bucket offsets must stay an int
    assert ws_fn(1, (1 << 29) - 1, 3, 8, C.byref(nb)) == 0
    assert ws_fn(2, 100, 3, 8, None) == -1
    # the existing entry's scratch is unchanged
    assert lib.egnn_knn_select_packed_workspace_bytes(2, 100, 3, 8, C.byref(nb)) == 0 and nb.value == 256

    G, T, Cd, k = 2, 100, 3, 8
    assert ws_fn(G, T, Cd, k, C.byref(nb)) == 0
    ws = (C.c_uint8 * (nb.value + 512))()
    base = (C.addressof(ws) + 255) // 256 * 256
    p = C.c_void_p(base)
    plain = getattr(lib, f"egnn_{grid}_select_packed")
    tri = getattr(lib, f"egnn_{grid}_select_packed_triclinic")

    def call(entry=plain, dtype=nat.DTYPE_F32, g=G, t=T, c=Cd, kk=k, ptr=p, coors=p, lat=None, out=p, ok=p, w=p,
             nbytes=nb.value):
        return entry(dtype, g, t, c, kk, 50, ptr, coors, None, lat, 1.0, out, ok, w, nbytes, None)

    assert call(ptr=None) == -1 and call(coors=None) == -1 and call(out=None) == -1 and call(w=None) == -1
    if grid == "radius":
        assert call(ok=None) == -1                          # the kept slots are the ok = 1 slots
    assert call(entry=tri, lat=None) == -1                  # a cell is required
    assert call(entry=tri, lat=p, c=4) == -2                # a cell is 2-D or 3-D
    assert call(kk=257) == -3 and call(dtype=nat.DTYPE_BF16) == -3
    assert call(g=0) == -2 and call(c=9) == -2 and call(t=1 << 29) == -2
    assert call(w=C.c_void_p(base + 16)) == -4
    assert call(nbytes=nb.value - 1) == -5


def test_entry_routing():
    from egnn_pytorch_b200.egnn import _PACKED_GRID_MAX_T, _packed_entry
    assert _packed_entry("knn", 1000, 3, 32) == "egnn_knn_grid_select_packed"
    assert _packed_entry("radius", 1000, 1, 256) == "egnn_radius_select_packed"
    # the existing entry where a grid cannot serve the call, and without a mode
    assert _packed_entry(None, 1000, 3, 32) == "egnn_knn_select_packed"
    assert _packed_entry("knn", 1000, 4, 32) == "egnn_knn_select_packed"
    assert _packed_entry("radius", 1000, 8, 32) == "egnn_knn_select_packed"
    assert _packed_entry("knn", 1000, 3, 257) == "egnn_knn_select_packed"
    assert _packed_entry("radius", _PACKED_GRID_MAX_T + 1, 3, 8) == "egnn_knn_select_packed"


@pytest.mark.parametrize("r2, dtype, want", [(2.25, torch.float32, True), (99999.0, torch.float64, True),
                                             (1e5, torch.float64, False), (99999.999, torch.float32, False),
                                             (math.inf, torch.float32, False), (1e-50, torch.float32, False),
                                             (1e-50, torch.float64, True)])
def test_radius_mode_needs_a_radius_the_grid_serves(r2, dtype, want):
    from egnn_pytorch_b200.egnn import _in_cell_radius
    assert _in_cell_radius(r2, dtype) is want


class _Recorder(Exception):
    pass


def _record_select(monkeypatch):
    """Replace _packed_select by a recorder that raises once it has seen its arguments."""
    from egnn_pytorch_b200 import egnn as E
    seen = []

    def fake(x, ptr, k, m, lattice, triclinic, valid_radius, mode=None, max_n=None):
        seen.append(dict(k=k, mask=m is not None, vr=valid_radius, mode=mode, max_n=max_n,
                         entry=E._packed_entry(mode, x.shape[1], x.shape[2], k)))
        raise _Recorder()
    monkeypatch.setattr(E, "_packed_select", fake)
    monkeypatch.setattr(E, "_compute_device", lambda t: torch.device("cpu"))
    monkeypatch.setattr(torch.cuda, "current_device", lambda: None)
    monkeypatch.setattr(E, "_NULL_CTX", __import__("contextlib").nullcontext())
    return seen


@pytest.mark.parametrize("vr, mask_on, c, k, want", [
    (math.inf, False, 3, 8, ("knn", "egnn_knn_grid_select_packed")),
    (math.inf, True, 3, 8, ("knn", "egnn_knn_grid_select_packed")),
    (2.0, True, 3, 8, ("radius", "egnn_radius_select_packed")),
    (2.0, False, 3, 8, ("knn", "egnn_knn_grid_select_packed")),       # no mask: every slot is kept
    (2e5, True, 3, 8, ("knn", "egnn_knn_grid_select_packed")),        # radius above the grid's
    (2.0, True, 5, 8, ("radius", "egnn_knn_select_packed")),          # C > 3
    (math.inf, False, 3, 300, ("knn", "egnn_knn_select_packed"))])    # k > 256
def test_layer_routing(monkeypatch, vr, mask_on, c, k, want):
    from egnn_pytorch_b200 import EGNN
    seen = _record_select(monkeypatch)
    lay = EGNN(dim=8, m_dim=8, num_nearest_neighbors=k, valid_radius=vr)
    t = 400
    ptr = torch.tensor([0, 100, t])
    mask = torch.ones(1, t, dtype=torch.bool) if mask_on else None
    with pytest.raises(_Recorder):
        lay(torch.randn(1, t, 8), torch.randn(1, t, c), mask=mask, ptr=ptr)
    assert (seen[0]["mode"], seen[0]["entry"]) == want
    assert seen[0]["max_n"] == 300 and seen[0]["k"] == min(k, 300)


@pytest.mark.parametrize("builder, cutoff, mask_on, want_mode, want_mask", [
    ("knn", None, True, "knn", True), ("knn", None, False, "knn", False),
    ("radius", 1.5, True, "radius", True), ("wide", 1.5, False, "radius", False),
    ("radius", 400.0, True, "radius", False)])     # cutoff^2 >= 1e5: masked nodes are made NaN instead
def test_builder_routing(monkeypatch, builder, cutoff, mask_on, want_mode, want_mask):
    from egnn_pytorch_b200 import knn_neighbors, radius_neighbors, radius_neighbors_wide
    seen = _record_select(monkeypatch)
    t = 300
    ptr = torch.tensor([0, 120, t])
    x = torch.randn(1, t, 3)
    mask = torch.ones(1, t, dtype=torch.bool) if mask_on else None
    call = {"knn": lambda: knn_neighbors(x, 16, mask=mask, ptr=ptr),
            "radius": lambda: radius_neighbors(x, cutoff, 16, mask=mask, ptr=ptr),
            "wide": lambda: radius_neighbors_wide(x, cutoff, 16, mask=mask, ptr=ptr)}[builder]
    with pytest.raises(_Recorder):
        call()
    assert seen[0]["mode"] == want_mode and seen[0]["mask"] == want_mask and seen[0]["max_n"] == 180
