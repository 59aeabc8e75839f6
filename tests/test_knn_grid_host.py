"""CPU checks of the kNN cell grid: the C-ABI entries agree with the header, their host checks return the documented
codes before anything launches, `knn_neighbors` rejects misuse, the module's select flags follow (k, N) only, a flagged
descriptor grows by exactly the kNN grid's scratch when eligible, and the numpy reference select that the GPU tests
compare against equals a brute-force ranking."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

from test_radius_select_host import _layer_descs, cell_bytes
from util import nat  # noqa: F401  (module-scoped fixture)

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ("egnn_knn_grid_select_workspace_bytes", "egnn_knn_grid_select", "egnn_knn_grid_select_triclinic")
KGRID_BYTES = 176          # sizeof(KGrid): per-graph grid parameters


def knn_bytes(B, N, Cd, coord_bytes):
    r = lambda v: (v + 255) // 256 * 256                # noqa: E731
    return cell_bytes(B, N, Cd, coord_bytes) + r(B * KGRID_BYTES) + r(4 * B * N) + r(4)


def test_symbols_match_the_header(nat):
    header = open(os.path.join(REPO, "include", "egnn_b200.h")).read()
    assert re.search(r"#define EGNN_FLAG_KNN_GRID \(1u << 12\)", header)
    assert nat.FLAG_KNN_GRID == 1 << 12
    for name in ENTRIES:
        assert name in nat.SYMBOLS
        m = re.search(r"\bint " + name + r"\(([^)]*)\);", header)
        assert m, name
        assert len(m.group(1).split(",")) == len(nat.SYMBOLS[name][1]), name
    # the radius entries' arguments: valid_radius in place of r2, ok bytes in place of counts
    assert nat.SYMBOLS["egnn_knn_grid_select"] == nat.SYMBOLS["egnn_radius_select_wide"]
    assert nat.SYMBOLS["egnn_knn_grid_select_triclinic"] == nat.SYMBOLS["egnn_radius_select_wide_triclinic"]


def test_workspace_formula_and_host_checks(nat):
    lib = nat.load()
    nb = C.c_size_t()
    for B, N, Cd, k in ((1, 1, 1, 1), (2, 1000, 3, 33), (3, 4096, 2, 256), (8, 4096, 3, 32)):
        assert lib.egnn_knn_grid_select_workspace_bytes(B, N, Cd, k, C.byref(nb)) == 0
        assert nb.value == knn_bytes(B, N, Cd, 8)
    for args, code in (((1, 1000, 3, 257), -3), ((1, 1000, 4, 8), -3), ((1, 100, 3, 101), -2), ((1, 100, 3, 0), -2),
                       ((0, 100, 3, 8), -2), ((1, 100, 0, 8), -2)):
        assert lib.egnn_knn_grid_select_workspace_bytes(*args, C.byref(nb)) == code, args
    assert lib.egnn_knn_grid_select_workspace_bytes(1, 100, 3, 8, None) == -1

    B, N, Cd, k = 1, 100, 3, 64
    assert lib.egnn_knn_grid_select_workspace_bytes(B, N, Cd, k, C.byref(nb)) == 0
    ws = (C.c_uint8 * (nb.value + 512))()
    base = (C.addressof(ws) + 255) // 256 * 256
    ptr = C.c_void_p(base)

    def call(entry=lib.egnn_knn_grid_select, dtype=nat.DTYPE_F32, b=B, n=N, c=Cd, kk=k, coors=ptr, lat=None, out=ptr,
             w=ptr, nbytes=nb.value):
        return entry(dtype, b, n, c, kk, coors, None, lat, math.inf, out, None, w, nbytes, None)

    assert call(kk=257, n=300) == nat.ERR_UNSUPPORTED
    assert call(c=4) == nat.ERR_UNSUPPORTED
    assert call(kk=N + 1) == -2 and call(kk=0) == -2
    assert call(w=None) == -1 and call(coors=None) == -1 and call(out=None) == -1
    assert call(w=C.c_void_p(base + 16)) == -4
    assert call(dtype=nat.DTYPE_F64, nbytes=nb.value - 1) == -5          # sized for float64 coordinates
    assert call(dtype=nat.DTYPE_BF16) == nat.ERR_UNSUPPORTED
    tri = lib.egnn_knn_grid_select_triclinic
    assert call(tri) == -1                                 # no cell
    assert call(tri, c=1, lat=ptr) == -2 and call(tri, c=4, lat=ptr) == -2
    assert call(tri, kk=257, n=300, lat=ptr) == nat.ERR_UNSUPPORTED


def test_knn_neighbors_rejects_misuse_before_launching():
    from egnn_pytorch_b200 import knn_neighbors
    x = torch.zeros(2, 300, 3)
    for kw, msg in (
        (dict(k=0), r"k must be an int in \[1, min\(256, N\)\] = \[1, 256\]"),
        (dict(k=257), "k must be"),
        (dict(coors=torch.zeros(2, 10, 3), k=11), r"\[1, 10\]"),
        (dict(k=8.0), "k must be"),
        (dict(k=True), "k must be"),
        (dict(coors=torch.zeros(2, 300, 4)), "knn_neighbors supports C <= 3"),
        (dict(coors=torch.zeros(300, 3)), r"\[B, N, C\]"),
        (dict(coors=torch.zeros(2, 300, 3, dtype=torch.float16)), "float32 or float64"),
        (dict(mask=torch.ones(2, 299)), "mask must be a"),
        (dict(box=torch.ones(3), cell=torch.eye(3)), "either box= or cell="),
        (dict(box=torch.tensor([1.0, -1.0, 1.0])), "box lengths"),
        (dict(cell=torch.ones(3, 3)), "lower-triangular"),
    ):
        args = dict(coors=x, k=8)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            knn_neighbors(args.pop("coors"), args.pop("k"), **args)


def test_knn_neighbors_is_exported():
    import egnn_pytorch_b200 as pkg
    from egnn_pytorch_b200 import egnn
    assert pkg.knn_neighbors is egnn.knn_neighbors and "knn_neighbors" in egnn.__all__


@pytest.mark.parametrize("k", [1, 32, 33, 256])
@pytest.mark.parametrize("n", [300, 16384, 16385, 131072])
@pytest.mark.parametrize("row_scan", [False, True])
def test_module_select_flags_follow_k_and_n_only(nat, k, n, row_scan):
    """The layer asks for the kNN grid whenever it ranks its own lists, except where a k > 32 layer beyond the block
    sort's limit keeps its error; mask and valid_radius do not enter (the library decides from the descriptor and
    the call)."""
    from egnn_pytorch_b200 import egnn
    fl, sort_limited = egnn._select_flags(k, n, row_scan)
    assert sort_limited == (k > 32 and n > egnn.SELECT_SORT_MAX_N and not row_scan)
    assert bool(fl & nat.FLAG_CELL_SELECT_WIDE) == (k > 32)
    assert bool(fl & nat.FLAG_KNN_GRID) == (not sort_limited)


def test_flagged_layer_workspace_grows_by_the_knn_scratch_only_when_eligible(nat):
    """Every layer descriptor of the case table with k = 8, 32, 40 (clipped at N), with and without a finite radius:
    EGNN_FLAG_KNN_GRID adds exactly the kNN grid's scratch (which replaces the radius grid's, if any) to an eligible
    descriptor and nothing to any other; without the flag sizes are unchanged."""
    lib = nat.load()
    seen = {True: 0, False: 0}
    for name, d0 in _layer_descs(nat):
        for k in (8, 32, 40):
            if d0.k == 0 or k > d0.N:
                continue
            for inf_r in (False, True):
                sizes = {}
                for extra in (0, nat.FLAG_KNN_GRID):
                    d = nat.LayerDesc()
                    C.memmove(C.byref(d), C.byref(d0), C.sizeof(nat.LayerDesc))
                    d.k = k
                    d.flags = d0.flags | extra | (nat.FLAG_CELL_SELECT_WIDE if k > 32 else 0)
                    d.valid_radius = math.inf if inf_r else d0.valid_radius
                    nb = C.c_size_t()
                    sizes[extra] = (lib.egnn_layer_workspace_bytes(C.byref(d), C.byref(nb)), nb.value)
                if sizes[0][0] != 0:
                    assert sizes[0][0] == sizes[nat.FLAG_KNN_GRID][0] == nat.ERR_UNSUPPORTED, (name, sizes)
                    continue
                bad = nat.FLAG_ONLY_SPARSE | nat.FLAG_ADJ_BATCHED | nat.FLAG_EDGES_PER_SLOT
                el = 1 <= d0.C <= 3 and not (d0.flags & bad)
                seen[el] += 1
                cb = 8 if d0.dtype == nat.DTYPE_F64 else 4
                vr = d0.valid_radius if cb == 8 else float(torch.tensor(d0.valid_radius, dtype=torch.float32))
                radius_el = el and not inf_r and 0.0 < vr < 1e5
                base = sizes[0][1] - (cell_bytes(d0.B, d0.N, d0.C, cb) if radius_el else 0)
                want = base + (knn_bytes(d0.B, d0.N, d0.C, cb) if el else (sizes[0][1] - base))
                assert sizes[nat.FLAG_KNN_GRID][1] == want, (name, k, inf_r, sizes)
    assert seen[True] > 10 and seen[False] > 10, seen


def test_backward_workspace_accepts_the_flag(nat):
    lib = nat.load()
    kw = dict(abi_version=nat.ABI_VERSION, dtype=nat.DTYPE_F32, B=1, N=5000, C=3, dim=16, edge_dim=0, label_dim=0,
              num_labels=0, m_dim=16, fourier=0, k=32, row_begin=0, row_end=0, reserved=0, clamp=0.0,
              valid_radius=math.inf)
    fl = nat.FLAG_UPDATE_FEATS | nat.FLAG_UPDATE_COORS
    a, b = C.c_size_t(), C.c_size_t()
    assert lib.egnn_layer_backward_workspace_bytes(C.byref(nat.LayerDesc(flags=fl, **kw)), C.byref(a)) == 0
    assert lib.egnn_layer_backward_workspace_bytes(C.byref(nat.LayerDesc(flags=fl | nat.FLAG_KNN_GRID, **kw)),
                                                   C.byref(b)) == 0


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_numpy_reference_select_equals_brute_force(dtype):
    """KS.ref_select (the exact restatement of the all-pairs select the GPU tests use beyond N = 16384) against a
    per-row Python ranking: (rank, j) order, 1e5 for padded pairs, NaN last by index, ok = rank <= valid_radius."""
    import test_gpu_knn_select as KS
    rng = np.random.default_rng(0)
    for c in (1, 2, 3):
        x = rng.integers(0, 6, size=(2, 60, c)).astype(dtype) / dtype(4)      # many exact ties
        x[0, 3, 0] = np.nan
        x[1, 7, c - 1] = np.inf
        mask = rng.random((2, 60)) < 0.8
        for k in (1, 7, 60):
            idx, ok = KS.ref_select(x, k, 0.5, mask=mask)
            T = dtype
            for b in range(2):
                for i in range(60):
                    keys = []
                    for j in range(60):
                        with np.errstate(invalid="ignore", over="ignore"):
                            d = T(0)
                            for a in range(c):
                                r = T(x[b, i, a] - x[b, j, a])
                                d = T(d + T(r * r))
                        if not (mask[b, i] and mask[b, j]):
                            d = T(1e5)
                        keys.append((1, 0.0, j) if d != d else (0, float(d), j))
                    keys.sort()
                    want = [kk[2] for kk in keys[:k]]
                    assert idx[b, i].tolist() == want, (c, k, b, i)
                    assert ok[b, i].tolist() == [kk[0] == 0 and kk[1] <= T(0.5) for kk in keys[:k]], (c, k, b, i)
