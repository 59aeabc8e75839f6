"""CPU checks of packed batches (`ptr=`): the C-ABI entries of the segmented select agree with the header, their host
checks return the documented codes before anything launches, `ptr` is validated and every combination `ptr=` does not
take is rejected with a ValueError before anything launches, and the numpy segmented reference that the GPU tests
compare against equals a brute-force ranking of each graph, including graphs smaller than k, single nodes and empty
graphs."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

from test_gpu_knn_select import ref_select
from util import nat  # noqa: F401  (module-scoped fixture)

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ("egnn_knn_select_packed_workspace_bytes", "egnn_knn_select_packed", "egnn_knn_select_packed_triclinic")


# ------------------------------------------------------------------ the segmented reference


def ref_packed_select(x, ptr, k, vr, mask=None, box=None):
    """The segmented select's lists, restated: each graph's egnn_knn_select lists (ref_select on it alone, B = 1,
    N = n_g, k' = min(k, n_g)) with indices shifted by ptr[g], -1 / False past n_g.  x [T, C] float32 / float64, mask
    [T] bool, box [C] shared by every graph -> (idx [T, k] int64, ok [T, k] bool)."""
    t = x.shape[0]
    idx = np.full((t, k), -1, np.int64)
    ok = np.zeros((t, k), bool)
    for g in range(len(ptr) - 1):
        lo, hi = int(ptr[g]), int(ptr[g + 1])
        if hi == lo:
            continue
        kk = min(k, hi - lo)
        i, o = ref_select(x[None, lo:hi], kk, vr, mask=None if mask is None else mask[None, lo:hi],
                          box=None if box is None else np.asarray(box)[None])
        idx[lo:hi, :kk] = i[0] + lo
        ok[lo:hi, :kk] = o[0]
    return idx, ok


def brute_packed_select(x, ptr, k, vr, mask=None):
    """One node at a time in Python scalars of x's type: rank every node of its graph (per axis r = x_i - x_j, d += r r;
    1e5 when either end is padded), order by (NaN last, rank, index), keep k."""
    T = x.dtype.type
    t = x.shape[0]
    idx = np.full((t, k), -1, np.int64)
    ok = np.zeros((t, k), bool)
    with np.errstate(invalid="ignore", over="ignore"):
        for g in range(len(ptr) - 1):
            lo, hi = int(ptr[g]), int(ptr[g + 1])
            for i in range(lo, hi):
                cand = []
                for j in range(lo, hi):
                    d = T(0)
                    for c in range(x.shape[1]):
                        r = T(x[i, c] - x[j, c])
                        d = T(d + T(r * r))
                    if mask is not None and not (mask[i] and mask[j]):
                        d = T(1e5)
                    cand.append((bool(np.isnan(d)), 0.0 if np.isnan(d) else float(d), j, d))
                cand.sort(key=lambda e: e[:3])
                for s, (_, _, j, d) in enumerate(cand[:k]):
                    idx[i, s] = j
                    ok[i, s] = bool(d <= T(vr))
    return idx, ok


PACKINGS = {
    "mixed": [0, 5, 5, 6, 20, 23],            # an empty graph, a single node, graphs above and below k
    "all_small": [0, 1, 3, 6],
    "empty_ends": [0, 0, 4, 4, 12, 12],
    "one_graph": [0, 9],
}


@pytest.mark.parametrize("packing", list(PACKINGS))
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("k", [1, 4, 8])
def test_segmented_reference_equals_brute_force(packing, dtype, k):
    ptr = np.array(PACKINGS[packing])
    t = int(ptr[-1])
    rs = np.random.RandomState(k + len(packing))
    x = rs.randint(-3, 4, size=(t, 3)).astype(dtype)          # integer coordinates: many ties
    x[t // 2 if t > 1 else 0, 1] = np.nan
    mask = rs.rand(t) > 0.25
    for m in (None, mask):
        for vr in (math.inf, 5.0):
            want = brute_packed_select(x, ptr, k, vr, m)
            got = ref_packed_select(x, ptr, k, vr, m)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (packing, m is None, vr)


def test_reference_marks_slots_past_a_small_graph_empty():
    x = np.arange(12, dtype=np.float64).reshape(4, 3)
    idx, ok = ref_packed_select(x, [0, 1, 1, 4], 3, math.inf)
    assert idx[0].tolist() == [0, -1, -1] and ok[0].tolist() == [True, False, False]
    assert idx[1].tolist() == [1, 2, 3] and idx[3].tolist() == [3, 2, 1]


# ------------------------------------------------------------------ the C ABI


def test_symbols_match_the_header(nat):
    header = open(os.path.join(REPO, "include", "egnn_b200.h")).read()
    for name in ENTRIES:
        assert name in nat.SYMBOLS
        m = re.search(r"\bint " + name + r"\(([^)]*)\);", header)
        assert m, name
        assert len(m.group(1).split(",")) == len(nat.SYMBOLS[name][1]), name
    assert nat.SYMBOLS["egnn_knn_select_packed"] == nat.SYMBOLS["egnn_knn_select_packed_triclinic"]
    assert "#define EGNN_ABI_VERSION 4 " in header and nat.ABI_VERSION == 4


def test_workspace_formula_and_host_checks(nat):
    lib = nat.load()
    nb = C.c_size_t()
    for G, T, Cd, k in ((1, 1, 1, 1), (2, 1000, 3, 33), (63, 4096, 8, 256), (64, 4096, 3, 32), (1000, 20000, 2, 16)):
        assert lib.egnn_knn_select_packed_workspace_bytes(G, T, Cd, k, C.byref(nb)) == 0
        assert nb.value == (4 * (G + 1) + 255) // 256 * 256           # the per-graph tile offsets, 256-byte rounded
    for args, code in (((1, 100, 3, 257), -3), ((1, 100, 9, 8), -2), ((1, 100, 0, 8), -2), ((1, 100, 3, 0), -2),
                       ((0, 100, 3, 8), -2), ((1, 0, 3, 8), -2), ((1, (1 << 30) + 1, 3, 8), -2)):
        assert lib.egnn_knn_select_packed_workspace_bytes(*args, C.byref(nb)) == code, args
    assert lib.egnn_knn_select_packed_workspace_bytes(2, 100, 3, 8, None) == -1
    # k above a graph's size is allowed: its slots past n_g are written empty
    assert lib.egnn_knn_select_packed_workspace_bytes(4, 10, 3, 200, C.byref(nb)) == 0

    G, T, Cd, k = 2, 100, 3, 8
    assert lib.egnn_knn_select_packed_workspace_bytes(G, T, Cd, k, C.byref(nb)) == 0
    ws = (C.c_uint8 * (nb.value + 512))()
    base = (C.addressof(ws) + 255) // 256 * 256
    p = C.c_void_p(base)

    def call(entry=lib.egnn_knn_select_packed, dtype=nat.DTYPE_F32, g=G, t=T, c=Cd, kk=k, ptr=p, coors=p, lat=None,
             out=p, w=p, nbytes=nb.value):
        return entry(dtype, g, t, c, kk, ptr, coors, None, lat, math.inf, out, None, w, nbytes, None)

    assert call(ptr=None) == -1 and call(coors=None) == -1 and call(out=None) == -1 and call(w=None) == -1
    assert call(entry=lib.egnn_knn_select_packed_triclinic, lat=None) == -1        # a cell is required
    assert call(entry=lib.egnn_knn_select_packed_triclinic, lat=p, c=4) == -2      # a cell is 2-D or 3-D
    assert call(kk=257) == -3 and call(dtype=nat.DTYPE_BF16) == -3
    assert call(g=0) == -2 and call(c=9) == -2
    assert call(w=C.c_void_p(base + 16)) == -4
    assert call(nbytes=nb.value - 1) == -5


# ------------------------------------------------------------------ Python checks, before anything launches


def _layer(**kw):
    from egnn_pytorch_b200 import EGNN
    return EGNN(dim=8, **kw).double()


def _inputs(t=10, c=3):
    return torch.randn(1, t, 8, dtype=torch.float64), torch.randn(1, t, c, dtype=torch.float64)


@pytest.mark.parametrize("ptr, msg", [
    (torch.tensor([0, 4, 10]).float(), "integer"),
    (torch.tensor([[0, 10]]), "1-D"),
    (torch.tensor([10]), "G \\+ 1 >= 2"),
    ([0, 10], "tensor"),
    (torch.tensor([1, 4, 10]), "start at 0"),
    (torch.tensor([0, 6, 4, 10]), "non-decreasing"),
    (torch.tensor([0, 4, 9]), "end at T = 10"),
    (torch.tensor([0, 4, 11]), "end at T = 10"),
])
def test_ptr_is_validated(ptr, msg):
    from egnn_pytorch_b200 import knn_neighbors
    feats, coors = _inputs()
    with pytest.raises(ValueError, match=msg):
        _layer(num_nearest_neighbors=4)(feats, coors, ptr=ptr)
    with pytest.raises(ValueError, match=msg):
        knn_neighbors(coors, 4, ptr=ptr)


def test_ptr_takes_one_batch_row():
    from egnn_pytorch_b200 import radius_neighbors
    with pytest.raises(ValueError, match="B=2"):
        _layer()(torch.randn(2, 5, 8, dtype=torch.float64), torch.randn(2, 5, 3, dtype=torch.float64),
                 ptr=torch.tensor([0, 5]))
    with pytest.raises(ValueError, match="B=2"):
        radius_neighbors(torch.randn(2, 5, 3), 1.0, 4, ptr=torch.tensor([0, 5]))


def test_ptr_check_is_cached_per_tensor_version(monkeypatch):
    from egnn_pytorch_b200 import egnn as E
    ptr = torch.tensor([0, 3, 10])
    assert E._check_ptr(ptr, 1, 10) == 7
    reads = []
    real = torch.Tensor.to
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **kw: reads.append(1) or real(self, *a, **kw))
    assert E._check_ptr(ptr, 1, 10) == 7 and not reads                # same object, same version: no host read
    ptr[1] = 4
    assert E._check_ptr(ptr, 1, 10) == 6 and reads                     # written in place: read again
    ptr[1] = 11
    with pytest.raises(ValueError, match="non-decreasing"):
        E._check_ptr(ptr, 1, 10)


@pytest.mark.parametrize("what, kw, msg", [
    ("neighbors", dict(neighbors=torch.zeros(1, 10, 2, dtype=torch.int32)), "neighbors="),
    ("adj_mat", dict(adj_mat=torch.ones(10, 10, dtype=torch.bool)), "adj_mat"),
    ("rows", dict(_rows=(0, 5)), "row range"),
    ("box_per_graph", dict(box=torch.ones(2, 3)), "per-graph boxes"),
    ("cell_per_graph", dict(cell=torch.eye(3).expand(2, 3, 3)), "per-graph cells"),
])
def test_layer_rejects_what_ptr_does_not_combine_with(what, kw, msg):
    feats, coors = _inputs()
    with pytest.raises(ValueError, match=msg):
        _layer(num_nearest_neighbors=4)(feats, coors, ptr=torch.tensor([0, 4, 10]), **kw)


def test_layer_rejects_dense_edges_and_only_sparse_with_ptr():
    feats, coors = _inputs()
    ptr = torch.tensor([0, 4, 10])
    with pytest.raises(ValueError, match="dense edges"):
        _layer(edge_dim=2)(feats, coors, torch.randn(1, 10, 10, 2, dtype=torch.float64), ptr=ptr)
    with pytest.raises(ValueError, match="only_sparse_neighbors"):
        _layer(num_nearest_neighbors=4, only_sparse_neighbors=True)(feats, coors, ptr=ptr)


def test_network_rejects_what_ptr_does_not_combine_with():
    from egnn_pytorch_b200 import EGNN_Network
    ptr = torch.tensor([0, 4, 10])
    tok, coors = torch.randint(0, 5, (1, 10)), torch.randn(1, 10, 3)
    net = EGNN_Network(depth=2, dim=8, num_tokens=5, num_adj_degrees=2, adj_dim=2)
    with pytest.raises(ValueError, match="adj_mat"):
        net(tok, coors, adj_mat=torch.ones(10, 10, dtype=torch.bool), ptr=ptr)
    net = EGNN_Network(depth=2, dim=8, num_tokens=5, global_linear_attn_every=1, global_linear_attn_dim_head=8)
    with pytest.raises(ValueError, match="global linear attention"):
        net(tok, coors, ptr=ptr)
    net = EGNN_Network(depth=2, dim=8, num_tokens=5, num_edge_tokens=3, edge_dim=2)
    with pytest.raises(ValueError, match="dense edges"):
        net(tok, coors, edges=torch.zeros(1, 10, 10, dtype=torch.long), ptr=ptr)
    with pytest.raises(ValueError, match="end at T"):
        EGNN_Network(depth=1, dim=8, num_tokens=5)(tok, coors, ptr=torch.tensor([0, 4, 9]))


def test_builders_check_k_against_their_limit_not_the_graph_sizes():
    from egnn_pytorch_b200 import knn_neighbors, radius_neighbors, radius_neighbors_wide
    coors, ptr = torch.randn(1, 10, 3), torch.tensor([0, 4, 10])
    with pytest.raises(ValueError, match=r"\[1, 256\]"):
        knn_neighbors(coors, 257, ptr=ptr)
    with pytest.raises(ValueError, match=r"\[1, 32\]"):
        radius_neighbors(coors, 1.0, 33, ptr=ptr)
    with pytest.raises(ValueError, match=r"\[1, 256\]"):
        radius_neighbors_wide(coors, 1.0, 0, ptr=ptr)
    with pytest.raises(ValueError, match="return_counts"):
        radius_neighbors(coors, 1.0, 4, ptr=ptr, return_counts=True)
    with pytest.raises(ValueError, match="per-graph boxes"):
        knn_neighbors(coors, 4, ptr=ptr, box=torch.ones(2, 3))
