"""Radius graphs with lists longer than 32 (csrc/radius_select.cu, radius_query_wide_kernel): `radius_neighbors_wide` /
egnn_radius_select_wide* and `valid_radius` layers with 32 < k <= 256 under EGNN_FLAG_CELL_SELECT_WIDE.

Reference: the all-pairs select.  The lists must equal its ok = 1 slots exactly and hold -1 elsewhere; the counts must
equal the number of in-radius ranks.  Ranks come from the exact restatements of the select's arithmetic in the coordinates'
type (`ranks` of test_gpu_knn_select.py without a lattice and under a box, `cell_ranks` of
test_gpu_lattice_tile_boundaries.py under a cell) or, up to N = 16384, from egnn_knn_select itself (its block sort).
The wide query keeps (rank, j) pairs in a shared-memory list of KP = next_pow2(k) entries and merges a queue of KP more
into it whenever the queue could not take another 32: the in-radius counts below put rows on both sides of k and of
several merges.

Inside a layer the two paths are switched with EGNN_B200_CELL_SELECT_MIN_N (0 = cell grid, huge = all pairs); forward
outputs must be bit-identical and gradients equal to the backward's atomics tolerance."""
import ctypes as C
import math
import time

import numpy as np
import pytest
import torch

import test_gpu_knn_select as KS
import test_gpu_radius_select as RS
from test_gpu_lattice_tile_boundaries import cell_ranks

pytestmark = pytest.mark.gpu

DEV = "cuda"
NEVER = RS.NEVER
WIDE_K = (33, 64, 65, 128, 200, 256)


@pytest.fixture(autouse=True)
def _time_and_peak_memory(request):
    """Prints each test's run time and peak device memory (visible with -s)."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n{request.node.name}: {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


@pytest.fixture(scope="module")
def lib():
    from egnn_pytorch_b200 import _native
    return _native.load()


def exact(x, k, r2, mask=None, box=None, cell=None, chunk=128):
    """-> (lists [B, N, k] with -1 in the slots the select leaves empty, counts [B, N]) of the all-pairs select."""
    T = x.dtype.type
    b, n, _ = x.shape
    lists, counts = [], []
    for s in range(0, n, chunk):
        rows = np.arange(s, min(n, s + chunk))
        if cell is not None:
            d = cell_ranks(x, rows, cell, mask)
        else:
            d = KS.ranks(x, rows, mask, None, box)
        inr = d <= T(r2)                                  # False for NaN
        o = np.argsort(d, axis=-1, kind="stable")[..., :k]
        ok = np.take_along_axis(inr, o, axis=-1)
        if o.shape[-1] < k:
            o = np.concatenate([o, np.zeros(o.shape[:-1] + (k - o.shape[-1],), o.dtype)], -1)
            ok = np.concatenate([ok, np.zeros(ok.shape[:-1] + (k - ok.shape[-1],), bool)], -1)
        lists.append(np.where(ok, o, -1))
        counts.append(inr.sum(-1))
    return np.concatenate(lists, 1).astype(np.int32), np.concatenate(counts, 1).astype(np.int32)


def wide(x, cutoff, k, **kw):
    from egnn_pytorch_b200 import radius_neighbors_wide
    got, cnt = radius_neighbors_wide(x, cutoff, k, return_counts=True, **kw)
    return got.cpu().numpy(), cnt.cpu().numpy()


def check(x, cutoff, k, what, mask=None, box=None, cell=None):
    """radius_neighbors_wide against `exact`, on numpy coordinates x in their own type -> counts."""
    tt = torch.float64 if x.dtype == np.float64 else torch.float32
    kw = {}
    if mask is not None:
        kw["mask"] = torch.from_numpy(np.asarray(mask, bool)).to(DEV)
    if box is not None:
        kw["box"] = torch.from_numpy(np.asarray(box, np.float64)).to(DEV, tt)
    if cell is not None:
        kw["cell"] = torch.from_numpy(np.asarray(cell, np.float64)).to(DEV, tt)
    got, cnt = wide(torch.from_numpy(x).to(DEV), cutoff, k, **kw)
    want, want_cnt = exact(x, k, cutoff * cutoff, mask, None if box is None else np.broadcast_to(
        np.asarray(box, x.dtype), (x.shape[0], x.shape[2])), None if cell is None else np.broadcast_to(
        np.asarray(cell, x.dtype), (x.shape[0], x.shape[2], x.shape[2])))
    bad = (got != want).any(-1)
    if bad.any():
        g, i = np.argwhere(bad)[0]
        raise AssertionError(f"{what}: {int(bad.sum())} rows differ, first ({g}, {i}): {got[g, i].tolist()} vs "
                             f"{want[g, i].tolist()}")
    assert np.array_equal(cnt, want_cnt), f"{what}: counts differ in {int((cnt != want_cnt).sum())} rows"
    return cnt


# ----------------------------------------------------------------------------- 1. in-radius counts around k


def star_graphs(k, dtype, rs):
    """One graph per count m in (k-1, k, k+1, 2k, 2k+1, 4k+37): a centre node with exactly m nodes within distance 1
    (itself included) and the others between 1.02 and 1.9, in random index order -> (x, {graph: (centre, m)})."""
    ms = (k - 1, k, k + 1, 2 * k, 2 * k + 1, 4 * k + 37)
    n = 4 * k + 100
    xs, centres = [], {}
    for g, m in enumerate(ms):
        u = rs.normal(size=(n, 3))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        rad = np.concatenate([[0.0], rs.uniform(0.05, 0.98, m - 1), rs.uniform(1.02, 1.9, n - m)])
        perm = rs.permutation(n)
        xs.append((u * rad[:, None])[perm])
        centres[g] = (int(np.argsort(perm)[0]), m)
    return np.stack(xs).astype(dtype), centres


@pytest.mark.parametrize("k", WIDE_K)
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["fp32", "fp64"])
def test_counts_around_k_and_the_merge_boundaries(dtype, k):
    rs = np.random.RandomState(k)
    x, centres = star_graphs(k, dtype, rs)
    cnt = check(x, 1.0, k, f"stars {dtype.__name__} k={k}")
    for g, (i, m) in centres.items():
        assert cnt[g, i] == m, (g, i, cnt[g, i], m)
    # a random cloud with a mask at about k / 2, k and 3k in-radius nodes per row
    for mean in (k // 2, k, 3 * k):
        side = (1500 * (4.0 / 3.0) * math.pi / mean) ** (1.0 / 3.0)
        x = (rs.uniform(size=(2, 1500, 3)) * side).astype(dtype)
        mask = rs.uniform(size=(2, 1500)) < 0.9
        cnt = check(x, 1.0, k, f"cloud {dtype.__name__} k={k} mean={mean}", mask=mask)
        if mean >= k:
            assert (cnt[mask] > k).any() and (cnt[mask] < k).any()


# ----------------------------------------------------------------------------- 2. ties, duplicates, lattices, non-finite


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["fp32", "fp64"])
def test_ties_duplicates_and_lattices(dtype):
    rs = np.random.RandomState(11)
    # duplicate points: whole groups at one identical distance, ties to the lower index
    base = rs.randint(0, 4, (2, 60, 3))
    x = base[:, rs.randint(0, 60, 900)].astype(dtype)
    for k in (33, 64, 128, 256):
        check(x, 1.5, k, f"duplicates k={k}")
    # more than k nodes at one distance from a node: every other node on one of the six unit axis points around node 0,
    # exactly at the cutoff
    y = np.zeros((1, 700, 3))
    y[0, 1:] = np.concatenate([np.eye(3), -np.eye(3)])[rs.randint(0, 6, 699)]
    check(y.astype(dtype), 1.0, 256, "one distance")
    # integer lattices: many pairs exactly at the cutoff and on cell faces (exact in both types)
    ax = np.arange(-5, 6, dtype=np.float64)
    lat = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(1, -1, 3)
    lat = lat[:, rs.permutation(lat.shape[1])].astype(dtype)
    lm = rs.uniform(size=lat.shape[:2]) < 0.9
    for r2, k in ((2.0, 33), (4.0, 64), (5.0, 65), (8.0, 128), (9.0, 200), (12.0, 256)):
        check(lat, math.sqrt(r2), k, f"lattice r2={r2} k={k}", mask=lm)
    for c in (1, 2):
        check(np.ascontiguousarray(lat[..., :c]), 3.0, 40 if c == 1 else 64, f"lattice C={c}", mask=lm)


@pytest.mark.parametrize("c", [1, 2, 3])
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["fp32", "fp64"])
def test_dimensions_batches_masks_and_non_finite_nodes(dtype, c):
    rs = np.random.RandomState(20 + c)
    n = 2000
    side = (n * {1: 2.0, 2: math.pi, 3: 4.0 / 3.0 * math.pi}[c] / 90.0) ** (1.0 / c)
    x = (rs.uniform(size=(3, n, c)) * side).astype(dtype)
    x[0, 5, 0] = np.nan
    x[1, 50, c - 1] = np.inf
    x[2, 150, 0] = -np.inf
    mask = rs.uniform(size=(3, n)) < 0.85
    for k in (33, 128, 256):
        for m in (None, mask):
            cnt = check(x, 1.0, k, f"C={c} k={k} mask={m is not None}", mask=m)
            assert cnt[0, 5] == 0 and cnt[1, 50] == 0 and cnt[2, 150] == 0


# ----------------------------------------------------------------------------- 3. periodic boxes and triclinic cells


BOXES = {
    # name: (C, box [C] or [B, C], cutoff, N) -- 1, 2 and 3 cells per axis, mixed 0 / inf / finite axes, per graph
    "one_cell": (3, [1.5, 1.5, 1.5], 1.0, 300),
    "two_cells": (3, [2.5, 2.5, 2.5], 1.0, 900),
    "three_cells": (3, [3.5, 3.5, 3.5], 1.0, 1500),
    "mixed_axes": (3, [3.0, 0.0, float("inf")], 1.0, 1200),
    "per_graph": (3, [[3.0, 3.5, 4.0], [2.5, 0.0, 3.3], [float("inf"), 3.1, 1.5]], 1.0, 1200),
    "c1": (1, [9.0], 1.0, 1200),
    "c2_mixed": (2, [[4.0, float("inf")], [2.2, 3.0], [0.0, 5.0]], 1.0, 1500),
}


@pytest.mark.parametrize("name", sorted(BOXES))
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["fp32", "fp64"])
def test_periodic_boxes(dtype, name):
    c, box, cut, n = BOXES[name]
    rs = np.random.RandomState(sum(map(ord, name)))
    b = 3
    boxa = np.broadcast_to(np.asarray(box, np.float64), (b, c))
    per = (boxa > 0) & np.isfinite(boxa)
    span = np.where(per, boxa, 4.0)
    x = (rs.uniform(size=(b, n, c)) * span[:, None, :]).astype(dtype)
    x = np.where(per[:, None, :] & (x >= boxa[:, None, :].astype(dtype)), dtype(0), x)      # keep [0, L)
    mask = rs.uniform(size=(b, n)) < 0.9
    for k in (33, 100, 256):
        check(x, cut, k, f"{name} k={k}", mask=mask, box=np.asarray(boxa, dtype))


def tilted_cell(rs, Ls, t):
    A = np.diag(np.asarray(Ls, np.float64))
    for r in range(1, len(Ls)):
        for q in range(r):
            A[r, q] = rs.uniform(-t, t) * A[q, q]
    return A


CELLS = {
    # name: (cell(rs) -> [C, C] or [B, C, C], N)
    "tilt": (lambda rs: tilted_cell(rs, [3.0, 3.2, 3.5], 0.5), 1500),
    "tilt095": (lambda rs: np.array([[3.0, 0, 0], [0.4, 3.2, 0], [0.95 * 3.0, -0.5, 3.5]]), 1500),
    "per_graph": (lambda rs: np.stack([tilted_cell(rs, rs.uniform(2.2, 3.6, 3), 0.5) for _ in range(3)]), 1200),
    "small": (lambda rs: tilted_cell(rs, [1.6, 1.7, 2.6], 0.3), 500),          # one and two cells per axis
    "hex_slab": (lambda rs: np.array([[3.0, 0, 0], [1.5, 3.0 * math.sqrt(3) / 2, 0], [0, 0, np.inf]]), 1200),
    "c2": (lambda rs: tilted_cell(rs, [3.0, 2.8], 0.5), 1200),
}
GRID = 2.0 ** -8


@pytest.mark.parametrize("name", sorted(CELLS))
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["fp32", "fp64"])
def test_triclinic_cells(dtype, name):
    """Coordinates and cells on a dyadic grid (fp64) or rounded to fp32, so that cell_ranks restates the wrap exactly."""
    make, n = CELLS[name]
    rs = np.random.RandomState(sum(map(ord, name)) + 7)
    b = 3
    cell = make(rs)
    cell = np.broadcast_to(cell, (b,) + cell.shape[-2:]).copy()
    c = cell.shape[-1]
    snap = (lambda a: np.where(np.isfinite(a), np.round(a / GRID) * GRID, a)) if dtype == np.float64 else \
        (lambda a: a.astype(np.float32).astype(np.float64))
    cell = snap(cell)
    diag = np.diagonal(cell, axis1=1, axis2=2)
    per = np.isfinite(diag) & (diag > 0)
    Af = np.where(np.isfinite(cell), cell, 0.0) + np.where(per, 0.0, 1.0)[:, :, None] * np.eye(c)
    s = rs.uniform(0, 1, (b, n, c)) * np.where(per, 1.0, 4.0)[:, None, :] + rs.randint(-2, 3, (b, n, c)) * per[:, None]
    x = snap(np.einsum("bnk,bkd->bnd", s, Af)).astype(dtype)
    mask = rs.uniform(size=(b, n)) < 0.9
    for k in (33, 100, 256):
        check(x, 1.0, k, f"{name} k={k}", mask=mask, cell=cell.astype(dtype))


# ----------------------------------------------------------------------------- 4. the library's own select


@pytest.mark.parametrize("n", [4096, 16384])
def test_equals_egnn_knn_select(lib, n):
    """Against egnn_knn_select's block sort (k > 32) at its largest N."""
    for dtype, k in ((torch.float32, 64), (torch.float64, 128)):
        x, mask, _ = RS.cloud(2, n, mean_count=1.3 * k, seed=n + k, dtype=dtype)
        from egnn_pytorch_b200 import radius_neighbors_wide
        got, cnt = radius_neighbors_wide(x, 1.0, k, mask=mask, return_counts=True)
        want, _ = RS.expected_from_all_pairs(lib, x, mask, k, 1.0) if n <= 4096 else (None, None)
        if want is None:                                  # N = 16384: no full ranking for the counts (N^2 memory)
            idx, ok = RS.knn_select(lib, x, mask, k, 1.0)
            want = torch.where(ok, idx, torch.full_like(idx, -1))
            assert torch.equal((got >= 0).sum(-1, dtype=torch.int32), cnt.clamp(max=k))
        assert torch.equal(got, want), f"{dtype} N={n} k={k}: {int((got != want).any(-1).sum())} rows differ"
        assert bool((cnt > k).any()) and bool(((cnt < k) & mask).any())


def c_call(lib, x, mask, k, r2, entry="egnn_radius_select_wide", fill=None):
    b, n, c = x.shape
    nb = C.c_size_t()
    assert getattr(lib, entry + "_workspace_bytes")(b, n, c, k, C.byref(nb)) == 0
    ws = torch.empty(nb.value, dtype=torch.uint8, device=DEV)
    if fill is not None:
        ws.fill_(fill)
    out = torch.empty((b, n, k), dtype=torch.int32, device=DEV)
    cnt = torch.empty((b, n), dtype=torch.int32, device=DEV)
    m = mask.to(torch.uint8).contiguous()
    rc = getattr(lib, entry)(RS._dt(x.dtype), b, n, c, k, C.c_void_p(x.data_ptr()), C.c_void_p(m.data_ptr()), None,
                             float(r2), C.c_void_p(out.data_ptr()), C.c_void_p(cnt.data_ptr()), C.c_void_p(ws.data_ptr()),
                             nb.value, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, rc
    return out, cnt


def test_k_up_to_32_equals_the_narrow_entry_and_the_workspace_contents_do_not_matter(lib):
    x, mask, _ = RS.cloud(2, 3000, mean_count=40.0, seed=3)
    for k in (1, 16, 32):
        a = c_call(lib, x, mask, k, 1.0, "egnn_radius_select")
        w = c_call(lib, x, mask, k, 1.0)
        assert torch.equal(a[0], w[0]) and torch.equal(a[1], w[1]), k
    for k in (33, 128, 256):
        a = c_call(lib, x, mask, k, 1.0, fill=0)
        w = c_call(lib, x, mask, k, 1.0, fill=0xFF)
        assert torch.equal(a[0], w[0]) and torch.equal(a[1], w[1]), k


def test_graph_capture(lib):
    from egnn_pytorch_b200 import radius_neighbors_wide
    x, mask, _ = RS.cloud(2, 3000, mean_count=80.0, seed=4)
    want = radius_neighbors_wide(x, 1.0, 96, mask=mask, return_counts=True)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = radius_neighbors_wide(x, 1.0, 96, mask=mask, return_counts=True)
    x.add_(0.25)                                          # the replay reads the new coordinates
    want = radius_neighbors_wide(x, 1.0, 96, mask=mask, return_counts=True)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


# ----------------------------------------------------------------------------- 5. layers: grid path == all pairs


def lattice_for(kind, side, dtype):
    if kind == "box":
        return dict(box=torch.tensor([side, side, 0.0], device=DEV, dtype=dtype))
    if kind == "cell":
        return dict(cell=torch.tensor([[side, 0, 0], [0.3 * side, side, 0], [0.2 * side, -0.4 * side, side]],
                                      device=DEV, dtype=dtype))
    return {}


@pytest.mark.parametrize("lattice", ["none", "box", "cell"])
@pytest.mark.parametrize("k", [33, 64, 128])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32, torch.bfloat16], ids=["fp64", "fp32", "bf16"])
def test_layer_outputs_bit_identical(lib, monkeypatch, dtype, k, lattice):
    from egnn_pytorch_b200 import EGNN
    torch.manual_seed(k)
    dim = 64 if dtype == torch.bfloat16 else 16
    mod = EGNN(dim=dim, num_nearest_neighbors=k, valid_radius=1.0, soft_edges=True).to(DEV, dtype).eval()
    cdt = torch.float64 if dtype == torch.float64 else torch.float32
    x, mask, side = RS.cloud(2, 4096, mean_count=1.2 * k, seed=k + 1, dtype=cdt)
    feats = torch.randn((2, 4096, dim), device=DEV).to(dtype)
    kw = dict(mask=mask, **lattice_for(lattice, side, cdt))
    cell, allp = RS.both_paths(lib, monkeypatch, lambda: mod(feats, x, **kw))
    if dtype == torch.bfloat16 and lattice != "cell":
        assert mod.last_path == "bf16-tc"
    for a, w, what in zip(cell, allp, ("feats", "coors")):
        assert torch.equal(RS.bits(a), RS.bits(w)), f"{what}: max diff {(a.float() - w.float()).abs().max()}"


@pytest.mark.parametrize("lattice", ["box", "cell"])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
def test_gradients_agree(lib, monkeypatch, dtype, lattice):
    from egnn_pytorch_b200 import EGNN
    torch.manual_seed(6)
    n, k = 4096, 64
    mod = EGNN(dim=16, num_nearest_neighbors=k, valid_radius=1.0, norm_coors=True).to(DEV, dtype)
    x0, mask, side = RS.cloud(2, n, mean_count=80.0, dtype=dtype, seed=12)
    f0 = torch.randn((2, n, 16), device=DEV, dtype=dtype)
    gf, gx = torch.randn_like(f0), torch.randn_like(x0)
    lat0 = next(iter(lattice_for(lattice, side, dtype).values()))

    def run():
        f, x = f0.clone().requires_grad_(True), x0.clone().requires_grad_(True)
        lat = lat0.clone().requires_grad_(True)
        mod.zero_grad(set_to_none=True)
        with torch.enable_grad():
            fo, xo = mod(f, x, mask=mask, lattice_grad=True, **{lattice: lat})
            ((fo * gf).sum() + (xo * gx).sum()).backward()
        grads = {"feats": f.grad, "coors": x.grad, lattice: lat.grad}
        grads.update({name: p.grad.clone() for name, p in mod.named_parameters()})
        return fo.detach(), xo.detach(), grads

    cell, allp = RS.both_paths(lib, monkeypatch, run)
    assert torch.equal(RS.bits(cell[0]), RS.bits(allp[0])) and torch.equal(RS.bits(cell[1]), RS.bits(allp[1]))
    for name, g in cell[2].items():
        w = allp[2][name]
        # the lists are the same, so the paths differ only in the order of the backward's atomic sums; the lattice
        # gradient sums over every pair
        tol = (1e-10 if dtype == torch.float64 else 2e-5) * (10 if name == lattice else 1)
        scale = max(1.0, float(w.abs().max()))
        assert float((g - w).abs().max()) <= tol * scale, f"{dtype} {name}: {float((g - w).abs().max())}"


def test_layer_beyond_the_sort_limit_runs_on_the_grid():
    """N = 20000 > SELECT_SORT_MAX_N: the layer selects on the grid and equals the layer given the exact lists."""
    from scipy.spatial import cKDTree
    from egnn_pytorch_b200 import EGNN
    n, k = 20000, 64
    x, mask, _ = RS.cloud(1, n, mean_count=80.0, seed=31)
    xn, mn = x[0].cpu().numpy(), mask[0].cpu().numpy()
    r2 = np.float32(1.0)
    lists = np.full((n, k), -1, np.int32)
    tree = cKDTree(xn.astype(np.float64))
    for i, cand in enumerate(tree.query_ball_point(xn.astype(np.float64), 1.0 + 1e-3)):
        if not mn[i]:
            continue
        cand = np.asarray(sorted(cand))
        cand = cand[mn[cand]]
        d = KS.ranks(xn[None], [i])[0, 0][cand]           # the select's rank, in fp32
        keep = d <= r2
        o = np.lexsort((cand[keep], d[keep]))[:k]
        lists[i, : len(o)] = cand[keep][o]
    torch.manual_seed(5)
    mod = EGNN(dim=16, num_nearest_neighbors=k, valid_radius=1.0).to(DEV).eval()
    f = torch.randn((1, n, 16), device=DEV)
    f1, x1 = mod(f, x, mask=mask)
    f2, x2 = mod(f, x, mask=mask, neighbors=torch.from_numpy(lists[None]).to(DEV))
    assert torch.equal(f1, f2) and torch.equal(x1, x2)


def test_network_outputs_bit_identical(lib, monkeypatch):
    from egnn_pytorch_b200 import EGNN_Network
    torch.manual_seed(4)
    net = EGNN_Network(depth=2, dim=32, num_nearest_neighbors=48, valid_radius=1.0).to(DEV)
    x, mask, _ = RS.cloud(2, 4096, mean_count=60.0, seed=9)
    feats = torch.randn((2, 4096, 32), device=DEV)
    cell, allp = RS.both_paths(lib, monkeypatch, lambda: net(feats, x, mask=mask))
    assert torch.equal(RS.bits(cell[0]), RS.bits(allp[0])) and torch.equal(RS.bits(cell[1]), RS.bits(allp[1]))


def test_graphed_forward_captures_the_grid_path(lib, monkeypatch):
    from egnn_pytorch_b200 import EGNN, GraphedForward
    torch.manual_seed(8)
    mod = EGNN(dim=32, num_nearest_neighbors=64, valid_radius=1.0).to(DEV).eval()
    x, mask, _ = RS.cloud(2, 4096, mean_count=80.0, seed=13)
    feats = torch.randn((2, 4096, 32), device=DEV)
    fast = GraphedForward(mod, feats, x, mask=mask)
    for s in range(2):
        x2 = x + 0.3 * torch.randn(x.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(s))
        f2 = torch.randn_like(feats)
        got = [t.clone() for t in fast(f2, x2)]
        want = mod(f2, x2, mask=mask)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    monkeypatch.setenv("EGNN_B200_CELL_SELECT_MIN_N", NEVER)
    want = mod(f2, x2, mask=mask)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
