"""k-nearest-neighbour lists on the cell grid (csrc/radius_select.cu, knn_grid_setup_kernel / knn_ring_kernel /
knn_scan_kernel): egnn_knn_grid_select*, `knn_neighbors` and layers under EGNN_FLAG_KNN_GRID.

Reference: the all-pairs select.  Without a lattice it is egnn_knn_select itself; under a box or a cell it is the exact
numpy restatement of its arithmetic (`ranks` of test_gpu_knn_select.py, `cell_ranks` of
test_gpu_lattice_tile_boundaries.py), as is every row beyond N = 16384 with k > 32, where the block sort cannot run.
Indices and ok bytes must be equal bit for bit.  Inside a layer the two paths are switched with
EGNN_B200_KNN_GRID_MIN_N (0 = kNN grid, huge = all pairs); forward outputs must be bit-identical."""
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


def grid_select(lib, x, mask, k, vr, box=None, cell=None):
    """egnn_knn_grid_select(_triclinic) -> (idx, ok) [B, N, k]; the workspace is filled with garbage first."""
    b, n, c = x.shape
    idx = torch.empty((b, n, k), dtype=torch.int32, device=DEV)
    ok = torch.empty((b, n, k), dtype=torch.uint8, device=DEV)
    nb = C.c_size_t()
    assert lib.egnn_knn_grid_select_workspace_bytes(b, n, c, k, C.byref(nb)) == 0
    ws = torch.randint(0, 255, (nb.value + 256,), dtype=torch.uint8, device=DEV)
    wp = (ws.data_ptr() + 255) // 256 * 256
    m = None if mask is None else mask.to(torch.uint8).contiguous()
    lat = cell if cell is not None else box
    lat = None if lat is None else lat.to(DEV, x.dtype).contiguous()
    entry = lib.egnn_knn_grid_select_triclinic if cell is not None else lib.egnn_knn_grid_select
    rc = entry(RS._dt(x.dtype), b, n, c, k, C.c_void_p(x.data_ptr()), None if m is None else C.c_void_p(m.data_ptr()),
               None if lat is None else C.c_void_p(lat.data_ptr()), float(vr), C.c_void_p(idx.data_ptr()),
               C.c_void_p(ok.data_ptr()), C.c_void_p(wp), nb.value, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, rc
    return idx, ok.bool()


def numpy_select(x, mask, k, vr, box=None, cell=None, rows=None):
    """The all-pairs select in numpy, in x's type -> (idx, ok) for rows `rows` (all if None)."""
    xn = x.cpu().numpy()
    T = xn.dtype.type
    mn = None if mask is None else mask.cpu().numpy()
    rows = np.arange(xn.shape[1]) if rows is None else np.asarray(rows)
    idx, ok = [], []
    for s in range(0, len(rows), 256):
        r = rows[s:s + 256]
        if cell is not None:
            d = cell_ranks(xn, r, cell.cpu().numpy().astype(xn.dtype), mn)
        else:
            d = KS.ranks(xn, r, mn, None, None if box is None else box.cpu().numpy().astype(xn.dtype))
        o = np.argsort(d, axis=-1, kind="stable")[..., :k]
        idx.append(o)
        ok.append(np.take_along_axis(d, o, axis=-1) <= T(vr))
    return np.concatenate(idx, 1).astype(np.int32), np.concatenate(ok, 1)


def coords(kind, b, n, c, dtype, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    if kind == "uniform":
        x = torch.rand((b, n, c), generator=g, dtype=torch.float64) * (1.0 + torch.arange(b).view(b, 1, 1))
    elif kind == "normal":
        x = torch.randn((b, n, c), generator=g, dtype=torch.float64)
    elif kind == "clusters":                         # two clusters 10^3 apart
        x = 0.1 * torch.randn((b, n, c), generator=g, dtype=torch.float64)
        x[:, n // 2:, 0] += 1e3
    elif kind == "line":
        t = torch.rand((b, n, 1), generator=g, dtype=torch.float64)
        x = t * torch.tensor([1.0, -2.0, 0.5][:c], dtype=torch.float64)
    elif kind == "coincident":
        x = torch.full((b, n, c), 0.25, dtype=torch.float64)
    elif kind == "lattice":                          # integer lattice: masses of exact ties
        side = max(2, round(n ** (1.0 / c)))
        i = torch.arange(n)
        x = torch.stack([(i // side ** a) % side for a in range(c)], -1).to(torch.float64).expand(b, n, c).clone()
    elif kind == "dyadic":
        x = torch.randint(0, 64, (b, n, c), generator=g).to(torch.float64) / 8.0
    else:
        raise ValueError(kind)
    return x.to(DEV, dtype).contiguous()


def masks(kind, b, n, k, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    if kind == "none":
        return None
    m = torch.rand((b, n), generator=g) < 0.8
    if kind == "padded_graph" and b > 1:
        m[1] = False
    if kind == "few":                                # graph 0 keeps fewer than k valid nodes
        m[0] = False
        m[0, : max(0, k - 1)] = True
    return m.to(DEV)


def check(lib, x, mask, k, vr, what, box=None, cell=None):
    gi, go = grid_select(lib, x, mask, k, vr, box, cell)
    if box is None and cell is None:
        wi, wo = RS.knn_select(lib, x, mask, k, vr)
        wi, wo = wi.cpu().numpy(), wo.cpu().numpy()
    else:
        wi, wo = numpy_select(x, mask, k, vr, box, cell)
    gi, go = gi.cpu().numpy(), go.cpu().numpy()
    bad = np.argwhere((gi != wi) | (go != wo))
    assert len(bad) == 0, f"{what}: {len(bad)} slots differ, first {bad[:3].tolist()}: grid {gi[tuple(bad[0][:2])]} " \
                          f"all-pairs {wi[tuple(bad[0][:2])]}"


@pytest.mark.parametrize("k", [1, 8, 31, 32, 33, 64, 255, 256])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
def test_equals_egnn_knn_select(lib, dtype, k):
    for c in (1, 2, 3):
        for kind in ("uniform", "normal", "clusters", "line", "lattice", "dyadic"):
            n = 1500 if c > 1 else 700
            x = coords(kind, 2, n, c, dtype, seed=k + 10 * c)
            mask = masks(("none", "rand", "padded_graph")[(k + c) % 3], 2, n, k, seed=c)
            check(lib, x, mask, k, 0.05, f"k={k} C={c} {kind} {dtype}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
def test_degenerate_inputs(lib, dtype):
    """k = N, all-coincident nodes, a single valid node, graphs with fewer than k valid nodes, NaN and inf nodes."""
    for k in (1, 17, 200):
        check(lib, coords("uniform", 2, 200, 3, dtype, 1), None, 200, math.inf, "k = N")
        check(lib, coords("coincident", 2, 900, 3, dtype, 2), masks("rand", 2, 900, k, 3), k, 0.0, f"coincident k={k}")
        check(lib, coords("normal", 3, 900, 2, dtype, 4), masks("few", 3, 900, k, 5), k, 1.0, f"few valid k={k}")
        m = torch.zeros((2, 900), dtype=torch.bool, device=DEV)
        m[:, 7] = True
        check(lib, coords("normal", 2, 900, 3, dtype, 6), m, k, math.inf, f"one valid node k={k}")
        x = coords("uniform", 2, 1200, 3, dtype, 7)
        x[0, 5, 1] = float("nan")
        x[0, 9] = float("inf")
        x[1, 100, 0] = -float("inf")
        x[1, 101:110, 2] = float("nan")
        for mk in ("none", "rand"):
            check(lib, x, masks(mk, 2, 1200, k, 8), k, 0.01, f"non-finite k={k} mask={mk}")


def boxes(kind, b, c, dtype):
    if kind == "cubic":
        return torch.full((b, c), 1.0, dtype=dtype)
    if kind == "mixed":                              # periodic, 0 and inf axes
        return torch.tensor([1.0, 0.0, math.inf][:c], dtype=dtype).expand(b, c).contiguous()
    if kind == "per_graph":
        return torch.tensor([[1.0, 0.7, 1.3][:c], [0.6, 1.0, 0.9][:c]], dtype=dtype)[:b]
    if kind == "tiny":                               # so small that the rings wrap fully
        return torch.full((b, c), 0.1, dtype=dtype)
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["cubic", "mixed", "per_graph", "tiny"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
def test_periodic_boxes(lib, dtype, kind):
    for c in (1, 2, 3):
        for k in (8, 32, 64):
            bx = boxes(kind, 2, c, dtype)
            # coordinates in [0, L) on periodic axes, so that the numpy minimum image is exact (KS.ranks)
            x = torch.rand((2, 1000, c), dtype=torch.float64, generator=torch.Generator().manual_seed(k + c))
            L = torch.where((bx > 0) & torch.isfinite(bx), bx.double(), torch.ones_like(bx, dtype=torch.float64))
            x = (x * L[:, None, :]).to(DEV, dtype)
            check(lib, x, masks("rand", 2, 1000, k, c), k, 0.02, f"box {kind} C={c} k={k}", box=bx)


def cells(kind, dtype):
    if kind == "tilt":                               # a tilt of 0.95 of the diagonal
        return torch.tensor([[[1.0, 0, 0], [0.95, 1.0, 0], [0.95, 0.95, 1.0]]], dtype=dtype)
    if kind == "hex_slab":                           # hexagonal in x-y, aperiodic z
        return torch.tensor([[[1.0, 0, 0], [0.5, math.sqrt(3) / 2, 0], [0, 0, 0]]], dtype=dtype)
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["tilt", "hex_slab"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
def test_triclinic_cells(lib, dtype, kind):
    cl = cells(kind, dtype)
    for k in (8, 32, 100):
        x = (torch.rand((1, 1200, 3), generator=torch.Generator().manual_seed(k), dtype=torch.float64) * 2 - 0.5)
        check(lib, x.to(DEV, dtype), masks("rand", 1, 1200, k, k), k, 0.05, f"cell {kind} k={k}", cell=cl)


def test_beyond_the_sort_limit_against_the_exact_reference(lib):
    """N = 20000 > 16384 with k > 32: rows of the grid's lists against the numpy restatement of the select."""
    n = 20000
    for k, kind, dtype in ((64, "uniform", torch.float32), (256, "normal", torch.float64)):
        x = coords(kind, 1, n, 3, dtype, seed=k)
        mask = masks("rand", 1, n, k, seed=k)
        gi, go = grid_select(lib, x, mask, k, 0.01)
        rows = np.random.default_rng(k).choice(n, 400, replace=False)
        wi, wo = numpy_select(x, mask, k, 0.01, rows=rows)
        assert np.array_equal(gi.cpu().numpy()[:, rows], wi) and np.array_equal(go.cpu().numpy()[:, rows], wo), k


def test_graph_capture(lib):
    x = coords("normal", 2, 5000, 3, torch.float32, 1)
    mask = masks("rand", 2, 5000, 16, 2)
    want = grid_select(lib, x, mask, 16, 0.1)
    from egnn_pytorch_b200 import knn_neighbors
    knn_neighbors(x, 16, mask=mask)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = knn_neighbors(x, 16, mask=mask)
    x.copy_(coords("uniform", 2, 5000, 3, torch.float32, 3))
    g.replay()
    torch.cuda.synchronize()
    again = knn_neighbors(x, 16, mask=mask)
    assert torch.equal(out, again)
    assert want[0].shape == out.shape


# ------------------------------------------------------------------ layers

def _both_paths(lib, monkeypatch, fn):
    monkeypatch.setenv("EGNN_B200_KNN_GRID_MIN_N", "0")
    grid, n_grid = RS._launches(lib, fn)
    monkeypatch.setenv("EGNN_B200_KNN_GRID_MIN_N", NEVER)
    allp, n_all = RS._launches(lib, fn)
    assert n_grid > n_all, (n_grid, n_all)
    return grid, allp


def _lattice(kind, dtype):
    if kind == "box":
        return dict(box=torch.tensor([4.0, 4.0, 4.0], device=DEV, dtype=dtype))
    if kind == "cell":
        return dict(cell=torch.tensor([[4.0, 0, 0], [1.0, 4.0, 0], [0.5, 1.0, 4.0]], device=DEV, dtype=dtype))
    return {}


@pytest.mark.parametrize("variant", ["plain", "mask", "box", "cell", "mean"])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32, torch.bfloat16], ids=["fp64", "fp32", "bf16"])
def test_layer_outputs_bit_identical(lib, monkeypatch, dtype, variant):
    from egnn_pytorch_b200 import EGNN
    torch.manual_seed(3)
    dim = 64 if dtype == torch.bfloat16 else 16
    kw_mod = dict(m_pool_method="mean") if variant == "mean" else {}
    mod = EGNN(dim=dim, num_nearest_neighbors=24, **kw_mod).to(DEV, dtype).eval()
    cdt = torch.float64 if dtype == torch.float64 else torch.float32
    x = (torch.rand((2, 3000, 3), device=DEV, dtype=cdt) * 4.0)
    feats = torch.randn((2, 3000, dim), device=DEV).to(dtype)
    kw = _lattice(variant, cdt)
    if variant in ("mask", "mean"):
        kw["mask"] = torch.rand((2, 3000), device=DEV) < 0.9
    grid, allp = _both_paths(lib, monkeypatch, lambda: mod(feats, x, **kw))
    for a, w, what in zip(grid, allp, ("feats", "coors")):
        assert torch.equal(RS.bits(a), RS.bits(w)), f"{what}: max diff {(a.float() - w.float()).abs().max()}"


def test_c4_shape_bit_identical(lib, monkeypatch):
    """BASELINE c4's layer: B = 8, N = 4096, k = 32, edge_dim = 4, bf16, N(0, 1) coordinates."""
    from egnn_pytorch_b200 import EGNN
    torch.manual_seed(4)
    mod = EGNN(dim=64, edge_dim=4, num_nearest_neighbors=32).to(DEV, torch.bfloat16).eval()
    x = torch.randn((8, 4096, 3), device=DEV)
    f = torch.randn((8, 4096, 64), device=DEV).to(torch.bfloat16)
    e = torch.randn((8, 4096, 4096, 4), device=DEV).to(torch.bfloat16)
    grid, allp = _both_paths(lib, monkeypatch, lambda: mod(f, x, e))
    assert torch.equal(RS.bits(grid[0]), RS.bits(allp[0])) and torch.equal(RS.bits(grid[1]), RS.bits(allp[1]))


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
def test_gradients_agree(lib, monkeypatch, dtype):
    from egnn_pytorch_b200 import EGNN
    torch.manual_seed(6)
    n = 3000
    mod = EGNN(dim=16, num_nearest_neighbors=40, norm_coors=True).to(DEV, dtype)
    x0 = torch.randn((2, n, 3), device=DEV, dtype=dtype)
    f0 = torch.randn((2, n, 16), device=DEV, dtype=dtype)
    mask = torch.rand((2, n), device=DEV) < 0.9
    gf, gx = torch.randn_like(f0), torch.randn_like(x0)

    def run():
        f, x = f0.clone().requires_grad_(True), x0.clone().requires_grad_(True)
        mod.zero_grad(set_to_none=True)
        with torch.enable_grad():
            fo, xo = mod(f, x, mask=mask)
            ((fo * gf).sum() + (xo * gx).sum()).backward()
        grads = {"feats": f.grad, "coors": x.grad}
        grads.update({name: p.grad.clone() for name, p in mod.named_parameters()})
        return fo.detach(), xo.detach(), grads

    grid, allp = _both_paths(lib, monkeypatch, run)
    assert torch.equal(RS.bits(grid[0]), RS.bits(allp[0])) and torch.equal(RS.bits(grid[1]), RS.bits(allp[1]))
    for name, g in grid[2].items():
        w = allp[2][name]
        tol = 1e-10 if dtype == torch.float64 else 2e-5
        assert float((g - w).abs().max()) <= tol * max(1.0, float(w.abs().max())), name


def test_network_and_row_shards_bit_identical(lib, monkeypatch):
    from egnn_pytorch_b200 import EGNN, EGNN_Network
    torch.manual_seed(7)
    net = EGNN_Network(depth=3, dim=32, num_nearest_neighbors=16).to(DEV)
    x = torch.randn((2, 3000, 3), device=DEV)
    feats = torch.randn((2, 3000, 32), device=DEV)
    grid, allp = _both_paths(lib, monkeypatch, lambda: net(feats, x))
    assert torch.equal(RS.bits(grid[0]), RS.bits(allp[0])) and torch.equal(RS.bits(grid[1]), RS.bits(allp[1]))
    mod = EGNN(dim=16, num_nearest_neighbors=16).to(DEV).eval()
    f = torch.randn((1, 3000, 16), device=DEV)
    grid, allp = _both_paths(lib, monkeypatch, lambda: mod(f, x[:1], _rows=(1000, 2000)))
    assert torch.equal(RS.bits(grid[0]), RS.bits(allp[0])) and torch.equal(RS.bits(grid[1]), RS.bits(allp[1]))


def test_graphed_forward_captures_the_grid_path(monkeypatch):
    from egnn_pytorch_b200 import EGNN, GraphedForward
    monkeypatch.setenv("EGNN_B200_KNN_GRID_MIN_N", "0")
    torch.manual_seed(8)
    mod = EGNN(dim=32, num_nearest_neighbors=32).to(DEV).eval()
    x = torch.randn((2, 4096, 3), device=DEV)
    mask = torch.rand((2, 4096), device=DEV) < 0.9
    feats = torch.randn((2, 4096, 32), device=DEV)
    fast = GraphedForward(mod, feats, x, mask=mask)
    for s in range(2):
        x2 = x + 0.3 * torch.randn(x.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(s))
        f2 = torch.randn_like(feats)
        got = [t.clone() for t in fast(f2, x2)]
    monkeypatch.setenv("EGNN_B200_KNN_GRID_MIN_N", NEVER)
    want = mod(f2, x2, mask=mask)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


@pytest.mark.parametrize("variant", ["plain", "mask", "box"])
def test_knn_neighbors_fed_back_equals_the_layers_select(monkeypatch, variant):
    from egnn_pytorch_b200 import EGNN, knn_neighbors
    monkeypatch.setenv("EGNN_B200_KNN_GRID_MIN_N", NEVER)
    torch.manual_seed(9)
    mod = EGNN(dim=16, num_nearest_neighbors=24).to(DEV).eval()
    x = torch.rand((2, 2000, 3), device=DEV) * 4.0
    f = torch.randn((2, 2000, 16), device=DEV)
    kw = _lattice("box" if variant == "box" else "", torch.float32)
    if variant == "mask":
        kw["mask"] = torch.rand((2, 2000), device=DEV) < 0.9
    nbr = knn_neighbors(x, 24, **kw)
    if "mask" in kw:
        assert bool((nbr[~kw["mask"]] == -1).all())
    want = mod(f, x, **kw)
    got = mod(f, x, neighbors=nbr, **kw)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
