"""Packed batches on the cell grids (egnn_radius_select_packed*, egnn_knn_grid_select_packed*): every graph of at least
the unpacked threshold's nodes (and k) goes on the radius or kNN grid in its segment form, the rest on the segmented
all-pairs select.

kNN mode: idx and ok equal egnn_knn_select_packed's bit for bit.  Radius mode: ok equals its ok, idx equals its idx in
every ok = 1 slot, so the kept lists idx.masked_fill(ok == 0, -1) are equal; they also equal the unpacked grid
(egnn_radius_select_wide, egnn_knn_grid_select) on each graph alone, shifted by ptr[g].  Thresholds are forced low
through EGNN_B200_CELL_SELECT_MIN_N / EGNN_B200_KNN_GRID_MIN_N (read at every call) and also run at their defaults.
Layers, networks and builders on grid-sized graphs equal the same calls with the grids forced off."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from test_gpu_packed import _ptr, packed_select

pytestmark = pytest.mark.gpu

DEV = "cuda"
ENV = {"knn": "EGNN_B200_KNN_GRID_MIN_N", "radius": "EGNN_B200_CELL_SELECT_MIN_N"}
OFF = str(1 << 40)


@pytest.fixture(scope="module")
def lib():
    from egnn_pytorch_b200 import _native
    return _native.load()


def grid_packed(lib, mode, x, ptr, k, vr, mask=None, box=None, cell=None):
    """egnn_{radius,knn_grid}_select_packed(_triclinic) on x [T, C] -> (idx, ok) numpy [T, k]; outputs poisoned and
    the workspace filled with garbage first."""
    from egnn_pytorch_b200 import _native as nat
    t, c = x.shape
    g = ptr.numel() - 1
    sizes = (ptr[1:] - ptr[:-1]).tolist()
    idx = torch.full((t, k), -7, dtype=torch.int32, device=DEV)
    ok = torch.full((t, k), 7, dtype=torch.uint8, device=DEV)
    name = "egnn_radius_select_packed" if mode == "radius" else "egnn_knn_grid_select_packed"
    nb = C.c_size_t()
    assert getattr(lib, name + "_workspace_bytes")(g, t, c, k, C.byref(nb)) == 0
    ws = torch.randint(0, 255, (nb.value + 256,), dtype=torch.uint8, device=DEV)
    wp = (ws.data_ptr() + 255) // 256 * 256
    p32 = ptr.to(DEV, torch.int32).contiguous()
    m = None if mask is None else mask.to(DEV, torch.uint8).contiguous()
    lat = cell if cell is not None else box
    lat = None if lat is None else lat.to(DEV, x.dtype).contiguous()
    entry = getattr(lib, name + ("_triclinic" if cell is not None else ""))
    rc = entry(nat.DTYPE_F64 if x.dtype == torch.float64 else nat.DTYPE_F32, g, t, c, k, max(sizes),
               C.c_void_p(p32.data_ptr()), C.c_void_p(x.data_ptr()), None if m is None else C.c_void_p(m.data_ptr()),
               None if lat is None else C.c_void_p(lat.data_ptr()), float(vr), C.c_void_p(idx.data_ptr()),
               C.c_void_p(ok.data_ptr()), C.c_void_p(wp), nb.value, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, rc
    torch.cuda.synchronize()
    return idx.cpu().numpy(), ok.cpu().numpy()


def points(sizes, c, dtype, seed, kind="rand"):
    """Graphs of `sizes` nodes at density ~1 per unit volume (per graph), with coincident points and non-finite
    coordinates for kind="degenerate"."""
    rs = np.random.RandomState(seed)
    parts = []
    for n in sizes:
        side = max(n, 1) ** (1.0 / c)
        p = rs.uniform(0, side, size=(n, c))
        if kind == "degenerate" and n > 4:
            p[n // 2:n // 2 + 4] = p[0]                          # coincident with node 0
            p[rs.choice(n, 3, replace=False), rs.randint(0, c, 3)] = [np.nan, np.inf, -np.inf]
        parts.append(p)
    x = np.concatenate(parts) if parts else np.zeros((0, c))
    return torch.from_numpy(x).to(DEV, dtype).contiguous()


def check_equal(lib, mode, x, ptr, k, vr, mask=None, box=None, cell=None, what=""):
    gi, go = grid_packed(lib, mode, x, ptr, k, vr, mask, box, cell)
    pi, po = packed_select(lib, x, ptr, k, vr, mask, box, cell)
    if mode == "knn":
        assert np.array_equal(gi, pi) and np.array_equal(go, po), f"kNN mode != egnn_knn_select_packed {what}"
    else:
        assert np.array_equal(go, po), f"radius mode ok != egnn_knn_select_packed's {what}"
        assert np.array_equal(np.where(go == 0, -1, gi), np.where(po == 0, -1, pi)), f"radius lists differ {what}"
    return gi, go


THR = 300
SIZES = [THR - 1, THR, THR + 1, 0, 5, 3, 40, THR + 257] + [17] * 30 + [2 * THR, 1]


def _lattice(lat, c, dtype):
    side = 9.0
    if lat == "box":
        return dict(box=torch.tensor([side] * (c - 1) + [0.0], dtype=dtype, device=DEV))   # the last axis aperiodic
    if lat == "cell":
        cell = torch.diag(torch.tensor([side] * c, dtype=dtype))
        cell[1, 0] = 1.5
        if c == 3:
            cell[2, 0], cell[2, 1] = -0.5, 1.0
        return dict(cell=cell.to(DEV))
    return {}


CASES = []
for i_, k_ in enumerate([1, 16, 32, 33, 96, 256]):
    for dt_ in (torch.float32, torch.float64):
        CASES.append(dict(k=k_, dtype=dt_, C=[1, 2, 3][(i_ + (dt_ == torch.float64)) % 3],
                          lat=[None, "box", "cell"][i_ % 3], mask=(i_ + (dt_ == torch.float64)) % 2 == 0))


@pytest.mark.parametrize("mode", ["knn", "radius"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: f"k{c['k']}-{str(c['dtype'])[6:]}-c{c['C']}-{c['lat']}"
                                                      f"{'-mask' if c['mask'] else ''}")
def test_forced_thresholds_equal_the_packed_select(lib, monkeypatch, mode, case):
    monkeypatch.setenv(ENV[mode], str(THR))
    k, c, dtype = case["k"], case["C"], case["dtype"]
    lat = case["lat"] if not (case["lat"] == "cell" and c == 1) else "box"
    sizes = [max(n, k + 1) if n >= THR else n for n in SIZES]
    ptr = _ptr(sizes)
    x = points(sizes, c, dtype, k + c)
    mask = torch.from_numpy(np.random.RandomState(k).rand(x.shape[0]) > 0.15) if case["mask"] else None
    vr = {"knn": [math.inf, 2.0][k % 2], "radius": 1.7 ** 2}[mode]
    kw = _lattice(lat, c, dtype)
    gi, go = check_equal(lib, mode, x, ptr, k, vr, mask, what=f"{case}", **kw)
    # the grid graphs against the unpacked grid on each graph alone, shifted by ptr[g]
    for g, n in enumerate(sizes):
        lo = int(ptr[g])
        if n < max(THR, k):
            continue
        xs = x[lo:lo + n][None].contiguous()
        ms = None if mask is None else mask[lo:lo + n][None].to(DEV)
        lat1 = {key: v[None] for key, v in kw.items()}
        if mode == "knn":
            from test_gpu_knn_grid import grid_select
            ui, uo = grid_select(lib, xs, ms, k, vr, **lat1)
            assert np.array_equal(gi[lo:lo + n], ui[0].cpu().numpy() + lo)
            assert np.array_equal(go[lo:lo + n].astype(bool), uo[0].cpu().numpy())
        else:
            want = unpacked_radius(lib, xs, ms, k, vr, **lat1)
            got = np.where(go[lo:lo + n] == 0, -1, gi[lo:lo + n])
            assert np.array_equal(got, np.where(want >= 0, want + lo, -1)), f"graph {g} vs the unpacked radius grid"


def unpacked_radius(lib, x, mask, k, r2, box=None, cell=None):
    """egnn_radius_select_wide(_triclinic) on one graph [1, n, C] -> idx numpy [n, k] (-1 empty)."""
    from egnn_pytorch_b200 import _native as nat
    _, n, c = x.shape
    out = torch.empty((1, n, k), dtype=torch.int32, device=DEV)
    nb = C.c_size_t()
    assert lib.egnn_radius_select_wide_workspace_bytes(1, n, c, k, C.byref(nb)) == 0
    ws = torch.empty(nb.value + 256, dtype=torch.uint8, device=DEV)
    wp = (ws.data_ptr() + 255) // 256 * 256
    m = None if mask is None else mask.to(torch.uint8).contiguous()
    lat = cell if cell is not None else box
    lat = None if lat is None else lat.contiguous()
    fn = lib.egnn_radius_select_wide_triclinic if cell is not None else lib.egnn_radius_select_wide
    rc = fn(nat.DTYPE_F64 if x.dtype == torch.float64 else nat.DTYPE_F32, 1, n, c, k, C.c_void_p(x.data_ptr()),
            None if m is None else C.c_void_p(m.data_ptr()), None if lat is None else C.c_void_p(lat.data_ptr()),
            float(r2), C.c_void_p(out.data_ptr()), None, C.c_void_p(wp), nb.value,
            C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, rc
    return out[0].cpu().numpy()


@pytest.mark.parametrize("mode", ["knn", "radius"])
@pytest.mark.parametrize("k", [32, 96])
def test_default_thresholds(lib, monkeypatch, mode, k):
    """Graphs across both default thresholds (4096 radius, 8192 kNN) and one above 16384 nodes."""
    monkeypatch.delenv(ENV[mode], raising=False)
    sizes = [4095, 4096, 4097, 8191, 8192, 8193, 16500] + [20] * 50
    ptr = _ptr(sizes)
    x = points(sizes, 3, torch.float32, k)
    mask = torch.from_numpy(np.random.RandomState(1).rand(x.shape[0]) > 0.05)
    check_equal(lib, mode, x, ptr, k, {"knn": math.inf, "radius": 1.6 ** 2}[mode], mask if mode == "radius" else None)


@pytest.mark.parametrize("mode", ["knn", "radius"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_degenerate_inputs(lib, monkeypatch, mode, dtype):
    """Coincident points, NaN / inf coordinates and a fully masked graph on the grid."""
    monkeypatch.setenv(ENV[mode], "64")
    sizes = [200, 64, 63, 300, 0, 90]
    ptr = _ptr(sizes)
    x = points(sizes, 3, dtype, 5, "degenerate")
    x[int(ptr[5]):int(ptr[6])] = x[int(ptr[5])]                  # a graph of 90 coincident points
    mask = torch.ones(x.shape[0], dtype=torch.bool)
    mask[int(ptr[3]):int(ptr[4])] = False                        # a fully masked graph
    mask[3] = False
    for k in (8, 40):
        for m in (None, mask):
            check_equal(lib, mode, x, ptr, k, {"knn": 1.0, "radius": 1.2}[mode], m, what=f"k{k} mask {m is not None}")


def test_below_threshold_equals_the_packed_select(lib, monkeypatch):
    """max_n under the default thresholds: the entries run the segmented select alone."""
    monkeypatch.delenv(ENV["knn"], raising=False)
    monkeypatch.delenv(ENV["radius"], raising=False)
    sizes = [100, 200, 50]
    ptr = _ptr(sizes)
    x = points(sizes, 3, torch.float32, 2)
    check_equal(lib, "knn", x, ptr, 8, math.inf)
    check_equal(lib, "radius", x, ptr, 8, 2.0)


# ------------------------------------------------------------------ builders, layers, networks, capture


def _big_batch(dtype, seed=0, c=3):
    sizes = [700, 9, 0, 520, 33, 260]
    ptr = _ptr(sizes)
    x = points(sizes, c, dtype, seed)[None]
    mask = torch.from_numpy(np.random.RandomState(seed).rand(1, x.shape[1]) > 0.1).to(DEV)
    return sizes, ptr, x, mask


@pytest.mark.parametrize("builder, k", [("knn", 16), ("knn", 96), ("radius", 16), ("wide", 64)])
@pytest.mark.parametrize("lattice", [None, "box", "cell"])
def test_builders_equal_the_per_graph_calls(monkeypatch, builder, k, lattice):
    from egnn_pytorch_b200 import knn_neighbors, radius_neighbors, radius_neighbors_wide
    monkeypatch.setenv(ENV["knn"], "250")
    monkeypatch.setenv(ENV["radius"], "250")
    sizes, ptr, x, mask = _big_batch(torch.float32, k)
    x[0, 5, 1] = float("nan")
    kw = {key: v for key, v in _lattice(lattice, 3, torch.float32).items()}
    call = {"knn": lambda xx, m, **a: knn_neighbors(xx, k, mask=m, **a),
            "radius": lambda xx, m, **a: radius_neighbors(xx, 1.5, k, mask=m, **a),
            "wide": lambda xx, m, **a: radius_neighbors_wide(xx, 2.0, k, mask=m, **a)}[builder]
    for m in (None, mask):
        got = call(x, m, ptr=ptr, **kw).cpu()
        monkeypatch.setenv(ENV["knn"], OFF)
        monkeypatch.setenv(ENV["radius"], OFF)
        off = call(x, m, ptr=ptr, **kw).cpu()
        monkeypatch.setenv(ENV["knn"], "250")
        monkeypatch.setenv(ENV["radius"], "250")
        assert torch.equal(got, off), f"{builder}: grids on != grids off"
        for g, n in enumerate(sizes):
            lo, hi = int(ptr[g]), int(ptr[g + 1])
            if n < k:
                continue
            want = call(x[:, lo:hi], None if m is None else m[:, lo:hi], **kw).cpu()
            assert torch.equal(got[:, lo:hi], torch.where(want >= 0, want + lo, want)), f"{builder} graph {g}"


def _layer(dtype, k, vr):
    from egnn_pytorch_b200 import EGNN
    torch.manual_seed(0)
    return EGNN(dim=16, m_dim=16, num_nearest_neighbors=k, valid_radius=vr, init_eps=0.1, norm_coors=True).to(DEV, dtype)


def _on_off(monkeypatch, fn):
    """fn() with the grids forced on for graphs of >= 250 nodes, then forced off."""
    monkeypatch.setenv(ENV["knn"], "250")
    monkeypatch.setenv(ENV["radius"], "250")
    on = fn()
    monkeypatch.setenv(ENV["knn"], OFF)
    monkeypatch.setenv(ENV["radius"], OFF)
    off = fn()
    return on, off


LAYER_CASES = [("knn", 16, math.inf, False), ("knn_vr_mask", 40, 1.5, True), ("radius_mask", 16, 1.7 ** 2, True)]


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32, torch.bfloat16])
@pytest.mark.parametrize("name, k, vr, mask_on", LAYER_CASES)
def test_layer_grids_on_equal_grids_off(monkeypatch, dtype, name, k, vr, mask_on):
    lay = _layer(dtype, k, vr)
    cdt = torch.float64 if dtype == torch.float64 else torch.float32
    sizes, ptr, x, mask = _big_batch(cdt, k)
    feats = torch.randn(1, x.shape[1], 16, device=DEV, dtype=dtype)
    m = mask if mask_on else None
    with torch.no_grad():
        on, off = _on_off(monkeypatch, lambda: lay(feats, x, mask=m, ptr=ptr))
    assert torch.equal(on[0], off[0]) and torch.equal(on[1], off[1]), f"{name}: inference differs"
    if dtype == torch.bfloat16:
        return
    wf, wx = torch.randn_like(feats), torch.randn_like(x)

    def train():
        fe, co = feats.clone().requires_grad_(), x.clone().requires_grad_()
        lay.zero_grad()
        with torch.enable_grad():
            f, xo = lay(fe, co, mask=m, ptr=ptr)
            ((f * wf).sum() + (xo * wx).sum()).backward()
        return [f.detach(), xo.detach(), fe.grad, co.grad] + [p.grad.clone() for p in lay.parameters()
                                                                if p.grad is not None]
    on, off = _on_off(monkeypatch, train)
    assert torch.equal(on[0], off[0]) and torch.equal(on[1], off[1]), f"{name}: training outputs differ"
    # the same lists (the outputs are bit-identical); the gradients to the rounding of the backward's atomic sums,
    # whose order varies from run to run of the same call
    for i, (a, b) in enumerate(zip(on[2:], off[2:])):
        scale = b.abs().max().item()
        assert (a - b).abs().max().item() <= (1e-12 if dtype == torch.float64 else 1e-4) * max(scale, 1e-30), i


def test_network_grids_on_equal_grids_off(monkeypatch):
    from egnn_pytorch_b200 import EGNN_Network
    torch.manual_seed(0)
    net = EGNN_Network(num_tokens=10, dim=16, depth=2, num_nearest_neighbors=16, num_positions=1024).to(DEV)
    sizes, ptr, x, mask = _big_batch(torch.float32, 3)
    tok = torch.randint(0, 10, (1, x.shape[1]), device=DEV)
    with torch.no_grad():
        on, off = _on_off(monkeypatch, lambda: net(tok, x, mask=mask, ptr=ptr))
    assert torch.equal(on[0], off[0]) and torch.equal(on[1], off[1])


def test_capture_replays_like_eager(monkeypatch):
    from egnn_pytorch_b200 import knn_neighbors
    from egnn_pytorch_b200.graphs import GraphedForward
    monkeypatch.setenv(ENV["knn"], "250")
    sizes, ptr, x, mask = _big_batch(torch.float32, 7)
    ptr_dev = ptr.to(DEV, torch.int32)
    lay = _layer(torch.float32, 16, math.inf).eval()
    feats = torch.randn(1, x.shape[1], 16, device=DEV)
    fast = GraphedForward(lay, feats, x, mask=mask, ptr=ptr_dev)
    got = [t.clone() for t in fast(feats, x)]
    with torch.no_grad():
        want = lay(feats, x, mask=mask, ptr=ptr_dev)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])

    eager = knn_neighbors(x, 32, ptr=ptr_dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        knn_neighbors(x, 32, ptr=ptr_dev)                         # warm-up: workspace and ptr check
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            out = knn_neighbors(x, 32, ptr=ptr_dev)
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
