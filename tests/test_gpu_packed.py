"""Packed batches of variable-size graphs (`ptr=`) on the device: the segmented select (csrc/segment_select.cu,
egnn_knn_select_packed*), the list builders, EGNN and EGNN_Network with `ptr`, and a CUDA-graph capture of a packed
layer.

Select: indices and ok bytes equal egnn_knn_select run on each graph alone (B = 1, N = n_g, k' = min(k, n_g)) bit for
bit, shifted by ptr[g]; under a box or a cell, egnn_knn_grid_select on each graph alone (which equals egnn_knn_select's
lists under a lattice bit for bit); and the exact numpy reference of test_packed_host.py, which also fixes the slots past
a graph's size (-1, ok 0) and leaves empty graphs unwritten.  Graph sizes straddle the row tile (SEG_WARPS = 8 rows) and
the staged chunk (SEG_JC = 1024 candidates), held by test_sizes_cross_the_launch_boundaries
(the launch rules are restated here, next to the tests that use them).

Layer: the packed layer's outputs equal the layer run on the packed lists with the mask it used, bit for bit (its
gradients to the rounding of the backward's atomic sums), and the per-graph calls concatenated to 1e-12 of scale in
fp64 (outputs and gradients), to the fp32 gate of util.TOL (gradients: 1e-4 of scale), and to 5e-2 of scale in bf16."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from launch_geometry import ceil_div
import test_gpu_knn_select as KS
from test_gpu_knn_grid import grid_select
from test_packed_host import ref_packed_select
from util import TOL

pytestmark = pytest.mark.gpu

DEV = "cuda"
SIZES = [0, 1, 7, 8, 9, 33, 5, 1023, 0, 1024, 1025, 2100, 64]

# The launch rules of egnn_knn_select_packed (segment_select.cu: SEG_WARPS rows per CTA, SEG_JC candidates staged per
# pass, the grid launched for the bound ceil(T / SEG_WARPS) + G), restated for the coverage check below.
SEG_WARPS, SEG_JC = 8, 1024


def launch_segment_select(sizes):
    """The launch for graphs of `sizes` nodes: ceil(n_g / SEG_WARPS) row tiles per graph (rows in each graph's last
    tile), staging passes of SEG_JC candidates per graph, and the grid bound that the tile count never exceeds."""
    tiles = [ceil_div(n, SEG_WARPS) for n in sizes]
    return dict(tiles=sum(tiles), grid=ceil_div(sum(sizes), SEG_WARPS) + len(sizes),
                last_tile_rows=[n - (t - 1) * SEG_WARPS for n, t in zip(sizes, tiles) if n],
                passes=[ceil_div(n, SEG_JC) for n in sizes])


def _ptr(sizes):
    return torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64)


@pytest.fixture(scope="module")
def lib():
    from egnn_pytorch_b200 import _native
    return _native.load()


def packed_select(lib, x, ptr, k, vr, mask=None, box=None, cell=None):
    """egnn_knn_select_packed(_triclinic) on device tensors x [T, C], ptr [G+1] -> (idx, ok) numpy [T, k].  Outputs are
    poisoned and the workspace filled with garbage first."""
    from egnn_pytorch_b200 import _native as nat
    t, c = x.shape
    g = ptr.numel() - 1
    idx = torch.full((t, k), -7, dtype=torch.int32, device=DEV)
    ok = torch.full((t, k), 7, dtype=torch.uint8, device=DEV)
    nb = C.c_size_t()
    assert lib.egnn_knn_select_packed_workspace_bytes(g, t, c, k, C.byref(nb)) == 0
    ws = torch.randint(0, 255, (nb.value + 256,), dtype=torch.uint8, device=DEV)
    wp = (ws.data_ptr() + 255) // 256 * 256
    p32 = ptr.to(DEV, torch.int32).contiguous()
    m = None if mask is None else mask.to(DEV, torch.uint8).contiguous()
    lat = cell if cell is not None else box
    lat = None if lat is None else lat.to(DEV, x.dtype).contiguous()
    entry = lib.egnn_knn_select_packed_triclinic if cell is not None else lib.egnn_knn_select_packed
    rc = entry(nat.DTYPE_F64 if x.dtype == torch.float64 else nat.DTYPE_F32, g, t, c, k, C.c_void_p(p32.data_ptr()),
               C.c_void_p(x.data_ptr()), None if m is None else C.c_void_p(m.data_ptr()),
               None if lat is None else C.c_void_p(lat.data_ptr()), float(vr), C.c_void_p(idx.data_ptr()),
               C.c_void_p(ok.data_ptr()), C.c_void_p(wp), nb.value, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, rc
    torch.cuda.synchronize()
    return idx.cpu().numpy(), ok.cpu().numpy()


def test_sizes_cross_the_launch_boundaries():
    g = launch_segment_select(SIZES)
    assert g["tiles"] <= g["grid"]
    assert {1, 7, 8} <= set(g["last_tile_rows"])                # partial and full last tiles
    assert {0, 1, 2, 3} <= set(g["passes"])                      # empty graphs, one, two and three staging passes
    assert any(n % SEG_JC == 0 and n for n in SIZES) and any(n % SEG_JC == 1 and n > 1 for n in SIZES)


def make_points(t, c, dtype, rs, kind):
    x = rs.uniform(0, 4, size=(t, c))
    if kind == "ties":
        x = np.floor(x * 2)                                      # a coarse integer lattice: many equal ranks
    x = x.astype(np.float64 if dtype == torch.float64 else np.float32)
    if kind == "nonfinite":
        x[rs.choice(t, 12, replace=False), rs.randint(0, c, 12)] = rs.choice([np.nan, np.inf, -np.inf], 12)
    return x


SELECT_CASES = []
for n_, k_ in enumerate([1, 8, 32, 33, 64, 256]):
    for dt_ in (torch.float32, torch.float64):
        SELECT_CASES.append(dict(k=k_, dtype=dt_, C=[1, 2, 3, 5, 8, 3][n_], kind=["rand", "ties", "nonfinite"][n_ % 3],
                                 mask=(n_ + (dt_ == torch.float64)) % 2 == 1, vr=[math.inf, 0.5][n_ % 2]))


@pytest.mark.parametrize("case", SELECT_CASES, ids=lambda c: f"k{c['k']}-{str(c['dtype'])[6:]}-c{c['C']}-{c['kind']}"
                                                          f"{'-mask' if c['mask'] else ''}-vr{c['vr']}")
def test_select_equals_the_per_graph_select(lib, case):
    k, dtype, c = case["k"], case["dtype"], case["C"]
    rs = np.random.RandomState(k * 7 + c)
    ptr = _ptr(SIZES)
    t = int(ptr[-1])
    xn = make_points(t, c, dtype, rs, case["kind"])
    mn = rs.rand(t) > 0.2 if case["mask"] else None
    x = torch.from_numpy(xn).to(DEV)
    idx, ok = packed_select(lib, x, ptr, k, case["vr"], None if mn is None else torch.from_numpy(mn))
    want_idx, want_ok = ref_packed_select(xn, ptr.numpy(), k, case["vr"], mn)
    assert np.array_equal(idx, want_idx), "lists differ from the exact reference"
    assert np.array_equal(ok.astype(bool), want_ok), "ok bytes differ from the exact reference"
    for g in range(len(SIZES)):
        lo, hi = int(ptr[g]), int(ptr[g + 1])
        if hi == lo:
            continue
        kk = min(k, hi - lo)
        rc, gi, go = KS.gpu_select(xn[None, lo:hi], kk, case["vr"], None if mn is None else mn[None, lo:hi])
        assert rc == 0
        assert np.array_equal(idx[lo:hi, :kk], gi[0] + lo), f"graph {g} ({hi - lo} nodes): lists differ"
        assert np.array_equal(ok[lo:hi, :kk], go[0]), f"graph {g}: ok bytes differ"
        assert (idx[lo:hi, kk:] == -1).all() and (ok[lo:hi, kk:] == 0).all()


LATTICE_CASES = [(torch.float32, 3, 8, "box"), (torch.float64, 2, 64, "box"), (torch.float32, 3, 33, "cell"),
                 (torch.float64, 3, 256, "cell"), (torch.float32, 2, 32, "cell"), (torch.float64, 1, 1, "box")]


@pytest.mark.parametrize("dtype, c, k, lat", LATTICE_CASES)
def test_select_under_a_shared_lattice_equals_the_per_graph_grid_select(lib, dtype, c, k, lat):
    rs = np.random.RandomState(c * 100 + k)
    sizes = [9, 1, 0, 300, 1030, 40]
    ptr = _ptr(sizes)
    t = int(ptr[-1])
    x = torch.from_numpy(make_points(t, c, dtype, rs, "rand")).to(DEV)
    mask = torch.from_numpy(rs.rand(t) > 0.15).to(DEV)
    if lat == "box":
        lattice = torch.tensor([4.0, 0.0, 4.0][:c], dtype=dtype, device=DEV)    # the middle axis aperiodic
        kw = dict(box=lattice)
    else:
        lattice = torch.diag(torch.full((c,), 4.0, dtype=dtype))
        lattice[1, 0] = 1.25
        if c == 3:
            lattice[2, 0], lattice[2, 1] = -0.5, 0.75
        lattice = lattice.to(DEV)
        kw = dict(cell=lattice)
    for vr in (math.inf, 1.5):
        idx, ok = packed_select(lib, x, ptr, k, vr, mask, **kw)
        for g in range(len(sizes)):
            lo, hi = int(ptr[g]), int(ptr[g + 1])
            if hi == lo:
                continue
            kk = min(k, hi - lo)
            one = {key: v.unsqueeze(0) for key, v in kw.items()}
            gi, go = grid_select(lib, x[None, lo:hi].contiguous(), mask[None, lo:hi], kk, vr, **one)
            assert np.array_equal(idx[lo:hi, :kk], gi[0].cpu().numpy() + lo), f"graph {g}: lists differ"
            assert np.array_equal(ok[lo:hi, :kk].astype(bool), go[0].cpu().numpy()), f"graph {g}: ok bytes differ"
            assert (idx[lo:hi, kk:] == -1).all()


# ------------------------------------------------------------------ the builders


@pytest.mark.parametrize("builder, k", [("knn", 8), ("knn", 64), ("radius", 16), ("wide", 40)])
@pytest.mark.parametrize("lattice", [None, "box", "cell"])
def test_builders_equal_the_shifted_per_graph_calls(builder, k, lattice):
    from egnn_pytorch_b200 import knn_neighbors, radius_neighbors, radius_neighbors_wide
    rs = np.random.RandomState(k)
    sizes = [50, 3, 0, 700, 64, 129]
    ptr = _ptr(sizes)
    t = int(ptr[-1])
    xn = make_points(t, 3, torch.float32, rs, "rand")
    xn[5, 0] = np.nan
    x = torch.from_numpy(xn).to(DEV)[None]
    mask = torch.from_numpy(rs.rand(1, t) > 0.1).to(DEV)
    kw = {}
    if lattice == "box":
        kw["box"] = torch.tensor([4.0, 4.0, 0.0], device=DEV)
    elif lattice == "cell":
        kw["cell"] = torch.tensor([[4.0, 0, 0], [1.0, 4.0, 0], [0.5, -0.5, 4.0]], device=DEV)
    call = {"knn": lambda xx, m, **a: knn_neighbors(xx, k, mask=m, **a),
            "radius": lambda xx, m, **a: radius_neighbors(xx, 0.9, k, mask=m, **a),
            "wide": lambda xx, m, **a: radius_neighbors_wide(xx, 1.3, k, mask=m, **a)}[builder]
    for m in (None, mask):
        got = call(x, m, ptr=ptr, **kw).cpu()
        assert got.shape == (1, t, k)
        for g, n in enumerate(sizes):
            lo, hi = int(ptr[g]), int(ptr[g + 1])
            if n < k:
                continue
            want = call(x[:, lo:hi], None if m is None else m[:, lo:hi], **kw).cpu()
            want = torch.where(want >= 0, want + lo, want)
            assert torch.equal(got[:, lo:hi], want), f"{builder} graph {g} ({n} nodes), mask {m is not None}"


# ------------------------------------------------------------------ the layer


def _layer(dtype, k, pool="sum", vr=math.inf, dim=16, seed=0):
    from egnn_pytorch_b200 import EGNN
    torch.manual_seed(seed)
    lay = EGNN(dim=dim, m_dim=16, num_nearest_neighbors=k, valid_radius=vr, m_pool_method=pool, init_eps=0.1,
               norm_coors=True)
    return lay.to(DEV, dtype)


def packed_lists(lay, coors, ptr, mask):
    """The lists and mask a packed layer runs with, rebuilt from the raw select (kNN) or index arithmetic (dense)."""
    t = coors.shape[1]
    sizes = (ptr[1:] - ptr[:-1]).tolist()
    cdt = torch.float64 if coors.dtype == torch.float64 else torch.float32
    if lay.num_nearest_neighbors > 0:
        from egnn_pytorch_b200 import _native
        idx, ok = packed_select(_native.load(), coors[0].to(cdt).contiguous(), ptr, min(lay.num_nearest_neighbors,
                                max(sizes)), lay.valid_radius, None if mask is None else mask[0])
        if mask is not None:
            idx = np.where(ok == 0, -1, idx)
    else:
        idx = np.full((t, max(sizes)), -1, np.int64)
        for g, n in enumerate(sizes):
            lo = int(ptr[g])
            idx[lo:lo + n, :n] = lo + np.arange(n)
    m = mask if mask is not None else torch.ones(1, t, dtype=torch.bool, device=DEV)
    return torch.from_numpy(np.ascontiguousarray(idx)).to(DEV, torch.int32)[None], m


def per_graph(lay, feats, coors, ptr, mask):
    """The layer on every graph alone (k = n_g where a graph has fewer than k nodes), outputs concatenated."""
    k0 = lay.num_nearest_neighbors
    fs, xs = [], []
    try:
        for g in range(ptr.numel() - 1):
            lo, hi = int(ptr[g]), int(ptr[g + 1])
            if hi == lo:
                continue
            lay.num_nearest_neighbors = min(k0, hi - lo)
            f, x = lay(feats[:, lo:hi], coors[:, lo:hi], mask=None if mask is None else mask[:, lo:hi])
            fs.append(f)
            xs.append(x)
    finally:
        lay.num_nearest_neighbors = k0
    return torch.cat(fs, 1), torch.cat(xs, 1)


def _scale_close(got, want, rel, what):
    got, want = got.double(), want.double()
    scale = want.abs().max().item()
    err = (got - want).abs().max().item()
    assert err <= rel * scale, f"{what}: max|err| {err:.3e} > {rel:g} x scale {scale:.3e}"


LAYER_CASES = [("knn", 8, "sum", False), ("knn", 16, "mean", False), ("radius_mask", 8, "mean", True),
               ("dense", 0, "sum", False), ("dense", 0, "mean", True), ("knn_small", 40, "mean", True)]
LAYER_SIZES = [30, 1, 0, 9, 70, 17, 5]


def _layer_inputs(dtype, mask_on, seed):
    rs = np.random.RandomState(seed)
    ptr = _ptr(LAYER_SIZES)
    t = int(ptr[-1])
    feats = torch.from_numpy(rs.standard_normal((1, t, 16))).to(DEV, dtype)
    coors = torch.from_numpy(rs.uniform(0, 3, (1, t, 3))).to(DEV, torch.float64 if dtype == torch.float64 else
                                                               torch.float32)
    mask = torch.from_numpy(rs.rand(1, t) > 0.2).to(DEV) if mask_on else None
    return feats, coors, ptr, mask


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32, torch.bfloat16])
@pytest.mark.parametrize("name, k, pool, mask_on", LAYER_CASES)
def test_layer_forward(dtype, name, k, pool, mask_on):
    lay = _layer(dtype, k, pool, vr=1.2 if name == "radius_mask" else math.inf)
    feats, coors, ptr, mask = _layer_inputs(dtype, mask_on, k + 3)
    with torch.no_grad():
        f, x = lay(feats, coors, mask=mask, ptr=ptr)
        lists, m = packed_lists(lay, coors, ptr, mask)
        f2, x2 = lay(feats, coors, mask=m, neighbors=lists)
        assert torch.equal(f, f2) and torch.equal(x, x2), "packed layer != the layer on its lists"
        fw, xw = per_graph(lay, feats, coors, ptr, mask)
    rel = {torch.float64: 1e-12, torch.float32: None, torch.bfloat16: 5e-2}[dtype]
    if rel is None:
        torch.testing.assert_close(f, fw, **TOL[torch.float32])
        torch.testing.assert_close(x, xw, **TOL[torch.float32])
    else:
        _scale_close(f, fw, rel, "feats")
        _scale_close(x, xw, rel, "coors")


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("name, k, pool, mask_on", LAYER_CASES)
def test_layer_training(dtype, name, k, pool, mask_on):
    lay = _layer(dtype, k, pool, vr=1.2 if name == "radius_mask" else math.inf, seed=1)
    feats0, coors0, ptr, mask = _layer_inputs(dtype, mask_on, k + 5)
    rs = np.random.RandomState(9)
    wf = torch.from_numpy(rs.standard_normal(feats0.shape)).to(DEV, dtype)
    wx = torch.from_numpy(rs.standard_normal(coors0.shape)).to(DEV, coors0.dtype)

    def grads(fn):
        feats, coors = feats0.clone().requires_grad_(), coors0.clone().requires_grad_()
        lay.zero_grad()
        with torch.enable_grad():
            f, x = fn(feats, coors)
            ((f * wf).sum() + (x * wx).sum()).backward()
        return [f.detach(), x.detach(), feats.grad, coors.grad] + [p.grad.clone() for p in lay.parameters()
                                                                    if p.grad is not None]

    got = grads(lambda fe, co: lay(fe, co, mask=mask, ptr=ptr))
    lists, m = packed_lists(lay, coors0, ptr, mask)
    same = grads(lambda fe, co: lay(fe, co, mask=m, neighbors=lists))
    # the outputs bit for bit; the gradients to the rounding of the backward's atomic sums, whose order varies from
    # run to run of the same call
    assert torch.equal(got[0], same[0]) and torch.equal(got[1], same[1]), "packed training != training on its lists"
    for i, (a, b) in enumerate(zip(got[2:], same[2:])):
        _scale_close(a, b, 1e-12 if dtype == torch.float64 else 1e-5, f"gradient {i} on the packed lists")
    want = grads(lambda fe, co: per_graph(lay, fe, co, ptr, mask))
    for i, (a, b) in enumerate(zip(got, want)):
        if dtype == torch.float64:
            _scale_close(a, b, 1e-12, f"tensor {i}")
        else:
            _scale_close(a, b, 1e-4, f"tensor {i}")


def test_graphed_packed_layer_replays_like_eager():
    from egnn_pytorch_b200.graphs import GraphedForward
    lay = _layer(torch.float32, 8).eval()
    feats, coors, ptr, mask = _layer_inputs(torch.float32, True, 4)
    ptr_dev = ptr.to(DEV, torch.int32)
    fast = GraphedForward(lay, feats, coors, mask=mask, ptr=ptr_dev)
    for s in range(2):
        f2 = torch.randn_like(feats)
        x2 = coors + 0.1 * s * torch.randn_like(coors)
        got = [t.clone() for t in fast(f2, x2)]
        with torch.no_grad():
            want = lay(f2, x2, mask=mask, ptr=ptr_dev)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


# ------------------------------------------------------------------ the network


@pytest.mark.parametrize("train", [False, True])
@pytest.mark.parametrize("k", [6, 0])
def test_network_equals_per_graph_calls(train, k):
    from egnn_pytorch_b200 import EGNN_Network
    torch.manual_seed(3)
    net = EGNN_Network(depth=3, dim=16, num_tokens=11, num_positions=80, num_nearest_neighbors=k, m_dim=16,
                       init_eps=0.1).to(DEV, torch.float64)
    net.train(train)
    rs = np.random.RandomState(5)
    ptr = _ptr(LAYER_SIZES)
    t = int(ptr[-1])
    tok = torch.from_numpy(rs.randint(0, 11, (1, t))).to(DEV)
    coors0 = torch.from_numpy(rs.uniform(0, 3, (1, t, 3))).to(DEV)
    mask = torch.from_numpy(rs.rand(1, t) > 0.2).to(DEV)

    def run(fn):
        coors = coors0.clone().requires_grad_(train)
        net.zero_grad()
        with torch.set_grad_enabled(train):
            f, x = fn(coors)
            if train:
                (f.sum() + (x * x).sum()).backward()
        out = [f.detach(), x.detach()]
        return out + ([coors.grad] + [p.grad.clone() for p in net.parameters() if p.grad is not None] if train else [])

    got = run(lambda co: net(tok, co, mask=mask, ptr=ptr))

    def each(co):
        fs, xs = [], []
        for g in range(len(LAYER_SIZES)):
            lo, hi = int(ptr[g]), int(ptr[g + 1])
            if hi == lo:
                continue
            for lay in net.modules():
                if hasattr(lay, "num_nearest_neighbors"):
                    lay.num_nearest_neighbors = min(k, hi - lo)
            f, x = net(tok[:, lo:hi], co[:, lo:hi], mask=mask[:, lo:hi])
            fs.append(f)
            xs.append(x)
        for lay in net.modules():
            if hasattr(lay, "num_nearest_neighbors"):
                lay.num_nearest_neighbors = k
        return torch.cat(fs, 1), torch.cat(xs, 1)

    want = run(each)
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        _scale_close(a, b, 1e-12, f"tensor {i}")


def test_network_rejects_a_graph_longer_than_num_positions():
    from egnn_pytorch_b200 import EGNN_Network
    net = EGNN_Network(depth=1, dim=8, num_tokens=5, num_positions=40).to(DEV)
    tok, coors = torch.randint(0, 5, (1, 60), device=DEV), torch.randn(1, 60, 3, device=DEV)
    net(tok, coors, ptr=torch.tensor([0, 30, 60]))                       # every graph fits
    with pytest.raises(AssertionError, match="number of positions"):
        net(tok, coors, ptr=torch.tensor([0, 10, 60]))
