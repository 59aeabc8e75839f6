"""Periodic boundaries in triclinic cells: `EGNN.forward(..., cell=)`, `EGNN_Network.forward(..., cell=)` and
`radius_neighbors(..., cell=)` (egnn_layer_forward_triclinic / egnn_layer_backward_triclinic /
egnn_radius_select_triclinic).

The triclinic restatement is tests/torch_reference.py's float64 layer with the sequential cell wrap in place of the
box wrap (`tri_layer`): for c = C-1 .. 0, n = round_half_even(r_c / L_c), r_d -= cell[c, d] n for d <= c.  It is
pinned without trusting its own wrap: a diagonal cell equals the box restatement; on a 3^C supercell of lattice images,
where every central node lists the nearest image of each partner, the existing edge-list oracles give its outputs and
gradients; its kNN selection equals a stable argsort of distances found by brute force over the 3^C images.

Inputs keep every wrap decision at least 1e-3 away from 1/2 (`wrap_margin`, the actual sequential wrap), and kNN
inputs are tie-free at rank k, so fp32 / bf16 rounding picks the image and the neighbours the fp64 restatement picks.

CPU: the restatement, argument errors, the new symbols.
GPU: a diagonal cell equals `box=` bit for bit on every path; tilted cells against the restatement on every path;
lattice-shift invariance; the README rotation recipe; gradients; the cell grid against the all-pairs select;
EGNN_Network; CUDA-graph replay after an in-place cell change."""
import contextlib
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

import cases
import torch_reference as R
import util
from oracle import egnn_oracle as O
from oracle import egnn_oracle_grad as G

NEVER = str(2 ** 40)


# ----------------------------------------------------------------------------- the triclinic restatement


def cell_wrap(rel, cell):
    """Sequential wrap of rel [..., C] under lower-triangular cells broadcastable to [..., C, C] (torch, any float)."""
    c_dim = rel.shape[-1]
    diag = torch.diagonal(cell, dim1=-2, dim2=-1)
    per = (diag > 0) & torch.isfinite(diag)
    L = torch.where(per, diag, torch.zeros_like(diag))
    inv = torch.where(per, 1.0 / torch.where(per, diag, torch.ones_like(diag)), torch.zeros_like(diag))
    r = list(rel.unbind(-1))
    for c in reversed(range(c_dim)):
        n = torch.round(r[c] * inv[..., c])           # half to even, as rint; no gradient (piecewise constant)
        for d in range(c + 1):
            coef = L[..., c] if d == c else cell[..., c, d]
            r[d] = r[d] - coef * n
    return torch.stack(r, -1)


@contextlib.contextmanager
def _cell_geometry():
    """torch_reference.layer with `box` read as a cell: [C, C] or [B, C, C] -> the sequential cell wrap."""
    saved = R.wrap, R.box_bc
    R.box_bc = lambda cell, b, c: None if cell is None else R._t(cell).expand(b, c, c)
    R.wrap = cell_wrap
    try:
        yield
    finally:
        R.wrap, R.box_bc = saved


def tri_layer(P, cfg, feats, coors, edges=None, mask=None, adj=None, cell=None, neighbors=None, slot_edges=None):
    with _cell_geometry():
        return R.layer(P, cfg, feats, coors, edges, mask, adj, cell, neighbors, slot_edges)


def tri_grads(case, cell, gf, gx):
    with _cell_geometry():
        return R.layer_grads(case, cell, gf, gx)


def cell_bc(cell, B, Cd):
    return np.broadcast_to(np.asarray(cell, np.float64), (B, Cd, Cd))


def wrap_margin(coors, cell):
    """Smallest distance from 1/2 of r_c / L_c at every decision of the sequential wrap, over all pairs and periodic
    axes (a fraction of L_c)."""
    x = np.asarray(coors, np.float64)
    B, N, Cd = x.shape
    A = cell_bc(cell, B, Cd)
    r = x[:, :, None] - x[:, None]
    m = np.ones((B, N, N))
    for c in reversed(range(Cd)):
        Lc = A[:, c, c]
        per = np.isfinite(Lc) & (Lc > 0)
        t = r[..., c] / np.where(per, Lc, 1.0)[:, None, None]
        m = np.where(per[:, None, None], np.minimum(m, np.abs(np.abs(t - np.rint(t)) - 0.5)), m)
        n = np.where(per[:, None, None], np.rint(t), 0.0)
        r[..., :c + 1] -= n[..., None] * np.where(per[:, None], A[:, c, :c + 1], 0.0)[:, None, None, :]
    return m


def wrapped_d2(x, cell):
    """Squared length of the sequentially wrapped pair vector, float64 [B, N, N]."""
    x = torch.as_tensor(np.asarray(x, np.float64))
    B, N, Cd = x.shape
    return (cell_wrap(x[:, :, None] - x[:, None], torch.as_tensor(cell_bc(cell, B, Cd).copy())[:, None, None]) ** 2).sum(-1)


def make_cell(kind, B, rs):
    """Lower-triangular cells: `tilt` (tilts up to 0.5 of the diagonal), `tilt09` (one tilt of 0.9), `per_graph` (a
    different tilted cell per graph), `hex_slab` (hexagonal, z aperiodic), `c2` (a 2-D oblique cell)."""
    def tilted(Ls, t):
        A = np.diag(np.asarray(Ls, np.float64))
        for r in range(1, len(Ls)):
            for c in range(r):
                A[r, c] = rs.uniform(-t, t) * A[c, c]
        return A
    if kind == "tilt":
        return tilted([3.0, 3.2, 3.5], 0.5)
    if kind == "tilt09":
        A = tilted([3.0, 3.2, 3.5], 0.3)
        A[2, 0] = 0.9 * A[0, 0]
        return A
    if kind == "per_graph":
        return np.stack([tilted(rs.uniform(2.8, 3.6, 3), 0.5) for _ in range(B)])
    if kind == "hex_slab":
        a = 3.0
        return np.array([[a, 0, 0], [a / 2, a * np.sqrt(3) / 2, 0], [0, 0, np.inf]])
    if kind == "c2":
        return tilted([3.0, 2.8], 0.5)
    raise KeyError(kind)


def cell_coors(rs, B, N, cell, shift=2, margin=1e-3, dtype=torch.float64):
    """Fractional positions u in [0, 1)^C (an aperiodic axis: [0, 3)), moved by whole lattice vectors in [-shift, shift],
    x = u A.  Nodes in a pair whose wrap decision lies within `margin` of 1/2 (after rounding to `dtype`) are drawn
    again."""
    Cd = np.shape(cell)[-1]
    A = cell_bc(cell, B, Cd)
    per = np.isfinite(np.diagonal(A, axis1=1, axis2=2)) & (np.diagonal(A, axis1=1, axis2=2) > 0)
    Af = np.where(np.isfinite(A), A, 0.0) + np.where(per, 0.0, 1.0)[:, :, None] * np.eye(Cd)   # aperiodic: unit axis
    u = rs.uniform(0, 1, (B, N, Cd)) * np.where(per, 1.0, 3.0)[:, None, :]

    def place(u):
        s = u + rs.randint(-shift, shift + 1, u.shape) * per[:, None, :]
        return util.rounded(np.einsum("bnk,bkd->bnd", s, Af), dtype)
    x = place(u)
    for _ in range(200):
        m = wrap_margin(x, util.rounded(cell, dtype))
        bad = (m < margin).any(-1)
        if not bad.any():
            return x
        u2 = rs.uniform(0, 1, u.shape) * np.where(per, 1.0, 3.0)[:, None, :]
        x = np.where(bad[..., None], place(u2), x)
    raise AssertionError("could not place the nodes off the wrap boundaries")


# name: (layer cfg, B, N, cell kind, mask)
TCASES = {
    "dense_tilt":        (dict(dim=16), 2, 40, "tilt", None),
    "dense_tilt09_soft": (dict(dim=16, soft_edges=True, m_pool_method="mean"), 2, 33, "tilt09", "padded"),
    "dense_per_graph_edges": (dict(dim=16, edge_dim=2, fourier_features=1, norm_coors=True), 3, 30, "per_graph", "random"),
    "dense_hex_slab":    (dict(dim=16), 2, 36, "hex_slab", None),
    "dense_c2":          (dict(dim=8), 2, 30, "c2", None),
    "knn_k8":            (dict(dim=16, num_nearest_neighbors=8, valid_radius=2.0), 2, 50, "tilt", "padded"),
    "knn_k16_edges":     (dict(dim=16, edge_dim=3, num_nearest_neighbors=16), 2, 60, "per_graph", None),
    "knn_k33":           (dict(dim=8, num_nearest_neighbors=33), 1, 70, "tilt09", "padded"),
    "knn_c2_fourier":    (dict(dim=16, fourier_features=1, num_nearest_neighbors=6), 2, 40, "c2", None),
    "knn_hex_slab":      (dict(dim=16, num_nearest_neighbors=8), 2, 40, "hex_slab", "full"),
}
BF16_OK = set(TCASES) - {"knn_k33"}


def build(name, seed=0, dtype=torch.float64):
    cfg, B, N, kind, mask = TCASES[name]
    Cd = 2 if kind == "c2" else 3
    spec = dict(kind="layer", cfg=cfg, B=B, N=N, C=Cd, seed=910 + seed, init="xavier", mask=mask or "none")
    case = cases.build_case(spec)
    rs = np.random.RandomState(710 + seed)
    cell = make_cell(kind, B, rs)
    cdt = torch.float64 if dtype == torch.float64 else torch.float32
    cell = util.rounded(cell, cdt)
    case["inputs"]["coors"] = cell_coors(rs, B, N, cell, dtype=cdt)
    if dtype == torch.bfloat16:
        case["params"] = {k: util.rounded(v, torch.bfloat16) for k, v in case["params"].items()}
        for k in ("feats", "edges"):
            if k in case["inputs"]:
                case["inputs"][k] = util.rounded(case["inputs"][k], torch.bfloat16)
    return case, cell


def knn_gap(case, cell):
    cfg, ins = case["cfg"], case["inputs"]
    k = cfg["num_nearest_neighbors"]
    n = ins["coors"].shape[1]
    if k == 0 or k >= n:
        return 1.0
    d = wrapped_d2(ins["coors"], cell)
    if ins.get("mask") is not None:
        mk = torch.as_tensor(ins["mask"])
        d = d.masked_fill(~(mk[:, :, None] & mk[:, None, :]), 1e5)
    s = torch.sort(d, -1).values
    live = s[..., k] < 1e5
    return float(((s[..., k] - s[..., k - 1]) / s[..., k].clamp_min(1e-12))[live].min())


# ----------------------------------------------------------------------------- CPU: pin the restatement


@pytest.mark.parametrize("name", ["dense_basic", "dense_mask_padded", "dense_fourier", "knn_basic", "knn_edges_mask",
                                  "knn_radius_mask"])
def test_a_diagonal_cell_is_the_box_restatement(name):
    case = cases.build_case(cases.SPECS[name])
    ins = case["inputs"]
    Cd = ins["coors"].shape[-1]
    assert Cd == 3                                     # (cells have C in {2, 3}; these cases are all 3-D)
    L = np.array([2.0, 2.5, np.inf])
    want = R.layer(case["params"], case["cfg"], ins["feats"], ins["coors"], ins.get("edges"), ins.get("mask"),
                   ins.get("adj_mat"), L)
    got = tri_layer(case["params"], case["cfg"], ins["feats"], ins["coors"], ins.get("edges"), ins.get("mask"),
                    ins.get("adj_mat"), np.diag(L))
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def supercell(x, cell, partners, per=None):
    """3^C lattice images of every graph (aperiodic axes are not copied) and, for each central node i and partner j, the
    image of j nearest to x_i.  -> (coors [B, S*N, C], neighbours [B, S*N, P]); central node i at index i.  `per`: the
    periodic axes (default: from the diagonal of a lower-triangular cell)."""
    B, N, Cd = x.shape
    A = cell_bc(cell, B, Cd)
    diag = np.diagonal(A, axis1=1, axis2=2)
    if per is None:
        per = (np.isfinite(diag) & (diag > 0))[0]
    Af = np.where(np.isfinite(A), A, 0.0)
    shifts = [np.array(s, np.float64) for s in itertools.product(*[(0, -1, 1) if p else (0,) for p in per])]
    xs = np.concatenate([x + np.einsum("k,bkd->bd", s, Af)[:, None, :] for s in shifts], 1)
    S = len(shifts)
    nb = np.full((B, S * N, partners.shape[-1]), -1, np.int64)
    for b in range(B):
        for i in range(N):
            for t, j in enumerate(partners[b, i]):
                d = ((xs[b, j::N] - x[b, i]) ** 2).sum(-1)
                s = int(np.argmin(d))
                assert np.sort(d)[1] - d[s] > 1e-6                  # a unique nearest image
                nb[b, i, t] = s * N + j
    return xs, nb


SUPER = [("dense_tilt", dict(dim=8, edge_dim=2, soft_edges=True), "tilt", "padded", None),
         ("dense_tilt09_normc", dict(dim=8, m_pool_method="mean", norm_coors=True, fourier_features=1), "tilt09", None, None),
         ("dense_hex_slab", dict(dim=8, coor_weights_clamp_value=0.3), "hex_slab", "random", None),
         ("knn_tilt", dict(dim=8, edge_dim=1, num_nearest_neighbors=4), "tilt", None, 4),
         ("knn_c2", dict(dim=8, num_nearest_neighbors=3), "c2", None, 3)]


@pytest.mark.parametrize("name,cfg,kind,mask,k", SUPER, ids=[s[0] for s in SUPER])
def test_supercell_of_images_gives_the_triclinic_forward_and_gradient(name, cfg, kind, mask, k):
    """Nodes clustered within 0.2 min L_c of a lattice point and then wrapped into the cell: every pair's minimum image is
    shorter than min L_c / 2, so the nearest image among the 3^C is the one the wrap must find."""
    B, N = 2, 6
    cell = make_cell(kind, B, np.random.RandomState(3))
    Cd = cell.shape[-1]
    spec = dict(kind="layer", cfg=cfg, B=B, N=N, C=Cd, seed=78, init="xavier", mask=mask or "none")
    case = cases.build_case(spec)
    rs = np.random.RandomState(6)
    diag = np.diag(cell)
    per = np.isfinite(diag) & (diag > 0)
    Lmin = diag[per].min()
    y = rs.uniform(-1, 1, (B, N, Cd))
    y = y / np.linalg.norm(y, axis=-1, keepdims=True) * rs.uniform(0, 0.2 * Lmin, (B, N, 1))
    Af = np.where(np.isfinite(cell), cell, 0.0) + np.diag(np.where(per, 0.0, 1.0))
    s = np.linalg.solve(Af.T, y.reshape(-1, Cd).T).T.reshape(B, N, Cd)           # fractional coordinates
    s = np.where(per, s - np.floor(s), s)                                       # wrapped into the cell
    x = s @ Af
    case["inputs"]["coors"] = x
    assert wrap_margin(x, cell).min() > 0.05
    ins, P, lc = case["inputs"], case["params"], case["cfg"]
    d = wrapped_d2(x, cell).numpy()
    partners = np.broadcast_to(np.arange(N), (B, N, N)) if k is None else np.argsort(d, -1, kind="stable")[..., :k]
    xs, nb = supercell(x, cell, partners)
    S = xs.shape[1] // N
    tile = lambda a, ax: np.concatenate([a] * S, ax)
    f = tile(ins["feats"], 1)
    m = None if ins.get("mask") is None else tile(ins["mask"], 1)
    e = None if ins.get("edges") is None else tile(tile(ins["edges"], 1), 2)
    got = tri_layer(P, lc, ins["feats"], x, ins.get("edges"), ins.get("mask"), None, cell)
    lcfg = dict(lc, num_nearest_neighbors=nb.shape[-1])
    want = O.egnn_layer_forward_edge_list(P, lcfg, f, xs, nb, e, m)
    assert np.abs(got[0].numpy() - want[0][:, :N]).max() <= 1e-12
    assert np.abs(got[1].numpy() - want[1][:, :N]).max() <= 1e-12

    gf, gx = rs.randn(B, N, lc["dim"]), rs.randn(B, N, Cd)
    g = tri_grads(case, cell, gf, gx)
    pad = lambda a: np.concatenate([a, np.zeros((B, (S - 1) * N) + a.shape[2:])], 1)
    gs = G.egnn_layer_backward(P, lcfg, f, xs, e, m, None, pad(gf), pad(gx), neighbors=nb)
    fold = lambda a, ax: sum(np.take(a, range(t * N, (t + 1) * N), axis=ax) for t in range(S))
    want = {"in.feats": fold(gs["feats"], 1), "in.coors": fold(gs["coors"], 1)}
    if e is not None:
        want["in.edges"] = fold(fold(gs["edges"], 1), 2)
    want.update({f"p.{k2}": v for k2, v in gs["params"].items()})
    tol = 1e-7 if lc["norm_coors"] else 1e-11
    util.compare(g, want, tol, f"{name}: triclinic restatement gradient vs supercell gradient oracle")


@pytest.mark.parametrize("name", ["knn_k8", "knn_k16_edges", "knn_c2_fourier", "knn_hex_slab", "knn_k33"])
def test_triclinic_knn_selection_is_a_stable_argsort_of_brute_force_image_distances(name):
    """For every pair whose minimum image is shorter than min L_c / 2 the restatement's rank equals the smallest squared
    distance over the 3^C images; its selection is the stable argsort of those ranks."""
    case, cell = build(name)
    x = np.asarray(case["inputs"]["coors"])
    B, N, Cd = x.shape
    A = cell_bc(cell, B, Cd)
    diag = np.diagonal(A, axis1=1, axis2=2)
    per = np.isfinite(diag) & (diag > 0)
    Af = np.where(np.isfinite(A), A, 0.0)
    rel = x[:, :, None] - x[:, None]
    best = np.full((B, N, N), np.inf)
    for s in itertools.product((-1, 0, 1), repeat=Cd):
        t = np.einsum("k,bkd->bd", np.asarray(s, np.float64), Af * per[:, :, None])
        best = np.minimum(best, ((rel - t[:, None, None, :]) ** 2).sum(-1))
    d = wrapped_d2(x, cell).numpy()
    Lmin = np.where(per, diag, np.inf).min(-1)[:, None, None]
    near = best < (Lmin / 2) ** 2
    assert near.mean() > 0.05
    assert np.allclose(d[near], best[near], rtol=1e-12, atol=1e-12)
    k = case["cfg"]["num_nearest_neighbors"]
    dm = np.where(near, best, d)
    if case["inputs"].get("mask") is not None:
        mk = case["inputs"]["mask"]
        dm = np.where(mk[:, :, None] & mk[:, None, :], dm, 1e5)
    want = np.argsort(dm, -1, kind="stable")[..., :k]
    got, _ = R.select(case["cfg"], torch.as_tensor(d), case["inputs"].get("mask"), None)     # the restatement's ranks
    assert (got.numpy() == want).all()
    assert knn_gap(case, cell) > 1e-5


@pytest.mark.parametrize("name", sorted(TCASES))
def test_inputs_keep_wrap_decisions_off_one_half_and_knn_ranks_tie_free(name):
    for dtype in (torch.float64, torch.float32, torch.bfloat16):
        case, cell = build(name, dtype=dtype)
        assert wrap_margin(case["inputs"]["coors"], cell).min() >= 1e-3
        assert knn_gap(case, cell) > 1e-5


def _layer():
    from egnn_pytorch_b200 import EGNN
    return EGNN(dim=8)


GOOD = torch.tensor([[3.0, 0, 0], [1.0, 3.0, 0], [0.5, -1.0, 3.0]])


def _with(idx, v, base=GOOD):
    t = base.clone()
    t[idx] = v
    return t


@pytest.mark.parametrize("bad,msg", [
    (torch.ones(3), "shape"), (torch.ones(2, 2), "shape"), (torch.ones(3, 3, 3), "shape"),
    (GOOD.to(torch.int64), "float"), ([[3.0, 0, 0], [0, 3.0, 0], [0, 0, 3.0]], "float"),
    (_with((0, 1), 0.5), "lower-triangular"), (_with((1, 2), float("nan")), "lower-triangular"),
    (_with((2, 1), float("nan")), "finite"), (_with((2, 0), float("inf")), "finite"),
    (_with((1, 1), -3.0), ">= 0"), (_with((2, 2), float("nan")), ">= 0"),
    (_with((2, 2), float("inf")), "aperiodic"), (_with((1, 1), 0.0), "aperiodic"),
    (GOOD.clone().requires_grad_(True), "requires_grad")])
def test_cell_misuse_raises_before_anything_launches(bad, msg):
    f, x = torch.randn(2, 5, 8), torch.randn(2, 5, 3)
    with pytest.raises(ValueError, match=msg):
        _layer()(f, x, cell=bad)


def test_cell_needs_two_or_three_coordinates_and_excludes_box():
    with pytest.raises(ValueError, match="C = 2 or 3"):
        _layer()(torch.randn(1, 4, 8), torch.randn(1, 4, 4), cell=torch.eye(4))
    with pytest.raises(ValueError, match="not both"):
        _layer()(torch.randn(1, 4, 8), torch.randn(1, 4, 3), box=torch.ones(3), cell=GOOD)
    from egnn_pytorch_b200 import radius_neighbors, EGNN_Network
    with pytest.raises(ValueError, match="not both"):
        radius_neighbors(torch.randn(1, 4, 3), 1.0, 2, box=torch.ones(3), cell=GOOD)
    with pytest.raises(ValueError, match="lower-triangular"):
        radius_neighbors(torch.randn(1, 4, 3), 1.0, 2, cell=GOOD.T.contiguous())
    with pytest.raises(ValueError, match="requires_grad"):
        EGNN_Network(depth=1, dim=8)(torch.randn(1, 4, 8), torch.randn(1, 4, 3), cell=GOOD.clone().requires_grad_(True))
    # a hexagonal slab is a valid cell
    from egnn_pytorch_b200.egnn import _check_cell
    _check_cell(torch.tensor([[3.0, 0, 0], [1.5, 2.6, 0], [0, 0, float("inf")]]), 1, 3, {})


def test_cell_check_follows_the_tensor_and_its_version():
    from egnn_pytorch_b200.egnn import _check_cell
    cache = {}
    good = GOOD.clone()
    _check_cell(good, 2, 3, cache)
    _check_cell(good, 2, 3, cache)
    good[0, 2] = 1.0                                          # an in-place write bumps the version
    with pytest.raises(ValueError, match="lower-triangular"):
        _check_cell(good, 2, 3, cache)


def test_triclinic_symbols_load_through_ctypes():
    from egnn_pytorch_b200 import _native as nat
    lib = nat.load()
    for name in ("egnn_layer_forward_triclinic", "egnn_layer_backward_triclinic", "egnn_radius_select_triclinic"):
        assert name in nat.SYMBOLS and getattr(lib, name).argtypes is not None
    assert lib.egnn_abi_version() == 4
    desc = nat.LayerDesc(abi_version=3, dtype=nat.DTYPE_F32, B=1, N=4, C=3, dim=8, m_dim=16,
                         flags=nat.FLAG_UPDATE_FEATS | nat.FLAG_UPDATE_COORS)
    dummy = C.c_void_p(16)
    assert lib.egnn_layer_forward_triclinic(C.byref(desc), None, None, None, dummy, None, 0, None) == -6
    assert lib.egnn_layer_backward_triclinic(C.byref(desc), None, None, None, dummy, None, None, None, 0, None) == -6
    desc.abi_version = 4
    desc.C = 4                                                # C outside {2, 3}: a shape error, before any pointer
    assert lib.egnn_layer_forward_triclinic(C.byref(desc), None, None, None, dummy, None, 0, None) == -2
    ws = C.c_void_p(256)
    for c in (1, 4):                                          # C outside {2, 3}: a shape error
        assert lib.egnn_radius_select_triclinic(nat.DTYPE_F32, 1, 8, c, 2, dummy, None, dummy, 1.0, dummy, None, ws,
                                                1 << 20, None) == -2


# ----------------------------------------------------------------------------- GPU


DT = {"fp64": torch.float64, "fp32": torch.float32, "bf16": torch.bfloat16}


def _cdt(dtype):
    return torch.float64 if dtype == torch.float64 else torch.float32


def _run(case, dtype, box=None, cell=None, mod=None, **kw):
    mod = mod or util.make_module(case, dtype, device="cuda")
    ins = case["inputs"]
    t = lambda name: util.to_torch(ins.get(name), dtype, "cuda")
    g = lambda a: None if a is None else torch.as_tensor(np.asarray(a), dtype=_cdt(dtype), device="cuda")
    with torch.no_grad():
        out = mod(t("feats"), util.to_torch(ins["coors"], _cdt(dtype), "cuda"), t("edges"), mask=t("mask"),
                  adj_mat=t("adj_mat"), box=g(box), cell=g(cell), **kw)
    return mod, out


def _check(case, out, want, dtype, what):
    if dtype == torch.bfloat16:
        f_scale = max(1e-3, float(np.abs(want[0]).max()))
        c_scale = float(np.abs(want[1] - case["inputs"]["coors"]).max())
        assert util.max_err(out[0], want[0]) <= 1e-2 * f_scale, what
        assert util.max_err(out[1], want[1]) <= 1e-2 * max(c_scale, 1.0), what
    else:
        for o, w, part in ((out[0], want[0], " feats"), (out[1], want[1], " coors")):
            s = max(1.0, float(np.abs(w).max()))
            tol = dict(atol=1e-10 * s, rtol=1e-10) if dtype == torch.float64 else dict(atol=2e-5 * s, rtol=1e-4)
            util.assert_close(o, w, what=what + part, **tol)


# every path: fp64 / fp32 SIMT dense and kNN (warp select k <= 32, block sort k > 32); bf16 tc_pair lean (plain dense)
# and generic (edges / fourier), tc_knn lean, edges and generic (fourier)
DIAG = [("dense_tilt", "fp64"), ("dense_tilt", "fp32"), ("knn_k8", "fp64"), ("knn_k8", "fp32"), ("knn_k33", "fp64"),
        ("knn_k33", "fp32"), ("dense_c2", "fp32"), ("knn_c2_fourier", "fp32"),
        ("dense_tilt", "bf16"), ("dense_per_graph_edges", "bf16"), ("knn_k8", "bf16"), ("knn_k16_edges", "bf16"),
        ("knn_c2_fourier", "bf16"), ("dense_per_graph_edges", "fp64")]


@pytest.mark.gpu
@pytest.mark.parametrize("name,dt", DIAG)
def test_a_diagonal_cell_is_the_box_bit_for_bit(name, dt):
    dtype = DT[dt]
    case, cell = build(name, dtype=dtype)
    B, Cd = case["inputs"]["coors"].shape[0], case["inputs"]["coors"].shape[-1]
    L = np.diagonal(cell_bc(cell, B, Cd), axis1=1, axis2=2).copy()            # [B, C]
    mod, ref = _run(case, dtype, box=L)
    diag = np.stack([np.diag(l) for l in L])
    _, out = _run(case, dtype, cell=diag, mod=mod)
    assert torch.equal(out[0], ref[0]) and torch.equal(out[1], ref[1])
    if dtype == torch.bfloat16:
        assert mod.last_path == "bf16-tc"


PARITY = [(n, d) for n in sorted(TCASES) for d in ("fp64", "fp32", "bf16") if d != "bf16" or n in BF16_OK]


@pytest.mark.gpu
@pytest.mark.parametrize("name,dt", PARITY)
def test_forward_matches_the_triclinic_restatement(name, dt):
    dtype = DT[dt]
    case, cell = build(name, dtype=dtype)
    ins = case["inputs"]
    want = [t.numpy() for t in tri_layer(case["params"], case["cfg"], ins["feats"], ins["coors"], ins.get("edges"),
                                         ins.get("mask"), None, cell)]
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("error" if dtype == torch.bfloat16 else "default")    # no fp32 fallback for bf16
        mod, out = _run(case, dtype, cell=cell)
    if dtype == torch.bfloat16:
        assert mod.last_path == "bf16-tc"
    _check(case, out, want, dtype, f"{name} [{dt}]")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32", "bf16"])
@pytest.mark.parametrize("name", ["dense_tilt", "knn_k8", "dense_c2", "dense_hex_slab"])
def test_lattice_shifts_of_single_nodes(name, dt):
    """Dyadic coordinates and an integer cell: moving nodes by integer combinations of lattice vectors changes no
    feature bit and moves their coordinates by the same shift."""
    dtype = DT[dt]
    case, _ = build(name, dtype=dtype)
    Cd = case["inputs"]["coors"].shape[-1]
    cell = np.array([[4.0, 0, 0], [1.0, 4.0, 0], [-2.0, 1.0, 4.0]])[:Cd, :Cd]
    if name == "dense_hex_slab":
        cell = np.array([[4.0, 0, 0], [2.0, 4.0, 0], [0, 0, np.inf]])
    B, N, _ = case["inputs"]["coors"].shape
    rs0 = np.random.RandomState(6)
    x = rs0.randint(0, 1024, (B, N, Cd)) / 512.0                  # in [0, 2): every pair inside the centred box
    case["inputs"]["coors"] = x
    _, ref = _run(case, dtype, cell=cell)
    rs = np.random.RandomState(1)
    per = np.isfinite(np.diag(cell))
    n = np.zeros_like(x)
    who = rs.uniform(size=(B, N)) < 0.3
    n[who] = rs.randint(-2, 3, (int(who.sum()), Cd)) * per
    shift = n @ np.where(np.isfinite(cell), cell, 0.0)
    case["inputs"]["coors"] = x + shift
    _, out = _run(case, dtype, cell=cell)
    assert torch.equal(out[0], ref[0])
    got = out[1].double().cpu().numpy() - shift
    tol = 1e-12 if dtype == torch.float64 else 1e-5
    assert np.abs(got - ref[1].double().cpu().numpy()).max() <= tol * max(1.0, np.abs(x + shift).max())


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
def test_the_readme_rotation_recipe(dt):
    """A random general cell: rotate to lower-triangular form (QR of cell^T, signs fixed so the diagonal is positive),
    run, rotate back.  The result equals the supercell oracle in the original frame."""
    dtype = DT[dt]
    rs = np.random.RandomState(12)
    B, N, Cd = 1, 6, 3
    cfg = dict(dim=8, edge_dim=0)
    case = cases.build_case(dict(kind="layer", cfg=cfg, B=B, N=N, C=Cd, seed=81, init="xavier"))
    Qr, _ = np.linalg.qr(rs.randn(3, 3))
    lower = np.array([[3.0, 0, 0], [1.2, 3.1, 0], [-0.8, 0.9, 3.3]])
    cell = lower @ Qr.T                                        # a general cell: rows are rotated lattice vectors
    y = rs.uniform(-1, 1, (B, N, Cd))
    y = y / np.linalg.norm(y, axis=-1, keepdims=True) * rs.uniform(0, 0.6, (B, N, 1))
    s = np.linalg.solve(cell.T, y.reshape(-1, Cd).T).T.reshape(B, N, Cd)
    x = (s - np.floor(s)) @ cell                               # clustered, then wrapped into the cell
    # the oracle in the original frame
    xs, nb = supercell(x, cell, np.broadcast_to(np.arange(N), (B, N, N)), per=np.ones(Cd, bool))
    S = xs.shape[1] // N
    f = np.concatenate([case["inputs"]["feats"]] * S, 1)
    want = O.egnn_layer_forward_edge_list(case["params"], dict(cfg, **dict(case["cfg"], num_nearest_neighbors=N)),
                                          f, xs, nb, None, None)
    # the recipe
    net = util.make_module(case, dtype)
    feats = util.to_torch(case["inputs"]["feats"], dtype, "cuda")
    cell = torch.as_tensor(cell, dtype=_cdt(dtype), device="cuda")
    coors = torch.as_tensor(x, dtype=_cdt(dtype), device="cuda")
    # the README's lines, verbatim
    q, r = torch.linalg.qr(cell.T)                  # cell: rows are lattice vectors, any orientation
    s = torch.sign(torch.diagonal(r)); q = q * s    # signs fixed so that the diagonal is positive
    with torch.no_grad():
        fo, xo = net(feats, coors @ q, cell=torch.tril(cell @ q))
    xo = xo @ q.T                                    # back to the original frame
    tol = 1e-10 if dtype == torch.float64 else 1e-4
    assert np.abs(fo.double().cpu().numpy() - want[0][:, :N]).max() <= tol * max(1.0, np.abs(want[0]).max())
    assert np.abs(xo.double().cpu().numpy() - want[1][:, :N]).max() <= tol * max(1.0, np.abs(want[1]).max())


def _gpu_grads(case, cell, dtype):
    mod = util.make_module(case, dtype).requires_grad_(True)
    ins = case["inputs"]
    t = lambda a: util.to_torch(a, dtype, "cuda")
    f, x = t(ins["feats"]).requires_grad_(True), t(ins["coors"]).requires_grad_(True)
    e = t(ins.get("edges"))
    leaves = {"in.feats": f, "in.coors": x}
    if e is not None:
        leaves["in.edges"] = e.requires_grad_(True)
    rs = np.random.RandomState(4)
    gf, gx = rs.randn(*ins["feats"].shape), rs.randn(*ins["coors"].shape)
    with torch.enable_grad():
        fo, xo = mod(f, x, e, mask=t(ins.get("mask")), cell=torch.as_tensor(cell, dtype=dtype, device="cuda"))
        ((fo * t(gf)).sum() + (xo * t(gx)).sum()).backward()
    got = {k: v.grad.double().cpu().numpy() for k, v in leaves.items()}
    got.update({f"p.{k}": (torch.zeros_like(p) if p.grad is None else p.grad).double().cpu().numpy()
                for k, p in mod.named_parameters()})
    return got, gf, gx


@pytest.mark.gpu
@pytest.mark.parametrize("saved", [True, False])
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name", ["dense_tilt09_soft", "dense_per_graph_edges", "knn_k8", "knn_k33", "dense_c2"])
def test_gradients_match_the_restatement(name, dt, saved, monkeypatch):
    if not saved:
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")
    dtype = DT[dt]
    case, cell = build(name, dtype=dtype)
    got, gf, gx = _gpu_grads(case, cell, dtype)
    want = tri_grads(case, cell, gf, gx)
    util.compare(got, want, util.grad_tol(case, dtype), f"{name} [{dt}] saved={saved}")


@pytest.mark.gpu
def test_fp64_gradient_matches_central_finite_differences():
    case, cell = build("dense_tilt09_soft")
    got, gf, gx = _gpu_grads(case, cell, torch.float64)
    ins = case["inputs"]
    mod = util.make_module(case, torch.float64)
    c = torch.as_tensor(cell, device="cuda")
    f = util.to_torch(ins["feats"], torch.float64, "cuda")
    m = util.to_torch(ins.get("mask"), torch.float64, "cuda")

    def loss(x):
        with torch.no_grad():
            fo, xo = mod(f, x, mask=m, cell=c)
        return float((fo.cpu().numpy() * gf).sum() + (xo.cpu().numpy() * gx).sum())
    x0 = util.to_torch(ins["coors"], torch.float64, "cuda")
    rs = np.random.RandomState(8)
    h = 1e-6
    for _ in range(6):
        b, i, a = rs.randint(x0.shape[0]), rs.randint(x0.shape[1]), rs.randint(x0.shape[2])
        xp, xm = x0.clone(), x0.clone()
        xp[b, i, a] += h
        xm[b, i, a] -= h
        fd = (loss(xp) - loss(xm)) / (2 * h)
        assert abs(fd - got["in.coors"][b, i, a]) <= 1e-5 * max(1.0, abs(fd))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
def test_dropout_with_a_fixed_seed_and_a_diagonal_cell_keeps_the_box_masks(dt):
    from egnn_pytorch_b200 import EGNN
    dtype = DT[dt]
    case, cell = build("knn_k8", dtype=dtype)
    ins = case["inputs"]
    B, Cd = ins["coors"].shape[0], ins["coors"].shape[-1]
    L = np.diagonal(cell_bc(cell, B, Cd), axis1=1, axis2=2)
    torch.manual_seed(0)
    mod = EGNN(dim=16, num_nearest_neighbors=8, valid_radius=2.0, dropout=0.2).to(dtype).cuda().train()
    f = util.to_torch(ins["feats"], dtype, "cuda").requires_grad_(True)
    x = util.to_torch(ins["coors"], _cdt(dtype), "cuda")
    m = util.to_torch(ins["mask"], dtype, "cuda")
    outs = []
    for kw in (dict(box=torch.as_tensor(L, dtype=_cdt(dtype), device="cuda")),
               dict(cell=torch.as_tensor(np.stack([np.diag(l) for l in L]), dtype=_cdt(dtype), device="cuda"))):
        torch.manual_seed(5)
        with torch.enable_grad():
            fo, xo = mod(f, x, mask=m, **kw)
            fo.sum().backward()
        outs.append((fo.detach(), xo.detach(), f.grad.clone()))
        f.grad = None
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert (outs[0][2] - outs[1][2]).abs().max().item() <= (1e-12 if dt == "fp64" else 1e-5) * max(1.0, outs[0][2].abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["dense_tilt09_soft", "knn_k8"])
def test_row_blocks_partition_forward_and_gradient(name):
    dtype = torch.float64
    case, cell = build(name, dtype=dtype)
    ins = case["inputs"]
    N = ins["feats"].shape[1]
    mod = util.make_module(case, dtype).requires_grad_(True)
    t = lambda a: util.to_torch(a, dtype, "cuda")
    c = torch.as_tensor(cell, device="cuda")
    f, x, m = t(ins["feats"]).requires_grad_(True), t(ins["coors"]).requires_grad_(True), t(ins.get("mask"))
    with torch.enable_grad():
        fo, xo = mod(f, x, mask=m, cell=c)
        (fo.sum() + xo.sum()).backward()
    gw = [p.grad.clone() for p in mod.parameters()]
    gx = x.grad.clone()
    mod.zero_grad(); x.grad = None
    cuts = [0, N // 3, N]
    fs, xs_ = [], []
    for r0, r1 in zip(cuts[:-1], cuts[1:]):
        with torch.enable_grad():
            fb, xb = mod(f, x, mask=m, cell=c, _rows=(r0, r1))
            fs.append(fb[:, r0:r1].detach()); xs_.append(xb[:, r0:r1].detach())
            (fb[:, r0:r1].sum() + xb[:, r0:r1].sum()).backward()
    assert torch.equal(torch.cat(fs, 1), fo.detach()) and torch.equal(torch.cat(xs_, 1), xo.detach())
    assert (x.grad - gx).abs().max().item() <= 1e-10 * max(1.0, gx.abs().max().item())
    for a, b in zip([p.grad for p in mod.parameters()], gw):
        assert (a - b).abs().max().item() <= 1e-10 * max(1.0, b.abs().max().item())


# ---- the cell grid


def _select_layer(cutoff, k, dtype):
    from egnn_pytorch_b200 import EGNN
    torch.manual_seed(0)
    return EGNN(dim=16, num_nearest_neighbors=k, valid_radius=cutoff ** 2).to(dtype).cuda().eval()


def _both_paths(monkeypatch, fn):
    monkeypatch.setenv("EGNN_B200_CELL_SELECT_MIN_N", "0")
    a = fn()
    monkeypatch.setenv("EGNN_B200_CELL_SELECT_MIN_N", NEVER)
    b = fn()
    return a, b


GRID = {   # name: (cell, fractional cells per axis roughly 1 / 2 / 3 from the cutoff, N, outside shift)
    "tilt_3cells":   (np.array([[3.0, 0, 0], [1.4, 3.0, 0], [-1.2, 0.9, 3.0]]), 0.95, 400, 2),
    "tilt_2cells":   (np.array([[3.0, 0, 0], [1.4, 3.0, 0], [-1.2, 0.9, 3.0]]), 1.35, 300, 4),
    "tilt_1cell":    (np.array([[3.0, 0, 0], [1.4, 3.0, 0], [-1.2, 0.9, 3.0]]), 1.45, 200, 6),
    "strong_tilt":   (np.array([[2.0, 0, 0], [1.9, 2.0, 0], [1.8, -1.9, 2.0]]), 0.6, 300, 3),
    "hex_slab":      (np.array([[3.0, 0, 0], [1.5, 3.0 * np.sqrt(3) / 2, 0], [0, 0, np.inf]]), 0.9, 300, 2),
    "c2":            (np.array([[3.0, 0], [1.2, 2.5]]), 0.8, 300, 3),
}


def _grid_inputs(name, dtype, seed=0, nonfinite=False):
    cell, cutoff, N, shift = GRID[name]
    rs = np.random.RandomState(seed)
    Cd = cell.shape[0]
    per = np.isfinite(np.diag(cell))
    Af = np.where(np.isfinite(cell), cell, 0.0) + np.diag(np.where(per, 0.0, 1.0))
    B = 2
    u = rs.uniform(0, 1, (B, N, Cd)) * np.where(per, 1.0, 4.0)
    u[:, : N // 4] = np.round(u[:, : N // 4] * 8) / 8          # points on a 1/8 lattice: tied distances, cell faces
    s = u + rs.randint(-shift, shift + 1, (B, N, Cd)) * per                     # several cells outside the cell
    x = torch.as_tensor(s @ Af, dtype=dtype)
    mask = torch.ones(B, N, dtype=torch.bool)
    mask[:, -7:] = False                                                        # padded
    if nonfinite:        # (lists only: in a layer, an ok = 0 slot of the all-pairs lists may hold such a node)
        x[0, 5, 0] = float("nan"); x[1, 9, -1] = float("inf")
    return x, mask, torch.as_tensor(cell, dtype=dtype), cutoff


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name", sorted(GRID))
def test_in_layer_cell_grid_equals_the_all_pairs_select(name, dt, monkeypatch):
    dtype = DT[dt]
    x, mask, cell, cutoff = _grid_inputs(name, dtype)
    x = x.cuda()
    mod = _select_layer(cutoff, 16, dtype)
    f = torch.randn(x.shape[0], x.shape[1], 16, dtype=dtype, device="cuda")
    with torch.no_grad():
        a, b = _both_paths(monkeypatch, lambda: mod(f, x, mask=mask.cuda(), cell=cell.cuda()))
    eq = lambda p, q: torch.equal(torch.nan_to_num(p, 7.0), torch.nan_to_num(q, 7.0))
    assert eq(a[0], b[0]) and eq(a[1], b[1])


def _brute_lists(x, mask, cell, cutoff, k):
    """The fp64 brute force of radius_neighbors: wrapped squared distances, ties to the lower index."""
    xd = x.double()
    B, N, Cd = xd.shape
    d = (cell_wrap(xd[:, :, None] - xd[:, None], cell.double()[None, None, None]) ** 2).sum(-1)
    thr = float(torch.tensor(cutoff * cutoff, dtype=x.dtype))          # r2 as the select compares it, in T
    ok = mask[:, :, None] & mask[:, None, :] & torch.isfinite(d) & (d <= thr)
    ok &= torch.isfinite(xd).all(-1)[:, :, None] & torch.isfinite(xd).all(-1)[:, None, :]
    key = torch.where(ok, d, torch.full_like(d, float("inf")))
    order = torch.sort(key, dim=-1, stable=True).indices[..., :k]
    kept = torch.gather(ok, -1, order)
    return torch.where(kept, order, torch.full_like(order, -1)).int(), ok.sum(-1).int(), d


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GRID))
def test_radius_neighbors_with_a_cell(name):
    """fp64 coordinates off the lattice (d^2 kept a relative 1e-6 from the cutoff), padded and non-finite nodes: the
    lists and counts equal the brute force; a diagonal cell gives the box's lists."""
    from egnn_pytorch_b200 import radius_neighbors
    x, mask, cell, cutoff = _grid_inputs(name, torch.float64, seed=1, nonfinite=True)
    x = x + 1e-3 * torch.randn(x.shape, generator=torch.Generator().manual_seed(3), dtype=x.dtype)
    nb, cnt = radius_neighbors(x.cuda(), cutoff, 16, mask=mask.cuda(), cell=cell.cuda(), return_counts=True)
    want, wcnt, d = _brute_lists(x, mask, cell, cutoff, 16)
    near = (d - cutoff ** 2).abs() < 1e-6 * cutoff ** 2
    assert not near[mask[:, :, None] & mask[:, None, :]].any()
    assert torch.equal(cnt.cpu(), wcnt) and torch.equal(nb.cpu(), want)
    # diagonal cell == box
    L = torch.diagonal(cell).clone()
    diag = torch.diag(L)
    xf = x.float().cuda()
    a = radius_neighbors(xf, cutoff, 16, mask=mask.cuda(), box=L.float().cuda(), return_counts=True)
    b = radius_neighbors(xf, cutoff, 16, mask=mask.cuda(), cell=diag.float().cuda(), return_counts=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


EXACT_CELLS = {"c3": np.array([[4.0, 0, 0], [1.0, 4.0, 0], [-2.0, 1.0, 4.0]]), "c2": np.array([[8.0, 0], [3.0, 6.0]])}
EXACT = [(c, r2) for c in ("c3", "c2") for r2 in (1, 2, 3, 4, 5) if not (c == "c2" and r2 == 3)]   # 3: no sum of 2 squares


def _exact_inputs(name, dtype, seed=0):
    """Integer coordinates (on 8 x 8 (x 8) sites, then moved by up to 3 whole lattice vectors per axis) in an integer
    cell: every wrap step and every squared distance is an exact integer in fp32 and fp64, so pairs sit exactly at an
    integer r2, and the fp64 brute force is the all-pairs select's own arithmetic."""
    cell = EXACT_CELLS[name]
    Cd = cell.shape[0]
    rs = np.random.RandomState(seed)
    B, N = 2, 40
    u = rs.randint(0, 8, (B, N, Cd)).astype(np.float64)
    x = u + rs.randint(-3, 4, (B, N, Cd)) @ cell
    mask = torch.ones(B, N, dtype=torch.bool)
    mask[:, -5:] = False
    return torch.as_tensor(x, dtype=dtype), mask, torch.as_tensor(cell, dtype=dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name,r2", EXACT)
def test_pairs_exactly_at_the_cutoff(name, r2, dt, monkeypatch):
    """The cell grid keeps every pair whose wrapped squared distance equals r2 exactly.  `radius_neighbors(cell=)`: lists
    and counts equal the exact brute force (the cutoff is sqrt(r2), raised by an ulp where its square would fall below
    r2, so the threshold in T is r2 itself, or r2 plus an ulp in fp64).  Inside a layer (valid_radius = r2, exact) the
    grid (MIN_N = 0) and the all-pairs select (MIN_N huge) give bit-identical outputs.  1 <= r2 <= 5 in a cell about 4
    wide gives 1 to 3 fractional cells per axis."""
    from egnn_pytorch_b200 import EGNN, radius_neighbors
    dtype = DT[dt]
    x, mask, cell = _exact_inputs(name, dtype)
    cutoff = float(np.sqrt(r2))
    if cutoff * cutoff < r2:
        cutoff = float(np.nextafter(cutoff, np.inf))
    k = 32
    want, wcnt, d = _brute_lists(x, mask, cell, cutoff, k)
    at = (d == r2) & mask[:, :, None] & mask[:, None, :]
    assert at.any(), "no pair sits exactly at the cutoff"
    nb, cnt = radius_neighbors(x.cuda(), cutoff, k, mask=mask.cuda(), cell=cell.cuda(), return_counts=True)
    assert torch.equal(cnt.cpu(), wcnt) and torch.equal(nb.cpu(), want)
    kept_at = torch.gather(at, -1, want.clamp_min(0).long()) & (want >= 0)
    assert kept_at.any(), "no pair at the cutoff made it into a list"
    torch.manual_seed(0)
    mod = EGNN(dim=16, num_nearest_neighbors=k, valid_radius=float(r2)).to(dtype).cuda().eval()
    f = torch.randn(x.shape[0], x.shape[1], 16, dtype=dtype, device="cuda")
    with torch.no_grad():
        a, b = _both_paths(monkeypatch, lambda: mod(f, x.cuda(), mask=mask.cuda(), cell=cell.cuda()))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp32", "bf16"])
def test_in_layer_cell_grid_with_a_diagonal_cell_is_the_box(dt, monkeypatch):
    dtype = DT[dt]
    x, mask, cell, cutoff = _grid_inputs("tilt_3cells", torch.float32)
    L = torch.tensor([3.0, 3.0, 3.0])
    mod = _select_layer(cutoff, 16, dtype)
    f = torch.randn(x.shape[0], x.shape[1], 16, device="cuda").to(dtype)
    monkeypatch.setenv("EGNN_B200_CELL_SELECT_MIN_N", "0")
    with torch.no_grad():
        a = mod(f, x.cuda(), mask=mask.cuda(), box=L.cuda())
        b = mod(f, x.cuda(), mask=mask.cuda(), cell=torch.diag(L).cuda())
    eq = lambda p, q: torch.equal(torch.nan_to_num(p, 7.0), torch.nan_to_num(q, 7.0))
    assert eq(a[0], b[0]) and eq(a[1], b[1])


# ---- network and graphs


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32", "bf16"])
def test_network_passes_the_cell_to_every_layer(dt):
    from egnn_pytorch_b200 import EGNN_Network
    dtype = DT[dt]
    torch.manual_seed(0)
    net = EGNN_Network(depth=3, dim=16, num_nearest_neighbors=6).to(dtype).cuda().eval()
    case, cell = build("knn_k8", dtype=dtype)
    f = util.to_torch(case["inputs"]["feats"], dtype, "cuda")
    x = util.to_torch(case["inputs"]["coors"], _cdt(dtype), "cuda").to(dtype)
    m = util.to_torch(case["inputs"]["mask"], dtype, "cuda")
    c = torch.as_tensor(cell, device="cuda", dtype=_cdt(dtype))
    with torch.no_grad():
        fo, xo = net(f, x, mask=m, cell=c)
        f2, x2 = f, x
        for _, egnn in net.layers:
            f2, x2 = egnn(f2, x2, None, m, None, cell=c)
        fn, xn = net(f, x, mask=m)
    assert torch.equal(fo, f2) and torch.equal(xo, x2)
    assert not torch.equal(xo, xn)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp32", "bf16"])
def test_graph_replay_follows_an_in_place_cell_change(dt):
    from egnn_pytorch_b200.graphs import GraphedForward
    dtype = DT[dt]
    case, cell = build("dense_tilt", dtype=dtype)
    mod = util.make_module(case, dtype)
    f = util.to_torch(case["inputs"]["feats"], dtype, "cuda")
    x = util.to_torch(case["inputs"]["coors"], torch.float32, "cuda")
    c = torch.as_tensor(cell, dtype=torch.float32, device="cuda")
    fast = GraphedForward(mod, f, x, cell=c)
    c[2, 0] += 0.25                                       # a shear step
    c.mul_(1.0625)
    got = [t.clone() for t in fast(f, x)]
    with torch.no_grad():
        want = mod(f, x, cell=c.clone())
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
