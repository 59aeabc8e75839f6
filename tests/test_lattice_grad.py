"""Gradients with respect to the periodic box and the triclinic cell (`lattice_grad=True`), for stress and virial
(egnn_layer_backward_periodic_lattice / egnn_layer_backward_triclinic_lattice).

The specification is torch autograd through the float64 restatements: tests/torch_reference.py's box wrap and
test_triclinic.py's sequential cell wrap, with the box / cell a leaf that requires grad.  It is pinned on the CPU
without trusting the wrap: on a 3^C supercell of lattice images the numpy gradient oracle gives dL/dx of every image,
and an image shifted by s (integer lattice coordinates) moves with the cell, so dL/dcell[c][d] = sum_images s_c g_d.

CPU: that pin; argument handling; the new symbols and their argument errors.
GPU: the library against the restatement (fp64 within 1e-12 of scale, fp32 within 4x the fp32 restatement's error) on
dense and kNN layers, boxes and cells, shared and per-graph lattices, C = 2 and 3, masks, soft edges, CoorsNorm,
fourier and edge features, saved and recomputed pre-activations, and a B = 8, N = 4096, k = 32 layer; central finite
differences; exact zeros; unchanged other gradients; row blocks; EGNN_Network; the README stress recipe."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

import cases
import torch_reference as R
import util
from oracle import egnn_oracle_grad as G
from test_triclinic import (SUPER, TCASES, _cell_geometry, build, cell_bc, cell_coors, knn_gap, make_cell, supercell,
                            wrap_margin, wrapped_d2)

DT = {"fp64": torch.float64, "fp32": torch.float32}
TAU64 = 1e-12            # fp64: error over the largest magnitude of the lattice gradient
FP32_RATIO = 4.0         # fp32: error over the fp32 restatement's error (tests/test_gpu_backward_at_size.py)
FP32_FLOOR = 1e-6        # ... which is floored at this fraction of the scale


def _cdt(dtype):
    return torch.float64 if dtype == torch.float64 else torch.float32


def ref_grads(case, lattice, kind, gf, gx, dtype=torch.float64, device="cpu", neighbors=None):
    """Restatement gradients of sum(fo gf) + sum(xo gx) with the lattice a leaf: {'in.*', 'p.*', 'lattice'}.
    kind: 'box' (lengths, [C] or [B, C]) or 'cell' ([C, C] or [B, C, C])."""
    ins = case["inputs"]
    lat = torch.as_tensor(np.array(lattice, np.float64)).to(device=device, dtype=dtype).requires_grad_(True)
    f = torch.as_tensor(np.asarray(ins["feats"], np.float64)).to(device=device, dtype=dtype)
    args = (case["params"], case["cfg"], f, ins["coors"], gf, gx, ins.get("edges"), ins.get("mask"), ins.get("adj_mat"),
            lat, neighbors)
    if kind == "cell":
        with _cell_geometry():
            g = R.layer_grads_chunked(*args)
    else:
        g = R.layer_grads_chunked(*args)
    g["lattice"] = lat.grad if lat.grad is not None else torch.zeros_like(lat)
    return g


# ----------------------------------------------------------------------------- CPU: pin the specification


LSUPER = [s for s in SUPER if s[0] in ("dense_tilt", "dense_tilt09_normc", "dense_hex_slab", "knn_c2")] + \
         [("dense_box", dict(dim=8, edge_dim=2, fourier_features=1), "box", "padded", None)]


@pytest.mark.parametrize("name,cfg,kind,mask,k", LSUPER, ids=[s[0] for s in LSUPER])
def test_supercell_of_images_gives_the_restatement_lattice_gradient(name, cfg, kind, mask, k):
    """The inputs of test_triclinic's supercell test (every pair's minimum image shorter than min L_c / 2).  The image
    of node j shifted by s sits at x_j + s A, so the gradient with respect to A is sum_images s_c dL/dx_d."""
    B, N = 2, 6
    box = kind == "box"
    cell = np.diag([3.0, 3.4, 2.8]) if box else make_cell(kind, B, np.random.RandomState(3))
    Cd = cell.shape[-1]
    case = cases.build_case(dict(kind="layer", cfg=cfg, B=B, N=N, C=Cd, seed=78, init="xavier", mask=mask or "none"))
    rs = np.random.RandomState(6)
    diag = np.diag(cell)
    per = np.isfinite(diag) & (diag > 0)
    y = rs.uniform(-1, 1, (B, N, Cd))
    y = y / np.linalg.norm(y, axis=-1, keepdims=True) * rs.uniform(0, 0.2 * diag[per].min(), (B, N, 1))
    Af = np.where(np.isfinite(cell), cell, 0.0) + np.diag(np.where(per, 0.0, 1.0))
    s = np.linalg.solve(Af.T, y.reshape(-1, Cd).T).T.reshape(B, N, Cd)
    x = np.where(per, s - np.floor(s), s) @ Af
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
    gf, gx = rs.randn(B, N, lc["dim"]), rs.randn(B, N, Cd)
    pad = lambda a: np.concatenate([a, np.zeros((B, (S - 1) * N) + a.shape[2:])], 1)
    lcfg = dict(lc, num_nearest_neighbors=nb.shape[-1])
    gs = G.egnn_layer_backward(P, lcfg, f, xs, e, m, None, pad(gf), pad(gx), neighbors=nb)
    shifts = [np.array(t, np.float64) for t in itertools.product(*[(0, -1, 1) if p else (0,) for p in per])]
    assert len(shifts) == S
    want = np.zeros((B, Cd, Cd))
    for t, sv in enumerate(shifts):
        g_img = gs["coors"][:, t * N:(t + 1) * N].sum(1)                    # [B, C]
        want += sv[None, :, None] * g_img[:, None, :]
    if box:
        want = np.diagonal(want, axis1=1, axis2=2)                          # a box moves image s by s_c L_c on axis c
        got = ref_grads(case, diag, "box", gf, gx)["lattice"].numpy()       # [C]: summed over the batch
        want = want.sum(0)
    else:
        got = ref_grads(case, cell, "cell", gf, gx)["lattice"].numpy()      # [C, C] shared: summed over the batch
        want = np.tril(want.sum(0))
    tol = 1e-7 if lc["norm_coors"] else 1e-11
    scale = max(1.0, float(np.abs(want).max()))
    assert np.abs(want).max() > 1e-3                                      # pairs do cross the boundary
    assert np.abs(got - want).max() <= tol * scale, (got, want)


def test_lattice_grad_needs_a_lattice_and_unlocks_requires_grad(monkeypatch):
    from egnn_pytorch_b200 import EGNN, EGNN_Network
    f, x = torch.randn(2, 5, 8), torch.randn(2, 5, 3)
    with pytest.raises(ValueError, match="lattice_grad=True needs box= or cell="):
        EGNN(dim=8)(f, x, lattice_grad=True)
    with pytest.raises(ValueError, match="lattice_grad=True needs box= or cell="):
        EGNN_Network(depth=1, dim=8)(f, x, lattice_grad=True)
    for kw in (dict(box=torch.ones(3, requires_grad=True)), dict(cell=torch.eye(3).requires_grad_(True))):
        with pytest.raises(ValueError, match="requires_grad.*lattice_grad=True"):
            EGNN(dim=8)(f, x, **kw)
    # accepted with the keyword: the checks pass and the training path is entered (checked without a device)
    calls = []
    layer = EGNN(dim=8).requires_grad_(False)
    monkeypatch.setattr(EGNN, "_forward_train", lambda self, *a, **k: calls.append(a[-1]) or (a[1], a[2]))
    cell = (3 * torch.eye(3)).requires_grad_(True)
    with torch.enable_grad():
        layer(f, x, cell=cell, lattice_grad=True)
    assert len(calls) == 1 and calls[0] is cell


def test_lattice_symbols_load_and_reject_bad_arguments_before_launching():
    from egnn_pytorch_b200 import _native as nat
    lib = nat.load()
    for name in ("egnn_layer_backward_periodic_lattice", "egnn_layer_backward_triclinic_lattice"):
        assert name in nat.SYMBOLS and getattr(lib, name).argtypes is not None
    assert lib.egnn_abi_version() == 4
    desc = nat.LayerDesc(abi_version=4, dtype=nat.DTYPE_F32, B=1, N=4, C=3, dim=8, m_dim=16,
                         flags=nat.FLAG_UPDATE_FEATS | nat.FLAG_UPDATE_COORS)
    dummy = C.c_void_p(256)
    per, tri = lib.egnn_layer_backward_periodic_lattice, lib.egnn_layer_backward_triclinic_lattice
    call = lambda fn, lat, g: fn(C.byref(desc), None, dummy, None, lat, dummy, None, g, dummy, 1 << 20, None)
    for fn in (per, tri):                                          # a NULL lattice or lattice gradient
        assert call(fn, None, dummy) == -1
        assert call(fn, dummy, None) == -1
    desc.dtype = nat.DTYPE_BF16                                    # bf16 has no backward
    assert call(per, dummy, dummy) == -3 and call(tri, dummy, dummy) == -3
    desc.dtype = nat.DTYPE_F32
    desc.C = 4                                                     # a cell needs C in {2, 3}
    assert call(tri, dummy, dummy) == -2


# ----------------------------------------------------------------------------- GPU


def _module(case, dtype):
    return util.make_module(case, dtype).requires_grad_(True)


def gpu_grads(case, lattice, kind, dtype, gf, gx, lattice_grad=True, mod=None, neighbors=None, rows=None):
    """Module gradients (autograd through the library) with the lattice a leaf -> {'in.*', 'p.*', ['lattice']} on the
    host in float64."""
    mod = mod or _module(case, dtype)
    ins = case["inputs"]
    t = lambda a: util.to_torch(a, dtype, "cuda")
    f, x = t(ins["feats"]).requires_grad_(True), util.to_torch(ins["coors"], _cdt(dtype), "cuda").requires_grad_(True)
    e = t(ins.get("edges"))
    leaves = {"in.feats": f, "in.coors": x}
    if e is not None:
        leaves["in.edges"] = e.requires_grad_(True)
    lat = torch.as_tensor(np.array(lattice, np.float64), dtype=_cdt(dtype), device="cuda")
    if lattice_grad:
        lat.requires_grad_(True)
    kw = dict(mask=t(ins.get("mask")), lattice_grad=lattice_grad, **{kind: lat})
    if neighbors is not None:
        kw["neighbors"] = torch.as_tensor(neighbors, device="cuda")
    if rows is not None:
        kw["_rows"] = rows
    with torch.enable_grad():
        fo, xo = mod(f, x, e, **kw)
        if rows is not None:
            fo, xo = fo[:, rows[0]:rows[1]], xo[:, rows[0]:rows[1]]
            gf, gx = gf[:, rows[0]:rows[1]], gx[:, rows[0]:rows[1]]
        ((fo * t(gf).to(fo.dtype)).sum() + (xo * t(gx).to(xo.dtype)).sum()).backward()
    got = {k: v.grad.double().cpu().numpy() for k, v in leaves.items()}
    got.update({f"p.{k}": (torch.zeros_like(p) if p.grad is None else p.grad).double().cpu().numpy()
                for k, p in mod.named_parameters()})
    if lattice_grad:
        assert lat.grad is not None and lat.grad.dtype == lat.dtype and lat.grad.shape == lat.shape
        got["lattice"] = lat.grad.double().cpu().numpy()
    return got


def _cotangents(case):
    rs = np.random.RandomState(4)
    return rs.randn(*case["inputs"]["feats"].shape), rs.randn(*case["inputs"]["coors"].shape)


def build_box(name, dtype=torch.float64):
    """test_triclinic.build with a box: the diagonal of the case's cell ([C] shared, [B, C] per graph), coordinates
    placed by cell_coors for that box (wrap decisions 1e-3 from 1/2) and kNN ranks 1e-5 from a tie."""
    cfg, B, N, kind, mask = TCASES[name]
    Cd = 2 if kind == "c2" else 3
    cdt = _cdt(dtype)
    case = cases.build_case(dict(kind="layer", cfg=cfg, B=B, N=N, C=Cd, seed=910, init="xavier", mask=mask or "none"))
    for seed in range(20):
        rs = np.random.RandomState(810 + seed)
        L = util.rounded(np.diagonal(make_cell(kind, B, rs), axis1=-2, axis2=-1).copy(), cdt)
        diag = np.eye(Cd) * L[..., None, :]
        diag[~np.isfinite(diag)] = 0.0
        diag[..., np.arange(Cd), np.arange(Cd)] = L
        case["inputs"]["coors"] = cell_coors(rs, B, N, diag, dtype=cdt)
        if knn_gap(case, diag) > 1e-5:
            return case, L
    raise AssertionError("no tie-free kNN inputs")


def inputs(name, kind, dtype=torch.float64):
    """(case, lattice) of a test_triclinic case with its cell, or (kind 'box') with a box."""
    return build(name, dtype=dtype) if kind == "cell" else build_box(name, dtype)


def check64(got, want, what, tau=TAU64):
    scale = float(np.abs(want).max())
    err = float(np.abs(got - want).max())
    print(f"{what}: fp64 lattice gradient error {err / max(scale, 1e-300):.2e} of scale {scale:.3e}")
    assert np.isfinite(got).all() and err <= tau * scale, (what, got, want)


def check32(got, ref32, want, what):
    scale = float(np.abs(want).max())
    ek, er = float(np.abs(got - want).max()), float(np.abs(ref32 - want).max())
    r = ek / max(er, FP32_FLOOR * scale, 1e-300)
    print(f"{what}: fp32 lattice gradient error {ek / scale:.2e} of scale, {r:.2f}x the fp32 restatement's")
    assert np.isfinite(got).all() and r <= FP32_RATIO, (what, ek, er)


# (test_triclinic case, box or cell): dense and kNN (warp select, k = 33 block sort), shared and per-graph lattices,
# C = 2 and 3, padded / random / full masks, soft edges with mean pooling, CoorsNorm, fourier and edge features
PARITY = [("dense_tilt09_soft", "cell"), ("dense_tilt09_soft", "box"), ("dense_per_graph_edges", "cell"),
          ("dense_per_graph_edges", "box"), ("dense_c2", "cell"), ("dense_hex_slab", "cell"), ("knn_k8", "cell"),
          ("knn_k8", "box"), ("knn_k16_edges", "cell"), ("knn_k33", "cell"), ("knn_k33", "box"),
          ("knn_c2_fourier", "cell"), ("knn_c2_fourier", "box")]


@pytest.mark.gpu
@pytest.mark.parametrize("saved", [True, False], ids=["saved", "recomputed"])
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name,kind", PARITY, ids=[f"{n}-{k}" for n, k in PARITY])
def test_lattice_gradient_matches_the_restatement(name, kind, dt, saved, monkeypatch):
    if not saved:
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")
    dtype = DT[dt]
    case, lat = inputs(name, kind, dtype)
    gf, gx = _cotangents(case)
    got = gpu_grads(case, lat, kind, dtype, gf, gx)
    want = ref_grads(case, lat, kind, gf, gx)
    assert float(want["lattice"].abs().max()) > 1e-3
    what = f"{name} {kind} [{dt}] {'saved' if saved else 'recomputed'}"
    if dtype == torch.float64:
        check64(got["lattice"], want["lattice"].numpy(), what)
        util.compare({k: v for k, v in got.items() if k != "lattice"},
                     {k: v.numpy() for k, v in want.items() if k != "lattice"}, util.grad_tol(case, dtype), what)
    else:
        ref32 = ref_grads(case, lat, kind, gf.astype(np.float32).astype(np.float64),
                          gx.astype(np.float32).astype(np.float64), dtype=torch.float32)["lattice"].double().numpy()
        check32(got["lattice"], ref32, want["lattice"].numpy(), what)


def _random_lists(rs, B, N, k, x, cell, margin):
    """k random partners per node (-1 in about 5 % of the slots, the node itself sometimes), redrawn while a partner's
    wrap decision lies within `margin` of 1/2 (so fp32 wraps every pair as fp64 does)."""
    nb = rs.randint(0, N, (B, N, k))
    A = cell_bc(cell, B, x.shape[-1])
    for _ in range(100):
        r = x[np.arange(B)[:, None, None], np.arange(N)[None, :, None]] - x[np.arange(B)[:, None, None], nb]
        m = np.ones(nb.shape)
        for c in reversed(range(x.shape[-1])):
            t = r[..., c] / A[:, c, c][:, None, None]
            m = np.minimum(m, np.abs(np.abs(t - np.rint(t)) - 0.5))
            r[..., :c + 1] -= np.rint(t)[..., None] * A[:, c, :c + 1][:, None, None, :]
        bad = m < margin
        if not bad.any():
            break
        nb = np.where(bad, rs.randint(0, N, nb.shape), nb)
    assert not bad.any()
    nb[rs.uniform(size=nb.shape) < 0.05] = -1
    return nb


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
def test_thousands_of_ctas_reduce_into_each_graph(dt):
    """B = 8, N = 4096, k = 32 neighbour lists (1024 bwd3 CTAs per graph) in per-graph tilted cells, against the
    row-chunked restatement on the device.  Random partners cross the cell up to several lattice vectors away."""
    dtype = DT[dt]
    B, N, k = 8, 4096, 32
    case = cases.build_case(dict(kind="layer", cfg=dict(dim=16, edge_dim=0), B=B, N=N, C=3, seed=4242, init="xavier",
                                 mask="padded"))
    rs = np.random.RandomState(17)
    cell = make_cell("per_graph", B, rs)
    cell = util.rounded(cell, _cdt(dtype))
    x = rs.uniform(-6, 6, (B, N, 3))
    x = x.astype(np.float32).astype(np.float64) if dtype == torch.float32 else x
    case["inputs"]["coors"] = x
    if dtype == torch.float32:
        case["params"] = {kk: np.asarray(v, np.float32).astype(np.float64) for kk, v in case["params"].items()}
        case["inputs"]["feats"] = case["inputs"]["feats"].astype(np.float32).astype(np.float64)
    nb = _random_lists(rs, B, N, k, x, cell, 1e-4)
    gf, gx = _cotangents(case)
    gf, gx = gf.astype(np.float32).astype(np.float64), gx.astype(np.float32).astype(np.float64)
    got = gpu_grads(case, cell, "cell", dtype, gf, gx, neighbors=nb)
    want = ref_grads(case, cell, "cell", gf, gx, device="cuda", neighbors=torch.as_tensor(nb, device="cuda"))
    w = want["lattice"].cpu().numpy()
    assert np.abs(w).max() > 1.0
    if dtype == torch.float64:
        check64(got["lattice"], w, "B=8 N=4096 k=32 cells")
    else:
        ref32 = ref_grads(case, cell, "cell", gf, gx, dtype=torch.float32, device="cuda",
                          neighbors=torch.as_tensor(nb, device="cuda"))["lattice"].double().cpu().numpy()
        check32(got["lattice"], ref32, w, "B=8 N=4096 k=32 cells")
    assert np.array_equal(np.triu(got["lattice"], 1), np.zeros_like(got["lattice"]))


def _loss(mod, case, kind, gf, gx):
    ins = case["inputs"]
    t = lambda a: util.to_torch(a, torch.float64, "cuda")
    f, m = t(ins["feats"]), t(ins.get("mask"))
    e = t(ins.get("edges"))

    def loss(x, lat):
        with torch.no_grad():
            fo, xo = mod(f, x, e, mask=m, **{kind: lat})
        return float((fo.cpu().numpy() * gf).sum() + (xo.cpu().numpy() * gx).sum())
    return loss


@pytest.mark.gpu
@pytest.mark.parametrize("name,kind", [("dense_tilt09_soft", "cell"), ("knn_k8", "cell"), ("dense_c2", "cell"),
                                       ("dense_per_graph_edges", "box"), ("knn_k8", "box")])
def test_fp64_lattice_gradient_matches_central_finite_differences(name, kind):
    """Every lower-triangular cell entry / every box length.  build() keeps wrap decisions 1e-3 and kNN ranks 1e-5
    from their discontinuities, far more than the step moves them."""
    case, lat0 = inputs(name, kind)
    gf, gx = _cotangents(case)
    got = gpu_grads(case, lat0, kind, torch.float64, gf, gx)["lattice"]
    loss = _loss(_module(case, torch.float64), case, kind, gf, gx)
    x0 = util.to_torch(case["inputs"]["coors"], torch.float64, "cuda")
    h = 1e-6
    entries = [idx for idx in np.ndindex(*np.shape(lat0)) if kind == "box" or idx[-1] <= idx[-2]]
    for idx in entries:
        lp, lm = np.array(lat0, np.float64), np.array(lat0, np.float64)
        lp[idx] += h
        lm[idx] -= h
        fd = (loss(x0, torch.as_tensor(lp, device="cuda")) - loss(x0, torch.as_tensor(lm, device="cuda"))) / (2 * h)
        assert abs(fd - got[idx]) <= 1e-6 * max(1.0, abs(fd)), (idx, fd, got[idx])


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
def test_exact_zeros_and_a_diagonal_cell_is_the_box(dt):
    dtype = DT[dt]
    case, cell = build("dense_tilt09_soft", dtype=dtype)
    gf, gx = _cotangents(case)
    x = case["inputs"]["coors"]
    # a box three times the coordinate spread wraps no pair: exactly 0
    spread = x.max((0, 1)) - x.min((0, 1))
    g = gpu_grads(case, 3 * spread, "box", dtype, gf, gx)["lattice"]
    assert np.array_equal(g, np.zeros_like(g))
    # aperiodic axes and rows, and the upper triangle: exactly 0
    case_h, cell_h = build("dense_hex_slab", dtype=dtype)
    g = gpu_grads(case_h, cell_h, "cell", dtype, *_cotangents(case_h))["lattice"]
    assert np.array_equal(g[2], np.zeros(3)) and np.array_equal(np.triu(g, 1), np.zeros((3, 3)))
    assert np.abs(g[:2, :2]).max() > 1e-3
    L = np.array([np.diag(cell)[0], np.inf, 0.0])                   # axes 1 and 2 aperiodic
    g = gpu_grads(case, L, "box", dtype, gf, gx)["lattice"]
    assert g[1] == 0 and g[2] == 0 and g[0] != 0
    # a diagonal cell's diagonal gradient is the box gradient (the wrap subtracts exact zeros off the diagonal)
    L = np.diag(cell).copy()
    gb = gpu_grads(case, L, "box", dtype, gf, gx)["lattice"]
    gc = gpu_grads(case, np.diag(L), "cell", dtype, gf, gx)["lattice"]
    tol = 1e-13 if dtype == torch.float64 else 1e-6
    assert np.abs(np.diag(gc) - gb).max() <= tol * np.abs(gb).max()
    assert np.array_equal(np.triu(gc, 1), np.zeros((3, 3)))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name,kind", [("dense_per_graph_edges", "cell"), ("knn_k8", "box"), ("knn_k33", "cell")])
def test_lattice_grad_leaves_every_other_gradient_unchanged(name, kind, dt):
    dtype = DT[dt]
    case, lat = inputs(name, kind, dtype)
    gf, gx = _cotangents(case)
    with_lat = gpu_grads(case, lat, kind, dtype, gf, gx, lattice_grad=True)
    without = gpu_grads(case, lat, kind, dtype, gf, gx, lattice_grad=False)
    with_lat.pop("lattice")
    util.compare(with_lat, without, 1e-13 if dtype == torch.float64 else 1e-5, f"{name} {kind} [{dt}]")


@pytest.mark.gpu
@pytest.mark.parametrize("name,kind", [("dense_tilt09_soft", "cell"), ("knn_k8", "cell"), ("knn_k8", "box")])
def test_row_block_lattice_gradients_sum_to_the_whole(name, kind):
    case, lat = inputs(name, kind)
    gf, gx = _cotangents(case)
    mod = _module(case, torch.float64)
    whole = gpu_grads(case, lat, kind, torch.float64, gf, gx, mod=mod)["lattice"]
    N = case["inputs"]["feats"].shape[1]
    cuts = [0, N // 3, N // 3, N]                       # (an empty block too)
    parts = [gpu_grads(case, lat, kind, torch.float64, gf, gx, mod=mod, rows=(r0, r1))["lattice"]
             for r0, r1 in zip(cuts[:-1], cuts[1:])]
    assert np.array_equal(parts[1], np.zeros_like(parts[1]))
    assert np.abs(sum(parts) - whole).max() <= 1e-13 * np.abs(whole).max()


def _net_case(seed=0):
    """A dense EGNN_Network of depth 2 in a tilted cell, its inputs off the wrap boundaries."""
    B, N = 2, 24
    case = cases.build_case(dict(kind="network", cfg=dict(depth=2, dim=16), B=B, N=N, C=3, seed=930 + seed,
                                 init="xavier", mask="padded"))
    rs = np.random.RandomState(730 + seed)
    cell = make_cell("tilt", B, rs)
    case["inputs"]["coors"] = cell_coors(rs, B, N, cell)
    return case, cell


@pytest.mark.gpu
def test_network_lattice_gradient_matches_the_restatement_network():
    """Autograd sums the layers' lattice gradients, and through the chained coordinates each layer's coordinate
    gradient reaches the earlier layers' lattice terms.  The second layer's inputs are the first layer's outputs, so
    wrap decisions there are checked too."""
    case, cell = _net_case()
    ins, ncfg = case["inputs"], case["ncfg"]
    with _cell_geometry():
        _, _, states = R.network(case["params"], ncfg, ins["feats"], ins["coors"], mask=ins["mask"], box=cell)
    for _, xs in states:
        assert wrap_margin(xs.detach().numpy(), cell).min() > 1e-4
    rs = np.random.RandomState(5)
    gf, gx = rs.randn(*ins["feats"].shape), rs.randn(*ins["coors"].shape)
    lat = torch.as_tensor(cell).requires_grad_(True)
    with _cell_geometry():
        want = R.network_grads(case["params"], ncfg, ins["feats"], ins["coors"], gf, gx, mask=ins["mask"], box=lat)
    want_lat = lat.grad.numpy()
    net = util.make_module(case, torch.float64).requires_grad_(True)
    t = lambda a: util.to_torch(a, torch.float64, "cuda")
    f, x = t(ins["feats"]).requires_grad_(True), t(ins["coors"]).requires_grad_(True)
    c = torch.as_tensor(cell, device="cuda").requires_grad_(True)
    with torch.enable_grad():
        fo, xo = net(f, x, mask=t(ins["mask"]), cell=c, lattice_grad=True)
        ((fo * t(gf)).sum() + (xo * t(gx)).sum()).backward()
    check64(c.grad.cpu().numpy(), want_lat, "EGNN_Network depth 2")
    assert np.abs(x.grad.cpu().numpy() - want["in.coors"].numpy()).max() <= 1e-9 * np.abs(want["in.coors"].numpy()).max()


def _energy(net, f, m):
    w = torch.as_tensor(np.random.RandomState(9).randn(f.shape[-1]), device="cuda")

    def E(x, cell, grad=False):
        with torch.set_grad_enabled(grad):
            fo, _ = net(f, x, mask=m, cell=cell, lattice_grad=grad)
            return (fo * w).sum()
    return E


@pytest.mark.gpu
def test_stress_recipe_lower_triangle_and_symmetric_strain():
    """An invariant energy (a weighted sum of a network's feats_out).  D = x^T dE/dx + cell^T dE/dcell on the lower
    triangle equals finite differences of E(x F, cell F) for lower-triangular F = I + h e_ab; a symmetric strain
    F = I + h (e_ab + e_ba), rotated back into lower-triangular form by the README's QR recipe, gives D_ab + D_ba =
    2 D_ab, so the lower triangle determines the symmetric stress."""
    case, cell = _net_case(1)
    ins = case["inputs"]
    net = util.make_module(case, torch.float64)
    t = lambda a: util.to_torch(a, torch.float64, "cuda")
    f, m = t(ins["feats"]), t(ins["mask"])
    E = _energy(net, f, m)
    x = t(ins["coors"]).requires_grad_(True)
    c = torch.as_tensor(cell, device="cuda").requires_grad_(True)
    with torch.enable_grad():
        gx, gc = torch.autograd.grad(E(x, c, grad=True), (x, c))
    D = (torch.einsum("bna,bnc->ac", x.detach(), gx) + c.detach().T @ gc).cpu().numpy()
    h = 1e-6
    x0, c0 = x.detach(), c.detach()
    for a in range(3):
        for b in range(a + 1):
            fd = []
            for sgn in (1, -1):
                F = torch.eye(3, dtype=torch.float64, device="cuda")
                F[a, b] += sgn * h
                fd.append(float(E(x0 @ F, c0 @ F)))
            fd = (fd[0] - fd[1]) / (2 * h)
            assert abs(fd - D[a, b]) <= 1e-6 * max(1.0, abs(fd)), ("lower", a, b, fd, D[a, b])
            if a == b:
                continue
            fd = []
            for sgn in (1, -1):
                F = torch.eye(3, dtype=torch.float64, device="cuda")
                F[a, b] += sgn * h
                F[b, a] += sgn * h
                cs, xs = c0 @ F, x0 @ F
                q, r = torch.linalg.qr(cs.T)                # the README's rotation into lower-triangular form
                s = torch.sign(torch.diagonal(r)); q = q * s
                fd.append(float(E(xs @ q, torch.tril(cs @ q))))
            fd = (fd[0] - fd[1]) / (2 * h)
            assert abs(fd - 2 * D[a, b]) <= 1e-6 * max(1.0, abs(fd)), ("symmetric", a, b, fd, D[a, b])
