"""Periodic boundaries: `EGNN.forward(..., box=)` / `EGNN_Network.forward(..., box=)`, the minimum-image pair geometry
rel = x_i - x_j - L rint((x_i - x_j) / L) on every axis with a finite L > 0 (egnn_layer_forward_periodic /
egnn_layer_backward_periodic).

The periodic restatement (tests/torch_reference.py) is the reference layer (egnn_pytorch.py:224-341) in float64 torch
with the wrapped rel in place of rel_coors, so gradients come from autograd.  It is pinned three ways without trusting its own
wrap: with no box and with a 2^20 box it equals the golden-pinned numpy oracle; on a 3^C supercell of images, where
every central node lists the nearest image of each partner, the existing edge-list oracles (forward and gradient) give
its outputs and gradients; its kNN selection equals a stable argsort of brute-force wrapped distances.

Inputs keep every pair at least 1e-3 L away from the half-box boundary (coordinates on an odd lattice of the box plus a
small jitter, then shifted by whole box lengths) and kNN inputs tie-free at the k-th rank, so fp32 / bf16 rounding picks
the image and the neighbours the fp64 restatement picks.

CPU: the restatement, the supercell checks, the kNN selection, validation errors, the new symbols.
GPU: forward parity on every path (fp64 / fp32 SIMT, bf16 tensor cores), huge box == no box, lattice-shift and
translation invariance, gradients (saved and recomputed pre-activations, finite differences), dropout, row blocks,
EGNN_Network, CUDA-graph replay after an in-place box change."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest
import torch

import cases
import util
from oracle import egnn_oracle as O
from oracle import egnn_oracle_grad as G

HUGE = 2.0 ** 20


# the periodic restatement: tests/torch_reference.py
from torch_reference import _t, box_bc, layer, layer_grads, select, wrap  # noqa: E402


# ----------------------------------------------------------------------------- inputs


def lattice_coors(rs, B, N, C, L, shift=2):
    """Coordinates on an odd lattice (101 cells per box length) plus a jitter below 0.0015 L, then moved by whole box
    lengths in [-shift, shift]: every pair difference sits >= 1e-3 L away from a half-box boundary on every periodic
    axis.  L: [C] lengths (a non-periodic axis: pass its scale)."""
    L = np.asarray(L, np.float64)
    u = rs.randint(0, 101, (B, N, C)) / 101.0 + rs.uniform(-0.0015, 0.0015, (B, N, C))
    return (u + rs.randint(-shift, shift + 1, (B, N, C))) * L


def half_box_margin(coors, box):
    """Smallest distance of |rel / L| (mod 1) from 1/2 over all pairs and periodic axes, as a fraction of L."""
    x = np.asarray(coors, np.float64)
    bx = np.broadcast_to(np.asarray(box, np.float64), (x.shape[0], x.shape[-1]))
    rel = x[:, :, None] - x[:, None]
    per = np.isfinite(bx) & (bx > 0)
    f = rel / np.where(per, bx, 1.0)[:, None, None]
    m = np.abs(np.abs(f - np.round(f)) - 0.5)
    return float(np.where(per[:, None, None], m, 1.0).min())


# name: (layer cfg, B, N, C, box [C] or None for [B, C], mask, adj).  inf / 0 entries: aperiodic axes.
PCASES = {
    "dense":          (dict(dim=16), 2, 40, 3, [3.0, 2.5, 4.0], None, None),
    "dense_mask_soft_mean": (dict(dim=16, soft_edges=True, m_pool_method="mean"), 3, 33, 3, None, "padded", None),
    "dense_everything_c5": (dict(dim=16, edge_dim=2, fourier_features=2, norm_coors=True, coor_weights_clamp_value=0.5,
                                 norm_feats=True), 2, 24, 5, [3.0, np.inf, 2.0, 0.0, 3.5], "random", None),
    "dense_c2":       (dict(dim=8), 2, 30, 2, [2.0, np.inf], None, None),
    "dense_n257":     (dict(dim=16), 1, 257, 3, [6.0, 6.0, 6.0], None, None),
    "dense_n129_edges": (dict(dim=16, edge_dim=3), 1, 129, 3, None, "padded", None),
    "knn_k8":         (dict(dim=16, num_nearest_neighbors=8, valid_radius=2.0), 2, 50, 3, [4.0, 4.0, 4.0], "padded", None),
    "knn_k32_edges":  (dict(dim=16, edge_dim=3, num_nearest_neighbors=32), 2, 97, 3, None, None, None),
    "knn_k33":        (dict(dim=8, num_nearest_neighbors=33), 1, 70, 3, [3.0, 3.0, 3.0], "padded", None),
    "knn_c2_fourier": (dict(dim=16, fourier_features=1, num_nearest_neighbors=6, m_pool_method="mean"), 2, 40, 2,
                       [3.0, 0.0], None, None),
    "knn_c5_normc":   (dict(dim=8, num_nearest_neighbors=7, norm_coors=True), 1, 45, 5, [3.0, 3.0, np.inf, 3.0, 3.0], "full", None),
    "adj_sparse":     (dict(dim=16, only_sparse_neighbors=True), 2, 30, 3, [3.0, 3.0, 3.0], "full", "chain"),
    "adj_knn":        (dict(dim=16, num_nearest_neighbors=5), 2, 26, 3, None, "padded", "chain"),
}


def build(name, seed=0, dtype=torch.float64):
    cfg, B, N, Cd, box, mask, adj = PCASES[name]
    spec = dict(kind="layer", cfg=cfg, B=B, N=N, C=Cd, seed=900 + seed, init="xavier", mask=mask or "none",
                adj=adj or "none")
    case = cases.build_case(spec)
    rs = np.random.RandomState(700 + seed)
    if box is None:                                  # [B, C]: one box per graph
        box = np.stack([rs.uniform(2.5, 4.0, Cd) for _ in range(B)])
        box[:, -1] = np.inf if Cd > 2 else box[:, -1]
    box = np.asarray(box, np.float64)
    scale = np.where(np.isfinite(box) & (box > 0), box, 3.0)
    case["inputs"]["coors"] = np.concatenate([lattice_coors(rs, 1, N, Cd, sc) for sc in np.broadcast_to(scale, (B, Cd))])
    if dtype != torch.float64:                       # the restatement sees the coordinates / features the kernels see
        case["inputs"]["coors"] = util.rounded(case["inputs"]["coors"], torch.float32)
    if dtype == torch.bfloat16:
        case["params"] = {k: util.rounded(v, torch.bfloat16) for k, v in case["params"].items()}
        for k in ("feats", "edges"):
            if k in case["inputs"]:
                case["inputs"][k] = util.rounded(case["inputs"][k], torch.bfloat16)
    return case, box


def knn_gap(case, box):
    """Smallest relative gap between the k-th and (k+1)-th rank over rows with k < N (tie-freedom of the inputs)."""
    cfg, ins = case["cfg"], case["inputs"]
    k = cfg["num_nearest_neighbors"]
    x = _t(ins["coors"])
    b, n, c = x.shape
    if k == 0 or k >= n or cfg["only_sparse_neighbors"] or ins.get("adj_mat") is not None:
        return 1.0
    d = (wrap(x[:, :, None] - x[:, None], box_bc(box, b, c)[:, None, None, :]) ** 2).sum(-1)
    if ins.get("mask") is not None:
        mk = torch.as_tensor(ins["mask"])
        d = d.masked_fill(~(mk[:, :, None] & mk[:, None, :]), 1e5)
    s = torch.sort(d, -1).values
    live = s[..., k] < 1e5                   # (masked candidates tie at 1e5; they never carry a message)
    return float(((s[..., k] - s[..., k - 1]) / s[..., k].clamp_min(1e-12))[live].min())


# ----------------------------------------------------------------------------- CPU: pin the restatement


ORACLE_CASES = ["dense_basic", "dense_mask_padded", "dense_fourier", "dense_everything", "dense_c5", "dense_mean_masked",
                "knn_basic", "knn_edges_mask", "knn_radius_mask", "knn_mean_fourier", "knn_k33",
                "adj_knn_chain", "adj_sparse_chain", "adj_sparse_random"]


@pytest.mark.parametrize("name", ORACLE_CASES)
@pytest.mark.parametrize("huge", [False, True])
def test_restatement_equals_the_oracle_without_a_box_and_with_a_huge_box(name, huge):
    case = cases.build_case(cases.SPECS[name])
    ins = case["inputs"]
    want = cases.run_oracle(case)
    box = np.full(ins["coors"].shape[-1], HUGE) if huge else None
    got = layer(case["params"], case["cfg"], ins["feats"], ins["coors"], ins.get("edges"), ins.get("mask"), ins.get("adj_mat"), box)
    assert np.abs(got[0].numpy() - want[0]).max() <= 1e-12 and np.abs(got[1].numpy() - want[1]).max() <= 1e-12


def supercell(case, box, k=None):
    """3^C images of every graph (aperiodic axes are not copied) and, for each central node, the nearest image of each
    partner: all N partners (dense) or its k nearest by wrapped distance.  -> (feats, coors, edges, mask, neighbors)
    of the supercell, central node i at index i; every other row lists nothing."""
    ins = case["inputs"]
    x = np.asarray(ins["coors"], np.float64)
    B, N, Cd = x.shape
    bx = np.broadcast_to(np.asarray(box, np.float64), (B, Cd))
    per = np.isfinite(bx[0]) & (bx[0] > 0)
    shifts = [np.array(s) for s in itertools.product(*[(0, -1, 1) if p else (0,) for p in per])]
    S = len(shifts)
    xs = np.concatenate([x + sh * np.where(per, bx, 0.0)[:, None, :] for sh in shifts], 1)      # [B, S*N, C]
    tile = lambda a, ax: np.concatenate([a] * S, ax)
    feats = tile(ins["feats"], 1)
    mask = None if ins.get("mask") is None else tile(ins["mask"], 1)
    edges = None
    if ins.get("edges") is not None:
        edges = tile(tile(ins["edges"], 1), 2)
    rel = x[:, :, None] - x[:, None]
    w = rel - np.where(per, bx, 0.0)[:, None, None] * np.round(rel / np.where(per, bx, 1.0)[:, None, None])
    if k is None:
        partners = np.broadcast_to(np.arange(N), (B, N, N))
    else:
        d = (w ** 2).sum(-1)
        partners = np.argsort(d, -1, kind="stable")[..., :k]
    nb = np.full((B, S * N, partners.shape[-1]), -1, np.int64)
    for b in range(B):
        for i in range(N):
            for s, j in enumerate(partners[b, i]):
                # the image of j at x_i - w_ij
                cand = np.where(np.abs(xs[b, j::N] - (x[b, i] - w[b, i, j])).max(-1) < 1e-9)[0]
                assert len(cand) == 1
                nb[b, i, s] = cand[0] * N + j
    return feats, xs, edges, mask, nb


SUPER = [("dense", dict(dim=8, edge_dim=2, soft_edges=True), 3, [2.0, 2.5, 3.0], "padded", None),
         ("dense_mean_normc", dict(dim=8, m_pool_method="mean", norm_coors=True, fourier_features=1), 3, [2.0, 2.5, 3.0], None, None),
         ("dense_c2_slab", dict(dim=8, coor_weights_clamp_value=0.3), 2, [2.5, np.inf], "random", None),
         ("knn", dict(dim=8, edge_dim=1, num_nearest_neighbors=4), 3, [2.0, 2.5, 3.0], None, 4),
         ("knn_c2_slab", dict(dim=8, num_nearest_neighbors=3), 2, [np.inf, 2.5], None, 3)]


@pytest.mark.parametrize("name,cfg,Cd,box,mask,k", SUPER, ids=[s[0] for s in SUPER])
def test_supercell_of_images_gives_the_periodic_forward_and_gradient(name, cfg, Cd, box, mask, k):
    """The central nodes of a 3^C supercell, each listing the nearest image of its partners, run through the existing
    edge-list oracles (forward and gradient) give the periodic layer; image gradients summed onto their originals give
    its gradients."""
    spec = dict(kind="layer", cfg=cfg, B=2, N=6, C=Cd, seed=77, init="xavier", mask=mask or "none")
    case = cases.build_case(spec)
    rs = np.random.RandomState(5)
    scale = np.where(np.isfinite(box), box, 3.0)
    case["inputs"]["coors"] = lattice_coors(rs, 2, 6, Cd, scale, shift=0)      # one box: 3^C images hold every nearest image
    ins, P, lc = case["inputs"], case["params"], case["cfg"]
    B, N = 2, 6
    f, xs, e, m, nb = supercell(case, box, k)
    S = xs.shape[1] // N
    got = layer(P, lc, ins["feats"], ins["coors"], ins.get("edges"), ins.get("mask"), None, np.asarray(box))
    # the edge-list oracle's rows follow its lists; a dense layer is the edge list over all N partners
    lcfg = dict(lc, num_nearest_neighbors=nb.shape[-1])
    want = O.egnn_layer_forward_edge_list(P, lcfg, f, xs, nb, e, m)
    assert np.abs(got[0].numpy() - want[0][:, :N]).max() <= 1e-12
    assert np.abs(got[1].numpy() - want[1][:, :N]).max() <= 1e-12

    gf, gx = rs.randn(B, N, lc["dim"]), rs.randn(B, N, Cd)
    g = layer_grads(case, np.asarray(box), gf, gx)
    pad = lambda a: np.concatenate([a, np.zeros((B, (S - 1) * N) + a.shape[2:])], 1)
    gs = G.egnn_layer_backward(P, lcfg, f, xs, e, m, None, pad(gf), pad(gx), neighbors=nb)
    fold = lambda a, ax: sum(np.take(a, range(s * N, (s + 1) * N), axis=ax) for s in range(S))
    want = {"in.feats": fold(gs["feats"], 1), "in.coors": fold(gs["coors"], 1)}
    if e is not None:
        want["in.edges"] = fold(fold(gs["edges"], 1), 2)
    want.update({f"p.{k2}": v for k2, v in gs["params"].items()})
    tol = 1e-7 if lc["norm_coors"] else 1e-11        # CoorsNorm: cancellation noise of the 1/eps self pair (util.grad_tol)
    util.compare(g, want, tol, f"{name}: periodic restatement gradient vs supercell gradient oracle")


@pytest.mark.parametrize("name", ["knn_k8", "knn_c2_fourier", "knn_c5_normc", "knn_k33"])
def test_periodic_knn_selection_is_a_stable_argsort_of_wrapped_distances(name):
    case, box = build(name)
    ins = case["inputs"]
    x = np.asarray(ins["coors"])
    B, N, Cd = x.shape
    bx = np.broadcast_to(box, (B, Cd))
    d = np.zeros((B, N, N))
    for c in range(Cd):                      # brute force, one axis at a time, in numpy
        r = x[:, :, None, c] - x[:, None, :, c]
        L = bx[:, c][:, None, None]
        if np.isfinite(L).all() and (L > 0).all():
            r = r - L * np.rint(r / L)
        d += r * r
    if ins.get("mask") is not None:
        mk = ins["mask"]
        d = np.where(mk[:, :, None] & mk[:, None, :], d, 1e5)
    want = np.argsort(d, -1, kind="stable")[..., :case["cfg"]["num_nearest_neighbors"]]
    got, _ = select(case["cfg"], (wrap(_t(x)[:, :, None] - _t(x)[:, None], _t(bx)[:, None, None, :]) ** 2).sum(-1),
                    ins.get("mask"), None)
    assert (got.numpy() == want).all()
    assert knn_gap(case, box) > 1e-5
    assert half_box_margin(x, box) >= 1e-3


@pytest.mark.parametrize("name", sorted(PCASES))
def test_inputs_keep_pairs_off_the_half_box_and_knn_ranks_tie_free(name):
    for dtype in (torch.float64, torch.float32, torch.bfloat16):
        case, box = build(name, dtype=dtype)
        assert half_box_margin(case["inputs"]["coors"], box) >= 1e-3
        assert knn_gap(case, box) > 1e-5


def _layer():
    from egnn_pytorch_b200 import EGNN
    return EGNN(dim=8)


@pytest.mark.parametrize("bad,msg", [
    (torch.ones(2), "shape"), (torch.ones(3, 3), "shape"), (torch.ones(2, 3, 1), "shape"),
    (torch.tensor([1.0, -1.0, 1.0]), ">= 0"), (torch.tensor([1.0, float("nan"), 1.0]), ">= 0"),
    (torch.ones(3, requires_grad=True), "requires_grad"), (torch.ones(3, dtype=torch.int64), "float"),
    ([1.0, 1.0, 1.0], "float")])
def test_box_misuse_raises_before_anything_launches(bad, msg):
    f, x = torch.randn(2, 5, 8), torch.randn(2, 5, 3)
    with pytest.raises(ValueError, match=msg):
        _layer()(f, x, box=bad)


def test_box_check_follows_the_tensor_not_its_address():
    """A checked box is not re-read while it is the same object at the same version; a new tensor (even one that
    reuses the freed storage of the last, at version 0) and an in-place write are checked again."""
    from egnn_pytorch_b200.egnn import _check_box
    cache = {}
    storage = torch.tensor([3.0, 3.0, 3.0, 7.0])
    good = storage[:3]
    _check_box(good, 2, 3, cache)
    _check_box(good, 2, 3, cache)                            # cached
    del good
    bad = storage[:3]                                        # same address, same version, a different tensor
    bad.data[1] = -1.0                                       # (a write that does not bump the version counter)
    assert bad.data_ptr() == storage.data_ptr() and bad._version == 0
    with pytest.raises(ValueError, match=">= 0"):
        _check_box(bad, 2, 3, cache)
    good = torch.tensor([3.0, 3.0, 3.0])
    _check_box(good, 2, 3, cache)
    good[1] = float("nan")                                   # an in-place write bumps the version
    with pytest.raises(ValueError, match=">= 0"):
        _check_box(good, 2, 3, cache)


def test_network_rejects_a_bad_box():
    from egnn_pytorch_b200 import EGNN_Network
    net = EGNN_Network(depth=1, dim=8)
    with pytest.raises(ValueError, match="requires_grad"):
        net(torch.randn(1, 4, 8), torch.randn(1, 4, 3), box=torch.ones(3, requires_grad=True))


def test_periodic_symbols_load_through_ctypes():
    from egnn_pytorch_b200 import _native as nat
    lib = nat.load()
    for name in ("egnn_layer_forward_periodic", "egnn_layer_backward_periodic"):
        assert name in nat.SYMBOLS and getattr(lib, name).argtypes is not None
    assert lib.egnn_abi_version() == 4
    # descriptor validation runs before anything touches the (absent) GPU
    desc = nat.LayerDesc(abi_version=3, dtype=nat.DTYPE_F32, B=1, N=4, C=3, dim=8, m_dim=16,
                         flags=nat.FLAG_UPDATE_FEATS | nat.FLAG_UPDATE_COORS)
    assert lib.egnn_layer_forward_periodic(C.byref(desc), None, None, None, None, None, 0, None) == -6
    assert lib.egnn_layer_backward_periodic(C.byref(desc), None, None, None, None, None, None, None, 0, None) == -6


# ----------------------------------------------------------------------------- GPU


DT = {"fp64": torch.float64, "fp32": torch.float32, "bf16": torch.bfloat16}
BF16_OK = {"dense", "dense_mask_soft_mean", "dense_everything_c5", "dense_c2", "dense_n257", "dense_n129_edges", "knn_k8",
           "knn_k32_edges", "knn_c2_fourier", "adj_sparse", "adj_knn"}


def _cdt(dtype):
    """Coordinates (and the box) are float64 on the fp64 path and float32 otherwise, bf16 layers included."""
    return torch.float64 if dtype == torch.float64 else torch.float32


def _run(case, box, dtype, dev="cuda"):
    mod = util.make_module(case, dtype, device=dev)
    ins = case["inputs"]
    t = lambda name: util.to_torch(ins.get(name), dtype, dev)
    b = None if box is None else torch.as_tensor(box, dtype=_cdt(dtype), device=dev)
    out = mod(t("feats"), util.to_torch(ins["coors"], _cdt(dtype), dev), t("edges"), mask=t("mask"), adj_mat=t("adj_mat"), box=b)
    return mod, out


def _check(case, out, want, dtype, what):
    if dtype == torch.bfloat16:                  # test_gpu_fast.py's tolerance of the tensor-core path
        f_scale = max(1e-3, float(np.abs(want[0]).max()))
        c_scale = float(np.abs(want[1] - case["inputs"]["coors"]).max())
        assert util.max_err(out[0], want[0]) <= 1e-2 * f_scale, what
        assert util.max_err(out[1], want[1]) <= 1e-2 * max(c_scale, 1.0), what
    else:                                        # the suite's tolerances, absolute ones scaled by the output's magnitude
        for o, w, part in ((out[0], want[0], " feats"), (out[1], want[1], " coors")):
            s = max(1.0, float(np.abs(w).max()))
            tol = dict(atol=1e-10 * s, rtol=1e-10) if dtype == torch.float64 else dict(atol=2e-5 * s, rtol=1e-4)
            util.assert_close(o, w, what=what + part, **tol)


PARITY = [(n, d) for n in sorted(PCASES) for d in ("fp64", "fp32", "bf16") if d != "bf16" or n in BF16_OK]


@pytest.mark.gpu
@pytest.mark.parametrize("name,dt", PARITY)
def test_forward_matches_the_periodic_restatement(name, dt):
    dtype = DT[dt]
    case, box = build(name, dtype=dtype)
    ins = case["inputs"]
    want = [t.numpy() for t in layer(case["params"], case["cfg"], ins["feats"], ins["coors"], ins.get("edges"),
                                     ins.get("mask"), ins.get("adj_mat"), box)]
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("error" if dtype == torch.bfloat16 else "default")    # no fp32 fallback for bf16
        mod, out = _run(case, box, dtype)
    if dtype == torch.bfloat16:
        assert mod.last_path == "bf16-tc"
    _check(case, out, want, dtype, f"{name} [{dt}]")


def _lists(case, k, seed=3):
    """Caller neighbour lists [B,N,k] with -1 slots, and per-slot edge features when the layer has edges."""
    B, N = case["inputs"]["feats"].shape[:2]
    rs = np.random.RandomState(seed)
    nb = np.stack([np.stack([rs.permutation(np.delete(np.arange(N), i))[:k] for i in range(N)]) for _ in range(B)])
    nb[:, ::3, -2:] = -1
    se = rs.randn(B, N, k, case["cfg"]["edge_dim"]) if case["cfg"]["edge_dim"] else None
    return nb, se


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32", "bf16"])
@pytest.mark.parametrize("name", ["dense_n129_edges", "dense_mask_soft_mean"])
def test_edge_list_mode_matches_the_restatement(name, dt):
    dtype = DT[dt]
    case, box = build(name, dtype=dtype)
    nb, se = _lists(case, 12)
    if se is not None and dtype == torch.bfloat16:
        se = util.rounded(se, torch.bfloat16)
    ins = case["inputs"]
    want = [t.numpy() for t in layer(case["params"], case["cfg"], ins["feats"], ins["coors"], None, ins.get("mask"),
                                     None, box, nb, se)]
    mod = util.make_module(case, dtype)
    t = lambda a: util.to_torch(a, dtype, "cuda")
    kw = dict(neighbors=torch.from_numpy(nb).cuda(), box=torch.as_tensor(box, dtype=torch.float64 if dt == "fp64" else torch.float32).cuda())
    if se is not None:
        kw["neighbor_edges"] = t(se)
    out = mod(t(ins["feats"]), util.to_torch(ins["coors"], _cdt(dtype), "cuda"), mask=t(ins.get("mask")), **kw)
    if dtype == torch.bfloat16:
        assert mod.last_path == "bf16-tc"
    _check(case, out, want, dtype, f"{name} lists [{dt}]")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32", "bf16"])
@pytest.mark.parametrize("name", ["dense", "dense_everything_c5", "knn_k8", "knn_k33", "adj_sparse"])
def test_a_huge_box_is_no_box(name, dt):
    dtype = DT[dt]
    if dt == "bf16" and name not in BF16_OK:
        pytest.skip("not a tensor-core configuration")
    case, box = build(name, dtype=dtype)
    _, ref = _run(case, None, dtype)
    _, out = _run(case, np.full(np.shape(box), HUGE), dtype)
    if dtype == torch.bfloat16:
        # the periodic tensor-core instantiations are compiled apart from the plain ones: the path's tolerance
        _check(case, out, [r.double().cpu().numpy() for r in ref], dtype, f"{name} huge box")
    else:                                        # same template, same arithmetic: bit for bit
        assert torch.equal(out[0], ref[0]) and torch.equal(out[1], ref[1])


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32", "bf16"])
@pytest.mark.parametrize("name", ["dense", "knn_k8", "knn_c5_normc", "dense_everything_c5"])
def test_lattice_shifts_of_single_nodes(name, dt):
    """Dyadic coordinates, power-of-two box: moving nodes by n L changes no feature bit and moves their coordinates by
    n L.  (The coordinates lie in [0, L/2) on periodic axes, so that no pair sits exactly on the half-box tie, where
    rounding half to even picks the image by the parity of n.)"""
    dtype = DT[dt]
    if dt == "bf16" and name not in BF16_OK:
        pytest.skip("not a tensor-core configuration")
    case, box = build(name, dtype=dtype)
    box = np.where(np.isfinite(box) & (box > 0), 4.0, box)
    rs0 = np.random.RandomState(6)
    x = rs0.randint(0, 2048, case["inputs"]["coors"].shape) / 1024.0
    case["inputs"]["coors"] = x
    _, ref = _run(case, box, dtype)
    rs = np.random.RandomState(1)
    B, N, Cd = x.shape
    n = np.zeros_like(x)
    who = rs.uniform(size=(B, N)) < 0.3
    per = np.isfinite(box) & (box > 0)
    n[who] = rs.randint(-2, 3, (int(who.sum()), Cd)) * per
    case["inputs"]["coors"] = x + n * 4.0
    _, out = _run(case, box, dtype)
    assert torch.equal(out[0], ref[0])
    got = out[1].double().cpu().numpy() - n * 4.0
    tol = 1e-12 if dtype == torch.float64 else 1e-5
    assert np.abs(got - ref[1].double().cpu().numpy()).max() <= tol * max(1.0, np.abs(x).max() + 8)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name", ["dense_mask_soft_mean", "knn_k8", "adj_knn"])
def test_translation_invariance(name, dt):
    dtype = DT[dt]
    case, box = build(name, dtype=dtype)
    _, ref = _run(case, box, dtype)
    t = np.random.RandomState(2).uniform(-7, 7, case["inputs"]["coors"].shape[-1])
    case["inputs"]["coors"] = case["inputs"]["coors"] + t
    _, out = _run(case, box, dtype)
    tol = dict(atol=1e-10, rtol=1e-10) if dtype == torch.float64 else dict(atol=1e-4, rtol=1e-4)
    util.assert_close(out[0], ref[0].double().cpu().numpy(), what="feats", **tol)
    util.assert_close(out[1], ref[1].double().cpu().numpy() + t, what="coors", **tol)


def _gpu_grads(case, box, dtype, neighbors=None, slot_edges=None):
    mod = util.make_module(case, dtype).requires_grad_(True)
    ins = case["inputs"]
    t = lambda a: util.to_torch(a, dtype, "cuda")
    f, x = t(ins["feats"]).requires_grad_(True), t(ins["coors"]).requires_grad_(True)
    e = t(slot_edges if slot_edges is not None else ins.get("edges"))
    leaves = {"in.feats": f, "in.coors": x}
    if e is not None:
        leaves["in.edges"] = e.requires_grad_(True)
    gf, gx = (torch.from_numpy(g).to(device="cuda", dtype=dtype) for g in cases.upstream_grads(case))
    bx = torch.as_tensor(box, dtype=dtype, device="cuda")
    kw = dict(mask=t(ins.get("mask")), box=bx)
    if neighbors is not None:
        kw["neighbors"] = torch.from_numpy(neighbors).cuda()
        if slot_edges is not None:
            kw["neighbor_edges"] = e
        e = None
    else:
        kw["adj_mat"] = t(ins.get("adj_mat"))
    with torch.enable_grad():
        fo, xo = mod(f, x, e, **kw)
        ((fo * gf).sum() + (xo * gx).sum()).backward()
    out = {k: v.grad.double().cpu().numpy() for k, v in leaves.items()}
    out.update({f"p.{k}": (torch.zeros_like(p) if p.grad is None else p.grad).double().cpu().numpy()
                for k, p in mod.named_parameters()})
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("saved", [True, False])
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name", ["dense_mask_soft_mean", "dense_everything_c5", "knn_k8", "knn_k33", "adj_knn", "lists"])
def test_gradients_match_the_restatement(name, dt, saved, monkeypatch):
    dtype = DT[dt]
    if not saved:
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")          # backward recomputes W2 silu(pre1)
    nb = se = None
    if name == "lists":
        case, box = build("dense_n129_edges", dtype=dtype)
        nb, se = _lists(case, 10)
    else:
        case, box = build(name, dtype=dtype)
    gf, gx = cases.upstream_grads(case)
    want = layer_grads(case, box, gf, gx, nb, se)
    got = _gpu_grads(case, box, dtype, nb, se)
    util.compare(got, want, 1e-9 if dtype == torch.float64 else 5e-4, f"{name} [{dt}] saved={saved}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["dense_everything_c5", "knn_k8"])
def test_fp64_gradient_matches_central_finite_differences(name):
    case, box = build(name)
    ins = case["inputs"]
    g = _gpu_grads(case, box, torch.float64)
    gf, gx = cases.upstream_grads(case)
    rs = np.random.RandomState(4)
    vf, vx = rs.randn(*ins["feats"].shape), rs.randn(*ins["coors"].shape)
    mod = util.make_module(case, torch.float64)
    bx = torch.as_tensor(box, device="cuda")

    def loss(s):
        c2 = dict(case, inputs=dict(ins, feats=ins["feats"] + s * vf, coors=ins["coors"] + s * vx))
        fo, xo = util.run_module(mod, c2, torch.float64, box=bx)
        return float((fo.cpu().numpy() * gf).sum() + (xo.cpu().numpy() * gx).sum())

    eps = 1e-6
    fd = (loss(eps) - loss(-eps)) / (2 * eps)
    an = float((g["in.feats"] * vf).sum() + (g["in.coors"] * vx).sum())
    assert abs(fd - an) <= 1e-6 * max(1.0, abs(an))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
def test_dropout_is_seeded_and_a_huge_box_keeps_its_masks(dt):
    dtype = DT[dt]
    case, box = build("knn_k8", dtype=dtype)
    mod = util.make_module(case, dtype, dropout=0.2).train()
    run = lambda b: util.run_module(mod, case, dtype, box=None if b is None else torch.as_tensor(b, dtype=dtype, device="cuda"))
    torch.manual_seed(3); a = run(box)
    torch.manual_seed(3); b = run(box)
    torch.manual_seed(3); c = run(np.full(3, HUGE))
    torch.manual_seed(3); d = run(None)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.equal(c[0], d[0]) and torch.equal(c[1], d[1])


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name", ["dense_mask_soft_mean", "knn_k8"])
def test_row_blocks_partition_forward_and_gradient(name, dt):
    dtype = DT[dt]
    case, box = build(name, dtype=dtype)
    ins = case["inputs"]
    N = ins["feats"].shape[1]
    mod = util.make_module(case, dtype).requires_grad_(True)
    t = lambda a: util.to_torch(a, dtype, "cuda")
    bx = torch.as_tensor(box, dtype=dtype, device="cuda")
    gf, gx = (torch.from_numpy(g).to(device="cuda", dtype=dtype) for g in cases.upstream_grads(case))

    def run(rows):
        f, x = t(ins["feats"]).requires_grad_(True), t(ins["coors"]).requires_grad_(True)
        mod.zero_grad()
        with torch.enable_grad():
            fo, xo = mod(f, x, mask=t(ins.get("mask")), box=bx, _rows=rows)
            ((fo * gf).sum() + (xo * gx).sum()).backward()
        grads = [f.grad, x.grad] + [p.grad.clone() for p in mod.parameters()]
        return fo.detach(), xo.detach(), grads

    fo, xo, gw = run(None)
    cut = [0, N // 3, N // 3 + 7, N]
    gsum = None
    for r0, r1 in zip(cut[:-1], cut[1:]):
        fb, xb, gb = run((r0, r1))
        assert torch.equal(fb[:, r0:r1], fo[:, r0:r1]) and torch.equal(xb[:, r0:r1], xo[:, r0:r1])
        # the identity rows outside the block carry the upstream gradient once per block: remove it before summing
        gb[0][:, :r0] -= gf[:, :r0]; gb[0][:, r1:] -= gf[:, r1:]
        gb[1][:, :r0] -= gx[:, :r0]; gb[1][:, r1:] -= gx[:, r1:]
        gsum = gb if gsum is None else [a + b for a, b in zip(gsum, gb)]
    tol = 1e-10 if dtype == torch.float64 else 1e-4
    for a, b in zip(gsum, gw):
        assert (a - b).abs().max().item() <= tol * max(1.0, b.abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32", "bf16"])
def test_network_passes_the_box_to_every_layer(dt):
    from egnn_pytorch_b200 import EGNN_Network
    dtype = DT[dt]
    torch.manual_seed(0)
    net = EGNN_Network(depth=3, dim=16, num_nearest_neighbors=6).to(dtype).cuda().eval()
    case, box = build("knn_k8", dtype=dtype)
    f = util.to_torch(case["inputs"]["feats"], dtype, "cuda")
    x = util.to_torch(case["inputs"]["coors"], torch.float64 if dt == "fp64" else torch.float32, "cuda").to(dtype)
    m = util.to_torch(case["inputs"]["mask"], dtype, "cuda")
    bx = torch.as_tensor(box, device="cuda", dtype=torch.float64 if dt == "fp64" else torch.float32)
    with torch.no_grad():
        fo, xo = net(f, x, mask=m, box=bx)
        f2, x2 = f, x
        for _, egnn in net.layers:
            f2, x2 = egnn(f2, x2, None, m, None, box=bx)
        fn, xn = net(f, x, mask=m)
    assert torch.equal(fo, f2) and torch.equal(xo, x2)
    assert not torch.equal(xo, xn)                          # the box changed the geometry


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
def test_network_with_degree_labels_trains_with_a_box(dt):
    from egnn_pytorch_b200 import EGNN_Network
    dtype = DT[dt]
    torch.manual_seed(0)
    net = EGNN_Network(depth=2, dim=16, num_tokens=10, num_adj_degrees=2, adj_dim=4, num_nearest_neighbors=5).to(dtype).cuda()
    B, N = 2, 24
    tok = torch.randint(0, 10, (B, N), device="cuda")
    rs = np.random.RandomState(9)
    x = torch.as_tensor(lattice_coors(rs, B, N, 3, [3.0, 3.0, 3.0]), dtype=dtype, device="cuda")
    adj = torch.as_tensor(cases.chain_adjacency(N), device="cuda")
    bx = torch.tensor([3.0, 3.0, 3.0], dtype=dtype, device="cuda")
    with torch.no_grad():
        a = net(tok, x, adj_mat=adj, box=torch.full((3,), HUGE, dtype=dtype, device="cuda"))
        b = net(tok, x, adj_mat=adj)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    target = x + 0.1
    losses = []
    for _ in range(20):
        opt.zero_grad()
        with torch.enable_grad():
            fo, xo = net(tok, x, adj_mat=adj, box=bx)
            loss = ((xo - target) ** 2).mean() + fo.pow(2).mean() * 1e-3
            loss.backward()
        opt.step()
        losses.append(loss.item())
    assert np.isfinite(losses).all() and losses[-1] < losses[0]


@pytest.mark.gpu
def test_the_same_module_rejects_a_bad_box_after_a_good_one():
    """Good box, then a new bad box of the same shape on the same module: the caching allocator hands the second the
    first one's block, and both are at version 0."""
    case, box = build("dense", dtype=torch.float32)
    mod = util.make_module(case, torch.float32)
    f = util.to_torch(case["inputs"]["feats"], torch.float32, "cuda")
    x = util.to_torch(case["inputs"]["coors"], torch.float32, "cuda")
    for bad in ([3.0, -1.0, 3.0], [3.0, float("nan"), 3.0]):
        good = torch.tensor([3.0, 3.0, 3.0], device="cuda")
        mod(f, x, box=good)
        del good
        b2 = torch.tensor(bad, device="cuda")
        assert b2._version == 0
        with pytest.raises(ValueError, match=">= 0"):
            mod(f, x, box=b2)
        del b2


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp32", "bf16"])
def test_graph_replay_follows_an_in_place_box_change(dt):
    from egnn_pytorch_b200.graphs import GraphedForward
    dtype = DT[dt]
    case, box = build("dense", dtype=dtype)
    mod = util.make_module(case, dtype)
    f = util.to_torch(case["inputs"]["feats"], dtype, "cuda")
    x = util.to_torch(case["inputs"]["coors"], torch.float32, "cuda")
    bx = torch.as_tensor(box, dtype=torch.float32, device="cuda")
    fast = GraphedForward(mod, f, x, box=bx)
    bx.mul_(1.125)                                        # a barostat step
    got = [t.clone() for t in fast(f, x)]
    with torch.no_grad():
        want = mod(f, x, box=bx.clone())
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
