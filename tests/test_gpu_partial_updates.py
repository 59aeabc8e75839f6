"""Layers that update only the features (`update_coors=False`) or only the coordinates (`update_feats=False`), and
coordinate dimensions C = 1, 4, 6 and 7, in every edge kernel, forward and backward.

Each update flag is a runtime branch in every kernel: the SIMT forward and its backward (bwd1's coordinate branch and
its pooled-message term, the GEMM roles, bwd2 / bwd3), the bf16 packer, tc_pair and tc_knn (the wide lists too), and
the identity copies of the output a layer does not update.  With `update_feats` off, `node_in` and `h1` take no
workspace and share their offset with the region after them, so a stale read or write there corrupts other scratch
without faulting: the poisoned-scratch test fills every workspace with 0xFF bytes (NaN in every float type) first.

Case tables (test_table_covers_every_boundary recomputes each boundary from the specs, through the launch mirrors
simt_layer and tc_layer of tests/launch_geometry.py):
  SIMT dense   PP = 2 and PP = 1 with a partial last 32-neighbour pass (N 33 / 70 / 97), the split hidden axis at 9 and
               32 CTAs, MP = 16 with a tail (m_dim 12) and MP = 32 (m_dim 20 / 24); soft edges, mean pooling over a
               mask, norm_feats (feats-only), CoorsNorm and clamp (coors-only)
  SIMT lists   TS = 1 / 4 / 8 / 32 and k = 33 (two slot passes), caller lists with -1 slots, per-slot edges, the kNN
               select with valid_radius and a mask, a depth-2 EGNN_Network with only_sparse_neighbors and degree labels
  lattices     a dense and a list case under a box and under a cell, with lattice_grad=True
  row blocks   a dense and a list partition whose blocks end inside a CTA
  new C        C = 1, 4, 6 and 7 with both flags on and with each flag off, dense and lists; boxes at C = 1 and 4
  bf16         tc_pair lean / generic at j-split 1 and > 1, N 63..65 / 127..129, a row range ending inside a row group;
               tc_knn lean / edges / generic at 8 and 16 rows, k = 1 / 31 / 32 and wide k = 33 / 64 / 65 with -1 slots;
               the small-node kernels and the tc_gemm tables + node GEMMs (feats-only); C = 1 / 4 / 6 / 7
Gates (each an existing, measured one):
  fp64 / fp32 forward   util.TOL against the float64 restatement (torch_reference, pinned here to the numpy oracle);
                        under a lattice test_triclinic._check
  gradients             util.grad_tol, with pre2 saved and recomputed (EGNN_B200_SAVE_PAIR_MB=0)
  lattice gradient      test_lattice_grad.check64 (1e-12 of scale) / check32 (4x the fp32 restatement's error)
  bf16                  test_gpu_tc_boundaries.TOL against tests/tc_reference.py, plus its fp64 oracle gate
  row blocks            the blocks' gradients sum to the whole gradient within 1e-12 of scale (fp64)
  dropout               test_gpu_dropout_reference's exact-mask gates, with stream 1 or 2 absent
  identity outputs      bit for bit: coors_out == coors without update_coors, feats_out == feats without update_feats
  poisoned scratch      outputs bit for bit against a zero-filled run; gradients at util.grad_tol and finite
CPU: the coverage tables, the restatement against the numpy oracle, and that each flag-off case fails its fp64 gate
against a reference that drops the only gradient path left (coors-only: the features detached from the edge MLP's
input; feats-only: the coordinates detached from the distance, which under a lattice is also the lattice gradient's
only source)."""
import contextlib
import ctypes as C
import functools

import numpy as np
import pytest
import torch

import cases
import launch_geometry as LG
import test_gpu_dropout_reference as DRT
import test_gpu_lattice_tile_boundaries as LTB
import test_gpu_radius_select as RS
import test_gpu_tc_boundaries as TCB
import test_gpu_tc_wide_lists as TCW
import test_triclinic as TRI
import torch_reference as R
import util
from test_edge_list import EDGE_CASES
from test_gpu_tile_boundaries import TILE_CASES
from test_lattice_grad import check32, check64

L, NW = "layer", "network"
FLAGS = {"feats": dict(update_coors=False), "coors": dict(update_feats=False), "both": {}}


def _variants(name, spec, tags=("feats", "coors"), feats=None, coors=None):
    """{name_tag: spec with the tag's flag}; `feats` / `coors`: options added to that variant only."""
    extra = {"feats": feats or {}, "coors": coors or {}, "both": {}}
    return {f"{name}_{t}": dict(spec, cfg=dict(spec["cfg"], **FLAGS[t], **extra[t])) for t in tags}


def _edge(name, **over):
    cfg, B, N, k, Cd, with_mask, init = EDGE_CASES[name]
    return dict(dict(kind=L, cfg=cfg, B=B, N=N, C=Cd, seed=1000, init=init, mask="padded" if with_mask else None, k=k),
                **over)


# spec: tests/cases.py spec plus [k] (caller lists of width k, -1 slots), [slot] (per-slot edges), [lat] (a lattice
# kind of test_gpu_lattice_tile_boundaries), [rows] (row-block cuts)
CASES = {}
# --- SIMT dense
CASES.update(_variants("n33_pp2_mean", TILE_CASES["dense_n33_hp72"], feats=dict(norm_feats=True)))
CASES.update(_variants("n70_hp144", TILE_CASES["dense_n70_hp144"]))
CASES.update(_variants("n97_hp296", TILE_CASES["dense_n97_hp296"]))
CASES.update(_variants("mdim12", TILE_CASES["dense_mdim12"], coors=dict(coor_weights_clamp_value=0.3)))
CASES.update(_variants("mdim20_soft", TILE_CASES["dense_mdim20_soft"]))
CASES.update(_variants("mdim24_pp1", TILE_CASES["dense_mdim24"], coors=dict(coor_weights_clamp_value=0.5)))
CASES.update(_variants("hsplit9", dict(kind=L, cfg=dict(dim=128), B=4, N=32, seed=1332, init="xavier", mask="padded")))
CASES.update(_variants("hsplit32", dict(kind=L, cfg=dict(dim=512), B=1, N=16, seed=1331, init="xavier")))
# --- SIMT lists
CASES.update(_variants("k1_ts1", dict(kind=L, cfg=dict(dim=16), B=2, N=20, seed=1401, init="xavier", k=1)))
CASES.update(_variants("k3_ts4", _edge("k3_q1")))
CASES.update(_variants("k6_ts8", _edge("plain"), coors=dict(norm_coors=True, coor_weights_clamp_value=0.5)))
CASES.update(_variants("k32_ts32", _edge("k32_q10")))
CASES.update(_variants("k33_two_passes", _edge("k33_mdim24")))
CASES.update(_variants("slot_k5", dict(kind=L, cfg=dict(dim=16, edge_dim=3, soft_edges=True), B=2, N=22, seed=1402,
                                       init="xavier", mask="random", k=5, slot=True)))
CASES.update(_variants("knn_radius", dict(kind=L, cfg=dict(dim=16, num_nearest_neighbors=7, valid_radius=1.2,
                                                            m_pool_method="mean"),
                                          B=2, N=30, seed=1403, init="xavier", mask="padded")))
CASES.update(_variants("net_sparse_labels", dict(kind=NW, cfg=dict(depth=2, dim=16, num_adj_degrees=2, adj_dim=4,
                                                                   only_sparse_neighbors=True),
                                                 B=2, N=24, seed=1404, init="xavier", adj="chain", mask="padded")))
# --- lattices (lattice_grad=True)
CASES.update(_variants("lat_dense_box", dict(TILE_CASES["dense_n33_hp72"], lat="box_per_graph")))
CASES.update(_variants("lat_dense_cell", dict(TILE_CASES["dense_n33_hp72"], lat="tilt")))
CASES.update(_variants("lat_list_box", _edge("k3_q1", lat="cubic")))
CASES.update(_variants("lat_list_cell", _edge("k3_q1", lat="tilt09")))
# --- row blocks ending inside a dense CTA (8 rows at PP = 2) and inside a list CTA (16 rows at TS = 8)
CASES.update(_variants("rows_dense", dict(TILE_CASES["dense_n45_hp128"], rows=[0, 13, 30, 45])))
CASES.update(_variants("rows_list", _edge("plain", rows=[0, 11, 24])))
# --- coordinate dimensions the other tables do not use, with both flags and with each flag off
NEW_C = (1, 4, 6, 7)
for _c in NEW_C:
    CASES.update(_variants(f"c{_c}_dense", dict(kind=L, cfg=dict(dim=16, edge_dim=1), B=2, N=35, C=_c, seed=1500 + _c,
                                                init="xavier", mask="padded"), tags=("both", "feats", "coors")))
    CASES.update(_variants(f"c{_c}_list", dict(kind=L, cfg=dict(dim=12, m_pool_method="mean"), B=2, N=30, C=_c,
                                               seed=1510 + _c, init="xavier", mask="random", k=9),
                           tags=("both", "feats", "coors")))
for _c, _lat in ((1, "box_per_graph"), (4, "cubic")):
    CASES.update(_variants(f"c{_c}_box", dict(kind=L, cfg=dict(dim=16), B=2, N=30, C=_c, seed=1520 + _c,
                                              init="xavier", lat=_lat), tags=("both", "feats", "coors")))


def flag_of(name):
    s = CASES[name]
    cfg = s["cfg"]
    return "coors" if cfg.get("update_feats") is False else ("feats" if cfg.get("update_coors") is False else "both")


def kind_of(name):
    return None if "lat" not in CASES[name] else LTB.lattice_kind(CASES[name])


def layer_cfg(case):
    return case["ncfg"]["layer"] if case["kind"] == NW else case["cfg"]


# ------------------------------------------------------------------ inputs and the float64 restatement


@functools.lru_cache(maxsize=None)
def build(name, dtype=torch.float64):
    """(case, lattice or None, caller lists or None, per-slot edges or None); a lattice case's coordinates and lattice
    are those of test_gpu_lattice_tile_boundaries (rounded to the compute type, wrap decisions off 1/2)."""
    s = CASES[name]
    if "lat" in s:
        case, lat, nb = LTB.build_spec(s, dtype)
        return case, lat, nb, None
    spec = {k: v for k, v in s.items() if k not in ("k", "rows", "slot")}
    spec["mask"] = spec.get("mask") or "none"
    if s.get("slot"):
        spec["dense_edges"] = False
    case = cases.build_case(spec)
    B, N = s["B"], s["N"]
    nb = LTB._lists(np.random.RandomState(77), B, N, s["k"]) if "k" in s else None
    se = np.random.RandomState(78).standard_normal((B, N, s["k"], s["cfg"]["edge_dim"])) if s.get("slot") else None
    return case, None, nb, se


def _rows(name):
    cuts = CASES[name].get("rows")
    return None if cuts is None else list(zip(cuts[:-1], cuts[1:]))


def ref_forward(name, dtype=torch.float64):
    case, lat, nb, se = build(name, dtype)
    if lat is not None:
        return LTB.ref_forward(case, lat, kind_of(name), nb)
    ins = case["inputs"]
    if case["kind"] == NW:
        fo, xo, _ = R.network(case["params"], case["ncfg"], ins["feats"], ins["coors"], ins.get("adj_mat"),
                              ins.get("edges"), ins.get("mask"))
    elif se is not None:
        fo, xo = R.layer(case["params"], case["cfg"], ins["feats"], ins["coors"], None, ins.get("mask"), None, None, nb,
                         se)
    else:
        fo, xo = R.layer_forward(case["params"], case["cfg"], ins["feats"], ins["coors"], ins.get("edges"),
                                 ins.get("mask"), ins.get("adj_mat"), None, nb)
    return fo.detach().numpy(), xo.detach().numpy()


def ref_grads(name, dtype=torch.float64, compute=torch.float64):
    """{'in.*', 'p.*', ['lattice']} of sum(fo gf) + sum(xo gx) in `compute` on the inputs of `dtype`, as numpy."""
    case, lat, nb, se = build(name, dtype)
    if lat is not None:
        return LTB.ref_grads(case, lat, kind_of(name), nb, dtype=compute)
    ins = case["inputs"]
    gf, gx = cases.upstream_grads(case)
    if case["kind"] == NW:
        g = R.network_grads(case["params"], case["ncfg"], ins["feats"], ins["coors"], gf, gx, ins.get("adj_mat"),
                            ins.get("edges"), ins.get("mask"), dtype=compute)
    else:
        g = R.layer_grads_chunked(case["params"], case["cfg"], ins["feats"], ins["coors"], gf, gx, ins.get("edges"),
                                  ins.get("mask"), ins.get("adj_mat"), None, nb, slot_edges=se)
    return {k: v.detach().double().numpy() for k, v in g.items()}


@functools.lru_cache(maxsize=None)
def _want(name, dtype):
    return ref_forward(name, dtype), ref_grads(name, dtype)


# ------------------------------------------------------------------ the layer on the device


def run(name, dtype, grad=False, rows=None, mod=None):
    """Forward (and with `grad` the backward of util's cotangents, the lattice a leaf) of the module ->
    ((fo, xo), (f_in, x_in), {'in.*', 'p.*', ['lattice']} float64 numpy or None, module)."""
    case, lat, nb, se = build(name, dtype)
    mod = mod or util.make_module(case, dtype)
    ins = case["inputs"]
    t = lambda a: util.to_torch(ins.get(a), dtype, "cuda")
    feats, edges = t("feats"), t("edges")
    x = util.to_torch(ins["coors"], LTB.cdt(dtype), "cuda")
    kw, leaves = {}, {}
    if lat is not None:
        kw[kind_of(name)] = LTB._lattice_tensor(lat, dtype, requires_grad=grad)
        kw["lattice_grad"] = grad
    if se is not None:
        edges = util.to_torch(se, dtype, "cuda")
    if grad:
        mod.requires_grad_(True)
        mod.zero_grad(set_to_none=True)
        leaves["in.coors"] = x.requires_grad_(True)
        if feats.is_floating_point():
            leaves["in.feats"] = feats.requires_grad_(True)
        if edges is not None:
            leaves["in.edges"] = edges.requires_grad_(True)
    with torch.enable_grad() if grad else torch.no_grad():
        if case["kind"] == NW:
            fo, xo = mod(feats, x, adj_mat=t("adj_mat"), edges=edges, mask=t("mask"), **kw)
        else:
            if nb is not None:
                kw["neighbors"] = torch.from_numpy(nb).cuda()
            if se is not None:
                kw["neighbor_edges"], edges = edges, None
            if rows is not None:
                kw["_rows"] = rows
            fo, xo = mod(feats, x, edges, mask=t("mask"), adj_mat=t("adj_mat"), **kw)
        if not grad:
            return (fo, xo), (feats, x), None, mod
        gf, gx = (torch.from_numpy(g).to(device="cuda", dtype=dtype) for g in cases.upstream_grads(case))
        fs, xs = fo, xo
        if rows is not None:
            fs, xs, gf, gx = (v[:, rows[0]:rows[1]] for v in (fo, xo, gf, gx))
        ((fs * gf).sum() + (xs * gx.to(xs.dtype)).sum()).backward()
    got = {k: v.grad.double().cpu().numpy() for k, v in leaves.items()}
    missing = [k for k, p in mod.named_parameters() if p.grad is None]
    assert not missing, f"{name}: parameters without a gradient: {missing}"
    got.update({f"p.{k}": p.grad.double().cpu().numpy() for k, p in mod.named_parameters()})
    if lat is not None:
        got["lattice"] = kw[kind_of(name)].grad.double().cpu().numpy()
    return (fo.detach(), xo.detach()), (feats.detach(), x.detach()), got, mod


def assert_identity(name, cfg, out, inp, rows=None):
    """The output a layer does not update is its input, bit for bit (all rows, inside and outside a row block)."""
    (fo, xo), (fi, xi) = out, inp
    if not cfg["update_coors"]:
        assert torch.equal(xo, xi), f"{name}: coors_out != coors in {int((xo != xi).any(-1).sum())} rows"
    if not cfg["update_feats"] and fi.is_floating_point():
        assert torch.equal(fo, fi), f"{name}: feats_out != feats in {int((fo != fi).any(-1).sum())} rows"


# ------------------------------------------------------------------ CPU: coverage


def case_geometry(name, rows=None):
    s = CASES[name]
    k = s.get("k") or s["cfg"].get("num_nearest_neighbors", 0)
    return dict(LG.simt_layer(s["kind"], s["cfg"], s["B"], s["N"], k=k, C=s.get("C", 3), rows=rows),
                flag=flag_of(name), lat=kind_of(name), net=s["kind"] == NW, slot=bool(s.get("slot")),
                select=bool(s["cfg"].get("num_nearest_neighbors")), radius="valid_radius" in s["cfg"],
                masked=s.get("mask") not in (None, "none"), cfg=s["cfg"])


def simt_boundaries():
    """{boundary: predicate over case_geometry} of the SIMT table; each must hold for a feats-only and a coors-only
    case (the new-C rows also for both flags on)."""
    dense = lambda g: g["k"] == 0 and not g["net"]
    lists = lambda g: g["k"] > 0
    return {
        "dense PP 2, partial last j pass": lambda g: dense(g) and g["PP"][4] == 2 and g["partial_j"] and g["j_passes"] >= 2,
        "dense PP 1 (fp64), partial last j pass": lambda g: dense(g) and g["PP"][8] == 1 and g["partial_j"],
        "dense N 97, Hp 296": lambda g: dense(g) and g["N"] == 97 and g["Hp"] == 296,
        "hsplit 9": lambda g: dense(g) and g["hsplit"] == 9,
        "hsplit 32": lambda g: dense(g) and g["hsplit"] == 32,
        "MP 16 with a tail": lambda g: dense(g) and g["MP"] == 16 and g["m"] < 16,
        "MP 32, m 20 and 24": lambda g: dense(g) and g["MP"] == 32 and g["m"] in (20, 24),
        "soft edges": lambda g: g["cfg"].get("soft_edges", False),
        "mean pooling over a mask": lambda g: g["cfg"].get("m_pool_method") == "mean" and g["masked"],
        "list TS 1": lambda g: lists(g) and g["TS"] == 1,
        "list TS 4": lambda g: lists(g) and g["TS"] == 4,
        "list TS 8": lambda g: lists(g) and g["TS"] == 8,
        "list TS 32": lambda g: lists(g) and g["TS"] == 32 and g["slot_passes"] == 1,
        "list k 33, two slot passes": lambda g: lists(g) and g["k"] == 33 and g["slot_passes"] == 2,
        "per-slot edges": lambda g: g["slot"],
        "kNN select, valid_radius, mask": lambda g: g["select"] and g["radius"] and g["masked"],
        "network, only_sparse_neighbors, degree labels": lambda g: g["net"] and g["labels"] > 0,
        "dense under a box": lambda g: dense(g) and g["lat"] == "box",
        "dense under a cell": lambda g: dense(g) and g["lat"] == "cell",
        "list under a box": lambda g: lists(g) and g["lat"] == "box",
        "list under a cell": lambda g: lists(g) and g["lat"] == "cell",
    }


FLAG_ONLY = {"norm_feats": "feats", "norm_coors": "coors", "coor_weights_clamp_value": "coors"}


def test_table_covers_every_boundary():
    """Each boundary of the SIMT, bf16 and new-C tables, for each flag, recomputed from the specs: removing a case
    (or editing its shape) so that a family x flag combination loses its partial tile fails here."""
    every = {n: case_geometry(n) for n in CASES}
    missing = [f"{what} [{flag}]" for what, ok in simt_boundaries().items() for flag in ("feats", "coors")
               if not any(ok(g) for g in every.values() if g["flag"] == flag)]
    for opt, flag in FLAG_ONLY.items():
        missing += [f"{opt} [{flag}]"] if not any(opt in g["cfg"] for g in every.values() if g["flag"] == flag) else []
    # row blocks ending inside a dense and a list CTA, for each flag
    for flag in ("feats", "coors"):
        for k_kind, inside in (("dense", lambda g: g["k"] == 0 and g["rows"] % (4 * g["PP"][8]) != 0),
                               ("list", lambda g: g["k"] > 0 and g["bwd3_partial"])):
            if not any(inside(case_geometry(n, r)) for n in CASES if flag_of(n) == flag and _rows(n) for r in _rows(n)):
                missing.append(f"row block ends inside a {k_kind} CTA [{flag}]")
    # C = 1, 4, 6, 7: dense and lists with each flag setting; boxes at C = 1 and 4
    for c in NEW_C:
        for flag in FLAGS:
            for fam, pick in (("dense", lambda g: g["k"] == 0), ("list", lambda g: g["k"] > 0)):
                if not any(pick(g) and g["C"] == c and g["flag"] == flag and g["lat"] is None for g in every.values()):
                    missing.append(f"C {c} {fam} [{flag}]")
    for c in (1, 4):
        for flag in FLAGS:
            if not any(g["C"] == c and g["flag"] == flag and g["lat"] == "box" for g in every.values()):
                missing.append(f"C {c} box [{flag}]")
    missing += tc_missing()
    missing += [f"dropout [{f}] {w}" for f, w in dropout_missing()]
    missing += [f"radius cell-grid select C {c} [{f}]" for c in (1, 2) for f in ("feats", "coors")
                if (c, f) not in {(c_, f_) for c_, f_, _ in RADIUS}]
    assert not missing, missing


# ------------------------------------------------------------------ CPU: the reference, and what the gates can see


PIN = [n for n in CASES if "lat" not in CASES[n] and not CASES[n].get("slot") and flag_of(n) != "both"
       and CASES[n]["B"] * CASES[n]["N"] <= 80]


@pytest.mark.parametrize("name", PIN)
def test_restatement_equals_the_numpy_oracle(name):
    """The float64 restatement the GPU tests compare with is the numpy oracle's function, with each flag off."""
    case, _, nb, _ = build(name)
    ins = case["inputs"]
    if nb is not None:
        want = cases.O.egnn_layer_forward_edge_list(case["params"], case["cfg"], ins["feats"], ins["coors"], nb,
                                                    edges=ins.get("edges"), mask=ins.get("mask"))
    else:
        want = cases.run_oracle(case)
    for g, w in zip(ref_forward(name), want):
        assert np.abs(g - w).max() <= 1e-12 * max(1.0, np.abs(w).max()), name


@contextlib.contextmanager
def dropped_path(flag):
    """torch_reference with the only gradient path a flag-off layer keeps cut: coors-only, the features detached from
    the edge MLP's input (features -> coordinate update); feats-only, the coordinates detached from the distance
    (coordinates -> features, and the lattice gradient's only source)."""
    real_cat, real_sum = torch.cat, torch.Tensor.sum
    state = {"on": False}

    def cat(ts, dim=0, **kw):
        if (flag == "coors" and len(ts) >= 3 and ts[0].dim() == 4 and (ts[0].stride(2) == 0 or ts[0].shape[2] == 1)
                and ts[1].shape[-1] == ts[0].shape[-1]):  # [f_i expanded over j, f_j, dist features, ...]: edge MLP input
            ts = [ts[0].detach(), ts[1].detach()] + list(ts[2:])
        return real_cat(ts, dim, **kw)

    def pow_sum(self, *a, **kw):
        out = real_sum(self, *a, **kw)
        if flag == "feats" and state["on"] and a == (-1,) and self.dim() == 4:
            out = out.detach()                         # dist = (rel ** 2).sum(-1)
        return out

    orig_layer = R.layer

    def layer(*a, **kw):
        state["on"] = True
        try:
            return orig_layer(*a, **kw)
        finally:
            state["on"] = False

    mp = pytest.MonkeyPatch()
    mp.setattr(R.torch, "cat", cat)
    mp.setattr(torch.Tensor, "sum", pow_sum)
    mp.setattr(R, "layer", layer)
    try:
        yield
    finally:
        mp.undo()


CUT = [n for n in CASES if flag_of(n) != "both" and CASES[n]["B"] * CASES[n]["N"] <= 100]


@pytest.mark.parametrize("name", CUT)
def test_a_dropped_gradient_path_fails_the_fp64_gate(name):
    """The restatement without the one gradient path the flag leaves fails util's fp64 gradient gate against the right
    one (under a lattice, the feats-only lattice gradient fails check64): a kernel that lost that path fails the case."""
    case, lat, _, _ = build(name)
    want = _want(name, torch.float64)[1]
    with dropped_path(flag_of(name)):
        got = ref_grads(name)
    glat, wlat = got.pop("lattice", None), want.get("lattice")
    with pytest.raises(AssertionError):
        util.compare(got, {k: v for k, v in want.items() if k != "lattice"}, util.grad_tol(case, torch.float64), name)
    if lat is not None and flag_of(name) == "feats":
        with pytest.raises(AssertionError):
            check64(glat, wlat, name)


# ------------------------------------------------------------------ GPU: SIMT forward, gradients, identity outputs

DT = {"fp64": torch.float64, "fp32": torch.float32}


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name", list(CASES))
def test_forward_matches_the_restatement(name, dt):
    dtype = DT[dt]
    case = build(name, dtype)[0]
    out, inp, _, mod = run(name, dtype)
    assert set(mod.state_dict()) == set(case["params"]), name
    assert_identity(name, layer_cfg(case), out, inp)
    want = _want(name, dtype)[0]
    LTB.report(f"forward-{dt}", name, [o.double().cpu().numpy() for o in out], want)
    if kind_of(name):
        TRI._check(case, out, want, dtype, f"{name} [{dt}]")
    else:
        util.assert_close(out[0], want[0], what=f"{name} feats [{dt}]", **util.TOL[dtype])
        util.assert_close(out[1], want[1], what=f"{name} coors [{dt}]", **util.TOL[dtype])


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["saved", "recomputed"])
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name", list(CASES))
def test_gradients_match_the_restatement(name, dt, mode, monkeypatch):
    """Every input and parameter gradient (parameters of the disabled MLP do not exist; every other one gets a
    gradient), and under a lattice the lattice gradient."""
    if mode == "recomputed":
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")
    dtype = DT[dt]
    case = build(name, dtype)[0]
    out, inp, got, _ = run(name, dtype, grad=True)
    assert_identity(name, layer_cfg(case), out, inp)
    want = _want(name, dtype)[1]
    what = f"{name} [{dt}] {mode}"
    glat, wlat = got.pop("lattice", None), want.get("lattice")
    plain = {k: v for k, v in want.items() if k != "lattice"}
    LTB.report(f"grads-{dt}", what, got, plain)
    util.compare(got, plain, util.grad_tol(case, dtype), what)
    if glat is not None:
        assert np.abs(wlat).max() > 1e-3
        if dtype == torch.float64:
            check64(glat, wlat, what)
        else:
            check32(glat, ref_grads(name, dtype, compute=torch.float32)["lattice"], wlat, what)


ROWS = [n for n in CASES if _rows(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ROWS)
def test_row_blocks_partition_forward_and_gradients(name):
    """fp64: a block's rows equal the whole forward bit for bit and its other rows equal the inputs; the blocks'
    gradients (EGNN_FLAG_ROW_PARTIAL_GRADS) sum to the whole gradient within 1e-12 of scale."""
    dtype = torch.float64
    case = build(name, dtype)[0]
    (fo, xo), _, whole, mod = run(name, dtype, grad=True)
    parts = []
    for r0, r1 in _rows(name):
        with torch.no_grad():
            out, inp, _, _ = run(name, dtype, rows=(r0, r1), mod=mod)
        assert_identity(name, layer_cfg(case), out, inp, rows=(r0, r1))
        for o, i in zip(out, inp):
            assert torch.equal(o[:, :r0], i[:, :r0]) and torch.equal(o[:, r1:], i[:, r1:]), (name, r0, r1)
        (fb, xb), _, g, _ = run(name, dtype, grad=True, rows=(r0, r1), mod=mod)
        assert torch.equal(fb[:, r0:r1], fo[:, r0:r1]) and torch.equal(xb[:, r0:r1], xo[:, r0:r1]), (name, r0, r1)
        parts.append(g)
    for k, w in whole.items():
        s = sum(p[k] for p in parts)
        LTB.report("rows-grads", f"{name} {k}", [s], [w])
        assert np.abs(s - w).max() <= 1e-12 * max(1.0, np.abs(w).max()), (name, k)


# ------------------------------------------------------------------ GPU: bf16 tensor cores

# test_gpu_tc_boundaries / test_gpu_tc_wide_lists specs (their `build`, `reference` and gates run them)
TC_CASES = {}
TC_CASES.update(_variants("pu_p_n63_lean", dict(kind=L, cfg=dict(dim=32, coor_weights_clamp_value=0.5), B=2, N=63,
                                                 seed=1601, mask="random")))
TC_CASES.update(_variants("pu_p_n64_mean", dict(kind=L, cfg=dict(dim=32, m_pool_method="mean"), B=2, N=64, seed=1602,
                                                 mask="padded"), feats=dict(norm_feats=True)))
TC_CASES.update(_variants("pu_p_n65_soft", dict(kind=L, cfg=dict(dim=24, soft_edges=True), B=2, N=65, seed=1603)))
TC_CASES.update(_variants("pu_p_n127_gen", dict(kind=L, cfg=dict(dim=16, fourier_features=1, edge_dim=2), B=2, N=127,
                                                 seed=1604, mask="padded")))
TC_CASES.update(_variants("pu_p_n128", dict(kind=L, cfg=dict(dim=32), B=2, N=128, seed=1605, mask="random"),
                          coors=dict(norm_coors=True)))
TC_CASES.update(_variants("pu_p_n129_gen", dict(kind=L, cfg=dict(dim=24, edge_dim=3, m_pool_method="mean"), B=2,
                                                 N=129, seed=1606)))
TC_CASES.update(_variants("pu_p_js4_range", dict(kind=L, cfg=dict(dim=24, fourier_features=2, edge_dim=4), B=2,
                                                  N=1024, seed=1607, rows=(0, 63), mask="padded")))
TC_CASES.update(_variants("pu_p_js8_range", dict(kind=L, cfg=dict(dim=16, coor_weights_clamp_value=2.0), B=1, N=2048,
                                                  seed=1608, rows=(5, 34))))
TC_CASES.update(_variants("pu_p_d72_gemm", dict(kind=L, cfg=dict(dim=72, m_pool_method="mean"), B=2, N=2100,
                                                 seed=1609, mask="padded",
                                                 check=[(0, 4), (1050, 1054), (2096, 2100)]), tags=("feats",)))
TC_CASES.update(_variants("pu_k1_lean8", dict(kind=L, cfg=dict(dim=32), B=2, N=203, k=1, seed=1621)))
TC_CASES.update(_variants("pu_k8_edges8_slot", dict(kind=L, cfg=dict(dim=64, edge_dim=4), B=2, N=150, k=8, seed=1622,
                                                     holes=True, slot_edges=True, mask="padded")))
TC_CASES.update(_variants("pu_k31_gen8_mean", dict(kind=L, cfg=dict(dim=32, fourier_features=2, m_pool_method="mean"),
                                                    B=2, N=100, k=31, seed=1623, holes=True)))
TC_CASES.update(_variants("pu_k32_lean16", dict(kind=L, cfg=dict(dim=344, coor_weights_clamp_value=3.0), B=1, N=150,
                                                 k=32, seed=1624, holes=True)))
TC_CASES.update(_variants("pu_k32_edges16", dict(kind=L, cfg=dict(dim=280, edge_dim=4), B=1, N=100, k=32, seed=1625,
                                                  holes=True, mask="random")))
TC_CASES.update(_variants("pu_k31_gen16_rows", dict(kind=L, cfg=dict(dim=264, fourier_features=2, edge_dim=1,
                                                                     m_pool_method="mean"), B=2, N=150, k=31,
                                                     seed=1626, holes=True, slot_edges=True, mask="padded",
                                                     rows=(19, 140))))
TC_CASES.update(_variants("pu_k8_gemm_tables", dict(kind=L, cfg=dict(dim=32, m_pool_method="mean"), B=1, N=5000, k=8,
                                                     seed=1627, holes=True,
                                                     check=[(0, 16), (2500, 2516), (4990, 5000)]), tags=("feats",)))
for _c in NEW_C:
    TC_CASES.update(_variants(f"pu_p_c{_c}", dict(kind=L, cfg=dict(dim=32, m_pool_method="mean"), B=2, N=90, C=_c,
                                                  seed=1640 + _c, mask="random"), tags=("both", "feats", "coors")))
    TC_CASES.update(_variants(f"pu_k_c{_c}", dict(kind=L, cfg=dict(dim=32, soft_edges=True), B=2, N=77, C=_c, k=8,
                                                  seed=1650 + _c, holes=True, mask="padded"),
                              tags=("both", "feats", "coors")))
WIDE_CASES = {}
WIDE_CASES.update(_variants("pu_w33_lean8", dict(kind=L, cfg=dict(dim=32), B=2, N=203, k=33, seed=1661, holes=True)))
WIDE_CASES.update(_variants("pu_w64_edges8_slot", dict(kind=L, cfg=dict(dim=64, edge_dim=4), B=2, N=150, k=64,
                                                       seed=1662, holes=True, slot_edges=True, mask="padded")))
WIDE_CASES.update(_variants("pu_w65_gen", dict(kind=L, cfg=dict(dim=264, fourier_features=1, m_pool_method="mean"),
                                                 B=1, N=120, k=65, seed=1663, holes=True, mask="random")))


# The rounded reference against the unrounded one at C = 1 (c_row of tc_reference with rounding=False): 0.34 on
# pu_k_c1_both and 0.15 on pu_p_c1_both, against 4.8e-3 on pu_k_c4_both.  test_c1_row_gate_is_dominated_by_rounding
# keeps that so.
C1_ROUNDING_C_ROW = 0.1


def _tc_flag(spec):
    cfg = spec["cfg"]
    return "coors" if cfg.get("update_feats") is False else ("feats" if cfg.get("update_coors") is False else "both")


def tc_missing():
    """The bf16 boundaries, for each flag (the node path: feats-only; the new C: each flag setting)."""
    geo = {n: dict(LG.tc_layer(s["kind"], s["cfg"], s["B"], s["N"], C=s.get("C", 3), k=s.get("k", 0), rows=s.get("rows")),
                   flag=_tc_flag(s), holes=bool(s.get("holes"))) for n, s in {**TC_CASES, **WIDE_CASES}.items()}
    missing = [n for n, g in geo.items() if not g["supported"]]
    pair = lambda g: g["k"] == 0
    want = {
        "tc_pair lean": lambda g: pair(g) and g["kernel"] == "tc_pair<lean>",
        "tc_pair generic": lambda g: pair(g) and g["kernel"] == "tc_pair<generic>",
        "tc_pair j-split 1": lambda g: pair(g) and g["jsplit"] == 1,
        "tc_pair j-split > 1": lambda g: pair(g) and g["jsplit"] > 1,
        "tc_pair N 63 / 64 / 65": None, "tc_pair N 127 / 128 / 129": None,
        "tc_pair j-split 4, row range ending with 3 valid rows": lambda g: pair(g) and g["rows_range"]
        and g["jsplit"] == 4 and g["last_rows_valid"] == 3,
        "tc_pair j-split 8, row range ending with 1 valid row": lambda g: pair(g) and g["rows_range"]
        and g["jsplit"] == 8 and g["last_rows_valid"] == 1,
        **{f"tc_knn<{m},{r}>": (lambda m, r: lambda g: g["k"] > 0 and g["kernel"] == f"tc_knn<{m},{r}>")(m, r)
           for m in ("LEAN", "EDGES", "GEN") for r in (8, 16)},
        **{f"tc_knn k {k}": (lambda k: lambda g: g["k"] == k)(k) for k in (1, 31, 32)},
        **{f"tc_knn wide k {k}, -1 slots": (lambda k: lambda g: g["k"] == k and g["holes"])(k) for k in (33, 64, 65)},
    }
    for flag in ("feats", "coors"):
        mine = [g for g in geo.values() if g["flag"] == flag]
        for what, ok in want.items():
            if ok is None:
                ns = {63, 64, 65} if "63" in what else {127, 128, 129}
                if not ns <= {g["N"] for g in mine if pair(g)}:
                    missing.append(f"bf16 {what} [{flag}]")
            elif not any(ok(g) for g in mine):
                missing.append(f"bf16 {what} [{flag}]")
    feats = [g for g in geo.values() if g["flag"] == "feats"]
    if not any(g["node"] == "small" and g["tables"] == "small" for g in feats):
        missing.append("bf16 small-node kernels [feats]")
    if not any(g["node"] == "tc_gemm" and g["tables"] == "tc_gemm" and g["B"] * g["N"] > 4096 for g in feats):
        missing.append("bf16 tc_gemm tables and node GEMMs [feats]")
    for c in NEW_C:
        for flag in FLAGS:
            for fam, pick in (("tc_pair", pair), ("tc_knn", lambda g: g["k"] > 0)):
                if not any(pick(g) and g["C"] == c and g["flag"] == flag for g in geo.values()):
                    missing.append(f"bf16 {fam} C {c} [{flag}]")
    return missing


def _tc_identity(spec, f, x, case):
    """Identity outputs of the bf16 path over every row (the whole graph outside a row range too, which the module
    copies from the inputs)."""
    ins = case["inputs"]
    cfg = spec["cfg"]
    if cfg.get("update_coors") is False:
        assert torch.equal(x.cpu().double(), torch.from_numpy(ins["coors"]))
    if cfg.get("update_feats") is False:
        assert torch.equal(f.cpu().double(), torch.from_numpy(ins["feats"]))


def test_c1_row_gate_is_dominated_by_rounding(monkeypatch):
    """At C = 1 the rounding the reference models moves some row's coordinate update by more than C1_ROUNDING_C_ROW of
    its value, far above TOL['c_row']: that gate cannot separate a kernel error from rounding there."""
    for name in ("pu_k_c1_both", "pu_p_c1_both"):
        monkeypatch.setitem(TCB.CASES, name, TC_CASES[name])
        g = TCB.gates(name, [(f, x) for _, f, x in TCB.reference(name, rounding=False)])
        assert g["c_row"] > C1_ROUNDING_C_ROW > TCB.TOL["c_row"], (name, g)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TC_CASES))
def test_bf16_matches_the_rounding_matched_reference(name, monkeypatch):
    monkeypatch.setitem(TCB.CASES, name, TC_CASES[name])
    f, x = TCB.run_gpu(name)
    _tc_identity(TC_CASES[name], f, x, TCB.build(name))
    assert np.isfinite(f.float().cpu().numpy()).all() and np.isfinite(x.cpu().numpy()).all()
    m = TCB.metrics(name, f, x)
    print(f"TCP {name} " + " ".join(f"{k}={v:.3e}" for k, v in m.items()))
    # At C = 1 a row's update is one signed sum whose rounding alone moves the worst row by C1_ROUNDING_C_ROW of its
    # value, so the per-row coordinate gate is reported there, not applied; the RMS and oracle gates still are.
    gated = [k for k in TCB.TOL if not (k == "c_row" and TC_CASES[name].get("C", 3) == 1)]
    bad = {k: m[k] for k in gated if not m[k] <= TCB.TOL[k]}
    assert not bad, (name, bad)
    x_in = TCB.build(name)["inputs"]["coors"]
    for w, of, ox in TCB.oracle(name):
        gf = f[:, w[0]:w[1]].double().cpu().numpy()
        gx = x[:, w[0]:w[1]].double().cpu().numpy()
        assert np.abs(gf - of).max() <= 1e-2 * max(1e-3, np.abs(of).max()), name
        assert np.abs(gx - ox).max() <= 1e-2 * max(np.abs(ox - x_in[:, w[0]:w[1]]).max(), 1.0), name


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(WIDE_CASES))
def test_bf16_wide_lists_match_the_rounding_matched_reference(name, monkeypatch):
    monkeypatch.setitem(TCW.CASES, name, WIDE_CASES[name])
    f, x = TCW.run_gpu(name)
    _tc_identity(WIDE_CASES[name], f, x, TCW.build(name))
    x_in = TCW.build(name)["inputs"]["coors"]
    m = TCW.gates(TCW.reference(name), x_in, [(f[:, w[0]:w[1]].double().cpu().numpy(),
                                               x[:, w[0]:w[1]].double().cpu().numpy()) for w in TCW.windows(name)])
    print(f"TCW {name} " + " ".join(f"{k}={v:.3e}" for k, v in m.items()))
    bad = {k: v for k, v in m.items() if not v <= TCB.TOL[k]}
    assert not bad, (name, bad)
    TCW.oracle_gate(name, TCW.oracle(name), x_in, f, x)


# ------------------------------------------------------------------ GPU: dropout with a flag off

DROPOUT_BASES = ["dense_pp2_soft", "dense_pp1_mdim24", "list_k40", "knn_k7_radius", "rows_knn"]
DROPOUT_CASES = {}
for _n in DROPOUT_BASES:
    DROPOUT_CASES.update(_variants(f"pu_{_n}", DRT.CASES[_n]))


def dropout_missing():
    """Each flag reaches the dense (PP 2 and PP 1), list, kNN-select and row-block dropout paths."""
    want = {"dense": lambda s: "lists" not in s and "rows" not in s, "lists": lambda s: s.get("lists") == "edge",
            "select": lambda s: s.get("lists") == "knn", "rows": lambda s: "rows" in s}
    return [(flag, what) for flag in ("feats", "coors") for what, ok in want.items()
            if not any(ok(s) and _tc_flag(s) == flag for s in DROPOUT_CASES.values())]


@pytest.fixture
def dropout_cases(monkeypatch):
    for n, s in DROPOUT_CASES.items():
        monkeypatch.setitem(DRT.CASES, n, s)


@pytest.mark.parametrize("name", list(DROPOUT_CASES))
def test_dropout_masks_bite_in_the_streams_the_flag_leaves(name, dropout_cases):
    """The restatement's masks drop and keep in every graph of each stream the layer has: edge (0), and coordinate (1)
    or node (2), never the disabled one."""
    _, ds = DRT._cpu_reference(name)
    want = {0, 1} if _tc_flag(DROPOUT_CASES[name]) == "coors" else {0, 2}
    for d in ds:
        assert set(d.seen) == want == DRT.streams(name), (name, sorted(d.seen))
        for stream, counts in d.seen.items():
            assert (counts > 0).all(), (name, stream, counts)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["saved", "recompute"])
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name", list(DROPOUT_CASES))
def test_dropout_matches_the_exact_mask_reference(name, dt, mode, dropout_cases, monkeypatch):
    if mode == "recompute":
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")
    got = DRT._minus_inputs(DRT.product(name, dt), name, dt, "cuda")
    want = DRT._gpu_reference(name, dt, torch.float64)
    assert set(got) == set(want), sorted(set(got) ^ set(want))
    if dt == "fp64":
        DRT.check_fp64(got, want, f"{name} [fp64, {mode}]")
    else:
        DRT.check_fp32(got, DRT._gpu_reference(name, dt, torch.float32), want, f"{name} [fp32, {mode}]")


# ------------------------------------------------------------------ GPU: poisoned scratch, NULL weights, back to back

_ES = {0: 4, 1: 8, 2: 2}          # element size per EGNN_DTYPE_*


class _Lib:
    """The native library with its layer entry points wrapped: each call records which weight and weight-gradient
    pointers were NULL, and with `fill` set the call's workspace -- and the outputs of whole-graph forwards and the input
    gradients of backwards -- are set to that byte first, on the call's stream."""

    def __init__(self, lib, fill=None):
        self._lib, self.fill, self.calls = lib, fill, []
        self._rt = C.CDLL("libcudart.so.12")

    def _memset(self, ptr, n, stream):
        if ptr and n:
            rc = self._rt.cudaMemsetAsync(C.c_void_p(ptr), C.c_int(self.fill), C.c_size_t(n), C.c_void_p(stream))
            assert rc == 0, rc

    def __getattr__(self, name):
        from egnn_pytorch_b200 import _native as nat
        fn = getattr(self._lib, name)
        if not name.startswith(("egnn_layer_forward", "egnn_layer_backward", "egnn_layer_pack_weights")) \
                or name.endswith("_bytes") or name == "egnn_layer_forward_host":
            return fn

        def call(*args):
            objs = [getattr(a, "_obj", None) for a in args]
            find = lambda t: next((o for o in objs if isinstance(o, t)), None)
            desc, w, io, gr = find(nat.LayerDesc), find(nat.LayerWeights), find(nat.LayerIO), find(nat.LayerGrads)
            null = lambda s: {f for f in nat.WEIGHT_FIELDS if not getattr(s, f)}
            self.calls.append((name, null(w), None if gr is None else null(gr.w)))
            if self.fill is not None and name != "egnn_layer_pack_weights":
                stream = args[-1].value
                self._memset(args[-3].value, args[-2], stream)
                ek, ec = _ES[desc.dtype], (8 if desc.dtype == 1 else 4)
                rows = desc.B * desc.N
                if gr is not None:
                    self._memset(gr.g_feats, rows * desc.dim * ek, stream)
                    self._memset(gr.g_coors, rows * desc.C * ec, stream)
                elif desc.row_begin == desc.row_end == 0:
                    self._memset(io.feats_out, rows * desc.dim * ek, stream)
                    self._memset(io.coors_out, rows * desc.C * ec, stream)
            return fn(*args)
        return call


@contextlib.contextmanager
def wrapped_lib(fill=None):
    from egnn_pytorch_b200 import _native as nat
    real = nat.load()
    lib = _Lib(real, fill)
    mp = pytest.MonkeyPatch()
    mp.setattr(nat, "load", lambda: lib)
    try:
        yield lib
    finally:
        mp.undo()


POISON = ["n33_pp2_mean_feats", "n33_pp2_mean_coors", "n97_hp296_feats", "n97_hp296_coors", "k6_ts8_feats",
          "k6_ts8_coors", "k33_two_passes_coors", "slot_k5_feats", "knn_radius_coors", "lat_list_cell_feats",
          "c4_dense_both", "c4_list_both", "c1_dense_coors", "hsplit32_feats"]
POISON_TC = ["pu_p_n129_gen_feats", "pu_p_n63_lean_coors", "pu_p_js8_range_coors", "pu_k8_edges8_slot_feats",
             "pu_k_c4_coors", "pu_k_c4_both"]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name", POISON)
def test_poisoned_scratch_changes_nothing(name, dt):
    """Workspaces (and the outputs the library writes) filled with 0xFF bytes before the forward and before the backward
    give the outputs of a zero-filled run bit for bit and finite gradients within util.grad_tol of it: no kernel reads
    scratch it did not write, and the backward reads only what the forward wrote."""
    dtype = DT[dt]
    case = build(name, dtype)[0]
    res = {}
    for fill in (0x00, 0xFF):
        with wrapped_lib(fill):
            out, inp, g, _ = run(name, dtype, grad=True)
            inf, _, _, _ = run(name, dtype)
        res[fill] = (out, inf, g)
        assert_identity(name, layer_cfg(case), out, inp)
    (o0, i0, g0), (o1, i1, g1) = res[0x00], res[0xFF]
    for a, b in zip(o0 + i0, o1 + i1):
        assert torch.equal(a, b), name
    for k, v in g1.items():
        assert np.isfinite(v).all(), (name, k)
    util.compare(g1, g0, util.grad_tol(case, dtype), f"{name} [{dt}] poisoned")
    if _rows(name) is None and CASES[name]["kind"] == L:
        r0, r1 = 3, CASES[name]["N"] - 5                     # one row-block forward
        outs = {}
        for fill in (0x00, 0xFF):
            with wrapped_lib(fill):
                outs[fill] = run(name, dtype, rows=(r0, r1))[0]
        assert all(torch.equal(a, b) for a, b in zip(outs[0x00], outs[0xFF])), name


@pytest.mark.gpu
@pytest.mark.parametrize("name", POISON_TC)
def test_poisoned_scratch_changes_nothing_bf16(name, monkeypatch):
    monkeypatch.setitem(TCB.CASES, name, TC_CASES[name])
    outs = {}
    for fill in (0x00, 0xFF):
        with wrapped_lib(fill):
            outs[fill] = TCB.run_gpu(name)
    assert all(torch.equal(a, b) for a, b in zip(outs[0x00], outs[0xFF])), name
    _tc_identity(TC_CASES[name], *outs[0xFF], TCB.build(name))


NULL_FIELDS = {"feats": {"coors_w1", "coors_b1", "coors_w2", "coors_b2"},
               "coors": {"node_w1", "node_b1", "node_w2", "node_b2"}}


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32", "bf16"])
@pytest.mark.parametrize("flag", ["feats", "coors"])
def test_the_library_takes_null_pointers_for_the_disabled_mlp(flag, dt):
    """egnn_layer_pack_weights, egnn_layer_forward and egnn_layer_backward run with NULL weight and weight-gradient
    pointers for the MLP the layer does not have (include/egnn_b200.h); the other pointers are all set."""
    from egnn_pytorch_b200 import EGNN
    torch.manual_seed(5)
    dtype = {"fp64": torch.float64, "fp32": torch.float32, "bf16": torch.bfloat16}[dt]
    mod = EGNN(dim=64, edge_dim=2, soft_edges=True, norm_feats=True, norm_coors=True, **FLAGS[flag]).to(dtype).cuda()
    f = torch.randn(2, 40, 64, device="cuda", dtype=dtype)
    x = torch.randn(2, 40, 3, device="cuda", dtype=torch.float64 if dt == "fp64" else torch.float32)
    e = torch.randn(2, 40, 40, 2, device="cuda", dtype=dtype)
    with wrapped_lib() as lib:
        if dt == "bf16":
            mod(f, x, e)
            assert mod.last_path == "bf16-tc"
        else:
            with torch.enable_grad():
                fo, xo = mod(f, x, e)
                (fo.sum() + xo.sum()).backward()
    names = {c[0] for c in lib.calls}
    assert "egnn_layer_pack_weights" in names and "egnn_layer_forward" in names
    assert dt == "bf16" or "egnn_layer_backward" in names
    for name, wnull, gnull in lib.calls:
        assert wnull == NULL_FIELDS[flag] | {"label_emb"}, (name, wnull)
        assert gnull is None or gnull == NULL_FIELDS[flag] | {"label_emb"}, (name, gnull)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_back_to_back_layers_on_one_stream(dtype, monkeypatch):
    """A feats-only, a full and a coors-only layer share the per-stream cached workspace; each gives exactly the
    outputs it gives run alone on a fresh workspace."""
    from egnn_pytorch_b200 import EGNN, egnn as E
    torch.manual_seed(11)
    B, N, d = 2, 150, 64
    layers = [EGNN(dim=d, m_pool_method="mean", **FLAGS[t]).to(dtype).cuda().eval() for t in ("feats", "both", "coors")]
    for l in layers:
        for p in l.parameters():
            torch.nn.init.normal_(p, std=0.2)
    f = torch.randn(B, N, d, device="cuda").to(dtype)
    x = torch.randn(B, N, 3, device="cuda")
    mask = torch.rand(B, N, device="cuda") < 0.9
    alone = []
    with torch.no_grad():
        for l in layers:
            monkeypatch.setattr(E, "_WORKSPACES", {})
            alone.append(l(f, x, mask=mask))
        monkeypatch.setattr(E, "_WORKSPACES", {})
        together = [l(f, x, mask=mask) for l in layers]
    for t, (a, b) in zip(("feats", "both", "coors"), zip(alone, together)):
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), t
    assert torch.equal(together[0][1], x) and torch.equal(together[2][0], f)


# ------------------------------------------------------------------ GPU: the layer's cell-grid select at C = 1 and 2

# (C, flag, dtype)
RADIUS = [(c, f, dt) for c in (1, 2) for f in ("feats", "coors") for dt in (torch.float64, torch.float32, torch.bfloat16)]


@pytest.mark.gpu
@pytest.mark.parametrize("c,flag,dtype", RADIUS, ids=[f"c{c}-{f}-{str(d)[6:]}" for c, f, d in RADIUS])
def test_cell_grid_select_in_the_layer_is_bit_identical_to_all_pairs(c, flag, dtype, monkeypatch):
    from egnn_pytorch_b200 import _native as nat, EGNN
    lib = nat.load()
    torch.manual_seed(3)
    dim = 64 if dtype == torch.bfloat16 else 24
    mod = EGNN(dim=dim, num_nearest_neighbors=16, valid_radius=1.0, **FLAGS[flag]).to(RS.DEV, dtype)
    x, mask, _ = RS.cloud(2, 700, c=c, dtype=torch.float64 if dtype == torch.float64 else torch.float32, seed=5 + c)
    feats = torch.randn((2, 700, dim), device=RS.DEV).to(dtype)
    with torch.no_grad():
        cell, allp = RS.both_paths(lib, monkeypatch, lambda: mod(feats, x, mask=mask))
    if dtype == torch.bfloat16:
        assert mod.last_path == "bf16-tc"
    for a, w, what in zip(cell, allp, ("feats", "coors")):
        assert torch.equal(RS.bits(a), RS.bits(w)), f"C {c} {flag} {dtype} {what}"
    assert torch.equal(cell[1] if flag == "feats" else cell[0], x if flag == "feats" else feats)
