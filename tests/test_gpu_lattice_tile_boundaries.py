"""Tile boundaries of the periodic fp32 / fp64 edge kernels, their backward and the lattice gradient (`box=`, `cell=`,
`lattice_grad=True`), against the float64 restatement.

Every periodic SIMT kernel is its own instantiation (PBC_BOX, PBC_CELL), and bwd3 has a fourth with LAT = true for the
lattice gradient.  The shapes of test_gpu_tile_boundaries.TILE_CASES and test_edge_list.EDGE_CASES run here under a
lattice, the kinds alternating along the table (boxes: cubic, per graph, an aperiodic axis given as 0 in one graph and
inf in another, C = 5 on the generic path; cells: tilt, tilt09, per_graph with B >= 3, hex_slab with z aperiodic, c2),
plus rows the non-periodic tables do not need: the split hidden axis (dim 512, N 16 and dim 128, B N^2 = 4096), the
largest fp64 configurations that still train (m_dim 30, and 23 with soft edges), row blocks that end inside a dense
and a list CTA, and networks with 4 and 16 degree-label rows.  test_table_covers_every_lattice_boundary recomputes
from the specs, through launch_geometry.simt_layer, that each boundary is reached under a box and under a cell.

Inputs: coordinates from test_triclinic.cell_coors (a box is a diagonal cell), rounded to the compute type, so every
wrap decision is at least 1e-3 from 1/2; each case wraps at least 20 % of the pairs it compares.

Gates (none looser than its neighbours'):
  forward            test_triclinic._check: fp64 atol 1e-10 of scale, rtol 1e-10; fp32 atol 2e-5 of scale, rtol 1e-4
  input / parameter  util.grad_tol: fp64 1e-9 (1e-7 with CoorsNorm), fp32 5e-4 of max(1, scale)
  lattice gradient   test_lattice_grad.check64 (fp64: 1e-12 of scale) and check32 (fp32: 4x the fp32 restatement's
                     error); exactly 0 above the diagonal and on aperiodic axes
  diagonal cell      the box's forward bit for bit; its lattice-gradient diagonal the box gradient to 1e-13 (fp64) /
                     1e-6 (fp32) of scale, the fp64 atomics' rounding
The all-pairs select under a cell (fp32 and fp64) and under fp64 boxes is checked through the layer: its own select
(the cell grid forced off) against the same layer run with `neighbors=` set to the exact reference lists of
`cell_select`, bit for bit, at 8 and 16 warps with 1 and 3 staging passes, the CDIM = 3 and generic instantiations, the
block sort at k = 40 and 64 around an Npad step, and mask + valid_radius.

CPU: the coverage tables, the input margins, the Fraction pin of the select reference, and that each lattice case fails
its fp64 gate under a wrong lattice (no lattice, the next graph's, a cell's diagonal, the axes wrapped first to last,
floor for rint).
GPU: the comparisons above, fp64 training rejected over the shared-memory budget under a lattice, row blocks, and the
launched kernels' template arguments and grids against launch_geometry.simt_layer under torch.profiler.

Worst measured value per gate, on an NVIDIA H100 80GB HBM3 at its 700 W power limit (error over max(1, scale)):
  forward            fp64 1.8e-15 (net_labels4_tilt09); fp32 7.3e-7 (net_labels4_cubic)
  input / parameter  fp64 1.4e-9 (list_k32_q10_hex_slab, CoorsNorm: gate 1e-7); fp32 5.1e-5 (net_labels16_aperiodic)
  lattice gradient   fp64 2.5e-15 of scale (hsplit512_cubic); fp32 1.23x the fp32 restatement's error, 1.2e-6 of
                     scale (list_k32_q10_box_pg)
  diagonal cell      fp64 3.8e-16, fp32 1.0e-7 of the box gradient's scale (hsplit512_cubic)
  row-block sums     gradients 8.7e-15 (rows_dense_cubic), lattice gradient 4.6e-16 (rows_list_box_pg)
  select             every list bit for bit
The file runs in 62 s with a peak of 88 MB of device memory."""
import contextlib
import functools
import json
import math
import os
import re
import tempfile

import numpy as np
import pytest
import torch

import cases
import launch_geometry as LG
import tc_reference as T
import test_triclinic as TRI
import torch_reference as R
import util
import test_edge_list
from test_edge_list import EDGE_CASES
from test_gpu_tile_boundaries import FP64_BACKWARD_REJECTED, TILE_CASES, _assert_training_forward_rejected
from test_lattice_grad import check32, check64

L, NW = "layer", "network"
BOXES = ("cubic", "box_per_graph", "box_aperiodic", "box_c5")
CELLS = ("tilt", "tilt09", "per_graph", "hex_slab", "c2")


def _tile(name, lat, **over):
    return dict(TILE_CASES[name], lat=lat, **over)


def _edge(name, lat, **over):
    cfg, B, N, k, Cd, with_mask, init = EDGE_CASES[name]
    spec = dict(kind=L, cfg=cfg, B=B, N=N, C=Cd, seed=1000, init=init, mask="padded" if with_mask else None, k=k, lat=lat)
    spec.update(over)
    return spec


# name: spec of tests/cases.py plus lat (lattice kind), [k] (neighbour lists of width k), [rows] (row-block cuts)
CASES = {
    # --- the dense shapes of TILE_CASES
    "n33_hp72_tilt":          _tile("dense_n33_hp72", "tilt"),
    "n70_hp144_per_graph":    _tile("dense_n70_hp144", "per_graph", B=3),
    "n97_hp296_box_pg":       _tile("dense_n97_hp296", "box_per_graph"),
    "n97_hp296_tilt09":       _tile("dense_n97_hp296", "tilt09"),
    "net_labels4_tilt09":     _tile("net_n45_labels4", "tilt09"),
    "net_labels4_cubic":      _tile("net_n45_labels4", "cubic"),
    "net_labels16_aperiodic": _tile("net_n45_labels16", "box_aperiodic"),
    "net_labels16_hex_slab":  _tile("net_n45_labels16", "hex_slab"),
    "mdim12_c2":              _tile("dense_mdim12", "c2", C=2),
    "mdim20_soft_cubic":      _tile("dense_mdim20_soft", "cubic"),
    "mdim24_hex_slab":        _tile("dense_mdim24", "hex_slab"),
    "mdim24_soft_box_pg":     _tile("dense_mdim24_soft", "box_per_graph"),
    "mdim32_aperiodic":       _tile("dense_mdim32", "box_aperiodic"),
    "q77_tilt":               _tile("dense_q77", "tilt"),
    "q77_cubic":              _tile("dense_q77", "cubic"),
    # --- the largest fp64 configurations that train, with the periodic kernels' static shared memory
    "mdim30_cubic":     dict(kind=L, cfg=dict(dim=12, m_dim=30, edge_dim=1), B=2, N=40, seed=321, init="xavier",
                             mask="random", lat="cubic"),
    "mdim30_tilt":      dict(kind=L, cfg=dict(dim=12, m_dim=30, edge_dim=1), B=2, N=40, seed=321, init="xavier",
                             mask="random", lat="tilt"),
    "mdim23_soft_box":  dict(kind=L, cfg=dict(dim=12, m_dim=23, soft_edges=True), B=2, N=35, seed=322, init="xavier",
                             mask="padded", lat="box_per_graph"),
    "mdim23_soft_cell": dict(kind=L, cfg=dict(dim=12, m_dim=23, soft_edges=True), B=3, N=35, seed=322, init="xavier",
                             mask="padded", lat="per_graph"),
    # --- the split hidden axis: 32 hidden CTAs (the README / BASELINE c1 shape) and 9 (B N^2 = 4096 exactly)
    "hsplit512_cubic":  dict(kind=L, cfg=dict(dim=512), B=1, N=16, seed=331, init="xavier", lat="cubic"),
    "hsplit512_tilt":   dict(kind=L, cfg=dict(dim=512), B=1, N=16, seed=331, init="xavier", lat="tilt"),
    "hsplit128_box_pg": dict(kind=L, cfg=dict(dim=128), B=4, N=32, seed=332, init="xavier", mask="padded",
                             lat="box_per_graph"),
    "hsplit128_cell_pg": dict(kind=L, cfg=dict(dim=128), B=4, N=32, seed=332, init="xavier", mask="padded",
                              lat="per_graph"),
    # --- row blocks ending inside a dense CTA (8 rows at PP = 2) and inside a list CTA (16 rows at TS = 8)
    "rows_dense_cubic": _tile("dense_n45_hp128", "cubic", rows=[0, 13, 30, 45]),
    "rows_dense_tilt":  _tile("dense_n45_hp128", "tilt", rows=[0, 13, 30, 45]),
    "rows_list_box_pg": _edge("plain", "box_per_graph", rows=[0, 11, 24]),
    "rows_list_tilt09": _edge("plain", "tilt09", rows=[0, 11, 24]),
    # --- the neighbour-list shapes of EDGE_CASES
    "list_edges_mask_cubic":  _edge("edges_mask", "cubic"),
    "list_mean_mask_per_graph": _edge("mean_mask", "per_graph", B=3),
    "list_mean_nomask_aperiodic": _edge("mean_nomask", "box_aperiodic"),
    "list_fourier_c5":        _edge("fourier_c5", "box_c5", B=2),
    "list_k33_tilt09":        _edge("k33", "tilt09"),
    "list_k3_q1_cubic":       _edge("k3_q1", "cubic"),
    "list_k3_q1_hex_slab":    _edge("k3_q1", "hex_slab"),
    "list_k17_q5_c2":         _edge("k17_q5_c2", "c2"),
    "list_k17_q5_c2_box":     _edge("k17_q5_c2", "box_per_graph"),
    "list_k32_q10_hex_slab":  _edge("k32_q10", "hex_slab"),
    "list_k32_q10_box_pg":    _edge("k32_q10", "box_per_graph", B=2),
    "list_k48_c5_mean":       _edge("k48_c5_mean", "box_c5"),
    "list_k64_q1_box_pg":     _edge("k64_q1", "box_per_graph", B=2),
    "list_k64_q1_tilt":       _edge("k64_q1", "tilt"),
    "list_k33_mdim24_per_graph": _edge("k33_mdim24", "per_graph", B=3),
    "list_k33_mdim24_aperiodic": _edge("k33_mdim24", "box_aperiodic"),
}
FP64_REJECTED = {n for n, s in CASES.items() if any(s["cfg"] == TILE_CASES[r]["cfg"] for r in FP64_BACKWARD_REJECTED)}


def kind_of(name):
    return lattice_kind(CASES[name])


# ------------------------------------------------------------------ inputs


def _diag_cell(Ls):
    """[..., C] box lengths -> the diagonal cell [..., C, C] (0 off the diagonal, also next to an inf)."""
    Ls = np.asarray(Ls, np.float64)
    A = np.zeros(Ls.shape + Ls.shape[-1:])
    A[..., np.arange(Ls.shape[-1]), np.arange(Ls.shape[-1])] = Ls
    return A


def make_lattice(kind, B, Cd, rs):
    """-> (lattice as the module takes it, the same lattice as a lower-triangular cell [B, C, C])."""
    if kind in CELLS:
        cell = TRI.make_cell(kind, B, rs)
        assert cell.shape[-1] == Cd, (kind, Cd)
        return cell, TRI.cell_bc(cell, B, Cd)
    if kind == "cubic":
        L = np.full(Cd, 3.1)
    elif kind in ("box_per_graph", "box_c5"):
        L = rs.uniform(2.8, 3.6, (B, Cd))
    elif kind == "box_aperiodic":
        assert B >= 2
        L = rs.uniform(2.8, 3.6, (B, Cd))
        L[0, Cd - 1], L[1, 1] = 0.0, np.inf
    else:
        raise KeyError(kind)
    return L, _diag_cell(np.broadcast_to(L, (B, Cd)))


def _lists(rs, B, N, k):
    """test_edge_list.build's lists: random partners, empty slots, a node without neighbours, a self edge."""
    nb = np.stack([np.stack([rs.permutation(N)[:k] for _ in range(N)]) for _ in range(B)]).astype(np.int64)
    nb[:, ::3, -2:] = -1
    nb[0, 5, :] = -1
    nb[:, 7, 0] = 7
    return nb


def cdt(dtype):
    return torch.float64 if dtype == torch.float64 else torch.float32


def lattice_kind(spec):
    return "box" if spec["lat"] in BOXES else "cell"


def build_spec(full, dtype=torch.float64):
    """(case, lattice, neighbour lists or None) of a table spec; lattice and coordinates rounded to the compute type."""
    spec = {k: v for k, v in full.items() if k not in ("lat", "k", "rows")}
    spec["mask"] = spec.get("mask") or "none"
    case = cases.build_case(spec)
    B, N, Cd = spec["B"], spec["N"], spec.get("C", 3)
    rs = np.random.RandomState(spec["seed"] + 17)
    lat, cell = make_lattice(full["lat"], B, Cd, rs)
    lat, cell = util.rounded(lat, cdt(dtype)), util.rounded(cell, cdt(dtype))
    case["inputs"]["coors"] = TRI.cell_coors(rs, B, N, cell, dtype=cdt(dtype))
    for _ in range(20):           # a network's later layers wrap the coordinates the earlier ones moved
        if case["kind"] != NW or _layer_margin(case, lat, cell, lattice_kind(full)) > 1e-4:
            break
        case["inputs"]["coors"] = TRI.cell_coors(rs, B, N, cell, dtype=cdt(dtype))
    nb = _lists(np.random.RandomState(77), B, N, full["k"]) if "k" in full else None
    return case, lat, nb


@functools.lru_cache(maxsize=None)
def build(name, dtype=torch.float64):
    """build_spec of a CASES entry, once per (name, dtype)."""
    return build_spec(CASES[name], dtype)


def _layer_margin(case, lat, cell, kind):
    """Smallest wrap margin over the inputs of a network's layers (the restatement's)."""
    ins = case["inputs"]
    with _reference_geometry(kind):
        _, _, states = R.network(case["params"], case["ncfg"], ins["feats"], ins["coors"], ins.get("adj_mat"),
                                 ins.get("edges"), ins.get("mask"), lat)
    return min(float(TRI.wrap_margin(xs.numpy(), cell).min()) for _, xs in states)


def _rows(name):
    cuts = CASES[name].get("rows")
    return None if cuts is None else list(zip(cuts[:-1], cuts[1:]))


# ------------------------------------------------------------------ the float64 restatement


def _reference_geometry(kind):
    return TRI._cell_geometry() if kind == "cell" else contextlib.nullcontext()


def ref_forward(case, lat, kind, nb):
    ins = case["inputs"]
    with _reference_geometry(kind):
        if case["kind"] == NW:
            fo, xo, _ = R.network(case["params"], case["ncfg"], ins["feats"], ins["coors"], ins.get("adj_mat"),
                                  ins.get("edges"), ins.get("mask"), lat)
        else:
            fo, xo = R.layer_forward(case["params"], case["cfg"], ins["feats"], ins["coors"], ins.get("edges"),
                                     ins.get("mask"), ins.get("adj_mat"), lat, nb)
    return fo.numpy(), xo.numpy()


def ref_grads(case, lat, kind, nb, dtype=torch.float64):
    """{'in.*', 'p.*', 'lattice'} of sum(fo gf) + sum(xo gx) (util's cotangents), the lattice a leaf, as numpy."""
    ins = case["inputs"]
    gf, gx = cases.upstream_grads(case)
    if dtype == torch.float32:
        gf, gx = gf.astype(np.float32).astype(np.float64), gx.astype(np.float32).astype(np.float64)
    leaf = torch.as_tensor(np.array(lat, np.float64)).to(dtype).requires_grad_(True)
    with _reference_geometry(kind):
        if case["kind"] == NW:
            g = R.network_grads(case["params"], case["ncfg"], ins["feats"], ins["coors"], gf, gx, ins.get("adj_mat"),
                                ins.get("edges"), ins.get("mask"), leaf, dtype=dtype)
        else:
            f = torch.as_tensor(np.asarray(ins["feats"], np.float64)).to(dtype)
            g = R.layer_grads_chunked(case["params"], case["cfg"], f, ins["coors"], gf, gx, ins.get("edges"),
                                      ins.get("mask"), ins.get("adj_mat"), leaf, nb)
    out = {k: v.detach().double().numpy() for k, v in g.items()}
    out["lattice"] = (leaf.grad if leaf.grad is not None else torch.zeros_like(leaf)).double().numpy()
    return out


@functools.lru_cache(maxsize=None)
def _want(name, dtype):
    """(forward, fp64 gradients) of the restatement on the inputs of `dtype`; computed once per case."""
    case, lat, nb = build(name, dtype)
    kind = kind_of(name)
    return ref_forward(case, lat, kind, nb), ref_grads(case, lat, kind, nb)


def _fp64_gate_fails(out, want):
    for o, w in zip(out, want):
        s = max(1.0, float(np.abs(w).max()))
        if (np.abs(np.asarray(o) - w) > 1e-10 * s + 1e-10 * np.abs(w)).any():
            return True
    return False


def _images(x, cell):
    """Whether the sequential wrap moves each pair by a lattice vector: bool [B, N, N]."""
    B, N, Cd = x.shape
    r = x[:, :, None] - x[:, None]
    moved = np.zeros((B, N, N), bool)
    for c in reversed(range(Cd)):
        Lc = cell[:, c, c]
        per = np.isfinite(Lc) & (Lc > 0)
        n = np.where(per[:, None, None], np.rint(r[..., c] / np.where(per, Lc, 1.0)[:, None, None]), 0.0)
        moved |= n != 0
        r[..., :c + 1] -= n[..., None] * np.where(per[:, None], cell[:, c, :c + 1], 0.0)[:, None, None, :]
    return moved


# ------------------------------------------------------------------ CPU: coverage


def case_geometry(name, rows=None):
    s = CASES[name]
    return dict(LG.simt_layer(s["kind"], s["cfg"], s["B"], s["N"], k=s.get("k", 0), C=s.get("C", 3), rows=rows),
                kind=kind_of(name), lat=s["lat"])


def test_table_covers_every_lattice_boundary():
    """Each boundary of the periodic instantiations, recomputed from the specs, reached under a box and under a cell,
    in each element size (8: fp64, 4: fp32) in which it exists.  Dropping a case or editing a shape so that it no
    longer reaches its boundary fails here."""
    every = {n: case_geometry(n) for n in CASES}
    blocks = {(n, r): case_geometry(n, r) for n in CASES if _rows(n) for r in _rows(n)}
    trained = {8: {n: g for n, g in every.items() if n not in FP64_REJECTED}, 4: every}
    dense = lambda es: [g for n, g in trained[es].items() if g["k"] == 0]
    lists = lambda es: [g for n, g in trained[es].items() if g["k"] > 0]
    want = {
        # forward and backward at MP = 32: pair_kernel, pair_dense_tiled_kernel, bwd1 / bwd3, recompute_pre2
        "dense MP 32": ((8, 4), lambda es: [g for g in dense(es) if g["MP"] == 32]),
        "list MP 32": ((8, 4), lambda es: [g for g in lists(es) if g["MP"] == 32]),
        # the dense forward at one row per thread (fp64 m_dim > 16 trains; q77 in fp64 infers there)
        "dense PP 1": ((8,), lambda es: [g for g in dense(es) if g["PP"][es] == 1]),
        "dense PP 1, shared-memory fallback": ((8,), lambda es: [g for g in every.values() if g["k"] == 0
                                                                 and g["MP"] == 16 and g["PP"][es] == 1]),
        "dense PP 2": ((8, 4), lambda es: [g for g in dense(es) if g["PP"][es] == 2]),
        # the split hidden axis: 32 and 9 hidden CTAs
        "hsplit 32": ((8, 4), lambda es: [g for g in dense(es) if g["hsplit"] == 32]),
        "hsplit 9": ((8, 4), lambda es: [g for g in dense(es) if g["hsplit"] == 9]),
        # hidden chunks, bwd2 channel CTAs, generic node GEMMs with split-K
        "Hp 296, partial chunk": ((8, 4), lambda es: [g for g in dense(es) if g["Hp"] == 296 and g["partial_chunk"]]),
        "bwd2 channel CTAs, partial last": ((8, 4), lambda es: [g for g in dense(es) if g["bwd2_ch_ctas"] >= 2
                                                                and g["partial_ch_cta"]]),
        "generic node GEMMs, partial split-K": ((8, 4), lambda es: [g for g in dense(es) if g["generic_node_gemm"]
                                                                    and g["splitk"] > 1 and g["partial_split"]]),
        "dense j passes >= 3, partial": ((8, 4), lambda es: [g for g in dense(es) if g["j_passes"] >= 3
                                                             and g["partial_j"]]),
        # lists: bwd2 at QR = 0, two full 32-slot passes, TS < 32, two 32-slot bwd2 steps
        "list QR 0": ((8, 4), lambda es: [g for g in lists(es) if g["QR"] == 0 and g["N"] > 32]),
        "list QR 1": ((8, 4), lambda es: [g for g in lists(es) if g["QR"] == 1 and g["N"] > 32]),
        "list QR 8": ((8, 4), lambda es: [g for g in lists(es) if g["QR"] == 8 and g["N"] > 32]),
        "list TS 32, two full slot passes": ((8, 4), lambda es: [g for g in lists(es) if g["TS"] == 32
                                                                 and g["slot_passes"] == 2 and not g["partial_slots"]]),
        "list TS 32, two slot passes, partial": ((8, 4), lambda es: [g for g in lists(es) if g["TS"] == 32
                                                                     and g["slot_passes"] == 2 and g["partial_slots"]]),
        "list TS < 32": ((8, 4), lambda es: [g for g in lists(es) if g["TS"] < 32]),
        "list TS 4, several CTAs, partial last": ((8, 4), lambda es: [g for g in lists(es) if g["TS"] == 4
                                                                      and g["bwd3_ctas"] >= 2 and g["bwd3_partial"]]),
        "list C 2": ((8, 4), lambda es: [g for g in lists(es) if g["C"] == 2]),
        # degree labels in a network
        "4 labels": ((8, 4), lambda es: [g for g in dense(es) if g["labels"] == 4]),
        "16 labels": ((8, 4), lambda es: [g for g in dense(es) if g["labels"] == 16]),
        # the largest fp64 configurations that train, beside the periodic kernels' static shared memory
        "fp64 m 30 trains": ((8,), lambda es: [g for g in dense(es) if g["m"] == 30]),
        "fp64 m 23 soft trains": ((8,), lambda es: [g for n, g in trained[es].items() if g["m"] == 23
                                                     and CASES[n]["cfg"].get("soft_edges")]),
        # bwd3 LAT: a partial last CTA at dense and list shapes; several CTAs per graph
        "LAT dense, partial last CTA": ((8, 4), lambda es: [g for g in dense(es) if g["bwd3_partial"]
                                                            and g["bwd3_ctas"] >= 2]),
        "LAT list, partial last CTA": ((8, 4), lambda es: [g for g in lists(es) if g["bwd3_partial"]
                                                           and g["bwd3_ctas"] >= 2]),
        # row blocks ending inside a dense forward CTA (4 PP rows) and inside a list CTA (128 / TS rows)
        "row block ends inside a dense CTA": ((8,), lambda es: [g for g in blocks.values() if g["k"] == 0
                                                                and g["rows"] % (4 * g["PP"][es]) != 0
                                                                and g["bwd3_partial"]]),
        "row block ends inside a list CTA": ((8,), lambda es: [g for g in blocks.values() if g["k"] > 0
                                                               and g["bwd3_partial"]]),
    }
    missing = []
    for what, (sizes, reach) in want.items():
        for es in sizes:
            kinds = {g["kind"] for g in reach(es)}
            missing += [f"{what} [{'fp64' if es == 8 else 'fp32'}] under a {k}" for k in ("box", "cell") if k not in kinds]
    assert not missing, missing
    # every shape of the non-periodic tables runs under a lattice (the row-block cases run the whole comparisons too)
    shape = lambda s: (repr(sorted(s["cfg"].items())), s["kind"], s["N"], s.get("k", 0))
    have = {shape(s) for s in CASES.values()}
    base = [shape(s) for s in TILE_CASES.values()] + [shape(_edge(n, None)) for n in test_edge_list.BACKWARD_CASES]
    assert not [b for b in base if b not in have], [b for b in base if b not in have]
    # every lattice kind is in the table, and the boxes include the generic C = 5 path
    assert {s["lat"] for s in CASES.values()} == set(BOXES) | set(CELLS)
    assert any(g["C"] == 5 and g["k"] > 0 for g in every.values())
    assert FP64_REJECTED and all(LG.simt_layer(s["kind"], s["cfg"], s["B"], s["N"])["m"]
                             for s in (TILE_CASES[r] for r in FP64_BACKWARD_REJECTED))
    # the q77 shape infers in fp64 at one row per thread
    assert every["q77_tilt"]["PP"][8] == 1 and every["q77_tilt"]["PP"][4] == 2
    # a row range turns the split hidden axis off, so no row-block case uses a split shape
    assert all(every[n]["hsplit"] == 1 for n in CASES if _rows(n))


@pytest.mark.parametrize("name", list(CASES))
def test_inputs_keep_wrap_decisions_off_one_half_and_wrap_a_fifth_of_the_pairs(name):
    for dtype in (torch.float64, torch.float32):
        case, lat, nb = build(name, dtype)
        x = case["inputs"]["coors"]
        B, N, Cd = x.shape
        cell = TRI.cell_bc(lat, B, Cd) if kind_of(name) == "cell" else _diag_cell(np.broadcast_to(lat, (B, Cd)))
        assert TRI.wrap_margin(x, cell).min() >= 1e-3
        moved = _images(np.asarray(x, np.float64), cell)
        if nb is not None:
            bi, ii = np.arange(B)[:, None, None], np.arange(N)[None, :, None]
            moved = moved[bi, ii, np.maximum(nb, 0)][nb >= 0]
        assert moved.mean() >= 0.2, (name, moved.mean())
        if CASES[name]["kind"] == NW:                 # the second layer's inputs are the first layer's outputs
            assert _layer_margin(case, lat, cell, kind_of(name)) > 1e-4


def wrong_lattices(name, lat):
    """[(what, lattice, (module, attribute, replacement) | None)]: mistakes a lattice case must see."""
    kind = kind_of(name)
    lat = np.asarray(lat)
    out = [("no lattice", None, None)]
    if lat.ndim == (2 if kind == "box" else 3):
        out.append(("each graph given the next graph's lattice", np.roll(lat, -1, 0), None))
    if kind == "cell":
        eye = np.eye(lat.shape[-1], dtype=bool)
        out.append(("the cell's diagonal", np.where(eye, lat, 0.0), None))

        def batched(first_to_last=False):
            return lambda rel, cell: torch.stack([T.wrap_cell(rel[b], cell[b].reshape(cell.shape[-2:]), rounding=False,
                                                              first_to_last=first_to_last) for b in range(rel.shape[0])])
        out.append(("axes wrapped first to last", lat, (TRI, "cell_wrap", batched(True))))
        out.append(("floor for rint", lat, (TRI, "cell_wrap", batched())))
    else:
        out.append(("floor for rint", lat, (R, "wrap", lambda rel, box: T.wrap_box(rel, box, rounding=False))))
    return out


@pytest.mark.parametrize("name", list(CASES))
def test_a_wrong_lattice_fails_the_fp64_gate(name, monkeypatch):
    """The float64 restatement under a wrong lattice fails the fp64 forward gate against the right one: a case that
    passed one could not see that mistake in a kernel."""
    case, lat, nb = build(name)
    want = _want(name, torch.float64)[0]
    for what, wrong, patch in wrong_lattices(name, lat):
        with monkeypatch.context() as m:
            if patch:
                m.setattr(*patch)
            if what == "floor for rint":
                m.setattr(T, "_rint", torch.floor)
            if wrong is None:
                got = ref_forward(case, None, "box", nb)
            else:
                got = ref_forward(case, wrong, kind_of(name), nb)
        assert _fp64_gate_fails(got, want), (name, what)


# ------------------------------------------------------------------ the GPU runs


def _lattice_tensor(lat, dtype, requires_grad=False):
    t = torch.as_tensor(np.array(lat, np.float64), dtype=cdt(dtype), device="cuda")
    return t.requires_grad_(True) if requires_grad else t


def run_forward(name, dtype, lattice=None, kind=None, rows=None, mod=None):
    case, lat, nb = build(name, dtype)
    mod = mod or util.make_module(case, dtype)
    kind = kind or kind_of(name)
    ins = case["inputs"]
    t = lambda a: util.to_torch(ins.get(a), dtype, "cuda")
    kw = {kind: _lattice_tensor(lat if lattice is None else lattice, dtype)}
    x = util.to_torch(ins["coors"], cdt(dtype), "cuda")
    with torch.no_grad():
        if case["kind"] == NW:
            return mod(t("feats"), x, adj_mat=t("adj_mat"), edges=t("edges"), mask=t("mask"), **kw)
        if nb is not None:
            kw["neighbors"] = torch.from_numpy(nb).cuda()
        if rows is not None:
            kw["_rows"] = rows
        return mod(t("feats"), x, t("edges"), mask=t("mask"), adj_mat=t("adj_mat"), **kw)


def gpu_grads(name, dtype, lattice=None, kind=None, rows=None, mod=None, lattice_grad=True, built=None):
    """Module gradients with the lattice a leaf -> ({'in.*', 'p.*', ['lattice']} float64 numpy, (fo, xo)).
    `built`: (case, lattice, lists) of build_spec to run instead of the CASES entry `name` (then `kind` is required)."""
    case, lat, nb = built or build(name, dtype)
    mod = (mod or util.make_module(case, dtype)).requires_grad_(True)
    mod.zero_grad(set_to_none=True)
    kind = kind or kind_of(name)
    ins = case["inputs"]
    t = lambda a: util.to_torch(ins.get(a), dtype, "cuda")
    feats, edges = t("feats"), t("edges")
    x = util.to_torch(ins["coors"], cdt(dtype), "cuda").requires_grad_(True)
    leaves = {"in.coors": x}
    if feats.is_floating_point():
        leaves["in.feats"] = feats.requires_grad_(True)
    if edges is not None and edges.is_floating_point():
        leaves["in.edges"] = edges.requires_grad_(True)
    latt = _lattice_tensor(lat if lattice is None else lattice, dtype, requires_grad=lattice_grad)
    kw = {kind: latt, "lattice_grad": lattice_grad}
    gf, gx = (torch.from_numpy(g).to(device="cuda", dtype=dtype) for g in cases.upstream_grads(case))
    with torch.enable_grad():
        if case["kind"] == NW:
            fo, xo = mod(feats, x, adj_mat=t("adj_mat"), edges=edges, mask=t("mask"), **kw)
        else:
            if nb is not None:
                kw["neighbors"] = torch.from_numpy(nb).cuda()
            if rows is not None:
                kw["_rows"] = rows
            fo, xo = mod(feats, x, edges, mask=t("mask"), adj_mat=t("adj_mat"), **kw)
        if rows is not None:
            fo, xo, gf, gx = (v[:, rows[0]:rows[1]] for v in (fo, xo, gf, gx))
        ((fo * gf).sum() + (xo * gx.to(xo.dtype)).sum()).backward()
    got = {k: v.grad.double().cpu().numpy() for k, v in leaves.items()}
    got.update({f"p.{k}": (torch.zeros_like(p) if p.grad is None else p.grad).double().cpu().numpy()
                for k, p in mod.named_parameters()})
    if lattice_grad:
        assert latt.grad is not None and latt.grad.shape == latt.shape and latt.grad.dtype == latt.dtype
        got["lattice"] = latt.grad.double().cpu().numpy()
    return got, (fo.detach(), xo.detach())


DT = {"fp64": torch.float64, "fp32": torch.float32}


def report(gate, what, got, want):
    """Print the largest error over the largest magnitude of the reference (at least 1) under `gate`; the module
    docstring quotes the worst of these."""
    pairs = [(got[k], want[k]) for k in want] if isinstance(want, dict) else list(zip(got, want))
    err = max(float(np.abs(np.asarray(g, np.float64) - np.asarray(w, np.float64)).max()) /
              max(1.0, float(np.abs(np.asarray(w, np.float64)).max())) for g, w in pairs)
    print(f"GATE {gate} {what} {err:.3e}")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name", list(CASES))
def test_forward_matches_the_restatement(name, dt):
    dtype = DT[dt]
    case, _, _ = build(name, dtype)
    out = run_forward(name, dtype)
    want = _want(name, dtype)[0]
    report(f"forward-{dt}", name, [o.double().cpu().numpy() for o in out], want)
    TRI._check(case, out, want, dtype, f"{name} [{dt}]")


def _assert_exact_zeros(name, g, lat):
    """The lattice gradient is 0 above the diagonal and on every aperiodic axis (its row, for a cell)."""
    lat = np.asarray(lat, np.float64)
    aper = ~(np.isfinite(lat) & (lat > 0)) if kind_of(name) == "box" else \
        ~(np.isfinite(np.diagonal(lat, axis1=-2, axis2=-1)) & (np.diagonal(lat, axis1=-2, axis2=-1) > 0))
    if kind_of(name) == "box":
        assert np.array_equal(g[aper], np.zeros(int(aper.sum()))), name
    else:
        C = g.shape[-1]
        assert np.array_equal(np.triu(g, 1), np.zeros_like(g)), name
        rows = np.broadcast_to(aper, g.shape[:-1])
        assert np.array_equal(g[rows], np.zeros((int(rows.sum()), C))), name


GRAD = [(n, dt) for n in CASES for dt in ("fp64", "fp32") if not (dt == "fp64" and n in FP64_REJECTED)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["saved", "recomputed"])
@pytest.mark.parametrize("name,dt", GRAD, ids=[f"{n}-{d}" for n, d in GRAD])
def test_gradients_and_lattice_gradient_match_the_restatement(name, dt, mode, monkeypatch):
    """recomputed: the backward recomputes W2 silu(pre1) with the forward's edge kernels (EGNN_B200_SAVE_PAIR_MB=0)."""
    if mode == "recomputed":
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")
    dtype = DT[dt]
    case, lat, nb = build(name, dtype)
    got, _ = gpu_grads(name, dtype)
    want = _want(name, dtype)[1]
    what = f"{name} [{dt}] {mode}"
    glat = got.pop("lattice")
    report(f"grads-{dt}", what, got, {k: v for k, v in want.items() if k != "lattice"})
    util.compare(got, {k: v for k, v in want.items() if k != "lattice"}, util.grad_tol(case, dtype), what)
    assert np.abs(want["lattice"]).max() > 1e-3
    if dtype == torch.float64:
        check64(glat, want["lattice"], what)
    else:
        ref32 = ref_grads(case, lat, kind_of(name), nb, dtype=torch.float32)["lattice"]
        check32(glat, ref32, want["lattice"], what)
    _assert_exact_zeros(name, glat, lat)


DIAG = [(n, dt) for n in CASES if kind_of(n) == "box" and CASES[n].get("C", 3) in (2, 3) for dt in ("fp64", "fp32")]


@pytest.mark.gpu
@pytest.mark.parametrize("name,dt", DIAG, ids=[f"{n}-{d}" for n, d in DIAG])
def test_a_diagonal_cell_is_the_box(name, dt):
    """Forward bit for bit; the cell's lattice-gradient diagonal is the box gradient to the rounding of the fp64
    atomics (the wrap subtracts exact zeros off the diagonal), and its upper triangle is exactly 0."""
    dtype = DT[dt]
    case, L, _ = build(name, dtype)
    B, Cd = case["inputs"]["coors"].shape[0], case["inputs"]["coors"].shape[-1]
    cell = _diag_cell(L)
    mod = util.make_module(case, dtype)
    ref = run_forward(name, dtype, mod=mod)
    out = run_forward(name, dtype, lattice=cell, kind="cell", mod=mod)
    assert torch.equal(out[0], ref[0]) and torch.equal(out[1], ref[1])
    if dt == "fp64" and name in FP64_REJECTED:
        return
    gb = gpu_grads(name, dtype)[0]["lattice"]
    gc = gpu_grads(name, dtype, lattice=cell, kind="cell")[0]["lattice"]
    tol = 1e-13 if dtype == torch.float64 else 1e-6
    err = float(np.abs(np.diagonal(gc, axis1=-2, axis2=-1) - gb).max() / np.abs(gb).max())
    print(f"GATE diagonal-{dt} {name} {err:.3e}")
    assert err <= tol, name
    upper = np.triu(np.ones((Cd, Cd), bool), 1)
    assert np.array_equal(gc[..., upper], np.zeros_like(gc[..., upper]))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["box", "cell"])
@pytest.mark.parametrize("name", sorted(FP64_BACKWARD_REJECTED))
def test_fp64_backward_over_the_shared_memory_budget_fails_at_the_training_forward(name, kind, monkeypatch):
    """Under a lattice, with and without lattice_grad=True, the fp64 training forward raises before it launches."""
    built = build_spec(_tile(name, {"box": "cubic", "cell": "tilt"}[kind]), torch.float64)
    for lg in (True, False):
        _assert_training_forward_rejected(None, torch.float64, monkeypatch,
                                          run=lambda: gpu_grads(None, torch.float64, kind=kind, built=built,
                                                                lattice_grad=lg))


ROWS = [n for n in CASES if _rows(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ROWS)
def test_row_blocks_partition_forward_and_gradients(name):
    """fp64: each block's rows of the forward equal the whole forward bit for bit; the gradients of the blocks, the
    lattice gradient included, sum to the whole gradient."""
    dtype = torch.float64
    case, _, _ = build(name, dtype)
    mod = util.make_module(case, dtype)
    whole, (fo, xo) = gpu_grads(name, dtype, mod=mod)
    parts = []
    for r0, r1 in _rows(name):
        g, (fb, xb) = gpu_grads(name, dtype, rows=(r0, r1), mod=mod)
        assert torch.equal(fb, fo[:, r0:r1]) and torch.equal(xb, xo[:, r0:r1]), (name, r0, r1)
        parts.append(g)
    for k, w in whole.items():
        s = sum(p[k] for p in parts)
        tol = 1e-13 if k == "lattice" else 1e-10
        report("rows-lattice" if k == "lattice" else "rows-grads", f"{name} {k}", [s], [w])
        assert np.abs(s - w).max() <= tol * max(1.0, np.abs(w).max()), (name, k)


# ------------------------------------------------------------------ the kernels the cases launch

_TPL = re.compile(r"egnn::(\w+)<([^>]*)>")


def _launched(fn):
    """Run fn under torch.profiler (CUDA activity only) -> [(kernel, [template arguments], grid)]."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    out = []
    for e in events:
        if e.get("cat") != "kernel":
            continue
        m = _TPL.search(e["name"])
        if m:
            out.append((m.group(1), [a.strip() for a in m.group(2).split(",")], tuple(e.get("args", {}).get("grid", ()))))
    return out


PROFILED = ["mdim30_tilt", "mdim20_soft_cubic", "q77_tilt", "hsplit512_tilt", "hsplit128_box_pg", "list_k64_q1_tilt",
            "list_k33_mdim24_aperiodic", "rows_dense_cubic"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", PROFILED)
def test_cases_launch_what_the_table_claims(name):
    """The demangled names of the launched kernels agree with launch_geometry.simt_layer: PBC, MP, PP, BLK and LAT, the
    phase-1 grid of the split hidden axis, and bwd3's grid."""
    g = case_geometry(name)
    pbc = "1" if g["kind"] == "box" else "2"
    for dt in ("fp64", "fp32"):
        dtype = DT[dt]
        es = 8 if dtype == torch.float64 else 4
        T_ = "double" if es == 8 else "float"
        rows = (_rows(name) or [None])[0]
        gr = case_geometry(name, rows) if rows else g
        blk = "true" if rows else "false"
        fwd = _launched(lambda: run_forward(name, dtype, rows=rows))
        if g["k"] == 0:
            tiled = [(a, grid) for n, a, grid in fwd if n == "pair_dense_tiled_kernel"]
            # (inference runs a row range in the whole-graph instantiation, over that range's CTAs)
            assert tiled and all(a == [T_, str(g["MP"]), str(g["PP"][es]), "false", pbc] for a, _ in tiled), (name, dt, tiled)
            assert tiled[-1][1][0] == math.ceil(gr["rows"] / (4 * g["PP"][es])), (name, dt, tiled)
            if g["hsplit"] > 1:
                assert [grid[2] for _, grid in tiled] == [g["hsplit"], 1], (name, dt, tiled)
        else:
            pk = [a for n, a, _ in fwd if n == "pair_kernel"]
            assert pk and all(a == [T_, str(g["MP"]), "false", pbc] for a in pk), (name, dt, pk)
        if dt == "fp64" and name in FP64_REJECTED:
            continue
        bwd = _launched(lambda: gpu_grads(name, dtype, rows=rows))
        b3 = [(a, grid) for n, a, grid in bwd if n == "pair_bwd3_kernel"]
        assert [a for a, _ in b3] == [[T_, "true" if g["k"] else "false", blk, pbc, "true"]], (name, dt, b3)
        assert b3[0][1][:2] == (gr["bwd3_ctas"], CASES[name]["B"]), (name, dt, b3)
        b1 = [a for n, a, _ in bwd if n == "pair_bwd1_kernel"]
        assert b1 and all(a[1] == str(g["MP"]) and a[-1] == pbc for a in b1), (name, dt, b1)


# ------------------------------------------------------------------ the all-pairs select under a cell (and fp64 boxes)
#
# knn_select.cu ranks a pair under a cell in the coordinates' type T as cell_staged / cell_wrap_n do: r_c = fl(x_i - x_j);
# from the last axis to the first, n = rint(fl(r_c fl(1 / L_c))) and r_d = fma(-a_cd, n, r_d) for d <= c; then
# d = fl(d + fl(r_c r_c)) over the axes in order (sq_acc).  An fp32 fma is the float64 sum rounded once
# (tc_reference._fma: a n has at most 29 significant bits, so the float64 sum is exact for the pairs here).  fp64 inputs
# lie on a dyadic grid (multiples of 2^-8 below 2^5), where n a and r - n a are exact, so the unfused float64 expression
# is the fma.  test_cell_ranks_are_pinned_to_exact_arithmetic checks both against fractions.Fraction.

SEL_GRID = 2.0 ** -8


def cell_ranks(x, rows, cell, mask=None):
    """Ranks [B, R, N] of rows `rows` under lower-triangular cells [B, C, C] (C = 2 or 3), in x's type (fp32 / fp64)."""
    Tt = x.dtype.type
    B, N, Cd = x.shape
    A = np.asarray(cell, Tt)
    rows = np.asarray(rows)
    diag = np.diagonal(A, axis1=1, axis2=2)
    per = (diag > 0) & np.isfinite(diag)
    L = np.where(per, diag, Tt(0)).astype(Tt)
    inv = np.where(per, Tt(1) / np.where(per, diag, Tt(1)), Tt(0)).astype(Tt)
    off = np.where(np.isfinite(A), A, Tt(0)).astype(Tt)
    r = [(x[:, rows, c][:, :, None] - x[:, None, :, c]).astype(Tt) for c in range(Cd)]
    fma = (lambda a, b, c: (a.astype(np.float64) * b + c).astype(np.float32)) if Tt is np.float32 else \
        (lambda a, b, c: a * b + c)
    for c in reversed(range(Cd)):
        n = np.rint(r[c] * inv[:, c, None, None]).astype(Tt)
        for d in range(c + 1):
            coef = L[:, c] if d == c else off[:, c, d]
            r[d] = fma(-coef[:, None, None], n, r[d]).astype(Tt)
    dd = np.zeros_like(r[0])
    for c in range(Cd):
        dd = (dd + (r[c] * r[c]).astype(Tt)).astype(Tt)
    if mask is not None:
        mask = np.asarray(mask, bool)
        dd = np.where(mask[:, rows, None] & mask[:, None, :], dd, Tt(1e5))
    return dd


def cell_select(x, k, vr, cell, mask=None, chunk=256):
    """-> (idx, ok) of the all-pairs select under a cell: stable argsort of cell_ranks, ok = rank <= T(vr)."""
    Tt = x.dtype.type
    idx, ok = [], []
    for s in range(0, x.shape[1], chunk):
        d = cell_ranks(x, np.arange(s, min(x.shape[1], s + chunk)), cell, mask)
        o = np.argsort(d, axis=-1, kind="stable")[..., :k]
        idx.append(o)
        ok.append(np.take_along_axis(d, o, axis=-1) <= Tt(vr))
    return np.concatenate(idx, 1), np.concatenate(ok, 1)


# name: (B, N, C, k, lattice kind, mask + valid_radius); C = 3 cells run the CDIM = 3 warp select, C = 2 the generic one
SELECT = {
    "sel_warp8_1pass":    (2, 300, 3, 16, "tilt", False),
    "sel_warp8_3pass":    (1, 2200, 3, 32, "per_graph", False),
    "sel_warp16_1pass":   (5, 1000, 3, 8, "tilt09", False),
    "sel_warp16_3pass":   (2, 2200, 3, 31, "per_graph", False),
    "sel_generic_c2":     (2, 500, 2, 8, "c2", False),
    "sel_sort_k40_n256":  (2, 256, 3, 40, "tilt", False),
    "sel_sort_k64_n257":  (1, 257, 3, 64, "hex_slab", False),
    "sel_warp_mask_r":    (2, 700, 3, 16, "tilt09", True),
    "sel_sort_mask_r":    (2, 200, 3, 33, "per_graph", True),
    # fp64 boxes (the box select is checked in fp32 by test_gpu_knn_select.py)
    "sel_box_warp16_3pass": (2, 2200, 3, 32, "box_per_graph", False),
    "sel_box_generic_c5": (2, 600, 5, 8, "box_c5", False),
    "sel_box_sort_k40":   (2, 256, 3, 40, "box_aperiodic", False),
    "sel_box_mask_r":     (2, 700, 3, 16, "cubic", True),
}
SELECT_DTYPES = {n: (("fp64",) if SELECT[n][4] in BOXES else ("fp64", "fp32")) for n in SELECT}


def select_inputs(name, dt):
    """(x [B, N, C], cell [B, C, C], lattice as the layer takes it, mask or None, valid_radius).  fp64: cell and
    coordinates on the dyadic grid; fp32: rounded to fp32."""
    B, N, Cd, k, kind, masked = SELECT[name]
    rs = np.random.RandomState(sum(map(ord, name)))
    lat, cell = make_lattice(kind, B, Cd, rs)
    snap = (lambda a: np.where(np.isfinite(a), np.round(a / SEL_GRID) * SEL_GRID, a)) if dt == "fp64" else \
        (lambda a: a.astype(np.float32).astype(np.float64))
    lat, cell = snap(np.asarray(lat, np.float64)), snap(cell)
    per = np.isfinite(np.diagonal(cell, axis1=1, axis2=2)) & (np.diagonal(cell, axis1=1, axis2=2) > 0)
    Af = np.where(np.isfinite(cell), cell, 0.0) + np.where(per, 0.0, 1.0)[:, :, None] * np.eye(Cd)
    s = rs.uniform(0, 1, (B, N, Cd)) * np.where(per, 1.0, 3.0)[:, None, :] + rs.randint(-2, 3, (B, N, Cd)) * per[:, None]
    x = snap(np.einsum("bnk,bkd->bnd", s, Af))
    assert np.abs(x).max() < 2 ** 5
    mask = rs.uniform(size=(B, N)) < 0.85 if masked else None
    Tt = np.float64 if dt == "fp64" else np.float32
    return x.astype(Tt), cell.astype(Tt), lat, mask, (4.0 if masked else math.inf)


def _exact_rank(xi, xj, A, Tt):
    """The rank of one pair by the same steps, each an exact Fraction rounded once to Tt."""
    from fractions import Fraction as Fr

    def rnd(q):                                    # round a Fraction to the nearest Tt, ties to even
        g = Tt(float(q))
        cands = [g, np.nextafter(g, Tt(np.inf)), np.nextafter(g, Tt(-np.inf))]
        return min(cands, key=lambda c: (abs(Fr(float(c)) - q), int(np.frexp(c)[0] * 2 ** 24) & 1 if Tt is np.float32
                                           else int(np.frexp(c)[0] * 2 ** 53) & 1))
    Cd = len(xi)
    r = [rnd(Fr(float(xi[c])) - Fr(float(xj[c]))) for c in range(Cd)]
    for c in reversed(range(Cd)):
        Lc = A[c][c]
        if not (Lc > 0 and np.isfinite(Lc)):
            continue
        inv = rnd(1 / Fr(float(Lc)))
        n = np.rint(rnd(Fr(float(r[c])) * Fr(float(inv))))
        for d in range(c + 1):
            r[d] = rnd(Fr(float(r[d])) - Fr(float(A[c][d])) * Fr(float(n)))
    acc = Tt(0)
    for c in range(Cd):
        acc = rnd(Fr(float(acc)) + Fr(float(rnd(Fr(float(r[c])) ** 2))))
    return acc


@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name", ["sel_warp8_1pass", "sel_generic_c2", "sel_sort_k64_n257"])
def test_cell_ranks_are_pinned_to_exact_arithmetic(name, dt):
    """A sample of pairs: cell_ranks (numpy, fp32 fma as one rounding of the float64 sum; fp64 unfused on the dyadic
    grid) equals the same steps carried out exactly in fractions and rounded once each."""
    x, cell, _, _, _ = select_inputs(name, dt)
    Tt = x.dtype.type
    rs = np.random.RandomState(3)
    B, N, _ = x.shape
    for _ in range(150):
        b, i, j = rs.randint(B), rs.randint(N), rs.randint(N)
        got = cell_ranks(x[b:b + 1], [i], cell[b:b + 1])[0, 0, j]
        want = _exact_rank(x[b, i], x[b, j], cell[b], Tt)
        assert got == want, (name, dt, b, i, j, got, want)


@pytest.mark.parametrize("name", list(SELECT))
def test_select_cases_wrap_and_reach_their_boundaries(name):
    """At least a fifth of each graph's selected pairs wrap; the launch geometry is the one the row names."""
    B, N, Cd, k, kind, masked = SELECT[name]
    for dt in SELECT_DTYPES[name]:
        x, cell, _, mask, vr = select_inputs(name, dt)
        idx, ok = cell_select(x, k, vr, cell, mask)
        moved = _images(x.astype(np.float64), cell.astype(np.float64))
        sel = np.take_along_axis(moved, idx, -1)
        assert sel.mean() >= 0.2, (name, dt, sel.mean())
        g = LG.launch_select(B, N, Cd, k, 8 if dt == "fp64" else 4)
        if k <= 32:
            assert g["kernel"] == "warp" and (g["cdim"] == 3) == (Cd == 3)
        else:
            assert g["kernel"] == "sort" and g["supported"]


def test_select_table_covers_the_schedule_boundaries():
    """Each schedule boundary of launch_select under a cell in fp32 and fp64, and under a box in fp64."""
    got = set()
    for name, (B, N, Cd, k, kind, masked) in SELECT.items():
        lk = "box" if kind in BOXES else "cell"
        for dt in SELECT_DTYPES[name]:
            g = LG.launch_select(B, N, Cd, k, 8 if dt == "fp64" else 4)
            m = " masked" if masked else ""
            if g["kernel"] == "warp":
                tags = [f"warp{g['warps']} passes{g['passes']} {'cdim3' if g['cdim'] == 3 else 'generic'}{m}"]
            else:
                tags = [f"sort k{k} npad{g['npad']}{m}"]
            got |= {(t, lk, dt) for t in tags}
    need = ["warp8 passes1 cdim3", "warp8 passes3 cdim3", "warp16 passes1 cdim3", "warp16 passes3 cdim3",
            "warp8 passes1 generic", "sort k40 npad256", "sort k64 npad512", "warp8 passes1 cdim3 masked",
            "sort k33 npad256 masked"]
    missing = [(t, "cell", dt) for t in need for dt in ("fp64", "fp32") if (t, "cell", dt) not in got]
    missing += [(t, "box", "fp64") for t in ("warp16 passes3 cdim3", "warp8 passes1 generic", "sort k40 npad256",
                                             "warp8 passes1 cdim3 masked")
                if (t, "box", "fp64") not in got]
    assert not missing, missing


SELECT_RUNS = [(n, dt) for n in SELECT for dt in SELECT_DTYPES[n]]


@pytest.mark.gpu
@pytest.mark.parametrize("name,dt", SELECT_RUNS, ids=[f"{n}-{d}" for n, d in SELECT_RUNS])
def test_select_under_a_lattice_through_the_layer(name, dt, monkeypatch):
    """The layer's own all-pairs select (cell grid forced off) equals the reference lists: the same layer run with
    `neighbors=` set to them (ok = 0 slots as -1) gives bit-identical outputs."""
    from egnn_pytorch_b200 import EGNN
    B, N, Cd, k, kind, masked = SELECT[name]
    dtype = DT[dt]
    x, cell, lat, mask, vr = select_inputs(name, dt)
    idx, ok = cell_select(x, k, vr, cell, mask)
    monkeypatch.setenv("EGNN_B200_CELL_SELECT_MIN_N", str(2 ** 40))
    torch.manual_seed(1)
    layer = EGNN(dim=8, num_nearest_neighbors=k, valid_radius=vr).to(dtype).cuda().eval()
    f = torch.randn(B, N, 8, device="cuda", dtype=dtype)
    tx = torch.from_numpy(x).cuda()
    lk = "box" if kind in BOXES else "cell"
    tl = torch.as_tensor(np.asarray(lat, np.float64), dtype=dtype, device="cuda")
    tm = None if mask is None else torch.from_numpy(mask).cuda()
    nbr = torch.from_numpy(np.where(ok, idx, -1)).cuda()
    with torch.no_grad():
        f1, x1 = layer(f, tx, mask=tm, **{lk: tl})
        f2, x2 = layer(f, tx, mask=tm, neighbors=nbr, **{lk: tl})
    assert torch.equal(f1, f2) and torch.equal(x1, x2), \
        f"{name} [{dt}]: outputs differ in {int(((f1 != f2).any(-1) | (x1 != x2).any(-1)).sum())} rows"
