"""Tile and schedule boundaries of the bf16 tensor-core layer, against a rounding-matched reference.

The fp64 oracle gate of test_gpu_fast.py (1e-2 of the output scale) has to allow for every bf16 rounding of the
kernels, so it cannot see errors of that size in the edge kernels.  tests/tc_reference.py rounds where the kernels
round; what is left between it and a correct kernel is tanh.approx, fp32 arithmetic and bf16 rounding-boundary flips,
so the gates below can be two orders of magnitude tighter on the coordinate output.

The case table crosses the boundaries of the launch code (fast_path.cu, tc_pair.cuh, tc_knn.cuh, small_node.cuh),
mirrored in `geometry` and held there by test_table_covers_every_boundary:
  tc_pair   j-split 1 / 2 / 4 / 8 (full graphs and row ranges); one active warpgroup (N <= 128); partial, full and
            empty warp and warpgroup tiles (N = 63..65 / 127..129 / 191..193 / 255..257); the widest lean layer
            (Hp = 2736); 1..3 valid rows in the last row group, at graph
            ends and at row-range ends; ring reuse (more than 2 items per CTA, odd laps); last hidden chunk of 1..4 K
            slabs; batches (the last graph reads B' into the table's pad rows); the generic instantiation at its
            limits (Q = 12 per-pair channels, C = 8) with fourier features, edges and degree labels through EGNN_Network;
            padded, random and fully masked graphs; mean pooling, clamp, soft edges, CoorsNorm
  tc_knn    k = 1 / 8 / 31 / 32; the lean, edges and generic instantiations at 8 and 16 rows per CTA, each with a
            partial last CTA; caller lists with -1 slots (mean without a mask too); per-slot edges; row ranges
  node path small-node kernels (dim <= 64, B*N <= 4096), tc_gemm tables at dim <= 64 with B*N > 4096, dim > 64
  lattices  the PBC_BOX and PBC_CELL instantiations of both kernels (cases "pb_" / "pc_" / "kb_" / "kc_"): the tc_pair
            and tc_knn boundaries above under a box and under a cell (k = 1 under a cell); ring slots refilled with
            a row group of another graph whose lattice differs (j-split 1 and 2, odd laps), the only route through
            the per-slot lattice staging; generic C = 5 / 8 boxes with aperiodic axes; 2-D, hexagonal-slab and 0.9-tilt cells;
            the c2 shape with a box and a cell, and c4 (B=8, N=4096, k=32, per-slot edges) with a box per graph
The lattice cases place nodes so that most compared pairs wrap (>= 20 %) and every wrap decision lies >= 1e-3 from
1/2, so the reference's fp32 wrap and the fp64 restatement pick the kernels' images; the CPU tests pin that fp32 wrap
to an exact rational evaluation and, unrounded, to torch_reference / test_triclinic's float64 restatements, and check
that each lattice case fails a gate when the reference is given a wrong lattice (none, the next graph's, a cell's
diagonal, the axes wrapped first to last, floor for rint).  A diagonal cell gives the box's outputs bit for bit.
Every case uses xavier weights, so that the coordinate update is O(1) and the messages move the features
(test_every_case_sees_the_edge_kernel checks that on the reference).

Gates against the rounding-matched reference, per case (measured: the worst value over the table on an H100 80GB HBM3;
each tolerance is 2.6x - 4x that, `TOL`):
  feats   max and mean |error| in bf16 ulps of the reference value (ulps below 1 % of the tensor's scale are
          counted at that floor)
  coors   per row: max |error| over the row / that row's update; over all rows: RMS error / RMS update
plus the gate of test_gpu_fast.py against the fp64 oracle (under a lattice: the float64 periodic restatement).  Large
cases compare row windows (`check`) that include the first and last rows of every graph and of the range."""
import contextlib
import functools
from fractions import Fraction

import numpy as np
import pytest
import torch

import cases
import launch_geometry as LG
import tc_reference as T
import test_periodic as PER
import test_triclinic as TRI
import torch_reference as R
import util
from oracle import egnn_oracle as O

L, NW = "layer", "network"

# Worst value over the table, measured on an H100 80GB HBM3 (700 W power limit), and the tolerance: 2.6x - 4x that.
#   f_ulp_max   33      (k8_edges8_slot: values near the 1 % floor)      -> 132
#   f_ulp_mean  0.078   (p_d680)                                          -> 0.26
#   c_row       3.1e-3  (p_n192_mean)                                     -> 8e-3
#   c_rms       9.1e-5  (k8_gemm_tables)                                  -> 3.6e-4
# For scale: packing the hidden values with round-toward-zero instead of round-to-nearest gives f_ulp_mean 0.1 - 1.6,
# c_row 1e-3 - 0.28 and c_rms 3e-4 - 7e-3 over the same table.
TOL = dict(f_ulp_max=132.0, f_ulp_mean=0.26, c_row=8e-3, c_rms=3.6e-4)

CASES = {
    # ---------------- dense all-pairs (tc_pair_kernel)
    # j-split 1, 7 items on the first CTAs (ring slots reused, odd laps), padded graphs
    "p_js1_ring":      dict(kind=L, cfg=dict(dim=16), B=5, N=700, seed=401, mask="padded",
                            check=[(0, 8), (344, 352), (690, 700)]),
    # j-split 2, 1 valid row in the last row group, 3-slab tail chunk, random mask
    "p_js2_n701":      dict(kind=L, cfg=dict(dim=24, soft_edges=True), B=2, N=701, seed=402, mask="random",
                            check=[(0, 8), (400, 404), (693, 701)]),
    # j-split 4 over a whole graph; generic instantiation (fourier + edges, Q = 9), 2-slab tail chunk
    "p_js4_full":      dict(kind=L, cfg=dict(dim=16, fourier_features=2, edge_dim=4), B=1, N=1100, seed=403,
                            check=[(0, 8), (548, 556), (1092, 1100)]),
    # j-split 4 on a row range ending with 3 valid rows; 4-slab last chunk (Hp = 128); two graphs
    "p_js4_range":     dict(kind=L, cfg=dict(dim=24, fourier_features=2, edge_dim=4, norm_coors=True), B=2, N=1024,
                            seed=404, rows=(0, 63), mask="padded"),
    # j-split 8 on a row range ending with 1 valid row
    "p_js8_range":     dict(kind=L, cfg=dict(dim=16, coor_weights_clamp_value=2.0), B=1, N=2048, seed=405, rows=(5, 34)),
    # one active warpgroup; mean over a mask with one fully masked graph
    "p_n100_empty":    dict(kind=L, cfg=dict(dim=64, m_pool_method="mean"), B=3, N=100, seed=406, mask="one_empty"),
    # warpgroup tiles: partial (127, 255), exactly full (128, 256), one pair in the second tile (129) / the next block (257)
    "p_n127_clamp":    dict(kind=L, cfg=dict(dim=32, coor_weights_clamp_value=0.3), B=2, N=127, seed=407),
    "p_n128_soft":     dict(kind=L, cfg=dict(dim=32, soft_edges=True), B=2, N=128, seed=408, mask="random"),
    "p_n129_norm":     dict(kind=L, cfg=dict(dim=32, norm_coors=True), B=2, N=129, seed=409),
    "p_n255_mean":     dict(kind=L, cfg=dict(dim=40, m_pool_method="mean"), B=2, N=255, seed=410),
    "p_n256":          dict(kind=L, cfg=dict(dim=48), B=2, N=256, seed=411, mask="padded"),
    "p_n257_rows":     dict(kind=L, cfg=dict(dim=32, edge_dim=2), B=3, N=257, seed=412, rows=(97, 257)),
    # warp tiles (32 pairs): partial / exactly full / one pair into the next warp at the end of 2, 4, 6 and 8 warps
    "p_n63_clamp":     dict(kind=L, cfg=dict(dim=32, coor_weights_clamp_value=0.5), B=2, N=63, seed=501, mask="random"),
    "p_n64_mean":      dict(kind=L, cfg=dict(dim=32, m_pool_method="mean"), B=2, N=64, seed=502, mask="padded"),
    "p_n65_soft":      dict(kind=L, cfg=dict(dim=24, soft_edges=True), B=2, N=65, seed=503),
    "p_n127_mean":     dict(kind=L, cfg=dict(dim=16, m_pool_method="mean", soft_edges=True), B=2, N=127, seed=504,
                            mask="random"),
    "p_n128":          dict(kind=L, cfg=dict(dim=32), B=2, N=128, seed=505, mask="padded"),
    "p_n129_clamp":    dict(kind=L, cfg=dict(dim=24, coor_weights_clamp_value=1.0), B=2, N=129, seed=506),
    "p_n191_soft":     dict(kind=L, cfg=dict(dim=16, soft_edges=True), B=2, N=191, seed=507, mask="padded"),
    "p_n192_mean":     dict(kind=L, cfg=dict(dim=32, m_pool_method="mean"), B=2, N=192, seed=508),
    "p_n193":          dict(kind=L, cfg=dict(dim=16), B=2, N=193, seed=509, mask="random"),
    "p_n255_clamp":    dict(kind=L, cfg=dict(dim=16, coor_weights_clamp_value=2.0, soft_edges=True), B=2, N=255,
                            seed=510),
    "p_n256_mean":     dict(kind=L, cfg=dict(dim=24, m_pool_method="mean"), B=2, N=256, seed=511, mask="padded"),
    "p_n257":          dict(kind=L, cfg=dict(dim=16), B=2, N=257, seed=512, mask="random"),
    # ... and the generic instantiation (fourier features + edges, edges + mean + clamp) with one and two warpgroups
    "p_gen_n60":       dict(kind=L, cfg=dict(dim=16, fourier_features=1, edge_dim=2, soft_edges=True), B=2, N=60,
                            seed=513, mask="padded"),
    "p_gen_n150":      dict(kind=L, cfg=dict(dim=16, edge_dim=3, m_pool_method="mean", coor_weights_clamp_value=1.0),
                            B=2, N=150, seed=514, mask="random"),
    # the widest lean layer: Hp = 2736, close to the shared-memory limit
    "p_d680":          dict(kind=L, cfg=dict(dim=680), B=1, N=70, seed=521, mask="padded"),
    # GEMM node path and GEMM tables (dim > 64), 2 valid rows in the last row group
    "p_d72_n258":      dict(kind=L, cfg=dict(dim=72, norm_feats=True, m_pool_method="mean"), B=2, N=258, seed=413,
                            mask="padded"),
    # GEMM tables at dim <= 64 (B*N > 4096) with the small node kernels
    "p_gemm_tables":   dict(kind=L, cfg=dict(dim=32), B=3, N=1400, seed=414, check=[(0, 4), (700, 704), (1396, 1400)]),
    # generic instantiation at its limits: C = 8, and Q = 12 (d, 2 x 2 fourier, 3 edges, 4 degree labels)
    "p_c8_mean_clamp": dict(kind=L, cfg=dict(dim=32, fourier_features=3, m_pool_method="mean",
                                             coor_weights_clamp_value=1.0), B=2, N=90, C=8, seed=415, mask="random"),
    "p_net_q12_c8":    dict(kind=NW, cfg=dict(depth=1, dim=16, fourier_features=2, edge_dim=3, num_adj_degrees=3,
                                              adj_dim=2, soft_edges=True), B=2, N=150, C=8, seed=416, adj="chain",
                            edges=True, mask="padded"),
    # ---------------- neighbour lists (tc_knn_kernel), caller-supplied lists
    "k1_lean8":        dict(kind=L, cfg=dict(dim=32), B=2, N=203, k=1, seed=420),
    "k8_edges8_slot":  dict(kind=L, cfg=dict(dim=64, edge_dim=4), B=2, N=150, k=8, seed=421, holes=True,
                            slot_edges=True, mask="padded"),
    "k31_gen8_mean":   dict(kind=L, cfg=dict(dim=32, fourier_features=2, m_pool_method="mean"), B=2, N=100, k=31,
                            seed=422, holes=True),
    "k8_gen8_c5":      dict(kind=L, cfg=dict(dim=32, edge_dim=2, soft_edges=True, norm_coors=True), B=2, N=77, C=5,
                            k=8, seed=423, mask="random"),
    "k32_lean16":      dict(kind=L, cfg=dict(dim=344, coor_weights_clamp_value=3.0), B=1, N=150, k=32, seed=424,
                            holes=True),
    "k32_edges16":     dict(kind=L, cfg=dict(dim=280, edge_dim=4), B=1, N=100, k=32, seed=425, holes=True,
                            mask="random"),
    "k31_gen16_rows":  dict(kind=L, cfg=dict(dim=264, fourier_features=2, edge_dim=1, m_pool_method="mean"), B=2, N=150,
                            k=31, seed=426, holes=True, slot_edges=True, mask="padded", rows=(19, 140)),
    "k32_d128_rows":   dict(kind=L, cfg=dict(dim=128, soft_edges=True), B=2, N=120, k=32, seed=427, rows=(3, 117)),
    "k8_gemm_tables":  dict(kind=L, cfg=dict(dim=32, m_pool_method="mean"), B=1, N=5000, k=8, seed=428, holes=True,
                            check=[(0, 16), (2500, 2516), (4990, 5000)]),
}

# ---------------- periodic boxes (`box`, key "pb_" / "kb_") and triclinic cells (`cell`, key "pc_" / "kc_")
# box: [C] lengths (0 / inf: aperiodic) or "per_graph" (one box per graph); cell: a kind of `lattice_inputs`.  Every
# lattice is smaller than the coordinate spread (nodes are moved by whole lattice vectors), so most pairs wrap.
BOX3, INF = [3.0, 3.25, 3.5], float("inf")
LATTICE_SHAPES = [
    # (name, spec, box, cell)
    # ring reuse with odd laps, where a CTA's consecutive items lie in graphs with different lattices: j-split 1
    # (875 items) and j-split 2 (800 items)
    ("js1_ring", dict(kind=L, cfg=dict(dim=16), B=5, N=700, seed=601, mask="padded",
                      check=[(0, 8), (172, 180), (344, 352), (690, 700)]), "per_graph", "per_graph"),
    ("js2_ring", dict(kind=L, cfg=dict(dim=24, fourier_features=1, soft_edges=True), B=2, N=800, seed=602,
                      mask="random",
                      check=[(0, 8), (396, 404), (792, 800)]), "per_graph", "per_graph"),
    # j-split 4 over a whole graph (generic: fourier + edges), on a row range ending with 3 valid rows; j-split 8 on a
    # row range ending with 1 valid row (lean)
    ("js4_full", dict(kind=L, cfg=dict(dim=16, fourier_features=2, edge_dim=4), B=1, N=1100, seed=603,
                      check=[(0, 8), (548, 556), (1092, 1100)]), BOX3, "tilt"),
    ("js4_range", dict(kind=L, cfg=dict(dim=24, fourier_features=2, edge_dim=4, norm_coors=True), B=2, N=1024,
                       seed=604, rows=(0, 63), mask="padded"), "per_graph", "per_graph"),
    ("js8_range", dict(kind=L, cfg=dict(dim=16, coor_weights_clamp_value=2.0), B=1, N=2048, seed=605, rows=(5, 34)),
     BOX3, "tilt"),
    # one active warpgroup, one fully masked graph
    ("n100_empty", dict(kind=L, cfg=dict(dim=64, m_pool_method="mean"), B=3, N=100, seed=606, mask="one_empty"),
     "per_graph", "per_graph"),
    # partial / full / one-more warp and warpgroup tiles
    ("n63", dict(kind=L, cfg=dict(dim=32, coor_weights_clamp_value=0.5), B=2, N=63, seed=607, mask="random"),
     "per_graph", "per_graph"),
    ("n64", dict(kind=L, cfg=dict(dim=32, m_pool_method="mean"), B=2, N=64, seed=608, mask="padded"), BOX3, "tilt"),
    ("n65", dict(kind=L, cfg=dict(dim=24, soft_edges=True), B=2, N=65, seed=609), "per_graph", "per_graph"),
    ("n127", dict(kind=L, cfg=dict(dim=32, norm_coors=True), B=2, N=127, seed=610), BOX3, "tilt"),
    ("n128", dict(kind=L, cfg=dict(dim=32, soft_edges=True), B=2, N=128, seed=611, mask="random"), "per_graph",
     "per_graph"),
    ("n129", dict(kind=L, cfg=dict(dim=24, coor_weights_clamp_value=1.0), B=2, N=129, seed=612), BOX3, "tilt"),
    ("n255", dict(kind=L, cfg=dict(dim=40, m_pool_method="mean"), B=2, N=255, seed=613), "per_graph", "per_graph"),
    ("n256", dict(kind=L, cfg=dict(dim=16, soft_edges=True, coor_weights_clamp_value=2.0), B=2, N=256, seed=614,
                  mask="padded"), BOX3, "tilt"),
    ("n257", dict(kind=L, cfg=dict(dim=16, norm_coors=True), B=2, N=257, seed=615, mask="random"), "per_graph",
     "per_graph"),
    # the widest lean layer (Hp = 2736)
    ("d680", dict(kind=L, cfg=dict(dim=680), B=1, N=70, seed=616, mask="padded"), BOX3, "tilt"),
    # generic: fourier features, edges and degree labels (Q = 12) through EGNN_Network
    ("net_q12", dict(kind=NW, cfg=dict(depth=1, dim=16, fourier_features=2, edge_dim=3, num_adj_degrees=3, adj_dim=2,
                                       soft_edges=True), B=2, N=150, seed=617, adj="chain", edges=True, mask="padded"),
     "per_graph", "per_graph"),
    # neighbour lists: k = 1 / 8 / 31 / 32, lean / edges / generic at 8 and 16 rows per CTA, partial last CTAs
    ("k8_edges8_slot", dict(kind=L, cfg=dict(dim=64, edge_dim=4), B=2, N=150, k=8, seed=622, holes=True,
                            slot_edges=True, mask="padded"), "per_graph", "per_graph"),
    ("k31_gen8_mean", dict(kind=L, cfg=dict(dim=32, fourier_features=2, m_pool_method="mean"), B=2, N=100, k=31,
                           seed=623, holes=True), BOX3, "tilt"),
    ("k32_lean16", dict(kind=L, cfg=dict(dim=344, coor_weights_clamp_value=3.0), B=1, N=150, k=32, seed=624,
                        holes=True), BOX3, "tilt"),
    ("k32_edges16", dict(kind=L, cfg=dict(dim=280, edge_dim=4), B=2, N=100, k=32, seed=625, holes=True,
                         mask="random"), "per_graph", "per_graph"),
    ("k31_gen16_rows", dict(kind=L, cfg=dict(dim=264, fourier_features=2, edge_dim=1, m_pool_method="mean"), B=2,
                            N=150, k=31, seed=628, holes=True, slot_edges=True, mask="padded", rows=(19, 140)),
     "per_graph", "per_graph"),
    # the BASELINE shapes as the lattice benches time them: c2 (dense dim 512, B=4, N=1024) with a box and with a
    # tilted cell
    ("c2", dict(kind=L, cfg=dict(dim=512), B=4, N=1024, seed=631, check=[(0, 8), (508, 516), (1016, 1024)]),
     [4.0, 4.0, 4.0], "tilt"),
]
LATTICE_CASES = {}
for _n, _s, _box, _cell in LATTICE_SHAPES:
    _k = "k" if _s.get("k") else "p"
    LATTICE_CASES[f"{_k}b_{_n}"] = dict(_s, box=_box)
    LATTICE_CASES[f"{_k}c_{_n}"] = dict(_s, cell=_cell, seed=_s["seed"] + 100)
LATTICE_CASES.update({
    # the lean 8-row list kernel: k = 1 under a cell, k = 8 under a box (at k = 1 the per-row coordinate gate compares
    # the error of one coordinate weight with its value; DESIGN section 5 gives what that measured under a box)
    "kc_k1_lean8":     dict(kind=L, cfg=dict(dim=32), B=2, N=203, k=1, seed=734, cell="per_graph"),
    "kb_k8_lean8":     dict(kind=L, cfg=dict(dim=32), B=2, N=203, k=8, seed=635, holes=True, box="per_graph"),
    # box only: the generic instantiation at C = 5 and C = 8 with aperiodic (0, inf) and periodic axes
    "pb_c5_mixed":     dict(kind=L, cfg=dict(dim=16, edge_dim=2, soft_edges=True), B=2, N=90, C=5, seed=641,
                            mask="random", box=[3.0, INF, 2.5, 0.0, 3.5]),
    "pb_c8_mixed":     dict(kind=L, cfg=dict(dim=32, fourier_features=1, m_pool_method="mean"), B=2, N=100, C=8,
                            seed=642, box=[3.0, 0.0, 2.75, INF, 3.25, 3.0, 0.0, 3.5]),
    "pb_net_q12_c8":   dict(kind=NW, cfg=dict(depth=1, dim=16, fourier_features=2, edge_dim=3, num_adj_degrees=3,
                                              adj_dim=2), B=2, N=120, C=8, seed=643, adj="chain", edges=True,
                            box=[2.5, INF, 3.0, 0.0, 3.5, 2.75, INF, 3.25]),
    # j-split 8 on a row range, generic (for the diagonal-cell identity)
    "pb_js8_range_gen": dict(kind=L, cfg=dict(dim=16, fourier_features=1), B=1, N=2048, seed=644, rows=(5, 34),
                             box=BOX3),
    # cell only: a 2-D cell (generic), a hexagonal slab, a tilt of 0.9
    "pc_c2_gen":       dict(kind=L, cfg=dict(dim=16, m_pool_method="mean"), B=2, N=300, C=2, seed=651, mask="padded",
                            cell="c2"),
    "pc_hex_slab":     dict(kind=L, cfg=dict(dim=32, soft_edges=True), B=2, N=60, seed=652, cell="hex_slab"),
    "pc_tilt09":       dict(kind=L, cfg=dict(dim=32, norm_coors=True), B=2, N=300, seed=653, mask="random",
                            cell="tilt09"),
    "kc_c2_gen8":      dict(kind=L, cfg=dict(dim=32), B=2, N=90, C=2, k=8, seed=654, holes=True, cell="c2"),
    # c4 (dim 256, edge_dim 4, B=8, N=4096) on caller lists of 32 with per-slot edges and a box per graph
    "kb_c4":           dict(kind=L, cfg=dict(dim=256, edge_dim=4), B=8, N=4096, k=32, seed=661, slot_edges=True,
                            box="per_graph", check=[(0, 16), (2040, 2056), (4080, 4096)]),
})
CASES.update(LATTICE_CASES)

# ------------------------------------------------------------------ launch geometry (launch_geometry.tc_layer)


def geometry(spec, sms=LG.H100_SMS):
    """What the launch code (fast_path.cu) runs a case with, and the case's lattice."""
    lat = spec.get("box", spec.get("cell"))
    g = LG.tc_layer(spec["kind"], spec["cfg"], spec["B"], spec["N"], C=spec.get("C", 3), k=spec.get("k", 0),
                    rows=spec.get("rows"), sms=sms)
    return dict(g, lattice=lattice_kind(spec), per_graph_lattice=lat == "per_graph" and spec["B"] > 1)


def test_table_covers_every_boundary():
    """Each boundary the table is meant to reach, recomputed from the specs: an edit to a shape that drops one fails
    here.  The SM count is the H100's 132, or the device's when one is present."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else LG.H100_SMS
    geo = {n: geometry(s, sms) for n, s in CASES.items()}
    assert all(g["supported"] for g in geo.values()), [n for n, g in geo.items() if not g["supported"]]
    pair = {n: g for n, g in geo.items() if g["k"] == 0}
    knn = {n: g for n, g in geo.items() if g["k"] > 0}
    want = {
        "jsplit 1 / 2 / 4 / 8": {g["jsplit"] for g in pair.values()} >= {1, 2, 4, 8},
        "jsplit 4 on a full graph": any(g["jsplit"] == 4 and not g["rows_range"] for g in pair.values()),
        "jsplit 4 and 8 on row ranges": {g["jsplit"] for g in pair.values() if g["rows_range"]} >= {4, 8},
        "one active warpgroup": any(g["active_wgs"] == 1 for g in pair.values()),
        "N 63..65 / 127..129 / 191..193 / 255..257": {g["N"] for g in pair.values()} >= {
            63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257},
        "dense lean at Hp 2736": any(g["kernel"] == "tc_pair<lean>" and g["Hp"] == 2736 for g in pair.values()),
        "last row group 1 / 2 / 3 rows at a graph end": {g["last_rows_valid"] for g in pair.values()
                                                         if not g["rows_range"]} >= {1, 2, 3},
        "last row group 1 / 3 rows at a range end": {g["last_rows_valid"] for g in pair.values()
                                                     if g["rows_range"]} >= {1, 3},
        "ring reuse, odd laps": any(g["items"] > 2 * g["grid"] and g["laps"] % 2 == 1 for g in pair.values()),
        "dense last chunk 1 / 2 / 3 / 4 slabs": {g["nsl_last"] for g in pair.values()} >= {1, 2, 3, 4},
        "dense batches": any(g["B"] >= 2 and g["N"] % 128 != 0 for g in pair.values()),
        "dense lean and generic": {g["kernel"] for g in pair.values()} == {"tc_pair<lean>", "tc_pair<generic>"},
        "dense Q 12, C 8, labels": any(g["Q"] == LG.TP_QMAX and g["C"] == LG.TP_CMAX and g["labels"] > 0
                                       for g in pair.values()),
        "dense fourier and edges": any(g["F"] > 0 and g["edge_dim"] > 0 for g in pair.values()),
        "knn k 1 / 8 / 31 / 32": {g["k"] for g in knn.values()} >= {1, 8, 31, 32},
        "knn every instantiation at 8 and 16 rows": {g["kernel"] for g in knn.values()} >= {
            f"tc_knn<{m},{r}>" for m in ("LEAN", "EDGES", "GEN") for r in (8, 16)},
        "knn partial last CTA at 8 and 16 rows": {g["ROWS"] for g in knn.values() if g["last_rows_valid"] < g["ROWS"]}
        == {8, 16},
        "knn 16 rows with more than 8 valid rows": any(g["ROWS"] == 16 and g["R"] > 8 for g in knn.values()),
        "knn row ranges": any(g["rows_range"] for g in knn.values()),
        "small tables + small node": any(g["tables"] == "small" and g["node"] == "small" for g in geo.values()),
        "tc_gemm tables at dim <= 64": any(g["tables"] == "tc_gemm" and g["dim"] <= 64 for g in geo.values())
        and any(g["tables"] == "tc_gemm" and g["dim"] <= 64 for g in pair.values()),
        "GEMM node path (dim > 64)": any(g["node"] == "tc_gemm" for g in pair.values())
        and any(g["node"] == "tc_gemm" for g in knn.values()),
    }
    missing = [k for k, v in want.items() if not v]
    assert not missing, missing
    opts = [(s.get("mask"), s["cfg"]) for s in CASES.values()]
    assert {m for m, _ in opts} >= {"padded", "random", "one_empty", None}
    for key in ("soft_edges", "norm_coors", "coor_weights_clamp_value", "norm_feats"):
        assert any(key in c for _, c in opts), key
    assert any(c.get("m_pool_method") == "mean" and s.get("k") and not s.get("mask") for s in CASES.values()
               for c in [s["cfg"]]), "mean over lists without a mask"
    assert any(s.get("holes") for s in CASES.values()) and any(s.get("slot_edges") for s in CASES.values())
    # ... and again under a box and under a cell
    for lat in ("box", "cell"):
        lp = {n: g for n, g in pair.items() if g["lattice"] == lat}
        lk = {n: g for n, g in knn.items() if g["lattice"] == lat}
        ls = [CASES[n] for n in list(lp) + list(lk)]
        want = {
            "jsplit 1 / 2 / 4 / 8": {g["jsplit"] for g in lp.values()} >= {1, 2, 4, 8},
            "jsplit 4 and 8 on row ranges ending with 3 / 1 valid rows": {
                (g["jsplit"], g["last_rows_valid"]) for g in lp.values() if g["rows_range"]} >= {(4, 3), (8, 1)},
            "ring refilled with another graph's row group, per-graph lattices, odd laps, at jsplit 1 and >= 2": {
                min(g["jsplit"], 2) for g in lp.values()
                if g["refill_other_graph"] and g["per_graph_lattice"] and g["laps"] % 2 == 1} == {1, 2},
            "one active warpgroup": any(g["active_wgs"] == 1 for g in lp.values()),
            "N 63..65 / 127..129 / 255..257": {g["N"] for g in lp.values()} >= {63, 64, 65, 127, 128, 129, 255, 256,
                                                                                257},
            "dense lean at Hp 2736": any(g["kernel"] == "tc_pair<lean>" and g["Hp"] == 2736 for g in lp.values()),
            "dense lean and generic": {g["kernel"] for g in lp.values()} == {"tc_pair<lean>", "tc_pair<generic>"},
            "network, Q 12 with labels, fourier and edges": any(
                CASES[n]["kind"] == NW and g["Q"] == LG.TP_QMAX and g["labels"] > 0 and g["F"] > 0 and g["edge_dim"] > 0
                for n, g in lp.items()),
            "knn k 1 (cell) / 8 / 31 / 32": {g["k"] for g in lk.values()} >= ({1} if lat == "cell" else set()) | {
                8, 31, 32},
            "knn every instantiation at 8 and 16 rows": {g["kernel"] for g in lk.values()} >= {
                f"tc_knn<{m},{r}>" for m in ("LEAN", "EDGES", "GEN") for r in (8, 16)},
            "knn partial last CTA at 8 and 16 rows": {
                g["ROWS"] for g in lk.values() if g["last_rows_valid"] < g["ROWS"]} == {8, 16},
            "knn row ranges": any(g["rows_range"] for g in lk.values()),
            "knn per-graph lattices": any(g["per_graph_lattice"] for g in lk.values()),
            "knn -1 slots and per-slot edges": any(s.get("holes") for s in ls if s.get("k"))
            and any(s.get("slot_edges") for s in ls if s.get("k")),
            "c2 (dense dim 512, B 4, N 1024)": any(g["dim"] == 512 and g["B"] == 4 and g["N"] == 1024 and g["k"] == 0
                                                   for g in lp.values()),
        }
        missing = [k for k, v in want.items() if not v]
        assert not missing, (lat, missing)
        assert {s.get("mask") for s in ls} >= {"padded", "random", "one_empty"}, lat
        for key in ("soft_edges", "norm_coors", "coor_weights_clamp_value"):
            assert any(key in s["cfg"] for s in ls), (lat, key)
        assert any(s["cfg"].get("m_pool_method") == "mean" for s in ls), lat
    # box only: the generic kernel at C = 5 and C = 8 with aperiodic (0, inf) and periodic axes
    mixed = lambda b: not isinstance(b, str) and {0.0, INF} <= set(b) and any(0 < v < INF for v in b)
    assert {g["C"] for n, g in pair.items() if g["kernel"] == "tc_pair<generic>" and mixed(CASES[n].get("box", "x"))
            } >= {5, 8}
    # cell only: a 2-D cell on the generic kernel, a hexagonal slab, a tilt of 0.9
    assert any(g["C"] == 2 and g["kernel"] == "tc_pair<generic>" and g["lattice"] == "cell" for g in pair.values())
    assert {CASES[n].get("cell") for n in pair} >= {"hex_slab", "tilt09"}
    # c4 (dim 256, edge_dim 4, k 32, B 8, N 4096) on caller lists with per-slot edges and a box per graph
    assert any(g["dim"] == 256 and g["edge_dim"] == 4 and g["k"] == 32 and g["B"] == 8 and g["N"] == 4096
               and g["lattice"] == "box" and g["per_graph_lattice"] and CASES[n].get("slot_edges")
               for n, g in knn.items())


# ------------------------------------------------------------------ inputs and the reference


def lattice_kind(spec):
    return "box" if "box" in spec else ("cell" if "cell" in spec else None)


# Cells: fractional coordinates on an odd 1/21 grid (plus a jitter below 1e-5) and tilts that are whole multiples of
# L_c / 21, so that every wrap decision r_c / L_c lies within 1e-4 of a multiple of 1/441, and 1/441 (odd) keeps
# those 1.13e-3 away from 1/2: fp32 and fp64 pick the same image at any N.  The hexagonal slab's a / 2 tilt is no
# such multiple; its nodes are redrawn until they clear the margin (test_triclinic.cell_coors), at small N.
CELL_GRID = 21


def _grid_cell(rs, Ls, tilt):
    A = np.diag(np.asarray(Ls, np.float64))
    m = int(tilt * CELL_GRID)
    for r in range(1, len(Ls)):
        for c in range(r):
            A[r, c] = rs.choice([-1, 1]) * rs.randint(3, m + 1) * Ls[c] / CELL_GRID
    return A


def lattice_inputs(spec, rs):
    """(lattice, coordinates [B, N, C]) of a case, both fp32 values as float64.  Box: coordinates on an odd lattice of
    the box (test_periodic.lattice_coors); cell: on the CELL_GRID; both moved by whole lattice vectors in [-2, 2]."""
    B, N, C = spec["B"], spec["N"], spec.get("C", 3)
    if "box" in spec:
        box = spec["box"]
        if isinstance(box, str):                                  # "per_graph"
            box = np.round(rs.uniform(2.5, 4.0, (B, C)) * 64) / 64
        box = np.asarray(box, np.float64)
        scale = np.where(np.isfinite(box) & (box > 0), box, 3.0)
        x = np.concatenate([PER.lattice_coors(rs, 1, N, C, sc) for sc in np.broadcast_to(scale, (B, C))])
        return box, util.rounded(x, torch.float32)
    kind = spec["cell"]
    if kind == "hex_slab":
        cell = util.rounded(TRI.make_cell(kind, B, rs), torch.float32)
        return cell, TRI.cell_coors(rs, B, N, cell, dtype=torch.float32)
    Ls = [3.0, 3.25, 3.5][:C] if kind != "c2" else [3.0, 2.75]
    if kind == "tilt":
        cell = _grid_cell(rs, Ls, 0.5)
    elif kind == "tilt09":
        cell = _grid_cell(rs, Ls, 0.3)
        cell[2, 0] = 19 * Ls[0] / CELL_GRID                       # 0.905 L_0
    elif kind == "c2":
        cell = _grid_cell(rs, Ls, 0.5)
    else:                                                         # "per_graph"
        cell = np.stack([_grid_cell(rs, np.round(rs.uniform(2.8, 3.6, C) * 64) / 64, 0.5) for _ in range(B)])
    cell = util.rounded(cell, torch.float32)
    A = np.broadcast_to(cell, (B, C, C))
    s = (rs.randint(0, CELL_GRID, (B, N, C)) / CELL_GRID + rs.uniform(-1e-5, 1e-5, (B, N, C))
         + rs.randint(-2, 3, (B, N, C)))
    return cell, util.rounded(np.einsum("bnk,bkd->bnd", s, A), torch.float32)


@functools.lru_cache(maxsize=None)
def build(name):
    """The case with bf16 parameters / features / edges and fp32 coordinates, plus its neighbour lists."""
    spec = CASES[name]
    lat = lattice_kind(spec)
    case = cases.build_case(dict({k: v for k, v in spec.items() if k not in ("check", "rows", "box", "cell")},
                                 init="xavier", dense_edges=not (lat and spec.get("slot_edges"))))
    ins = case["inputs"]
    if lat:
        case[lat], ins["coors"] = lattice_inputs(spec, np.random.RandomState(spec["seed"] + 11))
    case["params"] = {k: util.rounded(v, torch.bfloat16) for k, v in case["params"].items()}
    if np.issubdtype(np.asarray(ins["feats"]).dtype, np.floating):
        ins["feats"] = util.rounded(ins["feats"], torch.bfloat16)
    ins["coors"] = np.asarray(ins["coors"], np.float32).astype(np.float64)
    if ins.get("edges") is not None and np.issubdtype(np.asarray(ins["edges"]).dtype, np.floating):
        ins["edges"] = util.rounded(ins["edges"], torch.bfloat16)
    k = spec.get("k", 0)
    if k:
        B, N = spec["B"], spec["N"]
        rs = np.random.RandomState(spec["seed"] + 7)
        if spec.get("slot_edges") and not lat:   # distinct neighbours per row: the oracle takes per-slot edges as
            nbr = rs.uniform(size=(B, N, N)).argsort(-1)[..., :k]     # [B, N, N, e] (the restatement takes them per slot)
        else:
            nbr = rs.randint(0, N, (B, N, k))
        if spec.get("holes"):
            holes = rs.uniform(size=nbr.shape) < 0.2
            holes[:, ::2, -1] = False                                   # the last slot stays in use on half the rows
            nbr[holes] = -1
        ins["neighbors"] = nbr
        if spec.get("slot_edges"):
            ins["edges"] = util.rounded(rs.standard_normal((B, N, k, case["cfg"]["edge_dim"])), torch.bfloat16)
    return case


def windows(name):
    spec = CASES[name]
    return spec.get("check") or [spec.get("rows") or (0, spec["N"])]


def lattice_kw(name):
    """{'box': [C] | [B, C]} or {'cell': [C, C] | [B, C, C]} (fp32 values as float64) of a case, or {}."""
    case = build(name)
    return {k: case[k] for k in ("box", "cell") if k in case}


def reference(name, rounding=True, messages=True, lattice=None):
    """[(window, feats, coors)] of the reference over the case's check windows.  `lattice`: a {'box' | 'cell': ...}
    to use instead of the case's own ({} for none)."""
    case = build(name)
    ins = case["inputs"]
    lat = lattice_kw(name) if lattice is None else lattice
    if case["kind"] == NW:
        assert messages
        f, x = T.tc_network_forward(case["params"], case["ncfg"], ins["feats"], ins["coors"], ins.get("adj_mat"),
                                    ins.get("edges"), ins.get("mask"), rounding=rounding, **lat)
        return [((0, CASES[name]["N"]), f, x)]
    spec = CASES[name]
    out = []
    for w in windows(name):
        f, x = T.tc_layer_forward(case["params"], case["cfg"], ins["feats"], ins["coors"], edges=ins.get("edges"),
                                  mask=ins.get("mask"), neighbors=ins.get("neighbors"),
                                  slot_edges=bool(spec.get("slot_edges")), rows=w, rounding=rounding,
                                  messages=messages, **lat)
        out.append((w, f, x))
    return out


@functools.lru_cache(maxsize=None)
def reference_cached(name):
    return reference(name)


def oracle(name):
    """[(window, feats, coors)] of the fp64 oracle over the same windows (under a lattice: the float64 periodic
    restatement, torch_reference.layer / .network, with test_triclinic's cell wrap for a cell)."""
    case = build(name)
    ins = case["inputs"]
    if lattice_kind(CASES[name]):
        return restatement(name)
    if case["kind"] == NW:
        f, x = cases.run_oracle(case)
        return [((0, CASES[name]["N"]), f, x)]
    if "neighbors" in ins:
        e = ins.get("edges")
        if CASES[name].get("slot_edges"):          # per-slot edges -> the dense [B, N, N, e] tensor the oracle takes
            B, N, k = ins["neighbors"].shape
            dense = np.zeros((B, N, N, e.shape[-1]))
            b_, i_, s_ = np.nonzero(ins["neighbors"] >= 0)
            dense[b_, i_, ins["neighbors"][b_, i_, s_]] = e[b_, i_, s_]      # (`build` draws these lists without repeats)
            e = dense
        f, x = O.egnn_layer_forward_edge_list(case["params"], case["cfg"], ins["feats"], ins["coors"], ins["neighbors"],
                                              edges=e, mask=ins.get("mask"))
        return [(w, f[:, w[0]:w[1]], x[:, w[0]:w[1]]) for w in windows(name)]
    return [(w,) + tuple(O.egnn_layer_forward(case["params"], case["cfg"], ins["feats"], ins["coors"],
                                              edges=ins.get("edges"), mask=ins.get("mask"), rows=w))
            for w in windows(name)]


def restatement(name):
    case = build(name)
    ins = case["inputs"]
    lat = lattice_kw(name)
    geometry_ctx = TRI._cell_geometry() if "cell" in lat else contextlib.nullcontext()
    with geometry_ctx:
        lattice = next(iter(lat.values()))
        if case["kind"] == NW:
            f, x, _ = R.network(case["params"], case["ncfg"], ins["feats"], ins["coors"], ins.get("adj_mat"),
                                ins.get("edges"), ins.get("mask"), box=lattice)
            return [((0, CASES[name]["N"]), f.numpy(), x.numpy())]
        slot = CASES[name].get("slot_edges")
        out = []
        for w in windows(name):
            f, x = R.layer(case["params"], case["cfg"], ins["feats"], ins["coors"], None if slot else ins.get("edges"),
                           ins.get("mask"), None, lattice, ins.get("neighbors"), ins.get("edges") if slot else None,
                           rows=w)
            out.append((w, f.numpy(), x.numpy()))
    return out


def test_every_case_sees_the_edge_kernel():
    """On the reference: the coordinate update of every case is O(0.1 - 1) per row or larger, and the messages move
    the features by more than 2 % of their scale (several bf16 ulps), so an error in the edge kernel shows in both outputs."""
    for name in CASES:
        case = build(name)
        x_in = case["inputs"]["coors"]
        ref = reference_cached(name)
        upd = np.concatenate([np.abs(x - x_in[:, w[0]:w[1]]).max(-1).ravel() for w, _, x in ref])
        live = upd[upd > 0]
        assert live.size > 0.5 * upd.size and np.median(live) > 0.1, (name, np.median(live) if live.size else 0)
        if case["kind"] == NW:
            continue
        nomsg = reference(name, messages=False)
        share = max(float(np.abs(f - f0).max() / np.abs(f).max()) for (_, f, _), (_, f0, _) in zip(ref, nomsg))
        assert share > 0.02, (name, share)


@pytest.mark.parametrize("name", ["p_js2_n701", "p_js4_range", "p_c8_mean_clamp", "k8_edges8_slot", "k31_gen16_rows"])
def test_reference_rounding_stays_within_the_oracle_gate(name):
    """The rounded reference is within the bf16 gate of test_gpu_fast.py of the fp64 oracle (it models the kernels'
    rounding, not a different function)."""
    for (w, f, x), (_, fo, xo) in zip(reference_cached(name), oracle(name)):
        x_in = build(name)["inputs"]["coors"][:, w[0]:w[1]]
        assert np.abs(f - fo).max() <= 1e-2 * np.abs(fo).max(), name
        assert np.abs(x - xo).max() <= 1e-2 * max(np.abs(xo - x_in).max(), 1.0), name


# ------------------------------------------------------------------ the reference pinned to the oracles (CPU)

PIN_LAYER = ["dense_everything", "dense_c5", "dense_mean", "dense_clamp", "dense_soft_edges", "dense_norm_coors",
             "dense_mask_random", "dense_no_feats", "dense_no_coors", "knn_edges_mask", "knn_radius_mask",
             "knn_radius_nomask", "knn_mean_fourier", "knn_norm_coors", "knn_k32_c5", "adj_sparse_random"]
PIN_NETWORK = ["net_adj_dense", "net_adj_degrees", "net_c5_xavier", "net_edge_tokens", "net_c3_xavier"]


@pytest.mark.parametrize("name", PIN_LAYER + PIN_NETWORK)
def test_unrounded_reference_equals_the_oracle(name):
    c = cases.build_case(cases.SPECS[name])
    ins = c["inputs"]
    want = cases.run_oracle(c)
    if c["kind"] == NW:
        got = T.tc_network_forward(c["params"], c["ncfg"], ins["feats"], ins["coors"], ins.get("adj_mat"),
                                   ins.get("edges"), ins.get("mask"), rounding=False)
    else:
        cfg, nbr, ok = c["cfg"], None, None
        if cfg["num_nearest_neighbors"] > 0 or cfg["only_sparse_neighbors"]:
            nbr, ok, _ = O.neighbour_selection(cfg, ins["coors"], ins.get("mask"), ins.get("adj_mat"))
        got = T.tc_layer_forward(c["params"], cfg, ins["feats"], ins["coors"], edges=ins.get("edges"),
                                 mask=ins.get("mask"), neighbors=nbr, nbr_ok=ok, rounding=False)
    for g, w in zip(got, want):
        assert np.abs(g - w).max() <= 1e-12 * max(1.0, np.abs(w).max()), name


@pytest.mark.parametrize("mean", [False, True])
@pytest.mark.parametrize("masked", [False, True])
def test_unrounded_reference_equals_the_edge_list_oracle(masked, mean):
    """Caller lists with -1 slots and per-slot edges (edge-list mode) against oracle.egnn_layer_forward_edge_list."""
    spec = dict(kind=L, cfg=dict(dim=16, edge_dim=2, fourier_features=1, soft_edges=True, norm_coors=True,
                                 coor_weights_clamp_value=0.8, m_pool_method="mean" if mean else "sum"),
                B=2, N=23, seed=430, init="xavier", mask="random" if masked else "none")
    c = cases.build_case(spec)
    ins = c["inputs"]
    rs = np.random.RandomState(5)
    k = 6
    nbr = np.stack([np.stack([rs.permutation(23)[:k] for _ in range(23)]) for _ in range(2)])
    nbr[rs.uniform(size=nbr.shape) < 0.25] = -1
    slot = rs.standard_normal((2, 23, k, 2))
    dense = np.zeros((2, 23, 23, 2))
    b_, i_, s_ = np.nonzero(nbr >= 0)
    dense[b_, i_, nbr[b_, i_, s_]] = slot[b_, i_, s_]
    want = O.egnn_layer_forward_edge_list(c["params"], c["cfg"], ins["feats"], ins["coors"], nbr, edges=dense,
                                          mask=ins.get("mask"))
    for edges, per_slot in ((dense, False), (slot, True)):
        got = T.tc_layer_forward(c["params"], c["cfg"], ins["feats"], ins["coors"], edges=edges, mask=ins.get("mask"),
                                 neighbors=nbr, slot_edges=per_slot, rounding=False)
        for g, w in zip(got, want):
            assert np.abs(g - w).max() <= 1e-12 * max(1.0, np.abs(w).max())


def test_rounded_reference_stays_within_the_oracle_gate_on_pinned_cases():
    for name in ["dense_everything", "knn_edges_mask", "net_adj_dense"]:
        c = cases.build_case(cases.SPECS[name])
        c["params"] = {k: util.rounded(v, torch.bfloat16) for k, v in c["params"].items()}
        ins = c["inputs"]
        for key in ("feats", "coors", "edges"):
            if ins.get(key) is not None and np.issubdtype(np.asarray(ins[key]).dtype, np.floating):
                ins[key] = util.rounded(ins[key], torch.bfloat16)
        want = cases.run_oracle(c)
        if c["kind"] == NW:
            got = T.tc_network_forward(c["params"], c["ncfg"], ins["feats"], ins["coors"], ins.get("adj_mat"),
                                       ins.get("edges"), ins.get("mask"))
        else:
            nbr, ok = None, None
            if c["cfg"]["num_nearest_neighbors"] > 0:
                nbr, ok, _ = O.neighbour_selection(c["cfg"], ins["coors"], ins.get("mask"), None)
            got = T.tc_layer_forward(c["params"], c["cfg"], ins["feats"], ins["coors"], edges=ins.get("edges"),
                                     mask=ins.get("mask"), neighbors=nbr, nbr_ok=ok)
        assert np.abs(got[0] - want[0]).max() <= 1e-2 * np.abs(want[0]).max(), name
        assert np.abs(got[1] - want[1]).max() <= 1e-2 * max(np.abs(want[1] - ins["coors"]).max(), 1.0), name


# ------------------------------------------------------------------ periodic cases: inputs, the wrap, sensitivity (CPU)


def graph_lattice(name, b):
    kind = lattice_kind(CASES[name])
    lat = np.asarray(lattice_kw(name)[kind])
    return lat[b] if lat.ndim == (2 if kind == "box" else 3) else lat


def compared_pairs(name):
    """[(graph, rel [P, C])]: fp32(x_i - x_j) of every unmasked pair the gates compare (check windows, listed slots)."""
    ins = build(name)["inputs"]
    x, mk, nb = ins["coors"], ins.get("mask"), ins.get("neighbors")
    out = []
    for b in range(x.shape[0]):
        for w in windows(name):
            ii = np.arange(*w)
            if nb is None:
                jj = np.broadcast_to(np.arange(x.shape[1]), (len(ii), x.shape[1]))
                ok = np.ones(jj.shape, bool)
            else:
                jj = nb[b, w[0]:w[1]]
                ok = jj >= 0
                jj = np.where(ok, jj, ii[:, None])
            if mk is not None:
                ok = ok & mk[b, ii][:, None] & mk[b, jj]
            out.append((b, util.rounded(x[b, ii][:, None] - x[b, jj], torch.float32)[ok]))
    return out


def wrap_decisions(rel, kind, lat):
    """Float64 wrap of rel [P, C] under one graph's box [C] or cell [C, C] -> (smallest distance of r_c / L_c from 1/2
    (mod 1) over each pair's decisions, whether any image count of the pair is nonzero)."""
    A = np.diag(lat) if kind == "box" else np.asarray(lat)
    r = rel.copy()
    margin, moved = np.ones(len(r)), np.zeros(len(r), bool)
    for c in reversed(range(r.shape[-1])):
        Lc = A[c, c]
        if not (np.isfinite(Lc) and Lc > 0):
            continue
        t = r[:, c] / Lc
        margin = np.minimum(margin, np.abs(np.abs(t - np.rint(t)) - 0.5))
        n = np.rint(t)
        moved |= n != 0
        r[:, :c + 1] -= n[:, None] * A[c, :c + 1]
    return margin, moved


@pytest.mark.parametrize("name", list(LATTICE_CASES))
def test_lattice_inputs_wrap_often_and_stay_off_one_half(name):
    """Every wrap decision of a compared pair lies >= 1e-3 from 1/2, so fp32 and fp64 pick the same image (and the
    fp64 restatement's gate holds), and >= 20 % of the compared, unmasked pairs are moved by a lattice vector."""
    kind = lattice_kind(CASES[name])
    margin, moved, total = 1.0, 0, 0
    for b, rel in compared_pairs(name):
        m, mv = wrap_decisions(rel, kind, graph_lattice(name, b))
        margin = min(margin, float(m.min(initial=1.0)))
        moved += int(mv.sum())
        total += len(mv)
    assert margin >= 1e-3, (name, margin)
    assert moved >= 0.2 * total, (name, moved / total)


def _fp32_exact(q):
    """The Fraction q rounded to the nearest fp32 (ties to even; normal range)."""
    if q == 0:
        return Fraction(0)
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length() - 23
    while a / Fraction(2) ** e >= 2 ** 24:
        e += 1
    while a / Fraction(2) ** e < 2 ** 23:
        e -= 1
    return (1 if q > 0 else -1) * round(a / Fraction(2) ** e) * Fraction(2) ** e


def _exact_step(r, L, inv, coef=None):
    """n = rint(fp32(r * inv)) and fp32(-coef * n + r) (coef: L), exactly."""
    n = round(_fp32_exact(r * inv))
    return n, _fp32_exact(-(L if coef is None else coef) * n + r)


def _near_half(rs, L, size):
    """fp32 values within 3 ulps of (n + 1/2) L, n in [-4, 4]."""
    v = ((rs.randint(-4, 5, size) + 0.5) * L).astype(np.float32)
    for _ in range(3):
        step = rs.randint(-1, 2, size)
        v = np.where(step > 0, np.nextafter(v, np.float32(np.inf)),
                     np.where(step < 0, np.nextafter(v, np.float32(-np.inf)), v))
    return v


def test_rounded_wrap_is_the_kernels_fp32_sequence_exactly():
    """tc_reference's fp32 wrap (box: min_image, cell: cell_wrap_n) equals an exact rational evaluation of the same
    operation sequence, with one rounding to fp32 per operation, on 10^4 draws of each -- half of them within 3 ulps
    of (n + 1/2) L, where the image flips."""
    rs = np.random.RandomState(17)
    M = 10000
    L = rs.uniform(0.3, 12.0, M).astype(np.float32)
    r = np.where(rs.uniform(size=M) < 0.5, _near_half(rs, L, M), (rs.uniform(-6, 6, M) * L).astype(np.float32))
    got = T.wrap_box(torch.as_tensor(r, dtype=torch.float64)[None], torch.as_tensor(L, dtype=torch.float64))[0].numpy()
    for rv, Lv, g in zip(r, L, got):
        Lq = Fraction(float(Lv))
        inv = _fp32_exact(1 / Lq)
        assert Fraction(float(g)) == _exact_step(Fraction(float(rv)), Lq, inv)[1]
    for _ in range(200):
        A = np.tril(rs.uniform(-1.5, 1.5, (3, 3))) + np.diag(rs.uniform(0.5, 6.0, 3))
        if rs.uniform() < 0.2:
            A[rs.randint(3)] = 0.0                                # an aperiodic axis (its whole row: a slab)
        A = A.astype(np.float32)
        rv = (rs.uniform(-8, 8, (50, 3)) * np.abs(np.diag(A)).max()).astype(np.float32)
        if A[2, 2] > 0:
            rv[:25, 2] = _near_half(rs, np.full(25, A[2, 2], np.float32), 25)
        got = T.wrap_cell(torch.as_tensor(rv, dtype=torch.float64), torch.as_tensor(A, dtype=torch.float64)).numpy()
        Aq = [[Fraction(float(v)) for v in row] for row in A]
        invq = [_fp32_exact(1 / Aq[c][c]) if Aq[c][c] > 0 else Fraction(0) for c in range(3)]
        for v, g in zip(rv, got):
            x = [Fraction(float(t)) for t in v]
            for c in (2, 1, 0):
                Lc = Aq[c][c] if Aq[c][c] > 0 else Fraction(0)
                n = round(_fp32_exact(x[c] * invq[c]))
                for d in range(c + 1):
                    x[d] = _fp32_exact(-(Lc if d == c else Aq[c][d]) * n + x[d])
            assert [Fraction(float(t)) for t in g] == x


def _pin(case, **lat):
    """tc_layer_forward(rounding=False) under `lat` against torch_reference.layer (the float64 restatement), dense, or
    on the lists of the restatement's own selection."""
    ins, cfg = case["inputs"], case["cfg"]
    lattice = next(iter(lat.values()))
    want = R.layer(case["params"], cfg, ins["feats"], ins["coors"], ins.get("edges"), ins.get("mask"),
                   ins.get("adj_mat"), lattice)
    nbr = ok = None
    if cfg["num_nearest_neighbors"] > 0 or cfg["only_sparse_neighbors"]:
        x = R._t(ins["coors"])
        b, n, c = x.shape
        d = (R.wrap(x[:, :, None] - x[:, None], R.box_bc(lattice, b, c)[:, None, None, :]) ** 2).sum(-1)
        nbr, ok = R.select(cfg, d, ins.get("mask"), ins.get("adj_mat"))
    got = T.tc_layer_forward(case["params"], cfg, ins["feats"], ins["coors"], edges=ins.get("edges"),
                             mask=ins.get("mask"), neighbors=None if nbr is None else nbr.numpy(),
                             nbr_ok=None if ok is None else ok.numpy(), rounding=False, **lat)
    for g, w in zip(got, want):
        w = w.numpy()
        assert np.abs(g - w).max() <= 1e-12 * max(1.0, np.abs(w).max())


@pytest.mark.parametrize("name", sorted(PER.PCASES))
def test_unrounded_reference_equals_the_periodic_restatement(name):
    case, box = PER.build(name)
    _pin(case, box=box)


@pytest.mark.parametrize("name", sorted(TRI.TCASES))
def test_unrounded_reference_equals_the_triclinic_restatement(name):
    case, cell = TRI.build(name)
    with TRI._cell_geometry():
        _pin(case, cell=cell)


def wrong_lattices(name):
    """[(what, lattice, (tc_reference attribute, replacement) | None)]: mistakes a lattice case must see."""
    kind = lattice_kind(CASES[name])
    lat = np.asarray(lattice_kw(name)[kind])
    out = [("no lattice", {}, None)]
    if lat.ndim == (2 if kind == "box" else 3):
        out.append(("each graph given the next graph's lattice", {kind: np.roll(lat, -1, 0)}, None))
    if kind == "cell":
        eye = np.eye(lat.shape[-1], dtype=bool)
        out.append(("the cell's diagonal", {kind: np.where(eye, lat, 0.0)}, None))
        out.append(("axes wrapped first to last", {kind: lat},
                    ("wrap_cell", functools.partial(T.wrap_cell, first_to_last=True))))
    out.append(("floor for rint", {kind: lat}, ("_rint", torch.floor)))
    return out


@pytest.mark.parametrize("name", list(LATTICE_CASES))
def test_a_wrong_lattice_fails_a_gate(name, monkeypatch):
    """The rounded reference under a wrong lattice fails at least one TOL gate against the right one, for each
    mistake of `wrong_lattices`: a case that passes one could not see that mistake in a kernel."""
    for what, lat, patch in wrong_lattices(name):
        with monkeypatch.context() as m:
            if patch:
                m.setattr(T, *patch)
            g = gates(name, [(f, x) for _, f, x in reference(name, lattice=lat)])
        assert any(g[k] > TOL[k] for k in TOL), (name, what, g)


# ------------------------------------------------------------------ the GPU runs


def run_gpu(name, rows="spec", lattice=None):
    """Forward of the case on the bf16 path -> (feats [B,N,dim] bf16, coors [B,N,C] fp32) on the device.  `lattice`:
    a {'box' | 'cell': ...} to pass instead of the case's own."""
    case = build(name)
    spec = CASES[name]
    ins = case["inputs"]
    rows = spec.get("rows") if rows == "spec" else rows
    mod = util.make_module(case, torch.bfloat16)
    dev = "cuda"
    coors = torch.from_numpy(ins["coors"]).float().to(dev)
    mask = None if ins.get("mask") is None else torch.from_numpy(ins["mask"]).to(dev)
    tb = lambda a: None if a is None else torch.from_numpy(np.asarray(a, np.float64)).to(dev, torch.bfloat16)
    lat = {k: torch.as_tensor(np.asarray(v), dtype=torch.float32, device=dev)
           for k, v in (lattice_kw(name) if lattice is None else lattice).items()}
    with torch.no_grad():
        if case["kind"] == NW:
            f, x = mod(torch.from_numpy(ins["feats"]).to(dev) if not np.issubdtype(ins["feats"].dtype, np.floating)
                       else tb(ins["feats"]), coors, adj_mat=torch.from_numpy(ins["adj_mat"]).to(dev),
                       edges=tb(ins.get("edges")), mask=mask, **lat)
            layers = [l[1] for l in mod.layers]
        else:
            kw = dict(mask=mask, _rows=rows, **lat)
            edges = tb(ins.get("edges"))
            if "neighbors" in ins:
                kw["neighbors"] = torch.from_numpy(ins["neighbors"]).to(dev)
                if spec.get("slot_edges"):
                    kw["neighbor_edges"], edges = edges, None
            f, x = mod(tb(ins["feats"]), coors, edges, **kw)
            layers = [mod]
    assert all(l.last_path == "bf16-tc" for l in layers), name
    assert f.dtype == torch.bfloat16 and x.dtype == torch.float32
    return f, x


def metrics(name, f, x):
    """The four gate values of one GPU output against the rounding-matched reference."""
    return gates(name, [(f[:, w[0]:w[1]].double().cpu().numpy(), x[:, w[0]:w[1]].double().cpu().numpy())
                        for w in windows(name)])


def gates(name, outs):
    """The four gate values of outputs [(feats, coors)] over the case's windows against the rounding-matched reference."""
    x_in = build(name)["inputs"]["coors"]
    fu, fe, cr, ce, cu = [], [], [], [], []
    for (w, rf, rx), (gf, gx) in zip(reference_cached(name), outs):
        floor = 1e-2 * np.abs(rf).max()
        ulp = 2.0 ** (np.floor(np.log2(np.maximum(np.abs(rf), floor))) - 7)
        fu.append((np.abs(gf - rf) / ulp).ravel())
        upd = rx - x_in[:, w[0]:w[1]]
        err = np.abs(gx - rx).max(-1)
        row_upd = np.abs(upd).max(-1)
        cr.append((err / np.maximum(row_upd, 1e-3 * np.abs(upd).max() + 1e-30)).ravel())
        ce.append((gx - rx).ravel())
        cu.append(upd.ravel())
    fu, cr, ce, cu = (np.concatenate(a) for a in (fu, cr, ce, cu))
    return dict(f_ulp_max=float(fu.max()), f_ulp_mean=float(fu.mean()), c_row=float(cr.max()),
                c_rms=float(np.sqrt((ce ** 2).mean() / max((cu ** 2).mean(), 1e-300))))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_matches_rounding_matched_reference(name):
    f, x = run_gpu(name)
    assert np.isfinite(f.float().cpu().numpy()).all() and np.isfinite(x.cpu().numpy()).all()
    m = metrics(name, f, x)
    g = geometry(CASES[name], torch.cuda.get_device_properties(0).multi_processor_count)
    sched = f"jsplit={g['jsplit']}" if g["k"] == 0 else f"ROWS={g['ROWS']}"
    print(f"TCB {name} {g['kernel']} {sched} Hp={g['Hp']} nsl_last={g['nsl_last']} "
          + " ".join(f"{k}={v:.3e}" for k, v in m.items()))
    bad = {k: v for k, v in m.items() if not v <= TOL[k]}
    assert not bad, (name, bad)
    # ... and the gate of test_gpu_fast.py against the fp64 oracle
    x_in = build(name)["inputs"]["coors"]
    for w, of, ox in oracle(name):
        gf = f[:, w[0]:w[1]].double().cpu().numpy()
        gx = x[:, w[0]:w[1]].double().cpu().numpy()
        assert np.abs(gf - of).max() <= 1e-2 * max(1e-3, np.abs(of).max()), name
        assert np.abs(gx - ox).max() <= 1e-2 * max(np.abs(ox - x_in[:, w[0]:w[1]]).max(), 1.0), name


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["pb_js1_ring", "pb_js2_ring", "pb_js8_range", "pb_js8_range_gen"])
def test_a_diagonal_cell_is_the_box_bit_for_bit(name):
    """DESIGN's claim that the off-diagonal steps of a diagonal cell subtract exact zeros, at the ring-reuse (per-graph
    boxes) and j-split 8 row-range shapes, lean and generic."""
    box = np.asarray(lattice_kw(name)["box"])
    cell = np.stack([np.diag(b) for b in box]) if box.ndim == 2 else np.diag(box)
    f_box, x_box = run_gpu(name)
    f_cell, x_cell = run_gpu(name, lattice=dict(cell=cell))
    assert torch.equal(f_box, f_cell) and torch.equal(x_box, x_cell)


def test_the_diagonal_cell_cases_cover_ring_reuse_and_jsplit_8_ranges_lean_and_generic():
    geo = [geometry(CASES[n]) for n in ["pb_js1_ring", "pb_js2_ring", "pb_js8_range", "pb_js8_range_gen"]]
    assert {(g["refill_other_graph"], g["kernel"]) for g in geo if g["per_graph_lattice"]} == {
        (True, "tc_pair<lean>"), (True, "tc_pair<generic>")}
    assert {g["kernel"] for g in geo if g["jsplit"] == 8 and g["rows_range"]} == {"tc_pair<lean>", "tc_pair<generic>"}


@pytest.mark.gpu
@pytest.mark.parametrize("name,full_js", [("p_js8_range", 2), ("p_js4_range", 2), ("pb_js8_range", 2),
                                          ("pc_js8_range", 2)])
def test_jsplit_row_range_is_bit_identical_to_the_full_forward(name, full_js):
    """DESIGN's claim for the row-sharded dense kernel: the fp64 sums across tiles make the rows independent of how
    the j-blocks were dealt, so a row range run at j-split 4 / 8 equals the full forward (j-split 1 / 2) bit for bit.
    Two calls in a row are identical too: the j-split arrival counters are left at zero."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    spec = CASES[name]
    r0, r1 = spec["rows"]
    assert geometry(dict(spec, rows=None), sms)["jsplit"] == full_js and geometry(spec, sms)["jsplit"] > full_js
    f_full, x_full = run_gpu(name, rows=None)
    f1, x1 = run_gpu(name)
    f2, x2 = run_gpu(name)
    assert torch.equal(f1, f2) and torch.equal(x1, x2)
    assert torch.equal(f1[:, r0:r1], f_full[:, r0:r1]) and torch.equal(x1[:, r0:r1], x_full[:, r0:r1])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["k32_lean16", "k31_gen16_rows", "kb_k32_lean16", "kc_k31_gen16_rows"])
def test_knn_16_rows_row_range_is_bit_identical(name):
    """The 16-row neighbour-list kernel on a row range that starts off the CTA grid equals its full forward."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert geometry(CASES[name], sms)["ROWS"] == 16
    n = CASES[name]["N"]
    f_full, x_full = run_gpu(name, rows=None)
    for r0, r1 in [(5, n - 3), (37, 38)]:
        f, x = run_gpu(name, rows=(r0, r1))
        assert torch.equal(f[:, r0:r1], f_full[:, r0:r1]) and torch.equal(x[:, r0:r1], x_full[:, r0:r1])
