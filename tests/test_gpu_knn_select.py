"""The all-pairs neighbour select (csrc/knn_select.cu) against an exact reference, at its schedule boundaries.

Every kNN, `valid_radius` and adjacency layer starts here.  `ref_select` below ranks exactly as the kernels do, in the
coordinates' type (fp32 for fp32 and bf16 layers, fp64 for fp64): per axis r = fl(x_i - x_j), then d = fl(d + fl(r r))
(sq_acc: two roundings, no fma); a padded end -> 1e5; with an adjacency the diagonal -> -1 and adjacent pairs -> 0.  Then a
stable argsort (NaN last, ties to the lower index) keeps k, and ok = rank <= T(valid_radius).  Lists and ok are compared
exactly.  (The oracle's (rel**2).sum(-1) sums 8 axes pairwise, so its fp32 ranks can differ from the kernel's by an ulp.)

The case table crosses the boundaries of launch_select, mirrored in launch_geometry.py and held there by
test_table_covers_every_boundary:
  warp select (k <= 32)  8 and 16 warps per CTA on both sides of the switch (B ceil(N/16) >= 2 SMs); 1, 2 and 3 staging
                         passes of SEL_JC = 1024 candidates; partial 64-candidate groups and partial last CTAs; the CDIM = 3
                         and generic (C = 1, 2, 4, 5, 8) instantiations in fp32 and fp64; k = 1, 2, 16, 31, 32 and k = N
  block sort (k > 32)    k = 33, 64 and N around the power-of-two steps of Npad, up to its size limit N = 16384
  inputs                 farthest- and nearest-first candidate orders, all coincident, integer lattices, one and no valid
                         node; batched and unbatched adjacency with and without a mask; valid_radius equal to ranks, 0, inf;
                         NaN and +-inf coordinates on query nodes and candidates, masked and unmasked
Periodic boxes (which egnn_knn_select does not take) are checked through the layer: its own select against the same
layer run on the reference's periodic lists, bit for bit.  The adjacency row scan (adj_neighbors_kernel), which
select_neighbors runs for only_sparse_neighbors with a mask, is checked on its wide (4-byte) and narrow paths."""
import ctypes as C
import math
import warnings

import numpy as np
import pytest
import torch

import cases
import launch_geometry as LG

DEV = "cuda"
F32, F64 = "f32", "f64"
NP_T = {F32: np.float32, F64: np.float64}
TORCH_T = {F32: torch.float32, F64: torch.float64}

# ------------------------------------------------------------------ the exact reference


def ranks(x, rows, mask=None, adj=None, box=None):
    """Ranks of rows `rows` of every graph against all nodes, as the kernels compute them -> [B, R, N] in x's type.
    x [B, N, C] (float32 or float64), mask [B, N] bool, adj [N, N] or [B, N, N] bool, box [B, C] lengths (0 / inf: the
    axis is not periodic).  Periodic axes need |x_i - x_j| < 2 L, so that the minimum image is one exact subtraction
    (coordinates in [0, L): rint(r / L) is -1, 0 or 1 and r - n L is exact by Sterbenz, like the kernel's fma)."""
    T = x.dtype.type
    b, n, c = x.shape
    rows = np.asarray(rows)
    d = np.zeros((b, len(rows), n), T)
    with np.errstate(invalid="ignore", over="ignore"):
        for a in range(c):
            r = x[:, rows, a][:, :, None] - x[:, None, :, a]
            if box is not None:
                L = np.asarray(box, T)[:, a]
                per = (L > 0) & np.isfinite(L)
                Lp = np.where(per, L, T(0)).astype(T)[:, None, None]
                inv = np.where(per, T(1) / np.where(per, L, T(1)), T(0)).astype(T)[:, None, None]
                r = r - Lp * np.rint(r * inv)
            d = d + r * r
    assert d.dtype == T
    if mask is not None:
        mask = np.asarray(mask, bool)
        d = np.where(mask[:, rows, None] & mask[:, None, :], d, T(1e5))
    if adj is not None:
        a = np.broadcast_to(np.asarray(adj, bool), (b, n, n))[:, rows]
        eye = rows[:, None] == np.arange(n)[None, :]
        d = np.where(eye[None], T(-1), np.where(a, T(0), d))
    return d.astype(T)


def ref_select(x, k, valid_radius, rows=None, mask=None, adj=None, box=None, chunk=256):
    """-> (idx [B, R, k] int64, ok [B, R, k] bool) for rows `rows` (all rows if None)."""
    T = x.dtype.type
    rows = np.arange(x.shape[1]) if rows is None else np.asarray(rows)
    idx, ok = [], []
    for s in range(0, len(rows), chunk):
        d = ranks(x, rows[s:s + chunk], mask, adj, box)
        o = np.argsort(d, axis=-1, kind="stable")[..., :k]
        v = np.take_along_axis(d, o, axis=-1)
        idx.append(o)
        ok.append(v <= T(valid_radius))
    return np.concatenate(idx, 1), np.concatenate(ok, 1)


# ------------------------------------------------------------------ the case table

def _case(B, N, C, k, dt=F32, coords="rand", mask=None, adj=None, vr=math.inf, nonfinite=None, rows=None):
    return dict(B=B, N=N, C=C, k=k, dt=dt, coords=coords, mask=mask, adj=adj, vr=vr, nonfinite=nonfinite, rows=rows)


CASES = {
    # ---- warp select: the cases of the former test_gpu_parity.py::test_knn_select_kernel (dyadic coordinates)
    "w_k1_n5_f64":        _case(2, 5, 3, 1, F64, "dyadic", vr=1.0),
    "w_k8_n300_mask":     _case(2, 300, 3, 8, F32, "dyadic", mask="rand", vr=1.0),
    "w_k32_n1000_f64":    _case(2, 1000, 3, 32, F64, "dyadic", vr=1.0),
    "w_k7_n64_adj_mask":  _case(2, 64, 3, 7, F32, "dyadic", mask="rand", adj="chain", vr=1.0),
    "s_k40_n333_mask":    _case(2, 333, 3, 40, F64, "dyadic", mask="rand", vr=1.0),
    "s_k64_n64":          _case(2, 64, 3, 64, F32, "dyadic", vr=1.0),
    # k = N <= 32; k = 2 / 16 / 31 / 32 across 1, 2 and 3 staging passes; N % 64 = 1, 63, 0, 1
    "w_kN_n17":           _case(3, 17, 3, 17),
    "w_kN_n32_c2_f64":    _case(2, 32, 2, 32, F64),
    "w_k2_n1025":         _case(2, 1025, 3, 2),
    "w_k31_n1023_c1":     _case(2, 1023, 1, 31),
    "w_k32_n1024_f64":    _case(2, 1024, 3, 32, F64),
    "w_k16_n2049_c5":     _case(2, 2049, 5, 16),
    # partial groups: N % 64 = 31 and 33 (and partial last CTAs of 8 warps)
    "w_k31_n95_c4":       _case(2, 95, 4, 31),
    "w_k16_n97_c8_f64":   _case(2, 97, 8, 16, F64),
    "w_k16_n300_c8":      _case(2, 300, 8, 16, F32),
    "w_k8_n200_c4_f64":   _case(2, 200, 4, 8, F64),
    # 8 / 16 warps on both sides of the switch (B = 1: 263 / 264 CTAs of 16 rows), and BASELINE c4 (B = 8, N = 4096)
    "w_8w_n4208":         _case(1, 4208, 3, 16, rows="sample"),
    "w_16w_n4209":        _case(1, 4209, 3, 16, rows="sample"),
    "w_16w_n4209_f64":    _case(1, 4209, 3, 32, F64, rows="sample"),
    "w_16w_b8_n4096":     _case(8, 4096, 3, 32, rows="sample"),
    "w_16w_c8_f64":       _case(2, 2112, 8, 32, F64, rows="sample"),       # 78,912 B of dynamic shared memory
    "w_16w_c2_n2113":     _case(2, 2113, 2, 8, rows="sample"),
    # ---- candidate orders
    "o_line_f32":         _case(1, 2100, 3, 32, F32, "line", rows="sample"),   # last rows: farthest first; first rows: nearest
    "o_line_f64":         _case(1, 1100, 1, 32, F64, "line"),
    "o_line_16w":         _case(2, 2200, 3, 31, F32, "line", rows="sample"),
    "o_coincident":       _case(2, 700, 3, 32, F32, "zero"),
    "o_coincident_sort":  _case(1, 300, 3, 40, F64, "zero"),
    "o_lattice":          _case(2, 1500, 3, 32, F32, "lattice", vr="rank", rows="sample"),
    "o_lattice_c2_f64":   _case(2, 600, 2, 16, F64, "lattice", vr=0.0),
    "o_one_valid":        _case(2, 300, 3, 16, F32, mask="one", vr=1.0),
    "o_no_valid":         _case(2, 300, 3, 16, F64, mask="none", vr=1.0),
    "o_one_valid_sort":   _case(2, 100, 3, 40, F32, mask="one", vr=1.0),
    "o_no_valid_sort":    _case(2, 100, 2, 64, F64, mask="none", vr=1e5),
    # ---- mask, adjacency, radius
    "a_batched_mask":     _case(2, 200, 3, 16, F32, mask="rand", adj="batched", vr=0.5),
    "a_batched":          _case(2, 200, 5, 16, F64, adj="batched", vr=0.0),
    "a_chain_mask":       _case(2, 150, 3, 8, F64, mask="rand", adj="chain", vr=0.0),
    "a_chain":            _case(2, 150, 3, 8, F32, adj="chain"),
    "a_batched_mask_sort": _case(2, 257, 3, 40, F32, mask="rand", adj="batched", vr=0.0),
    "a_chain_sort":       _case(1, 65, 4, 64, F64, adj="chain", vr=1.0),
    "r_rank":             _case(2, 500, 3, 32, F32, mask="rand", vr="rank"),
    "r_rank_f64":         _case(2, 500, 3, 32, F64, vr="rank"),
    "r_zero":             _case(2, 500, 3, 16, F32, vr=0.0),
    "r_inf_mask":         _case(2, 500, 3, 16, F64, mask="rand", vr=math.inf),
    "r_rank_sort":        _case(2, 300, 3, 64, F32, mask="rand", vr="rank"),
    # ---- block sort: k = 33 / 64 / N around the steps of Npad (33 -> 64, 64, 65 -> 128, 256, 257 -> 512, 1000, 4097)
    "s_n33_k33":          _case(2, 33, 3, 33, F32),
    "s_n64_k33_f64":      _case(2, 64, 3, 33, F64),
    "s_n64_k64":          _case(2, 64, 2, 64, F32),
    "s_n65_k64_f64":      _case(2, 65, 3, 64, F64),
    "s_n65_kN":           _case(2, 65, 8, 65, F32),
    "s_n65_k33_mask":     _case(2, 65, 5, 33, F32, "lattice", mask="rand", vr=2.0),
    "s_n256_k64_f64":     _case(2, 256, 2, 64, F64, "line"),
    "s_n257_k33_c1":      _case(2, 257, 1, 33, F32, "lattice", vr="rank"),
    "s_n1000_k64_zero":   _case(1, 1000, 3, 64, F32, "zero"),
    "s_n4097_k33_f64":    _case(1, 4097, 8, 33, F64, rows="sample"),
    "s_n256_k33":         _case(2, 256, 3, 33, F32, mask="rand", vr=1.0),
    "s_n256_kN_f64":      _case(1, 256, 3, 256, F64),
    "s_n257_k64":         _case(2, 257, 1, 64, F32),
    "s_n257_kN_f64":      _case(1, 257, 3, 257, F64, "lattice"),
    "s_n1000_k33_f64":    _case(2, 1000, 3, 33, F64, mask="rand", vr="rank"),
    "s_n1000_kN":         _case(1, 1000, 3, 1000, F32, "lattice"),
    "s_n4097_k64":        _case(1, 4097, 3, 64, F32, rows="sample"),
    "s_n4097_kN_f64":     _case(1, 4097, 3, 4097, F64, rows="sample"),
    # the largest sort (Npad = 16384: 128 KiB fp32, 192 KiB fp64)
    "s_n16384_f32":       _case(1, 16384, 3, 33, F32, rows="sample"),
    "s_n16384_f64":       _case(1, 16384, 3, 40, F64, rows="sample"),
    # ---- non-finite coordinates: NaN and +-inf on query nodes and candidates
    "nf_warp_nan":        _case(2, 300, 3, 16, F32, nonfinite="nan"),
    "nf_warp_inf_f64":    _case(2, 300, 3, 16, F64, nonfinite="inf"),
    "nf_warp_mix_mask":   _case(2, 300, 3, 32, F32, mask="rand", vr=1.0, nonfinite="mix"),
    "nf_warp_c5_mix":     _case(2, 100, 5, 31, F64, nonfinite="mix"),
    "nf_warp_16w_nan":    _case(4, 2100, 3, 32, F32, nonfinite="mix", rows="sample"),
    "nf_warp_kN":         _case(1, 20, 3, 20, F32, nonfinite="mix"),
    "nf_warp_adj":        _case(2, 100, 3, 8, F32, adj="chain", nonfinite="mix"),
    "nf_sort_nan":        _case(2, 300, 3, 40, F32, nonfinite="nan"),
    "nf_sort_mix_mask":   _case(2, 257, 3, 64, F64, mask="rand", vr="rank", nonfinite="mix"),
    "nf_sort_kN":         _case(1, 70, 2, 70, F32, nonfinite="mix"),
}


def make_inputs(spec, seed):
    """-> (x [B, N, C] numpy of the case's type, mask or None, adj or None)."""
    rs = np.random.RandomState(seed)
    B, N, Cd, T = spec["B"], spec["N"], spec["C"], NP_T[spec["dt"]]
    kind = spec["coords"]
    if kind == "rand":
        x = rs.standard_normal((B, N, Cd)) * (N ** (1.0 / Cd))
    elif kind == "dyadic":                     # squared distances exact in fp32: frequent exact ties
        x = np.round(rs.standard_normal((B, N, Cd)) * 8) / 8
    elif kind == "line":                       # x_j = j on axis 0: row N-1 sees its candidates farthest first, row 0 nearest first
        x = np.zeros((B, N, Cd))
        x[:, :, 0] = np.arange(N)
    elif kind == "zero":
        x = np.zeros((B, N, Cd))
    elif kind == "lattice":
        x = rs.randint(0, 4, (B, N, Cd)).astype(np.float64)
    x = x.astype(T)
    nf = spec["nonfinite"]
    if nf:
        pts = []
        if nf in ("nan", "mix"):
            pts += [(0, 0, np.nan), (N // 2, Cd - 1, np.nan)]
        if nf in ("inf", "mix"):
            pts += [(min(5, N - 1), 0, np.inf), (N - 1, 0, np.inf), (N // 3, Cd - 1, -np.inf)]
        for j, a, v in pts:
            x[:, j, a] = v
    m = spec["mask"]
    mask = None
    if m == "rand":
        mask = rs.uniform(size=(B, N)) < 0.85
    elif m == "one":
        mask = np.zeros((B, N), bool)
        mask[:, N // 2] = True
    elif m == "none":
        mask = np.zeros((B, N), bool)
    adj = None
    if spec["adj"] == "chain":
        adj = cases.chain_adjacency(N, True)
    elif spec["adj"] == "batched":
        adj = rs.uniform(size=(B, N, N)) < 0.05
        adj = adj | adj.transpose(0, 2, 1)
    return x, mask, adj


def check_rows(spec, x):
    N = spec["N"]
    if spec["rows"] != "sample":
        return np.arange(N)
    rs = np.random.RandomState(N)
    r = set(range(min(N, 40))) | set(range(max(0, N - 40), N)) | set(rs.randint(0, N, 48).tolist())
    r |= {j for j in range(15, N, 16 * 37) for j in (j, j + 1)}                     # CTA edges through the graph
    r |= set(np.nonzero(~np.isfinite(x).all(-1).any(0))[0].tolist())               # non-finite nodes
    return np.array(sorted(j for j in r if j < N))


def resolve_vr(spec, x, mask, adj):
    """valid_radius "rank": a rank that occurs in row 0 (its k//2-th smallest finite one), so that `<=` meets equality."""
    if spec["vr"] != "rank":
        return float(spec["vr"])
    d = ranks(x, [0], mask, adj)[0, 0]
    d = np.sort(d[np.isfinite(d)])
    return float(d[min(spec["k"] // 2, len(d) - 1)])


# ------------------------------------------------------------------ CPU: the reference and the table


def test_reference_equals_oracle_on_dyadic_coordinates():
    """On a 1/8 grid every rank is exact, so the reference must reproduce the oracle's selection."""
    from oracle import egnn_oracle as O
    rs = np.random.RandomState(3)
    for B, N, Cd, k, masked, adj_kind, vr in [(2, 50, 3, 7, False, None, 1.0), (2, 64, 8, 33, True, None, 0.5),
                                              (3, 40, 2, 40, True, "chain", 0.0), (2, 45, 5, 9, False, "batched", 2.0),
                                              (1, 30, 1, 30, True, "batched", math.inf)]:
        for T in (np.float32, np.float64):
            x = (np.round(rs.standard_normal((B, N, Cd)) * 8) / 8).astype(T)
            mask = rs.uniform(size=(B, N)) < 0.8 if masked else None
            adj = cases.chain_adjacency(N, True) if adj_kind == "chain" else \
                (rs.uniform(size=(B, N, N)) < 0.1 if adj_kind == "batched" else None)
            cfg = O.layer_cfg(dim=4, num_nearest_neighbors=k, valid_radius=vr)
            want_idx, want_ok, _ = O.neighbour_selection(cfg, x, mask, adj)
            idx, ok = ref_select(x, k, vr, mask=mask, adj=adj)
            np.testing.assert_array_equal(idx, want_idx)
            np.testing.assert_array_equal(ok, want_ok)


def test_reference_orders_non_finite_like_a_stable_torch_sort():
    """NaN ranks (NaN coordinates, inf - inf) go last, +inf before them, ties to the lower index: torch.sort(stable=True)."""
    rs = np.random.RandomState(4)
    for T, tt in ((np.float32, torch.float32), (np.float64, torch.float64)):
        x = rs.randint(0, 3, (2, 60, 3)).astype(T)
        x[:, 3, 0] = np.nan
        x[:, 7, 1] = np.inf
        x[:, 8, 1] = np.inf
        x[:, 11, 2] = -np.inf
        x[1, 20, :] = np.nan
        d = ranks(x, np.arange(60))
        assert np.isnan(d[:, :, 3]).all() and np.isnan(d[:, 7, 8]).all() and np.isposinf(d[:, 7, 11]).all()
        want = torch.sort(torch.from_numpy(d).to(tt), dim=-1, stable=True).indices.numpy()
        idx, ok = ref_select(x, 60, math.inf)
        np.testing.assert_array_equal(idx, want)
        np.testing.assert_array_equal(ok, ~np.isnan(np.take_along_axis(d, idx, -1)))


def test_table_covers_every_boundary():
    geo = {name: LG.launch_select(s["B"], s["N"], s["C"], s["k"], 8 if s["dt"] == F64 else 4) for name, s in CASES.items()}
    warp = {n: g for n, g in geo.items() if g["kernel"] == "warp"}
    sort = {n: g for n, g in geo.items() if g["kernel"] == "sort"}
    assert {g["warps"] for g in warp.values()} == {8, 16}
    # both sides of the 8 / 16-warp switch at B = 1
    assert geo["w_8w_n4208"]["warps"] == 8 and geo["w_16w_n4209"]["warps"] == 16
    assert geo["w_16w_b8_n4096"]["warps"] == 16
    assert {g["passes"] for g in warp.values()} >= {1, 2, 3}
    assert {s["N"] for s in CASES.values()} >= {1023, 1024, 1025, 2049}
    assert {g["tail64"] for g in warp.values()} >= {0, 1, 31, 33, 63}
    assert any(g["last_cta_rows"] < g["warps"] for g in warp.values())
    assert any(g["last_cta_rows"] < g["warps"] and g["warps"] == 16 for g in warp.values())
    ks = {CASES[n]["k"] for n in warp}
    assert ks >= {1, 2, 16, 31, 32}
    assert any(CASES[n]["k"] == CASES[n]["N"] for n in warp)
    for dt in (F32, F64):
        assert {CASES[n]["C"] for n in warp if CASES[n]["dt"] == dt} >= {1, 2, 3, 4, 5, 8}
        assert {g["cdim"] for n, g in warp.items() if CASES[n]["dt"] == dt} == {0, 3}
        assert any(g["warps"] == 16 and g["cdim"] == 0 for n, g in warp.items() if CASES[n]["dt"] == dt)
    assert {CASES[n]["C"] for n in warp} >= {1, 2, 3, 4, 5, 8}
    assert max(g["smem"] for g in warp.values()) == 78912                            # fp64, C = 8, 16 warps
    # block sort: k = 33 / 64 / N at every listed N, the size limit in both types
    pairs = {(CASES[n]["N"], CASES[n]["k"]) for n in sort}
    for N in (33, 64, 65, 256, 257, 1000, 4097):
        want = {k for k in (33, 64, N) if k <= N}
        assert want <= {k for n, k in pairs if n == N}, N
    assert {g["npad"] for g in sort.values()} >= {64, 128, 256, 512, 1024, 8192, 16384}
    assert all(g["supported"] for g in sort.values())
    assert {CASES[n]["dt"] for n in sort if CASES[n]["N"] == 16384} == {F32, F64}
    assert not LG.launch_select(1, 16385, 3, 33, 4)["supported"] and not LG.launch_select(1, 16385, 3, 33, 8)["supported"]
    # inputs
    coords = {s["coords"] for s in CASES.values()}
    assert coords >= {"rand", "dyadic", "line", "zero", "lattice"}
    assert {s["mask"] for s in CASES.values()} >= {None, "rand", "one", "none"}
    for kern in (warp, sort):
        adj = {(CASES[n]["adj"], CASES[n]["mask"] is not None) for n in kern if CASES[n]["adj"]}
        assert {a for a, _ in adj} == {"chain", "batched"} and {m for _, m in adj} == {False, True}
        assert {"rank", 0.0, math.inf} <= {CASES[n]["vr"] for n in kern} | {math.inf}
        nf = {(CASES[n]["nonfinite"], CASES[n]["mask"] is not None) for n in kern if CASES[n]["nonfinite"]}
        assert {m for _, m in nf} == {False, True} and {"nan", "mix"} & {v for v, _ in nf}
    assert {CASES[n]["vr"] for n in warp} >= {"rank", 0.0, math.inf}
    assert any(g["warps"] == 16 for n, g in warp.items() if CASES[n]["nonfinite"])


# ------------------------------------------------------------------ GPU: egnn_knn_select vs the reference


def _nat():
    from egnn_pytorch_b200 import _native as nat
    return nat, nat.load()


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def gpu_select(x, k, vr, mask=None, adj=None, with_ok=True):
    """egnn_knn_select on numpy inputs -> (rc, idx [B, N, k], ok [B, N, k] bool or None)."""
    nat, lib = _nat()
    b, n, c = x.shape
    tx = torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
    tm = None if mask is None else torch.from_numpy(np.asarray(mask)).to(DEV, torch.uint8).contiguous()
    ta = None if adj is None else torch.from_numpy(np.ascontiguousarray(adj)).to(DEV, torch.uint8).contiguous()
    idx = torch.full((b, n, k), -7, dtype=torch.int32, device=DEV)
    ok = torch.full((b, n, k), 7, dtype=torch.uint8, device=DEV) if with_ok else None
    rc = lib.egnn_knn_select(nat.DTYPE_F64 if x.dtype == np.float64 else nat.DTYPE_F32, b, n, c, k, _p(tx), _p(tm), _p(ta),
                             1 if adj is not None and np.ndim(adj) == 3 else 0, float(vr), _p(idx), _p(ok),
                             C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, idx.cpu().numpy(), None if ok is None else ok.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_select_matches_exact_reference(name):
    spec = CASES[name]
    x, mask, adj = make_inputs(spec, seed=sum(map(ord, name)))
    k, N = spec["k"], spec["N"]
    vr = resolve_vr(spec, x, mask, adj)
    rows = check_rows(spec, x)
    rc, idx, ok = gpu_select(x, k, vr, mask, adj)
    assert rc == 0, rc
    # every index is a node of the graph (also in rows not compared below), every ok is 0 / 1
    assert idx.min() >= 0 and idx.max() < N, f"indices outside [0, {N}): {idx.min()}, {idx.max()}"
    assert set(np.unique(ok).tolist()) <= {0, 1}
    want_idx, want_ok = ref_select(x, k, vr, rows, mask, adj)
    got_idx, got_ok = idx[:, rows], ok[:, rows].astype(bool)
    bad = (got_idx != want_idx).any(-1) | (got_ok != want_ok).any(-1)
    if bad.any():
        g, r = np.argwhere(bad)[0]
        pytest.fail(f"{name}: {int(bad.sum())} of {bad.size} rows differ; graph {g} row {rows[r]}:\n"
                    f"  got  {got_idx[g, r].tolist()} ok {got_ok[g, r].astype(int).tolist()}\n"
                    f"  want {want_idx[g, r].tolist()} ok {want_ok[g, r].astype(int).tolist()}")
    if spec["nonfinite"]:
        # rows with at least k finite ranks keep exactly their finite lists, and a NaN rank is never ok
        d = ranks(x, rows, mask, adj)
        got_d = np.take_along_axis(d, got_idx, -1)
        full = np.isfinite(d).sum(-1) >= k
        assert np.isfinite(got_d[full]).all()
        assert not got_ok[np.isnan(got_d)].any()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, F64])
def test_select_without_ok_array(dt):
    spec = _case(2, 1100, 3, 24, dt, mask="rand")
    x, mask, _ = make_inputs(spec, seed=11)
    rc, idx, ok = gpu_select(x, 24, 1.0, mask, with_ok=False)
    assert rc == 0 and ok is None
    want_idx, _ = ref_select(x, 24, 1.0, mask=mask)
    np.testing.assert_array_equal(idx, want_idx)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, F64])
def test_sort_beyond_its_size_limit_is_rejected(dt):
    """N = 16385 needs Npad = 32768, beyond the sort's shared memory: EGNN_ERR_UNSUPPORTED, nothing written."""
    nat, _ = _nat()
    x = np.zeros((1, 16385, 3), NP_T[dt])
    rc, idx, ok = gpu_select(x, 33, math.inf)
    assert rc == nat.ERR_UNSUPPORTED
    assert (idx == -7).all() and (ok == 7).all()


@pytest.mark.gpu
def test_layer_with_k_above_32_beyond_the_sort_limit_raises_a_clear_error():
    from egnn_pytorch_b200 import EGNN
    torch.manual_seed(0)
    n = 16385
    for dtype in (torch.float32, torch.bfloat16):
        layer = EGNN(dim=16, num_nearest_neighbors=33).to(DEV).to(dtype).eval()
        f = torch.randn(1, n, 16, device=DEV, dtype=dtype)
        x = torch.randn(1, n, 3, device=DEV, dtype=dtype)
        with torch.no_grad(), pytest.raises(RuntimeError, match=r"num_nearest_neighbors=33 > 32 .* at most N=16384"):
            layer(f, x)
    # ... and at the limit it runs
    n = 16384
    layer = EGNN(dim=16, num_nearest_neighbors=33).to(DEV).eval()
    with torch.no_grad():
        out = layer(torch.randn(1, n, 16, device=DEV), torch.randn(1, n, 3, device=DEV))
    assert torch.isfinite(out[0]).all()


# ------------------------------------------------------------------ periodic boxes, through the layer

PBC_CASES = {
    # name: (B, N, C, k, box kind, mask + radius)
    "pbc_warp8_c3":       (2, 300, 3, 16, "cubic", False),
    "pbc_warp16_passes":  (2, 2200, 3, 32, "per_graph", False),         # 16 warps, 3 staging passes
    "pbc_warp_generic":   (2, 500, 2, 8, "slab", False),                 # C = 2: one axis periodic, one L = inf
    "pbc_warp16_c5":      (2, 2112, 5, 31, "mixed", False),
    "pbc_sort":           (2, 300, 3, 40, "per_graph", False),
    "pbc_sort_c4":        (1, 257, 4, 64, "mixed", False),
    "pbc_warp_mask_r":    (2, 700, 3, 16, "cubic", True),                # all-pairs path forced (no cell grid)
    "pbc_sort_mask_r":    (2, 200, 3, 33, "per_graph", True),
}


def _box(kind, B, Cd, rs):
    if kind == "cubic":
        return np.full((B, Cd), 7.0)
    if kind == "per_graph":
        return rs.uniform(5.0, 11.0, (B, Cd)).round(3)
    if kind == "slab":
        return np.array([[6.5] + [np.inf] * (Cd - 1)] * B)
    box = rs.uniform(5.0, 11.0, (B, Cd)).round(3)                       # mixed: 0 and inf axes, different per graph
    box[0, 0], box[-1, -1] = 0.0, np.inf
    return box


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PBC_CASES))
def test_periodic_select_through_the_layer(name, monkeypatch):
    """The layer's own periodic select equals the reference's periodic lists: the same layer run with `neighbors=` set to
    them (ok = 0 slots as -1) gives bit-identical outputs."""
    from egnn_pytorch_b200 import EGNN
    B, N, Cd, k, kind, masked = PBC_CASES[name]
    rs = np.random.RandomState(sum(map(ord, name)))
    box = _box(kind, B, Cd, rs)
    per = (box > 0) & np.isfinite(box)
    span = np.where(per, box, 8.0)
    x = (rs.uniform(size=(B, N, Cd)) * span[:, None, :]).astype(np.float32)
    x = np.where(per[:, None, :] & (x >= box[:, None, :].astype(np.float32)), np.float32(0), x)   # keep [0, L)
    vr = 4.0 if masked else math.inf
    mask = rs.uniform(size=(B, N)) < 0.85 if masked else None
    if masked:
        monkeypatch.setenv("EGNN_B200_CELL_SELECT_MIN_N", str(2 ** 40))
    torch.manual_seed(1)
    layer = EGNN(dim=8, num_nearest_neighbors=k, valid_radius=vr).to(DEV).eval()
    f = torch.randn(B, N, 8, device=DEV)
    tx = torch.from_numpy(x).to(DEV)
    tb = torch.from_numpy(box).to(DEV, torch.float32)
    tm = None if mask is None else torch.from_numpy(mask).to(DEV)
    idx, ok = ref_select(x, k, vr, mask=mask, box=box.astype(np.float32))
    nbr = torch.from_numpy(np.where(ok, idx, -1)).to(DEV)
    with torch.no_grad():
        f1, x1 = layer(f, tx, mask=tm, box=tb)
        f2, x2 = layer(f, tx, mask=tm, box=tb, neighbors=nbr)
    assert torch.equal(f1, f2) and torch.equal(x1, x2), \
        f"{name}: outputs differ in {int(((f1 != f2).any(-1) | (x1 != x2).any(-1)).sum())} rows"


# ------------------------------------------------------------------ non-finite coordinates in a layer (after the select)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [8, 40])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_layer_with_a_nan_node_keeps_every_other_row(dtype, k):
    """One NaN node: the layer runs, and every row whose list does not hold that node equals the layer run on the
    reference lists (which rank it last, as NaN)."""
    from egnn_pytorch_b200 import EGNN
    B, N, nan_node = 2, 300, 37
    torch.manual_seed(2)
    layer = EGNN(dim=32, num_nearest_neighbors=k).to(DEV).to(dtype).eval()
    f = torch.randn(B, N, 32, device=DEV, dtype=dtype)
    x = torch.randn(B, N, 3, device=DEV, dtype=dtype) * 3
    x[1, nan_node, 1] = float("nan")
    idx, ok = ref_select(x.float().cpu().numpy(), k, math.inf)
    nbr = torch.from_numpy(np.where(ok, idx, -1)).to(DEV)
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("ignore")               # k > 32 in bf16: the fp32 kernels run (a warning says so)
        f1, x1 = layer(f, x)
        f2, x2 = layer(f, x, neighbors=nbr)
        torch.cuda.synchronize()
    assert ok[1, :, :].sum() > 0 and not ok[1, nan_node].any()
    holds = (idx == nan_node) & ok
    holds[0] = False                                  # graph 0 has no NaN node
    keep = torch.from_numpy(~holds.any(-1)).to(DEV)
    keep[1, nan_node] = False
    assert int(keep.sum()) == B * N - 1               # ranked last and never ok: no other row holds the NaN node
    assert torch.equal(f1[keep], f2[keep]) and torch.equal(x1[keep], x2[keep])
    assert torch.isfinite(f1[keep]).all() and torch.isfinite(x1[keep]).all()


# ------------------------------------------------------------------ the adjacency row scan (adj_neighbors_kernel)

# (B, N, k, batched, with ok): N % 4 == 0 takes the 4-byte path, 128 columns per trip; 70 and 129 the byte path
ADJ_CASES = {
    "adj_n64_k6":            (2, 64, 6, True, True),
    "adj_n64_kN_unbatched":  (2, 64, 64, False, False),
    "adj_n96_k9":            (2, 96, 9, True, False),
    "adj_n132_k67":          (2, 132, 67, False, True),
    "adj_n4096_k200":        (1, 4096, 200, True, True),
    "adj_n4096_k4096":       (1, 4096, 4096, False, False),
    "adj_n70_k9":            (2, 70, 9, True, False),                    # the shape of test_gpu_list_cache's own check
    "adj_n70_k70_unbatched": (2, 70, 70, False, True),
    "adj_n129_k33":          (2, 129, 33, True, True),
    "adj_n129_k5_unbatched": (3, 129, 5, False, False),
}


def ref_adj_lists(adj, B, N, k, with_ok):
    """Slot 0 = the node, then its adjacent nodes ascending, truncated at k; unused slots: the node with ok = 0, or -1."""
    a = np.broadcast_to(adj, (B, N, N))
    idx = np.empty((B, N, k), np.int64)
    ok = np.zeros((B, N, k), bool)
    for b in range(B):
        for i in range(N):
            nb = [i] + [j for j in np.nonzero(a[b, i])[0].tolist() if j != i]
            nb = nb[:k]
            idx[b, i, :len(nb)] = nb
            ok[b, i, :len(nb)] = True
            idx[b, i, len(nb):] = i if with_ok else -1
    return idx, ok


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ADJ_CASES))
def test_adjacency_row_scan_matches_reference(name):
    nat, lib = _nat()
    B, N, k, batched, with_ok = ADJ_CASES[name]
    rs = np.random.RandomState(sum(map(ord, name)))
    # rows of every density: empty, sparse, and denser than k (cut inside a lane's word and inside a 128-column trip)
    shape = (B, N, N) if batched else (N, N)
    dens = rs.choice([0.0, 0.02, 0.3, 0.9], size=shape[:-1])
    adj = rs.uniform(size=shape) < dens[..., None]
    adj[..., 0, :] = False                       # an empty row (its diagonal set: the node is not its own neighbour)
    adj[..., 0, 0] = True
    adj[..., 1, :] = True                        # a full row
    ta = torch.from_numpy(adj).to(DEV, torch.uint8).contiguous()
    idx = torch.full((B, N, k), -7, dtype=torch.int32, device=DEV)
    ok = torch.full((B, N, k), 7, dtype=torch.uint8, device=DEV) if with_ok else None
    rc = lib.egnn_adj_neighbors(B, N, k, _p(ta), 1 if batched else 0, _p(idx), _p(ok),
                                C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, nat.strerror(rc)
    torch.cuda.synchronize()
    want_idx, want_ok = ref_adj_lists(adj, B, N, k, with_ok)
    got = idx.cpu().numpy()
    bad = (got != want_idx).any(-1)
    assert not bad.any(), f"{int(bad.sum())} rows differ, first {np.argwhere(bad)[0].tolist()}"
    if with_ok:
        np.testing.assert_array_equal(ok.cpu().numpy().astype(bool), want_ok)
    counts = np.broadcast_to(adj, (B, N, N)).sum(-1) - np.diagonal(np.broadcast_to(adj, (B, N, N)), axis1=1, axis2=2) + 1
    assert (counts > k).any() or k == N
    assert (counts == 1).any()
