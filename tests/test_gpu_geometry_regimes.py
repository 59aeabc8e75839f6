"""The edge kernels at physical coordinate scales and on degenerate geometry, against the float64 reference.

The rest of the suite draws coordinates from unit normals, a unit box or lattice coordinates within two box lengths of
the origin: pair distances are O(1), nodes sit near the origin, no two distinct nodes coincide and CoorsNorm's
max(|rel|, 1e-8) clamps only the self pair.  Real inputs differ.  Each regime below is a seeded generator whose stated
margin is pinned on the CPU (test_regime_*):
  angstrom      molecule-like blobs: a 1.3 A lattice thinned to 40 % and jittered by +-0.12 A (nearest neighbours
                ~1.0-1.6 A, radius ~1.1 N^(1/3) A), centred at (52.3, -37.9, 18.4); d^2 from ~1 to several 10^2 A^2,
                which goes raw into edge_mlp.0 and the fourier features.  kNN inputs tie-free at the k-th rank by >= 1e-5
                relative, valid_radius >= 1e-5 relative from every pair's d^2.  One case holds two such molecules
                ~25 A apart (d^2 to ~1.5e3) on a 1/16 A grid, where fp32 forms d^2 exactly, with edge_mlp.0's distance
                column zeroed, so that the fourier features alone carry the geometry
  far           unit normals translated by 2^10 .. 2^13 per axis (fp32 values, so x_i - x_j is exact in fp32)
  nano          unit normals scaled by 1e-4 and 1e-6 (CoorsNorm's 1/|rel| up to ~1e6)
  eps_straddle  unit normals plus planted pairs at |rel| in {0, 2e-9, 5e-9, 2e-8, 5e-8, 1e-7}, >= 10 % from CoorsNorm's
                1e-8 in fp32 and fp64
  coincident    groups of 2-4 distinct nodes at one position, and a fifth of the nodes (padding) stacked at the origin,
                masked and unmasked
  unwrapped     periodic inputs moved by up to +-64 box lengths, box and triclinic cell, every wrap decision >= 1e-3 L
                from 1/2
Paths: fp64 / fp32 SIMT dense (small-node stage dim <= 64, GEMM stage dim > 64 over several 64-row tiles) and neighbour
lists (k <= 32 and k > 32); bf16 tensor cores dense (lean and generic) and neighbour lists (lean and generic, k <= 32
and k > 32).  test_table_covers_every_path_and_regime holds that, through tests/launch_geometry.py; every GPU run
checks the module's `last_path`.  Parameters use Xavier init; all coordinates, features and parameters are fp32 values
(bf16 for the bf16 path), so fp64 and fp32 runs share one float64 reference.  Layers that select their own lists are
compared on test_gpu_knn_select.ref_select's lists (bit for bit the kernels' ranking in the coordinates' type).

References: torch_reference.layer / layer_grads_chunked in float64 (fp64, fp32), tc_reference.tc_layer_forward
(bf16: rounds where the kernels round), test_lattice_grad's restatement of the lattice gradient, and the all-pairs
select for the cell-grid selects (lists bit-equal).

Gates (`TOL`):
  forward   per output, max |error| / max |reference| for the features and max |error| / max |update| for the
            coordinates, where the coordinate error first drops 2 ulp(max |x|) of the coordinates' type (the rounding of
            x + update at a large offset)
  backward  per gradient max |error| / max |reference| (input gradients minus the cotangent, which passes unchanged);
            node-indexed gradients also per row, against the row's own max with a floor of 1e-3 of the median row.
            Where CoorsNorm's 1/eps branch runs the reference's ~1e8 gradient must be matched there, finite and nonzero,
            and no gradient may be non-finite where the reference's is finite
  lattice   test_lattice_grad.check64 / check32 (fp64 against scale; fp32 within 4x the fp32 restatement's error)
Measured on an H100 80GB HBM3 (700 W power limit): the worst value of each gate over its cases is listed beside TOL;
the whole file runs in about 21 s with a peak of 0.7 GiB of device memory."""
import contextlib
import functools
import time
import zlib

import numpy as np
import pytest
import torch

import cases
import launch_geometry as LG
import tc_reference as T
import test_gpu_knn_grid as KG
import test_gpu_radius_select as RS
import test_gpu_radius_select_wide as RSW
import test_lattice_grad as LGR
import test_periodic as PER
import test_triclinic as TRI
import torch_reference as TR
import util
from test_gpu_knn_select import ref_select

DEV = "cuda"
DT = {"fp64": torch.float64, "fp32": torch.float32, "bf16": torch.bfloat16}
PATH = {"fp64": "fp64-simt", "fp32": "fp32-simt", "bf16": "bf16-tc"}

# (gate, type): bound.  Beside it the worst value measured over the cases (H100 80GB HBM3, 700 W power limit).
TOL = {
    ("feats", "fp64"): 1e-14,    # 7.5e-16  ang_d16_fourier4
    ("coors", "fp64"): 1e-14,    # 7.6e-16  ang_d16_fourier4
    ("feats", "fp32"): 2e-6,     # 4.1e-7   ang_d96_normc
    ("coors", "fp32"): 2e-6,     # 4.5e-7   ang_d16_fourier4 (unwrapped inputs: UNWRAPPED_FP32_COORS)
    ("feats", "bf16"): 1e-2,     # 2.8e-3   ang_k48_normc
    ("coors", "bf16"): 1e-3,     # 3.1e-4   ang_k16_vr
    ("grad", "fp64"): 1e-12,     # 1.4e-13  ang_d16_fourier4 (p.edge_mlp.0.weight)
    ("grad_normc", "fp64"): 1e-7,  # 9.0e-9 eps_k8_normc (in.coors per row; see `grad_tol`)
    ("grad", "fp32"): 5e-4,      # 1.4e-4   unwrapped cell_lists_k10_normc (p.coors_mlp.3.bias); else 6.3e-5
}
# Unwrapped fp32 inputs: x_i - x_j of coordinates 64 lattice lengths out is rounded to fp32 (ulp 3e-5 there) before the
# wrap, which the float64 reference does not do; the coordinate update inherits that rounding.
UNWRAPPED_FP32_COORS = 4e-5    # 1.0e-5   cell_dense_tilt


def grad_tol(case, dt):
    """fp64 with CoorsNorm: the self pair's +-scale / 1e-8 terms (rel = 0) cancel in dL/dx_i, leaving ~1e-8 of their
    1e8 size as noise in the reference and the kernel alike (tests/util.grad_tol)."""
    if dt == "fp64" and case["cfg"]["norm_coors"]:
        return TOL[("grad_normc", dt)]
    return TOL[("grad", dt)]


@pytest.fixture(autouse=True)
def _time_and_peak_memory(request):
    """Prints each test's run time and peak device memory (visible with -s)."""
    if not torch.cuda.is_available():
        yield
        return
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n{request.node.name}: {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def f32(x):
    return util.rounded(np.asarray(x, np.float64), torch.float32)


def ulp(v, cdt):
    """ulp of |v| in the coordinates' type."""
    v = max(float(v), 1e-300)
    return 2.0 ** (np.floor(np.log2(v)) - (52 if cdt == torch.float64 else 23))


# ------------------------------------------------------------------ the regimes


CENTRE = (52.3, -37.9, 18.4)
SPACING, KEEP, JITTER = 1.3, 2.5, 0.12
PAIR_OFFSET = (22.0, 9.0, -6.0)


def angstrom(rs, B, N, pair=False):
    """Lattice points of spacing SPACING nearest the origin, KEEP N of them, N drawn per graph, jittered, centred at
    CENTRE (fp32 values).  `pair`: two blobs of N / 2, the second moved by PAIR_OFFSET (a complex of two molecules,
    d^2 up to ~10^3 across them), on a 1/16 A grid: with |x| < 128 fp32 then forms x_i - x_j and d^2 < 2^14 exactly, so
    the fourier features' arguments are the float64 reference's and only sin / cos themselves can differ."""
    if pair:
        a, b = angstrom(rs, B, N // 2), angstrom(rs, B, N - N // 2)
        return np.round(np.concatenate([a, b + np.asarray(PAIR_OFFSET)], 1) * 16) / 16
    m = int(KEEP * N)
    side = int(np.ceil((6 * m / np.pi) ** (1 / 3) / 2)) + 1
    ax = np.arange(-side, side + 1)
    g = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3) * SPACING
    g = g[np.argsort((g ** 2).sum(-1), kind="stable")[:m]]
    x = np.stack([g[rs.choice(m, N, replace=False)] for _ in range(B)])
    return f32(x + rs.uniform(-JITTER, JITTER, x.shape) + np.asarray(CENTRE))


def far(rs, B, N, offset):
    return f32(rs.standard_normal((B, N, 3)) + np.asarray(offset, np.float64))


def nano(rs, B, N, scale):
    return f32(rs.standard_normal((B, N, 3)) * scale)


EPS_REL = (0.0, 2e-9, 5e-9, 2e-8, 5e-8, 1e-7)


def eps_straddle(rs, B, N):
    """Nodes 2t, 2t+1 (t < 6): a pair |rel| = EPS_REL[t] apart along x, at 2^-12 (t+1, 1, -1), where fp32 resolves
    1e-10."""
    x = rs.standard_normal((B, N, 3))
    for t, v in enumerate(EPS_REL):
        base = 2.0 ** -12 * np.array([t + 1.0, 1.0, -1.0])
        x[:, 2 * t] = base
        x[:, 2 * t + 1] = base + np.array([v, 0.0, 0.0])
    return f32(x)


COINCIDENT_GROUPS = (2, 3, 4, 2, 3)


def coincident(rs, B, N):
    """-> (coordinates, padding mask): groups of COINCIDENT_GROUPS nodes at one position each, the last N // 5 nodes at
    the origin (the padding of the mask)."""
    x = rs.standard_normal((B, N, 3))
    s = 0
    for g in COINCIDENT_GROUPS:
        x[:, s:s + g] = x[:, s:s + 1]
        s += g
    pad = N // 5
    x[:, N - pad:] = 0.0
    return f32(x), np.broadcast_to(np.arange(N) < N - pad, (B, N)).copy()


def unwrapped_box(rs, B, N, L, shift=64):
    return f32(PER.lattice_coors(rs, B, N, len(L), L, shift=shift))


def unwrapped_cell(rs, B, N, cell, shift=64):
    return TRI.cell_coors(rs, B, N, cell, shift=shift, dtype=torch.float32)


def radius_with_margin(x, near, mask=None, lo=0.8, hi=1.25):
    """A valid_radius in [lo, hi] near: the middle of the widest gap between the pairs' d^2 there (float64 d^2 of the
    fp32 coordinates; masked pairs excluded)."""
    d = ((x[:, :, None] - x[:, None]) ** 2).sum(-1)
    if mask is not None:
        d = d[mask[:, :, None] & mask[:, None, :]]
    v = np.unique(d[(d > lo * near) & (d < hi * near)])
    v = np.concatenate([[lo * near], v, [hi * near]])
    i = int(np.argmax(np.diff(v)))
    return float((v[i] + v[i + 1]) / 2)


def radius_margin(x, vr, mask=None):
    d = ((x[:, :, None] - x[:, None]) ** 2).sum(-1)
    if mask is not None:
        d = d[mask[:, :, None] & mask[:, None, :]]
    return float(np.abs(d - vr).min() / vr)


# ------------------------------------------------------------------ forward and backward cases

# name: regime (generator, args), layer cfg, B, N, mask, paths.  `k` in cfg: num_nearest_neighbors (the layer selects);
# valid_radius "margin": radius_with_margin near VR_NEAR.
VR_NEAR = 16.0
CASES = {
    # ---- dense
    "ang_d16_fourier4": (("angstrom",), dict(dim=16, fourier_features=4, soft_edges=True), 1, 600, "none",
                         ("fp64", "fp32")),
    # without the raw distance column (zeroed), so that the fourier features alone carry the geometry: at d^2 ~ 10^3
    # the distance term otherwise dwarfs an error in sin / cos of d^2 / 2^q
    "ang_pair_d16_fourier4_nodist": (("angstrom", "pair"), dict(dim=16, fourier_features=4), 1, 400, "none",
                                     ("fp64", "fp32", "bf16")),
    "ang_d96_normc": (("angstrom",), dict(dim=96, norm_coors=True, coor_weights_clamp_value=2.0, m_pool_method="mean"),
                      2, 300, "padded", ("fp64", "fp32")),
    "ang_d32_fourier2": (("angstrom",), dict(dim=32, fourier_features=2, m_pool_method="mean"), 2, 200, "random",
                         ("bf16",)),
    "ang_d32_lean": (("angstrom",), dict(dim=32, soft_edges=True), 2, 200, "none", ("bf16",)),
    "far_d16_fourier2": (("far", (2.0 ** 10, -2.0 ** 12, 2.0 ** 13)),
                         dict(dim=16, fourier_features=2, norm_coors=True), 2, 200, "none", ("fp64", "fp32", "bf16")),
    "far13_d32_lean": (("far", (2.0 ** 13, 2.0 ** 13, -2.0 ** 13)), dict(dim=32, coor_weights_clamp_value=1.0), 2, 300,
                       "padded", ("fp64", "fp32", "bf16")),
    "nano4_d16_normc": (("nano", 1e-4), dict(dim=16, norm_coors=True), 2, 150, "none", ("fp64", "fp32", "bf16")),
    "nano6_d16_normc_fourier": (("nano", 1e-6), dict(dim=16, norm_coors=True, fourier_features=2), 2, 150, "random",
                                ("fp64", "fp32", "bf16")),
    "eps_d16_normc": (("eps_straddle",), dict(dim=16, norm_coors=True, soft_edges=True), 2, 64, "none",
                      ("fp64", "fp32", "bf16")),
    "coin_masked_normc": (("coincident", True), dict(dim=16, norm_coors=True, m_pool_method="mean"), 2, 80, "none",
                          ("fp64", "fp32", "bf16")),
    "coin_unmasked_normc": (("coincident", False), dict(dim=24, norm_coors=True, coor_weights_clamp_value=0.5), 2, 80,
                            "none", ("fp64", "fp32", "bf16")),
    # ---- neighbour lists
    "ang_k16_vr": (("angstrom",), dict(dim=16, num_nearest_neighbors=16, valid_radius="margin", fourier_features=2),
                   1, 800, "random", ("fp64", "fp32", "bf16")),
    "ang_k48_normc": (("angstrom",), dict(dim=32, num_nearest_neighbors=48, norm_coors=True), 1, 600, "none",
                      ("fp64", "fp32", "bf16")),
    "far_k8": (("far", (2.0 ** 12, 2.0 ** 10, -2.0 ** 11)), dict(dim=16, num_nearest_neighbors=8), 2, 300, "padded",
               ("fp64", "fp32", "bf16")),
    "eps_k8_normc": (("eps_straddle",), dict(dim=16, num_nearest_neighbors=8, norm_coors=True), 2, 64, "none",
                     ("fp64", "fp32", "bf16")),
    "coin_k12_fourier2": (("coincident", False), dict(dim=16, num_nearest_neighbors=12, fourier_features=2,
                                                      m_pool_method="mean"), 2, 100, "none", ("fp64", "fp32", "bf16")),
    "nano6_k40_fourier4": (("nano", 1e-6), dict(dim=16, num_nearest_neighbors=40, norm_coors=True, fourier_features=4),
                           1, 200, "random", ("fp64", "fp32", "bf16")),
}
NO_DISTANCE_COLUMN = {"ang_pair_d16_fourier4_nodist"}
FWD = [(n, dt) for n, c in CASES.items() for dt in c[5]]
GRAD = [n for n, c in CASES.items() if "fp64" in c[5]]


def regime_coors(regime, rs, B, N):
    """-> (coordinates, mask or None) of a regime."""
    kind = regime[0]
    if kind == "angstrom":
        return angstrom(rs, B, N, pair=regime[1:] == ("pair",)), None
    if kind == "far":
        return far(rs, B, N, regime[1]), None
    if kind == "nano":
        return nano(rs, B, N, regime[1]), None
    if kind == "eps_straddle":
        return eps_straddle(rs, B, N), None
    if kind == "coincident":
        x, m = coincident(rs, B, N)
        return x, (m if regime[1] else None)
    raise KeyError(kind)


@functools.lru_cache(maxsize=None)
def build(name):
    """The case (fp32 parameters, features and coordinates), its regime's coordinates and mask, and its valid_radius;
    angstrom kNN inputs are redrawn until tie-free at the k-th rank."""
    regime, cfg, B, N, mask_kind, _ = CASES[name]
    cfg = dict(cfg)
    k = cfg.get("num_nearest_neighbors", 0)
    seed = 3000 + zlib.crc32(name.encode()) % 10 ** 6
    case = cases.build_case(dict(kind="layer", cfg={**cfg, "valid_radius": 1.0} if cfg.get("valid_radius") else cfg,
                                 B=B, N=N, seed=seed, init="xavier", mask=mask_kind))
    mask = case["inputs"].get("mask")
    for attempt in range(20):
        x, m = regime_coors(regime, np.random.RandomState(seed + 101 * attempt), B, N)
        mk = m if m is not None else mask
        if regime[0] != "angstrom" or not k or TR.knn_gap(x, k, mk) >= 1e-5:
            break
    else:
        raise AssertionError(f"{name}: no tie-free draw")
    if cfg.get("valid_radius") == "margin":
        cfg["valid_radius"] = radius_with_margin(x, VR_NEAR, mk)
        case = cases.build_case(dict(kind="layer", cfg=cfg, B=B, N=N, seed=seed, init="xavier", mask=mask_kind))
    case["params"] = {p: f32(v) for p, v in case["params"].items()}
    if name in NO_DISTANCE_COLUMN:
        case["params"]["edge_mlp.0.weight"][:, 2 * cfg["dim"] + 2 * cfg["fourier_features"]] = 0.0
    case["inputs"]["feats"] = f32(case["inputs"]["feats"])
    case["inputs"]["coors"] = x
    case["inputs"]["mask"] = mk
    return case


def bf16_case(name):
    case = build(name)
    c = dict(case, params={p: util.rounded(v, torch.bfloat16) for p, v in case["params"].items()})
    c["inputs"] = dict(case["inputs"], feats=util.rounded(case["inputs"]["feats"], torch.bfloat16))
    return c


@functools.lru_cache(maxsize=None)
def lists(name, cdt_name):
    """The kernels' own lists (idx, ok) in the coordinates' type, or (None, None) for a dense case."""
    case = build(name)
    cfg = case["cfg"]
    if not cfg["num_nearest_neighbors"]:
        return None, None
    x = np.asarray(case["inputs"]["coors"], np.float64 if cdt_name == "fp64" else np.float32)
    return ref_select(x, cfg["num_nearest_neighbors"], cfg["valid_radius"], mask=case["inputs"]["mask"])


def cdt_name(dt):
    return "fp64" if dt == "fp64" else "fp32"


# ------------------------------------------------------------------ CPU: the regimes' margins


def test_regime_angstrom_spacing_radius_offset_and_margins():
    for name in ("ang_d16_fourier4", "ang_k16_vr", "ang_k48_normc", "ang_pair_d16_fourier4_nodist"):
        case = build(name)
        x, N = case["inputs"]["coors"], case["spec"]["N"]
        if CASES[name][0][1:] == ("pair",):                     # each blob on its own, then the d^2 across them
            d2 = ((x[:, :, None] - x[:, None]) ** 2).sum(-1)
            assert d2.max() > 1000.0 and np.abs(x).max() < 128 and (x * 16 == np.round(x * 16)).all(), d2.max()
            r = (x[:, :, None] - x[:, None]).astype(np.float32)              # fp32 forms rel and d^2 exactly
            d32 = r[..., 0] * r[..., 0] + r[..., 1] * r[..., 1] + r[..., 2] * r[..., 2]
            assert np.array_equal(d32.astype(np.float64), d2)
            h = N // 2
            x, N = np.concatenate([x[:, :h], x[:, h:] - np.asarray(PAIR_OFFSET)]), h
        for b in range(x.shape[0]):
            d = np.sqrt(((x[b][:, None] - x[b][None]) ** 2).sum(-1)) + np.diag(np.full(N, np.inf))
            nn = d.min(-1)
            assert nn.min() >= 0.85 and 1.0 <= np.median(nn) <= 1.6, (name, nn.min(), np.median(nn))
            c = x[b].mean(0)
            assert np.abs(c - np.asarray(CENTRE)).max() < 1.0, (name, c)
            radius = np.sqrt(((x[b] - c) ** 2).sum(-1)).max()
            assert 0.9 <= radius / N ** (1 / 3) <= 1.4, (name, radius / N ** (1 / 3))
            d2 = d[np.isfinite(d)] ** 2
            assert d2.min() < 1.5 and d2.max() > (300.0 if N >= 600 else 100.0), (name, d2.min(), d2.max())
        k = case["cfg"]["num_nearest_neighbors"]
        if k:
            assert TR.knn_gap(x, k, case["inputs"]["mask"]) >= 1e-5, name
    case = build("ang_k16_vr")
    vr = case["cfg"]["valid_radius"]
    assert 0.8 * VR_NEAR <= vr <= 1.25 * VR_NEAR
    assert radius_margin(case["inputs"]["coors"], vr, case["inputs"]["mask"]) >= 1e-5


def test_regime_far_differences_are_exact_in_fp32():
    for name in ("far_d16_fourier2", "far13_d32_lean", "far_k8"):
        x = build(name)["inputs"]["coors"]
        off = np.asarray(CASES[name][0][1])
        assert (np.abs(x.mean(1) - off) < 1.0).all()
        assert (np.sign(x) == np.sign(off)).all() and (np.abs(x) >= np.abs(off) / 2).all() and (
            np.abs(x) <= 2 * np.abs(off)).all()                                       # Sterbenz: x_i - x_j exact
        x32 = x.astype(np.float32)
        assert np.array_equal((x32[:, :, None] - x32[:, None]).astype(np.float64), x[:, :, None] - x[:, None])


def test_regime_nano_scales():
    for name, s in (("nano4_d16_normc", 1e-4), ("nano6_d16_normc_fourier", 1e-6), ("nano6_k40_fourier4", 1e-6)):
        x = build(name)["inputs"]["coors"]
        d = np.sqrt(((x[:, :, None] - x[:, None]) ** 2).sum(-1))
        off = d[d > 0]
        assert off.min() > 1e-3 * s and off.max() < 20 * s and off.min() > 1e-8 * 1.1, name


def test_regime_eps_straddle_pairs_are_a_tenth_from_the_clamp_in_fp32_and_fp64():
    for name in ("eps_d16_normc", "eps_k8_normc"):
        x = build(name)["inputs"]["coors"]
        for t, v in enumerate(EPS_REL):
            r64 = x[:, 2 * t + 1] - x[:, 2 * t]
            r32 = x[:, 2 * t + 1].astype(np.float32) - x[:, 2 * t].astype(np.float32)
            n64 = np.sqrt((r64 ** 2).sum(-1))
            n32 = np.sqrt((r32 * r32).sum(-1, dtype=np.float32)).astype(np.float64)
            if v == 0:
                assert (n64 == 0).all() and (n32 == 0).all()
            else:
                for n in (n64, n32):
                    assert (np.abs(n / v - 1) < 0.05).all() and (np.abs(n / 1e-8 - 1) >= 0.1).all(), (name, v, n)
        d = np.sqrt(((x[:, :, None] - x[:, None]) ** 2).sum(-1))
        pairs = {(2 * t, 2 * t + 1) for t in range(len(EPS_REL))}
        small = {(i, j) for b, i, j in np.argwhere(d < 1e-6) if i < j}
        assert small <= pairs                                      # no other distinct pair comes near the clamp


def test_regime_coincident_groups_and_stacked_padding():
    for name in ("coin_masked_normc", "coin_unmasked_normc", "coin_k12_fourier2"):
        case = build(name)
        x, N = case["inputs"]["coors"], case["spec"]["N"]
        s = 0
        for g in COINCIDENT_GROUPS:
            assert (x[:, s:s + g] == x[:, s:s + 1]).all() and (x[:, s] != 0).all()
            s += g
        assert (x[:, N - N // 5:] == 0).all()
        m = case["inputs"]["mask"]
        assert (m is not None) == CASES[name][0][1]
        if m is not None:
            assert (m[:, :N - N // 5]).all() and not m[:, N - N // 5:].any()


def test_regime_unwrapped_half_box_margin_and_shift():
    for name in PERIODIC:
        case, lat, kind = periodic_case(name)
        x = case["inputs"]["coors"]
        if kind == "box":
            assert PER.half_box_margin(x, lat) >= 1e-3, name
            A = np.diag(lat)
        else:
            assert TRI.wrap_margin(x, lat).min() >= 1e-3, name
            A = np.asarray(lat)
        frac = np.abs(x @ np.linalg.inv(A)).max()                  # lattice coordinates: tens of lattice vectors out
        assert 40 < frac <= 65, (name, frac)


# ------------------------------------------------------------------ coverage (tests/launch_geometry.py)


def path_geometry(name, dt):
    regime, cfg, B, N, _, _ = CASES[name]
    k = cfg.get("num_nearest_neighbors", 0)
    lcfg = {**cfg, "valid_radius": 1.0} if cfg.get("valid_radius") else cfg
    if dt == "bf16":
        g = LG.tc_layer("layer", lcfg, B, N, k=k)
        return dict(path=g["kernel"].split(",")[0].replace("<", ":").replace(">", "") + (":wide" if k > 32 else ""),
                    supported=g["supported"])
    g = LG.simt_layer("layer", lcfg, B, N, k=k)
    stage = "gemm" if g["generic_node_gemm"] else "small"
    if not k:
        return dict(path=f"simt:dense:{stage}", row_tiles=LG.ceil_div(B * N, 64), supported=True)
    return dict(path=f"simt:list:{'wide' if k > 32 else 'narrow'}", supported=True)


def test_table_covers_every_path_and_regime():
    geo = {(n, dt): path_geometry(n, dt) for n, dt in FWD}
    assert all(g["supported"] for g in geo.values())
    paths = {g["path"] for g in geo.values()}
    want = {"simt:dense:small", "simt:dense:gemm", "simt:list:narrow", "simt:list:wide", "tc_pair:lean",
            "tc_pair:generic", "tc_knn:LEAN", "tc_knn:GEN", "tc_knn:LEAN:wide", "tc_knn:GEN:wide"}
    assert paths >= want, sorted(want - paths)
    for dt in ("fp64", "fp32"):                                 # both SIMT types on every SIMT path
        assert {g["path"] for (n, d), g in geo.items() if d == dt} >= {p for p in want if p.startswith("simt")}, dt
    assert any(g.get("row_tiles", 0) > 1 and g["path"] == "simt:dense:gemm" for g in geo.values())
    assert any(CASES[n][1].get("fourier_features") and g["path"] == "tc_pair:generic" for (n, _), g in geo.items())
    regimes = {c[0][0] for c in CASES.values()} | {"unwrapped"}
    assert regimes == {"angstrom", "far", "nano", "eps_straddle", "coincident", "unwrapped"}
    assert {CASES[n][0][1] for n in CASES if CASES[n][0][0] == "nano"} == {1e-4, 1e-6}
    cfgs = [c[1] for c in CASES.values()]
    assert {c.get("fourier_features") for c in cfgs} >= {2, 4}
    for key in ("norm_coors", "coor_weights_clamp_value", "soft_edges"):
        assert any(key in c for c in cfgs), key
    assert any(c.get("m_pool_method") == "mean" for c in cfgs)
    assert {c[4] for c in CASES.values()} >= {"padded", "random"}
    assert {c[0][1] for c in CASES.values() if c[0][0] == "coincident"} == {True, False}
    assert {kind for _, _, kind in (periodic_case(n) for n in PERIODIC)} == {"box", "cell"}


# ------------------------------------------------------------------ GPU: forward


def run_layer(case, dt):
    dtype = DT[dt]
    cdt = torch.float64 if dt == "fp64" else torch.float32
    ins = case["inputs"]
    mod = util.make_module(case, dtype)
    m = None if ins["mask"] is None else torch.from_numpy(np.asarray(ins["mask"])).to(DEV)
    fo, xo = mod(util.to_torch(ins["feats"], dtype, DEV), util.to_torch(ins["coors"], cdt, DEV), None, mask=m)
    assert mod.last_path == PATH[dt], (mod.last_path, dt)
    return fo.double().cpu().numpy(), xo.double().cpu().numpy()


@functools.lru_cache(maxsize=None)
def reference(name, cdt):
    """float64 restatement on the kernels' lists of coordinate type `cdt` -> (feats, coors) numpy."""
    case = build(name)
    ins = case["inputs"]
    idx, ok = lists(name, cdt)
    f = torch.as_tensor(ins["feats"]).to(DEV, torch.float64)
    fo, xo = TR.layer_forward(case["params"], case["cfg"], f, ins["coors"], None, ins["mask"], None, None,
                              idx, ok)
    return fo.cpu().numpy(), xo.cpu().numpy()


@functools.lru_cache(maxsize=None)
def reference_bf16(name):
    case = bf16_case(name)
    ins = case["inputs"]
    idx, ok = lists(name, "fp32")
    return T.tc_layer_forward(case["params"], case["cfg"], ins["feats"], ins["coors"], mask=ins["mask"], neighbors=idx,
                              nbr_ok=ok)


def forward_errors(out, want, x_in, dt):
    cdt = torch.float64 if dt == "fp64" else torch.float32
    (f, x), (wf, wx) = out, want
    ef = float(np.abs(f - wf).max() / max(np.abs(wf).max(), 1e-300))
    allow = 2 * ulp(np.abs(x_in).max(), cdt)
    ex = float(max(0.0, np.abs(x - wx).max() - allow) / max(np.abs(wx - x_in).max(), 1e-300))
    return ef, ex


@pytest.mark.gpu
@pytest.mark.parametrize("name,dt", FWD, ids=[f"{n}-{d}" for n, d in FWD])
def test_forward_matches_the_float64_reference(name, dt):
    case = bf16_case(name) if dt == "bf16" else build(name)
    out = run_layer(case, dt)
    assert np.isfinite(out[0]).all() and np.isfinite(out[1]).all(), name
    want = reference_bf16(name) if dt == "bf16" else reference(name, cdt_name(dt))
    ef, ex = forward_errors(out, want, case["inputs"]["coors"], dt)
    print(f"GEO fwd {name} [{dt}] {path_geometry(name, dt)['path']}: feats {ef:.3e} coors {ex:.3e}")
    assert ef <= TOL[("feats", dt)] and ex <= TOL[("coors", dt)], (name, dt, ef, ex)


# ------------------------------------------------------------------ GPU: backward


def gpu_grads(case, dtype):
    mod = util.make_module(case, dtype).requires_grad_(True)
    ins = case["inputs"]
    t = lambda a: util.to_torch(a, dtype, DEV)
    f, x = t(ins["feats"]).requires_grad_(True), t(ins["coors"]).requires_grad_(True)
    gf, gx = (t(g) for g in cotangents(case))
    m = None if ins["mask"] is None else torch.from_numpy(np.asarray(ins["mask"])).to(DEV)
    with torch.enable_grad():
        fo, xo = mod(f, x, None, mask=m)
        ((fo * gf).sum() + (xo * gx).sum()).backward()
    assert mod.last_path == PATH["fp64" if dtype == torch.float64 else "fp32"]
    out = {"in.feats": f.grad, "in.coors": x.grad}
    out.update({f"p.{k}": p.grad for k, p in mod.named_parameters()})
    return {k: v.double().cpu().numpy() for k, v in out.items()}


def cotangents(case):
    return tuple(f32(g) for g in cases.upstream_grads(case))


@functools.lru_cache(maxsize=None)
def reference_grads(name, cdt):
    case = build(name)
    ins = case["inputs"]
    idx, ok = lists(name, cdt)
    gf, gx = cotangents(case)
    f = torch.as_tensor(ins["feats"]).to(DEV, torch.float64)
    if idx is not None:
        idx, ok = torch.from_numpy(idx).to(DEV), torch.from_numpy(ok).to(DEV)
    g = TR.layer_grads_chunked(case["params"], case["cfg"], f, ins["coors"], gf, gx, None, ins["mask"], None, None,
                               idx, ok)
    return {k: v.cpu().numpy() for k, v in g.items()}


def grad_errors(got, want, case):
    """{name: worst relative error} over tensors and (node-indexed) rows; asserts finiteness where the reference is.
    The fourier and distance columns of edge_mlp.0.weight count as tensors of their own: at d^2 ~ 10^2 the distance
    column's gradient would hide the fourier columns' in one scale."""
    gf, gx = cotangents(case)
    got, want = dict(got), dict(want)
    dim, F = case["cfg"]["dim"], case["cfg"]["fourier_features"]
    for g in (got, want):
        g["in.feats"] = g["in.feats"] - gf
        g["in.coors"] = g["in.coors"] - gx
        w1 = g["p.edge_mlp.0.weight"]
        g["p.edge_mlp.0.weight[distance]"] = w1[:, 2 * dim + 2 * F]
        if F:
            g["p.edge_mlp.0.weight[fourier]"] = w1[:, 2 * dim:2 * dim + 2 * F]
    worst = {}
    for k, w in want.items():
        g = got[k]
        assert g.shape == w.shape, k
        assert np.isfinite(g[np.isfinite(w)]).all(), f"{k}: non-finite where the reference is finite"
        e = np.abs(g - w)
        worst[k] = float(e.max() / max(np.abs(w).max(), 1e-300))
        if k.startswith("in."):
            rmax = np.abs(w).reshape(w.shape[0] * w.shape[1], -1).max(1)
            floor = 1e-3 * max(float(np.median(rmax)), 1e-300)
            worst[k + "[row]"] = float((e.reshape(len(rmax), -1).max(1) / np.maximum(rmax, floor)).max())
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("saved", [True, False], ids=["saved", "recomputed"])
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name", GRAD)
def test_backward_matches_the_float64_reference(name, dt, saved, monkeypatch):
    if not saved:
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")          # the backward recomputes W2 silu(pre1)
    case = build(name)
    got = gpu_grads(case, DT[dt])
    want = reference_grads(name, cdt_name(dt))
    worst = grad_errors(got, want, case)
    top = max(worst, key=worst.get)
    print(f"GEO bwd {name} [{dt}] {'saved' if saved else 'recomputed'}: worst {worst[top]:.3e} ({top})")
    if case["cfg"]["norm_coors"] and CASES[name][0][0] in ("eps_straddle", "coincident"):
        # CoorsNorm's 1/eps branch: distinct nodes closer than 1e-8 carry a ~1e8 coordinate gradient
        w = want["in.coors"] - cotangents(case)[1]
        g = got["in.coors"] - cotangents(case)[1]
        big = np.abs(w) > 1e6
        assert big.any(), name
        assert (g[big] != 0).all() and (np.abs(g[big] - w[big]) <= grad_tol(case, dt) * np.abs(w[big])).all(), name
    bad = {k: v for k, v in worst.items() if not v <= grad_tol(case, dt)}
    assert not bad, (name, dt, saved, bad)


# ------------------------------------------------------------------ periodic, unwrapped


# name: (layer cfg, B, N, lattice kind, lattice, neighbour lists k or 0)
PERIODIC = {
    "box_dense_normc_fourier": (dict(dim=16, norm_coors=True, fourier_features=1, soft_edges=True), 2, 60, "box",
                                [3.0, 2.5, 4.0], 0),
    "box_lists_k10": (dict(dim=16, m_pool_method="mean"), 2, 80, "box", [3.5, 3.0, 2.75], 10),
    "cell_dense_tilt": (dict(dim=16, coor_weights_clamp_value=1.0), 2, 60, "cell", "tilt", 0),
    "cell_lists_k10_normc": (dict(dim=16, norm_coors=True), 2, 80, "cell", "tilt09", 10),
}


@functools.lru_cache(maxsize=None)
def periodic_case(name):
    """(case with fp32 values, lattice, kind); neighbour lists (the float64 restatement's kNN) in inputs['neighbors']."""
    cfg, B, N, kind, lat, k = PERIODIC[name]
    seed = 3100 + sorted(PERIODIC).index(name)
    case = cases.build_case(dict(kind="layer", cfg=cfg, B=B, N=N, seed=seed, init="xavier"))
    case["params"] = {p: f32(v) for p, v in case["params"].items()}
    case["inputs"]["feats"] = f32(case["inputs"]["feats"])
    rs = np.random.RandomState(seed)
    if kind == "box":
        lat = np.asarray(lat, np.float64)
        x = unwrapped_box(rs, B, N, lat)
    else:
        lat = f32(TRI.make_cell(lat, B, rs))
        x = unwrapped_cell(rs, B, N, lat)
    case["inputs"]["coors"] = x
    case["inputs"]["mask"] = None
    nb = None
    if k:
        xt = torch.as_tensor(x)
        wrap = TRI.cell_wrap if kind == "cell" else TR.wrap
        latb = torch.as_tensor(np.asarray(lat, np.float64))
        d = (wrap(xt[:, :, None] - xt[:, None], latb) ** 2).sum(-1)
        nb = torch.sort(d, dim=-1, stable=True).indices[..., :k].numpy()
    case["inputs"]["neighbors"] = nb
    return case, lat, kind


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("name", list(PERIODIC))
def test_unwrapped_periodic_forward_gradients_and_lattice_gradient(name, dt):
    """Coordinates up to 64 lattice vectors out: pairs wrap by up to ~130 images, and the lattice gradient
    -sum n_c dL/drel_c carries those image counts."""
    case, lat, kind = periodic_case(name)
    dtype = DT[dt]
    cdt = torch.float64 if dt == "fp64" else torch.float32
    ins = case["inputs"]
    nb = ins["neighbors"]
    mod = util.make_module(case, dtype)
    kw = {kind: torch.as_tensor(np.asarray(lat), dtype=cdt, device=DEV)}
    if nb is not None:
        kw["neighbors"] = torch.from_numpy(nb).to(DEV)
    fo, xo = mod(util.to_torch(ins["feats"], dtype, DEV), util.to_torch(ins["coors"], cdt, DEV), **kw)
    assert mod.last_path == PATH[dt]
    with TRI._cell_geometry() if kind == "cell" else contextlib.nullcontext():
        want = [t.numpy() for t in TR.layer(case["params"], case["cfg"], ins["feats"], ins["coors"], None, None, None,
                                            lat, nb)]
    ef, ex = forward_errors((fo.double().cpu().numpy(), xo.double().cpu().numpy()), want, ins["coors"], dt)
    gf, gx = LGR._cotangents(case)
    gf, gx = f32(gf), f32(gx)
    got = LGR.gpu_grads(case, lat, kind, dtype, gf, gx, neighbors=nb)
    ref = {k: v.cpu().numpy() for k, v in LGR.ref_grads(case, lat, kind, gf, gx, neighbors=nb).items()}
    errs = {}
    for k, w in ref.items():
        if k == "lattice":
            continue
        g = got[k]
        assert np.isfinite(g).all(), (name, dt, k)
        errs[k] = float(np.abs(g - w).max() / max(np.abs(w).max(), 1e-300))
    top = max(errs, key=errs.get)
    L = np.diagonal(np.asarray(lat), axis1=-2, axis2=-1) if kind == "cell" else np.asarray(lat)
    n_img = np.abs(np.rint((ins["coors"][:, :, None] - ins["coors"][:, None]) / L.max())).max()
    print(f"GEO periodic {name} [{dt}]: feats {ef:.3e} coors {ex:.3e} grads {errs[top]:.3e} ({top}), image counts up "
          f"to {n_img:.0f}")
    assert ef <= TOL[("feats", dt)] and ex <= (UNWRAPPED_FP32_COORS if dt == "fp32" else TOL[("coors", dt)]), (
        name, dt, ef, ex)
    assert errs[top] <= grad_tol(case, dt), (name, dt, top, errs[top])
    assert float(np.abs(ref["lattice"]).max()) > 1e-3
    if dt == "fp64":
        LGR.check64(got["lattice"], ref["lattice"], f"{name} [{dt}]")
    else:
        ref32 = LGR.ref_grads(case, lat, kind, gf, gx, dtype=torch.float32, neighbors=nb)["lattice"].double().numpy()
        LGR.check32(got["lattice"], ref32, ref["lattice"], f"{name} [{dt}]")


TRANSLATION = 2.0 ** 12


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["fp32", "bf16"])
def test_translation_by_2_to_the_12_changes_no_feature_bit(dt):
    """Coordinates on the 2^-11 grid that fp32 keeps at 2^12 .. 2^13, so x + 2^12 and every x_i - x_j are exact: the
    pair vectors, their wrap and so the features are bit for bit those of the untranslated inputs; the coordinates move
    by 2^12 within the rounding of x + update there."""
    cfg, B, N, _, L, _ = PERIODIC["box_dense_normc_fourier"]
    case = cases.build_case(dict(kind="layer", cfg=cfg, B=B, N=N, seed=3200, init="xavier"))
    rs = np.random.RandomState(3200)
    x = np.round(PER.lattice_coors(rs, B, N, 3, L, shift=7) * 2 ** 11) / 2 ** 11
    assert PER.half_box_margin(x, L) >= 1e-3 and np.abs(x).max() < TRANSLATION
    dtype = DT[dt]
    mod = util.make_module(case, dtype)
    f = util.to_torch(case["inputs"]["feats"], dtype, DEV)
    box = torch.tensor(L, dtype=torch.float32, device=DEV)
    x0 = torch.from_numpy(x).to(DEV, torch.float32)
    f0, c0 = mod(f, x0, box=box)
    f1, c1 = mod(f, x0 + TRANSLATION, box=box)
    assert mod.last_path == PATH[dt]
    assert torch.equal(f0, f1)
    err = float((c1.double() - TRANSLATION - c0.double()).abs().max())
    print(f"GEO translation [{dt}]: coors moved by 2^12 within {err:.3e}")
    assert err <= ulp(TRANSLATION, torch.float32)


# ------------------------------------------------------------------ cell-grid selects at offsets and at the +-2^30 clamp


def offset_cloud(n, centre, extent, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand((2, n, 3), generator=g, dtype=torch.float64) - 0.5) * extent + torch.tensor(centre)
    return x.to(DEV, dtype).contiguous()


SELECT = [(1e4, torch.float32), (1e4, torch.float64), (1e5, torch.float32), (1e5, torch.float64)]


@pytest.mark.gpu
@pytest.mark.parametrize("centre,dtype", SELECT, ids=[f"{c:.0e}-{str(d)[6:]}" for c, d in SELECT])
def test_cell_grid_selects_at_an_offset_equal_the_all_pairs_select(centre, dtype):
    from egnn_pytorch_b200 import _native
    lib = _native.load()
    x = offset_cloud(1500, (centre, -centre, 0.5 * centre), 12.0, dtype, seed=int(centre) % 97)
    mask = torch.rand((2, 1500), generator=torch.Generator().manual_seed(5)).to(DEV) < 0.9
    cutoff = RS.cutoff_for(x, mask, 20)
    RS.check_vs_all_pairs(lib, x, mask, 32, cutoff, f"radius narrow at {centre:.0e}")
    RSW.check(x.cpu().numpy(), RS.cutoff_for(x, mask, 80), 64, f"radius wide at {centre:.0e}", mask=mask.cpu().numpy())
    for k in (16, 48):
        KG.check(lib, x, mask, k, cutoff * cutoff, f"knn grid k={k} at {centre:.0e}")


@pytest.mark.gpu
def test_cell_grid_selects_beyond_the_2_to_the_30_cell_clamp():
    """fp64, cutoff 1e-4 at |x| ~ 2e5: |x| / cs = 2e9 cells, beyond the +-2^30 the binning clamps to."""
    from egnn_pytorch_b200 import _native
    lib = _native.load()
    x = offset_cloud(600, (2e5, -2e5, 2e5), 1e-3, torch.float64, seed=7)
    cutoff = 1e-4
    assert float(x.abs().min()) / cutoff > 2 ** 30
    cnt = RS.check_vs_all_pairs(lib, x, None, 32, cutoff, "radius narrow at the clamp")
    assert int(cnt.max()) > 1                                         # pairs within the cutoff exist
    RSW.check(x.cpu().numpy(), 2 * cutoff, 48, "radius wide at the clamp")
    KG.check(lib, x, None, 16, cutoff * cutoff, "knn grid at the clamp")


@pytest.mark.gpu
def test_angstrom_layer_above_the_grid_threshold_is_bit_identical_on_both_selects(monkeypatch):
    """N = 5000 (above both grid thresholds), k = 16, valid_radius = 25 A^2: the cell-grid and all-pairs selects give
    the same outputs bit for bit."""
    from egnn_pytorch_b200 import EGNN, _native
    lib = _native.load()
    torch.manual_seed(11)
    x = torch.from_numpy(angstrom(np.random.RandomState(11), 1, 5000)).to(DEV, torch.float32)
    mod = EGNN(dim=32, num_nearest_neighbors=16, valid_radius=25.0, norm_coors=True).to(DEV).eval()
    f = torch.randn((1, 5000, 32), device=DEV)
    mask = torch.rand((1, 5000), device=DEV) < 0.95

    def run():
        return mod(f, x, mask=mask)
    monkeypatch.setenv("EGNN_B200_CELL_SELECT_MIN_N", "0")
    monkeypatch.setenv("EGNN_B200_KNN_GRID_MIN_N", "0")
    grid, n_grid = RS._launches(lib, run)
    monkeypatch.setenv("EGNN_B200_CELL_SELECT_MIN_N", RS.NEVER)
    monkeypatch.setenv("EGNN_B200_KNN_GRID_MIN_N", RS.NEVER)
    allp, n_all = RS._launches(lib, run)
    assert n_grid > n_all, (n_grid, n_all)
    for a, w in zip(grid, allp):
        assert torch.equal(RS.bits(a), RS.bits(w))
