"""The cell-grid radius select (csrc/radius_select.cu): `radius_neighbors` / egnn_radius_select and the layer's own use of it.

Reference: the all-pairs select egnn_knn_select with valid_radius = r2.  The cell lists must equal its ok = 1 slots exactly
(same rank arithmetic, ties to the lower index) and hold -1 elsewhere; the counts must equal the number of in-radius
valid nodes, taken from a full ranking (k = N) of the same select.  Periodic inputs, which egnn_knn_select does not take,
are checked against an fp64 numpy brute force on inputs whose squared distances keep a relative 1e-4 from r2 and from one
another within a row (nodes that would break this are padded out), so that rounding cannot decide a slot.

Inside a layer the two paths are switched with EGNN_B200_CELL_SELECT_MIN_N (0 = cell grid, huge = all pairs); outputs
must be bit-identical and gradients equal to the backward's atomics tolerance."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
NEVER = str(2 ** 40)


@pytest.fixture(scope="module")
def lib():
    from egnn_pytorch_b200 import _native
    return _native.load()


def _dt(dtype):
    from egnn_pytorch_b200 import _native as nat
    return nat.DTYPE_F64 if dtype == torch.float64 else nat.DTYPE_F32


def knn_select(lib, x, mask, k, r2):
    """egnn_knn_select with valid_radius = r2 -> (idx, ok) [B, N, k]."""
    b, n, c = x.shape
    idx = torch.empty((b, n, k), dtype=torch.int32, device=DEV)
    ok = torch.empty((b, n, k), dtype=torch.uint8, device=DEV)
    m = None if mask is None else mask.to(torch.uint8).contiguous()
    rc = lib.egnn_knn_select(_dt(x.dtype), b, n, c, k, C.c_void_p(x.data_ptr()), None if m is None else C.c_void_p(m.data_ptr()),
                             None, 0, float(r2), C.c_void_p(idx.data_ptr()), C.c_void_p(ok.data_ptr()),
                             C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, rc
    return idx, ok.bool()


def expected_from_all_pairs(lib, x, mask, k, r2):
    """The cell select's expected lists (ok slots of egnn_knn_select, -1 elsewhere) and counts (full ranking)."""
    idx, ok = knn_select(lib, x, mask, k, r2)
    want = torch.where(ok, idx, torch.full_like(idx, -1))
    _, ok_all = knn_select(lib, x, mask, x.shape[1], r2)
    return want, ok_all.sum(-1, dtype=torch.int32)


def cutoff_for(x, mask, m):
    """A cutoff whose in-radius count is about m for a typical row (median over up to 64 rows of the m-th smallest d^2)."""
    b, n, _ = x.shape
    rows = x[0, : min(n, 64)].double()
    d2 = ((rows[:, None] - x[0][None].double()) ** 2).sum(-1)
    if mask is not None:
        d2 = d2.masked_fill(~mask[0].bool()[None], float("inf"))
    d2 = d2.sort(-1).values[:, min(m, n) - 1]
    v = float(d2[torch.isfinite(d2)].median()) if torch.isfinite(d2).any() else 1.0
    return math.sqrt(v) if v > 0 else 1.0


def check_vs_all_pairs(lib, x, mask, k, cutoff, what):
    from egnn_pytorch_b200 import radius_neighbors
    r2 = cutoff * cutoff
    got, cnt = radius_neighbors(x, cutoff, k, mask=mask, return_counts=True)
    want, want_cnt = expected_from_all_pairs(lib, x, mask, k, r2)
    bad = (got != want).any(-1)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} rows differ, first {bad.nonzero()[0].tolist()}: " \
        f"{got[bad][0].tolist()} vs {want[bad][0].tolist()}"
    assert torch.equal(cnt, want_cnt), f"{what}: counts differ in {int((cnt != want_cnt).sum())} rows"
    return cnt


# ----------------------------------------------------------------------------- 1. lists vs the all-pairs select


@pytest.mark.parametrize("n", [1, 31, 33, 1000, 5000])
@pytest.mark.parametrize("c", [1, 2, 3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_lists_equal_all_pairs_select(lib, dtype, c, n):
    g = torch.Generator(device="cpu").manual_seed(1000 * c + n)
    for b in (1, 3):
        x = (torch.rand((b, n, c), generator=g, dtype=torch.float64) * (n ** (1.0 / c))).to(DEV, dtype)
        mask = (torch.rand((b, n), generator=g) < 0.85).to(DEV)
        mask[:, 0] = True
        for k in (1, 7, 16, 32):
            if k > n:
                continue
            seen_lo = seen_hi = False
            for m in (max(2, k // 2), 2 * k + 3):
                cut = cutoff_for(x, mask, m)
                cnt = check_vs_all_pairs(lib, x, mask, k, cut, f"{dtype} C={c} N={n} B={b} k={k} m={m}")
                seen_lo |= bool((cnt[mask] < k).any())
                seen_hi |= bool((cnt[mask] > k).any())
            if n >= 1000 and k > 1:                        # (k = 1: every valid row holds at least itself)
                assert seen_lo and seen_hi, "radii must give counts on both sides of k"


# ----------------------------------------------------------------------------- 2. adversarial inputs


def test_duplicates_one_cell_lattice_outlier(lib):
    g = torch.Generator(device="cpu").manual_seed(7)
    for dtype in (torch.float32, torch.float64):
        # duplicate coordinates: ties go to the lower index
        base = torch.randint(0, 6, (2, 400, 3), generator=g).to(dtype)
        x = base[:, torch.randint(0, 400, (400,), generator=g)].to(DEV)
        mask = torch.ones(2, 400, dtype=torch.bool, device=DEV)
        for k in (1, 7, 32):
            check_vs_all_pairs(lib, x, mask, k, 1.5, f"duplicates {dtype} k={k}")
        # every node in one cell
        x = (torch.rand((1, 300, 3), generator=g, dtype=torch.float64) * 0.1).to(DEV, dtype)
        check_vs_all_pairs(lib, x, torch.ones(1, 300, dtype=torch.bool, device=DEV), 32, 10.0, f"one cell {dtype}")
        # integer lattice: many pairs exactly at the cutoff and on cell faces (exact in both types)
        ax = torch.arange(-6, 7, dtype=torch.float64)
        lat = torch.stack(torch.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(1, -1, 3)
        lat = lat[:, torch.randperm(lat.shape[1], generator=g)].to(DEV, dtype)
        lm = (torch.rand(lat.shape[:2], generator=g) < 0.9).to(DEV)
        for r2 in (1.0, 2.0, 3.0, 4.0, 5.0):
            for k in (7, 16, 32):
                check_vs_all_pairs(lib, lat, lm, k, math.sqrt(r2), f"lattice {dtype} r2={r2} k={k}")
        for c in (1, 2):
            check_vs_all_pairs(lib, lat[..., :c].contiguous(), lm, 16, 1.0, f"lattice C={c} {dtype}")
        # a far outlier spreads the cell coordinates (and a node at exactly a huge coordinate)
        x = torch.rand((2, 500, 3), generator=g, dtype=torch.float64) * 8
        x[0, 17] = torch.tensor([1e6, -3e5, 2e4], dtype=torch.float64)
        x[1, 3] = torch.tensor([-1e9, 1e9, 0.5], dtype=torch.float64)
        x = x.to(DEV, dtype)
        check_vs_all_pairs(lib, x, torch.ones(2, 500, dtype=torch.bool, device=DEV), 16, 1.2, f"outlier {dtype}")


def test_non_finite_coordinates_are_never_neighbours(lib):
    from egnn_pytorch_b200 import radius_neighbors
    x = torch.rand((1, 200, 3), dtype=torch.float64, device=DEV) * 3
    bad = [5, 50, 150]
    x[0, 5, 0] = float("nan")
    x[0, 50, 1] = float("inf")
    x[0, 150, 2] = -float("inf")
    got, cnt = radius_neighbors(x, 1.0, 16, return_counts=True)
    for i in bad:
        assert (got[0, i] == -1).all() and int(cnt[0, i]) == 0
    assert not torch.isin(got, torch.tensor(bad, device=DEV, dtype=torch.int32)).any()
    keep = torch.ones(200, dtype=torch.bool, device=DEV)
    keep[bad] = False
    # the finite rows equal the all-pairs select on the finite nodes alone (masking the others out)
    want, want_cnt = expected_from_all_pairs(lib, x.nan_to_num(0.0, 0.0, 0.0), keep[None], 16, 1.0)
    assert torch.equal(got[0, keep], want[0, keep]) and torch.equal(cnt[0, keep], want_cnt[0, keep])


def brute_periodic(x, mask, box, k, r2):
    """fp64 numpy reference with minimum-image distances -> (lists with -1, counts, min relative gap to r2 / in row)."""
    x = np.asarray(x, np.float64)
    b, n, c = x.shape
    box = np.broadcast_to(np.asarray(box, np.float64), (b, c))
    out = np.full((b, n, k), -1, np.int32)
    cnt = np.zeros((b, n), np.int32)
    for g in range(b):
        L = box[g]
        per = (L > 0) & np.isfinite(L)
        rel = x[g][:, None] - x[g][None]
        Lp = np.where(per, L, 0.0)
        rel = rel - Lp * np.round(rel * np.where(per, 1.0 / np.where(per, L, 1.0), 0.0))
        d2 = (rel ** 2).sum(-1)
        valid = mask[g]
        d2[:, ~valid] = np.inf
        for i in range(n):
            if not valid[i]:
                continue
            order = np.lexsort((np.arange(n), d2[i]))
            inr = order[d2[i][order] <= r2]
            cnt[g, i] = len(inr)
            out[g, i, : min(k, len(inr))] = inr[:k]
    return out, cnt


def separate(x, mask, box, r2, k):
    """Pad out nodes until every valid pair's d^2 is 1e-4 (relative) away from r2 and from the next d^2 of its row."""
    x = np.asarray(x, np.float64)
    mask = np.array(mask, bool)
    b, n, c = x.shape
    box = np.broadcast_to(np.asarray(box, np.float64), (b, c))
    for g in range(b):
        L = box[g]
        per = (L > 0) & np.isfinite(L)
        rel = x[g][:, None] - x[g][None]
        rel = rel - np.where(per, L, 0.0) * np.round(rel * np.where(per, 1.0 / np.where(per, L, 1.0), 0.0))
        d2 = (rel ** 2).sum(-1)
        for i in range(n):
            if not mask[g, i]:
                continue
            while True:
                js = np.nonzero(mask[g])[0]
                js = js[js != i]
                dd = d2[i, js]
                near = js[np.abs(dd - r2) < 1e-4 * r2]
                o = np.argsort(dd)
                s = dd[o]
                close = np.nonzero(np.diff(s) < 1e-4 * np.maximum(s[1:], 1e-30))[0]
                if len(near):
                    mask[g, near[0]] = False
                elif len(close) and s[close[0]] <= r2 * 1.01:
                    mask[g, js[o][close[0] + 1]] = False
                else:
                    break
    return mask


PERIODIC = {
    # name: (C, box [C] or [B, C], cutoff, shift in box lengths)
    "cube_outside": (3, [6.0, 6.0, 6.0], 1.3, 3),          # coordinates several box lengths outside the box
    "one_cell": (1, [3.0], 2.0, 1),                         # L / cs in [1, 2): one cell
    "two_cells": (2, [5.0, 5.0], 2.0, 1),                   # two cells per axis
    "three_cells": (3, [7.0, 7.0, 7.0], 2.0, 2),            # three cells per axis
    "mixed_axes": (3, [6.0, 0.0, float("inf")], 1.2, 2),    # periodic, aperiodic (0), aperiodic (inf)
    "per_graph": (3, [[5.0, 7.0, 9.0], [4.0, 0.0, 6.5], [float("inf"), 3.0, 3.0]], 1.1, 2),
}


@pytest.mark.parametrize("name", sorted(PERIODIC))
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_periodic_against_brute_force(dtype, name):
    from egnn_pytorch_b200 import radius_neighbors
    c, box, cut, shift = PERIODIC[name]
    rs = np.random.RandomState(len(name) * 31 + c)
    b = 3
    boxa = np.broadcast_to(np.asarray(box, np.float64), (b, c))
    span = np.where(np.isfinite(boxa) & (boxa > 0), boxa, 6.0)
    n = 160
    x = rs.uniform(0, 1, (b, n, c)) * span[:, None, :]
    x = x + rs.randint(-shift, shift + 1, (b, n, c)) * np.where(np.isfinite(boxa) & (boxa > 0), boxa, 0.0)[:, None, :]
    x = x.astype(np.float32 if dtype == torch.float32 else np.float64).astype(np.float64)
    r2 = cut * cut
    mask = separate(x, rs.uniform(size=(b, n)) < 0.9, boxa, r2, 32)
    for k in (1, 7, 32):
        want, want_cnt = brute_periodic(x, mask, boxa, k, r2)
        got, cnt = radius_neighbors(torch.tensor(x, dtype=dtype, device=DEV), cut, k, mask=torch.tensor(mask, device=DEV),
                                    box=torch.tensor(np.ascontiguousarray(box), dtype=dtype, device=DEV), return_counts=True)
        assert np.array_equal(got.cpu().numpy(), want), f"{name} {dtype} k={k}"
        assert np.array_equal(cnt.cpu().numpy(), want_cnt), f"{name} {dtype} k={k} counts"


# ----------------------------------------------------------------------------- 3. layer outputs: cell path == all pairs


def _launches(lib, fn):
    lib.egnn_profile_read(None, None, None, 1)
    lib.egnn_profile_enable(1)
    try:
        out = fn()
        torch.cuda.synchronize()
        n = C.c_int64()
        lib.egnn_profile_read(None, None, C.byref(n), 1)
    finally:
        lib.egnn_profile_enable(0)
    return out, n.value


def both_paths(lib, monkeypatch, fn):
    """fn() on the cell path and on the all-pairs path -> (cell outputs, all-pairs outputs); checks which path ran by the
    launches of the select (4 for the cell grid, 1 for all pairs)."""
    monkeypatch.setenv("EGNN_B200_CELL_SELECT_MIN_N", "0")
    cell, n_cell = _launches(lib, fn)
    monkeypatch.setenv("EGNN_B200_CELL_SELECT_MIN_N", NEVER)
    allp, n_all = _launches(lib, fn)
    assert n_cell > n_all and (n_cell - n_all) % 3 == 0, (n_cell, n_all)
    return cell, allp


def cloud(b, n, c=3, mean_count=20.0, r2=1.0, seed=0, dtype=torch.float32, pad=0.9):
    g = torch.Generator(device="cpu").manual_seed(seed)
    side = (n * (4.0 / 3.0) * math.pi * r2 ** 1.5 / mean_count) ** (1.0 / 3.0)
    x = (torch.rand((b, n, c), generator=g, dtype=torch.float64) * side).to(DEV, dtype)
    mask = (torch.rand((b, n), generator=g) < pad).to(DEV)
    return x, mask, side


LAYER_VARIANTS = {
    "plain": dict(),
    "soft_edges": dict(soft_edges=True),
    "mean": dict(m_pool_method="mean"),
    "norm_coors": dict(norm_coors=True),
    "clamp": dict(coor_weights_clamp_value=0.05),
    "box": dict(),
}


def bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


@pytest.mark.parametrize("variant", sorted(LAYER_VARIANTS))
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32, torch.bfloat16])
def test_layer_outputs_bit_identical(lib, monkeypatch, dtype, variant):
    from egnn_pytorch_b200 import EGNN
    torch.manual_seed(3)
    k = 16
    dim = 64 if dtype == torch.bfloat16 else 24
    mod = EGNN(dim=dim, edge_dim=0, num_nearest_neighbors=k, valid_radius=1.0, **LAYER_VARIANTS[variant]).to(DEV, dtype)
    n, b = 700, 2
    x, mask, side = cloud(b, n, dtype=torch.float64 if dtype == torch.float64 else torch.float32, seed=5)
    feats = torch.randn((b, n, dim), device=DEV).to(dtype)
    kw = dict(mask=mask)
    if variant == "box":
        kw["box"] = torch.tensor([side, side, 0.0], device=DEV, dtype=x.dtype)
    cell, allp = both_paths(lib, monkeypatch, lambda: mod(feats, x, **kw))
    if dtype == torch.bfloat16:
        assert mod.last_path == "bf16-tc"
    for a, w, what in zip(cell, allp, ("feats", "coors")):
        assert torch.equal(bits(a), bits(w)), f"{dtype} {variant} {what}: max diff {(a.float() - w.float()).abs().max()}"


def test_network_outputs_bit_identical(lib, monkeypatch):
    from egnn_pytorch_b200 import EGNN_Network
    torch.manual_seed(4)
    net = EGNN_Network(depth=3, dim=32, num_nearest_neighbors=12, valid_radius=1.0, coor_weights_clamp_value=2.0).to(DEV)
    x, mask, _ = cloud(2, 600, seed=9)
    feats = torch.randn((2, 600, 32), device=DEV)
    cell, allp = both_paths(lib, monkeypatch, lambda: net(feats, x, mask=mask))
    assert torch.equal(bits(cell[0]), bits(allp[0])) and torch.equal(bits(cell[1]), bits(allp[1]))


# ----------------------------------------------------------------------------- 4. training


@pytest.mark.parametrize("saved", [True, False], ids=["saved_pre2", "recompute"])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_gradients_agree(lib, monkeypatch, dtype, saved):
    from egnn_pytorch_b200 import EGNN
    if not saved:
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")
    torch.manual_seed(6)
    mod = EGNN(dim=16, num_nearest_neighbors=12, valid_radius=1.0, norm_coors=True).to(DEV, dtype)
    x0, mask, side = cloud(2, 500, dtype=dtype, seed=11)
    f0 = torch.randn((2, 500, 16), device=DEV, dtype=dtype)
    gf = torch.randn_like(f0)
    gx = torch.randn_like(x0)

    def run():
        f, x = f0.clone().requires_grad_(True), x0.clone().requires_grad_(True)
        mod.zero_grad(set_to_none=True)
        with torch.enable_grad():
            fo, xo = mod(f, x, mask=mask, box=torch.tensor([side, side, side], device=DEV, dtype=dtype))
            ((fo * gf).sum() + (xo * gx).sum()).backward()
        grads = {"feats": f.grad, "coors": x.grad}
        grads.update({k: p.grad.clone() for k, p in mod.named_parameters()})
        return fo.detach(), xo.detach(), grads

    cell, allp = both_paths(lib, monkeypatch, run)
    assert torch.equal(bits(cell[0]), bits(allp[0])) and torch.equal(bits(cell[1]), bits(allp[1]))
    tol = 1e-10 if dtype == torch.float64 else 2e-5
    for k, g in cell[2].items():
        w = allp[2][k]
        scale = max(1.0, float(w.abs().max()))
        assert float((g - w).abs().max()) <= tol * scale, f"{dtype} {k}: {float((g - w).abs().max())}"


# ----------------------------------------------------------------------------- 5. graph capture


def test_graph_capture_on_the_cell_path(lib, monkeypatch):
    from egnn_pytorch_b200 import EGNN, GraphedForward
    monkeypatch.setenv("EGNN_B200_CELL_SELECT_MIN_N", "0")
    torch.manual_seed(8)
    mod = EGNN(dim=32, num_nearest_neighbors=16, valid_radius=1.0).to(DEV)
    x, mask, _ = cloud(2, 800, seed=13)
    feats = torch.randn((2, 800, 32), device=DEV)
    fast = GraphedForward(mod, feats, x, mask=mask)
    for s in range(3):
        x2 = x + 0.3 * torch.randn(x.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(s))
        f2 = torch.randn_like(feats)
        got = [t.clone() for t in fast(f2, x2)]
        want = mod(f2, x2, mask=mask)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    monkeypatch.setenv("EGNN_B200_CELL_SELECT_MIN_N", NEVER)
    want = mod(f2, x2, mask=mask)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


# ----------------------------------------------------------------------------- 6. large graph


def test_large_graph_equals_all_pairs(lib):
    from egnn_pytorch_b200 import radius_neighbors
    n, k = 131_072, 32
    x, mask, _ = cloud(1, n, mean_count=40.0, seed=21, pad=0.97)
    got, cnt = radius_neighbors(x, 1.0, k, mask=mask, return_counts=True)
    idx, ok = knn_select(lib, x, mask, k, 1.0)
    want = torch.where(ok, idx, torch.full_like(idx, -1))
    assert torch.equal(got, want)
    assert torch.equal((got >= 0).sum(-1, dtype=torch.int32), cnt.clamp(max=k))
    assert bool((cnt > k).any()) and bool(((cnt < k) & mask).any())
