"""The fp32 / fp64 backward (egnn_layer_backward) at the BASELINE shapes, against the row-chunked torch restatement of
tests/torch_reference.py run on the device in float64.

The small-graph gradient tests never reach the schedule branches that only large graphs take (mirrored in `geometry`
through tests/launch_geometry.py and held by test_table_covers_every_size_boundary, with H100_SMS = 132):
  gemm_acc   one CTA over all of K (tiles >= 2 SMs: g_h += gA W1_i at c2) and large splits with a partial last one
             (dWn2 at c2: K = 4096 in 3 splits of 1376)
  dsilu_mul  its grid-stride loop (the grid stops at 2048 CTAs: more than 524,288 elements)
  bwd2       dense: 17 channel CTAs (the last with 8 of its 128 channels) x 32 row CTAs x 4 graphs adding dL/dB_j with
             atomics, generic (Q = 9) with a partial last row CTA; kNN: TS = 32 and 9 channel CTAs over 4096 nodes
  pre2       saved by the forward, recomputed by the register-tiled kernel (budget 0), and per row block
  networks   token / position embeddings, kNN reselected on updated coordinates, degree-label gradients and the 8192-node
             per-node reductions of an adjacency network
Every case uses xavier weights (no path hides behind the biases) and seeded normal cotangents on both outputs.  Layer
cases take the kernels' neighbour lists from test_gpu_knn_select.ref_select (bit for bit the kernels' ranking, in the
layer's type); network cases select in the restatement, which asserts a relative k-th / (k+1)-th rank gap far beyond
the coordinates' deviation on every layer (c3 in fp32 runs one layer for that reason).

Gates (in.feats / in.coors compare grad - cotangent: the identity path is copied exactly):
  fp64   per tensor max|got - want| <= TAU64 max|want|; node-indexed tensors also per row, against the row's own max
         with a floor of 1e-3 of the tensor's scale
  fp32   per tensor, max and RMS error against the fp64 restatement <= 4x the fp32 restatement's own (TF32 off), with a
         floor of 1e-7 of the tensor's scale; 64x for the parameter gradients summed in long fp32 chains (FP32_CHAINED)
  exact  dense edge gradients are 0 outside the selected slots and on masked pairs; every gradient is finite and has
         its parameter's type
Measured on an H100 80GB HBM3 (700 W power limit): see DESIGN.md section 8."""
import time

import numpy as np
import pytest
import torch

import cases
import launch_geometry as LG
import torch_reference as TR
import util
from test_gpu_knn_select import ref_select

L, NW = "layer", "network"
DEV = "cuda"
DT = {"fp64": torch.float64, "fp32": torch.float32}
TAU64 = 3e-13
FP32_RATIO, FP32_FLOOR = 4.0, 1e-7
# Parameter gradients the kernels sum in long fp32 chains (bwd1's per-thread sums over every pair a CTA visits and
# bwd2's dW2, then one atomic per CTA): at size they carry up to 16x the error of torch's blocked sums, varying with the
# atomic order from run to run.  Their ratio is held at 4x the worst measured instead (DESIGN.md section 8).
FP32_CHAINED = ("coors_mlp.0.weight", "coors_mlp.0.bias", "coors_mlp.3.weight", "coors_mlp.3.bias", "edge_mlp.3.weight",
                "edge_mlp.3.bias", "edge_gate.0.weight", "edge_gate.0.bias", "coors_norm.scale")
FP32_CHAINED_RATIO = 64.0

SIZE_CASES = {
    "c2": dict(kind=L, cfg=dict(dim=512), B=4, N=1024, seed=1201, init="xavier"),
    "dense_generic": dict(kind=L, cfg=dict(dim=128, edge_dim=4, fourier_features=2, soft_edges=True, m_pool_method="mean",
                                           coor_weights_clamp_value=1.0, norm_feats=True), B=2, N=1000, seed=1202,
                          init="xavier", mask="random"),
    "c4": dict(kind=L, cfg=dict(dim=256, edge_dim=4, num_nearest_neighbors=32), B=2, N=4096, seed=1203, init="xavier"),
    "c4_box": dict(kind=L, cfg=dict(dim=256, edge_dim=4, num_nearest_neighbors=32), B=2, N=4096, seed=1204,
                   init="xavier"),
    "c3": dict(kind=NW, cfg=dict(depth=3, dim=32, num_tokens=21, num_positions=1024, num_nearest_neighbors=8,
                                 coor_weights_clamp_value=2.0), B=1, N=1024, seed=1205, init="xavier", mask="padded"),
    "c5": dict(kind=NW, cfg=dict(depth=3, dim=32, num_tokens=21, num_adj_degrees=3, adj_dim=8, only_sparse_neighbors=True),
               B=1, N=8192, seed=1206, init="xavier", adj="chain", mask="full"),
}
C4_BOX = 16.0                # 4096 nodes in [0, 16)^3: about one per unit volume, 32 neighbours within ~2


# ------------------------------------------------------------------ launch geometry (tests/launch_geometry.py)


def geometry(name, dt="fp64"):
    spec = SIZE_CASES[name]
    layer = LG.layer_dims(spec["kind"], spec["cfg"])[0]
    B, N, dim, m = spec["B"], spec["N"], layer["dim"], layer["m_dim"]
    k = 9 if layer["only_sparse_neighbors"] else layer["num_nearest_neighbors"]     # chain, 3 degrees: |i - j| <= 4
    g = LG.simt_layer(spec["kind"], spec["cfg"], B, N, k=k)
    M, H, acc = B * N, 2 * g["E"], LG.launch_gemm_acc
    g.update(M=M, gemm={"g_h_gA": acc(M, dim, H), "g_h_gB": acc(M, dim, H), "dW1_i": acc(H, dim, M),
                        "dWn2": acc(dim, 2 * dim, M), "ga": acc(M, 2 * dim, dim), "dWn1": acc(2 * dim, dim + m, M),
                        "g_node_in": acc(M, dim + m, 2 * dim)},
             dsilu_strides=LG.dsilu_strides(M * 2 * dim), bwd2_last_ch=g["Hp"] - (g["bwd2_ch_ctas"] - 1) * LG.BW2_TH,
             pre2_saved=LG.pre2_saved(B, N, k or N, m, 8 if dt == "fp64" else 4))
    if not k:
        g.update(bwd2_last_rows=N - (g["bwd2_row_ctas"] - 1) * LG.BW2_ROWS, generic_bwd2=g["Q"] > 1)
    return g


def test_table_covers_every_size_boundary():
    c2 = geometry("c2")
    assert c2["gemm"]["g_h_gA"][0] == 1 and c2["gemm"]["g_h_gB"][0] == 1          # one CTA reduces all of K = H
    splits, kper, last = c2["gemm"]["dWn2"]
    assert splits == 3 and kper == 1376 and 0 < last < kper                        # large splits, partial last one
    assert c2["dsilu_strides"] > 1                                                 # the grid-stride loop runs
    assert (c2["bwd2_ch_ctas"], c2["bwd2_last_ch"], c2["bwd2_row_ctas"]) == (17, 8, 32) and not c2["generic_bwd2"]
    assert c2["pre2_saved"] and geometry("c2", "fp32")["pre2_saved"]               # c2_recompute sets the budget to 0
    gen = geometry("dense_generic")
    assert gen["generic_bwd2"] and 0 < gen["bwd2_last_rows"] < LG.BW2_ROWS and gen["bwd2_ch_ctas"] > 1
    c4 = geometry("c4")
    assert c4["TS"] == 32 and c4["bwd2_ch_ctas"] == 9 and c4["dsilu_strides"] > 1
    c5 = geometry("c5")
    assert c5["labels"] == 4 and c5["k"] == 9 and c5["M"] == 8192
    assert any(s > 1 and 0 < l < kp for s, kp, l in c5["gemm"].values())         # split K over the 8192 node rows


# ------------------------------------------------------------------ inputs, the product, the reference


@pytest.fixture(autouse=True)
def _no_tf32():
    """The fp32 restatement measures fp32 arithmetic: no TF32 in its matmuls."""
    with util.no_tf32():
        yield


def build(name, dt, depth=None):
    """The case with its parameters and float inputs in the layer's type (so the fp64 reference differentiates what the
    kernels see), its cotangents, box and (layers) the kernels' neighbour lists."""
    spec = dict(SIZE_CASES[name])
    if depth is not None:
        spec["cfg"] = dict(spec["cfg"], depth=depth)
    case = cases.build_case(spec)
    dtype = DT[dt]
    rs = np.random.RandomState(spec["seed"] + 7)
    box = None
    if name == "c4_box":
        case["inputs"]["coors"] = rs.uniform(0.0, C4_BOX, case["inputs"]["coors"].shape)
        box = np.full(3, C4_BOX)
    case["params"] = {k: util.rounded(v, dtype) for k, v in case["params"].items()}
    case["inputs"] = {k: util.rounded(v, dtype) for k, v in case["inputs"].items()}
    gf, gx = cases.upstream_grads(case)
    case["grads"] = (util.rounded(gf, dtype), util.rounded(gx, dtype))
    case["box"] = box
    cfg = case["cfg"] if spec["kind"] == L else None
    if cfg is not None and cfg["num_nearest_neighbors"] > 0:
        x = np.asarray(case["inputs"]["coors"], np.float64 if dt == "fp64" else np.float32)
        B = x.shape[0]
        idx, ok = ref_select(x, cfg["num_nearest_neighbors"], cfg["valid_radius"],
                             box=None if box is None else np.broadcast_to(box, (B, 3)))
        case["lists"] = (idx, ok)
    return case


def product_grads(case, dtype, rows=None, gf=None, gx=None):
    """Gradients of the module (autograd through egnn_layer_backward) -> {name: tensor on the device}."""
    mod = util.make_module(case, dtype).requires_grad_(True)
    ins = case["inputs"]
    t = lambda a: util.to_torch(a, dtype, DEV)
    gf = t(case["grads"][0]) if gf is None else gf
    gx = t(case["grads"][1]) if gx is None else gx
    coors = t(ins["coors"]).requires_grad_(True)
    leaves = {"in.coors": coors}
    feats = t(ins["feats"])
    if feats.is_floating_point():
        leaves["in.feats"] = feats.requires_grad_(True)
    edges = t(ins.get("edges"))
    if edges is not None:
        leaves["in.edges"] = edges.requires_grad_(True)
    kw = {} if case["box"] is None else dict(box=torch.as_tensor(case["box"], dtype=dtype, device=DEV))
    if rows is not None:
        kw["_rows"] = rows
    with torch.enable_grad():
        if case["kind"] == NW:
            fo, xo = mod(feats, coors, adj_mat=t(ins.get("adj_mat")), mask=t(ins.get("mask")), **kw)
        else:
            fo, xo = mod(feats, coors, edges, mask=t(ins.get("mask")), **kw)
        ((fo * gf).sum() + (xo * gx).sum()).backward()
    out = {k: v.grad for k, v in leaves.items()}
    for k, p in mod.named_parameters():
        assert p.grad is not None, k
        out[f"p.{k}"] = p.grad
    return out


def reference_grads(case, dtype):
    """The restatement's gradients, float64 or float32, on the device."""
    ins = case["inputs"]
    gf, gx = case["grads"]
    if case["kind"] == NW:
        return TR.network_grads(case["params"], case["ncfg"], ins["feats"], ins["coors"], gf, gx, ins.get("adj_mat"),
                                None, ins.get("mask"), case["box"], dtype=dtype, device=DEV)
    f = torch.as_tensor(ins["feats"]).to(DEV, dtype)
    idx, ok = case.get("lists", (None, None))
    if idx is not None:
        idx, ok = torch.from_numpy(idx).to(DEV), torch.from_numpy(ok).to(DEV)
    return TR.layer_grads_chunked(case["params"], case["cfg"], f, ins["coors"], gf, gx, ins.get("edges"), ins.get("mask"),
                                  None, case["box"], idx, ok)


_REF = {}


def reference(name, dt, case, dtype=torch.float64, depth=None):
    """The restatement's gradients for (case, type of its inputs), kept for the next test of the same case only."""
    key = (name, dt, depth, dtype)
    if key not in _REF:
        _REF.clear()
        torch.cuda.empty_cache()
        _REF[key] = reference_grads(case, dtype)
    return _REF[key]


def _network_margins(case, name, dt):
    """The restatement's k-th / (k+1)-th rank gap on every layer's input coordinates."""
    ncfg, ins = case["ncfg"], case["inputs"]
    k = ncfg["layer"]["num_nearest_neighbors"]
    if k == 0 or ncfg["layer"]["only_sparse_neighbors"]:
        return None
    _, _, states = TR.network(case["params"], ncfg, ins["feats"], ins["coors"], ins.get("adj_mat"), None, ins.get("mask"),
                              dtype=torch.float64, device=DEV)
    return min(TR.knn_gap(x, k, ins.get("mask")) for _, x in states)


# ------------------------------------------------------------------ gates


NODE = ("in.feats", "in.coors", "in.edges")


def _minus_cotangent(g, case):
    g = dict(g)
    gf, gx = (torch.as_tensor(a).to(DEV, torch.float64) for a in case["grads"])
    if "in.feats" in g:
        g["in.feats"] = g["in.feats"].double() - gf
    g["in.coors"] = g["in.coors"].double() - gx
    return g


def check_fp64(got, want, case, what):
    got, want = _minus_cotangent(got, case), _minus_cotangent(want, case)
    worst, bad = {}, []
    for k, w in want.items():
        e = (got[k].double() - w).abs()
        scale = float(w.abs().max())
        worst[k] = float(e.max()) / max(scale, 1e-300)
        if worst[k] > TAU64:
            bad.append(f"{k}: {worst[k]:.2e}")
        if k in NODE:
            b, n = w.shape[:2]
            rmax = w.abs().reshape(b * n, -1).amax(1).clamp_min(1e-3 * scale)
            r = float((e.reshape(b * n, -1).amax(1) / rmax).max())
            worst[k + "[row]"] = r
            if r > TAU64:
                bad.append(f"{k} per row: {r:.2e}")
    print(f"{what}: worst fp64 error {max(worst.values()):.2e} of the scale ({max(worst, key=worst.get)})")
    assert not bad, f"{what}: " + "; ".join(bad)
    return worst


def check_fp32(got, ref32, want, case, what):
    got, ref32, want = (_minus_cotangent(g, case) for g in (got, ref32, want))
    ratios, bad = {}, []
    for k, w in want.items():
        scale = float(w.abs().max())
        floor = FP32_FLOOR * scale
        ek, er = got[k].double() - w, ref32[k].double() - w
        for stat, f in (("max", lambda e: float(e.abs().max())), ("rms", lambda e: float(e.pow(2).mean().sqrt()))):
            r = f(ek) / max(f(er), floor, 1e-300)
            ratios[f"{k}.{stat}"] = r
            if r > (FP32_CHAINED_RATIO if k.endswith(FP32_CHAINED) else FP32_RATIO):
                bad.append(f"{k} {stat}: kernel {f(ek):.2e} vs restatement {f(er):.2e}")
    top = max(ratios, key=ratios.get)
    rest = {k: v for k, v in ratios.items() if not k.rsplit(".", 1)[0].endswith(FP32_CHAINED)}
    top2 = max(rest, key=rest.get)
    print(f"{what}: worst fp32 ratio {ratios[top]:.2f} ({top}); outside the chained sums {rest[top2]:.2f} ({top2})")
    assert not bad, f"{what}: " + "; ".join(bad)
    return ratios


def check_exact(got, case, dtype, what):
    mod = util.make_module(case, dtype)
    params = dict(mod.named_parameters())
    for k, v in got.items():
        assert torch.isfinite(v).all(), f"{what}: {k} is not finite"
        want_dt = params[k[2:]].dtype if k.startswith("p.") else dtype
        assert v.dtype == want_dt, (what, k, v.dtype)
    ge = got.get("in.edges")
    if ge is None:
        return
    B, N = ge.shape[:2]
    live = torch.ones(B, N, N, dtype=torch.bool, device=DEV)
    if "lists" in case:
        live = torch.zeros_like(live)
        idx = torch.from_numpy(case["lists"][0]).to(DEV)
        live.scatter_(2, idx, True)
    mk = case["inputs"].get("mask")
    if mk is not None:
        m = torch.from_numpy(mk).to(DEV)
        live &= m[:, :, None] & m[:, None, :]
    assert not live.all()
    assert (ge[~live] == 0).all(), f"{what}: edge gradient outside the selected, unmasked pairs"


def _report(what, t0):
    torch.cuda.synchronize()
    print(f"{what}: {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


# ------------------------------------------------------------------ the cases


RUNS = [("c2", "fp64"), ("c2", "fp32"), ("dense_generic", "fp64"), ("dense_generic", "fp32"), ("c4", "fp64"),
        ("c4", "fp32"), ("c4_box", "fp64"), ("c4_box", "fp32"), ("c3", "fp64"), ("c3", "fp32"), ("c5", "fp64"),
        ("c5", "fp32")]


@pytest.mark.gpu
@pytest.mark.parametrize("name,dt", RUNS, ids=[f"{n}-{d}" for n, d in RUNS])
def test_backward_matches_the_chunked_reference(name, dt):
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    dtype = DT[dt]
    depth = 1 if (name == "c3" and dt == "fp32") else None      # fp32 coordinates: no reselection on updated ones
    case = build(name, dt, depth)
    if case["kind"] == NW:
        gap = _network_margins(case, name, dt)
        if gap is not None:
            assert gap > (1e-8 if dt == "fp64" else 1e-5), f"{name}: rank gap {gap:.2e}"
            print(f"{name} [{dt}]: smallest k-th rank gap {gap:.2e}")
    got = product_grads(case, dtype)
    check_exact(got, case, dtype, f"{name} [{dt}]")
    want = reference(name, dt, case, depth=depth)
    if dt == "fp64":
        check_fp64(got, want, case, f"{name} [fp64]")
    else:
        ref32 = reference_grads(case, torch.float32)
        check_fp32(got, ref32, want, case, f"{name} [fp32]")
    _report(f"{name} [{dt}]", t0)


@pytest.mark.gpu
def test_c2_recomputed_pre2_equals_saved(monkeypatch):
    """EGNN_B200_SAVE_PAIR_MB=0: the backward recomputes W2 silu(pre1) with the register-tiled forward kernel."""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    case = build("c2", "fp64")
    saved = product_grads(case, torch.float64)
    monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")
    got = product_grads(case, torch.float64)
    for k, v in saved.items():
        assert float((got[k] - v).abs().max()) <= 1e-12 * max(1.0, float(v.abs().max())), k
    check_fp64(got, reference("c2", "fp64", case), case, "c2_recompute [fp64]")
    _report("c2_recompute [fp64]", t0)


@pytest.mark.gpu
def test_c2_row_blocks_sum_to_the_whole_gradient():
    """Row blocks (0, 333), (333, 700), (700, 1024), each with the cotangents zero outside the block."""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    case = build("c2", "fp64")
    whole = product_grads(case, torch.float64)
    gf, gx = (util.to_torch(a, torch.float64, DEV) for a in case["grads"])
    total = None
    for r0, r1 in ((0, 333), (333, 700), (700, 1024)):
        keep = torch.zeros(1, gf.shape[1], 1, dtype=torch.float64, device=DEV)
        keep[:, r0:r1] = 1
        g = product_grads(case, torch.float64, rows=(r0, r1), gf=gf * keep, gx=gx * keep)
        total = g if total is None else {k: total[k] + v for k, v in g.items()}
    for k, v in whole.items():
        err = float((total[k] - v).abs().max()) / max(1.0, float(v.abs().max()))
        assert err <= 1e-12, (k, err)
    check_fp64(total, reference("c2", "fp64", case), case, "c2_rows [fp64]")
    _report("c2_rows [fp64]", t0)
