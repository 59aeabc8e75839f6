"""Training-mode dropout on the device against the float64 restatement given the kernels' own masks.

The kernels never store a mask: forward, recompute and backward regenerate each keep/drop decision from a counter hash
of (seed, stream, element key).  tests/dropout_reference.py ports that hash and the keys, and tests/torch_reference.py
applies the resulting masks (`drop=`), so every case here compares the layer's outputs and all its gradients with an
exact reference, not with statistics or finite differences (which cannot see masks that are consistently wrong in
forward and backward, nor a keep-scale that forward and backward share).

The case table crosses the launch code's boundaries under dropout, mirrored in `geometry` and held by
test_table_covers_every_dropout_path (at 132 SMs, an H100 SXM; the GPU test repeats the node-GEMM part with the device's
SM count):
  dense edge step   2 rows per thread (PP = 2) and 1 (fp64, m_dim 24), B = 3 with a partial last row CTA, Hp = 168
                    (H = 162, not a multiple of 8) in a partial third 64-channel chunk; the hidden axis split over 9 and
                    32 CTAs for tiny graphs (hsplit)
  dense bwd2        2 channel CTAs and 2 row CTAs, each with a partial last one
  node_mlp.0        the skinny GEMM at 1, 2 and 4 columns per warp and the tiled GEMM with partial 64 x 64 tiles (dropout
                    sits in their epilogues)
  lists             TS = 1, 4, 8 and 32 slots per row group; k = 40 (two slot passes) with -1 slots; per-slot edges with a
                    neighbour listed twice; the layer's own kNN select with valid_radius and a mask; only_sparse_neighbors
                    lists with degree labels in a depth-3 EGNN_Network; a box and a cell
  row blocks        `_rows=` against the restatement's `rows=`, dense and kNN
Drop rates p = 0.1, 0.25 and 0.3, where float32(1/(1-p)) differs from the double, and p = 0.5 as a control.

Each case runs in fp64 and fp32, forward and backward, with pre2 saved by the forward and recomputed by the backward
(EGNN_B200_SAVE_PAIR_MB=0).  Gates, per tensor (the outputs minus their inputs, in.feats / in.coors minus the cotangent,
and every other gradient):
  fp64   max|got - want| <= 1e-12 max|want|
  fp32   max and RMS error against the fp64 restatement <= 4x the fp32 restatement's own with the same masks (floor 1e-7
         of the scale), 64x for the parameter gradients summed per thread in bwd1 and bwd2 (the rule of
         test_gpu_backward_at_size.py)
On the CPU: the masks of every case drop and keep units in every graph and stream it exercises, and each case fails its
fp64 gate when the restatement is given a wrong key (dropout_reference.WRONG_KEYS) or the depth-3 network's seeds in
another order.  Measured on an H100: DESIGN.md section 8."""
import contextlib
import ctypes as C
import functools
import math

import numpy as np
import pytest
import torch

import cases
import dropout_reference as DR
import launch_geometry as LG
import test_gpu_backward_at_size as BAS
import test_triclinic as TRI
import torch_reference as TR
import util

L, NW = "layer", "network"
DT = {"fp64": torch.float64, "fp32": torch.float32}
TAU64 = 1e-12
SEED = 2024                  # torch.manual_seed before every training call: the module draws its dropout seeds from it

# spec: a cases.py spec (cfg carries dropout) plus
#   lists  "knn" (the layer's own select), "edge" (caller lists, neighbors=), "slot" (caller lists, neighbor_edges=)
#   k      width of caller lists;  lattice  "box" | "cell";  rows  a row block (r0, r1) run with `_rows=`
CASES = {
    # dense: PP = 2, B = 3, N = 37 (partial last row CTA and bwd2 row CTA), H = 162 / Hp = 168, soft edges
    "dense_pp2_soft":   dict(kind=L, cfg=dict(dim=40, dropout=0.1, soft_edges=True), B=3, N=37, seed=4101,
                             init="xavier", mask="padded"),
    # dense: fp64 at one row per thread (m_dim 24: MP = 32), clamp
    "dense_pp1_mdim24": dict(kind=L, cfg=dict(dim=40, m_dim=24, dropout=0.25, coor_weights_clamp_value=1.0), B=3,
                             N=37, seed=4102, init="xavier", mask="random"),
    # tiny graphs: the hidden axis split over 9 CTAs (Hp 520); mean pooling without a mask
    "hsplit9_mean":     dict(kind=L, cfg=dict(dim=128, dropout=0.3, m_pool_method="mean"), B=1, N=40, seed=4103,
                             init="xavier"),
    # the README example / BASELINE c1 width: 32 hidden splits, node_mlp.0 on the skinny GEMM at 1 column per warp
    "hsplit32_dim512":  dict(kind=L, cfg=dict(dim=512, dropout=0.1), B=1, N=12, seed=4104, init="xavier"),
    # skinny node GEMM at 2 columns per warp (Nout = 1056 = 132 SMs x 4 warps x 2)
    "skinny2_dim528":   dict(kind=L, cfg=dict(dim=528, dropout=0.25), B=1, N=8, seed=4105, init="xavier"),
    # skinny node GEMM at 4 columns per warp in fp32; fp64 stages K = 1072 in more than 96 KiB and takes the tiled GEMM
    "skinny4_dim1056":  dict(kind=L, cfg=dict(dim=1056, dropout=0.5), B=1, N=4, seed=4106, init="xavier"),
    # lists: k = 1 (TS 1)
    "list_k1_ts1":      dict(kind=L, cfg=dict(dim=16, dropout=0.5), B=2, N=20, seed=4107, init="xavier",
                             lists="edge", k=1),
    # lists: k = 4 (TS 4), per-slot edges with a neighbour listed twice and -1 slots, mean pooling, CoorsNorm
    "slot_k4_dup":      dict(kind=L, cfg=dict(dim=16, edge_dim=2, dropout=0.1, m_pool_method="mean", norm_coors=True),
                             B=2, N=22,
                             seed=4108, init="xavier", lists="slot", k=4, dense_edges=False),
    # lists: the layer's own kNN select with valid_radius and a mask, k = 7 (TS 8)
    "knn_k7_radius":    dict(kind=L, cfg=dict(dim=16, dropout=0.25, num_nearest_neighbors=7, valid_radius=1.2),
                             B=2, N=30, seed=4109, init="xavier", mask="padded", lists="knn"),
    # lists: k = 40 (TS 32, two slot passes, two bwd2 steps), -1 slots, N = 45 (partial 16-row bwd2 CTA), clamp and
    # CoorsNorm
    "list_k40":         dict(kind=L, cfg=dict(dim=16, dropout=0.3, coor_weights_clamp_value=0.5, norm_coors=True),
                             B=2, N=45,
                             seed=4110, init="xavier", mask="random", lists="edge", k=40),
    # only_sparse_neighbors with degree labels through a depth-3 network (one seed per layer, in layer order)
    "net3_sparse_labels": dict(kind=NW, cfg=dict(depth=3, dim=16, num_adj_degrees=3, adj_dim=4, dropout=0.1,
                                                 only_sparse_neighbors=True), B=2, N=24, seed=4111, init="xavier",
                               adj="chain", mask="padded"),
    # periodic: kNN under a box and under a tilted cell
    "knn_box":          dict(kind=L, cfg=dict(dim=16, dropout=0.25, num_nearest_neighbors=8), B=2,
                             N=40, seed=4112, init="xavier", lists="knn", lattice="box"),
    "knn_cell":         dict(kind=L, cfg=dict(dim=16, dropout=0.1, num_nearest_neighbors=6, m_pool_method="mean"), B=2,
                             N=40, seed=4113, init="xavier", mask="padded", lists="knn", lattice="cell"),
    # row blocks: block rows keep their global keys
    "rows_dense":       dict(kind=L, cfg=dict(dim=24, dropout=0.1), B=2, N=40, seed=4114, init="xavier", rows=(9, 30)),
    "rows_knn":         dict(kind=L, cfg=dict(dim=16, dropout=0.3, num_nearest_neighbors=8, soft_edges=True), B=2,
                             N=45, seed=4115, init="xavier", mask="padded", lists="knn", rows=(13, 37)),
}
# CoorsNorm runs only on caller lists without self pairs: at rel = 0 the restatement's rel / max(|rel|, 1e-8) carries
# ~1e-9 of cancellation noise into in.coors (util.grad_tol), above the fp64 gate.
# fp32 ratio for the dim-1056 layer, whose edge step sums 4232 hidden channels per pair in one thread (32 splits of 132)
# where the restatement's GEMM sums in blocks: measured 6.4 on out.feats with p = 0.5 (an exact keep-scale, and the
# fp64 run of the same masks within 5e-15).
FP32_RATIO_WIDE = {"skinny4_dim1056": 16.0}


# ------------------------------------------------------------------ launch geometry (tests/launch_geometry.py)


def _layer_cfg(spec):
    return LG.layer_dims(spec["kind"], spec["cfg"])[0]


def list_width(spec):
    """k of the layer's lists (0: dense)."""
    cfg = _layer_cfg(spec)
    if spec.get("lists") in ("edge", "slot"):
        return spec["k"]
    if spec["kind"] == NW and cfg["only_sparse_neighbors"]:
        return min(spec["N"], 1 + 2 * spec["cfg"]["num_adj_degrees"])        # a chain's expanded rows
    return cfg["num_nearest_neighbors"]


def geometry(name, dt, sms=LG.H100_SMS):
    """The case's SIMT launch (launch_geometry.simt_layer) at its element size, and node_mlp.0's GEMM (launch_gemm)."""
    spec = CASES[name]
    cfg = _layer_cfg(spec)
    dim, m = cfg["dim"], cfg["m_dim"]
    B, N = spec["B"], spec["N"]
    r0, r1 = spec.get("rows", (0, N))
    es = 8 if dt == "fp64" else 4
    k = list_width(spec)
    g = LG.simt_layer(spec["kind"], spec["cfg"], B, N, k=k, rows=spec.get("rows"))
    R, PP = g["rows"], g["PP"][es]
    g.update(B=B, R=R, H=2 * g["E"], p=cfg["dropout"], rows=r0 > 0 or r1 < N,
             node=LG.launch_gemm(B * R, dim + m, 2 * dim, es, sms), PP=PP)
    if k == 0:
        g.update(row_ctas=LG.ceil_div(R, 4 * PP), partial_row_cta=R % (4 * PP) != 0, partial_bwd2_rows=g["partial_rows"])
    return g


def test_table_covers_every_dropout_path():
    """Each boundary the table is meant to reach under dropout, recomputed from the specs."""
    geo = {(n, dt): geometry(n, dt) for n in CASES for dt in DT}
    dense = {key: g for key, g in geo.items() if g["k"] == 0}
    lists = {key: g for key, g in geo.items() if g["k"] > 0}
    want = {
        "dense PP 2, B >= 3, partial last row CTA": any(g["PP"] == 2 and g["B"] >= 3 and g["partial_row_cta"]
                                                        for g in dense.values()),
        "dense PP 1 in fp64, partial last row CTA": any(dt == "fp64" and g["PP"] == 1 and g["B"] >= 3 and
                                                        g["partial_row_cta"] for (_, dt), g in dense.items()),
        "Hp > 128 in a partial last chunk, H % 8 != 0": any(g["Hp"] > 128 and g["partial_chunk"] and g["H"] % 8
                                                            for g in dense.values()),
        "bwd2: 2 channel CTAs and 2 row CTAs, partial": any(g["bwd2_ch_ctas"] == 2 and g["partial_ch_cta"] and
                                                            g["bwd2_row_ctas"] == 2 and g["partial_bwd2_rows"]
                                                            for g in dense.values()),
        "hsplit 9": any(g["hsplit"] == 9 for g in dense.values()),
        "hsplit 32": any(g["hsplit"] == 32 for g in dense.values()),
        "skinny node GEMM, 1 column": any(g["node"] == ("skinny", 1) and g.get("hsplit") == 32 for g in geo.values()),
        "skinny node GEMM, 2 columns, fp64 and fp32": {dt for (_, dt), g in geo.items() if g["node"] == ("skinny", 2)}
                                                      == {"fp64", "fp32"},
        "skinny node GEMM, 4 columns": any(g["node"] == ("skinny", 4) for g in geo.values()),
        "tiled node GEMM, partial tiles": any(g["node"] == ("tiled", True) for g in geo.values()),
        "lists TS 1, 4, 8, 32": {g["TS"] for g in lists.values()} >= {1, 4, 8, 32},
        "k 40: two slot passes, two bwd2 steps": any(g["k"] == 40 and g["slot_passes"] == 2 and g["bwd2_steps"] == 2
                                                     for g in lists.values()),
        "row blocks, dense and lists": {g["k"] > 0 for g in geo.values() if g["rows"]} == {False, True},
        "p inexact in float and a p = 0.5 control": {g["p"] for g in geo.values()} >= {0.1, 0.25, 0.3, 0.5},
    }
    missing = [k for k, v in want.items() if not v]
    assert not missing, missing
    kinds = {s.get("lists") for s in CASES.values()} | {s.get("lattice") for s in CASES.values()}
    assert kinds >= {"knn", "edge", "slot", "box", "cell"}
    opts = {k for s in CASES.values() for k, v in s["cfg"].items() if v not in (None, False, "sum")}
    assert opts >= {"soft_edges", "norm_coors", "coor_weights_clamp_value", "m_pool_method", "valid_radius",
                    "only_sparse_neighbors", "num_adj_degrees"}
    assert any(s.get("mask") and s.get("lists") == "knn" and "valid_radius" in s["cfg"] for s in CASES.values())
    for name in ("slot_k4_dup", "list_k40"):                  # -1 slots and (per-slot edges) a neighbour listed twice
        nbr = build(name, "fp64")["nbr"]
        assert (nbr < 0).any(), name
    nbr = build("slot_k4_dup", "fp64")["nbr"]
    assert (nbr[..., 0] == nbr[..., 1]).any()


# ------------------------------------------------------------------ the cases' inputs


def _caller_lists(rs, B, N, k):
    """Random lists of distinct neighbours other than the node itself; a third of the rows end in -1 slots and one slot
    in the middle of some rows is -1 too."""
    other = lambda i: (lambda p: p + (p >= i))(rs.permutation(N - 1)[:k])
    nbr = np.stack([np.stack([other(i) for i in range(N)]) for _ in range(B)]).astype(np.int64)
    if k > 1:
        tail = rs.uniform(size=(B, N)) < 1 / 3
        cut = rs.randint(1, k, size=(B, N))
        nbr[tail[..., None] & (np.arange(k) >= cut[..., None])] = -1
        if k > 8:
            nbr[rs.uniform(size=(B, N)) < 0.2, k // 2] = -1
    return nbr


@functools.lru_cache(maxsize=None)
def build(name, dt):
    """The case with its parameters and float inputs in the layer's type (the fp64 restatement then differentiates what
    the kernels see), its cotangents, caller lists, lattice and the lists of its select."""
    spec = dict(CASES[name])
    case = cases.build_case(spec)
    dtype = DT[dt]
    rs = np.random.RandomState(spec["seed"] + 11)
    B, N = spec["B"], spec["N"]
    out = dict(case=case, nbr=None, slot_edges=None, box=None, cell=None)
    if spec.get("lists") in ("edge", "slot"):
        nbr = _caller_lists(rs, B, N, spec["k"])
        if spec["lists"] == "slot":
            dup = rs.uniform(size=(B, N)) < 0.5           # slot 1 repeats slot 0's neighbour: two slots, one mask
            nbr[..., 1] = np.where(dup & (nbr[..., 1] >= 0), nbr[..., 0], nbr[..., 1])
            out["slot_edges"] = rs.standard_normal((B, N, spec["k"], spec["cfg"]["edge_dim"]))
        out["nbr"] = nbr
    if spec.get("lattice"):
        cell = TRI.make_cell("tilt", B, rs)
        if spec["lattice"] == "box":
            cell = np.diag(np.diag(cell))
        case["inputs"]["coors"] = TRI.cell_coors(rs, B, N, cell, dtype=torch.float32)
        out["box" if spec["lattice"] == "box" else "cell"] = np.diag(cell).copy() if spec["lattice"] == "box" else cell
    case["params"] = {k: util.rounded(v, dtype) for k, v in case["params"].items()}
    case["inputs"] = {k: util.rounded(v, dtype) for k, v in case["inputs"].items()}
    if out["slot_edges"] is not None:
        out["slot_edges"] = util.rounded(out["slot_edges"], dtype)
    gf, gx = cases.upstream_grads(case)
    if spec.get("rows"):
        r0, r1 = spec["rows"]
        keep = ((np.arange(N) >= r0) & (np.arange(N) < r1))[None, :, None]
        gf, gx = gf * keep, gx * keep
    out["grads"] = (util.rounded(gf, dtype), util.rounded(gx, dtype))
    if spec.get("lists") == "knn":
        out["sel"] = _select(case, out)
    return out


@contextlib.contextmanager
def _geometry(b):
    """torch_reference with the case's lattice: a cell is read by its sequential wrap."""
    with (TRI._cell_geometry() if b["cell"] is not None else contextlib.nullcontext()):
        yield b["box"] if b["cell"] is None else b["cell"]


def _select(case, b):
    """The layer's select restated in float64 -> (idx, ok); asserts that the k-th and (k+1)-th ranks and valid_radius
    are far enough from every distance for the fp32 kernels to select the same lists."""
    cfg, ins = case["cfg"], case["inputs"]
    x = torch.as_tensor(ins["coors"])
    mask = ins.get("mask")
    with _geometry(b) as lat:
        rel = x[:, :, None] - x[:, None]
        if lat is not None:
            rel = TR.wrap(rel, TR.box_bc(TR._like(lat, x), x.shape[0], x.shape[-1])[:, None, None, :])
        dist = (rel ** 2).sum(-1)
        gap = TR.knn_gap(x, cfg["num_nearest_neighbors"], mask, lat)
    assert gap > 1e-4, gap
    idx, ok = TR.select(cfg, dist, mask, None)
    vr = cfg["valid_radius"]
    if math.isfinite(vr):
        d = torch.gather(dist, -1, idx)
        assert float(((d - vr).abs() / vr).min()) > 1e-4
        assert ok.any() and not ok.all()
    return idx.numpy(), ok.numpy()


# ------------------------------------------------------------------ the restatement


def drops(name, wrong=None, order=None):
    """The Drop of every layer call after torch.manual_seed(SEED).  `order`: the seeds handed out in another order."""
    spec = CASES[name]
    n = spec["cfg"]["depth"] if spec["kind"] == NW else 1
    seeds = DR.module_seeds(SEED, n)
    if order is not None:
        seeds = [seeds[i] for i in order]
    return [DR.Drop(spec["cfg"]["dropout"], s, wrong) for s in seeds]


def reference(name, dt, dtype=torch.float64, device="cpu", drop=None):
    """Outputs and gradients of the restatement with the kernels' masks -> {name: float64 tensor}: 'out.feats' /
    'out.coors' (the outputs of the case's rows), 'in.*' and 'p.<state-dict key>'."""
    spec, b = CASES[name], build(name, dt)
    case = b["case"]
    ins, cfg = case["inputs"], case.get("cfg")
    drop = drops(name) if drop is None else drop
    gf, gx = (torch.as_tensor(g).to(device, dtype) for g in b["grads"])
    with torch.enable_grad(), util.no_tf32():
        if spec["kind"] == NW:
            g = TR.network_grads(case["params"], case["ncfg"], ins["feats"], ins["coors"], gf, gx, ins.get("adj_mat"),
                                 None, ins.get("mask"), dtype=dtype, device=device, drop=drop)
            h, x, _ = TR.network(case["params"], case["ncfg"], ins["feats"], ins["coors"], ins.get("adj_mat"), None,
                                 ins.get("mask"), dtype=dtype, device=device, drop=drop)
            out = {"out.feats": h, "out.coors": x}
        else:
            leaf = lambda a: torch.as_tensor(a).to(device, dtype).requires_grad_(True)
            P = {k: leaf(v) for k, v in case["params"].items()}
            f, x = leaf(ins["feats"]), leaf(ins["coors"])
            e = None if ins.get("edges") is None else leaf(ins["edges"])
            se = None if b["slot_edges"] is None else leaf(b["slot_edges"])
            nbr, ok = b["nbr"], None
            if spec.get("lists") == "knn":
                nbr, ok = b["sel"]
            nbr = None if nbr is None else torch.from_numpy(nbr).to(device)
            ok = None if ok is None else torch.from_numpy(ok).to(device)
            rows = spec.get("rows")
            r0, r1 = rows or (0, spec["N"])
            with _geometry(b) as lat:
                fo, xo = TR.layer(P, cfg, f, x, e, ins.get("mask"), None, lat, nbr, se, ok, rows=rows, drop=drop[0])
            ((fo * gf[:, r0:r1]).sum() + (xo * gx[:, r0:r1]).sum()).backward()
            g = {"in.feats": f.grad, "in.coors": x.grad}
            if e is not None or se is not None:
                g["in.edges"] = (e if e is not None else se).grad
            g.update({f"p.{k}": (torch.zeros_like(v) if v.grad is None else v.grad) for k, v in P.items()})
            out = {"out.feats": fo, "out.coors": xo}
    out.update(g)
    return {k: v.detach().double() for k, v in out.items()}


def _minus_inputs(t, name, dt, device):
    """Outputs minus their inputs and input gradients minus the cotangents: the identity paths are exact and would
    only dilute the scale."""
    spec, b = CASES[name], build(name, dt)
    ins = b["case"]["inputs"]
    r0, r1 = spec.get("rows") or (0, spec["N"])
    t = dict(t)
    gf, gx = (torch.as_tensor(g, dtype=torch.float64, device=device) for g in b["grads"])
    if spec["kind"] == L:
        t["out.feats"] = t["out.feats"] - torch.as_tensor(ins["feats"], device=device)[:, r0:r1]
        t["in.feats"] = t["in.feats"] - gf
    t["out.coors"] = t["out.coors"] - torch.as_tensor(ins["coors"], device=device)[:, r0:r1]
    t["in.coors"] = t["in.coors"] - gx
    return t


def fp64_errors(got, want):
    """Per tensor max|got - want| / max|want|."""
    return {k: float((got[k].to(w.device) - w).abs().max()) / max(float(w.abs().max()), 1e-300) for k, w in want.items()}


def check_fp64(got, want, what):
    err = fp64_errors(got, want)
    worst = max(err, key=err.get)
    print(f"{what}: worst fp64 error {err[worst]:.2e} of the scale ({worst})")
    bad = [f"{k}: {v:.2e}" for k, v in err.items() if not v <= TAU64]
    assert not bad, f"{what}: " + "; ".join(bad)
    return err[worst]


def check_fp32(got, ref32, want, what, ratio=BAS.FP32_RATIO):
    ratios, bad = {}, []
    for k, w in want.items():
        scale = float(w.abs().max())
        floor = BAS.FP32_FLOOR * scale
        ek, er = got[k].to(w.device) - w, ref32[k].to(w.device) - w
        for stat, f in (("max", lambda e: float(e.abs().max())), ("rms", lambda e: float(e.pow(2).mean().sqrt()))):
            r = f(ek) / max(f(er), floor, 1e-300)
            ratios[f"{k}.{stat}"] = r
            if not r <= max(ratio, BAS.FP32_CHAINED_RATIO if k.endswith(BAS.FP32_CHAINED) else 0.0):
                bad.append(f"{k} {stat}: kernel {f(ek):.2e} vs restatement {f(er):.2e}")
    top = max(ratios, key=ratios.get)
    print(f"{what}: worst fp32 ratio {ratios[top]:.2f} ({top})")
    assert not bad, f"{what}: " + "; ".join(bad)
    return ratios[top]


# ------------------------------------------------------------------ CPU: the masks bite, and wrong keys fail


def streams(name):
    cfg = _layer_cfg(CASES[name])
    return {0} | ({1} if cfg["update_coors"] else set()) | ({2} if cfg["update_feats"] else set())


def applicable_wrong_keys(name):
    """The mistakes of dropout_reference.WRONG_KEYS that change this case's masks."""
    spec, g = CASES[name], geometry(name, "fp64")
    out = ["chunk-local h"] if g["H"] > 64 else []
    if g["H"] % 8:
        out.append("H for Hp")
    if spec["B"] > 1:
        out.append("no b")
    if spec.get("rows", (0,))[0] > 0:
        out.append("block-local rows")
    if g["k"] > 0:
        out.append("slot for j")
    if DR.keep_scale(g["p"], torch.float32) != DR.keep_scale(g["p"], torch.float64):
        out.append("float keep-scale")
    return out


def test_wrong_keys_cover_the_table():
    have = {w for n in CASES for w in applicable_wrong_keys(n)}
    assert have == set(DR.WRONG_KEYS), set(DR.WRONG_KEYS) - have
    assert not any("float keep-scale" in applicable_wrong_keys(n) for n in CASES if CASES[n]["cfg"]["dropout"] == 0.5)


@functools.lru_cache(maxsize=None)
def _cpu_reference(name):
    ds = drops(name)
    want = _minus_inputs(reference(name, "fp64", drop=ds), name, "fp64", "cpu")
    return want, ds


@pytest.mark.parametrize("name", list(CASES))
def test_masks_drop_and_keep_in_every_graph_and_stream(name):
    _, ds = _cpu_reference(name)
    for d in ds:
        assert set(d.seen) == streams(name), (name, sorted(d.seen))
        for stream, counts in d.seen.items():
            assert (counts > 0).all(), (name, stream, counts)
            rate = counts[:, 0].sum() / counts.sum()
            assert abs(rate - d.p) < 0.1, (name, stream, rate)


@pytest.mark.parametrize("name", list(CASES))
def test_a_wrong_key_fails_the_fp64_gate(name):
    """The restatement under each applicable wrong key misses the right one by more than the fp64 gate on at least one
    tensor (a wrong mask by far more than the fp32 gates): a kernel with that mistake fails this case."""
    want, _ = _cpu_reference(name)
    mistakes = [(w, drops(name, wrong=w)) for w in applicable_wrong_keys(name)]
    if CASES[name]["kind"] == NW:
        mistakes.append(("seeds in reverse layer order", drops(name, order=[2, 1, 0])))
    assert mistakes
    for what, ds in mistakes:
        got = _minus_inputs(reference(name, "fp64", drop=ds), name, "fp64", "cpu")
        worst = max(fp64_errors(got, want).values())
        assert worst > (10 * TAU64 if what == "float keep-scale" else 1e-4), (name, what, worst)


# ------------------------------------------------------------------ GPU


def _sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@pytest.mark.gpu
def test_node_gemm_paths_on_this_device():
    """The skinny GEMM's column count follows the device's SM count: the 1, 2 and 4 column cases must take them here."""
    sms = _sm_count()
    assert geometry("hsplit32_dim512", "fp64", sms)["node"] == ("skinny", 1)
    assert geometry("skinny2_dim528", "fp64", sms)["node"] == ("skinny", 2)
    assert geometry("skinny4_dim1056", "fp32", sms)["node"] == ("skinny", 4)
    assert geometry("skinny4_dim1056", "fp64", sms)["node"][0] == "tiled"


def product(name, dt):
    """Training forward + backward of the module after torch.manual_seed(SEED) -> {name: float64 tensor}."""
    spec, b = CASES[name], build(name, dt)
    case, dtype, dev = b["case"], DT[dt], "cuda"
    ins = case["inputs"]
    t = lambda a: util.to_torch(a, dtype, dev)
    mod = util.make_module(case, dtype).requires_grad_(True).train()
    gf, gx = t(b["grads"][0]), t(b["grads"][1])
    leaves = {"in.coors": t(ins["coors"]).requires_grad_(True), "in.feats": t(ins["feats"]).requires_grad_(True)}
    edges = t(ins.get("edges")) if b["slot_edges"] is None else t(b["slot_edges"])
    if edges is not None:
        leaves["in.edges"] = edges.requires_grad_(True)
    mask = t(ins.get("mask"))
    kw = {}
    if b["box"] is not None:
        kw["box"] = torch.as_tensor(b["box"], dtype=dtype, device=dev)
    if b["cell"] is not None:
        kw["cell"] = torch.as_tensor(b["cell"], dtype=dtype, device=dev)
    r0, r1 = spec.get("rows") or (0, spec["N"])
    with torch.enable_grad():
        torch.manual_seed(SEED)
        if spec["kind"] == NW:
            fo, xo = mod(leaves["in.feats"], leaves["in.coors"], adj_mat=t(ins["adj_mat"]), mask=mask)
        else:
            if spec.get("rows"):
                kw["_rows"] = spec["rows"]
            if b["nbr"] is not None:
                kw["neighbors"] = torch.from_numpy(b["nbr"]).to(dev)
            if b["slot_edges"] is not None:
                kw["neighbor_edges"] = edges
                edges = None
            fo, xo = mod(leaves["in.feats"], leaves["in.coors"], edges, mask=mask, **kw)
        ((fo * gf).sum() + (xo * gx).sum()).backward()
    out = {"out.feats": fo[:, r0:r1], "out.coors": xo[:, r0:r1]}
    out.update({k: v.grad for k, v in leaves.items()})
    out.update({f"p.{k}": p.grad for k, p in mod.named_parameters()})
    assert all(v is not None and torch.isfinite(v).all() for v in out.values()), name
    return {k: v.detach().double() for k, v in out.items()}


_REF = {}


def _gpu_reference(name, dt, dtype):
    key = (name, dt, dtype)
    if key not in _REF:
        if len(_REF) > 2:
            _REF.clear()
        _REF[key] = _minus_inputs(reference(name, dt, dtype, "cuda"), name, dt, "cuda")
    return _REF[key]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["saved", "recompute"])
@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("name", list(CASES))
def test_training_matches_the_exact_mask_reference(name, dt, mode, monkeypatch):
    """Forward outputs and every gradient, with W2 silu(pre1) saved by the forward or recomputed by the backward."""
    if mode == "recompute":
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")
    got = _minus_inputs(product(name, dt), name, dt, "cuda")
    want = _gpu_reference(name, dt, torch.float64)
    assert set(got) == set(want), sorted(set(got) ^ set(want))
    if dt == "fp64":
        check_fp64(got, want, f"{name} [fp64, {mode}]")
    else:
        check_fp32(got, _gpu_reference(name, dt, torch.float32), want, f"{name} [fp32, {mode}]",
                   FP32_RATIO_WIDE.get(name, BAS.FP32_RATIO))


@pytest.mark.gpu
@pytest.mark.parametrize("name,dt", [("dense_pp2_soft", "fp64"), ("list_k40", "fp32")])
def test_c_abi_forward_with_an_explicit_dropout_seed(name, dt):
    """egnn_layer_forward called directly with dropout_p and dropout_seed in the descriptor: the masks are a function of
    the seed alone."""
    from egnn_pytorch_b200 import _native as nat
    spec, b = CASES[name], build(name, dt)
    case, dtype = b["case"], DT[dt]
    ins = case["inputs"]
    lib = nat.load()
    mod = util.make_module(case, dtype)
    with torch.no_grad():
        util.run_module(mod, case, dtype, **({} if b["nbr"] is None else {"neighbors": torch.from_numpy(b["nbr"]).cuda()}))
    st = mod._staged(torch.device("cuda", 0), dtype)
    packed = next(iter(st["packed"].values()))
    B, N, d = ins["feats"].shape
    k = 0 if b["nbr"] is None else b["nbr"].shape[-1]
    seed = 0x1234_5678_9ABC_DEF
    desc = nat.LayerDesc(abi_version=nat.ABI_VERSION, dtype=nat.DTYPE_F64 if dt == "fp64" else nat.DTYPE_F32, B=B, N=N,
                         C=3, dim=d, edge_dim=0, label_dim=0, num_labels=0, m_dim=mod.m_dim, fourier=0, k=k,
                         flags=mod._flags(), valid_radius=float("inf"),
                         clamp=float(mod.coor_weights_clamp_value or 0.0), row_begin=0, row_end=0, reserved=0,
                         dropout_p=spec["cfg"]["dropout"], dropout_seed=seed)
    w = nat.LayerWeights(**{f: (st["tensors"][f].data_ptr() if f in st["tensors"] else None) for f in nat.WEIGHT_FIELDS})
    t = lambda a: util.to_torch(a, dtype, "cuda").contiguous()
    f, x = t(ins["feats"]), t(ins["coors"])
    m = None if ins.get("mask") is None else torch.from_numpy(ins["mask"]).to("cuda", torch.uint8)
    nbr = None if b["nbr"] is None else torch.from_numpy(b["nbr"]).to("cuda", torch.int32).contiguous()
    fo, xo = torch.empty_like(f), torch.empty_like(x)
    io = nat.LayerIO(feats=f.data_ptr(), coors=x.data_ptr(), edges=None, edge_labels=None,
                     mask=None if m is None else m.data_ptr(), adj=None, feats_out=fo.data_ptr(), coors_out=xo.data_ptr(),
                     nbr_idx=None if nbr is None else nbr.data_ptr(), pre2_out=None)
    nb = C.c_size_t()
    nat.check("egnn_layer_workspace_bytes", lib.egnn_layer_workspace_bytes(C.byref(desc), C.byref(nb)))
    ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    nat.check("egnn_layer_forward", lib.egnn_layer_forward(C.byref(desc), C.byref(w), C.c_void_p(packed.data_ptr()),
                                                           C.byref(io), C.c_void_p(ws.data_ptr()), ws.numel(), stream))
    want = reference(name, dt, dtype, "cuda", drop=[DR.Drop(spec["cfg"]["dropout"], seed)])
    got = {"out.feats": fo.double(), "out.coors": xo.double()}
    want = {k: want[k] for k in got}
    if dt == "fp64":
        check_fp64(got, want, f"{name} C ABI [fp64]")
    else:
        ref32 = reference(name, dt, torch.float32, "cuda", drop=[DR.Drop(spec["cfg"]["dropout"], seed)])
        check_fp32(got, {k: ref32[k] for k in got}, want, f"{name} C ABI [fp32]")


# ------------------------------------------------------------------ CUDA graphs refuse live dropout


def test_graphed_forward_refuses_a_module_with_live_dropout():
    """Checked before anything is cloned, warmed up or captured (so on any device)."""
    from egnn_pytorch_b200 import EGNN, EGNN_Network, GraphedForward
    f, x = torch.randn(1, 6, 8), torch.randn(1, 6, 3)
    with pytest.raises(ValueError, match="layers.1.1 applies dropout"):
        GraphedForward(EGNN_Network(depth=2, dim=8, dropout=0.1), f, x)
    with pytest.raises(ValueError, match="EGNN applies dropout"):
        GraphedForward(EGNN(dim=8, dropout=0.25), f, x)


@pytest.mark.gpu
def test_graphed_forward_refuses_to_replay_after_dropout_is_switched_on():
    from egnn_pytorch_b200 import EGNN_Network, GraphedForward
    net = EGNN_Network(depth=2, dim=8, dropout=0.1).cuda().eval()
    f, x = torch.randn(1, 6, 8, device="cuda"), torch.randn(1, 6, 3, device="cuda")
    fast = GraphedForward(net, f, x)
    before = fast(f, x)[0].clone()
    net.layers[1][1].train()
    with pytest.raises(ValueError, match="layers.1.1 applies dropout"):
        fast(f + 1, x)
    assert torch.equal(fast.static_in[0], f)          # refused before the inputs were copied in
    net.eval()
    assert torch.equal(fast(f, x)[0], before)


# ------------------------------------------------------------------ the hash's statistics (on the port)

KEYS = np.arange(1 << 20, dtype=np.int64) * 7 + 3         # a spread of element keys


@pytest.mark.parametrize("p", [1e-3, 0.1, 0.5, 0.9])
def test_drop_rate_is_p(p):
    rate = 1.0 - DR.keep(p, 0x5EED, 0, KEYS).mean()
    assert abs(rate - p) < 5 * math.sqrt(p * (1 - p) / KEYS.size), (p, rate)
    assert DR.threshold(p) == int(p * 2 ** 32)


def _corr(a, b):
    return float(np.corrcoef(a.astype(np.float64), b.astype(np.float64))[0, 1])


def test_masks_are_uncorrelated_across_streams_indices_graphs_and_seeds():
    """Pearson correlation of the keep decisions at p = 0.5 within 6 / sqrt(n) of 0 for: two streams at the same key,
    neighbouring keys, the same element of the next graph (dense edge keys of B = 4, N = 64, Hp = 168), and two
    seeds; and the high hash bits are uniform."""
    p, seed, n = 0.5, 0x1234ABCD, KEYS.size
    lim = 6 / math.sqrt(n)
    k = lambda s=seed, st=0, idx=KEYS: DR.keep(p, s, st, idx)
    assert abs(_corr(k(st=0), k(st=1))) < lim
    assert abs(_corr(k(st=1), k(st=2))) < lim
    assert abs(_corr(k(idx=KEYS), k(idx=KEYS + 1))) < lim
    assert abs(_corr(k(), k(s=seed + 1))) < lim
    N, Hp = 64, 168
    graph = N * N * Hp
    idx = np.arange(graph, dtype=np.int64)
    assert abs(_corr(k(idx=idx), k(idx=idx + graph))) < 6 / math.sqrt(graph)
    hist = np.bincount((DR.hash_hi(seed, 0, KEYS) >> np.uint64(28)).astype(np.int64), minlength=16)
    assert abs(hist / n - 1 / 16).max() < 6 * math.sqrt(1 / 16 / n)


def test_module_seeds_are_the_modules_draws():
    """module_seeds reproduces the draw sequence of torch.randint(0, 2**62, (1,)) after torch.manual_seed."""
    torch.manual_seed(SEED)
    want = [int(torch.randint(0, 2 ** 62, (1,)).item()) for _ in range(3)]
    assert DR.module_seeds(SEED, 3) == want
    assert len(set(want)) == 3
