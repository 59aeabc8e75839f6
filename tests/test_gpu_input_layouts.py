"""Every entry point on views of caller memory, against the same call on fresh contiguous copies.

Callers slice batches, broadcast masks and transpose adjacencies; the module's signature is the reference's, so each of
those views must give what the reference gives.  `place` builds each input in one of these layouts:

  canonical       a fresh contiguous copy (the form every other test passes)
  poisoned        the values as an aligned contiguous view in the middle of a larger buffer, with more poison on each
                  side than any kernel tile of that input spans (PAD_BYTES): NaN for float inputs, 1 for mask and
                  adjacency bytes, a valid but wrong node index for neighbour lists -- so a read past either end shows
                  up as a wrong value, never as an out-of-range address
  misaligned      the same with the start moved by whole elements off a 16-byte boundary, at every remainder the
                  element size allows (4 / 8 / 12 bytes for fp32, 8 for fp64, 2 .. 14 for bf16); every pointer stays
                  aligned for its element type
  batch_slice     `big[1:1 + B]` of a poisoned [B + 2, ...] tensor: contiguous, and off 16 bytes whenever one batch
                  entry is not a multiple of 16 bytes
  last_dim_slice  `big[..., 1:1 + D]` of a poisoned [..., D + 3] tensor (not contiguous)
  permuted        a contiguous tensor with its axes reversed, reversed back (not contiguous)
  expanded        a size-1 batch expanded to B with stride 0 (its own tests: the B graphs are then identical)

Gates: forward outputs are bit-identical (torch.equal) to the canonical call, and each canonical call is checked once
against the fp64 reference at the gate its path already uses (util.TOL for fp64 / fp32, test_gpu_fast's for bf16);
gradients agree with the canonical call to the backward's atomics tolerance (test_gpu_radius_select_wide) and with the
fp64 autograd reference at util.grad_tol; every input buffer, poison included, is unchanged byte for byte after forward
and backward, and no output shares storage with an input.  LAYOUT_COVERAGE lists which layouts reach which entry point;
tests/test_input_layouts_host.py holds it to the promise above."""
import contextlib

import numpy as np
import pytest
import torch

import cases
import tc_reference as TR
import torch_reference as TREF
import util
from oracle import egnn_oracle as O
from test_gpu_tile_boundaries import TILE_CASES
from tests import test_edge_list

DEV = "cuda"
L, NW = "layer", "network"
PAD_BYTES = 1 << 16          # poison on each side of an input: more than any tile of it a kernel reads (<= 32 KiB)
F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
CONTIGUOUS_FORMS = ("poisoned", "misaligned", "batch_slice")
STRIDED_FORMS = ("last_dim_slice", "permuted")
FORMS = CONTIGUOUS_FORMS + STRIDED_FORMS

# ----------------------------------------------------------------------------- layouts of caller memory


def offsets(t):
    """Element offsets that move an aligned start off a 16-byte boundary: every remainder the element size allows."""
    return list(range(1, 16 // t.element_size()))


def default_poison(t):
    return float("nan") if t.is_floating_point() else 1 if t.dtype in (torch.bool, torch.uint8) else 0


def place(t, form, i=0, poison=None):
    """-> (view, buffer): `t`'s values in layout `form` (the module docstring), and the allocation that holds them.  `i`
    picks the misaligned offset, cycling through offsets(t)."""
    t = t.to(DEV)
    poison = default_poison(t) if poison is None else poison
    full = lambda shape: torch.full(shape, poison, dtype=t.dtype, device=DEV)
    if form == "canonical":
        v = t.clone(memory_format=torch.contiguous_format)
        return v, v
    if form == "batch_slice":
        big = full((t.shape[0] + 2,) + tuple(t.shape[1:]))
        big[1:-1] = t
        return big[1:-1], big
    if form == "last_dim_slice":
        big = full(tuple(t.shape[:-1]) + (t.shape[-1] + 3,))
        big[..., 1:-2] = t
        return big[..., 1:-2], big
    if form == "permuted":
        rev = tuple(reversed(range(t.dim())))
        s = t.permute(rev).contiguous()
        return s.permute(rev), s
    assert form in ("poisoned", "misaligned"), form
    es, n = t.element_size(), t.numel()
    pad = -(-max(PAD_BYTES, n * es) // 256) * 256 // es          # a multiple of 256 bytes: the poisoned view is aligned
    off = 0 if form == "poisoned" else offsets(t)[i % len(offsets(t))]
    buf = full((2 * pad + n + 16,))
    buf[pad + off:pad + off + n] = t.reshape(-1)
    v = buf[pad + off:pad + off + n].view(t.shape)
    assert form == "poisoned" or v.data_ptr() % 16 != 0
    return v, buf


def _bytes(t):
    return t.detach().reshape(-1).view(torch.uint8)


class Caller:
    """The buffers handed to one call: checks afterwards that each is unchanged byte for byte and shares no storage with
    an output."""

    def __init__(self):
        self.bufs = []

    def place(self, t, form, i=0, poison=None):
        if t is None:
            return None
        v, buf = place(t, form, i, poison)
        self.bufs.append((buf, _bytes(buf).clone()))
        return v

    def check(self, outs, what):
        torch.cuda.synchronize()
        for buf, snap in self.bufs:
            assert torch.equal(_bytes(buf), snap), f"{what}: an input buffer was written ({tuple(buf.shape)} {buf.dtype})"
        ins = {b.untyped_storage().data_ptr() for b, _ in self.bufs}
        for o in outs:
            assert o.untyped_storage().data_ptr() not in ins, f"{what}: an output shares storage with an input"


def assert_bits(got, want, what):
    for g, w, nm in zip(got, want, ("feats", "coors")):
        assert g.shape == w.shape and g.dtype == w.dtype, (what, nm, g.shape, w.shape)
        assert torch.equal(g, w), f"{what} {nm}: max diff {(g.double() - w.double()).abs().max().item():.3e}"


@contextlib.contextmanager
def env(**kv):
    import os
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# ----------------------------------------------------------------------------- layer scenarios

CELL3 = np.array([[3.0, 0.0, 0.0], [0.5, 2.8, 0.0], [-0.4, 0.3, 3.2]])
BOX = {2: np.array([2.5, 3.0]), 3: np.array([3.0, np.inf, 2.6])}


def lists(B, N, k, seed):
    """Neighbour lists as test_edge_list builds them: distinct random nodes, two empty slots in every third row."""
    rs = np.random.RandomState(seed)
    nb = np.stack([np.stack([rs.permutation(N)[:k] for _ in range(N)]) for _ in range(B)]).astype(np.int64)
    nb[:, ::3, -2:] = -1
    return nb


# name: (source, options).  Sources: ("tile", TILE_CASES name) dense; ("list", EDGE_CASES name) caller lists; ("spec",
# spec) the layer's own select; options: lattice, slot_edges, env (select paths), k / rows for the bf16 cases.
LAYER_SCENARIOS = {
    # SIMT dense: several 32-neighbour passes with a partial last one, partial row CTAs, Hp 128 / 144 / 72
    "dense_n45_edges":    (("tile", "dense_n45_hp128"), {}),
    "dense_n70_box":      (("tile", "dense_n70_hp144"), dict(lattice="box")),
    "dense_n33_cell":     (("tile", "dense_n33_hp72"), dict(lattice="cell")),
    # SIMT lists: k = 33 (two slot passes, partial), TS 32 with C = 2 under a box, TS 4 under a cell, per-slot edges
    "list_k33":           (("list", "k33"), {}),
    "list_k17_box":       (("list", "k17_q5_c2"), dict(lattice="box")),
    "list_k3_cell":       (("list", "k3_q1"), dict(lattice="cell")),
    "list_slot_edges":    (("list", "edges_mask"), dict(slot_edges=True)),
    # the layer's own selects
    "select_knn":         (("spec", dict(kind=L, cfg=dict(dim=16, edge_dim=2, num_nearest_neighbors=8), B=2, N=70, seed=611,
                                         init="xavier", mask="padded")), {}),
    "select_sparse_adj":  (("spec", dict(kind=L, cfg=dict(dim=16, only_sparse_neighbors=True), B=2, N=37, seed=612,
                                         init="xavier", adj="random3d", mask="padded")), {}),
    "select_radius_grid": (("spec", dict(kind=L, cfg=dict(dim=16, num_nearest_neighbors=8, valid_radius=1.0), B=2, N=70,
                                         seed=613, init="xavier", mask="random")),
                           dict(env={"EGNN_B200_CELL_SELECT_MIN_N": "0"})),
    "select_knn_grid":    (("spec", dict(kind=L, cfg=dict(dim=16, num_nearest_neighbors=12), B=2, N=70, seed=614,
                                         init="xavier", mask="padded")), dict(env={"EGNN_B200_KNN_GRID_MIN_N": "0"})),
}

TC_SCENARIOS = {
    # tc_pair: N = 129 / 127 leave a partial j tile; a row range
    "tc_pair_n129":       (dict(kind=L, cfg=dict(dim=64), B=2, N=129, seed=621, init="xavier", mask="padded"), {}),
    "tc_pair_n127_rows":  (dict(kind=L, cfg=dict(dim=64, edge_dim=4), B=1, N=127, seed=622, init="xavier"),
                           dict(rows=(5, 100))),
    # tc_knn on caller lists: lean (no edge channels), edges, generic (fourier), k = 65 in 32-slot groups, per-slot edges
    "tc_knn_lean":        (dict(kind=L, cfg=dict(dim=64), B=2, N=101, seed=623, init="xavier", mask="padded"), dict(k=8)),
    "tc_knn_edges":       (dict(kind=L, cfg=dict(dim=64, edge_dim=4), B=2, N=67, seed=624, init="xavier"), dict(k=32)),
    "tc_knn_generic":     (dict(kind=L, cfg=dict(dim=64, fourier_features=2), B=1, N=75, seed=625, init="xavier",
                                mask="padded"), dict(k=7)),
    "tc_knn_k65":         (dict(kind=L, cfg=dict(dim=64), B=1, N=130, seed=626, init="xavier"), dict(k=65)),
    "tc_knn_slot_edges":  (dict(kind=L, cfg=dict(dim=64, edge_dim=2), B=2, N=45, seed=627, init="xavier", mask="padded",
                                dense_edges=False), dict(k=9, slot_edges=True)),
}


def build_scenario(name):
    """-> (case, inputs {name: float64 numpy | int numpy}, options).  inputs: feats, coors, edges, mask, adj_mat,
    neighbors, neighbor_edges, box, cell (None where absent)."""
    if name in TC_SCENARIOS:
        spec, opt = TC_SCENARIOS[name]
        src = ("tc", spec)
    else:
        src, opt = LAYER_SCENARIOS[name]
    nb = None
    if src[0] == "tile":
        case = cases.build_case(TILE_CASES[src[1]])
    elif src[0] == "list":
        case, nb = test_edge_list.build(src[1])
    else:
        case = cases.build_case(src[1])
        if "k" in opt:
            nb = lists(src[1]["B"], src[1]["N"], opt["k"], src[1]["seed"])
    ins = dict(case["inputs"])
    b, n, c = ins["coors"].shape
    slot = None
    if opt.get("slot_edges"):
        rs = np.random.RandomState(5)
        slot = rs.standard_normal((b, n, nb.shape[-1], case["cfg"]["edge_dim"]))
        ins.pop("edges", None)
    box = cell = None
    if opt.get("lattice") == "box":
        box = np.broadcast_to(BOX[c], (b, c)) * (1.0 + 0.1 * np.arange(b))[:, None]
    elif opt.get("lattice") == "cell":
        cell = np.broadcast_to(CELL3[:c, :c], (b, c, c)).copy()
    out = dict(feats=ins["feats"], coors=ins["coors"], edges=ins.get("edges"), mask=ins.get("mask"),
               adj_mat=ins.get("adj_mat"), neighbors=nb, neighbor_edges=slot, box=box, cell=cell)
    return case, out, dict(opt, select=src[0] == "spec")


def bf16_case(case, ins):
    """Parameters and float inputs rounded to bf16 (coordinates, box and cell as fp32 sees them stay bf16 values)."""
    case = dict(case, params={k: util.rounded(v, BF16) for k, v in case["params"].items()})
    ins = {k: (util.rounded(v, BF16) if k in ("feats", "coors", "edges", "neighbor_edges") else v) for k, v in ins.items()}
    return case, ins


def torch_inputs(ins, dtype):
    """numpy inputs -> tensors on the device: feats / edges in the module's type, coordinates / lattice in the
    coordinates' type, mask bool, adjacency bool, lists int32."""
    cdt = F64 if dtype == F64 else F32
    out = {}
    for k, v in ins.items():
        if v is None:
            out[k] = None
        elif k in ("mask", "adj_mat"):
            out[k] = torch.from_numpy(np.asarray(v).astype(bool)).to(DEV)
        elif k == "neighbors":
            out[k] = torch.from_numpy(np.asarray(v).astype(np.int32)).to(DEV)
        else:
            out[k] = torch.from_numpy(np.ascontiguousarray(v, np.float64)).to(DEV, cdt if k in ("coors", "box", "cell") else dtype)
    return out


def call_layer(mod, t, rows=None):
    kw = {k: t[k] for k in ("mask", "adj_mat", "neighbors", "neighbor_edges", "box", "cell") if t.get(k) is not None}
    if rows is not None:
        kw["_rows"] = rows
    return mod(t["feats"], t["coors"], t.get("edges"), **kw)


def placed_inputs(caller, t, form, i=0):
    """Every tensor input of `t` in layout `form`; lists poisoned with a valid but wrong node index (N - 1)."""
    n = t["feats"].shape[1]
    return {k: caller.place(v, form, i, poison=(n - 1) if k == "neighbors" else None) for k, v in t.items()}


def reference(case, ins, opt):
    """fp64 reference outputs of a scenario's canonical inputs: the oracle's own select for "spec" scenarios, the
    unrounded split form of tc_reference (which equals the oracle, test_gpu_tc_boundaries) for dense and list ones."""
    if opt["select"]:
        return cases.run_oracle(dict(case, inputs={k: v for k, v in ins.items() if v is not None}))
    nb = ins["neighbors"]
    slot = ins["neighbor_edges"] is not None
    return TR.tc_layer_forward(case["params"], case["cfg"], ins["feats"], ins["coors"],
                               edges=ins["neighbor_edges"] if slot else ins["edges"], mask=ins["mask"], neighbors=nb,
                               slot_edges=slot, rows=opt.get("rows"), rounding=False, box=ins["box"], cell=ins["cell"])


def check_reference(out, want, ins, dtype, opt, what):
    rows = opt.get("rows")
    got = out if rows is None else tuple(o[:, rows[0]:rows[1]] for o in out)
    if dtype != BF16:
        util.assert_close(got[0], want[0], what=f"{what} feats", **util.TOL[dtype])
        util.assert_close(got[1], want[1], what=f"{what} coors", **util.TOL[dtype])
        return
    x0 = ins["coors"] if rows is None else ins["coors"][:, rows[0]:rows[1]]
    f_err, c_err = util.max_err(got[0], want[0]), util.max_err(got[1], want[1])
    assert np.isfinite(got[0].float().cpu().numpy()).all() and np.isfinite(got[1].float().cpu().numpy()).all()
    assert f_err <= 1e-2 * max(1e-3, float(np.abs(want[0]).max())), (what, f_err)
    assert c_err <= 1e-2 * max(float(np.abs(want[1] - x0).max()), 1.0), (what, c_err)


_PATH = {F64: "fp64-simt", F32: "fp32-simt"}
SIMT_PARAMS = [(n, dt) for n in LAYER_SCENARIOS for dt in (F64, F32)] + [(n, BF16) for n in TC_SCENARIOS]


def _dt_id(dt):
    return {F64: "fp64", F32: "fp32", BF16: "bf16"}[dt]


@pytest.mark.gpu
@pytest.mark.parametrize("name,dtype", SIMT_PARAMS, ids=[f"{n}-{_dt_id(d)}" for n, d in SIMT_PARAMS])
def test_layer_forward_on_views_is_bit_identical(name, dtype):
    case, ins, opt = build_scenario(name)
    if dtype == BF16:
        case, ins = bf16_case(case, ins)
    mod = util.make_module(case, dtype)
    t = torch_inputs(ins, dtype)
    rows = opt.get("rows")
    with env(**opt.get("env", {})):
        caller = Caller()
        want = call_layer(mod, placed_inputs(caller, t, "canonical"), rows)
        caller.check(want, f"{name} canonical")
        if dtype == BF16:
            assert mod.last_path == "bf16-tc", (name, mod.last_path)
        check_reference(want, reference(case, ins, opt), ins, dtype, opt, name)
        for form in FORMS:
            for i in range(len(offsets(t["feats"])) if form == "misaligned" else 1):
                caller = Caller()
                got = call_layer(mod, placed_inputs(caller, t, form, i), rows)
                assert mod.last_path == ("bf16-tc" if dtype == BF16 else _PATH[dtype])
                what = f"{name} {form}{i if form == 'misaligned' else ''}"
                caller.check(got, what)
                assert_bits(got, want, what)


MASK_DTYPES = (torch.bool, torch.uint8, torch.int64, torch.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("name", ["select_sparse_adj", "select_knn"])
def test_mask_and_adjacency_types_and_views(name, dtype):
    """Mask and adjacency as bool, uint8, int64 and float tensors, each also as a transposed-back view."""
    case, ins, opt = build_scenario(name)
    mod = util.make_module(case, dtype)
    t = torch_inputs(ins, dtype)
    want = call_layer(mod, t)
    for mdt in MASK_DTYPES:
        for form in ("canonical", "permuted", "misaligned"):
            caller = Caller()
            v = dict(t)
            for k in ("mask", "adj_mat"):
                if t[k] is not None:
                    v[k] = caller.place(t[k].to(mdt), form, 3)
            got = call_layer(mod, v)
            caller.check(got, f"{name} {mdt} {form}")
            assert_bits(got, want, f"{name} {mdt} {form}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32, BF16], ids=["fp64", "fp32", "bf16"])
def test_expanded_size_one_batch(dtype):
    """feats, coors, mask and box of one graph expanded to B with stride 0 give the bits of their contiguous copies."""
    name = "dense_n70_box" if dtype != BF16 else "tc_pair_n129"
    case, ins, opt = build_scenario(name)
    if dtype == BF16:
        case, ins = bf16_case(case, ins)
        ins["box"] = BOX[3][None]
    B = 3
    one = {k: (None if v is None else np.asarray(v)[:1]) for k, v in ins.items()}
    mod = util.make_module(case, dtype)
    t1 = torch_inputs(one, dtype)
    expanded = {k: (None if v is None else v.expand((B,) + tuple(v.shape[1:]))) for k, v in t1.items()}
    want = call_layer(mod, {k: (None if v is None else v.contiguous()) for k, v in expanded.items()})
    got = call_layer(mod, expanded)
    assert_bits(got, want, f"{name} expanded")
    assert got[0].shape[0] == B and torch.equal(got[0][0], got[0][B - 1])


# ----------------------------------------------------------------------------- backward

GRAD_SCENARIOS = ["dense_n45_edges", "dense_n70_box", "list_k33", "list_slot_edges"]
GRAD_PARAMS = [(n, dt, m) for n in GRAD_SCENARIOS for dt in (F64, F32) for m in ("saved", "recompute")]


def grad_run(mod, t, gf, gx, leaves, make_inputs):
    """One forward + backward.  `make_inputs(leaves)` -> the layer's inputs built from the leaf tensors; the cotangents
    go in through torch.autograd.backward(grad_tensors=...) -> (outputs, {name: gradient})."""
    mod.zero_grad(set_to_none=True)
    for v in leaves.values():
        v.grad = None
    with torch.enable_grad():
        out = call_layer(mod, make_inputs(leaves))
        torch.autograd.backward(out, grad_tensors=(gf, gx))
    g = {f"leaf.{k}": v.grad for k, v in leaves.items()}
    g.update({f"p.{k}": p.grad for k, p in mod.named_parameters() if p.grad is not None})
    return tuple(o.detach() for o in out), g


def agree(got, want, dtype, what, factor=1.0):
    tol = (1e-10 if dtype == F64 else 2e-5) * factor
    for k, w in want.items():
        g = got[k]
        assert g is not None and g.shape == w.shape, (what, k)
        scale = max(1.0, float(w.abs().max()))
        err = float((g.double() - w.double()).abs().max())
        assert err <= tol * scale, f"{what} {k}: {err:.3e} (scale {scale:.3e})"


@pytest.mark.gpu
@pytest.mark.parametrize("name,dtype,mode", GRAD_PARAMS, ids=[f"{n}-{_dt_id(d)}-{m}" for n, d, m in GRAD_PARAMS])
def test_backward_on_views(name, dtype, mode, monkeypatch):
    """feats a misaligned view of a larger leaf, coors the transpose of a [B, C, N] leaf, edges a batch slice, the box a
    batch slice too; the cotangents a misaligned and a poisoned view."""
    if mode == "recompute":
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")
    case, ins, opt = build_scenario(name)
    mod = util.make_module(case, dtype)
    mod.requires_grad_(True)
    t = torch_inputs(ins, dtype)
    rs = np.random.RandomState(9)
    gf0 = torch.from_numpy(rs.standard_normal(t["feats"].shape)).to(DEV, dtype)
    gx0 = torch.from_numpy(rs.standard_normal(t["coors"].shape)).to(DEV, t["coors"].dtype)
    e_key = "neighbor_edges" if t["neighbor_edges"] is not None else "edges"

    # canonical: fresh contiguous leaves
    leaves_c = {"feats": t["feats"].clone().requires_grad_(True), "coors": t["coors"].clone().requires_grad_(True)}
    if t[e_key] is not None:
        leaves_c[e_key] = t[e_key].clone().requires_grad_(True)
    out_c, g_c = grad_run(mod, t, gf0.clone(), gx0.clone(), leaves_c, lambda lv: dict(t, **lv))

    # views: the leaves are the larger buffers
    caller = Caller()
    fv, fbuf = place(t["feats"], "misaligned", 1)
    cbuf = t["coors"].transpose(1, 2).contiguous()
    leaves_v = {"feats": fbuf.clone().requires_grad_(True), "coors": cbuf.clone().requires_grad_(True)}
    f_off = fv.data_ptr() - fbuf.data_ptr()
    f_lo = f_off // fbuf.element_size()
    if t[e_key] is not None:
        ebig = place(t[e_key], "batch_slice")[1]
        leaves_v[e_key] = ebig.clone().requires_grad_(True)
    for v in leaves_v.values():
        caller.bufs.append((v, _bytes(v).clone()))
    n_f = t["feats"].numel()

    def views(lv):
        v = dict(t, feats=lv["feats"][f_lo:f_lo + n_f].view(t["feats"].shape), coors=lv["coors"].transpose(1, 2))
        if e_key in lv:
            v[e_key] = lv[e_key][1:-1]
        for k in ("mask", "box", "neighbors"):
            if t[k] is not None:
                v[k] = caller.place(t[k], "batch_slice" if k != "neighbors" else "misaligned", 2,
                                    poison=t["feats"].shape[1] - 1 if k == "neighbors" else None)
        return v

    gf = caller.place(gf0, "misaligned", 2)
    gx = caller.place(gx0, "poisoned")
    out_v, g_v = grad_run(mod, t, gf, gx, leaves_v, views)
    caller.check(out_v, f"{name} {mode}")
    assert_bits(out_v, out_c, f"{name} {mode} forward")
    # the leaves' gradients: the views' share, zero in the poison
    gv = dict(g_v)
    gfeats = gv.pop("leaf.feats")
    assert not bool(gfeats[:f_lo].any()) and not bool(gfeats[f_lo + n_f:].any())
    gv["leaf.feats"] = gfeats[f_lo:f_lo + n_f].view(t["feats"].shape)
    gv["leaf.coors"] = gv.pop("leaf.coors").transpose(1, 2)
    if f"leaf.{e_key}" in gv:
        ge = gv.pop(f"leaf.{e_key}")
        assert not bool(ge[0].any()) and not bool(ge[-1].any())
        gv[f"leaf.{e_key}"] = ge[1:-1]
    agree(gv, g_c, dtype, f"{name} {mode} views vs canonical")
    # the canonical gradients against the fp64 autograd reference
    want = TREF.layer_grads_chunked(case["params"], case["cfg"], ins["feats"], ins["coors"], gf0.double().cpu(),
                                    gx0.double().cpu(), ins["edges"], ins["mask"], None, ins["box"], ins["neighbors"],
                                    slot_edges=ins["neighbor_edges"])
    got = {k.replace("leaf.", "in.").replace("neighbor_edges", "edges"): v.double().cpu().numpy() for k, v in g_c.items()}
    util.compare({k: got.get(k, np.zeros(v.shape)) for k, v in want.items()},
                 {k: v.numpy() for k, v in want.items()}, util.grad_tol(case, dtype), f"{name} {mode} vs reference")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
def test_backward_through_an_expanded_batch_and_a_box_view(dtype):
    """feats and coors of one graph expanded to B with stride 0 (their gradient is the batch sum), and lattice_grad=True
    with one box [C] for the batch given as a misaligned view of a larger leaf: gradients equal the contiguous call's,
    and the batch sum of the fp64 reference's."""
    case, ins, _ = build_scenario("dense_n70_box")
    B = 2
    one = {k: (None if v is None else np.asarray(v)[:1]) for k, v in ins.items()}
    one["box"] = BOX[3]
    mod = util.make_module(case, dtype)
    mod.requires_grad_(True)
    t = torch_inputs(one, dtype)
    rs = np.random.RandomState(10)
    ex = lambda v: v.expand((B,) + tuple(v.shape[1:]))
    gf = torch.from_numpy(rs.standard_normal(ex(t["feats"]).shape)).to(DEV, dtype)
    gx = torch.from_numpy(rs.standard_normal(ex(t["coors"]).shape)).to(DEV, t["coors"].dtype)
    bview, bbuf = place(t["box"], "misaligned", 1)
    b_lo = (bview.data_ptr() - bbuf.data_ptr()) // bbuf.element_size()
    c = t["box"].numel()

    def run(expanded, box_view):
        f, x = t["feats"].clone(), t["coors"].clone()
        if not expanded:
            f, x = ex(f).contiguous(), ex(x).contiguous()
        f.requires_grad_(True), x.requires_grad_(True)
        lat = (bbuf if box_view else t["box"]).clone().requires_grad_(True)
        mod.zero_grad(set_to_none=True)
        with torch.enable_grad():
            out = mod(ex(f) if expanded else f, ex(x) if expanded else x, ex(t["edges"]), mask=ex(t["mask"]),
                      box=lat[b_lo:b_lo + c] if box_view else lat, lattice_grad=True)
            torch.autograd.backward(out, grad_tensors=(gf, gx))
        g = {"in.feats": f.grad, "in.coors": x.grad, "box": lat.grad}
        g.update({f"p.{k}": p.grad for k, p in mod.named_parameters()})
        return tuple(o.detach() for o in out), g

    out_c, g_c = run(False, False)
    out_v, g_v = run(True, True)
    assert_bits(out_v, out_c, "expanded batch, box view")
    gb = g_v.pop("box")
    assert not bool(gb[:b_lo].any()) and not bool(gb[b_lo + c:].any())
    g_v["box"] = gb[b_lo:b_lo + c]
    g_c["in.feats"] = g_c["in.feats"].sum(0, keepdim=True)
    g_c["in.coors"] = g_c["in.coors"].sum(0, keepdim=True)
    agree(g_v, g_c, dtype, "expanded batch, box view", factor=10.0)
    full = {k: (None if v is None else np.broadcast_to(np.asarray(v)[:1], (B,) + np.shape(v)[1:]).copy())
            for k, v in ins.items()}
    want = TREF.layer_grads_chunked(case["params"], case["cfg"], full["feats"], full["coors"], gf.double().cpu(),
                                    gx.double().cpu(), full["edges"], full["mask"], None, BOX[3], None)
    want.pop("in.edges", None)
    want["in.feats"] = want["in.feats"].sum(0, keepdim=True)
    want["in.coors"] = want["in.coors"].sum(0, keepdim=True)
    util.compare({k: g_v[k].double().cpu().numpy() for k in want}, {k: v.numpy() for k, v in want.items()},
                 util.grad_tol(case, dtype), "expanded batch vs reference")


# ----------------------------------------------------------------------------- EGNN_Network

NET_SPECS = {
    # token ids, a mask, degree labels on dense layers
    "dense_adj":  dict(kind=NW, cfg=dict(depth=2, dim=16, num_tokens=21, num_adj_degrees=2, adj_dim=3, m_pool_method="mean",
                                         coor_weights_clamp_value=0.2), B=2, N=29, seed=631, init="xavier", mask="padded"),
    # only_sparse_neighbors with a mask: the adjacency's lists are built once and cached with the expansion
    "sparse_adj": dict(kind=NW, cfg=dict(depth=2, dim=16, num_tokens=21, num_adj_degrees=2, adj_dim=3,
                                         only_sparse_neighbors=True), B=2, N=29, seed=632, init="xavier", mask="padded"),
}


def directed_adjacency(n, b, seed):
    """A sparse directed graph with its diagonal ([N, N] for b = None, else [B, N, N]): A and A.T differ."""
    rs = np.random.RandomState(seed)
    shape = (n, n) if b is None else (b, n, n)
    a = (rs.uniform(size=shape) < 0.08) | np.eye(n, dtype=bool)
    a[..., 0, n - 1] = True
    a[..., n - 1, 0] = False
    return a


def net_oracle(case, adj):
    ins = dict(case["inputs"], adj_mat=np.asarray(adj))
    return cases.run_oracle(dict(case, inputs=ins))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("name", list(NET_SPECS))
def test_network_inputs_as_views(name, dtype):
    """Token ids (int64), mask and adjacency as views: outputs bit-identical to contiguous copies."""
    case = cases.build_case(NET_SPECS[name])
    adj = directed_adjacency(case["spec"]["N"], None, 7)
    case["inputs"]["adj_mat"] = adj
    mod = util.make_module(case, dtype)
    tok = torch.from_numpy(case["inputs"]["feats"]).to(DEV)
    x = torch.from_numpy(case["inputs"]["coors"]).to(DEV, dtype)
    m = torch.from_numpy(case["inputs"]["mask"]).to(DEV)
    a = torch.from_numpy(adj).to(DEV)
    want = mod(tok, x, adj_mat=a, mask=m)
    util.assert_close(want[0], net_oracle(case, adj)[0], what=f"{name} feats", **util.TOL[dtype])
    util.assert_close(want[1], net_oracle(case, adj)[1], what=f"{name} coors", **util.TOL[dtype])
    for form in FORMS:
        for i in range(3 if form == "misaligned" else 1):
            mod.__dict__.pop("_adj_cache", None)
            caller = Caller()
            got = mod(caller.place(tok, form, i), caller.place(x, form, i), adj_mat=caller.place(a, form, i),
                      mask=caller.place(m, form, i))
            caller.check(got, f"{name} {form}")
            assert_bits(got, want, f"{name} {form}{i}")


@pytest.mark.gpu
@pytest.mark.parametrize("batched", [False, True], ids=["unbatched", "batched"])
@pytest.mark.parametrize("name", list(NET_SPECS))
def test_network_adjacency_cache_follows_the_view(name, batched):
    """The expansion is cached per adjacency: A, then A.t() (same pointer, version and shape), then A.t().contiguous(),
    then A edited in place -- each call equals a fresh module's and the oracle on that matrix."""
    dtype = F64
    case = cases.build_case(NET_SPECS[name])
    b, n = case["spec"]["B"], case["spec"]["N"]
    A = torch.from_numpy(directed_adjacency(n, b if batched else None, 8)).to(DEV)
    T = lambda a: a.transpose(-1, -2)
    assert not torch.equal(A, T(A))
    mod = util.make_module(case, dtype)
    tok = torch.from_numpy(case["inputs"]["feats"]).to(DEV)
    x = torch.from_numpy(case["inputs"]["coors"]).to(DEV, dtype)
    m = torch.from_numpy(case["inputs"]["mask"]).to(DEV)

    def step(adj, what):
        got = mod(tok, x, adj_mat=adj, mask=m)
        fresh = util.make_module(case, dtype)(tok, x, adj_mat=adj.clone(), mask=m)
        assert_bits(got, fresh, f"{name} {what} vs a fresh module")
        a_np = adj.cpu().numpy()
        exp, lab = O.adjacency_degrees(a_np, case["ncfg"]["num_adj_degrees"], b)
        cached = mod.__dict__["_adj_cache"]
        assert np.array_equal(cached[1].cpu().numpy().astype(bool), exp), f"{what}: expanded adjacency"
        assert np.array_equal(cached[2].cpu().numpy().astype(np.int64), lab), f"{what}: degree labels"
        want = net_oracle(case, a_np)
        util.assert_close(got[0], want[0], what=f"{name} {what} feats", **util.TOL[dtype])
        util.assert_close(got[1], want[1], what=f"{name} {what} coors", **util.TOL[dtype])
        return got

    out_a = step(A, "A")
    out_t = step(T(A), "A.t()")
    assert not torch.equal(out_a[0], out_t[0])
    assert_bits(step(T(A).contiguous(), "A.t().contiguous()"), out_t, "A.t().contiguous() vs A.t()")
    with torch.no_grad():
        A[..., 1, n - 2] = ~A[..., 1, n - 2]
        A[..., n - 3, 2] = True
    step(A, "A edited in place")


# ----------------------------------------------------------------------------- GlobalLinearAttention

GA_CASES = ("n257", "cols4")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("name", GA_CASES)
def test_global_attention_inputs_as_views(name, dtype):
    """x, queries and mask as views, and as size-1 batches expanded with stride 0."""
    import test_gpu_global_attn as GA
    P, x, q, m = GA.make_case(name)
    mod = GA.make_module(name, P, dtype)
    tx = torch.from_numpy(x).to(DEV, dtype)
    tq = torch.from_numpy(q).to(DEV, dtype)
    tm = torch.from_numpy(m).to(DEV)
    want = mod(tx, tq, tm)
    GA.check(want, GA.oracle(P, x, q, m, GA.CASES[name]["heads"]), dtype, name)
    for form in FORMS:
        for i in range(3 if form == "misaligned" else 1):
            caller = Caller()
            got = mod(caller.place(tx, form, i), caller.place(tq, form, i), caller.place(tm.to(torch.uint8), form, i))
            caller.check(got, f"{name} {form}")
            assert_bits(got, want, f"{name} {form}{i}")
    B = x.shape[0]
    x1, q1, m1 = tx[:1], tq[:1], tm[:1]
    want = mod(x1.expand(B, -1, -1).contiguous(), q1.expand(B, -1, -1).contiguous(), m1.expand(B, -1).contiguous())
    for xs, qs, ms in ((x1.expand(B, -1, -1), q1.expand(B, -1, -1), m1.expand(B, -1)), (x1, q1.expand(B, -1, -1), m1)):
        caller = Caller()
        got = mod(caller.place(xs, "poisoned") if xs.shape[0] == 1 else xs, qs,
                  caller.place(ms, "misaligned") if ms.shape[0] == 1 else ms)
        caller.check(got, f"{name} expanded")
        assert_bits(got, want, f"{name} size-1 batches")


# ----------------------------------------------------------------------------- neighbour-list builders


def cloud(b, n, dtype, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn((b, n, 3), generator=g, dtype=torch.float64).to(DEV, dtype)
    m = (torch.rand((b, n), generator=g) < 0.85).to(DEV)
    return x, m


BUILDERS = [("radius_neighbors", 16), ("radius_neighbors_wide", 48), ("knn_neighbors", 12)]


@pytest.mark.gpu
@pytest.mark.parametrize("lattice", ["none", "box", "cell"])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("fn,k", BUILDERS, ids=[f for f, _ in BUILDERS])
def test_list_builders_on_views(fn, k, dtype, lattice):
    """coors, mask, box and cell as views: the lists equal the canonical call's exactly (and, without a lattice, the
    radius lists equal the all-pairs select's kept slots)."""
    import egnn_pytorch_b200 as E
    b, n = 2, 300
    x, m = cloud(b, n, dtype, 40 + k)
    lat = {}
    if lattice == "box":
        lat["box"] = torch.tensor(np.broadcast_to(BOX[3], (b, 3)).copy(), device=DEV, dtype=dtype)
    elif lattice == "cell":
        lat["cell"] = torch.tensor(np.broadcast_to(CELL3, (b, 3, 3)).copy(), device=DEV, dtype=dtype)
    cut = 1.0
    call = (lambda xs, ms, **kw: E.knn_neighbors(xs, k, mask=ms, **kw)) if fn == "knn_neighbors" else \
        (lambda xs, ms, **kw: getattr(E, fn)(xs, cut, k, mask=ms, **kw))
    want = call(x, m, **lat)
    if lattice == "none" and fn != "knn_neighbors":
        import test_gpu_radius_select as RS
        from egnn_pytorch_b200 import _native
        exp, _ = RS.expected_from_all_pairs(_native.load(), x, m, k, cut * cut)
        assert torch.equal(want, exp), f"{fn}: canonical lists differ from the all-pairs select"
    for form in FORMS:
        for i in range(len(offsets(x)) if form == "misaligned" else 1):
            caller = Caller()
            kw = {key: caller.place(v, form, i) for key, v in lat.items()}
            got = call(caller.place(x, form, i), caller.place(m, form, i), **kw)
            caller.check((got,), f"{fn} {form}")
            assert torch.equal(got, want), f"{fn} {form}{i}: {int((got != want).sum())} slots differ"


# ----------------------------------------------------------------------------- what this file covers

# entry point -> the layouts its inputs reach it in (tests/test_input_layouts_host.py checks it against the promise)
LAYOUT_COVERAGE = {
    "EGNN forward fp64/fp32 dense":      set(FORMS) | {"canonical", "expanded"},
    "EGNN forward fp64/fp32 lists":      set(FORMS) | {"canonical"},
    "EGNN forward bf16 tc_pair":         set(FORMS) | {"canonical", "expanded"},
    "EGNN forward bf16 tc_knn":          set(FORMS) | {"canonical"},
    "EGNN own selects":                  set(FORMS) | {"canonical"},
    "EGNN backward fp64/fp32":           {"canonical", "poisoned", "misaligned", "batch_slice", "permuted", "expanded"},
    "EGNN_Network":                      set(FORMS) | {"canonical"},
    "GlobalLinearAttention":             set(FORMS) | {"canonical", "expanded"},
    "radius_neighbors":                  set(FORMS) | {"canonical"},
    "radius_neighbors_wide":             set(FORMS) | {"canonical"},
    "knn_neighbors":                     set(FORMS) | {"canonical"},
}
SCENARIO_ENTRY = {n: ("EGNN forward fp64/fp32 dense" if n.startswith("dense") else "EGNN forward fp64/fp32 lists"
                      if n.startswith("list") else "EGNN own selects") for n in LAYER_SCENARIOS}
SCENARIO_ENTRY.update({n: "EGNN forward bf16 " + ("tc_pair" if "pair" in n else "tc_knn") for n in TC_SCENARIOS})
