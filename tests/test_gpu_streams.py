"""Every entry point on a side stream, and the module caches that one stream builds and another reuses.

The library enqueues all its work on the caller's stream and never synchronises; the Python modules keep device state
between calls (staged and packed parameters, `EGNN_Network`'s expanded adjacency, degree labels and neighbour lists,
`GlobalLinearAttention`'s staged parameters) that one call writes on its stream and a later call may read on another.

  A  side stream      inputs made on the default stream hold poison until a fresh stream, behind a ~50 ms sleep, copies
                      the real values in and calls: any work not ordered on that stream reads poison.  Forward outputs
                      equal the default stream's bit for bit, gradients within util.grad_tol (atomics), and one case of
                      each path meets its existing reference (the fp64 oracle, torch_reference, tc_reference, the
                      dropout restatement, the all-pairs select).
  B  read before      stream A builds a cache entry behind a sleep; stream B reuses it at once, with no wait.  A's call
     write            draws its memory from a private pool whose every byte is poison, and the test checks on the host
                      that the entry's tensors lie in that memory before B's call is issued (otherwise it fails as
                      inconclusive): a read that is not ordered after A's writes sees poison, never stale good values.
  C  free while       A builds an entry from a private pool; B reads it behind a sleep; A replaces it (parameters
     in use           updated in place, a new adjacency of the same shape) and then takes every free block of that pool,
                      filled with poison.  None of them may be a block of the old entry, and B's outputs must be those
                      of the old weights / adjacency.  Nothing but that poison is ever written to a block freed early.

Poison is always valid but wrong, so a library that mis-orders computes a wrong answer and never reads out of bounds:
0xFF bytes (NaN) for floating-point data, -1 for neighbour indices, 0 for masks, adjacency, degree labels and tokens.
The adjacency cases of B poison the pool with 0 bytes, the one value valid for everything the network's call allocates
there (labels, adjacency, list slots: node 0).  Calling one module from several host threads at once is not covered."""
import contextlib
import time

import numpy as np
import pytest
import torch

import cases
import test_gpu_global_attn as GA
import test_gpu_input_layouts as IL
import torch_reference as TREF
import util
from test_gpu_tile_boundaries import TILE_CASES

pytestmark = pytest.mark.gpu

DEV = "cuda"
L, NW = "layer", "network"
F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
SLEEP = 100_000_000          # cycles of torch.cuda._sleep: ~50 ms on an H100, far longer than any call below takes
SEGMENT = 1 << 20            # the largest block the caching allocator carves from its 2 MiB small segments
_POOLS = []                  # private pools stay alive for the session: module caches may still hold their blocks


@pytest.fixture(autouse=True)
def _time_and_peak_memory(request):
    """Prints each test's run time and peak device memory (visible with -s)."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n{request.node.name}: {time.perf_counter() - t0:.2f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def _dt_id(dt):
    return {F64: "fp64", F32: "fp32", BF16: "bf16"}[dt]


# ----------------------------------------------------------------------------- A: a side stream behind a sleep


def poisoned_like(key, v):
    if not torch.is_tensor(v):
        return v
    if v.is_floating_point():
        return torch.full_like(v, float("nan"))
    return torch.full_like(v, -1 if key == "neighbors" else 0)


def on_side_stream(real, fn):
    """`fn(inputs)` on a fresh stream behind a sleep, its inputs copied there from `real` into buffers that hold poison
    until then -> fn's result, after a device synchronise."""
    bufs = {k: poisoned_like(k, v) for k, v in real.items()}
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    assert s.cuda_stream != torch.cuda.current_stream().cuda_stream
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP)
        for k, v in real.items():
            if torch.is_tensor(v):
                bufs[k].copy_(v)
        out = fn(bufs)
    torch.cuda.synchronize()
    return out


# name: (source, options), as test_gpu_input_layouts.LAYER_SCENARIOS: the paths that file does not already name
EXTRA_SCENARIOS = {
    "dense_rows":         (("tile", "dense_n45_hp128"), dict(rows=(5, 40))),
    "select_radius_wide": (("spec", dict(kind=L, cfg=dict(dim=16, num_nearest_neighbors=40, valid_radius=1.0), B=2, N=70,
                                         seed=615, init="xavier", mask="random")),
                           dict(env={"EGNN_B200_CELL_SELECT_MIN_N": "0"})),
}


def build(name):
    if name not in EXTRA_SCENARIOS:
        return IL.build_scenario(name)
    (kind, arg), opt = EXTRA_SCENARIOS[name]
    case = cases.build_case(TILE_CASES[arg] if kind == "tile" else arg)
    ins = case["inputs"]
    out = dict(feats=ins["feats"], coors=ins["coors"], edges=ins.get("edges"), mask=ins.get("mask"),
               adj_mat=ins.get("adj_mat"), neighbors=None, neighbor_edges=None, box=None, cell=None)
    return case, out, dict(opt, select=kind == "spec")


# dense, the all-pairs kNN select, the kNN grid, the radius cell grid (k <= 32 and k > 32), caller lists with per-slot
# edges, a box, a cell, a row range
PATHS = ["dense_n45_edges", "select_knn", "select_knn_grid", "select_radius_grid", "select_radius_wide", "list_slot_edges",
         "dense_n70_box", "dense_n33_cell", "dense_rows"]
BF16_PATHS = ["tc_pair_n129", "tc_pair_n127_rows", "tc_knn_slot_edges", "select_knn", "select_knn_grid",
              "select_radius_grid", "select_radius_wide", "dense_n70_box", "dense_n33_cell"]
FWD_PARAMS = [(n, dt) for n in PATHS for dt in (F64, F32)] + [(n, BF16) for n in BF16_PATHS]


@pytest.mark.parametrize("name,dtype", FWD_PARAMS, ids=[f"{n}-{_dt_id(d)}" for n, d in FWD_PARAMS])
def test_layer_forward_on_a_side_stream(name, dtype):
    """A fresh module's first call on a side stream: its staging, packing, selects and edge kernels all there."""
    case, ins, opt = build(name)
    if dtype == BF16:
        case, ins = IL.bf16_case(case, ins)
    t = IL.torch_inputs(ins, dtype)
    rows = opt.get("rows")
    with IL.env(**opt.get("env", {})):
        want = IL.call_layer(util.make_module(case, dtype), t, rows)
        mod = util.make_module(case, dtype)
        got = on_side_stream(t, lambda v: IL.call_layer(mod, v, rows))
        IL.assert_bits(got, want, f"{name} side stream")
        if dtype != BF16 or name in IL.TC_SCENARIOS:
            IL.check_reference(got, IL.reference(case, ins, opt), ins, dtype, opt, name)


@pytest.mark.parametrize("dtype", [F64, F32, BF16], ids=["fp64", "fp32", "bf16"])
def test_training_dropout_on_a_side_stream(dtype):
    """Training-mode dropout with the same seed on both streams: the same masks, the same bits."""
    case = cases.build_case(dict(kind=L, cfg=dict(dim=24, edge_dim=2, dropout=0.25), B=2, N=33, seed=651, init="xavier",
                                 mask="padded"))
    ins = case["inputs"]
    t = IL.torch_inputs(dict(feats=ins["feats"], coors=ins["coors"], edges=ins["edges"], mask=ins["mask"]), dtype)

    def run(mod, v):
        torch.manual_seed(7)
        return mod(v["feats"], v["coors"], v["edges"], mask=v["mask"])

    want = run(util.make_module(case, dtype).train(), t)
    mod = util.make_module(case, dtype).train()
    got = on_side_stream(t, lambda v: run(mod, v))
    IL.assert_bits(got, want, "dropout side stream")
    assert not torch.equal(want[0], run(util.make_module(case, dtype).eval(), t)[0])


def test_training_dropout_on_a_side_stream_matches_the_mask_reference():
    """The dropout path's own exact reference (forward and every gradient), with the case built and run on a side
    stream behind a sleep."""
    import test_gpu_dropout_reference as DROP
    name = "dense_pp2_soft"
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP)
        got = DROP.product(name, "fp64")
    torch.cuda.synchronize()
    want = DROP._minus_inputs(DROP.reference(name, "fp64", torch.float64, "cuda"), name, "fp64", "cuda")
    DROP.check_fp64(DROP._minus_inputs(got, name, "fp64", "cuda"), want, f"{name} side stream")


def _layer_grads(mod, v, e_key, lattice_grad):
    leaves = {"feats": v["feats"], "coors": v["coors"]}
    if v.get(e_key) is not None:
        leaves[e_key] = v[e_key]
    if lattice_grad:
        leaves["box"] = v["box"]
    for x in leaves.values():
        x.requires_grad_(True)
    kw = {k: v[k] for k in ("mask", "neighbors", "neighbor_edges", "box", "cell") if v.get(k) is not None}
    mod.zero_grad(set_to_none=True)
    with torch.enable_grad():
        out = mod(v["feats"], v["coors"], v.get("edges"), lattice_grad=lattice_grad, **kw)
        torch.autograd.backward(out, grad_tensors=(v["gf"], v["gx"]))
    g = {("in.edges" if k in ("edges", "neighbor_edges") else k if k == "box" else f"in.{k}"): x.grad
         for k, x in leaves.items()}
    g.update({f"p.{k}": p.grad for k, p in mod.named_parameters() if p.grad is not None})
    return tuple(o.detach() for o in out), g


GRAD_PARAMS = [(n, dt, lg) for n, lg in (("dense_n45_edges", False), ("list_slot_edges", False), ("dense_n70_box", True))
               for dt in (F64, F32)]


@pytest.mark.parametrize("name,dtype,lattice_grad", GRAD_PARAMS,
                         ids=[f"{n}-{_dt_id(d)}{'-lattice_grad' if lg else ''}" for n, d, lg in GRAD_PARAMS])
def test_layer_backward_on_a_side_stream(name, dtype, lattice_grad):
    """Forward and backward (and the box's gradient) on a side stream, the cotangents poisoned until copied there."""
    case, ins, opt = build(name)
    t = IL.torch_inputs(ins, dtype)
    rs = np.random.RandomState(11)
    t["gf"] = torch.from_numpy(rs.standard_normal(t["feats"].shape)).to(DEV, dtype)
    t["gx"] = torch.from_numpy(rs.standard_normal(t["coors"].shape)).to(DEV, t["coors"].dtype)
    e_key = "neighbor_edges" if t["neighbor_edges"] is not None else "edges"
    clone = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in t.items()}
    out_w, g_w = _layer_grads(util.make_module(case, dtype).requires_grad_(True), clone, e_key, lattice_grad)
    mod = util.make_module(case, dtype).requires_grad_(True)
    out_s, g_s = on_side_stream(t, lambda v: _layer_grads(mod, v, e_key, lattice_grad))
    IL.assert_bits(out_s, out_w, f"{name} side stream forward")
    tol = util.grad_tol(case, dtype)
    npy = lambda g: {k: v.double().cpu().numpy() for k, v in g.items()}
    util.compare(npy(g_s), npy(g_w), tol, f"{name} side stream vs default stream")
    if not lattice_grad:
        want = TREF.layer_grads_chunked(case["params"], case["cfg"], ins["feats"], ins["coors"], t["gf"].double().cpu(),
                                        t["gx"].double().cpu(), ins["edges"], ins["mask"], None, ins["box"],
                                        ins["neighbors"], slot_edges=ins["neighbor_edges"])
        got = npy(g_s)
        util.compare({k: got.get(k, np.zeros(v.shape)) for k, v in want.items()}, {k: v.numpy() for k, v in want.items()},
                     tol, f"{name} side stream vs reference")


# ----------------------------------------------------------------------------- A: EGNN_Network, attention, builders

NET_SPECS = {
    # token, position and edge-token embeddings, degree labels with adj_emb, global attention on every layer
    "embeddings_labels_attention": dict(kind=NW, cfg=dict(depth=2, dim=16, num_tokens=21, num_positions=40,
                                                          num_edge_tokens=5, edge_dim=3, num_adj_degrees=2, adj_dim=3,
                                                          global_linear_attn_every=1, global_linear_attn_heads=2,
                                                          global_linear_attn_dim_head=8, num_global_tokens=3),
                                        B=2, N=29, seed=661, init="xavier", mask="padded", edges=True),
    # only_sparse_neighbors with a mask: the lists cached with the expansion
    "sparse_lists": IL.NET_SPECS["sparse_adj"],
}


def net_case(name, seed=7):
    case = cases.build_case(NET_SPECS[name])
    case["inputs"]["adj_mat"] = IL.directed_adjacency(case["spec"]["N"], case["spec"]["B"], seed)
    return case


def net_inputs(case, dtype):
    ins = case["inputs"]
    f = torch.from_numpy(ins["feats"]).to(DEV)
    t = dict(feats=f if not f.is_floating_point() else f.to(dtype), coors=torch.from_numpy(ins["coors"]).to(DEV, dtype),
             adj_mat=torch.from_numpy(ins["adj_mat"]).to(DEV), mask=torch.from_numpy(ins["mask"]).to(DEV))
    if ins.get("edges") is not None:
        t["edges"] = torch.from_numpy(ins["edges"]).to(DEV)
    return t


def call_net(mod, v):
    return mod(v["feats"], v["coors"], adj_mat=v["adj_mat"], edges=v.get("edges"), mask=v["mask"])


@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("name", list(NET_SPECS))
def test_network_on_a_side_stream(name, dtype):
    case = net_case(name)
    t = net_inputs(case, dtype)
    want = call_net(util.make_module(case, dtype), t)
    mod = util.make_module(case, dtype)
    got = on_side_stream(t, lambda v: call_net(mod, v))
    IL.assert_bits(got, want, f"{name} side stream")
    if dtype == F64:      # (fp32 against the oracle: test_gpu_parity; the embedding case's activations reach ~4e3)
        ref = cases.run_oracle(case)
        util.assert_close(got[0], ref[0], what=f"{name} feats", **util.TOL[dtype])
        util.assert_close(got[1], ref[1], what=f"{name} coors", **util.TOL[dtype])


def ga_setup(dtype, name="n257"):
    """-> (case params, module, inputs, x dtype): a bf16 module runs on fp32 inputs (fp32 staged copies)."""
    P, x, q, m = GA.make_case(name)
    mod = GA.make_module(name, P, dtype)
    xdt = F32 if dtype == BF16 else dtype
    t = dict(x=torch.from_numpy(x).to(DEV, xdt), q=torch.from_numpy(q).to(DEV, xdt), m=torch.from_numpy(m).to(DEV))
    return P, mod, t


@pytest.mark.parametrize("dtype", [F64, F32, BF16], ids=["fp64", "fp32", "bf16_module"])
def test_global_attention_on_a_side_stream(dtype):
    P, mod, t = ga_setup(dtype)
    want = ga_setup(dtype)[1](t["x"], t["q"], t["m"])
    got = on_side_stream(t, lambda v: mod(v["x"], v["q"], v["m"]))
    IL.assert_bits(got, want, "GlobalLinearAttention side stream")
    if dtype != BF16:
        _, x, q, m = GA.make_case("n257")
        GA.check(got, GA.oracle(P, x, q, m, GA.CASES["n257"]["heads"]), dtype, "side stream")


@pytest.mark.parametrize("lattice", ["none", "cell"])
@pytest.mark.parametrize("fn,k", IL.BUILDERS, ids=[f for f, _ in IL.BUILDERS])
def test_list_builders_on_a_side_stream(fn, k, lattice):
    import egnn_pytorch_b200 as E
    x, m = IL.cloud(2, 300, F32, 50 + k)
    t = dict(x=x, m=m)
    if lattice == "cell":
        t["cell"] = torch.tensor(np.broadcast_to(IL.CELL3, (2, 3, 3)).copy(), device=DEV, dtype=F32)
    call = (lambda v: E.knn_neighbors(v["x"], k, mask=v["m"], cell=v.get("cell"))) if fn == "knn_neighbors" else \
        (lambda v: getattr(E, fn)(v["x"], 1.0, k, mask=v["m"], cell=v.get("cell")))
    want = call(t)
    got = on_side_stream(t, call)
    assert torch.equal(got, want), f"{fn}: {int((got != want).sum())} slots differ"
    if lattice == "none" and fn != "knn_neighbors":
        import test_gpu_radius_select as RS
        from egnn_pytorch_b200 import _native
        exp, _ = RS.expected_from_all_pairs(_native.load(), x, m, k, 1.0)
        assert torch.equal(got, exp), f"{fn}: lists differ from the all-pairs select"


def test_edge_index_to_neighbors_on_a_side_stream():
    """Poison 0 for the edge index: a valid node, so a premature read gives other lists, not an indexing error."""
    from egnn_pytorch_b200 import edge_index_to_neighbors
    g = torch.Generator().manual_seed(3)
    n, e = 60, 400
    t = dict(ei=torch.randint(0, n, (2, e), generator=g).to(DEV), attr=torch.randn((e, 3), generator=g).to(DEV))
    call = lambda v: edge_index_to_neighbors(v["ei"], n, k=12, edge_attr=v["attr"])
    want = call(t)
    got = on_side_stream(t, call)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_graphed_forward_replays_on_a_side_stream():
    from egnn_pytorch_b200.graphs import GraphedForward
    case, ins, _ = build("dense_n45_edges")
    t = IL.torch_inputs(ins, F32)
    want = util.make_module(case, F32)(t["feats"], t["coors"], t["edges"], mask=t["mask"])
    fast = GraphedForward(util.make_module(case, F32), t["feats"].clone(), t["coors"].clone(), t["edges"].clone(),
                          mask=t["mask"].clone())
    args = dict(feats=t["feats"], coors=t["coors"], edges=t["edges"])
    got = on_side_stream(args, lambda v: tuple(o.clone() for o in fast(v["feats"], v["coors"], v["edges"])))
    IL.assert_bits(got, want, "graph replay on a side stream")


# ----------------------------------------------------------------------------- B: read before write


@contextlib.contextmanager
def poisoned_pool(fill):
    """Allocations inside go to a private pool of two 2 MiB segments whose every byte is `fill` -> their spans.  Used
    on the building stream: whatever its call allocates there reads as poison until that stream writes it."""
    pool = torch.cuda.MemPool()
    _POOLS.append(pool)
    with torch.cuda.use_mem_pool(pool):
        blocks = [torch.full((SEGMENT,), fill, dtype=torch.uint8, device=DEV) for _ in range(4)]
        spans = [(b.data_ptr(), b.data_ptr() + SEGMENT) for b in blocks]
        del blocks
        yield spans


def build_then_reuse(build_on_a, entry, call_b, fill=0xFF, around_a=contextlib.nullcontext):
    """Stream A: a poisoned private pool, a sleep, `build_on_a()`.  The host checks that every tensor of `entry()` lies
    in the poisoned memory (else the case is inconclusive and B's call is not issued); then stream B runs `call_b()`
    with no wait -> its result, after a device synchronise."""
    from egnn_pytorch_b200.egnn import _workspace
    torch.cuda.synchronize()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    assert a.cuda_stream != b.cuda_stream
    with torch.cuda.stream(a):
        _workspace(torch.device(DEV, torch.cuda.current_device()), 8 << 20)      # A's scratch arena, outside the pool
        with poisoned_pool(fill) as spans, around_a():
            torch.cuda._sleep(SLEEP)
            build_on_a()
    tensors = entry()
    assert tensors
    outside = [tuple(x.shape) for x in tensors if not any(lo <= x.data_ptr() < hi for lo, hi in spans)]
    if outside:
        torch.cuda.synchronize()
        pytest.fail(f"inconclusive: entry tensors {outside} were not allocated in the poisoned pool")
    with torch.cuda.stream(b):
        got = call_b()
    torch.cuda.synchronize()
    return got


LAYER_SPEC = dict(kind=L, cfg=dict(dim=24, edge_dim=2), B=2, N=33, seed=671, init="xavier", mask="padded")


def layer_inputs(case, dtype):
    ins = case["inputs"]
    return IL.torch_inputs(dict(feats=ins["feats"], coors=ins["coors"], edges=ins["edges"], mask=ins["mask"]), dtype)


def call_layer(mod, t):
    return mod(t["feats"], t["coors"], t["edges"], mask=t["mask"])


def packed_of(*mods):
    return [p for m in mods for st in m._stage.values() for p in st["packed"].values()]


def _bump(mod, factor=1.25):
    """Every parameter scaled in place, on the current stream."""
    with torch.no_grad():
        for p in mod.parameters():
            p.mul_(factor)


def _layer_case(when, dtype):
    """-> (build_on_a, entry, call_b, want) of one EGNN layer case."""
    case = cases.build_case(LAYER_SPEC)
    t = layer_inputs(case, dtype)
    mod = util.make_module(case, dtype)
    ref = util.make_module(case, dtype)
    if when == "first call":
        build = lambda: call_layer(mod, t)
    elif when == "parameter update":
        call_layer(mod, t)
        _bump(mod), _bump(ref)
        build = lambda: call_layer(mod, t)
    elif when == "invalidate_cache":
        call_layer(mod, t)
        mod.invalidate_cache()
        build = lambda: call_layer(mod, t)
    else:
        assert when == "cache_policy always"
        mod.cache_policy = "always"
        call_layer(mod, t)
        build = lambda: call_layer(mod, t)
    return build, lambda: packed_of(mod), lambda: call_layer(mod, t), call_layer(ref, t)


B_LAYER = [(w, dt) for w in ("first call", "parameter update", "invalidate_cache", "cache_policy always")
           for dt in (F64, F32, BF16)]


@pytest.mark.parametrize("when,dtype", B_LAYER, ids=[f"{w.replace(' ', '_')}-{_dt_id(d)}" for w, d in B_LAYER])
def test_packed_parameters_built_on_one_stream_reused_on_another(when, dtype):
    """With cache_policy "always" stream B packs its own copy: nothing is shared, so this case holds without any
    ordering between the streams."""
    build, entry, call_b, want = _layer_case(when, dtype)
    got = build_then_reuse(build, entry, call_b)
    IL.assert_bits(got, want, f"{when}: stream B")


def test_bf16_module_trained_on_one_stream_evaluated_on_another():
    """A bf16 module trains through fp32 staged copies of its parameters; an fp32-kernel evaluation on another stream
    reuses those copies and their packed form."""
    case = cases.build_case(LAYER_SPEC)
    t = layer_inputs(case, BF16)
    mod = util.make_module(case, BF16, precision="accurate").requires_grad_(True)
    ref = util.make_module(case, BF16, precision="accurate")

    def train_step():
        mod.train()
        with torch.enable_grad():
            f, x = call_layer(mod, t)
            (f.float().sum() + x.sum()).backward()
        mod.eval()

    def entry():
        st = mod._stage[(torch.device(DEV, torch.cuda.current_device()), F32)]
        return list(st["tensors"].values()) + list(st["packed"].values())

    got = build_then_reuse(train_step, entry, lambda: call_layer(mod, t))
    IL.assert_bits(got, call_layer(ref, t), "bf16 training then evaluation")


ADJ_SPEC = dict(kind=NW, cfg=dict(depth=2, dim=16, num_adj_degrees=2, adj_dim=3), B=2, N=29, seed=672, init="xavier",
                mask="padded")


def test_adj_emb_restaged_on_one_stream_reused_on_another():
    """An in-place update of adj_emb.weight re-stages every layer's label table and packed parameters."""
    case = cases.build_case(ADJ_SPEC)
    case["inputs"]["adj_mat"] = IL.directed_adjacency(29, 2, 5)
    t = net_inputs(case, F32)
    net, ref = util.make_module(case, F32), util.make_module(case, F32)
    call_net(net, t)
    for m in (net, ref):
        with torch.no_grad():
            m.adj_emb.weight.mul_(-1.5)
    layers = [egnn for _, egnn in net.layers]
    got = build_then_reuse(lambda: call_net(net, t), lambda: packed_of(*layers), lambda: call_net(net, t))
    IL.assert_bits(got, call_net(ref, t), "adj_emb restaged")


class _SleepBefore:
    """The native library with a sleep enqueued before one entry point: holds back work a host sync would release."""

    def __init__(self, lib, name):
        self._lib, self._name = lib, name

    def __getattr__(self, k):
        f = getattr(self._lib, k)
        if k != self._name:
            return f

        def held(*a):
            torch.cuda._sleep(SLEEP)
            return f(*a)
        return held


@pytest.mark.parametrize("name", ["dense_labels", "sparse_lists"])
def test_adjacency_cache_built_on_one_stream_reused_on_another(name, monkeypatch):
    """The expanded adjacency and degree labels (and, only-sparse with a mask, the lists, built after the expansion's
    one host sync: a second sleep holds them back) of a new adjacency, reused at once by another stream."""
    from egnn_pytorch_b200 import _native
    case = cases.build_case(ADJ_SPEC if name == "dense_labels" else NET_SPECS["sparse_lists"])
    b, n = case["spec"]["B"], case["spec"]["N"]
    case["inputs"]["adj_mat"] = IL.directed_adjacency(n, b, 5)
    t = net_inputs(case, F32)
    net, ref = util.make_module(case, F32), util.make_module(case, F32)
    call_net(net, t)                                       # parameters staged and packed: only the adjacency is new
    t1 = dict(t, adj_mat=torch.from_numpy(IL.directed_adjacency(n, b, 6)).to(DEV))
    want = call_net(ref, t1)
    lib = _native.load()

    @contextlib.contextmanager
    def held_lists():
        with monkeypatch.context() as mp:
            mp.setattr(_native, "load", lambda: _SleepBefore(lib, "egnn_adj_neighbors"))
            yield

    def entry():
        c = net.__dict__["_adj_cache"]
        return [c[1], c[2]] + ([] if c[5] is None else [c[5]])

    got = build_then_reuse(lambda: call_net(net, t1), entry, lambda: call_net(net, t1), fill=0,
                           around_a=held_lists if name == "sparse_lists" else contextlib.nullcontext)
    if name == "sparse_lists":
        assert net.__dict__["_adj_cache"][5] is not None
    IL.assert_bits(got, want, f"{name}: stream B")


def test_bf16_global_attention_staged_on_one_stream_reused_on_another():
    P, mod, t = ga_setup(BF16)
    want = ga_setup(BF16)[1](t["x"], t["q"], t["m"])
    got = build_then_reuse(lambda: mod(t["x"], t["q"], t["m"]),
                           lambda: [x for st in mod._stage.values() for x in st[1].values()],
                           lambda: mod(t["x"], t["q"], t["m"]))
    IL.assert_bits(got, want, "bf16 GlobalLinearAttention: stream B")


# ----------------------------------------------------------------------------- C: free while in use


def fill_free_blocks(pool, value):
    """Hands out every free block of `pool` on the current stream, filled with `value` bytes -> the tensors.  Largest
    first, in pieces of at most SEGMENT bytes, so that each request meets a free block of exactly its size."""
    sizes = []
    for seg in torch.cuda.memory_snapshot():
        if tuple(seg.get("segment_pool_id", ())) == tuple(pool.id):
            for blk in seg["blocks"]:
                if blk["state"] == "inactive":
                    n = blk["size"]
                    sizes += [SEGMENT] * (n // SEGMENT) + ([n % SEGMENT] if n % SEGMENT else [])
    assert sizes, "no free block of the private pool in the allocator's snapshot"
    with torch.cuda.use_mem_pool(pool):
        return [torch.full((n,), value, dtype=torch.uint8, device=DEV) for n in sorted(sizes, reverse=True)]


def reuse_then_replace(build_on_a, entry, call_b, replace_on_a, fill):
    """Stream A builds the entry from a private pool; stream B, behind a sleep, reads it; stream A replaces it (with its
    new blocks from the default pool) and then takes every free block of the private pool, filled with `fill` bytes ->
    (B's result, A's result), after a device synchronise.  The old entry's blocks must not be among them: B may still
    read them.  Only what this test writes ever lands there, so a library that frees them early computes a wrong
    answer, never reads an index it did not write."""
    pool = torch.cuda.MemPool()
    _POOLS.append(pool)
    torch.cuda.synchronize()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    assert a.cuda_stream != b.cuda_stream
    with torch.cuda.stream(a), torch.cuda.use_mem_pool(pool):
        build_on_a()
    old = entry()
    assert old and all(x.untyped_storage().data_ptr() for x in old)
    old_spans = [(x.data_ptr(), x.data_ptr() + x.untyped_storage().nbytes()) for x in old]
    del old
    torch.cuda.synchronize()
    with torch.cuda.stream(b):
        torch.cuda._sleep(SLEEP)
        got_b = call_b()
    with torch.cuda.stream(a):
        got_a = replace_on_a()
        taken = fill_free_blocks(pool, fill)
    reused = [(lo, hi) for lo, hi in old_spans
              if any(t.data_ptr() < hi and lo < t.data_ptr() + t.numel() for t in taken)]
    torch.cuda.synchronize()
    assert not reused, f"{len(reused)} of the {len(old_spans)} blocks stream B was reading were handed out again on stream A"
    return got_b, got_a


def test_layer_parameters_updated_while_another_stream_reads_them():
    """A bf16 module on the fp32 kernels (staged copies): stream B evaluates it while stream A updates the parameters in
    place and calls again."""
    case = cases.build_case(LAYER_SPEC)
    t = layer_inputs(case, BF16)
    mod = util.make_module(case, BF16, precision="accurate")
    old, new = util.make_module(case, BF16, precision="accurate"), util.make_module(case, BF16, precision="accurate")
    _bump(new)

    def replace():
        _bump(mod)
        return call_layer(mod, t)

    def entry():
        st = mod._stage[(torch.device(DEV, torch.cuda.current_device()), F32)]
        return list(st["tensors"].values()) + list(st["packed"].values())

    got_b, got_a = reuse_then_replace(lambda: call_layer(mod, t), entry, lambda: call_layer(mod, t), replace, 0xFF)
    IL.assert_bits(got_b, call_layer(old, t), "stream B: the old parameters")
    IL.assert_bits(got_a, call_layer(new, t), "stream A: the new parameters")


@pytest.mark.parametrize("name", ["dense_labels", "sparse_lists"])
def test_adjacency_replaced_while_another_stream_reads_it(name):
    """Stream A passes a new adjacency of the same shape while stream B still reads the cached expansion of the old one.
    The freed blocks are filled with 0 bytes: valid degree labels, adjacency and list slots (node 0)."""
    case = cases.build_case(ADJ_SPEC if name == "dense_labels" else NET_SPECS["sparse_lists"])
    b, n = case["spec"]["B"], case["spec"]["N"]
    case["inputs"]["adj_mat"] = IL.directed_adjacency(n, b, 5)
    t = net_inputs(case, F32)
    net, ref = util.make_module(case, F32), util.make_module(case, F32)
    t1 = dict(t, adj_mat=torch.from_numpy(IL.directed_adjacency(n, b, 6)).to(DEV))
    want_b, want_a = call_net(ref, t), call_net(ref, t1)

    def entry():
        c = net.__dict__["_adj_cache"]
        return [c[1], c[2]] + ([] if c[5] is None else [c[5]])

    got_b, got_a = reuse_then_replace(lambda: call_net(net, t), entry, lambda: call_net(net, t), lambda: call_net(net, t1), 0)
    IL.assert_bits(got_b, want_b, f"{name}: stream B, the old adjacency")
    IL.assert_bits(got_a, want_a, f"{name}: stream A, the new adjacency")


def test_bf16_global_attention_updated_while_another_stream_reads_it():
    P, mod, t = ga_setup(BF16)
    old, new = ga_setup(BF16)[1], ga_setup(BF16)[1]
    _bump(new, 0.75)
    call = lambda m: m(t["x"], t["q"], t["m"])

    def replace():
        _bump(mod, 0.75)
        return call(mod)

    got_b, got_a = reuse_then_replace(lambda: call(mod), lambda: [x for st in mod._stage.values() for x in st[1].values()],
                                      lambda: call(mod), replace, 0xFF)
    IL.assert_bits(got_b, call(old), "stream B: the old parameters")
    IL.assert_bits(got_a, call(new), "stream A: the new parameters")
