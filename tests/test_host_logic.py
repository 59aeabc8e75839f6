"""CPU-only checks of the host side: the C-ABI library loads and exports every declared symbol,
the ctypes structs match the C structs, the module mirrors the reference's state-dict contract,
and nothing computes without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import cases
from util import nat  # noqa: F401  (module-scoped fixture)

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(REPO, "include", "egnn_b200.h")


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(egnn_[a-z_0-9]+)\s*\(", src)))


def test_library_exports_every_declared_symbol(nat):
    names = declared_functions()
    assert len(names) >= 10
    out = subprocess.run(["nm", "-D", "--defined-only", nat.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r" T (egnn_[a-z_0-9]+)", out))
    assert set(names) <= exported, set(names) - exported
    assert set(names) == set(nat.SYMBOLS), set(names) ^ set(nat.SYMBOLS)


def test_library_is_sm90a_and_has_no_other_arch(nat):
    out = subprocess.run(["cuobjdump", "-lelf", nat.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    assert not re.search(r"sm_(?!90a)\d+", out), out


def test_ctypes_structs_match_c_layout(nat, tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "egnn_b200.h"\nint main(){\n'
                    'printf("%zu %zu %zu %zu %zu\\n", sizeof(EgnnLayerDesc), sizeof(EgnnLayerWeights), sizeof(EgnnLayerIO),'
                    ' sizeof(EgnnLayerWeightGrads), sizeof(EgnnLayerGrads));\n'
                    'printf("%zu %zu %zu %zu\\n", offsetof(EgnnLayerDesc, flags), offsetof(EgnnLayerDesc, valid_radius),'
                    ' offsetof(EgnnLayerDesc, row_end), offsetof(EgnnLayerIO, feats_out));\n'
                    'printf("%zu %zu\\n", offsetof(EgnnLayerGrads, g_edges), offsetof(EgnnLayerGrads, w));\nreturn 0;}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(REPO, "include"), str(prog), "-o", str(exe)], check=True)
    a, b, c = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.strip().split("\n")
    assert [int(x) for x in a.split()] == [C.sizeof(nat.LayerDesc), C.sizeof(nat.LayerWeights), C.sizeof(nat.LayerIO),
                                           C.sizeof(nat.LayerWeightGrads), C.sizeof(nat.LayerGrads)]
    assert [int(x) for x in c.split()] == [nat.LayerGrads.g_edges.offset, nat.LayerGrads.w.offset]
    assert [int(x) for x in b.split()] == [nat.LayerDesc.flags.offset, nat.LayerDesc.valid_radius.offset,
                                           nat.LayerDesc.row_end.offset, nat.LayerIO.feats_out.offset]


def test_host_side_validation_without_gpu(nat):
    lib = nat.load()
    nb = C.c_size_t()
    good = dict(abi_version=nat.ABI_VERSION, dtype=nat.DTYPE_F32, B=2, N=16, C=3, dim=32, edge_dim=0, label_dim=0, num_labels=0,
                m_dim=16, fourier=0, k=0, flags=nat.FLAG_UPDATE_FEATS | nat.FLAG_UPDATE_COORS, valid_radius=1e30,
                clamp=0.0, row_begin=0, row_end=0, reserved=0)
    d = nat.LayerDesc(**good)
    assert lib.egnn_layer_packed_bytes(C.byref(d), C.byref(nb)) == 0 and nb.value > 0
    assert lib.egnn_layer_workspace_bytes(C.byref(d), C.byref(nb)) == 0
    E = 2 * 32 + 1
    assert nb.value >= 2 * 16 * 2 * (2 * E) * 4          # the two per-node tables
    assert lib.egnn_layer_backward_workspace_bytes(C.byref(d), C.byref(nb)) == 0 and nb.value > 2 * 16 * 16 * 20 * 4
    for unsupported in (dict(dtype=nat.DTYPE_BF16), dict(row_begin=0, row_end=8), dict(label_dim=4, num_labels=40)):
        assert lib.egnn_layer_backward_workspace_bytes(C.byref(nat.LayerDesc(**dict(good, **unsupported))), C.byref(nb)) == -3
    for bad, code in [(dict(abi_version=7), -6), (dict(N=0), -2), (dict(C=9), -3), (dict(m_dim=64), -3),
                      (dict(k=17), -2), (dict(flags=0), -2), (dict(dtype=9), -3), (dict(row_begin=5, row_end=3), -2)]:
        d = nat.LayerDesc(**dict(good, **bad))
        assert lib.egnn_layer_packed_bytes(C.byref(d), C.byref(nb)) == code, bad
    assert lib.egnn_layer_packed_bytes(None, C.byref(nb)) == -1
    assert b"ABI" in lib.egnn_strerror(-6)
    assert lib.egnn_adj_workspace_bytes(1, 8192, C.byref(nb)) == 0 and nb.value == 2 * 8192 * 256 * 4


def test_backward_preflight_checks_the_shared_memory_of_the_backward_kernels(nat):
    """egnn_layer_backward_workspace_bytes (which the training forward calls before it launches anything) sizes bwd1 and
    bwd2 as their launches do and rejects what exceeds the 220 KB SIMT budget, dense and neighbour lists alike."""
    lib = nat.load()
    nb = C.c_size_t()
    uf_uc = nat.FLAG_UPDATE_FEATS | nat.FLAG_UPDATE_COORS
    base = dict(abi_version=nat.ABI_VERSION, B=2, N=40, C=3, dim=16, edge_dim=0, label_dim=0, num_labels=0, m_dim=16,
                fourier=0, k=0, flags=uf_uc, valid_radius=1e30, clamp=0.0, row_begin=0, row_end=0, reserved=0)
    soft = uf_uc | nat.FLAG_SOFT_EDGES
    over_in_fp64 = [dict(m_dim=32),                                  # bwd1: 234,032 B
                    dict(m_dim=24, flags=soft),                      # bwd1: 225,328 B
                    dict(dim=8, fourier=30, edge_dim=16)]            # dense bwd2: 77 channels, about 311 KB
    fits = [dict(m_dim=24), dict(m_dim=20, flags=soft), dict(m_dim=17), dict(label_dim=4, num_labels=16),
            dict(dim=8, fourier=30, edge_dim=16, m_dim=32)]         # (the last in fp32 only: see below)
    rc = lambda **kw: lib.egnn_layer_backward_workspace_bytes(C.byref(nat.LayerDesc(**dict(base, **kw))), C.byref(nb))
    for k in (0, 20):
        for cfg in over_in_fp64:
            assert rc(dtype=nat.DTYPE_F64, k=k, **cfg) == -3, (cfg, k)
            assert rc(dtype=nat.DTYPE_F32, k=k, **cfg) == 0, (cfg, k)
        for cfg in fits[:-1]:
            assert rc(dtype=nat.DTYPE_F64, k=k, **cfg) == 0, (cfg, k)
        assert rc(dtype=nat.DTYPE_F32, k=k, **fits[-1]) == 0
        for dt in (nat.DTYPE_F32, nat.DTYPE_F64):
            assert rc(dtype=dt, k=k, label_dim=4, num_labels=17) == -3        # label rows of bwd2's shared table


@pytest.mark.parametrize("name", ["dense_everything", "knn_edges_mask", "dense_no_feats", "dense_no_coors",
                                  "net_c5_xavier", "net_edge_tokens", "net_c3_small"])
def test_reference_state_dict_loads_unchanged(name):
    """The generated parameter dicts use the reference's keys (and loaded strictly into the
    reference when the fixtures were made, tests/golden/make_golden.py)."""
    from egnn_pytorch_b200 import EGNN, EGNN_Network
    case = cases.build_case(cases.SPECS[name])
    cfg = case["spec"]["cfg"]
    mod = EGNN_Network(**cfg) if case["kind"] == "network" else EGNN(**cfg)
    assert set(mod.state_dict().keys()) == set(case["params"].keys())
    for k, v in mod.state_dict().items():
        assert tuple(v.shape) == tuple(np.asarray(case["params"][k]).shape), k
    mod.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in case["params"].items()}, strict=True)


def test_default_init_follows_reference():
    from egnn_pytorch_b200 import EGNN
    torch.manual_seed(0)
    m = EGNN(dim=64, init_eps=1e-3)
    w = m.edge_mlp[0].weight
    assert abs(float(w.std()) - 1e-3) < 1e-4          # reference :219-222
    assert float(m.edge_mlp[0].bias.abs().max()) > 1e-2   # biases keep the PyTorch default
    assert EGNN(dim=8, norm_coors=True, norm_coors_scale_init=0.5).coors_norm.scale.item() == 0.5


def test_global_attention_network_keys():
    from egnn_pytorch_b200 import EGNN_Network
    net = EGNN_Network(depth=2, dim=16, global_linear_attn_every=1, num_global_tokens=3, global_linear_attn_heads=2,
                       global_linear_attn_dim_head=8)
    keys = set(net.state_dict())
    assert "global_tokens" in keys and "layers.0.0.attn1.to_kv.weight" in keys and "layers.1.0.ff.3.bias" in keys
    assert "layers.0.1.node_norm.weight" in keys


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    from egnn_pytorch_b200 import EGNN
    layer = EGNN(dim=8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        layer(torch.randn(1, 4, 8), torch.randn(1, 4, 3))


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from egnn_pytorch_b200 import _native
    monkeypatch.setattr(_native, "_lib", None)
    monkeypatch.setattr(_native, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_native.NativeLibraryError, match="no CPU fallback"):
        _native.load()


def test_product_never_imports_the_oracle():
    pkg = os.path.join(REPO, "egnn_pytorch_b200")
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(root, f)).read()
                assert "oracle" not in src.replace("the oracle", "").replace("fp64 oracle", ""), (f, "references oracle/")


def test_shard_range_partitions():
    from egnn_pytorch_b200.parallel import shard_range
    for total in (1, 7, 8, 64, 4096):
        for world in (1, 2, 3, 8):
            spans = [shard_range(total, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == total
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
            sizes = [e - s for s, e in spans]
            assert max(sizes) - min(sizes) <= 1


def test_edge_index_to_neighbors_cpu():
    """PyG-style edge_index -> padded neighbour lists (host glue of the edge-list mode, SURVEY.md section 8(f) rank 3)."""
    import torch
    from egnn_pytorch_b200 import edge_index_to_neighbors
    # messages flow source -> target; node 2 receives from 0, 1, 3; node 0 from 1; node 3 from nobody
    ei = torch.tensor([[0, 1, 3, 1], [2, 2, 2, 0]])
    nb = edge_index_to_neighbors(ei, 4)
    assert nb.shape == (1, 4, 3) and nb.dtype == torch.int32
    assert sorted(nb[0, 2].tolist()) == [0, 1, 3]
    assert nb[0, 0].tolist() == [1, -1, -1]
    assert nb[0, 1].tolist() == [-1, -1, -1] and nb[0, 3].tolist() == [-1, -1, -1]
    # a width cap keeps the first edges of each target in input order
    nb2 = edge_index_to_neighbors(ei, 4, k=2)
    assert nb2.shape == (1, 4, 2) and nb2[0, 2].tolist() == [0, 1]


def test_training_path_selection_without_gpu(monkeypatch):
    """Autograd semantics of the module mirror, checked without a device: under no_grad (or with nothing requiring
    grad) the inference path runs; otherwise the torch.autograd.Function bridge is entered."""
    import torch
    from egnn_pytorch_b200 import EGNN
    calls = []
    layer = EGNN(dim=8)
    monkeypatch.setattr(EGNN, "_forward_impl", lambda self, *a, **k: calls.append("infer") or (a[0], a[1]))
    monkeypatch.setattr(EGNN, "_forward_train", lambda self, *a, **k: calls.append("train") or (a[1], a[2]))
    f, x = torch.randn(1, 4, 8), torch.randn(1, 4, 3)
    with torch.no_grad():
        layer(f, x)
    with torch.enable_grad():                           # (the suite's autouse fixture switches grad mode off)
        layer.requires_grad_(False)
        layer(f, x)                                     # grad mode on, but nothing requires grad
        layer(f.clone().requires_grad_(True), x)        # an input requires grad
        layer.requires_grad_(True)
        layer(f, x)                                     # parameters require grad
    assert calls == ["infer", "infer", "train", "train"]


def test_flags_follow_attributes_changed_after_construction(nat):
    """Only the module structure is cached in the flag word: the pooling method and the clamp value are plain attributes
    and a change between calls must reach the descriptor (reference reads them per call, egnn_pytorch.py:308, :319)."""
    from egnn_pytorch_b200 import EGNN
    layer = EGNN(dim=8, norm_feats=True, soft_edges=True)
    f0 = layer._flags()
    assert f0 & nat.FLAG_NORM_FEATS and f0 & nat.FLAG_SOFT_EDGES and f0 & nat.FLAG_UPDATE_FEATS and f0 & nat.FLAG_UPDATE_COORS
    assert not f0 & nat.FLAG_CLAMP and not f0 & nat.FLAG_POOL_MEAN
    layer.coor_weights_clamp_value = 2.0
    layer.m_pool_method = "mean"
    f1 = layer._flags()
    assert f1 & nat.FLAG_CLAMP and f1 & nat.FLAG_POOL_MEAN and (f1 & f0) == f0
    layer.coor_weights_clamp_value = None
    assert not layer._flags() & nat.FLAG_CLAMP


def test_native_symbol_table_has_adj_neighbors(nat):
    assert "egnn_adj_neighbors" in nat.SYMBOLS and hasattr(nat.load(), "egnn_adj_neighbors")


def test_parameter_staging_cache_semantics():
    """The staged / packed parameter copies are keyed on (storage pointer, version) of every parameter: an in-place
    update, a replaced Parameter, `invalidate_cache()` and `cache_policy='always'` must each re-stage; nothing else may."""
    from egnn_pytorch_b200 import EGNN
    cpu = torch.device("cpu")
    layer = EGNN(dim=8).eval()
    s1 = layer._staged(cpu, torch.float32)
    assert layer._staged(cpu, torch.float32) is s1                       # unchanged parameters: cache hit
    w = layer.edge_mlp[0].weight
    with torch.no_grad():
        w.add_(1.0)                                                      # optimizer-style in-place step
    s2 = layer._staged(cpu, torch.float32)
    assert s2 is not s1 and torch.equal(s2["tensors"]["edge_w1"], w.detach())
    layer.edge_mlp[0].weight = torch.nn.Parameter(torch.zeros_like(w))   # Parameter object replaced
    s3 = layer._staged(cpu, torch.float32)
    assert s3 is not s2 and float(s3["tensors"]["edge_w1"].abs().max()) == 0.0
    layer.invalidate_cache()
    s4 = layer._staged(cpu, torch.float32)
    assert s4 is not s3
    layer.cache_policy = "always"
    assert layer._staged(cpu, torch.float32) is not s4
    layer.cache_policy = "version"
    s5 = layer._staged(cpu, torch.float32)
    assert layer._staged(cpu, torch.float32) is s5
    assert layer._staged(cpu, torch.float64) is not s5                   # one staging per (device, dtype)
