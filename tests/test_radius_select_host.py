"""CPU checks of the cell-grid radius select: `radius_neighbors` rejects misuse before anything launches, the new C-ABI
symbols load, and the layer workspace grows by exactly the documented cell scratch for eligible descriptors (1 <= k <=
32, C <= 3, 0 < (T)valid_radius < 1e5, no only_sparse / batched adjacency / per-slot edges) and not at all otherwise."""
import ctypes as C

import pytest
import torch

import cases
from oracle import egnn_oracle as O
from util import nat  # noqa: F401  (module-scoped fixture)


def _r256(n):
    return (n + 255) // 256 * 256


def cell_bytes(B, N, C, coord_bytes):
    """The documented scratch: bucket sizes and bucket ends (int32, B * next_pow2(2N) each), coordinates in cell order,
    node index in cell order; each region rounded up to 256 bytes."""
    tb = 2
    while tb < 2 * N:
        tb *= 2
    return 2 * _r256(B * tb * 4) + _r256(C * B * N * coord_bytes) + _r256(B * N * 4)


def _layer_descs(nat):
    """(name, LayerDesc) for every layer configuration of tests/cases.py, in each dtype, plus radius variants."""
    out = []
    for name, spec in cases.SPECS.items():
        if spec["kind"] == "layer":
            cfg = O.layer_cfg(**spec["cfg"])
            edge_dim = cfg["edge_dim"]
        else:
            ncfg = O.network_cfg(**spec["cfg"])
            cfg = ncfg["layer"]
            edge_dim = ncfg["edge_dim"]
        flags = nat.FLAG_NORM_FEATS if cfg["norm_feats"] or spec["kind"] != "layer" else 0
        flags |= nat.FLAG_NORM_COORS if cfg["norm_coors"] else 0
        flags |= nat.FLAG_UPDATE_FEATS if cfg["update_feats"] else 0
        flags |= nat.FLAG_UPDATE_COORS if cfg["update_coors"] else 0
        flags |= nat.FLAG_SOFT_EDGES if cfg["soft_edges"] else 0
        flags |= nat.FLAG_POOL_MEAN if cfg["m_pool_method"] == "mean" else 0
        flags |= nat.FLAG_CLAMP if cfg["coor_weights_clamp_value"] is not None else 0
        flags |= nat.FLAG_ONLY_SPARSE if cfg["only_sparse_neighbors"] else 0
        flags |= nat.FLAG_ADJ_BATCHED if spec.get("adj") == "random3d" else 0
        k = cfg["num_nearest_neighbors"] or (3 if cfg["only_sparse_neighbors"] else 0)
        for dt in (nat.DTYPE_F32, nat.DTYPE_F64, nat.DTYPE_BF16):
            for vr in (cfg["valid_radius"], 2.0, 0.0, 1e5, 2e5 if dt == nat.DTYPE_F64 else 99999.9):
                d = nat.LayerDesc(abi_version=nat.ABI_VERSION, dtype=dt, B=spec["B"], N=spec["N"], C=spec.get("C", 3),
                                  dim=cfg["dim"], edge_dim=edge_dim, label_dim=0, num_labels=0, m_dim=cfg["m_dim"],
                                  fourier=cfg["fourier_features"], k=min(k, spec["N"]), flags=flags, valid_radius=vr,
                                  clamp=float(cfg["coor_weights_clamp_value"] or 0.0), row_begin=0, row_end=0, reserved=0)
                out.append((f"{name}/dtype{dt}/vr{vr}", d))
    return out


def _eligible(nat, d):
    vr = d.valid_radius if d.dtype == nat.DTYPE_F64 else float(torch.tensor(d.valid_radius, dtype=torch.float32))
    bad_flags = nat.FLAG_ONLY_SPARSE | nat.FLAG_ADJ_BATCHED | nat.FLAG_EDGES_PER_SLOT
    return 1 <= d.k <= 32 and 1 <= d.C <= 3 and not (d.flags & bad_flags) and 0.0 < vr < 1e5


def test_layer_workspace_grows_by_the_cell_scratch_only_when_eligible(nat):
    lib = nat.load()
    seen = {True: 0, False: 0}
    for name, d in _layer_descs(nat):
        nb = C.c_size_t()
        rc = lib.egnn_layer_workspace_bytes(C.byref(d), C.byref(nb))
        # the same descriptor with an infinite radius is never eligible: the parent's layout (valid_radius sizes nothing else)
        base = nat.LayerDesc()
        C.memmove(C.byref(base), C.byref(d), C.sizeof(nat.LayerDesc))
        base.valid_radius = float("inf")
        nb0 = C.c_size_t()
        rc0 = lib.egnn_layer_workspace_bytes(C.byref(base), C.byref(nb0))
        assert rc == rc0, name
        if rc != 0:
            assert rc == nat.ERR_UNSUPPORTED and d.dtype == nat.DTYPE_BF16, (name, rc)
            continue
        el = _eligible(nat, d)
        seen[el] += 1
        grow = cell_bytes(d.B, d.N, d.C, 8 if d.dtype == nat.DTYPE_F64 else 4) if el else 0
        assert nb.value == nb0.value + grow, (name, nb.value, nb0.value, grow)
    assert seen[True] > 20 and seen[False] > 100, seen


def test_layer_workspace_sizes_at_large_n(nat):
    """About 50-70 bytes per node at the sizes the cell grid is for (two int32 arrays of next_pow2(2N) <= 4N buckets)."""
    lib = nat.load()
    for dt, cb in ((nat.DTYPE_F32, 4), (nat.DTYPE_BF16, 4), (nat.DTYPE_F64, 8)):
        for n in (4096, 100_000, 131_072):
            kw = dict(abi_version=nat.ABI_VERSION, dtype=dt, B=1, N=n, C=3, dim=64, edge_dim=0, label_dim=0, num_labels=0,
                      m_dim=16, fourier=0, k=32, flags=nat.FLAG_UPDATE_FEATS | nat.FLAG_UPDATE_COORS, row_begin=0,
                      row_end=0, reserved=0, clamp=0.0)
            a, b = C.c_size_t(), C.c_size_t()
            assert lib.egnn_layer_workspace_bytes(C.byref(nat.LayerDesc(valid_radius=4.0, **kw)), C.byref(a)) == 0
            assert lib.egnn_layer_workspace_bytes(C.byref(nat.LayerDesc(valid_radius=float("inf"), **kw)), C.byref(b)) == 0
            grow = a.value - b.value
            assert grow == cell_bytes(1, n, 3, cb)
            assert 20 * n <= grow <= 72 * n, (dt, n, grow / n)


def test_radius_select_symbols_and_host_checks(nat):
    lib = nat.load()
    assert "egnn_radius_select" in nat.SYMBOLS and "egnn_radius_select_workspace_bytes" in nat.SYMBOLS
    nb = C.c_size_t()
    assert lib.egnn_radius_select_workspace_bytes(2, 1000, 3, 16, C.byref(nb)) == 0
    assert nb.value == cell_bytes(2, 1000, 3, 8)
    for args, code in [((2, 1000, 3, 33), -3), ((2, 1000, 4, 16), -3), ((2, 10, 3, 11), -2), ((0, 10, 3, 1), -2),
                       ((1, 10, 0, 1), -2), ((1, 10, 3, 0), -2)]:
        assert lib.egnn_radius_select_workspace_bytes(*args, C.byref(nb)) == code, args
    assert lib.egnn_radius_select_workspace_bytes(1, 10, 3, 1, None) == -1
    ws = C.c_void_p(1 << 20)                          # never dereferenced: every call below fails its checks first
    x = C.c_void_p(1 << 21)
    out = C.c_void_p(1 << 22)
    call = lambda dtype=nat.DTYPE_F32, B=1, N=10, Cd=3, k=4, coors=x, r2=1.0, idx=out, w=ws, nbytes=1 << 30: \
        lib.egnn_radius_select(dtype, B, N, Cd, k, coors, None, None, r2, idx, None, w, nbytes, None)
    assert call(coors=None) == -1 and call(idx=None) == -1 and call(w=None) == -1
    assert call(k=33, N=40) == -3 and call(Cd=4) == -3 and call(k=11) == -2
    assert call(w=C.c_void_p((1 << 20) + 16)) == -4
    assert call(nbytes=64) == -5
    assert call(r2=0.0) == -2 and call(r2=-1.0) == -2 and call(r2=float("nan")) == -2
    assert call(r2=1e-60) == -2                       # 0 once cast to float32
    assert call(dtype=7) == -3


def test_radius_neighbors_rejects_misuse_before_launching():
    from egnn_pytorch_b200 import radius_neighbors
    x = torch.randn(2, 10, 3)
    bad = [
        (dict(coors=torch.randn(10, 3)), "coors must be a"),
        (dict(coors=x.to(torch.bfloat16)), "float32 or float64"),
        (dict(coors=x.half()), "float32 or float64"),
        (dict(coors=torch.randn(2, 0, 3)), "at least one node"),
        (dict(coors=torch.randn(2, 10, 4)), "C <= 3"),
        (dict(coors=torch.randn(2, 10, 0)), "C <= 3"),
        (dict(k=0), r"k must be an int in \[1, min\(32, N\)\] = \[1, 10\]"),
        (dict(k=11), "k must be"),
        (dict(coors=torch.randn(1, 50, 3), k=33), r"= \[1, 32\]"),
        (dict(k=2.0), "k must be"),
        (dict(k=True), "k must be"),
        (dict(cutoff=0.0), "cutoff must be a finite distance > 0"),
        (dict(cutoff=-1.0), "cutoff must be"),
        (dict(cutoff=float("nan")), "cutoff must be"),
        (dict(cutoff=float("inf")), "cutoff must be"),
        (dict(cutoff=1e-30), "squared is 0"),
        (dict(mask=torch.ones(2, 9)), "mask must be a"),
        (dict(mask=[1] * 10), "mask must be a"),
        (dict(box=torch.ones(4)), "box must have shape"),
        (dict(box=torch.tensor([1.0, -1.0, 1.0])), "box lengths must be >= 0"),
        (dict(box=[1.0, 1.0, 1.0]), "box must be a float tensor"),
        (dict(box=torch.ones(3, requires_grad=True)), "requires_grad"),
    ]
    for kw, msg in bad:
        args = dict(coors=x, cutoff=1.0, k=4)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            radius_neighbors(args.pop("coors"), args.pop("cutoff"), args.pop("k"), **args)


def test_radius_neighbors_is_exported():
    import egnn_pytorch_b200
    from egnn_pytorch_b200 import egnn
    assert egnn_pytorch_b200.radius_neighbors is egnn.radius_neighbors
    assert "radius_neighbors" in egnn.__all__
