"""Host side of caller-memory layouts (no GPU): the staging helpers realign what the library's 16-byte pointer contract
rejects and pass aligned contiguous tensors through uncopied, EGNN_Network's adjacency cache tells views of one storage
apart, and tests/test_gpu_input_layouts.py covers every layout at every entry point it promises."""
import pytest
import torch

from egnn_pytorch_b200 import egnn as E

CPU = torch.device("cpu")


def _misaligned_views(dtype):
    """Contiguous views of an aligned buffer at every element offset that leaves the start off 16 bytes."""
    base = torch.arange(256, dtype=torch.float64).to(dtype)
    assert base.data_ptr() % 16 == 0
    es = base.element_size()
    return [base[o:o + 97] for o in range(1, 16 // es)]


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32, torch.bfloat16, torch.int32])
def test_as_realigns_misaligned_views(dtype):
    for v in _misaligned_views(dtype):
        assert v.is_contiguous() and v.data_ptr() % 16 != 0
        out = E._as(v, CPU, dtype)
        assert out.data_ptr() % 16 == 0 and out.is_contiguous()
        assert torch.equal(out, v) and out.dtype == dtype


def test_as_realigns_a_batch_slice_and_a_single_graph_row_slice():
    big = torch.randn(4, 5, 3)                      # one graph: 15 floats = 60 bytes
    for v in (big[1:3], big[:1, 1:]):
        assert v.is_contiguous() and v.data_ptr() % 16 != 0
        out = E._as(v, CPU, torch.float32)
        assert out.data_ptr() % 16 == 0 and torch.equal(out, v) and out.shape == v.shape


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32, torch.bfloat16])
def test_as_passes_aligned_contiguous_tensors_through_uncopied(dtype):
    t = torch.randn(2, 8, 16).to(dtype)
    assert t.data_ptr() % 16 == 0
    assert E._as(t, CPU, dtype).data_ptr() == t.data_ptr()
    s = t[1:]                                       # 128 elements in: still 16-byte aligned
    assert E._as(s, CPU, dtype).data_ptr() == s.data_ptr()
    r = t.requires_grad_(True) if dtype != torch.bfloat16 else t
    out = E._as(r, CPU, dtype)
    assert out.data_ptr() == t.data_ptr() and not out.requires_grad


def test_as_copies_strided_and_converted_inputs():
    t = torch.randn(3, 7, 5)
    for v in (t.transpose(1, 2), t[..., 1:4], t[:1].expand(3, 7, 5)):
        out = E._as(v, CPU, torch.float32)
        assert out.is_contiguous() and out.data_ptr() % 16 == 0 and torch.equal(out, v)
    out = E._as(t[1:], CPU, torch.float64)
    assert out.dtype == torch.float64 and out.data_ptr() % 16 == 0 and torch.equal(out, t[1:].double())


@pytest.mark.parametrize("dtype", [torch.bool, torch.uint8, torch.int64, torch.float32])
def test_as_u8_realigns_and_converts_masks(dtype):
    base = (torch.arange(300) % 3 == 0).to(dtype)
    for o in range(0, 16):
        v = base[o:o + 150]
        out = E._as_u8(v, CPU)
        assert out.dtype == torch.uint8 and out.is_contiguous() and out.data_ptr() % 16 == 0
        assert torch.equal(out, v.ne(0).to(torch.uint8))
        if o == 0 and dtype in (torch.bool, torch.uint8):
            assert out.data_ptr() == v.data_ptr()      # aligned and already bytes: no copy
    m = (torch.rand(6, 9) < 0.5).to(dtype)
    assert torch.equal(E._as_u8(m.t(), CPU), m.t().ne(0).to(torch.uint8))


def test_adjacency_cache_key_tells_views_of_one_storage_apart():
    a = torch.rand(2, 9, 9) < 0.3
    t = a.transpose(1, 2)
    assert t.data_ptr() == a.data_ptr() and t._version == a._version and t.shape == a.shape
    key = E._adj_cache_key(a, 2, 2)
    assert key == E._adj_cache_key(a, 2, 2)
    assert E._adj_cache_key(t, 2, 2) != key
    assert E._adj_cache_key(a.view(torch.uint8), 2, 2) != key
    assert E._adj_cache_key(a, 2, 3) != key
    a2 = a[0]
    assert E._adj_cache_key(a2, 2, 2) != E._adj_cache_key(a2.t(), 2, 2)
    a[0, 1, 2] = True
    assert E._adj_cache_key(a, 2, 2) != key                 # an in-place write bumps the version


# ----------------------------------------------------------------------------- coverage of the GPU file

PROMISED = {
    # every entry point is run on contiguous placements (poison on both sides, every misaligned remainder, a batch
    # slice) and on strided views, next to its canonical call
    "EGNN forward fp64/fp32 dense": {"expanded"},
    "EGNN forward bf16 tc_pair": {"expanded"},
    "GlobalLinearAttention": {"expanded"},
    "EGNN backward fp64/fp32": {"expanded"},
}


def test_table_covers_every_layout_at_every_entry_point():
    import test_gpu_input_layouts as T
    everywhere = {"canonical", "poisoned", "misaligned", "batch_slice"}
    for entry in ("EGNN forward fp64/fp32 dense", "EGNN forward fp64/fp32 lists", "EGNN forward bf16 tc_pair",
                  "EGNN forward bf16 tc_knn", "EGNN own selects", "EGNN backward fp64/fp32", "EGNN_Network",
                  "GlobalLinearAttention", "radius_neighbors", "radius_neighbors_wide", "knn_neighbors"):
        want = everywhere | PROMISED.get(entry, set())
        if entry != "EGNN backward fp64/fp32":
            want |= {"last_dim_slice", "permuted"}
        else:
            want |= {"permuted"}                            # the transposed coordinate leaf
        missing = want - T.LAYOUT_COVERAGE.get(entry, set())
        assert not missing, (entry, sorted(missing))
    assert set(T.FORMS) == {"poisoned", "misaligned", "batch_slice", "last_dim_slice", "permuted"}


def test_scenarios_reach_the_boundaries_they_name():
    """Each forward entry point has a scenario; the SIMT ones come from the boundary tables, with a box and a cell among
    the dense and the list cases, k = 33 and per-slot edges among the lists, every own select path, and the bf16 ones
    cover tc_pair at N = 127 / 129 with a row range and tc_knn lean / edges / generic / k = 65 / per-slot edges."""
    import test_gpu_input_layouts as T
    entries = set(T.SCENARIO_ENTRY.values())
    assert {e for e in T.LAYOUT_COVERAGE if e.startswith("EGNN forward") or e == "EGNN own selects"} <= entries
    S = T.LAYER_SCENARIOS
    lat = lambda pre, kind: any(n.startswith(pre) and o.get("lattice") == kind for n, (_, o) in S.items())
    assert all(lat(pre, kind) for pre in ("dense", "list") for kind in ("box", "cell"))
    assert any(src == ("list", "k33") for src, _ in S.values())
    assert any(o.get("slot_edges") for _, o in S.values()) and any(o.get("slot_edges") for _, o in T.TC_SCENARIOS.values())
    envs = {k for _, o in S.values() for k in o.get("env", {})}
    assert envs == {"EGNN_B200_CELL_SELECT_MIN_N", "EGNN_B200_KNN_GRID_MIN_N"}
    assert any(src[0] == "spec" and src[1].get("adj") for src, _ in S.values())
    tc = T.TC_SCENARIOS
    assert {s["N"] for s, o in tc.values() if "k" not in o} >= {127, 129}
    assert any("rows" in o for _, o in tc.values())
    ks = {o["k"] for _, o in tc.values() if "k" in o}
    assert 65 in ks and any(k <= 32 for k in ks)
    assert any(s["cfg"].get("fourier_features") for s, o in tc.values() if "k" in o)
    assert any(s["cfg"].get("edge_dim") and not o.get("slot_edges") for s, o in tc.values() if "k" in o)
    # the misaligned placement reaches every remainder of every element size
    for dtype, rem in ((torch.float32, {4, 8, 12}), (torch.float64, {8}), (torch.bfloat16, set(range(2, 16, 2)))):
        t = torch.zeros(1, dtype=dtype)
        assert {o * t.element_size() for o in T.offsets(t)} == rem
