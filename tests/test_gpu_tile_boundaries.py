"""Tile boundaries of the fp32 / fp64 edge kernels and their backward, against the fp64 oracles.

Every SIMT edge kernel walks a fixed tile and has a partial last one: the dense forward takes 32 neighbours per pass
and 4*PP rows per CTA, stages the hidden axis in chunks of 64 channels, and at one row per thread (fp64 with 32-wide
accumulators) keeps its row sums in registers; the dense bwd2 takes 32 rows x 128 channels per CTA; bwd1 / bwd3 take
slot groups of TS lanes; the per-node backward GEMMs split K = B*N.  The cases below are sized so that each of these
runs with several tiles and a partial last one (test_table_covers_every_tile_boundary keeps them so), with xavier
weights and masks so that no path hides behind the biases.  The neighbour-list cases live in test_edge_list.py
(EDGE_CASES); the coverage check reads them from there.

Each case: forward in fp64 and fp32 at util.TOL; gradients in fp64 and fp32 at util.grad_tol, with W2 silu(pre1) saved
by the forward and recomputed by the backward.  Configurations whose backward needs more shared memory than the SIMT
budget must fail at the training forward, before it runs."""
import functools

import pytest
import torch

import cases
import launch_geometry as LG
import util
from tests import test_edge_list

L, NW = "layer", "network"

TILE_CASES = {
    # --- dense layers: N in {33, 45, 70, 97} gives 2-4 neighbour passes and bwd2 row CTAs, each with a partial last one
    "dense_n33_hp72":    dict(kind=L, cfg=dict(dim=16, m_pool_method="mean"), B=2, N=33, seed=301, init="xavier",
                              mask="random"),
    "dense_n45_hp128":   dict(kind=L, cfg=dict(dim=31, edge_dim=1, soft_edges=True), B=2, N=45, seed=302, init="xavier",
                              mask="padded"),
    "dense_n70_hp144":   dict(kind=L, cfg=dict(dim=32, fourier_features=2, edge_dim=3, norm_coors=True,
                                               coor_weights_clamp_value=0.5), B=2, N=70, seed=303, init="xavier",
                              mask="padded"),
    "dense_n97_hp296":   dict(kind=L, cfg=dict(dim=72, norm_feats=True, m_pool_method="mean",
                                               coor_weights_clamp_value=1.0), B=2, N=97, seed=304,
                              init="xavier", mask="random"),
    # --- networks of dense layers with degree labels (4 and 16 label rows in bwd2's shared table)
    "net_n45_labels4":   dict(kind=NW, cfg=dict(depth=2, dim=16, num_tokens=21, num_adj_degrees=3, adj_dim=4,
                                               m_pool_method="mean", coor_weights_clamp_value=0.2), B=2, N=45,
                              seed=305, init="xavier", adj="chain", mask="padded"),
    "net_n45_labels16":  dict(kind=NW, cfg=dict(depth=2, dim=16, num_adj_degrees=15, adj_dim=3, m_pool_method="mean",
                                               coor_weights_clamp_value=0.2),
                              B=2, N=45, seed=306, init="xavier", adj="chain", mask="random"),
    # --- m_dim: 16-wide accumulators with a partial tail, and 32-wide ones (fp64: one row per thread in the forward,
    # pre2 read again in bwd1)
    "dense_mdim12":      dict(kind=L, cfg=dict(dim=16, m_dim=12, edge_dim=2), B=2, N=40, seed=307, init="xavier",
                              mask="padded"),
    "dense_mdim20_soft": dict(kind=L, cfg=dict(dim=16, m_dim=20, soft_edges=True, m_pool_method="mean"), B=2, N=36,
                              seed=308, init="xavier", mask="random"),
    "dense_mdim24":      dict(kind=L, cfg=dict(dim=12, m_dim=24, norm_coors=True), B=1, N=50, seed=309, init="xavier",
                              mask="padded"),
    # --- over the shared-memory budget of the fp64 backward (bwd1: 225,328 B and 234,032 B; dense bwd2: 311 KB for
    # 77 per-pair channels), not of the fp32 one
    "dense_mdim24_soft": dict(kind=L, cfg=dict(dim=12, m_dim=24, soft_edges=True), B=2, N=35, seed=310, init="xavier",
                              mask="padded"),
    "dense_mdim32":      dict(kind=L, cfg=dict(dim=12, m_dim=32, edge_dim=1, coor_weights_clamp_value=1.0), B=2, N=40,
                              seed=311, init="xavier", mask="random"),
    "dense_q77":         dict(kind=L, cfg=dict(dim=8, fourier_features=30, edge_dim=16), B=1, N=40, seed=312,
                              init="xavier"),
}
FP64_BACKWARD_REJECTED = {"dense_mdim24_soft", "dense_mdim32", "dense_q77"}

# ------------------------------------------------------------------ tile geometry (launch_geometry.simt_layer)


def list_geometry(name):
    cfg, B, N, k, C, _, _ = test_edge_list.EDGE_CASES[name]
    return LG.simt_layer(L, cfg, B, N, k=k, C=C)


def test_table_covers_every_tile_boundary():
    """Each boundary the table is meant to reach, recomputed from the specs: an edit to a shape that drops one fails here."""
    dense = {n: LG.simt_layer(s["kind"], s["cfg"], s["B"], s["N"]) for n, s in TILE_CASES.items()}
    trained64 = {n: g for n, g in dense.items() if n not in FP64_BACKWARD_REJECTED}
    lists = {n: list_geometry(n) for n in test_edge_list.BACKWARD_CASES}
    want = {
        # dense forward: several 32-neighbour passes with a partial last one; the rows of a CTA (4 * PP) partial
        "dense j passes, partial last": any(g["j_passes"] >= 3 and g["partial_j"] for g in trained64.values()),
        "dense rows per CTA, partial last": any(g["N"] % 8 != 0 for g in trained64.values()),
        # hidden chunks of 64: Hp = 72 (partial second chunk), H = Hp = 128, Hp = 144 with Q = 8, Hp = 296
        "Hp 72": any(g["Hp"] == 72 and g["partial_chunk"] for g in trained64.values()),
        "H = Hp = 128": any(g["Hp"] == 128 and 2 * g["E"] == 128 for g in trained64.values()),
        "Hp 144, Q 8": any(g["Hp"] == 144 and g["Q"] == 8 for g in trained64.values()),
        "Hp 296": any(g["Hp"] == 296 for g in trained64.values()),
        # dense bwd2: several 32-row CTAs with a partial last one; a partial 128-channel CTA (hv false on some lanes)
        "bwd2 row CTAs, partial last": any(g["bwd2_row_ctas"] >= 3 and g["partial_rows"] for g in trained64.values()),
        "bwd2 channel CTAs, partial last": any(g["bwd2_ch_ctas"] >= 2 and g["partial_ch_cta"] for g in trained64.values()),
        # per-node stages: generic GEMMs above dim 64, split-K over B*N with a partial last split
        "generic node GEMMs, partial split-K": any(g["generic_node_gemm"] and g["splitk"] > 1 and g["partial_split"]
                                                   for g in trained64.values()),
        # m_dim: MP = 16 with a partial tail; MP = 32 (fp64: one row per thread with several passes, bwd1 REREAD)
        "MP 16 partial tail": any(g["MP"] == 16 and g["m"] < 16 for g in trained64.values()),
        "fp64 MP 32, several j passes": any(g["MP"] == 32 and g["j_passes"] >= 2 for g in trained64.values()),
        "fp64 REREAD with m in 17..32": {g["m"] for g in trained64.values() if g["MP"] == 32} >= {20, 24},
        "m 32 trained in fp32": any(g["m"] == 32 for g in dense.values()),
        "16 labels": any(g["labels"] == 16 for g in trained64.values()),
        "4 labels": any(g["labels"] == 4 for g in trained64.values()),
        # neighbour lists
        "list k in {3,17,32,33,48,64}": {g["k"] for g in lists.values()} >= {3, 17, 32, 33, 48, 64},
        "list N in {37,70,100}": {g["N"] for g in lists.values()} >= {37, 70, 100},
        "list TS 32, two slot passes, partial": any(g["TS"] == 32 and g["slot_passes"] == 2 and g["partial_slots"]
                                                    for g in lists.values()),
        "list TS 32, two full slot passes": any(g["TS"] == 32 and g["slot_passes"] == 2 and not g["partial_slots"]
                                                for g in lists.values()),
        "list TS < 32": any(g["TS"] < 32 for g in lists.values()),
        "list bwd2 two 32-slot steps": any(g["bwd2_steps"] == 2 and g["partial_step"] for g in lists.values()),
        "list bwd2 16-row CTAs, partial last": any(g["partial_rows"] and g["N"] > 32 for g in lists.values()),
        "list QR 1 / 8 / 0": {g["QR"] for g in lists.values() if g["N"] > 32} == {0, 1, 8},
        "list Q 1, 5, 10": {g["Q"] for g in lists.values()} >= {1, 5, 10},
        "list C 2 and 5": {g["C"] for g in lists.values()} >= {2, 5},
        "list fp64 MP 32": any(g["MP"] == 32 for g in lists.values()),
    }
    missing = [k for k, v in want.items() if not v]
    assert not missing, missing
    assert FP64_BACKWARD_REJECTED < set(TILE_CASES)
    # a mask must leave valid neighbours in the partial last j pass, or that pass adds nothing that could be wrong
    for name, spec in TILE_CASES.items():
        mask = cases.build_case(spec)["inputs"].get("mask")
        if mask is not None:
            assert mask[:, (spec["N"] - 1) // 32 * 32:].any(), name


# ------------------------------------------------------------------ the driver (GPU)


@functools.lru_cache(maxsize=None)
def _case(name):
    """(case, forward oracle, flat gradient oracle); the numpy oracles run once per case."""
    case = cases.build_case(TILE_CASES[name])
    return case, cases.run_oracle(case), cases.flatten_grads(cases.run_oracle_grad(case))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("name", list(TILE_CASES))
def test_forward_matches_oracle(name, dtype):
    case, want, _ = _case(name)
    mod = util.make_module(case, dtype)
    out = util.run_module(mod, case, dtype)
    util.assert_close(out[0], want[0], what=f"{name} feats", **util.TOL[dtype])
    util.assert_close(out[1], want[1], what=f"{name} coors", **util.TOL[dtype])


GRAD_PARAMS = [(n, dt) for n in TILE_CASES for dt in (torch.float64, torch.float32)
               if not (dt == torch.float64 and n in FP64_BACKWARD_REJECTED)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["saved", "recompute"])
@pytest.mark.parametrize("name,dtype", GRAD_PARAMS, ids=[f"{n}-{'fp64' if d == torch.float64 else 'fp32'}" for n, d in GRAD_PARAMS])
def test_grads_match_oracle(name, dtype, mode, monkeypatch):
    """saved: the forward keeps W2 silu(pre1) per pair for bwd1; recompute: the backward recomputes it with the dense
    forward kernel (EGNN_B200_SAVE_PAIR_MB=0).  fp32 is its own instantiation of every kernel (bwd2's sigmoid runs on
    ex2.approx)."""
    if mode == "recompute":
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")
    case, _, want = _case(name)
    got = util.module_grads(case, dtype)
    util.compare(got, want, util.grad_tol(case, dtype), f"{name} {mode}")


# ------------------------------------------------------------------ configurations the backward cannot run


class _LibWithoutForward:
    """The native library with egnn_layer_forward taken away: a call to it fails the test."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        if name == "egnn_layer_forward":
            raise AssertionError("egnn_layer_forward was called before the backward preflight rejected the configuration")
        return getattr(self._lib, name)


def _assert_training_forward_rejected(case, dtype, monkeypatch, run=None):
    """`run`: the training step to try (default: util.module_grads of the case)."""
    from egnn_pytorch_b200 import _native as nat
    real = nat.load()
    monkeypatch.setattr(nat, "load", lambda: _LibWithoutForward(real))
    with pytest.raises(RuntimeError, match="egnn_layer_backward_workspace_bytes"):
        (run or (lambda: util.module_grads(case, dtype)))()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FP64_BACKWARD_REJECTED))
def test_fp64_backward_over_the_shared_memory_budget_fails_at_the_training_forward(name, monkeypatch):
    """fp64 m_dim = 32 and m_dim = 24 with soft edges (bwd1), 77 per-pair channels (dense bwd2): the training forward
    raises before it launches anything; inference in fp64 and training in fp32 run (the tests above)."""
    case = cases.build_case(TILE_CASES[name])
    _assert_training_forward_rejected(case, torch.float64, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
def test_more_than_16_degree_labels_fail_at_the_training_forward(dtype, monkeypatch):
    spec = dict(TILE_CASES["net_n45_labels16"], cfg=dict(TILE_CASES["net_n45_labels16"]["cfg"], num_adj_degrees=16))
    _assert_training_forward_rejected(cases.build_case(spec), dtype, monkeypatch)
