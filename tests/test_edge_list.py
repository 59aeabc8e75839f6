"""Edge-list mode (`EGNN.forward(..., neighbors=)`, SURVEY.md section 8(f) rank 3) against the oracle's independent
flat-edge restatement (`oracle.egnn_oracle.egnn_layer_forward_edge_list`, following the message / aggregate
structure of reference egnn_pytorch_geometric.py:182-267 in the dense layer's conventions).

CPU part: the edge-list oracle is pinned to the reference-pinned gather oracle on the lists the top-k would pick,
and its gradient restatement to finite differences.  GPU part: random lists with empty (-1) slots, duplicate-free,
in fp64 / fp32 / bf16 forward and fp64 / fp32 backward (with W2 silu(pre1) saved by the forward or recomputed)."""
import functools

import numpy as np
import pytest
import torch

import cases
import util
from oracle import egnn_oracle as O
from oracle import egnn_oracle_grad as G

EDGE_CASES = {
    # name: (layer cfg, B, N, k, C, mask?, init)
    "plain":        (dict(dim=16), 2, 24, 6, 3, False, "xavier"),
    "edges_mask":   (dict(dim=16, edge_dim=3, soft_edges=True), 2, 20, 5, 3, True, "xavier"),
    "mean_mask":    (dict(dim=8, m_pool_method="mean", norm_coors=True, edge_dim=1), 1, 30, 7, 3, True, "xavier"),
    "mean_nomask":  (dict(dim=8, m_pool_method="mean", coor_weights_clamp_value=0.5), 2, 18, 4, 3, False, "xavier"),
    "fourier_c5":   (dict(dim=12, fourier_features=2, norm_feats=True), 1, 16, 5, 5, True, "xavier"),
    "k33":          (dict(dim=8, edge_dim=2), 1, 48, 33, 3, False, "xavier"),
    "default_init": (dict(dim=32, edge_dim=4), 2, 40, 9, 3, True, "default"),
    # tile boundaries of the neighbour-list kernels (test_gpu_tile_boundaries.py checks that they stay covered): the
    # slot group TS of pair_kernel / bwd1 / bwd3 (next power of two >= k, at most 32) with one or two slot passes,
    # the 32-slot steps and 16-row CTAs of bwd2 (N not a multiple of 16), and bwd2's per-pair channel instantiations
    # QR = 1 (Q = 1), 8 (Q <= 8) and 0 (Q > 8)
    "k3_q1":        (dict(dim=16, m_pool_method="mean"), 2, 37, 3, 3, True, "xavier"),
    "k17_q5_c2":    (dict(dim=16, fourier_features=2, soft_edges=True), 2, 70, 17, 2, True, "xavier"),
    "k32_q10":      (dict(dim=12, edge_dim=9, norm_coors=True), 1, 100, 32, 3, False, "xavier"),
    "k48_c5_mean":  (dict(dim=8, edge_dim=2, m_pool_method="mean", coor_weights_clamp_value=1.0), 2, 70, 48, 5, True, "xavier"),
    "k64_q1":       (dict(dim=8, m_pool_method="mean"), 1, 100, 64, 3, False, "xavier"),
    "k33_mdim24":   (dict(dim=12, m_dim=24, edge_dim=1), 2, 37, 33, 3, True, "xavier"),   # fp64: 32-wide accumulators
}


def build(name, seed=0):
    cfg, B, N, k, Cd, with_mask, init = EDGE_CASES[name]
    spec = dict(kind="layer", cfg=cfg, B=B, N=N, C=Cd, seed=1000 + seed, init=init, mask="padded" if with_mask else None)
    case = cases.build_case(spec)
    rs = np.random.RandomState(77 + seed)
    nb = np.stack([np.stack([rs.permutation(N)[:k] for _ in range(N)]) for _ in range(B)]).astype(np.int64)
    nb[:, ::3, -2:] = -1                    # every third node has two empty slots
    nb[0, 5, :] = -1                        # one node has no neighbours at all
    nb[:, 7, 0] = 7                         # a self edge
    return case, nb


@pytest.mark.parametrize("name", ["knn_edges_mask", "knn_mean_fourier", "knn_norm_coors", "knn_basic", "adj_sparse_random",
                                  "knn_k33", "knn_k32_c5", "knn_radius_nomask"])
def test_edge_list_oracle_is_pinned_to_the_gather_oracle(name):
    """On the lists top-k would pick (slots whose nbhd_mask is False dropped when a mask is given), the flat-edge
    restatement must reproduce the gather oracle, which is itself pinned to reference outputs."""
    case = cases.build_case(cases.SPECS[name])
    ins, cfg = case["inputs"], case["cfg"]
    idx, ok, _ = O.neighbour_selection(cfg, np.asarray(ins["coors"], np.float64), ins.get("mask"), ins.get("adj_mat"))
    nb = np.where(ok, idx, -1) if ins.get("mask") is not None else idx      # :296 -- nbhd_mask only acts with a mask
    want = O.egnn_layer_forward(case["params"], cfg, ins["feats"], ins["coors"], ins.get("edges"), ins.get("mask"), ins.get("adj_mat"))
    got = O.egnn_layer_forward_edge_list(case["params"], cfg, ins["feats"], ins["coors"], nb, ins.get("edges"), ins.get("mask"))
    assert np.abs(got[0] - want[0]).max() < 1e-12 and np.abs(got[1] - want[1]).max() < 1e-12


@pytest.mark.parametrize("name", ["edges_mask", "mean_mask", "mean_nomask", "fourier_c5"])
def test_edge_list_grad_oracle_against_finite_differences(name):
    case, nb = build(name)
    ins, cfg, P = case["inputs"], case["cfg"], case["params"]
    rs = np.random.RandomState(5)
    gf, gx = rs.randn(*ins["feats"].shape), rs.randn(*ins["coors"].shape)

    def loss(feats, coors, edges, params):
        fo, xo = O.egnn_layer_forward_edge_list(params, cfg, feats, coors, nb, edges, ins.get("mask"))
        return float((fo * gf).sum() + (xo * gx).sum())

    g = G.egnn_layer_backward(P, cfg, ins["feats"], ins["coors"], ins.get("edges"), ins.get("mask"), None, gf, gx, neighbors=nb)
    vf, vx = rs.randn(*ins["feats"].shape), rs.randn(*ins["coors"].shape)
    ve = None if ins.get("edges") is None else rs.randn(*ins["edges"].shape)
    vp = {k: rs.randn(*np.shape(v)) for k, v in P.items()}
    eps = 1e-6
    plus = loss(ins["feats"] + eps * vf, ins["coors"] + eps * vx, None if ve is None else ins["edges"] + eps * ve,
                {k: np.asarray(v) + eps * vp[k] for k, v in P.items()})
    minus = loss(ins["feats"] - eps * vf, ins["coors"] - eps * vx, None if ve is None else ins["edges"] - eps * ve,
                 {k: np.asarray(v) - eps * vp[k] for k, v in P.items()})
    fd = (plus - minus) / (2 * eps)
    an = (g["feats"] * vf).sum() + (g["coors"] * vx).sum() + sum((g["params"][k] * vp[k]).sum() for k in g["params"])
    if ve is not None:
        an += (g["edges"] * ve).sum()
    assert abs(fd - an) <= 2e-6 * max(1.0, abs(an)), (fd, an)


def _run_cuda(case, nb, dtype, **extra):
    mod = util.make_module(case, dtype, device="cuda", **extra)
    ins = case["inputs"]
    t = lambda key: util.to_torch(ins.get(key), dtype, "cuda")
    with torch.no_grad():
        out = mod(t("feats"), t("coors"), t("edges"), mask=t("mask"), neighbors=torch.from_numpy(nb).cuda())
    return mod, out


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(EDGE_CASES))
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
def test_edge_list_forward_matches_oracle(name, dtype):
    case, nb = build(name)
    ins = case["inputs"]
    want = O.egnn_layer_forward_edge_list(case["params"], case["cfg"], ins["feats"], ins["coors"], nb, ins.get("edges"), ins.get("mask"))
    _, got = _run_cuda(case, nb, dtype)
    atol, rtol = (1e-9, 1e-9) if dtype == torch.float64 else (2e-5, 1e-4)
    util.assert_close(got[0], want[0], atol=atol, rtol=rtol, what=f"{name} feats")
    util.assert_close(got[1], want[1], atol=atol, rtol=rtol, what=f"{name} coors")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(EDGE_CASES))
def test_edge_list_forward_bf16_matches_oracle(name):
    """bf16 modules: inputs / parameters rounded to bf16 first so the oracle sees the same numbers; gate 1e-2 of the
    output scale (feats) and of max(coordinate update scale, 1) (coors)."""
    case, nb = build(name)
    rnd = lambda v: torch.from_numpy(np.asarray(v, np.float64)).bfloat16().double().numpy()
    case["params"] = {k: rnd(v) for k, v in case["params"].items()}
    for key in ("feats", "edges", "coors"):             # a bf16 module is fed bf16 coordinates as well
        if case["inputs"].get(key) is not None:
            case["inputs"][key] = rnd(case["inputs"][key])
    ins = case["inputs"]
    want = O.egnn_layer_forward_edge_list(case["params"], case["cfg"], ins["feats"], ins["coors"], nb, ins.get("edges"), ins.get("mask"))
    mod, got = _run_cuda(case, nb, torch.bfloat16)
    ferr = util.max_err(got[0], want[0]) / max(1.0, float(np.abs(want[0]).max()))
    cscale = max(1.0, float(np.abs(want[1] - ins["coors"]).max()))        # coordinates are O(1): the gate of test_gpu_fast.py
    cerr = util.max_err(got[1], want[1]) / cscale
    cfg = case["cfg"]
    if cfg["dim"] % 8 == 0 and nb.shape[-1] <= 32 and cfg["m_dim"] == 16:      # what the tensor-core kernels cover
        assert mod.last_path == "bf16-tc"
    assert ferr < 1e-2 and cerr < 1e-2, (name, mod.last_path, ferr, cerr)


BACKWARD_CASES = ["plain", "edges_mask", "mean_mask", "mean_nomask", "fourier_c5", "k33", "k3_q1", "k17_q5_c2", "k32_q10",
                  "k48_c5_mean", "k64_q1", "k33_mdim24"]


@functools.lru_cache(maxsize=None)
def _grad_case(name):
    """(case, neighbour lists, flat oracle gradients) of an EDGE_CASES entry; the oracle runs once per case."""
    case, nb = build(name)
    return case, nb, cases.flatten_grads(cases.run_oracle_grad(case, neighbors=nb))


@pytest.mark.gpu
@pytest.mark.parametrize("name", BACKWARD_CASES)
def test_edge_list_backward_matches_grad_oracle(name):
    case, nb, want = _grad_case(name)
    got = util.module_grads(case, torch.float64, neighbors=nb)
    util.compare(got, want, 1e-8, f"{name} vs oracle")


@pytest.mark.gpu
@pytest.mark.parametrize("name", BACKWARD_CASES)
@pytest.mark.parametrize("dtype,mode", [(torch.float64, "recompute"), (torch.float32, "saved"), (torch.float32, "recompute")],
                         ids=["fp64-recompute", "fp32-saved", "fp32-recompute"])
def test_edge_list_backward_fp32_and_recompute_match_grad_oracle(name, dtype, mode, monkeypatch):
    """The other three instantiations of the list backward: the fp32 kernels (bwd2's ex2.approx sigmoid among them),
    and both types with W2 silu(pre1) recomputed by pair_kernel instead of saved by the forward."""
    if mode == "recompute":
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")
    case, nb, want = _grad_case(name)
    got = util.module_grads(case, dtype, neighbors=nb)
    util.compare(got, want, 1e-8 if dtype == torch.float64 else util.grad_tol(case, dtype), f"{name} {mode} vs oracle")
