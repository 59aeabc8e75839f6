"""The torch restatement of tests/torch_reference.py pinned on the CPU: forward and autograd gradients equal the
golden-pinned numpy oracles over every gradient case (layers and networks), and row blocks of any size give the
whole-graph gradient."""
import numpy as np
import pytest
import torch

import cases
import torch_reference as TR


def _forward(case):
    ins = case["inputs"]
    if case["kind"] == "network":
        f, x, _ = TR.network(case["params"], case["ncfg"], ins["feats"], ins["coors"], ins.get("adj_mat"), ins.get("edges"),
                             ins.get("mask"))
        return f, x
    return TR.layer(case["params"], case["cfg"], ins["feats"], ins["coors"], ins.get("edges"), ins.get("mask"),
                    ins.get("adj_mat"))


def _grads(case, chunk=None):
    ins = case["inputs"]
    gf, gx = cases.upstream_grads(case)
    if case["kind"] == "network":
        return TR.network_grads(case["params"], case["ncfg"], ins["feats"], ins["coors"], gf, gx, ins.get("adj_mat"),
                                ins.get("edges"), ins.get("mask"), chunk=chunk)
    return TR.layer_grads_chunked(case["params"], case["cfg"], ins["feats"], ins["coors"], gf, gx, ins.get("edges"),
                                  ins.get("mask"), ins.get("adj_mat"), chunk=chunk)


def _rel(got, want):
    return float(np.abs(np.asarray(got) - want).max()) / max(1.0, float(np.abs(want).max()))


@pytest.mark.parametrize("name", cases.GRAD_SPECS)
def test_forward_and_gradients_equal_the_oracles(name):
    case = cases.build_case(cases.SPECS[name])
    got = _forward(case)
    want = cases.run_oracle(case)
    assert _rel(got[0], want[0]) <= 1e-12 and _rel(got[1], want[1]) <= 1e-12
    g = {k: v.numpy() for k, v in _grads(case).items()}
    w = cases.flatten_grads(cases.run_oracle_grad(case))
    assert set(g) == set(w), sorted(set(g) ^ set(w))
    # CoorsNorm: both carry cancellation noise of the 1/eps self pair (util.grad_tol)
    tol = 1e-7 if case["spec"]["cfg"].get("norm_coors") else 1e-10
    bad = {k: _rel(g[k], w[k]) for k in w if _rel(g[k], w[k]) > tol}
    assert not bad, bad


@pytest.mark.parametrize("name", ["dense_mask_padded", "dense_fourier", "knn_edges_mask", "adj_sparse_random", "net_c5_xavier",
                                  "net_c3_xavier"])
def test_row_blocks_of_any_size_give_the_whole_gradient(name):
    case = cases.build_case(cases.SPECS[name])
    n = case["spec"]["N"]
    whole = _grads(case, chunk=n)
    for chunk in (1, 7):
        got = _grads(case, chunk=chunk)
        for k, v in whole.items():
            err = float((got[k] - v).abs().max()) / max(1.0, float(v.abs().max()))
            assert err <= 1e-13, (chunk, k, err)


def test_a_selects_lists_with_ok_flags_are_not_empty_slots():
    """A slot beyond valid_radius still carries a message without a mask (the reference masks it only through `mask`);
    an empty (-1) slot of edge-list mode never does."""
    case = cases.build_case(cases.SPECS["knn_radius_nomask"])
    ins, P, cfg = case["inputs"], case["params"], case["cfg"]
    want = TR.layer(P, cfg, ins["feats"], ins["coors"])
    x = torch.as_tensor(ins["coors"])
    idx, ok = TR.select(cfg, ((x[:, :, None] - x[:, None]) ** 2).sum(-1), None, None)
    assert not ok.all()
    got = TR.layer(P, cfg, ins["feats"], ins["coors"], neighbors=idx, ok=ok)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    empty = TR.layer(P, cfg, ins["feats"], ins["coors"], neighbors=torch.where(ok, idx, -1))
    assert not torch.equal(empty[1], want[1])
    masked = dict(mask=np.ones(ins["feats"].shape[:2], bool))
    got = TR.layer(P, cfg, ins["feats"], ins["coors"], neighbors=idx, ok=ok, **masked)
    assert torch.allclose(got[1], TR.layer(P, cfg, ins["feats"], ins["coors"], **masked)[1], rtol=0, atol=0)
