"""The bf16 tensor-core path (wgmma GEMMs + the fused edge kernels) against the fp64 oracle.

Inputs and parameters are rounded to bf16 first, so the comparison isolates the kernels' internal
rounding (bf16 B' table, bf16 hidden operand, bf16 m_i / h1, tanh.approx) from input quantisation.
Stated tolerance: max|err| <= 1e-2 * max|reference output| for feats and <= 1e-2 * max(max|coordinate
update|, 1) for coors (measured 2e-3 .. 7e-3 of the respective scale); the reference itself run in bf16 deviates from its fp32 self by
1.6e-2 / 4.7e-2 at default init and 0.10 / 0.52 with Xavier weights (BASELINE.md section 2)."""
import numpy as np
import pytest
import torch

import cases
import util

pytestmark = pytest.mark.gpu

L = "layer"
FAST_SPECS = {
    "d64_n160":        dict(kind=L, cfg=dict(dim=64), B=2, N=160, seed=99, init="xavier"),
    "d64_default":     dict(kind=L, cfg=dict(dim=64), B=1, N=257, seed=98),
    "d128_mask":       dict(kind=L, cfg=dict(dim=128), B=2, N=300, seed=97, init="xavier", mask="padded"),
    "d64_soft_norm":   dict(kind=L, cfg=dict(dim=64, soft_edges=True, norm_coors=True, norm_feats=True), B=2, N=96, seed=96,
                            init="xavier", mask="random"),
    "d72_clamp_mean":  dict(kind=L, cfg=dict(dim=72, coor_weights_clamp_value=0.5, m_pool_method="mean"), B=3, N=130, seed=95,
                            init="xavier", mask="padded"),
    "d64_mean_nomask": dict(kind=L, cfg=dict(dim=64, m_pool_method="mean"), B=1, N=64, seed=94, init="xavier"),
    "d64_tiny_n":      dict(kind=L, cfg=dict(dim=64), B=2, N=5, seed=93, init="xavier"),
    "d512_c1":         dict(kind=L, cfg=dict(dim=512), B=1, N=16, seed=92),
    "d512_n256":       dict(kind=L, cfg=dict(dim=512), B=1, N=256, seed=91, init="xavier"),
    "d64_no_coors":    dict(kind=L, cfg=dict(dim=64, update_coors=False), B=1, N=40, seed=90, init="xavier"),
    "d64_no_feats":    dict(kind=L, cfg=dict(dim=64, update_feats=False), B=1, N=40, seed=89, init="xavier"),
    # --- the generic instantiation of the dense kernel: dense edge channels (the reference's own test shape,
    #     tests/test_equivariance.py:13-30), fourier features, other coordinate dimensions (:40), hidden widths
    #     whose last chunk has 1..3 K slabs, degree labels through EGNN_Network
    "d512_edges4":     dict(kind=L, cfg=dict(dim=512, edge_dim=4), B=1, N=16, seed=70, mask="padded"),
    "d64_edges4":      dict(kind=L, cfg=dict(dim=64, edge_dim=4), B=2, N=140, seed=71, init="xavier", mask="padded"),
    "d64_edges2_soft": dict(kind=L, cfg=dict(dim=64, edge_dim=2, soft_edges=True, norm_coors=True, m_pool_method="mean"), B=2, N=70,
                            seed=72, init="xavier", mask="random"),
    "d32_fourier2":    dict(kind=L, cfg=dict(dim=32, fourier_features=2), B=2, N=90, seed=73, init="xavier"),
    "d64_fourier_e1":  dict(kind=L, cfg=dict(dim=64, fourier_features=3, edge_dim=1, coor_weights_clamp_value=0.7), B=1, N=130, seed=74,
                            init="xavier", mask="padded"),
    "d64_c5":          dict(kind=L, cfg=dict(dim=64), B=2, N=50, C=5, seed=75, init="xavier"),
    "d64_c2_edges":    dict(kind=L, cfg=dict(dim=64, edge_dim=3, norm_coors=True), B=1, N=33, C=2, seed=76, init="xavier", mask="padded"),
    "d40_tail":        dict(kind=L, cfg=dict(dim=40), B=2, N=130, seed=77, init="xavier"),            # H = 162 -> 176: last chunk 3 slabs
    "d48_tail_e1":     dict(kind=L, cfg=dict(dim=48, edge_dim=1), B=1, N=520, seed=78, init="xavier"),  # 2 tiles per warpgroup, 5 j-tiles
    "d64_many_rows":   dict(kind=L, cfg=dict(dim=64), B=3, N=700, seed=79, init="xavier", mask="padded"),   # > 2 row groups per CTA: ring reuse
    "net_dense_adj":   dict(kind="network", cfg=dict(depth=2, dim=32, num_tokens=11, num_adj_degrees=2, adj_dim=4), B=2, N=40, seed=69,
                            init="xavier", adj="chain", mask="padded"),
    "net_dense_adj_e": dict(kind="network", cfg=dict(depth=2, dim=32, num_tokens=11, num_edge_tokens=5, edge_dim=3, num_adj_degrees=3,
                                                     adj_dim=2), B=1, N=30, seed=68, init="xavier", adj="chain", edges=True),
    # --- neighbour lists on the tensor-core path (tc_knn_kernel)
    "knn_d64_k8":      dict(kind=L, cfg=dict(dim=64, num_nearest_neighbors=8), B=2, N=200, seed=80, init="xavier"),
    "knn_d64_k32_e4":  dict(kind=L, cfg=dict(dim=64, edge_dim=4, num_nearest_neighbors=32), B=2, N=100, seed=81, init="xavier",
                            mask="padded"),
    "knn_d32_k5_e2":   dict(kind=L, cfg=dict(dim=32, edge_dim=2, num_nearest_neighbors=5, soft_edges=True, norm_coors=True,
                                             coor_weights_clamp_value=1.0, m_pool_method="mean"), B=3, N=37, seed=82,
                            init="xavier", mask="random"),
    "knn_d64_radius":  dict(kind=L, cfg=dict(dim=64, num_nearest_neighbors=12, valid_radius=2.0), B=1, N=150, seed=83,
                            init="xavier", mask="full"),
    "knn_d256_c4":     dict(kind=L, cfg=dict(dim=256, edge_dim=4, num_nearest_neighbors=32), B=1, N=300, seed=84),
    "knn_k_eq_n":      dict(kind=L, cfg=dict(dim=64, num_nearest_neighbors=20), B=2, N=20, seed=85, init="xavier"),
    "adj_sparse_d64":  dict(kind=L, cfg=dict(dim=64, only_sparse_neighbors=True), B=2, N=50, seed=86, init="xavier", adj="chain",
                            mask="full"),
    "knn_mean_nomask": dict(kind=L, cfg=dict(dim=64, num_nearest_neighbors=7, m_pool_method="mean"), B=1, N=33, seed=87,
                            init="xavier"),
    # --- the generic instantiation of the neighbour-list kernel (fourier, > 4 edge channels, C != 3, degree labels)
    "knn_fourier2":    dict(kind=L, cfg=dict(dim=64, num_nearest_neighbors=7, fourier_features=2), B=2, N=60, seed=60, init="xavier",
                            mask="padded"),
    "knn_c5_e2":       dict(kind=L, cfg=dict(dim=32, num_nearest_neighbors=6, edge_dim=2, norm_coors=True), B=2, N=40, C=5, seed=61,
                            init="xavier"),
    "knn_e6_soft":     dict(kind=L, cfg=dict(dim=32, num_nearest_neighbors=5, edge_dim=6, soft_edges=True, m_pool_method="mean"), B=1, N=50,
                            seed=62, init="xavier", mask="random"),
    "net_c5_like":     dict(kind="network", cfg=dict(depth=3, dim=32, num_tokens=21, num_adj_degrees=3, adj_dim=8,
                                                     only_sparse_neighbors=True), B=1, N=96, seed=63, adj="chain", mask="full"),
    "net_c5_xavier":   dict(kind="network", cfg=dict(depth=2, dim=32, num_tokens=21, num_adj_degrees=2, adj_dim=4, edge_dim=2,
                                                     num_edge_tokens=4, only_sparse_neighbors=True), B=2, N=40, seed=64, init="xavier",
                            adj="chain", edges=True, mask="padded"),
    "net_global_bf16": dict(kind="network", cfg=dict(depth=2, dim=32, num_tokens=9, global_linear_attn_every=1, global_linear_attn_heads=2,
                                                     global_linear_attn_dim_head=16, num_global_tokens=3), B=2, N=24, seed=66,
                            init="xavier", mask="padded"),      # attention block in fp32 between bf16 tensor-core layers
    # depth 1: with more layers the bf16 coordinate round-off of layer 1 may flip a near-tie of layer 2's top-k, which is a
    # property of re-selecting neighbours, not of the kernels (the full c3 shape is covered in test_gpu_baseline_configs)
    "net_c3_like":     dict(kind="network", cfg=dict(depth=1, dim=32, num_tokens=21, num_positions=128, num_nearest_neighbors=8,
                                                     coor_weights_clamp_value=2.0), B=1, N=128, seed=65, mask="full"),
}


def bf16_round(a):
    return torch.from_numpy(np.asarray(a, np.float64)).bfloat16().double().numpy()


def run_fast(spec):
    case = cases.build_case(spec)
    case["params"] = {k: bf16_round(v) for k, v in case["params"].items()}
    if np.issubdtype(np.asarray(case["inputs"]["feats"]).dtype, np.floating):      # token ids stay integers
        case["inputs"]["feats"] = bf16_round(case["inputs"]["feats"])
    case["inputs"]["coors"] = bf16_round(case["inputs"]["coors"])      # a bf16 module is fed bf16 coordinates
    if case["inputs"].get("edges") is not None and np.issubdtype(np.asarray(case["inputs"]["edges"]).dtype, np.floating):
        case["inputs"]["edges"] = bf16_round(case["inputs"]["edges"])
    mod = util.make_module(case, torch.bfloat16)
    out = util.run_module(mod, case, torch.bfloat16)
    torch.cuda.synchronize()
    return case, mod, out


@pytest.mark.parametrize("name", list(FAST_SPECS))
def test_fast_path_matches_oracle(name):
    case, mod, out = run_fast(FAST_SPECS[name])
    layers = [l[1] for l in mod.layers] if hasattr(mod, "layers") else [mod]
    assert all(l.last_path == "bf16-tc" for l in layers)
    assert out[0].dtype == torch.bfloat16
    want = cases.run_oracle(case)
    f_scale = max(1e-3, float(np.abs(want[0]).max()))
    c_scale = float(np.abs(want[1] - case["inputs"]["coors"]).max())
    f_err, c_err = util.max_err(out[0], want[0]), util.max_err(out[1], want[1])
    print(f"{name}: feats err {f_err:.3e} (scale {f_scale:.3e}), coors err {c_err:.3e} (update scale {c_scale:.3e})")
    assert np.isfinite(out[0].float().cpu().numpy()).all() and np.isfinite(out[1].float().cpu().numpy()).all()
    assert f_err <= 1e-2 * f_scale
    assert c_err <= 1e-2 * max(c_scale, 1.0)           # coordinates are O(1): where the update nearly cancels, 1e-2 absolute


def test_fast_path_falls_back_to_fp32_simt_when_unsupported():
    case = cases.build_case(cases.SPECS["dense_mdim32"])          # m_dim = 32: not on the tensor-core path
    mod = util.make_module(case, torch.bfloat16)
    with pytest.warns(UserWarning, match="fp32"):
        out = util.run_module(mod, case, torch.bfloat16)
    assert mod.last_path == "fp32-simt" and out[0].dtype == torch.bfloat16


@pytest.mark.parametrize("name", ["d64_n160", "d64_edges4", "d128_mask", "knn_d64_k8", "knn_d64_k32_e4", "knn_fourier2"])
def test_fast_path_row_range_equals_full_forward(name):
    """Row-sharded use (EgnnLayerDesc.row_begin / row_end): rows inside the range are bit-identical to the full
    forward's, rows outside keep the inputs."""
    case, mod, full = run_fast(FAST_SPECS[name])
    ins = case["inputs"]
    n = ins["feats"].shape[1]
    t = lambda key: util.to_torch(ins.get(key), torch.bfloat16, "cuda")
    for (r0, r1) in [(0, n // 3), (n // 3, n - 5), (n - 5, n), (7, 8)]:
        with torch.no_grad():
            f, x = mod(t("feats"), t("coors"), t("edges"), mask=t("mask"), _rows=(r0, r1))
        assert mod.last_path == "bf16-tc"
        assert torch.equal(f[:, r0:r1], full[0][:, r0:r1]) and torch.equal(x[:, r0:r1], full[1][:, r0:r1])
        keep = torch.ones(n, dtype=torch.bool, device="cuda"); keep[r0:r1] = False
        assert torch.equal(f[:, keep], t("feats")[:, keep]) and torch.equal(x[:, keep].float(), t("coors")[:, keep].float())


def test_fast_equivariance():
    """tests/test_equivariance.py:8-34 on the bf16 path; coordinates and distances stay fp32, so the
    rotation only perturbs d_ij by fp32 rounding -- the error is far below bf16 epsilon."""
    spec = dict(kind=L, cfg=dict(dim=64), B=1, N=128, seed=5)
    case = cases.build_case(spec)
    mod = util.make_module(case, torch.bfloat16)
    f = util.to_torch(case["inputs"]["feats"], torch.bfloat16, "cuda")
    x = torch.from_numpy(case["inputs"]["coors"]).double()
    g = torch.Generator().manual_seed(1)
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    t = torch.randn(1, 1, 3, generator=g, dtype=torch.float64)
    f1, c1 = mod(f, (x @ q + t).float().cuda())
    f2, c2 = mod(f, x.float().cuda())
    ef = float((f1.float() - f2.float()).abs().max())
    ec = float((c1.double().cpu() - (c2.double().cpu() @ q + t)).abs().max())
    print(f"bf16 path equivariance: feats {ef:.3e} coors {ec:.3e}")
    assert ec < 1e-4
    assert ef <= 2 ** -7 * float(f2.float().abs().max())          # at most one bf16 ulp of the output


def test_tc_gemm_standalone():
    import ctypes as C
    from egnn_pytorch_b200 import _native as nat
    lib = nat.load()
    torch.manual_seed(0)
    for (M, N, K) in [(128, 128, 64), (200, 136, 72), (4096, 2112, 512), (77, 1024, 528)]:
        A = torch.randn(M, K, device="cuda").bfloat16()
        W = torch.randn(N, K, device="cuda").bfloat16()
        bias = torch.randn(N, device="cuda")
        o = torch.empty(M, N, device="cuda", dtype=torch.float32)
        rc = lib.egnn_gemm_bf16(M, N, K, A.data_ptr(), W.data_ptr(), bias.data_ptr(), 0.5, 0, o.data_ptr(), 1, None)
        assert rc == 0
        torch.cuda.synchronize()
        ref = 0.5 * (A.double() @ W.double().t() + bias.double())
        assert float((o.double() - ref).abs().max()) <= 1e-4 * float(ref.abs().max()) + 1e-4
