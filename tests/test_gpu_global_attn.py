"""GlobalLinearAttention (csrc/global_attn.cu) on the device against the fp64 oracle, at its kernels' boundaries.

The reference is `oracle.egnn_oracle.global_linear_attention` in fp64 (the net_global_* golden fixtures pin it to the
reference).  Each case's parameters come from its seed with the scheme of cases.gen_network_params: Linear weights
N(0, 1/fan_in), LayerNorm weights 1 + 0.2 N(0, 1), biases 0.1 N(0, 1), so that no path hides behind the biases.  Both
outputs (x_out and queries_out) are compared.

The case table crosses the boundaries of the launch code, mirrored in `geometry` and held there by
test_table_covers_every_boundary (at 132 SMs, an H100 SXM):
  launch_gemm           the eight Linear layers on the skinny kernel with 1, 2 and 4 columns per warp and on the tiled
                        kernel; the GELU epilogue on both; Mr <= 16 with K too large for the skinny kernel's 96 KiB of
                        staging (K > 1536 in fp32, K > 768 in fp64)
  ga_softmax_av_kernel  N = 1, 256, 257 and > 512 (1 to 3 strided passes); dh dividing 256, not dividing it (idle
                        threads), dh = 256 (one group) and dh = 320 (a partial second d0 pass)
  ga_attn2_kernel       T = 1 and T = 32 (sc[32] full), dh > 32 (lanes loop over channels); T = 33 takes the fallback
  ga_layernorm_kernel   dim < 32, dim not a multiple of 32, dim > 512
  masks                 none, padded, random, one graph fully masked, one valid node per graph; bool, uint8 and float
`big_logits` scales both to_q weights by 30, so that attention logits reach ~1e2 and exp overflows fp32 unless the
softmax subtracts its maximum.

Gates:
  fp64  util.TOL[float64] against the oracle, and 1e-10 against the module's own PyTorch arithmetic (_forward_autograd)
        in fp64, which ties the inference and training paths together
  fp32  max |error| / max(1, max |reference|) over both outputs, TOL_F32 (TOL_F32_BIG_LOGITS for big_logits, whose
        logits of ~1.3e2 turn the fp32 rounding of a logit into ~1e-5 of relative change in its exp)
  bf16  parameters and inputs rounded to bf16 (as in test_gpu_fast.run_fast), the block computed in fp32 and its
        outputs rounded to bf16: the same measure, TOL_BF16
Worst value over the table, measured on an H100 80GB HBM3 (700 W power limit), and the tolerance (2.6x - 4x that):
  fp32  7.7e-7  (d528, x_out)                        -> TOL_F32 2.5e-6
  fp32  1.7e-5  (big_logits, x_out)                  -> TOL_F32_BIG_LOGITS 5e-5
  bf16  3.3e-3  (dh256, queries_out)                 -> TOL_BF16 1e-2
  (fp64: at most 2.8e-14 of the output scale, big_logits; 1.6e-15 elsewhere)

Sensitivity: each of these kernel mutations (none of them reads or writes out of bounds), applied one at a time on the
same H100, fails test_matches_oracle in the cases named (both types unless a type is given):
  1. unbiased variance in ga_layernorm_kernel        every kernel-path case (relative error 9e-4 .. 3e-2)
  2. only the first d0 pass of ga_softmax_av_kernel  dh320 (fp64 0.23; fp32 NaN from the unwritten channels)
  3. the mask read as mask[n], not mask[b*N + n]     every case with a mask (3e-2 .. 0.95)
  4. no max subtraction in either softmax            dh320 (NaN: the fully masked graph), big_logits in fp32 (NaN)
  5. gelu_acc as the tanh approximation              every kernel-path case (8.7e-5 .. 1.4e-4)
  6. scale applied twice in ga_attn2_kernel          every case whose T tokens differ (9e-3 .. 0.19); not n1, t1 or dh256,
                                                     where one node or one token makes attn2 uniform
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import cases
import util
from launch_geometry import H100_SMS
from oracle import egnn_oracle as O
from util import nat  # noqa: F401  (module-scoped fixture)

SKINNY_WARPS, SKINNY_SMEM = 4, 96 * 1024
T_MAX = 32                     # ga_attn2_kernel's sc[32]; the module runs more tokens through PyTorch
TOL_F32 = 2.5e-6
TOL_F32_BIG_LOGITS = 5e-5      # logits ~1.3e2: fp32 rounding of a logit moves exp() by ~1e-5 relative
TOL_BF16 = 1e-2
F32, F64 = torch.float32, torch.float64


def _case(dim, heads, dh, T, B, N, mask=None, mask_dtype="bool", seed=0, q_scale=1.0):
    return dict(dim=dim, heads=heads, dh=dh, T=T, B=B, N=N, mask=mask, mask_dtype=mask_dtype, seed=seed, q_scale=q_scale)


CASES = {
    # the reference's defaults (heads 8, dim_head 64); two strided passes over N
    "default":     _case(64, 8, 64, 4, 2, 300, "padded", seed=1),
    # every GEMM skinny; a softmax over one node
    "n1":          _case(32, 2, 16, 3, 3, 1, seed=2),
    # 256 // 48 = 5 groups: 16 idle threads; partial last LayerNorm lane pass (dim 40)
    "n256":        _case(40, 3, 48, 5, 2, 256, "random", seed=3),
    "n257":        _case(40, 3, 48, 5, 2, 257, "random", seed=4),
    # dh not dividing 256 (10 groups, 16 idle threads); dim < 32; three passes over N
    "dh24":        _case(24, 3, 24, 5, 2, 700, "random", seed=5),
    # groups = 1 exactly; one head; one valid node per graph
    "dh256":       _case(64, 1, 256, 2, 2, 100, "one", seed=6),
    # a partial second d0 pass; kv2 skinny with 2 columns; the last graph fully masked
    "dh320":       _case(48, 2, 320, 4, 2, 90, "empty", seed=7),
    # kv1 / kv2 skinny with 4 columns, q with 2; a1_wo (K = 1088) tiled in fp64 only
    "cols4":       _case(64, 8, 136, 4, 2, 7, "random", "bool", seed=8),
    # the feed-forward GEMMs skinny (GELU; residual)
    "gelu_skinny": _case(40, 2, 16, 2, 2, 7, "random", "uint8", seed=9),
    # ff_w1 skinny with 4 columns and GELU; ff_w2 (K = 2112) tiled in both types; dim > 512
    "d528":        _case(528, 4, 32, 2, 2, 6, "random", "float", seed=10),
    # ff_w2 K = 800: skinny in fp32, tiled in fp64
    "d200_f64k":   _case(200, 4, 50, 3, 2, 8, seed=11),
    # T = 1; T = 32 fills sc[32] (and the T-side GEMMs go tiled); T = 33 runs through PyTorch
    "t1":          _case(32, 4, 8, 1, 2, 120, "padded", seed=12),
    "t32":         _case(32, 4, 8, 32, 2, 120, "padded", seed=13),
    "t33":         _case(32, 4, 8, 33, 2, 120, "padded", seed=14),
    # 64 groups of 4 channels; 16 heads; N > 512
    "h16":         _case(64, 16, 4, 4, 2, 520, "random", seed=15),
    # to_q x30: logits ~1e2, beyond exp's fp32 range unless the maximum is subtracted
    "big_logits":  _case(64, 4, 16, 4, 2, 200, "padded", seed=16, q_scale=30.0),
}


# ------------------------------------------------------------------ launch geometry (mirrors ga_forward / launch_gemm)


def gemm_kind(Mr, Nout, K, es, sms):
    V = 16 // es
    if Mr <= 16 and 16 * (-(-K // V) * V) * es <= SKINNY_SMEM:
        cols = 4 if Nout >= sms * SKINNY_WARPS * 4 else (2 if Nout >= sms * SKINNY_WARPS * 2 else 1)
        return f"skinny{cols}"
    return "tiled"


def geometry(case, dtype, sms=H100_SMS):
    """-> dict of the launch choices ga_forward makes for `case`; fallback=True when the module runs it in PyTorch."""
    if case["T"] > T_MAX:
        return dict(fallback=True, T=case["T"])
    es = 8 if dtype == F64 else 4
    dim, dh, T = case["dim"], case["dh"], case["T"]
    inner, BN, BT = case["heads"] * dh, case["B"] * case["N"], case["B"] * case["T"]
    gemms = {                  # name: (Mr, Nout, K); ff1 has the GELU epilogue
        "a1_q": (BT, inner, dim), "a1_kv": (BN, 2 * inner, dim), "a1_out": (BT, dim, inner),
        "a2_q": (BN, inner, dim), "a2_kv": (BT, 2 * inner, dim), "a2_out": (BN, dim, inner),
        "ff1": (BN, 4 * dim, dim), "ff2": (BN, dim, 4 * dim),
    }
    return dict(
        fallback=False,
        gemm={k: gemm_kind(*v, es, sms) for k, v in gemms.items()},
        k_fallback=sorted(k for k, (Mr, _, _) in gemms.items() if Mr <= 16 and gemm_kind(*gemms[k], es, sms) == "tiled"),
        # idle: threads without a channel in the last d0 pass
        softmax=dict(groups=max(1, 256 // dh), d0_passes=-(-dh // 256), n_passes=-(-case["N"] // 256),
                     idle=256 - (256 // dh) * dh if dh <= 256 else -dh % 256),
        attn2=dict(T=T, lane_passes=-(-dh // 32)),
        layernorm=dict(lane_passes=-(-dim // 32), partial=dim % 32 != 0),
    )


# ------------------------------------------------------------------ parameters, inputs, reference


def make_case(name):
    """-> (params {state-dict key: float64 array}, x [B,N,dim], queries [B,T,dim], mask [B,N] numpy or None)."""
    c = CASES[name]
    rs = np.random.RandomState(1000 + c["seed"])
    d, inner = c["dim"], c["heads"] * c["dh"]
    lin = lambda o, i: rs.standard_normal((o, i)) * math.sqrt(1.0 / i)
    P = {}
    for nm in ("norm_seq", "norm_queries", "ff.0"):
        P[nm + ".weight"] = 1.0 + 0.2 * rs.standard_normal((d,))
        P[nm + ".bias"] = 0.1 * rs.standard_normal((d,))
    for a in ("attn1", "attn2"):
        P[a + ".to_q.weight"] = lin(inner, d) * c["q_scale"]
        P[a + ".to_kv.weight"] = lin(2 * inner, d)
        P[a + ".to_out.weight"] = lin(d, inner)
        P[a + ".to_out.bias"] = 0.1 * rs.standard_normal((d,))
    P["ff.1.weight"] = lin(4 * d, d)
    P["ff.1.bias"] = 0.1 * rs.standard_normal((4 * d,))
    P["ff.3.weight"] = lin(d, 4 * d)
    P["ff.3.bias"] = 0.1 * rs.standard_normal((d,))
    B, N, T = c["B"], c["N"], c["T"]
    x = rs.standard_normal((B, N, d))
    q = rs.standard_normal((B, T, d))
    mk = c["mask"]
    if mk is None:
        m = None
    elif mk == "padded":
        m = np.arange(N)[None, :] < np.asarray([N - 1 - (37 * b) % max(1, N // 3) for b in range(B)])[:, None]
    elif mk == "random":
        m = rs.uniform(size=(B, N)) < 0.7
        m[:, 0] = True
    elif mk == "one":         # exactly one valid node per graph, at a different place in each
        m = np.zeros((B, N), bool)
        m[np.arange(B), rs.randint(0, N, B)] = True
    elif mk == "empty":       # the last graph has no valid node: it attends uniformly (reference :101-104)
        m = rs.uniform(size=(B, N)) < 0.7
        m[-1] = False
    return P, x, q, m


def mask_tensor(m, kind, device):
    if m is None:
        return None
    t = torch.from_numpy(m.copy())
    return {"bool": t, "uint8": t.to(torch.uint8), "float": t.to(torch.float32)}[kind].to(device)


def oracle(P, x, q, m, heads):
    return O.global_linear_attention(P, "", x, q, heads, m)


def make_module(name, P, dtype, device="cuda"):
    from egnn_pytorch_b200 import GlobalLinearAttention
    c = CASES[name]
    mod = GlobalLinearAttention(dim=c["dim"], heads=c["heads"], dim_head=c["dh"]).to(dtype)
    mod.load_state_dict({k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in P.items()}, strict=True)
    return mod.to(device).eval()


def rel_err(got, want):
    return util.max_err(got, want) / max(1.0, float(np.abs(want).max()))


def check(got, want, dtype, what):
    """fp64: util.TOL; fp32: max |error| / max(1, max |reference|) <= TOL_F32, on both outputs."""
    for g, w, out in zip(got, want, ("x_out", "queries_out")):
        if dtype == F64:
            util.assert_close(g, w, **util.TOL[F64], what=f"{what}: {out}")
        else:
            assert g.shape == w.shape and rel_err(g, w) <= TOL_F32, (what, out, g.shape, w.shape, rel_err(g, w))


def max_logits(P, x, q, m, heads):
    """Largest unmasked attention logit of attn1 and of attn2 (fp64)."""
    ln = lambda v, k: O.layer_norm(v, P[k + ".weight"], P[k + ".bias"])
    xn, qn = ln(x, "norm_seq"), ln(q, "norm_queries")

    def logits(pre, a, ctx):
        qq, kv = O.linear(a, P[pre + ".to_q.weight"]), O.linear(ctx, P[pre + ".to_kv.weight"])
        inner = qq.shape[-1]
        dh = inner // heads
        s = lambda t_: t_.reshape(t_.shape[0], t_.shape[1], heads, dh).transpose(0, 2, 1, 3)
        return np.einsum("bhid,bhjd->bhij", s(qq), s(kv[..., :inner])) * dh ** -0.5

    d1 = logits("attn1", qn, xn)
    if m is not None:
        d1 = np.where(m.astype(bool)[:, None, None, :], d1, -np.inf)
    induced = O.attention(P, "attn1.", qn, xn, heads, m)
    return float(d1.max()), float(logits("attn2", xn, induced).max())


# ------------------------------------------------------------------ the table reaches every boundary (no GPU)


@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32", "fp64"])
def test_table_covers_every_boundary(dtype):
    geo = {n: geometry(c, dtype) for n, c in CASES.items()}
    dev = {n: g for n, g in geo.items() if not g["fallback"]}
    kinds = {(k, v) for g in dev.values() for k, v in g["gemm"].items()}
    assert {v for _, v in kinds} == {"skinny1", "skinny2", "skinny4", "tiled"}, kinds
    assert ("ff1", "tiled") in kinds and any(("ff1", f"skinny{c}") in kinds for c in (1, 2, 4)), "GELU on both kernels"
    assert ("ff1", "skinny4") in kinds
    assert any(g["k_fallback"] for g in dev.values()), "Mr <= 16 with K beyond the skinny kernel's staging"
    ns = {CASES[n]["N"] for n in dev}
    assert {1, 256, 257} <= ns and max(ns) > 512
    assert {g["softmax"]["n_passes"] for g in dev.values()} >= {1, 2, 3}
    dhs = {CASES[n]["dh"] for n in dev}
    assert any(256 % d == 0 and d < 256 for d in dhs) and any(256 % d and d < 256 for d in dhs)
    assert 256 in dhs and any(d > 256 and d % 256 for d in dhs)
    assert any(g["softmax"]["idle"] > 0 for g in dev.values())
    assert any(g["softmax"]["d0_passes"] == 2 for g in dev.values())
    assert {1, T_MAX} <= {g["attn2"]["T"] for g in dev.values()}
    assert any(g["attn2"]["lane_passes"] > 1 for g in dev.values())
    assert any(g["fallback"] and g["T"] == T_MAX + 1 for g in geo.values())
    heads = {CASES[n]["heads"] for n in dev}
    assert 1 in heads and max(heads) >= 16
    dims = {CASES[n]["dim"] for n in dev}
    assert min(dims) < 32 and any(d % 32 for d in dims) and max(dims) > 512
    masks = {(c["mask"], c["mask_dtype"]) for c in CASES.values()}
    assert {None, "padded", "random", "one", "empty"} <= {m for m, _ in masks}
    assert {"bool", "uint8", "float"} <= {t for m, t in masks if m is not None}


def test_big_logits_overflow_exp_without_the_max():
    """exp overflows fp32 above 88.7: both softmaxes of `big_logits` need their maximum subtracted."""
    P, x, q, m = make_case("big_logits")
    l1, l2 = max_logits(P, x, q, m, CASES["big_logits"]["heads"])
    assert l1 > 89 and l2 > 89, (l1, l2)


def test_fully_masked_and_one_valid_masks_are_what_they_say():
    _, _, _, m = make_case("dh320")
    assert not m[-1].any() and m[0].any()
    _, _, _, m = make_case("dh256")
    assert (m.sum(1) == 1).all() and len({int(np.argmax(r)) for r in m}) == len(m)


# ------------------------------------------------------------------ shapes and the C ABI (no GPU, no launch)


@pytest.mark.parametrize("x_shape, q_shape, m_shape, match", [
    ((3, 10, 12), (3, 4, 16), (3, 10), "x must"),          # x's last axis is not dim
    ((3, 10, 16), (3, 4, 12), (3, 10), "queries must"),    # queries' last axis is not dim
    ((10, 16), (3, 4, 16), (3, 10), "x must"),             # no batch axis
    ((3, 10, 16), (2, 4, 16), (3, 10), "batch"),           # batches 3 and 2
    ((3, 10, 16), (3, 4, 16), (2, 10), "batch"),           # mask batch 2
    ((1, 10, 16), (2, 4, 16), (3, 10), "batch"),           # 2 and 3 besides 1
    ((3, 10, 16), (3, 4, 16), (10,), "mask must"),         # 1-D mask
    ((3, 10, 16), (3, 4, 16), (3, 9), "mask must"),        # wrong mask length
], ids=["x_dim", "q_dim", "x_2d", "batch_q", "batch_mask", "batch_three", "mask_1d", "mask_len"])
def test_shape_errors_raise_value_error_before_any_launch(x_shape, q_shape, m_shape, match):
    from egnn_pytorch_b200 import GlobalLinearAttention
    mod = GlobalLinearAttention(dim=16, heads=2, dim_head=8)
    with pytest.raises(ValueError, match=match):
        mod(torch.randn(x_shape), torch.randn(q_shape), torch.ones(m_shape, dtype=torch.bool))


def test_c_abi_return_codes_without_a_launch(nat):
    """Every call below returns before anything is enqueued: the pointers are placeholders."""
    lib = nat.load()
    good = dict(abi_version=nat.ABI_VERSION, dtype=nat.DTYPE_F32, B=2, N=50, T=4, dim=32, heads=2, dim_head=16)
    fake = 0x10000
    w = nat.GlobalAttnWeights(**{f: fake for f in nat.GA_WEIGHT_FIELDS})
    io = nat.GlobalAttnIO(x=fake, queries=fake, mask=None, x_out=fake, queries_out=fake)
    nb = C.c_size_t()

    def forward(desc, weights, nbytes):
        return lib.egnn_global_attn_forward(C.byref(desc), C.byref(weights), C.byref(io), C.c_void_p(fake), nbytes, None)

    t33 = nat.GlobalAttnDesc(**dict(good, T=T_MAX + 1))
    assert lib.egnn_global_attn_workspace_bytes(C.byref(t33), C.byref(nb)) == -3          # EGNN_ERR_UNSUPPORTED
    assert forward(t33, w, 1 << 30) == -3
    desc = nat.GlobalAttnDesc(**good)
    assert lib.egnn_global_attn_workspace_bytes(C.byref(desc), C.byref(nb)) == 0
    # the reported size carries 256 bytes of slack, like every workspace query of the library: one byte short of what
    # the forward needs is the report - 257
    need = nb.value - 256
    for i in range(len(nat.GA_WEIGHT_FIELDS)):
        w_null = nat.GlobalAttnWeights(**{f: (None if j == i else fake) for j, f in enumerate(nat.GA_WEIGHT_FIELDS)})
        assert forward(desc, w_null, nb.value) == -1, nat.GA_WEIGHT_FIELDS[i]             # EGNN_ERR_NULL
    assert forward(desc, w, need - 1) == -5                                                # EGNN_ERR_WORKSPACE
    assert forward(nat.GlobalAttnDesc(**dict(good, abi_version=nat.ABI_VERSION + 1)), w, nb.value) == -6   # EGNN_ERR_ABI
    assert lib.egnn_global_attn_workspace_bytes(C.byref(nat.GlobalAttnDesc(**dict(good, abi_version=3))), C.byref(nb)) == -6


# ------------------------------------------------------------------ on the device


def _sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _run(name, dtype, P=None, x=None, q=None, m=None):
    c = CASES[name]
    if P is None:
        P, x, q, m = make_case(name)
    mod = make_module(name, P, dtype)
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64)).to(device="cuda", dtype=dtype)
    xo, qo = mod(t(x), t(q), mask_tensor(m, c["mask_dtype"], "cuda"))
    torch.cuda.synchronize()
    return mod, (xo, qo)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("name", list(CASES))
def test_matches_oracle(name, dtype):
    sms = _sm_count()
    if geometry(CASES[name], dtype, sms) != geometry(CASES[name], dtype):
        print(f"{name}: at {sms} SMs the launch differs from the 132-SM mirror: {geometry(CASES[name], dtype, sms)}")
    P, x, q, m = make_case(name)
    mod, got = _run(name, dtype, P, x, q, m)
    want = oracle(P, x, q, m, CASES[name]["heads"])
    assert got[0].shape == want[0].shape and got[1].shape == want[1].shape
    errs = [rel_err(g, w) for g, w in zip(got, want)]
    print(f"{name} [{dtype}]: x_out rel err {errs[0]:.3e}, queries_out rel err {errs[1]:.3e}")
    for g, w, what in zip(got, want, ("x_out", "queries_out")):
        assert torch.isfinite(g).all(), f"{name} {what}: non-finite output"
        if dtype == F64:
            util.assert_close(g, w, **util.TOL[F64], what=f"{name} {what}")
    if dtype == F32:
        assert max(errs) <= (TOL_F32_BIG_LOGITS if CASES[name]["q_scale"] > 1 else TOL_F32), (name, errs)
    else:
        # the inference kernels and the module's own PyTorch arithmetic (the training path) agree
        c = CASES[name]
        t = lambda a: torch.from_numpy(np.asarray(a, np.float64)).cuda()
        ref = mod._forward_autograd(t(x), t(q), mask_tensor(m, c["mask_dtype"], "cuda"))
        for g, r, what in zip(got, ref, ("x_out", "queries_out")):
            assert util.max_err(g, r) <= 1e-10 * max(1.0, float(r.abs().max())), (name, what, util.max_err(g, r))


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in CASES if CASES[n]["T"] <= T_MAX])
def test_bf16_module_matches_oracle(name):
    """A bf16 module runs the block on fp32 copies of its parameters and rounds the outputs to bf16."""
    rnd = lambda a: torch.from_numpy(np.asarray(a, np.float64)).bfloat16().double().numpy()
    P, x, q, m = make_case(name)
    P = {k: rnd(v) for k, v in P.items()}
    x, q = rnd(x), rnd(q)
    mod, got = _run(name, torch.bfloat16, P, x, q, m)
    assert got[0].dtype == torch.bfloat16 and got[1].dtype == torch.bfloat16
    want = oracle(P, x, q, m, CASES[name]["heads"])
    errs = [rel_err(g, w) for g, w in zip(got, want)]
    print(f"{name} [bf16]: x_out rel err {errs[0]:.3e}, queries_out rel err {errs[1]:.3e}")
    assert max(errs) <= TOL_BF16, (name, errs)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
def test_size_one_batches_broadcast(dtype):
    """queries [1, T, dim] and mask [1, N] give the bits of the expanded tensors; x [1, N, dim] with queries [B, T, dim]
    is the reference run on the broadcast inputs, with batch B out."""
    name = "default"
    P, x, q, m = make_case(name)
    B = x.shape[0]
    mod = make_module(name, P, dtype)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(device="cuda", dtype=dtype)
    xs, q1, m1 = t(x), t(q[:1]), torch.from_numpy(m[:1].copy()).cuda()
    got = mod(xs, q1, m1)
    ref = mod(xs, q1.expand(B, -1, -1).contiguous(), m1.expand(B, -1).contiguous())
    assert got[0].shape == x.shape and got[1].shape == (B,) + q.shape[1:]
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    want = oracle(P, x, np.broadcast_to(q[:1], q.shape), np.broadcast_to(m[:1], m.shape), CASES[name]["heads"])
    check(got, want, dtype, "queries and mask of batch 1")
    # one graph's nodes against B sets of tokens
    got = mod(t(x[:1]), t(q), torch.from_numpy(m).cuda())
    assert got[0].shape == x.shape and got[1].shape == q.shape
    want = oracle(P, np.broadcast_to(x[:1], x.shape), q, m, CASES[name]["heads"])
    check(got, want, dtype, "x of batch 1")


NET_SPEC = dict(kind="network", cfg=dict(depth=2, dim=64, global_linear_attn_every=1), B=2, N=300, seed=67, mask="padded")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
def test_network_at_the_default_attention_shape(dtype):
    """EGNN_Network with a global attention block before each layer at heads 8, dim_head 64."""
    case = cases.build_case(NET_SPEC)
    mod = util.make_module(case, dtype)
    assert mod.layers[0][0].heads == 8 and mod.layers[0][0].dim_head == 64
    out = util.run_module(mod, case, dtype)
    want = cases.run_oracle(case)
    util.assert_close(out[0], want[0], **util.TOL[dtype], what="feats")
    util.assert_close(out[1], want[1], **util.TOL[dtype], what="coors")


@pytest.mark.gpu
def test_network_with_attention_replays_under_graph_capture():
    from egnn_pytorch_b200 import GraphedForward
    case = cases.build_case(NET_SPEC)
    mod = util.make_module(case, F32)
    ins = {k: util.to_torch(v, F32, "cuda") for k, v in case["inputs"].items()}
    args = (ins["feats"], ins["coors"])
    eager = mod(*args, mask=ins["mask"])
    fast = GraphedForward(mod, *args, mask=ins["mask"])
    out = fast(*args)
    assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])
    args2 = (args[0], args[1] * 1.25 + 0.5)
    out2 = [o.clone() for o in fast(*args2)]
    eager2 = mod(*args2, mask=ins["mask"])
    assert torch.equal(out2[0], eager2[0]) and torch.equal(out2[1], eager2[1])
