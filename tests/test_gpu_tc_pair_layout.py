"""The warpgroup layouts of the dense bf16 edge kernel (tc_pair.cuh), against the rounding-matched reference.

The kernel runs either 2 compute warpgroups of 32 pairs per warp (the default) or, for the lean instantiation with
EGNN_B200_TC_PAIR_WG=4 and where its shared memory fits, 4 warpgroups of 16 pairs per warp.  A warpgroup's j-tile is
128 pairs in the first layout and 64 in the second, so the cases here cross the 64-pair boundaries the second one adds:
N = 63 .. 257, one active warpgroup at N <= 64.  Every case is run in both layouts -- which one ran is read from the
library's launch counters -- and checked against tests/tc_reference.py with the gates of test_gpu_tc_boundaries.py
(`TOL`), and the two layouts against each other with the same gates."""
import functools
import os

import numpy as np
import pytest
import torch

import ctypes as C

import cases
import tc_reference as T
import util
from egnn_pytorch_b200 import _native as nat
from test_gpu_tc_boundaries import TOL, geometry

L = "layer"
CASES = {
    # one active warpgroup (N <= 64), then 2, 3 and 4 of them, each partial / exactly full / one pair into the next
    "w_n63_clamp":  dict(kind=L, cfg=dict(dim=32, coor_weights_clamp_value=0.5), B=2, N=63, seed=501, mask="random"),
    "w_n64_mean":   dict(kind=L, cfg=dict(dim=32, m_pool_method="mean"), B=2, N=64, seed=502, mask="padded"),
    "w_n65_soft":   dict(kind=L, cfg=dict(dim=24, soft_edges=True), B=2, N=65, seed=503),
    "w_n127_mean":  dict(kind=L, cfg=dict(dim=16, m_pool_method="mean", soft_edges=True), B=2, N=127, seed=504,
                         mask="random"),
    "w_n128":       dict(kind=L, cfg=dict(dim=32), B=2, N=128, seed=505, mask="padded"),
    "w_n129_clamp": dict(kind=L, cfg=dict(dim=24, coor_weights_clamp_value=1.0), B=2, N=129, seed=506),
    "w_n191_soft":  dict(kind=L, cfg=dict(dim=16, soft_edges=True), B=2, N=191, seed=507, mask="padded"),
    "w_n192_mean":  dict(kind=L, cfg=dict(dim=32, m_pool_method="mean"), B=2, N=192, seed=508),
    "w_n193":       dict(kind=L, cfg=dict(dim=16), B=2, N=193, seed=509, mask="random"),
    "w_n255_clamp": dict(kind=L, cfg=dict(dim=16, coor_weights_clamp_value=2.0, soft_edges=True), B=2, N=255, seed=510),
    "w_n256_mean":  dict(kind=L, cfg=dict(dim=24, m_pool_method="mean"), B=2, N=256, seed=511, mask="padded"),
    "w_n257":       dict(kind=L, cfg=dict(dim=16), B=2, N=257, seed=512, mask="random"),
    # the generic instantiation, which stays on 2 warpgroups when 4 are asked for (fourier features + edges)
    "w_gen_n60":    dict(kind=L, cfg=dict(dim=16, fourier_features=1, edge_dim=2, soft_edges=True), B=2, N=60,
                         seed=513, mask="padded"),
    "w_gen_n150":   dict(kind=L, cfg=dict(dim=16, edge_dim=3, m_pool_method="mean", coor_weights_clamp_value=1.0),
                         B=2, N=150, seed=514, mask="random"),
}
SMEM_MAX = 227 * 1024


def pair_smem(Hp, Q, Qf, gen, wg):
    """tc_pair_smem_bytes<GEN, WG> (tc_pair.cuh)."""
    cw, PW, XC = 4 * wg, (28 if gen else 20), (8 if gen else 4)
    n = Hp * 32 + Q * Hp * 4 + 2 * 4 * Hp * 4 + (64 * 16 + 64 + 64 + 16 + 16 + 4) * 4
    n += 2 * cw * 4 * PW * 8 + cw * (256 // cw) * 18 * 4
    n += 2 * 4 * XC * 4 + 2 * 4 * 4 + 64 + (0 if gen else 4 * 256 * 4)
    n += 4 * 256 * (Qf * 4 + (Q - Qf) * 2) if gen else 0
    return n + 64 + 256


def _bf16(a):
    return torch.from_numpy(np.asarray(a, np.float64)).float().bfloat16().double().numpy()


def make_case(spec):
    """bf16 parameters / features / edges and fp32 coordinates (as in test_gpu_tc_boundaries.build)."""
    case = cases.build_case(dict({k: v for k, v in spec.items() if k != "rows"}, init="xavier"))
    ins = case["inputs"]
    case["params"] = {k: _bf16(v) for k, v in case["params"].items()}
    ins["feats"] = _bf16(ins["feats"])
    ins["coors"] = np.asarray(ins["coors"], np.float32).astype(np.float64)
    if ins.get("edges") is not None:
        ins["edges"] = _bf16(ins["edges"])
    return case


@functools.lru_cache(maxsize=None)
def case_of(name):
    return make_case(CASES[name])


@functools.lru_cache(maxsize=None)
def reference(name):
    case = case_of(name)
    ins = case["inputs"]
    return T.tc_layer_forward(case["params"], case["cfg"], ins["feats"], ins["coors"], edges=ins.get("edges"),
                              mask=ins.get("mask"))


def run_gpu(case, wg=None, rows=None):
    """Forward on the bf16 path with EGNN_B200_TC_PAIR_WG set to `wg` for the call -> (feats, coors, warpgroups of the
    dense edge kernel's launch, from the library's launch counters)."""
    ins = case["inputs"]
    mod = util.make_module(case, torch.bfloat16)
    lib = nat.load()
    tb = lambda a: None if a is None else torch.from_numpy(np.asarray(a, np.float64)).to("cuda", torch.bfloat16)
    mask = None if ins.get("mask") is None else torch.from_numpy(ins["mask"]).to("cuda")
    old = os.environ.pop("EGNN_B200_TC_PAIR_WG", None)
    n2, n4 = C.c_int64(), C.c_int64()
    try:
        if wg is not None:
            os.environ["EGNN_B200_TC_PAIR_WG"] = str(wg)
        lib.egnn_profile_read(None, None, None, 1)
        lib.egnn_profile_enable(1)
        with torch.no_grad():
            f, x = mod(tb(ins["feats"]), torch.from_numpy(ins["coors"]).float().cuda(), tb(ins.get("edges")),
                       mask=mask, _rows=rows)
        torch.cuda.synchronize()
        assert lib.egnn_profile_pair_layouts(C.byref(n2), C.byref(n4)) == 0
    finally:
        lib.egnn_profile_enable(0)
        lib.egnn_profile_read(None, None, None, 1)
        os.environ.pop("EGNN_B200_TC_PAIR_WG", None)
        if old is not None:
            os.environ["EGNN_B200_TC_PAIR_WG"] = old
    assert mod.last_path == "bf16-tc"
    assert (n2.value, n4.value) in ((1, 0), (0, 1)), (n2.value, n4.value)
    return f, x, 4 if n4.value else 2


def metrics(x_in, rf, rx, f, x):
    """The four gates of test_gpu_tc_boundaries.metrics for one output (f, x) against (rf, rx)."""
    gf, gx = f.double().cpu().numpy(), x.double().cpu().numpy()
    rf, rx = np.asarray(rf, np.float64), np.asarray(rx, np.float64)
    floor = 1e-2 * np.abs(rf).max()
    ulp = 2.0 ** (np.floor(np.log2(np.maximum(np.abs(rf), floor))) - 7)
    fu = np.abs(gf - rf) / ulp
    upd = rx - x_in
    err = np.abs(gx - rx).max(-1)
    cr = err / np.maximum(np.abs(upd).max(-1), 1e-3 * np.abs(upd).max() + 1e-30)
    ce = (gx - rx).ravel()
    return dict(f_ulp_max=float(fu.max()), f_ulp_mean=float(fu.mean()), c_row=float(cr.max()),
                c_rms=float(np.sqrt((ce ** 2).mean() / max((upd ** 2).mean(), 1e-300))))


def test_cases_cross_the_warpgroup_tile_boundaries():
    geo = {n: geometry(s) for n, s in CASES.items()}
    assert all(g["supported"] and g["k"] == 0 for g in geo.values())
    assert {g["N"] for g in geo.values()} >= {63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257}
    active = {min(4, -(-g["N"] // 64)) for g in geo.values()}
    assert active == {1, 2, 3, 4}
    assert {g["kernel"] for g in geo.values()} == {"tc_pair<lean>", "tc_pair<generic>"}
    for n, g in geo.items():
        if g["kernel"] == "tc_pair<lean>":
            assert pair_smem(g["Hp"], 1, 1, False, 4) <= SMEM_MAX, n


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_both_layouts_match_the_reference_and_each_other(name):
    """The lean cases run 4 warpgroups when asked for, the generic ones always 2; the default is 2."""
    case = case_of(name)
    x_in = case["inputs"]["coors"]
    rf, rx = reference(name)
    lean = geometry(CASES[name])["kernel"] == "tc_pair<lean>"
    f4, x4, l4 = run_gpu(case, wg=4)
    f2, x2, l2 = run_gpu(case, wg=2)
    f0, x0, l0 = run_gpu(case)
    assert (l4, l2, l0) == ((4 if lean else 2), 2, 2)
    assert torch.equal(f0, f2) and torch.equal(x0, x2)
    if not lean:
        assert torch.equal(f4, f2) and torch.equal(x4, x2)
    for tag, (f, x) in (("wg4", (f4, x4)), ("wg2", (f2, x2))):
        assert torch.isfinite(f.float()).all() and torch.isfinite(x).all(), (name, tag)
        m = metrics(x_in, rf, rx, f, x)
        print(f"TPL {name} {tag} " + " ".join(f"{k}={v:.3e}" for k, v in m.items()))
        bad = {k: v for k, v in m.items() if not v <= TOL[k]}
        assert not bad, (name, tag, bad)
    m = metrics(x_in, f2.double().cpu().numpy(), x2.double().cpu().numpy(), f4, x4)
    bad = {k: v for k, v in m.items() if not v <= TOL[k]}
    assert not bad, (name, "wg4 vs wg2", bad)


@pytest.mark.gpu
def test_jsplit_row_ranges_are_bit_identical_to_the_full_forward():
    """4-warpgroup layout: row ranges dealt at j-split 2 and 4 equal the full forward (j-split 2) bit for bit."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    spec = dict(kind=L, cfg=dict(dim=16, soft_edges=True, coor_weights_clamp_value=1.5), B=2, N=1024, seed=520,
                mask="padded")
    ranges = [(100, 1000), (3, 62)]
    js = [geometry(dict(spec, rows=r), sms)["jsplit"] for r in ranges]
    assert geometry(spec, sms)["jsplit"] == 2 and js == [2, 4], js
    case = make_case(spec)
    f_full, x_full, wg = run_gpu(case, wg=4)
    assert wg == 4
    for r0, r1 in ranges:
        f, x, wg = run_gpu(case, wg=4, rows=(r0, r1))
        assert wg == 4
        assert torch.equal(f[:, r0:r1], f_full[:, r0:r1]) and torch.equal(x[:, r0:r1], x_full[:, r0:r1]), (r0, r1)


@pytest.mark.gpu
def test_lean_config_without_room_for_four_warpgroups_runs_two():
    """dim=680 (Hp = 2736): the 4-warpgroup layout needs more than 227 KB of shared memory (the fp64 partial sums per
    warp double), so a launch that asks for it takes the 2-warpgroup layout, still on the tensor cores."""
    spec = dict(kind=L, cfg=dict(dim=680), B=1, N=70, seed=521, mask="padded")
    g = geometry(spec)
    assert g["kernel"] == "tc_pair<lean>"
    assert pair_smem(g["Hp"], 1, 1, False, 4) > SMEM_MAX >= pair_smem(g["Hp"], 1, 1, False, 2)
    case = make_case(spec)
    ins = case["inputs"]
    rf, rx = T.tc_layer_forward(case["params"], case["cfg"], ins["feats"], ins["coors"], mask=ins["mask"])
    f, x, wg = run_gpu(case, wg=4)
    assert wg == 2
    m = metrics(ins["coors"], rf, rx, f, x)
    print("TPL lean_fallback " + " ".join(f"{k}={v:.3e}" for k, v in m.items()))
    bad = {k: v for k, v in m.items() if not v <= TOL[k]}
    assert not bad, bad
