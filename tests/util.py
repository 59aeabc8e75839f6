"""Helpers shared by the GPU parity tests, smoke() and bench.py: build the product modules from
a tests/cases.py case, move numpy inputs to torch, and run / compare forward and backward; plus the small helpers the
test files share (rounding, the native-library fixture, TF32 off)."""
from __future__ import annotations

import contextlib

import numpy as np
import pytest
import torch

import cases

# Forward tolerances against the fp64 oracle (stated per SURVEY.md section 8(c)):
#   fp64 kernels : atol 1e-9,  rtol 1e-9   (same algebra, different summation order)
#   fp32 kernels : atol 2e-5,  rtol 1e-4   (the reference's own fp32-vs-fp64 deviation is <= 5e-6 at these sizes,
#                  BASELINE.md section 2)
TOL = {torch.float64: dict(atol=1e-9, rtol=1e-9), torch.float32: dict(atol=2e-5, rtol=1e-4)}


def to_torch(x, dtype, device):
    if x is None:
        return None
    x = np.asarray(x)
    if x.dtype == bool:
        return torch.from_numpy(x.copy()).to(device)
    if np.issubdtype(x.dtype, np.integer):
        return torch.from_numpy(x.astype(np.int64)).to(device)
    return torch.from_numpy(x.astype(np.float64)).to(device=device, dtype=dtype)


def make_module(case, dtype, device="cuda", **extra):
    from egnn_pytorch_b200 import EGNN, EGNN_Network
    spec = case["spec"]
    mod = EGNN_Network(**spec["cfg"], **extra) if case["kind"] == "network" else EGNN(**spec["cfg"], **extra)
    mod = mod.to(dtype)                            # before loading: load_state_dict casts to the parameter dtype
    sd = {k: torch.from_numpy(np.asarray(v, dtype=np.float64)) for k, v in case["params"].items()}
    mod.load_state_dict(sd, strict=True)          # reference state-dict keys must load unchanged
    return mod.to(device).eval()


def run_module(mod, case, dtype, device="cuda", **kw):
    ins = case["inputs"]
    t = lambda name: to_torch(ins.get(name), dtype, device)
    if case["kind"] == "network":
        return mod(t("feats"), t("coors"), adj_mat=t("adj_mat"), edges=t("edges"), mask=t("mask"), **kw)
    return mod(t("feats"), t("coors"), t("edges"), mask=t("mask"), adj_mat=t("adj_mat"), **kw)


def module_grads(case, dtype, device="cuda", neighbors=None):
    """Run forward + backward of the product module; -> flat {name: float64 numpy gradient}.  `neighbors` (numpy
    [B,N,k], -1 = empty slot) runs a layer in edge-list mode."""
    mod = make_module(case, dtype, device=device)
    mod.requires_grad_(True)
    ins = case["inputs"]
    t = lambda name: to_torch(ins.get(name), dtype, device)
    feats, coors, edges = t("feats"), t("coors"), t("edges")
    leaves = {"coors": coors.requires_grad_(True)}
    if feats.is_floating_point():
        leaves["feats"] = feats.requires_grad_(True)
    if edges is not None and edges.is_floating_point():
        leaves["edges"] = edges.requires_grad_(True)
    gf, gx = (torch.from_numpy(g).to(device=device, dtype=dtype) for g in cases.upstream_grads(case))
    with torch.enable_grad():
        if case["kind"] == "network":
            fo, xo = mod(feats, coors, adj_mat=t("adj_mat"), edges=edges, mask=t("mask"))
        elif neighbors is not None:
            fo, xo = mod(feats, coors, edges, mask=t("mask"), neighbors=torch.from_numpy(neighbors).to(device))
        else:
            fo, xo = mod(feats, coors, edges, mask=t("mask"), adj_mat=t("adj_mat"))
        assert fo.requires_grad and xo.requires_grad
        ((fo * gf).sum() + (xo * gx).sum()).backward()
    out = {f"in.{k}": v.grad.double().cpu().numpy() for k, v in leaves.items()}
    for k, p in mod.named_parameters():
        out[f"p.{k}"] = (torch.zeros_like(p) if p.grad is None else p.grad).double().cpu().numpy()
    return out


def compare(got, want, tol, what):
    """Every gradient within `tol` of the reference, relative to max(1, its largest magnitude)."""
    assert set(got) == set(want), (what, sorted(set(got) ^ set(want)))
    bad = []
    for k in sorted(want):
        scale = max(1.0, float(np.abs(want[k]).max()))
        err = float(np.abs(got[k] - want[k]).max()) / scale
        if not np.isfinite(got[k]).all() or err > tol:
            bad.append(f"{k}: rel err {err:.3e}")
    assert not bad, f"{what}: " + "; ".join(bad)


def grad_tol(case, dtype):
    """Gradient tolerance of `compare` against the fp64 backward oracle."""
    if dtype == torch.float64:
        # CoorsNorm: the oracle (like the reference) carries ~1e-9 of cancellation noise from the 1/eps self pair
        return 1e-7 if "norm_coors" in str(case["spec"]["cfg"]) else 1e-9
    return 5e-4


def max_err(a, b):
    a = a.detach().double().cpu().numpy() if torch.is_tensor(a) else np.asarray(a, np.float64)
    b = b.detach().double().cpu().numpy() if torch.is_tensor(b) else np.asarray(b, np.float64)
    return float(np.abs(a - b).max())


def assert_close(got, want, atol, rtol, what=""):
    got = got.detach().double().cpu().numpy() if torch.is_tensor(got) else np.asarray(got, np.float64)
    want = np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    err = np.abs(got - want)
    tol = atol + rtol * np.abs(want)
    worst = float((err - tol).max())
    assert worst <= 0, f"{what}: max|err|={err.max():.3e} exceeds atol={atol} rtol={rtol} (|want|max={np.abs(want).max():.3e})"


def rounded(x, dtype):
    """`x` rounded to the torch float type `dtype` (a bfloat16 through float32, as torch converts) and returned as
    float64 numpy: the values a kernel of that type sees.  None and arrays that are not floating point are returned
    as they are (masks, token ids, adjacency)."""
    if x is None or not np.issubdtype(np.asarray(x).dtype, np.floating):
        return x
    return torch.as_tensor(np.asarray(x, np.float64)).to(dtype).double().numpy()


@pytest.fixture(scope="module")
def nat():
    """egnn_pytorch_b200._native with the library built for sm_90a (nvcc cross-compiles without a GPU) and loaded."""
    from egnn_pytorch_b200 import build, _native
    build.build()
    _native.load()
    return _native


@contextlib.contextmanager
def no_tf32():
    """fp32 matmuls in full fp32 (no TF32), so that an fp32 restatement measures fp32 arithmetic."""
    prev = torch.backends.cuda.matmul.allow_tf32, torch.get_float32_matmul_precision()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev[0]
        torch.set_float32_matmul_precision(prev[1])
