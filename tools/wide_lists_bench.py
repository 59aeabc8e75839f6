"""bf16 tensor cores vs fp32 SIMT on neighbour lists of 32 to 128 slots, and k = 32 against another build.

The c4 layer (EGNN(dim=256, edge_dim=4)) at B=8, N=4096 with per-slot edges, on lists from egnn_knn_select computed
once per k outside the timed window.  For k in {32, 64, 96, 128} the bf16 forward (tc_knn_kernel, slot groups of 32
for k > 32) and the fp32 forward (the SIMT kernels) are timed with CUDA events after a warm-up, alternated over
`--rounds` rounds; each entry is the median over the rounds, in ms and in edges (B * N * k) per second.  With
`--other-lib PATH` the k = 32 bf16 forward also runs on that build of the library (loaded like EGNN_B200_LIB, in the
same process, alternated with this one): the time of both and the largest output difference on the same inputs.
Prints one JSON line, with the GPU name and power limit.

    python tools/wide_lists_bench.py [--reps 10] [--warmup 3] [--rounds 5] [--other-lib PATH]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from egnn_pytorch_b200 import EGNN, _native as nat  # noqa: E402

B, N, DIM, EDIM = 8, 4096, 256, 4
KS = (32, 64, 96, 128)


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:      # noqa: BLE001  (reported as unknown)
        return None


def knn_lists(coors, k):
    b, n, cd = coors.shape
    idx = torch.empty(b, n, k, dtype=torch.int32, device=coors.device)
    nat.check("egnn_knn_select", nat.load().egnn_knn_select(
        nat.DTYPE_F32, b, n, cd, k, C.c_void_p(coors.data_ptr()), None, None, 0, float("inf"), C.c_void_p(idx.data_ptr()),
        None, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return idx


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def load_lib(path):
    """The library at `path`, typed and checked by the package's loader (as EGNN_B200_LIB would select it)."""
    saved, saved_path = nat._lib, nat.LIB_PATH
    nat._lib, nat.LIB_PATH = None, path
    try:
        return nat.load()
    finally:
        nat._lib, nat.LIB_PATH = saved, saved_path


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--other-lib", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    dev = "cuda"
    torch.manual_seed(0)
    torch.set_grad_enabled(False)
    this_lib = nat.load()
    mod16 = EGNN(dim=DIM, edge_dim=EDIM).to(dev).bfloat16().eval()
    mod32 = EGNN(dim=DIM, edge_dim=EDIM).to(dev).float().eval()
    mod32.load_state_dict(mod16.state_dict())
    feats = torch.randn(B, N, DIM, device=dev)
    coors = torch.randn(B, N, 3, device=dev) * 4.0
    f16, f32 = feats.bfloat16(), feats
    runs = {}
    for k in KS:
        nbr = knn_lists(coors, k)
        e = torch.randn(B, N, k, EDIM, device=dev)
        runs[("bf16-tc", k)] = (mod16, lambda m=mod16, n=nbr, e=e.bfloat16(): m(f16, coors, neighbors=n, neighbor_edges=e))
        runs[("fp32-simt", k)] = (mod32, lambda m=mod32, n=nbr, e=e: m(f32, coors, neighbors=n, neighbor_edges=e))
    other = load_lib(args.other_lib) if args.other_lib else None
    if other is not None:
        def on(lib, fn):
            def run():
                nat._lib = lib
                try:
                    return fn()
                finally:
                    nat._lib = this_lib
            return run
        base = runs[("bf16-tc", 32)][1]
        runs[("this", 32)] = (mod16, on(this_lib, base))
        runs[("other", 32)] = (mod16, on(other, base))
    for key, (mod, fn) in runs.items():
        for _ in range(args.warmup):
            fn()
        if key[0] in ("bf16-tc", "fp32-simt"):
            assert mod.last_path == key[0], (key, mod.last_path)
    torch.cuda.synchronize()
    times = {key: [] for key in runs}
    for _ in range(args.rounds):
        for key, (_, fn) in runs.items():
            times[key].append(timed(fn, args.reps))
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "B": B, "N": N, "dim": DIM,
           "edge_dim": EDIM, "reps": args.reps, "rounds": args.rounds}
    for k in KS:
        for path in ("bf16-tc", "fp32-simt"):
            t = times[(path, k)]
            med = statistics.median(t)
            res[f"{path}_k{k}_ms"] = round(med, 4)
            res[f"{path}_k{k}_spread_ms"] = round(max(t) - min(t), 4)
            res[f"{path}_k{k}_edges_per_s"] = float(f"{B * N * k / (med * 1e-3):.4g}")
        res[f"speedup_k{k}"] = round(res[f"fp32-simt_k{k}_ms"] / res[f"bf16-tc_k{k}_ms"], 3)
        res[f"bf16-tc_k{k}_ns_per_edge"] = round(res[f"bf16-tc_k{k}_ms"] * 1e6 / (B * N * k), 4)
    if other is not None:
        for who in ("this", "other"):
            t = times[(who, 32)]
            res[f"ab_k32_{who}_ms"] = round(statistics.median(t), 4)
            res[f"ab_k32_{who}_spread_ms"] = round(max(t) - min(t), 4)
        fa, xa = runs[("this", 32)][1]()
        fb, xb = runs[("other", 32)][1]()
        res["ab_k32_max_abs_diff_feats"] = float((fa.float() - fb.float()).abs().max())
        res["ab_k32_max_abs_diff_coors"] = float((xa - xb).abs().max())
        res["ab_k32_bit_identical"] = bool(torch.equal(fa, fb) and torch.equal(xa, xb))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
