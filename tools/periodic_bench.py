"""Cost of periodic boundaries (EGNN.forward(..., box=)): the same layer call with and without a box.

Three workloads, each timed with CUDA events in both modes, the modes alternated over several rounds after a warm-up:
  c2      : EGNN(dim=512) dense, bf16, B=4, N=1024 (bench.py's flagship layer)   (forward)
  c4      : EGNN(dim=256, edge_dim=4, num_nearest_neighbors=32), bf16, B=8, N=4096   (forward)
  c4_train: the c4 layer in fp32, forward + backward
The box is 2.5x the coordinate spread on every axis, so most pairs are not wrapped but every pair runs the wrap.
Prints one JSON line per workload: per-mode median and spread (min, max) of the rounds' milliseconds, the relative
overhead of the median, and the GPU name and power limit.

    python tools/periodic_bench.py [--reps 10] [--warmup 3] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from egnn_pytorch_b200 import EGNN  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:      # noqa: BLE001  (reported as unknown)
        return None


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def workload(name):
    torch.manual_seed(0)
    if name == "c2":
        mod, B, N, e, dt, train = EGNN(dim=512), 4, 1024, 0, torch.bfloat16, False
    else:
        mod, B, N, e = EGNN(dim=256, edge_dim=4, num_nearest_neighbors=32), 8, 4096, 4
        dt, train = (torch.float32, True) if name == "c4_train" else (torch.bfloat16, False)
    mod = mod.to(dt).cuda()
    feats = torch.randn(B, N, mod.dim, device="cuda", dtype=dt)
    coors = torch.randn(B, N, 3, device="cuda")
    edges = torch.randn(B, N, N, e, device="cuda", dtype=dt) if e else None
    box = torch.full((3,), 2.5 * float(coors.max() - coors.min()), device="cuda")
    if train:
        mod.train()
        feats.requires_grad_(True)
        coors.requires_grad_(True)

        def run(bx):
            fo, xo = mod(feats, coors, edges, box=bx)
            (fo.float().sum() + xo.sum()).backward()
    else:
        mod.eval()

        def run(bx):
            with torch.no_grad():
                mod(feats, coors, edges, box=bx)
    return run, box, mod


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--only", default=None, help="one workload: c2 | c4 | c4_train")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "periodic_bench needs a GPU"
    gpu, pl = torch.cuda.get_device_name(), power_limit_w()
    for name in [args.only] if args.only else ["c2", "c4", "c4_train"]:
        run, box, mod = workload(name)
        for _ in range(args.warmup):
            run(None)
            run(box)
        paths = {}
        t = {"plain": [], "periodic": []}
        for _ in range(args.rounds):
            for mode, bx in (("plain", None), ("periodic", box)):
                t[mode].append(timed(lambda: run(bx), args.reps))
                paths[mode] = mod.last_path
        med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
        print(json.dumps(dict(workload=name, gpu=gpu, power_limit_w=pl, paths=paths,
                              median_ms=med, min_ms={k: min(v) for k, v in t.items()}, max_ms={k: max(v) for k, v in t.items()},
                              overhead=med["periodic"] / med["plain"] - 1.0, rounds=args.rounds, reps=args.reps)), flush=True)
        del run, box, mod
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
