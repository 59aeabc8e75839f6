"""Cost of triclinic cells (EGNN.forward(..., cell=)): the same layer call with no box, with `box=`, with a diagonal
`cell=` and with a tilted `cell=`, the four arms alternated over several rounds after a warm-up, timed with CUDA events.

Workloads:
  c2       : EGNN(dim=512) dense, bf16, B=4, N=1024 (bench.py's flagship layer)                    (forward)
  c4       : EGNN(dim=256, edge_dim=4, num_nearest_neighbors=32), bf16, B=8, N=4096                 (forward)
  c4_train : the c4 layer in fp32, forward + backward
  radius   : EGNN(dim=64, num_nearest_neighbors=32, valid_radius=r^2) with a mask, bf16, B=1, N=65,536 on the cell grid
             (about 24 neighbours in radius per node)                                              (forward)
The box / cell diagonal is 2.5x the coordinate spread (radius: the cloud fills the cell), so most pairs are not
wrapped but every pair runs the wrap; the tilted cell leans every lattice vector by up to 0.5 of the diagonal.  Prints
one JSON line per workload: per-arm median and spread (min, max) of the rounds' milliseconds, the overhead of each
arm's median over no box, and the GPU name and power limit.

    python tools/triclinic_bench.py [--reps 10] [--warmup 3] [--rounds 7] [--only c2]
"""
import argparse
import copy
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
    mask = None
    if name == "c2":
        mod, B, N, e, dt, train = EGNN(dim=512), 4, 1024, 0, torch.bfloat16, False
    elif name == "radius":
        mod, B, N, e, dt, train = EGNN(dim=64, num_nearest_neighbors=32, valid_radius=1.0), 1, 65536, 0, torch.bfloat16, False
    else:
        mod, B, N, e = EGNN(dim=256, edge_dim=4, num_nearest_neighbors=32), 8, 4096, 4
        dt, train = (torch.float32, True) if name == "c4_train" else (torch.bfloat16, False)
    mod = mod.to(dt).cuda()
    feats = torch.randn(B, N, mod.dim, device="cuda", dtype=dt)
    if name == "radius":
        side = (N * 4.18879 / 24) ** (1 / 3)                       # density: ~24 nodes per unit ball
        coors = torch.rand(B, N, 3, device="cuda") * side
        L = side
        mask = torch.ones(B, N, dtype=torch.bool, device="cuda")
    else:
        coors = torch.randn(B, N, 3, device="cuda")
        L = 2.5 * float(coors.max() - coors.min())
    edges = torch.randn(B, N, N, e, device="cuda", dtype=dt) if e else None
    box = torch.full((3,), L, device="cuda")
    diag = torch.diag(box)
    tilt = torch.tensor([[1.0, 0, 0], [0.4, 1.0, 0], [-0.5, 0.3, 1.0]], device="cuda") * L
    arms = {"none": {}, "box": dict(box=box), "cell_diag": dict(cell=diag), "cell_tilt": dict(cell=tilt)}
    # one module per arm: a module re-reads a cell it did not check last, so two cells alternating on one module would
    # time that host check too
    mods = {arm: copy.deepcopy(mod) for arm in arms}
    if train:
        feats.requires_grad_(True)
        coors.requires_grad_(True)

        def run(arm):
            fo, xo = mods[arm].train()(feats, coors, edges, mask=mask, **arms[arm])
            (fo.float().sum() + xo.sum()).backward()
    else:
        def run(arm):
            with torch.no_grad():
                mods[arm].eval()(feats, coors, edges, mask=mask, **arms[arm])
    return run, arms, mods


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--only", default=None, help="one workload: c2 | c4 | c4_train | radius")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "triclinic_bench needs a GPU"
    gpu, pl = torch.cuda.get_device_name(), power_limit_w()
    for name in [args.only] if args.only else ["c2", "c4", "c4_train", "radius"]:
        run, arms, mods = workload(name)
        for _ in range(args.warmup):
            for arm in arms:
                run(arm)
        paths = {}
        t = {k: [] for k in arms}
        for _ in range(args.rounds):
            for arm in arms:
                t[arm].append(timed(lambda: run(arm), args.reps))
                paths[arm] = mods[arm].last_path
        med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
        print(json.dumps(dict(workload=name, gpu=gpu, power_limit_w=pl, paths=paths, median_ms=med,
                              min_ms={k: min(v) for k, v in t.items()}, max_ms={k: max(v) for k, v in t.items()},
                              overhead={k: med[k] / med["none"] - 1.0 for k in arms if k != "none"},
                              rounds=args.rounds, reps=args.reps)), flush=True)
        del run, arms, mods
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
