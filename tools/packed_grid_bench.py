"""Packed batches on the cell grids against the packed all-pairs select and the unpacked per-graph calls, on one GPU.

    python tools/packed_grid_bench.py [--reps 5] [--out results.json]

Workloads: atomistic graphs at density 0.1 A^-3 with a 5 A cutoff (8k-64k nodes), a mixed batch (a few large graphs
plus ~500 QM9-sized ones), and single graphs on both sides of each threshold.  For each, k = 32 and 96, it times with
CUDA events, alternating the three paths in every repetition so that they see the same clocks:
  select   kNN mode (egnn_knn_grid_select_packed, no mask) and radius mode (egnn_radius_select_packed, a mask and
           valid_radius = 25): packed with the grids (thresholds at their defaults), packed all-pairs (thresholds
           forced above every graph), and the unpacked grid entries graph by graph
  layer    one EGNN layer (dim 64, m_dim 16, kNN, no mask): bf16 forward under no_grad and fp32 forward + backward,
           packed with and without the grids (the unpacked column is the per-graph layer calls)
The median of --reps repetitions after one warm-up.  It prints the card name and power limit first, since every time
belongs to them, then one JSON line per configuration."""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from egnn_pytorch_b200 import EGNN, knn_neighbors, radius_neighbors_wide   # noqa: E402
from egnn_pytorch_b200.egnn import _packed_select                         # noqa: E402

DEV = "cuda"
ENVS = ("EGNN_B200_KNN_GRID_MIN_N", "EGNN_B200_CELL_SELECT_MIN_N")
OFF = str(1 << 40)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def atoms(n, rs):
    side = (n / 0.1) ** (1 / 3)                    # 0.1 atoms per cubic angstrom
    return rs.uniform(0, side, (n, 3))


WORKLOADS = {
    "atomistic 8k+16k+32k+64k": [8192, 16384, 32768, 65536],
    "mixed 2x20k + 500 QM9": [20000, 20000] + [18] * 500,
    "radius threshold 4095 / 4096": [4095, 4096],
    "kNN threshold 8191 / 8192": [8191, 8192],
    "below thresholds 2048 x 4": [2048] * 4,
}


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def set_grids(on):
    for e in ENVS:
        if on:
            os.environ.pop(e, None)
        else:
            os.environ[e] = OFF


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    print(f"# {card()}", flush=True)
    rs = np.random.RandomState(0)
    results = []
    for name, sizes in WORKLOADS.items():
        x = torch.from_numpy(np.concatenate([atoms(n, rs) for n in sizes])).to(DEV, torch.float32)[None].contiguous()
        ptr = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64)
        ptr_dev = ptr.to(DEV)
        t, max_n = x.shape[1], max(sizes)
        mask = torch.ones(1, t, dtype=torch.uint8, device=DEV)
        for k in (32, 96):
            paths = {
                "knn": (lambda: _packed_select(x, ptr_dev, k, None, None, False, math.inf, "knn", max_n),
                        lambda: [knn_neighbors(x[:, int(ptr[g]):int(ptr[g + 1])], min(k, sizes[g]))
                                 for g in range(len(sizes))]),
                "radius": (lambda: _packed_select(x, ptr_dev, k, mask, None, False, 25.0, "radius", max_n),
                           lambda: [radius_neighbors_wide(x[:, int(ptr[g]):int(ptr[g + 1])], 5.0, min(k, sizes[g]),
                                                          mask=mask[:, int(ptr[g]):int(ptr[g + 1])].bool())
                                    for g in range(len(sizes))]),
            }
            for mode, (packed, unpacked) in paths.items():
                ms = {"grid": [], "all_pairs": [], "unpacked": []}
                for rep in range(args.reps + 1):
                    set_grids(True)
                    g = timed(packed, 1)
                    set_grids(False)
                    a = timed(packed, 1)
                    set_grids(True)
                    u = timed(unpacked, 1)
                    if rep:
                        ms["grid"].append(g); ms["all_pairs"].append(a); ms["unpacked"].append(u)
                row = dict(workload=name, what=f"select {mode}", k=k, T=t, G=len(sizes),
                           **{p: float(np.median(v)) for p, v in ms.items()})
                print(json.dumps(row), flush=True)
                results.append(row)
            for dtype, train in ((torch.bfloat16, False), (torch.float32, True)):
                torch.manual_seed(0)
                lay = EGNN(dim=64, m_dim=16, num_nearest_neighbors=k).to(DEV, dtype)
                feats = torch.randn(1, t, 64, device=DEV, dtype=dtype)

                def layer():
                    if train:
                        f = feats.clone().requires_grad_()
                        with torch.enable_grad():
                            out = lay(f, x, ptr=ptr_dev)
                            (out[0].float().sum() + out[1].sum()).backward()
                    else:
                        with torch.no_grad():
                            lay(feats, x, ptr=ptr_dev)
                ms = {"grid": [], "all_pairs": []}
                for rep in range(args.reps + 1):
                    set_grids(True)
                    g = timed(layer, 1)
                    set_grids(False)
                    a = timed(layer, 1)
                    if rep:
                        ms["grid"].append(g); ms["all_pairs"].append(a)
                set_grids(True)
                row = dict(workload=name, what=f"layer {'fp32 fwd+bwd' if train else 'bf16 inference'}", k=k, T=t,
                           G=len(sizes), **{p: float(np.median(v)) for p, v in ms.items()})
                print(json.dumps(row), flush=True)
                results.append(row)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=card(), results=results), f, indent=1)


if __name__ == "__main__":
    main()
