"""Cost of the lattice gradient (EGNN.forward(..., lattice_grad=True)): an fp32 training step (forward + backward) of
the same layer with a box and with a tilted cell, each with and without the gradient with respect to the lattice.  The
four arms are alternated over several rounds after a warm-up and timed with CUDA events.

Workloads (fp32, forward + backward):
  c4 : EGNN(dim=256, edge_dim=4, num_nearest_neighbors=32), B=8, N=4096
  c2 : EGNN(dim=512) dense, B=4, N=1024
Nodes fill the box / cell uniformly (about one node per unit volume), so many pairs cross the boundary; the tilted cell
leans its lattice vectors by up to 0.5 of the diagonal.  Prints one JSON line per workload: per-arm median and spread
(min, max) of the rounds' milliseconds, the overhead of lattice_grad=True over the same lattice without it, and the
GPU name and power limit.

    python tools/lattice_grad_bench.py [--reps 5] [--warmup 2] [--rounds 7] [--only c4]
"""
import argparse
import copy
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from egnn_pytorch_b200 import EGNN  # noqa: E402
from triclinic_bench import power_limit_w, timed  # noqa: E402


def workload(name):
    torch.manual_seed(0)
    if name == "c2":
        mod, B, N, e = EGNN(dim=512), 4, 1024, 0
    else:
        mod, B, N, e = EGNN(dim=256, edge_dim=4, num_nearest_neighbors=32), 8, 4096, 4
    mod = mod.float().cuda().train()
    L = float(N) ** (1 / 3)
    feats = torch.randn(B, N, mod.dim, device="cuda").requires_grad_(True)
    u = torch.rand(B, N, 3, device="cuda")
    edges = torch.randn(B, N, N, e, device="cuda") if e else None
    box = torch.full((3,), L, device="cuda")
    tilt = torch.tensor([[1.0, 0, 0], [0.4, 1.0, 0], [-0.5, 0.3, 1.0]], device="cuda") * L
    lattices = {"box": ("box", box, (u * L).contiguous()), "cell": ("cell", tilt, (u @ tilt).contiguous())}
    arms = {f"{k}{'_grad' if g else ''}": (k, g) for k in lattices for g in (False, True)}
    # one module per arm: a module re-reads a lattice it did not check last
    mods = {arm: copy.deepcopy(mod) for arm in arms}

    def run(arm):
        k, g = arms[arm]
        kind, lat, x = lattices[k]
        lat = lat.detach().requires_grad_(g)
        x = x.detach().requires_grad_(True)
        fo, xo = mods[arm](feats, x, edges, **{kind: lat}, lattice_grad=g)
        (fo.sum() + xo.sum()).backward()
    return run, arms, mods


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--only", default=None, help="one workload: c4 | c2")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "lattice_grad_bench needs a GPU"
    gpu, pl = torch.cuda.get_device_name(), power_limit_w()
    for name in [args.only] if args.only else ["c4", "c2"]:
        run, arms, mods = workload(name)
        for _ in range(args.warmup):
            for arm in arms:
                run(arm)
        t = {k: [] for k in arms}
        for _ in range(args.rounds):
            for arm in arms:
                t[arm].append(timed(lambda: run(arm), args.reps))
        med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
        print(json.dumps(dict(workload=name, dtype="fp32", step="forward+backward", gpu=gpu, power_limit_w=pl,
                              paths={k: m.last_path for k, m in mods.items()}, median_ms=med,
                              min_ms={k: min(v) for k, v in t.items()}, max_ms={k: max(v) for k, v in t.items()},
                              overhead={k: med[k + "_grad"] / med[k] - 1.0 for k in ("box", "cell")},
                              rounds=args.rounds, reps=args.reps)), flush=True)
        del run, arms, mods
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
