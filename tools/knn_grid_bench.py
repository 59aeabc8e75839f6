"""k-nearest lists from the kNN cell grid (egnn_knn_grid_select) vs the all-pairs select (egnn_knn_select).

  select     : egnn_knn_select vs egnn_knn_grid_select, fp32, valid_radius inf, no mask; N in {2048, 4096, 8192,
               16384, 65536, 131072}, k in {8, 32, 64, 128}, B in {1, 8} (B * N <= 131072 for B = 8), clouds: uniform in
               a unit cube, N(0, 1) (what bench.py's c4 feeds), chain-like clusters (random walks of 64 nodes, blobs
               far apart) and a uniform cloud in a periodic unit box.  k > 32 beyond N = 16384 has no all-pairs arm
               (the block sort's limit): the grid is timed alone.
  layer_bf16 : EGNN(dim=64, num_nearest_neighbors=k) in bf16, inference forward on N(0, 1) coordinates,
               EGNN_B200_KNN_GRID_MIN_N = huge (all pairs) vs 0 (kNN grid), k in {8, 32}.

The arms of a pair are timed with CUDA events over --reps calls and alternated for --rounds rounds after a warm-up; one
JSON line per workload with the median and range of the rounds' milliseconds per call, the speed-up of the medians and
whether the two arms' outputs are bit-identical.  The first line names the card, its power limit and max SM clock.

    python tools/knn_grid_bench.py [--rounds 5] [--reps 5] [--quick] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from egnn_pytorch_b200 import EGNN, _native as nat  # noqa: E402
from egnn_pytorch_b200.egnn import _workspace  # noqa: E402
from radius_select_bench import alternate, card  # noqa: E402

NEVER = str(2 ** 40)


def make_cloud(kind, b, n, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    if kind == "normal":
        x = torch.randn((b, n, 3), generator=g)
    elif kind == "chains":
        steps = 0.05 * torch.randn((b, n // 64 + 1, 64, 3), generator=g)
        starts = 20.0 * torch.rand((b, n // 64 + 1, 1, 3), generator=g)
        x = (starts + steps.cumsum(2)).reshape(b, -1, 3)[:, :n]
    else:                                             # uniform, also the periodic box's cloud
        x = torch.rand((b, n, 3), generator=g)
    return x.contiguous().cuda()


def select_arms(lib, x, k, box):
    b, n, c = x.shape
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())      # noqa: E731
    idx_a, ok_a = torch.empty((b, n, k), dtype=torch.int32, device="cuda"), torch.empty((b, n, k), dtype=torch.uint8, device="cuda")
    idx_g, ok_g = torch.empty_like(idx_a), torch.empty_like(ok_a)
    nb = C.c_size_t()
    nat.check("egnn_knn_grid_select_workspace_bytes", lib.egnn_knn_grid_select_workspace_bytes(b, n, c, k, C.byref(nb)))
    ws = _workspace(x.device, nb.value)
    arms = {}
    if box is None and (k <= 32 or n <= 16384):
        arms["all_pairs"] = lambda: nat.check("egnn_knn_select", lib.egnn_knn_select(
            nat.DTYPE_F32, b, n, c, k, p(x), None, None, 0, float("inf"), p(idx_a), p(ok_a), st))
    arms["grid"] = lambda: nat.check("egnn_knn_grid_select", lib.egnn_knn_grid_select(
        nat.DTYPE_F32, b, n, c, k, p(x), None, p(box), float("inf"), p(idx_g), p(ok_g), p(ws), ws.numel(), st))
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    same = bool(torch.equal(idx_a, idx_g) and torch.equal(ok_a, ok_g)) if "all_pairs" in arms else None
    return arms, same


def layer_arms(k, b, n):
    torch.manual_seed(0)
    mod = EGNN(dim=64, num_nearest_neighbors=k).cuda().to(torch.bfloat16).eval()
    x = make_cloud("normal", b, n)
    f = torch.randn((b, n, 64), device="cuda").to(torch.bfloat16)
    outs = {}

    def arm(env):
        def run():
            os.environ["EGNN_B200_KNN_GRID_MIN_N"] = env
            with torch.no_grad():
                outs[env] = mod(f, x)
        return run
    arms = {"all_pairs": arm(NEVER), "grid": arm("0")}
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    same = all(torch.equal(a.view(torch.int16), g.view(torch.int16)) for a, g in zip(outs[NEVER], outs["0"]))
    return arms, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--quick", action="store_true", help="N <= 16384 and one cloud per N beyond")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = nat.load()
    lines = [dict(card=card())]
    print(json.dumps(lines[0]), flush=True)

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    for n in (2048, 4096, 8192, 16384, 65536, 131072):
        for b in (1, 8):
            if b * n > 131072:
                continue
            for kind in ("uniform", "normal", "chains", "box"):
                if a.quick and n > 16384 and kind != "normal":
                    continue
                for k in (8, 32, 64, 128):
                    x = make_cloud(kind, b, n, seed=n + k)
                    box = torch.ones((b, 3), device="cuda") if kind == "box" else None
                    arms, same = select_arms(lib, x, k, box)
                    r = alternate(arms, a.reps, a.rounds)
                    med = r["median_ms"]
                    emit(dict(workload="select", N=n, B=b, k=k, cloud=kind, median_ms=med, min_ms=r["min_ms"],
                              max_ms=r["max_ms"], identical=same,
                              speedup=(med["all_pairs"] / med["grid"]) if "all_pairs" in med else None))
    for n in (2048, 4096, 8192, 16384):
        for b in (1, 8):
            for k in (8, 32):
                arms, same = layer_arms(k, b, n)
                r = alternate(arms, a.reps, a.rounds)
                med = r["median_ms"]
                emit(dict(workload="layer_bf16", N=n, B=b, k=k, cloud="normal", median_ms=med, min_ms=r["min_ms"],
                          max_ms=r["max_ms"], identical=same, speedup=med["all_pairs"] / med["grid"]))
    if a.out:
        with open(a.out, "w") as fh:
            for d in lines:
                fh.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
