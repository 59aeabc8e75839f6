"""All-pairs select vs cell-grid radius select: the neighbour select alone and the whole bf16 layer.

Inputs: uniform clouds in a cube of side L with cutoff 1 (r2 = 1), the density set so that the mean in-radius count
(the node itself included) is about 24, or about 48 (then truncated at k = 32); every node valid (mask of ones).
Sizes: N in {1024, 2048, 4096, 8192, 16384, 65536, 131072} with B = 1, plus B = 8 at N = 4096.

  select : egnn_knn_select (all pairs, valid_radius = r2) vs egnn_radius_select (cell grid), k = 32, fp32, no box
  layer  : EGNN(dim=256, num_nearest_neighbors=32, valid_radius=1.0) in bf16 with the mask, without a box and with the
           cube as a periodic box, EGNN_B200_CELL_SELECT_MIN_N = huge (all pairs) vs 0 (cell grid)

Each pair of arms is timed with CUDA events over --reps calls, the two arms alternated for --rounds rounds after a
warm-up; one JSON line per (workload, size, density) with the median and range (min, max) of the rounds' milliseconds
per call and the speed-up of the medians.  The first line names the card, its power limit and its max SM clock.

    python tools/radius_select_bench.py [--rounds 7] [--sizes 1024,2048] [--skip-layer] [--out FILE]
"""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from egnn_pytorch_b200 import EGNN, _native as nat  # noqa: E402
from egnn_pytorch_b200.egnn import _workspace  # noqa: E402

SIZES = [(1, 1024), (1, 2048), (1, 4096), (1, 8192), (1, 16384), (1, 65536), (1, 131072), (8, 4096)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, pl, clk = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return dict(gpu=name, power_limit=pl, max_sm_clock=clk)
    except Exception as e:      # noqa: BLE001  (reported as unknown)
        return dict(gpu=torch.cuda.get_device_name(), power_limit=None, max_sm_clock=None, query_error=str(e))


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def alternate(arms, reps, rounds, warmup=2):
    for fn in arms.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    t = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            t[k].append(timed(fn, reps))
    med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
    return dict(median_ms=med, min_ms={k: min(v) for k, v in t.items()}, max_ms={k: max(v) for k, v in t.items()},
                all_ms=t)


def cloud(b, n, mean_count, seed=0):
    side = (n * (4.0 / 3.0) * math.pi / mean_count) ** (1.0 / 3.0)
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = (torch.rand((b, n, 3), generator=g, dtype=torch.float64) * side).float().cuda()
    return x, torch.ones((b, n), dtype=torch.uint8, device="cuda"), side


def select_arms(lib, x, mask, k):
    b, n, c = x.shape
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    idx_a = torch.empty((b, n, k), dtype=torch.int32, device="cuda")
    ok_a = torch.empty((b, n, k), dtype=torch.uint8, device="cuda")
    idx_c = torch.empty((b, n, k), dtype=torch.int32, device="cuda")
    nb = C.c_size_t()
    nat.check("egnn_radius_select_workspace_bytes", lib.egnn_radius_select_workspace_bytes(b, n, c, k, C.byref(nb)))
    ws = _workspace(x.device, nb.value)
    p = lambda t: C.c_void_p(t.data_ptr())
    arms = {
        "all_pairs": lambda: nat.check("egnn_knn_select", lib.egnn_knn_select(
            nat.DTYPE_F32, b, n, c, k, p(x), p(mask), None, 0, 1.0, p(idx_a), p(ok_a), st)),
        "cell": lambda: nat.check("egnn_radius_select", lib.egnn_radius_select(
            nat.DTYPE_F32, b, n, c, k, p(x), p(mask), None, 1.0, p(idx_c), None, p(ws), ws.numel(), st)),
    }
    arms["all_pairs"]()
    arms["cell"]()
    same = bool(torch.equal(torch.where(ok_a.bool(), idx_a, torch.full_like(idx_a, -1)), idx_c))
    return arms, same


def layer_arms(x, mask, box):
    torch.manual_seed(0)
    b, n, _ = x.shape
    mod = EGNN(dim=256, num_nearest_neighbors=32, valid_radius=1.0).to(torch.bfloat16).cuda().eval()
    feats = torch.randn((b, n, 256), device="cuda", dtype=torch.bfloat16)
    m = mask.bool()

    def run(env):
        os.environ["EGNN_B200_CELL_SELECT_MIN_N"] = env
        with torch.no_grad():
            return mod(feats, x, mask=m, box=box)

    outs = {e: run(e) for e in ("0", str(2 ** 40))}
    same = all(torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a, w.view(torch.int16) if w.dtype == torch.bfloat16 else w)
               for a, w in zip(outs["0"], outs[str(2 ** 40)]))
    return {"all_pairs": lambda: run(str(2 ** 40)), "cell": lambda: run("0")}, same, mod


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--sizes", default=None, help="comma-separated N (B = 1); default: the full list")
    ap.add_argument("--skip-layer", action="store_true")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "radius_select_bench needs a GPU"
    lib = nat.load()
    sink = open(args.out, "a") if args.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if sink:
            sink.write(line + "\n")
            sink.flush()

    emit(dict(card()))
    sizes = SIZES if args.sizes is None else [(1, int(s)) for s in args.sizes.split(",")]
    for b, n in sizes:
        for mean in (24, 48):
            x, mask, side = cloud(b, n, mean, seed=n + mean)
            # enough calls per measurement for ~20 ms of the slower arm (all pairs grows as N^2)
            reps = max(3, min(200, int(2e7 / (b * n * n / 4096 + 1))))
            arms, same = select_arms(lib, x, mask, 32)
            r = alternate(arms, reps, args.rounds)
            emit(dict(workload="select", B=b, N=n, mean_count=mean, k=32, reps=reps, identical=same,
                      speedup=r["median_ms"]["all_pairs"] / r["median_ms"]["cell"], **r))
            if args.skip_layer:
                continue
            for name, box in (("layer", None), ("layer_box", torch.full((3,), side, device="cuda"))):
                arms, same, mod = layer_arms(x, mask, box)
                r = alternate(arms, max(2, reps // 4), args.rounds, warmup=1)
                emit(dict(workload=name, B=b, N=n, mean_count=mean, k=32, reps=max(2, reps // 4), identical=same,
                          path=mod.last_path, speedup=r["median_ms"]["all_pairs"] / r["median_ms"]["cell"], **r))
                del arms, mod
            torch.cuda.empty_cache()
    os.environ.pop("EGNN_B200_CELL_SELECT_MIN_N", None)


if __name__ == "__main__":
    main()
