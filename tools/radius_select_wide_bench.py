"""Lists longer than 32 from the cell grid (egnn_radius_select_wide) vs the all-pairs block sort (egnn_knn_select, k > 32).

Inputs: uniform clouds in a cube with cutoff 1 (r2 = 1), every node valid (mask of ones), the density set by the mean
in-radius count (the node itself included), B = 1, fp32 coordinates.

  select     : egnn_knn_select (all pairs) vs egnn_radius_select_wide (cell grid), N in {4096, 8192, 16384},
               k in {64, 128}, mean count 1.5 k (most rows are truncated at k, some are not)
  grid       : egnn_radius_select_wide alone at N = 131072 (beyond the sort's N = 16384), mean count about 50 (k = 64)
               and about 100 (k = 128)
  layer_bf16 : EGNN(dim=128, num_nearest_neighbors=64, valid_radius=1.0) in bf16, inference forward, N = 16384,
               EGNN_B200_CELL_SELECT_MIN_N = huge (all pairs) vs 0 (cell grid)
  train_fp32 : the same layer in fp32 (dim=64), forward + backward of a training step, both paths

The arms of a pair are timed with CUDA events over --reps calls and alternated for --rounds rounds after a warm-up; one
JSON line per workload with the median and range of the rounds' milliseconds per call, the speed-up of the medians and
whether the two arms' outputs are identical.  The first line names the card, its power limit and its max SM clock.

    python tools/radius_select_wide_bench.py [--rounds 7] [--skip-layer] [--out FILE]
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
from radius_select_bench import alternate, card, cloud  # noqa: E402

NEVER = str(2 ** 40)


def select_arms(lib, x, mask, k):
    b, n, c = x.shape
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    idx_a = torch.empty((b, n, k), dtype=torch.int32, device="cuda")
    ok_a = torch.empty((b, n, k), dtype=torch.uint8, device="cuda")
    idx_c = torch.empty((b, n, k), dtype=torch.int32, device="cuda")
    nb = C.c_size_t()
    nat.check("egnn_radius_select_wide_workspace_bytes",
              lib.egnn_radius_select_wide_workspace_bytes(b, n, c, k, C.byref(nb)))
    ws = _workspace(x.device, nb.value)
    p = lambda t: C.c_void_p(t.data_ptr())
    arms = {
        "all_pairs": lambda: nat.check("egnn_knn_select", lib.egnn_knn_select(
            nat.DTYPE_F32, b, n, c, k, p(x), p(mask), None, 0, 1.0, p(idx_a), p(ok_a), st)),
        "cell": lambda: nat.check("egnn_radius_select_wide", lib.egnn_radius_select_wide(
            nat.DTYPE_F32, b, n, c, k, p(x), p(mask), None, 1.0, p(idx_c), None, p(ws), ws.numel(), st)),
    }
    for fn in arms.values():
        fn()
    same = bool(torch.equal(torch.where(ok_a.bool(), idx_a, torch.full_like(idx_a, -1)), idx_c))
    return arms, same


def bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def layer_arms(x, mask, dtype, train):
    torch.manual_seed(0)
    b, n, _ = x.shape
    dim = 128 if dtype == torch.bfloat16 else 64
    mod = EGNN(dim=dim, num_nearest_neighbors=64, valid_radius=1.0).to(dtype).cuda()
    mod.train(train)
    feats = torch.randn((b, n, dim), device="cuda", dtype=dtype)
    m = mask.bool()

    def run(env):
        os.environ["EGNN_B200_CELL_SELECT_MIN_N"] = env
        if not train:
            with torch.no_grad():
                return mod(feats, x, mask=m)
        f = feats.detach().requires_grad_(True)
        with torch.enable_grad():
            fo, xo = mod(f, x, mask=m)
            (fo.float().square().sum() + xo.float().sum()).backward()
        return fo.detach(), xo.detach()

    outs = {e: run(e) for e in ("0", NEVER)}
    same = all(torch.equal(bits(a), bits(w)) for a, w in zip(outs["0"], outs[NEVER]))
    return {"all_pairs": lambda: run(NEVER), "cell": lambda: run("0")}, same, mod


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--skip-layer", action="store_true")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "radius_select_wide_bench needs a GPU"
    lib = nat.load()
    sink = open(args.out, "a") if args.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if sink:
            sink.write(line + "\n")
            sink.flush()

    emit(dict(card()))
    for n in (4096, 8192, 16384):
        for k in (64, 128):
            x, mask, _ = cloud(1, n, 1.5 * k, seed=n + k)
            reps = max(3, int(2e6 / n))
            arms, same = select_arms(lib, x, mask, k)
            r = alternate(arms, reps, args.rounds)
            emit(dict(workload="select", B=1, N=n, k=k, mean_count=1.5 * k, reps=reps, identical=same,
                      speedup=r["median_ms"]["all_pairs"] / r["median_ms"]["cell"], **r))
    n = 131072
    for k, mean in ((64, 50), (128, 100)):
        x, mask, _ = cloud(1, n, mean, seed=n + k)
        arms, _ = select_arms(lib, x[:, :4096].contiguous(), mask[:, :4096].contiguous(), k)   # (workspace warm-up)
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        idx = torch.empty((1, n, k), dtype=torch.int32, device="cuda")
        cnt = torch.empty((1, n), dtype=torch.int32, device="cuda")
        nb = C.c_size_t()
        nat.check("egnn_radius_select_wide_workspace_bytes",
                  lib.egnn_radius_select_wide_workspace_bytes(1, n, 3, k, C.byref(nb)))
        ws = _workspace(x.device, nb.value)
        p = lambda t: C.c_void_p(t.data_ptr())
        fn = lambda: nat.check("egnn_radius_select_wide", lib.egnn_radius_select_wide(
            nat.DTYPE_F32, 1, n, 3, k, p(x), p(mask), None, 1.0, p(idx), p(cnt), p(ws), ws.numel(), st))
        r = alternate({"cell": fn}, 20, args.rounds)
        fn()
        emit(dict(workload="grid", B=1, N=n, k=k, mean_count=mean, measured_mean_count=float(cnt.float().mean()),
                  rows_over_k=float((cnt > k).float().mean()), reps=20, **r))
    if not args.skip_layer:
        x, mask, _ = cloud(1, 16384, 80, seed=7)
        for name, dtype, train in (("layer_bf16", torch.bfloat16, False), ("train_fp32", torch.float32, True)):
            arms, same, mod = layer_arms(x, mask, dtype, train)
            r = alternate(arms, 5, args.rounds, warmup=1)
            emit(dict(workload=name, B=1, N=16384, k=64, mean_count=80, reps=5, identical=same, path=mod.last_path,
                      speedup=r["median_ms"]["all_pairs"] / r["median_ms"]["cell"], **r))
            del arms, mod
            torch.cuda.empty_cache()
    os.environ.pop("EGNN_B200_CELL_SELECT_MIN_N", None)


if __name__ == "__main__":
    main()
