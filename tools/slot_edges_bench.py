"""Dense edge features vs the same features per neighbour slot, in edge-list mode (EGNN.forward(..., neighbors=)).

The c4 layer (EGNN(dim=256, edge_dim=4)) at B=8, N=4096, k=32.  The lists are computed once with egnn_knn_select,
outside the timed window.  Two modes, alternated in one run after a warm-up and timed with CUDA events:
  dense : edges [8, 4096, 4096, 4]
  slot  : neighbor_edges [8, 4096, 32, 4], the same features gathered from the dense tensor
for the bf16 forward and the fp32 forward + backward.  Inputs that require grad are made once, outside the timed
window; the dense mode's [8, 4096, 4096, 4] edge gradient is part of what the layer itself computes.  Prints one JSON
line: per-mode median milliseconds, the largest output difference between the modes (the forward must be exactly 0),
input bytes of each mode, and the GPU name and power limit.

    python tools/slot_edges_bench.py [--reps 20] [--warmup 3]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from egnn_pytorch_b200 import EGNN, _native as nat  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:      # noqa: BLE001  (reported as unknown)
        return None


def knn_lists(coors, k):
    B, N, Cd = coors.shape
    idx = torch.empty(B, N, k, dtype=torch.int32, device=coors.device)
    nat.check("egnn_knn_select", nat.load().egnn_knn_select(
        nat.DTYPE_F32, B, N, Cd, k, C.c_void_p(coors.data_ptr()), None, None, 0, float("inf"), C.c_void_p(idx.data_ptr()),
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    torch.manual_seed(0)
    B, N, k, dim, e = 8, 4096, 32, 256, 4
    dev = torch.device("cuda")
    feats = torch.randn(B, N, dim, device=dev)
    coors = torch.randn(B, N, 3, device=dev)
    edges = torch.randn(B, N, N, e, device=dev)
    nbr = knn_lists(coors, k)
    bi = torch.arange(B, device=dev)[:, None, None]
    ii = torch.arange(N, device=dev)[None, :, None]
    slot = edges[bi, ii, nbr.long()].contiguous()                   # [B, N, k, e]
    res = dict(config=dict(B=B, N=N, k=k, dim=dim, edge_dim=e), gpu=torch.cuda.get_device_name(), power_limit_w=power_limit_w())

    # ---- bf16 forward
    mod = EGNN(dim=dim, edge_dim=e).to(dev).to(torch.bfloat16)
    f16, d16, s16 = feats.bfloat16(), edges.bfloat16(), slot.bfloat16()
    res["input_bytes"] = dict(bf16=dict(dense=d16.numel() * 2, slot=s16.numel() * 2),
                              fp32=dict(dense=edges.numel() * 4, slot=slot.numel() * 4))
    runs = {"dense": lambda: mod(f16, coors, d16, neighbors=nbr), "slot": lambda: mod(f16, coors, neighbors=nbr, neighbor_edges=s16)}
    with torch.no_grad():
        outs = {m: fn() for m, fn in runs.items()}
        paths = {m: mod.last_path for m in runs}
        for m in runs:
            for _ in range(args.warmup):
                runs[m]()
        times = {m: [] for m in runs}
        for _ in range(args.rounds):
            for m in runs:
                times[m].append(timed(runs[m], args.reps))
    res["bf16_forward"] = dict(path=paths, ms={m: sorted(t)[len(t) // 2] for m, t in times.items()},
                               ms_all=times, max_abs_diff=[float((a - b).abs().max()) for a, b in zip(outs["dense"], outs["slot"])])

    # ---- fp32 forward + backward
    mod = EGNN(dim=dim, edge_dim=e).to(dev)
    gf, gx = torch.randn_like(feats), torch.randn_like(coors)

    # leaves made once, outside the timed window; torch.autograd.grad returns fresh gradients instead of accumulating
    # into .grad, so a timed step is exactly one layer forward + backward
    params = list(mod.parameters())
    leaves = {m: (feats.clone().requires_grad_(True), coors.clone().requires_grad_(True),
                  (edges if m == "dense" else slot).clone().requires_grad_(True)) for m in ("dense", "slot")}

    def step(mode):
        f, x, t = leaves[mode]
        with torch.enable_grad():
            fo, xo = mod(f, x, t, neighbors=nbr) if mode == "dense" else mod(f, x, neighbors=nbr, neighbor_edges=t)
            g = torch.autograd.grad((fo * gf).sum() + (xo * gx).sum(), [f, x, t] + params)
        return fo.detach(), xo.detach(), g[0], g[1]

    outs = {m: step(m) for m in ("dense", "slot")}
    for m in outs:
        for _ in range(args.warmup):
            step(m)
    times = {m: [] for m in outs}
    for _ in range(args.rounds):
        for m in outs:
            times[m].append(timed(lambda: step(m), max(1, args.reps // 4)))
    res["fp32_forward_backward"] = dict(
        path=mod.last_path, ms={m: sorted(t)[len(t) // 2] for m, t in times.items()}, ms_all=times,
        max_abs_diff_forward=[float((a - b).abs().max()) for a, b in zip(outs["dense"][:2], outs["slot"][:2])],
        max_abs_diff_input_grads=[float((a - b).abs().max()) for a, b in zip(outs["dense"][2:], outs["slot"][2:])])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
