"""A/B timing of the two warpgroup layouts of the dense bf16 edge kernel (tc_pair.cuh) on bench.py's c2 workload.

    python tools/tc_pair_ab.py [--rounds 7] [--calls 50] [--out DIR]

The layouts are switched with EGNN_B200_TC_PAIR_WG (2: 2 warpgroups x 32 pairs per warp, the default; 4: 4 warpgroups x
16 pairs per warp), which the library reads at every launch, and alternate within each round (the order flips every
round).  Per layout and round: the edge kernel's time from the library's CUDA-event stage brackets (as
tools/stage_times.py) and the whole call from CUDA events, L2 flushed between calls as bench.py does.  Prints one
JSON line: the card, its power limit, and per layout the median and the min / max over the rounds.  With --out, writes
the outputs of both layouts (feats_wg{2,4}.npy, coors_wg{2,4}.npy, float32) and reports how far apart they are."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

torch.set_grad_enabled(False)

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [REPO]
import bench  # noqa: E402
from egnn_pytorch_b200 import _native as nat  # noqa: E402

ENV = "EGNN_B200_TC_PAIR_WG"


def card():
    dev = torch.cuda.current_device()
    out = dict(name=torch.cuda.get_device_name(dev))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", str(dev)], capture_output=True, text=True, timeout=20).stdout.strip().split(",")
        out.update(power_limit_w=float(q[0]), sm_max_mhz=float(q[1]))
    except Exception as e:      # noqa: BLE001
        out["power_limit_w"] = f"unavailable ({type(e).__name__})"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tc_pair_ab.py needs a GPU"
    dev = torch.device("cuda", 0)
    lib = nat.load()
    mod, feats, coors = bench.build_workload("c2", torch.bfloat16, dev)
    f, x = feats.to(dev, torch.bfloat16), coors.to(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    info = card()
    saved = os.environ.pop(ENV, None)
    res = {2: dict(edge_ms=[], call_ms=[]), 4: dict(edge_ms=[], call_ms=[])}
    outs = {}
    try:
        for r in range(args.rounds):
            for wg in ((4, 2) if r % 2 == 0 else (2, 4)):
                os.environ[ENV] = str(wg)
                for _ in range(3):
                    mod(f, x)
                torch.cuda.synchronize()
                lib.egnn_profile_read(None, None, None, 1)
                lib.egnn_profile_enable(1)
                evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                       for _ in range(args.calls)]
                for a, b in evs:
                    flush.zero_()
                    a.record()
                    last = mod(f, x)
                    b.record()
                torch.cuda.synchronize()
                ms = (C.c_float * 4)(); spans = (C.c_int32 * 4)(); launches = C.c_int64()
                lib.egnn_profile_read(ms, spans, C.byref(launches), 1)
                lib.egnn_profile_enable(0)
                assert mod.last_path == "bf16-tc" and spans[2] == args.calls, (mod.last_path, spans[2])
                res[wg]["edge_ms"].append(ms[2] / spans[2])
                res[wg]["call_ms"].append(sum(a.elapsed_time(b) for a, b in evs) / args.calls)
                outs[wg] = [t.float().cpu().numpy() for t in last]
    finally:
        os.environ.pop(ENV, None)
        if saved is not None:
            os.environ[ENV] = saved
    summary = {}
    for wg, d in res.items():
        summary[f"wg{wg}"] = {k: dict(median=statistics.median(v), min=min(v), max=max(v), rounds=v) for k, v in d.items()}
    e2, e4 = summary["wg2"]["edge_ms"]["median"], summary["wg4"]["edge_ms"]["median"]
    c2, c4 = summary["wg2"]["call_ms"]["median"], summary["wg4"]["call_ms"]["median"]
    line = dict(workload=bench.WORKLOADS["c2"]["label"], card=info, rounds=args.rounds, calls_per_round=args.calls,
                layouts=summary, edge_speedup_wg4_over_wg2=e2 / e4, call_speedup_wg4_over_wg2=c2 / c4)
    diff = {}
    for i, name in enumerate(("feats", "coors")):
        a, b = outs[2][i].astype(np.float64), outs[4][i].astype(np.float64)
        diff[name] = dict(max_abs=float(np.abs(a - b).max()), scale=float(np.abs(a).max()),
                          identical_frac=float((a == b).mean()))
    line["wg4_vs_wg2_outputs"] = diff
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        for wg in (2, 4):
            np.save(os.path.join(args.out, f"feats_wg{wg}.npy"), outs[wg][0])
            np.save(os.path.join(args.out, f"coors_wg{wg}.npy"), outs[wg][1])
    print(json.dumps(line))


if __name__ == "__main__":
    main()
