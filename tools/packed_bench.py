"""Packed batches (`ptr=`) against the same graphs padded to the largest one (+ mask), on one GPU.

    python tools/packed_bench.py [--reps 7] [--out results.json]

For each size distribution (64 graphs of 64..1024 nodes; 1024 QM9-like graphs of 9..29 nodes), each graph kind (kNN
with k = 16, dense) and each precision (bf16 inference; fp32 forward + backward) it times, alternating the two layouts
in every repetition so that both see the same clocks:
  select   the neighbour select alone: egnn_knn_select on the padded [G, N_max] batch with its mask, against
           egnn_knn_select_packed on the [1, T] batch (kNN only; a dense layer ranks nothing)
  layer    one EGNN layer call (dim 64, m_dim 16), forward under no_grad (bf16) or forward + backward (fp32)
with CUDA events around each call, the median of --reps repetitions after two warm-up calls.  It prints the card name
and power limit first, since every time belongs to them, then one JSON line per configuration."""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from egnn_pytorch_b200 import EGNN, _native as nat   # noqa: E402
from egnn_pytorch_b200.egnn import _packed_select    # noqa: E402

DEV = "cuda"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def sizes_of(dist, rs):
    if dist == "uniform64-1024":
        return rs.randint(64, 1025, 64)
    return rs.randint(9, 30, 1024)          # QM9-like: at most 29 atoms


def timed(fn, reps):
    """-> list of milliseconds of `reps` calls of fn (events around each call)."""
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    lib = nat.load()
    print(f"# {card()}", flush=True)
    rows = []
    for dist in ("uniform64-1024", "qm9"):
        rs = np.random.RandomState(0)
        sizes = sizes_of(dist, rs)
        g, nmax, t = len(sizes), int(sizes.max()), int(sizes.sum())
        ptr = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), device=DEV)
        mask = torch.zeros(g, nmax, dtype=torch.bool, device=DEV)
        for i, n in enumerate(sizes):
            mask[i, :n] = True
        # about 8 nodes per unit volume in every graph
        extent = torch.tensor(sizes / 8.0, dtype=torch.float32, device=DEV).view(-1, 1, 1) ** (1 / 3)
        coors_pad = torch.rand(g, nmax, 3, device=DEV) * extent
        coors_pack = coors_pad[mask].unsqueeze(0).contiguous()
        for k in (16, 0):
            for prec in ("bf16", "fp32"):
                dtype = torch.bfloat16 if prec == "bf16" else torch.float32
                torch.manual_seed(0)
                lay = EGNN(dim=64, m_dim=16, num_nearest_neighbors=k).to(DEV, dtype)
                feats_pad = torch.randn(g, nmax, 64, device=DEV, dtype=dtype)
                feats_pack = feats_pad[mask].unsqueeze(0).contiguous()
                train = prec == "fp32"

                def layer(feats, coors, **kw):
                    if train:
                        f = feats.detach().requires_grad_()
                        x = coors.detach().requires_grad_()
                        fo, xo = lay(f, x, **kw)
                        (fo.float().sum() + xo.sum()).backward()
                    else:
                        with torch.no_grad():
                            lay(feats, coors, **kw)

                pad = lambda: layer(feats_pad, coors_pad, mask=mask)            # noqa: E731
                pack = lambda: layer(feats_pack, coors_pack, ptr=ptr)           # noqa: E731
                res = dict(dist=dist, graphs=g, nodes=t, n_max=nmax, padded_rows=g * nmax, k=k, prec=prec,
                           pairs_padded=g * nmax * (k or nmax), pairs_packed=int((sizes * np.minimum(k or 10 ** 9, sizes)).sum()))
                if k:
                    idx = torch.empty(g, nmax, k, dtype=torch.int32, device=DEV)
                    m8 = mask.to(torch.uint8)
                    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
                    sel_pad = lambda: nat.check("egnn_knn_select", lib.egnn_knn_select(           # noqa: E731
                        nat.DTYPE_F32, g, nmax, 3, k, C.c_void_p(coors_pad.data_ptr()), C.c_void_p(m8.data_ptr()), None, 0,
                        math.inf, C.c_void_p(idx.data_ptr()), None, st))
                    sel_pack = lambda: _packed_select(coors_pack, ptr, k, None, None, False, math.inf)   # noqa: E731
                    for f in (sel_pad, sel_pack):
                        f(); f()
                    a, b = [], []
                    for _ in range(args.reps):
                        a += timed(sel_pad, 1)
                        b += timed(sel_pack, 1)
                    res.update(select_padded_ms=float(np.median(a)), select_packed_ms=float(np.median(b)))
                for f in (pad, pack):
                    f(); f()
                a, b = [], []
                for _ in range(args.reps):
                    a += timed(pad, 1)
                    b += timed(pack, 1)
                res.update(layer_padded_ms=float(np.median(a)), layer_packed_ms=float(np.median(b)),
                           layer_speedup=float(np.median(a) / np.median(b)))
                print(json.dumps(res), flush=True)
                rows.append(res)
                del lay
                torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(dict(card=card(), rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
