"""Training-step timing (forward + backward) of the CUDA layer vs the reference's eager autograd on the same GPU.

    python tools/train_bench.py [--b 4] [--n 1024] [--dim 512] [--k 0] [--ref-b 1] [--iters 5] [--no-ref]

Prints one JSON line per arm.  The reference arm imports the unmodified reference from oracle/_ref; its batch is
`--ref-b` graphs (its autograd graph keeps ~35 GB per graph at dim=512, N=1024 in fp32) and its time is reported per
graph so the two arms compare per unit of work.
"""
import argparse
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def timed(fn, iters, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--b", type=int, default=4)
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--k", type=int, default=0)
    ap.add_argument("--edge-dim", type=int, default=0)
    ap.add_argument("--ref-b", type=int, default=1)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--no-ref", action="store_true")
    ap.add_argument("--fwd-only", action="store_true")
    a = ap.parse_args()
    dev = torch.device("cuda")
    torch.manual_seed(0)
    kw = dict(dim=a.dim, num_nearest_neighbors=a.k, edge_dim=a.edge_dim)

    def make_inputs(b):
        f = torch.randn(b, a.n, a.dim, device=dev, requires_grad=True)
        x = torch.randn(b, a.n, 3, device=dev, requires_grad=True)
        e = torch.randn(b, a.n, a.n, a.edge_dim, device=dev) if a.edge_dim else None
        return f, x, e

    def step_fn(mod, b):
        f, x, e = make_inputs(b)

        def step():
            for p in mod.parameters():
                p.grad = None
            f.grad = x.grad = None
            fo, xo = mod(f, x, e) if e is not None else mod(f, x)
            if not a.fwd_only:
                (fo.sum() + xo.sum()).backward()
        return step

    from egnn_pytorch_b200 import EGNN
    ours = EGNN(**kw).to(dev)
    pairs = a.b * a.n * (a.k or a.n)
    ms = timed(step_fn(ours, a.b), a.iters)
    print(json.dumps(dict(arm="ours fp32 fwd+bwd" if not a.fwd_only else "ours fp32 fwd (grad mode)", B=a.b, N=a.n, dim=a.dim,
                          k=a.k, ms_per_step=round(ms, 3), ms_per_graph=round(ms / a.b, 3),
                          edges_per_s=round(pairs / ms * 1e3, 1))))
    if a.no_ref:
        return
    sys.path.insert(0, os.path.join(REPO, "oracle", "_ref"))
    from egnn_pytorch import EGNN as RefEGNN
    ref = RefEGNN(**kw).to(dev)
    try:
        ms = timed(step_fn(ref, a.ref_b), max(2, a.iters // 2), warmup=1)
        print(json.dumps(dict(arm="reference eager fp32 fwd+bwd", B=a.ref_b, N=a.n, dim=a.dim, k=a.k,
                              ms_per_step=round(ms, 3), ms_per_graph=round(ms / a.ref_b, 3),
                              peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 1))))
    except torch.OutOfMemoryError as e:
        print(json.dumps(dict(arm="reference eager fp32 fwd+bwd", B=a.ref_b, error="out of memory")))


if __name__ == "__main__":
    main()
