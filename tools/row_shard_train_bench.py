"""Training one graph by row blocks: fp32 forward + backward of the whole graph against the same step split into W row
blocks (`EGNN.forward(..., _rows=)`, EGNN_FLAG_ROW_PARTIAL_GRADS), as W ranks of a row-sharded graph would run it.

    python tools/row_shard_train_bench.py [--reps 5] [--warmup 2]

For each shape (dense EGNN(dim=128) N=4096; kNN EGNN(256, edge_dim=4, k=32) N=4096, the c4 layer on one graph) and each
W in (2, 4) it reports the median time of every block, their sum against the whole step (the overhead of splitting),
the peak `torch.cuda.max_memory_allocated` of every block and of the whole step, and the largest difference between the
summed block gradients and the whole-graph gradient.  With two or more GPUs it also times the real sharded step
(`parallel.row_sharded_layer_call` forward + backward + `allreduce_gradients`, NCCL), max over ranks.  Prints one JSON line
with the GPU name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from egnn_pytorch_b200 import EGNN  # noqa: E402
from egnn_pytorch_b200 import egnn as egnn_module  # noqa: E402

SHAPES = {
    "dense_dim128_N4096": (dict(dim=128), 4096),
    "knn_c4_dim256_e4_k32_N4096": (dict(dim=256, edge_dim=4, num_nearest_neighbors=32), 4096),
}


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:      # noqa: BLE001  (reported as unknown)
        return None


def inputs(cfg, n, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(1, n, cfg["dim"], generator=g).to(dev)
    x = torch.randn(1, n, 3, generator=g).to(dev)
    e = torch.randn(1, n, n, cfg["edge_dim"], generator=g).to(dev) if cfg.get("edge_dim") else None
    gf = torch.randn(1, n, cfg["dim"], generator=g).to(dev)
    gx = torch.randn(1, n, 3, generator=g).to(dev)
    return f, x, e, gf, gx


def step(mod, f, x, e, gf, gx, rows=None):
    """One forward + backward; with `rows` the loss covers the block's rows (what its rank owns)."""
    for p in mod.parameters():
        p.grad = None
    f.grad = x.grad = None
    with torch.enable_grad():
        fo, xo = mod(f, x, e, _rows=rows)
        if rows is not None:
            fo, xo, gf, gx = fo[:, rows[0]:rows[1]], xo[:, rows[0]:rows[1]], gf[:, rows[0]:rows[1]], gx[:, rows[0]:rows[1]]
        ((fo * gf).sum() + (xo * gx).sum()).backward()


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def peak_mb(fn):
    """Peak allocated memory of one call of `fn`.  The backward's scratch arena is cached per stream and only ever
    grows, so it is dropped first: otherwise a block would be charged the arena of a larger call made before it."""
    egnn_module._WORKSPACES.clear()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() / 2 ** 20


def grads(mod, f, x):
    return [f.grad.clone(), x.grad.clone()] + [p.grad.clone() for p in mod.parameters()]


def one_gpu(name, reps, warmup, dev):
    cfg, n = SHAPES[name]
    torch.manual_seed(0)
    mod = EGNN(**cfg).to(dev)
    f, x, e, gf, gx = inputs(cfg, n, dev)
    f.requires_grad_(True)
    x.requires_grad_(True)
    res = dict(B=1, N=n, layer=cfg)
    run_full = lambda: step(mod, f, x, e, gf, gx)
    res["full"] = dict(ms=timed(run_full, reps, warmup), peak_mb=peak_mb(run_full))
    want = grads(mod, f, x)
    for w in (2, 4):
        bounds = [(n * r // w, n * (r + 1) // w) for r in range(w)]
        per, total = [], None
        for rows in bounds:
            run_blk = lambda rows=rows: step(mod, f, x, e, gf, gx, rows)
            per.append(dict(rows=list(rows), ms=timed(run_blk, reps, warmup), peak_mb=peak_mb(run_blk)))
            g = grads(mod, f, x)
            total = g if total is None else [a + b for a, b in zip(total, g)]
        err = max(float((a - b).abs().max()) / max(1.0, float(b.abs().max())) for a, b in zip(total, want))
        s = sum(p["ms"] for p in per)
        res[f"W{w}"] = dict(blocks=per, sum_ms=s, overhead_vs_full=s / res["full"]["ms"] - 1.0,
                            slowest_block_vs_full=max(p["ms"] for p in per) / res["full"]["ms"],
                            max_rel_grad_diff_vs_full=err)
    return res


def _rank_worker(rank, world, port, name, reps, warmup, q):
    import torch.distributed as dist
    from egnn_pytorch_b200 import parallel
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
        cfg, n = SHAPES[name]
        torch.manual_seed(0)
        mod = EGNN(**cfg).to(dev)
        f, x, e, gf, gx = inputs(cfg, n, dev)
        r0, r1 = parallel.shard_range(n, rank, world)
        fl, xl = f[:, r0:r1].clone().requires_grad_(True), x[:, r0:r1].clone().requires_grad_(True)
        params = list(mod.parameters())

        def sharded():
            for p in params:
                p.grad = None
            fl.grad = xl.grad = None
            with torch.enable_grad():
                fo, xo = parallel.row_sharded_layer_call(
                    lambda fa, xa, rows: mod(fa, xa, e, _rows=rows), fl, xl, n)
                ((fo * gf[:, r0:r1]).sum() + (xo * gx[:, r0:r1]).sum()).backward()
            parallel.allreduce_gradients(params)

        ms = timed(sharded, reps, warmup)
        t = torch.tensor([ms], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        q.put((rank, float(t.item())))
        dist.destroy_process_group()
    except Exception as ex:  # noqa: BLE001
        q.put((rank, f"{type(ex).__name__}: {ex}"[:300]))


def multi_gpu(name, reps, warmup, world):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 30500 + os.getpid() % 2000
    procs = [ctx.Process(target=_rank_worker, args=(r, world, port, name, reps, warmup, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(sorted(q.get(timeout=1800) for _ in procs))
    for p in procs:
        p.join(timeout=60)
    return dict(world=world, ms_max_over_ranks=res.get(0), ranks=res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    dev = torch.device("cuda")
    out = dict(what="fp32 forward + backward of one graph, whole vs the sum of W row blocks (median ms per block)",
               gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w())
    for name in SHAPES:
        out[name] = one_gpu(name, a.reps, a.warmup, dev)
        torch.cuda.empty_cache()
    world = torch.cuda.device_count()
    if world >= 2:
        out["sharded_step"] = {name: multi_gpu(name, a.reps, a.warmup, world) for name in SHAPES}
    else:
        out["sharded_step"] = "not measured: needs two or more GPUs"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
