"""Latency / throughput of the five BASELINE.json configurations on one GPU: this repo vs the unmodified
reference in PyTorch eager on the same GPU (if oracle/_ref is installed).  Writes one JSON line per config.
    python tools/bench_configs.py > configs.jsonl
c4 is run with the 8 graphs one GPU holds when B=64 is sharded over 8 GPUs."""
import json
import os
import sys

import torch

torch.set_grad_enabled(False)      # forward benchmark: no autograd state is kept

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [REPO, os.path.join(REPO, "tests")]
from egnn_pytorch_b200 import EGNN, EGNN_Network  # noqa: E402

ONLY = [t for t in os.environ.get("ONLY", "").split(",") if t]      # e.g. ONLY=c4 NOREF=1 for a profiler capture
DTYPES = [t for t in os.environ.get("DTYPES", "bf16,fp32").split(",") if t]


def want(tag):
    return not ONLY or tag in ONLY


try:
    if os.environ.get("NOREF"):
        raise ImportError
    sys.path.insert(0, os.path.join(REPO, "oracle", "_ref"))
    import egnn_pytorch as ref
except Exception:  # pragma: no cover
    ref = None

dev = torch.device("cuda", 0)


def chain(n):
    i = torch.arange(n)
    return (i[:, None] - i[None, :]).abs() <= 1


def timeit(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def build(cls_ours, cls_ref, kwargs, dtype):
    torch.manual_seed(0)
    ours = cls_ours(**kwargs).to(dtype).to(dev).eval()
    theirs = None
    if cls_ref is not None:
        theirs = cls_ref(**kwargs).to(dtype).to(dev).eval()
        theirs.load_state_dict(ours.state_dict())
    return ours, theirs


def run(name, ours, theirs, args, kwargs, pairs, edges, iters, ref_iters):
    with torch.no_grad():
        ms = timeit(lambda: ours(*args, **kwargs), iters)
        out = dict(config=name, ms=ms, all_pairs_per_s=pairs / ms * 1e3, edges_per_s=edges / ms * 1e3 if edges else None)
        if theirs is not None:
            try:
                rms = timeit(lambda: theirs(*args, **kwargs), ref_iters)
                o, r = ours(*args, **kwargs), theirs(*args, **kwargs)
                out.update(ref_eager_ms=rms, speedup=rms / ms,
                           max_diff_feats=float((o[0].float() - r[0].float()).abs().max()),
                           max_diff_coors=float((o[1].float() - r[1].float()).abs().max()))
            except Exception as e:  # noqa
                out.update(ref_eager_error=str(e)[:200])
        if ms < 2.0:      # launch-bound: also time the CUDA-graph replay of the same forward
            from egnn_pytorch_b200 import GraphedForward
            try:
                gf = GraphedForward(ours, *args, **kwargs)
                out["graphed_ms"] = timeit(lambda: gf(*args), iters)
                if "ref_eager_ms" in out:
                    out["graphed_speedup"] = out["ref_eager_ms"] / out["graphed_ms"]
            except Exception as e:  # noqa
                out["graphed_error"] = str(e)[:200]
    layer = ours.layers[0][1] if hasattr(ours, "layers") else ours
    out["kernel_path"] = layer.last_path
    print(json.dumps(out), flush=True)


g = torch.Generator().manual_seed(1)
R = ref.EGNN if ref else None
RN = ref.EGNN_Network if ref else None

# c1
if want("c1"):
  o, t = build(EGNN, R, dict(dim=512), torch.float32)
  run("c1 EGNN(512) B=1 N=16 fp32", o, t, (torch.randn(1, 16, 512, generator=g).to(dev), torch.randn(1, 16, 3, generator=g).to(dev)), {}, 256, None, 200, 50)
# c2 bf16 and fp32
for dt in [d for d in (torch.bfloat16, torch.float32) if want("c2") and str(d)[6:].replace("bfloat16", "bf16").replace("float32", "fp32") in DTYPES]:
    o, t = build(EGNN, R, dict(dim=512), dt)
    f, x = torch.randn(4, 1024, 512, generator=g).to(dev, dt), torch.randn(4, 1024, 3, generator=g).to(dev, dt)
    run(f"c2 EGNN(512) B=4 N=1024 {str(dt)[6:]}", o, t, (f, x), {}, 4 * 1024 * 1024, None, 20, 3)
# c3
if want("c3"):
  f, x, m = torch.randint(0, 21, (1, 1024), generator=g).to(dev), torch.randn(1, 1024, 3, generator=g).to(dev), torch.ones(1, 1024, dtype=torch.bool, device=dev)
  if "fp32" in DTYPES:
    o, t = build(EGNN_Network, RN, dict(num_tokens=21, num_positions=1024, dim=32, depth=3, num_nearest_neighbors=8, coor_weights_clamp_value=2.0), torch.float32)
    run("c3 Network depth3 dim32 N=1024 k=8 fp32", o, t, (f, x), dict(mask=m), 3 * 1024 * 1024, 3 * 1024 * 8, 100, 20)
  if "bf16" in DTYPES:
    o, t = build(EGNN_Network, RN, dict(num_tokens=21, num_positions=1024, dim=32, depth=3, num_nearest_neighbors=8, coor_weights_clamp_value=2.0), torch.bfloat16)
    run("c3 Network depth3 dim32 N=1024 k=8 bf16", o, t, (f, x.bfloat16()), dict(mask=m), 3 * 1024 * 1024, 3 * 1024 * 8, 100, 20)
# c4 (8 graphs = one GPU's share of B=64)
for dt in [d for d in (torch.bfloat16, torch.float32) if want("c4") and str(d)[6:].replace("bfloat16", "bf16").replace("float32", "fp32") in DTYPES]:
    o, t = build(EGNN, R, dict(dim=256, edge_dim=4, num_nearest_neighbors=32), dt)
    f, x = torch.randn(8, 4096, 256, generator=g).to(dev, dt), torch.randn(8, 4096, 3, generator=g).to(dev, dt)
    e = torch.randn(8, 4096, 4096, 4, generator=g).to(dev, dt)
    run(f"c4 EGNN(256,e4) k=32 N=4096 B=8/GPU {str(dt)[6:]}", o, t, (f, x, e), {}, 8 * 4096 * 4096, 8 * 4096 * 32, 10, 2)
    del e
# c5
n = 8192
for dt in [d for d in (torch.float32, torch.bfloat16) if want("c5") and str(d)[6:].replace("bfloat16", "bf16").replace("float32", "fp32") in DTYPES]:
    o, t = build(EGNN_Network, RN, dict(num_tokens=21, dim=32, depth=3, num_adj_degrees=3, adj_dim=8, only_sparse_neighbors=True), dt)
    f, x, m = torch.randint(0, 21, (1, n), generator=g).to(dev), torch.randn(1, n, 3, generator=g).to(dev, dt), torch.ones(1, n, dtype=torch.bool, device=dev)
    run(f"c5 Network only_sparse adj3 N=8192 {str(dt)[6:]}", o, t, (f, x), dict(adj_mat=chain(n).to(dev), mask=m), 3 * n * n, 3 * n * 9, 10, 2)
