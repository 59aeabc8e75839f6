"""Is the output of a layer call written after a CUDA-graph capture of the same module?  (bench.py's secondary block
reported a 0.0 difference to the reference for fp32 rows: stale memory or real?)"""
import sys, os, torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [REPO]
sys.path.insert(0, os.path.join(REPO, "oracle", "_ref"))
import egnn_pytorch as ref
import egnn_pytorch_b200 as ours_pkg
from egnn_pytorch_b200 import GraphedForward
torch.set_grad_enabled(False)
dev = torch.device("cuda", 0)
g = torch.Generator().manual_seed(1)
torch.manual_seed(0)
ours = ours_pkg.EGNN(dim=512).to(torch.float32).to(dev).eval()
theirs = ref.EGNN(dim=512).to(dev).eval()
theirs.load_state_dict(ours.state_dict())
f = torch.randn(1, 16, 512, generator=g).to(dev); x = torch.randn(1, 16, 3, generator=g).to(dev)


def cmp(tag):
    poison = [torch.full_like(f, float("nan")) for _ in range(8)]; del poison      # recycled blocks now hold NaN
    o = ours(f, x); r = theirs(f, x); torch.cuda.synchronize()
    print(tag, "diff feats %.3e coors %.3e nan %s" % (float((o[0] - r[0]).abs().max()), float((o[1] - r[1]).abs().max()), bool(torch.isnan(o[0]).any())))


cmp("fresh")
for _ in range(50): ours(f, x)
cmp("after 50 calls")
gf = GraphedForward(ours, f, x)
for _ in range(20): gf(f, x)
cmp("graph alive")
del gf
cmp("graph deleted")
for _ in range(30): theirs(f, x)
cmp("after reference loop")
