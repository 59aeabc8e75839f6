"""Host-side cost of one layer call (Python + ctypes, no GPU work): the native library is replaced by a stub whose entry
points return at once, so what is timed is exactly the per-call overhead that bounds the tiny configurations (c1 / c3)
in eager mode.  Runs on any machine:  python tools/host_overhead.py"""
import ctypes as C, os, sys, time, types
import torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path[:0] = [REPO]
from egnn_pytorch_b200 import _native as nat
import egnn_pytorch_b200.egnn as E


class _Stub:
    def __getattr__(self, name):
        def f(*a):
            if name.endswith("_bytes"):
                a[-1]._obj.value = 1 << 16
            return 0
        return f


nat.load = lambda: _Stub()
E.nat.load = nat.load
E._compute_device = lambda t: t.device
torch.cuda.current_stream = lambda dev=None: types.SimpleNamespace(cuda_stream=0)
torch.cuda.is_current_stream_capturing = lambda: False
torch.cuda.Event = lambda **kw: types.SimpleNamespace(record=lambda stream=None: None)
torch.cuda.current_device = lambda: None
import contextlib
torch.cuda.device = lambda dev=None: contextlib.nullcontext()


def bench(fn, n=2000):
    for _ in range(50): fn()
    t = time.perf_counter()
    for _ in range(n): fn()
    return (time.perf_counter() - t) / n * 1e6


torch.set_grad_enabled(False)
layer = E.EGNN(dim=32, num_nearest_neighbors=8).eval()
f, x = torch.randn(1, 1024, 32), torch.randn(1, 1024, 3)
print("EGNN(dim=32, k=8) layer call, host only: %.1f us" % bench(lambda: layer(f, x)))
net = E.EGNN_Network(num_tokens=21, dim=32, depth=3, num_nearest_neighbors=8).eval()
tok = torch.randint(0, 21, (1, 1024))
print("EGNN_Network(depth=3) forward, host only: %.1f us" % bench(lambda: net(tok, x), 500))
if "--profile" in sys.argv:
    import cProfile, pstats
    pr = cProfile.Profile(); pr.enable()
    for _ in range(500): layer(f, x)
    pr.disable(); pstats.Stats(pr).sort_stats("cumulative").print_stats(25)
