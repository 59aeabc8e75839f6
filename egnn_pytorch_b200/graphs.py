"""CUDA-graph capture of a forward call, for the launch-bound configurations (BASELINE configs 1, 3, 5: microseconds
of GPU work behind ~7 kernel launches and a Python/ctypes binding per layer).

    fast = GraphedForward(net, feats, coors, adj_mat=adj, mask=mask)     # warm-up + capture with these shapes
    feats_out, coors_out = fast(feats2, coors2)                          # copy-in, one graph launch

The library enqueues everything on the current stream and never synchronises, so a whole `EGNN` /
`EGNN_Network` forward is capturable as is; tensors passed as keyword arguments (adjacency, mask, edges) are treated
as static -- their CONTENT may be updated in place between replays, their identity may not.

Dropout cannot be captured: an `EGNN` with dropout > 0 in training mode draws a fresh mask seed on the host at every call,
and a graph would replay the seed of its capture, so every replay would apply the same masks.  Construction raises
ValueError for such a module, and so does a replay after one of its layers was put back into training mode."""
from __future__ import annotations

import torch


def _egnn_layers(module):
    """The EGNN layers of `module`, by name."""
    from .egnn import EGNN
    return [(name or type(m).__name__, m) for name, m in module.named_modules() if isinstance(m, EGNN)]


def _check_no_dropout(layers, when):
    """ValueError if one of `layers` would apply dropout (training mode, dropout > 0)."""
    live = [name for name, m in layers if m.training and m.dropout_p > 0]
    if live:
        raise ValueError(f"GraphedForward {when}: {', '.join(live)} applies dropout (training mode, dropout > 0), whose "
                         f"masks are seeded per call on the host; a CUDA graph would replay the same masks every time.  "
                         f"Call module.eval() (or build the layers with dropout=0) to capture the forward")


class GraphedForward:
    def __init__(self, module, *example_args, warmup: int = 3, **static_kwargs):
        self._layers = _egnn_layers(module)
        _check_no_dropout(self._layers, "cannot capture this module")
        self.module = module
        self.static_in = [a.clone() if torch.is_tensor(a) else a for a in example_args]
        self.kwargs = static_kwargs
        dev = next(t for t in self.static_in if torch.is_tensor(t)).device
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(warmup):                       # fills the packed-parameter / workspace / adjacency caches
                module(*self.static_in, **static_kwargs)
        torch.cuda.current_stream(dev).wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph), torch.no_grad():
            self.static_out = module(*self.static_in, **static_kwargs)

    def __call__(self, *args):
        _check_no_dropout(self._layers, "cannot replay")
        for dst, src in zip(self.static_in, args):
            if torch.is_tensor(dst):
                dst.copy_(src, non_blocking=True)
        self.graph.replay()
        return self.static_out
