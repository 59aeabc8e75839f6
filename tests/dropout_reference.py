"""The kernels' training-mode dropout restated exactly: the counter hash of `drop_mul` (egnn_pytorch_b200/csrc/common.cuh)
in numpy uint64 arithmetic, and the element keys every kernel hashes, so that the torch restatement
(tests/torch_reference.py, `drop=`) applies the very masks the kernels regenerate.

A kept hidden unit is scaled by 1/(1-p) in the layer's type: rounded to float32 for the fp32 kernels, the double itself
for the fp64 ones (as nn.Dropout does in each type).  The keys, with Hp = H rounded up to 8 (the SIMT padding of the hidden
axis) and j the global index of the neighbour (so two slots that list the same j share a mask):
  stream 0, edge_mlp hidden unit h of pair (b, i, j):    ((b N + i) N + j) Hp + h
  stream 1, coors_mlp hidden unit u of pair (b, i, j):   ((b N + i) N + j) 4m + u
  stream 2, node_mlp hidden unit c of node (b, i):       (b N + i) 2 dim + c
Row blocks keep these global keys.  `Drop(..., wrong=...)` builds the keys with one deliberate mistake (WRONG_KEYS), for
the tests that show a case would see that mistake in a kernel."""
import numpy as np
import torch

_M64 = (1 << 64) - 1
_GOLDEN = 0x9E3779B97F4A7C15
_STREAM = 0xD1B54A32D192ED03
_MIX1 = np.uint64(0xBF58476D1CE4E5B9)
_MIX2 = np.uint64(0x94D049BB133111EB)

# Mistakes a kernel could make consistently in forward and backward (finite differences cannot see them):
#   "H for Hp"           edge keys with the unpadded hidden width
#   "no b"               the graph index left out of every key (every graph of a batch gets the same masks)
#   "block-local rows"   row i counted from the start of the row block
#   "slot for j"         a neighbour-list slot keyed by its slot index instead of its neighbour
#   "chunk-local h"      the hidden channel counted within its 64-channel chunk
#   "float keep-scale"   the fp64 kernels' 1/(1-p) rounded to float32
WRONG_KEYS = ("H for Hp", "no b", "block-local rows", "slot for j", "chunk-local h", "float keep-scale")


def round_up(a, b):
    return (a + b - 1) // b * b


def threshold(p):
    """DropCfg::thr of make_drop: p 2^32 truncated to uint32 (saturating); an element is dropped when hash >> 32 < thr."""
    if p <= 0.0:
        return 0
    return int(min(p * 4294967296.0, 4294967295.0))


def keep_scale(p, dtype):
    """The multiplier of a kept unit in the kernels of `dtype`: float32(1/(1-p)) or the double 1/(1-p)."""
    s = 1.0 / (1.0 - p)
    return float(np.float32(s)) if dtype == torch.float32 else s


def hash_hi(seed, stream, idx):
    """The high 32 bits of drop_mul's splitmix64 finaliser of (idx, seed, stream), for an integer array idx."""
    z = np.asarray(idx).astype(np.uint64) * np.uint64(_GOLDEN)
    z = z + np.uint64((seed + stream * _STREAM) & _M64)
    z ^= z >> np.uint64(30)
    z *= _MIX1
    z ^= z >> np.uint64(27)
    z *= _MIX2
    z ^= z >> np.uint64(31)
    return z >> np.uint64(32)


def keep(p, seed, stream, idx):
    """bool array: the kernels keep element idx of `stream` under (p, seed)."""
    return hash_hi(seed, stream, idx) >= np.uint64(threshold(p))


def module_seeds(seed, n):
    """The per-call dropout seeds EGNN draws after torch.manual_seed(seed): one torch.randint(0, 2**62, (1,)) from the
    CPU generator per layer call with dropout active, in call order."""
    g = torch.Generator().manual_seed(seed)
    return [int(torch.randint(0, 2 ** 62, (1,), generator=g).item()) for _ in range(n)]


class Drop:
    """Dropout of one layer call: probability p and the call's seed.  Each method returns the multiplier of a hidden
    pre-activation -- 0 or keep_scale(p) -- as a tensor of `dtype` on `device`, and records which streams it served and
    how many units it dropped and kept per graph in `seen` (so a case can show that it exercised the mask)."""

    def __init__(self, p, seed, wrong=None):
        assert wrong is None or wrong in WRONG_KEYS, wrong
        self.p, self.seed, self.wrong = p, seed, wrong
        self.seen = {}

    def _mul(self, stream, keys, dtype, device):
        k = keep(self.p, self.seed, stream, keys)
        st = self.seen.setdefault(stream, np.zeros((k.shape[0], 2), np.int64))
        flat = k.reshape(k.shape[0], -1)
        st[:, 0] += (~flat).sum(1)
        st[:, 1] += flat.sum(1)
        scale = keep_scale(self.p, torch.float32 if self.wrong == "float keep-scale" else dtype)
        return torch.from_numpy(k).to(device=device, dtype=dtype) * torch.tensor(scale, dtype=dtype, device=device)

    def _bi(self, B, N, rows):
        """(b N + i) [B, R, 1] for global rows `rows`, under the key mistakes that change it."""
        b = np.arange(B, dtype=np.int64)[:, None] * (0 if self.wrong == "no b" else 1)
        i = np.asarray(rows, np.int64)
        if self.wrong == "block-local rows":
            i = i - i[0]
        return (b * N + i[None, :])[..., None]

    def _pairs(self, B, N, rows, nbr):
        """Pair index ((b N + i) N + j) [B, R, J]; nbr [B, R, J] global neighbour indices (or [J] for dense rows)."""
        j = np.broadcast_to(np.asarray(nbr, np.int64), (B, len(rows), np.shape(nbr)[-1]))
        if self.wrong == "slot for j":
            j = np.broadcast_to(np.arange(j.shape[-1]), j.shape)
        return self._bi(B, N, rows) * N + j

    def edge(self, B, N, rows, nbr, H, dtype, device):
        """[B, R, J, H] multipliers of edge_mlp.0's outputs (stream 0)."""
        Hp = H if self.wrong == "H for Hp" else round_up(H, 8)
        h = np.arange(H, dtype=np.int64)
        if self.wrong == "chunk-local h":
            h = h % 64
        return self._mul(0, self._pairs(B, N, rows, nbr)[..., None] * Hp + h, dtype, device)

    def coors(self, B, N, rows, nbr, U, dtype, device):
        """[B, R, J, U] multipliers of coors_mlp.0's outputs (stream 1, U = 4 m)."""
        return self._mul(1, self._pairs(B, N, rows, nbr)[..., None] * U + np.arange(U), dtype, device)

    def node(self, B, N, rows, D2, dtype, device):
        """[B, R, D2] multipliers of node_mlp.0's outputs (stream 2, D2 = 2 dim)."""
        return self._mul(2, self._bi(B, N, rows) * D2 + np.arange(D2), dtype, device)
