"""Rounding-matched CPU reference of the bf16 tensor-core layer (torch, float64).

The fp64 oracle (oracle/egnn_oracle.py) keeps the reference's own formulation and does not round the way the bf16 path
does, so a comparison against it has to allow for every bf16 rounding of the kernels -- which hides kernel bugs of that
size.  This module restates one layer in the kernels' split form (DESIGN.md section 2) and rounds at exactly the points
where the bf16 path rounds:

  inputs and parameters     bf16 (the caller rounds them; coordinates are fp32)
  B  = h W1_j^T             bf16 table (tc_gemm / tables_small_kernel store B' = 0.5 B as bf16; A' stays fp32)
  hidden = silu(A + B + sum_q s_q Wq)          packed to bf16 (tc_pair.cuh / tc_knn.cuh, cvt.rn.bf16x2)
  m_pre = hidden W2^T       bf16 x bf16 products, fp32 accumulation (mma.sync)
  m_ij, gate, coors MLP     fp32 (not rounded)
  m_i (after the mean)      bf16 (written into node_in)
  LN(h) | m_i, h1           bf16 on the GEMM node path (dim > 64); the small-node kernels (dim <= 64) keep LN(h) and
                            the hidden layer in fp32 -- `node_fp32`
  output (after residual)   bf16
  periodic pair vector      fp32, op for op (`box=` / `cell=`, below)

s_q are the per-pair scalar channels in the kernels' order: the squared distance, sin / cos of the fourier features,
the continuous edge channels, and the one-hot degree labels (whose weights are the label embedding folded through the
label columns of W1, computed in fp32).  The reference uses exact tanh and fp64 arithmetic elsewhere; what remains
between it and a correct kernel is tanh.approx in the SiLUs, fp32 arithmetic, and bf16 rounding-boundary flips.

Under a periodic box or triclinic cell the pair vector is formed and wrapped with the kernels' fp32 operations
(common.cuh: box_axis / min_image, cell_staged / cell_wrap_n), so the image of every pair is the kernels' bit for bit:
r = fp32(x_i - x_j); per periodic axis inv = fp32(1 / L), n = rint(fp32(r * inv)) (half to even) and r = fma(-L, n, r),
a cell from its last axis to its first.  The fma is fp32(float64(-L) * n + float64(r)): L n has at most about 28
significant bits and r 24, so the float64 sum is exact and only the final rounding to fp32 remains.

With `rounding=False` nothing is rounded, and the functions equal oracle.egnn_layer_forward /
egnn_layer_forward_edge_list / egnn_network_forward to fp64 accuracy (test_gpu_tc_boundaries pins that)."""
from __future__ import annotations

import numpy as np
import torch

from oracle import egnn_oracle as O

_CHUNK_ELEMS = 1 << 24          # bound on the [rows, J, H] hidden tensor of one chunk (128 MB in fp64)


def _t(x):
    return None if x is None else torch.as_tensor(np.asarray(x, dtype=np.float64))


def bf16(x, on=True):
    """Round to bf16 as the kernels do: from an fp32 value, round to nearest even."""
    return x.float().bfloat16().double() if on else x


def fp32(x, on=True):
    return x.float().double() if on else x


def _rint(x):
    """Round half to even, as rintf / rint."""
    return torch.round(x)


def _staged_axes(diag, rounding):
    """(L, 1/L) of each axis as the kernels stage them: both 0 on an axis that is not periodic (0 or inf)."""
    per = (diag > 0) & torch.isfinite(diag)
    L = torch.where(per, diag, torch.zeros_like(diag))
    one = torch.where(per, diag, torch.ones_like(diag))
    inv = (1.0 / one.float()).double() if rounding else 1.0 / one      # fp32 division, correctly rounded
    return L, torch.where(per, inv, torch.zeros_like(inv))


def _fma(a, b, c, rounding):
    """fmaf(a, b, c) for fp32 values a * b (<= 2^29) and c: the float64 sum is exact, one rounding to fp32."""
    return fp32(a * b + c, rounding)


def wrap_box(r, box, rounding=True):
    """min_image of r [..., C] under box lengths [C] (0 or inf: the axis is not periodic)."""
    L, inv = _staged_axes(fp32(_t(box), rounding), rounding)
    return _fma(-L, _rint(fp32(r * inv, rounding)), r, rounding)


def wrap_cell(r, cell, rounding=True, first_to_last=False):
    """cell_wrap of r [..., C] under a lower-triangular cell [C, C] (rows: lattice vectors; a diagonal entry of 0 or inf
    leaves that axis aperiodic): from the last axis to the first, n = rint(r_c / L_c), r_d -= cell[c, d] n for d <= c.
    `first_to_last` runs the axes the wrong way round (a mistake the tests must see)."""
    A = fp32(_t(cell), rounding)
    C = A.shape[-1]
    L, inv = _staged_axes(torch.diagonal(A), rounding)
    r = list(r.unbind(-1))
    for c in (range(C) if first_to_last else reversed(range(C))):
        n = _rint(fp32(r[c] * inv[c], rounding))
        for d in range(c + 1):
            r[d] = _fma(-(L[c] if d == c else A[c, d]), n, r[d], rounding)
    return torch.stack(r, -1)


def lattice_bc(box, cell, b, c):
    """The per-graph lattice: ('box', [B, C]) / ('cell', [B, C, C]) from [C] / [B, C] and [C, C] / [B, C, C], or None."""
    assert box is None or cell is None, "a box or a cell, not both"
    if box is not None:
        return "box", _t(box).expand(b, c)
    if cell is not None:
        return "cell", _t(cell).expand(b, c, c)
    return None


def _silu(x):
    return x * torch.sigmoid(x)


def _layer_norm(x, g, b, eps=1e-5):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * g + b


def tc_layer_forward(params, cfg, feats, coors, edges=None, mask=None, neighbors=None, nbr_ok=None, slot_edges=False,
                     labels=None, label_emb=None, rows=None, rounding=True, node_fp32=None, messages=True, box=None,
                     cell=None):
    """One layer as the bf16 path computes it.

    feats [B,N,dim], coors [B,N,C]; edges: continuous edge channels [B,N,N,e], or [B,N,k,e] per neighbour slot with
    `slot_edges`; mask [B,N] bool; neighbors [B,N,k] int (-1 = empty slot) selects the neighbour-list form, None the
    dense all-pairs form; nbr_ok [B,N,k] bool (the valid_radius test of a top-k selection; it only acts with a mask, like
    the reference); labels [B,N,N] int and label_emb [num_labels, label_dim] the degree labels of EGNN_Network (the
    layer's cfg edge_dim counts the continuous channels plus label_dim).  `rows=(r0, r1)` evaluates rows r0:r1 only
    and returns those rows.  `node_fp32` (default: dim <= 64, the small-node kernels) keeps LN(h) and the node MLP's
    hidden layer in fp32.  `messages=False` feeds m_i = 0 to the node MLP (how much of the output the edge step
    decides).  `box` ([C] or [B, C]) or `cell` ([C, C] or [B, C, C]) wraps x_i - x_j before the distance, the fourier
    features and the coordinate update use it (fp32 op for op with `rounding`, float64 without)."""
    rd = rounding
    P = {k: _t(v) for k, v in params.items()}
    h = _t(feats)
    x = _t(coors)
    b_, n, dim = h.shape
    F = cfg["fourier_features"]
    label_dim = 0 if label_emb is None else np.shape(label_emb)[1]
    ed = cfg["edge_dim"] - label_dim
    if node_fp32 is None:
        node_fp32 = dim <= 64
    W1, b1 = P["edge_mlp.0.weight"], P["edge_mlp.0.bias"]
    W2, b2 = P["edge_mlp.3.weight"], P["edge_mlp.3.bias"]
    H = W1.shape[0]
    # per-pair scalar columns of W1 in the kernels' channel order: d | sin | cos | continuous edges | label table
    qcols = [W1[:, 2 * dim + 2 * F]] + [W1[:, 2 * dim + q] for q in range(2 * F)]
    qcols += [W1[:, 2 * dim + 2 * F + 1 + e] for e in range(ed)]
    Wq = torch.stack(qcols, 0)                                                   # [Q0, H]
    if label_emb is not None:
        tab = fp32(_t(label_emb) @ W1[:, 2 * dim + 2 * F + 1 + ed:].T, rd)     # [num_labels, H]
        Wq = torch.cat([Wq, tab], 0)
    A = h @ W1[:, :dim].T + b1                                                   # [B,N,H] (fp32 in the kernels)
    Bt = bf16(h @ W1[:, dim:2 * dim].T, rd)                                      # [B,N,H] bf16 table
    e_t = _t(edges)
    mk = None if mask is None else torch.as_tensor(np.asarray(mask).astype(bool))
    lab = None if labels is None else torch.as_tensor(np.asarray(labels).astype(np.int64))
    nb = None if neighbors is None else torch.as_tensor(np.asarray(neighbors).astype(np.int64))
    ok = None if nbr_ok is None else torch.as_tensor(np.asarray(nbr_ok).astype(bool))
    nlab = 0 if label_emb is None else np.shape(label_emb)[0]
    r0, r1 = (0, n) if rows is None else rows
    lat = lattice_bc(box, cell, b_, x.shape[-1])
    R = r1 - r0
    J = n if nb is None else nb.shape[-1]
    feats_out = h[:, r0:r1].clone()
    coors_out = x[:, r0:r1].clone()
    m_i = torch.zeros(b_, R, W2.shape[0], dtype=torch.float64)
    step = max(1, _CHUNK_ELEMS // (J * H))
    for b in range(b_):
        for s in range(r0, r1, step):
            e = min(s + step, r1)
            ii = torch.arange(s, e)
            if nb is None:
                jj = torch.arange(n).expand(e - s, n)
                sv = torch.ones(e - s, n, dtype=torch.bool)
            else:
                jj = nb[b, s:e]
                sv = jj >= 0
                jj = torch.where(sv, jj, ii[:, None])                           # an empty slot reads the node itself
            rel = x[b, s:e, None, :] - x[b][jj]                                   # [R,J,C]  x_i - x_j
            if lat is not None:
                rel = fp32(rel, rd)
                rel = (wrap_box if lat[0] == "box" else wrap_cell)(rel, lat[1][b], rd)
            d = fp32((rel ** 2).sum(-1), rd)
            sc = [d]
            if F > 0:
                scaled = d[..., None] / (2.0 ** torch.arange(F, dtype=torch.float64))
                sc += list(torch.sin(scaled).unbind(-1)) + list(torch.cos(scaled).unbind(-1))
            if ed > 0:
                ev = e_t[b, s:e] if slot_edges else e_t[b][ii[:, None], jj]
                sc += list(ev.unbind(-1))
            if nlab > 0:
                lv = lab[b][ii[:, None], jj]
                sc += [(lv == l).double() for l in range(nlab)]
            S = torch.stack(sc, -1)                                               # [R,J,Q]
            pre = A[b, s:e, None, :] + Bt[b][jj] + S @ Wq
            hid = bf16(_silu(pre), rd)
            del pre
            m = _silu(hid @ W2.T + b2)                                            # [R,J,m]
            del hid
            if cfg["soft_edges"]:
                m = m * torch.sigmoid(m @ P["edge_gate.0.weight"].T + P["edge_gate.0.bias"])
            if mk is None:
                pm = sv
            else:
                pm = sv & mk[b, s:e, None] & mk[b][jj]
                if ok is not None:
                    pm = pm & ok[b, s:e]
            if cfg["update_coors"]:
                w = (_silu(m @ P["coors_mlp.0.weight"].T + P["coors_mlp.0.bias"]) @ P["coors_mlp.3.weight"].T
                     + P["coors_mlp.3.bias"])[..., 0]
                w = torch.where(pm, w, 0.0)
                cv = cfg["coor_weights_clamp_value"]
                if cv is not None:
                    w = w.clamp(-cv, cv)
                if cfg["norm_coors"]:
                    w = w * P["coors_norm.scale"] / torch.sqrt(d).clamp_min(1e-8)
                coors_out[b, s - r0:e - r0] = x[b, s:e] + (w[..., None] * rel).sum(1)
            mm = torch.where(pm[..., None], m, 0.0).sum(1)
            if cfg["m_pool_method"] == "mean":
                if mk is not None:
                    cnt = pm.sum(-1, keepdim=True).double()
                    mm = torch.where(cnt > 0, mm / cnt.clamp_min(1.0), 0.0)
                else:
                    mm = mm / J
            m_i[b, s - r0:e - r0] = mm
    if cfg["update_coors"]:
        coors_out = fp32(coors_out, rd)
    if cfg["update_feats"]:
        hr = h[:, r0:r1]
        normed = _layer_norm(hr, P["node_norm.weight"], P["node_norm.bias"]) if cfg["norm_feats"] else hr
        node_in = torch.cat([bf16(normed, rd and not node_fp32), bf16(m_i, rd) if messages else 0.0 * m_i], -1)
        h1 = _silu(node_in @ P["node_mlp.0.weight"].T + P["node_mlp.0.bias"])
        h1 = bf16(h1, rd and not node_fp32)
        feats_out = bf16(h1 @ P["node_mlp.3.weight"].T + P["node_mlp.3.bias"] + hr, rd)
    return feats_out.numpy(), coors_out.numpy()


def tc_network_forward(params, ncfg, feats, coors, adj_mat=None, edges=None, mask=None, rounding=True, box=None,
                       cell=None):
    """EGNN_Network as the bf16 path computes it: token (+ position) embedding rounded to bf16, edge tokens embedded,
    degree labels from the expanded adjacency handed to every layer as labels with the adjacency embedding as their
    table, layers chained on bf16 features and fp32 coordinates, `box` / `cell` passed to every layer.  Global
    attention blocks are not modelled, nor a neighbour selection under a lattice."""
    assert not ncfg.get("global_layers"), "global attention blocks are not part of this reference"
    P = {k: np.asarray(v, np.float64) for k, v in params.items()}
    b = np.shape(feats)[0]
    if ncfg["num_tokens"] is not None:
        h = P["token_emb.weight"][np.asarray(feats).astype(np.int64)]
        if ncfg["num_positions"] is not None:
            h = bf16(_t(h + P["pos_emb.weight"][:h.shape[1]][None]), rounding).numpy()
    else:
        h = np.asarray(feats, np.float64)
    if edges is not None and ncfg["num_edge_tokens"] is not None:
        edges = P["edge_emb.weight"][np.asarray(edges).astype(np.int64)]
    labels = label_emb = None
    adj = adj_mat
    if ncfg["num_adj_degrees"] is not None:
        adj, lab = O.adjacency_degrees(adj_mat, ncfg["num_adj_degrees"], b)
        if ncfg["adj_dim"] > 0:
            labels, label_emb = lab, P["adj_emb.weight"]
    cfg = ncfg["layer"]
    x = np.asarray(coors, np.float64)
    for l in range(ncfg["depth"]):
        pre = f"layers.{l}.1."
        lp = {k[len(pre):]: v for k, v in P.items() if k.startswith(pre)}
        nbr = ok = None
        if cfg["num_nearest_neighbors"] > 0 or cfg["only_sparse_neighbors"]:
            assert box is None and cell is None, "the oracle's neighbour selection has no lattice"
            nbr, ok, _ = O.neighbour_selection(cfg, x, None if mask is None else np.asarray(mask).astype(bool), adj)
        h, x = tc_layer_forward(lp, cfg, h, x, edges=edges, mask=mask, neighbors=nbr, nbr_ok=ok, labels=labels,
                                label_emb=label_emb, rounding=rounding, box=box, cell=cell)
    return h, x
