"""Torch-CPU restatement of the reference's dense `EGNN.forward` -- TEST / BENCH INFRASTRUCTURE, NOT PRODUCT.

Used ONLY as the fallback of `bench.py --impl reference` / `cpu_baseline` when the unmodified reference is not
installed under oracle/_ref (then `kind` = "port" instead of "reference").  It keeps the reference's formulation
and its ATen call sequence for the dense all-pairs branch (egnn_pytorch.py:224-341): broadcast both feature
operands to [B,N,N,d], concatenate [h_i | h_j | d] (:282-285), `Linear(E,2E) -> SiLU -> Linear(2E,m) -> SiLU`
over the concatenation (:287), coors MLP and both sums (:302-333), node MLP with residual (:335-337) -- so it
allocates the same [B,N,N,E] and [B,N,N,2E] intermediates and spends its time in the same addmm / silu / cat
kernels as the reference (BASELINE.md section 2).  Parameters: a dict keyed by the reference's state-dict names.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def egnn_dense_forward(P, feats, coors, mask=None):
    b, n, d = feats.shape
    rel_coors = coors[:, :, None, :] - coors[:, None, :, :]                      # :232
    rel_dist = (rel_coors ** 2).sum(dim=-1, keepdim=True)                        # :233
    feats_i = feats[:, :, None, :].expand(b, n, n, d)                            # :279-280
    feats_j = feats[:, None, :, :].expand(b, n, n, d)                            # :277
    edge_input = torch.cat((feats_i, feats_j, rel_dist), dim=-1)                 # :282
    hidden = F.silu(F.linear(edge_input, P["edge_mlp.0.weight"], P["edge_mlp.0.bias"]))
    m_ij = F.silu(F.linear(hidden, P["edge_mlp.3.weight"], P["edge_mlp.3.bias"]))   # :287
    del hidden, edge_input
    pair_mask = None
    if mask is not None:
        pair_mask = mask[:, :, None] & mask[:, None, :]                          # :292-295
    coor_w = F.linear(F.silu(F.linear(m_ij, P["coors_mlp.0.weight"], P["coors_mlp.0.bias"])),
                      P["coors_mlp.3.weight"], P["coors_mlp.3.bias"]).squeeze(-1)   # :303-304
    if pair_mask is not None:
        coor_w = coor_w.masked_fill(~pair_mask, 0.0)                             # :309
        m_ij = m_ij.masked_fill(~pair_mask[..., None], 0.0)                      # :322
    coors_out = torch.einsum("bij,bijc->bic", coor_w, rel_coors) + coors         # :315
    m_i = m_ij.sum(dim=-2)                                                       # :333
    node_in = torch.cat((feats, m_i), dim=-1)                                    # :336
    h1 = F.silu(F.linear(node_in, P["node_mlp.0.weight"], P["node_mlp.0.bias"]))
    feats_out = F.linear(h1, P["node_mlp.3.weight"], P["node_mlp.3.bias"]) + feats   # :337
    return feats_out, coors_out
