"""The reference layer (egnn_pytorch.py:224-341) and EGNN_Network (:390-454) restated in torch, so that gradients come
from autograd: on any device, in float64 (the reference gradient) or float32 (its own fp32 error), optionally with a
periodic box (minimum-image rel), and row by row.

`layer(..., rows=(r0, r1))` computes the outputs of rows r0..r1 only, with every node as a neighbour.  The loss
sum(feats_out * G_f) + sum(coors_out * G_x) is a sum over output rows, so running forward + backward block by block
with each block's rows of the cotangents and accumulating into the same leaves gives the whole gradient exactly
(`layer_grads_chunked`, `network_grads`); a block is sized so that its per-pair tensors stay near 1 GB
(`chunk_rows`).  Fixed neighbour lists come in two forms: edge-list mode (`neighbors` with -1 = empty slot, which never
carries a message) and a select's lists (`neighbors` with `ok`, the `valid_radius` flags: a slot that is not ok is
masked only when the layer has a mask, as in the reference).  Edge features may be an `Edges` of dense parts and
embedding look-ups, gathered per row block, so a [B, N, N, e] degree-label input is never built.

tests/test_periodic.py and tests/test_gpu_backward_at_size.py pin it to the golden-pinned numpy oracle."""
import numpy as np
import torch
import torch.nn.functional as TF

from oracle import egnn_oracle as O


def _t(x):
    return x if torch.is_tensor(x) else torch.as_tensor(np.array(x, np.float64))


def _like(x, ref):
    """x (numpy, list or tensor) as a tensor of ref's float type on ref's device (such a tensor passes unchanged)."""
    return _t(x).to(device=ref.device, dtype=ref.dtype)


def _bool(x, dev):
    return None if x is None else torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).to(dev).bool()


def wrap(rel, box):
    """Minimum image of rel [..., C] under box lengths broadcastable to it (0 or inf: the axis is not periodic)."""
    box = _like(box, rel)
    per = (box > 0) & torch.isfinite(box)
    L = torch.where(per, box, torch.zeros_like(box))
    inv = torch.where(per, 1.0 / torch.where(per, box, torch.ones_like(box)), torch.zeros_like(box))
    return rel - L * torch.round(rel * inv)


def box_bc(box, b, c):
    return None if box is None else _t(box).expand(b, c)


def select(cfg, rel_dist, mask, adj, r0=0):
    """Neighbour ranking + top-k of egnn_pytorch.py:237-260 for rows r0.. of the graph (rel_dist [B, R, N]), ties to the
    lowest index -> (idx [B,R,k], nbhd_mask).  mask [B, N], adj [N, N] or [B, N, N]: the whole graph's."""
    b, R, n = rel_dist.shape
    dev = rel_dist.device
    ranking = rel_dist.clone()
    k = cfg["num_nearest_neighbors"]
    vr = cfg["valid_radius"]
    if mask is not None:
        mk = _bool(mask, dev)
        ranking = ranking.masked_fill(~(mk[:, r0:r0 + R, None] & mk[:, None, :]), 1e5)
    if adj is not None:
        a = _bool(adj, dev)
        if a.dim() == 2:
            a = a.expand(b, n, n)
        if cfg["only_sparse_neighbors"]:
            k = int(a.sum(-1).max())                 # over the whole graph, not the block
            vr = 0.0
        eye = (torch.arange(R, device=dev)[:, None] + r0 == torch.arange(n, device=dev)[None])[None]
        a = a[:, r0:r0 + R] & ~eye
        ranking = ranking.masked_fill(eye, -1.0).masked_fill(a, 0.0)
    order = torch.sort(ranking, dim=-1, stable=True).indices[..., :k]
    return order, torch.gather(ranking, -1, order) <= vr


class Edges:
    """Edge features [B, N, N, e] given in parts concatenated on the last axis: dense tensors [B, N, N, e_p] and
    embedding look-ups (table [V, e_p], integer labels [B, N, N]).  Only the pairs a row block needs are gathered."""

    def __init__(self, *parts):
        self.parts = parts

    def rows(self, r0, r1, idx=None):
        out = []
        for p in self.parts:
            src = p[1] if isinstance(p, tuple) else p
            if idx is None:
                v = src[:, r0:r1]
            else:
                bi = torch.arange(idx.shape[0], device=idx.device)[:, None, None]
                v = src[bi, torch.arange(r0, r1, device=idx.device)[None, :, None], idx]
            out.append(p[0][v.long()] if isinstance(p, tuple) else v)
        return out[0] if len(out) == 1 else torch.cat(out, -1)


def _edge_rows(edges, ref, r0, r1, idx=None):
    if edges is None:
        return None
    if not isinstance(edges, Edges):
        edges = Edges(_like(edges, ref))
    return edges.rows(r0, r1, idx)


def layer(P, cfg, feats, coors, edges=None, mask=None, adj=None, box=None, neighbors=None, slot_edges=None, ok=None,
          rows=None, drop=None):
    """One EGNN layer (periodic geometry with `box`) in the type and on the device of `feats` (float64 for numpy).
    `neighbors` [B,N,k]: edge-list mode (-1 = empty slot), or with `ok` [B,N,k] a select's lists and their
    valid_radius flags; `slot_edges` [B,N,k,e] are per-slot edge features.  `rows` (r0, r1): the outputs of those rows
    only -> ([B, r1-r0, dim], [B, r1-r0, C]).  `drop`: training-mode dropout with the kernels' masks (a
    tests/dropout_reference.Drop), multiplying the outputs of edge_mlp.0, coors_mlp.0 and node_mlp.0, bias included."""
    feats = _t(feats)
    coors = _like(coors, feats)
    P = {k: _like(v, feats) for k, v in P.items()}
    dev = feats.device
    b, n, d = feats.shape
    c = coors.shape[-1]
    r0, r1 = (0, n) if rows is None else rows
    R = r1 - r0
    fi, xi = feats[:, r0:r1], coors[:, r0:r1]
    rel = xi[:, :, None] - coors[:, None]
    if box is not None:
        rel = wrap(rel, box_bc(_like(box, feats), b, c)[:, None, None, :])
    dist = (rel ** 2).sum(-1)
    mk = _bool(mask, dev)
    use_nearest = cfg["num_nearest_neighbors"] > 0 or cfg["only_sparse_neighbors"] or neighbors is not None
    bi = torch.arange(b, device=dev)[:, None, None]
    ii = torch.arange(R, device=dev)[None, :, None]
    valid = None
    if neighbors is not None:
        nb = torch.as_tensor(np.asarray(neighbors) if not torch.is_tensor(neighbors) else neighbors).to(dev).long()[:, r0:r1]
        if ok is None:
            valid = nb >= 0
            nbhd = valid
        else:
            nbhd = _bool(ok, dev)[:, r0:r1]
        idx = nb.clamp_min(0)
    elif use_nearest:
        idx, nbhd = select(cfg, dist, mk, adj, r0)
    if use_nearest:
        rel, dist = rel[bi, ii, idx], dist[bi, ii, idx]
        if slot_edges is not None:
            edges = _like(slot_edges, feats)[:, r0:r1]
        else:
            edges = _edge_rows(edges, feats, r0, r1, idx)
        feats_j = feats[bi, idx]
    else:
        feats_j = feats[:, None].expand(b, R, n, d)
        edges = _edge_rows(edges, feats, r0, r1)
    j = feats_j.shape[2]
    if drop is not None:                    # the neighbour of every (row, slot): the masks are keyed by it
        nbr_j = idx.cpu().numpy() if use_nearest else np.arange(n)
        rows_i = np.arange(r0, r1)
    F = cfg["fourier_features"]
    dfeat = dist[..., None]
    if F > 0:
        sc = dist[..., None] / (2.0 ** torch.arange(F, dtype=feats.dtype, device=dev))
        dfeat = torch.cat([torch.sin(sc), torch.cos(sc), dist[..., None]], -1)
    edge_in = torch.cat([fi[:, :, None].expand(b, R, j, d), feats_j, dfeat] + ([edges] if edges is not None else []), -1)
    lin = lambda x, key: x @ P[key + ".weight"].T + P[key + ".bias"]
    h1 = lin(edge_in, "edge_mlp.0")
    if drop is not None:
        h1 = h1 * drop.edge(b, n, rows_i, nbr_j, h1.shape[-1], feats.dtype, dev)
    m = TF.silu(lin(TF.silu(h1), "edge_mlp.3"))
    del h1
    del edge_in
    if cfg["soft_edges"]:
        m = m * torch.sigmoid(lin(m, "edge_gate.0"))
    live = valid
    if mk is not None:
        mj = mk[bi, idx] if use_nearest else mk[:, None, :].expand(b, R, n)
        live = mk[:, r0:r1, None] & mj
        if use_nearest:
            live = live & nbhd
    coors_out = xi
    if cfg["update_coors"]:
        t = lin(m, "coors_mlp.0")
        if drop is not None:
            t = t * drop.coors(b, n, rows_i, nbr_j, t.shape[-1], feats.dtype, dev)
        w = lin(TF.silu(t), "coors_mlp.3")[..., 0]
        if live is not None:
            w = torch.where(live, w, torch.zeros_like(w))
        cv = cfg["coor_weights_clamp_value"]
        if cv is not None:
            w = w.clamp(-cv, cv)
        if valid is not None:
            w = torch.where(valid, w, torch.zeros_like(w))
        r = rel
        if cfg["norm_coors"]:
            r = rel / torch.linalg.vector_norm(rel, dim=-1, keepdim=True).clamp_min(1e-8) * P["coors_norm.scale"]
        coors_out = xi + (w[..., None] * r).sum(2)
    feats_out = fi
    if cfg["update_feats"]:
        mm = m if live is None else torch.where(live[..., None], m, torch.zeros_like(m))
        m_i = mm.sum(2)
        if cfg["m_pool_method"] == "mean":
            if mk is not None:
                cnt = live.to(feats.dtype).sum(-1, keepdim=True)
                m_i = torch.where(cnt == 0, torch.zeros_like(m_i), m_i / cnt.clamp_min(1e-8))
            else:
                m_i = m_i / j
        normed = TF.layer_norm(fi, (d,), P["node_norm.weight"], P["node_norm.bias"], 1e-5) if cfg["norm_feats"] else fi
        t = lin(torch.cat([normed, m_i], -1), "node_mlp.0")
        if drop is not None:
            t = t * drop.node(b, n, rows_i, t.shape[-1], feats.dtype, dev)
        feats_out = lin(TF.silu(t), "node_mlp.3") + fi
    return feats_out, coors_out


# ----------------------------------------------------------------------------- row blocks


def chunk_rows(cfg, B, N, J, itemsize, budget=2 ** 30):
    """Rows per block so that one block's per-pair tensors, autograd's saved ones included, stay near `budget` bytes:
    about 4 E + 6 H + 16 m values per selected pair (edge input, both hidden layers and their gradients, the message
    MLPs) and 16 per candidate pair (rel, distances, the ranking and its sort)."""
    E = O.edge_input_dim(cfg)
    H = 2 * E
    per_row = B * J * itemsize * (4 * E + 6 * H + 16 * cfg["m_dim"] + 32) + B * N * 16 * 8
    return int(max(1, min(N, budget // per_row)))


def _blocks(n, chunk):
    return [(r0, min(n, r0 + chunk)) for r0 in range(0, n, chunk)]


def _width(cfg, n, neighbors, adj):
    if neighbors is not None:
        return neighbors.shape[-1]
    if cfg["only_sparse_neighbors"] and adj is not None:
        return int(_bool(adj, "cpu" if not torch.is_tensor(adj) else adj.device).sum(-1).max())
    return min(n, cfg["num_nearest_neighbors"]) if cfg["num_nearest_neighbors"] > 0 else n


def layer_forward(P, cfg, feats, coors, edges=None, mask=None, adj=None, box=None, neighbors=None, ok=None, chunk=None,
                  drop=None):
    """Whole-graph outputs of `layer`, computed block by block without a graph."""
    feats = _t(feats)
    b, n, _ = feats.shape
    chunk = chunk or chunk_rows(cfg, b, n, _width(cfg, n, neighbors, adj), feats.element_size())
    with torch.no_grad():
        outs = [layer(P, cfg, feats, coors, edges, mask, adj, box, neighbors, None, ok, rows=r, drop=drop)
                for r in _blocks(n, chunk)]
    return torch.cat([o[0] for o in outs], 1), torch.cat([o[1] for o in outs], 1)


def layer_grads_chunked(P, cfg, feats, coors, gf, gx, edges=None, mask=None, adj=None, box=None, neighbors=None,
                        ok=None, slot_edges=None, chunk=None, leaves=None, drop=None):
    """Gradients of sum(fo * gf) + sum(xo * gx) through `layer`, forward + backward one row block at a time, in the type
    and on the device of `feats` -> {'in.feats', 'in.coors', ['in.edges'], 'p.<key>'}.  `leaves`: existing leaf
    tensors (feats, coors, params) to accumulate into instead of fresh ones."""
    feats = _t(feats)
    lf = feats.detach().clone().requires_grad_(True)
    lx = _like(coors, feats).detach().clone().requires_grad_(True)
    LP = {k: _like(v, feats).detach().clone().requires_grad_(True) for k, v in P.items()}
    le = None
    e = slot_edges if slot_edges is not None else edges
    if e is not None and not isinstance(e, Edges):
        le = _like(e, feats).detach().clone().requires_grad_(True)
        e = le
    b, n, _ = feats.shape
    chunk = chunk or chunk_rows(cfg, b, n, _width(cfg, n, neighbors, adj), feats.element_size())
    gf, gx = _like(gf, feats), _like(gx, feats)
    with torch.enable_grad():
        for r0, r1 in _blocks(n, chunk):
            fo, xo = layer(LP, cfg, lf, lx, None if slot_edges is not None else e, mask, adj, box, neighbors,
                           e if slot_edges is not None else None, ok, rows=(r0, r1), drop=drop)
            ((fo * gf[:, r0:r1]).sum() + (xo * gx[:, r0:r1]).sum()).backward()
    out = {"in.feats": lf.grad, "in.coors": lx.grad}
    if le is not None:
        out["in.edges"] = le.grad
    out.update({f"p.{k}": (torch.zeros_like(v) if v.grad is None else v.grad) for k, v in LP.items()})
    return out


def layer_grads(case, box, gf, gx, neighbors=None, slot_edges=None):
    """`layer_grads_chunked` of a tests/cases.py layer case in float64 on the CPU, as numpy."""
    ins = case["inputs"]
    g = layer_grads_chunked(case["params"], case["cfg"], ins["feats"], ins["coors"], gf, gx, ins.get("edges"),
                            ins.get("mask"), ins.get("adj_mat"), box, neighbors, slot_edges=slot_edges)
    return {k: v.numpy() for k, v in g.items()}


# ----------------------------------------------------------------------------- EGNN_Network


def adjacency_degrees(adj_mat, num_adj_degrees, b, dev):
    """N-th degree adjacency by repeated squaring of the expanded matrix (egnn_pytorch.py:414-428) -> (adjacency bool
    [B,N,N], degree labels uint8 [B,N,N])."""
    adj = _bool(adj_mat, dev)
    if adj.dim() == 2:
        adj = adj.expand(b, *adj.shape)
    labels = adj.to(torch.uint8)
    for ind in range(num_adj_degrees - 1):
        a = adj.float()                              # counts below 2^24: exact
        nxt = (a @ a) > 0
        labels = torch.where(nxt ^ adj, torch.tensor(ind + 2, dtype=torch.uint8, device=dev), labels)
        adj = nxt
    return adj, labels


def _embed(P, ncfg, feats, dev):
    """Node features of the first layer: token and position embeddings (egnn_pytorch.py:401-408)."""
    h = feats
    if ncfg["num_tokens"] is not None:
        h = P["token_emb.weight"][torch.as_tensor(np.asarray(feats) if not torch.is_tensor(feats) else feats).to(dev).long()]
    if ncfg["num_positions"] is not None:
        h = h + P["pos_emb.weight"][:h.shape[1]][None]
    return h


def _edge_input(P, ncfg, edges, adj_mat, b, dev):
    """The layers' edge input as an `Edges` over the tables in P (edge tokens, degree labels; :410-432) and their
    adjacency.  The look-ups run per row block, so gradients reach the tables through every layer's blocks."""
    parts = []
    if edges is not None:
        if ncfg["num_edge_tokens"] is not None:
            parts.append((P["edge_emb.weight"], torch.as_tensor(np.asarray(edges)).to(dev)))
        else:
            parts.append(edges)
    adj = adj_mat
    if ncfg["num_adj_degrees"] is not None:
        adj, labels = adjacency_degrees(adj_mat, ncfg["num_adj_degrees"], b, dev)
        if ncfg["adj_dim"] > 0:
            parts.append((P["adj_emb.weight"], labels))
    return (Edges(*parts) if parts else None), adj


def _layer_params(P, l):
    prefix = f"layers.{l}.1."
    return {k[len(prefix):]: v for k, v in P.items() if k.startswith(prefix)}


def _is_float(a):
    return a.is_floating_point() if torch.is_tensor(a) else np.issubdtype(np.asarray(a).dtype, np.floating)


def _leaves(P, feats, edges, coors, ref):
    """Fresh leaves of ref's type: every parameter, the coordinates, and features / edges given as floats."""
    leaf = lambda a: _like(a, ref).detach().clone().requires_grad_(True)
    f = leaf(feats) if _is_float(feats) else feats
    e = leaf(edges) if edges is not None and _is_float(edges) else edges
    return {k: leaf(v) for k, v in P.items()}, f, e, leaf(coors)


def network(P, ncfg, feats, coors, adj_mat=None, edges=None, mask=None, box=None, chunk=None, dtype=torch.float64,
            device="cpu", drop=None):
    """`EGNN_Network.forward` (no global attention) -> (feats, coors, [(h, x) input of every layer]), without a graph.
    `drop`: one `layer` dropout per layer (a list), or None."""
    ref = torch.zeros((), dtype=dtype, device=device)
    LP, f, e, x = _leaves(P, feats, edges, coors, ref)
    with torch.no_grad():
        h = _embed(LP, ncfg, f, ref.device)
        E, adj = _edge_input(LP, ncfg, e, adj_mat, h.shape[0], ref.device)
        states = [(h, x)]
        for l in range(ncfg["depth"]):
            h, x = layer_forward(_layer_params(LP, l), ncfg["layer"], h, x, E, mask, adj, box, chunk=chunk,
                                 drop=None if drop is None else drop[l])
            states.append((h, x))
    return h, x, states[:-1]


def network_grads(P, ncfg, feats, coors, gf, gx, adj_mat=None, edges=None, mask=None, box=None, chunk=None,
                  dtype=torch.float64, device="cpu", drop=None):
    """Gradients of sum(fo * gf) + sum(xo * gx) through `network`: the layers' inputs by a forward without a graph,
    then each layer in reverse, block by block, then the embeddings -> {'in.coors', ['in.feats'], ['in.edges'],
    'p.<state-dict key>'}."""
    ref = torch.zeros((), dtype=dtype, device=device)
    LP, f, e, x = _leaves(P, feats, edges, coors, ref)
    cfg = ncfg["layer"]
    with torch.no_grad():
        h = _embed(LP, ncfg, f, ref.device)
    E, adj = _edge_input(LP, ncfg, e, adj_mat, h.shape[0], ref.device)
    states = [(h, x.detach())]
    for l in range(ncfg["depth"] - 1):
        states.append(layer_forward(_layer_params(LP, l), cfg, *states[-1], E, mask, adj, box, chunk=chunk,
                                    drop=None if drop is None else drop[l]))
    gh, gxx = _like(gf, ref), _like(gx, ref)
    b, n = gh.shape[:2]
    with torch.enable_grad():
        for l in reversed(range(ncfg["depth"])):
            hin = states[l][0].detach().clone().requires_grad_(True)
            xin = states[l][1].detach().clone().requires_grad_(True)
            lp = _layer_params(LP, l)
            c = chunk or chunk_rows(cfg, b, n, _width(cfg, n, None, adj), ref.element_size())
            for r0, r1 in _blocks(n, c):
                fo, xo = layer(lp, cfg, hin, xin, E, mask, adj, box, rows=(r0, r1), drop=None if drop is None else drop[l])
                ((fo * gh[:, r0:r1]).sum() + (xo * gxx[:, r0:r1]).sum()).backward()
            gh, gxx = hin.grad, xin.grad
        h0 = _embed(LP, ncfg, f, ref.device)
        if h0.requires_grad:
            h0.backward(gh)
    out = {"in.coors": gxx}
    if torch.is_tensor(f) and f.requires_grad:
        out["in.feats"] = f.grad
    if torch.is_tensor(e) and e.requires_grad:
        out["in.edges"] = e.grad
    out.update({f"p.{k}": (torch.zeros_like(v) if v.grad is None else v.grad) for k, v in LP.items()})
    return out


# ----------------------------------------------------------------------------- neighbour-rank margins


def knn_gap(coors, k, mask=None, box=None, chunk=512):
    """Smallest relative gap between the k-th and (k+1)-th smallest squared distance over rows with k < N (unmasked
    candidates only): how far the inputs are from a tie at the k-th rank."""
    x = _t(coors)
    b, n, c = x.shape
    if k == 0 or k >= n:
        return 1.0
    mk = _bool(mask, x.device)
    gap = 1.0
    for r0, r1 in _blocks(n, chunk):
        rel = x[:, r0:r1, None] - x[:, None]
        if box is not None:
            rel = wrap(rel, box_bc(_like(box, x), b, c)[:, None, None, :])
        d = (rel ** 2).sum(-1)
        if mk is not None:
            d = d.masked_fill(~(mk[:, r0:r1, None] & mk[:, None, :]), 1e5)
        s = torch.topk(d, k + 1, -1, largest=False).values
        live = s[..., k] < 1e5                       # (masked candidates tie at 1e5; they never carry a message)
        if live.any():
            gap = min(gap, float(((s[..., k] - s[..., k - 1]) / s[..., k].clamp_min(1e-12))[live].min()))
    return gap
