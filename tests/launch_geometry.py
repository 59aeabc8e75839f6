"""The host launch rules of the edge kernels, the node GEMMs and the neighbour select, restated once in Python for the
boundary tests' coverage checks (`test_table_covers_every_*`), which work out from a case's shape which tiles, grids and
instantiations the launch code picks.  Each function names the C++ function it mirrors."""
from oracle import egnn_oracle as O

H100_SMS = 132          # H100 SXM


def ceil_div(a, b):
    return -(-a // b)


def round_up(x, m):
    return ceil_div(x, m) * m


def layer_dims(kind, cfg):
    """(layer cfg, continuous edge channels, label_dim, degree labels) of an EGNN ("layer") or EGNN_Network
    ("network") built with the keyword arguments `cfg`: a network feeds its degree labels to the layer as label_dim
    more edge channels, one-hot over `labels` rows."""
    if kind == "network":
        ncfg = O.network_cfg(**cfg)
        layer = ncfg["layer"]
        label_dim = ncfg["adj_dim"] if ncfg["num_adj_degrees"] is not None else 0
        labels = ncfg["num_adj_degrees"] + 1 if label_dim else 0
        return layer, layer["edge_dim"] - label_dim, label_dim, labels
    layer = O.layer_cfg(**cfg)
    return layer, layer["edge_dim"], 0, 0


# ------------------------------------------------------------------ SIMT edge step, forward (simt_host.cuh)

SIMT_SMEM_MAX = 220 * 1024      # simt_host.cuh: the dense edge step falls back to one row per thread above it
PAIR_THREADS, PAIR_CH, PAIR_J = 128, 64, 32


def simt_mp(m):
    """MP, the width of the message accumulators (SimtPackLayout)."""
    return 16 if m <= 16 else 32


def pair_tiled_smem_bytes(MP, Q, m, PP, itemsize):
    """Dynamic shared memory of pair_dense_tiled_kernel at PP rows per thread (simt_kernels.cuh)."""
    n = 64 * MP + Q * 64 + 64 * 33 + (PP * Q * 128 if Q > 1 else 0) + 4 * m * MP + 8 * m + 2 * MP + 4
    if PP > 1:
        n += 4 * PP * (MP + 8 + 4)
    return round_up(n * itemsize, 16) + 16


def pair_dense_pp(MP, Q, m, itemsize):
    """Rows per thread of the dense edge step (launch_pair_dense): 2 where its shared memory fits, else 1; fp64 with
    MP = 32 always 1."""
    return 1 if (MP == 32 and itemsize == 8) or pair_tiled_smem_bytes(MP, Q, m, 2, itemsize) > SIMT_SMEM_MAX else 2


def simt_hsplit(B, N, Hp, k, row0, row1):
    """CTAs over the hidden axis of tiny dense graphs (simt_hsplit)."""
    whole = row0 == 0 and row1 == N
    return min(32, ceil_div(Hp, PAIR_CH)) if (k == 0 and B * N * N <= 4096 and Hp >= 512 and whole) else 1


def slot_group(k):
    """TS, the lanes per row of the neighbour-list kernels (launch_layer_simt, layer_backward)."""
    return min(32, 1 << (k - 1).bit_length())


# ------------------------------------------------------------------ SIMT backward (egnn_backward_impl.cuh)

BW2_TH, BW2_ROWS, BW2_LIST_ROWS = 128, 32, 16
DSILU_CTAS = 2048
SAVE_PAIR_MB = 1024             # egnn.py: EGNN_B200_SAVE_PAIR_MB's default


def bwd2_qr(Q, labels):
    """QR of the list bwd2 (launch_pair_bwd): 1 for the distance channel alone, 8 for up to 8 channels in registers,
    else 0."""
    return 1 if (Q == 1 and not labels) else (8 if Q <= 8 else 0)


def bwd3_rows(k):
    """Rows per CTA of bwd1 / bwd3 (launch_pair_bwd: PAIR_THREADS / TS, TS = 32 dense)."""
    return PAIR_THREADS // (slot_group(k) if k else 32)


def launch_gemm_acc(Mr, Nc, K, sms=H100_SMS):
    """(splits, K per split, K of the last split) of launch_gemm_acc."""
    tiles = ceil_div(Mr, 64) * ceil_div(Nc, 64)
    splits = max(1, min(ceil_div(2 * sms, tiles), ceil_div(K, 64)))
    kper = round_up(ceil_div(K, splits), 16)
    splits = ceil_div(K, kper)
    return splits, kper, K - (splits - 1) * kper


def dsilu_strides(n):
    """Grid-stride steps of dsilu_mul_kernel over n elements (256 threads, at most DSILU_CTAS CTAs)."""
    return ceil_div(n, min(DSILU_CTAS, ceil_div(n, 256)) * 256)


def pre2_saved(B, N, J, m, itemsize, budget_mb=SAVE_PAIR_MB):
    """Whether the training forward keeps W2 silu(pre1) per pair for the backward (egnn.py: within the budget)."""
    return B * N * J * simt_mp(m) * itemsize <= budget_mb * 2 ** 20


def simt_layer(kind, cfg, B, N, k=0, C=3, rows=None):
    """The SIMT launch of a layer (kind, cfg as layer_dims) on B graphs of N nodes: k > 0 neighbour lists of width k,
    `rows` a row block (r0, r1).  PP is per element size (8: fp64, 4: fp32)."""
    layer, _, label_dim, labels = layer_dims(kind, cfg)
    dim, m, F = layer["dim"], layer["m_dim"], layer["fourier_features"]
    E = O.edge_input_dim(layer)                      # 2 dim + Q + label_dim
    Q = E - 2 * dim - label_dim
    Hp = round_up(2 * E, 8)
    MP = simt_mp(m)
    r0, r1 = rows or (0, N)
    R = r1 - r0
    splits, kper, _ = launch_gemm_acc(dim, 2 * dim, B * N)          # dWn2 = go^T h1, K = B*N
    TI2, per_cta = BW2_LIST_ROWS if k else BW2_ROWS, bwd3_rows(k)           # rows per bwd2 CTA, per bwd1 / bwd3 CTA
    g = dict(E=E, Q=Q, Hp=Hp, MP=MP, m=m, dim=dim, N=N, C=C, labels=labels, k=k, F=F,
             chunks=ceil_div(Hp, PAIR_CH), partial_chunk=Hp % PAIR_CH != 0,
             bwd2_ch_ctas=ceil_div(Hp, BW2_TH), partial_ch_cta=Hp % BW2_TH != 0,
             bwd2_row_ctas=ceil_div(R, TI2), partial_rows=R % TI2 != 0,
             generic_node_gemm=dim > 64, splitk=splits, partial_split=splits > 1 and (B * N) % kper != 0,
             PP={es: pair_dense_pp(MP, Q, m, es) for es in (8, 4)},
             hsplit=simt_hsplit(B, N, Hp, k, r0, r1),
             rows=R, bwd3_rows_per_cta=per_cta, bwd3_ctas=ceil_div(R, per_cta), bwd3_partial=R % per_cta != 0)
    if k == 0:
        g.update(j_passes=ceil_div(N, PAIR_J), partial_j=N % PAIR_J != 0)
    else:
        TS = slot_group(k)
        g.update(TS=TS, slot_passes=ceil_div(k, TS), partial_slots=k % TS != 0,
                 bwd2_steps=ceil_div(k, 32), partial_step=k % 32 != 0, QR=bwd2_qr(Q, labels))
    return g


# ------------------------------------------------------------------ per-node GEMM (simt_host.cuh)

SKINNY_WARPS = 4


def launch_gemm(Mr, K, Nout, itemsize, sms=H100_SMS):
    """launch_gemm's kernel: ('skinny', columns per warp) or ('tiled', whether a 64 x 64 tile is partial)."""
    V = 16 // itemsize
    if Mr <= 16 and 16 * (ceil_div(K, V) * V) * itemsize <= 96 * 1024:
        return "skinny", 4 if Nout >= sms * SKINNY_WARPS * 4 else (2 if Nout >= sms * SKINNY_WARPS * 2 else 1)
    return "tiled", Mr % 64 != 0 or Nout % 64 != 0


# ------------------------------------------------------------------ tensor-core layer (fast_path.cu)

TP_TI, TP_JB, TP_KC, TP_JSPLIT_MAX, TP_QMAX, TP_CMAX = 4, 256, 64, 8, 12, 8
TP_EPI_FLOATS = 64 * 16 + 64 + 64 + 16 + 16 + 4
TK_QE, TK_LEAN, TK_EDGES, TK_GEN = 4, 0, 1, 2
SN_DIM_MAX, SN_TABLES_M_MAX = 64, 4096
TC_SMEM_MAX = 227 * 1024


def tc_knn_smem_bytes(Hp, mode, Q, rows):
    """tc_knn_smem_bytes (tc_knn.cuh)."""
    wq_rows = 1 if mode == TK_LEAN else (1 + TK_QE if mode == TK_EDGES else Q)
    n = Hp * 32 + rows * Hp * 4 + wq_rows * Hp * 4 + TP_EPI_FLOATS * 4
    n += rows * Q * 32 * 4 if mode == TK_GEN else 0
    return n + rows * 32 * 18 * 4 + 64 + 8 + 128


def tc_pair_smem_bytes(Hp, Q, Qf, gen):
    """tc_pair_smem_bytes (tc_pair.cuh)."""
    PW, XC = (28, 8) if gen else (20, 4)
    n = Hp * 32 + Q * Hp * 4 + 2 * TP_TI * Hp * 4 + TP_EPI_FLOATS * 4 + 2 * 8 * TP_TI * PW * 8 + 8 * 32 * 18 * 4
    n += 2 * TP_TI * XC * 4 + 2 * TP_TI * 4 + 64 + (0 if gen else TP_TI * TP_JB * 4)
    n += TP_TI * TP_JB * (Qf * 4 + (Q - Qf) * 2) if gen else 0
    return n + 64 + 256


def tc_pair(B, N, C, Hp, Q, F, row0, row1, sms=H100_SMS):
    """The tc_pair launch: instantiation, j-split, items, grid, ring refills across graphs, and `supported`."""
    R = row1 - row0
    gen = not (C == 3 and Q == 1)
    rg = ceil_div(R, TP_TI)
    items = B * rg
    njb = ceil_div(N, TP_JB)
    js = 1
    while js < TP_JSPLIT_MAX and items * js < 6 * sms and js * 2 <= njb:
        js *= 2
    n_items = items * js
    grid = min(n_items, sms)
    # a ring slot refilled with a row group of another graph (tc_pair.cuh: the last warpgroup stages item x + 2 grid
    # into the slot of item x)
    graph = lambda item: item // js // rg
    return dict(kernel="tc_pair<generic>" if gen else "tc_pair<lean>", jsplit=js, items=n_items, grid=grid,
                refill_other_graph=any(graph(x) != graph(x + 2 * grid) for x in range(n_items - 2 * grid)),
                laps=ceil_div(n_items, grid), active_wgs=min(2, ceil_div(N, 128)),
                last_rows_valid=R - TP_TI * (rg - 1),
                supported=Q <= TP_QMAX and C <= TP_CMAX and tc_pair_smem_bytes(Hp, Q, 1 + 2 * F, gen) <= TC_SMEM_MAX)


def tc_knn(k, C, Hp, Q, F, edge_dim, labels, R):
    """The tc_knn launch: mode, rows per CTA (tc_knn_rows_per_cta), 32-slot groups (WIDE = k > 32), `supported`."""
    mode = TK_LEAN if edge_dim == 0 else (TK_EDGES if edge_dim <= TK_QE else TK_GEN)
    if not (C == 3 and F == 0 and labels == 0):
        mode = TK_GEN
    rows = 8 if 2 * (tc_knn_smem_bytes(Hp, mode, Q, 8) + 1024) <= TC_SMEM_MAX else 16
    groups = ceil_div(k, 32)
    return dict(kernel=f"tc_knn<{['LEAN', 'EDGES', 'GEN'][mode]},{rows}>", mode=mode, ROWS=rows,
                last_rows_valid=R - rows * (ceil_div(R, rows) - 1), groups=groups, last_group=k - 32 * (groups - 1),
                wide=k > 32,
                supported=(mode != TK_GEN or Q <= TP_QMAX) and tc_knn_smem_bytes(Hp, mode, Q, 16) <= TC_SMEM_MAX)


def tc_layer(kind, cfg, B, N, C=3, k=0, rows=None, sms=H100_SMS):
    """The tensor-core launch of a layer (kind, cfg as layer_dims): the node path, and tc_pair (k = 0) or tc_knn."""
    layer, ed, label_dim, labels = layer_dims(kind, cfg)
    dim, F = layer["dim"], layer["fourier_features"]
    r0, r1 = rows or (0, N)
    E = 2 * dim + 1 + 2 * F + ed + label_dim
    Hp = round_up(2 * E, 16)
    Q = 1 + 2 * F + ed + labels
    nchunks = ceil_div(Hp, TP_KC)
    g = dict(dim=dim, B=B, N=N, C=C, k=k, R=r1 - r0, Hp=Hp, Q=Q, F=F, edge_dim=ed, labels=labels,
             nsl_last=(Hp - (nchunks - 1) * TP_KC) // 16, rows_range=rows is not None,
             tables="small" if dim <= SN_DIM_MAX and B * N <= SN_TABLES_M_MAX else "tc_gemm",
             node="small" if dim <= SN_DIM_MAX else "tc_gemm")
    g.update(tc_pair(B, N, C, Hp, Q, F, r0, r1, sms) if k == 0 else tc_knn(k, C, Hp, Q, F, ed, labels, r1 - r0))
    return g


# ------------------------------------------------------------------ all-pairs neighbour select (knn_select.cu)

SEL_JC, SORT_SMEM_MAX = 1024, 200 * 1024


def launch_select(B, N, C, k, itemsize, sms=H100_SMS):
    """The warp select (k <= 32: warps per CTA, staging passes of SEL_JC candidates) or the block sort."""
    if k <= 32:
        warps = 16 if B * ceil_div(N, 16) >= 2 * sms else 8
        passes = ceil_div(N, SEL_JC)
        tail = N - (passes - 1) * SEL_JC                      # candidates in the last staging pass
        return dict(kernel="warp", warps=warps, passes=passes, cdim=3 if C == 3 else 0, tail64=tail % 64,
                    last_cta_rows=N - (ceil_div(N, warps) - 1) * warps,
                    smem=C * SEL_JC * itemsize + SEL_JC + warps * 64 * (itemsize + 4) + 64)
    npad = 1 << max(0, (N - 1).bit_length())
    smem = npad * (itemsize + 4)
    return dict(kernel="sort", npad=npad, smem=smem, supported=smem <= SORT_SMEM_MAX)
