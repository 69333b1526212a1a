"""The engine's launch rules, restated once for the tests: the attention's key split (sets.cuh attn_set_split*,
attn_call_splits), the seed count and a set's sizes (sets.cuh num_seeds, set_sizes), the workspace layout (sets.cuh
plan_call, engine.cu carve, encoder_tc.cu tc_scratch), the front end's launch plans (frontend.cu, eig_power.cu, fpfh.cu) and the
spectral-matching baseline's rows per warp (spectral_matching.cu).
The tests assert that the engine reaches what these predict, and the memory contract that the restated workspace adds up
to pdsc_workspace_bytes(_packed), so the restatement cannot drift from the engine unnoticed."""
C_CH = 128                      # num_channels
RATIO = 0.1                     # cfg.ratio
TSI = 8                         # sets.cuh kAttnInvariantTiles
SPLIT_MAX_ITEMS = 320           # sets.cuh kAttnSplitMaxItems
PARTIAL_BYTES = 65536 + 1024    # encoder_tc.cu tc_scratch: one split work item's partial O and (m, l)
SETDESC_BYTES = 72              # sets.cuh SetDesc: 12 int32 + 3 int64


# ---------------------------------------------------------------------------------------------------
# the attention's key split
# ---------------------------------------------------------------------------------------------------
def attn_set_split(N, sms):
    QT, KT = -(-N // 128), -(-N // 64)
    if KT < 4:
        return 1, KT
    want = -(-sms // QT)
    ts = max(-(-KT // want), 2)
    s = -(-KT // ts)
    return (s, ts) if s >= 2 else (1, KT)


def attn_set_split_invariant(N):
    KT = -(-N // 64)
    sp = -(-KT // TSI)
    return sp, -(-KT // sp)


def call_splits(qtiles, items, sms, invariant):
    """Whether a call of `qtiles` query tiles, `items` work items when its sets are split, runs split."""
    return items > qtiles if invariant else (2 * qtiles <= sms and qtiles < items <= SPLIT_MAX_ITEMS)


def call_split(Ns, sms, invariant):
    """(split?, work items, [(sp, TS)] per set) of a tensor-core call; unsplit, every set is one item per query tile over
    all its key tiles."""
    per = [attn_set_split_invariant(n) if invariant else attn_set_split(n, sms) for n in Ns]
    qtiles = sum(-(-n // 128) for n in Ns)
    items = sum(-(-n // 128) * sp for n, (sp, _) in zip(Ns, per))
    split = call_splits(qtiles, items, sms, invariant)
    return split, (items if split else qtiles), (per if split else [(1, -(-n // 64)) for n in Ns])


def partial_items(split, items, invariant):
    """Work items whose partial O and (m, l) the tensor-core scratch holds."""
    return (items if split else 0) if invariant else SPLIT_MAX_ITEMS


# ---------------------------------------------------------------------------------------------------
# seeds and the workspace
# ---------------------------------------------------------------------------------------------------
def num_seeds(N, ratio=RATIO):
    """The reference's seed count: the length of argsort(...)[:int(N * ratio)] (PointDSC.py:174, :217)."""
    return len(range(N)[:int(N * ratio)])


def set_sizes(N, k_cfg, ratio=RATIO):
    """One set's terms of the workspace: seeds, neighbours, query / key tiles, the row length of the row-major SC, the floats
    of its SC block (row-major and tiled), of its seed-row distance block, and its neighbour slots."""
    S, k = num_seeds(N, ratio), max(min(k_cfg, N - 1), 0)
    QT, KT = -(-N // 128), -(-N // 64)
    return {"S": S, "k": k, "QT": QT, "KT": KT, "NS": KT * 64, "sc_rowmajor": N * KT * 64, "sc_tiled": KT * QT * 8192,
            "dist": (S * N + 3) & ~3, "knn": S * k}


def mirror_workspace(Ns, precision, invariant, k_cfg, sms, iters=10):
    """[(name, offset, bytes, kind)] and the total of carve(call_shape(Ns)); kind: float / index / mask / best / zero."""
    R = sum(Ns)
    B = len(Ns)
    sizes = [set_sizes(n, k_cfg) for n in Ns]
    seeds, dist, knn = (sum(z[key] for z in sizes) for key in ("S", "dist", "knn"))
    sc_row, sc_tiled = (sum(z[key] for z in sizes) for key in ("sc_rowmajor", "sc_tiled"))
    qtiles, ktiles = (sum(z[key] for z in sizes) for key in ("QT", "KT"))
    regions, off = [], 0

    def take(name, count, size, kind):
        nonlocal off
        off = -(-off // 256) * 256
        regions.append((name, off, count * size, kind))
        off += count * size

    take("sc", max(sc_row, sc_tiled), 4, "float")
    take("feat_a", R * C_CH, 4, "float")
    take("feat_b", -(-R // 128) * 128 * C_CH, 4, "float")
    take("msg", R * C_CH, 4, "float")
    if precision == "fp32":
        for name in ("q", "k", "v"):
            take(name, R * C_CH, 4, "float")
        take("h1", R * 64, 4, "float")
        take("h2", R * 64, 4, "float")
    else:
        split, items, _ = call_split(Ns, sms, invariant)
        take("tc_scratch", (qtiles + ktiles) * 65536 + 1024 + partial_items(split, items, invariant) * PARTIAL_BYTES, 1, "float")
    take("normed", R * C_CH, 4, "float")
    take("conf", R, 4, "float")
    take("key", R, 4, "float")
    take("seeds", seeds + 1, 4, "index")
    take("seedfeat", seeds * C_CH + 1, 4, "float")
    take("dist", dist + 1, 4, "float")
    take("knn", knn + 1, 4, "index")
    take("iterates", knn * iters + 1, 4, "float")
    take("seed_trans", seeds * 16 + 16, 4, "float")
    take("counts", seeds + 1, 4, "index")
    take("conv_mask", B, 4, "mask")
    take("best_key", B, 8, "best")
    take("sets", B * SETDESC_BYTES, 1, "zero")
    take("tile_set", -(-R // 128), 4, "zero")
    return regions, -(-off // 256) * 256


# ---------------------------------------------------------------------------------------------------
# the front end
# ---------------------------------------------------------------------------------------------------
MATCH_MAX_CHUNKS = 32           # frontend.cu kMatchMaxChunks
EIG_ROWS, EIG_COLS = 32, 512    # eig_power.cu: rows per CTA at most, columns per tile
CAND_CAP = 4096                 # fpfh.cu: candidates a warp of the neighbour search holds


def match_plan(rows, cols, D, fp64, sms):
    """(chunks, columns per chunk, dynamic shared memory) of one nearest_columns launch (frontend.cu)."""
    tt = 32 if fp64 else 64
    chunks = min(max(-(-4 * sms // -(-rows // 128)), 1), MATCH_MAX_CHUNKS)
    per = -(-(-(-cols // chunks)) // tt) * tt
    return -(-cols // per), per, (8 if fp64 else 4) * D * (128 + tt)


def eig_plan(B, N, ptr, sms):
    """launch_leading_eigenvector's choices: R and its regime, CTAs per set, the bulk-copy path, tiles, rows of the last CTA."""
    R, regime = EIG_ROWS, "waves"
    if B * -(-N // EIG_ROWS) < 4 * sms:
        raw = -(-(B * N) // (2 * sms))
        R = min(max(raw, 8), EIG_ROWS)
        regime = "clamp8" if raw < 8 else ("clamp32" if raw > EIG_ROWS else ("mid" if 8 < R < EIG_ROWS else "edge"))
    nparts = -(-N // R)
    return {"R": R, "regime": regime, "tma": N % 4 == 0 and ptr % 16 == 0, "ntiles": -(-N // EIG_COLS),
            "last_rows": N - (nparts - 1) * R}


def search_plan(max_nn):
    """(P, warps per CTA) of launch_hybrid_search."""
    P = 2
    while P < max_nn:
        P <<= 1
    per_warp = P * 8 + 1024 + CAND_CAP * 8
    return P, min(8, 200 * 1024 // per_warp)


# ---------------------------------------------------------------------------------------------------
# the spectral-matching baseline
# ---------------------------------------------------------------------------------------------------
SM_WARPS, SM_TILE = 8, 512      # spectral_matching.cu kSmWarps, kSmTile: warps per power CTA, columns staged per pass


def sm_rows_per_warp(Ns, sms):
    """RW of launch_spectral_matching: the most rows per warp (4, then 2) whose CTAs over the call's sets still number at
    least two per SM, else 1."""
    for rw in (4, 2):
        if sum(-(-n // (SM_WARPS * rw)) for n in Ns) >= 2 * sms:
            return rw
    return 1
