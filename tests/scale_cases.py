"""The batches tests/test_gpu_scale.py runs at the batch context's occurrence limit (pb_ctx_create: 2^24).  Plain numpy:
tests/test_scale_cases.py checks, without a GPU, that each one really has the multiplicities, spans, sizes and scan
trip counts it is meant to have, so that a change to a generator cannot quietly shrink a case."""
import numpy as np

from util import batch_with_multiplicities

CTX_LIMIT = 1 << 24  # id occurrences one context holds
HOT_WIN = 8192       # k_reduce_hot: occurrences of the item's slot per bitmap window
WARM_MAX = 32        # items of more occurrences are hot
SCAN_TILE = 1024     # exclusive_scan (pb_raw.cu): ids per tile ...
SPINE_TRIP = 1024    # ... and tiles per trip of k_scan_spine's one block
FILL_BASE = np.uint64(1 << 40)  # ids of the fill: never an item's id
MARKERS = np.array([2 ** 64 - 1, 2 ** 64 - 2, 2 ** 64 - 3], np.uint64)  # KEY_EMPTY and the index's other marker values


def lengths_summing_to(rng, batch, total, lo, hi, empty=()):
    """Sample lengths drawn from lo..hi, the samples in `empty` of none, nudged by one id at a time until they sum to
    total."""
    n = rng.integers(lo, hi + 1, size=batch).astype(np.int64)
    n[list(empty)] = 0
    live = np.setdiff1d(np.arange(batch), list(empty))
    while True:
        d = total - int(n.sum())
        if d == 0:
            return n
        k = rng.choice(live, size=min(abs(d), live.size), replace=False)
        ok = n[k] < hi if d > 0 else n[k] > lo
        n[k[ok]] += 1 if d > 0 else -1


def filled(rng, n, counts, spans, pool):
    """batch_with_multiplicities, then every position no item holds gets an id drawn from `pool` fill ids
    (FILL_BASE + 0..pool-1): fill ids repeat a few times each, so the items the case names stay the only hot ones while
    the distinct count stays near pool."""
    ids = batch_with_multiplicities(rng, n, counts, spans)
    free = ids >= np.uint64(len(counts))
    ids[free] = FILL_BASE + rng.integers(0, pool, size=int(free.sum())).astype(np.uint64)
    return ids


def window_straddle(k, count):
    """A span of exactly `count` occurrences across the boundary that starts window k: the item fills it whole."""
    lo = k * HOT_WIN - count // 2
    return lo, lo + count


# ---- 1. one summation slot at the context limit --------------------------------------------------------------------
SUM_B = 65535
SUM_N = CTX_LIMIT - 3  # within a few ids of the limit
SUM_EMPTY = (0, 40000)  # samples without ids
# (multiplicity, span of occurrences or None); constrained items first (batch_with_multiplicities places in order)
SUM_ITEMS = [
    (8193, window_straddle(1000, 8193)),         # one window of occurrences, across a boundary (two windows)
    (1025, ((SUM_N - 1) // HOT_WIN * HOT_WIN, SUM_N)),  # inside the last (short) window
    (257, window_straddle(7, 257)),
    (256, (2047 * HOT_WIN - 600, 2047 * HOT_WIN + 600)),  # across the boundary before the last window
    (33, window_straddle(5, 33)),                # the smallest hot item, across a boundary
    (32, window_straddle(3, 32)),                # the largest warm item, across a boundary
    (65537, (HOT_WIN * 100 - 40000, HOT_WIN * 100 + 40000)),  # dense over ten windows
    (4 * 1024 * 1024 + 1, None),                 # ~4 M: every window, the last one too
    (1024 * 1024 - 1, None),                     # ~1 M
    (1024, None), (2, None), (1, None),
]
SUM_POOL = 2_000_000  # distinct fill ids: ~5.8 occurrences each (cold and warm, never hot)


def summation_case(seed):
    """(ids u64 [SUM_N], row_off u32 [SUM_B + 1]); id k is item k of SUM_ITEMS."""
    rng = np.random.default_rng(seed)
    n = lengths_summing_to(rng, SUM_B, SUM_N, 128, 384, SUM_EMPTY)
    row_off = np.zeros(SUM_B + 1, np.uint32)
    row_off[1:] = np.cumsum(n)
    counts = [c for c, _ in SUM_ITEMS]
    spans = {k: sp for k, (_, sp) in enumerate(SUM_ITEMS) if sp is not None}
    return filled(rng, SUM_N, counts, spans, SUM_POOL), row_off


# ---- 2. the bitmap pool both ways -----------------------------------------------------------------------------------
POOL_B = 65535
POOL_N = 4_000_000
# a hot item wants ceil(POOL_N / 32) bitmap words, the pool holds max(4096, max_occurrences) = POOL_N: 32 of them fit
POOL_BITMAPS = max(4096, POOL_N) // ((POOL_N + 31) // 32)
POOL_ITEMS = [200_000, 50_000, 9000, 5000] + [40 + k for k in range(44)]  # 48 hot items: 16 go to occurrence lists
POOL_FILL = 1_000_000


def pool_case(seed):
    rng = np.random.default_rng(seed)
    n = lengths_summing_to(rng, POOL_B, POOL_N, 1, 121)
    row_off = np.zeros(POOL_B + 1, np.uint32)
    row_off[1:] = np.cumsum(n)
    return filled(rng, POOL_N, POOL_ITEMS, None, POOL_FILL), row_off


# ---- 2b. the pool's counter of words asked for, past 2^32 ------------------------------------------------------------
# Every hot item asks for its slot's bitmap words, also once the pool is used up: 36000 items of a 4 M slot ask for
# 36000 x 125000 = 4.5e9 words, more than a 32-bit counter holds.  All are of WRAP_MULT occurrences, so exactly
# POOL_BITMAPS of them get bitmaps and the occurrence lists hold the others' occurrences, a count the batch statistics
# show exactly.
WRAP_HOT, WRAP_MULT = 36_000, 40
WRAP_FILL = 1_000_000


def wrap_case(seed):
    """(ids u64 [POOL_N], row_off u32 [POOL_B + 1]); ids 0 .. WRAP_HOT - 1 occur WRAP_MULT times each."""
    rng = np.random.default_rng(seed)
    n = lengths_summing_to(rng, POOL_B, POOL_N, 1, 121)
    row_off = np.zeros(POOL_B + 1, np.uint32)
    row_off[1:] = np.cumsum(n)
    ids = FILL_BASE + rng.integers(0, WRAP_FILL, size=POOL_N).astype(np.uint64)
    ids[rng.permutation(POOL_N)[:WRAP_HOT * WRAP_MULT]] = np.repeat(np.arange(WRAP_HOT, dtype=np.uint64), WRAP_MULT)
    return ids, row_off


# ---- 2c. the work lists filled to their sizes -------------------------------------------------------------------------
# 128 slots of 65535 ragged samples, 2^24 occurrences in all, every occurrence in an item of one multiplicity (plus 16
# single ids where 2^24 does not divide): the warm list (n / 2 + 1 entries) holds 2^23 items of 2; the hot list
# (n / 33 entries below the giants') 508,400 items of 33; the giants' region (n / 1024 + 1 entries) 16,368 items of 1025.
CAP_S, CAP_B = 128, 65535
CAP_KINDS = {"pairs": 2, "hot33": 33, "giant": 1025}


def capacity_items(mult):
    """Items per slot (the slots' counts differ by at most one) and the single ids that fill the last slot."""
    total = CTX_LIMIT // mult
    q = np.full(CAP_S, total // CAP_S, np.int64)
    q[:total % CAP_S] += 1
    return q, CTX_LIMIT - total * mult


def capacity_case(kind, seed):
    """(ids u64 [2^24], row_off u32 [CAP_S * CAP_B + 1], slot_off [CAP_S + 1]); in every slot, ids 0 .. q - 1 occur
    CAP_KINDS[kind] times each, the last slot also holds the single ids FILL_BASE + 0, 1, ..."""
    rng = np.random.default_rng(seed)
    mult = CAP_KINDS[kind]
    q, extra = capacity_items(mult)
    parts, lens = [], []
    for s in range(CAP_S):
        x = np.repeat(np.arange(q[s], dtype=np.uint64), mult)
        if s == CAP_S - 1:
            x = np.concatenate([x, FILL_BASE + np.arange(extra, dtype=np.uint64)])
        parts.append(rng.permutation(x))
        lens.append(lengths_summing_to(rng, CAP_B, x.size, 1, 2 * x.size // CAP_B + 1))
    row_off = np.zeros(CAP_S * CAP_B + 1, np.uint32)
    row_off[1:] = np.cumsum(np.concatenate(lens))
    return np.concatenate(parts), row_off, [int(row_off[s * CAP_B]) for s in range(CAP_S + 1)]


# ---- 3. 128 slots x 65535 samples, one id each -----------------------------------------------------------------------
MANY_S, MANY_B = 128, 65535
MANY_CARD = 20_000


def many_slots_case(seed):
    """Zipf(1.1) ids per slot folded into MANY_CARD: the low ids of every slot are hot (thousands of occurrences)."""
    rng = np.random.default_rng(seed)
    ids = (rng.zipf(1.1, size=MANY_S * MANY_B) - 1) % MANY_CARD
    return ids.astype(np.uint64)


def many_slots_groups():
    """Feature groups: slots 0..7 one group, 60..67 another (across a slot-mask word), 120..127 a third, the rest alone."""
    return [0 if i < 8 else 1 if 60 <= i < 68 else 2 if i >= 120 else 3 + i for i in range(MANY_S)]


# ---- 4. U = N -------------------------------------------------------------------------------------------------------
UNIQUE_N = 16_000_000
UNIQUE_B = 65535


def unique_case(seed):
    """(ids u64 [UNIQUE_N], all distinct, row_off u32 [UNIQUE_B + 1]): ~244 ids per sample."""
    rng = np.random.default_rng(seed)
    lens = lengths_summing_to(rng, UNIQUE_B, UNIQUE_N, 1, 2 * UNIQUE_N // UNIQUE_B)
    row_off = np.zeros(UNIQUE_B + 1, np.uint32)
    row_off[1:] = np.cumsum(lens)
    return rng.permutation(UNIQUE_N).astype(np.uint64) * np.uint64(7919) + np.uint64(1 << 33), row_off


# ---- 5. raw slots past one spine trip -------------------------------------------------------------------------------
RAW_SIZES = [(1 << 20) - 1, 1 << 20, (1 << 20) + 1, (1 << 20) + 1025, CTX_LIMIT - 5]
RAW_FIXED = 3
RAW_B = 65535  # the most samples a batch holds


def scan_geometry(n):
    """(tiles, spine trips) of exclusive_scan over n values."""
    tiles = max(-(-n // SCAN_TILE), 1)
    return tiles, -(-tiles // SPINE_TRIP)


def raw_case(seed, n):
    """(ids u64 [n], row_off u32 [RAW_B + 1]): every tenth sample empty, the others of 1 .. 2 n / RAW_B ids (far longer
    than RAW_FIXED), the three marker ids at known positions, ids drawn from 0.7 n values."""
    rng = np.random.default_rng(seed)
    lens = lengths_summing_to(rng, RAW_B, n, 1, 2 * n // RAW_B, range(0, RAW_B, 10))
    row_off = np.zeros(RAW_B + 1, np.uint32)
    row_off[1:] = np.cumsum(lens)
    ids = rng.integers(0, max(int(n * 0.7), 1), size=n).astype(np.uint64)
    ids[[0, n // 2, n - 1]] = MARKERS
    return ids, row_off


# ---- 6. raw staging at persia_core's sizes --------------------------------------------------------------------------
STAGE_N = (1 << 23) - 7  # persia_core sizes the context at 2 x the ids: 2^24 - 14 occurrences
STAGE_B = 65535
STAGE_POOL = 4096


def stage_case(seed):
    rng = np.random.default_rng(seed)
    lens = lengths_summing_to(rng, STAGE_B, STAGE_N, 1, 2 * STAGE_N // STAGE_B)
    row_off = np.zeros(STAGE_B + 1, np.uint32)
    row_off[1:] = np.cumsum(lens)
    return rng.integers(0, STAGE_POOL, size=STAGE_N).astype(np.uint64), row_off
