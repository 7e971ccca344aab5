"""Keys crafted for the hash sets a batch goes through before anything reads a row (plain numpy, no torch).

Every step turns ids into signs (indices_add_prefix: `id % m + prefix` with m = 2^(64-b) - 1 for prefix bits b, no
change when the slot's prefix is 0) and signs into cells of one of these sets.  The homes restated here must follow the
kernels; a change to a set's layout changes them here too.

  batch scratch set   k_dedup (pb_dedup.cu) and its lookup again in k_link_items (find_in_slot, pb_shard.cu).  One region
                      per slot (set_region, pb_batch.cuh): slot s of n_s occurrences owns `size = 2 n_s + 1` cells from
                      `off = 2 occ_off[s] + 2 s`; the sign 2^64-1 (KEY_EMPTY) owns the reserved cell `off + size` that
                      sits between this region and the next.  Home: `off + umulhi(mix64(sign) >> 32, size)`; linear
                      probing wraps from `off + size - 1` to `off`.
  raw scratch set     k_raw_insert (pb_raw.cu).  `cells = next_pow2(max(1024, 2 max_occurrences))` (ensure_raw, pb_api_batch.cu:
                      the context's max_occurrences); home `mix64(sign) & (cells - 1)`, wrapping to 0; the sign 2^64-1 owns
                      the extra cell `cells`.
  incremental set     inc_find / inc_claim (pb_inc.cu).  `n_cells = next_pow2(max(1024, 2 capacity))`
                      (pb_table_enable_incremental, pb_api.cu), buckets of 8 cells; a sign's path starts at the first cell
                      of bucket `mix64(sign) & (n_cells / 8 - 1)` and wraps from cell n_cells - 1 to cell 0.

`homed_ids` returns raw ids whose prefixed signs are distinct and all land on one chosen home, so that a test can build a
cluster at a region's or a set's last cell and make its probes wrap."""
import numpy as np

M64 = (1 << 64) - 1
KEY_EMPTY = M64
BUCKET = 8


def mix64(k):
    """pb_common.cuh mix64 (MurmurHash3's fmix64), on uint64 numpy arrays (multiplication wraps)."""
    k = np.asarray(k, np.uint64).copy()
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xFF51AFD7ED558CCD)
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xC4CEB9FE1A85EC53)
        k ^= k >> np.uint64(33)
    return k


# ---- indices_add_prefix ---------------------------------------------------------------------------------------------
def spacing(b):
    """feature_spacing: m = 2^(64-b) - 1 (2^64 - 1 without prefix bits)."""
    return (1 << (64 - b)) - 1 if b else M64


def prefix_int(x, b, p):
    """One id's sign, in Python ints: `x % m + p`, or x itself when the slot's prefix p is 0."""
    return int(x) % spacing(b) + int(p) if p else int(x)


def prefix_np(ids, b, p):
    """prefix_int over a uint64 array."""
    ids = np.asarray(ids, np.uint64)
    if not p:
        return ids.copy()
    with np.errstate(over="ignore"):
        return ids % np.uint64(spacing(b)) + np.uint64(p)


PREFIX_BITS = (1, 2, 7, 8, 12, 31, 32, 33, 56, 62, 63)


def edge_ids(b, rng, n_random=8):
    """Ids at the edges of the residue mod m: 0, 1, m-1, m (residue m, which is 0), m+1, 2m, 3m and the largest
    multiple of m, 2^63, 2^64-1 and random ones (uint64, distinct)."""
    m = spacing(b)
    ids = {0, 1, m - 1, m, m + 1, 2 * m, 3 * m, (M64 // m) * m, 1 << 63, M64}
    ids.update(int(x) for x in rng.integers(0, 1 << 63, size=n_random, dtype=np.uint64) * 2 + 1)
    return np.array(sorted(x for x in ids if x <= M64), np.uint64)


def residues(ids, b, p):
    """Each id replaced by its residue mod m (ids unchanged without a prefix): the canonical id of its sign."""
    ids = np.asarray(ids, np.uint64)
    return ids % np.uint64(spacing(b)) if p else ids.copy()


# ---- the sets -------------------------------------------------------------------------------------------------------
def next_pow2(x):
    return 1 << (int(x) - 1).bit_length()


def set_region(slot_occ_off, slot):
    """(off, size) of a slot's region of the batch scratch set; the reserved cell is off + size."""
    n = int(slot_occ_off[slot + 1]) - int(slot_occ_off[slot])
    return 2 * int(slot_occ_off[slot]) + 2 * slot, 2 * n + 1


def dedup_home(signs, off, size):
    """k_dedup's first cell: off + umulhi(mix64(sign) >> 32, size)."""
    h = mix64(signs) >> np.uint64(32)
    return np.uint64(off) + ((h * np.uint64(size)) >> np.uint64(32))


def raw_cells(max_occurrences):
    return next_pow2(max(1024, 2 * int(max_occurrences)))


def raw_home(signs, cells):
    return mix64(signs) & np.uint64(cells - 1)


def inc_cells(capacity):
    return next_pow2(max(1024, 2 * int(capacity)))


def inc_bucket(signs, n_cells):
    """The bucket a sign's path starts in (its first cell is bucket * 8)."""
    return mix64(signs) & np.uint64(n_cells // BUCKET - 1)


def probe_cells(homes, off, size):
    """Linear probing of distinct signs inserted in the order given, in a region [off, off + size) that wraps: the cell
    each one takes."""
    used, out = set(), []
    for h in homes:
        c = int(h)
        while c in used:
            c = off if c + 1 == off + size else c + 1
        used.add(c)
        out.append(c)
    return out


def homed_ids(home_fn, target, count, b=0, p=0, start=1 << 32, avoid=()):
    """`count` raw ids, ascending from `start`, whose prefixed signs are distinct, not in `avoid` and have
    home_fn(signs) == target."""
    out, seen, base = [], set(int(s) for s in avoid), int(start)
    chunk = 1 << 20
    for _ in range(64):
        if len(out) == count:
            break
        assert base + chunk <= M64, "ran out of candidates"
        c = np.arange(base, base + chunk, dtype=np.uint64)
        s = prefix_np(c, b, p)
        for i in np.flatnonzero(home_fn(s) == np.uint64(target)):
            if int(s[i]) not in seen:
                seen.add(int(s[i]))
                out.append(int(c[i]))
                if len(out) == count:
                    break
        base += chunk
    assert len(out) == count, "too few distinct signs land on the target"
    return np.array(out, np.uint64)
