"""`.emb` list images laid out as the reference's writer can leave them (persia_b200/checkpoint.py's docstring): nodes
in any order, free nodes (flag 0, on the free list) and entries of several lengths in one list.  The reference's
ArrayLinkedList relinks nodes on every get_refresh and reuses freed slots, so its files list entries in an order
unrelated to node order."""
import numpy as np


def reference_layout(signs, dims, entries, rng, permute=True, free=0):
    """The list image of `signs` / `dims` / `entries` (list order; entries: float32 arrays of any lengths) over
    len(signs) + free nodes: the live ones at a random (permute) or in-order placement, the free ones interleaved and
    chained from the header's free index."""
    n = len(signs)
    m = n + int(free)
    place = rng.permutation(m) if permute else np.arange(m)
    live, unused = place[:n], place[n:]
    if not permute:  # free nodes spread through the live ones, the live ones still in list order
        slots = np.sort(rng.choice(m, size=n, replace=False)) if m else np.zeros(0, np.int64)
        live, unused = slots, np.setdiff1d(np.arange(m), slots)
    nodes = [None] * m
    for k in range(n):
        nxt = int(live[k + 1]) + 1 if k + 1 < n else 0
        prv = int(live[k - 1]) + 1 if k else 0
        e = np.ascontiguousarray(entries[k], dtype="<f4")
        nodes[live[k]] = (np.array([nxt, prv], "<u4").tobytes() + b"\x01" + np.array([e.size], "<u4").tobytes() +
                          e.tobytes() + np.array([dims[k], signs[k]], "<u8").tobytes())
    for k, i in enumerate(unused):
        nxt = int(unused[k + 1]) + 1 if k + 1 < len(unused) else 0
        nodes[i] = np.array([nxt, 0], "<u4").tobytes() + b"\x00"
    head = np.array([n], "<u8").tobytes() + np.array(
        [int(live[0]) + 1 if n else 0, int(live[-1]) + 1 if n else 0, int(unused[0]) + 1 if len(unused) else 0, m, m],
        "<u4").tobytes()
    return head + b"".join(nodes)
