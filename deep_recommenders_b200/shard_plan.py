"""Pure-Python partition arithmetic of the row-sharded embedding tables (SURVEY.md section 8e).

The reference is single-process; this is the multi-GPU design: all S tables of a model share one
global row space (row = slot_offset[s] + id), row r is owned by rank r mod G and stored at local
index r div G.  Shared by the CUDA path (sharded.py) and the gloo CPU protocol tests.
"""
from __future__ import annotations

from typing import List, NamedTuple, Sequence


def slot_offsets(rows: Sequence[int]) -> List[int]:
    out, o = [], 0
    for r in rows:
        out.append(o)
        o += int(r)
    return out


def owner(row: int, world: int) -> int:
    return row % world


def local_row(row: int, world: int) -> int:
    return row // world


def local_rows(total_rows: int, rank: int, world: int) -> int:
    """Number of global rows r in [0, total_rows) with r % world == rank."""
    return (total_rows - rank + world - 1) // world if total_rows > rank else 0


class P2PLayout(NamedTuple):
    max_rows: int      # rows allocated on every rank: local_rows(total, 0, world)
    vdim: int          # floats per row (the row stride)
    lin_in_row: bool   # first-order weight at float `dim` of the row (flags = DR_EMBED_LIN_IN_ROW)
    lin_offset: int    # floats from the shard base to the trailing first-order array (0: in the row)
    numel: int         # floats of the whole symmetric allocation


def p2p_layout(total_rows: int, dim: int, world: int) -> P2PLayout:
    """One rank's shard of the p2p exchange, the same size on every rank.  Narrow rows (dim + 1 <= 32) are
    [emb | w | pad] in ONE 128-B line; wide rows (dim = 32 ... 128) are exactly `dim` floats (whole lines, no
    padding), followed by the [max_rows] first-order weights rounded up to 4 floats."""
    max_rows = local_rows(total_rows, 0, world)
    if dim + 1 <= 32:
        return P2PLayout(max_rows, 32, True, 0, max_rows * 32)
    return P2PLayout(max_rows, dim, False, max_rows * dim, max_rows * dim + (max_rows + 3) // 4 * 4)


def capacity(n_lookups: int, world: int, slack: float = 0.04, floor: int = 4096) -> int:
    """Per-destination slots of the padded equal-split exchange: mean + slack, at least `floor`
    above the mean.  Owner = row mod G spreads even heavily repeated ids over the ranks unless ONE
    row dominates; uniform ids deviate by ~sqrt(n/G) (0.2 % at C2), so 4 % slack is ~20 sigma.
    The overflow flag catches skew (the caller re-plans with a larger slack)."""
    mean = (n_lookups + world - 1) // world
    return min(n_lookups, mean + max(floor, int(mean * slack))) if world > 1 else n_lookups


def own_first_order(rank: int, world: int) -> List[int]:
    """Block order of the all-gathered candidate embeddings seen by `rank` in the sharded two-tower step: its OWN
    block first (so the positive of local query i is candidate i and the in-batch-softmax kernel's eye(nq, nc)
    labels hold unchanged), the other ranks' blocks after it in rank order."""
    return [rank] + [r for r in range(world) if r != rank]


def inverse_order(order: Sequence[int]) -> List[int]:
    """inverse_order(o)[r] = position of block r in the order `o` (to bring gradients back to rank order)."""
    inv = [0] * len(order)
    for pos, r in enumerate(order):
        inv[r] = pos
    return inv
