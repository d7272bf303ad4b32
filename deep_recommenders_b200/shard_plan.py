"""Pure-Python partition arithmetic of the row-sharded embedding tables (SURVEY.md section 8e).

The reference is single-process; this is the multi-GPU design: all S tables of a model share one
global row space (row = slot_offset[s] + id), row r is owned by rank r mod G and stored at local
index r div G.  Shared by the CUDA path (sharded.py) and the gloo CPU protocol tests.
"""
from __future__ import annotations

from typing import List, Sequence


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
