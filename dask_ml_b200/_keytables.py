"""The per-column key tables of SimpleImputer's mode and of the encoders' categories (DESIGN.md, "Per-column key
tables"; the passes in csrc/bkm_keys.cu): their capacities, their allocation and their merge over ranks.

A group of g columns owns the tables ``keys`` / ``counts`` (uint64 held as int64, (total,)) on the device; column j owns
slots [off[j], off[j + 1]), a power of two or 0.  A table's content is a set of keys with integer counts, so whatever is
read from it does not depend on the slot layout.
"""
import numpy as np
import torch

# bits of the keys of each element type: a table never needs more than 2^bits entries
KEY_BITS = {torch.bfloat16: 16, torch.float32: 32, torch.float64: 64, torch.int32: 32, torch.int64: 64,
            torch.uint8: 8, torch.bool: 1}


def capacity(m, tdt):
    """The capacity of a table that receives ``m`` values of torch dtype ``tdt``: a power of two >= twice the distinct
    values it can hold (at most 2^KEY_BITS[tdt]), so that it never fills; 0 for m <= 0."""
    m = min(int(m), 1 << KEY_BITS[tdt])
    return 0 if m <= 0 else 1 << (2 * m - 1).bit_length()


def alloc(be, caps):
    """(keys, counts, off, total): uninitialised tables of capacities ``caps`` on ``be``'s device, ``off`` int64
    (g + 1,) on the device and ``total`` the sum of the capacities."""
    off = np.concatenate([[0], np.cumsum(caps)]).astype(np.int64)
    total = int(off[-1])
    keys = be.empty((max(total, 1),), torch.int64)
    counts = be.empty((max(total, 1),), torch.int64)
    return keys, counts, torch.as_tensor(off).to(be.device), total


def merge_ranks(be, comm, tables, g, tdt, distinct, flags=None):
    """Every rank's tables of the same g columns united into new tables, identical on every rank: each key with the sum
    of its counts over the ranks.  ``tables`` is ``alloc``'s tuple, ``distinct`` this rank's occupied slots per column
    (device tensor or numpy) and ``flags`` (g,) bool numpy or None: per-column flags or-ed over the ranks in the same
    all-reduce as the lengths.  Returns (merged tables, mode_best of them, the or-ed flags or None).

    The only collective is the sum all-reduce: every rank writes its lengths (and flags) into its own row of a zeroed
    [R][g] buffer and its compacted entries {column, key >> 32, key & 0xffffffff, count} into its own slice of a zeroed
    [sum of lengths][4] float64 buffer, whose sum is an exact all-gather (integers below 2^53)."""
    keys, counts, off, total = tables
    lens = be.zeros((comm.world, g if flags is None else 2 * g), torch.float64)
    lens[comm.rank, :g] = torch.as_tensor(distinct, dtype=torch.float64)
    if flags is not None:
        lens[comm.rank, g:] = torch.as_tensor(flags, dtype=torch.float64)
    comm.allreduce_sum_(lens.view(-1))
    L = lens.cpu().numpy()
    per_rank = L[:, :g].sum(1).astype(np.int64)
    start, E = int(per_rank[: comm.rank].sum()), int(per_rank.sum())
    entries = be.zeros((max(E, 1), 4), torch.float64)
    if per_rank[comm.rank] > 0:
        be.mode_compact(keys, counts, off, g, entries[start: start + int(per_rank[comm.rank])])
    comm.allreduce_sum_(entries.view(-1))
    keys, counts, off, total = alloc(be, [capacity(m, tdt) for m in L[:, :g].sum(0)])
    be.mode_merge(entries[:E], keys, counts, off, g, total)
    best = be.mode_best(keys, counts, off, g, total)
    return (keys, counts, off, total), best, None if flags is None else L[:, g:].sum(0) > 0
