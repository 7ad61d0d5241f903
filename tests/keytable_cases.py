"""Keys built to land where a test wants them in the per-column key tables (csrc/bkm_keys.cu), and a slot-exact numpy
restatement of the tables' distinct and count passes.

A key's home slot in a table of capacity ``cap`` (a power of two) is ``mix64(key) & (cap - 1)``; its slot in the
distinct pass's per-CTA cache is ``(mix64(key) >> 40) & (FS - 1)`` with FS = 4096 / CS slots per column and CS the
columns of one 32-byte sector.  ``mix64`` is a bijection of 64-bit words, so 64-bit keys with any hash are found by
inverting it; 32-bit keys are found by scanning a fixed range of candidates; 16-, 8- and 1-bit keys have key spaces
smaller than a probe chain and are tested whole instead.  Values come from keys through ``_encode.key_values`` and are
kept only when ``_encode.host_keys`` gives the key back (no NaN patterns but the canonical one, no -0.0)."""
import functools

import numpy as np
import torch

from dask_ml_b200.preprocessing import _encode

EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)          # the tables' empty slot
MAX_PROBE = 1024                               # the distinct pass's probe bound
FILTER_SLOTS = 4096                            # the distinct pass's per-CTA cache, shared by a sector's columns

DTYPES = {"f64": torch.float64, "i64": torch.int64, "f32": torch.float32, "i32": torch.int32,
          "bf16": torch.bfloat16, "u8": torch.uint8, "bool": torch.bool}
HOST = {torch.float64: np.float64, torch.int64: np.int64, torch.float32: np.float32, torch.int32: np.int32,
        torch.bfloat16: np.float32, torch.uint8: np.uint8, torch.bool: np.bool_}

_M1, _M2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53
_M1_INV, _M2_INV = pow(_M1, -1, 1 << 64), pow(_M2, -1, 1 << 64)
_S = np.uint64(33)


def mix64(k):
    """The tables' slot hash of uint64 keys (bkm_select.cuh)."""
    k = np.array(k, dtype=np.uint64, ndmin=1)
    k = k ^ (k >> _S)
    k = k * np.uint64(_M1)
    k = k ^ (k >> _S)
    k = k * np.uint64(_M2)
    return k ^ (k >> _S)


def unmix64(h):
    """The inverse of ``mix64``: x ^= x >> 33 is its own inverse (33 >= 32), a product by an odd constant is undone
    by its inverse modulo 2^64."""
    h = np.array(h, dtype=np.uint64, ndmin=1)
    h = h ^ (h >> _S)
    h = h * np.uint64(_M2_INV)
    h = h ^ (h >> _S)
    h = h * np.uint64(_M1_INV)
    return h ^ (h >> _S)


def home_slot(keys, cap):
    return (mix64(keys) & np.uint64(cap - 1)).astype(np.int64)


def cache_slot(keys, tdt):
    fs = FILTER_SLOTS // (32 // torch.empty(0, dtype=tdt).element_size())
    return ((mix64(keys) >> np.uint64(40)) & np.uint64(fs - 1)).astype(np.int64)


def key_bits(tdt):
    return {torch.float64: 64, torch.int64: 64, torch.float32: 32, torch.int32: 32}[tdt]


def values(keys, tdt):
    """The host values (``HOST[tdt]``) of ``keys``, all of which must round-trip."""
    keys = np.asarray(keys, dtype=np.uint64)
    v = _encode.key_values(keys, tdt, HOST[tdt])
    assert (_encode.host_keys(v, tdt) == keys).all()
    return v


def round_trips(keys, tdt):
    """Mask of the keys that stand for a value whose key is the same key, the empty marker excluded."""
    keys = np.asarray(keys, dtype=np.uint64)
    with np.errstate(invalid="ignore"):
        v = _encode.key_values(keys, tdt, HOST[tdt])
        return (_encode.host_keys(v, tdt) == keys) & (keys != EMPTY)


def device(v, tdt):
    """A CUDA tensor of dtype ``tdt`` holding the host values ``v`` (a column when 1-D)."""
    t = torch.from_numpy(np.ascontiguousarray(v)).to(tdt)
    return (t.reshape(-1, 1) if t.ndim == 1 else t).cuda()


# ------------------------------------------------ 32-bit candidates ------------------------------------------------
_BASE32 = 0x90000000          # keys of positive normal float32 values and of int32 values 0x10000000..: all round-trip


@functools.lru_cache(maxsize=None)
def _pool32(log2n):
    """(keys, mix64 of the keys) of 2^log2n consecutive 32-bit keys from _BASE32."""
    k = np.arange(_BASE32, _BASE32 + (1 << log2n), dtype=np.uint64)
    return k, mix64(k)


@functools.lru_cache(maxsize=None)
def _by_home32(cap):
    """(home slots, keys) of the 2^24 candidates, sorted by home slot in a table of capacity ``cap``."""
    k, h = _pool32(24)
    hs = (h & np.uint64(cap - 1)).astype(np.int64)
    order = np.argsort(hs, kind="stable")
    return hs[order], k[order]


@functools.lru_cache(maxsize=None)
def shared_low_bits32(bits, log2n=27, step=1 << 24):
    """The 32-bit keys among 2^log2n candidates whose hashes agree in their low ``bits`` bits with those of the most
    keys: about 2^(log2n - bits) of them (more than 1024 for bits = 17)."""
    mask = np.uint64((1 << bits) - 1)
    hist = np.zeros(1 << bits, dtype=np.int64)
    for s in range(0, 1 << log2n, step):
        k = np.arange(_BASE32 + s, _BASE32 + s + step, dtype=np.uint64)
        hist += np.bincount((mix64(k) & mask).astype(np.int64), minlength=1 << bits)
    want = np.uint64(int(hist.argmax()))
    out = []
    for s in range(0, 1 << log2n, step):
        k = np.arange(_BASE32 + s, _BASE32 + s + step, dtype=np.uint64)
        out.append(k[(mix64(k) & mask) == want])
    return np.concatenate(out)


# ------------------------------------------------ constructors ------------------------------------------------
def shared_low(tdt, bits, m, low=0, seed=0):
    """m distinct keys of a 64-bit dtype whose hashes all end in the ``bits``-bit pattern ``low`` (2 <= bits <= 62):
    mix64 inverted on random high bits above ``low``."""
    assert key_bits(tdt) == 64 and 2 <= bits <= 62
    rng = np.random.RandomState(seed)
    out = np.zeros(0, dtype=np.uint64)
    while len(out) < m:
        hi = rng.randint(0, 1 << 62, 2 * m + 16, dtype=np.int64).astype(np.uint64) << np.uint64(bits)
        k = unmix64(hi | np.uint64(low))
        out = np.unique(np.concatenate([out, k[round_trips(k, tdt)]]))
    return rng.permutation(out)[:m]


def home_keys(tdt, cap, slot, m, seed=0):
    """m distinct keys of ``tdt`` (64- or 32-bit) whose home slot in a table of capacity ``cap`` is ``slot``."""
    if key_bits(tdt) == 64:
        b = cap.bit_length() - 1
        k = shared_low(tdt, b, m, low=slot, seed=seed)
    else:
        k, h = _pool32(24)
        k = k[(h & np.uint64(cap - 1)) == np.uint64(slot)]
        assert len(k) >= m, (len(k), m)
        k = np.random.RandomState(seed).permutation(k)[:m]
    assert (home_slot(k, cap) == slot).all()
    return k


def home(dtype, cap, slot, m, seed=0):
    """m distinct values of ``dtype`` (a key of DTYPES) whose home slot in a table of capacity ``cap`` is ``slot``."""
    tdt = DTYPES[dtype]
    return values(home_keys(tdt, cap, slot, m, seed), tdt)


def placed_keys(tdt, cap, slots, seed=0):
    """One key per entry of ``slots`` with that home slot in a table of capacity ``cap``, all distinct."""
    slots = np.asarray(slots, dtype=np.int64)
    if key_bits(tdt) == 64:
        b = cap.bit_length() - 1
        rng = np.random.RandomState(seed)
        out = []
        for s in slots:
            while True:
                k = unmix64((np.uint64(rng.randint(1, 1 << 62)) << np.uint64(b)) | np.uint64(s))
                if round_trips(k, tdt)[0] and k[0] not in out:
                    out.append(k[0])
                    break
        k = np.array(out, dtype=np.uint64)
    else:
        hs, pk = _by_home32(cap)
        lo, hi = np.searchsorted(hs, slots), np.searchsorted(hs, slots, side="right")
        assert len(np.unique(slots)) == len(slots) and (hi > lo).all(), "no candidate for a slot"
        k = pk[lo + np.random.RandomState(seed).randint(0, 1 << 30, len(slots)) % (hi - lo)]
    assert (home_slot(k, cap) == slots).all()
    return k


def placed(dtype, cap, slots, seed=0):
    tdt = DTYPES[dtype]
    return values(placed_keys(tdt, cap, slots, seed), tdt)


def cache_mates_keys(tdt, cap, m, cslot=5, seed=0):
    """m distinct keys that share the distinct pass's cache slot ``cslot`` and have m different home slots in a
    table of capacity ``cap``."""
    fs = FILTER_SLOTS // (32 // torch.empty(0, dtype=tdt).element_size())
    if key_bits(tdt) == 64:
        fb = fs.bit_length() - 1
        rng = np.random.RandomState(seed)
        low = rng.permutation(cap)[: 2 * m].astype(np.uint64)
        mid = rng.randint(0, 1 << 28, 2 * m).astype(np.uint64) << np.uint64(12)
        hi = rng.randint(0, 1 << (24 - fb), 2 * m).astype(np.uint64) << np.uint64(40 + fb)
        k = unmix64(hi | (np.uint64(cslot) << np.uint64(40)) | mid | low)
        k = k[round_trips(k, tdt)][:m]
    else:
        pk, ph = _pool32(24)
        sel = ((ph >> np.uint64(40)) & np.uint64(fs - 1)) == np.uint64(cslot)
        k, h = pk[sel], (ph[sel] & np.uint64(cap - 1))
        _, first = np.unique(h, return_index=True)
        k = np.random.RandomState(seed).permutation(k[first])[:m]
        assert len(k) == m
    assert (cache_slot(k, tdt) == cslot).all() and len(np.unique(home_slot(k, cap))) == m
    return k


def cache_mates(dtype, cap, m, cslot=5, seed=0):
    tdt = DTYPES[dtype]
    return values(cache_mates_keys(tdt, cap, m, cslot, seed), tdt)


# ------------------------------------------------ the restatement ------------------------------------------------
class Table:
    """One column's table as the distinct pass (``count=False``) or the count pass (``count=True``) leaves it, with
    keys inserted one at a time: home slot ``mix64 & (cap - 1)``, linear probing with wrap-around, at most ``bound``
    slots examined per key (the distinct pass: min(cap, 1024), or cap with a full probe; the count pass: cap).  The
    distinct pass flags OVERFLOW when a probe fails or the occupancy passes half the capacity, and its column then
    takes no more keys; the key ~0 (INT64_MAX's) only sets MARKER.  Slots are held in a dict, so a table of any
    capacity costs memory only for its keys.

    Without deletions the set of occupied slots under linear probing does not depend on the insertion order as long as
    no insert fails, so whenever no flag is raised ``arrays()`` is what the kernels must leave, bit for bit."""

    def __init__(self, cap, count=False):
        self.cap, self.count = cap, count
        self.slots, self.counts = {}, {}
        self.overflow, self.marker = False, False

    @property
    def occ(self):
        return len(self.slots)

    def insert(self, keys, mult=None, full_probe=False):
        keys = np.asarray(keys, dtype=np.uint64)
        bound = self.cap if (self.count or full_probe) else min(self.cap, MAX_PROBE)
        homes = home_slot(keys, self.cap).tolist() if len(keys) else []
        mask, slots, empty = self.cap - 1, self.slots, int(EMPTY)
        for i, (k, h) in enumerate(zip(keys.tolist(), homes)):
            if self.overflow and not self.count:
                break
            if k == empty and not self.count:
                self.marker = True
                continue
            c = 1 if mult is None else int(mult[i])
            for _ in range(bound):
                cur = slots.get(h)
                if cur == k:
                    if self.count:
                        self.counts[h] += c
                    break
                if cur is None:
                    slots[h], self.counts[h] = k, c if self.count else 1
                    if not self.count and 2 * len(slots) > self.cap:
                        self.overflow = True
                    break
                h = (h + 1) & mask
            else:
                self.overflow = True
        return self

    def arrays(self):
        """(keys uint64 (cap,) with EMPTY in free slots, counts uint64 (cap,))."""
        k = np.full(self.cap, EMPTY, dtype=np.uint64)
        c = np.zeros(self.cap, dtype=np.uint64)
        if self.slots:
            idx = np.fromiter(self.slots.keys(), dtype=np.int64, count=len(self.slots))
            k[idx] = np.fromiter(self.slots.values(), dtype=np.uint64, count=len(self.slots))
            c[idx] = np.array([self.counts[i] for i in idx.tolist()], dtype=np.uint64)
        return k, c

    def occupied(self):
        return self.arrays()[0] != EMPTY


def first_seen(keys):
    """The distinct entries of ``keys`` in the order of their first occurrence."""
    u, i = np.unique(np.asarray(keys, dtype=np.uint64), return_index=True)
    return u[np.argsort(i)]
