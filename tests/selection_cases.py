"""Adversarial columns for the exact order-statistic passes (the radix selections of QuantileTransformer, RobustScaler
and SimpleImputer's median, and the key-table mode of SimpleImputer's most_frequent), in plain numpy.

Every case is named and seeded and aims at one mechanism of the selection (DESIGN.md, "The passes of
QuantileTransformer"): how many live prefixes a round carries, where the ranks fall in a bin's cumulative counts, the
sign of zero, the ends of the key range.  Columns are built as raw bit patterns of the dtype, so that bf16 columns hold
exactly the keys they are meant to hold.  ``plan()`` lists the (case, dtype, width, n_q, missing) runs of the selection
that the CPU coverage test and the GPU round-by-round replay share."""
import numpy as np
import torch

DTYPES = ("f32", "f64", "bf16")
BITS = {"f32": 32, "f64": 64, "bf16": 16}
EXP = {"f32": 8, "f64": 11, "bf16": 8}
UINT = {"f32": np.uint32, "f64": np.uint64, "bf16": np.uint16}
TORCH = {"f32": torch.float32, "f64": torch.float64, "bf16": torch.bfloat16}
ONE = {"f32": 0x3F800000, "f64": 0x3FF0000000000000, "bf16": 0x3F80}         # the bits of 1.0

SELECT_CASES = ("full_range", "one_prefix", "carry", "zero_carry", "boundary", "specials", "masked", "masked_zero")
MODE_CASES = ("mode_ties", "mode_many")
SPECIAL_KINDS = ("zeros", "inf_ends", "some_nan", "all_nan", "one_valid", "nq_minus_1", "nq", "nq_plus_1")


def sector(dt):
    """CS: the columns of one 32-byte sector of a row, the hist kernels' column group."""
    return 32 // (BITS[dt] // 8)


def widths(dt):
    c = sector(dt)
    return (1, c - 1, c, c + 1, 3 * c + 1)


def references(nq):
    """QuantileTransformer's references_ for n_q quantiles: the qf of the selection."""
    return np.linspace(0, 1, nq, endpoint=True)


def target_ranks(m, qf):
    """The distinct floor / floor + 1 ranks of numpy's 'linear' virtual index (m - 1) qf among m values."""
    vi = (m - 1.0) * np.asarray(qf, dtype=np.float64)
    lo, hi = np.floor(vi), np.floor(vi) + 1.0
    lo, hi = np.where(vi >= m - 1.0, m - 1.0, lo), np.where(vi >= m - 1.0, m - 1.0, hi)
    return np.unique(np.maximum(np.concatenate([lo, hi]), 0.0)).astype(np.int64) if m > 0 else np.zeros(1, np.int64)


# ------------------------------------------------ bits, keys, values ------------------------------------------------
def _u(dt, v):
    return np.asarray(v).astype(UINT[dt])


def key_of(dt, bits):
    """The order-preserving radix key of each bit pattern (bkm_select.cuh, radix_key), as uint64."""
    b = np.asarray(bits).astype(np.uint64)
    sign = np.uint64(1) << np.uint64(BITS[dt] - 1)
    mask = np.uint64(0xFFFFFFFFFFFFFFFF) if BITS[dt] == 64 else np.uint64((1 << BITS[dt]) - 1)
    return np.where(b & sign, ~b & mask, b | sign)


def bits_of_key(dt, keys):
    k = np.asarray(keys).astype(np.uint64)
    sign = np.uint64(1) << np.uint64(BITS[dt] - 1)
    mask = np.uint64(0xFFFFFFFFFFFFFFFF) if BITS[dt] == 64 else np.uint64((1 << BITS[dt]) - 1)
    return _u(dt, np.where(k & sign, k ^ sign, ~k & mask))


def bits_of_values(dt, v):
    """Bit patterns of float values that the dtype holds exactly."""
    if dt == "f64":
        return np.asarray(v, dtype=np.float64).view(np.uint64)
    u = np.asarray(v, dtype=np.float32).view(np.uint32)
    return u if dt == "f32" else _u(dt, u >> np.uint32(16))


def _finite_bits(dt, sign, exp, mant):
    m = BITS[dt] - 1 - EXP[dt]
    return _u(dt, (np.asarray(sign, np.uint64) << np.uint64(BITS[dt] - 1)) | (np.asarray(exp, np.uint64) << np.uint64(m))
              | np.asarray(mant, np.uint64))


def _mantissa(dt, rng, n):
    m = BITS[dt] - 1 - EXP[dt]
    return rng.randint(0, 1 << 31, size=n).astype(np.uint64) * np.uint64(1 << 21) + \
        rng.randint(0, 1 << 21, size=n).astype(np.uint64) & np.uint64((1 << m) - 1)


class Case(object):
    """One adversarial matrix: ``bits`` (n, d) of the dtype's unsigned type and the missing value of the masked pass
    (None: NaN only)."""

    def __init__(self, name, dt, bits, missing=None):
        self.name, self.dt, self.bits, self.missing = name, dt, np.ascontiguousarray(bits), missing

    def __repr__(self):
        return "%s-%s-d%d" % (self.name, self.dt, self.bits.shape[1])

    @property
    def n(self):
        return self.bits.shape[0]

    @property
    def d(self):
        return self.bits.shape[1]

    def tensor(self):
        """The rows as a CPU tensor of the case's dtype."""
        if self.dt == "bf16":
            return torch.from_numpy(self.bits.view(np.int16).copy()).view(torch.bfloat16)
        return torch.from_numpy(self.bits.view(np.float32 if self.dt == "f32" else np.float64).copy())

    def values(self):
        """The rows as numpy of the host dtype (float32 for bf16 rows, exact)."""
        if self.dt == "bf16":
            return (self.bits.astype(np.uint32) << np.uint32(16)).view(np.float32)
        return self.bits.view(np.float32 if self.dt == "f32" else np.float64).copy()

    def valid(self):
        v = self.values()
        ok = ~np.isnan(v)
        return ok & (v != self.missing) if self.missing is not None else ok


# ------------------------------------------------ columns ------------------------------------------------
def _full_range(dt, rng, n):
    """Random sign, exponent uniform over every finite binade (subnormals and the largest included), random mantissa:
    round 0 fills every one of the 256 bins."""
    return _finite_bits(dt, rng.randint(0, 2, n), rng.randint(0, (1 << EXP[dt]) - 1, n), _mantissa(dt, rng, n))


def _one_prefix(dt, rng, n):
    """Equal in every byte but the last: one live prefix up to the last round."""
    base = int(_finite_bits(dt, rng.randint(0, 2), rng.randint(1, (1 << EXP[dt]) - 2), _mantissa(dt, rng, 1))[0])
    return _u(dt, np.uint64(base & ~0xFF) | rng.randint(0, 256, n).astype(np.uint64))


def _carry(dt, rng, n, negative):
    """512 consecutive bit patterns about 1.0 (or -1.0): 0x3F7FFF00 ... 0x3F8000FF as f32, whose keys differ from
    the top byte down on the two sides of 1.0, so neighbouring ranks have different prefixes in every round."""
    b = _u(dt, ONE[dt] - 256 + rng.randint(0, 512, n))
    return b | _u(dt, 1 << (BITS[dt] - 1)) if negative else b


def _zero_carry(dt, rng, n):
    """+-(0 ... 255 units of the last place): subnormals and both zeros, whose keys straddle 0x7F..F / 0x80..0, a
    carry through every byte of the key."""
    return _finite_bits(dt, rng.randint(0, 2, n), np.zeros(n, np.int64), rng.randint(0, 256, n))


def _boundary(dt, rng, n, nq):
    """Runs of repeated values whose ends sit on the target ranks: for every target rank r of n_q quantiles (and of the
    median) the sorted column changes value just before r, just before r + 1, or both, so a rank equals a bin's
    exclusive or inclusive count in the round where the neighbouring values part.  Consecutive distinct values differ
    in a random byte, so the parting happens in every round."""
    cuts = set()
    for r in np.concatenate([target_ranks(n, references(nq)), target_ranks(n, [0.5])]):
        pick = rng.randint(0, 3)
        for p in ((r,), (r + 1,), (r, r + 1))[pick]:
            if 0 < p < n:
                cuts.add(int(p))
    pos = np.zeros(n, np.int64)
    pos[sorted(cuts)] = 1
    which = np.cumsum(pos)                                  # the distinct value of each sorted position
    D = int(which[-1]) + 1
    nb = BITS[dt] // 8
    top_p = min(1.0 / nb, 40.0 / D)
    p = np.full(nb, (1.0 - top_p) / (nb - 1))
    p[-1] = top_p
    byte = rng.choice(nb, size=D - 1, p=p)
    step = (np.uint64(1) << (np.uint64(8) * byte.astype(np.uint64))) * rng.randint(1, 3, D - 1).astype(np.uint64)
    k0 = key_of(dt, bits_of_values(dt, [-1000.0]))[0]
    keys = np.concatenate([[k0], k0 + np.cumsum(step)])
    col = bits_of_key(dt, keys[which])
    return col[rng.permutation(n)]


def _special(dt, rng, n, nq, kind):
    nan = bits_of_values(dt, [np.nan])[0]
    col = bits_of_values(dt, np.round(rng.standard_normal(n) * 4, 1))
    if kind == "zeros":                                      # -0.0 and +0.0 at every target rank
        col = bits_of_values(dt, rng.choice([-0.0, 0.0, -0.0, 0.0, -0.0, 0.0, 1.0, -1.5, 1e-30], n))
    elif kind == "inf_ends":
        col[rng.permutation(n)[: n // 10]] = bits_of_values(dt, [np.inf])[0]
        col[rng.permutation(n)[: n // 10]] = bits_of_values(dt, [-np.inf])[0]
    elif kind == "some_nan":
        col[rng.permutation(n)[: n // 7]] = nan
    elif kind == "all_nan":
        col[:] = nan
    else:
        keep = {"one_valid": 1, "nq_minus_1": nq - 1, "nq": nq, "nq_plus_1": nq + 1}[kind]
        col[rng.permutation(n)[keep:]] = nan
    return col


def _masked(dt, rng, n, zero):
    """Missing 2.0 at the column's median rank (removing it moves the median), or missing 0.0 among -0.0 / +0.0
    (both are missing).  No NaN: scikit-learn refuses NaN next to a numeric missing value (the plan runs the masked
    pass on the NaN-holding special columns too)."""
    k = rng.randint(n // 20, n // 3)
    below = rng.choice([-3.0, -1.0, 0.0, -0.0, 1.0] if zero else [-3.0, -1.0, 0.0, 1.0], (n - k) // 2)
    above = rng.choice([3.0, 5.0, 7.0], n - k - len(below))
    mid = rng.choice([0.0, -0.0], k) if zero else np.full(k, 2.0)
    return bits_of_values(dt, rng.permutation(np.concatenate([below, mid, above])))


def _mode(dt, rng, n, many):
    """Several values tied at the largest count (scikit-learn takes the smallest), -0.0 and +0.0 counted together, NaN
    (missing) among the rows; ``many``: mostly distinct values, so the tables grow, with a few small tied repeats."""
    if many:
        v = rng.standard_normal(n) * 1e3
        v = np.round(v, 3)
        for t in range(3):                                   # three values repeated 4 times: the tie at the top
            v[rng.permutation(n)[:4]] = rng.choice([-7.5, 2.25, 11.0, 0.5]) + t
        v[rng.permutation(n)[:2]] = -0.0
        v[rng.permutation(n)[:2]] = 0.0
    else:
        tied = rng.choice([-4.0, -2.5, 1.0, 3.0, 6.0], rng.randint(2, 5), replace=False)
        c = n // 12
        parts = [np.full(c, t) for t in tied]
        nz = rng.randint(0, c + 1)
        parts.append(np.concatenate([np.full(nz, -0.0), np.zeros(c - nz)]))          # zero ties too
        rest = n - c * len(parts)
        parts.append(rng.choice([-9.0, -1.0, 2.0, 8.0, 10.0], rest))                  # fewer of each
        v = rng.permutation(np.concatenate(parts))
    v[rng.permutation(n)[: n // 40]] = np.nan
    return bits_of_values(dt, v)


ROWS = {"full_range": 20000, "one_prefix": 6000, "carry": 6000, "zero_carry": 6000, "boundary": 5000,
        "specials": 3000, "masked": 2001, "masked_zero": 2001, "mode_ties": 6000, "mode_many": 20000}


def make(name, dt, d, nq=57, seed=0):
    """The case ``name`` for dtype ``dt`` with d columns (each its own draw), tuned to n_q quantiles where the case
    depends on the target ranks."""
    rng = np.random.RandomState([seed, SELECT_CASES.index(name) if name in SELECT_CASES else 20 + MODE_CASES.index(name),
                                 DTYPES.index(dt), d, nq])
    n = ROWS[name]
    if name == "specials":
        n = max(n, nq + 2)
    cols = []
    for j in range(d):
        if name == "full_range":
            c = _full_range(dt, rng, n)
        elif name == "one_prefix":
            c = _one_prefix(dt, rng, n)
        elif name == "carry":
            c = _carry(dt, rng, n, negative=j % 2 == 1)
        elif name == "zero_carry":
            c = _zero_carry(dt, rng, n)
        elif name == "boundary":
            c = _boundary(dt, rng, n, nq)
        elif name == "specials":
            c = _special(dt, rng, n, nq, SPECIAL_KINDS[j % len(SPECIAL_KINDS)])
        elif name in ("masked", "masked_zero"):
            c = _masked(dt, rng, n, zero=name == "masked_zero")
        else:
            c = _mode(dt, rng, n, many=name == "mode_many")
        cols.append(_u(dt, c))
    missing = {"masked": 2.0, "masked_zero": 0.0}.get(name)
    return Case(name, dt, np.stack(cols, axis=1), missing)


# ------------------------------------------------ the replay plan ------------------------------------------------
def plan():
    """(case, dtype, d, n_q, missing) of every selection the coverage test and the GPU replay run.  Every case and
    dtype at n_q 1, 2, 57 (3 CS + 1 columns) and 1000 (CS + 1 columns); every case at n_q = 10000 on two columns (the
    f32 / f64 rounds from round 2 on search their live lists in global memory); the full-range case at every width;
    the masked cases with and without their missing value, and missing = 0 on the signed-zero cases."""
    out = []
    for dt in DTYPES:
        c = sector(dt)
        for name in SELECT_CASES:
            miss = {"masked": 2.0, "masked_zero": 0.0}.get(name)
            for nq in (1, 2, 57, 1000, 10000):
                d = 3 * c + 1 if nq <= 57 else (c + 1 if nq == 1000 else 2)
                out.append((name, dt, d, nq, miss))
            if miss is not None:
                out.append((name, dt, c + 1, 57, None))
            if name in ("zero_carry", "specials"):
                out.append((name, dt, c + 1, 57, 0.0))
        for d in widths(dt)[:-1]:
            out.append(("full_range", dt, d, 57, None))
    return out
