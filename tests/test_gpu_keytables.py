"""The per-column key tables on the device (csrc/bkm_keys.cu) with keys built to collide (tests/keytable_cases.py),
against the slot-exact restatement of the passes, torch.unique / np.unique and scikit-learn 1.9: the 1024-slot probe
bound and the wrap at three home slots and four key widths, concurrent claims of one chain by many CTAs, the per-CTA
cache under keys that share its slots, table growth through LabelEncoder and OneHotEncoder with keys sharing 12 to 40
low hash bits, whole key spaces, count-pass chains past 1024 slots, the best entry at the edges of its 128 slices,
column grids past 65535, the cross-rank merge on one GPU with two threads as ranks, and the decode gather with codes out
of range.  The whole file peaks at about 150 MB of device memory."""
import os
import sys
import threading

import numpy as np
import pytest
import scipy.sparse
import sklearn.impute
import sklearn.preprocessing
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import keytable_cases as kc  # noqa: E402

from dask_ml_b200 import ChunkedArray, _keytables  # noqa: E402
from dask_ml_b200.cluster import k_means as km  # noqa: E402
from dask_ml_b200.preprocessing import _encode  # noqa: E402

CAP = 4096
WIDE = ["f64", "i64", "f32", "i32"]


def _chunks(t, rows):
    return [t[i: i + rows] for i in range(0, t.shape[0], rows)] or [t]


def distinct(X, caps, rows=None, full_probe=False):
    """The distinct pass over the CUDA block X (n, g) in chunks of ``rows``: (per-column (keys, counts) uint64 numpy,
    state (2, g) numpy)."""
    be = km._get_backend()
    keys, counts, off, total = _keytables.alloc(be, caps)
    state = be.zeros((2, X.shape[1]), torch.int64)
    for i, x in enumerate(_chunks(X, rows or X.shape[0])):
        be.distinct_chunk(x, keys, counts, off, total, state, first=i == 0, full_probe=full_probe)
    return _split(keys, counts, off), state.cpu().numpy()


def _split(keys, counts, off):
    k, c, o = keys.cpu().numpy().view(np.uint64), counts.cpu().numpy().view(np.uint64), off.cpu().numpy()
    return [(k[o[j]: o[j + 1]], c[o[j]: o[j + 1]]) for j in range(len(o) - 1)]


def assert_like(got, ref):
    """A table equal to the restatement's where the restatement raised no flag: the same occupied slots (bit for bit),
    the same keys and the same counts per key."""
    gk, gc = got
    rk, rc = ref.arrays()
    np.testing.assert_array_equal(gk != kc.EMPTY, rk != kc.EMPTY)
    occ = gk != kc.EMPTY
    assert dict(zip(gk[occ].tolist(), gc[occ].tolist())) == dict(zip(rk[occ].tolist(), rc[occ].tolist()))


def keys_of(v, dtype):
    return _encode.host_keys(v, kc.DTYPES[dtype])


# ------------------------------------------------ 1. probe bound and wrap ------------------------------------------------
@pytest.mark.parametrize("dtype", WIDE)
@pytest.mark.parametrize("slot", [0, 17, CAP - 5])
@pytest.mark.parametrize("m", [1024, 1025])
def test_probe_bound_and_wrap(dtype, slot, m):
    """m keys on one home slot of a 4096-slot table, as the middle column of three, each key twice in shuffled rows:
    1024 fill exactly [slot, slot + 1024) mod 4096; the 1025th overflows with 1024 keys in, and a full probe takes it."""
    tdt = kc.DTYPES[dtype]
    v = kc.home(dtype, CAP, slot, m, seed=slot + m)
    rng = np.random.RandomState(m)
    col = rng.permutation(np.concatenate([v, v]))
    side = np.asarray(rng.randint(0, 5, len(col)), dtype=col.dtype)
    X = kc.device(np.stack([side, col, side[::-1]], 1), tdt)
    run = np.zeros(CAP, bool)
    run[(slot + np.arange(1024)) % CAP] = True
    k = keys_of(v, dtype)
    (t0, (gk, gc), t2), st = distinct(X, [CAP] * 3, rows=768)
    assert list(st[1]) == [0, int(m > 1024), 0] and list(st[0]) == [5, 1024, 5]
    np.testing.assert_array_equal(gk != kc.EMPTY, run)
    assert set(gk[run].tolist()) <= set(k.tolist()) and (gc[run] == 1).all()
    if m == 1024:
        assert set(gk[run].tolist()) == set(k.tolist())
        assert_like((gk, gc), kc.Table(CAP).insert(k))
    for t in (t0, t2):
        assert_like(t, kc.Table(CAP).insert(kc.first_seen(keys_of(side, dtype))))
    (_, (gk, gc), _), st = distinct(X, [CAP] * 3, rows=768, full_probe=True)
    assert list(st[1]) == [0, 0, 0] and st[0][1] == m
    assert_like((gk, gc), kc.Table(CAP).insert(k, full_probe=True))


@pytest.mark.parametrize("dtype", ["i64", "f32"])
def test_merging_chains_across_the_wrap(dtype):
    """Two runs of 400 keys homed 200 slots apart before the end of the table merge into one chain of 800 that wraps
    to slot 0, among 300 keys elsewhere: the occupied slots are the restatement's."""
    tdt = kc.DTYPES[dtype]
    rng = np.random.RandomState(2)
    k = np.concatenate([kc.home_keys(tdt, CAP, CAP - 300, 400, seed=1), kc.home_keys(tdt, CAP, CAP - 100, 400, seed=2),
                        kc.placed_keys(tdt, CAP, rng.permutation(np.arange(1000, 3000))[:300], seed=3)])
    v = rng.permutation(kc.values(k, tdt))
    ((gk, gc),), st = distinct(kc.device(v, tdt), [CAP], rows=512)
    assert st[1][0] == 0 and st[0][0] == len(np.unique(k))
    ref = kc.Table(CAP).insert(k)
    assert not ref.overflow and ref.occupied()[: 500].any()
    assert_like((gk, gc), ref)


# ------------------------------------------------ 2. concurrent claims ------------------------------------------------
@pytest.mark.parametrize("dtype", ["i64", "f32"])
def test_concurrent_claims_of_one_chain(dtype):
    """2^20 rows in 4 chunks, every 256-row tile a permutation of the same 256 keys (200 of them on one home slot
    near the end of the table): thousands of CTAs race to claim the same chain.  Each key is claimed once: the
    occupancy is the distinct count, every count is 1, and the slots are the restatement's."""
    tdt = kc.DTYPES[dtype]
    k = np.concatenate([kc.home_keys(tdt, CAP, CAP - 60, 200, seed=4),
                        kc.placed_keys(tdt, CAP, np.arange(56) * 37 + 11, seed=5)])
    v = kc.values(k, tdt)
    rng = np.random.RandomState(6)
    tiles = 1 << 12
    idx = np.argsort(rng.uniform(size=(tiles, 256)), axis=1).reshape(-1)
    col0 = v[idx]
    col1 = v[::-1][idx]
    X = kc.device(np.stack([col0, col1], 1), tdt)
    tabs, st = distinct(X, [CAP, CAP], rows=1 << 18)
    assert list(st[1]) == [0, 0] and list(st[0]) == [256, 256]
    ref = kc.Table(CAP).insert(k)
    for t in tabs:
        assert_like(t, ref)


# ------------------------------------------------ 3. the CTA cache ------------------------------------------------
@pytest.mark.parametrize("dtype", WIDE)
def test_cache_mates(dtype):
    """Every column of a sector holds 64 keys that share one slot of the per-CTA cache and have different table
    slots; each warp of each tile alternates them, and a second set appears only from the middle of the rows on.  A
    cache that matched a mate for the key itself would drop keys."""
    tdt = kc.DTYPES[dtype]
    cs = 32 // torch.empty(0, dtype=tdt).element_size()
    n = 256 * 64
    cols, refs = [], []
    for j in range(cs):
        a = kc.cache_mates_keys(tdt, CAP, 64, cslot=9, seed=10 + j)
        b = kc.cache_mates_keys(tdt, CAP, 64, cslot=9, seed=100 + j)
        b = b[~np.isin(b, a)]
        r = np.arange(n)
        keys = np.where(r < n // 2, a[(r + j) % 64], np.where(r % 2 == 0, a[r % 64], b[(r // 2) % len(b)]))
        assert len(np.unique(keys)) == 64 + len(b)
        cols.append(kc.values(keys, tdt))
        refs.append(kc.Table(CAP).insert(np.concatenate([a, b])))
    X = kc.device(np.stack(cols, 1), tdt)
    tabs, st = distinct(X, [CAP] * cs, rows=n // 4)
    assert not st[1].any()
    for t, ref in zip(tabs, refs):
        assert_like(t, ref)
    assert list(st[0]) == [r.occ for r in refs]


# ------------------------------------------------ 4. growth through the public API ------------------------------------------------
@pytest.fixture
def caps_seen(monkeypatch):
    seen = []
    grow = _keytables.alloc

    def alloc(be, caps):
        seen.append([int(c) for c in caps])
        return grow(be, caps)

    monkeypatch.setattr(_keytables, "alloc", alloc)
    return seen


def _filler(dtype, n):
    """n distinct values of ``dtype`` away from the constructed keys."""
    a = np.arange(n)
    return {"f64": a * 0.5 - 7.0, "f32": (a * 0.25 + 1000.0).astype(np.float32), "i64": a * 7 - 10 ** 12,
            "i32": (a * 3 - 10 ** 6).astype(np.int32)}[dtype].astype(kc.HOST[kc.DTYPES[dtype]])


def _colliding(dtype, bits):
    tdt = kc.DTYPES[dtype]
    if bits == 12:
        k = kc.home_keys(tdt, CAP, 1234, 1100, seed=bits)
    elif kc.key_bits(tdt) == 32:
        k = kc.shared_low_bits32(bits)
    else:
        k = kc.shared_low(tdt, bits, 1100, low=0x3C3C3C & ((1 << bits) - 1), seed=bits)
    assert len(k) > 1024
    return kc.values(k, tdt)


@pytest.mark.parametrize("dtype,bits", [(d, 12) for d in WIDE] + [("f32", 17), ("i32", 17), ("f64", 24),
                                                                  ("i64", 24), ("f64", 40), ("i64", 40)])
def test_growth_with_colliding_keys(caps_seen, dtype, bits):
    """More than 1024 keys whose hashes share their low ``bits`` bits among 5000 other values: the encoders' tables
    grow to their limit and no further, and the categories, codes and CSR are scikit-learn's."""
    from dask_ml_b200.preprocessing import LabelEncoder, OneHotEncoder

    tdt = kc.DTYPES[dtype]
    rng = np.random.RandomState(bits)
    y = rng.permutation(np.concatenate([_colliding(dtype, bits), _filler(dtype, 5000)]))
    limit = _keytables.capacity(len(y), tdt)
    t = kc.device(y, tdt)
    le = LabelEncoder().fit(ChunkedArray([c.reshape(-1) for c in _chunks(t, 2000)]))
    np.testing.assert_array_equal(le.classes_, np.unique(y))
    np.testing.assert_array_equal(le.transform(t.reshape(-1)).compute(),
                                  sklearn.preprocessing.LabelEncoder().fit(y).transform(y))
    assert max(max(c) for c in caps_seen) <= limit, caps_seen
    X = np.stack([y, y[::-1]], 1)
    enc = OneHotEncoder(sparse=True, dtype=np.float64).fit(ChunkedArray(_chunks(kc.device(X, tdt), 3000)))
    sk = sklearn.preprocessing.OneHotEncoder(sparse_output=True, dtype=np.float64).fit(X)
    for g, w in zip(enc.categories_, sk.categories_):
        np.testing.assert_array_equal(g, w)
    got = enc.transform(ChunkedArray(_chunks(kc.device(X, tdt), 3000))).compute()
    want = sk.transform(X)
    assert scipy.sparse.issparse(got)
    for a in ("indptr", "indices", "data"):
        np.testing.assert_array_equal(getattr(got, a), getattr(want, a))
    assert max(max(c) for c in caps_seen) <= limit, caps_seen


# ------------------------------------------------ 5. whole key spaces ------------------------------------------------
def _whole(dtype):
    if dtype == "bf16":
        bits = torch.arange(-(1 << 15), 1 << 15, dtype=torch.int32).to(torch.int16)
        return bits.view(torch.bfloat16), bits.view(torch.bfloat16).float().numpy()
    if dtype == "u8":
        v = np.random.RandomState(1).permutation(np.tile(np.arange(256, dtype=np.uint8), 9))
    elif dtype == "bool":
        v = np.random.RandomState(1).randint(0, 2, 3000).astype(bool)
    else:
        i = np.iinfo(np.int32)
        v = np.concatenate([i.min + np.arange(300), i.max - np.arange(300), [0, -1, 1]]).astype(np.int32)
        v = np.random.RandomState(1).permutation(np.tile(v, 3))
    return torch.from_numpy(v), v


@pytest.mark.parametrize("dtype", ["bf16", "u8", "bool", "i32"])
def test_whole_key_spaces(dtype):
    """Every bf16 bit pattern (254 NaN patterns one key, +-0 one key), every uint8 value, both bools, and int32 at
    both ends of its range: the occupancy and the slots are the restatement's, the categories scikit-learn's."""
    from dask_ml_b200.preprocessing import LabelEncoder

    tdt = kc.DTYPES[dtype]
    t, h = _whole(dtype)
    k = _encode.host_keys(h, tdt)
    cap = _keytables.capacity(len(h), tdt)
    ((gk, gc),), st = distinct(t.reshape(-1, 1).cuda(), [cap], rows=4096)
    assert st[1][0] == 0 and st[0][0] == len(np.unique(k))
    assert_like((gk, gc), kc.Table(cap).insert(kc.first_seen(k)))
    if dtype == "bf16":
        assert st[0][0] == (1 << 16) - 254 + 1 - 1
    le = LabelEncoder().fit(t.cuda())
    want = np.unique(h)
    np.testing.assert_array_equal(le.classes_, want)
    np.testing.assert_array_equal(le.transform(t.cuda()).compute(), np.searchsorted(want, h) if dtype == "bf16"
                                  else sklearn.preprocessing.LabelEncoder().fit(h).transform(h))


# ------------------------------------------------ 6. count pass ------------------------------------------------
@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_count_pass_chains_past_the_bound(dtype):
    """1100 keys on one home slot of the count pass's table, with multiplicities 1 to 3 and NaN rows: the count pass
    probes up to the capacity, so every key is counted; the slots are the restatement's, the counts torch.unique's,
    and SimpleImputer's most_frequent statistic scikit-learn's (the smallest of the tied values)."""
    from dask_ml_b200.impute import SimpleImputer

    tdt = kc.DTYPES[dtype]
    rng = np.random.RandomState(8)
    mult = np.ones(1100, dtype=np.int64)
    mult[rng.permutation(1100)[:400]] = 2
    mult[rng.permutation(1100)[:6]] = 3
    valid = int(mult.sum())
    cap = _keytables.capacity(valid, tdt)
    assert cap == CAP
    k = kc.home_keys(tdt, cap, 77, 1100, seed=9)
    v = kc.values(k, tdt)
    col = rng.permutation(np.concatenate([np.repeat(v, mult), np.full(300, np.nan, dtype=v.dtype)]))
    be = km._get_backend()
    keys, counts, off, total = _keytables.alloc(be, [cap])
    X = kc.device(col, tdt)
    for i, x in enumerate(_chunks(X, 700)):
        be.mode_count_chunk(x, True, float("nan"), keys, counts, off, total, first=i == 0)
    ((gk, gc),) = _split(keys, counts, off)
    assert_like((gk, gc), kc.Table(cap, count=True).insert(k, mult))
    u, c = torch.unique(X[~torch.isnan(X)].double(), return_counts=True)
    occ = gk != kc.EMPTY
    assert dict(zip(gk[occ].tolist(), gc[occ].tolist())) == dict(zip(keys_of(u.cpu().numpy(), dtype).tolist(),
                                                                      c.cpu().numpy().tolist()))
    bk, bc, nd = (a.cpu().numpy() for a in be.mode_best(keys, counts, off, 1, total))
    assert int(bk.view(np.uint64)[0]) == int(k[mult == 3].min()) and bc[0] == 3 and nd[0] == 1100
    imp = SimpleImputer(strategy="most_frequent").fit(ChunkedArray(_chunks(X, 900)))
    sk = sklearn.impute.SimpleImputer(strategy="most_frequent").fit(col.reshape(-1, 1))
    np.testing.assert_array_equal(imp.statistics_, sk.statistics_)


# ------------------------------------------------ 7. best-entry slices ------------------------------------------------
def _tied(dtype, cap, pos, seed=0):
    """(smallest tied key at slot ``pos``, 4 larger tied keys in slice 0, 40 keys of count 1 in other slices) of a
    table of capacity ``cap``."""
    tdt = kc.DTYPES[dtype]
    rng = np.random.RandomState(seed)
    slots0 = rng.permutation(cap // 128)[:60]
    low = kc.placed_keys(tdt, cap, slots0, seed=seed)
    best = None
    for s in range(seed, seed + 200):
        cand = kc.placed_keys(tdt, cap, [pos], seed=s)[0]
        if (low > cand).sum() >= 4:
            best = cand
            break
    assert best is not None
    tied = np.concatenate([[best], low[low > best][:4]])
    ones = kc.placed_keys(tdt, cap, cap // 128 * (1 + rng.permutation(126)[:40]) + rng.randint(1, 50, 40), seed=seed)
    ones = ones[~np.isin(ones, tied)]
    return tied, ones


@pytest.mark.parametrize("dtype,cap", [("f64", 1 << 22), ("f32", 1 << 20)])
@pytest.mark.parametrize("where", ["last", "slice_start", "before_slice"])
def test_best_entry_slices(dtype, cap, where):
    """A table of 128 slices (the most bkm_mode_best splits one into): the smallest of five keys tied on the largest
    count sits in the last slot, at the first slot of slice 37 or in the slot before slice 90, the other four in slice
    0; then the same table in a group with tables of 4 and 0 slots."""
    tdt = kc.DTYPES[dtype]
    pos = {"last": cap - 1, "slice_start": cap // 128 * 37, "before_slice": cap // 128 * 90 - 1}[where]
    tied, ones = _tied(dtype, cap, pos)
    small = kc.values(kc.placed_keys(tdt, 4, [1, 3], seed=1), tdt)
    col = np.concatenate([np.repeat(kc.values(tied, tdt), 3), kc.values(ones, tdt)])
    n = len(col)
    col1 = np.concatenate([np.repeat(small, [2, 5]), np.full(n - 7, np.nan, dtype=col.dtype)])
    be = km._get_backend()
    for caps in ([cap], [cap, 4, 0]):
        g = len(caps)
        X = kc.device(np.stack([col, col1, col][:g], 1), tdt)
        keys, counts, off, total = _keytables.alloc(be, caps)
        be.mode_count_chunk(X, True, float("nan"), keys, counts, off, total, first=True)
        bk, bc, nd = (a.cpu().numpy() for a in be.mode_best(keys, counts, off, g, total))
        assert int(bk.view(np.uint64)[0]) == int(tied[0]) and bc[0] == 3 and nd[0] == len(tied) + len(ones)
        if g == 3:
            assert int(bk.view(np.uint64)[1]) == int(_encode.host_keys(small[1:], tdt)[0]) and bc[1] == 5
            assert nd[1] == 2 and bc[2] == 0 and nd[2] == 0 and int(bk.view(np.uint64)[2]) == int(kc.EMPTY)


def test_imputer_best_entry_in_the_last_slot():
    """SimpleImputer most_frequent on 2^19 valid float64 rows (a half-full 2^20-slot table of 128 slices) and NaN
    rows: the smallest of the values tied on count 3 has its home in the table's last slot, the larger ones in slice
    0."""
    from dask_ml_b200.impute import SimpleImputer

    cap = 1 << 20
    tied, _ = _tied("f64", cap, cap - 1, seed=3)
    tv = kc.values(tied, torch.float64)
    rng = np.random.RandomState(4)
    rest = (1 << 19) - 3 * len(tied)
    filler = np.arange(rest) * 0.5 + 1e6
    col = rng.permutation(np.concatenate([np.repeat(tv, 3), filler, np.full(1000, np.nan)]))
    X = np.stack([col, col[::-1]], 1)
    imp = SimpleImputer(strategy="most_frequent").fit(ChunkedArray(_chunks(kc.device(X, torch.float64), 200000)))
    sk = sklearn.impute.SimpleImputer(strategy="most_frequent").fit(X)
    np.testing.assert_array_equal(imp.statistics_, sk.statistics_)
    assert imp.statistics_[0] == tv[0]


# ------------------------------------------------ 8. wide groups ------------------------------------------------
def test_best_and_compact_past_65535_columns():
    """65537 columns of two rows: bkm_mode_best and bkm_mode_compact loop over columns in steps of their grid."""
    g = 65537
    rng = np.random.RandomState(5)
    X = rng.randint(0, 3, (2, g)).astype(np.float64)
    X[:, -1] = [7.0, np.nan]
    be = km._get_backend()
    caps = [4] * g
    keys, counts, off, total = _keytables.alloc(be, caps)
    be.mode_count_chunk(kc.device(X, torch.float64), True, float("nan"), keys, counts, off, total, first=True)
    bk, bc, nd = (a.cpu().numpy() for a in be.mode_best(keys, counts, off, g, total))
    kk = _encode.host_keys(X, torch.float64)
    same = X[0] == X[1]
    np.testing.assert_array_equal(bc[:-1], np.where(same, 2, 1)[:-1])
    np.testing.assert_array_equal(nd[:-1], np.where(same, 1, 2)[:-1])
    np.testing.assert_array_equal(bk.view(np.uint64)[:-1], np.minimum(kk[0], kk[1])[:-1])
    assert bc[-1] == 1 and nd[-1] == 1 and int(bk.view(np.uint64)[-1]) == int(kk[0, -1])
    E = int(nd.sum())
    e = be.zeros((E + 1, 4), torch.float64)
    be.mode_compact(keys, counts, off, g, e[:E])
    e = e.cpu().numpy()
    assert (e[E] == 0).all()
    got = sorted(zip(e[:E, 0].astype(np.int64).tolist(),
                     ((e[:E, 1].astype(np.uint64) << np.uint64(32)) | e[:E, 2].astype(np.uint64)).tolist(),
                     e[:E, 3].astype(np.int64).tolist()))
    want = []
    for j in range(g):
        col = X[:, j][~np.isnan(X[:, j])]
        u, c = np.unique(_encode.host_keys(col, torch.float64), return_counts=True)
        want += [(j, int(a), int(b)) for a, b in zip(u, c)]
    assert got == sorted(want)


def test_distinct_past_65535_sectors():
    """bf16, 16 x 65535 + 17 columns of two rows (tables of 4 slots, 67 MB): the sector scan loops over column
    sectors in steps of its grid, and every column's occupancy and distinct count are exact."""
    g = 16 * 65535 + 17
    j = np.arange(g)
    v0 = (j % 200).astype(np.float32)
    v1 = np.where(j % 3 == 0, v0, v0 + 1)
    X = torch.from_numpy(np.stack([v0, v1])).to(torch.bfloat16).cuda()
    be = km._get_backend()
    keys, counts, off, total = _keytables.alloc(be, [4] * g)
    state = be.zeros((2, g), torch.int64)
    be.distinct_chunk(X, keys, counts, off, total, state, first=True)
    st = state.cpu().numpy()
    want = np.where(j % 3 == 0, 1, 2)
    assert not st[1].any()
    np.testing.assert_array_equal(st[0], want)
    _, bc, nd = be.mode_best(keys, counts, off, g, total)
    np.testing.assert_array_equal(nd.cpu().numpy(), want)
    np.testing.assert_array_equal(bc.cpu().numpy(), np.ones(g))
    k = keys.cpu().numpy().view(np.uint64).reshape(g, 4)
    kk = _encode.host_keys(X.float().cpu().numpy(), torch.bfloat16)
    tail = j >= 16 * 65535 - 5
    for c in np.flatnonzero(tail):
        assert set(k[c][k[c] != kc.EMPTY].tolist()) == {int(kk[0, c]), int(kk[1, c])}


# ------------------------------------------------ 9. merge on one GPU ------------------------------------------------
class ThreadComm:
    """The sum all-reduce of ``engine.Comm`` between threads of one process, one thread per rank, each with its own
    backend: every rank's buffer is added in rank order."""

    def __init__(self, rank, world, shared):
        self.rank, self.world, self.shared = rank, world, shared

    def allreduce_sum_(self, t):
        s = self.shared
        torch.cuda.synchronize()
        s["bufs"][self.rank] = t.clone()
        torch.cuda.synchronize()
        s["barrier"].wait()
        total = s["bufs"][0].clone()
        for b in s["bufs"][1:]:
            total += b
        torch.cuda.synchronize()
        s["barrier"].wait()
        t.copy_(total)
        torch.cuda.synchronize()


def _run_ranks(world, fn):
    shared = {"bufs": [None] * world, "barrier": threading.Barrier(world)}
    out, errs = [None] * world, []

    def run(r):
        try:
            out[r] = fn(r, ThreadComm(r, world, shared))
        except BaseException as e:           # noqa: BLE001 - re-raised below
            errs.append(e)
            shared["barrier"].abort()

    th = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    if errs:
        raise errs[0]
    return out


@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_merge_ranks_on_one_gpu(dtype):
    """Two ranks count overlapping row sets that hold 600 keys on one home slot of the merged table: the merged
    tables are the same on both ranks, each key with the sum of its counts over the ranks, the slots the
    restatement's and the best entry the smallest of the keys tied on the largest summed count."""
    tdt = kc.DTYPES[dtype]
    rng = np.random.RandomState(11)
    m = 600
    merged_cap = 2048           # each rank holds 420 to 434 of the 640 keys: the merged tables take capacity(513..1024)
    k = np.concatenate([kc.home_keys(tdt, merged_cap, merged_cap - 7, m, seed=12),
                        kc.placed_keys(tdt, merged_cap, np.arange(40) * 50 + 3, seed=13)])
    v = kc.values(k, tdt)
    rows = rng.permutation(np.concatenate([v, v[:5], v[:5]]))
    parts = [rows[: 2 * len(rows) // 3], rows[len(rows) // 3:]]
    g = 2

    def rank(r, comm):
        be = km._get_backend()
        X = kc.device(np.stack([parts[r], parts[r][::-1]], 1), tdt)
        tab = _keytables.alloc(be, [_keytables.capacity(len(parts[r]), tdt)] * g)
        be.mode_count_chunk(X, True, float("nan"), *tab[:3], tab[3], first=True)
        _, _, nd = be.mode_best(*tab[:3], g, tab[3])
        (keys, counts, off, total), best, _ = _keytables.merge_ranks(be, comm, tab, g, tdt, nd)
        return _split(keys, counts, off), [b.cpu().numpy() for b in best]

    out = _run_ranks(2, rank)
    for a, b in zip(out[0][0], out[1][0]):          # the same content (where a chain's keys sit depends on timing)
        assert_like(a, kc.Table(len(b[0]), count=True).insert(b[0][b[0] != kc.EMPTY], b[1][b[0] != kc.EMPTY]))
    allk = np.concatenate([_encode.host_keys(p, tdt) for p in parts])
    u, c = np.unique(allk, return_counts=True)
    for j in range(g):
        t = out[0][0][j]
        assert len(t[0]) == merged_cap
        assert_like(t, kc.Table(merged_cap, count=True).insert(u, c))
    bk, bc, nd = out[0][1]
    top = u[c == c.max()].min()
    assert list(bk.view(np.uint64)) == [int(top)] * g and list(bc) == [c.max()] * g and list(nd) == [len(u)] * g


def test_mode_merge_synthetic_entries():
    """bkm_mode_merge on hand-made rows: keys whose high word is at least 2^31, counts up to 2^52 that add to an exact
    2^52 + 3, zero-count padding rows, and rows whose column is outside the group or has no table (all skipped)."""
    be = km._get_backend()
    caps = [16, 0, 8]
    keys, counts, off, total = _keytables.alloc(be, caps)
    K1, K2, K3 = 0xFFFFFFF0_00000001, 0x80000000_FFFFFFFF, 0x00000001_00000000
    rows = [(0, K1, 2.0 ** 52), (0, K1, 3.0), (0, K2, 5.0), (2, K3, 7.0), (2, K1, 1.0), (0, K3, 0.0),
            (1, K2, 9.0), (-1, K2, 4.0), (3, K2, 4.0), (70000, K3, 2.0), (0, 0, 0.0), (0, 0, 0.0)]
    e = np.array([[c, k >> 32, k & 0xFFFFFFFF, n] for c, k, n in rows], dtype=np.float64)
    be.mode_merge(torch.from_numpy(e).cuda(), keys, counts, off, 3, total)
    tabs = _split(keys, counts, off)
    got = [dict(zip(t[0][t[0] != kc.EMPTY].tolist(), t[1][t[0] != kc.EMPTY].tolist())) for t in tabs]
    assert got == [{K1: 2 ** 52 + 3, K2: 5}, {}, {K3: 7, K1: 1}]
    bk, bc, nd = (a.cpu().numpy() for a in be.mode_best(keys, counts, off, 3, total))
    assert list(bk.view(np.uint64)) == [K1, int(kc.EMPTY), K3] and list(bc) == [2.0 ** 52 + 3, 0, 7]
    assert list(nd) == [2, 0, 2]
    out = be.zeros((5, 4), torch.float64)
    be.mode_compact(keys, counts, off, 3, out[:4])
    o = out.cpu().numpy()
    assert sorted(map(tuple, o[:4].tolist())) == sorted(
        [(0.0, K1 >> 32, K1 & 0xFFFFFFFF, 2.0 ** 52 + 3), (0.0, K2 >> 32, K2 & 0xFFFFFFFF, 5.0),
         (2.0, K3 >> 32, K3 & 0xFFFFFFFF, 7.0), (2.0, K1 >> 32, K1 & 0xFFFFFFFF, 1.0)])
    assert (o[4] == 0).all()


# ------------------------------------------------ 10. decode ------------------------------------------------
@pytest.mark.parametrize("code_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("vals_dtype", [torch.uint8, torch.int16, torch.float32, torch.float64])
def test_decode_codes_out_of_range(code_dtype, vals_dtype):
    """bkm_decode_chunk over three columns of 5, 1 and 7 categories: in-range codes gather their value, -1, K and the
    largest code write zero bytes and are counted per column, with the first 8 of them kept."""
    be = km._get_backend()
    K = [5, 1, 7]
    rng = np.random.RandomState(1)
    vals = [rng.randint(1, 100, k) for k in K]
    cat_vals = torch.from_numpy(np.concatenate(vals)).to(vals_dtype).cuda()
    off = np.concatenate([[0], np.cumsum(K)]).astype(np.int64)
    big = torch.iinfo(code_dtype).max
    n = 300
    codes = np.stack([rng.randint(0, k, n) for k in K], 1).astype(np.int64)
    bad = {0: [(3, -1), (10, 5), (11, big)], 1: [(0, 1), (299, -1)], 2: [(i, 7 + i) for i in range(12)]}
    for j, lst in bad.items():
        for i, c in lst:
            codes[i, j] = c
    ct = torch.from_numpy(codes).to(code_dtype).cuda()
    out = torch.full((n, 3), 77, dtype=vals_dtype, device="cuda")
    unknown = be.zeros((1 + 3 + 3 * 8,), torch.int64)
    be.decode_chunk(ct, cat_vals, torch.from_numpy(off).cuda(), out, unknown)
    o, u = out.cpu().numpy(), unknown.cpu().numpy()
    flat = cat_vals.cpu().numpy()
    for j in range(3):
        ok = (codes[:, j] >= 0) & (codes[:, j] < K[j])
        np.testing.assert_array_equal(o[ok, j], flat[off[j] + codes[ok, j]])
        assert (o[~ok, j] == 0).all()
        assert u[1 + j] == len(bad[j])
        kept = u[4 + 8 * j: 4 + 8 * j + min(8, len(bad[j]))]
        assert set(kept.tolist()) <= {c for _, c in bad[j]} and len(set(kept.tolist())) == min(8, len(bad[j]))
    assert u[0] == sum(len(b) for b in bad.values())
