"""The per-column key tables without a GPU: the key constructors of tests/keytable_cases.py (home slots, cache slots,
round trips), the slot-exact restatement of the distinct and count passes at the probe bound and across the wrap, its
independence of the insertion order, and the encoders' growth loop (``_encode._group_keys``) on a CPU backend whose
distinct pass is that restatement: a table at its limit is run again with a full probe, never grown past it."""
import os
import sys

import numpy as np
import pytest
import sklearn.preprocessing
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import keytable_cases as kc  # noqa: E402
from test_encoders_host import EncodeOracleBackend, enc_keys  # noqa: E402

from dask_ml_b200.preprocessing import _encode  # noqa: E402

CAP = 4096
WIDE = ["f64", "i64", "f32", "i32"]


def test_mix64_inverse_round_trips():
    r = np.random.RandomState(0).randint(-(1 << 63), (1 << 63) - 1, 1000, dtype=np.int64).view(np.uint64)
    np.testing.assert_array_equal(kc.unmix64(kc.mix64(r)), r)
    np.testing.assert_array_equal(kc.mix64(kc.unmix64(r)), r)
    # against the device code's steps in Python integers
    M = (1 << 64) - 1
    for x in r[:20].tolist() + [0, 1, M]:
        h = x ^ (x >> 33)
        h = (h * 0xFF51AFD7ED558CCD) & M
        h ^= h >> 33
        h = (h * 0xC4CEB9FE1A85EC53) & M
        h ^= h >> 33
        assert int(kc.mix64(x)[0]) == h


@pytest.mark.parametrize("dtype", WIDE)
@pytest.mark.parametrize("slot", [0, 17, CAP - 5])
def test_home_keys_land_and_round_trip(dtype, slot):
    tdt = kc.DTYPES[dtype]
    v = kc.home(dtype, CAP, slot, 1025, seed=slot)
    k = _encode.host_keys(v, tdt)
    assert len(np.unique(k)) == 1025
    assert (kc.home_slot(k, CAP) == slot).all()
    if dtype[0] == "f":
        assert np.isfinite(v).all() and not (np.signbit(v) & (v == 0)).any()


@pytest.mark.parametrize("dtype", WIDE)
@pytest.mark.parametrize("slot", [0, 17, CAP - 5])
def test_probe_bound_and_wrap(dtype, slot):
    tdt = kc.DTYPES[dtype]
    k = kc.home_keys(tdt, CAP, slot, 1025, seed=slot)
    run = (slot + np.arange(1024)) % CAP
    t = kc.Table(CAP).insert(k[:1024])
    want = np.zeros(CAP, bool)
    want[run] = True
    np.testing.assert_array_equal(t.occupied(), want)
    assert not t.overflow and t.occ == 1024
    keys, counts = t.arrays()
    assert set(keys[run].tolist()) == set(k[:1024].tolist()) and (counts[run] == 1).all()
    t = kc.Table(CAP).insert(k)                     # the 1025th examines 1024 full slots
    assert t.overflow and t.occ == 1024
    np.testing.assert_array_equal(t.occupied(), want)
    t = kc.Table(CAP).insert(k, full_probe=True)    # a full probe takes it one slot further
    assert not t.overflow and t.occ == 1025 and t.occupied()[(slot + 1024) % CAP]
    c = kc.Table(CAP, count=True).insert(np.concatenate([k, k[:7]]))     # the count pass's bound is the capacity
    assert not c.overflow and c.occ == 1025 and sorted(c.counts.values()) == [1] * 1018 + [2] * 7


@pytest.mark.parametrize("seed", range(6))
def test_occupied_slots_do_not_depend_on_order(seed):
    """Two merging chains across the wrap, a third one apart and random keys: every insertion order leaves the same
    slots occupied when no insert fails (which key sits where does depend on the order)."""
    tdt = torch.int64
    k = np.concatenate([kc.home_keys(tdt, CAP, CAP - 300, 400, seed=1), kc.home_keys(tdt, CAP, CAP - 100, 400, seed=2),
                        kc.home_keys(tdt, CAP, 900, 40, seed=3),
                        np.random.RandomState(4).randint(0, 1 << 62, 300).astype(np.uint64)])
    ref = kc.Table(CAP).insert(k)
    assert not ref.overflow and ref.occ == len(np.unique(k))
    got = kc.Table(CAP).insert(np.random.RandomState(seed).permutation(k))
    assert not got.overflow
    np.testing.assert_array_equal(got.occupied(), ref.occupied())
    assert sorted(got.slots.values()) == sorted(ref.slots.values())
    if seed == 0:
        assert (got.arrays()[0] != ref.arrays()[0]).any()


@pytest.mark.parametrize("dtype", WIDE)
def test_cache_mates(dtype):
    tdt = kc.DTYPES[dtype]
    cs = 32 // torch.empty(0, dtype=tdt).element_size()
    k = kc.cache_mates_keys(tdt, CAP, 64, cslot=7, seed=1)
    assert (kc.cache_slot(k, tdt) == 7).all() and (kc.cache_slot(k, tdt) < kc.FILTER_SLOTS // cs).all()
    assert len(np.unique(kc.home_slot(k, CAP))) == 64
    kc.values(k, tdt)


@pytest.mark.parametrize("dtype", WIDE)
def test_placed_keys(dtype):
    tdt = kc.DTYPES[dtype]
    cap = 1 << 20
    slots = [cap - 1, 0, cap // 128 * 37, cap // 128 * 37 - 1]
    k = kc.placed_keys(tdt, cap, slots)
    np.testing.assert_array_equal(kc.home_slot(k, cap), slots)
    t = kc.Table(cap).insert(k)
    np.testing.assert_array_equal(np.flatnonzero(t.occupied()), sorted(slots))


# ------------------------------------------------ the growth loop ------------------------------------------------
class RestatedTablesBackend(EncodeOracleBackend):
    """The encoders' CPU backend with the distinct pass restated slot by slot (keytable_cases.Table, keys in the
    order of their first occurrence) on tables that hold only their keys, so a capacity of 2^30 slots costs nothing.
    ``calls`` records (capacities, full_probe) of every distinct pass."""

    calls = []

    def distinct_chunk(self, x, keys, counts, off, total, state, first=False, full_probe=False):
        self.launches += 1
        tabs = keys.tables
        if first:
            tabs[:] = [kc.Table(t.cap) for t in tabs]
            state.zero_()
            RestatedTablesBackend.calls.append(([t.cap for t in tabs], full_probe))
        K = enc_keys(x) if x.shape[0] else np.zeros((0, x.shape[1]), dtype=np.uint64)
        for j, t in enumerate(tabs):
            if t.cap:
                t.insert(kc.first_seen(K[:, j]), full_probe=full_probe)
            state[0, j] = t.occ
            state[1, j] = int(t.overflow) | 2 * int(t.marker)

    def mode_compact(self, keys, counts, off, g, entries):
        self.launches += 1
        rows = [[j, float(k >> 32), float(k & 0xFFFFFFFF), 1.0] for j, t in enumerate(keys.tables)
                for k in t.slots.values()]
        entries[: len(rows)] = torch.tensor(rows, dtype=torch.float64).reshape(-1, 4)


LIMIT_CAPS = 1 << 30          # a capacity sequence that passes this is unbounded (16 GiB of tables)


@pytest.fixture
def restated(monkeypatch):
    from dask_ml_b200 import _keytables
    from dask_ml_b200.cluster import k_means as km

    def alloc(be, caps):
        caps = [int(c) for c in caps]
        if max(caps) > LIMIT_CAPS:
            seq = [c for c, _ in RestatedTablesBackend.calls] + [caps]
            raise AssertionError("unbounded table growth: %s" % seq)
        keys = torch.zeros(1, dtype=torch.int64)
        keys.tables = [kc.Table(c) for c in caps]
        off = torch.as_tensor(np.concatenate([[0], np.cumsum(caps)]).astype(np.int64))
        return keys, torch.zeros(1, dtype=torch.int64), off, int(off[-1])

    monkeypatch.setattr(km, "_BACKEND_FACTORY", RestatedTablesBackend)
    monkeypatch.setattr(_keytables, "alloc", alloc)
    RestatedTablesBackend.calls = []
    return RestatedTablesBackend.calls


def _collide40(dtype, m, seed=0):
    """m values whose keys' hashes agree in their low 40 bits: no table of up to 2^40 slots separates them."""
    tdt = kc.DTYPES[dtype]
    return kc.values(kc.shared_low(tdt, 40, m, low=0x5A5A5, seed=seed), tdt)


@pytest.mark.parametrize("dtype", ["i64", "f64"])
def test_table_at_its_limit_takes_a_full_probe(restated, dtype):
    """1025 rows whose keys share 40 low hash bits: the table's limit is 4096 slots (2 x 1025 rows), where the chain
    of 1025 keys passes the 1024-slot bound.  Growing the table cannot separate them; the group runs again at the same
    capacity with a full probe."""
    from dask_ml_b200.preprocessing import LabelEncoder

    y = _collide40(dtype, 1025)
    le = LabelEncoder().fit(y)
    np.testing.assert_array_equal(le.classes_, np.unique(y))
    np.testing.assert_array_equal(le.transform(y).compute(), sklearn.preprocessing.LabelEncoder().fit(y).transform(y))
    assert restated == [([4096], False), ([4096], True)]


def test_column_below_its_limit_still_grows(restated):
    """Two columns of 21025 rows: one holds the 1025 colliding keys among 20000 distinct others (limit 65536 slots),
    the other three values.  The first grows x8 to its limit, then the group runs again with a full probe; the second
    stays at 4096 slots."""
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.preprocessing import OneHotEncoder

    rng = np.random.RandomState(3)
    a = np.concatenate([_collide40("i64", 1025), rng.permutation(np.arange(20000, dtype=np.int64) - 10000)])
    X = np.stack([rng.permutation(a), rng.randint(0, 3, len(a))], axis=1)
    enc = OneHotEncoder(sparse=True).fit(ChunkedArray.from_array(X, 8000))
    sk = sklearn.preprocessing.OneHotEncoder().fit(X)
    for g, w in zip(enc.categories_, sk.categories_):
        np.testing.assert_array_equal(g, w)
    got = enc.transform(ChunkedArray.from_array(X, 8000)).compute()
    want = sk.transform(X)
    np.testing.assert_array_equal(got.indices, want.indices)
    np.testing.assert_array_equal(got.indptr, want.indptr)
    assert restated == [([4096, 4096], False), ([32768, 4096], False), ([65536, 4096], False),
                        ([65536, 4096], True)]
