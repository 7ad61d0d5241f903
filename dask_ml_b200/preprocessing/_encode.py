"""The device side of LabelEncoder and OneHotEncoder: a native-dtype intake, the exact categories of every column and
the encoding passes (DESIGN.md, "The passes of the encoders"):

    fit (bkm_distinct_chunk, one read of X per column group and growth step): every distinct value's order-preserving
                    key in a per-column hash table that starts at INITIAL_SLOTS slots; a column whose table passes half
                    full is grown (x8, capped by its key space and rows) and its group runs again; one whose table is
                    at that cap runs again with probes bounded by the capacity.  The occupied keys are
                    compacted (bkm_mode_compact) and sorted per column in torch.  With several ranks the tables are
                    gathered by the sum all-reduce and merged (bkm_mode_merge), as SimpleImputer's mode does
    transform (bkm_encode_chunk, one read of X): codes, the dense one-hot matrix or the CSR indices, by binary search
                    of each element's key in its column's sorted keys; unknown keys are counted on the device and
                    checked once, after the last chunk, on every rank
    inverse (bkm_decode_chunk): codes -> category values

Keys (include/bkm_b200.h): floats the radix keys with -0.0 folded to +0.0 and every NaN one key, the largest; integers
the value with its sign bit flipped.  int8 / int16 / uint16 blocks are widened to int32, uint32 to int64 and float16 to
float32 by torch before the pass (exact); the categories are mapped back to the input's dtype.
"""
import numpy as np
import torch

from .. import _keytables, _lib
from ..chunked import ChunkedArray, _is_torch, block_dtype, is_dask_dataframe
from ..cluster import k_means as _km
from ..engine import DeviceData
from .data import keys_to_values

INITIAL_SLOTS = 4096          # a column's first table: 64 KiB of keys and counts
GROWTH = 8
ENCODE_BUDGET = 1 << 30       # bytes of one column group's first tables: wider data runs in column groups

# the element types the passes take, and what other dtypes are widened to
_NATIVE = (torch.float32, torch.float64, torch.bfloat16, torch.int32, torch.int64, torch.uint8, torch.bool)
_WIDEN = {torch.int8: torch.int32, torch.int16: torch.int32, torch.float16: torch.float32}
_NP_WIDEN = {np.dtype("int8"): torch.int32, np.dtype("int16"): torch.int32, np.dtype("uint16"): torch.int32,
             np.dtype("uint32"): torch.int64, np.dtype("float16"): torch.float32}
_NAN_KEY = {torch.bfloat16: 0xFFC0, torch.float32: 0xFFC00000, torch.float64: 0xFFF8000000000000}
_I64_MIN = -(1 << 63)


def device_dtype(dtype):
    """The torch dtype the passes run a block of ``dtype`` (numpy or torch) in, or None when it has none (strings,
    objects, complex, uint64)."""
    if isinstance(dtype, torch.dtype):
        return dtype if dtype in _NATIVE else _WIDEN.get(dtype)
    dtype = np.dtype(dtype)
    if dtype in _NP_WIDEN:
        return _NP_WIDEN[dtype]
    t = {np.dtype("float32"): torch.float32, np.dtype("float64"): torch.float64, np.dtype("int32"): torch.int32,
         np.dtype("int64"): torch.int64, np.dtype("uint8"): torch.uint8, np.dtype("bool"): torch.bool}
    return t.get(dtype)


def _blocks(X):
    try:
        import pandas as pd

        if isinstance(X, (pd.Series, pd.DataFrame)):
            X = X.to_numpy()
    except ImportError:  # pragma: no cover
        pass
    if is_dask_dataframe(X):
        raise TypeError("dask DataFrames and Series are not supported; pass a dask array")
    if isinstance(X, (list, tuple)):
        X = np.asarray(X)
    return _km._to_blocks(X)


def host_dtype(X):
    """The numpy dtype of X's blocks (float32 for bfloat16 blocks), or None for input that is not an array."""
    try:
        return block_dtype(_blocks(X)[0])
    except Exception:
        return None


def device_input(X):
    """True when X is an array kind whose values the passes take (numeric: not strings, objects or DataFrames)."""
    try:
        b = _blocks(X)[0]
    except Exception:
        return False
    dt = getattr(b, "dtype", None)
    return dt is not None and device_dtype(dt) is not None


def intake(X, ndim, backend=None):
    """X -> DeviceData of 2-D blocks in X's own dtype (widened as above, never cast to float), and the numpy dtype the
    categories take.  ``ndim`` 1 takes a 1-D y (each block a column), 2 a 2-D X.  Device blocks are not copied."""
    blocks = _blocks(X)
    hdt = block_dtype(blocks[0])
    first = blocks[0]
    tdt = device_dtype(first.dtype if _is_torch(first) else np.asarray(first).dtype)
    if tdt is None:
        raise TypeError("dtype %s cannot be encoded on the device" % hdt)
    be = backend or _km._get_backend()
    out = []
    for b in blocks:
        if b.ndim != ndim and not (ndim == 1 and b.ndim == 2 and b.shape[1] == 1):
            raise ValueError("Expected a %d-D array, got an array of shape %s" % (ndim, tuple(b.shape)))
        if _is_torch(b):
            t = b.to(device=be.device, dtype=tdt)
        else:
            a = np.asarray(b)
            np_dt = torch.empty(0, dtype=tdt).numpy().dtype
            a = np.array(a, dtype=np_dt) if (a.dtype != np_dt or not a.flags.writeable) else np.ascontiguousarray(a)
            t = torch.from_numpy(a).to(be.device)
        out.append(t.reshape(-1, 1) if ndim == 1 else (t if t.stride(-1) == 1 else t.contiguous()))
    return DeviceData(out, be), hdt


# ------------------------------------------------ keys ------------------------------------------------
def host_keys(values, tdt):
    """The device keys of ``values`` as data of torch dtype ``tdt`` would have them: uint64 numpy."""
    v = np.asarray(values)
    if tdt in (torch.float32, torch.float64, torch.bfloat16):
        f = v.astype(np.float64 if tdt == torch.float64 else np.float32)
        nan = np.isnan(f)
        f = np.where(f == 0, f.dtype.type(0), f)
        if tdt == torch.float64:
            u = f.view(np.uint64)
        elif tdt == torch.float32:
            u = f.view(np.uint32).astype(np.uint64)
        else:
            u = (f.view(np.uint32) >> np.uint32(16)).astype(np.uint64)
        bits = _keytables.KEY_BITS[tdt]
        sign = np.uint64(1 << (bits - 1))
        mask = np.uint64((1 << bits) - 1) if bits < 64 else np.uint64(0xFFFFFFFFFFFFFFFF)
        k = np.where(u & sign, ~u & mask, u | sign)
        k[nan] = np.uint64(_NAN_KEY[tdt])
        return k.astype(np.uint64)
    if tdt == torch.int32:
        return (v.astype(np.int64) + (1 << 31)).astype(np.uint64)
    if tdt == torch.int64:
        return v.astype(np.int64).view(np.uint64) ^ np.uint64(1 << 63)
    return v.astype(np.uint64)


def key_values(keys, tdt, hdt):
    """Keys (uint64 numpy) -> the values of numpy dtype ``hdt`` they stand for."""
    keys = np.asarray(keys, dtype=np.uint64)
    if tdt in (torch.float32, torch.float64, torch.bfloat16):
        vals = keys_to_values(keys, tdt)
    elif tdt == torch.int32:
        vals = (keys.astype(np.int64) - (1 << 31))
    elif tdt == torch.int64:
        vals = (keys ^ np.uint64(1 << 63)).view(np.int64)
    else:
        vals = keys
    return vals.astype(hdt)


def _entry_keys(entries):
    """(column, key int64 holding the uint64 key) of compacted rows {column, key >> 32, key & 0xffffffff, count}."""
    e = entries.to(torch.int64)
    return e[:, 0], (e[:, 1] << 32) | e[:, 2]


def _group_keys(X, j0, j1):
    """Every distinct key of columns [j0, j1) over every rank: (column within the group, key) int64 device tensors,
    unsorted."""
    be, comm, g = X.backend, X.comm, j1 - j0
    limit = _keytables.capacity(max(1, X.n_local), X.dtype)         # a table that is never more than half full
    caps = np.full(g, min(INITIAL_SLOTS, limit), dtype=np.int64)
    full = False
    while True:
        keys, counts, off, total = _keytables.alloc(be, caps)
        state = be.zeros((2, g), torch.int64)
        # full_probe is passed only when set: a backend without it still runs every group that does not need it
        probe = {"full_probe": True} if full else {}
        for i, x in enumerate(X.chunks):
            be.distinct_chunk(x[:, j0:j1], keys, counts, off, total, state, first=i == 0, **probe)
        st = state.cpu().numpy()
        over = (st[1] & 1) != 0
        if not over.any():
            break
        # a table at its limit overflows only by a probe chain past 1024 slots, which a larger table need not
        # shorten (keys may share any number of low hash bits): the group runs again with probes bounded by the
        # capacity, which such a table never fills
        at_limit = over & (caps >= limit)
        if full and at_limit.any():
            raise RuntimeError("a key table at its limit overflowed under a full probe")
        full = full or bool(at_limit.any())
        grow = over & ~at_limit
        caps[grow] = np.minimum(caps[grow] * GROWTH, limit)
    occupied, marker = st[0], (st[1] & 2) != 0
    if comm.world > 1:
        (keys, counts, off, total), (_, _, nd), marker = _keytables.merge_ranks(
            be, comm, (keys, counts, off, total), g, X.dtype, occupied, marker)
        occupied = nd.cpu().numpy().astype(np.int64)
    E = int(occupied.sum())
    entries = be.zeros((max(E, 1), 4), torch.float64)
    if E:
        be.mode_compact(keys, counts, off, g, entries[:E])
    col, key = _entry_keys(entries[:E])
    if marker.any():
        mcol = torch.as_tensor(np.flatnonzero(marker), dtype=torch.int64).to(be.device)
        col = torch.cat([col, mcol])
        key = torch.cat([key, torch.full_like(mcol, -1)])
    return col, key


def fit_keys(X):
    """(cat_keys, counts): every column's sorted distinct keys, concatenated (int64 device tensor holding uint64 keys),
    and the number of categories of every column (numpy int64).  Identical on every rank."""
    be, d = X.backend, X.d
    per_col = 16 * min(INITIAL_SLOTS, _keytables.capacity(max(1, X.n_local), X.dtype))
    step = max(1, ENCODE_BUDGET // per_col)      # the same on every rank: columns are grouped by the first tables
    cols, keys = [], []
    for j0 in range(0, d, step):
        j1 = min(d, j0 + step)
        c, k = _group_keys(X, j0, j1)
        cols.append(c + j0)
        keys.append(k)
    col, key = torch.cat(cols), torch.cat(keys)
    order = torch.argsort(key ^ _I64_MIN, stable=True)          # unsigned order of the keys
    col, key = col[order], key[order]
    order = torch.argsort(col, stable=True)
    counts = torch.bincount(col, minlength=d).cpu().numpy().astype(np.int64)
    return key[order].contiguous(), counts


def categories_from_keys(cat_keys, counts, tdt, hdt):
    """The categories of every column as numpy arrays of ``hdt``."""
    vals = key_values(cat_keys.cpu().numpy().view(np.uint64), tdt, hdt)
    return np.split(vals, np.cumsum(counts)[:-1])


def common_dtype(fit_tdt, x_tdt):
    """The dtype in which data of ``x_tdt`` is compared with categories fitted on ``fit_tdt``."""
    if fit_tdt == x_tdt:
        return x_tdt
    t = torch.promote_types(fit_tdt, x_tdt)
    return t if t in _NATIVE else device_dtype(t) or torch.float64


def device_lists(categories, tdt, device):
    """(cat_keys, cat_off, n_cats) on the device for numpy ``categories`` (one sorted array per column) compared as
    data of ``tdt``."""
    keys = [host_keys(c, tdt) for c in categories]
    off = np.concatenate([[0], np.cumsum([len(k) for k in keys])]).astype(np.int64)
    allk = np.concatenate(keys) if keys else np.zeros(0, dtype=np.uint64)
    cat_keys = torch.from_numpy(allk.view(np.int64).copy()).to(device)
    return cat_keys, torch.from_numpy(off).to(device), int(off[-1])


def unknown_buffer(be, d):
    return be.zeros((1 + d + d * _lib.ENCODE_KEEP,), torch.int64)


def unknown_values(X, unknown, tdt, hdt):
    """After the last chunk of a pass, on every rank: None when no rank met an unknown key, else per column the sorted
    unknown values seen (up to ENCODE_KEEP per column and rank)."""
    comm, d = X.comm, X.d
    u = unknown.cpu().numpy()
    total = torch.tensor([float(u[0])], dtype=torch.float64, device=unknown.device)
    comm.allreduce_sum_(total)
    if float(total.item()) == 0.0:
        return None
    per = u[1: 1 + d]
    kept = u[1 + d:].reshape(d, _lib.ENCODE_KEEP)
    mine = [kept[j, : min(int(per[j]), _lib.ENCODE_KEEP)].view(np.uint64) for j in range(d)]
    parts = comm.allgather_obj(mine)
    out = []
    for j in range(d):
        k = np.unique(np.concatenate([p[j] for p in parts]))
        out.append(np.unique(key_values(k, tdt, hdt)) if tdt is not None else np.unique(k.view(np.int64)))
    return out


def encode(X, categories, fit_tdt, layout, out_dtype=torch.int64):
    """One encoding pass over X (DeviceData): the output blocks (codes (n, d) int64, dense (n, W) or (indices, data)
    pairs for CSR) and the unknown values per column (None when there are none)."""
    be, d = X.backend, X.d
    tdt = common_dtype(fit_tdt, X.dtype)
    cat_keys, cat_off, W = device_lists(categories, tdt, be.device)
    unknown = unknown_buffer(be, d)
    blocks = []
    for x in X.chunks:
        x = x if x.dtype == tdt else x.to(tdt)
        n = int(x.shape[0])
        if layout == _lib.ENCODE_CODES:
            o = be.empty((n, d), torch.int64)
            be.encode_chunk(x, cat_keys, cat_off, W, layout, o, unknown)
            blocks.append(o)
        elif layout == _lib.ENCODE_DENSE:
            o = be.empty((n, W), out_dtype)
            be.encode_chunk(x, cat_keys, cat_off, W, layout, o, unknown)
            blocks.append(o)
        else:
            idx = be.empty((n * d,), torch.int64)
            data = be.empty((n * d,), out_dtype)
            be.encode_chunk(x, cat_keys, cat_off, W, layout, data, unknown, indices=idx)
            blocks.append((idx, data))
    hdt = np.result_type(*[np.asarray(c).dtype for c in categories]) if categories else np.dtype("float64")
    return blocks, unknown_values(X, unknown, tdt, hdt), W


def csr_block(idx, data, n, d, W):
    """A device torch.sparse_csr_tensor (n, W) with d nonzeros per row."""
    crow = torch.arange(0, n * d + 1, d, dtype=torch.int64, device=idx.device)
    return torch.sparse_csr_tensor(crow, idx, data, size=(n, W), check_invariants=False)


def decode(codes, categories, backend=None):
    """codes (anything ``intake`` takes with ndim 1 or 2, integer) -> device blocks of category values, and the bad
    codes per column (None when there are none)."""
    C, _ = intake(codes, 2 if len(categories) > 1 else 1, backend)
    be, d = C.backend, C.d
    if C.dtype not in (torch.int32, torch.int64):
        if C.dtype in (torch.float32, torch.float64, torch.bfloat16):
            raise ValueError("codes must be integers, got %s" % C.dtype)
    vals = np.concatenate([np.asarray(c) for c in categories])
    cat_vals = torch.from_numpy(np.ascontiguousarray(vals)).to(be.device)
    off = np.concatenate([[0], np.cumsum([len(c) for c in categories])]).astype(np.int64)
    cat_off = torch.from_numpy(off).to(be.device)
    unknown = unknown_buffer(be, d)
    blocks = []
    for c in C.chunks:
        c = c if c.dtype in (torch.int32, torch.int64) else c.to(torch.int64)
        o = be.empty((int(c.shape[0]), d), cat_vals.dtype)
        be.decode_chunk(c, cat_vals, cat_off, o, unknown)
        blocks.append(o)
    bad = unknown_values(C, unknown, None, None)
    return blocks, bad
