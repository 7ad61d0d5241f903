"""The fp32 tensor-core chunk kernel's variants without a GPU: the layout query (bkm_debug_tc_layout) over every supported
shape, the ring depths S it gives (the wrap points tests/test_gpu_tc_ring.py aims at), and the row-count guard of the
transform and Nystrom entry points."""
import ctypes

import pytest

ARGMIN, XFORM, COLSUM, EMBED = 0, 1, 2, 3          # TcEpi of bkm_tc.cu
SMEM_CAP = 227 * 1024                              # dynamic shared memory of one H100 CTA
SLOT_BYTES = 64 * 64 * 4                           # one ring slot: a 64-row tile of up to 64 fp32 features
EUNSUPPORTED, EINVAL = -3, -1


@pytest.fixture(scope="module")
def lib():
    from dask_ml_b200 import _lib

    return _lib.load()


def _mma_n(k):
    cols = (k + 15) // 16 * 16
    return next(n for n in (16, 32, 64, 128, 256) if cols <= n)


def _variants():
    """(epi, mstep, kw) of every variant a chunk call can run."""
    yield ARGMIN, 1, 0
    yield ARGMIN, 0, 0
    yield XFORM, 0, 0
    yield COLSUM, 0, 0
    for kw in range(1, 65):
        yield EMBED, 0, kw


def _expected_s(epi, mstep, kw, n):
    """The ring depths of an H100: the M-step at N = 256 keeps 5 slots (an odd count, which the turn order allows), the
    embedding at N = 256 gives up slots to its staged weights as kw grows, everything else has the full 8."""
    if epi == ARGMIN and mstep and n == 256:
        return 5
    if epi == EMBED and n == 256 and kw > 56:
        return 4
    if epi == EMBED and n == 256 and kw > 24:
        return 6
    return 8


def test_layout_of_every_supported_shape(lib):
    out = (ctypes.c_int * 4)()
    seen = set()
    for epi, mstep, kw in _variants():
        for k in range(1, 257):
            n = _mma_n(k)
            want_s = _expected_s(epi, mstep, kw, n)
            for d in range(1, 65):
                assert lib.bkm_debug_tc_layout(d, k, epi, mstep, kw, out) == 0, (d, k, epi, mstep, kw)
                ks, nn, s, smem = out
                assert ks == (d + 15) // 16 and nn == n, (d, k, epi, mstep, kw, list(out))
                assert 4 <= s <= 8 and (mstep or s % 2 == 0), (d, k, epi, mstep, kw, s)
                assert s * SLOT_BYTES < smem <= SMEM_CAP, (d, k, epi, mstep, kw, smem)
                assert s == want_s, (d, k, epi, mstep, kw, s)
                seen.add((epi, mstep, n, s))
    # the table the GPU ring tests rely on
    assert (ARGMIN, 1, 256, 5) in seen and (EMBED, 0, 256, 4) in seen and (EMBED, 0, 256, 6) in seen
    for kw, s in ((1, 8), (7, 8), (24, 8), (25, 6), (32, 6), (33, 6), (56, 6), (57, 4), (64, 4)):
        assert lib.bkm_debug_tc_layout(64, 256, EMBED, 0, kw, out) == 0 and out[2] == s, (kw, list(out))


@pytest.mark.parametrize("d,k,epi,mstep,kw,rc", [
    (65, 10, ARGMIN, 0, 0, EUNSUPPORTED),         # d > 64
    (0, 10, XFORM, 0, 0, EUNSUPPORTED),
    (16, 257, COLSUM, 0, 0, EUNSUPPORTED),        # k > 256
    (16, 0, ARGMIN, 1, 0, EUNSUPPORTED),
    (16, 100, EMBED, 0, 65, EUNSUPPORTED),        # more than 64 embedding outputs
    (16, 100, EMBED, 0, 0, EUNSUPPORTED),
    (16, 100, 4, 0, 0, EINVAL),                   # no such epilogue
    (16, 100, XFORM, 1, 0, EINVAL),               # the M-step belongs to the arg-min epilogue only
])
def test_layout_refusals(lib, d, k, epi, mstep, kw, rc):
    out = (ctypes.c_int * 4)(-7, -7, -7, -7)
    assert lib.bkm_debug_tc_layout(d, k, epi, mstep, kw, out) == rc
    assert list(out) == [-7] * 4
    assert lib.bkm_debug_tc_layout(16, 100, ARGMIN, 0, 0, None) == EINVAL


def test_entry_points_refuse_chunks_beyond_32_bit_row_indices(lib):
    """n = 2^31 rows would give the tensor path negative TMA row coordinates (rows the copy engine reads as zeros):
    refused before any pointer is read or kernel launched (X is null: without the check the calls stop at it with
    BKM_EINVAL)."""
    n = 1 << 31
    dummy = ctypes.c_void_p(0x1000)
    null = ctypes.c_void_p(0)
    assert lib.bkm_transform_chunk(null, n, 8, 8, 0, dummy, 4, dummy, 4, 0, 0.0, 0, null) == EUNSUPPORTED
    assert lib.bkm_kernel_colsum_chunk(null, n, 8, 8, 0, dummy, 4, 0.5, dummy, dummy, 1 << 30, 0, null) == EUNSUPPORTED
    assert lib.bkm_nystrom_embed_chunk(null, n, 8, 8, 0, dummy, 4, 0.5, dummy, 2, dummy, 2, 0, null) == EUNSUPPORTED
    # one row fewer is a valid row count: the same calls reach the null X
    n -= 1
    assert lib.bkm_transform_chunk(null, n, 8, 8, 0, dummy, 4, dummy, 4, 0, 0.0, 0, null) == EINVAL
    assert lib.bkm_kernel_colsum_chunk(null, n, 8, 8, 0, dummy, 4, 0.5, dummy, dummy, 1 << 30, 0, null) == EINVAL
    assert lib.bkm_nystrom_embed_chunk(null, n, 8, 8, 0, dummy, 4, 0.5, dummy, 2, dummy, 2, 0, null) == EINVAL
