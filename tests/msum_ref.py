"""Order-exact references of the M-step sums (numpy, CPU).

The fused kernels promise bit-reproducible sums because every partial sum is formed in a fixed order.  This module
restates those orders as executable references that take the kernel's own labels, so that a test can demand the
kernel's sums bit for bit:

* family 1 (``tc_chunk_kernel``, bkm_tc.cu): ``grid = max(1, min(ceil(n / 64), sm_count))`` CTAs; CTA b owns the 64-row
  tiles b, b + grid, ...; its partial ``P[b][c][f]`` is the fp32 sum, from +0.0f, of ``X[r][f]`` over its rows with
  label c, in increasing row order (deferred rows are left out: the float64 re-check adds them later).
* family 3 (``rowpass_mstep_kernel``, bkm_rowpass.cu): rows are cut into row blocks of ``tiles_per_block`` 4096-row
  tiles; ``P[rb][c][f]`` is the fp32 sum of the rows of block rb with label c, in row order (bf16 widened exactly).
* ``reduce_partials_kernel`` (bkm_aux.cu): chain y in 0..7 adds ``(double)P[g]`` for g = y, y + 8, ... in float64; the
  total is ``((s0 + s1) + ...) + s7``; the output is that total (first chunk) or ``old + total``.

Every sequential sum is written with its order explicit: a loop over the rank within each segment, vectorised across
segments (np.sum / reduceat leave their association unspecified).
"""
import numpy as np

TC_TILE = 64          # family 1: rows per warpgroup tile (wgmma M)
RP_TILE = 4096        # family 3: rows per binning tile of the label-indexed row pass
CHAINS = 8            # reduce_partials: independent float64 chains per output


def sequential_sums(X32, seg, nseg, rank_key=None):
    """fp32 sums ``S[s] = ((0 + x_a) + x_b) + ...`` of the rows of X32 with ``seg == s`` (``seg < 0``: left out), in
    increasing order of ``rank_key`` (default: the row index), one rounded fp32 addition per row."""
    X32 = np.asarray(X32, dtype=np.float32)
    d = X32.shape[1]
    seg = np.asarray(seg, dtype=np.int64)
    keep = np.nonzero(seg >= 0)[0]
    key = keep if rank_key is None else np.asarray(rank_key)[keep]
    order = keep[np.lexsort((key, seg[keep]))]              # by segment, then by key
    cnt = np.bincount(seg[order], minlength=nseg)
    start = np.concatenate(([0], np.cumsum(cnt)[:-1]))
    by_len = np.argsort(-cnt, kind="stable")                # segments by decreasing length
    neg_len = -cnt[by_len]
    out = np.zeros((nseg, d), dtype=np.float32)
    for r in range(int(cnt.max()) if nseg else 0):
        act = by_len[:np.searchsorted(neg_len, -r, side="left")]      # the segments with more than r rows
        out[act] += X32[order[start[act] + r]]
    return out


# ------------------------------------------------------------------------------------------------ family 1
def tc_grid(n, sm_count):
    """CTAs of the fp32 fused E+M kernel (tc_grid in bkm_tc.cu)."""
    return max(1, min(-(-n // TC_TILE), sm_count))


def tc_partials(X32, labels, k, sm_count, keep=None, grid=None, rank_key=None):
    """Per-CTA partials ``P[b][c][f]`` of family 1 for the kernel's labels; ``keep`` masks out deferred rows.
    ``grid`` and ``rank_key`` override the kernel's grid and row order (to show that a changed order is visible)."""
    n, d = X32.shape
    g = tc_grid(n, sm_count) if grid is None else grid
    seg = (np.arange(n) // TC_TILE) % g * k + np.asarray(labels, dtype=np.int64)
    if keep is not None:
        seg = np.where(keep, seg, -1)
    return sequential_sums(X32, seg, g * k, rank_key).reshape(g, k, d)


# ------------------------------------------------------------------------------------------------ family 3
def tc2_slices(k, d):
    """DS of tc2_geom (bkm_common.cuh): cluster slices so that a slice's fp32 sums fit one CTA."""
    dpad = 32 if d <= 32 else (64 if d <= 64 else 128)
    ds = 1
    while -(-k // ds) * dpad * 4 + -(-k // ds) * 4 + 40 * 1024 > 210 * 1024:
        ds <<= 1
    return ds


def rowpass_blocks(n, k, d, sm_count):
    """(RB, tiles_per_block) of make_rp_cfg (bkm_rowpass.cu), with psum_slots = max(1, sm_count // DS) (ws_layout)."""
    ds = tc2_slices(k, d)
    ntiles = -(-n // RP_TILE)
    rb = max(1, sm_count // ds)                             # (the psum_slots cap is the same number)
    if rb > ntiles:
        rb = ntiles if ntiles > 0 else 1
    tpb = -(-ntiles // rb)
    return -(-ntiles // tpb), tpb


def rowpass_partials(X32, labels, k, sm_count):
    """Per-row-block partials ``P[rb][c][f]`` of family 3 (X32: the bf16 rows widened to fp32)."""
    n, d = X32.shape
    rb, tpb = rowpass_blocks(n, k, d, sm_count)
    seg = np.arange(n) // RP_TILE // tpb * k + np.asarray(labels, dtype=np.int64)
    return sequential_sums(X32, seg, rb * k).reshape(rb, k, d)


# ------------------------------------------------------------------------------------------------ reduce_partials
def reduce_partials(P, first=True, old=None, fold=tuple(range(CHAINS))):
    """float64 fold of the partials ``P[g]`` (any shape after the first axis) as reduce_partials_kernel does it.
    ``fold`` is the order in which the chain sums are added (to show that a changed order is visible)."""
    P = np.asarray(P)
    G = P.shape[0]
    flat = P.reshape(G, -1)
    chains = np.zeros((CHAINS, flat.shape[1]), dtype=np.float64)
    for g in range(G):
        chains[g % CHAINS] += flat[g].astype(np.float64)
    t = chains[fold[0]].copy()
    for y in fold[1:]:
        t += chains[y]
    t = t.reshape(P.shape[1:])
    return t if first else np.asarray(old, dtype=np.float64) + t


# ------------------------------------------------------------------------------------------------ designed data
def zero_features(d):
    """Features whose centre coordinate is 0 (every third one): their rows carry only noise."""
    return np.arange(d) % 3 == 2


def lattice_centres(k, d, spacing=32.0, offset=100.0):
    """k float64 centres, pairwise at least ``spacing`` apart: the features that are not zero features hold
    ``offset + spacing * digit`` (the base-B digits of the cluster index), the zero features hold 0."""
    off = np.nonzero(~zero_features(d))[0]
    base = 2
    while base ** len(off) < k:
        base += 1
    C = np.zeros((k, d))
    C[:, off] = offset
    c = np.arange(k)
    for f in off:
        C[:, f] += spacing * (c % base)
        c = c // base
    return C


def designed_rows(pattern, C, seed):
    """``X[r] = C[pattern[r]] + noise`` in float64, order-sensitive: the noise of row r is ``2^-u * U(-1, 1)`` in the
    offset features (u uniform in [0, 12]: an offset of ~100 plus noise down to 2^-12 fills the low bits of fp32 sums)
    and ``2^-v * U(-1, 1)`` in the zero features (v uniform in [0, 60]: partials of very different magnitudes, so that
    even the float64 fold rounds).  |noise| <= 1 per feature keeps every row nearest to its own centre."""
    rng = np.random.RandomState(seed)
    pattern = np.asarray(pattern, dtype=np.int64)
    n, d = len(pattern), C.shape[1]
    u = rng.uniform(0, 12, size=(n, 1))
    v = rng.uniform(0, 60, size=(n, 1))
    scale = np.where(zero_features(d)[None, :], 2.0 ** -v, 2.0 ** -u)
    return C[pattern] + scale * rng.uniform(-1, 1, size=(n, d))
