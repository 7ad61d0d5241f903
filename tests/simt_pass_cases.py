"""Cases built to reach the limits of the two CUDA-core passes that serve every shape the tensor path does not take, and a
numpy restatement of the host rules that pick their geometry.

The passes, both in bkm_aux.cu: ``nystrom_kernel`` (SpectralClustering's column sums, COLSUM, and embedding rows, EMBED)
and ``transform_kernel`` (KMeans.transform, euclidean_distances and rbf_kernel).  Each picks its geometry on the host from
(n, d, l or k, k outputs, element size, SM count); the rules are restated below with the source lines they follow, each
taking the SM count as a parameter, so that a test can assert which limits a case reaches.

The data is made of small integers, so that every dot product and norm the kernels form is exact in fp32 and fp64
whatever the order of its terms: the distances are then bit-exact against numpy, the column sums at a large gamma are
exact counts (exp(0) = 1 for a row equal to a keep row, an underflow to 0 for every other pair), and an embedding row
equal to keep row j is exactly W_j / ||W_j||."""
import types

import numpy as np

ES = {"f32": 4, "f64": 8}
BUDGET, LIMIT = 200 * 1024, 227 * 1024    # the shared-memory target and the BKM_EUNSUPPORTED limit: bkm_aux.cu:650-652, 780-787
TPB = 256                                  # transform threads per CTA: bkm_aux.cu:602, 657
TC_MAX_D, TC_MAX_K, TC_EMBED_MAX_K = 64, 256, 64   # tc_supported (bkm_tc.cu:720-725), the EMBED k <= 64 (bkm_api.cu:336)
SMS = (132, 114)                           # H100 SXM and H100 PCIe


def _al(x, a):
    return (x + a - 1) // a * a


def d4_of(d):
    """The SIMT row pitch of the centre pack, d rounded up to a multiple of 4: pack_layout, bkm_common.cuh:151."""
    return (d + 3) // 4 * 4


# ---------------------------------------------------------------------------------------------------------------------
# routing: bkm_transform_chunk, bkm_kernel_colsum_chunk, bkm_nystrom_embed_chunk (bkm_api.cu:247-345)
# ---------------------------------------------------------------------------------------------------------------------
def tc_supported(d, k, dt):
    """bkm_tc.cu:720-725."""
    return dt == "f32" and 1 <= d <= TC_MAX_D and 1 <= k <= TC_MAX_K


def aligned16(base_bytes, ldx):
    """The tensor path's TMA row copies need a 16-byte base and a row pitch of a multiple of 4 floats: launch_tc_transform,
    launch_tc_colsum and launch_tc_embed return BKM_EALIGN otherwise (bkm_tc.cu:846, 859, 876)."""
    return base_bytes % 16 == 0 and ldx % 4 == 0


def route(op, dt, d, l, kw=0, force_simt=False, base_bytes=0, ldx=None):
    """("tc" | "simt", counted): the kernel an entry point runs, and whether bkm_debug_fallback_count counts the call (a
    tensor-path shape whose rows are not 16-byte aligned).  ``op`` is "transform" (l = k centres), "colsum" or "embed"
    (kw outputs)."""
    ldx = d if ldx is None else ldx
    tc = dt == "f32" and tc_supported(d, l, dt) and not force_simt
    if op == "embed":
        tc = tc and kw <= TC_EMBED_MAX_K
    if not tc:
        return "simt", False
    if not aligned16(base_bytes, ldx):
        return "simt", True
    return "tc", False


# ---------------------------------------------------------------------------------------------------------------------
# nystrom_kernel: launch_nystrom, bkm_aux.cu:771-815
# ---------------------------------------------------------------------------------------------------------------------
def nystrom_smem(mode, nw, lb, d, kw, es):
    """smem_of (bkm_aux.cu:776-778): COLSUM's float64 column sums [nw][lb], then per warp the row, lb kernel values and
    kw outputs, each warp's share rounded up to 16 bytes (an odd number of fp32 / fp64 elements gains a pad)."""
    return (_al(nw * lb * 8, 16) if mode == 0 else 0) + nw * _al((d4_of(d) + lb + kw) * es, 16)


def nystrom_geom(mode, n, d, l, kw, dt, sms):
    """The geometry of one launch_nystrom call.  COLSUM (mode 0) passes kw = 0 (bkm_api.cu:319).  The (nw, lb) loop:
    bkm_aux.cu:779-785; the limit: :787; the grid: :788-790; COLSUM's launches and the short last block: :800-801."""
    es = ES[dt]
    kw = kw if mode == 1 else 0
    nw, lb = 8, l
    while nystrom_smem(mode, nw, lb, d, kw, es) > BUDGET:
        if lb > 1024:
            lb = (lb // 2 + 31) // 32 * 32
        elif nw > 1:
            nw >>= 1
        elif lb > 32:
            lb = (lb // 2 + 31) // 32 * 32
        else:
            break
    smem = nystrom_smem(mode, nw, lb, d, kw, es)
    grid = max(1, min((n + nw - 1) // nw, 4 * sms))
    blocks = (l + lb - 1) // lb
    return types.SimpleNamespace(
        nw=nw, lb=lb, smem=smem, ok=smem <= LIMIT, grid=grid, one=l <= lb, blocks=blocks,
        launches=blocks if mode == 0 else 1, last=l - (blocks - 1) * lb,
        turns=(n + grid * nw - 1) // (grid * nw),                 # rows per warp, at most
        last_turn=n - ((n + grid * nw - 1) // (grid * nw) - 1) * grid * nw)   # rows in the last grid-stride turn


def embed_fixed(d, kw):
    """The per-warp width that does not depend on lb: d4 + kw elements (the row and the outputs)."""
    return d4_of(d) + kw


def first_blocked_total(dt, nw=8):
    """The smallest d4 + l + kw at which EMBED at nw warps no longer fits the budget (per warp BUDGET / nw bytes, after the
    16-byte rounding)."""
    t = 1
    while nw * _al(t * ES[dt], 16) <= BUDGET:
        t += 1
    return t


# ---------------------------------------------------------------------------------------------------------------------
# transform_kernel: launch_transform, bkm_aux.cu:643-665
# ---------------------------------------------------------------------------------------------------------------------
def transform_smem(TR, d, es):
    """TR staged rows of d4 + 1 elements, TR norms and 16 bytes: bkm_aux.cu:650-651."""
    return TR * (d4_of(d) + 1) * es + TR * es + 16


def transform_geom(n, d, k, dt, sms):
    """The row tile TR (64 halved while over budget: :649-650), the limit (:652), the tiles and the grid (:653-654)."""
    es = ES[dt]
    TR = 64
    while TR > 1 and transform_smem(TR, d, es) > BUDGET:
        TR >>= 1
    smem = transform_smem(TR, d, es)
    ntiles = (n + TR - 1) // TR
    grid = min(4 * sms, ntiles)
    return types.SimpleNamespace(TR=TR, smem=smem, ok=smem <= LIMIT, ntiles=ntiles, grid=grid,
                                 last_rows=n - (ntiles - 1) * TR, tile_turns=(ntiles + grid - 1) // grid)


def first_d_of_tr(TR, dt):
    """The smallest d (a multiple of 4, so d == d4) at which the row tile is TR: each TR at its first d4."""
    d = 4
    while transform_geom(1, d, 1, dt, 132).TR > TR:
        d += 4
    return d


# ---------------------------------------------------------------------------------------------------------------------
# the cases
# ---------------------------------------------------------------------------------------------------------------------
def d_for_nw(mode, dt, nw, l, kw=0):
    """The smallest d (a multiple of 4) at which (l, kw) runs nw warps per CTA."""
    d = 4
    while nystrom_geom(mode, 1, d, l, kw, dt, 132).nw > nw:
        d += 4
    return d


def _nw1_chain(l):
    """The keep-row blocks the nw = 1 halving walks through from min(l, 1024): bkm_aux.cu:783."""
    b, out = min(l, 1024), []
    while True:
        out.append(b)
        if b <= 32:
            return out
        b = (b // 2 + 31) // 32 * 32


def d_for_lb_at_nw1(dt, l, lb, kw):
    """The smallest d (a multiple of 4) whose nw = 1 halving stops at lb: lb fits one warp's budget, the block before it
    in the chain does not."""
    d = 4
    while True:
        g = nystrom_geom(1, 1, d, l, kw, dt, 132)
        if g.nw == 1 and g.lb <= lb:
            return d if g.lb == lb else None
        d += 4


def short_last_block(dt, r, kw=2):
    """(d, l, kw) of the narrowest EMBED shape whose nw = 1 halving below 1024 leaves a last block of r keep rows."""
    for l in range(r + 1, 1025):
        for lb in _nw1_chain(l)[1:]:
            if l % lb == r:
                d = d_for_lb_at_nw1(dt, l, lb, kw)
                if d is not None:
                    return d, l, kw
    raise AssertionError("no shape")


def lb1024_chain(l):
    """The keep-row blocks of the halving while lb > 1024 (bkm_aux.cu:781): each step takes floor(lb / 2) up to a
    multiple of 32."""
    out = [l]
    while out[-1] > 1024:
        out.append((out[-1] // 2 + 31) // 32 * 32)
    return out


def kw_for_lb1024(dt, l, d=4):
    """The smallest kw at which rows of d features and l keep rows stop the nw = 8 halving at lb = 1024: the block before
    1024 in the chain no longer fits, 1024 does."""
    kw = 1
    while nystrom_geom(1, 1, d, l, kw, dt, 132).lb > 1024:
        kw += 1
    return kw


# lb = 1024 with a last block of 31, 32 and 33 keep rows: l = 31 x 1024 + r halves five times, 31775 -> 15904 -> 7968
# -> 4000 -> 2016 -> 1024, and leaves 31 full blocks and one of r rows.  Rows of 4 features with kw outputs wide enough
# to stop the chain at 1024 keep the keep rows small; W (l x kw, up to 139M fp32 elements) is built on the device.  Each
# row walks the whole W, so these run at n = 1, nw - 1 and nw + 1 only.
LB1024_SHORT = tuple("lb1024_last%d" % r for r in (31, 32, 33))


def embed_shapes(dt):
    """(name, d, l, kw) of the EMBED cases of one precision: the last total d4 + l + kw that fits at nw = 8 and the first
    that does not, with kw = 1, 32, 33 and 65; lb = 1024 with a last block of 1, 31, 32 and 33 keep rows; last blocks of
    31, 32 and 33 keep rows after the halving below 1024 at nw = 1; nw = 4, 2 and 1 through wide rows; and the halving
    below 1024 at nw = 1 from l = 300."""
    t = first_blocked_total(dt)
    out = []
    for kw, d in ((1, 4), (32, 9), (33, 5), (65, 40)):
        l = t - 1 - embed_fixed(d, kw)
        out.append(("fits_kw%d" % kw, d, l, kw))
        out.append(("blocked_kw%d" % kw, d, l + 1, kw))
    # lb = 1024: l = 2049 halves to 1024, and rows this wide keep it from fitting at 2049 but not at 1024
    d = (t - 1024 - 8) // 4 * 4 - 64
    out.append(("lb1024_last1", d, 2049, 8))
    for r in (31, 32, 33):
        l = 31 * 1024 + r
        out.append(("lb1024_last%d" % r, 4, l, kw_for_lb1024(dt, l)))
    for r in (31, 32, 33):
        out.append(("nw1_last%d" % r,) + short_last_block(dt, r))
    for nw in (4, 2, 1):
        out.append(("nw%d" % nw, d_for_nw(1, dt, nw, 300, 3), 300, 3))
    d = d_for_nw(1, dt, 1, 300, 3)
    while nystrom_geom(1, 1, d, 300, 3, dt, 132).lb == 300:
        d += 4
    out.append(("nw1_halved", d, 300, 3))
    return out


def colsum_shapes(dt):
    """(name, d, l) of the COLSUM cases: one launch, two launches, many launches, a last block of exactly one keep row
    (lb = 1024 for fp64, 2048 for fp32), nw = 4, 2 and 1 through wide rows, and nw = 1 with two launches."""
    two = 1700 if dt == "f64" else 4000
    last1 = 2049 if dt == "f64" else 4097
    out = [("one", 5, 300), ("two", 4, two), ("many", 4, 20000), ("last1", 4, last1)]
    for nw in (4, 2, 1):
        out.append(("nw%d" % nw, d_for_nw(0, dt, nw, 300), 300))
    d = d_for_nw(0, dt, 1, 300)
    while nystrom_geom(0, 1, d, 300, 0, dt, 132).lb == 300:
        d += 4
    out.append(("nw1_two", d, 300))
    return out


def row_counts(nw, sms, big=True):
    """n = 1, nw - 1, nw + 1, and one row past a full grid turn of 4 SMs x nw rows: the grid walks a second turn that
    holds one row."""
    ns = sorted({1, max(nw - 1, 1), nw + 1})
    if big:
        ns.append(4 * sms * nw + 1)
    return ns


def transform_shapes(dt):
    """(name, d, k) of the transform cases: every row tile TR = 64 ... 1 at its first d4, once with d = d4 and once with
    d = d4 - 3 (the same tile, a padded pack row); k = 7 and 37 (k % 4 != 0)."""
    out = []
    for TR in (64, 32, 16, 8, 4, 2, 1):
        d = first_d_of_tr(TR, dt)
        out.append(("TR%d" % TR, d, 7 if TR > 4 else 37))
        if d > 4:
            out.append(("TR%d_pad" % TR, d - 3, 37 if TR > 4 else 7))
    return out


def transform_rows(TR, sms):
    """More tiles than the 4 x SMs CTAs of the grid, and a last tile of one row."""
    return TR * (4 * sms + 2) + 1


# ---------------------------------------------------------------------------------------------------------------------
# exact data
# ---------------------------------------------------------------------------------------------------------------------
GAMMA_COUNT = 1000.0        # exp(-gamma y) underflows to 0 in fp32 and fp64 for every integer y >= 1
GAMMA_LO, GAMMA_HI = 745.12, 745.14      # either side of the NaN threshold 745.13 (bkm_aux.cu:741) at m = 1
COPY, NEAR, ODD = 0, 1, 2   # row kinds: a keep row (m = 0), a keep row +- e_c (m = 1), all coordinates odd (m >= d)


def keep_radius(l, d):
    """R with (2R + 1)^d >= 8 l: enough even integers in [-2R, 2R] for l distinct keep rows."""
    R = 1
    while (2 * R + 1) ** min(d, 64) < 8 * l:
        R += 1
    return R


def keep_rows(l, d, seed):
    """l distinct keep rows (int8) of even integers in [-2R, 2R]: two distinct keep rows lie at a squared distance >= 4."""
    rng = np.random.RandomState(seed)
    R = keep_radius(l, d)
    K = np.unique((2 * rng.randint(-R, R + 1, (2 * l, d))).astype(np.int8), axis=0)
    assert len(K) >= l
    return K[rng.permutation(len(K))[:l]]


def exact_rows(keep, n, seed):
    """n rows of three kinds over the keep rows ``keep`` (int8): COPY rows equal keep row j, NEAR rows keep row j +- 1 in
    one coordinate (their squared distance to the nearest keep row is exactly 1: every keep row is even), ODD rows have
    every coordinate odd (at least d from every keep row).  Rows 0 and n - 1 are copies of keep rows l - 1 and 0.
    Returns (X int8, kind, j)."""
    rng = np.random.RandomState(seed)
    l, d = keep.shape
    kind = rng.choice([COPY, NEAR, ODD], n, p=[0.6, 0.25, 0.15])
    j = rng.randint(0, l, n)
    kind[0] = kind[-1] = COPY
    j[0], j[-1] = l - 1, 0
    X = keep[j].copy()
    near = np.nonzero(kind == NEAR)[0]
    X[near, rng.randint(0, d, len(near))] += rng.choice([-1, 1], len(near)).astype(np.int8)
    odd = np.nonzero(kind == ODD)[0]
    R = keep_radius(l, d)
    X[odd] = (2 * rng.randint(-R, R + 1, (len(odd), d)) + 1).astype(np.int8)
    return X, kind, j


def one_hot_parts(l, kw, seed):
    """(column, sign) of each row of a signed one-hot W (l, kw)."""
    rng = np.random.RandomState(seed)
    return rng.randint(0, kw, l), rng.choice([-1.0, 1.0], l)


def signed_one_hot(l, kw, seed):
    """W (l, kw): row j is +-1 in one column, 0 elsewhere."""
    col, sgn = one_hot_parts(l, kw, seed)
    W = np.zeros((l, kw))
    W[np.arange(l), col] = sgn
    return W


def exact_bound(R, d):
    """The largest |squared distance| or norm the exact data can form: every coordinate difference is at most 4R + 1."""
    return d * (4 * R + 1) ** 2
