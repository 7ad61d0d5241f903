"""The large-shape tensor path (bf16 rows, d <= 128, k <= 4096: bkm_tc2.cu, bkm_rowpass.cu) restated on the host, the
cases that reach its limits, and data designed so that every distance it forms is exact.

Host rules, each with the source it follows; every rule takes the SM count as a parameter:

* ``tc2_geom`` (bkm_common.cuh): S = ceil(k / 256) centre slices of NS = ceil(ceil(k / S) / 16) * 16 columns, KB
  64-feature blocks, DS cluster slices of the M-step row pass (msum_ref.tc2_slices).
* ``mma_n`` (bkm_wgmma.cuh): the wgmma width N of a slice, 16 / 32 / 64 / 128 / 256.
* ``make_cfg2`` (bkm_tc2.cu): G = SMs // S row-tile groups (SMs - G S of them idle), the shared-memory carve-up and
  its 227 KB limit; ``launch_tc2`` clamps G to the row tiles, launches the slice combine on min(ceil(n / 256), 8 SMs)
  CTAs and the float64 re-check on 4 SMs CTAs of 16 deferred rows per turn.
* the tile dealing of ``tc2_assign_kernel``: CTA b serves slice b % S for group b // S; the group's tile lt holds
  rows (group + lt G) * 64 ...; warpgroup lt & 1 takes it in pair lt >> 1.
* ``make_rp_cfg`` / ``launch_rowpass_*`` (bkm_rowpass.cu): CS = DS, NB = 16 CS buckets (<= RP_MAXB = 256), KL,
  RB / tiles_per_block (msum_ref.rowpass_blocks), the binning grid min(ntiles, 4 SMs) and the distance grid
  min(ceil(n / 8), 8 SMs).
* ``ws_layout`` (bkm_common.cuh) for bf16 rows: the slice records, the label buffer and the bins.

The designed data (``design``): centre j holds the bits of j in B spread-out features, so centres are distinct 0/1
vectors.  A few centres are rewritten into pairs (a, b):

* "pair": c_b = c_a + e_E + 2^-9 e_T (one extra feature E, one tilt feature T).  The row c_a + e_E / 2 + t e_T is
  1/4 + O(2^-18) from both and >= 1 + 1/4 from every other centre; t = 0 makes a the winner by 2^-18, t = 2^-9 makes b
  the winner by 2^-18, t = 2^-10 is an exact tie.
* "dup": c_b = c_a; the row c_a ties exactly at distance 0.

Every row value is 0, 1/2, 1, 2^-10 or 2^-9 and every centre value 0, 1 or 2^-9, all exact in bf16, and -2 c is its
own bf16 ``hi`` (lo = 0).  Each product x_i (-2 c_i) is a multiple of 2^-18, and every partial sum of them, as well as
||c||^2 = popcount + 2^-18 and the distance ||c||^2 - 2 x.c, is a multiple of 2^-18 below 2^6 in magnitude: 24
significant bits, exact in fp32 whatever order (and whatever alignment window of at least 24 bits) the tensor cores
accumulate in.  So the kernel's distances equal the float64 ones: a gap of 2^-18 lies inside the near-tie bound
tau (||x||^2 + max ||c||^2) > 2^-17 and is deferred for certain, an exact tie is deferred and goes to the lower index,
and every other gap is >= 1, far outside the bound (< 1e-3).
"""
import math

import numpy as np

import msum_ref as mr

T2_BM = 64             # rows per warpgroup tile
R2_ROWS = 16           # deferred rows per re-check CTA and turn
RP_TILE = 4096         # rows per binning tile of the row pass
RP_NW = 16             # warps of a row-pass CTA
RP_MAXB = 256          # bucket bound of the binning kernel (cntw, base_s, 257-entry tile_off rows)
SMEM_MAX = 227 * 1024
SM_COUNTS = (132, 114)                 # H100 SXM and H100 PCIe
LAYOUT_FIELDS = ("S", "NS", "N", "KB", "KS", "G", "smem", "combine_grid", "recheck_grid", "DS", "NB", "KL", "RB",
                 "tiles_per_block", "bin_grid", "dist_grid", "FPL", "rp_smem")
TILT = 2.0 ** -9


def _cdiv(a, b):
    return -(-a // b)


def _align(x, a):
    return _cdiv(x, a) * a


def tau(d):
    """tau_for(d, BF16, 0, family 3) of bkm_api.cu, in float32 as the library forms it."""
    f = np.float32
    eps = f(1.0) / f(16777216.0)
    return float(f(1.0) / f(131072.0) + (f(8.0) * np.sqrt(f(2.0) * f((d + 7) // 8), dtype=f) + f(16.0)) * eps)


def mma_n(cols):
    """wg::mma_n (bkm_wgmma.cuh)."""
    return 16 if cols <= 16 else 32 if cols <= 32 else 64 if cols <= 64 else 128 if cols <= 128 else 256


def tc2_geom(k, d):
    """Tc2Geom of tc2_geom (bkm_common.cuh)."""
    S = _cdiv(k, 256)
    per = _cdiv(k, S)
    NS = _cdiv(per, 16) * 16
    KB = _cdiv(d, 64)
    return dict(S=S, per=per, NS=NS, kp2=S * NS, KB=KB, dk2=KB * 64, DS=mr.tc2_slices(k, d))


def make_cfg2(d, k, sms):
    """Tc2Cfg of make_cfg2 (bkm_tc2.cu) before the launch clamps G; None where the shape cannot run."""
    g = tc2_geom(k, d)
    if g["S"] > sms:
        return None
    N = mma_n(g["NS"])
    o = 0
    off_b = o; o += 2 * g["KB"] * N * 128            # (hi, lo) x K-blocks of the slice
    off_x = o; o += 2 * 2 * g["KB"] * T2_BM * 128     # 2 warpgroups x 2 stages
    off_cn = o; o += N * 4
    off_xn = o; o += 2 * 2 * T2_BM * 4
    if o > SMEM_MAX:
        return None
    return dict(S=g["S"], NS=g["NS"], N=N, KB=g["KB"], KS=_cdiv(d, 16), G=sms // g["S"], off_b=off_b, off_x=off_x,
                off_cn=off_cn, off_xn=off_xn, total=o)


def ws_layout(n, d, k, sms):
    """ws_layout (bkm_common.cuh) of a bf16 call: the offsets of the family-3 buffers and the total."""
    g = tc2_geom(k, d)
    slot = k * d * 4
    part_slots = sms * 8
    psum_slots = max(1, sms // g["DS"])
    W = {}
    o = 0
    W["bal"] = o; o = _align(o + 16 + 4096, 256)
    W["psum"] = o; o = _align(o + max(psum_slots * slot, k * d * 8), 256)
    W["pcnt"] = o; o = _align(o + part_slots * k * 4, 256)
    W["pin"] = o; o = _align(o + part_slots * 8, 256)
    W["flag"] = o; o = _align(o + 256, 256)
    W["defer"] = o; o = _align(o + n * 4, 256)
    W["rec"] = o
    if g["S"] > 1:
        o = _align(o + g["S"] * n * 16, 256)
    W["lab"] = o; o = _align(o + n * 4, 256)
    ntile = _cdiv(n, RP_TILE)
    W["bin"] = o; o = _align(o + ntile * RP_TILE * 4, 256)
    W["binoff"] = o; o = _align(o + ntile * (RP_MAXB + 1) * 4, 256)
    W["total"] = o
    W["psum_slots"], W["part_slots"] = psum_slots, part_slots
    return W


def layout(d, k, n, sms):
    """The 18 numbers bkm_debug_tc2_layout returns (LAYOUT_FIELDS), restated; None where the shape cannot run."""
    c = make_cfg2(d, k, sms)
    if c is None:
        return None
    G = max(1, min(c["G"], _cdiv(n, T2_BM)))                       # launch_tc2's clamp to the row tiles
    DS = mr.tc2_slices(k, d)
    NB = DS * RP_NW
    if NB > RP_MAXB:
        return None
    fpl = 1 if d <= 32 else 2 if d <= 64 else 4
    KL = _cdiv(k, DS)
    rp_smem = KL * 32 * fpl * 4 + _align(KL * 4, 16)
    if rp_smem > SMEM_MAX:
        return None
    RB, tpb = mr.rowpass_blocks(n, k, d, sms)
    ntiles = _cdiv(n, RP_TILE)
    dist = max(1, min(_cdiv(n, 8), 8 * sms, ws_layout(n, d, k, sms)["part_slots"]))
    return (c["S"], c["NS"], c["N"], c["KB"], c["KS"], G, c["total"], min(_cdiv(n, 256), 8 * sms), 4 * sms, DS, NB, KL,
            RB, tpb, min(ntiles, 4 * sms), dist, fpl, rp_smem)


def lay(d, k, n, sms):
    """layout() as a dict."""
    t = layout(d, k, n, sms)
    return None if t is None else dict(zip(LAYOUT_FIELDS, t))


def dealing(d, k, n, sms):
    """[(cta, slice, group, lt, warpgroup, pair, row0)] of every tile tc2_assign_kernel stages."""
    L = lay(d, k, n, sms)
    S, G = L["S"], L["G"]
    ntiles = _cdiv(n, T2_BM)
    out = []
    for b in range(G * S):
        s, grp = b % S, b // S
        my_tiles = _cdiv(ntiles - grp, G) if grp < ntiles else 0
        for lt in range(my_tiles):
            out.append((b, s, grp, lt, lt & 1, lt >> 1, (grp + lt * G) * T2_BM))
    return out


# ------------------------------------------------------------------------------------------------ cases
def ds_transitions(dpad, kmax=4096):
    """k where DS doubles at the padded width dpad (32 / 64 / 128): DS(k - 1) < DS(k)."""
    return [k for k in range(2, kmax + 1) if mr.tc2_slices(k, dpad) > mr.tc2_slices(k - 1, dpad)]


def _case(cid, d, k, n, n_defer=None, tags=()):
    return dict(id=cid, d=d, k=k, n=n, n_defer=n_defer, tags=tuple(tags))


def cases(sms):
    """Integer cases (d, k, n) that reach the path's limits on ``sms`` SMs; ``tags`` name the limits a case is for."""
    out = []
    for k in (1, 16, 17, 32, 33, 40, 64, 65, 128, 129, 256):                      # every MMA width, padded and full
        out.append(_case("mma-k%d" % k, 128, k, 3000, tags=("N%d" % mma_n(tc2_geom(k, 128)["NS"]),)))
    for S in range(1, 17):                                                          # every slice count
        for k in ((256 * (S - 1) + 1,) if S > 1 else ()) + (256 * S,):
            # n > k + the special rows: a far row, decided on the tensor path, at every column of every slice
            out.append(_case("S%d-k%d" % (S, k), 64 if S % 2 else 128, k, k + 800 + 37 * S, tags=("S%d" % S,)))
    for d in (1, 8, 9, 16, 63, 64, 65, 100, 127, 128):                               # K-blocks and partial K-steps
        out.append(_case("d%d" % d, d, min(300, 2 ** max(1, d - 2)), 2500, tags=("d%d" % d,)))
    for dpad in (32, 64, 128):                                                      # DS transitions at every FPL
        for kt in ds_transitions(dpad):
            for k in (kt - 1, kt):
                out.append(_case("ds%d-k%d" % (dpad, k), dpad, k, 9000, tags=("DS%d" % mr.tc2_slices(k, dpad),)))
    for d, k in ((128, 1280), (40, 200)):                                           # row counts around the groups
        G = lay(d, k, 1 << 30, sms)["G"]
        rows = {"n1": 1, "n63": 63, "tiles=G-1": 64 * (G - 1) - 5, "tiles=G": 64 * G - 5, "tiles=G+1": 64 * (G + 1) - 5,
                "tiles=2G": 64 * 2 * G - 5, "tiles=2G+1": 64 * (2 * G + 1) - 5}
        for name, n in rows.items():           # the single row of n1 is one the tensor path decides
            out.append(_case("rows-d%d-k%d-%s" % (d, k, name), d, k, n, n_defer=0 if n == 1 else None, tags=(name,)))
    out.append(_case("bin-turn2", 8, 64, 4 * sms * RP_TILE + 1, tags=("bin-turn2",)))
    R = 4 * sms
    for S_k in (200, 4096):               # S = 1, and S = 16 with a duplicate at every re-check reduction level
        for name, nd in (("0", 0), ("1", 1), ("16", 16), ("17", 17), ("16R-1", 16 * R - 1), ("16R", 16 * R),
                         ("16R+1", 16 * R + 1)):
            out.append(_case("defer%s-k%d" % (name, S_k), 64, S_k, max(4096, 2 * nd + 1000), n_defer=nd,
                             tags=("defer" + name,)))
    return out


# ------------------------------------------------------------------------------------------------ designed data
def features(d, k):
    """(bit features, E, T) positions spread over [0, d): the last one is feature d - 1, so the bits reach the last
    K-block and the partial last K-step.  E and T are None where d leaves no room for them."""
    B = max(1, math.ceil(math.log2(k))) if k > 1 else 1
    assert 2 ** B >= k and d >= B, (d, k)
    m = B + 2 if d >= B + 2 else B
    pos = np.unique(np.round(np.linspace(0, d - 1, m)).astype(int)) if m > 1 else np.array([d - 1])
    assert len(pos) == m
    if m == B:
        return pos, None, None
    return pos[:B], int(pos[B]), int(pos[B + 1])


def _pair_plan(k, d):
    """[(a, b, kind)] of the pairs of a (d, k) design: pairs at the MMA fragment neighbours inside every slice,
    between slice 0 and the last column, across every slice border, and the duplicate centres of the re-check's
    reduction levels.  Every a and every b appear once, and no column is both: the first of two pairs that want the same
    column keeps it (at k = 3841 the last slice's single column goes to the pair with slice 0, not to the border pair
    (3839, 3840))."""
    g = tc2_geom(k, d)
    NS, S, N = g["NS"], g["S"], mma_n(g["NS"])
    want = []
    for s in range(S):
        base = s * NS
        sh = 2 * (s % 4)        # offsets move between slices: a column one slice bit away from a pair is free
        for o, p in ((4 + sh, 5 + sh), (9 + sh, 10 + sh), (16 + sh, 24 + sh), (N // 2 - 1, N // 2), (NS - 3, NS - 2)):
            want.append((base + o, base + p, "pair"))
    if S > 1:
        want.append((1, k - 1, "pair"))                                 # slice 0 and the last slice's last column
    for s in range(1, S):
        want.append((s * NS - 1, s * NS, "pair"))                       # straddles the slice border
    for a, b in ((48, 49), (50, 82), (52, 308), (54, 3894)):             # same warp / other warps / same thread
        want.append((a, b, "dup"))
    used, plan = set(), []
    for a, b, kind in want:
        if 0 <= a < b < k and a not in used and b not in used:
            used |= {a, b}
            plan.append((a, b, kind))
    return plan


def centres(k, d):
    """(C float64 (k, d), plan, bits, E, T) of the design."""
    bits, E, T = features(d, k)
    C = np.zeros((k, d))
    for i, f in enumerate(bits):
        C[:, f] = (np.arange(k) >> i) & 1
    plan = [p for p in _pair_plan(k, d) if E is not None or p[2] == "dup"]
    for a, b, kind in plan:
        C[b] = C[a]
        if kind == "pair":
            C[b, E] = 1.0
            C[b, T] = TILT
    return C, plan, bits, E, T


def special_rows(C, plan, bits, E, T, NS):
    """[(x, kind)] of the rows built on the pairs: the near-ties in either order and the exact tie of every pair,
    the exact tie of every duplicate, and rows that win in one slice while another slice holds a near-tie."""
    k = C.shape[0]
    rows = []
    pair_cols = {c for a, b, _ in plan for c in (a, b)}
    for a, b, kind in plan:
        if kind == "dup":
            rows.append((C[a].copy(), "dup"))
            continue
        for t, name in ((0.0, "near-a"), (TILT, "near-b"), (TILT / 2, "equal")):
            x = C[a].copy()
            x[E] = 0.5
            x[T] = t
            rows.append((x, name))
        # inner-losing: the winner w is one bit away from a in another slice, not in a pair
        for i in range(len(bits)):
            w = a ^ (1 << i)
            if w < k and w // NS != a // NS and w not in pair_cols:
                x = C[w].copy()
                x[E] = 0.5
                rows.append((x, "inner-losing"))
                break
    return rows


def decide(X, C, k, d, NS, S):
    """(label, deferred) of every row of X under the kernel's rules with exact arithmetic: the lowest-index float64
    arg-min, and the near-tie test of the single slice (S = 1) or of the slice combine (S > 1)."""
    X = np.asarray(X, dtype=np.float64)
    cn = (C * C).sum(1)
    e = cn[None, :] - 2.0 * (X @ C.T)                      # exact: every term is a multiple of 2^-18 below 2^6
    lab = e.argmin(1)
    bound = tau(d) * ((X * X).sum(1) + cn.max())
    if k == 1:
        return lab, np.zeros(len(X), dtype=bool)
    mins, ties = [], []
    for s in range(S):
        es = e[:, s * NS:min((s + 1) * NS, k)]
        two = np.sort(es, axis=1)[:, :2] if es.shape[1] > 1 else np.concatenate([es, np.full_like(es, 3e38)], 1)
        mins.append(two[:, 0])
        ties.append(~(two[:, 1] > two[:, 0] + bound))
    mins, ties = np.stack(mins, 1), np.stack(ties, 1)
    win = mins.argmin(1)                                   # first slice of the smallest minimum
    best = mins[np.arange(len(X)), win]
    if S == 1:
        deferred = ties[:, 0]
    else:
        second = np.sort(mins, axis=1)[:, 1]
        deferred = ties[np.arange(len(X)), win] | ~(second - best > bound)
    return lab, deferred


def design(d, k, n, seed, n_defer=None):
    """Designed case: (X float64 (n, d), C float64 (k, d), labels, deferred mask, kinds per row).  Special rows
    (``special_rows``) sit at spread positions, the last row among them; the other rows are far rows, centres: every
    column but the duplicates' once when there is room (so every slice, the padded last one included, labels rows on
    the tensor path), then columns at random.  ``n_defer``: exactly that many deferred rows (the deferring special rows
    cycled), else every special row once."""
    g = tc2_geom(k, d)
    C, plan, bits, E, T = centres(k, d)
    rng = np.random.RandomState(seed)
    dup_cols = {c for a, b, kind in plan if kind == "dup" for c in (a, b)}
    free = np.array([j for j in range(k) if j not in dup_cols])
    sp = special_rows(C, plan, bits, E, T, g["NS"])
    pick, spX = [], None
    if sp:
        spX = np.stack([x for x, _ in sp])
        _, spdef = decide(spX, C, k, d, g["NS"], g["S"])
        if n_defer is not None:
            dfr = [i for i in range(len(sp)) if spdef[i]]
            keep = [i for i in range(len(sp)) if not spdef[i]]
            assert n_defer == 0 or dfr
            pick = ([dfr[i % len(dfr)] for i in range(n_defer)] if dfr else []) + keep
        else:
            pick = list(range(len(sp)))
        pick = pick[:n]
    where = np.unique(np.round(np.linspace(n - 1, 0, len(pick))).astype(int)) if pick else np.zeros(0, dtype=int)
    assert len(where) == len(pick), "too few rows for the special rows"
    nfar = n - len(pick)
    far = np.concatenate([free, free[rng.randint(0, len(free), max(0, nfar - len(free)))]])[:nfar]
    rng.shuffle(far)
    is_far = np.ones(n, dtype=bool)
    is_far[where] = False
    X = np.zeros((n, d))
    X[is_far] = C[far]
    kinds = np.array(["far"] * n, dtype=object)
    lab = np.zeros(n, dtype=np.int64)
    lab[is_far] = far
    deferred = np.zeros(n, dtype=bool)
    if pick:
        X[where] = spX[pick]
        kinds[where] = [sp[i][1] for i in pick]
        lab[where], deferred[where] = decide(X[where], C, k, d, g["NS"], g["S"])
    return X, C, lab, deferred, kinds


# ------------------------------------------------------------------------------------------------ references
def dist_sum_ref(v, sms):
    """The distance sum of rowpass_dist_kernel + reduce_partials_kernel for the per-row values v (float64): warp gw of
    a grid of min(ceil(n / 8), 8 SMs) CTAs adds rows gw, gw + 8 grid, ... in order, each CTA adds its 8 warps in order;
    lane l of one warp adds the CTA sums l, l + 32, ... in order, then a shuffle tree over the 32 lanes."""
    v = np.asarray(v, dtype=np.float64)
    n = len(v)
    grid = max(1, min(_cdiv(n, 8), 8 * sms))
    nw = grid * 8
    pad = np.zeros(_cdiv(n, nw) * nw)
    pad[:n] = v
    per_warp = np.zeros(nw)
    for r in pad.reshape(-1, nw):                         # row turn by row turn: each warp's sum in row order
        per_warp += r
    cta = np.zeros(grid)
    for w in range(8):
        cta += per_warp.reshape(grid, 8)[:, w]
    lanes = np.zeros(32)
    for g0 in range(0, grid, 32):
        part = cta[g0:g0 + 32]
        lanes[:len(part)] += part
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[idx ^ o]
    return float(lanes[0])
