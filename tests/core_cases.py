"""The CUDA-core chunk kernels behind bkm_lloyd_chunk / bkm_assign_chunk, restated: the generic kernel (family 0,
bkm_simt.cu) and the two streaming kernels (family 2, bkm_stream.cu), with the data the limit tests run on.

Geometry (``layout`` equals bkm_debug_core_layout, test_core_cases_host.py):
* generic: J = 8 or 16 centres per register block (16 for fp32 when it pads k no more than 8 does), GLOBAL mode when
  centres + sums do not fit beside a 32-row tile, SMALLK (lane-owns-cluster M-step) for k <= 32 and d <= 16 in SMEM
  mode, and a row tile rt of 256 rows stepping down by 32 to 32, then halving, until the staged tile fits;
* streaming: two rows per thread for k <= 24 at a pitch of at most 32 floats (KC centres, a ring of 3 stages of 64 rows
  per warp, an M-step pair stride msS = 16 >> trailing zero bits of the pitch), else one row per thread (KPT centre
  pairs, 4 stages of 32 rows); a pitch over 64 floats, a ring too large for shared memory or a base address that is
  not 16-byte aligned goes to the generic kernel.
``grid`` restates each launch's clamp; the tests measure the SM occupancy it needs.

Data (every result exact, so numpy's float64 is a bit-exact reference):
* ``lattice``: small-integer centres and rows around them; every product, partial sum and distance the fp32 kernels
  form is an integer below 2^24, with duplicate centres placed at the designed tie pairs;
* ``near_tie``: centres 64 apart around a base point far from the origin (||x||^2 + max ||c||^2 >= 2^25), and pairs
  of centres one unit apart along feature 0 with rows next to the higher-index one: the two best distances are small
  integers that differ by 1, far inside the re-check bound, so the fp32 GEMM form cannot order them while float64 and
  the fp32 direct form are exact.
"""
import math

import numpy as np

F32, F64 = 0, 1
FORCE_SIMT, FORCE_TC, NO_RECHECK = 1, 2, 4
SMEM_BUDGET = 227 * 1024
TILE = 256                          # generic kernel: threads per CTA, the largest row tile
SW = 8                              # streaming kernels: warps per CTA
SNSTG, S2_NSTG = 4, 3               # ring stages per warp: one-row, two-row kernel
GENERIC, ONE_ROW, TWO_ROW = 0, 1, 2
FIELDS = ("kernel", "J", "GLOBAL", "SMALLK", "rt", "pitch", "DH", "KB", "msS", "stages", "rows", "stage_bytes", "smem")
SM_COUNTS = (132, 114)


def _align(x, a):
    return (x + a - 1) // a * a


def _cdiv(a, b):
    return -(-a // b)


def tau(d):
    """The re-check coefficient of both CUDA-core kernels (bkm_api.cu tau_for), in float64."""
    return 8.0 * (math.sqrt(d) + 2.0) * 2.0 ** -24


# ------------------------------------------------------------------------------------------------ geometry
def kernel_family(d, k, dtype, flags=0):
    """bkm_kernel_family for fp32 / float64 rows; None where it refuses."""
    tc = dtype == F32 and 1 <= d <= 64 and 1 <= k <= 256
    if flags & FORCE_SIMT:
        return 0
    if flags & FORCE_TC:
        return 1 if tc else None
    if dtype == F32 and d <= 16 and k <= 32 and k * d < 512:
        return 2
    return 1 if tc and k * d >= 512 else 0


def tile_pitch(d4, esz):
    return ((d4 * esz // 16) | 1) * 16 // esz


def simt_smem(k, d, J, mstep, glob, rt, esz):
    psz = 8 if esz == 8 else 4
    d4 = _align(d, 4)
    kJ = _align(k, J)
    o = 0 if glob else kJ * d4 * esz
    o = _align(o, 16) + kJ * esz
    o = _align(o, 16) + rt * tile_pitch(d4, esz) * esz
    o = _align(o, 16) + TILE * 4 + TILE * 8 + TILE * 4
    if mstep and not glob:
        o += k * d * psz
    o = _align(o, 16)
    if mstep:
        o += k * 4
    return _align(o, 16) + 256


def simt_plan(d, k, dtype, mstep):
    esz = 8 if dtype == F64 else 4
    w8, w16 = _align(k, 8) - k, _align(k, 16) - k
    J = 16 if (w16 <= w8 and dtype == F32) else 8
    glob = simt_smem(k, d, J, mstep, False, 32, esz) > SMEM_BUDGET
    rt = TILE
    while rt > 1 and simt_smem(k, d, J, mstep, glob, rt, esz) > SMEM_BUDGET:
        rt = rt - 32 if rt > 32 else rt // 2
    total = simt_smem(k, d, J, mstep, glob, rt, esz)
    if total > SMEM_BUDGET:
        return None
    return dict(kernel=GENERIC, J=J, GLOBAL=int(glob), SMALLK=int(mstep and not glob and k <= 32 and d <= 16), rt=rt,
                pitch=tile_pitch(_align(d, 4), esz), smem=total)


def pair_stride(L):
    tz = 0
    while tz < 4 and not (L >> tz) & 1:
        tz += 1
    return 16 >> tz


def stream_plan(d, k, ldx):
    """The streaming kernel of an aligned call, or None where it falls back to the generic kernel."""
    if ldx > 64:
        return None
    DH = 2 if d <= 4 else 4 if d <= 8 else 6 if d <= 12 else 7 if d <= 14 else 8
    if k <= 24 and ldx <= 32:
        KC = _align(k, 4)
        dp = _align(2 * DH, 4)
        o = KC * dp * 4 + KC * 4
        o = _align(o, 16) + k * 4
        o = _align(o, 16) + SW * 8 + SW * S2_NSTG * 8 + SW * 64 * 4 + SW * 64 * 4
        o = _align(o, 128) + SW * (KC + 1) * 32 * 4
        stage = 64 * ldx * 4
        o = _align(o, 128) + SW * S2_NSTG * stage + 128
        p = dict(kernel=TWO_ROW, DH=DH, KB=KC, msS=pair_stride(ldx), stages=S2_NSTG, rows=64, stage_bytes=stage, smem=o)
    else:
        KPT = _cdiv(k, 4) * 2
        dp = 2 * DH
        o = KPT * dp * 8 + KPT * 8
        o = _align(o, 16) + k * d * 4
        o = _align(o, 16) + k * 4
        o = _align(o, 16) + SW * 8 + SW * SNSTG * 8 + SW * 32 * 4
        stage = 32 * ldx * 4
        o = _align(o, 128) + SW * SNSTG * stage
        p = dict(kernel=ONE_ROW, DH=DH, KB=KPT, msS=0, stages=SNSTG, rows=32, stage_bytes=stage, smem=o)
    return p if p["smem"] <= SMEM_BUDGET else None


def plan(d, k, ldx, dtype, flags=0, mstep=True, aligned16=True):
    """The kernel a chunk call runs and its configuration (a dict of FIELDS); None where the tensor path runs."""
    fam = kernel_family(d, k, dtype, flags)
    if fam is None or (fam == 1 and ((aligned16 and ldx % 4 == 0) or flags & FORCE_TC)):
        return None
    p = stream_plan(d, k, ldx) if fam == 2 and aligned16 else None
    if p is None:
        p = simt_plan(d, k, dtype, mstep)
    if p is None:
        return None
    return {f: int(p.get(f, 0)) for f in FIELDS}


def layout(d, k, ldx, dtype, flags=0, mstep=True, aligned16=True):
    """The 13 numbers bkm_debug_core_layout returns, restated; None where it answers BKM_EUNSUPPORTED."""
    p = plan(d, k, ldx, dtype, flags, mstep, aligned16)
    return None if p is None else tuple(p[f] for f in FIELDS)


def ws_layout(n, d, k, dtype, sms):
    """ws_layout (bkm_common.cuh) of an fp32 / float64 call: offsets of the per-CTA partials and the total."""
    esz = 8 if dtype == F64 else 4
    slot = k * d * esz
    part = sms * 8
    psum_slots = 1 if 2 * slot > SMEM_BUDGET else sms * min(8, max(1, SMEM_BUDGET // (2 * slot)))
    W = {}
    o = _align(16 + 4096, 256)
    W["psum"] = o; o = _align(o + max(psum_slots * slot, k * d * 8), 256)
    W["pcnt"] = o; o = _align(o + part * k * 4, 256)
    W["pin"] = o; o = _align(o + part * 8, 256)
    W["flag"] = o; o = _align(o + 256, 256)
    W["defer"] = o; o = _align(o + n * 4, 256)
    W["total"] = o
    W["psum_slots"], W["part_slots"] = psum_slots, part
    return W


def grid(p, d, k, n, dtype, mstep, sms, occ):
    """The grid the launch picks for a call of plan ``p`` on n rows: SMs x occupancy, clamped to the workspace's
    partial slots and to the row tiles (generic: one tile per CTA at least; streaming: 8 warps' tiles per CTA)."""
    W = ws_layout(n, d, k, dtype, sms)
    g = sms * occ
    if p["kernel"] == GENERIC:
        if mstep and not p["GLOBAL"]:
            g = min(g, W["psum_slots"])
        g = min(g, W["part_slots"], _cdiv(n, p["rt"]))
    else:
        g = min(g, W["psum_slots"], W["part_slots"], _cdiv(_cdiv(n, p["rows"]), SW))
    return max(1, g)


# ------------------------------------------------------------------------------------------------ designed data
def lattice(d, k, n, seed, ties=(), R=6, r=2):
    """(X, C): centres with integer coordinates in [-R, R], rows = a centre + integers in [-r, r].  For each tie pair
    (a, b) centre b duplicates centre a, and the first rows sit on the tied centres (distance 0 to both)."""
    rng = np.random.RandomState(seed)
    C = rng.randint(-R, R + 1, size=(k, d)).astype(np.float64)
    for a, b in ties:
        C[b] = C[a]
    X = C[rng.randint(0, k, size=n)] + rng.randint(-r, r + 1, size=(n, d))
    for i, (a, b) in enumerate(ties):
        if 2 * i + 1 < n:
            X[2 * i] = C[a]
            X[2 * i + 1] = C[b] + (rng.randint(-1, 2, size=d) if i % 2 else 0)
    return X, C


def near_tie(d, k, n, seed, pairs, ties=()):
    """(X, C, near): centres on a lattice of step 64 around a base point B with ||B||^2 >= 2^25; for each near pair
    (a, b), a < b, centre b sits one unit from centre a along feature 0 and 16 rows sit next to centre b, on it or
    one unit off it in features other than 0 (distances |w|^2 to b, |w|^2 + 1 to a: the higher index wins by less than
    the bound); for each tie pair centre b duplicates centre a.  The other
    rows sit within 2 of a random centre.  ``near`` marks the near-tie rows."""
    rng = np.random.RandomState(seed)
    M = int(math.ceil(math.sqrt(2.0 ** 25.3 / d)))
    B = M + rng.randint(0, 8, size=d)
    side = max(2, int(math.ceil(k ** (1.0 / d) / 2)) + 1) if d < 8 else 2
    g = set()
    cells = []
    while len(cells) < k:
        v = tuple(rng.randint(-side, side + 1, size=d))
        if v not in g:
            g.add(v)
            cells.append(v)
    C = (B[None, :] + 64 * np.array(cells)).astype(np.float64)
    for a, b in pairs:
        C[b] = C[a]
        C[b, 0] += 1
    for a, b in ties:
        C[b] = C[a]
    X = C[rng.randint(0, k, size=n)] + rng.randint(-2, 3, size=(n, d))
    near = np.zeros(n, dtype=bool)
    # 16 distinct rows per near pair, x = c_b + w with w_0 = 0 and w_i in {-1, 0, 1} otherwise: distances |w|^2 to b
    # and |w|^2 + 1 to a, each row with its own fp32 rounding; two rows on each duplicated centre
    i = 0
    for a, b in pairs:
        for r in range(16):
            w = rng.randint(-1, 2, size=d) if r else np.zeros(d, dtype=np.int64)
            w[0] = 0
            X[i] = C[b] + w
            near[i] = True
            i += 1
    for a, b in ties:
        for r in range(2):
            X[i] = C[a]
            near[i] = True
            i += 1
    return X, C, near


def reference(X, C):
    """(labels, squared distances) of the float64 arg-min, lowest index on exact ties."""
    n = X.shape[0]
    lab = np.empty(n, dtype=np.int64)
    d2 = np.empty(n)
    cn = (C * C).sum(1)
    for s in range(0, n, 16384):
        blk = X[s:s + 16384]
        e = (blk * blk).sum(1)[:, None] - 2.0 * blk @ C.T + cn[None, :]
        lab[s:s + 16384] = e.argmin(1)
        d2[s:s + 16384] = e[np.arange(blk.shape[0]), lab[s:s + 16384]]
    return lab, d2


def generic_fp32_argmin(X, C):
    """Labels the generic kernel's fp32 E-step gives without the re-check: per centre the FMA chain
    acc = fma(x_4q, c_4q, fma(x_4q+1, c_4q+1, fma(x_4q+2, c_4q+2, fma(x_4q+3, c_4q+3, acc)))) over the 4-feature chunks,
    dist = fma(-2, acc, ||c||^2 rounded to fp32), the first index of the smallest.  Exact emulation on integer data
    below 2^24 per product: every product and sum is exact in float64, so each fma rounds once, as on the device."""
    n, d = X.shape
    acc = np.zeros((n, C.shape[0]), dtype=np.float32)
    for ch in range(0, d, 4):
        for i in range(min(ch + 3, d - 1), ch - 1, -1):
            acc = (X[:, i, None] * C[None, :, i] + acc.astype(np.float64)).astype(np.float32)
    cn = (C * C).sum(1).astype(np.float32)
    dist = (-2.0 * acc.astype(np.float64) + cn.astype(np.float64)[None, :]).astype(np.float32)
    return dist.argmin(1)


def sums_ref(X, lab, k):
    """(float64 sums, counts) per cluster: exact on the designed data, in any order."""
    sums = np.stack([np.bincount(lab, weights=X[:, i], minlength=k) for i in range(X.shape[1])], 1)
    return sums, np.bincount(lab, minlength=k)


# ------------------------------------------------------------------------------------------------ cases
DH_D = {2: 3, 4: 7, 6: 11, 7: 13, 8: 16}          # a d of every feature-pair count DH
GENERIC_TIES = ((3, 5), (6, 21), (40, 140), (7, 263), (100, 261))   # k = 300: in one J block, across J blocks,
# across warps, j and j + 256 (one re-check thread), and a lower index held by a higher warp than its duplicate's
STREAM_TIES = ((1, 2), (0, 7))


def rt_shape(dtype, rt, odd=True):
    """The smallest d (odd when asked) whose assign-only call (k = 4) runs the generic kernel with row tile rt."""
    d = 64 + (1 if odd else 0)
    step = 2 if odd else 1
    while True:
        p = simt_plan(d, 4, dtype, False)
        if p["rt"] == rt:
            return d
        assert p["rt"] > rt, (dtype, rt, d)
        d += step if p["rt"] > 2 * rt or p["rt"] <= 32 else 16 * step


def global_boundary(d, dtype, mstep):
    """The smallest k whose call runs the generic kernel in GLOBAL mode at d."""
    k = 1
    while not simt_plan(d, k, dtype, mstep)["GLOBAL"]:
        k += 1
    return k


def _c(cid, d, k, n, dtype=F32, flags=0, pitch=None, data="lattice", ties=(), pairs=(), base_off=0, pad="big"):
    return dict(id=cid, d=d, k=k, n=n, dtype=dtype, flags=flags, pitch=pitch or d, data=data, ties=tuple(ties),
                pairs=tuple(pairs), base_off=base_off, pad=pad)


def cases():
    """The exact-data cases of test_gpu_core_limits.py (each runs its Lloyd and its assign-only call)."""
    cs = []
    # ---- family 2: every two-row instance (DH x KC) and every one-row instance (DH x KPT), pitches of every msS class
    two_pitch = (None, 16, 20, 17, 32, 18, 24, 28, 31, 12)
    for i, (DH, d) in enumerate(sorted(DH_D.items())):
        for j, KC in enumerate(range(4, 25, 4)):
            k = max(1, KC - (i + j) % 4)
            p = two_pitch[(i + 2 * j) % len(two_pitch)]
            p = max(d, p) if p else None
            cs.append(_c("s2-DH%d-KC%d" % (DH, KC), d, k, 64 * 29 + 1 + 7 * j, pitch=p, pad=("big", "nan")[j % 2]))
        for j, KPT in enumerate(range(2, 17, 2)):
            k = 2 * KPT - (i + j) % 4 if KPT >= 14 else 2 * KPT - (i + j) % 2
            k = min(k, 511 // d)
            pitch = d if KPT >= 14 and k > 24 else 33 + (3 * i + 5 * j) % 22
            cs.append(_c("s1-DH%d-KPT%d" % (DH, KPT), d, k, 32 * 53 + 3 + 5 * j, pitch=pitch,
                         pad=("nan", "big")[j % 2]))
    for L in (3, 4, 5, 6, 8, 12, 16, 20, 24, 28, 32):                          # every msS class at d = 3, k = 20
        cs.append(_c("msS-d3-L%d" % L, 3, 20, 64 * 41 + 9, pitch=L))
    for L in (12, 13, 14, 16, 20, 28):
        cs.append(_c("msS-d12-L%d" % L, 12, 24, 64 * 23 + 63, pitch=L))
    for k in (24, 25):
        cs.append(_c("k%d-L16" % k, 16, k, 5000, pitch=16))
    for L in (32, 33, 56, 57, 65):
        cs.append(_c("d13-k20-L%d" % L, 13, 20, 3001, pitch=L))
    cs.append(_c("misaligned-d13-k20", 13, 20, 3001, pitch=16, base_off=1))
    cs.append(_c("misaligned-d8-k24", 8, 24, 777, pitch=8, base_off=2))
    for d in (1, 13):
        cs.append(_c("k1-d%d" % d, d, 1, 1111))
    cs.append(_c("s2-ties", 13, 20, 4000, ties=STREAM_TIES))
    cs.append(_c("s1-ties", 13, 28, 4000, ties=STREAM_TIES))
    # ---- family 0, fp32 and float64: J padding, SMALLK, SMEM / GLOBAL, row tiles, FORCE_SIMT
    for dtype, tag in ((F32, "f32"), (F64, "f64")):
        for k in ((16, 17, 31, 15, 24, 23, 255, 257) if dtype == F32 else (8, 9, 15, 16, 17, 263)):
            cs.append(_c("J-%s-k%d" % (tag, k), 70, k, 256 * 5 + 3, dtype))
        for d, k in ((16, 32), (16, 33), (17, 32), (1, 1)):
            cs.append(_c("smallk-%s-d%d-k%d" % (tag, d, k), d, k, 256 * 9 + 255, dtype, FORCE_SIMT))
        for mstep in (True, False):
            kb = global_boundary(96, dtype, mstep)
            for k in (kb - 1, kb):
                cs.append(_c("global-%s-%s-k%d" % (tag, "lloyd" if mstep else "assign", k), 96, k, 1500, dtype))
        for rt in (256, 160, 32, 16, 2, 1):
            d = rt_shape(dtype, rt)
            cs.append(_c("rt%d-%s-d%d" % (rt, tag, d), d, 4, 3 * rt + 1 if rt > 2 else 37, dtype))
        cs.append(_c("ties-%s-k300" % tag, 20, 300, 3000, dtype, ties=GENERIC_TIES))
    cs.append(_c("force-simt-d64-k256", 64, 256, 5000, F32, FORCE_SIMT, pitch=68))
    cs.append(_c("force-simt-d13-k20", 13, 20, 5000, F32, FORCE_SIMT, pitch=16))
    cs.append(_c("misaligned-d41-k100", 41, 100, 2000, F32, pitch=44, base_off=1))
    # ---- near-ties only float64 can decide (fp32: the re-check of both kernels)
    cs.append(_c("near-generic-d100-k40", 100, 40, 1500, data="near", pairs=((2, 3), (10, 30), (5, 39))))
    cs.append(_c("near-generic-d20-k300", 20, 300, 1500, data="near", pairs=((2, 4), (10, 30), (8, 299)),
                 ties=GENERIC_TIES))
    cs.append(_c("near-generic-d13-k20", 13, 20, 1500, flags=FORCE_SIMT, pitch=16, data="near",
                 pairs=((0, 1), (4, 19))))
    cs.append(_c("near-s2-d13-k20", 13, 20, 1500, pitch=16, data="near", pairs=((0, 1), (4, 19)), ties=((6, 7),)))
    cs.append(_c("near-s2-d3-k8", 3, 8, 1500, pitch=4, data="near", pairs=((0, 1), (2, 7))))
    cs.append(_c("near-s1-d13-k28", 13, 28, 1500, pitch=16, data="near", pairs=((0, 1), (4, 27)), ties=((6, 7),)))
    cs.append(_c("near-s1-d5-k20", 5, 20, 1500, pitch=40, data="near", pairs=((0, 1), (4, 19))))
    return cs


def design(c, seed=0):
    """(X, C, near) of a case; ``near`` marks the designed near-tie rows (none in the lattice cases)."""
    d, k, n = c["d"], c["k"], c["n"]
    if c["data"] == "near":
        return near_tie(d, k, n, seed + 17 * k + d, c["pairs"], c["ties"])
    ties = tuple((a, b) for a, b in c["ties"] if b < k)
    R, r = (6, 2) if d <= 64 else (2, 1)
    X, C = lattice(d, k, n, seed + 31 * k + d, ties, R, r)
    return X, C, np.zeros(n, dtype=bool)
