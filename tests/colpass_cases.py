"""Cases built to reach the layout and grid limits of the column-block passes, a numpy restatement of the host rules
that pick their geometry, and the column reduction's fold restated in the kernel's order.

The passes: the scalers' statistics pass (bkm_colstats_chunk, bkm_scale.cu), SimpleImputer's statistics and fill passes
(bkm_impute_stats_chunk, bkm_impute_chunk, bkm_impute.cu), the scoring metrics' pass (bkm_metric_chunk, bkm_metrics.cu),
the sparse KMeans pack (bkm_sparse_pack_centers, bkm_sparse_finalize_step, bkm_kmeans_sparse.cu), the affine pass
(bkm_affine_chunk) and QuantileTransformer's transform (bkm_quantile_transform_chunk, bkm_quantile.cu).  The reductions
share column_reduce's layout (bkm_select.cuh): CB columns per pass, G = 256 / CB interleaved row groups, one contiguous
row range per CTA.  ``fold`` restates that reduction literally, so its result is the kernel's bit for bit:

  - each (CTA, row group, column) starts from the identity and adds its rows rb + g, rb + g + G, ... in row order;
  - the row groups combine as ((f_0 + f_1) + f_2) ...;
  - the last CTA folds identity + p_0 + p_1 ... in CTA order;
  - the store is ``first ? v : acc + v``.

The kernels square with fma(t, t, f); numpy has no fma, so the restatement writes f + t * t, which is the same only
while t * t is exact: t has at most 26 significant bits.  The builders guarantee it (values m 2^k with m below 2^12, or
2^8 for bfloat16, and differences on one exponent grid) and ``short_ok`` checks it.  The sums of such values still
round, so the bits depend on the order: ``fold`` can also run with the row groups or the CTAs reversed, and the host
test asserts that every case gives other bits that way, which is what lets the device comparison catch a wrong order."""
import types

import numpy as np

KT = 256                                  # threads per CTA: bkm_select.cuh:13
STAGE_BYTES = 96 * 1024                   # kStageBytes: bkm_quantile.cu:472
QCS = {"f32": 8, "f64": 4, "bf16": 8}     # TCols<T>: min(32 / sizeof(T), 8), bkm_quantile.cu:429
MBITS = {"f32": 12, "f64": 12, "bf16": 8}

# widths: every CB with and without spare threads (256 mod CB threads with bg >= G), and two and three column passes
WIDTHS = [1, 31, 32, 33, 64, 65, 96, 97, 128, 129, 160, 161, 192, 193, 224, 225, 256, 257, 513]
METRIC_M = [1, 2, 3, 5, 7, 85, 100, 129, 255, 256, 257]
METRIC_ROW_M = [1, 4, 40]                 # EQ / LOGLOSS: CB = 1, G = 256
PACK_K = [1, 32, 33, 96, 97, 160, 257]


# ---------------------------------------------------------------------------------------------------------------------
# host rules
# ---------------------------------------------------------------------------------------------------------------------
def cdiv(a, b):
    return -(-a // b)


def col_block(d):
    """bkm_select.cuh:21."""
    return min(KT, cdiv(d, 32) * 32)


def spare(cb):
    """Threads of a CTA whose row group is past G."""
    return KT % cb


def col_pass_grid(n, cols, sms):
    """bkm_select.cuh:25: at least 8 rows per thread, at most 8 CTAs per SM."""
    G = KT // col_block(cols)
    return max(1, min(cdiv(n, 8 * G), 8 * sms))


def reduce_grid(n, G, cap_per_sm, sms):
    """bkm_select.cuh:35: at least 16 rows per thread, at most cap_per_sm CTAs per SM."""
    return max(1, min(cdiv(n, 16 * G), cap_per_sm * sms))


def metric_cb(m, mode):
    """CB of bkm_metric_chunk (bkm_metrics.cu:59, :131): min(m, 256) output columns for ERR, 1 for EQ / LOGLOSS."""
    return min(m, KT) if mode == "err" else 1


def metric_grid(n, m, mode, sms):
    """bkm_metrics.cu:62."""
    return reduce_grid(n, KT // metric_cb(m, mode), 8, sms)


def partials_bytes(grid, per_cta):
    """bkm_common.cuh:63."""
    return cdiv(grid * per_cta * 8, 256) * 256 + 256


def pack_grid_sparse(p, k, sms):
    """bkm_kmeans_sparse.cu:616."""
    return reduce_grid(p, KT // col_block(k), 4, sms)


def pack_ws(p, k, sms):
    """bkm_kmeans_sparse.cu:617: the k shift terms, then the partials."""
    return cdiv(k * 8, 256) * 256 + partials_bytes(pack_grid_sparse(p, k, sms), 2 * k)


def layout(n, cols, cb, cap, sms):
    """(CB, G, grid) of a column_reduce pass."""
    G = KT // cb
    return cb, G, reduce_grid(n, G, cap, sms)


def qtransform_geom(n, d, nq, dt, sms):
    """launch_qtransform (bkm_quantile.cu:498-509): (CS, staged, per_sm, gx, gy)."""
    CS = QCS[dt]
    smem = (CS + 1) * nq * 8
    staged = smem <= STAGE_BYTES
    per_sm = (8 if smem <= 24 * 1024 else 4 if smem <= 48 * 1024 else 2) if staged else 8
    gx = cdiv(d, CS)
    gy = cdiv(per_sm * sms, gx)
    gy = max(1, min(gy, cdiv(n, (KT // CS) * 8), 65535))
    return CS, staged, per_sm, gx, gy


def cta_rows(n, grid):
    """Each CTA's row range [rb, re) (empty past n): per = ceil(n / grid)."""
    per = cdiv(n, grid) if n else 0
    rb = np.arange(grid, dtype=np.int64) * per
    return np.minimum(rb, n), np.minimum(rb + per, n), per


# ---------------------------------------------------------------------------------------------------------------------
# row counts
# ---------------------------------------------------------------------------------------------------------------------
def reduce_rows(G, cap, sms):
    """{label: n} of a column_reduce layout with G row groups: no row, one row, one row past a 16 G boundary, one CTA
    under the grid cap, at it, past it (with empty trailing CTAs where 16 G < cap * sms) and a last CTA of one row
    (where one exists: 16 G <= cap * sms)."""
    capn = cap * sms
    out = {"0": 0, "1": 1, "16G+1": 16 * G + 1, "cap-1": 16 * G * (capn - 1), "cap": 16 * G * capn,
           "past": 16 * G * capn + 1}
    if 16 * G <= capn:
        out["tail1"] = 16 * G * (16 * G - 1) + 1
    return out


def pass_rows(cols, sms):
    """{label: n} of an element pass over `cols` columns: one row, one past an 8 G boundary, at the 8-per-SM cap and
    past it."""
    G = KT // col_block(cols)
    capn = 8 * sms
    return {"1": 1, "8G+1": 8 * G + 1, "cap": 8 * G * capn, "past": 8 * G * capn + 3}


def grid_facts(n, G, grid):
    """(CTAs with rows, empty trailing CTAs, rows of the last CTA with rows)."""
    rb, re, per = cta_rows(n, grid)
    used = int((re > rb).sum())
    return used, grid - used, int(re[used - 1] - rb[used - 1]) if used else 0


# ---------------------------------------------------------------------------------------------------------------------
# data
# ---------------------------------------------------------------------------------------------------------------------
def short_ok(t):
    """Every finite t has at most 26 significant bits, so t * t is exact in float64."""
    t = np.asarray(t, dtype=np.float64)
    t = t[np.isfinite(t) & (t != 0)]
    m, _ = np.frexp(t)
    q = m * 2.0 ** 26
    return bool((q == np.round(q)).all())


def wide(rng, shape, dt, kspan=30):
    """m 2^k, |m| < 2^12 (2^8 for bfloat16), k in [-kspan, kspan]: exact in the dtype, exact squares, rounding sums."""
    m = rng.randint(1, 1 << MBITS[dt], shape).astype(np.float64) * rng.choice([-1.0, 1.0], shape)
    return np.ldexp(m, rng.randint(-kspan, kspan + 1, shape))


def ints(rng, shape, dt):
    """Integers of every size below 2^26, exact in the dtype: m 2^e with m < 2^12 (2^8), e in [0, 26 - 12 (8)]."""
    mb = MBITS[dt]
    m = rng.randint(0, 1 << mb, shape).astype(np.float64)
    return np.ldexp(m, rng.randint(0, 26 - mb + 1, shape))


SPECIALS = [np.nan, np.inf, -np.inf, 0.0, -0.0, "miss"]


def special_rows(n, G, grid):
    """Rows that matter to the layout: the first and last rows of the first, a middle and the last CTA with rows, the
    first row of row group G - 1 and the row a spare group would revisit first (rb + G, row group 0's second row)."""
    rb, re, _ = cta_rows(n, grid)
    used = [c for c in range(grid) if re[c] > rb[c]]
    rows = set()
    for c in sorted({used[0], used[len(used) // 2], used[-1]}) if used else []:
        for r in (rb[c], re[c] - 1, rb[c] + G - 1, rb[c] + G):
            if rb[c] <= r < re[c]:
                rows.add(int(r))
    return sorted(rows)


def place_specials(X, rows, miss, seed):
    """NaN, +-inf, +-0 and the missing value at the given rows, a few columns each; returns X."""
    n, d = X.shape
    rng = np.random.RandomState(seed)
    for i, r in enumerate(rows):
        for q in range(min(d, 3)):
            v = SPECIALS[(i + q) % len(SPECIALS)]
            X[r, rng.randint(0, d)] = miss if isinstance(v, str) else v
    return X


def plant(X, n, G, grid, big, cancel):
    """Make the fold's order show in the sums.  cancel: +big and -big in the first rows of row groups 1 and 2 of every
    CTA, and +-4 big in CTA 0 and CTA 1, so that the forward order cancels them before the small values arrive and a
    reversed order rounds the small values at their scale.  Otherwise (positive sums) big in row group 1's first row of
    every CTA: the order decides which small values round at big's scale."""
    rb, re, _ = cta_rows(n, grid)
    for c in range(grid):
        m = re[c] - rb[c]
        if m >= 2:
            X[rb[c] + 1] = big
        if cancel and m >= 3:
            X[rb[c] + 2] = -big
        if cancel and c < 2 and m >= 4:
            X[rb[c] + 3] = 4 * big if c == 0 else -4 * big
    return X


def stat_case(n, d, dt, sms, cap, seed, shifted, miss=-1.0):
    """Rows for the statistics passes: wide-exponent values (no shift), or integers of every size below 2^26 with a
    small integer shift, planted to make the order show (``plant``), with the special values placed for this geometry."""
    rng = np.random.RandomState(seed)
    X = ints(rng, (n, d), dt) if shifted else wide(rng, (n, d), dt)
    shift = rng.randint(0, 1 << 12, d).astype(np.float64) if shifted else None
    cb = col_block(d)
    _, G, grid = layout(n, d, cb, cap, sms)
    big = np.ldexp((1 << MBITS[dt]) - 1.0, 26 - MBITS[dt]) if shifted else 2.0 ** 60
    plant(X, n, G, grid, big, cancel=not shifted)
    place_specials(X, special_rows(n, G, grid), miss, seed + 1)
    return X, shift


# ---------------------------------------------------------------------------------------------------------------------
# the fold
# ---------------------------------------------------------------------------------------------------------------------
def fold(n, cols, G, grid, ident, comb, add, rev_groups=False, rev_ctas=False):
    """column_reduce restated (bkm_select.cuh:52-100): the (N, cols) result before the store.  ``ident`` the N
    identities, ``comb(k, v, p)`` the fold rule, ``add(f, R, ok)`` a thread step: rows R (grid, G), ok where R < re."""
    N = len(ident)
    rb, re, per = cta_rows(n, grid)
    f = [np.full((grid, G, cols), ident[k], dtype=np.float64) for k in range(N)]
    g = np.arange(G, dtype=np.int64)
    for t in range(cdiv(per, G) if per else 0):
        R = rb[:, None] + g[None, :] + t * G
        ok = R < re[:, None]
        if not ok.any():
            break
        add(f, np.minimum(R, n - 1), ok)
    gorder = list(range(G))[::-1] if rev_groups else list(range(G))
    corder = list(range(grid))[::-1] if rev_ctas else list(range(grid))
    out = []
    with np.errstate(all="ignore"):
        for k in range(N):
            p = f[k][:, gorder[0]]
            for gg in gorder[1:]:
                p = comb(k, p, f[k][:, gg])
            v = np.full(cols, ident[k], dtype=np.float64)
            for c in corder:
                v = comb(k, v, p[c])
            out.append(v)
    return np.stack(out)


def _sum(k, v, p):
    return v + p


def _w(ok, new, old):
    return np.where(ok, new, old)


# scalers: acc [sum | sq | nan | +inf | -inf], minmax [min | max] (bkm_scale.cu:28-95)
CS_IDENT = [0.0, 0.0, 0.0, 0.0, 0.0, np.inf, -np.inf]


def dev_fmin(a, b):
    """CUDA's fmin on float64: np.fmin, except that -0.0 is below +0.0 in either order (np.fmin returns its first
    argument for two zeros)."""
    z = (a == 0) & (b == 0)
    return np.where(z, np.where(np.signbit(a), a, b), np.fmin(a, b))


def dev_fmax(a, b):
    """CUDA's fmax on float64: np.fmax, except that +0.0 is above -0.0 in either order."""
    z = (a == 0) & (b == 0)
    return np.where(z, np.where(np.signbit(a), b, a), np.fmax(a, b))


def cs_comb(k, v, p):
    return dev_fmin(v, p) if k == 5 else dev_fmax(v, p) if k == 6 else v + p


def colstats_fold(X, shift, G, grid, **kw):
    n, d = X.shape
    s = 0.0 if shift is None else shift

    def add(f, R, ok):
        x = X[R]
        ok = ok[..., None]
        nan = np.isnan(x)
        f[2] = _w(ok & nan, f[2] + 1.0, f[2])
        nn = ok & ~nan
        f[5] = _w(nn, dev_fmin(f[5], x), f[5])
        f[6] = _w(nn, dev_fmax(f[6], x), f[6])
        inf = np.isinf(x)
        f[3] = _w(nn & inf & (x > 0), f[3] + 1.0, f[3])
        f[4] = _w(nn & inf & (x < 0), f[4] + 1.0, f[4])
        fin = nn & ~inf
        t = x - s
        f[0] = _w(fin, f[0] + t, f[0])
        f[1] = _w(fin, f[1] + t * t, f[1])             # fma(t, t, f): t is short

    with np.errstate(all="ignore"):
        return fold(n, d, G, grid, CS_IDENT, cs_comb, add, **kw)


def colstats_store(prev, v, first):
    """(acc (5, d), minmax (2, d)) after a call (StatsFold::store, bkm_scale.cu:91)."""
    if first or prev is None:
        return v[:5].copy(), v[5:].copy()
    acc, mm = prev
    return acc + v[:5], np.stack([dev_fmin(mm[0], v[5]), dev_fmax(mm[1], v[6])])


# imputer: acc [missing | nan | inf | sum] (bkm_impute.cu:17-101)
def impute_fold(X, shift, miss_is_nan, miss, G, grid, **kw):
    n, d = X.shape
    s = 0.0 if shift is None else shift

    def add(f, R, ok):
        x = X[R]
        ok = ok[..., None]
        nan, inf = np.isnan(x), np.isinf(x)
        f[1] = _w(ok & nan, f[1] + 1.0, f[1])
        f[2] = _w(ok & ~nan & inf, f[2] + 1.0, f[2])
        m = nan if miss_is_nan else x == miss
        f[0] = _w(ok & m, f[0] + 1.0, f[0])
        fin = ok & ~m & np.isfinite(x)
        f[3] = _w(fin, f[3] + (x - s), f[3])

    with np.errstate(all="ignore"):
        return fold(n, d, G, grid, [0.0] * 4, _sum, add, **kw)


def sum_store(prev, v, first):
    return v.copy() if first or prev is None else prev + v


# metrics (bkm_metrics.cu:70-124)
def metric_err_fold(A, B, shift, G, grid, **kw):
    n, m = A.shape
    s = 0.0 if shift is None else shift

    def add(f, R, ok):
        x, y = A[R], B[R]
        ok = ok[..., None]
        dl, t = y - x, x - s
        f[0] = _w(ok, f[0] + dl * dl, f[0])              # fma(dl, dl, f): dl is short
        f[1] = _w(ok, f[1] + np.abs(dl), f[1])
        f[2] = _w(ok, f[2] + t, f[2])
        f[3] = _w(ok, f[3] + t * t, f[3])

    with np.errstate(all="ignore"):
        return fold(n, m, G, grid, [0.0] * 4, _sum, add, **kw)


def metric_row_fold(term0, w, G, grid, sub=False, **kw):
    """EQ (f0 += eq ? w : w 0.0) and LOGLOSS (f0 -= w log(pick / sum)) over per-row terms; f1 += w."""
    n = len(w)

    def add(f, R, ok):
        a, b = term0[R][..., None], w[R][..., None]
        ok = ok[..., None]
        f[0] = _w(ok, f[0] - a if sub else f[0] + a, f[0])
        f[1] = _w(ok, f[1] + b, f[1])

    with np.errstate(all="ignore"):
        return fold(n, 1, G, grid, [0.0, 0.0], _sum, add, **kw)


def eq_terms(A, B, w):
    eq = (A == B).all(1)
    with np.errstate(all="ignore"):
        return np.where(eq, w, w * 0.0)


def logloss_terms(cls, P, w, eps):
    """w log(pick / sum) per row in numpy (CUDA's log is not numpy's: held to a tolerance)."""
    with np.errstate(all="ignore"):
        q = np.clip(P, eps, 1.0 - eps)
        if q.shape[1] == 1:
            p1 = q[:, 0]
            q = np.stack([1.0 - p1, p1], 1)
        tot = np.zeros(len(q))
        for j in range(q.shape[1]):
            tot = tot + q[:, j]
        ok = (cls >= 0) & (cls < q.shape[1])
        pick = np.where(ok, q[np.arange(len(cls)), np.where(ok, cls, 0)], np.nan)
        return w * np.log(pick / tot)


# sparse pack: CT [p][k], f0 = sum (ct_in - c)^2, f1 = sum c^2 (bkm_kmeans_sparse.cu:566-614)
def pack_fold(Cp, ct_in, G, grid, **kw):
    """Cp (p, k) the new CT; ct_in (p, k) or None."""
    p, k = Cp.shape

    def add(f, R, ok):
        c = Cp[R]
        ok = ok[..., None]
        if ct_in is not None:
            df = ct_in[R] - c
            f[0] = _w(ok, f[0] + df * df, f[0])
        f[1] = _w(ok, f[1] + c * c, f[1])

    with np.errstate(all="ignore"):
        return fold(p, k, G, grid, [0.0, 0.0], _sum, add, **kw)


def pack_case(p, k, sms, seed):
    """Centres C (k, p) for the pack, and the finalize step's inputs: red = [p k sumsT | k counts | inertia] with
    power-of-two counts (0 for some clusters), and the current pack's CT on the same exponent grid as the new one.
    Both planted (``plant``) for the layout of p rows and k columns."""
    rng = np.random.RandomState(seed)
    G = KT // col_block(k)
    grid = pack_grid_sparse(p, k, sms)
    e = rng.randint(-10, 11, (p, k))
    C = plant(np.ldexp(rng.randint(-4095, 4096, (p, k)).astype(np.float64), e), p, G, grid, 2.0 ** 35, False)
    cnt = np.ldexp(1.0, rng.randint(0, 12, k))
    cnt[::5] = 0.0
    e = plant(e, p, G, grid, 23, False)
    S = np.ldexp(rng.randint(-4095, 4096, (p, k)).astype(np.float64), e)
    new = S / np.maximum(cnt, 1.0)[None, :]
    ct_in = new + np.ldexp(rng.randint(-4095, 4096, (p, k)).astype(np.float64), e - 12)
    red = np.concatenate([S.ravel(), cnt, [0.0]])
    return types.SimpleNamespace(C=C.T.copy(), red=red, ct_in=ct_in, new=new)


def pack_rows(k, sms):
    """{label: p} of the pack over k clusters: reduce_rows at its layout, capped to keep the pack small."""
    G = KT // col_block(k)
    return {lab: p for lab, p in reduce_rows(G, 4, sms).items() if p > 0}
