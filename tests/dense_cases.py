"""Exact-data cases built to reach the geometry limits of the dense row-chunk passes, and a numpy restatement of the host
rules that pick those geometries.

The passes: the GaussianNB moments / class-count pass and log-likelihood pass and the discrete-NB linear jll pass
(bkm_nb.cu), the DMMA Gram pass, its weighted variant and the projection (bkm_pca.cu), and the fused GLM pass
(bkm_glm.cu).  Each picks its geometry on the host from (n, d, K, SM count); the rules are restated below with the
source lines they follow, each taking the SM count as a parameter, so a test can assert which limits a case reaches.

Every case holds small integers, integer theta and shifts, and dyadic weights, inverse variances, W, beta and
log-priors, so that every partial sum a kernel can form is exact (below 2^53, and below 2^24 for the fp32 sums of the
fp32 jll path): every summation order gives the same bits, and numpy's float64 result is a bit-exact reference at every
geometry.  ``two_orders`` checks that claim for each case."""
import types

import numpy as np

# ---------------------------------------------------------------------------------------------------------------------
# host rules
# ---------------------------------------------------------------------------------------------------------------------
MT, MR, MBUDGET = 256, 256, 96 * 1024     # moments threads, rows per member tile, accumulator budget: bkm_nb.cu:49-51
JT, JC, JBUDGET = 128, 32, 100 * 1024     # jll rows per tile, feature chunk, shared budget: bkm_nb.cu:219-221
LR = 64                                   # linear jll rows per tile: bkm_nb.cu:564
GB, GR = 64, 32                           # Gram feature block, rows per staged tile: bkm_pca.cu:28-29
PR = 64                                   # projection rows per tile: bkm_pca.cu:31
GLM_T, GLM_TR = 256, 32                   # GLM threads, rows per tile: bkm_glm.cu:36-38
ES = {"f32": 4, "f64": 8, "bf16": 2}


def _al(x, a):
    return (x + a - 1) // a * a


def jll_path(dt, d):
    """(FC, CH) of launch_jll_f32 / launch_jll_f64 (bkm_nb.cu:546-560): FC-wide registers, CH = 32-wide chunks."""
    for fc in ((8, 16, 32) if dt == "f64" else (8, 16, 32, 64)):
        if d <= fc:
            return fc, False
    return JC, True


def jll_smem(es, kb, dp, fc, ch, out):
    """JllSmem.total of jll_smem<TC> (bkm_nb.cu:286-299); es = sizeof(TC)."""
    o = _al(kb * dp * 2 * es, 16)
    o = _al(o + kb * 4, 16)
    o = _al(o + kb * 8, 16)
    o = _al(o + JT * (fc + 1) * es, 16)
    o = _al(o + (kb * JT * es if ch else 0), 16)
    o = _al(o + (JT * (kb + 1) * 8 if out else 0), 16)
    return _al(o + (JT * 8 if out else 0), 16)


def jll_kb(dt, d, K, out):
    """Classes per block of launch_jll_fc (bkm_nb.cu:515-530): all K while they fit JBUDGET, else as many as fit."""
    es = 8 if dt == "f64" else 4                  # the compute type: fp32 for f32 / bf16 rows
    fc, ch = jll_path(dt, d)

    def fits(kb):
        return jll_smem(es, kb, fc, fc, ch, out) <= JBUDGET

    kb = K
    if not fits(kb):
        fixed = jll_smem(es, 0, fc, fc, ch, out) + 64
        per = fc * 2 * es + 12 + (JT * es if ch else 0) + (JT * 8 if out else 0)
        kb = max(1, (JBUDGET - fixed) // per)
        while kb > 1 and not fits(kb):
            kb -= 1
    return kb


def jll_kb_max(dt, d, out):
    """The block size of any K too large to stay resident."""
    return jll_kb(dt, d, 1 << 20, out)


def linear_geom(K):
    """(NT, classes per block CW, blocks) of launch_linear (bkm_nb.cu:733-738) and linear_jll_kernel (:593, :604)."""
    nt = 1 if K <= 16 else 2 if K <= 32 else 4
    cw = 16 * nt
    return nt, cw, (K + cw - 1) // cw


def project_geom(n, k, sms):
    """(NT, columns per CTA CW, gy, gx) of launch_project / launch_project_nt: bkm_pca.cu:406-425."""
    nt = 1 if k <= 16 else 2 if k <= 32 else 4
    cw = 16 * nt
    gy = (k + cw - 1) // cw
    gx = max(1, min((4 * sms + gy - 1) // gy, (n + PR - 1) // PR))
    return nt, cw, gy, gx


def gram_geom(n, d, sms):
    """GramGeom of gram_geom (bkm_pca.cu:48-66): feature blocks, upper tile pairs, row splits, rows per split and the
    workspace bytes."""
    nb = (d + GB - 1) // GB
    pairs = nb * (nb + 1) // 2
    tiles = (n + GR - 1) // GR
    s = max(1, min((2 * sms + pairs - 1) // pairs, tiles))
    rps = max(GR, ((tiles + s - 1) // s) * GR)
    splits = max(1, (n + rps - 1) // rps)
    o = _al(pairs * splits * GB * GB * 8, 256)
    o = _al(o + nb * splits * GB * 8, 256)
    o = _al(o + pairs * 4, 256)
    return types.SimpleNamespace(nb=nb, pairs=pairs, splits=splits, rows_per_split=rps, total=o)


def gram_one_split_d(sms):
    """The smallest d whose tile pairs alone fill two CTAs per SM (pairs >= 2 SMs): from there every pair gets one CTA
    and no split fold runs."""
    nb = 1
    while nb * (nb + 1) // 2 < 2 * sms:
        nb += 1
    return GB * (nb - 1) + 1


def bulk_ok(base_bytes, ldx, d, dt):
    """The Gram pass bulk-copies rows whose base, pitch and width are multiples of 16 bytes (bkm_pca.cu:442); the GLM
    pass reads them with 16-byte vector loads on the same condition (bkm_glm.cu:319)."""
    es = ES[dt]
    return base_bytes % 16 == 0 and (ldx * es) % 16 == 0 and (d * es) % 16 == 0


def glm_grid(n, sms):
    """CTAs of the GLM pass: three per SM, at most one per 32-row tile (bkm_glm.cu:268-274)."""
    return max(1, min(3 * sms, (n + GLM_TR - 1) // GLM_TR))


def glm_phase_b(d):
    """(CB, G, column passes) of phase B (bkm_glm.cu:115-118, :203): CB columns per pass, G row groups."""
    cb = min(GLM_T, (d + 31) // 32 * 32)
    return cb, GLM_T // cb, (d + cb - 1) // cb


def glm_ws(n, d, sms):
    """partials_bytes(glm_grid, 2 d + 3) (bkm_glm.cu:276, bkm_common.cuh:63-65)."""
    return _al(glm_grid(n, sms) * (2 * d + 3) * 8, 256) + 256


def mom_geom(n, d, K, sms):
    """MomGeom of mom_geom (bkm_nb.cu:67-91): feature slices, row groups, class slices, row splits and workspace bytes."""
    fs = min(d, MT)
    nf = (d + fs - 1) // fs
    groups = MT // fs
    ks = min(max(1, MBUDGET // (groups * (fs + 1) * 8)), K)
    nk = (K + ks - 1) // ks
    tiles = (n + MR - 1) // MR
    s = max(1, min((2 * sms + nk * nf - 1) // (nk * nf), tiles))
    rps = max(MR, ((tiles + s - 1) // s) * MR)
    splits = (n + rps - 1) // rps if n > 0 else 0
    sp = max(splits, 1)
    total = _al(_al(sp * K * d * 8, 256) + sp * K * 8, 256)
    return types.SimpleNamespace(fs=fs, nf=nf, groups=groups, ks=ks, nk=nk, splits=splits, rows_per_split=rps,
                                 total=total)


def mom_ks(d):
    """The class-slice size of a d-wide moments pass (any K above it)."""
    return mom_geom(1, d, 1 << 20, 1).ks


# ---------------------------------------------------------------------------------------------------------------------
# the cases
# ---------------------------------------------------------------------------------------------------------------------
SMS = (132, 114)                                   # H100 SXM and H100 PCIe
JLL_D = {("f32", 8, False): 7, ("f32", 16, False): 13, ("f32", 32, False): 32, ("f32", 64, False): 50,
         ("f32", 32, True): 100, ("f64", 8, False): 8, ("f64", 16, False): 11, ("f64", 32, False): 31,
         ("f64", 32, True): 70}                    # a d for every (precision, FC, CH) path
JLL_N = 3 * JT + 37                                # three full tiles and a partial one
LIN_K = [16, 17, 32, 33, 64, 65, 129]
LIN_D = [31, 32, 33]
MOM_D = [255, 256, 257, 513]
GLM_D = [31, 64, 95, 128, 129, 192, 200, 256, 513]  # CB 32, 64, ..., 256 and three passes of 256


def jll_paths():
    """(precision, d, FC, CH) of every jll path; bf16 rows share the fp32 kernels."""
    return [(dt, d, fc, ch) for (dt, fc, ch), d in JLL_D.items()]


def jll_resident_max(dt, d, out):
    """The largest K that stays resident.  The block size leaves 64 bytes for alignment, so this is a few classes
    above ``jll_kb_max``."""
    K = jll_kb_max(dt, d, out)
    while jll_kb(dt, d, K + 1, out) == K + 1:
        K += 1
    return K


def jll_ks(dt, d, out):
    """K at the block size (resident), the first K that is cut into blocks (two), and two blocks and one class."""
    kb = jll_kb_max(dt, d, out)
    return [kb, jll_resident_max(dt, d, out) + 1, 2 * kb + 1]


def _perm_place(rng, n, groups):
    """Row indices for each of ``groups`` (counts), spread over the tiles at random."""
    p = rng.permutation(n)
    out, o = [], 0
    for c in groups:
        out.append(p[o:o + c])
        o += c
    return out


def jll_case(dt, d, K, kb, seed=0, nan_class=None, n=JLL_N):
    """GaussianNB's predict pass on exact data.  theta integers in [-3, 3], 1/sigma in {1/2, 1, 2}, log-priors multiples
    of 1/2 in [-6, -1], rows integers in [-3, 3]: every (x - theta)^2 w is a multiple of 1/2 and every jll a multiple of
    1/4, far from the fp32 bound E.  Classes kb - 1 and kb (either side of the first block boundary; 0 and K - 2 when K
    fits one block) are copies with log-prior 0, and rows equal to their theta tie on them; class K - 1 (in the last
    block) has log-prior 0 and rows equal to its theta pick it alone.  ``nan_class`` gets a NaN log-prior."""
    rng = np.random.RandomState(seed)
    theta = rng.randint(-3, 4, (K, d)).astype(np.float64)
    w = rng.choice([0.5, 1.0, 2.0], (K, d))
    logc = rng.randint(-12, -1, K) / 2.0
    a, b = (kb - 1, kb) if K > kb else (0, K - 2)
    theta[b], w[b] = theta[a], w[a]
    logc[a] = logc[b] = 0.0
    last = K - 1 if K - 1 not in (a, b) else None
    if last is not None:
        logc[last] = 0.0
    tie_rows, last_rows, rest = _perm_place(rng, n, [12, 12 if last is not None else 0, n])
    y = rng.randint(0, K, n)
    x = np.clip(theta[y] + rng.randint(-1, 2, (n, d)), -3, 3)
    x[tie_rows] = theta[a]
    if last is not None:
        x[last_rows] = theta[last]
    if nan_class is not None:
        logc[nan_class] = np.nan
    return types.SimpleNamespace(dt=dt, x=x, theta=theta, w=w, logc=logc, K=K, tie=(a, b), last=last,
                                 tie_rows=tie_rows, last_rows=last_rows)


def jll_ref(c, order=1):
    """(jll, labels, rows whose maximum is attained twice, log-softmax) in float64; ``order`` -1 sums the features
    backwards."""
    s = np.zeros((c.x.shape[0], c.K))
    for j in range(c.x.shape[1])[::order]:
        u = c.x[:, j:j + 1] - c.theta[None, :, j]
        s += u * u * c.w[None, :, j]
    jll = c.logc[None] - 0.5 * s
    lab = np.argmax(jll, 1)
    mx = np.nanmax(jll, 1) if not np.isnan(c.logc).any() else None
    ties = int(((jll == mx[:, None]).sum(1) > 1).sum()) if mx is not None else 0
    with np.errstate(invalid="ignore"):
        vmax = jll.max(1, keepdims=True)
        lp = jll - (np.log(np.exp(jll - vmax).sum(1, keepdims=True)) + vmax)
    return jll, lab, ties, lp


def fp32_bound(c):
    """The largest fp32 error bound E = tau (s + sqrt(s sum_j w theta^2)) + 2^-50 |jll| of the case (DESIGN.md, A21)."""
    d = c.x.shape[1]
    s = np.zeros((c.x.shape[0], c.K))
    for j in range(d):
        u = c.x[:, j:j + 1] - c.theta[None, :, j]
        s += u * u * c.w[None, :, j]
    big = (c.w * c.theta ** 2).sum(1)
    jll = np.nan_to_num(c.logc)[None] - 0.5 * s
    return float(((d + 8) * 2.0 ** -25 * (s + np.sqrt(s * big[None])) + 2.0 ** -50 * np.abs(jll)).max())


def linear_case(K, d, seed=0, n=3 * LR + 21, binarize=None):
    """The discrete-NB jll f(x) W^T + b on exact data: counts in [0, 3], W multiples of 1/8 in [-2, 0], b multiples of
    1/8 in [-4, -1].  Classes CW - 1 and CW (either side of the first block boundary; 1 and K - 2 when K fits one
    block) are copies with W[:, 0] = 0 and b = -1/2, and rows 3 e_0 tie on them; class K - 1 has b = 0, and zero rows
    pick it alone."""
    rng = np.random.RandomState(seed)
    _, cw, _ = linear_geom(K)
    W = -rng.randint(0, 17, (K, d)) / 8.0
    b = -rng.randint(8, 33, K) / 8.0
    a, bb = (cw - 1, cw) if K > cw else (1, K - 2)
    W[:, 0] = -2.0
    W[bb], W[a, 0], W[bb, 0] = W[a], 0.0, 0.0
    b[a] = b[bb] = -0.5
    last = K - 1 if K - 1 not in (a, bb) else None
    if last is not None:
        b[last] = 0.0
    x = rng.randint(0, 4, (n, d)).astype(np.float64)
    tie_rows, zero_rows = _perm_place(rng, n, [10, 10])
    x[tie_rows] = 0.0
    x[tie_rows, 0] = 3.0
    x[zero_rows] = 0.0
    return types.SimpleNamespace(x=x, W=W, b=b, K=K, tie=(a, bb), last=last, binarize=binarize, zero_rows=zero_rows,
                                 tie_rows=tie_rows)


def linear_ref(c, order=1):
    f = c.x if c.binarize is None else (c.x > c.binarize).astype(np.float64)
    jll = f[:, ::order] @ c.W[:, ::order].T + c.b[None]
    vmax = jll.max(1, keepdims=True)
    lp = jll - (np.log(np.exp(jll - vmax).sum(1, keepdims=True)) + vmax)
    return jll, np.argmax(jll, 1), lp


def project_case(k, d, seed=0, n=None, shift=True):
    """(x - s) W^T on exact data: s integers in [-2, 2], x - s integers in [-4, 4], W multiples of 1/8 in [-2, 2].  For
    every column c one row is s + 4 sign(W_c) (the column's largest |out|) and one is s - 4 sign(W_c) (the same |out|,
    the other sign), at random places: the arg-max record must take the lower row."""
    rng = np.random.RandomState(seed)
    n = n or 2 * k + 3 * PR + 5
    s = rng.randint(-2, 3, d).astype(np.float64) if shift else np.zeros(d)
    W = rng.randint(-16, 17, (k, d)) / 8.0
    u = rng.randint(-4, 5, (n, d)).astype(np.float64)
    pos, neg = _perm_place(rng, n, [k, k])
    u[pos] = 4.0 * np.sign(W)
    u[neg] = -4.0 * np.sign(W)
    return types.SimpleNamespace(x=u + s[None], shift=s if shift else None, W=W, k=k)


def project_ref(c, order=1, row_offset=0):
    """out and the (k, 3) arg-max records [|out| max, lowest row, signed value]."""
    s = c.shift if c.shift is not None else 0.0
    out = (c.x - s)[:, ::order] @ c.W[:, ::order].T
    r = np.argmax(np.abs(out), 0)
    cols = np.arange(c.k)
    return out, np.stack([np.abs(out[r, cols]), (r + row_offset).astype(np.float64), out[r, cols]], 1)


def colmax_merge(a, b):
    """Two arg-max records of the same columns: the larger |out|, then the lower row."""
    take_b = (b[:, 0] > a[:, 0]) | ((b[:, 0] == a[:, 0]) & (b[:, 1] < a[:, 1]))
    return np.where(take_b[:, None], b, a)


def rows_last_split_one(d, sms, n0, geom=gram_geom):
    """The smallest n >= n0 whose last row split holds one row (the first n >= n0 when every n has one split)."""
    for n in range(n0, n0 + 4096):
        g = geom(n, d, sms)
        if g.splits > 1 and n - (g.splits - 1) * g.rows_per_split == 1:
            return n
    return n0


def gram_ds(sms):
    """Gram widths: either side of the one-split threshold, 2049, and 64 m + 1, 64 m + 63 for m = 1, 2."""
    t = gram_one_split_d(sms)
    return [t - 1, t, 2049, 65, 127, 129, 191]


def gram_case(d, sms, seed=0):
    """Two blocks of d columns (a first call and an accumulating call with other row splits): integers in [-3, 3],
    shift integers in [-1, 1], row weights in {1/4, 1/2, 1, 2}.  Block A has one row in its last split."""
    rng = np.random.RandomState(seed)
    nA = rows_last_split_one(d, sms, 40)
    nB = max(1, nA // 2 + 7)
    xs = [rng.randint(-3, 4, (n, d)).astype(np.float64) for n in (nA, nB)]
    ws = [rng.choice([0.25, 0.5, 1.0, 2.0], n) for n in (nA, nB)]
    return types.SimpleNamespace(xs=xs, ws=ws, shift=rng.randint(-1, 2, d).astype(np.float64), d=d)


def gram_ref(c, order=1):
    """(colsum, Gram, weighted Gram) of both blocks."""
    cs, G, H = 0.0, 0.0, 0.0
    for x, w in zip(c.xs, c.ws):
        u = (x - c.shift[None])[::order]
        cs = cs + u.sum(0)
        G = G + u.T @ u
        H = H + (x[::order] * w[::order, None]).T @ x[::order]
    return cs, G, H


def mom_case(d, K, seed=0):
    """Two blocks of d columns (600 and 300 rows: other row splits): integers in [-3, 3], class indices in [-1, K]
    (-1 and K are skipped), integer theta, row weights in {1/4, 1/2, 1, 2}."""
    rng = np.random.RandomState(seed)
    xs = [rng.randint(-3, 4, (n, d)).astype(np.float64) for n in (600, 300)]
    cls = [rng.randint(-1, K + 1, n) for n in (600, 300)]
    for c in cls:
        c[:3] = [0, K - 1, K - 1]
    ws = [rng.choice([0.25, 0.5, 1.0, 2.0], n) for n in (600, 300)]
    return types.SimpleNamespace(xs=xs, cls=cls, ws=ws, theta=rng.randint(-2, 3, (K, d)).astype(np.float64), d=d, K=K)


def mom_ref(c, order=1, binarize=None):
    """(sums, counts, squared deviations, weighted feature counts, weighted class counts) over both blocks."""
    K, d = c.K, c.d
    S, C, Q, F, CC = (np.zeros((K, d)), np.zeros(K), np.zeros((K, d)), np.zeros((K, d)), np.zeros(K))
    for x, y, w in zip(c.xs, c.cls, c.ws):
        x, y, w = x[::order], y[::order], w[::order]
        keep = (y >= 0) & (y < K)
        oh = np.zeros((len(y), K))
        oh[np.nonzero(keep)[0], y[keep]] = 1.0
        f = x if binarize is None else (x > binarize).astype(np.float64)
        S += oh.T @ x
        C += oh.sum(0)
        Q += np.stack([((x[y == k] - c.theta[k]) ** 2).sum(0) for k in range(K)])
        F += (oh * w[:, None]).T @ f
        CC += (oh * w[:, None]).sum(0)
    return S, C, Q, F, CC


def glm_case(d, sms, seed=0, family=1):
    """Two blocks of d columns: A of 3 SMs x 32 + 45 rows (every CTA of the grid, some with two tiles, a partial last
    tile), B of 700 rows (another grid).  x integers in [-2, 2], beta multiples of 1/16 in [-1, 1] (1/256 for the
    logistic and Poisson families, so that eta stays moderate), y integers (counts for Poisson, 0 / 1 for logistic)."""
    rng = np.random.RandomState(seed)
    ns = (3 * sms * GLM_TR + 45, 700)
    xs = [rng.randint(-2, 3, (n, d)).astype(np.float64) for n in ns]
    den = 16.0 if family == 1 else 256.0
    beta = rng.randint(-16, 17, d + 1) / den
    if family == 0:
        ys = [rng.randint(0, 2, n).astype(np.float64) for n in ns]
    elif family == 2:
        ys = [rng.randint(0, 5, n).astype(np.float64) for n in ns]
    else:
        ys = [rng.randint(-20, 21, n).astype(np.float64) for n in ns]
    return types.SimpleNamespace(xs=xs, ys=ys, beta=beta, d=d, family=family)


def glm_terms(c, x, y, order=1):
    """(mu, loss, r, w) per row of one block, as family_terms (bkm_glm.cu:79-99)."""
    eta = x[:, ::order] @ c.beta[:c.d][::order] + c.beta[c.d]
    if c.family == 0:
        e = np.exp(-np.abs(eta))
        mu = np.where(eta >= 0, 1.0 / (1.0 + e), e / (1.0 + e))
        return mu, (np.maximum(eta, 0) + np.log1p(e)) - y * eta, mu - y, mu * (1.0 - mu)
    if c.family == 1:
        return eta, (y - eta) ** 2, 2.0 * (eta - y), np.full_like(eta, 2.0)
    mu = np.exp(eta)
    return mu, mu - y * eta, mu - y, mu


def glm_ref(c, order=1):
    """(grad [d + 2], hrow [d + 1], w of each block, mu of each block, and the scales |r| |x|, |w| |x| of the sums)."""
    grad, hrow, gs, hs = np.zeros(c.d + 2), np.zeros(c.d + 1), np.zeros(c.d + 2), np.zeros(c.d + 1)
    ws, mus = [], []
    for x, y in zip(c.xs, c.ys):
        mu, loss, r, w = glm_terms(c, x, y, order)
        xo, ro, wo = x[::order], r[::order], w[::order]
        grad += np.concatenate([xo.T @ ro, [ro.sum(), loss[::order].sum()]])
        hrow += np.concatenate([xo.T @ wo, [wo.sum()]])
        gs += np.concatenate([np.abs(x).T @ np.abs(r), [np.abs(r).sum(), np.abs(loss).sum()]])
        hs += np.concatenate([np.abs(x).T @ np.abs(w), [np.abs(w).sum()]])
        ws.append(w)
        mus.append(mu)
    return grad, hrow, ws, mus, gs, hs
