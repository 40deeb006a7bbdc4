"""Float64 references of the operations that turn vectors into codes, tables and cell orders, each with the bound that
an fp32 evaluation of it must stay inside, and the acceptance rules every check of those kernels uses.

Each helper computes the reference's formula in float64 (its own rounding is far below the fp32 bounds) and returns the
bound of the standard form  gamma_n * sum|terms| + n * eta:
  u     = 2^-24, the unit roundoff of fp32 round-to-nearest;
  gamma_n = n u / (1 - n u), the relative error of n chained roundings;
  eta   = 2^-150, half the smallest fp32 subnormal: the absolute error of a product that underflows (additions and
          subtractions are exact when their result is subnormal, so only products contribute it);
  n     = the length of the sequential chain, plus the warp-tree depth where a kernel reduces across lanes.
The bounds hold whatever order the sum runs in (any order's error is within gamma_(terms - 1)), so they serve the
oracle's fp32 restatements, numpy, and the CUDA kernels alike; they are not a model of any one rounding order.

Acceptance rules (written once here, used by tests/test_numeric_bounds.py and tests/test_gpu_numeric_edges.py):
  values          |fp32 - ref64| <= bound;
  argmin outputs  the chosen index c is accepted only if ref64[c] - bound(c) <= min over a of (ref64[a] + bound(a))
                  (c could be the minimum under some admissible rounding); fp32 overflow is part of the model;
  exact ties      duplicate codewords and all-+inf rows: the lower index, exactly (checked by the tests directly).
"""
import numpy as np

U = 2.0 ** -24
ETA = 2.0 ** -150
FLT_MAX = float(np.finfo(np.float32).max)
EPS32 = float(np.finfo(np.float32).eps)
# annlite.math.l2_normalize's switch `norms < 10 * eps`, evaluated in fp32 as the reference and the kernel do
NORM_FLOOR = float(np.float32(10) * np.float32(EPS32))
WARP_TREE = 5  # log2(32): the shuffle reductions of l2_normalize and the probe's |x|^2


def gamma(n):
    n = np.asarray(n, dtype=np.float64)
    return n * U / (1.0 - n * U)


def _f64(a):
    return np.asarray(a, dtype=np.float64)


# ---- squared L2 to every codeword (PQ encode, VQ assignment, the L2 ADC table) ------------------------------------
def sq_l2(x, w):
    """x (B, ds), w (K, ds) -> (ref (B, K), bound (B, K)): sum_j (x_j - w_j)^2.

    fp32: t = fl(x_j - w_j) = (x_j - w_j)(1 + d1); fl(t * t) = t^2 (1 + d2) (+ eta if it underflows); then a chain of
    ds - 1 additions.  Every term carries at most (1 + u)^(2 + 1 + ds - 1) - 1 <= gamma_(ds + 2) of relative error,
    and the ds underflow errors, carried through the chain, stay below 2 ds eta."""
    x, w = _f64(x), _f64(w)
    ds = x.shape[1]
    ref = np.stack([((w - r[None, :]) ** 2).sum(-1) for r in x]) if len(x) else np.zeros((0, len(w)))
    return ref, gamma(ds + 2) * ref + 2 * ds * ETA


def ip_table(x, w, bias):
    """x (B, ds), w (K, ds) -> (ref, bound): bias - sum_j w_j x_j, with bias = fp32(1/Ks) (or 0 for the raw form).

    fp32: ds products (1 + d) each, ds - 1 chained additions: gamma_ds * sum|w x| on the sum; the final subtraction
    adds u * |bias - acc| <= u (|bias| + sum|w x|) (1 + gamma_ds).  Together within gamma_(ds + 1) (|bias| + sum|w x|)
    plus the underflow term."""
    x, w = _f64(x), _f64(w)
    ds = x.shape[1]
    ref = float(bias) - x @ w.T
    return ref, gamma(ds + 1) * (abs(float(bias)) + np.abs(x) @ np.abs(w).T) + 2 * ds * ETA


def table_ref(q, cb, metric, bias=None):
    """The (B, M, Ks) ADC table of queries q (B, M*ds) over codebooks cb (M, Ks, ds) in float64, and its bound.
    `metric` 'euclidean' or 'inner_product' (a cosine table is the inner-product table of the normalised query)."""
    q, cb = _f64(q), _f64(cb)
    M, Ks, ds = cb.shape
    if bias is None:
        bias = float(np.float32(1.0 / Ks))
    ref = np.empty((q.shape[0], M, Ks))
    bnd = np.empty_like(ref)
    for m in range(M):
        sub = q[:, m * ds:(m + 1) * ds]
        r, b = sq_l2(sub, cb[m]) if metric == 'euclidean' else ip_table(sub, cb[m], bias)
        ref[:, m], bnd[:, m] = r, b
    return ref, bnd


# ---- argmin acceptance -----------------------------------------------------------------------------------------
def argmin_ok(ref, bound, chosen):
    """ref, bound (B, K) float64; chosen (B,) -> bool (B,): could an fp32 evaluation within `bound` of `ref`, with fp32
    overflow to +inf, have `chosen` as its first minimum?  Where every value must overflow, the first minimum of an
    all-+inf row is index 0, and only 0 is accepted."""
    ref, bound = _f64(ref), _f64(bound)
    chosen = np.asarray(chosen, dtype=np.int64)
    K = ref.shape[1]
    if (chosen < 0).any() or (chosen >= K).any():
        return np.zeros(len(chosen), dtype=bool)
    lo, hi = ref - bound, ref + bound
    lo = np.where(lo > FLT_MAX, np.inf, lo)
    hi = np.where(hi > FLT_MAX, np.inf, hi)
    rows = np.arange(len(chosen))
    lo_c = lo[rows, chosen]
    ok = lo_c <= hi.min(1)
    must_inf = np.isinf(lo_c)
    return np.where(must_inf, np.isinf(hi).all(1) & (chosen == 0), ok)


def encode_ok(x, cb, codes):
    """PQ / VQ codes (B, M) of rows x (B, M*ds) over codebooks cb (M, Ks, ds): bool (B, M) by the argmin rule."""
    M, Ks, ds = cb.shape
    codes = np.asarray(codes).astype(np.int64)
    out = np.empty(codes.shape, dtype=bool)
    for m in range(M):
        ref, bnd = sq_l2(np.asarray(x)[:, m * ds:(m + 1) * ds], cb[m])
        out[:, m] = argmin_ok(ref, bnd, codes[:, m])
    return out


# ---- l2_normalize ------------------------------------------------------------------------------------------------
def l2_normalize_ref(x, n):
    """x (B, D) -> (ref, bound, mode): annlite.math.l2_normalize, x / max(|x|, 1 if |x| < 10 eps), in float64.

    The sum of squares s is a chain of n roundings (n = the longest chain plus tree depth of the evaluation), so
    |s^ - s| <= gamma_n s + 2 D eta; sqrt adds u and halves the relative error of s; the division adds u.  An output
    element is therefore within (gamma_n / 2 + 2u) (1 + 2^-20) |ref| + 2 eta of ref64.  `mode` per row:
      'scaled'       the norm is clear of the switch: the output is x / |x|;
      'unchanged'    the norm is clear below the switch: x / 1, exactly x;
      'either'       |x| lies within its own bound of 10 eps: either outcome is accepted, and only there;
      'overflow'     s must exceed FLT_MAX in fp32: the norm is +inf, so the output is exactly 0 (numpy's fp32 formula
                     gives the same)."""
    x = _f64(x)
    D = x.shape[1]
    s = (x * x).sum(1)
    g = gamma(n)
    s_err = g * s + 2 * D * ETA
    norm = np.sqrt(s)
    # the norm's own error, from s's: sqrt(s + e) - sqrt(s) <= e / (2 sqrt(s)) or sqrt(e) near 0; plus the sqrt's u
    norm_err = np.minimum(np.sqrt(s_err), s_err / np.maximum(2 * norm, 1e-300)) + U * norm
    mode = np.full(len(x), 'scaled', dtype=object)
    mode[norm + norm_err < NORM_FLOOR] = 'unchanged'
    mode[np.abs(norm - NORM_FLOOR) <= norm_err] = 'either'
    mode[s * (1 - g) > FLT_MAX] = 'overflow'
    ref = x / np.where(mode == 'unchanged', 1.0, norm)[:, None]
    bound = (g / 2 + 2 * U) * (1 + 2.0 ** -20) * np.abs(ref) + 2 * ETA
    return ref, bound, mode


def l2_normalize_ok(x, got, n):
    """bool (B,): every element of row i of `got` accepted for the l2_normalize of x[i] (rule of l2_normalize_ref)."""
    ref, bound, mode = l2_normalize_ref(x, n)
    x = _f64(x)
    got = _f64(got)
    scaled = (np.abs(got - ref) <= bound).all(1)
    same = (got == x).all(1)
    zero = (got == 0).all(1)
    return np.where(mode == 'scaled', scaled,
                    np.where(mode == 'unchanged', same,
                             np.where(mode == 'either', scaled | same, zero)))


def l2_normalize_chain(D):
    """n of l2_normalize_kernel: a lane's chain of ceil(D / 32) products and sums, then the 5-level shuffle tree."""
    return -(-D // 32) + 1 + WARP_TREE


# ---- cell probe (annlite.math.cdist) -----------------------------------------------------------------------------
def probe_ref(x, cen, cosine, n):
    """Query x (D,) against centroids cen (C, D) -> (val, bound) per centroid, the quantity the probe orders by.

    Euclidean: the radicand |y|^2 + |x|^2 - 2 x.y, not its sqrt: the three sums are chains of at most n roundings
    (gamma_n on each), the two combining operations add 2u, and the final sqrt may merge radicands within 2u of
    each other (ties then go by index): bound = gamma_(n+4) (|x|^2 + |y|^2 + 2 |x||.|y|) + 4 n eta.  A radicand within
    its bound of 0 may round below zero, where sqrt gives NaN and the probe sorts the cell last.
    Cosine: d = 1 - clip(r, -1, 1) with r = (x.y + eps) / (|x| |y| + eps).  The numerator is within
    gamma_(n+1) (|x||.|y| + eps); each norm within gamma_n / 2 + u relative, their product and + eps within 2u more, the
    division u: |r^ - r| <= (num_err + |r| den_err) / (den - den_err) + u |r|, clip is 1-Lipschitz, and `1 -` adds at
    most u |d| <= 2u.  The bound is on d, derived from that of the ratio (the output's own relative error is useless
    near d = 0)."""
    x, cen = _f64(x), _f64(cen)
    xx = (x * x).sum()
    yy = (cen * cen).sum(1)
    axy = (np.abs(x)[None, :] * np.abs(cen)).sum(1)
    xy = (x[None, :] * cen).sum(1)
    D = x.shape[0]
    if not cosine:
        val = yy + xx - 2 * xy
        return val, gamma(n + 4) * (xx + yy + 2 * axy) + 4 * D * ETA
    g = gamma(n)
    den = np.sqrt(xx) * np.sqrt(yy) + EPS32
    num = xy + EPS32
    num_err = gamma(n + 1) * (axy + EPS32) + 2 * D * ETA
    den_err = (g + 3 * U) * np.sqrt(xx) * np.sqrt(yy) + U * den + 2 * D * ETA
    r = num / den
    r_err = (num_err + np.abs(r) * den_err) / np.maximum(den - den_err, 1e-300) + U * np.abs(r)
    d = 1 - np.clip(r, -1, 1)
    return d, (r_err + 2 * U) * (1 + 2.0 ** -20)


def probe_order_ok(x, cen, cosine, order, n):
    """bool: `order` (a permutation prefix of the centroids) is an ascending order of the probe distances under some
    admissible rounding: for every adjacent pair (a, b), val[a] - val[b] <= bound(a) + bound(b), unless b's radicand
    may have rounded below zero (a NaN distance, sorted last)."""
    val, bnd = probe_ref(x, cen, cosine, n)
    order = np.asarray(order, dtype=np.int64)
    a, b = order[:-1], order[1:]
    ok = val[a] - val[b] <= bnd[a] + bnd[b]
    if not cosine:
        ok |= val[b] <= bnd[b]
    return bool(ok.all())


def probe_chain(D):
    """n of cell_probe_kernel's sums: |x|^2 is a lane chain plus the shuffle tree, |y|^2 and x.y one chain of D fused
    multiply-adds; D + 1 + 5 covers both (and any summation order numpy or BLAS may use for D terms)."""
    return D + 1 + WARP_TREE


# ---- the input grids, shared by the CPU self-check and the GPU tests ----------------------------------------------
ENCODE_KS = (1, 2, 31, 32, 33, 255, 256, 257, 1000, 65536)
ENCODE_DS = (1, 3, 4, 5, 40, 256)
# one subspace per magnitude: subnormal, small, unit, large (ds >= 40 at 1e18 reaches fp32 overflow)
ENCODE_SCALES = (1e-40, 1e-20, 1.0, 1e18)
OVERFLOW_COORD = 3e19   # (3e19)^2 = 9e38 > FLT_MAX: every fp32 distance of its subspace is +inf


def encode_grid():
    """(Ks, ds) pairs of the encode checks; a 65536-codeword book stays at ds <= 5 (268 MB at ds = 256)."""
    return [(ks, ds) for ks in ENCODE_KS for ds in ENCODE_DS if ks < 65536 or ds <= 5]


def encode_case(Ks, ds, seed=0):
    """Codebooks (4, Ks, ds), subspace m at ENCODE_SCALES[m], and rows (B, 4 * ds): Gaussian rows, rows equal to a
    codeword, rows equal to a duplicated codeword (the duplicate one lane over and, for Ks > 35, in the same lane 32
    codewords on), and two rows whose unit-scale subspace holds OVERFLOW_COORD.  Returns (cb, x, ties): ties lists
    (row, subspace, code) where the fp32 minimum is an exact tie at distance 0 that the lower index must win."""
    rng = np.random.default_rng(seed + 1000 * Ks + ds)
    M = len(ENCODE_SCALES)
    scale = np.repeat(np.asarray(ENCODE_SCALES), ds)
    cb = np.stack([rng.standard_normal((Ks, ds)) * s for s in ENCODE_SCALES]).astype(np.float32)
    pairs = sorted({(a, b) for a, b in ((0, 1), (3, 35), (Ks - 2, Ks - 1)) if 0 <= a < b < Ks})
    for a, b in pairs:
        cb[:, b] = cb[:, a]
    gauss = rng.standard_normal((8, M * ds)) * scale
    at_code = np.concatenate([cb[m, rng.integers(0, Ks, size=4)] for m in range(M)], 1)
    at_dup = np.stack([cb[:, b].reshape(-1) for _a, b in pairs]) if pairs else np.zeros((0, M * ds))
    over = rng.standard_normal((2, M * ds)) * scale
    over[:, 2 * ds + (ds - 1) // 2] = OVERFLOW_COORD
    x = np.ascontiguousarray(np.concatenate([gauss, at_code, at_dup, over]), dtype=np.float32)
    # subspaces 0 and 1: squares of differences near the codewords' spacing underflow to 0, so other codewords can tie
    # there too; subspace 0's every distance is 0 (checked by its own rule)
    base = len(gauss) + len(at_code)
    ties = [(base + i, m, a) for i, (a, _b) in enumerate(pairs) for m in (2, 3)]
    return cb, x, ties


def overflow_rows(x):
    """Rows of an encode_case holding OVERFLOW_COORD (their subspace 2 distances are all +inf in fp32)."""
    return np.nonzero((np.asarray(x) == np.float32(OVERFLOW_COORD)).any(1))[0]


K1_DS = (1, 2, 7, 41, 42, 64, 200, 201, 256, 512)
K1_KS = (1, 7, 256, 257)


def k1_case(ds, Ks, seed=0, B=40):
    """Codebooks (2, Ks, ds) and B queries (B, 2 * ds); B = 40 spans a full and a partial 32-query tile."""
    rng = np.random.default_rng(seed + 7 * ds + Ks)
    cb = rng.standard_normal((2, Ks, ds)).astype(np.float32)
    q = rng.standard_normal((B, 2 * ds)).astype(np.float32)
    return cb, q


NORM_D = (1, 31, 32, 33, 768, 1000)


def norm_rows(D, seed=0):
    """Rows for l2_normalize at dimension D: Gaussian, zero, norms just either side of 10 eps (by less than the
    bound's width and by clearly more), overflowing sums of squares, subnormal rows, and mixed magnitudes."""
    rng = np.random.default_rng(seed + D)
    g = rng.standard_normal((6, D))
    unit = g / np.linalg.norm(g, axis=1, keepdims=True)
    rows = [g, np.zeros((1, D))]
    for f in (1 - 1e-7, 1 + 1e-7, 0.5, 2.0):            # straddling the switch, then clear of it
        rows.append(unit[:1] * NORM_FLOOR * f)
    rows.append(unit[:2] * 1e30)                       # sum of squares overflows fp32
    rows.append(np.full((1, D), 2e19))                 # each square overflows
    rows.append(unit[:2] * 1e-40 * np.sqrt(D))         # subnormal coordinates: the squares underflow
    mixed = g[:1].copy()
    mixed[0, 0] = 1e18
    rows.append(mixed)
    return np.ascontiguousarray(np.concatenate(rows), dtype=np.float32)


PROBE_CELLS = (1, 31, 32, 33, 255, 256)
PROBE_D = (1, 33, 768)


def probe_case(n_cells, D, seed=0, B=24):
    """Centroids (n_cells, D) and queries (B, D)."""
    rng = np.random.default_rng(seed + 31 * n_cells + D)
    cen = rng.standard_normal((n_cells, D)).astype(np.float32)
    q = rng.standard_normal((B, D)).astype(np.float32)
    return cen, q
