"""Deterministic inputs of the wide-code-row golden fixtures (tests/golden/wide_*.npz) -- TEST INFRASTRUCTURE ONLY.

oracle/make_wide_golden.py feeds these to the compiled reference and stores only what the reference returned; the
tests rebuild the same inputs here instead of reading them from the fixture, which keeps the files small.  Nothing
depends on numpy's random streams: every value comes from a splitmix64 hash of its position, and the PQ codes come
from the C oracle's encoder (plain sequential fp32, first minimum), which both sides run on the same inputs.

* X (N, D), Q (nq, D): sums of four hash bytes on a 1/128 grid (roughly gaussian, std ~1.15), exact in fp32;
* codebook (M, Ks, ds): rows of X picked by the hash, divided by 32 for COSINE (exact; no normalisation involved);
* codes (N, M): the oracle's encoding of X (of X / 32 for COSINE), handed to the reference's add_items;
* labels: a hash permutation of 0..N-1, times 2 plus 5; `allow`: the labels whose hash bit is set; deleted: every 9th.
"""
import numpy as np

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def _mix(x):
    """splitmix64 finaliser over a uint64 array (wrapping arithmetic)."""
    with np.errstate(over='ignore'):
        z = (np.asarray(x, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)) & _M64
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def _hash(seed, stream, n):
    base = (np.uint64(seed) << np.uint64(40)) ^ (np.uint64(stream) << np.uint64(32))
    return _mix(base + np.arange(n, dtype=np.uint64))


def _grid(seed, stream, rows, cols):
    h = _hash(seed, stream, rows * cols)
    b = sum(((h >> np.uint64(8 * i)) & np.uint64(0xFF)).astype(np.int32) for i in range(4))
    return ((b - 510).astype(np.float32) / np.float32(128)).reshape(rows, cols)


def wide_inputs(N, D, M, Ks, metric, seed, nq):
    """-> dict(X, Q, codebook, codes, labels, allow, deleted) for one fixture."""
    import oracle as O
    X = _grid(seed, 1, N, D)
    Q = _grid(seed, 2, nq, D)
    ds = D // M
    pick = np.argsort(_hash(seed, 3, M * N).reshape(M, N), axis=1, kind='stable')[:, :Ks]
    cb = np.stack([X[pick[m], m * ds:(m + 1) * ds] for m in range(M)]).astype(np.float32)
    if metric == 'cosine':
        cb = cb / np.float32(32)
    codes = O.encode(X / np.float32(32) if metric == 'cosine' else X, cb)
    labels = np.argsort(_hash(seed, 4, N), kind='stable').astype(np.uint64) * 2 + 5
    allow = np.sort(labels[(_hash(seed, 5, N) & np.uint64(1)) == 1])
    return dict(X=X, Q=Q, codebook=cb, codes=codes, labels=labels, allow=allow, deleted=labels[::9].copy())
