"""float32 restatement of fcn_rank_fold (the rank-ordered sum of G rows) and inputs on which the order of the adds
shows in the bits."""
import numpy as np

F32 = np.float32


def left_fold(rows):
    """((rows[0] + rows[1]) + rows[2]) + ... in float32, each add rounded to nearest even (numpy's float32 add)."""
    rows = np.asarray(rows, dtype=F32)
    acc = rows[0].copy()
    with np.errstate(invalid="ignore", over="ignore"):
        for r in rows[1:]:
            acc = np.add(acc, r, dtype=F32)
    return acc


def same_bits(a, b):
    """Equal bit for bit, except that any NaN equals any NaN (a NaN's payload is not part of the contract)."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a.view(np.uint32)[~na], b.view(np.uint32)[~nb]))


SPECIALS = np.array([1.0, -1.0, 2.0 ** 24, -(2.0 ** 24), 2.0 ** -140, -(2.0 ** -140), 2.0 ** -149, 3 * 2.0 ** -149,
                     2.0 ** -126, 0.0, -0.0, 0.5, 3.0, 2.0 ** 23], dtype=F32)
PZERO, NZERO = F32(0.0), F32(-0.0)


def order_sensitive(G, n, seed, with_inf=True, with_nan=True):
    """(G, n) float32 rows: mostly values drawn from SPECIALS (1, +-2^24, subnormals, +-0) and scaled normals, a few
    +-inf and NaN.  Column i % 4 == 0 of the first 1024 columns holds the pattern 2^24, 1, 1, ..., whose left fold
    (2^24, since each 2^24 + 1 rounds back) differs from the reverse fold (2^24 + G - 1, for G >= 3 even)."""
    rng = np.random.default_rng(seed)
    pick = rng.integers(0, len(SPECIALS), size=(G, n))
    rows = SPECIALS[pick]
    normal = rng.random((G, n)) < 0.4
    rows[normal] = (rng.standard_normal(int(normal.sum())) * np.exp2(rng.integers(-20, 25, int(normal.sum())))
                    ).astype(F32)
    if with_inf:
        rows[rng.random((G, n)) < 0.002] = np.inf
        rows[rng.random((G, n)) < 0.002] = -np.inf
    if with_nan:
        rows[rng.random((G, n)) < 0.001] = np.nan
    if n >= 8:
        if with_nan:
            rows[G - 1, 5] = np.nan
        if with_inf:
            rows[:, 6:8] = F32(1.0)
            rows[0, 6], rows[G - 1, 7] = np.inf, -np.inf
    cols = np.arange(0, min(n, 1024), 4)
    rows[:, cols] = F32(1.0)
    rows[0, cols] = F32(2.0 ** 24)
    return np.ascontiguousarray(rows, dtype=F32)
