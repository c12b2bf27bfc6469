"""Inputs at the top of the fp32 range, shared by the grid, segmentation and mean-shift edge tests. Nothing here calls
the product or the oracle.

top_range_cloud: columns whose x and y take a few values in [2^126, FLT_MAX] (most with |x| + |y| + |z| >= 3e38) and
whose z is a dyadic lattice of step 1/4, so every d2 inside a column is an exact small dyadic number and every d2
between columns is Inf (the coordinate gaps are >= 2^104, their squares overflow). Exact duplicates included.
raised_origin_cloud: columns at x = -2^127 and x = 2^127 - 5 * 2^104, an x extent of FLT_MAX - 2^106 that leaves no
room for a margin cell below the box.
wide_cloud: clusters near -FLT_MAX and +FLT_MAX, an extent no fp32 difference can hold."""
import numpy as np

F32 = np.float32
FMAX = float(np.finfo(np.float32).max)
TOP = 2.0**127
GUARD = 3.0e38  # the sum of magnitudes above which the searches used to give up on a finite query
COLUMNS = ((TOP, TOP), (TOP + 2.0**105, TOP), (FMAX, FMAX), (FMAX, 1.5 * TOP), (1.5 * TOP, 2.0**126),
           (2.0**126, 2.0**126))


def _columns(cols, nz, seed, dups):
    rng = np.random.default_rng(seed)
    z = np.arange(nz, dtype=np.float64) * 0.25
    pts = np.array([[x, y, zz] for x, y in cols for zz in z], np.float64)
    pts = np.vstack([pts, pts[rng.choice(len(pts), dups, replace=False)]])
    pts = pts[rng.permutation(len(pts))]
    out = pts.astype(F32)
    assert np.array_equal(out.astype(np.float64), pts)  # every coordinate is exact in fp32
    return out


def top_range_cloud(seed=0, nz=48, dups=40, cols=COLUMNS):
    pts = _columns(cols, nz, seed, dups)
    assert (np.abs(pts.astype(np.float64)).sum(axis=1) >= GUARD).mean() > 0.7
    assert np.isin(FMAX, pts)
    return pts


def raised_origin_cloud(seed=1, nz=40, dups=20):
    hi = TOP - 5 * 2.0**104
    pts = _columns(((-TOP, TOP), (hi, TOP), (hi, 1.5 * TOP)), nz, seed, dups)
    assert np.ptp(pts[:, 0].astype(np.float64)) == FMAX - 2.0**106
    return pts


def wide_cloud(seed=2, n=200):
    rng = np.random.default_rng(seed)
    lo = np.column_stack([-FMAX + rng.integers(0, 8, n) * 2.0**104, rng.integers(0, 8, (n, 2)) * 0.5])
    hi = np.column_stack([FMAX - rng.integers(0, 8, n) * 2.0**104, rng.integers(0, 8, (n, 2)) * 0.5])
    return np.vstack([lo, hi]).astype(F32)


def top_range_queries(pts, seed=3):
    """The cloud itself, the cloud shifted by an eighth along z (exact), and queries at the corners of its x-y extent
    (a query cloud is indexed too, so it keeps to the cloud's extent), far along z, and non-finite."""
    rng = np.random.default_rng(seed)
    shifted = pts[rng.choice(len(pts), 200)].copy()
    shifted[:, 2] += F32(0.125)
    lo, hi = pts.min(axis=0), pts.max(axis=0)
    far = np.array([[hi[0], hi[1], 100.0], [lo[0], lo[1], 0.0], [lo[0], hi[1], 1e30], [hi[0], lo[1], -0.125],
                    [hi[0], hi[1], -1e30], [np.nan, hi[1], 0.0], [np.inf, hi[1], 0.0]], np.float64)
    return np.vstack([pts, shifted, far.astype(F32)]).astype(F32)
