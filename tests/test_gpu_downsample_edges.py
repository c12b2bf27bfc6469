"""GPU voxel-grid downsampling at its edges, bit for bit against the oracle in both bin orders, with normals and
colours: non-finite points (they belong to no bin, so the output equals the output for the cloud without them, through
cb_grid_downsample and cb_cloud_grid_downsample), NaN normals on finite points, point counts at the radix sort's
4096-element tile, bin keys of exactly 1, 8, 9, 16, 17 and 58 bits (odd and even pass counts), the first-occurrence
re-sort at 8 and 9 index bits, and points on exact bin faces."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _same(got, want):
    """Equal bit patterns, except that any NaN matches any NaN (the device's NaN payload is canonical)."""
    for g, w in zip(got, want):
        assert (g is None) == (w is None)
        if g is not None:
            g, w = np.ascontiguousarray(g, np.float32), np.ascontiguousarray(w, np.float32)
            assert g.shape == w.shape, (g.shape, w.shape)
            ok = (g.view(np.uint32) == w.view(np.uint32)) | (np.isnan(g) & np.isnan(w))
            assert ok.all(), f"{(~ok).sum()} differing words"


def _unit(rng, n):
    v = rng.normal(size=(n, 3))
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


def _dense(n, seed):
    rng = np.random.default_rng(seed)
    pts = rng.random((n, 3), dtype=np.float32)
    nrm = _unit(rng, n)
    nrm[rng.random(n) < 0.3] *= -1
    col = rng.random((n, 3), dtype=np.float32)
    return pts, nrm, col


def _insert(pts, nrm, col, bad, rng):
    """pts / nrm / col with the rows `bad` inserted at random positions (finite normals and colours)."""
    n, k = len(pts), len(bad)
    pos = np.sort(rng.choice(n + k, size=k, replace=False))
    keep = np.ones(n + k, bool)
    keep[pos] = False
    out = []
    for a, fill in ((pts, bad), (nrm, _unit(rng, k)), (col, rng.random((k, 3), dtype=np.float32))):
        full = np.empty((n + k, 3), np.float32)
        full[keep] = a
        full[pos] = fill
        out.append(full)
    return out


def _bad_rows(pts, rng):
    """Rows whose finite coordinates sit inside the dense cloud, so that clamping a NaN / Inf coordinate into the grid
    would land them in occupied bins of the first and last x-slabs; plus all-NaN / all-Inf rows."""
    yz = pts[rng.choice(len(pts), 8)][:, 1:]
    rows = [[np.nan, *yz[0]], [np.inf, *yz[1]], [-np.inf, *yz[2]], [np.nan, *yz[3]], [np.inf, *yz[4]],
            [yz[5][0], np.nan, yz[5][1]], [yz[6][0], yz[6][1], -np.inf], [-np.inf, *yz[7]],
            [np.nan] * 3, [np.inf] * 3, [-np.inf] * 3, [np.inf, -np.inf, np.nan]]
    return np.array(rows, np.float32)


@pytest.mark.parametrize("order", [0, 1])
def test_nonfinite_points_belong_to_no_bin(cb, ctx, orc, order):
    rng = np.random.default_rng(30)
    pts, nrm, col = _dense(20000, 31)
    dp, dn, dc = _insert(pts, nrm, col, _bad_rows(pts, rng), rng)
    for minp in (1, 3):
        want = orc.grid_downsample(pts, 0.05, normals=nrm, colors=col, min_points=minp, order=order)
        _same(cb.grid_downsample(ctx, dp, 0.05, normals=dn, colors=dc, min_points=minp, order=order), want)
        ds = cb.Cloud(ctx, dp, dn).grid_downsample(0.05, min_points=minp, order=order)
        p, q = ds.download(normals=True)
        _same((p, q), want[:2])


def test_all_nonfinite_cloud_gives_empty_output(cb, ctx):
    bad = np.array([[np.nan, 0, 0], [np.inf, 1, 1], [0, -np.inf, 0], [np.nan] * 3] * 3, np.float32)
    nrm = np.tile(np.float32([0, 0, 1]), (len(bad), 1))
    for order in (0, 1):
        p, q, c = cb.grid_downsample(ctx, bad, 0.1, normals=nrm, colors=nrm, order=order)
        assert p.shape == q.shape == c.shape == (0, 3)
        assert cb.Cloud(ctx, bad, nrm).grid_downsample(0.1, order=order).n == 0


@pytest.mark.parametrize("order", [0, 1])
def test_nan_normals_on_finite_points_propagate_like_the_oracle(cb, ctx, orc, order):
    """Normal estimation leaves NaN normals below 3 neighbours; a bin holding one has a NaN normal, as in the
    reference."""
    rng = np.random.default_rng(32)
    pts, nrm, col = _dense(30000, 33)
    nrm[rng.random(len(nrm)) < 0.02] = np.nan
    got = cb.grid_downsample(ctx, pts, 0.05, normals=nrm, colors=col, order=order)
    want = orc.grid_downsample(pts, 0.05, normals=nrm, colors=col, order=order)
    _same(got, want)
    assert np.isnan(want[1]).any() and not np.isnan(want[1]).all()


@pytest.mark.parametrize("n", [4095, 4096, 4097, 8193])
def test_sizes_at_radix_tile_edges(cb, ctx, orc, n):
    pts, nrm, col = _dense(n, n)
    for order in (0, 1):
        _same(cb.grid_downsample(ctx, pts, 0.2, normals=nrm, colors=col, order=order),
              orc.grid_downsample(pts, 0.2, normals=nrm, colors=col, order=order))


def _bits_for(count):
    return max(1, int(count - 1).bit_length())


# bins per axis (bin size 1); the key range is their product plus one key for non-finite points
KEY_DIMS = {1: (1, 1, 1), 8: (200, 1, 1), 9: (300, 1, 1), 16: (200, 200, 1), 17: (400, 250, 1),
            58: (1 << 20, 1 << 20, 1 << 17)}


@pytest.mark.parametrize("bits", list(KEY_DIMS))
def test_key_widths(cb, ctx, orc, bits):
    dims = np.array(KEY_DIMS[bits], np.int64)
    assert _bits_for(int(np.prod(dims)) + 1) == bits
    rng = np.random.default_rng(bits)
    cells = np.vstack([np.zeros(3, np.int64), dims - 1, (rng.random((60, 3)) * dims).astype(np.int64)])
    which = np.concatenate([np.arange(len(cells)), rng.integers(0, len(cells), 3000)])
    pts = (cells[which] + rng.uniform(0.25, 0.75, (len(which), 3))).astype(np.float32)
    nrm, col = _unit(rng, len(pts)), rng.random((len(pts), 3), dtype=np.float32)
    for order in (0, 1):
        _same(cb.grid_downsample(ctx, pts, 1.0, normals=nrm, colors=col, order=order),
              orc.grid_downsample(pts, 1.0, normals=nrm, colors=col, order=order))


@pytest.mark.parametrize("n", [256, 257])
def test_first_occurrence_resort_index_bits(cb, ctx, orc, n):
    rng = np.random.default_rng(n)
    pts = rng.random((n, 3), dtype=np.float32)
    for b in (0.1, 0.3):  # most points alone in their bin; then several per bin
        _same(cb.grid_downsample(ctx, pts, b, order=1), orc.grid_downsample(pts, b, order=1))


def test_exact_bin_faces(cb, ctx, orc):
    """p * (1 / bin) exactly an integer (bin 0.25, inverse 4 exactly), on both sides of zero, and -0.0."""
    rng = np.random.default_rng(34)
    pts = (rng.integers(-12, 13, (3000, 3)) * 0.25).astype(np.float32)
    pts[:50] = -0.0
    pts[50:60, 0] = -0.0
    nrm, col = _unit(rng, len(pts)), rng.random((len(pts), 3), dtype=np.float32)
    for order in (0, 1):
        got = cb.grid_downsample(ctx, pts, 0.25, normals=nrm, colors=col, order=order)
        _same(got, orc.grid_downsample(pts, 0.25, normals=nrm, colors=col, order=order))
        assert got[0].shape[0] == len(np.unique(pts + np.float32(0.0), axis=0))
