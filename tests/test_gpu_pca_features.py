"""Covariance, PCA, projection and reconstruction over D-dimensional vector sets on the device (cb_vectors_mean_cov,
cb_vectors_pca, cb_vectors_project, cb_vectors_reconstruct) against the float64 / fp32 restatement of
pca_features_ref.py: the accuracy bound of DESIGN §4.18 on both sides of every tile and MMA edge, the non-finite rule,
the sample-size expressions, bit identities (repeat calls, subsets, D = 3 against the cloud path), PCA against eigh,
bit-exact projection and reconstruction, argument errors, constant launch counts and no device-memory growth."""
import numpy as np
import pytest

import kmeans_features_ref as kf
import pca_features_ref as pf
from test_gpu_device_memory import pool_used  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

# both sides of the 8 / 16 / 32 / 64 column tiles and of the 8-wide MMA fragments
DIMS = [1, 2, 4, 5, 6, 7, 8, 9, 15, 16, 17, 24, 31, 32, 33, 40, 63, 64, 65, 127, 128, 129, 200, 1024]


def _same_f32(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


def _rows(kind, n, D, rng):
    x = rng.standard_normal((n, D))
    if kind == "plain":
        return x.astype(np.float32)
    if kind == "offset_1e4":
        return (x + 1e4).astype(np.float32)
    if kind == "offset_1e6":
        return (x * 3 + 1e6).astype(np.float32)
    if kind == "far_pivot":  # the pivot rows sit far from the rest
        x[:4096] += 1e3
        return x.astype(np.float32)
    if kind == "zero_var":
        x[:, ::2] = 7.25
        return x.astype(np.float32)
    if kind == "rank_deficient":
        r = max(1, D // 3)
        return (rng.standard_normal((n, r)) @ rng.standard_normal((r, D)) + 5).astype(np.float32)
    if kind == "scales":
        return (x * np.logspace(-20, 18, D)).astype(np.float32)
    raise ValueError(kind)


def _check(cb, ctx, rows, subset=None):
    v = cb.Vectors(ctx, rows)
    mean, cov, ok = cb.mean_cov(ctx, v, subset=subset)
    rm, rc, rok = pf.mean_cov(rows, subset=subset)
    assert ok == rok
    assert pf.within_cov_bound(mean, cov, rm, rc), (np.nanmax(np.abs(mean - rm)), np.nanmax(np.abs(cov - rc)))
    return v, mean, cov


@pytest.mark.parametrize("D", DIMS)
def test_mean_cov_dims(cb, ctx, D):
    rng = np.random.default_rng(D)
    _check(cb, ctx, _rows("plain", 5000, D, rng))


@pytest.mark.parametrize("D", [6, 65])
@pytest.mark.parametrize("n", [2, 3, 31, 32, 33, 255, 256, 257, 4095, 4096, 4097, (1 << 20) + 1])
def test_mean_cov_sizes(cb, ctx, D, n):
    rng = np.random.default_rng(n + D)
    _check(cb, ctx, _rows("offset_1e4", n, D, rng))


@pytest.mark.parametrize("kind", ["offset_1e4", "offset_1e6", "far_pivot", "zero_var", "rank_deficient", "scales"])
@pytest.mark.parametrize("D", [5, 9, 40])
def test_mean_cov_inputs(cb, ctx, kind, D):
    rng = np.random.default_rng(D * 31 + len(kind))
    _check(cb, ctx, _rows(kind, 20000, D, rng))


def test_mean_cov_10m_rows_d6(cb, ctx):
    rng = np.random.default_rng(10)
    rows = (rng.standard_normal((10_000_000, 6), dtype=np.float32) * np.float32([1, 2, 3, 0.5, 10, 0.1]) +
            np.float32([1e3, -5, 0, 2e4, 1, 3]))
    _check(cb, ctx, rows)


@pytest.mark.parametrize("where", ["inside", "outside"])
def test_nonfinite_pattern(cb, ctx, where):
    rng = np.random.default_rng(11)
    rows = rng.standard_normal((6000, 9)).astype(np.float32)
    r = 100 if where == "inside" else 5000
    rows[r, 1] = np.nan
    rows[r, 3] = np.inf
    rows[r + 1, 4] = -np.inf
    rows[r + 2, 6], rows[r + 3, 6] = np.inf, -np.inf
    _, mean, cov = _check(cb, ctx, rows)
    assert np.isnan(cov[[1, 3, 4, 6], :]).all() and np.isfinite(cov[np.ix_([0, 2, 5, 7, 8], [0, 2, 5, 7, 8])]).all()
    assert np.isnan(mean[1]) and mean[3] == np.inf and mean[4] == -np.inf and np.isnan(mean[6])


@pytest.mark.parametrize("D", [3, 5])
@pytest.mark.parametrize("n", [0, 1, 2])
@pytest.mark.parametrize("min_size", [0, 1, 2, 5])
@pytest.mark.parametrize("use_subset", [False, True])
def test_min_sample_size(cb, ctx, D, n, min_size, use_subset):
    rows = (np.arange(4 * D, dtype=np.float32).reshape(4, D) * 0.5 - 1)
    full = rows[:n] if not use_subset else rows
    subset = list(range(n))[::-1] if use_subset else None
    v = cb.Vectors(ctx, full)
    mean, cov, ok = cb.mean_cov(ctx, v, subset=subset, min_sample_size=min_size)
    rm, rc, rok = pf.mean_cov(full, subset=subset, min_sample_size=min_size)
    assert ok == rok and pf.within_cov_bound(mean, cov, rm, rc)
    if n == 0 and ok:
        assert (cov == 0).all() and np.array_equal(np.signbit(cov), np.signbit(rc.astype(np.float32)))
    r = cb.pca(ctx, v, subset=subset, min_sample_size=min_size)
    assert r["ok"] == ok and _same_f32(r["mean"], mean) and _same_f32(r["cov"], cov)
    if not ok or (n == 1 and D != 3):
        assert np.isnan(r["eigenvalues"]).all() and np.isnan(r["eigenvectors"]).all()


@pytest.mark.parametrize("D", [2, 7, 64, 130])
def test_bit_identities(cb, ctx, D):
    rng = np.random.default_rng(D + 5)
    rows = _rows("offset_1e4", 9000, D, rng)
    v = cb.Vectors(ctx, rows)
    a = cb.pca(ctx, v)
    b = cb.pca(ctx, v)
    for key in ("mean", "cov", "eigenvalues", "eigenvectors"):
        assert _same_f32(a[key], b[key]), key
    subset = np.concatenate([rng.integers(0, 9000, 5000), [17, 17, 17]])
    s = cb.pca(ctx, v, subset=subset)
    g = cb.pca(ctx, cb.Vectors(ctx, rows[subset]))
    for key in ("mean", "cov", "eigenvalues", "eigenvectors"):
        assert _same_f32(s[key], g[key]), key


def test_d3_equals_cloud_path(cb, ctx):
    rng = np.random.default_rng(33)
    for n in (3, 4097, 100_000):
        pts = (rng.standard_normal((n, 3)) * [1, 2, 3] + [1e3, 0, -4]).astype(np.float32)
        mc, cc, okc = cb.mean_cov(ctx, cb.Cloud(ctx, pts))
        v = cb.Vectors(ctx, pts)
        mv, cv, okv = cb.mean_cov(ctx, v)
        assert okc == okv and _same_f32(mc, mv) and _same_f32(cc, cv)
        pc, pv = cb.pca(ctx, cb.Cloud(ctx, pts)), cb.pca(ctx, v)
        for key in ("mean", "cov", "eigenvalues", "eigenvectors"):
            assert _same_f32(pc[key], pv[key]), key


def _clusters(w, tol):
    groups, cur = [], [0]
    for j in range(1, len(w)):
        if abs(w[j - 1] - w[j]) <= tol:
            cur.append(j)
        else:
            groups.append(cur)
            cur = [j]
    return groups + [cur]


@pytest.mark.parametrize("D,kind", [(2, "plain"), (6, "offset_1e4"), (9, "rank_deficient"), (64, "plain"),
                                    (130, "zero_var"), (200, "plain")])
def test_pca_against_eigh(cb, ctx, D, kind):
    rng = np.random.default_rng(D * 3)
    rows = _rows(kind, 30000, D, rng)
    r = cb.pca(ctx, cb.Vectors(ctx, rows))
    assert r["ok"]
    w, V = np.linalg.eigh(r["cov"].astype(np.float64))
    w, V = w[::-1], V[:, ::-1]
    lmax = max(abs(w).max(), np.finfo(np.float64).tiny)
    ev = r["eigenvalues"].astype(np.float64)
    assert np.abs(ev - w).max() <= 1e-6 * lmax
    E = r["eigenvectors"].astype(np.float64)
    assert np.abs(E.T @ E - np.eye(D)).max() <= 4 * np.sqrt(D) * 2.0 ** -24 and np.linalg.det(E) > 0
    # separated eigenvectors within the angle bound 1e-6 lmax / gap; clustered ones by the largest principal angle
    # between the two subspaces
    for g in _clusters(w, 1e-5 * lmax):
        rest = [i for i in range(D) if i not in g]
        if not rest:
            continue
        gap = min(abs(w[i] - w[j]) for i in g for j in rest)
        bound = 1e-6 * lmax / gap
        if bound >= 0.1:
            continue
        Q = np.linalg.qr(E[:, g])[0]
        sin_max = np.linalg.norm(Q - V[:, g] @ (V[:, g].T @ Q), 2)
        assert sin_max <= bound + 4 * np.sqrt(D) * 2.0 ** -24, (g, sin_max, bound)


@pytest.mark.parametrize("D,ks", [(1, [1]), (6, [1, 3, 6]), (17, [1, 16, 17]), (130, [1, 129, 130])])
def test_project_reconstruct_bit_exact(cb, ctx, D, ks):
    rng = np.random.default_rng(D + 77)
    rows = _rows("offset_1e4", 3001, D, rng)
    rows[5, 0] = np.nan
    v = cb.Vectors(ctx, rows)
    r = cb.pca(ctx, v)
    for k in ks:
        proj = cb.pca_project(ctx, v, r["mean"], r["eigenvectors"], k)
        assert _same_f32(proj, pf.project(rows, r["mean"], r["eigenvectors"], k)), k
        q = cb.pca_project(ctx, v, r["mean"], r["eigenvectors"], k, to_device=True)
        assert q.n == 3001 and q.D == k
        rec = cb.pca_reconstruct(ctx, q, r["mean"], r["eigenvectors"])
        assert _same_f32(rec, pf.reconstruct(proj, r["mean"], r["eigenvectors"])), k
        rec_dev = cb.pca_reconstruct(ctx, q, r["mean"], r["eigenvectors"], to_device=True)
        assert rec_dev.D == D


def test_projected_device_set_feeds_kmeans(cb, ctx):
    rng = np.random.default_rng(8)
    rows = _rows("plain", 50000, 32, rng)
    v = cb.Vectors(ctx, rows)
    r = cb.pca(ctx, v)
    q_dev = cb.pca_project(ctx, v, r["mean"], r["eigenvectors"], 8, to_device=True)
    q_host = cb.pca_project(ctx, v, r["mean"], r["eigenvectors"], 8)
    c0 = q_host[rng.choice(50000, 16, replace=False)]
    a = cb.kmeans_cluster(ctx, q_dev, c0, max_iter=10, tol=0.0)
    b = cb.kmeans_cluster(ctx, cb.Vectors(ctx, q_host), c0, max_iter=10, tol=0.0)
    assert np.array_equal(a["labels"], b["labels"]) and _same_f32(a["centroids"], b["centroids"])
    assert np.array_equal(kf.assign(q_host, c0), cb.kmeans_assign(ctx, q_dev, c0)[0])


def test_argument_errors(cb, ctx):
    import ctypes as C

    rows = np.random.default_rng(1).standard_normal((100, 5)).astype(np.float32)
    v = cb.Vectors(ctx, rows)
    r = cb.pca(ctx, v)
    for k in (0, 6):
        with pytest.raises(cb.CbError):
            cb.pca_project(ctx, v, r["mean"], r["eigenvectors"], k)
    with pytest.raises(cb.CbError):  # 5-wide q into 4 dimensions
        cb.pca_reconstruct(ctx, v, r["mean"][:4], r["eigenvectors"][:4, :4])
    with pytest.raises(cb.CbError):
        cb.mean_cov(ctx, v, subset=[0, 100])
    mean, cov = np.empty(5, np.float32), np.empty((5, 5), np.float32)
    lib = cb.lib()
    assert lib.cb_vectors_mean_cov(ctx.h, None, None, C.c_size_t(0), C.c_size_t(2), cb._p(mean), cb._p(cov)) < 0
    assert lib.cb_vectors_mean_cov(ctx.h, v.h, None, C.c_size_t(0), C.c_size_t(2), None, cb._p(cov)) < 0
    assert lib.cb_vectors_project(ctx.h, v.h, cb._p(r["mean"]), cb._p(r["eigenvectors"]), C.c_int(2), None, None) < 0


def test_launch_counts_constant(cb, ctx):
    counts = set()
    sub_counts = set()
    rng = np.random.default_rng(2)
    for n, D in ((10, 2), (5000, 6), (70000, 40), (3000, 200)):
        v = cb.Vectors(ctx, rng.standard_normal((n, D)).astype(np.float32))
        l0 = ctx.kernel_launches()
        cb.mean_cov(ctx, v)
        counts.add(ctx.kernel_launches() - l0)
        l0 = ctx.kernel_launches()
        cb.mean_cov(ctx, v, subset=np.arange(n)[::-1])
        sub_counts.add(ctx.kernel_launches() - l0)
    assert counts == {3} and sub_counts == {4}, (counts, sub_counts)


def test_no_device_memory_growth(cb, ctx, pool_used):
    rows = np.random.default_rng(4).standard_normal((3000, 20)).astype(np.float32)

    def once():
        v = cb.Vectors(ctx, rows)
        r = cb.pca(ctx, v, subset=np.arange(0, 3000, 2))
        q = cb.pca_project(ctx, v, r["mean"], r["eigenvectors"], 5, to_device=True)
        cb.pca_reconstruct(ctx, q, r["mean"], r["eigenvectors"])
        with pytest.raises(cb.CbError):
            cb.pca_project(ctx, v, r["mean"], r["eigenvectors"], 0)
        q.close()
        v.close()

    once()
    before = pool_used()
    for _ in range(100):
        once()
    assert pool_used() <= before


def _slab_rows(n, D, sm_count):
    """The row-slab length of the covariance grid for n rows of dimension D (pca_features.cu, cov_launch)."""
    T = 8 if D <= 8 else 16 if D <= 16 else 32 if D <= 32 else 64
    rows = 2048 // T
    nt = (D + T - 1) // T
    npairs = nt * (nt + 1) // 2
    chunks = max(1, (n + rows - 1) // rows)
    want = max(1, (sm_count * 4 + npairs - 1) // npairs)
    s0 = min(chunks, want)
    return ((chunks + s0 - 1) // s0) * rows


@pytest.mark.parametrize("D", [6, 40, 65])
@pytest.mark.parametrize("residue", ["full", "one", "one_short"])
def test_mean_cov_slab_edges(cb, ctx, D, residue):
    """Sizes whose last row slab is full, holds one row, or lacks one row, derived from the grid's slab formula."""
    sm = ctx.device_info()["sm_count"]
    start = 300_000
    for n in range(start, start + 20_000):
        L = _slab_rows(n, D, sm)
        r = n % L
        if (residue == "full" and r == 0) or (residue == "one" and r == 1) or (residue == "one_short" and r == L - 1):
            break
    else:
        pytest.fail("no size found")
    assert _slab_rows(n, D, sm) < n  # several slabs
    rng = np.random.default_rng(n)
    _check(cb, ctx, _rows("offset_1e4", n, D, rng))
