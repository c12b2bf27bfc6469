"""Classical multidimensional scaling on the device (cb_vectors_mds) against the float64 restatement of mds_ref.py
(numpy.linalg.eigh of the explicitly formed B): the accuracy bounds of DESIGN §4.19 at the block, strip, chunk and
means-slab edges and at n = 32 768, the clamp and order rules on non-Euclidean and non-symmetric input, offsets and
scales, the non-finite and argument rules, bit identities, device output into k-means and PCA, and no memory growth."""
import numpy as np
import pytest

import mds_ref as mr
from test_gpu_device_memory import pool_used  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _points(n, rng, dims=(3.0, 2.0, 1.0, 0.5, 0.25)):
    """n points in len(dims) dimensions with distinct spreads: B has a gap after every eigenvalue."""
    return (rng.standard_normal((n, len(dims))) * np.asarray(dims)).astype(np.float32)


def _check_eigenvalues(ev, ref):
    """|lambda - lambda_ref| <= 1e-6 |lambda_ref| + 1e-9 |lambda_1|, lambda_1 the largest magnitude of the spectrum."""
    lam1 = np.max(np.abs(ref["all_eigenvalues"]))
    want = ref["eigenvalues"]
    err = np.abs(ev.astype(np.float64) - want)
    assert np.all(err <= 1e-6 * np.abs(want) + 1e-9 * lam1), (ev, want)


def _check_embedding(emb, ref, tol=1e-5):
    """The Gram matrix X X^T and the pairwise distances of the embedding against the restatement's, Frobenius-relative."""
    x = np.asarray(emb, np.float64)
    y = ref["embedding"]
    assert x.shape == y.shape
    gx, gy = x @ x.T, y @ y.T
    scale = max(np.linalg.norm(gy), 1e-300)
    assert np.linalg.norm(gx - gy) <= tol * scale + 1e-30, np.linalg.norm(gx - gy) / scale
    dx = np.sqrt(np.maximum(np.diag(gx)[:, None] + np.diag(gx)[None, :] - 2 * gx, 0))
    dy = np.sqrt(np.maximum(np.diag(gy)[:, None] + np.diag(gy)[None, :] - 2 * gy, 0))
    assert np.max(np.abs(dx - dy)) <= np.sqrt(tol) * max(dy.max(), 1e-300)


def _run(cb, ctx, dm, max_dim, estimate_dim=False, squared=True):
    r = cb.mds(ctx, dm, max_dim, estimate_dim=estimate_dim, squared=squared)
    ref = mr.mds(dm, max_dim, estimate_dim=estimate_dim, squared=squared)
    assert r["ok"]
    assert r["dim"] == ref["dim"]
    _check_eigenvalues(r["eigenvalues"], ref)
    return r, ref


@pytest.mark.parametrize("max_dim,estimate", [(2, False), (3, False), (2, True), (3, True)])
def test_ring(cb, ctx, max_dim, estimate):
    """The reference example's wavy ring: lambda_1 = lambda_2, so only the Gram matrix and distances are compared."""
    _, dm = mr.ring(1000)
    r, ref = _run(cb, ctx, dm, max_dim, estimate)
    _check_embedding(r["embedding"], ref)


# block (8 / 16 columns; the whole space up to 2 b rows), chunk (32), strip (256) and means (64 rows, 1024 columns)
# edges, each +-1
SIZES = [3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 255, 256, 257, 511, 513, 1000, 1023, 1024, 1025]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("max_dim", [1, 2, 3])
def test_sizes(cb, ctx, n, max_dim):
    if max_dim > n - 1:
        pytest.skip("nev > n - 1")
    rng = np.random.default_rng(n * 10 + max_dim)
    p = _points(n, rng)
    squared = (n + max_dim) % 2 == 0
    dm = mr.points_distances(p, squared=squared)
    r, ref = _run(cb, ctx, dm, max_dim, False, squared)
    if n > 8:  # the spectrum has a gap after every kept eigenvalue: columns are compared with the pinned signs
        assert np.allclose(r["embedding"], ref["embedding"], rtol=0,
                           atol=1e-4 * np.abs(ref["embedding"]).max())
    _check_embedding(r["embedding"], ref)


@pytest.mark.parametrize("n", [4, 17, 300])
def test_estimate_dim(cb, ctx, n):
    rng = np.random.default_rng(n)
    p = _points(n, rng, dims=(5.0, 4.0, 0.01, 0.005, 0.001))
    dm = mr.points_distances(p)
    for max_dim in (1, 2, 3):
        if max_dim > n - 1:
            continue
        r, ref = _run(cb, ctx, dm, max_dim, True)
        _check_embedding(r["embedding"], ref)


@pytest.mark.parametrize("n", [700, 3000])
def test_clustered_spectrum_restarts(cb, ctx, n):
    """16-D points with spreads 1.00, 0.98, ..., 0.70: eigenvalue gaps of a few percent need several restarts."""
    rng = np.random.default_rng(n)
    p = _points(n, rng, dims=tuple(1.0 - 0.02 * k for k in range(16)))
    dm = mr.points_distances(p)
    for max_dim in (3, 10):
        r, ref = _run(cb, ctx, dm, max_dim)
        _check_embedding(r["embedding"], ref)


def test_non_euclidean_negative_eigenvalues(cb, ctx):
    """Pseudo-Euclidean distances |x_i - x_j|^2 - 3 |y_i - y_j|^2: the largest-magnitude eigenvalue of B is negative,
    takes the first slot and gives a zero embedding column."""
    rng = np.random.default_rng(7)
    x = rng.standard_normal((200, 3)) * np.array([3.0, 2.0, 1.0])
    y = rng.standard_normal((200, 1)) * 2.0
    dm = (mr.points_distances(x) - 3 * mr.points_distances(y)).astype(np.float32)
    ref = mr.mds(dm, 3)
    assert ref["eigenvalues"][0] == 0.0, "the case needs a clamped leading eigenvalue"
    r, ref = _run(cb, ctx, dm, 3)
    _check_embedding(r["embedding"], ref)
    zero = ref["eigenvalues"] == 0.0
    assert np.all(r["eigenvalues"][zero] == 0.0)
    assert np.all(r["embedding"][:, zero] == 0.0)


def test_non_symmetric_lower_triangle(cb, ctx):
    """A non-symmetric matrix gives the lower-triangle restatement's result."""
    rng = np.random.default_rng(8)
    p = _points(300, rng)
    dm = mr.points_distances(p) + rng.uniform(0, 0.5, (300, 300)).astype(np.float32)
    r, ref = _run(cb, ctx, dm, 3)
    _check_embedding(r["embedding"], ref, tol=1e-4)


@pytest.mark.parametrize("scale", [1e-20, 1e-10, 1.0, 1e10, 1e18])
def test_scales(cb, ctx, scale):
    rng = np.random.default_rng(9)
    dm = (mr.points_distances(_points(400, rng)) * np.float32(scale)).astype(np.float32)
    r, ref = _run(cb, ctx, dm, 3)
    _check_embedding(r["embedding"], ref)


@pytest.mark.parametrize("offset", [1e2, 1e4])
def test_far_offsets(cb, ctx, offset):
    """A constant added to every entry cancels in B; the entries keep their fp32 rounding."""
    rng = np.random.default_rng(10)
    dm = (mr.points_distances(_points(400, rng)) + np.float32(offset)).astype(np.float32)
    r, ref = _run(cb, ctx, dm, 3)
    _check_embedding(r["embedding"], ref, tol=1e-4)


def test_large(cb, ctx):
    """n = 32 768 built on the device: squared Euclidean distances of 5-D points, so the eigenvalues are those of the
    centred points' 5 x 5 scatter matrix (float64), up to the fp32 rounding of the entries."""
    import torch

    n = 32768
    g = torch.Generator(device="cuda").manual_seed(11)
    p = torch.randn(n, 5, device="cuda", generator=g, dtype=torch.float64) * torch.tensor(
        [3.0, 2.0, 1.0, 0.5, 0.25], device="cuda", dtype=torch.float64)
    dm = torch.cdist(p, p).pow(2).to(torch.float32).contiguous()
    torch.cuda.synchronize()  # the library copies on its own stream
    v = cb.Vectors(ctx, device_ptr=dm.data_ptr(), n=n, D=n)
    r = cb.mds(ctx, v, 3)
    assert r["ok"]
    pc = (p - p.mean(dim=0)).cpu().numpy()
    want = np.sort(np.linalg.eigvalsh(pc.T @ pc))[::-1][:3]
    assert np.allclose(r["eigenvalues"], want, rtol=1e-4), (r["eigenvalues"], want)
    # embedded distances of sampled pairs against the distances of the points projected on the top 3 directions
    w, E = np.linalg.eigh(pc.T @ pc)
    proj = pc @ E[:, ::-1][:, :3]
    idx = np.random.default_rng(0).integers(0, n, (4000, 2))
    de = np.linalg.norm(r["embedding"][idx[:, 0]] - r["embedding"][idx[:, 1]], axis=1)
    dp = np.linalg.norm(proj[idx[:, 0]] - proj[idx[:, 1]], axis=1)
    assert np.max(np.abs(de - dp)) <= 1e-3 * dp.max()
    v.close()


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
@pytest.mark.parametrize("squared", [True, False])
def test_non_finite(cb, ctx, bad, squared):
    rng = np.random.default_rng(12)
    dm = mr.points_distances(_points(50, rng), squared=squared)
    dm[31, 7] = bad
    r = cb.mds(ctx, dm, 2, squared=squared)
    assert not r["ok"]
    assert r["dim"] == 2 and np.all(np.isnan(r["eigenvalues"])) and np.all(np.isnan(r["embedding"]))


def test_unsquared_overflow_is_non_finite(cb, ctx):
    """An entry whose fp32 square overflows counts as non-finite."""
    dm = np.ones((10, 10), np.float32)
    dm[3, 4] = 3e20
    r = cb.mds(ctx, dm, 2, squared=False)
    assert not r["ok"]


def test_argument_errors(cb, ctx):
    dm = mr.points_distances(_points(6, np.random.default_rng(13)))
    for max_dim, est in ((0, False), (6, False), (7, False), (6, True)):
        with pytest.raises(cb.CbError):
            cb.mds(ctx, dm, max_dim, estimate_dim=est)
    v = cb.Vectors(ctx, np.zeros((6, 5), np.float32))
    with pytest.raises(cb.CbError):
        cb.mds(ctx, v, 2)
    v.close()
    assert cb.mds(ctx, dm, 5)["ok"]  # nev = n - 1 is allowed
    assert cb.mds(ctx, dm, 5, estimate_dim=True)["ok"]


def test_bit_identities_and_device_output(cb, ctx):
    _, dm = mr.ring(1000)
    a = cb.mds(ctx, dm, 3)
    b = cb.mds(ctx, dm, 3)
    assert np.array_equal(_bits(a["eigenvalues"]), _bits(b["eigenvalues"]))
    assert np.array_equal(_bits(a["embedding"]), _bits(b["embedding"]))
    d = cb.mds(ctx, dm, 3, to_device=True)
    assert np.array_equal(_bits(a["eigenvalues"]), _bits(d["eigenvalues"]))
    out = d["embedding"]
    assert (out.n, out.D) == (1000, 3)
    host = cb.Vectors(ctx, a["embedding"])
    pd, ph = cb.pca(ctx, out), cb.pca(ctx, host)  # the device set holds the host embedding's bytes
    assert pd["ok"] and all(np.array_equal(_bits(pd[k]), _bits(ph[k])) for k in ("mean", "cov", "eigenvalues"))
    cent = a["embedding"][::250].copy()
    k1 = cb.kmeans_cluster(ctx, out, cent, max_iter=20)
    k2 = cb.kmeans_cluster(ctx, host, cent, max_iter=20)
    assert np.array_equal(k1["labels"], k2["labels"]) and np.array_equal(_bits(k1["centroids"]), _bits(k2["centroids"]))
    out.close()
    host.close()


def test_launch_counts_repeat(cb, ctx):
    """The launch count of a call is a function of its restart count: the same input gives the same count."""
    dm = mr.points_distances(_points(700, np.random.default_rng(15)))
    counts = set()
    for _ in range(3):
        l0 = ctx.kernel_launches()
        cb.mds(ctx, dm, 2)
        counts.add(ctx.kernel_launches() - l0)
    assert len(counts) == 1


def test_no_device_memory_growth(cb, ctx, pool_used):
    dm = mr.points_distances(_points(300, np.random.default_rng(14)))

    def once():
        r = cb.mds(ctx, dm, 3, to_device=True)
        r["embedding"].close()
        with pytest.raises(cb.CbError):
            cb.mds(ctx, dm, 0)

    once()
    before = pool_used()
    for _ in range(20):
        once()
    assert pool_used() <= before
