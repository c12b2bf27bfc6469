"""The robust-normal oracle (oracle/robust_normals_oracle.cpp) on the host, no GPU:
  * against an independent float64 restatement in numpy of MinimumCovarianceDeterminant::operator()
    (core/covariance.hpp:185-371) under the draws of DESIGN §4.15: the same kept subsets and covariances within fp32
    rounding;
  * with inlier_ratio = 1 (h == size), the bits of the plain normal-estimation oracle;
  * the reference example's point: on a noisy plane with 20 % planted off-plane outliers (k = 24, default trials), the
    median robust normal of the inliers is within 1 degree of the true normal while the plain one is tilted by more
    than 4, and the chi-square test (6.25) flags more than 95 % of the outliers and fewer than 10 % of the inliers.
"""
import numpy as np
import pytest

import oracle
from oracle import robust_normals as orn

M = 2147483647


def _fmix32(x):
    x ^= x >> 16
    x = (x * 0x85EBCA6B) & 0xFFFFFFFF
    x ^= x >> 13
    x = (x * 0xC2B2AE35) & 0xFFFFFFFF
    x ^= x >> 16
    return x


class _Minstd:
    """std::minstd_rand0 and libstdc++'s uniform_int_distribution<size_t> downscale on it, from their definitions."""

    def __init__(self, seed):
        self.x = seed % M or 1

    def below(self, n):
        scaling = (M - 2) // n  # engine range max - min = (M - 1) - 1
        past = n * scaling
        while True:
            self.x = self.x * 16807 % M
            r = self.x - 1
            if r < past:
                return r // scaling


def _inv(a):
    """Inverse by the adjugate: a singular matrix gives Inf / NaN entries, as the fp32 rule does, instead of raising."""
    adj = np.array([[np.linalg.det(np.delete(np.delete(a, i, 0), j, 1)) * (-1) ** (i + j) for i in range(3)]
                    for j in range(3)])
    with np.errstate(all="ignore"):
        return adj / np.linalg.det(a)


def _mcd64(p, i, trials, refinements, ratio, min_size, seed):
    """One neighbourhood p (m x 3, search order) of point i: (kept indices of the winner, mean, cov) in float64."""
    m = p.shape[0]
    h = min(max(min_size, int(np.floor(np.float32(ratio) * np.float32(m) + np.float32(0.5)))), m)
    if m <= min_size or h == m:
        return np.arange(m), p.mean(0), np.cov(p.T)
    rng = _Minstd(_fmix32(seed ^ _fmix32((i + 0x9E3779B9) & 0xFFFFFFFF)))
    best = (np.finfo(np.float32).max, None, None, None)
    for _ in range(trials):
        kept = np.array([rng.below(m) for _ in range(min_size)])
        mean, cov = p[kept].mean(0), np.cov(p[kept].T)
        for _ in range(refinements):
            with np.errstate(all="ignore"):
                d = p - mean
                q = np.einsum("ij,jk,ik->i", d, _inv(cov), d)
            q = np.where(np.isnan(q), np.inf, q)
            kept = np.lexsort((np.arange(m), q))[:h]
            mean, cov = p[kept].mean(0), np.cov(p[kept].T)
        det = np.linalg.det(cov)
        if np.isfinite(det) and det < best[0]:
            best = (det, kept, mean, cov)
    return best[1], best[2], best[3]


# Three points span a plane, so the first refinement of a 3-point sample ranks by the inverse of a singular matrix:
# round-off decides, in fp32 and float64 differently. The refined cases therefore draw larger samples.
@pytest.mark.parametrize("k,trials,refinements,ratio,min_size", [(12, 6, 3, 0.75, 6), (12, 2, 1, 0.75, 6),
                                                                 (8, 1, 0, 0.5, 3), (33, 6, 3, 0.5, 8),
                                                                 (128, 2, 2, 0.75, 8)])
def test_oracle_matches_float64_restatement(k, trials, refinements, ratio, min_size):
    rng = np.random.default_rng(k + trials)
    pts = rng.random((600, 3)).astype(np.float32)
    pts[:, 2] *= 0.05  # a thick slab: well-conditioned covariances with one short axis
    seed = 17
    got = orn.estimate_normals_mcd(pts, k=k, num_trials=trials, num_refinements=refinements, inlier_ratio=ratio,
                                   min_sample_size=min_size, seed=seed)
    assert (got["status"] == 0).all()
    same, total = 0, 0
    for i in range(pts.shape[0]):
        nb = got["nbr"][i, :got["cnt"][i]]
        kept, _, cov = _mcd64(pts[nb].astype(np.float64), i, trials, refinements, ratio, min_size, seed)
        h = int(got["h"][i])
        mine = got["kept"][i, :len(kept)] if refinements == 0 or h == len(nb) else got["kept"][i, :h]
        total += 1
        if set(mine.tolist()) == set(nb[kept].tolist()):
            same += 1
            c6 = got["cov6"][i].astype(np.float64)
            ref6 = cov[[0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
            assert np.all(np.abs(c6 - ref6) <= 1e-4 * max(np.abs(ref6).max(), 1e-10)), (i, c6, ref6)
    # near-equal determinants or keys (a sample of few distinct points is nearly singular) may order differently in
    # float64 than in the pinned fp32
    assert same >= 0.95 * total, (same, total)


@pytest.mark.parametrize("k", [3, 12, 64])
def test_whole_neighbourhood_is_the_plain_oracle_bit_for_bit(k):
    rng = np.random.default_rng(k)
    pts = rng.random((3000, 3), dtype=np.float32)
    vp = [0.5, 0.5, 4.0]
    got = orn.estimate_normals_mcd(pts, k=k, inlier_ratio=1.0, view_point=vp)
    n, curv, cov6, _ = oracle.estimate_normals(pts, oracle.BruteKnn(pts), k=k, view_point=vp)
    for a, b in ((got["normals"], n), (got["curvature"], curv), (got["cov6"], cov6)):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_robust_normals_resist_planted_outliers():
    rng = np.random.default_rng(21)
    n = 20000
    pts = np.zeros((n, 3), np.float32)
    pts[:, :2] = rng.random((n, 2))
    pts[:, 2] = 0.0003 * rng.standard_normal(n)
    out = rng.random(n) < 0.2
    pts[out, 2] = rng.uniform(0.005, 0.015, out.sum()) * rng.choice([-1, 1], out.sum())
    plain = oracle.estimate_normals(pts, oracle.BruteKnn(pts), k=24)[0]
    rob = orn.estimate_normals_mcd(pts, k=24, chi_square_threshold=6.25, seed=3)  # 6 trials, 3 refinements

    def tilt(nn):
        return np.degrees(np.arccos(np.clip(np.abs(nn[:, 2].astype(np.float64)), 0, 1)))

    inl = ~out & (rob["status"] == 0)
    t_rob, t_plain = tilt(rob["normals"][inl]), tilt(plain[inl])
    print(f"median tilt: robust {np.median(t_rob):.2f} deg, plain {np.median(t_plain):.2f} deg; outliers flagged "
          f"{(rob['status'][out] == 2).mean():.3f}, inliers flagged {(rob['status'][~out] == 2).mean():.3f}")
    assert np.median(t_rob) < 1.0 and np.median(t_plain) > 4.0
    assert (rob["status"][out] == 2).mean() > 0.95
    assert (rob["status"][~out] == 2).mean() < 0.1
