"""The feature-ICP oracle (oracle/feature_icp_oracle.cpp) pinned on the CPU: its 1-NN lists on D = 6 / 9 feature vectors
equal those of the reference's own nanoflann kd-tree built over the same features (the same index, or an alternative at a
bit-equal d2; d2 bit for bit), with a finite radius and unbounded, and agree with a float64 brute force."""
import numpy as np
import pytest

from cilantro_b200 import synth

FLT_MAX = float(np.finfo(np.float32).max)
KINDS = ["point_normal", "point_color", "point_normal_color"]


@pytest.fixture(scope="module")
def F(orc):
    from oracle import feature_icp

    feature_icp.build()
    return feature_icp


def _features(F, kind, n, seed):
    s = synth.textured_sheet_pair(n, seed=seed)
    rng = np.random.default_rng(seed)
    # a few exact duplicates (ties) and far outliers
    s["dst"][:20] = s["dst"][20:40]
    s["dst_colors"][:20] = s["dst_colors"][20:40]
    s["dst_normals"][:20] = s["dst_normals"][20:40]
    s["src"][-5:] = rng.normal(0, 30, (5, 3)).astype(np.float32)
    nrm, col = "normal" in kind, "color" in kind
    dt = F.tails(kind, s["dst_normals"] if nrm else None, s["dst_colors"] if col else None, 0.5, 5.0)
    st = F.tails(kind, s["src_normals"] if nrm else None, s["src_colors"] if col else None, 0.5, 5.0)
    T = synth.rigid_from_axis_angle([0.2, -0.3, 1.0], 0.02, [0.02, -0.01, 0.001]).astype(np.float32)
    return F.features(kind, np.hstack([np.eye(3), np.zeros((3, 1))]), s["dst"], dt), F.features(kind, T, s["src"], st)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("max_d2", [0.02, FLT_MAX])
def test_brute_force_equals_reference_nanoflann(F, kind, max_d2):
    if not F.have_ref():
        pytest.skip("oracle/_ref was not built (no reference checkout)")
    ref, qry = _features(F, kind, 4000, seed=7)
    i0, d0 = F.knn1(ref, qry, max_d2)
    i1, d1 = F.ref_knn1(ref, qry, max_d2)
    assert np.array_equal(d0.view(np.uint32), d1.view(np.uint32))
    same = i0 == i1
    # an alternative index is only acceptable at a bit-equal distance
    alt = ~same
    assert np.all(i0[alt] >= 0) and np.all(i1[alt] >= 0)
    assert np.array_equal(F.knn1(ref[i1[alt]], qry[alt], FLT_MAX)[1].view(np.uint32), d0[alt].view(np.uint32)) or \
        not alt.any()
    assert (i0 >= 0).sum() > 0.9 * len(i0) if max_d2 == FLT_MAX else (i0 >= 0).sum() > 0


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("max_d2", [0.02, FLT_MAX])
def test_brute_force_agrees_with_float64(F, kind, max_d2):
    ref, qry = _features(F, kind, 2000, seed=3)
    idx, d2 = F.knn1(ref, qry, max_d2)
    r64, q64 = ref.astype(np.float64), qry.astype(np.float64)
    full = ((q64[:, None, :] - r64[None, :, :]) ** 2).sum(-1)
    best = full.min(1)
    found = idx >= 0
    # the fp32 distance is the float64 one up to a few roundings per term
    assert np.allclose(d2[found], full[np.arange(len(idx))[found], idx[found]], rtol=1e-5, atol=1e-30)
    # the chosen point is the nearest up to that rounding, and nothing missed lies clearly inside the radius
    assert np.all(full[np.arange(len(idx))[found], idx[found]] <= best[found] * (1 + 2e-5) + 1e-30)
    assert np.all(best[~found] >= max_d2 * (1 - 2e-5))
