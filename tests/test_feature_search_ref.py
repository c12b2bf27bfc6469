"""The scalable feature 1-NN restatement (tests/feature_search_ref.py) against the brute-force oracle
(feature_icp.knn1): the same index and the same value bits for every query, for every feature kind, on exact ties and
duplicates, a radius hit exactly, non-finite xyz and tails, and tails whose squares underflow or overflow. The GPU
tests of the feature search (test_gpu_feature_icp_edges.py) take their expected answers from this restatement."""
import numpy as np
import pytest

import feature_search_ref as fsr
from cilantro_b200 import synth

FLT_MAX = float(np.finfo(np.float32).max)
KINDS = ["point_normal", "point_color", "point_normal_color"]
T1 = np.array([[0.9998, -0.0175, 0.0, 0.025], [0.0175, 0.9998, 0.0, -0.015], [0.0, 0.0, 1.0, 0.0005]], np.float32)
I34 = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)


@pytest.fixture(scope="module")
def F(orc):
    from oracle import feature_icp

    return feature_icp


def _sheet(n, seed):
    s = synth.textured_sheet_pair(n, seed=seed)
    s["T"] = T1
    return s


def _lattice(n, seed):
    s = fsr.lattice_scene(n, n, seed)
    s["T"] = I34
    return s


def _nonfinite(n, seed):
    s = _sheet(n, seed)
    rng = np.random.default_rng(seed)
    for key in ("dst", "src", "dst_colors", "src_colors", "dst_normals", "src_normals"):
        rows = rng.choice(n, 40, replace=False)
        s[key][rows[:15], rng.integers(0, 3)] = np.nan
        s[key][rows[15:30], rng.integers(0, 3)] = np.inf
        s[key][rows[30:], rng.integers(0, 3)] = -np.inf
    return s


def _far_colours(n, seed):
    s = _sheet(n, seed)
    s["src_colors"][:20] = 4.0  # no destination colour near: with w_c = 1e20 every distance of these queries is +inf
    return s


SCENES = {  # name: (scene, w_n, w_c)
    "sheet": (_sheet, 0.5, 5.0),
    "lattice_ties": (_lattice, 0.5, 1.0),
    "non_finite": (_nonfinite, 0.5, 5.0),
    "tails_underflow": (_sheet, 2.0 ** -70, 2.0 ** -70),  # tail squares subnormal or zero
    "tails_overflow": (_far_colours, 1.0, 1e20),               # colour squares +inf unless the colours nearly agree
}


def _features(F, kind, s, w_n, w_c):
    nrm, col = "normal" in kind, "color" in kind
    dt = F.tails(kind, s["dst_normals"] if nrm else None, s["dst_colors"] if col else None, w_n, w_c)
    st = F.tails(kind, s["src_normals"] if nrm else None, s["src_colors"] if col else None, w_n, w_c)
    return np.hstack([s["dst"], dt]), F.features(kind, s["T"], s["src"], st)


def _ties(ref, qry, best):
    """per query, the number of reference points whose fp32 distance equals best"""
    return np.concatenate([(fsr.feature_d2(qry[i:i + 256, None, :], ref[None, :, :]) == best[i:i + 256, None]).sum(1)
                           for i in range(0, qry.shape[0], 256)])


def _same(got, want):
    assert np.array_equal(got[0], want[0]), int((got[0] != want[0]).sum())
    assert np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32)), int((got[1] != want[1]).sum())


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("scene", list(SCENES))
def test_restatement_matches_brute_force(F, kind, scene):
    make, w_n, w_c = SCENES[scene]
    s = make(3000, seed=len(scene))
    ref, qry = _features(F, kind, s, w_n, w_c)
    want = F.knn1(ref, qry, FLT_MAX)
    _same(fsr.knn1(ref, qry, FLT_MAX), want)
    hit = want[0] >= 0
    assert hit.mean() > 0.5, hit.mean()
    # a radius equal to an attained distance: the queries at exactly that distance find nothing (strict d2 < max_d2)
    r = np.sort(want[1][hit])[hit.sum() // 2]
    at = want[1] == r
    assert at.any()
    bounded = F.knn1(ref, qry, r)
    assert (bounded[0][at] == -1).all() and (bounded[0][want[1] < r] >= 0).all()
    _same(fsr.knn1(ref, qry, r), bounded)
    # and just above it
    r_up = np.nextafter(r, np.float32(np.inf))
    _same(fsr.knn1(ref, qry, r_up), F.knn1(ref, qry, r_up))
    if scene == "lattice_ties":
        # the scene does what it is for: most answers are an exact tie between several points
        ties = _ties(ref, qry, want[1])
        assert (ties[hit] > 1).mean() > 0.4, (ties[hit] > 1).mean()
    if scene == "tails_overflow" and "color" in kind:
        assert (~hit[:20]).all() and hit[20:].all()
    if scene == "non_finite":
        bad_q = ~np.isfinite(qry).all(1)
        bad_r = np.flatnonzero(~np.isfinite(ref).all(1))
        assert bad_q.any() and bad_r.size and (want[0][bad_q] == -1).all() and not np.isin(want[0], bad_r).any()


@pytest.mark.parametrize("kind", KINDS)
def test_restatement_matches_nanoflann_where_the_nearest_is_unique(F, kind):
    """Where oracle/_ref exists: the reference's own kd-tree search agrees on every query whose fp32 nearest distance is
    attained by one point only (on ties nanoflann's answer depends on its traversal order)."""
    if not F.have_ref():
        pytest.skip("oracle/_ref (the reference's nanoflann) is not built")
    s = _sheet(3000, seed=7)
    ref, qry = _features(F, kind, s, 0.5, 5.0)
    got = fsr.knn1(ref, qry, FLT_MAX)
    unique = _ties(ref, qry, got[1]) == 1
    assert unique.mean() > 0.9
    nf = F.ref_knn1(ref, qry, FLT_MAX)
    assert np.array_equal(nf[0][unique], got[0][unique])
    assert np.array_equal(nf[1][unique].view(np.uint32), got[1][unique].view(np.uint32))
