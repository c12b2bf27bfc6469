"""The C++ drop-in surface of plane RANSAC (include/cilantro/model_estimation/ransac_hyperplane_estimator.hpp) and the
PointCloud3f index subsets: they compile without Eigen, and on the GPU the shim gives what capi gives, estimateModel
is cb_pca's plane, the subsets follow the reference's set semantics, and the example runs."""
import os

import numpy as np
import pytest

import cxx
from cilantro_b200 import synth

ROOT = cxx.ROOT
SHIM = os.path.join(ROOT, "tests", "cpp", "test_ransac_plane_shim.cpp")
EXAMPLE = os.path.join(ROOT, "examples", "ransac_plane_cloud.cpp")


def test_shim_and_example_compile_without_eigen():
    for path in (SHIM, EXAMPLE):
        r = cxx.syntax(path)
        assert r.returncode == 0, r.stderr


def ref_subset(n, idx, negate):
    """utilities/point_cloud.hpp:32-45: a std::set of the indices (or of their complement)."""
    s = set(idx)
    return sorted(set(range(n)) - s) if negate else sorted(s)


def ref_remove(n, idx):
    """utilities/point_cloud.hpp:154-199 on a list of original positions."""
    order = list(range(n))
    drop = sorted(set(idx))
    if len(drop) >= n:
        return []
    valid = n - 1
    while valid in drop:
        valid -= 1
    for i in drop:
        if i >= valid:
            break
        order[i], order[valid] = order[valid], order[i]
        valid -= 1
        while i < valid and valid in drop:
            valid -= 1
    return order[:valid + 1]


@pytest.mark.gpu
def test_shim_matches_capi(cb, ctx, tmp_path):
    pts = synth.plane_scene(30000, seed=4)["points"]
    pts.tofile(tmp_path / "pts.bin")
    out = cxx.run(cxx.build(SHIM, str(tmp_path / "shim")), tmp_path / "pts.bin", 6)
    rows = {ln.split()[0]: ln.split()[1:] for ln in out.splitlines() if ln.strip()}
    cloud = cb.Cloud(ctx, pts)
    got = cb.ransac_plane(ctx, cloud, 6, max_iter=250, thresh=0.01, inlier_count_thresh=int(0.15 * 30000),
                          re_estimate=False)
    assert int(rows["iterations"][0]) == got["iterations"] and int(rows["inliers"][0]) == got["num_inliers"]
    assert np.array_equal(np.array(rows["plane"], np.uint32), got["plane"].view(np.uint32))
    assert np.array_equal(np.array(rows["inlier_list"][1:], np.int64), got["inliers"])
    assert int(rows["recount"][0]) == got["num_inliers"]
    assert int(rows["cut"][0]) == 30000 - got["num_inliers"]
    for key, sel in (("model_all", np.arange(30000)), ("model_subset", np.array([0, 5, 9, 13, 21, 40]))):
        p = cb.pca(ctx, cb.Cloud(ctx, pts[sel]))
        nrm = p["eigenvectors"][:, 2]
        m = p["mean"]
        want = np.array([nrm[0], nrm[1], nrm[2], -(nrm[0] * m[0] + (nrm[1] * m[1] + nrm[2] * m[2]))], np.float32)
        assert np.array_equal(np.array(rows[key], np.uint32), want.view(np.uint32)), key
    x = lambda key: np.array(rows[key][1:], np.float64).reshape(-1, 3)  # noqa: E731
    idx = [5, 1, 5, 3]
    assert np.array_equal(x("subset")[:, 0], ref_subset(8, idx, False))
    assert np.array_equal(x("subset_normals")[:, 1], ref_subset(8, idx, False))
    assert np.array_equal(x("negate")[:, 0], ref_subset(8, idx, True))
    assert np.array_equal(x("remove")[:, 0], ref_remove(8, [1, 6, 1, 3]))
    assert np.array_equal(x("remove_normals")[:, 1], ref_remove(8, [1, 6, 1, 3]))


@pytest.mark.gpu
def test_example_runs(cb, tmp_path):
    out = cxx.run(cxx.build(EXAMPLE, str(tmp_path / "ransac_plane_cloud")), cwd=str(tmp_path))
    assert "RANSAC iterations:" in out and "left" in out
    line = [ln for ln in out.splitlines() if ln.startswith("plane:")][0]
    assert abs(abs(float(line.split()[3])) - 1.0) < 1e-3  # the floor, z = 0
