"""The hypothesis loop shared by the rigid and plane RANSAC estimators, on the host. tests/cpp/test_ransac_loop.cpp
compiles cilantro_b200/csrc/ransac_loop.hpp with g++ and checks it, under four batch schedules, against a direct
restatement of RandomSampleConsensusBase::estimate (ransac_base.hpp:64-114). No GPU involved."""
import os
import re

import cxx

ROOT, CSRC = cxx.ROOT, cxx.CSRC


def test_ransac_loop_matches_the_sequential_loop(tmp_path):
    exe = cxx.build(os.path.join(ROOT, "tests", "cpp", "test_ransac_loop.cpp"), str(tmp_path / "test_ransac_loop"),
                    ["-O2", "-Wall", "-I", CSRC], link=False)
    out = cxx.run(exe, timeout=600)
    assert "all ransac-loop checks passed" in out and "FAIL" not in out


def test_the_estimators_use_the_shared_loop_and_compaction():
    """ransac.cu and ransac_plane.cu run the loop of ransac_loop.hpp and list their inliers through ransac_inliers;
    neither draws samples, keeps a best count or tests the target itself."""
    for name in ("ransac.cu", "ransac_plane.cu"):
        with open(os.path.join(CSRC, name)) as f:
            src = re.sub(r"//[^\n]*", "", f.read())
        assert "ransac_loop(" in src and "ransac_inliers(" in src, name
        assert "sampler.next(" not in src and "std::mt19937" not in src, name
        assert not re.search(r"best_count\s*=|best_it\b|>=\s*inlier_count_thresh", src), name
        if name == "ransac_plane.cu":
            assert "exclusive_scan_u32" not in src and "inlier_scatter_kernel" not in src
