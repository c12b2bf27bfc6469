"""The pinned rule of the robust normal estimation, on the host. tests/cpp/test_mcd_rule.cpp compiles
cilantro_b200/csrc/mcd_rule.hpp for the host and checks the per-point generator and draws against the installed
libstdc++ (std::minstd_rand0, std::uniform_int_distribution<size_t>), the selection order of the Mahalanobis keys, the
subset size and the 3x3 determinant and inverse against float64. No GPU involved."""
import os
import re

import cxx

ROOT, CSRC = cxx.ROOT, cxx.CSRC


def test_mcd_rule_matches_libstdcxx_and_float64(tmp_path):
    exe = cxx.build(os.path.join(ROOT, "tests", "cpp", "test_mcd_rule.cpp"), str(tmp_path / "test_mcd_rule"),
                    ["-O2", "-ffp-contract=off", "-Wall", "-I", CSRC], link=False)
    out = cxx.run(exe, timeout=600)
    assert "all mcd-rule checks passed" in out and "FAIL" not in out


def test_the_kernel_uses_the_shared_rule():
    """robust_normals.cu takes its draws, keys, subset size and 3x3 algebra from the header."""
    with open(os.path.join(CSRC, "robust_normals.cu")) as f:
        src = re.sub(r"//[^\n]*", "", f.read())
    for fn in ("mcd::point_seed(", "mcd::uniform_below(", "mcd::sort_key(", "mcd::subset_size(", "mcd::inverse(",
               "mcd::determinant(", "mcd::mahalanobis2(", "mcd::mean_cov("):
        assert fn in src, fn
