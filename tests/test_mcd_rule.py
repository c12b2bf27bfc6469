"""The pinned rule of the robust normal estimation, on the host. tests/cpp/test_mcd_rule.cpp compiles
cilantro_b200/csrc/mcd_rule.hpp for the host and checks the per-point generator and draws against the installed
libstdc++ (std::minstd_rand0, std::uniform_int_distribution<size_t>), the selection order of the Mahalanobis keys, the
subset size and the 3x3 determinant and inverse against float64. No GPU involved."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cilantro_b200", "csrc")


def test_mcd_rule_matches_libstdcxx_and_float64(tmp_path):
    exe = str(tmp_path / "test_mcd_rule")
    env = dict(os.environ)
    env.pop("CXX", None)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-I", CSRC,
                           os.path.join(ROOT, "tests", "cpp", "test_mcd_rule.cpp"), "-o", exe], env=env)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "all mcd-rule checks passed" in out.stdout and "FAIL" not in out.stdout


def test_the_kernel_uses_the_shared_rule():
    """robust_normals.cu takes its draws, keys, subset size and 3x3 algebra from the header."""
    with open(os.path.join(CSRC, "robust_normals.cu")) as f:
        src = re.sub(r"//[^\n]*", "", f.read())
    for fn in ("mcd::point_seed(", "mcd::uniform_below(", "mcd::sort_key(", "mcd::subset_size(", "mcd::inverse(",
               "mcd::determinant(", "mcd::mahalanobis2(", "mcd::mean_cov("):
        assert fn in src, fn
