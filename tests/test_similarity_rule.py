"""The angle test of the connected-component extraction, on the host. cilantro_b200/csrc/similarity_rule.hpp derives
from an angle threshold the dot-product intervals the device compares against; tests/cpp/test_similarity_rule.cpp
compiles that header for the host and checks, over every float in [-1, 1], that the intervals give the verdict of
std::acos (and that acosf is monotone there, which the derivation relies on). No GPU involved."""
import os
import re

import cxx

ROOT, CSRC = cxx.ROOT, cxx.CSRC


def test_angle_intervals_match_acos_on_every_float(tmp_path):
    exe = cxx.build(os.path.join(ROOT, "tests", "cpp", "test_similarity_rule.cpp"),
                    str(tmp_path / "test_similarity_rule"),
                    ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-Wall", "-pthread", "-I", CSRC], link=False)
    out = cxx.run(exe, timeout=1200)
    assert "all similarity-rule checks passed" in out and "FAIL" not in out


def test_the_kernel_uses_the_shared_rule():
    """segment.cu derives the intervals with the header's function and never evaluates acos on the device."""
    with open(os.path.join(CSRC, "segment.cu")) as f:
        src = re.sub(r"//[^\n]*", "", f.read())
    assert "sim::derive_angle_intervals(" in src and "sim::dot_passes(" in src
    assert "acos" not in src
