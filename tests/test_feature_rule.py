"""The feature-distance rule of the ICP's feature search, on the host. cilantro_b200/csrc/feature_rule.hpp is the one
source of the rule: feature_search.cu compiles it for the device, tests/cpp/test_feature_rule.cpp for the host, where it
is checked bit for bit against the reference's own nanoflann L2_Adaptor::evalMetric (D = 3, 6, 9), for the inequality
feature_d2 >= contract_d2(xyz part) that keeps the grid search exact, and for the rotated weighted normal against
float64. No GPU involved; the device side is tests/test_gpu_feature_icp.py."""
import os
import re

import numpy as np
import pytest

import cxx

ROOT, CSRC = cxx.ROOT, cxx.CSRC
NANOFLANN = "/root/reference/include/cilantro/3rd_party/nanoflann"


def _run(tmp_path, extra, args=()):
    exe = cxx.build(os.path.join(ROOT, "tests", "cpp", "test_feature_rule.cpp"), str(tmp_path / "test_feature_rule"),
                    ["-O2", "-frounding-math", "-ffp-contract=off", "-Wall", "-I", CSRC, *extra], link=False)
    out = cxx.run(exe, *args, timeout=600)
    assert "all feature-rule checks passed" in out and "FAIL" not in out
    return out


def test_feature_rule_inequality_and_rotation_on_the_host(tmp_path):
    out = _run(tmp_path, [])
    assert int(re.search(r"monotonicity checks: (\d+)", out).group(1)) >= 10**6


def test_feature_rule_matches_reference_nanoflann_bits(tmp_path):
    if not os.path.exists(os.path.join(NANOFLANN, "nanoflann.hpp")):
        pytest.skip("the reference checkout is not present")
    out = _run(tmp_path, ["-DCB_NANOFLANN", "-I", NANOFLANN])
    assert int(re.search(r"bit checks against nanoflann: (\d+)", out).group(1)) >= 10**6


def test_feature_rule_matches_the_prebuilt_reference_bits(tmp_path, orc):
    """The same samples against the reference's evalMetric as built into oracle/_ref (which travels with the tree where
    the reference checkout itself is absent)."""
    from oracle import feature_icp

    if not feature_icp.have_ref():
        pytest.skip("oracle/_ref was never built (no reference checkout when it was built)")
    path = tmp_path / "samples.bin"
    _run(tmp_path, [], [str(path)])
    x = np.fromfile(path, np.float32).reshape(-1, 21)
    assert x.shape[0] >= 400000
    for v, D in enumerate((3, 6, 9)):
        ref = feature_icp.ref_l2_eval(x[:, :D], x[:, 9:9 + D])
        rule = x[:, 18 + v]
        same = (ref.view(np.uint32) == rule.view(np.uint32)) | (np.isnan(ref) & np.isnan(rule))
        assert same.all(), (D, int((~same).sum()))


def test_the_feature_search_compiles_the_same_rule():
    """feature_search.cu computes its distance through rule::contract_d2 + rule::feature_d2 and its transform through
    rule::transform_point / rule::rotate_tail, never a private copy."""
    with open(os.path.join(CSRC, "feature_search.cu")) as f:
        src = re.sub(r"//[^\n]*", "", f.read())
    for call in ("rule::contract_d2(", "rule::feature_d2<", "rule::transform_point(", "rule::rotate_tail("):
        assert call in src, call
    assert "__fmul_rn" not in src and "__fadd_rn" not in src
