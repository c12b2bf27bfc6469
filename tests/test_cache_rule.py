"""The exclusion-cache rule of the device-resident ICP loop, on the host. cilantro_b200/csrc/cache_rule.hpp is the one
source of the rule: the cached-pass kernel of icp_loop.cu compiles it for the device, tests/cpp/test_cache_rule.cpp
compiles it for the host (directed rounding through <cfenv>) and checks every verdict against a brute-force search with
the contract arithmetic — tightest valid exclusion radius, converging transform sequences, lattice inputs with exact ties,
and an inflated radius that must be caught. No GPU involved; the device side of the same claim is
tests/test_gpu_loop.py (cache equals a fresh exact search, loops bit-identical with the host-driven loop)."""
import os
import re

import cxx

ROOT, CSRC = cxx.ROOT, cxx.CSRC


def test_cache_rule_against_brute_force_on_the_host(tmp_path):
    exe = cxx.build(os.path.join(ROOT, "tests", "cpp", "test_cache_rule.cpp"), str(tmp_path / "test_cache_rule"),
                    ["-O2", "-frounding-math", "-ffp-contract=off", "-Wall", "-I", CSRC], link=False)
    out = cxx.run(exe, timeout=600)
    assert "all cache-rule checks passed" in out and "FAIL" not in out


def test_the_cached_pass_kernel_compiles_the_same_rule():
    """The one cached-pass kernel calls rule::cached_match_test, searches store rule::cache_radius, and icp_loop.cu keeps
    no private copy of the bound arithmetic (the directed-rounding intrinsics of the test live in cache_rule.hpp only)."""
    with open(os.path.join(CSRC, "icp_loop.cu")) as f:
        src = re.sub(r"//[^\n]*", "", f.read())
    cached_kernels = re.findall(r"__global__\s+void\s+__launch_bounds__\(.*?\)\s*(\w*cached\w*)\(", src)
    assert cached_kernels == ["icp_cached_pipe_kernel"]
    assert len(re.findall(r"rule::cached_match_test\(", src)) == 1
    assert len(re.findall(r"rule::cache_radius\(", src)) >= 1
    assert "__fsub_rd" not in src and "__fmul_rd" not in src and "kDown17" not in src
    with open(os.path.join(CSRC, "cache_rule.hpp")) as f:
        rule = f.read()
    for intrinsic in ("__fsub_rd", "__fmul_rd", "__fmul_ru", "__fmaf_ru", "__fsqrt_ru", "__fsqrt_rd"):
        assert intrinsic in rule
    # the searches compute the contract distance through rule::contract_d2, never a private copy of it
    for name in ("nn_search.cuh", "warp_search.cuh", "warp_search_wide.cuh", "radius_lists.cuh", "knn_k.cu",
                 "segment.cu", "mean_shift.cu"):
        with open(os.path.join(CSRC, name)) as f:
            assert "__fmul_rn(dx, dx)" not in f.read(), name
