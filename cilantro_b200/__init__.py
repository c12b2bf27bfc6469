"""cilantro_b200 — H100-native (sm_90a) rigid-ICP / k-means / RANSAC / PCA hot path of cilantro.

The product is the shared library cilantro_b200/libcilantro_b200.so (hand-written CUDA behind the
C ABI of include/cilantro_b200.h) plus the C++ header shims in include/cilantro/. This Python
package only holds the build script, a ctypes binding used by tests/ and bench.py, and the seeded
synthetic workloads of SURVEY.md §8(d).
"""
from . import capi  # noqa: F401

__all__ = ["capi"]
