"""Host-only: the PLY passthrough of the PointCloud3f shim (tests/cpp/test_ply.cpp) — round trips in ascii and
binary, a hand-written file with another property layout and a face element, append / clear, a missing file."""
import os

import cxx

ROOT = cxx.ROOT
PLY = os.path.join(ROOT, "tests", "cpp", "test_ply.cpp")


def test_ply_passthrough(tmp_path):
    out = cxx.run(cxx.build(PLY, str(tmp_path / "test_ply"), ["-O1", "-Wall"]), tmp_path, timeout=120)
    assert "PLY checks passed" in out


def test_reads_the_reference_scans(tmp_path):
    """An excerpt of the reference's bundled scan, in its layout (binary little endian; colours between xyz and the
    normals, an extra 'radius' property), through the shim reader, compared with a direct numpy parse of the bytes."""
    import numpy as np
    import sys

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from golden.make_config1_fixture import EXCERPT as scan, read_test_ply

    out = cxx.run(cxx.build(PLY, str(tmp_path / "test_ply"), ["-O1"]), tmp_path, scan, timeout=120)
    lines = out.strip().splitlines()
    p, n, c = read_test_ply(scan)
    assert lines[0].split() == ["scan", str(p.shape[0]), "1", "1"]
    for ln in lines[1:]:
        f = ln.split()
        i = int(f[1])
        got = np.array([float(x) for x in f[2:5] + f[6:9] + f[10:13]], np.float32)
        want = np.concatenate([p[i], n[i], c[i]]).astype(np.float32)
        assert np.array_equal(got, want), (i, got, want)
