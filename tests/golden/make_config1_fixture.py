"""Generate the committed fixtures of BASELINE config 1 (the reference's own CPU-runnable case) from the reference's
bundled scan examples/test_clouds/test.ply (573 663 vertices with normals and colours), so that the tests run the
rigid_icp.cpp recipe on REAL scan data without the reference checkout:

  config1_cloud.npz  the scan voxel-downsampled with the ORACLE's restatement of PointCloud::gridDownsample at 12 mm
                     (the example uses 5 mm; a coarser grid keeps the fixture under 1 MB): points, normals (float32),
                     plus the oracle's 5 mm bin count as a known answer;
  scan_excerpt.ply   every vertex of a seeded choice of 12 mm bins, bytes and header layout as in test.ply (binary
                     little endian: float x y z, uchar r g b, float nx ny nz, float radius). The bins are complete, so
                     downsampling the excerpt reproduces those bins of config1_cloud.npz bit for bit.

    python tests/golden/make_config1_fixture.py <cilantro checkout>/examples/test_clouds/test.ply [--check]

--check compares the committed fixtures with a fresh derivation instead of writing them.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
EXCERPT = os.path.join(HERE, "scan_excerpt.ply")
EXCERPT_BINS = 160


def _read(path):
    with open(path, "rb") as f:
        header = b""
        while not header.endswith(b"end_header\n"):
            header += f.readline()
        n = int([ln for ln in header.decode().splitlines() if ln.startswith("element vertex")][0].split()[-1])
        dt = np.dtype([("p", "<f4", 3), ("c", "u1", 3), ("n", "<f4", 3), ("radius", "<f4")])
        v = np.frombuffer(f.read(n * dt.itemsize), dtype=dt, count=n)
    return header, v


def read_test_ply(path):
    _, v = _read(path)
    return (np.ascontiguousarray(v["p"]), np.ascontiguousarray(v["n"]),
            (np.float32(1.0 / 255.0) * v["c"].astype(np.float32)).astype(np.float32))


def excerpt_bytes(path):
    """test.ply restricted to every vertex of EXCERPT_BINS seeded 12 mm bins (index order kept)."""
    header, v = _read(path)
    key = np.floor(v["p"] * np.float32(1.0 / 0.012)).astype(np.int64)
    bins, inverse = np.unique(key, axis=0, return_inverse=True)
    pick = np.random.default_rng(12).choice(bins.shape[0], EXCERPT_BINS, replace=False)
    keep = np.isin(inverse.reshape(-1), pick)
    lines = header.decode().splitlines(keepends=True)
    lines = [f"element vertex {int(keep.sum())}\n" if ln.startswith("element vertex") else ln for ln in lines]
    return "".join(lines).encode() + v[keep].tobytes()


def derive(path):
    import oracle

    oracle.build()
    pts, nrm, col = read_test_ply(path)
    p5, _, _ = oracle.grid_downsample(pts, 0.005, normals=nrm, colors=col)
    p12, n12, _ = oracle.grid_downsample(pts, 0.012, normals=nrm)
    return dict(points=p12, normals=n12, n_source=np.int64(pts.shape[0]), n_bins_5mm=np.int64(p5.shape[0]))


if __name__ == "__main__":
    ply = sys.argv[1]
    fixture, excerpt = derive(ply), excerpt_bytes(ply)
    if "--check" in sys.argv:
        z = np.load(os.path.join(HERE, "config1_cloud.npz"))
        for k, v in fixture.items():
            assert np.asarray(v).tobytes() == np.asarray(z[k]).tobytes(), k
        with open(EXCERPT, "rb") as f:
            assert f.read() == excerpt, "scan_excerpt.ply"
        print("fixtures match the scan")
    else:
        np.savez_compressed(os.path.join(HERE, "config1_cloud.npz"), **fixture)
        with open(EXCERPT, "wb") as f:
            f.write(excerpt)
        print(f"{int(fixture['n_source'])} vertices -> {int(fixture['n_bins_5mm'])} bins at 5 mm, "
              f"{fixture['points'].shape[0]} at 12 mm (fixture); excerpt of {len(excerpt)} bytes")
