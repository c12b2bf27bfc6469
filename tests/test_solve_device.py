"""The O(1) solves of the ICP iteration as compiled for the GPU, against numpy float64 and against a g++ build of the
same headers.

tests/cuda/solve_harness.cu includes the shipped headers (solve_core.hpp, solve_warp.cuh, sym3_eigen.cuh) and is
compiled at test time with the library's own nvcc flags (cilantro_b200/build.py), so the device code tested here -
FMA-contracted, run inside a kernel - is the code the device-resident ICP loop and the normal estimation run. The
cases sit where these solves branch or lose accuracy:
  - nearest_rotation / kabsch_from_moments: the polar (Newton) path and the Jacobi SVD fallback on both sides of the
    acceptance threshold det(sigma) = 1e-6 |sigma|_F^3, reflections, rank 2 / 1 / 0, scales 1e-12 .. 1e12;
  - solve6_warp vs la::solve6: every partial-pivoting row swap, in particular the pivot rows 4 and 5 (second register)
    while k < 4, exact zero pivots and NaN entries;
  - sym3_smallest (normal estimation): planar, linear, isotropic and degenerate (w0 = w1) covariances, scales
    1e-20 .. 1e20.
Each GPU test prints its largest error against float64.
"""
import os

import numpy as np
import pytest

import cxx
import icp_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cilantro_b200", "csrc")
HARNESS = os.path.join(ROOT, "tests", "cuda", "solve_harness.cu")
EPS = np.finfo(np.float64).eps


def build_harness(outdir, device, include_first=()):
    """Compile the harness: nvcc with the library's flags (device) or g++ (host). include_first: directories searched
    before the library's sources (to build the harness against another version of a header)."""
    inc = [f"-I{d}" for d in include_first] + [f"-I{CSRC}"]
    exe = os.path.join(outdir, "solve_harness_dev" if device else "solve_harness_host")
    return cxx.harness(HARNESS, exe, inc, device)


def run(exe, mode, cases, tmpdir):
    dt = np.float32 if mode == "sym3" else np.float64
    rec = {"rotation": 20, "kabsch": 13, "solve6": 14, "sym3": 7}[mode]
    src, dst = os.path.join(tmpdir, f"{mode}.in"), os.path.join(tmpdir, f"{mode}.out")
    np.ascontiguousarray(cases, dt).tofile(src)
    cxx.run(exe, mode, src, dst)
    return np.fromfile(dst, dt).reshape(-1, rec)


@pytest.fixture(scope="module")
def host_exe(tmp_path_factory):
    return build_harness(str(tmp_path_factory.mktemp("solve_host")), device=False)


@pytest.fixture(scope="module")
def dev_exe(tmp_path_factory):
    return build_harness(str(tmp_path_factory.mktemp("solve_dev")), device=True)


# ---- cases -------------------------------------------------------------------------------------------------------
def _rot(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def _ratio_e(target):
    """e such that diag(1, 1, e) has det / |.|_F^3 = target."""
    e = target * 2 ** 1.5
    for _ in range(6):
        e = target * (2 + e * e) ** 1.5
    return e


def rotation_cases():
    """(sigma 3x3, kind). kind: 'unique' (U V^T unique under both reflection rules), 'rank2' (unique under the Kabsch
    rule only), 'rank1', 'zero'."""
    rng = np.random.default_rng(11)
    out = []
    for _ in range(40):
        out.append((rng.normal(size=(3, 3)), "unique"))  # random: either sign of det
    for c in (1e-3, 0.08, 1.0, 250.0):
        for _ in range(4):
            out.append((c * _rot(rng), "unique"))  # isotropic sigma = c R (a uniform cube)
    for target in (1e-6 * (1 - 1e-2), 1e-6 * (1 + 1e-2)):
        for _ in range(8):
            out.append((_rot(rng) @ np.diag([1.0, 1.0, _ratio_e(target)]) @ _rot(rng).T, "unique"))
    for sv in ([3.0, 2.0, 1.0], [1.0, 0.5, 1e-3], [2.0, 1.0, 0.9]):
        for _ in range(4):
            out.append((_rot(rng) @ np.diag(sv) @ np.diag([1, 1, -1]) @ _rot(rng).T, "unique"))  # reflections
    for _ in range(6):
        out.append((_rot(rng) @ np.diag([2.0, 0.7, 0.0]) @ _rot(rng).T, "rank2"))
        out.append((_rot(rng) @ np.diag([1.5, 0.0, 0.0]) @ _rot(rng).T, "rank1"))
    out.append((np.zeros((3, 3)), "zero"))
    for k in range(-12, 13, 2):
        out.append((10.0 ** k * (_rot(rng) @ np.diag([1.0, 0.6, 0.3]) @ _rot(rng).T), "unique"))
        out.append((10.0 ** k * (_rot(rng) @ np.diag([1.0, 0.6, -0.3]) @ _rot(rng).T), "unique"))
    return out


def _rotation_tol(sigma, flip_col):
    """Forward error bound of U V^T: eps |sigma| / (smallest sum of two signed singular values), where the singular
    value the reflection rule flips counts negative."""
    U, s, Vt = np.linalg.svd(sigma)
    sg = s.copy()
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        sg[2 if flip_col == 2 else 0] *= -1
    gap = min(abs(sg[0] + sg[1]), abs(sg[0] + sg[2]), abs(sg[1] + sg[2]))
    return 64 * EPS * s[0] / gap


def check_rotations(res, cases, label):
    worst = {}
    for (sigma, kind), r in zip(cases, res):
        R2, R0, polar = r[:9].reshape(3, 3), r[9:18].reshape(3, 3), bool(r[18])
        # the branch: polar_rotation's entry test (icp_ref.polar_accepts). Outside |sigma|_F ~ 1e-6 .. 1e6 its single-
        # precision Frobenius scaling is switched off and the plain Newton steps may run out before converging: the
        # SVD then answers instead, which is still correct
        acc = icp_ref.polar_accepts(sigma)
        if 1e-6 < np.linalg.norm(sigma) < 1e6:
            assert polar == acc, (label, kind, icp_ref.det_ratio(sigma))
        else:
            assert acc or not polar, (label, kind, icp_ref.det_ratio(sigma))
        for R, col in ((R2, 2), (R0, 0)):
            assert abs(np.linalg.det(R) - 1) < 1e-12 and np.abs(R @ R.T - np.eye(3)).max() < 1e-12, (label, kind)
        if kind == "unique":
            for R, col, ref in ((R2, 2, icp_ref.kabsch_rotation(sigma)), (R0, 0, icp_ref.rotation(sigma))):
                err = np.abs(R - ref).max()
                tol = max(_rotation_tol(sigma, col), 1e-13)
                assert err < tol, (label, kind, col, err, tol)
                key = "polar" if polar else "svd"
                worst[key] = max(worst.get(key, 0.0), err / tol)
        elif kind == "rank2":  # Kabsch rule: the proper rotation taking v0, v1 to u0, u1 is unique
            err = np.abs(R2 - icp_ref.kabsch_rotation(sigma)).max()
            assert err < 1e-12, (label, kind, err)
        elif kind == "rank1":  # R v0 = u0
            U, _, Vt = np.linalg.svd(sigma)
            assert np.abs(R2 @ Vt[0] - U[:, 0]).max() < 1e-12, (label, kind)
        else:
            assert np.array_equal(R2, np.eye(3)) and np.array_equal(R0, np.eye(3))
    return worst


def kabsch_cases():
    """(moments16, d, q) of small matched sets: 0, 1, 2 pairs, collinear and planar sets, and general ones."""
    rng = np.random.default_rng(12)
    out = []
    for n, shape in ((0, None), (1, None), (2, None), (3, None), (3, "line"), (8, "plane"), (50, None), (50, "plane"),
                     (50, "line"), (50, "point"), (400, None)):
        for _ in range(3):
            q = rng.normal(size=(n, 3)) * [1.0, 0.6, 0.3]
            if shape == "plane":
                q[:, 2] = 0.0
            if shape == "line":
                q[:, 1:] = 0.0
            if shape == "point":
                q[:] = q[:1]
            T = np.hstack([_rot(rng), rng.normal(size=(3, 1))])
            d = icp_ref.apply(T, q)
            s = np.zeros(16)
            s[0] = n
            s[1:4] = d.sum(0)
            s[4:7] = q.sum(0)
            s[7:16] = (d.T @ q).ravel()
            out.append((s, d, q))
    return out


def check_kabsch(res, cases, label):
    worst = 0.0
    for (s, d, q), r in zip(cases, res):
        T, ok = r[:12].reshape(3, 4), bool(r[12])
        n = len(d)
        assert ok == (n >= 3), (label, n)
        if n == 0:
            assert np.array_equal(T, icp_ref.identity()), label
            continue
        R = T[:, :3]
        assert abs(np.linalg.det(R) - 1) < 1e-6 and np.abs(R @ R.T - np.eye(3)).max() < 1e-6, (label, n)
        # every configuration here is an exact rigid copy: whether or not R is unique, it must map q onto d
        err = np.abs(icp_ref.apply(T, q) - d).max()
        assert err < 4e-6 * (1 + np.abs(d).max()), (label, n, err)
        worst = max(worst, err)
    return worst


def _pivots(A):
    """The row la::solve6 picks in each column: first row of largest |M[i][k]| (float64 elimination without FMA)."""
    M = np.array(A, np.float64)
    piv = []
    for k in range(6):
        p = k
        for i in range(k + 1, 6):
            if abs(M[i, k]) > abs(M[p, k]):
                p = i
        piv.append(p)
        M[[k, p]] = M[[p, k]]
        if M[k, k] == 0 or np.isnan(M[k, k]):
            continue
        r = 1.0 / M[k, k]
        for i in range(k + 1, 6):
            f = M[i, k] * r
            if f != 0:
                M[i, k:] -= f * M[k, k:]
    return piv


def _s28(A, b):
    s = np.zeros(28)
    s[0] = 1.0
    s[1:22] = np.asarray(A)[np.triu_indices(6)]
    s[22:] = b
    return s


def solve6_cases():
    """(s28, A, b, pattern). Random SPD (B B^T) and symmetric indefinite systems chosen so that the pivot sequence
    covers: a swap in every column k < 5, every pair (k < 4, pivot 4 / 5) and (4, 5); then exact zero pivots and NaN
    entries."""
    rng = np.random.default_rng(13)
    want = {(k, p) for k in range(4) for p in (4, 5)} | {(4, 5)}
    want_all_cols = 3  # systems with a swap in every column k = 0..4
    got = {}
    all_cols = []
    for trial in range(200000):
        B = rng.normal(size=(6, 6)) * rng.choice([1.0, 10.0], size=(6, 6))
        A = B @ B.T if trial % 2 == 0 else B + B.T
        piv = _pivots(A)
        pairs = {(k, p) for k, p in enumerate(piv) if p != k}
        for pr in pairs & want:
            if pr not in got:
                got[pr] = A
        if len(pairs) == 5 and len(all_cols) < 2 * want_all_cols:
            all_cols.append(A)
        if set(got) == want and len(all_cols) >= 2 * want_all_cols:
            break
    assert set(got) == want, sorted(want - set(got))
    out = []
    for pr, A in sorted(got.items()):
        out.append((A, f"swap k={pr[0]} piv={pr[1]}"))
    for A in all_cols:
        out.append((A, "swap in every column"))
    for _ in range(4):
        out.append((np.diag(rng.uniform(1, 2, 6)) * 10 + rng.normal(size=(6, 6)) * 0.1, "no swap"))
    out = [((A + A.T) / 2, pat) for A, pat in out]
    # exact zero pivots: a zero row / column (pivot 0 at k = 2), and a duplicated row and column of small integers
    Z = np.round(rng.normal(size=(6, 6)) * 4)
    Z = Z + Z.T
    Z[2, :] = 0
    Z[:, 2] = 0
    out.append((Z, "zero pivot"))
    # rows 4 and 5 equal (an exactly representable 2x2 block [[2, 2], [2, 2]] beside an SPD block): M[5][5] = 0 at k = 5
    D = np.zeros((6, 6))
    B = rng.normal(size=(4, 4))
    D[:4, :4] = B @ B.T + np.eye(4)
    D[4:, 4:] = 2.0
    out.append((D, "zero pivot"))
    # NaN entries: in the pivot row of a column that other rows already have exact zeros in
    for (i, j) in ((0, 3), (4, 5), (1, 1)):
        N = np.diag([4.0, 3.0, 5.0, 2.0, 6.0, 7.0])
        N[0, 1] = N[1, 0] = 1.0
        N[i, j] = N[j, i] = np.nan
        out.append((N, "nan"))
    cases = []
    for A, pat in out:
        b = rng.normal(size=6)
        cases.append((_s28(A, b), A, b, pat))
    return cases


def check_solve6(res, cases, label, warp):
    """res rows: la::solve6 (x, ok), solve6_warp (x, ok). Returns the largest |x - x_numpy| / bound per pattern."""
    worst = {}
    for (s, A, b, pat), r in zip(cases, res):
        x_s, ok_s, x_w, ok_w = r[:6], bool(r[6]), r[7:13], bool(r[13])
        if warp:  # the warp solve runs the same elimination: same flag, same NaN pattern, x to rounding
            assert ok_w == ok_s, (label, pat)
            assert np.array_equal(np.isnan(x_w), np.isnan(x_s)), (label, pat, x_s, x_w)
            fin = np.isfinite(x_s)
            dev = np.abs(x_w[fin] - x_s[fin]).max() if fin.any() else 0.0
            assert dev <= 1e-12 * max(1.0, np.abs(x_s[fin]).max() if fin.any() else 1.0), (label, pat, x_s, x_w)
            worst["warp vs serial " + pat.split(" k=")[0]] = max(worst.get("warp vs serial " + pat.split(" k=")[0], 0.0),
                                                                 dev)
        if pat == "nan":  # a NaN entry reaches a pivot: the solve reports it
            assert not ok_s, (label, x_s)
            continue
        if pat == "zero pivot":
            assert not ok_s, (label, pat)
            assert not np.isnan(x_s).any(), (label, pat, x_s)
            continue
        assert ok_s, (label, pat)
        x = np.linalg.solve(A, b)
        bound = 64 * EPS * np.linalg.cond(A) * np.abs(x).max()
        for xx, who in ((x_s, "serial"), (x_w, "warp") if warp else (x_s, "serial")):
            err = np.abs(xx - x).max()
            assert err < bound, (label, who, pat, err, bound)
            key = f"{who} {pat.split(' k=')[0]}"
            worst[key] = max(worst.get(key, 0.0), err / bound)
    return worst


# ---- host build (no GPU): the same headers through g++ -------------------------------------------------------------
def test_host_build_rotations(host_exe, tmp_path):
    cases = rotation_cases()
    res = run(host_exe, "rotation", np.array([c[0].ravel() for c in cases]), str(tmp_path))
    worst = check_rotations(res, cases, "host")
    assert "polar" in worst and "svd" in worst  # both branches ran


def test_host_build_kabsch(host_exe, tmp_path):
    cases = kabsch_cases()
    res = run(host_exe, "kabsch", np.array([c[0] for c in cases]), str(tmp_path))
    check_kabsch(res, cases, "host")


def test_host_build_solve6(host_exe, tmp_path):
    cases = solve6_cases()
    res = run(host_exe, "solve6", np.array([c[0] for c in cases]), str(tmp_path))
    check_solve6(res, cases, "host", warp=False)


# ---- device build ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_rotations_match_float64_and_host_build(dev_exe, host_exe, tmp_path):
    cases = rotation_cases()
    inp = np.array([c[0].ravel() for c in cases])
    dev = run(dev_exe, "rotation", inp, str(tmp_path))
    worst = check_rotations(dev, cases, "device")
    host = run(host_exe, "rotation", inp, str(tmp_path))
    assert np.array_equal(dev[:, 18], host[:, 18])  # same branch on the device as on the host
    # where the rotation is unique the two builds agree to rounding (rank-deficient input leaves a free rotation about
    # the null space that rounding decides: checked above for what is determined)
    uniq = np.array([k == "unique" for _, k in cases])
    diff = np.abs(dev[uniq, :18] - host[uniq, :18]).max()
    assert diff < 1e-12, diff
    print(f"\nrotation: max err / bound vs float64: {worst}; max |device - host| (unique cases) = {diff:.2e}")


@pytest.mark.gpu
def test_device_kabsch_from_moments(dev_exe, host_exe, tmp_path):
    cases = kabsch_cases()
    inp = np.array([c[0] for c in cases])
    dev = run(dev_exe, "kabsch", inp, str(tmp_path))
    worst = check_kabsch(dev, cases, "device")
    host = run(host_exe, "kabsch", inp, str(tmp_path))
    assert np.array_equal(dev[:, 12], host[:, 12])
    # general position (>= 3 points, not collinear): a unique rotation, the same from both builds
    uniq = np.array([len(d) >= 3 and np.linalg.matrix_rank(q - q.mean(0), tol=1e-9) >= 2 for _, d, q in cases])
    diff = np.abs(dev[uniq, :12] - host[uniq, :12]).max()
    assert diff < 1e-5, diff
    print(f"\nkabsch_from_moments: max |T q - d| = {worst:.2e}; max |device - host| (unique cases) = {diff:.2e}")


@pytest.mark.gpu
def test_device_solve6_warp_and_serial(dev_exe, host_exe, tmp_path):
    cases = solve6_cases()
    inp = np.array([c[0] for c in cases])
    dev = run(dev_exe, "solve6", inp, str(tmp_path))
    worst = check_solve6(dev, cases, "device", warp=True)
    host = run(host_exe, "solve6", inp, str(tmp_path))
    assert np.array_equal(dev[:, 6], host[:, 6]) and np.array_equal(np.isnan(dev[:, :6]), np.isnan(host[:, :6]))
    print("\nsolve6: max err / (64 eps cond |x|) vs float64, and max |warp - serial|:")
    for k in sorted(worst):
        print(f"  {k:32s} {worst[k]:.3e}")


def sym3_cases():
    """(cov6 float32, kind)."""
    rng = np.random.default_rng(14)
    out = []

    def cov(R, w, scale=1.0):
        C = scale * (R @ np.diag(w) @ R.T)
        return np.array([C[0, 0], C[0, 1], C[0, 2], C[1, 1], C[1, 2], C[2, 2]], np.float32)

    for _ in range(20):
        out.append((cov(_rot(rng), [0.0, 0.3, 1.0]), "planar"))
        out.append((cov(_rot(rng), [0.0, 0.0, 1.0]), "linear"))
        out.append((cov(_rot(rng), [0.5, 0.5, 1.0]), "w0=w1"))
        out.append((cov(_rot(rng), [1e-4, 0.4, 1.0]), "near-planar"))
        out.append((cov(_rot(rng), [1e-3, 0.2, 1.0]), "near-planar"))
        out.append((cov(_rot(rng), [0.05, 0.3, 1.0]), "generic"))
    for _ in range(3):
        out.append((cov(np.eye(3), [0.7, 0.7, 0.7]), "isotropic"))
        out.append((cov(_rot(rng), [0.7, 0.7, 0.7]), "isotropic"))
    for k in range(-20, 21, 4):
        for _ in range(3):
            out.append((cov(_rot(rng), [0.02, 0.3, 1.0], 10.0 ** k), "generic"))
    return out


@pytest.mark.gpu
def test_device_sym3_smallest(dev_exe, tmp_path):
    """Eigenvalues within 1e-6 w2; curvature w0 / (w0 + w1 + w2) relative where w0 > 1e-5 w2; the normal within
    eps / gap of the eigenvector (in the eigenspace when w0 = w1)."""
    cases = sym3_cases()
    res = run(dev_exe, "sym3", np.array([c[0] for c in cases]), str(tmp_path))
    worst = {}
    for (cv, kind), r in zip(cases, res):
        C = np.array([[cv[0], cv[1], cv[2]], [cv[1], cv[3], cv[4]], [cv[2], cv[4], cv[5]]], np.float64)
        wr, V = np.linalg.eigh(C)
        w, n, curv = r[:3].astype(np.float64), r[3:6].astype(np.float64), float(r[6])
        w2 = wr[2]
        ew = np.abs(w - wr).max() / w2
        assert ew < 1e-6, (kind, w, wr)
        assert abs(np.linalg.norm(n) - 1) < 1e-6, kind
        if kind == "isotropic":
            en = 0.0
        elif kind in ("w0=w1", "linear"):  # a two-dimensional eigenspace: any unit vector of it is right
            en = np.linalg.norm(C @ n - wr[0] * n) / w2
            assert en < 1e-6, (kind, en)
        else:
            gap = (wr[1] - wr[0]) / w2
            en = np.linalg.norm(np.cross(n, V[:, 0])) / np.linalg.norm(n)  # sin of the angle (1 - cos^2 would lose it)
            assert en < 1e-6 / gap, (kind, en, gap)
        kr = wr[0] / wr.sum()
        if wr[0] > 1e-5 * w2:
            ec = abs(curv - kr) / kr
            assert ec < 1e-6 * w2 / wr[0], (kind, curv, kr)
        else:
            ec = abs(curv - kr)
            assert ec < 1e-6, (kind, curv, kr)
        for key, v in (("eigenvalue / w2", ew), ("normal", en), ("curvature", ec)):
            worst[(kind, key)] = max(worst.get((kind, key), 0.0), v)
    print("\nsym3_smallest: max error vs float64")
    for (kind, key) in sorted(worst):
        print(f"  {kind:12s} {key:16s} {worst[(kind, key)]:.3e}")
