"""numpy restatement of cb_vectors_mds (DESIGN §4.19): computeDistancePreservingSpectralEmbedding
(utilities/multidimensional_scaling.hpp:35-83) with the eigen-solve done by numpy.linalg.eigh in float64."""
import numpy as np


def nev_of(n, max_dim, estimate_dim):
    """Number of eigenpairs; None when Spectra's rule 1 <= nev <= n - 1 (or the estimation bound) rejects it."""
    nev = min(max_dim + 1, n - 1) if estimate_dim else max_dim
    if nev < 1 or nev > n - 1 or (estimate_dim and max_dim > n - 1):
        return None
    return nev


def xf_args(n, max_dim, estimate_dim):
    """MultidimensionalScalingXf's constructor: dim 2 without estimation when max_dim == 0 or max_dim >= n."""
    return (max_dim, estimate_dim) if 0 < max_dim < n else (2, False)


def entries(dm, squared):
    """The fp32 entries E: the input, or its fp32 square (one rounding)."""
    dm = np.asarray(dm, np.float32)
    return dm if squared else (dm * dm).astype(np.float32)


def b_matrix(dm, squared):
    """The symmetric B whose entries for i >= j are -1/2 (E_ij - r_i - c_j + g), in float64."""
    e = entries(dm, squared).astype(np.float64)
    r, c, g = e.mean(axis=1), e.mean(axis=0), e.mean()
    full = -0.5 * (e - r[:, None] - c[None, :] + g)
    low = np.tril(full)
    return low + np.tril(full, -1).T


def magnitude_order(w):
    """Indices by descending |w|, the positive value first at equal magnitude, then the lower index."""
    return sorted(range(len(w)), key=lambda i: (-abs(w[i]), -w[i], i))


def sign_rule(v):
    """v signed so that its largest-magnitude component is positive (the lowest index on ties)."""
    big = int(np.argmax(np.abs(v)))
    return v if v[big] >= 0 else -v


def eigengap_dim(ev, max_dim):
    """estimateEmbeddingDimensionEigengap (:9-31) in float32."""
    ev = np.asarray(ev, np.float32)
    m = ev.size
    best, ind = -np.inf, 0
    for i in range(m - 1):
        d = np.float32(ev[i] - ev[i + 1])
        if d > best:
            best, ind = d, i
    spread = np.float32(ev.max() - ev.min()) if np.all(np.isfinite(ev)) else np.float32(-np.inf)
    if not spread >= np.finfo(np.float32).eps:
        return max_dim
    return ind + 1


def mds(dm, max_dim, estimate_dim=False, squared=True):
    """dict(eigenvalues (fp64, clamped), eigenvalues32, dim, vectors (n x nev, signed), embedding (n x dim fp64), B)."""
    n = np.asarray(dm).shape[0]
    nev = nev_of(n, max_dim, estimate_dim)
    if nev is None:
        raise ValueError("invalid number of eigenvalues")
    B = b_matrix(dm, squared)
    w, V = np.linalg.eigh(B)
    order = magnitude_order(w)[:nev]
    lam = np.maximum(w[order], 0.0)
    vecs = np.stack([sign_rule(V[:, i]) for i in order], axis=1)
    lam32 = lam.astype(np.float32)
    dim = eigengap_dim(lam32, max_dim) if estimate_dim else max_dim
    emb = vecs[:, :dim] * np.sqrt(lam32[:dim].astype(np.float64))[None, :]
    return {"eigenvalues": lam, "eigenvalues32": lam32, "dim": dim, "vectors": vecs, "embedding": emb, "B": B,
            "all_eigenvalues": w}


def ring(n=1000):
    """The wavy ring of the reference example: (cos t, sin t, 0.1 sin 10 t), fp32, and its squared distances."""
    t = (2.0 * np.pi * np.arange(n)) / n
    p = np.stack([np.cos(t), np.sin(t), 0.1 * np.sin(10.0 * t)], axis=1).astype(np.float32)
    d = p[:, None, :] - p[None, :, :]
    return p, (d * d).sum(axis=2).astype(np.float32)


def points_distances(p, squared=True):
    """fp32 Euclidean distances (or squared distances) of the rows of p, computed in float64 and rounded once."""
    p = np.asarray(p, np.float64)
    g = (p * p).sum(axis=1)
    d2 = np.maximum(g[:, None] + g[None, :] - 2.0 * p @ p.T, 0.0)
    np.fill_diagonal(d2, 0.0)
    return (d2 if squared else np.sqrt(d2)).astype(np.float32)
