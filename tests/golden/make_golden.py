"""Generate tests/golden/oracle_golden.json (committed fixture).

Run where a reference checkout exists and oracle/_ref has been built from the
reference's own nanoflann:   python tests/golden/make_golden.py
The kNN entries are produced with the REFERENCE kd-tree (oracle.RefKnn) when available, so the
fixture pins the brute-force restatement to the reference's own code on a case without exact ties.
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def compute(orc, use_ref=False):
    from cilantro_b200 import synth

    out = {}
    dst, src, nrm, T_ref = synth.icp_pair(20000, seed=42, noise=0.002, with_normals=True)
    T = T_ref.astype(np.float32)
    q = orc.transform_points(T, src)
    knn = orc.RefKnn(dst) if (use_ref and orc.have_ref()) else orc.BruteKnn(dst)
    idx, d2 = knn.query(q, np.float32(0.01**2))
    out["knn_idx_sha"] = _sha(idx.astype(np.int64))
    out["knn_d2_sha"] = _sha(d2.astype(np.float32))
    out["knn_backend"] = knn.kind
    bk = orc.BruteKnn(dst)
    r = orc.icp(dst, src, bk, metric="p2p", max_iter=8, tol=0.0, max_d2=np.float32(0.05**2))
    out["icp_p2p_T"] = r["T"].astype(np.float64).reshape(-1).tolist()
    r = orc.icp(dst, src, bk, metric="combined", dst_n=nrm, max_iter=6, tol=0.0, max_d2=np.float32(0.05**2),
                w_pt=0.1, w_pl=1.0)
    out["icp_combined_T"] = r["T"].astype(np.float64).reshape(-1).tolist()
    pts, cent = synth.kmeans_data(20000, 50, seed=42)
    labels, _ = orc.kmeans_assign(pts, cent)
    out["kmeans_labels_sha"] = _sha(labels.astype(np.int64))
    d, s, Tr, _ = synth.ransac_pairs(20000, 0.3, seed=42)
    T_h = orc.ransac_fit_samples(d, s, orc.ransac_samples(20000, 3, 16, 42))
    T_h[0] = Tr.astype(np.float32)
    out["ransac_counts"] = [int(c) for c in orc.ransac_score(d, s, T_h, 0.01)]
    out["pca_eigenvalues"] = orc.pca(pts)["eigenvalues"].astype(np.float64).tolist()
    # §8(f) rows: neighbourhoods (reference nanoflann when use_ref), normals, downsampling, engine lists
    sp, _ = synth.surface_cloud(8000, seed=42, noise=0.001)
    nk = orc.RefKnn(sp) if (use_ref and orc.have_ref()) else orc.BruteKnn(sp)
    ni, nd, nc = nk.neighborhoods(sp, 9, np.float32(0.05**2))
    out["nbr_idx_sha"], out["nbr_d2_sha"], out["nbr_cnt_sha"] = _sha(ni), _sha(nd), _sha(nc)
    nrm_o, curv_o, cov_o, _ = orc.estimate_normals(sp, nk, k=9, radius2=np.float32(0.05**2), view_point=[0.5, 0.5, 5.0])
    out["normals_cov_sha"] = _sha(cov_o)
    out["normals_first"] = nrm_o[:4].astype(np.float64).reshape(-1).tolist()
    out["curvature_first"] = curv_o[:4].astype(np.float64).tolist()
    ri, rd, rc = nk.neighborhoods(sp[:200], 0, np.float32(0.03**2), stride=64)
    out["radius_cnt_sha"], out["radius_d2_sha"] = _sha(rc), _sha(rd)
    for order in (0, 1):
        dp, dn, _ = orc.grid_downsample(sp, 0.04, normals=nrm_o, order=order)
        out[f"downsample_order{order}_sha"] = _sha(dp) + _sha(np.nan_to_num(dn))
    f, s_, v = orc.engine_correspondences(dst, src, T, bk, np.float32(0.02**2), search_dir="both",
                                          require_reciprocal=True, inlier_fraction=0.8)
    out["engine_both_recip_frac_sha"] = _sha(f) + _sha(s_) + _sha(v)
    f, s_, v = orc.engine_correspondences(dst, src, T, bk, np.float32(0.02**2), search_dir="first_to_second",
                                          one_to_one=True)
    out["engine_f2s_1to1_sha"] = _sha(f) + _sha(s_) + _sha(v)
    return out


if __name__ == "__main__":
    import oracle

    oracle.build()
    g = compute(oracle, use_ref=True)
    b = compute(oracle, use_ref=False)
    assert g["knn_idx_sha"] == b["knn_idx_sha"] and g["knn_d2_sha"] == b["knn_d2_sha"], \
        "brute-force restatement disagrees with the reference nanoflann on the golden case"
    for key in ("nbr_idx_sha", "nbr_d2_sha", "nbr_cnt_sha", "normals_cov_sha", "radius_cnt_sha", "radius_d2_sha"):
        assert g[key] == b[key], f"{key}: brute-force neighbourhoods disagree with the reference nanoflann"
    with open(os.path.join(HERE, "oracle_golden.json"), "w") as f:
        json.dump(g, f, indent=1)
    print("wrote oracle_golden.json; kNN backend:", g["knn_backend"])
