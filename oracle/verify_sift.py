"""The verification chain of cvb_verify_noncentral_relative_pose_sift_seeded_batch composed from the existing oracles — TEST
INFRASTRUCTURE ONLY.

verify_noncentral_sift_seeded is oracle/verify.py:verify_noncentral_seeded with the pairwise matching done by the L2 matching
oracle (oracle/knn_oracle.c: exact L2 2-NN of CV_32F rows, then the same ratio filter): its glue steps (gather_matches,
merge_inliers) and the seeded 5-point, 17-point and covariance drivers of oracle/seeded.py are the ORB chain's.  It adds no
numerical oracle of its own."""
import numpy as np

from . import knn as oknn
from . import seeded as osd
from .verify import gather_matches, merge_inliers


def verify_noncentral_sift_seeded(kf_ptr, desc, bearings, sigma, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2, cam_rot2, pair_ptr, pairs,
                                  seeds5, seeds, img_match_thres, ratio_thres, threshold5, max_iterations5, threshold17, max_iterations17,
                                  probability=0.99, n_cov_samples=300):
    """same arguments (desc [R,128] float32) and result dict (with the full correspondence list) as
    covins_b200.placerec.verify_noncentral_relative_pose_sift_seeded, composed from the matching oracle and the seeded drivers"""
    kf_ptr = np.asarray(kf_ptr, np.int64); desc = np.asarray(desc, np.float32).reshape(-1, 128)
    bearings = np.asarray(bearings, np.float64).reshape(-1, 3); sigma = np.asarray(sigma, np.float64).reshape(-1)
    pairs = np.asarray(pairs, np.int64).reshape(-1, 4); pair_ptr = np.asarray(pair_ptr, np.int64)
    rig = dict(cam_ptr1=cam_ptr1, cam_off1=cam_off1, cam_rot1=cam_rot1, cam_ptr2=cam_ptr2, cam_off2=cam_off2, cam_rot2=cam_rot2)
    match_train, n_matches = [], []
    for a, b, _, _ in pairs:
        q = desc[kf_ptr[a]:kf_ptr[a + 1]]; t = desc[kf_ptr[b]:kf_ptr[b + 1]]
        if len(q) == 0:                   # no query rows: no matches
            match_train.append(np.zeros(0, np.int32)); n_matches.append(0)
            continue
        idx, dist = oknn.knn_l2_batch(q, t, np.array([0, len(t)], np.int32), 2)
        mt, _, cnt = oknn.ratio_filter(idx, dist, img_match_thres, ratio_thres)
        match_train.append(mt[0]); n_matches.append(int(cnt[0]))
    g = gather_matches(kf_ptr, bearings, sigma, pairs, match_train)
    r5 = osd.ransac_central_relative_pose_seeded(g["prob_ptr"], g["f1"], g["f2"], g["sigma1"], g["sigma2"], seeds5, threshold5, max_iterations5, probability)
    m = merge_inliers(pair_ptr, pairs, g, r5["inlier_mask"])
    b17 = {k: m[k] for k in ("prob_ptr", "f1", "f2", "sigma1", "sigma2", "cam1", "cam2")}
    r17 = osd.ransac_noncentral_relative_pose_seeded(**b17, **rig, seeds=seeds, threshold=threshold17, max_iterations=max_iterations17,
                                                     probability=probability)
    rc = osd.relative_pose_covariance_seeded(m["prob_ptr"], m["f1"], m["f2"], m["cam1"], m["cam2"], inlier_mask=r17["inlier_mask"], seeds=seeds,
                                             ref_model=r17["best_model"], n_samples=n_cov_samples, **rig)
    n_total = int(g["prob_ptr"][-1])
    inl17 = np.zeros(n_total, np.int32)
    inl17[m["src"]] = r17["inlier_mask"]
    pairing = np.repeat(np.arange(len(pairs), dtype=np.int32), np.diff(g["prob_ptr"]))
    corr = np.stack([pairing, g["row1"], g["row2"], r5["inlier_mask"].astype(np.int32), inl17], 1).astype(np.int32).reshape(-1, 5)
    out = dict(n_matches=np.array(n_matches, np.int32), n_total=n_total, corr=corr, cov=rc["cov"], n_valid=rc["n_valid"])
    for k in ("best_sample", "best_model", "best_count", "iterations", "consumed"):
        out[k + "5"] = r5[k]; out[k] = r17[k]
    return out
