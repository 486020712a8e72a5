"""The verification chain of cvb_verify_noncentral_relative_pose_seeded_batch composed from the existing oracles — TEST
INFRASTRUCTURE ONLY.

verify_noncentral_seeded runs the matching oracle (oracle/knn_oracle.c: 2-NN and the ratio filter) per pairing, then the seeded
5-point, 17-point and covariance drivers of oracle/seeded.py (the C sampler feeding the unchanged C oracles); gather_matches and
merge_inliers are its two glue steps.  It adds no numerical oracle of its own."""
import numpy as np

from . import knn as oknn
from . import seeded as osd


def gather_matches(kf_ptr, bearings, sigma, pairs, match_train):
    """the 5-point problems of the pairings: match_train [P] per pairing (accepted train row per query row of kf1, or -1) →
    dict(prob_ptr, f1, f2, sigma1, sigma2, row1, row2), the accepted matches of each pairing in query order"""
    ptr, f1, f2, s1, s2, r1, r2 = [0], [], [], [], [], [], []
    for (a, b, _, _), mt in zip(pairs, match_train):
        for i, t in enumerate(mt):
            if t < 0:
                continue
            qa, tb = kf_ptr[a] + i, kf_ptr[b] + t
            f1.append(bearings[qa]); f2.append(bearings[tb]); s1.append(sigma[qa]); s2.append(sigma[tb]); r1.append(i); r2.append(t)
        ptr.append(len(f1))
    return dict(prob_ptr=np.array(ptr, np.int32), f1=np.array(f1, np.float64).reshape(-1, 3), f2=np.array(f2, np.float64).reshape(-1, 3),
                sigma1=np.array(s1, np.float64), sigma2=np.array(s2, np.float64), row1=np.array(r1, np.int32), row2=np.array(r2, np.int32))


def merge_inliers(pair_ptr, pairs, g, mask5):
    """the 17-point problems of the candidates: their pairings in order, of each the 5-point inliers in match order with the
    pairing's cameras → dict(prob_ptr, f1, f2, sigma1, sigma2, cam1, cam2, src), src the 5-point correspondence of each entry"""
    ptr, src, c1, c2 = [0], [], [], []
    for c in range(len(pair_ptr) - 1):
        for q in range(pair_ptr[c], pair_ptr[c + 1]):
            for j in range(g["prob_ptr"][q], g["prob_ptr"][q + 1]):
                if mask5[j]:
                    src.append(j); c1.append(pairs[q][2]); c2.append(pairs[q][3])
        ptr.append(len(src))
    src = np.array(src, np.int64)
    return dict(prob_ptr=np.array(ptr, np.int32), f1=g["f1"][src].reshape(-1, 3), f2=g["f2"][src].reshape(-1, 3), sigma1=g["sigma1"][src],
                sigma2=g["sigma2"][src], cam1=np.array(c1, np.int32), cam2=np.array(c2, np.int32), src=src)


def verify_noncentral_seeded(kf_ptr, desc, bearings, sigma, cam_ptr1, cam_off1, cam_rot1, cam_ptr2, cam_off2, cam_rot2, pair_ptr, pairs, seeds5,
                             seeds, img_match_thres, ratio_thres, threshold5, max_iterations5, threshold17, max_iterations17, probability=0.99,
                             n_cov_samples=300):
    """same arguments and result dict (with the full correspondence list) as
    covins_b200.placerec.verify_noncentral_relative_pose_seeded, composed from the matching oracle and the seeded drivers"""
    kf_ptr = np.asarray(kf_ptr, np.int64); desc = np.asarray(desc, np.uint8).reshape(-1, 32)
    bearings = np.asarray(bearings, np.float64).reshape(-1, 3); sigma = np.asarray(sigma, np.float64).reshape(-1)
    pairs = np.asarray(pairs, np.int64).reshape(-1, 4); pair_ptr = np.asarray(pair_ptr, np.int64)
    rig = dict(cam_ptr1=cam_ptr1, cam_off1=cam_off1, cam_rot1=cam_rot1, cam_ptr2=cam_ptr2, cam_off2=cam_off2, cam_rot2=cam_rot2)
    match_train, n_matches = [], []
    for a, b, _, _ in pairs:
        q = desc[kf_ptr[a]:kf_ptr[a + 1]]; t = desc[kf_ptr[b]:kf_ptr[b + 1]]
        if len(q) == 0:                   # no query rows: no matches
            match_train.append(np.zeros(0, np.int32)); n_matches.append(0)
            continue
        idx, dist = oknn.knn_hamming_batch(q, t, np.array([0, len(t)], np.int32), 2)
        mt, _, cnt = oknn.ratio_filter(idx, dist.astype(np.float32), img_match_thres, ratio_thres)
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
