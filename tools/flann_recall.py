"""SURVEY §8a M2: the reference's SIFT branch calls cv::FlannBasedMatcher (approximate, randomised kd-forest); the CUDA path
computes the EXACT brute-force 2-NN (== cv::BFMatcher(NORM_L2)).  This script reports how much of FLANN's output the exact
matcher reproduces on SIFT-like synthetic keyframes — as recall of FLANN against the exact result (CPU only, cv2)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import cv2
from covins_b200 import synth

THR, RATIO = 500.0, 0.8      # SIFT thresholds of the place recognition (img_match_thres / ratio_thres for SIFT, SURVEY §8a M3)
desc, lm = synth.sift_keyframes(seed=7, n_kf=41, n_feat=300)
q = desc[0]
tot = dict(pairs=0, nn1=0, nn2=0, acc_exact=0, acc_flann=0, acc_both=0)
cv2.setRNGSeed(0)
for c in range(1, 41):
    t = desc[c]
    ex = cv2.BFMatcher(cv2.NORM_L2).knnMatch(q, t, k=2)
    fl = cv2.FlannBasedMatcher().knnMatch(q, t, k=2)
    for e, f in zip(ex, fl):
        tot["pairs"] += 1
        tot["nn1"] += e[0].trainIdx == f[0].trainIdx
        tot["nn2"] += {e[0].trainIdx, e[1].trainIdx} == {f[0].trainIdx, f[1].trainIdx}
        ae = e[0].distance <= THR and e[0].distance < RATIO * e[1].distance
        af = f[0].distance <= THR and f[0].distance < RATIO * f[1].distance
        tot["acc_exact"] += ae; tot["acc_flann"] += af; tot["acc_both"] += ae and af and e[0].trainIdx == f[0].trainIdx
print(f"cv2 {cv2.__version__}; 300 SIFT-like queries vs 40 candidate keyframes x 300 rows (synth.sift_keyframes, seed 7)")
print(f"FLANN (default kd-forest) vs exact brute force, per query row: nearest neighbour identical {tot['nn1']/tot['pairs']:.4f}, "
      f"both neighbours identical {tot['nn2']/tot['pairs']:.4f}")
print(f"matches accepted by the distance + ratio filter (thr {THR}, ratio {RATIO}): exact {tot['acc_exact']}, FLANN {tot['acc_flann']}, "
      f"identical in both {tot['acc_both']}  → recall of FLANN's accepted matches by the exact matcher "
      f"{tot['acc_both']/max(tot['acc_flann'],1):.4f}, of the exact ones by FLANN {tot['acc_both']/max(tot['acc_exact'],1):.4f}")
