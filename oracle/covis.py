"""CPU oracle of cvb_covisibility: Keyframe::UpdateCovisibilityConnections (keyframe_be.cpp:559-608) for every keyframe.

ASSUMPTION (parity unpinned beyond the source): the reference's source is not in this tree; the loop below restates the
ORB-SLAM / CCM-SLAM lineage that function follows — per keyframe, count in a map how often every other keyframe
observes one of its landmarks; connect those reaching the threshold (15 in the lineage), or only the single best one when
none does, adding the connection on the other side too (AddConnectedKeyframe); keep the list sorted by weight.  The
reference's own result depends on the order the keyframes were updated in and, for equal weights, on pointer order; the
library defines the canonical, order-independent result (include/covins_b200.h, cvb_covisibility, rules 1-4):
  1. an observation takes part iff obs_skip is None or 0 for it, its landmark iff lm_valid is None or 1 for it
     (lm && !lm->IsInvalid());
  2. w(i, j), i != j = the number of participating landmarks both keyframes observe;
  3. i and j are connected iff w(i, j) >= min_weight, or i has no neighbour reaching min_weight, w(i, j) > 0 and j is
     i's best neighbour (largest weight, lowest index among equals), or the same with i and j exchanged;
  4. keyframe i's list: its connected keyframes by weight descending, then keyframe index ascending.
Plain Python, written for clarity; test infrastructure only.
"""
from collections import Counter

import numpy as np


def covisibility(lm_obs_ptr, obs_kf, K, obs_skip=None, lm_valid=None, min_weight=15):
    """→ (nbr_ptr [K+1] i32, nbr_kf [n] i32, nbr_w [n] i32)"""
    lm_obs_ptr = np.asarray(lm_obs_ptr); obs_kf = np.asarray(obs_kf)
    L = len(lm_obs_ptr) - 1
    # the containers: every landmark's observers, every keyframe's landmarks (rule 1)
    observers = [[] for _ in range(L)]
    landmarks_of = [[] for _ in range(K)]
    for l in range(L):
        if lm_valid is not None and not lm_valid[l]:
            continue
        for o in range(lm_obs_ptr[l], lm_obs_ptr[l + 1]):
            if obs_skip is not None and obs_skip[o]:
                continue
            k = int(obs_kf[o])
            assert k not in observers[l], f"keyframe {k} observes landmark {l} twice"
            observers[l].append(k)
            landmarks_of[k].append(l)
    # the reference's loop, one keyframe at a time: KFcounter[other]++ over the observers of its landmarks (rule 2)
    counter = []
    for i in range(K):
        c = Counter()
        for l in landmarks_of[i]:
            c.update(observers[l])
        c.pop(i, None)
        counter.append(c)
    # rule 3: the keyframes reaching the threshold, else the single best one; either side's choice connects both
    connected = [dict() for _ in range(K)]
    for i in range(K):
        chosen = [j for j, w in counter[i].items() if w >= min_weight]
        if not chosen and counter[i]:
            chosen = [min(counter[i], key=lambda j: (-counter[i][j], j))]
        for j in chosen:
            connected[i][j] = counter[i][j]
            connected[j][i] = counter[i][j]
    # rule 4
    nbr_ptr, nbr_kf, nbr_w = [0], [], []
    for i in range(K):
        for j in sorted(connected[i], key=lambda j: (-connected[i][j], j)):
            nbr_kf.append(j); nbr_w.append(connected[i][j])
        nbr_ptr.append(len(nbr_kf))
    return np.array(nbr_ptr, np.int32), np.array(nbr_kf, np.int32), np.array(nbr_w, np.int32)
