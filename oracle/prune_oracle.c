/* CPU oracle of cvb_redundant_keyframes: the sequential culling pass of Map::Clean's redundancy pruning
 * (map_be.cpp:745-811), incremental and single-threaded like the reference, which runs it on one thread under the map lock.
 *
 * ASSUMPTION (parity unpinned beyond the source): the reference's source is not in this tree; the rule is restated from
 * the ORB-SLAM3 KeyFrameCulling lineage the pass follows.  Every clause below is an assumption, and the library defines
 * the one canonical result (include/covins_b200.h, cvb_redundant_keyframes):
 *   - an observation takes part iff obs_skip is NULL or 0 for it, its landmark iff lm_valid is NULL or 1 for it;
 *   - Λ(k) = k's participating landmarks, fixed for the whole pass (landmarks are not erased), n(k) = |Λ(k)|;
 *   - for the set C culled so far, l in Λ(k) is redundant iff at least th_obs keyframes k' not in C, k' != k, observe l
 *     with octave(k', l) <= octave(k, l) + 1; red_C(k) counts them;
 *   - pred_C(k) = k's nearest chain ancestor not in C, succ(k) = its original successor;
 *   - for k = 0 .. K-1: cull k iff not protected, n(k) > 0, (double)red_C(k) > th_red * (double)n(k), pred_C(k) and
 *     succ(k) exist, and kf_time[succ(k)] - kf_time[pred_C(k)] <= max_time_dist.
 * Incremental state: a culled flag per keyframe (the observers' scan skips culled keyframes) and pred_C, re-linked on
 * every cull (pred_C[succ(k)] = pred_C[k]).  Test infrastructure only; built with -ffp-contract=off. */
#include <stdint.h>
#include <stdlib.h>

#define EXPORT __attribute__((visibility("default")))

/* → 0, or -1 for input the pass is not defined on (an index out of range, kf_pred[k] >= k, two successors) */
EXPORT int ora_redundant_keyframes(int K, int L, const int32_t* lm_obs_ptr, const int32_t* obs_kf, const int32_t* obs_octave,
                                   const uint8_t* obs_skip, const uint8_t* lm_valid, const int32_t* kf_pred, const double* kf_time,
                                   const uint8_t* kf_protect, double th_red, double max_time_dist, int th_obs, uint8_t* culled) {
  int rc = -1;
  int32_t* succ = malloc(sizeof(int32_t) * (size_t)(K + 1));
  int32_t* pred_c = malloc(sizeof(int32_t) * (size_t)(K + 1));
  int32_t* kf_ptr = calloc((size_t)K + 2, sizeof(int32_t));
  const int n_obs = L ? lm_obs_ptr[L] : 0;
  int32_t* kf_obs = malloc(sizeof(int32_t) * (size_t)(n_obs + 1));   /* participating observation indices by keyframe */
  int32_t* obs_lm = malloc(sizeof(int32_t) * (size_t)(n_obs + 1));
  if (!succ || !pred_c || !kf_ptr || !kf_obs || !obs_lm) goto out;
  for (int k = 0; k < K; k++) succ[k] = -1;
  for (int k = 0; k < K; k++) {
    if (kf_pred[k] < -1 || kf_pred[k] >= k) goto out;
    if (kf_pred[k] >= 0) {
      if (succ[kf_pred[k]] >= 0) goto out;
      succ[kf_pred[k]] = k;
    }
    pred_c[k] = kf_pred[k];
    culled[k] = 0;
  }
  for (int l = 0; l < L; l++)
    for (int o = lm_obs_ptr[l]; o < lm_obs_ptr[l + 1]; o++) {
      if (obs_kf[o] < 0 || obs_kf[o] >= K) goto out;
      obs_lm[o] = l;
      if ((!lm_valid || lm_valid[l]) && !(obs_skip && obs_skip[o])) kf_ptr[obs_kf[o] + 2]++;
    }
  for (int k = 0; k < K; k++) kf_ptr[k + 2] += kf_ptr[k + 1];
  for (int l = 0; l < L; l++)
    for (int o = lm_obs_ptr[l]; o < lm_obs_ptr[l + 1]; o++)
      if ((!lm_valid || lm_valid[l]) && !(obs_skip && obs_skip[o])) kf_obs[kf_ptr[obs_kf[o] + 1]++] = o;
  /* kf_ptr[k] .. kf_ptr[k+1] now holds k's participating observations */
  for (int k = 0; k < K; k++) {
    const int n = kf_ptr[k + 1] - kf_ptr[k];
    if (kf_protect[k] || n == 0 || pred_c[k] < 0 || succ[k] < 0) continue;
    int red = 0;
    for (int t = kf_ptr[k]; t < kf_ptr[k + 1]; t++) {
      const int o = kf_obs[t], l = obs_lm[o];
      int others = 0;
      for (int q = lm_obs_ptr[l]; q < lm_obs_ptr[l + 1]; q++) {
        const int k2 = obs_kf[q];
        if (k2 == k || culled[k2] || (obs_skip && obs_skip[q])) continue;
        if (obs_octave[q] <= obs_octave[o] + 1) others++;
      }
      red += others >= th_obs;
    }
    if (!((double)red > th_red * (double)n)) continue;
    if (!(kf_time[succ[k]] - kf_time[pred_c[k]] <= max_time_dist)) continue;
    culled[k] = 1;
    pred_c[succ[k]] = pred_c[k];
  }
  rc = 0;
out:
  free(succ); free(pred_c); free(kf_ptr); free(kf_obs); free(obs_lm);
  return rc;
}
