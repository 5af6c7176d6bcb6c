/*
 * fixedtime_ref.c — fixed-time mode of the CPU oracle (TEST INFRASTRUCTURE ONLY): oracle/tsc_sim_ref.c compiled as it
 * stands, plus one control step whose signals come from a static program instead of an action, the reference the
 * FIXED instantiations of tsc_step_kernel are pinned against (tests/test_fixedtime_gpu.py).
 *
 * The oracle's node_signal derives a node's signal from (action, previous action) through the net's phase tables.  With
 * a table of two entries per program phase k, 2k = (open_k, major_k) and 2k + 1 = (open_k | yellow_k, major_k), the
 * pair (a = 2k, p = 2k + 1) of a yellow sub-step shows exactly (open_k, major_k, yellow_k) (yellow_k and open_k are
 * disjoint, major_k lies in open_k), and (2k, 2k) shows (open_k, major_k, no yellow).  So every simulated second runs
 * the oracle's own substep with the program's link masks; prev_action is left as it was, as the device leaves it.
 */
#include "../oracle/tsc_sim_ref.c"

/* program phase of node i during simulated second `sec` (envs/fixedtime.py:phase_at) */
static int fx_phase(int P, const int32_t* n_phases, const int32_t* dur, const int32_t* offset, int i, int sec) {
  int cycle = 0;
  for (int k = 0; k < n_phases[i]; ++k) cycle += dur[i * P + k];
  int t = (sec - offset[i]) % cycle;
  if (t < 0) t += cycle;
  int k = 0;
  while (k < n_phases[i] - 1 && t >= dur[i * P + k]) { t -= dur[i * P + k]; ++k; }
  return k;
}

/* one control step of every replica on the program ([n_nodes][P] tables as tsc_set_signal_program takes them).
 * sub_stats [R][control_interval_sec][8] or NULL, as ref_step_record; phase [R][n_nodes] or NULL receives the program
 * phase of the interval's first second (the device's phase tap). */
void ref_step_fixed(ref_sim* s, int32_t P, const int32_t* n_phases, const int32_t* dur, const uint32_t* open,
                    const uint32_t* major, const uint32_t* yellow, const int32_t* offset, const float* fp, float* obs,
                    float* reward, float* greward, uint8_t* done, float* sub_stats, int32_t* phase) {
  tsc_net* n = &s->net;
  const tsc_cfg* c = &s->cfg;
  const int N = n->n_nodes, ci = c->control_interval_sec;
  uint32_t* g2 = (uint32_t*)calloc((size_t)N * 2 * P + 1, 4);
  uint32_t* m2 = (uint32_t*)calloc((size_t)N * 2 * P + 1, 4);
  for (int i = 0; i < N; ++i)
    for (int k = 0; k < P; ++k) {
      const size_t e = (size_t)i * P + k;
      g2[i * 2 * P + 2 * k] = open[e]; g2[i * 2 * P + 2 * k + 1] = open[e] | yellow[e];
      m2[i * 2 * P + 2 * k] = major[e]; m2[i * 2 * P + 2 * k + 1] = major[e];
    }
  const uint32_t* g_save = n->node_green; const uint32_t* m_save = n->node_major;
  const int32_t mp_save = n->max_phases;
  n->node_green = g2; n->node_major = m2; n->max_phases = 2 * P;
  int32_t* prev = (int32_t*)malloc(4 * (size_t)s->R * N + 4);
  for (int r = 0; r < s->R; ++r) {
    memcpy(prev + (size_t)r * N, s->rep[r].prev_action, 4 * (size_t)N);
    if (phase)
      for (int i = 0; i < N; ++i) phase[(size_t)r * N + i] = fx_phase(P, n_phases, dur, offset, i, s->rep[r].cur_sec);
  }
  float* vnew = (float*)malloc(4 * (size_t)n->n_slots + 4);
  float* xnew = (float*)malloc(4 * (size_t)n->n_slots + 4);
  uint8_t* flag = (uint8_t*)calloc((size_t)n->n_slots + 1, 1);
  uint8_t* hblk = (uint8_t*)calloc((size_t)n->n_lanes + 1, 1);
  float* head_lim = (float*)malloc(4 * (size_t)n->n_lanes + 4);
  uint32_t* approach = (uint32_t*)malloc(4 * (size_t)N + 4);
  uint32_t* o = (uint32_t*)malloc(4 * (size_t)N + 4);
  uint32_t* m = (uint32_t*)malloc(4 * (size_t)N + 4);
  uint32_t* ymask = (uint32_t*)malloc(4 * (size_t)N + 4);
  uint8_t* accepted = (uint8_t*)malloc((size_t)n->n_lanes + 1);
  int32_t* cnt_add = (int32_t*)malloc(4 * (size_t)n->n_lanes + 4);
  float* st = (float*)malloc(4 * 8 * (size_t)s->R);
  for (int t = 0; t < ci; ++t) {
    for (int r = 0; r < s->R; ++r) {
      replica_t* rp = &s->rep[r];
      for (int i = 0; i < N; ++i) {
        const int k = fx_phase(P, n_phases, dur, offset, i, rp->cur_sec);
        rp->cur_action[i] = 2 * k;
        rp->prev_action[i] = yellow[i * P + k] ? 2 * k + 1 : 2 * k;
      }
      substep(s, rp, 1, vnew, xnew, flag, hblk, head_lim, approach, o, m, ymask, accepted, cnt_add);
    }
    if (sub_stats) {
      ref_traffic_stats(s, st);
      for (int r = 0; r < s->R; ++r) memcpy(sub_stats + ((size_t)r * ci + t) * 8, st + 8 * (size_t)r, 32);
    }
  }
  n->node_green = g_save; n->node_major = m_save; n->max_phases = mp_save;
  for (int r = 0; r < s->R; ++r) {
    replica_t* rp = &s->rep[r];
    memcpy(rp->prev_action, prev + (size_t)r * N, 4 * (size_t)N);
    memcpy(rp->cur_action, prev + (size_t)r * N, 4 * (size_t)N);
    measure(s, rp);
    outputs(s, rp, fp ? fp + (size_t)r * N * n->max_na : 0, obs ? obs + (size_t)r * n->n_obs : 0,
            reward ? reward + (size_t)r * N : 0, greward ? greward + r : 0, done ? done + r : 0);
  }
  free(g2); free(m2); free(prev); free(vnew); free(xnew); free(flag); free(hblk); free(head_lim); free(approach);
  free(o); free(m); free(ymask); free(accepted); free(cnt_add); free(st);
}
