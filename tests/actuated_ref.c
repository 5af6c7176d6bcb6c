/*
 * actuated_ref.c — actuated mode of the CPU oracle (TEST INFRASTRUCTURE ONLY): oracle/tsc_sim_ref.c compiled as it
 * stands, plus one control step whose signals come from a vehicle-actuated program, the reference the ACTUATED
 * instantiations of tsc_step_kernel are pinned against (tests/test_actuated_gpu.py).
 *
 * Signals are shown as tests/fixedtime_ref.c shows them: a table of two entries per program phase k, 2k = (open_k,
 * major_k) and 2k + 1 = (open_k | yellow_k, major_k), and the action pair (2k, 2k + 1) when phase k has a yellow link,
 * (2k, 2k) otherwise.  Every simulated second runs the oracle's own substep.  The loop rule and the decision are
 * restated here, in the kernel's order: coverage from each vehicle's stored position before the second and the one its
 * move in B computed (the substep's xnew / flag scratch, indexed by the vehicle's slot, which C, D and E do not reuse
 * for a vehicle that was on the lane before the second), then the gap fold, then the per-node decision.
 */
#include "../oracle/tsc_sim_ref.c"

/* state [R][n_nodes][2] = {phase, seconds run before the next second}, gap [R][n_lanes]: updated in place.
 * sub_stats [R][control_interval_sec][8] or NULL, as ref_step_record; phase [R][n_nodes] or NULL receives the phase in
 * force during the interval's first second (the device's phase tap). */
void ref_step_actuated(ref_sim* s, int32_t P, const int32_t* n_phases, const int32_t* min_dur, const int32_t* max_dur,
                       const uint32_t* open, const uint32_t* major, const uint32_t* yellow, const int32_t* max_gap,
                       const int32_t* loop_pos, int32_t* state, uint8_t* gap, const float* fp, float* obs,
                       float* reward, float* greward, uint8_t* done, float* sub_stats, int32_t* phase) {
  tsc_net* n = &s->net;
  const tsc_cfg* c = &s->cfg;
  const int N = n->n_nodes, L = n->n_lanes, ci = c->control_interval_sec;
  const int Lq = (int)(c->veh_len * 64.0f);
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
      for (int i = 0; i < N; ++i) phase[(size_t)r * N + i] = state[((size_t)r * N + i) * 2];
  }
  float* vnew = (float*)malloc(4 * (size_t)n->n_slots + 4);
  float* xnew = (float*)malloc(4 * (size_t)n->n_slots + 4);
  uint8_t* flag = (uint8_t*)calloc((size_t)n->n_slots + 1, 1);
  uint8_t* hblk = (uint8_t*)calloc((size_t)L + 1, 1);
  float* head_lim = (float*)malloc(4 * (size_t)L + 4);
  uint32_t* approach = (uint32_t*)malloc(4 * (size_t)N + 4);
  uint32_t* o = (uint32_t*)malloc(4 * (size_t)N + 4);
  uint32_t* m = (uint32_t*)malloc(4 * (size_t)N + 4);
  uint32_t* ymask = (uint32_t*)malloc(4 * (size_t)N + 4);
  uint8_t* accepted = (uint8_t*)malloc((size_t)L + 1);
  int32_t* cnt_add = (int32_t*)malloc(4 * (size_t)L + 4);
  int32_t* head0 = (int32_t*)malloc(4 * (size_t)L + 4);
  int32_t* cnt0 = (int32_t*)malloc(4 * (size_t)L + 4);
  int32_t* xq0 = (int32_t*)malloc(4 * (size_t)n->n_slots + 4);
  uint8_t* cov = (uint8_t*)malloc((size_t)L + 1);
  float* st = (float*)malloc(4 * 8 * (size_t)s->R);
  for (int t = 0; t < ci; ++t) {
    for (int r = 0; r < s->R; ++r) {
      replica_t* rp = &s->rep[r];
      int32_t* sr = state + (size_t)r * N * 2;
      uint8_t* gr = gap + (size_t)r * L;
      for (int i = 0; i < N; ++i) {
        const int k = sr[2 * i];
        rp->cur_action[i] = 2 * k;
        rp->prev_action[i] = yellow[i * P + k] ? 2 * k + 1 : 2 * k;
      }
      for (int l = 0; l < L; ++l) {      /* positions before the second */
        head0[l] = rp->head[l]; cnt0[l] = rp->cnt[l];
        for (int k = 0; k < cnt0[l]; ++k) {
          const int slot = (int)(veh_at(n, rp, l, k) - rp->ring);
          xq0[slot] = (int)(rp->ring[slot].xv & 0xffffu);
        }
      }
      substep(s, rp, 1, vnew, xnew, flag, hblk, head_lim, approach, o, m, ymask, accepted, cnt_add);
      /* B: loop coverage; xq - Lq <= X <= xnq, a crossing or arriving head vehicle at xnq = +inf */
      for (int l = 0; l < L; ++l) {
        cov[l] = 0;
        const int X = loop_pos[l];
        if (X < 0) continue;
        for (int k = 0; k < cnt0[l]; ++k) {
          int idx = head0[l] + k;
          if (idx >= n->lane_cap[l]) idx -= n->lane_cap[l];
          const int slot = n->lane_slot0[l] + idx;
          const int xnq = (int)(pack_xv(xnew[slot], 0.0f) & 0xffffu);
          if (xq0[slot] - Lq <= X && (flag[slot] != 0 || X <= xnq)) cov[l] = 1;
        }
      }
      for (int l = 0; l < L; ++l) gr[l] = cov[l] ? 0 : (gr[l] < 255 ? gr[l] + 1 : 255);
      /* the switch point: phase k has run e seconds including this one */
      for (int i = 0; i < N; ++i) {
        int k = sr[2 * i], e = sr[2 * i + 1] + 1;
        const size_t pe = (size_t)i * P + k;
        int end = e >= max_dur[pe];
        if (!end && e >= min_dur[pe]) {
          end = 1;
          for (int j = 0; j < n->n_links; ++j)
            if (n->link_node[j] == i && n->link_from[j] >= 0 && ((open[pe] >> n->link_tlidx[j]) & 1u) &&
                gr[n->link_from[j]] < max_gap[i])
              end = 0;
        }
        if (end) { k = k + 1 < n_phases[i] ? k + 1 : 0; e = 0; }
        sr[2 * i] = k; sr[2 * i + 1] = e;
      }
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
  free(o); free(m); free(ymask); free(accepted); free(cnt_add); free(head0); free(cnt0); free(xq0); free(cov); free(st);
}

/* test set-up: appends one vehicle record {xv, m0} (tsc.h vehicle record) at the tail of lane `lane` of replica r;
 * -1 when the lane is full */
int32_t ref_put_vehicle(ref_sim* s, int32_t r, int32_t lane, uint32_t xv, uint32_t m0) {
  const tsc_net* n = &s->net;
  replica_t* rp = &s->rep[r];
  const int cap = n->lane_cap[lane];
  if (rp->cnt[lane] >= cap) return -1;
  int idx = rp->head[lane] + rp->cnt[lane];
  if (idx >= cap) idx -= cap;
  const int slot = n->lane_slot0[lane] + idx;
  rp->ring[slot].xv = xv; rp->ring[slot].m0 = m0;
  if (rp->trip) rp->trip[slot] = 0;
  rp->cnt[lane]++;
  return 0;
}
