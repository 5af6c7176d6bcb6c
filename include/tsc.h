/*
 * tsc.h — C ABI of libtsc (traffic-signal-control simulator, H100 / sm_90a).
 *
 * This is the drop-in boundary for the hot path of cts198859/deeprl_signal_control:
 *   TrafficSimulator.step()/reset()            reference envs/env.py:544-631
 *   which today talks to SUMO through TraCI    reference envs/env.py:291-294, 455-471, 325-407
 * Each entry point below names the reference call sites it replaces.  The reference has no
 * FFI of its own (its "FFI" is the TraCI TCP socket), so the binding a maintainer adds is a
 * ctypes stub; INTEGRATION.md shows it.
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error (tsc_last_error() has the message);
 *     nothing throws across the boundary;
 *   - pointers named *_dev are caller-owned DEVICE pointers (e.g. torch tensors' data_ptr),
 *     pointers named *_host are caller-owned HOST pointers; no torch types appear here;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream); calls are
 *     stream-ordered and asynchronous unless stated otherwise;
 *   - one host thread per handle (the reference isolates envs per thread by port,
 *     envs/env.py:90-91).
 *
 * The same structs (tsc_net, tsc_cfg) are consumed by the CPU oracle (oracle/tsc_sim_ref.c),
 * which is TEST INFRASTRUCTURE ONLY and is never linked into this library.
 */
#ifndef TSC_H_
#define TSC_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TSC_MAX_NODE_LINKS 32 /* TLS link masks are uint32 (Monaco max = 22, envs/real_net_env.py:49-68) */

/* ---- static road network + demand, flattened by the Python host (net/ package) -------------------- */
typedef struct tsc_net {
  /* sizes */
  int32_t n_lanes;    /* normal lanes (grid: 180)                                                  */
  int32_t n_links;    /* lane->lane connections (grid: 300, 12 per junction)                       */
  int32_t n_nodes;    /* signalised nodes = agents, in SORTED-NAME order (envs/env.py:232)         */
  int32_t n_routes;   /* distinct vehicle routes                                                   */
  int32_t max_hops;   /* row stride of route_lane / route_link                                     */
  int32_t n_src;      /* demand sources (origin lane, route)                                       */
  int32_t horizon;    /* seconds covered by src_due                                                */
  int32_t n_det;      /* detector lanes = sum over nodes of de-duplicated incoming lanes           */
  int32_t n_obs;      /* sum_i n_s_i : floats per replica in the observation                       */
  int32_t max_phases; /* row stride of node_green / node_major                                     */
  int32_t max_na;     /* row stride of the fingerprint input [R][n_nodes][max_na]                  */
  int32_t n_slots;    /* sum of lane_cap : vehicle slots per replica                               */
  /* lanes */
  const float*   lane_len;      /* [n_lanes] m                                                     */
  const float*   lane_vmax;     /* [n_lanes] m/s  (large_grid/data/build_file.py:15-16,53-58)      */
  const int32_t* lane_cap;      /* [n_lanes] ring capacity (vehicles)                              */
  const int32_t* lane_slot0;    /* [n_lanes] first slot of the lane's ring                         */
  const int32_t* lane_inl_off;  /* [n_lanes+1] CSR into lane_inl                                   */
  const int32_t* lane_inl;      /* links ENTERING each lane, in merge-priority order               */
  /* links */
  const int32_t*  link_from;    /* [n_links]                                                       */
  const int32_t*  link_to;      /* [n_links]                                                       */
  const int32_t*  link_node;    /* [n_links] controlling node or -1 (uncontrolled)                 */
  const int32_t*  link_tlidx;   /* [n_links] position in the node's phase string                   */
  const float*    link_vmax;    /* [n_links] turning-speed limit, m/s                              */
  const uint32_t* link_cross;   /* [n_links] foes to yield to when own state is 'g'                */
  const uint32_t* link_merge;   /* [n_links] foes to yield to when own state is 'g' or 'G'         */
  /* routes */
  const int32_t* route_len;     /* [n_routes] hops                                                 */
  const int16_t* route_lane;    /* [n_routes][max_hops] lane of hop h                              */
  const int16_t* route_link;    /* [n_routes][max_hops] link leaving hop h, -1 = arrival           */
  /* signal programs: phase strings of envs/large_grid_env.py:40-41 / envs/real_net_env.py:49-68   */
  const int32_t*  node_n_phases;/* [n_nodes] = n_a_i                                               */
  const uint32_t* node_green;   /* [n_nodes][max_phases] bit i set iff char i in 'Gg'              */
  const uint32_t* node_major;   /* [n_nodes][max_phases] bit i set iff char i == 'G'               */
  /* detectors (ilds_in, envs/env.py:225-230) and neighbours (envs/env.py:209-216) */
  const int32_t* node_det_off;  /* [n_nodes+1] CSR into det_lane                                   */
  const int32_t* det_lane;      /* [n_det] lane id                                                 */
  const int32_t* node_nbr_off;  /* [n_nodes+1] CSR into node_nbr                                   */
  const int32_t* node_nbr;      /* neighbour node indices in neighbor_map list order               */
  /* observation gather program (envs/env.py:163-205): obs[k] = scale * source(kind, idx)          */
  const int32_t* node_obs_off;  /* [n_nodes+1] offsets of each agent's slice in the obs row        */
  const int32_t* obs_kind;      /* [n_obs] 0 = wave(det idx) 1 = wait(det idx) 2 = fingerprint     */
  const int32_t* obs_idx;       /* [n_obs] det index, or node*max_na + a for fingerprints          */
  const float*   obs_scale;     /* [n_obs] 1 or coop_gamma (envs/env.py:186-188)                   */
  /* demand (large_grid/data/build_file.py:268-326, real_net/data/build_file.py:15-105)            */
  const int32_t* src_lane;      /* [n_src] origin lane                                             */
  const int32_t* src_route;     /* [n_src]                                                         */
  const uint8_t* src_due;       /* [horizon][n_src] vehicles becoming due in second t              */
  /* stochastic demand (small_grid: JTRRouter turn ratios and `probability=` flows,
   * small_grid/data/build_file.py:167-307).  A due vehicle of source q with src_group[q] = g >= 0 is kept iff
   * src_plo[iv][q] <= u < src_phi[iv][q], u = U[0,1) drawn per (replica seed, second, g), iv = min(t / pint_sec,
   * n_pint - 1): sources of one group share u, so route choice among them is exclusive.  NULL / -1: off. */
  const int32_t* src_group;     /* [n_src] or NULL                                                 */
  const float*   src_plo;       /* [n_pint][n_src]                                                 */
  const float*   src_phi;       /* [n_pint][n_src]                                                 */
  int32_t n_pint, pint_sec;
} tsc_net;

/* ---- scalar configuration: vType + [ENV_CONFIG] (config/config_ma2c_large.ini:24-48) ---------- */
typedef struct tsc_cfg {
  /* vType (large_grid/data/build_file.py:279) + SUMO passenger defaults (SURVEY App. A) */
  float veh_len, min_gap, accel, decel, tau, sigma, speed_dev;
  /* detectors */
  float det_len;        /* E2 length from the stop line; <=0 = whole lane (real_net)               */
  float halt_speed;     /* 1.39 (E2 halting, grid reward) or 0.1 (lane halting, real_net)          */
  int32_t queue_cap;    /* per-lane cap in the reward: 10 for real_net (envs/env.py:333), else big */
  /* control protocol (envs/env.py:85-88, 566-579) */
  int32_t control_interval_sec, yellow_interval_sec, episode_length_sec, teleport_sec;
  /* state / reward (envs/env.py:96-100, 325-367, 439-442, 591-631) */
  float norm_wave, norm_wait, clip_wave, clip_wait, coef_wait, coop_gamma;
  int32_t objective;    /* 0 queue, 1 wait, 2 hybrid                                               */
  int32_t agent_mode;   /* 0 local rewards (greedy / test mode), 1 ia2c+iql (global), 2 ma2c       */
  int32_t real_net_norm;/* 1: divide as envs/env.py:599-601,625-629 (REALNET_REWARD_NORM = 20)     */
  int32_t use_wait;     /* 'wait' in state_names                                                   */
} tsc_cfg;

typedef struct tsc_handle tsc_handle;

/* Message of the last failing call on this thread. */
const char* tsc_last_error(void);

/* Replaces TrafficSimulator.__init__/_init_sim/_init_nodes (envs/env.py:83-110,207-242,271-294):
 * builds `n_replicas` lock-stepped copies of the network on CUDA device `device`.  The tables
 * are copied; the caller may free them afterwards. */
int tsc_create(const tsc_net* net, const tsc_cfg* cfg, int32_t n_replicas, int32_t device,
               tsc_handle** out);
int tsc_destroy(tsc_handle* h);

/* Replaces reset() (envs/env.py:544-561): empties every replica, sets prev_action = 0,
 * cur_sec = 0 and re-keys replica r's random streams with seeds_host[r] (the reference
 * re-seeds SUMO per episode, envs/env.py:278,560).  Host pointer, synchronous copy. */
int tsc_reset(tsc_handle* h, const uint64_t* seeds_host, void* stream);

/* Switch reward shaping between train (agent_mode) and test mode (local rewards,
 * envs/env.py:591-592). */
int tsc_set_train_mode(tsc_handle* h, int32_t train_mode);

/* Per-replica MA2C spatial discount (a hyperparameter sweep over coop_gamma in one simulator): cg_host [R] host floats,
 * copied (synchronous).  While set, replica r uses cg_host[r] wherever the process-wide cfg->coop_gamma applies: the
 * neighbour sum of the ma2c reward (envs/env.py:595-609) and the scale of the observation entries the network was
 * built to scale (neighbour waves, envs/env.py:184-188); every step / observe / record / host-range call reads it.
 * Replica r is then bit-identical to a simulator built with coop_gamma = cg_host[r] (the network must have been built
 * with a coop_gamma != 1, else no observation entry is marked as scaled).  NULL returns to cfg->coop_gamma. */
int tsc_set_replica_coop_gamma(tsc_handle* h, const float* cg_host);

/* Demand per replica (synchronous: synchronises the device, then replaces the previous setting).  n_levels demand
 * levels of the built net, each given by its three demand tables:
 *   due_host    uint8 [n_levels][horizon][n_src]        (tsc_net.src_due of that level)
 *   plo_host    float [n_levels][n_pint][n_src] or NULL (tsc_net.src_plo), phi_host likewise (tsc_net.src_phi):
 *               given exactly when the net has stochastic demand (src_group)
 *   level_host  int32 [R] level of each replica, each in [0, n_levels)
 * Every step / observe / record / host-range call then takes replica r's demand from level level_host[r], so replica
 * r is bit-identical to a simulator built with that level's tables (all other tables equal).  level_host NULL
 * returns to the built tables.  */
int tsc_set_replica_demand(tsc_handle* h, int32_t n_levels, const uint8_t* due_host, const float* plo_host,
                           const float* phi_host, const int32_t* level_host);

/* Fixed-time signal control (synchronous: synchronises the device, then replaces the previous program; call right
 * after tsc_reset, like tsc_set_record).  Node i runs a static program of n_phases_host[i] phases (1 <= n <= max_phases);
 * phase k (entry [i][k] of the [n_nodes][max_phases] host arrays) lasts dur_host[i][k] >= 1 seconds and shows the link
 * masks open_host ('G' or 'g'), major_host ('G') and yellow_host ('y'), bit j = link j of the node's phase string.
 * The cycle is C_i = sum of the durations; the simulated second s -> s + 1 runs with the phase k whose window
 * [start_k, start_k + d_k) holds (s - offset_host[i]) mod C_i.
 * While a program is set, tsc_step, tsc_step_record, tsc_step_host and both host-range calls run every replica on it:
 * they read no action (action_dev / action_host may be NULL), leave prev_action as it is, and the phase tap of
 * tsc_get_counts holds the program phase in force during the first second of the interval.  n_phases_host NULL
 * returns to action-driven stepping. */
int tsc_set_signal_program(tsc_handle* h, int32_t max_phases, const int32_t* n_phases_host, const int32_t* dur_host,
                           const uint32_t* open_host, const uint32_t* major_host, const uint32_t* yellow_host,
                           const int32_t* offset_host);

/* Fixed-time signal control with one program per replica (synchronous, like tsc_set_signal_program).  n_plans >= 1
 * programs, stacked: n_phases_host and offset_host [n_plans][n_nodes], dur_host, open_host, major_host and yellow_host
 * [n_plans][n_nodes][max_phases]; plan p is a program as tsc_set_signal_program takes it.  plan_host [R]: replica r runs
 * plan plan_host[r] (0 <= plan_host[r] < n_plans), bit-identical to a handle that runs that plan alone through
 * tsc_set_signal_program.  Every plan and every plan index is checked before anything is replaced; the error names the
 * plan.  The setting persists over tsc_reset, replaces the current fixed-time program and turns an actuated program off;
 * tsc_set_signal_program is the case of one plan run by every replica.  n_phases_host NULL turns it off. */
int tsc_set_replica_signal_programs(tsc_handle* h, int32_t n_plans, int32_t max_phases, const int32_t* n_phases_host,
                                    const int32_t* dur_host, const uint32_t* open_host, const uint32_t* major_host,
                                    const uint32_t* yellow_host, const int32_t* offset_host, const int32_t* plan_host);

/* Vehicle-actuated signal control (synchronous, like tsc_set_signal_program; validates every table before it replaces
 * anything).  Node i runs n_phases_host[i] phases in order (1 <= n <= max_phases); phase k (entry [i][k] of the
 * [n_nodes][max_phases] host arrays) shows the link masks open_host, major_host and yellow_host as in
 * tsc_set_signal_program and lasts between min_dur_host[i][k] and max_dur_host[i][k] seconds
 * (1 <= min_dur <= max_dur <= 2^30).  loop_pos_host[n_lanes]: the induction loop of each lane, in 1/64 m from the
 * lane start (0..65535), or -1 for none; every from-lane of a controlled link needs one.  Each lane keeps a gap g, the
 * seconds since its loop was last covered (saturating at 255, 255 after a reset): a vehicle covers it in a second iff
 * xq - Lq <= X <= xnq, xq / xnq its stored front position before / after the second's move (1/64 m; a head vehicle
 * that crosses or arrives has xnq = +inf), Lq = veh_len in 1/64 m.  At the end of every simulated second a node whose
 * phase k has run e seconds (this one included) advances to k + 1 mod n when e >= max_dur, or when e >= min_dur and
 * every loop on the from-lane of a link open in k has g >= max_gap_host[i] (>= 0; 0 ends every phase at min_dur, 256
 * or more runs it to max_dur); the new phase shows from the next second on.  init_host [n_nodes][2] = {phase,
 * elapsed seconds} of every node at simulated second 0 (0 <= elapsed <= 2^30).
 * Allocates the per-replica state ([R][n_nodes] phases, [R][lanes] gaps) and initialises every replica; tsc_reset
 * re-initialises it.  When the record-mode actuated state does not fit in shared memory, this call refuses while
 * record mode is on and tsc_set_record refuses while a program is set.  While set, the step calls behave as under tsc_set_signal_program (no action read, prev_action
 * kept, the phase tap holding the phase in force during the interval's first second).  Setting it turns a
 * tsc_set_signal_program program off, and setting that turns this one off; n_phases_host NULL turns it off and frees
 * the state. */
int tsc_set_actuated_program(tsc_handle* h, int32_t max_phases, const int32_t* n_phases_host,
                             const int32_t* min_dur_host, const int32_t* max_dur_host, const uint32_t* open_host,
                             const uint32_t* major_host, const uint32_t* yellow_host, const int32_t* init_host,
                             const int32_t* max_gap_host, const int32_t* loop_pos_host);

/* phase_dev [R][n_nodes] int32: the phase of every node's signal program (tsc_set_signal_program or
 * tsc_set_actuated_program) in force during the next simulated second.  Fails when no program is set. */
int tsc_get_program_phase(tsc_handle* h, int32_t* phase_dev, void* stream);

/* Replaces _get_state() without stepping (the observation reset() returns,
 * envs/env.py:561,163-205).  fp_dev: [R][n_nodes][max_na] policy probabilities installed by
 * update_fingerprint (envs/env.py:633-635) or NULL (zeros).  obs_dev: [R][n_obs]. */
int tsc_observe(tsc_handle* h, const float* fp_dev, float* obs_dev, void* stream);

/* Replaces step(action) (envs/env.py:566-631): yellow phase, yellow_interval 1-s sub-steps,
 * green phase, remaining sub-steps, state + reward measurement, reward shaping.
 *   action_dev  int32 [R][n_nodes]
 *   fp_dev      float [R][n_nodes][max_na] or NULL
 *   obs_dev     float [R][n_obs]
 *   reward_dev  float [R][n_nodes]   (shaped per agent_mode / train mode)
 *   greward_dev float [R]            (global_reward = sum of local rewards, envs/env.py:580)
 *   done_dev    uint8 [R]
 * Any output pointer may be NULL. */
int tsc_step(tsc_handle* h, const int32_t* action_dev, const float* fp_dev, float* obs_dev,
             float* reward_dev, float* greward_dev, uint8_t* done_dev, void* stream);

/* Same call with HOST buffers (pinned or pageable): copies action/fp in, runs the step and
 * copies the outputs back; synchronises the stream before returning.  This is the call the
 * reference-facing Python env uses for n_replicas == 1 and the one bench.py times as "e2e". */
int tsc_step_host(tsc_handle* h, const int32_t* action_host, const float* fp_host, float* obs_host,
                  float* reward_host, float* greward_host, uint8_t* done_host, void* stream);

/* The same call for the replica range [rep0, rep0 + count): host pointers are the bases of that range's slices
 * (action [count][n_nodes], obs [count][n_obs], ...).  Ranges are independent, so a caller can keep one range on the
 * PCIe link while another one computes (one stream per range; see agents/trainer.py:control_step_host_pipelined). */
int tsc_step_host_range(tsc_handle* h, int32_t rep0, int32_t count, const int32_t* action_host, const float* fp_host,
                        float* obs_host, float* reward_host, float* greward_host, uint8_t* done_host, void* stream);
/* Same without the final synchronisation: the copies and the kernel are only enqueued on `stream` (host buffers must be
 * page-locked and stay valid); the results are on the host once the caller has synchronised that stream. */
int tsc_step_host_range_async(tsc_handle* h, int32_t rep0, int32_t count, const int32_t* action_host,
                              const float* fp_host, float* obs_host, float* reward_host, float* greward_host,
                              uint8_t* done_host, void* stream);

/* ---- evaluation / recording path (replaces the per-second TraCI reads of `_measure_traffic_step` and SUMO's
 * --tripinfo-output; reference envs/env.py:409-437, 461-471, 498-542) ------------------------------------------
 * tsc_set_record(on): keep a trip word per vehicle (depart second, total waiting seconds, waiting episodes) and log
 *   one row per arrival.  Call right after tsc_reset; costs one more 4-byte word per vehicle slot in shared memory.
 * tsc_step_record: tsc_step advanced one simulated second per launch; sub_stats_dev [R][control_interval_sec][8]
 *   (may be NULL) receives the tsc_get_traffic_stats fields after every second.  Results equal tsc_step's.
 * tsc_get_trips: the arrival log of one replica, rows_host [max_rows][2] uint32:
 *   word 0 = depart_sec:12 | arrival_sec:12 | route:8,  word 1 = waiting seconds:16 | waiting episodes:16. */
int tsc_set_record(tsc_handle* h, int32_t on);
int tsc_step_record(tsc_handle* h, const int32_t* action_dev, const float* fp_dev, float* obs_dev, float* reward_dev,
                    float* greward_dev, uint8_t* done_dev, float* sub_stats_dev, void* stream);
int tsc_get_trips(tsc_handle* h, int32_t replica, uint32_t* rows_host, int32_t max_rows, int32_t* n_rows);

/* ---- greedy controllers (reference envs/large_grid_env.py:45-60, envs/real_net_env.py:78-111,
 * envs/small_grid_env.py:41-57) as one table-driven rule ------------------------------------------------------------
 * tsc_set_greedy_program: per node i and candidate c < max_cand (k = i * max_cand + c), the candidate scores the sum of
 *   the observation entries idx_host[off_host[k] .. off_host[k+1]) (offsets into the [n_obs] row) and maps to action
 *   act_host[k] (-1: no such candidate).  off_host [n_nodes * max_cand + 1].  Host arrays, copied (synchronous).
 * tsc_greedy_actions: action_dev int32 [R][n_nodes] = per node, the action of the FIRST candidate with the largest score,
 *   scores summed in float64 in table order (np.argmax over the reference's float64 sums, ties included).
 *   obs_dev float [R][n_obs]. */
int tsc_set_greedy_program(tsc_handle* h, int32_t max_cand, const int32_t* off_host, const int32_t* idx_host,
                           const int32_t* act_host);
int tsc_greedy_actions(tsc_handle* h, const float* obs_dev, int32_t* action_dev, void* stream);

/* ---- max-pressure controller (Varaiya 2013) ---------------------------------------------------------------------------
 * tsc_pressure_actions: action_dev int32 [R][n_nodes] = per replica r and node i, the FIRST phase p < node_n_phases[i]
 *   with the largest pressure
 *     P(r, i, p) = sum over links l with link_node[l] == i and bit link_tlidx[l] set in node_green[i][p]
 *                  of lane_cnt[r][link_from[l]] - lane_cnt[r][link_to[l]]
 *   (integer; lane_cnt = whole-lane vehicle counts, as tsc_dump_state returns them), read from the state the last
 *   tsc_step / tsc_step_record / tsc_observe left, the instant that call's observation describes.  Uncontrolled links
 *   (link_node = -1) and links into a lane outside the net (link_to = -1: no vehicle takes them) do not count.  The per-node link list is built from the net given to tsc_create on the first call
 *   (synchronous then); later calls are one stream-ordered launch. */
int tsc_pressure_actions(tsc_handle* h, int32_t* action_dev, void* stream);

/* Integer parity taps measured at the end of the last step, per detector lane
 * (lanearea.getLastStepVehicleNumber / getLastStepHaltingNumber / head getWaitingTime,
 * envs/env.py:333-349,377-395) and per node (the phase index = action applied).
 * All device pointers, int32; any may be NULL. */
int tsc_get_counts(tsc_handle* h, int32_t* veh_dev /*[R][n_det]*/, int32_t* halt_dev /*[R][n_det]*/,
                   int32_t* headwait_dev /*[R][n_det]*/, int32_t* phase_dev /*[R][n_nodes]*/,
                   void* stream);

/* Per-replica traffic statistics of the last simulated second (_measure_traffic_step,
 * envs/env.py:409-437): stats_dev float [R][8] =
 * {n_live, n_departed_total, n_arrived_total, avg_wait, avg_speed, avg_queue, std_queue, backlog};
 * avg/std_queue = lane halting number (speed < 0.1 m/s) over the detector lanes. */
int tsc_get_traffic_stats(tsc_handle* h, float* stats_dev, void* stream);

/* Debug / parity: copy replica r's full vehicle state to the host in canonical form:
 * lane_cnt_host int32[n_lanes], veh_host uint32[3*n_slots] (lane-major, front vehicle first,
 * 12-byte records {pos f32, speed f32, meta0 = wait:10|hop:6|route:8|speedFactor:8}); *n_veh = vehicles written.
 * Synchronous.
 * "vehicle record": on the device (HBM and shared memory) a vehicle is 8 bytes — word 0 = position:16 (1/64 m) |
 * speed:16 (1/1024 m/s), word 1 = meta0.  Both scales are powers of two, so this dump is the exact stored state;
 * positions are truncated and speeds rounded when a record is written (once per simulated second).  Limits checked by
 * tsc_create: lanes <= 959 m, speed limits <= 42 m/s. */
int tsc_dump_state(tsc_handle* h, int32_t replica, int32_t* lane_cnt_host, uint32_t* veh_host,
                   int32_t* n_veh);

/* Geometry of the compiled kernels / buffers, for bench.py's roofline arithmetic. */
int tsc_info(tsc_handle* h, int64_t* state_bytes_per_replica, int32_t* threads_per_block,
             int32_t* smem_bytes);

/* Mean live vehicles per replica right now (device reduction; synchronous). */
int tsc_mean_live(tsc_handle* h, double* mean_live);

#ifdef __cplusplus
}
#endif
#endif /* TSC_H_ */
