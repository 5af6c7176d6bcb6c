// tsc_sim.cu — sm_90a (H100) control-step kernel + C ABI (include/tsc.h) of libtsc.
//
// One CTA advances ONE road-network replica through one whole control interval
// (reference envs/env.py:566-631: yellow phase, 2 x 1 s, green phase, 3 x 1 s, detector reads,
// reward, observation) with the replica's entire vehicle state resident in shared memory:
//
//   HBM  (compact, lane-major, SoA 8 B/vehicle)   --coalesced loads-->  per-lane FIFO rings in smem
//   5 x { A1 lane summaries + scan | A2 junction limits | B per-vehicle Krauss update |
//         C junction transfers | D pops | E insertion }
//   detector scan -> reward -> shaping -> observation gather -> compact store back to HBM
//
// so state crosses HBM exactly once per direction per control step (the five 1-second
// sub-steps are fused).  Threads map to LIVE vehicles (prefix sum over lane counts + binary
// search), not to ring slots, so SIMT lanes are not wasted on empty slots.
//
// Arithmetic contract (bit-exact against oracle/tsc_sim_ref.c): IEEE binary32, compiled with
// -fmad=false, default -prec-div/-prec-sqrt, only + - * / sqrt floor; integer counter-based RNG.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/tsc.h"

#ifndef TSC_THREADS
#define TSC_THREADS 256
#endif
#ifndef TSC_MIN_BLOCKS
#define TSC_MIN_BLOCKS 5   /* 8-byte vehicle records: 38.7 KB of shared memory per 5x5-grid replica -> 5 CTAs/SM */
#endif
#define INF_SPEED 1.0e9f
#define F_CROSS 1
#define F_ARRIVE 2
#define F_CLOSED 4 /* set by A2 on the lane's head flag: its stop line is closed (red / yellow-and-can-brake / yielding) */
#define CTL_FIXED 8 /* cur_sec, seed_lo, seed_hi, n_departed, n_arrived, 3 spare */

// ------------------------------------------------------------------------------------------------
struct __align__(16) LaneC { float len, vmax; int32_t slot0, cap; };                       // 16 B, one LDG.128
struct __align__(16) LinkC { int32_t from, node, tlidx; float vmax; uint32_t cross, merge; int32_t pad0, pad1; };  // 32 B

struct DevNet {
  int32_t n_lanes, n_links, n_nodes, n_routes, max_hops, n_src, horizon, n_det, n_obs, max_phases,
      max_na, n_slots, src_shared, lpad;
  const LaneC* lane;
  const int32_t* lane_inl_off;
  const int32_t* lane_inl;
  const LinkC* link;
  const int16_t* route_lane;
  const int16_t* route_link;
  const uint32_t* node_green;
  const uint32_t* node_major;
  const int32_t* node_det_off;
  const int32_t* det_lane;
  const int32_t* node_nbr_off;
  const int32_t* node_nbr;
  const int32_t* obs_kind;
  const int32_t* obs_idx;
  const float* obs_scale;
  const uint32_t* obs_prog;   // packed gather program: kind:2 | scaled:1 | index:29 (scale is 1 or obs_scale_val)
  float obs_scale_val;        // the one non-unit scale of the program (coop_gamma, envs/env.py:186-188)
  const int32_t* src_lane;
  const int32_t* src_route;
  const uint8_t* src_due;
  const int32_t* lane_src0;  // [n_lanes] first demand source entering at this lane or -1
  const int32_t* src_next;   // [n_src]   next source on the same lane (ascending index) or -1
  const int32_t* src_group;  // stochastic demand (tsc.h) or null
  const float* src_plo;
  const float* src_phi;
  int32_t n_pint, pint_sec;
};

struct StepArgs {
  DevNet net;
  tsc_cfg cfg;
  // state (HBM)
  uint32_t* veh;      // [R][2][n_slots]  compact lane-major records, SoA: pos:16|speed:16 fixed point, meta0
  uint8_t* lane_cnt;  // [R][lpad]
  int32_t* ctl;       // [R][ctl_words]
  int32_t* meas;      // [R][3*n_det + n_nodes]  parity taps
  int32_t ctl_words;
  int32_t n_sub;      // sub-steps to run (0 = observe only)
  int32_t train_mode;
  int32_t rep0;       // first replica of this launch (replica-range launches of the host-buffer pipeline)
  int32_t sub0;       // first sub-step of this launch within the control interval (0 except in record mode, which
                      // advances one simulated second per launch so that per-second traffic statistics can be read)
  // record mode (evaluation runs, envs/env.py:498-542): per-vehicle trip word and the arrival log
  uint32_t* trip;     // [R][n_slots]  depart:12 | total wait s:12 | wait episodes:8, parallel to veh
  uint32_t* trip_log; // [R][trip_cap][2]  {depart:12 | arrival:12 | route:8, wait s:16 | wait episodes:16}
  int32_t* trip_cnt;  // [R]
  int32_t trip_cap;
  // io
  const int32_t* action;
  const float* fp;
  float* obs;
  float* reward;
  float* greward;
  uint8_t* done;
  const float* cg;    // [R] per-replica coop_gamma (tsc_set_replica_coop_gamma) or null: cfg.coop_gamma / obs_scale_val
};

// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t mix32(uint32_t h) {
  h ^= h >> 16; h *= 0x7feb352dU; h ^= h >> 15; h *= 0x846ca68bU; h ^= h >> 16;
  return h;
}
// key of one simulated second of one replica (two rounds, computed once per sub-step), then ONE round per draw
__device__ __forceinline__ uint32_t rng_key(uint32_t s0, uint32_t s1, uint32_t a) {
  return mix32(mix32(s0 ^ (a * 0x9E3779B1U)) ^ s1);
}
__device__ __forceinline__ uint32_t rng_draw(uint32_t key, uint32_t b, uint32_t c) {
  return mix32(key ^ (b * 0x85EBCA77U + c * 0xC2B2AE3DU));
}
__device__ __forceinline__ float u01(uint32_t h) { return (float)(h >> 8) * (1.0f / 16777216.0f); }

// Krauss / Euler helpers (SUMO MSCFModel restated; same operation order as the oracle)
// ib = 1 / b, formed once by a float division and multiplied here (same in the oracle)
__device__ __forceinline__ float brake_gap(float v, float b, float ib) {
  int steps = (int)(v * ib);
  float fs = (float)steps;
  float t1 = fs * v;
  float t2 = b * fs;
  float t3 = fs + 1.0f;
  float t4 = t2 * t3;
  float t5 = t4 * 0.5f;
  return t1 - t5;
}
__device__ __forceinline__ float stop_speed(float gap, float b, float ib, float tau) {
  float g = gap - 0.001f;
  if (g < 0.0f) return 0.0f;
  float q = (2.0f * g) * ib;
  q = q - tau;
  float tt = tau * tau;
  float disc = 1.0f + 4.0f * (q + tt);
  float sq = sqrtf(disc);
  float n = floorf(0.5f - (tau + sq * -0.5f));
  float h1 = 0.5f * n;
  h1 = h1 * (n - 1.0f);
  h1 = h1 * b;
  float h2 = n * b;
  h2 = h2 * tau;
  float h = h1 + h2;
  float r = (g - h) / (n + tau);
  return n * b + r;
}
__device__ __forceinline__ float follow_speed(float gap, float v_lead, float b, float ib, float tau) {
  return stop_speed(gap + brake_gap(v_lead, b, ib), b, ib, tau);
}
__device__ __forceinline__ float free_speed(float dist, float target, float b) {
  if (dist < target) return target;
  float bb = b + 2.0f * target;
  float disc = bb * bb + (8.0f * b) * dist;
  float y = ((sqrtf(disc) - b) * 0.5f - target) / b;
  if (y < 0.0f) y = 0.0f;
  float yf = floorf(y);
  float eg = (yf * yf + yf) * 0.5f;
  eg = eg * b;
  eg = eg + yf * target;
  if (y > yf) eg = eg + target;
  float rem = dist - eg;
  if (rem < 0.0f) rem = 0.0f;
  float res = rem / (yf + 1.0f);
  res = res + yf * b;
  return res + target;
}
__device__ __forceinline__ float clipf(float x, float hi) {
  if (hi < 0.0f) return x;
  if (x < 0.0f) x = 0.0f;
  if (x > hi) x = hi;
  return x;
}

// Vehicle record = 8 bytes {pos:16 (1/64 m) | speed:16 (1/1024 m/s), meta0}; stored SoA both in HBM and in shared
// memory.  Power-of-two scales: unpacking is exact; positions are truncated when packed (a vehicle that stops 1 mm
// short of a stop line stays short of it), speeds rounded to nearest.  Same functions as in the oracle.
struct Ring { uint32_t* xv; uint32_t* m; uint32_t* t; };   // t: trip word (record mode only, else null)
__device__ __forceinline__ float veh_x(uint32_t xv) { return (float)(xv & 0xffffu) * 0.015625f; }
__device__ __forceinline__ float veh_v(uint32_t xv) { return (float)(xv >> 16) * 0.0009765625f; }
__device__ __forceinline__ uint32_t pack_xv(float x, float v) {
  int xq = (int)(x * 64.0f), vq = (int)(v * 1024.0f + 0.5f);
  xq = min(max(xq, 0), 65535);
  vq = min(max(vq, 0), 65535);
  return (uint32_t)xq | ((uint32_t)vq << 16);
}
#define T1_DEPART(t) ((t) & 4095u)
#define T1_WAIT(t) (((t) >> 12) & 4095u)
#define T1_WCNT(t) ((t) >> 24)
__device__ __forceinline__ uint2 ld2(const Ring& r, int i) { return make_uint2(r.xv[i], r.m[i]); }
__device__ __forceinline__ void st2(const Ring& r, int i, const uint2 e) { r.xv[i] = e.x; r.m[i] = e.y; }
#define M0_WAIT(m) ((m) & 1023u)
#define M0_HOP(m) (((m) >> 10) & 63u)
#define M0_ROUTE(m) (((m) >> 16) & 255u)
#define M0_SFQ(m) ((m) >> 24)

// Block-wide exclusive scan of cnt[0..n) into pre[0..n], pre[n] = total.  n <= 4*TSC_THREADS.
// Warp-shuffle scans + one smem hop; two __syncthreads.
__device__ __forceinline__ void block_scan(const int32_t* __restrict__ cnt, int32_t* __restrict__ pre,
                                           int32_t* __restrict__ wsum, int n) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int per = (n + TSC_THREADS - 1) / TSC_THREADS;
  int base = tid * per;
  int loc[4];
  int s = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int v = (j < per && base + j < n) ? cnt[base + j] : 0;
    loc[j] = s;
    s += v;
  }
  int incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  int woff = 0;
#pragma unroll
  for (int w = 0; w < TSC_THREADS / 32; ++w) woff += (w < warp) ? wsum[w] : 0;
  int excl = woff + incl - s;
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (j < per && base + j < n) pre[base + j] = excl + loc[j];
  if (tid == TSC_THREADS - 1) pre[n] = woff + incl;
  __syncthreads();
}

// The same scan split in two halves so that its two barriers can be shared with neighbouring phases:
// part 1 (before the barrier) leaves warp totals in wsum, part 2 (after it) writes pre[].
struct ScanCarry { int loc[4]; int incl; int s; };
__device__ __forceinline__ ScanCarry scan_part1(const int32_t* __restrict__ cnt, int32_t* __restrict__ wsum, int n) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int per = (n + TSC_THREADS - 1) / TSC_THREADS;
  const int base = tid * per;
  ScanCarry c;
  int s = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int v = (j < per && base + j < n) ? cnt[base + j] : 0;
    c.loc[j] = s;
    s += v;
  }
  int incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) wsum[warp] = incl;
  c.incl = incl; c.s = s;
  return c;
}
__device__ __forceinline__ void scan_part2(const ScanCarry& c, int32_t* __restrict__ pre, const int32_t* __restrict__ wsum, int n) {
  const int tid = threadIdx.x, warp = tid >> 5;
  const int per = (n + TSC_THREADS - 1) / TSC_THREADS;
  const int base = tid * per;
  int woff = 0;
#pragma unroll
  for (int w = 0; w < TSC_THREADS / 32; ++w) woff += (w < warp) ? wsum[w] : 0;
  const int excl = woff + c.incl - c.s;
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (j < per && base + j < n) pre[base + j] = excl + c.loc[j];
  if (tid == TSC_THREADS - 1) pre[n] = woff + c.incl;
}

// largest l in [0, n) with pre[l] <= k   (k < pre[n])
__device__ __forceinline__ int find_lane(const int32_t* __restrict__ pre, int n, int k) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (pre[mid] <= k) lo = mid; else hi = mid;
  }
  return lo;
}

// lane of compact vehicle index kk, warp-cooperatively: s_blk[j] = lane of compact index 32 j (written by the lane
// owners after the scan); the 32 lane boundaries that follow the lane of the warp's first vehicle are searched with
// shuffles (33 possible outcomes -> 6 halvings); falls back to the block-wide binary search when the warp spans more.
__device__ __forceinline__ int find_lane_warp(const int32_t* __restrict__ pre, const int32_t* __restrict__ blk, int L, int kk) {
  const int lane0 = blk[(kk & ~31) >> 5];
  const int bi = lane0 + 1 + (threadIdx.x & 31);
  const int bnd = pre[bi < L ? bi : L];
  int lo = 0, hi = 32;
#pragma unroll
  for (int itb = 0; itb < 6; ++itb) {
    const int mid = (lo + hi) >> 1;
    const int vb = __shfl_sync(0xffffffffu, bnd, mid & 31);
    if (lo < hi) { if (vb <= kk) lo = mid + 1; else hi = mid; }
  }
  return lo < 32 ? lane0 + lo : find_lane(pre, L, kk);
}
// s_blk for the current scan (own lanes of every thread)
__device__ __forceinline__ void fill_blk(const int32_t* __restrict__ pre, const int32_t* __restrict__ cnt, int32_t* __restrict__ blk,
                                         int l_lo, int l_hi) {
  for (int l = l_lo; l < l_hi; ++l) {
    const int p0 = pre[l], p1 = p0 + cnt[l];
    for (int j = (p0 + 31) >> 5; (j << 5) < p1; ++j) blk[j] = l;
  }
}

// signal state of node i for the yellow or the green part of the interval (envs/env.py:128-152)
__device__ __forceinline__ void node_signal(const DevNet& n, int i, int a, int p, bool yellow_phase,
                                            uint32_t* open, uint32_t* major, uint32_t* ymask) {
  uint32_t g1 = __ldg(&n.node_green[i * n.max_phases + a]);
  uint32_t m1 = __ldg(&n.node_major[i * n.max_phases + a]);
  uint32_t o = g1, m = m1, y = 0;
  if (yellow_phase && p >= 0 && p != a) {
    uint32_t g0 = __ldg(&n.node_green[i * n.max_phases + p]);
    uint32_t sw_red = g0 & ~g1;
    uint32_t sw_green = ~g0 & g1;
    if (sw_red) { y = sw_red; o = g1 & ~sw_green; m = m1 & ~sw_green; }
  }
  open[i] = o; major[i] = m; ymask[i] = y;
}

// ------------------------------------------------------------------------------------------------
extern __shared__ __align__(16) unsigned char smem_raw[];

// REC = record mode: a fourth ring word per vehicle (trip word) and the arrival log; compiled out of the hot variant.
template <bool REC>
__global__ void __launch_bounds__(TSC_THREADS, TSC_MIN_BLOCKS)
tsc_step_kernel(const StepArgs A) {
  const DevNet& n = A.net;
  const tsc_cfg& c = A.cfg;
  const int tid = threadIdx.x;
  const int rep = blockIdx.x + A.rep0;
  const int L = n.n_lanes, N = n.n_nodes;

  // ---- shared-memory carve-up ----
  Ring ring;
  ring.xv = reinterpret_cast<uint32_t*>(smem_raw);
  ring.m = ring.xv + n.n_slots;
  ring.t = REC ? ring.m + n.n_slots : nullptr;
  int32_t* s_cnt = reinterpret_cast<int32_t*>(ring.m + (REC ? 2 : 1) * n.n_slots);
  int32_t* s_head = s_cnt + L;
  int32_t* s_pre = s_head + L;              // L + 1
  float* s_headlim = reinterpret_cast<float*>(s_pre + L + 1);
  int32_t* s_cntadd = reinterpret_cast<int32_t*>(s_headlim + L);
  uint8_t* s_hflag = reinterpret_cast<uint8_t*>(s_cntadd + L);
  uint8_t* s_acc = s_hflag + L;
  // 4-byte align after the two byte arrays
  int32_t* s_open = reinterpret_cast<int32_t*>(smem_raw + (((s_acc + L) - smem_raw + 3) & ~3));
  uint32_t* s_opn = reinterpret_cast<uint32_t*>(s_open);
  uint32_t* s_maj = s_opn + N;
  uint32_t* s_yel = s_maj + N;
  uint32_t* s_appr = s_yel + N;
  int32_t* s_act = reinterpret_cast<int32_t*>(s_appr + N);
  int32_t* s_prev = s_act + N;
  int32_t* s_backlog = s_prev + N;          // n_src
  int32_t* s_det = s_backlog + n.n_src;     // 3 * n_det
  float* s_loc = reinterpret_cast<float*>(s_det + 3 * n.n_det);  // N
  int32_t* s_misc = reinterpret_cast<int32_t*>(s_loc + N);         // [0..7] ctl fixed, [8..15] wsum
  int32_t* s_wsum = s_misc + 8;
  int32_t* s_blk = s_wsum + TSC_THREADS / 32;                      // lane of compact vehicle 32*j
  float* s_obsv = reinterpret_cast<float*>(s_blk + (n.n_slots + 31) / 32 + 1);   // [2*n_det] normalised wave | wait
  // static tables staged once per CTA (they sit on the dependent-load chains of every phase): lane constants and the
  // route tables (hop -> lane, hop -> link)
  LaneC* s_lane = reinterpret_cast<LaneC*>(smem_raw + ((reinterpret_cast<unsigned char*>(s_obsv + 2 * n.n_det) - smem_raw + 15) & ~15));
  int16_t* s_rlane = reinterpret_cast<int16_t*>(s_lane + L);
  int16_t* s_rlink = s_rlane + n.n_routes * n.max_hops;

  // ---- load replica state -------------------------------------------------------------------
  const uint8_t* g_cnt = A.lane_cnt + (size_t)rep * n.lpad;
  int32_t* g_ctl = A.ctl + (size_t)rep * A.ctl_words;
  uint32_t* g_x = A.veh + (size_t)rep * 2 * n.n_slots;
  uint32_t* g_m = g_x + n.n_slots;
  for (int l = tid; l < L; l += TSC_THREADS) { s_cnt[l] = g_cnt[l]; s_head[l] = 0; s_lane[l] = n.lane[l]; }
  for (int i = tid; i < n.n_routes * n.max_hops; i += TSC_THREADS) {
    s_rlane[i] = __ldg(&n.route_lane[i]); s_rlink[i] = __ldg(&n.route_link[i]);
  }
  if (tid < CTL_FIXED) s_misc[tid] = g_ctl[tid];
  for (int i = tid; i < N; i += TSC_THREADS) {
    s_prev[i] = g_ctl[CTL_FIXED + i];
    s_act[i] = A.n_sub > 0 ? A.action[(size_t)rep * N + i] : s_prev[i];
    s_appr[i] = 0;
  }
  for (int q = tid; q < n.n_src; q += TSC_THREADS) s_backlog[q] = g_ctl[CTL_FIXED + N + q];
  __syncthreads();
  block_scan(s_cnt, s_pre, s_wsum, L);
  {
    const int per0 = (L + TSC_THREADS - 1) / TSC_THREADS;
    fill_blk(s_pre, s_cnt, s_blk, tid * per0, min(L, tid * per0 + per0));
    __syncthreads();
    const int V = s_pre[L];
    for (int k0 = 0; k0 < V; k0 += TSC_THREADS) {      // warp-uniform trip count: the lane lookup uses shuffles
      const int k = k0 + tid;
      const int lane = find_lane_warp(s_pre, s_blk, L, k < V ? k : V - 1);
      if (k < V) {
        const int rank = k - s_pre[lane];
        st2(ring, s_lane[lane].slot0 + rank, make_uint2(g_x[k], g_m[k]));
        if constexpr (REC) ring.t[s_lane[lane].slot0 + rank] = A.trip[(size_t)rep * n.n_slots + k];
      }
    }
  }
  for (int i = tid; i < N; i += TSC_THREADS)
    node_signal(n, i, s_act[i], s_prev[i], A.sub0 < c.yellow_interval_sec, s_opn, s_maj, s_yel);
  __syncthreads();

  const uint32_t seed_lo = (uint32_t)s_misc[1], seed_hi = (uint32_t)s_misc[2];
  int cur_sec = s_misc[0];
  int n_dep_add = 0;  // per-thread partial (sources), reduced at the end via atomics
  const float ib = 1.0f / c.decel;

  // ---- sub-steps: each is one traci.simulationStep() (envs/env.py:461-471) -------------------
  // Lane phases use BLOCKED ownership (thread tid owns lanes [tid*per, tid*per+per)), identical in every
  // phase and in the scan, so data a thread only exchanges with itself needs no barrier:
  //   [A1 + scan part 1] | [scan part 2 + A2] | B (1 barrier per batch + 1) | C | [D + E]  -> 6 barriers.
  const int per = (L + TSC_THREADS - 1) / TSC_THREADS;
  const int l_lo = tid * per, l_hi = min(L, l_lo + per);
  for (int sub = A.sub0; sub < A.sub0 + A.n_sub; ++sub) {
    const uint32_t t_abs = (uint32_t)cur_sec;
    const uint32_t key = rng_key(seed_lo, seed_hi, t_abs);
    // A1: approach masks + reset of per-lane scratch (own lanes)
    for (int l = l_lo; l < l_hi; ++l) {
      s_hflag[l] = 0; s_acc[l] = 0; s_cntadd[l] = 0;
      if (s_cnt[l] > 0) {
        const LaneC lc = s_lane[l];
        const uint2 h = ld2(ring, lc.slot0 + s_head[l]);
        int link = (int)s_rlink[M0_ROUTE(h.y) * n.max_hops + M0_HOP(h.y)];
        if (link >= 0) {
          const LinkC* lk = &n.link[link];
          int node = __ldg(&lk->node);
          if (node >= 0) {
            uint32_t bit = 1u << __ldg(&lk->tlidx);
            float d = lc.len - veh_x(h.x);
            if ((s_opn[node] & bit) && d <= 3.0f * veh_v(h.x) + 7.5f) atomicOr(&s_appr[node], bit);
          }
        }
      }
    }
    const ScanCarry sc = scan_part1(s_cnt, s_wsum, L);
    __syncthreads();
    scan_part2(sc, s_pre, s_wsum, L);
    fill_blk(s_pre, s_cnt, s_blk, l_lo, l_hi);      // own lanes: which compact indices 32*j fall into lane l
    // A2: head-vehicle speed limit from the junction ahead (own lanes; reads other lanes' tails)
    for (int l = l_lo; l < l_hi; ++l) {
      float lim = INF_SPEED;
      if (s_cnt[l] > 0) {
        const LaneC lc = s_lane[l];
        const uint2 h = ld2(ring, lc.slot0 + s_head[l]);
        const uint32_t route = M0_ROUTE(h.y), hop = M0_HOP(h.y);
        const int link = (int)s_rlink[route * n.max_hops + hop];
        if (link >= 0) {
          const LinkC lk = n.link[link];
          const float hx = veh_x(h.x), hv = veh_v(h.x);
          const float d = lc.len - hx;
          bool blocked = false;
          if (lk.node >= 0 && (int)M0_WAIT(h.y) < c.teleport_sec) {
            const uint32_t bit = 1u << lk.tlidx;
            if (s_yel[lk.node] & bit) {
              blocked = brake_gap(hv, c.decel, ib) <= d;
            } else if (!(s_opn[lk.node] & bit)) {
              blocked = true;
            } else {
              uint32_t foes = lk.merge;
              if (!(s_maj[lk.node] & bit)) foes |= lk.cross;
              if (s_appr[lk.node] & foes) blocked = true;
            }
          }
          if (blocked) {
            lim = stop_speed(d, c.decel, ib, c.tau);
            s_hflag[l] = F_CLOSED;        // own lane; read by the lane's rank-0 vehicle thread in B after the barrier
          } else {
            if (lk.vmax < 1.0e8f) lim = free_speed(d, lk.vmax, c.decel);
            const int nl = (int)s_rlane[route * n.max_hops + hop + 1];
            const int nc = s_cnt[nl];
            if (nc > 0) {
              const LaneC nlc = s_lane[nl];
              int idx = s_head[nl] + nc - 1;
              if (idx >= nlc.cap) idx -= nlc.cap;
              const uint32_t txv = ring.xv[nlc.slot0 + idx];
              float gap = d + (veh_x(txv) - c.veh_len);
              gap = gap - c.min_gap;
              float fs = follow_speed(gap, veh_v(txv), c.decel, ib, c.tau);
              if (fs < lim) lim = fs;
            }
          }
        }
      }
      s_headlim[l] = lim;
    }
    __syncthreads();
    // B: every live vehicle plans from the OLD state, then writes (back-to-front batches so a
    //    batch never overwrites a leader that a later batch still has to read)
    {
      const int V = s_pre[L];
      const int iters = (V + TSC_THREADS - 1) / TSC_THREADS;
      for (int it = iters - 1; it >= 0; --it) {
        const int k = it * TSC_THREADS + tid;
        const bool act = k < V;
        int slot = 0, lane = 0, rank = 0;
        uint2 me = make_uint2(0, 0);
        uint8_t f = 0;
        lane = find_lane_warp(s_pre, s_blk, L, act ? k : V - 1);
        if (act) {
          rank = k - s_pre[lane];
          const LaneC lc = s_lane[lane];
          int idx = s_head[lane] + rank;
          if (idx >= lc.cap) idx -= lc.cap;
          slot = lc.slot0 + idx;
          me = ld2(ring, slot);
          const float x = veh_x(me.x), v = veh_v(me.x);
          const float sf = 0.5f + (float)M0_SFQ(me.y) * (1.0f / 256.0f);
          const float vmax = lc.vmax * sf;
          float vfree = v + c.accel;
          if (vmax < vfree) vfree = vmax;
          float vsafe;
          if (rank == 0) {
            vsafe = s_headlim[lane];
          } else {
            int lidx = idx - 1;
            if (lidx < 0) lidx += lc.cap;
            const uint32_t lxv = ring.xv[lc.slot0 + lidx];
            float gap = veh_x(lxv) - c.veh_len;
            gap = gap - x;
            gap = gap - c.min_gap;
            vsafe = follow_speed(gap, veh_v(lxv), c.decel, ib, c.tau);
          }
          const float vnm = vfree < vsafe ? vfree : vsafe;
          float vmin = v - c.decel;
          if (vmin < 0.0f) vmin = 0.0f;
          if (vnm < vmin) vmin = vnm;
          const float u = u01(rng_draw(key, (uint32_t)lane, (uint32_t)rank));
          const float basev = vnm < c.accel ? vnm : c.accel;
          const float vd = vnm - (c.sigma * basev) * u;
          float vn = vd > vmin ? vd : vmin;
          float xn = x + vn;
          if (xn >= lc.len) {
            // a head vehicle whose stop line is closed never passes it (tau < 1 s makes the Euler stop speed
            // overshoot: SUMO's "emergency stop at the end of the lane"); followers: one discharge per lane and second
            if (rank == 0 && s_hflag[lane] != F_CLOSED) {
              int link = (int)s_rlink[M0_ROUTE(me.y) * n.max_hops + M0_HOP(me.y)];
              f = link < 0 ? F_ARRIVE : F_CROSS;
            } else {
              xn = lc.len - 0.01f;
              vn = xn - x;
              if (vn < 0.0f) { vn = 0.0f; xn = x; }
            }
          }
          uint32_t w = M0_WAIT(me.y);
          if constexpr (REC) {      // tripinfo waitingTime / waitingCount (envs/env.py:498-515)
            if (vn < 0.1f) {
              uint32_t t1 = ring.t[slot];
              uint32_t wt = T1_WAIT(t1), wc = T1_WCNT(t1);
              if (wt < 4095u) wt++;
              if (w == 0 && wc < 255u) wc++;
              ring.t[slot] = T1_DEPART(t1) | (wt << 12) | (wc << 24);     // own slot: nobody else reads the trip word
            }
          }
          if (vn < 0.1f) {
            if (w < 1023u) w++;
          } else {
            w = 0;
          }
          me.x = pack_xv(xn, vn);       // waiting was decided on the computed speed; the record stores it rounded
          me.y = (me.y & ~1023u) | w;
        }
        __syncthreads();
        if (act) {
          st2(ring, slot, me);
          if (rank == 0) s_hflag[lane] = f;
        }
      }
      __syncthreads();
    }
    // C: junction transfers — the owner of each destination lane pulls from its source lanes in
    //    merge-priority order (no atomics).  Also: clear approach masks, switch yellow -> green.
    for (int t = l_lo; t < l_hi; ++t) {
      const int q0 = __ldg(&n.lane_inl_off[t]), q1 = __ldg(&n.lane_inl_off[t + 1]);
      if (q0 == q1) continue;
      const LaneC tc = s_lane[t];
      int cur = s_cnt[t];
      bool have_tail = cur > 0;
      float tail_x = 0.0f;
      if (have_tail) {
        int idx = s_head[t] + cur - 1;
        if (idx >= tc.cap) idx -= tc.cap;
        tail_x = veh_x(ring.xv[tc.slot0 + idx]);
      }
      for (int q = q0; q < q1; ++q) {
        const int link = __ldg(&n.lane_inl[q]);
        const int src = __ldg(&n.link[link].from);
        if (s_cnt[src] == 0 || s_hflag[src] != F_CROSS) continue;
        const LaneC sc2 = s_lane[src];
        const uint2 h = ld2(ring, sc2.slot0 + s_head[src]);
        const uint32_t route = M0_ROUTE(h.y), hop = M0_HOP(h.y);
        if ((int)s_rlink[route * n.max_hops + hop] != link) continue;
        if ((int)s_rlane[route * n.max_hops + hop + 1] != t) continue;
        if (cur >= tc.cap) continue;
        float x = veh_x(h.x) - sc2.len;
        if (have_tail) {
          float lim = tail_x - c.veh_len;
          lim = lim - c.min_gap;
          if (x > lim) x = lim;
        }
        if (x < 0.0f) continue;
        int idx = s_head[t] + cur;
        if (idx >= tc.cap) idx -= tc.cap;
        uint2 e;
        e.x = pack_xv(x, veh_v(h.x));
        e.y = (h.y & ~(63u << 10)) | ((hop + 1) << 10);
        st2(ring, tc.slot0 + idx, e);
        if constexpr (REC) ring.t[tc.slot0 + idx] = ring.t[sc2.slot0 + s_head[src]];
        cur++; tail_x = veh_x(e.x); have_tail = true;   // the next source sees the stored (truncated) position
        s_acc[src] = 1;
      }
      s_cntadd[t] = cur - s_cnt[t];
    }
    for (int i = tid; i < N; i += TSC_THREADS) {
      s_appr[i] = 0;
      // green part starts after the yellow sub-steps (envs/env.py:571-573)
      if (sub + 1 == c.yellow_interval_sec) node_signal(n, i, s_act[i], s_prev[i], false, s_opn, s_maj, s_yel);
    }
    __syncthreads();
    // D + E (own lanes only, so no barrier in between and none before the next A1):
    // D pops / arrivals / refused crossings; E insertion (departPos random_free restated on the free
    // tail segment; at most one insertion per lane per second, lowest source index first)
    for (int l = l_lo; l < l_hi; ++l) {
      int cl = s_cnt[l];
      const LaneC lc = s_lane[l];
      if (cl > 0) {
        const uint8_t f = s_hflag[l];
        bool pop = false;
        if (f == F_ARRIVE) {
          pop = true; atomicAdd(&s_misc[4], 1);
          if constexpr (REC) {      // one tripinfo row
            const int slot_h = lc.slot0 + s_head[l];
            const uint32_t t1 = ring.t[slot_h], m0 = ring.m[slot_h];
            const int at = atomicAdd(&s_misc[5], 1);
            if (at < A.trip_cap) {
              uint32_t* row = A.trip_log + ((size_t)rep * A.trip_cap + at) * 2;
              row[0] = T1_DEPART(t1) | (((uint32_t)(cur_sec + 1) & 4095u) << 12) | (M0_ROUTE(m0) << 24);
              row[1] = T1_WAIT(t1) | (T1_WCNT(t1) << 16);
            }
          }
        }
        else if (f == F_CROSS) {
          if (s_acc[l]) pop = true;
          else {
            ring.xv[lc.slot0 + s_head[l]] = pack_xv(lc.len - 0.01f, 0.0f);
          }
        }
        if (pop) {
          int hd = s_head[l] + 1;
          if (hd >= lc.cap) hd = 0;
          s_head[l] = hd;
          cl--;
        }
      }
      cl += s_cntadd[l];
      int q = __ldg(&n.lane_src0[l]);
      if (q >= 0) {
        const bool in_h = (int)t_abs < n.horizon;
        bool lane_free = true;   // the lane belongs to the first source (by index) with a backlog
        int pick = -1;
        if (n.src_group) {
          // stochastic demand: first update every backlog of the lane with this second's draws, then the lane goes to
          // the source with the LONGEST backlog (ties: lowest index), which keeps the realised route shares at the
          // turn ratios when the entry lane saturates (a fixed order would starve the later siblings)
          int best = 0;
          for (int q2 = q; q2 >= 0; q2 = __ldg(&n.src_next[q2])) {
            int due = in_h ? (int)__ldg(&n.src_due[t_abs * n.n_src + q2]) : 0;
            const int gq = __ldg(&n.src_group[q2]);
            if (gq >= 0 && due > 0) {
              const float ug = u01(rng_draw(key, 0x20000u + (uint32_t)gq, 7u));
              int iv = (int)t_abs / n.pint_sec;
              if (iv >= n.n_pint) iv = n.n_pint - 1;
              if (!(ug >= __ldg(&n.src_plo[iv * n.n_src + q2]) && ug < __ldg(&n.src_phi[iv * n.n_src + q2]))) due = 0;
            }
            int b2 = s_backlog[q2] + due;
            if (b2 > 65535) b2 = 65535;
            s_backlog[q2] = b2;
            if (b2 > best) { best = b2; pick = q2; }
          }
        }
        for (; q >= 0; q = __ldg(&n.src_next[q])) {
          int b_new = n.src_group ? s_backlog[q] : s_backlog[q] + (in_h ? (int)__ldg(&n.src_due[t_abs * n.n_src + q]) : 0);
          if (b_new > 65535) b_new = 65535;
          if (n.src_group ? (q == pick) : (b_new > 0 && lane_free)) {
            lane_free = false;
            bool ok = cl < lc.cap;
            float free_back = lc.len;
            if (ok && cl > 0) {
              int idx = s_head[l] + cl - 1;
              if (idx >= lc.cap) idx -= lc.cap;
              free_back = veh_x(ring.xv[lc.slot0 + idx]) - c.veh_len;
              free_back = free_back - c.min_gap;
            }
            if (ok && !(free_back < c.veh_len)) {
              const uint32_t qq = (uint32_t)q;
              const float u = u01(rng_draw(key, qq, (1u << 16)));
              const float pos = c.veh_len + u * (free_back - c.veh_len);
              float su = 0.0f;
              for (uint32_t j = 1; j <= 4; ++j) su = su + u01(rng_draw(key, qq, (1u << 16) | j));
              const float sfr = 1.0f + (c.speed_dev * 1.7320508f) * (su - 2.0f);
              int sfq = (int)((sfr - 0.5f) * 256.0f);
              if (sfq < 0) sfq = 0;
              if (sfq > 255) sfq = 255;
              int idx = s_head[l] + cl;
              if (idx >= lc.cap) idx -= lc.cap;
              uint2 e;
              e.x = pack_xv(pos, 0.0f);
              e.y = ((uint32_t)__ldg(&n.src_route[q]) << 16) | ((uint32_t)sfq << 24);
              st2(ring, lc.slot0 + idx, e);
              if constexpr (REC) ring.t[lc.slot0 + idx] = (uint32_t)t_abs & 4095u;      // depart second
              cl++;
              b_new--;
              n_dep_add++;
            }
          }
          s_backlog[q] = b_new;
        }
      }
      s_cnt[l] = cl;
    }
    cur_sec++;
  }
  __syncthreads();
  if (n_dep_add) atomicAdd(&s_misc[3], n_dep_add);

  // ---- detector reads (envs/env.py:325-407): one thread per detector lane ---------------------
  for (int d = tid; d < n.n_det; d += TSC_THREADS) {
    const int l = __ldg(&n.det_lane[d]);
    const LaneC lc = s_lane[l];
    int veh = 0, halt = 0, wait = 0;
    const int cl = s_cnt[l];
    int idx = s_head[l];
    for (int k = 0; k < cl; ++k) {
      const uint2 v = ld2(ring, lc.slot0 + idx);
      const float x = veh_x(v.x);
      if (c.det_len > 0.0f && !(x > lc.len - c.det_len)) break;
      veh++;
      if (veh_v(v.x) < c.halt_speed) halt++;
      if (k == 0 && x > 0.0f) wait = (int)M0_WAIT(v.y);
      if (++idx >= lc.cap) idx = 0;
    }
    s_det[d] = veh; s_det[n.n_det + d] = halt; s_det[2 * n.n_det + d] = wait;
  }
  __syncthreads();
  // local rewards
  for (int i = tid; i < N; i += TSC_THREADS) {
    int queue = 0, wait = 0;
    for (int d = __ldg(&n.node_det_off[i]); d < __ldg(&n.node_det_off[i + 1]); ++d) {
      int h = s_det[n.n_det + d];
      if (h > c.queue_cap) h = c.queue_cap;
      queue += h; wait += s_det[2 * n.n_det + d];
    }
    float rw;
    if (c.objective == 0) rw = -(float)queue;
    else if (c.objective == 1) rw = -(float)wait;
    else rw = -(float)queue - c.coef_wait * (float)wait;
    s_loc[i] = rw;
  }
  __syncthreads();
  if (A.n_sub > 0) {
    float g = 0.0f;   // every thread that needs it recomputes the same sequential sum
    const int mode = A.train_mode ? c.agent_mode : 0;
    if (tid < N || tid == TSC_THREADS - 1) {
      if (mode == 1 || tid == TSC_THREADS - 1)
        for (int i = 0; i < N; ++i) g = g + s_loc[i];
    }
    if (tid == TSC_THREADS - 1) {
      if (A.greward) A.greward[rep] = g;
      if (A.done) A.done[rep] = cur_sec >= c.episode_length_sec;
    }
    if (A.reward)
      for (int i = tid; i < N; i += TSC_THREADS) {
        float rw;
        if (mode == 0) rw = s_loc[i];
        else if (mode == 1) {
          rw = g;
          if (c.real_net_norm) rw = rw / ((float)N * 20.0f);
        } else {
          rw = s_loc[i];
          const int q0 = __ldg(&n.node_nbr_off[i]), q1 = __ldg(&n.node_nbr_off[i + 1]);
          const float cg = A.cg ? __ldg(&A.cg[rep]) : c.coop_gamma;
          for (int q = q0; q < q1; ++q) rw = rw + cg * s_loc[__ldg(&n.node_nbr[q])];
          if (c.real_net_norm) rw = rw / ((float)(1 + q1 - q0) * 20.0f);
        }
        A.reward[(size_t)rep * N + i] = rw;
      }
  }
  // observation gather (envs/env.py:163-205), coalesced row write
  if (A.obs) {
    for (int dd = tid; dd < n.n_det; dd += TSC_THREADS) {
      s_obsv[dd] = clipf((float)s_det[dd] / c.norm_wave, c.clip_wave);
      s_obsv[n.n_det + dd] = clipf((float)s_det[2 * n.n_det + dd] / c.norm_wait, c.clip_wait);
    }
    __syncthreads();
    const float* fp = A.fp ? A.fp + (size_t)rep * N * n.max_na : nullptr;
    float* o = A.obs + (size_t)rep * n.n_obs;
    const float sv = A.cg ? __ldg(&A.cg[rep]) : n.obs_scale_val;
    for (int k = tid; k < n.n_obs; k += TSC_THREADS) {
      const uint32_t pw = __ldg(&n.obs_prog[k]);
      const int kind = (int)(pw & 3u), idx = (int)(pw >> 3);
      float v;
      if (kind == 0) v = s_obsv[idx];
      else if (kind == 1) v = s_obsv[n.n_det + idx];
      else v = fp ? fp[idx] : 0.0f;
      o[k] = ((pw & 4u) ? sv : 1.0f) * v;      // same product as obs_scale[k] * v
    }
  }
  if (A.n_sub == 0) return;  // observe only: state untouched

  // ---- store replica state (compact) + parity taps --------------------------------------------
  block_scan(s_cnt, s_pre, s_wsum, L);
  {
    fill_blk(s_pre, s_cnt, s_blk, l_lo, l_hi);
    __syncthreads();
    const int V = s_pre[L];
    for (int k0 = 0; k0 < V; k0 += TSC_THREADS) {
      const int k = k0 + tid;
      const int lane = find_lane_warp(s_pre, s_blk, L, k < V ? k : V - 1);
      if (k < V) {
        const int rank = k - s_pre[lane];
        const LaneC lc = s_lane[lane];
        int idx = s_head[lane] + rank;
        if (idx >= lc.cap) idx -= lc.cap;
        const uint2 e = ld2(ring, lc.slot0 + idx);
        g_x[k] = e.x; g_m[k] = e.y;
        if constexpr (REC) A.trip[(size_t)rep * n.n_slots + k] = ring.t[lc.slot0 + idx];
      }
    }
  }
  uint8_t* g_cnt_w = A.lane_cnt + (size_t)rep * n.lpad;
  for (int l = tid; l < L; l += TSC_THREADS) g_cnt_w[l] = (uint8_t)s_cnt[l];
  if (tid == 0) {
    g_ctl[0] = cur_sec; g_ctl[3] = s_misc[3]; g_ctl[4] = s_misc[4];
    if constexpr (REC) { g_ctl[5] = s_misc[5]; A.trip_cnt[rep] = s_misc[5] < A.trip_cap ? s_misc[5] : A.trip_cap; }
  }
  if (A.sub0 + A.n_sub >= c.control_interval_sec)      // the interval is complete: prev_action = action
    for (int i = tid; i < N; i += TSC_THREADS) g_ctl[CTL_FIXED + i] = s_act[i];
  for (int q = tid; q < n.n_src; q += TSC_THREADS) g_ctl[CTL_FIXED + N + q] = s_backlog[q];
  if (A.meas) {
    int32_t* m = A.meas + (size_t)rep * (3 * n.n_det + N);
    for (int d = tid; d < 3 * n.n_det; d += TSC_THREADS) m[d] = s_det[d];
    for (int i = tid; i < N; i += TSC_THREADS) m[3 * n.n_det + i] = s_act[i];
  }
}

// reset(): envs/env.py:544-561
__global__ void tsc_reset_kernel(uint8_t* lane_cnt, int32_t* ctl, int32_t* meas, const uint64_t* seeds,
                                 int lpad, int ctl_words, int meas_words, int R) {
  const int rep = blockIdx.x;
  if (rep >= R) return;
  for (int l = threadIdx.x; l < lpad; l += blockDim.x) lane_cnt[(size_t)rep * lpad + l] = 0;
  for (int w = threadIdx.x; w < ctl_words; w += blockDim.x) {
    int32_t v = 0;
    if (w == 1) v = (int32_t)(uint32_t)(seeds[rep] & 0xffffffffull);
    if (w == 2) v = (int32_t)(uint32_t)(seeds[rep] >> 32);
    ctl[(size_t)rep * ctl_words + w] = v;
  }
  for (int w = threadIdx.x; w < meas_words; w += blockDim.x) meas[(size_t)rep * meas_words + w] = 0;
}

// _measure_traffic_step (envs/env.py:409-437) for every replica: one CTA per replica over the compact state.
// stats[r] = {n_live, n_departed_total, n_arrived_total, avg_wait, avg_speed, avg_queue, std_queue, backlog}
// avg/std_queue: lane halting number (speed < 0.1 m/s, whole lane) over the detector lanes (envs/env.py:422-427).
__global__ void tsc_stats_kernel(const DevNet n, const uint32_t* __restrict__ veh, const uint8_t* __restrict__ lane_cnt,
                                 const int32_t* __restrict__ ctl, int ctl_words, float* __restrict__ stats,
                                 int row_stride) {
  extern __shared__ int32_t sh[];
  int32_t* s_pre = sh;                 // [L + 1]
  int32_t* s_halt = sh + n.n_lanes + 1; // [L]
  __shared__ float red[3];
  const int rep = blockIdx.x, tid = threadIdx.x, L = n.n_lanes;
  const uint8_t* cnt = lane_cnt + (size_t)rep * n.lpad;
  if (tid == 0) {
    int s = 0;
    for (int l = 0; l < L; ++l) { s_pre[l] = s; s += cnt[l]; }
    s_pre[L] = s;
    red[0] = red[1] = 0.f;
  }
  for (int l = tid; l < L; l += blockDim.x) s_halt[l] = 0;
  __syncthreads();
  const int V = s_pre[L];
  float w = 0.f, sp = 0.f;
  for (int k = tid; k < V; k += blockDim.x) {
    const float vy = veh_v(veh[((size_t)rep * 2 + 0) * n.n_slots + k]);
    w += (float)(veh[((size_t)rep * 2 + 1) * n.n_slots + k] & 1023u);
    sp += vy;
    if (vy < 0.1f) {
      int lo = 0, hi = L;
      while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (s_pre[mid] <= k) lo = mid; else hi = mid; }
      atomicAdd(&s_halt[lo], 1);
    }
  }
  atomicAdd(&red[0], w); atomicAdd(&red[1], sp);
  __syncthreads();
  if (tid == 0) {
    const int32_t* c = ctl + (size_t)rep * ctl_words;
    float q = 0.f, q2 = 0.f;
    for (int d = 0; d < n.n_det; ++d) { const float h = (float)s_halt[n.det_lane[d]]; q += h; q2 += h * h; }
    const float nd = (float)(n.n_det > 0 ? n.n_det : 1);
    const float mq = q / nd;
    float var = q2 / nd - mq * mq;
    if (var < 0.f) var = 0.f;
    int backlog = 0;
    for (int s2 = 0; s2 < n.n_src; ++s2) backlog += c[CTL_FIXED + n.n_nodes + s2];
    float* o = stats + (size_t)rep * row_stride;
    o[0] = (float)V; o[1] = (float)c[3]; o[2] = (float)c[4];
    o[3] = V > 0 ? red[0] / (float)V : 0.f; o[4] = V > 0 ? red[1] / (float)V : 0.f;
    o[5] = mq; o[6] = sqrtf(var); o[7] = (float)backlog;
  }
}

__global__ void tsc_live_kernel(const uint8_t* lane_cnt, int lpad, int L, int R, unsigned long long* out) {
  unsigned long long s = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)R * lpad; i += (size_t)gridDim.x * blockDim.x)
    if ((int)(i % lpad) < L) s += lane_cnt[i];
  for (int o = 16; o; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(out, s);
}

// ================================================================================================
// host side: C ABI
// ================================================================================================
static thread_local std::string g_err;
static int fail(const std::string& m) { g_err = m; return -1; }
int tsc_set_error(const std::string& m) { return fail(m); }   // shared with tsc_learn.cu
#define CK(call)                                                                      \
  do {                                                                                \
    cudaError_t e__ = (call);                                                         \
    if (e__ != cudaSuccess)                                                           \
      return fail(std::string(#call) + ": " + cudaGetErrorString(e__));               \
  } while (0)

struct tsc_handle {
  int device = 0;
  int R = 0;
  StepArgs args{};
  int smem = 0, smem_rec = 0;
  bool record = false;       // record mode (tsc_set_record): trip words + arrival log, one simulated second per launch
  uint32_t* d_trip = nullptr; uint32_t* d_trip_log = nullptr; int32_t* d_trip_cnt = nullptr; int trip_cap = 0;
  std::vector<void*> owned;  // device allocations
  // io scratch for the host-buffer entry point
  int32_t* d_action = nullptr; float* d_fp = nullptr; float* d_obs = nullptr; float* d_reward = nullptr;
  float* d_greward = nullptr; uint8_t* d_done = nullptr;
  unsigned long long* d_scalar = nullptr;
  float* d_cg = nullptr;     // per-replica coop_gamma (tsc_set_replica_coop_gamma), allocated on first use
  int n_nodes = 0, n_obs = 0, max_na = 0, n_det = 0;
  int meas_words = 0;
  // greedy program (tsc_set_greedy_program): CSR over (node, candidate) of observation offsets + action per candidate
  int gp_max_cand = 0;
  int32_t* d_gp_off = nullptr; int32_t* d_gp_idx = nullptr; int32_t* d_gp_act = nullptr;
};

template <class T>
static int upload(tsc_handle* h, const T* src, size_t count, const T** dst) {
  void* p = nullptr;
  CK(cudaMalloc(&p, count ? count * sizeof(T) : 16));
  if (count) CK(cudaMemcpy(p, src, count * sizeof(T), cudaMemcpyHostToDevice));
  h->owned.push_back(p);
  *dst = static_cast<const T*>(p);
  return 0;
}
template <class T>
static int dalloc(tsc_handle* h, size_t count, T** dst) {
  void* p = nullptr;
  CK(cudaMalloc(&p, count ? count * sizeof(T) : 16));
  CK(cudaMemset(p, 0, count ? count * sizeof(T) : 16));
  h->owned.push_back(p);
  *dst = static_cast<T*>(p);
  return 0;
}

extern "C" const char* tsc_last_error(void) { return g_err.c_str(); }

extern "C" int tsc_create(const tsc_net* net, const tsc_cfg* cfg, int32_t R, int32_t device, tsc_handle** out) {
  if (!net || !cfg || !out || R <= 0) return fail("tsc_create: bad argument");
  if (net->n_lanes > 4 * TSC_THREADS) return fail("tsc_create: too many lanes for one CTA");
  if (net->n_nodes > TSC_THREADS - 1) return fail("tsc_create: too many nodes");
  if (net->n_src > TSC_THREADS) return fail("tsc_create: too many demand sources");
  if (net->max_hops > 63 || net->n_routes > 255) return fail("tsc_create: route table too large");
  for (int l = 0; l < net->n_lanes; ++l) {
    if (net->lane_cap[l] > 255) return fail("tsc_create: lane capacity > 255");
    // fixed-point vehicle records: 16-bit position in 1/64 m (a crossing vehicle may overshoot by one step's travel),
    // 16-bit speed in 1/1024 m/s; speedFactor <= 1.5
    if (net->lane_len[l] + 64.0f > 1023.0f) return fail("tsc_create: lane longer than 959 m (16-bit position field)");
    if (net->lane_vmax[l] * 1.5f > 63.9f) return fail("tsc_create: lane speed limit above 42 m/s (16-bit speed field)");
  }
  CK(cudaSetDevice(device));
  tsc_handle* h = new tsc_handle();
  h->device = device; h->R = R;
  DevNet& d = h->args.net;
  d.n_lanes = net->n_lanes; d.n_links = net->n_links; d.n_nodes = net->n_nodes; d.n_routes = net->n_routes;
  d.max_hops = net->max_hops; d.n_src = net->n_src; d.horizon = net->horizon; d.n_det = net->n_det;
  d.n_obs = net->n_obs; d.max_phases = net->max_phases; d.max_na = net->max_na; d.n_slots = net->n_slots;
  d.lpad = (net->n_lanes + 15) & ~15;
  d.src_shared = 0;
  for (int q = 0; q < net->n_src; ++q)
    for (int p = 0; p < q; ++p)
      if (net->src_lane[p] == net->src_lane[q]) d.src_shared = 1;
  std::vector<LaneC> lanes(net->n_lanes);
  for (int l = 0; l < net->n_lanes; ++l)
    lanes[l] = LaneC{net->lane_len[l], net->lane_vmax[l], net->lane_slot0[l], net->lane_cap[l]};
  std::vector<LinkC> links(net->n_links);
  for (int k = 0; k < net->n_links; ++k)
    links[k] = LinkC{net->link_from[k], net->link_node[k], net->link_tlidx[k], net->link_vmax[k],
                     net->link_cross[k], net->link_merge[k], 0, 0};
  int rc = 0;
  const int L = net->n_lanes, N = net->n_nodes;
  rc |= upload(h, lanes.data(), lanes.size(), &d.lane);
  rc |= upload(h, links.data(), links.size(), &d.link);
  rc |= upload(h, net->lane_inl_off, (size_t)L + 1, &d.lane_inl_off);
  rc |= upload(h, net->lane_inl, (size_t)net->lane_inl_off[L], &d.lane_inl);
  rc |= upload(h, net->route_lane, (size_t)net->n_routes * net->max_hops, &d.route_lane);
  rc |= upload(h, net->route_link, (size_t)net->n_routes * net->max_hops, &d.route_link);
  rc |= upload(h, net->node_green, (size_t)N * net->max_phases, &d.node_green);
  rc |= upload(h, net->node_major, (size_t)N * net->max_phases, &d.node_major);
  rc |= upload(h, net->node_det_off, (size_t)N + 1, &d.node_det_off);
  rc |= upload(h, net->det_lane, (size_t)net->n_det, &d.det_lane);
  rc |= upload(h, net->node_nbr_off, (size_t)N + 1, &d.node_nbr_off);
  rc |= upload(h, net->node_nbr, (size_t)net->node_nbr_off[N], &d.node_nbr);
  rc |= upload(h, net->obs_kind, (size_t)net->n_obs, &d.obs_kind);
  rc |= upload(h, net->obs_idx, (size_t)net->n_obs, &d.obs_idx);
  rc |= upload(h, net->obs_scale, (size_t)net->n_obs, &d.obs_scale);
  {
    std::vector<uint32_t> prog(net->n_obs > 0 ? net->n_obs : 1, 0u);
    float sv = 1.0f;
    for (int k = 0; k < net->n_obs; ++k)
      if (net->obs_scale[k] != 1.0f) sv = net->obs_scale[k];
    for (int k = 0; k < net->n_obs; ++k) {
      const float sc = net->obs_scale[k];
      if (sc != 1.0f && sc != sv) { tsc_destroy(h); return fail("tsc_create: more than one non-unit observation scale"); }
      prog[k] = (uint32_t)(net->obs_kind[k] & 3) | (sc != 1.0f ? 4u : 0u) | ((uint32_t)net->obs_idx[k] << 3);
    }
    d.obs_scale_val = sv;
    rc |= upload(h, prog.data(), prog.size(), &d.obs_prog);
  }
  rc |= upload(h, net->src_lane, (size_t)net->n_src, &d.src_lane);
  rc |= upload(h, net->src_route, (size_t)net->n_src, &d.src_route);
  rc |= upload(h, net->src_due, (size_t)net->horizon * net->n_src, &d.src_due);
  d.src_group = nullptr; d.src_plo = d.src_phi = nullptr; d.n_pint = 0; d.pint_sec = 1;
  if (net->src_group && net->n_pint > 0 && net->pint_sec > 0) {
    rc |= upload(h, net->src_group, (size_t)net->n_src, &d.src_group);
    rc |= upload(h, net->src_plo, (size_t)net->n_pint * net->n_src, &d.src_plo);
    rc |= upload(h, net->src_phi, (size_t)net->n_pint * net->n_src, &d.src_phi);
    d.n_pint = net->n_pint; d.pint_sec = net->pint_sec;
  }
  {
    std::vector<int32_t> lane_src0(net->n_lanes, -1), src_next(net->n_src > 0 ? net->n_src : 1, -1);
    for (int q = net->n_src - 1; q >= 0; --q) {      // descending, so the lists come out in ascending index order
      src_next[q] = lane_src0[net->src_lane[q]];
      lane_src0[net->src_lane[q]] = q;
    }
    rc |= upload(h, lane_src0.data(), lane_src0.size(), &d.lane_src0);
    rc |= upload(h, src_next.data(), src_next.size(), &d.src_next);
  }
  h->args.cfg = *cfg;
  h->args.ctl_words = (CTL_FIXED + N + net->n_src + 3) & ~3;
  h->meas_words = 3 * net->n_det + N;
  h->n_nodes = N; h->n_obs = net->n_obs; h->max_na = net->max_na; h->n_det = net->n_det;
  rc |= dalloc(h, (size_t)R * 2 * net->n_slots, &h->args.veh);
  rc |= dalloc(h, (size_t)R * d.lpad, &h->args.lane_cnt);
  rc |= dalloc(h, (size_t)R * h->args.ctl_words, &h->args.ctl);
  rc |= dalloc(h, (size_t)R * h->meas_words, &h->args.meas);
  rc |= dalloc(h, (size_t)R * N, &h->d_action);
  rc |= dalloc(h, (size_t)R * N * net->max_na, &h->d_fp);
  rc |= dalloc(h, (size_t)R * net->n_obs, &h->d_obs);
  rc |= dalloc(h, (size_t)R * N, &h->d_reward);
  rc |= dalloc(h, (size_t)R, &h->d_greward);
  rc |= dalloc(h, (size_t)R, &h->d_done);
  rc |= dalloc(h, 2, &h->d_scalar);
  if (rc) { tsc_destroy(h); return -1; }
  h->args.train_mode = 1;
  // shared memory: must mirror the carve-up in the kernel
  size_t sm = (size_t)net->n_slots * 8;
  sm += (size_t)L * 4 * 2 + ((size_t)L + 1) * 4 + (size_t)L * 4 * 2 + (size_t)L * 2;
  sm = (sm + 3) & ~(size_t)3;
  sm += (size_t)N * 4 * 6 + (size_t)net->n_src * 4 + (size_t)net->n_det * 12 + (size_t)N * 4 + (8 + TSC_THREADS / 32) * 4 +
        ((size_t)(net->n_slots + 31) / 32 + 1) * 4 + (size_t)net->n_det * 8;
  sm = (sm + 15) & ~(size_t)15;
  sm += (size_t)L * sizeof(LaneC) + (size_t)net->n_routes * net->max_hops * 2 * 2;
  h->smem = (int)sm + 16;
  if (sm > 227 * 1024) { tsc_destroy(h); return fail("tsc_create: replica state exceeds 227 KB of shared memory"); }
  CK(cudaFuncSetAttribute(tsc_step_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem));
  h->smem_rec = h->smem + (int)net->n_slots * 4 + 16;   // + slack: the 16-byte alignment of the table block can shift
  if (h->smem_rec <= 232448)
    CK(cudaFuncSetAttribute(tsc_step_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_rec));
  std::vector<uint64_t> seeds(R, 0);
  *out = h;
  return tsc_reset(h, seeds.data(), nullptr);
}

extern "C" int tsc_destroy(tsc_handle* h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  for (void* p : h->owned) cudaFree(p);
  cudaFree(h->d_gp_off); cudaFree(h->d_gp_idx); cudaFree(h->d_gp_act);
  delete h;
  return 0;
}

extern "C" int tsc_reset(tsc_handle* h, const uint64_t* seeds_host, void* stream) {
  if (!h || !seeds_host) return fail("tsc_reset: bad argument");
  CK(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  uint64_t* d_seeds = nullptr;
  CK(cudaMalloc(&d_seeds, sizeof(uint64_t) * h->R));
  CK(cudaMemcpyAsync(d_seeds, seeds_host, sizeof(uint64_t) * h->R, cudaMemcpyHostToDevice, st));
  tsc_reset_kernel<<<h->R, 64, 0, st>>>(h->args.lane_cnt, h->args.ctl, h->args.meas, d_seeds, h->args.net.lpad,
                                        h->args.ctl_words, h->meas_words, h->R);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(st));
  CK(cudaFree(d_seeds));
  return 0;
}

extern "C" int tsc_set_train_mode(tsc_handle* h, int32_t m) {
  if (!h) return fail("tsc_set_train_mode: null handle");
  h->args.train_mode = m ? 1 : 0;
  return 0;
}

extern "C" int tsc_set_replica_coop_gamma(tsc_handle* h, const float* cg_host) {
  if (!h) return fail("tsc_set_replica_coop_gamma: null handle");
  if (!cg_host) { h->args.cg = nullptr; return 0; }
  CK(cudaSetDevice(h->device));
  if (!h->d_cg && dalloc(h, (size_t)h->R, &h->d_cg)) return -1;
  CK(cudaDeviceSynchronize());          // no launch in flight still reads the previous values
  CK(cudaMemcpy(h->d_cg, cg_host, (size_t)h->R * 4, cudaMemcpyHostToDevice));
  h->args.cg = h->d_cg;
  return 0;
}

static int launch(tsc_handle* h, int n_sub, const int32_t* action, const float* fp, float* obs, float* reward,
                  float* greward, uint8_t* done, cudaStream_t st, int rep0 = 0, int count = -1, int sub0 = 0) {
  StepArgs a = h->args;
  a.n_sub = n_sub; a.action = action; a.fp = fp; a.obs = obs; a.reward = reward; a.greward = greward; a.done = done;
  a.rep0 = rep0;
  if (h->record) {
    a.trip = h->d_trip; a.trip_log = h->d_trip_log; a.trip_cnt = h->d_trip_cnt; a.trip_cap = h->trip_cap;
    a.sub0 = sub0;
    tsc_step_kernel<true><<<count < 0 ? h->R : count, TSC_THREADS, h->smem_rec, st>>>(a);
  } else {
    a.sub0 = sub0;
    tsc_step_kernel<false><<<count < 0 ? h->R : count, TSC_THREADS, h->smem, st>>>(a);
  }
  CK(cudaGetLastError());
  return 0;
}

extern "C" int tsc_observe(tsc_handle* h, const float* fp_dev, float* obs_dev, void* stream) {
  if (!h || !obs_dev) return fail("tsc_observe: bad argument");
  CK(cudaSetDevice(h->device));
  return launch(h, 0, nullptr, fp_dev, obs_dev, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}

extern "C" int tsc_step(tsc_handle* h, const int32_t* action_dev, const float* fp_dev, float* obs_dev,
                        float* reward_dev, float* greward_dev, uint8_t* done_dev, void* stream) {
  if (!h || !action_dev) return fail("tsc_step: bad argument");
  CK(cudaSetDevice(h->device));
  return launch(h, h->args.cfg.control_interval_sec, action_dev, fp_dev, obs_dev, reward_dev, greward_dev, done_dev,
                (cudaStream_t)stream);
}

extern "C" int tsc_step_host(tsc_handle* h, const int32_t* action_host, const float* fp_host, float* obs_host,
                             float* reward_host, float* greward_host, uint8_t* done_host, void* stream) {
  if (!h || !action_host) return fail("tsc_step_host: bad argument");
  CK(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t R = h->R, N = h->n_nodes;
  CK(cudaMemcpyAsync(h->d_action, action_host, R * N * 4, cudaMemcpyHostToDevice, st));
  if (fp_host) CK(cudaMemcpyAsync(h->d_fp, fp_host, R * N * h->max_na * 4, cudaMemcpyHostToDevice, st));
  if (launch(h, h->args.cfg.control_interval_sec, h->d_action, fp_host ? h->d_fp : nullptr, obs_host ? h->d_obs : nullptr,
             reward_host ? h->d_reward : nullptr, greward_host ? h->d_greward : nullptr,
             done_host ? h->d_done : nullptr, st))
    return -1;
  if (obs_host) CK(cudaMemcpyAsync(obs_host, h->d_obs, R * h->n_obs * 4, cudaMemcpyDeviceToHost, st));
  if (reward_host) CK(cudaMemcpyAsync(reward_host, h->d_reward, R * N * 4, cudaMemcpyDeviceToHost, st));
  if (greward_host) CK(cudaMemcpyAsync(greward_host, h->d_greward, R * 4, cudaMemcpyDeviceToHost, st));
  if (done_host) CK(cudaMemcpyAsync(done_host, h->d_done, R, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}

static int step_host_range(tsc_handle* h, int32_t rep0, int32_t count, const int32_t* action_host,
                           const float* fp_host, float* obs_host, float* reward_host, float* greward_host,
                           uint8_t* done_host, void* stream, bool sync) {
  if (!h || !action_host || rep0 < 0 || count <= 0 || rep0 + count > h->R) return fail("tsc_step_host_range: bad argument");
  CK(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t N = h->n_nodes, r0 = (size_t)rep0, n = (size_t)count;
  // the kernel indexes its io arrays by absolute replica: device scratch is used at offset rep0, host pointers are slice bases
  CK(cudaMemcpyAsync(h->d_action + r0 * N, action_host, n * N * 4, cudaMemcpyHostToDevice, st));
  if (fp_host) CK(cudaMemcpyAsync(h->d_fp + r0 * N * h->max_na, fp_host, n * N * h->max_na * 4, cudaMemcpyHostToDevice, st));
  if (launch(h, h->args.cfg.control_interval_sec, h->d_action, fp_host ? h->d_fp : nullptr, obs_host ? h->d_obs : nullptr,
             reward_host ? h->d_reward : nullptr, greward_host ? h->d_greward : nullptr,
             done_host ? h->d_done : nullptr, st, rep0, count))
    return -1;
  if (obs_host) CK(cudaMemcpyAsync(obs_host, h->d_obs + r0 * h->n_obs, n * h->n_obs * 4, cudaMemcpyDeviceToHost, st));
  if (reward_host) CK(cudaMemcpyAsync(reward_host, h->d_reward + r0 * N, n * N * 4, cudaMemcpyDeviceToHost, st));
  if (greward_host) CK(cudaMemcpyAsync(greward_host, h->d_greward + r0, n * 4, cudaMemcpyDeviceToHost, st));
  if (done_host) CK(cudaMemcpyAsync(done_host, h->d_done + r0, n, cudaMemcpyDeviceToHost, st));
  if (sync) CK(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int tsc_step_host_range(tsc_handle* h, int32_t rep0, int32_t count, const int32_t* action_host,
                                   const float* fp_host, float* obs_host, float* reward_host, float* greward_host,
                                   uint8_t* done_host, void* stream) {
  return step_host_range(h, rep0, count, action_host, fp_host, obs_host, reward_host, greward_host, done_host, stream, true);
}

extern "C" int tsc_step_host_range_async(tsc_handle* h, int32_t rep0, int32_t count, const int32_t* action_host,
                                         const float* fp_host, float* obs_host, float* reward_host, float* greward_host,
                                         uint8_t* done_host, void* stream) {
  return step_host_range(h, rep0, count, action_host, fp_host, obs_host, reward_host, greward_host, done_host, stream, false);
}

// ---- evaluation / recording path (envs/env.py:409-437, 498-542) ---------------------------------------------------
extern "C" int tsc_set_record(tsc_handle* h, int32_t on) {
  if (!h) return fail("tsc_set_record: null handle");
  CK(cudaSetDevice(h->device));
  CK(cudaDeviceSynchronize());
  if (on && !h->d_trip) {
    if (h->smem_rec > 232448) return fail("tsc_set_record: the record-mode ring image does not fit in shared memory");
    h->trip_cap = 8192;
    if (dalloc(h, (size_t)h->R * h->args.net.n_slots, &h->d_trip)) return -1;
    if (dalloc(h, (size_t)h->R * h->trip_cap * 2, &h->d_trip_log)) return -1;
    if (dalloc(h, (size_t)h->R, &h->d_trip_cnt)) return -1;
  }
  if (on) {      // a fresh log; trip words of vehicles already in the network start from zero
    CK(cudaMemset(h->d_trip, 0, (size_t)h->R * h->args.net.n_slots * 4));
    CK(cudaMemset(h->d_trip_cnt, 0, (size_t)h->R * 4));
  }
  h->record = on != 0;
  return 0;
}

extern "C" int tsc_step_record(tsc_handle* h, const int32_t* action_dev, const float* fp_dev, float* obs_dev,
                               float* reward_dev, float* greward_dev, uint8_t* done_dev, float* sub_stats_dev,
                               void* stream) {
  if (!h || !action_dev) return fail("tsc_step_record: bad argument");
  if (!h->record) return fail("tsc_step_record: record mode is off (tsc_set_record)");
  CK(cudaSetDevice(h->device));
  const int ci = h->args.cfg.control_interval_sec;
  const DevNet& d = h->args.net;
  for (int t = 0; t < ci; ++t) {
    const bool last = t + 1 == ci;
    if (launch(h, 1, action_dev, fp_dev, last ? obs_dev : nullptr, last ? reward_dev : nullptr,
               last ? greward_dev : nullptr, last ? done_dev : nullptr, (cudaStream_t)stream, 0, -1, t))
      return -1;
    if (sub_stats_dev) {
      tsc_stats_kernel<<<h->R, 128, (2 * d.n_lanes + 1) * 4, (cudaStream_t)stream>>>(
          d, h->args.veh, h->args.lane_cnt, h->args.ctl, h->args.ctl_words, sub_stats_dev + (size_t)t * 8, ci * 8);
      CK(cudaGetLastError());
    }
  }
  return 0;
}

extern "C" int tsc_get_trips(tsc_handle* h, int32_t replica, uint32_t* rows_host, int32_t max_rows, int32_t* n_rows) {
  if (!h || replica < 0 || replica >= h->R || !rows_host || !n_rows) return fail("tsc_get_trips: bad argument");
  if (!h->d_trip_log) { *n_rows = 0; return 0; }
  CK(cudaSetDevice(h->device));
  CK(cudaDeviceSynchronize());
  int32_t cnt = 0;
  CK(cudaMemcpy(&cnt, h->d_trip_cnt + replica, 4, cudaMemcpyDeviceToHost));
  if (cnt > max_rows) cnt = max_rows;
  if (cnt > 0) CK(cudaMemcpy(rows_host, h->d_trip_log + (size_t)replica * h->trip_cap * 2, (size_t)cnt * 8, cudaMemcpyDeviceToHost));
  *n_rows = cnt;
  return 0;
}

extern "C" int tsc_get_counts(tsc_handle* h, int32_t* veh_dev, int32_t* halt_dev, int32_t* headwait_dev,
                              int32_t* phase_dev, void* stream) {
  if (!h) return fail("tsc_get_counts: null handle");
  CK(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t mw = h->meas_words, nd = h->n_det;
  int32_t* outs[4] = {veh_dev, halt_dev, headwait_dev, phase_dev};
  const size_t offs[4] = {0, nd, 2 * nd, 3 * nd};
  const size_t widths[4] = {nd, nd, nd, (size_t)h->n_nodes};
  for (int k = 0; k < 4; ++k)
    if (outs[k])
      CK(cudaMemcpy2DAsync(outs[k], widths[k] * 4, h->args.meas + offs[k], mw * 4, widths[k] * 4, h->R,
                           cudaMemcpyDeviceToDevice, st));
  return 0;
}

extern "C" int tsc_dump_state(tsc_handle* h, int32_t replica, int32_t* lane_cnt_host, uint32_t* veh_host,
                              int32_t* n_veh) {
  if (!h || replica < 0 || replica >= h->R) return fail("tsc_dump_state: bad argument");
  CK(cudaSetDevice(h->device));
  CK(cudaDeviceSynchronize());
  const DevNet& d = h->args.net;
  std::vector<uint8_t> cnt(d.lpad);
  CK(cudaMemcpy(cnt.data(), h->args.lane_cnt + (size_t)replica * d.lpad, d.lpad, cudaMemcpyDeviceToHost));
  int V = 0;
  for (int l = 0; l < d.n_lanes; ++l) { lane_cnt_host[l] = cnt[l]; V += cnt[l]; }
  if (V) {   // packed SoA on the device -> canonical [V][3] records {pos f32, speed f32, meta0} on the host
    std::vector<uint32_t> tmp((size_t)2 * V);
    for (int a = 0; a < 2; ++a)
      CK(cudaMemcpy(tmp.data() + (size_t)a * V, h->args.veh + ((size_t)replica * 2 + a) * d.n_slots, (size_t)V * 4,
                    cudaMemcpyDeviceToHost));
    for (int k = 0; k < V; ++k) {
      const uint32_t xv = tmp[k];
      const float fx = (float)(xv & 0xffffu) * 0.015625f, fv = (float)(xv >> 16) * 0.0009765625f;
      memcpy(&veh_host[(size_t)k * 3 + 0], &fx, 4);
      memcpy(&veh_host[(size_t)k * 3 + 1], &fv, 4);
      veh_host[(size_t)k * 3 + 2] = tmp[(size_t)V + k];
    }
  }
  *n_veh = V;
  return 0;
}

extern "C" int tsc_info(tsc_handle* h, int64_t* state_bytes_per_replica, int32_t* threads_per_block, int32_t* smem_bytes) {
  if (!h) return fail("tsc_info: null handle");
  const DevNet& d = h->args.net;
  if (state_bytes_per_replica)
    *state_bytes_per_replica = (int64_t)d.n_slots * 8 + d.lpad + (int64_t)h->args.ctl_words * 4 + (int64_t)h->meas_words * 4;
  if (threads_per_block) *threads_per_block = TSC_THREADS;
  if (smem_bytes) *smem_bytes = h->smem;
  return 0;
}

extern "C" int tsc_mean_live(tsc_handle* h, double* mean_live) {
  if (!h || !mean_live) return fail("tsc_mean_live: bad argument");
  CK(cudaSetDevice(h->device));
  CK(cudaMemset(h->d_scalar, 0, 8));
  int n_sm = 0;
  CK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, h->device));
  tsc_live_kernel<<<n_sm, 256>>>(h->args.lane_cnt, h->args.net.lpad, h->args.net.n_lanes, h->R, h->d_scalar);
  CK(cudaGetLastError());
  unsigned long long s = 0;
  CK(cudaMemcpy(&s, h->d_scalar, 8, cudaMemcpyDeviceToHost));
  *mean_live = (double)s / (double)h->R;
  return 0;
}

extern "C" int tsc_get_traffic_stats(tsc_handle* h, float* stats_dev, void* stream) {
  if (!h || !stats_dev) return fail("tsc_get_traffic_stats: bad argument");
  CK(cudaSetDevice(h->device));
  const DevNet& d = h->args.net;
  tsc_stats_kernel<<<h->R, 128, (2 * d.n_lanes + 1) * 4, (cudaStream_t)stream>>>(d, h->args.veh, h->args.lane_cnt,
                                                                                   h->args.ctl, h->args.ctl_words, stats_dev, 8);
  CK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Greedy controllers (reference envs/large_grid_env.py:45-60, envs/real_net_env.py:78-111, envs/small_grid_env.py:41-57):
// per node, every candidate phase scores the sum of a fixed list of that node's observation entries, accumulated in
// float64 in list order (the reference sums float64 copies of the observation), and the FIRST maximum wins (np.argmax).
// One thread per (replica, node).
__global__ void tsc_greedy_kernel(const float* __restrict__ obs, int32_t* __restrict__ action, int64_t RN, int n_nodes,
                                  int n_obs, int max_cand, const int32_t* __restrict__ off, const int32_t* __restrict__ idx,
                                  const int32_t* __restrict__ act) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= RN) return;
  const int64_t r = i / n_nodes;
  const int node = (int)(i - r * n_nodes);
  const float* o = obs + r * n_obs;
  double best = 0.0;
  int pick = 0;
  bool any = false;
  for (int c = 0; c < max_cand; ++c) {
    const int k = node * max_cand + c;
    if (act[k] < 0) continue;             // padding: the node has fewer candidates
    double s = 0.0;
    for (int e = off[k]; e < off[k + 1]; ++e) s += (double)o[idx[e]];
    if (!any || s > best) { best = s; pick = act[k]; any = true; }
  }
  action[i] = pick;
}

extern "C" int tsc_set_greedy_program(tsc_handle* h, int32_t max_cand, const int32_t* off_host, const int32_t* idx_host,
                                      const int32_t* act_host) {
  if (!h || max_cand <= 0 || !off_host || !act_host) return fail("tsc_set_greedy_program: bad argument");
  const int nk = h->n_nodes * max_cand;
  if (off_host[0] != 0) return fail("tsc_set_greedy_program: off[0] must be 0");
  for (int k = 0; k < nk; ++k)
    if (off_host[k + 1] < off_host[k]) return fail("tsc_set_greedy_program: offsets must not decrease");
  const int n_idx = off_host[nk];
  if (n_idx > 0 && !idx_host) return fail("tsc_set_greedy_program: bad argument");
  for (int e = 0; e < n_idx; ++e)
    if (idx_host[e] < 0 || idx_host[e] >= h->n_obs) return fail("tsc_set_greedy_program: observation offset out of range");
  CK(cudaSetDevice(h->device));
  cudaFree(h->d_gp_off); cudaFree(h->d_gp_idx); cudaFree(h->d_gp_act);
  h->d_gp_off = h->d_gp_idx = h->d_gp_act = nullptr;
  h->gp_max_cand = 0;
  CK(cudaMalloc(&h->d_gp_off, sizeof(int32_t) * (nk + 1)));
  CK(cudaMalloc(&h->d_gp_idx, sizeof(int32_t) * (n_idx > 0 ? n_idx : 1)));
  CK(cudaMalloc(&h->d_gp_act, sizeof(int32_t) * nk));
  CK(cudaMemcpy(h->d_gp_off, off_host, sizeof(int32_t) * (nk + 1), cudaMemcpyHostToDevice));
  if (n_idx > 0) CK(cudaMemcpy(h->d_gp_idx, idx_host, sizeof(int32_t) * n_idx, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(h->d_gp_act, act_host, sizeof(int32_t) * nk, cudaMemcpyHostToDevice));
  h->gp_max_cand = max_cand;
  return 0;
}

extern "C" int tsc_greedy_actions(tsc_handle* h, const float* obs_dev, int32_t* action_dev, void* stream) {
  if (!h || !obs_dev || !action_dev) return fail("tsc_greedy_actions: bad argument");
  if (h->gp_max_cand <= 0) return fail("tsc_greedy_actions: no greedy program (call tsc_set_greedy_program)");
  CK(cudaSetDevice(h->device));
  const int64_t RN = (int64_t)h->R * h->n_nodes;
  tsc_greedy_kernel<<<(unsigned)((RN + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      obs_dev, action_dev, RN, h->n_nodes, h->n_obs, h->gp_max_cand, h->d_gp_off, h->d_gp_idx, h->d_gp_act);
  CK(cudaGetLastError());
  return 0;
}
