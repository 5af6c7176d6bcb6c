// tsc_q.cu — test-mode forward of the IQL Q networks for R replicas and all A agents at once (include/tsc_learn.h,
// tscl_q_*).  Replaces the per-agent `sess.run(qvalues)` + host argmax / sample of the reference's
// IQL.forward(obs, mode='act', stochastic) (agents/models.py:347-363) on the networks of agents/policies.py:341-389:
//   LRQPolicy     q = S.W + b
//   DeepQPolicy   h0 = relu(S[:, :n_s-n_w].W_fcw + b), h1 = relu(S[:, n_s-n_w:].W_fct + b) (n_w > 0 only),
//                 h = relu([h0 | h1].W_fc0 + b), q = h.W_q + b
// fp32 SIMT FMAs on purpose: the action is an argmax over q, and bf16 / tf32 operands (relative error ~1e-3) would flip
// near-ties that an fp32 host forward keeps.
//
// One CTA per (agent, group of 64-row tiles), persistent over its tiles; the agent's weights stay in shared memory.
// 256 threads; thread (ty, tx) = (tid / 16, tid % 16) owns rows 4 ty .. 4 ty + 3 of a tile and the columns tx + 16 j of
// the two hidden layers.  Activations are kept column-major in shared memory ([column][row], row pitch QT_LD), so one
// 128-bit load gives a thread its four rows and the weight loads of a half-warp are 16 consecutive floats.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/tsc_learn.h"

int tsc_set_error(const std::string& m);  // defined in tsc_sim.cu

#define LCK(call)                                                                  \
  do {                                                                             \
    cudaError_t e__ = (call);                                                      \
    if (e__ != cudaSuccess) return tsc_set_error(std::string(#call) + ": " + cudaGetErrorString(e__)); \
  } while (0)

#define QT_ROWS 64               // rows per tile
#define QT_LD (QT_ROWS + 4)      // row pitch of the column-major activation tiles (16-byte aligned columns)
#define QT_FC_MAX 128            // q_fcw width: 8 columns per thread
#define QT_FT_MAX 32             // q_fct width: 2 columns per thread
#define QT_H_MAX 64              // q_fc_0 width: 4 columns per thread
#define QT_NA 8                  // padded action dimension in shared memory

struct QDims {
  int A, n_obs, max_na, model, n_fc, n_ft, n_h;
  const int32_t *obs_off, *n_s, *n_w, *n_a;
  const int64_t *off_fcw_w, *off_fcw_b, *off_fct_w, *off_fct_b, *off_fc0_w, *off_fc0_b, *off_q_w, *off_q_b;
  // shared-memory extents (maxima over the agents, so every CTA uses the same layout), in floats
  int s_max;     // widest observation slice
  int wave_max;  // widest wave block (dqn)
  int w_max;     // widest wait block (dqn)
  int in2_max;   // widest input of q_fc_0 (dqn)
  int q_in;      // rows of the resident q weight: n_h (dqn) or s_max (lr)
};

#define QG_MAX 64                // members of one grouped launch (their per-member scalars travel by value)

// Per-member scalars of a grouped launch (ε, γ, lr_t, max_grad_norm, reward scaling), copied from a host array into the
// kernel's parameters: no upload and no host sync per call.
struct QMemberF {
  float v[QG_MAX];
};

static QMemberF q_member_f(const float* host, int K) {
  QMemberF o{};
  for (int k = 0; k < K; ++k) o.v[k] = host[k];
  return o;
}

struct tscl_qhandle {
  int device = 0;
  QDims d{};
  std::vector<void*> owned;
  size_t smem = 0;
  int ctas_per_sm = 1, n_sm = 1;
  int64_t n_params = 0;
  size_t td_smem = 0;            // 0: the TD kernel's layout does not fit a CTA (tscl_q_td refuses)
  int td_ctas_per_sm = 1;
  const int64_t* blk = nullptr;  // [A + 1] first float of every agent's block in the flat vector, then n_params
  float* part = nullptr;         // TD partials [groups][n_params + 3 A]
  float* part_g = nullptr;       // grouped TD partials [K][groups][n_params + 3 A] (tscl_q_td_g)
  int part_g_k = 0;              // members part_g holds
};

struct QSmem {          // float offsets of the shared-memory regions
  int w1, b1, wt, w2, b2, wq, bq, s, h1, h2, q, total;
};

__host__ __device__ inline QSmem q_smem_layout(const QDims& d) {
  QSmem o;
  int p = 0;
  const int h1w = d.n_fc + d.n_ft;
  o.w1 = p; p += d.wave_max * d.n_fc;
  o.b1 = p; p += h1w;
  o.wt = p; p += d.w_max * d.n_ft;
  o.w2 = p; p += d.in2_max * d.n_h;
  o.b2 = p; p += d.n_h;
  o.wq = p; p += d.q_in * QT_NA;
  o.bq = p; p += QT_NA;
  p = (p + 3) & ~3;                    // 16-byte aligned activation tiles
  o.s = p; p += d.s_max * QT_LD;
  o.h1 = p; p += h1w * QT_LD;
  o.h2 = p; p += d.n_h * QT_LD;
  o.q = p; p += QT_ROWS * QT_NA;
  o.total = p;
  return o;
}

// The TD kernel's shared memory: the forward's regions, except that the q_fc_0 weight lives at an odd row pitch in w2p
// (the transposed reads of the backward are then free of bank conflicts) and the forward's unpadded w2 region holds that
// weight's gradient.  Then the other weight-gradient accumulators, at the weights' unpadded shapes (their order in the
// flat vector), and three per-row arrays of a tile: TD target, dL/dq of the taken action, the action.
struct QTdSmem {
  QSmem f;
  int ld2, w2p, gw1, gb1, gwt, gw2, gb2, gwq, gbq, tq, dq, act, total;
};

__host__ __device__ inline QTdSmem q_td_smem_layout(const QDims& d) {
  QTdSmem o;
  o.f = q_smem_layout(d);
  int p = o.f.total;
  o.ld2 = d.n_h + 1;
  o.gw2 = o.f.w2;
  o.w2p = p; p += d.in2_max * o.ld2;
  o.gw1 = p; p += d.wave_max * d.n_fc;
  o.gb1 = p; p += d.n_fc + d.n_ft;
  o.gwt = p; p += d.w_max * d.n_ft;
  o.gb2 = p; p += d.n_h;
  o.gwq = p; p += d.q_in * QT_NA;
  o.gbq = p; p += QT_NA;
  o.tq = p; p += QT_ROWS;
  o.dq = p; p += QT_ROWS;
  o.act = p; p += QT_ROWS;
  o.total = p;
  return o;
}

__device__ __forceinline__ uint32_t qmix32(uint32_t h) {   // the counter hash of the A2C sampling kernels
  h ^= h >> 16; h *= 0x7feb352dU; h ^= h >> 15; h *= 0x846ca68bU; h ^= h >> 16;
  return h;
}

// One hidden layer on a 64-row tile: out[c][row] = relu(sum_k in[k][row] W[k][c] + b[c]) for the columns c = tx + 16 j,
// j < ncol (ncol <= NJ), k < K.  `in` / `out` column-major with pitch QT_LD; W row-major with `ldw` columns.
// BWD: the same layer's input gradient, in place: out[c][row] = (sum_k in[k][row] W[c][k]) * (out[c][row] > 0), with
// `in` the output gradient and `out` holding the layer input's relu activations (b unused).
template <int NJ, bool BWD = false>
__device__ __forceinline__ void q_dense_relu(const float* __restrict__ in, int K, const float* __restrict__ W, int ldw,
                                             const float* __restrict__ b, int ncol, float* __restrict__ out, int ty,
                                             int tx) {
  float acc[4][NJ];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc[i][j] = 0.f;
#pragma unroll 4
  for (int k = 0; k < K; ++k) {                // unrolled: the shared-memory loads of 4 k run ahead of their FMAs
    const float4 x = *reinterpret_cast<const float4*>(in + k * QT_LD + ty * 4);
    const float* w = W + k * ldw + tx;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      if (j < ncol) {
        const float wj = BWD ? W[(tx + 16 * j) * ldw + k] : w[16 * j];
        acc[0][j] = fmaf(x.x, wj, acc[0][j]); acc[1][j] = fmaf(x.y, wj, acc[1][j]);
        acc[2][j] = fmaf(x.z, wj, acc[2][j]); acc[3][j] = fmaf(x.w, wj, acc[3][j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    if (j < ncol) {
      float4* o = reinterpret_cast<float4*>(out + (tx + 16 * j) * QT_LD + ty * 4);
      if (BWD) {
        const float4 h = *o;
        *o = make_float4(h.x > 0.f ? acc[0][j] : 0.f, h.y > 0.f ? acc[1][j] : 0.f, h.z > 0.f ? acc[2][j] : 0.f,
                         h.w > 0.f ? acc[3][j] : 0.f);
      } else {
        const float bj = b[tx + 16 * j];
        *o = make_float4(fmaxf(acc[0][j] + bj, 0.f), fmaxf(acc[1][j] + bj, 0.f), fmaxf(acc[2][j] + bj, 0.f),
                         fmaxf(acc[3][j] + bj, 0.f));
      }
    }
  }
}

// The network on one tile whose observation slice is in sS: q of the 64 rows into sQ [row][QT_NA] (hidden activations
// left in sH1 / sH2), with q_fc_0's weight at row pitch ld2.  Ends before the barrier that publishes sQ.  The TD kernel's
// forward; q_fwd_kernel keeps the same statements inline so that its evaluation instantiations compile as before.
template <bool DQN>
__device__ __forceinline__ void q_tile_forward(const QDims& d, const float* sS, const float* sW1, const float* sB1,
                                               const float* sWt, const float* sW2, int ld2, const float* sB2,
                                               const float* sWq, const float* sBq, float* sH1, float* sH2, float* sQ,
                                               int n_wave, int n_w, int n_ft, int q_in, int tid, int ty, int tx) {
  const float* qin = sS;
  if (DQN) {
    q_dense_relu<QT_FC_MAX / 16>(sS, n_wave, sW1, d.n_fc, sB1, d.n_fc / 16, sH1, ty, tx);
    if (n_ft > 0)
      q_dense_relu<QT_FT_MAX / 16>(sS + n_wave * QT_LD, n_w, sWt, n_ft, sB1 + d.n_fc, n_ft / 16,
                                   sH1 + d.n_fc * QT_LD, ty, tx);
    __syncthreads();
    q_dense_relu<QT_H_MAX / 16>(sH1, d.n_fc + n_ft, sW2, ld2, sB2, d.n_h / 16, sH2, ty, tx);
    __syncthreads();
    qin = sH2;
  }
  // output layer (linear): thread = (row, two actions)
  const int row = tid & (QT_ROWS - 1), j0 = (tid >> 6) * 2;
  float q0 = 0.f, q1 = 0.f;
#pragma unroll 4
  for (int k = 0; k < q_in; ++k) {
    const float x = qin[k * QT_LD + row];
    q0 = fmaf(x, sWq[k * QT_NA + j0], q0);
    q1 = fmaf(x, sWq[k * QT_NA + j0 + 1], q1);
  }
  sQ[row * QT_NA + j0] = q0 + sBq[j0];
  sQ[row * QT_NA + j0 + 1] = q1 + sBq[j0 + 1];
}

// The counter hash keyed (seed, step, replica, agent) of ε-greedy exploration: the chain of mode 1 in q_fwd_kernel.
__device__ __forceinline__ uint32_t q_row_hash(uint32_t seed_lo, uint32_t seed_hi, uint32_t step, int64_t replica, int a) {
  uint32_t hsh = qmix32(seed_lo ^ (step * 0x9E3779B1U));
  hsh = qmix32(hsh ^ seed_hi ^ ((uint32_t)replica * 0x85EBCA77U));
  return qmix32(hsh ^ ((uint32_t)a * 0xC2B2AE3DU));
}

// grid (groups, A), 256 threads.  DQN = false: LRQPolicy, true: DeepQPolicy.
// EXPLORE: IQL.forward(obs, mode='explore') — the first maximum of q, replaced by a uniform action when the row's
// uniform is below eps; also stores act (int8) and, from the agent-0 CTAs, whole observation rows into a replay slot.
template <bool DQN, bool EXPLORE = false>
__global__ void __launch_bounds__(256)
q_fwd_kernel(const QDims d, const float* __restrict__ P, const float* __restrict__ obs, int64_t R,
             float* __restrict__ q, int32_t* __restrict__ act, int mode, uint32_t seed_lo, uint32_t seed_hi,
             uint32_t step, int64_t replica0, unsigned long long* __restrict__ bad, float eps,
             float* __restrict__ ring_s, int8_t* __restrict__ ring_a) {
  extern __shared__ __align__(16) float qsm[];
  const QSmem L = q_smem_layout(d);
  const int a = blockIdx.y, tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int n_s = d.n_s[a], n_a = d.n_a[a], ooff = d.obs_off[a];
  const int n_w = DQN ? d.n_w[a] : 0, n_wave = n_s - n_w;
  const int n_ft = n_w > 0 ? d.n_ft : 0;            // agents without a wait block have no q_fct layer
  const int q_in = DQN ? d.n_h : n_s;
  float *sW1 = qsm + L.w1, *sB1 = qsm + L.b1, *sWt = qsm + L.wt, *sW2 = qsm + L.w2, *sB2 = qsm + L.b2;
  float *sWq = qsm + L.wq, *sBq = qsm + L.bq, *sS = qsm + L.s, *sH1 = qsm + L.h1, *sH2 = qsm + L.h2, *sQ = qsm + L.q;

  // resident weights of agent a
  if (DQN) {
    for (int i = tid; i < n_wave * d.n_fc; i += 256) sW1[i] = P[d.off_fcw_w[a] + i];
    for (int i = tid; i < d.n_fc; i += 256) sB1[i] = P[d.off_fcw_b[a] + i];
    for (int i = tid; i < n_w * n_ft; i += 256) sWt[i] = P[d.off_fct_w[a] + i];
    for (int i = tid; i < n_ft; i += 256) sB1[d.n_fc + i] = P[d.off_fct_b[a] + i];
    for (int i = tid; i < (d.n_fc + n_ft) * d.n_h; i += 256) sW2[i] = P[d.off_fc0_w[a] + i];
    for (int i = tid; i < d.n_h; i += 256) sB2[i] = P[d.off_fc0_b[a] + i];
  }
  for (int i = tid; i < q_in * QT_NA; i += 256) {
    const int k = i / QT_NA, j = i - k * QT_NA;
    sWq[i] = j < n_a ? P[d.off_q_w[a] + (int64_t)k * n_a + j] : 0.f;
  }
  for (int i = tid; i < QT_NA; i += 256) sBq[i] = i < n_a ? P[d.off_q_b[a] + i] : 0.f;

  const int64_t n_tiles = (R + QT_ROWS - 1) / QT_ROWS;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t m0 = tile * QT_ROWS;
    __syncthreads();
    // observation slice of agent a, transposed into [k][row]; rows past R are zero (never written back)
    for (int i = tid; i < QT_ROWS * n_s; i += 256) {
      const int row = i / n_s, k = i - row * n_s;
      const int64_t m = m0 + row;
      sS[k * QT_LD + row] = m < R ? __ldg(obs + m * d.n_obs + ooff + k) : 0.f;
    }
    if (EXPLORE && blockIdx.y == 0 && ring_s) {
      const int64_t nr = R - m0 < QT_ROWS ? R - m0 : QT_ROWS;
      for (int64_t i = tid; i < nr * d.n_obs; i += 256) ring_s[m0 * d.n_obs + i] = obs[m0 * d.n_obs + i];
    }
    __syncthreads();
    const float* qin = sS;
    if (DQN) {
      q_dense_relu<QT_FC_MAX / 16>(sS, n_wave, sW1, d.n_fc, sB1, d.n_fc / 16, sH1, ty, tx);
      if (n_ft > 0)
        q_dense_relu<QT_FT_MAX / 16>(sS + n_wave * QT_LD, n_w, sWt, n_ft, sB1 + d.n_fc, n_ft / 16,
                                     sH1 + d.n_fc * QT_LD, ty, tx);
      __syncthreads();
      q_dense_relu<QT_H_MAX / 16>(sH1, d.n_fc + n_ft, sW2, d.n_h, sB2, d.n_h / 16, sH2, ty, tx);
      __syncthreads();
      qin = sH2;
    }
    // output layer (linear): thread = (row, two actions)
    {
      const int row = tid & (QT_ROWS - 1), j0 = (tid >> 6) * 2;
      float q0 = 0.f, q1 = 0.f;
#pragma unroll 4
      for (int k = 0; k < q_in; ++k) {
        const float x = qin[k * QT_LD + row];
        q0 = fmaf(x, sWq[k * QT_NA + j0], q0);
        q1 = fmaf(x, sWq[k * QT_NA + j0 + 1], q1);
      }
      sQ[row * QT_NA + j0] = q0 + sBq[j0];
      sQ[row * QT_NA + j0 + 1] = q1 + sBq[j0 + 1];
    }
    __syncthreads();
    if (tid < QT_ROWS && m0 + tid < R) {
      const int64_t r = m0 + tid;
      float qv[QT_NA];
#pragma unroll
      for (int j = 0; j < QT_NA; ++j) qv[j] = sQ[tid * QT_NA + j];
      float* qo = q + (r * d.A + a) * d.max_na;
#pragma unroll
      for (int j = 0; j < QT_NA; ++j)
        if (j < d.max_na) qo[j] = j < n_a ? qv[j] : 0.f;
      int pick = 0;
      if (mode == 0) {                        // np.argmax: the first maximum
        float best = qv[0];
#pragma unroll
        for (int j = 1; j < QT_NA; ++j)
          if (j < n_a && qv[j] > best) { best = qv[j]; pick = j; }
        if (EXPLORE) {                        // np.random.random() < eps: np.random.randint(n_a)
          const uint32_t hsh = q_row_hash(seed_lo, seed_hi, step, replica0 + r, a);
          if ((float)(hsh >> 8) * (1.0f / 16777216.0f) < eps)
            pick = (int)(((uint64_t)qmix32(hsh ^ 0x5BD1E995U) * (uint32_t)n_a) >> 32);
          if (ring_a) ring_a[r * d.A + a] = (int8_t)pick;
        }
      } else {                                // qs / np.sum(qs); np.random.choice(n_a, p=qs)
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < QT_NA; ++j)
          if (j < n_a) s = __fadd_rn(s, qv[j]);
        bool ok = isfinite(s) && s != 0.f;
        float p[QT_NA];
#pragma unroll
        for (int j = 0; j < QT_NA; ++j) {
          p[j] = j < n_a ? __fdiv_rn(qv[j], s) : 0.f;
          ok = ok && (j >= n_a || (p[j] >= 0.f && isfinite(p[j])));
        }
        if (ok) {
          uint32_t hsh = qmix32(seed_lo ^ (step * 0x9E3779B1U));
          hsh = qmix32(hsh ^ seed_hi ^ ((uint32_t)(replica0 + r) * 0x85EBCA77U));
          hsh = qmix32(hsh ^ ((uint32_t)a * 0xC2B2AE3DU));
          const float uu = (float)(hsh >> 8) * (1.0f / 16777216.0f);
          float cum = 0.f;
          bool found = false;
          pick = n_a - 1;
#pragma unroll
          for (int j = 0; j < QT_NA; ++j) {
            if (j < n_a) {
              cum = __fadd_rn(cum, p[j]);
              if (!found && uu < cum) { pick = j; found = true; }
            }
          }
        } else if (bad) {                     // np.random.choice would raise: report (replica, step, agent), act 0
          const unsigned long long key = ((unsigned long long)(replica0 + r) << 40) |
                                         ((unsigned long long)(step & 0xFFFFFFu) << 16) | (unsigned long long)a;
          atomicMin(bad, key);
        }
      }
      act[r * d.A + a] = pick;
    }
  }
}

// Grouped form (tscl_q_step_g): grid (groups, A, K); CTA (g, a, k) walks tiles g, g + groups, .. of member k, whose rows
// are rows[k] .. rows[k+1] - 1 (ragged: a member's last tile is partial), with member k's weights of agent a (P + k
// p_stride) resident.  Per row the statements of q_fwd_kernel's evaluation path (the network through q_tile_forward at
// q_fc_0's own pitch, the same chain of fp32 operations), keyed with seeds[k] and the member-local replica index, and
// a failed sample reported into bad[k]: member k's outputs are those of its own tscl_q_step launch.
// EXPLORE (tscl_q_explore_g): q_fwd_kernel's explore path per member, with ε eps.v[k] and the draws keyed by `seed`
// and the member-local replica; the ring slot's rows ring_s / ring_a are the lock-step's (row0 + r): member k's outputs
// are those of its own tscl_q_explore launch with replica0 = 0.
template <bool DQN, bool EXPLORE = false>
__global__ void __launch_bounds__(256)
q_fwd_g_kernel(const QDims d, const float* __restrict__ P0, int64_t p_stride, const float* __restrict__ obs,
               const int64_t* __restrict__ rows, float* __restrict__ q, int32_t* __restrict__ act, int mode,
               const uint64_t* __restrict__ seeds, uint32_t step, unsigned long long* __restrict__ bad,
               const QMemberF eps, uint64_t seed, float* __restrict__ ring_s, int8_t* __restrict__ ring_a) {
  extern __shared__ __align__(16) float qsm[];
  const int k = blockIdx.z;
  const int64_t row0 = rows[k], S = rows[k + 1] - row0;
  const int64_t n_tiles = (S + QT_ROWS - 1) / QT_ROWS;
  if (blockIdx.x >= n_tiles) return;                 // the whole CTA: no barrier is pending
  const QSmem L = q_smem_layout(d);
  const float* P = P0 + (int64_t)k * p_stride;
  const int a = blockIdx.y, tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int n_s = d.n_s[a], n_a = d.n_a[a], ooff = d.obs_off[a];
  const int n_w = DQN ? d.n_w[a] : 0, n_wave = n_s - n_w;
  const int n_ft = n_w > 0 ? d.n_ft : 0;
  const int q_in = DQN ? d.n_h : n_s;
  float *sW1 = qsm + L.w1, *sB1 = qsm + L.b1, *sWt = qsm + L.wt, *sW2 = qsm + L.w2, *sB2 = qsm + L.b2;
  float *sWq = qsm + L.wq, *sBq = qsm + L.bq, *sS = qsm + L.s, *sH1 = qsm + L.h1, *sH2 = qsm + L.h2, *sQ = qsm + L.q;
  if (DQN) {
    for (int i = tid; i < n_wave * d.n_fc; i += 256) sW1[i] = P[d.off_fcw_w[a] + i];
    for (int i = tid; i < d.n_fc; i += 256) sB1[i] = P[d.off_fcw_b[a] + i];
    for (int i = tid; i < n_w * n_ft; i += 256) sWt[i] = P[d.off_fct_w[a] + i];
    for (int i = tid; i < n_ft; i += 256) sB1[d.n_fc + i] = P[d.off_fct_b[a] + i];
    for (int i = tid; i < (d.n_fc + n_ft) * d.n_h; i += 256) sW2[i] = P[d.off_fc0_w[a] + i];
    for (int i = tid; i < d.n_h; i += 256) sB2[i] = P[d.off_fc0_b[a] + i];
  }
  for (int i = tid; i < q_in * QT_NA; i += 256) {
    const int kk = i / QT_NA, j = i - kk * QT_NA;
    sWq[i] = j < n_a ? P[d.off_q_w[a] + (int64_t)kk * n_a + j] : 0.f;
  }
  for (int i = tid; i < QT_NA; i += 256) sBq[i] = i < n_a ? P[d.off_q_b[a] + i] : 0.f;
  const uint64_t sk = EXPLORE ? seed : seeds[k];
  const uint32_t seed_lo = (uint32_t)(sk & 0xFFFFFFFFu), seed_hi = (uint32_t)(sk >> 32);

  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t m0 = tile * QT_ROWS;               // member-local
    __syncthreads();
    for (int i = tid; i < QT_ROWS * n_s; i += 256) {
      const int row = i / n_s, kk = i - row * n_s;
      const int64_t m = m0 + row;
      sS[kk * QT_LD + row] = m < S ? __ldg(obs + (row0 + m) * d.n_obs + ooff + kk) : 0.f;
    }
    if (EXPLORE && blockIdx.y == 0 && ring_s) {
      const int64_t nr = S - m0 < QT_ROWS ? S - m0 : QT_ROWS, o = (row0 + m0) * d.n_obs;
      for (int64_t i = tid; i < nr * d.n_obs; i += 256) ring_s[o + i] = obs[o + i];
    }
    __syncthreads();
    q_tile_forward<DQN>(d, sS, sW1, sB1, sWt, sW2, d.n_h, sB2, sWq, sBq, sH1, sH2, sQ, n_wave, n_w, n_ft, q_in, tid, ty,
                        tx);
    __syncthreads();
    if (tid < QT_ROWS && m0 + tid < S) {
      const int64_t r = m0 + tid, g = row0 + r;
      float qv[QT_NA];
#pragma unroll
      for (int j = 0; j < QT_NA; ++j) qv[j] = sQ[tid * QT_NA + j];
      float* qo = q + (g * d.A + a) * d.max_na;
#pragma unroll
      for (int j = 0; j < QT_NA; ++j)
        if (j < d.max_na) qo[j] = j < n_a ? qv[j] : 0.f;
      int pick = 0;
      if (mode == 0) {
        float best = qv[0];
#pragma unroll
        for (int j = 1; j < QT_NA; ++j)
          if (j < n_a && qv[j] > best) { best = qv[j]; pick = j; }
        if (EXPLORE) {
          const uint32_t hsh = q_row_hash(seed_lo, seed_hi, step, r, a);
          if ((float)(hsh >> 8) * (1.0f / 16777216.0f) < eps.v[k])
            pick = (int)(((uint64_t)qmix32(hsh ^ 0x5BD1E995U) * (uint32_t)n_a) >> 32);
          if (ring_a) ring_a[g * d.A + a] = (int8_t)pick;
        }
      } else {
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < QT_NA; ++j)
          if (j < n_a) s = __fadd_rn(s, qv[j]);
        bool ok = isfinite(s) && s != 0.f;
        float p[QT_NA];
#pragma unroll
        for (int j = 0; j < QT_NA; ++j) {
          p[j] = j < n_a ? __fdiv_rn(qv[j], s) : 0.f;
          ok = ok && (j >= n_a || (p[j] >= 0.f && isfinite(p[j])));
        }
        if (ok) {
          const float uu = (float)(q_row_hash(seed_lo, seed_hi, step, r, a) >> 8) * (1.0f / 16777216.0f);
          float cum = 0.f;
          bool found = false;
          pick = n_a - 1;
#pragma unroll
          for (int j = 0; j < QT_NA; ++j) {
            if (j < n_a) {
              cum = __fadd_rn(cum, p[j]);
              if (!found && uu < cum) { pick = j; found = true; }
            }
          }
        } else if (bad) {
          const unsigned long long key = ((unsigned long long)r << 40) | ((unsigned long long)(step & 0xFFFFFFu) << 16) |
                                         (unsigned long long)a;
          atomicMin(bad + k, key);
        }
      }
      act[g * d.A + a] = pick;
    }
  }
}


// ================================================================================================
// Training (IQL.backward, agents/models.py:305-312): minibatch sampler, fused TD forward / backward, reduction, clip + Adam.

// Counter-hash key of agent a's minibatch draws in one round of one update, for global replica `replica`.
__device__ __forceinline__ uint32_t q_sample_key(uint32_t seed_lo, uint32_t seed_hi, uint32_t update, uint32_t round,
                                                 int64_t replica, int a) {
  uint32_t hsh = qmix32(seed_lo ^ (update * 0x9E3779B1U));
  hsh = qmix32(hsh ^ seed_hi ^ ((uint32_t)replica * 0x85EBCA77U));
  return qmix32(hsh ^ ((uint32_t)a * 0xC2B2AE3DU) ^ (round * 0x27D4EB2FU));
}

// random.sample(range(size), batch) per (agent, replica): Floyd's algorithm, draw d picks t uniform in [0, j] with
// j = size - batch + d by multiply-shift (bias <= size / 2^32) and keeps j instead when t was already taken.  One thread
// per (agent, replica); idx [A][R][batch].
__global__ void q_sample_kernel(int A, int64_t R, int batch, int size, uint32_t seed_lo, uint32_t seed_hi,
                                uint32_t update, uint32_t round, int64_t replica0, int32_t* __restrict__ idx) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)A * R) return;
  const int a = (int)(i / R);
  const int64_t r = i - (int64_t)a * R;
  const uint32_t key = q_sample_key(seed_lo, seed_hi, update, round, replica0 + r, a);
  int32_t* out = idx + i * batch;
  for (int dd = 0; dd < batch; ++dd) {
    const uint32_t j = (uint32_t)(size - batch + dd);
    const uint32_t x = qmix32(key ^ ((uint32_t)(dd + 1) * 0x165667B1U));
    const int32_t t = (int32_t)(((uint64_t)x * (j + 1u)) >> 32);
    bool taken = false;
    for (int e = 0; e < dd; ++e) taken |= out[e] == t;
    out[dd] = taken ? (int32_t)j : t;
  }
}

// G[k][c] += sum over the tile's rows of A[k][row] B[c][row] for k < K and the columns c = tx + 16 j, j < ncol (<= NJ);
// A / B column-major tiles (pitch QT_LD), G row-major with ldg columns.  Every G element has one owner thread.
template <int KI, int NJ>
__device__ __forceinline__ void q_wgrad(const float* __restrict__ A, int K, const float* __restrict__ B, int ncol,
                                        float* __restrict__ G, int ldg, int ty, int tx) {
  for (int k0 = 0; k0 < K; k0 += 16 * KI) {
    float acc[KI][NJ];
#pragma unroll
    for (int i = 0; i < KI; ++i)
#pragma unroll
      for (int j = 0; j < NJ; ++j) acc[i][j] = 0.f;
    for (int r = 0; r < QT_ROWS; r += 4) {
      float4 b[NJ];
#pragma unroll
      for (int j = 0; j < NJ; ++j)
        if (j < ncol) b[j] = *reinterpret_cast<const float4*>(B + (tx + 16 * j) * QT_LD + r);
#pragma unroll
      for (int i = 0; i < KI; ++i) {
        const int k = k0 + ty + 16 * i;
        if (k < K) {
          const float4 x = *reinterpret_cast<const float4*>(A + k * QT_LD + r);
#pragma unroll
          for (int j = 0; j < NJ; ++j)
            if (j < ncol) {
              acc[i][j] = fmaf(x.x, b[j].x, acc[i][j]); acc[i][j] = fmaf(x.y, b[j].y, acc[i][j]);
              acc[i][j] = fmaf(x.z, b[j].z, acc[i][j]); acc[i][j] = fmaf(x.w, b[j].w, acc[i][j]);
            }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < KI; ++i) {
      const int k = k0 + ty + 16 * i;
#pragma unroll
      for (int j = 0; j < NJ; ++j)
        if (k < K && j < ncol) G[k * ldg + tx + 16 * j] += acc[i][j];
    }
  }
}

// Gb[c] += sum over the tile's rows of B[c][row], c < n
__device__ __forceinline__ void q_bgrad(const float* __restrict__ B, int n, float* __restrict__ Gb, int tid) {
  for (int c = tid; c < n; c += 256) {
    float s = 0.f;
    for (int r = 0; r < QT_ROWS; ++r) s += B[c * QT_LD + r];
    Gb[c] += s;
  }
}

// One round of QPolicy.backward for every agent (agents/policies.py:307-338): rows m < R * batch of agent a are the
// ring entries (slot idx[a][r][m % batch], replica r = m / batch).  tq = done ? r : r + gamma max_j q(s1)_j (no gradient,
// same network), e = q(s)[act] - tq, loss = sum e^2 * inv_n, dq = 2 e inv_n.  grid (groups, A), 256 threads; CTA (g, a)
// walks tiles g, g + groups, .. with agent a's weights resident, accumulates its weight gradients in shared memory, and
// writes them at the agent's flat offsets into partial row g (part [groups][ld]); the tail columns n_params + a,
// n_params + A + a and n_params + 2 A + a get inv_n times the CTA's sums of e^2, q(s)[act] and tq (the summaries of
// QPolicy, agents/policies.py:331-338: loss, mean q, mean tq).
// GROUPED (tscl_q_td_g): grid (groups, A, K); member k = blockIdx.z owns the ring's replica columns k R .. k R + R - 1 of
// R_ring, reads P + k p_stride, uses gam.v[k] and writes partial row k groups + g: CTA (g, a, k) does exactly what CTA
// (g, a) of member k's own launch does.
template <bool DQN, bool GROUPED = false>
__global__ void __launch_bounds__(256)
q_td_kernel(const QDims d, const float* __restrict__ P0, const float* __restrict__ ring_s,
            const float* __restrict__ ring_s1, const int8_t* __restrict__ ring_a, const float* __restrict__ ring_r,
            const uint8_t* __restrict__ ring_done, const int32_t* __restrict__ idx, int64_t R, int batch, float gamma0,
            float inv_n, int64_t n_params, float* __restrict__ part, int64_t ld, int64_t R_ring, int64_t p_stride,
            const QMemberF gam) {
  extern __shared__ __align__(16) float qsm[];
  const int mk = GROUPED ? (int)blockIdx.z : 0;
  const float* __restrict__ P = GROUPED ? P0 + mk * p_stride : P0;
  const float gamma = GROUPED ? gam.v[mk] : gamma0;
  const int64_t Rr = GROUPED ? R_ring : R, rc0 = GROUPED ? (int64_t)mk * R : 0;
  const QTdSmem T = q_td_smem_layout(d);
  const QSmem& L = T.f;
  const int a = blockIdx.y, tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int n_s = d.n_s[a], n_a = d.n_a[a], ooff = d.obs_off[a];
  const int n_w = DQN ? d.n_w[a] : 0, n_wave = n_s - n_w;
  const int n_ft = n_w > 0 ? d.n_ft : 0;
  const int q_in = DQN ? d.n_h : n_s, h1w = d.n_fc + n_ft;
  float *sW1 = qsm + L.w1, *sB1 = qsm + L.b1, *sWt = qsm + L.wt, *sW2 = qsm + T.w2p, *sB2 = qsm + L.b2;
  float *sWq = qsm + L.wq, *sBq = qsm + L.bq, *sS = qsm + L.s, *sH1 = qsm + L.h1, *sH2 = qsm + L.h2, *sQ = qsm + L.q;
  float *gW1 = qsm + T.gw1, *gB1 = qsm + T.gb1, *gWt = qsm + T.gwt, *gW2 = qsm + T.gw2, *gB2 = qsm + T.gb2;
  float *gWq = qsm + T.gwq, *gBq = qsm + T.gbq, *sTq = qsm + T.tq, *sDq = qsm + T.dq;
  int* sAct = reinterpret_cast<int*>(qsm + T.act);

  if (DQN) {
    for (int i = tid; i < n_wave * d.n_fc; i += 256) { sW1[i] = P[d.off_fcw_w[a] + i]; gW1[i] = 0.f; }
    for (int i = tid; i < h1w; i += 256) {
      sB1[i] = i < d.n_fc ? P[d.off_fcw_b[a] + i] : P[d.off_fct_b[a] + i - d.n_fc];
      gB1[i] = 0.f;
    }
    for (int i = tid; i < n_w * n_ft; i += 256) { sWt[i] = P[d.off_fct_w[a] + i]; gWt[i] = 0.f; }
    for (int i = tid; i < h1w * d.n_h; i += 256) {
      const int k = i / d.n_h, c = i - k * d.n_h;
      sW2[k * T.ld2 + c] = P[d.off_fc0_w[a] + i];
      gW2[i] = 0.f;
    }
    for (int i = tid; i < d.n_h; i += 256) { sB2[i] = P[d.off_fc0_b[a] + i]; gB2[i] = 0.f; }
  }
  for (int i = tid; i < q_in * QT_NA; i += 256) {
    const int k = i / QT_NA, j = i - k * QT_NA;
    sWq[i] = j < n_a ? P[d.off_q_w[a] + (int64_t)k * n_a + j] : 0.f;
    gWq[i] = 0.f;
  }
  for (int i = tid; i < QT_NA; i += 256) { sBq[i] = i < n_a ? P[d.off_q_b[a] + i] : 0.f; gBq[i] = 0.f; }

  float loss = 0.f, qsum = 0.f, tqsum = 0.f;          // threads < QT_ROWS: their rows' e^2, q(s)[act] and tq
  const int64_t rows = R * batch, n_tiles = (rows + QT_ROWS - 1) / QT_ROWS;
  const int32_t* ia = idx + (int64_t)a * rows;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t m0 = tile * QT_ROWS;
    for (int pass = 0; pass < 2; ++pass) {           // 0: s1 -> TD target, 1: s -> q and the activations kept
      const float* src = pass ? ring_s : ring_s1;
      __syncthreads();
      for (int i = tid; i < QT_ROWS * n_s; i += 256) {
        const int row = i / n_s, k = i - row * n_s;
        const int64_t m = m0 + row;
        float x = 0.f;
        if (m < rows) {
          const int64_t r = m / batch;
          x = __ldg(src + ((int64_t)ia[m] * Rr + rc0 + r) * d.n_obs + ooff + k);
        }
        sS[k * QT_LD + row] = x;
      }
      __syncthreads();
      q_tile_forward<DQN>(d, sS, sW1, sB1, sWt, sW2, T.ld2, sB2, sWq, sBq, sH1, sH2, sQ, n_wave, n_w, n_ft, q_in, tid,
                          ty, tx);
      __syncthreads();
      if (tid < QT_ROWS) {
        const int64_t m = m0 + tid;
        if (pass == 0) {                              // tq = done ? r : r + gamma * max q(s1)  (torch.where, fp32 ops)
          float tq = 0.f;
          int act = -1;
          if (m < rows) {
            const int64_t r = m / batch, e = (int64_t)ia[m] * Rr + rc0 + r;
            float best = sQ[tid * QT_NA];
            for (int j = 1; j < n_a; ++j) best = fmaxf(best, sQ[tid * QT_NA + j]);
            const float rw = ring_r[e * d.A + a];
            tq = ring_done[e] ? rw : __fadd_rn(rw, __fmul_rn(gamma, best));
            act = ring_a[e * d.A + a];
          }
          sTq[tid] = tq;
          sAct[tid] = act;
        } else {
          float dq = 0.f;
          if (m < rows) {
            const float q0 = sQ[tid * QT_NA + sAct[tid]];
            const float e = __fsub_rn(q0, sTq[tid]);
            loss = fmaf(e, e, loss);
            qsum += q0;
            tqsum += sTq[tid];
            dq = 2.f * e * inv_n;
          }
          sDq[tid] = dq;
        }
      }
    }
    __syncthreads();
    // output layer: gWq[k][j] += sum_rows in[k][row] dq[row] [act[row] == j], gBq[j] += sum_rows dq[row] [act == j]
    const float* qin = DQN ? sH2 : sS;
    for (int i = tid; i < q_in * QT_NA; i += 256) {
      const int k = i / QT_NA, j = i - k * QT_NA;
      if (j < n_a) {
        float acc = 0.f;
        for (int r = 0; r < QT_ROWS; ++r) acc = fmaf(qin[k * QT_LD + r], sAct[r] == j ? sDq[r] : 0.f, acc);
        gWq[i] += acc;
      }
    }
    if (tid < n_a) {
      float acc = 0.f;
      for (int r = 0; r < QT_ROWS; ++r) acc += sAct[r] == tid ? sDq[r] : 0.f;
      gBq[tid] += acc;
    }
    if (DQN) {
      __syncthreads();
      // dh2 = dq Wq[:, act]^T masked by h2 > 0, in place of h2
      for (int i = tid; i < d.n_h * QT_ROWS; i += 256) {
        const int c = i / QT_ROWS, r = i - c * QT_ROWS;
        const float h = sH2[c * QT_LD + r];
        sH2[c * QT_LD + r] = (h > 0.f && sAct[r] >= 0) ? sDq[r] * sWq[c * QT_NA + sAct[r]] : 0.f;
      }
      __syncthreads();
      q_wgrad<4, QT_H_MAX / 16>(sH1, h1w, sH2, d.n_h / 16, gW2, d.n_h, ty, tx);
      q_bgrad(sH2, d.n_h, gB2, tid);
      __syncthreads();
      // dh1 = dh2 W2^T masked by h1 > 0, in place of h1
      q_dense_relu<(QT_FC_MAX + QT_FT_MAX) / 16, true>(sH2, d.n_h, sW2, T.ld2, nullptr, h1w / 16, sH1, ty, tx);
      __syncthreads();
      q_wgrad<2, QT_FC_MAX / 16>(sS, n_wave, sH1, d.n_fc / 16, gW1, d.n_fc, ty, tx);
      if (n_ft > 0) q_wgrad<1, QT_FT_MAX / 16>(sS + n_wave * QT_LD, n_w, sH1 + d.n_fc * QT_LD, n_ft / 16, gWt, n_ft, ty, tx);
      q_bgrad(sH1, h1w, gB1, tid);
    }
  }
  // the CTA's loss, q and tq sums: fixed-order shuffle reductions over the 64 row threads
  if (tid < QT_ROWS) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      loss += __shfl_down_sync(0xffffffffu, loss, o);
      qsum += __shfl_down_sync(0xffffffffu, qsum, o);
      tqsum += __shfl_down_sync(0xffffffffu, tqsum, o);
    }
    if ((tid & 31) == 0) { sTq[tid >> 5] = loss; sTq[2 + (tid >> 5)] = qsum; sTq[4 + (tid >> 5)] = tqsum; }
  }
  __syncthreads();
  float* out = part + ((GROUPED ? (int64_t)mk * gridDim.x : 0) + blockIdx.x) * ld;
  if (tid == 0) {
    out[n_params + a] = (sTq[0] + sTq[1]) * inv_n;
    out[n_params + d.A + a] = (sTq[2] + sTq[3]) * inv_n;
    out[n_params + 2 * d.A + a] = (sTq[4] + sTq[5]) * inv_n;
  }
  if (DQN) {
    for (int i = tid; i < n_wave * d.n_fc; i += 256) out[d.off_fcw_w[a] + i] = gW1[i];
    for (int i = tid; i < d.n_fc; i += 256) out[d.off_fcw_b[a] + i] = gB1[i];
    for (int i = tid; i < n_w * n_ft; i += 256) out[d.off_fct_w[a] + i] = gWt[i];
    for (int i = tid; i < n_ft; i += 256) out[d.off_fct_b[a] + i] = gB1[d.n_fc + i];
    for (int i = tid; i < h1w * d.n_h; i += 256) out[d.off_fc0_w[a] + i] = gW2[i];
    for (int i = tid; i < d.n_h; i += 256) out[d.off_fc0_b[a] + i] = gB2[i];
  }
  for (int i = tid; i < q_in * n_a; i += 256) {
    const int k = i / n_a, j = i - k * n_a;
    out[d.off_q_w[a] + i] = gWq[k * QT_NA + j];
  }
  for (int i = tid; i < n_a; i += 256) out[d.off_q_b[a] + i] = gBq[i];
}

// grad[i] = sum over the partial rows g = 0, 1, .. of part[g][i], in that order (no atomics: bit-reproducible)
__global__ void q_reduce_kernel(const float* __restrict__ part, int groups, int64_t ld, float* __restrict__ grad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ld) return;
  float s = 0.f;
  for (int g = 0; g < groups; ++g) s += part[(int64_t)g * ld + i];
  grad[i] = s;
}

// Grouped form: grid (x, K); grad[k][i] = sum over member k's partial rows part[k][g][i], g = 0, 1, .. in that order
__global__ void q_reduce_g_kernel(const float* __restrict__ part, int groups, int64_t ld, float* __restrict__ grad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ld) return;
  const float* p = part + (int64_t)blockIdx.y * groups * ld;
  float s = 0.f;
  for (int g = 0; g < groups; ++g) s += p[(int64_t)g * ld + i];
  grad[(int64_t)blockIdx.y * ld + i] = s;
}

// Per agent (one CTA of 512 threads): tf.clip_by_global_norm and the TF1 Adam step of IQL.td_update
// (agents/models.py:290-302) on the agent's block [blk[a], blk[a+1]) of the flat vector, loss / norm written out, and
// with rec_out the agent's row (loss, mean q, mean tq, norm) of the round's summaries.
// GROUPED (tscl_q_adam_g): grid (A, K); member k = blockIdx.y steps P / m / v + k p_stride with grad + k (n_params + 3 A),
// lr.v[k] and clip.v[k], and writes loss / norm at + k out_stride and its rec row at + k rec_stride.
template <bool GROUPED = false>
__global__ void __launch_bounds__(512)
q_adam_kernel(float* __restrict__ P0, const float* __restrict__ grad0, float* __restrict__ m0, float* __restrict__ v0,
              const int64_t* __restrict__ blk, int64_t n_params, int A, float lr_t0, float max_norm0,
              float* __restrict__ loss_out0, float* __restrict__ norm_out0, float* __restrict__ rec_out0,
              int64_t p_stride, int64_t out_stride, int64_t rec_stride, const QMemberF lr, const QMemberF clip) {
  __shared__ float red[512];
  const int a = blockIdx.x, tid = threadIdx.x, mk = GROUPED ? (int)blockIdx.y : 0;
  float* __restrict__ P = GROUPED ? P0 + mk * p_stride : P0;
  float* __restrict__ m = GROUPED ? m0 + mk * p_stride : m0;
  float* __restrict__ v = GROUPED ? v0 + mk * p_stride : v0;
  const float* __restrict__ grad = GROUPED ? grad0 + mk * (n_params + 3 * A) : grad0;
  float* __restrict__ loss_out = GROUPED ? loss_out0 + mk * out_stride : loss_out0;
  float* __restrict__ norm_out = GROUPED ? norm_out0 + mk * out_stride : norm_out0;
  float* __restrict__ rec_out = GROUPED && rec_out0 ? rec_out0 + mk * rec_stride : rec_out0;
  const float lr_t = GROUPED ? lr.v[mk] : lr_t0, max_norm = GROUPED ? clip.v[mk] : max_norm0;
  const int64_t b0 = blk[a], b1 = blk[a + 1];
  float ss = 0.f;
  for (int64_t i = b0 + tid; i < b1; i += 512) ss = fmaf(grad[i], grad[i], ss);
  red[tid] = ss;
  __syncthreads();
  for (int o = 256; o > 0; o >>= 1) {
    if (tid < o) red[tid] += red[tid + o];
    __syncthreads();
  }
  const float norm = sqrtf(red[0]);
  const float scale = max_norm > 0.f ? __fdiv_rn(max_norm, fmaxf(norm, max_norm)) : 1.f;
  const float c1 = (float)(1.0 - 0.9), c2 = (float)(1.0 - 0.999);
  for (int64_t i = b0 + tid; i < b1; i += 512) {
    const float g = max_norm > 0.f ? __fmul_rn(grad[i], scale) : grad[i];
    const float mi = __fadd_rn(m[i], __fmul_rn(__fsub_rn(g, m[i]), c1));
    const float vi = __fadd_rn(v[i], __fmul_rn(__fsub_rn(__fmul_rn(g, g), v[i]), c2));
    m[i] = mi;
    v[i] = vi;
    P[i] = __fsub_rn(P[i], __fdiv_rn(__fmul_rn(lr_t, mi), __fadd_rn(__fsqrt_rn(vi), 1e-8f)));
  }
  if (tid == 0) {
    loss_out[a] = grad[n_params + a];
    norm_out[a] = norm;
    if (rec_out) {
      float* r = rec_out + 4 * a;
      r[0] = grad[n_params + a]; r[1] = grad[n_params + A + a]; r[2] = grad[n_params + 2 * A + a]; r[3] = norm;
    }
  }
}

// IQL.add_transition's reward (r / reward_norm, then clipped) and the post-step done into one replay slot, and the
// episode's global-reward sum.  GROUPED (tscl_q_transition_g): row r belongs to member r / R_m and takes its
// reward_norm / reward_clip from norms / clips.
template <bool GROUPED = false>
__global__ void q_transition_kernel(const float* __restrict__ rew, int64_t RA, float reward_norm0, float reward_clip0,
                                    float* __restrict__ ring_r, const float* __restrict__ grew, float* __restrict__ rew_acc,
                                    uint8_t* __restrict__ ring_done, int64_t R, int done, int64_t R_m,
                                    const QMemberF norms, const QMemberF clips) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < RA) {
    const int mk = GROUPED ? (int)(i / (RA / R) / R_m) : 0;
    const float reward_norm = GROUPED ? norms.v[mk] : reward_norm0, reward_clip = GROUPED ? clips.v[mk] : reward_clip0;
    float x = rew[i];
    if (reward_norm != 0.f) x = __fdiv_rn(x, reward_norm);
    if (reward_clip != 0.f) x = fminf(fmaxf(x, -reward_clip), reward_clip);
    ring_r[i] = x;
  }
  if (i < R) {
    ring_done[i] = (uint8_t)done;
    if (rew_acc) rew_acc[i] += grew[i];
  }
}

// ================================================================================================
template <class T>
static int qup(tscl_qhandle* h, const T* src, size_t n, const T** dst) {
  void* p = nullptr;
  LCK(cudaMalloc(&p, n ? n * sizeof(T) : 16));
  if (n) LCK(cudaMemcpy(p, src, n * sizeof(T), cudaMemcpyHostToDevice));
  h->owned.push_back(p);
  *dst = static_cast<const T*>(p);
  return 0;
}

extern "C" int tscl_q_create(const tscl_qdims* x, int32_t device, tscl_qhandle** out) {
  if (!x || !out || x->n_agents <= 0 || x->n_obs <= 0 || x->max_na <= 0 || !x->obs_off || !x->n_s || !x->n_w || !x->n_a ||
      !x->off_q_w || !x->off_q_b)
    return tsc_set_error("tscl_q_create: bad argument");
  if (x->model != 0 && x->model != 1) return tsc_set_error("tscl_q_create: model must be 0 (lr) or 1 (dqn)");
  if (x->max_na > QT_NA) return tsc_set_error("tscl_q_create: max_na > 8");
  const bool dqn = x->model == 1;
  const int A = x->n_agents;
  QDims d{};
  int any_w = 0;
  for (int a = 0; a < A; ++a) {
    if (x->n_a[a] < 1 || x->n_a[a] > x->max_na || x->n_s[a] < 1 || x->obs_off[a] < 0 ||
        x->obs_off[a] + x->n_s[a] > x->n_obs || x->n_w[a] < 0 || x->n_w[a] >= x->n_s[a])
      return tsc_set_error("tscl_q_create: agent " + std::to_string(a) + " has an inconsistent observation / action shape");
    d.s_max = std::max(d.s_max, (int)x->n_s[a]);
    if (dqn) {
      d.wave_max = std::max(d.wave_max, (int)(x->n_s[a] - x->n_w[a]));
      d.w_max = std::max(d.w_max, (int)x->n_w[a]);
      any_w |= x->n_w[a] > 0;
    }
  }
  if (dqn) {
    if (!x->off_fcw_w || !x->off_fcw_b || !x->off_fc0_w || !x->off_fc0_b || (any_w && (!x->off_fct_w || !x->off_fct_b)))
      return tsc_set_error("tscl_q_create: missing dqn offsets");
    if (x->n_fc < 16 || x->n_fc > QT_FC_MAX || x->n_fc % 16 || x->n_h < 16 || x->n_h > QT_H_MAX || x->n_h % 16 ||
        (any_w && (x->n_ft < 16 || x->n_ft > QT_FT_MAX || x->n_ft % 16)))
      return tsc_set_error("tscl_q_create: dqn widths must be multiples of 16 with num_fc <= 128, num_fc/4 <= 32, "
                           "num_h <= 64");
    d.n_fc = x->n_fc; d.n_ft = any_w ? x->n_ft : 0; d.n_h = x->n_h;
    d.in2_max = d.n_fc + d.n_ft;
    d.q_in = d.n_h;
  } else {
    d.q_in = d.s_max;
  }
  d.A = A; d.n_obs = x->n_obs; d.max_na = x->max_na; d.model = x->model;
  LCK(cudaSetDevice(device));
  tscl_qhandle* h = new tscl_qhandle();
  h->device = device;
  int rc = 0;
  rc |= qup(h, x->obs_off, A, &d.obs_off); rc |= qup(h, x->n_s, A, &d.n_s); rc |= qup(h, x->n_w, A, &d.n_w);
  rc |= qup(h, x->n_a, A, &d.n_a); rc |= qup(h, x->off_q_w, A, &d.off_q_w); rc |= qup(h, x->off_q_b, A, &d.off_q_b);
  if (dqn) {
    rc |= qup(h, x->off_fcw_w, A, &d.off_fcw_w); rc |= qup(h, x->off_fcw_b, A, &d.off_fcw_b);
    rc |= qup(h, x->off_fc0_w, A, &d.off_fc0_w); rc |= qup(h, x->off_fc0_b, A, &d.off_fc0_b);
    if (any_w) { rc |= qup(h, x->off_fct_w, A, &d.off_fct_w); rc |= qup(h, x->off_fct_b, A, &d.off_fct_b); }
  }
  // agent blocks of the flat vector, in agent order (QLayout): the per-agent clip + Adam ranges
  std::vector<int64_t> blk(A + 1);
  for (int a = 0; a < A; ++a) blk[a] = dqn ? x->off_fcw_w[a] : x->off_q_w[a];
  blk[A] = x->n_params;
  for (int a = 0; a < A; ++a)
    if (blk[a] < 0 || blk[a] >= blk[a + 1]) rc = tsc_set_error("tscl_q_create: agent blocks are not in agent order");
  if (!rc) rc |= qup(h, blk.data(), A + 1, &h->blk);
  if (rc) { tscl_q_destroy(h); return -1; }
  h->d = d;
  h->n_params = x->n_params;
  h->smem = (size_t)q_smem_layout(d).total * sizeof(float);
  int optin = 0;
  LCK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  LCK(cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, device));
  if (h->smem > (size_t)optin) {
    tscl_q_destroy(h);
    return tsc_set_error("tscl_q_create: the weights and tiles of one agent need more shared memory than a CTA has");
  }
  // the shared-memory limit belongs to the kernel, not the handle: the opt-in maximum, so that a handle created later
  // for a smaller layout does not lower it below what a live handle's launches need
  const void* fn = dqn ? (const void*)q_fwd_kernel<true> : (const void*)q_fwd_kernel<false>;
  LCK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
  LCK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&h->ctas_per_sm, fn, 256, h->smem));
  if (h->ctas_per_sm < 1) h->ctas_per_sm = 1;
  const void* ex = dqn ? (const void*)q_fwd_kernel<true, true> : (const void*)q_fwd_kernel<false, true>;
  LCK(cudaFuncSetAttribute(ex, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
  const void* fg = dqn ? (const void*)q_fwd_g_kernel<true> : (const void*)q_fwd_g_kernel<false>;
  LCK(cudaFuncSetAttribute(fg, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
  const void* eg = dqn ? (const void*)q_fwd_g_kernel<true, true> : (const void*)q_fwd_g_kernel<false, true>;
  LCK(cudaFuncSetAttribute(eg, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
  const size_t td_smem = (size_t)q_td_smem_layout(d).total * sizeof(float);
  if (td_smem <= (size_t)optin) {
    const void* td = dqn ? (const void*)q_td_kernel<true> : (const void*)q_td_kernel<false>;
    LCK(cudaFuncSetAttribute(td, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
    LCK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&h->td_ctas_per_sm, td, 256, td_smem));
    const void* tg = dqn ? (const void*)q_td_kernel<true, true> : (const void*)q_td_kernel<false, true>;
    LCK(cudaFuncSetAttribute(tg, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
    if (h->td_ctas_per_sm < 1) h->td_ctas_per_sm = 1;
    h->td_smem = td_smem;
  }
  *out = h;
  return 0;
}

extern "C" int tscl_q_destroy(tscl_qhandle* h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  for (void* p : h->owned) cudaFree(p);
  if (h->part) cudaFree(h->part);
  if (h->part_g) cudaFree(h->part_g);
  delete h;
  return 0;
}

extern "C" int tscl_q_info(tscl_qhandle* h, int64_t* fwd_smem_bytes, int64_t* td_smem_bytes) {
  if (!h || !fwd_smem_bytes || !td_smem_bytes) return tsc_set_error("tscl_q_info: bad argument");
  *fwd_smem_bytes = (int64_t)h->smem;
  *td_smem_bytes = (int64_t)h->td_smem;
  return 0;
}

extern "C" int tscl_q_step(tscl_qhandle* h, const float* params, const float* obs, int64_t R, float* q, int32_t* act,
                           int32_t mode, uint64_t seed, int64_t step, int64_t replica0, int64_t* bad_flag, void* stream) {
  if (!h || !params || !obs || !q || !act || R <= 0 || replica0 < 0 || (mode != 0 && mode != 1))
    return tsc_set_error("tscl_q_step: bad argument");
  LCK(cudaSetDevice(h->device));
  const int64_t n_tiles = (R + QT_ROWS - 1) / QT_ROWS;
  // enough CTAs to fill the device once, spread over the agents; each walks its agent's tiles with the weights resident
  int64_t groups = ((int64_t)h->n_sm * h->ctas_per_sm + h->d.A - 1) / h->d.A;
  if (groups > n_tiles) groups = n_tiles;
  dim3 grid((unsigned)groups, (unsigned)h->d.A);
  unsigned long long* bad = reinterpret_cast<unsigned long long*>(bad_flag);
  const uint32_t lo = (uint32_t)(seed & 0xFFFFFFFFu), hi = (uint32_t)(seed >> 32);
  if (h->d.model == 1)
    q_fwd_kernel<true><<<grid, 256, h->smem, (cudaStream_t)stream>>>(h->d, params, obs, R, q, act, mode, lo, hi,
                                                                      (uint32_t)step, replica0, bad, 0.f, nullptr,
                                                                      nullptr);
  else
    q_fwd_kernel<false><<<grid, 256, h->smem, (cudaStream_t)stream>>>(h->d, params, obs, R, q, act, mode, lo, hi,
                                                                       (uint32_t)step, replica0, bad, 0.f, nullptr,
                                                                       nullptr);
  LCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_q_step_g(tscl_qhandle* h, const float* params, int64_t p_stride, const float* obs, int32_t K,
                             const int64_t* rows, int64_t R, float* q, int32_t* act, int32_t mode, const uint64_t* seeds,
                             int64_t step, int64_t* bad_flags, void* stream) {
  if (!h || !params || !obs || !rows || !seeds || !q || !act || K < 1 || K > 65535 || R < K || (mode != 0 && mode != 1) ||
      (K > 1 && p_stride < h->n_params))
    return tsc_set_error("tscl_q_step_g: bad argument");
  LCK(cudaSetDevice(h->device));
  // a member has at most ceil(R / 64) tiles; CTAs past a member's tiles return at once
  const int64_t max_tiles = (R + QT_ROWS - 1) / QT_ROWS;
  int64_t groups = ((int64_t)h->n_sm * h->ctas_per_sm + (int64_t)h->d.A * K - 1) / ((int64_t)h->d.A * K);
  if (groups > max_tiles) groups = max_tiles;
  dim3 grid((unsigned)groups, (unsigned)h->d.A, (unsigned)K);
  unsigned long long* bad = reinterpret_cast<unsigned long long*>(bad_flags);
  if (h->d.model == 1)
    q_fwd_g_kernel<true><<<grid, 256, h->smem, (cudaStream_t)stream>>>(h->d, params, p_stride, obs, rows, q, act, mode,
                                                                        seeds, (uint32_t)step, bad, QMemberF{}, 0,
                                                                        nullptr, nullptr);
  else
    q_fwd_g_kernel<false><<<grid, 256, h->smem, (cudaStream_t)stream>>>(h->d, params, p_stride, obs, rows, q, act, mode,
                                                                         seeds, (uint32_t)step, bad, QMemberF{}, 0,
                                                                         nullptr, nullptr);
  LCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_q_explore(tscl_qhandle* h, const float* params, const float* obs, int64_t R, float* q, int32_t* act,
                              float eps, uint64_t seed, int64_t step, int64_t replica0, float* ring_s, int8_t* ring_a,
                              void* stream) {
  if (!h || !params || !obs || !q || !act || R <= 0 || replica0 < 0) return tsc_set_error("tscl_q_explore: bad argument");
  LCK(cudaSetDevice(h->device));
  const int64_t n_tiles = (R + QT_ROWS - 1) / QT_ROWS;
  int64_t groups = ((int64_t)h->n_sm * h->ctas_per_sm + h->d.A - 1) / h->d.A;
  if (groups > n_tiles) groups = n_tiles;
  dim3 grid((unsigned)groups, (unsigned)h->d.A);
  const uint32_t lo = (uint32_t)(seed & 0xFFFFFFFFu), hi = (uint32_t)(seed >> 32);
  if (h->d.model == 1)
    q_fwd_kernel<true, true><<<grid, 256, h->smem, (cudaStream_t)stream>>>(h->d, params, obs, R, q, act, 0, lo, hi,
                                                                          (uint32_t)step, replica0, nullptr, eps, ring_s,
                                                                          ring_a);
  else
    q_fwd_kernel<false, true><<<grid, 256, h->smem, (cudaStream_t)stream>>>(h->d, params, obs, R, q, act, 0, lo, hi,
                                                                           (uint32_t)step, replica0, nullptr, eps, ring_s,
                                                                           ring_a);
  LCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_q_sample(tscl_qhandle* h, int64_t R, int32_t batch, int32_t size, uint64_t seed, int64_t update,
                             int32_t round, int64_t replica0, int32_t* idx, void* stream) {
  if (!h || !idx || R <= 0 || batch <= 0 || size < batch || replica0 < 0 || round < 0)
    return tsc_set_error("tscl_q_sample: bad argument (the ring must hold at least batch entries)");
  LCK(cudaSetDevice(h->device));
  const int64_t n = (int64_t)h->d.A * R;
  q_sample_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      h->d.A, R, batch, size, (uint32_t)(seed & 0xFFFFFFFFu), (uint32_t)(seed >> 32), (uint32_t)update, (uint32_t)round,
      replica0, idx);
  LCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_q_td(tscl_qhandle* h, const float* params, const float* ring_s, const float* ring_s1,
                         const int8_t* ring_a, const float* ring_r, const uint8_t* ring_done, const int32_t* idx, int64_t R,
                         int32_t batch, float gamma, float inv_n, float* grad, void* stream) {
  if (!h || !params || !ring_s || !ring_s1 || !ring_a || !ring_r || !ring_done || !idx || !grad || R <= 0 || batch <= 0)
    return tsc_set_error("tscl_q_td: bad argument");
  if (!h->td_smem)
    return tsc_set_error("tscl_q_td: the weights, gradients and tiles of one agent need more shared memory than a CTA has");
  LCK(cudaSetDevice(h->device));
  const int A = h->d.A;
  const int64_t ld = h->n_params + 3 * A, n_tiles = (R * batch + QT_ROWS - 1) / QT_ROWS;
  const int64_t max_groups = ((int64_t)h->n_sm * h->td_ctas_per_sm + A - 1) / A;
  int64_t groups = max_groups < n_tiles ? max_groups : n_tiles;
  if (!h->part) LCK(cudaMalloc(&h->part, (size_t)max_groups * ld * sizeof(float)));
  dim3 grid((unsigned)groups, (unsigned)A);
  if (h->d.model == 1)
    q_td_kernel<true><<<grid, 256, h->td_smem, (cudaStream_t)stream>>>(h->d, params, ring_s, ring_s1, ring_a, ring_r,
                                                                        ring_done, idx, R, batch, gamma, inv_n,
                                                                        h->n_params, h->part, ld, 0, 0, QMemberF{});
  else
    q_td_kernel<false><<<grid, 256, h->td_smem, (cudaStream_t)stream>>>(h->d, params, ring_s, ring_s1, ring_a, ring_r,
                                                                         ring_done, idx, R, batch, gamma, inv_n,
                                                                         h->n_params, h->part, ld, 0, 0, QMemberF{});
  LCK(cudaGetLastError());
  q_reduce_kernel<<<(unsigned)((ld + 255) / 256), 256, 0, (cudaStream_t)stream>>>(h->part, (int)groups, ld, grad);
  LCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_q_adam(tscl_qhandle* h, float* params, const float* grad, float* adam_m, float* adam_v, float lr_t,
                           float max_grad_norm, float* loss_out, float* norm_out, float* rec_out, void* stream) {
  if (!h || !params || !grad || !adam_m || !adam_v || !loss_out || !norm_out) return tsc_set_error("tscl_q_adam: bad argument");
  LCK(cudaSetDevice(h->device));
  q_adam_kernel<<<h->d.A, 512, 0, (cudaStream_t)stream>>>(params, grad, adam_m, adam_v, h->blk, h->n_params, h->d.A,
                                                          lr_t, max_grad_norm, loss_out, norm_out, rec_out, 0, 0, 0,
                                                          QMemberF{}, QMemberF{});
  LCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_q_transition(tscl_qhandle* h, const float* rew, int64_t R, float reward_norm, float reward_clip,
                                 float* ring_r, const float* grew, float* rew_acc, uint8_t* ring_done, int32_t done,
                                 void* stream) {
  if (!h || !rew || !ring_r || !ring_done || R <= 0 || (rew_acc && !grew)) return tsc_set_error("tscl_q_transition: bad argument");
  LCK(cudaSetDevice(h->device));
  const int64_t RA = R * h->d.A;
  q_transition_kernel<<<(unsigned)((RA + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      rew, RA, reward_norm, reward_clip, ring_r, grew, rew_acc, ring_done, R, done, 0, QMemberF{}, QMemberF{});
  LCK(cudaGetLastError());
  return 0;
}

// ================================================================================================
// Grouped training (a population or sweep of K members, R_m replicas each, in one lock-step of K R_m replicas)

extern "C" int tscl_q_explore_g(tscl_qhandle* h, const float* params, int64_t p_stride, const float* obs, int32_t K,
                                const int64_t* rows, int64_t R, float* q, int32_t* act, const float* eps, uint64_t seed,
                                int64_t step, float* ring_s, int8_t* ring_a, void* stream) {
  if (!h || !params || !obs || !rows || !q || !act || !eps || K < 1 || K > QG_MAX || R < K ||
      (K > 1 && p_stride < h->n_params))
    return tsc_set_error("tscl_q_explore_g: bad argument (1 <= K <= 64 members)");
  LCK(cudaSetDevice(h->device));
  const int64_t max_tiles = (R + QT_ROWS - 1) / QT_ROWS;
  int64_t groups = ((int64_t)h->n_sm * h->ctas_per_sm + (int64_t)h->d.A * K - 1) / ((int64_t)h->d.A * K);
  if (groups > max_tiles) groups = max_tiles;
  dim3 grid((unsigned)groups, (unsigned)h->d.A, (unsigned)K);
  const QMemberF e = q_member_f(eps, K);
  if (h->d.model == 1)
    q_fwd_g_kernel<true, true><<<grid, 256, h->smem, (cudaStream_t)stream>>>(
        h->d, params, p_stride, obs, rows, q, act, 0, nullptr, (uint32_t)step, nullptr, e, seed, ring_s, ring_a);
  else
    q_fwd_g_kernel<false, true><<<grid, 256, h->smem, (cudaStream_t)stream>>>(
        h->d, params, p_stride, obs, rows, q, act, 0, nullptr, (uint32_t)step, nullptr, e, seed, ring_s, ring_a);
  LCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_q_td_g(tscl_qhandle* h, const float* params, int64_t p_stride, int32_t K, const float* ring_s,
                           const float* ring_s1, const int8_t* ring_a, const float* ring_r, const uint8_t* ring_done,
                           const int32_t* idx, int64_t R_m, int32_t batch, const float* gamma, float inv_n, float* grad,
                           void* stream) {
  if (!h || !params || !ring_s || !ring_s1 || !ring_a || !ring_r || !ring_done || !idx || !gamma || !grad || R_m <= 0 ||
      batch <= 0 || K < 1 || K > QG_MAX || (K > 1 && p_stride < h->n_params))
    return tsc_set_error("tscl_q_td_g: bad argument (1 <= K <= 64 members)");
  if (!h->td_smem)
    return tsc_set_error("tscl_q_td_g: the weights, gradients and tiles of one agent need more shared memory than a CTA "
                         "has");
  LCK(cudaSetDevice(h->device));
  const int A = h->d.A;
  // member k's partial rows are cut as its own tscl_q_td launch on R_m replicas cuts them
  const int64_t ld = h->n_params + 3 * A, n_tiles = (R_m * batch + QT_ROWS - 1) / QT_ROWS;
  const int64_t max_groups = ((int64_t)h->n_sm * h->td_ctas_per_sm + A - 1) / A;
  const int64_t groups = max_groups < n_tiles ? max_groups : n_tiles;
  if (h->part_g_k < K) {
    if (h->part_g) LCK(cudaFree(h->part_g));
    h->part_g = nullptr;
    h->part_g_k = 0;
    LCK(cudaMalloc(&h->part_g, (size_t)K * max_groups * ld * sizeof(float)));
    h->part_g_k = K;
  }
  dim3 grid((unsigned)groups, (unsigned)A, (unsigned)K);
  const QMemberF g = q_member_f(gamma, K);
  if (h->d.model == 1)
    q_td_kernel<true, true><<<grid, 256, h->td_smem, (cudaStream_t)stream>>>(
        h->d, params, ring_s, ring_s1, ring_a, ring_r, ring_done, idx, R_m, batch, 0.f, inv_n, h->n_params, h->part_g,
        ld, (int64_t)K * R_m, p_stride, g);
  else
    q_td_kernel<false, true><<<grid, 256, h->td_smem, (cudaStream_t)stream>>>(
        h->d, params, ring_s, ring_s1, ring_a, ring_r, ring_done, idx, R_m, batch, 0.f, inv_n, h->n_params, h->part_g,
        ld, (int64_t)K * R_m, p_stride, g);
  LCK(cudaGetLastError());
  q_reduce_g_kernel<<<dim3((unsigned)((ld + 255) / 256), (unsigned)K), 256, 0, (cudaStream_t)stream>>>(
      h->part_g, (int)groups, ld, grad);
  LCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_q_adam_g(tscl_qhandle* h, int32_t K, float* params, int64_t p_stride, const float* grad,
                             float* adam_m, float* adam_v, const float* lr_t, const float* max_grad_norm, float* loss_out,
                             float* norm_out, int64_t out_stride, float* rec_out, int64_t rec_stride, void* stream) {
  if (!h || !params || !grad || !adam_m || !adam_v || !lr_t || !max_grad_norm || !loss_out || !norm_out || K < 1 ||
      K > QG_MAX || (K > 1 && (p_stride < h->n_params || out_stride < h->d.A || (rec_out && rec_stride < 4 * h->d.A))))
    return tsc_set_error("tscl_q_adam_g: bad argument (1 <= K <= 64 members)");
  LCK(cudaSetDevice(h->device));
  q_adam_kernel<true><<<dim3((unsigned)h->d.A, (unsigned)K), 512, 0, (cudaStream_t)stream>>>(
      params, grad, adam_m, adam_v, h->blk, h->n_params, h->d.A, 0.f, 0.f, loss_out, norm_out, rec_out, p_stride,
      out_stride, rec_stride, q_member_f(lr_t, K), q_member_f(max_grad_norm, K));
  LCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_q_transition_g(tscl_qhandle* h, const float* rew, int32_t K, int64_t R_m, const float* reward_norm,
                                   const float* reward_clip, float* ring_r, const float* grew, float* rew_acc,
                                   uint8_t* ring_done, int32_t done, void* stream) {
  if (!h || !rew || !ring_r || !ring_done || !reward_norm || !reward_clip || R_m <= 0 || K < 1 || K > QG_MAX ||
      (rew_acc && !grew))
    return tsc_set_error("tscl_q_transition_g: bad argument (1 <= K <= 64 members)");
  LCK(cudaSetDevice(h->device));
  const int64_t R = (int64_t)K * R_m, RA = R * h->d.A;
  q_transition_kernel<true><<<(unsigned)((RA + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      rew, RA, 0.f, 0.f, ring_r, grew, rew_acc, ring_done, R, done, R_m, q_member_f(reward_norm, K),
      q_member_f(reward_clip, K));
  LCK(cudaGetLastError());
  return 0;
}
