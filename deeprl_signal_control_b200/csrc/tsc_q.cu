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

struct tscl_qhandle {
  int device = 0;
  QDims d{};
  std::vector<void*> owned;
  size_t smem = 0;
  int ctas_per_sm = 1, n_sm = 1;
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

__device__ __forceinline__ uint32_t qmix32(uint32_t h) {   // the counter hash of the A2C sampling kernels
  h ^= h >> 16; h *= 0x7feb352dU; h ^= h >> 15; h *= 0x846ca68bU; h ^= h >> 16;
  return h;
}

// One hidden layer on a 64-row tile: out[c][row] = relu(sum_k in[k][row] W[k][c] + b[c]) for the columns c = tx + 16 j,
// j < ncol (ncol <= NJ), k < K.  `in` / `out` column-major with pitch QT_LD; W row-major with `ldw` columns.
template <int NJ>
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
        const float wj = w[16 * j];
        acc[0][j] = fmaf(x.x, wj, acc[0][j]); acc[1][j] = fmaf(x.y, wj, acc[1][j]);
        acc[2][j] = fmaf(x.z, wj, acc[2][j]); acc[3][j] = fmaf(x.w, wj, acc[3][j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    if (j < ncol) {
      const float bj = b[tx + 16 * j];
      *reinterpret_cast<float4*>(out + (tx + 16 * j) * QT_LD + ty * 4) =
          make_float4(fmaxf(acc[0][j] + bj, 0.f), fmaxf(acc[1][j] + bj, 0.f), fmaxf(acc[2][j] + bj, 0.f),
                      fmaxf(acc[3][j] + bj, 0.f));
    }
  }
}

// grid (groups, A), 256 threads.  DQN = false: LRQPolicy, true: DeepQPolicy.
template <bool DQN>
__global__ void __launch_bounds__(256)
q_fwd_kernel(const QDims d, const float* __restrict__ P, const float* __restrict__ obs, int64_t R,
             float* __restrict__ q, int32_t* __restrict__ act, int mode, uint32_t seed_lo, uint32_t seed_hi,
             uint32_t step, int64_t replica0, unsigned long long* __restrict__ bad) {
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
  if (rc) { tscl_q_destroy(h); return -1; }
  h->d = d;
  h->smem = (size_t)q_smem_layout(d).total * sizeof(float);
  int optin = 0;
  LCK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  LCK(cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, device));
  if (h->smem > (size_t)optin) {
    tscl_q_destroy(h);
    return tsc_set_error("tscl_q_create: the weights and tiles of one agent need more shared memory than a CTA has");
  }
  const void* fn = dqn ? (const void*)q_fwd_kernel<true> : (const void*)q_fwd_kernel<false>;
  LCK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem));
  LCK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&h->ctas_per_sm, fn, 256, h->smem));
  if (h->ctas_per_sm < 1) h->ctas_per_sm = 1;
  *out = h;
  return 0;
}

extern "C" int tscl_q_destroy(tscl_qhandle* h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  for (void* p : h->owned) cudaFree(p);
  delete h;
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
                                                                      (uint32_t)step, replica0, bad);
  else
    q_fwd_kernel<false><<<grid, 256, h->smem, (cudaStream_t)stream>>>(h->d, params, obs, R, q, act, mode, lo, hi,
                                                                       (uint32_t)step, replica0, bad);
  LCK(cudaGetLastError());
  return 0;
}
