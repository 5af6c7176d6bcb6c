// tsc_policy_tc.cu — fused per-control-step policy forward and the learner's GEMMs on the Hopper tensor cores (sm_90a).
//
// Policy forward v1 (tscl_policy_step; the shipping v2 kernel, warp-specialised with register accumulators, is described
// at policy_step_tc2_kernel).  One persistent CTA (1 per SM, up to ~223 KB smem) walks (unit, 128-replica tile) work items:
//   1. fc front end (agents/policies.py:191-201): relu(fc) of the observation slice, written as bf16 straight into
//      the A-operand tile in shared memory (K-major, no swizzle), followed by the previous hidden state h (masked by
//      the pre-decision done flag, agents/utils.py:104-105);
//   2. warps 0-7 (two warpgroups, 64 rows each) run wgmma.mma_async m64nNk16 (bf16 x bf16 -> fp32) against the packed
//      [Wx;Wh] operand that stays resident in shared memory, and store the accumulators to the CTA's accumulator tile;
//   3. epilogue: every thread owns one replica row and a group of hidden units: the four gate pre-activations, bias,
//      LSTM cell (agents/utils.py:106-113), state write-back, head dot products (agents/policies.py:18-26), then
//      softmax / value / categorical sample (utils.py:155-157) for the row.
// Replaces per step: fc_embed_kernel + library GEMM + lstm_seq_fwd_kernel(T=1) + heads_kernel.
//
// Operand layouts (bytes, 16-byte "core rows", no swizzle; canonical ((8,n),2):((1,SBO),LBO)):
//   A tile  [KC][128 rows][16 B]   : LBO = 2048 (next K chunk of 8 bf16), SBO = 128 (next 8 rows)
//   B tile  [KC][256 cols][16 B]   : LBO = 4096,                          SBO = 128
#include <cuda.h>
#include <cstdlib>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/tsc_learn.h"

int tsc_set_error(const std::string& m);
#define PCK(call)                                                                  \
  do {                                                                             \
    cudaError_t e__ = (call);                                                      \
    if (e__ != cudaSuccess) return tsc_set_error(std::string(#call) + ": " + cudaGetErrorString(e__)); \
  } while (0)

struct DDimsTC {   // mirror of DDims in tsc_learn.cu (kept in sync by tscl_handle)
  int A, n_obs, max_na, fw, ff, ft, h, dx;
  const int32_t *obs_off, *n_wave, *n_wait, *n_fp, *n_a;
  const int64_t *off_fcw_w, *off_fcw_b, *off_fcf_w, *off_fcf_b, *off_fct_w, *off_fct_b;
  int64_t off_wx, off_wh, off_bl, off_wo, off_bo, n_params;
  int kw, ones_slot;
};
const DDimsTC* tscl_dims_of(tscl_handle* h);   // defined in tsc_learn.cu
int tscl_device_of(tscl_handle* h);
float* tscl_acc_tiles(tscl_handle* h, void* stream, size_t bytes);   // defined in tsc_learn.cu

#define TC_M 128
#define TC_N 256
#define TC_H 64
#define TC_THREADS 256
#define TC_STAGE_ROWS 16
#define TC_KW 32
#define TC_KF 16
#define TC_KT 16
#define TC_KTOT (TC_KW + TC_KF + TC_KT)

// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// ---- Hopper tensor cores ------------------------------------------------------------------------------
// wgmma.mma_async: a warpgroup (4 warps) computes a 64-row slab of a product whose operands sit in shared memory,
// described by matrix descriptors (core matrices of 8 rows x 16 bytes).  The two warpgroups of warps 0-7 cover the
// 128 rows of a tile.  Their fp32 accumulator fragments are stored to the CTA's accumulator tile, 128 rows x ACC_COLS
// fp32 in global memory (one tile per CTA and stream, see acc_tiles(); the tile of a CTA is written and read back by
// the same SM within microseconds, so the round trip normally stays in L1/L2), which the row-per-thread epilogues read
// back at address (row base << 16) + column, row = row base + lane.  This keeps the epilogues' thread = row mapping
// (v1 policy forward, BPTT, fp32 weight gradients); the other kernels keep their fragments in registers.
#define ACC_COLS 512
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)((lbo >> 4) & 0x3FFFu) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3FFFu) << 32);   // layout type 0: no swizzle
}
// the same operand `n` rows / columns further along M or N (n a multiple of 8): core-matrix groups are SBO apart
__device__ __forceinline__ uint64_t desc_adv_mn(uint64_t desc, int n) {
  return desc + ((desc >> 32) & 0x3FFFu) * (uint64_t)(n >> 3);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  } while (!ok);
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t accum) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
               : "l"(da), "l"(db), "r"(accum), "n"(TA), "n"(TB) : "memory");
}
// (a larger fragment array: its first 16 registers)
template <int TA, int TB, int N>
__device__ __forceinline__ void wgmma_n32(float (&d)[N], uint64_t da, uint64_t db, uint32_t accum) {
  static_assert(N >= 16, "m64n32 accumulator needs 16 registers");
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "l"(da), "l"(db), "r"(accum), "n"(TA), "n"(TB) : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t accum) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(da), "l"(db), "r"(accum), "n"(TA), "n"(TB) : "memory");
}

// one NC-column chunk of D[128 x N] = sum_ks A_ks . B_ks into columns col0 + c .. of the accumulator tile
// (accum: add to what the tile holds).  descs(ks, da, db) gives the descriptors of the whole 128-row A tile and of B.
template <int NC, int TA, int TB, class F>
__device__ __forceinline__ void wg_mma_chunk(float* tile, int col0, int c, int KS, bool accum, const F& descs) {
  constexpr int NR = NC / 2;
  const int tid = threadIdx.x, g = tid >> 7, lane = tid & 31;
  const int row = g * 64 + ((tid >> 5) & 3) * 16 + (lane >> 2);
  float* p0 = tile + (size_t)row * ACC_COLS + col0 + c + 2 * (lane & 3);
  float* p1 = p0 + 8 * ACC_COLS;
  float dd[NR];
#pragma unroll
  for (int j = 0; j < NR / 4; ++j) {
    float2 x = make_float2(0.f, 0.f), y = x;
    if (accum) { x = *reinterpret_cast<const float2*>(p0 + 8 * j); y = *reinterpret_cast<const float2*>(p1 + 8 * j); }
    dd[4 * j] = x.x; dd[4 * j + 1] = x.y; dd[4 * j + 2] = y.x; dd[4 * j + 3] = y.y;
  }
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
  for (int ks = 0; ks < KS; ++ks) {
    uint64_t da, db;
    descs(ks, da, db);
    da = desc_adv_mn(da, 64 * g);
    db = desc_adv_mn(db, c);
    const uint32_t acc = (accum || ks > 0) ? 1u : 0u;
    if constexpr (NC == 64) wgmma_n64<TA, TB>(dd, da, db, acc);
    else if constexpr (NC == 32) wgmma_n32<TA, TB>(dd, da, db, acc);
    else wgmma_n16<TA, TB>(dd, da, db, acc);
  }
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
  for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(dd[i])::"memory");
#pragma unroll
  for (int j = 0; j < NR / 4; ++j) {
    *reinterpret_cast<float2*>(p0 + 8 * j) = make_float2(dd[4 * j], dd[4 * j + 1]);
    *reinterpret_cast<float2*>(p1 + 8 * j) = make_float2(dd[4 * j + 2], dd[4 * j + 3]);
  }
}
// D[128 x N] (N a multiple of 16) into tile columns col0 .. col0 + N; executed by all threads of warps 0-7.
// TA / TB: 0 = K-major, 1 = MN-major operand.
template <int TA, int TB, class F>
__device__ __forceinline__ void wg_mma(float* tile, int col0, int N, int KS, bool accum, const F& descs) {
  int c = 0;
  for (; c + 64 <= N; c += 64) wg_mma_chunk<64, TA, TB>(tile, col0, c, KS, accum, descs);
  if (c + 32 <= N) { wg_mma_chunk<32, TA, TB>(tile, col0, c, KS, accum, descs); c += 32; }
  if (c + 16 <= N) wg_mma_chunk<16, TA, TB>(tile, col0, c, KS, accum, descs);
}
// Register-accumulator form, for products that accumulate over many tiles: issues the KS k-steps of one NC-column slab
// of this warpgroup into the fragment `dd` (accum: add to what it holds) without committing or waiting.  descs(ks, da, db)
// gives the descriptors of this warpgroup's 64-row A slab and of the B columns.  The caller brackets a batch of these
// with wg_fence() and wg_commit(), and reads dd only after wg_wait<0>() (fragment layout: row 16 (warp & 3) + lane / 4
// (+ 8 for dd[4i + 2], dd[4i + 3]), column 8 i + 2 (lane & 3) (+ 1 for the odd entries)).
template <int NC, int TA, int TB, class F>
__device__ __forceinline__ void wg_mma_regs(float (&dd)[NC / 2], int KS, bool accum, const F& descs) {
  for (int ks = 0; ks < KS; ++ks) {
    uint64_t da, db;
    descs(ks, da, db);
    const uint32_t acc = (accum || ks > 0) ? 1u : 0u;
    if constexpr (NC == 64) wgmma_n64<TA, TB>(dd, da, db, acc);
    else if constexpr (NC == 32) wgmma_n32<TA, TB>(dd, da, db, acc);
    else wgmma_n16<TA, TB>(dd, da, db, acc);
  }
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of a fragment across a wg_wait (the asm of the wgmma only names it at issue)
template <int NR>
__device__ __forceinline__ void wg_frag_fence(float (&dd)[NR]) {
#pragma unroll
  for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(dd[i])::"memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// warps 0-7 have stored their fragments: publish them to the CTA and arrive (once) on `bar`
__device__ __forceinline__ void wg_mma_done(uint32_t bar) {
  __threadfence_block();
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (threadIdx.x == 0) mbar_arrive(bar);
}
// 16 / 8 consecutive accumulator columns of row (addr >> 16) + lane
__device__ __forceinline__ void acc_ld16(const float* tile, uint32_t addr, float* v) {
  const float4* p = reinterpret_cast<const float4*>(tile + (size_t)((addr >> 16) + (threadIdx.x & 31)) * ACC_COLS + (addr & 0xFFFFu));
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float4 x = p[i]; v[4 * i] = x.x; v[4 * i + 1] = x.y; v[4 * i + 2] = x.z; v[4 * i + 3] = x.w; }
}
__device__ __forceinline__ void acc_ld8(const float* tile, uint32_t addr, float* v) {
  const float4* p = reinterpret_cast<const float4*>(tile + (size_t)((addr >> 16) + (threadIdx.x & 31)) * ACC_COLS + (addr & 0xFFFFu));
#pragma unroll
  for (int i = 0; i < 2; ++i) { const float4 x = p[i]; v[4 * i] = x.x; v[4 * i + 1] = x.y; v[4 * i + 2] = x.z; v[4 * i + 3] = x.w; }
}

__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// MUFU tanh (tanh.approx.f32, max rel. error ~2^-11: below the bf16 operand rounding of this path)
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float sigm(float x) { return fmaf(0.5f, tanh_fast(0.5f * x), 0.5f); }
__device__ __forceinline__ uint32_t pmix32(uint32_t h) {
  h ^= h >> 16; h *= 0x7feb352dU; h ^= h >> 15; h *= 0x846ca68bU; h ^= h >> 16;
  return h;
}

// ---------------------------------------------------------------------------------------------------
// Accumulator tiles of the tensor-core kernels: one [128][ACC_COLS] fp32 tile per CTA, grids of at most two CTAs per SM
// (tscl_acc_tiles: owned by the handle, one set per stream, so that kernels running concurrently on different streams
// never share one)
static float* acc_tiles(tscl_handle* h, void* stream) {
  int n_sm = 0;
  if (cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, tscl_device_of(h)) != cudaSuccess) return nullptr;
  return tscl_acc_tiles(h, stream, (size_t)2 * n_sm * TC_M * ACC_COLS * sizeof(float));
}

// per-unit stride of the packed image: main [KC][256][8] followed by the fc image [8][dx][8]
__host__ __device__ inline int64_t wp_stride(int dx) { return (int64_t)((dx + TC_H) / 8) * TC_N * 8 + (int64_t)8 * dx * 8; }

// pack [Wx;Wh] of every unit into the bf16 UMMA B-operand image  Wp[u][kc][n][8]
__global__ void pack_wxh_kernel(const DDimsTC d, const float* __restrict__ P, __nv_bfloat16* __restrict__ Wp) {
  const int u = blockIdx.y;
  const int K = d.dx + TC_H, KC = K / 8;
  const float* Wx = P + d.off_wx + (int64_t)u * d.dx * TC_N;
  const float* Wh = P + d.off_wh + (int64_t)u * TC_H * TC_N;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < KC * TC_N; i += gridDim.x * blockDim.x) {
    const int kc = i / TC_N, n = i - kc * TC_N;
    __align__(16) __nv_bfloat16 v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = kc * 8 + e;
      const float w = k < d.dx ? Wx[(int64_t)k * TC_N + n] : Wh[(int64_t)(k - d.dx) * TC_N + n];
      v[e] = __float2bfloat16_rn(w);
    }
    *reinterpret_cast<uint4*>(Wp + (int64_t)u * wp_stride(d.dx) + ((int64_t)kc * TC_N + n) * 8) = *reinterpret_cast<const uint4*>(v);
  }
}


// block-diagonal fc weights as UMMA B operand: rows k = {wave 0..31 | fp 32..47 | wait 48..63}, cols = X columns
__global__ void pack_fc_kernel(const DDimsTC d, const float* __restrict__ P, __nv_bfloat16* __restrict__ Wp) {
  const int u = blockIdx.y, ag = u >> 1;
  const int nw = d.n_wave[ag], nt = d.n_wait[ag], nf = d.ff > 0 ? d.n_fp[ag] : 0;
  __nv_bfloat16* W0 = Wp + (int64_t)u * wp_stride(d.dx) + (int64_t)((d.dx + TC_H) / 8) * TC_N * 8;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 8 * d.dx; i += gridDim.x * blockDim.x) {
    const int kc = i / d.dx, n = i - kc * d.dx;
    __align__(16) __nv_bfloat16 v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = kc * 8 + e;
      float w = 0.f;
      if (n < d.fw) { if (k < d.kw && k < nw) w = P[d.off_fcw_w[u] + (int64_t)k * d.fw + n]; }
      else if (n < d.fw + d.ff) { const int kk = k - d.kw; if (kk >= 0 && kk < TC_KF && kk < nf) w = P[d.off_fcf_w[u] + (int64_t)kk * d.ff + (n - d.fw)]; }
      else { const int kk = k - d.kw - TC_KF; if (kk >= 0 && kk < nt) w = P[d.off_fct_w[u] + (int64_t)kk * d.ft + (n - d.fw - d.ff)]; }
      v[e] = __float2bfloat16_rn(w);
    }
    *reinterpret_cast<uint4*>(W0 + ((int64_t)kc * d.dx + n) * 8) = *reinterpret_cast<const uint4*>(v);
  }
}

struct StepTC {
  float* acc;                // accumulator tiles, one [128][ACC_COLS] fp32 tile per CTA (acc_tiles)
  const float* P;
  const __nv_bfloat16* Wp;
  const float* obs;        // [R][n_obs]
  const float* c_in;       // [2A][R][64]
  const float* h_in;
  float* c_out;
  float* h_out;
  float* pi;               // [R][A][max_na]
  float* val;              // [R][A]
  int32_t* act;            // [R][A] or null
  float* zdbg;             // [2A][R][256] raw accumulators (debug) or null
  int64_t R;
  int done;                // pre-decision done flag
  int swap_lbo_sbo;        // debug: exchange the two descriptor strides
  uint32_t seed_lo, seed_hi, step;
  int64_t replica0;
  // optional activation store for the update (v2 only): bf16 [R/rc][2A][T][rc][w], w = dx / 256 / 64 / 64
  // (replica-chunk major, so that each update chunk is one contiguous block)
  __nv_bfloat16 *st_x, *st_g, *st_c, *st_h;
  int t, T;
  int64_t rc;
  // replica-range launches (v2 only): the per-unit state arrays have `ld` rows per unit (0: R) and the activation
  // store is indexed by the absolute replica row0 + r; every pointer is the base of the range's slice
  int64_t ld, row0;
  unsigned long long* prof;   // optional: per-phase clock64 sums of thread 0 of every CTA (tools/profile only)
  int act_mode;               // pi-only instantiation: 0 = counter-RNG sample, 1 = first argmax of pi
  // grouped (population) instantiation: K members of Rm rows each; member k's parameters and bf16 image start at
  // P + k p_stride and Wp + k wp_stride, and it samples with seeds[k] (device array) and replica index r - k Rm
  int64_t Rm, p_stride, wp_stride;
  const uint64_t* seeds;
  // grouped pi-only instantiation (EVAL && GRP): ragged members, member k owns rows rows[k] .. rows[k+1] - 1 (device
  // array of K + 1 ascending boundaries); Rm is unused
  const int64_t* rows;
  int K;
};

extern __shared__ __align__(1024) unsigned char tc_smem[];

__global__ void __launch_bounds__(TC_THREADS, 1)
policy_step_tc_kernel(const DDimsTC d, const StepTC a) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = d.dx + TC_H, KC = K / 8, KS = K / 16;
  // ---- shared memory carve-up ----
  unsigned char* sB = tc_smem;                                  // KC * 4096
  unsigned char* sA = sB + (size_t)KC * 4096;                   // KC * 2048
  float* sStage = reinterpret_cast<float*>(sA + (size_t)KC * 2048);   // 16 x 64 floats; aliased by sRed [128][8]
  float* sWo = sStage + TC_STAGE_ROWS * TC_KTOT;                // [64][8]
  float* sBo = sWo + TC_H * 8;                                  // [8]
  float* sBias = sBo + 8;                                       // [256]
  uint64_t* sBar = reinterpret_cast<uint64_t*>(sBias + TC_N);   // mbarrier
  float* sRed = sStage;

  const uint32_t bar = smem_u32(sBar);
  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  float* const acc = a.acc + (size_t)blockIdx.x * TC_M * ACC_COLS;
  // instruction descriptor: D=f32, A=B=bf16, K-major both, N=256, M=128

  const int64_t n_tiles = (a.R + TC_M - 1) / TC_M;
  const int64_t n_items = n_tiles * 2 * d.A;
  const int64_t it_lo = n_items * blockIdx.x / gridDim.x, it_hi = n_items * (blockIdx.x + 1) / gridDim.x;
  int cur_u = -1;
  uint32_t parity = 0;
  // per-thread fc role: output column `col` of X
  const int col = tid;
  float w[TC_KW];
  float bias = 0.f;
  int kbase = 0, nk4 = 0, nw = 0, nt = 0, nf = 0, ooff = 0, n_in = 0, na = 0;

  for (int64_t it = it_lo; it < it_hi; ++it) {
    const int u = (int)(it / n_tiles);
    const int64_t r0 = (it - (int64_t)u * n_tiles) * TC_M;
    const int ag = u >> 1;
    if (u != cur_u) {
      cur_u = u;
      __syncthreads();
      // B operand image of this unit: plain 16-byte copies (async proxy will read it: fence below)
      const uint4* src = reinterpret_cast<const uint4*>(a.Wp + (int64_t)u * wp_stride(d.dx));
      uint4* dst = reinterpret_cast<uint4*>(sB);
      for (int i = tid; i < KC * TC_N; i += TC_THREADS) dst[i] = src[i];
      nw = d.n_wave[ag]; nt = d.n_wait[ag]; nf = d.ff > 0 ? d.n_fp[ag] : 0;
      n_in = nw + nt + nf; ooff = d.obs_off[ag]; na = d.n_a[ag];
#pragma unroll
      for (int k = 0; k < TC_KW; ++k) w[k] = 0.f;
      int nk = 0;
      if (col < d.dx) {
        if (col < d.fw) {
          nk = nw; kbase = 0;
#pragma unroll
          for (int k = 0; k < TC_KW; ++k) if (k < nw) w[k] = a.P[d.off_fcw_w[u] + (int64_t)k * d.fw + col];
          bias = a.P[d.off_fcw_b[u] + col];
        } else if (col < d.fw + d.ff) {
          nk = nf; kbase = TC_KW;
#pragma unroll
          for (int k = 0; k < TC_KF; ++k) if (k < nf) w[k] = a.P[d.off_fcf_w[u] + (int64_t)k * d.ff + (col - d.fw)];
          bias = a.P[d.off_fcf_b[u] + (col - d.fw)];
        } else {
          nk = nt; kbase = TC_KW + TC_KF;
#pragma unroll
          for (int k = 0; k < TC_KT; ++k) if (k < nt) w[k] = a.P[d.off_fct_w[u] + (int64_t)k * d.ft + (col - d.fw - d.ff)];
          bias = a.P[d.off_fct_b[u] + (col - d.fw - d.ff)];
        }
      }
      nk4 = (nk + 3) >> 2;
      for (int i = tid; i < TC_H * 8; i += TC_THREADS) {
        const int k = i >> 3, j = i & 7;
        sWo[i] = j < d.max_na ? a.P[d.off_wo + ((int64_t)u * TC_H + k) * d.max_na + j] : 0.f;
      }
      if (tid < 8) sBo[tid] = tid < d.max_na ? a.P[d.off_bo + (int64_t)u * d.max_na + tid] : 0.f;
      for (int i = tid; i < TC_N; i += TC_THREADS) sBias[i] = a.P[d.off_bl + (int64_t)u * TC_N + i];
    }
    // ---- 1. A tile: fc front end (cols 0..dx) in 16-row sub-blocks, then h_prev (cols dx..dx+64) ----
    for (int sb = 0; sb < TC_M / TC_STAGE_ROWS; ++sb) {
      __syncthreads();
      for (int i = tid; i < TC_STAGE_ROWS * TC_KTOT; i += TC_THREADS) sStage[i] = 0.f;
      __syncthreads();
      for (int i = tid; i < TC_STAGE_ROWS * n_in; i += TC_THREADS) {
        const int row = i / n_in, k = i - row * n_in;
        const int64_t r = r0 + sb * TC_STAGE_ROWS + row;
        if (r < a.R) {
          int dst;
          if (k < nw) dst = k;
          else if (k < nw + nt) dst = TC_KW + TC_KF + (k - nw);
          else dst = TC_KW + (k - nw - nt);
          sStage[row * TC_KTOT + dst] = a.obs[r * d.n_obs + ooff + k];
        }
      }
      __syncthreads();
      if (col < d.dx) {
        __nv_bfloat16* acol = reinterpret_cast<__nv_bfloat16*>(sA + (size_t)(col >> 3) * 2048) + (col & 7);
#pragma unroll 4
        for (int row = 0; row < TC_STAGE_ROWS; ++row) {
          const float4* in4 = reinterpret_cast<const float4*>(&sStage[row * TC_KTOT + kbase]);
          float acc = bias;
#pragma unroll
          for (int k4 = 0; k4 < TC_KW / 4; ++k4) {
            if (k4 < nk4) {
              const float4 x = in4[k4];
              acc = fmaf(x.x, w[4 * k4], acc); acc = fmaf(x.y, w[4 * k4 + 1], acc);
              acc = fmaf(x.z, w[4 * k4 + 2], acc); acc = fmaf(x.w, w[4 * k4 + 3], acc);
            }
          }
          acol[(sb * TC_STAGE_ROWS + row) * 8] = __float2bfloat16_rn(fmaxf(acc, 0.f));
        }
      }
    }
    {   // h_prev -> A columns dx .. dx+63 : thread = (row, 32-column half)
      const int row = tid >> 1, half = tid & 1;
      const int64_t r = r0 + row;
      const bool live = r < a.R && !a.done;
      const float4* hp = reinterpret_cast<const float4*>(a.h_in + ((int64_t)u * a.R + (r < a.R ? r : 0)) * TC_H + half * 32);
#pragma unroll
      for (int c8 = 0; c8 < 4; ++c8) {
        __align__(16) __nv_bfloat16 v[8];
        float4 x0 = make_float4(0.f, 0.f, 0.f, 0.f), x1 = x0;
        if (live) { x0 = hp[2 * c8]; x1 = hp[2 * c8 + 1]; }
        v[0] = __float2bfloat16_rn(x0.x); v[1] = __float2bfloat16_rn(x0.y); v[2] = __float2bfloat16_rn(x0.z); v[3] = __float2bfloat16_rn(x0.w);
        v[4] = __float2bfloat16_rn(x1.x); v[5] = __float2bfloat16_rn(x1.y); v[6] = __float2bfloat16_rn(x1.z); v[7] = __float2bfloat16_rn(x1.w);
        const int kc = (d.dx >> 3) + half * 4 + c8;
        *reinterpret_cast<uint4*>(sA + (size_t)kc * 2048 + row * 16) = *reinterpret_cast<const uint4*>(v);
      }
    }
    // generic-proxy smem writes -> visible to the tensor core (async proxy)
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    // ---- 2. MMA: D[128 x 256] = A[128 x K] . B[K x 256] ----
    if (warp < 8) {
      const uint32_t aA = smem_u32(sA), aB = smem_u32(sB);
      wg_mma<0, 0>(acc, 0, TC_N, KS, false, [&](int ks, uint64_t& da, uint64_t& db) {
        if (!a.swap_lbo_sbo) {
          da = make_desc(aA + ks * 2 * 2048, 2048, 128);
          db = make_desc(aB + ks * 2 * 4096, 4096, 128);
        } else {
          da = make_desc(aA + ks * 2 * 2048, 128, 2048);
          db = make_desc(aB + ks * 2 * 4096, 128, 4096);
        }
      });
      wg_mma_done(bar);
    }
    mbar_wait(bar, parity);
    parity ^= 1;
    // ---- 3. epilogue: thread = (row of the accumulator tile, 32 hidden units) ----
    {
      const int q = warp & 3, half = warp >> 2;
      const int row = q * 32 + lane;
      const int64_t r = r0 + row;
      const bool valid = r < a.R;
      const int64_t srow = ((int64_t)u * a.R + (valid ? r : 0)) * TC_H + half * 32;
      float lg[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) lg[j] = 0.f;
#pragma unroll
      for (int jb = 0; jb < 2; ++jb) {
        float zi[16], zf[16], zo[16], zu[16];
        const uint32_t tbase = ((uint32_t)(q * 32) << 16) + (uint32_t)(half * 32 + jb * 16);
        acc_ld16(acc, tbase, zi); acc_ld16(acc, tbase + 64, zf); acc_ld16(acc, tbase + 128, zo); acc_ld16(acc, tbase + 192, zu);
        if (a.zdbg && valid) {
          float* z = a.zdbg + ((int64_t)u * a.R + r) * TC_N + half * 32 + jb * 16;
#pragma unroll
          for (int e = 0; e < 16; ++e) { z[e] = zi[e]; z[64 + e] = zf[e]; z[128 + e] = zo[e]; z[192 + e] = zu[e]; }
        }
        float cprev[16];
        if (valid && !a.done) {
          const float4* cp = reinterpret_cast<const float4*>(a.c_in + srow + jb * 16);
#pragma unroll
          for (int e4 = 0; e4 < 4; ++e4) {
            const float4 x = cp[e4];
            cprev[4 * e4] = x.x; cprev[4 * e4 + 1] = x.y; cprev[4 * e4 + 2] = x.z; cprev[4 * e4 + 3] = x.w;
          }
        } else {
#pragma unroll
          for (int e = 0; e < 16; ++e) cprev[e] = 0.f;
        }
        float cn[16], hn[16];
#pragma unroll
        for (int e = 0; e < 16; ++e) {
          const int j = half * 32 + jb * 16 + e;
          const float gi = sigm(zi[e] + sBias[j]), gf = sigm(zf[e] + sBias[64 + j]);
          const float go = sigm(zo[e] + sBias[128 + j]), gu = tanh_fast(zu[e] + sBias[192 + j]);
          cn[e] = gf * cprev[e] + gi * gu;
          hn[e] = go * tanh_fast(cn[e]);
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) lg[jj] = fmaf(hn[e], sWo[j * 8 + jj], lg[jj]);
        }
        if (valid) {
          float4* co = reinterpret_cast<float4*>(a.c_out + srow + jb * 16);
          float4* ho = reinterpret_cast<float4*>(a.h_out + srow + jb * 16);
#pragma unroll
          for (int e4 = 0; e4 < 4; ++e4) {
            co[e4] = make_float4(cn[4 * e4], cn[4 * e4 + 1], cn[4 * e4 + 2], cn[4 * e4 + 3]);
            ho[e4] = make_float4(hn[4 * e4], hn[4 * e4 + 1], hn[4 * e4 + 2], hn[4 * e4 + 3]);
          }
        }
      }
      // all accumulator reads of this tile are done before the next tile's MMA may overwrite the accumulator
      __syncthreads();     // also: sStage (aliased by sRed) is free
      if (half == 1) {
#pragma unroll
        for (int j = 0; j < 8; ++j) sRed[row * 8 + j] = lg[j];
      }
      __syncthreads();
      if (half == 0 && valid) {
#pragma unroll
        for (int j = 0; j < 8; ++j) lg[j] += sRed[row * 8 + j] + sBo[j];
        if ((u & 1) == 0) {        // policy unit
          float mx = -1e30f;
#pragma unroll
          for (int j = 0; j < 8; ++j) if (j < na) mx = fmaxf(mx, lg[j]);
          float s = 0.f;
#pragma unroll
          for (int j = 0; j < 8; ++j) { lg[j] = j < na ? __expf(lg[j] - mx) : 0.f; s += lg[j]; }
          const float inv = 1.0f / s;
          float* po = a.pi + ((int64_t)r * d.A + ag) * d.max_na;
#pragma unroll
          for (int j = 0; j < 8; ++j) if (j < d.max_na) po[j] = lg[j] * inv;
          if (a.act) {
            uint32_t hsh = pmix32(a.seed_lo ^ (a.step * 0x9E3779B1U));
            hsh = pmix32(hsh ^ a.seed_hi ^ ((uint32_t)(a.replica0 + r) * 0x85EBCA77U));
            hsh = pmix32(hsh ^ ((uint32_t)ag * 0xC2B2AE3DU));
            const float uu = (float)(hsh >> 8) * (1.0f / 16777216.0f);
            float cum = 0.f;
            int pick = na - 1;
            bool found = false;
#pragma unroll
            for (int j = 0; j < 8; ++j)
              if (j < na) { cum += lg[j] * inv; if (!found && uu < cum) { pick = j; found = true; } }
            a.act[(int64_t)r * d.A + ag] = pick;
          }
        } else {
          a.val[(int64_t)r * d.A + ag] = lg[0];
        }
      }
    }
  }
  __syncthreads();
}

// ===================================================================================================
static size_t tc_smem_bytes(int K) {
  const int KC = K / 8;
  return (size_t)KC * 4096 + (size_t)KC * 2048 + (TC_STAGE_ROWS * TC_KTOT + TC_H * 8 + 8 + TC_N) * 4 + 16;
}

extern "C" int tscl_pack_weights(tscl_handle* h, const float* params, void* wpack_bf16, void* stream) {
  if (!h || !params || !wpack_bf16) return tsc_set_error("tscl_pack_weights: bad argument");
  PCK(cudaSetDevice(tscl_device_of(h)));
  const DDimsTC& d = *tscl_dims_of(h);
  if ((d.dx % 16) != 0) return tsc_set_error("tscl_pack_weights: dx must be a multiple of 16");
  dim3 grid(8, 2 * d.A);
  pack_wxh_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(d, params, (__nv_bfloat16*)wpack_bf16);
  pack_fc_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(d, params, (__nv_bfloat16*)wpack_bf16);
  PCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_policy_step(tscl_handle* h, const float* params, const void* wpack_bf16, const float* obs,
                                int64_t R, const float* c_in, const float* h_in, float* c_out, float* h_out, float* pi,
                                float* val, int32_t* act, int32_t done, uint64_t seed, int64_t step, int64_t replica0,
                                float* zdbg, int32_t swap_lbo_sbo, void* stream) {
  if (!h || !params || !wpack_bf16 || !obs || R <= 0) return tsc_set_error("tscl_policy_step: bad argument");
  PCK(cudaSetDevice(tscl_device_of(h)));
  const DDimsTC& d = *tscl_dims_of(h);
  const int K = d.dx + TC_H;
  if ((d.dx % 16) != 0 || d.dx > TC_THREADS) return tsc_set_error("tscl_policy_step: unsupported dx");
  if (d.kw != 32) return tsc_set_error("tscl_policy_step: v1 kernel supports wave widths <= 32 only (use tscl_policy_step_v2)");
  const size_t smem = tc_smem_bytes(K);
  if (smem > 232448) return tsc_set_error("tscl_policy_step: operand tiles exceed shared memory");
  static int attr_dev = -1;
  if (attr_dev != tscl_device_of(h)) {      // the largest opt-in, so that a later handle with a wider dx can launch too
    PCK(cudaFuncSetAttribute(policy_step_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    attr_dev = tscl_device_of(h);
  }
  int n_sm = 0;
  PCK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, tscl_device_of(h)));
  const int64_t n_items = ((R + TC_M - 1) / TC_M) * 2 * d.A;
  const int grid = (int)(n_items < n_sm ? n_items : n_sm);
  StepTC a;
  a.acc = acc_tiles(h, stream);
  if (!a.acc) return tsc_set_error("accumulator tiles: cudaMalloc failed");
  a.P = params; a.Wp = (const __nv_bfloat16*)wpack_bf16; a.obs = obs; a.c_in = c_in; a.h_in = h_in; a.c_out = c_out;
  a.h_out = h_out; a.pi = pi; a.val = val; a.act = act; a.zdbg = zdbg; a.R = R; a.done = done;
  a.swap_lbo_sbo = swap_lbo_sbo; a.seed_lo = (uint32_t)seed; a.seed_hi = (uint32_t)(seed >> 32);
  a.step = (uint32_t)step; a.replica0 = replica0;
  a.st_x = a.st_g = a.st_c = a.st_h = nullptr; a.t = 0; a.T = 1; a.rc = R; a.prof = nullptr;
  policy_step_tc_kernel<<<grid, TC_THREADS, smem, (cudaStream_t)stream>>>(d, a);
  PCK(cudaGetLastError());
  return 0;
}

// ===================================================================================================
// v2: the fc front end also runs on the tensor cores, and the kernel is warp-specialised: 384 threads, three warpgroups.
// A work item is (unit, 64 replica rows); a CTA walks a contiguous range of items, the items of one unit at a time.
//   warpgroup 0, producer: stages the items in turn into two A tiles (item parity = tile): the unit's fc-weight block
//     B0 [8][dx][16 B] by one bulk copy into the X chunks of the tile (it fills exactly dx / 8 chunks: a region that is
//     dead until the fc result is written), and the observation slice A0 [64 x 64] (bf16) into the last 8 chunks (dead
//     until h_{t-1} is written); L2 prefetch of the state rows of the item after next.
//   warpgroups 1 and 2, consumers: consumer c takes the items of parity c, in tile c, so that one consumer's MMAs and
//     operand loads overlap the other's epilogue:
//       MMA0  D0[64 x dx] = A0 . B0 into registers; + bias, relu, bf16 -> X chunks of the tile (and the activation
//             store st_x, copied out of shared memory in whole sectors); h_{t-1} -> the last 8 chunks;
//       MMA1  gates[64 x 256] = [X | h] . [Wx;Wh] into registers, one m64n64 fragment per gate;
//       LSTM cell, state and activation-store writes and the head dot products straight from the fragments.
// The resident [Wx;Wh] image is copied into shared memory with its gate columns permuted: packed column 8i + 2q + e holds
// gate i / 8, hidden unit 16q + 2(i % 8) + e (gate_col).  So lane q of each quad holds all four gates of hidden units
// 16q .. 16q + 15 of its two fragment rows: thread = (row, 16 hidden units), the cell's natural assignment.  The MMAs
// are the same m64nN k16 instructions in the same k order as a 128-row tile walked 64 columns at a time, and the cell,
// store and head arithmetic is per element what it was, so the outputs do not depend on this organisation.
#define P2_ROWS 64
#define P2_DX_OK(dx) ((dx) == 128 || (dx) == 160 || (dx) == 192 || (dx) == 224)   // keep in sync with learner.V2_DX
#define P2_THREADS 384
// setmaxnreg: the producer gives registers back, the consumers (four m64n64 gate fragments = 128 per thread, plus the
// cell state) take them.  setmaxnreg.inc only draws on what the CTA was launched with (168 per thread at 384 threads =
// 64512; a larger request waits forever), so 128 * P2_PROD_REGS + 256 * P2_CONS_REGS must not exceed 384 * 168.
#define P2_PROD_REGS 40
#define P2_CONS_REGS 232
static_assert(128 * P2_PROD_REGS + 256 * P2_CONS_REGS <= P2_THREADS * 168, "setmaxnreg split exceeds the CTA's registers");

// v -> bf16 (round to nearest even) into the low (hi = 0) or high half of w
__device__ __forceinline__ void bf16_pack(uint32_t& w, float v, int hi) {
  const uint32_t b = __bfloat16_as_ushort(__float2bfloat16_rn(v));
  w = hi ? (w | (b << 16)) : b;
}
// unpermuted gate-image column ([i | f | o | u] x 64) held by packed column n of the consumers' B operand
__host__ __device__ inline int gate_col(int n) {
  const int i = n >> 3, q = (n >> 1) & 3, e = n & 1;
  return (i >> 3) * 64 + 16 * q + 2 * (i & 7) + e;
}

// EVAL && GRP: the item block (member mk, pi unit ui) holding item `seg`.  Member k's items are its A units times its
// ceil(S_k / 64) tiles, in member order; the item count the launcher sizes the grid with is an upper bound, so an item
// past the last member returns false.  rofs: the block's first row minus 64 times its first item.
__device__ __forceinline__ bool grp_block(const DDimsTC& d, const StepTC& a, int64_t seg, int64_t it_hi, int& mk, int& ui,
                                          int64_t& seg_hi, int64_t& rofs) {
  int64_t t0 = 0;
  for (int k = 0; k < a.K; ++k) {
    const int64_t r0 = a.rows[k], nt = (a.rows[k + 1] - r0 + P2_ROWS - 1) / P2_ROWS, ni = nt * d.A;
    if (seg < t0 + ni) {
      mk = k;
      ui = (int)((seg - t0) / nt);
      const int64_t b0 = t0 + (int64_t)ui * nt;
      seg_hi = b0 + nt < it_hi ? b0 + nt : it_hi;
      rofs = r0 - b0 * P2_ROWS;
      return true;
    }
    t0 += ni;
  }
  return false;
}

// DX = d.dx: the fragment sizes and the k loops are compile-time.  Instantiated for the fc widths of the shipped
// configurations (P2_DX_OK): 224 (grid MA2C), 192 (Monaco), 160 (grid IA2C: no fingerprint block), 128 (Monaco IA2C:
// no fingerprint or wait block)
// EVAL: the pi-only forward of test-mode evaluation (tscl_policy_step_pi).  Work items are (pi unit u = 2 * agent, 64 rows),
// n_tiles * A of them; V units are never loaded, multiplied or stored.  The recurrent state is compact, [A][ld][h] (row
// (u >> 1) * ld + r); there is no activation store, no zdbg and no value output.  Per element the arithmetic is the
// training instantiation's, so pi, c and h are bit-identical to its pi units.
// GRP: the population forward (tscl_policy_step_v2g).  Rows are K members of a.Rm (a multiple of 64) each; work items
// are (member, unit, tile), so one member's [Wx;Wh] image stays resident over its tiles, and a block of items never
// spans two members.  Member k reads its parameters and image at stride offsets and samples with the key
// (seeds[k], step, replica0 + r - k Rm) of its own one-member launch; per element the arithmetic is unchanged.
// EVAL && GRP: the grouped pi-only forward (tscl_policy_step_pi_g).  Members are ragged (grp_block): items are (member,
// pi unit, tile of the member), a member's last tile is partial and its rows past the member's end are neither loaded
// nor stored; member k samples with (seeds[k], step, r - rows[k]).
template <int DX, bool PROF, bool EVAL, bool GRP = false>
__global__ void __launch_bounds__(P2_THREADS, 1)
policy_step_tc2_kernel(const DDimsTC d, const StepTC a) {
  const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31;
  constexpr int K = DX + TC_H, KC = K / 8, KS = K / 16, KCX = DX / 8, NXF = (DX + 63) / 64;
  unsigned char* sB = tc_smem;                                               // KC * 4096, gate columns permuted
  unsigned char* sA0 = sB + (size_t)KC * 4096;                               // two A tiles [KC][64 rows][16 B]
  float* sWo = reinterpret_cast<float*>(sA0 + (size_t)2 * KC * 1024);        // [64][8]
  float* sBo = sWo + TC_H * 8;                                               // [8]
  float* sBias = sBo + 8;                                                    // [256]  lstm bias
  float* sBias0 = sBias + TC_N;                                              // [256]  fc biases
  uint64_t* sBar = reinterpret_cast<uint64_t*>(sBias0 + TC_N);               // full[2], empty[2]
  // GRP only (16 more bytes): the block's row offset rofs (int64), the member's sampling key and the low word of its
  // first row, kept in shared memory rather than in the consumers' full register budget; EVAL && GRP (8 more): the
  // member's end row
  int64_t* sGrp = reinterpret_cast<int64_t*>(sBar + 4);
  const uint32_t aB = smem_u32(sB);
  if (tid == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(smem_u32(sBar + s), 128 + 1);        // producer threads + the fc-weight copy's expect_tx
      mbar_init(smem_u32(sBar + 2 + s), 128);        // consumer threads: the tile is dead
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int64_t n_tiles = (a.R + P2_ROWS - 1) / P2_ROWS;
  const int64_t ld = a.ld > 0 ? a.ld : a.R;
  const int64_t n_items = (EVAL && GRP ? n_tiles + a.K - 1 : n_tiles) * (EVAL ? 1 : 2) * d.A;   // EVAL && GRP: bound
  const int64_t it_lo = n_items * blockIdx.x / gridDim.x, it_hi = n_items * (blockIdx.x + 1) / gridDim.x;

  // phase clocks of the producer's thread 0 and consumer 0's thread 0, added straight into the counters (no register
  // arrays: the producer's budget is small)
  long long pc = 0;
  const bool prof_thread = PROF && (tid == 0 || tid == 128);
#define PROF_MARK(i) do { if (PROF && prof_thread) { const long long c_ = clock64(); atomicAdd(a.prof + (i), (unsigned long long)(c_ - pc)); pc = c_; } } while (0)
  if (PROF && prof_thread) pc = clock64();

  // the constants of unit u, written by the 256 consumer threads between two CTA barriers that every role passes (all
  // roles have retired the previous unit); the producer, with its small register budget, only takes the barriers
  auto load_unit = [&](int u, int mk, int64_t rofs, bool consumer) {
    __syncthreads();
    if (consumer) {
      const int t = tid - 128;
      if (GRP && t == 0) {
        const uint64_t sk = a.seeds[mk];
        sGrp[0] = rofs;
        reinterpret_cast<uint32_t*>(sGrp)[2] = pmix32((uint32_t)sk ^ (a.step * 0x9E3779B1U)) ^ (uint32_t)(sk >> 32);
        if constexpr (EVAL) {
          reinterpret_cast<uint32_t*>(sGrp)[3] = (uint32_t)a.rows[mk];
          sGrp[2] = a.rows[mk + 1];
        } else {
          reinterpret_cast<uint32_t*>(sGrp)[3] = (uint32_t)((int64_t)mk * a.Rm);
        }
      }
      const float* P = GRP ? a.P + (int64_t)mk * a.p_stride : a.P;
      const uint4* src = reinterpret_cast<const uint4*>((GRP ? a.Wp + (int64_t)mk * a.wp_stride : a.Wp) + (int64_t)u * wp_stride(DX));
      uint4* dst = reinterpret_cast<uint4*>(sB);
#pragma unroll 4
      for (int i = t; i < KC * TC_N; i += 256) dst[i] = src[(i & ~(TC_N - 1)) + gate_col(i & (TC_N - 1))];
      for (int i = t; i < TC_H * 8; i += 256) {
        const int k = i >> 3, j = i & 7;
        sWo[i] = j < d.max_na ? P[d.off_wo + ((int64_t)u * TC_H + k) * d.max_na + j] : 0.f;
      }
      if (t < 8) sBo[t] = t < d.max_na ? P[d.off_bo + (int64_t)u * d.max_na + t] : 0.f;
      for (int i = t; i < TC_N; i += 256) {
        sBias[i] = P[d.off_bl + (int64_t)u * TC_N + i];
        float b0 = 0.f;
        if (i < d.fw) b0 = P[d.off_fcw_b[u] + i];
        else if (i < d.fw + d.ff) b0 = P[d.off_fcf_b[u] + (i - d.fw)];
        else if (i < d.dx) b0 = P[d.off_fct_b[u] + (i - d.fw - d.ff)];
        sBias0[i] = b0;
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // the B image is read by wgmma
    }
    __syncthreads();
  };

  if (wg == 0) {
    // ================= producer =================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(P2_PROD_REGS));
    const int warp = tid >> 5;
    uint32_t ph_empty = 0;
    for (int64_t seg = it_lo; seg < it_hi;) {
      int mk, ui;                 // ui: item block = state unit
      int64_t seg_hi, rofs;
      if constexpr (EVAL && GRP) {
        if (!grp_block(d, a, seg, it_hi, mk, ui, seg_hi, rofs)) break;
      } else {
        // GRP: item block blk = (member mk, unit ui) of bt tiles; items (item counts < 2^31) in 32-bit arithmetic
        const int bt = GRP ? (int)(a.Rm / P2_ROWS) : 1, blk = GRP ? (int)seg / bt : 0;
        mk = GRP ? blk / (2 * d.A) : 0;
        ui = GRP ? blk - mk * 2 * d.A : (int)(seg / n_tiles);
        seg_hi = GRP ? ((int64_t)(blk + 1) * bt < it_hi ? (int64_t)(blk + 1) * bt : it_hi)
                     : ((int64_t)(ui + 1) * n_tiles < it_hi ? (int64_t)(ui + 1) * n_tiles : it_hi);
        rofs = GRP ? (int64_t)mk * a.Rm - (int64_t)blk * bt * P2_ROWS : 0;
      }
      const int u = EVAL ? 2 * ui : ui, ag = u >> 1;
      load_unit(u, mk, rofs, false);
      PROF_MARK(8);      // producer: unit constants
      const int nw = d.n_wave[ag], nt = d.n_wait[ag], nf = d.ff > 0 ? d.n_fp[ag] : 0, ooff = d.obs_off[ag];
      // observation index of this lane's two input slots 2 lane, 2 lane + 1 (-1: unused slot)
      auto slot_src = [&](int c) -> int {
        if (c < d.kw) return c < nw ? c : -1;
        if (c < d.kw + TC_KF) return c - d.kw < nf ? nw + nt + (c - d.kw) : -1;
        return c - d.kw - TC_KF < nt ? nw + (c - d.kw - TC_KF) : -1;
      };
      const int src_a = slot_src(2 * lane), src_b = slot_src(2 * lane + 1);
      const __nv_bfloat16* Wfc = (GRP ? a.Wp + (int64_t)mk * a.wp_stride : a.Wp) + (int64_t)u * wp_stride(DX) + (int64_t)KC * TC_N * 8;
      for (int64_t it = seg; it < seg_hi; ++it) {
        const int s = (int)((it - it_lo) & 1);
        const int64_t r0 = GRP ? sGrp[0] + it * P2_ROWS : (it - (int64_t)ui * n_tiles) * P2_ROWS;
        const int64_t rlim = EVAL && GRP ? sGrp[2] : a.R;      // end of the rows this item may touch
        unsigned char* sA = sA0 + (size_t)s * KC * 1024;
        const uint32_t full = smem_u32(sBar + s), empty = smem_u32(sBar + 2 + s);
        mbar_wait(empty, ((ph_empty >> s) & 1) ^ 1);       // the tile's previous item has left it (first use: passes)
        ph_empty ^= 1u << s;
        PROF_MARK(9);    // producer: waiting for a free tile
        if (tid == 0) {
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          mbar_expect_tx(full, (uint32_t)(8 * DX * 16));
          bulk_g2s(smem_u32(sA), Wfc, (uint32_t)(8 * DX * 16), full);
        }
        // L2 prefetch of the state rows and observations of the next item of this tile (GRP: within the block only)
        if (GRP ? it + 2 < seg_hi : it + 2 < it_hi) {
          int un;
          int64_t rn;
          if (GRP) {
            un = ui;
            rn = r0 + 2 * P2_ROWS + (tid & 63);
          } else {
            un = (int)((it + 2) / n_tiles);
            rn = ((it + 2) - (int64_t)un * n_tiles) * P2_ROWS + (tid & 63);
          }
          if (rn < rlim) {
            const int64_t so = ((int64_t)un * ld + rn) * TC_H + (tid >> 6) * 32;
            asm volatile("prefetch.global.L2 [%0];" ::"l"(a.c_in + so));
            asm volatile("prefetch.global.L2 [%0];" ::"l"(a.h_in + so));
            asm volatile("prefetch.global.L2 [%0];" ::"l"(a.obs + rn * d.n_obs + d.obs_off[EVAL ? un : un >> 1] + (tid >> 6) * 32));
          }
        }
        // observation slice: warp w takes rows 16 w .. 16 w + 15, lane l the input slots 2l, 2l + 1 of each (the slice of
        // a row is one contiguous <= 256 B run of the observation vector); the two values leave as one packed store
#pragma unroll
        for (int h4 = 0; h4 < 4; ++h4) {
          const int rb = warp * 16 + h4 * 4;
          float xa[4], xb[4];
#pragma unroll
          for (int rr = 0; rr < 4; ++rr) {
            const int64_t r = r0 + rb + rr;
            const bool ok = r < rlim;
            const float* op = a.obs + (ok ? r : 0) * d.n_obs + ooff;
            xa[rr] = (src_a >= 0 && ok) ? __ldg(op + src_a) : 0.f;
            xb[rr] = (src_b >= 0 && ok) ? __ldg(op + src_b) : 0.f;
          }
#pragma unroll
          for (int rr = 0; rr < 4; ++rr)
            *reinterpret_cast<__nv_bfloat162*>(sA + (size_t)(KC - 8 + (lane >> 2)) * 1024 + (rb + rr) * 16 + (lane & 3) * 4) =
                __floats2bfloat162_rn(xa[rr], xb[rr]);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_arrive(full);
        PROF_MARK(10);   // producer: fc-weight copy issue + observation staging
      }
      seg = seg_hi;
    }
  } else {
    // ================= consumers =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(P2_CONS_REGS));
    const int c = wg - 1, ct = tid & 127, q = lane & 3;
    const int rq = 16 * (ct >> 5) + (lane >> 2);                  // fragment rows rq, rq + 8
    unsigned char* sA = sA0 + (size_t)c * KC * 1024;
    const uint32_t aA = smem_u32(sA), full = smem_u32(sBar + c), empty = smem_u32(sBar + 2 + c);
    uint32_t ph_full = 0;
    for (int64_t seg = it_lo; seg < it_hi;) {
      int mk, ui;
      int64_t seg_hi, rofs;
      if constexpr (EVAL && GRP) {
        if (!grp_block(d, a, seg, it_hi, mk, ui, seg_hi, rofs)) break;
      } else {
        const int bt = GRP ? (int)(a.Rm / P2_ROWS) : 1, blk = GRP ? (int)seg / bt : 0;
        mk = GRP ? blk / (2 * d.A) : 0;
        ui = GRP ? blk - mk * 2 * d.A : (int)(seg / n_tiles);
        seg_hi = GRP ? ((int64_t)(blk + 1) * bt < it_hi ? (int64_t)(blk + 1) * bt : it_hi)
                     : ((int64_t)(ui + 1) * n_tiles < it_hi ? (int64_t)(ui + 1) * n_tiles : it_hi);
        rofs = GRP ? (int64_t)mk * a.Rm - (int64_t)blk * bt * P2_ROWS : 0;
      }
      const int u = EVAL ? 2 * ui : ui, ag = u >> 1;
      load_unit(u, mk, rofs, true);
      PROF_MARK(0);      // unit constants
      const int na = d.n_a[ag];
      for (int64_t it = seg + (((seg - it_lo) & 1) != c ? 1 : 0); it < seg_hi; it += 2) {
        const int64_t r0 = GRP ? sGrp[0] + it * P2_ROWS : (it - (int64_t)ui * n_tiles) * P2_ROWS;
        const int64_t rlim = EVAL && GRP ? sGrp[2] : a.R;
        // row of the activation store (chunk-outermost [R/rc][2A][T][rc][w]) for tile row `row`
        const int64_t st_c0 = (a.row0 + r0) / a.rc, st_rin0 = (a.row0 + r0) - st_c0 * a.rc;
        auto store_row = [&](int row) -> int64_t {
          int64_t cc = st_c0, rin = st_rin0 + row;
          while (rin >= a.rc) { rin -= a.rc; ++cc; }
          return ((cc * (2 * d.A) + u) * a.T + a.t) * a.rc + rin;
        };
        mbar_wait(full, ph_full);
        ph_full ^= 1;
        PROF_MARK(1);    // waiting for the staged operands
        // ---- MMA0: D0[64 x dx] = A0[64 x 64] . B0[64 x dx], 64 columns at a time (a last 32-column piece if dx % 64) ----
        float x[NXF][32];
        wg_fence();
#pragma unroll
        for (int j = 0; j < NXF; ++j)
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            const uint64_t da = make_desc(aA + (KC - 8 + 2 * ks) * 1024, 1024, 128);
            const uint64_t db = desc_adv_mn(make_desc(aA + ks * 2 * (DX * 16), DX * 16, 128), 64 * j);
            if (64 * j + 64 <= DX) wgmma_n64<0, 0>(x[j], da, db, ks > 0 ? 1u : 0u);
            else wgmma_n32<0, 0>(x[j], da, db, ks > 0 ? 1u : 0u);
          }
        wg_commit();
        wg_wait<0>();
#pragma unroll
        for (int j = 0; j < NXF; ++j) wg_frag_fence(x[j]);
        PROF_MARK(2);    // MMA0 issue + wait
        // ---- X = relu(D0 + b) as bf16 -> chunks 0 .. dx/8 (B0 is dead); h_{t-1} -> the last 8 (A0 is dead) ----
#pragma unroll
        for (int j = 0; j < NXF; ++j)
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int col = 64 * j + 8 * i;
            if (col < DX) {
              const float b0 = sBias0[col + 2 * q], b1 = sBias0[col + 2 * q + 1];
#pragma unroll
              for (int hr = 0; hr < 2; ++hr)
                *reinterpret_cast<__nv_bfloat162*>(sA + (size_t)(col >> 3) * 1024 + (rq + 8 * hr) * 16 + q * 4) =
                    __floats2bfloat162_rn(fmaxf(x[j][4 * i + 2 * hr] + b0, 0.f), fmaxf(x[j][4 * i + 2 * hr + 1] + b1, 0.f));
            }
          }
        // h_{t-1} of row ct & 63, hidden units 32 (ct >> 6) .. (the producer prefetched it to L2)
        float4 hpre[8];
        {
          const int64_t r = r0 + (ct & 63);
          const bool live = r < rlim && !a.done;
          const float4* hp = reinterpret_cast<const float4*>(a.h_in + ((int64_t)ui * ld + (r < rlim ? r : 0)) * TC_H + (ct >> 6) * 32);
#pragma unroll
          for (int i = 0; i < 8; ++i) hpre[i] = live ? hp[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int c8 = 0; c8 < 4; ++c8) {
          __align__(16) __nv_bfloat16 v[8];
          const float4 x0 = hpre[2 * c8], x1 = hpre[2 * c8 + 1];
          v[0] = __float2bfloat16_rn(x0.x); v[1] = __float2bfloat16_rn(x0.y); v[2] = __float2bfloat16_rn(x0.z); v[3] = __float2bfloat16_rn(x0.w);
          v[4] = __float2bfloat16_rn(x1.x); v[5] = __float2bfloat16_rn(x1.y); v[6] = __float2bfloat16_rn(x1.z); v[7] = __float2bfloat16_rn(x1.w);
          *reinterpret_cast<uint4*>(sA + (size_t)(KCX + (ct >> 6) * 4 + c8) * 1024 + (ct & 63) * 16) = *reinterpret_cast<const uint4*>(v);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        if (c == 0) asm volatile("bar.sync 1, 128;" ::: "memory");     // the whole tile of this consumer is written
        else asm volatile("bar.sync 2, 128;" ::: "memory");
        // st_x out of the tile, 32 bytes of a row per thread (the 8 lanes of a quarter-warp read 8 rows of one chunk
        // pair: no bank conflicts)
        if (!EVAL && a.st_x) {
          constexpr int np = DX / 16;
#pragma unroll 2
          for (int p = ct; p < P2_ROWS * np; p += 128) {
            const int rest = p >> 3, pcol = rest % np, row = (rest / np) * 8 + (p & 7);
            if (r0 + row < a.R) {
              const uint4 lo = *reinterpret_cast<const uint4*>(sA + (size_t)(2 * pcol) * 1024 + row * 16);
              const uint4 hi = *reinterpret_cast<const uint4*>(sA + (size_t)(2 * pcol + 1) * 1024 + row * 16);
              uint4* o = reinterpret_cast<uint4*>(a.st_x + store_row(row) * DX + 16 * pcol);
              o[0] = lo; o[1] = hi;
            }
          }
        }
        PROF_MARK(3);    // relu epilogue + h staging + st_x copy-out
        // ---- MMA1: gates[64 x 256] = [X | h][64 x K] . [Wx;Wh][K x 256], one m64n64 fragment per gate ----
        float g[4][32];
        // descriptors = base + address offset >> 4 (no carry out of the 14-bit field: shared addresses < 256 KB); the base
        // is made opaque here so that the 2 x 4 KS descriptors are formed at issue, not hoisted out of the item loop
        uint64_t dA1 = make_desc(aA, 1024, 128), dB1 = make_desc(aB, 4096, 128);
        asm volatile("" : "+l"(dA1), "+l"(dB1));
        wg_fence();
#pragma unroll
        for (int gi = 0; gi < 4; ++gi)
#pragma unroll
          for (int ks = 0; ks < KS; ++ks)
            wgmma_n64<0, 0>(g[gi], dA1 + (uint64_t)((ks * 2 * 1024) >> 4), dB1 + (uint64_t)((ks * 2 * 4096 + gi * 1024) >> 4),
                            ks > 0 ? 1u : 0u);
        wg_commit();
        wg_wait<0>();
#pragma unroll
        for (int gi = 0; gi < 4; ++gi) wg_frag_fence(g[gi]);
        mbar_arrive(empty);      // this thread is done with the tile (its st_x reads have returned)
        PROF_MARK(4);    // gate MMA issue + wait
        // ---- epilogue: the two fragment rows of this thread, 16 hidden units 16 q .. each ----
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int row = rq + 8 * hr;
          const int64_t r = r0 + row;
          const bool valid = r < rlim;
          const int64_t srow = ((int64_t)ui * ld + (valid ? r : 0)) * TC_H + 16 * q;
          float cprev[16];      // c_{t-1} of (row, hidden units 16 q ..), prefetched to L2 by the producer
          if (valid && !a.done) {
#pragma unroll
            for (int e4 = 0; e4 < 4; ++e4) {
              const float4 v = reinterpret_cast<const float4*>(a.c_in + srow)[e4];
              cprev[4 * e4] = v.x; cprev[4 * e4 + 1] = v.y; cprev[4 * e4 + 2] = v.z; cprev[4 * e4 + 3] = v.w;
            }
          } else {
#pragma unroll
            for (int e = 0; e < 16; ++e) cprev[e] = 0.f;
          }
          // fragment entry of (this row, hidden unit 16 q + e) in a gate's fragment
#define GF(gate, e) g[gate][4 * ((e) >> 1) + 2 * hr + ((e) & 1)]
          if (!EVAL && a.zdbg && valid) {
            float* z = a.zdbg + ((int64_t)u * ld + r) * TC_N + 16 * q;
#pragma unroll
            for (int e = 0; e < 16; ++e) { z[e] = GF(0, e); z[64 + e] = GF(1, e); z[128 + e] = GF(2, e); z[192 + e] = GF(3, e); }
          }
          float lg[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) lg[j] = 0.f;
          // bf16 gates / c / h packed in pairs as they are produced; the fp32 state leaves 4 units at a time
          uint32_t gw[4][8], cw[8], hw[8];
          float cn[4], hn[4];
          const bool st_row = !EVAL && valid && a.st_g;
          const int64_t m = st_row ? store_row(row) : 0;
#pragma unroll
          for (int e = 0; e < 16; ++e) {
            const int j = 16 * q + e;
            const float gi = sigm(GF(0, e) + sBias[j]), gf = sigm(GF(1, e) + sBias[64 + j]);
            const float go = sigm(GF(2, e) + sBias[128 + j]), gu = tanh_fast(GF(3, e) + sBias[192 + j]);
            const float c1 = gf * cprev[e] + gi * gu;
            const float h1 = go * tanh_fast(c1);
            cn[e & 3] = c1; hn[e & 3] = h1;
            const float gv[4] = {gi, gf, go, gu};
#pragma unroll
            for (int gg = 0; gg < 4; ++gg) bf16_pack(gw[gg][e >> 1], gv[gg], e & 1);
            bf16_pack(cw[e >> 1], c1, e & 1);
            bf16_pack(hw[e >> 1], h1, e & 1);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) lg[jj] = fmaf(h1, sWo[j * 8 + jj], lg[jj]);
            if ((e & 3) == 3 && valid) {
              reinterpret_cast<float4*>(a.c_out + srow)[e >> 2] = make_float4(cn[0], cn[1], cn[2], cn[3]);
              reinterpret_cast<float4*>(a.h_out + srow)[e >> 2] = make_float4(hn[0], hn[1], hn[2], hn[3]);
            }
            if ((e & 7) == 7 && st_row) {      // 16-byte halves of the 32-byte pieces
              const int hv = e >> 3;
#pragma unroll
              for (int gg = 0; gg < 4; ++gg)
                reinterpret_cast<uint4*>(a.st_g + m * TC_N + gg * 64 + 16 * q)[hv] =
                    make_uint4(gw[gg][4 * hv], gw[gg][4 * hv + 1], gw[gg][4 * hv + 2], gw[gg][4 * hv + 3]);
              reinterpret_cast<uint4*>(a.st_c + m * TC_H + 16 * q)[hv] = make_uint4(cw[4 * hv], cw[4 * hv + 1], cw[4 * hv + 2], cw[4 * hv + 3]);
              reinterpret_cast<uint4*>(a.st_h + m * TC_H + 16 * q)[hv] = make_uint4(hw[4 * hv], hw[4 * hv + 1], hw[4 * hv + 2], hw[4 * hv + 3]);
            }
          }
#undef GF
          // head sums over the quad's four 16-unit groups as ((g0 + g1) + (g2 + g3)) + bo (fp32 addition commutes, so
          // every lane ends with the same bits); lane q = hr finishes the row
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            lg[j] += __shfl_xor_sync(0xffffffffu, lg[j], 1);
            lg[j] += __shfl_xor_sync(0xffffffffu, lg[j], 2);
            lg[j] += sBo[j];
          }
          if (q == hr && valid) {
            if (EVAL || (u & 1) == 0) {
              float mx = -1e30f;
#pragma unroll
              for (int j = 0; j < 8; ++j) if (j < na) mx = fmaxf(mx, lg[j]);
              float sm = 0.f;
#pragma unroll
              for (int j = 0; j < 8; ++j) { lg[j] = j < na ? __expf(lg[j] - mx) : 0.f; sm += lg[j]; }
              const float inv = 1.0f / sm;
              float* po = a.pi + ((int64_t)r * d.A + ag) * d.max_na;
#pragma unroll
              for (int j = 0; j < 8; ++j) if (j < d.max_na) po[j] = lg[j] * inv;
              if (EVAL && a.act && a.act_mode == 1) {      // first maximum of the pi values written above (np.argmax)
                float best = lg[0] * inv;
                int pick = 0;
#pragma unroll
                for (int j = 1; j < 8; ++j)
                  if (j < na && lg[j] * inv > best) { best = lg[j] * inv; pick = j; }
                a.act[(int64_t)r * d.A + ag] = pick;
              } else if (a.act) {
                uint32_t hsh;
                if (GRP) {
                  // the member's key up to the replica term (xor is associative: the bits of the step-wise hash),
                  // and its replica index r - k Rm, of which the uint32 key sees the low word only
                  const uint32_t* g32 = reinterpret_cast<const uint32_t*>(sGrp);
                  hsh = pmix32(g32[2] ^ (((uint32_t)r - g32[3]) * 0x85EBCA77U));
                } else {
                  hsh = pmix32(a.seed_lo ^ (a.step * 0x9E3779B1U));
                  hsh = pmix32(hsh ^ a.seed_hi ^ ((uint32_t)(a.replica0 + r) * 0x85EBCA77U));
                }
                hsh = pmix32(hsh ^ ((uint32_t)ag * 0xC2B2AE3DU));
                const float uu = (float)(hsh >> 8) * (1.0f / 16777216.0f);
                float cum = 0.f;
                int pick = na - 1;
                bool found = false;
#pragma unroll
                for (int j = 0; j < 8; ++j)
                  if (j < na) { cum += lg[j] * inv; if (!found && uu < cum) { pick = j; found = true; } }
                a.act[(int64_t)r * d.A + ag] = pick;
              }
            } else if (!EVAL) {
              a.val[(int64_t)r * d.A + ag] = lg[0];
            }
          }
        }
        PROF_MARK(5);    // cell + stores + heads
      }
      seg = seg_hi;
    }
  }
#undef PROF_MARK
}

static size_t tc2_smem_bytes(int K) {
  const int KC = K / 8;
  return (size_t)KC * 4096 + (size_t)2 * KC * 1024 + (TC_H * 8 + 8 + TC_N + TC_N) * 4 + 4 * sizeof(uint64_t);
}

static unsigned long long* g_policy_prof = nullptr;
// tools only: device pointer to 16 uint64 counters that receive per-phase clock64 sums of the v2 kernel (NULL = off)
extern "C" int tscl_debug_policy_prof(void* counters_dev) { g_policy_prof = (unsigned long long*)counters_dev; return 0; }
static unsigned long long* g_bptt_prof = nullptr;
extern "C" int tscl_debug_bptt_prof(void* counters_dev) { g_bptt_prof = (unsigned long long*)counters_dev; return 0; }

extern "C" int tscl_policy_step_v2r(tscl_handle* h, const float* params, const void* wpack_bf16, const float* obs,
                                   int64_t R, const float* c_in, const float* h_in, float* c_out, float* h_out,
                                   float* pi, float* val, int32_t* act, int32_t done, uint64_t seed, int64_t step,
                                   int64_t replica0, float* zdbg, void* st_x, void* st_g, void* st_c, void* st_h,
                                   int32_t t, int32_t T, int64_t rc, int64_t ld_state, int64_t row0, void* stream) {
  if (!h || !params || !wpack_bf16 || !obs || R <= 0) return tsc_set_error("tscl_policy_step_v2r: bad argument");
  if (st_x && (rc <= 0 || (ld_state > 0 ? ld_state : R) % rc != 0)) return tsc_set_error("tscl_policy_step_v2r: store chunk must divide the replica count");
  if (ld_state > 0 && (row0 < 0 || row0 + R > ld_state)) return tsc_set_error("tscl_policy_step_v2r: replica range outside [0, ld_state)");
  PCK(cudaSetDevice(tscl_device_of(h)));
  const DDimsTC& d = *tscl_dims_of(h);
  const int K = d.dx + TC_H;
  if (!P2_DX_OK(d.dx)) return tsc_set_error("tscl_policy_step_v2r: no kernel for this dx (128, 160, 192 or 224)");
  if (d.kw == 0) return tsc_set_error("tscl_policy_step_v2r: observation slice does not fit the 64-column input tile");
  const size_t smem = tc2_smem_bytes(K);
  if (smem > 232448) return tsc_set_error("tscl_policy_step_v2r: operand tiles exceed shared memory");
  void (*kern)(const DDimsTC, const StepTC) = nullptr;
  const bool prof = g_policy_prof != nullptr;
#define P2_CASE(n) case n: kern = prof ? policy_step_tc2_kernel<n, true, false> : policy_step_tc2_kernel<n, false, false>; break;
  switch (d.dx) { P2_CASE(128) P2_CASE(160) P2_CASE(192) P2_CASE(224) }
#undef P2_CASE
  static int attr_dev = -1;
  static void (*attr_kern)(const DDimsTC, const StepTC) = nullptr;
  if (attr_dev != tscl_device_of(h) || attr_kern != kern) {
    PCK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    attr_dev = tscl_device_of(h); attr_kern = kern;
  }
  int n_sm = 0;
  PCK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, tscl_device_of(h)));
  const int64_t n_items = ((R + P2_ROWS - 1) / P2_ROWS) * 2 * d.A;
  const int grid = (int)(n_items < n_sm ? n_items : n_sm);
  StepTC a;
  a.acc = nullptr;
  a.P = params; a.Wp = (const __nv_bfloat16*)wpack_bf16; a.obs = obs; a.c_in = c_in; a.h_in = h_in; a.c_out = c_out;
  a.h_out = h_out; a.pi = pi; a.val = val; a.act = act; a.zdbg = zdbg; a.R = R; a.done = done; a.swap_lbo_sbo = 0;
  a.seed_lo = (uint32_t)seed; a.seed_hi = (uint32_t)(seed >> 32); a.step = (uint32_t)step; a.replica0 = replica0;
  a.st_x = (__nv_bfloat16*)st_x; a.st_g = (__nv_bfloat16*)st_g; a.st_c = (__nv_bfloat16*)st_c; a.st_h = (__nv_bfloat16*)st_h;
  a.t = t; a.T = T > 0 ? T : 1; a.rc = rc > 0 ? rc : R; a.ld = ld_state; a.row0 = ld_state > 0 ? row0 : 0;
  a.prof = g_policy_prof;
  a.act_mode = 0;
  kern<<<grid, P2_THREADS, smem, (cudaStream_t)stream>>>(d, a);
  PCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_policy_step_v2(tscl_handle* h, const float* params, const void* wpack_bf16, const float* obs, int64_t R,
                                   const float* c_in, const float* h_in, float* c_out, float* h_out, float* pi, float* val,
                                   int32_t* act, int32_t done, uint64_t seed, int64_t step, int64_t replica0, float* zdbg,
                                   void* st_x, void* st_g, void* st_c, void* st_h, int32_t t, int32_t T, int64_t rc,
                                   void* stream) {
  return tscl_policy_step_v2r(h, params, wpack_bf16, obs, R, c_in, h_in, c_out, h_out, pi, val, act, done, seed, step, replica0,
                              zdbg, st_x, st_g, st_c, st_h, t, T, rc, 0, 0, stream);
}

extern "C" int tscl_policy_step_v2g(tscl_handle* h, const float* params, int64_t p_stride, const void* wpack_bf16,
                                   int64_t wp_stride_m, const float* obs, int32_t K, int64_t Rm, const float* c_in,
                                   const float* h_in, float* c_out, float* h_out, float* pi, float* val, int32_t* act,
                                   int32_t done, const uint64_t* seeds, int64_t step, void* st_x, void* st_g, void* st_c,
                                   void* st_h, int32_t t, int32_t T, int64_t rc, void* stream) {
  if (!h || !params || !wpack_bf16 || !obs || !seeds || K < 1 || Rm <= 0) return tsc_set_error("tscl_policy_step_v2g: bad argument");
  if (Rm % P2_ROWS != 0) return tsc_set_error("tscl_policy_step_v2g: the member replica count must be a multiple of 64");
  if (st_x && (rc <= 0 || Rm % rc != 0)) return tsc_set_error("tscl_policy_step_v2g: store chunk must divide the member replica count");
  PCK(cudaSetDevice(tscl_device_of(h)));
  const DDimsTC& d = *tscl_dims_of(h);
  if (!P2_DX_OK(d.dx)) return tsc_set_error("tscl_policy_step_v2g: no kernel for this dx (128, 160, 192 or 224)");
  if (d.kw == 0) return tsc_set_error("tscl_policy_step_v2g: observation slice does not fit the 64-column input tile");
  if (K > 1 && (p_stride < d.n_params || wp_stride_m < 2 * d.A * wp_stride(d.dx)))
    return tsc_set_error("tscl_policy_step_v2g: member strides smaller than one member's parameters / image");
  const size_t smem = tc2_smem_bytes(d.dx + TC_H) + 16;      // + the block constants (sGrp)
  if (smem > 232448) return tsc_set_error("tscl_policy_step_v2g: operand tiles exceed shared memory");
  void (*kern)(const DDimsTC, const StepTC) = nullptr;
  switch (d.dx) {
    case 128: kern = policy_step_tc2_kernel<128, false, false, true>; break;
    case 160: kern = policy_step_tc2_kernel<160, false, false, true>; break;
    case 192: kern = policy_step_tc2_kernel<192, false, false, true>; break;
    case 224: kern = policy_step_tc2_kernel<224, false, false, true>; break;
  }
  static int attr_dev = -1;
  static void (*attr_kern)(const DDimsTC, const StepTC) = nullptr;
  if (attr_dev != tscl_device_of(h) || attr_kern != kern) {
    PCK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    attr_dev = tscl_device_of(h); attr_kern = kern;
  }
  int n_sm = 0;
  PCK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, tscl_device_of(h)));
  const int64_t R = (int64_t)K * Rm;
  const int64_t n_items = (R / P2_ROWS) * 2 * d.A;
  if (n_items > INT32_MAX) return tsc_set_error("tscl_policy_step_v2g: more than 2^31 work items");
  const int grid = (int)(n_items < n_sm ? n_items : n_sm);
  StepTC a{};
  a.P = params; a.Wp = (const __nv_bfloat16*)wpack_bf16; a.obs = obs; a.c_in = c_in; a.h_in = h_in; a.c_out = c_out;
  a.h_out = h_out; a.pi = pi; a.val = val; a.act = act; a.R = R; a.done = done;
  a.step = (uint32_t)step; a.replica0 = 0;
  a.st_x = (__nv_bfloat16*)st_x; a.st_g = (__nv_bfloat16*)st_g; a.st_c = (__nv_bfloat16*)st_c; a.st_h = (__nv_bfloat16*)st_h;
  a.t = t; a.T = T > 0 ? T : 1; a.rc = rc > 0 ? rc : Rm; a.ld = 0; a.row0 = 0;
  a.Rm = Rm; a.p_stride = p_stride; a.wp_stride = wp_stride_m; a.seeds = seeds;
  kern<<<grid, P2_THREADS, smem, (cudaStream_t)stream>>>(d, a);
  PCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_policy_step_pi(tscl_handle* h, const float* params, const void* wpack_bf16, const float* obs, int64_t R,
                                   const float* c_in, const float* h_in, float* c_out, float* h_out, float* pi, int32_t* act,
                                   int32_t act_mode, int32_t done, uint64_t seed, int64_t step, int64_t replica0,
                                   int64_t ld_state, int64_t row0, void* stream) {
  if (!h || !params || !wpack_bf16 || !obs || !c_in || !h_in || !c_out || !h_out || !pi || R <= 0)
    return tsc_set_error("tscl_policy_step_pi: bad argument");
  if (act_mode != 0 && act_mode != 1) return tsc_set_error("tscl_policy_step_pi: act_mode must be 0 (sample) or 1 (argmax)");
  if (ld_state > 0 && (row0 < 0 || row0 + R > ld_state)) return tsc_set_error("tscl_policy_step_pi: replica range outside [0, ld_state)");
  PCK(cudaSetDevice(tscl_device_of(h)));
  const DDimsTC& d = *tscl_dims_of(h);
  if (!P2_DX_OK(d.dx)) return tsc_set_error("tscl_policy_step_pi: no kernel for this dx (128, 160, 192 or 224)");
  if (d.kw == 0) return tsc_set_error("tscl_policy_step_pi: observation slice does not fit the 64-column input tile");
  const size_t smem = tc2_smem_bytes(d.dx + TC_H);
  if (smem > 232448) return tsc_set_error("tscl_policy_step_pi: operand tiles exceed shared memory");
  void (*kern)(const DDimsTC, const StepTC) = nullptr;
  switch (d.dx) {
    case 128: kern = policy_step_tc2_kernel<128, false, true>; break;
    case 160: kern = policy_step_tc2_kernel<160, false, true>; break;
    case 192: kern = policy_step_tc2_kernel<192, false, true>; break;
    case 224: kern = policy_step_tc2_kernel<224, false, true>; break;
  }
  static int attr_dev = -1;
  static void (*attr_kern)(const DDimsTC, const StepTC) = nullptr;
  if (attr_dev != tscl_device_of(h) || attr_kern != kern) {
    PCK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    attr_dev = tscl_device_of(h); attr_kern = kern;
  }
  int n_sm = 0;
  PCK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, tscl_device_of(h)));
  const int64_t n_items = ((R + P2_ROWS - 1) / P2_ROWS) * d.A;
  const int grid = (int)(n_items < n_sm ? n_items : n_sm);
  StepTC a{};
  a.P = params; a.Wp = (const __nv_bfloat16*)wpack_bf16; a.obs = obs; a.c_in = c_in; a.h_in = h_in; a.c_out = c_out;
  a.h_out = h_out; a.pi = pi; a.act = act; a.R = R; a.done = done;
  a.seed_lo = (uint32_t)seed; a.seed_hi = (uint32_t)(seed >> 32); a.step = (uint32_t)step; a.replica0 = replica0;
  a.t = 0; a.T = 1; a.rc = R; a.ld = ld_state; a.row0 = ld_state > 0 ? row0 : 0;
  a.act_mode = act_mode;
  kern<<<grid, P2_THREADS, smem, (cudaStream_t)stream>>>(d, a);
  PCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_policy_step_pi_g(tscl_handle* h, const float* params, int64_t p_stride, const void* wpack_bf16,
                                     int64_t wp_stride_m, const float* obs, int32_t K, const int64_t* rows, int64_t R,
                                     const float* c_in, const float* h_in, float* c_out, float* h_out, float* pi,
                                     int32_t* act, int32_t act_mode, int32_t done, const uint64_t* seeds, int64_t step,
                                     void* stream) {
  if (!h || !params || !wpack_bf16 || !obs || !rows || !seeds || !c_in || !h_in || !c_out || !h_out || !pi || K < 1 || R < K)
    return tsc_set_error("tscl_policy_step_pi_g: bad argument");
  if (act_mode != 0 && act_mode != 1) return tsc_set_error("tscl_policy_step_pi_g: act_mode must be 0 (sample) or 1 (argmax)");
  PCK(cudaSetDevice(tscl_device_of(h)));
  const DDimsTC& d = *tscl_dims_of(h);
  if (!P2_DX_OK(d.dx)) return tsc_set_error("tscl_policy_step_pi_g: no kernel for this dx (128, 160, 192 or 224)");
  if (d.kw == 0) return tsc_set_error("tscl_policy_step_pi_g: observation slice does not fit the 64-column input tile");
  if (K > 1 && (p_stride < d.n_params || wp_stride_m < 2 * d.A * wp_stride(d.dx)))
    return tsc_set_error("tscl_policy_step_pi_g: member strides smaller than one member's parameters / image");
  const size_t smem = tc2_smem_bytes(d.dx + TC_H) + 32;      // + the block constants (sGrp with the member's end row)
  if (smem > 232448) return tsc_set_error("tscl_policy_step_pi_g: operand tiles exceed shared memory");
  void (*kern)(const DDimsTC, const StepTC) = nullptr;
  switch (d.dx) {
    case 128: kern = policy_step_tc2_kernel<128, false, true, true>; break;
    case 160: kern = policy_step_tc2_kernel<160, false, true, true>; break;
    case 192: kern = policy_step_tc2_kernel<192, false, true, true>; break;
    case 224: kern = policy_step_tc2_kernel<224, false, true, true>; break;
  }
  static int attr_dev = -1;
  static void (*attr_kern)(const DDimsTC, const StepTC) = nullptr;
  if (attr_dev != tscl_device_of(h) || attr_kern != kern) {
    PCK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    attr_dev = tscl_device_of(h); attr_kern = kern;
  }
  int n_sm = 0;
  PCK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, tscl_device_of(h)));
  // the members' tiles sum to at most ceil(R / 64) + K - 1 (one partial tile per member); items past the last member's
  // are empty (grp_block), so the row boundaries stay on the device
  const int64_t n_items = ((R + P2_ROWS - 1) / P2_ROWS + K - 1) * d.A;
  if (n_items > INT32_MAX) return tsc_set_error("tscl_policy_step_pi_g: more than 2^31 work items");
  const int grid = (int)(n_items < n_sm ? n_items : n_sm);
  StepTC a{};
  a.P = params; a.Wp = (const __nv_bfloat16*)wpack_bf16; a.obs = obs; a.c_in = c_in; a.h_in = h_in; a.c_out = c_out;
  a.h_out = h_out; a.pi = pi; a.act = act; a.R = R; a.done = done;
  a.step = (uint32_t)step; a.replica0 = 0;
  a.t = 0; a.T = 1; a.rc = R; a.ld = R; a.row0 = 0;
  a.act_mode = act_mode;
  a.p_stride = p_stride; a.wp_stride = wp_stride_m; a.seeds = seeds; a.rows = rows; a.K = K;
  kern<<<grid, P2_THREADS, smem, (cudaStream_t)stream>>>(d, a);
  PCK(cudaGetLastError());
  return 0;
}

// ===================================================================================================
// BPTT through the LSTM on the tensor cores (replaces lstm_seq_bwd_kernel of tsc_learn.cu).
// One CTA walks (unit, 128-replica tile) items; for t = T-1 .. 0:
//   thread = (replica row, 32 hidden units): cell backward from gate activations, c_t, c_{t-1} and the
//   incoming dh / dc  ->  dz (4 x 32) written fp32 in place over the gates (operand of the weight-gradient
//   GEMMs) and as bf16 into the A tile [128 x 256];  wgmma  D[128 x 64] = dz . Wh^T  (K = 256, N = 64)
//   -> accumulator tile -> the thread's 32 columns = dh_{t-1} carry.  dc / dh carries stay in registers.
#define BW_KC 32            // 256 / 8 K-chunks
__global__ void pack_wht_kernel(const DDimsTC d, const float* __restrict__ P, __nv_bfloat16* __restrict__ Wt) {
  const int u = blockIdx.y;
  const float* Wh = P + d.off_wh + (int64_t)u * TC_H * TC_N;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < BW_KC * TC_H; i += gridDim.x * blockDim.x) {
    const int kc = i / TC_H, n = i - kc * TC_H;
    __align__(16) __nv_bfloat16 v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = __float2bfloat16_rn(Wh[(int64_t)n * TC_N + kc * 8 + e]);
    *reinterpret_cast<uint4*>(Wt + (((int64_t)u * BW_KC + kc) * TC_H + n) * 8) = *reinterpret_cast<const uint4*>(v);
  }
}

// B operand of the fused dX = dZ . Wx^T product: element (kc, n, e) = Wx[n][kc * 8 + e], n = fc-output column (< dx)
__global__ void pack_wxt_kernel(const DDimsTC d, const float* __restrict__ P, __nv_bfloat16* __restrict__ Wxt) {
  const int u = blockIdx.y;
  const float* Wx = P + d.off_wx + (int64_t)u * d.dx * TC_N;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < BW_KC * d.dx; i += gridDim.x * blockDim.x) {
    const int kc = i / d.dx, n = i - kc * d.dx;
    __align__(16) __nv_bfloat16 v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = __float2bfloat16_rn(Wx[(int64_t)n * TC_N + kc * 8 + e]);
    *reinterpret_cast<uint4*>(Wxt + (((int64_t)u * BW_KC + kc) * d.dx + n) * 8) = *reinterpret_cast<const uint4*>(v);
  }
}
struct BwdTC {
  float* acc;                // accumulator tiles, one [128][ACC_COLS] fp32 tile per CTA (acc_tiles)
  const __nv_bfloat16* Wxt;  // optional [2A][32][dx][8] (tscl_pack_wxt): with dXb, dX = dZ . Wx^T is fused into the step
  __nv_bfloat16* dXb;        // optional [2A][T*Rc][dx] bf16
  const __nv_bfloat16* Wt;   // [2A][32][64][8]
  float* ZG;                 // [2A][T*Rc][256] gates in, dZ out
  const float* C;            // [2A][T*Rc][64]
  const float* dH;           // [2A][T*Rc][64]
  const float* c0;           // [2A][ld_state][64]
  const float* done;         // [T]
  int T;
  int64_t Rc, ld_state, r0;
  const __nv_bfloat16* Gb;   // optional: gate activations / c_t straight from the bf16 activation store
  const __nv_bfloat16* Cb;   //           ([2A][T*Rc][256] / [..][64]); when set, ZG is write-only and C is unused
  __nv_bfloat16* dZb;        // optional: dZ as bf16 [2A][T*Rc][256] (operand of the tensor-core weight-gradient kernels);
                             //           ZG may then be null (needs Gb / Cb)
  unsigned long long* prof;  // optional: phase counters of lstm_bwd_tc_regs_kernel (tscl_debug_bptt_prof)
  // lstm_bwd_tc_regs_kernel<., true> (tscl_lstm_seq_bwd_tc_heads): dH from h_t and the heads instead of a dH tensor
  const float* P;            // parameters (head weights / biases at off_wo / off_bo)
  const int32_t* act;        // [T][..][A] at the first chunk's first replica, row (t, r, a) at t * stride_t + r * A + a
  const float* Rs;
  const float* Adv;
  int64_t stride_t;
  float v_coef, beta, scale;
  float* stats;              // optional: agent 0's loss sums (policy, value, entropy) x scale
  float* G;                  // head weight / bias gradients are added here
  int n_chunks;              // consecutive chunks of Rc replicas ([n_chunks][2A][T][Rc][w] store blocks)
};

// NT = 512: thread = (replica row, 16 hidden units), one CTA per SM.
// NT = 256: thread = (replica row, 32 hidden units) processed 8 at a time, TWO CTAs per SM (<= 128 registers): while one
//           tile waits for its per-step MMA / barrier the other one has its loads in flight.
template <int NT>
__global__ void __launch_bounds__(NT, NT == 256 ? 2 : 1)
lstm_bwd_tc_kernel(const DDimsTC d, const BwdTC a) {
  constexpr int HPT = 8192 / NT;            // hidden units per thread
  constexpr int NSUB = HPT / 8;
  constexpr int NQ = NT / 128;              // hidden groups (threads per row)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const bool fuse_dx = a.dXb != nullptr;             // second product of the same dz tile: dX = dz . Wx^T (N = dx)
  const int dx = d.dx;
  unsigned char* sB = tc_smem;                       // 32 * 1024  : Wh^T image
  unsigned char* sA = sB + BW_KC * 1024;             // 32 * 2048  : dz tile
  uint64_t* sBar = reinterpret_cast<uint64_t*>(sA + BW_KC * 2048);
  unsigned char* sBx = sA + BW_KC * 2048 + 16;       // 32 * dx * 16 : Wx^T image (only when fuse_dx)
  const uint32_t bar = smem_u32(sBar);
  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  float* const acc = a.acc + (size_t)blockIdx.x * TC_M * ACC_COLS;
  const uint32_t aA = smem_u32(sA), aB = smem_u32(sB), aBx = smem_u32(sBx);
  const int64_t n_tiles = (a.Rc + TC_M - 1) / TC_M;
  const int64_t n_items = n_tiles * 2 * d.A;
  int cur_u = -1;
  uint32_t parity = 0;
  const int q = warp & 3, qt = warp >> 2;            // row quadrant of the accumulator tile, hidden-unit group
  const int row = q * 32 + lane, jq = qt * HPT;
  auto bf8 = [](const uint4 v, float* o) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) { o[2 * i] = __uint_as_float(w[i] << 16); o[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u); }
  };
  auto f8 = [](const float* p, float* o) {
    const float4 x = reinterpret_cast<const float4*>(p)[0], y = reinterpret_cast<const float4*>(p)[1];
    o[0] = x.x; o[1] = x.y; o[2] = x.z; o[3] = x.w; o[4] = y.x; o[5] = y.y; o[6] = y.z; o[7] = y.w;
  };
  for (int64_t it = blockIdx.x; it < n_items; it += gridDim.x) {
    const int u = (int)(it / n_tiles);
    const int64_t r = (it - (int64_t)u * n_tiles) * TC_M + row;
    const bool valid = r < a.Rc;
    __syncthreads();
    if (u != cur_u) {
      cur_u = u;
      const uint4* src = reinterpret_cast<const uint4*>(a.Wt + (int64_t)u * BW_KC * TC_H * 8);
      uint4* dst = reinterpret_cast<uint4*>(sB);
      for (int i = tid; i < BW_KC * TC_H; i += NT) dst[i] = src[i];
      if (fuse_dx) {
        const uint4* sx = reinterpret_cast<const uint4*>(a.Wxt + (int64_t)u * BW_KC * dx * 8);
        uint4* dxs = reinterpret_cast<uint4*>(sBx);
        for (int i = tid; i < BW_KC * dx; i += NT) dxs[i] = sx[i];
      }
    }
    float dc[HPT], dhc[HPT];
#pragma unroll
    for (int e = 0; e < HPT; ++e) { dc[e] = 0.f; dhc[e] = 0.f; }
    for (int t = a.T - 1; t >= 0; --t) {
      const float keep = 1.0f - a.done[t];
      const int64_t m = ((int64_t)u * a.T + t) * a.Rc + (valid ? r : 0);
      if (t > 0 && valid) {      // pull step t-1's operands towards L2 while step t is being processed
        const int64_t mp = m - a.Rc;
        constexpr int LP = 4 / NQ;                 // 128-byte lines of a 512-byte row per thread
#pragma unroll
        for (int ln = 0; ln < LP; ++ln) {
          const int li = qt * LP + ln;             // 0..3
          if (a.Gb) {
            asm volatile("prefetch.global.L2 [%0];" ::"l"(a.Gb + mp * TC_N + li * 64));
            if (li == 0) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.Cb + mp * TC_H));
            if (li == 1 && t > 1) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.Cb + (mp - a.Rc) * TC_H));
          } else {
            asm volatile("prefetch.global.L2 [%0];" ::"l"(a.ZG + mp * TC_N + li * 64));
            asm volatile("prefetch.global.L2 [%0];" ::"l"(a.ZG + mp * TC_N + li * 64 + 32));
            if (li < 2) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.C + mp * TC_H + li * 32));
          }
          if (li >= 2) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.dH + mp * TC_H + (li - 2) * 32));
        }
      }
#pragma unroll
      for (int jb = 0; jb < NSUB; ++jb) {
        const int jo = jq + jb * 8;
        float gi[8], gf[8], go[8], gu[8], ct[8], cp[8], dh[8];
        if (valid) {
          if (a.Gb) {
            const __nv_bfloat16* zb = a.Gb + m * TC_N + jo;
            bf8(*reinterpret_cast<const uint4*>(zb), gi); bf8(*reinterpret_cast<const uint4*>(zb + 64), gf);
            bf8(*reinterpret_cast<const uint4*>(zb + 128), go); bf8(*reinterpret_cast<const uint4*>(zb + 192), gu);
            bf8(*reinterpret_cast<const uint4*>(a.Cb + m * TC_H + jo), ct);
            if (t > 0) bf8(*reinterpret_cast<const uint4*>(a.Cb + (m - a.Rc) * TC_H + jo), cp);
            if (t == 0) f8(a.c0 + ((int64_t)u * a.ld_state + a.r0 + r) * TC_H + jo, cp);
            f8(a.dH + m * TC_H + jo, dh);
          } else {
            const float* z = a.ZG + m * TC_N + jo;
            f8(z, gi); f8(z + 64, gf); f8(z + 128, go); f8(z + 192, gu);
            f8(a.C + m * TC_H + jo, ct);
            f8(t > 0 ? a.C + (m - a.Rc) * TC_H + jo : a.c0 + ((int64_t)u * a.ld_state + a.r0 + r) * TC_H + jo, cp);
            f8(a.dH + m * TC_H + jo, dh);
          }
#pragma unroll
          for (int e = 0; e < 8; ++e) cp[e] *= keep;
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e) { gi[e] = gf[e] = go[e] = gu[e] = ct[e] = cp[e] = dh[e] = 0.f; }
        }
        float dzi[8], dzf[8], dzo[8], dzu[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int k = jb * 8 + e;
          const float dht = dh[e] + dhc[k];
          const float tc = tanh_fast(ct[e]);
          const float dcc = dc[k] + dht * go[e] * (1.0f - tc * tc);
          dzi[e] = dcc * gu[e] * gi[e] * (1.0f - gi[e]);
          dzf[e] = dcc * cp[e] * gf[e] * (1.0f - gf[e]);
          dzo[e] = dht * tc * go[e] * (1.0f - go[e]);
          dzu[e] = dcc * gi[e] * (1.0f - gu[e] * gu[e]);
          dc[k] = dcc * gf[e] * keep;
        }
        const float* srcs[4] = {dzi, dzf, dzo, dzu};
        if (valid && a.ZG) {
          float4* z = reinterpret_cast<float4*>(a.ZG + m * TC_N + jo);
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            z[g * 16] = make_float4(srcs[g][0], srcs[g][1], srcs[g][2], srcs[g][3]);
            z[g * 16 + 1] = make_float4(srcs[g][4], srcs[g][5], srcs[g][6], srcs[g][7]);
          }
        }
        // bf16 copies into the A tile: columns g*64 + jo .. +8  ->  chunk (g*64 + jo)/8, row `row`
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          __align__(16) __nv_bfloat16 v[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) v[e] = __float2bfloat16_rn(srcs[g][e]);
          *reinterpret_cast<uint4*>(sA + (size_t)((g * 64 + jo) >> 3) * 2048 + row * 16) = *reinterpret_cast<const uint4*>(v);
          if (valid && a.dZb) *reinterpret_cast<uint4*>(a.dZb + m * TC_N + g * 64 + jo) = *reinterpret_cast<const uint4*>(v);
        }
      }
      const bool need_dh = keep != 0.f && t > 0;
      if (need_dh || fuse_dx) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        if (warp < 8) {
          if (need_dh)
            wg_mma<0, 0>(acc, 0, TC_H, 16, false, [&](int ks, uint64_t& da, uint64_t& db) {
              da = make_desc(aA + ks * 2 * 2048, 2048, 128);
              db = make_desc(aB + ks * 2 * 1024, 1024, 128);
            });
          if (fuse_dx)      // same A tile, B = Wx^T image: chunk stride dx * 16 B, 8-row groups 128 B apart
            wg_mma<0, 0>(acc, 64, dx, 16, false, [&](int ks, uint64_t& da, uint64_t& db) {
              da = make_desc(aA + ks * 2 * 2048, 2048, 128);
              db = make_desc(aBx + (uint32_t)(ks * 2 * dx * 16), (uint32_t)(dx * 16), 128);
            });
          wg_mma_done(bar);
        }
        mbar_wait(bar, parity);
        parity ^= 1;
        if (need_dh) {
          float dhp[HPT];
#pragma unroll
          for (int c16 = 0; c16 < HPT / 16; ++c16)
            acc_ld16(acc, ((uint32_t)(q * 32) << 16) + (uint32_t)(jq + c16 * 16), dhp + c16 * 16);
#pragma unroll
          for (int e = 0; e < HPT; ++e) dhc[e] = dhp[e] * keep;
        } else {
#pragma unroll
          for (int e = 0; e < HPT; ++e) dhc[e] = 0.f;
        }
        if (fuse_dx) {        // this thread's share of the row: dx / NQ columns, 8 at a time -> bf16 -> one 16-byte store
          const int per = dx / NQ;
          for (int c8 = 0; c8 < per; c8 += 8) {
            float xv[8];
            acc_ld8(acc, ((uint32_t)(q * 32) << 16) + (uint32_t)(64 + qt * per + c8), xv);
            if (valid) {
              __align__(16) __nv_bfloat16 v[8];
#pragma unroll
              for (int e = 0; e < 8; ++e) v[e] = __float2bfloat16_rn(xv[e]);
              *reinterpret_cast<uint4*>(a.dXb + m * dx + qt * per + c8) = *reinterpret_cast<const uint4*>(v);
            }
          }
        }
      } else {
#pragma unroll
        for (int e = 0; e < HPT; ++e) dhc[e] = 0.f;
      }
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------
// BPTT with the recurrence in registers: the activation-store path of the training loop (gates / c from the bf16 store,
// dZ written as bf16).  Same operands, k-step order, per-element formulas and bf16 rounding points as
// lstm_bwd_tc_kernel<512>, hence the same bits.  A CTA takes the same (unit, 128-row tile) items; each of its two
// warpgroups owns 64 of the rows and runs its own step loop, and the two meet only between items (they share the
// unit's Wh^T image).
// Why no accumulator tile is needed: with k = gate * 64 + unit, k-step 4 g + c of an RS-form wgmma m64n64k16 takes from
// thread (warp w of the warpgroup, lane l) rows 16 w + l / 4 (+ 8) and units 16 c + 2 (l % 4) + {0, 1, 8, 9} of gate g.
// Over c = 0..3 those are units 8 j + 2 (l % 4) + {0, 1}, j = 0..7: exactly the accumulator columns the same thread
// holds for the same rows.  So the thread that computes dz for (row, unit, all four gates) supplies it as the A
// operand, and receives dh_{t-1} for that (row, unit) in its own accumulator.
// Per step and warpgroup:
//   1. wait on the warpgroup's mbarrier for step t's operands (TMA copies, 128-byte swizzle);
//   2. ldmatrix (gates, c_t, c_{t-1}: the fragment layout straight out of the swizzled boxes), 8-byte reads for dH;
//   3. warpgroup barrier, then one thread issues step t-1's copies into the buffers just read;
//   4. cell backward -> the 16 A fragments (bf16 pairs, lower column in the low half) and the dc carry;
//   5. stmatrix of the fragments into a swizzled staging tile, 16 RS wgmmas, warpgroup barrier, TMA store of dZ;
//   6. wait for the MMA: dh_{t-1} = accumulator * keep is the next step's carry.
// The tensor maps are 3-D [2A * T][Rc][cols], so every copy is clipped at Rc: rows past Rc read as zero and are never
// written, and no copy reaches another step's rows.
#define BR_WG_BYTES (96 * 1024)   // per warpgroup: gates 4 x 8 KB | dH 2 x 8 KB | c ring 2 x 8 KB | dZ staging 4 x 8 KB
#define BR_SMEM (BW_KC * 1024 + 2 * BR_WG_BYTES + 16)
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void stsm_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};"
               ::"r"(addr), "r"(r0), "r"(r1), "r"(r2), "r"(r3) : "memory");
}
// bf16 pair, `lo` in the low half (round to nearest even, as __float2bfloat16_rn)
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
// m64n64k16 with A from registers (this thread's four bf16 pairs) and B K-major in shared memory
__device__ __forceinline__ void wgmma_n64_rs(float (&d)[32], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t db,
                                             uint32_t accum) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(db), "r"(accum) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, int x, int y, int z, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(x), "r"(y), "r"(z), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, int x, int y, int z, uint32_t src) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(x), "r"(y), "r"(z), "r"(src) : "memory");
}

// Loss gradients at the heads for one step of a warpgroup of lstm_bwd_tc_regs_kernel<., true>: the thread's rows
// rr0, rr0 + 8 of the chunk (rg0, rg0 + 8 of the update), h_t in the swizzled tile sH.  Writes dht = dH + dhc for the
// thread's 16 units (the register layout of the kernel), the rows' dlog into sDl (value unit: dv in slot 0) and adds
// agent 0's loss terms.  The per-row arithmetic is heads_loss_kernel's (tsc_learn.cu), expression for expression.
__device__ __forceinline__ void heads_step(const DDimsTC& d, const BwdTC& a, const unsigned char* sH, const float* sHW,
                                           float* sDl, bool pol, int ag, int na, int rq, int rr0, int lane, int q,
                                           int64_t rg0, int t, const float (&dhc)[8][4], float (&dht)[8][4], float& pl,
                                           float& vl, float& el) {
  constexpr int HB_DL = 12;
  const float* sWp = sHW;                  // [64][8]
  const float* sWv = sHW + 512;            // [64]
  const float* sBo = sHW + 576;            // [8]
  bool valid[2];
  int64_t io[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    valid[h] = rr0 + 8 * h < a.Rc;
    io[h] = valid[h] ? (int64_t)t * a.stride_t + (rg0 + 8 * h) * d.A + ag : 0;
  }
  auto row8 = [&](int h, int c, float* x) {   // h[row rq + 8 h][8 c .. 8 c + 7] as fp32
    const uint4 v = *reinterpret_cast<const uint4*>(sH + (rq + 8 * h) * 128 + ((c ^ (rq & 7)) << 4));
    const uint32_t wv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) { x[2 * i] = __uint_as_float(wv[i] << 16); x[2 * i + 1] = __uint_as_float(wv[i] & 0xffff0000u); }
  };
  if (pol) {
    // logits 2 q, 2 q + 1 of both rows: each its own sequential chain over k
    float l[2][2];
#pragma unroll
    for (int h = 0; h < 2; ++h) { l[h][0] = sBo[2 * q]; l[h][1] = sBo[2 * q + 1]; }
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      float x[2][8];
      row8(0, c, x[0]); row8(1, c, x[1]);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float2 wv = *reinterpret_cast<const float2*>(sWp + (8 * c + e) * 8 + 2 * q);
#pragma unroll
        for (int h = 0; h < 2; ++h) { l[h][0] = fmaf(x[h][e], wv.x, l[h][0]); l[h][1] = fmaf(x[h][e], wv.y, l[h][1]); }
      }
    }
    float dl[2][8];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float lg[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) lg[j] = __shfl_sync(0xffffffffu, l[h][j & 1], (lane & ~3) | (j >> 1));
#pragma unroll
      for (int j = 0; j < 8; ++j) dl[h][j] = 0.f;
      if (valid[h]) {
        float mx = -1e30f;
#pragma unroll
        for (int j = 0; j < 8; ++j) if (j < na) mx = fmaxf(mx, lg[j]);
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) { lg[j] = j < na ? __expf(lg[j] - mx) : 0.f; s += lg[j]; }
        const float inv = 1.0f / s;
        const int at = a.act[io[h]];
        const float adv = a.Adv[io[h]];
        // log(clip(pi, 1e-10, 1)) and its gradient: see heads_loss_kernel
        float lp[8], ent = 0.f, clip_mass = 0.f;
        bool in_at = true;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          lg[j] *= inv;                                             // pi_j
          lp[j] = j < na ? __logf(fminf(fmaxf(lg[j], 1e-10f), 1.0f)) : 0.f;
          ent -= lg[j] * lp[j];
          const bool clipped = j < na && !(lg[j] >= 1e-10f && lg[j] <= 1.0f);
          if (clipped) clip_mass += lg[j];
          if (clipped && j == at) in_at = false;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float g = 0.f;
          if (j < na) {
            const bool clipped = !(lg[j] >= 1e-10f && lg[j] <= 1.0f);
            const float pg = in_at ? -adv * ((j == at ? 1.f : 0.f) - lg[j]) : 0.f;
            g = a.scale * (pg + a.beta * lg[j] * (lp[j] + ent + clip_mass - (clipped ? 1.f : 0.f)));
          }
          dl[h][j] = g;
        }
        if (ag == 0 && q == 0) {
#pragma unroll
          for (int j = 0; j < 8; ++j) if (j == at) pl += -lp[j] * adv;
          el += -a.beta * ent;
        }
      }
      float s0 = 0.f, s1 = 0.f;              // this thread's share of the staging row: dlog 2 q, 2 q + 1
#pragma unroll
      for (int j = 0; j < 8; j += 2) if ((j >> 1) == q) { s0 = dl[h][j]; s1 = dl[h][j + 1]; }
      *reinterpret_cast<float2*>(sDl + (rq + 8 * h) * HB_DL + 2 * q) = make_float2(s0, s1);
    }
    // dH[k] = sum_j dlog_j Wp[k][j] in heads_loss_kernel's order, for the thread's units k = 8 j + 2 q + e
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int k = 8 * j + 2 * q + e;
        const float4 w0 = *reinterpret_cast<const float4*>(sWp + k * 8), w1 = *reinterpret_cast<const float4*>(sWp + k * 8 + 4);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float tt = 0.f;
          tt = fmaf(dl[h][0], w0.x, tt); tt = fmaf(dl[h][1], w0.y, tt); tt = fmaf(dl[h][2], w0.z, tt); tt = fmaf(dl[h][3], w0.w, tt);
          tt = fmaf(dl[h][4], w1.x, tt); tt = fmaf(dl[h][5], w1.y, tt); tt = fmaf(dl[h][6], w1.z, tt); tt = fmaf(dl[h][7], w1.w, tt);
          dht[j][2 * h + e] = (valid[h] ? tt : 0.f) + dhc[j][2 * h + e];
        }
      }
  } else {
    float v[2] = {sBo[0], sBo[0]};
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      float x[2][8];
      row8(0, c, x[0]); row8(1, c, x[1]);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float wv = sWv[8 * c + e];
        v[0] = fmaf(x[0][e], wv, v[0]); v[1] = fmaf(x[1][e], wv, v[1]);
      }
    }
    float dv[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      dv[h] = 0.f;
      if (valid[h]) {
        const float ret = a.Rs[io[h]];
        dv[h] = a.scale * a.v_coef * (v[h] - ret);
        if (ag == 0 && q == 0) vl += 0.5f * a.v_coef * (ret - v[h]) * (ret - v[h]);
      }
      *reinterpret_cast<float2*>(sDl + (rq + 8 * h) * HB_DL + 2 * q) = make_float2(q == 0 ? dv[h] : 0.f, 0.f);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float wv = sWv[8 * j + 2 * q + e];
#pragma unroll
        for (int h = 0; h < 2; ++h) dht[j][2 * h + e] = (valid[h] ? __fmul_rn(dv[h], wv) : 0.f) + dhc[j][2 * h + e];
      }
  }
}

// PROF: clock64 phase sums of thread 0 of every warpgroup into a.prof[0..3] (operand wait | smem -> regs + cell backward |
// MMA issue -> wait | dZ store), a separate instantiation (tscl_debug_bptt_prof)
//
// HEADS: the loss gradients at the heads are computed here instead of read from a dH tensor (tscl_lstm_seq_bwd_tc_heads).
// mapD is then the bf16 h store ([.][T][Rc][64]); the warpgroup's 8 KB h_t tile takes the first half of the dH space,
// on its own mbarrier, and is refilled with h_{t-1} once the step's readers are past the staging barrier.  Per step:
//   after the operand wait, the quad of threads that share rows rq, rq + 8 computes each row's logits (policy unit:
//   thread q the logits 2 q, 2 q + 1, the sequential fmaf chain over k = 0..63 of heads_loss_kernel; value unit: every
//   thread the whole v chain), gathers them by shuffles (no arithmetic), and repeats heads_loss_kernel's per-row loss
//   arithmetic and its 8-term dH chains for the thread's own 16 units.  dH is therefore the bits tscl_heads_loss
//   writes, and dZ the bits of the tscl_heads_loss -> tscl_lstm_seq_bwd_tc pair.  The rows' dlog go to a small
//   staging tile; while the step's MMA runs, thread (k, logits 4 hh..4 hh + 3) adds h[row][k] * dlog[row][j] over the
//   warpgroup's 64 rows into registers, flushed to G with one atomic per output at every unit change.
// Items run over n_chunks consecutive chunks (chunk-outermost, the activation store's order).
template <bool PROF, bool HEADS = false>
__global__ void __launch_bounds__(256, 1)
lstm_bwd_tc_regs_kernel(const DDimsTC d, const BwdTC a, const __grid_constant__ CUtensorMap mapG,
                        const __grid_constant__ CUtensorMap mapC, const __grid_constant__ CUtensorMap mapD,
                        const __grid_constant__ CUtensorMap mapZ) {
  const int tid = threadIdx.x, wg = tid >> 7, w = (tid >> 5) & 3, lane = tid & 31, q = lane & 3;
  const bool lead = (tid & 127) == 0;
  long long bp[4] = {0, 0, 0, 0}, pc = 0;
#define BR_MARK(i) do { if (PROF && lead) { const long long c_ = clock64(); bp[i] += c_ - pc; pc = c_; } } while (0)
  unsigned char* sB = tc_smem;                                       // 32 KB: Wh^T image, shared by both warpgroups
  unsigned char* sW = sB + BW_KC * 1024 + wg * BR_WG_BYTES;          // this warpgroup's buffers (1024-byte aligned)
  const uint32_t aB = smem_u32(sB), aG = smem_u32(sW), aD = aG + 32768, aC = aG + 49152, aZ = aG + 65536;
  const uint32_t ldbar = smem_u32(sB + BW_KC * 1024 + 2 * BR_WG_BYTES) + 8 * wg;
  // HEADS: in the dH space of each warpgroup, h_t tile [64][128 B] | dlog staging [64][HB_DL] fp32 | (warpgroup 0 only)
  // the unit's head weights [64][8] (padded to 8 logits), Wv [64], biases [8] | h mbarrier
  constexpr int HB_DL = 12;
  const unsigned char* sH = sW + 32768;
  float* sDl = reinterpret_cast<float*>(sW + 40960);
  float* sHW = reinterpret_cast<float*>(sB + BW_KC * 1024 + 40960 + 64 * HB_DL * 4);
  const uint32_t hbar = aG + 47104;
  if (lead) {
    mbar_init(ldbar, 1);
    if (HEADS) mbar_init(hbar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // ldmatrix / stmatrix lane address in a [64 rows][128 B] swizzled box for 16-byte chunks 2 c, 2 c + 1: lanes 0-7 / 8-15 /
  // 16-23 / 24-31 give the rows of matrices (rows 16 w.., chunk 2 c) / (rows 16 w + 8.., 2 c) / (16 w.., 2 c + 1) /
  // (16 w + 8.., 2 c + 1), which are this thread's fragment registers (j = 2 c, row r) (2 c, r + 8) (2 c + 1, r) (2 c + 1, r + 8)
  const uint32_t lm_row = (uint32_t)(16 * w + (lane & 7) + ((lane >> 3) & 1) * 8) * 128, lm_sw = lane & 7, lm_hi = lane >> 4;
  auto lm = [&](uint32_t box, int c) { return box + lm_row + (((2 * c + lm_hi) ^ lm_sw) << 4); };
  const int rq = 16 * w + (lane >> 2);                               // the thread's rows: rq, rq + 8 of the warpgroup's 64
  const int64_t n_tiles = (a.Rc + TC_M - 1) / TC_M;
  const int64_t per_chunk = n_tiles * 2 * d.A;
  const int64_t n_items = per_chunk * (HEADS ? a.n_chunks : 1);
  int cur_u = -1;
  uint32_t ldpar = 0, hpar = 0;
  // HEADS: head weight / bias gradient sums of the current unit, thread = (hidden unit hk, logits 4 hh .. 4 hh + 3)
  const int hk = tid & 63, hh = (tid >> 6) & 1;
  float gw[4] = {0.f, 0.f, 0.f, 0.f}, gb = 0.f, pl = 0.f, vl = 0.f, el = 0.f;
  auto flush = [&](int uu) {
    const int nl = (uu & 1) ? 1 : d.max_na;                          // value units have one output
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      if (hh * 4 + jj < nl) atomicAdd(&a.G[d.off_wo + ((int64_t)uu * TC_H + hk) * d.max_na + hh * 4 + jj], gw[jj]);
      gw[jj] = 0.f;
    }
    if ((tid & 127) < nl) atomicAdd(&a.G[d.off_bo + (int64_t)uu * d.max_na + (tid & 127)], gb);
    gb = 0.f;
  };
  for (int64_t it = blockIdx.x; it < n_items; it += gridDim.x) {
    const int ci = HEADS ? (int)(it / per_chunk) : 0;                // chunk of the item
    const int64_t ic = it - (int64_t)ci * per_chunk;
    const int u = (int)(ic / n_tiles);
    const int rw0 = (int)((ic - (int64_t)u * n_tiles) * TC_M) + 64 * wg;   // first row of this warpgroup
    __syncthreads();                                                 // both warpgroups are done with the previous item
    if (u != cur_u) {
      if (HEADS && cur_u >= 0) flush(cur_u);
      cur_u = u;
      const uint4* src = reinterpret_cast<const uint4*>(a.Wt + (int64_t)u * BW_KC * TC_H * 8);
      uint4* dst = reinterpret_cast<uint4*>(sB);
      for (int i = tid; i < BW_KC * TC_H; i += 256) dst[i] = src[i];
      if (HEADS) {       // the unit's head weights and biases, padded to 8 logits as heads_loss_kernel pads them
        const int mna = d.max_na;
        const float* wo = a.P + d.off_wo + (int64_t)u * TC_H * mna;
        for (int i = tid; i < TC_H * 8; i += 256) { const int k = i >> 3, j = i & 7; sHW[i] = j < mna ? wo[k * mna + j] : 0.f; }
        if (tid < TC_H) sHW[512 + tid] = wo[tid * mna];
        if (tid < 8) sHW[576 + tid] = tid < mna ? a.P[d.off_bo + (int64_t)u * mna + tid] : 0.f;
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic writes -> operand of the wgmmas
      __syncthreads();
    }
    if (rw0 >= a.Rc) continue;                                       // a partial tile with no row for this warpgroup
    const int z0 = (ci * 2 * d.A + u) * a.T;                         // plane of step 0 in the [2A * T][Rc][cols] maps
    // step t's gates and dH, c_{t-1} into its ring slot, and c_t as well for the item's first step (lead thread)
    auto fetch = [&](int t, bool with_c_t) {
      mbar_expect_tx(ldbar, (uint32_t)(32768 + (HEADS ? 0 : 16384) + (with_c_t ? 8192 : 0) + (t > 0 ? 8192 : 0)));
#pragma unroll
      for (int g = 0; g < 4; ++g) tma_load_3d(aG + g * 8192, &mapG, g * 64, rw0, z0 + t, ldbar);
      if (!HEADS) {
        tma_load_3d(aD, &mapD, 0, rw0, z0 + t, ldbar);
        tma_load_3d(aD + 8192, &mapD, 32, rw0, z0 + t, ldbar);
      }
      if (with_c_t) tma_load_3d(aC + (t & 1) * 8192, &mapC, 0, rw0, z0 + t, ldbar);
      if (t > 0) tma_load_3d(aC + ((t - 1) & 1) * 8192, &mapC, 0, rw0, z0 + t - 1, ldbar);
    };
    auto fetch_h = [&](int t) {                                      // HEADS: h_t of this warpgroup's rows
      mbar_expect_tx(hbar, 8192u);
      tma_load_3d(aD, &mapD, 0, rw0, z0 + t, hbar);
    };
    if (lead) {
      fetch(a.T - 1, true);
      if (HEADS) fetch_h(a.T - 1);
    }
    // HEADS: the item's agent, and this thread's rows as rows of the whole update (act / Rs / Adv index)
    const int ag = u >> 1, na = HEADS ? d.n_a[ag] : 0;
    const bool pol = (u & 1) == 0;
    const int64_t rg0 = (int64_t)ci * a.Rc + rw0 + rq;
    // per-thread state, entry [j][e]: row rq + 8 (e >> 1), unit 8 j + 2 q + (e & 1) (= accumulator entry 4 j + e)
    float dc[8][4], dhc[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) { dc[j][e] = 0.f; dhc[j][e] = 0.f; }
    if (PROF && lead) pc = clock64();
    for (int t = a.T - 1; t >= 0; --t) {
      const float keep = 1.0f - a.done[t];
      mbar_wait(ldbar, ldpar); ldpar ^= 1;                           // step t's operands have landed
      if (HEADS) { mbar_wait(hbar, hpar); hpar ^= 1; }               // and h_t
      BR_MARK(0);
      float dht[8][4];                                               // dH + dh carry
      if constexpr (HEADS) heads_step(d, a, sH, sHW, sDl, pol, ag, na, rq, rw0 + rq, lane, q, rg0, t, dhc, dht, pl, vl, el);
      // shared memory -> registers; bf16 pairs [j][h]: row rq + 8 h, units 8 j + 2 q + {0 (low half), 1}
      uint32_t gr[4][8][2], cr[8][2], pr[8][2];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        uint32_t r[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          ldsm_x4(r, lm(aG + g * 8192, c));
          gr[g][2 * c][0] = r[0]; gr[g][2 * c][1] = r[1]; gr[g][2 * c + 1][0] = r[2]; gr[g][2 * c + 1][1] = r[3];
        }
        ldsm_x4(r, lm(aC + (t & 1) * 8192, c));
        cr[2 * c][0] = r[0]; cr[2 * c][1] = r[1]; cr[2 * c + 1][0] = r[2]; cr[2 * c + 1][1] = r[3];
        if (t > 0) {
          ldsm_x4(r, lm(aC + ((t - 1) & 1) * 8192, c));
          pr[2 * c][0] = r[0]; pr[2 * c][1] = r[1]; pr[2 * c + 1][0] = r[2]; pr[2 * c + 1][1] = r[3];
        }
      }
      if constexpr (!HEADS) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = rq + 8 * h;
            const float2 v = *reinterpret_cast<const float2*>(sW + 32768 + (j >> 2) * 8192 + row * 128 +
                                                             (((2 * (j & 3) + (q >> 1)) ^ (row & 7)) << 4) + 8 * (q & 1));
            dht[j][2 * h] = v.x + dhc[j][2 * h];
            dht[j][2 * h + 1] = v.y + dhc[j][2 * h + 1];
          }
      }
      if (lead) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // the last dZ store has left the staging tile
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");    // the operand buffers are free
      if (lead && t > 0) fetch(t - 1, false);
      // cell backward (the formulas of lstm_bwd_tc_kernel) -> A fragments af[g][j][h]
      uint32_t af[4][8][2];
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float cp2[2];
          if (t > 0) {
            cp2[0] = bf16_lo(pr[j][h]); cp2[1] = bf16_hi(pr[j][h]);
          } else {
            const int64_t r = rw0 + rq + 8 * h;
            float2 v = make_float2(0.f, 0.f);
            if (r < a.Rc)
              v = *reinterpret_cast<const float2*>(a.c0 + ((int64_t)u * a.ld_state + a.r0 + (int64_t)ci * a.Rc + r) * TC_H +
                                                   8 * j + 2 * q);
            cp2[0] = v.x; cp2[1] = v.y;
          }
          float z[4][2];
#pragma unroll
          for (int ee = 0; ee < 2; ++ee) {
            const int e = 2 * h + ee;
            const float gi = ee ? bf16_hi(gr[0][j][h]) : bf16_lo(gr[0][j][h]);
            const float gf = ee ? bf16_hi(gr[1][j][h]) : bf16_lo(gr[1][j][h]);
            const float go = ee ? bf16_hi(gr[2][j][h]) : bf16_lo(gr[2][j][h]);
            const float gu = ee ? bf16_hi(gr[3][j][h]) : bf16_lo(gr[3][j][h]);
            const float ct = ee ? bf16_hi(cr[j][h]) : bf16_lo(cr[j][h]);
            const float cp = cp2[ee] * keep;
            const float dh = dht[j][e];
            const float tc = tanh_fast(ct);
            const float dcc = dc[j][e] + dh * go * (1.0f - tc * tc);
            z[0][ee] = dcc * gu * gi * (1.0f - gi);
            z[1][ee] = dcc * cp * gf * (1.0f - gf);
            z[2][ee] = dh * tc * go * (1.0f - go);
            z[3][ee] = dcc * gi * (1.0f - gu * gu);
            dc[j][e] = dcc * gf * keep;
          }
#pragma unroll
          for (int g = 0; g < 4; ++g) af[g][j][h] = pack_bf16x2(z[g][0], z[g][1]);
        }
      BR_MARK(1);
#pragma unroll
      for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int c = 0; c < 4; ++c)
          stsm_x4(lm(aZ + g * 8192, c), af[g][2 * c][0], af[g][2 * c][1], af[g][2 * c + 1][0], af[g][2 * c + 1][1]);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // staging tile -> the TMA store
      BR_MARK(3);
      // The MMA is issued on every step (a branch around it makes ptxas serialise the wgmmas); its result is used only
      // where lstm_bwd_tc_kernel runs it, keep != 0 and t > 0.
      float acc[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] = 0.f;
      wg_fence();
#pragma unroll
      for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int c = 0; c < 4; ++c)                                  // k-step 4 g + c, in order
          wgmma_n64_rs(acc, af[g][2 * c][0], af[g][2 * c][1], af[g][2 * c + 1][0], af[g][2 * c + 1][1],
                       make_desc(aB + (4 * g + c) * 2 * 1024, 1024, 128), (g | c) != 0);
      wg_commit();
      BR_MARK(2);
      if constexpr (HEADS) {     // head weight / bias gradients of step t while the MMA runs (dlog staged before bar 1)
#pragma unroll 8
        for (int row = 0; row < 64; ++row) {
          const uint16_t hb = *reinterpret_cast<const uint16_t*>(sH + row * 128 + (((hk >> 3) ^ (row & 7)) << 4) + (hk & 7) * 2);
          const float x = __uint_as_float((uint32_t)hb << 16);
          const float4 g4 = *reinterpret_cast<const float4*>(sDl + row * HB_DL + hh * 4);
          gw[0] = fmaf(x, g4.x, gw[0]); gw[1] = fmaf(x, g4.y, gw[1]);
          gw[2] = fmaf(x, g4.z, gw[2]); gw[3] = fmaf(x, g4.w, gw[3]);
        }
        if ((tid & 127) < 8)
          for (int row = 0; row < 64; ++row) gb += sDl[row * HB_DL + (tid & 127)];
      }
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");    // the whole staging tile is written
      if (lead) {
#pragma unroll
        for (int g = 0; g < 4; ++g) tma_store_3d(&mapZ, g * 64, rw0, z0 + t, aZ + g * 8192);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        if (HEADS && t > 0) fetch_h(t - 1);                          // every reader of h_t / dlog is past the barrier
      }
      BR_MARK(3);
      wg_wait<0>();
      wg_frag_fence(acc);
      const bool need_dh = keep != 0.f && t > 0;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) dhc[j][e] = need_dh ? acc[4 * j + e] * keep : 0.f;
      BR_MARK(2);
    }
  }
  if (lead) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // dZ stores complete before the CTA leaves
  if (HEADS) {
    if (cur_u >= 0) flush(cur_u);
    if (a.stats) {
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        pl += __shfl_down_sync(0xffffffffu, pl, o);
        vl += __shfl_down_sync(0xffffffffu, vl, o);
        el += __shfl_down_sync(0xffffffffu, el, o);
      }
      if (lane == 0 && (pl != 0.f || vl != 0.f || el != 0.f)) {
        atomicAdd(&a.stats[0], pl * a.scale); atomicAdd(&a.stats[1], vl * a.scale); atomicAdd(&a.stats[2], el * a.scale);
      }
    }
  }
  if (PROF && lead)
    for (int i = 0; i < 4; ++i) atomicAdd(a.prof + i, (unsigned long long)bp[i]);
#undef BR_MARK
}

// 3-D tiled tensor map over row-major [planes][rows][cols] (box = box_cols x box_rows x 1, inner box = 128 bytes,
// 128-byte swizzle unless `sw` says otherwise) through the driver entry point (no link-time dependency on libcuda)
static bool make_tmap_3d(CUtensorMap* m, CUtensorMapDataType dt, int elem_bytes, const void* base, uint64_t planes,
                         uint64_t rows, uint64_t cols, uint32_t box_cols, uint32_t box_rows,
                         CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B) {
  typedef CUresult (*encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static encode_fn fn = []() -> encode_fn {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      return nullptr;
    return (encode_fn)p;
  }();
  if (!fn || !base) return false;
  memset(m, 0, sizeof(*m));
  const cuuint64_t dims[3] = {cols, rows, planes};
  const cuuint64_t strides[2] = {cols * (uint64_t)elem_bytes, rows * cols * (uint64_t)elem_bytes};
  const cuuint32_t box[3] = {box_cols, box_rows, 1};
  const cuuint32_t es[3] = {1, 1, 1};
  return fn(m, dt, 3, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// 16-byte cp.async global -> shared (the dX kernel's operand loader)
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}

extern "C" int tscl_pack_wxt(tscl_handle* h, const float* params, void* wxt_bf16, void* stream) {
  if (!h || !params || !wxt_bf16) return tsc_set_error("tscl_pack_wxt: bad argument");
  PCK(cudaSetDevice(tscl_device_of(h)));
  const DDimsTC& d = *tscl_dims_of(h);
  pack_wxt_kernel<<<dim3(8, 2 * d.A), 256, 0, (cudaStream_t)stream>>>(d, params, (__nv_bfloat16*)wxt_bf16);
  PCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_pack_wht(tscl_handle* h, const float* params, void* wt_bf16, void* stream) {
  if (!h || !params || !wt_bf16) return tsc_set_error("tscl_pack_wht: bad argument");
  PCK(cudaSetDevice(tscl_device_of(h)));
  const DDimsTC& d = *tscl_dims_of(h);
  pack_wht_kernel<<<dim3(2, 2 * d.A), 256, 0, (cudaStream_t)stream>>>(d, params, (__nv_bfloat16*)wt_bf16);
  PCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_lstm_seq_bwd_tc(tscl_handle* h, const void* wt_bf16, float* ZG, const float* C, const float* dH,
                                    const float* c0, const float* done, int32_t T, int64_t Rc, int64_t ld_state,
                                    int64_t r0, const void* gates_bf16, const void* c_bf16, void* dz_bf16, void* stream) {
  return tscl_lstm_seq_bwd_tc_dx(h, wt_bf16, ZG, C, dH, c0, done, T, Rc, ld_state, r0, gates_bf16, c_bf16, dz_bf16, nullptr,
                                 nullptr, stream);
}

extern "C" int tscl_lstm_seq_bwd_tc_dx(tscl_handle* h, const void* wt_bf16, float* ZG, const float* C, const float* dH,
                                       const float* c0, const float* done, int32_t T, int64_t Rc, int64_t ld_state,
                                       int64_t r0, const void* gates_bf16, const void* c_bf16, void* dz_bf16,
                                       const void* wxt_bf16, void* dx_bf16, void* stream) {
  if (!h || !wt_bf16 || T <= 0 || Rc <= 0) return tsc_set_error("tscl_lstm_seq_bwd_tc: bad argument");
  if ((wxt_bf16 == nullptr) != (dx_bf16 == nullptr)) return tsc_set_error("tscl_lstm_seq_bwd_tc_dx: wxt_bf16 and dx_bf16 go together");
  if (!ZG && !(gates_bf16 && c_bf16 && dz_bf16)) return tsc_set_error("tscl_lstm_seq_bwd_tc: ZG may be null only with gates_bf16, c_bf16 and dz_bf16");
  if ((gates_bf16 == nullptr) != (c_bf16 == nullptr)) return tsc_set_error("tscl_lstm_seq_bwd_tc: gates_bf16 and c_bf16 go together");
  PCK(cudaSetDevice(tscl_device_of(h)));
  const DDimsTC& d = *tscl_dims_of(h);
  if (dx_bf16 && (d.dx % 32 != 0 || d.dx > 256)) return tsc_set_error("tscl_lstm_seq_bwd_tc_dx: dx must be a multiple of 32, <= 256");
  const size_t smem_max = BW_KC * 1024 + BW_KC * 2048 + 16 + (size_t)BW_KC * 256 * 16;
  const size_t smem = BW_KC * 1024 + BW_KC * 2048 + 16 + (dx_bf16 ? (size_t)BW_KC * d.dx * 16 : 0);
  static int attr_dev = -1;
  if (attr_dev != tscl_device_of(h)) {
    PCK(cudaFuncSetAttribute(lstm_bwd_tc_kernel<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max));
    PCK(cudaFuncSetAttribute(lstm_bwd_tc_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max));
    attr_dev = tscl_device_of(h);
  }
  int n_sm = 0;
  PCK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, tscl_device_of(h)));
  const int64_t n_items = ((Rc + TC_M - 1) / TC_M) * 2 * d.A;
  // 96 KB smem: two 512-thread CTAs per SM when registers allow; the fused-dX variant (up to 211 KB) is
  // one CTA per SM
  const int64_t max_ctas = dx_bf16 ? n_sm : 2 * n_sm;
  const int grid = (int)(n_items < max_ctas ? n_items : max_ctas);
  BwdTC a;
  a.acc = acc_tiles(h, stream);
  if (!a.acc) return tsc_set_error("accumulator tiles: cudaMalloc failed");
  a.Wt = (const __nv_bfloat16*)wt_bf16; a.ZG = ZG; a.C = C; a.dH = dH; a.c0 = c0; a.done = done; a.T = T; a.Rc = Rc;
  a.ld_state = ld_state; a.r0 = r0; a.Gb = (const __nv_bfloat16*)gates_bf16; a.Cb = (const __nv_bfloat16*)c_bf16; a.dZb = (__nv_bfloat16*)dz_bf16;
  a.Wxt = (const __nv_bfloat16*)wxt_bf16; a.dXb = (__nv_bfloat16*)dx_bf16;
  // default: the one-CTA-per-SM 512-thread variant; TSC_BPTT_THREADS=256 selects the two-CTA-per-SM 256-thread variant
  // for experiments (same arithmetic, same bits)
  static const int bw_threads = []() { const char* e = getenv("TSC_BPTT_THREADS"); return e && atoi(e) == 256 ? 256 : 512; }();
  // store path without fused dX: the register-recurrence kernel (TSC_BPTT_STAGED=0 selects lstm_bwd_tc_kernel, same bits)
  static const int bw_staged = []() { const char* e = getenv("TSC_BPTT_STAGED"); return e ? atoi(e) : 1; }();
  if (bw_staged && bw_threads == 512 && a.Gb && a.Cb && a.dZb && !a.ZG && !a.dXb) {
    // tensor maps [2A * T][Rc][cols] over this chunk's gates / c / dH / dZ; if they cannot be encoded,
    // lstm_bwd_tc_kernel<512> below gives the same bits
    CUtensorMap mG, mC, mD, mZ;
    const uint64_t planes = (uint64_t)2 * d.A * T;
    if (make_tmap_3d(&mG, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, gates_bf16, planes, Rc, TC_N, 64, 64) &&
        make_tmap_3d(&mC, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, c_bf16, planes, Rc, TC_H, 64, 64) &&
        make_tmap_3d(&mD, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, dH, planes, Rc, TC_H, 32, 64) &&
        make_tmap_3d(&mZ, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, dz_bf16, planes, Rc, TC_N, 64, 64)) {
      static int attr_r = -1;
      if (attr_r != tscl_device_of(h)) {
        PCK(cudaFuncSetAttribute(lstm_bwd_tc_regs_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, BR_SMEM));
        PCK(cudaFuncSetAttribute(lstm_bwd_tc_regs_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, BR_SMEM));
        attr_r = tscl_device_of(h);
      }
      const int grid_r = (int)(n_items < n_sm ? n_items : n_sm);
      a.prof = g_bptt_prof;
      if (a.prof) lstm_bwd_tc_regs_kernel<true><<<grid_r, 256, BR_SMEM, (cudaStream_t)stream>>>(d, a, mG, mC, mD, mZ);
      else lstm_bwd_tc_regs_kernel<false><<<grid_r, 256, BR_SMEM, (cudaStream_t)stream>>>(d, a, mG, mC, mD, mZ);
      PCK(cudaGetLastError());
      return 0;
    }
  }
  if (bw_threads == 512) lstm_bwd_tc_kernel<512><<<grid, 512, smem, (cudaStream_t)stream>>>(d, a);
  else lstm_bwd_tc_kernel<256><<<grid, 256, smem, (cudaStream_t)stream>>>(d, a);
  PCK(cudaGetLastError());
  return 0;
}

extern "C" int tscl_lstm_seq_bwd_tc_heads(tscl_handle* h, const void* wt_bf16, const float* params, const void* gates_bf16,
                                          const void* c_bf16, const void* h_bf16, const float* c0, const float* done,
                                          const int32_t* act, const float* Rs, const float* Adv, int32_t T, int64_t Rc,
                                          int32_t n_chunks, int64_t ld_state, int64_t r0, int64_t stride_t, float v_coef,
                                          float beta, float scale, void* dz_bf16, float* stats, float* grads, void* stream) {
  if (!h || !wt_bf16 || !params || !gates_bf16 || !c_bf16 || !h_bf16 || !c0 || !done || !act || !Rs || !Adv || !dz_bf16 ||
      !grads || T <= 0 || Rc <= 0 || n_chunks <= 0)
    return tsc_set_error("tscl_lstm_seq_bwd_tc_heads: bad argument");
  PCK(cudaSetDevice(tscl_device_of(h)));
  const DDimsTC& d = *tscl_dims_of(h);
  if (d.max_na > 8) return tsc_set_error("tscl_lstm_seq_bwd_tc_heads: more than 8 actions");
  if ((uint64_t)n_chunks * 2 * d.A * T > 0x7fffffffu) return tsc_set_error("tscl_lstm_seq_bwd_tc_heads: too many planes");
  CUtensorMap mG, mC, mH, mZ;
  const uint64_t planes = (uint64_t)n_chunks * 2 * d.A * T;
  if (!(make_tmap_3d(&mG, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, gates_bf16, planes, Rc, TC_N, 64, 64) &&
        make_tmap_3d(&mC, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, c_bf16, planes, Rc, TC_H, 64, 64) &&
        make_tmap_3d(&mH, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, h_bf16, planes, Rc, TC_H, 64, 64) &&
        make_tmap_3d(&mZ, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, dz_bf16, planes, Rc, TC_N, 64, 64)))
    return tsc_set_error("tscl_lstm_seq_bwd_tc_heads: cannot encode the tensor maps (cuTensorMapEncodeTiled)");
  static int attr_r = -1;
  if (attr_r != tscl_device_of(h)) {
    PCK(cudaFuncSetAttribute(lstm_bwd_tc_regs_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, BR_SMEM));
    PCK(cudaFuncSetAttribute(lstm_bwd_tc_regs_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, BR_SMEM));
    attr_r = tscl_device_of(h);
  }
  int n_sm = 0;
  PCK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, tscl_device_of(h)));
  const int64_t n_items = (int64_t)n_chunks * ((Rc + TC_M - 1) / TC_M) * 2 * d.A;
  const int grid = (int)(n_items < n_sm ? n_items : n_sm);
  BwdTC a = {};
  a.Wt = (const __nv_bfloat16*)wt_bf16; a.c0 = c0; a.done = done; a.T = T; a.Rc = Rc; a.ld_state = ld_state; a.r0 = r0;
  a.Gb = (const __nv_bfloat16*)gates_bf16; a.Cb = (const __nv_bfloat16*)c_bf16; a.dZb = (__nv_bfloat16*)dz_bf16;
  a.P = params; a.act = act; a.Rs = Rs; a.Adv = Adv; a.stride_t = stride_t; a.v_coef = v_coef; a.beta = beta;
  a.scale = scale; a.stats = stats; a.G = grads; a.n_chunks = n_chunks;
  a.prof = g_bptt_prof;
  if (a.prof) lstm_bwd_tc_regs_kernel<true, true><<<grid, 256, BR_SMEM, (cudaStream_t)stream>>>(d, a, mG, mC, mH, mZ);
  else lstm_bwd_tc_regs_kernel<false, true><<<grid, 256, BR_SMEM, (cudaStream_t)stream>>>(d, a, mG, mC, mH, mZ);
  PCK(cudaGetLastError());
  return 0;
}

// ===================================================================================================
// fc front-end weight gradients on the tensor cores (replaces fc_bwd_kernel of tsc_learn.cu).
//   dW[k][c] = sum_m In[m][k] * dXm[m][c],   dXm = dX * (X > 0),   m = (t, replica) rows of one chunk
// is a GEMM whose reduction index is the ROW index, so both operands are staged MN-major: the row-major global
// data lands as [col/8][128 rows][8 cols] bf16 without a transposition, and
//   D[dX column (four 64-column slabs)][64 input slots] += A^T B      (wgmma, A and B MN-major, K = 128 rows)
// Two warpgroups: warpgroup g owns slabs g and g + 2 and keeps their m64n64 fp32 fragments in registers (64 per thread;
// at 256 threads a thread may use 255) over all tiles of a unit.  A spare input slot holds 1.0: its D column is the bias
// gradient.  Persistent: CTA b owns the tile range [b NT / grid, (b + 1) NT / grid) of the (unit, tile) list and adds its
// fragments to G with atomics whenever the unit changes (<= 3 flushes per CTA).  Two smem stages: the first half of tile
// j + 1 is loaded into registers while the MMAs of tile j run.
#define FBT_ROWS 128
#define FBT_SBO 2064                       // chunk stride: 128 rows * 16 B + 16 B pad (conflict-free transposing stores)
#define FBT_A_BYTES (32 * FBT_SBO)
#define FBT_B_BYTES (8 * FBT_SBO)
#define FBT_STAGE (FBT_A_BYTES + FBT_B_BYTES)
#define FBT_THREADS 512                    // the weight-gradient kernels below
#define FBB_THREADS 256                    // fc_bwd_tc_kernel
struct FcBwdTC {
  const float* obs;            // rows as tscl_fc_embed
  const float* X;              // [2A][M][dx] fp32 activations, or
  const __nv_bfloat16* Xb;     // [2A][M][dx] bf16 activations (one chunk of the activation store)
  const float* dX;             // [2A][M][dx] fp32, or
  const __nv_bfloat16* dXb;    // [2A][M][dx] bf16
  float* G;
  int64_t M, rows_per_t, stride_t;
  int variant;                 // 1: LBO/SBO swapped (descriptor diagnosis)
};

__global__ void __launch_bounds__(FBB_THREADS, 1)
fc_bwd_tc_kernel(const DDimsTC d, const FcBwdTC a) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  // bf16 x bf16 -> f32, A and B MN-major, N = 64, M = 64 per slab
  const uint32_t lbo = a.variant ? FBT_SBO : 128, sbo = a.variant ? 128 : FBT_SBO;
  const int dx = d.dx, ng = dx >> 3, n_items = FBT_ROWS * ng;
  const uint32_t ng_magic = (1u << 20) / (uint32_t)ng + 1u;      // i / ng == (i * magic) >> 20 for i < 4096, ng <= 32
  const int64_t tpu = (a.M + FBT_ROWS - 1) / FBT_ROWS;
  const int64_t NT = tpu * 2 * d.A;
  const int64_t j0 = NT * blockIdx.x / gridDim.x, j1 = NT * (blockIdx.x + 1) / gridDim.x;
  float f0[32], f1[32];                        // slabs wg and wg + 2
  bool first = true;
  int cur_u = -1, nw = 0, nt = 0, nf = 0, ooff = 0;
  int src[8];                                  // observation index of each of this thread's 8 input slots (-1 none, -2 one)
  const int bc = tid & 7;                      // this thread's B chunk (8 input slots)

  // a fragment into G: dX column c = 64 sl + 16 (warp & 3) + lane / 4 (+ 8), input slot 8 i + 2 (lane & 3) (+ 1).
  // Columns past dx come from A chunks that are never staged: they are dropped here.
  auto flush_slab = [&](const float (&f)[32], int sl, int u) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int c = sl * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * hh;
      if (c < dx) {
        int64_t wo, bo; int ld, cc, s0, n;
        if (c < d.fw) { wo = d.off_fcw_w[u]; bo = d.off_fcw_b[u]; ld = d.fw; cc = c; s0 = 0; n = nw; }
        else if (c < d.fw + d.ff) { wo = d.off_fcf_w[u]; bo = d.off_fcf_b[u]; ld = d.ff; cc = c - d.fw; s0 = d.kw; n = nf; }
        else { wo = d.off_fct_w[u]; bo = d.off_fct_b[u]; ld = d.ft; cc = c - d.fw - d.ff; s0 = d.kw + TC_KF; n = nt; }
#pragma unroll
        for (int e = 0; e < 16; ++e) {
          const int slot = 8 * (e >> 1) + 2 * (lane & 3) + (e & 1), kin = slot - s0;
          const float v = f[4 * (e >> 1) + 2 * hh + (e & 1)];
          if (kin >= 0 && kin < n) atomicAdd(&a.G[wo + (int64_t)kin * ld + cc], v);
          if (slot == d.ones_slot) atomicAdd(&a.G[bo + cc], v);
        }
      }
    }
  };
  auto flush = [&](int u) {
    wg_wait<0>();
    wg_frag_fence(f0); wg_frag_fence(f1);
    flush_slab(f0, wg, u);
    flush_slab(f1, wg + 2, u);
  };

  for (int64_t j = j0; j < j1; ++j) {
    const int u = (int)(j / tpu);
    const int64_t m0 = (j - (int64_t)u * tpu) * FBT_ROWS;
    const int s = (int)((j - j0) & 1);
    if (u != cur_u) {
      if (cur_u >= 0) flush(cur_u);
      cur_u = u; first = true;
      const int ag = u >> 1;
      nw = d.n_wave[ag]; nt = d.n_wait[ag]; nf = d.ff > 0 ? d.n_fp[ag] : 0; ooff = d.obs_off[ag];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int slot = bc * 8 + e;
        int sidx = -1;
        if (slot < d.kw) { if (slot < nw) sidx = slot; }
        else if (slot < d.kw + TC_KF) { if (slot - d.kw < nf) sidx = nw + nt + (slot - d.kw); }
        else { if (slot - d.kw - TC_KF < nt) sidx = nw + (slot - d.kw - TC_KF); }
        if (slot == d.ones_slot) sidx = -2;
        src[e] = sidx;
      }
    }
    unsigned char* sA = tc_smem + (size_t)s * FBT_STAGE;
    unsigned char* sB = sA + FBT_A_BYTES;
    const int rows_valid = (a.M - m0) < FBT_ROWS ? (int)(a.M - m0) : FBT_ROWS;
    const int items_valid = rows_valid * ng;
    const int64_t base = ((int64_t)u * a.M + m0) * dx;
    if (j + 1 < j1) {      // pull the next tile towards L2 while this one is converted and multiplied
      const int un = (int)((j + 1) / tpu);
      const int64_t m0n = (j + 1 - (int64_t)un * tpu) * FBT_ROWS;
      const int rvn = (a.M - m0n) < FBT_ROWS ? (int)(a.M - m0n) : FBT_ROWS;
      const int64_t basen = ((int64_t)un * a.M + m0n) * dx;
      const int64_t nbytes = (int64_t)rvn * dx * 4;
      if (a.dXb) {
        const char* pd = reinterpret_cast<const char*>(a.dXb + basen);
        for (int64_t o = (int64_t)tid * 128; o < nbytes / 2; o += FBB_THREADS * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(pd + o));
      } else {
        const char* pd = reinterpret_cast<const char*>(a.dX + basen);
        for (int64_t o = (int64_t)tid * 128; o < nbytes; o += FBB_THREADS * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(pd + o));
      }
      if (a.Xb) {
        const char* px = reinterpret_cast<const char*>(a.Xb + basen);
        for (int64_t o = (int64_t)tid * 128; o < nbytes / 2; o += FBB_THREADS * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(px + o));
      }
      if (tid < rvn) {
        const int64_t m = m0n + tid;
        const float* op = a.obs + (m / a.rows_per_t) * a.stride_t + (m % a.rows_per_t) * d.n_obs + d.obs_off[un >> 1];
        asm volatile("prefetch.global.L2 [%0];" ::"l"(op));
        asm volatile("prefetch.global.L2 [%0];" ::"l"(op + 32));
      }
    }
    // ---- B loads first (observation slice of this thread's 8 input slots, 2 rows): their latency overlaps the A staging ----
    uint4 ov[(FBT_ROWS * 8) / FBB_THREADS];      // 8 bf16 each
    {
      const int64_t tq = m0 / a.rows_per_t, rem0 = m0 - tq * a.rows_per_t;      // one division per tile
#pragma unroll
      for (int r = 0; r < (FBT_ROWS * 8) / FBB_THREADS; ++r) {
        const int row = (r * FBB_THREADS + tid) >> 3;
        ov[r] = make_uint4(0, 0, 0, 0);
        if (row < rows_valid) {
          int64_t tt = tq, rem = rem0 + row;
          while (rem >= a.rows_per_t) { rem -= a.rows_per_t; ++tt; }
          const float* op = a.obs + tt * a.stride_t + rem * d.n_obs + ooff;
          __align__(16) __nv_bfloat16 o[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) o[e] = __float2bfloat16_rn(src[e] >= 0 ? __ldg(op + src[e]) : (src[e] == -2 ? 1.0f : 0.f));
          ov[r] = *reinterpret_cast<const uint4*>(o);
        }
      }
    }
    // ---- A, bf16 in / bf16 out: the loads of half a tile in flight at once, relu mask as packed 16-bit integer ops.
    //      The first half is loaded before the barrier that frees this stage ----
    const bool all_bf16 = a.dXb && a.Xb;
    uint4 gb[8], xm[8];
    auto load_half = [&](int h) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int i = (8 * h + k) * FBB_THREADS + tid;
        gb[k] = make_uint4(0, 0, 0, 0); xm[k] = make_uint4(0, 0, 0, 0);
        if (i < items_valid) {
          gb[k] = __ldg(reinterpret_cast<const uint4*>(a.dXb + base) + i);
          xm[k] = __ldg(reinterpret_cast<const uint4*>(a.Xb + base) + i);
        }
      }
    };
    auto store_half = [&](int h) {
      auto keep2 = [](uint32_t x) -> uint32_t {      // 0xFFFF per 16-bit half where the bf16 value is > 0
        const uint32_t nz = ((x & 0x7FFF7FFFu) + 0x7FFF7FFFu) & ~x & 0x80008000u;
        return (nz >> 15) * 0xFFFFu;
      };
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int i = (8 * h + k) * FBB_THREADS + tid;
        if (i < n_items) {
          const uint4 o = make_uint4(gb[k].x & keep2(xm[k].x), gb[k].y & keep2(xm[k].y), gb[k].z & keep2(xm[k].z),
                                     gb[k].w & keep2(xm[k].w));
          const int row = (int)(((uint32_t)i * ng_magic) >> 20), cg = i - row * ng;
          *reinterpret_cast<uint4*>(sA + (size_t)cg * FBT_SBO + row * 16) = o;
        }
      }
    };
    if (all_bf16) load_half(0);
    __syncthreads();      // every warpgroup has waited for its MMAs of tile j - 1: stage s is free
    if (all_bf16) {
      store_half(0);
      if (n_items > 8 * FBB_THREADS) { load_half(1); store_half(1); }
    } else {
      // ---- A: masked dX, 8 columns (one 16 B chunk row) per item; items are contiguous in global memory ----
      for (int ib = 0; ib < n_items; ib += 2 * FBB_THREADS) {
        float4 g0[2], g1[2];
        uint4 xb[2];
        float4 x0[2], x1[2];
  #pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int i = ib + r * FBB_THREADS + tid;
          g0[r] = g1[r] = make_float4(0.f, 0.f, 0.f, 0.f);
          xb[r] = make_uint4(0, 0, 0, 0);
          x0[r] = x1[r] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (i < items_valid) {
            if (a.dXb) {
              const uint4 gb = __ldg(reinterpret_cast<const uint4*>(a.dXb + base) + i);
              g0[r] = make_float4(__uint_as_float(gb.x << 16), __uint_as_float(gb.x & 0xffff0000u), __uint_as_float(gb.y << 16),
                                  __uint_as_float(gb.y & 0xffff0000u));
              g1[r] = make_float4(__uint_as_float(gb.z << 16), __uint_as_float(gb.z & 0xffff0000u), __uint_as_float(gb.w << 16),
                                  __uint_as_float(gb.w & 0xffff0000u));
            } else {
              const float4* gp = reinterpret_cast<const float4*>(a.dX + base) + 2 * (int64_t)i;
              g0[r] = __ldg(gp); g1[r] = __ldg(gp + 1);
            }
            if (a.Xb) xb[r] = __ldg(reinterpret_cast<const uint4*>(a.Xb + base) + i);
            else {
              const float4* xp = reinterpret_cast<const float4*>(a.X + base) + 2 * (int64_t)i;
              x0[r] = __ldg(xp); x1[r] = __ldg(xp + 1);
            }
          }
        }
  #pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int i = ib + r * FBB_THREADS + tid;
          if (i < n_items) {
            const float gv[8] = {g0[r].x, g0[r].y, g0[r].z, g0[r].w, g1[r].x, g1[r].y, g1[r].z, g1[r].w};
            bool pos[8];
            if (a.Xb) {
              const uint32_t w[4] = {xb[r].x, xb[r].y, xb[r].z, xb[r].w};
  #pragma unroll
              for (int e = 0; e < 4; ++e) {
                const uint32_t lo = w[e] & 0xffffu, hi = w[e] >> 16;
                pos[2 * e] = (lo & 0x8000u) == 0 && (lo & 0x7fffu) != 0;
                pos[2 * e + 1] = (hi & 0x8000u) == 0 && (hi & 0x7fffu) != 0;
              }
            } else {
              const float xv[8] = {x0[r].x, x0[r].y, x0[r].z, x0[r].w, x1[r].x, x1[r].y, x1[r].z, x1[r].w};
  #pragma unroll
              for (int e = 0; e < 8; ++e) pos[e] = xv[e] > 0.f;
            }
            __align__(16) __nv_bfloat16 o[8];
  #pragma unroll
            for (int e = 0; e < 8; ++e) o[e] = __float2bfloat16_rn(pos[e] ? gv[e] : 0.f);
            const int row = i / ng, cg = i - row * ng;
            *reinterpret_cast<uint4*>(sA + (size_t)cg * FBT_SBO + row * 16) = *reinterpret_cast<const uint4*>(o);
          }
        }
      }
    }
    // ---- B: the unit's observation slice scattered into the 64 input slots ----
#pragma unroll
    for (int r = 0; r < (FBT_ROWS * 8) / FBB_THREADS; ++r) {
      const int row = (r * FBB_THREADS + tid) >> 3;
      *reinterpret_cast<uint4*>(sB + (size_t)bc * FBT_SBO + row * 16) = ov[r];
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    // both slabs of each warpgroup are multiplied whatever dx is: rows past dx are never flushed
    const uint32_t aA = smem_u32(sA), aB = smem_u32(sB);
    wg_fence();
    wg_mma_regs<64, 1, 1>(f0, FBT_ROWS / 16, !first, [&](int ks, uint64_t& da, uint64_t& db) {
      da = make_desc(aA + wg * 8 * FBT_SBO + ks * 256, lbo, sbo);
      db = make_desc(aB + ks * 256, lbo, sbo);
    });
    wg_mma_regs<64, 1, 1>(f1, FBT_ROWS / 16, !first, [&](int ks, uint64_t& da, uint64_t& db) {
      da = make_desc(aA + (wg + 2) * 8 * FBT_SBO + ks * 256, lbo, sbo);
      db = make_desc(aB + ks * 256, lbo, sbo);
    });
    wg_commit();
    // wait_group 0, not 1: with a group still in flight across the staging code below (divergent per thread), ptxas
    // serialises the wgmma of this kernel.  The MMAs of a tile are short next to its staging.
    wg_wait<0>();
    first = false;
  }
  if (cur_u >= 0) flush(cur_u);
}

extern "C" int tscl_fc_bwd_tc(tscl_handle* h, const float* obs, const float* X, const void* x_bf16, const float* dX,
                              const void* dx_bf16, int64_t M, int64_t rows_per_t, int64_t stride_t, float* grads,
                              int32_t variant, void* stream) {
  if (!h || !obs || (!X && !x_bf16) || (!dX && !dx_bf16) || !grads || M <= 0) return tsc_set_error("tscl_fc_bwd_tc: bad argument");
  PCK(cudaSetDevice(tscl_device_of(h)));
  const DDimsTC& d = *tscl_dims_of(h);
  if ((d.dx % 8) != 0 || d.dx > 256) return tsc_set_error("tscl_fc_bwd_tc: dx must be a multiple of 8, <= 256");
  if (d.kw == 0 || d.ones_slot < 0) return tsc_set_error("tscl_fc_bwd_tc: no free input slot for the bias column (use tscl_fc_bwd)");
  const size_t smem = 2 * FBT_STAGE;
  static int attr_dev = -1;
  if (attr_dev != tscl_device_of(h)) {
    PCK(cudaFuncSetAttribute(fc_bwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_dev = tscl_device_of(h);
  }
  int n_sm = 0;
  PCK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, tscl_device_of(h)));
  const int64_t NT = ((M + FBT_ROWS - 1) / FBT_ROWS) * 2 * d.A;
  const int grid = (int)(NT < n_sm ? NT : n_sm);
  FcBwdTC a;
  a.obs = obs; a.X = X; a.Xb = (const __nv_bfloat16*)x_bf16; a.dX = dX; a.dXb = (const __nv_bfloat16*)dx_bf16; a.G = grads; a.M = M;
  a.rows_per_t = rows_per_t;
  a.stride_t = stride_t; a.variant = variant;
  fc_bwd_tc_kernel<<<grid, FBB_THREADS, smem, (cudaStream_t)stream>>>(d, a);
  PCK(cudaGetLastError());
  return 0;
}

// ===================================================================================================
// LSTM weight gradients on the tensor cores (replaces two cuBLAS GEMMs, a column reduction and the fp32 unpacking of
// X / Hp):   dWx += X^T dZ,   dWh += Hp^T dZ,   dbl += 1^T dZ      over the rows m = (t, replica) of one chunk.
// Same MN-major staging as fc_bwd_tc_kernel.  A = [X | Hp | 1] (dx + 64 + 1 columns = up to three M = 128 blocks),
// B = one 128-column half of dZ; D[block][128 gate columns] accumulates in the accumulator tile (384 columns).  A CTA owns a
// contiguous tile range of the (unit, half, tile) list and flushes with atomics when (unit, half) changes.
// Hp is rebuilt from the bf16 activation store: Hp[t] = (1 - done[t]) * (t > 0 ? H[t-1] : h0).
#define WG_A_CHUNKS 40
#define WG_Z_CHUNKS 16
#define WG_STAGE ((WG_A_CHUNKS + WG_Z_CHUNKS) * FBT_SBO)
struct WGradTC {
  float* acc;                // accumulator tiles, one [128][ACC_COLS] fp32 tile per CTA (acc_tiles)
  const float* dZ;             // [2A][M][256] fp32, or
  const __nv_bfloat16* dZb;    // [2A][M][256] bf16
  const float* X;              // [2A][M][dx] fp32, or
  const __nv_bfloat16* Xb;     // [2A][M][dx] bf16
  const float* Hp;             // [2A][M][64] fp32, or
  const __nv_bfloat16* Hb;     // [2A][T][rc][64] bf16 with h0 / done / T / rc / ld_state / r0
  const float* h0;
  const float* done;
  float* G;
  int64_t M, rc, ld_state, r0;
  int T, variant;
};

__global__ void __launch_bounds__(FBT_THREADS, 1)
wgrad_tc_kernel(const DDimsTC d, const WGradTC a) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint64_t* sBar = reinterpret_cast<uint64_t*>(tc_smem + 2 * WG_STAGE);
  const uint32_t bar0 = smem_u32(sBar);
  if (tid == 0) {
    mbar_init(bar0, 1); mbar_init(bar0 + 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // never-written A chunks are read by the last M block: keep them finite
  for (int i = tid; i < 2 * WG_STAGE / 16; i += FBT_THREADS) reinterpret_cast<uint4*>(tc_smem)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  float* const acc = a.acc + (size_t)blockIdx.x * TC_M * ACC_COLS;
  const uint32_t lbo = a.variant ? FBT_SBO : 128, sbo = a.variant ? 128 : FBT_SBO;
  const int dx = d.dx, ng = dx >> 3, n_xitems = FBT_ROWS * ng;
  const int nb = (dx + TC_H + 1 + 127) >> 7;        // M blocks
  const int64_t tpu = (a.M + FBT_ROWS - 1) / FBT_ROWS;
  const int64_t NT = tpu * 4 * d.A;
  const int64_t j0 = NT * blockIdx.x / gridDim.x, j1 = NT * (blockIdx.x + 1) / gridDim.x;
  uint32_t ph0 = 0, ph1 = 0;
  bool pend0 = false, pend1 = false, first = true;
  int cur_pu = -1;

  auto flush = [&](int pu) {
    if (pend0) { mbar_wait(bar0, ph0); ph0 ^= 1; pend0 = false; }
    if (pend1) { mbar_wait(bar0 + 8, ph1); ph1 ^= 1; pend1 = false; }
    const int u = pu >> 1, nh = pu & 1;
    const int q = warp & 3, cq = warp >> 2;
    const int g0 = nh * 128 + cq * 32;
    for (int b = 0; b < nb; ++b) {
      const int ci = b * 128 + q * 32 + lane;
      float v[32];
      const uint32_t tb = ((uint32_t)(q * 32) << 16) + (uint32_t)(b * 128 + cq * 32);
      acc_ld16(acc, tb, v); acc_ld16(acc, tb + 16, v + 16);
      float* dst = nullptr;
      if (ci < dx) dst = a.G + d.off_wx + ((int64_t)u * dx + ci) * TC_N + g0;
      else if (ci < dx + TC_H) dst = a.G + d.off_wh + ((int64_t)u * TC_H + (ci - dx)) * TC_N + g0;
      else if (ci == dx + TC_H) dst = a.G + d.off_bl + (int64_t)u * TC_N + g0;
      if (dst) {
#pragma unroll
        for (int e = 0; e < 32; ++e) atomicAdd(dst + e, v[e]);
      }
    }
    __syncthreads();
  };

  for (int64_t j = j0; j < j1; ++j) {
    const int pu = (int)(j / tpu), u = pu >> 1, nh = pu & 1;
    const int64_t m0 = (j - (int64_t)pu * tpu) * FBT_ROWS;
    const int s = (int)((j - j0) & 1);
    if (pu != cur_pu) {
      if (cur_pu >= 0) flush(cur_pu);
      cur_pu = pu; first = true;
    }
    if (s == 0) { if (pend0) { mbar_wait(bar0, ph0); ph0 ^= 1; pend0 = false; } }
    else { if (pend1) { mbar_wait(bar0 + 8, ph1); ph1 ^= 1; pend1 = false; } }
    unsigned char* sA = tc_smem + (size_t)s * WG_STAGE;
    unsigned char* sZ = sA + (size_t)WG_A_CHUNKS * FBT_SBO;
    const int rows_valid = (a.M - m0) < FBT_ROWS ? (int)(a.M - m0) : FBT_ROWS;
    const int64_t rowbase = (int64_t)u * a.M + m0;
    if (j + 1 < j1) {      // pull the next tile towards L2 while this one is converted and multiplied
      const int pun = (int)((j + 1) / tpu), un = pun >> 1, nhn = pun & 1;
      const int64_t m0n = (j + 1 - (int64_t)pun * tpu) * FBT_ROWS;
      const int rvn = (a.M - m0n) < FBT_ROWS ? (int)(a.M - m0n) : FBT_ROWS;
      const int64_t rbn = (int64_t)un * a.M + m0n;
      if ((tid >> 2) < rvn) {
        if (a.dZb) { if ((tid & 3) < 2) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.dZb + (rbn + (tid >> 2)) * TC_N + nhn * 128 + (tid & 3) * 64)); }
        else asm volatile("prefetch.global.L2 [%0];" ::"l"(a.dZ + (rbn + (tid >> 2)) * TC_N + nhn * 128 + (tid & 3) * 32));
      }
      if (a.Xb) {
        const char* px = reinterpret_cast<const char*>(a.Xb + rbn * dx);
        const int64_t nbytes = (int64_t)rvn * dx * 2;
        for (int64_t o = (int64_t)tid * 128; o < nbytes; o += FBT_THREADS * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(px + o));
      }
      if (a.Hb && tid < rvn && m0n + tid >= a.rc) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.Hb + (rbn + tid - a.rc) * TC_H));
    }
    // ---- B: this half of dZ (fp32 -> bf16), 8 gate columns per item ----
    {
      float4 z0[4], z1[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i = r * FBT_THREADS + tid, row = i >> 4, g = i & 15;
        z0[r] = z1[r] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < rows_valid) {
          if (a.dZb) {       // already bf16: carried bit-for-bit in z0
            const uint4 zb = __ldg(reinterpret_cast<const uint4*>(a.dZb + (rowbase + row) * TC_N + nh * 128 + g * 8));
            z0[r] = make_float4(__uint_as_float(zb.x), __uint_as_float(zb.y), __uint_as_float(zb.z), __uint_as_float(zb.w));
          } else {
            const float4* zp = reinterpret_cast<const float4*>(a.dZ + (rowbase + row) * TC_N + nh * 128 + g * 8);
            z0[r] = __ldg(zp); z1[r] = __ldg(zp + 1);
          }
        }
      }
      // ---- A: X, 8 columns per item; items are contiguous in global memory ----
      for (int ib = 0; ib < n_xitems; ib += 4 * FBT_THREADS) {
        uint4 xb[4];
        float4 x0[4], x1[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int i = ib + r * FBT_THREADS + tid;
          xb[r] = make_uint4(0, 0, 0, 0);
          x0[r] = x1[r] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (i < rows_valid * ng) {
            if (a.Xb) xb[r] = __ldg(reinterpret_cast<const uint4*>(a.Xb + rowbase * dx) + i);
            else {
              const float4* xp = reinterpret_cast<const float4*>(a.X + rowbase * dx) + 2 * (int64_t)i;
              x0[r] = __ldg(xp); x1[r] = __ldg(xp + 1);
            }
          }
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int i = ib + r * FBT_THREADS + tid;
          if (i < n_xitems) {
            uint4 o = xb[r];
            if (!a.Xb) {
              __align__(16) __nv_bfloat16 t[8] = {__float2bfloat16_rn(x0[r].x), __float2bfloat16_rn(x0[r].y),
                                                  __float2bfloat16_rn(x0[r].z), __float2bfloat16_rn(x0[r].w),
                                                  __float2bfloat16_rn(x1[r].x), __float2bfloat16_rn(x1[r].y),
                                                  __float2bfloat16_rn(x1[r].z), __float2bfloat16_rn(x1[r].w)};
              o = *reinterpret_cast<const uint4*>(t);
            }
            const int row = i / ng, cg = i - row * ng;
            *reinterpret_cast<uint4*>(sA + (size_t)cg * FBT_SBO + row * 16) = o;
          }
        }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i = r * FBT_THREADS + tid, row = i >> 4, g = i & 15;
        __align__(16) __nv_bfloat16 t[8] = {__float2bfloat16_rn(z0[r].x), __float2bfloat16_rn(z0[r].y),
                                            __float2bfloat16_rn(z0[r].z), __float2bfloat16_rn(z0[r].w),
                                            __float2bfloat16_rn(z1[r].x), __float2bfloat16_rn(z1[r].y),
                                            __float2bfloat16_rn(z1[r].z), __float2bfloat16_rn(z1[r].w)};
        uint4 zo = *reinterpret_cast<const uint4*>(t);
        if (a.dZb) zo = make_uint4(__float_as_uint(z0[r].x), __float_as_uint(z0[r].y), __float_as_uint(z0[r].z), __float_as_uint(z0[r].w));
        *reinterpret_cast<uint4*>(sZ + (size_t)g * FBT_SBO + row * 16) = zo;
      }
    }
    // ---- A: Hp (8 hidden units per item) and the ones column ----
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int i = r * FBT_THREADS + tid, row = i >> 3, c = i & 7;
      uint4 o = make_uint4(0, 0, 0, 0);
      if (row < rows_valid) {
        if (a.Hb) {
          const int64_t m = m0 + row;
          const int t = (int)(m / a.rc);
          if (a.done[t] == 0.f) {
            if (t > 0) o = __ldg(reinterpret_cast<const uint4*>(a.Hb + (rowbase + row - a.rc) * TC_H + c * 8));
            else {
              const float4* hp = reinterpret_cast<const float4*>(a.h0 + ((int64_t)u * a.ld_state + a.r0 + m) * TC_H + c * 8);
              const float4 p = __ldg(hp), qv = __ldg(hp + 1);
              __align__(16) __nv_bfloat16 tt[8] = {__float2bfloat16_rn(p.x), __float2bfloat16_rn(p.y), __float2bfloat16_rn(p.z),
                                                   __float2bfloat16_rn(p.w), __float2bfloat16_rn(qv.x), __float2bfloat16_rn(qv.y),
                                                   __float2bfloat16_rn(qv.z), __float2bfloat16_rn(qv.w)};
              o = *reinterpret_cast<const uint4*>(tt);
            }
          }
        } else {
          const float4* hp = reinterpret_cast<const float4*>(a.Hp + (rowbase + row) * TC_H + c * 8);
          const float4 p = __ldg(hp), qv = __ldg(hp + 1);
          __align__(16) __nv_bfloat16 tt[8] = {__float2bfloat16_rn(p.x), __float2bfloat16_rn(p.y), __float2bfloat16_rn(p.z),
                                               __float2bfloat16_rn(p.w), __float2bfloat16_rn(qv.x), __float2bfloat16_rn(qv.y),
                                               __float2bfloat16_rn(qv.z), __float2bfloat16_rn(qv.w)};
          o = *reinterpret_cast<const uint4*>(tt);
        }
      }
      *reinterpret_cast<uint4*>(sA + (size_t)(ng + c) * FBT_SBO + row * 16) = o;
    }
    if (tid < FBT_ROWS)
      *reinterpret_cast<uint4*>(sA + (size_t)(ng + 8) * FBT_SBO + tid * 16) = make_uint4(tid < rows_valid ? 0x3f80u : 0u, 0, 0, 0);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (warp < 8) {
      const uint32_t aA = smem_u32(sA), aZ = smem_u32(sZ);
      for (int b = 0; b < nb; ++b)
        wg_mma<1, 1>(acc, b * 128, 128, FBT_ROWS / 16, !first, [&](int ks, uint64_t& da, uint64_t& db) {
          da = make_desc(aA + b * 16 * FBT_SBO + ks * 256, lbo, sbo);
          db = make_desc(aZ + ks * 256, lbo, sbo);
        });
      wg_mma_done(bar0 + 8 * s);
    }
    if (s == 0) pend0 = true; else pend1 = true;
    first = false;
  }
  if (cur_pu >= 0) flush(cur_pu);
}

// All-bf16 variant (the training loop's): 64-row tiles, two smem stages + one register stage, accumulators in registers.
// The A columns [X | Hp | 1] (dx + 65 <= 320) form nsl 64-column slabs; CTA 5p + k (for nsl = 5) owns slab k of the
// (unit, tile) range of group p, and its warpgroup q the gate columns 64 q .. 64 q + 63, so every warpgroup holds one
// m64n64 fragment (32 registers per thread) for as long as the CTA stays on one unit.  The CTAs of a group walk the same
// range, so the later readers of a dZ tile find it in L2.
#define WGA_ROWS 64
#define WGA_SBO (WGA_ROWS * 16 + 16)
#define WGA_A_CHUNKS 8
#define WGA_STAGE ((WGA_A_CHUNKS + 32) * WGA_SBO)
#define WGA_STAGES 2
#define WGA_MAXT 256
__host__ __device__ inline int wga_slabs(int dx) { return (dx + TC_H + 1 + 63) >> 6; }
__global__ void __launch_bounds__(FBT_THREADS, 1)
wgrad_tc_async_kernel(const DDimsTC d, const WGradTC a) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wq = warp >> 2;
  float* sDone = reinterpret_cast<float*>(tc_smem + WGA_STAGES * WGA_STAGE);
  for (int i = tid; i < a.T; i += FBT_THREADS) sDone[i] = a.done[i];
  __syncthreads();
  const uint32_t lbo = a.variant ? WGA_SBO : 128, sbo = a.variant ? 128 : WGA_SBO;
  const int dx = d.dx, ng = dx >> 3;
  const int nsl = wga_slabs(dx);
  const int64_t tpu = (a.M + WGA_ROWS - 1) / WGA_ROWS;
  const int64_t NT = tpu * 2 * d.A;
  const int ngrp = gridDim.x / nsl, pb = blockIdx.x / nsl, sl = blockIdx.x - pb * nsl;
  const int64_t j0 = NT * pb / ngrp, j1 = NT * (pb + 1) / ngrp;
  // this thread's A piece: 8 columns (chunk cg of [X | Hp | 1 | 0]) of one row
  const int arow = tid >> 3, cg = sl * 8 + (tid & 7);
  float f[32];
  bool first = true;
  int cur_u = -1;
  // the fragment into G: A column sl * 64 + 16 (warp & 3) + lane / 4 (+ 8), gate column 64 wq + 8 i + 2 (lane & 3) (+ 1)
  auto flush = [&](int u) {
    wg_wait<0>();
    wg_frag_fence(f);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int ci = sl * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * hh;
      float* dst = nullptr;
      if (ci < dx) dst = a.G + d.off_wx + ((int64_t)u * dx + ci) * TC_N;
      else if (ci < dx + TC_H) dst = a.G + d.off_wh + ((int64_t)u * TC_H + (ci - dx)) * TC_N;
      else if (ci == dx + TC_H) dst = a.G + d.off_bl + (int64_t)u * TC_N;
      if (dst) {
        dst += wq * 64 + 2 * (lane & 3);
#pragma unroll
        for (int i = 0; i < 8; ++i) { atomicAdd(dst + 8 * i, f[4 * i + 2 * hh]); atomicAdd(dst + 8 * i + 1, f[4 * i + 2 * hh + 1]); }
      }
    }
  };

  // running position of the NEXT tile to load: unit, first row, and (t, row within t) of that row
  int iu = (int)(j0 / tpu);
  int64_t im0 = (j0 - (int64_t)iu * tpu) * WGA_ROWS;
  int64_t it_t = im0 / a.rc, it_rem = im0 - it_t * a.rc;
  // Register-staged pipeline: the 5 pieces (16 B each: 4 of dZ, 1 of A) of tile j + 2 are loaded into registers while
  // tile j is multiplied and tile j + 1 sits in the other smem stage; they are stored one iteration later, when their
  // latency has passed.  (cp.async is slower here: LDGSTS keeps its address registers reserved until the copy
  // completes, and the allocator's reuse of them stalls the warp for a memory latency.)
  uint4 pv[5];
  auto load_tile = [&]() {
    const int u = iu;
    const int64_t m0 = im0;
    const int rows_valid = (a.M - m0) < WGA_ROWS ? (int)(a.M - m0) : WGA_ROWS;
    const int64_t rowbase = (int64_t)u * a.M + m0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i = k * FBT_THREADS + tid, row = i >> 5, g = i & 31;
      pv[k] = make_uint4(0, 0, 0, 0);
      if (row < rows_valid) pv[k] = __ldg(reinterpret_cast<const uint4*>(a.dZb + (rowbase + row) * TC_N + g * 8));
    }
    pv[4] = make_uint4(0, 0, 0, 0);
    if (arow < rows_valid) {
      if (cg < ng) pv[4] = __ldg(reinterpret_cast<const uint4*>(a.Xb + (rowbase + arow) * dx) + cg);
      else if (cg < ng + 8) {
        const int hc = cg - ng;
        int64_t t = it_t, rem = it_rem + arow;
        while (rem >= a.rc) { rem -= a.rc; ++t; }
        if (sDone[t] == 0.f) {
          if (t > 0) pv[4] = __ldg(reinterpret_cast<const uint4*>(a.Hb + (rowbase + arow - a.rc) * TC_H + hc * 8));
          else {       // first step of the rollout: Hp = h0 (fp32 state)
            const float4* hp = reinterpret_cast<const float4*>(a.h0 + ((int64_t)u * a.ld_state + a.r0 + rem) * TC_H + hc * 8);
            const float4 p = __ldg(hp), qv = __ldg(hp + 1);
            __align__(16) __nv_bfloat16 tt[8] = {__float2bfloat16_rn(p.x), __float2bfloat16_rn(p.y), __float2bfloat16_rn(p.z),
                                                 __float2bfloat16_rn(p.w), __float2bfloat16_rn(qv.x), __float2bfloat16_rn(qv.y),
                                                 __float2bfloat16_rn(qv.z), __float2bfloat16_rn(qv.w)};
            pv[4] = *reinterpret_cast<const uint4*>(tt);
          }
        }
      } else if (cg == ng + 8) pv[4].x = 0x3f80u;      // the ones column (bias gradient)
    }
    // advance the running position
    im0 += WGA_ROWS; it_rem += WGA_ROWS;
    while (it_rem >= a.rc) { it_rem -= a.rc; ++it_t; }
    if (im0 >= a.M) { ++iu; im0 = 0; it_t = 0; it_rem = 0; }
  };
  auto store_tile = [&](int s) {
    unsigned char* sA = tc_smem + (size_t)s * WGA_STAGE;
    unsigned char* sZ = sA + (size_t)WGA_A_CHUNKS * WGA_SBO;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i = k * FBT_THREADS + tid;
      *reinterpret_cast<uint4*>(sZ + (size_t)(i & 31) * WGA_SBO + (i >> 5) * 16) = pv[k];
    }
    *reinterpret_cast<uint4*>(sA + (size_t)(tid & 7) * WGA_SBO + arow * 16) = pv[4];
  };

  if (j0 < j1) { load_tile(); store_tile(0); }
  if (j0 + 1 < j1) load_tile();
  for (int64_t j = j0; j < j1; ++j) {
    const int u = (int)(j / tpu);
    const int s = (int)((j - j0) & 1);
    if (u != cur_u) {
      if (cur_u >= 0) flush(cur_u);
      cur_u = u; first = true;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const uint32_t aA = smem_u32(tc_smem + (size_t)s * WGA_STAGE), aZ = aA + WGA_A_CHUNKS * WGA_SBO;
    wg_fence();
    wg_mma_regs<64, 1, 1>(f, WGA_ROWS / 16, !first, [&](int ks, uint64_t& da, uint64_t& db) {
      da = make_desc(aA + ks * 256, lbo, sbo);
      db = make_desc(aZ + wq * 8 * WGA_SBO + ks * 256, lbo, sbo);
    });
    wg_commit();
    first = false;
    if (j + 1 < j1) {
      wg_wait<1>();                 // this warpgroup's MMAs of tile j - 1 are done ...
      __syncthreads();              // ... and every warpgroup's: the other stage is free
      store_tile(s ^ 1);            // tile j + 1, loaded one iteration ago
      if (j + 2 < j1) load_tile();
    }
  }
  if (cur_u >= 0) flush(cur_u);
}

extern "C" int tscl_wgrad_tc(tscl_handle* h, const float* dZ, const void* dz_bf16, const float* X, const void* x_bf16,
                             const float* Hp, const void* h_bf16, const float* h0, const float* done, int32_t T, int64_t rc,
                             int64_t ld_state, int64_t r0, float* grads, int32_t variant, void* stream) {
  if (!h || (!dZ && !dz_bf16) || (!X && !x_bf16) || (!Hp && !h_bf16) || !grads || T <= 0 || rc <= 0)
    return tsc_set_error("tscl_wgrad_tc: bad argument");
  if (h_bf16 && (!h0 || !done)) return tsc_set_error("tscl_wgrad_tc: h_bf16 needs h0 and done");
  PCK(cudaSetDevice(tscl_device_of(h)));
  const DDimsTC& d = *tscl_dims_of(h);
  if ((d.dx % 8) != 0 || d.dx / 8 + 9 > WG_A_CHUNKS) return tsc_set_error("tscl_wgrad_tc: dx must be a multiple of 8, <= 240");
  const size_t smem = 2 * (size_t)WG_STAGE + 32;
  const size_t smem_async = (size_t)WGA_STAGES * WGA_STAGE + 4 * WGA_MAXT;
  static int attr_dev = -1;
  if (attr_dev != tscl_device_of(h)) {
    PCK(cudaFuncSetAttribute(wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PCK(cudaFuncSetAttribute(wgrad_tc_async_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_async));
    attr_dev = tscl_device_of(h);
  }
  int n_sm = 0;
  PCK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, tscl_device_of(h)));
  const int64_t M = (int64_t)T * rc;
  const int64_t NT = ((M + FBT_ROWS - 1) / FBT_ROWS) * 4 * d.A;
  const int grid = (int)(NT < n_sm ? NT : n_sm);
  WGradTC a;
  a.acc = nullptr;
  a.dZ = dZ; a.dZb = (const __nv_bfloat16*)dz_bf16; a.X = X; a.Xb = (const __nv_bfloat16*)x_bf16; a.Hp = Hp; a.Hb = (const __nv_bfloat16*)h_bf16; a.h0 = h0;
  a.done = done; a.G = grads; a.M = M; a.rc = rc; a.ld_state = ld_state; a.r0 = r0; a.T = T; a.variant = variant;
  if (a.dZb && a.Xb && a.Hb && T <= WGA_MAXT) {
    const int64_t nt2 = ((M + WGA_ROWS - 1) / WGA_ROWS) * 2 * d.A;
    const int nsl = wga_slabs(d.dx);
    const int g2 = (int)(nt2 < n_sm / nsl ? nt2 : n_sm / nsl) * nsl;      // groups of nsl CTAs, one per A slab
    wgrad_tc_async_kernel<<<g2, FBT_THREADS, smem_async, (cudaStream_t)stream>>>(d, a);
  }
  else {
    a.acc = acc_tiles(h, stream);
    if (!a.acc) return tsc_set_error("accumulator tiles: cudaMalloc failed");
    wgrad_tc_kernel<<<grid, FBT_THREADS, smem, (cudaStream_t)stream>>>(d, a);
  }
  PCK(cudaGetLastError());
  return 0;
}

// ===================================================================================================
// dX = dZ . Wx^T  (input gradient of the LSTM's x-projection, agents/utils.py:103-105 differentiated): a streaming GEMM
// [M x 256] . [256 x dx] per unit, 960 B of HBM traffic per row.  Warp-specialised persistent kernel:
//   warps 8-11  loaders : 16-byte cp.async of one swizzle atom (128 rows x 64 K, 16 KB) per stage, written in the
//                         SWIZZLE_128B K-major pattern (chunk ^ (row & 7)); 3 stages, completion signalled one stage late
//   warps 0-7   MMA     : two warpgroups (64 rows each), 4 x wgmma (N = dx, K = 16) per atom into register fragments
//                         (dx / 2 fp32 per thread, 168 registers at 384 threads), B = the unit's Wx^T image resident in
//                         shared memory (fetched by one cp.async.bulk per unit); an atom's stage is released as soon as
//                         the MMAs of the next atom are issued and its own have completed (wait_group 1)
//              epilogue : after the tile's 4 atoms, the same warps convert their fragments to bf16 into padded rows in
//                         shared memory, and one cp.async.bulk store per row (448 B) drains them while the next tile is
//                         multiplied
// A CTA owns a contiguous range of the (unit, 128-row tile) list, so it changes unit at most twice.
#define DXK_THREADS 384
#define DXK_STAGES 3
#define DXK_STAGE_BYTES 16384
struct DxTC {
  const __nv_bfloat16* dZb;    // [2A][M][256]
  const __nv_bfloat16* Wxt;    // [2A][32][dx][8]  (tscl_pack_wxt)
  __nv_bfloat16* dXb;          // [2A][M][dx]
  int64_t M;
};
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t saddr) {      // K-major, 128-byte swizzle, 8-row groups 1024 B apart
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);   // layout type 1: 128B swizzle
}

template <int DXT>
__global__ void __launch_bounds__(DXK_THREADS, 1)
dx_tc_kernel(const DDimsTC d, const DxTC a) {
  constexpr int N64 = DXT / 64, R32 = (DXT % 64) >= 32, R16 = (DXT % 32) >= 16;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int dx = DXT, row_bytes = dx * 2, out_stride = row_bytes + 16;
  unsigned char* sStage = tc_smem;
  unsigned char* sB = sStage + DXK_STAGES * DXK_STAGE_BYTES;
  unsigned char* sOut = sB + (size_t)BW_KC * dx * 16;
  uint64_t* sBar = reinterpret_cast<uint64_t*>(sOut + (size_t)128 * out_stride);
  const uint32_t bar_full = smem_u32(sBar), bar_empty = bar_full + 24, bar_b = bar_full + 48;
  if (tid == 0) {
    for (int s = 0; s < DXK_STAGES; ++s) { mbar_init(bar_full + 8 * s, 128); mbar_init(bar_empty + 8 * s, 8); }
    mbar_init(bar_b, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int64_t tpu = (a.M + 127) / 128;
  const int64_t NT = tpu * 2 * d.A;
  const int64_t j0 = NT * blockIdx.x / gridDim.x, j1 = NT * (blockIdx.x + 1) / gridDim.x;

  if (warp >= 8) {
    // ---------------- loaders ----------------
    const int lt = tid - 256;
    const uint32_t aS = smem_u32(sStage);
    int64_t it = 0;
    for (int64_t j = j0; j < j1; ++j) {
      const int u = (int)(j / tpu);
      const int64_t m0 = (j - (int64_t)u * tpu) * 128;
      const __nv_bfloat16* src0 = a.dZb + (int64_t)u * a.M * TC_N;
      for (int at = 0; at < 4; ++at, ++it) {
        const int s = (int)(it % DXK_STAGES);
        const int64_t n = it / DXK_STAGES;
        if (n > 0) mbar_wait(bar_empty + 8 * s, (uint32_t)((n - 1) & 1));
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int id = i * 128 + lt, rw = id >> 3, c = id & 7;
          const int64_t rr = m0 + rw < a.M ? m0 + rw : a.M - 1;
          cp_async16(aS + s * DXK_STAGE_BYTES + rw * 128 + ((c ^ (rw & 7)) << 4), src0 + rr * TC_N + at * 64 + c * 8);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        // one atom of lag, not two: the MMA warps release an atom's stage only once the next atom's MMAs are issued
        // (wait_group 1), so holding back the atom before that one would close a wait cycle
        if (it >= 1) {
          asm volatile("cp.async.wait_group 1;" ::: "memory");
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          mbar_arrive(bar_full + 8 * (int)((it - 1) % DXK_STAGES));
        }
      }
    }
    if (it >= 1) {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      mbar_arrive(bar_full + 8 * (int)((it - 1) % DXK_STAGES));
    }
  } else {
    // ---------------- MMA + epilogue: warps 0-7, one warpgroup per 64-row half ----------------
    const int wg = warp >> 2, tl = tid & 127;
    const uint32_t aS = smem_u32(sStage), aB = smem_u32(sB);
    const uint32_t b_lbo = (uint32_t)dx * 16;
    float f64[N64 > 0 ? N64 : 1][32], f32[16], f16[8];
    int64_t it = 0;
    int cur_u = -1, prev_s = 0;
    uint32_t bph = 0;
    // this thread's fragment rows within the tile, and the padded output row it stores (tl < 64)
    const int fr = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const uint32_t my_s = smem_u32(sOut + (size_t)(wg * 64 + tl) * out_stride);
    auto put = [&](int col, float x, float y, int r) {
      const __nv_bfloat162 v = __floats2bfloat162_rn(x, y);
      *reinterpret_cast<__nv_bfloat162*>(sOut + (size_t)r * out_stride + col * 2) = v;
    };
    for (int64_t j = j0; j < j1; ++j) {
      const int u = (int)(j / tpu);
      const int64_t m0 = (j - (int64_t)u * tpu) * 128;
      if (u != cur_u) {      // both warpgroups have waited for every MMA of the previous unit (end of its last tile)
        cur_u = u;
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (tid == 0) {
          const uint32_t bytes = (uint32_t)BW_KC * dx * 16;
          mbar_expect_tx(bar_b, bytes);
          bulk_g2s(aB, a.Wxt + (int64_t)u * BW_KC * dx * 8, bytes, bar_b);
        }
        mbar_wait(bar_b, bph); bph ^= 1;
      }
      for (int at = 0; at < 4; ++at, ++it) {
        const int s = (int)(it % DXK_STAGES);
        mbar_wait(bar_full + 8 * s, (uint32_t)((it / DXK_STAGES) & 1));
        const uint32_t a0 = aS + s * DXK_STAGE_BYTES + wg * 8192;
        const uint32_t b0 = aB + (uint32_t)(at * 8) * b_lbo;
        wg_fence();
#pragma unroll
        for (int q = 0; q < N64; ++q)
          wg_mma_regs<64, 0, 0>(f64[q], 4, at > 0, [&](int k, uint64_t& da, uint64_t& db) {
            da = make_desc_sw128(a0 + k * 32);
            db = make_desc(b0 + (uint32_t)(k * 2) * b_lbo + q * 64 * 16, b_lbo, 128);
          });
        if constexpr (R32)
          wg_mma_regs<32, 0, 0>(f32, 4, at > 0, [&](int k, uint64_t& da, uint64_t& db) {
            da = make_desc_sw128(a0 + k * 32);
            db = make_desc(b0 + (uint32_t)(k * 2) * b_lbo + N64 * 64 * 16, b_lbo, 128);
          });
        if constexpr (R16)
          wg_mma_regs<16, 0, 0>(f16, 4, at > 0, [&](int k, uint64_t& da, uint64_t& db) {
            da = make_desc_sw128(a0 + k * 32);
            db = make_desc(b0 + (uint32_t)(k * 2) * b_lbo + (N64 * 64 + R32 * 32) * 16, b_lbo, 128);
          });
        wg_commit();
        if (at > 0) {        // the MMAs of the previous atom have completed: release its stage
          wg_wait<1>();
          if (lane == 0) mbar_arrive(bar_empty + 8 * prev_s);
        }
        prev_s = s;
      }
      wg_wait<0>();
      if (lane == 0) mbar_arrive(bar_empty + 8 * prev_s);
#pragma unroll
      for (int q = 0; q < N64; ++q) wg_frag_fence(f64[q]);
      if constexpr (R32) wg_frag_fence(f32);
      if constexpr (R16) wg_frag_fence(f16);
      // ---- epilogue: fragments -> bf16 rows in shared memory -> one bulk store per row ----
      if (tl < 64) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");      // the previous tile's stores have left
      asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
      const int c0 = 2 * (lane & 3);
#pragma unroll
      for (int q = 0; q < N64; ++q)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          put(q * 64 + 8 * i + c0, f64[q][4 * i], f64[q][4 * i + 1], fr);
          put(q * 64 + 8 * i + c0, f64[q][4 * i + 2], f64[q][4 * i + 3], fr + 8);
        }
      if constexpr (R32)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          put(N64 * 64 + 8 * i + c0, f32[4 * i], f32[4 * i + 1], fr);
          put(N64 * 64 + 8 * i + c0, f32[4 * i + 2], f32[4 * i + 3], fr + 8);
        }
      if constexpr (R16)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          put(N64 * 64 + R32 * 32 + 8 * i + c0, f16[4 * i], f16[4 * i + 1], fr);
          put(N64 * 64 + R32 * 32 + 8 * i + c0, f16[4 * i + 2], f16[4 * i + 3], fr + 8);
        }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
      if (tl < 64) {
        const int64_t m = m0 + wg * 64 + tl;
        if (m < a.M) {
          __nv_bfloat16* dst = a.dXb + ((int64_t)u * a.M + m) * dx;
          asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(my_s), "r"(row_bytes) : "memory");
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
    }
    if (tl < 64) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
  __syncthreads();
}

extern "C" int tscl_dx_tc(tscl_handle* h, const void* dz_bf16, const void* wxt_bf16, void* dx_bf16, int64_t M, void* stream) {
  if (!h || !dz_bf16 || !wxt_bf16 || !dx_bf16 || M <= 0) return tsc_set_error("tscl_dx_tc: bad argument");
  PCK(cudaSetDevice(tscl_device_of(h)));
  const DDimsTC& d = *tscl_dims_of(h);
  if (d.dx % 16 != 0 || d.dx > 224 || d.dx < 16) return tsc_set_error("tscl_dx_tc: dx must be a multiple of 16 in [16, 224]");
  const size_t smem = (size_t)DXK_STAGES * DXK_STAGE_BYTES + (size_t)BW_KC * d.dx * 16 + (size_t)128 * (d.dx * 2 + 16) + 12 * 8 + 16;
  if (smem > 232448) return tsc_set_error("tscl_dx_tc: shared memory budget exceeded");
  void (*kern)(const DDimsTC, const DxTC) = nullptr;
  switch (d.dx) {      // the fragment size of the register accumulators is a compile-time constant
#define DXK_CASE(n) case n: kern = dx_tc_kernel<n>; break;
    DXK_CASE(16) DXK_CASE(32) DXK_CASE(48) DXK_CASE(64) DXK_CASE(80) DXK_CASE(96) DXK_CASE(112) DXK_CASE(128)
    DXK_CASE(144) DXK_CASE(160) DXK_CASE(176) DXK_CASE(192) DXK_CASE(208) DXK_CASE(224)
#undef DXK_CASE
  }
  static int attr_dev = -1;
  static void (*attr_kern)(const DDimsTC, const DxTC) = nullptr;
  if (attr_dev != tscl_device_of(h) || attr_kern != kern) {
    PCK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    attr_dev = tscl_device_of(h); attr_kern = kern;
  }
  int n_sm = 0;
  PCK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, tscl_device_of(h)));
  const int64_t NT = ((M + 127) / 128) * 2 * d.A;
  const int grid = (int)(NT < n_sm ? NT : n_sm);
  DxTC a;
  a.dZb = (const __nv_bfloat16*)dz_bf16; a.Wxt = (const __nv_bfloat16*)wxt_bf16; a.dXb = (__nv_bfloat16*)dx_bf16; a.M = M;
  kern<<<grid, DXK_THREADS, smem, (cudaStream_t)stream>>>(d, a);
  PCK(cudaGetLastError());
  return 0;
}

// ===================================================================================================
// dX fused into the fc front-end weight gradients: per (unit, 128-row tile) the kernel forms dX = dZ . Wx^T exactly as
// dx_tc_kernel does (same operands, same 4 atoms x 4 k16 order, so the bf16-rounded dX has the same bits), masks it by
// X > 0 (fc_bwd_tc_kernel's bf16 test) in registers, and multiplies it straight into the fc weight gradients:
//   D[64 input slots][dx] += In^T . dXm      (wgmma, A = In and B = dXm both MN-major in shared memory, K = 128 rows)
// dX never leaves the SM: per row the kernel reads dZ (512 B), X (2 dx B) and the observation slice, and writes nothing.
//   warp 8, lane 0    : TMA issue: dZ one swizzle atom (128 rows x 64 K, 16 KB) per stage, 2 stages; the tile's X as
//                       dx / 8 boxes of [128 rows][8 columns] straight into the MN-major dXm buffer
//   warps 9-11        : the observation tile In, gathered into the 64 input slots (plus the ones slot of the bias)
//   warps 0-7         : two warpgroups (64 rows each) run the dX MMAs into register fragments (dx / 2 per thread), then
//                       overwrite each X word in shared memory with the masked bf16 dX of the same (row, column pair), meet
//                       at a 256-thread barrier and multiply: warpgroup g owns dX columns [g dx / 2, (g + 1) dx / 2) of D,
//                       dx / 4 fp32 per thread, kept over all tiles of a unit and flushed to G with atomics when the unit
//                       changes (the column -> fcw / fcf / fct and slot -> input mapping of fc_bwd_tc_kernel)
// Shared memory at dx = 224: 32 KB dZ stages + 112 KB Wx^T image + 56 KB dXm + 16.1 KB In = 216 KB.  setmaxnreg gives the
// consumers 216 registers at dx = 224 (dX 112 + fc 56 fragments), the producer warps 72.
#define DXF_THREADS 384
#define DXF_STAGES 2
#define DXF_SBO 2048                       // dXm chunk stride: 128 rows x 16 B (a TMA destination: 128-byte aligned)
#define DXF_BUILDERS 96                    // warps 9-11
// (dx = 224 needs 8 more consumer registers than the narrower widths, which leave the producer warps 80)
#define DXF_CONS_REGS(dx) ((dx) > 192 ? 216 : 208)
#define DXF_PROD_REGS(dx) ((dx) > 192 ? 72 : 80)
static_assert(128 * DXF_PROD_REGS(224) + 256 * DXF_CONS_REGS(224) <= DXF_THREADS * 168 &&
              128 * DXF_PROD_REGS(160) + 256 * DXF_CONS_REGS(160) <= DXF_THREADS * 168,
              "setmaxnreg split exceeds the CTA's registers");
static size_t dxf_smem(int dx) {
  return (size_t)DXF_STAGES * DXK_STAGE_BYTES + (size_t)BW_KC * dx * 16 + (size_t)(dx / 8) * DXF_SBO + 8 * FBT_SBO + 8 * 8;
}
struct DxFcTC {
  const float* obs;            // rows as tscl_fc_embed
  const __nv_bfloat16* Wxt;    // [2A][32][dx][8]  (tscl_pack_wxt)
  float* G;
  int64_t M, rows_per_t, stride_t;
};
// 0xFFFF per 16-bit half of x where that bf16 value is > 0
__device__ __forceinline__ uint32_t bf16x2_pos_mask(uint32_t x) {
  const uint32_t nz = ((x & 0x7FFF7FFFu) + 0x7FFF7FFFu) & ~x & 0x80008000u;
  return (nz >> 15) * 0xFFFFu;
}
// an fc fragment of unit u into G: input slot 16 (warp & 3) + lane / 4 (+ 8 for entries 4 i + 2, 4 i + 3),
// dX column cb + 8 i + 2 (lane & 3) (+ 1 for the odd entries)
template <int NR>
__device__ __forceinline__ void dxf_flush(const DDimsTC& d, float* G, int u, const float (&f)[NR], int cb) {
  const int lane = threadIdx.x & 31, w4 = (threadIdx.x >> 5) & 3, ag = u >> 1;
  const int nw = d.n_wave[ag], nt = d.n_wait[ag], nf = d.ff > 0 ? d.n_fp[ag] : 0;
#pragma unroll
  for (int e = 0; e < NR; ++e) {
    const int slot = 16 * w4 + (lane >> 2) + 8 * ((e >> 1) & 1);
    const int c = cb + 8 * (e >> 2) + 2 * (lane & 3) + (e & 1);
    int64_t wo, bo; int ld, cc, s0, n;
    if (c < d.fw) { wo = d.off_fcw_w[u]; bo = d.off_fcw_b[u]; ld = d.fw; cc = c; s0 = 0; n = nw; }
    else if (c < d.fw + d.ff) { wo = d.off_fcf_w[u]; bo = d.off_fcf_b[u]; ld = d.ff; cc = c - d.fw; s0 = d.kw; n = nf; }
    else { wo = d.off_fct_w[u]; bo = d.off_fct_b[u]; ld = d.ft; cc = c - d.fw - d.ff; s0 = d.kw + TC_KF; n = nt; }
    const int kin = slot - s0;
    if (kin >= 0 && kin < n) atomicAdd(&G[wo + (int64_t)kin * ld + cc], f[e]);
    if (slot == d.ones_slot) atomicAdd(&G[bo + cc], f[e]);
  }
}

template <int DX>
__global__ void __launch_bounds__(DXF_THREADS, 1)
dx_fc_bwd_tc_kernel(const DDimsTC d, const DxFcTC a, const __grid_constant__ CUtensorMap mapZ,
                    const __grid_constant__ CUtensorMap mapX) {
  constexpr int N64 = DX / 64, R32 = (DX % 64) >= 32, R16 = (DX % 32) >= 16;      // dX fragments: the tile's dx columns
  constexpr int HN = DX / 2, H32 = (HN % 64) >= 32, H16 = (HN % 32) >= 16;        // fc fragments: this warpgroup's half
  static_assert(HN >= 64 && HN < 128 && HN % 16 == 0, "fc half width must be 64 + {0, 16, 32, 48}");
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  unsigned char* sStage = tc_smem;
  unsigned char* sW = sStage + DXF_STAGES * DXK_STAGE_BYTES;
  unsigned char* sA = sW + (size_t)BW_KC * DX * 16;              // X, then masked dX: [dx / 8][128 rows][8] bf16
  unsigned char* sB = sA + (size_t)(DX / 8) * DXF_SBO;           // In: [8][128 rows][8] bf16, chunk stride FBT_SBO
  uint64_t* sBar = reinterpret_cast<uint64_t*>(sB + 8 * FBT_SBO);
  const uint32_t bar_full = smem_u32(sBar), bar_empty = bar_full + 16, bar_w = bar_full + 32, bar_x = bar_full + 40,
                 bar_in = bar_full + 48, bar_free = bar_full + 56;
  if (tid == 0) {
    for (int s = 0; s < DXF_STAGES; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 8); }
    mbar_init(bar_w, 1); mbar_init(bar_x, 1); mbar_init(bar_in, DXF_BUILDERS); mbar_init(bar_free, 8);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // the CTA's contiguous range [j0, j1) of the (unit, tile) list, formed in each role after its setmaxnreg
#define DXF_RANGE                                                                                   \
  const int64_t tpu = (a.M + 127) / 128;                                                            \
  const int64_t NT = tpu * 2 * d.A;                                                                 \
  const int64_t j0 = NT * blockIdx.x / gridDim.x, j1 = NT * (blockIdx.x + 1) / gridDim.x;

  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(DXF_PROD_REGS(DX)));
    DXF_RANGE
    if (warp == 8) {
      // ---------------- TMA issue ----------------
      if (lane == 0) {
        const uint32_t aS = smem_u32(sStage), aA = smem_u32(sA);
        int64_t it = 0;
        for (int64_t j = j0; j < j1; ++j) {
          const int u = (int)(j / tpu), m0 = (int)((j - (int64_t)u * tpu) * 128);
          auto atom = [&](int at) {
            const int s = (int)(it % DXF_STAGES);
            const int64_t n = it / DXF_STAGES;
            if (n > 0) mbar_wait(bar_empty + 8 * s, (uint32_t)((n - 1) & 1));
            mbar_expect_tx(bar_full + 8 * s, DXK_STAGE_BYTES);
            tma_load_3d(aS + s * DXK_STAGE_BYTES, &mapZ, at * 64, m0, u, bar_full + 8 * s);
            ++it;
          };
          atom(0); atom(1);
          // X of this tile once both warpgroups have multiplied the previous tile's dXm
          if (j > j0) mbar_wait(bar_free, (uint32_t)((j - j0 - 1) & 1));
          mbar_expect_tx(bar_x, (DX / 8) * DXF_SBO);
#pragma unroll 1
          for (int cg = 0; cg < DX / 8; ++cg) tma_load_3d(aA + cg * DXF_SBO, &mapX, cg * 8, m0, u, bar_x);
          atom(2); atom(3);
        }
      }
    } else {
      // ---------------- observation tile: item i = (row i / 8, input-slot chunk i % 8) ----------------
      const int bt = tid - 288, bc = bt & 7;      // DXF_BUILDERS is a multiple of 8: every item of a thread has chunk bc
      int cur_u = -1, ooff = 0;
      int src[8];                                 // observation index of each of the chunk's 8 slots (-1 none, -2 one)
      for (int64_t j = j0; j < j1; ++j) {
        const int u = (int)(j / tpu);
        const int64_t m0 = (j - (int64_t)u * tpu) * 128;
        if (u != cur_u) {
          cur_u = u;
          const int ag = u >> 1;
          const int nw = d.n_wave[ag], nt = d.n_wait[ag], nf = d.ff > 0 ? d.n_fp[ag] : 0;
          ooff = d.obs_off[ag];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const int slot = bc * 8 + e;
            int sidx = -1;
            if (slot < d.kw) { if (slot < nw) sidx = slot; }
            else if (slot < d.kw + TC_KF) { if (slot - d.kw < nf) sidx = nw + nt + (slot - d.kw); }
            else { if (slot - d.kw - TC_KF < nt) sidx = nw + (slot - d.kw - TC_KF); }
            if (slot == d.ones_slot) sidx = -2;
            src[e] = sidx;
          }
        }
        const int rows_valid = (a.M - m0) < 128 ? (int)(a.M - m0) : 128;
        const int64_t tq = m0 / a.rows_per_t, rem0 = m0 - tq * a.rows_per_t;
        if (j > j0) mbar_wait(bar_free, (uint32_t)((j - j0 - 1) & 1));
#pragma unroll 1
        for (int i = bt; i < 128 * 8; i += 2 * DXF_BUILDERS) {      // two items (rows i / 8, i / 8 + 12) per pass
          float v[2][8];
#pragma unroll
          for (int p = 0; p < 2; ++p) {
            const int row = (i + p * DXF_BUILDERS) >> 3;
#pragma unroll
            for (int e = 0; e < 8; ++e) v[p][e] = 0.f;
            if (i + p * DXF_BUILDERS < 128 * 8 && row < rows_valid) {
              int64_t tt = tq, rem = rem0 + row;
              while (rem >= a.rows_per_t) { rem -= a.rows_per_t; ++tt; }
              const float* op = a.obs + tt * a.stride_t + rem * d.n_obs + ooff;
#pragma unroll
              for (int e = 0; e < 8; ++e) v[p][e] = src[e] >= 0 ? __ldg(op + src[e]) : (src[e] == -2 ? 1.0f : 0.f);
            }
          }
#pragma unroll
          for (int p = 0; p < 2; ++p) {
            const int ii = i + p * DXF_BUILDERS;
            if (ii < 128 * 8) {
              __align__(16) __nv_bfloat16 o[8];
#pragma unroll
              for (int e = 0; e < 8; ++e) o[e] = __float2bfloat16_rn(v[p][e]);
              *reinterpret_cast<uint4*>(sB + (size_t)bc * FBT_SBO + (ii >> 3) * 16) = *reinterpret_cast<const uint4*>(o);
            }
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic writes -> operand of the wgmmas
        mbar_arrive(bar_in);
        if (j + 1 < j1) {      // pull the next tile's observation rows towards L2 while this tile is multiplied
          const int un = (int)((j + 1) / tpu);
          const int ooff_n = d.obs_off[un >> 1];
          for (int r = bt; r < 128; r += DXF_BUILDERS) {
            const int64_t m = (j + 1 - (int64_t)un * tpu) * 128 + r;
            if (m >= a.M) break;
            const float* op = a.obs + (m / a.rows_per_t) * a.stride_t + (m % a.rows_per_t) * d.n_obs + ooff_n;
            asm volatile("prefetch.global.L2 [%0];" ::"l"(op));
            asm volatile("prefetch.global.L2 [%0];" ::"l"(op + 32));
          }
        }
      }
    }
  } else {
    // ---------------- dX MMA, mask, fc MMA: warps 0-7, one warpgroup per 64-row half ----------------
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(DXF_CONS_REGS(DX)));
    DXF_RANGE
    const int wg = warp >> 2;
    const uint32_t aS = smem_u32(sStage), aW = smem_u32(sW), aA = smem_u32(sA), aB = smem_u32(sB);
    const uint32_t b_lbo = (uint32_t)DX * 16;
    float f64[N64][32], f32[R32 ? 16 : 1], f16[R16 ? 8 : 1];
    float g64[32], g32[H32 ? 16 : 1], g16[H16 ? 8 : 1];
    const int n0 = wg * HN;                       // this warpgroup's first dX column of D
    int64_t it = 0;
    int cur_u = -1, prev_s = 0;
    uint32_t wph = 0;
    bool first = true;
    const int fr = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
    // the X word of (row r, columns col, col + 1) becomes the masked bf16 dX of the same pair
    auto mask_put = [&](int col, float x, float y, int r) {
      uint32_t* p = reinterpret_cast<uint32_t*>(sA + (size_t)(col >> 3) * DXF_SBO + r * 16 + (col & 7) * 2);
      const __nv_bfloat162 v = __floats2bfloat162_rn(x, y);
      *p = *reinterpret_cast<const uint32_t*>(&v) & bf16x2_pos_mask(*p);
    };
    auto flush = [&](int u) {
      dxf_flush(d, a.G, u, g64, n0);
      if constexpr (H32) dxf_flush(d, a.G, u, g32, n0 + 64);
      if constexpr (H16) dxf_flush(d, a.G, u, g16, n0 + 64 + 32 * H32);
    };
    for (int64_t j = j0; j < j1; ++j) {
      const int u = (int)(j / tpu);
      const uint32_t ph = (uint32_t)((j - j0) & 1);
      if (u != cur_u) {
        if (cur_u >= 0) flush(cur_u);
        cur_u = u; first = true;
        asm volatile("bar.sync 1, 256;" ::: "memory");      // both warpgroups' MMAs of the previous unit have completed
        if (tid == 0) {
          const uint32_t bytes = (uint32_t)BW_KC * DX * 16;
          mbar_expect_tx(bar_w, bytes);
          bulk_g2s(aW, a.Wxt + (int64_t)u * BW_KC * DX * 8, bytes, bar_w);
        }
        mbar_wait(bar_w, wph); wph ^= 1;
      }
      // ---- dX = dZ . Wx^T: dx_tc_kernel's MMA sequence ----
      for (int at = 0; at < 4; ++at, ++it) {
        const int s = (int)(it % DXF_STAGES);
        mbar_wait(bar_full + 8 * s, (uint32_t)((it / DXF_STAGES) & 1));
        const uint32_t a0 = aS + s * DXK_STAGE_BYTES + wg * 8192;
        const uint32_t b0 = aW + (uint32_t)(at * 8) * b_lbo;
        wg_fence();
#pragma unroll
        for (int q = 0; q < N64; ++q)
          wg_mma_regs<64, 0, 0>(f64[q], 4, at > 0, [&](int k, uint64_t& da, uint64_t& db) {
            da = make_desc_sw128(a0 + k * 32);
            db = make_desc(b0 + (uint32_t)(k * 2) * b_lbo + q * 64 * 16, b_lbo, 128);
          });
        if constexpr (R32)
          wg_mma_regs<32, 0, 0>(f32, 4, at > 0, [&](int k, uint64_t& da, uint64_t& db) {
            da = make_desc_sw128(a0 + k * 32);
            db = make_desc(b0 + (uint32_t)(k * 2) * b_lbo + N64 * 64 * 16, b_lbo, 128);
          });
        if constexpr (R16)
          wg_mma_regs<16, 0, 0>(f16, 4, at > 0, [&](int k, uint64_t& da, uint64_t& db) {
            da = make_desc_sw128(a0 + k * 32);
            db = make_desc(b0 + (uint32_t)(k * 2) * b_lbo + (N64 * 64 + R32 * 32) * 16, b_lbo, 128);
          });
        wg_commit();
        if (at > 0) {        // the MMAs of the previous atom have completed: release its stage
          wg_wait<1>();
          if (lane == 0) mbar_arrive(bar_empty + 8 * prev_s);
        }
        prev_s = s;
      }
      wg_wait<0>();
      if (lane == 0) mbar_arrive(bar_empty + 8 * prev_s);
#pragma unroll
      for (int q = 0; q < N64; ++q) wg_frag_fence(f64[q]);
      if constexpr (R32) wg_frag_fence(f32);
      if constexpr (R16) wg_frag_fence(f16);
      // ---- mask in place: X -> dX (bf16) where X > 0, else 0 (rows past M: X is zero-filled by the TMA) ----
      mbar_wait(bar_x, ph);
#pragma unroll
      for (int q = 0; q < N64; ++q)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          mask_put(q * 64 + 8 * i + c0, f64[q][4 * i], f64[q][4 * i + 1], fr);
          mask_put(q * 64 + 8 * i + c0, f64[q][4 * i + 2], f64[q][4 * i + 3], fr + 8);
        }
      if constexpr (R32)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          mask_put(N64 * 64 + 8 * i + c0, f32[4 * i], f32[4 * i + 1], fr);
          mask_put(N64 * 64 + 8 * i + c0, f32[4 * i + 2], f32[4 * i + 3], fr + 8);
        }
      if constexpr (R16)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          mask_put(N64 * 64 + R32 * 32 + 8 * i + c0, f16[4 * i], f16[4 * i + 1], fr);
          mask_put(N64 * 64 + R32 * 32 + 8 * i + c0, f16[4 * i + 2], f16[4 * i + 3], fr + 8);
        }
      mbar_wait(bar_in, ph);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      asm volatile("bar.sync 1, 256;" ::: "memory");      // the whole 128-row dXm tile is in place
      // ---- D[slot][n0 ..] += In^T . dXm over the tile's 128 rows ----
      wg_fence();
      wg_mma_regs<64, 1, 1>(g64, 8, !first, [&](int ks, uint64_t& da, uint64_t& db) {
        da = make_desc(aB + ks * 256, 128, FBT_SBO);
        db = make_desc(aA + (n0 / 8) * DXF_SBO + ks * 256, 128, DXF_SBO);
      });
      if constexpr (H32)
        wg_mma_regs<32, 1, 1>(g32, 8, !first, [&](int ks, uint64_t& da, uint64_t& db) {
          da = make_desc(aB + ks * 256, 128, FBT_SBO);
          db = make_desc(aA + ((n0 + 64) / 8) * DXF_SBO + ks * 256, 128, DXF_SBO);
        });
      if constexpr (H16)
        wg_mma_regs<16, 1, 1>(g16, 8, !first, [&](int ks, uint64_t& da, uint64_t& db) {
          da = make_desc(aB + ks * 256, 128, FBT_SBO);
          db = make_desc(aA + ((n0 + 64 + 32 * H32) / 8) * DXF_SBO + ks * 256, 128, DXF_SBO);
        });
      wg_commit();
      wg_wait<0>();
      wg_frag_fence(g64);
      if constexpr (H32) wg_frag_fence(g32);
      if constexpr (H16) wg_frag_fence(g16);
      if (lane == 0) mbar_arrive(bar_free);      // this warp is done reading dXm and In
      first = false;
    }
    if (cur_u >= 0) flush(cur_u);
  }
#undef DXF_RANGE
}

extern "C" int tscl_dx_fc_bwd_tc(tscl_handle* h, const float* obs, const void* x_bf16, const void* dz_bf16,
                                 const void* wxt_bf16, int64_t M, int64_t rows_per_t, int64_t stride_t, float* grads,
                                 void* stream) {
  if (!h || !obs || !x_bf16 || !dz_bf16 || !wxt_bf16 || !grads || M <= 0 || rows_per_t <= 0)
    return tsc_set_error("tscl_dx_fc_bwd_tc: bad argument");
  if (M >= ((int64_t)1 << 31) - 128) return tsc_set_error("tscl_dx_fc_bwd_tc: M must be below 2^31 - 128 rows");
  PCK(cudaSetDevice(tscl_device_of(h)));
  const DDimsTC& d = *tscl_dims_of(h);
  if (!P2_DX_OK(d.dx)) return tsc_set_error("tscl_dx_fc_bwd_tc: dx must be 128, 160, 192 or 224 (use tscl_dx_tc + tscl_fc_bwd_tc)");
  if (d.kw == 0 || d.ones_slot < 0) return tsc_set_error("tscl_dx_fc_bwd_tc: no free input slot for the bias column");
  CUtensorMap mZ, mX;
  if (!make_tmap_3d(&mZ, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, dz_bf16, 2 * d.A, M, TC_N, 64, 128) ||
      !make_tmap_3d(&mX, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, x_bf16, 2 * d.A, M, d.dx, 8, 128, CU_TENSOR_MAP_SWIZZLE_NONE))
    return tsc_set_error("tscl_dx_fc_bwd_tc: cannot build the tensor maps (dz_bf16 / x_bf16 must be 16-byte aligned)");
  void (*kern)(const DDimsTC, const DxFcTC, const CUtensorMap, const CUtensorMap) =
      d.dx == 224 ? dx_fc_bwd_tc_kernel<224> : d.dx == 192 ? dx_fc_bwd_tc_kernel<192> :
      d.dx == 160 ? dx_fc_bwd_tc_kernel<160> : dx_fc_bwd_tc_kernel<128>;
  const size_t smem = dxf_smem(d.dx);
  static int attr_dev = -1;
  if (attr_dev != tscl_device_of(h)) {
    PCK(cudaFuncSetAttribute(dx_fc_bwd_tc_kernel<224>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dxf_smem(224)));
    PCK(cudaFuncSetAttribute(dx_fc_bwd_tc_kernel<192>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dxf_smem(192)));
    PCK(cudaFuncSetAttribute(dx_fc_bwd_tc_kernel<160>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dxf_smem(160)));
    PCK(cudaFuncSetAttribute(dx_fc_bwd_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dxf_smem(128)));
    attr_dev = tscl_device_of(h);
  }
  int n_sm = 0;
  PCK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, tscl_device_of(h)));
  const int64_t NT = ((M + 127) / 128) * 2 * d.A;
  const int grid = (int)(NT < n_sm ? NT : n_sm);
  DxFcTC a;
  a.obs = obs; a.Wxt = (const __nv_bfloat16*)wxt_bf16; a.G = grads; a.M = M; a.rows_per_t = rows_per_t; a.stride_t = stride_t;
  kern<<<grid, DXF_THREADS, smem, (cudaStream_t)stream>>>(d, a, mZ, mX);
  PCK(cudaGetLastError());
  return 0;
}
