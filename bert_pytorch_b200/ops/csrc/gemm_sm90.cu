// Warp-specialised wgmma GEMM for sm_90a with fused epilogues.
//
//   D[M,N] = epilogue( A[M,K] * B[N,K]^T )        bf16 (or fp8) operands, fp32 accumulation in registers
//
// Persistent: a work unit is one 128 x BLOCK_N output tile and K range, and min(units, SMs) CTAs each walk the units
// blockIdx.x, blockIdx.x + gridDim.x, ...  Warpgroup 0 is the producer: one thread moves operand tiles global ->
// shared memory with cp.async.bulk.tensor (TMA, 128B swizzle) through a STAGES-deep mbarrier ring, running straight
// across unit boundaries, so the next unit's operands arrive while the consumers are still in an epilogue.
// Warpgroups 1 and 2 issue wgmma.mma_async straight from the ring, keep one group in flight, hand a slot back as soon
// as the group that read it has retired, and run the epilogue from their accumulator registers.  Two schedules:
//   BLOCK_N 256, cooperative: both warpgroups work on every unit, 64 rows each (half the A traffic per FLOP of
//                128 x 128; the tensor cores idle while both run the epilogue).
//   BLOCK_N 128, ping-pong:   the warpgroups take alternate units, each the whole 128 x 128 tile, and a pair of named
//                barriers orders their main loops, so one warpgroup's epilogue runs under the other's MMAs.
//
// Both bf16 operands can be K-major (reduction dim contiguous) or MN-major, selected per instantiation, so the same
// kernel serves the three GEMMs of a linear layer without any transpose copy:
//     forward  Y  = X  W^T        A K-major (X[M,K]),     B K-major  (W[N,K])
//     dgrad    dX = dY W          A K-major (dY[M,N']),   B MN-major (W[N',K'] read as [Kred][N])
//     wgrad    dW = dY^T X        A MN-major (dY[M,N']),  B MN-major (X[M,K'])   (+ split-K, fp32 reductions)
// fp8 wgmma reads K-major operands only: an MN-major fp8 operand is transposed once into a stream-ordered scratch
// buffer (fp8_transpose_kernel) and the GEMM runs in the NT form.
//
// Epilogues (a template argument: every kernel carries the straight-line code of one epilogue): bias, bias+GELU(erf)
// with the derivative saved for backward, bias+dropout+residual, residual add, multiply by a saved factor, fp32
// accumulate-into (wgrad into the gradient arena), bias+tanh, plain fp32.  gemm_bf16 lists the (operand form,
// epilogue) pairs that are built.  The accumulator fragment is regrouped inside each quad (quad_transpose) so that a
// thread owns 8 consecutive output columns: one 16-byte store, one Philox draw and one keep-bit byte per group.  The
// bf16 epilogues that read a residual or saved factor, and bias and bias + tanh, stage their output through shared
// memory and store it with TMA (staged_epilogue); the others store from registers (fragment_epilogue).
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "gemm_sm90.h"
#include "wgmma.cuh"

namespace b200 {

constexpr int BLOCK_M = 128;
constexpr int TILE_K_BYTES = 128;    // one swizzle atom row: 64 bf16 or 128 fp8 along K
constexpr int NUM_THREADS = 384;     // warpgroup 0: TMA producer, warpgroups 1-2: MMA + epilogue
constexpr int SMEM_BUDGET = 196608;  // bytes for the operand ring (192 of the 227 KB a block may use)

template <int BLOCK_N>
struct Cfg {
  static constexpr int A_BYTES = BLOCK_M * TILE_K_BYTES;
  static constexpr int B_BYTES = BLOCK_N * TILE_K_BYTES;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = SMEM_BUDGET / STAGE_BYTES;      // 6 (BLOCK_N 128) or 4 (256)
  static constexpr int SMEM_TOTAL = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
  // bf16-output epilogues add two 8 KB staging subtiles and a BLOCK_N bias slice per consumer warpgroup (see
  // staged_epilogue)
  static constexpr int SMEM_STAGED = SMEM_TOTAL + 2 * (2 * 8192 + BLOCK_N * 2);
  static_assert(SMEM_STAGED <= 232448, "more dynamic shared memory than an sm_90 block may use");
};

struct GemmArgs {
  int M, N, K;
  int m_blocks, n_blocks, k_blocks, k_splits, k_per_split;
  int units;                 // m_blocks * n_blocks * k_splits
  void* out;
  int ldo;
  __nv_bfloat16* aux_out;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* res;
  int ldr;
  float* colsum;             // optional fp32 column sums of the bf16 output (bias gradients)
  unsigned char* mask_out;   // optional dropout keep bits, [M][N / 8] bytes (GemmCall::mask_out)
  const unsigned char* mask_in;   // the same bits as input: applied instead of generated (GemmCall::mask_in)
  Seed seed;
  unsigned int stream;
  unsigned int drop_thresh16;
  float drop_scale;
  float alpha;
  const float* scale_a;      // fp8: device dequantisation factors (nullptr for bf16 operands)
  const float* scale_b;
  unsigned int fp8_fmt;      // bit0: A is e5m2 (else e4m3), bit1: B is e5m2
  // GEMM -> reduce-scatter fusion (EPI_ACCUM_F32 into a gradient arena that lives in NVLink symmetric memory):
  // peer_world > 1 makes every accumulation a system-scope reduction (peers add into this arena concurrently);
  // peer_push adds the tile -- plus, once per tile, the locally accumulated value -- straight into the arena of the
  // rank that owns that shard, so the gradient is reduced tile by tile while the backward pass is still running.
  int peer_world, peer_rank, peer_push;
  long long peer_off;        // element offset of `out` inside the arena
  long long peer_per;        // shard size in elements: owner(e) = min(e / peer_per, world - 1)
  float* peer_base[16];      // gradient arena of every rank (symmetric-memory mapping)
#ifdef B200_GEMM_TIMELINE
  long long* timeline;       // [units][TL_STRIDE] clock64 stamps (nullptr: not recorded), see gemm_set_timeline
#endif
};

// In-kernel timeline (build with -DB200_GEMM_TIMELINE, read by tools/gemm_timeline.py).  Record of unit u:
//   [6 cw + 0..5]  consumer warpgroup cw that ran the unit: turn taken, first full_bar passed, last MMA issued,
//                  wgmma_wait<0> returned, epilogue done, cycles spent waiting on full_bar
//   [12] cycles the producer was blocked on empty_bar while loading the unit   [13] gridDim.x
// SM clock cycles (clock64): stamps are compared only within one CTA.  Register reads only, so the define adds no
// call to the wgmma pipeline.
#ifdef B200_GEMM_TIMELINE
constexpr int TL_STRIDE = 16;
struct UnitStamps {
  long long start, full0, last_mma, wait0, epi_done, op_wait;
};
#define TL(...) __VA_ARGS__
#else
#define TL(...)
#endif

// bf16-output epilogue math of W consecutive output columns of one row (W even).  `f` holds alpha * accumulator,
// `bias` and `res` the packed bf16 bias and residual / saved-factor values of those columns (read only when p.bias /
// p.res is set), `kb` their dropout keep bits (bit t: column t; applied when the epilogue drops).  Writes the packed
// bf16 output to `out` and, for EPI_BIAS_GELU_DG, gelu' to `aux`.
template <int E, int W>
__device__ __forceinline__ void epilogue_math(const GemmArgs& p, float (&f)[W], const uint32_t (&bias)[W / 2],
                                              uint32_t kb, const uint32_t (&res)[W / 2], uint32_t (&out)[W / 2],
                                              uint32_t (&aux)[W / 2]) {
  if constexpr (epilogue_spec(E).bias) {
    if (p.bias != nullptr) {
#pragma unroll
      for (int t = 0; t < W / 2; ++t) {
        const float2 bb = unpack_bf16(bias[t]);
        f[2 * t] += bb.x;
        f[2 * t + 1] += bb.y;
      }
    }
  }
  if constexpr (E == EPI_BIAS_GELU_DG) {
    float dg[W];
#pragma unroll
    for (int j = 0; j < W; ++j) {
      const GeluParts gp = gelu_parts(f[j]);
      dg[j] = fmaf(f[j] * 0.3989422804014327f, gp.e, gp.Phi);
      f[j] *= gp.Phi;
    }
#pragma unroll
    for (int t = 0; t < W / 2; ++t) aux[t] = pack_bf16(dg[2 * t], dg[2 * t + 1]);
  } else if constexpr (E == EPI_BIAS_TANH) {
#pragma unroll
    for (int j = 0; j < W; ++j) f[j] = tanhf(f[j]);
  } else if constexpr (E == EPI_BIAS_DROP_RES || E == EPI_ADD || E == EPI_MUL) {
    if constexpr (epilogue_spec(E).keep_bits) {
      if (p.drop_thresh16 != 0) {
#pragma unroll
        for (int t = 0; t < W; ++t) f[t] = (kb >> t) & 1u ? __fmul_rn(f[t], p.drop_scale) : 0.f;
      }
    }
    if (p.res != nullptr) {
#pragma unroll
      for (int t = 0; t < W / 2; ++t) {
        const float2 rr = unpack_bf16(res[t]);
        if constexpr (E == EPI_MUL) {
          f[2 * t] *= rr.x;
          f[2 * t + 1] *= rr.y;
        } else {
          f[2 * t] += rr.x;
          f[2 * t + 1] += rr.y;
        }
      }
    }
  }
#pragma unroll
  for (int t = 0; t < W / 2; ++t) out[t] = pack_bf16(f[2 * t], f[2 * t + 1]);
}

// Work unit u of a launch: output tile (mb, nb) and k-blocks [kb0, kb0 + nkb) -- split-major, then m-block, then
// n-block, so the units that run at the same time share their A rows in L2.
struct Unit {
  int mb, nb, ks, kb0, nkb;
};
__device__ __forceinline__ Unit unit_of(const GemmArgs& p, int u) {
  Unit w;
  w.nb = u % p.n_blocks;
  w.mb = (u / p.n_blocks) % p.m_blocks;
  w.ks = u / (p.n_blocks * p.m_blocks);
  w.kb0 = w.ks * p.k_per_split;
  w.nkb = min(p.k_blocks, w.kb0 + p.k_per_split) - w.kb0;   // >= 1: the launcher leaves no empty split
  return w;
}

// Main loop of one consumer warpgroup over one unit: acc[r] (+)= A[64 rows, chunk a_chunk + r] * B over the unit's
// nkb k-blocks, which sit at ring positions it, it + 1, ...  `arrive_bar` >= 0: once every MMA is issued, let the
// other warpgroup start its main loop (ping-pong order).
template <bool A_MN, bool B_MN, int BLOCK_N, int R, bool FP8, int AE5, int BE5>
__device__ __forceinline__ void consumer_mainloop(float (&acc)[R][BLOCK_N / 2], uint8_t* smem, uint64_t* full_bar,
                                                  uint64_t* empty_bar, int a_chunk, uint32_t it, int nkb,
                                                  int arrive_bar TL(, UnitStamps& st)) {
  using C = Cfg<BLOCK_N>;
  const int lane = threadIdx.x & 31;
  int s = it % C::STAGES, prev = -1;
  uint32_t ph = (it / C::STAGES) & 1;
#pragma unroll
  for (int r = 0; r < R; ++r) wgmma_fence_regs(acc[r]);
  for (int i = 0; i < nkb; ++i) {
#ifdef B200_GEMM_TIMELINE
    if (!mbar_try_wait(&full_bar[s], ph)) {
      const long long t = clock64();
      mbar_wait_mma(&full_bar[s], ph);
      st.op_wait += clock64() - t;
    }
    if (i == 0) st.full0 = clock64();
#else
    mbar_wait_mma(&full_bar[s], ph);
#endif
    const uint32_t sa = smem_u32(smem + s * C::STAGE_BYTES) + a_chunk * 8192;   // 64 rows (or a 64-wide MN chunk) of A
    const uint32_t sb = smem_u32(smem + s * C::STAGE_BYTES) + C::A_BYTES;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      // advance inside the tile: K-major +32 B per MMA (16 bf16 / 32 fp8), MN-major +16 k-rows * 128 B
      const uint64_t db = B_MN ? wgmma_desc_sw128(sb + kk * 2048, 8192, 1024) : wgmma_desc_sw128(sb + kk * 32, 16, 1024);
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const uint32_t sr = sa + r * 8192;
        const uint64_t da = A_MN ? wgmma_desc_sw128(sr + kk * 2048, 8192, 1024) : wgmma_desc_sw128(sr + kk * 32, 16, 1024);
        if constexpr (FP8) WgmmaFp8SS<BLOCK_N, AE5, BE5>::mma(acc[r], da, db, (i > 0 || kk > 0) ? 1 : 0);
        else WgmmaBf16SS<BLOCK_N, A_MN ? 1 : 0, B_MN ? 1 : 0>::mma(acc[r], da, db, (i > 0 || kk > 0) ? 1 : 0);
      }
    }
    wgmma_commit();
    TL(st.last_mma = clock64();)
    wgmma_wait<1>();                              // the group that read slot `prev` has retired
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    prev = s;
    if (++s == C::STAGES) { s = 0; ph ^= 1; }
  }
  if (arrive_bar >= 0) asm volatile("bar.arrive %0, 256;" ::"r"(arrive_bar) : "memory");
  wgmma_wait<0>();
#pragma unroll
  for (int r = 0; r < R; ++r) wgmma_fence_regs(acc[r]);
  TL(st.wait0 = clock64();)
  if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
}

// Register epilogue of 8 consecutive output columns [n0, n0 + 8) of one row (n0 % 8 == 0, N % 8 == 0), stored
// straight from registers (the epilogues that do not stage their output, see staged_epi).  `f` holds alpha *
// accumulator.  Returns through `f` the values that were stored (bf16-rounded) for the column sums.
template <int E>
__device__ __forceinline__ void epilogue_group(const GemmArgs& p, float (&f)[8], int row, int n0, bool add_local) {
  const size_t ooff = (size_t)row * p.ldo + n0;
  if constexpr (E == EPI_ACCUM_F32) {
    float* o = reinterpret_cast<float*>(p.out) + ooff;
    if (p.peer_world > 1) {
      // an 8-column group crosses at most one shard boundary (shards are multiples of 2048 elements)
      const long long e0 = p.peer_off + (long long)ooff;
      const int own0 = (int)min((long long)(p.peer_world - 1), e0 / p.peer_per);
      const long long bound = own0 + 1 < p.peer_world ? (long long)(own0 + 1) * p.peer_per : (1ll << 62);
#pragma unroll
      for (int j = 0; j < 8; j += 4) {
        const int owner = (e0 + j >= bound) ? own0 + 1 : own0;
        if (!p.peer_push || owner == p.peer_rank) {
          asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(o + j), "f"(f[j]),
                       "f"(f[j + 1]), "f"(f[j + 2]), "f"(f[j + 3]) : "memory");
        } else {
          float4 v = make_float4(f[j], f[j + 1], f[j + 2], f[j + 3]);
          if (add_local) {                       // what the earlier micro-steps accumulated here
            const float4 cur = *reinterpret_cast<const float4*>(o + j);
            v.x += cur.x; v.y += cur.y; v.z += cur.z; v.w += cur.w;
          }
          float* dst = p.peer_base[owner] + (e0 + j);
          asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(v.x), "f"(v.y),
                       "f"(v.z), "f"(v.w) : "memory");
        }
      }
      return;
    }
    // fire-and-forget reduction at the L2 (one contributor per element and launch unless split-K)
#pragma unroll
    for (int j = 0; j < 8; j += 4)
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(o + j), "f"(f[j]), "f"(f[j + 1]),
                   "f"(f[j + 2]), "f"(f[j + 3]) : "memory");
    return;
  }
  if constexpr (E == EPI_F32) {
    float* o = reinterpret_cast<float*>(p.out) + ooff;
    *reinterpret_cast<float4*>(o) = make_float4(f[0], f[1], f[2], f[3]);
    *reinterpret_cast<float4*>(o + 4) = make_float4(f[4], f[5], f[6], f[7]);
    return;
  }
  uint32_t bias[4] = {0, 0, 0, 0}, ow[4], aux[4];
  const uint32_t none[4] = {0, 0, 0, 0};
  if constexpr (epilogue_spec(E).bias) {
    if (p.bias != nullptr) {
      const uint4 b = __ldg(reinterpret_cast<const uint4*>(p.bias + n0));
      bias[0] = b.x; bias[1] = b.y; bias[2] = b.z; bias[3] = b.w;
    }
  }
  epilogue_math<E, 8>(p, f, bias, 0, none, ow, aux);
  *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + ooff) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
  if constexpr (epilogue_spec(E).aux)
    *reinterpret_cast<uint4*>(p.aux_out + ooff) = make_uint4(aux[0], aux[1], aux[2], aux[3]);
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const float2 v = unpack_bf16(ow[t]);
    f[2 * t] = v.x;
    f[2 * t + 1] = v.y;
  }
}

// Accumulator values of 8 output columns of one row after the quad regrouping: 32-column chunk i of the fragment,
// row half h, as alpha * acc.  __fmul_rn: alpha * acc is rounded to fp32 before the bias or residual add that follows,
// so that add is never contracted into an fma.  The outputs are defined with that rounding.
__device__ __forceinline__ void regroup8(float (&f)[8], const uint32_t (&lo_in)[4], const uint32_t (&hi_in)[4],
                                         float alpha) {
  uint32_t lo[4] = {lo_in[0], lo_in[1], lo_in[2], lo_in[3]}, hi[4] = {hi_in[0], hi_in[1], hi_in[2], hi_in[3]};
  quad_transpose(lo);
  quad_transpose(hi);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    f[2 * k] = __fmul_rn(__uint_as_float(lo[k]), alpha);
    f[2 * k + 1] = __fmul_rn(__uint_as_float(hi[k]), alpha);
  }
}

// Register epilogue of one warpgroup's 64 x NCOLS accumulator fragment: output rows [row64, row64 + 64), columns from
// col0.
template <int NCOLS, int E>
__device__ __forceinline__ void fragment_epilogue(const GemmArgs& p, float (&acc)[NCOLS / 2], int row64, int col0,
                                                  float alpha, bool add_local) {
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  const int c = lane & 3;
  const int row_base = row64 + warp * 16 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < NCOLS / 32; ++i) {           // unrolled: the accumulator must stay in registers
    const int n0 = col0 + i * 32 + c * 8;                    // after the regrouping this lane owns columns [n0, n0 + 8)
    if (col0 + i * 32 >= p.N) break;                         // warp uniform
    float cs[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) cs[t] = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint32_t lo[4], hi[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        lo[k] = __float_as_uint(acc[(i * 4 + k) * 4 + 2 * h]);
        hi[k] = __float_as_uint(acc[(i * 4 + k) * 4 + 2 * h + 1]);
      }
      float f[8];
      regroup8(f, lo, hi, alpha);
      const int row = row_base + h * 8;
      if (row < p.M && n0 < p.N) {
        epilogue_group<E>(p, f, row, n0, add_local);
#pragma unroll
        for (int t = 0; t < 8; ++t) cs[t] += f[t];
      }
    }
    if constexpr (epilogue_spec(E).colsum) {
      if (p.colsum != nullptr) {                 // bias gradients: rows of this warp, then one atomic per column
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          cs[t] += __shfl_xor_sync(0xffffffffu, cs[t], 4);
          cs[t] += __shfl_xor_sync(0xffffffffu, cs[t], 8);
          cs[t] += __shfl_xor_sync(0xffffffffu, cs[t], 16);
        }
        if (lane < 4 && n0 < p.N) {
#pragma unroll
          for (int t = 0; t < 8; ++t) atomicAdd(p.colsum + n0 + t, cs[t]);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// bf16-output epilogue through shared memory.  Each consumer warpgroup owns two 8 KB staging buffers, each one 64 x 64
// bf16 subtile with 128-byte rows in the SWIZZLE_128B layout of a [64][64] tensor-map box.  Per subtile the warpgroup
// converts its accumulator fragment, reads its residual / saved factor from the buffer (loaded by TMA, ahead of use),
// writes the output to the same addresses, and one thread stores the buffer with a TMA bulk store.  TMA clips the
// ragged M / N edges, so nothing outside the [M, N] window is written.
// ---------------------------------------------------------------------------------------------------------------------
// Which epilogues stage their output.  The plain store (EPI_NONE) and bias + GELU + GELU' (EPI_BIAS_GELU_DG) read no
// [M, N] input and measured faster on H100 with their stores issued straight from registers; the fp32 outputs are
// reductions or plain stores that need no staging.
__host__ __device__ constexpr bool staged_epi(int E) { return !epilogue_spec(E).f32_out && E != EPI_NONE && E != EPI_BIAS_GELU_DG; }

constexpr int SUB_BYTES = 64 * 128;
constexpr int STAGE_BUFS = 2;                   // per consumer warpgroup

// byte offset of 16-byte chunk `chunk` (0..7) of row `row` in a swizzled subtile
__device__ __forceinline__ uint32_t sw128(int row, int chunk) { return row * 128 + ((chunk ^ (row & 7)) << 4); }

// the 128 threads of consumer warpgroup cw (named barriers 1 and 2 are the ping-pong turn barriers).  Not the .aligned
// form (bar.sync): the thread that issues the bulk copies reaches it from its own branch and mbarrier wait loop.
__device__ __forceinline__ void wg_sync(int cw) { asm volatile("barrier.sync %0, 128;" ::"r"(3 + cw) : "memory"); }

// Where a warpgroup's bf16 epilogue runs in a unit: its `nsub` 64-column subtiles hold output columns and its `rlive`
// 64-row fragments hold output rows.  Subtile t = s * rlive + r uses staging buffer (q + t) & 1, where q counts the
// subtiles the warpgroup staged in its earlier units.
struct StagedUnit {
  int row64, col0, nsub, rlive;
  uint32_t q;
  __device__ int count() const { return nsub * rlive; }
};

template <int BLOCK_N, int R>
__device__ __forceinline__ StagedUnit staged_unit(const GemmArgs& p, int row64, int nb, uint32_t q) {
  StagedUnit su;
  su.row64 = row64;
  su.col0 = nb * BLOCK_N;
  su.nsub = (min(BLOCK_N, p.N - su.col0) + 63) / 64;
  const int rows_left = p.M - row64;
  su.rlive = rows_left <= 0 ? 0 : (R == 2 && rows_left > 64 ? 2 : 1);
  su.q = q;
  return su;
}

// staging buffers and their load barriers (one per buffer) of consumer warpgroup cw
template <int BLOCK_N>
__device__ __forceinline__ uint8_t* staging(uint8_t* smem, int cw) {
  return smem + Cfg<BLOCK_N>::STAGES * Cfg<BLOCK_N>::STAGE_BYTES + cw * STAGE_BUFS * SUB_BYTES;
}
template <int BLOCK_N>
__device__ __forceinline__ uint64_t* in_bars(uint8_t* smem, int cw) {
  return reinterpret_cast<uint64_t*>(staging<BLOCK_N>(smem, 2)) + 2 * Cfg<BLOCK_N>::STAGES + cw * STAGE_BUFS;
}

// bias slice of consumer warpgroup cw's unit, after the barriers
template <int BLOCK_N>
__device__ __forceinline__ uint32_t bias_slice(uint8_t* smem, int cw) {
  return smem_u32(staging<BLOCK_N>(smem, 2) + 256) + cw * BLOCK_N * 2;
}

// TMA load of the residual / saved factor of subtile t = s * rlive + r into its staging buffer
__device__ __forceinline__ void load_input(const CUtensorMap* tm_res, uint8_t* buf, uint64_t* in_bar,
                                           const StagedUnit& su, int t, int s, int r) {
  const uint32_t b = (su.q + t) & 1;
  mbar_arrive_expect_tx(&in_bar[b], SUB_BYTES);
  tma_load_2d(buf + b * SUB_BYTES, tm_res, &in_bar[b], su.col0 + s * 64, su.row64 + r * 64);
}

template <int BLOCK_N, int R, int E>
__device__ __forceinline__ void staged_epilogue(const GemmArgs& p, float (&acc)[R][BLOCK_N / 2], const CUtensorMap* tm_out,
                                                const CUtensorMap* tm_res, uint8_t* smem,
                                                const StagedUnit& su, int cw, float alpha, unsigned long long seed,
                                                const uint32_t (&kwords)[R][2][BLOCK_N / 128]) {
  constexpr EpilogueSpec SP = epilogue_spec(E);
  int tid = threadIdx.x & 127;
  asm volatile("" : "+r"(tid));    // derived addresses are recomputed per unit, not held across the main loop
  const int lane = tid & 31, warp = tid >> 5, c = lane & 3;
  const bool issuer = tid == 0;
  const bool has_in = (SP.res || E == EPI_ADD) && p.res != nullptr;   // residual or saved factor, loaded by TMA
  uint8_t* buf = staging<BLOCK_N>(smem, cw);
  uint64_t* in_bar = in_bars<BLOCK_N>(smem, cw);
  const uint32_t buf_s = smem_u32(buf);
  const int n_staged = su.count();
  const uint32_t bias_s = bias_slice<BLOCK_N>(smem, cw);
  if constexpr (SP.bias) {                       // the unit's bias slice, copied in before the main loop
    if (p.bias != nullptr) {
      asm volatile("cp.async.wait_all;" ::: "memory");
      wg_sync(cw);
    }
  }
#pragma unroll
  for (int s = 0; s < BLOCK_N / 64; ++s) {
    if (s >= su.nsub) break;                                   // warpgroup uniform
    float cs[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (r >= su.rlive) break;                                // warpgroup uniform
      const int t = s * su.rlive + r;
      const uint32_t b = (su.q + t) & 1;
      const uint32_t sub = buf_s + b * SUB_BYTES;
      if (has_in) mbar_wait_mma(&in_bar[b], ((su.q + t) >> 1) & 1);
      // The accumulator is used in its wgmma layout: this lane owns columns 8 j + 2 c, + 1 of each 8-column group j,
      // rows rr and rr + 8.  Its 4-byte reads and writes of a row's group sit in 16-byte chunk j, which the swizzle
      // spreads over the 8 rows of the warp: no bank conflicts.
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int rr = warp * 16 + (lane >> 2) + h * 8;        // row inside the subtile
        const int row = su.row64 + r * 64 + rr;
        // keep bits drawn here (no mask_in): lane c draws groups c and 4 + c of the row, one Philox evaluation per
        // group as before, and the quad shares the bytes
        uint32_t kq[2] = {0, 0};
        if constexpr (SP.keep_bits) {
          if (p.drop_thresh16 != 0 && p.mask_in == nullptr) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int n0 = su.col0 + s * 64 + (4 * e + c) * 8;
              const Keep8 keep =
                  dropout_keep8(seed, p.stream, ((uint64_t)row * (uint64_t)p.N + (uint64_t)n0) >> 3, p.drop_thresh16);
#pragma unroll
              for (int t = 0; t < 8; ++t) kq[e] |= (keep[t] ? 1u : 0u) << t;
              if (p.mask_out != nullptr && row < p.M && n0 < p.N)
                p.mask_out[(size_t)row * (size_t)(p.N >> 3) + (size_t)(n0 >> 3)] = (unsigned char)kq[e];
            }
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int jb = s * 8 + j;                            // 8-column group of the fragment
          float f[2] = {__fmul_rn(acc[r][jb * 4 + 2 * h], alpha), __fmul_rn(acc[r][jb * 4 + 2 * h + 1], alpha)};
          const uint32_t addr = sub + sw128(rr, j) + c * 4;
          uint32_t res[1] = {0}, bias[1] = {0}, out[1], aux[1];
          if (has_in) asm volatile("ld.shared.b32 %0, [%1];" : "=r"(res[0]) : "r"(addr) : "memory");
          if constexpr (SP.bias)
            if (p.bias != nullptr)
              asm volatile("ld.shared.b32 %0, [%1];" : "=r"(bias[0]) : "r"(bias_s + (jb * 8 + c * 2) * 2) : "memory");
          uint32_t kb = 0;
          if constexpr (SP.keep_bits) {
            if (p.drop_thresh16 != 0) {
              // keep byte of group jb: from mask_in, byte jb % 16 of the row's 16 bytes of 128-column chunk jb / 16,
              // held in word (jb % 16) / 4 by that quad lane; or drawn above by lane j % 4
              const uint32_t byte =
                  p.mask_in != nullptr
                      ? __shfl_sync(0xffffffffu, kwords[r][h][jb >> 4], (lane & ~3) | ((jb & 15) >> 2)) >> (8 * (jb & 3))
                      : __shfl_sync(0xffffffffu, kq[j >> 2], (lane & ~3) | (j & 3));
              kb = (byte >> (2 * c)) & 3u;
            }
          }
          epilogue_math<E, 2>(p, f, bias, kb, res, out, aux);
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(out[0]) : "memory");
        }
      }
      fence_proxy_async();                                     // the generic-proxy writes -> the TMA store
      if (issuer) tma_store_wait_read<0>();                    // the other buffer is free once this barrier is passed
      wg_sync(cw);
      if (issuer) {
        tma_store_2d(tm_out, buf + b * SUB_BYTES, su.col0 + s * 64, su.row64 + r * 64);
        tma_store_commit();
      }
      if constexpr (SP.colsum) {
        if (p.colsum != nullptr) {
          // column pair cp of the subtile, rows 16 qd .. 16 qd + 15 in a rotated order (conflict-free reads)
          int l2 = lane;
          asm volatile("" : "+r"(l2));
          const int cp = warp * 8 + (l2 & 7), qd = l2 >> 3;
#pragma unroll 1
          for (int j = 0; j < 16; ++j) {
            const int rs = 16 * qd + ((j + 2 * qd) & 15);
            uint32_t v;
            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(sub + sw128(rs, cp >> 2) + (cp & 3) * 4) : "memory");
            if (su.row64 + r * 64 + rs < p.M) {
              const float2 x = unpack_bf16(v);
              cs[0] += x.x;
              cs[1] += x.y;
            }
          }
          if (has_in) wg_sync(cw);                             // every read of the buffer is done before it is reloaded
        }
      }
      if (has_in && issuer && t + 2 < n_staged) {
        tma_store_wait_read<0>();
        if (su.rlive == 2) load_input(tm_res, buf, in_bar, su, t + 2, s + 1, r);
        else load_input(tm_res, buf, in_bar, su, t + 2, s + 2, 0);
      }
    }
    if constexpr (SP.colsum) {
      if (p.colsum != nullptr) {                 // bias gradients: one atomic per column, subtile and warpgroup
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          cs[e] += __shfl_xor_sync(0xffffffffu, cs[e], 8);
          cs[e] += __shfl_xor_sync(0xffffffffu, cs[e], 16);
        }
        const int n = su.col0 + s * 64 + 2 * (warp * 8 + (lane & 7));
        if (lane < 8 && n < p.N) {
          atomicAdd(p.colsum + n, cs[0]);
          atomicAdd(p.colsum + n + 1, cs[1]);
        }
      }
    }
  }
}

// The consumer warpgroup `cw` (0 or 1) over this CTA's units.  Ping-pong (BLOCK_N 128): warpgroup cw takes the
// CTA's units j = cw, cw + 2, ...; it waits on named barrier 1 + cw for its turn to issue MMAs and, if the other
// warpgroup has a next unit, hands the turn over on barrier 2 - cw once its own MMAs are issued.  The order also keeps
// a warpgroup from running more than one ring phase ahead of the producer.
template <bool A_MN, bool B_MN, int BLOCK_N, bool FP8, int AE5, int BE5, int E>
__device__ __forceinline__ void consumer(const GemmArgs& p, const CUtensorMap* tm_out, const CUtensorMap* tm_res,
                                         uint8_t* smem, uint64_t* full_bar,
                                         uint64_t* empty_bar, int cw) {
  constexpr bool PINGPONG = BLOCK_N == 128;
  constexpr int R = PINGPONG ? 2 : 1;            // 64-row accumulator fragments per warpgroup
  constexpr EpilogueSpec SP = epilogue_spec(E);
  float acc[R][BLOCK_N / 2];                     // the first MMA of a unit overwrites it (scale-d = 0)
  float alpha = p.alpha;
  if constexpr (FP8) alpha *= __ldg(p.scale_a) * __ldg(p.scale_b);   // per-tensor dequantisation
  const unsigned long long seed = p.drop_thresh16 != 0 ? p.seed.value() : 0ull;
  const bool issuer = (threadIdx.x & 127) == 0;  // issues this warpgroup's TMA loads and stores
  uint32_t q = 0;                                // subtiles this warpgroup has staged
  if (PINGPONG && cw == 1) asm volatile("bar.arrive 1, 256;" ::: "memory");   // warpgroup 0 goes first
  uint32_t it = 0;                               // ring position of the unit: k-blocks of this CTA's earlier units
  int j = 0;
  for (int u = blockIdx.x; u < p.units; u += gridDim.x, ++j) {
    const Unit w = unit_of(p, u);
    if (PINGPONG && (j & 1) != cw) {
      it += w.nkb;
      continue;
    }
    if (PINGPONG) asm volatile("bar.sync %0, 256;" ::"r"(1 + cw) : "memory");
    TL(UnitStamps st{}; st.start = clock64();)
    const int row64 = w.mb * BLOCK_M + (PINGPONG ? 0 : cw * 64);
    if constexpr (staged_epi(E)) {
      if (issuer && p.res != nullptr && (SP.res || E == EPI_ADD)) {   // the first two subtiles land under the MMAs
        const StagedUnit su = staged_unit<BLOCK_N, R>(p, row64, w.nb, q);
        tma_store_wait_read<0>();
        uint8_t* buf = staging<BLOCK_N>(smem, cw);
        uint64_t* in_bar = in_bars<BLOCK_N>(smem, cw);
        if (su.count() > 0) load_input(tm_res, buf, in_bar, su, 0, 0, 0);
        if (su.count() > 1) load_input(tm_res, buf, in_bar, su, 1, su.rlive == 2 ? 0 : 1, su.rlive == 2 ? 1 : 0);
      }
    }
    // the unit's bias slice goes to shared memory and its mask_in keep bytes to registers while the MMAs run: for each
    // of the thread's rows and 128-column chunks, word c of the row's 16 keep bytes (the quad shares them)
    uint32_t kwords[R][2][BLOCK_N / 128];
    if constexpr (staged_epi(E)) {
      const int tid = threadIdx.x & 127;
      if constexpr (SP.bias) {
        const int n = w.nb * BLOCK_N + tid * 2;
        if (p.bias != nullptr && tid < BLOCK_N / 2)
          asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(bias_slice<BLOCK_N>(smem, cw) + tid * 4),
                       "l"(p.bias + (n < p.N ? n : 0)), "r"(n < p.N ? 4 : 0) : "memory");
      }
      if constexpr (SP.keep_bits) {
        if (p.drop_thresh16 != 0 && p.mask_in != nullptr) {
#pragma unroll
          for (int r = 0; r < R; ++r)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = row64 + r * 64 + (tid >> 5) * 16 + ((tid & 31) >> 2) + h * 8;
#pragma unroll
              for (int x = 0; x < BLOCK_N / 128; ++x) {
                const int n = w.nb * BLOCK_N + x * 128;
                kwords[r][h][x] =
                    row < p.M && n < p.N
                        ? __ldg(reinterpret_cast<const uint32_t*>(p.mask_in + (size_t)row * (p.N >> 3) + (n >> 3)) + (tid & 3))
                        : 0u;
              }
            }
        }
      }
    }
    const int arrive_bar = PINGPONG && u + (int)gridDim.x < p.units ? 2 - cw : -1;
    consumer_mainloop<A_MN, B_MN, BLOCK_N, R, FP8, AE5, BE5>(acc, smem, full_bar, empty_bar, PINGPONG ? 0 : cw, it,
                                                            w.nkb, arrive_bar TL(, st));
    it += w.nkb;
    if constexpr (!staged_epi(E)) {
#pragma unroll
      for (int r = 0; r < R; ++r)
        fragment_epilogue<BLOCK_N, E>(p, acc[r], row64 + r * 64, w.nb * BLOCK_N, alpha, w.ks == 0);
    } else {
      const StagedUnit su = staged_unit<BLOCK_N, R>(p, row64, w.nb, q);
      staged_epilogue<BLOCK_N, R, E>(p, acc, tm_out, tm_res, smem, su, cw, alpha, seed, kwords);
      q += su.count();
    }
#ifdef B200_GEMM_TIMELINE
    st.epi_done = clock64();
    if (p.timeline != nullptr && (threadIdx.x & 127) == 0) {
      long long* rec = p.timeline + (size_t)u * TL_STRIDE + cw * 6;
      rec[0] = st.start; rec[1] = st.full0; rec[2] = st.last_mma; rec[3] = st.wait0; rec[4] = st.epi_done;
      rec[5] = st.op_wait;
    }
#endif
  }
  if (staged_epi(E) && issuer) tma_store_wait<0>();   // the bulk stores have read the staging buffers before exit
}

// E: the epilogue (GemmEpilogue), see epilogue_group
template <bool A_MN, bool B_MN, int BLOCK_N, bool FP8, int E>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
            const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_res,
            const GemmArgs p) {
  using C = Cfg<BLOCK_N>;
  static_assert(!FP8 || (!A_MN && !B_MN), "fp8 wgmma reads K-major operands only");
  constexpr bool STAGED = staged_epi(E);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // operand ring, then (bf16 epilogues) the staging subtiles, then full_bar, empty_bar and in_bar
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging<BLOCK_N>(smem, 0) + (STAGED ? 2 * STAGE_BUFS * SUB_BYTES : 0));
  uint64_t* empty_bar = full_bar + C::STAGES;
  uint64_t* in_bar = in_bars<BLOCK_N>(smem, 0);

  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], BLOCK_N == 128 ? 4 : 8);   // one arrival per warp of the warpgroup(s) reading the slot
    }
    if (STAGED)
      for (int b = 0; b < 2 * STAGE_BUFS; ++b) mbar_init(&in_bar[b], 1);
    fence_barrier_init();
  }
  __syncthreads();
  constexpr int BK = FP8 ? 128 : 64;             // elements along K per stage

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
        const Unit w = unit_of(p, u);
        TL(long long blocked = 0;)
        for (int kb = w.kb0; kb < w.kb0 + w.nkb; ++kb) {
          TL(const long long t = clock64();)
          mbar_wait_mma(&empty_bar[s], ph ^ 1);
          TL(blocked += clock64() - t;)
          uint8_t* sa = smem + s * C::STAGE_BYTES;
          uint8_t* sb = sa + C::A_BYTES;
          mbar_arrive_expect_tx(&full_bar[s], C::STAGE_BYTES);
          if constexpr (!A_MN) {
            tma_load_2d(sa, &tmap_a, &full_bar[s], kb * BK, w.mb * BLOCK_M);
          } else {
#pragma unroll
            for (int j = 0; j < BLOCK_M / 64; ++j)
              tma_load_2d(sa + j * 8192, &tmap_a, &full_bar[s], w.mb * BLOCK_M + j * 64, kb * BK);
          }
          if constexpr (!B_MN) {
            tma_load_2d(sb, &tmap_b, &full_bar[s], kb * BK, w.nb * BLOCK_N);
          } else {
#pragma unroll
            for (int j = 0; j < BLOCK_N / 64; ++j)
              tma_load_2d(sb + j * 8192, &tmap_b, &full_bar[s], w.nb * BLOCK_N + j * 64, kb * BK);
          }
          if (++s == C::STAGES) { s = 0; ph ^= 1; }
        }
#ifdef B200_GEMM_TIMELINE
        if (p.timeline != nullptr) {
          p.timeline[(size_t)u * TL_STRIDE + 12] = blocked;
          p.timeline[(size_t)u * TL_STRIDE + 13] = gridDim.x;
        }
#endif
      }
    }
    return;
  }
  // -------------------------------------------------------------------- MMA + epilogue (two warpgroups)
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int cw = wg - 1;
  if constexpr (FP8) {
    switch (p.fp8_fmt & 3u) {
      case 0: consumer<A_MN, B_MN, BLOCK_N, true, 0, 0, E>(p, &tmap_out, &tmap_res, smem, full_bar, empty_bar, cw); break;
      case 1: consumer<A_MN, B_MN, BLOCK_N, true, 1, 0, E>(p, &tmap_out, &tmap_res, smem, full_bar, empty_bar, cw); break;
      case 2: consumer<A_MN, B_MN, BLOCK_N, true, 0, 1, E>(p, &tmap_out, &tmap_res, smem, full_bar, empty_bar, cw); break;
      default: consumer<A_MN, B_MN, BLOCK_N, true, 1, 1, E>(p, &tmap_out, &tmap_res, smem, full_bar, empty_bar, cw); break;
    }
  } else {
    consumer<A_MN, B_MN, BLOCK_N, false, 0, 0, E>(p, &tmap_out, &tmap_res, smem, full_bar, empty_bar, cw);
  }
}

// [R][ld_in] bytes -> [C][ld_out] bytes (fp8 operand transposition: MN-major -> K-major)
__global__ void __launch_bounds__(256) fp8_transpose_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                                                            int R, int Cn, long long ld_in, long long ld_out) {
  __shared__ uint8_t t[64][65];
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  for (int i = threadIdx.x; i < 64 * 64; i += 256) {
    const int r = i >> 6, c = i & 63;
    t[r][c] = (r0 + r < R && c0 + c < Cn) ? in[(long long)(r0 + r) * ld_in + c0 + c] : (uint8_t)0;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 64 * 64; i += 256) {
    const int c = i >> 6, r = i & 63;
    if (c0 + c < Cn && r0 + r < R) out[(long long)(c0 + c) * ld_out + r0 + r] = t[r][c];
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || f == nullptr) {
      fprintf(stderr, "[b200] cuTensorMapEncodeTiled is unavailable (%s)\n", cudaGetErrorString(e));
      abort();
    }
    fn = reinterpret_cast<EncodeTiledFn>(f);
  });
  return fn;
}

// 2D bf16 tensor map: `inner` contiguous elements per row, `outer` rows, row pitch `ld` elements,
// box = [box_outer][box_inner], 128B swizzle (box_inner must be 64 bf16).
static CUtensorMap make_tmap_2d(const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                                uint32_t box_outer, uint32_t esize);

CUtensorMap make_tmap_2d_bf16(const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                              uint32_t box_outer) {
  return make_tmap_2d(ptr, inner, outer, ld, box_inner, box_outer, 2);
}

// `esize` 2: bf16 (box_inner 64), 1: fp8 bytes (box_inner 128)
static CUtensorMap make_tmap_2d(const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                                uint32_t box_outer, uint32_t esize) {
  struct Key {
    const void* p; uint64_t i, o, l; uint32_t bi, bo, es;
    bool operator==(const Key& k) const {
      return p == k.p && i == k.i && o == k.o && l == k.l && bi == k.bi && bo == k.bo && es == k.es;
    }
  };
  struct Hash {
    size_t operator()(const Key& k) const {
      size_t h = reinterpret_cast<size_t>(k.p);
      h = h * 1000003u ^ k.i; h = h * 1000003u ^ k.o; h = h * 1000003u ^ k.l; h = h * 1000003u ^ k.bi;
      h = h * 1000003u ^ k.es;
      return h * 1000003u ^ k.bo;
    }
  };
  static std::unordered_map<Key, CUtensorMap, Hash> cache;
  static std::mutex mu;
  Key key{ptr, inner, outer, ld, box_inner, box_outer, esize};
  std::lock_guard<std::mutex> lock(mu);
  auto itf = cache.find(key);
  if (itf != cache.end()) return itf->second;
  CUtensorMap m;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld * esize};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode_fn()(&m, esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box,
                               estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[b200] cuTensorMapEncodeTiled failed (%d): ptr=%p inner=%llu outer=%llu ld=%llu box=%ux%u\n",
            (int)r, ptr, (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)ld, box_inner,
            box_outer);
    abort();
  }
  if (cache.size() > 4096) cache.clear();
  cache.emplace(key, m);
  return m;
}

CUtensorMap make_tmap_2d_u8(const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                            uint32_t box_outer) {
  return make_tmap_2d(ptr, inner, outer, ld, box_inner, box_outer, 1);
}


static long long* g_timeline = nullptr;
static long long g_timeline_units = 0;

bool gemm_set_timeline(long long* buf, long long units) {
  g_timeline = buf;
  g_timeline_units = buf != nullptr ? units : 0;
#ifdef B200_GEMM_TIMELINE
  return true;
#else
  return false;
#endif
}

template <bool A_MN, bool B_MN, int BLOCK_N, bool FP8, int E>
static void launch(const GemmCall& c, cudaStream_t st) {
  using C = Cfg<BLOCK_N>;
  constexpr int BK = FP8 ? 128 : 64;
  GemmArgs p;
  p.M = c.M; p.N = c.N; p.K = c.K;
  p.m_blocks = (c.M + BLOCK_M - 1) / BLOCK_M;
  p.n_blocks = (c.N + BLOCK_N - 1) / BLOCK_N;
  p.k_blocks = (c.K + BK - 1) / BK;
  if (p.m_blocks <= 0 || p.n_blocks <= 0 || p.k_blocks <= 0) return;
  int splits = E == EPI_ACCUM_F32 ? c.k_splits : 1;           // only the reducing epilogue can merge K ranges
  if (splits < 0) {                                            // automatic: fill the machine, >= 4 k-blocks per CTA
    splits = num_sms() / (p.m_blocks * p.n_blocks);
    if (splits > p.k_blocks / 4) splits = p.k_blocks / 4;
  }
  p.k_splits = splits < 1 ? 1 : splits;
  if (p.k_splits > p.k_blocks) p.k_splits = p.k_blocks;
  p.k_per_split = (p.k_blocks + p.k_splits - 1) / p.k_splits;
  p.k_splits = (p.k_blocks + p.k_per_split - 1) / p.k_per_split;   // no empty splits
  p.out = c.out; p.ldo = c.ldo; p.aux_out = reinterpret_cast<__nv_bfloat16*>(c.aux_out);
  p.bias = reinterpret_cast<const __nv_bfloat16*>(c.bias);
  p.res = reinterpret_cast<const __nv_bfloat16*>(c.res); p.ldr = c.ldr;
  p.colsum = c.colsum; p.mask_out = c.mask_out; p.mask_in = c.mask_in;
  p.seed = Seed{c.seed, c.seed_step}; p.stream = c.stream;
  const float pd = c.p_drop;
  p.drop_thresh16 = pd > 0.f ? (unsigned)(pd * 65536.f + 0.5f) : 0u;
  p.drop_scale = pd > 0.f ? 65536.f / (65536.f - (float)p.drop_thresh16) : 1.f;
  p.alpha = c.alpha;
  p.peer_world = c.peer_world; p.peer_rank = c.peer_rank; p.peer_push = c.peer_push;
  p.peer_off = c.peer_off; p.peer_per = c.peer_per;
  for (int i = 0; i < 16; ++i) p.peer_base[i] = i < c.peer_world ? c.peer_base[i] : nullptr;
  p.scale_a = c.scale_a; p.scale_b = c.scale_b;
  p.fp8_fmt = (c.a_e5m2 ? 1u : 0u) | (c.b_e5m2 ? 2u : 0u);
  constexpr uint32_t ES = FP8 ? 1 : 2;
  CUtensorMap ta = A_MN ? make_tmap_2d(c.A, c.M, c.K, c.lda, 64, BK, ES)
                        : make_tmap_2d(c.A, c.K, c.M, c.lda, BK, 64 * 2, ES);
  CUtensorMap tb = B_MN ? make_tmap_2d(c.B, c.N, c.K, c.ldb, 64, BK, ES)
                        : make_tmap_2d(c.B, c.K, c.N, c.ldb, BK, BLOCK_N, ES);
  // out and res of the bf16 epilogues: box [64][64], dims [M, N] and the tensor's own row stride, so TMA clips the
  // ragged edges and never touches a column past N of a wider tensor
  constexpr bool STAGED = staged_epi(E);
  const CUtensorMap to = STAGED ? make_tmap_2d(c.out, c.N, c.M, c.ldo, 64, 64, 2) : ta;
  const CUtensorMap tres = STAGED && c.res != nullptr ? make_tmap_2d(c.res, c.N, c.M, c.ldr, 64, 64, 2) : to;
  constexpr int SMEM = STAGED ? C::SMEM_STAGED : C::SMEM_TOTAL;
  auto kern = gemm_kernel<A_MN, B_MN, BLOCK_N, FP8, E>;
  static bool configured = false;
  if (!configured) {
    B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    configured = true;
  }
  p.units = p.m_blocks * p.n_blocks * p.k_splits;
#ifdef B200_GEMM_TIMELINE
  p.timeline = p.units <= g_timeline_units ? g_timeline : nullptr;
#endif
  const int grid = p.units < num_sms() ? p.units : num_sms();       // persistent: one CTA per SM walks the units
  kern<<<grid, NUM_THREADS, SMEM, st>>>(ta, tb, to, tres, p);
}

// fp8: bring an MN-major operand ([K][ld], the M or N index contiguous) into the K-major form [MN][Kp]
static const void* fp8_k_major(const void* src, int mn, int K, int ld, int* ld_out, cudaStream_t st) {
  const int Kp = (K + 15) & ~15;                // TMA row pitch: multiple of 16 bytes
  void* buf = nullptr;
  B200_CUDA_CHECK(cudaMallocAsync(&buf, (size_t)mn * Kp, st));
  fp8_transpose_kernel<<<dim3((mn + 63) / 64, (K + 63) / 64), 256, 0, st>>>((const uint8_t*)src, (uint8_t*)buf, K, mn, ld, Kp);
  *ld_out = Kp;
  return buf;
}

typedef void (*LaunchFn)(const GemmCall&, cudaStream_t);

// 128 x 256 tiles (wide) or 128 x 128
template <bool A_MN, bool B_MN, bool FP8, int E>
static LaunchFn tile_width(bool wide) {
  return wide ? launch<A_MN, B_MN, 256, FP8, E> : launch<A_MN, B_MN, 128, FP8, E>;
}

// Operand forms: GEMM_NT, GEMM_NN and GEMM_TN with bf16 operands, and FORM_FP8: fp8 operands in any layout, which run
// in the NT form once their MN-major operands are transposed.
constexpr int FORM_FP8 = 3;
constexpr int form_epi(int form, int epi) { return form * 16 + epi; }

// Every (operand form, epilogue) pair that is built: the pairs the engine, the K-FAC factors, the pretraining and
// fine-tuning heads, tools/ and the tests call.  nullptr for any other pair.
static LaunchFn kernel_for(int form, int epi, bool wide) {
  constexpr bool K_MAJOR = false, MN_MAJOR = true;
  switch (form_epi(form, epi)) {
    case form_epi(GEMM_NT, EPI_NONE): return tile_width<K_MAJOR, K_MAJOR, false, EPI_NONE>(wide);
    case form_epi(GEMM_NT, EPI_BIAS): return tile_width<K_MAJOR, K_MAJOR, false, EPI_BIAS>(wide);
    case form_epi(GEMM_NT, EPI_BIAS_DROP_RES): return tile_width<K_MAJOR, K_MAJOR, false, EPI_BIAS_DROP_RES>(wide);
    case form_epi(GEMM_NT, EPI_ADD): return tile_width<K_MAJOR, K_MAJOR, false, EPI_ADD>(wide);
    case form_epi(GEMM_NT, EPI_MUL): return tile_width<K_MAJOR, K_MAJOR, false, EPI_MUL>(wide);
    case form_epi(GEMM_NT, EPI_BIAS_GELU_DG): return tile_width<K_MAJOR, K_MAJOR, false, EPI_BIAS_GELU_DG>(wide);
    case form_epi(GEMM_NT, EPI_BIAS_TANH): return tile_width<K_MAJOR, K_MAJOR, false, EPI_BIAS_TANH>(wide);
    case form_epi(GEMM_NT, EPI_F32): return tile_width<K_MAJOR, K_MAJOR, false, EPI_F32>(wide);
    case form_epi(GEMM_NN, EPI_NONE): return tile_width<K_MAJOR, MN_MAJOR, false, EPI_NONE>(wide);
    case form_epi(GEMM_NN, EPI_ADD): return tile_width<K_MAJOR, MN_MAJOR, false, EPI_ADD>(wide);
    case form_epi(GEMM_NN, EPI_MUL): return tile_width<K_MAJOR, MN_MAJOR, false, EPI_MUL>(wide);
    case form_epi(GEMM_TN, EPI_ACCUM_F32): return tile_width<MN_MAJOR, MN_MAJOR, false, EPI_ACCUM_F32>(wide);
    case form_epi(GEMM_TN, EPI_F32): return tile_width<MN_MAJOR, MN_MAJOR, false, EPI_F32>(wide);
    case form_epi(FORM_FP8, EPI_NONE): return tile_width<K_MAJOR, K_MAJOR, true, EPI_NONE>(wide);
    case form_epi(FORM_FP8, EPI_BIAS): return tile_width<K_MAJOR, K_MAJOR, true, EPI_BIAS>(wide);
    case form_epi(FORM_FP8, EPI_BIAS_DROP_RES): return tile_width<K_MAJOR, K_MAJOR, true, EPI_BIAS_DROP_RES>(wide);
    case form_epi(FORM_FP8, EPI_ADD): return tile_width<K_MAJOR, K_MAJOR, true, EPI_ADD>(wide);
    case form_epi(FORM_FP8, EPI_ACCUM_F32): return tile_width<K_MAJOR, K_MAJOR, true, EPI_ACCUM_F32>(wide);
    case form_epi(FORM_FP8, EPI_F32): return tile_width<K_MAJOR, K_MAJOR, true, EPI_F32>(wide);
    default: return nullptr;
  }
}

bool gemm_bf16(const GemmCall& c, cudaStream_t st) {
  if (c.layout != GEMM_NT && c.layout != GEMM_NN && c.layout != GEMM_TN) {
    fprintf(stderr, "[b200] bad gemm layout %d\n", c.layout);
    abort();
  }
  const bool wide = c.block_n != 128 && c.N > 128;             // 128 x 256 tiles unless the caller asks for 128 x 128
  const LaunchFn run = kernel_for(c.fp8 ? FORM_FP8 : c.layout, c.epi, wide);
  if (run == nullptr) return false;
  if (!c.fp8) {
    run(c, st);
    return true;
  }
  if (c.scale_a == nullptr || c.scale_b == nullptr) {
    fprintf(stderr, "[b200] fp8 gemm needs the device dequantisation factors of both operands\n");
    abort();
  }
  GemmCall k = c;
  k.layout = GEMM_NT;
  void* ta = nullptr; void* tb = nullptr;
  if (c.layout == GEMM_TN) k.A = ta = const_cast<void*>(fp8_k_major(c.A, c.M, c.K, c.lda, &k.lda, st));
  if (c.layout != GEMM_NT) k.B = tb = const_cast<void*>(fp8_k_major(c.B, c.N, c.K, c.ldb, &k.ldb, st));
  run(k, st);
  if (ta) B200_CUDA_CHECK(cudaFreeAsync(ta, st));
  if (tb) B200_CUDA_CHECK(cudaFreeAsync(tb, st));
  return true;
}

}  // namespace b200
