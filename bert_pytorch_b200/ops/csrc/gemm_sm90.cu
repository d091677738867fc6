// Warp-specialised wgmma GEMM for sm_90a with fused epilogues.
//
//   D[M,N] = epilogue( A[M,K] * B[N,K]^T )        bf16 (or fp8) operands, fp32 accumulation in registers
//
// One CTA per 128 x BLOCK_N output tile (and K split).  Warpgroup 0 is the producer: one thread moves operand tiles
// global -> shared memory with cp.async.bulk.tensor (TMA, 128B swizzle) through a STAGES-deep mbarrier ring.
// Warpgroups 1 and 2 each own 64 rows of the tile: they issue wgmma.mma_async straight from the ring, keep one
// group in flight, hand a slot back as soon as the group that read it has retired, and run the epilogue from their
// accumulator registers.
//
// Both bf16 operands can be K-major (reduction dim contiguous) or MN-major, selected per instantiation, so the same
// kernel serves the three GEMMs of a linear layer without any transpose copy:
//     forward  Y  = X  W^T        A K-major (X[M,K]),     B K-major  (W[N,K])
//     dgrad    dX = dY W          A K-major (dY[M,N']),   B MN-major (W[N',K'] read as [Kred][N])
//     wgrad    dW = dY^T X        A MN-major (dY[M,N']),  B MN-major (X[M,K'])   (+ split-K, fp32 reductions)
// fp8 wgmma reads K-major operands only: an MN-major fp8 operand is transposed once into a stream-ordered scratch
// buffer (fp8_transpose_kernel) and the GEMM runs in the NT form.
//
// Epilogues (runtime switch, warp uniform): bias, bias+GELU(erf) with the pre-activation or the derivative saved for
// backward, bias+dropout+residual, residual add, multiply by GELU'(aux) or by a saved factor, fp32 accumulate-into
// (wgrad into the gradient arena), bias+tanh, plain fp32.  The accumulator fragment is regrouped inside each quad
// (quad_transpose) so that a thread owns 8 consecutive output columns: one 16-byte store, one Philox draw and one
// keep-bit byte per group.
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
};

struct GemmArgs {
  int M, N, K;
  int m_blocks, n_blocks, k_blocks, k_splits, k_per_split;
  int epi;
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
};

// Epilogue of 8 consecutive output columns [n0, n0 + 8) of one row (n0 % 8 == 0, N % 8 == 0).  `f` holds
// alpha * accumulator.  Returns through `f` the values that were stored (bf16-rounded) for the column sums.
__device__ __forceinline__ void epilogue_group(const GemmArgs& p, float (&f)[8], int row, int n0, unsigned long long seed,
                                               bool add_local) {
  const size_t ooff = (size_t)row * p.ldo + n0;
  if (p.epi == EPI_ACCUM_F32) {
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
  if (p.epi == EPI_F32) {
    float* o = reinterpret_cast<float*>(p.out) + ooff;
    *reinterpret_cast<float4*>(o) = make_float4(f[0], f[1], f[2], f[3]);
    *reinterpret_cast<float4*>(o + 4) = make_float4(f[4], f[5], f[6], f[7]);
    return;
  }
  if (p.bias != nullptr && (p.epi == EPI_BIAS || p.epi == EPI_BIAS_GELU || p.epi == EPI_BIAS_DROP_RES ||
                            p.epi == EPI_BIAS_TANH || p.epi == EPI_BIAS_GELU_DG)) {
    const uint4 b = __ldg(reinterpret_cast<const uint4*>(p.bias + n0));
    const uint32_t w[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 bb = unpack_bf16(w[t]);
      f[2 * t] += bb.x;
      f[2 * t + 1] += bb.y;
    }
  }
  if (p.epi == EPI_BIAS_GELU) {                  // save the pre-activation, then activate
    *reinterpret_cast<uint4*>(p.aux_out + ooff) =
        make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = gelu_erf(f[j]);
  } else if (p.epi == EPI_BIAS_GELU_DG) {
    float dg[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const GeluParts gp = gelu_parts(f[j]);
      dg[j] = fmaf(f[j] * 0.3989422804014327f, gp.e, gp.Phi);
      f[j] *= gp.Phi;
    }
    *reinterpret_cast<uint4*>(p.aux_out + ooff) =
        make_uint4(pack_bf16(dg[0], dg[1]), pack_bf16(dg[2], dg[3]), pack_bf16(dg[4], dg[5]), pack_bf16(dg[6], dg[7]));
  } else if (p.epi == EPI_BIAS_TANH) {
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = tanhf(f[j]);
  } else if (p.epi == EPI_BIAS_DROP_RES || p.epi == EPI_ADD || p.epi == EPI_DGELU || p.epi == EPI_MUL) {
    if (p.epi == EPI_BIAS_DROP_RES && p.drop_thresh16 != 0) {
      const size_t moff = (size_t)row * (size_t)(p.N >> 3) + (size_t)(n0 >> 3);
      uint32_t kb;
      if (p.mask_in != nullptr) {
        kb = __ldg(p.mask_in + moff);
      } else {
        const uint64_t e8 = ((uint64_t)row * (uint64_t)p.N + (uint64_t)n0) >> 3;
        const Keep8 keep = dropout_keep8(seed, p.stream, e8, p.drop_thresh16);
        kb = 0;
#pragma unroll
        for (int t = 0; t < 8; ++t) kb |= (keep[t] ? 1u : 0u) << t;
        if (p.mask_out != nullptr) p.mask_out[moff] = (unsigned char)kb;
      }
#pragma unroll
      for (int t = 0; t < 8; ++t) f[t] = (kb >> t) & 1u ? f[t] * p.drop_scale : 0.f;
    }
    if (p.res != nullptr) {
      const uint4 r = *reinterpret_cast<const uint4*>(p.res + (size_t)row * p.ldr + n0);
      const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 rr = unpack_bf16(w[t]);
        if (p.epi == EPI_DGELU) {
          f[2 * t] *= dgelu_erf(rr.x);
          f[2 * t + 1] *= dgelu_erf(rr.y);
        } else if (p.epi == EPI_MUL) {
          f[2 * t] *= rr.x;
          f[2 * t + 1] *= rr.y;
        } else {
          f[2 * t] += rr.x;
          f[2 * t + 1] += rr.y;
        }
      }
    }
  }
  const uint4 o = make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
  *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + ooff) = o;
  const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const float2 v = unpack_bf16(ow[t]);
    f[2 * t] = v.x;
    f[2 * t + 1] = v.y;
  }
}

// main loop of one consumer warpgroup: acc (+)= A[64 rows] * B over k-blocks [kb0, kb1)
template <bool A_MN, bool B_MN, int BLOCK_N, bool FP8, int AE5, int BE5>
__device__ __forceinline__ void consumer_mainloop(float (&acc)[BLOCK_N / 2], uint8_t* smem, uint64_t* full_bar,
                                                  uint64_t* empty_bar, int wg, int nkb) {
  using C = Cfg<BLOCK_N>;
  const int lane = threadIdx.x & 31;
  int s = 0, prev = -1;
  uint32_t ph = 0;
  for (int i = 0; i < nkb; ++i) {
    mbar_wait_mma(&full_bar[s], ph);
    const uint32_t sa = smem_u32(smem + s * C::STAGE_BYTES) + wg * 8192;   // this warpgroup's 64 rows (or 64-wide MN chunk)
    const uint32_t sb = smem_u32(smem + s * C::STAGE_BYTES) + C::A_BYTES;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      // advance inside the tile: K-major +32 B per MMA (16 bf16 / 32 fp8), MN-major +16 k-rows * 128 B
      const uint64_t da = A_MN ? wgmma_desc_sw128(sa + kk * 2048, 8192, 1024) : wgmma_desc_sw128(sa + kk * 32, 16, 1024);
      const uint64_t db = B_MN ? wgmma_desc_sw128(sb + kk * 2048, 8192, 1024) : wgmma_desc_sw128(sb + kk * 32, 16, 1024);
      if constexpr (FP8) WgmmaFp8SS<BLOCK_N, AE5, BE5>::mma(acc, da, db, (i > 0 || kk > 0) ? 1 : 0);
      else WgmmaBf16SS<BLOCK_N, A_MN ? 1 : 0, B_MN ? 1 : 0>::mma(acc, da, db, (i > 0 || kk > 0) ? 1 : 0);
    }
    wgmma_commit();
    wgmma_wait<1>();                              // the group that read slot `prev` has retired
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    prev = s;
    if (++s == C::STAGES) { s = 0; ph ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
  if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
}

template <bool A_MN, bool B_MN, int BLOCK_N, bool FP8>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
            const GemmArgs p) {
  using C = Cfg<BLOCK_N>;
  static_assert(!FP8 || (!A_MN && !B_MN), "fp8 wgmma reads K-major operands only");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + C::STAGES;

  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);               // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  const int tile = blockIdx.x;
  const int nb = tile % p.n_blocks;
  const int mb = (tile / p.n_blocks) % p.m_blocks;
  const int ks = tile / (p.n_blocks * p.m_blocks);
  const int kb0 = ks * p.k_per_split;
  const int kb1 = min(p.k_blocks, kb0 + p.k_per_split);
  constexpr int BK = FP8 ? 128 : 64;             // elements along K per stage

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
    if (threadIdx.x == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait_mma(&empty_bar[s], ph ^ 1);
        uint8_t* sa = smem + s * C::STAGE_BYTES;
        uint8_t* sb = sa + C::A_BYTES;
        mbar_arrive_expect_tx(&full_bar[s], C::STAGE_BYTES);
        if constexpr (!A_MN) {
          tma_load_2d(sa, &tmap_a, &full_bar[s], kb * BK, mb * BLOCK_M);
        } else {
#pragma unroll
          for (int j = 0; j < BLOCK_M / 64; ++j)
            tma_load_2d(sa + j * 8192, &tmap_a, &full_bar[s], mb * BLOCK_M + j * 64, kb * BK);
        }
        if constexpr (!B_MN) {
          tma_load_2d(sb, &tmap_b, &full_bar[s], kb * BK, nb * BLOCK_N);
        } else {
#pragma unroll
          for (int j = 0; j < BLOCK_N / 64; ++j)
            tma_load_2d(sb + j * 8192, &tmap_b, &full_bar[s], nb * BLOCK_N + j * 64, kb * BK);
        }
        if (++s == C::STAGES) { s = 0; ph ^= 1; }
      }
    }
    return;
  }
  // -------------------------------------------------------------------- MMA + epilogue (two warpgroups x 64 rows)
  asm volatile("setmaxnreg.inc.sync.aligned.u32 240;");
  const int cw = wg - 1;
  float acc[BLOCK_N / 2];                       // the first MMA of the tile overwrites it (scale-d = 0)
  const int nkb = kb1 - kb0;
  if constexpr (FP8) {
    switch (p.fp8_fmt & 3u) {
      case 0: consumer_mainloop<A_MN, B_MN, BLOCK_N, true, 0, 0>(acc, smem, full_bar, empty_bar, cw, nkb); break;
      case 1: consumer_mainloop<A_MN, B_MN, BLOCK_N, true, 1, 0>(acc, smem, full_bar, empty_bar, cw, nkb); break;
      case 2: consumer_mainloop<A_MN, B_MN, BLOCK_N, true, 0, 1>(acc, smem, full_bar, empty_bar, cw, nkb); break;
      default: consumer_mainloop<A_MN, B_MN, BLOCK_N, true, 1, 1>(acc, smem, full_bar, empty_bar, cw, nkb); break;
    }
  } else {
    consumer_mainloop<A_MN, B_MN, BLOCK_N, false, 0, 0>(acc, smem, full_bar, empty_bar, cw, nkb);
  }
  if (nkb <= 0) return;

  float alpha = p.alpha;
  if constexpr (FP8) alpha *= __ldg(p.scale_a) * __ldg(p.scale_b);   // per-tensor dequantisation
  const unsigned long long seed = p.drop_thresh16 != 0 ? p.seed.value() : 0ull;
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  const int c = lane & 3;
  const int row_base = mb * BLOCK_M + cw * 64 + warp * 16 + (lane >> 2);
  const bool bf16_out = p.epi != EPI_ACCUM_F32 && p.epi != EPI_F32;
#pragma unroll
  for (int i = 0; i < BLOCK_N / 32; ++i) {         // unrolled: the accumulator must stay in registers
    const int n0 = nb * BLOCK_N + i * 32 + c * 8;            // after the regrouping this lane owns columns [n0, n0 + 8)
    if (nb * BLOCK_N + i * 32 >= p.N) break;                 // warp uniform
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
      quad_transpose(lo);
      quad_transpose(hi);
      const int row = row_base + h * 8;
      if (row < p.M && n0 < p.N) {
        float f[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          f[2 * k] = __uint_as_float(lo[k]) * alpha;
          f[2 * k + 1] = __uint_as_float(hi[k]) * alpha;
        }
        epilogue_group(p, f, row, n0, seed, ks == 0);
#pragma unroll
        for (int t = 0; t < 8; ++t) cs[t] += f[t];
      }
    }
    if (p.colsum != nullptr && bf16_out) {       // bias gradients: rows of this warp, then one atomic per column
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


template <bool A_MN, bool B_MN, int BLOCK_N, bool FP8>
static void launch(const GemmCall& c, cudaStream_t st) {
  using C = Cfg<BLOCK_N>;
  constexpr int BK = FP8 ? 128 : 64;
  GemmArgs p;
  p.M = c.M; p.N = c.N; p.K = c.K;
  p.m_blocks = (c.M + BLOCK_M - 1) / BLOCK_M;
  p.n_blocks = (c.N + BLOCK_N - 1) / BLOCK_N;
  p.k_blocks = (c.K + BK - 1) / BK;
  if (p.m_blocks <= 0 || p.n_blocks <= 0 || p.k_blocks <= 0) return;
  int splits = c.epi == EPI_ACCUM_F32 ? c.k_splits : 1;       // only the reducing epilogue can merge K ranges
  if (splits < 0) {                                            // automatic: fill the machine, >= 4 k-blocks per CTA
    splits = num_sms() / (p.m_blocks * p.n_blocks);
    if (splits > p.k_blocks / 4) splits = p.k_blocks / 4;
  }
  p.k_splits = splits < 1 ? 1 : splits;
  if (p.k_splits > p.k_blocks) p.k_splits = p.k_blocks;
  p.k_per_split = (p.k_blocks + p.k_splits - 1) / p.k_splits;
  p.k_splits = (p.k_blocks + p.k_per_split - 1) / p.k_per_split;   // no empty splits
  p.epi = c.epi;
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
  auto kern = gemm_kernel<A_MN, B_MN, BLOCK_N, FP8>;
  static bool configured = false;
  if (!configured) {
    B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_TOTAL));
    configured = true;
  }
  const int grid = p.m_blocks * p.n_blocks * p.k_splits;
  launch_pdl(kern, dim3(grid), dim3(NUM_THREADS), C::SMEM_TOTAL, st, ta, tb, p);
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

void gemm_bf16(const GemmCall& c, cudaStream_t st) {
  if (c.layout != GEMM_NT && c.layout != GEMM_NN && c.layout != GEMM_TN) {
    fprintf(stderr, "[b200] bad gemm layout %d\n", c.layout);
    abort();
  }
  const bool wide = c.block_n != 128 && c.N > 128;             // 128 x 256 tiles unless the caller asks for 128 x 128
  if (c.fp8) {
    if (c.scale_a == nullptr || c.scale_b == nullptr) {
      fprintf(stderr, "[b200] fp8 gemm needs the device dequantisation factors of both operands\n");
      abort();
    }
    GemmCall k = c;
    k.layout = GEMM_NT;
    void* ta = nullptr; void* tb = nullptr;
    if (c.layout == GEMM_TN) k.A = ta = const_cast<void*>(fp8_k_major(c.A, c.M, c.K, c.lda, &k.lda, st));
    if (c.layout != GEMM_NT) k.B = tb = const_cast<void*>(fp8_k_major(c.B, c.N, c.K, c.ldb, &k.ldb, st));
    wide ? launch<false, false, 256, true>(k, st) : launch<false, false, 128, true>(k, st);
    if (ta) B200_CUDA_CHECK(cudaFreeAsync(ta, st));
    if (tb) B200_CUDA_CHECK(cudaFreeAsync(tb, st));
    return;
  }
  switch (c.layout) {
    case GEMM_NT: wide ? launch<false, false, 256, false>(c, st) : launch<false, false, 128, false>(c, st); break;
    case GEMM_NN: wide ? launch<false, true, 256, false>(c, st) : launch<false, true, 128, false>(c, st); break;
    default: wide ? launch<true, true, 256, false>(c, st) : launch<true, true, 128, false>(c, st); break;
  }
}

}  // namespace b200
