// Fused multi-head attention for BERT (non-causal, key-padding mask given as per-sequence valid length,
// head_dim 64, S <= 512) on wgmma (sm_90a): scores, softmax, dropout and P V never leave the SM.
// Padded form: the valid keys of sequence b are its first min(seqlens[b], S); seqlens[b] <= 0 (an all-zero mask row)
// makes all S keys valid, which is what the model's additive -10000 mask computes, so every output stays finite.
//
// Data layout: qkv is the QKV-GEMM output [B*S, 3H] (token-major, q|k|v, head-major inside), so the Q / K / V tiles
// of a head are 64-column TMA boxes of that matrix; ctx / dctx are [B*S, H].
//
// Forward   attn_fwd_kernel: one warpgroup per (batch, head, 64-query block).  K and V of the valid key range arrive by
//           TMA in 128-key blocks, one mbarrier each.  Per block: S = Q K^T (wgmma, operands in shared memory), online
//           softmax on the accumulator fragment (fp32, exp2), dropout on the probabilities, and P~ goes straight from
//           the accumulator registers into the A operand of O += P~ V (V is read MN-major: no transpose).
// Backward  attn_bwd_kernel: one CTA per (batch, head, 128-key block), two warpgroups of 64 keys each, looping over
//           64-query blocks (Q / dO double buffered).  S = Q K^T and dP = dO V^T on the tensor cores; P~ and dS are
//           formed in registers; dQ += dS K takes dS from registers; P~ and dS pass through shared memory once and
//           are read MN-major for dV += P~^T dO and dK += dS^T Q.  dQ is reduced across key blocks with fp32 reductions
//           into dq_acc and converted to bf16 by attn_dq_convert_kernel; delta = <dO, O> comes from attn_delta_kernel.
//           S <= 128 (one key block) runs attn_bwd_onepass_kernel instead: the same per-block math in a persistent
//           CTA per (batch, head) item, with delta and the dQ sum inside.
// Varlen (VARLEN = true): qkv is packed [T, 3H] and ctx / dctx / dq_acc are [T, H]; sequence b owns rows
// cu_seqlens[b] .. cu_seqlens[b + 1] (passed in AttnArgs::seqlens).  S is the padded length: it sizes the grid and is
// the stride of the dropout counter, so the keep decisions equal the padded kernel's for the same batch.  lse and
// delta stay [B, h, S], indexed by the position inside the sequence.  CTAs whose query block (forward) or key block
// (backward) starts at or past the sequence's end exit at once; TMA boxes that run into the next sequence (or past T,
// zero fill) are masked as keys, and every store is bounded by the sequence length so no neighbour row is written.
// Dropout: Philox counter RNG, one draw per 8 consecutive keys of a (batch, head, query) row; the backward regenerates
// the forward's keep decisions.  A draw serves the four lanes of a quad (each owns two of the eight keys): lane c of
// the quad draws for key groups c, 4 + c, ... and quad_transpose hands every lane its 32-bit word of each draw.
#include "common.cuh"
#include "gemm_sm90.h"
#include "kernels.h"
#include "wgmma.cuh"

namespace b200 {

constexpr int QT = 64;             // query rows per block (one wgmma M)
constexpr int KT = 128;            // keys per block
constexpr int HD = 64;             // head dim
constexpr float LOG2E = 1.4426950408889634f;

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct AttnArgs {
  int B, S, h, H;
  const int* seqlens;
  __nv_bfloat16* ctx;      // fwd out [B*S, H]
  float* lse;              // [B, h, S] natural-log LSE of the scaled scores
  float scale;
  Seed seed;
  unsigned int stream;
  unsigned int thresh16;
  float inv_keep;
  // backward
  const float* delta;      // [B, h, S]
  __nv_bfloat16* dqkv;     // [B*S, 3H]
  float* dq_acc;           // [B*S, H] fp32
  Fp8Out f8;               // optional fp8 copy of the output (ctx in the forward, dqkv in the backward)
};

// keep decisions of the two keys (8 j + 2 c, 8 j + 2 c + 1) this lane owns in key group j, from its word of the draw
__device__ __forceinline__ void keep_pair(uint32_t word, uint32_t thresh16, bool& k0, bool& k1) {
  k0 = (word & 0xFFFFu) >= thresh16;
  k1 = (word >> 16) >= thresh16;
}

// Philox words for NG key groups (NG % 4 == 0) of one row: w[j] = this lane's word of group j's draw
template <int NG>
__device__ __forceinline__ void draw_row(uint32_t (&w)[NG], const PhiloxKeys& keys, uint64_t e8_row, uint32_t stream) {
  const int c = threadIdx.x & 3;
#pragma unroll
  for (int u = 0; u < NG / 4; ++u) {
    const uint4 r = philox7(keys, e8_row + (uint64_t)(4 * u + c), stream);
    uint32_t a[4] = {r.x, r.y, r.z, r.w};
    quad_transpose(a);
#pragma unroll
    for (int k = 0; k < 4; ++k) w[4 * u + k] = a[k];
  }
}

// Regroup row half `h` of four 8-column accumulator groups (acc4 = &acc[16 u]) so that lane c of a quad holds the
// 8 consecutive columns of group 4 u + c.
__device__ __forceinline__ void regroup8(const float* acc4, int h, float (&f)[8]) {
  uint32_t lo[4], hi[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    lo[k] = __float_as_uint(acc4[4 * k + 2 * h]);
    hi[k] = __float_as_uint(acc4[4 * k + 2 * h + 1]);
  }
  quad_transpose(lo);
  quad_transpose(hi);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    f[2 * k] = __uint_as_float(lo[k]);
    f[2 * k + 1] = __uint_as_float(hi[k]);
  }
}

// Store NU 32-column halves of a [64 rows x 64 columns] accumulator tile (acc: 16 NU fragment values) as bf16
// (16 bytes per lane and row half) + optional fp8 copy.  row_lo: this lane's first row inside the tile; n_valid: rows of
// the tile that exist; dst: element (0, 0) of the first half.
template <int NU>
__device__ __forceinline__ void store_cols64(const float* acc, float mul_lo, float mul_hi, int row_lo, int n_valid,
                                             __nv_bfloat16* dst, size_t ld, const Fp8Out& f8, size_t f8_off, float qscale,
                                             float& amax) {
  const int c = threadIdx.x & 3;
#pragma unroll
  for (int u = 0; u < NU; ++u) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float f[8];
      regroup8(&acc[16 * u], h, f);
      const int row = row_lo + 8 * h;
      const float mul = h ? mul_hi : mul_lo;
#pragma unroll
      for (int t = 0; t < 8; ++t) f[t] *= mul;
      if (row < n_valid) {
        const size_t off = (size_t)row * ld + (4 * u + c) * 8;
        *reinterpret_cast<uint4*>(dst + off) =
            make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
        if (f8.q) fp8_emit8(f8, f8_off + off, f, qscale, amax);
      }
    }
  }
}

// the whole tile
__device__ __forceinline__ void store_tile64(const float (&acc)[32], float mul_lo, float mul_hi, int row_lo, int n_valid,
                                             __nv_bfloat16* dst, size_t ld, const Fp8Out& f8, size_t f8_off, float qscale,
                                             float& amax) {
  store_cols64<2>(acc, mul_lo, mul_hi, row_lo, n_valid, dst, ld, f8, f8_off, qscale, amax);
}

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
template <bool VARLEN>
__global__ void __launch_bounds__(128)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_kv, const AttnArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int qb = blockIdx.x, bh = blockIdx.y;
  const int b = bh / p.h, head = bh % p.h;
  int seqlen, row0;
  if constexpr (VARLEN) {
    row0 = p.seqlens[b];
    seqlen = min(p.seqlens[b + 1] - row0, p.S);
    if (qb * QT >= seqlen) return;                      // CTA uniform, before any mbarrier or TMA work
  } else {
    seqlen = min(p.seqlens[b], p.S);
    if (seqlen <= 0) seqlen = p.S;                      // a fully masked sequence attends to every key
    row0 = b * p.S;
  }
  const int nkb = max(1, (seqlen + KT - 1) / KT);       // key blocks that contain valid keys
  uint8_t* sQ = smem;                                   // 8 KB
  uint8_t* sKV = smem + 8192;                           // per key block: K 16 KB | V 16 KB
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + (size_t)nkb * 32768);   // [0]: Q, [1 + j]: key block j

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_kv);
    for (int i = 0; i <= nkb; ++i) mbar_init(&bars[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&bars[0], 8192);
    tma_load_2d(sQ, &tmap_q, &bars[0], head * HD, row0 + qb * QT);
    for (int j = 0; j < nkb; ++j) {
      mbar_arrive_expect_tx(&bars[1 + j], 32768);
      tma_load_2d(sKV + j * 32768, &tmap_kv, &bars[1 + j], p.H + head * HD, row0 + j * KT);
      tma_load_2d(sKV + j * 32768 + 16384, &tmap_kv, &bars[1 + j], 2 * p.H + head * HD, row0 + j * KT);
    }
  }

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, c = lane & 3;
  const int r_lo = warp * 16 + (lane >> 2);             // this lane's rows inside the block: r_lo, r_lo + 8
  const int q_lo = qb * QT + r_lo;
  const float c_scale = p.scale * LOG2E;
  const bool drop = p.thresh16 != 0;
  const PhiloxKeys keys = philox_keys(drop ? p.seed.value() : 0ull);
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[32];
#pragma unroll
  for (int t = 0; t < 32; ++t) o[t] = 0.f;

  mbar_wait_mma(&bars[0], 0);
  for (int j = 0; j < nkb; ++j) {
    mbar_wait_mma(&bars[1 + j], 0);
    const uint32_t aq = smem_u32(sQ), ak = smem_u32(sKV + j * 32768), av = ak + 16384;
    float s[64];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk)
      WgmmaBf16SS<128, 0, 0>::mma(s, wgmma_desc_sw128(aq + kk * 32, 16, 1024), wgmma_desc_sw128(ak + kk * 32, 16, 1024), kk > 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    const int k0 = j * KT;
    const bool full = k0 + KT <= seqlen;                // every key of this block is valid (CTA uniform)
    uint32_t pk[2][16];                                 // P~ of this lane, bf16 pairs: [row half][key group]
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int g = 0; g < 16; ++g) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = k0 + 8 * g + 2 * c + e;
          if (full || key < seqlen) mx = fmaxf(mx, s[4 * g + 2 * h + e]);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[h], mx * c_scale);    // c_scale > 0: max commutes with the scaling
      const float alpha = (m[h] == -INFINITY) ? 0.f : exp2f(m[h] - m_new);
      uint32_t w[16];
      if (drop) {
        const uint64_t erow = ((uint64_t)bh * p.S + (uint64_t)(q_lo + 8 * h)) * (uint64_t)p.S;
        draw_row<16>(w, keys, (erow + (uint64_t)k0) >> 3, p.stream);
      }
      float rowsum = 0.f;
#pragma unroll
      for (int g = 0; g < 16; ++g) {
        float e0 = ex2_approx(fmaf(s[4 * g + 2 * h], c_scale, -m_new));
        float e1 = ex2_approx(fmaf(s[4 * g + 2 * h + 1], c_scale, -m_new));
        const int key = k0 + 8 * g + 2 * c;
        if (!full && key >= seqlen) e0 = 0.f;
        if (!full && key + 1 >= seqlen) e1 = 0.f;
        rowsum += e0 + e1;
        if (drop) {
          bool ka, kb;
          keep_pair(w[g], p.thresh16, ka, kb);
          e0 = ka ? e0 * p.inv_keep : 0.f;
          e1 = kb ? e1 * p.inv_keep : 0.f;
        }
        pk[h][g] = pack_bf16(e0, e1);
      }
      l[h] = l[h] * alpha + rowsum;                     // this lane's share of the denominator
      m[h] = m_new;
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        o[4 * g + 2 * h] *= alpha;
        o[4 * g + 2 * h + 1] *= alpha;
      }
    }
    wgmma_fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KT / 16; ++kk) {              // O += P~[:, 16 kk ..] V[16 kk .., :]   (V MN-major)
      const uint32_t a[4] = {pk[0][2 * kk], pk[1][2 * kk], pk[0][2 * kk + 1], pk[1][2 * kk + 1]};
      WgmmaBf16RS<64, 1>::mma(o, a, wgmma_desc_sw128(av + kk * 2048, 8192, 1024), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
  }
  float amax = 0.f;
  const float qscale = p.f8.q ? p.f8.meta[1] : 0.f;
  const size_t tile_off = (size_t)(row0 + qb * QT) * p.H + head * HD;
  const int q_end = VARLEN ? seqlen : p.S;              // query rows that exist
  store_tile64(o, 1.f / l[0], 1.f / l[1], r_lo, q_end - qb * QT, p.ctx + tile_off, (size_t)p.H, p.f8, tile_off, qscale, amax);
  if (p.f8.q) fp8_amax_commit(p.f8, amax);
  if (c == 0) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (q_lo + 8 * h < q_end) p.lse[(size_t)bh * p.S + q_lo + 8 * h] = (m[h] + log2f(l[h])) * 0.6931471805599453f;
  }
}

// ------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------
template <bool VARLEN>
__global__ void __launch_bounds__(256)
attn_delta_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ dout, float* __restrict__ delta,
                  int B, int S, int h, int H, const int* __restrict__ cu_seqlens) {
  // one 8-lane group per (token, head): 64 elements = 8 x 16 B; varlen: per (sequence, position < seqlen, head)
  const long long gid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  const int sub = threadIdx.x & 7;
  const long long total = (long long)B * S * h;
  if (gid >= total) return;
  const int head = (int)(gid % h);
  const long long tok = gid / h;                       // (sequence, position) of this group
  long long row = tok;                                  // its row of o / dout
  if constexpr (VARLEN) {
    const int bb = (int)(tok / S), ss = (int)(tok % S);
    const int r0 = cu_seqlens[bb];
    if (ss >= cu_seqlens[bb + 1] - r0) return;
    row = r0 + ss;
  }
  const size_t off = (size_t)row * H + head * HD + sub * 8;
  const uint4 a = *reinterpret_cast<const uint4*>(o + off), d = *reinterpret_cast<const uint4*>(dout + off);
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, dw[4] = {d.x, d.y, d.z, d.w};
  float s = 0.f;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const float2 x = unpack_bf16(aw[t]), y = unpack_bf16(dw[t]);
    s += x.x * y.x + x.y * y.y;
  }
  // varlen: groups past their sequence's end have returned, so each group reduces among its own 8 lanes only
  const unsigned gm = VARLEN ? (0xFFu << (threadIdx.x & 24)) : 0xffffffffu;
  s += __shfl_xor_sync(gm, s, 1);
  s += __shfl_xor_sync(gm, s, 2);
  s += __shfl_xor_sync(gm, s, 4);
  if (sub == 0) {
    const int bb = (int)(tok / S), ss = (int)(tok % S);
    delta[((size_t)bb * h + head) * S + ss] = s;
  }
}


// [64 rows][64 columns] bf16 tile, rows of 128 B, 128B swizzle: byte offset of the pair (row r, columns 8 g + 2 c, + 1)
__device__ __forceinline__ uint32_t tile_pair_offset(int r, int g, int c) {
  return (uint32_t)(r * 128 + ((g ^ (r & 7)) << 4) + 4 * c);
}

constexpr int ATT_BWD_THREADS = 256;
constexpr int ATT_BWD_SMEM = 16384 * 2 + 8192 * 8 + 1024 + 64;

// SLICED (deterministic mode): key block kb adds its dQ into its own fp32 slice dq_acc + kb * slice, which
// attn_dq_convert_kernel<true> sums in key-block order.  The two warpgroups of a CTA add onto a zeroed slice, and
// 0 + a + b == 0 + b + a exactly, so each slice is order-free.  For the same reason a single key block (S <= 128)
// needs no slices: attn_bwd_kernel is deterministic there as it is.
template <bool VARLEN, bool SLICED>
__device__ __forceinline__ void attn_bwd_body(const CUtensorMap& tmap_q, const CUtensorMap& tmap_kv,
                                              const CUtensorMap& tmap_do, const AttnArgs& p, size_t slice) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;                        // 16 KB: 128 keys, warpgroup w reads rows [64 w, 64 w + 64)
  uint8_t* sV = smem + 16384;                // 16 KB
  uint8_t* sQ = smem + 32768;                // 2 stages x 8 KB
  uint8_t* sDO = sQ + 16384;                 // 2 stages x 8 KB
  uint8_t* sP = sDO + 16384;                 // 2 warpgroups x 8 KB: P~ [64 q][64 keys]
  uint8_t* sDS = sP + 16384;                 // 2 warpgroups x 8 KB: dS
  uint64_t* bars = reinterpret_cast<uint64_t*>(sDS + 16384);   // [0]: K / V, [1], [2]: Q / dO stages

  const int kb = blockIdx.x, bh = blockIdx.y;
  const int b = bh / p.h, head = bh % p.h;
  int seqlen, row0;
  if constexpr (VARLEN) {
    row0 = p.seqlens[b];
    seqlen = min(p.seqlens[b + 1] - row0, p.S);
    if (kb * KT >= seqlen) return;                      // CTA uniform, before any mbarrier or TMA work
  } else {
    seqlen = min(p.seqlens[b], p.S);
    if (seqlen <= 0) seqlen = p.S;                      // a fully masked sequence attends to every key
    row0 = b * p.S;
  }
  const int q_end = VARLEN ? seqlen : p.S;              // query rows (and rows of dK / dV) that exist
  const int nqb = (q_end + QT - 1) / QT;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_kv);
    tma_prefetch_desc(&tmap_do);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto load_q = [&](int i) {                 // Q and dO of query block i into stage i & 1
    const int st = i & 1;
    mbar_arrive_expect_tx(&bars[1 + st], 16384);
    tma_load_2d(sQ + st * 8192, &tmap_q, &bars[1 + st], head * HD, row0 + i * QT);
    tma_load_2d(sDO + st * 8192, &tmap_do, &bars[1 + st], head * HD, row0 + i * QT);
  };
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&bars[0], 32768);
    tma_load_2d(sK, &tmap_kv, &bars[0], p.H + head * HD, row0 + kb * KT);
    tma_load_2d(sV, &tmap_kv, &bars[0], 2 * p.H + head * HD, row0 + kb * KT);
    load_q(0);
    if (nqb > 1) load_q(1);
  }

  const int wg = threadIdx.x >> 7;
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, c = lane & 3;
  const int r_lo = warp * 16 + (lane >> 2);
  const int key0 = kb * KT + wg * 64;        // first key of this warpgroup
  const float c_scale = p.scale * LOG2E;
  const bool drop = p.thresh16 != 0;
  const PhiloxKeys keys = philox_keys(drop ? p.seed.value() : 0ull);
  const uint32_t ak = smem_u32(sK) + wg * 8192, av = smem_u32(sV) + wg * 8192;
  uint8_t* myP = sP + wg * 8192;
  uint8_t* myDS = sDS + wg * 8192;
  const uint32_t ap = smem_u32(myP), ads = smem_u32(myDS);
  float dv[32], dk[32];
#pragma unroll
  for (int t = 0; t < 32; ++t) dv[t] = dk[t] = 0.f;

  mbar_wait_mma(&bars[0], 0);
  for (int i = 0; i < nqb; ++i) {
    const int st = i & 1;
    mbar_wait_mma(&bars[1 + st], (i >> 1) & 1);
    const uint32_t aq = smem_u32(sQ + st * 8192), ado = smem_u32(sDO + st * 8192);
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
      WgmmaBf16SS<64, 0, 0>::mma(s, wgmma_desc_sw128(aq + kk * 32, 16, 1024), wgmma_desc_sw128(ak + kk * 32, 16, 1024), kk > 0);
      WgmmaBf16SS<64, 0, 0>::mma(dp, wgmma_desc_sw128(ado + kk * 32, 16, 1024), wgmma_desc_sw128(av + kk * 32, 16, 1024), kk > 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    wgmma_fence_regs(dp);
    uint32_t dsp[2][8];                      // dS of this lane, bf16 pairs: [row half][key group]
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r_lo + 8 * h, q = i * QT + r;
      const bool q_ok = q < q_end;
      const float lse2 = q_ok ? __ldg(p.lse + (size_t)bh * p.S + q) * LOG2E : 0.f;
      const float dlt = q_ok ? __ldg(p.delta + (size_t)bh * p.S + q) : 0.f;
      uint32_t w[8];
      if (drop) {
        const uint64_t erow = ((uint64_t)bh * p.S + (uint64_t)q) * (uint64_t)p.S;
        draw_row<8>(w, keys, (erow + (uint64_t)key0) >> 3, p.stream);
      }
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        const int key = key0 + 8 * g + 2 * c;
        const float pr0 = (q_ok && key < seqlen) ? ex2_approx(fmaf(s[4 * g + 2 * h], c_scale, -lse2)) : 0.f;
        const float pr1 = (q_ok && key + 1 < seqlen) ? ex2_approx(fmaf(s[4 * g + 2 * h + 1], c_scale, -lse2)) : 0.f;
        bool ka = true, kb2 = true;
        if (drop) keep_pair(w[g], p.thresh16, ka, kb2);
        const float dp0 = ka ? dp[4 * g + 2 * h] * p.inv_keep : 0.f;
        const float dp1 = kb2 ? dp[4 * g + 2 * h + 1] * p.inv_keep : 0.f;
        const uint32_t pd = pack_bf16(ka ? pr0 * p.inv_keep : 0.f, kb2 ? pr1 * p.inv_keep : 0.f);
        const uint32_t ds = pack_bf16(pr0 * (dp0 - dlt) * p.scale, pr1 * (dp1 - dlt) * p.scale);
        dsp[h][g] = ds;
        *reinterpret_cast<uint32_t*>(myP + tile_pair_offset(r, g, c)) = pd;
        *reinterpret_cast<uint32_t*>(myDS + tile_pair_offset(r, g, c)) = ds;
      }
    }
    fence_proxy_async();                     // generic-proxy smem writes -> visible to wgmma (async proxy)
    asm volatile("bar.sync %0, 128;" ::"r"(wg + 1) : "memory");
    float dq[32];
    wgmma_fence_regs(dv);
    wgmma_fence_regs(dk);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < QT / 16; ++kk) {   // reduction over the 64 queries: P~ / dS and dO / Q all read MN-major
      WgmmaBf16SS<64, 1, 1>::mma(dv, wgmma_desc_sw128(ap + kk * 2048, 8192, 1024), wgmma_desc_sw128(ado + kk * 2048, 8192, 1024), 1);
      WgmmaBf16SS<64, 1, 1>::mma(dk, wgmma_desc_sw128(ads + kk * 2048, 8192, 1024), wgmma_desc_sw128(aq + kk * 2048, 8192, 1024), 1);
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {         // dQ (partial: this warpgroup's 64 keys) = dS K
      const uint32_t a[4] = {dsp[0][2 * kk], dsp[1][2 * kk], dsp[0][2 * kk + 1], dsp[1][2 * kk + 1]};
      WgmmaBf16RS<64, 1>::mma(dq, a, wgmma_desc_sw128(ak + kk * 2048, 8192, 1024), kk > 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(dv);
    wgmma_fence_regs(dk);
    wgmma_fence_regs(dq);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int q = i * QT + r_lo + 8 * h;
      if (q < q_end) {
        float* dst = p.dq_acc + (size_t)(row0 + q) * p.H + head * HD + 2 * c;
        if constexpr (SLICED) dst += kb * slice;
#pragma unroll
        for (int g = 0; g < 8; ++g)
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst + 8 * g), "f"(dq[4 * g + 2 * h]),
                       "f"(dq[4 * g + 2 * h + 1]) : "memory");
      }
    }
    __syncthreads();                         // both warpgroups are done with stage st
    if (threadIdx.x == 0 && i + 2 < nqb) load_q(i + 2);
  }
  // dK -> k slots, dV -> v slots of dqkv (rows = keys of this warpgroup)
  float amax = 0.f;
  const float qscale = p.f8.q ? p.f8.meta[1] : 0.f;
  const size_t k_off = (size_t)(row0 + key0) * 3 * p.H + p.H + head * HD;
  store_tile64(dk, 1.f, 1.f, r_lo, q_end - key0, p.dqkv + k_off, (size_t)3 * p.H, p.f8, k_off, qscale, amax);
  store_tile64(dv, 1.f, 1.f, r_lo, q_end - key0, p.dqkv + k_off + p.H, (size_t)3 * p.H, p.f8, k_off + p.H, qscale, amax);
  if (p.f8.q) fp8_amax_commit(p.f8, amax);
}

template <bool VARLEN>
__global__ void __launch_bounds__(ATT_BWD_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_kv,
                const __grid_constant__ CUtensorMap tmap_do, const AttnArgs p) {
  attn_bwd_body<VARLEN, false>(tmap_q, tmap_kv, tmap_do, p, 0);
}

template <bool VARLEN>
__global__ void __launch_bounds__(ATT_BWD_THREADS, 1)
attn_bwd_sliced_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_kv,
                       const __grid_constant__ CUtensorMap tmap_do, const AttnArgs p, long long slice) {
  attn_bwd_body<VARLEN, true>(tmap_q, tmap_kv, tmap_do, p, (size_t)slice);
}

// dq_acc (fp32 [B*S, H]) -> q slots of dqkv (bf16 [B*S, 3H]).  SLICED: dq_acc is [nslices, rows, H], summed in slice
// order (a varlen CTA past the end of its sequence leaves its slice zero).
template <bool SLICED>
__device__ __forceinline__ void attn_dq_convert_body(const float* __restrict__ acc, __nv_bfloat16* __restrict__ dqkv,
                                                     long long rows, int H, const Fp8Out& f8, int nslices) {
  const int per_row = H / 8;
  const float qscale = f8.q ? f8.meta[1] : 0.f;
  float amax = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < rows * per_row;
       i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / per_row;
    const int col = (int)(i % per_row) * 8;
    float4 a = *reinterpret_cast<const float4*>(acc + row * H + col);
    float4 c = *reinterpret_cast<const float4*>(acc + row * H + col + 4);
    if constexpr (SLICED) {
      for (int k = 1; k < nslices; ++k) {
        const float* sl = acc + (size_t)k * rows * H + row * H + col;
        const float4 a2 = *reinterpret_cast<const float4*>(sl), c2 = *reinterpret_cast<const float4*>(sl + 4);
        a.x += a2.x; a.y += a2.y; a.z += a2.z; a.w += a2.w;
        c.x += c2.x; c.y += c2.y; c.z += c2.z; c.w += c2.w;
      }
    }
    *reinterpret_cast<uint4*>(dqkv + row * 3 * H + col) =
        make_uint4(pack_bf16(a.x, a.y), pack_bf16(a.z, a.w), pack_bf16(c.x, c.y), pack_bf16(c.z, c.w));
    if (f8.q) {
      const float t8[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
      fp8_emit8(f8, (size_t)(row * 3 * H + col), t8, qscale, amax);
    }
  }
  if (f8.q) fp8_amax_commit(f8, amax);
}

__global__ void __launch_bounds__(256)
attn_dq_convert_kernel(const float* __restrict__ acc, __nv_bfloat16* __restrict__ dqkv, long long rows, int H, const Fp8Out f8) {
  attn_dq_convert_body<false>(acc, dqkv, rows, H, f8, 1);
}

__global__ void __launch_bounds__(256)
attn_dq_convert_sliced_kernel(const float* __restrict__ acc, __nv_bfloat16* __restrict__ dqkv, long long rows, int H,
                              const Fp8Out f8, int nslices) {
  attn_dq_convert_body<true>(acc, dqkv, rows, H, f8, nslices);
}

// ------------------------------------------------------------------------------------------------
// one-pass backward (S <= 128: one key block holds every key of a sequence)
// ------------------------------------------------------------------------------------------------
// attn_bwd_onepass_kernel: persistent; CTA x walks the (batch, head) items x, x + gridDim.x, ...  The CTA of an item
// sees every query and key of its head, so the whole backward is one pass:
//  - delta = <dO, O> of a query block from its dO and O tiles in shared memory, with attn_delta_kernel's arithmetic
//    (same 8-column partial sums and contraction, same xor 1, 2, 4 combine), so it is bit-identical;
//  - the two warpgroups' dQ partials are summed through shared memory as 0 + a + b (the value the fp32 reductions
//    into a zeroed dq_acc produce, signed zeros included) and stored as bf16 into the q slots of dqkv.
// Loads run ahead of the MMAs: K / V are double buffered per item, and Q | dO | O per query block ("job"), so while
// an item computes, the K / V of the next item and the first query block of the next item are in flight.
constexpr int ATT_OP_SMEM_TILES = 2 * 32768 + 3 * 2 * 8192 + 2 * 16384;   // K|V x2, Q / dO / O x2, P~ / dS
constexpr int ATT_OP_SMEM = ATT_OP_SMEM_TILES + 1024 + 64 + 64 * 4;

template <bool VARLEN>
__device__ __forceinline__ void onepass_item(const AttnArgs& p, int it, int& row0, int& nrows) {
  const int b = it / p.h;
  if constexpr (VARLEN) {
    row0 = p.seqlens[b];
    nrows = min(p.seqlens[b + 1] - row0, p.S);          // rows (queries = keys) of the sequence; 0: nothing to do
  } else {
    row0 = b * p.S;
    nrows = p.S;                                        // every row of a padded sequence gets dQ, dK and dV
  }
}

template <bool VARLEN>
__device__ __forceinline__ int onepass_next(const AttnArgs& p, int it) {   // the next item of this CTA with rows
  const int n = p.B * p.h;
  for (it += gridDim.x; VARLEN && it < n; it += gridDim.x) {
    int r0, nr;
    onepass_item<VARLEN>(p, it, r0, nr);
    if (nr > 0) break;
  }
  return it;
}

template <bool VARLEN>
__global__ void __launch_bounds__(ATT_BWD_THREADS, 1)
attn_bwd_onepass_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_kv,
                        const __grid_constant__ CUtensorMap tmap_do, const __grid_constant__ CUtensorMap tmap_o,
                        const AttnArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sKV = smem;                       // 2 stages x (K 16 KB | V 16 KB); warpgroup w reads key rows [64 w, 64 w + 64)
  uint8_t* sQ = smem + 65536;                // 2 stages x 8 KB
  uint8_t* sDO = sQ + 16384;                 // 2 stages x 8 KB
  uint8_t* sO = sDO + 16384;                 // 2 stages x 8 KB
  uint8_t* sP = sO + 16384;                  // 2 warpgroups x 8 KB: P~, then this warpgroup's dQ half for the other one
  uint8_t* sDS = sP + 16384;                 // 2 warpgroups x 8 KB: dS
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + ATT_OP_SMEM_TILES);   // [0], [1]: K / V stages, [2], [3]: jobs
  float* sDelta = reinterpret_cast<float*>(bars + 8);                      // [64] delta of the current query block

  const int nitems = p.B * p.h;
  int first = blockIdx.x;
  if (VARLEN && first < nitems) {
    int r0, nr;
    onepass_item<VARLEN>(p, first, r0, nr);
    if (nr == 0) first = onepass_next<VARLEN>(p, first);
  }
  if (first >= nitems) return;                          // CTA uniform, before any mbarrier or TMA work

  // producer state (thread 0): the next item whose K / V to load, the next job (item, query block) whose Q / dO / O
  int kv_it = first, kv_n = 0, job_it = first, job_qb = 0, job_n = 0;
  auto issue_kv = [&]() {
    if (kv_it >= nitems) return;
    int r0, nr;
    onepass_item<VARLEN>(p, kv_it, r0, nr);
    const int head = kv_it % p.h, st = kv_n & 1;
    mbar_arrive_expect_tx(&bars[st], 32768);
    tma_load_2d(sKV + st * 32768, &tmap_kv, &bars[st], p.H + head * HD, r0);
    tma_load_2d(sKV + st * 32768 + 16384, &tmap_kv, &bars[st], 2 * p.H + head * HD, r0);
    ++kv_n;
    kv_it = onepass_next<VARLEN>(p, kv_it);
  };
  auto issue_job = [&]() {
    if (job_it >= nitems) return;
    int r0, nr;
    onepass_item<VARLEN>(p, job_it, r0, nr);
    const int head = job_it % p.h, st = job_n & 1, row = r0 + job_qb * QT;
    mbar_arrive_expect_tx(&bars[2 + st], 3 * 8192);
    tma_load_2d(sQ + st * 8192, &tmap_q, &bars[2 + st], head * HD, row);
    tma_load_2d(sDO + st * 8192, &tmap_do, &bars[2 + st], head * HD, row);
    tma_load_2d(sO + st * 8192, &tmap_o, &bars[2 + st], head * HD, row);
    ++job_n;
    if (++job_qb * QT >= nr) {
      job_qb = 0;
      job_it = onepass_next<VARLEN>(p, job_it);
    }
  };
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_kv);
    tma_prefetch_desc(&tmap_do);
    tma_prefetch_desc(&tmap_o);
    for (int i = 0; i < 4; ++i) mbar_init(&bars[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    issue_kv(); issue_kv();
    issue_job(); issue_job();
  }

  const int wg = threadIdx.x >> 7, tw = threadIdx.x & 127;
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, c = lane & 3;
  const int r_lo = warp * 16 + (lane >> 2);
  const int key0 = wg * 64;                  // first key of this warpgroup
  const float c_scale = p.scale * LOG2E;
  const bool drop = p.thresh16 != 0;
  const PhiloxKeys keys = philox_keys(drop ? p.seed.value() : 0ull);
  uint8_t* myP = sP + wg * 8192;
  uint8_t* myDS = sDS + wg * 8192;
  const uint32_t ap = smem_u32(myP), ads = smem_u32(myDS);
  const float* otherDq = reinterpret_cast<const float*>(sP + (wg ^ 1) * 8192);
  float amax = 0.f;
  const float qscale = p.f8.q ? p.f8.meta[1] : 0.f;
  const size_t ld = (size_t)3 * p.H;
  int j = 0;                                 // jobs done by this CTA

  for (int it = first, n = 0; it < nitems; it = onepass_next<VARLEN>(p, it), ++n) {
    const int bh = it, head = it % p.h;
    int row0, q_end;
    onepass_item<VARLEN>(p, it, row0, q_end);
    int seqlen = q_end;                      // valid keys
    if constexpr (!VARLEN) {
      seqlen = min(p.seqlens[it / p.h], p.S);
      if (seqlen <= 0) seqlen = p.S;                    // a fully masked sequence attends to every key
    }
    const int nqb = (q_end + QT - 1) / QT;
    const uint32_t ak = smem_u32(sKV + (n & 1) * 32768) + wg * 8192, av = ak + 16384;
    float dv[32], dk[32];
#pragma unroll
    for (int t = 0; t < 32; ++t) dv[t] = dk[t] = 0.f;

    mbar_wait_mma(&bars[n & 1], (n >> 1) & 1);
    for (int i = 0; i < nqb; ++i, ++j) {
      const int st = j & 1;
      mbar_wait_mma(&bars[2 + st], (j >> 1) & 1);
      {                                      // delta of the 64 rows: 8 lanes per row, 8 columns per lane
        const uint8_t* o_t = sO + st * 8192;
        const uint8_t* d_t = sDO + st * 8192;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int r = (threadIdx.x >> 3) + 32 * k, sub = threadIdx.x & 7;
          const uint32_t off = r * 128 + ((sub ^ (r & 7)) << 4);
          const uint4 a = *reinterpret_cast<const uint4*>(o_t + off), d = *reinterpret_cast<const uint4*>(d_t + off);
          const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, dw[4] = {d.x, d.y, d.z, d.w};
          float s = 0.f;
#pragma unroll
          for (int t = 0; t < 4; ++t) {          // attn_delta_kernel's contraction: s + fma(x.x, y.x, x.y * y.y)
            const float2 x = unpack_bf16(aw[t]), y = unpack_bf16(dw[t]);
            s = __fadd_rn(s, __fmaf_rn(x.x, y.x, __fmul_rn(x.y, y.y)));
          }
          s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 1));
          s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 2));
          s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 4));
          if (sub == 0) sDelta[r] = s;
        }
      }
      __syncthreads();
      const uint32_t aq = smem_u32(sQ + st * 8192), ado = smem_u32(sDO + st * 8192);
      float s[32], dp[32];
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk) {
        WgmmaBf16SS<64, 0, 0>::mma(s, wgmma_desc_sw128(aq + kk * 32, 16, 1024), wgmma_desc_sw128(ak + kk * 32, 16, 1024), kk > 0);
        WgmmaBf16SS<64, 0, 0>::mma(dp, wgmma_desc_sw128(ado + kk * 32, 16, 1024), wgmma_desc_sw128(av + kk * 32, 16, 1024), kk > 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(s);
      wgmma_fence_regs(dp);
      uint32_t dsp[2][8];                    // dS of this lane, bf16 pairs: [row half][key group]
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r_lo + 8 * h, q = i * QT + r;
        const bool q_ok = q < q_end;
        const float lse2 = q_ok ? __ldg(p.lse + (size_t)bh * p.S + q) * LOG2E : 0.f;
        const float dlt = q_ok ? sDelta[r] : 0.f;
        uint32_t w[8];
        if (drop) {
          const uint64_t erow = ((uint64_t)bh * p.S + (uint64_t)q) * (uint64_t)p.S;
          draw_row<8>(w, keys, (erow + (uint64_t)key0) >> 3, p.stream);
        }
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          const int key = key0 + 8 * g + 2 * c;
          const float pr0 = (q_ok && key < seqlen) ? ex2_approx(fmaf(s[4 * g + 2 * h], c_scale, -lse2)) : 0.f;
          const float pr1 = (q_ok && key + 1 < seqlen) ? ex2_approx(fmaf(s[4 * g + 2 * h + 1], c_scale, -lse2)) : 0.f;
          bool ka = true, kb2 = true;
          if (drop) keep_pair(w[g], p.thresh16, ka, kb2);
          const float dp0 = ka ? dp[4 * g + 2 * h] * p.inv_keep : 0.f;
          const float dp1 = kb2 ? dp[4 * g + 2 * h + 1] * p.inv_keep : 0.f;
          const uint32_t pd = pack_bf16(ka ? pr0 * p.inv_keep : 0.f, kb2 ? pr1 * p.inv_keep : 0.f);
          const uint32_t ds = pack_bf16(pr0 * (dp0 - dlt) * p.scale, pr1 * (dp1 - dlt) * p.scale);
          dsp[h][g] = ds;
          *reinterpret_cast<uint32_t*>(myP + tile_pair_offset(r, g, c)) = pd;
          *reinterpret_cast<uint32_t*>(myDS + tile_pair_offset(r, g, c)) = ds;
        }
      }
      fence_proxy_async();                   // generic-proxy smem writes -> visible to wgmma (async proxy)
      asm volatile("bar.sync %0, 128;" ::"r"(wg + 1) : "memory");
      float dq[32];
      wgmma_fence_regs(dv);
      wgmma_fence_regs(dk);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < QT / 16; ++kk) { // reduction over the 64 queries: P~ / dS and dO / Q all read MN-major
        WgmmaBf16SS<64, 1, 1>::mma(dv, wgmma_desc_sw128(ap + kk * 2048, 8192, 1024), wgmma_desc_sw128(ado + kk * 2048, 8192, 1024), 1);
        WgmmaBf16SS<64, 1, 1>::mma(dk, wgmma_desc_sw128(ads + kk * 2048, 8192, 1024), wgmma_desc_sw128(aq + kk * 2048, 8192, 1024), 1);
      }
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {       // dQ (partial: this warpgroup's 64 keys) = dS K
        const uint32_t a[4] = {dsp[0][2 * kk], dsp[1][2 * kk], dsp[0][2 * kk + 1], dsp[1][2 * kk + 1]};
        WgmmaBf16RS<64, 1>::mma(dq, a, wgmma_desc_sw128(ak + kk * 2048, 8192, 1024), kk > 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(dv);
      wgmma_fence_regs(dk);
      wgmma_fence_regs(dq);
      // dQ: warpgroup w stores columns [32 w, 32 w + 32).  It hands the other half of its partial to the other
      // warpgroup through its own P~ buffer (its MMAs are done with it), fragment-major so the reads match lanes.
      float* give = reinterpret_cast<float*>(myP);
      float mine[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        give[k * 128 + tw] = wg ? dq[k] : dq[16 + k];
        mine[k] = wg ? dq[16 + k] : dq[k];
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 16; ++k) mine[k] = __fadd_rn(__fadd_rn(0.f, mine[k]), otherDq[k * 128 + tw]);
      const size_t q_off = (size_t)(row0 + i * QT) * ld + head * HD + wg * 32;
      store_cols64<1>(mine, 1.f, 1.f, r_lo, q_end - i * QT, p.dqkv + q_off, ld, p.f8, q_off, qscale, amax);
      __syncthreads();                       // both warpgroups are done with stage st and with the P~ buffers
      if (threadIdx.x == 0) issue_job();
    }
    // dK -> k slots, dV -> v slots of dqkv (rows = keys of this warpgroup)
    const size_t k_off = (size_t)(row0 + key0) * ld + p.H + head * HD;
    store_tile64(dk, 1.f, 1.f, r_lo, q_end - key0, p.dqkv + k_off, ld, p.f8, k_off, qscale, amax);
    store_tile64(dv, 1.f, 1.f, r_lo, q_end - key0, p.dqkv + k_off + p.H, ld, p.f8, k_off + p.H, qscale, amax);
    __syncthreads();                         // K / V stage n & 1 is free
    if (threadIdx.x == 0) issue_kv();
  }
  if (p.f8.q) fp8_amax_commit(p.f8, amax);
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
// head_dim 64, S <= 512 and S % 8 == 0 are checked by the bindings
static void fill_args(AttnArgs& a, int B, int S, int h, int d, const int* seqlens, float scale,
                      Seed seed, unsigned int stream, float p_drop) {
  a.B = B; a.S = S; a.h = h; a.H = h * d; a.seqlens = seqlens; a.scale = scale; a.seed = seed; a.stream = stream;
  a.thresh16 = p_drop > 0.f ? (unsigned)(p_drop * 65536.f + 0.5f) : 0u;
  a.inv_keep = p_drop > 0.f ? 65536.f / (65536.f - (float)a.thresh16) : 1.f;
  a.ctx = nullptr; a.lse = nullptr; a.delta = nullptr; a.dqkv = nullptr; a.dq_acc = nullptr;
}

template <bool VARLEN>
static void launch_fwd(const void* qkv, const AttnArgs& a, long long rows, cudaStream_t st) {
  const int S = a.S, H = a.H;
  CUtensorMap tq = make_tmap_2d_bf16(qkv, 3 * H, (uint64_t)rows, 3 * H, 64, QT);
  CUtensorMap tkv = make_tmap_2d_bf16(qkv, 3 * H, (uint64_t)rows, 3 * H, 64, KT);
  const int nkb = (S + KT - 1) / KT;
  const int smem = 8192 + nkb * 32768 + 1024 + 64;
  static int configured = 0;
  if (smem > configured) {
    B200_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_kernel<VARLEN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = smem;
  }
  attn_fwd_kernel<VARLEN><<<dim3((S + QT - 1) / QT, a.B * a.h), 128, smem, st>>>(tq, tkv, a);
}

void attention_fwd(const void* qkv, const int* seqlens, void* ctx, float* lse, int B, int S, int h, int d,
                   float scale, Seed seed, unsigned int stream, float p_drop, Fp8Out f8, cudaStream_t st,
                   const int* cu_seqlens, long long T) {
  AttnArgs a;
  fill_args(a, B, S, h, d, cu_seqlens ? cu_seqlens : seqlens, scale, seed, stream, p_drop);
  a.ctx = (__nv_bfloat16*)ctx; a.lse = lse; a.f8 = f8;
  if (cu_seqlens) launch_fwd<true>(qkv, a, T, st);
  else launch_fwd<false>(qkv, a, (long long)B * S, st);
}

template <bool VARLEN>
static void launch_bwd_onepass(const void* qkv, const void* ctx, const void* dctx, const AttnArgs& a, long long rows,
                               cudaStream_t st) {
  const int H = a.H;
  CUtensorMap tq = make_tmap_2d_bf16(qkv, 3 * H, (uint64_t)rows, 3 * H, 64, QT);
  CUtensorMap tkv = make_tmap_2d_bf16(qkv, 3 * H, (uint64_t)rows, 3 * H, 64, KT);
  CUtensorMap td = make_tmap_2d_bf16(dctx, H, (uint64_t)rows, H, 64, QT);
  CUtensorMap to = make_tmap_2d_bf16(ctx, H, (uint64_t)rows, H, 64, QT);
  static int resident = 0;                                // CTAs of the kernel one SM holds
  if (resident == 0) {
    B200_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_onepass_kernel<VARLEN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         ATT_OP_SMEM));
    B200_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, attn_bwd_onepass_kernel<VARLEN>,
                                                                  ATT_BWD_THREADS, ATT_OP_SMEM));
    if (resident < 1) { fprintf(stderr, "[b200] attn_bwd_onepass_kernel does not fit on an SM\n"); abort(); }
  }
  const long long items = (long long)a.B * a.h;
  const int grid = (int)std::min<long long>(items, (long long)num_sms() * resident);
  if (grid > 0) attn_bwd_onepass_kernel<VARLEN><<<grid, ATT_BWD_THREADS, ATT_OP_SMEM, st>>>(tq, tkv, td, to, a);
}

template <bool VARLEN>
static void launch_bwd(const void* qkv, const void* ctx, const void* dctx, const AttnArgs& a, long long rows,
                       cudaStream_t st, bool deterministic) {
  const int B = a.B, S = a.S, h = a.h, H = a.H;
  const int nkb = (S + KT - 1) / KT;
  const bool sliced = deterministic && nkb > 1;           // dq_acc then holds nkb slices of [rows, H]
  const long long groups = (long long)B * S * h;
  attn_delta_kernel<VARLEN><<<(unsigned)((groups * 8 + 255) / 256), 256, 0, st>>>(
      (const __nv_bfloat16*)ctx, (const __nv_bfloat16*)dctx, const_cast<float*>(a.delta), B, S, h, H, a.seqlens);
  B200_CUDA_CHECK(cudaMemsetAsync(a.dq_acc, 0, sizeof(float) * (size_t)(sliced ? nkb : 1) * rows * H, st));
  CUtensorMap tq = make_tmap_2d_bf16(qkv, 3 * H, (uint64_t)rows, 3 * H, 64, QT);
  CUtensorMap tkv = make_tmap_2d_bf16(qkv, 3 * H, (uint64_t)rows, 3 * H, 64, KT);
  CUtensorMap td = make_tmap_2d_bf16(dctx, H, (uint64_t)rows, H, 64, QT);
  static bool once = false;
  if (!once) {
    B200_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_kernel<VARLEN>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_BWD_SMEM));
    B200_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_sliced_kernel<VARLEN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         ATT_BWD_SMEM));
    once = true;
  }
  if (sliced)
    attn_bwd_sliced_kernel<VARLEN><<<dim3(nkb, B * h), ATT_BWD_THREADS, ATT_BWD_SMEM, st>>>(tq, tkv, td, a, rows * H);
  else
    attn_bwd_kernel<VARLEN><<<dim3(nkb, B * h), ATT_BWD_THREADS, ATT_BWD_SMEM, st>>>(tq, tkv, td, a);
  const long long work = rows * (H / 8);
  int g = (int)((work + 255) / 256);
  if (g > num_sms() * 16) g = num_sms() * 16;
  if (sliced) attn_dq_convert_sliced_kernel<<<g, 256, 0, st>>>(a.dq_acc, a.dqkv, rows, H, a.f8, nkb);
  else attn_dq_convert_kernel<<<g, 256, 0, st>>>(a.dq_acc, a.dqkv, rows, H, a.f8);
}

bool attention_bwd_onepass(int S, bool force_general) { return S <= KT && !force_general; }

void attention_bwd(const void* qkv, const int* seqlens, const void* ctx, const void* dctx, const float* lse,
                   void* dqkv, float* delta_ws, float* dq_acc, int B, int S, int h, int d, float scale,
                   Seed seed, unsigned int stream, float p_drop, Fp8Out f8, cudaStream_t st,
                   const int* cu_seqlens, long long T, bool deterministic, bool force_general) {
  AttnArgs a;
  fill_args(a, B, S, h, d, cu_seqlens ? cu_seqlens : seqlens, scale, seed, stream, p_drop);
  a.f8 = f8;
  a.lse = const_cast<float*>(lse); a.delta = delta_ws; a.dqkv = (__nv_bfloat16*)dqkv; a.dq_acc = dq_acc;
  a.ctx = (__nv_bfloat16*)const_cast<void*>(ctx);
  if (attention_bwd_onepass(S, force_general)) {
    if (cu_seqlens) launch_bwd_onepass<true>(qkv, ctx, dctx, a, T, st);
    else launch_bwd_onepass<false>(qkv, ctx, dctx, a, (long long)B * S, st);
    return;
  }
  if (dq_acc == nullptr || delta_ws == nullptr) {
    fprintf(stderr, "[b200] attention_bwd needs delta and dq accumulation buffers\n");
    abort();
  }
  if (cu_seqlens) launch_bwd<true>(qkv, ctx, dctx, a, T, st, deterministic);
  else launch_bwd<false>(qkv, ctx, dctx, a, (long long)B * S, st, deterministic);
}

}  // namespace b200
