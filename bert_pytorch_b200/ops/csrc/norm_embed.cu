// Bandwidth-bound kernels around the GEMMs: LayerNorm forward/backward (with the dropout-masked copy of
// the gradient and all column reductions fused), embedding gather+LN+dropout forward and its backward
// scatter, MLM position compaction / row gather / scatter, column sums for bias gradients.
// (SURVEY.md K1-K3, K15, K18, K22 and their backward call sites; apex FusedLayerNorm contract N4:
// fp32 statistics, eps inside the sqrt.)
//
// Layout: one warp per row, lane l owns columns {c*256 + l*8 .. +7}, so per-column reductions over rows
// stay in registers of a fixed lane and 16-byte loads/stores are fully coalesced.
#include "common.cuh"
#include "kernels.h"

namespace b200 {

constexpr int LN_WARPS = 4;

template <int CHUNKS>
__device__ __forceinline__ void load_row(const __nv_bfloat16* p, int H, int lane, float (&v)[CHUNKS][8]) {
#pragma unroll
  for (int c = 0; c < CHUNKS; ++c) {
    const int col = c * 256 + lane * 8;
    if (col < H) {
      const uint4 u = *reinterpret_cast<const uint4*>(p + col);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 f = unpack_bf16(w[t]);
        v[c][2 * t] = f.x;
        v[c][2 * t + 1] = f.y;
      }
    } else {
#pragma unroll
      for (int t = 0; t < 8; ++t) v[c][t] = 0.f;
    }
  }
}
template <int CHUNKS>
__device__ __forceinline__ void store_row(__nv_bfloat16* p, int H, int lane, const float (&v)[CHUNKS][8]) {
#pragma unroll
  for (int c = 0; c < CHUNKS; ++c) {
    const int col = c * 256 + lane * 8;
    if (col < H)
      *reinterpret_cast<uint4*>(p + col) = make_uint4(pack_bf16(v[c][0], v[c][1]), pack_bf16(v[c][2], v[c][3]),
                                                      pack_bf16(v[c][4], v[c][5]), pack_bf16(v[c][6], v[c][7]));
  }
}
template <int CHUNKS>
__device__ __forceinline__ void load_vec_f32(const float* p, int H, int lane, float (&v)[CHUNKS][8]) {
#pragma unroll
  for (int c = 0; c < CHUNKS; ++c) {
    const int col = c * 256 + lane * 8;
    if (col < H) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(p + col));
      const float4 b = __ldg(reinterpret_cast<const float4*>(p + col + 4));
      v[c][0] = a.x; v[c][1] = a.y; v[c][2] = a.z; v[c][3] = a.w;
      v[c][4] = b.x; v[c][5] = b.y; v[c][6] = b.z; v[c][7] = b.w;
    } else {
#pragma unroll
      for (int t = 0; t < 8; ++t) v[c][t] = 0.f;
    }
  }
}

template <int CHUNKS>
__device__ __forceinline__ void row_stats(const float (&x)[CHUNKS][8], int H, int lane, float eps, float& mean,
                                          float& rstd) {
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < CHUNKS; ++c)
#pragma unroll
    for (int t = 0; t < 8; ++t) s += x[c][t];
  mean = warp_sum(s) / (float)H;
  float q = 0.f;
#pragma unroll
  for (int c = 0; c < CHUNKS; ++c) {
    const int col = c * 256 + lane * 8;
    if (col < H) {
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const float d = x[c][t] - mean;
        q += d * d;
      }
    }
  }
  rstd = rsqrtf(warp_sum(q) / (float)H + eps);
}

// 16-byte streaming load (read once: do not keep it in L1)
__device__ __forceinline__ uint4 ld_stream16(const __nv_bfloat16* p) {
  uint4 u;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(p));
  return u;
}
__device__ __forceinline__ void unpack8(const uint4& u, float (&v)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const float2 f = unpack_bf16(w[t]);
    v[2 * t] = f.x;
    v[2 * t + 1] = f.y;
  }
}
__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const float2 f = unpack_bf16(w[t]);
    v[2 * t] = f.x;
    v[2 * t + 1] = f.y;
  }
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&v)[8]) {
  *reinterpret_cast<uint4*>(p) = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]),
                                            pack_bf16(v[6], v[7]));
}

// ------------------------------------------------------------------------------------------------
// LayerNorm forward / backward.  Both are instruction bound at these sizes (per-row reductions and address arithmetic
// amortised over few elements per lane), so they keep the instructions per element low:
//   forward : one warp owns a whole row (8 columns per lane and 256-column chunk): shuffle-only statistics, exact
//             two-pass variance in registers, gamma / beta from shared memory (conflict-free float4 layout)
//   backward: WPR warps share a row and every lane owns 8 columns (the column sums for dgamma / dbeta / dbias stay in
//             registers of a fixed lane), the per-row constants are folded into two FFMAs per element, one 64-bit
//             Philox counter computation per row.
// TAIL = false: H is CHUNKS * 256 (WPR * 256) at compile time, no bounds predicates.  TAIL = true: H (a multiple of 8)
// is a kernel argument and the 8-column groups at or past H are predicated off.  FP8: the fp8 copy of the output
// (Fp8Out) is written in the same pass.
// ------------------------------------------------------------------------------------------------
template <int CHUNKS, bool TAIL, bool FP8>
__global__ void __launch_bounds__(256)
ln_fwd_row_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                  __nv_bfloat16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, int M,
                  float eps, int h, const Fp8Out f8) {
  const int H = TAIL ? h : CHUNKS * 256;
  __shared__ float4 sg[CHUNKS][2][32], sb[CHUNKS][2][32];   // [chunk][half of the lane's 8 columns][lane]
  for (int i = threadIdx.x; i < CHUNKS * 64; i += blockDim.x) {
    const int c = i >> 6, hf = (i >> 5) & 1, l = i & 31;
    const int col = c * 256 + l * 8 + hf * 4;
    if (!TAIL || col < H) {
      sg[c][hf][l] = __ldg(reinterpret_cast<const float4*>(gamma + col));
      sb[c][hf][l] = __ldg(reinterpret_cast<const float4*>(beta + col));
    }
  }
  __syncthreads();
  const float qscale = FP8 ? f8.meta[1] : 0.f;
  float amax = 0.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int lane_cols = H - lane * 8;      // chunk c of this lane lies inside the row iff c * 256 < lane_cols
  auto live = [&](int c) { return !TAIL || c * 256 < lane_cols; };
  const int stride = gridDim.x * 8;
  int row = blockIdx.x * 8 + warp;
  uint4 nx[CHUNKS];
  if constexpr (TAIL) {                    // columns past H read as zeros: they add nothing to the row sum
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) nx[c] = make_uint4(0, 0, 0, 0);
  }
  if (row < M) {
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c)
      if (live(c)) nx[c] = ld_stream16(x + (size_t)row * H + c * 256 + lane * 8);
  }
  for (; row < M; row += stride) {
    float v[CHUNKS][8];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) unpack8(nx[c], v[c]);
    const int nrow = row + stride;
    if (nrow < M) {                        // next row in flight while this one is reduced
#pragma unroll
      for (int c = 0; c < CHUNKS; ++c)
        if (live(c)) nx[c] = ld_stream16(x + (size_t)nrow * H + c * 256 + lane * 8);
    }
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c)
#pragma unroll
      for (int t = 0; t < 8; ++t) s += v[c][t];
    // a true division: a row of equal values then has its own value as mean and a variance of exactly 0 (the sum is
    // exact, but sum * (1/H) can land one ulp off for H not a power of two, which rstd ~ 1/sqrt(eps) turns into
    // an error of order 0.1 * gamma)
    const float mean = warp_sum(s) / (float)H;
    float q = 0.f;
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c)
      if (live(c)) {
#pragma unroll
        for (int t = 0; t < 8; ++t) { v[c][t] -= mean; q = fmaf(v[c][t], v[c][t], q); }
      }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / (float)H) + eps);
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
      if (!live(c)) continue;
      const float4 g0 = sg[c][0][lane], g1 = sg[c][1][lane], b0 = sb[c][0][lane], b1 = sb[c][1][lane];
      const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int t = 0; t < 8; ++t) v[c][t] = fmaf(v[c][t] * rstd, g[t], b[t]);
      store8(y + (size_t)row * H + c * 256 + lane * 8, v[c]);
      if constexpr (FP8) fp8_emit8(f8, (size_t)row * H + c * 256 + lane * 8, v[c], qscale, amax);
    }
    if (lane == 0) {
      if (mean_out) mean_out[row] = mean;
      if (rstd_out) rstd_out[row] = rstd;
    }
  }
  if constexpr (FP8) fp8_amax_commit(f8, amax);
}

// LayerNorm backward, GROUPS rows per block at a time.
//   in : dy [M,H] grad wrt the LN output; with `in_stream` given (TAIL instantiations only), dy is first multiplied by
//        the output dropout of that stream -- the embedding LN, whose output was dropped out
//        x [M,H] pre-LN input, mean / rstd [M], gamma [H]
//   out: dx [M,H]  grad wrt the pre-LN input (also the residual-branch gradient)
//        dxd [M,H] optional: dx * dropout_mask(stream `drop_stream`) * scale, the gradient of the GEMM output that was
//                  dropped out before the residual add.  The keep decisions are READ from `keep_mask` (one byte per 8
//                  elements, written by dropout_mask_kernel or by the producing GEMM epilogue: GemmCall::mask_out)
//                  instead of regenerated with Philox whenever the caller has them.
//        partial [grid, 3, H]: per-block column sums of (dy * xhat, dy, dxd) -> dgamma, dbeta, dbias
template <int WPR, int GROUPS, bool TAIL, bool FP8>
__global__ void __launch_bounds__(GROUPS * WPR * 32)
ln_bwd3_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
               const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
               __nv_bfloat16* __restrict__ dx, __nv_bfloat16* __restrict__ dxd, float* __restrict__ partial, int M,
               Seed seed_in, unsigned int drop_stream, unsigned int thresh16, float drop_scale,
               const uint8_t* __restrict__ keep_mask, int h, unsigned int in_stream, const Fp8Out f8) {
  const int H = TAIL ? h : WPR * 256;
  __shared__ float2 xchg[GROUPS][2][WPR];
  __shared__ float comb[GROUPS - 1 > 0 ? GROUPS - 1 : 1][3][WPR * 256];
  const unsigned long long seed = thresh16 != 0 ? seed_in.value() : 0ull;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int group = warp / WPR, wi = warp % WPR;
  const int col = (wi * 32 + lane) * 8;
  const bool live = !TAIL || col < H;      // this lane's 8 columns lie inside the row
  const bool in_drop = TAIL && in_stream != 0xFFFFFFFFu && thresh16 != 0;
  const float qscale = FP8 ? f8.meta[1] : 0.f;
  float amax = 0.f;
  f32x2 g2[4], ag2[4], ab2[4], ad2[4];
  {
    float4 g0 = make_float4(0.f, 0.f, 0.f, 0.f), g1 = g0;
    if (live) {
      g0 = __ldg(reinterpret_cast<const float4*>(gamma + col));
      g1 = __ldg(reinterpret_cast<const float4*>(gamma + col + 4));
    }
    g2[0] = f2_pack(g0.x, g0.y); g2[1] = f2_pack(g0.z, g0.w); g2[2] = f2_pack(g1.x, g1.y); g2[3] = f2_pack(g1.z, g1.w);
  }
#pragma unroll
  for (int t = 0; t < 4; ++t) ag2[t] = ab2[t] = ad2[t] = f2_splat(0.f);
  const int stride = gridDim.x * GROUPS;
  int row = blockIdx.x * GROUPS + group;
  uint4 nd = make_uint4(0, 0, 0, 0), nv = make_uint4(0, 0, 0, 0);
  float nmu = 0.f, nrs = 0.f;
  uint32_t nmask = 0;
  const bool use_mask = keep_mask != nullptr && dxd != nullptr && thresh16 != 0;
  if (row < M) {                           // columns past H read as zeros: they add nothing to the sums
    if (live) {
      nd = ld_stream16(dy + (size_t)row * H + col);
      nv = ld_stream16(x + (size_t)row * H + col);
    }
    nmu = __ldg(mean + row);
    nrs = __ldg(rstd + row);
    if (use_mask && live) nmask = __ldg(keep_mask + (size_t)row * (H / 8) + (col >> 3));
  }
  const float invH = 1.0f / (float)H;
  for (int it = 0; row < M; row += stride, ++it) {
    const uint32_t dw[4] = {nd.x, nd.y, nd.z, nd.w}, vw[4] = {nv.x, nv.y, nv.z, nv.w};
    const float rs = nrs, nmr = -nmu * nrs;
    const uint32_t mask = nmask;
    const int nrow = row + stride;
    if (nrow < M) {                        // next row's loads are in flight across this row's barrier
      if (live) {
        nd = ld_stream16(dy + (size_t)nrow * H + col);
        nv = ld_stream16(x + (size_t)nrow * H + col);
      }
      nmu = __ldg(mean + nrow);
      nrs = __ldg(rstd + nrow);
      if (use_mask && live) nmask = __ldg(keep_mask + (size_t)nrow * (H / 8) + (col >> 3));
    }
    Keep8 in_keep = Keep8::all();
    if (in_drop) in_keep = dropout_keep8(seed, in_stream, (uint64_t)row * (uint64_t)(H / 8) + (uint64_t)(col >> 3), thresh16);
    const f32x2 rs2 = f2_splat(rs), nmr2 = f2_splat(nmr);
    f32x2 xh[4], dg[4], s1p = f2_splat(0.f), s2p = f2_splat(0.f);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      f32x2 d = f2_from_bf16x2(dw[t]);
      if (in_drop) d = f2_mul(d, f2_pack(in_keep[2 * t] ? drop_scale : 0.f, in_keep[2 * t + 1] ? drop_scale : 0.f));
      xh[t] = f2_fma(f2_from_bf16x2(vw[t]), rs2, nmr2);
      dg[t] = f2_mul(d, g2[t]);
      ag2[t] = f2_fma(d, xh[t], ag2[t]);
      ab2[t] = f2_add(ab2[t], d);
      s1p = f2_add(s1p, dg[t]);
      s2p = f2_fma(dg[t], xh[t], s2p);
    }
    // row sums across the WPR warps of this group: one named barrier per row, slots double buffered by parity
    const float2 s1f = f2_unpack(s1p), s2f = f2_unpack(s2p);
    float s1 = warp_sum(s1f.x + s1f.y);
    float s2 = warp_sum(s2f.x + s2f.y);
    if (WPR > 1) {
      float2* slot = xchg[group][it & 1];
      if (lane == 0) slot[wi] = make_float2(s1, s2);
      asm volatile("bar.sync %0, %1;" ::"r"(group + 1), "n"(WPR * 32) : "memory");
      s1 = 0.f; s2 = 0.f;
#pragma unroll
      for (int w = 0; w < WPR; ++w) { const float2 u = slot[w]; s1 += u.x; s2 += u.y; }
    }
    const f32x2 c1 = f2_splat(-rs * s1 * invH), c2 = f2_splat(-rs * s2 * invH);
    f32x2 o[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) o[t] = f2_fma(xh[t], c2, f2_fma(dg[t], rs2, c1));   // rs (dg - mean(dg) - xh mean(dg xh))
    if (!live) continue;
    const size_t off = (size_t)row * H + col;
    *reinterpret_cast<uint4*>(dx + off) = make_uint4(f2_to_bf16x2(o[0]), f2_to_bf16x2(o[1]), f2_to_bf16x2(o[2]), f2_to_bf16x2(o[3]));
    if (dxd != nullptr) {
      if (thresh16 != 0) {
        if (use_mask) {
#pragma unroll
          for (int t = 0; t < 4; ++t)
            o[t] = f2_mul(o[t], f2_pack((mask >> (2 * t)) & 1u ? drop_scale : 0.f, (mask >> (2 * t + 1)) & 1u ? drop_scale : 0.f));
        } else {
          const Keep8 keep = dropout_keep8(seed, drop_stream, (uint64_t)row * (uint64_t)(H / 8) + (uint64_t)(col >> 3), thresh16);
#pragma unroll
          for (int t = 0; t < 4; ++t)
            o[t] = f2_mul(o[t], f2_pack(keep[2 * t] ? drop_scale : 0.f, keep[2 * t + 1] ? drop_scale : 0.f));
        }
      }
#pragma unroll
      for (int t = 0; t < 4; ++t) ad2[t] = f2_add(ad2[t], o[t]);
      *reinterpret_cast<uint4*>(dxd + off) = make_uint4(f2_to_bf16x2(o[0]), f2_to_bf16x2(o[1]), f2_to_bf16x2(o[2]), f2_to_bf16x2(o[3]));
      if constexpr (FP8) {
        float r[8];
#pragma unroll
        for (int t = 0; t < 4; ++t) { r[2 * t] = o[t].x; r[2 * t + 1] = o[t].y; }
        fp8_emit8(f8, off, r, qscale, amax);
      }
    }
  }
  if constexpr (FP8) fp8_amax_commit(f8, amax);
  float ag[8], ab[8], ad[8];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const float2 a = f2_unpack(ag2[t]), b = f2_unpack(ab2[t]), c = f2_unpack(ad2[t]);
    ag[2 * t] = a.x; ag[2 * t + 1] = a.y; ab[2 * t] = b.x; ab[2 * t + 1] = b.y; ad[2 * t] = c.x; ad[2 * t + 1] = c.y;
  }
  // combine the row groups of the block in shared memory, then one atomic per column and quantity
  if (GROUPS > 1) {
    if (group > 0) {
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        comb[group - 1][0][col + t] = ag[t];
        comb[group - 1][1][col + t] = ab[t];
        comb[group - 1][2][col + t] = ad[t];
      }
    }
    __syncthreads();
    if (group == 0) {
#pragma unroll
      for (int gidx = 0; gidx < GROUPS - 1; ++gidx)
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          ag[t] += comb[gidx][0][col + t];
          ab[t] += comb[gidx][1][col + t];
          ad[t] += comb[gidx][2][col + t];
        }
    }
  }
  if (group == 0 && live) {   // per-block partial column sums; colsum_finalize_kernel adds them into the gradient arena
    // (444 blocks x 3072 same-address atomics at the end of the kernel serialise in L2: measured 2x slower)
    float* dst = partial + (size_t)blockIdx.x * 3 * H + col;
    *reinterpret_cast<float4*>(dst) = make_float4(ag[0], ag[1], ag[2], ag[3]);
    *reinterpret_cast<float4*>(dst + 4) = make_float4(ag[4], ag[5], ag[6], ag[7]);
    *reinterpret_cast<float4*>(dst + H) = make_float4(ab[0], ab[1], ab[2], ab[3]);
    *reinterpret_cast<float4*>(dst + H + 4) = make_float4(ab[4], ab[5], ab[6], ab[7]);
    *reinterpret_cast<float4*>(dst + 2 * H) = make_float4(ad[0], ad[1], ad[2], ad[3]);
    *reinterpret_cast<float4*>(dst + 2 * H + 4) = make_float4(ad[4], ad[5], ad[6], ad[7]);
  }
}

// dst[k][col] += sum over blocks of partial[block][k][col]   (k = 0..2, any dst may be null)
// grid (ceil(H/32), 3, Z), 256 threads: warp w sums rows w, w+8, ... of a 32-column strip (coalesced 128 B
// per row), then the 8 warps are combined through shared memory.  Z > 1 cuts the partial rows into Z slices that
// finish with an atomic add: the kernel is a chain of ~55 dependent loads per warp at Z = 1 (8 us for 444 partial
// rows), i.e. latency bound.
__global__ void __launch_bounds__(256)
colsum_finalize_kernel(const float* __restrict__ partial, int nblocks, int H, float* dgamma, float* dbeta,
                       float* dbias) {
  const int qn = blockIdx.y;
  float* dst = qn == 0 ? dgamma : (qn == 1 ? dbeta : dbias);
  if (dst == nullptr) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int col = blockIdx.x * 32 + lane;
  float s = 0.f;
  if (col < H) {
    const int per = (nblocks + gridDim.z - 1) / gridDim.z;
    const int b_lo = blockIdx.z * per, b_hi = min(nblocks, b_lo + per);
#pragma unroll 4
    for (int b = b_lo + warp; b < b_hi; b += 8) s += partial[((size_t)b * 3 + qn) * H + col];
  }
  __shared__ float sm[8][32];
  sm[warp][lane] = s;
  __syncthreads();
  if (warp == 0 && col < H) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += sm[w][lane];
    if (gridDim.z == 1) dst[col] += t;
    else atomicAdd(dst + col, t);
  }
}

// ------------------------------------------------------------------------------------------------
// column sum of a bf16 matrix into an fp32 vector (bias gradients): out[n] += sum_m x[m][n]
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) colsum_bf16_kernel(const __nv_bfloat16* __restrict__ x, int M, int N, int ld,
                                                         float* __restrict__ out) {
  // block: 32 column-groups (8 cols each = 256 columns) x 8 row lanes
  const int cg = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int col = blockIdx.x * 256 + cg * 8;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (col < N) {
    for (int row = blockIdx.y * 8 + rl; row < M; row += gridDim.y * 8) {
      const uint4 u = *reinterpret_cast<const uint4*>(x + (size_t)row * ld + col);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 f = unpack_bf16(w[t]);
        acc[2 * t] += f.x;
        acc[2 * t + 1] += f.y;
      }
    }
  }
  __shared__ float sm[8][256];
#pragma unroll
  for (int t = 0; t < 8; ++t) sm[rl][cg * 8 + t] = acc[t];
  __syncthreads();
  const int c = threadIdx.x;
  float s = 0.f;
#pragma unroll
  for (int r = 0; r < 8; ++r) s += sm[r][c];
  if (blockIdx.x * 256 + c < N) atomicAdd(out + blockIdx.x * 256 + c, s);
}

// ------------------------------------------------------------------------------------------------
// GELU as bandwidth kernels.  With K = 1024 the FFN-1 / FFN-2-dgrad GEMM tiles give the epilogue only
// ~8k cycles for 32k elements; erf-GELU (~20 instructions per element on 4 issue ports) does not fit under
// that main loop (measured in situ: 192 us and 202 us per GEMM instead of ~83), so the activation runs here
// where the instruction budget per byte is 10x larger: one pass at HBM speed forward, and the backward pass
// also produces the FFN-1 bias gradient (column sums) that used to be a separate kernel.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gelu_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                      long long n8, const Fp8Out f8) {
  const float qscale = f8.q ? f8.meta[1] : 0.f;
  float amax = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const uint4 u = reinterpret_cast<const uint4*>(x)[i];
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    uint32_t o[4];
    float r[8];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 f = unpack_bf16(w[t]);
      r[2 * t] = gelu_erf(f.x);
      r[2 * t + 1] = gelu_erf(f.y);
      o[t] = pack_bf16(r[2 * t], r[2 * t + 1]);
    }
    reinterpret_cast<uint4*>(y)[i] = make_uint4(o[0], o[1], o[2], o[3]);
    if (f8.q) fp8_emit8(f8, (size_t)i * 8, r, qscale, amax);
  }
  if (f8.q) fp8_amax_commit(f8, amax);
}

// dx[m][n] = dy[m][n] * gelu'(x[m][n]);  dbias[n] += sum_m dx[m][n] (the fp32 products, before the bf16 rounding)
// PART (deterministic mode): block (x, y) stores its column sums to dbias[y * N + col] for ordered_sum instead
template <bool PART>
__device__ __forceinline__ void dgelu_bwd_body(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                               __nv_bfloat16* __restrict__ dx, float* __restrict__ dbias, int M, int N,
                                               const Fp8Out& f8) {
  const int cg = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int col = blockIdx.x * 256 + cg * 8;
  const float qscale = f8.q ? f8.meta[1] : 0.f;
  float amax = 0.f;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (col < N) {
    auto body = [&](size_t off, const uint4& a, const uint4& b) {
      const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
      uint32_t o[4];
      float r[8];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 g = unpack_bf16(aw[t]), v = unpack_bf16(bw[t]);
        const float r0 = g.x * dgelu_erf(v.x), r1 = g.y * dgelu_erf(v.y);
        acc[2 * t] += r0;
        acc[2 * t + 1] += r1;
        r[2 * t] = r0; r[2 * t + 1] = r1;
        o[t] = pack_bf16(r0, r1);
      }
      *reinterpret_cast<uint4*>(dx + off) = make_uint4(o[0], o[1], o[2], o[3]);
      if (f8.q) fp8_emit8(f8, off, r, qscale, amax);
    };
    // two rows per iteration: four 16-byte loads in flight per thread (the kernel is latency bound otherwise)
    const int stride = gridDim.y * 8;
    int row = blockIdx.y * 8 + rl;
    for (; row + stride < M; row += 2 * stride) {
      const size_t off0 = (size_t)row * N + col, off1 = (size_t)(row + stride) * N + col;
      const uint4 a0 = ld_stream16(dy + off0), b0 = ld_stream16(x + off0);
      const uint4 a1 = ld_stream16(dy + off1), b1 = ld_stream16(x + off1);
      body(off0, a0, b0);
      body(off1, a1, b1);
    }
    if (row < M) {
      const size_t off = (size_t)row * N + col;
      body(off, ld_stream16(dy + off), ld_stream16(x + off));
    }
  }
  if (f8.q) fp8_amax_commit(f8, amax);
  if (dbias == nullptr) return;
  __shared__ float sm[8][256];
#pragma unroll
  for (int t = 0; t < 8; ++t) sm[rl][cg * 8 + t] = acc[t];
  __syncthreads();
  const int c = threadIdx.x;
  float sum = 0.f;
#pragma unroll
  for (int r = 0; r < 8; ++r) sum += sm[r][c];
  if constexpr (PART) { if (blockIdx.x * 256 + c < N) dbias[(size_t)blockIdx.y * N + blockIdx.x * 256 + c] = sum; }
  else if (blockIdx.x * 256 + c < N) atomicAdd(dbias + blockIdx.x * 256 + c, sum);
}

__global__ void __launch_bounds__(256)
dgelu_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ dx,
                 float* __restrict__ dbias, int M, int N, const Fp8Out f8) {
  dgelu_bwd_body<false>(dy, x, dx, dbias, M, N, f8);
}

__global__ void __launch_bounds__(256)
dgelu_bwd_part_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                      __nv_bfloat16* __restrict__ dx, float* __restrict__ dbias_part, int M, int N, const Fp8Out f8) {
  dgelu_bwd_body<true>(dy, x, dx, dbias_part, M, N, f8);
}

// ------------------------------------------------------------------------------------------------
// Embedding forward: e = word[id] + pos[s] (+ type[seg]); y = dropout(LN(e)); saves e, mean, rstd.
// s = row % S for a padded [B, S] batch; POS_IDS: s = pos_ids[row] (packed rows of an unpadded batch).
// ------------------------------------------------------------------------------------------------
template <int CHUNKS, bool POS_IDS = false>
__global__ void __launch_bounds__(LN_WARPS * 32)
embed_fwd_kernel(const int* __restrict__ ids, const int* __restrict__ seg, const __nv_bfloat16* __restrict__ word,
                 const __nv_bfloat16* __restrict__ pos, const __nv_bfloat16* __restrict__ type,
                 const float* __restrict__ gamma, const float* __restrict__ beta, __nv_bfloat16* __restrict__ e_out,
                 __nv_bfloat16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, int M,
                 int S, int H, float eps, Seed seed_in, unsigned int stream, unsigned int thresh16,
                 float drop_scale, const int* __restrict__ pos_ids) {
  const unsigned long long seed = seed_in.value();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float g[CHUNKS][8], b[CHUNKS][8];
  load_vec_f32<CHUNKS>(gamma, H, lane, g);
  load_vec_f32<CHUNKS>(beta, H, lane, b);
  for (int row = blockIdx.x * LN_WARPS + warp; row < M; row += gridDim.x * LN_WARPS) {
    float v[CHUNKS][8], t0[CHUNKS][8];
    load_row<CHUNKS>(word + (size_t)ids[row] * H, H, lane, v);
    load_row<CHUNKS>(pos + (size_t)(POS_IDS ? pos_ids[row] : row % S) * H, H, lane, t0);
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c)
#pragma unroll
      for (int t = 0; t < 8; ++t) v[c][t] += t0[c][t];
    if (type != nullptr) {
      load_row<CHUNKS>(type + (size_t)seg[row] * H, H, lane, t0);
#pragma unroll
      for (int c = 0; c < CHUNKS; ++c)
#pragma unroll
        for (int t = 0; t < 8; ++t) v[c][t] += t0[c][t];
    }
    // round the sum to bf16 first so the saved copy and the statistics agree exactly
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c)
#pragma unroll
      for (int t = 0; t < 8; ++t) v[c][t] = __bfloat162float(__float2bfloat16(v[c][t]));
    store_row<CHUNKS>(e_out + (size_t)row * H, H, lane, v);
    float mean, rstd;
    row_stats<CHUNKS>(v, H, lane, eps, mean, rstd);
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
      const int col = c * 256 + lane * 8;
      Keep8 keep = Keep8::all();
      if (thresh16 != 0 && col < H) keep = dropout_keep8(seed, stream, ((uint64_t)row * H + col) >> 3, thresh16);
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        float o = (v[c][t] - mean) * rstd * g[c][t] + b[c][t];
        if (thresh16 != 0) o = keep[t] ? o * drop_scale : 0.f;
        v[c][t] = o;
      }
    }
    store_row<CHUNKS>(y + (size_t)row * H, H, lane, v);
    if (lane == 0) {
      mean_out[row] = mean;
      rstd_out[row] = rstd;
    }
  }
}

// Embedding backward scatter: de [M,H] (bf16) is added into the fp32 gradient tables (position row: pos_ids[row] when
// given, else row % S; token-type row seg[row], or 0 without segment ids).
__global__ void __launch_bounds__(256)
embed_bwd_scatter_kernel(const __nv_bfloat16* __restrict__ de, const int* __restrict__ ids,
                         const int* __restrict__ seg, float* __restrict__ gword, float* __restrict__ gpos,
                         float* __restrict__ gtype, int M, int S, int H, const int* __restrict__ pos_ids) {
  const int per_row = H / 8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)M * per_row;
       i += (size_t)gridDim.x * blockDim.x) {
    const int row = (int)(i / per_row), col = (int)(i % per_row) * 8;
    const uint4 u = *reinterpret_cast<const uint4*>(de + (size_t)row * H + col);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    float f[8];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 p = unpack_bf16(w[t]);
      f[2 * t] = p.x;
      f[2 * t + 1] = p.y;
    }
    float* dst[3] = {gword + (size_t)ids[row] * H + col,
                     gpos ? gpos + (size_t)(pos_ids ? pos_ids[row] : row % S) * H + col : nullptr,
                     gtype ? gtype + (size_t)(seg ? seg[row] : 0) * H + col : nullptr};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (dst[k] == nullptr) continue;
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst[k]), "f"(f[0]), "f"(f[1]), "f"(f[2]),
                   "f"(f[3]) : "memory");
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst[k] + 4), "f"(f[4]), "f"(f[5]),
                   "f"(f[6]), "f"(f[7]) : "memory");
    }
  }
}

// Position / token-type gradients as REDUCTIONS instead of atomics (12288 rows hammering the two token-type rows and
// 96 rows per position row serialise in L2).  Thread (s, 8 columns)
// walks the batch dimension: the position row s has exactly one owner (plain read-modify-write), the two token-type
// rows are reduced over the 8 positions of a block in shared memory and leave as one atomic per block and column.
__global__ void __launch_bounds__(256)
embed_bwd_postype_kernel(const __nv_bfloat16* __restrict__ de, const int* __restrict__ seg, float* __restrict__ gpos,
                         float* __restrict__ gtype, int B, int S, int H) {
  const int cg = threadIdx.x & 31, sl = threadIdx.x >> 5;
  const int col = blockIdx.x * 256 + cg * 8;
  const int s = blockIdx.y * 8 + sl;
  float ap[8], a1[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) ap[j] = a1[j] = 0.f;
  const bool live = col < H && s < S;
  if (live) {
#pragma unroll 4
    for (int b = 0; b < B; ++b) {
      const size_t row = (size_t)b * S + s;
      float f[8];
      unpack8(ld_stream16(de + row * H + col), f);
      const float m = (seg != nullptr && seg[row] != 0) ? 1.f : 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) { ap[j] += f[j]; a1[j] = fmaf(m, f[j], a1[j]); }
    }
    float4* gp = reinterpret_cast<float4*>(gpos + (size_t)s * H + col);
    float4 x = gp[0], y = gp[1];
    x.x += ap[0]; x.y += ap[1]; x.z += ap[2]; x.w += ap[3];
    y.x += ap[4]; y.y += ap[5]; y.z += ap[6]; y.w += ap[7];
    gp[0] = x; gp[1] = y;
  }
  if (gtype == nullptr) return;
  __shared__ float sm[2][8][256];
#pragma unroll
  for (int j = 0; j < 8; ++j) { sm[0][sl][cg * 8 + j] = live ? ap[j] - a1[j] : 0.f; sm[1][sl][cg * 8 + j] = live ? a1[j] : 0.f; }
  __syncthreads();
  const int c = threadIdx.x;
  if (blockIdx.x * 256 + c < H) {
    float t0 = 0.f, t1 = 0.f;
#pragma unroll
    for (int r = 0; r < 8; ++r) { t0 += sm[0][r][c]; t1 += sm[1][r][c]; }
    atomicAdd(gtype + blockIdx.x * 256 + c, t0);
    atomicAdd(gtype + H + blockIdx.x * 256 + c, t1);
  }
}

// ------------------------------------------------------------------------------------------------
// Deterministic mode (ops.api.deterministic()): fixed-order forms of the reductions above.  None of these kernels
// waits on another CTA; the order of every floating-point sum depends only on the shapes.
// ------------------------------------------------------------------------------------------------
constexpr int ORD_THREADS = 256;

// out[s * W + w] += sum over the rows r of segment s of part[r * W + w].  A block owns CW (a power of two <= 32)
// columns; its R = 256 / CW row lanes sum rows lo + j, lo + j + R, ... each, and a fixed binary tree combines the
// lanes.  Segment s is every row when row_seg is null (one segment), else the rows whose row_seg (ascending) is s.
__global__ void __launch_bounds__(ORD_THREADS)
ordered_sum_kernel(const float* __restrict__ part, int rows, int W, int CW, const int* __restrict__ row_seg,
                   float* __restrict__ out) {
  const int s = blockIdx.y;
  int lo = 0, hi = rows;
  if (row_seg != nullptr) {
    auto lower = [&](int v) {
      int a = 0, b = rows;
      while (a < b) { const int m = (a + b) >> 1; if (row_seg[m] < v) a = m + 1; else b = m; }
      return a;
    };
    lo = lower(s);
    hi = lower(s + 1);
  }
  const int cl = threadIdx.x & (CW - 1), rl = threadIdx.x / CW, R = ORD_THREADS / CW;
  const int w = blockIdx.x * CW + cl;
  float acc = 0.f;
  if (w < W) {
#pragma unroll 4
    for (int r = lo + rl; r < hi; r += R) acc += part[(size_t)r * W + w];
  }
  __shared__ float sm[ORD_THREADS];
  sm[threadIdx.x] = acc;
  __syncthreads();
  for (int half = R >> 1; half > 0; half >>= 1) {
    if (rl < half) sm[threadIdx.x] += sm[threadIdx.x + half * CW];
    __syncthreads();
  }
  if (rl == 0 && w < W) out[(size_t)s * W + w] += sm[cl];
}

// colsum_bf16_kernel with the block's column sums stored to part[blockIdx.y][N] instead of added to the output
__global__ void __launch_bounds__(256) colsum_bf16_part_kernel(const __nv_bfloat16* __restrict__ x, int M, int N, int ld,
                                                              float* __restrict__ part) {
  const int cg = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int col = blockIdx.x * 256 + cg * 8;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (col < N) {
    for (int row = blockIdx.y * 8 + rl; row < M; row += gridDim.y * 8) {
      float f[8];
      unpack8(*reinterpret_cast<const uint4*>(x + (size_t)row * ld + col), f);
#pragma unroll
      for (int t = 0; t < 8; ++t) acc[t] += f[t];
    }
  }
  __shared__ float sm[8][256];
#pragma unroll
  for (int t = 0; t < 8; ++t) sm[rl][cg * 8 + t] = acc[t];
  __syncthreads();
  const int c = threadIdx.x;
  float s = 0.f;
#pragma unroll
  for (int r = 0; r < 8; ++r) s += sm[r][c];
  if (blockIdx.x * 256 + c < N) part[(size_t)blockIdx.y * N + blockIdx.x * 256 + c] = s;
}

// Embedding backward as "sort, then one owner per table row".  sort_rows_kernel orders the token rows by table row:
// it sorts the unique keys table_row * M + token_row (bitonic, one CTA, in shared memory), so the rows of one table
// row end up adjacent and in token order.  sorted_piece_sum_kernel cuts the sorted rows into tiles of SORT_TILE; a
// piece (the rows of one table row inside one tile) is summed in order and stored at ws[first row of the piece].
// sorted_run_finish_kernel: the first sorted row of each table row adds the pieces of its run in order (one per tile
// the run touches) and does the single read-modify-write of that table row.  Long runs ([PAD] in a padded batch, the
// two token-type rows) thus cost one tile sum plus one add per tile rather than a serial walk.
constexpr int SORT_THREADS = 1024;
constexpr int SORT_CAP = 32768;       // token rows per sort: 128 KB of shared memory
constexpr int SORT_TILE = 64;

__global__ void __launch_bounds__(SORT_THREADS)
sort_rows_kernel(const int* __restrict__ key, int key_mod, int row0, int M, unsigned* __restrict__ out) {
  extern __shared__ unsigned sk[];
  int N = 1;
  while (N < M) N <<= 1;
  for (int i = threadIdx.x; i < N; i += SORT_THREADS)
    sk[i] = i < M ? (unsigned)(key != nullptr ? key[i] : (row0 + i) % key_mod) * (unsigned)M + (unsigned)i : 0xFFFFFFFFu;
  __syncthreads();
  for (int k = 2; k <= N; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < N; i += SORT_THREADS) {
        const int q = i ^ j;
        if (q > i) {
          const unsigned a = sk[i], b = sk[q];
          if ((a > b) == ((i & k) == 0)) { sk[i] = b; sk[q] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < M; i += SORT_THREADS) out[i] = sk[i];
}

// block: SORT_TILE sorted rows x 1024 columns (128 threads x 8)
__global__ void __launch_bounds__(128)
sorted_piece_sum_kernel(const __nv_bfloat16* __restrict__ de, const unsigned* __restrict__ sorted, int M, int H,
                        float* __restrict__ ws) {
  __shared__ unsigned sk[SORT_TILE];
  const int p0 = blockIdx.x * SORT_TILE, n = min(M - p0, SORT_TILE);
  if (threadIdx.x < n) sk[threadIdx.x] = sorted[p0 + threadIdx.x];
  __syncthreads();
  const int col = (blockIdx.y * 128 + threadIdx.x) * 8;
  if (col >= H) return;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  int head = 0;
  auto flush = [&](int at) {
    float4* d = reinterpret_cast<float4*>(ws + (size_t)(p0 + at) * H + col);
    d[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    d[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
#pragma unroll
    for (int t = 0; t < 8; ++t) acc[t] = 0.f;
  };
  for (int g = 0; g < n; g += 8) {           // eight row loads in flight, then the adds in sorted order
    uint4 u[8];
#pragma unroll
    for (int t = 0; t < 8; ++t)
      if (g + t < n) u[t] = ld_stream16(de + (size_t)(sk[g + t] % (unsigned)M) * H + col);
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int i = g + t;
      if (i >= n) break;
      if (i > 0 && sk[i] / (unsigned)M != sk[i - 1] / (unsigned)M) { flush(head); head = i; }
      float f[8];
      unpack8(u[t], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
  }
  flush(head);
}

// grid (M, ceil(H / 1024)): block p is a no-op unless sorted row p is the first of its table row
__global__ void __launch_bounds__(128)
sorted_run_finish_kernel(const unsigned* __restrict__ sorted, const float* __restrict__ ws, int M, int H,
                         float* __restrict__ table) {
  const int p = blockIdx.x;
  const unsigned key = sorted[p] / (unsigned)M;
  if (p > 0 && sorted[p - 1] / (unsigned)M == key) return;
  const int col = (blockIdx.y * 128 + threadIdx.x) * 8;
  if (col >= H) return;
  const float4* w0 = reinterpret_cast<const float4*>(ws + (size_t)p * H + col);
  float4 a = w0[0], b = w0[1];
  for (int q = (p / SORT_TILE + 1) * SORT_TILE; q < M && sorted[q] / (unsigned)M == key; q += SORT_TILE) {
    const float4* w = reinterpret_cast<const float4*>(ws + (size_t)q * H + col);
    const float4 c = w[0], d = w[1];
    a.x += c.x; a.y += c.y; a.z += c.z; a.w += c.w;
    b.x += d.x; b.y += d.y; b.z += d.z; b.w += d.w;
  }
  float4* t = reinterpret_cast<float4*>(table + (size_t)key * H + col);
  float4 x = t[0], y = t[1];
  x.x += a.x; x.y += a.y; x.z += a.z; x.w += a.w;
  y.x += b.x; y.y += b.y; y.z += b.z; y.w += b.w;
  t[0] = x; t[1] = y;
}

// ------------------------------------------------------------------------------------------------
// MLM position compaction: per sequence, the positions with label >= 0 (at most max_pred) are written to
// idx[b*max_pred + j] (global row index b*S+s), the tail is -1; tgt gets the labels (-1 tail);
// count accumulates the number of valid targets.  Deterministic order (ascending position).
// REMAP (unpadded pre-training): idx holds the packed row row_map[b*S+s] instead, and a label whose token is masked
// (row_map -1) is dropped -- neither written nor counted.
// ------------------------------------------------------------------------------------------------
template <bool REMAP>
__global__ void mlm_compact_kernel(const int* __restrict__ labels, int S, int max_pred, int* __restrict__ idx,
                                   int* __restrict__ tgt, int* __restrict__ count, const int* __restrict__ row_map) {
  const int b = blockIdx.x;
  __shared__ int n;
  if (threadIdx.x == 0) n = 0;
  __syncthreads();
  // single warp, ordered compaction with ballots
  const int lane = threadIdx.x;
  int base = 0;
  for (int s0 = 0; s0 < S; s0 += 32) {
    const int s = s0 + lane;
    int lab = s < S ? labels[b * S + s] : -1;
    const int row = REMAP && lab >= 0 ? row_map[b * S + s] : b * S + s;
    if (REMAP && row < 0) lab = -1;
    const unsigned m = __ballot_sync(0xffffffffu, lab >= 0);
    if (lab >= 0) {
      const int j = base + __popc(m & ((1u << lane) - 1));
      if (j < max_pred) {
        idx[b * max_pred + j] = row;
        tgt[b * max_pred + j] = lab;
      }
    }
    base += __popc(m);
  }
  const int valid = min(base, max_pred);
  for (int j = valid + lane; j < max_pred; j += 32) {
    idx[b * max_pred + j] = -1;
    tgt[b * max_pred + j] = -1;
  }
  if (lane == 0) atomicAdd(count, valid);
}

// ------------------------------------------------------------------------------------------------
// Token packing of a [B, S] pre-training batch on the device (no host sync: it runs inside a captured graph).  One CTA;
// every output has a fixed shape and is written completely on each call:
//   ids / seg / pos [T_cap]  the T unmasked tokens in b*S+s order (id, segment, position s), then the pad tail rows
//                            T .. T_cap-1: id 0, segment 0, position = offset inside its dummy sequence
//   cu [B + D + 1]           the B real sequences, then D dummy sequences of at most S rows that cover the pad tail
//                            (length 0 where the tail does not need them)
//   cls [B]                  first packed row of every sequence
//   row_map [B*S]            packed row of token (b, s), -1 where the token is masked
// A row without any unmasked token packs as S valid tokens: the padded program computes such a row with every key
// valid (the attention length-0 rule), so both modes see the same values and cls always points at a real row.  The
// tail rows are real [PAD] tokens and each tail chunk attends only to itself, so they stay finite and inert.  Nothing
// is written at or past T_cap: a T_cap below T truncates (the host sizes T_cap and D from the same mask).
// ------------------------------------------------------------------------------------------------
constexpr int PACK_THREADS = 512;
constexpr int PACK_MAX_B = 1024;

__global__ void __launch_bounds__(PACK_THREADS) pack_tokens_kernel(
    const int* __restrict__ mask, const int* __restrict__ ids_in, const int* __restrict__ seg_in, int B, int S,
    int T_cap, int D, int* __restrict__ ids, int* __restrict__ seg, int* __restrict__ pos, int* __restrict__ cu,
    int* __restrict__ cls, int* __restrict__ row_map) {
  __shared__ int off[PACK_MAX_B + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  // 1. packed length of every sequence (warp per row)
  for (int b = warp; b < B; b += warps) {
    int n = 0;
    for (int s0 = 0; s0 < S; s0 += 32) {
      const int s = s0 + lane;
      n += __popc(__ballot_sync(0xffffffffu, s < S && mask[(size_t)b * S + s] != 0));
    }
    if (lane == 0) off[b + 1] = n > 0 ? n : S;
  }
  __syncthreads();
  // 2. inclusive scan of the lengths (warp 0) -> off[b] = first packed row of sequence b, off[B] = T
  if (warp == 0) {
    int carry = 0;
    for (int b0 = 0; b0 < B; b0 += 32) {
      const int b = b0 + lane;
      int v = b < B ? off[b + 1] : 0;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += t;
      }
      if (b < B) off[b + 1] = v + carry;
      carry += __shfl_sync(0xffffffffu, v, 31);
    }
    if (lane == 0) off[0] = 0;
  }
  __syncthreads();
  const int T = min(off[B], T_cap);
  // 3. the real tokens (warp per row, ordered compaction with ballots); a full-length row keeps every token, which
  //    covers the empty rows
  for (int b = warp; b < B; b += warps) {
    const bool all = off[b + 1] - off[b] == S;
    int base = off[b];
    for (int s0 = 0; s0 < S; s0 += 32) {
      const int s = s0 + lane;
      const size_t i = (size_t)b * S + s;
      const bool keep = s < S && (all || mask[i] != 0);
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (s < S) {
        const int r = keep ? base + __popc(m & ((1u << lane) - 1)) : -1;
        const bool in = r >= 0 && r < T_cap;
        row_map[i] = in ? r : -1;
        if (in) {
          ids[r] = ids_in[i];
          seg[r] = seg_in != nullptr ? seg_in[i] : 0;
          pos[r] = s;
        }
      }
      base += __popc(m);
    }
    if (lane == 0) {
      cu[b] = min(off[b], T_cap);
      cls[b] = min(off[b], T_cap - 1);
    }
  }
  // 4. the pad tail and its dummy sequences
  for (int r = T + threadIdx.x; r < T_cap; r += blockDim.x) {
    ids[r] = 0;
    seg[r] = 0;
    pos[r] = (r - T) % S;
  }
  if (threadIdx.x == 0) cu[B] = T;
  for (int j = threadIdx.x; j < D; j += blockDim.x) cu[B + 1 + j] = (int)min((long long)T_cap, T + (long long)(j + 1) * S);
}

// rows[i] = src[idx[i]] (zeros when idx < 0)
__global__ void gather_rows_kernel(const __nv_bfloat16* __restrict__ src, const int* __restrict__ idx,
                                   __nv_bfloat16* __restrict__ dst, int n, int H) {
  const int per_row = H / 8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)n * per_row;
       i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / per_row), col = (int)(i % per_row) * 8;
    const int s = idx[r];
    uint4 u = make_uint4(0, 0, 0, 0);
    if (s >= 0) u = *reinterpret_cast<const uint4*>(src + (size_t)s * H + col);
    *reinterpret_cast<uint4*>(dst + (size_t)r * H + col) = u;
  }
}
// dst[idx[i]] = src[i]  (dst pre-zeroed, indices unique)
__global__ void scatter_rows_kernel(const __nv_bfloat16* __restrict__ src, const int* __restrict__ idx,
                                    __nv_bfloat16* __restrict__ dst, int n, int H) {
  const int per_row = H / 8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)n * per_row;
       i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / per_row), col = (int)(i % per_row) * 8;
    const int s = idx[r];
    if (s >= 0) *reinterpret_cast<uint4*>(dst + (size_t)s * H + col) = *reinterpret_cast<const uint4*>(src + (size_t)r * H + col);
  }
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
static inline void drop_params(float p, unsigned int& thresh, float& scale) {
  thresh = p > 0.f ? (unsigned)(p * 65536.f + 0.5f) : 0u;
  scale = p > 0.f ? 65536.f / (65536.f - (float)thresh) : 1.f;
}
static inline int ln_grid(int M) {
  int g = (M + LN_WARPS - 1) / LN_WARPS;
  return g < num_sms() * 8 ? g : num_sms() * 8;
}

#define DISPATCH_CHUNKS(H, ...)                                    \
  do {                                                             \
    const int chunks_ = ((H) + 255) / 256;                         \
    if (chunks_ <= 1) { constexpr int CH = 1; __VA_ARGS__; }       \
    else if (chunks_ <= 2) { constexpr int CH = 2; __VA_ARGS__; }  \
    else if (chunks_ <= 3) { constexpr int CH = 3; __VA_ARGS__; }  \
    else if (chunks_ <= 4) { constexpr int CH = 4; __VA_ARGS__; }  \
    else if (chunks_ <= 8) { constexpr int CH = 8; __VA_ARGS__; }  \
    else { fprintf(stderr, "[b200] hidden size %d too large for the LN kernels\n", (H)); abort(); } \
  } while (0)

void layer_norm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* mean, float* rstd, int M,
                    int H, float eps, Fp8Out f8, cudaStream_t st) {
  if (M == 0) return;                    // no rows: a zero-sized grid is a launch error
  decltype(&ln_fwd_row_kernel<1, false, false>) k;
  if (f8.q == nullptr && H % 256 == 0 && H <= 1024)      // the encoder LNs of the bf16 path
    k = H == 256 ? ln_fwd_row_kernel<1, false, false> : H == 512 ? ln_fwd_row_kernel<2, false, false>
      : H == 768 ? ln_fwd_row_kernel<3, false, false> : ln_fwd_row_kernel<4, false, false>;
  else if (f8.q == nullptr)
    k = H <= 512 ? ln_fwd_row_kernel<2, true, false> : H <= 1024 ? ln_fwd_row_kernel<4, true, false>
                                                                 : ln_fwd_row_kernel<8, true, false>;
  else
    k = H <= 512 ? ln_fwd_row_kernel<2, true, true> : H <= 1024 ? ln_fwd_row_kernel<4, true, true>
                                                                : ln_fwd_row_kernel<8, true, true>;
  int g = (M + 7) / 8;
  if (g > num_sms() * 4) g = num_sms() * 4;
  k<<<g, 256, 0, st>>>((const __nv_bfloat16*)x, gamma, beta, (__nv_bfloat16*)y, mean, rstd, M, eps, H, f8);
}

// Rows per block of the LN backward: 256 threads, WPR = 8 / groups warps per row (the H = 768 kernel: 3 x 2 warps).
static inline int ln_bwd_groups(int H) { return H <= 256 ? 8 : (H <= 512 ? 4 : (H <= 1024 ? 2 : 1)); }
// ~80 registers x 256 threads -> 3 blocks per SM are co-resident; one exact wave (a grid of 4 per SM ran a 1/3-full
// second wave).  The per-block partial column sums are sized by the same grid.
static inline int ln_bwd_grid(int M, int H) {
  const int g = (M + ln_bwd_groups(H) - 1) / ln_bwd_groups(H);
  return g < num_sms() * 3 ? g : num_sms() * 3;
}

int ln_bwd_workspace_floats(int M, int H) { return ln_bwd_grid(M, H) * 3 * H; }

void layer_norm_bwd(const void* dy, const void* x, const float* mean, const float* rstd, const float* gamma, void* dx,
                    void* dxd, float* dgamma, float* dbeta, float* dbias, float* workspace, int M, int H,
                    Seed seed, unsigned int drop_stream, unsigned int in_stream, float p_drop, Fp8Out f8,
                    cudaStream_t st, const uint8_t* keep_mask, bool deterministic) {
  if (M == 0) return;                    // nothing to add to the column sums either
  unsigned int th; float sc;
  drop_params(p_drop, th, sc);
  decltype(&ln_bwd3_kernel<1, 8, false, false>) k;
  int wpr;
  if (f8.q == nullptr && (in_stream == 0xFFFFFFFFu || th == 0) && H % 256 == 0 && H <= 1024) {   // the encoder LNs of the bf16 path
    wpr = H / 256;
    k = wpr == 1 ? ln_bwd3_kernel<1, 8, false, false> : wpr == 2 ? ln_bwd3_kernel<2, 4, false, false>
      : wpr == 3 ? ln_bwd3_kernel<3, 2, false, false> : ln_bwd3_kernel<4, 2, false, false>;
  } else {
    wpr = 8 / ln_bwd_groups(H);
    if (f8.q == nullptr)
      k = wpr == 1 ? ln_bwd3_kernel<1, 8, true, false> : wpr == 2 ? ln_bwd3_kernel<2, 4, true, false>
        : wpr == 4 ? ln_bwd3_kernel<4, 2, true, false> : ln_bwd3_kernel<8, 1, true, false>;
    else
      k = wpr == 1 ? ln_bwd3_kernel<1, 8, true, true> : wpr == 2 ? ln_bwd3_kernel<2, 4, true, true>
        : wpr == 4 ? ln_bwd3_kernel<4, 2, true, true> : ln_bwd3_kernel<8, 1, true, true>;
  }
  const int grid = ln_bwd_grid(M, H);
  k<<<grid, wpr * ln_bwd_groups(H) * 32, 0, st>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, mean, rstd, gamma,
                                                  (__nv_bfloat16*)dx, (__nv_bfloat16*)dxd, workspace, M, seed,
                                                  drop_stream, th, sc, keep_mask, H, in_stream, f8);
  // deterministic: one slice, so every column is finished by a plain += in a fixed order
  colsum_finalize_kernel<<<dim3((H + 31) / 32, 3, deterministic ? 1 : 8), 256, 0, st>>>(workspace, grid, H, dgamma, dbeta,
                                                                                       dxd ? dbias : nullptr);
}

// Keep bits of one hidden-dropout site, one byte per 8 elements ([M][N / 8], bit t of byte j = element 8 j + t kept):
// the same decisions as dropout_keep8(seed, stream, e8) with e8 = (row * N + col) / 8.  Generated here, with every warp
// of the machine busy, instead of inside the GEMM epilogue that applies them (where the tensor cores idle
// meanwhile) and instead of being regenerated by the LayerNorm backward.
__global__ void __launch_bounds__(256) dropout_mask_kernel(unsigned int* __restrict__ out, long long n_words, Seed seed_in,
                                                           unsigned int stream, unsigned int thresh16) {
  const PhiloxKeys keys = philox_keys(seed_in.value());
  const uint32_t T = thresh16 << 16;
  for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (long long)gridDim.x * blockDim.x) {
    uint32_t bits = 0;                        // 32 elements = 4 groups of 8
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const uint4 r = philox7(keys, (uint64_t)(w * 4 + g), stream);
#pragma unroll
      for (int t = 0; t < 8; ++t) bits |= (keep_bit(r, t, T) ? 1u : 0u) << (g * 8 + t);
    }
    out[w] = bits;
  }
}

void dropout_mask(void* out, long long n_elems, Seed seed, unsigned int stream, float p_drop, cudaStream_t st) {
  unsigned int th; float sc;
  drop_params(p_drop, th, sc);
  const long long n_words = n_elems / 32;
  long long g = (n_words + 255) / 256;
  if (g > num_sms() * 16) g = num_sms() * 16;
  if (g > 0) dropout_mask_kernel<<<(unsigned)g, 256, 0, st>>>((unsigned int*)out, n_words, seed, stream, th);
}

void colsum_bf16(const void* x, int M, int N, int ld, float* out, cudaStream_t st) {
  dim3 grid((N + 255) / 256, M >= 4096 ? 64 : (M >= 512 ? 16 : 1));
  colsum_bf16_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, M, N, ld, out);
}

void gelu_fwd(const void* x, void* y, long long n, Fp8Out f8, cudaStream_t st) {
  const long long n8 = n >> 3;
  long long g = (n8 + 255) / 256;
  if (g > num_sms() * 32) g = num_sms() * 32;
  if (g > 0) gelu_fwd_kernel<<<(unsigned)g, 256, 0, st>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, n8, f8);
}
static inline int dgelu_rows(int M) { return M >= 4096 ? 74 : (M >= 512 ? 16 : 1); }
int dgelu_det_workspace_floats(int M, int N) { return dgelu_rows(M) * N; }

void dgelu_bwd(const void* dy, const void* x, void* dx, float* dbias, int M, int N, Fp8Out f8, cudaStream_t st,
               float* dbias_ws) {
  dim3 grid((N + 255) / 256, dgelu_rows(M));
  if (dbias != nullptr && dbias_ws != nullptr) {
    dgelu_bwd_part_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, (__nv_bfloat16*)dx,
                                                dbias_ws, M, N, f8);
    ordered_sum(dbias_ws, grid.y, N, nullptr, 1, dbias, st);
    return;
  }
  dgelu_bwd_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, (__nv_bfloat16*)dx, dbias, M, N, f8);
}

void embedding_fwd(const int* ids, const int* seg, const void* word, const void* pos, const void* type,
                   const float* gamma, const float* beta, void* e_out, void* y, float* mean, float* rstd, int M, int S,
                   int H, float eps, Seed seed, unsigned int stream, float p_drop, cudaStream_t st, const int* pos_ids) {
  if (M == 0) return;
  unsigned int th; float sc;
  drop_params(p_drop, th, sc);
  if (pos_ids != nullptr)
    DISPATCH_CHUNKS(H, (embed_fwd_kernel<CH, true><<<ln_grid(M), LN_WARPS * 32, 0, st>>>(
        ids, seg, (const __nv_bfloat16*)word, (const __nv_bfloat16*)pos, (const __nv_bfloat16*)type, gamma, beta,
        (__nv_bfloat16*)e_out, (__nv_bfloat16*)y, mean, rstd, M, S, H, eps, seed, stream, th, sc, pos_ids)));
  else
    DISPATCH_CHUNKS(H, (embed_fwd_kernel<CH><<<ln_grid(M), LN_WARPS * 32, 0, st>>>(
        ids, seg, (const __nv_bfloat16*)word, (const __nv_bfloat16*)pos, (const __nv_bfloat16*)type, gamma, beta,
        (__nv_bfloat16*)e_out, (__nv_bfloat16*)y, mean, rstd, M, S, H, eps, seed, stream, th, sc, nullptr)));
}

void embedding_bwd_scatter(const void* de, const int* ids, const int* seg, float* gword, float* gpos, float* gtype,
                           int M, int S, int H, int type_rows, cudaStream_t st, const int* pos_ids) {
  if (M == 0) return;
  const size_t work = (size_t)M * (H / 8);
  int grid = (int)((work + 255) / 256);
  if (grid > num_sms() * 16) grid = num_sms() * 16;
  if (pos_ids == nullptr && M % S == 0 && H % 8 == 0 && (gtype == nullptr || type_rows == 2)) {
    // word rows: scatter with atomics (30 k rows, little contention); position / token-type rows: reductions
    embed_bwd_scatter_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)de, ids, seg, gword, nullptr, nullptr, M, S, H,
                                                   nullptr);
    dim3 g2((H + 255) / 256, (S + 7) / 8);
    embed_bwd_postype_kernel<<<g2, 256, 0, st>>>((const __nv_bfloat16*)de, seg, gpos, gtype, M / S, S, H);
    return;
  }
  // packed rows (pos_ids) or a ragged batch: every table row by atomics
  if (grid > 0)
    embed_bwd_scatter_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)de, ids, seg, gword, gpos, gtype, M, S, H,
                                                   pos_ids);
}

void ordered_sum(const float* part, int rows, int W, const int* row_seg, int nseg, float* out, cudaStream_t st) {
  int cw = 1;
  while (cw < W && cw < 32) cw <<= 1;
  if (W > 0 && nseg > 0)
    ordered_sum_kernel<<<dim3((W + cw - 1) / cw, nseg), ORD_THREADS, 0, st>>>(part, rows, W, cw, row_seg, out);
}

static inline int colsum_rows(int M) { return M >= 4096 ? 64 : (M >= 512 ? 16 : 1); }
int colsum_det_workspace_floats(int M, int N) { return colsum_rows(M) * N; }

void colsum_bf16_det(const void* x, int M, int N, int ld, float* out, float* ws, cudaStream_t st) {
  const int rows = colsum_rows(M);
  colsum_bf16_part_kernel<<<dim3((N + 255) / 256, rows), 256, 0, st>>>((const __nv_bfloat16*)x, M, N, ld, ws);
  ordered_sum(ws, rows, N, nullptr, 1, out, st);
}

int embedding_det_chunk_rows() { return SORT_CAP; }

// table[key(i)] += de[i] for the M token rows i of a chunk that starts at row row0; key(i) = key[i], or
// (row0 + i) % key_mod without key (de and key point at the chunk)
static void sorted_scatter(const void* de, const int* key, int key_mod, int row0, int M, int H, float* table,
                           unsigned* sort_ws, float* sum_ws, cudaStream_t st) {
  static bool configured = false;
  if (!configured) {
    B200_CUDA_CHECK(cudaFuncSetAttribute(sort_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         SORT_CAP * (int)sizeof(unsigned)));
    configured = true;
  }
  int n = 1;
  while (n < M) n <<= 1;
  sort_rows_kernel<<<1, SORT_THREADS, n * sizeof(unsigned), st>>>(key, key_mod, row0, M, sort_ws);
  const dim3 g2((M + SORT_TILE - 1) / SORT_TILE, (H + 1023) / 1024);
  sorted_piece_sum_kernel<<<g2, 128, 0, st>>>((const __nv_bfloat16*)de, sort_ws, M, H, sum_ws);
  sorted_run_finish_kernel<<<dim3(M, (H + 1023) / 1024), 128, 0, st>>>(sort_ws, sum_ws, M, H, table);
}

void embedding_bwd_det(const void* de, const int* ids, const int* seg, float* gword, float* gpos, float* gtype,
                       int M, int S, int H, const int* pos_ids, unsigned* sort_ws, float* sum_ws, cudaStream_t st) {
  // chunks of at most SORT_CAP rows, each added to the tables in row order; a null seg keys every row to type row 0
  for (int r0 = 0; r0 < M; r0 += SORT_CAP) {
    const int m = M - r0 < SORT_CAP ? M - r0 : SORT_CAP;
    const void* d = (const __nv_bfloat16*)de + (size_t)r0 * H;
    sorted_scatter(d, ids + r0, 0, r0, m, H, gword, sort_ws, sum_ws, st);
    sorted_scatter(d, pos_ids ? pos_ids + r0 : nullptr, S, r0, m, H, gpos, sort_ws, sum_ws, st);
    if (gtype != nullptr) sorted_scatter(d, seg ? seg + r0 : nullptr, 1, r0, m, H, gtype, sort_ws, sum_ws, st);
  }
}

void mlm_compact(const int* labels, int B, int S, int max_pred, int* idx, int* tgt, int* count, cudaStream_t st,
                 const int* row_map) {
  B200_CUDA_CHECK(cudaMemsetAsync(count, 0, sizeof(int), st));
  if (row_map != nullptr)
    mlm_compact_kernel<true><<<B, 32, 0, st>>>(labels, S, max_pred, idx, tgt, count, row_map);
  else
    mlm_compact_kernel<false><<<B, 32, 0, st>>>(labels, S, max_pred, idx, tgt, count, nullptr);
}

int pack_tokens_max_batch() { return PACK_MAX_B; }

void pack_tokens(const int* mask, const int* ids_in, const int* seg_in, int B, int S, int T_cap, int D, int* ids,
                 int* seg, int* pos, int* cu, int* cls, int* row_map, cudaStream_t st) {
  pack_tokens_kernel<<<1, PACK_THREADS, 0, st>>>(mask, ids_in, seg_in, B, S, T_cap, D, ids, seg, pos, cu, cls, row_map);
}

void gather_rows(const void* src, const int* idx, void* dst, int n, int H, cudaStream_t st) {
  const size_t work = (size_t)n * (H / 8);
  int grid = (int)((work + 255) / 256);
  if (grid > num_sms() * 16) grid = num_sms() * 16;
  if (grid > 0) gather_rows_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)src, idx, (__nv_bfloat16*)dst, n, H);
}
void scatter_rows(const void* src, const int* idx, void* dst, int n, int H, cudaStream_t st) {
  const size_t work = (size_t)n * (H / 8);
  int grid = (int)((work + 255) / 256);
  if (grid > num_sms() * 16) grid = num_sms() * 16;
  if (grid > 0) scatter_rows_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)src, idx, (__nv_bfloat16*)dst, n, H);
}

}  // namespace b200
