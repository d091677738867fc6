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

// ------------------------------------------------------------------------------------------------
// LayerNorm forward / backward, occupancy-friendly layout: WPR warps share one row, every lane owns ONE
// 16-byte chunk (8 columns), a block holds two such row groups.  ~70-90 registers per thread instead of
// 255 -> 4-6x more warps in flight, which is what a pure streaming kernel needs to reach HBM speed
// (first version, one warp per row with 32 columns per lane: 38 us for a 100 MB backward pass).
// Row statistics travel through shared memory + a named barrier per row group.
// ------------------------------------------------------------------------------------------------
// two sums at once across the WPR warps of a row group: ONE named barrier per row -- the exchange slots are
// double buffered by row parity (a warp can only overwrite parity p again after the barrier of the row in
// between, which the slowest reader of parity p has to reach first).
template <int WPR>
__device__ __forceinline__ float2 group_sum2(float a, float b, float2* slot, int wi, int group) {
  a = warp_sum(a);
  b = warp_sum(b);
  if (WPR == 1) return make_float2(a, b);
  if ((threadIdx.x & 31) == 0) slot[wi] = make_float2(a, b);
  if (group == 0) asm volatile("bar.sync 1, %0;" ::"n"(WPR * 32) : "memory");
  else asm volatile("bar.sync 2, %0;" ::"n"(WPR * 32) : "memory");
  float2 t = make_float2(0.f, 0.f);
#pragma unroll
  for (int w = 0; w < WPR; ++w) { const float2 v = slot[w]; t.x += v.x; t.y += v.y; }
  return t;
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

template <int WPR>
__global__ void __launch_bounds__(2 * WPR * 32)
ln_fwd2_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
               __nv_bfloat16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, int M, int H,
               float eps, Seed seed_in, unsigned int stream, unsigned int thresh16, float drop_scale, const Fp8Out f8) {
  const unsigned long long seed = seed_in.value();
  const float qscale = f8.q ? f8.meta[1] : 0.f;
  float amax = 0.f;
  __shared__ float2 xchg[2][2][8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int group = warp / WPR, wi = warp % WPR;
  const int col = (wi * 32 + lane) * 8;
  const bool live = col < H;
  float g[8], b[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) { g[t] = live ? gamma[col + t] : 0.f; b[t] = live ? beta[col + t] : 0.f; }
  const int stride = gridDim.x * 2;
  int row = blockIdx.x * 2 + group;
  uint4 nx = make_uint4(0, 0, 0, 0);
  float nshift = 0.f;
  if (row < M) {
    if (live) nx = ld_stream16(x + (size_t)row * H + col);
    nshift = __bfloat162float(x[(size_t)row * H]);
  }
  for (int it = 0; row < M; row += stride, ++it) {
    float v[8];
    unpack8(nx, v);
    const float shift = nshift;           // first element of the row: keeps sum / sum-of-squares well conditioned
    const int nrow = row + stride;
    if (nrow < M) {                        // prefetch the next row before this row's barrier
      if (live) nx = ld_stream16(x + (size_t)nrow * H + col);
      nshift = __bfloat162float(x[(size_t)nrow * H]);
    }
    float s = 0.f, q = 0.f;
    if (live) {
#pragma unroll
      for (int t = 0; t < 8; ++t) { const float d = v[t] - shift; s += d; q += d * d; }
    }
    const float2 r = group_sum2<WPR>(s, q, xchg[group][it & 1], wi, group);
    const float ms = r.x / (float)H;
    const float mean = shift + ms;
    const float rstd = rsqrtf(fmaxf(r.y / (float)H - ms * ms, 0.f) + eps);
    if (live) {
      Keep8 keep = Keep8::all();
      if (thresh16 != 0) keep = dropout_keep8(seed, stream, ((uint64_t)row * H + col) >> 3, thresh16);
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        float o = (v[t] - mean) * rstd * g[t] + b[t];
        if (thresh16 != 0) o = keep[t] ? o * drop_scale : 0.f;
        v[t] = o;
      }
      store8(y + (size_t)row * H + col, v);
      if (f8.q) fp8_emit8(f8, (size_t)row * H + col, v, qscale, amax);
    }
    if (wi == 0 && lane == 0) {
      if (mean_out) mean_out[row] = mean;
      if (rstd_out) rstd_out[row] = rstd;
    }
  }
  if (f8.q) fp8_amax_commit(f8, amax);
}

// Opt-in variant (B200_LN_ROWS=2): every group of WPR warps works on TWO rows per iteration -- twice the bytes in
// flight per thread (the kernel above is latency bound: 16 B per thread and one barrier per row) and one barrier per
// two rows.  Same arithmetic per row, so the results are bit-identical to ln_fwd2_kernel.
template <int WPR>
__device__ __forceinline__ float4 group_sum4(float a, float b, float c, float d, float4* slot, int wi, int group) {
  a = warp_sum(a); b = warp_sum(b); c = warp_sum(c); d = warp_sum(d);
  if (WPR == 1) return make_float4(a, b, c, d);
  if ((threadIdx.x & 31) == 0) slot[wi] = make_float4(a, b, c, d);
  if (group == 0) asm volatile("bar.sync 1, %0;" ::"n"(WPR * 32) : "memory");
  else asm volatile("bar.sync 2, %0;" ::"n"(WPR * 32) : "memory");
  float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int w = 0; w < WPR; ++w) { const float4 v = slot[w]; t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w; }
  return t;
}

template <int WPR>
__global__ void __launch_bounds__(2 * WPR * 32)
ln_fwd2x2_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                 __nv_bfloat16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, int M, int H,
                 float eps, Seed seed_in, unsigned int stream, unsigned int thresh16, float drop_scale, const Fp8Out f8) {
  const unsigned long long seed = seed_in.value();
  const float qscale = f8.q ? f8.meta[1] : 0.f;
  float amax = 0.f;
  __shared__ float4 xchg[2][2][8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int group = warp / WPR, wi = warp % WPR;
  const int col = (wi * 32 + lane) * 8;
  const bool live = col < H;
  float g[8], b[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) { g[t] = live ? gamma[col + t] : 0.f; b[t] = live ? beta[col + t] : 0.f; }
  const int stride = gridDim.x * 4;                 // 2 groups x 2 rows per block and iteration
  int row = (blockIdx.x * 2 + group) * 2;           // this group's rows: row, row + 1
  uint4 nx[2] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
  float nshift[2] = {0.f, 0.f};
#pragma unroll
  for (int r = 0; r < 2; ++r)
    if (row + r < M) {
      if (live) nx[r] = ld_stream16(x + (size_t)(row + r) * H + col);
      nshift[r] = __bfloat162float(x[(size_t)(row + r) * H]);
    }
  for (int it = 0; row < M; row += stride, ++it) {
    float v[2][8], shift[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) { unpack8(nx[r], v[r]); shift[r] = nshift[r]; }
    const int nrow = row + stride;
#pragma unroll
    for (int r = 0; r < 2; ++r)
      if (nrow + r < M) {                  // prefetch the next pair before this pair's barrier
        if (live) nx[r] = ld_stream16(x + (size_t)(nrow + r) * H + col);
        nshift[r] = __bfloat162float(x[(size_t)(nrow + r) * H]);
      }
    float s[2] = {0.f, 0.f}, q[2] = {0.f, 0.f};
    if (live) {
#pragma unroll
      for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int t = 0; t < 8; ++t) { const float d = v[r][t] - shift[r]; s[r] += d; q[r] += d * d; }
    }
    const float4 red = group_sum4<WPR>(s[0], q[0], s[1], q[1], xchg[group][it & 1], wi, group);
    const float rs[2] = {red.x, red.z}, rq[2] = {red.y, red.w};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int rr = row + r;
      if (rr >= M) continue;
      const float ms = rs[r] / (float)H;
      const float mean = shift[r] + ms;
      const float rstd = rsqrtf(fmaxf(rq[r] / (float)H - ms * ms, 0.f) + eps);
      if (live) {
        Keep8 keep = Keep8::all();
        if (thresh16 != 0) keep = dropout_keep8(seed, stream, ((uint64_t)rr * H + col) >> 3, thresh16);
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          float o = (v[r][t] - mean) * rstd * g[t] + b[t];
          if (thresh16 != 0) o = keep[t] ? o * drop_scale : 0.f;
          v[r][t] = o;
        }
        store8(y + (size_t)rr * H + col, v[r]);
        if (f8.q) fp8_emit8(f8, (size_t)rr * H + col, v[r], qscale, amax);
      }
      if (wi == 0 && lane == 0) {
        if (mean_out) mean_out[rr] = mean;
        if (rstd_out) rstd_out[rr] = rstd;
      }
    }
  }
  if (f8.q) fp8_amax_commit(f8, amax);
}

// LayerNorm backward.
//   in : dy [M,H] (grad wrt LN output; with `in_stream` given, dy is first multiplied by the *output* dropout
//        mask of that stream -- used by the embedding LN whose output was dropped out)
//        x  [M,H] pre-LN input, mean/rstd [M], gamma [H]
//   out: dx [M,H]          grad wrt the pre-LN input (this is also the residual-branch gradient)
//        dxd [M,H] optional: dx * dropout_mask(stream `drop_stream`) * scale  -> gradient of the GEMM output
//                            that was dropped out before the residual add (K14/K18)
//        partial [grid, 3, H]: per-block column sums of (dy*xhat, dy, dxd) -> dgamma, dbeta, dbias
template <int WPR>
__global__ void __launch_bounds__(2 * WPR * 32)
ln_bwd2_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
               const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
               __nv_bfloat16* __restrict__ dx, __nv_bfloat16* __restrict__ dxd, float* __restrict__ partial, int M,
               int H, Seed seed_in, unsigned int drop_stream, unsigned int in_stream,
               unsigned int thresh16, float drop_scale, const Fp8Out f8) {
  const unsigned long long seed = seed_in.value();
  const float qscale = f8.q ? f8.meta[1] : 0.f;
  float amax = 0.f;
  __shared__ float2 xchg[2][2][8];
  __shared__ float comb[3][WPR * 256];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int group = warp / WPR, wi = warp % WPR;
  const int col = (wi * 32 + lane) * 8;
  const bool live = col < H;
  float g[8], ag[8], ab[8], ad[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) { g[t] = live ? gamma[col + t] : 0.f; ag[t] = ab[t] = ad[t] = 0.f; }
  const int stride = gridDim.x * 2;
  int row = blockIdx.x * 2 + group;
  uint4 nd = make_uint4(0, 0, 0, 0), nv = make_uint4(0, 0, 0, 0);
  float nmu = 0.f, nrs = 0.f;
  if (row < M) {
    if (live) { nd = ld_stream16(dy + (size_t)row * H + col); nv = ld_stream16(x + (size_t)row * H + col); }
    nmu = mean[row]; nrs = rstd[row];
  }
  for (int it = 0; row < M; row += stride, ++it) {
    float d[8], v[8];
    unpack8(nd, d);
    unpack8(nv, v);
    const float mu = nmu, rs = nrs;
    const int nrow = row + stride;
    if (nrow < M) {                        // next row's loads are in flight across this row's barrier
      if (live) { nd = ld_stream16(dy + (size_t)nrow * H + col); nv = ld_stream16(x + (size_t)nrow * H + col); }
      nmu = mean[nrow]; nrs = rstd[nrow];
    }
    if (in_stream != 0xFFFFFFFFu && thresh16 != 0 && live) {
      const Keep8 keep = dropout_keep8(seed, in_stream, ((uint64_t)row * H + col) >> 3, thresh16);
#pragma unroll
      for (int t = 0; t < 8; ++t) d[t] = keep[t] ? d[t] * drop_scale : 0.f;
    }
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const float xh = live ? (v[t] - mu) * rs : 0.f;
      const float dg = d[t] * g[t];
      ag[t] += d[t] * xh;
      ab[t] += d[t];
      v[t] = xh;
      d[t] = dg;
      s1 += dg;
      s2 += dg * xh;
    }
    const float2 r = group_sum2<WPR>(s1, s2, xchg[group][it & 1], wi, group);
    s1 = r.x / (float)H;
    s2 = r.y / (float)H;
    if (live) {
#pragma unroll
      for (int t = 0; t < 8; ++t) d[t] = rs * (d[t] - s1 - v[t] * s2);
      store8(dx + (size_t)row * H + col, d);
      if (dxd != nullptr) {
        if (thresh16 != 0) {
          const Keep8 keep = dropout_keep8(seed, drop_stream, ((uint64_t)row * H + col) >> 3, thresh16);
#pragma unroll
          for (int t = 0; t < 8; ++t) d[t] = keep[t] ? d[t] * drop_scale : 0.f;
        }
#pragma unroll
        for (int t = 0; t < 8; ++t) ad[t] += d[t];
        store8(dxd + (size_t)row * H + col, d);
        if (f8.q) fp8_emit8(f8, (size_t)row * H + col, d, qscale, amax);
      }
    }
  }
  if (f8.q) fp8_amax_commit(f8, amax);
  // combine the two row groups of the block and write the per-block partial column sums
  const int cbase = (wi * 32 + lane) * 8;
  if (group == 1) {
#pragma unroll
    for (int t = 0; t < 8; ++t) { comb[0][cbase + t] = ag[t]; comb[1][cbase + t] = ab[t]; comb[2][cbase + t] = ad[t]; }
  }
  __syncthreads();
  if (group == 0 && live) {
    float* dst = partial + (size_t)blockIdx.x * 3 * H + col;
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      dst[t] = ag[t] + comb[0][cbase + t];
      dst[H + t] = ab[t] + comb[1][cbase + t];
      dst[2 * H + t] = ad[t] + comb[2][cbase + t];
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Fast paths (H == CHUNKS * 256, no fp8 side output).  The kernels above are instruction bound (per-row reductions,
// barriers and address arithmetic amortised over only 8 elements per lane), so these variants cut instructions per element:
//   forward : one warp owns a whole row (32 elements per lane): shuffle-only statistics, exact two-pass variance in
//             registers, gamma / beta from shared memory (conflict-free float4 layout); ~8 instructions per element
//   backward: same lane-owns-8-columns layout as ln_bwd2 (the column sums for dgamma / dbeta / dbias must stay in
//             registers of a fixed lane) but without bounds predicates, with the per-row constants folded into two
//             FFMAs per element, one 64-bit Philox counter computation per row.
// ------------------------------------------------------------------------------------------------
template <int CHUNKS>
__global__ void __launch_bounds__(256)
ln_fwd_row_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                  __nv_bfloat16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, int M,
                  float eps) {
  constexpr int H = CHUNKS * 256;
  __shared__ float4 sg[CHUNKS][2][32], sb[CHUNKS][2][32];   // [chunk][half of the lane's 8 columns][lane]
  pdl_trigger_small();
  pdl_wait();
  for (int i = threadIdx.x; i < CHUNKS * 64; i += blockDim.x) {
    const int c = i >> 6, h = (i >> 5) & 1, l = i & 31;
    sg[c][h][l] = __ldg(reinterpret_cast<const float4*>(gamma + c * 256 + l * 8 + h * 4));
    sb[c][h][l] = __ldg(reinterpret_cast<const float4*>(beta + c * 256 + l * 8 + h * 4));
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int stride = gridDim.x * 8;
  int row = blockIdx.x * 8 + warp;
  uint4 nx[CHUNKS];
  if (row < M) {
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) nx[c] = ld_stream16(x + (size_t)row * H + c * 256 + lane * 8);
  }
  for (; row < M; row += stride) {
    float v[CHUNKS][8];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) unpack8(nx[c], v[c]);
    const int nrow = row + stride;
    if (nrow < M) {                        // next row in flight while this one is reduced
#pragma unroll
      for (int c = 0; c < CHUNKS; ++c) nx[c] = ld_stream16(x + (size_t)nrow * H + c * 256 + lane * 8);
    }
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c)
#pragma unroll
      for (int t = 0; t < 8; ++t) s += v[c][t];
    const float mean = warp_sum(s) * (1.0f / (float)H);
    float q = 0.f;
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c)
#pragma unroll
      for (int t = 0; t < 8; ++t) { v[c][t] -= mean; q = fmaf(v[c][t], v[c][t], q); }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / (float)H) + eps);
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
      const float4 g0 = sg[c][0][lane], g1 = sg[c][1][lane], b0 = sb[c][0][lane], b1 = sb[c][1][lane];
      const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int t = 0; t < 8; ++t) v[c][t] = fmaf(v[c][t] * rstd, g[t], b[t]);
      store8(y + (size_t)row * H + c * 256 + lane * 8, v[c]);
    }
    if (lane == 0) {
      if (mean_out) mean_out[row] = mean;
      if (rstd_out) rstd_out[row] = rstd;
    }
  }
}

template <int WPR, int GROUPS>
__global__ void __launch_bounds__(GROUPS * WPR * 32)
ln_bwd3_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
               const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
               __nv_bfloat16* __restrict__ dx, __nv_bfloat16* __restrict__ dxd, float* __restrict__ partial, int M,
               Seed seed_in, unsigned int drop_stream, unsigned int thresh16, float drop_scale,
               const uint8_t* __restrict__ keep_mask) {
  // The dropout decisions of the residual branch are READ (one byte per 8 elements, written by dropout_mask_kernel
  // or by the producing GEMM epilogue: GemmCall::mask_out) instead of regenerated with Philox whenever the caller
  // has them.
  constexpr int H = WPR * 256;
  __shared__ float2 xchg[GROUPS][2][WPR];
  __shared__ float comb[GROUPS - 1 > 0 ? GROUPS - 1 : 1][3][H];
  pdl_trigger_small();
  pdl_wait();
  const unsigned long long seed = thresh16 != 0 ? seed_in.value() : 0ull;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int group = warp / WPR, wi = warp % WPR;
  const int col = (wi * 32 + lane) * 8;
  f32x2 g2[4], ag2[4], ab2[4], ad2[4];
  {
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + col));
    const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + col + 4));
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
  if (row < M) {
    nd = ld_stream16(dy + (size_t)row * H + col);
    nv = ld_stream16(x + (size_t)row * H + col);
    nmu = __ldg(mean + row);
    nrs = __ldg(rstd + row);
    if (use_mask) nmask = __ldg(keep_mask + (size_t)row * (H / 8) + (col >> 3));
  }
  constexpr float invH = 1.0f / (float)H;
  for (int it = 0; row < M; row += stride, ++it) {
    const uint32_t dw[4] = {nd.x, nd.y, nd.z, nd.w}, vw[4] = {nv.x, nv.y, nv.z, nv.w};
    const float rs = nrs, nmr = -nmu * nrs;
    const uint32_t mask = nmask;
    const int nrow = row + stride;
    if (nrow < M) {                        // next row's loads are in flight across this row's barrier
      nd = ld_stream16(dy + (size_t)nrow * H + col);
      nv = ld_stream16(x + (size_t)nrow * H + col);
      nmu = __ldg(mean + nrow);
      nrs = __ldg(rstd + nrow);
      if (use_mask) nmask = __ldg(keep_mask + (size_t)nrow * (H / 8) + (col >> 3));
    }
    const f32x2 rs2 = f2_splat(rs), nmr2 = f2_splat(nmr);
    f32x2 xh[4], dg[4], s1p = f2_splat(0.f), s2p = f2_splat(0.f);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const f32x2 d = f2_from_bf16x2(dw[t]);
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
    }
  }
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
  if (group == 0) {           // per-block partial column sums; colsum_finalize_kernel adds them into the gradient arena
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
// per row), then the 8 warps are combined through shared memory.  Z > 1 (B200_LN_FINALIZE_SPLIT, opt-in) cuts the
// partial rows into Z slices that finish with an atomic add: the kernel is a chain of ~55 dependent loads per warp
// at Z = 1 (8 us for 444 partial rows), i.e. latency bound.
__global__ void __launch_bounds__(256)
colsum_finalize_kernel(const float* __restrict__ partial, int nblocks, int H, float* dgamma, float* dbeta,
                       float* dbias) {
  pdl_trigger_small();
  pdl_wait();
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
  pdl_trigger_small();
  pdl_wait();
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

// dx[m][n] = dy[m][n] * gelu'(x[m][n]);  dbias[n] += sum_m dx[m][n]
__global__ void __launch_bounds__(256)
dgelu_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ dx,
                 float* __restrict__ dbias, int M, int N, const Fp8Out f8) {
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
  if (blockIdx.x * 256 + c < N) atomicAdd(dbias + blockIdx.x * 256 + c, sum);
}

// ------------------------------------------------------------------------------------------------
// Embedding forward: e = word[id] + pos[s] (+ type[seg]); y = dropout(LN(e)); saves e, mean, rstd
// ------------------------------------------------------------------------------------------------
template <int CHUNKS>
__global__ void __launch_bounds__(LN_WARPS * 32)
embed_fwd_kernel(const int* __restrict__ ids, const int* __restrict__ seg, const __nv_bfloat16* __restrict__ word,
                 const __nv_bfloat16* __restrict__ pos, const __nv_bfloat16* __restrict__ type,
                 const float* __restrict__ gamma, const float* __restrict__ beta, __nv_bfloat16* __restrict__ e_out,
                 __nv_bfloat16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, int M,
                 int S, int H, float eps, Seed seed_in, unsigned int stream, unsigned int thresh16,
                 float drop_scale) {
  const unsigned long long seed = seed_in.value();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float g[CHUNKS][8], b[CHUNKS][8];
  load_vec_f32<CHUNKS>(gamma, H, lane, g);
  load_vec_f32<CHUNKS>(beta, H, lane, b);
  for (int row = blockIdx.x * LN_WARPS + warp; row < M; row += gridDim.x * LN_WARPS) {
    float v[CHUNKS][8], t0[CHUNKS][8];
    load_row<CHUNKS>(word + (size_t)ids[row] * H, H, lane, v);
    load_row<CHUNKS>(pos + (size_t)(row % S) * H, H, lane, t0);
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

// Embedding backward scatter: de [M,H] (bf16) is added into the fp32 gradient tables.
__global__ void __launch_bounds__(256)
embed_bwd_scatter_kernel(const __nv_bfloat16* __restrict__ de, const int* __restrict__ ids,
                         const int* __restrict__ seg, float* __restrict__ gword, float* __restrict__ gpos,
                         float* __restrict__ gtype, int M, int S, int H) {
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
    float* dst[3] = {gword + (size_t)ids[row] * H + col, gpos ? gpos + (size_t)(row % S) * H + col : nullptr,
                     gtype ? gtype + (size_t)seg[row] * H + col : nullptr};
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
// MLM position compaction: per sequence, the positions with label >= 0 (at most max_pred) are written to
// idx[b*max_pred + j] (global row index b*S+s), the tail is -1; tgt gets the labels (-1 tail);
// count accumulates the number of valid targets.  Deterministic order (ascending position).
// ------------------------------------------------------------------------------------------------
__global__ void mlm_compact_kernel(const int* __restrict__ labels, int S, int max_pred, int* __restrict__ idx,
                                   int* __restrict__ tgt, int* __restrict__ count) {
  const int b = blockIdx.x;
  __shared__ int n;
  if (threadIdx.x == 0) n = 0;
  __syncthreads();
  // single warp, ordered compaction with ballots
  const int lane = threadIdx.x;
  int base = 0;
  for (int s0 = 0; s0 < S; s0 += 32) {
    const int s = s0 + lane;
    const int lab = s < S ? labels[b * S + s] : -1;
    const unsigned m = __ballot_sync(0xffffffffu, lab >= 0);
    if (lab >= 0) {
      const int j = base + __popc(m & ((1u << lane) - 1));
      if (j < max_pred) {
        idx[b * max_pred + j] = b * S + s;
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

#define DISPATCH_WPR(H, ...)                                         \
  do {                                                               \
    const int wpr_ = ((H) + 255) / 256;                              \
    if (wpr_ <= 1) { constexpr int WPR = 1; __VA_ARGS__; }           \
    else if (wpr_ <= 2) { constexpr int WPR = 2; __VA_ARGS__; }      \
    else if (wpr_ <= 3) { constexpr int WPR = 3; __VA_ARGS__; }      \
    else if (wpr_ <= 4) { constexpr int WPR = 4; __VA_ARGS__; }      \
    else if (wpr_ <= 8) { constexpr int WPR = 8; __VA_ARGS__; }      \
    else { fprintf(stderr, "[b200] hidden size %d too large for the LN kernels\n", (H)); abort(); } \
  } while (0)

static inline int ln2_grid(int M) {     // 2 rows per block at a time; 4 resident blocks per SM
  int g = (M + 1) / 2;
  return g < num_sms() * 4 ? g : num_sms() * 4;
}

static bool ln_fast_enabled() {
  static const bool on = []() { const char* e = getenv("B200_LN_FAST"); return !(e && e[0] == '0'); }();
  return on;
}

void layer_norm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* mean, float* rstd, int M,
                    int H, float eps, Seed seed, unsigned int stream, float p_drop, Fp8Out f8, cudaStream_t st) {
  unsigned int th; float sc;
  drop_params(p_drop, th, sc);
  if (ln_fast_enabled() && th == 0 && f8.q == nullptr && H % 256 == 0 && H <= 1024) {   // warp-per-row fast path
    int g = (M + 7) / 8;
    if (g > num_sms() * 4) g = num_sms() * 4;
    const __nv_bfloat16* xp = (const __nv_bfloat16*)x;
    __nv_bfloat16* yp = (__nv_bfloat16*)y;
    switch (H / 256) {
      case 1: launch_pdl(ln_fwd_row_kernel<1>, dim3(g), dim3(256), 0, st, xp, gamma, beta, yp, mean, rstd, M, eps); break;
      case 2: launch_pdl(ln_fwd_row_kernel<2>, dim3(g), dim3(256), 0, st, xp, gamma, beta, yp, mean, rstd, M, eps); break;
      case 3: launch_pdl(ln_fwd_row_kernel<3>, dim3(g), dim3(256), 0, st, xp, gamma, beta, yp, mean, rstd, M, eps); break;
      default: launch_pdl(ln_fwd_row_kernel<4>, dim3(g), dim3(256), 0, st, xp, gamma, beta, yp, mean, rstd, M, eps); break;
    }
    return;
  }
  static const bool two_rows = []() { const char* e = getenv("B200_LN_ROWS"); return e && e[0] == '2'; }();
  if (two_rows) {                        // measured slower than one row (24.6 vs 22.6 us): kept for reference only
    int g4 = (M + 3) / 4;
    if (g4 > num_sms() * 3) g4 = num_sms() * 3;
    DISPATCH_WPR(H, (ln_fwd2x2_kernel<WPR><<<g4, 2 * WPR * 32, 0, st>>>(
        (const __nv_bfloat16*)x, gamma, beta, (__nv_bfloat16*)y, mean, rstd, M, H, eps, seed, stream, th, sc, f8)));
    return;
  }
  DISPATCH_WPR(H, (ln_fwd2_kernel<WPR><<<ln2_grid(M), 2 * WPR * 32, 0, st>>>(
      (const __nv_bfloat16*)x, gamma, beta, (__nv_bfloat16*)y, mean, rstd, M, H, eps, seed, stream, th, sc, f8)));
}

// backward: ~80 registers x 256 threads -> 3 blocks per SM are co-resident; one exact wave (a grid of 4 per SM
// ran a 1/3-full second wave)
static inline int ln2_bwd_grid(int M) {
  int g = (M + 1) / 2;
  return g < num_sms() * 3 ? g : num_sms() * 3;
}

int ln_bwd_workspace_floats(int M, int H) { return ln2_grid(M) * 3 * H; }

void layer_norm_bwd(const void* dy, const void* x, const float* mean, const float* rstd, const float* gamma, void* dx,
                    void* dxd, float* dgamma, float* dbeta, float* dbias, float* workspace, int M, int H,
                    Seed seed, unsigned int drop_stream, unsigned int in_stream, float p_drop, Fp8Out f8,
                    cudaStream_t st, const uint8_t* keep_mask) {
  unsigned int th; float sc;
  drop_params(p_drop, th, sc);
  static const int split = []() {
    const char* e = getenv("B200_LN_FINALIZE_SPLIT");
    const int z = e ? atoi(e) : 8;
    return z < 1 ? 1 : (z > 32 ? 32 : z);
  }();
  if (ln_fast_enabled() && f8.q == nullptr && (in_stream == 0xFFFFFFFFu || th == 0) && H % 256 == 0 && H <= 1024) {
    const __nv_bfloat16 *dyp = (const __nv_bfloat16*)dy, *xp = (const __nv_bfloat16*)x;
    __nv_bfloat16 *dxp = (__nv_bfloat16*)dx, *dxdp = (__nv_bfloat16*)dxd;
    const int wpr = H / 256;
    const int groups = wpr == 4 ? 2 : (wpr == 3 ? 2 : (wpr == 2 ? 4 : 8));
    int g = (M + groups - 1) / groups;
    const int cap = ln2_bwd_grid(M);     // the workspace is sized for ln2_grid(M) >= this
    if (g > cap) g = cap;
    switch (wpr) {
      case 1: launch_pdl(ln_bwd3_kernel<1, 8>, dim3(g), dim3(256), 0, st, dyp, xp, mean, rstd, gamma, dxp, dxdp, workspace, M, seed, drop_stream, th, sc, keep_mask); break;
      case 2: launch_pdl(ln_bwd3_kernel<2, 4>, dim3(g), dim3(256), 0, st, dyp, xp, mean, rstd, gamma, dxp, dxdp, workspace, M, seed, drop_stream, th, sc, keep_mask); break;
      case 3: launch_pdl(ln_bwd3_kernel<3, 2>, dim3(g), dim3(192), 0, st, dyp, xp, mean, rstd, gamma, dxp, dxdp, workspace, M, seed, drop_stream, th, sc, keep_mask); break;
      default: launch_pdl(ln_bwd3_kernel<4, 2>, dim3(g), dim3(256), 0, st, dyp, xp, mean, rstd, gamma, dxp, dxdp, workspace, M, seed, drop_stream, th, sc, keep_mask); break;
    }
    dim3 g2((H + 31) / 32, 3, split);
    launch_pdl(colsum_finalize_kernel, g2, dim3(256), 0, st, (const float*)workspace, g, H, dgamma, dbeta, dxd ? dbias : (float*)nullptr);
    return;
  }
  const int grid = ln2_bwd_grid(M);
  DISPATCH_WPR(H, (ln_bwd2_kernel<WPR><<<grid, 2 * WPR * 32, 0, st>>>(
      (const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, mean, rstd, gamma, (__nv_bfloat16*)dx, (__nv_bfloat16*)dxd,
      workspace, M, H, seed, drop_stream, in_stream, th, sc, f8)));
  dim3 g2((H + 31) / 32, 3, split);
  launch_pdl(colsum_finalize_kernel, g2, dim3(256), 0, st, (const float*)workspace, grid, H, dgamma, dbeta, dxd ? dbias : (float*)nullptr);
}

// Keep bits of one hidden-dropout site, one byte per 8 elements ([M][N / 8], bit t of byte j = element 8 j + t kept):
// the same decisions as dropout_keep8(seed, stream, e8) with e8 = (row * N + col) / 8.  Generated here, with every warp
// of the machine busy, instead of inside the GEMM epilogue that applies them (where the tensor cores idle
// meanwhile) and instead of being regenerated by the LayerNorm backward.
__global__ void __launch_bounds__(256) dropout_mask_kernel(unsigned int* __restrict__ out, long long n_words, Seed seed_in,
                                                           unsigned int stream, unsigned int thresh16) {
  pdl_trigger_small();
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
  if (g > 0) launch_pdl(dropout_mask_kernel, dim3((unsigned)g), dim3(256), 0, st, (unsigned int*)out, n_words, seed, stream, th);
}

void colsum_bf16(const void* x, int M, int N, int ld, float* out, cudaStream_t st) {
  dim3 grid((N + 255) / 256, M >= 4096 ? 64 : (M >= 512 ? 16 : 1));
  launch_pdl(colsum_bf16_kernel, grid, dim3(256), 0, st, (const __nv_bfloat16*)x, M, N, ld, out);
}

void gelu_fwd(const void* x, void* y, long long n, Fp8Out f8, cudaStream_t st) {
  const long long n8 = n >> 3;
  long long g = (n8 + 255) / 256;
  if (g > num_sms() * 32) g = num_sms() * 32;
  if (g > 0) gelu_fwd_kernel<<<(unsigned)g, 256, 0, st>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, n8, f8);
}
void dgelu_bwd(const void* dy, const void* x, void* dx, float* dbias, int M, int N, Fp8Out f8, cudaStream_t st) {
  dim3 grid((N + 255) / 256, M >= 4096 ? 74 : (M >= 512 ? 16 : 1));
  dgelu_bwd_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, (__nv_bfloat16*)dx, dbias, M, N, f8);
}

void embedding_fwd(const int* ids, const int* seg, const void* word, const void* pos, const void* type,
                   const float* gamma, const float* beta, void* e_out, void* y, float* mean, float* rstd, int M, int S,
                   int H, float eps, Seed seed, unsigned int stream, float p_drop, cudaStream_t st) {
  unsigned int th; float sc;
  drop_params(p_drop, th, sc);
  DISPATCH_CHUNKS(H, (embed_fwd_kernel<CH><<<ln_grid(M), LN_WARPS * 32, 0, st>>>(
      ids, seg, (const __nv_bfloat16*)word, (const __nv_bfloat16*)pos, (const __nv_bfloat16*)type, gamma, beta,
      (__nv_bfloat16*)e_out, (__nv_bfloat16*)y, mean, rstd, M, S, H, eps, seed, stream, th, sc)));
}

void embedding_bwd_scatter(const void* de, const int* ids, const int* seg, float* gword, float* gpos, float* gtype,
                           int M, int S, int H, int type_rows, cudaStream_t st) {
  const size_t work = (size_t)M * (H / 8);
  int grid = (int)((work + 255) / 256);
  if (grid > num_sms() * 16) grid = num_sms() * 16;
  static const bool reduce_ok = []() { const char* e = getenv("B200_EMBED_REDUCE"); return !(e && e[0] == '0'); }();
  if (reduce_ok && M % S == 0 && H % 8 == 0 && (gtype == nullptr || type_rows == 2)) {
    // word rows: scatter with atomics (30 k rows, little contention); position / token-type rows: reductions
    embed_bwd_scatter_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)de, ids, seg, gword, nullptr, nullptr, M, S, H);
    dim3 g2((H + 255) / 256, (S + 7) / 8);
    embed_bwd_postype_kernel<<<g2, 256, 0, st>>>((const __nv_bfloat16*)de, seg, gpos, gtype, M / S, S, H);
    return;
  }
  embed_bwd_scatter_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)de, ids, seg, gword, gpos, gtype, M, S, H);
}

void mlm_compact(const int* labels, int B, int S, int max_pred, int* idx, int* tgt, int* count, cudaStream_t st) {
  B200_CUDA_CHECK(cudaMemsetAsync(count, 0, sizeof(int), st));
  mlm_compact_kernel<<<B, 32, 0, st>>>(labels, S, max_pred, idx, tgt, count);
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
