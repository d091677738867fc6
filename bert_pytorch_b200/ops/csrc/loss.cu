// Softmax cross-entropy over the (masked-position) MLM logits, forward + backward in one kernel
// (SURVEY.md K23/K24).  logits are bf16 [R, V]; rows whose target is < 0 are ignored (gradient zero).
// The mean is taken over the device-side count of valid targets, so no host sync is needed to know how
// many positions were masked.  The gradient overwrites the logits in place:
//     dlogits = (softmax - onehot) * grad_scale / count          loss += sum_r (lse_r - logit_r[t_r]) / count
#include "common.cuh"
#include "kernels.h"

namespace b200 {

constexpr int CE_THREADS = 256;

// ROWS (deterministic mode): loss_out[r] receives row r's term (0 for an ignored row) instead of an atomic add into
// loss_out[0]; ordered_sum then adds the rows in order.
template <bool ROWS>
__device__ __forceinline__ void softmax_ce_body(__nv_bfloat16* __restrict__ logits, int ld, const int* __restrict__ targets,
                                                const int* __restrict__ count, float grad_scale,
                                                float* __restrict__ loss_out, int V) {
  __shared__ float sm[32];
  __shared__ float s_max, s_sum;
  const int r = blockIdx.x;
  __nv_bfloat16* row = logits + (size_t)r * ld;
  const int tgt = targets[r];
  const int nvec = V >> 3;  // V % 8 == 0
  uint4* row4 = reinterpret_cast<uint4*>(row);
  if (tgt < 0) {  // ignored position: zero gradient row
    if constexpr (ROWS) if (threadIdx.x == 0) loss_out[r] = 0.f;
    for (int i = threadIdx.x; i < nvec; i += CE_THREADS) row4[i] = make_uint4(0, 0, 0, 0);
    return;
  }
  // pass 1: online max / sum of exp
  float m = -INFINITY, s = 0.f;
  for (int i = threadIdx.x; i < nvec; i += CE_THREADS) {
    const uint4 u = row4[i];
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    float f[8];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 p = unpack_bf16(w[t]);
      f[2 * t] = p.x; f[2 * t + 1] = p.y;
    }
    float lm = f[0];
#pragma unroll
    for (int t = 1; t < 8; ++t) lm = fmaxf(lm, f[t]);
    const float nm = fmaxf(m, lm);
    float acc = 0.f;
#pragma unroll
    for (int t = 0; t < 8; ++t) acc += __expf(f[t] - nm);
    s = s * __expf(m - nm) + acc;
    m = nm;
  }
  // block combine (max first, then rescaled sums)
  float wm = warp_max(m);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) sm[warp] = wm;
  __syncthreads();
  if (warp == 0) {
    float v = lane < CE_THREADS / 32 ? sm[lane] : -INFINITY;
    v = warp_max(v);
    if (lane == 0) s_max = v;
  }
  __syncthreads();
  const float gmax = s_max;
  float part = (m == -INFINITY) ? 0.f : s * __expf(m - gmax);
  part = warp_sum(part);
  if (lane == 0) sm[warp] = part;
  __syncthreads();
  if (warp == 0) {
    float v = lane < CE_THREADS / 32 ? sm[lane] : 0.f;
    v = warp_sum(v);
    if (lane == 0) s_sum = v;
  }
  __syncthreads();
  const float inv_sum = 1.f / s_sum;
  const float cnt = (float)max(*count, 1);
  const float gs = grad_scale / cnt;
  if (threadIdx.x == 0) {
    const float lt = __bfloat162float(row[tgt]);
    if constexpr (ROWS) loss_out[r] = (logf(s_sum) + gmax - lt) / cnt;
    else atomicAdd(loss_out, (logf(s_sum) + gmax - lt) / cnt);
  }
  __syncthreads();  // the target logit was read before anyone overwrites it
  // pass 2: gradient in place
  for (int i = threadIdx.x; i < nvec; i += CE_THREADS) {
    const uint4 u = row4[i];
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    float f[8];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 p = unpack_bf16(w[t]);
      f[2 * t] = p.x; f[2 * t + 1] = p.y;
    }
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      float pr = __expf(f[t] - gmax) * inv_sum;
      if (i * 8 + t == tgt) pr -= 1.f;
      f[t] = pr * gs;
    }
    row4[i] = make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
  }
}

__global__ void __launch_bounds__(CE_THREADS)
softmax_ce_kernel(__nv_bfloat16* __restrict__ logits, int ld, const int* __restrict__ targets,
                  const int* __restrict__ count, float grad_scale, float* __restrict__ loss_out, int V) {
  softmax_ce_body<false>(logits, ld, targets, count, grad_scale, loss_out, V);
}

__global__ void __launch_bounds__(CE_THREADS)
softmax_ce_rows_kernel(__nv_bfloat16* __restrict__ logits, int ld, const int* __restrict__ targets,
                       const int* __restrict__ count, float grad_scale, float* __restrict__ loss_rows, int V) {
  softmax_ce_body<true>(logits, ld, targets, count, grad_scale, loss_rows, V);
}

void softmax_ce(void* logits, int ld, const int* targets, const int* count, float grad_scale, float* loss_out, int R,
                int V, cudaStream_t st, float* loss_rows) {
  if (R <= 0) return;
  if (loss_rows == nullptr) {
    softmax_ce_kernel<<<R, CE_THREADS, 0, st>>>((__nv_bfloat16*)logits, ld, targets, count, grad_scale, loss_out, V);
    return;
  }
  softmax_ce_rows_kernel<<<R, CE_THREADS, 0, st>>>((__nv_bfloat16*)logits, ld, targets, count, grad_scale, loss_rows, V);
  ordered_sum(loss_rows, R, 1, nullptr, 1, loss_out, st);
}

// ------------------------------------------------------------------------------------------------
// NSP head, everything after the pooler GEMM in ONE launch (SURVEY.md K20 / K25): the [B,H] x [H,2] classifier,
// its cross-entropy (ignore_index -1, mean over the valid rows), and the backward: dW[2,H], db[2] accumulated with
// atomics and the gradient of the pooler pre-activation  dz = (dlogits . W) * (1 - pooled^2)  (tanh' folded in).
// One block per sequence; pooled is the bf16 output of the pooler GEMM's bias+tanh epilogue.
// ------------------------------------------------------------------------------------------------
// ROWS (deterministic mode): sequence b stores its loss term, db and dW contributions to loss_out[b], db[2 b + k] and
// dw[2 H b + k H + i] (zeros when it contributes nothing) for ordered_sum, instead of atomics.
template <bool ROWS>
__device__ __forceinline__ void nsp_head_body(const __nv_bfloat16* __restrict__ pooled, const __nv_bfloat16* __restrict__ w,
                                              const float* __restrict__ bias, const long long* __restrict__ labels, int B,
                                              int H, float grad_scale, float* __restrict__ loss_out,
                                              __nv_bfloat16* __restrict__ dz, float* __restrict__ dw, float* __restrict__ db) {
  __shared__ float sm[32];
  __shared__ float s_bc[3];
  const int b = blockIdx.x;
  int n_valid = 0;
  for (int i = 0; i < B; ++i) n_valid += labels[i] >= 0 ? 1 : 0;      // B is ~100: cheaper than a second launch
  const long long y = labels[b];
  const __nv_bfloat16* x = pooled + (size_t)b * H;
  float a0 = 0.f, a1 = 0.f;
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    const float xv = __bfloat162float(x[i]);
    a0 += xv * __bfloat162float(w[i]);
    a1 += xv * __bfloat162float(w[H + i]);
  }
  auto block_sum = [&](float v) -> float {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) r += sm[k];
    __syncthreads();
    return r;
  };
  const float l0 = block_sum(a0) + bias[0], l1 = block_sum(a1) + bias[1];
  float d0 = 0.f, d1 = 0.f;
  if constexpr (ROWS) {
    if (threadIdx.x == 0) loss_out[b] = 0.f;
    loss_out += b; db += 2 * b; dw += (size_t)2 * H * b;
  }
  if (y >= 0 && n_valid > 0) {
    const float m = fmaxf(l0, l1);
    const float lse = m + logf(expf(l0 - m) + expf(l1 - m));
    const float p0 = expf(l0 - lse), p1 = expf(l1 - lse);
    const float inv = 1.f / (float)n_valid;
    if constexpr (ROWS) { if (threadIdx.x == 0) *loss_out = (lse - (y == 0 ? l0 : l1)) * inv; }
    else if (threadIdx.x == 0) atomicAdd(loss_out, (lse - (y == 0 ? l0 : l1)) * inv);
    d0 = (p0 - (y == 0 ? 1.f : 0.f)) * inv * grad_scale;
    d1 = (p1 - (y == 1 ? 1.f : 0.f)) * inv * grad_scale;
  }
  if constexpr (ROWS) {
    if (threadIdx.x == 0) { db[0] = d0; db[1] = d1; }
  } else if (threadIdx.x == 0 && (d0 != 0.f || d1 != 0.f)) {
    atomicAdd(db, d0);
    atomicAdd(db + 1, d1);
  }
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    const float xv = __bfloat162float(x[i]);
    const float g = d0 * __bfloat162float(w[i]) + d1 * __bfloat162float(w[H + i]);
    dz[(size_t)b * H + i] = __float2bfloat16(g * (1.f - xv * xv));
    if constexpr (ROWS) {
      const bool live = d0 != 0.f || d1 != 0.f;
      dw[i] = live ? d0 * xv : 0.f;
      dw[H + i] = live ? d1 * xv : 0.f;
    } else if (d0 != 0.f || d1 != 0.f) {
      atomicAdd(dw + i, d0 * xv);
      atomicAdd(dw + H + i, d1 * xv);
    }
  }
}

__global__ void __launch_bounds__(128)
nsp_head_kernel(const __nv_bfloat16* __restrict__ pooled, const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias,
                const long long* __restrict__ labels, int B, int H, float grad_scale, float* __restrict__ loss_out,
                __nv_bfloat16* __restrict__ dz, float* __restrict__ dw, float* __restrict__ db) {
  nsp_head_body<false>(pooled, w, bias, labels, B, H, grad_scale, loss_out, dz, dw, db);
}

__global__ void __launch_bounds__(128)
nsp_head_rows_kernel(const __nv_bfloat16* __restrict__ pooled, const __nv_bfloat16* __restrict__ w,
                     const float* __restrict__ bias, const long long* __restrict__ labels, int B, int H, float grad_scale,
                     float* __restrict__ loss_rows, __nv_bfloat16* __restrict__ dz, float* __restrict__ dw_rows,
                     float* __restrict__ db_rows) {
  nsp_head_body<true>(pooled, w, bias, labels, B, H, grad_scale, loss_rows, dz, dw_rows, db_rows);
}

void nsp_head(const void* pooled, const void* w, const float* bias, const long long* labels, int B, int H, float grad_scale,
              float* loss_out, void* dz, float* dw, float* db, cudaStream_t st, float* rows_ws) {
  if (B <= 0) return;
  if (rows_ws == nullptr) {
    nsp_head_kernel<<<B, 128, 0, st>>>((const __nv_bfloat16*)pooled, (const __nv_bfloat16*)w, bias, labels, B, H, grad_scale,
                                       loss_out, (__nv_bfloat16*)dz, dw, db);
    return;
  }
  float* loss_rows = rows_ws;                 // [B], then db [B, 2], then dW [B, 2, H]
  float* db_rows = rows_ws + B;
  float* dw_rows = rows_ws + 3 * B;
  nsp_head_rows_kernel<<<B, 128, 0, st>>>((const __nv_bfloat16*)pooled, (const __nv_bfloat16*)w, bias, labels, B, H,
                                          grad_scale, loss_rows, (__nv_bfloat16*)dz, dw_rows, db_rows);
  ordered_sum(loss_rows, B, 1, nullptr, 1, loss_out, st);
  ordered_sum(db_rows, B, 2, nullptr, 1, db, st);
  ordered_sum(dw_rows, B, 2 * H, nullptr, 1, dw, st);
}

// ------------------------------------------------------------------------------------------------
// Sequence-classification head (GLUE fine-tuning), everything after the pooler GEMM in ONE launch: dropout on the
// pooled row (keep decisions from Philox stream `stream` at element index b * H + i, rescale 1 / (1 - p)), the
// [B, H] x [H, C] classifier, its cross-entropy (mean over the rows whose label lies in [0, C); any other label is
// ignored), and the backward: db[C], dW[C, H] and  dz = (dlogits . W) * keep / (1 - p) * (1 - pooled^2).  One block per
// sequence; C (2 or 3, the GLUE classification tasks) is a template parameter so that the logits stay in registers.
// ROWS (deterministic mode): sequence b stores its loss term, db and dW contributions to loss_out[b], db[C b + c] and
// dw[C H b + c H + i] (zeros when it contributes nothing) for ordered_sum, instead of atomics.
// ------------------------------------------------------------------------------------------------
constexpr int CLS_THREADS = 128;

// 8 consecutive pooled values of group g (elements 8 g .. 8 g + 7 of the row) and their dropout multipliers
__device__ __forceinline__ void cls_load8(const __nv_bfloat16* __restrict__ x, int g, float (&xv)[8]) {
  const uint4 u = reinterpret_cast<const uint4*>(x)[g];
  const uint32_t wd[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const float2 p = unpack_bf16(wd[t]);
    xv[2 * t] = p.x; xv[2 * t + 1] = p.y;
  }
}

__device__ __forceinline__ void cls_keep8(unsigned long long seed, unsigned stream, unsigned thresh16, float keep_scale,
                                          unsigned long long e8, float (&mul)[8]) {
  if (thresh16 == 0u) {
#pragma unroll
    for (int t = 0; t < 8; ++t) mul[t] = 1.f;
    return;
  }
  const Keep8 k = dropout_keep8(seed, stream, e8, thresh16);
#pragma unroll
  for (int t = 0; t < 8; ++t) mul[t] = k[t] ? keep_scale : 0.f;
}

// the C partial sums of every thread added over the block in a fixed order; every thread gets the totals
template <int C>
__device__ __forceinline__ void cls_block_sum(float (&a)[C], float* sm) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const float v = warp_sum(a[c]);
    if (lane == 0) sm[warp * C + c] = v;
  }
  __syncthreads();
#pragma unroll
  for (int c = 0; c < C; ++c) {
    float r = 0.f;
    for (int k = 0; k < CLS_THREADS / 32; ++k) r += sm[k * C + c];
    a[c] = r;
  }
  __syncthreads();
}

// logits of row x (H % 8 == 0) after the dropout multipliers of its elements (all 1 without dropout)
template <int C>
__device__ __forceinline__ void cls_logits_row(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                                               const float* __restrict__ bias, int H, unsigned long long seed,
                                               unsigned stream, unsigned thresh16, float keep_scale,
                                               unsigned long long e8_row, float (&l)[C], float* sm) {
#pragma unroll
  for (int c = 0; c < C; ++c) l[c] = 0.f;
  for (int g = threadIdx.x; g < (H >> 3); g += CLS_THREADS) {
    float xv[8], mul[8];
    cls_load8(x, g, xv);
    cls_keep8(seed, stream, thresh16, keep_scale, e8_row + (unsigned long long)g, mul);
#pragma unroll
    for (int c = 0; c < C; ++c) {
      float wv[8];
      cls_load8(w + (size_t)c * H, g, wv);
#pragma unroll
      for (int t = 0; t < 8; ++t) l[c] += xv[t] * mul[t] * wv[t];
    }
  }
  cls_block_sum<C>(l, sm);
#pragma unroll
  for (int c = 0; c < C; ++c) l[c] += bias[c];
}

template <int C, bool ROWS>
__global__ void __launch_bounds__(CLS_THREADS)
cls_head_kernel(const __nv_bfloat16* __restrict__ pooled, const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias,
                const long long* __restrict__ labels, int B, int H, float grad_scale, Seed seed, unsigned stream,
                unsigned thresh16, float keep_scale, float* __restrict__ loss_out, __nv_bfloat16* __restrict__ dz,
                float* __restrict__ dw, float* __restrict__ db) {
  __shared__ float sm[(CLS_THREADS / 32) * C];
  const int b = blockIdx.x;
  int n_valid = 0;
  for (int i = 0; i < B; ++i) n_valid += (labels[i] >= 0 && labels[i] < C) ? 1 : 0;   // B is small: no second launch
  const long long y = labels[b];
  const bool live = y >= 0 && y < C;                 // then n_valid >= 1
  const __nv_bfloat16* x = pooled + (size_t)b * H;
  const unsigned long long sd = seed.value();
  const unsigned long long e8_row = (unsigned long long)b * (unsigned long long)(H >> 3);
  float l[C];
  cls_logits_row<C>(x, w, bias, H, sd, stream, thresh16, keep_scale, e8_row, l, sm);
  float d[C];
#pragma unroll
  for (int c = 0; c < C; ++c) d[c] = 0.f;
  if constexpr (ROWS) {
    loss_out += b; db += C * b; dw += (size_t)C * H * b;
  }
  float term = 0.f;
  if (live) {
    float m = l[0], ly = l[0];
#pragma unroll
    for (int c = 1; c < C; ++c) {
      m = fmaxf(m, l[c]);
      if (c == y) ly = l[c];
    }
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) s += expf(l[c] - m);
    const float lse = m + logf(s);
    const float inv = 1.f / (float)n_valid;
    term = (lse - ly) * inv;
#pragma unroll
    for (int c = 0; c < C; ++c) d[c] = (expf(l[c] - lse) - (c == y ? 1.f : 0.f)) * inv * grad_scale;
  }
  if (threadIdx.x == 0) {
    if constexpr (ROWS) {
      *loss_out = term;
#pragma unroll
      for (int c = 0; c < C; ++c) db[c] = d[c];
    } else if (live) {
      atomicAdd(loss_out, term);
#pragma unroll
      for (int c = 0; c < C; ++c) atomicAdd(db + c, d[c]);
    }
  }
  for (int g = threadIdx.x; g < (H >> 3); g += CLS_THREADS) {
    float xv[8], mul[8], dx[8];
    cls_load8(x, g, xv);
    cls_keep8(sd, stream, thresh16, keep_scale, e8_row + (unsigned long long)g, mul);
#pragma unroll
    for (int t = 0; t < 8; ++t) dx[t] = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      float wv[8];
      cls_load8(w + (size_t)c * H, g, wv);
#pragma unroll
      for (int t = 0; t < 8; ++t) dx[t] += d[c] * wv[t];
    }
    float o[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) o[t] = dx[t] * mul[t] * (1.f - xv[t] * xv[t]);
    reinterpret_cast<uint4*>(dz + (size_t)b * H)[g] =
        make_uint4(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]), pack_bf16(o[4], o[5]), pack_bf16(o[6], o[7]));
#pragma unroll
    for (int c = 0; c < C; ++c) {
      float* dwc = dw + (size_t)c * H + 8 * g;
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const float v = d[c] * xv[t] * mul[t];
        if constexpr (ROWS) dwc[t] = live ? v : 0.f;
        else if (live) atomicAdd(dwc + t, v);
      }
    }
  }
}

// evaluation form: fp32 logits [B, C] of the pooled rows, no dropout, the training kernel's dot-product order
template <int C>
__global__ void __launch_bounds__(CLS_THREADS)
cls_logits_kernel(const __nv_bfloat16* __restrict__ pooled, const __nv_bfloat16* __restrict__ w,
                  const float* __restrict__ bias, int H, float* __restrict__ logits) {
  __shared__ float sm[(CLS_THREADS / 32) * C];
  float l[C];
  cls_logits_row<C>(pooled + (size_t)blockIdx.x * H, w, bias, H, 0ull, 0u, 0u, 1.f, 0ull, l, sm);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int c = 0; c < C; ++c) logits[(size_t)blockIdx.x * C + c] = l[c];
  }
}

template <int C>
static void cls_head_launch(const void* pooled, const void* w, const float* bias, const long long* labels, int B, int H,
                            float grad_scale, Seed seed, unsigned stream, float p_drop, float* loss_out, void* dz,
                            float* dw, float* db, cudaStream_t st, float* rows_ws) {
  const unsigned thresh = p_drop > 0.f ? (unsigned)(p_drop * 65536.f + 0.5f) : 0u;
  const float scale = p_drop > 0.f ? 65536.f / (65536.f - (float)thresh) : 1.f;
  const auto* x = (const __nv_bfloat16*)pooled;
  const auto* wb = (const __nv_bfloat16*)w;
  if (rows_ws == nullptr) {
    cls_head_kernel<C, false><<<B, CLS_THREADS, 0, st>>>(x, wb, bias, labels, B, H, grad_scale, seed, stream, thresh,
                                                         scale, loss_out, (__nv_bfloat16*)dz, dw, db);
    return;
  }
  float* loss_rows = rows_ws;                 // [B], then db [B, C], then dW [B, C, H]
  float* db_rows = rows_ws + B;
  float* dw_rows = rows_ws + (size_t)(1 + C) * B;
  cls_head_kernel<C, true><<<B, CLS_THREADS, 0, st>>>(x, wb, bias, labels, B, H, grad_scale, seed, stream, thresh, scale,
                                                      loss_rows, (__nv_bfloat16*)dz, dw_rows, db_rows);
  ordered_sum(loss_rows, B, 1, nullptr, 1, loss_out, st);
  ordered_sum(db_rows, B, C, nullptr, 1, db, st);
  ordered_sum(dw_rows, B, C * H, nullptr, 1, dw, st);
}

void cls_head(const void* pooled, const void* w, const float* bias, const long long* labels, int B, int H, int C,
              float grad_scale, Seed seed, unsigned stream, float p_drop, float* loss_out, void* dz, float* dw, float* db,
              cudaStream_t st, float* rows_ws) {
  if (B <= 0) return;
  if (C == 2) cls_head_launch<2>(pooled, w, bias, labels, B, H, grad_scale, seed, stream, p_drop, loss_out, dz, dw, db, st, rows_ws);
  else if (C == 3) cls_head_launch<3>(pooled, w, bias, labels, B, H, grad_scale, seed, stream, p_drop, loss_out, dz, dw, db, st, rows_ws);
}

void cls_logits(const void* pooled, const void* w, const float* bias, int B, int H, int C, float* logits, cudaStream_t st) {
  if (B <= 0) return;
  const auto* x = (const __nv_bfloat16*)pooled;
  const auto* wb = (const __nv_bfloat16*)w;
  if (C == 2) cls_logits_kernel<2><<<B, CLS_THREADS, 0, st>>>(x, wb, bias, H, logits);
  else if (C == 3) cls_logits_kernel<3><<<B, CLS_THREADS, 0, st>>>(x, wb, bias, H, logits);
}

// ------------------------------------------------------------------------------------------------
// Evaluation metrics (forward only; the inputs are only read).  Every row r writes rows[r] = {loss, correct, valid}:
// the cross-entropy of its target, whether the argmax is the target, and 1 -- or {0, 0, 0} for an ignored row.  The
// rows are then added by ordered_sum in a fixed order: no atomics, so the sums are the same bits in every mode.
// ------------------------------------------------------------------------------------------------

// (value, index) pair that wins an argmax: the larger value, and the lower index among equal values
__device__ __forceinline__ void argmax_take(float& v, int& i, float ov, int oi) {
  if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
}

// One block per row of bf16 logits [R, V] (V % 8 == 0, row stride ld).  The loss is the forward half of
// softmax_ce_body with the same block shape and the same arithmetic, so that both give the same per-row term.  A target
// outside [0, V) counts as ignored.
__global__ void __launch_bounds__(CE_THREADS)
mlm_eval_kernel(const __nv_bfloat16* __restrict__ logits, int ld, const int* __restrict__ targets, int V,
                float* __restrict__ rows) {
  __shared__ float sm[32];
  __shared__ int si[32];
  __shared__ float s_max, s_sum;
  __shared__ int s_arg;
  const int r = blockIdx.x;
  const __nv_bfloat16* row = logits + (size_t)r * ld;
  const int tgt = targets[r];
  if (tgt < 0 || tgt >= V) {
    if (threadIdx.x < 3) rows[(size_t)r * 3 + threadIdx.x] = 0.f;
    return;
  }
  const int nvec = V >> 3;
  const uint4* row4 = reinterpret_cast<const uint4*>(row);
  float m = -INFINITY, s = 0.f;
  float bv = -INFINITY;
  int bi = V;                        // no index yet (a row of NaN has no argmax and is never correct)
  for (int i = threadIdx.x; i < nvec; i += CE_THREADS) {
    const uint4 u = row4[i];
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    float f[8];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 p = unpack_bf16(w[t]);
      f[2 * t] = p.x; f[2 * t + 1] = p.y;
    }
    float lm = f[0];
#pragma unroll
    for (int t = 1; t < 8; ++t) lm = fmaxf(lm, f[t]);
    const float nm = fmaxf(m, lm);
    float acc = 0.f;
#pragma unroll
    for (int t = 0; t < 8; ++t) acc += __expf(f[t] - nm);
    s = s * __expf(m - nm) + acc;
    m = nm;
#pragma unroll
    for (int t = 0; t < 8; ++t)      // a thread visits its indices in increasing order: strict > keeps the lowest
      if (f[t] > bv) { bv = f[t]; bi = i * 8 + t; }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // block combine of the softmax statistics: softmax_ce_body's order
  float wm = warp_max(m);
  if (lane == 0) sm[warp] = wm;
  __syncthreads();
  if (warp == 0) {
    float v = lane < CE_THREADS / 32 ? sm[lane] : -INFINITY;
    v = warp_max(v);
    if (lane == 0) s_max = v;
  }
  __syncthreads();
  const float gmax = s_max;
  float part = (m == -INFINITY) ? 0.f : s * __expf(m - gmax);
  part = warp_sum(part);
  if (lane == 0) sm[warp] = part;
  __syncthreads();
  if (warp == 0) {
    float v = lane < CE_THREADS / 32 ? sm[lane] : 0.f;
    v = warp_sum(v);
    if (lane == 0) s_sum = v;
  }
  // block combine of the argmax
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    argmax_take(bv, bi, __shfl_xor_sync(0xffffffffu, bv, o), __shfl_xor_sync(0xffffffffu, bi, o));
  __syncthreads();                   // sm is free again (warp 0 has read it)
  if (lane == 0) { sm[warp] = bv; si[warp] = bi; }
  __syncthreads();
  if (warp == 0) {
    float v = lane < CE_THREADS / 32 ? sm[lane] : -INFINITY;
    int k = lane < CE_THREADS / 32 ? si[lane] : V;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
      argmax_take(v, k, __shfl_xor_sync(0xffffffffu, v, o), __shfl_xor_sync(0xffffffffu, k, o));
    if (lane == 0) s_arg = k;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const float lt = __bfloat162float(row[tgt]);
    rows[(size_t)r * 3 + 0] = logf(s_sum) + gmax - lt;
    rows[(size_t)r * 3 + 1] = s_arg == tgt ? 1.f : 0.f;
    rows[(size_t)r * 3 + 2] = 1.f;
  }
}

void mlm_eval(const void* logits, int ld, const int* targets, int R, int V, float* rows, float* sums, cudaStream_t st) {
  if (R <= 0) return;
  mlm_eval_kernel<<<R, CE_THREADS, 0, st>>>((const __nv_bfloat16*)logits, ld, targets, V, rows);
  ordered_sum(rows, R, 3, nullptr, 1, sums, st);
}

// One block per sequence: the NSP classifier and its cross-entropy with nsp_head_body's block shape and arithmetic.  The
// prediction is class 1 only when its logit is strictly larger (a tie goes to class 0, torch.argmax's rule).
__global__ void __launch_bounds__(128)
nsp_eval_kernel(const __nv_bfloat16* __restrict__ pooled, const __nv_bfloat16* __restrict__ w,
                const float* __restrict__ bias, const long long* __restrict__ labels, int H, float* __restrict__ rows) {
  __shared__ float sm[32];
  const int b = blockIdx.x;
  const long long y = labels[b];
  float* out = rows + (size_t)b * 3;
  if (y < 0 || y > 1) {
    if (threadIdx.x < 3) out[threadIdx.x] = 0.f;
    return;
  }
  const __nv_bfloat16* x = pooled + (size_t)b * H;
  float a0 = 0.f, a1 = 0.f;
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    const float xv = __bfloat162float(x[i]);
    a0 += xv * __bfloat162float(w[i]);
    a1 += xv * __bfloat162float(w[H + i]);
  }
  auto block_sum = [&](float v) -> float {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) r += sm[k];
    __syncthreads();
    return r;
  };
  const float l0 = block_sum(a0) + bias[0], l1 = block_sum(a1) + bias[1];
  if (threadIdx.x == 0) {
    const float m = fmaxf(l0, l1);
    const float lse = m + logf(expf(l0 - m) + expf(l1 - m));
    out[0] = lse - (y == 0 ? l0 : l1);
    out[1] = (l1 > l0 ? 1 : 0) == y ? 1.f : 0.f;
    out[2] = 1.f;
  }
}

void nsp_eval(const void* pooled, const void* w, const float* bias, const long long* labels, int B, int H, float* rows,
              float* sums, cudaStream_t st) {
  if (B <= 0) return;
  nsp_eval_kernel<<<B, 128, 0, st>>>((const __nv_bfloat16*)pooled, (const __nv_bfloat16*)w, bias, labels, H, rows);
  ordered_sum(rows, B, 3, nullptr, 1, sums, st);
}

// ------------------------------------------------------------------------------------------------
// Per-token heads (SQuAD start / end, NER token classifier): a [M, H] x [H, N] classifier over every row of the
// sequence output, N in 1..64, with Philox dropout on the seq elements (index row * H + i).  Dropped elements are
// zeroed in bf16 (exact) and the keep scale 1 / (1 - p) multiplies the fp32 result, so the kept products are never
// rounded again.  Forward (token_logits): bf16 mma.sync with fp32 accumulation, seq read once, W staged through shared
// memory in 64-column chunks.  Losses (token_ce, span_ce): in place on the fp32 logits.  Backward (token_head_bwd):
// d_seq = (dlogits . W) * keep * scale on fp32 FMAs, and dW / db accumulated per CTA over a fixed 512-row partition of
// the rows, then added with one atomic per CTA and element (or stored per partition and added by ordered_sum in
// deterministic mode).
// ------------------------------------------------------------------------------------------------
constexpr int TOK_THREADS = 128;            // forward: 4 warps x 16 rows
constexpr int TOK_ROWS = 64;
constexpr int TOK_KC = 64;                  // H columns per staged chunk
constexpr int TOK_LD = TOK_KC + 8;          // padded smem row: 36 words, so the fragment loads hit 32 distinct banks

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
               "{%0,%1,%2,%3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 8 consecutive bf16 values with the dropped ones zeroed (keep bits of group e8; thresh16 == 0: no dropout)
__device__ __forceinline__ uint4 tok_keep(uint4 u, const Keep8& k, unsigned thresh16) {
  if (thresh16 == 0u) return u;
  uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int t = 0; t < 4; ++t) w[t] &= (k[2 * t] ? 0x0000FFFFu : 0u) | (k[2 * t + 1] ? 0xFFFF0000u : 0u);
  return make_uint4(w[0], w[1], w[2], w[3]);
}

__device__ __forceinline__ Keep8 tok_keep8(unsigned long long seed, unsigned stream, unsigned long long e8,
                                           unsigned thresh16) {
  return thresh16 == 0u ? Keep8::all() : dropout_keep8(seed, stream, e8, thresh16);
}

// NT n-tiles of 8 outputs (N <= 8 NT).  Thread tid stages 16-byte group (tid & 7) of rows tid / 8 + 16 i of the x chunk.
template <int NT>
__global__ void __launch_bounds__(TOK_THREADS)
token_logits_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                    const float* __restrict__ bias, int M, int H, int N, Seed seed, unsigned stream, unsigned thresh16,
                    float keep_scale, float* __restrict__ out) {
  __shared__ __align__(16) __nv_bfloat16 xs[TOK_ROWS * TOK_LD];
  __shared__ __align__(16) __nv_bfloat16 wsm[8 * NT * TOK_LD];
  constexpr int WV = (64 * NT + TOK_THREADS - 1) / TOK_THREADS;    // 16-byte W groups per thread and chunk
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int row0 = blockIdx.x * TOK_ROWS, hg = H >> 3;
  const unsigned long long sd = seed.value();
  const uint4 zero = make_uint4(0, 0, 0, 0);
  float acc[NT][4];
#pragma unroll
  for (int n = 0; n < NT; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;
  uint4 xr[4], wr[WV];
  auto load = [&](int k0) {
    const int gi = (k0 >> 3) + (tid & 7);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = row0 + (tid >> 3) + 16 * i;
      xr[i] = (r < M && gi < hg) ? __ldg(reinterpret_cast<const uint4*>(x + (size_t)r * H) + gi) : zero;
    }
#pragma unroll
    for (int j = 0; j < WV; ++j) {
      const int idx = tid + j * TOK_THREADS, n = idx >> 3, gj = (k0 >> 3) + (idx & 7);
      wr[j] = (n < N && gj < hg) ? __ldg(reinterpret_cast<const uint4*>(w + (size_t)n * H) + gj) : zero;
    }
  };
  auto store = [&](int k0) {
    const int gi = (k0 >> 3) + (tid & 7);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int rl = (tid >> 3) + 16 * i;
      const Keep8 k = tok_keep8(sd, stream, (unsigned long long)(row0 + rl) * hg + gi, thresh16);
      *reinterpret_cast<uint4*>(xs + rl * TOK_LD + (tid & 7) * 8) = tok_keep(xr[i], k, thresh16);
    }
#pragma unroll
    for (int j = 0; j < WV; ++j) {
      const int idx = tid + j * TOK_THREADS;
      if (idx < 64 * NT) *reinterpret_cast<uint4*>(wsm + (idx >> 3) * TOK_LD + (idx & 7) * 8) = wr[j];
    }
  };
  load(0);
  for (int k0 = 0; k0 < H; k0 += TOK_KC) {
    store(k0);
    __syncthreads();
    if (k0 + TOK_KC < H) load(k0 + TOK_KC);          // the next chunk's loads fly under this chunk's MMAs
#pragma unroll
    for (int kk = 0; kk < TOK_KC; kk += 16) {
      const __nv_bfloat16* xa = xs + (warp * 16 + g) * TOK_LD + kk + 2 * t;
      uint32_t a[4];
      a[0] = *reinterpret_cast<const uint32_t*>(xa);
      a[1] = *reinterpret_cast<const uint32_t*>(xa + 8 * TOK_LD);
      a[2] = *reinterpret_cast<const uint32_t*>(xa + 8);
      a[3] = *reinterpret_cast<const uint32_t*>(xa + 8 * TOK_LD + 8);
#pragma unroll
      for (int n = 0; n < NT; ++n) {
        const __nv_bfloat16* wb = wsm + (n * 8 + g) * TOK_LD + kk + 2 * t;
        mma_bf16_16816(acc[n], a, *reinterpret_cast<const uint32_t*>(wb), *reinterpret_cast<const uint32_t*>(wb + 8));
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int n = 0; n < NT; ++n) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row0 + warp * 16 + g + 8 * h;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = n * 8 + 2 * t + e;
        if (r < M && c < N) out[(size_t)r * N + c] = acc[n][2 * h + e] * keep_scale + bias[c];
      }
    }
  }
}

static unsigned tok_thresh(float p_drop) { return p_drop > 0.f ? (unsigned)(p_drop * 65536.f + 0.5f) : 0u; }
static float tok_scale(unsigned thresh) { return thresh ? 65536.f / (65536.f - (float)thresh) : 1.f; }

void token_logits(const void* x, const void* w, const float* bias, int M, int H, int N, Seed seed, unsigned stream,
                  float p_drop, float* out, cudaStream_t st) {
  if (M <= 0) return;
  const unsigned th = tok_thresh(p_drop);
  const float sc = tok_scale(th);
  const auto* xb = (const __nv_bfloat16*)x;
  const auto* wb = (const __nv_bfloat16*)w;
  const int grid = (M + TOK_ROWS - 1) / TOK_ROWS;
  if (N <= 8) token_logits_kernel<1><<<grid, TOK_THREADS, 0, st>>>(xb, wb, bias, M, H, N, seed, stream, th, sc, out);
  else if (N <= 16) token_logits_kernel<2><<<grid, TOK_THREADS, 0, st>>>(xb, wb, bias, M, H, N, seed, stream, th, sc, out);
  else if (N <= 32) token_logits_kernel<4><<<grid, TOK_THREADS, 0, st>>>(xb, wb, bias, M, H, N, seed, stream, th, sc, out);
  else token_logits_kernel<8><<<grid, TOK_THREADS, 0, st>>>(xb, wb, bias, M, H, N, seed, stream, th, sc, out);
}

// out [P, N]: the logits of packed row row_map[p], or the bias at a masked position (mask[p] == 0; the packed rows of
// an all-zero mask row are computed, but belong to no position)
__global__ void token_unpack_kernel(const float* __restrict__ logits, const int* __restrict__ row_map,
                                    const int* __restrict__ mask, const float* __restrict__ bias, int P, int N,
                                    float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)P * N) return;
  const int p = (int)(i / N), n = (int)(i - (long long)p * N);
  const int r = row_map[p];
  out[i] = (mask[p] != 0 && r >= 0) ? logits[(size_t)r * N + n] : bias[n];
}

void token_unpack(const float* logits, const int* row_map, const int* mask, const float* bias, int P, int N, float* out,
                  cudaStream_t st) {
  const long long n = (long long)P * N;
  if (n <= 0) return;
  token_unpack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(logits, row_map, mask, bias, P, N, out);
}

// ---- NER cross-entropy.  Position p counts iff mask[p] == 1 (no mask: always) and 0 <= labels[p] < N; its logits row
// is row_map[p] (packed) or p.  Pass 1 (one CTA): inv[row] = the counted position of every logits row or -1, and the
// count.  Pass 2: one warp per row, 64 rows per CTA; counted rows get (softmax - onehot) * grad_scale / count, every
// other row zero, and each CTA adds its rows' loss terms in a fixed order.
constexpr int TCE_ROWS = 64;

__global__ void __launch_bounds__(1024)
token_ce_index_kernel(const int* __restrict__ labels, const int* __restrict__ mask, const int* __restrict__ row_map,
                      int P, int R, int N, int* __restrict__ inv, int* __restrict__ count) {
  __shared__ int s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  for (int i = threadIdx.x; i < R; i += blockDim.x) inv[i] = -1;
  __syncthreads();
  int c = 0;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const int y = labels[p];
    const int r = row_map != nullptr ? row_map[p] : p;
    if ((mask == nullptr || mask[p] == 1) && y >= 0 && y < N && r >= 0 && r < R) {
      inv[r] = p;
      ++c;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_cnt, c);        // integer adds: the same count in every order
  __syncthreads();
  if (threadIdx.x == 0) *count = s_cnt;
}

template <bool PART>
__global__ void __launch_bounds__(256)
token_ce_kernel(float* __restrict__ logits, const int* __restrict__ labels, const int* __restrict__ inv,
                const int* __restrict__ count, int R, int N, float grad_scale, float* __restrict__ loss_out) {
  __shared__ float sm[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float cnt = (float)max(*count, 1);
  const float gs = grad_scale / cnt;
  float wloss = 0.f;
  for (int i = 0; i < TCE_ROWS / 8; ++i) {
    const int r = blockIdx.x * TCE_ROWS + warp * (TCE_ROWS / 8) + i;
    if (r >= R) break;
    float* row = logits + (size_t)r * N;
    const int p = inv[r];
    if (p < 0) {
      if (lane < N) row[lane] = 0.f;
      if (lane + 32 < N) row[lane + 32] = 0.f;
      continue;
    }
    const int y = labels[p];
    const float v0 = lane < N ? row[lane] : -INFINITY, v1 = lane + 32 < N ? row[lane + 32] : -INFINITY;
    const float m = warp_max(fmaxf(v0, v1));
    const float e0 = lane < N ? __expf(v0 - m) : 0.f, e1 = lane + 32 < N ? __expf(v1 - m) : 0.f;
    const float s = warp_sum(e0 + e1);
    const float a0 = __shfl_sync(0xffffffffu, v0, y & 31), a1 = __shfl_sync(0xffffffffu, v1, y & 31);
    const float ly = y < 32 ? a0 : a1;
    if (lane == 0) wloss += (logf(s) + m - ly) / cnt;
    const float inv_s = 1.f / s;
    if (lane < N) row[lane] = (e0 * inv_s - (lane == y ? 1.f : 0.f)) * gs;
    if (lane + 32 < N) row[lane + 32] = (e1 * inv_s - (lane + 32 == y ? 1.f : 0.f)) * gs;
  }
  if (lane == 0) sm[warp] = wloss;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f;
    for (int k = 0; k < 8; ++k) tot += sm[k];
    if constexpr (PART) loss_out[blockIdx.x] = tot;
    else if (tot != 0.f) atomicAdd(loss_out, tot);
  }
}

int token_ce_parts(int R) { return (R + TCE_ROWS - 1) / TCE_ROWS; }

void token_ce(float* logits, const int* labels, const int* mask, const int* row_map, int P, int R, int N,
              float grad_scale, float* loss_out, int* idx_ws, float* part, cudaStream_t st) {
  if (R <= 0) return;
  int* inv = idx_ws;
  int* count = idx_ws + R;
  token_ce_index_kernel<<<1, 1024, 0, st>>>(labels, mask, row_map, P, R, N, inv, count);
  const int grid = token_ce_parts(R);
  if (part == nullptr) {
    token_ce_kernel<false><<<grid, 256, 0, st>>>(logits, labels, inv, count, R, N, grad_scale, loss_out);
    return;
  }
  token_ce_kernel<true><<<grid, 256, 0, st>>>(logits, labels, inv, count, R, N, grad_scale, part);
  ordered_sum(part, grid, 1, nullptr, 1, loss_out, st);
}

// ---- SQuAD span cross-entropy: one CTA per sequence, softmax over its S positions, separately for the start (column
// 0) and end (column 1) logits.  Positions are clamped to [0, S] and S is ignored; each column's mean is over its own
// count of non-ignored sequences, and the loss is the average of the two means.
constexpr int SPAN_THREADS = 256;

__device__ __forceinline__ float span_block_reduce(float v, bool is_max, float* sm) {
  v = is_max ? warp_max(v) : warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) sm[warp] = v;
  __syncthreads();
  float r = sm[0];
  for (int k = 1; k < SPAN_THREADS / 32; ++k) r = is_max ? fmaxf(r, sm[k]) : r + sm[k];
  __syncthreads();
  return r;
}

template <bool PART>
__global__ void __launch_bounds__(SPAN_THREADS)
span_ce_kernel(float* __restrict__ logits, const int* __restrict__ start, const int* __restrict__ end, int B, int S,
               float grad_scale, float* __restrict__ loss_out) {
  __shared__ float sm[SPAN_THREADS / 32];
  const int b = blockIdx.x;
  auto clampS = [S](int v) { return v < 0 ? 0 : (v > S ? S : v); };
  int cnt[2] = {0, 0};
  for (int i = 0; i < B; ++i) {                       // B is small: cheaper than a second launch
    cnt[0] += clampS(start[i]) != S ? 1 : 0;
    cnt[1] += clampS(end[i]) != S ? 1 : 0;
  }
  const int ys[2] = {clampS(start[b]), clampS(end[b])};
  float* base = logits + (size_t)b * S * 2;
  float term = 0.f;
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const int y = ys[c];
    if (y == S) {                                     // ignored: zero gradient
      for (int s = threadIdx.x; s < S; s += SPAN_THREADS) base[2 * s + c] = 0.f;
      continue;
    }
    const float ly = base[2 * y + c];                 // read before any thread writes (the reductions sync)
    float m = -INFINITY;
    for (int s = threadIdx.x; s < S; s += SPAN_THREADS) m = fmaxf(m, base[2 * s + c]);
    m = span_block_reduce(m, true, sm);
    float sum = 0.f;
    for (int s = threadIdx.x; s < S; s += SPAN_THREADS) sum += __expf(base[2 * s + c] - m);
    sum = span_block_reduce(sum, false, sm);
    const float w = 0.5f / (float)cnt[c];
    term += (logf(sum) + m - ly) * w;
    const float gs = grad_scale * w, inv_s = 1.f / sum;
    for (int s = threadIdx.x; s < S; s += SPAN_THREADS)
      base[2 * s + c] = (__expf(base[2 * s + c] - m) * inv_s - (s == y ? 1.f : 0.f)) * gs;
  }
  if (threadIdx.x == 0) {
    if constexpr (PART) loss_out[b] = term;
    else if (term != 0.f) atomicAdd(loss_out, term);
  }
}

void span_ce(float* logits, const int* start, const int* end, int B, int S, float grad_scale, float* loss_out,
             float* part, cudaStream_t st) {
  if (B <= 0 || S <= 0) return;
  if (part == nullptr) {
    span_ce_kernel<false><<<B, SPAN_THREADS, 0, st>>>(logits, start, end, B, S, grad_scale, loss_out);
    return;
  }
  span_ce_kernel<true><<<B, SPAN_THREADS, 0, st>>>(logits, start, end, B, S, grad_scale, part);
  ordered_sum(part, B, 1, nullptr, 1, loss_out, st);
}

// ---- backward.  CTA (x, y): H columns 64 x .. 64 x + 63 of rows 512 y .. 512 y + 511, walked in 64-row tiles.  Thread
// (tr = tid / 8, tc = tid % 8) stages and computes 8 columns of rows tr and tr + 32 of a tile (one Philox call per
// 8 elements), and accumulates dW for outputs tr + 32 j (j < NJ) over all the partition's rows.
constexpr int TB_THREADS = 256, TB_ROWS = 64, TB_COLS = 64, TB_PART_ROWS = 512;

template <int NJ>
__global__ void __launch_bounds__(TB_THREADS)
token_head_bwd_kernel(const float* __restrict__ dl, const __nv_bfloat16* __restrict__ x,
                      const __nv_bfloat16* __restrict__ w, int M, int H, int N, Seed seed, unsigned stream,
                      unsigned thresh16, float keep_scale, __nv_bfloat16* __restrict__ dx, float* __restrict__ dw,
                      float* __restrict__ db, float* __restrict__ ws_dw, float* __restrict__ ws_db) {
  __shared__ float dls[TB_ROWS][65];
  __shared__ __align__(16) __nv_bfloat16 wsm[64][TB_COLS];
  __shared__ __align__(16) __nv_bfloat16 xk[TB_ROWS][TB_COLS];
  const int tid = threadIdx.x, tc = tid & 7, tr = tid >> 3;
  const int c0 = blockIdx.x * TB_COLS, hg = H >> 3, gcol = (c0 >> 3) + tc;
  const bool colok = gcol < hg;
  const int rbeg = blockIdx.y * TB_PART_ROWS, rend = min(M, rbeg + TB_PART_ROWS);
  const unsigned long long sd = seed.value();
  const uint4 zero = make_uint4(0, 0, 0, 0);
  for (int i = tid; i < 64 * 8; i += TB_THREADS) {
    const int n = i >> 3, gg = (c0 >> 3) + (i & 7);
    *reinterpret_cast<uint4*>(&wsm[n][(i & 7) * 8]) =
        (n < N && gg < hg) ? __ldg(reinterpret_cast<const uint4*>(w + (size_t)n * H) + gg) : zero;
  }
  float acc[NJ][8];
#pragma unroll
  for (int j = 0; j < NJ; ++j)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[j][e] = 0.f;
  float dbacc = 0.f;
  for (int r0 = rbeg; r0 < rend; r0 += TB_ROWS) {
    __syncthreads();                                  // the previous tile's shared reads are done
    for (int i = tid; i < TB_ROWS * N; i += TB_THREADS) {
      const int rl = i / N, n = i - rl * N;
      dls[rl][n] = r0 + rl < rend ? dl[(size_t)(r0 + rl) * N + n] : 0.f;
    }
    Keep8 keep[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int rl = tr + 32 * h, r = r0 + rl;
      const bool ok = r < rend && colok;
      keep[h] = tok_keep8(sd, stream, (unsigned long long)r * hg + gcol, ok ? thresh16 : 0u);
      const uint4 u = ok ? __ldg(reinterpret_cast<const uint4*>(x + (size_t)r * H) + gcol) : zero;
      *reinterpret_cast<uint4*>(&xk[rl][tc * 8]) = tok_keep(u, keep[h], thresh16);
    }
    __syncthreads();
    // d_seq of this thread's two rows
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int rl = tr + 32 * h, r = r0 + rl;
      if (r >= rend || !colok) continue;
      float d[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) d[e] = 0.f;
      for (int n = 0; n < N; ++n) {
        const float gv = dls[rl][n];
        const uint4 u = *reinterpret_cast<const uint4*>(&wsm[n][tc * 8]);
        const uint32_t wd[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 p = unpack_bf16(wd[q]);
          d[2 * q] += gv * p.x;
          d[2 * q + 1] += gv * p.y;
        }
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) d[e] = keep[h][e] ? d[e] * keep_scale : 0.f;
      reinterpret_cast<uint4*>(dx + (size_t)r * H)[gcol] =
          make_uint4(pack_bf16(d[0], d[1]), pack_bf16(d[2], d[3]), pack_bf16(d[4], d[5]), pack_bf16(d[6], d[7]));
    }
    // dW += dlogits^T . dropped x over the tile's rows, in row order
    const int nrows = min(TB_ROWS, rend - r0);
    for (int rl = 0; rl < nrows; ++rl) {
      const uint4 u = *reinterpret_cast<const uint4*>(&xk[rl][tc * 8]);
      const uint32_t xd[4] = {u.x, u.y, u.z, u.w};
      float xv[8];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 p = unpack_bf16(xd[q]);
        xv[2 * q] = p.x; xv[2 * q + 1] = p.y;
      }
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int n = tr + 32 * j;
        const float gv = n < N ? dls[rl][n] : 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[j][e] += gv * xv[e];
      }
    }
    if (blockIdx.x == 0 && tid < N)
      for (int rl = 0; rl < nrows; ++rl) dbacc += dls[rl][tid];
  }
  if (colok) {
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int n = tr + 32 * j;
      if (n >= N) continue;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float v = acc[j][e] * keep_scale;
        const size_t at = (size_t)n * H + gcol * 8 + e;
        if (ws_dw != nullptr) ws_dw[(size_t)blockIdx.y * N * H + at] = v;
        else atomicAdd(dw + at, v);
      }
    }
  }
  if (blockIdx.x == 0 && tid < N) {
    if (ws_db != nullptr) ws_db[blockIdx.y * N + tid] = dbacc;
    else atomicAdd(db + tid, dbacc);
  }
}

int token_head_bwd_parts(int M) { return (M + TB_PART_ROWS - 1) / TB_PART_ROWS; }

void token_head_bwd(const float* dl, const void* x, const void* w, int M, int H, int N, Seed seed, unsigned stream,
                    float p_drop, void* dx, float* dw, float* db, float* ws, cudaStream_t st) {
  if (M <= 0) return;
  const unsigned th = tok_thresh(p_drop);
  const float sc = tok_scale(th);
  const int parts = token_head_bwd_parts(M);
  const dim3 grid((H + TB_COLS - 1) / TB_COLS, parts);
  float* ws_dw = ws;
  float* ws_db = ws != nullptr ? ws + (size_t)parts * N * H : nullptr;
  const auto* xb = (const __nv_bfloat16*)x;
  const auto* wb = (const __nv_bfloat16*)w;
  auto* dxb = (__nv_bfloat16*)dx;
  if (N <= 32)
    token_head_bwd_kernel<1><<<grid, TB_THREADS, 0, st>>>(dl, xb, wb, M, H, N, seed, stream, th, sc, dxb, dw, db, ws_dw, ws_db);
  else
    token_head_bwd_kernel<2><<<grid, TB_THREADS, 0, st>>>(dl, xb, wb, M, H, N, seed, stream, th, sc, dxb, dw, db, ws_dw, ws_db);
  if (ws != nullptr) {
    ordered_sum(ws_dw, parts, N * H, nullptr, 1, dw, st);
    ordered_sum(ws_db, parts, N, nullptr, 1, db, st);
  }
}

}  // namespace b200
