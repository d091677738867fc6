// Per-tensor scaled fp8 (e4m3 / e5m2) operand preparation for the wgmma fp8 GEMM path.
//
// Recipe (delayed scaling; the reference has no fp8 path -- BASELINE.json's RoBERTa fp8 config is an addition of this project):
//   every GEMM operand site owns a 4-float record  meta = {amax, scale, inv_scale, _}  on the device
//   quantise:     q = sat_fp8(x * scale)      and   amax = max(amax, |x|)      (one pass over x, 3 B/element)
//   GEMM:         D = (qa . qb) * inv_scale_a * inv_scale_b                     (read by the epilogue from meta)
//   end of step:  scale = 2^e with e the largest integer such that amax * margin * 2^e <= fmax, clamped to
//                 [-126, 126] (power of two, so re-scaling is exact; scale and inv_scale = 1 / scale are both finite,
//                 normal floats for any amax), then amax = 0.  amax = 0 or non-finite keeps the old scale.
// Nothing syncs with the host; the first step after enabling fp8 calibrates with fp8_amax + fp8_update.
#include <cuda_fp8.h>

#include "common.cuh"
#include "kernels.h"

namespace b200 {

__device__ __forceinline__ void atomic_max_nonneg(float* addr, float v) {
  // non-negative floats order like their bit patterns
  atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
}

template <bool E5M2>
__device__ __forceinline__ uint32_t cvt4(float a, float b, float c, float d) {
  constexpr __nv_fp8_interpretation_t K = E5M2 ? __NV_E5M2 : __NV_E4M3;
  const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, K);
  const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, K);
  return lo | (hi << 16);
}

// x: bf16 [n] (n % 16 == 0), q: fp8 bytes [n].  16 elements per thread and iteration: 32 B in, 16 B out.
template <bool E5M2>
__global__ void __launch_bounds__(256) fp8_quantize_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q,
                                                           long long n16, float* __restrict__ meta) {
  const float scale = meta[1];
  float amax = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (long long)gridDim.x * blockDim.x) {
    const uint4 u0 = __ldg(reinterpret_cast<const uint4*>(x) + 2 * i);
    const uint4 u1 = __ldg(reinterpret_cast<const uint4*>(x) + 2 * i + 1);
    const uint32_t w[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
    uint32_t o[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 a = unpack_bf16(w[2 * t]), b = unpack_bf16(w[2 * t + 1]);
      amax = fmaxf(amax, fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(b.x), fabsf(b.y))));
      o[t] = cvt4<E5M2>(a.x * scale, a.y * scale, b.x * scale, b.y * scale);
    }
    reinterpret_cast<uint4*>(q)[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
  amax = warp_max(amax);
  if ((threadIdx.x & 31) == 0 && amax > 0.f) {
    if (!isfinite(amax)) amax = 3.0e38f;            // keep the record finite; the GradScaler handles the overflow
    atomic_max_nonneg(meta, amax);
  }
}

__global__ void __launch_bounds__(256) fp8_amax_kernel(const __nv_bfloat16* __restrict__ x, long long n8,
                                                       float* __restrict__ meta) {
  float amax = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(x) + i);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 a = unpack_bf16(w[t]);
      amax = fmaxf(amax, fmaxf(fabsf(a.x), fabsf(a.y)));
    }
  }
  amax = warp_max(amax);
  if ((threadIdx.x & 31) == 0 && amax > 0.f) atomic_max_nonneg(meta, isfinite(amax) ? amax : 3.0e38f);
}

// one thread per record; is_e5m2[i] != 0 -> record i quantises to e5m2 (max 57344) else e4m3 (448)
__global__ void fp8_update_kernel(float* __restrict__ meta, int nrec, const int* __restrict__ is_e5m2, float margin_pow2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nrec) return;
  float* m = meta + 4 * i;
  const float amax = m[0];
  if (amax > 0.f && isfinite(amax)) {
    // largest e with amax * margin * 2^e <= fmax, from exact mantissas and exponents: fmax / (amax * margin) in fp32
    // overflows for a tiny amax (< 1.3e-36 for e4m3) and amax * margin for one near FLT_MAX
    int e_x, e_f;
    const double m_x = frexp((double)amax * (double)margin_pow2, &e_x);   // exact: a 48-bit product
    const double m_f = frexp(is_e5m2[i] ? 57344.0 : 448.0, &e_f);
    int e = e_f - e_x - (m_x > m_f ? 1 : 0);
    e = min(126, max(-126, e));                      // scale and inv_scale both finite, normal powers of two
    m[1] = ldexpf(1.f, e);
    m[2] = ldexpf(1.f, -e);
  }
  m[0] = 0.f;
}

void fp8_quantize(const void* x, void* q, long long n, float* meta, bool e5m2, cudaStream_t st) {
  const long long n16 = n / 16;
  if (n16 == 0) return;
  const int grid = (int)std::min<long long>((n16 + 255) / 256, num_sms() * 8);
  if (e5m2) fp8_quantize_kernel<true><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, (uint8_t*)q, n16, meta);
  else fp8_quantize_kernel<false><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, (uint8_t*)q, n16, meta);
}

void fp8_amax(const void* x, long long n, float* meta, cudaStream_t st) {
  const long long n8 = n / 8;
  if (n8 == 0) return;
  const int grid = (int)std::min<long long>((n8 + 255) / 256, num_sms() * 8);
  fp8_amax_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, n8, meta);
}

void fp8_update(float* meta, int nrec, const int* is_e5m2, float margin_pow2, cudaStream_t st) {
  if (nrec <= 0) return;
  fp8_update_kernel<<<(nrec + 127) / 128, 128, 0, st>>>(meta, nrec, is_e5m2, margin_pow2);
}

}  // namespace b200
