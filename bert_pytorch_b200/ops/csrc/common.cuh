// Shared device helpers for the sm_90a kernels: mbarrier / TMA PTX wrappers (wgmma: wgmma.cuh),
// Philox counter RNG for dropout, bf16 packing.
// Everything here is inline PTX written against the CUDA 12.9 ISA (no CUTLASS dependency).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <cstdio>
#include <cstdlib>

#include <cuda_fp8.h>

#include "seed.h"

#ifndef B200_WATCHDOG_NS
#define B200_WATCHDOG_NS 4000000000ull  // a barrier wait longer than 4 s traps instead of hanging the GPU
#endif

namespace b200 {

// ------------------------------------------------------------------------------------------------
// small utilities
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(0x4000u)   // suspend-time hint (ns): park the thread in hardware instead of
      : "memory");                                        // spinning through the issue slots
  return ok != 0;
}
// Blocking wait with a watchdog: a protocol bug must trap (visible error), never hang the box.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  uint64_t t0 = 0;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {          // try_wait itself suspends the thread for a HW-defined time
    if ((++spins & 255u) == 0) {                 // look at the clock only now and then (keeps issue slots free)
      const uint64_t now = globaltimer_ns();
      if (t0 == 0) t0 = now;
      if (now - t0 > B200_WATCHDOG_NS) {
        printf("[b200] mbarrier watchdog: block (%d,%d) thread %d parity %u\n", blockIdx.x, blockIdx.y,
               threadIdx.x, parity);
        __trap();
      }
    }
  }
}

// The same wait for threads that have wgmma groups in flight: no printf (a function call inside the wgmma pipeline
// makes ptxas serialise the MMAs), the watchdog only traps.
__device__ __forceinline__ void mbar_wait_mma(uint64_t* bar, uint32_t parity) {
  uint64_t t0 = 0;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 255u) == 0) {
      const uint64_t now = globaltimer_ns();
      if (t0 == 0) t0 = now;
      if (now - t0 > B200_WATCHDOG_NS) __trap();
    }
  }
}

// ------------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0,
                                            int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* m, int32_t c0, int32_t c1) {   // box -> L2 only
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(m)),
               "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0,
                                            int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0,
                                            int32_t c1, int32_t c2, int32_t c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ------------------------------------------------------------------------------------------------
// Philox4x32-7 counter RNG (7 rounds: the Crush-resistant variant of Random123; 10 buys nothing for dropout)
// Philox counter RNG (dropout masks are a pure function of (seed, stream, element index) so the
// backward pass and any recompute regenerate them instead of storing them).
// ------------------------------------------------------------------------------------------------
struct Philox {
  static constexpr uint32_t kA = 0xD2511F53u, kB = 0xCD9E8D57u, kW0 = 0x9E3779B9u, kW1 = 0xBB67AE85u;
  __host__ __device__ static inline uint4 round(uint4 c, uint2 k) {
#ifdef __CUDA_ARCH__
    uint32_t hi0 = __umulhi(kA, c.x), lo0 = kA * c.x;
    uint32_t hi1 = __umulhi(kB, c.z), lo1 = kB * c.z;
#else
    uint64_t p0 = (uint64_t)kA * c.x, p1 = (uint64_t)kB * c.z;
    uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
#endif
    return make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  // 128 random bits for counter (idx, stream) under key `seed`.
  __host__ __device__ static inline uint4 gen(uint64_t seed, uint64_t idx, uint32_t stream) {
    uint2 k = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    uint4 c = make_uint4((uint32_t)idx, (uint32_t)(idx >> 32), stream, 0x5EEDu);
#pragma unroll
    for (int i = 0; i < 7; ++i) {
      c = round(c, k);
      k.x += kW0;
      k.y += kW1;
    }
    return c;
  }
};
// Dropout decisions for 8 consecutive elements: element index `e8*8 + j` keeps iff its 16 random bits
// are >= threshold (threshold = round(p * 65536)).  Returns an 8-bit keep mask.
// Keep decisions of 8 consecutive elements: 16 random bits each, compared at the use site (keep[t] with a
// compile-time t is one bit-field extract + one integer compare feeding the select directly; assembling and
// re-testing a bit mask cost ~3 more instructions per element in kernels that are instruction bound).
struct Keep8 {
  uint32_t w[4];
  uint32_t th;
  __host__ __device__ static inline Keep8 all() {
    Keep8 k;
    k.w[0] = k.w[1] = k.w[2] = k.w[3] = 0xFFFFFFFFu;
    k.th = 0u;
    return k;
  }
  __host__ __device__ inline bool operator[](int t) const {
    const uint32_t x = w[t >> 1];
    return ((t & 1) ? (x >> 16) : (x & 0xFFFFu)) >= th;
  }
};
__host__ __device__ inline Keep8 dropout_keep8(uint64_t seed, uint32_t stream, uint64_t e8, uint32_t thresh16) {
  const uint4 r = Philox::gen(seed, e8, stream);
  Keep8 k;
  k.w[0] = r.x; k.w[1] = r.y; k.w[2] = r.z; k.w[3] = r.w;
  k.th = thresh16;
  return k;
}

// Lean evaluation of the same generator for instruction-bound kernels: round keys hoisted out of the element loops,
// one 64-bit product per multiply, 16-bit keep fields compared in place (same bits as dropout_keep8 / Keep8).
struct PhiloxKeys { uint32_t a[7], b[7]; };
__device__ __forceinline__ PhiloxKeys philox_keys(unsigned long long seed) {
  PhiloxKeys k;
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    k.a[i] = (uint32_t)seed + (uint32_t)i * Philox::kW0;
    k.b[i] = (uint32_t)(seed >> 32) + (uint32_t)i * Philox::kW1;
  }
  return k;
}
// same value as Philox::gen(seed, idx, stream), round keys hoisted, 64-bit products (one IMAD.WIDE each)
__device__ __forceinline__ uint4 philox7(const PhiloxKeys& k, uint64_t idx, uint32_t stream) {
  uint32_t x = (uint32_t)idx, y = (uint32_t)(idx >> 32), z = stream, w = 0x5EEDu;
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    const uint64_t p0 = (uint64_t)Philox::kA * x, p1 = (uint64_t)Philox::kB * z;
    const uint32_t nx = (uint32_t)(p1 >> 32) ^ y ^ k.a[i];
    const uint32_t nz = (uint32_t)(p0 >> 32) ^ w ^ k.b[i];
    y = (uint32_t)p1;
    w = (uint32_t)p0;
    x = nx;
    z = nz;
  }
  return make_uint4(x, y, z, w);
}
// element t (0..7) of a dropout group is kept iff its 16-bit field (word t/2, low half for even t) >= thresh16;
// `T` = thresh16 << 16.  High halves compare in place, low halves after a 16-bit shift.
__device__ __forceinline__ bool keep_bit(const uint4& r, int t, uint32_t T) {
  const uint32_t wds[4] = {r.x, r.y, r.z, r.w};
  const uint32_t w = wds[t >> 1];
  return (t & 1) ? (w >= T) : ((w << 16) >= T);
}
// ------------------------------------------------------------------------------------------------
// bf16 helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
// erf-GELU through the complementary error function of Abramowitz & Stegun 7.1.26:
//   erfc(z) = (a1 t + ... + a5 t^5) exp(-z^2),  t = 1/(1 + p z),  z >= 0,  |error| <= 1.5e-7
// so  Phi(x) = 0.5 erfc(|x|/sqrt2)  for x < 0  and  1 - that  for x >= 0  (no cancellation in the negative tail),
// gelu(x) = x Phi(x)  and  gelu'(x) = Phi(x) + x phi(x)  with  phi(x) = exp(-x^2/2)/sqrt(2 pi)  sharing the SAME
// exponential.  One rcp.approx + one ex2.approx + ~10 FMA-class instructions (erff() needs ~3x as many; the
// GELU kernels and epilogues are instruction bound).
struct GeluParts { float Phi, e; };   // e = exp(-x^2/2)
__device__ __forceinline__ GeluParts gelu_parts(float x) {
  // 11 instructions: the 0.5 of 0.5 erfc and the 1/sqrt2 of z are folded into the constants
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(fabsf(x), 0.3275911f * 0.70710678118654752f, 1.0f)));
  float poly = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);
  poly = fmaf(poly, t, 0.5f * 1.421413741f);
  poly = fmaf(poly, t, 0.5f * -0.284496736f);
  poly = fmaf(poly, t, 0.5f * 0.254829592f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * x * (-0.5f * 1.4426950408889634f)));
  const float h = poly * t * e;                        // 0.5 erfc(|x| / sqrt2)
  GeluParts r;
  r.Phi = x < 0.f ? h : 1.0f - h;
  r.e = e;
  return r;
}
__device__ __forceinline__ float erf_fast(float x) { return 2.0f * gelu_parts(x * 1.4142135623730951f).Phi - 1.0f; }
__device__ __forceinline__ float gelu_erf(float x) { return x * gelu_parts(x).Phi; }
__device__ __forceinline__ float dgelu_erf(float x) {
  const GeluParts g = gelu_parts(x);
  return fmaf(x * 0.3989422804014327f, g.e, g.Phi);
}

// ------------------------------------------------------------------------------------------------
// fp32 pairs: two independent lanes of fp32 math behind one name (sm_90 has no packed fp32 instructions; each
// operation is two scalar FFMA / FMUL / FADD with the same rounding as the scalar code).
// ------------------------------------------------------------------------------------------------
struct f32x2 { float x, y; };
__device__ __forceinline__ f32x2 f2_pack(float lo, float hi) { return f32x2{lo, hi}; }
__device__ __forceinline__ f32x2 f2_pack_u(uint32_t lo, uint32_t hi) { return f32x2{__uint_as_float(lo), __uint_as_float(hi)}; }
__device__ __forceinline__ float2 f2_unpack(f32x2 v) { return make_float2(v.x, v.y); }
__device__ __forceinline__ f32x2 f2_splat(float c) { return f32x2{c, c}; }
__device__ __forceinline__ f32x2 f2_fma(f32x2 a, f32x2 b, f32x2 c) { return f32x2{fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)}; }
__device__ __forceinline__ f32x2 f2_mul(f32x2 a, f32x2 b) { return f32x2{a.x * b.x, a.y * b.y}; }
__device__ __forceinline__ f32x2 f2_add(f32x2 a, f32x2 b) { return f32x2{a.x + b.x, a.y + b.y}; }
__device__ __forceinline__ f32x2 f2_from_bf16x2(uint32_t w) {       // {lo, hi} bf16 -> two fp32 (exact)
  return f2_pack_u(w << 16, w & 0xffff0000u);
}
__device__ __forceinline__ uint32_t f2_to_bf16x2(f32x2 v) { return pack_bf16(v.x, v.y); }
// gelu(x) and gelu'(x) of two values: the same arithmetic as gelu_parts()
struct GeluDg2 { f32x2 g, dg; };
__device__ __forceinline__ GeluDg2 gelu_dg2(f32x2 x) {
  const float2 xf = f2_unpack(x);
  float t0, t1, e0, e1;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t0) : "f"(fmaf(fabsf(xf.x), 0.3275911f * 0.70710678118654752f, 1.0f)));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t1) : "f"(fmaf(fabsf(xf.y), 0.3275911f * 0.70710678118654752f, 1.0f)));
  const f32x2 t = f2_pack(t0, t1);
  f32x2 poly = f2_fma(f2_splat(0.5f * 1.061405429f), t, f2_splat(0.5f * -1.453152027f));
  poly = f2_fma(poly, t, f2_splat(0.5f * 1.421413741f));
  poly = f2_fma(poly, t, f2_splat(0.5f * -0.284496736f));
  poly = f2_fma(poly, t, f2_splat(0.5f * 0.254829592f));
  const float2 s = f2_unpack(f2_mul(f2_mul(x, f2_splat(-0.5f * 1.4426950408889634f)), x));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(s.x));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(s.y));
  const f32x2 e = f2_pack(e0, e1);
  const f32x2 h = f2_mul(f2_mul(poly, t), e);                          // 0.5 erfc(|x| / sqrt2)
  const float2 hf = f2_unpack(h), omh = f2_unpack(f2_fma(h, f2_splat(-1.0f), f2_splat(1.0f)));
  const f32x2 Phi = f2_pack(xf.x < 0.f ? hf.x : omh.x, xf.y < 0.f ? hf.y : omh.y);
  GeluDg2 r;
  r.g = f2_mul(x, Phi);
  r.dg = f2_fma(f2_mul(x, f2_splat(0.3989422804014327f)), e, Phi);
  return r;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------------------------------
// fp8 side outputs (see Fp8Out in seed.h)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t fp8_cvt4(float a, float b, float c, float d, bool e5m2) {
  uint32_t lo, hi;
  if (e5m2) {
    lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E5M2);
    hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E5M2);
  } else {
    lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
    hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
  }
  return lo | (hi << 16);
}
// 8 consecutive elements starting at element offset `off` (multiple of 8)
__device__ __forceinline__ void fp8_emit8(const Fp8Out& f, size_t off, const float (&v)[8], float scale, float& amax) {
#pragma unroll
  for (int t = 0; t < 8; ++t) amax = fmaxf(amax, fabsf(v[t]));
  const uint2 o = make_uint2(fp8_cvt4(v[0] * scale, v[1] * scale, v[2] * scale, v[3] * scale, f.e5m2 != 0),
                             fp8_cvt4(v[4] * scale, v[5] * scale, v[6] * scale, v[7] * scale, f.e5m2 != 0));
  *reinterpret_cast<uint2*>(f.q + off) = o;
}
__device__ __forceinline__ void fp8_amax_commit(const Fp8Out& f, float amax) {
  amax = warp_max(amax);
  if ((threadIdx.x & 31) == 0 && amax > 0.f)
    atomicMax(reinterpret_cast<int*>(f.meta), __float_as_int(isfinite(amax) ? amax : 3.0e38f));
}

}  // namespace b200

// host side: error checking + tensor-map encode through the runtime's driver entry point (no -lcuda)
#define B200_CUDA_CHECK(x)                                                                      \
  do {                                                                                          \
    cudaError_t e_ = (x);                                                                       \
    if (e_ != cudaSuccess) {                                                                    \
      fprintf(stderr, "[b200] CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      abort();                                                                                  \
    }                                                                                           \
  } while (0)

namespace b200 {
inline int num_sms() {                   // SMs of the current device (132 on an H100 SXM)
  static int n = 0;
  if (n == 0) {
    int dev;
    B200_CUDA_CHECK(cudaGetDevice(&dev));
    B200_CUDA_CHECK(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  }
  return n;
}
}  // namespace b200
