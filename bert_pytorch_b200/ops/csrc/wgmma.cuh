// wgmma (sm_90a warpgroup MMA) wrappers: one function template per instruction shape, fp32 accumulators in
// registers.  Accumulator fragment of a 64 x N tile: thread t of the warpgroup (warp w = t / 32, lane l = t % 32) holds,
// for every 8-column group j, d[4 j + {0, 1}] = row 16 w + l / 4, columns 8 j + 2 (l % 4) + {0, 1} and
// d[4 j + {2, 3}] = the same columns of row 16 w + l / 4 + 8.
#pragma once
#include <stdint.h>

namespace b200 {

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// 64-bit shared-memory matrix descriptor, 128-byte swizzle:
//   bits [0,14) start address >> 4   [16,30) leading byte offset >> 4   [32,46) stride byte offset >> 4   [62,64) 1 = 128B swizzle
// K-major tile (rows of 128 B): LBO unused, SBO = 1024 (8 rows).  MN-major tile ([k][64 mn] chunks of 128-byte rows):
// LBO = byte distance between 64-wide MN chunks, SBO = 1024 (8 k-rows).
__host__ __device__ constexpr uint64_t wgmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32) | ((uint64_t)1 << 62);
}

// wgmma.wait_group orders the asynchronous MMAs, not the compiler: an accumulator read may be scheduled above the
// wait (and a write below the next MMA) unless the registers themselves pass through a volatile statement.  Call on
// every accumulator array right after the wait that completes it and right before the first MMA that reuses it.
template <int N>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Operand lists of the MMA statements: WG_ACC_n(d) = the n accumulator registers as "+f" operands (%0 .. %n-1),
// WG_REGS_n = the matching register list of the instruction text; the inputs follow as %n, %n+1, ...
#define WG_ACC8(d, i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define WG_ACC_32(d) WG_ACC8(d, 0), WG_ACC8(d, 8), WG_ACC8(d, 16), WG_ACC8(d, 24)
#define WG_ACC_64(d) WG_ACC_32(d), WG_ACC8(d, 32), WG_ACC8(d, 40), WG_ACC8(d, 48), WG_ACC8(d, 56)
#define WG_ACC_128(d) WG_ACC_64(d), WG_ACC8(d, 64), WG_ACC8(d, 72), WG_ACC8(d, 80), WG_ACC8(d, 88), WG_ACC8(d, 96), WG_ACC8(d, 104), WG_ACC8(d, 112), WG_ACC8(d, 120)
#define WG_REGS_32 \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, " \
  "%23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define WG_REGS_64 \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, " \
  "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, " \
  "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define WG_REGS_128 \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, " \
  "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, " \
  "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, " \
  "%65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, " \
  "%86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, " \
  "%106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, " \
  "%124, %125, %126, %127}"
#define WG_PRED(i) "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #i ", 0;\n\t"

// D (+)= A B with both operands in shared memory (descriptors), bf16: TA / TB = 1 reads that operand MN-major.
// `acc` = 0 overwrites the accumulator (it need not be initialised).
template <int N, int TA, int TB> struct WgmmaBf16SS;
// A from registers (the accumulator fragment of a previous MMA, packed to bf16), B from shared memory
template <int N, int TB> struct WgmmaBf16RS;
// fp8 operands (K-major only): AE5 / BE5 = 1 selects e5m2 for that operand, else e4m3
template <int N, int AE5, int BE5> struct WgmmaFp8SS;

#define WG_DEFINE_BF16_SS(N, n, i0, i1, i2, i3, i4)                                                                    \
  template <int TA, int TB> struct WgmmaBf16SS<N, TA, TB> {                                                            \
    __device__ __forceinline__ static void mma(float (&d)[n], uint64_t da, uint64_t db, int acc) {                     \
      asm volatile(WG_PRED(i2) "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 " WG_REGS_##n                 \
                   ", %" #i0 ", %" #i1 ", p, 1, 1, %" #i3 ", %" #i4 ";\n\t}"                                            \
                   : WG_ACC_##n(d) : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));                                    \
    }                                                                                                                  \
  };
WG_DEFINE_BF16_SS(64, 32, 32, 33, 34, 35, 36)
WG_DEFINE_BF16_SS(128, 64, 64, 65, 66, 67, 68)
WG_DEFINE_BF16_SS(256, 128, 128, 129, 130, 131, 132)

template <int TB> struct WgmmaBf16RS<64, TB> {
  __device__ __forceinline__ static void mma(float (&d)[32], const uint32_t (&a)[4], uint64_t db, int acc) {
    asm volatile(WG_PRED(37) "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " WG_REGS_32
                 ", {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}"
                 : WG_ACC_32(d) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc), "n"(TB));
  }
};

#define WG_DEFINE_FP8_SS(N, n, i0, i1, i2, AE5, BE5, TA, TB)                                                           \
  template <> struct WgmmaFp8SS<N, AE5, BE5> {                                                                         \
    __device__ __forceinline__ static void mma(float (&d)[n], uint64_t da, uint64_t db, int acc) {                     \
      asm volatile(WG_PRED(i2) "wgmma.mma_async.sync.aligned.m64n" #N "k32.f32." TA "." TB " " WG_REGS_##n             \
                   ", %" #i0 ", %" #i1 ", p, 1, 1;\n\t}"                                                                \
                   : WG_ACC_##n(d) : "l"(da), "l"(db), "r"(acc));                                                      \
    }                                                                                                                  \
  };
#define WG_DEFINE_FP8_ALL(N, n, i0, i1, i2)                                                                            \
  WG_DEFINE_FP8_SS(N, n, i0, i1, i2, 0, 0, "e4m3", "e4m3") WG_DEFINE_FP8_SS(N, n, i0, i1, i2, 1, 0, "e5m2", "e4m3")    \
  WG_DEFINE_FP8_SS(N, n, i0, i1, i2, 0, 1, "e4m3", "e5m2") WG_DEFINE_FP8_SS(N, n, i0, i1, i2, 1, 1, "e5m2", "e5m2")
WG_DEFINE_FP8_ALL(128, 64, 64, 65, 66)
WG_DEFINE_FP8_ALL(256, 128, 128, 129, 130)

// 4 x 4 transpose inside a quad (lanes 4 q .. 4 q + 3): lane c holds a[k] = M[c][k] and receives M[k][c].
// Used to regroup accumulator fragments (lane c owns column pair c of every 8-column group) into runs of 8
// consecutive columns per lane, and back.
__device__ __forceinline__ void quad_transpose(uint32_t (&a)[4]) {
  const int c = threadIdx.x & 3;
  {
    const bool hi = c & 1;
    const uint32_t s0 = hi ? a[0] : a[1], s1 = hi ? a[2] : a[3];
    const uint32_t r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
    if (hi) { a[0] = r0; a[2] = r1; } else { a[1] = r0; a[3] = r1; }
  }
  {
    const bool hi = c & 2;
    const uint32_t s0 = hi ? a[0] : a[2], s1 = hi ? a[1] : a[3];
    const uint32_t r0 = __shfl_xor_sync(0xffffffffu, s0, 2), r1 = __shfl_xor_sync(0xffffffffu, s1, 2);
    if (hi) { a[0] = r0; a[1] = r1; } else { a[2] = r0; a[3] = r1; }
  }
}

}  // namespace b200
