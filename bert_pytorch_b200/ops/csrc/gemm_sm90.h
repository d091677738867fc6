// Host API of the wgmma GEMM (see gemm_sm90.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

enum GemmLayout : int {
  GEMM_NT = 0,  // D[M,N] = A[M,K] * B[N,K]^T        A stored [M][lda], B stored [N][ldb]   (forward)
  GEMM_NN = 1,  // D[M,N] = A[M,K] * B[K,N]          A stored [M][lda], B stored [K][ldb]   (dgrad)
  GEMM_TN = 2,  // D[M,N] = A[K,M]^T * B[K,N]        A stored [K][lda], B stored [K][ldb]   (wgrad)
};

enum GemmEpilogue : int {
  EPI_NONE = 0,           // out(bf16) = alpha*acc
  EPI_BIAS = 1,           // + bias[n]
  EPI_BIAS_GELU = 2,      // aux_out = acc + bias ; out = gelu(aux_out)
  EPI_BIAS_DROP_RES = 3,  // out = res + dropout(acc + bias)
  EPI_ADD = 4,            // out = acc + res          (res may be null)
  EPI_DGELU = 5,          // out = acc * gelu'(res)
  EPI_ACCUM_F32 = 6,      // out(fp32) += alpha*acc   (atomic when split-K)
  EPI_BIAS_TANH = 7,      // out = tanh(acc + bias)
  EPI_F32 = 8,            // out(fp32) = alpha*acc
  EPI_BIAS_GELU_DG = 9,   // x = acc + bias ; out = gelu(x) ; aux_out = gelu'(x)   (FFN-1: the activation and its
                          // derivative leave the GEMM together, the backward pass only multiplies -- K16)
  EPI_MUL = 10,           // out = acc * res          (FFN-2 dgrad: res = gelu'(x) saved by EPI_BIAS_GELU_DG)
};

struct GemmCall {
  int layout = GEMM_NT;
  int epi = EPI_NONE;
  int block_n = 256;   // 128: 128 x 128 tiles, anything else: 128 x 256 (when N > 128)
  int M = 0, N = 0, K = 0;
  const void* A = nullptr; int lda = 0;
  const void* B = nullptr; int ldb = 0;
  void* out = nullptr; int ldo = 0;
  void* aux_out = nullptr;
  const void* bias = nullptr;
  const void* res = nullptr; int ldr = 0;
  // optional (EPI_BIAS_DROP_RES): keep decisions of the dropout, one byte per 8 output columns
  // ([M][N / 8], bit t = column 8 j + t kept) -- the LayerNorm backward reads them back instead of re-running Philox
  unsigned char* mask_out = nullptr;
  // the same bits as INPUT (written beforehand by dropout_mask()): the epilogue applies them instead of running Philox
  const unsigned char* mask_in = nullptr;
  float* colsum = nullptr;   // optional (bf16 epilogues): colsum[n] += sum_m out[m][n]  (bias gradients, fp32 atomics)
  int k_splits = 1;      // EPI_ACCUM_F32 only; < 0: as many K ranges as fill the SMs
  unsigned long long seed = 0; unsigned int stream = 0; float p_drop = 0.f;
  const unsigned long long* seed_step = nullptr;   // device step counter mixed into the seed (CUDA-graph replays)
  float alpha = 1.f;
  // fp8 operands: A/B are e4m3 (default) or e5m2 bytes, lda/ldb in elements (= bytes);
  // scale_a/scale_b point at the device-resident per-tensor dequantisation factors (x = q * scale)
  bool fp8 = false, a_e5m2 = false, b_e5m2 = false;
  const float* scale_a = nullptr;
  const float* scale_b = nullptr;
  // EPI_ACCUM_F32 into a gradient arena shared over NVLink (see GemmArgs::peer_*)
  int peer_world = 0, peer_rank = 0, peer_push = 0;
  long long peer_off = 0, peer_per = 0;
  float* peer_base[16] = {};
};

void gemm_bf16(const GemmCall& c, cudaStream_t st);

CUtensorMap make_tmap_2d_bf16(const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                              uint32_t box_outer);

}  // namespace b200
