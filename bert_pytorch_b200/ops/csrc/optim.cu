// Multi-tensor optimizer kernels (replacing apex amp_C / FusedLAMB / FusedAdam: SURVEY.md N1-N3, O2-O8).
//
// All kernels are driven by a *chunk table*: chunk c covers elements [chunk_start[c], chunk_start[c] +
// chunk_len[c]) of tensor chunk_tensor[c]; a chunk never straddles tensors, so per-tensor reductions are a
// block reduce + one atomic per block.  For the parameter arena the "tensors" are slots of one flat
// buffer (pointer table = base + offset), for the generic multi_tensor_* entry points they are arbitrary
// fp32 / bf16 / fp16 tensors.
//
// LAMB over the arena is three launches:
//   1. sumsq:   sum (g * inv_scale)^2  + inf/nan flag                       -> global grad norm
//   2. stage 1: clip, moments, update u (written over g), per-tensor ||p||^2, ||u||^2
//   3. stage 2: p -= lr * trust_ratio * u ; refresh bf16 shadow ; zero g
// A set found_inf flag turns stages 1-2 into "zero the gradients only" (GradScaler skip semantics,
// decided on the device: no host synchronisation anywhere).
#include "common.cuh"
#include "kernels.h"

namespace b200 {

constexpr int OPT_THREADS = 512;

__device__ __forceinline__ float block_sum(float v, float* sm) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) sm[warp] = v;
  __syncthreads();
  float r = 0.f;
  if (warp == 0) {
    r = lane < (blockDim.x >> 5) ? sm[lane] : 0.f;
    r = warp_sum(r);
  }
  __syncthreads();
  return r;  // valid in warp 0
}

template <typename T>
__device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <typename T>
__device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16(v); }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half(v); }

// ------------------------------------------------------------------------------------------------
// generic multi-tensor l2norm / scale over a pointer table
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(OPT_THREADS)
mt_l2norm_kernel(const long long* __restrict__ ptrs, const int* __restrict__ chunk_tensor,
                 const long long* __restrict__ chunk_start, const int* __restrict__ chunk_len,
                 float* __restrict__ per_tensor_sq, float* __restrict__ total_sq) {
  __shared__ float sm[32];
  const int c = blockIdx.x;
  const int t = chunk_tensor[c];
  const T* p = reinterpret_cast<const T*>(ptrs[t]) + chunk_start[c];
  const int n = chunk_len[c];
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float v = to_f<T>(p[i]);
    s += v * v;
  }
  s = block_sum(s, sm);
  if (threadIdx.x == 0) {
    if (per_tensor_sq) atomicAdd(per_tensor_sq + t, s);
    atomicAdd(total_sq, s);
  }
}

// deterministic mode: chunk c stores its sum of squares to chunk_sq[c]; ordered_sum finishes per tensor and in total
template <typename T>
__global__ void __launch_bounds__(OPT_THREADS)
mt_l2norm_part_kernel(const long long* __restrict__ ptrs, const int* __restrict__ chunk_tensor,
                      const long long* __restrict__ chunk_start, const int* __restrict__ chunk_len,
                      float* __restrict__ chunk_sq) {
  __shared__ float sm[32];
  const int c = blockIdx.x;
  const T* p = reinterpret_cast<const T*>(ptrs[chunk_tensor[c]]) + chunk_start[c];
  const int n = chunk_len[c];
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float v = to_f<T>(p[i]);
    s += v * v;
  }
  s = block_sum(s, sm);
  if (threadIdx.x == 0) chunk_sq[c] = s;
}

template <typename TI, typename TO>
__global__ void __launch_bounds__(OPT_THREADS)
mt_scale_kernel(const long long* __restrict__ in_ptrs, const long long* __restrict__ out_ptrs,
                const int* __restrict__ chunk_tensor, const long long* __restrict__ chunk_start,
                const int* __restrict__ chunk_len, const float* __restrict__ scale_dev, float scale_host,
                int* __restrict__ overflow) {
  const int c = blockIdx.x;
  const int t = chunk_tensor[c];
  const TI* in = reinterpret_cast<const TI*>(in_ptrs[t]) + chunk_start[c];
  TO* out = reinterpret_cast<TO*>(out_ptrs[t]) + chunk_start[c];
  const float sc = scale_dev ? *scale_dev : scale_host;
  const int n = chunk_len[c];
  bool bad = false;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float v = to_f<TI>(in[i]) * sc;
    bad |= !isfinite(v);
    out[i] = from_f<TO>(v);
  }
  if (bad) *overflow = 1;
}

// ------------------------------------------------------------------------------------------------
// arena kernels
// ------------------------------------------------------------------------------------------------
// stats[0] = sum (g*inv_scale)^2, found_inf set to 1 on inf/nan.  Grid-stride over the whole arena.
// PART (deterministic mode): block b stores its sum to stats[b] for ordered_sum instead of adding it to stats[0]
template <bool PART>
__device__ __forceinline__ void flat_sumsq_body(const float* __restrict__ g, long long n, const float* __restrict__ inv_scale,
                                                float* __restrict__ stats, float* __restrict__ found_inf) {
  __shared__ float sm[32];
  const float is = inv_scale ? *inv_scale : 1.f;
  float s = 0.f;
  bool bad = false;
  const long long n4 = n >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v = g4[i];
    v.x *= is; v.y *= is; v.z *= is; v.w *= is;
    const float q = v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    bad |= !isfinite(q);
    s += q;
  }
  s = block_sum(s, sm);
  if constexpr (PART) { if (threadIdx.x == 0) stats[blockIdx.x] = s; }
  else if (threadIdx.x == 0) atomicAdd(stats, s);
  if (bad && found_inf) *found_inf = 1.f;
}

__global__ void __launch_bounds__(OPT_THREADS)
flat_sumsq_kernel(const float* __restrict__ g, long long n, const float* __restrict__ inv_scale,
                  float* __restrict__ stats, float* __restrict__ found_inf) {
  flat_sumsq_body<false>(g, n, inv_scale, stats, found_inf);
}

__global__ void __launch_bounds__(OPT_THREADS)
flat_sumsq_part_kernel(const float* __restrict__ g, long long n, const float* __restrict__ inv_scale,
                       float* __restrict__ block_sq, float* __restrict__ found_inf) {
  flat_sumsq_body<true>(g, n, inv_scale, block_sq, found_inf);
}

// grads *= inv_scale in place + inf flag (GradScaler.unscale_ for the K-FAC path)
__global__ void __launch_bounds__(OPT_THREADS)
flat_unscale_kernel(float* __restrict__ g, long long n, const float* __restrict__ inv_scale,
                    float* __restrict__ found_inf) {
  const float is = *inv_scale;
  bool bad = false;
  const long long n4 = n >> 2;
  float4* g4 = reinterpret_cast<float4*>(g);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v = g4[i];
    v.x *= is; v.y *= is; v.z *= is; v.w *= is;
    // per element: the sum of four finite values can overflow (3e38 + 3e38) and would flag a clean step
    bad |= !(isfinite(v.x) && isfinite(v.y) && isfinite(v.z) && isfinite(v.w));
    g4[i] = v;
  }
  if (bad) *found_inf = 1.f;
}

struct LambHyper {
  float lr, beta1, beta2, beta3, eps, weight_decay, bc1, bc2, max_grad_norm;
  int adam_w_mode, use_nvlamb;
};

// stage 1 over chunks of the arena; u overwrites g; norms[t] = {sum p^2, sum u^2}
// PART (deterministic mode): chunk c stores {sum p^2, sum u^2} to norms[2 c], norms[2 c + 1] for ordered_sum
template <bool PART>
__device__ __forceinline__ void lamb_stage1_body(float* __restrict__ g, const float* __restrict__ p, float* __restrict__ m,
                                                 float* __restrict__ v, const int* __restrict__ chunk_tensor,
                                                 const long long* __restrict__ chunk_start,
                                                 const int* __restrict__ chunk_len, const int* __restrict__ decay_flag,
                                                 const float* __restrict__ stats, const float* __restrict__ inv_scale,
                                                 const float* __restrict__ found_inf, float* __restrict__ norms,
                                                 const LambHyper& h) {
  __shared__ float sm[32];
  const int c = blockIdx.x;
  if (found_inf && *found_inf != 0.f) {
    if constexpr (PART) if (threadIdx.x == 0) norms[2 * c] = norms[2 * c + 1] = 0.f;
    return;
  }
  const int t = chunk_tensor[c];
  const long long off = chunk_start[c];
  const int n = chunk_len[c];
  const float is = inv_scale ? *inv_scale : 1.f;
  const float gnorm = sqrtf(stats[0]);
  const float clip = (h.max_grad_norm > 0.f && gnorm > h.max_grad_norm) ? gnorm / h.max_grad_norm : 1.f;
  const float gs = is / clip;
  const float wd = decay_flag[t] ? h.weight_decay : 0.f;
  float sp = 0.f, su = 0.f;
  const int n4 = n >> 2;   // chunk starts/lengths are multiples of 4 except a tensor's tail
  float4* g4 = reinterpret_cast<float4*>(g + off);
  const float4* p4 = reinterpret_cast<const float4*>(p + off);
  float4* m4 = reinterpret_cast<float4*>(m + off);
  float4* v4 = reinterpret_cast<float4*>(v + off);
  const bool aligned = (off & 3) == 0;
  auto upd = [&](float gg, float pp, float& mm, float& vv) -> float {
    gg *= gs;
    if (!h.adam_w_mode) gg += wd * pp;
    mm = h.beta1 * mm + h.beta3 * gg;
    vv = h.beta2 * vv + (1.f - h.beta2) * gg * gg;
    float u = (mm / h.bc1) / (sqrtf(vv / h.bc2) + h.eps);
    if (h.adam_w_mode) u += wd * pp;
    sp += pp * pp;
    su += u * u;
    return u;
  };
  if (aligned) {
    for (int i = threadIdx.x; i < n4; i += blockDim.x) {
      float4 gg = g4[i], pp = p4[i], mm = m4[i], vv = v4[i];
      gg.x = upd(gg.x, pp.x, mm.x, vv.x);
      gg.y = upd(gg.y, pp.y, mm.y, vv.y);
      gg.z = upd(gg.z, pp.z, mm.z, vv.z);
      gg.w = upd(gg.w, pp.w, mm.w, vv.w);
      g4[i] = gg; m4[i] = mm; v4[i] = vv;
    }
    for (int i = (n4 << 2) + threadIdx.x; i < n; i += blockDim.x) {
      float mm = m[off + i], vv = v[off + i];
      g[off + i] = upd(g[off + i], p[off + i], mm, vv);
      m[off + i] = mm; v[off + i] = vv;
    }
  } else {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      float mm = m[off + i], vv = v[off + i];
      g[off + i] = upd(g[off + i], p[off + i], mm, vv);
      m[off + i] = mm; v[off + i] = vv;
    }
  }
  sp = block_sum(sp, sm);
  su = block_sum(su, sm);
  if constexpr (PART) {
    if (threadIdx.x == 0) { norms[2 * c] = sp; norms[2 * c + 1] = su; }
  } else if (threadIdx.x == 0) {
    atomicAdd(norms + 2 * t, sp);
    atomicAdd(norms + 2 * t + 1, su);
  }
}

__global__ void __launch_bounds__(OPT_THREADS)
lamb_stage1_kernel(float* __restrict__ g, const float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                   const int* __restrict__ chunk_tensor, const long long* __restrict__ chunk_start,
                   const int* __restrict__ chunk_len, const int* __restrict__ decay_flag,
                   const float* __restrict__ stats, const float* __restrict__ inv_scale,
                   const float* __restrict__ found_inf, float* __restrict__ norms, LambHyper h) {
  lamb_stage1_body<false>(g, p, m, v, chunk_tensor, chunk_start, chunk_len, decay_flag, stats, inv_scale, found_inf,
                          norms, h);
}

__global__ void __launch_bounds__(OPT_THREADS)
lamb_stage1_part_kernel(float* __restrict__ g, const float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                        const int* __restrict__ chunk_tensor, const long long* __restrict__ chunk_start,
                        const int* __restrict__ chunk_len, const int* __restrict__ decay_flag,
                        const float* __restrict__ stats, const float* __restrict__ inv_scale,
                        const float* __restrict__ found_inf, float* __restrict__ chunk_norms, LambHyper h) {
  lamb_stage1_body<true>(g, p, m, v, chunk_tensor, chunk_start, chunk_len, decay_flag, stats, inv_scale, found_inf,
                         chunk_norms, h);
}

// stage 2: apply, refresh shadow, zero the gradient arena slot
__global__ void __launch_bounds__(OPT_THREADS)
lamb_stage2_kernel(float* __restrict__ g, float* __restrict__ p, __nv_bfloat16* __restrict__ shadow,
                   const int* __restrict__ chunk_tensor, const long long* __restrict__ chunk_start,
                   const int* __restrict__ chunk_len, const int* __restrict__ decay_flag,
                   const float* __restrict__ found_inf, const float* __restrict__ norms, LambHyper h) {
  const int c = blockIdx.x;
  const int t = chunk_tensor[c];
  const long long off = chunk_start[c];
  const int n = chunk_len[c];
  if (found_inf && *found_inf != 0.f) {  // skipped step: just clear the gradients
    for (int i = threadIdx.x; i < n; i += blockDim.x) g[off + i] = 0.f;
    return;
  }
  float ratio = h.lr;
  if (h.use_nvlamb || (decay_flag[t] && h.weight_decay != 0.f)) {
    const float pn = sqrtf(norms[2 * t]), un = sqrtf(norms[2 * t + 1]);
    if (pn > 0.f && un > 0.f) ratio = h.lr * pn / un;
  }
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float np = p[off + i] - ratio * g[off + i];
    p[off + i] = np;
    if (shadow) shadow[off + i] = __float2bfloat16(np);
    g[off + i] = 0.f;
  }
}

struct AdamHyper {
  float lr, beta1, beta2, eps, weight_decay, bc1, bc2;
  int adam_w_mode;
};

__global__ void __launch_bounds__(OPT_THREADS)
adam_kernel(float* __restrict__ g, float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
            __nv_bfloat16* __restrict__ shadow, const int* __restrict__ chunk_tensor,
            const long long* __restrict__ chunk_start, const int* __restrict__ chunk_len,
            const int* __restrict__ decay_flag, const float* __restrict__ inv_scale,
            const float* __restrict__ found_inf, AdamHyper h) {
  const int c = blockIdx.x;
  const int t = chunk_tensor[c];
  const long long off = chunk_start[c];
  const int n = chunk_len[c];
  if (found_inf && *found_inf != 0.f) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) g[off + i] = 0.f;
    return;
  }
  const float is = inv_scale ? *inv_scale : 1.f;
  const float wd = decay_flag[t] ? h.weight_decay : 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float gg = g[off + i] * is;
    const float pp = p[off + i];
    if (!h.adam_w_mode) gg += wd * pp;
    const float mm = h.beta1 * m[off + i] + (1.f - h.beta1) * gg;
    const float vv = h.beta2 * v[off + i] + (1.f - h.beta2) * gg * gg;
    float u = (mm / h.bc1) / (sqrtf(vv / h.bc2) + h.eps);
    if (h.adam_w_mode) u += wd * pp;
    const float np = pp - h.lr * u;
    m[off + i] = mm; v[off + i] = vv; p[off + i] = np;
    if (shadow) shadow[off + i] = __float2bfloat16(np);
    g[off + i] = 0.f;
  }
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
void mt_l2norm(int dtype, const long long* ptrs, const int* chunk_tensor, const long long* chunk_start,
               const int* chunk_len, int nchunks, float* per_tensor_sq, float* total_sq, cudaStream_t st,
               float* chunk_ws, int ntensors) {
  if (nchunks <= 0) return;
  if (chunk_ws != nullptr) {
    if (dtype == 0) mt_l2norm_part_kernel<float><<<nchunks, OPT_THREADS, 0, st>>>(ptrs, chunk_tensor, chunk_start, chunk_len, chunk_ws);
    else if (dtype == 1) mt_l2norm_part_kernel<__nv_bfloat16><<<nchunks, OPT_THREADS, 0, st>>>(ptrs, chunk_tensor, chunk_start, chunk_len, chunk_ws);
    else mt_l2norm_part_kernel<__half><<<nchunks, OPT_THREADS, 0, st>>>(ptrs, chunk_tensor, chunk_start, chunk_len, chunk_ws);
    if (per_tensor_sq) ordered_sum(chunk_ws, nchunks, 1, chunk_tensor, ntensors, per_tensor_sq, st);
    ordered_sum(chunk_ws, nchunks, 1, nullptr, 1, total_sq, st);
    return;
  }
  if (dtype == 0) mt_l2norm_kernel<float><<<nchunks, OPT_THREADS, 0, st>>>(ptrs, chunk_tensor, chunk_start, chunk_len, per_tensor_sq, total_sq);
  else if (dtype == 1) mt_l2norm_kernel<__nv_bfloat16><<<nchunks, OPT_THREADS, 0, st>>>(ptrs, chunk_tensor, chunk_start, chunk_len, per_tensor_sq, total_sq);
  else mt_l2norm_kernel<__half><<<nchunks, OPT_THREADS, 0, st>>>(ptrs, chunk_tensor, chunk_start, chunk_len, per_tensor_sq, total_sq);
}

template <typename TI>
static void mt_scale_out(int out_dtype, const long long* in_ptrs, const long long* out_ptrs, const int* ct,
                         const long long* cs, const int* cl, int nchunks, const float* sd, float sh, int* ovf,
                         cudaStream_t st) {
  if (out_dtype == 0) mt_scale_kernel<TI, float><<<nchunks, OPT_THREADS, 0, st>>>(in_ptrs, out_ptrs, ct, cs, cl, sd, sh, ovf);
  else if (out_dtype == 1) mt_scale_kernel<TI, __nv_bfloat16><<<nchunks, OPT_THREADS, 0, st>>>(in_ptrs, out_ptrs, ct, cs, cl, sd, sh, ovf);
  else mt_scale_kernel<TI, __half><<<nchunks, OPT_THREADS, 0, st>>>(in_ptrs, out_ptrs, ct, cs, cl, sd, sh, ovf);
}
void mt_scale(int in_dtype, int out_dtype, const long long* in_ptrs, const long long* out_ptrs,
              const int* chunk_tensor, const long long* chunk_start, const int* chunk_len, int nchunks,
              const float* scale_dev, float scale_host, int* overflow, cudaStream_t st) {
  if (nchunks <= 0) return;
  if (in_dtype == 0) mt_scale_out<float>(out_dtype, in_ptrs, out_ptrs, chunk_tensor, chunk_start, chunk_len, nchunks, scale_dev, scale_host, overflow, st);
  else if (in_dtype == 1) mt_scale_out<__nv_bfloat16>(out_dtype, in_ptrs, out_ptrs, chunk_tensor, chunk_start, chunk_len, nchunks, scale_dev, scale_host, overflow, st);
  else mt_scale_out<__half>(out_dtype, in_ptrs, out_ptrs, chunk_tensor, chunk_start, chunk_len, nchunks, scale_dev, scale_host, overflow, st);
}

int flat_sumsq_det_blocks() { return 512; }

void flat_sumsq(const float* g, long long n, const float* inv_scale, float* stats, float* found_inf, cudaStream_t st,
                float* block_ws) {
  B200_CUDA_CHECK(cudaMemsetAsync(stats, 0, sizeof(float), st));
  if (block_ws == nullptr) {
    flat_sumsq_kernel<<<num_sms() * 4, OPT_THREADS, 0, st>>>(g, n, inv_scale, stats, found_inf);
    return;
  }
  // a fixed grid: the block partition of the sum does not depend on the device either
  flat_sumsq_part_kernel<<<flat_sumsq_det_blocks(), OPT_THREADS, 0, st>>>(g, n, inv_scale, block_ws, found_inf);
  ordered_sum(block_ws, flat_sumsq_det_blocks(), 1, nullptr, 1, stats, st);
}
void flat_unscale(float* g, long long n, const float* inv_scale, float* found_inf, cudaStream_t st) {
  flat_unscale_kernel<<<num_sms() * 4, OPT_THREADS, 0, st>>>(g, n, inv_scale, found_inf);
}

void arena_lamb(float* g, float* p, float* m, float* v, void* shadow, const int* chunk_tensor,
                const long long* chunk_start, const int* chunk_len, int nchunks, const int* decay_flag,
                int ntensors, float* stats, float* norms, const float* inv_scale, const float* found_inf,
                float lr, float beta1, float beta2, float eps, float weight_decay, int step, int bias_correction,
                int grad_averaging, float max_grad_norm, int adam_w_mode, int use_nvlamb, cudaStream_t st,
                float* chunk_ws) {
  LambHyper h;
  h.lr = lr; h.beta1 = beta1; h.beta2 = beta2; h.beta3 = grad_averaging ? 1.f - beta1 : 1.f; h.eps = eps;
  h.weight_decay = weight_decay;
  h.bc1 = bias_correction ? 1.f - powf(beta1, (float)step) : 1.f;
  h.bc2 = bias_correction ? 1.f - powf(beta2, (float)step) : 1.f;
  h.max_grad_norm = max_grad_norm; h.adam_w_mode = adam_w_mode; h.use_nvlamb = use_nvlamb;
  B200_CUDA_CHECK(cudaMemsetAsync(norms, 0, sizeof(float) * 2 * ntensors, st));
  if (chunk_ws == nullptr) {
    lamb_stage1_kernel<<<nchunks, OPT_THREADS, 0, st>>>(g, p, m, v, chunk_tensor, chunk_start, chunk_len, decay_flag,
                                                       stats, inv_scale, found_inf, norms, h);
  } else {
    lamb_stage1_part_kernel<<<nchunks, OPT_THREADS, 0, st>>>(g, p, m, v, chunk_tensor, chunk_start, chunk_len,
                                                            decay_flag, stats, inv_scale, found_inf, chunk_ws, h);
    ordered_sum(chunk_ws, nchunks, 2, chunk_tensor, ntensors, norms, st);
  }
  lamb_stage2_kernel<<<nchunks, OPT_THREADS, 0, st>>>(g, p, (__nv_bfloat16*)shadow, chunk_tensor, chunk_start,
                                                     chunk_len, decay_flag, found_inf, norms, h);
}

void arena_adam(float* g, float* p, float* m, float* v, void* shadow, const int* chunk_tensor,
                const long long* chunk_start, const int* chunk_len, int nchunks, const int* decay_flag,
                const float* inv_scale, const float* found_inf, float lr, float beta1, float beta2, float eps,
                float weight_decay, int step, int bias_correction, int adam_w_mode, cudaStream_t st) {
  AdamHyper h;
  h.lr = lr; h.beta1 = beta1; h.beta2 = beta2; h.eps = eps; h.weight_decay = weight_decay;
  h.bc1 = bias_correction ? 1.f - powf(beta1, (float)step) : 1.f;
  h.bc2 = bias_correction ? 1.f - powf(beta2, (float)step) : 1.f;
  h.adam_w_mode = adam_w_mode;
  adam_kernel<<<nchunks, OPT_THREADS, 0, st>>>(g, p, m, v, (__nv_bfloat16*)shadow, chunk_tensor, chunk_start,
                                              chunk_len, decay_flag, inv_scale, found_inf, h);
}

}  // namespace b200
