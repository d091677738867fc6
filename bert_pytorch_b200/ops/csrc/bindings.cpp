// torch <-> kernel glue.  Every function takes torch tensors, checks what the kernels assume (device,
// dtype, contiguity, alignment) and launches on the current CUDA stream.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "gemm_sm90.h"
#include "kernels.h"

namespace {

using torch::Tensor;

inline cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }
// fp32 workspace of a deterministic-mode kernel chain, from the caching allocator on the current stream (stream-ordered:
// it is only reused by work queued after the chain)
inline Tensor f32_workspace(const Tensor& like, int64_t n) {
  return at::empty({std::max<int64_t>(n, 1)}, like.options().dtype(at::kFloat));
}
inline void check_bf16(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
  TORCH_CHECK(t.scalar_type() == at::kBFloat16, name, " must be bf16");
  TORCH_CHECK(t.stride(-1) == 1, name, " must have a unit inner stride");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0, name, " must be 16-byte aligned");
}
// Device-resident dropout step counter mixed into every seed (set by the engine when it captures CUDA graphs:
// the pointer is baked into the captured launches, the counter is advanced inside the graph).
const unsigned long long* g_seed_step = nullptr;
Tensor g_seed_step_keepalive;
void set_seed_step(c10::optional<Tensor> t) {
  if (t.has_value() && t->defined()) {
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kLong && t->numel() == 1, "seed step must be a CUDA int64 scalar");
    g_seed_step_keepalive = *t;
    g_seed_step = reinterpret_cast<const unsigned long long*>(t->data_ptr<int64_t>());
  } else {
    g_seed_step = nullptr;
    g_seed_step_keepalive = Tensor();
  }
}
inline b200::Seed mk_seed(int64_t seed) { return b200::Seed{static_cast<unsigned long long>(seed), g_seed_step}; }

// Gradient arenas in NVLink symmetric memory: once registered, every fp32-accumulate GEMM whose output lies inside
// the local arena adds atomically (peers may be adding into it), and with `push` on the tile goes straight to
// the owner rank's arena (GEMM -> reduce-scatter in one kernel).
struct GradPeers {
  int world = 0, rank = 0, push = 0;
  int64_t numel = 0, per = 0;
  float* base[16] = {};
} g_grad_peers;
void set_grad_peers(int64_t world, int64_t rank, std::vector<int64_t> ptrs, int64_t numel, int64_t per) {
  TORCH_CHECK(world <= 16 && (int64_t)ptrs.size() == world, "set_grad_peers: <= 16 ranks, one pointer each");
  g_grad_peers = GradPeers();
  g_grad_peers.world = (int)world; g_grad_peers.rank = (int)rank; g_grad_peers.numel = numel; g_grad_peers.per = per;
  for (int i = 0; i < world; ++i) g_grad_peers.base[i] = reinterpret_cast<float*>(ptrs[i]);
}
void set_grad_push(bool on) { g_grad_peers.push = on ? 1 : 0; }
int64_t grad_peers_world() { return g_grad_peers.world; }

// optional fp8 side output: (q bytes, meta record, e5m2)
inline b200::Fp8Out mk_fp8(const c10::optional<Tensor>& q, const c10::optional<Tensor>& meta, bool e5m2, int64_t numel) {
  b200::Fp8Out f;
  if (q.has_value() && q->defined()) {
    TORCH_CHECK(meta.has_value() && meta->defined() && meta->scalar_type() == at::kFloat && meta->numel() >= 4, "fp8 meta");
    TORCH_CHECK(q->is_cuda() && q->is_contiguous() && q->element_size() == 1 && q->numel() == numel, "fp8 side output shape");
    f.q = reinterpret_cast<unsigned char*>(q->data_ptr());
    f.meta = meta->data_ptr<float>();
    f.e5m2 = e5m2 ? 1 : 0;
  }
  return f;
}

inline const void* opt_ptr(const c10::optional<Tensor>& t) { return t.has_value() && t->defined() ? t->data_ptr() : nullptr; }
inline float* opt_f32(const c10::optional<Tensor>& t) {
  if (!t.has_value() || !t->defined()) return nullptr;
  TORCH_CHECK(t->scalar_type() == at::kFloat && t->is_cuda(), "expected a CUDA fp32 tensor");
  return t->data_ptr<float>();
}

// D = epilogue(A op B).  a/b are 2-D bf16 (row stride arbitrary, multiple of 8 elements).
//   layout 0 (NT): a [M,K], b [N,K]     1 (NN): a [M,K], b [K,N]     2 (TN): a [K,M], b [K,N]
// fp8 mode (scale_a/scale_b given): a/b are 1-byte e4m3 (or e5m2, per flag) tensors, row strides multiples of 16,
// scale_* are the device inv_scale floats (views into the fp8 meta table).
static inline bool p_drop_is_zero(double p) { return !(p > 0.0); }

void gemm(Tensor a, Tensor b, Tensor out, int64_t layout, int64_t epi, c10::optional<Tensor> bias,
          c10::optional<Tensor> res, c10::optional<Tensor> aux_out, int64_t k_splits, int64_t block_n, double alpha,
          double p_drop, int64_t seed, int64_t stream_id, c10::optional<Tensor> scale_a, c10::optional<Tensor> scale_b,
          bool a_e5m2, bool b_e5m2, bool allow_push, c10::optional<Tensor> colsum, c10::optional<Tensor> mask_out,
          c10::optional<Tensor> mask_in) {
  const bool fp8 = scale_a.has_value() && scale_a->defined();
  if (fp8) {
    TORCH_CHECK(a.is_cuda() && b.is_cuda() && a.element_size() == 1 && b.element_size() == 1 && a.stride(1) == 1 &&
                b.stride(1) == 1, "fp8 gemm operands must be CUDA 1-byte tensors with unit inner stride");
    TORCH_CHECK(scale_b.has_value() && scale_b->defined(), "fp8 gemm needs both dequantisation factors");
    TORCH_CHECK(a.stride(0) % 16 == 0 && b.stride(0) % 16 == 0 && reinterpret_cast<uintptr_t>(a.data_ptr()) % 16 == 0 &&
                reinterpret_cast<uintptr_t>(b.data_ptr()) % 16 == 0, "fp8 operands must be 16-byte aligned");
  } else {
    check_bf16(a, "a");
    check_bf16(b, "b");
  }
  TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && out.dim() == 2, "gemm operands must be 2-D");
  TORCH_CHECK(layout == b200::GEMM_NT || layout == b200::GEMM_NN || layout == b200::GEMM_TN, "unknown GEMM layout ", layout);
  const b200::EpilogueSpec spec = b200::epilogue_spec((int)epi);
  TORCH_CHECK(spec.name != nullptr, "unknown GEMM epilogue ", epi);
  c10::cuda::CUDAGuard guard(a.device());
  b200::GemmCall c;
  c.layout = (int)layout;
  c.epi = (int)epi;
  c.block_n = (int)block_n;
  int64_t M, N, K;
  if (layout == b200::GEMM_NT) { M = a.size(0); K = a.size(1); N = b.size(0); TORCH_CHECK(b.size(1) == K, "K mismatch"); }
  else if (layout == b200::GEMM_NN) { M = a.size(0); K = a.size(1); N = b.size(1); TORCH_CHECK(b.size(0) == K, "K mismatch"); }
  else { K = a.size(0); M = a.size(1); N = b.size(1); TORCH_CHECK(b.size(0) == K, "K mismatch"); }
  TORCH_CHECK(out.size(0) == M && out.size(1) == N, "output shape mismatch");
  TORCH_CHECK(a.stride(0) % 8 == 0 && b.stride(0) % 8 == 0, "row strides must be multiples of 8 elements");
  TORCH_CHECK(N % 8 == 0, "N must be a multiple of 8");
  // an empty reduction launches nothing: right for the accumulate-into epilogue (out += 0), but any other epilogue
  // would leave its output unwritten
  TORCH_CHECK(K > 0 || epi == b200::EPI_ACCUM_F32, "gemm: K == 0 leaves the ", spec.name, " output unwritten");
  TORCH_CHECK(block_n == 128 || block_n == 256, "gemm: block_n must be 128 or 256 (the tile widths), got ", block_n);
  // only the fp32 accumulate-into epilogue merges K ranges (split-K); any other epilogue would ignore the split
  TORCH_CHECK(k_splits == 1 || epi == b200::EPI_ACCUM_F32, "gemm: k_splits = ", k_splits, " needs EPI_ACCUM_F32, not ",
              spec.name);
  TORCH_CHECK(p_drop_is_zero(p_drop) || spec.keep_bits, "gemm: p_drop > 0 but ", spec.name, " applies no dropout");
  TORCH_CHECK(out.is_cuda() && out.stride(1) == 1, "out must be CUDA with unit inner stride");
  TORCH_CHECK(out.scalar_type() == (spec.f32_out ? at::kFloat : at::kBFloat16), "out dtype does not match the epilogue");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(out.data_ptr()) % 16 == 0 && out.stride(0) % (spec.f32_out ? 4 : 8) == 0,
              "out must be 16-byte aligned with an aligned row stride");
  c.M = (int)M; c.N = (int)N; c.K = (int)K;
  if (fp8) {
    c.fp8 = true; c.a_e5m2 = a_e5m2; c.b_e5m2 = b_e5m2;
    c.scale_a = opt_f32(scale_a); c.scale_b = opt_f32(scale_b);
  }
  c.A = a.data_ptr(); c.lda = (int)a.stride(0);
  c.B = b.data_ptr(); c.ldb = (int)b.stride(0);
  c.out = out.data_ptr(); c.ldo = (int)out.stride(0);
  // an input or output the epilogue does not read or write is refused rather than ignored
  if (aux_out.has_value() && aux_out->defined()) {
    TORCH_CHECK(spec.aux, "aux_out is not written by ", spec.name);
    check_bf16(*aux_out, "aux_out");
    TORCH_CHECK(aux_out->dim() == 2 && aux_out->size(0) == M && aux_out->size(1) == N, "aux_out must be [M, N]");
    TORCH_CHECK(aux_out->stride(0) == out.stride(0), "aux_out must share out's row stride");
    c.aux_out = aux_out->data_ptr();
  }
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(spec.bias, "bias is not read by ", spec.name);
    check_bf16(*bias, "bias");
    TORCH_CHECK(bias->numel() == N, "bias length");
    c.bias = bias->data_ptr();
  }
  if (res.has_value() && res->defined()) {
    TORCH_CHECK(spec.res || epi == b200::EPI_ADD, "res is not read by ", spec.name);
    check_bf16(*res, "res");
    TORCH_CHECK(res->size(0) == M && res->size(1) == N && res->stride(0) % 8 == 0, "res shape");
    c.res = res->data_ptr(); c.ldr = (int)res->stride(0);
  }
  TORCH_CHECK(!spec.bias || c.bias != nullptr, spec.name, " needs a bias");
  TORCH_CHECK(!spec.aux || c.aux_out != nullptr, spec.name, " needs aux_out");
  TORCH_CHECK(!spec.res || c.res != nullptr, spec.name, " needs res");
  if (colsum.has_value() && colsum->defined()) {
    TORCH_CHECK(spec.colsum, "column sums are not fused into ", spec.name);
    TORCH_CHECK(colsum->numel() == N && colsum->is_contiguous(), "colsum length");
    c.colsum = opt_f32(colsum);
  }
  if (mask_out.has_value() && mask_out->defined()) {
    TORCH_CHECK(spec.keep_bits && !p_drop_is_zero(p_drop), "mask_out: dropout epilogue only");
    TORCH_CHECK(mask_out->is_cuda() && mask_out->scalar_type() == at::kByte && mask_out->is_contiguous() &&
                mask_out->numel() == M * (N / 8) && reinterpret_cast<uintptr_t>(mask_out->data_ptr()) % 16 == 0 && N % 128 == 0,
                "mask_out: uint8 [M, N / 8], 16-byte aligned, N % 128 == 0");
    c.mask_out = mask_out->data_ptr<uint8_t>();
  }
  if (mask_in.has_value() && mask_in->defined()) {
    TORCH_CHECK(spec.keep_bits && !p_drop_is_zero(p_drop), "mask_in: dropout epilogue only");
    TORCH_CHECK(mask_in->is_cuda() && mask_in->scalar_type() == at::kByte && mask_in->is_contiguous() &&
                mask_in->numel() == M * (N / 8) && reinterpret_cast<uintptr_t>(mask_in->data_ptr()) % 16 == 0 && N % 128 == 0,
                "mask_in: uint8 [M, N / 8], 16-byte aligned, N % 128 == 0");
    c.mask_in = mask_in->data_ptr<uint8_t>();
  }
  c.k_splits = (int)k_splits;
  c.alpha = (float)alpha;
  c.p_drop = (float)p_drop;
  c.seed = (unsigned long long)seed;
  c.seed_step = g_seed_step;
  if (epi == b200::EPI_ACCUM_F32 && g_grad_peers.world > 1) {
    const float* lo = g_grad_peers.base[g_grad_peers.rank];
    const float* o = reinterpret_cast<const float*>(out.data_ptr());
    if (o >= lo && o < lo + g_grad_peers.numel) {
      c.peer_world = g_grad_peers.world; c.peer_rank = g_grad_peers.rank;
      c.peer_push = (g_grad_peers.push && allow_push) ? 1 : 0;   // only tensors the fused step knows to be pre-reduced
      c.peer_off = (long long)(o - lo); c.peer_per = g_grad_peers.per;
      for (int i = 0; i < g_grad_peers.world; ++i) c.peer_base[i] = g_grad_peers.base[i];
    }
  }
  c.stream = (unsigned int)stream_id;
  static const char* const form[] = {"NT bf16", "NN bf16", "TN bf16"};
  TORCH_CHECK(b200::gemm_bf16(c, cur_stream()), "gemm: no kernel is built for ", fp8 ? "fp8" : form[layout],
              " operands with ", spec.name);
}

// In-kernel GEMM timeline (tools/gemm_timeline.py): `buf` is int64 [units, 16]; None turns recording off.
bool gemm_timeline(c10::optional<Tensor> buf) {
  if (!buf.has_value() || !buf->defined()) return b200::gemm_set_timeline(nullptr, 0);
  TORCH_CHECK(buf->is_cuda() && buf->scalar_type() == at::kLong && buf->is_contiguous() && buf->dim() == 2 &&
              buf->size(1) == 16, "gemm_timeline: int64 CUDA tensor [units, 16]");
  return b200::gemm_set_timeline(reinterpret_cast<long long*>(buf->data_ptr<int64_t>()), buf->size(0));
}

// the LayerNorm kernels cover H % 8 == 0 up to 2048 (8 columns per lane, at most 8 warps or chunks of 256 per row)
inline void check_ln_width(int64_t H) {
  TORCH_CHECK(H > 0 && H % 8 == 0 && H <= 2048, "LayerNorm: hidden size ", H, " is not a multiple of 8 in [8, 2048]");
}
// fp32 CUDA vector of n elements; `vec16`: read with 16-byte loads (gamma / beta), so its start must be 16-byte aligned
inline void check_f32_vec(const Tensor& t, int64_t n, const char* name, bool vec16) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat && t.is_contiguous(), name, " must be a contiguous CUDA fp32 tensor");
  TORCH_CHECK(t.numel() == n, name, " has ", t.numel(), " elements, expected ", n);
  TORCH_CHECK(!vec16 || reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0, name, " must be 16-byte aligned");
}
inline void check_opt_f32_vec(const c10::optional<Tensor>& t, int64_t n, const char* name) {
  if (t.has_value() && t->defined()) check_f32_vec(*t, n, name, false);
}

void layer_norm_fwd(Tensor x,Tensor gamma, Tensor beta, Tensor y, c10::optional<Tensor> mean,
                    c10::optional<Tensor> rstd, double eps, c10::optional<Tensor> q8, c10::optional<Tensor> meta8,
                    bool e5m2) {
  check_ln_width(x.size(-1));
  check_bf16(x, "x"); check_bf16(y, "y");
  TORCH_CHECK(x.is_contiguous() && y.is_contiguous() && y.numel() == x.numel(), "x/y must be contiguous and of one size");
  const int H = (int)x.size(-1), M = (int)(x.numel() / H);
  check_f32_vec(gamma, H, "gamma", true); check_f32_vec(beta, H, "beta", true);
  check_opt_f32_vec(mean, M, "mean"); check_opt_f32_vec(rstd, M, "rstd");
  c10::cuda::CUDAGuard guard(x.device());
  b200::layer_norm_fwd(x.data_ptr(), gamma.data_ptr<float>(), beta.data_ptr<float>(), y.data_ptr(), opt_f32(mean),
                       opt_f32(rstd), M, H, (float)eps, mk_fp8(q8, meta8, e5m2, x.numel()), cur_stream());
}

int64_t ln_bwd_workspace(int64_t M, int64_t H) { return b200::ln_bwd_workspace_floats((int)M, (int)H); }

void layer_norm_bwd(Tensor dy, Tensor x, Tensor mean, Tensor rstd, Tensor gamma, Tensor dx, c10::optional<Tensor> dxd,
                    c10::optional<Tensor> dgamma, c10::optional<Tensor> dbeta, c10::optional<Tensor> dbias,
                    Tensor workspace, double p_drop, int64_t seed, int64_t drop_stream, int64_t in_stream,
                    c10::optional<Tensor> q8, c10::optional<Tensor> meta8, bool e5m2, c10::optional<Tensor> keep_mask,
                    bool deterministic) {
  check_ln_width(x.size(-1));
  check_bf16(dy, "dy"); check_bf16(x, "x"); check_bf16(dx, "dx");
  TORCH_CHECK(x.is_contiguous() && dy.is_contiguous() && dx.is_contiguous() && dy.numel() == x.numel() &&
              dx.numel() == x.numel(), "dy/x/dx must be contiguous and of one size");
  const int H = (int)x.size(-1), M = (int)(x.numel() / H);
  check_f32_vec(mean, M, "mean", false); check_f32_vec(rstd, M, "rstd", false);
  check_f32_vec(gamma, H, "gamma", true);
  check_opt_f32_vec(dgamma, H, "dgamma"); check_opt_f32_vec(dbeta, H, "dbeta"); check_opt_f32_vec(dbias, H, "dbias");
  TORCH_CHECK(workspace.numel() >= b200::ln_bwd_workspace_floats(M, H), "LN workspace too small");
  c10::cuda::CUDAGuard guard(x.device());
  void* dxd_p = nullptr;
  if (dxd.has_value() && dxd->defined()) {
    check_bf16(*dxd, "dxd");
    TORCH_CHECK(dxd->is_contiguous() && dxd->numel() == x.numel(), "dxd must be contiguous and of the size of x");
    dxd_p = dxd->data_ptr();
  }
  const uint8_t* km = nullptr;
  if (keep_mask.has_value() && keep_mask->defined()) {   // keep bits written by the producing GEMM (GemmCall::mask_out)
    TORCH_CHECK(keep_mask->is_cuda() && keep_mask->scalar_type() == at::kByte && keep_mask->is_contiguous() &&
                keep_mask->numel() == (int64_t)M * (H / 8), "keep_mask: uint8 [M, H / 8]");
    km = keep_mask->data_ptr<uint8_t>();
  }
  b200::layer_norm_bwd(dy.data_ptr(), x.data_ptr(), mean.data_ptr<float>(), rstd.data_ptr<float>(),
                       gamma.data_ptr<float>(), dx.data_ptr(), dxd_p, opt_f32(dgamma), opt_f32(dbeta), opt_f32(dbias),
                       workspace.data_ptr<float>(), M, H, mk_seed(seed), (unsigned)drop_stream,
                       (unsigned)in_stream, (float)p_drop, mk_fp8(q8, meta8, e5m2, x.numel()), cur_stream(), km,
                       deterministic);
}

void gelu_fwd(Tensor x, Tensor y, c10::optional<Tensor> q8, c10::optional<Tensor> meta8, bool e5m2) {
  check_bf16(x, "x"); check_bf16(y, "y");
  TORCH_CHECK(x.is_contiguous() && y.is_contiguous() && x.numel() == y.numel() && x.numel() % 8 == 0, "gelu_fwd shapes");
  c10::cuda::CUDAGuard guard(x.device());
  b200::gelu_fwd(x.data_ptr(), y.data_ptr(), x.numel(), mk_fp8(q8, meta8, e5m2, x.numel()), cur_stream());
}
void dgelu_bwd(Tensor dy, Tensor x, Tensor dx, c10::optional<Tensor> dbias, c10::optional<Tensor> q8,
               c10::optional<Tensor> meta8, bool e5m2, bool deterministic) {
  check_bf16(dy, "dy"); check_bf16(x, "x"); check_bf16(dx, "dx");
  TORCH_CHECK(dy.dim() == 2 && dy.is_contiguous() && x.is_contiguous() && dx.is_contiguous() && dy.size(1) % 8 == 0,
              "dgelu_bwd: contiguous [M,N] with N % 8 == 0");
  c10::cuda::CUDAGuard guard(x.device());
  const int M = (int)dy.size(0), N = (int)dy.size(1);
  Tensor ws;
  if (deterministic && opt_f32(dbias) != nullptr) ws = f32_workspace(dy, b200::dgelu_det_workspace_floats(M, N));
  b200::dgelu_bwd(dy.data_ptr(), x.data_ptr(), dx.data_ptr(), opt_f32(dbias), M, N, mk_fp8(q8, meta8, e5m2, dy.numel()),
                  cur_stream(), ws.defined() ? ws.data_ptr<float>() : nullptr);
}

void colsum(Tensor x, Tensor out, bool deterministic) {
  check_bf16(x, "x");
  TORCH_CHECK(x.dim() == 2 && out.scalar_type() == at::kFloat && out.numel() == x.size(1), "colsum shapes");
  c10::cuda::CUDAGuard guard(x.device());
  TORCH_CHECK(out.is_cuda() && out.is_contiguous(), "colsum: out must be a contiguous CUDA tensor");
  const int M = (int)x.size(0), N = (int)x.size(1);
  // both kernels read 8 columns with one 16-byte load: unit column stride (check_bf16), N and the row stride in 8s
  TORCH_CHECK(N % 8 == 0 && x.stride(0) % 8 == 0, "colsum: N and the row stride must be multiples of 8");
  if (M == 0 || N == 0) return;
  if (deterministic) {
    Tensor ws = f32_workspace(out, b200::colsum_det_workspace_floats(M, N));
    b200::colsum_bf16_det(x.data_ptr(), M, N, (int)x.stride(0), out.data_ptr<float>(), ws.data_ptr<float>(), cur_stream());
    return;
  }
  b200::colsum_bf16(x.data_ptr(), M, N, (int)x.stride(0), out.data_ptr<float>(), cur_stream());
}

// out[W] += part[rows, W] summed over the rows in row order (deterministic mode)
void ordered_sum(Tensor part, Tensor out) {
  TORCH_CHECK(part.is_cuda() && part.scalar_type() == at::kFloat && part.is_contiguous() && part.dim() >= 2,
              "ordered_sum: contiguous fp32 part [rows, ...]");
  TORCH_CHECK(out.scalar_type() == at::kFloat && out.is_contiguous() && out.numel() * part.size(0) == part.numel(),
              "ordered_sum: out must be a contiguous fp32 tensor of one row of part");
  c10::cuda::CUDAGuard guard(part.device());
  b200::ordered_sum(part.data_ptr<float>(), (int)part.size(0), (int)out.numel(), nullptr, 1, out.data_ptr<float>(),
                    cur_stream());
}

// pos_ids (optional int32 [M]): position of every token row (packed rows of an unpadded batch); else row % S
inline const int* opt_pos_ids(const c10::optional<Tensor>& pos_ids, const Tensor& ids) {
  if (!pos_ids.has_value() || !pos_ids->defined()) return nullptr;
  TORCH_CHECK(pos_ids->scalar_type() == at::kInt && pos_ids->is_contiguous() && pos_ids->numel() == ids.numel() &&
              pos_ids->device() == ids.device(), "pos_ids must be a contiguous int32 tensor like ids");
  return pos_ids->data_ptr<int>();
}

void embedding_fwd(Tensor ids, c10::optional<Tensor> seg, Tensor word, Tensor pos, c10::optional<Tensor> type,
                   Tensor gamma, Tensor beta, Tensor e_out, Tensor y, Tensor mean, Tensor rstd, int64_t S, double eps,
                   double p_drop, int64_t seed, int64_t stream_id, c10::optional<Tensor> pos_ids) {
  TORCH_CHECK(ids.scalar_type() == at::kInt && ids.is_contiguous(), "ids must be contiguous int32");
  check_bf16(word, "word"); check_bf16(pos, "pos"); check_bf16(e_out, "e_out"); check_bf16(y, "y");
  TORCH_CHECK(word.dim() == 2 && pos.dim() == 2 && word.is_contiguous() && pos.is_contiguous(),
              "word / position tables must be contiguous [rows, H]");
  const int H = (int)word.size(1), M = (int)ids.numel();
  check_ln_width(H);
  TORCH_CHECK(pos.size(1) == H, "position table width ", pos.size(1), " != ", H);
  TORCH_CHECK(S > 0, "embedding_fwd: S must be positive");
  TORCH_CHECK(e_out.is_contiguous() && y.is_contiguous() && e_out.numel() == (int64_t)M * H && y.numel() == (int64_t)M * H,
              "e_out / y must be contiguous [M, H]");
  check_f32_vec(gamma, H, "gamma", true); check_f32_vec(beta, H, "beta", true);
  check_f32_vec(mean, M, "mean", false); check_f32_vec(rstd, M, "rstd", false);
  c10::cuda::CUDAGuard guard(ids.device());
  const int* seg_p = nullptr;
  const void* type_p = nullptr;
  if (type.has_value() && type->defined()) {
    TORCH_CHECK(seg.has_value() && seg->defined() && seg->scalar_type() == at::kInt && seg->is_contiguous() &&
                seg->numel() == M, "segment ids must be a contiguous int32 tensor like ids");
    check_bf16(*type, "type");
    TORCH_CHECK(type->dim() == 2 && type->is_contiguous() && type->size(1) == H, "token-type table must be contiguous [rows, H]");
    seg_p = seg->data_ptr<int>();
    type_p = type->data_ptr();
  }
  if (M == 0) return;
  b200::embedding_fwd(ids.data_ptr<int>(), seg_p, word.data_ptr(), pos.data_ptr(), type_p, gamma.data_ptr<float>(),
                      beta.data_ptr<float>(), e_out.data_ptr(), y.data_ptr(), mean.data_ptr<float>(),
                      rstd.data_ptr<float>(), M, (int)S, H, (float)eps, mk_seed(seed), (unsigned)stream_id,
                      (float)p_drop, cur_stream(), opt_pos_ids(pos_ids, ids));
}

void embedding_bwd_scatter(Tensor de, Tensor ids, c10::optional<Tensor> seg, Tensor gword, Tensor gpos,
                           c10::optional<Tensor> gtype, int64_t S, c10::optional<Tensor> pos_ids, bool deterministic) {
  check_bf16(de, "de");
  const int H = (int)de.size(-1), M = (int)ids.numel();
  check_ln_width(H);
  TORCH_CHECK(ids.scalar_type() == at::kInt && ids.is_contiguous(), "ids must be contiguous int32");
  TORCH_CHECK(de.is_contiguous() && de.numel() == (int64_t)M * H, "de must be contiguous [M, H]");
  TORCH_CHECK(S > 0, "embedding backward: S must be positive");
  auto check_table = [&](const Tensor& t, const char* name) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat && t.is_contiguous() && t.dim() == 2 && t.size(1) == H &&
                reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0, name, " must be a contiguous 16-byte aligned fp32 [rows, H]");
  };
  check_table(gword, "gword"); check_table(gpos, "gpos");
  if (gtype.has_value() && gtype->defined()) check_table(*gtype, "gtype");
  if (seg.has_value() && seg->defined())
    TORCH_CHECK(seg->scalar_type() == at::kInt && seg->is_contiguous() && seg->numel() == M,
                "segment ids must be a contiguous int32 tensor like ids");
  if (M == 0) return;
  c10::cuda::CUDAGuard guard(de.device());
  if (deterministic) {
    const int chunk = std::min(M, b200::embedding_det_chunk_rows());   // rows sorted at a time
    int64_t rows = std::max(gword.size(0), gpos.size(0));
    if (gtype.has_value() && gtype->defined()) rows = std::max(rows, gtype->size(0));
    TORCH_CHECK(rows * (int64_t)chunk < (int64_t(1) << 32), "deterministic embedding backward: table rows x ", chunk,
                " must stay below 2^32");
    Tensor sort_ws = at::empty({std::max(chunk, 1)}, ids.options().dtype(at::kInt));
    Tensor sum_ws = f32_workspace(gword, (int64_t)chunk * H);
    b200::embedding_bwd_det(de.data_ptr(), ids.data_ptr<int>(),
                            seg.has_value() && seg->defined() ? seg->data_ptr<int>() : nullptr, gword.data_ptr<float>(),
                            gpos.data_ptr<float>(), opt_f32(gtype), M, (int)S, H, opt_pos_ids(pos_ids, ids),
                            reinterpret_cast<unsigned*>(sort_ws.data_ptr<int>()), sum_ws.data_ptr<float>(), cur_stream());
    return;
  }
  b200::embedding_bwd_scatter(de.data_ptr(), ids.data_ptr<int>(),
                              seg.has_value() && seg->defined() ? seg->data_ptr<int>() : nullptr,
                              gword.data_ptr<float>(), gpos.data_ptr<float>(), opt_f32(gtype), M, (int)S, H,
                              gtype.has_value() && gtype->defined() ? (int)gtype->size(0) : 0, cur_stream(),
                              opt_pos_ids(pos_ids, ids));
}

inline void check_i32(const Tensor& t, const Tensor& like, int64_t numel, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.device() == like.device(), name, " must be a CUDA tensor on the device of the batch");
  TORCH_CHECK(t.scalar_type() == at::kInt && t.is_contiguous() && t.numel() == numel, name, " must be a contiguous int32 "
              "tensor of ", numel, " elements");
}

// row_map (optional, int32 [B*S], from pack_tokens): idx gets packed rows, labels of masked tokens are dropped
void mlm_compact(Tensor labels, int64_t max_pred, Tensor idx, Tensor tgt, Tensor count, c10::optional<Tensor> row_map) {
  TORCH_CHECK(labels.scalar_type() == at::kInt && labels.dim() == 2 && labels.is_contiguous(), "labels: int32 [B,S]");
  const int* rm = nullptr;
  if (row_map.has_value() && row_map->defined()) {
    TORCH_CHECK(labels.is_cuda(), "labels must be a CUDA tensor");
    check_i32(*row_map, labels, labels.numel(), "row_map");
    check_i32(idx, labels, labels.size(0) * max_pred, "idx");
    check_i32(tgt, labels, labels.size(0) * max_pred, "tgt");
    check_i32(count, labels, 1, "count");
    rm = row_map->data_ptr<int>();
  }
  c10::cuda::CUDAGuard guard(labels.device());
  b200::mlm_compact(labels.data_ptr<int>(), (int)labels.size(0), (int)labels.size(1), (int)max_pred,
                    idx.data_ptr<int>(), tgt.data_ptr<int>(), count.data_ptr<int>(), cur_stream(), rm);
}

// Device packing of a [B, S] batch (see pack_tokens_kernel in norm_embed.cu).  mask / ids / seg: int32 [B, S] (seg
// optional); outputs ids, seg, pos [T_cap], cu [B + D + 1], cls [B], row_map [B * S], all int32.
void pack_tokens(Tensor mask, Tensor ids_in, c10::optional<Tensor> seg_in, int64_t T_cap, int64_t D, Tensor ids,
                 Tensor seg, Tensor pos, Tensor cu, Tensor cls, Tensor row_map) {
  TORCH_CHECK(mask.is_cuda(), "pack_tokens: mask must be a CUDA tensor");
  TORCH_CHECK(mask.dim() == 2, "pack_tokens: mask must be [B, S]");
  const int64_t B = mask.size(0), S = mask.size(1);
  TORCH_CHECK(B >= 1 && B <= b200::pack_tokens_max_batch() && S >= 1, "pack_tokens: 1 <= B <= ",
              b200::pack_tokens_max_batch(), " and S >= 1");
  TORCH_CHECK(T_cap >= 1 && D >= 0 && T_cap <= B * S + D * S, "pack_tokens: T_cap in [1, (B + D) * S], D >= 0");
  check_i32(mask, mask, B * S, "mask");
  check_i32(ids_in, mask, B * S, "input_ids");
  const int* seg_p = nullptr;
  if (seg_in.has_value() && seg_in->defined()) {
    check_i32(*seg_in, mask, B * S, "segment_ids");
    seg_p = seg_in->data_ptr<int>();
  }
  check_i32(ids, mask, T_cap, "ids");
  check_i32(seg, mask, T_cap, "seg");
  check_i32(pos, mask, T_cap, "pos_ids");
  check_i32(cu, mask, B + D + 1, "cu_seqlens");
  check_i32(cls, mask, B, "cls_rows");
  check_i32(row_map, mask, B * S, "row_map");
  c10::cuda::CUDAGuard guard(mask.device());
  b200::pack_tokens(mask.data_ptr<int>(), ids_in.data_ptr<int>(), seg_p, (int)B, (int)S, (int)T_cap, (int)D,
                    ids.data_ptr<int>(), seg.data_ptr<int>(), pos.data_ptr<int>(), cu.data_ptr<int>(),
                    cls.data_ptr<int>(), row_map.data_ptr<int>(), cur_stream());
}
void gather_rows(Tensor src, Tensor idx, Tensor dst) {
  check_bf16(src, "src"); check_bf16(dst, "dst");
  c10::cuda::CUDAGuard guard(src.device());
  b200::gather_rows(src.data_ptr(), idx.data_ptr<int>(), dst.data_ptr(), (int)idx.numel(), (int)src.size(-1), cur_stream());
}
void scatter_rows(Tensor src, Tensor idx, Tensor dst) {
  check_bf16(src, "src"); check_bf16(dst, "dst");
  c10::cuda::CUDAGuard guard(src.device());
  b200::scatter_rows(src.data_ptr(), idx.data_ptr<int>(), dst.data_ptr(), (int)idx.numel(), (int)src.size(-1), cur_stream());
}

void softmax_ce(Tensor logits, Tensor targets, Tensor count, double grad_scale, Tensor loss_out, bool deterministic) {
  check_bf16(logits, "logits");
  TORCH_CHECK(logits.dim() == 2 && logits.size(1) % 8 == 0 && logits.stride(0) % 8 == 0, "logits: [R,V], V%8==0");
  c10::cuda::CUDAGuard guard(logits.device());
  Tensor rows;
  if (deterministic) rows = f32_workspace(loss_out, logits.size(0));
  b200::softmax_ce(logits.data_ptr(), (int)logits.stride(0), targets.data_ptr<int>(), count.data_ptr<int>(),
                   (float)grad_scale, loss_out.data_ptr<float>(), (int)logits.size(0), (int)logits.size(1), cur_stream(),
                   deterministic ? rows.data_ptr<float>() : nullptr);
}

inline int dtype_code(const Tensor& t) {
  if (t.scalar_type() == at::kFloat) return 0;
  if (t.scalar_type() == at::kBFloat16) return 1;
  if (t.scalar_type() == at::kHalf) return 2;
  TORCH_CHECK(false, "unsupported dtype for multi-tensor op");
  return -1;
}

void mt_l2norm(int64_t dtype, Tensor ptrs, Tensor chunk_tensor, Tensor chunk_start, Tensor chunk_len,
               c10::optional<Tensor> per_tensor_sq, Tensor total_sq, bool deterministic) {
  c10::cuda::CUDAGuard guard(ptrs.device());
  Tensor ws;
  if (deterministic) ws = f32_workspace(total_sq, chunk_tensor.numel());
  b200::mt_l2norm((int)dtype, (const long long*)ptrs.data_ptr<int64_t>(), chunk_tensor.data_ptr<int>(),
                  (const long long*)chunk_start.data_ptr<int64_t>(), chunk_len.data_ptr<int>(),
                  (int)chunk_tensor.numel(), opt_f32(per_tensor_sq), total_sq.data_ptr<float>(), cur_stream(),
                  deterministic ? ws.data_ptr<float>() : nullptr, (int)ptrs.numel());
}
void mt_scale(int64_t in_dtype, int64_t out_dtype, Tensor in_ptrs, Tensor out_ptrs, Tensor chunk_tensor,
              Tensor chunk_start, Tensor chunk_len, c10::optional<Tensor> scale_dev, double scale_host, Tensor overflow) {
  c10::cuda::CUDAGuard guard(in_ptrs.device());
  b200::mt_scale((int)in_dtype, (int)out_dtype, (const long long*)in_ptrs.data_ptr<int64_t>(),
                 (const long long*)out_ptrs.data_ptr<int64_t>(), chunk_tensor.data_ptr<int>(),
                 (const long long*)chunk_start.data_ptr<int64_t>(), chunk_len.data_ptr<int>(), (int)chunk_tensor.numel(),
                 opt_f32(scale_dev), (float)scale_host, overflow.data_ptr<int>(), cur_stream());
}
void flat_sumsq(Tensor g, c10::optional<Tensor> inv_scale, Tensor stats, c10::optional<Tensor> found_inf,
                bool deterministic) {
  c10::cuda::CUDAGuard guard(g.device());
  TORCH_CHECK(g.numel() % 4 == 0, "arena size must be a multiple of 4");
  Tensor ws;
  if (deterministic) ws = f32_workspace(stats, b200::flat_sumsq_det_blocks());
  b200::flat_sumsq(g.data_ptr<float>(), g.numel(), opt_f32(inv_scale), stats.data_ptr<float>(), opt_f32(found_inf), cur_stream(),
                   deterministic ? ws.data_ptr<float>() : nullptr);
}
void flat_unscale(Tensor g, Tensor inv_scale, Tensor found_inf) {
  c10::cuda::CUDAGuard guard(g.device());
  TORCH_CHECK(g.numel() % 4 == 0, "arena size must be a multiple of 4");
  b200::flat_unscale(g.data_ptr<float>(), g.numel(), inv_scale.data_ptr<float>(), found_inf.data_ptr<float>(), cur_stream());
}
void arena_lamb(Tensor g, Tensor p, Tensor m, Tensor v, c10::optional<Tensor> shadow, Tensor chunk_tensor,
                Tensor chunk_start, Tensor chunk_len, Tensor decay_flag, Tensor stats, Tensor norms,
                c10::optional<Tensor> inv_scale, c10::optional<Tensor> found_inf, double lr, double beta1, double beta2,
                double eps, double weight_decay, int64_t step, bool bias_correction, bool grad_averaging,
                double max_grad_norm, bool adam_w_mode, bool use_nvlamb, bool deterministic) {
  c10::cuda::CUDAGuard guard(g.device());
  Tensor ws;
  if (deterministic) ws = f32_workspace(norms, 2 * chunk_tensor.numel());
  b200::arena_lamb(g.data_ptr<float>(), p.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(),
                   shadow.has_value() && shadow->defined() ? shadow->data_ptr() : nullptr, chunk_tensor.data_ptr<int>(),
                   (const long long*)chunk_start.data_ptr<int64_t>(), chunk_len.data_ptr<int>(), (int)chunk_tensor.numel(),
                   decay_flag.data_ptr<int>(), (int)decay_flag.numel(), stats.data_ptr<float>(), norms.data_ptr<float>(),
                   opt_f32(inv_scale), opt_f32(found_inf), (float)lr, (float)beta1, (float)beta2, (float)eps,
                   (float)weight_decay, (int)step, bias_correction, grad_averaging, (float)max_grad_norm, adam_w_mode,
                   use_nvlamb, cur_stream(), deterministic ? ws.data_ptr<float>() : nullptr);
}
void arena_adam(Tensor g, Tensor p, Tensor m, Tensor v, c10::optional<Tensor> shadow, Tensor chunk_tensor,
                Tensor chunk_start, Tensor chunk_len, Tensor decay_flag, c10::optional<Tensor> inv_scale,
                c10::optional<Tensor> found_inf, double lr, double beta1, double beta2, double eps, double weight_decay,
                int64_t step, bool bias_correction, bool adam_w_mode) {
  c10::cuda::CUDAGuard guard(g.device());
  b200::arena_adam(g.data_ptr<float>(), p.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(),
                   shadow.has_value() && shadow->defined() ? shadow->data_ptr() : nullptr, chunk_tensor.data_ptr<int>(),
                   (const long long*)chunk_start.data_ptr<int64_t>(), chunk_len.data_ptr<int>(), (int)chunk_tensor.numel(),
                   decay_flag.data_ptr<int>(), opt_f32(inv_scale), opt_f32(found_inf), (float)lr, (float)beta1,
                   (float)beta2, (float)eps, (float)weight_decay, (int)step, bias_correction, adam_w_mode, cur_stream());
}

// The attention kernels need head_dim 64 and S <= 512 with S % 8 == 0.  Padded form: qkv [B, S, 3H] with per-sequence
// valid lengths `seqlens` (int32 [B]), clamped to S; a length <= 0 (an all-zero mask row) attends to all S keys, as the
// model's additive mask does.  Varlen form (`cu_seqlens` given): qkv packed [T, 3H], sequence b is rows
// cu_seqlens[b] .. cu_seqlens[b + 1] (int32 [B + 1], B = lse.size(0)), S the padded length that sizes lse [B, h, S];
// it writes no fp8 side output.  Everything is checked before anything is launched.
struct AttnShape {
  int B, S, H;
  long long rows;                  // token rows of qkv: B * S, or T
  const int* seqlens;              // seqlens (padded) or nullptr
  const int* cu;                   // cu_seqlens (varlen) or nullptr
};
AttnShape check_attention(const Tensor& qkv, const c10::optional<Tensor>& seqlens, const Tensor& lse, int64_t heads,
                          const c10::optional<Tensor>& cu_seqlens, int64_t S_arg, bool fp8) {
  const bool varlen = cu_seqlens.has_value() && cu_seqlens->defined();
  TORCH_CHECK(qkv.dim() == (varlen ? 2 : 3) && qkv.is_contiguous(),
              varlen ? "attention: qkv must be a contiguous packed [T, 3H] tensor" : "attention: qkv must be a contiguous [B, S, 3H] tensor");
  AttnShape a;
  a.H = (int)(qkv.size(-1) / 3);
  TORCH_CHECK(heads > 0 && qkv.size(-1) % 3 == 0 && a.H % heads == 0 && a.H / heads == 64,
              "attention: the kernels need head dim 64 (got hidden ", a.H, " over ", heads, " heads)");
  const int64_t S = varlen ? S_arg : qkv.size(1);
  TORCH_CHECK(S <= 512 && S % 8 == 0, "attention: the kernels need S <= 512 and S % 8 == 0 (got S = ", S, ")");
  a.S = (int)S;
  if (varlen) {
    TORCH_CHECK(!fp8, "attention: the varlen form writes no fp8 side output");
    TORCH_CHECK(lse.dim() == 3 && lse.size(1) == heads && lse.size(2) == S, "attention: lse must be [B, heads, S]");
    a.B = (int)lse.size(0);
    const Tensor& cu = *cu_seqlens;
    TORCH_CHECK(cu.scalar_type() == at::kInt && cu.is_contiguous() && cu.dim() == 1 && cu.numel() == a.B + 1,
                "attention: cu_seqlens must be a contiguous int32 tensor of B + 1 = ", a.B + 1, " entries");
    TORCH_CHECK(cu.device() == qkv.device(), "attention: cu_seqlens must be on the device of qkv");
    a.rows = qkv.size(0);
    a.seqlens = nullptr;
    a.cu = cu.data_ptr<int>();
  } else {
    TORCH_CHECK(seqlens.has_value() && seqlens->defined(), "attention: the padded form needs seqlens");
    a.B = (int)qkv.size(0);
    a.rows = (long long)a.B * a.S;
    a.seqlens = seqlens->data_ptr<int>();
    a.cu = nullptr;
  }
  return a;
}

void attention_fwd(Tensor qkv, c10::optional<Tensor> seqlens, Tensor ctx, Tensor lse, int64_t heads, double scale,
                   double p_drop, int64_t seed, int64_t stream_id, c10::optional<Tensor> q8, c10::optional<Tensor> meta8,
                   bool e5m2, c10::optional<Tensor> cu_seqlens, int64_t S) {
  const AttnShape a = check_attention(qkv, seqlens, lse, heads, cu_seqlens, S, q8.has_value() && q8->defined());
  check_bf16(qkv, "qkv"); check_bf16(ctx, "ctx");
  TORCH_CHECK(ctx.numel() == a.rows * a.H && ctx.is_contiguous(), "attention_fwd: ctx must be contiguous [rows, H]");
  c10::cuda::CUDAGuard guard(qkv.device());
  b200::attention_fwd(qkv.data_ptr(), a.seqlens, ctx.data_ptr(), lse.data_ptr<float>(), a.B, a.S, (int)heads,
                      a.H / (int)heads, (float)scale, mk_seed(seed), (unsigned)stream_id, (float)p_drop,
                      mk_fp8(q8, meta8, e5m2, ctx.numel()), cur_stream(), a.cu, a.rows);
}
// S <= 128 runs the one-pass kernel, which needs neither delta_ws nor dq_acc, unless force_general.
void attention_bwd(Tensor qkv, c10::optional<Tensor> seqlens, Tensor ctx, Tensor dctx, Tensor lse, Tensor dqkv,
                   c10::optional<Tensor> delta_ws, c10::optional<Tensor> dq_acc, int64_t heads, double scale, double p_drop,
                   int64_t seed, int64_t stream_id, c10::optional<Tensor> q8, c10::optional<Tensor> meta8, bool e5m2,
                   c10::optional<Tensor> cu_seqlens, int64_t S, bool deterministic, bool force_general) {
  const AttnShape a = check_attention(qkv, seqlens, lse, heads, cu_seqlens, S, q8.has_value() && q8->defined());
  check_bf16(qkv, "qkv"); check_bf16(ctx, "ctx"); check_bf16(dctx, "dctx"); check_bf16(dqkv, "dqkv");
  TORCH_CHECK(qkv.is_contiguous() && ctx.is_contiguous() && dctx.is_contiguous() && dqkv.is_contiguous(), "attention_bwd needs contiguous tensors");
  TORCH_CHECK(ctx.numel() == a.rows * a.H && dctx.numel() == ctx.numel() && dqkv.numel() == qkv.numel(),
              "attention_bwd: ctx / dctx [rows, H] and dqkv like qkv");
  const int slices = b200::attention_dq_slices(a.S, deterministic);
  TORCH_CHECK(!dq_acc.has_value() || !dq_acc->defined() || dq_acc->numel() >= slices * a.rows * a.H,
              "attention_bwd: dq_acc must hold ", slices, " x [rows, H] floats");
  const bool onepass = b200::attention_bwd_onepass(a.S, force_general);
  if (!onepass) {
    TORCH_CHECK(delta_ws.has_value() && delta_ws->defined() && dq_acc.has_value() && dq_acc->defined(),
                "attention_bwd: the multi-block path (S > 128 or force_general) needs delta_ws and dq_acc");
  }
  if (delta_ws.has_value() && delta_ws->defined())
    TORCH_CHECK(delta_ws->scalar_type() == at::kFloat && delta_ws->numel() >= (int64_t)a.B * heads * a.S,
                "attention_bwd: delta_ws must hold [B, heads, S] floats");
  c10::cuda::CUDAGuard guard(qkv.device());
  b200::attention_bwd(qkv.data_ptr(), a.seqlens, ctx.data_ptr(), dctx.data_ptr(), lse.data_ptr<float>(),
                      dqkv.data_ptr(), opt_f32(delta_ws), opt_f32(dq_acc), a.B, a.S, (int)heads, a.H / (int)heads,
                      (float)scale, mk_seed(seed), (unsigned)stream_id, (float)p_drop,
                      mk_fp8(q8, meta8, e5m2, dqkv.numel()), cur_stream(), a.cu, a.rows, deterministic, force_general);
}

void fused_allreduce_lamb(int64_t rank, int64_t world, bool use_multicast, std::vector<int64_t> grad_ptrs,
                          std::vector<int64_t> param_ptrs, std::vector<int64_t> shadow_ptrs, std::vector<int64_t> pad_ptrs,
                          std::vector<int64_t> flag_ptrs, int64_t grad_mc, int64_t param_mc, int64_t shadow_mc, Tensor m,
                          Tensor v, int64_t numel, int64_t lo, int64_t hi, Tensor chunk_tensor, Tensor chunk_start,
                          Tensor chunk_len, Tensor decay_flag, Tensor stats, Tensor norms, Tensor grid_bar, int64_t epoch,
                          double grad_mul, double lr, double beta1, double beta2, double eps, double weight_decay,
                          double max_grad_norm, int64_t step, bool bias_correction, bool grad_averaging,
                          bool adam_w_mode, bool use_nvlamb, bool push_master, c10::optional<Tensor> prereduced) {
  TORCH_CHECK((int64_t)grad_ptrs.size() == world && world <= 16, "peer pointer lists must have `world` (<= 16) entries");
  TORCH_CHECK(lo % 4 == 0 && hi % 4 == 0 && numel % 4 == 0, "shard bounds must be multiples of 4 elements");
  c10::cuda::CUDAGuard guard(m.device());
  b200::FusedLambLaunch L;
  L.rank = (int)rank; L.world = (int)world; L.use_multicast = use_multicast ? 1 : 0;
  for (int p = 0; p < world; ++p) {
    L.grad_ptrs[p] = reinterpret_cast<const void*>(grad_ptrs[p]);
    L.param_ptrs[p] = reinterpret_cast<const void*>(param_ptrs[p]);
    L.shadow_ptrs[p] = reinterpret_cast<const void*>(shadow_ptrs[p]);
    L.pad_ptrs[p] = reinterpret_cast<const void*>(pad_ptrs[p]);
    L.flag_ptrs[p] = reinterpret_cast<const void*>(flag_ptrs[p]);
  }
  L.grad_mc = reinterpret_cast<void*>(grad_mc); L.param_mc = reinterpret_cast<void*>(param_mc);
  L.shadow_mc = reinterpret_cast<void*>(shadow_mc);
  L.m = m.data_ptr<float>(); L.v = v.data_ptr<float>();
  L.numel = numel; L.lo = lo; L.hi = hi;
  L.chunk_tensor = chunk_tensor.data_ptr<int>(); L.chunk_start = (const long long*)chunk_start.data_ptr<int64_t>();
  L.chunk_len = chunk_len.data_ptr<int>(); L.nchunks = (int)chunk_tensor.numel(); L.ntensors = (int)decay_flag.numel();
  L.decay_flag = decay_flag.data_ptr<int>();
  TORCH_CHECK(stats.numel() >= 16, "fused_allreduce_lamb: stats needs 16 floats ([8..15] carry the in-kernel timeline)");
  L.stats = stats.data_ptr<float>(); L.norms = norms.data_ptr<float>();
  L.grid_bar = reinterpret_cast<unsigned int*>(grid_bar.data_ptr<int>());
  L.epoch = (unsigned int)epoch;
  L.grad_mul = (float)grad_mul; L.lr = (float)lr; L.beta1 = (float)beta1; L.beta2 = (float)beta2; L.eps = (float)eps;
  L.weight_decay = (float)weight_decay; L.max_grad_norm = (float)max_grad_norm; L.step = (int)step;
  L.bias_correction = bias_correction; L.grad_averaging = grad_averaging; L.adam_w_mode = adam_w_mode;
  L.use_nvlamb = use_nvlamb; L.push_master = push_master ? 1 : 0;
  if (prereduced.has_value() && prereduced->defined()) {
    TORCH_CHECK(prereduced->scalar_type() == at::kInt && prereduced->numel() == decay_flag.numel(), "prereduced flags");
    L.prereduced = prereduced->data_ptr<int>();
  }
  b200::fused_allreduce_lamb(L, cur_stream());
}

void nsp_head(Tensor pooled, Tensor w, Tensor bias, Tensor labels, double grad_scale, Tensor loss_out, Tensor dz, Tensor dw,
              Tensor db, bool deterministic) {
  check_bf16(pooled, "pooled"); check_bf16(w, "w"); check_bf16(dz, "dz");
  TORCH_CHECK(pooled.dim() == 2 && pooled.is_contiguous() && dz.is_contiguous() && dz.sizes() == pooled.sizes(), "nsp_head: pooled/dz");
  const int64_t B = pooled.size(0), H = pooled.size(1);
  TORCH_CHECK(w.is_contiguous() && w.size(0) == 2 && w.size(1) == H, "nsp_head: w must be [2, H]");
  TORCH_CHECK(bias.scalar_type() == at::kFloat && bias.numel() == 2 && labels.scalar_type() == at::kLong && labels.numel() == B,
              "nsp_head: bias fp32 [2], labels int64 [B]");
  TORCH_CHECK(dw.scalar_type() == at::kFloat && dw.is_contiguous() && dw.numel() == 2 * H && db.scalar_type() == at::kFloat &&
              db.numel() == 2 && loss_out.scalar_type() == at::kFloat, "nsp_head: fp32 gradient / loss buffers");
  c10::cuda::CUDAGuard guard(pooled.device());
  b200::nsp_head(pooled.data_ptr(), w.data_ptr(), bias.data_ptr<float>(), reinterpret_cast<const long long*>(labels.data_ptr<int64_t>()), (int)B, (int)H,
                 (float)grad_scale, loss_out.data_ptr<float>(), dz.data_ptr(), dw.data_ptr<float>(), db.data_ptr<float>(),
                 cur_stream(), deterministic ? f32_workspace(dw, B * (3 + 2 * H)).data_ptr<float>() : nullptr);
}

inline void check_cls(const Tensor& pooled, const Tensor& w, const Tensor& bias, const char* name) {
  check_bf16(pooled, "pooled"); check_bf16(w, "w");
  TORCH_CHECK(pooled.dim() == 2 && pooled.is_contiguous() && pooled.size(1) % 8 == 0, name,
              ": pooled must be a contiguous [B, H] with H % 8 == 0");
  TORCH_CHECK(w.dim() == 2 && w.is_contiguous() && (w.size(0) == 2 || w.size(0) == 3) && w.size(1) == pooled.size(1), name,
              ": w must be a contiguous [C, H] with C = 2 or 3");
  TORCH_CHECK(bias.is_cuda() && bias.device() == pooled.device() && bias.scalar_type() == at::kFloat && bias.is_contiguous() &&
              bias.numel() == w.size(0), name, ": bias must be a contiguous fp32 CUDA tensor [C]");
}

void cls_head(Tensor pooled, Tensor w, Tensor bias, Tensor labels, double grad_scale, int64_t seed, int64_t stream_id,
              double p_drop, Tensor loss_out, Tensor dz, Tensor dw, Tensor db, bool deterministic) {
  check_cls(pooled, w, bias, "cls_head");
  check_bf16(dz, "dz");
  const int64_t B = pooled.size(0), H = pooled.size(1), C = w.size(0);
  TORCH_CHECK(dz.is_contiguous() && dz.sizes() == pooled.sizes(), "cls_head: dz must be a contiguous tensor of pooled's shape");
  TORCH_CHECK(labels.is_cuda() && labels.device() == pooled.device() && labels.scalar_type() == at::kLong &&
              labels.is_contiguous() && labels.numel() == B, "cls_head: labels must be a contiguous int64 CUDA tensor [B]");
  TORCH_CHECK(dw.is_cuda() && dw.scalar_type() == at::kFloat && dw.is_contiguous() && dw.numel() == C * H &&
              db.is_cuda() && db.scalar_type() == at::kFloat && db.is_contiguous() && db.numel() == C &&
              loss_out.is_cuda() && loss_out.scalar_type() == at::kFloat && loss_out.numel() >= 1,
              "cls_head: fp32 gradient buffers dw [C, H], db [C] and loss");
  TORCH_CHECK(p_drop >= 0.0 && p_drop < 1.0, "cls_head: p_drop must lie in [0, 1)");
  c10::cuda::CUDAGuard guard(pooled.device());
  b200::cls_head(pooled.data_ptr(), w.data_ptr(), bias.data_ptr<float>(),
                 reinterpret_cast<const long long*>(labels.data_ptr<int64_t>()), (int)B, (int)H, (int)C, (float)grad_scale,
                 mk_seed(seed), (unsigned)stream_id, (float)p_drop, loss_out.data_ptr<float>(), dz.data_ptr(),
                 dw.data_ptr<float>(), db.data_ptr<float>(), cur_stream(),
                 deterministic ? f32_workspace(dw, B * (1 + C + C * H)).data_ptr<float>() : nullptr);
}

void cls_logits(Tensor pooled, Tensor w, Tensor bias, Tensor logits) {
  check_cls(pooled, w, bias, "cls_logits");
  const int64_t B = pooled.size(0), C = w.size(0);
  TORCH_CHECK(logits.is_cuda() && logits.device() == pooled.device() && logits.scalar_type() == at::kFloat &&
              logits.is_contiguous() && logits.numel() == B * C, "cls_logits: logits must be a contiguous fp32 [B, C]");
  c10::cuda::CUDAGuard guard(pooled.device());
  b200::cls_logits(pooled.data_ptr(), w.data_ptr(), bias.data_ptr<float>(), (int)B, (int)pooled.size(1), (int)C,
                   logits.data_ptr<float>(), cur_stream());
}

// per-token heads: seq bf16 [M, H] (H % 8 == 0), w bf16 [N, H] with 1 <= N <= 64, fp32 bias [N], all on one device
inline void check_token_head(const Tensor& seq, const Tensor& w, const Tensor& bias, double p_drop, const char* name) {
  check_bf16(seq, "seq"); check_bf16(w, "w");
  TORCH_CHECK(seq.dim() == 2 && seq.is_contiguous() && seq.size(1) % 8 == 0, name,
              ": seq must be a contiguous [M, H] with H % 8 == 0");
  TORCH_CHECK(w.dim() == 2 && w.is_contiguous() && w.size(0) >= 1 && w.size(0) <= 64 && w.size(1) == seq.size(1), name,
              ": w must be a contiguous [N, H] with 1 <= N <= 64");
  TORCH_CHECK(w.device() == seq.device(), name, ": w must be on seq's device");
  TORCH_CHECK(bias.is_cuda() && bias.device() == seq.device() && bias.scalar_type() == at::kFloat && bias.is_contiguous() &&
              bias.numel() == w.size(0), name, ": bias must be a contiguous fp32 CUDA tensor [N] on seq's device");
  TORCH_CHECK(p_drop >= 0.0 && p_drop < 1.0, name, ": p_drop must lie in [0, 1)");
}

inline void check_f32_on(const Tensor& t, const Tensor& like, int64_t numel, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.device() == like.device() && t.scalar_type() == at::kFloat && t.is_contiguous() &&
              t.numel() == numel, name, " must be a contiguous fp32 CUDA tensor of ", numel, " elements on the batch's device");
}

void token_logits(Tensor seq, Tensor w, Tensor bias, double p_drop, int64_t seed, int64_t stream_id, Tensor out) {
  check_token_head(seq, w, bias, p_drop, "token_logits");
  const int64_t M = seq.size(0), H = seq.size(1), N = w.size(0);
  check_f32_on(out, seq, M * N, "token_logits: out");
  c10::cuda::CUDAGuard guard(seq.device());
  b200::token_logits(seq.data_ptr(), w.data_ptr(), bias.data_ptr<float>(), (int)M, (int)H, (int)N, mk_seed(seed),
                     (unsigned)stream_id, (float)p_drop, out.data_ptr<float>(), cur_stream());
}

void token_unpack(Tensor logits, Tensor row_map, Tensor mask, Tensor bias, Tensor out) {
  TORCH_CHECK(logits.is_cuda() && logits.scalar_type() == at::kFloat && logits.is_contiguous() && logits.dim() == 2,
              "token_unpack: logits must be a contiguous fp32 CUDA tensor [T, N]");
  const int64_t N = logits.size(1), P = row_map.numel();
  check_i32(row_map, logits, P, "token_unpack: row_map");
  check_i32(mask, logits, P, "token_unpack: mask");
  check_f32_on(bias, logits, N, "token_unpack: bias");
  check_f32_on(out, logits, P * N, "token_unpack: out");
  c10::cuda::CUDAGuard guard(logits.device());
  b200::token_unpack(logits.data_ptr<float>(), row_map.data_ptr<int>(), mask.data_ptr<int>(), bias.data_ptr<float>(),
                     (int)P, (int)N, out.data_ptr<float>(), cur_stream());
}

// logits fp32 [R, N] (in place), labels int32 [P], mask int32 [P] (optional), row_map int32 [P] (optional; without it
// P == R), loss fp32
void token_ce(Tensor logits, Tensor labels, c10::optional<Tensor> mask, c10::optional<Tensor> row_map, double grad_scale,
              Tensor loss_out, bool deterministic) {
  TORCH_CHECK(logits.is_cuda() && logits.scalar_type() == at::kFloat && logits.is_contiguous() && logits.dim() == 2 &&
              logits.size(1) >= 1 && logits.size(1) <= 64, "token_ce: logits must be a contiguous fp32 CUDA tensor [R, N], "
              "1 <= N <= 64");
  const int64_t R = logits.size(0), N = logits.size(1), P = labels.numel();
  check_i32(labels, logits, P, "token_ce: labels");
  const int* mask_p = nullptr;
  const int* rm_p = nullptr;
  if (mask.has_value() && mask->defined()) {
    check_i32(*mask, logits, P, "token_ce: mask");
    mask_p = mask->data_ptr<int>();
  }
  if (row_map.has_value() && row_map->defined()) {
    check_i32(*row_map, logits, P, "token_ce: row_map");
    rm_p = row_map->data_ptr<int>();
  } else {
    TORCH_CHECK(P == R, "token_ce: without a row_map there must be one label per logits row");
  }
  TORCH_CHECK(loss_out.is_cuda() && loss_out.device() == logits.device() && loss_out.scalar_type() == at::kFloat &&
              loss_out.numel() >= 1, "token_ce: loss_out must be an fp32 CUDA tensor");
  TORCH_CHECK(R < (int64_t(1) << 31) && P < (int64_t(1) << 31), "token_ce: too many rows");
  c10::cuda::CUDAGuard guard(logits.device());
  Tensor idx = at::empty({R + 1}, labels.options());
  Tensor part;
  if (deterministic) part = f32_workspace(logits, b200::token_ce_parts((int)R));
  b200::token_ce(logits.data_ptr<float>(), labels.data_ptr<int>(), mask_p, rm_p, (int)P, (int)R, (int)N, (float)grad_scale,
                 loss_out.data_ptr<float>(), idx.data_ptr<int>(), deterministic ? part.data_ptr<float>() : nullptr,
                 cur_stream());
}

// logits fp32 [B * S, 2] (in place), start / end int32 [B]
void span_ce(Tensor logits, Tensor start, Tensor end, int64_t S, double grad_scale, Tensor loss_out, bool deterministic) {
  TORCH_CHECK(S >= 1, "span_ce: S must be positive");
  TORCH_CHECK(logits.is_cuda() && logits.scalar_type() == at::kFloat && logits.is_contiguous() && logits.dim() == 2 &&
              logits.size(1) == 2 && logits.size(0) % S == 0, "span_ce: logits must be a contiguous fp32 CUDA tensor "
              "[B * S, 2]");
  const int64_t B = logits.size(0) / S;
  check_i32(start, logits, B, "span_ce: start_positions");
  check_i32(end, logits, B, "span_ce: end_positions");
  TORCH_CHECK(loss_out.is_cuda() && loss_out.device() == logits.device() && loss_out.scalar_type() == at::kFloat &&
              loss_out.numel() >= 1, "span_ce: loss_out must be an fp32 CUDA tensor");
  c10::cuda::CUDAGuard guard(logits.device());
  Tensor part;
  if (deterministic) part = f32_workspace(logits, B);
  b200::span_ce(logits.data_ptr<float>(), start.data_ptr<int>(), end.data_ptr<int>(), (int)B, (int)S, (float)grad_scale,
                loss_out.data_ptr<float>(), deterministic ? part.data_ptr<float>() : nullptr, cur_stream());
}

void token_head_bwd(Tensor dlogits, Tensor seq, Tensor w, Tensor dw, Tensor db, double p_drop, int64_t seed,
                    int64_t stream_id, Tensor dseq, bool deterministic) {
  TORCH_CHECK(p_drop >= 0.0 && p_drop < 1.0, "token_head_bwd: p_drop must lie in [0, 1)");
  check_bf16(seq, "seq"); check_bf16(w, "w"); check_bf16(dseq, "dseq");
  TORCH_CHECK(seq.dim() == 2 && seq.is_contiguous() && seq.size(1) % 8 == 0,
              "token_head_bwd: seq must be a contiguous [M, H] with H % 8 == 0");
  const int64_t M = seq.size(0), H = seq.size(1);
  TORCH_CHECK(w.dim() == 2 && w.is_contiguous() && w.size(0) >= 1 && w.size(0) <= 64 && w.size(1) == H &&
              w.device() == seq.device(), "token_head_bwd: w must be a contiguous [N, H] with 1 <= N <= 64 on seq's device");
  const int64_t N = w.size(0);
  check_f32_on(dlogits, seq, M * N, "token_head_bwd: dlogits");
  check_f32_on(dw, seq, N * H, "token_head_bwd: dw");
  check_f32_on(db, seq, N, "token_head_bwd: db");
  TORCH_CHECK(dseq.device() == seq.device() && dseq.is_contiguous() && dseq.sizes() == seq.sizes(),
              "token_head_bwd: dseq must be a contiguous tensor of seq's shape");
  c10::cuda::CUDAGuard guard(seq.device());
  Tensor ws;
  if (deterministic) ws = f32_workspace(dw, (int64_t)b200::token_head_bwd_parts((int)M) * (N * H + N));
  b200::token_head_bwd(dlogits.data_ptr<float>(), seq.data_ptr(), w.data_ptr(), (int)M, (int)H, (int)N, mk_seed(seed),
                       (unsigned)stream_id, (float)p_drop, dseq.data_ptr(), dw.data_ptr<float>(), db.data_ptr<float>(),
                       deterministic ? ws.data_ptr<float>() : nullptr, cur_stream());
}

// evaluation metrics: rows fp32 [R, 3] ({loss, correct, valid} per row), sums fp32 [3] += their column sums (in order)
inline void check_eval_out(const Tensor& rows, const Tensor& sums, int64_t R, const Tensor& like, const char* name) {
  TORCH_CHECK(rows.is_cuda() && rows.device() == like.device() && rows.scalar_type() == at::kFloat && rows.is_contiguous() &&
              rows.numel() == 3 * R, name, ": rows must be a contiguous fp32 CUDA tensor [R, 3]");
  TORCH_CHECK(sums.is_cuda() && sums.device() == like.device() && sums.scalar_type() == at::kFloat && sums.is_contiguous() &&
              sums.numel() == 3, name, ": sums must be a contiguous fp32 CUDA tensor [3]");
}

void mlm_eval(Tensor logits, Tensor targets, Tensor rows, Tensor sums) {
  check_bf16(logits, "logits");
  TORCH_CHECK(logits.dim() == 2 && logits.size(1) % 8 == 0 && logits.stride(0) % 8 == 0, "mlm_eval: logits [R, V], V % 8 == 0");
  const int64_t R = logits.size(0);
  check_i32(targets, logits, R, "mlm_eval: targets");
  check_eval_out(rows, sums, R, logits, "mlm_eval");
  c10::cuda::CUDAGuard guard(logits.device());
  b200::mlm_eval(logits.data_ptr(), (int)logits.stride(0), targets.data_ptr<int>(), (int)R, (int)logits.size(1),
                 rows.data_ptr<float>(), sums.data_ptr<float>(), cur_stream());
}

void nsp_eval(Tensor pooled, Tensor w, Tensor bias, Tensor labels, Tensor rows, Tensor sums) {
  check_bf16(pooled, "pooled"); check_bf16(w, "w");
  TORCH_CHECK(pooled.dim() == 2 && pooled.is_contiguous(), "nsp_eval: pooled must be a contiguous [B, H]");
  const int64_t B = pooled.size(0), H = pooled.size(1);
  TORCH_CHECK(w.is_contiguous() && w.dim() == 2 && w.size(0) == 2 && w.size(1) == H, "nsp_eval: w must be [2, H]");
  TORCH_CHECK(bias.is_cuda() && bias.device() == pooled.device() && bias.scalar_type() == at::kFloat && bias.is_contiguous() &&
              bias.numel() == 2, "nsp_eval: bias must be a contiguous fp32 CUDA tensor [2]");
  TORCH_CHECK(labels.is_cuda() && labels.device() == pooled.device() && labels.scalar_type() == at::kLong &&
              labels.is_contiguous() && labels.numel() == B, "nsp_eval: labels must be a contiguous int64 CUDA tensor [B]");
  check_eval_out(rows, sums, B, pooled, "nsp_eval");
  c10::cuda::CUDAGuard guard(pooled.device());
  b200::nsp_eval(pooled.data_ptr(), w.data_ptr(), bias.data_ptr<float>(),
                 reinterpret_cast<const long long*>(labels.data_ptr<int64_t>()), (int)B, (int)H, rows.data_ptr<float>(),
                 sums.data_ptr<float>(), cur_stream());
}

void peer_allreduce(int64_t rank, int64_t world, bool use_multicast, std::vector<int64_t> buf_ptrs,
                    std::vector<int64_t> flag_ptrs, int64_t buf_mc, Tensor grid_bar, int64_t epoch, int64_t n, double scale) {
  TORCH_CHECK((int64_t)buf_ptrs.size() == world && (int64_t)flag_ptrs.size() == world && world <= 16, "peer pointer lists");
  TORCH_CHECK(n % 4 == 0 && n > 0, "peer_allreduce: element count must be a positive multiple of 4");
  c10::cuda::CUDAGuard guard(grid_bar.device());
  b200::PeerAllreduceLaunch L;
  L.rank = (int)rank; L.world = (int)world; L.use_multicast = use_multicast ? 1 : 0;
  for (int p = 0; p < world; ++p) {
    L.buf_ptrs[p] = reinterpret_cast<const void*>(buf_ptrs[p]);
    L.flag_ptrs[p] = reinterpret_cast<const void*>(flag_ptrs[p]);
  }
  L.buf_mc = reinterpret_cast<void*>(buf_mc);
  L.grid_bar = reinterpret_cast<unsigned int*>(grid_bar.data_ptr<int>());
  L.epoch = (unsigned int)epoch; L.n = n; L.scale = (float)scale;
  b200::peer_allreduce(L, cur_stream());
}

void fp8_quantize(Tensor x, Tensor q, Tensor meta, bool e5m2) {
  check_bf16(x, "x");
  TORCH_CHECK(x.is_contiguous() && q.is_contiguous() && q.is_cuda() && q.element_size() == 1 && q.numel() == x.numel(),
              "fp8_quantize: q must be a contiguous 1-byte tensor of x's size");
  TORCH_CHECK(x.numel() % 16 == 0, "fp8_quantize: numel must be a multiple of 16");
  TORCH_CHECK(meta.scalar_type() == at::kFloat && meta.is_cuda() && meta.numel() >= 4, "fp8 meta record");
  c10::cuda::CUDAGuard guard(x.device());
  b200::fp8_quantize(x.data_ptr(), q.data_ptr(), x.numel(), meta.data_ptr<float>(), e5m2, cur_stream());
}

void fp8_amax(Tensor x, Tensor meta) {
  check_bf16(x, "x");
  TORCH_CHECK(x.is_contiguous() && x.numel() % 8 == 0, "fp8_amax: contiguous, numel % 8 == 0");
  c10::cuda::CUDAGuard guard(x.device());
  b200::fp8_amax(x.data_ptr(), x.numel(), meta.data_ptr<float>(), cur_stream());
}

void fp8_update(Tensor meta, Tensor is_e5m2, double margin_pow2) {
  TORCH_CHECK(meta.scalar_type() == at::kFloat && meta.is_cuda() && meta.is_contiguous() && meta.numel() % 4 == 0, "meta");
  TORCH_CHECK(is_e5m2.scalar_type() == at::kInt && is_e5m2.numel() * 4 == meta.numel(), "is_e5m2 flags");
  c10::cuda::CUDAGuard guard(meta.device());
  b200::fp8_update(meta.data_ptr<float>(), (int)(meta.numel() / 4), is_e5m2.data_ptr<int>(), (float)margin_pow2, cur_stream());
}

// keep bits of the dropout stream (seed, stream) for a [.., N] tensor of `out.numel() * 8` elements (see dropout_mask_kernel)
void dropout_mask(Tensor out, double p_drop, int64_t seed, int64_t stream_id) {
  TORCH_CHECK(out.is_cuda() && out.scalar_type() == at::kByte && out.is_contiguous() && out.numel() % 4 == 0 &&
              reinterpret_cast<uintptr_t>(out.data_ptr()) % 16 == 0, "dropout_mask: uint8, contiguous, numel % 4 == 0");
  c10::cuda::CUDAGuard guard(out.device());
  b200::dropout_mask(out.data_ptr(), out.numel() * 8, mk_seed(seed), (unsigned)stream_id, (float)p_drop, cur_stream());
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("dropout_mask", &dropout_mask);
  m.doc() = "bert_pytorch_b200 sm_90a kernels";
  m.def("gemm", &gemm);
  m.def("gemm_timeline", &gemm_timeline);
  m.def("set_seed_step", &set_seed_step);
  m.def("set_grad_peers", &set_grad_peers);
  m.def("set_grad_push", &set_grad_push);
  m.def("grad_peers_world", &grad_peers_world);
  m.def("peer_allreduce", &peer_allreduce);
  m.def("fp8_quantize", &fp8_quantize);
  m.def("fp8_amax", &fp8_amax);
  m.def("fp8_update", &fp8_update);
  m.def("layer_norm_fwd", &layer_norm_fwd);
  m.def("layer_norm_bwd", &layer_norm_bwd, pybind11::arg("dy"), pybind11::arg("x"), pybind11::arg("mean"),
        pybind11::arg("rstd"), pybind11::arg("gamma"), pybind11::arg("dx"), pybind11::arg("dxd"),
        pybind11::arg("dgamma"), pybind11::arg("dbeta"), pybind11::arg("dbias"), pybind11::arg("workspace"),
        pybind11::arg("p_drop"), pybind11::arg("seed"), pybind11::arg("drop_stream"), pybind11::arg("in_stream"),
        pybind11::arg("q8"), pybind11::arg("meta8"), pybind11::arg("e5m2"), pybind11::arg("keep_mask"),
        pybind11::arg("deterministic") = false);
  m.def("ln_bwd_workspace", &ln_bwd_workspace);
  m.def("colsum", &colsum);
  m.def("ordered_sum", &ordered_sum);
  m.def("gelu_fwd", &gelu_fwd);
  m.def("dgelu_bwd", &dgelu_bwd);
  m.def("embedding_fwd", &embedding_fwd);
  m.def("embedding_bwd_scatter", &embedding_bwd_scatter);
  m.def("mlm_compact", &mlm_compact, pybind11::arg("labels"), pybind11::arg("max_pred"), pybind11::arg("idx"),
        pybind11::arg("tgt"), pybind11::arg("count"), pybind11::arg("row_map") = pybind11::none());
  m.def("pack_tokens", &pack_tokens);
  m.def("gather_rows", &gather_rows);
  m.def("scatter_rows", &scatter_rows);
  m.def("softmax_ce", &softmax_ce);
  m.def("nsp_head", &nsp_head);
  m.def("cls_head", &cls_head);
  m.def("cls_logits", &cls_logits);
  m.def("token_logits", &token_logits);
  m.def("token_unpack", &token_unpack);
  m.def("token_ce", &token_ce);
  m.def("span_ce", &span_ce);
  m.def("token_head_bwd", &token_head_bwd);
  m.def("mlm_eval", &mlm_eval);
  m.def("nsp_eval", &nsp_eval);
  m.def("mt_l2norm", &mt_l2norm);
  m.def("mt_scale", &mt_scale);
  m.def("flat_sumsq", &flat_sumsq);
  m.def("flat_unscale", &flat_unscale);
  m.def("arena_lamb", &arena_lamb);
  m.def("arena_adam", &arena_adam);
  m.def("attention_fwd", &attention_fwd);
  m.def("attention_bwd", &attention_bwd, pybind11::arg("qkv"), pybind11::arg("seqlens"), pybind11::arg("ctx"),
        pybind11::arg("dctx"), pybind11::arg("lse"), pybind11::arg("dqkv"), pybind11::arg("delta_ws"),
        pybind11::arg("dq_acc"), pybind11::arg("heads"), pybind11::arg("scale"), pybind11::arg("p_drop"),
        pybind11::arg("seed"), pybind11::arg("stream_id"), pybind11::arg("q8"), pybind11::arg("meta8"),
        pybind11::arg("e5m2"), pybind11::arg("cu_seqlens"), pybind11::arg("S"),
        pybind11::arg("deterministic") = false, pybind11::arg("force_general") = false);
  m.def("fused_allreduce_lamb", &fused_allreduce_lamb);
}
