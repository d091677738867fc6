// Host launch API of the non-GEMM kernels (raw pointers + stream; the torch binding layer is bindings.cpp).
#pragma once
#include <cuda_runtime.h>

#include "seed.h"

namespace b200 {

// norm_embed.cu
// LayerNorm: H % 8 == 0 and H <= 2048 (the bindings check it)
void layer_norm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* mean, float* rstd, int M,
                    int H, float eps, Fp8Out f8, cudaStream_t st);
int ln_bwd_workspace_floats(int M, int H);
void layer_norm_bwd(const void* dy, const void* x, const float* mean, const float* rstd, const float* gamma, void* dx,
                    void* dxd, float* dgamma, float* dbeta, float* dbias, float* workspace, int M, int H,
                    Seed seed, unsigned int drop_stream, unsigned int in_stream, float p_drop, Fp8Out f8,
                    cudaStream_t st, const uint8_t* keep_mask = nullptr, bool deterministic = false);
void gelu_fwd(const void* x, void* y, long long n, Fp8Out f8, cudaStream_t st);
// dbias_ws (deterministic mode, dgelu_det_workspace_floats(M, N) floats): the blocks' fp32 column sums are stored there
// and added to dbias in order
int dgelu_det_workspace_floats(int M, int N);
void dgelu_bwd(const void* dy, const void* x, void* dx, float* dbias, int M, int N, Fp8Out f8, cudaStream_t st,
               float* dbias_ws = nullptr);
// keep bits ([n_elems / 8] bytes, n_elems % 32 == 0) of the dropout stream (seed, stream): see dropout_mask_kernel
void dropout_mask(void* out, long long n_elems, Seed seed, unsigned int stream, float p_drop, cudaStream_t st);
void colsum_bf16(const void* x, int M, int N, int ld, float* out, cudaStream_t st);

// Deterministic mode: fixed-order forms of the reductions (no atomics; the order of every sum depends on the shapes only).
// out[s * W + w] += sum over the rows r of segment s, in a fixed order, of part[r * W + w]; row_seg (ascending, int32
// [rows]) assigns rows to the nseg segments, or is null for one segment of every row
void ordered_sum(const float* part, int rows, int W, const int* row_seg, int nseg, float* out, cudaStream_t st);
// colsum_bf16 through a workspace of colsum_det_workspace_floats(M, N) floats
int colsum_det_workspace_floats(int M, int N);
void colsum_bf16_det(const void* x, int M, int N, int ld, float* out, float* ws, cudaStream_t st);
// embedding_bwd_scatter by sorting the rows by table row, embedding_det_chunk_rows() rows at a time (chunks added in
// order; table rows * chunk < 2^32); workspaces: sort_ws [chunk], sum_ws [chunk, H].  A null seg means segment 0.
int embedding_det_chunk_rows();
void embedding_bwd_det(const void* de, const int* ids, const int* seg, float* gword, float* gpos, float* gtype,
                       int M, int S, int H, const int* pos_ids, unsigned* sort_ws, float* sum_ws, cudaStream_t st);
void embedding_fwd(const int* ids, const int* seg, const void* word, const void* pos, const void* type,
                   const float* gamma, const float* beta, void* e_out, void* y, float* mean, float* rstd, int M, int S,
                   int H, float eps, Seed seed, unsigned int stream, float p_drop, cudaStream_t st,
                   const int* pos_ids = nullptr);
// pos_ids (int32 [M], optional): position row of every token row; without it the position is row % S
void embedding_bwd_scatter(const void* de, const int* ids, const int* seg, float* gword, float* gpos, float* gtype,
                           int M, int S, int H, int type_rows, cudaStream_t st, const int* pos_ids = nullptr);
// row_map (int32 [B*S], optional): idx gets packed rows, and labels of masked tokens (row_map -1) are dropped
void mlm_compact(const int* labels, int B, int S, int max_pred, int* idx, int* tgt, int* count, cudaStream_t st,
                 const int* row_map = nullptr);
// device packing of a [B, S] batch into T_cap rows + D dummy sequences (see pack_tokens_kernel); B <= pack_tokens_max_batch()
int pack_tokens_max_batch();
void pack_tokens(const int* mask, const int* ids_in, const int* seg_in, int B, int S, int T_cap, int D, int* ids,
                 int* seg, int* pos, int* cu, int* cls, int* row_map, cudaStream_t st);
void gather_rows(const void* src, const int* idx, void* dst, int n, int H, cudaStream_t st);
void scatter_rows(const void* src, const int* idx, void* dst, int n, int H, cudaStream_t st);

// loss.cu
// loss_rows (float [R], deterministic mode): per-row terms, then added to loss_out in row order
void softmax_ce(void* logits, int ld, const int* targets, const int* count, float grad_scale, float* loss_out, int R,
                int V, cudaStream_t st, float* loss_rows = nullptr);

// optim.cu   (dtype codes: 0 = fp32, 1 = bf16, 2 = fp16)
void mt_l2norm(int dtype, const long long* ptrs, const int* chunk_tensor, const long long* chunk_start,
               const int* chunk_len, int nchunks, float* per_tensor_sq, float* total_sq, cudaStream_t st,
               float* chunk_ws = nullptr, int ntensors = 0);   // chunk_ws [nchunks]: deterministic mode
void mt_scale(int in_dtype, int out_dtype, const long long* in_ptrs, const long long* out_ptrs,
              const int* chunk_tensor, const long long* chunk_start, const int* chunk_len, int nchunks,
              const float* scale_dev, float scale_host, int* overflow, cudaStream_t st);
// block_ws [flat_sumsq_det_blocks()]: deterministic mode
int flat_sumsq_det_blocks();
void flat_sumsq(const float* g, long long n, const float* inv_scale, float* stats, float* found_inf, cudaStream_t st,
                float* block_ws = nullptr);
void flat_unscale(float* g, long long n, const float* inv_scale, float* found_inf, cudaStream_t st);
void arena_lamb(float* g, float* p, float* m, float* v, void* shadow, const int* chunk_tensor,
                const long long* chunk_start, const int* chunk_len, int nchunks, const int* decay_flag,
                int ntensors, float* stats, float* norms, const float* inv_scale, const float* found_inf,
                float lr, float beta1, float beta2, float eps, float weight_decay, int step, int bias_correction,
                int grad_averaging, float max_grad_norm, int adam_w_mode, int use_nvlamb, cudaStream_t st,
                float* chunk_ws = nullptr);   // chunk_ws [2 * nchunks]: deterministic mode
void arena_adam(float* g, float* p, float* m, float* v, void* shadow, const int* chunk_tensor,
                const long long* chunk_start, const int* chunk_len, int nchunks, const int* decay_flag,
                const float* inv_scale, const float* found_inf, float lr, float beta1, float beta2, float eps,
                float weight_decay, int step, int bias_correction, int adam_w_mode, cudaStream_t st);

// attention_sm90.cu
// Padded form (cu_seqlens == nullptr): qkv [B*S, 3H], the valid keys of sequence b are a prefix of length seqlens[b]
// (clamped to S; a length <= 0 means all S keys).
// Varlen form: qkv [T, 3H] packed, sequence b is rows cu_seqlens[b] .. cu_seqlens[b + 1] (int32 [B + 1]); S is the
// padded length (grid, lse / delta [B, h, S], dropout counter stride) and seqlens is unused.  No fp8 side outputs.
void attention_fwd(const void* qkv, const int* seqlens, void* ctx, float* lse, int B, int S, int h, int d,
                   float scale, Seed seed, unsigned int stream, float p_drop, Fp8Out f8, cudaStream_t st,
                   const int* cu_seqlens = nullptr, long long T = 0);
void attention_bwd(const void* qkv, const int* seqlens, const void* ctx, const void* dctx, const float* lse,
                   void* dqkv, float* delta_ws, float* dq_acc, int B, int S, int h, int d, float scale,
                   Seed seed, unsigned int stream, float p_drop, Fp8Out f8, cudaStream_t st,
                   const int* cu_seqlens = nullptr, long long T = 0, bool deterministic = false,
                   bool force_general = false);
// Whether attention_bwd runs the one-pass kernel (S <= 128 unless force_general): it needs no delta_ws / dq_acc.  The
// general path computes delta with attn_delta_kernel and reduces dQ through dq_acc.
bool attention_bwd_onepass(int S, bool force_general);
// deterministic attention_bwd: dq_acc holds attention_dq_slices(S) slices of [rows, H]
inline int attention_dq_slices(int S, bool deterministic) { return deterministic && S > 128 ? (S + 127) / 128 : 1; }

// comm.cu -- fused peer-memory all-reduce + partitioned LAMB (one cooperative kernel per step)
struct FusedLambLaunch {
  int rank, world, use_multicast;
  const void* grad_ptrs[16]; const void* param_ptrs[16]; const void* shadow_ptrs[16];
  const void* pad_ptrs[16]; const void* flag_ptrs[16];
  void* grad_mc; void* param_mc; void* shadow_mc;
  float* m; float* v;
  long long numel, lo, hi;
  const int* chunk_tensor; const long long* chunk_start; const int* chunk_len; int nchunks, ntensors;
  const int* decay_flag;
  const int* prereduced = nullptr;   // per tensor flags: already reduced into the owner's arena by the wgrad GEMMs
  float* stats; float* norms; unsigned int* grid_bar;
  unsigned int epoch;
  float grad_mul, lr, beta1, beta2, eps, weight_decay, max_grad_norm;
  int step, bias_correction, grad_averaging, adam_w_mode, use_nvlamb;
  int push_master = 1;   // 0: peers receive only the bf16 shadow; the fp32 master stays with its owner
};
void fused_allreduce_lamb(const FusedLambLaunch& L, cudaStream_t st);

// in-place fp32 all-reduce (sum * scale) of a symmetric staging buffer, one kernel, P2P or NVLS multicast
struct PeerAllreduceLaunch {
  int rank, world, use_multicast;
  const void* buf_ptrs[16]; const void* flag_ptrs[16];
  void* buf_mc;
  unsigned int* grid_bar;
  unsigned int epoch;
  long long n;
  float scale;
};
void peer_allreduce(const PeerAllreduceLaunch& L, cudaStream_t st);

// loss.cu: NSP classifier + CE + backward in one launch
void nsp_head(const void* pooled_bf16, const void* w_bf16, const float* bias, const long long* labels, int B, int H,
              float grad_scale, float* loss_out, void* dz_bf16, float* dw, float* db, cudaStream_t st,
              float* rows_ws = nullptr);   // rows_ws [B * (3 + 2 H)]: deterministic mode

// loss.cu: sequence-classification head (dropout + [B,H] x [H,C] classifier + CE + backward) in one launch, C = 2 or 3;
// pooled / w / dz bf16 with H % 8 == 0, labels int64 (outside [0, C): ignored)
void cls_head(const void* pooled_bf16, const void* w_bf16, const float* bias, const long long* labels, int B, int H, int C,
              float grad_scale, Seed seed, unsigned int stream, float p_drop, float* loss_out, void* dz_bf16, float* dw,
              float* db, cudaStream_t st, float* rows_ws = nullptr);   // rows_ws [B * (1 + C + C H)]: deterministic mode
// evaluation form: fp32 logits [B, C], no dropout
void cls_logits(const void* pooled_bf16, const void* w_bf16, const float* bias, int B, int H, int C, float* logits,
                cudaStream_t st);

// loss.cu: per-token heads (SQuAD, NER).  seq / w bf16 [M, H] / [N, H], H % 8 == 0, 1 <= N <= 64; fp32 logits [M, N].
// Dropout p_drop on the seq elements (Philox stream `stream`, element row * H + i).
void token_logits(const void* seq_bf16, const void* w_bf16, const float* bias, int M, int H, int N, Seed seed,
                  unsigned int stream, float p_drop, float* logits, cudaStream_t st);
// out [P, N] = logits[row_map[p]], or bias where mask[p] == 0
void token_unpack(const float* logits, const int* row_map, const int* mask, const float* bias, int P, int N, float* out,
                  cudaStream_t st);
// in place: logits [R, N] <- d loss / d logits; loss_out += the mean CE over the counted positions p < P (mask[p] == 1
// or no mask, 0 <= labels[p] < N; row row_map[p] or p).  idx_ws int32 [R + 1]; part [token_ce_parts(R)]: deterministic.
int token_ce_parts(int R);
void token_ce(float* logits, const int* labels, const int* mask, const int* row_map, int P, int R, int N,
              float grad_scale, float* loss_out, int* idx_ws, float* part, cudaStream_t st);
// in place on logits [B * S, 2] (start, end): span cross-entropy with positions clamped to [0, S], S ignored.
// part [B]: deterministic mode.
void span_ce(float* logits, const int* start, const int* end, int B, int S, float grad_scale, float* loss_out,
             float* part, cudaStream_t st);
// d_seq bf16 [M, H] = (dlogits . W) * keep / (1 - p); dw [N, H] += dlogits^T . dropout(seq); db [N] += column sums.
// ws [parts * (N H + N)], parts = token_head_bwd_parts(M): deterministic mode (per-partition partials, ordered_sum).
int token_head_bwd_parts(int M);
void token_head_bwd(const float* dlogits, const void* seq_bf16, const void* w_bf16, int M, int H, int N, Seed seed,
                    unsigned int stream, float p_drop, void* dseq_bf16, float* dw, float* db, float* ws, cudaStream_t st);

// loss.cu: evaluation metrics, forward only.  rows [R, 3] receives {loss, correct, valid} of every row ({0, 0, 0} for an
// ignored one); sums [3] += the column sums of rows, added by ordered_sum (no atomics, the same bits in every mode).
// mlm_eval: bf16 logits [R, V] (V % 8 == 0, row stride ld), targets int32 (< 0: ignored).  nsp_eval: pooled bf16 [B, H],
// classifier w bf16 [2, H], fp32 bias [2], int64 labels (< 0: ignored).
void mlm_eval(const void* logits, int ld, const int* targets, int R, int V, float* rows, float* sums, cudaStream_t st);
void nsp_eval(const void* pooled, const void* w, const float* bias, const long long* labels, int B, int H, float* rows,
              float* sums, cudaStream_t st);

// fp8.cu: per-tensor scaled fp8 operand preparation; meta records are {amax, scale, inv_scale, _}
void fp8_quantize(const void* x_bf16, void* q, long long n, float* meta, bool e5m2, cudaStream_t st);
void fp8_amax(const void* x_bf16, long long n, float* meta, cudaStream_t st);
void fp8_update(float* meta, int nrec, const int* is_e5m2, float margin_pow2, cudaStream_t st);

}  // namespace b200
