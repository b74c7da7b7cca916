/*
 * hqq_b200 -- C ABI of the H100 (sm_90a) HQQ quantize-and-infer hot path.
 *
 * This is the drop-in boundary: plain pointers (device memory owned by the caller),
 * sizes and a cudaStream_t passed as void*.  No torch types, no allocation, no host
 * synchronisation inside any call; every call is safe under CUDA-graph capture.
 *
 * Each entry point names the reference (mobiusml/hqq @ e0b1d00) interface it replaces.
 * All functions return 0 on success, a negative HQQ_E_* code otherwise; the message is
 * available (thread-local) through hqq_b200_last_error().
 *
 * Tensor conventions (identical to the reference):
 *   W          [N, K] row-major (nn.Linear.weight), any of f32/f16/bf16
 *   groups     axis=1: W.reshape(-1, gs)  -> R = N*K/gs rows of gs columns, meta [R,1]
 *              axis=0: W.reshape(gs, -1)  -> gs rows of C = N*K/gs columns,  meta [1,C]
 *   W_q        the packed tensor produced by BitPack.pack_* on the grouped matrix:
 *              "slab interleave" along dim 0 -- field f of packed row i holds unpacked row
 *              i + f*step (hqq/core/bitpack.py:24-28,43-52,69-91,115-128);
 *              8/4/2/1 bit -> uint8 (1/2/4/8 fields per byte, most significant first),
 *              3 bit -> int32 (10 fields, bits 29..0, rows zero-padded to a multiple of 10)
 *   scale,zero one value per group, dequantisation form  W ~= (W_q - zero) * scale
 */
#ifndef HQQ_B200_H
#define HQQ_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HQQ_B200_ABI_VERSION 2

/* element types */
enum {
  HQQ_F32 = 0,
  HQQ_F16 = 1,
  HQQ_BF16 = 2,
  HQQ_U8 = 3,
  HQQ_I32 = 4,
  HQQ_I64 = 5
};

/* error codes */
enum {
  HQQ_OK = 0,
  HQQ_E_INVALID = -1,     /* bad argument (shape, dtype, alignment, null pointer)        */
  HQQ_E_UNSUPPORTED = -2, /* valid request outside what this build implements            */
  HQQ_E_WORKSPACE = -3,   /* workspace too small                                         */
  HQQ_E_CUDA = -4         /* CUDA launch/driver error (message carries cudaGetErrorString) */
};

int hqq_b200_abi_version(void);
const char* hqq_b200_last_error(void);

/* ---------------------------------------------------------------------------------------
 * BitPack.pack_{8,4,2,1}bit_u8 / pack_3bit_32            hqq/core/bitpack.py:14-15,24-28,43-52,69-91,115-128
 *   in : [rows, cols] of in_dtype (any HQQ_* type; values are the integer levels)
 *   out: uint8 [rows*nbits/8, cols]   (nbits 8/4/2/1; rows must be a multiple of 8/nbits)
 *        int32 [ceil(rows/10), cols]  (nbits 3)
 * ------------------------------------------------------------------------------------- */
int hqq_b200_pack(int nbits, const void* in, int in_dtype, void* out,
                  int64_t rows, int64_t cols, void* stream);

/* BitPack.unpack_* and hqq_aten.unpack_{4,2,1}bit_u8 / unpack_3bit_32
 *   hqq/core/bitpack.py:18-19,31-38,55-64,95-110,131-144 ; hqq/kernels/hqq_aten_cuda.cpp:59-71
 *   in : packed [packed_rows, cols] (uint8, or int32 for nbits 3)
 *   out: out_dtype [packed_rows * fields, cols]  (fields = 8/nbits, or 10 for 3 bit:
 *        like the reference the 3-bit output keeps the padded rows; callers slice)      */
int hqq_b200_unpack(int nbits, const void* in, void* out, int out_dtype,
                    int64_t packed_rows, int64_t cols, void* stream);

/* Quantizer.dequantize and hqq_aten.dequantize (which only handles axis 0)
 *   hqq/core/quantize.py:184-199 ; hqq/kernels/hqq_aten_cuda.cpp:32-54
 *   out[N,K] = ((unpack(W_q) as dtype) - zero) * scale, two roundings in `dtype`,
 *   scale/zero given in `dtype` (as stored in HQQLinear.meta after .cuda()).
 *   W_q may be the float "view" of the packed bytes (view_as_float): same pointer.   */
int hqq_b200_dequantize(const void* W_q, const void* scale, const void* zero, void* out,
                        int64_t N, int64_t K, int group_size, int nbits, int axis,
                        int dtype, void* stream);

/* Quantizer.quantize incl. Quantizer.optimize_weights (= optimize_weights_proximal_legacy)
 * and BitPack.pack      hqq/core/quantize.py:76-180 ; hqq/core/optimize.py:96-108,201-255
 *   W        [N,K] of src_dtype (f32/f16/bf16), device memory
 *   optimize 0: W_q = round(W*s+z) only ; 1: proximal solver (lp_norm, beta, iters; the
 *            reference defaults are 0.7, 10.0, 20) with the reference's whole-tensor early stop
 *   W_q_out  packed as above; scale_out/zero_out float32, one per group (scale is the
 *            dequantisation scale, i.e. already inverted, quantize.py:154)
 *   info_out optional int32[4] device: {iterations executed, selected zero slot, 0, 0}
 *   err_out  optional float[iters] device: whole-tensor mean |W - W_r| per iteration
 *   workspace: hqq_b200_quantize_workspace_bytes() bytes of device scratch              */
size_t hqq_b200_quantize_workspace_bytes(int64_t N, int64_t K, int group_size, int nbits,
                                         int axis, int iters);
int hqq_b200_quantize(const void* W, int src_dtype, int64_t N, int64_t K,
                      int group_size, int nbits, int axis, int round_zero, int optimize,
                      float lp_norm, float beta, int iters,
                      void* W_q_out, float* scale_out, float* zero_out,
                      int32_t* info_out, float* err_out,
                      void* workspace, size_t workspace_bytes, void* stream);

/* Quantizer.optimize_weights seam (hqq/core/quantize.py:38,137-145): same as hqq_b200_quantize but
 *   inv_scale_init / zero_init  optional float32 [groups]: the caller's initial inverse scale and zero
 *                               (what optimize_weights_proximal receives as `scale`, `zero`); NULL = min/max init
 *   max_level                   upper clamp (min_max[1]); lower clamp is 0 as in the reference
 * With nbits = 8 the output is one level per byte, i.e. the unpacked W_q the seam returns.            */
int hqq_b200_quantize_ex(const void* W, int src_dtype, int64_t N, int64_t K,
                         int group_size, int nbits, int max_level, int axis, int round_zero, int optimize,
                         float lp_norm, float beta, int iters,
                         const float* inv_scale_init, const float* zero_init,
                         void* W_q_out, float* scale_out, float* zero_out,
                         int32_t* info_out, float* err_out,
                         void* workspace, size_t workspace_bytes, void* stream);

/* Quantising a layer whose rows / groups are spread over several GPUs (tensor-parallel shards) with the reference's result:
 * the groups are independent except for the early stop, which compares the mean |W - W_r| of the WHOLE tensor per iteration
 * (hqq/core/optimize.py:239-247).  _begin runs init + solver on this shard and writes its `iters` float64 error sums to
 * err_sums_out (device memory; the zero-point trajectories stay in `workspace`); the caller adds the shards' sums (one all-reduce of
 * iters x 8 bytes) and calls _finish with the global sums and the global element count: early stop, round, pack -- every shard
 * then holds exactly the levels / scale / zero of the unsharded quantisation.  Same workspace (hqq_b200_quantize_workspace_bytes)
 * for both calls, untouched in between.                                                                                        */
int hqq_b200_quantize_shard_begin(const void* W, int src_dtype, int64_t N, int64_t K, int group_size, int nbits, int axis,
                                  int round_zero, float lp_norm, float beta, int iters, double* err_sums_out,
                                  void* workspace, size_t workspace_bytes, void* stream);
int hqq_b200_quantize_shard_finish(const void* W, int src_dtype, int64_t N, int64_t K, int group_size, int nbits, int axis,
                                   int round_zero, float lp_norm, float beta, int iters, const double* err_sums,
                                   int64_t total_elements, void* W_q_out, float* scale_out, float* zero_out,
                                   int32_t* info_out, float* err_out, void* workspace, size_t workspace_bytes, void* stream);

/* HQQLinear.forward under HQQBackend.PYTORCH (forward_pytorch / forward_pytorch_backprop),
 * i.e. y = x @ dequantize(W_q).T + bias, as ONE fused unpack->dequant->MMA kernel.
 *   hqq/core/quantize.py:880-898 ; semantic template hqq/kernels/hqq_aten_torch.cpp:79-107
 *   x [M,K], y [M,N], bias [N] or NULL, scale/zero [N*K/gs], all of `dtype` (f16/bf16)
 *   Routes (hqq_b200_linear_fwd_route): 1 = small-M weight-streaming kernel (M <= 16; M <= 32 on matrices of up to 2^24 weights),
 *   2 = fused wgmma GEMM -- both axis 1,
 *   nbits 8/4/2/1, group_size 64/128, K % 256 == 0 -- and 3 = everything else hqq_b200_dequantize accepts (3-bit, axis 0, other
 *   group sizes, ragged K): the dequantize kernel writes W_r into `workspace`, the dense wgmma GEMM multiplies.  Returns
 *   HQQ_E_UNSUPPORTED where none applies (fp32 compute).
 *   workspace: hqq_b200_linear_fwd_workspace_bytes() bytes, 256-byte aligned scratch owned by the caller: 0 for route 1
 *   (split-K partials of the small-M kernel meet in shared memory); route 2: 0 unless the problem has so few output tiles
 *   (roughly M <= 512 on a 4096-row matrix) that the kernel splits K over CTAs -- then the fp32 partial tiles, summed in slice
 *   order by a second pass (deterministic); route 3: N*K*sizeof(dtype) for W_r.  Contents on entry are irrelevant.           */
size_t hqq_b200_linear_fwd_workspace_bytes(int64_t M, int64_t N, int64_t K, int group_size,
                                           int nbits, int axis, int dtype);
int hqq_b200_linear_fwd(const void* x, const void* W_q, const void* scale, const void* zero,
                        const void* bias, void* y, int64_t M, int64_t N, int64_t K,
                        int group_size, int nbits, int axis, int dtype,
                        void* workspace, size_t workspace_bytes, void* stream);

/* y[M,N] = x[M,K] @ W[N,K]^T (+ bias) for an ordinary fp16/bf16 matrix W: the persistent wgmma kernel of route 2 with both
 * operands on TMA.  Used by route 3 and by the backward pass of HQQMatmulNoCacheMul (grad_out @ W_r, hqq/core/quantize.py:322-352:
 * W = W_r^T).  K % 8 == 0 (16-byte row pitch), x / W 16-byte aligned.                                                        */
int hqq_b200_dense_gemm(const void* x, const void* W, const void* bias, void* y, int64_t M, int64_t N, int64_t K,
                        int dtype, void* stream);

/* Log-probabilities over an lm_head shard without materialising the logits (prompt scoring, perplexity).  x [M, K] and the shard
 * W [N, K] (vocabulary rows index_offset .. index_offset + N - 1) of `dtype` (f16/bf16); targets int64 [M]: a vocabulary index or -1.
 *   l[m][v] = T(sum_k x[m][k] * W[v][k])   -- fp32 accumulation, one rounding to T: what hqq_b200_dense_gemm stores (no bias)
 *   per vocabulary tile j (rows 128 j .. 128 j + 127 that are < N) and position m, in fp32:
 *     m_j = max_v l[m][v],  s_j = sum_v expf(l[m][v] - m_j)                      (the wgmma kernel's epilogue; logits never stored)
 *   then over the tiles, in tile order:  M = max_j m_j,  S = sum_j s_j * expf(m_j - M),  lse[m] = M + logf(S)      (fp32)
 *   tgt[m] = l[m][targets[m] - index_offset] when that row lies in the shard, else -inf                          (fp32)
 * log p(target | x) = tgt - lse on one shard; shards merge their lse the same way (max, then sum of exp in rank order).  The
 * value of a position depends on its x row alone: not on M, the other rows or the schedule.  No atomics.
 * workspace: hqq_b200_lm_logprob_workspace_bytes(M, N) = ceil(N / 128) * M * 8 bytes (8-byte aligned) of tile partials; the
 * caller bounds M per call (4096 rows at vocabulary 128256: 33 MB).  HQQ_E_INVALID for null or unaligned pointers (x, W 16 bytes;
 * targets, workspace 8; lse, tgt 4) or K % 8 != 0; HQQ_E_UNSUPPORTED outside f16 / bf16.                                      */
size_t hqq_b200_lm_logprob_workspace_bytes(int64_t M, int64_t N);
int hqq_b200_lm_logprob(const void* x, const void* W, const int64_t* targets, float* lse, float* tgt, void* workspace, int64_t M,
                        int64_t N, int64_t K, int64_t index_offset, int dtype, void* stream);

/* Several HQQLinear layers that consume the SAME activation (q/k/v, gate/up) in one launch of the small-M kernel:
 * the 16-row tiles of all `count` (<= 4) matrices form one stream-K work list, so small matrices no longer pay a
 * launch each.  Arrays hold `count` device pointers / sizes; bias may be NULL or hold NULL entries; all matrices share
 * K, group_size, nbits, dtype.  Same math per layer as hqq_b200_linear_fwd (quantize.py:880-898).
 * Workspace: hqq_b200_linear_fwd_workspace_bytes(M, ...) bytes (currently 0).                                         */
int hqq_b200_linear_fwd_multi(const void* x, int count, const void* const* W_q, const void* const* scale,
                              const void* const* zero, const void* const* bias, void* const* y, const int64_t* N,
                              int64_t M, int64_t K, int group_size, int nbits, int axis, int dtype,
                              void* workspace, size_t workspace_bytes, void* stream);

/* Which kernels hqq_b200_linear_fwd would use: 0 none (unsupported), 1 small-M mma.sync weight-streaming kernel,
 * 2 fused wgmma/TMA GEMM, 3 dequantize kernel + dense wgmma GEMM.                                         */
int hqq_b200_linear_fwd_route(int64_t M, int64_t N, int64_t K, int group_size, int nbits,
                              int axis, int dtype);

/* ---------------------------------------------------------------------------------------
 * Decode-harness glue (SURVEY.md 8 f-2, the CALLER of HQQLinear.forward -- not part of the
 * hot path and with no counterpart inside hqq/core): the handful of tiny batch-1 ops between
 * the fused linears of a Llama-style block, so that one decoded token is 8 launches per
 * block (hqq/utils/generation_hf.py:270-289 leaves these to HF transformers + torch.compile).
 * fp16/bf16 only; every kernel is launched with programmatic dependent launch.
 * ------------------------------------------------------------------------------------- */
/* One-token linear(s) with the activation prologue folded into the kernel's x staging, so a block needs 5 launches:
 *   x_op 0: y_i = x @ W_i^T                               (== hqq_b200_linear_fwd_multi at M = 1)
 *   x_op 1: t = x + x2 (x2 may be NULL); h_out = t (may be NULL); y_i = (rmsnorm(t, eps) * x_weight) @ W_i^T
 *   x_op 2: y_i = (silu(x) * x2) @ W_i^T
 *   x_op | HQQ_YOP_SILU_MUL_PAIR (count == 2, N[0] == N[1], nbits < 8): y[0] = silu(x' @ W_0^T) * (x' @ W_1^T) with both
 *     products rounded to `dtype` first (the MLP's act(gate) * up, models/llama semantics); y[1] is not written.
 * Roundings follow the stand-alone glue kernels (every intermediate is rounded to `dtype`).  h_out must not alias x. */
#define HQQ_YOP_SILU_MUL_PAIR 16
int hqq_b200_decode_linear_fwd(const void* x, int x_op, const void* x2, const void* x_weight, void* h_out, float eps,
                               int count, const void* const* W_q, const void* const* scale, const void* const* zero,
                               const void* const* bias, void* const* y, const int64_t* N, int64_t K,
                               int group_size, int nbits, int dtype, void* stream);
/* Chained / tensor-parallel variant.  Kernels exchange one-token activations as 32-bit words {tag16 : value16} ("LL" protocol:
 * a consumer polls until the tag matches, so there are no fences, flags or collective launches):
 *   - SURVEY.md 8e, row-parallel o_proj / down_proj: with peer_data the producer scatters its [1, hidden] partial to
 *     peer_data[dst][parity][rank][n] on all `tp` ranks over NVLink peer memory; the consumer (x_op 1, red_data) sums the `tp`
 *     partials into the residual delta.  This IS the all-reduce, fused into the kernels that produce and consume it.
 *   - on one GPU the same words chain kernels: y_tagged[i] keeps a tagged copy [2][N_i] of output i, x_tagged / x2_tagged feed
 *     the SiLU*mul prologue, red_data with tp == 1 feeds the residual delta.
 * tag = low 16 bits of the exchange number (*step_ctr * x_per_step + x_index), parity = its bit 0.  step_ctr is an int in local
 * device memory that hqq_b200_glue_add_rmsnorm_tp bumps once per token, so a captured CUDA graph can be replayed.  Buffers
 * start filled with 0xFF.  All other fields as in hqq_b200_decode_linear_fwd.                                                  */
typedef struct hqq_b200_decode_desc {
  const void* x; int x_op; const void* x2; const void* x_weight; void* h_out; float eps;
  int count; const void* const* W_q; const void* const* scale; const void* const* zero; const void* const* bias;
  void* const* y; const int64_t* N; int64_t K; int group_size; int nbits; int dtype;
  int tp; int rank;
  void* const* peer_data;   /* `tp` peer-mapped pointers, each [2][tp][N] uint32, or NULL */
  const void* red_data;     /* local [2][tp][K] uint32 to reduce into the delta (x_op 1), or NULL */
  void* const* y_tagged;    /* `count` local [2][N_i] uint32 buffers, or NULL */
  const void* x_tagged;     /* local [2][K] uint32 (x_op 2), or NULL */
  const void* x2_tagged;
  const int* step_ctr; int x_index; int x_per_step;
} hqq_b200_decode_desc;
int hqq_b200_decode_linear_fwd_desc(const hqq_b200_decode_desc* desc, void* stream);
/* final-norm consumer of the same exchange: h += sum_r red_data[parity][r]; y = rmsnorm(h) * weight; ++*step_ctr */
int hqq_b200_glue_add_rmsnorm_tp(void* h, const void* red_data, int* step_ctr, int x_index, int x_per_step, int tp,
                                 const void* weight, void* y, int H, float eps, int dtype, void* stream);
/* h += delta (delta may be NULL);  y = rmsnorm(h) * weight          (one token, H <= 8192) */
int hqq_b200_glue_add_rmsnorm(void* h, const void* delta, const void* weight, void* y,
                              int H, float eps, int dtype, void* stream);
/* the same on `rows` sequences decoding in lock-step: h, delta, y are [rows, H] row-major, one CTA per row */
int hqq_b200_glue_add_rmsnorm_rows(void* h, const void* delta, const void* weight, void* y,
                                   int rows, int H, float eps, int dtype, void* stream);
/* y = silu(gate) * up */
int hqq_b200_glue_silu_mul(const void* gate, const void* up, void* y, int n, int dtype, void* stream);
/* RoPE(q,k at *pos) + KV-cache append + one-token GQA attention over cache[0..*pos];
 * caches [n_kv_heads, cache_len, head_dim], cos/sin tables [cache_len, head_dim], pos on device.
 * *pos and cache rows [0, *pos) are read BEFORE the programmatic-dependency wait (L2 prefetch under the previous kernel's
 * tail): they must have been written by an earlier, completed launch, not by the kernel directly in front of this one. */
int hqq_b200_glue_rope_attn_decode(const void* q, const void* k, const void* v,
                                   const void* cos_table, const void* sin_table,
                                   void* k_cache, void* v_cache, const int64_t* pos, void* out,
                                   int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                   int dtype, void* stream);
/* the same for `batch` sequences at the SAME position *pos: q / out [batch, n_q_heads*head_dim], k / v [batch, n_kv_heads*head_dim],
 * caches [batch, n_kv_heads, cache_len, head_dim]; grid = (n_q_heads, batch) */
int hqq_b200_glue_rope_attn_decode_batch(const void* q, const void* k, const void* v,
                                         const void* cos_table, const void* sin_table,
                                         void* k_cache, void* v_cache, const int64_t* pos, void* out,
                                         int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                         int batch, int dtype, void* stream);
/* Long-context form of hqq_b200_glue_rope_attn_decode_batch (same layouts, same RoPE and cache rows bit for bit, cache_len up to
 * 131072 instead of 8192; the decode harness uses it above 8192).  The cached positions are split into S contiguous chunks,
 * S = max(1, min(SMs / n_kv_heads, ceil(cache_len / 16))), one CTA per (chunk, kv head, sequence) serving all query heads of its
 * group with tensor-core products; the last CTA of each (sequence, kv head) combines the partials in chunk order.  S does not
 * depend on batch: a sequence of a batch gets bit for bit what it gets alone.  Like split-K, the result is a function of
 * (inputs, *pos, SM count).
 * workspace: hqq_b200_glue_rope_attn_decode_split_workspace_bytes(...) bytes on the device, 4-byte aligned: fp32 partials
 * [batch, n_kv_heads, S, n_q_heads / n_kv_heads, 2 + head_dim] (laid out for S = max(1, SMs / n_kv_heads)) followed by
 * batch * n_kv_heads uint32 tickets.  The caller zeroes it once after allocating it; every launch leaves the tickets at zero, so a
 * captured graph replays without a memset.  One workspace serves any number of launches in stream order.
 * Needs head_dim 128 and n_q_heads / n_kv_heads <= 8.  The precondition on *pos and cache rows [0, *pos) of
 * hqq_b200_glue_rope_attn_decode applies. */
int hqq_b200_glue_rope_attn_decode_split(const void* q, const void* k, const void* v,
                                         const void* cos_table, const void* sin_table,
                                         void* k_cache, void* v_cache, const int64_t* pos, void* out, void* workspace,
                                         int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                         int batch, int dtype, void* stream);
/* Workspace bytes of hqq_b200_glue_rope_attn_decode_split on the current device (0 for invalid head counts).  The same
 * workspace serves hqq_b200_glue_rope_attn_decode_split_kv8. */
size_t hqq_b200_glue_rope_attn_decode_split_workspace_bytes(int n_q_heads, int n_kv_heads, int head_dim, int batch);
/* hqq_b200_glue_rope_attn_decode_split over an 8-bit HQQ KV cache: the same grid, split count, merge order, workspace and RoPE
 * rounding.  A cache row of one kv head is Quantizer.quantize(row, nbits=8, group_size, axis=1, optimize=False) with the meta cast to
 * dtype: k_q / v_q uint8 [batch, n_kv_heads, cache_len, head_dim] (16-byte aligned), k_scale / k_zero / v_scale / v_zero
 * [batch, n_kv_heads, cache_len, head_dim / group_size] in dtype, and the attended row is (q - zero) * scale with one rounding to
 * dtype per operation, as hqq_b200_dequantize computes it.  Row *pos is quantised from rope(k) and v in this launch and written
 * there; every attended row, row *pos included, is the dequantised row, so the output is attention over exactly the cache the next
 * step reads.  group_size 64 or 128; the other limits and the precondition on *pos are those of hqq_b200_glue_rope_attn_decode_split. */
int hqq_b200_glue_rope_attn_decode_split_kv8(const void* q, const void* k, const void* v,
                                             const void* cos_table, const void* sin_table,
                                             void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                             const int64_t* pos, void* out, void* workspace,
                                             int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int group_size,
                                             int batch, int dtype, void* stream);
/* Prompt prefill, step 1: a chunk of T positions pos0 .. pos0 + T - 1 of `batch` sequences.  q [batch*T, n_q_heads*head_dim],
 * k / v [batch*T, n_kv_heads*head_dim] as the q/k/v linears produce them (token row b*T + t); caches [batch, n_kv_heads, cache_len,
 * head_dim].  Writes rope(k) and v into cache rows [pos0, pos0 + T) and rope(q) into q_out (same layout as q).  RoPE rounds as
 * hqq_b200_glue_rope_attn_decode does (each product and the sum rounded to dtype), so a cache row written here is bit for bit the
 * row a decode step writes at the same position from the same k and v.
 * Needs head_dim 128, n_q_heads % n_kv_heads == 0, n_q_heads / n_kv_heads <= 8, 1 <= T, pos0 + T <= cache_len <= 131072,
 * batch <= 65535. */
int hqq_b200_glue_rope_append_rows(const void* q, const void* k, const void* v,
                                   const void* cos_table, const void* sin_table,
                                   void* k_cache, void* v_cache, void* q_out, int pos0, int T,
                                   int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                   int batch, int dtype, void* stream);
/* hqq_b200_glue_rope_append_rows for an 8-bit cache (see hqq_b200_glue_rope_attn_decode_split_kv8 for the format): q_out as
 * hqq_b200_glue_rope_append_rows writes it, bit for bit; rope(k) and v of rows [pos0, pos0 + T) quantised into the levels and meta
 * exactly as the decode kernel quantises row *pos; and their dequantised rows written to k_stage / v_stage
 * [batch, n_kv_heads, cache_len, head_dim] in dtype at the same rows, for hqq_b200_glue_attn_prefill to read.  group_size 64 or 128;
 * other limits as hqq_b200_glue_rope_append_rows. */
int hqq_b200_glue_rope_append_rows_kv8(const void* q, const void* k, const void* v,
                                       const void* cos_table, const void* sin_table,
                                       void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                       void* k_stage, void* v_stage, void* q_out, int pos0, int T,
                                       int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int group_size,
                                       int batch, int dtype, void* stream);
/* Prompt prefill, step 2: causal GQA attention of the chunk's queries over the cache.  Query t (row b*T + t of q_rot, rotated as
 * hqq_b200_glue_rope_append_rows leaves it) sits at position pos0 + t and attends to cache rows 0 .. pos0 + t; out has the layout
 * of q_rot, ready for o_proj.  Cache rows at or past pos0 + T are never read.  A row's output depends only on its q row and cache
 * rows 0 .. pos0 + t: it is bit for bit the same whatever pos0 / T chunking or batch produced it.  No workspace, no atomics.
 * Same argument limits as hqq_b200_glue_rope_append_rows. */
int hqq_b200_glue_attn_prefill(const void* q_rot, const void* k_cache, const void* v_cache, void* out,
                               int pos0, int T, int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                               int batch, int dtype, void* stream);
/* Ragged batches: the three decode attention entry points with one position per sequence.  Same arguments, layouts, split count,
 * workspace (hqq_b200_glue_rope_attn_decode_split_workspace_bytes) and limits as hqq_b200_glue_rope_attn_decode_batch /
 * _split / _split_kv8, except that pos is a device int64 [batch] and sequence b decodes at position pos[b]: its RoPE row, its
 * cache row written, its attended rows 0 .. pos[b] and, for the split forms, its chunking all follow pos[b].  Sequence b's output
 * and cache rows are bit for bit those of the lock-step entry point called with batch 1 on sequence b's slices at position pos[b].
 * Every pos[b] and cache rows [0, pos[b]) of every sequence are read BEFORE the programmatic-dependency wait: they must have been
 * written by an earlier, completed launch, not by the kernel directly in front of this one. */
int hqq_b200_glue_rope_attn_decode_batch_seqpos(const void* q, const void* k, const void* v,
                                                const void* cos_table, const void* sin_table,
                                                void* k_cache, void* v_cache, const int64_t* pos, void* out,
                                                int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                                int batch, int dtype, void* stream);
int hqq_b200_glue_rope_attn_decode_split_seqpos(const void* q, const void* k, const void* v,
                                                const void* cos_table, const void* sin_table,
                                                void* k_cache, void* v_cache, const int64_t* pos, void* out, void* workspace,
                                                int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                                int batch, int dtype, void* stream);
int hqq_b200_glue_rope_attn_decode_split_kv8_seqpos(const void* q, const void* k, const void* v,
                                                    const void* cos_table, const void* sin_table,
                                                    void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                                    const int64_t* pos, void* out, void* workspace,
                                                    int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int group_size,
                                                    int batch, int dtype, void* stream);
/* Variable-length prefill: the three prefill entry points with prompts of different lengths in one launch.  pos0 and n_tok are
 * HOST arrays of `batch` entries: slot b contributes n_tok[b] >= 0 rows at positions pos0[b] .. pos0[b] + n_tok[b] - 1.  Token rows
 * of q, k, v, q_out and out are packed in slot order: slot b's rows start at row n_tok[0] + ... + n_tok[b - 1] (with equal lengths
 * T this is the b*T + t layout of the fixed-length calls).  A slot with n_tok[b] == 0 is neither read nor written.  Every row, cache
 * row and attention row is bit for bit what the fixed-length entry point gives when called with batch 1 on that slot alone.
 * Needs 1 <= batch <= 256, 0 <= pos0[b], pos0[b] + n_tok[b] <= cache_len, 1 <= n_tok[0] + ... + n_tok[batch - 1] <= 65535;
 * the other limits are those of the fixed-length calls. */
int hqq_b200_glue_rope_append_rows_varlen(const void* q, const void* k, const void* v,
                                          const void* cos_table, const void* sin_table,
                                          void* k_cache, void* v_cache, void* q_out, const int* pos0, const int* n_tok,
                                          int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                          int batch, int dtype, void* stream);
int hqq_b200_glue_rope_append_rows_kv8_varlen(const void* q, const void* k, const void* v,
                                              const void* cos_table, const void* sin_table,
                                              void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                              void* k_stage, void* v_stage, void* q_out, const int* pos0, const int* n_tok,
                                              int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int group_size,
                                              int batch, int dtype, void* stream);
int hqq_b200_glue_attn_prefill_varlen(const void* q_rot, const void* k_cache, const void* v_cache, void* out,
                                      const int* pos0, const int* n_tok, int n_q_heads, int n_kv_heads, int cache_len,
                                      int head_dim, int batch, int dtype, void* stream);
/* Paged KV cache: the _seqpos decode and _varlen prefill entry points over page pools.  A page holds 64 positions of one sequence
 * for every kv head: the pools are [n_pages + 1, n_kv_heads, 64, head_dim] (fp16 / bf16 rows, or uint8 levels) and, for the 8-bit
 * cache, [n_pages + 1, n_kv_heads, 64, head_dim / group_size] meta.  table is a device int32 [batch, cache_len / 64]: position p of
 * sequence b, kv head h lives at pool row (table[b][p / 64] * n_kv_heads + h) * 64 + p % 64.  Every entry must lie in
 * [0, n_pages]; page n_pages is conventionally the sink the unbacked entries point at.  Nothing else differs from the contiguous
 * entry points: a sequence's output, tickets and written rows are bit for bit theirs on the cache gathered through the table.
 * Needs cache_len % 64 == 0 and n_pages >= 1.  The table entries, like pos, are read BEFORE the programmatic-dependency wait: they
 * must have been written by an earlier, completed launch, not by the kernel directly in front of this one.  The 8-bit prefill keeps
 * its staging pair [batch, n_kv_heads, cache_len, head_dim]; hqq_b200_glue_kv8_stage_paged refills staging rows [0, pos0[b]) of
 * every slot with n_tok[b] > 0 from the pools, bit for bit the rows hqq_b200_dequantize gives. */
int hqq_b200_glue_rope_attn_decode_batch_paged(const void* q, const void* k, const void* v,
                                               const void* cos_table, const void* sin_table,
                                               void* k_pool, void* v_pool, const int* table, const int64_t* pos, void* out,
                                               int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                               int batch, int n_pages, int dtype, void* stream);
int hqq_b200_glue_rope_attn_decode_split_paged(const void* q, const void* k, const void* v,
                                               const void* cos_table, const void* sin_table,
                                               void* k_pool, void* v_pool, const int* table, const int64_t* pos, void* out, void* workspace,
                                               int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                               int batch, int n_pages, int dtype, void* stream);
int hqq_b200_glue_rope_attn_decode_split_kv8_paged(const void* q, const void* k, const void* v,
                                                   const void* cos_table, const void* sin_table,
                                                   void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                                   const int* table, const int64_t* pos, void* out, void* workspace,
                                                   int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int group_size,
                                                   int batch, int n_pages, int dtype, void* stream);
int hqq_b200_glue_rope_append_rows_paged(const void* q, const void* k, const void* v,
                                         const void* cos_table, const void* sin_table,
                                         void* k_pool, void* v_pool, const int* table, void* q_out, const int* pos0, const int* n_tok,
                                         int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                         int batch, int n_pages, int dtype, void* stream);
int hqq_b200_glue_rope_append_rows_kv8_paged(const void* q, const void* k, const void* v,
                                             const void* cos_table, const void* sin_table,
                                             void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                             const int* table, void* k_stage, void* v_stage, void* q_out, const int* pos0, const int* n_tok,
                                             int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int group_size,
                                             int batch, int n_pages, int dtype, void* stream);
int hqq_b200_glue_kv8_stage_paged(const void* k_q, const void* k_scale, const void* k_zero,
                                  const void* v_q, const void* v_scale, const void* v_zero, const int* table,
                                  void* k_stage, void* v_stage, const int* pos0, const int* n_tok,
                                  int n_kv_heads, int cache_len, int head_dim, int group_size,
                                  int batch, int n_pages, int dtype, void* stream);
int hqq_b200_glue_attn_prefill_paged(const void* q_rot, const void* k_pool, const void* v_pool, const int* table, void* out,
                                     const int* pos0, const int* n_tok, int n_q_heads, int n_kv_heads, int cache_len,
                                     int head_dim, int batch, int n_pages, int dtype, void* stream);

/* Speculative decoding (greedy, DecodeModel(ragged=True, spec_k=K), 1 <= K <= 7).  Slot b sits at position pos[b] with next input
 * tok[b].  One verify step feeds the window [tok, d1 .. dK] at positions pos .. pos + K (row b T + t, T = K + 1); only the
 * n[b] = min(T, cache_len - pos[b]) rows that fit in the cache are valid.  Row r's target is t_r = argmax(logits_r) (first index on
 * ties).  a = the largest r < n[b] with d_i == t_{i-1} for every i <= r; the slot emits d1 .. da, t_a (a + 1 tokens), then
 * pos <- (pos + a + 1) mod cache_len, tok <- t_a, next_tok <- t_a.  Cache rows past the new position may hold rejected rows; they
 * are never read.  A draft of -1 matches no target.
 *
 * rope_append_rows_devpos: the rows kernel with device positions: row b T + t goes to position pos[b] + t; rows t >= n[b] are
 * neither written nor rotated into q_out.  Written rows are bit for bit those of the _varlen entry point called with pos0 = pos.
 * pos is read before the programmatic wait: it must come from an earlier, completed launch.  1 <= T <= 8, T * n_q / n_kv <= 64.
 * The _paged twin writes through the page table. */
int hqq_b200_glue_rope_append_rows_devpos(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                          void* k_cache, void* v_cache, void* q_out, const int64_t* pos, int T, int n_q_heads,
                                          int n_kv_heads, int cache_len, int head_dim, int batch, int dtype, void* stream);
int hqq_b200_glue_rope_append_rows_devpos_paged(const void* q, const void* k, const void* v, const void* cos_table,
                                                const void* sin_table, void* k_pool, void* v_pool, const int* table, void* q_out,
                                                const int64_t* pos, int T, int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                                int batch, int n_pages, int dtype, void* stream);
/* Verify attention: out row b T + t, head h = softmax over cache rows 0 .. pos[b] + t of q_rot row b T + t (rotated, as the
 * rows kernel leaves it) against the cache, every row read from the cache (the devpos append writes rows pos .. just before).
 * Split-KV like rope_attn_decode_split (grid (S, n_kv * n_cg, batch), S = max(1, min(SMs / n_kv, ceil(cache_len / 16)))); the
 * (t, head) pairs of a GQA group are the MMA columns, 16 per CTA, n_cg = ceil(T * n_q / n_kv / 16) column groups per kv head.
 * Rows t >= n[b] are undefined (their q_rot rows are not written).  workspace: hqq_b200_glue_attn_verify_split_workspace_bytes() =
 * batch * n_kv * n_cg * max(1, SMs / n_kv) * 16 * (head_dim + 2) * 4 bytes of partials, one per column, then
 * batch * n_kv * n_cg uint32 tickets, zeroed once (every launch leaves them at zero).  1 <= T <= 8, T * n_q / n_kv <= 64. */
size_t hqq_b200_glue_attn_verify_split_workspace_bytes(int n_q_heads, int n_kv_heads, int head_dim, int T, int batch);
int hqq_b200_glue_attn_verify_split(const void* q_rot, const void* k_cache, const void* v_cache, const int64_t* pos, void* out,
                                    void* workspace, int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int T, int batch,
                                    int dtype, void* stream);
int hqq_b200_glue_attn_verify_split_paged(const void* q_rot, const void* k_pool, const void* v_pool, const int* table,
                                          const int64_t* pos, void* out, void* workspace, int n_q_heads, int n_kv_heads, int cache_len,
                                          int head_dim, int T, int batch, int n_pages, int dtype, void* stream);
/* 8-bit HQQ cache (levels uint8 and meta [.., 128 / gs] T, as hqq_b200_glue_rope_append_rows_kv8): the devpos append quantises
 * the valid rows into the cache exactly as the _varlen kv8 append does and writes no staging rows; the verify attention
 * dequantises every attended row, T(T(q - z) * s) as hqq_b200_dequantize gives it, into the 16-bit tile the 16-bit form uses.
 * Same workspace.  group_size 64 or 128. */
int hqq_b200_glue_rope_append_rows_kv8_devpos(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                              void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                              void* q_out, const int64_t* pos, int T, int n_q_heads, int n_kv_heads, int cache_len,
                                              int head_dim, int group_size, int batch, int dtype, void* stream);
int hqq_b200_glue_rope_append_rows_kv8_devpos_paged(const void* q, const void* k, const void* v, const void* cos_table,
                                                    const void* sin_table, void* k_q, void* k_scale, void* k_zero, void* v_q,
                                                    void* v_scale, void* v_zero, const int* table, void* q_out, const int64_t* pos, int T,
                                                    int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int group_size, int batch,
                                                    int n_pages, int dtype, void* stream);
int hqq_b200_glue_attn_verify_split_kv8(const void* q_rot, const void* k_q, const void* k_scale, const void* k_zero, const void* v_q,
                                        const void* v_scale, const void* v_zero, const int64_t* pos, void* out, void* workspace,
                                        int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int group_size, int T, int batch,
                                        int dtype, void* stream);
int hqq_b200_glue_attn_verify_split_kv8_paged(const void* q_rot, const void* k_q, const void* k_scale, const void* k_zero,
                                              const void* v_q, const void* v_scale, const void* v_zero, const int* table,
                                              const int64_t* pos, void* out, void* workspace, int n_q_heads, int n_kv_heads,
                                              int cache_len, int head_dim, int group_size, int T, int batch, int n_pages, int dtype,
                                              void* stream);

/* ---- 4-bit HQQ KV cache.
 * A cache row of one kv head is HQQ's Quantizer.quantize(row[1, 128], nbits=4, group_size=gs, axis=1, optimize=False,
 * round_zero=False) in fp32: inverse scale s = 15 / (max - min) (1 where |max - min| <= 1e-4, at most 2e4), zero z = -min * s,
 * levels round(x * s + z) clamped to [0, 15] with the product and the sum rounded separately; stored meta scale = 1 / s and zero,
 * both cast to T.  The levels are packed as the reference's 4bit_u8 packing of that row: 64 bytes, byte d = q[d] << 4 | q[d + 64].
 * group_size is 32 or 64 (a one-group row has no 4bit_u8 packing).  Levels uint8 [batch, n_kv_heads, cache_len, 64] (pages
 * [n_pages + 1, n_kv_heads, 64, 64]), meta [.., 128 / group_size] T.  The attended row is T(T(q - z) * s), what
 * Quantizer.dequantize gives.  Each entry point below is its kv8 twin with the same arguments, grid, split count, merge order,
 * workspace (the decode and verify forms use the existing workspace-size functions), RoPE rounding and preconditions, on this
 * format: the decode kernel quantises and packs the fresh k / v row and attends to its dequantisation, split 0 writing it to the
 * cache; the rows kernels write the rows the decode kernel writes and (not _devpos) stage their dequantisation. */
int hqq_b200_glue_rope_attn_decode_split_kv4(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                             void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                             const int64_t* pos, void* out, void* workspace, int n_q_heads, int n_kv_heads, int cache_len,
                                             int head_dim, int group_size, int batch, int dtype, void* stream);
int hqq_b200_glue_rope_attn_decode_split_kv4_seqpos(const void* q, const void* k, const void* v, const void* cos_table,
                                                    const void* sin_table, void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale,
                                                    void* v_zero, const int64_t* pos, void* out, void* workspace, int n_q_heads,
                                                    int n_kv_heads, int cache_len, int head_dim, int group_size, int batch, int dtype,
                                                    void* stream);
int hqq_b200_glue_rope_attn_decode_split_kv4_paged(const void* q, const void* k, const void* v, const void* cos_table,
                                                   const void* sin_table, void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale,
                                                   void* v_zero, const int* table, const int64_t* pos, void* out, void* workspace,
                                                   int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int group_size, int batch,
                                                   int n_pages, int dtype, void* stream);
int hqq_b200_glue_rope_append_rows_kv4(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                       void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero, void* k_stage,
                                       void* v_stage, void* q_out, int pos0, int T, int n_q_heads, int n_kv_heads, int cache_len,
                                       int head_dim, int group_size, int batch, int dtype, void* stream);
int hqq_b200_glue_rope_append_rows_kv4_varlen(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                              void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                              void* k_stage, void* v_stage, void* q_out, const int* pos0, const int* n_tok, int n_q_heads,
                                              int n_kv_heads, int cache_len, int head_dim, int group_size, int batch, int dtype,
                                              void* stream);
int hqq_b200_glue_rope_append_rows_kv4_paged(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                             void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                             const int* table, void* k_stage, void* v_stage, void* q_out, const int* pos0, const int* n_tok,
                                             int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int group_size, int batch,
                                             int n_pages, int dtype, void* stream);
/* Staging rows [0, pos0[b]) of every slot with n_tok[b] > 0 (host pos0 / n_tok, as the _varlen appends take them), dequantised from
 * the 4-bit cache: the contiguous caches (hqq_b200_dequantize cannot serve them: it unpacks slabs spanning all rows, while here
 * every row is packed on its own), or the page pools through the table.  Staging [batch, n_kv_heads, cache_len, 128] T. */
int hqq_b200_glue_kv4_stage(const void* k_q, const void* k_scale, const void* k_zero, const void* v_q, const void* v_scale,
                            const void* v_zero, void* k_stage, void* v_stage, const int* pos0, const int* n_tok, int n_kv_heads,
                            int cache_len, int head_dim, int group_size, int batch, int dtype, void* stream);
int hqq_b200_glue_kv4_stage_paged(const void* k_q, const void* k_scale, const void* k_zero, const void* v_q, const void* v_scale,
                                  const void* v_zero, const int* table, void* k_stage, void* v_stage, const int* pos0, const int* n_tok,
                                  int n_kv_heads, int cache_len, int head_dim, int group_size, int batch, int n_pages, int dtype,
                                  void* stream);
int hqq_b200_glue_rope_append_rows_kv4_devpos(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                              void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                              void* q_out, const int64_t* pos, int T, int n_q_heads, int n_kv_heads, int cache_len,
                                              int head_dim, int group_size, int batch, int dtype, void* stream);
int hqq_b200_glue_rope_append_rows_kv4_devpos_paged(const void* q, const void* k, const void* v, const void* cos_table,
                                                    const void* sin_table, void* k_q, void* k_scale, void* k_zero, void* v_q,
                                                    void* v_scale, void* v_zero, const int* table, void* q_out, const int64_t* pos, int T,
                                                    int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int group_size, int batch,
                                                    int n_pages, int dtype, void* stream);
int hqq_b200_glue_attn_verify_split_kv4(const void* q_rot, const void* k_q, const void* k_scale, const void* k_zero, const void* v_q,
                                        const void* v_scale, const void* v_zero, const int64_t* pos, void* out, void* workspace,
                                        int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int group_size, int T, int batch,
                                        int dtype, void* stream);
int hqq_b200_glue_attn_verify_split_kv4_paged(const void* q_rot, const void* k_q, const void* k_scale, const void* k_zero,
                                              const void* v_q, const void* v_scale, const void* v_zero, const int* table,
                                              const int64_t* pos, void* out, void* workspace, int n_q_heads, int n_kv_heads,
                                              int cache_len, int head_dim, int group_size, int T, int batch, int n_pages, int dtype,
                                              void* stream);

/* Prompt-lookup drafts: slot b knows L = pos[b] + 1 tokens, hist[b][0 .. pos - 1] (int32 [batch, cache_len]) and tok[b] at pos.
 * Take the longest g in {3, 2, 1} for which some j with j + g <= L - 1 has hist[j .. j+g-1] == the last g tokens, the largest such
 * j, and write drafts[b][i] = token j + g + i while j + g + i < L, else -1 (int64 [batch, K]); no match: every draft -1. */
int hqq_b200_glue_ngram_draft(const int32_t* hist, const int64_t* pos, const int64_t* tok, int64_t* drafts, int cache_len, int K,
                              int batch, void* stream);
/* Accept and advance: from targets int64 [batch, K + 1] and drafts int64 [batch, K], as defined above: tokens int64 [batch, K + 1]
 * (d1 .. da, t_a, then -1), n_new[b] = a + 1, hist[b][pos .. pos + a] = the accepted window, and pos, tok, next_tok advanced. */
int hqq_b200_glue_spec_accept(const int64_t* targets, const int64_t* drafts, int64_t* pos, int64_t* tok, int64_t* next_tok,
                              int32_t* hist, int64_t* tokens, int64_t* n_new, int cache_len, int K, int batch, void* stream);
/* out[0] = argmax(logits[0..n)) (first index on ties) */
int hqq_b200_glue_argmax(const void* logits, int n, int64_t* out, int dtype, void* stream);
/* Vocabulary-sharded lm_head (tensor parallel decode): out_key[0] = a signed 64-bit key {ordered(max) : 0xFFFFFFFF - (index_offset +
 * argmax)} of this rank's logits slice; the MAX of the keys over the ranks (one 8-byte all-reduce) names the global argmax, first
 * index on ties: token = 0xFFFFFFFF - (key & 0xFFFFFFFF). */
int hqq_b200_glue_argmax_key(const void* logits, int n, int64_t index_offset, int64_t* out_key, int dtype, void* stream);
/* The same pick with the key exchange inside the launch (tensor-parallel decode over peer-mapped memory, no collective library
 * call in the step): peer_keys[r] is rank r's key area, uint64 [2][tp], initialised to 0xFF bytes; *step_ctr >= 1 is the token
 * counter every rank advances in step (hqq_b200_glue_add_rmsnorm_tp bumps it).  Each rank stores its key, tagged with 12 bits of
 * the counter in key bits that are equal for all 16-bit values of one sign, into slot [ctr & 1][rank] of every peer, waits for
 * the tp keys of this step in its own area and writes the global argmax (first index on ties) to out[0]. */
int hqq_b200_glue_argmax_tp(const void* logits, int n, int64_t index_offset, void* const* peer_keys, int tp, int rank,
                            const int* step_ctr, int64_t* out, int dtype, void* stream);
/* Sampling in place of the argmax: row b of `rows` starts at logits + b * ld (elements; 16-byte aligned rows: logits 16-byte
 * aligned, ld % 8 == 0) and out[b] receives its token.  For a row l[0..n) and temperature > 0, top_k >= 0 (0: off), top_p in
 * (0, 1] (1: off), in the order of transformers' warpers:
 *   1. top-k: v_k = the top_k-th largest value of l, repeats counted; keep every i with l[i] >= v_k (ties at the pivot are all
 *      kept).  Off when top_k == 0 or top_k >= n.  The selection compares the 16-bit values as stored (-0 == +0), not l / T.
 *   2. top-p: p_i ~ exp((l[i] - max l) / T) over the kept set; v_p = the largest value such that the kept elements with l >= v_p
 *      carry at least top_p of the mass; keep those (ties again all kept; the maximum always survives).  The masses are fixed
 *      point, round(exp((l[i] - max) / T) * 2^32) of the fp32 exponential, summed in 64-bit integers.
 *   3. race: the token is the kept i with the largest l[i] / T + g_i (fp32), lowest index on equal keys; g_i = -log(-log u_i) with
 *      u_i = ((x >> 9) + 0.5) * 2^-23 (exact in fp32, in (0, 1)), x = word i % 4 of Philox4x32-10 with key (seed & 0xFFFFFFFF,
 *      seed >> 32) and counter (i / 4, b, *counter & 0xFFFFFFFF, *counter >> 32).
 * The token is a function of (row bits, n, temperature, top_k, top_p, seed, *counter, b) alone: not of the grid, rows, ld or the
 * GPU.  top_k = 1 gives the argmax when the maximum is unique.  *counter is read, never written (the decode harness advances it
 * by one per sampled token).  No workspace, no atomics outside shared memory.  Needs rows <= 65535. */
int hqq_b200_glue_sample(const void* logits, int n, int ld, int rows, float temperature, int top_k, float top_p, uint64_t seed,
                         const uint64_t* counter, int64_t* out, int dtype, void* stream);
/* Position keys: the same kept set and race, with the random numbers of each token keyed by the slot, the sequence and the
 * position of the row whose logits are sampled, so that a sequence's token at a given position draws the same numbers whichever
 * step (one-token decode, prefill, speculative verify) samples it and whatever the other slots do.  Row r of `rows` is slot
 * b = r / T at position p = pos[b] + r % T (T = rows_per_slot in [1, 8], dividing rows; pos and seq device int64 [rows / T]);
 * its race uses counter (i / 4, b, p & 0xFFFFFFFF, 0x80000000 | (seq[b] & 0x7FFFFFFF)) under the same key.  The high bit of
 * the last word keeps these counters apart from every counter of hqq_b200_glue_sample below 2^63.  The token is a function of
 * (row bits, n, temperature, top_k, top_p, seed, b, p, seq[b]) alone: not of the grid, the row's index in the launch or the
 * other slots.  The decode harness's seq[b] is a per-slot sequence number: zeroed by a reset, + 1 when a prefill starts the
 * slot at position 0, copied by a fork.  pos and seq are read, never written. */
int hqq_b200_glue_sample_pos(const void* logits, int n, int ld, int rows, float temperature, int top_k, float top_p, uint64_t seed,
                             int rows_per_slot, const int64_t* pos, const int64_t* seq, int64_t* out, int dtype, void* stream);

/* Number of kernels launched by this library on the calling thread since the last reset
 * (used by bench.py for its gpu_launches claim).                                        */
int64_t hqq_b200_launch_count(void);
void hqq_b200_launch_count_reset(void);

/* The few HQQ_B200_* switches the library reads (test / measurement hooks: HQQ_B200_GEMM_CTAS, HQQ_B200_GEMM_KSPLIT,
 * HQQ_B200_SMALL_M_MAX, HQQ_B200_PDL, HQQ_B200_PLAIN_SOLVER) are parsed once and cached; after changing one with setenv() call
 * this to have the next launch parse them again.  Not thread-safe against concurrent launches. */
void hqq_b200_reload_env(void);

#ifdef __cplusplus
}
#endif
#endif /* HQQ_B200_H */
