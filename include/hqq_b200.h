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

/* Number of kernels launched by this library on the calling thread since the last reset
 * (used by bench.py for its gpu_launches claim).                                        */
int64_t hqq_b200_launch_count(void);
void hqq_b200_launch_count_reset(void);

/* The few HQQ_B200_* switches the library reads (test hooks: HQQ_B200_GEMM_CTAS, HQQ_B200_DECODE1, HQQ_B200_PDL,
 * HQQ_B200_PLAIN_SOLVER) are parsed once and cached; after changing one with setenv() call this to have the next launch parse
 * them again.  Not thread-safe against concurrent launches. */
void hqq_b200_reload_env(void);

#ifdef __cplusplus
}
#endif
#endif /* HQQ_B200_H */
