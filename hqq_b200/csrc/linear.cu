// hqq_b200_linear_fwd / hqq_b200_linear_fwd_multi: routing between the fused forward kernels.
#include "linear_internal.cuh"

namespace hqq {
bool small_route_ok(int64_t M, int64_t N, int64_t K, int gs, int nbits, int axis, int dtype);
size_t small_workspace_bytes(int64_t M);
int linear_small_multi(const void* x, int nprob, const void* const* Wq, const void* const* scale, const void* const* zero,
                       const void* const* bias, void* const* y, const int64_t* N, int64_t M, int64_t K, int gs, int nbits, int dtype,
                       void* ws, size_t ws_bytes, cudaStream_t st, int xop = 0, const void* x2 = nullptr, const void* xw = nullptr,
                       void* h_out = nullptr, float eps = 0.0f, const TpExchange* tpx = nullptr);
bool small_xop_ok(int64_t M, int64_t K);
int linear_small_grouped(const void* x, const int* x_rows, int nprob, const void* const* Wq, const void* const* scale, const void* const* zero,
                         void* const* y, const int64_t* N, int64_t K, int n_experts, const int* expert_off, const int* expert_cnt,
                         int64_t max_pairs, int gs, int nbits, int dtype, cudaStream_t st);
bool gemm_route_ok(int64_t M, int64_t N, int64_t K, int gs, int nbits, int axis, int dtype);
size_t gemm_workspace_bytes(int64_t M, int64_t N, int64_t K, int gs, int nbits, int dtype);
int linear_gemm(const void* x, const void* Wq, const void* scale, const void* zero, const void* bias, void* y, int64_t M,
                int64_t N, int64_t K, int gs, int nbits, int dtype, void* ws, size_t ws_bytes, cudaStream_t st);
bool dense_route_ok(int64_t M, int64_t N, int64_t K, int dtype);
int linear_dense(const void* x, const void* W, const void* bias, void* y, int64_t M, int64_t N, int64_t K, int dtype, cudaStream_t st);
size_t lm_logprob_ws_bytes(int64_t M, int64_t N);
int lm_logprob(const void* x, const void* W, const int64_t* targets, float* lse, float* tgt, void* ws, int64_t M, int64_t N, int64_t K,
               int64_t index_offset, int dtype, cudaStream_t st);
}  // namespace hqq

using namespace hqq;

// what hqq_b200_dequantize accepts (bitpack.cu): every width, both axes, any group size that divides the tensor
static bool dequant_ok(int64_t N, int64_t K, int gs, int nbits, int axis) {
  if (!valid_nbits(nbits) || !(axis == 0 || axis == 1) || gs <= 0 || N <= 0 || K <= 0 || (N * K) % gs != 0) return false;
  const int64_t R = axis == 1 ? N * K / gs : gs;
  return nbits == 3 || R % fields_of(nbits) == 0;
}

static size_t dense_ws_bytes(int64_t N, int64_t K, int dtype) { return (size_t)((N * K * (int64_t)dtype_size(dtype) + 255) & ~(int64_t)255); }

// Where the single-matrix entry point hands over from the small-M kernel (mma.sync, streams x per tile) to the wgmma kernel when
// both take the shape: up to M = 16 everywhere, and up to M = 32 on matrices of at most 2^24 weights, where the weight stream the
// small kernel is bound by still dominates; larger problems go to the wgmma kernel.  tools/prof_route_boundary.py times both
// sides.  HQQ_B200_SMALL_M_MAX=<m> (measurement hook) replaces the rule by "small kernel up to M = m".
static bool prefer_small(int64_t M, int64_t N, int64_t K) {
  HQQ_ENV_KNOB(m, ([] { const char* e = getenv("HQQ_B200_SMALL_M_MAX"); return e ? atoi(e) : 0; })());
  if (m > 0) return M <= m;
  return M <= 16 || N * K <= (int64_t(1) << 24);
}

extern "C" int hqq_b200_linear_fwd_route(int64_t M, int64_t N, int64_t K, int group_size, int nbits, int axis, int dtype) {
  const bool small = small_route_ok(M, N, K, group_size, nbits, axis, dtype);
  if (small && (prefer_small(M, N, K) || !gemm_route_ok(M, N, K, group_size, nbits, axis, dtype))) return 1;
  if (gemm_route_ok(M, N, K, group_size, nbits, axis, dtype)) return 2;
  if (dequant_ok(N, K, group_size, nbits, axis) && dense_route_ok(M, N, K, dtype)) return 3;  // dequantize kernel -> dense wgmma GEMM
  return 0;
}

extern "C" size_t hqq_b200_linear_fwd_workspace_bytes(int64_t M, int64_t N, int64_t K, int group_size, int nbits, int axis, int dtype) {
  switch (hqq_b200_linear_fwd_route(M, N, K, group_size, nbits, axis, dtype)) {
    case 1: return small_workspace_bytes(M);
    case 2: return gemm_workspace_bytes(M, N, K, group_size, nbits, dtype);
    case 3: return dense_ws_bytes(N, K, dtype);  // W_r, written by the dequantize kernel and read back (mostly from L2) by the GEMM
  }
  return 0;
}

static int check_common(const void* x, int64_t M, int64_t K, int group_size, int nbits, int axis) {
  HQQ_REQUIRE(x, HQQ_E_INVALID, "hqq_b200_linear_fwd: null pointer");
  HQQ_REQUIRE(M > 0 && K > 0 && group_size > 0, HQQ_E_INVALID, "hqq_b200_linear_fwd: bad shape M=%lld K=%lld gs=%d", (long long)M, (long long)K, group_size);
  HQQ_REQUIRE(valid_nbits(nbits), HQQ_E_INVALID, "nbits=%d not supported.", nbits);
  HQQ_REQUIRE(axis == 0 || axis == 1, HQQ_E_INVALID, "axis should be either 0 or 1");
  return HQQ_OK;
}

extern "C" int hqq_b200_linear_fwd(const void* x, const void* W_q, const void* scale, const void* zero, const void* bias, void* y,
                                   int64_t M, int64_t N, int64_t K, int group_size, int nbits, int axis, int dtype, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  int rc = check_common(x, M, K, group_size, nbits, axis);
  if (rc) return rc;
  HQQ_REQUIRE(W_q && scale && zero && y && N > 0, HQQ_E_INVALID, "hqq_b200_linear_fwd: null pointer or empty matrix");
  cudaStream_t st = (cudaStream_t)stream;
  const int route = hqq_b200_linear_fwd_route(M, N, K, group_size, nbits, axis, dtype);
  if (route == 1) return linear_small_multi(x, 1, &W_q, &scale, &zero, &bias, &y, &N, M, K, group_size, nbits, dtype, workspace, workspace_bytes, st);
  if (route == 2) return linear_gemm(x, W_q, scale, zero, bias, y, M, N, K, group_size, nbits, dtype, workspace, workspace_bytes, st);
  if (route == 3) {
    HQQ_REQUIRE(workspace != nullptr && workspace_bytes >= dense_ws_bytes(N, K, dtype) && aligned(workspace, 256), HQQ_E_WORKSPACE,
                "hqq_b200_linear_fwd: this configuration runs dequantize + dense GEMM and needs a 256-byte aligned workspace of %zu bytes (got %zu)",
                dense_ws_bytes(N, K, dtype), workspace_bytes);
    rc = hqq_b200_dequantize(W_q, scale, zero, workspace, N, K, group_size, nbits, axis, dtype, stream);
    if (rc) return rc;
    return linear_dense(x, workspace, bias, y, M, N, K, dtype, st);
  }
  set_error("hqq_b200_linear_fwd: no fused kernel for M=%lld N=%lld K=%lld gs=%d nbits=%d axis=%d dtype=%d", (long long)M, (long long)N,
            (long long)K, group_size, nbits, axis, dtype);
  return HQQ_E_UNSUPPORTED;
}

extern "C" int hqq_b200_dense_gemm(const void* x, const void* W, const void* bias, void* y, int64_t M, int64_t N, int64_t K, int dtype,
                                   void* stream) {
  return linear_dense(x, W, bias, y, M, N, K, dtype, (cudaStream_t)stream);
}

extern "C" size_t hqq_b200_lm_logprob_workspace_bytes(int64_t M, int64_t N) { return lm_logprob_ws_bytes(M, N); }

extern "C" int hqq_b200_lm_logprob(const void* x, const void* W, const int64_t* targets, float* lse, float* tgt, void* workspace, int64_t M,
                                   int64_t N, int64_t K, int64_t index_offset, int dtype, void* stream) {
  return lm_logprob(x, W, targets, lse, tgt, workspace, M, N, K, index_offset, dtype, (cudaStream_t)stream);
}

extern "C" int hqq_b200_linear_fwd_multi(const void* x, int count, const void* const* W_q, const void* const* scale,
                                         const void* const* zero, const void* const* bias, void* const* y, const int64_t* N, int64_t M,
                                         int64_t K, int group_size, int nbits, int axis, int dtype, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  int rc = check_common(x, M, K, group_size, nbits, axis);
  if (rc) return rc;
  HQQ_REQUIRE(count >= 1 && count <= 4 && W_q && scale && zero && y && N, HQQ_E_INVALID, "hqq_b200_linear_fwd_multi: 1..4 matrices, non-null arrays");
  for (int i = 0; i < count; ++i) {
    if (!small_route_ok(M, N[i], K, group_size, nbits, axis, dtype)) {
      set_error("hqq_b200_linear_fwd_multi: matrix %d (N=%lld K=%lld gs=%d nbits=%d axis=%d dtype=%d M=%lld) is outside the fused small-M kernel",
                i, (long long)N[i], (long long)K, group_size, nbits, axis, dtype, (long long)M);
      return HQQ_E_UNSUPPORTED;
    }
  }
  return linear_small_multi(x, count, W_q, scale, zero, bias, y, N, M, K, group_size, nbits, dtype, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int hqq_b200_linear_fwd_grouped(const void* x, const int32_t* x_rows, int count, const void* const* W_q, const void* const* scale,
                                           const void* const* zero, void* const* y, const int64_t* N, int64_t K, int n_experts,
                                           const int32_t* expert_off, const int32_t* expert_cnt, int64_t max_pairs, int group_size, int nbits,
                                           int dtype, void* stream) {
  int rc = check_common(x, 1, K, group_size, nbits, 1);
  if (rc) return rc;
  HQQ_REQUIRE(count >= 1 && count <= 4 && W_q && scale && zero && y && N, HQQ_E_INVALID, "hqq_b200_linear_fwd_grouped: 1..4 matrices, non-null arrays");
  HQQ_REQUIRE(n_experts >= 1 && n_experts <= 64, HQQ_E_INVALID, "hqq_b200_linear_fwd_grouped: 1..64 experts (got %d)", n_experts);
  HQQ_REQUIRE(expert_off && expert_cnt, HQQ_E_INVALID, "hqq_b200_linear_fwd_grouped: null expert tables");
  HQQ_REQUIRE(max_pairs >= 1 && max_pairs <= 65535LL * 8, HQQ_E_INVALID, "hqq_b200_linear_fwd_grouped: max_pairs must be in [1, 524280] (got %lld)",
              (long long)max_pairs);
  HQQ_REQUIRE(aligned(x, 16), HQQ_E_INVALID, "hqq_b200_linear_fwd_grouped: x must be 16-byte aligned");
  for (int i = 0; i < count; ++i) {
    HQQ_REQUIRE(W_q[i] && scale[i] && zero[i] && y[i] && N[i] > 0, HQQ_E_INVALID, "hqq_b200_linear_fwd_grouped: null pointer or empty matrix %d", i);
    HQQ_REQUIRE(aligned(W_q[i], 16) && aligned(scale[i], 8) && aligned(zero[i], 8), HQQ_E_INVALID,
                "hqq_b200_linear_fwd_grouped: W_q must be 16-byte and scale/zero 8-byte aligned");
    if (!small_route_ok(1, N[i], K, group_size, nbits, 1, dtype)) {
      set_error("hqq_b200_linear_fwd_grouped: matrix %d (N=%lld K=%lld gs=%d nbits=%d dtype=%d) is outside the small-M kernel", i, (long long)N[i],
                (long long)K, group_size, nbits, dtype);
      return HQQ_E_UNSUPPORTED;
    }
  }
  return linear_small_grouped(x, x_rows, count, W_q, scale, zero, y, N, K, n_experts, expert_off, expert_cnt, max_pairs, group_size, nbits, dtype,
                              (cudaStream_t)stream);
}

extern "C" int hqq_b200_decode_linear_fwd(const void* x, int x_op, const void* x2, const void* x_weight, void* h_out, float eps, int count,
                                          const void* const* W_q, const void* const* scale, const void* const* zero,
                                          const void* const* bias, void* const* y, const int64_t* N, int64_t K, int group_size, int nbits,
                                          int dtype, void* stream) {
  int rc = check_common(x, 1, K, group_size, nbits, 1);
  if (rc) return rc;
  HQQ_REQUIRE(count >= 1 && count <= 4 && W_q && scale && zero && y && N, HQQ_E_INVALID, "hqq_b200_decode_linear_fwd: 1..4 matrices, non-null arrays");
  HQQ_REQUIRE(x_op >= 0 && (x_op & 15) <= 2 && (x_op >> 4) <= 1, HQQ_E_INVALID,
              "hqq_b200_decode_linear_fwd: x_op must be 0 (none), 1 (add+rmsnorm) or 2 (silu*mul), optionally | HQQ_YOP_SILU_MUL_PAIR");
  for (int i = 0; i < count; ++i) {
    if (!small_route_ok(1, N[i], K, group_size, nbits, 1, dtype) || (x_op != 0 && !small_xop_ok(1, K))) {
      set_error("hqq_b200_decode_linear_fwd: matrix %d (N=%lld K=%lld gs=%d nbits=%d dtype=%d) is outside the fused M=1 kernel", i, (long long)N[i],
                (long long)K, group_size, nbits, dtype);
      return HQQ_E_UNSUPPORTED;
    }
  }
  return linear_small_multi(x, count, W_q, scale, zero, bias, y, N, 1, K, group_size, nbits, dtype, nullptr, 0, (cudaStream_t)stream, x_op, x2,
                            x_weight, h_out, eps);
}

extern "C" int hqq_b200_decode_linear_fwd_desc(const hqq_b200_decode_desc* d, void* stream) {
  HQQ_REQUIRE(d != nullptr, HQQ_E_INVALID, "hqq_b200_decode_linear_fwd_desc: null descriptor");
  int rc = check_common(d->x ? d->x : d->x_tagged, 1, d->K, d->group_size, d->nbits, 1);
  if (rc) return rc;
  HQQ_REQUIRE(d->count >= 1 && d->count <= 4 && d->W_q && d->scale && d->zero && d->y && d->N, HQQ_E_INVALID,
              "hqq_b200_decode_linear_fwd_desc: 1..4 matrices, non-null arrays");
  HQQ_REQUIRE(d->x_op >= 0 && (d->x_op & 15) <= 2 && (d->x_op >> 4) <= 1, HQQ_E_INVALID,
              "hqq_b200_decode_linear_fwd_desc: x_op must be 0, 1 or 2, optionally | HQQ_YOP_SILU_MUL_PAIR");
  HQQ_REQUIRE(d->x || ((d->x_op & 15) == 2 && d->x_tagged), HQQ_E_INVALID, "hqq_b200_decode_linear_fwd_desc: no activation given");
  for (int i = 0; i < d->count; ++i) {
    if (!small_route_ok(1, d->N[i], d->K, d->group_size, d->nbits, 1, d->dtype) || !small_xop_ok(1, d->K)) {
      set_error("hqq_b200_decode_linear_fwd_desc: matrix %d (N=%lld K=%lld gs=%d nbits=%d dtype=%d) is outside the fused M=1 kernel", i,
                (long long)d->N[i], (long long)d->K, d->group_size, d->nbits, d->dtype);
      return HQQ_E_UNSUPPORTED;
    }
  }
  TpExchange t{d->tp, d->rank, d->peer_data, d->red_data, d->y_tagged, d->x_tagged, d->x2_tagged, d->step_ctr, d->x_index, d->x_per_step};
  const bool exchange = d->step_ctr != nullptr;
  // a tagged x still needs a mapped pointer for the alignment checks / unused plain path: reuse the tagged buffer itself
  const void* x = d->x ? d->x : d->x_tagged;
  return linear_small_multi(x, d->count, d->W_q, d->scale, d->zero, d->bias, d->y, d->N, 1, d->K, d->group_size, d->nbits, d->dtype, nullptr, 0,
                            (cudaStream_t)stream, d->x_op, d->x2, d->x_weight, d->h_out, d->eps, exchange ? &t : nullptr);
}
