// Shared helpers for the hqq_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "../../include/hqq_b200.h"

namespace hqq {

// ---- error plumbing -----------------------------------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;
extern std::atomic<int> g_env_epoch;  // bumped by hqq_b200_reload_env(): cached HQQ_B200_* knobs are parsed again

// `static int var`, parsed from the environment by `expr` on first use and again after every hqq_b200_reload_env()
#define HQQ_ENV_KNOB(var, expr)                                                     \
  static int var = 0;                                                               \
  {                                                                                 \
    static int epoch__ = -1;                                                        \
    const int now__ = ::hqq::g_env_epoch.load(std::memory_order_relaxed);           \
    if (epoch__ != now__) { var = (expr); epoch__ = now__; }                        \
  }

#define HQQ_REQUIRE(cond, code, ...)            \
  do {                                          \
    if (!(cond)) {                              \
      ::hqq::set_error(__VA_ARGS__);            \
      return (code);                            \
    }                                           \
  } while (0)

// Launch check that is legal under stream capture (no sync).
#define HQQ_LAUNCH_CHECK(name)                                                 \
  do {                                                                         \
    cudaError_t e__ = cudaGetLastError();                                      \
    ::hqq::g_launches.fetch_add(1, std::memory_order_relaxed);                 \
    if (e__ != cudaSuccess) {                                                  \
      ::hqq::set_error("%s: CUDA launch failed: %s", name, cudaGetErrorString(e__)); \
      return HQQ_E_CUDA;                                                       \
    }                                                                          \
  } while (0)

static inline bool aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) % a) == 0; }
static inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

constexpr int kNumSMs = 132;  // H100 SXM

// ---- host launch path ------------------------------------------------------------------------
// Function attributes and SM counts belong to ONE device: the caches are indexed by the calling thread's current device, so
// layers living on several GPUs of one process each get their own setup.
constexpr int kMaxDevices = 64;
int current_device();  // 0 when it cannot be queried or lies outside the caches
int sm_count();        // of the current device, cached; kNumSMs when it cannot be queried
bool pdl_enabled();    // HQQ_B200_PDL=0 (test hook) launches without the programmatic-dependency attribute

// Opts KERNEL into `bytes` of dynamic shared memory on the current device (kept per device: the largest request so far).
template <auto KERNEL>
static int reserve_smem(int bytes) {
  static int reserved[kMaxDevices] = {};
  int& r = reserved[current_device()];
  if (bytes > r) {
    cudaError_t e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    HQQ_REQUIRE(e == cudaSuccess, HQQ_E_CUDA, "hqq_b200_linear_fwd: cannot reserve %d bytes of shared memory: %s", bytes, cudaGetErrorString(e));
    r = bytes;
  }
  return HQQ_OK;
}

// Launches with programmatic dependent launch (the kernel's prologue may overlap the tail of the previous kernel on the
// stream; the kernel calls pdl_wait() before it reads what that kernel wrote) and counts the launch.
template <typename K, typename... Args>
static int launch_pdl(const char* name, K kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, args...);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  HQQ_REQUIRE(e == cudaSuccess, HQQ_E_CUDA, "%s: CUDA launch failed: %s", name, cudaGetErrorString(e));
  return HQQ_OK;
}

static inline int fields_of(int nbits) { return nbits == 3 ? 10 : 8 / nbits; }
static inline bool valid_nbits(int nbits) { return nbits == 8 || nbits == 4 || nbits == 3 || nbits == 2 || nbits == 1; }
static inline size_t dtype_size(int dt) {
  switch (dt) {
    case HQQ_F32: case HQQ_I32: return 4;
    case HQQ_F16: case HQQ_BF16: return 2;
    case HQQ_U8: return 1;
    case HQQ_I64: return 8;
  }
  return 0;
}

// ---- device-side scalar conversions ---------------------------------------------------
template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

// integer level -> T (levels are < 256: exact in every type)
template <typename T> __device__ __forceinline__ T level_to(unsigned q);
template <> __device__ __forceinline__ float level_to<float>(unsigned q) { return (float)q; }
template <> __device__ __forceinline__ __half level_to<__half>(unsigned q) { return __ushort2half_rn((unsigned short)q); }
template <> __device__ __forceinline__ __nv_bfloat16 level_to<__nv_bfloat16>(unsigned q) { return __ushort2bfloat16_rn((unsigned short)q); }
template <> __device__ __forceinline__ uint8_t level_to<uint8_t>(unsigned q) { return (uint8_t)q; }
template <> __device__ __forceinline__ int32_t level_to<int32_t>(unsigned q) { return (int32_t)q; }
template <> __device__ __forceinline__ int64_t level_to<int64_t>(unsigned q) { return (int64_t)q; }

// (q - z) * s with one rounding per operation in T -- the reference's two-rounding dequant
// (hqq/core/quantize.py:198).  __fsub_rn/__fmul_rn forbid FMA contraction.
template <typename T> __device__ __forceinline__ T dequant_one(unsigned q, T z, T s);
template <> __device__ __forceinline__ float dequant_one<float>(unsigned q, float z, float s) {
  return __fmul_rn(__fsub_rn((float)q, z), s);
}
template <> __device__ __forceinline__ __half dequant_one<__half>(unsigned q, __half z, __half s) {
  return __hmul(__hsub(level_to<__half>(q), z), s);
}
template <> __device__ __forceinline__ __nv_bfloat16 dequant_one<__nv_bfloat16>(unsigned q, __nv_bfloat16 z, __nv_bfloat16 s) {
  return __hmul(__hsub(level_to<__nv_bfloat16>(q), z), s);
}

// ---- quantisation of one group (csrc/quantize.cu and the 8-bit KV cache of csrc/decode_glue.cu) ----------------------------
__device__ __forceinline__ float rint_magic(float t) {
  // round-half-even for |t| < 2^22; beyond that the result is still >= 2^22-ish in magnitude with the
  // right sign, so the clamp that always follows yields the same level as rintf would.
  return __fsub_rn(__fadd_rn(t, 12582912.0f), 12582912.0f);
}

struct GroupState {
  float s, rs, z;
};

__device__ __forceinline__ void init_group(float mn, float mx, int maxv, int round_zero, GroupState& st) {
  // quantize.py:126-134 ; `max_v / denom` is reciprocal(denom) * max_v in torch (two roundings)
  float denom = __fsub_rn(mx, mn);
  float s = __fmul_rn(__frcp_rn(denom), (float)maxv);
  if (fabsf(denom) <= 1e-4f) s = 1.0f;
  s = fminf(s, 2e4f);
  float z = __fmul_rn(-mn, s);
  if (round_zero) z = rintf(z);
  st.s = s;
  st.rs = __frcp_rn(s);
  st.z = z;
}

// optimize.py:254 / quantize.py:147: round(W*scale + zero).clamp(min,max); mul and add round separately
__device__ __forceinline__ float quant_level(float w, float s, float z, float fmaxv) {
  const float t = rint_magic(__fadd_rn(__fmul_rn(w, s), z));
  return fminf(fmaxf(t, 0.0f), fmaxv);
}

// ---- vector of N elements of T with 16/8/4-byte aligned storage ------------------------
template <typename T, int N>
struct alignas(sizeof(T) * N >= 16 ? 16 : sizeof(T) * N) Vec {
  T v[N];
};

// ---- device primitives ----------------------------------------------------------------------
// Programmatic dependent launch.  Under the CPU emulator (tests/emu) kernels run one after another: nothing to wait for.
#ifdef HQQ_EMU
__device__ __forceinline__ void pdl_wait() {}
__device__ __forceinline__ void pdl_launch_dependents() {}
#else
// blocks until the grids this one depends on have completed and their writes are visible
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// lets the next kernel on the stream launch; it still waits for this grid in its own pdl_wait()
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#endif

// byte permute (prmt.b32, default mode): result byte i is byte ((s >> 4i) & 7) of the eight bytes {b, a}, a being bytes 0-3
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t s) {
#ifdef HQQ_EMU
  return ::emu::prmt(a, b, s);
#else
  uint32_t r;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(s));
  return r;
#endif
}

// streaming 16-byte global load that does not pollute L1 (weights are read exactly once)
__device__ __forceinline__ uint4 ldg_stream_v4(const void* p) {
#ifdef HQQ_EMU
  return *reinterpret_cast<const uint4*>(p);
#endif
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

}  // namespace hqq
