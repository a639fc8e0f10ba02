// Shared host/device helpers of libcvvae_b200: error reporting, launch accounting, dtype conversion,
// cuTensorMapEncodeTiled access without linking libcuda.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "../../include/cvvae_b200.h"

namespace cvvae {

// ---- error plumbing (api.cu owns the storage)
void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define CVVAE_CHECK_ARG(cond, ...)              \
  do {                                          \
    if (!(cond)) {                              \
      ::cvvae::set_error(__VA_ARGS__);          \
      return CVVAE_E_ARG;                       \
    }                                           \
  } while (0)

#define CVVAE_CUDA(expr)                                                                        \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) {                                                                    \
      ::cvvae::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return CVVAE_E_CUDA;                                                                      \
    }                                                                                           \
  } while (0)

#define CVVAE_LAUNCH_CHECK()                                                                    \
  do {                                                                                          \
    cudaError_t _e = cudaGetLastError();                                                        \
    if (_e != cudaSuccess) {                                                                    \
      ::cvvae::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return CVVAE_E_CUDA;                                                                      \
    }                                                                                           \
    ::cvvae::count_launch();                                                                    \
  } while (0)

// ---- driver entry point for TMA descriptors
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();

// fp32 -> nearest TF32 value (ties to even), kept in fp32 storage with the low 13 mantissa bits zero.  Written out in
// integer arithmetic so that it is the same function everywhere (kernels and the test-suite's reference).
__device__ __forceinline__ float tf32_rn(float v) {
  uint32_t u = __float_as_uint(v);
  if ((u & 0x7F800000u) != 0x7F800000u) u += 0xFFFu + ((u >> 13) & 1u);
  return __uint_as_float(u & 0xFFFFE000u);
}

// ---- storage <-> fp32
// T: stored element; P: a channel pair as one word (32 bit in 16-bit storage, 64 bit in fp32);
// from_f: the stored value of an output that is read as data (residual stream, conv outputs);
// mma_in: the value to store when the output's only consumers are tensor-core products (identity unless the
//         storage is wider than the MMA operand, i.e. F32: round to nearest TF32 instead of letting the MMA drop bits).
template <int DT>
struct Elem;
template <>
struct Elem<CVVAE_F16> {
  using T = __half;
  using T2 = __half2;
  using P = uint32_t;
  static __device__ __forceinline__ float to_f(T v) { return __half2float(v); }
  static __device__ __forceinline__ T from_f(float v) { return __float2half_rn(v); }
  static __device__ __forceinline__ float mma_in(float v) { return v; }
  static __device__ __forceinline__ float2 to_f2(uint32_t u) {
    return __half22float2(*reinterpret_cast<const __half2*>(&u));
  }
  static __device__ __forceinline__ uint32_t pack2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
};
template <>
struct Elem<CVVAE_BF16> {
  using T = __nv_bfloat16;
  using T2 = __nv_bfloat162;
  using P = uint32_t;
  static __device__ __forceinline__ float to_f(T v) { return __bfloat162float(v); }
  static __device__ __forceinline__ T from_f(float v) { return __float2bfloat16_rn(v); }
  static __device__ __forceinline__ float mma_in(float v) { return v; }
  static __device__ __forceinline__ float2 to_f2(uint32_t u) {
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u));
  }
  static __device__ __forceinline__ uint32_t pack2(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
};
template <>
struct Elem<CVVAE_F32> {
  using T = float;
  using T2 = float2;
  using P = float2;
  static __device__ __forceinline__ float to_f(T v) { return v; }
  static __device__ __forceinline__ T from_f(float v) { return v; }
  static __device__ __forceinline__ float mma_in(float v) { return tf32_rn(v); }
  static __device__ __forceinline__ float2 to_f2(float2 u) { return u; }
  static __device__ __forceinline__ float2 pack2(float a, float b) { return make_float2(a, b); }
};

// Eight consecutive channels of a 16-byte aligned channels-last row: one 16-byte vector in 16-bit storage, two in fp32.
template <int DT>
struct Vec8 {
  static constexpr int kN = static_cast<int>(sizeof(typename Elem<DT>::T)) / 2;   // 16-byte vectors
  uint4 v[kN];
};
template <int DT>
__device__ __forceinline__ Vec8<DT> ld8(const typename Elem<DT>::T* p) {
  Vec8<DT> r;
#pragma unroll
  for (int i = 0; i < Vec8<DT>::kN; ++i) r.v[i] = __ldg(reinterpret_cast<const uint4*>(p) + i);
  return r;
}
template <int DT>
__device__ __forceinline__ void st8(typename Elem<DT>::T* p, const Vec8<DT>& r) {
#pragma unroll
  for (int i = 0; i < Vec8<DT>::kN; ++i) reinterpret_cast<uint4*>(p)[i] = r.v[i];
}
template <int DT>
__device__ __forceinline__ void unpack8(const Vec8<DT>& r, float (&f)[8]) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(r.v);
  if constexpr (DT == CVVAE_F32) {
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = __uint_as_float(w[j]);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 t = Elem<DT>::to_f2(w[j]);
      f[2 * j] = t.x;
      f[2 * j + 1] = t.y;
    }
  }
}
template <int DT>
__device__ __forceinline__ Vec8<DT> pack8(const float (&f)[8]) {
  Vec8<DT> r;
  uint32_t* w = reinterpret_cast<uint32_t*>(r.v);
  if constexpr (DT == CVVAE_F32) {
#pragma unroll
    for (int j = 0; j < 8; ++j) w[j] = __float_as_uint(f[j]);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) w[j] = Elem<DT>::pack2(f[2 * j], f[2 * j + 1]);
  }
  return r;
}

#define CVVAE_DISPATCH_DTYPE(dt, ...)                          \
  do {                                                         \
    if ((dt) == CVVAE_F16) {                                   \
      constexpr int DT = CVVAE_F16;                            \
      __VA_ARGS__                                              \
    } else if ((dt) == CVVAE_BF16) {                           \
      constexpr int DT = CVVAE_BF16;                           \
      __VA_ARGS__                                              \
    } else if ((dt) == CVVAE_F32) {                            \
      constexpr int DT = CVVAE_F32;                            \
      __VA_ARGS__                                              \
    } else {                                                   \
      ::cvvae::set_error("unsupported dtype %d", (int)(dt));   \
      return CVVAE_E_ARG;                                      \
    }                                                          \
  } while (0)

// Entry points that exist for 16-bit storage only (video I/O, the tap-stacked conv_out kernel).
#define CVVAE_DISPATCH_DTYPE16(dt, what, ...)                                               \
  do {                                                                                      \
    if ((dt) == CVVAE_F16) {                                                                \
      constexpr int DT = CVVAE_F16;                                                         \
      __VA_ARGS__                                                                           \
    } else if ((dt) == CVVAE_BF16) {                                                        \
      constexpr int DT = CVVAE_BF16;                                                        \
      __VA_ARGS__                                                                           \
    } else {                                                                                \
      ::cvvae::set_error("%s: float16 / bfloat16 only, got dtype %d", (what), (int)(dt));   \
      return CVVAE_E_ARG;                                                                   \
    }                                                                                       \
  } while (0)

// GroupNorm statistics are accumulated as 64-bit FIXED-POINT integers (sum * 2^20, sum of squares * 2^18) so that
// the many atomic contributions add up to the same bits in any order: results stay deterministic run to run.
// Range: |sum| < 8.8e12, sum^2 < 3.5e13 per (sample, group) - e.g. 22.6 M elements of rms magnitude up to 1.2e3.
// The range is the same for fp32 activations as for 16-bit ones (the sums are formed in fp32 either way): it is the
// limit of the F32 path too.
constexpr double kGnSumScale = 1048576.0;   // 2^20
constexpr double kGnSqScale = 262144.0;     // 2^18
__device__ __forceinline__ unsigned long long gn_fix(float v, double scale) {
  return static_cast<unsigned long long>(__double2ll_rn(static_cast<double>(v) * scale));
}

// x * sigmoid(x); fast reciprocal (2 ulp) is far below the 16-bit output rounding
__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }

// ---- per-device state.  The library may be driven on several GPUs from one process (a model per device): everything
// cached about "the device" is keyed by the CURRENT device ordinal at the time of the call (the caller guarantees the
// current device is the one the pointers live on; cvvae_b200/ops.py enforces that).
constexpr int kMaxDevices = 64;
inline int cur_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return (dev >= 0 && dev < kMaxDevices) ? dev : 0;
}
inline int num_sms() {
  static std::atomic<int> n[kMaxDevices];
  const int dev = cur_device();
  int v = n[dev].load(std::memory_order_relaxed);
  if (v == 0) {
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    if (v <= 0) v = 132;
    n[dev].store(v, std::memory_order_relaxed);
  }
  return v;
}
// "has this one-time set-up (cudaFuncSetAttribute ...) been done on the current device?"  One static instance per call site.
struct PerDeviceOnce {
  std::atomic<bool> done[kMaxDevices];
  bool need() const { return !done[cur_device()].load(std::memory_order_acquire); }
  void mark() { done[cur_device()].store(true, std::memory_order_release); }
};

inline bool tensor_ok(const cvvae_tensor5* t) {
  return t && t->ptr && t->B > 0 && t->T > 0 && t->H > 0 && t->W > 0 && t->C > 0;
}

}  // namespace cvvae
