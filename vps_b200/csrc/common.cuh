// Shared device/host helpers for libvps_b200.so (sm_90a).
#pragma once
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <type_traits>

#include "../../include/vps_b200.h"

namespace vps {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);
// SM count of the current device (cached; 0 without a device)
int num_sms();
// the driver's cuTensorMapEncodeTiled (cached; nullptr, with the error set, if the driver lacks it)
PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder();
// Tensor map over the NHWC tensor t: dims {c, w, h, n}, box {box_c, box_w, box_h, 1} read every {1, sw, sh, 1} elements,
// no interleave or OOB NaN fill.  The pixel, row and image strides come from `strides` (default t): cs, w * cs and h * w * cs
// elements of type `type` (fp32 or a 16-bit type).  On failure the error, prefixed by `who`, is set and false returned.
bool encode_nhwc(CUtensorMap* m, const vps_tensor& t, CUtensorMapDataType type, int box_c, int box_w, int box_h, int sw, int sh,
                 CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2, const char* who, const vps_tensor* strides = nullptr);

#define VPS_CHECK_ARG(cond, ...)          \
  do {                                    \
    if (!(cond)) {                        \
      vps::set_error(__VA_ARGS__);        \
      return VPS_E_ARG;                   \
    }                                     \
  } while (0)

#define VPS_CUDA_LAST(name)                                                        \
  do {                                                                             \
    cudaError_t e__ = cudaGetLastError();                                          \
    if (e__ != cudaSuccess) {                                                      \
      vps::set_error("%s: %s", name, cudaGetErrorString(e__));                     \
      return VPS_E_CUDA;                                                           \
    }                                                                              \
    vps::count_launch();                                                           \
  } while (0)

static inline int cdiv(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// blocks of a grid-stride launch over `total` items, capped at 148 * 32: 32 blocks per SM of the 148-SM B200 (an H100 has
// 132 SMs; the cap has not been retuned for it)
static inline int grid_for(int64_t total, int threads = 256) {
  int64_t b = (total + threads - 1) / threads;
  const int64_t cap = 148 * 32;
  return (int)(b > cap ? cap : (b < 1 ? 1 : b));
}

#define VPS_GRID_STRIDE(i, total) \
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < (total); i += (int64_t)gridDim.x * blockDim.x)

// decompose flat index over [n,h,w,c] with c fastest
#define VPS_DECOMP_NHWC(i, T_, n_, y_, x_, c_)  \
  const int c_ = (int)((i) % (T_).c);           \
  int64_t t__ = (i) / (T_).c;                   \
  const int x_ = (int)(t__ % (T_).w);           \
  t__ /= (T_).w;                                \
  const int y_ = (int)(t__ % (T_).h);           \
  const int n_ = (int)(t__ / (T_).h)

// ---- typed element access (activations are f32 or bf16) ----
template <typename T>
__device__ __forceinline__ float ldf(const T* p);
template <>
__device__ __forceinline__ float ldf<float>(const float* p) { return __ldg(p); }
template <>
__device__ __forceinline__ float ldf<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __bfloat162float(*p);
}
template <typename T>
__device__ __forceinline__ void stf(T* p, float v);
template <>
__device__ __forceinline__ void stf<float>(float* p, float v) { *p = v; }
template <>
__device__ __forceinline__ void stf<__nv_bfloat16>(__nv_bfloat16* p, float v) {
  *p = __float2bfloat16_rn(v);
}

// Device view of vps_tensor.
template <typename T>
struct TV {
  T* p;
  int n, h, w, c, cs;
  __device__ __forceinline__ int64_t off(int b, int y, int x) const {
    return (((int64_t)b * h + y) * w + x) * cs;
  }
};
template <typename T>
static inline TV<T> tv(const vps_tensor& t) {
  TV<T> v;
  v.p = (T*)t.ptr;
  v.n = t.n; v.h = t.h; v.w = t.w; v.c = t.c; v.cs = t.cs;
  return v;
}

// binds T to the element type of `dtype` (f32 or bf16); nest it to bind a second type (input / output, data / flow)
#define VPS_DISPATCH_T(dtype, T, ...)                         \
  do {                                                        \
    if ((dtype) == VPS_F32) { using T = float; __VA_ARGS__; } \
    else { using T = __nv_bfloat16; __VA_ARGS__; }            \
  } while (0)

__device__ __forceinline__ float apply_act(float v, int act, float slope) {
  if (act == VPS_ACT_RELU) return v > 0.f ? v : 0.f;
  if (act == VPS_ACT_LRELU) return v > 0.f ? v : v * slope;
  if (act == VPS_ACT_SIGMOID) return 1.f / (1.f + expf(-v));
  return v;
}

}  // namespace vps

// ---- vectorised channel access: V consecutive channels per thread (V = 16 bytes / sizeof(T), or 1) ----
namespace vps {
template <typename T> struct VecW;
template <> struct VecW<float> { static constexpr int value = 4; };
template <> struct VecW<__nv_bfloat16> { static constexpr int value = 8; };

template <typename T, int V>
__device__ __forceinline__ void ldv(const T* p, float (&v)[V]) {
  if constexpr (V == 1) {
    v[0] = ldf<T>(p);
  } else if constexpr (sizeof(T) == 4) {
    static_assert(V == 4, "fp32 vector width");
    const float4 f = *reinterpret_cast<const float4*>(p);
    v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
  } else {
    static_assert(V == 8, "bf16 vector width");
    const uint4 raw = *reinterpret_cast<const uint4*>(p);
    const __nv_bfloat162* b2 = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __bfloat1622float2(b2[j]);
      v[2 * j] = f.x; v[2 * j + 1] = f.y;
    }
  }
}
template <typename T, int V>
__device__ __forceinline__ void stv(T* p, const float (&v)[V]) {
  if constexpr (V == 1) {
    stf<T>(p, v[0]);
  } else if constexpr (sizeof(T) == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    uint4 o;
    __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) o2[j] = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
    *reinterpret_cast<uint4*>(p) = o;
  }
}
// can tensor t be accessed with V-wide vectors of its dtype over its first `c` channels?
static inline bool vec_ok(const vps_tensor& t, int c) {
  int V;
  VPS_DISPATCH_T(t.dtype, T, V = VecW<T>::value);
  return c % V == 0 && t.cs % V == 0 && ((uintptr_t)t.ptr & 15) == 0;
}
// launch geometry of the (x*chunks, y, n) pixel grid
static inline dim3 pix_grid(int w, int chunks, int h, int n, int threads = 256) {
  return dim3((unsigned)cdiv((int64_t)w * chunks, threads), (unsigned)h, (unsigned)n);
}
}  // namespace vps

// bilinear blend with an explicit operation order: `hx*a + lx*b` leaves the compiler free to fuse either product into the
// FMA, and two kernels computing the same interpolation (resize_bilinear / the fused FlowNet2 stage kernel) must agree bit
// for bit
__device__ __forceinline__ float vps_bilerp(float v00, float v01, float v10, float v11, float hx, float lx, float hy, float ly) {
  const float top = __fmaf_rn(hx, v00, __fmul_rn(lx, v01));
  const float bot = __fmaf_rn(hx, v10, __fmul_rn(lx, v11));
  return __fmaf_rn(hy, top, __fmul_rn(ly, bot));
}

// per-thread coordinates for kernels launched with vps::pix_grid: V channels starting at `c`, pixel (n,y,x)
#define VPS_PIX_COORDS(OUT, V, c_, x_, y_, n_)                           \
  const int chunks__ = (OUT).c / (V);                                    \
  const int t__ = blockIdx.x * blockDim.x + threadIdx.x;                 \
  if (t__ >= (OUT).w * chunks__) return;                                 \
  const int c_ = (t__ % chunks__) * (V), x_ = t__ / chunks__, y_ = blockIdx.y, n_ = blockIdx.z

// channel width V of a VPS_PIX_COORDS launch, bound at compile time: VW if `vec` (every tensor passed vps::vec_ok), else 1
#define VPS_WITH_V(VW, vec, V, ...)                     \
  do {                                                  \
    if (vec) { constexpr int V = VW; __VA_ARGS__; }     \
    else { constexpr int V = 1; __VA_ARGS__; }          \
  } while (0)
// binds T from `dtype` and V = VecW<T>::value if `vec`, else 1; the launch covers vps::pix_grid(w, c / V, h, n)
#define VPS_DISPATCH_V(dtype, vec, T, V, ...) VPS_DISPATCH_T(dtype, T, VPS_WITH_V(vps::VecW<T>::value, vec, V, __VA_ARGS__))
// input / output pair: the vector arm exists only where TI == TO (a mixed pair has no vector instances, V = 1)
#define VPS_DISPATCH_IN_OUT_V(in_dtype, out_dtype, vec, TI, TO, V, ...)                  \
  VPS_DISPATCH_T(in_dtype, TI, VPS_DISPATCH_T(out_dtype, TO,                             \
    VPS_WITH_V((std::is_same<TI, TO>::value ? vps::VecW<TI>::value : 1), vec, V, __VA_ARGS__)))
