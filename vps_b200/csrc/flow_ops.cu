// FlowNet2 native ops: correlation, resample2d, channelnorm (NHWC, f32 or bf16 storage, fp32 math).
// Semantics follow correlation_cuda_kernel.cu:74-147, resample2d_kernel.cu:16-71,
// channelnorm_kernel.cu:19-60 of the reference (see include/vps_b200.h).
#include "common.cuh"

namespace {

// ------------------------------------------------------------------ correlation (CUDA-core version)
// Block = one output row segment of 32 pixels; lane = pixel, warp w owns displacement rows
// tj = w, w+8, w+16 and all D column displacements.  Channel chunks of CK are staged in shared memory
// channel-major so lanes read consecutive words (no bank conflicts); the reference's separate
// NCHW->padded-NHWC repack pass (correlation_cuda_kernel.cu:47-70) does not exist here: zero padding
// is applied while staging.
constexpr int CK = 16;

template <typename T, int D, int S2>
__global__ void __launch_bounds__(256) correlation_kernel(vps::TV<const T> f1, vps::TV<const T> f2,
                                                          vps::TV<T> out, int act, float slope) {
  constexpr int R = (D - 1) / 2;
  constexpr int PW = 32 + (D - 1) * S2;
  constexpr int JT = (D + 7) / 8;
  extern __shared__ float sm[];
  float* f1s = sm;                 // [CK][32]
  float* f2s = sm + CK * 32;       // [CK][D][PW]
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int x0 = blockIdx.x * 32, y = blockIdx.y, n = blockIdx.z;
  const int H = f1.h, W = f1.w, C = f1.c;
  float acc[JT][D];
#pragma unroll
  for (int a = 0; a < JT; ++a)
#pragma unroll
    for (int b = 0; b < D; ++b) acc[a][b] = 0.f;

  for (int c0 = 0; c0 < C; c0 += CK) {
    // stage f1: 32 px x CK ch
    for (int i = threadIdx.x; i < 32 * CK; i += 256) {
      const int c = i % CK, px = i / CK;
      const int x = x0 + px;
      float v = 0.f;
      if (x < W && c0 + c < C) v = vps::ldf<T>(f1.p + f1.off(n, y, x) + c0 + c);
      f1s[c * 32 + px] = v;
    }
    // stage f2: D rows x PW px x CK ch
    for (int i = threadIdx.x; i < D * PW * CK; i += 256) {
      const int c = i % CK;
      const int t = i / CK;
      const int px = t % PW, row = t / PW;
      const int x = x0 + px - R * S2, yy = y + (row - R) * S2;
      float v = 0.f;
      if (x >= 0 && x < W && yy >= 0 && yy < H && c0 + c < C) v = vps::ldf<T>(f2.p + f2.off(n, yy, x) + c0 + c);
      f2s[(c * D + row) * PW + px] = v;
    }
    __syncthreads();
#pragma unroll 4
    for (int c = 0; c < CK; ++c) {
      const float a = f1s[c * 32 + lane];
#pragma unroll
      for (int jt = 0; jt < JT; ++jt) {
        const int tj = w + 8 * jt;
        if (tj < D) {
          const float* rowp = f2s + (c * D + tj) * PW + lane;
#pragma unroll
          for (int ti = 0; ti < D; ++ti) acc[jt][ti] = fmaf(a, rowp[ti * S2], acc[jt][ti]);
        }
      }
    }
    __syncthreads();
  }
  const int x = x0 + lane;
  if (x < W) {
    const float inv = 1.f / (float)C;
    T* op = out.p + out.off(n, y, x);
#pragma unroll
    for (int jt = 0; jt < JT; ++jt) {
      const int tj = w + 8 * jt;
      if (tj < D) {
#pragma unroll
        for (int ti = 0; ti < D; ++ti) {
          float v = acc[jt][ti] * inv;
          v = vps::apply_act(v, act, slope);
          vps::stf<T>(op + tj * D + ti, v);
        }
      }
    }
  }
}

template <typename T, int D, int S2>
int launch_corr(const vps_tensor* f1, const vps_tensor* f2, const vps_tensor* out, int act, float slope,
                cudaStream_t st) {
  constexpr int PW = 32 + (D - 1) * S2;
  const int smem = (CK * 32 + CK * D * PW) * 4;
  auto kern = correlation_kernel<T, D, S2>;
  if (smem > 48 * 1024) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) {
      vps::set_error("correlation: smem attr: %s", cudaGetErrorString(cudaGetLastError()));
      return VPS_E_CUDA;
    }
  }
  dim3 grid(vps::cdiv(f1->w, 32), f1->h, f1->n);
  kern<<<grid, 256, smem, st>>>(vps::tv<const T>(*f1), vps::tv<const T>(*f2), vps::tv<T>(*out), act, slope);
  VPS_CUDA_LAST("correlation_kernel");
  return VPS_OK;
}

// ------------------------------------------------------------------ resample2d
template <typename T, typename TF, int V>
__global__ void resample2d_kernel(vps::TV<const T> src, vps::TV<const TF> flow, vps::TV<T> out) {
  VPS_PIX_COORDS(out, V, c, x, y, n);
  const TF* fp = flow.p + flow.off(n, y, x);
  const float dx = vps::ldf<TF>(fp), dy = vps::ldf<TF>(fp + 1);
  const float xf = (float)x + dx, yf = (float)y + dy;
  const float alpha = xf - floorf(xf), beta = yf - floorf(yf);
  // border clamp of the tap coordinates, fractional weights NOT renormalised (resample2d_kernel.cu:44-52)
  const int xL = max(min((int)floorf(xf), src.w - 1), 0);
  const int xR = max(min((int)floorf(xf) + 1, src.w - 1), 0);
  const int yT = max(min((int)floorf(yf), src.h - 1), 0);
  const int yB = max(min((int)floorf(yf) + 1, src.h - 1), 0);
  float a[V], b[V], cc[V], d[V];
  vps::ldv<T, V>(src.p + src.off(n, yT, xL) + c, a);
  vps::ldv<T, V>(src.p + src.off(n, yT, xR) + c, b);
  vps::ldv<T, V>(src.p + src.off(n, yB, xL) + c, cc);
  vps::ldv<T, V>(src.p + src.off(n, yB, xR) + c, d);
#pragma unroll
  for (int j = 0; j < V; ++j) {
    float v = 0.f;
    v += (1.f - alpha) * (1.f - beta) * a[j];
    v += (alpha) * (1.f - beta) * b[j];
    v += (1.f - alpha) * (beta) * cc[j];
    v += (alpha) * (beta) * d[j];
    a[j] = v;
  }
  vps::stv<T, V>(out.p + out.off(n, y, x) + c, a);
}

// ------------------------------------------------------------------ channelnorm
template <typename T, typename TO>
__global__ void channelnorm_kernel(vps::TV<const T> a, vps::TV<const T> b, int has_b, vps::TV<TO> out,
                                   int64_t total) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % a.w);
    int64_t t = i / a.w;
    const int y = (int)(t % a.h);
    const int n = (int)(t / a.h);
    const T* ap = a.p + a.off(n, y, x);
    const T* bp = has_b ? b.p + b.off(n, y, x) : nullptr;
    float s = 0.f;
    for (int c = 0; c < a.c; ++c) {
      float v = vps::ldf<T>(ap + c);
      if (has_b) v -= vps::ldf<T>(bp + c);
      s += v * v;
    }
    vps::stf<TO>(out.p + out.off(n, y, x), sqrtf(s));
  }
}

}  // namespace

extern "C" int vps_correlation_tc(const vps_tensor* f1, const vps_tensor* f2, const vps_tensor* out, int pad, int max_disp,
                                  int stride1, int stride2, int act, float slope, void* stream);

extern "C" int vps_correlation_simt(const vps_tensor* f1, const vps_tensor* f2, const vps_tensor* out, int pad,
                                    int max_disp, int stride1, int stride2, int act, float slope, void* stream);

// dispatcher: bf16 features with C % 64 == 0 (<= 256) and 16-byte aligned views go to the tensor-core kernel
extern "C" int vps_correlation(const vps_tensor* f1, const vps_tensor* f2, const vps_tensor* out, int pad,
                               int max_disp, int stride1, int stride2, int act, float slope, void* stream) {
  const bool tc = f1->dtype == VPS_BF16 && f2->dtype == VPS_BF16 && f1->c % 64 == 0 && f1->c <= 256 && f1->cs % 8 == 0 &&
                  f2->cs % 8 == 0 && ((uintptr_t)f1->ptr & 15) == 0 && ((uintptr_t)f2->ptr & 15) == 0 && stride1 == 1 &&
                  pad == max_disp && ((max_disp == 20 && stride2 == 2) || (max_disp == 4 && stride2 == 1)) &&
                  (act == VPS_ACT_NONE || act == VPS_ACT_LRELU);
  if (tc) return vps_correlation_tc(f1, f2, out, pad, max_disp, stride1, stride2, act, slope, stream);
  return vps_correlation_simt(f1, f2, out, pad, max_disp, stride1, stride2, act, slope, stream);
}

extern "C" int vps_correlation_simt(const vps_tensor* f1, const vps_tensor* f2, const vps_tensor* out, int pad,
                                    int max_disp, int stride1, int stride2, int act, float slope, void* stream) {
  VPS_CHECK_ARG(stride1 == 1 && pad == max_disp, "correlation: only stride1=1, pad==max_displacement");
  VPS_CHECK_ARG(f1->dtype == f2->dtype && f1->dtype == out->dtype, "correlation: dtype mismatch");
  VPS_CHECK_ARG(f1->h == f2->h && f1->w == f2->w && f1->c == f2->c && out->h == f1->h && out->w == f1->w,
                "correlation: shape mismatch");
  const int R = max_disp / stride2, D = 2 * R + 1;
  VPS_CHECK_ARG(out->c == D * D, "correlation: out.c %d != %d", out->c, D * D);
  cudaStream_t st = (cudaStream_t)stream;
  if (D == 21 && stride2 == 2) {
    VPS_DISPATCH_T(f1->dtype, T, return (launch_corr<T, 21, 2>(f1, f2, out, act, slope, st)));
  } else if (D == 9 && stride2 == 1) {
    VPS_DISPATCH_T(f1->dtype, T, return (launch_corr<T, 9, 1>(f1, f2, out, act, slope, st)));
  }
  vps::set_error("correlation: unsupported (max_disp %d, stride2 %d)", max_disp, stride2);
  return VPS_E_ARG;
}

extern "C" int vps_resample2d(const vps_tensor* src, const vps_tensor* flow, const vps_tensor* out, void* stream) {
  VPS_CHECK_ARG(src->dtype == out->dtype && src->c == out->c && flow->c >= 2, "resample2d: bad args");
  VPS_CHECK_ARG(flow->h == out->h && flow->w == out->w, "resample2d: flow/out size");
  if (!((int64_t)out->n * out->h * out->w * out->c)) return VPS_OK;
  const bool vec = vps::vec_ok(*src, out->c) && vps::vec_ok(*out, out->c);
  VPS_DISPATCH_T(flow->dtype, TF, VPS_DISPATCH_V(out->dtype, vec, T, V,
      (resample2d_kernel<T, TF, V><<<vps::pix_grid(out->w, out->c / V, out->h, out->n), 256, 0, (cudaStream_t)stream>>>(
          vps::tv<const T>(*src), vps::tv<const TF>(*flow), vps::tv<T>(*out)))));
  VPS_CUDA_LAST("resample2d_kernel");
  return VPS_OK;
}

extern "C" int vps_channelnorm(const vps_tensor* a, const vps_tensor* b, const vps_tensor* out, void* stream) {
  VPS_CHECK_ARG(out->c == 1 && out->h == a->h && out->w == a->w, "channelnorm: out shape");
  if (b) VPS_CHECK_ARG(b->dtype == a->dtype && b->c == a->c && b->h == a->h && b->w == a->w, "channelnorm: b");
  const int64_t total = (int64_t)a->n * a->h * a->w;
  if (!total) return VPS_OK;
  vps_tensor bb = b ? *b : *a;
  VPS_DISPATCH_T(a->dtype, T, VPS_DISPATCH_T(out->dtype, TO,
      (channelnorm_kernel<T, TO><<<vps::grid_for(total), 256, 0, (cudaStream_t)stream>>>(
          vps::tv<const T>(*a), vps::tv<const T>(bb), b != nullptr, vps::tv<TO>(*out), total))));
  VPS_CUDA_LAST("channelnorm_kernel");
  return VPS_OK;
}

// ------------------------------------------------------------------ FlowNet2 input preparation
// compute_flow + FlowNet2.forward head (panoptic_fusetrack.py:119-121, flow_utils.py:5-10,
// flownet2.py:135-139): rgb = img*std + mean for both frames, per-channel mean over both frames and all
// pixels, x = (rgb - rgb_mean) / rgb_max, frames concatenated on channels (img0 -> 0..2, img1 -> 3..5).
namespace {
struct F3 { float v[3]; };

__global__ void flownet_sums_kernel(const float* __restrict__ img, const float* __restrict__ ref, int64_t hw, F3 std_, F3 mean_,
                                    double* __restrict__ sums) {
  const int c = blockIdx.y;
  double s = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < hw; i += (int64_t)gridDim.x * blockDim.x) {
    s += (double)(img[c * hw + i] * std_.v[c] + mean_.v[c]);
    s += (double)(ref[c * hw + i] * std_.v[c] + mean_.v[c]);
  }
  __shared__ double sh[32];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) atomicAdd(sums + c, s);
  }
}

template <typename T>
__global__ void flownet_input_kernel(const float* __restrict__ img, const float* __restrict__ ref, int64_t hw, F3 std_,
                                     F3 mean_, const double* __restrict__ sums, float rgb_max, vps::TV<T> x) {
  const int64_t total = hw * 6;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c6 = (int)(i % 6);
    const int64_t pix = i / 6;
    const int c = c6 % 3;
    const float* s = c6 < 3 ? img : ref;
    const float m = (float)(sums[c] / (double)(2 * hw));
    const float v = (s[c * hw + pix] * std_.v[c] + mean_.v[c] - m) / rgb_max;
    vps::stf<T>(x.p + pix * x.cs + c6, v);
  }
}
}  // namespace

extern "C" int vps_flownet_input(const float* img_nchw, const float* ref_nchw, int H, int W, const float* std3,
                                 const float* mean3, float rgb_max, double* sums_ws, const vps_tensor* x, void* stream) {
  VPS_CHECK_ARG(x->c == 6 && x->h == H && x->w == W && x->n == 1, "flownet_input: x must be [1,H,W,6]");
  cudaStream_t st = (cudaStream_t)stream;
  F3 s, m;
  for (int i = 0; i < 3; ++i) { s.v[i] = std3[i]; m.v[i] = mean3[i]; }
  const int64_t hw = (int64_t)H * W;
  cudaMemsetAsync(sums_ws, 0, 3 * sizeof(double), st);
  dim3 g1(148, 3);
  flownet_sums_kernel<<<g1, 256, 0, st>>>(img_nchw, ref_nchw, hw, s, m, sums_ws);
  VPS_CUDA_LAST("flownet_sums");
  VPS_DISPATCH_T(x->dtype, T, (flownet_input_kernel<T><<<vps::grid_for(hw * 6), 256, 0, st>>>(img_nchw, ref_nchw, hw, s, m,
                                                                                            sums_ws, rgb_max, vps::tv<T>(*x))));
  VPS_CUDA_LAST("flownet_input");
  return VPS_OK;
}

// ------------------------------------------------------------------ 2->2 channel flow up-sampler
// nn.ConvTranspose2d(2, 2, 4, 2, 1) -- `upsampled_flow*_to_*` of every FlowNet (FlowNetS.py:45-48 etc.).
// One thread per output pixel, both output channels; weights [ci][co][ky][kx] (torch IOHW) in registers.
namespace {
struct DeconvW { float w[2][2][4][4]; float b[2]; };

template <typename TI, typename TO>
__global__ void flow_deconv_kernel(vps::TV<const TI> x, vps::TV<TO> y, DeconvW W) {
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y, n = blockIdx.z;
  if (ox >= y.w) return;
  const int qy = oy >> 1, py = oy & 1, qx = ox >> 1, px = ox & 1;
  // out[2q+p]: p=0 -> (iy=q-1, ky=3), (iy=q, ky=1);  p=1 -> (iy=q, ky=2), (iy=q+1, ky=0)
  const int iy0 = py ? qy : qy - 1, ky0 = py ? 2 : 3, ky1 = py ? 0 : 1;
  const int ix0 = px ? qx : qx - 1, kx0 = px ? 2 : 3, kx1 = px ? 0 : 1;
  float acc0 = W.b[0], acc1 = W.b[1];
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    const int iy = iy0 + a, ky = a ? ky1 : ky0;
    if (iy < 0 || iy >= x.h) continue;
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int ix = ix0 + b, kx = b ? kx1 : kx0;
      if (ix < 0 || ix >= x.w) continue;
      const TI* xp = x.p + x.off(n, iy, ix);
      const float v0 = vps::ldf<TI>(xp), v1 = vps::ldf<TI>(xp + 1);
      acc0 += v0 * W.w[0][0][ky][kx] + v1 * W.w[1][0][ky][kx];
      acc1 += v0 * W.w[0][1][ky][kx] + v1 * W.w[1][1][ky][kx];
    }
  }
  TO* yp = y.p + y.off(n, oy, ox);
  vps::stf<TO>(yp, acc0);
  vps::stf<TO>(yp + 1, acc1);
}
}  // namespace

extern "C" int vps_flow_deconv(const vps_tensor* x, const float* w_iohw_host, const float* bias_host, const vps_tensor* y,
                               void* stream) {
  VPS_CHECK_ARG(x->c == 2 && y->c == 2 && y->h == 2 * x->h && y->w == 2 * x->w && y->n == x->n, "flow_deconv: shapes");
  DeconvW W;
  for (int i = 0; i < 64; ++i) (&W.w[0][0][0][0])[i] = w_iohw_host[i];
  W.b[0] = bias_host ? bias_host[0] : 0.f;
  W.b[1] = bias_host ? bias_host[1] : 0.f;
  dim3 grid(vps::cdiv(y->w, 128), y->h, y->n);
  VPS_DISPATCH_T(x->dtype, TI, VPS_DISPATCH_T(y->dtype, TO,
      (flow_deconv_kernel<TI, TO><<<grid, 128, 0, (cudaStream_t)stream>>>(vps::tv<const TI>(*x), vps::tv<TO>(*y), W))));
  VPS_CUDA_LAST("flow_deconv");
  return VPS_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Fused FlowNet2 glue.  Between its sub-networks FlowNet2 builds two concat inputs per pixel from 2-3 channel tensors
// (flownet2.py:142-153 and :176-189).  As separate ops that is 5 / 11 launches of scalar 2-byte traffic at full
// resolution; here ONE kernel per concat reads the pixel's inputs once and writes the whole 12 / 11-channel pixel.  The
// arithmetic (and every rounding to the storage type T) is the same as in resize_bilinear / resize_nearest / axpby /
// resample2d / channelnorm above and in pointwise.cu, expression by expression, so the results are bit-identical.
namespace {
template <typename T> __device__ __forceinline__ float round_T(float v);
template <> __device__ __forceinline__ float round_T<float>(float v) { return v; }
template <> __device__ __forceinline__ float round_T<__nv_bfloat16>(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

// resample2d of channels [c0, c0+3) of `src` at (x + dx, y + dy): border-clamped taps, weights not renormalised
template <typename T>
__device__ __forceinline__ void warp3(const vps::TV<const T>& src, int n, int x, int y, int c0, float dx, float dy, float (&o)[3]) {
  const float xf = (float)x + dx, yf = (float)y + dy;
  const float alpha = xf - floorf(xf), beta = yf - floorf(yf);
  const int xL = max(min((int)floorf(xf), src.w - 1), 0);
  const int xR = max(min((int)floorf(xf) + 1, src.w - 1), 0);
  const int yT = max(min((int)floorf(yf), src.h - 1), 0);
  const int yB = max(min((int)floorf(yf) + 1, src.h - 1), 0);
  const T* pa = src.p + src.off(n, yT, xL) + c0;
  const T* pb = src.p + src.off(n, yT, xR) + c0;
  const T* pc = src.p + src.off(n, yB, xL) + c0;
  const T* pd = src.p + src.off(n, yB, xR) + c0;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    float v = 0.f;
    v += (1.f - alpha) * (1.f - beta) * vps::ldf<T>(pa + j);
    v += (alpha) * (1.f - beta) * vps::ldf<T>(pb + j);
    v += (1.f - alpha) * (beta) * vps::ldf<T>(pc + j);
    v += (alpha) * (beta) * vps::ldf<T>(pd + j);
    o[j] = round_T<T>(v);                         // resample2d stores T
  }
}
template <typename T>
__device__ __forceinline__ void store_pixel(T* op, const float* v, int c, int cs_pad) {
  // whole-pixel store: c channels + zeroed padding up to cs_pad (the destination is a full buffer, never a slice)
  if (sizeof(T) == 2 && cs_pad % 8 == 0 && (((uintptr_t)op) & 15) == 0) {
    for (int g = 0; g < cs_pad / 8; ++g) {
      uint32_t pk[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int i0 = 8 * g + 2 * t;
        __nv_bfloat162 b = __floats2bfloat162_rn(i0 < c ? v[i0] : 0.f, i0 + 1 < c ? v[i0 + 1] : 0.f);
        pk[t] = *reinterpret_cast<uint32_t*>(&b);
      }
      *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(op) + 8 * g) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    }
  } else {
    for (int i = 0; i < c; ++i) vps::stf<T>(op + i, v[i]);
  }
}

// concat(x6, resample(img1, flow), flow / div_flow, |img0 - resampled|) with flow = bilinear-upsampled flow_lo * mul
template <typename T>
__global__ void __launch_bounds__(256) flownet_stage_kernel(vps::TV<const T> x6, vps::TV<const float> flow_lo, float mul, float inv,
                                                            vps::TV<T> cat, int cs_pad) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, n = blockIdx.z;
  if (x >= cat.w) return;
  // resize_bilinear (align_corners = False) of the 2-channel flow, times mul
  const float sy = (float)flow_lo.h / (float)cat.h, sx = (float)flow_lo.w / (float)cat.w;
  const float fy = fmaxf(sy * ((float)y + 0.5f) - 0.5f, 0.f);
  const float fx = fmaxf(sx * ((float)x + 0.5f) - 0.5f, 0.f);
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < flow_lo.h - 1 ? 1 : 0), x1 = x0 + (x0 < flow_lo.w - 1 ? 1 : 0);
  const float ly = fy - (float)y0, lx = fx - (float)x0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  const float* f00 = flow_lo.p + flow_lo.off(n, y0, x0);
  const float* f01 = flow_lo.p + flow_lo.off(n, y0, x1);
  const float* f10 = flow_lo.p + flow_lo.off(n, y1, x0);
  const float* f11 = flow_lo.p + flow_lo.off(n, y1, x1);
  float fl[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) fl[j] = vps_bilerp(f00[j], f01[j], f10[j], f11[j], hx, lx, hy, ly) * mul;
  float v[12];
  const T* xp = x6.p + x6.off(n, y, x);
#pragma unroll
  for (int j = 0; j < 6; ++j) v[j] = 1.0f * vps::ldf<T>(xp + j) + 0.f;     // copy_scale(x6, cat[..., 0:6]) = axpby: alpha * a + 0
  float wv[3];
  warp3<T>(x6, n, x, y, 3, fl[0], fl[1], wv);
#pragma unroll
  for (int j = 0; j < 3; ++j) v[6 + j] = wv[j];
  v[9] = inv * fl[0] + 0.f; v[10] = inv * fl[1] + 0.f;                       // copy_scale(flow, cat[..., 9:11], 1 / div_flow)
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < 3; ++j) { float d = vps::ldf<T>(xp + j); d -= wv[j]; s += d * d; }
  v[11] = sqrtf(s);                                                          // channelnorm(img0 - resampled)
  store_pixel<T>(cat.p + cat.off(n, y, x), v, 12, cs_pad);
}

// concat3 = (img0, sd_flow, s2_flow, |sd_flow|, |s2_flow|, |img0 - warp(img1, sd_flow)|, |img0 - warp(img1, s2_flow)|)
template <typename T>
__global__ void __launch_bounds__(256) flownet_cat3_kernel(vps::TV<const T> x6, vps::TV<const float> s2_lo, vps::TV<const float> sd_lo,
                                                           float mul_s2, float mul_sd, vps::TV<T> cat, int cs_pad) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, n = blockIdx.z;
  if (x >= cat.w) return;
  float s2[2], sd[2];
  {   // resize_nearest * mul of both low-resolution flows
    const float sy = (float)s2_lo.h / (float)cat.h, sx = (float)s2_lo.w / (float)cat.w;
    const int ys = min((int)floorf((float)y * sy), s2_lo.h - 1), xs = min((int)floorf((float)x * sx), s2_lo.w - 1);
    const float* p = s2_lo.p + s2_lo.off(n, ys, xs);
    s2[0] = p[0] * mul_s2 + 0.f; s2[1] = p[1] * mul_s2 + 0.f;
  }
  {
    const float sy = (float)sd_lo.h / (float)cat.h, sx = (float)sd_lo.w / (float)cat.w;
    const int ys = min((int)floorf((float)y * sy), sd_lo.h - 1), xs = min((int)floorf((float)x * sx), sd_lo.w - 1);
    const float* p = sd_lo.p + sd_lo.off(n, ys, xs);
    sd[0] = p[0] * mul_sd + 0.f; sd[1] = p[1] * mul_sd + 0.f;
  }
  float v[11];
  const T* xp = x6.p + x6.off(n, y, x);
#pragma unroll
  for (int j = 0; j < 3; ++j) v[j] = 1.0f * vps::ldf<T>(xp + j) + 0.f;
  v[3] = 1.0f * sd[0] + 0.f; v[4] = 1.0f * sd[1] + 0.f;
  v[5] = 1.0f * s2[0] + 0.f; v[6] = 1.0f * s2[1] + 0.f;
  {   // channelnorm of a 2-channel fp32 flow: the same accumulation loop as channelnorm_kernel
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int j = 0; j < 2; ++j) { const float p = sd[j]; a += p * p; const float q = s2[j]; b += q * q; }
    v[7] = sqrtf(a); v[8] = sqrtf(b);
  }
  float wv[3];
  warp3<T>(x6, n, x, y, 3, sd[0], sd[1], wv);
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < 3; ++j) { float d = vps::ldf<T>(xp + j); d -= wv[j]; s += d * d; }
  v[9] = sqrtf(s);
  warp3<T>(x6, n, x, y, 3, s2[0], s2[1], wv);
  s = 0.f;
#pragma unroll
  for (int j = 0; j < 3; ++j) { float d = vps::ldf<T>(xp + j); d -= wv[j]; s += d * d; }
  v[10] = sqrtf(s);
  store_pixel<T>(cat.p + cat.off(n, y, x), v, 11, cs_pad);
}
}  // namespace

static int cat_pad(const vps_tensor* cat) {      // channels a whole-pixel store may touch: only for a full (non-slice) buffer view
  return cat->cs;
}

extern "C" int vps_flownet_stage(const vps_tensor* x6, const vps_tensor* flow_lo, float mul, float inv, const vps_tensor* cat, void* stream) {
  VPS_CHECK_ARG(x6->c == 6 && flow_lo->c == 2 && flow_lo->dtype == VPS_F32 && cat->c == 12 && cat->dtype == x6->dtype &&
                    cat->h == x6->h && cat->w == x6->w && cat->n == x6->n && flow_lo->n == x6->n, "flownet_stage: shapes");
  if (!((int64_t)cat->n * cat->h * cat->w)) return VPS_OK;
  dim3 grid((unsigned)vps::cdiv(cat->w, 256), (unsigned)cat->h, (unsigned)cat->n);
  VPS_DISPATCH_T(cat->dtype, T,
                 (flownet_stage_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>(vps::tv<const T>(*x6), vps::tv<const float>(*flow_lo), mul,
                                                                                 inv, vps::tv<T>(*cat), cat_pad(cat))));
  VPS_CUDA_LAST("flownet_stage");
  return VPS_OK;
}

extern "C" int vps_flownet_cat3(const vps_tensor* x6, const vps_tensor* s2_flow_lo, const vps_tensor* sd_flow_lo, float mul_s2, float mul_sd,
                                const vps_tensor* cat, void* stream) {
  VPS_CHECK_ARG(x6->c == 6 && s2_flow_lo->c == 2 && sd_flow_lo->c == 2 && s2_flow_lo->dtype == VPS_F32 && sd_flow_lo->dtype == VPS_F32 &&
                    cat->c == 11 && cat->dtype == x6->dtype && cat->h == x6->h && cat->w == x6->w && cat->n == x6->n, "flownet_cat3: shapes");
  if (!((int64_t)cat->n * cat->h * cat->w)) return VPS_OK;
  dim3 grid((unsigned)vps::cdiv(cat->w, 256), (unsigned)cat->h, (unsigned)cat->n);
  VPS_DISPATCH_T(cat->dtype, T,
                 (flownet_cat3_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>(vps::tv<const T>(*x6), vps::tv<const float>(*s2_flow_lo),
                                                                                vps::tv<const float>(*sd_flow_lo), mul_s2, mul_sd,
                                                                                vps::tv<T>(*cat), cat_pad(cat))));
  VPS_CUDA_LAST("flownet_cat3");
  return VPS_OK;
}
