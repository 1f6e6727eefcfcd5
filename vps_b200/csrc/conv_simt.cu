// fp32-FMA direct convolution on CUDA cores: the parity-mode conv (bit-faithful fp32 accumulation,
// only the summation order differs from the oracle) and the path for layers too small/odd for the
// tensor-core kernel (2->2 ConvTranspose flow upsamplers, first layers when running fp32 storage).
// Same argument contract as vps_conv2d_tc; weights are f32 [kh][kw][cin][cout].
#include "common.cuh"

namespace {

struct ConvSimtParams {
  const void* x; int x_n, x_h, x_w, x_cs;
  void* y; int y_h, y_w, y_cs;
  const void* res; int res_cs; int res_after_act;
  const float* w; const float* bias;
  int kh, kw, sh, sw, ph, pw, oh, ow;
  int oy_mul, oy_off, ox_mul, ox_off;
  int cin, cout, act;
  float slope, out_scale;
  int64_t total_pix;
};

constexpr int TP = 64;   // pixels per block
constexpr int TC = 64;   // couts per block
constexpr int KC = 16;   // cin chunk

template <typename TI, typename TO, typename TR>
__global__ void __launch_bounds__(256) conv_simt_kernel(const ConvSimtParams p) {
  __shared__ float xs[KC][TP + 1];
  __shared__ float ws[KC][TC];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t pix0 = (int64_t)blockIdx.x * TP;
  const int co0 = blockIdx.y * TC;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  // loader assignments: x tile: thread -> (pixel lp = tid % 64, cin rows tid/64 + 4*i)
  const int lp = threadIdx.x & 63, lc = threadIdx.x >> 6;
  const int64_t lpix = pix0 + lp;
  int ln = 0, loy = 0, lox = 0;
  const bool lvalid = lpix < p.total_pix;
  if (lvalid) {
    ln = (int)(lpix / ((int64_t)p.oh * p.ow));
    const int rem = (int)(lpix - (int64_t)ln * p.oh * p.ow);
    loy = rem / p.ow; lox = rem - loy * p.ow;
  }
  const TI* xin = (const TI*)p.x;

  for (int r = 0; r < p.kh; ++r) {
    for (int s = 0; s < p.kw; ++s) {
      const int iy = loy * p.sh - p.ph + r, ix = lox * p.sw - p.pw + s;
      const bool inb = lvalid && iy >= 0 && iy < p.x_h && ix >= 0 && ix < p.x_w;
      const int64_t xoff = inb ? (((int64_t)ln * p.x_h + iy) * p.x_w + ix) * p.x_cs : 0;
      const float* wrs = p.w + (int64_t)(r * p.kw + s) * p.cin * p.cout;
      for (int c0 = 0; c0 < p.cin; c0 += KC) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int ci = c0 + lc + 4 * i;
          xs[lc + 4 * i][lp] = (inb && ci < p.cin) ? vps::ldf<TI>(xin + xoff + ci) : 0.f;
        }
        // w tile: thread -> (cout = tid % 64, cin rows tid/64 + 4*i)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int ci = c0 + lc + 4 * i, co = co0 + lp;
          ws[lc + 4 * i][lp] = (ci < p.cin && co < p.cout) ? __ldg(wrs + (int64_t)ci * p.cout + co) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < KC; ++k) {
          float xv[4], wv[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) xv[i] = xs[k][ty * 4 + i];
#pragma unroll
          for (int j = 0; j < 4; ++j) wv[j] = ws[k][tx * 4 + j];
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(xv[i], wv[j], acc[i][j]);
        }
        __syncthreads();
      }
    }
  }

  TO* yout = (TO*)p.y;
  const TR* rin = (const TR*)p.res;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t pix = pix0 + ty * 4 + i;
    if (pix >= p.total_pix) continue;
    const int n = (int)(pix / ((int64_t)p.oh * p.ow));
    const int rem = (int)(pix - (int64_t)n * p.oh * p.ow);
    const int oy = rem / p.ow, ox = rem - oy * p.ow;
    const int64_t opix = ((int64_t)n * p.y_h + oy * p.oy_mul + p.oy_off) * p.y_w + ox * p.ox_mul + p.ox_off;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int co = co0 + tx * 4 + j;
      if (co >= p.cout) continue;
      float v = acc[i][j];
      if (p.bias) v += __ldg(p.bias + co);
      float rv = 0.f;
      if (rin) rv = vps::ldf<TR>(rin + opix * p.res_cs + co);
      if (rin && !p.res_after_act) v += rv;
      v = vps::apply_act(v, p.act, p.slope) * p.out_scale;
      if (rin && p.res_after_act) v += rv;
      vps::stf<TO>(yout + opix * p.y_cs + co, v);
    }
  }
}

__global__ void pack_weights_simt_kernel(const float* __restrict__ src, const float* __restrict__ scale,
                                         float* __restrict__ dst, int cout, int cin, int kh, int kw,
                                         int transposed) {
  const int64_t total = (int64_t)cout * cin * kh * kw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int co = (int)(i % cout);
    int64_t t = i / cout;
    const int ci = (int)(t % cin); t /= cin;
    const int s = (int)(t % kw); t /= kw;
    const int r = (int)t;
    const int64_t si = transposed ? ((((int64_t)ci * cout + co) * kh + r) * kw + s)
                                  : ((((int64_t)co * cin + ci) * kh + r) * kw + s);
    float v = src[si];
    if (scale) v *= scale[co];
    dst[i] = v;
  }
}

}  // namespace

extern "C" int vps_pack_weights_simt(const float* w, const float* scale, float* dst, int cout, int cin, int kh,
                                     int kw, int transposed, void* stream) {
  const int64_t total = (int64_t)cout * cin * kh * kw;
  const int blocks = (int)((total + 255) / 256 > 4096 ? 4096 : (total + 255) / 256);
  pack_weights_simt_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, scale, dst, cout, cin, kh, kw, transposed);
  VPS_CUDA_LAST("pack_weights_simt");
  return VPS_OK;
}

extern "C" int vps_conv2d_simt(const vps_conv_args* a, void* stream) {
  VPS_CHECK_ARG(a->cin <= a->x.c, "conv2d_simt: cin %d > x.c %d", a->cin, a->x.c);
  VPS_CHECK_ARG((a->oh - 1) * a->oy_mul + a->oy_off < a->y.h && (a->ow - 1) * a->ox_mul + a->ox_off < a->y.w,
                "conv2d_simt: output mapping out of range");
  ConvSimtParams p;
  p.x = a->x.ptr; p.x_n = a->x.n; p.x_h = a->x.h; p.x_w = a->x.w; p.x_cs = a->x.cs;
  p.y = a->y.ptr; p.y_h = a->y.h; p.y_w = a->y.w; p.y_cs = a->y.cs;
  p.res = a->res.ptr; p.res_cs = a->res.cs; p.res_after_act = a->res_after_act;
  p.w = (const float*)a->w; p.bias = a->bias;
  p.kh = a->kh; p.kw = a->kw; p.sh = a->sh; p.sw = a->sw; p.ph = a->ph; p.pw = a->pw; p.oh = a->oh; p.ow = a->ow;
  p.oy_mul = a->oy_mul; p.oy_off = a->oy_off; p.ox_mul = a->ox_mul; p.ox_off = a->ox_off;
  p.cin = a->cin; p.cout = a->cout; p.act = a->act; p.slope = a->slope; p.out_scale = a->out_scale;
  p.total_pix = (int64_t)a->x.n * a->oh * a->ow;
  if (p.total_pix == 0) return VPS_OK;
  dim3 grid((unsigned)((p.total_pix + TP - 1) / TP), (unsigned)((a->cout + TC - 1) / TC));
  // without a residual the kernel never reads one: the fp32-residual instance runs
  VPS_DISPATCH_T(a->x.dtype, TI, VPS_DISPATCH_T(a->y.dtype, TO, VPS_DISPATCH_T(a->res.ptr ? a->res.dtype : VPS_F32, TR,
      (conv_simt_kernel<TI, TO, TR><<<grid, 256, 0, (cudaStream_t)stream>>>(p)))));
  VPS_CUDA_LAST("conv_simt_kernel");
  return VPS_OK;
}
