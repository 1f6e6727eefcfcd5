// BFPTcea / UPSNetFPN memory-bound kernels: BFP gather & scatter, flow warp (grid_sample),
// TCEA temporal attention + combine, deformable im2col.  NHWC, fp32 math.
#include "common.cuh"

namespace {

constexpr int MAXLEV = 8;
template <typename T>
struct Levels {
  vps::TV<const T> l[MAXLEV];
  int n;
};

// bfp_tcea.py:96-109 with refine_level 0: every level nearest-resized to level-0 size, summed in level
// order, divided by the level count -- one pass, the five resized maps are never materialised.
template <typename T, int V>
__global__ void bfp_gather_kernel(Levels<T> lv, vps::TV<T> out) {
  VPS_PIX_COORDS(out, V, c, x, y, n);
  float s[V];
  for (int k = 0; k < lv.n; ++k) {
    const vps::TV<const T>& L = lv.l[k];
    const float sy = (float)L.h / (float)out.h, sx = (float)L.w / (float)out.w;
    const int ys = min((int)floorf((float)y * sy), L.h - 1);
    const int xs = min((int)floorf((float)x * sx), L.w - 1);
    float v[V];
    vps::ldv<T, V>(L.p + L.off(n, ys, xs) + c, v);
#pragma unroll
    for (int j = 0; j < V; ++j) s[j] = (k == 0) ? v[j] : s[j] + v[j];
  }
#pragma unroll
  for (int j = 0; j < V; ++j) s[j] /= (float)lv.n;
  vps::stv<T, V>(out.p + out.off(n, y, x) + c, s);
}

// bfp_tcea.py:141-147: adaptive_max_pool2d(bsf, size_i) + inputs[i]
template <typename T, int V>
__global__ void bfp_scatter_kernel(vps::TV<const T> bsf, vps::TV<const T> in, vps::TV<T> out) {
  VPS_PIX_COORDS(out, V, c, x, y, n);
  // adaptive pooling window: [floor(i*in/out), ceil((i+1)*in/out))
  const int y0 = (int)(((int64_t)y * bsf.h) / out.h), y1 = (int)((((int64_t)(y + 1)) * bsf.h + out.h - 1) / out.h);
  const int x0 = (int)(((int64_t)x * bsf.w) / out.w), x1 = (int)((((int64_t)(x + 1)) * bsf.w + out.w - 1) / out.w);
  float m[V], v[V];
#pragma unroll
  for (int j = 0; j < V; ++j) m[j] = -INFINITY;
  for (int yy = y0; yy < y1; ++yy)
    for (int xx = x0; xx < x1; ++xx) {
      vps::ldv<T, V>(bsf.p + bsf.off(n, yy, xx) + c, v);
#pragma unroll
      for (int j = 0; j < V; ++j) m[j] = fmaxf(m[j], v[j]);
    }
  vps::ldv<T, V>(in.p + in.off(n, y, x) + c, v);
#pragma unroll
  for (int j = 0; j < V; ++j) m[j] += v[j];
  vps::stv<T, V>(out.p + out.off(n, y, x) + c, m);
}

// torch.linspace(-1, 1, steps)[i] as the CPU kernel computes it (symmetric halves)
__device__ __forceinline__ float linspace_m1p1(int i, int steps) {
  const float step = 2.0f / (float)(steps - 1);
  return (i < steps / 2) ? (-1.0f + step * (float)i) : (1.0f - step * (float)(steps - i - 1));
}

// WarpingLayer (flow_modules.py:126-148) = grid_sample(bilinear, zeros, align_corners=False)
template <typename T, typename TF, int V>
__global__ void flow_warp_kernel(vps::TV<const T> src, vps::TV<const TF> flow, vps::TV<T> out) {
  const int H = src.h, W = src.w;
  VPS_PIX_COORDS(out, V, c, x, y, n);
  const TF* fp = flow.p + flow.off(n, y, x);
  const float gx = linspace_m1p1(x, W) + vps::ldf<TF>(fp) / (((float)flow.w - 1.0f) / 2.0f);
  const float gy = linspace_m1p1(y, H) + vps::ldf<TF>(fp + 1) / (((float)flow.h - 1.0f) / 2.0f);
  const float ix = ((gx + 1.f) * (float)W - 1.f) / 2.f;
  const float iy = ((gy + 1.f) * (float)H - 1.f) / 2.f;
  const int x0 = (int)floorf(ix), y0 = (int)floorf(iy), x1 = x0 + 1, y1 = y0 + 1;
  const float wts[4] = {((float)x1 - ix) * ((float)y1 - iy), (ix - (float)x0) * ((float)y1 - iy),
                        ((float)x1 - ix) * (iy - (float)y0), (ix - (float)x0) * (iy - (float)y0)};
  const int xs[4] = {x0, x1, x0, x1}, ys[4] = {y0, y0, y1, y1};
  float acc[V], v[V];
#pragma unroll
  for (int j = 0; j < V; ++j) acc[j] = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (xs[q] < 0 || xs[q] >= W || ys[q] < 0 || ys[q] >= H) continue;
    vps::ldv<T, V>(src.p + src.off(n, ys[q], xs[q]) + c, v);
#pragma unroll
    for (int j = 0; j < V; ++j) acc[j] += v[j] * wts[q];
  }
  vps::stv<T, V>(out.p + out.off(n, y, x) + c, acc);
}

// tcea_modules.py:52-61: one warp per pixel; out[:, 0:C] = fea0 * sigmoid(<emb0, emb_ref>), out[:, C:2C] = fea1 * ...
template <typename T, int V>
__global__ void tcea_temporal_kernel(vps::TV<const T> fea0, vps::TV<const T> fea1, vps::TV<const T> emb0,
                                     vps::TV<const T> emb1, vps::TV<const T> embr, vps::TV<T> out, int64_t npix) {
  // a lane owns V consecutive channels (16-byte vectors when V > 1): one warp-wide load covers 32*V channels of a pixel
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int C = fea0.c;
  for (int64_t pix = warp; pix < npix; pix += nwarps) {
    const int x = (int)(pix % fea0.w);
    const int64_t t = pix / fea0.w;
    const int y = (int)(t % fea0.h), n = (int)(t / fea0.h);
    const T* e0 = emb0.p + emb0.off(n, y, x);
    const T* e1 = emb1.p + emb1.off(n, y, x);
    const T* er = embr.p + embr.off(n, y, x);
    float d0 = 0.f, d1 = 0.f;
    for (int c = lane * V; c < C; c += 32 * V) {
      float r[V], a[V], b[V];
      vps::ldv<T, V>(er + c, r);
      vps::ldv<T, V>(e0 + c, a);
      vps::ldv<T, V>(e1 + c, b);
#pragma unroll
      for (int j = 0; j < V; ++j) { d0 += a[j] * r[j]; d1 += b[j] * r[j]; }
    }
    for (int o = 16; o > 0; o >>= 1) { d0 += __shfl_xor_sync(0xffffffffu, d0, o); d1 += __shfl_xor_sync(0xffffffffu, d1, o); }
    const float p0 = 1.f / (1.f + expf(-d0)), p1 = 1.f / (1.f + expf(-d1));
    const T* f0 = fea0.p + fea0.off(n, y, x);
    const T* f1 = fea1.p + fea1.off(n, y, x);
    T* op = out.p + out.off(n, y, x);
    for (int c = lane * V; c < C; c += 32 * V) {
      float a[V], b[V];
      vps::ldv<T, V>(f0 + c, a);
      vps::ldv<T, V>(f1 + c, b);
#pragma unroll
      for (int j = 0; j < V; ++j) { a[j] *= p0; b[j] *= p1; }
      vps::stv<T, V>(op + c, a);
      vps::stv<T, V>(op + C + c, b);
    }
  }
}

// tcea_modules.py:75-77: fea * sigmoid(att) * 2 + att_add
template <typename T, int V>
__global__ void tcea_combine_kernel(vps::TV<const T> fea, vps::TV<const T> att, vps::TV<const T> add, vps::TV<T> out) {
  VPS_PIX_COORDS(out, V, c, x, y, n);
  float f[V], a[V], d[V];
  vps::ldv<T, V>(fea.p + fea.off(n, y, x) + c, f);
  vps::ldv<T, V>(att.p + att.off(n, y, x) + c, a);
  vps::ldv<T, V>(add.p + add.off(n, y, x) + c, d);
#pragma unroll
  for (int j = 0; j < V; ++j) f[j] = f[j] * (1.f / (1.f + expf(-a[j]))) * 2.f + d[j];
  vps::stv<T, V>(out.p + out.off(n, y, x) + c, f);
}

// deformable_im2col (deform_conv_cuda_kernel.cu:83-113,189-242), 3x3 s1 p1 d1, deformable_group 1.
// cols[n,y,x, k*C + c]: the sampled value of input channel c at tap k; consumed by the GEMM as a 1x1 conv.
template <typename T, typename TOF>
__global__ void deform_im2col_kernel(vps::TV<const T> x, vps::TV<const TOF> off, vps::TV<T> cols, int64_t total) {
  const int C = x.c, H = x.h, W = x.w;
  VPS_GRID_STRIDE(i, total) {
    const int c = (int)(i % C);
    int64_t t = i / C;
    const int k = (int)(t % 9); t /= 9;
    const int xo = (int)(t % W); t /= W;
    const int yo = (int)(t % H);
    const int n = (int)(t / H);
    const TOF* op = off.p + off.off(n, yo, xo);
    const float oh = vps::ldf<TOF>(op + 2 * k), ow = vps::ldf<TOF>(op + 2 * k + 1);
    const float h = (float)(yo - 1 + k / 3) + oh;
    const float w = (float)(xo - 1 + k % 3) + ow;
    float val = 0.f;
    if (h > -1.f && w > -1.f && h < (float)H && w < (float)W) {
      const int hl = (int)floorf(h), wl = (int)floorf(w);
      const int hh_ = hl + 1, wh_ = wl + 1;
      const float lh = h - (float)hl, lw = w - (float)wl;
      const float hh = 1.f - lh, hw = 1.f - lw;
      float v1 = 0.f, v2 = 0.f, v3 = 0.f, v4 = 0.f;
      if (hl >= 0 && wl >= 0) v1 = vps::ldf<T>(x.p + x.off(n, hl, wl) + c);
      if (hl >= 0 && wh_ <= W - 1) v2 = vps::ldf<T>(x.p + x.off(n, hl, wh_) + c);
      if (hh_ <= H - 1 && wl >= 0) v3 = vps::ldf<T>(x.p + x.off(n, hh_, wl) + c);
      if (hh_ <= H - 1 && wh_ <= W - 1) v4 = vps::ldf<T>(x.p + x.off(n, hh_, wh_) + c);
      val = hh * hw * v1 + hh * lw * v2 + lh * hw * v3 + lh * lw * v4;
    }
    vps::stf<T>(cols.p + cols.off(n, yo, xo) + k * C + c, val);
  }
}

// bf16 fast path: thread = (pixel, tap, 8 channels): offsets / bilinear weights once per thread, four 16-byte gathers,
// one 16-byte store.
template <typename TOF>
__global__ void deform_im2col_bf16x8_kernel(vps::TV<const __nv_bfloat16> x, vps::TV<const TOF> off,
                                            vps::TV<__nv_bfloat16> cols, int64_t total) {
  const int C = x.c, H = x.h, W = x.w;
  const uint32_t C8 = (uint32_t)x.c / 8u;
  // 32-bit index arithmetic (host guarantees total < 2^31): 64-bit div/mod chains were the whole cost of this kernel
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < (uint32_t)total; i += gridDim.x * blockDim.x) {
    const uint32_t c8 = i % C8;
    uint32_t t = i / C8;
    const int k = (int)(t % 9u); t /= 9u;
    const int xo = (int)(t % (uint32_t)W); t /= (uint32_t)W;
    const int yo = (int)(t % (uint32_t)H);
    const int n = (int)(t / (uint32_t)H);
    const TOF* op = off.p + off.off(n, yo, xo);
    const float oh = vps::ldf<TOF>(op + 2 * k), ow = vps::ldf<TOF>(op + 2 * k + 1);
    const float h = (float)(yo - 1 + k / 3) + oh;
    const float w = (float)(xo - 1 + k % 3) + ow;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    if (h > -1.f && w > -1.f && h < (float)H && w < (float)W) {
      const int hl = (int)floorf(h), wl = (int)floorf(w);
      const int hh_ = hl + 1, wh_ = wl + 1;
      const float lh = h - (float)hl, lw = w - (float)wl;
      const float hh = 1.f - lh, hw = 1.f - lw;
      const float wts[4] = {hh * hw, hh * lw, lh * hw, lh * lw};
      const int ys[4] = {hl, hl, hh_, hh_}, xs[4] = {wl, wh_, wl, wh_};
      const bool ok[4] = {hl >= 0 && wl >= 0, hl >= 0 && wh_ <= W - 1, hh_ <= H - 1 && wl >= 0, hh_ <= H - 1 && wh_ <= W - 1};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (!ok[q]) continue;
        const uint4 raw = *(const uint4*)(x.p + x.off(n, ys[q], xs[q]) + c8 * 8);
        const __nv_bfloat162* b2 = (const __nv_bfloat162*)&raw;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __bfloat1622float2(b2[j]);
          acc[2 * j] += wts[q] * f.x;
          acc[2 * j + 1] += wts[q] * f.y;
        }
      }
    }
    uint4 o;
    __nv_bfloat162* o2 = (__nv_bfloat162*)&o;
#pragma unroll
    for (int j = 0; j < 4; ++j) o2[j] = __floats2bfloat162_rn(acc[2 * j], acc[2 * j + 1]);
    *(uint4*)(cols.p + cols.off(n, yo, xo) + k * C + c8 * 8) = o;
  }
}

}  // namespace

extern "C" int vps_bfp_gather(const vps_tensor* levels, int nlev, const vps_tensor* out, void* stream) {
  VPS_CHECK_ARG(nlev >= 1 && nlev <= MAXLEV, "bfp_gather: nlev");
  if (!((int64_t)out->n * out->h * out->w * out->c)) return VPS_OK;
  bool vec = vps::vec_ok(*out, out->c);
  for (int i = 0; i < nlev; ++i) {
    VPS_CHECK_ARG(levels[i].dtype == out->dtype && levels[i].c >= out->c, "bfp_gather: level %d", i);
    vec = vec && vps::vec_ok(levels[i], out->c);
  }
  VPS_DISPATCH_V(out->dtype, vec, T, V, {
    Levels<T> lv; lv.n = nlev;
    for (int i = 0; i < nlev; ++i) lv.l[i] = vps::tv<const T>(levels[i]);
    bfp_gather_kernel<T, V><<<vps::pix_grid(out->w, out->c / V, out->h, out->n), 256, 0, (cudaStream_t)stream>>>(lv, vps::tv<T>(*out));
  });
  VPS_CUDA_LAST("bfp_gather");
  return VPS_OK;
}

extern "C" int vps_bfp_scatter(const vps_tensor* bsf, const vps_tensor* in, const vps_tensor* out, void* stream) {
  VPS_CHECK_ARG(in->h == out->h && in->w == out->w && bsf->dtype == out->dtype && in->dtype == out->dtype, "bfp_scatter: args");
  if (!((int64_t)out->n * out->h * out->w * out->c)) return VPS_OK;
  const bool vec = vps::vec_ok(*bsf, out->c) && vps::vec_ok(*in, out->c) && vps::vec_ok(*out, out->c);
  VPS_DISPATCH_V(out->dtype, vec, T, V,
                 (bfp_scatter_kernel<T, V><<<vps::pix_grid(out->w, out->c / V, out->h, out->n), 256, 0, (cudaStream_t)stream>>>(
                     vps::tv<const T>(*bsf), vps::tv<const T>(*in), vps::tv<T>(*out))));
  VPS_CUDA_LAST("bfp_scatter");
  return VPS_OK;
}

extern "C" int vps_flow_warp(const vps_tensor* src, const vps_tensor* flow, const vps_tensor* out, void* stream) {
  VPS_CHECK_ARG(src->dtype == out->dtype && flow->h == out->h && flow->w == out->w && src->h == out->h && src->w == out->w,
                "flow_warp: args");
  if (!((int64_t)out->n * out->h * out->w * out->c)) return VPS_OK;
  const bool vec = vps::vec_ok(*src, out->c) && vps::vec_ok(*out, out->c);
  VPS_DISPATCH_T(flow->dtype, TF, VPS_DISPATCH_V(out->dtype, vec, T, V,
      (flow_warp_kernel<T, TF, V><<<vps::pix_grid(out->w, out->c / V, out->h, out->n), 256, 0, (cudaStream_t)stream>>>(
          vps::tv<const T>(*src), vps::tv<const TF>(*flow), vps::tv<T>(*out)))));
  VPS_CUDA_LAST("flow_warp");
  return VPS_OK;
}

extern "C" int vps_tcea_temporal(const vps_tensor* fea0, const vps_tensor* fea1, const vps_tensor* emb0,
                                 const vps_tensor* emb1, const vps_tensor* emb_ref, const vps_tensor* out, void* stream) {
  VPS_CHECK_ARG(out->c == 2 * fea0->c && fea1->c == fea0->c && emb0->c == emb_ref->c && emb1->c == emb_ref->c, "tcea_temporal: channels");
  VPS_CHECK_ARG(fea0->dtype == out->dtype && fea1->dtype == out->dtype && emb0->dtype == out->dtype &&
                    emb1->dtype == out->dtype && emb_ref->dtype == out->dtype, "tcea_temporal: dtype");
  const int64_t npix = (int64_t)out->n * out->h * out->w;
  if (!npix) return VPS_OK;
  const int C = fea0->c;
  const bool vec = vps::vec_ok(*fea0, C) && vps::vec_ok(*fea1, C) && vps::vec_ok(*emb0, C) && vps::vec_ok(*emb1, C) &&
                   vps::vec_ok(*emb_ref, C) && vps::vec_ok(*out, 2 * C);
  VPS_DISPATCH_V(out->dtype, vec, T, V,
                 (tcea_temporal_kernel<T, V><<<vps::grid_for(npix * 32), 256, 0, (cudaStream_t)stream>>>(
                     vps::tv<const T>(*fea0), vps::tv<const T>(*fea1), vps::tv<const T>(*emb0), vps::tv<const T>(*emb1),
                     vps::tv<const T>(*emb_ref), vps::tv<T>(*out), npix)));
  VPS_CUDA_LAST("tcea_temporal");
  return VPS_OK;
}

extern "C" int vps_tcea_combine(const vps_tensor* fea, const vps_tensor* att, const vps_tensor* att_add,
                                const vps_tensor* out, void* stream) {
  VPS_CHECK_ARG(fea->dtype == out->dtype && att->dtype == out->dtype && att_add->dtype == out->dtype, "tcea_combine: dtype");
  if (!((int64_t)out->n * out->h * out->w * out->c)) return VPS_OK;
  const bool vec = vps::vec_ok(*fea, out->c) && vps::vec_ok(*att, out->c) && vps::vec_ok(*att_add, out->c) && vps::vec_ok(*out, out->c);
  VPS_DISPATCH_V(out->dtype, vec, T, V,
                 (tcea_combine_kernel<T, V><<<vps::pix_grid(out->w, out->c / V, out->h, out->n), 256, 0, (cudaStream_t)stream>>>(
                     vps::tv<const T>(*fea), vps::tv<const T>(*att), vps::tv<const T>(*att_add), vps::tv<T>(*out))));
  VPS_CUDA_LAST("tcea_combine");
  return VPS_OK;
}

extern "C" int vps_deform_im2col(const vps_tensor* x, const vps_tensor* offset, const vps_tensor* cols, void* stream) {
  VPS_CHECK_ARG(offset->c >= 18 && cols->c == 9 * x->c && cols->dtype == x->dtype && cols->h == x->h && cols->w == x->w,
                "deform_im2col: args");
  const int64_t total = (int64_t)x->n * x->h * x->w * 9 * x->c;
  if (!total) return VPS_OK;
  if (x->dtype == VPS_BF16 && x->c % 8 == 0 && x->cs % 8 == 0 && cols->cs % 8 == 0 && ((uintptr_t)x->ptr & 15) == 0 &&
      ((uintptr_t)cols->ptr & 15) == 0) {
    const int64_t tot8 = total / 8;
    VPS_CHECK_ARG(tot8 < (1ll << 31) - (148ll * 64 * 256), "deform_im2col: tensor too large for 32-bit indexing");
    int64_t blocks = (tot8 + 255) / 256;
    if (blocks > 148 * 64) blocks = 148 * 64;
    VPS_DISPATCH_T(offset->dtype, TOF,
                   (deform_im2col_bf16x8_kernel<TOF><<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(
                       vps::tv<const __nv_bfloat16>(*x), vps::tv<const TOF>(*offset), vps::tv<__nv_bfloat16>(*cols), tot8)));
    VPS_CUDA_LAST("deform_im2col_bf16x8");
    return VPS_OK;
  }
  VPS_DISPATCH_T(x->dtype, T, VPS_DISPATCH_T(offset->dtype, TOF,
      (deform_im2col_kernel<T, TOF><<<vps::grid_for(total), 256, 0, (cudaStream_t)stream>>>(
          vps::tv<const T>(*x), vps::tv<const TOF>(*offset), vps::tv<T>(*cols), total))));
  VPS_CUDA_LAST("deform_im2col");
  return VPS_OK;
}
