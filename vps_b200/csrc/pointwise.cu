// HBM-bound layout / pointwise / resampling kernels (NHWC, f32 or bf16 storage, fp32 math).
// One thread per output element with the channel index fastest => coalesced, 128-bit where the
// channel count allows.  Torch semantics are reproduced exactly where index arithmetic matters
// (align_corners=False bilinear, floor nearest, adaptive pooling windows).
#include <algorithm>

#include "common.cuh"

namespace {

template <typename TO>
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ src, vps::TV<TO> dst, int64_t total) {
  VPS_GRID_STRIDE(i, total) {
    VPS_DECOMP_NHWC(i, dst, n, y, x, c);
    vps::stf<TO>(dst.p + dst.off(n, y, x) + c, src[(((int64_t)n * dst.c + c) * dst.h + y) * dst.w + x]);
  }
}
template <typename TI>
__global__ void nhwc_to_nchw_kernel(vps::TV<const TI> src, float* __restrict__ dst, int64_t total) {
  VPS_GRID_STRIDE(i, total) {
    // iterate in NCHW order for coalesced writes
    const int x = (int)(i % src.w);
    int64_t t = i / src.w;
    const int y = (int)(t % src.h); t /= src.h;
    const int c = (int)(t % src.c);
    const int n = (int)(t / src.c);
    dst[i] = vps::ldf<TI>(src.p + src.off(n, y, x) + c);
  }
}

// All kernels below use the (x*chunks, y, n) pixel grid of vps::pix_grid: no 64-bit index division, and V
// consecutive channels (16 bytes) per thread when every tensor involved allows it (V = 1 otherwise).
template <typename TI, typename TO, int V>
__global__ void axpby_kernel(vps::TV<const TI> a, vps::TV<const TI> b, int has_b, vps::TV<TO> out, float alpha, float beta) {
  VPS_PIX_COORDS(out, V, c, x, y, n);
  float va[V], vb[V];
  vps::ldv<TI, V>(a.p + a.off(n, y, x) + c, va);
  if (has_b) vps::ldv<TI, V>(b.p + b.off(n, y, x) + c, vb);
#pragma unroll
  for (int j = 0; j < V; ++j) va[j] = alpha * va[j] + (has_b ? beta * vb[j] : 0.f);
  vps::stv<TO, V>(out.p + out.off(n, y, x) + c, va);
}

template <typename TI, typename TO, int V>
__global__ void resize_bilinear_kernel(vps::TV<const TI> src, vps::TV<TO> out, float sy, float sx, float mul) {
  VPS_PIX_COORDS(out, V, c, x, y, n);
  // area_pixel_compute_source_index(align_corners=False): max(scale*(dst+0.5)-0.5, 0)
  const float fy = fmaxf(sy * ((float)y + 0.5f) - 0.5f, 0.f);
  const float fx = fmaxf(sx * ((float)x + 0.5f) - 0.5f, 0.f);
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < src.h - 1 ? 1 : 0), x1 = x0 + (x0 < src.w - 1 ? 1 : 0);
  const float ly = fy - (float)y0, lx = fx - (float)x0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  float v00[V], v01[V], v10[V], v11[V];
  vps::ldv<TI, V>(src.p + src.off(n, y0, x0) + c, v00);
  vps::ldv<TI, V>(src.p + src.off(n, y0, x1) + c, v01);
  vps::ldv<TI, V>(src.p + src.off(n, y1, x0) + c, v10);
  vps::ldv<TI, V>(src.p + src.off(n, y1, x1) + c, v11);
#pragma unroll
  for (int j = 0; j < V; ++j) v00[j] = vps_bilerp(v00[j], v01[j], v10[j], v11[j], hx, lx, hy, ly) * mul;
  vps::stv<TO, V>(out.p + out.off(n, y, x) + c, v00);
}

template <typename TI, typename TO, int V>
__global__ void resize_nearest_kernel(vps::TV<const TI> src, vps::TV<TO> out, float sy, float sx, float mul, int accumulate) {
  VPS_PIX_COORDS(out, V, c, x, y, n);
  const int ys = min((int)floorf((float)y * sy), src.h - 1);
  const int xs = min((int)floorf((float)x * sx), src.w - 1);
  float v[V], o[V];
  vps::ldv<TI, V>(src.p + src.off(n, ys, xs) + c, v);
  TO* op = out.p + out.off(n, y, x) + c;
  if (accumulate) vps::ldv<TO, V>(op, o);
#pragma unroll
  for (int j = 0; j < V; ++j) v[j] = v[j] * mul + (accumulate ? o[j] : 0.f);
  vps::stv<TO, V>(op, v);
}

template <typename TI, typename TO, int V>
__global__ void pool2d_kernel(vps::TV<const TI> src, vps::TV<TO> out, int k, int s, int p, int is_avg) {
  VPS_PIX_COORDS(out, V, c, x, y, n);
  const int ys = y * s - p, xs = x * s - p;
  float acc[V];
#pragma unroll
  for (int j = 0; j < V; ++j) acc[j] = is_avg ? 0.f : -INFINITY;
  for (int r = 0; r < k; ++r) {
    const int yy = ys + r;
    if (yy < 0 || yy >= src.h) continue;
    for (int q = 0; q < k; ++q) {
      const int xx = xs + q;
      if (xx < 0 || xx >= src.w) continue;
      float v[V];
      vps::ldv<TI, V>(src.p + src.off(n, yy, xx) + c, v);
#pragma unroll
      for (int j = 0; j < V; ++j) acc[j] = is_avg ? acc[j] + v[j] : fmaxf(acc[j], v[j]);
    }
  }
  if (is_avg) {
#pragma unroll
    for (int j = 0; j < V; ++j) acc[j] /= (float)(k * k);   // count_include_pad=True (torch default, tcea_modules.py:28)
  }
  vps::stv<TO, V>(out.p + out.off(n, y, x) + c, acc);
}

// space-to-depth (block 2): y[n, Y, X, (dy*2+dx)*C + c] = x[n, 2Y+dy, 2X+dx, c]; out-of-range reads (odd sizes) are 0.
// Turns a stride-2 convolution over C channels into a stride-1 convolution over 4C channels (first layers).
template <typename TI, typename TO>
__global__ void space_to_depth2_kernel(vps::TV<const TI> x, vps::TV<TO> y) {
  VPS_PIX_COORDS(y, 1, k, X, Y, n);
  const int C = x.c;
  const int c = k % C, q = k / C;
  const int iy = 2 * Y + (q >> 1), ix = 2 * X + (q & 1);
  float v = 0.f;
  if (q < 4 && iy < x.h && ix < x.w) v = vps::ldf<TI>(x.p + x.off(n, iy, ix) + c);
  vps::stf<TO>(y.p + y.off(n, Y, X) + k, v);
}

// bf16 fast path: one thread assembles 8 consecutive output channels (scalar, L1-resident reads of the four source
// pixels) and writes them with one 16-byte store; the channel padding up to the pixel stride is written as zeros.
__global__ void space_to_depth2_bf16x8_kernel(vps::TV<const __nv_bfloat16> x, vps::TV<__nv_bfloat16> y) {
  const int chunks = y.cs / 8;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= y.w * chunks) return;
  const int k0 = (t % chunks) * 8, X = t / chunks, Y = blockIdx.y, n = blockIdx.z;
  const int C = x.c;
  int c = k0 % C, q = k0 / C;
  uint32_t pk[4];
#pragma unroll
  for (int j2 = 0; j2 < 4; ++j2) {
    unsigned short v[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int iy = 2 * Y + (q >> 1), ix = 2 * X + (q & 1);
      v[e] = 0;
      if (q < 4 && iy < x.h && ix < x.w) v[e] = *reinterpret_cast<const unsigned short*>(x.p + x.off(n, iy, ix) + c);
      if (++c == C) { c = 0; ++q; }
    }
    pk[j2] = (uint32_t)v[0] | ((uint32_t)v[1] << 16);
  }
  *reinterpret_cast<uint4*>(y.p + y.off(n, Y, X) + k0) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
}

// ---- GroupNorm: pass 1 = per-block partial statistics of every (n, group); pass 2 = one block per (n, group) merges them
// into mean / rstd; pass 3 = apply.  A thread keeps a running (count, mean, M2) in fp32 of x - shift, shift = the first value
// it reads: a constant group gives mean = shift and M2 = 0 exactly, and x - shift stays exact where the mean dwarfs the
// spread.  Partials are merged with Chan's formula in fp64 in a fixed order (no atomics), so the result does not depend on
// the order in which blocks finish.
struct GnPart {
  double n, mean, m2;
};

// a <- a merged with b (Chan et al.); an empty b leaves a as it is, an empty a becomes b
__device__ __forceinline__ void gn_merge(GnPart& a, const GnPart& b) {
  if (b.n == 0.0) return;
  const double n = a.n + b.n, d = b.mean - a.mean, w = b.n / n;
  a.mean += d * w;
  a.m2 += b.m2 + d * d * a.n * w;
  a.n = n;
}

// lane 0 <- the merge of the warp's 32 partials, as a fixed shuffle tree
__device__ __forceinline__ void gn_warp_merge(GnPart& p) {
  for (int o = 16; o > 0; o >>= 1) {
    GnPart q;
    q.n = __shfl_down_sync(0xffffffffu, p.n, o);
    q.mean = __shfl_down_sync(0xffffffffu, p.mean, o);
    q.m2 = __shfl_down_sync(0xffffffffu, p.m2, o);
    gn_merge(p, q);
  }
}

struct GnAcc {
  float shift, mean, m2;   // mean and M2 of x - shift
  int n;
  // merges a batch of k values (x - shift) with mean bm and M2 bm2 about bm
  __device__ __forceinline__ void push(int k, float bm, float bm2) {
    const int n1 = n + k;
    const float d = bm - mean, w = (float)k / (float)n1;
    mean = fmaf(d, w, mean);
    m2 += bm2 + d * d * (float)n * w;
    n = n1;
  }
  __device__ __forceinline__ GnPart part() const {
    GnPart p;
    p.n = n; p.mean = (double)shift + (double)mean; p.m2 = m2;
    return p;
  }
};

// scalar arm: grid (P, groups, n), block (p, g, n) strides over the group's elements and writes part[(n*groups + g)*P + p]
template <typename TI>
__global__ void __launch_bounds__(256) gn_stats_kernel(vps::TV<const TI> x, int groups, GnPart* __restrict__ part) {
  const int g = blockIdx.y, n = blockIdx.z;
  const int cg = x.c / groups;
  const int64_t npix = (int64_t)x.h * x.w;
  const int64_t total = npix * cg;
  GnAcc acc = {0.f, 0.f, 0.f, 0};
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % cg);
    const int64_t pix = i / cg;
    const float v = vps::ldf<TI>(x.p + ((int64_t)n * npix + pix) * x.cs + g * cg + c);
    if (acc.n == 0) acc.shift = v;
    acc.push(1, v - acc.shift, 0.f);
  }
  // fixed-order tree: shuffles within each warp, then over the warps' partials
  GnPart p = acc.part();
  gn_warp_merge(p);
  __shared__ GnPart sh[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) sh[w] = p;
  __syncthreads();
  if (w == 0) {
    p = lane < (blockDim.x >> 5) ? sh[lane] : GnPart{0.0, 0.0, 0.0};
    gn_warp_merge(p);
    if (lane == 0) part[((int64_t)n * groups + g) * gridDim.x + blockIdx.x] = p;
  }
}

// vector arm: a thread owns one 16-byte channel chunk (V channels of one group, or of two when TWO: V == 2 * cg) and strides
// over pixels, so a warp reads whole pixels (fully coalesced).  block = (C/V chunks) x (256*V/C pixel rows); grid (P, 1, n):
// each block merges its rows per chunk, then its chunks per group, and writes part[(n*groups + g)*P + blockIdx.x].
template <typename TI, int V, bool TWO>
__global__ void __launch_bounds__(256) gn_stats_vec_kernel(vps::TV<const TI> x, int groups, GnPart* __restrict__ part) {
  constexpr int S = TWO ? 2 : 1, VS = V / S;   // groups per chunk, channels per (chunk, group)
  const int chunks = x.c / V;
  const int rows = blockDim.x / chunks;
  const int ch = threadIdx.x % chunks, row = threadIdx.x / chunks;
  const int n = blockIdx.z;
  const int64_t npix = (int64_t)x.h * x.w;
  GnAcc acc[S];
#pragma unroll
  for (int s = 0; s < S; ++s) acc[s] = GnAcc{0.f, 0.f, 0.f, 0};
  // 4 independent 16-byte loads in flight per thread (one was latency bound: 1.7 TB/s on an L2/HBM-resident map)
  constexpr int U = 4;
  const int64_t stride = (int64_t)gridDim.x * rows;
  for (int64_t pix = (int64_t)blockIdx.x * rows + row; pix < npix; pix += U * stride) {
    float v[U][V];
    int k = 0;                                       // loads in range: a prefix of the U
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t q = pix + u * stride;
      if (q < npix) {
        vps::ldv<TI, V>(x.p + ((int64_t)n * npix + q) * x.cs + ch * V, v[u]);
        ++k;
      } else {
#pragma unroll
        for (int j = 0; j < V; ++j) v[u][j] = 0.f;
      }
    }
#pragma unroll
    for (int s = 0; s < S; ++s) {
      if (acc[s].n == 0) acc[s].shift = v[0][s * VS];
      float sum = 0.f;
#pragma unroll
      for (int u = 0; u < U; ++u) {
#pragma unroll
        for (int j = s * VS; j < (s + 1) * VS; ++j) {
          v[u][j] -= acc[s].shift;
          if (u < k) sum += v[u][j];
        }
      }
      const int cnt = k * VS;
      const float bm = sum / (float)cnt;
      float bm2 = 0.f;
#pragma unroll
      for (int u = 0; u < U; ++u) {
#pragma unroll
        for (int j = s * VS; j < (s + 1) * VS; ++j) {
          const float e = v[u][j] - bm;
          if (u < k) bm2 = fmaf(e, e, bm2);
        }
      }
      acc[s].push(cnt, bm, bm2);
    }
  }
  __shared__ GnPart sh[256][S];
#pragma unroll
  for (int s = 0; s < S; ++s) sh[threadIdx.x][s] = acc[s].part();
  __syncthreads();
  if (row == 0) {
#pragma unroll
    for (int s = 0; s < S; ++s) {
      GnPart a = sh[ch][s];
      for (int r = 1; r < rows; ++r) gn_merge(a, sh[r * chunks + ch][s]);
      sh[ch][s] = a;
    }
  }
  __syncthreads();
  const int g = threadIdx.x;
  if (g < groups) {
    GnPart a;
    if constexpr (TWO) {
      a = sh[g / 2][g % 2];
    } else {
      const int per = x.c / groups / V;             // chunks per group
      a = sh[g * per][0];
      for (int i = 1; i < per; ++i) gn_merge(a, sh[g * per + i][0]);
    }
    part[((int64_t)n * groups + g) * gridDim.x + blockIdx.x] = a;
  }
}

// grid (groups, n): merges the P partials of one (n, group) in a fixed order; mean and rstd are each rounded once to fp32
__global__ void __launch_bounds__(128) gn_finalize_kernel(const GnPart* __restrict__ part, int P, float eps,
                                                          float2* __restrict__ stats) {
  const int64_t ng = (int64_t)blockIdx.y * gridDim.x + blockIdx.x;
  GnPart a = {0.0, 0.0, 0.0};
  for (int p = threadIdx.x; p < P; p += blockDim.x) gn_merge(a, part[ng * P + p]);
  __shared__ GnPart sh[128];
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int s = 64; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      a = sh[threadIdx.x];
      gn_merge(a, sh[threadIdx.x + s]);
      sh[threadIdx.x] = a;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double var = fmax(a.m2 / a.n, 0.0);       // biased, clamped at 0 as torch does
    stats[ng] = make_float2((float)a.mean, (float)(1.0 / sqrt(var + (double)eps)));
  }
}

constexpr int GN_MAX_C = 1024;
// the group's mean / rstd are copied per channel into shared memory once per block, so the element loop needs no group
// index; per-element global loads of gamma / beta made this kernel LSU-bound
template <typename TI, typename TO, int V>
__global__ void gn_apply_kernel(vps::TV<const TI> x, vps::TV<TO> y, const float2* __restrict__ stats,
                                const float* __restrict__ gamma, const float* __restrict__ beta, int groups, int relu) {
  __shared__ float s_mean[GN_MAX_C], s_rstd[GN_MAX_C], s_gamma[GN_MAX_C], s_beta[GN_MAX_C];
  const int cg = x.c / groups;
  const float2* st = stats + (int64_t)blockIdx.z * groups;      // pix_grid: z = image index
  for (int c = threadIdx.x; c < x.c; c += blockDim.x) {
    const float2 mr = st[c / cg];
    s_mean[c] = mr.x; s_rstd[c] = mr.y; s_gamma[c] = gamma[c]; s_beta[c] = beta[c];
  }
  __syncthreads();
  VPS_PIX_COORDS(y, V, c, xx, yy, n);
  float v[V];
  vps::ldv<TI, V>(x.p + x.off(n, yy, xx) + c, v);
#pragma unroll
  for (int j = 0; j < V; ++j) {
    const float o = (v[j] - s_mean[c + j]) * s_rstd[c + j] * s_gamma[c + j] + s_beta[c + j];
    v[j] = relu ? fmaxf(o, 0.f) : o;
  }
  vps::stv<TO, V>(y.p + y.off(n, yy, xx) + c, v);
}

template <typename TI, typename TO>
__global__ void im2col_kernel(vps::TV<const TI> x, vps::TV<TO> cols, int kh, int kw, int sh, int sw, int ph, int pw,
                              int64_t total) {
  const int kk = kh * kw * x.c;
  VPS_GRID_STRIDE(i, total) {
    VPS_DECOMP_NHWC(i, cols, n, oy, ox, k);
    float v = 0.f;
    if (k < kk) {
      const int ci = k % x.c;
      const int rs = k / x.c;
      const int s = rs % kw, r = rs / kw;
      const int iy = oy * sh - ph + r, ix = ox * sw - pw + s;
      if (iy >= 0 && iy < x.h && ix >= 0 && ix < x.w) v = vps::ldf<TI>(x.p + x.off(n, iy, ix) + ci);
    }
    vps::stf<TO>(cols.p + cols.off(n, oy, ox) + k, v);
  }
}

// bf16 fast path: one thread = one output pixel x 8 consecutive k (one 16-byte store); (r,s,ci) is decomposed once
// with 32-bit arithmetic and then incremented.
__global__ void im2col_bf16x8_kernel(vps::TV<const __nv_bfloat16> x, vps::TV<__nv_bfloat16> cols, int kh, int kw, int sh,
                                     int sw, int ph, int pw, int chunks, int64_t total) {
  const int kk = kh * kw * x.c;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % chunks);
    const int64_t pix = i / chunks;
    const int ox = (int)(pix % cols.w);
    const int64_t t = pix / cols.w;
    const int oy = (int)(t % cols.h), n = (int)(t / cols.h);
    int k = ch * 8;
    int ci = k % x.c;
    int rs = k / x.c;
    int s = rs % kw, r = rs / kw;
    __align__(16) __nv_bfloat16 v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float f = 0.f;
      if (k < kk) {
        const int iy = oy * sh - ph + r, ix = ox * sw - pw + s;
        if (iy >= 0 && iy < x.h && ix >= 0 && ix < x.w) f = __bfloat162float(x.p[x.off(n, iy, ix) + ci]);
      }
      v[j] = __float2bfloat16_rn(f);
      ++k;
      if (++ci == x.c) { ci = 0; if (++s == kw) { s = 0; ++r; } }
    }
    *(uint4*)(cols.p + pix * cols.cs + ch * 8) = *(const uint4*)v;
  }
}

template <typename TI>
__global__ void sigmoid_flat_kernel_t(vps::TV<const TI> src, float* __restrict__ dst, int64_t total) {
  VPS_GRID_STRIDE(i, total) {
    VPS_DECOMP_NHWC(i, src, n, y, x, c);
    const float v = vps::ldf<TI>(src.p + src.off(n, y, x) + c);
    dst[i] = 1.f / (1.f + expf(-v));
  }
}

}  // namespace

extern "C" int vps_nchw_to_nhwc(const float* src, const vps_tensor* dst, void* stream) {
  const int64_t total = (int64_t)dst->n * dst->h * dst->w * dst->c;
  if (!total) return VPS_OK;
  VPS_DISPATCH_T(dst->dtype, TO,
                 (nchw_to_nhwc_kernel<TO><<<vps::grid_for(total), 256, 0, (cudaStream_t)stream>>>(src, vps::tv<TO>(*dst), total)));
  VPS_CUDA_LAST("nchw_to_nhwc");
  return VPS_OK;
}
extern "C" int vps_nhwc_to_nchw(const vps_tensor* src, float* dst, void* stream) {
  const int64_t total = (int64_t)src->n * src->h * src->w * src->c;
  if (!total) return VPS_OK;
  VPS_DISPATCH_T(src->dtype, TI,
                 (nhwc_to_nchw_kernel<TI><<<vps::grid_for(total), 256, 0, (cudaStream_t)stream>>>(vps::tv<const TI>(*src), dst, total)));
  VPS_CUDA_LAST("nhwc_to_nchw");
  return VPS_OK;
}
extern "C" int vps_axpby(const vps_tensor* a, const vps_tensor* b, const vps_tensor* out, float alpha, float beta,
                         void* stream) {
  VPS_CHECK_ARG(a->h == out->h && a->w == out->w && a->c >= out->c && a->n == out->n, "axpby: shape");
  if (b) VPS_CHECK_ARG(b->dtype == a->dtype && b->h == out->h && b->w == out->w && b->c >= out->c, "axpby: b");
  if (!((int64_t)out->n * out->h * out->w * out->c)) return VPS_OK;
  const vps_tensor bb = b ? *b : *a;
  const bool vec = vps::vec_ok(*a, out->c) && vps::vec_ok(bb, out->c) && vps::vec_ok(*out, out->c);
  VPS_DISPATCH_IN_OUT_V(a->dtype, out->dtype, vec, TI, TO, V,
                        (axpby_kernel<TI, TO, V><<<vps::pix_grid(out->w, out->c / V, out->h, out->n), 256, 0, (cudaStream_t)stream>>>(
                            vps::tv<const TI>(*a), vps::tv<const TI>(bb), b != nullptr, vps::tv<TO>(*out), alpha, beta)));
  VPS_CUDA_LAST("axpby");
  return VPS_OK;
}
extern "C" int vps_copy_scale(const vps_tensor* src, const vps_tensor* dst, float alpha, void* stream) {
  return vps_axpby(src, nullptr, dst, alpha, 0.f, stream);
}
extern "C" int vps_resize_bilinear(const vps_tensor* src, const vps_tensor* out, float mul, void* stream) {
  VPS_CHECK_ARG(src->c >= out->c && src->n == out->n, "resize_bilinear: shape");
  if (!((int64_t)out->n * out->h * out->w * out->c)) return VPS_OK;
  const float sy = (float)src->h / (float)out->h, sx = (float)src->w / (float)out->w;
  const bool vec = vps::vec_ok(*src, out->c) && vps::vec_ok(*out, out->c);
  VPS_DISPATCH_IN_OUT_V(src->dtype, out->dtype, vec, TI, TO, V,
                        (resize_bilinear_kernel<TI, TO, V><<<vps::pix_grid(out->w, out->c / V, out->h, out->n), 256, 0, (cudaStream_t)stream>>>(
                            vps::tv<const TI>(*src), vps::tv<TO>(*out), sy, sx, mul)));
  VPS_CUDA_LAST("resize_bilinear");
  return VPS_OK;
}
extern "C" int vps_resize_nearest(const vps_tensor* src, const vps_tensor* out, float mul, int accumulate,
                                  void* stream) {
  VPS_CHECK_ARG(src->c >= out->c && src->n == out->n, "resize_nearest: shape");
  if (!((int64_t)out->n * out->h * out->w * out->c)) return VPS_OK;
  const float sy = (float)src->h / (float)out->h, sx = (float)src->w / (float)out->w;
  const bool vec = vps::vec_ok(*src, out->c) && vps::vec_ok(*out, out->c);
  VPS_DISPATCH_IN_OUT_V(src->dtype, out->dtype, vec, TI, TO, V,
                        (resize_nearest_kernel<TI, TO, V><<<vps::pix_grid(out->w, out->c / V, out->h, out->n), 256, 0, (cudaStream_t)stream>>>(
                            vps::tv<const TI>(*src), vps::tv<TO>(*out), sy, sx, mul, accumulate)));
  VPS_CUDA_LAST("resize_nearest");
  return VPS_OK;
}
extern "C" int vps_pool2d(const vps_tensor* src, const vps_tensor* out, int k, int s, int p, int is_avg,
                          void* stream) {
  VPS_CHECK_ARG(src->c >= out->c && src->n == out->n, "pool2d: shape");
  VPS_CHECK_ARG(out->h == (src->h + 2 * p - k) / s + 1 && out->w == (src->w + 2 * p - k) / s + 1, "pool2d: out size");
  if (!((int64_t)out->n * out->h * out->w * out->c)) return VPS_OK;
  const bool vec = vps::vec_ok(*src, out->c) && vps::vec_ok(*out, out->c);
  VPS_DISPATCH_IN_OUT_V(src->dtype, out->dtype, vec, TI, TO, V,
                        (pool2d_kernel<TI, TO, V><<<vps::pix_grid(out->w, out->c / V, out->h, out->n), 256, 0, (cudaStream_t)stream>>>(
                            vps::tv<const TI>(*src), vps::tv<TO>(*out), k, s, p, is_avg)));
  VPS_CUDA_LAST("pool2d");
  return VPS_OK;
}

// statistics scratch: a ring of slots, one per call, so GroupNorm calls on parallel streams / graph branches never share one.
// A slot holds the block partials of every (n, group) and their merged (mean, rstd).
namespace {
constexpr int GN_SLOTS = 16, GN_MAX_NG = 2048, GN_SLOT_PARTS = 32768;
struct GnSlot {
  GnPart part[GN_SLOT_PARTS];
  float2 stats[GN_MAX_NG];
};
GnSlot* g_gn_ring = nullptr;
unsigned g_gn_next = 0;
}  // namespace

extern "C" int vps_groupnorm(const vps_tensor* x, const vps_tensor* y, const float* gamma, const float* beta,
                             int groups, float eps, int relu, void* stream) {
  VPS_CHECK_ARG(groups >= 1 && groups <= 64 && x->c <= GN_MAX_C, "groupnorm: groups %d not in [1, 64] or c %d > %d", groups, x->c, GN_MAX_C);
  VPS_CHECK_ARG(x->c % groups == 0 && x->c == y->c && x->h == y->h && x->w == y->w && x->n == y->n, "groupnorm: shape");
  const int64_t ng = (int64_t)x->n * groups;
  VPS_CHECK_ARG(ng <= GN_MAX_NG, "groupnorm: n * groups too large (%lld)", (long long)ng);
  const int64_t total = (int64_t)x->n * x->h * x->w * x->c;
  if (!total) return VPS_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (!g_gn_ring && cudaMalloc(&g_gn_ring, sizeof(GnSlot) * GN_SLOTS) != cudaSuccess) {
    vps::set_error("groupnorm: malloc");
    return VPS_E_CUDA;
  }
  GnSlot* slot = g_gn_ring + g_gn_next++ % GN_SLOTS;
  const int max_parts = (int)(GN_SLOT_PARTS / ng);    // partials per (n, group) the slot has room for (>= 16)
  const int cg = x->c / groups;
  int P;
  VPS_DISPATCH_T(x->dtype, TI, {
    constexpr int V = vps::VecW<TI>::value;
    const int chunks = x->c / V;
    if (vps::vec_ok(*x, x->c) && chunks <= 256 && 256 % chunks == 0 && (cg % V == 0 || V == 2 * cg)) {
      const int rows = 256 / chunks;
      int64_t slices = ((int64_t)x->h * x->w + rows * 32 - 1) / (rows * 32);
      if (slices > 148 * 4) slices = 148 * 4;
      P = (int)std::min<int64_t>(slices, max_parts);
      const dim3 grid((unsigned)P, 1, x->n);
      if (V == 2 * cg) gn_stats_vec_kernel<TI, V, true><<<grid, 256, 0, st>>>(vps::tv<const TI>(*x), groups, slot->part);
      else gn_stats_vec_kernel<TI, V, false><<<grid, 256, 0, st>>>(vps::tv<const TI>(*x), groups, slot->part);
    } else {
      const int64_t per_group = (int64_t)x->h * x->w * cg;
      P = (int)std::min<int64_t>(std::min<int64_t>((per_group + 256 * 32 - 1) / (256 * 32), 64), max_parts);
      gn_stats_kernel<TI><<<dim3(P, groups, x->n), 256, 0, st>>>(vps::tv<const TI>(*x), groups, slot->part);
    }
  });
  VPS_CUDA_LAST("gn_stats");
  gn_finalize_kernel<<<dim3(groups, x->n), 128, 0, st>>>(slot->part, P, eps, slot->stats);
  VPS_CUDA_LAST("gn_finalize");
  const bool vec = vps::vec_ok(*x, x->c) && vps::vec_ok(*y, x->c);
  VPS_DISPATCH_IN_OUT_V(x->dtype, y->dtype, vec, TI, TO, V,
                        (gn_apply_kernel<TI, TO, V><<<vps::pix_grid(y->w, y->c / V, y->h, y->n), 256, 0, st>>>(
                            vps::tv<const TI>(*x), vps::tv<TO>(*y), slot->stats, gamma, beta, groups, relu)));
  VPS_CUDA_LAST("gn_apply");
  return VPS_OK;
}

extern "C" int vps_im2col(const vps_tensor* x, const vps_tensor* cols, int kh, int kw, int sh, int sw, int ph, int pw,
                          void* stream) {
  VPS_CHECK_ARG(cols->c >= kh * kw * x->c, "im2col: cols.c %d < %d", cols->c, kh * kw * x->c);
  const int64_t total = (int64_t)cols->n * cols->h * cols->w * cols->c;
  if (!total) return VPS_OK;
  if (x->dtype == VPS_BF16 && cols->dtype == VPS_BF16 && cols->c % 8 == 0 && cols->cs % 8 == 0 &&
      ((uintptr_t)cols->ptr & 15) == 0) {
    const int chunks = cols->c / 8;
    const int64_t tot8 = total / 8;
    int64_t blocks = (tot8 + 255) / 256;
    if (blocks > 148 * 64) blocks = 148 * 64;
    im2col_bf16x8_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(vps::tv<const __nv_bfloat16>(*x),
                                                                        vps::tv<__nv_bfloat16>(*cols), kh, kw, sh, sw, ph,
                                                                        pw, chunks, tot8);
    VPS_CUDA_LAST("im2col_bf16x8");
    return VPS_OK;
  }
  VPS_DISPATCH_T(x->dtype, TI, VPS_DISPATCH_T(cols->dtype, TO,
      (im2col_kernel<TI, TO><<<vps::grid_for(total), 256, 0, (cudaStream_t)stream>>>(
          vps::tv<const TI>(*x), vps::tv<TO>(*cols), kh, kw, sh, sw, ph, pw, total))));
  VPS_CUDA_LAST("im2col");
  return VPS_OK;
}

// RPN objectness: sigmoid of an NHWC score map flattened to the reference's (h, w, anchor) order
// (rpn_head.py:69-72).
extern "C" int vps_sigmoid_flat(const vps_tensor* t, float* dst, void* stream) {
  const int64_t total = (int64_t)t->n * t->h * t->w * t->c;
  if (!total) return VPS_OK;
  VPS_DISPATCH_T(t->dtype, TI,
                 (sigmoid_flat_kernel_t<TI><<<vps::grid_for(total), 256, 0, (cudaStream_t)stream>>>(vps::tv<const TI>(*t), dst, total)));
  VPS_CUDA_LAST("sigmoid_flat");
  return VPS_OK;
}

extern "C" int vps_space_to_depth2(const vps_tensor* x, const vps_tensor* y, void* stream) {
  VPS_CHECK_ARG(y->c == 4 * x->c && y->h == (x->h + 1) / 2 && y->w == (x->w + 1) / 2 && y->n == x->n, "space_to_depth2: shapes");
  if (!((int64_t)y->n * y->h * y->w * y->c)) return VPS_OK;
  if (x->dtype == VPS_BF16 && y->dtype == VPS_BF16 && y->cs % 8 == 0 && ((uintptr_t)y->ptr & 15) == 0 && y->cs >= y->c) {
    space_to_depth2_bf16x8_kernel<<<vps::pix_grid(y->w, y->cs / 8, y->h, y->n), 256, 0, (cudaStream_t)stream>>>(
        vps::tv<const __nv_bfloat16>(*x), vps::tv<__nv_bfloat16>(*y));
    VPS_CUDA_LAST("space_to_depth2");
    return VPS_OK;
  }
  VPS_DISPATCH_T(x->dtype, TI, VPS_DISPATCH_T(y->dtype, TO,
      (space_to_depth2_kernel<TI, TO><<<vps::pix_grid(y->w, y->c, y->h, y->n), 256, 0, (cudaStream_t)stream>>>(
          vps::tv<const TI>(*x), vps::tv<TO>(*y)))));
  VPS_CUDA_LAST("space_to_depth2");
  return VPS_OK;
}

// ---------------------------------------------------------------- input stage (SURVEY 8f rank 4): Normalize + Pad + to-tensor
// What the reference's test pipeline does on the host between LoadImageFromFile and the model for img and ref_img
// (mmdet/datasets/pipelines/transforms.py:295-318 Normalize -> mmcv.imnormalize: float32(img), BGR->RGB, (img - mean) / std;
// :238-270 Pad(size_divisor=32) -> zero pad bottom / right; formating.py:46-68 ImageToTensor: HWC -> CHW): one pass from the
// uint8 HWC BGR frame to the fp32 NCHW padded tensor simple_test takes.  (x - mean) / std with IEEE fp32 subtract and divide:
// bit-identical to numpy's float32 arithmetic.  Uploading uint8 frames cuts the host->device bytes of a pair from 50 MB to 12.6 MB.
namespace {
__global__ void preprocess_u8_kernel(const uint8_t* __restrict__ src, int h, int w, float m0, float m1, float m2, float s0, float s1,
                                     float s2, int to_rgb, float* __restrict__ out, int hp, int wp) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= wp) return;
  float v0 = 0.f, v1 = 0.f, v2 = 0.f;                     // pad_val = 0 (after normalisation, as in the reference: Pad follows Normalize)
  if (y < h && x < w) {
    const uint8_t* p = src + ((int64_t)y * w + x) * 3;
    const float b = (float)p[0], g = (float)p[1], r = (float)p[2];
    const float c0 = to_rgb ? r : b, c2 = to_rgb ? b : r;
    v0 = __fdiv_rn(__fsub_rn(c0, m0), s0);
    v1 = __fdiv_rn(__fsub_rn(g, m1), s1);
    v2 = __fdiv_rn(__fsub_rn(c2, m2), s2);
  }
  const int64_t plane = (int64_t)hp * wp, o = (int64_t)y * wp + x;
  out[o] = v0; out[plane + o] = v1; out[2 * plane + o] = v2;
}
}  // namespace

extern "C" int vps_preprocess_u8(const uint8_t* bgr_hwc, int h, int w, const float* mean3, const float* std3, int to_rgb,
                                 float* out_nchw, int hp, int wp, void* stream) {
  VPS_CHECK_ARG(h > 0 && w > 0 && hp >= h && wp >= w, "preprocess_u8: shapes %dx%d -> %dx%d", h, w, hp, wp);
  dim3 grid((unsigned)((wp + 255) / 256), (unsigned)hp);
  preprocess_u8_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(bgr_hwc, h, w, mean3[0], mean3[1], mean3[2], std3[0], std3[1], std3[2],
                                                              to_rgb, out_nchw, hp, wp);
  VPS_CUDA_LAST("preprocess_u8");
  return VPS_OK;
}

// Resize(img_scale, keep_ratio) of the same pipeline (transforms.py:107-121: mmcv.imrescale -> cv2.resize(..., INTER_LINEAR)
// on the uint8 frame) fused in front of Normalize + Pad + ImageToTensor.  OpenCV's fixed-point bilinear path for uint8,
// bit for bit; the taps are computed here, so there is no per-shape host table or upload and the stage stays capturable:
//   per axis: scale = 1 / (dst / src) (double); f = (float)((d + 0.5) * scale - 0.5); s = floor(f); f -= s (float);
//   x: f = 0 where s < 0 (s = 0) or s >= src - 1 (s = src - 1), second tap min(s + 1, src - 1);
//   y: f kept, both rows clamped to [0, src - 1];   a1 = rint(f * 2048), a0 = rint((1 - f) * 2048) (half to even);
//   R = S[s0] * a0 + S[s1] * a1 per row; out = clamp((((R0 >> 4) * b0 >> 16) + ((R1 >> 4) * b1 >> 16) + 2) >> 2, 0, 255)
// (the vertical arithmetic of OpenCV's SIMD VResizeLinearVec_32s8u, which cv2 uses for every column).  Explicitly rounded
// double operations keep nvcc from contracting (d + 0.5) * scale - 0.5 into an FMA, which would change f.
namespace {
struct LinearTap {
  int s0, s1, a0, a1;
};
__device__ __forceinline__ LinearTap linear_tap(int d, int src, double scale, bool clamp_frac) {
  float f = __double2float_rn(__dadd_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), -0.5));
  int s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  if (clamp_frac) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= src - 1) { f = 0.f; s = src - 1; }
  }
  LinearTap t;
  t.s0 = min(max(s, 0), src - 1);
  t.s1 = min(max(s + 1, 0), src - 1);
  t.a1 = __float2int_rn(__fmul_rn(f, 2048.f));
  t.a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  return t;
}

// grid (cdiv(wp, 256), hp): one thread per output pixel of the padded tensor; source bytes are read one at a time, so any
// alignment of the frame works (neighbouring threads share most of their taps, which L1 serves)
__global__ void preprocess_resize_u8_kernel(const uint8_t* __restrict__ src, int h, int w, int oh, int ow, double sy, double sx,
                                            float m0, float m1, float m2, float s0, float s1, float s2, int to_rgb,
                                            float* __restrict__ out, int hp, int wp) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= wp) return;
  float v0 = 0.f, v1 = 0.f, v2 = 0.f;                     // pad_val = 0 after normalisation
  if (y < oh && x < ow) {
    const LinearTap tx = linear_tap(x, w, sx, true), ty = linear_tap(y, h, sy, false);
    const uint8_t* r0 = src + (int64_t)ty.s0 * w * 3;
    const uint8_t* r1 = src + (int64_t)ty.s1 * w * 3;
    float c[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int R0 = (int)r0[tx.s0 * 3 + k] * tx.a0 + (int)r0[tx.s1 * 3 + k] * tx.a1;
      const int R1 = (int)r1[tx.s0 * 3 + k] * tx.a0 + (int)r1[tx.s1 * 3 + k] * tx.a1;
      const int t = (((R0 >> 4) * ty.a0) >> 16) + (((R1 >> 4) * ty.a1) >> 16);
      c[k] = (float)min(max((t + 2) >> 2, 0), 255);
    }
    const float c0 = to_rgb ? c[2] : c[0], c2 = to_rgb ? c[0] : c[2];
    v0 = __fdiv_rn(__fsub_rn(c0, m0), s0);
    v1 = __fdiv_rn(__fsub_rn(c[1], m1), s1);
    v2 = __fdiv_rn(__fsub_rn(c2, m2), s2);
  }
  const int64_t plane = (int64_t)hp * wp, o = (int64_t)y * wp + x;
  out[o] = v0; out[plane + o] = v1; out[2 * plane + o] = v2;
}
}  // namespace

extern "C" int vps_preprocess_resize_u8(const uint8_t* bgr_hwc, int h, int w, int oh, int ow, const float* mean3,
                                        const float* std3, int to_rgb, float* out_nchw, int hp, int wp, void* stream) {
  VPS_CHECK_ARG(h > 0 && w > 0 && oh > 0 && ow > 0 && hp >= oh && wp >= ow, "preprocess_resize_u8: shapes %dx%d -> %dx%d -> %dx%d",
                h, w, oh, ow, hp, wp);
  const double sy = 1.0 / ((double)oh / (double)h), sx = 1.0 / ((double)ow / (double)w);     // cv2: scale = 1 / inv_scale
  dim3 grid((unsigned)((wp + 255) / 256), (unsigned)hp);
  preprocess_resize_u8_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(bgr_hwc, h, w, oh, ow, sy, sx, mean3[0], mean3[1], mean3[2],
                                                                     std3[0], std3[1], std3[2], to_rgb, out_nchw, hp, wp);
  VPS_CUDA_LAST("preprocess_resize_u8");
  return VPS_OK;
}

// ---------------------------------------------------------------- 3x3 convolutions with <= 3 output channels (predict_flow)
// FlowNet2's predict_flow layers (submodules.py:27-28: Conv2d(cin, 2, 3, 1, 1), 19 launches per pair) have K = 9*cin up to
// 9234 but N = 2: as implicit GEMMs they cost one K step per (tap, 32 channels) at any N.  They run as a 1x1 tensor-core
// convolution with the taps moved to the output-channel axis, z[p][t*cout+co] = sum_c x[p][c] * w[co][c][t] (9x fewer K
// steps, the input is read once instead of once per tap), followed by this gather:
//     out[n,y,x,co] = act(bias[co] + sum_t z[n, y + t/3 - 1, x + t%3 - 1, t*cout + co]) * out_scale    (zero outside the map)
namespace {
template <int CO>
__global__ void tap_gather3x3_kernel(vps::TV<const float> z, vps::TV<float> out, const float* __restrict__ bias, int act, float slope,
                                     float out_scale) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, n = blockIdx.z;
  if (x >= out.w) return;
  float acc[CO];
#pragma unroll
  for (int c = 0; c < CO; ++c) acc[c] = 0.f;
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
    if (yy < 0 || yy >= z.h || xx < 0 || xx >= z.w) continue;
    const float* zp = z.p + z.off(n, yy, xx) + t * CO;
#pragma unroll
    for (int c = 0; c < CO; ++c) acc[c] += __ldg(zp + c);
  }
  float* op = out.p + out.off(n, y, x);
#pragma unroll
  for (int c = 0; c < CO; ++c) {
    float v = acc[c];
    if (bias) v += __ldg(bias + c);
    op[c] = vps::apply_act(v, act, slope) * out_scale;
  }
}
}  // namespace

extern "C" int vps_tap_gather3x3(const vps_tensor* z, const vps_tensor* out, const float* bias, int act, float slope,
                                 float out_scale, void* stream) {
  VPS_CHECK_ARG(z->dtype == VPS_F32 && out->dtype == VPS_F32, "tap_gather3x3: fp32 tensors");
  VPS_CHECK_ARG(out->c >= 1 && out->c <= 3 && z->c == 9 * out->c, "tap_gather3x3: z.c %d != 9 * out.c %d", z->c, out->c);
  VPS_CHECK_ARG(z->n == out->n && z->h == out->h && z->w == out->w, "tap_gather3x3: shapes");
  if (!((int64_t)out->n * out->h * out->w)) return VPS_OK;
  dim3 grid((unsigned)vps::cdiv(out->w, 128), (unsigned)out->h, (unsigned)out->n);
  cudaStream_t st = (cudaStream_t)stream;
  if (out->c == 1) tap_gather3x3_kernel<1><<<grid, 128, 0, st>>>(vps::tv<const float>(*z), vps::tv<float>(*out), bias, act, slope, out_scale);
  else if (out->c == 2) tap_gather3x3_kernel<2><<<grid, 128, 0, st>>>(vps::tv<const float>(*z), vps::tv<float>(*out), bias, act, slope, out_scale);
  else tap_gather3x3_kernel<3><<<grid, 128, 0, st>>>(vps::tv<const float>(*z), vps::tv<float>(*out), bias, act, slope, out_scale);
  VPS_CUDA_LAST("tap_gather3x3");
  return VPS_OK;
}
