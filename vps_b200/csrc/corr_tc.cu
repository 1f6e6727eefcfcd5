// Correlation (cost volume) on Hopper tensor cores (wgmma) -- the FlowNetC (pad 20, d 20, s2 2 -> 441 ch) and
// LiteFlowNetCorr (pad 4, d 4, s2 1 -> 81 ch) call sites of correlation_cuda.forward
// (correlation_cuda.cc:10-87, correlation_cuda_kernel.cu:74-147), bf16 features, fp32 accumulation.
//
// Banded GEMM:  D[n, m] = sum_c f2[n, c] * f1[m, c]
//   m = one of 96 output pixels of a TH x TW tile (pixels of ONE stride2-parity class, so that every needed f2
//       pixel has the same parity and element-strided TMA boxes fetch exactly the useful pixels),
//   n = f2 pixels of the tile's displacement neighbourhood, (TH + 2R) rows x 32 columns, 4 rows (128 pixels) per block;
//       each consumer warpgroup multiplies 2 of those rows (M = 64, N = 96, K = 16).
// Accumulator element (n, m) is output pixel m = (i, j) at displacement (tj, ti) = (i' - i, j' - j) for the
// neighbourhood pixel n = (i', j'); the band is stored straight from the register fragments.
//
//   warp 0         : TMA producer (f1 tile resident & double-buffered per tile; f2 blocks streamed through a 6-stage ring)
//   warpgroups 1, 2: wgmma + band extraction
#include "conv_tc_common.cuh"

namespace {

constexpr int NPIX = 96;           // output pixels per tile (MMA N)
constexpr int KC = 64;             // channels per K chunk (128-byte rows, SWIZZLE_128B)
constexpr int A_BYTES = 128 * KC * 2;       // one f2 block chunk  (16 KiB)
constexpr int B_BYTES = NPIX * KC * 2;      // one f1 tile chunk   (12 KiB)
constexpr int A_STAGES = 6;
constexpr int MAX_KCH = 4;         // C <= 256

struct CorrParams {
  int H, W, C, kch;
  int tiles_x, tiles_y, total_tiles;   // total = tiles_y * tiles_x * S2*S2 * n_img
  int n_img;
  void* out; int out_cs, out_dtype;
  int act; float slope;
  float scale;        // result = accumulator * scale (1/C; the correction passes of the fp32-parity mode carry 2^-11 as well)
  int accumulate;     // 1: add to the fp32 value already in `out` before the activation
  int f16;            // 1: fp16 operands (the split planes of fp32 features), 0: bf16
};

// Shared memory from the 1024-byte aligned `base`: f2 ring, two f1 tile buffers, barriers; smem = the launch's dynamic size
struct CorrSmem {
  uint32_t a_ring, b_buf, bars, smem;
  __device__ __forceinline__ uint32_t afull(int s) const { return bars + 8u * s; }
  __device__ __forceinline__ uint32_t aempty(int s) const { return bars + 8u * (A_STAGES + s); }
  __device__ __forceinline__ uint32_t bfull(int s) const { return bars + 8u * (2 * A_STAGES + s); }
  __device__ __forceinline__ uint32_t bempty(int s) const { return bars + 8u * (2 * A_STAGES + 2 + s); }
};
__host__ __device__ __forceinline__ CorrSmem corr_smem(uint32_t base) {
  const uint32_t b_buf = base + A_STAGES * A_BYTES, bars = b_buf + 2 * MAX_KCH * B_BYTES;
  return {base, b_buf, bars, bars + 8u * (2 * A_STAGES + 12) + 1024u - base};     // 2 * A_STAGES + 4 barriers used
}

// Tile `tile` (tiles_per_par per stride2-parity class): image, parity (py, px), first output pixel (y0, x0) less the parity
struct CorrTile { int img, py, px, y0, x0; };
template <int R, int S2>
__device__ __forceinline__ CorrTile corr_tile(const CorrParams& p, int tiles_per_par, int tile) {
  constexpr int TW = 32 - 2 * R, TH = NPIX / TW;
  const int per_img = tiles_per_par * S2 * S2;
  CorrTile c;
  c.img = tile / per_img;
  int t = tile - c.img * per_img;
  const int par = t / tiles_per_par;
  t -= par * tiles_per_par;
  c.py = par / S2; c.px = par % S2;
  c.y0 = (t / p.tiles_x) * TH * S2; c.x0 = (t % p.tiles_x) * TW * S2;
  return c;
}

template <int R, int S2, bool F16>
__device__ __forceinline__ void corr_consumer(const CorrParams& p, const CorrSmem& sm, int wg) {
  constexpr int D = 2 * R + 1, TW = 32 - 2 * R, TH = NPIX / TW, NBLK = (TH + 2 * R) / 4;
  const bool leader = (threadIdx.x & 127) == 0;
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const int tiles_per_par = p.tiles_y * p.tiles_x;
  RingPos ap, bp;       // f2 ring, f1 double buffer
  float d[NPIX / 2];
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const CorrTile t = corr_tile<R, S2>(p, tiles_per_par, tile);
    bp.wait_full(sm.bfull(bp.slot));
    for (int b = 0; b < NBLK; ++b) {
      for (int kc = 0; kc < p.kch; ++kc) {
        ap.wait_full(sm.afull(ap.slot));
        // K-major, 128-byte rows (SWIZZLE_128B), 8-row groups 1 KiB apart
        const uint64_t adesc = desc_at(desc_hi(128, 1024), sm.a_ring + ap.slot * A_BYTES + (uint32_t)wg * 64u * 128u);
        const uint64_t bdesc = desc_at(desc_hi(128, 1024), sm.b_buf + bp.slot * MAX_KCH * B_BYTES + kc * B_BYTES);
        wg::fence();
#pragma unroll
        for (int k = 0; k < KC / 16; ++k)
          wg::Mma<NPIX, F16>::run(d, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (uint32_t)((kc | k) != 0));
        wg::commit();
        wg::wait<0>();
        if (leader) mbar_arrive(sm.aempty(ap.slot));
        ap.next(A_STAGES);
      }
      wg::fence_regs(d);
      // fragment element d[4q + 2h + e]: neighbourhood pixel n = 64 wg + 16 w + lane/4 + 8h, output pixel m = 8q + 2(lane%4) + e.
      // The per-pixel index math below does not depend on the block; recomputing it here (opaque lane copy) keeps the
      // compiler from hoisting ~100 values out of the block loop and spilling them.
      int ln = lane;
      asm volatile("" : "+r"(ln));
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = 64 * wg + 16 * w + (ln >> 2) + 8 * h;
        const int ip = 4 * b + (n >> 5), jp = n & 31;
#pragma unroll
        for (int q = 0; q < NPIX / 8; ++q) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int m = 8 * q + 2 * (ln & 3) + e;
            const int i = m / TW, j = m - (m / TW) * TW;
            const int tj = ip - i, ti = jp - j;
            const int y = t.y0 + t.py + i * S2, x = t.x0 + t.px + j * S2;
            if (tj >= 0 && tj < D && ti >= 0 && ti < D && y < p.H && x < p.W) {
              float v = d[4 * q + 2 * h + e] * p.scale;
              const int64_t o = (((int64_t)t.img * p.H + y) * p.W + x) * p.out_cs + tj * D + ti;
              if (p.accumulate) v += ((const float*)p.out)[o];
              if (p.act == VPS_ACT_LRELU) v = v > 0.f ? v : v * p.slope;
              if (p.out_dtype == VPS_BF16) ((__nv_bfloat16*)p.out)[o] = __float2bfloat16_rn(v);
              else ((float*)p.out)[o] = v;
            }
          }
        }
      }
    }
    if (leader) mbar_arrive(sm.bempty(bp.slot));      // every MMA reading this f1 tile has completed
    bp.next(2);
  }
}

// R = max_displacement / stride2, S2 = stride2.  TW = 32 - 2R so the neighbourhood is exactly 32 columns wide.
template <int R, int S2>
__global__ void __launch_bounds__(384, 1)
corr_tc_kernel(const __grid_constant__ CUtensorMap tmF1, const __grid_constant__ CUtensorMap tmF2, const CorrParams p) {
  constexpr int TW = 32 - 2 * R, TH = NPIX / TW, NBLK = (TH + 2 * R) / 4;
  static_assert(TW * TH == NPIX && (TH + 2 * R) % 4 == 0, "tile geometry");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const CorrSmem sm = corr_smem((smem_u32(smem_raw) + 1023u) & ~1023u);
  const uint32_t b_tile_bytes = (uint32_t)p.kch * B_BYTES;
  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;     // warp-uniform role index

  if (threadIdx.x == 0) {      // full: one TMA arrival; empty: one arrival per consumer warpgroup
    for (int s = 0; s < A_STAGES; ++s) { mbar_init(sm.afull(s), 1); mbar_init(sm.aempty(s), 2); }
    for (int s = 0; s < 2; ++s) { mbar_init(sm.bfull(s), 1); mbar_init(sm.bempty(s), 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int tiles_per_par = p.tiles_y * p.tiles_x;
  if (warp == 0) {
    if (lane == 0) {
      RingPos ap, bp;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const CorrTile t = corr_tile<R, S2>(p, tiles_per_par, tile);
        // f1 tile (MMA B operand): resident for the whole tile, double-buffered across tiles
        bp.wait_empty(sm.bempty(bp.slot));
        mbar_expect_tx(sm.bfull(bp.slot), b_tile_bytes);
        for (int kc = 0; kc < p.kch; ++kc)
          tma_load_4d(sm.b_buf + bp.slot * MAX_KCH * B_BYTES + kc * B_BYTES, &tmF1, sm.bfull(bp.slot), kc * KC, t.x0 + t.px, t.y0 + t.py, t.img);
        // f2 neighbourhood blocks (MMA A operand): 4 rows x 32 columns of same-parity pixels each
        for (int b = 0; b < NBLK; ++b) {
          for (int kc = 0; kc < p.kch; ++kc) {
            ap.wait_empty(sm.aempty(ap.slot));
            mbar_expect_tx(sm.afull(ap.slot), A_BYTES);
            tma_load_4d(sm.a_ring + ap.slot * A_BYTES, &tmF2, sm.afull(ap.slot), kc * KC, t.x0 + t.px - R * S2,
                        t.y0 + t.py + (4 * b - R) * S2, t.img);
            ap.next(A_STAGES);
          }
        }
        bp.next(2);
      }
    }
  } else if (warp >= 4) {
    if (p.f16) corr_consumer<R, S2, true>(p, sm, (warp - 4) >> 2);
    else corr_consumer<R, S2, false>(p, sm, (warp - 4) >> 2);
  }
}

template <int R, int S2>
int launch(const vps_tensor* f1, const vps_tensor* f2, const vps_tensor* out, int act, float slope, cudaStream_t st,
           float scale = 0.f, int accumulate = 0, int f16 = 0) {
  constexpr int TW = 32 - 2 * R, TH = NPIX / TW;
  CorrParams p;
  p.H = f1->h; p.W = f1->w; p.C = f1->c; p.kch = f1->c / KC; p.n_img = f1->n;
  p.tiles_y = vps::cdiv(vps::cdiv(f1->h, S2), TH);
  p.tiles_x = vps::cdiv(vps::cdiv(f1->w, S2), TW);
  p.total_tiles = p.tiles_y * p.tiles_x * S2 * S2 * f1->n;
  p.out = out->ptr; p.out_cs = out->cs; p.out_dtype = out->dtype; p.act = act; p.slope = slope;
  p.scale = scale != 0.f ? scale : 1.0f / (float)f1->c; p.accumulate = accumulate; p.f16 = f16;
  // f1: the tile's output pixels; f2: blocks of 4 rows x 32 columns of its neighbourhood (same-parity pixels)
  const CUtensorMapDataType type = f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUtensorMap tm1, tm2;
  if (!vps::encode_nhwc(&tm1, *f1, type, KC, TW * S2, TH * S2, S2, S2, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        "correlation_tc: encode f1") ||
      !vps::encode_nhwc(&tm2, *f2, type, KC, 32 * S2, 4 * S2, S2, S2, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        "correlation_tc: encode f2"))
    return VPS_E_CUDA;
  const int smem = (int)corr_smem(0).smem;
  auto kern = corr_tc_kernel<R, S2>;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) {
      vps::set_error("correlation_tc: smem attr: %s", cudaGetErrorString(cudaGetLastError()));
      return VPS_E_CUDA;
    }
    attr_set = true;
  }
  // a plain launch: the kernel has no griddepcontrol.wait, so it must not start before the previous kernel has completed
  const int sms = vps::num_sms();
  const int grid = p.total_tiles < sms ? p.total_tiles : sms;
  kern<<<grid, 384, smem, st>>>(tm1, tm2, p);
  VPS_CUDA_LAST("corr_tc_kernel");
  return VPS_OK;
}

// fp32 features -> two fp16 planes (dense NHWC, cs = c):  hi = fp16(v),  lo = fp16(2^11 * (v - hi))  -- the operand split of the
// fp32-parity convolutions (split_f16): v = hi + 2^-11 * lo to ~2^-22 relative
__global__ void split_f16_planes_kernel(const float* __restrict__ x, int64_t npix, int c, int cs, __half* __restrict__ hi,
                                        __half* __restrict__ lo, unsigned int* overflow) {
  const int64_t total = npix * (c / 4);
  bool over = false;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pix = i / (c / 4);
    const int c4 = (int)(i - pix * (c / 4)) * 4;
    const float4 v = *reinterpret_cast<const float4*>(x + pix * cs + c4);
    const float vv[4] = {v.x, v.y, v.z, v.w};
    __half h[4], l[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      unsigned short hb, lb;
      split_f16(vv[k], hb, lb);
      over = over || f16_over(vv[k]);
      h[k] = __ushort_as_half(hb); l[k] = __ushort_as_half(lb);
    }
    *reinterpret_cast<uint2*>(hi + pix * c + c4) = *reinterpret_cast<const uint2*>(h);
    *reinterpret_cast<uint2*>(lo + pix * c + c4) = *reinterpret_cast<const uint2*>(l);
  }
  if (over && overflow) atomicAdd(overflow, 1u);
}

}  // namespace

extern "C" unsigned int* vps_tc32_overflow_flag();      // conv_tc32.cu: device address of the saturation counter

extern "C" int64_t vps_correlation_tc32_ws_bytes(const vps_tensor* f1) {
  return 4 * (int64_t)f1->n * f1->h * f1->w * f1->c * 2 + 1024;
}

// Correlation of fp32 features on the tensor cores in the parity precision: both maps are split into fp16 planes
// (v = hi + 2^-11 lo) and the banded GEMM runs three times, hi.hi, then hi.lo and lo.hi scaled by 2^-11 and accumulated
// into the fp32 output (the activation is applied by the last pass).  Unlike the stacked convolutions a correlation is a
// single K = C <= 256 contraction (16 MMAs per accumulator chain) whose result is not fed through further layers of the same
// kind, so the accumulation inside the tensor core needs no promotion here.
// `ws`: vps_correlation_tc32_ws_bytes() of scratch, 256-byte aligned.  Same supported geometries as vps_correlation_tc.
extern "C" int vps_correlation_tc32(const vps_tensor* f1, const vps_tensor* f2, const vps_tensor* out, int pad, int max_disp,
                                    int stride1, int stride2, int act, float slope, void* ws, void* stream) {
  VPS_CHECK_ARG(stride1 == 1 && pad == max_disp, "correlation_tc32: only stride1=1, pad==max_displacement");
  VPS_CHECK_ARG(f1->dtype == VPS_F32 && f2->dtype == VPS_F32 && out->dtype == VPS_F32, "correlation_tc32: fp32 tensors only");
  VPS_CHECK_ARG(f1->h == f2->h && f1->w == f2->w && f1->c == f2->c && f1->n == f2->n && out->h == f1->h && out->w == f1->w,
                "correlation_tc32: shape mismatch");
  VPS_CHECK_ARG(f1->c % KC == 0 && f1->c <= KC * MAX_KCH, "correlation_tc32: C must be a multiple of 64, <= 256");
  VPS_CHECK_ARG(f1->cs % 4 == 0 && f2->cs % 4 == 0 && ((uintptr_t)f1->ptr & 15) == 0 && ((uintptr_t)f2->ptr & 15) == 0 &&
                    ws && ((uintptr_t)ws & 255) == 0, "correlation_tc32: features / scratch must be aligned");
  VPS_CHECK_ARG(act == VPS_ACT_NONE || act == VPS_ACT_LRELU, "correlation_tc32: act");
  const int R = max_disp / stride2, D = 2 * R + 1;
  VPS_CHECK_ARG(out->c == D * D, "correlation_tc32: out.c %d != %d", out->c, D * D);
  VPS_CHECK_ARG((R == 10 && stride2 == 2) || (R == 4 && stride2 == 1), "correlation_tc32: unsupported (max_disp %d, stride2 %d)",
                max_disp, stride2);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t npix = (int64_t)f1->n * f1->h * f1->w, plane = npix * f1->c;
  __half* base = (__half*)ws;
  vps_tensor t[4];      // f1 hi, f1 lo, f2 hi, f2 lo
  for (int i = 0; i < 4; ++i) {
    t[i] = *f1; t[i].ptr = base + i * plane; t[i].cs = f1->c; t[i].dtype = VPS_BF16;      // (2-byte elements; the kernel is told f16)
  }
  unsigned int* flag = vps_tc32_overflow_flag();
  const int blocks = (int)((npix * (f1->c / 4) + 255) / 256 > 8192 ? 8192 : (npix * (f1->c / 4) + 255) / 256);
  split_f16_planes_kernel<<<blocks, 256, 0, st>>>((const float*)f1->ptr, npix, f1->c, f1->cs, base, base + plane, flag);
  VPS_CUDA_LAST("split_f16_planes");
  split_f16_planes_kernel<<<blocks, 256, 0, st>>>((const float*)f2->ptr, npix, f1->c, f2->cs, base + 2 * plane, base + 3 * plane, flag);
  VPS_CUDA_LAST("split_f16_planes");
  const float s1 = 1.0f / (float)f1->c, s2 = s1 * T32_LO_INV;
  int rc;
#define CORR_PASS(A, B, SC, ACC, ACT)                                                                        \
  rc = (R == 10) ? launch<10, 2>(&t[A], &t[B], out, ACT, slope, st, SC, ACC, 1) : launch<4, 1>(&t[A], &t[B], out, ACT, slope, st, SC, ACC, 1); \
  if (rc != VPS_OK) return rc;
  CORR_PASS(0, 2, s1, 0, VPS_ACT_NONE)      // f1.hi x f2.hi
  CORR_PASS(0, 3, s2, 1, VPS_ACT_NONE)      // f1.hi x f2.lo
  CORR_PASS(1, 2, s2, 1, act)               // f1.lo x f2.hi, then the activation
#undef CORR_PASS
  return VPS_OK;
}

// Tensor-core correlation; returns VPS_E_ARG (without launching) when the geometry is not one of the two supported
// call sites -- vps_correlation then uses the CUDA-core kernel.
extern "C" int vps_correlation_tc(const vps_tensor* f1, const vps_tensor* f2, const vps_tensor* out, int pad, int max_disp,
                                  int stride1, int stride2, int act, float slope, void* stream) {
  VPS_CHECK_ARG(stride1 == 1 && pad == max_disp, "correlation_tc: only stride1=1, pad==max_displacement");
  VPS_CHECK_ARG(f1->dtype == VPS_BF16 && f2->dtype == VPS_BF16, "correlation_tc: bf16 features only");
  VPS_CHECK_ARG(f1->h == f2->h && f1->w == f2->w && f1->c == f2->c && f1->n == f2->n && out->h == f1->h && out->w == f1->w,
                "correlation_tc: shape mismatch");
  VPS_CHECK_ARG(f1->c % KC == 0 && f1->c <= KC * MAX_KCH, "correlation_tc: C must be a multiple of 64, <= 256");
  VPS_CHECK_ARG(f1->cs % 8 == 0 && f2->cs % 8 == 0 && ((uintptr_t)f1->ptr & 15) == 0 && ((uintptr_t)f2->ptr & 15) == 0,
                "correlation_tc: features must be 16-byte aligned");
  VPS_CHECK_ARG(act == VPS_ACT_NONE || act == VPS_ACT_LRELU, "correlation_tc: act");
  const int R = max_disp / stride2, D = 2 * R + 1;
  VPS_CHECK_ARG(out->c == D * D, "correlation_tc: out.c %d != %d", out->c, D * D);
  cudaStream_t st = (cudaStream_t)stream;
  if (R == 10 && stride2 == 2) return launch<10, 2>(f1, f2, out, act, slope, st);
  if (R == 4 && stride2 == 1) return launch<4, 1>(f1, f2, out, act, slope, st);
  vps::set_error("correlation_tc: unsupported (max_disp %d, stride2 %d)", max_disp, stride2);
  return VPS_E_ARG;
}
