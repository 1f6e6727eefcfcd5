// Shared code of the wgmma kernels (conv_tc.cu: bf16 operands; conv_tc32.cu: fp32 operands split on the fly into fp16 main +
// correction planes; corr_tc.cu): launch parameters, PTX wrappers (mbarrier / TMA), shared-memory matrix descriptors, the fp16
// operand split, the DCN sampling set-up, the epilogue (register accumulators -> bias / activation / residual -> NHWC store),
// and the host side common to the convolution launchers.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace {

constexpr int BLOCK_M = 128;
constexpr int MAX_STAGES = 8;

constexpr int MAX_PROB = 4;   // stride-phase sub-convolutions of one transposed conv share a launch

struct ConvTcParams {
  int bk;                     // K elements per pipeline stage: 64 (SWIZZLE_128B rows) or 16 (SWIZZLE_32B rows)
  int nprob, tiles_per_prob;  // problems differ only in weights, padding and output pixel offset
  int ph_[MAX_PROB], pw_[MAX_PROB], oy_off_[MAX_PROB], ox_off_[MAX_PROB];
  int n_img, oh, ow;
  int th, tw, tiles_y, tiles_x;
  int n_tiles_n, block_n;
  int kh, kw, sh, sw;
  int cin_chunks;
  int a_stages, b_stages;     // operand rings (A: activation boxes, B: weight boxes)
  int halo;                   // 1: one (th+kh-1) x (tw+kw-1) activation box per channel chunk feeds all kh*kw taps
  int halo_w;                 // tw + kw - 1 (pixels per halo row)
  int a_stage_bytes;          // bytes of one A ring slot (multiple of 1024)
  int a_box_bytes;            // bytes one A TMA box delivers
  int rowg;                   // halo mode: 1 = one B ring slot holds the kw taps of a filter row (one barrier round per row)
  int gsub;                   // flat (non-halo) mode: K steps per ring slot (one barrier round covers gsub steps)
  int nk_last;                // K16 slabs of the last channel chunk that hold real channels (the rest is zero padding)
  int total_tiles;
  void* y;
  int y_h, y_w, y_cs, y_dtype, y_vec;
  int oy_mul, ox_mul;
  const void* res;
  int res_cs, res_dtype, res_after_act, res_vec;
  const float* bias;
  int cout;
  int act;
  float slope, out_scale;
};

#ifndef VPS_MBAR_SPIN_LOG2
#define VPS_MBAR_SPIN_LOG2 26     // debugging builds: VPS_NVCC_EXTRA=-DVPS_MBAR_SPIN_LOG2=20 python -m vps_b200.build -f
#endif
// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// The retry loop lives inside the PTX block: a C++ loop around try_wait (with a diagnostic printf) is a divergent path with a
// function call to the compiler, and a wait between two wgmma batches then makes ptxas serialise the wgmma pipeline.  A lost
// arrival still fails loudly: after 2^VPS_MBAR_SPIN_LOG2 unsuccessful polls the kernel traps instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      ".reg .u32 n;\n"
      "mov.u32 n, 0;\n"
      "VPS_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra.uni VPS_DONE;\n"
      "add.u32 n, n, 1;\n"
      "setp.lt.u32 p, n, %2;\n"
      "@p bra.uni VPS_WAIT;\n"
      "trap;\n"
      "VPS_DONE:\n"
      "}\n" ::"r"(bar), "r"(parity), "n"(1u << VPS_MBAR_SPIN_LOG2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4, %5, %6}], [%2];" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2, int c3,
                                            int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4, %5, %6, %7}], [%2];" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4, %5}], [%2];" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4}], [%2];" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// shared -> global tensor store of one box (clipped at the tensor bounds), in the issuing thread's bulk async-group
__device__ __forceinline__ void tma_store_4d(const void* tmap, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(tmap), "r"(src),
               "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
// true in exactly one lane of the (converged) warp -- the same lane every time for a full mask
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "elect.sync _|P, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}
// High word of a wgmma matrix descriptor for a K-major operand tile whose rows are `row_bytes` long: 128 -> SWIZZLE_128B,
// 64 -> SWIZZLE_64B, 32 -> SWIZZLE_32B (the swizzle TMA wrote the tile with); `sbo` = byte distance between consecutive
// 8-row groups (8 * row bytes for a dense tile; the halo row pitch when the 8 rows of a group are 8 consecutive pixels of
// one halo row).  The low word is (shared address & 0x3FFFF) >> 4; a K16 slab further along a row is +2 per 32 bytes.
__host__ __device__ __forceinline__ uint64_t desc_hi(uint32_t row_bytes, uint32_t sbo) {
  uint64_t d = (uint64_t)1 << 16;                                    // leading byte offset (unused by swizzled K-major tiles)
  d |= (uint64_t)(sbo >> 4) << 32;
  d |= (uint64_t)(row_bytes == 128 ? 1 : (row_bytes == 64 ? 2 : 3)) << 62;
  return d;
}
__device__ __forceinline__ uint64_t desc_at(uint64_t hi, uint32_t smem_addr) { return hi | (uint64_t)((smem_addr & 0x3FFFF) >> 4); }

// ---------------------------------------------------------------- fp16 operand split of the fp32-parity precision
// v = hi + 2^-11 lo:  hi = fp16(v),  lo = fp16(2^11 (v - hi))  (round to nearest, saturating; see conv_tc32.cu)
constexpr float T32_LO_SCALE = 2048.f, T32_LO_INV = 1.f / 2048.f;

// |v| > 65504 (or NaN): outside the fp16 range, so the split saturates hi
__device__ __forceinline__ bool f16_over(float v) { return !(fabsf(v) <= 65504.f); }

// split of one value (round to nearest, saturating).  The range check is left to the caller (f16_over): with a flag passed
// by reference the compiler no longer folds the checks of consecutive values into one predicate chain.
__device__ __forceinline__ void split_f16(float v, unsigned short& hi, unsigned short& lo) {
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(hi) : "f"(v));
  const float r = (v - __half2float(__ushort_as_half(hi))) * T32_LO_SCALE;      // exact in fp32; never exceeds |v|
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(lo) : "f"(r));
}

// split of two values at once: hi = packed fp16x2 of (v0, v1), lo = packed fp16x2 of 2^11 * (v - fp16(v)).  Same values as two
// split_f16() calls with 10 instead of 14 instructions; `over` collects f16_over of both values (the converter and the deformable sampler are bound by exactly this
// arithmetic).
__device__ __forceinline__ void split_pair_f16(float v0, float v1, uint32_t& hi, uint32_t& lo, bool& over) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(v1), "f"(v0));       // first source -> upper half
  over = over || !(fabsf(v0) <= 65504.f) || !(fabsf(v1) <= 65504.f);
  const float2 h = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  const float r0 = (v0 - h.x) * T32_LO_SCALE, r1 = (v1 - h.y) * T32_LO_SCALE;          // exact in fp32
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(r1), "f"(r0));
}

// ---------------------------------------------------------------- weight packing
// element i of a packed [cout_pad][kh][kw][cin_pad] weight buffer: the source weight times scale[co] (if given), 0 in the
// padding; src OIHW, or IOHW when transposed
__device__ __forceinline__ float packed_weight(const float* __restrict__ src, const float* __restrict__ scale, int64_t i, int cout,
                                               int cin, int kh, int kw, int cin_pad, int transposed) {
  const int ci = (int)(i % cin_pad);
  int64_t t = i / cin_pad;
  const int s = (int)(t % kw); t /= kw;
  const int r = (int)(t % kh); t /= kh;
  const int co = (int)t;
  float v = 0.f;
  if (co < cout && ci < cin) {
    const int64_t si = transposed ? ((((int64_t)ci * cout + co) * kh + r) * kw + s) : ((((int64_t)co * cin + ci) * kh + r) * kw + s);
    v = src[si];
    if (scale) v *= scale[co];
  }
  return v;
}

// ---------------------------------------------------------------- deformable convolution (DCNv1, 3x3, pad 1)
// input x (bf16 or fp32 NHWC) and the fp32 NHWC offsets, (dy, dx) per tap
template <class T>
struct DcnParams {
  const T* x;
  const float* off;
  int x_cs, off_cs, H, W;
};
// bytes of a tile's sampling set-up table: one 32-byte entry (4 bilinear weights + 4 element offsets) per (tap, pixel)
__host__ __device__ constexpr int dcn_setup_bytes(int rows) { return 9 * rows * 32; }

// Sampling set-up of tap k of output pixel (yo, xo) of image img -- the 4 bilinear corner weights and the 4 element offsets of
// the corners in x (0 / 0 outside the image) -- as one 32-byte shared-memory entry at `sa`.
template <class T>
__device__ __forceinline__ void dcn_setup_entry(const DcnParams<T>& d, uint32_t sa, int img, int yo, int xo, int k) {
  const int H = d.H, W = d.W;
  float wts[4] = {0.f, 0.f, 0.f, 0.f};
  int offs[4] = {0, 0, 0, 0};
  if (yo < H && xo < W) {
    const float* op = d.off + ((int64_t)(img * H + yo) * W + xo) * d.off_cs;
    const float oh = __ldg(op + 2 * k), ow = __ldg(op + 2 * k + 1);
    const float h = (float)(yo - 1 + k / 3) + oh;
    const float w = (float)(xo - 1 + k % 3) + ow;
    if (h > -1.f && w > -1.f && h < (float)H && w < (float)W) {
      const int hl = (int)floorf(h), wl = (int)floorf(w);
      const int hh_ = hl + 1, wh_ = wl + 1;
      const float lh = h - (float)hl, lw = w - (float)wl;
      const float hh = 1.f - lh, hw = 1.f - lw;
      const int base = img * H;
      if (hl >= 0 && wl >= 0) { wts[0] = hh * hw; offs[0] = ((base + hl) * W + wl) * d.x_cs; }
      if (hl >= 0 && wh_ <= W - 1) { wts[1] = hh * lw; offs[1] = ((base + hl) * W + wh_) * d.x_cs; }
      if (hh_ <= H - 1 && wl >= 0) { wts[2] = lh * hw; offs[2] = ((base + hh_) * W + wl) * d.x_cs; }
      if (hh_ <= H - 1 && wh_ <= W - 1) { wts[3] = lh * lw; offs[3] = ((base + hh_) * W + wh_) * d.x_cs; }
    }
  }
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(sa), "f"(wts[0]), "f"(wts[1]), "f"(wts[2]), "f"(wts[3]) : "memory");
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sa + 16u), "r"(offs[0]), "r"(offs[1]), "r"(offs[2]), "r"(offs[3]) : "memory");
}

// ---------------------------------------------------------------- ring positions and the K walk shared by the roles
// Position in a ring of `slots` mbarrier-guarded slots: the slot and the parity of its current use.  A reader waits for the
// slot's full barrier at `phase`; a writer waits for its empty barrier at `phase ^ 1`, which the barrier's initial phase
// satisfies on the first pass through the ring.
struct RingPos {
  int slot = 0;
  uint32_t phase = 0;
  // the position of use n (counted from 0)
  __device__ __forceinline__ static RingPos at(uint32_t n, uint32_t slots) { return {(int)(n % slots), (n / slots) & 1u}; }
  __device__ __forceinline__ void wait_full(uint32_t bar) const { mbar_wait(bar, phase); }
  __device__ __forceinline__ void wait_empty(uint32_t bar) const { mbar_wait(bar, phase ^ 1u); }
  // advance by `step` (0 or 1), without a branch on it: the tc32 consumers need more registers with `if (step)`
  __device__ __forceinline__ void next(int slots, bool step = true) {
    slot += step;
    if (slot == slots) { slot = 0; phase ^= 1; }
  }
};

// The filter tap of a K step and its (r, s).  K steps run chunk-major and tap-minor: within a channel chunk the tap
// advances fastest, s before r.
struct Tap {
  int k = 0, r = 0, s = 0;
  __device__ __forceinline__ void next(int kw) { ++k; if (++s == kw) { s = 0; ++r; } }
};

struct TileCoord {
  int prob, n_idx, img, ty, tx;
};
__device__ __forceinline__ TileCoord tile_coord(const ConvTcParams& p, int tile) {
  TileCoord t;
  t.prob = tile / p.tiles_per_prob;
  const int t_in = tile - t.prob * p.tiles_per_prob;
  t.n_idx = t_in % p.n_tiles_n;
  const int m_idx = t_in / p.n_tiles_n;
  const int tiles_per_img = p.tiles_y * p.tiles_x;
  t.img = m_idx / tiles_per_img;
  const int rem = m_idx - t.img * tiles_per_img;
  t.ty = rem / p.tiles_x;
  t.tx = rem - t.ty * p.tiles_x;
  return t;
}

// ---------------------------------------------------------------- epilogue
// bias / residual / activation / scale of one channel pair (b = bias, r = residual).  Every epilogue goes through this
// function, so the fp32 operations and their order are the same whichever way the values are loaded and stored.
__device__ __forceinline__ float2 epi_math(const ConvTcParams& p, float v0, float v1, float b0, float b1, float r0, float r1) {
  if (p.bias) { v0 += b0; v1 += b1; }
  if (p.res && !p.res_after_act) { v0 += r0; v1 += r1; }
  float v[2] = {v0, v1};
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    float t = v[j];
    if (p.act == VPS_ACT_RELU) t = fmaxf(t, 0.f);
    else if (p.act == VPS_ACT_LRELU) t = t > 0.f ? t : t * p.slope;
    else if (p.act == VPS_ACT_SIGMOID) t = 1.f / (1.f + __expf(-t));
    v[j] = t * p.out_scale;
  }
  if (p.res && p.res_after_act) { v[0] += r0; v[1] += r1; }
  return make_float2(v[0], v[1]);
}

// bias and residual of the channel pair (c, c + 1) of output pixel `pix` (c + 1 only if `two`)
__device__ __forceinline__ void epi_load(const ConvTcParams& p, int64_t pix, int c, bool two, float& b0, float& b1, float& r0,
                                         float& r1) {
  b0 = b1 = r0 = r1 = 0.f;
  if (p.bias) {
    b0 = __ldg(p.bias + c);
    if (two) b1 = __ldg(p.bias + c + 1);
  }
  if (p.res) {
    const int64_t ro = pix * p.res_cs + c;       // even element index: pair loads are aligned when res_vec
    if (p.res_dtype == VPS_BF16) {
      const __nv_bfloat16* rp = (const __nv_bfloat16*)p.res + ro;
      if (two && p.res_vec) {
        const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(rp));
        r0 = f.x; r1 = f.y;
      } else {
        r0 = __bfloat162float(rp[0]);
        if (two) r1 = __bfloat162float(rp[1]);
      }
    } else {
      const float* rp = (const float*)p.res + ro;
      if (two && p.res_vec) {
        const float2 f = *reinterpret_cast<const float2*>(rp);
        r0 = f.x; r1 = f.y;
      } else {
        r0 = rp[0];
        if (two) r1 = rp[1];
      }
    }
  }
}

// store of the channel pair (c, c + 1) of output pixel `pix` (c + 1 only if `two`)
__device__ __forceinline__ void epi_store(const ConvTcParams& p, float2 v, int64_t pix, int c, bool two) {
  const int64_t yo = pix * p.y_cs + c;           // even element index: pair stores are aligned when y_vec
  if (p.y_dtype == VPS_BF16) {
    __nv_bfloat16* yp = (__nv_bfloat16*)p.y + yo;
    if (two && p.y_vec) *reinterpret_cast<__nv_bfloat162*>(yp) = __floats2bfloat162_rn(v.x, v.y);
    else { yp[0] = __float2bfloat16_rn(v.x); if (two) yp[1] = __float2bfloat16_rn(v.y); }
  } else {
    float* yp = (float*)p.y + yo;
    if (two && p.y_vec) *reinterpret_cast<float2*>(yp) = v;
    else { yp[0] = v.x; if (two) yp[1] = v.y; }
  }
}

// One consumer warpgroup's m64nN accumulator (rows row0 .. row0 + 63, channels c_off .. c_off + N - 1 of the tile) -> NHWC
// output.  Fragment layout of wgmma:
// warp w of the group, lane l holds d[4j + 2h + e] = D[16w + l/4 + 8h][8j + 2(l%4) + e].
// y may alias the bias and the residual as far as the compiler knows, so a load written after a store waits for it.  The
// loads of PAIRS channel pairs of a row are therefore all issued before any of their stores: one global round trip per
// group instead of one per pair.  PAIRS is the most the caller's register budget holds without spilling.
template <int N, int PAIRS>
__device__ __forceinline__ void epi_frag(const ConvTcParams& p, const float (&d)[N / 2], int tile, int row0, int c_off = 0) {
  constexpr int G = N / 8 < PAIRS ? N / 8 : PAIRS;
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const TileCoord t = tile_coord(p, tile);
  const int nbase = t.n_idx * p.block_n + c_off;
  const int nlim = min(p.cout, nbase + N);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + 16 * w + (lane >> 2) + 8 * h;
    const int ty_in = row / p.tw, tx_in = row - ty_in * p.tw;
    const int oy = t.ty * p.th + ty_in, ox = t.tx * p.tw + tx_in;
    if (oy >= p.oh || ox >= p.ow) continue;
    const int64_t pix = ((int64_t)t.img * p.y_h + (oy * p.oy_mul + p.oy_off_[t.prob])) * p.y_w + (ox * p.ox_mul + p.ox_off_[t.prob]);
#pragma unroll
    for (int j0 = 0; j0 < N / 8; j0 += G) {
      float b[G][2], r[G][2];
#pragma unroll
      for (int j = 0; j < G; ++j) {
        const int c = nbase + 8 * (j0 + j) + 2 * (lane & 3);
        if (c < nlim) epi_load(p, pix, c, c + 1 < nlim, b[j][0], b[j][1], r[j][0], r[j][1]);
      }
#pragma unroll
      for (int j = 0; j < G; ++j) {
        const int c = nbase + 8 * (j0 + j) + 2 * (lane & 3);
        const int k = 4 * (j0 + j) + 2 * h;
        if (c < nlim) epi_store(p, epi_math(p, d[k], d[k + 1], b[j][0], b[j][1], r[j][0], r[j][1]), pix, c, c + 1 < nlim);
      }
    }
  }
}

// ---------------------------------------------------------------- host
// Width of the output patch of `pixels` pixels (tw x pixels / tw) with the smallest padded area over oh x ow.  The first
// minimum in candidate order wins; a candidate whose TMA box extents tw * sw or th * sh exceed 256 is skipped.
inline int patch_tw(int oh, int ow, int pixels, int sh, int sw) {
  int best_tw = 16;
  int64_t best_area = -1;
  for (const int tw : {16, 8, 32, 64, 128, 256}) {
    const int th = pixels / tw;
    if (th == 0 || tw * sw > 256 || th * sh > 256) continue;
    const int64_t area = (int64_t)vps::cdiv(ow, tw) * tw * vps::cdiv(oh, th) * th;
    if (best_area < 0 || area < best_area) { best_area = area; best_tw = tw; }
  }
  return best_tw;
}

// Tile walk of a launch: th x tw output pixels x block_n channels per tile, K in chunks of kc channels, nprob problems.
inline void set_tiles(ConvTcParams& p, const vps_conv_args* a, int nprob, int tw, int th, int block_n, int kc) {
  p.n_img = a->x.n; p.oh = a->oh; p.ow = a->ow;
  p.tw = tw; p.th = th;
  p.tiles_x = vps::cdiv(a->ow, tw); p.tiles_y = vps::cdiv(a->oh, th);
  p.block_n = block_n; p.n_tiles_n = vps::cdiv((a->cout + 15) / 16 * 16, block_n);
  p.kh = a->kh; p.kw = a->kw; p.sh = a->sh; p.sw = a->sw;
  p.cin_chunks = vps::cdiv(a->cin, kc);
  p.nk_last = vps::cdiv(a->cin - (p.cin_chunks - 1) * kc, 16);
  p.nprob = nprob;
  p.tiles_per_prob = p.n_img * p.tiles_y * p.tiles_x * p.n_tiles_n;
  p.total_tiles = p.tiles_per_prob * nprob;
}

// A DCN layer as the convolution whose tiles and epilogue it shares: 3x3, stride 1, pad 1, no bias, x's size.  The caller
// sets the output y.
inline vps_conv_args dcn_args(const vps_tensor& x, int cout) {
  vps_conv_args a = {};
  a.x = x;
  a.kh = a.kw = 3; a.sh = a.sw = 1; a.ph = a.pw = 1;
  a.oh = x.h; a.ow = x.w; a.oy_mul = a.ox_mul = 1;
  a.cin = x.c; a.cout = cout;
  a.act = VPS_ACT_NONE; a.out_scale = 1.f;
  return a;
}

// the output tensor of the epilogue; pair stores are 128-bit (y_vec 1) or 256-bit (y_vec 2) aligned where the layout allows
inline void set_output(ConvTcParams& p, const vps_tensor& y) {
  p.y = y.ptr; p.y_h = y.h; p.y_w = y.w; p.y_cs = y.cs; p.y_dtype = y.dtype;
  const int esz = y.dtype == VPS_BF16 ? 2 : 4;
  p.y_vec = (((uintptr_t)y.ptr & 15) == 0) && ((y.cs * esz) % 16 == 0);
  if (p.y_vec && (((uintptr_t)y.ptr & 31) == 0) && ((y.cs * esz) % 32 == 0)) p.y_vec = 2;
}

// Padding, output mapping and epilogue of the nprob problems of one convolution launch; `who` prefixes the error messages.
inline int set_problems(ConvTcParams& p, const vps_conv_args* args, int nprob, const char* who) {
  const vps_conv_args* a = &args[0];
  set_output(p, a->y);
  p.oy_mul = a->oy_mul; p.ox_mul = a->ox_mul;
  for (int i = 0; i < MAX_PROB; ++i) {
    const vps_conv_args* q = &args[i < nprob ? i : 0];
    p.ph_[i] = q->ph; p.pw_[i] = q->pw; p.oy_off_[i] = q->oy_off; p.ox_off_[i] = q->ox_off;
    VPS_CHECK_ARG((a->oh - 1) * a->oy_mul + q->oy_off < a->y.h && (a->ow - 1) * a->ox_mul + q->ox_off < a->y.w,
                  "%s: output mapping out of range", who);
  }
  p.res = a->res.ptr; p.res_cs = a->res.cs; p.res_dtype = a->res.dtype; p.res_after_act = a->res_after_act;
  p.res_vec = a->res.ptr && (((uintptr_t)a->res.ptr & 15) == 0) && (a->res.cs % 8 == 0);
  if (p.res_vec && (((uintptr_t)a->res.ptr & 31) == 0) && (a->res.cs % 16 == 0)) p.res_vec = 2;       // 256-bit loads
  VPS_CHECK_ARG(!a->bias || ((uintptr_t)a->bias & 15) == 0, "%s: bias must be 16-byte aligned", who);
  p.bias = a->bias; p.cout = a->cout; p.act = a->act; p.slope = a->slope; p.out_scale = a->out_scale;
  if (a->res.ptr) VPS_CHECK_ARG(a->res.h == a->y.h && a->res.w == a->y.w, "%s: residual geometry", who);
  return VPS_OK;
}

// Persistent launch of the tile kernel K: grid = min(tiles, SMs), with programmatic stream serialization, so that the kernel's
// prologue (barrier init, tensor-map prefetch) overlaps the previous kernel's tail until its griddepcontrol.wait.  Only for
// kernels that execute griddepcontrol.wait before they touch global memory.  The dynamic shared-memory limit is raised once
// per kernel.  `who` prefixes the error messages.
template <auto K, typename... A>
int launch_persistent(int tiles, int threads, int smem, void* stream, const char* who, const A&... args) {
  static bool smem_raised = false;
  if (!smem_raised) {
    if (cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess) {
      vps::set_error("%s: cannot raise dynamic smem: %s", who, cudaGetErrorString(cudaGetLastError()));
      return VPS_E_CUDA;
    }
    smem_raised = true;
  }
  const int sms = vps::num_sms();
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(tiles < sms ? tiles : sms)); cfg.blockDim = dim3((unsigned)threads);
  cfg.dynamicSmemBytes = (size_t)smem; cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = &attr; cfg.numAttrs = 1;
  const cudaError_t le = cudaLaunchKernelEx(&cfg, K, args...);
  if (le != cudaSuccess) { vps::set_error("%s: launch failed: %s", who, cudaGetErrorString(le)); return VPS_E_CUDA; }
  VPS_CUDA_LAST(who);
  return VPS_OK;
}

}  // namespace
