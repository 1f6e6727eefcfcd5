// fp32-parity convolution on Hopper tensor cores (wgmma, sm_90a): the "tc32" precision.
//
// The reference computes every convolution in fp32 (cuDNN, e.g. resnet.py:506-517, flownet2.py:133-198) and
// north_star asks for label maps / track ids bit-exact and logits within 1e-3 of it -- which a single bf16 pass
// (8 significant bits per operand) cannot give.  This kernel keeps activations and results fp32 in HBM and feeds the
// tensor cores three fp16 products per K slab that together carry ~23 significant bits of every operand:
//
//     a = A + 2^-11 * A2,   A = fp16(a) (round to nearest),  A2 = fp16(2^11 * (a - A))      [b = B + 2^-11 * B2 likewise]
//     a*b ~= A*B  +  2^-11 * (A2*B + A*B2)                      (all kind::f16, f16 x f16, fp32 accumulate)
//
// a - A is exact in fp32 and at most half an fp16 ulp of a, so 2^11 * (a - A) never exceeds |a| (no overflow) and stays
// a normal fp16 number whenever a is one; dropped are a_lo*b_lo <= 2^-24 |ab| and the fp16 rounding of A2 / B2 (2^-23).
// Cost: 3 tensor-core passes -- against 6 for a three-way bf16 split of the same accuracy class; a two-way bf16 split
// (bf16x3) is NOT enough: its CPU emulation through the whole FuseTrack path (tools/emulate_split.py) flips proposals /
// ids / label pixels.  fp16's narrow exponent range is harmless below (values under 2^-14 are carried by A2: the residual
// of a subnormal A is <= 2^-25, i.e. 2^-14 after scaling); values above 65504 are saturated and counted in a device
// flag the caller must check (vps_tc32_overflow) -- the result then only has fp16-saturation accuracy.
//
// The tensor core's fp32 accumulation is not guaranteed to round to nearest (on the previous tensor-core generation it was
// measured to truncate: a bias that compounds over ~60 stacked layers), so no long chain of MMA additions is trusted:
//   * per K step the correction products (A2*B + A*B2) start a fresh accumulator, are scaled by 2^-11 in registers, and the
//     main product A*B is added on top -- a chain of 2 main MMAs;
//   * that step result is promoted into a per-thread register sum with a round-to-nearest fp32 add.
//
// Pipeline per CTA (persistent, one (64 * P)-pixel x block_n tile at a time, K consumed 32 channels per step):
//   warp 0          : TMA producer: raw fp32 activation boxes {32 ch, pixels} into a staging ring; pre-split weight tiles
//                     [B | B2] (vps_pack_weights_tc32) into the B ring.
//   warps 1-3       : converters: staging box -> two SWIZZLE_64B operand planes A, A2 (generic-proxy writes ->
//                     fence.proxy.async -> mbarrier).  In halo mode (stride 1, > 1 tap) one converted (th+kh-1) x (tw+kw-1)
//                     box feeds all kh*kw taps through shifted descriptor start addresses.
//   warpgroups 1..NWG: consumers: wgmma.kind f16 (M64 x N x K16) into registers, promotion, then bias / activation /
//                     residual and the NHWC store.  Flat tiles (N <= 64, aligned fp32 output) stage the result in
//                     shared-memory output boxes and store them by TMA while the next tile's K steps run, the residual
//                     having arrived by TMA during the K steps; halo tiles and outputs no tensor map expresses store straight
//                     from the accumulator fragments.
// Layout (P, Q), P * Q = NWG: the tile holds 64 P pixels x block_n = Q N channels, and consumer warpgroup w takes pixels
// 64 (w / Q) .. + 63 and channels N (w % Q) .. + N - 1 of it (Tc32Share).  All NWG warpgroups read the one converted box and
// the one weight tile of a step.  NWG = 2 (384 threads, N <= 128): (2, 1); NWG = 4 (640 threads, N <= 64): (4, 1), and
// (2, 2), (1, 4) at N = 64 (tc32_plan).  A K step is two dependent wgmma round trips (the promotion order above), so a warpgroup spends a few
// hundred clocks per step however small N is; four warpgroups overlap those round trips, and Q > 1 lets them do so on
// layers of 128 and more channels without converting the same activations once per N tile.  At 640 threads the register
// cap is 96, which holds the N = 64 step accumulator + sum.  vps_conv2d_tc32_plan picks (NWG, Q, N).
#include "conv_tc_common.cuh"

namespace {

constexpr int T32_CONV_WARPS = 3;           // warps 1..3 (warp 0 = TMA)
constexpr int T32_KC = 32;                  // channels per K step: 64-byte operand rows (SWIZZLE_64B), 2 x K16
constexpr int T32_MAX_N = 128;              // step accumulator + promoted sum: 2 x 64 registers per thread at N = 128
constexpr int T32_WIDE_MAX_N = 64;          // NWG = 4: 2 x 32 registers at N = 64 under the 96-register cap of 640 threads
// warpgroup 0: producer + converters; warpgroups 1..NWG: consumers
constexpr int t32_threads(int nwg) { return 128 * (nwg + 1); }
constexpr int T32_STAGE_SLOTS = 2;          // fp32 staging boxes (TMA -> converters)
constexpr int T32_PLANES = 2;               // operand planes: fp16(v), fp16(2^11 (v - fp16(v)))

__device__ unsigned int g_tc32_overflow = 0;     // activations / weights that exceeded the fp16 range of the main product

struct Tc32Extra {
  int rows;                  // activation rows (pixels) per A item: halo_h * halo_w, or the tile's 64 * P pixels
  int plane_bytes;           // bytes of one operand plane of an A item (rows * 64, padded to 1024)
  int stage_bytes;           // bytes of one fp32 staging slot (rows * 128, padded to 1024)
  int b_plane_bytes;         // block_n * 64: one weight plane of one step
  int dcn;                   // 1: the operand planes are produced by the deformable-sampling warps (no activation TMA)
  int wg_n;                  // Q: channel groups of consumer warpgroups; each warpgroup takes block_n / Q of the tile's channels
};

// Consumer warpgroup wg's share of a tile: pixels row0 .. row0 + 63, channels c_off .. c_off + n - 1 (n = block_n / Q).
struct Tc32Share {
  int row0, c_off, n;
};
__host__ __device__ __forceinline__ Tc32Share tc32_share(const ConvTcParams& p, const Tc32Extra& e, int wg) {
  const int n = p.block_n / e.wg_n, lg = e.wg_n >> 1;    // Q is 1, 2 or 4: shifts, not divisions, in the epilogue
  return {64 * (wg >> lg), n * (wg & (e.wg_n - 1)), n};
}

// the fused DCN kernel is bound by its sampling warps (CUDA-core issue + L1 latency), so it runs 4 warpgroups: warp 0 = weight
// TMA, warps 1-3 and 12-15 = 7 sampling warps, warpgroups 1 and 2 = consumers.  setmaxnreg moves registers from warpgroups 0
// and 3 to the consumers, whose 176 hold the step accumulator and the promoted sum at N = 128 per warpgroup.  Each sample is
// taken once per tile, so a tile spans every output channel where it can (dcn32_plan):
//   split-M: 128-pixel tile, warpgroup w takes pixels 64 w .. 64 w + 63 and all bn channels of the tile;
//   split-N:  64-pixel tile, both warpgroups read the same operand planes, warpgroup w takes channels w bn .. w bn + bn - 1.
constexpr int DCN32_THREADS = 512;
constexpr int DCN32_GATHER_WARPS = 7;
constexpr int DCN32_MAX_N = 128;                         // per consumer warpgroup
constexpr int DCN32_LO_REGS = 80, DCN32_HI_REGS = 176;   // warpgroups 0, 3 / consumer warpgroups 1, 2
// __launch_bounds__(512, 1) gives every thread 128 registers: a split asking for more than that pool makes setmaxnreg.inc
// wait forever
static_assert(128 * (2 * DCN32_LO_REGS + 2 * DCN32_HI_REGS) == DCN32_THREADS * (65536 / DCN32_THREADS),
              "the DCN register split must use exactly the launch allocation");
static_assert(DCN32_LO_REGS % 8 == 0 && DCN32_HI_REGS % 8 == 0 && DCN32_LO_REGS >= 24 && DCN32_HI_REGS <= 256,
              "setmaxnreg counts are multiples of 8 in [24, 256]");

struct Ring32 {
  uint32_t s_base, s_bytes;      // staging ring
  uint32_t a_base, a_bytes;      // operand-plane ring (T32_PLANES planes per slot)
  uint32_t b_base, b_bytes;      // weight ring (T32_PLANES planes per slot)
  uint32_t e_base, bias_base;    // TMA epilogue: the consumers' output boxes, their block_n bias values
  uint32_t setup_base;           // DCN: the tile's sampling set-up table
  uint32_t bar_base;
  uint32_t smem;                 // the launch's dynamic shared memory: all of the above + 1 KB of slack for aligning the base
  __device__ __forceinline__ uint32_t sfull(int s) const { return bar_base + 8u * s; }
  __device__ __forceinline__ uint32_t sempty(int s) const { return bar_base + 8u * (MAX_STAGES + s); }
  __device__ __forceinline__ uint32_t pfull(int s) const { return bar_base + 8u * (2 * MAX_STAGES + s); }
  __device__ __forceinline__ uint32_t pempty(int s) const { return bar_base + 8u * (3 * MAX_STAGES + s); }
  __device__ __forceinline__ uint32_t bfull(int s) const { return bar_base + 8u * (4 * MAX_STAGES + s); }
  __device__ __forceinline__ uint32_t bempty(int s) const { return bar_base + 8u * (5 * MAX_STAGES + s); }
  __device__ __forceinline__ uint32_t unit_ctr() const { return bar_base + 8u * (6 * MAX_STAGES); }   // DCN sampling units
  __device__ __forceinline__ uint32_t rfull(int wg) const { return bar_base + 8u * (6 * MAX_STAGES + 1 + wg); }  // residual box
};
constexpr int T32_NBAR = 6 * MAX_STAGES;
constexpr int T32_BAR_BYTES = 8 * (T32_NBAR + 2 + 4);
// TMA epilogue: a warpgroup's 64 x N result is stored as N / t32_box_c(N) boxes of t32_box_c(N) channels (128- or 64-byte
// rows, SWIZZLE_128B / SWIZZLE_64B) x 64 pixels (min(tw, 64) wide)
constexpr int t32_box_c(int n) { return n >= 32 ? 32 : 16; }
// At N = 128 the sum alone takes 64 of the 168 registers of a 384-thread CTA, and the TMA epilogue's unrolled pass over it
// spills around the slow-path call of the sigmoid's IEEE division; those tiles keep the fragment epilogue.
constexpr int T32_EPI_MAX_N = 64;

// Shared memory of the tc32 kernels from the 1024-byte aligned `base`, in this order: the convolution's staging ring,
// operand-plane ring, weight ring, with the TMA epilogue the 64 x N output boxes and N bias values of each of the nwg consumer
// warpgroups, the DCN's set-up table, then the barriers.  The ring slots are multiples of 1 KB, so every region after them is
// 1024-byte aligned.
__host__ __device__ __forceinline__ Ring32 ring32(uint32_t base, const ConvTcParams& p, const Tc32Extra& e, int nwg, bool epi_tma,
                                                  bool dcn) {
  Ring32 rg;
  const uint32_t n = (uint32_t)(p.block_n / e.wg_n);
  rg.s_base = base; rg.s_bytes = dcn ? 0u : (uint32_t)e.stage_bytes;
  rg.a_base = rg.s_base + T32_STAGE_SLOTS * rg.s_bytes; rg.a_bytes = (uint32_t)T32_PLANES * (uint32_t)e.plane_bytes;
  rg.b_base = rg.a_base + (uint32_t)p.a_stages * rg.a_bytes; rg.b_bytes = (uint32_t)T32_PLANES * (uint32_t)e.b_plane_bytes;
  rg.e_base = rg.b_base + (uint32_t)p.b_stages * rg.b_bytes;
  rg.bias_base = rg.e_base + (epi_tma ? 64u * nwg * n * 4u : 0u);
  rg.setup_base = rg.bias_base + (epi_tma ? (uint32_t)nwg * n * 4u : 0u);
  rg.bar_base = rg.setup_base + (dcn ? (uint32_t)dcn_setup_bytes(e.rows) : 0u);
  rg.smem = rg.bar_base + T32_BAR_BYTES + 1024u - base;
  return rg;
}

// The K walk of a tile, which every role follows: T32_KC channels of one filter tap per step, chunk-major and tap-minor
// (a loop over chunks around a loop over Tap).  An A item -- one converted or sampled box -- feeds all taps of a chunk in
// halo mode and one step otherwise.  The second K16 slab of a step is padding only in the last chunk, when p.nk_last is 1.
struct Tc32Walk {
  int chunks, taps, kw;
  bool halo;
  __host__ __device__ __forceinline__ int steps() const { return chunks * taps; }
  __host__ __device__ __forceinline__ int items() const { return chunks * (halo ? 1 : taps); }
  __device__ __forceinline__ bool opens_item(int tap) const { return !halo || tap == 0; }
};
__host__ __device__ __forceinline__ Tc32Walk tc32_walk(const ConvTcParams& p) { return {p.cin_chunks, p.kh * p.kw, p.kw, p.halo != 0}; }

// ---------------------------------------------------------------- warp 0: TMA producer
__device__ __forceinline__ void producer32(const ConvTcParams& p, const Tc32Extra& e, const Ring32& rg, const CUtensorMap* tmA,
                                           const CUtensorMap* tmB) {
  const Tc32Walk walk = tc32_walk(p);
  const uint32_t a_box_bytes = (uint32_t)p.a_box_bytes, b_bytes = (uint32_t)T32_PLANES * (uint32_t)e.b_plane_bytes;
  const int bn = p.block_n;
  RingPos sp, bp;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const TileCoord t = tile_coord(p, tile);
    const int x_base = t.tx * p.tw * p.sw - p.pw_[t.prob];
    const int y_base = t.ty * p.th * p.sh - p.ph_[t.prob];
    const int n0 = t.n_idx * bn;
    for (int cc = 0; cc < walk.chunks; ++cc) {
      for (Tap tap; tap.k < walk.taps; tap.next(walk.kw)) {
        if (!e.dcn && walk.opens_item(tap.k)) {
          sp.wait_empty(rg.sempty(sp.slot));
          if (elect_one()) {
            mbar_expect_tx(rg.sfull(sp.slot), a_box_bytes);
            tma_load_4d(rg.s_base + sp.slot * rg.s_bytes, tmA, rg.sfull(sp.slot), cc * T32_KC,
                        walk.halo ? x_base : x_base + tap.s, walk.halo ? y_base : y_base + tap.r, t.img);
          }
          sp.next(T32_STAGE_SLOTS);
        }
        bp.wait_empty(rg.bempty(bp.slot));
        if (elect_one()) {     // both weight planes of this (tap, chunk) in one 5-D box
          mbar_expect_tx(rg.bfull(bp.slot), b_bytes);
          tma_load_5d(rg.b_base + bp.slot * rg.b_bytes, tmB, rg.bfull(bp.slot), cc * T32_KC, n0, tap.k, t.prob, 0);
        }
        bp.next(p.b_stages);
      }
    }
  }
}

// ---------------------------------------------------------------- warps 1..3: fp32 box -> fp16 main / correction operand planes
__device__ __forceinline__ void converter32(const ConvTcParams& p, const Tc32Extra& e, const Ring32& rg, int ctid, int nthreads) {
  const int items_per_tile = tc32_walk(p).items();
  const int tasks = e.rows * 4;                       // 8 channels (two 16-byte fp32 chunks) per task
  RingPos sp, ap;
  bool over = false;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    for (int it = 0; it < items_per_tile; ++it) {
      sp.wait_full(rg.sfull(sp.slot));
      ap.wait_empty(rg.pempty(ap.slot));
      const uint32_t src = rg.s_base + sp.slot * rg.s_bytes;
      const uint32_t dst = rg.a_base + ap.slot * rg.a_bytes;
      for (int task = ctid; task < tasks; task += nthreads) {
        const int r = task >> 2, j = task & 3;
        // staging rows are 128 bytes, SWIZZLE_128B (written by TMA): 16-byte chunk c of row r sits at chunk c ^ (r & 7)
        const uint32_t row_s = src + (uint32_t)r * 128u;
        const uint32_t sw = (uint32_t)(r & 7);
        float v[8];
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3])
                     : "r"(row_s + (((uint32_t)(2 * j) ^ sw) << 4)));
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v[4]), "=f"(v[5]), "=f"(v[6]), "=f"(v[7])
                     : "r"(row_s + (((uint32_t)(2 * j + 1) ^ sw) << 4)));
        uint32_t hp[4], lp[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) split_pair_f16(v[2 * q], v[2 * q + 1], hp[q], lp[q], over);
        // operand planes: 64-byte rows, SWIZZLE_64B: 16-byte chunk j of row r sits at chunk j ^ ((r >> 1) & 3)
        const uint32_t off = (uint32_t)r * 64u + ((((uint32_t)j) ^ ((uint32_t)(r >> 1) & 3u)) << 4);
        const uint32_t pm = dst + off, pl = pm + (uint32_t)e.plane_bytes;
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(pm), "r"(hp[0]), "r"(hp[1]), "r"(hp[2]), "r"(hp[3]) : "memory");
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(pl), "r"(lp[0]), "r"(lp[1]), "r"(lp[2]), "r"(lp[3]) : "memory");
      }
      mbar_arrive(rg.sempty(sp.slot));                                   // staging slot may be refilled
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // generic-proxy writes -> tensor-core reads
      mbar_arrive(rg.pfull(ap.slot));
      sp.next(T32_STAGE_SLOTS);
      ap.next(p.a_stages);
    }
  }
  if (over) atomicAdd(&g_tc32_overflow, 1u);
}


// ---------------------------------------------------------------- DCNv1: the sampling warps fill the operand planes (fused im2col)
// deformable_im2col (deform_conv_cuda_kernel.cu:189-242) for a 3x3 / stride 1 / pad 1 / dilation 1 kernel with one deformable
// group: column (tap k, channel c) of output pixel (y, x) = bilinear sample of x[c] at (y - 1 + k/3 + dy_k, x - 1 + k%3 + dx_k),
// zero outside (-1, H) x (-1, W), corner taps outside the image contribute 0.  The sampled fp32 value is split into the two
// fp16 planes straight into the operand ring -- the 9x column matrix (1.2 GB per P2 layer in fp32) never exists.  K steps run
// chunk-major / tap-minor: the nine taps of a 32-channel chunk re-read the same few KB of input from L1.  A tile has e.rows
// (128 or 64) pixels, i.e. e.rows / 8 sampling units per K step.
__device__ __forceinline__ void dcn_gather32(const ConvTcParams& p, const Tc32Extra& e, const DcnParams<float>& d, const Ring32& rg,
                                             uint32_t setup_base, uint32_t ctr_addr, int gtid) {
  constexpr int NT = 32 * DCN32_GATHER_WARPS;
  const int lane = gtid & 31;
  const int j = lane & 3;                    // 8-channel group of the 32-channel chunk
  const int rlog = e.rows == 128 ? 7 : 6, ulog = rlog - 3;
  const Tc32Walk walk = tc32_walk(p);
  const int steps_per_tile = walk.steps();
  const uint32_t units_per_tile = (uint32_t)steps_per_tile << ulog;   // a unit = 8 rows (pixels) x 32 channels of one K step
  uint32_t step_base = 0;                    // K steps of the tiles this CTA has finished
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const TileCoord t = tile_coord(p, tile);
    if (gtid == 0) asm volatile("st.volatile.shared.u32 [%0], %1;" ::"r"(ctr_addr), "r"(0u) : "memory");
    // ---- sampling set-up of all (tap, pixel) pairs of this tile
    for (int item = gtid; item < 9 << rlog; item += NT) {
      const int k = item >> rlog, r = item & ((1 << rlog) - 1);
      const int ty_in = r / p.tw, tx_in = r - ty_in * p.tw;
      dcn_setup_entry(d, setup_base + (uint32_t)item * 32u, t.img, t.ty * p.th + ty_in, t.tx * p.tw + tx_in, k);
    }
    asm volatile("bar.sync 1, %0;" ::"n"(NT) : "memory");
    // ---- units are claimed dynamically (any number of gather warps stays balanced; a warp may run ahead into the next
    //      K step's ring slot): unit u = (K step u / units, rows 8 * (u % units) ..), K steps chunk-major / tap-minor
    while (true) {
      uint32_t u = 0;
      if (lane == 0) asm volatile("atom.shared.add.u32 %0, [%1], 1;" : "=r"(u) : "r"(ctr_addr) : "memory");
      u = __shfl_sync(0xffffffffu, u, 0);
      if (u >= units_per_tile) break;
      const uint32_t step = u >> ulog, part = u & ((1u << ulog) - 1u);
      const uint32_t cc = step / (uint32_t)walk.taps, k = step - cc * (uint32_t)walk.taps;
      const RingPos ap = RingPos::at(step_base + step, (uint32_t)p.a_stages);   // K step counted over this CTA's tiles
      ap.wait_empty(rg.pempty(ap.slot));
      const uint32_t dst = rg.a_base + ap.slot * rg.a_bytes;
      const int r = (int)(part * 8u) + (lane >> 2);
      const float* xc = d.x + cc * T32_KC + j * 8;
      {
        const uint32_t sa = setup_base + (uint32_t)((k << rlog) + r) * 32u;
        float wq[4];
        int oq[4];
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(wq[0]), "=f"(wq[1]), "=f"(wq[2]), "=f"(wq[3]) : "r"(sa));
        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(oq[0]), "=r"(oq[1]), "=r"(oq[2]), "=r"(oq[3]) : "r"(sa + 16u));
        float acc[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = 0.f;
        // the reference accumulates w1*v1 + w2*v2 + w3*v3 + w4*v4 left to right (dmcn_im2col_bilinear); same order here
        float4 v0[4], v1[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {           // corners outside the image carry weight 0 (branch-free: finite inputs)
          v0[c] = __ldg(reinterpret_cast<const float4*>(xc + oq[c]));
          v1[c] = __ldg(reinterpret_cast<const float4*>(xc + oq[c]) + 1);
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          acc[0] += wq[c] * v0[c].x; acc[1] += wq[c] * v0[c].y; acc[2] += wq[c] * v0[c].z; acc[3] += wq[c] * v0[c].w;
          acc[4] += wq[c] * v1[c].x; acc[5] += wq[c] * v1[c].y; acc[6] += wq[c] * v1[c].z; acc[7] += wq[c] * v1[c].w;
        }
        uint32_t hp[4], lp[4];
        bool over = false;
#pragma unroll
        for (int q = 0; q < 4; ++q) split_pair_f16(acc[2 * q], acc[2 * q + 1], hp[q], lp[q], over);
        if (over) atomicAdd(&g_tc32_overflow, 1u);
        const uint32_t off = (uint32_t)r * 64u + ((((uint32_t)j) ^ ((uint32_t)(r >> 1) & 3u)) << 4);
        const uint32_t pm = dst + off, pl = pm + (uint32_t)e.plane_bytes;
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(pm), "r"(hp[0]), "r"(hp[1]), "r"(hp[2]), "r"(hp[3]) : "memory");
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(pl), "r"(lp[0]), "r"(lp[1]), "r"(lp[2]), "r"(lp[3]) : "memory");
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy writes -> tensor-core reads
      __syncwarp();
      if (lane == 0) mbar_arrive(rg.pfull(ap.slot));                   // e.rows / 8 warp-units complete a K step's operand planes
    }
    step_base += (uint32_t)steps_per_tile;
    asm volatile("bar.sync 1, %0;" ::"n"(NT) : "memory");      // the set-up table and the unit counter are rewritten for the next tile
  }
}

// ---------------------------------------------------------------- TMA epilogue
// Byte address of (pixel q of the warpgroup, tile channel c) in the warpgroup's output boxes, swizzled as TMA reads and writes
// them: 16-byte chunk k of pixel row q sits at k ^ (q & 7) (SWIZZLE_128B, 32-channel rows) or k ^ ((q >> 1) & 3)
// (SWIZZLE_64B, 16-channel rows).  The float2 stores of a warp then cover every bank twice: two wavefronts, no conflict.
template <int N>
__device__ __forceinline__ uint32_t epi_box_addr(uint32_t box, int q, int c) {
  constexpr int BC = t32_box_c(N);
  const uint32_t k = (uint32_t)((c % BC) >> 2);
  const uint32_t sw = BC == 32 ? (uint32_t)(q & 7) : (uint32_t)((q >> 1) & 3);
  return box + (uint32_t)(c / BC) * (64u * BC * 4u) + (uint32_t)q * (BC * 4u) + ((k ^ sw) << 4) + (uint32_t)(c & 3) * 4u;
}

// The output box of warpgroup wg in tile `tile` (its tc32_share): channels n0.., pixels (x0, y0).. of image img; live = any
// pixel in range.  Recomputed where it is needed rather than held in registers across the K steps.
struct EpiBox {
  int n0, x0, y0, img;
  bool live;
};
__device__ __forceinline__ EpiBox epi_box(const ConvTcParams& p, const Tc32Extra& e, int tile, int wg) {
  const TileCoord t = tile_coord(p, tile);
  const Tc32Share s = tc32_share(p, e, wg);
  EpiBox b;
  b.n0 = t.n_idx * p.block_n + s.c_off; b.img = t.img;
  b.x0 = t.tx * p.tw + s.row0 % p.tw; b.y0 = t.ty * p.th + s.row0 / p.tw;
  b.live = b.x0 < p.ow && b.y0 < p.oh;
  return b;
}

// One warpgroup's 64 x N result -> its output boxes (residual read from, and the result written over, the box the TMA load
// filled) -> TMA store of the boxes.  The store stays in flight while the warpgroup runs the next tile's K steps.  The
// boxes are written again only after the leader's cp.async.bulk.wait_group.read, i.e. once the store has read them.
template <int N>
__device__ __forceinline__ void epi_tma32(const ConvTcParams& p, const Tc32Extra& e, const CUtensorMap* tmY, const float (&d)[N / 2], uint32_t box,
                                          uint32_t bias_s, float bias_v, uint32_t rbar, uint32_t rphase, int wg, int tile) {
  constexpr int BC = t32_box_c(N);
  const int i = threadIdx.x & 127, lane = threadIdx.x & 31, w = i >> 5;
  if (i < N) asm volatile("st.shared.f32 [%0], %1;" ::"r"(bias_s + 4u * i), "f"(bias_v) : "memory");
  if (i == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");        // bias visible, boxes free
  if (p.res) mbar_wait(rbar, rphase);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = 16 * w + (lane >> 2) + 8 * h;
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
      const int c = 8 * j + 2 * (lane & 3);
      const uint32_t a = epi_box_addr<N>(box, q, c);
      float b0, b1, r0 = 0.f, r1 = 0.f;
      asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(b0), "=f"(b1) : "r"(bias_s + 4u * c));
      if (p.res) asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(r0), "=f"(r1) : "r"(a));
      const float2 v = epi_math(p, d[4 * j + 2 * h], d[4 * j + 2 * h + 1], b0, b1, r0, r1);
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(v.x), "f"(v.y) : "memory");
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");        // generic-proxy writes -> TMA reads
  asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
  const EpiBox eb = epi_box(p, e, tile, wg);
  if (i == 0 && eb.live) {
#pragma unroll
    for (int b = 0; b < N / BC; ++b) tma_store_4d(tmY, box + (uint32_t)b * (64u * BC * 4u), eb.n0 + b * BC, eb.x0, eb.y0, eb.img);
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  }
}

// ---------------------------------------------------------------- consumer warpgroups: MMA, promotion, epilogue
// Per K step: acc = A2*B + A*B2 (fresh chain), acc *= 2^-11, acc += A*B, sum += acc (round to nearest).  The operand planes
// and weight tiles of the step are released as soon as its MMAs have completed (one arrival per consumer warpgroup).
// With the TMA epilogue the leader loads the tile's residual boxes after the first K step: by then the previous tile's store
// has long read the boxes, so its wait does not hold up the first MMAs.
// The warpgroup's share of the tile (tc32_share, N = its channel count): pixels row0 .. row0 + 63, tile channels
// c_off .. c_off + N - 1, whose weight rows start at byte c_off * 64 of each weight plane.  The epilogue recomputes the share
// rather than holding it in registers across the K steps.
template <int N, bool TMA_EPI>
__device__ __forceinline__ void consumer32(const ConvTcParams& p, const Tc32Extra& e, const Ring32& rg, int wg, const CUtensorMap* tmY,
                                           const CUtensorMap* tmR) {
  constexpr int BC = t32_box_c(N);
  const bool leader = (threadIdx.x & 127) == 0;
  constexpr bool epi_tma = TMA_EPI;
  const Tc32Share s = tc32_share(p, e, wg);
  const uint32_t b_base = rg.b_base + (uint32_t)s.c_off * 64u;     // 64-byte weight rows
  const uint32_t box = rg.e_base + (uint32_t)wg * (64u * N * 4u), bias_s = rg.bias_base + (uint32_t)wg * (N * 4u);
  const uint32_t rbar = rg.rfull(wg);
  uint32_t rphase = 0;
  // The K walk is Tc32Walk's, spelled out: the same expressions through Tc32Walk's members make ptxas allocate 4 more
  // registers to the 640-thread TMA-epilogue kernel.
  const bool halo = p.halo != 0;
  const int ntaps = p.kh * p.kw, kw = p.kw, last_cc = p.cin_chunks - 1;
  const uint32_t a_pitch = halo ? (uint32_t)p.halo_w * 64u : 512u;      // byte distance of the A planes' 8-row groups
  const uint64_t a_hi = desc_hi(64u, a_pitch), b_hi = desc_hi(64u, 512u);
  // this warpgroup's 64 pixels: row0 / 8 halo rows (of 8 tile pixels each) down, or row0 dense rows
  const uint32_t a_wg = halo ? (uint32_t)(s.row0 >> 3) * a_pitch : (uint32_t)s.row0 * 64u;
  const uint32_t plane = (uint32_t)e.plane_bytes, b_plane = (uint32_t)e.b_plane_bytes;
  float acc[N / 2], sum[N / 2];
  RingPos ap, bp;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    float bias_v = 0.f;
    if (epi_tma) {        // this thread's bias value of the tile: loaded now, written to shared memory in the epilogue
      const int c = tile_coord(p, tile).n_idx * p.block_n + tc32_share(p, e, wg).c_off + (threadIdx.x & 127);
      if (p.bias && (threadIdx.x & 127) < N && c < p.cout) bias_v = __ldg(p.bias + c);
    }
#pragma unroll
    for (int i = 0; i < N / 2; ++i) sum[i] = 0.f;
    for (int cc = 0; cc <= last_cc; ++cc) {
      const bool two = cc != last_cc || p.nk_last > 1;
      uint32_t a_item = 0;
      for (Tap tap; tap.k < ntaps; tap.next(kw)) {
        if (!halo || tap.k == 0) {
          ap.wait_full(rg.pfull(ap.slot));
          a_item = rg.a_base + ap.slot * rg.a_bytes + a_wg;
        }
        bp.wait_full(rg.bfull(bp.slot));
        const uint32_t a_addr = halo ? a_item + (uint32_t)tap.r * a_pitch + (uint32_t)tap.s * 64u : a_item;
        const uint32_t b_addr = b_base + bp.slot * rg.b_bytes;
        const uint64_t A = desc_at(a_hi, a_addr), A2 = desc_at(a_hi, a_addr + plane);
        const uint64_t B = desc_at(b_hi, b_addr), B2 = desc_at(b_hi, b_addr + b_plane);
        wg::fence();
        wg::Mma<N, true>::run(acc, A2, B, 0u);
        if (two) wg::Mma<N, true>::run(acc, A2 + 2, B + 2, 1u);
        wg::Mma<N, true>::run(acc, A, B2, 1u);
        if (two) wg::Mma<N, true>::run(acc, A + 2, B2 + 2, 1u);
        wg::commit();
        wg::wait<0>();
        wg::fence_regs(acc);
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc[i] *= T32_LO_INV;
        wg::fence();
        wg::Mma<N, true>::run(acc, A, B, 1u);
        if (two) wg::Mma<N, true>::run(acc, A + 2, B + 2, 1u);
        wg::commit();
        wg::wait<0>();
        wg::fence_regs(acc);
#pragma unroll
        for (int i = 0; i < N / 2; ++i) sum[i] += acc[i];
        const bool item_done = !halo || tap.k == ntaps - 1;
        if (leader) {
          mbar_arrive(rg.bempty(bp.slot));
          if (item_done) mbar_arrive(rg.pempty(ap.slot));
          if (epi_tma && p.res && cc == 0 && tap.k == 0) {
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            const EpiBox eb = epi_box(p, e, tile, wg);
            if (eb.live) {
              mbar_expect_tx(rbar, 64u * N * 4u);
#pragma unroll
              for (int b = 0; b < N / BC; ++b)
                tma_load_4d(box + (uint32_t)b * (64u * BC * 4u), tmR, rbar, eb.n0 + b * BC, eb.x0, eb.y0, eb.img);
            } else {
              mbar_arrive(rbar);
            }
          }
        }
        ap.next(p.a_stages, item_done);
        bp.next(p.b_stages);
      }
    }
    if (epi_tma) {
      epi_tma32<N>(p, e, tmY, sum, box, bias_s, bias_v, rbar, rphase, wg, tile);
      if (p.res) rphase ^= 1u;
    } else {
      const Tc32Share s = tc32_share(p, e, wg);
      epi_frag<N, 4>(p, sum, tile, s.row0, s.c_off);
    }
  }
  // the boxes must stay allocated until the last store has read them, and the stores must be complete before the grid is
  // (a dependent launch's griddepcontrol.wait reads the output)
  if (epi_tma && leader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

template <int NWG, bool TMA_EPI>
__device__ __forceinline__ void consumer32_n(const ConvTcParams& p, const Tc32Extra& e, const Ring32& rg, int wg,
                                             const CUtensorMap* tmY, const CUtensorMap* tmR) {
  switch (p.block_n / e.wg_n) {
    case 16: consumer32<16, TMA_EPI>(p, e, rg, wg, tmY, tmR); break;
    case 32: consumer32<32, TMA_EPI>(p, e, rg, wg, tmY, tmR); break;
    case 64: consumer32<64, TMA_EPI>(p, e, rg, wg, tmY, tmR); break;
    default:
      if constexpr (NWG == 2 && !TMA_EPI) consumer32<T32_MAX_N, false>(p, e, rg, wg, tmY, tmR);
      else __trap();                      // the host plan pairs N > T32_EPI_MAX_N with neither NWG = 4 nor the TMA epilogue
      break;
  }
}

// barrier arrival counts: sfull / bfull = one TMA arrival, sempty = every converter thread, pfull = every converter thread
// (convolution) or one arrival per 8-row sampling unit (DCN), pempty / bempty = one arrival per consumer warpgroup
__device__ __forceinline__ void init_bars32(const Ring32& rg, uint32_t pfull_count, uint32_t sempty_count, uint32_t consumers) {
  for (int i = threadIdx.x & 31; i < T32_NBAR; i += 32) {
    const int kind = i / MAX_STAGES;       // 0 sfull, 1 sempty, 2 pfull, 3 pempty, 4 bfull, 5 bempty
    const uint32_t count = kind == 1 ? sempty_count : (kind == 2 ? pfull_count : ((kind == 3 || kind == 5) ? consumers : 1u));
    mbar_init(rg.bar_base + 8u * i, count);
  }
  if ((threadIdx.x & 31) < 4) mbar_init(rg.rfull(threadIdx.x & 31), 1u);     // residual boxes: one TMA arrival
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// ---------------------------------------------------------------- kernel
template <int NWG, bool TMA_EPI>
__global__ void __launch_bounds__(t32_threads(NWG), 1)
conv_igemm_tc32_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tmR, const ConvTcParams p,
                       const Tc32Extra e) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const Ring32 rg = ring32((smem_u32(smem_raw) + 1023u) & ~1023u, p, e, NWG, TMA_EPI, false);
  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0);     // warp-uniform role index (wgmma issue is not treated as divergent)
  if (warp == 0) init_bars32(rg, 32 * T32_CONV_WARPS, 32 * T32_CONV_WARPS, NWG);
  if (threadIdx.x == 32) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    if (TMA_EPI) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmY) : "memory");
      if (p.res) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmR) : "memory");
    }
  }
  __syncthreads();
  // programmatic dependent launch: the prologue above overlaps the previous kernel's tail (see conv_tc.cu)
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (warp == 0) producer32(p, e, rg, &tmA, &tmB);
  else if (warp < 4) converter32(p, e, rg, (int)threadIdx.x - 32, 32 * T32_CONV_WARPS);
  else consumer32_n<NWG, TMA_EPI>(p, e, rg, (warp - 4) >> 2, &tmY, &tmR);
}

// ---------------------------------------------------------------- fused DCNv1 kernel (same pipeline, sampling warps feed the ring)
__global__ void __launch_bounds__(DCN32_THREADS, 1)
dcn_igemm_tc32_kernel(const __grid_constant__ CUtensorMap tmB, const ConvTcParams p, const Tc32Extra e, const DcnParams<float> d) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const Ring32 rg = ring32((smem_u32(smem_raw) + 1023u) & ~1023u, p, e, 2, false, true);
  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0);     // warp-uniform role index (wgmma issue is not treated as divergent)
  if (warp == 0) init_bars32(rg, (uint32_t)e.rows / 8u, 1, 2);
  if (threadIdx.x == 32) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
  __syncthreads();
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (warp >= 4 && warp < 12) {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(DCN32_HI_REGS));
    const int wg = (warp - 4) >> 2;
    switch (p.block_n / e.wg_n) {
      case 16: consumer32<16, false>(p, e, rg, wg, nullptr, nullptr); break;
      case 32: consumer32<32, false>(p, e, rg, wg, nullptr, nullptr); break;
      case 64: consumer32<64, false>(p, e, rg, wg, nullptr, nullptr); break;
      default: consumer32<DCN32_MAX_N, false>(p, e, rg, wg, nullptr, nullptr); break;
    }
  } else {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(DCN32_LO_REGS));
    if (warp == 0) producer32(p, e, rg, &tmB, &tmB);
    else dcn_gather32(p, e, d, rg, rg.setup_base, rg.unit_ctr(), warp < 4 ? (int)threadIdx.x - 32 : (int)threadIdx.x - 384 + 96);
  }
}

// ---------------------------------------------------------------- weight packing
// two planes of fp16 words, each [nprob][cout_pad][tap][cin_pad]:  B = fp16(w),  B2 = fp16(2^11 * (w - B))
__global__ void pack_weights_tc32_kernel(const float* __restrict__ src, const float* __restrict__ scale, unsigned short* __restrict__ bm,
                                         unsigned short* __restrict__ bl, int cout, int cin, int kh, int kw, int cout_pad,
                                         int cin_pad, int transposed) {
  const int64_t total = (int64_t)cout_pad * kh * kw * cin_pad;
  bool over = false;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = packed_weight(src, scale, i, cout, cin, kh, kw, cin_pad, transposed);
    unsigned short h, l;
    split_f16(v, h, l);
    over = over || f16_over(v);
    bm[i] = h;
    bl[i] = l;
  }
  if (over) atomicAdd(&g_tc32_overflow, 1u);
}

inline int64_t plane_elems(int cout, int cin, int kh, int kw) {
  const int64_t cout_pad = (cout + 15) / 16 * 16, cin_pad = (cin + T32_KC - 1) / T32_KC * T32_KC;
  return cout_pad * kh * kw * cin_pad;
}

// Packed weights [plane][prob][cout_pad][tap][cin_pad] (vps_pack_weights_tc32): a box is {T32_KC channels, block_n rows} of
// one tap and problem in both planes.  `who` prefixes the error message.
bool encode_weights_tc32(CUtensorMap* m, const void* w, int nprob, int cout, int taps, int cin_pad, int block_n, const char* who) {
  const auto encode = vps::tensor_map_encoder();
  if (!encode) return false;
  const int cout_pad = (cout + 15) / 16 * 16;
  const int64_t n_plane = (int64_t)cout_pad * taps * cin_pad;
  cuuint64_t dims[5] = {(cuuint64_t)cin_pad, (cuuint64_t)cout_pad, (cuuint64_t)taps, (cuuint64_t)nprob, T32_PLANES};
  cuuint64_t strides[4] = {(cuuint64_t)taps * cin_pad * 2, (cuuint64_t)cin_pad * 2, (cuuint64_t)n_plane * 2,
                           (cuuint64_t)n_plane * nprob * 2};
  cuuint32_t box[5] = {(cuuint32_t)T32_KC, (cuuint32_t)block_n, 1, 1, T32_PLANES};
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  const CUresult r = encode(m, CU_TENSOR_MAP_DATA_TYPE_UINT16, 5, (void*)w, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { vps::set_error("%s: encode B failed (%d)", who, (int)r); return false; }
  return true;
}

constexpr int T32_SMEM_MAX = 227 * 1024 - 64;    // dynamic shared memory of a tc32 convolution

// One tc32 launch: the kernel parameters and the choices only the host needs.  Everything here follows from the shapes (and
// the SM count); the launchers launch exactly this plan and the plan queries report it.
struct Tc32Plan {
  ConvTcParams p;
  Tc32Extra e;
  int nwg;                   // convolution: consumer warpgroups, the tile holds 64 * nwg / e.wg_n output pixels
  int epi_tma;               // 1: TMA epilogue (output boxes in shared memory), 0: stores from the accumulator fragments
  int smem;                  // dynamic shared memory
};

// A tensor map can express the output (and the residual) of one problem written at unit output strides into fp32 tensors
// whose channel-slice base and pixel stride are 16-byte aligned.  The stride phases of a transposed convolution (nprob > 1,
// doubled output strides), bf16 outputs or residuals and unaligned slices keep the fragment epilogue.
bool tc32_epi_expressible(const vps_conv_args* a, int nprob) {
  if (nprob != 1 || a->oy_mul != 1 || a->ox_mul != 1 || a->y.dtype != VPS_F32) return false;
  const int64_t px = (int64_t)a->oy_off * a->y.w + a->ox_off;       // the first output pixel
  if ((((uintptr_t)a->y.ptr + px * a->y.cs * 4) & 15) || a->y.cs % 4) return false;
  if (a->res.ptr && (a->res.dtype != VPS_F32 || (((uintptr_t)a->res.ptr + px * a->res.cs * 4) & 15) || a->res.cs % 4))
    return false;
  return true;
}

// The tile of nwg consumer warpgroups in layout (nwg / wg_n, wg_n), n channels each, and its A items; tc32_plan sets the
// weight ring depth.
Tc32Plan tc32_tile(const vps_conv_args* a, int nprob, int nwg, int wg_n, int n) {
  Tc32Plan g = {};
  ConvTcParams& p = g.p;
  g.nwg = nwg;
  g.e.wg_n = wg_n;
  const int px = 64 * (nwg / wg_n), block_n = wg_n * n;
  p.halo = a->sh == 1 && a->sw == 1 && a->kh * a->kw > 1 && a->kh <= 8 && a->kw <= 8;
  // 8-pixel halo rows: the consumer's descriptors step one halo row per 8-row group
  const int tw = p.halo ? 8 : patch_tw(a->oh, a->ow, px, a->sh, a->sw);
  set_tiles(p, a, nprob, tw, px / tw, block_n, T32_KC);
  p.halo_w = tw + a->kw - 1;
  p.a_stages = p.halo ? 2 : 3;
  g.e.rows = p.halo ? (p.th + a->kh - 1) * p.halo_w : px;
  p.a_box_bytes = g.e.rows * 128;
  g.e.stage_bytes = (g.e.rows * 128 + 1023) / 1024 * 1024;
  g.e.plane_bytes = (g.e.rows * 64 + 1023) / 1024 * 1024;
  g.e.b_plane_bytes = block_n * 64;
  return g;
}

// (NWG, Q, N) minimising waves * (steps * step clocks + epilogue) over the candidates whose rings fit (>= 2 weight
// stages).  N (channels per warpgroup) is <= 128 at NWG 2 and <= 64 at NWG 4 (the register cap), and block_n = Q N is a
// power-of-two divisor of cout_pad.  The layouts: NWG 2 as (2, 1); NWG 4 as (4, 1), and as (2, 2) and (1, 4) at N = 64.
// Channel groups of fewer than 64 channels, and (1, 2) at NWG 2, never measured faster than a (P, 1) layout on the
// production shapes, so they are not candidates.  The step costs are fitted to H100 per-layer times of every candidate on
// the shapes of tools/diag_tc32.py (DESIGN.md §5.0) and add up rather than overlap:
//   * a fixed 410 clocks (the two dependent wgmma round trips, barrier waits), 70 more at 640 threads;
//   * the tensor pipe: 6 NWG MMAs of m64 x N x k16 at 2048 MAC/clk = 3 NWG N clocks; at NWG 2, 0.4 N more (one warpgroup's
//     longer MMA chain is hidden only by the other);
//   * the converters: 6 clocks per activation row they convert (an A item per step in flat mode, per channel chunk in halo
//     mode), so a tile that spans more channels converts each input row for more of them;
//   * the weight tile: 1 clock per 200 bytes of it.
// The epilogue costs 40 N + 1500 clocks per tile.  A shared-memory read term (every MMA reading its A and B slabs at
// 128 B/clk) did not fit the timings: (1, 4), which reads the most, is the fastest layout wherever it fits.
constexpr double T32_STEP_CLK = 410.0, T32_STEP_CLK_640 = 70.0, T32_MMA_CLK_N2 = 0.4, T32_CONV_CLK = 6.0, T32_B_BYTES_PER_CLK = 200.0;
int tc32_plan(const vps_conv_args* a, int nprob, Tc32Plan& out) {
  VPS_CHECK_ARG(nprob >= 1 && nprob <= MAX_PROB, "conv2d_tc32: nprob %d", nprob);
  VPS_CHECK_ARG(a->sh >= 1 && a->sh <= 2 && a->sw >= 1 && a->sw <= 2, "conv2d_tc32: stride must be 1 or 2");
  VPS_CHECK_ARG(a->kh >= 1 && a->kw >= 1 && a->cin >= 1 && a->cout >= 1 && a->oh >= 0 && a->ow >= 0 && a->x.n >= 0,
                "conv2d_tc32: bad geometry (k %dx%d, cin %d, cout %d, out %dx%d)", a->kh, a->kw, a->cin, a->cout, a->oh, a->ow);
  const int sms = vps::num_sms();
  if (sms <= 0) { vps::set_error("no device"); return VPS_E_NODEV; }
  const int cout_pad = (a->cout + 15) / 16 * 16;
  double best = -1.0;
  for (int wg_n = 1; wg_n <= 4; wg_n *= 2) {
    for (int nwg = 2; nwg <= 4; nwg += 2) {
      if (wg_n > 1 && nwg == 2) continue;
      for (int n = 16; n <= (nwg == 2 ? T32_MAX_N : T32_WIDE_MAX_N) && wg_n * n <= cout_pad; n *= 2) {
        if (cout_pad % (wg_n * n) || (wg_n > 1 && n != T32_WIDE_MAX_N)) continue;
        Tc32Plan g = tc32_tile(a, nprob, nwg, wg_n, n);
        g.p.b_stages = 2;
        if ((int)ring32(0, g.p, g.e, nwg, false, false).smem > T32_SMEM_MAX) continue;
        const int64_t tiles = g.p.total_tiles;
        const double waves = (double)((tiles + sms - 1) / sms);
        const double rows = g.p.halo ? (double)g.e.rows / (a->kh * a->kw) : (double)g.e.rows;
        const double step = T32_STEP_CLK + (nwg == 4 ? T32_STEP_CLK_640 : T32_MMA_CLK_N2 * n) + 3.0 * nwg * n + T32_CONV_CLK * rows +
                            (double)(g.p.block_n * 64 * T32_PLANES) / T32_B_BYTES_PER_CLK;
        const double t = waves * ((double)tc32_walk(g.p).steps() * step + 40.0 * n + 1500.0);
        if (best < 0 || t < best * 0.999) {
          best = t;
          out = g;
        }
      }
    }
  }
  if (best < 0) {
    vps::set_error("conv2d_tc32: ring does not fit (k %dx%d)", a->kh, a->kw);
    return VPS_E_ARG;
  }
  // Epilogue: the TMA epilogue on flat tiles (one A item per K step: 1x1 and strided layers, a few K steps per tile, so the
  // exposed epilogue was up to half of the layer) where it is expressible and its output boxes fit next to >= 2 weight
  // stages, giving up the third operand-plane slot if need be (NWG 4 at block_n 64: 256-pixel A items).  Halo tiles keep the
  // fragment epilogue: they run tens of K steps per tile, and the boxes would take the weight stages their taps stream
  // through (NWG 4 at block_n 32 drops from 6 to 2 and ran 13-16% slower; per-layer H100 timings in DESIGN.md §5.0).
  ConvTcParams& p = out.p;
  p.b_stages = 2;
  const auto epi_fits = [&] { return (int)ring32(0, p, out.e, out.nwg, true, false).smem <= T32_SMEM_MAX; };
  if (!p.halo && p.block_n / out.e.wg_n <= T32_EPI_MAX_N && tc32_epi_expressible(a, nprob)) {
    if (!epi_fits() && p.a_stages == 3) {
      p.a_stages = 2;
      if (!epi_fits()) p.a_stages = 3;
    }
    out.epi_tma = epi_fits();
  }
  p.b_stages = 0;
  const Ring32 rg = ring32(0, p, out.e, out.nwg, out.epi_tma, false);
  const int bst = (T32_SMEM_MAX - (int)rg.smem) / (int)rg.b_bytes;
  p.b_stages = bst > MAX_STAGES ? MAX_STAGES : bst;
  out.smem = (int)ring32(0, p, out.e, out.nwg, out.epi_tma, false).smem;
  return VPS_OK;
}

// Shared memory stays at most 132 KB so that L1 keeps room: the sampling warps read 4 x 128 B per (tap, pixel, 32-channel
// chunk) through L1, and the nine taps of a chunk re-read the same ~60 KB footprint of the tile.
constexpr int DCN32_SMEM_MAX = 132 * 1024;
// Clocks of the CTA's 7 sampling warps per 8-pixel x 32-channel unit, from per-layer H100 timings of the 128-pixel x 64
// tiling (DESIGN.md §5.0: about 120 ns at every layer and level; the units are latency bound, 7 in flight per CTA), and the
// latency floor of a consumer K step (two dependent wgmma round trips).
constexpr double DCN32_UNIT_CLK = 220.0, DCN32_STEP_CLK = 300.0;

// (layout, bn) minimising waves * (K steps * step clocks + epilogue), among those whose tile width divides cout_pad and whose
// rings fit.  A K step costs the larger of: the sampling of rows / 8 units; the consumers' latency floor or their 12 MMAs of
// m64 x bn x k16 (6 bn clocks of the tensor pipe); the weight tile (2 planes x block_n x 64 B) at the L2 rate of 56 B/clk.
// Every N tile samples the same input again, so a tile as wide as cout_pad samples each input once; narrower tiles win where
// the grid would otherwise leave SMs idle.  Equal costs go to the plan that samples less.
int dcn32_plan(const vps_conv_args* a, Tc32Plan& out) {
  const int sms = vps::num_sms();
  if (sms <= 0) { vps::set_error("no device"); return VPS_E_NODEV; }
  const int cout_pad = (a->cout + 15) / 16 * 16;
  double best = -1.0, best_units = 0.0;
  for (int split_n = 0; split_n <= 1; ++split_n) {
    const int rows = split_n ? 64 : 128;        // tile pixels: split-M or split-N
    const int tw = patch_tw(a->oh, a->ow, rows, 1, 1);
    for (int bn = 16; bn <= DCN32_MAX_N; bn *= 2) {
      const int block_n = split_n ? 2 * bn : bn;
      if (block_n > cout_pad || cout_pad % block_n) continue;
      Tc32Plan g = {};
      set_tiles(g.p, a, 1, tw, rows / tw, block_n, T32_KC);
      g.p.a_stages = 2;
      g.e.rows = rows; g.e.plane_bytes = rows * 64; g.e.b_plane_bytes = block_n * 64; g.e.dcn = 1; g.e.wg_n = split_n ? 2 : 1;
      const Ring32 rg = ring32(0, g.p, g.e, 2, false, true);
      const int bst = (DCN32_SMEM_MAX - (int)rg.smem) / (int)rg.b_bytes;
      if (bst < 2) continue;
      const int64_t tiles = g.p.total_tiles;
      const double waves = (double)((tiles + sms - 1) / sms);
      const double step = fmax(fmax(rows / 8 * DCN32_UNIT_CLK, fmax(DCN32_STEP_CLK, 6.0 * bn)), rg.b_bytes / 56.0);
      const double t = waves * ((double)tc32_walk(g.p).steps() * step + 40.0 * bn + 1500.0), units = waves * rows;
      if (best < 0 || t < best * 0.999 || (t <= best * 1.001 && units < best_units)) {
        best = t; best_units = units;
        g.p.b_stages = bst > 3 ? 3 : bst;
        g.smem = (int)ring32(0, g.p, g.e, 2, false, true).smem;
        out = g;
      }
    }
  }
  if (best < 0) {
    vps::set_error("deform_conv_tc32: no tiling fits (cout %d)", a->cout);
    return VPS_E_ARG;
  }
  return VPS_OK;
}

}  // namespace

extern "C" int64_t vps_packed_tc32_bytes(int cout, int cin, int kh, int kw, int nprob) {
  return plane_elems(cout, cin, kh, kw) * 2 * T32_PLANES * nprob;
}

// device address of the saturation counter (library-internal: the correlation's operand split in corr_tc.cu reports into the
// same flag)
extern "C" unsigned int* vps_tc32_overflow_flag() {
  unsigned int* p = nullptr;
  if (cudaGetSymbolAddress((void**)&p, g_tc32_overflow) != cudaSuccess) return nullptr;
  return p;
}

// number of converter / packing threads that met |value| > 65504 (or NaN) since the last reset; synchronises the device
extern "C" int vps_tc32_overflow(int reset) {
  unsigned int v = 0;
  if (cudaMemcpyFromSymbol(&v, g_tc32_overflow, sizeof(v)) != cudaSuccess) return -1;
  if (reset && v) {
    const unsigned int z = 0;
    cudaMemcpyToSymbol(g_tc32_overflow, &z, sizeof(z));
  }
  return (int)v;
}

// problem `prob` of `nprob` (the stride phases of a transposed convolution share one packed buffer; nprob = 1 otherwise)
extern "C" int vps_pack_weights_tc32(const float* w, const float* scale, void* dst, int cout, int cin, int kh, int kw,
                                     int transposed, int prob, int nprob, void* stream) {
  VPS_CHECK_ARG(nprob >= 1 && nprob <= MAX_PROB && prob >= 0 && prob < nprob, "pack_weights_tc32: prob %d of %d", prob, nprob);
  const int cout_pad = (cout + 15) / 16 * 16, cin_pad = (cin + T32_KC - 1) / T32_KC * T32_KC;
  const int64_t n = plane_elems(cout, cin, kh, kw);
  unsigned short* base = (unsigned short*)dst;
  unsigned short* bm = base + (int64_t)prob * n;
  unsigned short* bl = base + n * nprob + (int64_t)prob * n;
  const int blocks = (int)((n + 255) / 256 > 4096 ? 4096 : (n + 255) / 256);
  pack_weights_tc32_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, scale, bm, bl, cout, cin, kh, kw, cout_pad, cin_pad, transposed);
  VPS_CUDA_LAST("pack_weights_tc32");
  return VPS_OK;
}

// fp32 activations, fp32 (or bf16) output; args[i].w = the shared buffer of vps_pack_weights_tc32(.., prob i, nprob)
extern "C" int vps_conv2d_tc32_multi(const vps_conv_args* args, int nprob, void* stream) {
  VPS_CHECK_ARG(nprob >= 1 && nprob <= MAX_PROB, "conv2d_tc32: nprob %d", nprob);
  const vps_conv_args* a = &args[0];
  VPS_CHECK_ARG(a->x.dtype == VPS_F32, "conv2d_tc32: x must be fp32");
  VPS_CHECK_ARG(a->x.cs % 4 == 0 && ((uintptr_t)a->x.ptr & 15) == 0, "conv2d_tc32: x not 16B aligned (cs=%d)", a->x.cs);
  VPS_CHECK_ARG(a->cin == a->x.c, "conv2d_tc32: cin %d != x.c %d", a->cin, a->x.c);
  VPS_CHECK_ARG(((uintptr_t)a->w & 127) == 0, "conv2d_tc32: weights not aligned");
  for (int i = 0; i < nprob; ++i) {
    VPS_CHECK_ARG(args[i].w == a->w && args[i].x.ptr == a->x.ptr && args[i].y.ptr == a->y.ptr && args[i].kh == a->kh &&
                      args[i].kw == a->kw && args[i].oh == a->oh && args[i].ow == a->ow && args[i].cout == a->cout &&
                      args[i].bias == a->bias && args[i].act == a->act && args[i].oy_mul == a->oy_mul && args[i].ox_mul == a->ox_mul,
                  "conv2d_tc32_multi: problems must share geometry and the packed weight buffer");
  }
  Tc32Plan g;
  int st = tc32_plan(a, nprob, g);
  if (st != VPS_OK) return st;
  ConvTcParams& p = g.p;
  const int halo_h = p.th + p.kh - 1;
  VPS_CHECK_ARG(p.b_stages >= 2, "conv2d_tc32: ring does not fit (%d x %d px halo, bn %d)", halo_h, p.halo_w, p.block_n);
  st = set_problems(p, args, nprob, "conv2d_tc32");
  if (st != VPS_OK) return st;
  if (p.total_tiles == 0) return VPS_OK;

  CUtensorMap tmA, tmB;
  if (!vps::encode_nhwc(&tmA, a->x, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, T32_KC, p.halo ? p.halo_w : p.tw * a->sw,
                        p.halo ? halo_h : p.th * a->sh, a->sw, a->sh, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        "conv2d_tc32: encode A"))
    return VPS_E_CUDA;
  if (!encode_weights_tc32(&tmB, a->w, nprob, a->cout, a->kh * a->kw, p.cin_chunks * T32_KC, p.block_n, "conv2d_tc32"))
    return VPS_E_CUDA;
  // TMA epilogue: output and residual as [n][oh][ow][cout] from the first output pixel (a channel slice of a wider tensor
  // keeps its pixel stride); TMA clips the boxes at oh / ow / cout, so partial tiles and the neighbouring channels are safe
  CUtensorMap tmY = {}, tmR = {};
  if (g.epi_tma) {
    const int bc = t32_box_c(p.block_n / g.e.wg_n), box_w = p.tw < 64 ? p.tw : 64;
    const int64_t px = (int64_t)a->oy_off * a->y.w + a->ox_off;
    for (int m = 0; m < (a->res.ptr ? 2 : 1); ++m) {
      const vps_tensor& t = m ? a->res : a->y;          // the residual has the output's geometry
      vps_tensor v = t;
      v.ptr = (float*)t.ptr + px * t.cs; v.n = a->x.n; v.h = a->oh; v.w = a->ow; v.c = a->cout;
      if (!vps::encode_nhwc(m ? &tmR : &tmY, v, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, bc, box_w, 64 / box_w, 1, 1,
                            bc == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                            m ? "conv2d_tc32: encode residual" : "conv2d_tc32: encode output", &t))
        return VPS_E_CUDA;
    }
  }
#define VPS_TC32_LAUNCH(NWG, EPI)                                                                                              \
  launch_persistent<conv_igemm_tc32_kernel<NWG, EPI>>(p.total_tiles, t32_threads(NWG), g.smem, stream, "conv2d_tc32", tmA, tmB,  \
                                                      tmY, tmR, p, g.e)
  if (g.nwg == 4) return g.epi_tma ? VPS_TC32_LAUNCH(4, true) : VPS_TC32_LAUNCH(4, false);
  return g.epi_tma ? VPS_TC32_LAUNCH(2, true) : VPS_TC32_LAUNCH(2, false);
#undef VPS_TC32_LAUNCH
}

extern "C" int vps_conv2d_tc32(const vps_conv_args* a, void* stream) { return vps_conv2d_tc32_multi(a, 1, stream); }

extern "C" int vps_conv2d_tc32_plan(const vps_conv_args* a, int nprob, int* plan) {
  Tc32Plan g;
  const int st = tc32_plan(a, nprob, g);
  if (st != VPS_OK) return st;
  plan[0] = g.nwg; plan[1] = g.p.block_n; plan[2] = g.p.tw; plan[3] = g.p.th; plan[4] = g.p.halo; plan[5] = g.epi_tma;
  plan[6] = g.e.wg_n;
  return VPS_OK;
}


// Fused DCNv1 3x3 / stride 1 / pad 1 / dilation 1 / 1 deformable group in the tc32 precision (deform_conv.py:15-87 forward,
// deform_conv_cuda.cpp:152-260): x fp32 NHWC (c % 32 == 0), offset fp32 NHWC [.., 18] = (dy, dx) per tap,
// w = vps_pack_weights_tc32 buffer of the [cout, cin, 3, 3] kernel, y fp32 NHWC.  No bias (DeformConv has none).
extern "C" int vps_deform_conv_tc32(const vps_tensor* x, const vps_tensor* offset, const void* w, int cout, const vps_tensor* y,
                                    void* stream) {
  VPS_CHECK_ARG(x->dtype == VPS_F32 && offset->dtype == VPS_F32 && offset->c >= 18, "deform_conv_tc32: dtypes");
  VPS_CHECK_ARG(x->c % T32_KC == 0 && x->cs % 8 == 0 && ((uintptr_t)x->ptr & 31) == 0,
                "deform_conv_tc32: x must have cin %% 32 == 0 and 32-byte aligned pixel rows (256-bit sampling loads)");
  VPS_CHECK_ARG(offset->n == x->n && offset->h == x->h && offset->w == x->w && y->n == x->n && y->h == x->h && y->w == x->w &&
                    y->c == cout, "deform_conv_tc32: shapes");
  VPS_CHECK_ARG((int64_t)x->n * x->h * x->w * x->cs < (1ll << 31), "deform_conv_tc32: tensor too large for 32-bit offsets");
  VPS_CHECK_ARG(((uintptr_t)w & 127) == 0, "deform_conv_tc32: weights not aligned");
  VPS_CHECK_ARG(y->dtype == VPS_F32, "deform_conv_tc32: y must be fp32");
  vps_conv_args a = dcn_args(*x, cout);
  a.y = *y;
  Tc32Plan g;
  int st = dcn32_plan(&a, g);
  if (st != VPS_OK) return st;
  st = set_problems(g.p, &a, 1, "deform_conv_tc32");
  if (st != VPS_OK) return st;
  if (g.p.total_tiles == 0) return VPS_OK;
  const DcnParams<float> d = {(const float*)x->ptr, (const float*)offset->ptr, x->cs, offset->cs, x->h, x->w};
  CUtensorMap tmB;
  if (!encode_weights_tc32(&tmB, w, 1, cout, 9, x->c, g.p.block_n, "deform_conv_tc32")) return VPS_E_CUDA;
  // a hint only: the driver picks the smallest carve-out that holds the launch's dynamic shared memory (<= DCN32_SMEM_MAX)
  static bool carveout_set = false;
  if (!carveout_set) {
    cudaFuncSetAttribute(dcn_igemm_tc32_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 58);
    (void)cudaGetLastError();
    carveout_set = true;
  }
  return launch_persistent<dcn_igemm_tc32_kernel>(g.p.total_tiles, DCN32_THREADS, g.smem, stream, "deform_conv_tc32", tmB, g.p, g.e,
                                                  d);
}

extern "C" int vps_deform_conv_tc32_plan(const vps_tensor* x, int cout, int* plan) {
  VPS_CHECK_ARG(x->c % T32_KC == 0 && x->c > 0 && cout > 0, "deform_conv_tc32_plan: cin %d, cout %d", x->c, cout);
  const vps_conv_args a = dcn_args(*x, cout);
  Tc32Plan g;
  const int st = dcn32_plan(&a, g);
  if (st != VPS_OK) return st;
  plan[0] = g.e.rows; plan[1] = g.p.block_n / g.e.wg_n; plan[2] = g.e.wg_n == 2; plan[3] = g.p.n_tiles_n;
  return VPS_OK;
}
