// Implicit-GEMM convolution on Hopper tensor cores (wgmma, sm_90a).
//
//   M = 128 output pixels (a th x tw patch of one image), N = block_n output channels (<= 256),
//   K = kh*kw*cin_pad consumed 64 channels (=128 B, one SWIZZLE_128B row) per pipeline stage.
//
//   warp 0      : TMA producer.  The A tile of one (r,s,channel-chunk) K-step is ONE 4-D TMA box
//                 {64 ch, tw, th, 1} of the NHWC activation tensor, shifted by the filter tap; the
//                 tensor map's element strides implement the conv stride and TMA's out-of-bounds zero
//                 fill implements the padding -- im2col is never materialised.  B tile = 2-D box of the
//                 packed weights [cout_pad][K].
//   warpgroups 1, 2: consumers, pixels 0-63 / 64-127 of the tile: wgmma (M=64, N=block_n, K=16) from shared memory into
//                 register accumulators, one batch in flight while the previous one's ring slots are released; then bias +
//                 activation + residual + scale, convert, NHWC store (also into a channel slice of a concat buffer /
//                 interleaved pixels for transposed convs) straight from the accumulator fragments.
//   Persistent: grid = #SMs, static round-robin over tiles; the producer runs ahead into the next tile during the epilogue.
//
// Replaces the cuDNN/cuBLAS calls behind every nn.Conv2d/ConvTranspose2d/Linear of the reference path.
#include "conv_tc_common.cuh"

namespace {

constexpr int NUM_THREADS = 384;     // warpgroup 0: warp 0 = TMA producer (warps 1-3 idle); warpgroups 1, 2: MMA + epilogue
constexpr int TC_BAR_BYTES = 8 * (4 * MAX_STAGES + 8);

// Shared memory of the bf16 kernels from the 1024-byte aligned `base`: A ring, B ring, the DCN's sampling set-up table, the
// barriers.  smem = the launch's dynamic size, with 1 KB of slack for aligning the base.
struct Ring {
  uint32_t a_base, a_stage_bytes, b_base, b_stage_bytes, setup_base, bar_base, smem;
  __device__ __forceinline__ uint32_t afull(int s) const { return bar_base + 8u * s; }
  __device__ __forceinline__ uint32_t aempty(int s) const { return bar_base + 8u * (MAX_STAGES + s); }
  __device__ __forceinline__ uint32_t bfull(int s) const { return bar_base + 8u * (2 * MAX_STAGES + s); }
  __device__ __forceinline__ uint32_t bempty(int s) const { return bar_base + 8u * (3 * MAX_STAGES + s); }
};
// a B slot holds the weights of one tap, of a filter row (halo mode, rowg) or of gsub K steps (flat mode)
__host__ __device__ __forceinline__ Ring tc_ring(uint32_t base, const ConvTcParams& p, bool dcn) {
  Ring rg;
  rg.a_base = base; rg.a_stage_bytes = (uint32_t)p.a_stage_bytes;
  rg.b_base = rg.a_base + (uint32_t)p.a_stages * rg.a_stage_bytes;
  rg.b_stage_bytes = (uint32_t)p.block_n * ((uint32_t)p.bk * 2u) * (p.halo ? (p.rowg ? (uint32_t)p.kw : 1u) : (uint32_t)p.gsub);
  rg.setup_base = rg.b_base + (uint32_t)p.b_stages * rg.b_stage_bytes;
  rg.bar_base = rg.setup_base + (dcn ? (uint32_t)dcn_setup_bytes(BLOCK_M) : 0u);
  rg.smem = rg.bar_base + TC_BAR_BYTES + 1024u - base;
  return rg;
}

// The K walk of a tile, which every role follows: bk channels of one filter tap per K step, chunk-major and tap-minor (a
// chunk's taps in Tap order).  Halo mode: one A item per chunk feeds `rounds` B barrier rounds, of a filter row each (rowg)
// or of one tap.  Flat mode: the tile's `steps` K steps fill ring slots of gsub steps, the last slot possibly fewer.  A step
// of the last chunk has nk_last K16 slabs (bk = 64), the others 4.
struct TcWalk {
  const ConvTcParams& p;
  __host__ __device__ __forceinline__ int chunks() const { return p.cin_chunks; }
  __host__ __device__ __forceinline__ int taps() const { return p.kh * p.kw; }
  __host__ __device__ __forceinline__ int rounds() const { return p.rowg ? p.kh : p.kh * p.kw; }
  __host__ __device__ __forceinline__ int steps() const { return p.cin_chunks * p.kh * p.kw; }
  __host__ __device__ __forceinline__ int slot_steps(int q0) const { return min(p.gsub, steps() - q0); }
  __device__ __forceinline__ int chunk_nk(int cc) const { return cc == p.cin_chunks - 1 ? p.nk_last : 4; }
  __device__ __forceinline__ int step_nk(int q) const { return q >= steps() - taps() ? p.nk_last : 4; }
};
__host__ __device__ __forceinline__ TcWalk tc_walk(const ConvTcParams& p) { return {p}; }

// ---------------------------------------------------------------- TMA producer (warp 0)
// The loop runs warp-uniformly and picks the issuing lane with elect.sync: code under `if (lane == 0)` is divergent to the
// compiler, which then wraps every TMA instruction in a uniformity loop.  In halo mode one barrier round covers a whole
// filter row (kw taps) when the row's weights fit one ring slot.

// ---- halo mode: one activation box per channel chunk (A ring), weights per tap or per filter row (B ring)
template <bool ROWG>
__device__ __forceinline__ void producer_halo(const ConvTcParams& p, const Ring& rg, const CUtensorMap* tmA,
                                              const CUtensorMap* tmB0, const CUtensorMap* tmB1, const CUtensorMap* tmB2,
                                              const CUtensorMap* tmB3) {
  const int bk = p.bk, kw = p.kw, a_stages = p.a_stages, b_stages = p.b_stages;
  const TcWalk walk = tc_walk(p);
  const uint32_t a_box_bytes = (uint32_t)p.a_box_bytes;
  RingPos ap, bp;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const TileCoord t = tile_coord(p, tile);
    const int x_base = t.tx * p.tw - p.pw_[t.prob];
    const int y_base = t.ty * p.th - p.ph_[t.prob];
    const int n0 = t.n_idx * p.block_n;
    const CUtensorMap* tmB = t.prob == 0 ? tmB0 : (t.prob == 1 ? tmB1 : (t.prob == 2 ? tmB2 : tmB3));
    for (int cc = 0; cc < walk.chunks(); ++cc) {
      ap.wait_empty(rg.aempty(ap.slot));
      if (elect_one()) {
        mbar_expect_tx(rg.afull(ap.slot), a_box_bytes);
        tma_load_4d(rg.a_base + ap.slot * rg.a_stage_bytes, tmA, rg.afull(ap.slot), cc * bk, x_base, y_base, t.img);
      }
      ap.next(a_stages);
      for (int g = 0; g < walk.rounds(); ++g) {
        bp.wait_empty(rg.bempty(bp.slot));
        if (elect_one()) {
          mbar_expect_tx(rg.bfull(bp.slot), rg.b_stage_bytes);
          tma_load_3d(rg.b_base + bp.slot * rg.b_stage_bytes, tmB, rg.bfull(bp.slot), cc * bk, n0, ROWG ? g * kw : g);
        }
        bp.next(b_stages);
      }
    }
  }
}

// ---- flat mode (strided / 1x1 convolutions): K steps in (chunk, tap) order, gsub steps share one ring slot and one
// barrier round (both operands arrive on the slot's `afull` barrier; the B barriers are unused)
__device__ __forceinline__ void producer_flat(const ConvTcParams& p, const Ring& rg, const CUtensorMap* tmA,
                                              const CUtensorMap* tmB0, const CUtensorMap* tmB1, const CUtensorMap* tmB2,
                                              const CUtensorMap* tmB3) {
  const int bk = p.bk, stages = p.a_stages;
  const TcWalk walk = tc_walk(p);
  const uint32_t a_box_bytes = (uint32_t)p.a_box_bytes;
  const uint32_t b_tile_bytes = (uint32_t)p.block_n * (uint32_t)bk * 2u;
  RingPos sp;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const TileCoord t = tile_coord(p, tile);
    const int x_base = t.tx * p.tw * p.sw - p.pw_[t.prob];
    const int y_base = t.ty * p.th * p.sh - p.ph_[t.prob];
    const int n0 = t.n_idx * p.block_n;
    const CUtensorMap* tmB = t.prob == 0 ? tmB0 : (t.prob == 1 ? tmB1 : (t.prob == 2 ? tmB2 : tmB3));
    int cc = 0;
    Tap tap;
    for (int q0 = 0; q0 < walk.steps(); q0 += p.gsub) {
      const int cnt = walk.slot_steps(q0);
      sp.wait_empty(rg.aempty(sp.slot));
      const uint32_t a_slot = rg.a_base + sp.slot * rg.a_stage_bytes, b_slot = rg.b_base + sp.slot * rg.b_stage_bytes;
      if (elect_one()) mbar_expect_tx(rg.afull(sp.slot), (uint32_t)cnt * (a_box_bytes + b_tile_bytes));
      __syncwarp();
      for (int j = 0; j < cnt; ++j) {
        if (elect_one()) {
          tma_load_4d(a_slot + j * a_box_bytes, tmA, rg.afull(sp.slot), cc * bk, x_base + tap.s, y_base + tap.r, t.img);
          tma_load_3d(b_slot + j * b_tile_bytes, tmB, rg.afull(sp.slot), cc * bk, n0, tap.k);
        }
        tap.next(p.kw);
        if (tap.r == p.kh) { tap = Tap(); ++cc; }
      }
      sp.next(stages);
    }
  }
}

// ---------------------------------------------------------------- consumer warpgroups (MMA + epilogue)
// the (up to) four K16 MMAs of one tap: 64 channels = one SWIZZLE_128B row; +2 in the (addr >> 4) field = 32 bytes
template <int N, bool BK64>
__device__ __forceinline__ void issue_tap(float (&d)[N / 2], uint64_t a_hi, uint64_t b_hi, uint32_t a_addr, uint32_t b_addr, int nk,
                                          uint32_t& accumulate) {
  const uint64_t adesc = desc_at(a_hi, a_addr), bdesc = desc_at(b_hi, b_addr);
  wg::Mma<N, false>::run(d, adesc, bdesc, accumulate);
  if (BK64) {
    if (nk > 1) wg::Mma<N, false>::run(d, adesc + 2, bdesc + 2, 1u);
    if (nk > 2) wg::Mma<N, false>::run(d, adesc + 4, bdesc + 4, 1u);
    if (nk > 3) wg::Mma<N, false>::run(d, adesc + 6, bdesc + 6, 1u);
  }
  accumulate = 1u;
}

// Ring slots are released one batch late: after batch i is committed, wgmma.wait_group 1 guarantees batch i - 1 has read
// its operands, so its slots go back to the producer while batch i runs.  One elected thread per warpgroup arrives (the
// empty barriers count both consumer warpgroups).
struct Release {
  int b = -1, a = -1;
  __device__ __forceinline__ void flush(const Ring& rg, bool leader) {
    if (leader) {
      if (b >= 0) mbar_arrive(rg.bempty(b));
      if (a >= 0) mbar_arrive(rg.aempty(a));
    }
    b = a = -1;
  }
};

template <int N, bool BK64>
__device__ __forceinline__ void consumer_tc(const ConvTcParams& p, const Ring& rg, int wg) {
  constexpr uint32_t row_bytes = BK64 ? 128u : 32u;
  const bool leader = (threadIdx.x & 127) == 0;
  const int kw = p.kw;
  const TcWalk walk = tc_walk(p);
  const uint32_t tap_b_bytes = (uint32_t)N * row_bytes;
  const uint64_t b_hi = desc_hi(row_bytes, 8u * row_bytes);
  float d[N / 2];
  RingPos ap, bp;
  Release rel;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    uint32_t accumulate = 0;
    if (p.halo) {
      // the 8 rows of an MMA row group are 8 pixels of one halo row; this warpgroup's 64 pixels start 8 halo rows down
      const uint32_t halo_pitch = (uint32_t)p.halo_w * row_bytes;
      const uint64_t a_hi = desc_hi(row_bytes, halo_pitch);
      for (int cc = 0; cc < walk.chunks(); ++cc) {
        const int nk = walk.chunk_nk(cc);
        ap.wait_full(rg.afull(ap.slot));
        uint32_t a_row = rg.a_base + ap.slot * rg.a_stage_bytes + (uint32_t)wg * 8u * halo_pitch, a_tap = a_row;
        const int a_cur = ap.slot;
        int sx = 0;
        ap.next(p.a_stages);
        for (int g = 0; g < walk.rounds(); ++g) {
          bp.wait_full(rg.bfull(bp.slot));
          const uint32_t b_addr = rg.b_base + bp.slot * rg.b_stage_bytes;
          wg::fence();
          if (p.rowg) {      // the kw taps of filter row g: A start moves one pixel (row_bytes) per tap
            for (int j = 0; j < kw; ++j) issue_tap<N, BK64>(d, a_hi, b_hi, a_row + j * row_bytes, b_addr + j * tap_b_bytes, nk, accumulate);
          } else {
            issue_tap<N, BK64>(d, a_hi, b_hi, a_tap, b_addr, nk, accumulate);
          }
          wg::commit();
          wg::wait<1>();
          rel.flush(rg, leader);
          rel.b = bp.slot;
          if (g == walk.rounds() - 1) rel.a = a_cur;
          bp.next(p.b_stages);
          if (p.rowg) {
            a_row += halo_pitch;
          } else {          // next tap: one pixel to the right, or the start of the next halo row
            a_tap += row_bytes;
            if (++sx == kw) { sx = 0; a_row += halo_pitch; a_tap = a_row; }
          }
        }
      }
    } else {
      // flat mode: gsub K steps per ring slot, operands of both kinds on the slot's `afull` barrier
      const uint32_t a_box_bytes = (uint32_t)p.a_box_bytes;
      const uint64_t a_hi = desc_hi(row_bytes, 8u * row_bytes);
      for (int q0 = 0; q0 < walk.steps(); q0 += p.gsub) {
        const int cnt = walk.slot_steps(q0);
        ap.wait_full(rg.afull(ap.slot));
        const uint32_t a_slot = rg.a_base + ap.slot * rg.a_stage_bytes + (uint32_t)wg * 64u * row_bytes;
        const uint32_t b_slot = rg.b_base + ap.slot * rg.b_stage_bytes;
        wg::fence();
        for (int j = 0; j < cnt; ++j)
          issue_tap<N, BK64>(d, a_hi, b_hi, a_slot + j * a_box_bytes, b_slot + j * tap_b_bytes, walk.step_nk(q0 + j), accumulate);
        wg::commit();
        wg::wait<1>();
        rel.flush(rg, leader);
        rel.a = ap.slot;
        ap.next(p.a_stages);
      }
    }
    wg::wait<0>();
    wg::fence_regs(d);
    rel.flush(rg, leader);
    epi_frag<N, 2>(p, d, tile, wg * 64);
  }
}

template <bool BK64>
__device__ __forceinline__ void consumer_tc_n(const ConvTcParams& p, const Ring& rg, int wg) {
  switch (p.block_n) {
    case 16: consumer_tc<16, BK64>(p, rg, wg); break;
    case 32: consumer_tc<32, BK64>(p, rg, wg); break;
    case 64: consumer_tc<64, BK64>(p, rg, wg); break;
    case 128: consumer_tc<128, BK64>(p, rg, wg); break;
    default: consumer_tc<256, BK64>(p, rg, wg); break;
  }
}

// ---------------------------------------------------------------- kernel
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_igemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB0,
                     const __grid_constant__ CUtensorMap tmB1, const __grid_constant__ CUtensorMap tmB2,
                     const __grid_constant__ CUtensorMap tmB3, const ConvTcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte aligned operand ring (SWIZZLE_128B requirement)
  const Ring rg = tc_ring((smem_u32(smem_raw) + 1023u) & ~1023u, p, false);
  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0);     // warp-uniform role index (wgmma issue is not treated as divergent)
  const int lane = threadIdx.x & 31;

  // full = one TMA arrival, empty = one arrival per consumer warpgroup
  if (warp == 0) {
    if (lane < MAX_STAGES) { mbar_init(rg.afull(lane), 1); mbar_init(rg.aempty(lane), 2); }
    else if (lane < 2 * MAX_STAGES) { mbar_init(rg.bfull(lane - MAX_STAGES), 1); mbar_init(rg.bempty(lane - MAX_STAGES), 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x == 32) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB0) : "memory");
  }
  __syncthreads();
  // Programmatic dependent launch: the prologue above overlaps the tail of the previous kernel in the stream; no global
  // memory is touched before the wait.  Our own dependents are released immediately -- they block at their own wait until
  // this grid has completed and flushed.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (warp == 0) {
    if (!p.halo) producer_flat(p, rg, &tmA, &tmB0, &tmB1, &tmB2, &tmB3);
    else if (p.rowg) producer_halo<true>(p, rg, &tmA, &tmB0, &tmB1, &tmB2, &tmB3);
    else producer_halo<false>(p, rg, &tmA, &tmB0, &tmB1, &tmB2, &tmB3);
  } else if (warp >= 4) {
    if (p.bk == 64) consumer_tc_n<true>(p, rg, (warp - 4) >> 2);
    else consumer_tc_n<false>(p, rg, (warp - 4) >> 2);
  }
}


// ---------------------------------------------------------------- fused deformable convolution (DCNv1, 3x3, pad 1)
// Same implicit GEMM, but the A tile of a K step is not a TMA box: eight producer warps bilinearly sample the input
// at the learned offsets (deform_conv_cuda_kernel.cu: deformable_im2col) straight into the SWIZZLE_128B operand slot,
// so the 9x column matrix is never written to HBM.  K steps run chunk-major / tap-minor: for one 64-channel chunk the
// nine taps of a tile touch the same ~(th+2) x (tw+2) x 128 B of input, which stays in L1.  Per tile the sampling
// set-up of every (pixel, tap) -- 4 corner element offsets + 4 weights -- is computed once into shared memory.
// 512 threads: warp 0 = weight TMA, warps 1-3 and 12-15 = sampling, warpgroups 1 and 2 = MMA + epilogue.  At 128 registers
// per thread a consumer holds at most an N = 128 accumulator, so wider layers run as several N tiles.
constexpr int DCN_GATHER_WARPS = 7;
constexpr int DCN_THREADS = 512;
constexpr int DCN_MAX_N = 128;

__device__ __forceinline__ void dcn_gather_loop(const ConvTcParams& p, const DcnParams<__nv_bfloat16>& d, const Ring& rg,
                                                uint32_t setup_base, int gtid) {
  const int stages = p.a_stages;
  const TcWalk walk = tc_walk(p);
  RingPos sp;
  const int j = gtid & 7;                    // 16-byte channel chunk of the 128-byte row
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const TileCoord tc = tile_coord(p, tile);
    const int img = tc.img, ty = tc.ty, tx = tc.tx;
    // ---- sampling set-up of all (tap, pixel) pairs of this tile
    for (int item = gtid; item < 9 * BLOCK_M; item += 32 * DCN_GATHER_WARPS) {
      const int k = item >> 7, r = item & (BLOCK_M - 1);
      const int ty_in = r / p.tw, tx_in = r - ty_in * p.tw;
      dcn_setup_entry(d, setup_base + (uint32_t)item * 32u, img, ty * p.th + ty_in, tx * p.tw + tx_in, k);
    }
    asm volatile("bar.sync 1, %0;" ::"n"(32 * DCN_GATHER_WARPS) : "memory");
    // ---- K steps: chunk-major, tap-minor
    for (int cc = 0; cc < walk.chunks(); ++cc) {
      const __nv_bfloat16* xc = d.x + cc * 64 + j * 8;
      for (int k = 0; k < walk.taps(); ++k) {
        sp.wait_empty(rg.aempty(sp.slot));
        const uint32_t a_slot = rg.a_base + sp.slot * rg.a_stage_bytes;
        constexpr int ROWS_PER_PASS = 32 * DCN_GATHER_WARPS / 8;       // 8 lanes (16-byte chunks) per pixel row
        for (int r = gtid >> 3; r < BLOCK_M; r += ROWS_PER_PASS) {
          const uint32_t sa = setup_base + (uint32_t)(k * BLOCK_M + r) * 32u;
          float w0, w1, w2, w3;
          int o0, o1, o2, o3;
          asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(w0), "=f"(w1), "=f"(w2), "=f"(w3) : "r"(sa));
          asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(o0), "=r"(o1), "=r"(o2), "=r"(o3) : "r"(sa + 16u));
          const uint4 q0 = __ldg(reinterpret_cast<const uint4*>(xc + o0));
          const uint4 q1 = __ldg(reinterpret_cast<const uint4*>(xc + o1));
          const uint4 q2 = __ldg(reinterpret_cast<const uint4*>(xc + o2));
          const uint4 q3 = __ldg(reinterpret_cast<const uint4*>(xc + o3));
          const float wq[4] = {w0, w1, w2, w3};
          const uint4 qs[4] = {q0, q1, q2, q3};
          float acc[8];
#pragma unroll
          for (int t = 0; t < 8; ++t) acc[t] = 0.f;
#pragma unroll
          for (int q = 0; q < 4; ++q) {           // corners outside the image carry weight 0 (branch-free: finite inputs)
            const __nv_bfloat162* b2 = reinterpret_cast<const __nv_bfloat162*>(&qs[q]);
#pragma unroll
            for (int t = 0; t < 4; ++t) {
              const float2 f = __bfloat1622float2(b2[t]);
              acc[2 * t] += wq[q] * f.x;
              acc[2 * t + 1] += wq[q] * f.y;
            }
          }
          uint32_t pk[4];
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            __nv_bfloat162 b = __floats2bfloat162_rn(acc[2 * t], acc[2 * t + 1]);
            pk[t] = *reinterpret_cast<uint32_t*>(&b);
          }
          const uint32_t da = a_slot + (uint32_t)r * 128u + (uint32_t)((j ^ (r & 7)) << 4);
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(da), "r"(pk[0]), "r"(pk[1]), "r"(pk[2]), "r"(pk[3]) : "memory");
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy writes -> tensor-core reads
        mbar_arrive(rg.afull(sp.slot));
        sp.next(stages);
      }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(32 * DCN_GATHER_WARPS) : "memory");   // set-up cache is rewritten next tile
  }
}

__global__ void __launch_bounds__(DCN_THREADS, 1)
dcn_igemm_tc_kernel(const __grid_constant__ CUtensorMap tmB, const ConvTcParams p, const DcnParams<__nv_bfloat16> d) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const Ring rg = tc_ring((smem_u32(smem_raw) + 1023u) & ~1023u, p, true);
  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0);     // warp-uniform role index (wgmma issue is not treated as divergent)
  if (threadIdx.x == 0) {
    for (int s = 0; s < MAX_STAGES; ++s) {
      mbar_init(rg.afull(s), 1 + 32 * DCN_GATHER_WARPS);     // weight TMA (expect_tx arrival) + every gather thread
      mbar_init(rg.aempty(s), 2);                            // one arrival per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
  }
  __syncthreads();
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (warp >= 4 && warp < 12) {
    if (p.block_n <= 64) consumer_tc<64, true>(p, rg, (warp - 4) >> 2);
    else consumer_tc<DCN_MAX_N, true>(p, rg, (warp - 4) >> 2);
  } else {
    if (warp == 0) {
      // weight producer: one {64 ch, block_n, 1 tap} box per K step, completing on the step's `afull` barrier
      const TcWalk walk = tc_walk(p);
      RingPos sp;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int n0 = tile_coord(p, tile).n_idx * p.block_n;
        for (int cc = 0; cc < walk.chunks(); ++cc) {
          for (int k = 0; k < walk.taps(); ++k) {
            sp.wait_empty(rg.aempty(sp.slot));
            if (elect_one()) {
              mbar_expect_tx(rg.afull(sp.slot), rg.b_stage_bytes);
              tma_load_3d(rg.b_base + sp.slot * rg.b_stage_bytes, &tmB, rg.afull(sp.slot), cc * 64, n0, k);
            }
            sp.next(p.a_stages);
          }
        }
      }
    } else {
      dcn_gather_loop(p, d, rg, rg.setup_base, warp < 4 ? (int)threadIdx.x - 32 : (int)threadIdx.x - 384 + 96);
    }
  }
}

// ---------------------------------------------------------------- weight packing
// dst[co][ (r*kw+s)*cin_pad + ci ] (bf16), zero padded; src OIHW (or IOHW when transposed)
__global__ void pack_weights_tc_kernel(const float* __restrict__ src, const float* __restrict__ scale,
                                       __nv_bfloat16* __restrict__ dst, int cout, int cin, int kh, int kw,
                                       int cout_pad, int cin_pad, int transposed) {
  const int64_t total = (int64_t)cout_pad * kh * kw * cin_pad;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = __float2bfloat16_rn(packed_weight(src, scale, i, cout, cin, kh, kw, cin_pad, transposed));
}

// Packed weights [cout_pad][taps][cin_pad] viewed as {cin_pad, cout_pad, taps}: a box is {bk, block_n, box_taps}, i.e.
// consecutive K-major [block_n][bk] tiles, one per tap.  `who` prefixes the error message.
bool encode_weights_tc(CUtensorMap* m, const void* w, int cout, int taps, int cin_pad, int bk, int block_n, int box_taps,
                       const char* who) {
  const auto encode = vps::tensor_map_encoder();
  if (!encode) return false;
  cuuint64_t dims[3] = {(cuuint64_t)cin_pad, (cuuint64_t)((cout + 15) / 16 * 16), (cuuint64_t)taps};
  cuuint64_t strides[2] = {(cuuint64_t)taps * cin_pad * 2, (cuuint64_t)cin_pad * 2};
  cuuint32_t box[3] = {(cuuint32_t)bk, (cuuint32_t)block_n, (cuuint32_t)box_taps};
  cuuint32_t estr[3] = {1, 1, 1};
  const CUresult r = encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, (void*)w, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { vps::set_error("%s: encode B failed (%d)", who, (int)r); return false; }
  return true;
}

}  // namespace

static inline int cin_pad_for(int cin, int gran) { return (cin + gran - 1) / gran * gran; }

extern "C" int64_t vps_packed_tc_bytes(int cout, int cin, int kh, int kw, int cin_gran) {
  const int64_t cout_pad = (cout + 15) / 16 * 16, cin_pad = cin_pad_for(cin, cin_gran == 16 ? 16 : 64);
  return cout_pad * kh * kw * cin_pad * 2;
}

extern "C" int vps_pack_weights_tc(const float* w, const float* scale, void* dst, int cout, int cin, int kh, int kw,
                                   int transposed, int cin_gran, void* stream) {
  const int cout_pad = (cout + 15) / 16 * 16, cin_pad = cin_pad_for(cin, cin_gran == 16 ? 16 : 64);
  const int64_t total = (int64_t)cout_pad * kh * kw * cin_pad;
  const int blocks = (int)((total + 255) / 256 > 4096 ? 4096 : (total + 255) / 256);
  pack_weights_tc_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, scale, (__nv_bfloat16*)dst, cout, cin, kh,
                                                                  kw, cout_pad, cin_pad, transposed);
  VPS_CUDA_LAST("pack_weights_tc");
  return VPS_OK;
}

// The tiling and rings of vps_conv2d_tc_multi(a, nprob), from the shapes in `a` and the current device's SM count (no pointer
// is read); set_problems() adds the output, residual and epilogue.
static int tc_plan(const vps_conv_args* a, int nprob, ConvTcParams& p) {
  VPS_CHECK_ARG(nprob >= 1 && nprob <= MAX_PROB, "conv2d_tc: nprob %d", nprob);
  VPS_CHECK_ARG(a->sh >= 1 && a->sh <= 2 && a->sw >= 1 && a->sw <= 2, "conv2d_tc: stride must be 1 or 2");
  const int sms = vps::num_sms();
  if (sms <= 0) { vps::set_error("no device"); return VPS_E_NODEV; }

  p = {};
  const int bk = a->cin_gran == 16 ? 16 : 64;
  p.bk = bk;
  const int cin_pad = cin_pad_for(a->cin, bk);
  const int cout_pad = (a->cout + 15) / 16 * 16;
  // halo mode (stride 1, more than one tap): the 8 rows of an MMA row group are 8 consecutive pixels of one halo row,
  // so the tile is 16 x 8 pixels and every tap reads the same (16+kh-1) x (8+kw-1) box at a shifted start address.
  const bool halo = a->sh == 1 && a->sw == 1 && a->kh * a->kw > 1 && a->kh <= 8 && a->kw <= 8;
  p.halo = halo ? 1 : 0;
  const int tw = halo ? 8 : patch_tw(a->oh, a->ow, BLOCK_M, a->sh, a->sw), th = BLOCK_M / tw;
  p.halo_w = tw + a->kw - 1;
  const int halo_h = th + a->kh - 1;
  p.a_box_bytes = halo ? halo_h * p.halo_w * bk * 2 : BLOCK_M * bk * 2;
  p.a_stage_bytes = (p.a_box_bytes + 1023) / 1024 * 1024;
  // N tile: pick the divisor of cout_pad (multiple of 16, <= 256) that minimises a simple time model
  //   waves(bn) * k_steps * max(fixed per-step latency, MMA time 2*bn clk, stage bytes / per-SM L2 bandwidth)
  // -- large tiles when there is enough parallelism, smaller N tiles to fill the persistent grid otherwise.
  int block_n = 16;
  {
    const int64_t m_tiles = (int64_t)a->x.n * vps::cdiv(a->oh, th) * vps::cdiv(a->ow, tw) * nprob;
    double best = -1.0;
    for (int bn = 16; bn <= 256 && bn <= cout_pad; bn *= 2) {     // the N extents the consumer is instantiated for
      if (cout_pad % bn) continue;
      const int64_t tiles = m_tiles * (cout_pad / bn);
      const double waves = (double)((tiles + sms - 1) / sms);
      const double epi = 40.0 * bn;     // epilogue clocks per tile (not hidden when a CTA runs a single tile)
      double t;
      if (halo) {   // per tap: MMA time / operand reads from smem / weight box; per chunk: one halo box
        const double step = fmax(fmax(215.0, 2.0 * bn), (double)(bn * bk * 2) / 40.0);
        t = waves * ((double)(cin_pad / bk) * ((double)(a->kh * a->kw) * step + (double)p.a_box_bytes / 20.0) + epi);
      } else {
        const double step = fmax(fmax(350.0, 2.0 * bn), (double)((BLOCK_M + bn) * bk * 2) / 80.0);
        t = waves * ((double)(a->kh * a->kw * (cin_pad / bk)) * step + epi);
      }
      if (best < 0 || t < best * 0.999) { best = t; block_n = bn; }
    }
  }
  set_tiles(p, a, nprob, tw, th, block_n, bk);
  // halo mode: one B ring slot = the kw taps of a filter row when that fits (<= 48 KB) -- one barrier round per row
  p.rowg = (halo && a->kw > 1 && a->kw * block_n * bk * 2 <= 48 * 1024) ? 1 : 0;
  // flat mode: gsub consecutive K steps share a ring slot (<= 48 KB of operands per barrier round, at most 4 steps)
  p.gsub = 1;
  if (!halo) {
    const int step_bytes = p.a_box_bytes + block_n * bk * 2;
    int g = (48 * 1024) / step_bytes;
    const int steps = tc_walk(p).steps();
    if (g > 4) g = 4;
    if (g > steps) g = steps;
    if (g < 1) g = 1;
    p.gsub = g;
    p.a_stage_bytes = g * p.a_box_bytes;
  }
  const int b_stage_bytes = (int)tc_ring(0, p, false).b_stage_bytes;
  if (halo) {
    p.a_stages = p.cin_chunks >= 3 ? 3 : 2;
    int bst = (200 * 1024 - p.a_stages * p.a_stage_bytes) / b_stage_bytes;
    p.b_stages = bst > MAX_STAGES ? MAX_STAGES : bst;
    VPS_CHECK_ARG(p.b_stages >= 2, "conv2d_tc: halo ring does not fit");
  } else {
    int stages = (200 * 1024) / (p.a_stage_bytes + b_stage_bytes);
    if (stages > MAX_STAGES) stages = MAX_STAGES;
    p.a_stages = p.b_stages = stages;
  }
  return VPS_OK;
}

// nprob problems (<= 4) that share x / y / geometry / epilogue and differ in weights, padding and output pixel
// offset: the four stride phases of a transposed convolution run as ONE persistent launch.
extern "C" int vps_conv2d_tc_multi(const vps_conv_args* args, int nprob, void* stream) {
  VPS_CHECK_ARG(nprob >= 1 && nprob <= MAX_PROB, "conv2d_tc: nprob %d", nprob);
  const vps_conv_args* a = &args[0];
  VPS_CHECK_ARG(a->x.dtype == VPS_BF16, "conv2d_tc: x must be bf16");
  VPS_CHECK_ARG(a->x.cs % 8 == 0 && ((uintptr_t)a->x.ptr & 15) == 0, "conv2d_tc: x not 16B aligned (cs=%d)",
                a->x.cs);
  VPS_CHECK_ARG(a->cin == a->x.c, "conv2d_tc: cin %d != x.c %d", a->cin, a->x.c);
  for (int i = 0; i < nprob; ++i) {
    VPS_CHECK_ARG(((uintptr_t)args[i].w & 15) == 0, "conv2d_tc: weights not aligned");
    VPS_CHECK_ARG(args[i].x.ptr == a->x.ptr && args[i].y.ptr == a->y.ptr && args[i].kh == a->kh && args[i].kw == a->kw &&
                      args[i].oh == a->oh && args[i].ow == a->ow && args[i].cout == a->cout && args[i].bias == a->bias &&
                      args[i].act == a->act && args[i].oy_mul == a->oy_mul && args[i].ox_mul == a->ox_mul &&
                      args[i].cin_gran == a->cin_gran,
                  "conv2d_tc_multi: problems must share geometry");
  }
  ConvTcParams p;
  int st = tc_plan(a, nprob, p);
  if (st != VPS_OK) return st;
  st = set_problems(p, args, nprob, "conv2d_tc");
  if (st != VPS_OK) return st;
  if (p.total_tiles == 0) return VPS_OK;

  const int bk = p.bk, halo_h = p.th + a->kh - 1;
  CUtensorMap tmA, tmB[MAX_PROB];
  if (!vps::encode_nhwc(&tmA, a->x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, bk, p.halo ? p.halo_w : p.tw * a->sw, p.halo ? halo_h : p.th * a->sh,
                        a->sw, a->sh, bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_32B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "conv2d_tc: encode A"))
    return VPS_E_CUDA;
  for (int i = 0; i < MAX_PROB; ++i)
    if (!encode_weights_tc(&tmB[i], args[i < nprob ? i : 0].w, a->cout, a->kh * a->kw, cin_pad_for(a->cin, bk), bk, p.block_n,
                           p.rowg ? a->kw : 1, "conv2d_tc"))
      return VPS_E_CUDA;
  return launch_persistent<conv_igemm_tc_kernel>(p.total_tiles, NUM_THREADS, (int)tc_ring(0, p, false).smem, stream, "conv2d_tc",
                                                 tmA, tmB[0], tmB[1], tmB[2], tmB[3], p);
}

extern "C" int vps_conv2d_tc(const vps_conv_args* a, void* stream) { return vps_conv2d_tc_multi(a, 1, stream); }

extern "C" int vps_conv2d_tc_plan(const vps_conv_args* a, int nprob, int* plan) {
  ConvTcParams p;
  const int st = tc_plan(a, nprob, p);
  if (st != VPS_OK) return st;
  const int v[10] = {p.block_n, p.tw, p.th, p.halo, p.rowg, p.gsub, p.bk, p.a_stages, p.b_stages, p.total_tiles};
  for (int i = 0; i < 10; ++i) plan[i] = v[i];
  return VPS_OK;
}


// Fused DCNv1 3x3 / stride 1 / pad 1 / dilation 1 / 1 deformable group (deform_conv.py:15-87 forward):
// x bf16 NHWC, offset f32 NHWC [.., 18] = (dy, dx) per tap, w = vps_pack_weights_tc layout of the [cout, cin, 3, 3]
// kernel (cin % 64 == 0, cout <= 256), y bf16 / f32 NHWC.  No bias (the reference's DeformConv has none).
extern "C" int vps_deform_conv_tc(const vps_tensor* x, const vps_tensor* offset, const void* w, int cout, const vps_tensor* y,
                                  void* stream) {
  VPS_CHECK_ARG(x->dtype == VPS_BF16 && offset->dtype == VPS_F32 && offset->c >= 18, "deform_conv_tc: dtypes");
  VPS_CHECK_ARG(x->c % 64 == 0 && x->cs % 8 == 0 && ((uintptr_t)x->ptr & 15) == 0, "deform_conv_tc: x must have cin %% 64 == 0");
  VPS_CHECK_ARG(offset->n == x->n && offset->h == x->h && offset->w == x->w && y->n == x->n && y->h == x->h && y->w == x->w &&
                    y->c == cout, "deform_conv_tc: shapes");
  VPS_CHECK_ARG((int64_t)x->n * x->h * x->w * x->cs < (1ll << 31), "deform_conv_tc: tensor too large for 32-bit offsets");
  const int cout_pad = (cout + 15) / 16 * 16;
  VPS_CHECK_ARG(cout_pad <= 256 && ((uintptr_t)w & 15) == 0, "deform_conv_tc: cout %d > 256", cout);
  if (vps::num_sms() <= 0) { vps::set_error("no device"); return VPS_E_NODEV; }
  vps_conv_args a = dcn_args(*x, cout);
  a.y = *y;
  ConvTcParams p = {};
  p.bk = 64;
  // weight rows past cout_pad are TMA zero fill
  const int tw = patch_tw(x->h, x->w, BLOCK_M, 1, 1);
  set_tiles(p, &a, 1, tw, BLOCK_M / tw, cout_pad <= 64 ? 64 : DCN_MAX_N, 64);
  p.gsub = 1;
  p.a_box_bytes = BLOCK_M * 128; p.a_stage_bytes = p.a_box_bytes;
  int stages = (200 * 1024 - dcn_setup_bytes(BLOCK_M)) / (p.a_stage_bytes + (int)tc_ring(0, p, true).b_stage_bytes);
  if (stages > MAX_STAGES) stages = MAX_STAGES;
  VPS_CHECK_ARG(stages >= 2, "deform_conv_tc: ring does not fit");
  p.a_stages = p.b_stages = stages;
  const int st = set_problems(p, &a, 1, "deform_conv_tc");
  if (st != VPS_OK) return st;
  if (p.total_tiles == 0) return VPS_OK;
  const DcnParams<__nv_bfloat16> d = {(const __nv_bfloat16*)x->ptr, (const float*)offset->ptr, x->cs, offset->cs, x->h, x->w};
  CUtensorMap tmB;
  if (!encode_weights_tc(&tmB, w, cout, 9, x->c, 64, p.block_n, 1, "deform_conv_tc")) return VPS_E_CUDA;
  return launch_persistent<dcn_igemm_tc_kernel>(p.total_tiles, DCN_THREADS, (int)tc_ring(0, p, true).smem, stream, "deform_conv_tc",
                                                tmB, p, d);
}
