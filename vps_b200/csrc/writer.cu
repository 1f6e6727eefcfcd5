// Segment table of one sampled frame for the video writer (reference tools/dataset/cityscapes_vps.py:96-140,
// converter_2ch_track_core): the per-key pixel counts and bounding boxes the converter takes from np.unique / np.where over
// pan = 1000 * semantic + track, and the pan_pred PNG (id2rgb of the segment id), in one pass over the unified result.
// The image converter (tools/dataset/base_dataset.py:287-335, _converter_2ch_single_core) does the same over
// pan = 1000 * semantic + instance rank: KEY_CH selects the key channel, 2 (track) or 1 (instance), as in vpq.cu.
//
// Keys are (semantic < 19, key-channel byte): at most 19 * 256 of them, so a block keeps the whole table in shared memory
// (5 planes x 4864 words = 95 KiB).  Each thread walks strips of 16 pixels inside one row and issues one set of shared
// atomics per run of equal keys; a block then adds each key it touched into the global table with one atomic per plane.
#include "common.cuh"

namespace {
constexpr int SEG_RUN = 16;
constexpr uint32_t NKEY = VPS_SEG_NKEY;

__device__ __forceinline__ uint32_t seg_id(uint32_t sem, uint32_t trk, uint32_t num_stuff) {
  return sem == 255u ? 0u : 1000u * sem + (sem < num_stuff ? 0u : trk) + 1u;
}

__global__ void seg_table_init_kernel(uint32_t* __restrict__ table) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < VPS_SEG_TABLE_WORDS; i += gridDim.x * blockDim.x)
    table[i] = (i >= VPS_SEG_X0 * NKEY && i < VPS_SEG_X1 * NKEY) ? 0xFFFFFFFFu : 0u;
}

// vec: W % 16 == 0 and both images 16-byte aligned, so every strip is three aligned uint4 of input and of output
template <int KEY_CH>
__global__ void __launch_bounds__(256) pan2ch_segments_kernel(const uint8_t* __restrict__ p2, int H, int W, uint32_t num_stuff,
                                                              uint32_t* __restrict__ table, uint8_t* __restrict__ rgb, bool vec) {
  extern __shared__ uint32_t s[];                                  // planes area, x0, y0, x1, y1 of NKEY words
  __shared__ uint32_t s_bad;
  for (uint32_t i = threadIdx.x; i < VPS_SEG_PLANES * NKEY; i += blockDim.x)
    s[i] = (i >= VPS_SEG_X0 * NKEY && i < VPS_SEG_X1 * NKEY) ? 0xFFFFFFFFu : 0u;
  if (threadIdx.x == 0) s_bad = 0;
  __syncthreads();

  const int nsx = (W + SEG_RUN - 1) / SEG_RUN;
  const int64_t nstrip = (int64_t)H * nsx;
  VPS_GRID_STRIDE(r, nstrip) {
    const int y = (int)(r / nsx), x0 = (int)(r % nsx) * SEG_RUN;
    const int cnt = min(SEG_RUN, W - x0);
    const int64_t base = ((int64_t)y * W + x0) * 3;
    alignas(16) uint8_t px[3 * SEG_RUN];          // read / written as three uint4 on the vector path
    if (vec) {
      const uint4* src = reinterpret_cast<const uint4*>(p2 + base);
#pragma unroll
      for (int q = 0; q < 3; ++q) reinterpret_cast<uint4*>(px)[q] = src[q];
    } else {
#pragma unroll
      for (int e = 0; e < 3 * SEG_RUN; ++e) px[e] = e < 3 * cnt ? p2[base + e] : 0;
    }
    alignas(16) uint8_t out[3 * SEG_RUN];
    int cur = -1, xs = x0;
    unsigned n = 0;
    auto flush = [&](int key, int xa, int xb, unsigned m) {
      if (key >= 0) {
        atomicAdd(&s[VPS_SEG_AREA * NKEY + key], m);
        atomicMin(&s[VPS_SEG_X0 * NKEY + key], (uint32_t)xa);
        atomicMin(&s[VPS_SEG_Y0 * NKEY + key], (uint32_t)y);
        atomicMax(&s[VPS_SEG_X1 * NKEY + key], (uint32_t)xb);
        atomicMax(&s[VPS_SEG_Y1 * NKEY + key], (uint32_t)y);
      } else if (key == -2) {
        atomicAdd(&s_bad, m);
      }
    };
#pragma unroll
    for (int e = 0; e < SEG_RUN; ++e) {
      if (e < cnt) {
        const uint32_t sem = px[3 * e], trk = px[3 * e + KEY_CH];
        const int key = sem == 255u ? -1 : (sem < (uint32_t)VPS_SEG_NSEM ? (int)(sem * 256u + trk) : -2);
        const uint32_t id = key == -2 ? 0u : seg_id(sem, trk, num_stuff);
        out[3 * e] = (uint8_t)(id & 255u);
        out[3 * e + 1] = (uint8_t)((id >> 8) & 255u);
        out[3 * e + 2] = (uint8_t)(id >> 16);
        if (e == 0) { cur = key; n = 1; }
        else if (key == cur) { ++n; }
        else { flush(cur, xs, x0 + e - 1, n); cur = key; xs = x0 + e; n = 1; }
      } else {
        out[3 * e] = out[3 * e + 1] = out[3 * e + 2] = 0;
      }
    }
    flush(cur, xs, x0 + cnt - 1, n);
    if (rgb != nullptr) {
      if (vec) {
        uint4* dst = reinterpret_cast<uint4*>(rgb + base);
#pragma unroll
        for (int q = 0; q < 3; ++q) dst[q] = reinterpret_cast<const uint4*>(out)[q];
      } else {
#pragma unroll
        for (int e = 0; e < 3 * SEG_RUN; ++e)
          if (e < 3 * cnt) rgb[base + e] = out[e];
      }
    }
  }
  __syncthreads();
  for (uint32_t k = threadIdx.x; k < NKEY; k += blockDim.x) {
    const uint32_t a = s[VPS_SEG_AREA * NKEY + k];
    if (a == 0) continue;
    atomicAdd(&table[VPS_SEG_AREA * NKEY + k], a);
    atomicMin(&table[VPS_SEG_X0 * NKEY + k], s[VPS_SEG_X0 * NKEY + k]);
    atomicMin(&table[VPS_SEG_Y0 * NKEY + k], s[VPS_SEG_Y0 * NKEY + k]);
    atomicMax(&table[VPS_SEG_X1 * NKEY + k], s[VPS_SEG_X1 * NKEY + k]);
    atomicMax(&table[VPS_SEG_Y1 * NKEY + k], s[VPS_SEG_Y1 * NKEY + k]);
  }
  if (threadIdx.x == 0 && s_bad != 0) atomicAdd(&table[VPS_SEG_PLANES * NKEY], s_bad);
}
template <int KEY_CH>
int pan2ch_segments(const uint8_t* pan_2ch, int H, int W, int num_stuff, uint32_t* table, uint8_t* rgb_out, void* stream) {
  VPS_CHECK_ARG(H >= 0 && W >= 0 && table != nullptr, "pan2ch_segments: bad arguments (H %d, W %d)", H, W);
  cudaStream_t st = (cudaStream_t)stream;
  seg_table_init_kernel<<<vps::cdiv(VPS_SEG_TABLE_WORDS, 256), 256, 0, st>>>(table);
  VPS_CUDA_LAST("pan2ch_segments_init");
  if ((int64_t)H * W == 0) return VPS_OK;
  const int sms = vps::num_sms();
  if (sms <= 0) { vps::set_error("pan2ch_segments: no device"); return VPS_E_NODEV; }
  const size_t smem = (size_t)VPS_SEG_PLANES * NKEY * sizeof(uint32_t);
  cudaError_t e = cudaFuncSetAttribute(pan2ch_segments_kernel<KEY_CH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { vps::set_error("pan2ch_segments: smem attribute: %s", cudaGetErrorString(e)); return VPS_E_CUDA; }
  const bool vec = W % SEG_RUN == 0 && ((uintptr_t)pan_2ch & 15) == 0 && ((uintptr_t)rgb_out & 15) == 0;
  const int64_t nstrip = (int64_t)H * ((W + SEG_RUN - 1) / SEG_RUN);
  // about four strips per thread, at most two resident blocks per SM (the table fills 95 KiB of shared memory)
  const int64_t want = (nstrip + 256 * 4 - 1) / (256 * 4);
  const int blocks = (int)(want < 2 * sms ? (want < 1 ? 1 : want) : 2 * sms);
  pan2ch_segments_kernel<KEY_CH><<<blocks, 256, smem, st>>>(pan_2ch, H, W, (uint32_t)num_stuff, table, rgb_out, vec);
  VPS_CUDA_LAST("pan2ch_segments");
  return VPS_OK;
}
}  // namespace

extern "C" int vps_pan2ch_segments(const uint8_t* pan_2ch, int H, int W, int num_stuff, uint32_t* table, uint8_t* rgb_out,
                                   void* stream) {
  return pan2ch_segments<2>(pan_2ch, H, W, num_stuff, table, rgb_out, stream);
}

extern "C" int vps_pan2ch_image_segments(const uint8_t* pan_2ch, int H, int W, int num_stuff, uint32_t* table,
                                         uint8_t* rgb_out, void* stream) {
  return pan2ch_segments<1>(pan_2ch, H, W, num_stuff, table, rgb_out, stream);
}
