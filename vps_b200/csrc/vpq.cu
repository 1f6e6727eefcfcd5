// SURVEY 8f rank 2: the pixel-level step of the VPQ evaluator (reference tools/eval_vpq.py:138-145):
//   vid_pan_gt_pred = gt.astype(uint64) * 2^24 + pred;  labels, counts = np.unique(vid_pan_gt_pred, return_counts=True)
// over a tube of nframes id maps.  On the device: pack -> 64-bit radix sort (CUB) -> run-length encode (CUB); the few
// hundred (gt, pred, count) triples go back to the host, where the matching logic of the reference runs unchanged.
#include <cub/cub.cuh>

#include "common.cuh"

namespace {
__global__ void pack_pairs_kernel(const uint32_t* __restrict__ gt, const uint32_t* __restrict__ pred, int64_t n,
                                  unsigned long long offset, unsigned long long* __restrict__ keys) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    keys[i] = (unsigned long long)gt[i] * offset + (unsigned long long)pred[i];
}
// r + 256 g + 65536 b of an RGB-coded id image (eval_vpq.py:87-89)
__global__ void rgb_to_id_kernel(const uint8_t* __restrict__ rgb, int64_t n, uint32_t* __restrict__ ids) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    ids[i] = (uint32_t)rgb[3 * i] + 256u * rgb[3 * i + 1] + 65536u * rgb[3 * i + 2];
}

// segment id of a pixel of the unified 3-channel result (semantic, instance rank, track id).  The reference's converter
// (tools/dataset/cityscapes_vps.py:104-140) walks the keys OFFSET * semantic + track channel, skips VOID (semantic 255) and
// makes the segment id the COLOUR panopticapi's IdGenerator returns: one fixed colour per stuff category -- so every key of
// a stuff category (the native stuff pixels carry their pan value in the track channel, a thing region demoted to stuff
// carries 0) collapses into ONE segment per frame -- and one colour per (thing category, track) key, kept across frames.
// Deterministic stand-in for the colours: stuff -> 1000 * semantic + 1, thing -> 1000 * semantic + track + 1, VOID -> 0.
// KEY_CH = 2 is that video converter.  KEY_CH = 1 is the image converter (tools/dataset/base_dataset.py:287-335), which
// keys pixels by 1000 * semantic + instance rank: one segment per thing instance, and, since the image-level unify leaves
// the instance channel 0 on every stuff pixel, one per stuff category.
template <int KEY_CH>
__global__ void pan2ch_ids_kernel(const uint8_t* __restrict__ p2, int64_t n, uint32_t num_stuff, uint32_t* __restrict__ ids) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t sem = p2[3 * i], key = p2[3 * i + KEY_CH];
    ids[i] = sem == 255u ? 0u : 1000u * sem + (sem < num_stuff ? 0u : key) + 1u;
  }
}

template <int KEY_CH>
int pan2ch_ids(const uint8_t* pan_2ch, int64_t npix, int num_stuff, uint32_t* ids, void* stream) {
  if (npix <= 0) return VPS_OK;
  const int blocks = (int)((npix + 255) / 256 > 148 * 16 ? 148 * 16 : (npix + 255) / 256);
  pan2ch_ids_kernel<KEY_CH><<<blocks, 256, 0, (cudaStream_t)stream>>>(pan_2ch, npix, (uint32_t)num_stuff, ids);
  VPS_CUDA_LAST("pan2ch_ids");
  return VPS_OK;
}

struct Layout { size_t keys, sorted, temp, temp_bytes, total; };
Layout layout(int64_t n, int cap) {
  Layout l;
  size_t t1 = 0, t2 = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, t1, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)n, 0, 64);
  cub::DeviceRunLengthEncode::Encode(nullptr, t2, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (unsigned int*)nullptr,
                                     (int*)nullptr, (int)n);
  l.temp_bytes = (t1 > t2 ? t1 : t2);
  auto up = [](size_t v) { return (v + 255) / 256 * 256; };
  l.keys = 0;
  l.sorted = up(l.keys + (size_t)n * 8);
  l.temp = up(l.sorted + (size_t)n * 8);
  l.total = up(l.temp + l.temp_bytes);
  (void)cap;
  return l;
}
}  // namespace

extern "C" int64_t vps_tube_confusion_ws_bytes(int64_t npix) { return npix > 0 ? (int64_t)layout(npix, 0).total : 256; }

extern "C" int vps_pan2ch_ids(const uint8_t* pan_2ch, int64_t npix, int num_stuff, uint32_t* ids, void* stream) {
  return pan2ch_ids<2>(pan_2ch, npix, num_stuff, ids, stream);
}

extern "C" int vps_pan2ch_image_ids(const uint8_t* pan_2ch, int64_t npix, int num_stuff, uint32_t* ids, void* stream) {
  return pan2ch_ids<1>(pan_2ch, npix, num_stuff, ids, stream);
}

extern "C" int vps_rgb_to_id(const uint8_t* rgb, int64_t npix, uint32_t* ids, void* stream) {
  if (npix <= 0) return VPS_OK;
  const int blocks = (int)((npix + 255) / 256 > 148 * 16 ? 148 * 16 : (npix + 255) / 256);
  rgb_to_id_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(rgb, npix, ids);
  VPS_CUDA_LAST("rgb_to_id");
  return VPS_OK;
}

// pairs_out / counts_out must hold one entry per DISTINCT pair; the exact number is written to *nruns_dev (device).  If it
// exceeds `cap` the results are still written (CUB needs room for npix runs in the worst case), so cap must be >= npix or the
// caller must size the outputs for the worst case; the host wrapper allocates npix entries and reads back only *nruns.
extern "C" int vps_tube_confusion(const uint32_t* gt_ids, const uint32_t* pred_ids, int64_t npix, uint64_t offset, uint64_t* pairs_out,
                                  uint32_t* counts_out, int* nruns_dev, void* ws, int64_t ws_bytes, void* stream) {
  VPS_CHECK_ARG(npix >= 0 && npix < (1ll << 31), "tube_confusion: npix %lld", (long long)npix);
  cudaStream_t st = (cudaStream_t)stream;
  if (npix == 0) { cudaMemsetAsync(nruns_dev, 0, sizeof(int), st); return VPS_OK; }
  const Layout l = layout(npix, 0);
  VPS_CHECK_ARG(ws_bytes >= (int64_t)l.total && ((uintptr_t)ws & 255) == 0, "tube_confusion: workspace %lld < %lld", (long long)ws_bytes,
                (long long)l.total);
  unsigned long long* keys = (unsigned long long*)((char*)ws + l.keys);
  unsigned long long* sorted = (unsigned long long*)((char*)ws + l.sorted);
  void* temp = (char*)ws + l.temp;
  size_t tb = l.temp_bytes;
  const int blocks = (int)((npix + 255) / 256 > 148 * 16 ? 148 * 16 : (npix + 255) / 256);
  pack_pairs_kernel<<<blocks, 256, 0, st>>>(gt_ids, pred_ids, npix, (unsigned long long)offset, keys);
  VPS_CUDA_LAST("pack_pairs");
  cudaError_t e = cub::DeviceRadixSort::SortKeys(temp, tb, keys, sorted, (int)npix, 0, 64, st);
  if (e != cudaSuccess) { vps::set_error("tube_confusion: sort: %s", cudaGetErrorString(e)); return VPS_E_CUDA; }
  tb = l.temp_bytes;
  e = cub::DeviceRunLengthEncode::Encode(temp, tb, sorted, (unsigned long long*)pairs_out, counts_out, nruns_dev, (int)npix, st);
  if (e != cudaSuccess) { vps::set_error("tube_confusion: rle: %s", cudaGetErrorString(e)); return VPS_E_CUDA; }
  vps::count_launch(4);
  return VPS_OK;
}
