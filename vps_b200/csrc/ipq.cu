// The pixel pass of the semantic-segmentation evaluation of the reference (Cityscapes.evaluate_ssegs,
// tools/dataset/cityscapes.py:112-166, with get_confusion_matrix of tools/dataset/base_dataset.py:449-467): a C x C
// confusion matrix of ground-truth trainIds against predicted labels, accumulated over frames on the device.
//   index = gt * C + pred over the pixels with gt != 255; np.bincount; bins index < C * C go to [index / C][index % C].
// So a prediction >= C aliases into the next row, and a gt in [C, 255) is dropped unless its index is still < C * C.
// One pass over (gt, pred): per-block shared-memory bins fed one atomic per run of equal labels in a 16-pixel strip
// (label_runs.cuh), then one 64-bit global atomic per non-zero bin per block.
#include "label_runs.cuh"

namespace {
constexpr int MAX_SEG_CLASSES = 64;

template <typename TL>
__global__ void __launch_bounds__(256) seg_confusion_kernel(const uint8_t* __restrict__ gt, const TL* __restrict__ pred,
                                                            int64_t npix, int C, unsigned long long* __restrict__ conf) {
  __shared__ unsigned int s_bin[MAX_SEG_CLASSES * MAX_SEG_CLASSES];
  const int nbin = C * C;
  for (int i = threadIdx.x; i < nbin; i += blockDim.x) s_bin[i] = 0;
  __syncthreads();
  vps::walk_label_runs(gt, pred, npix, [&](int g, int p, unsigned int n) {
    const int idx = g * C + p;
    if (g != 255 && idx < nbin) atomicAdd(&s_bin[idx], n);
  });
  __syncthreads();
  for (int i = threadIdx.x; i < nbin; i += blockDim.x)
    if (s_bin[i]) atomicAdd(&conf[i], (unsigned long long)s_bin[i]);
}
}  // namespace

extern "C" int vps_seg_confusion(const uint8_t* gt, const void* pred, int label_bytes, int64_t npix, int num_classes,
                                 uint64_t* conf, void* stream) {
  VPS_CHECK_ARG(label_bytes == 1 || label_bytes == 8, "seg_confusion: label_bytes %d", label_bytes);
  VPS_CHECK_ARG(num_classes >= 1 && num_classes <= MAX_SEG_CLASSES, "seg_confusion: num_classes %d (1..%d)", num_classes,
                MAX_SEG_CLASSES);
  VPS_CHECK_ARG(npix >= 0 && ((uintptr_t)conf & 7) == 0, "seg_confusion: npix %lld / matrix alignment", (long long)npix);
  if (npix == 0) return VPS_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int blocks = vps::grid_for((npix + vps::LABEL_RUN - 1) / vps::LABEL_RUN);
  unsigned long long* c = (unsigned long long*)conf;
  if (label_bytes == 1) seg_confusion_kernel<uint8_t><<<blocks, 256, 0, st>>>(gt, (const uint8_t*)pred, npix, num_classes, c);
  else seg_confusion_kernel<int64_t><<<blocks, 256, 0, st>>>(gt, (const int64_t*)pred, npix, num_classes, c);
  VPS_CUDA_LAST("seg_confusion");
  return VPS_OK;
}
