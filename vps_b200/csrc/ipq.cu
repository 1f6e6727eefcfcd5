// The pixel pass of the semantic-segmentation evaluation of the reference (Cityscapes.evaluate_ssegs,
// tools/dataset/cityscapes.py:112-166, with get_confusion_matrix of tools/dataset/base_dataset.py:449-467): a C x C
// confusion matrix of ground-truth trainIds against predicted labels, accumulated over frames on the device.
//   index = gt * C + pred over the pixels with gt != 255; np.bincount; bins index < C * C go to [index / C][index % C].
// So a prediction >= C aliases into the next row, and a gt in [C, 255) is dropped unless its index is still < C * C.
// One pass over (gt, pred): per-block shared-memory bins fed one atomic per run of equal labels in a 16-pixel strip
// (label_runs.cuh), then one 64-bit global atomic per non-zero bin per block.  vps_seg_confusion_nearest is the same pass
// for a prediction of another shape, read through Image.NEAREST index tables.
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

// The prediction of another shape, read through the Image.NEAREST resize evaluate_ssegs applies to it
// (cityscapes.py:125-126): pixel (y, x) of the gt takes the prediction at (ytab[y], xtab[x]); an index < 0 stands for
// Pillow's fill value 0.  Nothing resized is written: the strip walker fetches the gathered labels directly.
template <typename TL>
struct NearestStrip {
  const TL* __restrict__ pred;
  const int* __restrict__ xtab;
  const int* __restrict__ ytab;
  int gw, pw;
  __device__ __forceinline__ void operator()(int64_t i0, int cnt, int (&v)[vps::LABEL_RUN]) const {
    int y = (int)(i0 / gw), x = (int)(i0 - (int64_t)y * gw);
    int yi = __ldg(ytab + y);
#pragma unroll
    for (int e = 0; e < vps::LABEL_RUN; ++e) {
      if (e < cnt) {
        const int xi = __ldg(xtab + x);
        v[e] = (yi < 0 || xi < 0) ? 0 : vps::lab(pred, (int64_t)yi * pw + xi);
        if (++x == gw && e + 1 < cnt) { x = 0; yi = __ldg(ytab + ++y); }
      } else {
        v[e] = -1;
      }
    }
  }
};

// the per-pixel rule of seg_confusion_kernel with the prediction gathered through the index tables.  The reference wraps
// the prediction with np.uint8 before it resizes it; vps::lab reads the low byte, which is that wrap, and fcn_outputs
// (semantic argmaxes < C) are unchanged by it anyway.
template <typename TL>
__global__ void __launch_bounds__(256) seg_confusion_nearest_kernel(const uint8_t* __restrict__ gt, int gh, int gw,
                                                                    NearestStrip<TL> pred, int C,
                                                                    unsigned long long* __restrict__ conf) {
  __shared__ unsigned int s_bin[MAX_SEG_CLASSES * MAX_SEG_CLASSES];
  const int nbin = C * C;
  for (int i = threadIdx.x; i < nbin; i += blockDim.x) s_bin[i] = 0;
  __syncthreads();
  vps::walk_label_runs_by(vps::StripOf<uint8_t>{gt}, pred, (int64_t)gh * gw, [&](int g, int p, unsigned int n) {
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

extern "C" int vps_seg_confusion_nearest(const uint8_t* gt, int gh, int gw, const void* pred, int pred_elem, int ph, int pw,
                                         const int* xtab, const int* ytab, int num_classes, uint64_t* conf, void* stream) {
  VPS_CHECK_ARG(pred_elem == 1 || pred_elem == 8, "seg_confusion_nearest: pred_elem %d", pred_elem);
  VPS_CHECK_ARG(num_classes >= 1 && num_classes <= MAX_SEG_CLASSES, "seg_confusion_nearest: num_classes %d (1..%d)", num_classes,
                MAX_SEG_CLASSES);
  VPS_CHECK_ARG(gh >= 0 && gw >= 0 && ph > 0 && pw > 0 && ((uintptr_t)conf & 7) == 0,
                "seg_confusion_nearest: shapes gt %dx%d pred %dx%d / matrix alignment", gh, gw, ph, pw);
  const int64_t npix = (int64_t)gh * gw;
  if (npix == 0) return VPS_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int blocks = vps::grid_for((npix + vps::LABEL_RUN - 1) / vps::LABEL_RUN);
  unsigned long long* c = (unsigned long long*)conf;
  if (pred_elem == 1)
    seg_confusion_nearest_kernel<uint8_t><<<blocks, 256, 0, st>>>(
        gt, gh, gw, NearestStrip<uint8_t>{(const uint8_t*)pred, xtab, ytab, gw, pw}, num_classes, c);
  else
    seg_confusion_nearest_kernel<int64_t><<<blocks, 256, 0, st>>>(
        gt, gh, gw, NearestStrip<int64_t>{(const int64_t*)pred, xtab, ytab, gw, pw}, num_classes, c);
  VPS_CUDA_LAST("seg_confusion_nearest");
  return VPS_OK;
}
