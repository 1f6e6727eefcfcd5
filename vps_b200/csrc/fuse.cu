// Panoptic fusion kernels: MaskRemoval (mask_removal.py:29-92) and the final per-pixel fusion
// (SegTerm unary_logits.py:81-108 + mask paste mask_removal.py:86 + argmax panoptic_fusetrack.py:588-593).
// Neither the [1,k,H,W] mask_energy tensor nor the [1,11+k,H,W] logits tensor of the reference is
// ever materialised: resized mask logits are recomputed from the 28x28 maps wherever they are needed.
#include <cooperative_groups.h>

#include "common.cuh"

namespace {

// cv2.resize(src[ms x ms] f32, (w, h), INTER_LINEAR) value at (dy, dx): half-pixel centres, taps clamped
// with the fractional weight zeroed at the borders (OpenCV resize.cpp linear coefficient tables).
__device__ __forceinline__ float cv_resize_linear(const float* __restrict__ src, int ms, int w, int h, int dy, int dx) {
  const double scale_x = (double)ms / (double)w, scale_y = (double)ms / (double)h;
  float fx = (float)(((double)dx + 0.5) * scale_x - 0.5);
  int sx = (int)floorf(fx);
  fx -= (float)sx;
  if (sx < 0) { fx = 0.f; sx = 0; }
  if (sx >= ms - 1) { fx = 0.f; sx = ms - 1; }
  float fy = (float)(((double)dy + 0.5) * scale_y - 0.5);
  int sy = (int)floorf(fy);
  fy -= (float)sy;
  if (sy < 0) { fy = 0.f; sy = 0; }
  if (sy >= ms - 1) { fy = 0.f; sy = ms - 1; }
  const int sx1 = min(sx + 1, ms - 1), sy1 = min(sy + 1, ms - 1);
  const float a0 = 1.f - fx, a1 = fx, b0 = 1.f - fy, b1 = fy;
  const float r0 = src[sy * ms + sx] * a0 + src[sy * ms + sx1] * a1;
  const float r1 = src[sy1 * ms + sx] * a0 + src[sy1 * ms + sx1] * a1;
  return r0 * b0 + r1 * b1;
}

constexpr int MAX_DET_K = 128;
struct BoxI { int x1, y1, x2, y2, w, h, x_0, x_1, y_0, y_1; };
__device__ __forceinline__ BoxI int_box(const float* b, int H, int W) {
  BoxI r;
  r.x1 = (int)b[0]; r.y1 = (int)b[1]; r.x2 = (int)b[2]; r.y2 = (int)b[3];   // astype(np.int32): trunc toward 0
  r.w = max(r.x2 - r.x1 + 1, 1); r.h = max(r.y2 - r.y1 + 1, 1);
  r.x_0 = max(r.x1, 0); r.x_1 = min(r.x2 + 1, W);
  r.y_0 = max(r.y1, 0); r.y_1 = min(r.y2 + 1, H);
  return r;
}

// pass A for sorted position `pos`: count mask pixels and pixels already claimed by the same class
__global__ void mr_count_kernel(const float* __restrict__ boxes, const int32_t* __restrict__ order, int pos, int k,
                                const int* __restrict__ k_dev, const float* __restrict__ mask_logit, int ms,
                                const int32_t* __restrict__ cls_idx, int H, int W, const uint8_t* __restrict__ occ,
                                unsigned int* __restrict__ counters) {
  const int kk = k_dev ? min(*k_dev, k) : k;
  if (pos >= kk) return;
  const int det = order[pos];
  const int cls = cls_idx[det] - 1;
  if (cls < 0) return;
  const BoxI b = int_box(boxes + (int64_t)det * 4, H, W);
  const int cw = b.x_1 - b.x_0, ch = b.y_1 - b.y_0;
  if (cw <= 0 || ch <= 0) return;
  const float* ml = mask_logit + (int64_t)det * ms * ms;
  const uint8_t* oc = occ + (int64_t)cls * H * W;
  unsigned int msum = 0, osum = 0;
  const int64_t total = (int64_t)cw * ch;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = b.x_0 + (int)(i % cw), y = b.y_0 + (int)(i / cw);
    const float v = cv_resize_linear(ml, ms, b.w, b.h, y - b.y1, x - b.x1);
    if (v > 0.f) {
      msum++;
      if (oc[(int64_t)y * W + x] >= 1) osum++;
    }
  }
  for (int o = 16; o > 0; o >>= 1) { msum += __shfl_xor_sync(0xffffffffu, msum, o); osum += __shfl_xor_sync(0xffffffffu, osum, o); }
  if ((threadIdx.x & 31) == 0 && (msum | osum)) {
    atomicAdd(counters + 2 * pos, msum);
    atomicAdd(counters + 2 * pos + 1, osum);
  }
}

// pass B: decide keep (mask_removal.py:81-83) and, if kept, add the mask into the class occupancy image
__global__ void mr_apply_kernel(const float* __restrict__ boxes, const int32_t* __restrict__ order, int pos, int k,
                                const int* __restrict__ k_dev, const float* __restrict__ mask_logit, int ms,
                                const int32_t* __restrict__ cls_idx, int H, int W, float frac_thr, uint8_t* __restrict__ occ,
                                const unsigned int* __restrict__ counters, int32_t* __restrict__ keep_flag) {
  const int kk = k_dev ? min(*k_dev, k) : k;
  if (pos >= kk) return;
  const int det = order[pos];
  const int cls = cls_idx[det] - 1;
  const unsigned int msum = counters[2 * pos], osum = counters[2 * pos + 1];
  // numpy: int / int -> float64 true division compared with the python float 0.3
  const bool keep = cls >= 0 && msum != 0 && !((double)osum / (double)msum > (double)frac_thr);
  if (blockIdx.x == 0 && threadIdx.x == 0) keep_flag[pos] = keep ? 1 : 0;
  if (!keep) return;
  const BoxI b = int_box(boxes + (int64_t)det * 4, H, W);
  const int cw = b.x_1 - b.x_0, ch = b.y_1 - b.y_0;
  const float* ml = mask_logit + (int64_t)det * ms * ms;
  uint8_t* oc = occ + (int64_t)cls * H * W;
  const int64_t total = (int64_t)cw * ch;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = b.x_0 + (int)(i % cw), y = b.y_0 + (int)(i / cw);
    const float v = cv_resize_linear(ml, ms, b.w, b.h, y - b.y1, x - b.x1);
    if (v > 0.f) oc[(int64_t)y * W + x] += 1;   // uint8 += (wraps like numpy)
  }
}

// ---- class-parallel MaskRemoval: boxes of different classes never interact (the occupancy image is per class,
// mask_removal.py:44,81-85), so the sequential dependence only runs along each class's score-ordered chain.
// Boxes grouped by class in score order (MaskRemoval only compares boxes of the same class, mask_removal.py:40-58).
struct MrSched { int slot[8][MAX_DET_K]; int count[8]; int steps; };

__global__ void mr_schedule_kernel(const int32_t* __restrict__ order, const int32_t* __restrict__ cls_idx, int k,
                                   const int* __restrict__ k_dev, int num_things, MrSched* __restrict__ sc) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int kk = k_dev ? min(*k_dev, k) : k;
  for (int c = 0; c < 8; ++c) sc->count[c] = 0;
  int steps = 0;
  for (int pos = 0; pos < kk; ++pos) {
    const int c = cls_idx[order[pos]] - 1;
    if (c < 0 || c >= num_things || c >= 8) continue;       // dummy / invalid class: never kept
    sc->slot[c][sc->count[c]++] = pos;
    steps = max(steps, sc->count[c]);
  }
  sc->steps = steps;
}

// One 8-CTA thread-block cluster per thing class: the boxes of a class are handled in score order with two hardware
// cluster barriers per box (count -> decide/apply); classes never wait for each other and no grid-wide sync exists.
constexpr int MR_CLUSTER = 8;
__global__ void __cluster_dims__(MR_CLUSTER, 1, 1) __launch_bounds__(256)
mr_cluster_kernel(const float* __restrict__ boxes, const int32_t* __restrict__ order, const float* __restrict__ mask_logit,
                  int ms, const int32_t* __restrict__ cls_idx, int H, int W, float frac_thr, uint8_t* __restrict__ occ,
                  unsigned int* __restrict__ counters, int32_t* __restrict__ keep_flag, const MrSched* __restrict__ sc) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int cls = blockIdx.x / MR_CLUSTER;
  const int part = (int)cluster.block_rank(), nparts = MR_CLUSTER;
  const int cnt = sc->count[cls];
  uint8_t* oc = occ + (int64_t)cls * H * W;
  for (int t = 0; t < cnt; ++t) {
    const int pos = sc->slot[cls][t];
    const int det = order[pos];
    const BoxI b = int_box(boxes + (int64_t)det * 4, H, W);
    const int cw = b.x_1 - b.x_0, ch = b.y_1 - b.y_0;
    const float* ml = mask_logit + (int64_t)det * ms * ms;
    const int total = (cw > 0 && ch > 0) ? cw * ch : 0;
    // ---- count mask pixels and those already occupied by a kept box of this class
    unsigned int msum = 0, osum = 0;
    for (int i = part * blockDim.x + threadIdx.x; i < total; i += nparts * blockDim.x) {
      const int x = b.x_0 + i % cw, y = b.y_0 + i / cw;
      const float v = cv_resize_linear(ml, ms, b.w, b.h, y - b.y1, x - b.x1);
      if (v > 0.f) { msum++; if (__ldcg(oc + (int64_t)y * W + x) >= 1) osum++; }   // L2 reads: other SMs wrote it
    }
    for (int o = 16; o > 0; o >>= 1) { msum += __shfl_xor_sync(0xffffffffu, msum, o); osum += __shfl_xor_sync(0xffffffffu, osum, o); }
    if ((threadIdx.x & 31) == 0 && (msum | osum)) { atomicAdd(counters + 2 * pos, msum); atomicAdd(counters + 2 * pos + 1, osum); }
    cluster.sync();
    // ---- decide + apply
    const unsigned int ms_all = __ldcg(counters + 2 * pos), os_all = __ldcg(counters + 2 * pos + 1);
    const bool keep = ms_all != 0 && !((double)os_all / (double)ms_all > (double)frac_thr);
    if (part == 0 && threadIdx.x == 0) keep_flag[pos] = keep ? 1 : 0;
    if (keep) {
      for (int i = part * blockDim.x + threadIdx.x; i < total; i += nparts * blockDim.x) {
        const int x = b.x_0 + i % cw, y = b.y_0 + i / cw;
        const float v = cv_resize_linear(ml, ms, b.w, b.h, y - b.y1, x - b.x1);
        if (v > 0.f) { uint8_t* q = oc + (int64_t)y * W + x; __stcg(q, (uint8_t)(__ldcg(q) + 1)); }
      }
    }
    cluster.sync();
  }
}

// compact kept detections in sorted order: keep_sorted[j] = det index of the j-th kept one
__global__ void mr_compact_kernel(const int32_t* __restrict__ order, const int32_t* __restrict__ keep_flag, int k,
                                  const int* __restrict__ k_dev, int32_t* __restrict__ keep_sorted, int* __restrict__ nkeep) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int kk = k_dev ? min(*k_dev, k) : k;
  int n = 0;
  for (int i = 0; i < kk; ++i)
    if (keep_flag[i]) keep_sorted[n++] = order[i];
  *nkeep = n;
}

// ------------------------------------------------------------------ final fusion
constexpr int MAX_INST = 128;
struct InstParams {
  // SegTerm box (unary_logits.py:99-103) and paste box (mask_removal.py:59-86), per kept instance
  int sy0[MAX_INST], sy1[MAX_INST], sx0[MAX_INST], sx1[MAX_INST];
  int bx1[MAX_INST], by1[MAX_INST], bw[MAX_INST], bh[MAX_INST], px0[MAX_INST], px1[MAX_INST], py0[MAX_INST], py1[MAX_INST];
  int seg_ch[MAX_INST];   // channel of fcn_output feeding inst_seg, -1 for the dummy instance
  int det[MAX_INST];
};

__global__ void fuse_prepare_kernel(const float* __restrict__ boxes, const int32_t* __restrict__ cls_idx,
                                    const int32_t* __restrict__ keep_sorted, const int* __restrict__ nkeep_dev, int kcap,
                                    int num_stuff, int H, int W, InstParams* __restrict__ ip, int* __restrict__ ninst) {
  const int j = threadIdx.x;
  // MaskRemoval kept nothing: the reference falls back to keep_inds = [0] with an all-zero mask energy
  // (mask_removal.py:89-91), so detection 0 (original order) still adds its SegTerm channel
  const int nkeep = *nkeep_dev;
  const bool fallback = nkeep == 0;
  const int nk = min(fallback ? 1 : nkeep, kcap);
  if (j == 0) *ninst = nk;
  if (j >= nk) return;
  const int det = fallback ? 0 : keep_sorted[j];
  const float* b = boxes + (int64_t)det * 4;
  const int cls = cls_idx[det];
  ip->det[j] = det;
  ip->seg_ch[j] = cls > 0 ? (num_stuff - 1 + cls) : -1;   // class_mapping {1..8 -> 11..18} (fusetrack.py:148)
  // SegTerm: boxes*(1/4) of mask_rois*4 is exact; y0=int(y1), y1=int(round(y2)+1) (np.round = half-to-even)
  ip->sy0[j] = (int)b[1]; ip->sy1[j] = (int)(rintf(b[3]) + 1.f);
  ip->sx0[j] = (int)b[0]; ip->sx1[j] = (int)(rintf(b[2]) + 1.f);
  const BoxI r = int_box(b, H, W);
  ip->bx1[j] = r.x1; ip->by1[j] = r.y1; ip->bw[j] = r.w; ip->bh[j] = r.h;
  ip->px0[j] = r.x_0; ip->px1[j] = r.x_1; ip->py0[j] = r.y_0; ip->py1[j] = r.y_1;
  if (fallback) { ip->px0[j] = ip->px1[j] = ip->py0[j] = ip->py1[j] = 0; }   // empty paste box: no mask energy
}

// One block = one 32 x 8 pixel tile.  Instances whose SegTerm box and paste box both miss the tile contribute the
// constant logit 0 there; only the FIRST of them can ever win the first-max argmax, so the tile's candidate list is
// {instances overlapping the tile} + {first non-overlapping instance}, in instance order -- identical results to the
// reference's dense [stuff | instances] argmax, without looping over every instance at every pixel.
constexpr int FUSE_TW = 32, FUSE_TH = 8;
template <typename T, typename TL>
__global__ void __launch_bounds__(FUSE_TW * FUSE_TH) panoptic_fuse_kernel(vps::TV<const T> score, const float* __restrict__ mask_logit,
                                                            int ms, const InstParams* __restrict__ ipg,
                                                            const int* __restrict__ ninst_dev, int num_stuff, int dummy,
                                                            int H, int W, TL* __restrict__ pano, TL* __restrict__ sem) {
  __shared__ int s_cnt[4], s_first[4];
  __shared__ int s_j[MAX_INST], s_seg[MAX_INST], s_det[MAX_INST];
  __shared__ int s_sy0[MAX_INST], s_sy1[MAX_INST], s_sx0[MAX_INST], s_sx1[MAX_INST];
  __shared__ int s_py0[MAX_INST], s_py1[MAX_INST], s_px0[MAX_INST], s_px1[MAX_INST];
  __shared__ int s_bx1[MAX_INST], s_by1[MAX_INST], s_bw[MAX_INST], s_bh[MAX_INST];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tx0 = blockIdx.x * FUSE_TW, ty0 = blockIdx.y * FUSE_TH;
  const int ninst = dummy ? 0 : *ninst_dev;
  // ---- candidate list of this tile (threads 0..127 = instances)
  bool hit = false, valid = false;
  int rank_in_warp = 0;
  int sy0 = 0, sy1 = 0, sx0 = 0, sx1 = 0, py0 = 0, py1 = 0, px0 = 0, px1 = 0, seg = -1;
  if (tid < MAX_INST) {
    valid = tid < ninst;
    if (valid) {
      sy0 = ipg->sy0[tid]; sy1 = ipg->sy1[tid]; sx0 = ipg->sx0[tid]; sx1 = ipg->sx1[tid];
      py0 = ipg->py0[tid]; py1 = ipg->py1[tid]; px0 = ipg->px0[tid]; px1 = ipg->px1[tid];
      seg = ipg->seg_ch[tid];
      const bool hs = seg >= 0 && sy0 < ty0 + FUSE_TH && sy1 > ty0 && sx0 < tx0 + FUSE_TW && sx1 > tx0;
      const bool hp = py0 < ty0 + FUSE_TH && py1 > ty0 && px0 < tx0 + FUSE_TW && px1 > tx0;
      hit = hs || hp;
    }
    const unsigned miss = __ballot_sync(0xffffffffu, valid && !hit);
    if (lane == 0) s_first[warp] = miss ? warp * 32 + (__ffs(miss) - 1) : 0x7fffffff;
  }
  __syncthreads();
  if (tid < MAX_INST) {
    const int first_miss = min(min(s_first[0], s_first[1]), min(s_first[2], s_first[3]));
    const bool listed = hit || tid == first_miss;
    const unsigned bal = __ballot_sync(0xffffffffu, listed);
    if (lane == 0) s_cnt[warp] = __popc(bal);
    rank_in_warp = __popc(bal & ((1u << lane) - 1u));
    hit = listed;
  }
  __syncthreads();
  if (tid < MAX_INST && hit) {
    int base = 0;
    for (int w = 0; w < warp; ++w) base += s_cnt[w];
    const int slot = base + rank_in_warp;
    s_j[slot] = tid; s_seg[slot] = seg; s_det[slot] = ipg->det[tid];
    s_sy0[slot] = sy0; s_sy1[slot] = sy1; s_sx0[slot] = sx0; s_sx1[slot] = sx1;
    s_py0[slot] = py0; s_py1[slot] = py1; s_px0[slot] = px0; s_px1[slot] = px1;
    s_bx1[slot] = ipg->bx1[tid]; s_by1[slot] = ipg->by1[tid]; s_bw[slot] = ipg->bw[tid]; s_bh[slot] = ipg->bh[tid];
  }
  __syncthreads();
  const int nlist = s_cnt[0] + s_cnt[1] + s_cnt[2] + s_cnt[3];
  const int X = tx0 + lane, Y = ty0 + warp;
  if (X >= W || Y >= H) return;
  const int NC = score.c;
  const float sy = (float)score.h / (float)H, sx = (float)score.w / (float)W;
  const int64_t i = (int64_t)Y * W + X;
  {
    // fcn_output = bilinear x4 (align_corners False) of fcn_score (upsnetFPN.py:59,80)
    const float fy = fmaxf(sy * ((float)Y + 0.5f) - 0.5f, 0.f), fx = fmaxf(sx * ((float)X + 0.5f) - 0.5f, 0.f);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < score.h - 1 ? 1 : 0), x1 = x0 + (x0 < score.w - 1 ? 1 : 0);
    const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
    const T* p00 = score.p + score.off(0, y0, x0);
    const T* p01 = score.p + score.off(0, y0, x1);
    const T* p10 = score.p + score.off(0, y1, x0);
    const T* p11 = score.p + score.off(0, y1, x1);
    float fo[24];
#pragma unroll
    for (int c = 0; c < 24; ++c) {
      if (c < NC)
        fo[c] = hy * (hx * vps::ldf<T>(p00 + c) + lx * vps::ldf<T>(p01 + c)) +
                ly * (hx * vps::ldf<T>(p10 + c) + lx * vps::ldf<T>(p11 + c));
      else
        fo[c] = -INFINITY;
    }
    // semantic argmax (first max)
    float bs = fo[0]; int bsi = 0;
#pragma unroll
    for (int c = 1; c < 24; ++c) if (c < NC && fo[c] > bs) { bs = fo[c]; bsi = c; }
    sem[i] = (TL)bsi;
    // panoptic argmax over [stuff | instances]
    float bp = fo[0]; int bpi = 0;
#pragma unroll
    for (int c = 1; c < 24; ++c) if (c < num_stuff && fo[c] > bp) { bp = fo[c]; bpi = c; }
    if (dummy) {
      // MaskROI dummy detection (mask_roi.py:136-142): one all-zero instance channel
      if (0.f > bp) { bp = 0.f; bpi = num_stuff; }
    } else {
      for (int q = 0; q < nlist; ++q) {
        float v = 0.f;
        const int ch = s_seg[q];
        if (ch >= 0 && Y >= s_sy0[q] && Y < s_sy1[q] && X >= s_sx0[q] && X < s_sx1[q]) {
          float sv = 0.f;
#pragma unroll
          for (int c = 0; c < 24; ++c) if (c == ch) sv = fo[c];
          v = sv;
        }
        if (Y >= s_py0[q] && Y < s_py1[q] && X >= s_px0[q] && X < s_px1[q])
          v += cv_resize_linear(mask_logit + (int64_t)s_det[q] * ms * ms, ms, s_bw[q], s_bh[q], Y - s_by1[q], X - s_bx1[q]);
        if (v > bp) { bp = v; bpi = num_stuff + s_j[q]; }
      }
    }
    pano[i] = (TL)bpi;
  }
}

InstParams* g_ip = nullptr;
int* g_ninst = nullptr;

}  // namespace

extern "C" int vps_mask_removal(const float* boxes, const int32_t* order, int k, const int* k_dev,
                                const float* mask_logit, int msize, const int32_t* cls_idx, int H, int W, float frac_thr,
                                uint8_t* occ, int num_things, unsigned int* counters, int32_t* keep_flag,
                                int32_t* keep_sorted, int* nkeep, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(occ, 0, (size_t)num_things * H * W, st);
  cudaMemsetAsync(counters, 0, sizeof(unsigned int) * 2 * k, st);
  cudaMemsetAsync(keep_flag, 0, sizeof(int32_t) * k, st);
  static MrSched* d_sched = nullptr;
  if (!d_sched && cudaMalloc(&d_sched, sizeof(MrSched)) != cudaSuccess) { vps::set_error("mask_removal: malloc"); return VPS_E_CUDA; }
  if (k <= MAX_DET_K && num_things <= 8) {
    mr_schedule_kernel<<<1, 32, 0, st>>>(order, cls_idx, k, k_dev, num_things, d_sched);
    mr_cluster_kernel<<<num_things * MR_CLUSTER, 256, 0, st>>>(boxes, order, mask_logit, msize, cls_idx, H, W, frac_thr, occ,
                                                               counters, keep_flag, d_sched);
    vps::count_launch(1);
  } else {
    for (int pos = 0; pos < k; ++pos) {
      mr_count_kernel<<<148, 256, 0, st>>>(boxes, order, pos, k, k_dev, mask_logit, msize, cls_idx, H, W, occ, counters);
      mr_apply_kernel<<<148, 256, 0, st>>>(boxes, order, pos, k, k_dev, mask_logit, msize, cls_idx, H, W, frac_thr, occ,
                                           counters, keep_flag);
    }
    vps::count_launch(2 * k);
  }
  mr_compact_kernel<<<1, 32, 0, st>>>(order, keep_flag, k, k_dev, keep_sorted, nkeep);
  VPS_CUDA_LAST("mask_removal");
  return VPS_OK;
}

extern "C" int vps_panoptic_fuse(const vps_tensor* fcn_score, const float* boxes, const int32_t* cls_idx,
                                 const float* mask_logit, int msize, const int32_t* keep_sorted, const int* nkeep_dev,
                                 int kcap, int num_stuff, int dummy, int H, int W, void* pano_out, void* sem_out,
                                 int label_bytes, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  VPS_CHECK_ARG(label_bytes == 8 || (label_bytes == 1 && num_stuff + kcap <= 255), "panoptic_fuse: label_bytes %d", label_bytes);
  VPS_CHECK_ARG(fcn_score->c <= 24 && kcap <= MAX_INST && fcn_score->n == 1, "panoptic_fuse: args (c %d kcap %d)", fcn_score->c, kcap);
  if (!g_ip) {
    if (cudaMalloc(&g_ip, sizeof(InstParams)) != cudaSuccess || cudaMalloc(&g_ninst, sizeof(int)) != cudaSuccess) {
      vps::set_error("panoptic_fuse: malloc");
      return VPS_E_CUDA;
    }
  }
  if (dummy) {
    cudaMemsetAsync(g_ninst, 0, sizeof(int), st);
  } else {
    fuse_prepare_kernel<<<1, MAX_INST, 0, st>>>(boxes, cls_idx, keep_sorted, nkeep_dev, kcap, num_stuff, H, W, g_ip, g_ninst);
    VPS_CUDA_LAST("fuse_prepare");
  }
  const dim3 fgrid((unsigned)vps::cdiv(W, FUSE_TW), (unsigned)vps::cdiv(H, FUSE_TH));
  if (label_bytes == 8) {
    VPS_DISPATCH_T(fcn_score->dtype, T, (panoptic_fuse_kernel<T, int64_t><<<fgrid, FUSE_TW * FUSE_TH, 0, st>>>(
                                            vps::tv<const T>(*fcn_score), mask_logit, msize, g_ip, g_ninst, num_stuff, dummy,
                                            H, W, (int64_t*)pano_out, (int64_t*)sem_out)));
  } else {
    VPS_DISPATCH_T(fcn_score->dtype, T, (panoptic_fuse_kernel<T, uint8_t><<<fgrid, FUSE_TW * FUSE_TH, 0, st>>>(
                                            vps::tv<const T>(*fcn_score), mask_logit, msize, g_ip, g_ninst, num_stuff, dummy,
                                            H, W, (uint8_t*)pano_out, (uint8_t*)sem_out)));
  }
  VPS_CUDA_LAST("panoptic_fuse");
  return VPS_OK;
}
