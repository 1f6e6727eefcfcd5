// Detection-side kernels: RoIAlign with FPN level mapping, stable descending sort (CUB radix sort),
// RPN decode, greedy NMS entirely on device, MaskROI candidate generation, tracker assignment.
// All index-producing kernels are deterministic (no atomics in ordering decisions).
#include <cub/cub.cuh>

#include "common.cuh"

namespace {

// ------------------------------------------------------------------ RoIAlign
constexpr int MAXLEV = 4;
template <typename T>
struct Feats {
  vps::TV<const T> l[MAXLEV];
  float scale[MAXLEV];
  int n;
};

// roi_align_kernel.cu:16-45, V channels at once: acc += bilinear(feature, y, x)
template <typename T, int V>
__device__ __forceinline__ void bilinear_legacy_acc(const vps::TV<const T>& f, int b, int c, float y, float x, float (&acc)[V]) {
  const int H = f.h, W = f.w;
  if (y < -1.0f || y > (float)H || x < -1.0f || x > (float)W) return;
  if (y <= 0.f) y = 0.f;
  if (x <= 0.f) x = 0.f;
  int y_low = (int)y, x_low = (int)x, y_high, x_high;
  if (y_low >= H - 1) { y_high = y_low = H - 1; y = (float)y_low; } else { y_high = y_low + 1; }
  if (x_low >= W - 1) { x_high = x_low = W - 1; x = (float)x_low; } else { x_high = x_low + 1; }
  const float ly = y - (float)y_low, lx = x - (float)x_low;
  const float hy = 1.f - ly, hx = 1.f - lx;
  const float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
  float lt[V], rt[V], lb[V], rb[V];
  vps::ldv<T, V>(f.p + f.off(b, y_low, x_low) + c, lt);
  vps::ldv<T, V>(f.p + f.off(b, y_low, x_high) + c, rt);
  vps::ldv<T, V>(f.p + f.off(b, y_high, x_low) + c, lb);
  vps::ldv<T, V>(f.p + f.off(b, y_high, x_high) + c, rb);
#pragma unroll
  for (int j = 0; j < V; ++j) acc[j] += w1 * lt[j] + w2 * rt[j] + w3 * lb[j] + w4 * rb[j];
}

// ROIAlignForward (roi_align_kernel.cu:64-128) + map_roi_levels (single_level.py:54-73), one launch for all levels.
// grid: (pw * channel-chunks, ph, roi)
template <typename T, int V>
__global__ void roi_align_kernel(Feats<T> fs, const float* __restrict__ rois, int nroi, const int* __restrict__ nroi_dev,
                                 vps::TV<T> out, int ps, int sample_num) {
  VPS_PIX_COORDS(out, V, c, pw, ph, r);
  const int nvalid = nroi_dev ? min(*nroi_dev, nroi) : nroi;
  T* op = out.p + out.off(r, ph, pw) + c;
  float acc[V];
#pragma unroll
  for (int j = 0; j < V; ++j) acc[j] = 0.f;
  if (r < nvalid) {
    const float* roi = rois + (int64_t)r * 5;
    const int b = (int)roi[0];
    const float x1 = roi[1], y1 = roi[2], x2 = roi[3], y2 = roi[4];
    const float sc = sqrtf((x2 - x1 + 1.f) * (y2 - y1 + 1.f));
    int lvl = (int)floorf(log2f(sc / 56.f + 1e-6f));
    lvl = max(0, min(lvl, fs.n - 1));
    const float ss = fs.scale[lvl];
    const float rsw = x1 * ss, rsh = y1 * ss, rew = (x2 + 1.f) * ss, reh = (y2 + 1.f) * ss;
    const float rw = fmaxf(rew - rsw, 0.f), rh = fmaxf(reh - rsh, 0.f);
    const float bh = rh / (float)ps, bw = rw / (float)ps;
    for (int iy = 0; iy < sample_num; ++iy) {
      const float y = rsh + (float)ph * bh + ((float)iy + 0.5f) * bh / (float)sample_num;
      for (int ix = 0; ix < sample_num; ++ix) {
        const float x = rsw + (float)pw * bw + ((float)ix + 0.5f) * bw / (float)sample_num;
        // level is warp-divergent at most across RoIs (blockIdx.z), never inside a block
        switch (lvl) {
          case 0: bilinear_legacy_acc<T, V>(fs.l[0], b, c, y, x, acc); break;
          case 1: bilinear_legacy_acc<T, V>(fs.l[1], b, c, y, x, acc); break;
          case 2: bilinear_legacy_acc<T, V>(fs.l[2], b, c, y, x, acc); break;
          default: bilinear_legacy_acc<T, V>(fs.l[3], b, c, y, x, acc); break;
        }
      }
    }
#pragma unroll
    for (int j = 0; j < V; ++j) acc[j] /= (float)(sample_num * sample_num);
  }
  vps::stv<T, V>(op, acc);
}

// ------------------------------------------------------------------ RPN decode (rpn_head.py:73-85, transforms.py:34-68)
template <typename T>
__global__ void rpn_decode_kernel(const float* __restrict__ scores_sorted, const int32_t* __restrict__ idx_sorted, int k,
                                  vps::TV<const T> deltas, int feat_w, int stride, const float* __restrict__ base,
                                  int A, float img_h, float img_w, float* __restrict__ dets) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k) return;
  const int idx = idx_sorted[i];
  const int a = idx % A, pix = idx / A;
  const int x = pix % feat_w, y = pix / feat_w;
  const float ax1 = base[a * 4 + 0] + (float)(x * stride), ay1 = base[a * 4 + 1] + (float)(y * stride);
  const float ax2 = base[a * 4 + 2] + (float)(x * stride), ay2 = base[a * 4 + 3] + (float)(y * stride);
  const T* dp = deltas.p + deltas.off(0, y, x) + a * 4;
  const float dx = vps::ldf<T>(dp), dy = vps::ldf<T>(dp + 1);
  float dw = vps::ldf<T>(dp + 2), dh = vps::ldf<T>(dp + 3);
  const float max_ratio = 4.135166556742356f;  // |log(16/1000)|
  dw = fminf(fmaxf(dw, -max_ratio), max_ratio);
  dh = fminf(fmaxf(dh, -max_ratio), max_ratio);
  const float px = (ax1 + ax2) * 0.5f, py = (ay1 + ay2) * 0.5f;
  const float pw = ax2 - ax1 + 1.0f, ph = ay2 - ay1 + 1.0f;
  const float gw = pw * expf(dw), gh = ph * expf(dh);
  const float gx = px + pw * dx, gy = py + ph * dy;
  float bx1 = gx - gw * 0.5f + 0.5f, by1 = gy - gh * 0.5f + 0.5f;
  float bx2 = gx + gw * 0.5f - 0.5f, by2 = gy + gh * 0.5f - 0.5f;
  bx1 = fminf(fmaxf(bx1, 0.f), img_w - 1.f);
  by1 = fminf(fmaxf(by1, 0.f), img_h - 1.f);
  bx2 = fminf(fmaxf(bx2, 0.f), img_w - 1.f);
  by2 = fminf(fmaxf(by2, 0.f), img_h - 1.f);
  float* o = dets + (int64_t)i * 5;
  o[0] = bx1; o[1] = by1; o[2] = bx2; o[3] = by2; o[4] = scores_sorted[i];
}

// ------------------------------------------------------------------ NMS (nms_kernel.cu:13-131)
__device__ __forceinline__ float dev_iou(const float* a, const float* b) {
  const float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
  const float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
  const float width = fmaxf(right - left + 1.f, 0.f), height = fmaxf(bottom - top + 1.f, 0.f);
  const float inter = width * height;
  const float sa = (a[2] - a[0] + 1.f) * (a[3] - a[1] + 1.f);
  const float sb = (b[2] - b[0] + 1.f) * (b[3] - b[1] + 1.f);
  return inter / (sa + sb - inter);
}

// nb independent problems per launch (the RPN levels): problem b = rows [b*seg, b*seg + n_b) of dets
struct NmsBatch {
  int n[8];
};
__device__ __forceinline__ int nms_count(const NmsBatch& nb, const int* __restrict__ n_dev, int b) {
  return n_dev ? min(n_dev[b], nb.n[b]) : nb.n[b];
}

__global__ void nms_mask_kernel(NmsBatch nb, int seg, const int* __restrict__ n_dev, float thr, const float* __restrict__ boxes_all,
                                unsigned long long* __restrict__ mask_all, int col_blocks) {
  const int b = blockIdx.z;
  const int n = nms_count(nb, n_dev, b);
  const float* boxes = boxes_all + (int64_t)b * seg * 5;
  unsigned long long* mask = mask_all + (int64_t)b * seg * col_blocks;
  const int row_start = blockIdx.y, col_start = blockIdx.x;
  if (row_start * 64 >= n || col_start * 64 >= n) return;
  const int row_size = min(n - row_start * 64, 64), col_size = min(n - col_start * 64, 64);
  __shared__ float bb[64 * 5];
  if (threadIdx.x < col_size) {
    for (int j = 0; j < 5; ++j) bb[threadIdx.x * 5 + j] = boxes[(int64_t)(64 * col_start + threadIdx.x) * 5 + j];
  }
  __syncthreads();
  if (threadIdx.x < row_size) {
    const int cur = 64 * row_start + threadIdx.x;
    const float* cb = boxes + (int64_t)cur * 5;
    unsigned long long t = 0;
    const int start = (row_start == col_start) ? threadIdx.x + 1 : 0;
    for (int i = start; i < col_size; ++i)
      if (dev_iou(cb, bb + i * 5) > thr) t |= 1ULL << i;
    mask[(int64_t)cur * col_blocks + col_start] = t;
  }
}

// The host greedy loop of the reference (nms_kernel.cu:104-123) as a device pass, one block per problem: no D2H.
// The suppression words live in shared memory.  Per chunk of 64 boxes: (1) the 64 diagonal mask words are fetched in
// parallel, (2) one thread resolves the intra-chunk greedy order (the only serial part), (3) 8 x 128 threads OR the
// rows of the boxes kept in this chunk into the remaining words -- independent loads, one L2 round trip per chunk.
__global__ void __launch_bounds__(1024) nms_reduce_kernel(NmsBatch nb, int seg, const int* __restrict__ n_dev,
                                                          const unsigned long long* __restrict__ mask_all, int col_blocks,
                                                          int32_t* __restrict__ keep_all, int* __restrict__ nkeep) {
  __shared__ unsigned long long s_remv[128], diag[64];
  __shared__ int s_rows[64];
  __shared__ int s_nk, s_num;
  const int b = blockIdx.x;
  const int n = nms_count(nb, n_dev, b);
  const unsigned long long* mask = mask_all + (int64_t)b * seg * col_blocks;
  int32_t* keep = keep_all + (int64_t)b * seg;
  const int cb = (n + 63) / 64;
  const int tid = threadIdx.x;
  if (tid < 128) s_remv[tid] = 0ULL;
  if (tid == 0) s_num = 0;
  __syncthreads();
  for (int c = 0; c < cb; ++c) {
    if (tid < 64) {
      const int i = c * 64 + tid;
      diag[tid] = (i < n) ? mask[(int64_t)i * col_blocks + c] : 0ULL;
    }
    __syncthreads();
    if (tid == 0) {
      unsigned long long cur = s_remv[c];
      const int lim = min(64, n - c * 64);
      int num = s_num, nk = 0;
      for (int i = 0; i < lim; ++i) {
        if (!((cur >> i) & 1ULL)) {
          cur |= diag[i];
          keep[num++] = c * 64 + i;
          s_rows[nk++] = c * 64 + i;
        }
      }
      s_nk = nk;
      s_num = num;
    }
    __syncthreads();
    {
      const int j = tid & 127, r = tid >> 7;
      if (j > c && j < cb) {
        const int nk = s_nk;
        unsigned long long acc = 0ULL;
#pragma unroll 8
        for (int q = r; q < nk; q += 8) acc |= mask[(int64_t)s_rows[q] * col_blocks + j];
        if (acc) atomicOr(&s_remv[j], acc);
      }
    }
    __syncthreads();
  }
  if (tid == 0) nkeep[b] = s_num;
}

__global__ void gather_rows_kernel(const float* __restrict__ src, const int32_t* __restrict__ idx, int n_cap,
                                   const int* __restrict__ n_dev, int width, float* __restrict__ dst) {
  const int n = n_dev ? min(*n_dev, n_cap) : n_cap;
  const int64_t total = (int64_t)n_cap * width;
  VPS_GRID_STRIDE(i, total) {
    const int r = (int)(i / width), c = (int)(i % width);
    dst[i] = r < n ? src[(int64_t)idx[r] * width + c] : 0.f;
  }
}

__global__ void iota_kernel(int32_t* p, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = i;
}

// ------------------------------------------------------------------ MaskROI candidates (mask_roi.py:37-93)
__global__ void maskroi_candidates_kernel(const float* __restrict__ rois, const float* __restrict__ cls_score,
                                          const float* __restrict__ bbox_pred, int row_stride, int nroi,
                                          const int* __restrict__ nroi_dev,
                                          int num_classes, float thr, float img_h, float img_w, float* __restrict__ cand,
                                          int32_t* __restrict__ cand_cls, float* __restrict__ cand_prob,
                                          int* __restrict__ ncand) {
  const int nvalid = nroi_dev ? min(*nroi_dev, nroi) : nroi;
  const int nfg = num_classes - 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nroi * nfg) return;
  const int r = i / nfg, c = i % nfg + 1;
  float prob = -1.f;
  float bx[4] = {0.f, 0.f, 0.f, 0.f};
  if (r < nvalid) {
    const float* s = cls_score + (int64_t)r * row_stride;
    float m = s[0];
    for (int j = 1; j < num_classes; ++j) m = fmaxf(m, s[j]);
    float sum = 0.f;
    for (int j = 0; j < num_classes; ++j) sum += expf(s[j] - m);
    const float p = expf(s[c] - m) / sum;
    // upsnet bbox_transform (bbox_transform.py:290-330), weights (10,10,5,5), then clip_boxes (:45-60)
    const float* b = rois + (int64_t)r * 5 + 1;
    const float* d = bbox_pred + (int64_t)r * row_stride + c * 4;
    const float w = b[2] - b[0] + 1.0f, h = b[3] - b[1] + 1.0f;
    const float cx = b[0] + 0.5f * w, cy = b[1] + 0.5f * h;
    const float dx = d[0] / 10.0f, dy = d[1] / 10.0f;
    const float lim = 4.135166556742356f;  // log(1000/16)
    const float dw = fminf(d[2] / 5.0f, lim), dh = fminf(d[3] / 5.0f, lim);
    const float pcx = dx * w + cx, pcy = dy * h + cy;
    const float pw = expf(dw) * w, ph = expf(dh) * h;
    bx[0] = fmaxf(fminf(pcx - 0.5f * pw, img_w - 1.f), 0.f);
    bx[1] = fmaxf(fminf(pcy - 0.5f * ph, img_h - 1.f), 0.f);
    bx[2] = fmaxf(fminf(pcx + 0.5f * pw - 1.f, img_w - 1.f), 0.f);
    bx[3] = fmaxf(fminf(pcy + 0.5f * ph - 1.f, img_h - 1.f), 0.f);
    if (p > thr) { prob = p; atomicAdd(ncand, 1); }
  }
  float* o = cand + (int64_t)i * 5;
  o[0] = bx[0]; o[1] = bx[1]; o[2] = bx[2]; o[3] = bx[3]; o[4] = prob;
  cand_cls[i] = c;
  cand_prob[i] = prob;
}

// ------------------------------------------------------------------ tracker
// dots[i][j] = <emb_i, ref_j>.  The bits are those of one warp per pair: lane l runs an fmaf chain from 0 over the columns
// c = l (mod 32) in increasing c, then the xor butterfly s += shfl_xor(s, o) for o = 16, 8, 4, 2, 1 (lane 0's value; the
// comp scores of the tracker, and so its ids, depend on these bits).
//
// Tiling: a block owns TD_BI detections x TD_BJ memory slots (blockIdx.x = slot tile * detection tiles + detection tile,
// so the blocks that read the same memory rows run together and each row comes from DRAM about once), stages the rows
// through shared memory TD_CK columns at a time (cp.async, double-buffered), and each warp keeps a TD_TI x TD_TJ
// register tile of pairs: lane l holds the partial sums of column class l of all 64 pairs.  The butterfly then runs as
// a reduce-scatter: step o exchanges half of the sums a lane holds with lane l ^ o and adds, so every pair goes through
// the same additions as above (IEEE addition commutes), and lane l ends with pairs 2l and 2l + 1.
constexpr int TD_TI = 8, TD_TJ = 8;              // register tile of a warp: detections x slots
constexpr int TD_WI = 2, TD_WJ = 4;              // warps of a block: detections x slots
constexpr int TD_BI = TD_TI * TD_WI, TD_BJ = TD_TJ * TD_WJ, TD_CK = 128, TD_THREADS = 32 * TD_WI * TD_WJ;
static_assert((TD_BI + TD_BJ) * TD_CK % TD_THREADS == 0 && 2 * (TD_BI + TD_BJ) * TD_CK * 4 <= 48 * 1024, "staging");
static_assert(TD_TI * TD_TJ == 64, "the reduce-scatter below leaves 2 of 64 pairs per lane");

// one butterfly step over the first H sums of v: keep one half (by lane bit O), add the partner's sums of that half
template <int O, int H>
__device__ __forceinline__ void dot_scatter_step(float (&v)[TD_TI * TD_TJ], int lane) {
  const bool up = (lane & O) != 0;
#pragma unroll
  for (int r = 0; r < H / 2; ++r) {
    const float send = up ? v[r] : v[r + H / 2];
    const float keep = up ? v[r + H / 2] : v[r];
    v[r] = keep + __shfl_xor_sync(0xffffffffu, send, O);
  }
}

// 4-byte asynchronous global -> shared copy; src_bytes 0 stores a zero (rows past k / m, columns past dim)
__device__ __forceinline__ void cp_async4(float* dst, const float* src, int src_bytes) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(src), "r"(src_bytes) : "memory");
}

__global__ void __launch_bounds__(TD_THREADS, 2)
track_dot_kernel(const float* __restrict__ emb, const float* __restrict__ ref, int k, int m, int dim,
                 float* __restrict__ dots) {
  // two stages of TD_CK columns: detection rows [0, TD_BI), memory rows [TD_BI, TD_BI + TD_BJ); the copy of the next
  // chunk runs while the warps multiply the current one
  __shared__ float st[2][TD_BI + TD_BJ][TD_CK];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int wi = warp / TD_WJ, wj = warp % TD_WJ;
  const int ntile_i = (k + TD_BI - 1) / TD_BI;
  const int i0 = (int)(blockIdx.x % ntile_i) * TD_BI;
  const int64_t j0 = (int64_t)(blockIdx.x / ntile_i) * TD_BJ;
  auto stage = [&](int buf, int c0) {
#pragma unroll 1
    for (int it = 0; it < (TD_BI + TD_BJ) * TD_CK / TD_THREADS; ++it) {
      const int e = it * TD_THREADS + threadIdx.x;
      const int r = e / TD_CK, c = e % TD_CK;
      const float* src = emb;
      bool ok = c0 + c < dim;
      if (r < TD_BI) {
        ok = ok && i0 + r < k;
        if (ok) src = emb + (int64_t)(i0 + r) * dim + c0 + c;
      } else {
        const int64_t j = j0 + r - TD_BI;
        ok = ok && j < m;
        if (ok) src = ref + j * dim + c0 + c;
      }
      // a staged zero leaves the chain unchanged: fmaf(0, 0, s) == s for every s the chain can hold (never -0)
      cp_async4(&st[buf][r][c], src, ok ? 4 : 0);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  float acc[TD_TI * TD_TJ];
#pragma unroll
  for (int q = 0; q < TD_TI * TD_TJ; ++q) acc[q] = 0.f;
  stage(0, 0);
  for (int c0 = 0, buf = 0; c0 < dim; c0 += TD_CK, buf ^= 1) {
    if (c0 + TD_CK < dim) {
      stage(buf ^ 1, c0 + TD_CK);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();                                   // chunk c0 is in st[buf] for every thread
#pragma unroll
    for (int t = 0; t < TD_CK / 32; ++t) {           // columns c0 + 32 t + lane: increasing c per lane
      float a[TD_TI], b[TD_TJ];
#pragma unroll
      for (int ti = 0; ti < TD_TI; ++ti) a[ti] = st[buf][wi * TD_TI + ti][t * 32 + lane];
#pragma unroll
      for (int tj = 0; tj < TD_TJ; ++tj) b[tj] = st[buf][TD_BI + wj * TD_TJ + tj][t * 32 + lane];
#pragma unroll
      for (int ti = 0; ti < TD_TI; ++ti)
#pragma unroll
        for (int tj = 0; tj < TD_TJ; ++tj) acc[ti * TD_TJ + tj] = fmaf(a[ti], b[tj], acc[ti * TD_TJ + tj]);
    }
    __syncthreads();                                   // st[buf] is read before the copy two chunks on refills it
  }
  dot_scatter_step<16, 64>(acc, lane);
  dot_scatter_step<8, 32>(acc, lane);
  dot_scatter_step<4, 16>(acc, lane);
  dot_scatter_step<2, 8>(acc, lane);
  dot_scatter_step<1, 4>(acc, lane);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = 2 * lane + r;
    const int i = i0 + wi * TD_TI + q / TD_TJ;
    const int64_t j = j0 + wj * TD_TJ + q % TD_TJ;
    if (i < k && j < m) dots[(int64_t)i * m + j] = acc[r];
  }
}

// comp scores + row argmax (track_head.py:73-91, panoptic_fusetrack.py:412-424); one warp per detection
__global__ void track_score_kernel(const float* __restrict__ dots, int k, int m, const float* __restrict__ det_boxes,
                                   const float* __restrict__ ref_boxes, const int32_t* __restrict__ det_labels,
                                   const int32_t* __restrict__ ref_labels, const float* __restrict__ cls_prob, float c0,
                                   float c1, float c2, float* __restrict__ comp, int32_t* __restrict__ match_ids,
                                   float* __restrict__ match_like) {
  const int lane = threadIdx.x & 31;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= k) return;
  const float* d = dots + (int64_t)i * m;
  // log_softmax over [0 | dots]
  float mx = 0.f;
  for (int j = lane; j < m; j += 32) mx = fmaxf(mx, d[j]);
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = (lane == 0) ? expf(0.f - mx) : 0.f;
  for (int j = lane; j < m; j += 32) sum += expf(d[j] - mx);
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float lse = mx + logf(sum);
  const float lp = c0 * logf(cls_prob[i]);
  const float* a = det_boxes + (int64_t)i * 4;
  float best = -INFINITY;
  int besti = 0x7fffffff;
  for (int j = lane; j <= m; j += 32) {
    float v;
    if (j == 0) {
      v = (0.f - lse) + lp + c1 * 0.f + c2 * 1.f;
    } else {
      const float* b = ref_boxes + (int64_t)(j - 1) * 4;
      const float ltx = fmaxf(a[0], b[0]), lty = fmaxf(a[1], b[1]);
      const float rbx = fminf(a[2], b[2]), rby = fminf(a[3], b[3]);
      const float w = fmaxf(rbx - ltx + 1.f, 0.f), h = fmaxf(rby - lty + 1.f, 0.f);
      const float ov = w * h;
      const float a1 = (a[2] - a[0] + 1.f) * (a[3] - a[1] + 1.f), a2 = (b[2] - b[0] + 1.f) * (b[3] - b[1] + 1.f);
      const float iou = ov / (a1 + a2 - ov);
      const float ld = (ref_labels[j - 1] == det_labels[i]) ? 1.f : 0.f;
      v = (d[j - 1] - lse) + lp + c1 * iou + c2 * ld;
    }
    comp[(int64_t)i * (m + 1) + j] = v;
    if (v > best) { best = v; besti = j; }   // ascending j per lane => first max per lane
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
    if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
  }
  if (lane == 0) { match_ids[i] = besti; match_like[i] = best; }
}

// state of the id-assignment loop: no slot written, no best match per memory slot yet
__global__ void track_assign_init_kernel(int m, int cap, int32_t* __restrict__ mem_src, float* __restrict__ best_scores,
                                         int32_t* __restrict__ best_ids) {
  VPS_GRID_STRIDE(j, cap) {
    mem_src[j] = -1;
    if (j < m) { best_scores[j] = -100.f; best_ids[j] = -1; }
  }
}

// the sequential id-assignment loop (panoptic_fusetrack.py:430-469) on one thread, O(k).
// mem_src[slot] = index of the detection whose features/box end up in memory slot `slot` (-1: unchanged).
__global__ void track_assign_kernel(const int32_t* __restrict__ match_ids, const float* __restrict__ match_like, int k,
                                    int m, int cap, int32_t* __restrict__ det_obj_ids, int32_t* __restrict__ mem_src,
                                    float* __restrict__ best_scores, int32_t* __restrict__ best_ids, int* __restrict__ new_m) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int cur = m;
  for (int i = 0; i < k; ++i) det_obj_ids[i] = -1;
  for (int i = 0; i < k; ++i) {
    const int mid = match_ids[i];
    if (mid == 0) {
      if (cur < cap) { det_obj_ids[i] = cur; mem_src[cur] = i; cur++; }
    } else {
      const int obj = mid - 1;
      const float sc = match_like[i];
      if (sc > best_scores[obj]) {
        det_obj_ids[i] = obj;
        if (best_ids[obj] >= 0) det_obj_ids[best_ids[obj]] = -1;
        best_scores[obj] = sc;
        best_ids[obj] = i;
        mem_src[obj] = i;
      }
    }
  }
  for (int i = 0; i < k; ++i) {
    if (det_obj_ids[i] >= 0) continue;
    if (cur < cap) { det_obj_ids[i] = cur; mem_src[cur] = i; cur++; }
  }
  *new_m = cur;
}


// ------------------------------------------------------------------ small glue kernels (device-side bookkeeping)
// RPN: concatenated per-level kept proposals -> final stable top-k (rpn_head.py:94-103).  dets_cat holds
// nlev segments of `seg` rows; segment l has counts[l] valid rows.  Writes compact scores for sorting.
__global__ void rpn_concat_scores_kernel(const float* __restrict__ dets_cat, const int* __restrict__ counts, int nlev,
                                         int seg, float* __restrict__ scores, int* __restrict__ total, int cap) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {
    int t = 0;
    for (int l = 0; l < nlev; ++l) t += min(counts[l], seg);
    *total = min(t, cap);
  }
  if (i >= nlev * seg) return;
  const int l = i / seg, r = i % seg;
  scores[i] = (r < min(counts[l], seg)) ? dets_cat[(int64_t)i * 5 + 4] : -1.0f;   // sigmoid scores are > 0
}
__global__ void rpn_finalize_kernel(const float* __restrict__ dets_cat, const int32_t* __restrict__ idx_sorted,
                                    const int* __restrict__ total, int cap, float* __restrict__ proposals,
                                    float* __restrict__ rois) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap) return;
  float v[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
  if (i < *total) {
    const float* s = dets_cat + (int64_t)idx_sorted[i] * 5;
    for (int j = 0; j < 5; ++j) v[j] = s[j];
  }
  for (int j = 0; j < 5; ++j) proposals[(int64_t)i * 5 + j] = v[j];
  rois[(int64_t)i * 5] = 0.f;   // bbox2roi batch index (transforms.py:106-125)
  for (int j = 0; j < 4; ++j) rois[(int64_t)i * 5 + 1 + j] = v[j];
}

// MaskROI tail (mask_roi.py:95-147): NMS survivors (score order) -> max_det rule (keep scores >= the
// max_det-th best) -> det_rois [cap,5] (batch 0), cls_idx, cls_prob; dummy result when nothing survives.
__global__ void maskroi_finalize_kernel(const float* __restrict__ cand_sorted, const int32_t* __restrict__ slot_sorted,
                                        const int32_t* __restrict__ cand_cls, const int32_t* __restrict__ keep,
                                        const int* __restrict__ nkeep, int max_det, int cap, float* __restrict__ det_rois,
                                        int32_t* __restrict__ cls_idx, float* __restrict__ cls_prob, int* __restrict__ kout) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int n = *nkeep;
  if (max_det > 0 && n > max_det) {
    const float thresh = cand_sorted[(int64_t)keep[max_det - 1] * 5 + 4];
    int m = max_det;
    while (m < n && cand_sorted[(int64_t)keep[m] * 5 + 4] >= thresh) ++m;
    n = m;
  }
  if (n > cap) n = cap;
  for (int i = 0; i < cap; ++i) {
    float* r = det_rois + (int64_t)i * 5;
    if (i < n) {
      const float* c = cand_sorted + (int64_t)keep[i] * 5;
      r[0] = 0.f; r[1] = c[0]; r[2] = c[1]; r[3] = c[2]; r[4] = c[3];
      cls_prob[i] = c[4];
      cls_idx[i] = cand_cls[slot_sorted[keep[i]]];
    } else {
      r[0] = r[1] = r[2] = r[3] = r[4] = 0.f;
      cls_prob[i] = 0.f; cls_idx[i] = 0;
    }
  }
  if (n == 0) {            // dummy detection (mask_roi.py:136-142): score 1, zero box, class 0
    cls_prob[0] = 1.f; cls_idx[0] = 0;
    kout[0] = 1; kout[1] = 1;
  } else {
    kout[0] = n; kout[1] = 0;
  }
}

// mask_score.gather(1, cls_idx) (panoptic_fusetrack.py:566-568): pick the class channel of each RoI's 28x28x9 logits
template <typename T>
__global__ void select_class_kernel(vps::TV<const T> logits, const int32_t* __restrict__ cls_idx, int k,
                                    float* __restrict__ out) {
  const int64_t per = (int64_t)logits.h * logits.w;
  const int64_t total = (int64_t)k * per;
  VPS_GRID_STRIDE(i, total) {
    const int r = (int)(i / per);
    const int64_t pix = i % per;
    out[i] = vps::ldf<T>(logits.p + ((int64_t)r * per + pix) * logits.cs + cls_idx[r]);
  }
}

// tracker memory update (panoptic_fusetrack.py:441-443,458-459,467-469): slot j <- detection mem_src[j].
// Block b owns the slots j = b (mod gridDim.x): it reads their mem_src entries TU_THREADS at a time, lists the written
// ones in shared memory and copies each listed row with all its threads, so the work is one scan of mem_src[0, new_m)
// plus the written rows, and consecutive written slots (the appended ones) go to different blocks.
constexpr int TU_THREADS = 256, TU_BLOCKS = 512;
template <typename T>
__global__ void __launch_bounds__(TU_THREADS)
track_update_kernel(T* __restrict__ mem_feats, const T* __restrict__ det_feats, int64_t feat_len,
                    float* __restrict__ mem_boxes, const float* __restrict__ det_boxes, int32_t* __restrict__ mem_labels,
                    const int32_t* __restrict__ det_labels, const int32_t* __restrict__ mem_src, int old_m,
                    const int* __restrict__ new_m_dev) {
  __shared__ int64_t slot[TU_THREADS];
  __shared__ int src[TU_THREADS];
  __shared__ int nlist;
  const int64_t n = *new_m_dev;
  for (int64_t s0 = 0; blockIdx.x + s0 * gridDim.x < n; s0 += TU_THREADS) {
    if (threadIdx.x == 0) nlist = 0;
    __syncthreads();
    const int64_t j = blockIdx.x + (s0 + threadIdx.x) * gridDim.x;
    const int s = j < n ? mem_src[j] : -1;
    if (s >= 0) {
      const int p = atomicAdd(&nlist, 1);
      slot[p] = j;
      src[p] = s;
    }
    __syncthreads();
    for (int q = 0; q < nlist; ++q) {
      const int64_t jj = slot[q], ss = src[q];
      for (int64_t i = threadIdx.x; i < feat_len; i += TU_THREADS) mem_feats[jj * feat_len + i] = det_feats[ss * feat_len + i];
      if (mem_boxes != nullptr && threadIdx.x < 4) mem_boxes[jj * 4 + threadIdx.x] = det_boxes[ss * 4 + threadIdx.x];
      if (mem_labels != nullptr && threadIdx.x == 0 && jj >= old_m) mem_labels[jj] = det_labels[ss];
    }
    __syncthreads();                                   // the list is read before the next round resets it
  }
}


// det_bboxes = roi2bbox(det_rois) (transforms.py:128-135), det_labels = cls_idx - 1 (panoptic_fusetrack.py:386)
__global__ void det_split_kernel(const float* __restrict__ det_rois, const int32_t* __restrict__ cls_idx, int cap,
                                 float* __restrict__ boxes, int32_t* __restrict__ labels) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap) return;
  for (int j = 0; j < 4; ++j) boxes[i * 4 + j] = det_rois[i * 5 + 1 + j];
  labels[i] = cls_idx[i] - 1;
}

}  // namespace

extern "C" int vps_roi_align(const vps_tensor* feats, const int* strides, int nlev, const float* rois, int nroi,
                             const int* nroi_dev, const vps_tensor* out, int sample_num, void* stream) {
  VPS_CHECK_ARG(nlev >= 1 && nlev <= MAXLEV && out->h == out->w && out->n >= nroi, "roi_align: args");
  if (!((int64_t)nroi * out->h * out->w * out->c)) return VPS_OK;
  bool vec = vps::vec_ok(*out, out->c);
  for (int i = 0; i < nlev; ++i) {
    VPS_CHECK_ARG(feats[i].dtype == out->dtype && feats[i].c >= out->c, "roi_align: level %d dtype/channels", i);
    vec = vec && vps::vec_ok(feats[i], out->c);
  }
  VPS_DISPATCH_V(out->dtype, vec, T, V, {
    Feats<T> fs;
    fs.n = nlev;
    for (int i = 0; i < nlev; ++i) { fs.l[i] = vps::tv<const T>(feats[i]); fs.scale[i] = 1.0f / (float)strides[i]; }
    for (int i = nlev; i < MAXLEV; ++i) { fs.l[i] = fs.l[nlev - 1]; fs.scale[i] = fs.scale[nlev - 1]; }
    roi_align_kernel<T, V><<<vps::pix_grid(out->w, out->c / V, out->h, nroi, 128), 128, 0, (cudaStream_t)stream>>>(
        fs, rois, nroi, nroi_dev, vps::tv<T>(*out), out->h, sample_num);
  });
  VPS_CUDA_LAST("roi_align");
  return VPS_OK;
}

extern "C" int vps_sort_desc(const float* keys, float* keys_out, int32_t* idx_out, int n, void* ws, int64_t ws_bytes,
                             void* stream) {
  if (n <= 0) return VPS_OK;
  cudaStream_t st = (cudaStream_t)stream;
  size_t need = 0;
  cub::DeviceRadixSort::SortPairsDescending(nullptr, need, keys, keys_out, (const int32_t*)nullptr, idx_out, n, 0, 32, st);
  const int64_t iota_bytes = ((int64_t)n * 4 + 255) / 256 * 256;
  VPS_CHECK_ARG(ws_bytes >= (int64_t)need + iota_bytes, "sort_desc: workspace %lld < %lld", (long long)ws_bytes,
                (long long)(need + iota_bytes));
  int32_t* iota = (int32_t*)ws;
  iota_kernel<<<vps::cdiv(n, 256), 256, 0, st>>>(iota, n);
  VPS_CUDA_LAST("iota");
  cudaError_t e = cub::DeviceRadixSort::SortPairsDescending((char*)ws + iota_bytes, need, keys, keys_out, iota, idx_out, n,
                                                            0, 32, st);
  if (e != cudaSuccess) { vps::set_error("sort_desc: %s", cudaGetErrorString(e)); return VPS_E_CUDA; }
  vps::count_launch(3);
  return VPS_OK;
}

extern "C" int vps_rpn_decode(const float* scores_sorted, const int32_t* idx_sorted, int k, const vps_tensor* deltas,
                              int feat_h, int feat_w, int stride, const float* base_anchors, int num_anchors, float img_h,
                              float img_w, float* dets, void* stream) {
  if (k <= 0) return VPS_OK;
  VPS_CHECK_ARG(deltas->h == feat_h && deltas->w == feat_w && deltas->c >= 4 * num_anchors, "rpn_decode: deltas shape");
  VPS_DISPATCH_T(deltas->dtype, T, (rpn_decode_kernel<T><<<vps::cdiv(k, 128), 128, 0, (cudaStream_t)stream>>>(
                                       scores_sorted, idx_sorted, k, vps::tv<const T>(*deltas), feat_w, stride,
                                       base_anchors, num_anchors, img_h, img_w, dets)));
  VPS_CUDA_LAST("rpn_decode");
  return VPS_OK;
}

extern "C" int vps_nms_batch(const float* dets, int nb, int seg, const int* ns, const int* n_dev, float thr,
                             int32_t* keep_idx, int* nkeep, void* ws, int64_t ws_bytes, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  VPS_CHECK_ARG(nb >= 1 && nb <= 8 && seg >= 0, "nms_batch: nb %d (max 8)", nb);
  NmsBatch b;
  int nmax = 0;
  for (int i = 0; i < 8; ++i) {
    b.n[i] = i < nb ? ns[i] : 0;
    VPS_CHECK_ARG(b.n[i] >= 0 && b.n[i] <= seg, "nms_batch: n[%d] = %d exceeds the segment %d", i, b.n[i], seg);
    if (b.n[i] > nmax) nmax = b.n[i];
  }
  if (nmax <= 0) { cudaMemsetAsync(nkeep, 0, sizeof(int) * nb, st); return VPS_OK; }
  const int col_blocks = (nmax + 63) / 64;
  VPS_CHECK_ARG(ws_bytes >= (int64_t)nb * seg * col_blocks * 8, "nms: workspace too small");
  VPS_CHECK_ARG(col_blocks <= 128, "nms: n %d too large (max 8192)", nmax);
  dim3 grid(col_blocks, col_blocks, nb);
  nms_mask_kernel<<<grid, 64, 0, st>>>(b, seg, n_dev, thr, dets, (unsigned long long*)ws, col_blocks);
  VPS_CUDA_LAST("nms_mask");
  nms_reduce_kernel<<<nb, 1024, 0, st>>>(b, seg, n_dev, (const unsigned long long*)ws, col_blocks, keep_idx, nkeep);
  VPS_CUDA_LAST("nms_reduce");
  return VPS_OK;
}

extern "C" int vps_nms(const float* dets, int n, const int* n_dev, float thr, int32_t* keep_idx, int* nkeep, void* ws,
                       int64_t ws_bytes, void* stream) {
  return vps_nms_batch(dets, 1, n, &n, n_dev, thr, keep_idx, nkeep, ws, ws_bytes, stream);
}

extern "C" int vps_gather_rows(const float* src, const int32_t* idx, int n, const int* n_dev, int width, float* dst,
                               void* stream) {
  if (n <= 0) return VPS_OK;
  gather_rows_kernel<<<vps::grid_for((int64_t)n * width), 256, 0, (cudaStream_t)stream>>>(src, idx, n, n_dev, width, dst);
  VPS_CUDA_LAST("gather_rows");
  return VPS_OK;
}

extern "C" int vps_maskroi_candidates(const float* rois, const float* cls_score, const float* bbox_pred,
                                      int row_stride, int nroi, const int* nroi_dev, int num_classes, float score_thr, float img_h, float img_w,
                                      float* cand, int32_t* cand_cls, float* cand_prob, int* ncand, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(ncand, 0, sizeof(int), st);
  const int total = nroi * (num_classes - 1);
  if (total <= 0) return VPS_OK;
  maskroi_candidates_kernel<<<vps::cdiv(total, 128), 128, 0, st>>>(rois, cls_score, bbox_pred, row_stride, nroi, nroi_dev, num_classes,
                                                                 score_thr, img_h, img_w, cand, cand_cls, cand_prob, ncand);
  VPS_CUDA_LAST("maskroi_candidates");
  return VPS_OK;
}

// ws layout (floats/ints): dots[k*m] | match_like[k] | best_scores[cap] | best_ids[cap]
extern "C" int vps_track_assign(const float* emb, const float* ref_emb, int k, int m, int dim, const float* det_boxes,
                                const float* ref_boxes, const int32_t* det_labels, const int32_t* ref_labels,
                                const float* cls_prob, float c0, float c1, float c2, int cap, int32_t* det_obj_ids,
                                int32_t* match_ids, float* comp_scores, int32_t* mem_src, int* new_m, void* ws,
                                int64_t ws_bytes, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  VPS_CHECK_ARG(k >= 1 && m >= 1 && m <= cap, "track_assign: k %d m %d cap %d", k, m, cap);
  const int64_t need = ((int64_t)k * m + k + 2 * cap) * 4;
  VPS_CHECK_ARG(ws_bytes >= need, "track_assign: workspace %lld < %lld", (long long)ws_bytes, (long long)need);
  float* dots = (float*)ws;
  float* match_like = dots + (int64_t)k * m;
  float* best_scores = match_like + k;
  int32_t* best_ids = (int32_t*)(best_scores + cap);
  const int64_t dot_blocks = (int64_t)vps::cdiv(k, TD_BI) * vps::cdiv(m, TD_BJ);
  VPS_CHECK_ARG(dot_blocks <= 0x7fffffff, "track_assign: k %d x m %d exceeds one grid", k, m);
  track_dot_kernel<<<(unsigned)dot_blocks, TD_THREADS, 0, st>>>(emb, ref_emb, k, m, dim, dots);
  VPS_CUDA_LAST("track_dot");
  track_assign_init_kernel<<<vps::grid_for(cap), 256, 0, st>>>(m, cap, mem_src, best_scores, best_ids);
  VPS_CUDA_LAST("track_assign_init");
  track_score_kernel<<<vps::cdiv((int64_t)k * 32, 128), 128, 0, st>>>(dots, k, m, det_boxes, ref_boxes, det_labels,
                                                                     ref_labels, cls_prob, c0, c1, c2, comp_scores,
                                                                     match_ids, match_like);
  VPS_CUDA_LAST("track_score");
  track_assign_kernel<<<1, 32, 0, st>>>(match_ids, match_like, k, m, cap, det_obj_ids, mem_src, best_scores, best_ids, new_m);
  VPS_CUDA_LAST("track_assign");
  return VPS_OK;
}

extern "C" int vps_rpn_finalize(const float* dets_cat, const int* counts, int nlev, int seg, int cap, float* scores_ws,
                                float* scores_sorted_ws, int32_t* idx_sorted_ws, void* sort_ws, int64_t sort_ws_bytes,
                                float* proposals, float* rois, int* total, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int n = nlev * seg;
  rpn_concat_scores_kernel<<<vps::cdiv(n, 256), 256, 0, st>>>(dets_cat, counts, nlev, seg, scores_ws, total, cap);
  VPS_CUDA_LAST("rpn_concat_scores");
  int rc = vps_sort_desc(scores_ws, scores_sorted_ws, idx_sorted_ws, n, sort_ws, sort_ws_bytes, stream);
  if (rc != VPS_OK) return rc;
  rpn_finalize_kernel<<<vps::cdiv(cap, 128), 128, 0, st>>>(dets_cat, idx_sorted_ws, total, cap, proposals, rois);
  VPS_CUDA_LAST("rpn_finalize");
  return VPS_OK;
}

extern "C" int vps_maskroi_finalize(const float* cand_sorted, const int32_t* slot_sorted, const int32_t* cand_cls,
                                    const int32_t* keep, const int* nkeep, int max_det, int cap, float* det_rois,
                                    int32_t* cls_idx, float* cls_prob, int* kout, void* stream) {
  maskroi_finalize_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(cand_sorted, slot_sorted, cand_cls, keep, nkeep, max_det, cap,
                                                             det_rois, cls_idx, cls_prob, kout);
  VPS_CUDA_LAST("maskroi_finalize");
  return VPS_OK;
}

extern "C" int vps_select_class(const vps_tensor* logits, const int32_t* cls_idx, int k, float* out, void* stream) {
  if (k <= 0) return VPS_OK;
  VPS_CHECK_ARG(logits->n >= k, "select_class: k");
  const int64_t total = (int64_t)k * logits->h * logits->w;
  VPS_DISPATCH_T(logits->dtype, T, (select_class_kernel<T><<<vps::grid_for(total), 256, 0, (cudaStream_t)stream>>>(
                                       vps::tv<const T>(*logits), cls_idx, k, out)));
  VPS_CUDA_LAST("select_class");
  return VPS_OK;
}

extern "C" int vps_track_update(void* mem_feats, const void* det_feats, int dtype, int64_t feat_len, float* mem_boxes,
                                const float* det_boxes, int32_t* mem_labels, const int32_t* det_labels,
                                const int32_t* mem_src, int old_m, int cap, const int* new_m_dev, void* stream) {
  if (cap <= 0) return VPS_OK;
  VPS_DISPATCH_T(dtype, T, (track_update_kernel<T><<<TU_BLOCKS, TU_THREADS, 0, (cudaStream_t)stream>>>(
                               (T*)mem_feats, (const T*)det_feats, feat_len, mem_boxes, det_boxes, mem_labels, det_labels,
                               mem_src, old_m, new_m_dev)));
  VPS_CUDA_LAST("track_update");
  return VPS_OK;
}

extern "C" int vps_det_split(const float* det_rois, const int32_t* cls_idx, int cap, float* boxes, int32_t* labels,
                             void* stream) {
  if (cap <= 0) return VPS_OK;
  det_split_kernel<<<vps::cdiv(cap, 128), 128, 0, (cudaStream_t)stream>>>(det_rois, cls_idx, cap, boxes, labels);
  VPS_CUDA_LAST("det_split");
  return VPS_OK;
}
