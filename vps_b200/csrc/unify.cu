// SURVEY 8f rank 1: get_unified_pan_result (reference tools/dataset/cityscapes_vps.py:183-224) for one frame, and its
// image-level sibling (tools/dataset/base_dataset.py:232-274, vps_unify_pan_image).
//
// Everything the reference decides per REGION (= per panoptic id) depends only on two histograms: how many pixels each
// panoptic id has, and, per id, how the semantic map votes inside it.  So the frame is processed as
//   1. unify_hist_kernel   one pass over (seg, pan): per-block shared-memory histograms -> global  [HBM: 2 label maps in]
//   2. unify_decide_kernel one block: region rank, majority vote, stuff/thing decision, stuff-area filter
//                          -> a 256-entry look-up table  pan value -> (semantic, instance rank, track id)
//   3. unify_apply_kernel  out[pixel] = LUT[pan[pixel]]                                  [HBM: 1 map in, 3 channels out]
// Bit-exact with the reference's numpy (uint8 wrap-around included); no per-region passes, no host round trip.
#include <stddef.h>

#include "label_runs.cuh"

namespace {
constexpr int NID = 256;            // panoptic ids are uint8 in the reference (test_vpq.py:52-56)
constexpr int NCLS_FAST = 32;       // semantic classes kept in the per-block shared histogram (Cityscapes: 19)
constexpr int NID_FAST = 128;       // instance slots kept in the per-block shared histogram

constexpr int MAX_UNIFY_K = 256;
struct UnifyIds {                   // per-instance host arrays travel as a kernel argument (no H2D copy, no device buffer)
  short cls[MAX_UNIFY_K];
  int obj[MAX_UNIFY_K];
};

struct UnifyWs {
  unsigned int vote[NID][NID];      // vote[id][semantic class]
  unsigned int area[NID];           // pixels per panoptic id
  unsigned char lut[NID][4];        // (semantic, instance, track, unused)
  int error;
};

using vps::lab;

// one shared-memory atomic per run of equal (pan, seg) labels in a 16-pixel strip (label_runs.cuh)
template <typename TL>
__global__ void __launch_bounds__(256) unify_hist_kernel(const TL* __restrict__ seg, const TL* __restrict__ pan, int64_t npix,
                                                         int id_last_stuff, UnifyWs* __restrict__ ws) {
  __shared__ unsigned int s_vote[NID_FAST][NCLS_FAST];
  __shared__ unsigned int s_area[NID];
  for (int i = threadIdx.x; i < NID_FAST * NCLS_FAST; i += blockDim.x) (&s_vote[0][0])[i] = 0;
  for (int i = threadIdx.x; i < NID; i += blockDim.x) s_area[i] = 0;
  __syncthreads();
  const int first_inst = id_last_stuff + 1;
  auto flush = [&](int p, int sg, unsigned int n) {
    atomicAdd(&s_area[p], n);
    if (p > id_last_stuff) {
      const int j = p - first_inst;
      if (j < NID_FAST && sg < NCLS_FAST) atomicAdd(&s_vote[j][sg], n);
      else atomicAdd(&ws->vote[p][sg], n);
    }
  };
  vps::walk_label_runs(pan, seg, npix, flush);
  __syncthreads();
  for (int i = threadIdx.x; i < NID; i += blockDim.x)
    if (s_area[i]) atomicAdd(&ws->area[i], s_area[i]);
  for (int i = threadIdx.x; i < NID_FAST * NCLS_FAST; i += blockDim.x) {
    const unsigned int v = (&s_vote[0][0])[i];
    if (v) atomicAdd(&ws->vote[first_inst + i / NCLS_FAST][i % NCLS_FAST], v);
  }
}

// one block of NID threads; thread t decides the fate of panoptic id t
// obj_mode: what the third channel holds -- OBJ_COPY (a copy of pan, the video function without track ids), OBJ_TRACK
// (track id + 1) or OBJ_ZERO (the image-level function, tools/dataset/base_dataset.py:232-274, leaves it 0)
enum { OBJ_COPY = 0, OBJ_TRACK = 1, OBJ_ZERO = 2 };
__global__ void __launch_bounds__(NID) unify_decide_kernel(UnifyWs* __restrict__ ws, const __grid_constant__ UnifyIds ids,
                                                           int obj_mode, int k, int id_last_stuff,
                                                           unsigned int stuff_area_limit) {
  __shared__ unsigned int s_area[NID];
  __shared__ int s_seg[NID];
  __shared__ int s_kill[NID];
  const int t = threadIdx.x;
  const unsigned int area = ws->area[t];
  s_area[t] = area;
  s_kill[t] = 0;
  __syncthreads();
  int seg = t, ins = t, obj = t;                     // all three channels start as copies of pan (:185-187)
  if (t <= id_last_stuff) {
    ins = 0;                                         // :191
  } else if (area) {
    int rank = 0;                                    // idx of :193 = number of PRESENT instance ids below this one
    for (int u = id_last_stuff + 1; u < t; ++u) rank += s_area[u] ? 1 : 0;
    if (t == 255) {
      seg = 255; ins = 0;                            // :195-198
    } else {
      const int j = t - id_last_stuff - 1;
      unsigned int best = 0;
      int winner = 0;
      for (int c = 0; c < NID; ++c) {                // np.unique + argmax: first maximum = smallest class id
        const unsigned int v = ws->vote[t][c];
        if (v > best) { best = v; winner = c; }
      }
      if (j >= k) { ws->error = 1; }                 // the reference would raise IndexError
      const int want = (j < k ? (int)ids.cls[j] : 0) + id_last_stuff;
      const bool to_stuff = winner != want && 2ull * best >= (unsigned long long)area && winner <= id_last_stuff;   // :203
      if (to_stuff) {
        seg = winner; ins = 0; obj = 0;
      } else {
        seg = want & 255; ins = (rank + 1) & 255;
        if (obj_mode == OBJ_TRACK) obj = (ids.obj[rank < MAX_UNIFY_K ? rank : 0] + 1) & 255;   // looked up with the RANK, as the reference does (:201, :211)
      }
    }
  }
  s_seg[t] = seg;
  __syncthreads();
  // stuff classes covering fewer than stuff_area_limit pixels of the final semantic channel -> 255 (:214-219)
  if (t <= id_last_stuff) {
    unsigned long long a = 0;
    for (int u = 0; u < NID; ++u)
      if (s_area[u] && s_seg[u] == t) a += s_area[u];
    if (a > 0 && a < stuff_area_limit) s_kill[t] = 1;
  }
  __syncthreads();
  if (seg <= id_last_stuff && s_kill[seg]) seg = 255;
  if (obj_mode == OBJ_ZERO) obj = 0;
  ws->lut[t][0] = (unsigned char)seg; ws->lut[t][1] = (unsigned char)ins; ws->lut[t][2] = (unsigned char)obj; ws->lut[t][3] = 0;
}

template <typename TL>
__global__ void __launch_bounds__(256) unify_apply_kernel(const TL* __restrict__ pan, int64_t npix, const UnifyWs* __restrict__ ws,
                                                          uint8_t* __restrict__ out) {
  __shared__ unsigned char s_lut[NID][4];
  for (int i = threadIdx.x; i < NID; i += blockDim.x) *(uint32_t*)s_lut[i] = *(const uint32_t*)ws->lut[i];
  __syncthreads();
  // 4 pixels per thread: 12 output bytes = three 32-bit stores
  const int64_t nquad = npix >> 2;
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < nquad; q += (int64_t)gridDim.x * blockDim.x) {
    unsigned char b[12];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const unsigned char* l = s_lut[lab(pan, 4 * q + e)];
      b[3 * e] = l[0]; b[3 * e + 1] = l[1]; b[3 * e + 2] = l[2];
    }
    uint32_t* o = reinterpret_cast<uint32_t*>(out + 12 * q);
    o[0] = b[0] | (b[1] << 8) | (b[2] << 16) | ((uint32_t)b[3] << 24);
    o[1] = b[4] | (b[5] << 8) | (b[6] << 16) | ((uint32_t)b[7] << 24);
    o[2] = b[8] | (b[9] << 8) | (b[10] << 16) | ((uint32_t)b[11] << 24);
  }
  if (blockIdx.x == 0 && threadIdx.x < (npix & 3)) {
    const int64_t i = (nquad << 2) + threadIdx.x;
    const unsigned char* l = s_lut[lab(pan, i)];
    out[3 * i] = l[0]; out[3 * i + 1] = l[1]; out[3 * i + 2] = l[2];
  }
}
}  // namespace

extern "C" int64_t vps_unify_pan_ws_bytes(void) { return (int64_t)sizeof(UnifyWs); }

static int unify_pan(const void* seg, const void* pan, int label_bytes, int H, int W, const int32_t* cls_ind,
                     const int32_t* obj_id, int obj_mode, int k, int id_last_stuff, int stuff_area_limit, uint8_t* out,
                     void* ws, int64_t ws_bytes, void* stream) {
  VPS_CHECK_ARG(label_bytes == 1 || label_bytes == 8, "unify_pan: label_bytes %d", label_bytes);
  VPS_CHECK_ARG(ws_bytes >= (int64_t)sizeof(UnifyWs) && ((uintptr_t)ws & 15) == 0, "unify_pan: workspace");
  VPS_CHECK_ARG(id_last_stuff >= 0 && id_last_stuff < 255 && k >= 0 && k <= MAX_UNIFY_K && ((uintptr_t)out & 3) == 0, "unify_pan: args (k %d)", k);
  UnifyIds ids;
  for (int i = 0; i < MAX_UNIFY_K; ++i) {
    ids.cls[i] = (short)(i < k ? cls_ind[i] : 0);
    ids.obj[i] = (i < k && obj_id) ? obj_id[i] : 0;
  }
  const int64_t npix = (int64_t)H * W;
  if (!npix) return VPS_OK;
  cudaStream_t st = (cudaStream_t)stream;
  UnifyWs* w = (UnifyWs*)ws;
  cudaMemsetAsync(w, 0, sizeof(UnifyWs), st);
  const int blocks = (int)(((npix + 255) / 256) < 148 * 8 ? ((npix + 255) / 256) : 148 * 8);
  if (label_bytes == 1) unify_hist_kernel<uint8_t><<<blocks, 256, 0, st>>>((const uint8_t*)seg, (const uint8_t*)pan, npix, id_last_stuff, w);
  else unify_hist_kernel<int64_t><<<blocks, 256, 0, st>>>((const int64_t*)seg, (const int64_t*)pan, npix, id_last_stuff, w);
  VPS_CUDA_LAST("unify_hist");
  unify_decide_kernel<<<1, NID, 0, st>>>(w, ids, obj_mode, k, id_last_stuff, (unsigned int)stuff_area_limit);
  VPS_CUDA_LAST("unify_decide");
  if (label_bytes == 1) unify_apply_kernel<uint8_t><<<blocks, 256, 0, st>>>((const uint8_t*)pan, npix, w, out);
  else unify_apply_kernel<int64_t><<<blocks, 256, 0, st>>>((const int64_t*)pan, npix, w, out);
  VPS_CUDA_LAST("unify_apply");
  return VPS_OK;
}

extern "C" int vps_unify_pan(const void* seg, const void* pan, int label_bytes, int H, int W, const int32_t* cls_ind,
                             const int32_t* obj_id, int k, int id_last_stuff, int stuff_area_limit, uint8_t* out, void* ws,
                             int64_t ws_bytes, void* stream) {
  return unify_pan(seg, pan, label_bytes, H, W, cls_ind, obj_id, obj_id ? OBJ_TRACK : OBJ_COPY, k, id_last_stuff,
                   stuff_area_limit, out, ws, ws_bytes, stream);
}

// the image-level function (tools/dataset/base_dataset.py:232-274): same histograms and decisions, no track ids, and the
// third channel stays 0
extern "C" int vps_unify_pan_image(const void* seg, const void* pan, int label_bytes, int H, int W, const int32_t* cls_ind,
                                   int k, int id_last_stuff, int stuff_area_limit, uint8_t* out, void* ws, int64_t ws_bytes,
                                   void* stream) {
  return unify_pan(seg, pan, label_bytes, H, W, cls_ind, nullptr, OBJ_ZERO, k, id_last_stuff, stuff_area_limit, out, ws,
                   ws_bytes, stream);
}

// the reference raises IndexError when a panoptic instance id has no cls_ind entry (cityscapes_vps.py:197: cls_ind[id - id_last_stuff - 1]);
// the decide kernel records that case in the workspace.  Returns the flag of the LAST vps_unify_pan call on `ws` (synchronises `stream`).
extern "C" int vps_unify_pan_error(const void* ws, void* stream) {
  int flag = 0;
  if (cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess) return -1;
  if (cudaMemcpy(&flag, (const char*)ws + offsetof(UnifyWs, error), sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  return flag;
}

// byte offset of the error word inside the workspace (callers that must not synchronise copy it asynchronously)
extern "C" int64_t vps_unify_pan_error_offset(void) { return (int64_t)offsetof(UnifyWs, error); }
