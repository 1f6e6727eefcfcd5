// Run-length walk over pairs of label maps, shared by the unify histogram (unify.cu) and the semantic confusion matrix
// (ipq.cu).  Label maps are piecewise constant: every thread walks strips of 16 consecutive pixels and reports each run of
// equal (a, b) labels once, so a histogram issues one shared-memory atomic per run instead of one per pixel.
#pragma once
#include "common.cuh"

namespace vps {

// label value of pixel i: the low byte (int64 maps carry uint8 values, as the reference's collector casts them)
template <typename TL>
__device__ __forceinline__ int lab(const TL* p, int64_t i) { return (int)((unsigned long long)p[i] & 0xFFull); }

constexpr int LABEL_RUN = 16;

// the 16 labels of the strip starting at i0 (cnt valid pixels; -1 past the end): one uint4 load for an aligned uint8 map
template <typename TL>
__device__ __forceinline__ void load_strip(const TL* __restrict__ p, int64_t i0, int cnt, int (&v)[LABEL_RUN]) {
  if (sizeof(TL) == 1 && cnt == LABEL_RUN && ((uintptr_t)p & 15) == 0) {
    const uint4 a = *reinterpret_cast<const uint4*>((const uint8_t*)p + i0);
    const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int e = 0; e < LABEL_RUN; ++e) v[e] = (w[e >> 2] >> (8 * (e & 3))) & 255;
  } else {
#pragma unroll
    for (int e = 0; e < LABEL_RUN; ++e) v[e] = e < cnt ? lab(p, i0 + e) : -1;
  }
}

// a label map read in place: fetch(i0, cnt, v) fills the strip starting at pixel i0
template <typename TL>
struct StripOf {
  const TL* __restrict__ p;
  __device__ __forceinline__ void operator()(int64_t i0, int cnt, int (&v)[LABEL_RUN]) const { load_strip(p, i0, cnt, v); }
};

// grid-stride walk over the 16-pixel strips of two label sources of npix pixels; fetch_a / fetch_b(i0, cnt, v) give each
// strip's labels (-1 past the end), flush(a, b, n) is called once per run of n equal pairs
template <typename FA, typename FB, typename F>
__device__ __forceinline__ void walk_label_runs_by(FA&& fetch_a, FB&& fetch_b, int64_t npix, F&& flush) {
  const int64_t nrun = (npix + LABEL_RUN - 1) / LABEL_RUN;
  VPS_GRID_STRIDE(r, nrun) {
    const int64_t i0 = r * LABEL_RUN;
    const int cnt = (int)min((int64_t)LABEL_RUN, npix - i0);
    int av[LABEL_RUN], bv[LABEL_RUN];
    fetch_a(i0, cnt, av);
    fetch_b(i0, cnt, bv);
    int ca = av[0], cb = bv[0];
    unsigned int n = 1;
#pragma unroll
    for (int e = 1; e < LABEL_RUN; ++e) {
      if (av[e] < 0) break;
      if (av[e] == ca && bv[e] == cb) { ++n; }
      else { flush(ca, cb, n); ca = av[e]; cb = bv[e]; n = 1; }
    }
    flush(ca, cb, n);
  }
}

// the same walk over two maps stored in place
template <typename TA, typename TB, typename F>
__device__ __forceinline__ void walk_label_runs(const TA* __restrict__ a, const TB* __restrict__ b, int64_t npix, F&& flush) {
  walk_label_runs_by(StripOf<TA>{a}, StripOf<TB>{b}, npix, flush);
}

}  // namespace vps
