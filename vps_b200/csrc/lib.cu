// Library-level state of libvps_b200.so: last-error string, launch counter, version; the device queries and the tensor-map
// encoder shared by the tensor-core kernels.
#include <stdarg.h>

#include <atomic>

#include "common.cuh"

namespace vps {
static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int num_sms() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  return sms;
}

PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess) {
      set_error("cuTensorMapEncodeTiled unavailable");
      return nullptr;
    }
    fn = (PFN_cuTensorMapEncodeTiled_v12000)p;
  }
  return fn;
}

bool encode_nhwc(CUtensorMap* m, const vps_tensor& t, CUtensorMapDataType type, int box_c, int box_w, int box_h, int sw, int sh,
                 CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2, const char* who, const vps_tensor* strides) {
  const auto encode = tensor_map_encoder();
  if (!encode) return false;
  const vps_tensor& s = strides ? *strides : t;
  const cuuint64_t esz = type == CU_TENSOR_MAP_DATA_TYPE_FLOAT32 ? 4 : 2;
  cuuint64_t dims[4] = {(cuuint64_t)t.c, (cuuint64_t)t.w, (cuuint64_t)t.h, (cuuint64_t)t.n};
  cuuint64_t bytes[3] = {(cuuint64_t)s.cs * esz, (cuuint64_t)s.w * s.cs * esz, (cuuint64_t)s.h * s.w * s.cs * esz};
  cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  cuuint32_t estr[4] = {1, (cuuint32_t)sw, (cuuint32_t)sh, 1};
  const CUresult r = encode(m, type, 4, t.ptr, dims, bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("%s failed (%d) dims %d,%d,%d,%d cs %d box %d,%d,%d", who, (int)r, t.c, t.w, t.h, t.n, s.cs, box_c, box_w, box_h);
    return false;
  }
  return true;
}
}  // namespace vps

extern "C" const char* vps_last_error(void) { return vps::g_err; }
extern "C" int vps_version(void) { return 100; }
extern "C" int64_t vps_launch_count(void) { return vps::g_launches.load(std::memory_order_relaxed); }
// kernels replayed through a captured CUDA graph do not pass through the launch wrappers: the host adds them here
extern "C" void vps_add_launch_count(int64_t n) { vps::count_launch((int)n); }
