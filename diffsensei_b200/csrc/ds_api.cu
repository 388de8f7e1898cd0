// ds_api.cu — library-wide C-ABI plumbing: version, error text, launch counter, device query,
// TMA tensor-map encoding (driver entry point resolved at run time, so the .so has no link-time
// dependency on libcuda and can be dlopen'ed for symbol checks on a box without a GPU).
#include <mutex>
#include <string>

#include "ds_host.h"

namespace ds {

static thread_local std::string t_last_error;
std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  t_last_error = buf;
}

bool get_device(DeviceInfo* out) {
  static std::mutex mu;
  static DeviceInfo cache[64];
  static bool have[64] = {false};
  int dev = -1;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess || dev < 0 || dev >= 64) {
    set_error("no CUDA device available (%s); libdsengine has no CPU fallback", cudaGetErrorString(e));
    (void)cudaGetLastError();
    return false;
  }
  std::lock_guard<std::mutex> lock(mu);
  if (!have[dev]) {
    DeviceInfo d;
    if (cudaDeviceGetAttribute(&d.num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&d.cc_major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&d.cc_minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) {
      set_error("cudaDeviceGetAttribute failed");
      (void)cudaGetLastError();
      return false;
    }
    cache[dev] = d;
    have[dev] = true;
  }
  *out = cache[dev];
  if (out->cc_major != 9 || out->cc_minor != 0) {
    set_error("device compute capability %d.%d is not sm_90: libdsengine is built for sm_90a only", out->cc_major,
              out->cc_minor);
    return false;
  }
  return true;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<EncodeTiledFn>(p);
    } else {
      (void)cudaGetLastError();
    }
  });
  return fn;
}

bool encode_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                      const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled driver entry point not available");
    return false;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = elem_strides ? elem_strides[i] : 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim,
                  gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d, dims %llu,%llu, box %u,%u, base %p)", (int)r,
              rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0],
              rank > 1 ? box[1] : 0, base);
    return false;
  }
  return true;
}

}  // namespace ds

extern "C" {

int ds_version(void) { return 100; }  // 0.1.0

const char* ds_last_error(void) { return ds::t_last_error.c_str(); }

uint64_t ds_launch_count(void) { return ds::g_launches.load(std::memory_order_relaxed); }

int ds_zero_async(void* ptr, int64_t bytes, void* stream) {
  using namespace ds;
  DS_REQUIRE(ptr != nullptr && bytes >= 0, "ds_zero_async: bad arguments");
  if (bytes > 0) DS_CUDA_OK(cudaMemsetAsync(ptr, 0, static_cast<size_t>(bytes), static_cast<cudaStream_t>(stream)));
  return DS_OK;
}

}  // extern "C"
