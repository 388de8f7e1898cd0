// ds_host.h — host-side helpers shared by the C-ABI translation units of libdsengine.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>

#include "../../include/dsengine.h"

namespace ds {

// thread-local last-error text + process-wide launch counter (defined in ds_api.cu)
void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;
inline void count_launch(uint64_t n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

// Device properties of the current device (cached). Fails (returns false + error text) when the
// current device is not an sm_90 part — there is no fallback path.
struct DeviceInfo {
  int num_sms;
  int cc_major;
  int cc_minor;
};
bool get_device(DeviceInfo* out);

// Function attributes (dynamic-smem opt-in) and occupancy answers are PER DEVICE: every cache of them is an array
// indexed by the current device's ordinal (a process may drive several GPUs through the same library).
constexpr int kMaxDevices = 64;
inline int device_slot() {
  int d = 0;
  (void)cudaGetDevice(&d);
  return d & (kMaxDevices - 1);
}

#define DS_REQUIRE(cond, ...)        \
  do {                               \
    if (!(cond)) {                   \
      ::ds::set_error(__VA_ARGS__);  \
      return DS_ERR_INVALID;         \
    }                                \
  } while (0)

#define DS_CUDA_OK(expr)                                                                       \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      ::ds::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return DS_ERR_CUDA;                                                                      \
    }                                                                                          \
  } while (0)

// check the launch that was just enqueued
#define DS_LAUNCH_OK(name)                                                           \
  do {                                                                               \
    cudaError_t _e = cudaGetLastError();                                             \
    if (_e != cudaSuccess) {                                                         \
      ::ds::set_error("launch of %s failed: %s", name, cudaGetErrorString(_e));      \
      return DS_ERR_CUDA;                                                            \
    }                                                                                \
    ::ds::count_launch();                                                            \
  } while (0)

// Fills one launch attribute: programmatic dependent launch (the kernel's prologue may overlap the previous kernel's
// tail).
inline void pdl_attr(cudaLaunchAttribute* a) {
  a->id = cudaLaunchAttributeProgrammaticStreamSerialization;
  a->val.programmaticStreamSerializationAllowed = 1;
}

// bf16 tensor map (tile mode, 128-byte swizzle, zero OOB fill). dims/strides innermost first;
// strides_bytes has rank-1 entries (dim 0 is contiguous). Returns false + error text on failure.
bool encode_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                      const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides);

}  // namespace ds
