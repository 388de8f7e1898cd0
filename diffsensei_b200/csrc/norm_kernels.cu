// norm_kernels.cu — GroupNorm(+SiLU) and LayerNorm for channels-last bf16 activations (HBM-bound).
//
// GroupNorm on NHWC: a group's channels are interleaved with every other group's inside each pixel, so the
// coalesced decomposition is by PIXEL RANGE, not by group: a CTA streams a contiguous run of pixels (all
// channels, 16-byte vectors, every thread pinned to the same 8 channels).
//   statistics : per-(sample, CHANNEL) {sum, sum of squares} in fp64, [B][C][2].  Normally they come for free from
//                the epilogue of the GEMM / conv that PRODUCED the tensor (gemm_wgmma.cu, `chan_stats`); tensors
//                without such a producer (conv_in output, unaligned shapes) get them from chan_stats_kernel.
//                Per-channel (not per-group) sums make them composable: the statistics of torch.cat([h, skip], 1)
//                are the two tensors' statistics side by side, whatever the group boundaries of the result.
//   apply      : gn_apply2_kernel reads x ONCE (from one or two source tensors — the up-block concatenation is never
//                written), folds the channel sums into the 32 groups' mean / rstd in shared memory (fixed order),
//                normalises, applies gamma / beta (+ SiLU) in fp32 and rounds once to bf16.
// Algorithmic bytes: read x + write y = 4 B/element — which is all the apply kernel moves.
//
// Replaces diffusers ResnetBlock2D.norm1/norm2+SiLU, Transformer2DModel.norm, conv_norm_out+conv_act
// (reached from src/models/unet.py:251-261,281-290,316-338) and BasicTransformerBlock / Resampler LayerNorms
// (src/models/resampler.py:14,40-41,104).
#include "ds_common.cuh"
#include "ds_host.h"

namespace ds {

// Launch shape: threads per CTA of the apply and statistics kernels, the apply kernel's independent 16-byte loads in
// flight per thread, and its cap on resident CTAs per SM.
constexpr int kGnApplyThreads = 256;
constexpr int kGnStatsThreads = 512;
constexpr int kGnUnroll = 8;
constexpr int kGnMaxOcc = 8;

// L2 residency control for the two-pass GroupNorm: the stats pass marks x evict_last so that the apply pass
// re-reads it from the L2 instead of HBM; the apply pass reads x with the evict_normal policy.
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_normal() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint4 ldg_hint(const uint4* ptr, uint64_t pol) {
  uint4 v;
  asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(ptr), "l"(pol));
  return v;
}

// Work decomposition: the tensor is cut into ITEMS of `ipx` consecutive pixels of one sample (item id = sample *
// items_per_sample + k); a launch has exactly one resident wave of CTAs (grid = SMs x occupancy) and CTA c owns the
// contiguous item range [c*I/G, (c+1)*I/G) — so no tail wave, and a CTA touches at most a couple of samples.
// blockDim.x = cv * rpb (cv = C/8 16-byte vectors per pixel, rpb pixel rows per sweep); every thread stays pinned to
// the same 8 channels.
__device__ __forceinline__ void gn_item_range(int total_items, int& i0, int& i1) {
  const long long g = gridDim.x, c = blockIdx.x;
  i0 = static_cast<int>(c * total_items / g);
  i1 = static_cast<int>((c + 1) * total_items / g);
}

// Per-(sample, channel) {sum, sum of squares} of a [B][HW][C] bf16 tensor -> fp64 [B][C][2] (accumulated: the caller
// zeroes it).  Threads keep fp32 partials over <= a few hundred pixels, the CTA's pixel rows are combined in a fixed
// order in shared memory and every channel adds ONE fp64 pair per (CTA, sample) — fp64 sums of a few hundred fp32
// partials are exact, so the result does not depend on the arrival order.
__global__ void chan_stats_kernel(const uint4* __restrict__ x, double* __restrict__ stats, int HW, int C,
                                  int items_per_sample, int ipx, int total_items) {
  extern __shared__ float shs[];  // [rpb][C][2]
  const int cv = C >> 3;
  const int rpb = blockDim.x / cv;
  const int cvec = threadIdx.x % cv;
  const int prow = threadIdx.x / cv;
  int i0, i1;
  gn_item_range(total_items, i0, i1);
  pdl_launch_dependents();  // programmatic dependent launch: our launch latency overlapped the producer's tail ...
  pdl_wait();               // ... and nothing of the producer's output is touched before it has completed
  if (i0 >= i1) return;
  float s[8], q[8];
  auto reset = [&]() {
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
  };
  auto accum = [&](const uint4& u) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a = bf16_lo(w[j]), c = bf16_hi(w[j]);
      s[2 * j] += a;
      q[2 * j] = fmaf(a, a, q[2 * j]);
      s[2 * j + 1] += c;
      q[2 * j + 1] = fmaf(c, c, q[2 * j + 1]);
    }
  };
  auto flush = [&](int b) {
    float* row = shs + (static_cast<size_t>(prow) * C + cvec * 8) * 2;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      row[2 * j] = s[j];
      row[2 * j + 1] = q[j];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      float ts = 0.f, tq = 0.f;
      for (int r = 0; r < rpb; ++r) {
        ts += shs[(static_cast<size_t>(r) * C + c) * 2];
        tq += shs[(static_cast<size_t>(r) * C + c) * 2 + 1];
      }
      double* gp = stats + (static_cast<size_t>(b) * C + c) * 2;
      atomicAdd(gp, static_cast<double>(ts));
      atomicAdd(gp + 1, static_cast<double>(tq));
    }
    __syncthreads();
  };
  reset();
  const uint64_t pol = l2_policy_evict_last();  // the GroupNorm apply pass that follows re-reads x
  int cur_b = i0 / items_per_sample;
  for (int it = i0; it < i1; ++it) {
    const int b = it / items_per_sample;
    if (b != cur_b) {  // CTA-uniform
      flush(cur_b);
      reset();
      cur_b = b;
    }
    const int p0 = (it - b * items_per_sample) * ipx;
    const int p1 = min(p0 + ipx, HW);
    const uint4* base = x + (static_cast<size_t>(b) * HW) * cv + cvec;
    int p = p0 + prow;
    for (; p + 7 * rpb < p1; p += 8 * rpb) {  // 8 independent 16-byte loads in flight per thread
      uint4 u[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) u[k] = ldg_hint(base + static_cast<size_t>(p + k * rpb) * cv, pol);
#pragma unroll
      for (int k = 0; k < 8; ++k) accum(u[k]);
    }
    for (; p < p1; p += rpb) accum(ldg_hint(base + static_cast<size_t>(p) * cv, pol));
  }
  flush(cur_b);
}

// GroupNorm(+SiLU) apply from per-channel statistics; x = [x1 | x2] along channels (x2 may be NULL).
// kU = independent 16-byte loads in flight per thread.
template <bool kSilu, int kU>
__global__ void gn_apply2_kernel(const uint4* __restrict__ x1, const uint4* __restrict__ x2, uint4* __restrict__ y,
                                 const double* __restrict__ st1, const double* __restrict__ st2,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, int HW, int C1, int C2,
                                 int groups, float eps, int items_per_sample, int ipx, int total_items) {
  extern __shared__ double shd[];  // [C][2] channel sums of the current sample, then [groups][2] {mean, rstd}
  const int C = C1 + C2;
  const int cv = C >> 3, cv1 = C1 >> 3;
  const int rpb = blockDim.x / cv;
  const int cvec = threadIdx.x % cv;
  const int prow = threadIdx.x / cv;
  const int cpg = C / groups;
  const double inv_n = 1.0 / (static_cast<double>(HW) * cpg);
  float* sh_coef = reinterpret_cast<float*>(shd + 2 * static_cast<size_t>(C));  // [groups][2]
  int i0, i1;
  gn_item_range(total_items, i0, i1);
  pdl_launch_dependents();
  if (i0 >= i1) {
    pdl_wait();
    return;
  }
  // this thread's source: its 8 channels live entirely in x1 or entirely in x2 (C1 % 8 == 0)
  const bool second = cvec >= cv1;
  const uint4* xsrc = second ? x2 : x1;
  const int scv = second ? (cv - cv1) : cv1;        // row pitch of the source in 16-byte vectors
  const int svec = second ? (cvec - cv1) : cvec;
  float ga[8], be[8], sc[8], sf[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    ga[j] = __ldg(gamma + cvec * 8 + j);   // parameters: not written by the predecessor kernel
    be[j] = __ldg(beta + cvec * 8 + j);
  }
  pdl_wait();  // x and the statistics come from the predecessor
  const uint64_t pol = l2_policy_normal();
  // group coefficients of sample b: channel sums -> smem -> 32 threads fold cpg channels each, in order
  auto load_coeffs = [&](int b) {
    __syncthreads();                                 // previous sample's coefficients no longer in use
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const double* gp = (c < C1) ? st1 + (static_cast<size_t>(b) * C1 + c) * 2
                                  : st2 + (static_cast<size_t>(b) * C2 + (c - C1)) * 2;
      const double2 v = *reinterpret_cast<const double2*>(gp);
      shd[2 * c] = v.x;
      shd[2 * c + 1] = v.y;
    }
    __syncthreads();
    if (threadIdx.x < groups) {
      double ts = 0.0, tq = 0.0;
      const double* gp = shd + 2 * static_cast<size_t>(threadIdx.x) * cpg;
      for (int k = 0; k < cpg; ++k) {
        ts += gp[2 * k];
        tq += gp[2 * k + 1];
      }
      const double mean = ts * inv_n;
      double var = tq * inv_n - mean * mean;
      var = var < 0.0 ? 0.0 : var;
      sh_coef[2 * threadIdx.x] = static_cast<float>(mean);
      sh_coef[2 * threadIdx.x + 1] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int g = (cvec * 8 + j) / cpg;
      const float mean = sh_coef[2 * g], rstd = sh_coef[2 * g + 1];
      sc[j] = rstd * ga[j];
      sf[j] = be[j] - mean * rstd * ga[j];
    }
  };
  auto norm8 = [&](const uint4& u) -> uint4 {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float a = fmaf(bf16_lo(w[j]), sc[2 * j], sf[2 * j]);
      float c = fmaf(bf16_hi(w[j]), sc[2 * j + 1], sf[2 * j + 1]);
      if (kSilu) {
        a = silu_tanh_f(a);
        c = silu_tanh_f(c);
      }
      o[j] = pack_bf16_alu(a, c);
    }
    return make_uint4(o[0], o[1], o[2], o[3]);
  };
  int cur_b = -1;
  for (int it = i0; it < i1; ++it) {
    const int b = it / items_per_sample;
    const int p0 = (it - b * items_per_sample) * ipx;
    const int p1 = min(p0 + ipx, HW);
    const uint4* xb = xsrc + (static_cast<size_t>(b) * HW) * scv + svec;
    uint4* yb = y + (static_cast<size_t>(b) * HW) * cv + cvec;
    int p = p0 + prow;
    // the first batch of loads is issued BEFORE the (CTA-wide, L2-latency-bound) coefficient fold of a new sample
    uint4 u[kU];
    const bool full = p + (kU - 1) * rpb < p1;
    if (full) {
#pragma unroll
      for (int k = 0; k < kU; ++k) u[k] = ldg_hint(xb + static_cast<size_t>(p + k * rpb) * scv, pol);
    }
    if (b != cur_b) {  // CTA-uniform
      load_coeffs(b);
      cur_b = b;
    }
    if (full) {
#pragma unroll
      for (int k = 0; k < kU; ++k) yb[static_cast<size_t>(p + k * rpb) * cv] = norm8(u[k]);
      p += kU * rpb;
    }
    for (; p + (kU - 1) * rpb < p1; p += kU * rpb) {
#pragma unroll
      for (int k = 0; k < kU; ++k) u[k] = ldg_hint(xb + static_cast<size_t>(p + k * rpb) * scv, pol);
#pragma unroll
      for (int k = 0; k < kU; ++k) yb[static_cast<size_t>(p + k * rpb) * cv] = norm8(u[k]);
    }
    for (; p < p1; p += rpb) yb[static_cast<size_t>(p) * cv] = norm8(ldg_hint(xb + static_cast<size_t>(p) * scv, pol));
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, the whole row held in registers (two-pass mean / variance, fp32).
// ------------------------------------------------------------------------------------------------
template <int MAXV>
__global__ void layernorm_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, int rows, int C, float eps) {
  const int cv = C >> 3;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const uint4* xr = x + static_cast<size_t>(warp) * cv;
  uint4* yr = y + static_cast<size_t>(warp) * cv;
  float v[MAXV][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + 32 * i;
    if (vi < cv) {
      const uint4 u = __ldg(xr + vi);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        v[i][2 * j] = bf16_lo(w[j]);
        v[i][2 * j + 1] = bf16_hi(w[j]);
        sum += v[i][2 * j] + v[i][2 * j + 1];
      }
    }
  }
  const float mean = warp_sum(sum) / static_cast<float>(C);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + 32 * i;
    if (vi < cv) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[i][j] - mean;
        sq += d * d;
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / static_cast<float>(C) + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + 32 * i;
    if (vi < cv) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * vi);
      const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * vi + 1);
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta) + 2 * vi);
      const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta) + 2 * vi + 1);
      const float ga[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float be[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
        o[j] = pack_bf16_alu((v[i][2 * j] - mean) * rstd * ga[2 * j] + be[2 * j],
                             (v[i][2 * j + 1] - mean) * rstd * ga[2 * j + 1] + be[2 * j + 1]);
      yr[vi] = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

}  // namespace ds

namespace {
struct GnPlan {
  int threads, rpb, ipx, items_per_sample, total_items;
};
// blockDim = cv * rpb threads (<= target), items of `sweeps` sweeps of the CTA's pixel rows
static bool gn_plan(int B, int HW, int C, int target_threads, int sweeps, GnPlan* pl) {
  const int cv = C / 8;
  if (cv > 1024) return false;
  int rpb = target_threads / cv;
  if (rpb < 1) rpb = 1;
  pl->rpb = rpb;
  pl->threads = cv * rpb;
  pl->ipx = sweeps * rpb;
  pl->items_per_sample = (HW + pl->ipx - 1) / pl->ipx;
  const long long t = static_cast<long long>(B) * pl->items_per_sample;
  if (t >= (1ll << 30)) return false;
  pl->total_items = static_cast<int>(t);
  return true;
}
}  // namespace

extern "C" int ds_channel_stats(const void* x, double* stats, int B, int HW, int C, void* stream) {
  using namespace ds;
  DS_REQUIRE(x && stats, "ds_channel_stats: NULL pointer");
  DS_REQUIRE(B > 0 && HW > 0 && C > 0 && C % 8 == 0 && C <= 8192, "ds_channel_stats: bad shape (C %% 8 == 0, C <= 8192)");
  DS_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(stats) & 15) == 0,
             "ds_channel_stats: x / stats must be 16-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  GnPlan pl;
  DS_REQUIRE(gn_plan(B, HW, C, kGnStatsThreads, 8, &pl), "ds_channel_stats: tensor too large");
  const size_t smem = static_cast<size_t>(pl.rpb) * C * 2 * sizeof(float);
  static size_t attr[kMaxDevices] = {};
  if (smem > 48 * 1024 && smem > attr[device_slot()]) {
    DS_CUDA_OK(cudaFuncSetAttribute(chan_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    attr[device_slot()] = smem;
  }
  int occ = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, chan_stats_kernel, pl.threads, smem) != cudaSuccess || occ < 1) {
    (void)cudaGetLastError();
    occ = 1;
  }
  if (occ > 2) occ = 2;  // few, fat CTAs: every CTA ends with 2*C fp64 atomics per sample it touched
  const long long g = static_cast<long long>(occ) * dev.num_sms;
  const int grid = static_cast<int>(g < pl.total_items ? g : pl.total_items);
  {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(pl.threads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    pdl_attr(&attr[0]);
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    DS_CUDA_OK(cudaLaunchKernelEx(&cfg, chan_stats_kernel, static_cast<const uint4*>(x), stats, HW, C,
                                  pl.items_per_sample, pl.ipx, pl.total_items));
  }
  DS_LAUNCH_OK("chan_stats_kernel");
  return DS_OK;
}

extern "C" int ds_groupnorm_apply(const void* x1, const double* stats1, int C1, const void* x2, const double* stats2,
                                  int C2, void* y, const float* gamma, const float* beta, int B, int HW, int groups,
                                  float eps, int apply_silu, void* stream) {
  using namespace ds;
  DS_REQUIRE(x1 && stats1 && y && gamma && beta, "ds_groupnorm_apply: NULL pointer");
  DS_REQUIRE((x2 == nullptr) == (C2 == 0) && (x2 == nullptr) == (stats2 == nullptr),
             "ds_groupnorm_apply: x2 / stats2 / C2 must be given together");
  const int C = C1 + C2;
  DS_REQUIRE(B > 0 && HW > 0 && C1 > 0 && C2 >= 0 && groups > 0 && groups <= 64, "ds_groupnorm_apply: bad shape");
  DS_REQUIRE(C1 % 8 == 0 && C2 % 8 == 0 && C % groups == 0 && C <= 8192,
             "ds_groupnorm_apply: C1, C2 must be multiples of 8 and C1 + C2 (%d) a multiple of groups (%d)", C, groups);
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  DS_REQUIRE(al16(x1) && al16(y) && al16(stats1) && (!x2 || (al16(x2) && al16(stats2))),
             "ds_groupnorm_apply: x / y / stats must be 16-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  GnPlan pl;
  DS_REQUIRE(gn_plan(B, HW, C, kGnApplyThreads, kGnUnroll, &pl), "ds_groupnorm_apply: tensor too large");
  const size_t smem = static_cast<size_t>(C) * 2 * sizeof(double) + static_cast<size_t>(groups) * 2 * sizeof(float);
  auto* fn = apply_silu ? gn_apply2_kernel<true, kGnUnroll> : gn_apply2_kernel<false, kGnUnroll>;
  static size_t attr[kMaxDevices][2] = {};
  size_t& a = attr[device_slot()][apply_silu ? 1 : 0];
  if (smem > 48 * 1024 && smem > a) {
    DS_CUDA_OK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    a = smem;
  }
  int occ = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, pl.threads, smem) != cudaSuccess || occ < 1) {
    (void)cudaGetLastError();
    occ = 1;
  }
  if (occ > kGnMaxOcc) occ = kGnMaxOcc;
  const long long g = static_cast<long long>(occ) * dev.num_sms;
  const int grid = static_cast<int>(g < pl.total_items ? g : pl.total_items);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(pl.threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute lattr[1];
  pdl_attr(&lattr[0]);
  cfg.attrs = lattr;
  cfg.numAttrs = 1;
  DS_CUDA_OK(cudaLaunchKernelEx(&cfg, fn, static_cast<const uint4*>(x1), static_cast<const uint4*>(x2),
                                static_cast<uint4*>(y), stats1, stats2, gamma, beta, HW, C1, C2, groups, eps,
                                pl.items_per_sample, pl.ipx, pl.total_items));
  DS_LAUNCH_OK("gn_apply2_kernel");
  return DS_OK;
}

extern "C" int ds_groupnorm_silu(const void* x, void* y, const float* gamma, const float* beta, float* stats, int B,
                                 int HW, int C, int groups, float eps, int apply_silu, void* stream) {
  using namespace ds;
  DS_REQUIRE(x && y && gamma && beta && stats, "ds_groupnorm_silu: NULL pointer");
  DS_REQUIRE(B > 0 && HW > 0 && C > 0 && groups > 0, "ds_groupnorm_silu: bad shape");
  DS_REQUIRE((reinterpret_cast<uintptr_t>(stats) & 15) == 0, "ds_groupnorm_silu: stats scratch must be 16-byte aligned");
  // stand-alone form (no producer statistics): one statistics pass + the apply pass.  scratch = fp64 [B][C][2]
  double* dstats = reinterpret_cast<double*>(stats);
  DS_CUDA_OK(cudaMemsetAsync(dstats, 0, sizeof(double) * 2 * static_cast<size_t>(B) * C, static_cast<cudaStream_t>(stream)));
  int rc = ds_channel_stats(x, dstats, B, HW, C, stream);
  if (rc != DS_OK) return rc;
  return ds_groupnorm_apply(x, dstats, C, nullptr, nullptr, 0, y, gamma, beta, B, HW, groups, eps, apply_silu, stream);
}

extern "C" int64_t ds_groupnorm_scratch_floats(int B, int C) {
  if (B <= 0 || C <= 0) return 0;
  return static_cast<int64_t>(4) * B * C;  // fp64 [B][C][2]
}

extern "C" int ds_layernorm(const void* x, void* y, const float* gamma, const float* beta, int rows, int C, float eps,
                            void* stream) {
  using namespace ds;
  DS_REQUIRE(x && y && gamma && beta, "ds_layernorm: NULL pointer");
  DS_REQUIRE(rows > 0 && C > 0 && C % 8 == 0, "ds_layernorm: rows>0 and C %% 8 == 0 required (rows=%d C=%d)", rows, C);
  DS_REQUIRE(C <= 5120, "ds_layernorm: C (%d) > 5120 unsupported", C);
  DS_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(gamma) & 15) == 0 && (reinterpret_cast<uintptr_t>(beta) & 15) == 0,
             "ds_layernorm: pointers must be 16-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int threads = 256;
  const int blocks = (rows + 7) / 8;
  const int cv = C / 8;
  const int per_lane = (cv + 31) / 32;  // 16-byte vectors each lane holds: exact-fit instantiation keeps registers low
#define DS_LN_CASE(V)                                                                                             \
  layernorm_kernel<V><<<blocks, threads, 0, st>>>(static_cast<const uint4*>(x), static_cast<uint4*>(y), gamma, beta, \
                                                  rows, C, eps)
  switch (per_lane) {
    case 1: DS_LN_CASE(1); break;
    case 2: DS_LN_CASE(2); break;
    case 3: DS_LN_CASE(3); break;
    case 4: DS_LN_CASE(4); break;
    case 5: DS_LN_CASE(5); break;
    case 6: DS_LN_CASE(6); break;
    case 7:
    case 8: DS_LN_CASE(8); break;
    case 9: case 10: case 11: case 12: case 13: case 14: case 15:
    case 16: DS_LN_CASE(16); break;
    default: DS_LN_CASE(20); break;
  }
#undef DS_LN_CASE
  DS_LAUNCH_OK("layernorm_kernel");
  return DS_OK;
}
