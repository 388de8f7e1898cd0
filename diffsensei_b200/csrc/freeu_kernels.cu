// freeu_kernels.cu — FreeU's skip-connection Fourier filter and backbone scaling on channels-last bf16 (HBM-bound).
//
// diffusers' apply_freeu (diffusers.utils.torch_utils, reached from every up-block of UNet2DConditionModel once
// enable_freeu has set s1, s2, b1, b2) runs in front of each up-block resnet of up-blocks 0 and 1:
//   hidden[:, :C/2] *= b;   skip = fourier_filter(skip, threshold=1, scale=s)
// fourier_filter takes fftshift(fftn(skip)) over (H, W), multiplies the block [H/2-1, H/2+1) x [W/2-1, W/2+1) by s
// and returns ifftn(ifftshift(.)).real.  That block holds the frequencies Ky x Kx with Ky = {0, -1 mod H} and
// Kx = {0, -1 mod W} as SETS (a size-1 axis gives {0} alone), so no FFT is needed:
//   y[h,w] = x[h,w] - (1 - s) / (HW) * Re sum_{ky in Ky, kx in Kx} X[ky,kx] e^{+2 pi i (ky h / H + kx w / W)}
// and with th = 2 pi h / H, ph = 2 pi w / W, ps = th + ph the frequency (-1, 0) contributes Ch cos th + Sh sin th where
// Ch = sum x cos th, Sh = sum x sin th, and likewise (0, -1) with ph and (-1, -1) with ps.  Per (sample, channel)
// that is 7 real moments: sum x, then {sum x cos, sum x sin} of th, ph and ps.
//   freeu_moments_kernel : the 7 moments (one read of the skip), in chan_stats_kernel's way: one fp32 partial per ITEM
//                          (a run of pixels of one sample that depends only on H, W and C), combined with fp64
//                          atomics, so a sample's moments are the same bits at any batch size and in any CTA.
//   freeu_apply_kernel   : one launch per site.  blockIdx.y = 0 filters the skip, blockIdx.y = 1 scales the hidden
//                          channels [0, C/2) by b; both accumulate the GroupNorm statistics of what they wrote with
//                          chan_stats_kernel's items and fp32 partials, so those equal ds_channel_stats of the output
//                          bit for bit (the up-block resnet's norm1 consumes them; the producers' are stale).
// The twiddles cos/sin(2 pi k / n) come from sincospif(2k / n) (exact multiplication by pi), one table per CTA in
// shared memory.
#include "ds_common.cuh"
#include "ds_host.h"

namespace ds {

constexpr int kFuMaxSide = 2048;  // H, W <= this: the twiddle table takes 8 (H + W) bytes of shared memory
constexpr int kFuMomUnroll = 4;   // independent 16-byte loads in flight per thread
constexpr int kFuMomSweeps = 16;  // pixel-row sweeps per moments item: C * 7 fp64 atomics per item
constexpr int kFuApplyUnroll = 2;  // (the filter keeps 56 coefficients in registers)

// tw[k] = {cos, sin}(2 pi k / H) for k < H, then tw[H + k] = {cos, sin}(2 pi k / W)
__device__ __forceinline__ void fu_twiddles(float2* tw, int H, int W) {
  for (int i = threadIdx.x; i < H + W; i += blockDim.x) {
    const int n = i < H ? H : W;
    const int k = i < H ? i : i - H;
    float sv, cv;
    sincospif(static_cast<float>(2 * k) / static_cast<float>(n), &sv, &cv);
    tw[i] = make_float2(cv, sv);
  }
}

// {cos th, sin th, cos ph, sin ph, cos ps, sin ps} of pixel p
__device__ __forceinline__ void fu_phase(const float2* tw, int p, int H, int W, float (&f)[6]) {
  const int h = p / W;
  const float2 a = tw[h], b = tw[H + p - h * W];
  f[0] = a.x;
  f[1] = a.y;
  f[2] = b.x;
  f[3] = b.y;
  f[4] = a.x * b.x - a.y * b.y;
  f[5] = a.y * b.x + a.x * b.y;
}

__global__ void __launch_bounds__(kGnStatsThreads) freeu_moments_kernel(const uint4* __restrict__ x,
                                                                         double* __restrict__ mom, int H, int W,
                                                                         int C, int items_per_sample, int ipx,
                                                                         int total_items) {
  extern __shared__ float4 fu_smem[];
  float2* tw = reinterpret_cast<float2*>(fu_smem);
  float* red = reinterpret_cast<float*>(tw + H + W);  // [rpb][C][7]
  const int HW = H * W, cv = C >> 3, rpb = blockDim.x / cv;
  const int cvec = threadIdx.x % cv, prow = threadIdx.x / cv;
  int i0, i1;
  gn_item_range(total_items, i0, i1);
  pdl_launch_dependents();
  fu_twiddles(tw, H, W);  // no global memory: overlaps the producer's tail
  pdl_wait();
  if (i0 >= i1) return;
  __syncthreads();
  float acc[7][8];
  auto reset = [&]() {
#pragma unroll
    for (int k = 0; k < 7; ++k)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[k][j] = 0.f;
  };
  auto accum = [&](const uint4& u, int p) {
    float f[6];
    fu_phase(tw, p, H, W, f);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float a = (j & 1) ? bf16_hi(w[j >> 1]) : bf16_lo(w[j >> 1]);
      acc[0][j] += a;
#pragma unroll
      for (int k = 0; k < 6; ++k) acc[k + 1][j] = fmaf(a, f[k], acc[k + 1][j]);
    }
  };
  // one fp64 add per (channel, moment) per item: the CTA's pixel rows are summed in shared memory in a fixed order
  auto flush = [&](int b) {
    float* row = red + (static_cast<size_t>(prow) * C + cvec * 8) * 7;
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int k = 0; k < 7; ++k) row[j * 7 + k] = acc[k][j];
    __syncthreads();
    for (int i = threadIdx.x; i < C * 7; i += blockDim.x) {
      float t = 0.f;
      for (int r = 0; r < rpb; ++r) t += red[static_cast<size_t>(r) * C * 7 + i];
      atomicAdd(mom + static_cast<size_t>(b) * C * 7 + i, static_cast<double>(t));
    }
    __syncthreads();
  };
  for (int it = i0; it < i1; ++it) {
    const int b = it / items_per_sample;
    reset();
    const int p0 = (it - b * items_per_sample) * ipx;
    const int p1 = min(p0 + ipx, HW);
    const uint4* base = x + (static_cast<size_t>(b) * HW) * cv + cvec;
    int p = p0 + prow;
    for (; p + (kFuMomUnroll - 1) * rpb < p1; p += kFuMomUnroll * rpb) {
      uint4 u[kFuMomUnroll];
#pragma unroll
      for (int k = 0; k < kFuMomUnroll; ++k) u[k] = __ldg(base + static_cast<size_t>(p + k * rpb) * cv);
#pragma unroll
      for (int k = 0; k < kFuMomUnroll; ++k) accum(u[k], p + k * rpb);
    }
    for (; p < p1; p += rpb) accum(__ldg(base + static_cast<size_t>(p) * cv), p);
    flush(b);
  }
}

struct FuSeg {
  const uint4* x;  // read, then written through y by the same thread: y may alias x
  uint4* y;
  double* stats;   // fp64 [B][C][2], accumulated
  int C, threads, rpb, ipx, items_per_sample, total_items;
};

struct FuApplyParams {
  FuSeg seg[2];        // 0: skip (filtered), 1: hidden (channels < half scaled by b)
  const double* mom;   // fp64 [B][C_skip][7]
  double kscale;       // (1 - s) / (H W)
  float b;
  int H, W, half;
};

__global__ void __launch_bounds__(kGnStatsThreads) freeu_apply_kernel(const FuApplyParams P) {
  extern __shared__ float4 fu_smem[];
  const bool filt = blockIdx.y == 0;
  const FuSeg sg = filt ? P.seg[0] : P.seg[1];
  const int H = P.H, W = P.W, HW = H * W, C = sg.C, cv = C >> 3, rpb = sg.rpb;
  float2* tw = reinterpret_cast<float2*>(fu_smem);
  float* shs = reinterpret_cast<float*>(tw + (filt ? H + W : 0));  // [rpb][C][2]
  const bool active = threadIdx.x < sg.threads;
  const int cvec = threadIdx.x % cv, prow = threadIdx.x / cv;
  int i0, i1;
  gn_item_range(sg.total_items, i0, i1);
  pdl_launch_dependents();
  if (filt) fu_twiddles(tw, H, W);
  pdl_wait();
  if (i0 >= i1) return;
  __syncthreads();
  // the skip's per-channel coefficients of the low-frequency part, A_k = (1 - s) / (HW) * moment_k, with the terms of
  // a frequency that coincides with 0 (a size-1 axis) dropped
  float A[7][8];
  const bool use_h = H > 1, use_w = W > 1;
  auto load_coef = [&](int b) {
    const double* m = P.mom + (static_cast<size_t>(b) * C + cvec * 8) * 7;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const bool on[7] = {true, use_h, use_h, use_w, use_w, use_h && use_w, use_h && use_w};
#pragma unroll
      for (int k = 0; k < 7; ++k) A[k][j] = on[k] ? static_cast<float>(m[j * 7 + k] * P.kscale) : 0.f;
    }
  };
  // identical arithmetic to chan_stats_kernel: s += v, q = fma(v, v, q) in pixel order, rows summed in order
  float s[8] = {}, q[8] = {};
  auto stat = [&](uint32_t o, int j) {
    const float a = bf16_lo(o), c = bf16_hi(o);
    s[2 * j] += a;
    q[2 * j] = fmaf(a, a, q[2 * j]);
    s[2 * j + 1] += c;
    q[2 * j + 1] = fmaf(c, c, q[2 * j + 1]);
  };
  auto flush = [&](int b) {
    if (active) {
      float* row = shs + (static_cast<size_t>(prow) * C + cvec * 8) * 2;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        row[2 * j] = s[j];
        row[2 * j + 1] = q[j];
      }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      float ts = 0.f, tq = 0.f;
      for (int r = 0; r < rpb; ++r) {
        ts += shs[(static_cast<size_t>(r) * C + c) * 2];
        tq += shs[(static_cast<size_t>(r) * C + c) * 2 + 1];
      }
      double* gp = sg.stats + (static_cast<size_t>(b) * C + c) * 2;
      atomicAdd(gp, static_cast<double>(ts));
      atomicAdd(gp + 1, static_cast<double>(tq));
    }
    __syncthreads();
  };
  // hidden: channel c0 + j is scaled when c0 + j < half; a vector above half is only stored when y is another tensor
  const int c0 = cvec * 8;
  const bool keep_vec = !filt && c0 >= P.half && sg.y == sg.x;
  auto process = [&](const uint4& u, int p) -> uint4 {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    uint32_t o[4];
    if (filt) {
      float f[6];
      fu_phase(tw, p, H, W, f);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float y[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int ch = 2 * j + e;
          float l = A[0][ch];
#pragma unroll
          for (int k = 0; k < 6; ++k) l = fmaf(A[k + 1][ch], f[k], l);
          y[e] = (e ? bf16_hi(w[j]) : bf16_lo(w[j])) - l;
        }
        o[j] = pack_bf16(y[0], y[1]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float lo = bf16_lo(w[j]), hi = bf16_hi(w[j]);
        o[j] = pack_bf16(c0 + 2 * j < P.half ? lo * P.b : lo, c0 + 2 * j + 1 < P.half ? hi * P.b : hi);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) stat(o[j], j);
    return make_uint4(o[0], o[1], o[2], o[3]);
  };
  int cur = -1;
  for (int it = i0; it < i1; ++it) {
    const int b = it / sg.items_per_sample;
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
    if (active) {
      if (filt && b != cur) {
        load_coef(b);
        cur = b;
      }
      const int p0 = (it - b * sg.items_per_sample) * sg.ipx;
      const int p1 = min(p0 + sg.ipx, HW);
      const size_t off = (static_cast<size_t>(b) * HW) * cv + cvec;
      const uint4* xb = sg.x + off;
      uint4* yb = sg.y + off;
      int p = p0 + prow;
      for (; p + (kFuApplyUnroll - 1) * rpb < p1; p += kFuApplyUnroll * rpb) {
        uint4 u[kFuApplyUnroll];
#pragma unroll
        for (int k = 0; k < kFuApplyUnroll; ++k) u[k] = xb[static_cast<size_t>(p + k * rpb) * cv];
#pragma unroll
        for (int k = 0; k < kFuApplyUnroll; ++k) {
          const uint4 v = process(u[k], p + k * rpb);
          if (!keep_vec) yb[static_cast<size_t>(p + k * rpb) * cv] = v;
        }
      }
      for (; p < p1; p += rpb) {
        const uint4 v = process(xb[static_cast<size_t>(p) * cv], p);
        if (!keep_vec) yb[static_cast<size_t>(p) * cv] = v;
      }
    }
    flush(b);
  }
}

}  // namespace ds

namespace {
bool fu_shape_ok(int B, int H, int W, int C) {
  return B > 0 && H > 0 && W > 0 && H <= ds::kFuMaxSide && W <= ds::kFuMaxSide && C > 0 && C % 8 == 0 &&
         C <= 8 * ds::kGnStatsThreads;
}
bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// gridDim.x of a launch with `ny` rows of CTAs: ny * gridDim.x CTAs are one resident wave (at most 2 CTAs per SM),
// and a row never has more CTAs than items
int fu_grid(const void* fn, int threads, size_t smem, int items, int num_sms, int ny) {
  int occ = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, threads, smem) != cudaSuccess || occ < 1) {
    (void)cudaGetLastError();
    occ = 1;
  }
  if (occ > 2) occ = 2;
  long long g = static_cast<long long>(occ) * num_sms / ny;
  if (g < 1) g = 1;
  return static_cast<int>(g < items ? g : items);
}

// dynamic shared memory beyond the 48 KB default: opted in once per device and kernel
cudaError_t fu_smem_attr(const void* fn, size_t smem, size_t* attr) {
  if (smem > 48 * 1024 && smem > attr[ds::device_slot()]) {
    const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    attr[ds::device_slot()] = smem;
  }
  return cudaSuccess;
}
}  // namespace

extern "C" int ds_freeu_moments(const void* skip, double* moments, int B, int H, int W, int C, void* stream) {
  using namespace ds;
  DS_REQUIRE(skip && moments, "ds_freeu_moments: NULL pointer");
  DS_REQUIRE(fu_shape_ok(B, H, W, C), "ds_freeu_moments: bad shape (C %% 8 == 0, C <= 4096, H, W <= 2048)");
  DS_REQUIRE(aligned16(skip) && (reinterpret_cast<uintptr_t>(moments) & 7) == 0,
             "ds_freeu_moments: skip must be 16-byte and moments 8-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  GnPlan pl;
  DS_REQUIRE(gn_plan(B, H * W, C, kGnStatsThreads, kFuMomSweeps, &pl), "ds_freeu_moments: tensor too large");
  const size_t smem = static_cast<size_t>(H + W) * sizeof(float2) + static_cast<size_t>(pl.rpb) * C * 7 * sizeof(float);
  static size_t attr[kMaxDevices] = {};
  const void* fn = reinterpret_cast<const void*>(freeu_moments_kernel);
  DS_CUDA_OK(fu_smem_attr(fn, smem, attr));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(fu_grid(fn, pl.threads, smem, pl.total_items, dev.num_sms, 1));
  cfg.blockDim = dim3(pl.threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute la[1];
  pdl_attr(&la[0]);
  cfg.attrs = la;
  cfg.numAttrs = 1;
  DS_CUDA_OK(cudaLaunchKernelEx(&cfg, freeu_moments_kernel, static_cast<const uint4*>(skip), moments, H, W, C,
                                pl.items_per_sample, pl.ipx, pl.total_items));
  DS_LAUNCH_OK("freeu_moments_kernel");
  return DS_OK;
}

extern "C" int ds_freeu_apply(const void* skip, const double* moments, void* skip_out, double* skip_stats, int C_skip,
                              const void* hidden, void* hidden_out, double* hidden_stats, int C_hidden, float s,
                              float b, int B, int H, int W, void* stream) {
  using namespace ds;
  DS_REQUIRE(skip && moments && skip_out && skip_stats && hidden && hidden_out && hidden_stats,
             "ds_freeu_apply: NULL pointer");
  DS_REQUIRE(fu_shape_ok(B, H, W, C_skip) && fu_shape_ok(B, H, W, C_hidden),
             "ds_freeu_apply: bad shape (C_skip, C_hidden %% 8 == 0 and <= 4096, H, W <= 2048)");
  DS_REQUIRE(aligned16(skip) && aligned16(skip_out) && aligned16(hidden) && aligned16(hidden_out) &&
                 aligned16(skip_stats) && aligned16(hidden_stats) && (reinterpret_cast<uintptr_t>(moments) & 7) == 0,
             "ds_freeu_apply: tensors / statistics must be 16-byte and moments 8-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  FuApplyParams P = {};
  const int Cs[2] = {C_skip, C_hidden};
  const void* xs[2] = {skip, hidden};
  void* ys[2] = {skip_out, hidden_out};
  double* sts[2] = {skip_stats, hidden_stats};
  int threads = 0, items = 0;
  size_t smem = 0;
  for (int g = 0; g < 2; ++g) {
    GnPlan pl;
    DS_REQUIRE(gn_plan(B, H * W, Cs[g], kGnStatsThreads, kGnStatsSweeps, &pl), "ds_freeu_apply: tensor too large");
    P.seg[g] = FuSeg{static_cast<const uint4*>(xs[g]), static_cast<uint4*>(ys[g]), sts[g], Cs[g], pl.threads, pl.rpb,
                     pl.ipx, pl.items_per_sample, pl.total_items};
    threads = pl.threads > threads ? pl.threads : threads;
    items = pl.total_items > items ? pl.total_items : items;
    const size_t sm = (g == 0 ? static_cast<size_t>(H + W) * sizeof(float2) : 0) +
                      static_cast<size_t>(pl.rpb) * Cs[g] * 2 * sizeof(float);
    smem = sm > smem ? sm : smem;
  }
  P.mom = moments;
  P.kscale = (1.0 - static_cast<double>(s)) / (static_cast<double>(H) * W);
  P.b = b;
  P.H = H;
  P.W = W;
  P.half = C_hidden / 2;
  static size_t attr[kMaxDevices] = {};
  const void* fn = reinterpret_cast<const void*>(freeu_apply_kernel);
  DS_CUDA_OK(fu_smem_attr(fn, smem, attr));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(fu_grid(fn, threads, smem, items, dev.num_sms, 2), 2);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute la[1];
  pdl_attr(&la[0]);
  cfg.attrs = la;
  cfg.numAttrs = 1;
  DS_CUDA_OK(cudaLaunchKernelEx(&cfg, freeu_apply_kernel, P));
  DS_LAUNCH_OK("freeu_apply_kernel");
  return DS_OK;
}
