// adapter_kernels.cu — the SDXL T2I-Adapter (diffusers' T2IAdapter, adapter_type "full_adapter_xl") on channels-last
// bf16 (HBM-bound).
//
// The adapter network runs once per panel; its 3x3 convs are ds_conv3x3_nhwc and its 1x1 convs (+ residual)
// ds_gemm_bf16.  What those do not cover:
//   adapter_relu_kernel    : AdapterResnetBlock.act, nn.ReLU between block1 and block2.
//   adapter_avgpool_kernel : AdapterBlock.downsample, nn.AvgPool2d(2, 2, ceil_mode=True) without padding: the window
//                            of a partial edge is divided by its in-bounds pixel count, as torch does.
//   adapter_add_kernel     : the per-step hot path, UNet2DConditionModel's `sample += down_intrablock_residual`, in
//                            place, with the GroupNorm statistics of the result in chan_stats_kernel's items and fp32
//                            partials (the next GroupNorm reads them; the producer's are stale), so they equal
//                            ds_channel_stats of the output bit for bit.
// The preprocess (Pillow LANCZOS, / 255, PixelUnshuffle(16)) is the adapter epilogue of ds_vae_preprocess.
#include "ds_common.cuh"
#include "ds_host.h"

namespace ds {

constexpr int kAdUnroll = 2;  // independent 16-byte loads of h and f in flight per thread

__global__ void adapter_relu_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, long long n_vec) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_vec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 u = x[i];
    uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      // a negative half (sign bit set, not NaN) becomes +0; NaN propagates as in torch.relu
      uint32_t o = 0;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const uint32_t h = (w[j] >> (16 * e)) & 0xffffu;
        const bool neg = (h & 0x8000u) && (h & 0x7fffu) <= 0x7f80u;
        o |= (neg ? 0u : h) << (16 * e);
      }
      w[j] = o;
    }
    y[i] = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

// one thread per (output pixel, 8-channel vector); the window sum in torch's order (row by row), in fp32, / count
__global__ void adapter_avgpool_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int H, int W, int Ho,
                                       int Wo, int cv, long long total) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % cv);
    const long long px = i / cv;
    const int ox = static_cast<int>(px % Wo);
    const long long r = px / Wo;
    const int oy = static_cast<int>(r % Ho);
    const long long b = r / Ho;
    const int y0 = 2 * oy, x0 = 2 * ox, y1 = min(y0 + 2, H), x1 = min(x0 + 2, W);
    float acc[8] = {};
    for (int yy = y0; yy < y1; ++yy)
      for (int xx = x0; xx < x1; ++xx) {
        const uint4 u = x[((b * H + yy) * W + xx) * cv + c];
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          acc[2 * j] += bf16_lo(w[j]);
          acc[2 * j + 1] += bf16_hi(w[j]);
        }
      }
    const float n = static_cast<float>((y1 - y0) * (x1 - x0));
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = pack_bf16(__fdiv_rn(acc[2 * j], n), __fdiv_rn(acc[2 * j + 1], n));
    y[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

struct AdAddParams {
  uint4* h;              // [B][HW][C], updated in place
  const uint4* f;        // [F][HW][C]
  double* stats;         // fp64 [B][C][2], accumulated
  const float* gate;     // device scalar
  int HW, C, F, row0, rpb, ipx, items_per_sample, total_items;
};

__global__ void __launch_bounds__(kGnStatsThreads) adapter_add_kernel(const AdAddParams P) {
  extern __shared__ float ad_smem[];  // [rpb][C][2]
  const int HW = P.HW, C = P.C, cv = C >> 3, rpb = P.rpb;
  const int cvec = threadIdx.x % cv, prow = threadIdx.x / cv;
  int i0, i1;
  gn_item_range(P.total_items, i0, i1);
  pdl_launch_dependents();
  pdl_wait();
  if (i0 >= i1) return;
  const float g = *P.gate;
  // identical arithmetic to chan_stats_kernel: s += v, q = fma(v, v, q) in pixel order, rows summed in order
  float s[8], q[8];
  auto process = [&](const uint4& hv, const uint4& fv) -> uint4 {
    const uint32_t a[4] = {hv.x, hv.y, hv.z, hv.w}, b[4] = {fv.x, fv.y, fv.z, fv.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      // torch's bf16 `h + f`: an fp32 add, one rounding; gate 0 leaves h as it is
      o[j] = g != 0.f ? pack_bf16(fmaf(g, bf16_lo(b[j]), bf16_lo(a[j])), fmaf(g, bf16_hi(b[j]), bf16_hi(a[j])))
                      : a[j];
      const float lo = bf16_lo(o[j]), hi = bf16_hi(o[j]);
      s[2 * j] += lo;
      q[2 * j] = fmaf(lo, lo, q[2 * j]);
      s[2 * j + 1] += hi;
      q[2 * j + 1] = fmaf(hi, hi, q[2 * j + 1]);
    }
    return make_uint4(o[0], o[1], o[2], o[3]);
  };
  auto flush = [&](int b) {
    float* row = ad_smem + (static_cast<size_t>(prow) * C + cvec * 8) * 2;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      row[2 * j] = s[j];
      row[2 * j + 1] = q[j];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      float ts = 0.f, tq = 0.f;
      for (int r = 0; r < rpb; ++r) {
        ts += ad_smem[(static_cast<size_t>(r) * C + c) * 2];
        tq += ad_smem[(static_cast<size_t>(r) * C + c) * 2 + 1];
      }
      double* gp = P.stats + (static_cast<size_t>(b) * C + c) * 2;
      atomicAdd(gp, static_cast<double>(ts));
      atomicAdd(gp + 1, static_cast<double>(tq));
    }
    __syncthreads();
  };
  for (int it = i0; it < i1; ++it) {
    const int b = it / P.items_per_sample;
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
    const int p0 = (it - b * P.items_per_sample) * P.ipx;
    const int p1 = min(p0 + P.ipx, HW);
    uint4* hb = P.h + (static_cast<size_t>(b) * HW) * cv + cvec;
    const uint4* fb = P.f + (static_cast<size_t>((b + P.row0) % P.F) * HW) * cv + cvec;
    int p = p0 + prow;
    for (; p + (kAdUnroll - 1) * rpb < p1; p += kAdUnroll * rpb) {
      uint4 hv[kAdUnroll], fv[kAdUnroll];
#pragma unroll
      for (int k = 0; k < kAdUnroll; ++k) {
        hv[k] = hb[static_cast<size_t>(p + k * rpb) * cv];
        fv[k] = __ldg(fb + static_cast<size_t>(p + k * rpb) * cv);
      }
#pragma unroll
      for (int k = 0; k < kAdUnroll; ++k) hb[static_cast<size_t>(p + k * rpb) * cv] = process(hv[k], fv[k]);
    }
    for (; p < p1; p += rpb)
      hb[static_cast<size_t>(p) * cv] =
          process(hb[static_cast<size_t>(p) * cv], __ldg(fb + static_cast<size_t>(p) * cv));
    flush(b);
  }
}

}  // namespace ds

namespace {
bool ad_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// a grid-stride launch of `total` work items: at most 8 CTAs of 256 threads per SM
unsigned ad_blocks(long long total, int num_sms) {
  const long long need = (total + 255) / 256, cap = 8LL * num_sms;
  return static_cast<unsigned>(need < 1 ? 1 : need < cap ? need : cap);
}

cudaLaunchConfig_t ad_config(unsigned grid, unsigned threads, size_t smem, void* stream, cudaLaunchAttribute* la) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = static_cast<cudaStream_t>(stream);
  ds::pdl_attr(&la[0]);
  cfg.attrs = la;
  cfg.numAttrs = 1;
  return cfg;
}
}  // namespace

extern "C" int ds_adapter_relu(const void* x, void* y, int64_t n, void* stream) {
  using namespace ds;
  DS_REQUIRE(x && y && n > 0 && n % 8 == 0, "ds_adapter_relu: bad arguments (n > 0, n %% 8 == 0)");
  DS_REQUIRE(ad_aligned16(x) && ad_aligned16(y), "ds_adapter_relu: x / y must be 16-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long nv = n / 8;
  cudaLaunchAttribute la[1];
  const cudaLaunchConfig_t cfg = ad_config(ad_blocks(nv, dev.num_sms), 256, 0, stream, la);
  DS_CUDA_OK(cudaLaunchKernelEx(&cfg, adapter_relu_kernel, static_cast<const uint4*>(x), static_cast<uint4*>(y), nv));
  DS_LAUNCH_OK("adapter_relu_kernel");
  return DS_OK;
}

extern "C" int ds_adapter_avgpool(const void* x, void* y, int B, int H, int W, int C, void* stream) {
  using namespace ds;
  DS_REQUIRE(x && y && B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0,
             "ds_adapter_avgpool: bad arguments (B, H, W > 0, C %% 8 == 0)");
  DS_REQUIRE(ad_aligned16(x) && ad_aligned16(y), "ds_adapter_avgpool: x / y must be 16-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2, cv = C / 8;
  const long long total = static_cast<long long>(B) * Ho * Wo * cv;
  cudaLaunchAttribute la[1];
  const cudaLaunchConfig_t cfg = ad_config(ad_blocks(total, dev.num_sms), 256, 0, stream, la);
  DS_CUDA_OK(cudaLaunchKernelEx(&cfg, adapter_avgpool_kernel, static_cast<const uint4*>(x), static_cast<uint4*>(y), H,
                                W, Ho, Wo, cv, total));
  DS_LAUNCH_OK("adapter_avgpool_kernel");
  return DS_OK;
}

extern "C" int ds_adapter_add(void* h, const void* f, int F, int row0, const float* gate, double* stats, int B, int HW,
                              int C, void* stream) {
  using namespace ds;
  DS_REQUIRE(h && f && gate && stats, "ds_adapter_add: NULL pointer");
  DS_REQUIRE(B > 0 && HW > 0 && F > 0 && row0 >= 0 && C > 0 && C % 8 == 0 && C <= 8 * kGnStatsThreads,
             "ds_adapter_add: bad shape (B, HW, F > 0, row0 >= 0, C %% 8 == 0, C <= 4096)");
  DS_REQUIRE(ad_aligned16(h) && ad_aligned16(f) && ad_aligned16(stats) && (reinterpret_cast<uintptr_t>(gate) & 3) == 0,
             "ds_adapter_add: h / f / stats must be 16-byte and gate 4-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  GnPlan pl;
  DS_REQUIRE(gn_plan(B, HW, C, kGnStatsThreads, kGnStatsSweeps, &pl), "ds_adapter_add: tensor too large");
  const size_t smem = static_cast<size_t>(pl.rpb) * C * 2 * sizeof(float);
  static size_t attr[kMaxDevices] = {};
  if (smem > 48 * 1024 && smem > attr[device_slot()]) {
    DS_CUDA_OK(cudaFuncSetAttribute(adapter_add_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    static_cast<int>(smem)));
    attr[device_slot()] = smem;
  }
  int occ = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, adapter_add_kernel, pl.threads, smem) != cudaSuccess ||
      occ < 1) {
    (void)cudaGetLastError();
    occ = 1;
  }
  if (occ > 2) occ = 2;
  const long long g = static_cast<long long>(occ) * dev.num_sms;
  const AdAddParams P = {static_cast<uint4*>(h), static_cast<const uint4*>(f), stats, gate, HW, C, F, row0 % F, pl.rpb,
                         pl.ipx, pl.items_per_sample, pl.total_items};
  cudaLaunchAttribute la[1];
  const cudaLaunchConfig_t cfg =
      ad_config(static_cast<unsigned>(g < pl.total_items ? g : pl.total_items), pl.threads, smem, stream, la);
  DS_CUDA_OK(cudaLaunchKernelEx(&cfg, adapter_add_kernel, P));
  DS_LAUNCH_OK("adapter_add_kernel");
  return DS_OK;
}
