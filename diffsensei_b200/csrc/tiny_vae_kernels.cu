// tiny_vae_kernels.cu — the decoder of the tiny SDXL autoencoder (TAESDXL: diffusers' AutoencoderTiny / DecoderTiny).
//
// DecoderTiny is a first conv (4 -> 64) and then nothing but 3x3 convs with 64 input channels: 64 -> 64 (+ bias, + ReLU,
// + the block's skip), the nearest-x2 upsample's conv (no bias), and the final 64 -> 3 conv.  Three kernels cover it:
//
//   ds_tiny_latent_in : x = latents * inv_scale (`latents / scaling_factor`), tanh(x / 3) * 3 (DecoderTiny's latent
//                       clamp) -> conv 4 -> 64 + bias -> ReLU; fp32 NCHW latents in, bf16 NHWC out; CUDA cores
//                       (K = 36), one pass.
//   ds_tiny_conv64    : 3x3 / pad 1 conv, 64 -> 64 channels, bf16 NHWC, on wgmma (fp32 accumulation).  Epilogue: fp32
//                       bias, bf16 residual (same shape as the output), ReLU last — any combination.  upsample2:
//                       conv3x3(nearest_x2(x)) as four 2x2 phase convs of x (weights.pack_conv3x3_up2), the upsampled
//                       tensor never written.
//   ds_tiny_conv_out  : the 64 -> 3 conv + bias on the same kernel with an 8-column MMA (filter rows 3..7 zero).
//
// tiny_conv_kernel<N, UP2>: one persistent CTA per SM, 384 threads.  Warpgroup 0 is the producer (one lane drives TMA),
// warpgroups 1-2 are the consumers.  At start the producer loads the WHOLE packed filter into shared memory (9 taps x
// [N][64] bf16 = 72 KiB for N = 64; 4 phases x 4 taps = 128 KiB with UP2), where it stays for the CTA's lifetime.  Then
// the CTA walks its work items (static round-robin: item = (tile, phase), tile = 8 x 16 output pixels of one image,
// or low-res pixels of one upsample phase) and streams, per filter tap, the tap's shifted 8 x 16 x 64 input box
// through a multi-stage ring of 16 KiB stages (4-D TMA tensor map over the NHWC input; its out-of-bounds zero fill is
// the conv's padding, and masks partial tiles).  Each consumer warpgroup owns 64 of the tile's 128 pixels: per tap
// four wgmma m64nNk16 against the resident filter slice, the stage freed once the MMAs that read it retired.  The
// epilogue runs from the accumulator registers and stores bf16 straight to global memory, while the producer already
// fills the ring with the next item's taps.
// Every output element is one item's fixed-order K loop: no split-K and no batch-dependent schedule, so an image's
// output bits do not depend on the batch around it.
#include "ds_common.cuh"
#include "ds_host.h"
#include "wgmma.cuh"

namespace ds {

constexpr int kTinyThreads = 384;      // warpgroup 0: TMA producer; warpgroups 1-2: MMA + epilogue
constexpr int kTinyConsumers = 256;
constexpr int kTinyTileH = 8;
constexpr int kTinyTileW = 16;         // 128 pixels per tile
constexpr int kTinyC = 64;             // input channels: one 64-wide k-block per filter tap
constexpr int kTinyABytes = kTinyTileH * kTinyTileW * kTinyC * 2;   // 16 KiB per ring stage
constexpr int kTinySmemLimit = 232448;  // sm_90 opt-in limit: 227 KiB

template <int N, bool UP2>
struct TinyCfg {
  static constexpr int kPhases = UP2 ? 4 : 1;
  static constexpr int kTaps = UP2 ? 4 : 9;
  static constexpr int kTapsX = UP2 ? 2 : 3;
  static constexpr int kSliceBytes = N * kTinyC * 2;                  // one tap of the filter, [N][64] bf16
  static constexpr int kFilterBytes = kPhases * kTaps * kSliceBytes;
  static constexpr int kFixedBytes = 1024 /*align slack*/ + 256 /*barriers*/;
  static constexpr int kFit = (kTinySmemLimit - kFilterBytes - kFixedBytes) / kTinyABytes;
  static constexpr int kStages = kFit > 8 ? 8 : kFit;
  static constexpr int kSmemBytes = kFilterBytes + kStages * kTinyABytes + kFixedBytes;
  static_assert(kStages >= 4, "ring too shallow");
  static_assert(kSliceBytes % 1024 == 0, "filter slices must keep the 1024-byte swizzle alignment");
};

struct TinyConvParams {
  const float* bias;                  // [n_out] fp32 or NULL
  const __nv_bfloat16* residual;      // same shape as out, or NULL
  __nv_bfloat16* out;                 // [B][Ho][Wo][n_out]
  int B, H, W;                        // input geometry
  int tiles_x, tiles_y, num_items;
  int n_out;                          // output channels written (64, or 3 for the output conv)
  int relu;
};

struct TinyConvLaunch {
  CUtensorMap tm_x;                   // 4-D {64, W, H, B}, box {64, 16, 8, 1}
  CUtensorMap tm_w;                   // 2-D {taps * 64, phases * N}, box {64, N}
  TinyConvParams p;
};

// D[64 x 8] (+)= A(smem) * B(smem), both K-major; scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_m64n8_ss(float* d, uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %6, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 {%0, %1, %2, %3}, %4, %5, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

template <int N>
__device__ __forceinline__ void tiny_mma(float* acc, uint64_t adesc, uint64_t bdesc, int scale_d) {
  if constexpr (N == 64)
    wgmma_m64n64_ss(acc, adesc, bdesc, scale_d);
  else
    wgmma_m64n8_ss(acc, adesc, bdesc, scale_d);
}

// item -> (image, tile origin y0 / x0 in input pixels, phase)
__device__ __forceinline__ void tiny_item(const TinyConvParams& p, int phases, int item, int& img, int& y0, int& x0,
                                          int& ph) {
  ph = item % phases;
  const int tile = item / phases;
  const int per_img = p.tiles_x * p.tiles_y;
  img = tile / per_img;
  const int rem = tile - img * per_img;
  y0 = (rem / p.tiles_x) * kTinyTileH;
  x0 = (rem % p.tiles_x) * kTinyTileW;
}

template <int N, bool UP2>
__global__ void __launch_bounds__(kTinyThreads, 1) tiny_conv_kernel(const __grid_constant__ TinyConvLaunch L) {
  using Cfg = TinyCfg<N, UP2>;
  constexpr int STAGES = Cfg::kStages;
  constexpr int ACC = N / 2;          // fp32 accumulator registers per consumer thread (64 rows x N per warpgroup)
  const TinyConvParams& p = L.p;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sW = smem;                                   // [phases * taps][N][64] bf16, 128-B swizzled
  uint8_t* sA = smem + Cfg::kFilterBytes;               // [STAGES][128][64] bf16, 128-B swizzled
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sA + STAGES * kTinyABytes);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* w_bar = empty_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&L.tm_x);
    tma_prefetch_desc(&L.tm_w);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kTinyConsumers);  // every consumer thread arrives once its warpgroup's MMAs retired
    }
    mbar_init(w_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer (one lane)
    if (warp != 0 || lane != 0) return;
    mbar_arrive_expect_tx(w_bar, Cfg::kFilterBytes);
    for (int ph = 0; ph < Cfg::kPhases; ++ph)
      for (int t = 0; t < Cfg::kTaps; ++t)
        tma_load_2d(sW + (ph * Cfg::kTaps + t) * Cfg::kSliceBytes, &L.tm_w, w_bar, t * kTinyC, ph * N);
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < p.num_items; item += gridDim.x) {
      int img, y0, x0, ph;
      tiny_item(p, Cfg::kPhases, item, img, y0, x0, ph);
      // 3x3 / pad 1: taps at offsets -1..1; upsample phase (a, b): 2x2 taps from offset -1 (parity 0) or 0 (parity 1)
      const int off_y = UP2 ? ((ph >> 1) ? 0 : -1) : -1;
      const int off_x = UP2 ? ((ph & 1) ? 0 : -1) : -1;
      for (int t = 0; t < Cfg::kTaps; ++t) {
        const int r = t / Cfg::kTapsX, s = t - r * Cfg::kTapsX;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_arrive_expect_tx(&full_bar[stage], kTinyABytes);
        tma_load_4d(sA + stage * kTinyABytes, &L.tm_x, &full_bar[stage], 0, x0 + s + off_x, y0 + r + off_y, img);
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: MMA + epilogue
  const int ct = threadIdx.x - 128;    // consumer thread 0..255
  const int wg = ct >> 7;              // rows [64 wg, +64) of the tile
  const int cw = ct >> 5;              // consumer warp 0..7: rows [16 cw, +16)
  const int cq = 2 * (lane & 3);       // first of the two columns this thread holds in every 8-column block
  int r_loc[2];                        // the two tile rows this thread holds (cw already counts the warpgroup's 64)
  r_loc[0] = cw * 16 + (lane >> 2);
  r_loc[1] = r_loc[0] + 8;
  const uint32_t a_base = smem_u32(sA) + static_cast<uint32_t>(wg) * 64 * 128;
  const uint32_t w_base = smem_u32(sW);
  float bias[N / 8][2];
#pragma unroll
  for (int j = 0; j < N / 8; ++j)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int c = 8 * j + cq + e;
      bias[j][e] = (p.bias && c < p.n_out) ? __ldg(p.bias + c) : 0.0f;
    }
  const int Ho = UP2 ? 2 * p.H : p.H, Wo = UP2 ? 2 * p.W : p.W;
  float acc[ACC];
  int stage = 0;
  uint32_t phase = 0;
  mbar_wait(w_bar, 0);                 // the filter is resident
  for (int item = blockIdx.x; item < p.num_items; item += gridDim.x) {
    int img, y0, x0, ph;
    tiny_item(p, Cfg::kPhases, item, img, y0, x0, ph);
    const uint32_t w_item = w_base + ph * Cfg::kTaps * Cfg::kSliceBytes;
    int prev = -1;
    for (int t = 0; t < Cfg::kTaps; ++t) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_addr = a_base + stage * kTinyABytes;
      const uint32_t b_addr = w_item + t * Cfg::kSliceBytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kTinyC / 16; ++k)
        tiny_mma<N>(acc, make_wgmma_desc(a_addr + k * 32, 1024, 16), make_wgmma_desc(b_addr + k * 32, 1024, 16),
                    (t != 0 || k != 0) ? 1 : 0);
      wgmma_commit();
      wgmma_wait<1>();                 // the previous tap's MMAs have retired: its stage may be refilled
      if (prev >= 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    fence_regs<ACC>(acc);
    mbar_arrive(&empty_bar[prev]);

    // epilogue: acc + bias (+ residual), ReLU last, one rounding to bf16
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r_loc[h];         // tile row = output pixel (y0 + r / 16, x0 + r % 16)
      const int py = y0 + r / kTinyTileW, px = x0 + r % kTinyTileW;
      if (py >= p.H || px >= p.W) continue;
      const int oy = UP2 ? 2 * py + (ph >> 1) : py;
      const int ox = UP2 ? 2 * px + (ph & 1) : px;
      const size_t o = ((static_cast<size_t>(img) * Ho + oy) * Wo + ox) * p.n_out;
#pragma unroll
      for (int j = 0; j < N / 8; ++j) {
        const int c = 8 * j + cq;
        float v0 = acc[4 * j + 2 * h] + bias[j][0];
        float v1 = acc[4 * j + 2 * h + 1] + bias[j][1];
        if constexpr (N == 64) {
          if (p.residual) {
            const uint32_t rv = __ldg(reinterpret_cast<const unsigned int*>(p.residual + o + c));
            v0 += bf16_lo(rv);
            v1 += bf16_hi(rv);
          }
          if (p.relu) {
            v0 = fmaxf(v0, 0.0f);
            v1 = fmaxf(v1, 0.0f);
          }
          *reinterpret_cast<uint32_t*>(p.out + o + c) = pack_bf16(v0, v1);
        } else {
          if (p.relu) {
            v0 = fmaxf(v0, 0.0f);
            v1 = fmaxf(v1, 0.0f);
          }
          if (c < p.n_out) p.out[o + c] = __float2bfloat16_rn(v0);
          if (c + 1 < p.n_out) p.out[o + c + 1] = __float2bfloat16_rn(v1);
        }
      }
    }
  }
}

template <int N, bool UP2>
static int launch_tiny_conv(const void* x, const void* w, const TinyConvParams& p_in, cudaStream_t stream,
                            const char* name) {
  using Cfg = TinyCfg<N, UP2>;
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  TinyConvLaunch L;
  {
    const uint64_t dims[4] = {static_cast<uint64_t>(kTinyC), static_cast<uint64_t>(p_in.W),
                              static_cast<uint64_t>(p_in.H), static_cast<uint64_t>(p_in.B)};
    const uint64_t strides[3] = {static_cast<uint64_t>(kTinyC) * 2, static_cast<uint64_t>(p_in.W) * kTinyC * 2,
                                 static_cast<uint64_t>(p_in.H) * p_in.W * kTinyC * 2};
    const uint32_t box[4] = {kTinyC, kTinyTileW, kTinyTileH, 1};
    if (!encode_tmap_bf16(&L.tm_x, x, 4, dims, strides, box, nullptr)) return DS_ERR_CUDA;
  }
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(Cfg::kTaps * kTinyC), static_cast<uint64_t>(Cfg::kPhases * N)};
    const uint64_t strides[1] = {static_cast<uint64_t>(Cfg::kTaps * kTinyC) * 2};
    const uint32_t box[2] = {kTinyC, N};
    if (!encode_tmap_bf16(&L.tm_w, w, 2, dims, strides, box, nullptr)) return DS_ERR_CUDA;
  }
  L.p = p_in;
  L.p.tiles_x = (p_in.W + kTinyTileW - 1) / kTinyTileW;
  L.p.tiles_y = (p_in.H + kTinyTileH - 1) / kTinyTileH;
  const long long items = static_cast<long long>(p_in.B) * L.p.tiles_x * L.p.tiles_y * Cfg::kPhases;
  DS_REQUIRE(items < (1ll << 31), "%s: too many tiles (%lld)", name, items);
  L.p.num_items = static_cast<int>(items);
  const int slot = device_slot();
  static bool attr_set[kMaxDevices] = {};  // per device; benign race: idempotent
  if (!attr_set[slot]) {
    DS_CUDA_OK(cudaFuncSetAttribute(tiny_conv_kernel<N, UP2>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    Cfg::kSmemBytes));
    attr_set[slot] = true;
  }
  const int grid = L.p.num_items < dev.num_sms ? L.p.num_items : dev.num_sms;
  tiny_conv_kernel<N, UP2><<<grid, kTinyThreads, Cfg::kSmemBytes, stream>>>(L);
  DS_LAUNCH_OK(name);
  return DS_OK;
}

// DecoderTiny's first layer, one thread per (pixel, 8 output channels): the 3x3 x 4 neighbourhood of the clamped
// latents tanh(x * inv_scale / 3) * 3 (zero outside the image: the conv pads the clamped tensor), 36 x 8 FMAs against the
// shared-memory filter, + bias, ReLU, one 16-byte store.
__global__ void __launch_bounds__(256) tiny_latent_in_kernel(const float* __restrict__ lat, const float* __restrict__ w,
                                                             const float* __restrict__ bias, uint4* __restrict__ out,
                                                             float inv_scale, int H, int W, long long total) {
  __shared__ float sw[36][64];  // [tap * 4 + c][cout]
  __shared__ float sb[64];
  for (int i = threadIdx.x; i < 36 * 64; i += blockDim.x) {
    const int co = i / 36, k = i - co * 36;
    sw[k][co] = w[i];
  }
  if (threadIdx.x < 64) sb[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;  // (pixel, channel group)
  if (i >= total) return;
  const int cg = static_cast<int>(i & 7);
  const long long pix = i >> 3;
  const int HW = H * W;
  const long long b = pix / HW;
  const int pp = static_cast<int>(pix - b * HW);
  const int y = pp / W, x = pp - (pp / W) * W;
  const float* src = lat + b * 4 * HW;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = sb[cg * 8 + j];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int yy = y + r - 1;
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const int xx = x + s - 1;
      if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float v = __ldg(src + static_cast<size_t>(c) * HW + yy * W + xx);
        const float z = __fmul_rn(tanhf(__fdiv_rn(__fmul_rn(v, inv_scale), 3.0f)), 3.0f);
        const float* wr = sw[(r * 3 + s) * 4 + c] + cg * 8;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(wr[j], z, acc[j]);
      }
    }
  }
  uint4 o;
  o.x = pack_bf16(fmaxf(acc[0], 0.f), fmaxf(acc[1], 0.f));
  o.y = pack_bf16(fmaxf(acc[2], 0.f), fmaxf(acc[3], 0.f));
  o.z = pack_bf16(fmaxf(acc[4], 0.f), fmaxf(acc[5], 0.f));
  o.w = pack_bf16(fmaxf(acc[6], 0.f), fmaxf(acc[7], 0.f));
  out[i] = o;
}

}  // namespace ds

extern "C" int ds_tiny_latent_in(const float* latents, const float* w, const float* bias, void* out, float inv_scale,
                                 int B, int H, int W, void* stream) {
  using namespace ds;
  DS_REQUIRE(latents && w && bias && out, "ds_tiny_latent_in: NULL pointer");
  DS_REQUIRE(B > 0 && H > 0 && W > 0, "ds_tiny_latent_in: bad geometry %d x %d x %d", B, H, W);
  DS_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "ds_tiny_latent_in: out must be 16-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long total = static_cast<long long>(B) * H * W * 8;
  tiny_latent_in_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      latents, w, bias, static_cast<uint4*>(out), inv_scale, H, W, total);
  DS_LAUNCH_OK("tiny_latent_in_kernel");
  return DS_OK;
}

extern "C" int ds_tiny_conv64(const void* x, const void* w, const float* bias, const void* residual, void* out, int B,
                              int H, int W, int relu, int upsample2, void* stream) {
  using namespace ds;
  DS_REQUIRE(x && w && out, "ds_tiny_conv64: x/w/out must be non-NULL");
  DS_REQUIRE(B > 0 && H > 0 && W > 0, "ds_tiny_conv64: bad geometry %d x %d x %d", B, H, W);
  DS_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0,
             "ds_tiny_conv64: x and w must be 16-byte aligned");
  DS_REQUIRE((reinterpret_cast<uintptr_t>(out) & 3) == 0 && (reinterpret_cast<uintptr_t>(residual) & 3) == 0,
             "ds_tiny_conv64: out and residual must be 4-byte aligned");
  TinyConvParams p{};
  p.bias = bias;
  p.residual = static_cast<const __nv_bfloat16*>(residual);
  p.out = static_cast<__nv_bfloat16*>(out);
  p.B = B;
  p.H = H;
  p.W = W;
  p.n_out = 64;
  p.relu = relu != 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (upsample2) return launch_tiny_conv<64, true>(x, w, p, st, "tiny_conv_kernel<64, up2>");
  return launch_tiny_conv<64, false>(x, w, p, st, "tiny_conv_kernel<64>");
}

extern "C" int ds_tiny_conv_out(const void* x, const void* w, const float* bias, void* out, int B, int H, int W,
                                void* stream) {
  using namespace ds;
  DS_REQUIRE(x && w && bias && out, "ds_tiny_conv_out: NULL pointer");
  DS_REQUIRE(B > 0 && H > 0 && W > 0, "ds_tiny_conv_out: bad geometry %d x %d x %d", B, H, W);
  DS_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0,
             "ds_tiny_conv_out: x and w must be 16-byte aligned");
  TinyConvParams p{};
  p.bias = bias;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.B = B;
  p.H = H;
  p.W = W;
  p.n_out = 3;
  return launch_tiny_conv<8, false>(x, w, p, static_cast<cudaStream_t>(stream), "tiny_conv_kernel<8>");
}
