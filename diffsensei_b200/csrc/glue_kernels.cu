// glue_kernels.cu — small HBM-bound kernels around the tensor-core ops: conv_in (Cin = 4), layout changes at
// the diffusers-facing boundary, nearest upsample, channel concat, SiLU, sinusoidal timestep features, and the
// fused CFG + DDIM update.  All vectorised to 16-byte accesses where the shape allows.
#include "ds_common.cuh"
#include "ds_host.h"

namespace ds {

// ------------------------------------------------------------------------------------------------
// conv_in: 3x3, pad 1, Cin = 4 -> Cout.  x NHWC bf16 (8 B / pixel), w fp32 [Cout][3][3][4].
// One thread = one pixel x 8 output channels; weights transposed into smem as [36][Cout].
// Replaces UNet2DConditionModel.conv_in (src/models/unet.py:206).
// ------------------------------------------------------------------------------------------------
__global__ void conv_in_kernel(const uint2* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                               uint4* __restrict__ out, int H, int W, int Cout, int grp_per_cta) {
  // Work item = 4 consecutive output pixels of one row x 8 output channels: every weight read from shared memory
  // feeds 4 FMAs (a one-pixel version would re-read all 36 x 8 weights per output vector from shared memory).
  extern __shared__ float sw[];  // [36][Cout] then bias [Cout]
  float* sb = sw + 36 * Cout;
  for (int i = threadIdx.x; i < 36 * Cout; i += blockDim.x) {
    const int co = i / 36, k = i - co * 36;
    sw[k * Cout + co] = w[i];
  }
  for (int i = threadIdx.x; i < Cout; i += blockDim.x) sb[i] = bias ? bias[i] : 0.f;
  __syncthreads();
  const int cv = Cout >> 3;
  const int b = blockIdx.y;
  const int HW = H * W;
  const int gpr = (W + 3) >> 2;            // 4-pixel groups per row
  const int n_grp = H * gpr;
  const int g_begin = blockIdx.x * grp_per_cta;
  const int g_end = min(g_begin + grp_per_cta, n_grp);
  const uint2* xb = x + static_cast<size_t>(b) * HW;
  for (int idx = threadIdx.x; idx < (g_end - g_begin) * cv; idx += blockDim.x) {
    const int grp = g_begin + idx / cv;
    const int cvec = idx % cv;
    const int y = grp / gpr, x0 = (grp - y * gpr) * 4;
    float acc[4][8];
#pragma unroll
    for (int px = 0; px < 4; ++px)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[px][j] = sb[cvec * 8 + j];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int iy = y + r - 1;
      if (iy < 0 || iy >= H) continue;
      float in[6][4];  // input columns x0-1 .. x0+4 of row iy (zero outside the image)
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        const int ix = x0 + c - 1;
        uint2 u = make_uint2(0u, 0u);
        if (ix >= 0 && ix < W) u = __ldg(xb + iy * W + ix);
        in[c][0] = bf16_lo(u.x);
        in[c][1] = bf16_hi(u.x);
        in[c][2] = bf16_lo(u.y);
        in[c][3] = bf16_hi(u.y);
      }
#pragma unroll
      for (int s = 0; s < 3; ++s) {
#pragma unroll
        for (int ci = 0; ci < 4; ++ci) {
          const float* wk = sw + ((r * 3 + s) * 4 + ci) * Cout + cvec * 8;
          const float4 w0 = *reinterpret_cast<const float4*>(wk);
          const float4 w1 = *reinterpret_cast<const float4*>(wk + 4);
#pragma unroll
          for (int px = 0; px < 4; ++px) {
            const float v = in[px + s][ci];
            acc[px][0] = fmaf(v, w0.x, acc[px][0]);
            acc[px][1] = fmaf(v, w0.y, acc[px][1]);
            acc[px][2] = fmaf(v, w0.z, acc[px][2]);
            acc[px][3] = fmaf(v, w0.w, acc[px][3]);
            acc[px][4] = fmaf(v, w1.x, acc[px][4]);
            acc[px][5] = fmaf(v, w1.y, acc[px][5]);
            acc[px][6] = fmaf(v, w1.z, acc[px][6]);
            acc[px][7] = fmaf(v, w1.w, acc[px][7]);
          }
        }
      }
    }
#pragma unroll
    for (int px = 0; px < 4; ++px) {
      if (x0 + px < W)
        out[(static_cast<size_t>(b) * HW + y * W + x0 + px) * cv + cvec] =
            make_uint4(pack_bf16(acc[px][0], acc[px][1]), pack_bf16(acc[px][2], acc[px][3]),
                       pack_bf16(acc[px][4], acc[px][5]), pack_bf16(acc[px][6], acc[px][7]));
    }
  }
}

// ------------------------------------------------------------------------------------------------
// NCHW <-> NHWC (small C; used for the 4-channel latents at the module boundary)
// ------------------------------------------------------------------------------------------------
template <typename SrcT>
__global__ void nchw_to_nhwc_kernel(const SrcT* __restrict__ src, __nv_bfloat16* __restrict__ dst, int C, int HW,
                                    long long total) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;  // index into dst
  if (i >= total) return;
  const int c = static_cast<int>(i % C);
  const long long bp = i / C;
  const int p = static_cast<int>(bp % HW);
  const long long b = bp / HW;
  dst[i] = __float2bfloat16(static_cast<float>(src[(b * C + c) * HW + p]));
}
template <typename DstT>
__global__ void nhwc_to_nchw_kernel(const __nv_bfloat16* __restrict__ src, DstT* __restrict__ dst, int C, int HW,
                                    long long total) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;  // index into dst
  if (i >= total) return;
  const int p = static_cast<int>(i % HW);
  const long long bc = i / HW;
  const int c = static_cast<int>(bc % C);
  const long long b = bc / C;
  dst[i] = static_cast<DstT>(__bfloat162float(src[(b * HW + p) * C + c]));
}

// ------------------------------------------------------------------------------------------------
// nearest resize (F.interpolate(mode="nearest"): src = floor(dst * in / out), computed in fp32 like ATen)
// ------------------------------------------------------------------------------------------------
__global__ void upsample_nearest_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int H, int W, int cv,
                                        int Ho, int Wo, float sh, float sw_, long long total) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = static_cast<int>(i % cv);
  long long r = i / cv;
  const int ox = static_cast<int>(r % Wo);
  r /= Wo;
  const int oy = static_cast<int>(r % Ho);
  const long long b = r / Ho;
  const int iy = min(static_cast<int>(floorf(oy * sh)), H - 1);
  const int ix = min(static_cast<int>(floorf(ox * sw_)), W - 1);
  y[i] = __ldg(x + ((b * H + iy) * W + ix) * cv + c);
}

__global__ void concat_channels_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* __restrict__ y,
                                       int cv1, int cv2, long long total) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int cv = cv1 + cv2;
  const int c = static_cast<int>(i % cv);
  const long long p = i / cv;
  y[i] = (c < cv1) ? __ldg(a + p * cv1 + c) : __ldg(b + p * cv2 + (c - cv1));
}

__global__ void silu_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, long long n) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) y[i] = __float2bfloat16(silu_f(__bfloat162float(x[i])));
}

// Timesteps(dim, flip_sin_to_cos=True, downscale_freq_shift=0): out[r] = [cos(t*w_i) | sin(t*w_i)],
// w_i = exp(-ln(10000) * i / (dim/2)).  Accurate sincosf/expf: the arguments reach ~1000 rad.
__global__ void timestep_embedding_kernel(const float* __restrict__ t, __nv_bfloat16* __restrict__ out, int rows,
                                          int dim) {
  const int half = dim >> 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * half) return;
  const int r = i / half, k = i - r * half;
  const float freq = expf(-9.210340371976184f * static_cast<float>(k) / static_cast<float>(half));
  const float arg = t[r] * freq;
  float s, c;
  sincosf(arg, &s, &c);
  out[static_cast<size_t>(r) * dim + k] = __float2bfloat16(c);
  out[static_cast<size_t>(r) * dim + half + k] = __float2bfloat16(s);
}

// ------------------------------------------------------------------------------------------------
// CFG blend + DDIM step (eta = 0, epsilon prediction), src/pipelines/pipeline_diffsensei.py:315,332-337.
// C == 4: one thread per pixel (8-byte bf16 vectors, 16-byte fp32 vector).
// ------------------------------------------------------------------------------------------------
__global__ void cfg_ddim_kernel(const uint2* __restrict__ noise_pred, float4* __restrict__ latents,
                                uint2* __restrict__ model_in, const float* __restrict__ coef, float guidance,
                                long long n_pix /* bs*HW */) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_pix) return;
  const float a_t = coef[0], a_prev = coef[1];
  const float sqrt_at = sqrtf(a_t), sqrt_1mat = sqrtf(1.0f - a_t);
  const float sqrt_ap = sqrtf(a_prev), sqrt_1map = sqrtf(1.0f - a_prev);
  const uint2 eu = __ldg(noise_pred + i);          // uncond half
  const uint2 et = __ldg(noise_pred + n_pix + i);  // text half
  const float u[4] = {bf16_lo(eu.x), bf16_hi(eu.x), bf16_lo(eu.y), bf16_hi(eu.y)};
  const float tt[4] = {bf16_lo(et.x), bf16_hi(et.x), bf16_lo(et.y), bf16_hi(et.y)};
  float4 x = latents[i];
  float xv[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float eps = u[j] + guidance * (tt[j] - u[j]);
    const float x0 = (xv[j] - sqrt_1mat * eps) / sqrt_at;
    xv[j] = sqrt_ap * x0 + sqrt_1map * eps;
  }
  latents[i] = make_float4(xv[0], xv[1], xv[2], xv[3]);
  const uint2 o = make_uint2(pack_bf16(xv[0], xv[1]), pack_bf16(xv[2], xv[3]));
  model_in[i] = o;
  model_in[n_pix + i] = o;
}

}  // namespace ds

using namespace ds;

extern "C" int ds_conv_in_3x3(const void* x, const float* w, const float* bias, void* out, int B, int H, int W,
                              int Cout, void* stream) {
  DS_REQUIRE(x && w && out, "ds_conv_in_3x3: NULL pointer");
  DS_REQUIRE(B > 0 && H > 0 && W > 0 && Cout > 0 && Cout % 8 == 0, "ds_conv_in_3x3: bad shape (Cout %% 8 == 0)");
  DS_REQUIRE(37 * Cout * 4 <= 160 * 1024, "ds_conv_in_3x3: Cout too large");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const int smem = 37 * Cout * 4;
  static bool attr_set[kMaxDevices] = {};
  if (!attr_set[device_slot()] && smem > 48 * 1024) {
    DS_CUDA_OK(cudaFuncSetAttribute(conv_in_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    attr_set[device_slot()] = true;
  }
  const int n_grp = H * ((W + 3) / 4);  // 4-pixel groups per image
  int gpc = (B * n_grp + dev.num_sms * 4 - 1) / (dev.num_sms * 4);  // ~4 CTAs per SM: amortise the weight staging
  if (gpc < 8) gpc = 8;
  dim3 grid((n_grp + gpc - 1) / gpc, B);
  conv_in_kernel<<<grid, 256, smem, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint2*>(x), w, bias, static_cast<uint4*>(out), H, W, Cout, gpc);
  DS_LAUNCH_OK("conv_in_kernel");
  return DS_OK;
}

// im2col of the 4-channel latent for a 3x3 / pad 1 conv: A[b*HW + p][tap*4 + c] = x[b][y+r-1][x+s-1][c] (zero outside
// the image), taps 0..8 = (r, s) row-major, columns 36..63 zero -> one K = 64 block of the wgmma GEMM.  16 threads
// per pixel, 8 bytes each: every 128-byte row of A is one coalesced store.
__global__ void im2col_latent_kernel(const uint2* __restrict__ x, uint2* __restrict__ a, int H, int W, long long total) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;  // (pixel, tap slot)
  if (i >= total) return;
  const int tap = static_cast<int>(i & 15);
  const long long pix = i >> 4;
  uint2 v = make_uint2(0u, 0u);
  if (tap < 9) {
    const int HW = H * W;
    const long long b = pix / HW;
    const int p = static_cast<int>(pix - b * HW);
    const int y = p / W + tap / 3 - 1, xx = p % W + tap % 3 - 1;
    if (y >= 0 && y < H && xx >= 0 && xx < W) v = __ldg(x + b * HW + static_cast<long long>(y) * W + xx);
  }
  a[i] = v;
}

extern "C" int ds_im2col_latent(const void* x, void* a, int B, int H, int W, void* stream) {
  DS_REQUIRE(x && a && B > 0 && H > 0 && W > 0, "ds_im2col_latent: bad arguments");
  DS_REQUIRE((reinterpret_cast<uintptr_t>(x) & 7) == 0 && (reinterpret_cast<uintptr_t>(a) & 7) == 0,
             "ds_im2col_latent: pointers must be 8-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long total = static_cast<long long>(B) * H * W * 16;
  im2col_latent_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint2*>(x), static_cast<uint2*>(a), H, W, total);
  DS_LAUNCH_OK("im2col_latent_kernel");
  return DS_OK;
}

extern "C" int ds_nchw_to_nhwc(const void* src, int src_is_fp32, void* dst, int B, int C, int H, int W, void* stream) {
  DS_REQUIRE(src && dst && B > 0 && C > 0 && H > 0 && W > 0, "ds_nchw_to_nhwc: bad arguments");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long total = static_cast<long long>(B) * C * H * W;
  const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (src_is_fp32)
    nchw_to_nhwc_kernel<float><<<blocks, 256, 0, st>>>(static_cast<const float*>(src),
                                                       static_cast<__nv_bfloat16*>(dst), C, H * W, total);
  else
    nchw_to_nhwc_kernel<__nv_bfloat16><<<blocks, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(src),
                                                               static_cast<__nv_bfloat16*>(dst), C, H * W, total);
  DS_LAUNCH_OK("nchw_to_nhwc_kernel");
  return DS_OK;
}

extern "C" int ds_nhwc_to_nchw(const void* src, void* dst, int dst_is_fp32, int B, int C, int H, int W, void* stream) {
  DS_REQUIRE(src && dst && B > 0 && C > 0 && H > 0 && W > 0, "ds_nhwc_to_nchw: bad arguments");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long total = static_cast<long long>(B) * C * H * W;
  const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dst_is_fp32)
    nhwc_to_nchw_kernel<float><<<blocks, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(src),
                                                       static_cast<float*>(dst), C, H * W, total);
  else
    nhwc_to_nchw_kernel<__nv_bfloat16><<<blocks, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(src),
                                                               static_cast<__nv_bfloat16*>(dst), C, H * W, total);
  DS_LAUNCH_OK("nhwc_to_nchw_kernel");
  return DS_OK;
}

extern "C" int ds_upsample_nearest(const void* x, void* y, int B, int H, int W, int C, int Ho, int Wo, void* stream) {
  DS_REQUIRE(x && y && B > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && C > 0 && C % 8 == 0,
             "ds_upsample_nearest: bad arguments (C %% 8 == 0)");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const int cv = C / 8;
  const long long total = static_cast<long long>(B) * Ho * Wo * cv;
  // ATen nearest: scale = in / out as float (exact 0.5 for the x2 case)
  const float sh = static_cast<float>(H) / static_cast<float>(Ho);
  const float sw = static_cast<float>(W) / static_cast<float>(Wo);
  upsample_nearest_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(x), static_cast<uint4*>(y), H, W, cv, Ho, Wo, sh, sw, total);
  DS_LAUNCH_OK("upsample_nearest_kernel");
  return DS_OK;
}

extern "C" int ds_concat_channels(const void* a, const void* b, void* y, int pixels, int C1, int C2, void* stream) {
  DS_REQUIRE(a && b && y && pixels > 0 && C1 > 0 && C2 > 0 && C1 % 8 == 0 && C2 % 8 == 0,
             "ds_concat_channels: bad arguments (C1, C2 %% 8 == 0)");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long total = static_cast<long long>(pixels) * ((C1 + C2) / 8);
  concat_channels_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(a), static_cast<const uint4*>(b), static_cast<uint4*>(y), C1 / 8, C2 / 8, total);
  DS_LAUNCH_OK("concat_channels_kernel");
  return DS_OK;
}

extern "C" int ds_silu(const void* x, void* y, int64_t n, void* stream) {
  DS_REQUIRE(x && y && n > 0, "ds_silu: bad arguments");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  silu_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), n);
  DS_LAUNCH_OK("silu_kernel");
  return DS_OK;
}

extern "C" int ds_timestep_embedding(const float* t, void* out, int rows, int dim, void* stream) {
  DS_REQUIRE(t && out && rows > 0 && dim > 0 && dim % 2 == 0, "ds_timestep_embedding: bad arguments");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const int total = rows * (dim / 2);
  timestep_embedding_kernel<<<(total + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      t, static_cast<__nv_bfloat16*>(out), rows, dim);
  DS_LAUNCH_OK("timestep_embedding_kernel");
  return DS_OK;
}

extern "C" int ds_cfg_ddim_step(const void* noise_pred, float* latents, void* model_in, const float* coef,
                                float guidance, int bs, int HW, int C, void* stream) {
  DS_REQUIRE(noise_pred && latents && model_in && coef, "ds_cfg_ddim_step: NULL pointer");
  DS_REQUIRE(bs > 0 && HW > 0 && C == 4, "ds_cfg_ddim_step: only C == 4 latents are supported (got C=%d)", C);
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long n_pix = static_cast<long long>(bs) * HW;
  cfg_ddim_kernel<<<static_cast<unsigned>((n_pix + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint2*>(noise_pred), reinterpret_cast<float4*>(latents), static_cast<uint2*>(model_in), coef,
      guidance, n_pix);
  DS_LAUNCH_OK("cfg_ddim_kernel");
  return DS_OK;
}
