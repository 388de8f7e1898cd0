// vae_kernels.cu — the three small kernels the AutoencoderKL decoder needs beyond the UNet's (everything else in the
// decoder — 3x3 convs, GroupNorm+SiLU, linears, nearest upsample — runs on the kernels in gemm_wgmma.cu /
// norm_kernels.cu / glue_kernels.cu):
//   ds_latent_pointwise : latents / scaling_factor -> post_quant_conv (1x1, 4 -> 4) -> NHWC bf16
//                         (src/pipelines/pipeline_diffsensei.py:346-361; diffusers AutoencoderKL.decode)
//   ds_softmax_rows     : P = softmax(scale * S) row-wise, fp32 scores in, bf16 probabilities out — the mid-block
//                         attention of the decoder has ONE head of width 512 over all H*W tokens (no flash kernel for
//                         that head size: QK^T and PV run as plain wgmma GEMMs with this kernel between them)
//   ds_image_postprocess: (x / 2 + 0.5).clamp(0, 1), NHWC bf16 -> NCHW fp32 (VaeImageProcessor.postprocess/denormalize)
// and one the encoder needs after its conv_out:
//   ds_vae_posterior    : quant_conv (1x1, 8 -> 8) -> DiagonalGaussianDistribution sample / mode -> * scaling_factor
//                         -> repeat to num_samples -> scheduler.add_noise (diffusers AutoencoderKL.encode and
//                         StableDiffusionXLImg2ImgPipeline.prepare_latents)
// All four are HBM-bound one-pass kernels.
#include "ds_common.cuh"
#include "ds_host.h"

namespace ds {

__global__ void latent_pointwise_kernel(const float* __restrict__ lat, const float* __restrict__ w,
                                        const float* __restrict__ bias, uint2* __restrict__ out, float inv_scale,
                                        int HW, long long total) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;  // pixel of (batch, hw)
  if (i >= total) return;
  const long long b = i / HW;
  const int p = static_cast<int>(i - b * HW);
  const float* src = lat + b * 4 * HW + p;  // NCHW fp32
  float z[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) z[c] = src[static_cast<size_t>(c) * HW] * inv_scale;
  float o[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float a = bias ? __ldg(bias + k) : 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) a = fmaf(__ldg(w + k * 4 + c), z[c], a);
    o[k] = a;
  }
  out[i] = make_uint2(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]));
}

// One CTA per row; the row lives in registers (kPer values per thread), so S is read once and P written once.
template <int kPer>
__global__ void __launch_bounds__(512) softmax_rows_kernel(const float* __restrict__ S, __nv_bfloat16* __restrict__ P,
                                                            int n, long long lds, long long ldp, float scale_log2) {
  __shared__ float red[16];
  const float* s = S + static_cast<long long>(blockIdx.x) * lds;
  __nv_bfloat16* pr = P + static_cast<long long>(blockIdx.x) * ldp;
  float v[kPer];
  float m = -INFINITY;
#pragma unroll
  for (int k = 0; k < kPer; ++k) {
    const int i = threadIdx.x + k * 512;
    v[k] = i < n ? s[i] * scale_log2 : -INFINITY;
    m = fmaxf(m, v[k]);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  m = warp_max(m);
  if (lane == 0) red[warp] = m;
  __syncthreads();
  m = red[lane & 15];
  m = warp_max(m);
  __syncthreads();
  float l = 0.f;
#pragma unroll
  for (int k = 0; k < kPer; ++k) {
    v[k] = exp2f(v[k] - m);  // -inf -> 0 beyond n
    l += v[k];
  }
  l = warp_sum(l);
  if (lane == 0) red[warp] = l;
  __syncthreads();
  l = red[lane & 15];
  l = warp_sum(l) * 0.5f;  // lanes 16..31 re-read the 16 partials: every partial was counted twice
  const float inv = 1.0f / l;
#pragma unroll
  for (int k = 0; k < kPer; ++k) {
    const int i = threadIdx.x + k * 512;
    if (i < n) pr[i] = __float2bfloat16(v[k] * inv);
  }
}

__global__ void image_postprocess_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ out, int HW, int C,
                                         long long total) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;  // index into NCHW output
  if (i >= total) return;
  const int p = static_cast<int>(i % HW);
  const long long bc = i / HW;
  const int c = static_cast<int>(bc % C);
  const long long b = bc / C;
  const float v = __bfloat162float(x[(b * HW + p) * C + c]);
  out[i] = fminf(fmaxf(fmaf(v, 0.5f, 0.5f), 0.f), 1.f);
}

// The AutoencoderKL posterior from the encoder's conv_out (fp32 NHWC [B][HW][8]), one pixel per thread:
//   moments = quant_conv(x) (1x1, 8 -> 8, fp32), mean = moments[0:4], logvar = clamp(moments[4:8], -30, 20),
//   z = mean + exp(0.5 * logvar) * eps (eps NULL: z = mean, DiagonalGaussianDistribution.mode()), z *= scale,
//   then for each of the `repeat` copies r: out[b * repeat + r] = c0 * z + c1 * noise[b * repeat + r] (noise NULL:
//   out = z).  Each fp32 operation is rounded on its own, as torch's eager ops are.  All planes fp32 NCHW.
__global__ void vae_posterior_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                     const float* __restrict__ bias, const float* __restrict__ eps, float scale,
                                     const float* __restrict__ noise, const float* __restrict__ coef, int repeat,
                                     float* __restrict__ mean_out, float* __restrict__ logvar_out,
                                     float* __restrict__ out, int HW, long long total) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;  // pixel of (batch, hw)
  if (i >= total) return;
  const long long b = i / HW;
  const long long p = i - b * HW;
  const float4* src = reinterpret_cast<const float4*>(x + i * 8);
  const float4 u0 = src[0], u1 = src[1];
  const float in[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
  float m[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    float a = __ldg(bias + k);
#pragma unroll
    for (int c = 0; c < 8; ++c) a = fmaf(__ldg(w + k * 8 + c), in[c], a);
    m[k] = a;
  }
  float c0 = 1.0f, c1 = 0.0f;
  if (noise) {
    c0 = __ldg(coef);
    c1 = __ldg(coef + 1);
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const long long at = (b * 4 + c) * HW + p;
    const float mu = m[c];
    const float lv = fminf(fmaxf(m[4 + c], -30.0f), 20.0f);
    if (mean_out) mean_out[at] = mu;
    if (logvar_out) logvar_out[at] = lv;
    float z = mu;
    if (eps) z = __fadd_rn(mu, __fmul_rn(expf(__fmul_rn(0.5f, lv)), eps[at]));
    z = __fmul_rn(scale, z);
    if (!out) continue;
    for (int r = 0; r < repeat; ++r) {
      const long long o = ((b * repeat + r) * 4 + c) * HW + p;
      out[o] = noise ? __fadd_rn(__fmul_rn(c0, z), __fmul_rn(c1, noise[o])) : z;
    }
  }
}

}  // namespace ds

extern "C" int ds_latent_pointwise(const float* latents, const float* w, const float* bias, void* out,
                                   float inv_scale, int B, int HW, void* stream) {
  using namespace ds;
  DS_REQUIRE(latents && w && out && B > 0 && HW > 0, "ds_latent_pointwise: bad arguments");
  DS_REQUIRE((reinterpret_cast<uintptr_t>(out) & 7) == 0, "ds_latent_pointwise: out must be 8-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long total = static_cast<long long>(B) * HW;
  latent_pointwise_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      latents, w, bias, static_cast<uint2*>(out), inv_scale, HW, total);
  DS_LAUNCH_OK("latent_pointwise_kernel");
  return DS_OK;
}

extern "C" int ds_softmax_rows(const float* S, void* P, int rows, int n, int64_t lds, int64_t ldp, float scale,
                               void* stream) {
  using namespace ds;
  DS_REQUIRE(S && P && rows > 0 && n > 0 && lds >= n && ldp >= n, "ds_softmax_rows: bad arguments");
  DS_REQUIRE(n <= 512 * 64, "ds_softmax_rows: rows longer than 32768 are not supported (got %d)", n);
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const float sl2 = scale * 1.4426950408889634f;
  __nv_bfloat16* p = static_cast<__nv_bfloat16*>(P);
  const int per = (n + 511) / 512;
#define DS_SM_CASE(K) softmax_rows_kernel<K><<<rows, 512, 0, st>>>(S, p, n, lds, ldp, sl2)
  if (per <= 1) DS_SM_CASE(1);
  else if (per <= 2) DS_SM_CASE(2);
  else if (per <= 4) DS_SM_CASE(4);
  else if (per <= 8) DS_SM_CASE(8);
  else if (per <= 16) DS_SM_CASE(16);
  else if (per <= 32) DS_SM_CASE(32);
  else DS_SM_CASE(64);
#undef DS_SM_CASE
  DS_LAUNCH_OK("softmax_rows_kernel");
  return DS_OK;
}

extern "C" int ds_image_postprocess(const void* x, float* out, int B, int HW, int C, void* stream) {
  using namespace ds;
  DS_REQUIRE(x && out && B > 0 && HW > 0 && C > 0, "ds_image_postprocess: bad arguments");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long total = static_cast<long long>(B) * HW * C;
  image_postprocess_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), out, HW, C, total);
  DS_LAUNCH_OK("image_postprocess_kernel");
  return DS_OK;
}

extern "C" int ds_vae_posterior(const float* x, const float* w, const float* bias, const float* eps, float scale,
                                const float* noise, const float* coef, int repeat, float* mean, float* logvar,
                                float* out, int B, int HW, void* stream) {
  using namespace ds;
  DS_REQUIRE(x && w && bias && B > 0 && HW > 0 && repeat >= 1 && (mean || logvar || out),
             "ds_vae_posterior: bad arguments");
  DS_REQUIRE(!noise || (coef && out), "ds_vae_posterior: noise needs coef and out");
  DS_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "ds_vae_posterior: x must be 16-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long total = static_cast<long long>(B) * HW;
  vae_posterior_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, w, bias, eps, scale, noise, coef, repeat, mean, logvar, out, HW, total);
  DS_LAUNCH_OK("vae_posterior_kernel");
  return DS_OK;
}
