// vae_kernels.cu — the three small kernels the AutoencoderKL decoder needs beyond the UNet's (everything else in the
// decoder — 3x3 convs, GroupNorm+SiLU, linears, nearest upsample — runs on the kernels in gemm_wgmma.cu /
// norm_kernels.cu / glue_kernels.cu):
//   ds_latent_pointwise : latents / scaling_factor -> post_quant_conv (1x1, 4 -> 4) -> NHWC bf16
//                         (src/pipelines/pipeline_diffsensei.py:346-361; diffusers AutoencoderKL.decode)
//   ds_softmax_rows     : P = softmax(scale * S) row-wise, fp32 scores in, bf16 probabilities out — the mid-block
//                         attention of the decoder has ONE head of width 512 over all H*W tokens (no flash kernel for
//                         that head size: QK^T and PV run as plain wgmma GEMMs with this kernel between them)
//   ds_image_postprocess: (x / 2 + 0.5).clamp(0, 1), NHWC bf16 -> NCHW fp32 (VaeImageProcessor.postprocess/denormalize)
// All three are HBM-bound one-pass kernels.
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
