// image_kernels.cu — the CLIP / ViT image processors of the reference (CLIPImageProcessor, ViTImageProcessor with
// their shipped defaults, src/pipelines/pipeline_diffsensei.py:70-71,125-126) on the GPU: uint8 RGB HWC images of any
// size in, the fp32 NCHW [n][3][224][224] pixel values the vision encoders read out.
//
// The resize restates Pillow's 8-bit separable resampler bit for bit (transformers' PIL backend calls
// Image.resize(size, resample) with no box and no reducing_gap):
//   per output index xx, in double:  scale = in/out, fs = max(scale, 1), support = filter_support * fs,
//     center = (xx + 0.5) * scale, xmin = max((int)(center - support + 0.5), 0),
//     xmax = min((int)(center + support + 0.5), in) - xmin, w[x] = filter((x + xmin - center + 0.5) * (1/fs)),
//     w /= sum(w) (summed in x order; skipped when the sum is 0), k[x] = (int)(w * 2^22 +- 0.5)
//   per pass: acc = 2^21 + sum u8 * k, out = clamp(acc >> 22, 0, 255); horizontal pass first into a uint8
//   intermediate, then the vertical pass; a pass whose size does not change is skipped.
// Every double / float operation is an explicit round-to-nearest intrinsic, so no FMA contraction can change a
// coefficient or a normalised value.  CLIP: shortest edge -> 224 bicubic (a = -0.5), centre crop 224 x 224 — only
// the 224 kept columns and rows are ever resampled (each output index has its own coefficients, so this is the same
// arithmetic as resize-then-crop).  ViT: 224 x 224 bilinear.  Then float32(u8 * (1/255 as double)) and
// (x - mean) / std in fp32.
//
// Three launches per batch of up to kMaxImages images: coefficient tables, horizontal pass, vertical pass fused with
// crop / rescale / normalise.  Tables and the intermediate live in the caller's scratch; the tap count per output
// index is not bounded by anything but the image size.
//
// The same resampler also serves the AutoencoderKL encoder's preprocessing (ds_vae_image_preprocess: Pillow LANCZOS
// to any size, then 2 * u8 / 255 - 1) and the inpaint mask's (ds_vae_mask_preprocess: LANCZOS on the mask's own 1 or
// 3 channels, RGB -> L, threshold), with host-built tap tables; see the section below plan_images.
#include <cuda_bf16.h>

#include <cmath>
#include <vector>

#include "ds_host.h"

namespace ds {

constexpr int kOut = 224;          // crop / resize target of both processors
constexpr int kMaxImages = 16;     // images per launch (descriptors travel as kernel parameters)
constexpr int kMaxSide = 65535;
constexpr int kPrecisionBits = 22;

struct ImgDesc {
  long long src;                       // byte offset of the image in `src`
  long long coef_h, coef_v, inter;     // byte offsets into scratch
  int H, W;                            // source size
  int rh, rw;                          // resized size (before the crop)
  int top, left;                       // crop origin in resized coordinates
  int kh, kv;                          // taps per output index of each pass; 0: pass skipped
};

struct ImgBatch {
  ImgDesc d[kMaxImages];
  int n;
  int bicubic;
};

__constant__ float kClipMean[3] = {static_cast<float>(0.48145466), static_cast<float>(0.4578275),
                                   static_cast<float>(0.40821073)};
__constant__ float kClipStd[3] = {static_cast<float>(0.26862954), static_cast<float>(0.26130258),
                                  static_cast<float>(0.27577711)};

__device__ __forceinline__ double resample_filter(double x, bool bicubic) {
  if (x < 0.0) x = -x;
  if (bicubic) {  // a = -0.5: ((a + 2) x - (a + 3)) x x + 1 on [0, 1), (((x - 5) x + 8) x - 4) a on [1, 2)
    if (x < 1.0) return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(1.5, x), 2.5), x), x), 1.0);
    if (x < 2.0) return __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(x, 5.0), x), 8.0), x), 4.0), -0.5);
    return 0.0;
  }
  return x < 1.0 ? __dsub_rn(1.0, x) : 0.0;
}

__device__ __forceinline__ int clip8(int acc) { return min(max(acc >> kPrecisionBits, 0), 255); }

// grid (n, 2 axes), kOut threads: thread t writes {xmin, xmax, k[0 .. ksize)} of output index first + t.
__global__ void image_coef_kernel(ImgBatch b, unsigned char* __restrict__ scratch) {
  const ImgDesc& d = b.d[blockIdx.x];
  const bool vert = blockIdx.y == 1;
  const int ksize = vert ? d.kv : d.kh;
  if (ksize == 0) return;
  const int in = vert ? d.H : d.W, out = vert ? d.rh : d.rw;
  const int xx = (vert ? d.top : d.left) + static_cast<int>(threadIdx.x);
  int* row = reinterpret_cast<int*>(scratch + (vert ? d.coef_v : d.coef_h)) + threadIdx.x * (2 + ksize);
  const bool bicubic = b.bicubic != 0;
  const double scale = __ddiv_rn(static_cast<double>(in), static_cast<double>(out));
  const double fs = scale < 1.0 ? 1.0 : scale;
  const double support = __dmul_rn(bicubic ? 2.0 : 1.0, fs);
  const double center = __dmul_rn(__dadd_rn(static_cast<double>(xx), 0.5), scale);
  const double ss = __ddiv_rn(1.0, fs);
  const int xmin = max(__double2int_rz(__dadd_rn(__dsub_rn(center, support), 0.5)), 0);
  const int xmax = min(min(__double2int_rz(__dadd_rn(__dadd_rn(center, support), 0.5)), in) - xmin, ksize);
  double ww = 0.0;
  for (int x = 0; x < xmax; ++x)
    ww = __dadd_rn(ww, resample_filter(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss),
                                       bicubic));
  for (int x = 0; x < xmax; ++x) {
    double w = resample_filter(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss), bicubic);
    if (ww != 0.0) w = __ddiv_rn(w, ww);
    row[2 + x] = __double2int_rz(__dadd_rn(w < 0.0 ? -0.5 : 0.5, __dmul_rn(w, static_cast<double>(1 << kPrecisionBits))));
  }
  row[0] = xmin;
  row[1] = xmax;
}

// grid (x-blocks, n): every source row, the kOut kept output columns, 3 channels -> uint8 intermediate [H][kOut][3].
__global__ void image_hpass_kernel(ImgBatch b, const unsigned char* __restrict__ src, unsigned char* __restrict__ scratch) {
  const ImgDesc& d = b.d[blockIdx.y];
  if (d.kh == 0) return;
  const long long total = static_cast<long long>(d.H) * kOut;
  const int* coef = reinterpret_cast<const int*>(scratch + d.coef_h);
  unsigned char* inter = scratch + d.inter;
  const unsigned char* img = src + d.src;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long y = i / kOut;
    const int x = static_cast<int>(i - y * kOut);
    const int* k = coef + x * (2 + d.kh);
    const int xmin = k[0], xmax = k[1];
    const unsigned char* p = img + (y * d.W + xmin) * 3;
    int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
    for (int t = 0; t < xmax; ++t) {
      const int w = k[2 + t];
      a0 += p[3 * t] * w;
      a1 += p[3 * t + 1] * w;
      a2 += p[3 * t + 2] * w;
    }
    unsigned char* o = inter + i * 3;
    o[0] = static_cast<unsigned char>(clip8(a0));
    o[1] = static_cast<unsigned char>(clip8(a1));
    o[2] = static_cast<unsigned char>(clip8(a2));
  }
}

// grid (kOut*kOut/256, n): one output pixel per thread — vertical pass (or the crop rows), rescale, normalise, NCHW.
__global__ void image_vpass_normalise_kernel(ImgBatch b, const unsigned char* __restrict__ src,
                                             const unsigned char* __restrict__ scratch, float* __restrict__ out) {
  const ImgDesc& d = b.d[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= kOut * kOut) return;
  const int y = i / kOut, x = i - (i / kOut) * kOut;
  const unsigned char* base;
  long long pitch;
  if (d.kh) {
    base = scratch + d.inter + x * 3;
    pitch = kOut * 3;
  } else {
    base = src + d.src + static_cast<long long>(d.left + x) * 3;
    pitch = static_cast<long long>(d.W) * 3;
  }
  int v[3];
  if (d.kv) {
    const int* k = reinterpret_cast<const int*>(scratch + d.coef_v) + y * (2 + d.kv);
    const int ymin = k[0], ymax = k[1];
    int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
    for (int t = 0; t < ymax; ++t) {
      const unsigned char* p = base + (ymin + t) * pitch;
      const int w = k[2 + t];
      a0 += p[0] * w;
      a1 += p[1] * w;
      a2 += p[2] * w;
    }
    v[0] = clip8(a0);
    v[1] = clip8(a1);
    v[2] = clip8(a2);
  } else {
    const unsigned char* p = base + (d.top + y) * pitch;
    v[0] = p[0];
    v[1] = p[1];
    v[2] = p[2];
  }
  float* o = out + static_cast<long long>(blockIdx.y) * 3 * kOut * kOut + i;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float f = __double2float_rn(__dmul_rn(static_cast<double>(v[c]), 1.0 / 255.0));
    const float mean = b.bicubic ? kClipMean[c] : 0.5f, stdv = b.bicubic ? kClipStd[c] : 0.5f;
    o[c * kOut * kOut] = __fdiv_rn(__fsub_rn(f, mean), stdv);
  }
}

// Host plan shared by the size query and the entry point: resized size, crop, taps per pass and scratch offsets
// (every section 16-byte aligned).  Returns false on an unsupported size.
static bool plan_images(const int* sizes, int n, int mode, ImgDesc* descs, long long* total) {
  long long cur = 0;
  auto take = [&cur](long long bytes) {
    const long long at = cur;
    cur += (bytes + 15) / 16 * 16;
    return at;
  };
  for (int i = 0; i < n; ++i) {
    const int H = sizes[2 * i], W = sizes[2 * i + 1];
    if (H < 1 || W < 1 || H > kMaxSide || W > kMaxSide) return false;
    ImgDesc d{};
    d.H = H;
    d.W = W;
    double support;
    if (mode == DS_IMG_CLIP) {  // transformers get_resize_output_image_size(shortest_edge=224, default_to_square=False)
      const int s = W <= H ? W : H, l = W <= H ? H : W;
      const int nl = static_cast<int>(static_cast<double>(static_cast<long long>(kOut) * l) / static_cast<double>(s));
      d.rh = W <= H ? nl : kOut;
      d.rw = W <= H ? kOut : nl;
      d.top = (d.rh - kOut) / 2;
      d.left = (d.rw - kOut) / 2;
      support = 2.0;
    } else {
      d.rh = d.rw = kOut;
      support = 1.0;
    }
    auto taps = [support](int in, int out) {
      double fs = static_cast<double>(in) / static_cast<double>(out);
      if (fs < 1.0) fs = 1.0;
      return static_cast<int>(std::ceil(support * fs)) * 2 + 1;
    };
    d.kh = d.rw != W ? taps(W, d.rw) : 0;
    d.kv = d.rh != H ? taps(H, d.rh) : 0;
    d.coef_h = d.kh ? take(4LL * kOut * (2 + d.kh)) : 0;
    d.coef_v = d.kv ? take(4LL * kOut * (2 + d.kv)) : 0;
    d.inter = d.kh ? take(3LL * kOut * H) : 0;
    if (descs) descs[i] = d;
  }
  *total = cur;
  return true;
}

// ------------------------------------------------------------------------------------------------
// VAE image preprocessing (diffusers VaeImageProcessor.preprocess, default config: Pillow LANCZOS resize to the
// panel size, float32(u8) / 255, 2x - 1).  Same fixed-point two-pass resampler as above, any output size.  The
// Lanczos taps need sin(), and one ulp of a device sin() can flip a 22-bit coefficient, so the coefficient tables are
// built on the HOST with the host libm's sin — the function Pillow's precompute_coeffs calls, in the same double
// arithmetic — and copied into the scratch; the kernels only do the integer passes.
constexpr double kLanczosSupport = 3.0;

static double sinc_filter(double x) {
  if (x == 0.0) return 1.0;
  x = x * M_PI;
  return std::sin(x) / x;
}

static double lanczos_filter(double x) {
  if (-3.0 <= x && x < 3.0) return sinc_filter(x) * sinc_filter(x / 3.0);
  return 0.0;
}

static int lanczos_taps(int in, int out) {
  double fs = static_cast<double>(in) / static_cast<double>(out);
  if (fs < 1.0) fs = 1.0;
  return static_cast<int>(std::ceil(kLanczosSupport * fs)) * 2 + 1;
}

// {xmin, xmax, k[0 .. ksize)} per output index, as Pillow's precompute_coeffs + normalize_coeffs_8bpc.
static void lanczos_coeffs(int in, int out, int ksize, int* table) {
  const double scale = static_cast<double>(in) / static_cast<double>(out);
  const double fs = scale < 1.0 ? 1.0 : scale;
  const double support = kLanczosSupport * fs;
  const double ss = 1.0 / fs;
  std::vector<double> k(ksize);
  for (int xx = 0; xx < out; ++xx) {
    const double center = (xx + 0.5) * scale;
    int xmin = static_cast<int>(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = static_cast<int>(center + support + 0.5);
    if (xmax > in) xmax = in;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      k[x] = lanczos_filter((x + xmin - center + 0.5) * ss);
      ww += k[x];
    }
    int* row = table + static_cast<size_t>(xx) * (2 + ksize);
    row[0] = xmin;
    row[1] = xmax;
    for (int x = 0; x < ksize; ++x) {
      double w = x < xmax ? k[x] : 0.0;
      if (x < xmax && ww != 0.0) w /= ww;
      row[2 + x] = w < 0 ? static_cast<int>(-0.5 + w * (1 << kPrecisionBits))
                         : static_cast<int>(0.5 + w * (1 << kPrecisionBits));
    }
  }
}

struct VaePlan {
  int kh, kv;                          // taps per output index of each pass; 0: pass skipped
  long long coef_h, coef_v, inter, total;
};

static VaePlan plan_vae(int H, int W, int oh, int ow, int C) {
  VaePlan p{};
  long long cur = 0;
  auto take = [&cur](long long bytes) {
    const long long at = cur;
    cur += (bytes + 15) / 16 * 16;
    return at;
  };
  p.kh = ow != W ? lanczos_taps(W, ow) : 0;
  p.kv = oh != H ? lanczos_taps(H, oh) : 0;
  p.coef_h = p.kh ? take(4LL * ow * (2 + p.kh)) : 0;
  p.coef_v = p.kv ? take(4LL * oh * (2 + p.kv)) : 0;
  p.inter = p.kh ? take(static_cast<long long>(C) * ow * H) : 0;
  p.total = cur;
  return p;
}

// every source row, the ow output columns, C channels -> uint8 intermediate [H][ow][C]
template <int C>
__global__ void vae_image_hpass_kernel(const unsigned char* __restrict__ img, const int* __restrict__ coef,
                                       unsigned char* __restrict__ inter, int W, int ow, int kh, long long total) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long y = i / ow;
    const int x = static_cast<int>(i - y * ow);
    const int* k = coef + static_cast<size_t>(x) * (2 + kh);
    const int xmin = k[0], xmax = k[1];
    const unsigned char* p = img + (y * W + xmin) * C;
    int a[C];
#pragma unroll
    for (int c = 0; c < C; ++c) a[c] = 1 << (kPrecisionBits - 1);
    for (int t = 0; t < xmax; ++t) {
      const int w = k[2 + t];
#pragma unroll
      for (int c = 0; c < C; ++c) a[c] += p[C * t + c] * w;
    }
    unsigned char* o = inter + i * C;
#pragma unroll
    for (int c = 0; c < C; ++c) o[c] = static_cast<unsigned char>(clip8(a[c]));
  }
}

// output pixel (y, x) of the vertical pass (or a copy when kv == 0) over C-channel uint8 rows of `pitch` bytes
template <int C>
__device__ __forceinline__ void vae_vpass_pixel(const unsigned char* __restrict__ base, long long pitch,
                                                const int* __restrict__ coef, int kv, int y, int x, int v[C]) {
  const unsigned char* col = base + static_cast<long long>(x) * C;
  if (kv) {
    const int* k = coef + static_cast<size_t>(y) * (2 + kv);
    const int ymin = k[0], ymax = k[1];
#pragma unroll
    for (int c = 0; c < C; ++c) v[c] = 1 << (kPrecisionBits - 1);
    for (int t = 0; t < ymax; ++t) {
      const unsigned char* p = col + (ymin + t) * pitch;
      const int w = k[2 + t];
#pragma unroll
      for (int c = 0; c < C; ++c) v[c] += p[c] * w;
    }
#pragma unroll
    for (int c = 0; c < C; ++c) v[c] = clip8(v[c]);
  } else {
    const unsigned char* p = col + y * pitch;
#pragma unroll
    for (int c = 0; c < C; ++c) v[c] = p[c];
  }
}

// one output pixel per thread: vertical pass (or a copy), float32(u8) / 255, 2x - 1 -> fp32 NCHW and / or bf16 NHWC
// with a zero 4th channel (the input of the encoder's conv_in)
__global__ void vae_image_vpass_kernel(const unsigned char* __restrict__ base, long long pitch,
                                       const int* __restrict__ coef, int kv, int oh, int ow, float* __restrict__ out,
                                       uint2* __restrict__ out4) {
  const long long hw = static_cast<long long>(oh) * ow;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= hw) return;
  const int y = static_cast<int>(i / ow), x = static_cast<int>(i - static_cast<long long>(y) * ow);
  int v[3];
  vae_vpass_pixel<3>(base, pitch, coef, kv, y, x, v);
  float o[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    o[c] = __fsub_rn(__fmul_rn(2.0f, __fdiv_rn(static_cast<float>(v[c]), 255.0f)), 1.0f);
    if (out) out[c * hw + i] = o[c];
  }
  if (out4) {
    __nv_bfloat162 lo = __floats2bfloat162_rn(o[0], o[1]), hi = __floats2bfloat162_rn(o[2], 0.0f);
    out4[i] = make_uint2(*reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
  }
}

// float NCHW [B][3][HW] -> (normalize ? 2x - 1 : x) as fp32 NCHW (may alias x) and / or bf16 NHWC with a zero 4th channel
__global__ void vae_image_pack_kernel(const float* x, float* out, uint2* __restrict__ out4, int HW, int normalize,
                                      long long total) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;  // pixel of (batch, hw)
  if (i >= total) return;
  const long long b = i / HW;
  const long long p = i - b * HW;
  float o[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const long long at = (b * 3 + c) * HW + p;
    o[c] = normalize ? __fsub_rn(__fmul_rn(2.0f, x[at]), 1.0f) : x[at];
    if (out) out[at] = o[c];
  }
  if (out4) {
    __nv_bfloat162 lo = __floats2bfloat162_rn(o[0], o[1]), hi = __floats2bfloat162_rn(o[2], 0.0f);
    out4[i] = make_uint2(*reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
  }
}

// ------------------------------------------------------------------------------------------------
// Inpaint mask preprocessing (diffusers VaeImageProcessor(do_normalize=False, do_binarize=True,
// do_convert_grayscale=True).preprocess + prepare_mask_latents' nearest downsample): the same resampler on the mask's
// own channels (1: "L", 3: "RGB"), then for RGB Pillow's RGB -> L conversion of the resized pixels,
// L = (19595 R + 38470 G + 7471 B + 0x8000) >> 16, then float32(L) / 255 >= 0.5, i.e. L >= 128.  One output pixel per
// thread; the pixel at (8i, 8j) also writes latent pixel (i, j) (F.interpolate nearest to H/8 x W/8).
template <int C>
__global__ void vae_mask_vpass_kernel(const unsigned char* __restrict__ base, long long pitch,
                                      const int* __restrict__ coef, int kv, int oh, int ow, float* __restrict__ out,
                                      unsigned char* __restrict__ out_latent) {
  const long long hw = static_cast<long long>(oh) * ow;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= hw) return;
  const int y = static_cast<int>(i / ow), x = static_cast<int>(i - static_cast<long long>(y) * ow);
  int v[C];
  vae_vpass_pixel<C>(base, pitch, coef, kv, y, x, v);
  const int l = C == 3 ? (v[0] * 19595 + v[1] * 38470 + v[2] * 7471 + 0x8000) >> 16 : v[0];
  const bool keep = l >= 128;
  if (out) out[i] = keep ? 1.0f : 0.0f;
  if (out_latent && (y & 7) == 0 && (x & 7) == 0) out_latent[(y >> 3) * (ow >> 3) + (x >> 3)] = keep;
}

// a float mask already at its size [H][W] -> (x >= 0.5) as fp32 and / or the uint8 latent mask [H/8][W/8]
__global__ void vae_mask_pack_kernel(const float* __restrict__ x, float* __restrict__ out,
                                     unsigned char* __restrict__ out_latent, int H, int W) {
  const long long hw = static_cast<long long>(H) * W;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= hw) return;
  const int y = static_cast<int>(i / W), xx = static_cast<int>(i - static_cast<long long>(y) * W);
  const bool keep = x[i] >= 0.5f;
  if (out) out[i] = keep ? 1.0f : 0.0f;
  if (out_latent && (y & 7) == 0 && (xx & 7) == 0) out_latent[(y >> 3) * (W >> 3) + (xx >> 3)] = keep;
}

// The host half of the VAE resampler: the Lanczos tap tables into the scratch and the horizontal pass.  Returns the
// rows the vertical pass reads (the source, or the intermediate) and their pitch.
template <int C>
static int vae_resample_begin(const uint8_t* src, int H, int W, int out_h, int out_w, const VaePlan& p,
                              unsigned char* scr, cudaStream_t st, const unsigned char** base, long long* pitch) {
  // host-built tap tables (pageable source: the copy is staged before the call returns)
  std::vector<int> table;
  if (p.kh) {
    table.assign(static_cast<size_t>(out_w) * (2 + p.kh), 0);
    lanczos_coeffs(W, out_w, p.kh, table.data());
    DS_CUDA_OK(cudaMemcpyAsync(scr + p.coef_h, table.data(), table.size() * 4, cudaMemcpyHostToDevice, st));
  }
  if (p.kv) {
    table.assign(static_cast<size_t>(out_h) * (2 + p.kv), 0);
    lanczos_coeffs(H, out_h, p.kv, table.data());
    DS_CUDA_OK(cudaMemcpyAsync(scr + p.coef_v, table.data(), table.size() * 4, cudaMemcpyHostToDevice, st));
  }
  *base = src;
  *pitch = static_cast<long long>(C) * W;
  if (p.kh) {
    const long long total = static_cast<long long>(H) * out_w;
    const long long blocks = (total + 255) / 256;
    vae_image_hpass_kernel<C><<<static_cast<unsigned>(blocks < 4096 ? blocks : 4096), 256, 0, st>>>(
        src, reinterpret_cast<const int*>(scr + p.coef_h), scr + p.inter, W, out_w, p.kh, total);
    DS_LAUNCH_OK("vae_image_hpass_kernel");
    *base = scr + p.inter;
    *pitch = static_cast<long long>(C) * out_w;
  }
  return DS_OK;
}

}  // namespace ds

extern "C" int64_t ds_image_preprocess_scratch_bytes(const int* sizes, int n, int mode) {
  long long total = 0;
  if (!sizes || n < 1 || (mode != DS_IMG_CLIP && mode != DS_IMG_VIT) || !ds::plan_images(sizes, n, mode, nullptr, &total))
    return -1;
  return total;
}

extern "C" int ds_image_preprocess(const uint8_t* src, const int64_t* offsets, const int* sizes, int n, int mode,
                                   float* out, void* scratch, int64_t scratch_bytes, void* stream) {
  using namespace ds;
  DS_REQUIRE(src && offsets && sizes && out && n > 0, "ds_image_preprocess: bad arguments");
  DS_REQUIRE(mode == DS_IMG_CLIP || mode == DS_IMG_VIT, "ds_image_preprocess: unknown mode %d", mode);
  DS_REQUIRE((reinterpret_cast<uintptr_t>(out) & 3) == 0, "ds_image_preprocess: out must be 4-byte aligned");
  for (int i = 0; i < n; ++i) {
    DS_REQUIRE(sizes[2 * i] >= 1 && sizes[2 * i + 1] >= 1 && sizes[2 * i] <= kMaxSide && sizes[2 * i + 1] <= kMaxSide,
               "ds_image_preprocess: image %d is %d x %d; sides must be in [1, %d]", i, sizes[2 * i], sizes[2 * i + 1],
               kMaxSide);
    DS_REQUIRE(offsets[i] >= 0, "ds_image_preprocess: negative offset for image %d", i);
  }
  long long need = 0;
  std::vector<ImgDesc> all(n);
  plan_images(sizes, n, mode, all.data(), &need);
  DS_REQUIRE(need == 0 || (scratch && scratch_bytes >= need && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0),
             "ds_image_preprocess: needs %lld bytes of 16-byte aligned scratch (ds_image_preprocess_scratch_bytes), "
             "got %lld", need, static_cast<long long>(scratch_bytes));
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  unsigned char* scr = static_cast<unsigned char*>(scratch);
  for (int first = 0; first < n; first += kMaxImages) {
    ImgBatch b;
    b.n = n - first < kMaxImages ? n - first : kMaxImages;
    b.bicubic = mode == DS_IMG_CLIP;
    bool any_resize = false;
    long long max_rows = 0;  // rows of the tallest image that needs the horizontal pass
    for (int j = 0; j < b.n; ++j) {
      b.d[j] = all[first + j];
      b.d[j].src = offsets[first + j];
      any_resize |= b.d[j].kh || b.d[j].kv;
      if (b.d[j].kh && b.d[j].H > max_rows) max_rows = b.d[j].H;
    }
    if (any_resize) {
      image_coef_kernel<<<dim3(b.n, 2), kOut, 0, st>>>(b, scr);
      DS_LAUNCH_OK("image_coef_kernel");
    }
    if (max_rows) {
      const long long blocks = (max_rows * kOut + 255) / 256;
      image_hpass_kernel<<<dim3(static_cast<unsigned>(blocks < 2048 ? blocks : 2048), b.n), 256, 0, st>>>(b, src, scr);
      DS_LAUNCH_OK("image_hpass_kernel");
    }
    image_vpass_normalise_kernel<<<dim3(kOut * kOut / 256, b.n), 256, 0, st>>>(
        b, src, scr, out + static_cast<long long>(first) * 3 * kOut * kOut);
    DS_LAUNCH_OK("image_vpass_normalise_kernel");
  }
  return DS_OK;
}

extern "C" int64_t ds_vae_image_preprocess_scratch_bytes(int H, int W, int out_h, int out_w) {
  if (H < 1 || W < 1 || H > ds::kMaxSide || W > ds::kMaxSide || out_h < 1 || out_w < 1 || out_h > ds::kMaxSide ||
      out_w > ds::kMaxSide)
    return -1;
  return ds::plan_vae(H, W, out_h, out_w, 3).total;
}

extern "C" int ds_vae_image_preprocess(const uint8_t* src, int H, int W, int out_h, int out_w, float* out,
                                       void* out_nhwc4, void* scratch, int64_t scratch_bytes, void* stream) {
  using namespace ds;
  DS_REQUIRE(src && (out || out_nhwc4), "ds_vae_image_preprocess: bad arguments");
  DS_REQUIRE(H >= 1 && W >= 1 && H <= kMaxSide && W <= kMaxSide && out_h >= 1 && out_w >= 1 && out_h <= kMaxSide &&
                 out_w <= kMaxSide,
             "ds_vae_image_preprocess: %d x %d -> %d x %d; sides must be in [1, %d]", H, W, out_h, out_w, kMaxSide);
  DS_REQUIRE((reinterpret_cast<uintptr_t>(out) & 3) == 0 && (reinterpret_cast<uintptr_t>(out_nhwc4) & 7) == 0,
             "ds_vae_image_preprocess: out must be 4-byte and out_nhwc4 8-byte aligned");
  const VaePlan p = plan_vae(H, W, out_h, out_w, 3);
  DS_REQUIRE(p.total == 0 || (scratch && scratch_bytes >= p.total && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0),
             "ds_vae_image_preprocess: needs %lld bytes of 16-byte aligned scratch "
             "(ds_vae_image_preprocess_scratch_bytes), got %lld", p.total, static_cast<long long>(scratch_bytes));
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  unsigned char* scr = static_cast<unsigned char*>(scratch);
  const unsigned char* base;
  long long pitch;
  const int rc = vae_resample_begin<3>(src, H, W, out_h, out_w, p, scr, st, &base, &pitch);
  if (rc != DS_OK) return rc;
  const long long hw = static_cast<long long>(out_h) * out_w;
  vae_image_vpass_kernel<<<static_cast<unsigned>((hw + 255) / 256), 256, 0, st>>>(
      base, pitch, reinterpret_cast<const int*>(scr + p.coef_v), p.kv, out_h, out_w, out,
      static_cast<uint2*>(out_nhwc4));
  DS_LAUNCH_OK("vae_image_vpass_kernel");
  return DS_OK;
}

extern "C" int ds_vae_image_pack(const float* x, float* out, void* out_nhwc4, int B, int HW, int normalize,
                                 void* stream) {
  using namespace ds;
  DS_REQUIRE(x && (out || out_nhwc4) && B > 0 && HW > 0, "ds_vae_image_pack: bad arguments");
  DS_REQUIRE((reinterpret_cast<uintptr_t>(out_nhwc4) & 7) == 0, "ds_vae_image_pack: out_nhwc4 must be 8-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long total = static_cast<long long>(B) * HW;
  vae_image_pack_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, out, static_cast<uint2*>(out_nhwc4), HW, normalize, total);
  DS_LAUNCH_OK("vae_image_pack_kernel");
  return DS_OK;
}

extern "C" int64_t ds_vae_mask_preprocess_scratch_bytes(int H, int W, int C, int out_h, int out_w) {
  if (H < 1 || W < 1 || H > ds::kMaxSide || W > ds::kMaxSide || out_h < 1 || out_w < 1 || out_h > ds::kMaxSide ||
      out_w > ds::kMaxSide || (C != 1 && C != 3))
    return -1;
  return ds::plan_vae(H, W, out_h, out_w, C).total;
}

extern "C" int ds_vae_mask_preprocess(const uint8_t* src, int H, int W, int C, int out_h, int out_w, float* out,
                                      uint8_t* out_latent, void* scratch, int64_t scratch_bytes, void* stream) {
  using namespace ds;
  DS_REQUIRE(src && (out || out_latent), "ds_vae_mask_preprocess: bad arguments");
  DS_REQUIRE(C == 1 || C == 3, "ds_vae_mask_preprocess: C must be 1 (L) or 3 (RGB), got %d", C);
  DS_REQUIRE(H >= 1 && W >= 1 && H <= kMaxSide && W <= kMaxSide && out_h >= 1 && out_w >= 1 && out_h <= kMaxSide &&
                 out_w <= kMaxSide,
             "ds_vae_mask_preprocess: %d x %d -> %d x %d; sides must be in [1, %d]", H, W, out_h, out_w, kMaxSide);
  DS_REQUIRE(!out_latent || (out_h % 8 == 0 && out_w % 8 == 0),
             "ds_vae_mask_preprocess: the latent mask needs an output size that is a multiple of 8, got %d x %d", out_h,
             out_w);
  DS_REQUIRE((reinterpret_cast<uintptr_t>(out) & 3) == 0, "ds_vae_mask_preprocess: out must be 4-byte aligned");
  const VaePlan p = plan_vae(H, W, out_h, out_w, C);
  DS_REQUIRE(p.total == 0 || (scratch && scratch_bytes >= p.total && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0),
             "ds_vae_mask_preprocess: needs %lld bytes of 16-byte aligned scratch "
             "(ds_vae_mask_preprocess_scratch_bytes), got %lld", p.total, static_cast<long long>(scratch_bytes));
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  unsigned char* scr = static_cast<unsigned char*>(scratch);
  const unsigned char* base;
  long long pitch;
  const int rc = C == 3 ? vae_resample_begin<3>(src, H, W, out_h, out_w, p, scr, st, &base, &pitch)
                        : vae_resample_begin<1>(src, H, W, out_h, out_w, p, scr, st, &base, &pitch);
  if (rc != DS_OK) return rc;
  const long long hw = static_cast<long long>(out_h) * out_w;
  const unsigned blocks = static_cast<unsigned>((hw + 255) / 256);
  const int* coef_v = reinterpret_cast<const int*>(scr + p.coef_v);
  if (C == 3)
    vae_mask_vpass_kernel<3><<<blocks, 256, 0, st>>>(base, pitch, coef_v, p.kv, out_h, out_w, out, out_latent);
  else
    vae_mask_vpass_kernel<1><<<blocks, 256, 0, st>>>(base, pitch, coef_v, p.kv, out_h, out_w, out, out_latent);
  DS_LAUNCH_OK("vae_mask_vpass_kernel");
  return DS_OK;
}

extern "C" int ds_vae_mask_pack(const float* x, int H, int W, float* out, uint8_t* out_latent, void* stream) {
  using namespace ds;
  DS_REQUIRE(x && (out || out_latent) && H > 0 && W > 0, "ds_vae_mask_pack: bad arguments");
  DS_REQUIRE(!out_latent || (H % 8 == 0 && W % 8 == 0),
             "ds_vae_mask_pack: the latent mask needs a size that is a multiple of 8, got %d x %d", H, W);
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long hw = static_cast<long long>(H) * W;
  vae_mask_pack_kernel<<<static_cast<unsigned>((hw + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, out, out_latent, H, W);
  DS_LAUNCH_OK("vae_mask_pack_kernel");
  return DS_OK;
}
