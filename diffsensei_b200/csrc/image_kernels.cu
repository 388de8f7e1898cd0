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
// The same resampler also serves diffusers' VaeImageProcessor.preprocess (ds_vae_preprocess: an optional crop, Pillow
// LANCZOS to any size or _resize_and_fill, then the AutoencoderKL encoder's 2 * u8 / 255 - 1 or the inpaint mask's
// RGB -> L and threshold, or the T2I-Adapter's u8 / 255 written pixel-unshuffled) and apply_overlay (ds_vae_overlay),
// with host-built tap tables; see the sections below plan_images.
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

// Pillow's bicubic_filter (a = -0.5), the default filter of Image.resize: the fill stripes use it
static double bicubic_filter(double x) {
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((-0.5 + 2.0) * x - (-0.5 + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * -0.5;
  return 0.0;
}

constexpr double kBicubicSupport = 2.0;

// taps per output index of a pass over a source span of `span` pixels (Pillow: ceil(support * filterscale) * 2 + 1)
static int filter_taps(double span, int out, double support) {
  double fs = span / static_cast<double>(out);
  if (fs < 1.0) fs = 1.0;
  return static_cast<int>(std::ceil(support * fs)) * 2 + 1;
}

static int lanczos_taps(int in, int out) { return filter_taps(static_cast<double>(in), out, kLanczosSupport); }

// {xmin, xmax, k[0 .. ksize)} per output index, as Pillow's precompute_coeffs(inSize, in0, in1, outSize) +
// normalize_coeffs_8bpc: the source box [in0, in1) of an axis of `in` pixels (in0 == in1 is a zero-width box: every
// output index takes the same taps around in0, Pillow's edge rows).
static void box_coeffs(int in, double in0, double in1, int out, int ksize, int* table, bool bicubic) {
  const double scale = (in1 - in0) / static_cast<double>(out);
  const double fs = scale < 1.0 ? 1.0 : scale;
  const double support = (bicubic ? kBicubicSupport : kLanczosSupport) * fs;
  const double ss = 1.0 / fs;
  std::vector<double> k(ksize);
  for (int xx = 0; xx < out; ++xx) {
    const double center = in0 + (xx + 0.5) * scale;
    int xmin = static_cast<int>(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = static_cast<int>(center + support + 0.5);
    if (xmax > in) xmax = in;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      const double arg = (x + xmin - center + 0.5) * ss;
      k[x] = bicubic ? bicubic_filter(arg) : lanczos_filter(arg);
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

// the whole axis (box [0, in)), LANCZOS: Image.resize without a box
static void lanczos_coeffs(int in, int out, int ksize, int* table) {
  box_coeffs(in, 0.0, static_cast<double>(in), out, ksize, table, false);
}

struct VaePlan {
  int kh, kv;                          // taps per output index of each pass; 0: pass skipped
  long long coef_h, coef_v, inter, total;
};

// `n` images of one size share the tables; each has its own horizontal-pass intermediate
static VaePlan plan_vae(int H, int W, int oh, int ow, int C, int n = 1) {
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
  p.inter = p.kh ? take(static_cast<long long>(n) * C * ow * H) : 0;
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

// The host-built LANCZOS tap tables of plan `p` (an H x W source to out_h x out_w) into the scratch (pageable
// source: the copy is staged before the call returns).
static int upload_lanczos_tables(int H, int W, int out_h, int out_w, const VaePlan& p, unsigned char* scr,
                                 cudaStream_t st) {
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
  return DS_OK;
}

// The host half of the VAE resampler: the Lanczos tap tables into the scratch and the horizontal pass over an
// H x W source whose rows are `row_px` pixels apart (W for a whole image, the image's width for a crop).  Returns the
// rows the vertical pass reads (the source, or the intermediate) and their pitch.
template <int C>
static int vae_resample_begin(const uint8_t* src, int H, int W, long long row_px, int out_h, int out_w,
                              const VaePlan& p, unsigned char* scr, cudaStream_t st, const unsigned char** base,
                              long long* pitch) {
  const int rc = upload_lanczos_tables(H, W, out_h, out_w, p, scr, st);
  if (rc != DS_OK) return rc;
  *base = src;
  *pitch = static_cast<long long>(C) * row_px;
  if (p.kh) {
    const long long total = static_cast<long long>(H) * out_w;
    const long long blocks = (total + 255) / 256;
    vae_image_hpass_kernel<C><<<static_cast<unsigned>(blocks < 4096 ? blocks : 4096), 256, 0, st>>>(
        src, reinterpret_cast<const int*>(scr + p.coef_h), scr + p.inter, static_cast<int>(row_px), out_w, p.kh,
        total);
    DS_LAUNCH_OK("vae_image_hpass_kernel");
    *base = scr + p.inter;
    *pitch = static_cast<long long>(C) * out_w;
  }
  return DS_OK;
}

// ------------------------------------------------------------------------------------------------
// diffusers VaeImageProcessor.preprocess(..., crops_coords, resize_mode) of one uint8 image or mask:
// Image.crop(crops_coords) (the whole image without them; the SDXL inpaint pipeline's padding_mask_crop passes them),
// then
//   resize_mode "fill"    (_resize_and_fill): ratio = w / h, src_ratio = cw / ch (crop size), the crop resized with
//                         LANCZOS to fit, rw = ratio < src_ratio ? w : cw * h // ch, rh = ratio >= src_ratio ? h :
//                         ch * w // cw, pasted at (w // 2 - rw // 2, h // 2 - rh // 2) on a black w x h canvas; when
//                         the crop is wider (taller) than the frame, the `fill` = h // 2 - rh // 2 rows above and below
//                         (w // 2 - rw // 2 columns left and right) are resized.resize(..., box=(0, 0, w, 0)) and
//                         box=(0, rh, w, rh) (the column equivalents): Pillow's default BICUBIC over a zero-height
//                         (zero-width) source box, every stripe row the same weighted mix of the resized image's
//                         first (last) rows; a canvas row or column neither covers stays black;
//   resize_mode "default" (Image.resize): the crop resized with LANCZOS to w x h.
// Then the epilogue of the processor's configuration:
//   image (the default one, the AutoencoderKL encoder's input): float32(u8) / 255, 2x - 1 -> fp32 NCHW and / or bf16
//         NHWC with a zero 4th channel (the input of the encoder's conv_in);
//   mask  (do_normalize=False, do_binarize=True, do_convert_grayscale=True; resized in its own mode, C = 1 "L" or
//         3 "RGB"): for RGB Pillow's RGB -> L conversion of the resized pixels, L = (19595 R + 38470 G + 7471 B +
//         0x8000) >> 16, then float32(L) / 255 >= 0.5, i.e. L >= 128 -> fp32; the pixel at (8i, 8j) also writes
//         latent pixel (i, j) (prepare_mask_latents' F.interpolate nearest to H/8 x W/8).
//   adapter (diffusers' _preprocess_adapter_image + T2IAdapter's PixelUnshuffle(16); resized in its own mode, C = 1
//         "L" or 3 "RGB"): float32(u8) / 255, no normalisation, rounded to bf16 and written pixel-unshuffled.
// One launch of the horizontal pass over the crop (the source rows keep the image's pitch; skipped when the width
// does not change), then one thread per output pixel: the vertical pass of the resized pixel (a copy when the height
// does not change), or of the 2 resized rows (columns) a stripe pixel mixes, then the epilogue.
struct FillPlan {
  VaePlan main;           // the crop (ch x cw) -> rh x rw resize
  int x1, y1, cw, ch;     // crop origin and size in the source
  int rw, rh, ox, oy;     // resized size, paste offset on the canvas
  int stripe;             // 0: none, 1: rows above / below, 2: columns left / right
  int fill;               // stripe thickness
  int ks;                 // taps of a stripe table
  long long coef_s0, coef_s1, total;
};

static bool plan_fill(int H, int W, int C, int x1, int y1, int x2, int y2, int oh, int ow, int fill_mode,
                      FillPlan* out) {
  if (H < 1 || W < 1 || H > kMaxSide || W > kMaxSide || oh < 1 || ow < 1 || oh > kMaxSide || ow > kMaxSide ||
      (C != 1 && C != 3) || x1 < 0 || y1 < 0 || x2 > W || y2 > H || x2 <= x1 || y2 <= y1 ||
      (fill_mode != 0 && fill_mode != 1))
    return false;
  FillPlan p{};
  p.x1 = x1;
  p.y1 = y1;
  p.cw = x2 - x1;
  p.ch = y2 - y1;
  if (fill_mode) {
    const double ratio = static_cast<double>(ow) / static_cast<double>(oh);
    const double src_ratio = static_cast<double>(p.cw) / static_cast<double>(p.ch);
    p.rw = ratio < src_ratio ? ow : static_cast<int>(static_cast<long long>(p.cw) * oh / p.ch);
    p.rh = ratio >= src_ratio ? oh : static_cast<int>(static_cast<long long>(p.ch) * ow / p.cw);
    p.ox = ow / 2 - p.rw / 2;
    p.oy = oh / 2 - p.rh / 2;
    if (ratio < src_ratio) {
      p.fill = oh / 2 - p.rh / 2;
      p.stripe = p.fill > 0 ? 1 : 0;
    } else if (ratio > src_ratio) {
      p.fill = ow / 2 - p.rw / 2;
      p.stripe = p.fill > 0 ? 2 : 0;
    }
  } else {
    p.rw = ow;
    p.rh = oh;
  }
  if (p.rw < 1 || p.rh < 1 || p.rw > ow || p.rh > oh) return false;   // Pillow: "height and width must be > 0"
  p.main = plan_vae(p.ch, p.cw, p.rh, p.rw, C);
  long long cur = p.main.total;
  if (p.stripe) {
    p.ks = filter_taps(0.0, p.fill, kBicubicSupport);
    const long long bytes = (4LL * p.fill * (2 + p.ks) + 15) / 16 * 16;
    p.coef_s0 = cur;
    p.coef_s1 = cur + bytes;
    cur += 2 * bytes;
  }
  p.total = cur;
  *out = p;
  return true;
}

struct FillArgs {
  const unsigned char* base;   // rows the vertical pass reads: the crop in the source, or the intermediate
  long long pitch;             // bytes between those rows
  const int* coef_v;
  const int* coef_s0;          // stripe tables (top / left, bottom / right)
  const int* coef_s1;
  int kv, ks;
  int rw, rh, ox, oy, stripe, fill;
  int oh, ow;
  float* out;                  // image: fp32 NCHW [3][oh][ow]; mask: fp32 [oh][ow]; adapter: unused
  void* out2;                  // image: bf16 NHWC4 [oh][ow][4]; mask: uint8 latent [oh/8][ow/8];
                               // adapter: bf16 NHWC [oh/16][ow/16][C*256]
};

// one stripe pixel: clip8(2^21 + sum_t k[t] * resized[...]) over the 1-D taps of its stripe table row
template <int C>
__device__ __forceinline__ void fill_stripe_pixel(const FillArgs& a, const int* table, int idx, int ry, int rx,
                                                  bool rows, int v[C]) {
  const int* k = table + static_cast<size_t>(idx) * (2 + a.ks);
  const int lo = k[0], n = k[1];
  int acc[C];
#pragma unroll
  for (int c = 0; c < C; ++c) acc[c] = 1 << (kPrecisionBits - 1);
  for (int t = 0; t < n; ++t) {
    int r[C];
    vae_vpass_pixel<C>(a.base, a.pitch, a.coef_v, a.kv, rows ? lo + t : ry, rows ? rx : lo + t, r);
    const int w = k[2 + t];
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] += r[c] * w;
  }
#pragma unroll
  for (int c = 0; c < C; ++c) v[c] = clip8(acc[c]);
}

template <int C, int kEpi>
__global__ void vae_preprocess_kernel(FillArgs a) {
  const long long hw = static_cast<long long>(a.oh) * a.ow;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= hw) return;
  const int y = static_cast<int>(i / a.ow), x = static_cast<int>(i - static_cast<long long>(y) * a.ow);
  const int ry = y - a.oy, rx = x - a.ox;
  int v[C];
#pragma unroll
  for (int c = 0; c < C; ++c) v[c] = 0;                            // the black canvas
  if (ry >= 0 && ry < a.rh && rx >= 0 && rx < a.rw) {
    vae_vpass_pixel<C>(a.base, a.pitch, a.coef_v, a.kv, ry, rx, v);
  } else if (a.stripe == 1) {                                      // rows: ox == 0, rw == ow
    if (y < a.fill) fill_stripe_pixel<C>(a, a.coef_s0, y, 0, x, true, v);
    else if (ry >= a.rh && ry - a.rh < a.fill) fill_stripe_pixel<C>(a, a.coef_s1, ry - a.rh, 0, x, true, v);
  } else if (a.stripe == 2) {                                      // columns: oy == 0, rh == oh
    if (x < a.fill) fill_stripe_pixel<C>(a, a.coef_s0, x, y, 0, false, v);
    else if (rx >= a.rw && rx - a.rw < a.fill) fill_stripe_pixel<C>(a, a.coef_s1, rx - a.rw, y, 0, false, v);
  }
  if constexpr (kEpi == DS_VAE_EPI_MASK) {
    const int l = C == 3 ? (v[0] * 19595 + v[1] * 38470 + v[2] * 7471 + 0x8000) >> 16 : v[0];
    const bool keep = l >= 128;
    if (a.out) a.out[i] = keep ? 1.0f : 0.0f;
    if (a.out2 && (y & 7) == 0 && (x & 7) == 0)
      static_cast<unsigned char*>(a.out2)[(y >> 3) * (a.ow >> 3) + (x >> 3)] = keep;
  } else if constexpr (kEpi == DS_VAE_EPI_ADAPTER) {
    // PixelUnshuffle(16): pixel (16 Y + i, 16 X + j) of channel c -> [Y][X][c * 256 + i * 16 + j]
    __nv_bfloat16* o = static_cast<__nv_bfloat16*>(a.out2) +
                       (static_cast<long long>(y >> 4) * (a.ow >> 4) + (x >> 4)) * (C * 256) + (y & 15) * 16 + (x & 15);
#pragma unroll
    for (int c = 0; c < C; ++c) o[c * 256] = __float2bfloat16_rn(__fdiv_rn(static_cast<float>(v[c]), 255.0f));
  } else {
    float o[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      o[c] = __fsub_rn(__fmul_rn(2.0f, __fdiv_rn(static_cast<float>(v[c]), 255.0f)), 1.0f);
      if (a.out) a.out[c * hw + i] = o[c];
    }
    if (a.out2) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(o[0], o[1]), hi = __floats2bfloat162_rn(o[2], 0.0f);
      static_cast<uint2*>(a.out2)[i] = make_uint2(*reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
    }
  }
}

// ------------------------------------------------------------------------------------------------
// diffusers VaeImageProcessor.apply_overlay(mask, init_image, image, crop_coords) after numpy_to_pil, for a batch of
// decoded crops sharing one original and one mask:
//   u8 = round(float32(x) * 255) (ties to even) of the decoded fp32 NCHW [0, 1] image (h x w);
//   _resize_and_crop to the crop (cw x ch): ratio = cw / ch, src_ratio = w / h, rw = ratio > src_ratio ? cw :
//     w * ch // h, rh = ratio <= src_ratio ? ch : h * cw // w, LANCZOS, pasted at (cw // 2 - rw // 2, ch // 2 - rh // 2)
//     (negative offsets crop), then at (x1, y1) on a transparent canvas, convert("RGB"), convert("RGBA"): the canvas
//     pixel d is that resized pixel inside the crop and black outside, alpha 255;
//   the masked original: a = 255 - L (ImageOps.invert), paste onto a zero RGBa image with mask a: p = DIV255(init * a),
//     alpha = DIV255(255 a); convert("RGBA"): s = alpha in {0, 255} ? p : CLIP8(255 p / alpha);
//   alpha_composite(canvas, masked) with Pillow's 7-bit-precision integer blend (alpha 0: the canvas pixel), "RGB".
// One horizontal-pass launch (reading and rounding the fp32 image) when the width changes, then one output pixel per
// thread; a pixel outside the crop does no resampling.
struct OverlayPlan {
  VaePlan main;           // the decoded (h x w) -> rh x rw resize, one intermediate per sample
  int x1, y1, cw, ch;
  int rw, rh, ox, oy;
};

static bool plan_overlay(int n, int h, int w, int H, int W, int x1, int y1, int x2, int y2, OverlayPlan* out) {
  if (n < 1 || h < 1 || w < 1 || h > kMaxSide || w > kMaxSide || H < 1 || W < 1 || H > kMaxSide || W > kMaxSide ||
      x1 < 0 || y1 < 0 || x2 > W || y2 > H || x2 <= x1 || y2 <= y1)
    return false;
  OverlayPlan p{};
  p.x1 = x1;
  p.y1 = y1;
  p.cw = x2 - x1;
  p.ch = y2 - y1;
  const double ratio = static_cast<double>(p.cw) / static_cast<double>(p.ch);
  const double src_ratio = static_cast<double>(w) / static_cast<double>(h);
  p.rw = ratio > src_ratio ? p.cw : static_cast<int>(static_cast<long long>(w) * p.ch / h);
  p.rh = ratio <= src_ratio ? p.ch : static_cast<int>(static_cast<long long>(h) * p.cw / w);
  if (p.rw < 1 || p.rh < 1 || p.rw > kMaxSide || p.rh > kMaxSide) return false;
  p.ox = p.cw / 2 - p.rw / 2;
  p.oy = p.ch / 2 - p.rh / 2;
  p.main = plan_vae(h, w, p.rh, p.rw, 3, n);
  *out = p;
  return true;
}

__device__ __forceinline__ int round_u8(float x) {
  return min(max(__float2int_rn(__fmul_rn(x, 255.0f)), 0), 255);
}

// every row of every sample, the rw output columns: the horizontal pass over the rounded fp32 NCHW image
__global__ void overlay_hpass_kernel(const float* __restrict__ img, const int* __restrict__ coef,
                                     unsigned char* __restrict__ inter, int h, int w, int rw, int kh,
                                     long long total) {
  const long long hw = static_cast<long long>(h) * w;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / rw;                                   // b * h + y
    const int x = static_cast<int>(i - row * rw);
    const long long b = row / h;
    const int* k = coef + static_cast<size_t>(x) * (2 + kh);
    const int xmin = k[0], xmax = k[1];
    const float* p = img + b * 3 * hw + (row - b * h) * w + xmin;
    int a[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) a[c] = 1 << (kPrecisionBits - 1);
    for (int t = 0; t < xmax; ++t) {
      const int wt = k[2 + t];
#pragma unroll
      for (int c = 0; c < 3; ++c) a[c] += round_u8(p[c * hw + t]) * wt;
    }
    unsigned char* o = inter + i * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = static_cast<unsigned char>(clip8(a[c]));
  }
}

struct OverlayArgs {
  const float* img;            // decoded fp32 NCHW [n][3][h][w]
  const unsigned char* inter;  // horizontal-pass intermediate [n][h][rw][3], or NULL (kh == 0)
  const int* coef_v;
  const unsigned char* init;   // uint8 RGB [H][W][3]
  const unsigned char* mask;   // uint8 L [H][W]
  unsigned char* out;          // uint8 RGB [n][H][W][3]
  int n, h, w, H, W;
  int x1, y1, cw, ch, rw, rh, ox, oy, kv;
};

__global__ void vae_overlay_kernel(OverlayArgs a) {
  const long long HW = static_cast<long long>(a.H) * a.W;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= HW * a.n) return;
  const long long b = i / HW, px = i - b * HW;
  const int Y = static_cast<int>(px / a.W), X = static_cast<int>(px - static_cast<long long>(Y) * a.W);
  // the canvas pixel: the resized crop inside the crop box, black outside
  int d[3] = {0, 0, 0};
  const int cy = Y - a.y1 - a.oy, cx = X - a.x1 - a.ox;
  if (X >= a.x1 && X < a.x1 + a.cw && Y >= a.y1 && Y < a.y1 + a.ch && cy >= 0 && cy < a.rh && cx >= 0 && cx < a.rw) {
    if (a.inter) {
      vae_vpass_pixel<3>(a.inter + b * a.h * a.rw * 3, static_cast<long long>(a.rw) * 3, a.coef_v, a.kv, cy, cx, d);
    } else {                                                        // width unchanged: read and round the fp32 image
      const long long hw = static_cast<long long>(a.h) * a.w;
      const float* col = a.img + b * 3 * hw + cx;
      if (a.kv) {
        const int* k = a.coef_v + static_cast<size_t>(cy) * (2 + a.kv);
        const int ymin = k[0], ymax = k[1];
#pragma unroll
        for (int c = 0; c < 3; ++c) d[c] = 1 << (kPrecisionBits - 1);
        for (int t = 0; t < ymax; ++t) {
          const int wt = k[2 + t];
#pragma unroll
          for (int c = 0; c < 3; ++c) d[c] += round_u8(col[c * hw + static_cast<long long>(ymin + t) * a.w]) * wt;
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) d[c] = clip8(d[c]);
      } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) d[c] = round_u8(col[c * hw + static_cast<long long>(cy) * a.w]);
      }
    }
  }
  // the masked original, premultiplied by the inverted mask and converted back to straight alpha
  const unsigned int alpha_in = 255u - a.mask[px];
  auto div255 = [](unsigned int v) {
    const unsigned int t = v + 128u;
    return ((t >> 8) + t) >> 8;
  };
  const unsigned int alpha = div255(255u * alpha_in);
  const unsigned char* p0 = a.init + px * 3;
  unsigned char* o = a.out + i * 3;
  if (alpha == 0) {
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = static_cast<unsigned char>(d[c]);
    return;
  }
  const unsigned int outa255 = alpha * 255u + 255u * (255u - alpha);
  const unsigned int coef1 = alpha * 255u * 255u * (1u << 7) / outa255;
  const unsigned int coef2 = 255u * (1u << 7) - coef1;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const unsigned int prem = div255(static_cast<unsigned int>(p0[c]) * alpha_in);
    const unsigned int s = alpha == 255u ? prem : min(255u * prem / alpha, 255u);
    const unsigned int tmp = s * coef1 + static_cast<unsigned int>(d[c]) * coef2 + (0x80u << 7);
    o[c] = static_cast<unsigned char>((((tmp >> 8) + tmp) >> 8) >> 7);
  }
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

extern "C" int64_t ds_vae_preprocess_scratch_bytes(int H, int W, int C, int x1, int y1, int x2, int y2, int out_h,
                                                   int out_w, int fill) {
  ds::FillPlan p;
  if (!ds::plan_fill(H, W, C, x1, y1, x2, y2, out_h, out_w, fill, &p)) return -1;
  return p.total;
}

extern "C" int ds_vae_preprocess(const uint8_t* src, int H, int W, int C, int x1, int y1, int x2, int y2, int out_h,
                                 int out_w, int fill, int epilogue, float* out, void* out2, void* scratch,
                                 int64_t scratch_bytes, void* stream) {
  using namespace ds;
  DS_REQUIRE(src && (out || out2), "ds_vae_preprocess: bad arguments");
  DS_REQUIRE(epilogue == DS_VAE_EPI_IMAGE || epilogue == DS_VAE_EPI_MASK || epilogue == DS_VAE_EPI_ADAPTER,
             "ds_vae_preprocess: unknown epilogue %d", epilogue);
  const bool mask = epilogue == DS_VAE_EPI_MASK, adapter = epilogue == DS_VAE_EPI_ADAPTER;
  DS_REQUIRE(epilogue != DS_VAE_EPI_IMAGE ? (C == 1 || C == 3) : C == 3, "ds_vae_preprocess: C must be 3 for an "
             "image, 1 or 3 for a mask or an adapter input, got %d", C);
  DS_REQUIRE(!adapter || (!out && out2 && out_h % 16 == 0 && out_w % 16 == 0 &&
                          (reinterpret_cast<uintptr_t>(out2) & 1) == 0),
             "ds_vae_preprocess: the adapter epilogue writes out2 only (2-byte aligned) and needs an output size that "
             "is a multiple of 16, got %d x %d", out_h, out_w);
  FillPlan p;
  DS_REQUIRE(plan_fill(H, W, C, x1, y1, x2, y2, out_h, out_w, fill, &p),
             "ds_vae_preprocess: crop (%d, %d, %d, %d) of a %d x %d image -> %d x %d (fill %d) is not supported: "
             "the crop must lie inside the image, sides in [1, %d], and the resized crop must be at least 1 x 1",
             x1, y1, x2, y2, H, W, out_h, out_w, fill, kMaxSide);
  DS_REQUIRE(!(mask && out2) || (out_h % 8 == 0 && out_w % 8 == 0),
             "ds_vae_preprocess: the latent mask needs an output size that is a multiple of 8, got %d x %d", out_h,
             out_w);
  DS_REQUIRE((reinterpret_cast<uintptr_t>(out) & 3) == 0 && (epilogue != DS_VAE_EPI_IMAGE ||
                                                             (reinterpret_cast<uintptr_t>(out2) & 7) == 0),
             "ds_vae_preprocess: out must be 4-byte and an image's out2 8-byte aligned");
  DS_REQUIRE(p.total == 0 || (scratch && scratch_bytes >= p.total && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0),
             "ds_vae_preprocess: needs %lld bytes of 16-byte aligned scratch "
             "(ds_vae_preprocess_scratch_bytes), got %lld", p.total, static_cast<long long>(scratch_bytes));
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  unsigned char* scr = static_cast<unsigned char*>(scratch);
  if (p.stripe) {                                   // rows: the resized image's height; columns: its width
    const int in = p.stripe == 1 ? p.rh : p.rw;
    std::vector<int> table(static_cast<size_t>(p.fill) * (2 + p.ks), 0);
    box_coeffs(in, 0.0, 0.0, p.fill, p.ks, table.data(), true);
    DS_CUDA_OK(cudaMemcpyAsync(scr + p.coef_s0, table.data(), table.size() * 4, cudaMemcpyHostToDevice, st));
    std::vector<int> table1(table.size(), 0);
    box_coeffs(in, static_cast<double>(in), static_cast<double>(in), p.fill, p.ks, table1.data(), true);
    DS_CUDA_OK(cudaMemcpyAsync(scr + p.coef_s1, table1.data(), table1.size() * 4, cudaMemcpyHostToDevice, st));
  }
  const uint8_t* crop = src + (static_cast<long long>(p.y1) * W + p.x1) * C;
  FillArgs a{};
  const int rc = C == 3 ? vae_resample_begin<3>(crop, p.ch, p.cw, W, p.rh, p.rw, p.main, scr, st, &a.base, &a.pitch)
                        : vae_resample_begin<1>(crop, p.ch, p.cw, W, p.rh, p.rw, p.main, scr, st, &a.base, &a.pitch);
  if (rc != DS_OK) return rc;
  a.coef_v = reinterpret_cast<const int*>(scr + p.main.coef_v);
  a.coef_s0 = reinterpret_cast<const int*>(scr + p.coef_s0);
  a.coef_s1 = reinterpret_cast<const int*>(scr + p.coef_s1);
  a.kv = p.main.kv;
  a.ks = p.ks;
  a.rw = p.rw;
  a.rh = p.rh;
  a.ox = p.ox;
  a.oy = p.oy;
  a.stripe = p.stripe;
  a.fill = p.fill;
  a.oh = out_h;
  a.ow = out_w;
  a.out = out;
  a.out2 = out2;
  const unsigned blocks = static_cast<unsigned>((static_cast<long long>(out_h) * out_w + 255) / 256);
  if (!mask && !adapter)
    vae_preprocess_kernel<3, DS_VAE_EPI_IMAGE><<<blocks, 256, 0, st>>>(a);
  else if (mask && C == 3)
    vae_preprocess_kernel<3, DS_VAE_EPI_MASK><<<blocks, 256, 0, st>>>(a);
  else if (mask)
    vae_preprocess_kernel<1, DS_VAE_EPI_MASK><<<blocks, 256, 0, st>>>(a);
  else if (C == 3)
    vae_preprocess_kernel<3, DS_VAE_EPI_ADAPTER><<<blocks, 256, 0, st>>>(a);
  else
    vae_preprocess_kernel<1, DS_VAE_EPI_ADAPTER><<<blocks, 256, 0, st>>>(a);
  DS_LAUNCH_OK("vae_preprocess_kernel");
  return DS_OK;
}

extern "C" int64_t ds_vae_overlay_scratch_bytes(int n, int h, int w, int H, int W, int x1, int y1, int x2, int y2) {
  ds::OverlayPlan p;
  if (!ds::plan_overlay(n, h, w, H, W, x1, y1, x2, y2, &p)) return -1;
  return p.main.total;
}

extern "C" int ds_vae_overlay(const float* image, int n, int h, int w, const uint8_t* init, const uint8_t* mask, int H,
                              int W, int x1, int y1, int x2, int y2, uint8_t* out, void* scratch,
                              int64_t scratch_bytes, void* stream) {
  using namespace ds;
  DS_REQUIRE(image && init && mask && out, "ds_vae_overlay: bad arguments");
  OverlayPlan p;
  DS_REQUIRE(plan_overlay(n, h, w, H, W, x1, y1, x2, y2, &p),
             "ds_vae_overlay: %d images of %d x %d onto crop (%d, %d, %d, %d) of a %d x %d image is not supported: the "
             "crop must lie inside the image, sides in [1, %d]", n, h, w, x1, y1, x2, y2, H, W, kMaxSide);
  DS_REQUIRE(p.main.total == 0 ||
                 (scratch && scratch_bytes >= p.main.total && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0),
             "ds_vae_overlay: needs %lld bytes of 16-byte aligned scratch (ds_vae_overlay_scratch_bytes), got %lld",
             p.main.total, static_cast<long long>(scratch_bytes));
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  unsigned char* scr = static_cast<unsigned char*>(scratch);
  const int rc = upload_lanczos_tables(h, w, p.rh, p.rw, p.main, scr, st);
  if (rc != DS_OK) return rc;
  OverlayArgs a{};
  if (p.main.kh) {
    const long long total = static_cast<long long>(n) * h * p.rw;
    const long long blocks = (total + 255) / 256;
    overlay_hpass_kernel<<<static_cast<unsigned>(blocks < 4096 ? blocks : 4096), 256, 0, st>>>(
        image, reinterpret_cast<const int*>(scr + p.main.coef_h), scr + p.main.inter, h, w, p.rw, p.main.kh, total);
    DS_LAUNCH_OK("overlay_hpass_kernel");
    a.inter = scr + p.main.inter;
  }
  a.img = image;
  a.coef_v = reinterpret_cast<const int*>(scr + p.main.coef_v);
  a.init = init;
  a.mask = mask;
  a.out = out;
  a.n = n;
  a.h = h;
  a.w = w;
  a.H = H;
  a.W = W;
  a.x1 = p.x1;
  a.y1 = p.y1;
  a.cw = p.cw;
  a.ch = p.ch;
  a.rw = p.rw;
  a.rh = p.rh;
  a.ox = p.ox;
  a.oy = p.oy;
  a.kv = p.main.kv;
  const long long total = static_cast<long long>(n) * H * W;
  vae_overlay_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(a);
  DS_LAUNCH_OK("vae_overlay_kernel");
  return DS_OK;
}
