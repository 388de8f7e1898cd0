// glue_kernels.cu — small HBM-bound kernels around the tensor-core ops: conv_in (Cin = 4), layout changes at
// the diffusers-facing boundary, nearest upsample, channel concat, SiLU, sinusoidal timestep features, and the
// fused CFG + DDIM and CFG + Euler updates (plain and inpaint, with or without guidance_rescale), the same update on a
// canvas denoised as overlapping views or under per-region prompts (MultiDiffusion), and the per-sample factors of that
// rescale.  All vectorised to 16-byte accesses where the shape allows.
#include <array>
#include <cmath>

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
// The end of every denoise step, fused: the guidance blend of the UNet's eps chunks, the scheduler update
// (src/pipelines/pipeline_diffsensei.py:315-317,332-337) and the next step's UNet input, optionally followed by the
// inpaint blend.  C == 4: one thread per pixel (8-byte bf16 vectors, 16-byte fp32 vector).  See ds_cfg_step in
// dsengine.h for the coefficient row and the formulas.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void load_cfg_halves(const uint2* __restrict__ noise_pred, long long i, long long n_pix,
                                                float u[4], float tt[4]) {
  const uint2 eu = __ldg(noise_pred + i);          // uncond half
  const uint2 et = __ldg(noise_pred + n_pix + i);  // text half
  u[0] = bf16_lo(eu.x), u[1] = bf16_hi(eu.x), u[2] = bf16_lo(eu.y), u[3] = bf16_hi(eu.y);
  tt[0] = bf16_lo(et.x), tt[1] = bf16_hi(et.x), tt[2] = bf16_lo(et.y), tt[3] = bf16_hi(et.y);
}

// A step kernel's eps of pixel i: the uncond and text halves, or with one chunk (no guidance: noise_pred holds the
// text chunk only) the text eps into tt, u left unread.
template <int kChunks>
__device__ __forceinline__ void load_eps(const uint2* __restrict__ noise_pred, long long i, long long n_pix,
                                         float u[4], float tt[4]) {
  if constexpr (kChunks == 1) {
    const uint2 et = __ldg(noise_pred + i);
    tt[0] = bf16_lo(et.x), tt[1] = bf16_hi(et.x), tt[2] = bf16_lo(et.y), tt[3] = bf16_hi(et.y);
  } else {
    load_cfg_halves(noise_pred, i, n_pix, u, tt);
  }
}

// xv <- DDIM(CFG(u, tt)) in place, the compiler free to contract into FMAs; coef = {alpha_prod_t, alpha_prod_t_prev}
__device__ __forceinline__ void cfg_ddim_pixel(const float u[4], const float tt[4], float xv[4],
                                               const float* __restrict__ coef, float guidance) {
  const float a_t = coef[0], a_prev = coef[1];
  const float sqrt_at = sqrtf(a_t), sqrt_1mat = sqrtf(1.0f - a_t);
  const float sqrt_ap = sqrtf(a_prev), sqrt_1map = sqrtf(1.0f - a_prev);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float eps = u[j] + guidance * (tt[j] - u[j]);
    const float x0 = (xv[j] - sqrt_1mat * eps) / sqrt_at;
    xv[j] = sqrt_ap * x0 + sqrt_1map * eps;
  }
}

// diffusers' DDIMScheduler.step (eta = 0) on a guided eps, each operation rounded on its own; coef = {a_t, a_prev}
__device__ __forceinline__ void ddim_update_rn(const float eps[4], float xv[4], const float* __restrict__ coef) {
  const float a_t = coef[0], a_prev = coef[1];
  const float sqrt_at = __fsqrt_rn(a_t), sqrt_1mat = __fsqrt_rn(__fsub_rn(1.0f, a_t));
  const float sqrt_ap = __fsqrt_rn(a_prev), sqrt_1map = __fsqrt_rn(__fsub_rn(1.0f, a_prev));
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float x0 = __fdiv_rn(__fsub_rn(xv[j], __fmul_rn(sqrt_1mat, eps[j])), sqrt_at);
    xv[j] = __fadd_rn(__fmul_rn(sqrt_ap, x0), __fmul_rn(sqrt_1map, eps[j]));
  }
}

// diffusers' EulerDiscreteScheduler.step (s_churn = 0) on a guided eps, each operation rounded on its own;
// coef = {sigma_i, sigma_{i+1}, ...}
__device__ __forceinline__ void euler_update_rn(const float eps[4], float xv[4], const float* __restrict__ coef) {
  const float sigma = coef[0], sigma_next = coef[1];
  const float dt = __fsub_rn(sigma_next, sigma);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float x0 = __fsub_rn(xv[j], __fmul_rn(sigma, eps[j]));
    const float d = __fdiv_rn(__fsub_rn(xv[j], x0), sigma);
    xv[j] = __fadd_rn(xv[j], __fmul_rn(d, dt));
  }
}

// diffusers' 4-channel inpaint blend after the scheduler step: where mask == 0 the pixel becomes init_proper =
// c0 * z + c1 * n (add_noise of the image latents z at the next timestep, each product and the sum rounded on its
// own as torch eager does; {c0, c1} = {1, 0} on the last step gives z); where mask == 1 it keeps the update.
__device__ __forceinline__ void inpaint_blend(float xv[4], long long i, const float4* __restrict__ image_latents,
                                              const float4* __restrict__ noise, const unsigned char* __restrict__ mask,
                                              float c0, float c1) {
  if (__ldg(mask + i)) return;
  const float4 z = __ldg(image_latents + i), n = __ldg(noise + i);
  xv[0] = __fadd_rn(__fmul_rn(c0, z.x), __fmul_rn(c1, n.x));
  xv[1] = __fadd_rn(__fmul_rn(c0, z.y), __fmul_rn(c1, n.y));
  xv[2] = __fadd_rn(__fmul_rn(c0, z.z), __fmul_rn(c1, n.z));
  xv[3] = __fadd_rn(__fmul_rn(c0, z.w), __fmul_rn(c1, n.w));
}

// The guided eps of one pixel, each operation rounded on its own: u + g (t - u), then + s (t - p) with 3 chunks (the
// perturbed chunk read here).  The step kernel and the rescale factors both use it, so the values the factors reduce
// are bit for bit the values the step rescales.
template <int kChunks>
__device__ __forceinline__ void guided_eps_rn(const uint2* __restrict__ noise_pred, long long i, long long n_pix,
                                              const float u[4], const float tt[4], float guidance, float s,
                                              float eps[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) eps[j] = __fadd_rn(u[j], __fmul_rn(guidance, __fsub_rn(tt[j], u[j])));
  if constexpr (kChunks == 3) {
    const uint2 ep = __ldg(noise_pred + 2 * n_pix + i);  // perturbed chunk
    const float pp[4] = {bf16_lo(ep.x), bf16_hi(ep.x), bf16_lo(ep.y), bf16_hi(ep.y)};
#pragma unroll
    for (int j = 0; j < 4; ++j) eps[j] = __fadd_rn(eps[j], __fmul_rn(s, __fsub_rn(tt[j], pp[j])));
  }
}

// diffusers' rescale_noise_cfg on one pixel of the guided eps, in its eager fp32 order:
// phi * (eps * r) + (1 - phi) * eps, each product and the sum rounded on its own; one_m_phi = fp32(1 - phi).
__device__ __forceinline__ void rescale_eps(float eps[4], float r, float phi, float one_m_phi) {
#pragma unroll
  for (int j = 0; j < 4; ++j) eps[j] = __fadd_rn(__fmul_rn(phi, __fmul_rn(eps[j], r)), __fmul_rn(one_m_phi, eps[j]));
}

// the next UNet input of one pixel in bf16: xv / in_div, or xv when in_div is NULL
__device__ __forceinline__ uint2 next_input(const float xv[4], const float* in_div) {
  if (!in_div) return make_uint2(pack_bf16(xv[0], xv[1]), pack_bf16(xv[2], xv[3]));
  const float d = *in_div;
  return make_uint2(pack_bf16(__fdiv_rn(xv[0], d), __fdiv_rn(xv[1], d)),
                    pack_bf16(__fdiv_rn(xv[2], d), __fdiv_rn(xv[3], d)));
}

// The guided scheduler update of one pixel: xv (the latents, loaded by the caller) <- update(guide(u, tt)), u / tt
// the pixel's uncond / text eps at index i of noise_pred, kS the PAG scale's column of coef; kRescale: the factor of
// sample i / HW is rescale[i / HW].  The step kernels share it, so a tiled step's views update exactly as untiled samples.
template <bool kEuler, int kChunks, bool kRescale, int kS>
__device__ __forceinline__ void guided_update(const uint2* __restrict__ noise_pred, long long i, long long n_pix,
                                              const float u[4], const float tt[4], float xv[4],
                                              const float* __restrict__ coef, float guidance,
                                              const float* __restrict__ rescale, int HW, float phi,
                                              float one_m_phi) {
  static_assert(kChunks > 1 || !kRescale, "guidance_rescale needs the guided eps");
  if constexpr (kChunks == 1) {
    // no guidance: the text eps as it comes, diffusers' eager scheduler.step(noise_pred_text)
    if constexpr (kEuler)
      euler_update_rn(tt, xv, coef);
    else
      ddim_update_rn(tt, xv, coef);
  } else if constexpr (!kEuler && kChunks == 2 && !kRescale) {
    // the CFG-only DDIM step has always let the compiler contract into FMAs; rounding it op by op changes its bits
    cfg_ddim_pixel(u, tt, xv, coef, guidance);
  } else {
    float eps[4];
    guided_eps_rn<kChunks>(noise_pred, i, n_pix, u, tt, guidance, kChunks == 3 ? coef[kS] : 0.f, eps);
    if constexpr (kRescale) rescale_eps(eps, __ldg(rescale + i / HW), phi, one_m_phi);
    if constexpr (kEuler)
      euler_update_rn(eps, xv, coef);
    else
      ddim_update_rn(eps, xv, coef);
  }
}

// The UNet rows of a step kernel's canvas.  noise_pred / model_in hold kChunks chunks of chunk_pixels() row pixels;
// every covering row pixel of canvas pixel i (`covering`, from its pixel(i) state) gives an update of it, their mean is
// the new canvas pixel, and every row pixel `inputs` visits gets the next UNet input.  A row pixel j's rescale factor
// is rescale[j / row_hw()].

// The plain layout: row pixel i is canvas pixel i, sample b's eps is row b of each chunk.
struct PlainRows {
  static constexpr bool kOneRow = true;  // the update is the new pixel as it is: no 0 + x (it turns -0 into +0), no / 1
  int bs, HW;
  __device__ long long canvas_pixels() const { return static_cast<long long>(bs) * HW; }
  __device__ long long chunk_pixels() const { return canvas_pixels(); }
  __device__ int row_hw() const { return HW; }
  __device__ long long pixel(long long i) const { return i; }
  template <class F>
  __device__ void covering(long long i, F&& f) const { f(i); }
  template <class F>
  __device__ void inputs(long long i, F&& f) const { f(i); }
};

// MultiDiffusion's view grid on one latent axis: n views of `size` pixels, view k at min(k * stride, dim - size) (the
// last one flush with the far edge), 0 < stride <= size <= dim.  Every coordinate has at least one covering view.
struct TileAxis {
  int dim, size, stride, n;
};

__device__ __forceinline__ int tile_origin(const TileAxis& a, int k) { return min(k * a.stride, a.dim - a.size); }

// the views [lo, hi] that cover coordinate p: a contiguous range, from integer arithmetic on the grid alone
__device__ __forceinline__ void tile_cover(const TileAxis& a, int p, int& lo, int& hi) {
  lo = p < a.size ? 0 : min((p - a.size) / a.stride + 1, a.n - 1);
  hi = p >= a.dim - a.size ? a.n - 1 : p / a.stride;
}

// The tiled layout (MultiDiffusion, Bar-Tal et al. 2023): the canvas [bs][ay.dim][ax.dim] denoised as bs * V views
// (row b * V + v, v = vy * ax.n + vx) of ay.size x ax.size pixels.  The covering views of a canvas pixel, in view
// order, update it, and the same views get its next UNet input (diffusers' panorama loop: value += x_view, then
// value / count).
struct TileRows {
  static constexpr bool kOneRow = false;
  TileAxis ay, ax;
  int bs;
  __device__ long long canvas_pixels() const { return static_cast<long long>(bs) * ay.dim * ax.dim; }
  __device__ long long chunk_pixels() const { return static_cast<long long>(bs) * ay.n * ax.n * row_hw(); }
  __device__ int row_hw() const { return ay.size * ax.size; }
  struct Pixel {
    int b, y, x, ylo, yhi, xlo, xhi;  // the canvas pixel and its covering views [ylo, yhi] x [xlo, xhi]
  };
  __device__ Pixel pixel(long long i) const {
    Pixel p;
    p.x = static_cast<int>(i % ax.dim);
    const long long by = i / ax.dim;
    p.y = static_cast<int>(by % ay.dim);
    p.b = static_cast<int>(by / ay.dim);
    tile_cover(ay, p.y, p.ylo, p.yhi);
    tile_cover(ax, p.x, p.xlo, p.xhi);
    return p;
  }
  template <class F>
  __device__ void covering(const Pixel& p, F&& f) const {
    const int views = ay.n * ax.n, view_hw = row_hw();
    for (int vy = p.ylo; vy <= p.yhi; ++vy) {
      const long long row0 = (static_cast<long long>(p.b) * views + vy * ax.n) * view_hw +
                             static_cast<long long>(p.y - tile_origin(ay, vy)) * ax.size;
      for (int vx = p.xlo; vx <= p.xhi; ++vx)
        f(row0 + vx * static_cast<long long>(view_hw) + (p.x - tile_origin(ax, vx)));
    }
  }
  template <class F>
  __device__ void inputs(const Pixel& p, F&& f) const { covering(p, f); }
};

// The regional layout (MultiDiffusion's region-based generation, Bar-Tal et al. 2023 sec. 4.2): the canvas [bs][HW]
// under R1 prompts, row b * R1 + r sample b under prompt r (r = 0 the background, r = 1 .. R1 - 1 the regions), every
// row's input the whole canvas.  cover: uint8 [bs][HW], bit r - 1 set <=> region r covers the pixel (bits at or above
// R1 - 1 are ignored); the background covers exactly the pixels whose byte is 0.  The covering rows, in row order,
// update a canvas pixel; all R1 rows get its next UNet input.
struct RegionRows {
  static constexpr bool kOneRow = false;
  const unsigned char* cover;
  int R1, bs, HW;
  __device__ long long canvas_pixels() const { return static_cast<long long>(bs) * HW; }
  __device__ long long chunk_pixels() const { return static_cast<long long>(bs) * R1 * HW; }
  __device__ int row_hw() const { return HW; }
  struct Pixel {
    long long row0;  // the pixel in row b * R1 (the background)
    unsigned rows;   // bit r set <=> row r covers the pixel
  };
  __device__ Pixel pixel(long long i) const {
    const long long b = i / HW;
    const unsigned bits = __ldg(cover + i) & ((1u << (R1 - 1)) - 1u);
    return {b * R1 * HW + (i - b * HW), bits ? bits << 1 : 1u};
  }
  template <class F>
  __device__ void covering(const Pixel& p, F&& f) const {
    for (unsigned m = p.rows; m != 0; m &= m - 1) f(p.row0 + static_cast<long long>(__ffs(m) - 1) * HW);
  }
  template <class F>
  __device__ void inputs(const Pixel& p, F&& f) const {
    for (int r = 0; r < R1; ++r) f(p.row0 + static_cast<long long>(r) * HW);
  }
};

// The step, one thread per canvas pixel.  noise_pred holds kChunks chunks of the layout's rows, [uncond ; text
// (; perturbed)], or [text] with no guidance; coef is the step's row {update (2 DDIM, 3 Euler) | c0, c1 if kInpaint |
// s if kChunks == 3}.  kRescale: the guided eps of row pixel j is rescaled with the factor rescale[j / row_hw()]
// (cfg_rescale_factors_kernel) before the update.  Every covering row's x_new is computed from the canvas pixel by
// guided_update; their fp32 sum, in the layout's order from 0, over the count is the new canvas pixel (one row in the
// plain layout: its x_new itself), then the inpaint blend on the canvas, then the canvas and the next UNet input into
// every chunk of the rows `inputs` visits.  Each output element is written by one thread once.
template <class Rows, bool kEuler, int kChunks, bool kInpaint, bool kRescale>
__global__ void cfg_step_kernel(const uint2* __restrict__ noise_pred, float4* __restrict__ latents,
                                uint2* __restrict__ model_in, const float* __restrict__ coef, float guidance, Rows rows,
                                const float4* __restrict__ image_latents, const float4* __restrict__ noise,
                                const unsigned char* __restrict__ mask, const float* __restrict__ rescale, float phi,
                                float one_m_phi) {
  static_assert(1 <= kChunks && kChunks <= 3, "no guidance (1 chunk), CFG (2) or CFG + PAG (3)");
  constexpr int kC0 = kEuler ? 3 : 2;                 // {c0, c1} follow the update's coefficients
  constexpr int kS = kC0 + (kInpaint ? 2 : 0);         // then the PAG scale
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= rows.canvas_pixels()) return;
  const long long n_pix = rows.chunk_pixels();
  const auto px = rows.pixel(i);
  const float4 xc = latents[i];
  // x_new of the canvas pixel from row pixel j's eps
  auto update = [&](long long j, float xv[4]) {
    float u[4], tt[4];
    load_eps<kChunks>(noise_pred, j, n_pix, u, tt);
    xv[0] = xc.x, xv[1] = xc.y, xv[2] = xc.z, xv[3] = xc.w;
    guided_update<kEuler, kChunks, kRescale, kS>(noise_pred, j, n_pix, u, tt, xv, coef, guidance, rescale,
                                                 rows.row_hw(), phi, one_m_phi);
  };
  float xv[4];
  if constexpr (Rows::kOneRow) {
    update(i, xv);
  } else {
    float sum[4] = {0.f, 0.f, 0.f, 0.f};
    int count = 0;
    rows.covering(px, [&](long long j) {
      float x[4];
      update(j, x);
#pragma unroll
      for (int c = 0; c < 4; ++c) sum[c] = __fadd_rn(sum[c], x[c]);
      ++count;
    });
#pragma unroll
    for (int c = 0; c < 4; ++c) xv[c] = __fdiv_rn(sum[c], static_cast<float>(count));
  }
  if constexpr (kInpaint) inpaint_blend(xv, i, image_latents, noise, mask, coef[kC0], coef[kC0 + 1]);
  latents[i] = make_float4(xv[0], xv[1], xv[2], xv[3]);
  const uint2 o = next_input(xv, kEuler ? coef + 2 : nullptr);
  rows.inputs(px, [&](long long j) {
#pragma unroll
    for (int c = 0; c < kChunks; ++c) model_in[c * n_pix + j] = o;
  });
}

// The 20 step kernels of one row layout, [update][chunks - 1][inpaint][rescale]; 1 chunk has no rescale kernel.
template <class Rows>
struct StepKernels {
  using Fn = void (*)(const uint2*, float4*, uint2*, const float*, float, Rows, const float4*, const float4*,
                      const unsigned char*, const float*, float, float);
  using Variants = std::array<std::array<Fn, 2>, 2>;  // [inpaint][rescale]
  template <bool kEuler, int kChunks, bool kInpaint, bool kRescale>
  static constexpr Fn kernel() {
    if constexpr (kChunks == 1 && kRescale)
      return nullptr;  // guidance_rescale needs the guided eps
    else
      return cfg_step_kernel<Rows, kEuler, kChunks, kInpaint, kRescale>;
  }
  template <bool kEuler, int kChunks>
  static constexpr Variants variants() {
    return {{{kernel<kEuler, kChunks, false, false>(), kernel<kEuler, kChunks, false, true>()},
             {kernel<kEuler, kChunks, true, false>(), kernel<kEuler, kChunks, true, true>()}}};
  }
  static constexpr std::array<std::array<Variants, 3>, 2> kTable = {{
      {variants<false, 1>(), variants<false, 2>(), variants<false, 3>()},
      {variants<true, 1>(), variants<true, 2>(), variants<true, 3>()}}};
};

template <class Rows>
void launch_step(const Rows& rows, long long n_canvas, int update, int chunks, bool inpaint, bool rescale,
                 const void* noise_pred, float* latents, void* model_in, const float* coef, float guidance,
                 const float* image_latents, const float* noise, const uint8_t* mask, const float* rescale_factors,
                 double guidance_rescale, cudaStream_t stream) {
  StepKernels<Rows>::kTable[update][chunks - 1][inpaint][rescale]<<<static_cast<unsigned>((n_canvas + 255) / 256), 256,
                                                                    0, stream>>>(
      static_cast<const uint2*>(noise_pred), reinterpret_cast<float4*>(latents), static_cast<uint2*>(model_in), coef,
      guidance, rows, reinterpret_cast<const float4*>(image_latents), reinterpret_cast<const float4*>(noise), mask,
      // phi and 1 - phi (in double) each rounded to fp32 once: torch's values of the Python scalars for an fp32 tensor
      rescale_factors, static_cast<float>(guidance_rescale), static_cast<float>(1.0 - guidance_rescale));
}

// guidance_rescale's per-sample factor r_b = fp32(std(text_b)) / fp32(std(guided_b)), both unbiased over the sample's
// 4 * HW values.  One CTA per sample: every thread walks a fixed set of pixels, accumulating in fp64 the sums of
// x - k and (x - k)^2 (k: the sample's first value, so a constant sample gives exactly 0), then a fixed-order tree
// (warp shuffles, then the warps in order) combines them.  No atomics: a sample's factor has the same bits whatever
// the batch around it.
constexpr int kRescaleThreads = 512;

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

template <int kChunks>
__global__ void __launch_bounds__(kRescaleThreads) cfg_rescale_factors_kernel(
    const uint2* __restrict__ noise_pred, const float* __restrict__ coef, int s_col, float guidance,
    float* __restrict__ factors, int HW, long long n_pix) {
  __shared__ double part[kRescaleThreads / 32][4];
  const long long base = static_cast<long long>(blockIdx.x) * HW;
  const float s = kChunks == 3 ? coef[s_col] : 0.f;
  float u[4], tt[4], e[4];
  load_cfg_halves(noise_pred, base, n_pix, u, tt);
  guided_eps_rn<kChunks>(noise_pred, base, n_pix, u, tt, guidance, s, e);
  const double kt = tt[0], kc = e[0];
  double st = 0.0, st2 = 0.0, sc = 0.0, sc2 = 0.0;
  for (int p = threadIdx.x; p < HW; p += kRescaleThreads) {
    load_cfg_halves(noise_pred, base + p, n_pix, u, tt);
    guided_eps_rn<kChunks>(noise_pred, base + p, n_pix, u, tt, guidance, s, e);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const double dt = static_cast<double>(tt[j]) - kt, dc = static_cast<double>(e[j]) - kc;
      st += dt;
      st2 = fma(dt, dt, st2);
      sc += dc;
      sc2 = fma(dc, dc, sc2);
    }
  }
  st = warp_sum_f64(st), st2 = warp_sum_f64(st2), sc = warp_sum_f64(sc), sc2 = warp_sum_f64(sc2);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) part[warp][0] = st, part[warp][1] = st2, part[warp][2] = sc, part[warp][3] = sc2;
  __syncthreads();
  if (threadIdx.x == 0) {
    double a[4] = {0.0, 0.0, 0.0, 0.0};
    for (int w = 0; w < kRescaleThreads / 32; ++w)
#pragma unroll
      for (int k = 0; k < 4; ++k) a[k] += part[w][k];
    const double n = 4.0 * HW;
    // unbiased variance of the shifted values; rounding can leave it a hair below 0 only when it is ~0
    const double var_t = fmax((a[1] - a[0] * a[0] / n) / (n - 1.0), 0.0);
    const double var_c = fmax((a[3] - a[2] * a[2] / n) / (n - 1.0), 0.0);
    factors[blockIdx.x] = __fdiv_rn(__double2float_rn(sqrt(var_t)), __double2float_rn(sqrt(var_c)));
  }
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

extern "C" int ds_cfg_step(const void* noise_pred, float* latents, void* model_in, const float* coef, float guidance,
                           int update, int chunks, const float* image_latents, const float* noise, const uint8_t* mask,
                           const float* rescale_factors, double guidance_rescale, const ds_step_rows* rows, int bs,
                           int H, int W, int C, void* stream) {
  const bool inpaint = image_latents || noise || mask;
  const bool rescale = rescale_factors != nullptr;
  const bool views = rows && (rows->tile_h || rows->tile_w || rows->stride_h || rows->stride_w);
  const bool regions = rows && (rows->cover || rows->n_regions);
  DS_REQUIRE(noise_pred && latents && model_in && coef && (!regions || rows->cover), "ds_cfg_step: NULL pointer");
  DS_REQUIRE(!inpaint || (image_latents && noise && mask),
             "ds_cfg_step: image_latents / noise / mask must all be given or all be NULL");
  DS_REQUIRE(update == 0 || update == 1, "ds_cfg_step: update must be 0 (DDIM) or 1 (Euler), got %d", update);
  DS_REQUIRE(1 <= chunks && chunks <= 3,
             "ds_cfg_step: chunks must be 2 or 3 (CFG, CFG + PAG) or 1 (no guidance), got %d", chunks);
  DS_REQUIRE(chunks > 1 || !rescale, "ds_cfg_step: rescale_factors must be NULL with 1 chunk (no guidance)");
  DS_REQUIRE(!(views && regions), "ds_cfg_step: rows sets both views and regions");
  DS_REQUIRE(!regions || (1 <= rows->n_regions && rows->n_regions <= 8),
             "ds_cfg_step: n_regions must be in [1, 8], got %d", rows->n_regions);
  DS_REQUIRE(bs > 0 && H > 0 && W > 0 && C == 4, "ds_cfg_step: only C == 4 latents are supported (got C=%d)", C);
  DS_REQUIRE(!views || (0 < rows->tile_h && rows->tile_h <= H && 0 < rows->tile_w && rows->tile_w <= W),
             "ds_cfg_step: the view (%d x %d) must fit the canvas (%d x %d)", rows->tile_h, rows->tile_w, H, W);
  DS_REQUIRE(!views || (0 < rows->stride_h && rows->stride_h <= rows->tile_h && 0 < rows->stride_w &&
                        rows->stride_w <= rows->tile_w),
             "ds_cfg_step: the stride (%d, %d) must be in (0, view size]", rows->stride_h, rows->stride_w);
  DS_REQUIRE((reinterpret_cast<uintptr_t>(latents) & 15) == 0 && (reinterpret_cast<uintptr_t>(noise_pred) & 7) == 0 &&
                 (reinterpret_cast<uintptr_t>(model_in) & 7) == 0,
             "ds_cfg_step: latents must be 16-byte and noise_pred / model_in 8-byte aligned");
  DS_REQUIRE(!inpaint || ((reinterpret_cast<uintptr_t>(image_latents) & 15) == 0 &&
                          (reinterpret_cast<uintptr_t>(noise) & 15) == 0),
             "ds_cfg_step: image_latents / noise must be 16-byte aligned");
  DS_REQUIRE(rescale ? std::isfinite(guidance_rescale) : guidance_rescale == 0.0,
             "ds_cfg_step: guidance_rescale must be finite, and 0 when rescale_factors is NULL (got %g)",
             guidance_rescale);
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long n_canvas = static_cast<long long>(bs) * H * W;
  const auto s = static_cast<cudaStream_t>(stream);
  if (views) {
    const ds_step_rows& v = *rows;
    // n views per axis: ceil((dim - size) / stride) + 1, the last one flush with the far edge
    const TileAxis ay{H, v.tile_h, v.stride_h, (H - v.tile_h + v.stride_h - 1) / v.stride_h + 1};
    const TileAxis ax{W, v.tile_w, v.stride_w, (W - v.tile_w + v.stride_w - 1) / v.stride_w + 1};
    launch_step(TileRows{ay, ax, bs}, n_canvas, update, chunks, inpaint, rescale, noise_pred, latents, model_in, coef,
                guidance, image_latents, noise, mask, rescale_factors, guidance_rescale, s);
  } else if (regions) {
    launch_step(RegionRows{static_cast<const unsigned char*>(rows->cover), rows->n_regions + 1, bs, H * W}, n_canvas,
                update, chunks, inpaint, rescale, noise_pred, latents, model_in, coef, guidance, image_latents, noise,
                mask, rescale_factors, guidance_rescale, s);
  } else {
    launch_step(PlainRows{bs, H * W}, n_canvas, update, chunks, inpaint, rescale, noise_pred, latents, model_in, coef,
                guidance, image_latents, noise, mask, rescale_factors, guidance_rescale, s);
  }
  DS_LAUNCH_OK("cfg_step_kernel");
  return DS_OK;
}

extern "C" int ds_cfg_rescale_factors(const void* noise_pred, const float* coef, int ncoef, float guidance, int chunks,
                                      float* factors, int bs, int HW, int C, void* stream) {
  DS_REQUIRE(noise_pred && coef && factors, "ds_cfg_rescale_factors: NULL pointer");
  DS_REQUIRE(chunks == 2 || chunks == 3, "ds_cfg_rescale_factors: chunks must be 2 or 3, got %d", chunks);
  DS_REQUIRE(chunks == 2 || ncoef > 0, "ds_cfg_rescale_factors: 3 chunks read the PAG scale at coef[ncoef - 1]");
  DS_REQUIRE(bs > 0 && HW > 0 && C == 4, "ds_cfg_rescale_factors: only C == 4 latents are supported (got C=%d)", C);
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long n_pix = static_cast<long long>(bs) * HW;
  auto kernel = chunks == 2 ? cfg_rescale_factors_kernel<2> : cfg_rescale_factors_kernel<3>;
  kernel<<<bs, kRescaleThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint2*>(noise_pred), coef, ncoef - 1, guidance, factors, HW, n_pix);
  DS_LAUNCH_OK("cfg_rescale_factors_kernel");
  return DS_OK;
}
