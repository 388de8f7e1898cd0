// llm_kernels.cu — the LLaMA decoder of the MLLM agent (SURVEY.md §8f-4: ContinuousLVLM.generate,
// src/models/mllm/seed_x.py:90-171, around LlamaForCausalLM of src/models/mllm/modeling_llama_xformer.py).
//
// A greedy decode at batch 1 reads every weight once per token (25.7 GB at 13B in bf16), so the decode linears are a
// weight-streaming GEMV rather than a tensor-core GEMM; the prefill linears run on ds_gemm_bf16.  Everything else a
// decode step needs is here too, and every kernel reads the current position from DEVICE memory, so one captured
// graph serves every step:
//   ds_gemv_bf16        : y[M][N] = x[M][K] W[N][K]^T (+ residual), M <= 8, K-major W streamed once with 16-byte
//                         non-allocating loads, x staged in shared memory, rows reduced with warp shuffles
//   ds_rmsnorm          : LlamaRMSNorm, fp32 statistics, one rounding
//   ds_rope_kv_append   : rotate-half RoPE of q and k, append k / v to the layer's [2][H][L_max][D] cache
//   ds_attention_kv     : split-KV attention of M query rows against the cache (bottom-right causal) + combine pass
//   ds_silu_mul         : silu(gate) * up of the fused gate|up projection
//   ds_agent_next_token : the image-token logits rule + greedy argmax + stop flag + next input row, on the device
// and, for B <= 8 sequences decoded together (one row each, each with its own position and cache slice):
//   ds_rope_kv_append_rows, ds_attention_kv_rows, ds_agent_next_token_rows
// The per-row arithmetic of each *_rows kernel is the same __device__ function its batch-1 kernel calls, so a row
// computes bit for bit what the batch-1 decode computes for that sequence alone.
// Every kernel is launched with programmatic dependent launch and waits for its predecessor before its first access
// to global memory.
#include "ds_common.cuh"
#include "ds_host.h"

namespace ds {

// ----------------------------------------------------------------------------------------------- GEMV
constexpr int kGemvThreads = 256;    // 8 warps
constexpr int kGemvRowsPerWarp = 2;  // output rows a warp streams side by side
constexpr int kGemvUnroll = 4;       // 16-byte chunks per row in flight per lane

__device__ __forceinline__ uint4 ld_stream(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

__device__ __forceinline__ float dot8(const uint4 w, const uint4 x) {
  float a = bf16_lo(w.x) * bf16_lo(x.x);
  a = fmaf(bf16_hi(w.x), bf16_hi(x.x), a);
  a = fmaf(bf16_lo(w.y), bf16_lo(x.y), a);
  a = fmaf(bf16_hi(w.y), bf16_hi(x.y), a);
  a = fmaf(bf16_lo(w.z), bf16_lo(x.z), a);
  a = fmaf(bf16_hi(w.z), bf16_hi(x.z), a);
  a = fmaf(bf16_lo(w.w), bf16_lo(x.w), a);
  a = fmaf(bf16_hi(w.w), bf16_hi(x.w), a);
  return a;
}

template <int M>
__global__ void __launch_bounds__(kGemvThreads)
gemv_bf16_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                 const __nv_bfloat16* residual, void* y, int N, int K, int out_fp32) {   // y may alias residual
  extern __shared__ uint4 sx[];                       // [M][K/8]
  const int kc = K >> 3;
  pdl_wait();
  pdl_launch_dependents();
  for (int i = threadIdx.x; i < M * kc; i += kGemvThreads) sx[i] = reinterpret_cast<const uint4*>(x)[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = (blockIdx.x * (kGemvThreads / 32) + warp) * kGemvRowsPerWarp;
  if (n0 >= N) return;
  const uint4* wr[kGemvRowsPerWarp];
#pragma unroll
  for (int r = 0; r < kGemvRowsPerWarp; ++r)
    wr[r] = reinterpret_cast<const uint4*>(w + static_cast<size_t>(min(n0 + r, N - 1)) * K);   // odd N: row re-read
  float acc[kGemvRowsPerWarp][M];
#pragma unroll
  for (int r = 0; r < kGemvRowsPerWarp; ++r)
#pragma unroll
    for (int m = 0; m < M; ++m) acc[r][m] = 0.f;
  int c = lane;
  for (; c + 32 * (kGemvUnroll - 1) < kc; c += 32 * kGemvUnroll) {
    uint4 wv[kGemvRowsPerWarp][kGemvUnroll];
#pragma unroll
    for (int r = 0; r < kGemvRowsPerWarp; ++r)
#pragma unroll
      for (int u = 0; u < kGemvUnroll; ++u) wv[r][u] = ld_stream(wr[r] + c + 32 * u);
#pragma unroll
    for (int u = 0; u < kGemvUnroll; ++u)
#pragma unroll
      for (int m = 0; m < M; ++m) {
        const uint4 xv = sx[m * kc + c + 32 * u];
#pragma unroll
        for (int r = 0; r < kGemvRowsPerWarp; ++r) acc[r][m] += dot8(wv[r][u], xv);
      }
  }
  for (; c < kc; c += 32) {
    uint4 wv[kGemvRowsPerWarp];
#pragma unroll
    for (int r = 0; r < kGemvRowsPerWarp; ++r) wv[r] = ld_stream(wr[r] + c);
#pragma unroll
    for (int m = 0; m < M; ++m) {
      const uint4 xv = sx[m * kc + c];
#pragma unroll
      for (int r = 0; r < kGemvRowsPerWarp; ++r) acc[r][m] += dot8(wv[r], xv);
    }
  }
#pragma unroll
  for (int r = 0; r < kGemvRowsPerWarp; ++r)
#pragma unroll
    for (int m = 0; m < M; ++m) acc[r][m] = warp_sum(acc[r][m]);
  // lane (r * M + m) writes output (m, n0 + r)
#pragma unroll
  for (int r = 0; r < kGemvRowsPerWarp; ++r)
#pragma unroll
    for (int m = 0; m < M; ++m) {
      const int n = n0 + r;
      if (lane == r * M + m && n < N) {
        float v = acc[r][m];
        const size_t o = static_cast<size_t>(m) * N + n;
        if (residual) v += __bfloat162float(residual[o]);
        if (out_fp32) static_cast<float*>(y)[o] = v;
        else static_cast<__nv_bfloat16*>(y)[o] = __float2bfloat16_rn(v);
      }
    }
}

// ----------------------------------------------------------------------------------------------- RMSNorm
constexpr int kNormThreads = 256;

__global__ void __launch_bounds__(kNormThreads)
rmsnorm_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma, __nv_bfloat16* __restrict__ y,
               int C, float eps) {
  __shared__ float red[kNormThreads / 32];
  pdl_wait();
  pdl_launch_dependents();
  const uint4* xr = reinterpret_cast<const uint4*>(x + static_cast<size_t>(blockIdx.x) * C);
  uint4* yr = reinterpret_cast<uint4*>(y + static_cast<size_t>(blockIdx.x) * C);
  constexpr int kMaxVec = 8192 / 8 / kNormThreads;    // C <= 8192
  uint4 v[kMaxVec];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int c = threadIdx.x + i * kNormThreads;
    if (c < C / 8) {
      v[i] = xr[c];
      const uint32_t* p = &v[i].x;
#pragma unroll
      for (int j = 0; j < 4; ++j) ss += bf16_lo(p[j]) * bf16_lo(p[j]) + bf16_hi(p[j]) * bf16_hi(p[j]);
    }
  }
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < kNormThreads / 32; ++i) tot += red[i];
  const float rstd = rsqrtf(tot / C + eps);
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int c = threadIdx.x + i * kNormThreads;
    if (c < C / 8) {
      const float4 g0 = reinterpret_cast<const float4*>(gamma)[2 * c];
      const float4 g1 = reinterpret_cast<const float4*>(gamma)[2 * c + 1];
      uint4 o;
      o.x = pack_bf16(bf16_lo(v[i].x) * rstd * g0.x, bf16_hi(v[i].x) * rstd * g0.y);
      o.y = pack_bf16(bf16_lo(v[i].y) * rstd * g0.z, bf16_hi(v[i].y) * rstd * g0.w);
      o.z = pack_bf16(bf16_lo(v[i].z) * rstd * g1.x, bf16_hi(v[i].z) * rstd * g1.y);
      o.w = pack_bf16(bf16_lo(v[i].w) * rstd * g1.z, bf16_hi(v[i].w) * rstd * g1.w);
      yr[c] = o;
    }
  }
}

// ----------------------------------------------------------------------------------------------- RoPE + KV append
// One row at position p: rotates q and k of `row` ([3][H][D]), writes q to qo and appends k / v at row p of the
// [2][H][L_max][D] cache kv.  Shared by the prefill / batch-1 kernel and the one-sequence-per-row kernel.
__device__ __forceinline__ void rope_kv_append_row(const __nv_bfloat16* __restrict__ row, __nv_bfloat16* __restrict__ qo,
                                                   __nv_bfloat16* __restrict__ kv, int p, int H, int D, int L_max,
                                                   float theta) {
  const int half = D / 2, C = H * D;
  for (int t = threadIdx.x; t < H * half; t += blockDim.x) {
    const int h = t / half, i = t - h * half;
    // inv_freq = theta^(-2i/D) in fp32, angle = p * inv_freq in fp32 (LlamaRotaryEmbedding)
    const float inv_freq = 1.0f / powf(theta, static_cast<float>(2 * i) / static_cast<float>(D));
    float s, c;
    sincosf(static_cast<float>(p) * inv_freq, &s, &c);
    const int a = h * D + i, b = a + half;
    const float q1 = __bfloat162float(row[a]), q2 = __bfloat162float(row[b]);
    const float k1 = __bfloat162float(row[C + a]), k2 = __bfloat162float(row[C + b]);
    qo[a] = __float2bfloat16_rn(q1 * c - q2 * s);
    qo[b] = __float2bfloat16_rn(q2 * c + q1 * s);
    __nv_bfloat16* kr = kv + (static_cast<size_t>(h) * L_max + p) * D;
    kr[i] = __float2bfloat16_rn(k1 * c - k2 * s);
    kr[i + half] = __float2bfloat16_rn(k2 * c + k1 * s);
  }
  __nv_bfloat16* vbase = kv + static_cast<size_t>(H) * L_max * D;
  for (int t = threadIdx.x; t < C; t += blockDim.x) {
    const int h = t / D, d = t - h * D;
    vbase[(static_cast<size_t>(h) * L_max + p) * D + d] = row[2 * C + t];
  }
}

// row m of one sequence at position *pos_ptr + m (prefill and batch-1 decode)
__global__ void __launch_bounds__(256)
rope_kv_append_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ q_out,
                      __nv_bfloat16* __restrict__ kv, const int* __restrict__ pos_ptr, int H, int D, int L_max,
                      float theta) {
  pdl_wait();
  pdl_launch_dependents();
  const int m = blockIdx.x;
  const int p = *pos_ptr + m;
  if (p < 0 || p >= L_max) return;
  const int C = H * D;
  rope_kv_append_row(qkv + static_cast<size_t>(m) * 3 * C, q_out + static_cast<size_t>(m) * C, kv, p, H, D, L_max,
                     theta);
}

// row b is its own sequence at position pos[b * pos_stride], with its cache slice at kv + b * seq_stride
__global__ void __launch_bounds__(256)
rope_kv_append_rows_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ q_out,
                           __nv_bfloat16* __restrict__ kv, long long seq_stride, const int* __restrict__ pos,
                           int pos_stride, int H, int D, int L_cap, float theta) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.x;
  const int p = pos[static_cast<size_t>(b) * pos_stride];
  if (p < 0 || p >= L_cap) return;
  const int C = H * D;
  rope_kv_append_row(qkv + static_cast<size_t>(b) * 3 * C, q_out + static_cast<size_t>(b) * C, kv + b * seq_stride,
                     p, H, D, L_cap, theta);
}

// ----------------------------------------------------------------------------------------------- attention
constexpr int kAttnWarps = 4;
constexpr int kAttnMaxVec = 4;   // D / 32 values per lane: D = 128 -> 4, D = 64 -> 2

// Keys j0 .. j1-1 of one split for one (query row, head): the CTA's warps stride over the keys with an online softmax
// per warp, merge in shared memory, and leave {max, sum, o[D]} of the split in `part` for the combine pass.
// qr: the row's q of this head [D]; kh / vh: this head's keys / values [L][D].
template <int DV>
__device__ __forceinline__ void attention_kv_split_part(const __nv_bfloat16* __restrict__ qr,
                                                        const __nv_bfloat16* __restrict__ kh,
                                                        const __nv_bfloat16* __restrict__ vh, float* __restrict__ part,
                                                        int j0, int j1, float scale) {
  constexpr int D = DV * 32;
  __shared__ float s_m[kAttnWarps], s_l[kAttnWarps];
  __shared__ float s_o[kAttnWarps][D];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float qf[DV];
#pragma unroll
  for (int i = 0; i < DV; ++i) qf[i] = __bfloat162float(qr[lane * DV + i]) * scale;
  const __nv_bfloat16* kb = kh + lane * DV;
  const __nv_bfloat16* vb = vh + lane * DV;
  float mx = -INFINITY, l = 0.f, o[DV];
#pragma unroll
  for (int i = 0; i < DV; ++i) o[i] = 0.f;
  for (int j = j0 + warp; j < j1; j += kAttnWarps) {
    float kf[DV], vf[DV];
    if constexpr (DV == 4) {
      const uint2 ku = *reinterpret_cast<const uint2*>(kb + static_cast<size_t>(j) * D);
      const uint2 vu = *reinterpret_cast<const uint2*>(vb + static_cast<size_t>(j) * D);
      kf[0] = bf16_lo(ku.x); kf[1] = bf16_hi(ku.x); kf[2] = bf16_lo(ku.y); kf[3] = bf16_hi(ku.y);
      vf[0] = bf16_lo(vu.x); vf[1] = bf16_hi(vu.x); vf[2] = bf16_lo(vu.y); vf[3] = bf16_hi(vu.y);
    } else {
      const uint32_t ku = *reinterpret_cast<const uint32_t*>(kb + static_cast<size_t>(j) * D);
      const uint32_t vu = *reinterpret_cast<const uint32_t*>(vb + static_cast<size_t>(j) * D);
      kf[0] = bf16_lo(ku); kf[1] = bf16_hi(ku);
      vf[0] = bf16_lo(vu); vf[1] = bf16_hi(vu);
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < DV; ++i) s = fmaf(qf[i], kf[i], s);
    s = warp_sum(s);
    const float mn = fmaxf(mx, s);
    const float corr = __expf(mx - mn), p = __expf(s - mn);
    l = l * corr + p;
#pragma unroll
    for (int i = 0; i < DV; ++i) o[i] = fmaf(o[i], corr, p * vf[i]);
    mx = mn;
  }
  if (lane == 0) { s_m[warp] = mx; s_l[warp] = l; }
#pragma unroll
  for (int i = 0; i < DV; ++i) s_o[warp][lane * DV + i] = o[i];
  __syncthreads();
  if (warp != 0) return;
  float M_ = -INFINITY;
#pragma unroll
  for (int w = 0; w < kAttnWarps; ++w) M_ = fmaxf(M_, s_m[w]);
  float L_ = 0.f, acc[DV];
#pragma unroll
  for (int i = 0; i < DV; ++i) acc[i] = 0.f;
#pragma unroll
  for (int w = 0; w < kAttnWarps; ++w) {
    const float f = s_m[w] == -INFINITY ? 0.f : __expf(s_m[w] - M_);   // a warp that saw no key
    L_ += s_l[w] * f;
#pragma unroll
    for (int i = 0; i < DV; ++i) acc[i] += s_o[w][lane * DV + i] * f;
  }
  if (lane == 0) { part[0] = M_; part[1] = L_; }
#pragma unroll
  for (int i = 0; i < DV; ++i) part[2 + lane * DV + i] = acc[i];
}

// Merges the `used` split partials at `base` (stride D + 2) into element d of the output row.
__device__ __forceinline__ void attention_kv_combine_part(const float* __restrict__ base, __nv_bfloat16* __restrict__ o,
                                                          int used, int D, int d) {
  float M_ = -INFINITY;
  for (int s = 0; s < used; ++s) M_ = fmaxf(M_, base[s * (D + 2)]);
  float L_ = 0.f, acc = 0.f;
  for (int s = 0; s < used; ++s) {
    const float f = __expf(base[s * (D + 2)] - M_);
    L_ += base[s * (D + 2) + 1] * f;
    acc += base[s * (D + 2) + 2 + d] * f;
  }
  o[d] = __float2bfloat16_rn(acc / L_);
}

// One CTA per (split, head, query row) of one sequence; row m sees keys 0 .. *pos_ptr + m (bottom-right causal).
template <int DV>
__global__ void __launch_bounds__(kAttnWarps * 32)
attention_kv_split_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ kv,
                          float* __restrict__ ws, const int* __restrict__ pos_ptr, int H, int L_max, int chunk,
                          int splits, float scale) {
  constexpr int D = DV * 32;
  pdl_wait();
  pdl_launch_dependents();
  const int split = blockIdx.x, h = blockIdx.y, m = blockIdx.z;
  const int nkeys = min(*pos_ptr + m + 1, L_max);
  const int j0 = split * chunk, j1 = min(j0 + chunk, nkeys);
  if (j0 >= j1) return;
  const __nv_bfloat16* kh = kv + static_cast<size_t>(h) * L_max * D;
  attention_kv_split_part<DV>(q + (static_cast<size_t>(m) * H + h) * D, kh, kh + static_cast<size_t>(H) * L_max * D,
                              ws + ((static_cast<size_t>(m) * H + h) * splits + split) * (D + 2), j0, j1, scale);
}

__global__ void attention_kv_combine_kernel(const float* __restrict__ ws, __nv_bfloat16* __restrict__ out,
                                            const int* __restrict__ pos_ptr, int H, int D, int L_max, int chunk,
                                            int splits) {
  pdl_wait();
  pdl_launch_dependents();
  const int h = blockIdx.x, m = blockIdx.y;
  const int nkeys = min(*pos_ptr + m + 1, L_max);
  const int used = min((nkeys + chunk - 1) / chunk, splits);
  attention_kv_combine_part(ws + (static_cast<size_t>(m) * H + h) * splits * (D + 2),
                            out + (static_cast<size_t>(m) * H + h) * D, used, D, threadIdx.x);
}

// One CTA per (split, head, row b); row b is its own sequence: keys 0 .. pos[b * pos_stride] of the cache slice at
// kv + b * seq_stride.  With the same chunk, every split covers the same keys as the batch-1 decode's.
template <int DV>
__global__ void __launch_bounds__(kAttnWarps * 32)
attention_kv_rows_split_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ kv,
                               long long seq_stride, float* __restrict__ ws, const int* __restrict__ pos,
                               int pos_stride, int H, int L_cap, int chunk, int splits, float scale) {
  constexpr int D = DV * 32;
  pdl_wait();
  pdl_launch_dependents();
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int nkeys = min(pos[static_cast<size_t>(b) * pos_stride] + 1, L_cap);
  const int j0 = split * chunk, j1 = min(j0 + chunk, nkeys);
  if (j0 >= j1) return;
  const __nv_bfloat16* kh = kv + b * seq_stride + static_cast<size_t>(h) * L_cap * D;
  attention_kv_split_part<DV>(q + (static_cast<size_t>(b) * H + h) * D, kh, kh + static_cast<size_t>(H) * L_cap * D,
                              ws + ((static_cast<size_t>(b) * H + h) * splits + split) * (D + 2), j0, j1, scale);
}

__global__ void attention_kv_rows_combine_kernel(const float* __restrict__ ws, __nv_bfloat16* __restrict__ out,
                                                 const int* __restrict__ pos, int pos_stride, int H, int D, int L_cap,
                                                 int chunk, int splits) {
  pdl_wait();
  pdl_launch_dependents();
  const int h = blockIdx.x, b = blockIdx.y;
  const int nkeys = min(pos[static_cast<size_t>(b) * pos_stride] + 1, L_cap);
  const int used = min((nkeys + chunk - 1) / chunk, splits);
  attention_kv_combine_part(ws + (static_cast<size_t>(b) * H + h) * splits * (D + 2),
                            out + (static_cast<size_t>(b) * H + h) * D, used, D, threadIdx.x);
}

// ----------------------------------------------------------------------------------------------- SiLU * up
__global__ void silu_mul_kernel(const uint4* __restrict__ gu, uint4* __restrict__ out, int I8, long long total) {
  pdl_wait();
  pdl_launch_dependents();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long m = i / I8;
  const int c = static_cast<int>(i - m * I8);
  const uint4 g = gu[m * 2 * I8 + c], u = gu[m * 2 * I8 + I8 + c];
  uint4 o;
  o.x = pack_bf16(silu_f(bf16_lo(g.x)) * bf16_lo(u.x), silu_f(bf16_hi(g.x)) * bf16_hi(u.x));
  o.y = pack_bf16(silu_f(bf16_lo(g.y)) * bf16_lo(u.y), silu_f(bf16_hi(g.y)) * bf16_hi(u.y));
  o.z = pack_bf16(silu_f(bf16_lo(g.z)) * bf16_lo(u.z), silu_f(bf16_hi(g.z)) * bf16_hi(u.z));
  o.w = pack_bf16(silu_f(bf16_lo(g.w)) * bf16_lo(u.w), silu_f(bf16_hi(g.w)) * bf16_hi(u.w));
  out[i] = o;
}

// ----------------------------------------------------------------------------------------------- next token
constexpr int kTokThreads = 1024;

// (value, index) argmax of one block, ranked as torch.argmax ranks: NaN above every number, ties (NaN included) to
// the smaller index.  The merge is order-independent, so the index is the first maximum however the block splits V,
// and any V > 0 yields an index in [0, V).
__device__ __forceinline__ void argmax_merge(float& v, int& i, float v2, int i2) {
  const bool n = isnan(v), n2 = isnan(v2);
  const bool take = n2 != n ? n2 : (v2 > v || ((n || v2 == v) && i2 < i));
  if (take) { v = v2; i = i2; }
}

__device__ __forceinline__ void block_argmax(const float* s, int V, float* sv, int* si, float& best_v, int& best_i) {
  float v = -INFINITY;
  int idx = 0x7fffffff;
  for (int j = threadIdx.x; j < V; j += kTokThreads) argmax_merge(v, idx, s[j], j);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v2 = __shfl_xor_sync(0xffffffffu, v, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, idx, o);
    argmax_merge(v, idx, v2, i2);
  }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = v; si[threadIdx.x >> 5] = idx; }
  __syncthreads();
  v = sv[0];
  idx = si[0];
  for (int w = 1; w < kTokThreads / 32; ++w) argmax_merge(v, idx, sv[w], si[w]);
  best_v = v;
  best_i = idx;
  __syncthreads();
}

// One greedy step of one sequence (the ds_agent_next_token contract); sv / si: the block's shared argmax scratch.
__device__ __forceinline__ void agent_next_token_row(float* logits, int V, const int* __restrict__ img_ids, int n_img,
                                                     int* state, int* __restrict__ out_ids, int max_new, int eos,
                                                     const uint4* __restrict__ embed, uint4* __restrict__ next_x,
                                                     const uint4* __restrict__ hidden_src, uint4* __restrict__ hidden,
                                                     int C8, float* sv, int* si) {
  // state: {pos, generated, done, last token}
  const int pos = state[0], n = state[1], done = state[2], last = state[3];
  if (done) return;
  if (hidden_src)
    for (int c = threadIdx.x; c < C8; c += kTokThreads) hidden[static_cast<size_t>(pos) * C8 + c] = hidden_src[c];
  // the image-token rule (generation.py:18-30), applied to the scores in place as the processor does
  int forced = -1;
  for (int t = 0; t + 1 < n_img; ++t)
    if (img_ids[t] == last) { forced = img_ids[t + 1]; break; }
  if (forced >= 0) {
    float mx;
    int unused;
    block_argmax(logits, V, sv, si, mx, unused);
    if (threadIdx.x == 0) logits[forced] = mx + 10.0f;
  } else {
    for (int t = 1 + threadIdx.x; t < n_img; t += kTokThreads) logits[img_ids[t]] = 0.0f;
  }
  __syncthreads();
  float bv;
  int tok;
  block_argmax(logits, V, sv, si, bv, tok);
  for (int c = threadIdx.x; c < C8; c += kTokThreads) next_x[c] = embed[static_cast<size_t>(tok) * C8 + c];
  if (threadIdx.x == 0) {
    out_ids[n] = tok;
    state[0] = pos + 1;
    state[1] = n + 1;
    state[2] = (tok == eos || n + 1 >= max_new) ? 1 : 0;
    state[3] = tok;
  }
}

__global__ void __launch_bounds__(kTokThreads)
agent_next_token_kernel(float* logits, int V, const int* __restrict__ img_ids, int n_img, int* state,
                        int* __restrict__ out_ids, int max_new, int eos, const uint4* __restrict__ embed,
                        uint4* __restrict__ next_x, const uint4* __restrict__ hidden_src, uint4* __restrict__ hidden,
                        int C8) {
  __shared__ float sv[kTokThreads / 32];
  __shared__ int si[kTokThreads / 32];
  pdl_wait();
  pdl_launch_dependents();
  agent_next_token_row(logits, V, img_ids, n_img, state, out_ids, max_new, eos, embed, next_x, hidden_src, hidden, C8,
                       sv, si);
}

// One CTA per row b, each its own sequence: logits[b], state[b], out_ids[b] (stride max_new), next_x[b],
// hidden[b] (stride hidden_stride8 uint4s) and hidden_src[b]; img_ids, eos and max_new are shared.
__global__ void __launch_bounds__(kTokThreads)
agent_next_token_rows_kernel(float* logits, int V, const int* __restrict__ img_ids, int n_img, int* state,
                             int* __restrict__ out_ids, int max_new, int eos, const uint4* __restrict__ embed,
                             uint4* __restrict__ next_x, const uint4* __restrict__ hidden_src,
                             uint4* __restrict__ hidden, long long hidden_stride8, int C8) {
  __shared__ float sv[kTokThreads / 32];
  __shared__ int si[kTokThreads / 32];
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.x;
  agent_next_token_row(logits + static_cast<size_t>(b) * V, V, img_ids, n_img, state + 4 * b,
                       out_ids + static_cast<size_t>(b) * max_new, max_new, eos, embed,
                       next_x + static_cast<size_t>(b) * C8, hidden_src ? hidden_src + static_cast<size_t>(b) * C8 : nullptr,
                       hidden + b * hidden_stride8, C8, sv, si);
}

template <typename Kern, typename... Args>
int launch_pdl(const char* name, Kern kern, dim3 grid, dim3 block, size_t smem, void* stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  pdl_attr(&attr[0]);
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = static_cast<cudaStream_t>(stream);
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  DS_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, args...));
  DS_LAUNCH_OK(name);
  return DS_OK;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <int M>
int gemv_launch(const void* x, const void* w, const void* residual, void* y, int N, int K, int out_fp32,
                void* stream) {
  const size_t smem = static_cast<size_t>(M) * K * 2;
  static size_t attr[kMaxDevices] = {};
  if (smem > 48 * 1024 && smem > attr[device_slot()]) {
    DS_CUDA_OK(cudaFuncSetAttribute(gemv_bf16_kernel<M>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    static_cast<int>(smem)));
    attr[device_slot()] = smem;
  }
  const int rows_per_cta = kGemvThreads / 32 * kGemvRowsPerWarp;
  return launch_pdl("gemv_bf16_kernel", gemv_bf16_kernel<M>, dim3((N + rows_per_cta - 1) / rows_per_cta),
                    dim3(kGemvThreads), smem, stream, static_cast<const __nv_bfloat16*>(x),
                    static_cast<const __nv_bfloat16*>(w), static_cast<const __nv_bfloat16*>(residual), y, N, K,
                    out_fp32);
}

}  // namespace ds

extern "C" int ds_gemv_bf16(const void* x, const void* w, const void* residual, void* y, int M, int N, int K,
                            int out_fp32, void* stream) {
  using namespace ds;
  DS_REQUIRE(x && w && y, "ds_gemv_bf16: NULL pointer");
  DS_REQUIRE(M >= 1 && M <= 8 && N > 0 && K > 0 && K % 8 == 0, "ds_gemv_bf16: need 1 <= M <= 8, K %% 8 == 0");
  DS_REQUIRE(static_cast<size_t>(M) * K * 2 <= 227 * 1024, "ds_gemv_bf16: M*K bf16 must fit in shared memory");
  DS_REQUIRE(aligned16(x) && aligned16(w), "ds_gemv_bf16: x and w must be 16-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  switch (M) {
    case 1: return gemv_launch<1>(x, w, residual, y, N, K, out_fp32, stream);
    case 2: return gemv_launch<2>(x, w, residual, y, N, K, out_fp32, stream);
    case 3: return gemv_launch<3>(x, w, residual, y, N, K, out_fp32, stream);
    case 4: return gemv_launch<4>(x, w, residual, y, N, K, out_fp32, stream);
    case 5: return gemv_launch<5>(x, w, residual, y, N, K, out_fp32, stream);
    case 6: return gemv_launch<6>(x, w, residual, y, N, K, out_fp32, stream);
    case 7: return gemv_launch<7>(x, w, residual, y, N, K, out_fp32, stream);
    default: return gemv_launch<8>(x, w, residual, y, N, K, out_fp32, stream);
  }
}

extern "C" int ds_rmsnorm(const void* x, const float* gamma, void* y, int rows, int C, float eps, void* stream) {
  using namespace ds;
  DS_REQUIRE(x && gamma && y && rows > 0, "ds_rmsnorm: bad arguments");
  DS_REQUIRE(C > 0 && C % 8 == 0 && C <= 8192, "ds_rmsnorm: C %% 8 == 0 and C <= 8192");
  DS_REQUIRE(aligned16(x) && aligned16(gamma) && aligned16(y), "ds_rmsnorm: pointers must be 16-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  return launch_pdl("rmsnorm_kernel", rmsnorm_kernel, dim3(rows), dim3(kNormThreads), 0, stream,
                    static_cast<const __nv_bfloat16*>(x), gamma, static_cast<__nv_bfloat16*>(y), C, eps);
}

extern "C" int ds_rope_kv_append(const void* qkv, void* q_out, void* kv_layer, const int* pos, int M, int H, int D,
                                 int L_max, float theta, void* stream) {
  using namespace ds;
  DS_REQUIRE(qkv && q_out && kv_layer && pos, "ds_rope_kv_append: NULL pointer");
  DS_REQUIRE(M > 0 && H > 0 && L_max > 0 && (D == 64 || D == 128), "ds_rope_kv_append: bad shape (D = 64 or 128)");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  return launch_pdl("rope_kv_append_kernel", rope_kv_append_kernel, dim3(M), dim3(256), 0, stream,
                    static_cast<const __nv_bfloat16*>(qkv), static_cast<__nv_bfloat16*>(q_out),
                    static_cast<__nv_bfloat16*>(kv_layer), pos, H, D, L_max, theta);
}

extern "C" int ds_attention_kv(const void* q, const void* kv_layer, void* out, float* ws, int64_t ws_bytes,
                               const int* pos, int M, int H, int D, int L_max, int chunk, void* stream) {
  using namespace ds;
  DS_REQUIRE(q && kv_layer && out && ws && pos, "ds_attention_kv: NULL pointer");
  DS_REQUIRE(M > 0 && H > 0 && L_max > 0 && chunk > 0 && (D == 64 || D == 128),
             "ds_attention_kv: bad shape (D = 64 or 128)");
  const int splits = (L_max + chunk - 1) / chunk;
  const int64_t need = static_cast<int64_t>(M) * H * splits * (D + 2) * 4;
  DS_REQUIRE(ws_bytes >= need, "ds_attention_kv: workspace of %lld bytes < %lld", static_cast<long long>(ws_bytes),
             static_cast<long long>(need));
  DS_REQUIRE(static_cast<int64_t>(M) * H <= 65535LL * 65535LL && M <= 65535, "ds_attention_kv: too many rows");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const float scale = 1.0f / sqrtf(static_cast<float>(D));
  const auto* qq = static_cast<const __nv_bfloat16*>(q);
  const auto* kv = static_cast<const __nv_bfloat16*>(kv_layer);
  int rc = D == 128 ? launch_pdl("attention_kv_split_kernel", attention_kv_split_kernel<4>, dim3(splits, H, M),
                                 dim3(kAttnWarps * 32), 0, stream, qq, kv, ws, pos, H, L_max, chunk, splits, scale)
                    : launch_pdl("attention_kv_split_kernel", attention_kv_split_kernel<2>, dim3(splits, H, M),
                                 dim3(kAttnWarps * 32), 0, stream, qq, kv, ws, pos, H, L_max, chunk, splits, scale);
  if (rc != DS_OK) return rc;
  return launch_pdl("attention_kv_combine_kernel", attention_kv_combine_kernel, dim3(H, M), dim3(D), 0, stream,
                    static_cast<const float*>(ws), static_cast<__nv_bfloat16*>(out), pos, H, D, L_max, chunk, splits);
}

extern "C" int ds_rope_kv_append_rows(const void* qkv, void* q_out, void* kv, int64_t seq_stride, const int* pos,
                                      int pos_stride, int B, int H, int D, int L_cap, float theta, void* stream) {
  using namespace ds;
  DS_REQUIRE(qkv && q_out && kv && pos, "ds_rope_kv_append_rows: NULL pointer");
  DS_REQUIRE(B > 0 && H > 0 && L_cap > 0 && pos_stride >= 0 && (D == 64 || D == 128),
             "ds_rope_kv_append_rows: bad shape (D = 64 or 128)");
  DS_REQUIRE(seq_stride >= 2LL * H * L_cap * D || B == 1, "ds_rope_kv_append_rows: seq_stride < 2 * H * L_cap * D");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  return launch_pdl("rope_kv_append_rows_kernel", rope_kv_append_rows_kernel, dim3(B), dim3(256), 0, stream,
                    static_cast<const __nv_bfloat16*>(qkv), static_cast<__nv_bfloat16*>(q_out),
                    static_cast<__nv_bfloat16*>(kv), static_cast<long long>(seq_stride), pos, pos_stride, H, D, L_cap,
                    theta);
}

extern "C" int ds_attention_kv_rows(const void* q, const void* kv, int64_t seq_stride, void* out, float* ws,
                                    int64_t ws_bytes, const int* pos, int pos_stride, int B, int H, int D, int L_cap,
                                    int chunk, void* stream) {
  using namespace ds;
  DS_REQUIRE(q && kv && out && ws && pos, "ds_attention_kv_rows: NULL pointer");
  DS_REQUIRE(B > 0 && B <= 65535 && H > 0 && H <= 65535 && L_cap > 0 && chunk > 0 && pos_stride >= 0 &&
                 (D == 64 || D == 128),
             "ds_attention_kv_rows: bad shape (D = 64 or 128)");
  DS_REQUIRE(seq_stride >= 2LL * H * L_cap * D || B == 1, "ds_attention_kv_rows: seq_stride < 2 * H * L_cap * D");
  const int splits = (L_cap + chunk - 1) / chunk;
  const int64_t need = static_cast<int64_t>(B) * H * splits * (D + 2) * 4;
  DS_REQUIRE(ws_bytes >= need, "ds_attention_kv_rows: workspace of %lld bytes < %lld",
             static_cast<long long>(ws_bytes), static_cast<long long>(need));
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const float scale = 1.0f / sqrtf(static_cast<float>(D));
  const auto* qq = static_cast<const __nv_bfloat16*>(q);
  const auto* kk = static_cast<const __nv_bfloat16*>(kv);
  const long long ss = seq_stride;
  int rc = D == 128 ? launch_pdl("attention_kv_rows_split_kernel", attention_kv_rows_split_kernel<4>,
                                 dim3(splits, H, B), dim3(kAttnWarps * 32), 0, stream, qq, kk, ss, ws, pos, pos_stride,
                                 H, L_cap, chunk, splits, scale)
                    : launch_pdl("attention_kv_rows_split_kernel", attention_kv_rows_split_kernel<2>,
                                 dim3(splits, H, B), dim3(kAttnWarps * 32), 0, stream, qq, kk, ss, ws, pos, pos_stride,
                                 H, L_cap, chunk, splits, scale);
  if (rc != DS_OK) return rc;
  return launch_pdl("attention_kv_rows_combine_kernel", attention_kv_rows_combine_kernel, dim3(H, B), dim3(D), 0,
                    stream, static_cast<const float*>(ws), static_cast<__nv_bfloat16*>(out), pos, pos_stride, H, D,
                    L_cap, chunk, splits);
}

extern "C" int ds_silu_mul(const void* gate_up, void* out, int M, int I, void* stream) {
  using namespace ds;
  DS_REQUIRE(gate_up && out && M > 0 && I > 0 && I % 8 == 0, "ds_silu_mul: bad arguments (I %% 8 == 0)");
  DS_REQUIRE(aligned16(gate_up) && aligned16(out), "ds_silu_mul: pointers must be 16-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long total = static_cast<long long>(M) * (I / 8);
  return launch_pdl("silu_mul_kernel", silu_mul_kernel, dim3(static_cast<unsigned>((total + 255) / 256)), dim3(256), 0,
                    stream, static_cast<const uint4*>(gate_up), static_cast<uint4*>(out), I / 8, total);
}

extern "C" int ds_agent_next_token(float* logits, int V, const int* img_ids, int n_img, int* state, int* out_ids,
                                   int max_new, int eos, const void* embed, void* next_x, const void* hidden_src,
                                   void* hidden, int C, void* stream) {
  using namespace ds;
  DS_REQUIRE(logits && state && out_ids && embed && next_x && hidden && V > 0 && max_new > 0,
             "ds_agent_next_token: bad arguments");
  DS_REQUIRE(n_img >= 0 && (n_img == 0 || img_ids), "ds_agent_next_token: img_ids missing");
  DS_REQUIRE(C > 0 && C % 8 == 0 && aligned16(embed) && aligned16(next_x) && aligned16(hidden) &&
                 (!hidden_src || aligned16(hidden_src)),
             "ds_agent_next_token: C %% 8 == 0 and 16-byte aligned rows");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  return launch_pdl("agent_next_token_kernel", agent_next_token_kernel, dim3(1), dim3(kTokThreads), 0, stream, logits,
                    V, img_ids, n_img, state, out_ids, max_new, eos, static_cast<const uint4*>(embed),
                    static_cast<uint4*>(next_x), static_cast<const uint4*>(hidden_src), static_cast<uint4*>(hidden),
                    C / 8);
}

extern "C" int ds_agent_next_token_rows(float* logits, int V, const int* img_ids, int n_img, int* state, int* out_ids,
                                        int max_new, int eos, const void* embed, void* next_x, const void* hidden_src,
                                        void* hidden, int64_t hidden_stride, int C, int B, void* stream) {
  using namespace ds;
  DS_REQUIRE(logits && state && out_ids && embed && next_x && hidden && V > 0 && max_new > 0 && B > 0,
             "ds_agent_next_token_rows: bad arguments");
  DS_REQUIRE(n_img >= 0 && (n_img == 0 || img_ids), "ds_agent_next_token_rows: img_ids missing");
  DS_REQUIRE(C > 0 && C % 8 == 0 && hidden_stride >= C && hidden_stride % 8 == 0 && aligned16(embed) &&
                 aligned16(next_x) && aligned16(hidden) && (!hidden_src || aligned16(hidden_src)),
             "ds_agent_next_token_rows: C %% 8 == 0, hidden_stride %% 8 == 0 and 16-byte aligned rows");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  return launch_pdl("agent_next_token_rows_kernel", agent_next_token_rows_kernel, dim3(B), dim3(kTokThreads), 0,
                    stream, logits, V, img_ids, n_img, state, out_ids, max_new, eos, static_cast<const uint4*>(embed),
                    static_cast<uint4*>(next_x), static_cast<const uint4*>(hidden_src), static_cast<uint4*>(hidden),
                    static_cast<long long>(hidden_stride / 8), C / 8);
}
