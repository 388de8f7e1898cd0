// encoder_kernels.cu — what the conditioning encoders need beyond the UNet's kernels (SURVEY.md §8f ranks 2-3:
// the CLIP ViT-H and Magi ViT-MAE image encoders of prepare_ip_image_embeds, src/pipelines/pipeline_diffsensei.py:125-128,
// and the two SDXL CLIP text encoders of encode_prompt, :232-245).  Their linears / MLPs run on the wgmma GEMM
// (ds_gemm_bf16, bias / GELU / quick-GELU / residual epilogues) and their LayerNorms on ds_layernorm; this file adds
//   ds_attention_small : softmax(scale * Q K^T [+ causal mask]) V for SHORT sequences (<= 320 keys, fewer above head
//                        width 168: K and V must fit in shared memory) and any head width that is a multiple of 8 up
//                        to 256 — 77 text tokens (causal), 197 / 257 image tokens, heads
//                        of 64 (text, ViT-MAE) and 80 (ViT-H, outside the flash kernel's head_dim 64).  These encoders
//                        run once per panel (1.3 TFLOP of GEMMs for four 224x224 character crops, 43 GFLOP of
//                        attention), so the attention is a plain CUDA-core kernel: K / V of one (batch, head) staged
//                        in shared memory, one warp per query row, fp32 softmax.                   [latency-bound]
//   ds_embed_tokens    : out[b][t][:] = token_embedding[ids[b][t]][:] + position_embedding[t][:]   (CLIPTextEmbeddings)
//   ds_prompt_emphasis : AUTOMATIC1111's "Original" prompt emphasis on each encoder's chunk of hidden_states[-2],
//                        written into the concatenated [chunks][L][C1 + C2] prompt embedding (prompt_weighting.py)
#include "ds_common.cuh"
#include "ds_host.h"

namespace ds {

constexpr int kSmallAttnThreads = 128;   // 4 warps, one query row each per sweep
constexpr int kSmallAttnRows = 32;       // query rows per CTA
constexpr int kSmallAttnMaxKeys = 320;   // 10 keys per lane

__global__ void __launch_bounds__(kSmallAttnThreads)
attention_small_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                       const __nv_bfloat16* __restrict__ v, __nv_bfloat16* __restrict__ out, int Nq, int Nk, int hd,
                       long long ldq, long long ldk, long long ldv, long long ldo, float scale_log2, int causal) {
  extern __shared__ uint32_t sm[];
  const int hw = hd >> 1;        // bf16x2 words per row
  const int row_words = (hw & 1) ? hw : hw + 1;           // odd word stride: lane j reads row j without bank conflicts
  uint32_t* sK = sm;                                      // [Nk][row_words]
  uint32_t* sV = sK + static_cast<size_t>(Nk) * row_words;
  float* sQ = reinterpret_cast<float*>(sV + static_cast<size_t>(Nk) * row_words);   // [4 warps][hd]
  float* sP = sQ + 4 * hd;                                                         // [4 warps][Nk]
  const int b = blockIdx.z, head = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const __nv_bfloat16* kb = k + static_cast<long long>(b) * Nk * ldk + head * hd;
  const __nv_bfloat16* vb = v + static_cast<long long>(b) * Nk * ldv + head * hd;
  // stage K and V of this (batch, head): 16-byte global loads, 4-byte shared stores into the padded rows
  const int vec_per_row = hd >> 3;
  for (int i = threadIdx.x; i < Nk * vec_per_row; i += blockDim.x) {
    const int j = i / vec_per_row, c = i - j * vec_per_row;
    const uint4 uk = __ldg(reinterpret_cast<const uint4*>(kb + static_cast<long long>(j) * ldk) + c);
    const uint4 uv = __ldg(reinterpret_cast<const uint4*>(vb + static_cast<long long>(j) * ldv) + c);
    uint32_t* dk = sK + static_cast<size_t>(j) * row_words + c * 4;
    uint32_t* dv = sV + static_cast<size_t>(j) * row_words + c * 4;
    dk[0] = uk.x; dk[1] = uk.y; dk[2] = uk.z; dk[3] = uk.w;
    dv[0] = uv.x; dv[1] = uv.y; dv[2] = uv.z; dv[3] = uv.w;
  }
  __syncthreads();
  const int r_end = min(Nq, (static_cast<int>(blockIdx.x) + 1) * kSmallAttnRows);
  float* myQ = sQ + warp * hd;
  float* myP = sP + static_cast<size_t>(warp) * Nk;
  for (int r = blockIdx.x * kSmallAttnRows + warp; r < r_end; r += 4) {
    const __nv_bfloat16* qr = q + (static_cast<long long>(b) * Nq + r) * ldq + head * hd;
    for (int d = lane; d < hd; d += 32) myQ[d] = __bfloat162float(qr[d]);
    __syncwarp();
    const int kmax = causal ? min(Nk, r + 1) : Nk;       // keys a causal row may see
    float s[kSmallAttnMaxKeys / 32];
    float m = -INFINITY;
#pragma unroll
    for (int t = 0; t < kSmallAttnMaxKeys / 32; ++t) {
      const int j = lane + 32 * t;
      float acc = -INFINITY;
      if (j < kmax) {
        const uint32_t* kr = sK + static_cast<size_t>(j) * row_words;
        float a0 = 0.f, a1 = 0.f;
        for (int w = 0; w < hw; ++w) {
          const uint32_t kw = kr[w];
          const float2 qq = *reinterpret_cast<const float2*>(myQ + 2 * w);
          a0 = fmaf(qq.x, bf16_lo(kw), a0);
          a1 = fmaf(qq.y, bf16_hi(kw), a1);
        }
        acc = (a0 + a1) * scale_log2;
      }
      s[t] = acc;
      m = fmaxf(m, acc);
    }
    m = warp_max(m);
    float l = 0.f;
#pragma unroll
    for (int t = 0; t < kSmallAttnMaxKeys / 32; ++t) {
      const int j = lane + 32 * t;
      const float pj = j < kmax ? exp2f(s[t] - m) : 0.f;
      l += pj;
      if (j < Nk) myP[j] = pj;
    }
    l = warp_sum(l);
    __syncwarp();
    const float inv = 1.0f / l;
    __nv_bfloat16* orow = out + (static_cast<long long>(b) * Nq + r) * ldo + head * hd;
    for (int w = lane; w < hw; w += 32) {
      float o0 = 0.f, o1 = 0.f;
      for (int j = 0; j < kmax; ++j) {
        const float pj = myP[j];
        const uint32_t vw = sV[static_cast<size_t>(j) * row_words + w];
        o0 = fmaf(pj, bf16_lo(vw), o0);
        o1 = fmaf(pj, bf16_hi(vw), o1);
      }
      *reinterpret_cast<uint32_t*>(orow + 2 * w) = pack_bf16(o0 * inv, o1 * inv);
    }
    __syncwarp();
  }
}

__global__ void embed_tokens_kernel(const int* __restrict__ ids, const uint4* __restrict__ tok,
                                    const uint4* __restrict__ pos, uint4* __restrict__ out, int L, int cv, int vocab,
                                    long long total) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = static_cast<int>(i % cv);
  const long long row = i / cv;
  const int t = static_cast<int>(row % L);
  int id = ids[row];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  const uint4 a = __ldg(tok + static_cast<long long>(id) * cv + c), p = __ldg(pos + static_cast<long long>(t) * cv + c);
  uint4 o;
  o.x = pack_bf16(bf16_lo(a.x) + bf16_lo(p.x), bf16_hi(a.x) + bf16_hi(p.x));
  o.y = pack_bf16(bf16_lo(a.y) + bf16_lo(p.y), bf16_hi(a.y) + bf16_hi(p.y));
  o.z = pack_bf16(bf16_lo(a.z) + bf16_lo(p.z), bf16_hi(a.z) + bf16_hi(p.z));
  o.w = pack_bf16(bf16_lo(a.w) + bf16_lo(p.w), bf16_hi(a.w) + bf16_hi(p.w));
  out[i] = o;
}

constexpr int kEmphasisThreads = 256;

// One CTA per (entry, encoder).  z = the source chunk [L][C], w = its per-token weights [L]:
//   m0 = mean(z), z' = z * w, m1 = mean(z'), out = z' * (m0 / m1)   (out = z' where m1 == 0),
// fp32 throughout; each thread sums a fixed stride of elements and the CTA adds the 8 warp sums in warp order, so a
// chunk's bits depend on nothing but the chunk.  A chunk whose weights are all 1 is copied unchanged.
__global__ void __launch_bounds__(kEmphasisThreads)
prompt_emphasis_kernel(const uint4* __restrict__ h1, const uint4* __restrict__ h2, const float* __restrict__ w1,
                       const float* __restrict__ w2, const int* __restrict__ entries, uint4* __restrict__ out, int L,
                       int C1, int C2) {
  __shared__ float red[2][kEmphasisThreads / 32];
  const int e = blockIdx.x, enc = blockIdx.y, tid = threadIdx.x;
  const int src = entries[3 * e + enc], dst = entries[3 * e + 2];
  const int cv = (enc ? C2 : C1) >> 3;
  const int ldo = (C1 + C2) >> 3;
  const uint4* z = (enc ? h2 : h1) + static_cast<long long>(src) * L * cv;
  const float* w = (enc ? w2 : w1) + static_cast<long long>(src) * L;
  uint4* o = out + static_cast<long long>(dst) * L * ldo + (enc ? C1 >> 3 : 0);
  bool ones = true;
  for (int t = tid; t < L; t += kEmphasisThreads) ones &= w[t] == 1.0f;
  const int n = L * cv;
  if (__syncthreads_and(ones)) {
    for (int i = tid; i < n; i += kEmphasisThreads) {
      const int t = i / cv;
      o[static_cast<long long>(t) * ldo + (i - t * cv)] = __ldg(z + i);
    }
    return;
  }
  float s0 = 0.f, s1 = 0.f;
  for (int i = tid; i < n; i += kEmphasisThreads) {
    const float wt = w[i / cv];
    const uint4 u = __ldg(z + i);
    const uint32_t q[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float a = bf16_lo(q[k]), b = bf16_hi(q[k]);
      s0 += a;
      s0 += b;
      s1 += __fmul_rn(a, wt);
      s1 += __fmul_rn(b, wt);
    }
  }
  s0 = warp_sum(s0);
  s1 = warp_sum(s1);
  if ((tid & 31) == 0) {
    red[0][tid >> 5] = s0;
    red[1][tid >> 5] = s1;
  }
  __syncthreads();
  float t0 = 0.f, t1 = 0.f;
#pragma unroll
  for (int k = 0; k < kEmphasisThreads / 32; ++k) {
    t0 += red[0][k];
    t1 += red[1][k];
  }
  const float count = static_cast<float>(n) * 8.0f;
  const float m0 = t0 / count, m1 = t1 / count;
  const bool guard = m1 == 0.0f;
  const float ratio = guard ? 1.0f : m0 / m1;
  for (int i = tid; i < n; i += kEmphasisThreads) {
    const int t = i / cv;
    const float wt = w[t];
    const uint4 u = __ldg(z + i);
    const uint32_t q[4] = {u.x, u.y, u.z, u.w};
    uint32_t r[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float a = __fmul_rn(bf16_lo(q[k]), wt), b = __fmul_rn(bf16_hi(q[k]), wt);
      r[k] = guard ? pack_bf16(a, b) : pack_bf16(__fmul_rn(a, ratio), __fmul_rn(b, ratio));
    }
    o[static_cast<long long>(t) * ldo + (i - t * cv)] = make_uint4(r[0], r[1], r[2], r[3]);
  }
}

}  // namespace ds

extern "C" int ds_prompt_emphasis(const void* h1, const void* h2, const float* w1, const float* w2,
                                  const int* entries, int n_entries, int L, int C1, int C2, void* out, void* stream) {
  using namespace ds;
  DS_REQUIRE(h1 && h2 && w1 && w2 && entries && out, "ds_prompt_emphasis: NULL pointer");
  DS_REQUIRE(n_entries > 0 && L > 0 && C1 > 0 && C2 > 0 && C1 % 8 == 0 && C2 % 8 == 0,
             "ds_prompt_emphasis: bad shape (n_entries, L > 0; C1, C2 > 0 and multiples of 8)");
  DS_REQUIRE(n_entries <= 0x7fffffff / 3, "ds_prompt_emphasis: too many entries");
  DS_REQUIRE((reinterpret_cast<uintptr_t>(h1) & 15) == 0 && (reinterpret_cast<uintptr_t>(h2) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(out) & 15) == 0 && (reinterpret_cast<uintptr_t>(w1) & 3) == 0 &&
                 (reinterpret_cast<uintptr_t>(w2) & 3) == 0 && (reinterpret_cast<uintptr_t>(entries) & 3) == 0,
             "ds_prompt_emphasis: h1 / h2 / out must be 16-byte aligned, w1 / w2 / entries 4-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  prompt_emphasis_kernel<<<dim3(n_entries, 2), kEmphasisThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(h1), static_cast<const uint4*>(h2), w1, w2, entries, static_cast<uint4*>(out), L, C1,
      C2);
  DS_LAUNCH_OK("prompt_emphasis_kernel");
  return DS_OK;
}

extern "C" int ds_attention_small(const void* q, const void* k, const void* v, void* out, int B, int Nq, int Nk,
                                  int heads, int head_dim, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo,
                                  float scale, int causal, void* stream) {
  using namespace ds;
  DS_REQUIRE(q && k && v && out, "ds_attention_small: NULL pointer");
  DS_REQUIRE(B > 0 && Nq > 0 && Nk > 0 && heads > 0, "ds_attention_small: bad shape");
  DS_REQUIRE(Nk <= kSmallAttnMaxKeys, "ds_attention_small: at most %d keys (got %d); long sequences use ds_attention_self",
             kSmallAttnMaxKeys, Nk);
  DS_REQUIRE(head_dim >= 8 && head_dim <= 256 && head_dim % 8 == 0, "ds_attention_small: head_dim %% 8 == 0, <= 256");
  DS_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 2 == 0 && ldq >= heads * head_dim &&
                 ldk >= heads * head_dim && ldv >= heads * head_dim && ldo >= heads * head_dim,
             "ds_attention_small: row strides must cover heads*head_dim and be multiples of 8 elements");
  DS_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(k) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(v) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0,
             "ds_attention_small: q / k / v must be 16-byte aligned");
  DS_REQUIRE(!causal || Nq == Nk, "ds_attention_small: the causal mask needs Nq == Nk");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const int hw = head_dim / 2;
  const int row_words = (hw & 1) ? hw : hw + 1;
  // K and V rows [Nk][row_words] words, the 4 warps' q rows [4][hd] and probabilities [4][Nk] floats
  const size_t per_key = static_cast<size_t>(2) * row_words * 4 + 4 * 4;
  const size_t smem = per_key * Nk + 4 * head_dim * 4;
  DS_REQUIRE(smem <= static_cast<size_t>(dev.smem_optin),
             "ds_attention_small: %d keys at head_dim %d need %zu bytes of shared memory > %d; at most %d keys fit",
             Nk, head_dim, smem, dev.smem_optin,
             static_cast<int>((static_cast<size_t>(dev.smem_optin) - 4 * head_dim * 4) / per_key));
  static size_t attr[kMaxDevices] = {};
  if (smem > 48 * 1024 && smem > attr[device_slot()]) {
    DS_CUDA_OK(cudaFuncSetAttribute(attention_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    attr[device_slot()] = smem;
  }
  dim3 grid((Nq + kSmallAttnRows - 1) / kSmallAttnRows, heads, B);
  attention_small_kernel<<<grid, kSmallAttnThreads, smem, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(k), static_cast<const __nv_bfloat16*>(v),
      static_cast<__nv_bfloat16*>(out), Nq, Nk, head_dim, ldq, ldk, ldv, ldo, scale * 1.4426950408889634f, causal);
  DS_LAUNCH_OK("attention_small_kernel");
  return DS_OK;
}

extern "C" int ds_embed_tokens(const int* ids, const void* tok_emb, const void* pos_emb, void* out, int B, int L, int C,
                               int vocab, void* stream) {
  using namespace ds;
  DS_REQUIRE(ids && tok_emb && pos_emb && out && B > 0 && L > 0 && C > 0 && C % 8 == 0 && vocab > 0,
             "ds_embed_tokens: bad arguments (C %% 8 == 0)");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const long long total = static_cast<long long>(B) * L * (C / 8);
  embed_tokens_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      ids, static_cast<const uint4*>(tok_emb), static_cast<const uint4*>(pos_emb), static_cast<uint4*>(out), L, C / 8,
      vocab, total);
  DS_LAUNCH_OK("embed_tokens_kernel");
  return DS_OK;
}
