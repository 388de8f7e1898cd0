// attn_wgmma.cu — fused attention for head_dim 64 on sm_90a warpgroup tensor cores.
//
// One kernel serves three entry points:
//   ds_attention_self      self-attention (AttnProcessor2_0, src/models/attention_processor.py:69-81):
//                          softmax(Q K^T / 8) V over the fused [B][N][3C] projection, no mask;
//   ds_resampler_attn      the Resampler's perceiver attention (src/models/resampler.py:64-74), same math;
//   ds_attention_cross_ip  out = softmax(Q Kt^T/8) Vt + scale * softmax(Q Kip^T/8 + M(bbox)) Vip
//                          (MaskedIPAttnProcessor2_0, :231-258) in ONE pass over both key sets; the additive bbox mask
//                          M in {0,-10000} (:115-169) is evaluated in registers with the reference's closed-interval /
//                          derived-(H',W') semantics (ip_mask.cuh).
// Q/K/V are addressed by 3-D tensor maps {columns, tokens, batch} over the projection outputs, so the head split /
// transposes of the reference are never materialised.
//
// CTA = 128 query rows of one (batch, head), 384 threads:
//   warpgroup 0     one TMA lane: the Q tile, then 64-key K|V tiles through a RING-deep shared-memory ring
//   warpgroups 1-2  64 query rows each: S = Q K^T (wgmma, both operands in smem), online softmax in registers (a row
//                   lives in the 4 threads of a quad), O += P V (wgmma with P as a register A operand, V MN-major)
// Keys past the end of a key set arrive as TMA zero fill and are masked to -inf.
#include <cstdlib>

#include "ds_common.cuh"
#include "ds_host.h"
#include "ip_mask.cuh"
#include "wgmma.cuh"

namespace ds {

constexpr int kQTile = 128;  // query rows per CTA
constexpr int kKTile = 64;   // keys per pipeline stage
constexpr int kHd = 64;      // head dim
constexpr int kRing = 4;
constexpr int kAttnThreads = 384;
constexpr int kQBytes = kQTile * kHd * 2;   // 16 KiB
constexpr int kKVBytes = kKTile * kHd * 2;  // 8 KiB each for K and V
constexpr int kAttnSmemBytes = kQBytes + kRing * 2 * kKVBytes + 1024 /*align*/ + 256 /*barriers*/;
constexpr float kLog2e = 1.4426950408889634f;

struct AttnParams {
  __nv_bfloat16* out;  // [B][Nq][ldo], head h at columns [64 h, +64)
  int Nq, ldo;
  int n_keys[2];       // keys of set 0 (self / text) and set 1 (IP; 0 = no second set)
  int k_col0, v_col0;  // column of head 0's K / V inside the key tensor maps
  float scale_log2;    // softmax scale * log2(e)
  // IP mask (set 1 only)
  const float* bbox;   // [B][num_ips][4]
  int num_ips, tokens_per_ip, num_dummy, Hd, Wd;
  float ip_scale;
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__global__ void __launch_bounds__(kAttnThreads, 1)
attn_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK0,
                  const __grid_constant__ CUtensorMap tmK1, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sRing = sQ + kQBytes;  // stage s: K at s * 16 KiB, V at s * 16 KiB + 8 KiB
  uint64_t* q_bar = reinterpret_cast<uint64_t*>(sRing + kRing * 2 * kKVBytes);
  uint64_t* full_bar = q_bar + 1;
  uint64_t* empty_bar = full_bar + kRing;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kQTile, head = blockIdx.y, b = blockIdx.z;
  const int tiles0 = (p.n_keys[0] + kKTile - 1) / kKTile;
  const int tiles1 = (p.n_keys[1] + kKTile - 1) / kKTile;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK0);
    if (tiles1 > 0) tma_prefetch_desc(&tmK1);
    mbar_init(q_bar, 1);
    for (int i = 0; i < kRing; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 256);  // every consumer thread, once its warpgroup's MMAs on the stage retired
    }
    fence_mbar_init();
  }
  pdl_launch_dependents();
  __syncthreads();
  pdl_wait();

  if (warp < 4) {
    if (warp == 0 && lane == 0) {
      mbar_arrive_expect_tx(q_bar, kQBytes);
      tma_load_3d(sQ, &tmQ, q_bar, head * kHd, q0, b);
      int stage = 0;
      uint32_t phase = 0;
      for (int t = 0; t < tiles0 + tiles1; ++t) {
        const bool second = t >= tiles0;
        const CUtensorMap* m = second ? &tmK1 : &tmK0;
        const int key0 = (second ? t - tiles0 : t) * kKTile;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_arrive_expect_tx(&full_bar[stage], 2 * kKVBytes);
        uint8_t* sK = sRing + stage * 2 * kKVBytes;
        tma_load_3d(sK, m, &full_bar[stage], p.k_col0 + head * kHd, key0, b);
        tma_load_3d(sK + kKVBytes, m, &full_bar[stage], p.v_col0 + head * kHd, key0, b);
        if (++stage == kRing) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumers
  const int ct = threadIdx.x - 128;
  const int wg = ct >> 7;
  const int r0 = (ct >> 5) * 16 + (lane >> 2);  // tile rows r0 and r0 + 8
  const int cq = 2 * (lane & 3);
  uint32_t ip_bits[2] = {0u, 0u};
  if (tiles1 > 0) {
    const float* bb = p.bbox + static_cast<size_t>(b) * p.num_ips * 4;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = q0 + r0 + 8 * h;
      if (n < p.Nq) ip_bits[h] = ip_inside_bits(bb, p.num_ips, n, p.Hd, p.Wd);
    }
  }
  const uint32_t q_addr = smem_u32(sQ) + wg * 64 * 128;
  mbar_wait(q_bar, 0);

  float o[32], res[32];
  float m_run[2], l_run[2];
  int stage = 0;
  uint32_t phase = 0;
  for (int set = 0; set < (tiles1 > 0 ? 2 : 1); ++set) {
    const int n_tiles = set ? tiles1 : tiles0;
    const int nk = set ? p.n_keys[1] : p.n_keys[0];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    m_run[0] = m_run[1] = -INFINITY;
    l_run[0] = l_run[1] = 0.f;
    for (int t = 0; t < n_tiles; ++t) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t k_addr = smem_u32(sRing + stage * 2 * kKVBytes);
      const uint32_t v_addr = k_addr + kKVBytes;
      float s[32];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kHd / 16; ++k)
        wgmma_m64n64_ss(s, make_wgmma_desc(q_addr + k * 32, 1024, 16), make_wgmma_desc(k_addr + k * 32, 1024, 16),
                        k != 0);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<32>(s);

      // scores -> log2 domain with the mask applied; row max over the quad
      const int key0 = t * kKTile;
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = key0 + j * 8 + cq + (e & 1);
          const int h = e >> 1;
          float v = s[4 * j + e] * p.scale_log2;
          if (set == 1 && !ip_key_open(ip_bits[h], key, p.tokens_per_ip, p.num_dummy)) v -= 10000.0f * kLog2e;
          if (key >= nk) v = -INFINITY;
          s[4 * j + e] = v;
          mx[h] = fmaxf(mx[h], v);
        }
      }
      float corr[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        const float m_new = fmaxf(m_run[h], mx[h]);
        corr[h] = ex2(m_run[h] - m_new);  // 0 on the first tile (m_run = -inf)
        m_run[h] = m_new;
        l_run[h] *= corr[h];
      }
      uint32_t pa[4][4];  // P as the bf16 A fragments of the four 16-key MMA slices
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float p0 = ex2(s[4 * j + 2 * h] - m_run[h]);
          const float p1 = ex2(s[4 * j + 2 * h + 1] - m_run[h]);
          l_run[h] += p0 + p1;
          pa[j >> 1][(j & 1) * 2 + h] = pack_bf16(p0, p1);
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[4 * j + 0] *= corr[0];
        o[4 * j + 1] *= corr[0];
        o[4 * j + 2] *= corr[1];
        o[4 * j + 3] *= corr[1];
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kKTile / 16; ++kk)
        wgmma_m64n64_rs_tb(o, pa[kk], make_wgmma_desc(v_addr + kk * 2048, 1024, 1024), 1);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<32>(o);
      mbar_arrive(&empty_bar[stage]);
      if (++stage == kRing) {
        stage = 0;
        phase ^= 1;
      }
    }
    // normalise this key set's result
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
      l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
    }
    const float w = set ? p.ip_scale : 1.0f;
    const float inv[2] = {w / l_run[0], w / l_run[1]};
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float v = o[i] * inv[(i >> 1) & 1];
      res[i] = set ? res[i] + v : v;
    }
  }

  // bf16 output, two columns per store
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int n = q0 + r0 + 8 * h;
    if (n >= p.Nq) continue;
    __nv_bfloat16* orow = p.out + (static_cast<size_t>(b) * p.Nq + n) * p.ldo + head * kHd + cq;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(orow + j * 8) = pack_bf16(res[4 * j + 2 * h], res[4 * j + 2 * h + 1]);
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static bool make_tok_map(CUtensorMap* m, const void* base, int cols, int ld, int tokens, int batch, int box_rows) {
  const uint64_t dims[3] = {static_cast<uint64_t>(cols), static_cast<uint64_t>(tokens), static_cast<uint64_t>(batch)};
  const uint64_t strides[2] = {static_cast<uint64_t>(ld) * 2, static_cast<uint64_t>(tokens) * ld * 2};
  const uint32_t box[3] = {kHd, static_cast<uint32_t>(box_rows), 1};
  return encode_tmap_bf16(m, base, 3, dims, strides, box, nullptr);
}

static int launch_attn(const CUtensorMap& tmQ, const CUtensorMap& tmK0, const CUtensorMap& tmK1, const AttnParams& p,
                       int B, int heads, cudaStream_t st) {
  static bool attr_set[kMaxDevices] = {};
  bool& set = attr_set[device_slot()];
  if (!set) {
    DS_CUDA_OK(cudaFuncSetAttribute(attn_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmemBytes));
    set = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((p.Nq + kQTile - 1) / kQTile, heads, B);
  cfg.blockDim = dim3(kAttnThreads);
  cfg.dynamicSmemBytes = kAttnSmemBytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  pdl_attr(&attr[0]);
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  DS_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_wgmma_kernel, tmQ, tmK0, tmK1, p));
  DS_LAUNCH_OK("attn_wgmma_kernel");
  return DS_OK;
}

// Q [B][Nq][ldq] (head h at column q_col0 + 64 h) against K / V [B][Nkv][ldkv] at columns k_col0 / v_col0 + 64 h
static int launch_flash(const void* q, int ldq, int q_cols, const void* kv, int ldkv, int kv_cols, int k_col0,
                        int v_col0, void* out, int ldo, int B, int Nq, int Nkv, int heads, float scale, cudaStream_t st) {
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  CUtensorMap tmQ, tmK;
  if (!make_tok_map(&tmQ, q, q_cols, ldq, Nq, B, kQTile)) return DS_ERR_CUDA;
  if (!make_tok_map(&tmK, kv, kv_cols, ldkv, Nkv, B, kKTile)) return DS_ERR_CUDA;
  AttnParams p{};
  p.out = static_cast<__nv_bfloat16*>(out);
  p.Nq = Nq;
  p.ldo = ldo;
  p.n_keys[0] = Nkv;
  p.n_keys[1] = 0;
  p.k_col0 = k_col0;
  p.v_col0 = v_col0;
  p.scale_log2 = scale * kLog2e;
  return launch_attn(tmQ, tmK, tmK, p, B, heads, st);
}

}  // namespace ds

using namespace ds;

extern "C" int ds_attention_self(const void* qkv, void* out, int B, int N, int heads, void* stream) {
  DS_REQUIRE(qkv && out, "ds_attention_self: NULL pointer");
  DS_REQUIRE(B > 0 && N > 0 && heads > 0, "ds_attention_self: bad shape");
  DS_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
             "ds_attention_self: pointers must be 16-byte aligned");
  const int C = heads * kHd;
  // tensor maps over the fused [B][N][3C] projection; K and V are column offsets C and 2C
  return launch_flash(qkv, 3 * C, 3 * C, qkv, 3 * C, 3 * C, C, 2 * C, out, C, B, N, N, heads, 0.125f,
                      static_cast<cudaStream_t>(stream));
}

extern "C" int ds_resampler_attn(const void* q, const void* kv, void* out, int Bc, int nq, int n_kv, int heads,
                                 void* stream) {
  DS_REQUIRE(q && kv && out, "ds_resampler_attn: NULL pointer");
  DS_REQUIRE(Bc > 0 && nq > 0 && n_kv > 0 && heads > 0, "ds_resampler_attn: bad shape");
  DS_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(kv) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(out) & 15) == 0,
             "ds_resampler_attn: pointers must be 16-byte aligned");
  const int C = heads * kHd;
  // (q * d^-1/4)(k * d^-1/4)^T == q k^T / sqrt(d)   (src/models/resampler.py:69-70)
  return launch_flash(q, C, C, kv, 2 * C, 2 * C, 0, C, out, C, Bc, nq, n_kv, heads, 0.125f,
                      static_cast<cudaStream_t>(stream));
}

extern "C" int ds_attention_cross_ip(const ds_cross_ip_args* a, void* stream) {
  DS_REQUIRE(a != nullptr, "ds_attention_cross_ip: args is NULL");
  DS_REQUIRE(a->q && a->kv_text && a->kv_ip && a->bbox && a->out, "ds_attention_cross_ip: NULL pointer");
  DS_REQUIRE(a->B > 0 && a->N > 0 && a->heads > 0, "ds_attention_cross_ip: bad shape");
  DS_REQUIRE(a->n_text > 0 && a->n_ip > 0, "ds_attention_cross_ip: n_text and n_ip must be positive");
  DS_REQUIRE(a->num_ips > 0 && a->num_ips <= kMaxIps && a->tokens_per_ip > 0 && a->num_dummy >= 0 &&
                 a->num_dummy + a->num_ips * a->tokens_per_ip == a->n_ip,
             "ds_attention_cross_ip: n_ip (%d) != num_dummy (%d) + num_ips (%d) * tokens_per_ip (%d)", a->n_ip,
             a->num_dummy, a->num_ips, a->tokens_per_ip);
  DS_REQUIRE((reinterpret_cast<uintptr_t>(a->q) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->kv_text) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(a->kv_ip) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->out) & 15) == 0,
             "ds_attention_cross_ip: pointers must be 16-byte aligned");
  int Hd, Wd;
  if (!derive_hw(a->N, a->aspect_ratio, &Hd, &Wd)) {
    set_error("ds_attention_cross_ip: cannot factor N=%d for aspect_ratio=%f", a->N, a->aspect_ratio);
    return DS_ERR_INVALID;
  }
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  const int C = a->heads * kHd;
  CUtensorMap tmQ, tmT, tmI;
  if (!make_tok_map(&tmQ, a->q, C, C, a->N, a->B, kQTile)) return DS_ERR_CUDA;
  if (!make_tok_map(&tmT, a->kv_text, 2 * C, 2 * C, a->n_text, a->B, kKTile)) return DS_ERR_CUDA;
  if (!make_tok_map(&tmI, a->kv_ip, 2 * C, 2 * C, a->n_ip, a->B, kKTile)) return DS_ERR_CUDA;
  AttnParams p{};
  p.out = static_cast<__nv_bfloat16*>(a->out);
  p.Nq = a->N;
  p.ldo = C;
  p.n_keys[0] = a->n_text;
  p.n_keys[1] = a->n_ip;
  p.k_col0 = 0;
  p.v_col0 = C;
  p.scale_log2 = 0.125f * kLog2e;
  p.bbox = a->bbox;
  p.num_ips = a->num_ips;
  p.tokens_per_ip = a->tokens_per_ip;
  p.num_dummy = a->num_dummy;
  p.Hd = Hd;
  p.Wd = Wd;
  p.ip_scale = a->ip_scale;
  return launch_attn(tmQ, tmT, tmI, p, a->B, a->heads, static_cast<cudaStream_t>(stream));
}
