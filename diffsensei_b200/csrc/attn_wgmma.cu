// attn_wgmma.cu — fused attention for head_dim 64 on sm_90a warpgroup tensor cores.
//
// Four entry points:
//   ds_attention_self      self-attention (AttnProcessor2_0, src/models/attention_processor.py:69-81):
//                          softmax(Q K^T / 8) V over the fused [B][N][3C] projection, no mask;
//   ds_attention_self_pag  the same launch for perturbed-attention guidance: batch rows from first_perturbed_row on
//                          take the identity attention map (out = V, diffusers' PAGCFGIdentitySelfAttnProcessor2_0),
//                          their CTAs copy V instead of running the flash pipeline;
//   ds_resampler_attn      the Resampler's perceiver attention (src/models/resampler.py:64-74), same math;
//   ds_attention_cross_ip  out = softmax(Q Kt^T/8) Vt + scale * softmax(Q Kip^T/8 + M(bbox)) Vip
//                          (MaskedIPAttnProcessor2_0, :231-258) in ONE pass over both key sets; the additive bbox mask
//                          M in {0,-10000} (:115-169) is evaluated in registers with the reference's closed-interval /
//                          derived-(H',W') semantics (ip_mask.cuh).
// Q/K/V are addressed by 3-D tensor maps {columns, tokens, batch} over the projection outputs, so the head split /
// transposes of the reference are never materialised.
//
// Two kernels share the per-tile steps (S = Q K^T, masked online-softmax step, O += P V, normalise, store):
//   attn_stream_kernel    CTA = 128 query rows of one (batch, head); its keys stream through a RING-deep ring of
//                         64-key K|V tiles.  Self-attention, the Resampler, and cross-attention whose key sets are too
//                         long to stay resident.
//   attn_cross_kernel     persistent; a CTA walks a contiguous range of (batch, head, 128-row query tile) items.  Both
//                         key sets of the current (batch, head) stay resident in shared memory and the query tiles
//                         stream through a double buffer, so a tile's load overlaps the previous tile's MMAs.
// Both: 384 threads; warpgroup 0 is one TMA lane, warpgroups 1-2 own 64 query rows each (a row lives in the 4 threads
// of a quad).  Within a key set the consumer loop is software-pipelined: tile t+1's S = Q K^T and tile t's O += P V
// are in flight while tile t+1's exponentials run.  Keys past the end of a key set arrive as TMA zero fill and are
// masked to -inf; only a set's partial last tile and the IP set take the masked softmax step.
#include <cstdlib>

#include "ds_common.cuh"
#include "ds_host.h"
#include "ip_mask.cuh"
#include "wgmma.cuh"

namespace ds {

constexpr int kQTile = 128;  // query rows per CTA / per item
constexpr int kKTile = 64;   // keys per pipeline stage
constexpr int kHd = 64;      // head dim
constexpr int kRing = 4;
constexpr int kAttnThreads = 384;
constexpr int kQBytes = kQTile * kHd * 2;   // 16 KiB
constexpr int kKVBytes = kKTile * kHd * 2;  // 8 KiB each for K and V
constexpr int kStreamSmemBytes = kQBytes + kRing * 2 * kKVBytes + 1024 /*align*/ + 256 /*barriers*/;
// cross-attention with resident keys: up to kResidentTiles K|V tiles of both sets together, two Q buffers
constexpr int kResidentTiles = 4;
constexpr int kQBufs = 2;
constexpr int kCrossSmemBytes = kResidentTiles * 2 * kKVBytes + kQBufs * kQBytes + 1024 + 256;
constexpr float kLog2e = 1.4426950408889634f;
// Register budgets after setmaxnreg (the launch gives every thread 168): one TMA lane in the producer warpgroup, the
// pipelined consumers hold O, two score tiles' worth of S / P and the softmax state.  128 * 40 + 256 * 232 <= 65536.
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;

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
  // attn_cross_kernel: items are (batch, head, query tile) in that nesting; CTA c walks [c * items / ctas, ...)
  int heads, q_tiles, items;
  // attn_stream_kernel, perturbed-attention guidance: when v_src is set, the CTAs of batch rows >= pag_b0 copy their
  // rows of V (v_src [B][Nq][ld_src], head h at columns [64 h, +64)) to out instead of attending (identity map)
  const __nv_bfloat16* v_src;
  int ld_src, pag_b0;
};

// The identity-attention rows of one CTA: out rows [q0, q0 + 128) of (b, head) = V, 16-byte vectors.  Every thread of
// the CTA takes part; no shared memory, no barrier.
__device__ __forceinline__ void copy_v_rows(const AttnParams& p, int b, int head, int q0) {
  const int rows = min(kQTile, p.Nq - q0);
  const size_t src0 = (static_cast<size_t>(b) * p.Nq + q0) * p.ld_src + head * kHd;
  const size_t dst0 = (static_cast<size_t>(b) * p.Nq + q0) * p.ldo + head * kHd;
  for (int i = threadIdx.x; i < rows * (kHd / 8); i += kAttnThreads) {
    const int r = i >> 3, c = (i & 7) * 8;
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(p.v_src + src0 + static_cast<size_t>(r) * p.ld_src + c));
    *reinterpret_cast<uint4*>(p.out + dst0 + static_cast<size_t>(r) * p.ldo + c) = v;
  }
}

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// What the softmax step masks in one key set
struct SetMask {
  int nk;               // keys at or past nk score -inf
  bool ip;              // the bbox mask applies (IP set)
  uint32_t ip_bits[2];  // rows r0 and r0 + 8: bit i set <=> the row's pixel lies in box i
  int tokens_per_ip, num_dummy;
};

// S[64 x 64] = Q K^T for one 64-key tile, both operands K-major in shared memory (issued, not waited)
__device__ __forceinline__ void issue_qk(float (&s)[32], uint32_t q_addr, uint32_t k_addr) {
#pragma unroll
  for (int k = 0; k < kHd / 16; ++k)
    wgmma_m64n64_ss(s, make_wgmma_desc(q_addr + k * 32, 1024, 16), make_wgmma_desc(k_addr + k * 32, 1024, 16), k != 0);
}

// O[64 x 64] += P V, P as the register A operand, V MN-major in shared memory (issued, not waited)
__device__ __forceinline__ void issue_pv(float (&o)[32], const uint32_t (&pa)[4][4], uint32_t v_addr) {
#pragma unroll
  for (int kk = 0; kk < kKTile / 16; ++kk)
    wgmma_m64n64_rs_tb(o, pa[kk], make_wgmma_desc(v_addr + kk * 2048, 1024, 1024), 1);
}

// O and P are written by ordinary instructions (zeroing, rescale, the P copy) that must all precede the next wgmma
// fence: ptxas serialises every wgmma of a pipeline stage whose register inputs are defined inside it.
__device__ __forceinline__ void fence_operands(float (&o)[32], uint32_t (&pa)[4][4]) {
  fence_regs<32>(o);
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(pa[kk][i])::"memory");
}

// One 64-key online-softmax step: scores -> log2 domain (+ mask), running max / sum update, P as the bf16 A fragments
// of the four 16-key MMA slices, and the factor corr by which O must be rescaled before P V is added.
// open[h]: the IP keys open to row h (ip_open_keys64), shifted down by the thread's column cq.
template <bool kMasked>
__device__ __forceinline__ void softmax_step(const float (&s)[32], int key0, const SetMask& mk,
                                             const uint64_t (&open)[2], float scale_log2, int cq, float (&m_run)[2],
                                             float (&l_run)[2], float (&corr)[2], uint32_t (&pa)[4][4]) {
  float x[32];  // not in place: s may be the accumulator of an MMA group still open
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int key = key0 + j * 8 + cq + (e & 1);
      const int h = e >> 1;
      float v = s[4 * j + e] * scale_log2;
      if (kMasked) {
        if (mk.ip && !((open[h] >> (j * 8 + (e & 1))) & 1u)) v -= 10000.0f * kLog2e;
        if (key >= mk.nk) v = -INFINITY;
      }
      x[4 * j + e] = v;
      mx[h] = fmaxf(mx[h], v);
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    const float m_new = fmaxf(m_run[h], mx[h]);
    corr[h] = ex2(m_run[h] - m_new);  // 0 on the first tile (m_run = -inf)
    m_run[h] = m_new;
    l_run[h] *= corr[h];
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float p0 = ex2(x[4 * j + 2 * h] - m_run[h]);
      const float p1 = ex2(x[4 * j + 2 * h + 1] - m_run[h]);
      l_run[h] += p0 + p1;
      pa[j >> 1][(j & 1) * 2 + h] = pack_bf16(p0, p1);
    }
  }
}

__device__ __forceinline__ void softmax_tile(const float (&s)[32], int key0, const SetMask& mk, float scale_log2, int cq,
                                             float (&m_run)[2], float (&l_run)[2], float (&corr)[2],
                                             uint32_t (&pa)[4][4]) {
  uint64_t open[2] = {0ull, 0ull};
  if (mk.ip) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      open[h] = ip_open_keys64(mk.ip_bits[h], key0, mk.tokens_per_ip, mk.num_dummy) >> cq;
  }
  if (mk.ip || key0 + kKTile > mk.nk)
    softmax_step<true>(s, key0, mk, open, scale_log2, cq, m_run, l_run, corr, pa);
  else
    softmax_step<false>(s, key0, mk, open, scale_log2, cq, m_run, l_run, corr, pa);
}

// o = unnormalised softmax(Q K^T) V over one key set of n_tiles 64-key tiles; l_run = the quad-partial row sums.
// tile_addr(t) waits for tile t and returns its K address (V follows at + kKVBytes); release(t) hands it back once
// the MMAs reading it have retired.  Tile t+1's S and tile t's P V are in flight while tile t+1's softmax step runs,
// so P alternates between two register sets: the step writes the one the MMA in flight does not read.
template <class TileAddr, class Release>
__device__ __forceinline__ void attend_set(float (&o)[32], float (&l_run)[2], uint32_t q_addr, int n_tiles,
                                           const SetMask& mk, float scale_log2, int cq, TileAddr tile_addr,
                                           Release release) {
  float m_run[2] = {-INFINITY, -INFINITY};
  l_run[0] = l_run[1] = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float s[32], corr[2];
  uint32_t pa[4][4], pb[4][4];
  uint32_t k_addr = tile_addr(0);
  wgmma_fence();
  issue_qk(s, q_addr, k_addr);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs<32>(s);
  softmax_tile(s, 0, mk, scale_log2, cq, m_run, l_run, corr, pa);  // O is still zero: no rescale

  // tile t's P V (P in cur) and tile t+1's S; tile t+1's softmax step writes next
  auto step = [&](int t, uint32_t(&cur)[4][4], uint32_t(&next)[4][4]) {
    const uint32_t k_next = tile_addr(t + 1);
    fence_operands(o, cur);
    wgmma_fence();
    issue_qk(s, q_addr, k_next);
    wgmma_commit();
    issue_pv(o, cur, k_addr + kKVBytes);
    wgmma_commit();
    wgmma_wait<1>();
    fence_regs<32>(s);
    softmax_tile(s, (t + 1) * kKTile, mk, scale_log2, cq, m_run, l_run, corr, next);
    wgmma_wait<0>();
    fence_regs<32>(o);
    release(t);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[4 * j + 0] *= corr[0];
      o[4 * j + 1] *= corr[0];
      o[4 * j + 2] *= corr[1];
      o[4 * j + 3] *= corr[1];
    }
    k_addr = k_next;
  };
  auto last = [&](int t, uint32_t(&cur)[4][4]) {
    fence_operands(o, cur);
    wgmma_fence();
    issue_pv(o, cur, k_addr + kKVBytes);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<32>(o);
    release(t);
  };
  for (int t = 0;; t += 2) {
    if (t + 1 == n_tiles) {
      last(t, pa);
      break;
    }
    step(t, pa, pb);
    if (t + 2 == n_tiles) {
      last(t + 1, pb);
      break;
    }
    step(t + 1, pb, pa);
  }
}

// res (= or +=) w * o / l, with the row sums completed over the quad
__device__ __forceinline__ void normalise_into(float (&res)[32], const float (&o)[32], float (&l_run)[2], float w,
                                               bool accumulate) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
  }
  const float inv[2] = {w / l_run[0], w / l_run[1]};
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const float v = o[i] * inv[(i >> 1) & 1];
    res[i] = accumulate ? res[i] + v : v;
  }
}

// bf16 output, two columns per store; rows past Nq (TMA zero fill of the last query tile) are dropped
__device__ __forceinline__ void store_rows(const AttnParams& p, const float (&res)[32], int b, int head, int row0,
                                           int cq) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int n = row0 + 8 * h;
    if (n >= p.Nq) continue;
    __nv_bfloat16* orow = p.out + (static_cast<size_t>(b) * p.Nq + n) * p.ldo + head * kHd + cq;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(orow + j * 8) = pack_bf16(res[4 * j + 2 * h], res[4 * j + 2 * h + 1]);
  }
}

__device__ __forceinline__ void ip_row_bits(const AttnParams& p, int b, int row0, uint32_t (&bits)[2]) {
  const float* bb = p.bbox + static_cast<size_t>(b) * p.num_ips * 4;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int n = row0 + 8 * h;
    bits[h] = n < p.Nq ? ip_inside_bits(bb, p.num_ips, n, p.Hd, p.Wd) : 0u;
  }
}

__device__ __forceinline__ SetMask set_mask(const AttnParams& p, int set, const uint32_t (&bits)[2]) {
  SetMask mk;
  mk.nk = set ? p.n_keys[1] : p.n_keys[0];
  mk.ip = set == 1;
  mk.ip_bits[0] = bits[0];
  mk.ip_bits[1] = bits[1];
  mk.tokens_per_ip = p.tokens_per_ip;
  mk.num_dummy = p.num_dummy;
  return mk;
}

__global__ void __launch_bounds__(kAttnThreads, 1)
attn_stream_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK0,
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

  if (p.v_src != nullptr && b >= p.pag_b0) {  // a perturbed row (uniform per CTA): identity attention, out = V
    pdl_launch_dependents();
    pdl_wait();
    copy_v_rows(p, b, head, q0);
    return;
  }

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
    setmaxnreg_dec<kProducerRegs>();
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
  setmaxnreg_inc<kConsumerRegs>();
  const int ct = threadIdx.x - 128;
  const int wg = ct >> 7;
  const int r0 = (ct >> 5) * 16 + (lane >> 2);  // tile rows r0 and r0 + 8
  const int cq = 2 * (lane & 3);
  uint32_t ip_bits[2] = {0u, 0u};
  if (tiles1 > 0) ip_row_bits(p, b, q0 + r0, ip_bits);
  const uint32_t q_addr = smem_u32(sQ) + wg * 64 * 128;
  const uint32_t ring_addr = smem_u32(sRing);
  mbar_wait(q_bar, 0);

  float o[32], res[32], l_run[2];
  int stage = 0;
  uint32_t phase = 0;
  auto tile_addr = [&](int) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t a = ring_addr + stage * 2 * kKVBytes;
    if (++stage == kRing) {
      stage = 0;
      phase ^= 1;
    }
    return a;
  };
  int rstage = 0;
  auto release = [&](int) {
    mbar_arrive(&empty_bar[rstage]);
    if (++rstage == kRing) rstage = 0;
  };
  for (int set = 0; set < (tiles1 > 0 ? 2 : 1); ++set) {
    const SetMask mk = set_mask(p, set, ip_bits);
    attend_set(o, l_run, q_addr, set ? tiles1 : tiles0, mk, p.scale_log2, cq, tile_addr, release);
    normalise_into(res, o, l_run, set ? p.ip_scale : 1.0f, set != 0);
  }
  store_rows(p, res, b, head, q0 + r0, cq);
}

__global__ void __launch_bounds__(kAttnThreads, 1)
attn_cross_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK0,
                  const __grid_constant__ CUtensorMap tmK1, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sKV = smem;  // tile t (set 0's tiles, then set 1's): K at t * 16 KiB, V at t * 16 KiB + 8 KiB
  uint8_t* sQ = sKV + kResidentTiles * 2 * kKVBytes;
  uint64_t* kv_full = reinterpret_cast<uint64_t*>(sQ + kQBufs * kQBytes);
  uint64_t* kv_empty = kv_full + 1;
  uint64_t* q_full = kv_empty + 1;
  uint64_t* q_empty = q_full + kQBufs;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles0 = (p.n_keys[0] + kKTile - 1) / kKTile;
  const int tiles1 = (p.n_keys[1] + kKTile - 1) / kKTile;
  const int item_lo = static_cast<int>(static_cast<long long>(blockIdx.x) * p.items / gridDim.x);
  const int item_hi = static_cast<int>(static_cast<long long>(blockIdx.x + 1) * p.items / gridDim.x);

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK0);
    tma_prefetch_desc(&tmK1);
    mbar_init(kv_full, 1);
    mbar_init(kv_empty, 256);
    for (int i = 0; i < kQBufs; ++i) {
      mbar_init(&q_full[i], 1);
      mbar_init(&q_empty[i], 256);
    }
    fence_mbar_init();
  }
  pdl_launch_dependents();
  __syncthreads();
  pdl_wait();

  if (warp < 4) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      int pair = -1;
      uint32_t kv_phase = 0;
      for (int item = item_lo, it = 0; item < item_hi; ++item, ++it) {
        const int ip = item / p.q_tiles, qt = item - ip * p.q_tiles;
        const int b = ip / p.heads, head = ip - b * p.heads;
        if (ip != pair) {  // the next (batch, head): its keys replace the previous ones once those are released
          pair = ip;
          mbar_wait(kv_empty, kv_phase ^ 1);
          kv_phase ^= 1;
          mbar_arrive_expect_tx(kv_full, (tiles0 + tiles1) * 2 * kKVBytes);
          for (int t = 0; t < tiles0 + tiles1; ++t) {
            const bool second = t >= tiles0;
            const CUtensorMap* m = second ? &tmK1 : &tmK0;
            const int key0 = (second ? t - tiles0 : t) * kKTile;
            uint8_t* sK = sKV + t * 2 * kKVBytes;
            tma_load_3d(sK, m, kv_full, p.k_col0 + head * kHd, key0, b);
            tma_load_3d(sK + kKVBytes, m, kv_full, p.v_col0 + head * kHd, key0, b);
          }
        }
        const int buf = it & 1;
        mbar_wait(&q_empty[buf], ((it >> 1) & 1) ^ 1);
        mbar_arrive_expect_tx(&q_full[buf], kQBytes);
        tma_load_3d(sQ + buf * kQBytes, &tmQ, &q_full[buf], head * kHd, qt * kQTile, b);
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumers
  setmaxnreg_inc<kConsumerRegs>();
  const int ct = threadIdx.x - 128;
  const int wg = ct >> 7;
  const int r0 = (ct >> 5) * 16 + (lane >> 2);  // tile rows r0 and r0 + 8
  const int cq = 2 * (lane & 3);
  const uint32_t kv_addr = smem_u32(sKV);
  const uint32_t q_base = smem_u32(sQ) + wg * 64 * 128;
  int pair = -1;
  uint32_t kv_phase = 0;
  for (int item = item_lo, it = 0; item < item_hi; ++item, ++it) {
    const int ip = item / p.q_tiles, qt = item - ip * p.q_tiles;
    const int b = ip / p.heads, head = ip - b * p.heads;
    const int q0 = qt * kQTile;
    if (ip != pair) {
      if (pair >= 0) mbar_arrive(kv_empty);
      pair = ip;
      mbar_wait(kv_full, kv_phase);
      kv_phase ^= 1;
    }
    uint32_t ip_bits[2];
    ip_row_bits(p, b, q0 + r0, ip_bits);
    const int buf = it & 1;
    const uint32_t q_addr = q_base + buf * kQBytes;
    mbar_wait(&q_full[buf], (it >> 1) & 1);
    float o[32], res[32], l_run[2];
    for (int set = 0; set < 2; ++set) {
      const SetMask mk = set_mask(p, set, ip_bits);
      const uint32_t set_addr = kv_addr + (set ? tiles0 : 0) * 2 * kKVBytes;
      attend_set(o, l_run, q_addr, set ? tiles1 : tiles0, mk, p.scale_log2, cq,
                 [&](int t) { return set_addr + t * 2 * kKVBytes; }, [](int) {});
      normalise_into(res, o, l_run, set ? p.ip_scale : 1.0f, set != 0);
    }
    mbar_arrive(&q_empty[buf]);
    store_rows(p, res, b, head, q0 + r0, cq);
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

using AttnKernel = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, AttnParams);

// attr_set: one flag per device, for the kernel's dynamic shared memory opt-in
static int launch_attn(AttnKernel kernel, const char* name, int smem_bytes, bool* attr_set, dim3 grid,
                       const CUtensorMap& tmQ, const CUtensorMap& tmK0, const CUtensorMap& tmK1, const AttnParams& p,
                       cudaStream_t st) {
  bool& set = attr_set[device_slot()];
  if (!set) {
    DS_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    set = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(kAttnThreads);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  pdl_attr(&attr[0]);
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  DS_CUDA_OK(cudaLaunchKernelEx(&cfg, kernel, tmQ, tmK0, tmK1, p));
  DS_LAUNCH_OK(name);
  return DS_OK;
}

static int launch_stream(const CUtensorMap& tmQ, const CUtensorMap& tmK0, const CUtensorMap& tmK1,
                         const AttnParams& p, int B, int heads, cudaStream_t st) {
  static bool attr_set[kMaxDevices] = {};
  return launch_attn(attn_stream_kernel, "attn_stream_kernel", kStreamSmemBytes, attr_set,
                     dim3((p.Nq + kQTile - 1) / kQTile, heads, B), tmQ, tmK0, tmK1, p, st);
}

// Q [B][Nq][ldq] (head h at column q_col0 + 64 h) against K / V [B][Nkv][ldkv] at columns k_col0 / v_col0 + 64 h
static int launch_flash(const void* q, int ldq, int q_cols, const void* kv, int ldkv, int kv_cols, int k_col0,
                        int v_col0, void* out, int ldo, int B, int Nq, int Nkv, int heads, float scale, cudaStream_t st,
                        const void* v_src = nullptr, int pag_b0 = 0) {
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
  p.v_src = static_cast<const __nv_bfloat16*>(v_src);
  p.ld_src = ldkv;
  p.pag_b0 = pag_b0;
  return launch_stream(tmQ, tmK, tmK, p, B, heads, st);
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

extern "C" int ds_attention_self_pag(const void* qkv, void* out, int B, int N, int heads, int first_perturbed_row,
                                     void* stream) {
  DS_REQUIRE(qkv && out, "ds_attention_self_pag: NULL pointer");
  DS_REQUIRE(B > 0 && N > 0 && heads > 0, "ds_attention_self_pag: bad shape");
  DS_REQUIRE(first_perturbed_row >= 0 && first_perturbed_row <= B,
             "ds_attention_self_pag: first_perturbed_row (%d) must be in [0, B = %d]", first_perturbed_row, B);
  DS_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
             "ds_attention_self_pag: pointers must be 16-byte aligned");
  const int C = heads * kHd;
  // ds_attention_self's launch; the CTAs of rows >= first_perturbed_row copy the V third instead of attending
  return launch_flash(qkv, 3 * C, 3 * C, qkv, 3 * C, 3 * C, C, 2 * C, out, C, B, N, N, heads, 0.125f,
                      static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(qkv) + 2 * C,
                      first_perturbed_row);
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
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int tiles = (a->n_text + kKTile - 1) / kKTile + (a->n_ip + kKTile - 1) / kKTile;
  if (tiles > kResidentTiles) return launch_stream(tmQ, tmT, tmI, p, a->B, a->heads, st);
  // both key sets stay resident: one persistent CTA per SM over contiguous runs of (batch, head, query tile)
  p.heads = a->heads;
  p.q_tiles = (a->N + kQTile - 1) / kQTile;
  const long long items = static_cast<long long>(a->B) * a->heads * p.q_tiles;
  DS_REQUIRE(items <= INT32_MAX, "ds_attention_cross_ip: too many query tiles");
  p.items = static_cast<int>(items);
  const int ctas = static_cast<int>(items < dev.num_sms ? items : dev.num_sms);
  static bool attr_set[kMaxDevices] = {};
  return launch_attn(attn_cross_kernel, "attn_cross_kernel", kCrossSmemBytes, attr_set, dim3(ctas), tmQ, tmT, tmI,
                     p, st);
}
