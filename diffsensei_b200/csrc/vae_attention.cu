// vae_attention.cu — ds_attention_single_head: one-head flash attention of width 128 or 512 on sm_90a.
//
// The AutoencoderKL decoder's mid-block attention (diffusers Attention(heads=1, dim_head=C), residual_connection) is
// ONE head as wide as the last block_out_channels (512 in SDXL's VAE, 128 in TINY_VAE) over all H*W latent tokens.
// A softmax over a 512-wide dot product cannot be split into the flash kernel's 64-wide heads (attn_wgmma.cu), so it
// has its own kernel:  O[b] = softmax(Q[b] K[b]^T / sqrt(D)) V[b]  for a batch of B images in one launch, with no
// scratch memory and no alignment condition on N.
//
// CTA = 64 query rows of one image, NWG = D / 128 warpgroups; warpgroup w owns the 128-wide slice [128 w, 128 w + 128)
// of d and of the output.  Thread 0 issues the TMA loads: the 64 x D Q tile, then 32-key K|V tiles (32 x D each)
// through a kRing-deep ring of stages (a stage is refilled once every warpgroup is past the tile that used it; a
// separate producer warp would cost registers: 17 warps leave 96 per thread, 16 leave 128).  Per key tile:
//     1. partial scores S_w = Q[:, slice] K[:, slice]^T (wgmma, both operands in smem), stored fp32 to smem;
//     2. each thread sums the NWG partials of one row over 32 / (2 NWG) keys and takes the online-softmax
//        step for them (fp32 running max and sum, shared by the 2 NWG threads of the row through shuffles), then
//        writes P (bf16) and the row's rescale factor to smem: every score is exponentiated once, not once per
//        warpgroup;
//     3. O_w = corr * O_w + P V[:, slice] (wgmma with P as the register A operand, V MN-major).
//   Two CTA barriers per tile separate the phases.  P lives in the stage's K buffer, dead once every S_w is done.
// Q/K/V rows past N arrive as TMA zero fill (the 3-D tensor maps end at N tokens per image), keys >= N are masked to
// -inf before the softmax, and rows >= N are never stored.  P is rounded to bf16 before the PV MMA, as in
// attn_wgmma.cu; scores, running max / sum and the output accumulator are fp32.
#include <cmath>

#include "ds_common.cuh"
#include "ds_host.h"
#include "wgmma.cuh"

namespace ds {

template <int D>
struct SingleHead {
  static constexpr int kWG = D / 128;                 // warpgroups
  static constexpr int kThreads = kWG * 128;
  static constexpr int kRows = 64;                    // query rows per CTA
  static constexpr int kKeys = 32;                    // keys per pipeline stage
  static constexpr int kRing = D == 512 ? 2 : 4;
  static constexpr int kQBox = kRows * 128;           // one 64-column TMA box of the Q tile (128 B rows)
  static constexpr int kKBox = kKeys * 128;           // ... of a K or V tile
  static constexpr int kQBytes = kRows * D * 2;
  static constexpr int kKVBytes = kKeys * D * 2;      // K (or V) of one stage
  static constexpr int kRedFloats = kWG * kRows * kKeys;
  static constexpr int kSmemBytes =
      1024 /*align*/ + kQBytes + kRing * 2 * kKVBytes + kRedFloats * 4 + kRows * 4 + 8 * (1 + kRing);
  static_assert(kSmemBytes <= 227 * 1024, "shared memory");
};

constexpr int kShPld = 40;  // P row stride in bf16: 80-byte rows keep the A-fragment loads free of bank conflicts
constexpr float kShLog2e = 1.4426950408889634f;

__device__ __forceinline__ float sh_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// column of (row, col) inside a 32-float partial-score row: rows r and r + 1..3 land on different banks
__device__ __forceinline__ int red_col(int row, int col) { return col ^ ((row & 3) << 3); }

template <int D>
__global__ void __launch_bounds__(SingleHead<D>::kThreads, 1)
attn_single_head_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmV, __nv_bfloat16* __restrict__ out, int N,
                        float scale_log2) {
  using T = SingleHead<D>;
  constexpr int kWG = T::kWG, kRows = T::kRows, kKeys = T::kKeys, kRing = T::kRing;
  constexpr int kTpr = 2 * kWG;          // softmax threads per row
  constexpr int kKpt = kKeys / kTpr;     // keys per softmax thread
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sRing = sQ + T::kQBytes;  // stage s: K at s * 2 * kKVBytes, V kKVBytes later
  float* sRed = reinterpret_cast<float*>(sRing + kRing * 2 * T::kKVBytes);  // [kWG][64][32] partial scores
  float* sCorr = sRed + T::kRedFloats;                                       // [64] per-row rescale, then 1 / sum
  uint64_t* q_bar = reinterpret_cast<uint64_t*>(sCorr + kRows);
  uint64_t* full_bar = q_bar + 1;

  const int ct = threadIdx.x, lane = ct & 31;
  const int q0 = blockIdx.x * kRows, b = blockIdx.y;
  const int tiles = (N + kKeys - 1) / kKeys;
  auto load_tile = [&](int t) {  // K|V keys [32 t, 32 t + 32) into stage t % kRing
    const int st = t % kRing;
    uint8_t* sK = sRing + st * 2 * T::kKVBytes;
    mbar_arrive_expect_tx(&full_bar[st], 2 * T::kKVBytes);
#pragma unroll
    for (int c = 0; c < D / 64; ++c) {
      tma_load_3d(sK + c * T::kKBox, &tmK, &full_bar[st], c * 64, t * kKeys, b);
      tma_load_3d(sK + T::kKVBytes + c * T::kKBox, &tmV, &full_bar[st], c * 64, t * kKeys, b);
    }
  };

  if (ct == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_bar, 1);
    for (int i = 0; i < kRing; ++i) mbar_init(&full_bar[i], 1);
    fence_mbar_init();
  }
  pdl_launch_dependents();
  __syncthreads();
  pdl_wait();
  if (ct == 0) {
    mbar_arrive_expect_tx(q_bar, T::kQBytes);
#pragma unroll
    for (int c = 0; c < D / 64; ++c) tma_load_3d(sQ + c * T::kQBox, &tmQ, q_bar, c * 64, q0, b);
    for (int t = 0; t < kRing && t < tiles; ++t) load_tile(t);
  }

  const int wg = ct >> 7;
  const int r0 = ((ct >> 5) & 3) * 16 + (lane >> 2);  // accumulator rows r0 and r0 + 8 of this warpgroup's tiles
  const int cq = 2 * (lane & 3);
  const int sr = ct / kTpr, sk0 = (ct % kTpr) * kKpt;  // softmax: row sr, keys [sk0, sk0 + kKpt) of each tile
  const uint32_t q_addr = smem_u32(sQ) + wg * 2 * T::kQBox;
  float* red_own = sRed + wg * kRows * kKeys;

  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_run = -INFINITY, l_run = 0.f;
  mbar_wait(q_bar, 0);

  int stage = 0;
  uint32_t phase = 0;
  for (int t = 0; t < tiles; ++t) {
    mbar_wait(&full_bar[stage], phase);
    uint8_t* sK = sRing + stage * 2 * T::kKVBytes;
    const uint32_t k_addr = smem_u32(sK) + wg * 2 * T::kKBox;
    const uint32_t v_addr = smem_u32(sK + T::kKVBytes) + wg * 2 * T::kKBox;

    // 1. partial scores over this warpgroup's 128 columns of d (two 64-column boxes, four 16-wide k steps each)
    float s[16];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 8; ++k)
      wgmma_m64n32_ss(s, make_wgmma_desc(q_addr + (k >> 2) * T::kQBox + (k & 3) * 32, 1024, 16),
                      make_wgmma_desc(k_addr + (k >> 2) * T::kKBox + (k & 3) * 32, 1024, 16), k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<16>(s);
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        *reinterpret_cast<float2*>(red_own + row * kKeys + red_col(row, 8 * j + cq)) =
            make_float2(s[4 * j + 2 * h], s[4 * j + 2 * h + 1]);
      }
    __syncthreads();
    // every warpgroup is past tile t - 1 (its PV MMAs retired, its P stores fenced): refill that stage
    if (ct == 0 && t >= 1 && t - 1 + kRing < tiles) load_tile(t - 1 + kRing);

    // 2. full scores of (row sr, kKpt keys), online-softmax step, P and the row's rescale factor to smem
    float v[kKpt];
#pragma unroll
    for (int i = 0; i < kKpt; ++i) v[i] = 0.f;
#pragma unroll
    for (int w = 0; w < kWG; ++w) {
      const float* rr = sRed + (w * kRows + sr) * kKeys;
#pragma unroll
      for (int i = 0; i < kKpt; i += 4) {
        const float4 x = *reinterpret_cast<const float4*>(rr + red_col(sr, sk0 + i));
        v[i] += x.x;
        v[i + 1] += x.y;
        v[i + 2] += x.z;
        v[i + 3] += x.w;
      }
    }
    const int key0 = t * kKeys + sk0;
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < kKpt; ++i) {
      v[i] = key0 + i < N ? v[i] * scale_log2 : -INFINITY;
      mx = fmaxf(mx, v[i]);
    }
#pragma unroll
    for (int x = 1; x < kTpr; x <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, x));
    const float m_new = fmaxf(m_run, mx);  // finite: key 0 of the first tile is always valid
    const float corr = sh_ex2(m_run - m_new);  // 0 on the first tile (m_run = -inf)
    m_run = m_new;
    uint32_t pk[kKpt / 2];
    float ls = 0.f;
#pragma unroll
    for (int i = 0; i < kKpt / 2; ++i) {
      const float p0 = sh_ex2(v[2 * i] - m_new), p1 = sh_ex2(v[2 * i + 1] - m_new);
      ls += p0 + p1;
      pk[i] = pack_bf16(p0, p1);
    }
    l_run = l_run * corr + ls;
    __nv_bfloat16* sP = reinterpret_cast<__nv_bfloat16*>(sK);  // [64][kShPld] over the consumed K tile
#pragma unroll
    for (int i = 0; i < kKpt / 4; ++i)
      *reinterpret_cast<uint2*>(sP + sr * kShPld + sk0 + 4 * i) = make_uint2(pk[2 * i], pk[2 * i + 1]);
    if (ct % kTpr == 0) sCorr[sr] = corr;
    __syncthreads();

    // 3. O = corr * O + P V over this warpgroup's 128 output columns
    uint32_t pa[2][4];
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      const __nv_bfloat16* p0 = sP + r0 * kShPld + 16 * kk + cq;
      const __nv_bfloat16* p1 = p0 + 8 * kShPld;
      pa[kk][0] = *reinterpret_cast<const uint32_t*>(p0);
      pa[kk][1] = *reinterpret_cast<const uint32_t*>(p1);
      pa[kk][2] = *reinterpret_cast<const uint32_t*>(p0 + 8);
      pa[kk][3] = *reinterpret_cast<const uint32_t*>(p1 + 8);
    }
    const float c0 = sCorr[r0], c1 = sCorr[r0 + 8];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      o[4 * j + 0] *= c0;
      o[4 * j + 1] *= c0;
      o[4 * j + 2] *= c1;
      o[4 * j + 3] *= c1;
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 2; ++kk)
      wgmma_m64n128_rs_tb(o, pa[kk], make_wgmma_desc(v_addr + kk * 2048, 1024, T::kKBox), 1);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<64>(o);
    fence_proxy_async_smem();  // the P stores (generic proxy) before TMA refills this stage
    if (++stage == kRing) {
      stage = 0;
      phase ^= 1;
    }
  }

  // normalise: the row sum lives in the kTpr softmax threads of the row
#pragma unroll
  for (int x = 1; x < kTpr; x <<= 1) l_run += __shfl_xor_sync(0xffffffffu, l_run, x);
  __syncthreads();  // every warpgroup has read the last tile's rescale factors
  if (ct % kTpr == 0) sCorr[sr] = 1.0f / l_run;
  __syncthreads();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int n = q0 + r0 + 8 * h;
    if (n >= N) continue;
    const float inv = sCorr[r0 + 8 * h];
    __nv_bfloat16* orow = out + (static_cast<size_t>(b) * N + n) * D + wg * 128 + cq;
#pragma unroll
    for (int j = 0; j < 16; ++j)
      *reinterpret_cast<uint32_t*>(orow + j * 8) = pack_bf16(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv);
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// [B][N][D] rows of stride ld elements, images N * ld apart; 64-column boxes of box_rows rows
static bool make_head_map(CUtensorMap* m, const void* base, int D, int64_t ld, int N, int B, int box_rows) {
  const uint64_t dims[3] = {static_cast<uint64_t>(D), static_cast<uint64_t>(N), static_cast<uint64_t>(B)};
  const uint64_t strides[2] = {static_cast<uint64_t>(ld) * 2, static_cast<uint64_t>(N) * ld * 2};
  const uint32_t box[3] = {64, static_cast<uint32_t>(box_rows), 1};
  return encode_tmap_bf16(m, base, 3, dims, strides, box, nullptr);
}

template <int D>
static int launch_single_head(const void* q, const void* k, const void* v, void* out, int B, int N, int64_t ld,
                              cudaStream_t st) {
  using T = SingleHead<D>;
  CUtensorMap tmQ, tmK, tmV;
  if (!make_head_map(&tmQ, q, D, ld, N, B, T::kRows)) return DS_ERR_CUDA;
  if (!make_head_map(&tmK, k, D, ld, N, B, T::kKeys)) return DS_ERR_CUDA;
  if (!make_head_map(&tmV, v, D, ld, N, B, T::kKeys)) return DS_ERR_CUDA;
  static bool attr_set[kMaxDevices] = {};
  bool& set = attr_set[device_slot()];
  if (!set) {
    DS_CUDA_OK(cudaFuncSetAttribute(attn_single_head_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    T::kSmemBytes));
    set = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((N + T::kRows - 1) / T::kRows, B);
  cfg.blockDim = dim3(T::kThreads);
  cfg.dynamicSmemBytes = T::kSmemBytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  pdl_attr(&attr[0]);
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  DS_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_single_head_kernel<D>, tmQ, tmK, tmV, static_cast<__nv_bfloat16*>(out), N,
                                kShLog2e / sqrtf(static_cast<float>(D))));
  DS_LAUNCH_OK("attn_single_head_kernel");
  return DS_OK;
}

}  // namespace ds

using namespace ds;

extern "C" int ds_attention_single_head(const void* q, const void* k, const void* v, void* out, int B, int N, int D,
                                        int64_t ld, void* stream) {
  DS_REQUIRE(q && k && v && out, "ds_attention_single_head: NULL pointer");
  DS_REQUIRE(B > 0 && B <= 65535 && N > 0, "ds_attention_single_head: bad shape B=%d N=%d", B, N);
  DS_REQUIRE(D == 128 || D == 512, "ds_attention_single_head: head width D=%d is not supported (128 or 512)", D);
  DS_REQUIRE(ld >= D && ld % 8 == 0, "ds_attention_single_head: row stride ld=%lld must be >= D and a multiple of 8",
             static_cast<long long>(ld));
  DS_REQUIRE(static_cast<int64_t>(N) * ld * 2 < (int64_t{1} << 40), "ds_attention_single_head: images too large");
  DS_REQUIRE(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
               reinterpret_cast<uintptr_t>(out)) & 15) == 0,
             "ds_attention_single_head: pointers must be 16-byte aligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return D == 512 ? launch_single_head<512>(q, k, v, out, B, N, ld, st)
                  : launch_single_head<128>(q, k, v, out, B, N, ld, st);
}
