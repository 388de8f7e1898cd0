// gemm_wgmma.cu — persistent, warp-specialised bf16 GEMM / implicit-GEMM conv3x3 for sm_90a.
//
//   out[M][Nout] = epilogue( A[M][K] * W[N][K]^T ),  fp32 accumulation in registers.
//
// One CTA per SM, persistent, 384 threads = 3 warpgroups; a CTA owns a 128 x BN output tile (BN = 256; 192 for
// N = 320; 128 for N <= 128), static round-robin over the tiles:
//   warpgroup 0     TMA producer : one lane streams A (128x64) and W (BN x 64) k-slices into a 4-6-stage shared-memory
//                                  ring (128-byte swizzle), arming a "full" mbarrier per stage
//   warpgroups 1-2  consumers    : each issues wgmma (M=64, N=BN, K=16) for its 64 rows of the tile and frees a stage
//                                  once the MMAs that read it have retired; then the epilogue runs from the
//                                  accumulator registers: bias / LayerNorm-on-A / row-bias / GEGLU / activation in
//                                  fp32, residual, one rounding; bf16 outputs are staged as 128-B-swizzled [128][64]
//                                  smem tiles and written with TMA stores (residual tiles arrive by TMA loads into the
//                                  same staging tile), so all epilogue global traffic is full-line and coalesced;
//                                  optional per-row (sum, sum of squares) of the outputs for the next LayerNorm and
//                                  per-channel statistics for the next GroupNorm.  The producer keeps filling the ring
//                                  while the epilogue runs, so the next tile's first k-blocks are resident by then.
// Split-K tail (big 3x3 convs): see GemmParams.  Programmatic dependent launch: the prologue (barriers, tensor map
// prefetch) runs while the previous kernel drains.
//
// conv3x3 mode (ds_conv3x3_nhwc): identical MMA pipeline; only the producer and the row->address map
// change.  An M tile is an 8x16 patch of output pixels of one image; for filter tap (r,s) and channel
// chunk c the A slice is the 4-D TMA box {64 ch, 16 px, 8 px, 1 img} of the NHWC input at pixel offset
// (r-1, s-1) — halo and zero padding come from TMA out-of-bounds fill, stride-2 from the tensor map's
// element strides.  K runs over (tap, channel): weights are packed [Cout][3][3][Cin].
//
// Reference arithmetic replaced: every nn.Linear / nn.Conv2d on the UNet sampling path
// (src/models/attention_processor.py:56-84,207-261; diffusers blocks reached from src/models/unet.py:190-338).
#include <cstdlib>
#include <functional>
#include <map>
#include <mutex>
#include <queue>
#include <vector>

#include "ds_common.cuh"
#include "ds_host.h"
#include "wgmma.cuh"

namespace ds {

constexpr int kBM = 128;
constexpr int kBK = 64;
constexpr int kGemmThreads = 384;  // 1 producer warpgroup + 2 consumer warpgroups
constexpr int kConsumers = 256;
constexpr int kABytes = kBM * kBK * 2;  // 16 KiB per stage
constexpr int kConvTileH = 8;
constexpr int kConvTileW = 16;
constexpr int kNarrowBN = 128;  // width of the narrow units of the mixed-width schedule (any BN > 128 instantiation)
constexpr int kMaxSmemPerBlock = 232448;  // sm_90 opt-in limit: 227 KiB

struct GemmParams {
  const float* bias;
  const float* rowbias;
  const __nv_bfloat16* residual;
  void* out;
  int M, N, K;
  int n_out;  // output columns (N, or N/2 for GEGLU)
  int ldo, ldres, rows_per_batch, ldrb;
  int epilogue, out_fp32;
  int tma_epilogue;  // 1: stage bf16 output tiles in smem and TMA-store them (residual tiles TMA-loaded)
  float out_scale;
  // LayerNorm fusion: consumer side (A rows are un-normalised; W/bias pre-folded) and producer side (row sums out)
  const double* ln_stats;  // [M][2] {sum, sum of squares} of A's rows (fp64), or NULL
  const float* ln_colsum;  // [N] sum_k W'[n][k]
  float ln_eps, ln_inv_k;
  double* row_stats_out;   // [M][2] fp64, accumulated with atomics (zeroed by the host wrapper), or NULL.  fp64 sums of
                           // the <= n-tiles fp32 partials of a row are exact: the result is order-independent
  double* zero_rows;       // [M][2] buffer whose rows this launch resets to 0 (the statistics buffer two hops ahead)
  int num_m_tiles, num_n_tiles, num_k_iters;
  // split-K tail: work items [0, tail_start) are whole 128 x BN units.  Each of the remaining `left` units (the
  // partial last wave of the persistent schedule) is cut along K into tail_parts slices that run on different CTAs;
  // every slice adds its fp32 accumulator into the unit's tile of `ws` (vector red.global.add), and the slice that
  // arrives last (per-unit counter) runs the normal epilogue from `ws` instead of its registers, clearing the tile and
  // the counter behind it.  tail_parts = 1: off.
  int tail_start, tail_parts, total_items;
  float* ws;  // [256 uint32 counters][left][128][BN] fp32, all zero between launches
  // Mixed-width schedule (BN = 256 instantiations only; see prepare_gemm): units [0, wide_units) are 256-column tiles
  // over the m-tiles [0, wide_m_tiles); the remaining units are HALF-width (128-column) tiles over the last m-tiles,
  // nt_narrow of them per m-tile — the m-rows of the under-filled last round of the persistent schedule are cut
  // into twice as many, half as long units instead of costing a whole round.  Off: wide_units >= all units.
  int wide_units, wide_m_tiles, nt_narrow;
  // last_narrow: the LAST n-tile of every m-tile is a 128-column unit instead of a (mostly padding) BN-wide one —
  // N = 640 runs as 256 | 256 | 128 and N = 320 as 192 | 128: no MMA work is spent on zero columns
  int last_narrow;
  // 1: the weight operand is constant data (never written by a kernel that may still be in flight), so the producer
  // may request its first tiles BEFORE griddepcontrol.wait.  0 (e.g. K / V^T of the VAE attention used as `w`): after.
  int w_const;
  // second A operand: k-blocks [k1_iters, num_k_iters) of a plain GEMM come from tmA2 (the channel concatenation
  // [a | a2] along K is never materialised); k1_iters == num_k_iters: off
  int k1_iters;
  // per-(sample, channel) {sum, sum of squares} of the bf16 OUTPUT, fp64 [B][n_out][2], accumulated with atomics:
  // the statistics the next GroupNorm needs, taken while the output tile still sits in shared memory
  double* chan_stats;
  int stats_rows_per_sample;  // GEMM mode: rows per sample (multiple of 128); conv mode: unused (tile = one image)
  // conv geometry
  int conv, stride, Ho, Wo, tiles_x, tiles_y, cin_chunks, conv_B;
  // filter-tap geometry: taps are enumerated row-major over a taps_x-wide window whose first tap sits at input offset
  // (off_x, off_y) from the output pixel: 3x3 / pad 1 = {3, -1, -1}; one phase of the fused nearest-x2-upsample conv =
  // {2, -1|0, -1|0}.  out_stride: the output patch is written to every out_stride-th pixel of the output tensor map
  // (2 for an upsample phase, whose map starts at that phase's first pixel).
  int taps_x, off_x, off_y, out_stride;
};

template <int BN>
struct GemmCfg {
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStageOutBytes = kBM * 64 * 2;      // one [128][64] bf16 epilogue staging tile
  static constexpr int kVecBytes = 2 * 2 * BN * 4;         // double-buffered per-tile copies of bias[BN] and ln_colsum[BN]
  static constexpr int kStatBytes = 8 * 64 * 2 * 4;        // channel statistics: [consumer warp][64 cols][2]
  static constexpr int kFixedBytes = kStageOutBytes + kVecBytes + kStatBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static constexpr int kFit = (kMaxSmemPerBlock - kFixedBytes) / kStageBytes;
  static constexpr int kStages = kFit > 8 ? 8 : kFit;
  static constexpr int kSmemBytes = kStages * kStageBytes + kFixedBytes;
  static_assert(kStages >= 3, "shared-memory ring too shallow");
};

// One launch = 1 problem (MAXQ = 1), or a CHAIN of up to kMaxChain dependent GEMMs over the same M rows (ds_gemm_chain):
// problem q+1 reads the output of problem q as its A operand.  The persistent CTAs walk the problems in order with
// their pipeline state (smem ring, barrier phases) carried across; a unit of problem q+1 on the 128-row block m waits —
// in the TMA producer, spinning on a global counter — until all n-tiles of problem q for that row block have been
// written (the epilogue bumps the counter after its stores have completed).  What this buys: one launch + prologue +
// drain instead of one per GEMM, and the CTAs that run out of problem-q units start on problem q+1 instead of idling
// through the partial last round.
constexpr int kMaxChain = 4;
template <int MAXQ>
struct GemmLaunch {
  CUtensorMap tm[MAXQ][6];  // per problem: A, B, C (output), R (residual), A2, B2 (narrow units)
  GemmParams p[MAXQ];
  int nq;
  int* dep;        // [nq][dep_stride] finished n-tiles per (problem, 128-row block), all zero at launch; NULL: nq == 1
  int dep_stride;
  // chain schedule (host-built, see chain_schedule): for CTA g, the items of problem q are
  // sched[sched_items + i] for i in [sched[g * (kMaxChain + 1) + q], sched[g * (kMaxChain + 1) + q + 1])
  const int* sched;
  int sched_items;
};

__device__ __forceinline__ int ld_acquire_gpu(const int* ptr) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(ptr) : "memory");
  return v;
}

// Register budgets after setmaxnreg (the launch gives every thread 168): the producer warpgroup needs a handful for
// one lane's TMA loop, the consumers hold a 64 x 256 fp32 accumulator (128 registers) beside the epilogue state.
// 128 * 40 + 256 * 232 = 64512 <= 65536.
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;

template <int W>
__device__ __forceinline__ void wgmma_tile(float* acc, uint64_t adesc, uint64_t bdesc, int scale_d) {
  if constexpr (W == 256)
    wgmma_m64n256_ss(acc, adesc, bdesc, scale_d);
  else if constexpr (W == 192)
    wgmma_m64n192_ss(acc, adesc, bdesc, scale_d);
  else
    wgmma_m64n128_ss(acc, adesc, bdesc, scale_d);
}

// One item's main loop, 4 x wgmma (64 x W x 16) per 64-wide k-block; kb + 1 is issued before the MMAs of kb are
// waited for, and kb's stage is freed once they retired.  `narrow` (CTA-uniform) runs a 128-column unit of a wider
// tile; callers that never have one pass a constant false, so their kernel has only the W-wide wgmma (the chain: a
// data-dependent wgmma shape there made ptxas serialise its MMAs).
template <int W, int STAGES, int BBYTES>
__device__ __forceinline__ void mma_mainloop(float* acc, uint32_t a_base, uint32_t b_base, uint64_t* full_bar,
                                             uint64_t* empty_bar, int& stage, uint32_t& phase, int k0, int k1,
                                             bool narrow) {
  int prev = -1;
  for (int kb = k0; kb < k1; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t a_addr = a_base + stage * kABytes;
    const uint32_t b_addr = b_base + stage * BBYTES;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k)
      if (W > kNarrowBN && narrow)
        wgmma_tile<kNarrowBN>(acc, make_wgmma_desc(a_addr + k * 32, 1024, 16),
                              make_wgmma_desc(b_addr + k * 32, 1024, 16), (kb != k0 || k != 0) ? 1 : 0);
      else
        wgmma_tile<W>(acc, make_wgmma_desc(a_addr + k * 32, 1024, 16), make_wgmma_desc(b_addr + k * 32, 1024, 16),
                      (kb != k0 || k != 0) ? 1 : 0);
    wgmma_commit();
    wgmma_wait<1>();  // the previous k-block's MMAs have retired: its stage may be refilled
    if (prev >= 0) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
  fence_regs<W / 2>(acc);
  if (prev >= 0) mbar_arrive(&empty_bar[prev]);
}

// item -> (unit, k-block range [k0, k1), index of the unit among the tail units or -1)
__device__ __forceinline__ void decode_item(const GemmParams& p, int item, int& unit, int& k0, int& k1, int& tail_idx) {
  if (item < p.tail_start) {
    unit = item;
    k0 = 0;
    k1 = p.num_k_iters;
    tail_idx = -1;
  } else {
    const int s = item - p.tail_start;
    tail_idx = s / p.tail_parts;
    const int part = s - tail_idx * p.tail_parts;
    unit = p.tail_start + tail_idx;
    k0 = part * p.num_k_iters / p.tail_parts;
    k1 = (part + 1) * p.num_k_iters / p.tail_parts;
  }
}

// unit -> (m-tile, first weight row of its columns, tile width)
template <int BN>
__device__ __forceinline__ void unit_geom(const GemmParams& p, int unit, int& m_tile, int& n_org, int& bn) {
  if (unit < p.wide_units) {
    m_tile = unit / p.num_n_tiles;
    const int k = unit - m_tile * p.num_n_tiles;
    n_org = k * BN;
    bn = (p.last_narrow && k == p.num_n_tiles - 1) ? kNarrowBN : BN;
  } else {
    const int j = unit - p.wide_units;
    const int mt = j / p.nt_narrow;
    m_tile = p.wide_m_tiles + mt;
    n_org = (j - mt * p.nt_narrow) * kNarrowBN;
    bn = kNarrowBN;
  }
}

// this CTA's items of problem q: round-robin over the grid, or — chain — its row of the host-built schedule
// (item i of [beg, end) is sched_items[i] then)
template <int MAXQ>
__device__ __forceinline__ void item_range(const GemmLaunch<MAXQ>& L, int q, int& beg, int& end, int& step,
                                           const int*& sched_items) {
  beg = blockIdx.x;
  end = L.p[q].total_items;
  step = gridDim.x;
  sched_items = nullptr;
  if (MAXQ > 1) {
    const int* hdr = L.sched + blockIdx.x * (kMaxChain + 1);
    beg = __ldg(hdr + q);
    end = __ldg(hdr + q + 1);
    step = 1;
    sched_items = L.sched + L.sched_items;
  }
}

template <int BN, bool STATS, int MAXQ>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_wgmma(const __grid_constant__ GemmLaunch<MAXQ> L) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::kStages;
  constexpr int ACC = BN / 2;  // fp32 accumulator registers per consumer thread (64 rows x BN per warpgroup)
  const int unit0 = blockIdx.x;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * kABytes;
  uint8_t* sOut = sB + STAGES * Cfg::kBBytes;  // [128][64] bf16, 128-B swizzled (TMA store / residual load)
  float* sVec = reinterpret_cast<float*>(sOut + Cfg::kStageOutBytes);  // [2 tiles in flight][bias | colsum][BN]
  float* sStat = reinterpret_cast<float*>(sOut + Cfg::kStageOutBytes + Cfg::kVecBytes);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sOut + Cfg::kStageOutBytes + Cfg::kVecBytes + Cfg::kStatBytes);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* res_bar = empty_bar + STAGES;  // residual tile landed
  volatile uint32_t* s_flag = reinterpret_cast<uint32_t*>(res_bar + 1);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    for (int q = 0; q < (MAXQ == 1 ? 1 : L.nq); ++q) {
      const GemmParams& pq = L.p[q];
      tma_prefetch_desc(&L.tm[q][0]);
      tma_prefetch_desc(&L.tm[q][1]);
      if (pq.tma_epilogue) {
        tma_prefetch_desc(&L.tm[q][2]);
        if (pq.residual) tma_prefetch_desc(&L.tm[q][3]);
      }
      if (pq.k1_iters < pq.num_k_iters) tma_prefetch_desc(&L.tm[q][4]);
      if (pq.nt_narrow > 0 || pq.last_narrow) tma_prefetch_desc(&L.tm[q][5]);
    }
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kConsumers);  // every consumer thread arrives once its warpgroup's MMAs retired
    }
    mbar_init(res_bar, 1);
    fence_mbar_init();
  }
  pdl_launch_dependents();  // the next kernel may start its prologue on SMs this grid has already left
  __syncthreads();
  // Everything above overlapped the previous kernel's tail; from here on we touch its outputs.  The TMA producer lane
  // may wait later: it first requests the WEIGHT tiles of its first pipeline stages when they are constant data.
  const bool is_producer_lane = (warp == 0) && (lane == 0);
  const int nq = MAXQ == 1 ? 1 : L.nq;

  // Each role walks all problems of the chain inside its own branch, so that the register budget set by setmaxnreg at
  // the head of the branch holds for all of the role's code.  The pipeline state (ring slot, barrier phases) carries
  // from one problem to the next.
  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer (warpgroup 0, one lane)
    setmaxnreg_dec<kProducerRegs>();
    if (!is_producer_lane) pdl_wait();
    if (is_producer_lane) {
      int stage = 0;
      uint32_t phase = 0;
      for (int q = 0; q < nq; ++q) {
      const GemmParams& p = L.p[q];
      const CUtensorMap& tmA = L.tm[q][0];
      const CUtensorMap& tmB = L.tm[q][1];
      const CUtensorMap& tmA2 = L.tm[q][4];
      const CUtensorMap& tmB2 = L.tm[q][5];
      int it_beg, it_end, it_step;
      const int* sched_items;
      item_range(L, q, it_beg, it_end, it_step, sched_items);
      // chain dependency: the A rows of row block m_blk are the output rows of ALL n-tiles of the previous problem
      auto wait_chain_dep = [&](int m_blk) {
        const int* cnt = L.dep + (q - 1) * L.dep_stride + m_blk;
        const int need = L.p[q - 1].num_n_tiles;
        if (ld_acquire_gpu(cnt) < need) {
          const long long t0 = clock64();
          while (ld_acquire_gpu(cnt) < need) {
            if (clock64() - t0 > 4000000000LL) __trap();  // a protocol bug becomes a launch error, not a hang
          }
        }
        asm volatile("fence.proxy.async;" ::: "memory");  // generic-proxy acquire -> async-proxy (TMA) reads
      };
      int pre_b = 0;  // k-blocks of the FIRST item whose weight tile was requested before griddepcontrol.wait
      if (MAXQ == 1 && p.w_const && unit0 < p.total_items) {
        int unit, k0, k1, tail_idx, m_tile, n_org, bn;
        decode_item(p, unit0, unit, k0, k1, tail_idx);
        unit_geom<BN>(p, unit, m_tile, n_org, bn);
        const CUtensorMap* bm = (bn != BN) ? &tmB2 : &tmB;
        pre_b = (k1 - k0) < STAGES ? (k1 - k0) : STAGES;
        for (int i = 0; i < pre_b; ++i)  // stage i, first pass: the slot is free, its barrier is in phase 0
          tma_load_2d(sB + i * Cfg::kBBytes, bm, &full_bar[i], (k0 + i) * kBK, n_org);
      }
      if (q == 0) pdl_wait();
      for (int it = it_beg; it < it_end; it += it_step) {
        const int tile = MAXQ > 1 ? __ldg(sched_items + it) : it;
        int unit, k0, k1, tail_idx;
        decode_item(p, tile, unit, k0, k1, tail_idx);
        int m_blk, n_org, bn;
        unit_geom<BN>(p, unit, m_blk, n_org, bn);
        const bool narrow = bn != BN;
        if (MAXQ > 1 && q > 0 && L.dep != nullptr) wait_chain_dep(m_blk);
        const uint32_t stage_bytes = kABytes + bn * kBK * 2;
        int img = 0, x0 = 0, y0 = 0;
        if (p.conv) {
          const int per_img = p.tiles_x * p.tiles_y;
          img = m_blk / per_img;
          const int rem = m_blk - img * per_img;
          y0 = (rem / p.tiles_x) * kConvTileH;
          x0 = (rem % p.tiles_x) * kConvTileW;
        }
        const CUtensorMap* bm = narrow ? &tmB2 : &tmB;
        for (int kb = k0; kb < k1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], stage_bytes);
          if (p.conv) {
            const int tap = kb / p.cin_chunks;
            const int cc = kb - tap * p.cin_chunks;
            const int r = tap / p.taps_x, s = tap - r * p.taps_x;
            tma_load_4d(sA + stage * kABytes, &tmA, &full_bar[stage], cc * kBK, x0 * p.stride + s + p.off_x,
                        y0 * p.stride + r + p.off_y, img);
          } else {
            const bool second = kb >= p.k1_iters;  // [a | a2] along K
            const CUtensorMap* am = second ? &tmA2 : &tmA;
            const int kc = (second ? kb - p.k1_iters : kb) * kBK;
            tma_load_2d(sA + stage * kABytes, am, &full_bar[stage], kc, m_blk * kBM);
          }
          if (MAXQ == 1 && tile == unit0 && kb - k0 < pre_b) {
            // weight tile already in flight (requested before griddepcontrol.wait); its bytes count towards the
            // expect_tx above — complete_tx may precede expect_tx within a phase (the tx-count is signed)
          } else {
            tma_load_2d(sB + stage * Cfg::kBBytes, bm, &full_bar[stage], kb * kBK, n_org);
          }
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
      }  // problems of the chain
    }
  } else {
    // ------------------------------------------------------------------ consumers (warpgroups 1-2): MMA + epilogue
    setmaxnreg_inc<kConsumerRegs>();
    pdl_wait();
    const int ct = threadIdx.x - 128;     // consumer thread 0..255
    const int wg = ct >> 7;               // consumer warpgroup: rows [64 wg, +64) of the tile
    const int cw = ct >> 5;               // consumer warp 0..7: rows [16 cw, +16)
    const int cq = 2 * (lane & 3);        // first of the two columns this thread holds in every 8-column block
    int r_loc[2];                         // the two tile rows this thread holds
    r_loc[0] = cw * 16 + (lane >> 2);
    r_loc[1] = r_loc[0] + 8;
    const bool issuer = ct == 0;          // drives the TMA engine for the epilogue
    const uint32_t a_base = smem_u32(sA) + static_cast<uint32_t>(wg) * 64 * 128;  // this warpgroup's 64 A rows
    const uint32_t b_base = smem_u32(sB);
    float acc[ACC];

    int stage = 0, iter = 0;
    uint32_t phase = 0, res_phase = 0;
    for (int q = 0; q < nq; ++q) {
    const GemmParams& p = L.p[q];
    const CUtensorMap& tmC = L.tm[q][2];
    const CUtensorMap& tmR = L.tm[q][3];
    int it_beg, it_end, it_step;
    const int* sched_items;
    item_range(L, q, it_beg, it_end, it_step, sched_items);
    const bool geglu = p.epilogue == DS_EPI_GEGLU;
    // chain: "this n-tile of row block m is written" is published one tile LATE: after the main loop of the CTA's
    // next tile (or at the end of the problem).  By then the tile's bulk stores have long completed (the wait is
    // free), and every consumer is past its trailing statistics atomics (the barrier at the head of the next tile).
    // A consumer needs num_n_tiles signals per row block.
    const bool chain_sig = MAXQ > 1 && L.dep != nullptr && q + 1 < nq;
    int pend_blk = -1;  // row block whose signal is pending (CTA-uniform)
    auto post_signal = [&]() {  // issuer thread, after a barrier of the consumers
      asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // the bulk stores have been WRITTEN
      asm volatile("fence.proxy.async;" ::: "memory");
      asm volatile("red.release.gpu.global.add.s32 [%0], 1;" ::"l"(L.dep + q * L.dep_stride + pend_blk) : "memory");
    };
    for (int it = it_beg; it < it_end; it += it_step, ++iter) {
      const int tile = MAXQ > 1 ? __ldg(sched_items + it) : it;
      int unit, k0, k1, tail_idx;
      decode_item(p, tile, unit, k0, k1, tail_idx);
      int m_blk, n_org, bn_cur;  // n_org: first weight row of the tile's columns; bn_cur: BN, or 128 (narrow unit)
      unit_geom<BN>(p, unit, m_blk, n_org, bn_cur);
      const int bn_out = geglu ? bn_cur / 2 : bn_cur;  // output columns of this item
      const int no_org = geglu ? n_org / 2 : n_org;    // first output column

      // row -> (valid, output row index, batch index)
      bool row_ok[2];
      long long orow[2];
      int batch[2];
      int cx = 0, cy = 0, cimg = 0;  // conv: tile origin in the output tensor map
      if (p.conv) {
        const int per_img = p.tiles_x * p.tiles_y;
        cimg = m_blk / per_img;
        const int rem = m_blk - cimg * per_img;
        cy = (rem / p.tiles_x) * kConvTileH;
        cx = (rem % p.tiles_x) * kConvTileW;
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (p.conv) {
          const int y = cy + r_loc[h] / kConvTileW;
          const int x = cx + r_loc[h] % kConvTileW;
          row_ok[h] = (y < p.Ho) && (x < p.Wo) && (cimg < p.conv_B);
          orow[h] = (static_cast<long long>(cimg) * p.Ho + y) * p.Wo + x;
          batch[h] = cimg;
        } else {
          const int row = m_blk * kBM + r_loc[h];
          row_ok[h] = row < p.M;
          orow[h] = row;
          batch[h] = p.rowbias ? row / p.rows_per_batch : 0;
        }
      }

      // Per-tile column vectors -> shared memory (double-buffered by iteration parity), read back as broadcasts:
      //   vec[0..BN)    = bias[n] (+ the time-embedding row bias of this tile's image in conv mode), 0 beyond N
      //   vec[BN..2BN)  = ln_colsum[n]
      float* vec = sVec + (iter & 1) * 2 * BN;
      {
        const float* rb_row = nullptr;  // conv: every row of the tile belongs to one image
        if (p.conv && p.rowbias && cimg < p.conv_B) rb_row = p.rowbias + static_cast<long long>(cimg) * p.ldrb;
        for (int i = ct; i < bn_cur; i += kConsumers) {
          const int nn = n_org + i;
          float b = 0.f, c = 0.f;
          if (nn < p.N) {
            if (p.bias) b = __ldg(p.bias + nn);
            if (rb_row) b += __ldg(rb_row + nn);
            if (p.ln_stats) c = __ldg(p.ln_colsum + nn);
          }
          vec[i] = b;
          vec[BN + i] = c;
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
      const bool gemm_rowbias = p.rowbias && !p.conv;  // GEMM mode: rows of a tile may belong to different samples

      // LayerNorm-on-A: v = rstd * (acc - mean * colsum[n]) (+ folded bias); statistics of this thread's rows
      float ln_mean[2] = {0.f, 0.f}, ln_rstd[2] = {1.f, 1.f};
      auto row_stats_io = [&]() {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (p.ln_stats && row_ok[h]) {
            // chain: the statistics were written by an earlier problem of THIS launch -> no read-only (nc) path
            const double2 st = MAXQ > 1 ? __ldcg(reinterpret_cast<const double2*>(p.ln_stats) + orow[h])
                                        : __ldg(reinterpret_cast<const double2*>(p.ln_stats) + orow[h]);
            const double dmean = st.x * static_cast<double>(p.ln_inv_k);
            ln_mean[h] = static_cast<float>(dmean);
            const float var = fmaxf(static_cast<float>(st.y * static_cast<double>(p.ln_inv_k) - dmean * dmean), 0.f);
            ln_rstd[h] = rsqrtf(var + p.ln_eps);
          }
          if (p.zero_rows && n_org == 0 && (lane & 3) == 0 && row_ok[h])
            *reinterpret_cast<double2*>(p.zero_rows + 2 * orow[h]) = make_double2(0.0, 0.0);
        }
      };
      // One problem per launch: ahead of the main loop, so the load's latency hides behind the MMAs.  Chain: the
      // statistics (and the buffer to clear) belong to earlier problems of this launch — only touch them once the
      // tile's operands have arrived, i.e. after the producer saw the row block's dependency counter complete.
      if (MAXQ == 1) row_stats_io();

      // ---------------- main loop.  Narrow (128-column) units only exist in single-problem launches of the wider
      // tiles (last_narrow, mixed-width tail): prepare_gemm sets neither for a chain link, so the chain kernel has only
      // the BN-wide loop.
      mma_mainloop<BN, STAGES, Cfg::kBBytes>(acc, a_base, b_base, full_bar, empty_bar, stage, phase, k0, k1,
                                             MAXQ == 1 && bn_cur != BN);
      if (MAXQ > 1) row_stats_io();
      if (chain_sig && pend_blk >= 0) {  // the previous item: see post_signal
        if (issuer) post_signal();
        pend_blk = -1;
      }

      // ---- split-K tail: add this K-slice's accumulator into the unit's workspace tile; only the last slice to
      // arrive goes on to the epilogue proper, reading the sums back from the workspace
      if (tail_idx >= 0) {
        float* ws_t = p.ws + 256 + static_cast<size_t>(tail_idx) * kBM * BN;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          if (j * 8 >= bn_cur) continue;
#pragma unroll
          for (int h = 0; h < 2; ++h)
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(ws_t + r_loc[h] * BN + j * 8 + cq),
                         "f"(acc[4 * j + 2 * h]), "f"(acc[4 * j + 2 * h + 1])
                         : "memory");
        }
        __threadfence();  // this thread's reductions are performed before the arrival below becomes visible
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (issuer) {
          unsigned int* cnt = reinterpret_cast<unsigned int*>(p.ws) + tail_idx;
          const unsigned int old = atomicAdd(cnt, 1u);
          const bool last = old == static_cast<unsigned int>(p.tail_parts - 1);
          if (last) *cnt = 0u;  // every slice has arrived: leave the counter clean for the next launch
          *s_flag = last ? 1u : 0u;
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (*s_flag == 0u) continue;  // CTA-uniform
        __threadfence();
        // sums of all K-slices; clear behind us so the workspace is zero again for the next launch
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          if (j * 8 >= bn_cur) continue;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float2* wp = reinterpret_cast<float2*>(ws_t + r_loc[h] * BN + j * 8 + cq);
            const float2 f = __ldcg(wp);
            acc[4 * j + 2 * h] = f.x;
            acc[4 * j + 2 * h + 1] = f.y;
            __stcg(wp, make_float2(0.f, 0.f));
          }
        }
      }

      // accumulator -> fp32 values with LayerNorm / bias / row-bias / GEGLU / activation applied (no residual yet).
      // The GEGLU pass is a loop of its own: in one loop with the other epilogues, the value | gate pairs of every
      // column block stay live across all branches and the accumulator no longer fits the register budget.
      auto ln_bias = [&](float& v0, float& v1, int h, int c) {  // tile column c (value or gate)
        if (p.ln_stats) {
          const float nm = -ln_mean[h] * ln_rstd[h];
          v0 = fmaf(v0, ln_rstd[h], nm * vec[BN + c]);
          v1 = fmaf(v1, ln_rstd[h], nm * vec[BN + c + 1]);
        }
        v0 += vec[c];
        v1 += vec[c + 1];
      };
      auto add_rowbias = [&](float& v0, float& v1, int h, int c) {
        if (gemm_rowbias && row_ok[h]) {
          const float* rb = p.rowbias + static_cast<long long>(batch[h]) * p.ldrb + n_org + c;
          if (n_org + c < p.N) v0 += __ldg(rb);
          if (n_org + c + 1 < p.N) v1 += __ldg(rb + 1);
        }
      };
      if (geglu) {
        // value columns [0, bn/2) of the tile, gates [bn/2, bn) — the same thread holds both.  GEGLU only runs on
        // 256-column tiles (prepare_gemm refuses anything else), so narrower instantiations leave this pass out.
        if constexpr (BN >= 256) {
          constexpr int G = BN / 16;  // first gate block
#pragma unroll
          for (int j = 0; j < BN / 16; ++j) {
            if (j * 8 >= bn_out) continue;
            const int c = j * 8 + cq;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
              ln_bias(v0, v1, h, c);
              add_rowbias(v0, v1, h, c);
              float g0 = acc[4 * (j + G) + 2 * h], g1 = acc[4 * (j + G) + 2 * h + 1];
              ln_bias(g0, g1, h, BN / 2 + c);
              acc[4 * j + 2 * h] = v0 * gelu_sig5(g0);
              acc[4 * j + 2 * h + 1] = v1 * gelu_sig5(g1);
            }
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          if (j * 8 >= bn_out) continue;
          const int c = j * 8 + cq;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
            ln_bias(v0, v1, h, c);
            add_rowbias(v0, v1, h, c);
            if (p.epilogue == DS_EPI_GELU) {
              v0 = gelu_sig5(v0);
              v1 = gelu_sig5(v1);
            } else if (p.epilogue == DS_EPI_SILU) {
              v0 = silu_f(v0);
              v1 = silu_f(v1);
            } else if (p.epilogue == DS_EPI_QUICKGELU) {  // CLIP "quick_gelu": x * sigmoid(1.702 x)
              v0 = __fdividef(v0, 1.0f + __expf(-1.702f * v0));
              v1 = __fdividef(v1, 1.0f + __expf(-1.702f * v1));
            }
            acc[4 * j + 2 * h] = v0;
            acc[4 * j + 2 * h + 1] = v1;
          }
        }
      }

      if (p.tma_epilogue) {
        // ---------------- coalesced path: 64-column blocks staged in swizzled smem, moved by TMA
        float rs_sum[2] = {0.f, 0.f}, rs_sq[2] = {0.f, 0.f};  // producer side: this thread's share of its rows' sums
#pragma unroll
        for (int cbi = 0; cbi < BN / 64; ++cbi) {
          const int no0 = no_org + cbi * 64;  // first output column of this 64-wide block
          if (cbi * 64 >= bn_out || no0 >= p.n_out) break;  // CTA-uniform
          // the previous TMA store must have finished READING the staging tile before anyone overwrites it
          if (issuer) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
          asm volatile("bar.sync 1, 256;" ::: "memory");
          if (p.residual) {
            if (issuer) {
              mbar_arrive_expect_tx(res_bar, kBM * 64 * 2);
              if (p.conv)
                tma_load_4d(sOut, &tmR, res_bar, no0, cx, cy, cimg);
              else
                tma_load_2d(sOut, &tmR, res_bar, no0, m_blk * kBM);
            }
            mbar_wait(res_bar, res_phase);
            res_phase ^= 1;
          }
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = cbi * 8 + jj;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = r_loc[h];
              const uint32_t sp = smem_u32(sOut) + r * 128 + ((jj ^ (r & 7)) << 4) + cq * 2;
              float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
              if (p.residual) {
                uint32_t u;
                asm volatile("ld.shared.b32 %0, [%1];" : "=r"(u) : "r"(sp));
                v0 += bf16_lo(u);
                v1 += bf16_hi(u);
              }
              if (p.out_scale != 0.0f) {
                v0 *= p.out_scale;
                v1 *= p.out_scale;
              }
              if (p.row_stats_out) {  // statistics for the next LayerNorm, from the fp32 values (the bf16 rounding
                                      // of 1e3 row elements is unbiased: it moves mean / rstd by < 1e-4 relative)
                rs_sum[h] += v0;
                rs_sum[h] += v1;
                rs_sq[h] = fmaf(v0, v0, rs_sq[h]);
                rs_sq[h] = fmaf(v1, v1, rs_sq[h]);
              }
              asm volatile("st.shared.b32 [%0], %1;" ::"r"(sp), "r"(pack_bf16(v0, v1)) : "memory");
            }
          }
          fence_proxy_async_smem();  // st.shared -> visible to the TMA (async proxy)
          asm volatile("bar.sync 1, 256;" ::: "memory");
          if (issuer) {
            if (p.conv)
              asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                               &tmC),
                           "r"(smem_u32(sOut)), "r"(no0), "r"(cx * p.out_stride), "r"(cy * p.out_stride), "r"(cimg)
                           : "memory");
            else
              asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(&tmC),
                           "r"(smem_u32(sOut)), "r"(no0), "r"(m_blk * kBM)
                           : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
          }
          if (STATS && p.chan_stats) {
            // Channel statistics of the staged [128 rows][64 cols] bf16 block (exactly the values the next GroupNorm
            // will read), while the TMA store drains it: warp cw reads rows [16 cw, +16), lane <-> column pair; a
            // warp reads 128 contiguous (swizzled) bytes of one row per step — conflict-free.  Rows outside the
            // tensor (partial conv patches, M tail) are masked.  The 8 warps' partials are combined in a fixed order
            // and each column adds ONE fp64 pair per (tile, column) to global memory: fp64 sums of <= 2^11 fp32
            // partials are exact, so the result does not depend on the arrival order.
            uint32_t vmask;
            int sbatch;
            if (p.conv) {  // rows [16 cw, +16) are pixel row cy + cw of the patch
              uint32_t mx = 0;
#pragma unroll
              for (int i = 0; i < kConvTileW; ++i) mx |= (cx + i < p.Wo) ? (1u << i) : 0u;
              vmask = (cy + cw < p.Ho && cimg < p.conv_B) ? mx : 0u;
              sbatch = cimg;
            } else {
              const int nv = p.M - (m_blk * kBM + cw * 16);
              vmask = nv >= 16 ? 0xffffu : (nv <= 0 ? 0u : ((1u << nv) - 1u));
              sbatch = (m_blk * kBM) / p.stats_rows_per_sample;
            }
            float s0 = 0.f, q0 = 0.f, s1 = 0.f, q1 = 0.f;
            const uint32_t sbase = smem_u32(sOut) + (cw * 16) * 128 + (lane & 3) * 4;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const int r = cw * 16 + i;
              uint32_t wv;
              asm volatile("ld.shared.b32 %0, [%1];" : "=r"(wv) : "r"(sbase + i * 128 + (((lane >> 2) ^ (r & 7)) << 4)));
              if (!((vmask >> i) & 1u)) wv = 0u;
              const float a = bf16_lo(wv), c = bf16_hi(wv);
              s0 += a;
              q0 = fmaf(a, a, q0);
              s1 += c;
              q1 = fmaf(c, c, q1);
            }
            // lane read columns 8 (lane / 4) + 2 (lane % 4) + {0, 1} = 2 lane + {0, 1}: [col][2] entries
            *reinterpret_cast<float4*>(sStat + cw * 128 + lane * 4) = make_float4(s0, q0, s1, q1);
            asm volatile("bar.sync 1, 256;" ::: "memory");
            const bool tile_ok = p.conv ? (cimg < p.conv_B) : (m_blk * kBM < p.M);
            if (ct < 64 && tile_ok && no0 + ct < p.n_out) {
              const float* sc = sStat + ct * 2;
              float ts = 0.f, tq = 0.f;
#pragma unroll
              for (int w = 0; w < 8; ++w) {
                ts += sc[w * 128];
                tq += sc[w * 128 + 1];
              }
              double* gp = p.chan_stats + (static_cast<size_t>(sbatch) * p.n_out + (no0 + ct)) * 2;
              atomicAdd(gp, static_cast<double>(ts));
              atomicAdd(gp + 1, static_cast<double>(tq));
            }
          }
        }
        if (p.row_stats_out) {  // columns beyond N contributed exact zeros; a row's 4 column-sharing threads combine
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float s = rs_sum[h], sq = rs_sq[h];
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            sq += __shfl_xor_sync(0xffffffffu, sq, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            sq += __shfl_xor_sync(0xffffffffu, sq, 2);
            if ((lane & 3) == 0 && row_ok[h]) {
              atomicAdd(p.row_stats_out + 2 * orow[h], static_cast<double>(s));
              atomicAdd(p.row_stats_out + 2 * orow[h] + 1, static_cast<double>(sq));
            }
          }
        }
        if (chain_sig) pend_blk = m_blk;
        continue;
      }

      // ---------------- direct path (fp32 output or rows that are not 16-byte addressable): per-thread stores
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        if (j * 8 >= bn_out) continue;
        const int no = no_org + j * 8 + cq;  // output column of this thread's first element in the block
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!row_ok[h]) continue;
          float v[2] = {acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]};
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (no + e >= p.n_out) continue;
            if (p.residual) v[e] += __bfloat162float(p.residual[orow[h] * p.ldres + no + e]);
            if (p.out_scale != 0.0f) v[e] *= p.out_scale;
            if (p.out_fp32)
              reinterpret_cast<float*>(p.out)[orow[h] * p.ldo + no + e] = v[e];
            else
              reinterpret_cast<__nv_bfloat16*>(p.out)[orow[h] * p.ldo + no + e] = __float2bfloat16(v[e]);
          }
        }
      }
    }
    if (chain_sig && pend_blk >= 0) {  // the last item of this problem
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (issuer) post_signal();
    }
    // the staging tile must outlive the store's READ of it; global visibility of the bulk stores is the grid's
    // completion (what griddepcontrol.wait / stream order of the consumer waits for)
    if (p.tma_epilogue && issuer) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    }  // problems of the chain
  }

  // ---------------------------------------------------------------------- teardown
  __syncthreads();
  if (MAXQ > 1 && L.dep != nullptr && warp == 0) {
    // the last CTA to get here (every CTA's dependency reads are behind it) hands the counters back zeroed, so the
    // same buffer serves the next chain launch — and every replay of a captured graph — without a memset node
    int* ticket = L.dep + kMaxChain * L.dep_stride;
    int last = 0;
    if (lane == 0) {
      __threadfence();
      last = atomicAdd(ticket, 1) == static_cast<int>(gridDim.x) - 1;
    }
    last = __shfl_sync(0xffffffffu, last, 0);
    if (last) {
      for (int i = lane; i < (nq - 1) * L.dep_stride; i += 32) L.dep[i] = 0;
      if (lane == 0) *ticket = 0;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// One prepared problem: tensor maps {A, B, C, R, A2, B2}, parameters and the tile shape run_gemm chose for it.
struct PreparedGemm {
  CUtensorMap tm[6];
  GemmParams p;
  int bn;
};

// Launches gemm_bf16_wgmma<BN, STATS, MAXQ> on `groups` CTAs with programmatic dependent launch.  The schedule is
// persistent with a static stride, so every CTA must be resident: callers pass at most one CTA per SM.  The dynamic
// shared-memory opt-in is set once per device for each instantiation.
template <int BN, bool STATS, int MAXQ>
static int launch_wgmma(const GemmLaunch<MAXQ>& L, int groups, cudaStream_t stream, const char* name) {
  const int slot = device_slot();
  static bool attr_set[kMaxDevices] = {};  // per device; benign race: idempotent
  if (!attr_set[slot]) {
    DS_CUDA_OK(cudaFuncSetAttribute(gemm_bf16_wgmma<BN, STATS, MAXQ>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    GemmCfg<BN>::kSmemBytes));
    attr_set[slot] = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(groups);
  cfg.blockDim = dim3(kGemmThreads);
  cfg.dynamicSmemBytes = GemmCfg<BN>::kSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  pdl_attr(&attr[0]);
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  DS_CUDA_OK(cudaLaunchKernelEx(&cfg, gemm_bf16_wgmma<BN, STATS, MAXQ>, L));
  DS_LAUNCH_OK(name);
  return DS_OK;
}

template <int BN, bool STATS>
static int launch_gemm_t(const PreparedGemm& g, int num_sms, cudaStream_t stream, void* splitk_ws,
                         long long splitk_ws_bytes) {
  GemmParams p = g.p;
  const int m_groups = p.num_m_tiles;
  const bool mixed = p.nt_narrow > 0;  // run_gemm chose the mixed-width tail (BN == 256 only)
  if (!mixed) {
    p.wide_units = m_groups * p.num_n_tiles;
    p.wide_m_tiles = m_groups;
    p.nt_narrow = 0;
  }
  const int units = mixed ? p.wide_units + (m_groups - p.wide_m_tiles) * p.nt_narrow : m_groups * p.num_n_tiles;
  const int groups = units < num_sms ? units : num_sms;
  // split-K tail (see GemmParams): the units of the partial last wave are cut along K so that every CTA gets a slice.
  // Needs the bf16 TMA epilogue, no GEGLU (its accumulator pairs value | gate columns) and a caller-provided zeroed
  // workspace.  The fp32 reductions through the L2 and the second epilogue pass cost a fixed amount per launch, so it
  // only pays when one unit's main loop is much longer than that (the big 3x3 convs), and the fp32 atomics make those
  // outputs non-reproducible at the last ulp: the feature is OPT-IN, DS_GEMM_SPLITK = minimum k-blocks per unit
  // (e.g. 128); unset / 0 = off.  The native harness (and its pytest wrapper) exercise it.
  static const int splitk_env = [] {
    const char* e = getenv("DS_GEMM_SPLITK");
    return e ? atoi(e) : 0;
  }();
  p.tail_start = units;
  p.tail_parts = 1;
  p.total_items = units;
  p.ws = nullptr;
  if (splitk_env > 0 && !mixed && p.num_k_iters >= splitk_env && splitk_ws && p.tma_epilogue &&
      p.epilogue != DS_EPI_GEGLU && units > groups) {
    const int full = (units / groups) * groups, left = units - full;
    if (left > 0 && left <= 128) {
      int parts = groups / left;
      if (parts > 8) parts = 8;
      if (parts > p.num_k_iters / 2) parts = p.num_k_iters / 2;
      const long long need = 1024 + static_cast<long long>(left) * kBM * BN * 4;
      if (parts >= 2 && need <= splitk_ws_bytes && (reinterpret_cast<uintptr_t>(splitk_ws) & 15) == 0) {
        p.tail_start = full;
        p.tail_parts = parts;
        p.total_items = full + left * parts;
        p.ws = static_cast<float*>(splitk_ws);
      }
    }
  }
  GemmLaunch<1> L;
  for (int i = 0; i < 6; ++i) L.tm[0][i] = g.tm[i];
  L.p[0] = p;
  L.nq = 1;
  L.dep = nullptr;
  L.dep_stride = 0;
  L.sched = nullptr;
  L.sched_items = 0;
  return launch_wgmma<BN, STATS, 1>(L, groups, stream, "gemm_bf16_wgmma");
}

// Static schedule of a chain: which CTA runs which units, in which order.  Round-robin per problem (what a single
// launch does) leaves every problem's partial last round on the same low-numbered CTAs; here the units of ALL
// problems, in (problem, unit) order, go through list scheduling — each unit to the CTA that becomes free first under
// the cost model "k-blocks + alpha" — which is what a dynamic tile scheduler would do, without a per-tile atomic and a
// broadcast in the kernel.  Dependencies only point to earlier problems and every CTA walks the problems
// in order, so any assignment is deadlock-free.  The table depends only on (CTAs, per-problem units, k-blocks): it is
// built once per distinct chain shape and kept in device memory (first use must be outside a graph capture).
struct ChainSchedule {
  int* dev = nullptr;
  int items_off = 0;
};

constexpr double kChainAlpha = 6.0;  // per-unit fixed cost of the schedule's cost model, in k-blocks

static int chain_schedule(const PreparedGemm* pr, int n, int groups, cudaStream_t stream, ChainSchedule* out) {
  static std::mutex mu;
  static std::map<std::vector<int>, ChainSchedule> cache[kMaxDevices];
  std::vector<int> key = {groups, n};
  for (int q = 0; q < n; ++q) {
    key.push_back(pr[q].p.total_items);
    key.push_back(pr[q].p.num_k_iters);
  }
  std::lock_guard<std::mutex> lock(mu);
  auto& tab = cache[device_slot()];
  auto it = tab.find(key);
  if (it != tab.end()) {
    *out = it->second;
    return DS_OK;
  }
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  DS_CUDA_OK(cudaStreamIsCapturing(stream, &cs));
  DS_REQUIRE(cs == cudaStreamCaptureStatusNone,
             "ds_gemm_chain: first use of a chain shape must happen outside a graph capture (it uploads its schedule)");
  const int hdr = groups * (kMaxChain + 1);
  std::vector<std::vector<int>> mine(static_cast<size_t>(groups) * kMaxChain);
  using Slot = std::pair<double, int>;  // (time the CTA becomes free, CTA)
  std::priority_queue<Slot, std::vector<Slot>, std::greater<Slot>> free_at;
  for (int g = 0; g < groups; ++g) free_at.push({0.0, g});
  int total = 0;
  for (int q = 0; q < n; ++q) {
    const double cost = static_cast<double>(pr[q].p.num_k_iters) + kChainAlpha;
    for (int u = 0; u < pr[q].p.total_items; ++u) {
      Slot s = free_at.top();
      free_at.pop();
      mine[static_cast<size_t>(s.second) * kMaxChain + q].push_back(u);
      s.first += cost;
      free_at.push(s);
    }
    total += pr[q].p.total_items;
  }
  std::vector<int> host(static_cast<size_t>(hdr) + total);
  int pos = 0;
  for (int g = 0; g < groups; ++g) {
    for (int q = 0; q < kMaxChain; ++q) {
      host[g * (kMaxChain + 1) + q] = pos;
      for (int u : mine[static_cast<size_t>(g) * kMaxChain + q]) host[hdr + pos++] = u;
    }
    host[g * (kMaxChain + 1) + kMaxChain] = pos;
  }
  ChainSchedule sc;
  sc.items_off = hdr;
  DS_CUDA_OK(cudaMalloc(&sc.dev, host.size() * sizeof(int)));
  DS_CUDA_OK(cudaMemcpy(sc.dev, host.data(), host.size() * sizeof(int), cudaMemcpyHostToDevice));
  tab.emplace(std::move(key), sc);
  *out = sc;
  return DS_OK;
}

// ds_gemm_chain: n dependent GEMMs (problem q+1 reads problem q's output rows) as ONE persistent launch of
// 128 x 256 tiles; see GemmLaunch.  `dep` = kMaxChain * dep_stride + 1 zeroed ints the kernel hands back zeroed.
static int launch_chain(PreparedGemm* pr, int n, int* dep, int dep_len, int num_sms, cudaStream_t stream) {
  GemmLaunch<kMaxChain> L;
  const int m_groups = pr[0].p.num_m_tiles;
  int max_units = 0;
  for (int q = 0; q < n; ++q) {
    GemmParams& p = pr[q].p;
    const int units = m_groups * p.num_n_tiles;
    p.wide_units = units;
    p.wide_m_tiles = m_groups;
    p.nt_narrow = 0;
    p.tail_start = units;
    p.tail_parts = 1;
    p.total_items = units;
    p.ws = nullptr;
    if (units > max_units) max_units = units;
    for (int i = 0; i < 6; ++i) L.tm[q][i] = pr[q].tm[i];
    L.p[q] = p;
  }
  for (int q = n; q < kMaxChain; ++q) {  // unused slots: defined bytes
    for (int i = 0; i < 6; ++i) L.tm[q][i] = pr[0].tm[i];
    L.p[q] = pr[0].p;
  }
  L.nq = n;
  L.dep = dep;
  L.dep_stride = m_groups;
  DS_REQUIRE(kMaxChain * L.dep_stride + 1 <= dep_len,
             "ds_gemm_chain: dependency buffer too small (%d ints for %d row blocks)", dep_len, L.dep_stride);
  const int groups = max_units < num_sms ? max_units : num_sms;
  ChainSchedule sc;
  const int rc = chain_schedule(pr, n, groups, stream, &sc);
  if (rc != DS_OK) return rc;
  L.sched = sc.dev;
  L.sched_items = sc.items_off;
  return launch_wgmma<256, false, kMaxChain>(L, groups, stream, "gemm_bf16_wgmma(chain)");
}

template <int BN>
static int launch_gemm(const PreparedGemm& g, int num_sms, cudaStream_t stream, void* splitk_ws,
                       long long splitk_ws_bytes) {
  // the statistics epilogue is a separate instantiation: the default one keeps its register budget
  if (g.p.chan_stats) return launch_gemm_t<BN, true>(g, num_sms, stream, splitk_ws, splitk_ws_bytes);
  return launch_gemm_t<BN, false>(g, num_sms, stream, splitk_ws, splitk_ws_bytes);
}

static int pick_bn(int N, int epilogue) {
  if (epilogue == DS_EPI_GEGLU) return 256;
  if (N <= 128) return 128;
  // wide tiles read less shared memory per MMA (the A slice is shared by more columns), so BN = 256 is the default;
  // BN = 192 (3 x 64-column blocks) is used where it trims >= 15 % of the padded columns.
  const int c256 = ((N + 255) / 256) * 256, c192 = ((N + 191) / 192) * 192;
  return (c192 * 100 <= c256 * 85) ? 192 : 256;
}

// Output / residual tensor maps for the TMA epilogue: plain GEMM = 2-D {n_out, M}, box {64, 128};
// conv = 4-D NHWC {Cout, Wo, Ho, B}, box {64, 16, 8, 1} (the same 8x16 pixel patch as the M tile).
static bool make_out_map(CUtensorMap* m, const void* base, const GemmParams& p, int ld, int conv_B) {
  if (p.conv && p.out_stride == 2) {
    // one phase of the fused nearest-x2 upsample: `base` points at the phase's first pixel of the FULL-resolution
    // [B][2Ho][2Wo][C] output; the 8x16 patch lands on every second pixel in x and y (tensor-map element strides)
    const uint64_t Wf = 2ull * p.Wo, Hf = 2ull * p.Ho;
    const uint64_t dims[4] = {static_cast<uint64_t>(p.n_out), Wf - 1, Hf - 1, static_cast<uint64_t>(conv_B)};
    const uint64_t strides[3] = {static_cast<uint64_t>(ld) * 2, Wf * ld * 2, Hf * Wf * ld * 2};
    const uint32_t box[4] = {64, 2 * kConvTileW, 2 * kConvTileH, 1};
    const uint32_t es[4] = {1, 2, 2, 1};
    return encode_tmap_bf16(m, base, 4, dims, strides, box, es);
  }
  if (p.conv) {
    const uint64_t dims[4] = {static_cast<uint64_t>(p.n_out), static_cast<uint64_t>(p.Wo), static_cast<uint64_t>(p.Ho),
                              static_cast<uint64_t>(conv_B)};
    const uint64_t strides[3] = {static_cast<uint64_t>(ld) * 2, static_cast<uint64_t>(p.Wo) * ld * 2,
                                 static_cast<uint64_t>(p.Ho) * p.Wo * ld * 2};
    const uint32_t box[4] = {64, kConvTileW, kConvTileH, 1};
    return encode_tmap_bf16(m, base, 4, dims, strides, box, nullptr);
  }
  const uint64_t dims[2] = {static_cast<uint64_t>(p.n_out), static_cast<uint64_t>(p.M)};
  const uint64_t strides[1] = {static_cast<uint64_t>(ld) * 2};
  const uint32_t box[2] = {64, kBM};
  return encode_tmap_bf16(m, base, 2, dims, strides, box, nullptr);
}

// Everything run_gemm decides about one problem except the launch: tile shape, epilogue kind, output / residual /
// weight tensor maps, the narrow-tile schedule.  `chain`: the problem is a link of ds_gemm_chain (256-column tiles, no
// mixed-width tail — its row blocks must all have num_n_tiles units).
static int prepare_gemm(const CUtensorMap& tmA, const CUtensorMap& tmA2, const void* w, int ldw, GemmParams& p,
                        int conv_B, cudaStream_t stream, bool row_stats_zeroed, bool chain, const DeviceInfo& dev,
                        PreparedGemm* out) {
  const int bn = chain ? 256 : pick_bn(p.N, p.epilogue);
  // the kernel's GEGLU pass pairs value | gate columns of a 256-wide tile; narrower instantiations do not compile it
  DS_REQUIRE(p.epilogue != DS_EPI_GEGLU || bn == 256, "ds_gemm_bf16: GEGLU needs 256-column tiles (got %d)", bn);
  // coalesced TMA epilogue whenever the bf16 output (and residual) rows are 16-byte addressable
  auto aligned16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  p.tma_epilogue = !p.out_fp32 && p.n_out % 8 == 0 && p.ldo % 8 == 0 && aligned16(p.out) &&
                   (!p.residual || (p.ldres % 8 == 0 && aligned16(p.residual)));
  if (p.row_stats_out) {
    DS_REQUIRE(p.tma_epilogue, "ds_gemm_bf16: row_stats_out needs a 16-byte addressable bf16 output");
    if (!row_stats_zeroed)
      DS_CUDA_OK(cudaMemsetAsync(p.row_stats_out, 0, sizeof(double) * 2 * static_cast<size_t>(p.M), stream));
  }
  if (p.chan_stats) {
    DS_REQUIRE(p.tma_epilogue && p.epilogue != DS_EPI_GEGLU,
               "chan_stats needs a 16-byte addressable bf16 output and no GEGLU epilogue");
    DS_REQUIRE((reinterpret_cast<uintptr_t>(p.chan_stats) & 15) == 0, "chan_stats must be 16-byte aligned");
    if (!p.conv)
      DS_REQUIRE(p.stats_rows_per_sample > 0 && p.stats_rows_per_sample % kBM == 0,
                 "ds_gemm_bf16: chan_stats needs stats_rows_per_sample %% 128 == 0 (got %d)", p.stats_rows_per_sample);
  }
  CUtensorMap tmC = tmA, tmR = tmA;  // placeholders when the direct epilogue is used
  if (p.tma_epilogue) {
    if (!make_out_map(&tmC, p.out, p, p.ldo, conv_B)) return DS_ERR_CUDA;
    if (p.residual && !make_out_map(&tmR, p.residual, p, p.ldres, conv_B)) return DS_ERR_CUDA;
  }
  p.conv_B = conv_B;
  // DS_GEMM_EARLY_W=1: request the first weight tiles BEFORE griddepcontrol.wait.  Opt-in: it is only legal when `w`
  // is constant data (w_is_constant).
  static const int early_w_env = [] {
    const char* e = getenv("DS_GEMM_EARLY_W");
    return e ? atoi(e) : 0;
  }();
  if (!early_w_env) p.w_const = 0;
  p.num_n_tiles = (p.N + bn - 1) / bn;
  p.wide_units = 0;
  p.wide_m_tiles = 0;
  p.nt_narrow = 0;
  // narrow last n-tile: when the last BN-wide tile of a row would hold <= 128 real columns (N = 640 -> 256|256|128,
  // N = 320 -> 192|128, N = 1920 -> 7 x 256|128) it runs as a 128-column unit: same unit count, no padded MMAs.
  // Not in a chain: the chain kernel has only the 256-wide wgmma (a data-dependent wgmma width there makes ptxas
  // serialise its MMAs), so its last tile is a full 256-row weight box whose rows beyond N are TMA zero fill; the
  // epilogue stops at n_out, so the outputs are the same.
  p.last_narrow = 0;
  if (!chain && bn > kNarrowBN && p.epilogue != DS_EPI_GEGLU) {
    const int last_cols = p.N - (p.num_n_tiles - 1) * bn;
    if (last_cols <= kNarrowBN) p.last_narrow = 1;
  }
  // ---- mixed-width schedule: when the last round of the persistent schedule would fill less than ~45 % of the CTAs,
  // the m-rows that fall into it are cut into 128-column units instead (twice as many, half as long; same kernel, same
  // launch: the MMA width, the B box and the epilogue's column range are per unit) and appended after the wide units,
  // so the round-robin hands them to the CTAs that would otherwise idle.  Bit-identical outputs (same K order per
  // output element).  Not with row_stats_out: a unit sums its rows' statistics in fp32 over its own columns before the
  // fp64 add, so a row in a narrow unit would get differently rounded LayerNorm statistics, and whether the schedule
  // runs depends on M — a sample's statistics would change with the batch it runs in.  DS_GEMM_TAIL=0: off.
  static const int tail_env = [] {
    const char* e = getenv("DS_GEMM_TAIL");
    return e ? atoi(e) : 1;
  }();
  if (tail_env && !chain && bn == 256 && p.epilogue != DS_EPI_GEGLU && p.N % 128 == 0 &&
      !p.last_narrow && !p.row_stats_out) {
    const int G = dev.num_sms;  // one persistent CTA per SM
    const int mp = p.num_m_tiles, nt = p.num_n_tiles;
    const int units = mp * nt;
    const int full = units / G, rem = units - full * G;
    if (full >= 1 && rem > 0 && rem * 100 < G * 45) {
      const int R = (full * G) / nt;                 // m-tiles whose wide tiles fill exactly `full` rounds
      const int nt128 = p.N / 128;
      const int narrow = (mp - R) * nt128;
      // rounds in units of a wide tile: the narrow units run at ~0.6 of a wide unit each
      const int total = R * nt + narrow;
      const float cost = static_cast<float>(full) + 0.6f * static_cast<float>((total - full * G + G - 1) / G);
      if (R >= 1 && R < mp && cost < 0.95f * static_cast<float>(full + 1)) {
        p.wide_units = R * nt;
        p.wide_m_tiles = R;
        p.nt_narrow = nt128;
      }
    }
  }
  CUtensorMap tmB, tmB2;
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(p.K), static_cast<uint64_t>(p.N)};
    const uint64_t strides[1] = {static_cast<uint64_t>(ldw) * 2};
    const uint32_t box[2] = {kBK, static_cast<uint32_t>(bn)};
    if (!encode_tmap_bf16(&tmB, w, 2, dims, strides, box, nullptr)) return DS_ERR_CUDA;
    tmB2 = tmB;
    if (p.nt_narrow > 0 || p.last_narrow) {
      const uint32_t box2[2] = {kBK, static_cast<uint32_t>(kNarrowBN)};
      if (!encode_tmap_bf16(&tmB2, w, 2, dims, strides, box2, nullptr)) return DS_ERR_CUDA;
    }
  }
  out->tm[0] = tmA;
  out->tm[1] = tmB;
  out->tm[2] = tmC;
  out->tm[3] = tmR;
  out->tm[4] = tmA2;
  out->tm[5] = tmB2;
  out->p = p;
  out->bn = bn;
  return DS_OK;
}

static int run_gemm(const CUtensorMap& tmA_in, const CUtensorMap& tmA2_in, const void* w, int ldw, GemmParams& p_in,
                    int conv_B, cudaStream_t stream, bool row_stats_zeroed, void* splitk_ws,
                    long long splitk_ws_bytes) {
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  PreparedGemm g;
  const int rc = prepare_gemm(tmA_in, tmA2_in, w, ldw, p_in, conv_B, stream, row_stats_zeroed, false, dev, &g);
  if (rc != DS_OK) return rc;
  if (g.bn == 256) return launch_gemm<256>(g, dev.num_sms, stream, splitk_ws, splitk_ws_bytes);
  if (g.bn == 192) return launch_gemm<192>(g, dev.num_sms, stream, splitk_ws, splitk_ws_bytes);
  return launch_gemm<128>(g, dev.num_sms, stream, splitk_ws, splitk_ws_bytes);
}

// argument checks + A tensor map(s) + GemmParams of one ds_gemm_args (shared by ds_gemm_bf16 and ds_gemm_chain)
static int build_problem(const ds_gemm_args* a, CUtensorMap* tmA_out, CUtensorMap* tmA2_out, GemmParams* p_out) {
  DS_REQUIRE(a != nullptr, "ds_gemm_bf16: args is NULL");
  DS_REQUIRE(a->a && a->w && a->out, "ds_gemm_bf16: a/w/out must be non-NULL");
  DS_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0, "ds_gemm_bf16: M,N,K must be positive (got %d,%d,%d)", a->M, a->N,
             a->K);
  DS_REQUIRE(a->K % 8 == 0 && a->lda % 8 == 0 && a->ldw % 8 == 0,
             "ds_gemm_bf16: K, lda, ldw must be multiples of 8 (got %d,%d,%d)", a->K, a->lda, a->ldw);
  DS_REQUIRE((a->a2 || a->lda >= a->K) && a->ldw >= a->K, "ds_gemm_bf16: lda/ldw smaller than K");
  DS_REQUIRE((reinterpret_cast<uintptr_t>(a->a) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->w) & 15) == 0,
             "ds_gemm_bf16: a and w must be 16-byte aligned");
  DS_REQUIRE(a->epilogue >= DS_EPI_NONE && a->epilogue <= DS_EPI_QUICKGELU, "ds_gemm_bf16: bad epilogue %d", a->epilogue);
  if (a->epilogue == DS_EPI_GEGLU) {
    DS_REQUIRE(a->N % 256 == 0, "ds_gemm_bf16: GEGLU needs N %% 256 == 0 (128 value + 128 gate rows per block)");
    // the GEGLU pass adds the row bias to the value columns only (one more per-element load for the gates spills
    // the 256-wide accumulator): refuse the combination rather than return value * gelu(gate without row bias)
    DS_REQUIRE(a->rowbias == nullptr, "ds_gemm_bf16: GEGLU takes no rowbias");
  }
  if (a->rowbias) DS_REQUIRE(a->rows_per_batch > 0, "ds_gemm_bf16: rowbias needs rows_per_batch > 0");
  const int n_out = a->epilogue == DS_EPI_GEGLU ? a->N / 2 : a->N;
  DS_REQUIRE(a->ldo >= n_out, "ds_gemm_bf16: ldo (%d) smaller than output width (%d)", a->ldo, n_out);
  if (a->residual) DS_REQUIRE(a->ldres >= n_out, "ds_gemm_bf16: ldres smaller than output width");

  CUtensorMap& tmA = *tmA_out;
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(a->K), static_cast<uint64_t>(a->M)};
    const uint64_t strides[1] = {static_cast<uint64_t>(a->lda) * 2};
    const uint32_t box[2] = {kBK, kBM};
    if (!encode_tmap_bf16(&tmA, a->a, 2, dims, strides, box, nullptr)) return DS_ERR_CUDA;
  }
  GemmParams& p = *p_out;
  p = GemmParams{};
  p.bias = a->bias;
  p.rowbias = a->rowbias;
  p.residual = static_cast<const __nv_bfloat16*>(a->residual);
  p.out = a->out;
  p.M = a->M;
  p.N = a->N;
  p.K = a->K;
  p.n_out = n_out;
  p.ldo = a->ldo;
  p.ldres = a->ldres;
  p.rows_per_batch = a->rows_per_batch > 0 ? a->rows_per_batch : 1;
  p.ldrb = a->rowbias_ld > 0 ? a->rowbias_ld : a->N;
  p.epilogue = a->epilogue;
  p.out_fp32 = a->out_fp32;
  p.out_scale = a->out_scale == 1.0f ? 0.0f : a->out_scale;
  if (a->ln_stats) {
    DS_REQUIRE(a->ln_colsum != nullptr, "ds_gemm_bf16: ln_stats needs ln_colsum");
    DS_REQUIRE(a->rowbias == nullptr, "ds_gemm_bf16: ln_stats and rowbias are mutually exclusive");
    DS_REQUIRE((reinterpret_cast<uintptr_t>(a->ln_stats) & 15) == 0, "ds_gemm_bf16: ln_stats must be 16-byte aligned");
  }
  p.ln_stats = a->ln_stats;
  p.ln_colsum = a->ln_colsum;
  p.ln_eps = a->ln_eps;
  p.ln_inv_k = 1.0f / static_cast<float>(a->K);
  p.row_stats_out = a->row_stats_out;
  if (a->row_stats_out)
    DS_REQUIRE((reinterpret_cast<uintptr_t>(a->row_stats_out) & 15) == 0, "ds_gemm_bf16: row_stats_out must be 16-byte aligned");
  p.zero_rows = a->zero_rows;
  if (a->zero_rows)
    DS_REQUIRE((reinterpret_cast<uintptr_t>(a->zero_rows) & 15) == 0 && a->zero_rows != a->row_stats_out &&
                   a->zero_rows != a->ln_stats,
               "ds_gemm_bf16: zero_rows must be 16-byte aligned and distinct from ln_stats / row_stats_out");
  p.num_m_tiles = (a->M + kBM - 1) / kBM;
  p.num_k_iters = (a->K + kBK - 1) / kBK;
  p.k1_iters = p.num_k_iters;
  p.conv = 0;
  p.taps_x = 3;
  p.out_stride = 1;
  p.chan_stats = a->chan_stats;
  p.stats_rows_per_sample = a->stats_rows_per_sample;
  p.w_const = a->w_is_constant != 0;
  CUtensorMap& tmA2 = *tmA2_out;
  tmA2 = tmA;
  if (a->a2) {
    DS_REQUIRE(a->K1 > 0 && a->K1 < a->K && a->K1 % kBK == 0, "ds_gemm_bf16: a2 needs 0 < K1 < K and K1 %% 64 == 0");
    DS_REQUIRE(a->lda >= a->K1 && a->lda2 >= a->K - a->K1 && a->lda2 % 8 == 0 &&
                   (reinterpret_cast<uintptr_t>(a->a2) & 15) == 0,
               "ds_gemm_bf16: bad lda / lda2 / alignment for the two-operand form");
    const uint64_t dims1[2] = {static_cast<uint64_t>(a->K1), static_cast<uint64_t>(a->M)};
    const uint64_t strides1[1] = {static_cast<uint64_t>(a->lda) * 2};
    const uint64_t dims2[2] = {static_cast<uint64_t>(a->K - a->K1), static_cast<uint64_t>(a->M)};
    const uint64_t strides2[1] = {static_cast<uint64_t>(a->lda2) * 2};
    const uint32_t box[2] = {kBK, kBM};
    if (!encode_tmap_bf16(&tmA, a->a, 2, dims1, strides1, box, nullptr)) return DS_ERR_CUDA;
    if (!encode_tmap_bf16(&tmA2, a->a2, 2, dims2, strides2, box, nullptr)) return DS_ERR_CUDA;
    p.k1_iters = a->K1 / kBK;
  }
  return DS_OK;
}

}  // namespace ds

extern "C" int ds_gemm_bf16(const ds_gemm_args* a, void* stream) {
  using namespace ds;
  CUtensorMap tmA, tmA2;
  GemmParams p;
  const int rc = build_problem(a, &tmA, &tmA2, &p);
  if (rc != DS_OK) return rc;
  return run_gemm(tmA, tmA2, a->w, a->ldw, p, 0, static_cast<cudaStream_t>(stream), a->row_stats_zeroed != 0,
                  a->splitk_ws, a->splitk_ws_bytes);
}

extern "C" int ds_gemm_chain(const ds_gemm_args* args, int n, int* dep, int dep_len, void* stream) {
  using namespace ds;
  DS_REQUIRE(args != nullptr && n >= 1 && n <= kMaxChain, "ds_gemm_chain: 1..%d problems (got %d)", kMaxChain, n);
  DS_REQUIRE(dep != nullptr && (reinterpret_cast<uintptr_t>(dep) & 3) == 0, "ds_gemm_chain: dep is NULL / unaligned");
  DeviceInfo dev;
  if (!get_device(&dev)) return DS_ERR_CUDA;
  PreparedGemm pr[kMaxChain];
  for (int q = 0; q < n; ++q) {
    const ds_gemm_args* a = args + q;
    CUtensorMap tmA, tmA2;
    GemmParams p;
    const int rc = build_problem(a, &tmA, &tmA2, &p);
    if (rc != DS_OK) return rc;
    DS_REQUIRE(a->M == args[0].M && a->M > kBM, "ds_gemm_chain: every problem must have the same M > 128");
    DS_REQUIRE(!a->chan_stats && !a->out_fp32, "ds_gemm_chain: no chan_stats / fp32 outputs in a chain");
    if (q > 0)
      DS_REQUIRE(a->a == args[q - 1].out && a->a2 == nullptr,
                 "ds_gemm_chain: problem %d must read problem %d's output as its A operand", q, q - 1);
    const int rc2 = prepare_gemm(tmA, tmA2, a->w, a->ldw, p, 0, static_cast<cudaStream_t>(stream),
                                 a->row_stats_zeroed != 0, true, dev, &pr[q]);
    if (rc2 != DS_OK) return rc2;
    DS_REQUIRE(pr[q].p.tma_epilogue, "ds_gemm_chain: problem %d needs a 16-byte addressable bf16 output", q);
  }
  return launch_chain(pr, n, dep, dep_len, dev.num_sms, static_cast<cudaStream_t>(stream));
}

extern "C" int ds_gemm_chain_max(void) { return ds::kMaxChain; }

extern "C" int64_t ds_gemm_splitk_ws_bytes(void) {
  int sms = 256;
  ds::DeviceInfo dev;
  if (ds::get_device(&dev)) sms = dev.num_sms;
  // at most (CTAs - 1) tail units of 128 x 256 fp32, plus the counter header
  return 1024 + static_cast<int64_t>(sms) * 128 * 256 * 4;
}

namespace ds {
// one launch of the implicit-GEMM conv: `taps_y x taps_x` window at offset (off_x, off_y), weights [Cout][taps][Cin]
static int conv_launch(const ds_conv3x3_args* a, const void* w, void* out, int Ho, int Wo, int taps_y, int taps_x,
                       int off_x, int off_y, int out_stride, cudaStream_t stream) {
  CUtensorMap tmA;
  {
    const uint64_t dims[4] = {static_cast<uint64_t>(a->Cin), static_cast<uint64_t>(a->W),
                              static_cast<uint64_t>(a->H), static_cast<uint64_t>(a->B)};
    const uint64_t strides[3] = {static_cast<uint64_t>(a->Cin) * 2, static_cast<uint64_t>(a->W) * a->Cin * 2,
                                 static_cast<uint64_t>(a->H) * a->W * a->Cin * 2};
    const uint32_t box[4] = {kBK, static_cast<uint32_t>(kConvTileW * a->stride),
                             static_cast<uint32_t>(kConvTileH * a->stride), 1};
    const uint32_t es[4] = {1, static_cast<uint32_t>(a->stride), static_cast<uint32_t>(a->stride), 1};
    if (!encode_tmap_bf16(&tmA, a->x, 4, dims, strides, box, es)) return DS_ERR_CUDA;
  }
  const int taps = taps_y * taps_x;
  GemmParams p{};
  p.bias = a->bias;
  p.rowbias = a->rowbias;
  p.residual = static_cast<const __nv_bfloat16*>(a->residual);
  p.out = out;
  p.tiles_x = (Wo + kConvTileW - 1) / kConvTileW;
  p.tiles_y = (Ho + kConvTileH - 1) / kConvTileH;
  p.M = a->B * Ho * Wo;
  p.N = a->Cout;
  p.K = taps * a->Cin;
  p.n_out = a->Cout;
  p.ldo = a->Cout;
  p.ldres = a->Cout;
  p.rows_per_batch = 1;
  p.ldrb = a->rowbias_ld > 0 ? a->rowbias_ld : a->Cout;
  p.epilogue = DS_EPI_NONE;
  p.out_fp32 = a->out_fp32;
  p.out_scale = a->out_scale == 1.0f ? 0.0f : a->out_scale;
  p.num_m_tiles = a->B * p.tiles_x * p.tiles_y;
  p.num_k_iters = taps * (a->Cin / kBK);
  p.conv = 1;
  p.stride = a->stride;
  p.Ho = Ho;
  p.Wo = Wo;
  p.cin_chunks = a->Cin / kBK;
  p.taps_x = taps_x;
  p.off_x = off_x;
  p.off_y = off_y;
  p.out_stride = out_stride;
  p.k1_iters = p.num_k_iters;
  p.chan_stats = a->chan_stats;
  p.w_const = 1;  // conv filters are parameters
  return run_gemm(tmA, tmA, w, taps * a->Cin, p, a->B, stream, false, a->splitk_ws, a->splitk_ws_bytes);
}
}  // namespace ds

extern "C" int ds_conv3x3_nhwc(const ds_conv3x3_args* a, void* stream) {
  using namespace ds;
  DS_REQUIRE(a != nullptr, "ds_conv3x3_nhwc: args is NULL");
  DS_REQUIRE(a->x && a->w && a->out, "ds_conv3x3_nhwc: x/w/out must be non-NULL");
  DS_REQUIRE(a->B > 0 && a->H > 0 && a->W > 0 && a->Cin > 0 && a->Cout > 0, "ds_conv3x3_nhwc: bad geometry");
  DS_REQUIRE(a->Cin % 64 == 0, "ds_conv3x3_nhwc: Cin must be a multiple of 64 (got %d)", a->Cin);
  DS_REQUIRE(a->stride == 1 || a->stride == 2, "ds_conv3x3_nhwc: stride must be 1 or 2 (got %d)", a->stride);
  DS_REQUIRE((reinterpret_cast<uintptr_t>(a->x) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->w) & 15) == 0,
             "ds_conv3x3_nhwc: x and w must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (a->upsample2) {
    // conv3x3(nearest_x2(x)) as FOUR 2x2 convolutions of x, one per output-pixel parity (a, b): the 3x3 taps that read
    // the same low-resolution pixel are pre-summed (weights.pack_conv3x3_up2), so the op does 16 instead of 36 MACs per
    // (low-res pixel, Cin, Cout) and the upsampled tensor is never written.  Phase (a, b) writes pixels (2i+a, 2j+b).
    DS_REQUIRE(a->stride == 1 && !a->pad_bottom_right && !a->residual && !a->rowbias && !a->out_fp32 && a->Cout % 8 == 0 &&
                   (reinterpret_cast<uintptr_t>(a->out) & 15) == 0,
               "ds_conv3x3_nhwc: upsample2 needs stride 1, bf16 output with Cout %% 8 == 0, no residual / rowbias");
    const size_t wph = static_cast<size_t>(a->Cout) * 4 * a->Cin;  // elements per phase: [Cout][2][2][Cin]
    for (int ph = 0; ph < 4; ++ph) {
      const int pa = ph >> 1, pb = ph & 1;
      const __nv_bfloat16* w = static_cast<const __nv_bfloat16*>(a->w) + ph * wph;
      __nv_bfloat16* o = static_cast<__nv_bfloat16*>(a->out) + (static_cast<size_t>(pa) * 2 * a->W + pb) * a->Cout;
      const int rc = conv_launch(a, w, o, a->H, a->W, 2, 2, pb ? 0 : -1, pa ? 0 : -1, 2, st);
      if (rc != DS_OK) return rc;
    }
    return DS_OK;
  }
  if (a->pad_bottom_right) {
    // diffusers Downsample2D(padding=0) of the VAE encoder: F.pad(x, (0, 1, 0, 1)) then a stride-2 conv without
    // padding.  Output pixel i reads input rows / columns 2i .. 2i+2: the tap window starts at offset 0 instead of -1,
    // and the one padded row and column are the tensor map's out-of-bounds zero fill.
    DS_REQUIRE(a->stride == 2 && a->H >= 2 && a->W >= 2,
               "ds_conv3x3_nhwc: pad_bottom_right needs stride 2 and H, W >= 2 (got stride %d, %d x %d)", a->stride,
               a->H, a->W);
    return conv_launch(a, a->w, a->out, a->H / 2, a->W / 2, 3, 3, 0, 0, 1, st);
  }
  const int Ho = (a->H - 1) / a->stride + 1;
  const int Wo = (a->W - 1) / a->stride + 1;
  return conv_launch(a, a->w, a->out, Ho, Wo, 3, 3, -1, -1, 1, st);
}
