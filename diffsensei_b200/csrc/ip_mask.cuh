// ip_mask.cuh — the bbox -> key-visibility predicate of MaskedIPAttnProcessor2_0.prepare_attention_mask_ip
// (src/models/attention_processor.py:115-169), shared by the stand-alone mask kernel and the fused
// cross-attention kernel so both evaluate bit-identical membership.
//
// Reference semantics reproduced exactly (SURVEY.md §3.4):
//   * (H', W') are re-derived on the host from (N, aspect_ratio) in double precision like the Python code
//     (:131-139) — NOT the true feature-map shape;
//   * pixel coordinates are torch.linspace(0, 1, steps) in fp32 (:146-147).  ATen evaluates it as
//     step = 1/(steps-1);  i < steps/2 ? step*i : fma(-step, steps-1-i, 1)   [probed against torch 2.11 CPU];
//   * membership is the CLOSED interval test x1<=x<=x2 && y1<=y<=y2 on fp32 boxes (:159), so a padded
//     [0,0,0,0] box still captures pixel (0,0);
//   * key layout [num_dummy dummy | tokens_per_ip x ip0 | ip1 | ...] (:165-167); ip-i keys are visible iff the
//     pixel is in box i, dummy keys iff it is in no box (:143,162-163).
#pragma once
#include <math.h>
#include <stdint.h>

namespace ds {

constexpr int kMaxIps = 16;

// Host: Python's  width = int((N / ar) ** 0.5); height = N // width; while width*height != N: ...
inline bool derive_hw(int N, double aspect_ratio, int* Hd, int* Wd) {
  if (N <= 0 || !(aspect_ratio > 0.0)) return false;
  long long width = static_cast<long long>(pow(static_cast<double>(N) / aspect_ratio, 0.5));
  if (width < 1) return false;  // the reference would raise ZeroDivisionError
  long long height = N / width;
  while (width * height != N) {
    if (width * height < N)
      width += 1;
    else
      width -= 1;
    if (width < 1 || width > N) return false;
    height = N / width;
  }
  *Hd = static_cast<int>(height);
  *Wd = static_cast<int>(width);
  return true;
}

__device__ __forceinline__ float linspace01(int i, int steps) {
  if (steps <= 1) return 0.0f;
  const float step = __fdiv_rn(1.0f, static_cast<float>(steps - 1));
  return (i < steps / 2) ? __fmul_rn(step, static_cast<float>(i))
                         : __fmaf_rn(-step, static_cast<float>(steps - 1 - i), 1.0f);
}

// bit i set <=> token n (row-major over the derived H' x W' grid) lies inside box i
__device__ __forceinline__ uint32_t ip_inside_bits(const float* __restrict__ bbox, int num_ips, int n, int Hd, int Wd) {
  const int yi = n / Wd, xi = n - yi * Wd;
  const float x = linspace01(xi, Wd), y = linspace01(yi, Hd);
  uint32_t bits = 0;
  for (int i = 0; i < num_ips; ++i) {
    const float x1 = bbox[4 * i], y1 = bbox[4 * i + 1], x2 = bbox[4 * i + 2], y2 = bbox[4 * i + 3];
    if (x >= x1 && x <= x2 && y >= y1 && y <= y2) bits |= 1u << i;
  }
  return bits;
}

__device__ __forceinline__ bool ip_key_open(uint32_t bits, int key, int tokens_per_ip, int num_dummy) {
  if (key < num_dummy) return bits == 0;
  return (bits >> ((key - num_dummy) / tokens_per_ip)) & 1u;
}

// bits [lo, hi) of a 64-bit word, the range clipped to [0, 64)
__device__ __forceinline__ uint64_t bit_range64(int lo, int hi) {
  lo = max(lo, 0);
  hi = min(hi, 64);
  if (lo >= hi) return 0ull;
  const uint64_t below_hi = hi == 64 ? ~0ull : (1ull << hi) - 1ull;
  return below_hi & ~((1ull << lo) - 1ull);
}

// ip_key_open for the 64 keys [key0, key0 + 64) at once: bit k set <=> key key0 + k is open.  Keys past the last IP
// token are closed, as ip_key_open has them (their box index is >= num_ips).  A few range operations per open box
// instead of an integer division per key.
__device__ __forceinline__ uint64_t ip_open_keys64(uint32_t bits, int key0, int tokens_per_ip, int num_dummy) {
  uint64_t m = bits == 0 ? bit_range64(-key0, num_dummy - key0) : 0ull;
  for (uint32_t r = bits; r != 0; r &= r - 1) {
    const int lo = num_dummy + (__ffs(r) - 1) * tokens_per_ip - key0;
    m |= bit_range64(lo, lo + tokens_per_ip);
  }
  return m;
}

}  // namespace ds
