// Native (torch-free) check of ds_gemm_bf16 / ds_conv3x3_nhwc through the C ABI against a scalar CPU
// restatement.  Usage: test_gemm <case-id> ; prints one line "CASE <id> <name> PASS|FAIL ..." and timing.
// Run each case in its own process so a device trap in one case cannot poison the next.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "dsengine.h"

static uint16_t f2bf(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  uint32_t r = u + 0x7FFF + ((u >> 16) & 1);
  return (uint16_t)(r >> 16);
}
static float bf2f(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
static uint32_t rng_state = 12345;
static float frand() {  // uniform in [-1, 1)
  rng_state = rng_state * 1664525u + 1013904223u;
  return ((rng_state >> 8) & 0xFFFFFF) / 8388608.0f - 1.0f;
}
static double gelu(double x) { return 0.5 * x * (1.0 + erf(x * 0.70710678118654752440)); }

#define CK(x)                                                                    \
  do {                                                                           \
    cudaError_t e = (x);                                                         \
    if (e != cudaSuccess) {                                                      \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
      exit(2);                                                                   \
    }                                                                            \
  } while (0)

struct Case {
  const char* name;
  int conv;
  int M, N, K;  // gemm
  int B, H, W, Cin, Cout, stride;  // conv
  int epi, bias, rowbias, residual, out_fp32;
  int sampled;  // 0 = full check
  int time_it;
};

static const Case cases[] = {
    {"gemm_basic_256x256x128", 0, 256, 256, 128, 0, 0, 0, 0, 0, 0, DS_EPI_NONE, 0, 0, 0, 0, 0, 0},
    {"gemm_k64_single", 0, 128, 128, 64, 0, 0, 0, 0, 0, 0, DS_EPI_NONE, 0, 0, 0, 0, 0, 0},
    {"gemm_tails_300x200x72", 0, 300, 200, 72, 0, 0, 0, 0, 0, 0, DS_EPI_NONE, 1, 0, 0, 0, 0, 0},
    {"gemm_bn128_640", 0, 384, 640, 320, 0, 0, 0, 0, 0, 0, DS_EPI_NONE, 1, 0, 1, 0, 0, 0},
    {"gemm_geglu_256x512x128", 0, 256, 512, 128, 0, 0, 0, 0, 0, 0, DS_EPI_GEGLU, 1, 0, 0, 0, 0, 0},
    {"gemm_rowbias_res_fp32", 0, 512, 256, 192, 0, 0, 0, 0, 0, 0, DS_EPI_NONE, 1, 1, 1, 1, 0, 0},
    {"gemm_smallN_4", 0, 200, 4, 128, 0, 0, 0, 0, 0, 0, DS_EPI_NONE, 1, 0, 0, 0, 0, 0},
    {"gemm_many_tiles_4096x1024x512", 0, 4096, 1024, 512, 0, 0, 0, 0, 0, 0, DS_EPI_SILU, 1, 0, 1, 0, 1, 0},
    {"conv_s1_2x16x24_64_128", 1, 0, 0, 0, 2, 16, 24, 64, 128, 1, DS_EPI_NONE, 1, 1, 1, 0, 0, 0},
    {"conv_s1_tails_2x20x12_128_64", 1, 0, 0, 0, 2, 20, 12, 128, 64, 1, DS_EPI_NONE, 1, 0, 0, 0, 0, 0},
    {"conv_s2_2x16x32_64_128", 1, 0, 0, 0, 2, 16, 32, 64, 128, 2, DS_EPI_NONE, 1, 0, 0, 0, 0, 0},
    {"conv_s2_odd_1x18x14_64_64", 1, 0, 0, 0, 1, 18, 14, 64, 64, 2, DS_EPI_NONE, 0, 0, 0, 0, 0, 0},
    // split-K tail (DS_GEMM_SPLITK=1, see test_native_harness_gpu.py): the units of the partial last round of the
    // persistent schedule are cut along K into slices on different CTAs that add into the fp32 workspace.  It needs
    // more units than SMs, a last round of <= SMs / 2 units, >= 4 k-blocks and no mixed-width schedule (which takes
    // over when a BN = 256 launch's last round is under 45 % full).  On the H100's 132 SMs:
    //   21979 x 128 (BN 128): 172 units, 40 left over -> 3 slices of 8 k-blocks, M tail
    //   11515 x 360 (BN 192, TMA block clipped to 40 columns): 180 units, 48 left -> 2 slices, residual
    //   conv 6 x 40 x 40, 64 -> 320 (192 | 128 narrow): 180 units, 48 left -> 2 slices of 9 k-blocks
    {"gemm_tailsplit_bn128_21979x128x512", 0, 21979, 128, 512, 0, 0, 0, 0, 0, 0, DS_EPI_NONE, 1, 0, 0, 0, 0, 0},
    {"gemm_tailsplit_bn192_11515x360x256_res", 0, 11515, 360, 256, 0, 0, 0, 0, 0, 0, DS_EPI_NONE, 1, 0, 1, 0, 0, 0},
    {"conv_tailsplit_6x40x40_64_320", 1, 0, 0, 0, 6, 40, 40, 64, 320, 1, DS_EPI_NONE, 1, 1, 1, 0, 0, 0},
    // timing cases (cfg2 shapes), sampled check
    {"T_gemm_attnproj_32768x640x640", 0, 32768, 640, 640, 0, 0, 0, 0, 0, 0, DS_EPI_NONE, 1, 0, 1, 0, 1, 1},
    {"T_gemm_qkv_8192x3840x1280", 0, 8192, 3840, 1280, 0, 0, 0, 0, 0, 0, DS_EPI_NONE, 0, 0, 0, 0, 1, 1},
    {"T_gemm_ff1_geglu_8192x10240x1280", 0, 8192, 10240, 1280, 0, 0, 0, 0, 0, 0, DS_EPI_GEGLU, 1, 0, 0, 0, 1, 1},
    {"T_gemm_ff2_8192x1280x5120", 0, 8192, 1280, 5120, 0, 0, 0, 0, 0, 0, DS_EPI_NONE, 1, 0, 1, 0, 1, 1},
    {"T_gemm_ff1_geglu_32768x5120x640", 0, 32768, 5120, 640, 0, 0, 0, 0, 0, 0, DS_EPI_GEGLU, 1, 0, 0, 0, 1, 1},
    {"T_conv_8x64x64_640_640", 1, 0, 0, 0, 8, 64, 64, 640, 640, 1, DS_EPI_NONE, 1, 1, 1, 0, 1, 1},
    {"T_conv_8x32x32_1280_1280", 1, 0, 0, 0, 8, 32, 32, 1280, 1280, 1, DS_EPI_NONE, 1, 1, 1, 0, 1, 1},
    {"T_conv_8x128x128_320_320", 1, 0, 0, 0, 8, 128, 128, 320, 320, 1, DS_EPI_NONE, 1, 1, 1, 0, 1, 1},
    {"T_conv_s2_8x128x128_320_320", 1, 0, 0, 0, 8, 128, 128, 320, 320, 2, DS_EPI_NONE, 1, 0, 0, 0, 1, 1},
};
static const int num_cases = sizeof(cases) / sizeof(cases[0]);

int main(int argc, char** argv) {
  if (argc < 2) {
    printf("%d\n", num_cases);
    return 0;
  }
  const int id = atoi(argv[1]);
  if (id < 0 || id >= num_cases) return 1;
  const Case c = cases[id];
  rng_state = 1000 + id;

  int M, N, K, n_out, Ho = 0, Wo = 0;
  if (c.conv) {
    Ho = (c.H - 1) / c.stride + 1;
    Wo = (c.W - 1) / c.stride + 1;
    M = c.B * Ho * Wo;
    N = c.Cout;
    K = 9 * c.Cin;
  } else {
    M = c.M;
    N = c.N;
    K = c.K;
  }
  n_out = c.epi == DS_EPI_GEGLU ? N / 2 : N;
  const int rows_per_batch = c.conv ? Ho * Wo : 128;
  const int nbatch = c.conv ? c.B : (M + rows_per_batch - 1) / rows_per_batch;

  const size_t a_elems = c.conv ? (size_t)c.B * c.H * c.W * c.Cin : (size_t)M * K;
  std::vector<uint16_t> hA(a_elems), hW((size_t)N * K), hRes;
  std::vector<float> hBias, hRow;
  for (auto& v : hA) v = f2bf(frand());
  const float wscale = 1.0f / sqrtf((float)K);
  for (auto& v : hW) v = f2bf(frand() * wscale * 2.0f);
  if (c.bias) {
    hBias.resize(N);
    for (auto& v : hBias) v = frand() * 0.5f;
  }
  if (c.rowbias) {
    hRow.resize((size_t)nbatch * N);
    for (auto& v : hRow) v = frand() * 0.5f;
  }
  if (c.residual) {
    hRes.resize((size_t)M * n_out);
    for (auto& v : hRes) v = f2bf(frand());
  }

  void *dA, *dW, *dOut, *dRes = nullptr;
  float *dBias = nullptr, *dRow = nullptr;
  const size_t out_bytes = (size_t)M * n_out * (c.out_fp32 ? 4 : 2);
  CK(cudaMalloc(&dA, a_elems * 2));
  CK(cudaMalloc(&dW, hW.size() * 2));
  CK(cudaMalloc(&dOut, out_bytes));
  CK(cudaMemcpy(dA, hA.data(), a_elems * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dW, hW.data(), hW.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemset(dOut, 0xFF, out_bytes));
  if (c.bias) {
    CK(cudaMalloc(&dBias, N * 4));
    CK(cudaMemcpy(dBias, hBias.data(), N * 4, cudaMemcpyHostToDevice));
  }
  if (c.rowbias) {
    CK(cudaMalloc(&dRow, hRow.size() * 4));
    CK(cudaMemcpy(dRow, hRow.data(), hRow.size() * 4, cudaMemcpyHostToDevice));
  }
  if (c.residual) {
    CK(cudaMalloc(&dRes, hRes.size() * 2));
    CK(cudaMemcpy(dRes, hRes.data(), hRes.size() * 2, cudaMemcpyHostToDevice));
  }

  // split-K workspace: all zero on entry, the kernels must leave it all zero (checked below)
  const long long ws_bytes = ds_gemm_splitk_ws_bytes();
  void* dWs = nullptr;
  CK(cudaMalloc(&dWs, ws_bytes));
  CK(cudaMemset(dWs, 0, ws_bytes));
  auto run = [&]() -> int {
    if (c.conv) {
      ds_conv3x3_args a;
      memset(&a, 0, sizeof(a));
      a.x = dA;
      a.w = dW;
      a.out = dOut;
      a.bias = dBias;
      a.rowbias = dRow;
      a.residual = dRes;
      a.B = c.B;
      a.H = c.H;
      a.W = c.W;
      a.Cin = c.Cin;
      a.Cout = c.Cout;
      a.stride = c.stride;
      a.out_fp32 = c.out_fp32;
      a.splitk_ws = dWs;
      a.splitk_ws_bytes = ws_bytes;
      return ds_conv3x3_nhwc(&a, nullptr);
    }
    ds_gemm_args a;
    memset(&a, 0, sizeof(a));
    a.a = dA;
    a.w = dW;
    a.out = dOut;
    a.bias = dBias;
    a.rowbias = dRow;
    a.residual = dRes;
    a.M = M;
    a.N = N;
    a.K = K;
    a.lda = K;
    a.ldw = K;
    a.ldo = n_out;
    a.ldres = n_out;
    a.rows_per_batch = rows_per_batch;
    a.epilogue = c.epi;
    a.out_fp32 = c.out_fp32;
    a.splitk_ws = dWs;
    a.splitk_ws_bytes = ws_bytes;
    return ds_gemm_bf16(&a, nullptr);
  };

  int rc = run();
  if (rc == DS_OK) rc = run();  // a second launch on the same workspace: it must have been left clean
  if (rc != DS_OK) {
    printf("CASE %d %s FAIL rc=%d err=%s\n", id, c.name, rc, ds_last_error());
    return 1;
  }
  cudaError_t se = cudaDeviceSynchronize();
  if (se != cudaSuccess) {
    printf("CASE %d %s FAIL sync: %s\n", id, c.name, cudaGetErrorString(se));
    return 1;
  }
  std::vector<uint8_t> hOut(out_bytes);
  CK(cudaMemcpy(hOut.data(), dOut, out_bytes, cudaMemcpyDeviceToHost));
  {
    std::vector<uint32_t> hWs((size_t)ws_bytes / 4);
    CK(cudaMemcpy(hWs.data(), dWs, ws_bytes, cudaMemcpyDeviceToHost));
    size_t dirty = 0;
    for (uint32_t v : hWs) dirty += (v & 0x7fffffffu) != 0;  // -0.0f counts as clean
    if (dirty) {
      printf("CASE %d %s FAIL split-K workspace not left clean: %zu non-zero words\n", id, c.name, dirty);
      return 1;
    }
  }

  // ---- CPU restatement on all / sampled outputs
  auto a_at = [&](int m, int k) -> float {
    if (!c.conv) return bf2f(hA[(size_t)m * K + k]);
    const int img = m / (Ho * Wo), rem = m % (Ho * Wo), oy = rem / Wo, ox = rem % Wo;
    const int tap = k / c.Cin, ci = k % c.Cin, r = tap / 3, s = tap % 3;
    const int iy = oy * c.stride + r - 1, ix = ox * c.stride + s - 1;
    if (iy < 0 || iy >= c.H || ix < 0 || ix >= c.W) return 0.0f;
    return bf2f(hA[(((size_t)img * c.H + iy) * c.W + ix) * c.Cin + ci]);
  };
  // sum a w and sum |a||w| of one output element
  auto dot = [&](int m, int wrow, double* abs_sum) -> double {
    double acc = 0, aacc = 0;
    const uint16_t* wr = &hW[(size_t)wrow * K];
    for (int k = 0; k < K; ++k) {
      const double p = (double)a_at(m, k) * (double)bf2f(wr[k]);
      acc += p;
      aacc += fabs(p);
    }
    *abs_sum = aacc;
    return acc;
  };
  // the reference and its bound (tests/gemm_check.py): |got - ref| <= 2^-8 |ref| + 2^-9 absref + act_abs, where
  // absref = sum |a||w| + |bias| + |rowbias| + |residual| through the activation's Lipschitz constant and act_abs
  // covers gelu_sig5 (2.6e-5 + 2^-21 |x|) and __expf / __fdividef in SiLU (2^-21 |x| (1 + |x|))
  auto ref_at = [&](int m, int j, double* tol) -> double {
    const int batch = m / rows_per_batch;
    double v, absref, act_abs = 0;
    if (c.epi == DS_EPI_GEGLU) {
      const int blk = j / 128, jj = j % 128;
      const int hrow = blk * 256 + jj, grow = hrow + 128;
      double eh, eg;
      const double h = dot(m, hrow, &eh) + (c.bias ? hBias[hrow] : 0.0);
      const double g = dot(m, grow, &eg) + (c.bias ? hBias[grow] : 0.0);
      if (c.bias) {
        eh += fabs(hBias[hrow]);
        eg += fabs(hBias[grow]);
      }
      v = h * gelu(g);
      absref = fabs(gelu(g)) * eh + 1.13 * fabs(h) * eg;
      act_abs = (2.6e-5 + ldexp(fabs(g), -21)) * fabs(h);
    } else {
      v = dot(m, j, &absref);
      if (c.bias) {
        v += hBias[j];
        absref += fabs(hBias[j]);
      }
      if (c.rowbias) {
        v += hRow[(size_t)batch * N + j];
        absref += fabs(hRow[(size_t)batch * N + j]);
      }
      if (c.epi == DS_EPI_GELU) {
        act_abs = 2.6e-5 + ldexp(fabs(v), -21);
        v = gelu(v);
        absref *= 1.13;
      }
      if (c.epi == DS_EPI_SILU) {
        act_abs = ldexp(fabs(v) * (1.0 + fabs(v)), -21);
        v = v / (1.0 + exp(-v));
        absref *= 1.1;
      }
    }
    if (c.residual) {
      v += bf2f(hRes[(size_t)m * n_out + j]);
      absref += fabs(bf2f(hRes[(size_t)m * n_out + j]));
    }
    *tol = ldexp(fabs(v), -8) + ldexp(absref, -9) + act_abs;
    return v;
  };
  auto got_at = [&](int m, int j) -> double {
    if (c.out_fp32) return ((float*)hOut.data())[(size_t)m * n_out + j];
    return bf2f(((uint16_t*)hOut.data())[(size_t)m * n_out + j]);
  };

  double max_err = 0, max_ref = 0, worst = 0;
  long long bad = 0, checked = 0;
  int shown = 0;
  auto check = [&](int m, int j) {
    double tol;
    const double r = ref_at(m, j, &tol), g = got_at(m, j);
    const double err = fabs(r - g);
    if (err > 0 && err / tol > worst) worst = err / tol;
    if (!(err <= tol)) {
      ++bad;
      if (shown < 8) {
        printf("  mismatch m=%d j=%d ref=%.5f got=%.5f tol=%.3g\n", m, j, r, g, tol);
        ++shown;
      }
    }
    if (err > max_err) max_err = err;
    if (fabs(r) > max_ref) max_ref = fabs(r);
    ++checked;
  };
  if (!c.sampled) {
    for (int m = 0; m < M; ++m)
      for (int j = 0; j < n_out; ++j) check(m, j);
  } else {
    for (int t = 0; t < 6000; ++t) {
      rng_state = rng_state * 1664525u + 1013904223u;
      const int m = (rng_state >> 4) % M;
      rng_state = rng_state * 1664525u + 1013904223u;
      const int j = (rng_state >> 4) % n_out;
      check(m, j);
    }
    // plus the four corners of the output and the last row/col explicitly
    check(0, 0);
    check(M - 1, n_out - 1);
    check(0, n_out - 1);
    check(M - 1, 0);
  }

  double ms = 0, tflops = 0;
  if (c.time_it && bad == 0) {
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    for (int i = 0; i < 3; ++i) run();
    CK(cudaDeviceSynchronize());
    const int iters = 10;
    CK(cudaEventRecord(e0));
    for (int i = 0; i < iters; ++i) run();
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float t;
    CK(cudaEventElapsedTime(&t, e0, e1));
    ms = t / iters;
    tflops = 2.0 * M * (double)N * K / (ms * 1e-3) / 1e12;
  }
  printf("CASE %d %s %s checked=%lld bad=%lld max_err=%.4g max_ref=%.4g worst=%.3f", id, c.name,
         bad == 0 ? "PASS" : "FAIL", checked, bad, max_err, max_ref, worst);
  if (ms > 0) printf(" ms=%.4f TFLOPs=%.1f", ms, tflops);
  printf("\n");
  return bad == 0 ? 0 : 1;
}
