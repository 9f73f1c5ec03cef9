// Standalone GPU check of the fused dense-FFN kernels (ffn_fused.cu) against a double-precision CPU reference, plus
// CUDA-event timings at the benchmarked stage-0 / stage-1 shapes.
// Build: make build/ffn_test      Run: build/ffn_test [check|time|all]
#include "ffn_fused.cuh"
#include "gemm_tc.cuh"
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

namespace sm3 { const char* last_error(); }
using namespace sm3;

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(2); } } while (0)

template <class T> T* dev(const std::vector<T>& h) {
  T* d; CK(cudaMalloc(&d, std::max<size_t>(16, h.size() * sizeof(T))));
  CK(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice)); return d;
}
template <class T> T* dalloc(size_t n) { T* d; CK(cudaMalloc(&d, std::max<size_t>(16, n * sizeof(T)))); CK(cudaMemset(d, 0, n * sizeof(T))); return d; }
static double gelu(double x) { return 0.5 * x * (1.0 + erf(x / sqrt(2.0))); }
static double dgelu(double x) { return 0.5 * (1.0 + erf(x / sqrt(2.0))) + x * exp(-0.5 * x * x) / sqrt(2.0 * M_PI); }
static int g_fail = 0;

struct Dev {
  int M, C, H4;
  float *v, *dz, *w1, *b1, *w2, *b2, *gamma, *rs, *x, *w2g;
  uint16_t *v_img, *dz_img;
};

static uint16_t* pack_k(const float* X, long long rows, int cols) {
  uint16_t* out; CK(cudaMalloc(&out, (size_t)gemm::packed_act_elems(rows, cols, 0, 128) * 2));
  if (gemm::pack_act(X, cols, nullptr, rows, cols, 0, 128, out, 0) != 0) { printf("pack_act failed: %s\n", last_error()); exit(2); }
  return out;
}
static uint16_t* pack_w(const float* W, long long s_mn, long long s_k, int N, int K, int tile) {
  uint16_t* out; CK(cudaMalloc(&out, (size_t)gemm::packed_elems(N, K) * 2));
  if (gemm::pack_b(W, s_mn, s_k, 0, 1, N, K, out, 0, tile) != 0) { printf("pack_b failed: %s\n", last_error()); exit(2); }
  return out;
}

__global__ void scale_rows_k(const float* w, const float* g, float* o, int C, int H4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (long long)C * H4) o[i] = w[i] * g[i / H4];
}

static int g_cols = 0;     // row length of the tensor being compared (for the non-finite pattern dump)
static double maxrel(const std::vector<float>& got, const std::vector<double>& ref) {
  double mx = 0, sc = 0;
  size_t bad = 0;
  std::vector<int> by_col_mod8(8, 0);
  long long rmin = 1LL << 60, rmax = -1;
  std::vector<char> colhit(g_cols > 0 ? g_cols : 1, 0);
  for (size_t i = 0; i < ref.size(); ++i) {
    if (!std::isfinite(got[i])) {
      if (bad++ < 3) printf("    non-finite value %g at flat index %zu (of %zu)\n", got[i], i, ref.size());
      if (g_cols > 0) { const long long r = i / g_cols; const int c = (int)(i % g_cols); by_col_mod8[c % 8]++; colhit[c] = 1; rmin = std::min(rmin, r); rmax = std::max(rmax, r); }
      continue;
    }
    mx = std::max(mx, fabs((double)got[i] - ref[i])); sc = std::max(sc, fabs(ref[i]));
  }
  if (bad) {
    printf("    %zu non-finite values", bad);
    if (g_cols > 0) {
      printf("; rows %lld..%lld; by (col %% 8):", rmin, rmax);
      for (int m = 0; m < 8; ++m) printf(" %d", by_col_mod8[m]);
      printf("; columns hit:");
      for (int c = 0; c < g_cols; ++c) if (colhit[c]) printf(" %d", c);
    }
    printf("\n");
    return 1e30;
  }
  return mx / (sc + 1e-30);
}

static void check(int M, int C, bool with_rs) {
  const int H4 = 4 * C;
  std::mt19937 rng(77 + M + C);
  std::normal_distribution<float> nd(0.f, 1.f);
  std::vector<float> v((size_t)M * C), dz((size_t)M * C), x((size_t)M * C), w1((size_t)H4 * C), b1(H4), w2((size_t)C * H4), b2(C), gm(C), rs(M);
  for (auto& t : v) t = nd(rng);
  for (auto& t : dz) t = nd(rng) * 0.1f;
  for (auto& t : x) t = nd(rng);
  for (auto& t : w1) t = nd(rng) / sqrtf((float)C);
  for (auto& t : w2) t = nd(rng) / sqrtf((float)H4);
  for (auto& t : b1) t = nd(rng) * 0.2f;
  for (auto& t : b2) t = nd(rng) * 0.2f;
  for (auto& t : gm) t = 0.1f + 0.9f * (float)(rng() % 1000) / 1000.f;
  for (auto& t : rs) t = (rng() % 4 == 0) ? 0.f : 1.25f;
  float *dv = dev(v), *ddz = dev(dz), *dx = dev(x), *dw1 = dev(w1), *db1 = dev(b1), *dw2 = dev(w2), *db2 = dev(b2), *dgm = dev(gm), *drs = dev(rs);
  float* dw2g = dalloc<float>((size_t)C * H4);
  scale_rows_k<<<(C * H4 + 255) / 256, 256>>>(dw2, dgm, dw2g, C, H4);
  uint16_t* v_img = pack_k(dv, M, C);
  uint16_t* dz_img = pack_k(ddz, M, C);
  // ---------------- CPU reference (double) ----------------
  std::vector<double> h((size_t)M * H4), y2((size_t)M * C), out((size_t)M * C), dvr((size_t)M * C), dh((size_t)M * H4);
  std::vector<double> rdw1((size_t)H4 * C, 0.0), rdw2((size_t)C * H4, 0.0), rdb1(H4, 0.0);
  for (int m = 0; m < M; ++m) {
    for (int j = 0; j < H4; ++j) {
      double s = b1[j];
      for (int c = 0; c < C; ++c) s += (double)v[(size_t)m * C + c] * w1[(size_t)j * C + c];
      h[(size_t)m * H4 + j] = s;
    }
    for (int c = 0; c < C; ++c) {
      double s = b2[c];
      for (int j = 0; j < H4; ++j) s += gelu(h[(size_t)m * H4 + j]) * w2[(size_t)c * H4 + j];
      y2[(size_t)m * C + c] = s;
      out[(size_t)m * C + c] = x[(size_t)m * C + c] + (with_rs ? rs[m] : 1.0) * gm[c] * s;
    }
    for (int j = 0; j < H4; ++j) {
      double da = 0;
      for (int c = 0; c < C; ++c) da += (double)dz[(size_t)m * C + c] * gm[c] * w2[(size_t)c * H4 + j];
      dh[(size_t)m * H4 + j] = da * dgelu(h[(size_t)m * H4 + j]);
      rdb1[j] += dh[(size_t)m * H4 + j];
    }
    for (int c = 0; c < C; ++c) {
      double s = 0;
      for (int j = 0; j < H4; ++j) s += dh[(size_t)m * H4 + j] * w1[(size_t)j * C + c];
      dvr[(size_t)m * C + c] = s;
    }
    for (int j = 0; j < H4; ++j)
      for (int c = 0; c < C; ++c) {
        rdw1[(size_t)j * C + c] += dh[(size_t)m * H4 + j] * v[(size_t)m * C + c];
        rdw2[(size_t)c * H4 + j] += gm[c] * (double)dz[(size_t)m * C + c] * gelu(h[(size_t)m * H4 + j]);
      }
  }
  // ---------------- forward ----------------
  {
    const int HC = ffn::chain_chunk(0, C);
    if (HC == 0) { printf("fwd  M=%-6d C=%-4d unsupported\n", M, C); }
    else {
      ffn::ChainParams p{};
      p.a1 = v_img; p.wa1 = pack_w(dw1, C, 1, H4, C, HC); p.wb = pack_w(dw2, H4, 1, C, H4, C);
      p.bias1 = db1; p.bias2 = db2; p.col_scale = dgm; p.row_scale = with_rs ? drs : nullptr; p.resid = dx;
      float* dout = dalloc<float>((size_t)M * C); float* daux = dalloc<float>((size_t)M * C);
      p.out = dout; p.aux_out = daux; p.M = M; p.C = C; p.H4 = H4; p.HC = HC; p.passes = 3; p.mode = 0;
      const int rc = ffn::chain(p, 0);
      cudaError_t e = cudaDeviceSynchronize();
      if (rc != 0 || e != cudaSuccess) { printf("fwd  M=%-6d C=%-4d LAUNCH FAILED rc=%d %s %s\n", M, C, rc, last_error(), cudaGetErrorString(e)); g_fail++; exit(3); }
      std::vector<float> go((size_t)M * C), ga((size_t)M * C);
      CK(cudaMemcpy(go.data(), dout, go.size() * 4, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(ga.data(), daux, ga.size() * 4, cudaMemcpyDeviceToHost));
      const double e1 = maxrel(go, out), e2 = maxrel(ga, y2);
      const bool ok = e1 < 1e-4 && e2 < 1e-4;
      printf("fwd  M=%-6d C=%-4d chunk=%d rs=%d  out err %.2e  y2 err %.2e  %s\n", M, C, HC, (int)with_rs, e1, e2, ok ? "ok" : "FAIL");
      if (!ok) g_fail++;
    }
  }
  // ---------------- backward into dv ----------------
  {
    const int HC = ffn::chain_chunk(1, C);
    if (HC == 0) { printf("bwd  M=%-6d C=%-4d unsupported\n", M, C); }
    else {
      ffn::ChainParams p{};
      p.a1 = v_img; p.a2 = dz_img; p.wa1 = pack_w(dw1, C, 1, H4, C, HC); p.wa2 = pack_w(dw2g, 1, H4, H4, C, HC);
      p.wb = pack_w(dw1, 1, C, C, H4, C);
      p.bias1 = db1;
      float* dout = dalloc<float>((size_t)M * C);
      p.out = dout; p.M = M; p.C = C; p.H4 = H4; p.HC = HC; p.passes = 3; p.mode = 1;
      const int rc = ffn::chain(p, 0);
      cudaError_t e = cudaDeviceSynchronize();
      if (rc != 0 || e != cudaSuccess) { printf("bwd  M=%-6d C=%-4d LAUNCH FAILED rc=%d %s %s\n", M, C, rc, last_error(), cudaGetErrorString(e)); g_fail++; exit(3); }
      std::vector<float> go((size_t)M * C);
      CK(cudaMemcpy(go.data(), dout, go.size() * 4, cudaMemcpyDeviceToHost));
      const double e1 = maxrel(go, dvr);
      const bool ok = e1 < 1e-4;
      printf("bwd  M=%-6d C=%-4d chunk=%d        dv err %.2e  %s\n", M, C, HC, e1, ok ? "ok" : "FAIL");
      if (!ok) g_fail++;
    }
  }
}

static int g_passes = 3, g_debug = 0;
static void timeit(int M, int C) {
  const int H4 = 4 * C;
  std::vector<float> w1((size_t)H4 * C, 0.01f), w2((size_t)C * H4, 0.01f), b1(H4, 0.1f), b2(C, 0.1f), gm(C, 0.5f);
  float* dv = dalloc<float>((size_t)M * C); float* ddz = dalloc<float>((size_t)M * C); float* dx = dalloc<float>((size_t)M * C);
  CK(cudaMemset(dv, 0x3c, (size_t)M * C * 4)); CK(cudaMemset(ddz, 0x3b, (size_t)M * C * 4));
  float *dw1 = dev(w1), *dw2 = dev(w2), *db1 = dev(b1), *db2 = dev(b2), *dgm = dev(gm);
  uint16_t* v_img = pack_k(dv, M, C); uint16_t* dz_img = pack_k(ddz, M, C);
  float* dout = dalloc<float>((size_t)M * C); float* daux = dalloc<float>((size_t)M * C);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  const double unit = 2.0 * M * C * (double)H4;     // FLOPs of one [M,C]x[C,4C] GEMM
  for (int mode = 0; mode < 2; ++mode) {
    const int HC = ffn::chain_chunk(mode, C);
    if (HC == 0) { printf("time mode %d M=%d C=%d: unsupported\n", mode, M, C); continue; }
    ffn::ChainParams p{};
    uint16_t* wa1 = pack_w(dw1, C, 1, H4, C, HC); uint16_t* wa2 = pack_w(dw2, 1, H4, H4, C, HC);
    {
      p.a1 = v_img; p.a2 = dz_img; p.wa1 = wa1; p.wa2 = wa2;
      p.wb = mode == 0 ? pack_w(dw2, H4, 1, C, H4, C) : pack_w(dw1, 1, C, C, H4, C);
      p.bias1 = db1; p.bias2 = mode == 0 ? db2 : nullptr; p.col_scale = mode == 0 ? dgm : nullptr; p.resid = mode == 0 ? dx : nullptr;
      p.out = dout; p.aux_out = mode == 0 ? daux : nullptr; p.M = M; p.C = C; p.H4 = H4; p.HC = HC; p.passes = g_passes; p.mode = mode; p.debug = g_debug;
    }
    auto launch = [&]() { return ffn::chain(p, 0); };
    for (int i = 0; i < 2; ++i) if (launch() != 0) { printf("launch failed: %s\n", last_error()); exit(3); }
    CK(cudaDeviceSynchronize());
    const int it = 10;
    cudaEventRecord(e0);
    for (int i = 0; i < it; ++i) launch();
    cudaEventRecord(e1);
    CK(cudaDeviceSynchronize());
    float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= it;
    const double alg = 2 * unit;                                           // GEMMs the algorithm needs (recomputation not counted)
    const double issued = (mode == 0 ? 2 : 3) * unit;
    const double bytes = mode == 0 ? 4.0 * M * C * 4 : 3.0 * M * C * 4;
    printf("time mode %d (%s) M=%d C=%d chunk=%d: %.3f ms  algorithmic %.1f TFLOP/s  issued %.1f TFLOP/s  min-HBM %.0f GB/s\n", mode,
           mode == 0 ? "fwd" : "bwd-dv", M, C, HC, ms, alg / ms * 1e-9, issued / ms * 1e-9, bytes / ms * 1e-6);
  }
}

int main(int argc, char** argv) {
  const std::string what = argc > 1 ? argv[1] : "all";
  if (argc > 2) g_passes = atoi(argv[2]);
  if (argc > 3) g_debug = atoi(argv[3]);
  if (what == "check640") { check(640, 96, true); printf(g_fail ? "FAILED\n" : "PASSED\n"); return g_fail; }
  if (what == "one") { printf("passes=%d debug=%d\n", g_passes, g_debug); timeit(524288, 96); return 0; }
  if (what == "check" || what == "all") {
    check(128, 96, false);
    check(640, 96, true);
    check(200, 96, true);       // ragged last tile
    check(45000, 96, false);    // > 132 x 2 tiles: every CTA loops, all ring phases wrap
    check(512, 64, true);
    check(384, 128, true);
    check(384, 192, false);
    printf(g_fail ? "FFN TEST FAILED (%d)\n" : "FFN TEST PASSED\n", g_fail);
  }
  if (what == "time" || what == "all") {
    timeit(524288, 96);
    timeit(131072, 192);
    timeit(262144, 96);
  }
  return g_fail ? 1 : 0;
}
