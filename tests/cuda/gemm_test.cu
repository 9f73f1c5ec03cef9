// Standalone GPU check of the split-bf16 wgmma GEMM against a double-precision CPU reference.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I sm3det_b200/csrc \
//        tests/cuda/gemm_test.cu sm3det_b200/csrc/gemm_tc.cu sm3det_b200/csrc/common.cu -o build/gemm_test
#include "gemm_tc.cuh"
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <string>
#include <vector>

namespace sm3 { const char* last_error(); }
using namespace sm3;
using namespace sm3::gemm;

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(2); } } while (0)

template <class T> T* dev(const std::vector<T>& h) {
  T* d; CK(cudaMalloc(&d, std::max<size_t>(16, h.size() * sizeof(T))));
  CK(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice)); return d;
}
static double gelu(double x) { return 0.5 * x * (1.0 + erf(x / sqrt(2.0))); }
static double dgelu(double x) { return 0.5 * (1.0 + erf(x / sqrt(2.0))) + x * exp(-0.5 * x * x) / sqrt(2.0 * M_PI); }

static int g_fail = 0;
static int g_debug = 0;

struct Case {
  std::string name;
  int M, N, K, BN = 0;
  bool a_mn = false, b_mn = false;
  bool gather = false, ints = false, kgather = false, packed = false, apacked = false;
  int sched = SCHED_DENSE, groups = 1, k_splits = 1;
  int epi = 0;
};

static void run(const Case& c) {
  std::mt19937 rng(1234);
  std::normal_distribution<float> nd(0.f, 1.f);
  std::uniform_int_distribution<int> id(-3, 3);
  auto val = [&]() { return c.ints ? (float)id(rng) : nd(rng); };
  const int M = c.M, N = c.N, K = c.K, G = c.groups;
  // physical storage
  const int a_rows_phys = c.gather ? M + 37 : M;
  std::vector<float> A((size_t)a_rows_phys * K), B((size_t)G * N * K);
  for (auto& v : A) v = val();
  for (auto& v : B) v = val();
  // A logical (m,k): K-major: A[m*K+k]; MN-major: A[k*M+m]  (only without gather)
  // B logical (g,n,k): K-major: B[g*N*K + n*K + k]; MN-major: B[g*N*K + k*N + n]
  std::vector<int> ridx;
  if (c.gather) {
    ridx.resize(M);
    std::uniform_int_distribution<int> rd(0, a_rows_phys - 1);
    for (int m = 0; m < M; ++m) ridx[m] = (m % 11 == 5) ? -1 : rd(rng);
  }
  std::vector<int> kidx;
  if (c.kgather) {
    kidx.resize(K);
    std::uniform_int_distribution<int> rd(0, K - 1);
    for (int k = 0; k < K; ++k) kidx[k] = (k % 13 == 7) ? -1 : rd(rng);
  }
  // grouped schedule: m tiles -> group
  std::vector<int> tile_group; std::vector<int> nmt(1);
  const int m_tiles = (M + BM - 1) / BM;
  if (c.sched == SCHED_GROUPED) {
    tile_group.resize(m_tiles);
    for (int t = 0; t < m_tiles; ++t) tile_group[t] = (t * G) / m_tiles;
    nmt[0] = m_tiles;
  }
  // split-K segments along K per group
  std::vector<int> segb, sege;
  if (c.sched == SCHED_SPLITK && G > 1) {
    segb.resize(G); sege.resize(G);
    int pos = 0;
    for (int g = 0; g < G; ++g) {
      int len = (g == 1) ? 0 : (K / G + (g % 2 ? 13 : -7));   // one empty group, ragged others
      if (g == G - 1) len = K - pos - 5;
      segb[g] = pos; sege[g] = pos + len; pos += len + 3;      // 3 unused rows between groups
    }
  }
  std::vector<float> bias((size_t)G * N), cs(N), rs(M), resid((size_t)M * N), aux((size_t)M * N);
  for (auto& v : bias) v = nd(rng);
  for (auto& v : cs) v = nd(rng);
  for (auto& v : rs) v = nd(rng);
  for (auto& v : resid) v = nd(rng);
  for (auto& v : aux) v = nd(rng);
  const int Gout = (c.sched == SCHED_SPLITK) ? G : 1;
  std::vector<float> D((size_t)Gout * M * N, 0.f), AUXO((size_t)M * N, 0.f);

  Params p{};
  float* dA = dev(A); float* dB = dev(B);
  p.A = dA; p.B = dB;
  if (!c.a_mn) { p.a_smn = K; p.a_sk = 1; } else { p.a_smn = 1; p.a_sk = M; }
  if (!c.b_mn) { p.b_smn = K; p.b_sk = 1; } else { p.b_smn = 1; p.b_sk = N; }
  p.b_group_stride = (c.sched == SCHED_GROUPED) ? (long long)N * K : 0;
  int* dridx = c.gather ? dev(ridx) : nullptr; p.a_row_index = dridx;
  int* dkidx = c.kgather ? dev(kidx) : nullptr; p.b_k_index = dkidx;
  p.M = M; p.N = N; p.K = K; p.BN = c.BN;
  p.sched = c.sched; p.k_splits = c.k_splits; p.num_groups = G;
  int* dtg = tile_group.empty() ? nullptr : dev(tile_group); int* dnmt = dev(nmt);
  p.tile_group = dtg; p.num_m_tiles_dev = dnmt;
  int* dsb = segb.empty() ? nullptr : dev(segb); int* dse = sege.empty() ? nullptr : dev(sege);
  p.seg_begin = dsb; p.seg_end = dse;
  float* dD = dev(D); p.D = dD; p.ldd = N; p.d_group_stride = (c.sched == SCHED_SPLITK) ? (long long)M * N : 0;
  float* dbias = dev(bias); p.bias = dbias; p.bias_group_stride = (c.sched == SCHED_GROUPED) ? N : 0;
  p.epi = c.epi;
  float* dauxo = dev(AUXO); float* daux = dev(aux);
  p.aux_out = (c.epi & EPI_GELU) ? dauxo : nullptr; p.aux_in = daux; p.ld_aux = N;
  std::vector<float> colsum_h((size_t)G * N, 0.f);
  float* dcolsum = dev(colsum_h); p.colsum = dcolsum; p.colsum_group_stride = (c.sched == SCHED_GROUPED) ? N : 0;
  float* dcs = dev(cs); float* drs = dev(rs); float* dres = dev(resid);
  p.col_scale = dcs; p.row_scale = drs; p.resid = dres; p.ld_resid = N;

  uint16_t* dpack = nullptr;
  if (c.packed) {
    const long long per = packed_elems(N, K);
    const int pg = (c.sched == SCHED_GROUPED) ? G : 1;
    CK(cudaMalloc(&dpack, (size_t)pg * per * 2));
    int prc = pack_b(dB, c.b_mn ? 1 : K, c.b_mn ? N : 1, (long long)N * K, pg, N, K, dpack, 0);
    if (prc != 0) { printf("CASE %-28s PACK FAILED (%s)\n", c.name.c_str(), last_error()); g_fail++; return; }
    p.b_packed = dpack; p.b_packed_group_stride = per;
  }
  uint16_t* dpa = nullptr; uint16_t* dpb2 = nullptr;
  if (c.apacked) {
    // A: activation pack (K-major with optional row gather, or MN-major for the wgrad form)
    const long long ea = c.a_mn ? packed_act_elems(K, M, 1, 128) : packed_act_elems(M, K, 0, 128);
    CK(cudaMalloc(&dpa, (size_t)ea * 2));
    int prc = c.a_mn ? pack_act(dA, M, nullptr, K, M, 1, 128, dpa, 0) : pack_act(dA, K, dridx, M, K, 0, 128, dpa, 0);
    if (prc != 0) { printf("CASE %-28s PACK_A FAILED (%s)\n", c.name.c_str(), last_error()); g_fail++; return; }
    p.a_packed = dpa; p.a_row_index = nullptr;
    if (c.a_mn) {   // wgrad: B is an activation too, MN-major tiles of the GEMM tile width, optional k gather
      const int bn = pick_bn(N);
      CK(cudaMalloc(&dpb2, (size_t)packed_act_elems(K, N, 1, bn) * 2));
      prc = pack_act(dB, N, dkidx, K, N, 1, bn, dpb2, 0);
      if (prc != 0) { printf("CASE %-28s PACK_B FAILED (%s)\n", c.name.c_str(), last_error()); g_fail++; return; }
      p.b_packed = dpb2; p.b_packed_group_stride = 0; p.b_k_index = nullptr;
    }
  }
  int rc = launch(p, 0);
  cudaError_t e = cudaDeviceSynchronize();
  if (rc != 0 || e != cudaSuccess) {
    printf("CASE %-28s LAUNCH FAILED rc=%d (%s) cuda=%s\n", c.name.c_str(), rc, last_error(), cudaGetErrorString(e));
    g_fail++; if (e != cudaSuccess) exit(3); return;
  }
  CK(cudaMemcpy(D.data(), dD, D.size() * sizeof(float), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(AUXO.data(), dauxo, AUXO.size() * sizeof(float), cudaMemcpyDeviceToHost));

  CK(cudaMemcpy(colsum_h.data(), dcolsum, colsum_h.size() * sizeof(float), cudaMemcpyDeviceToHost));
  std::vector<double> colsum_ref((size_t)G * N, 0.0);
  // reference
  double max_err = 0, max_ref = 0, max_aux_err = 0; long long nbad = 0; int bad_m = -1, bad_n = -1;
  const double max_ref_bound = c.ints ? 1e-9 : (3.0 * sqrt((double)K) + 10.0);   // ~ scale of |sum_k a*b| for N(0,1) data
  for (int go = 0; go < Gout; ++go)
  for (int m = 0; m < M; ++m) {
    int g = 0;
    if (c.sched == SCHED_GROUPED) g = tile_group[m / BM];
    if (c.sched == SCHED_SPLITK) g = go;
    int kb = 0, ke = K;
    if (!segb.empty()) { kb = segb[g]; ke = sege[g]; }
    for (int n = 0; n < N; ++n) {
      double acc = 0;
      const int bg = (c.sched == SCHED_GROUPED) ? g : 0;
      long long arow = m;
      bool zero = false;
      if (c.gather) { if (ridx[m] < 0) zero = true; else arow = ridx[m]; }
      if (!zero)
        for (int k = kb; k < ke; ++k) {
          const double a = c.a_mn ? A[(size_t)k * M + m] : A[(size_t)arow * K + k];
          double b;
          if (c.kgather) { if (kidx[k] < 0) continue; b = B[(size_t)kidx[k] * N + n]; }
          else b = c.b_mn ? B[(size_t)bg * N * K + (size_t)k * N + n] : B[(size_t)bg * N * K + (size_t)n * K + k];
          acc += a * b;
        }
      double pre = acc;
      if (c.epi & EPI_BIAS) acc += bias[(size_t)bg * N + n];
      if (c.epi & EPI_GELU) { pre = acc; acc = gelu(acc); }
      if (c.epi & EPI_DGELU) acc *= dgelu(aux[(size_t)m * N + n]);
      if (c.epi & EPI_COLSCALE) acc *= cs[n];
      if (c.epi & EPI_ROWSCALE) acc *= rs[m];
      if (c.epi & EPI_RESID) acc += resid[(size_t)m * N + n];
      if (c.epi & EPI_COLSUM) colsum_ref[(size_t)((c.sched == SCHED_GROUPED) ? g : 0) * N + n] += acc;
      const double got = D[(size_t)go * M * N + (size_t)m * N + n];
      const double err = fabs(got - acc);
      if (err > max_err) { max_err = err; }
      if (fabs(acc) > max_ref) max_ref = fabs(acc);
      if (err > 5e-5 * max_ref_bound) { if (nbad == 0) { bad_m = m; bad_n = n; } nbad++; }
      if (c.epi & EPI_GELU) max_aux_err = std::max(max_aux_err, fabs((double)AUXO[(size_t)m * N + n] - pre));
    }
  }
  double cs_err = 0, cs_ref = 0;
  if (c.epi & EPI_COLSUM) for (size_t i = 0; i < colsum_ref.size(); ++i) { cs_err = std::max(cs_err, fabs(colsum_ref[i] - colsum_h[i])); cs_ref = std::max(cs_ref, fabs(colsum_ref[i])); }
  if (cs_err > 1e-4 * (cs_ref + 1.0)) { nbad++; printf("   colsum mismatch: err %.3e ref %.3e\n", cs_err, cs_ref); }
  const double rel = max_err / (max_ref + 1e-30);
  const bool ok = (c.ints ? max_err == 0.0 : rel < 4e-5) && nbad == 0 && max_aux_err < 1e-3;
  printf("CASE %-28s M=%d N=%d K=%d BN=%d a_mn=%d b_mn=%d : max_abs_err=%.3e max_ref=%.3e rel=%.3e aux_err=%.2e bad=%lld first_bad=(%d,%d) %s\n",
         c.name.c_str(), M, N, K, c.BN, c.a_mn, c.b_mn, max_err, max_ref, rel, max_aux_err, nbad, bad_m, bad_n, ok ? "OK" : "FAIL");
  if (!ok) {
    g_fail++;
    // print a small corner to help diagnose layout bugs
    for (int m = 0; m < 4 && m < M; ++m) { printf("   row %d got:", m); for (int n = 0; n < 8; ++n) printf(" %9.3f", D[(size_t)m * N + n]); printf("\n"); }
  }
  cudaFree(dA); cudaFree(dB); cudaFree(dD); cudaFree(dbias); cudaFree(dauxo); cudaFree(daux); cudaFree(dcs); cudaFree(drs); cudaFree(dres);
  if (dridx) cudaFree(dridx); if (dtg) cudaFree(dtg); cudaFree(dnmt); if (dsb) cudaFree(dsb); if (dse) cudaFree(dse);
}

static void bench(const char* name, int M, int N, int K, bool a_mn, bool b_mn, int epi, int sched = SCHED_DENSE, int splits = 1, bool packed = false, bool apacked = false) {
  float *A, *B, *D, *bias, *aux;
  CK(cudaMalloc(&A, (size_t)M * K * 4)); CK(cudaMalloc(&B, (size_t)N * K * 4)); CK(cudaMalloc(&D, (size_t)M * N * 4));
  CK(cudaMalloc(&bias, (size_t)N * 4)); CK(cudaMalloc(&aux, (size_t)M * N * 4));
  CK(cudaMemset(A, 0, (size_t)M * K * 4)); CK(cudaMemset(B, 0, (size_t)N * K * 4)); CK(cudaMemset(bias, 0, N * 4));
  Params p{};
  p.A = A; p.B = B; p.D = D; p.ldd = N; p.M = M; p.N = N; p.K = K; p.bias = bias; p.epi = epi; p.aux_out = (epi & EPI_GELU) ? aux : nullptr; p.ld_aux = N;
  if (!a_mn) { p.a_smn = K; p.a_sk = 1; } else { p.a_smn = 1; p.a_sk = M; }
  if (!b_mn) { p.b_smn = K; p.b_sk = 1; } else { p.b_smn = 1; p.b_sk = N; }
  p.sched = sched; p.k_splits = splits; p.num_groups = 1; p.debug = g_debug;
  uint16_t* dpack = nullptr;
  if (packed) { CK(cudaMalloc(&dpack, (size_t)packed_elems(N, K) * 2)); pack_b(B, b_mn ? 1 : K, b_mn ? N : 1, 0, 1, N, K, dpack, 0); p.b_packed = dpack; }
  uint16_t* dpa = nullptr; uint16_t* dpb2 = nullptr;
  if (apacked) {
    if (a_mn) {
      const int bn = pick_bn(N);
      CK(cudaMalloc(&dpa, (size_t)packed_act_elems(K, M, 1, 128) * 2)); pack_act(A, M, nullptr, K, M, 1, 128, dpa, 0);
      CK(cudaMalloc(&dpb2, (size_t)packed_act_elems(K, N, 1, bn) * 2)); pack_act(B, N, nullptr, K, N, 1, bn, dpb2, 0);
      p.b_packed = dpb2;
    } else {
      CK(cudaMalloc(&dpa, (size_t)packed_act_elems(M, K, 0, 128) * 2)); pack_act(A, K, nullptr, M, K, 0, 128, dpa, 0);
    }
    p.a_packed = dpa;
    cudaEvent_t q0, q1; cudaEventCreate(&q0); cudaEventCreate(&q1);
    cudaEventRecord(q0);
    for (int i = 0; i < 5; ++i) { if (a_mn) pack_act(A, M, nullptr, K, M, 1, 128, dpa, 0); else pack_act(A, K, nullptr, M, K, 0, 128, dpa, 0); }
    cudaEventRecord(q1); cudaEventSynchronize(q1);
    float pms; cudaEventElapsedTime(&pms, q0, q1);
    printf("      pack A: %.3f ms per call (%.0f GB/s)\n", pms / 5, 8.0 * M * K / (pms / 5) * 1e-6);
  }
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int i = 0; i < 3; ++i) launch(p, 0);
  cudaEventRecord(e0);
  const int iters = 10;
  for (int i = 0; i < iters; ++i) launch(p, 0);
  cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
  float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= iters;
  const double flops = 2.0 * M * N * K;
  const double bytes = 4.0 * ((double)M * K + (double)N * K + (double)M * N * ((epi & EPI_GELU) ? 2 : 1));
  printf("BENCH %-26s M=%d N=%d K=%d : %.3f ms  %.1f TFLOP/s (algorithmic)  %.1f GB/s (min traffic)\n", name, M, N, K, ms, flops / ms * 1e-9, bytes / ms * 1e-6);
  cudaFree(A); cudaFree(B); cudaFree(D); cudaFree(bias); cudaFree(aux);
}

int main(int argc, char** argv) {
  const bool quick = argc > 1 && std::string(argv[1]) == "quick";
  const bool only_bench = argc > 1 && std::string(argv[1]) == "bench";
  const int bench_idx = argc > 2 ? atoi(argv[2]) : -1;
  g_debug = argc > 3 ? atoi(argv[3]) : 0;
  if (g_debug) printf("DEBUG FLAGS %d (results invalid)\n", g_debug);
  std::vector<Case> cases;
  auto add = [&](Case c) { cases.push_back(c); };
  { Case c; c.name = "nt_int_128x32x32";   c.M = 128; c.N = 32;  c.K = 32;  c.ints = true; add(c); }
  { Case c; c.name = "nt_int_128x256x64";  c.M = 128; c.N = 256; c.K = 64;  c.ints = true; add(c); }
  { Case c; c.name = "nt_int_tail";        c.M = 300; c.N = 96;  c.K = 96;  c.ints = true; add(c); }
  { Case c; c.name = "nt_f32_384";         c.M = 1000; c.N = 384; c.K = 96; add(c); }
  { Case c; c.name = "nt_f32_bn128";       c.M = 520; c.N = 384; c.K = 160; c.BN = 128; add(c); }
  { Case c; c.name = "nt_f32_bigK";        c.M = 256; c.N = 768; c.K = 3072; add(c); }
  { Case c; c.name = "nt_gather";          c.M = 700; c.N = 192; c.K = 192; c.gather = true; add(c); }
  { Case c; c.name = "nt_bias_gelu";       c.M = 333; c.N = 256; c.K = 128; c.epi = EPI_BIAS | EPI_GELU; add(c); }
  { Case c; c.name = "nt_bias_cs_resid";   c.M = 333; c.N = 96;  c.K = 384; c.epi = EPI_BIAS | EPI_COLSCALE | EPI_RESID; add(c); }
  { Case c; c.name = "nt_rowscale";        c.M = 200; c.N = 64;  c.K = 64;  c.epi = EPI_BIAS | EPI_ROWSCALE; add(c); }
  { Case c; c.name = "nn_int (B MN-major)"; c.M = 128; c.N = 128; c.K = 64; c.b_mn = true; c.ints = true; add(c); }
  { Case c; c.name = "nn_f32_dgelu";       c.M = 450; c.N = 384; c.K = 96;  c.b_mn = true; c.epi = EPI_DGELU; add(c); }
  { Case c; c.name = "nn_f32_bn96";        c.M = 450; c.N = 96;  c.K = 384; c.b_mn = true; add(c); }
  { Case c; c.name = "nn_f32_bn192";       c.M = 130; c.N = 192; c.K = 768; c.b_mn = true; add(c); }
  { Case c; c.name = "tn_int (A,B MN-major)"; c.M = 128; c.N = 128; c.K = 64; c.a_mn = true; c.b_mn = true; c.ints = true; add(c); }
  { Case c; c.name = "tn_f32_wgrad_splitk"; c.M = 384; c.N = 96; c.K = 5000; c.a_mn = true; c.b_mn = true; c.sched = SCHED_SPLITK; c.k_splits = 7; c.epi = EPI_ATOMIC; add(c); }
  { Case c; c.name = "tn_f32_wgrad_groups"; c.M = 96; c.N = 384; c.K = 4000; c.a_mn = true; c.b_mn = true; c.sched = SCHED_SPLITK; c.k_splits = 3; c.groups = 4; c.epi = EPI_ATOMIC; add(c); }
  { Case c; c.name = "tn_f32_wgrad_kgather"; c.M = 384; c.N = 96; c.K = 3000; c.a_mn = true; c.b_mn = true; c.sched = SCHED_SPLITK; c.k_splits = 5; c.groups = 3; c.epi = EPI_ATOMIC; c.kgather = true; add(c); }
  { Case c; c.name = "nn_dgelu_colsum";   c.M = 450; c.N = 384; c.K = 96;  c.b_mn = true; c.epi = EPI_DGELU | EPI_COLSUM; add(c); }
  { Case c; c.name = "grouped_nn_packed_colsum"; c.M = 640; c.N = 96; c.K = 384; c.sched = SCHED_GROUPED; c.groups = 4; c.b_mn = true; c.packed = true; c.epi = EPI_COLSUM; add(c); }
  { Case c; c.name = "nt_ALLpacked";       c.M = 1000; c.N = 384; c.K = 96;  c.packed = true; c.apacked = true; c.epi = EPI_BIAS | EPI_GELU; add(c); }
  { Case c; c.name = "nt_ALLpacked_ktail"; c.M = 333; c.N = 96;  c.K = 48;  c.packed = true; c.apacked = true; add(c); }
  { Case c; c.name = "nt_ALLpacked_bigK";  c.M = 256; c.N = 768; c.K = 3072; c.packed = true; c.apacked = true; add(c); }
  { Case c; c.name = "nn_ALLpacked dgrad"; c.M = 450; c.N = 384; c.K = 96;  c.b_mn = true; c.packed = true; c.apacked = true; c.epi = EPI_DGELU | EPI_COLSUM; add(c); }
  { Case c; c.name = "grouped_ALLpacked_gather"; c.M = 1024; c.N = 384; c.K = 96; c.sched = SCHED_GROUPED; c.groups = 3; c.gather = true; c.packed = true; c.apacked = true; c.epi = EPI_BIAS | EPI_GELU; add(c); }
  { Case c; c.name = "tn_ALLpacked_splitk"; c.M = 384; c.N = 96; c.K = 4992; c.a_mn = true; c.b_mn = true; c.sched = SCHED_SPLITK; c.k_splits = 7; c.epi = EPI_ATOMIC; c.apacked = true; add(c); }
  { Case c; c.name = "tn_ALLpacked_ragged"; c.M = 96; c.N = 384; c.K = 1000; c.a_mn = true; c.b_mn = true; c.sched = SCHED_SPLITK; c.k_splits = 3; c.epi = EPI_ATOMIC; c.apacked = true; add(c); }
  { Case c; c.name = "tn_ALLpacked_kgather"; c.M = 384; c.N = 192; c.K = 3008; c.a_mn = true; c.b_mn = true; c.sched = SCHED_SPLITK; c.k_splits = 5; c.epi = EPI_ATOMIC; c.kgather = true; c.apacked = true; add(c); }
  { Case c; c.name = "nt_packed";         c.M = 1000; c.N = 384; c.K = 96;  c.packed = true; c.epi = EPI_BIAS | EPI_GELU; add(c); }
  { Case c; c.name = "nt_packed_ktail48"; c.M = 333; c.N = 96;  c.K = 48;  c.packed = true; add(c); }
  { Case c; c.name = "nt_packed_bigK";    c.M = 256; c.N = 768; c.K = 3072; c.packed = true; add(c); }
  { Case c; c.name = "nn_packed (dgrad)"; c.M = 450; c.N = 384; c.K = 96;  c.b_mn = true; c.packed = true; c.epi = EPI_DGELU; add(c); }
  { Case c; c.name = "nn_packed_bn192";   c.M = 130; c.N = 192; c.K = 768; c.b_mn = true; c.packed = true; add(c); }
  { Case c; c.name = "grouped_packed_gather"; c.M = 1024; c.N = 384; c.K = 96; c.sched = SCHED_GROUPED; c.groups = 3; c.gather = true; c.packed = true; c.epi = EPI_BIAS | EPI_GELU; add(c); }
  { Case c; c.name = "grouped_nn_packed"; c.M = 640; c.N = 96; c.K = 384; c.sched = SCHED_GROUPED; c.groups = 4; c.b_mn = true; c.packed = true; add(c); }
  { Case c; c.name = "grouped_nt_gelu";    c.M = 1024; c.N = 384; c.K = 96; c.sched = SCHED_GROUPED; c.groups = 3; c.gather = true; c.epi = EPI_BIAS | EPI_GELU; add(c); }
  { Case c; c.name = "grouped_nn";         c.M = 640; c.N = 96; c.K = 384; c.sched = SCHED_GROUPED; c.groups = 4; c.b_mn = true; add(c); }
  if (!only_bench) for (auto& c : cases) run(c);
  if (!quick) {
    int bi = 0;
#define B_(...) do { if (bench_idx < 0 || bench_idx == bi) bench(__VA_ARGS__); ++bi; } while (0)
    B_("ffn1 stage2 ALLPACKED", 32768, 1536, 384, false, false, EPI_BIAS | EPI_GELU, SCHED_DENSE, 1, true, true);
    B_("ffn2 stage2 ALLPACKED", 32768, 384, 1536, false, false, EPI_BIAS, SCHED_DENSE, 1, true, true);
    B_("ffn1 stage0 ALLPACKED", 524288, 384, 96, false, false, EPI_BIAS | EPI_GELU, SCHED_DENSE, 1, true, true);
    B_("ffn2 stage0 ALLPACKED", 524288, 96, 384, false, false, EPI_BIAS, SCHED_DENSE, 1, true, true);
    B_("ffn1 stage3 ALLPACKED", 8192, 3072, 768, false, false, EPI_BIAS, SCHED_DENSE, 1, true, true);
    B_("wgrad stage2 ALLPACKED", 1536, 384, 32768, true, true, EPI_ATOMIC, SCHED_SPLITK, 16, false, true);
    B_("wgrad stage0 ALLPACKED", 384, 96, 524288, true, true, EPI_ATOMIC, SCHED_SPLITK, 64, false, true);
    B_("square 8192 ALLPACKED", 8192, 8192, 8192, false, false, 0, SCHED_DENSE, 1, true, true);
    B_("ffn1 stage2 PACKED", 32768, 1536, 384, false, false, EPI_BIAS | EPI_GELU, SCHED_DENSE, 1, true);
    B_("ffn2 stage2 PACKED", 32768, 384, 1536, false, false, EPI_BIAS, SCHED_DENSE, 1, true);
    B_("ffn1 stage0 PACKED", 524288, 384, 96, false, false, EPI_BIAS | EPI_GELU, SCHED_DENSE, 1, true);
    B_("ffn2 stage0 PACKED", 524288, 96, 384, false, false, EPI_BIAS, SCHED_DENSE, 1, true);
    B_("ffn1 stage3 PACKED", 8192, 3072, 768, false, false, EPI_BIAS, SCHED_DENSE, 1, true);
    B_("dgrad stage2 PACKED", 32768, 384, 1536, false, true, 0, SCHED_DENSE, 1, true);
    B_("square 8192 PACKED", 8192, 8192, 8192, false, false, 0, SCHED_DENSE, 1, true);
    B_("ffn1 stage2 (gelu)", 32768, 1536, 384, false, false, EPI_BIAS | EPI_GELU);
    B_("ffn2 stage2", 32768, 384, 1536, false, false, EPI_BIAS);
    B_("ffn1 stage0 (gelu)", 524288, 384, 96, false, false, EPI_BIAS | EPI_GELU);
    B_("ffn2 stage0", 524288, 96, 384, false, false, EPI_BIAS);
    B_("ffn1 stage3", 8192, 3072, 768, false, false, EPI_BIAS);
    B_("ffn2 stage3", 8192, 768, 3072, false, false, EPI_BIAS);
    B_("dgrad stage2 (NN)", 32768, 384, 1536, false, true, 0);
    B_("wgrad stage2 (TN)", 1536, 384, 32768, true, true, EPI_ATOMIC, SCHED_SPLITK, 16);
    B_("square 8192", 8192, 8192, 8192, false, false, 0);
  }
  printf("SUMMARY: %d failed of %zu\n", g_fail, cases.size());
  return g_fail ? 1 : 0;
}
