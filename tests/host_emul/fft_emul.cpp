// Host emulation of the FFT kernels' arithmetic (lama_b200/csrc/fft_core.cuh compiled with g++).
// For each (H, W) it runs rfft2 -> spectrum and spectrum -> irfft2 the way fft.cu orchestrates
// the passes (two-for-one rows, column pass, C2R rule) for ONE lane and checks against a
// double-precision DFT.  Exit code 0 = all sizes within tolerance.  Usage: fft_emul [verbose]
#include <cmath>
#include <complex>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../lama_b200/csrc/fft_core.cuh"

using namespace ffcb::fftc;
typedef std::complex<double> cd;

static std::vector<float2> twiddles(int n) {
  std::vector<float2> tw(n);
  for (int t = 0; t < n; ++t) {
    // device: sincospif(2t/n) in float
    float a = 2.0f * (float)t / (float)n;
    tw[t] = make_float2((float)cos(M_PI * (double)a), (float)-sin(M_PI * (double)a));
  }
  return tw;
}

static bool g_mixed_radix = false;

template <int N, bool INV>
static float2* run_pow2(float2* a, float2* b, const float2* tw) {
  const int nw = workers_for(N);
  for (int w = 0; w < nw; ++w) stockham_pass<N, 0, INV, 1>(a, b, tw, 0, w, nw);
  if (Plan<N>::P == 1) return b;
  for (int w = 0; w < nw; ++w) stockham_pass<N, 1, INV, 1>(b, a, tw, 0, w, nw);
  if (Plan<N>::P == 2) return a;
  for (int w = 0; w < nw; ++w) stockham_pass<N, 2, INV, 1>(a, b, tw, 0, w, nw);
  return b;
}

template <bool INV>
static float2* run_any(int n, float2* a, float2* b, const float2* tw) {
  bool pow2 = (n & (n - 1)) == 0 && n >= 4 && n <= 256;
  if (pow2) {
    switch (n) {
      case 4: return run_pow2<4, INV>(a, b, tw);
      case 8: return run_pow2<8, INV>(a, b, tw);
      case 16: return run_pow2<16, INV>(a, b, tw);
      case 32: return run_pow2<32, INV>(a, b, tw);
      case 64: return run_pow2<64, INV>(a, b, tw);
      case 128: return run_pow2<128, INV>(a, b, tw);
      case 256: return run_pow2<256, INV>(a, b, tw);
    }
  }
  if (!g_mixed_radix) {
    const int nw = 8;
    for (int w = 0; w < nw; ++w) dft_pass<INV, 1>(a, b, tw, n, 0, w, nw);
    return b;
  }
  // runtime mixed-radix Stockham (fft.cu: fft_dispatch<0> with an RtPlan)
  const RtPlan rp = make_rt_plan(n);
  const int nw = 12;
  int ns = 1, prod = 1;
  for (int p = 0; p < rp.np; ++p) {
    for (int w = 0; w < nw; ++w) generic_pass<INV, 1>(a, b, tw, n, rp.radix[p], ns, 0, w, nw);
    ns *= rp.radix[p];
    prod *= rp.radix[p];
    std::swap(a, b);
  }
  if (prod != (n < 2 ? 1 : n)) { printf("bad plan for n=%d\n", n); exit(2); }
  return a;
}

static double check(int H, int W, bool verbose) {
  const int wf = W / 2 + 1;
  std::vector<float> x(H * W);
  for (auto& v : x) v = (float)(rand() / (double)RAND_MAX * 2.0 - 1.0);
  // ---- forward (rfft_rows_kernel + fft_cols_fwd_kernel)
  std::vector<float2> ws(H * wf), spec(H * wf);
  auto tww = twiddles(W), twh = twiddles(H);
  std::vector<float2> a(std::max(H, W)), b(std::max(H, W));
  for (int y0 = 0; y0 < H; y0 += 2) {
    const bool row1 = y0 + 1 < H;
    for (int xx = 0; xx < W; ++xx) a[xx] = make_float2(x[y0 * W + xx], row1 ? x[(y0 + 1) * W + xx] : 0.f);
    const float2* r = run_any<false>(W, a.data(), b.data(), tww.data());
    for (int k = 0; k < wf; ++k) {
      float2 p, q;
      r2c_pair_post<1>(r, W, k, 0, p, q);
      ws[y0 * wf + k] = p;
      if (row1) ws[(y0 + 1) * wf + k] = q;
    }
  }
  const float scale = (float)(1.0 / std::sqrt((double)H * W));
  for (int k = 0; k < wf; ++k) {
    for (int y = 0; y < H; ++y) a[y] = ws[y * wf + k];
    const float2* r = run_any<false>(H, a.data(), b.data(), twh.data());
    for (int y = 0; y < H; ++y) spec[y * wf + k] = make_float2(r[y].x * scale, r[y].y * scale);
  }
  // double-precision reference, separable (row DFT, then column DFT) with tabulated roots of unity
  std::vector<cd> rw(W), rh(H);
  for (int t = 0; t < W; ++t) rw[t] = std::polar(1.0, -2 * M_PI * t / W);
  for (int t = 0; t < H; ++t) rh[t] = std::polar(1.0, -2 * M_PI * t / H);
  std::vector<cd> rowdft(H * wf);
  for (int y = 0; y < H; ++y)
    for (int kx = 0; kx < wf; ++kx) {
      cd acc = 0;
      for (int xx = 0; xx < W; ++xx) acc += (double)x[y * W + xx] * rw[(kx * xx) % W];
      rowdft[y * wf + kx] = acc;
    }
  double err_f = 0, mag = 0;
  for (int ky = 0; ky < H; ++ky)
    for (int kx = 0; kx < wf; ++kx) {
      cd acc = 0;
      for (int y = 0; y < H; ++y) acc += rowdft[y * wf + kx] * rh[(ky * y) % H];
      acc /= std::sqrt((double)H * W);
      err_f = std::max(err_f, std::abs(acc - cd(spec[ky * wf + kx].x, spec[ky * wf + kx].y)));
      mag = std::max(mag, std::abs(acc));
    }
  // ---- inverse on a NON-Hermitian spectrum (post-ReLU like): fft_cols_inv_kernel + irfft_rows_kernel
  std::vector<float2> z(H * wf);
  for (auto& v : z) v = make_float2(std::max(0.f, (float)(rand() / (double)RAND_MAX * 2 - 1)),
                                    std::max(0.f, (float)(rand() / (double)RAND_MAX * 2 - 1)));
  for (int k = 0; k < wf; ++k) {
    for (int y = 0; y < H; ++y) a[y] = z[y * wf + k];
    const float2* r = run_any<true>(H, a.data(), b.data(), twh.data());
    for (int y = 0; y < H; ++y) ws[y * wf + k] = r[y];
  }
  std::vector<float> out(H * W);
  for (int y0 = 0; y0 < H; y0 += 2) {
    const bool row1 = y0 + 1 < H;
    for (int k = 0; k < wf; ++k)
      c2r_pair_pre<1>(a.data(), W, k, 0, ws[y0 * wf + k], row1 ? ws[(y0 + 1) * wf + k] : make_float2(0.f, 0.f));
    const float2* r = run_any<true>(W, a.data(), b.data(), tww.data());
    for (int xx = 0; xx < W; ++xx) {
      out[y0 * W + xx] = r[xx].x * scale;
      if (row1) out[(y0 + 1) * W + xx] = r[xx].y * scale;
    }
  }
  // reference: inverse along H (all columns), then C2R along W dropping Im of bins 0 and W/2
  double err_i = 0, mag_i = 0;
  std::vector<cd> t(H * wf);
  for (int k = 0; k < wf; ++k)
    for (int y = 0; y < H; ++y) {
      cd acc = 0;
      for (int q = 0; q < H; ++q) acc += cd(z[q * wf + k].x, z[q * wf + k].y) * std::conj(rh[(q * y) % H]);
      t[y * wf + k] = acc / std::sqrt((double)H);
    }
  for (int y = 0; y < H; ++y)
    for (int n = 0; n < W; ++n) {
      double acc = t[y * wf].real();
      const int last = (W % 2 == 0) ? wf - 1 : wf;
      for (int k = 1; k < last; ++k) acc += 2.0 * (t[y * wf + k] * std::conj(rw[(k * n) % W])).real();
      if (W % 2 == 0) acc += t[y * wf + wf - 1].real() * ((n % 2) ? -1.0 : 1.0);
      acc /= std::sqrt((double)W);
      err_i = std::max(err_i, std::abs(acc - (double)out[y * W + n]));
      mag_i = std::max(mag_i, std::abs(acc));
    }
  const double rel = std::max(err_f / mag, err_i / mag_i);
  if (verbose) printf("H=%3d W=%3d  fwd %.2e / %.2e   inv %.2e / %.2e\n", H, W, err_f, mag, err_i, mag_i);
  return rel;
}

// rfft2_plane64_kernel (fft_plane.cu): same per-thread functors, one channel, S[y][kx] — the 32 row-pair tasks, then
// one complex column task for each of the 33 columns.
static double check_plane64(bool verbose) {
  const int N = 64, WF = 33;
  std::vector<float> x(N * N);
  for (auto& v : x) v = (float)(rand() / (double)RAND_MAX * 2.0 - 1.0);
  std::vector<float2> S(N * WF), spec(N * WF);
  const float scale = 1.0f / 64.0f;
  for (int g = 0; g < 32; ++g)
    plane64_rows_fwd([&](int n) { return make_float2(x[(2 * g) * N + n], x[(2 * g + 1) * N + n]); },
                     [&](int k, float2 a, float2 b) { S[(2 * g) * WF + k] = a; S[(2 * g + 1) * WF + k] = b; });
  for (int kx = 0; kx < WF; ++kx)
    plane64_col<false>([&](int y) { return S[y * WF + kx]; },
                       [&](int ky, float2 z) { spec[ky * WF + kx] = make_float2(z.x * scale, z.y * scale); });
  double err_f = 0, mag = 0;
  for (int ky = 0; ky < N; ++ky)
    for (int kx = 0; kx < WF; ++kx) {
      cd acc = 0;
      for (int y = 0; y < N; ++y)
        for (int xx = 0; xx < N; ++xx)
          acc += (double)x[y * N + xx] * std::polar(1.0, -2 * M_PI * ((double)ky * y / N + (double)kx * xx / N));
      acc /= 64.0;
      err_f = std::max(err_f, std::abs(acc - cd(spec[ky * WF + kx].x, spec[ky * WF + kx].y)));
      mag = std::max(mag, std::abs(acc));
    }
  if (verbose) printf("plane64 forward   %.2e / %.2e\n", err_f, mag);
  return err_f / mag;
}

// irfft2_plane64_v2_kernel (fft_plane.cu): emulate ONE CTA (8 channels) thread by thread, phase by phase, with the
// kernel's index expressions: column tasks -> S, row tasks -> results staged in place of their rows (after every
// thread of the row's group has its inputs in registers), channels-last epilogue slots -> output (+ residual).
static double check_plane64_inv_v2(bool verbose) {
  const int N = 64, WF = 33, CH = 8, P = kP64Pitch;
  std::vector<float> spec((size_t)N * WF * 2 * CH), res((size_t)N * N * CH), out((size_t)N * N * CH, -1e30f);
  for (auto& v : spec) v = std::max(0.f, (float)(rand() / (double)RAND_MAX * 2 - 1));
  for (auto& v : res) v = (float)(rand() / (double)RAND_MAX);
  const unsigned spec_sx = 2 * CH, spec_sy = WF * 2 * CH, res_sx = CH, res_sy = N * CH;
  const float scale = 1.0f / 64.0f;
  std::vector<float2> S((size_t)N * P, make_float2(1e30f, 1e30f));
  for (int tid = 0; tid < WF * CH; ++tid) {           // phase A
    const int c = tid & 7, g = tid >> 3;
    const unsigned o0 = (unsigned)g * spec_sx + 2u * c;
    plane64_col<true>([&](int ky) { const float* q = spec.data() + (o0 + (unsigned)ky * spec_sy); return make_float2(q[0], q[1]); },
                      [&](int y, float2 z) { S[y * P + g * 8 + c] = z; });
  }
  float* R = reinterpret_cast<float*>(S.data());
  for (int warp = 0; warp < 8; ++warp) {              // phase B, one warp at a time: compute all lanes, then write
    std::vector<float2> held(32 * 64);
    for (int lane = 0; lane < 32; ++lane) {
      const int tid = warp * 32 + lane, c = tid & 7, g = tid >> 3;
      plane64_rows_inv([&](int k, float2& x1, float2& x2) { x1 = S[(2 * g) * P + k * 8 + c]; x2 = S[(2 * g + 1) * P + k * 8 + c]; },
                       [&](int n0, const float2* zb) { for (int j = 0; j < 16; ++j) held[lane * 64 + n0 + j] = zb[j]; });
    }
    for (int lane = 0; lane < 32; ++lane) {
      const int tid = warp * 32 + lane, c = tid & 7, g = tid >> 3;
      for (int n = 0; n < 64; ++n) {
        R[p64_stage_index(2 * g, n, c)] = held[lane * 64 + n].x;
        R[p64_stage_index(2 * g + 1, n, c)] = held[lane * 64 + n].y;
      }
    }
    for (int lane = 0; lane < 32; ++lane)             // phase C
      for (int i = 0; i < 16; ++i) {
        int row, x;
        p64_store_slot(warp, lane, i, row, x);
        for (int c = 0; c < CH; ++c)
          out[(size_t)row * res_sy + x * res_sx + c] =
              std::fma(R[p64_stage_index(row, x, 0) + c], scale, res[(size_t)row * res_sy + x * res_sx + c]);
      }
  }
  double err = 0, mag = 0;
  for (int c = 0; c < CH; ++c) {
    std::vector<cd> t(N * WF);
    for (int k = 0; k < WF; ++k)
      for (int y = 0; y < N; ++y) {
        cd acc = 0;
        for (int q = 0; q < N; ++q)
          acc += cd(spec[(size_t)q * spec_sy + k * spec_sx + 2 * c], spec[(size_t)q * spec_sy + k * spec_sx + 2 * c + 1]) *
                 std::polar(1.0, 2 * M_PI * (double)q * y / N);
        t[y * WF + k] = acc / 8.0;
      }
    for (int y = 0; y < N; ++y)
      for (int n = 0; n < N; ++n) {
        double acc = t[y * WF].real();
        for (int k = 1; k < 32; ++k) acc += 2.0 * (t[y * WF + k] * std::polar(1.0, 2 * M_PI * (double)k * n / N)).real();
        acc += t[y * WF + 32].real() * ((n % 2) ? -1.0 : 1.0);
        acc = acc / 8.0 + res[(size_t)y * res_sy + n * res_sx + c];
        err = std::max(err, std::abs(acc - (double)out[(size_t)y * res_sy + n * res_sx + c]));
        mag = std::max(mag, std::abs(acc));
      }
  }
  if (verbose) printf("plane64 inverse v2 (one CTA, 8 channels)   %.2e / %.2e\n", err, mag);
  return err / mag;
}

int main(int argc, char** argv) {
  const bool verbose = argc > 1;
  const int sizes[][2] = {{4, 4}, {8, 8}, {16, 16}, {32, 32}, {64, 64}, {128, 128}, {256, 256}, {8, 32}, {64, 16},
                          {256, 4}, {15, 15}, {6, 9}, {20, 24}, {5, 9}, {7, 6}, {3, 2}, {1, 8}, {2, 2}, {125, 188},
                          {64, 33}, {9, 64}};
  double worst = 0;
  for (auto& s : sizes) worst = std::max(worst, check(s[0], s[1], verbose));
  worst = std::max(worst, check_plane64(verbose));
  worst = std::max(worst, check_plane64_inv_v2(verbose));
  // runtime mixed-radix plans (row f2): composite, prime-power, prime and large-prime-factor lengths
  g_mixed_radix = true;
  const int mixed[][2] = {{15, 15}, {6, 9}, {20, 24}, {5, 9}, {7, 6}, {3, 2}, {1, 8}, {2, 2}, {125, 188}, {96, 128},
                          {135, 240}, {100, 36}, {47, 94}, {243, 12}, {27, 250}, {49, 98}, {192, 160}, {13, 26}};
  for (auto& s : mixed) worst = std::max(worst, check(s[0], s[1], verbose));
  for (int n = 2; n <= 320; ++n) {            // every plan multiplies back to n with radices >= 2
    const RtPlan rp = make_rt_plan(n);
    int prod = 1, sum = 0;
    for (int p = 0; p < rp.np; ++p) { prod *= rp.radix[p]; sum += rp.radix[p]; if (rp.radix[p] < 2) return 3; }
    if (prod != n || rp.np > kMaxRtPasses) { printf("plan(%d) broken\n", n); return 3; }
    if (verbose && (n % 8 == 0)) { printf("plan(%3d) =", n); for (int p = 0; p < rp.np; ++p) printf(" %d", rp.radix[p]); printf("  (sum %d)\n", sum); }
  }
  printf("worst relative error %.3e\n", worst);
  return worst < 2e-6 ? 0 : 1;
}
