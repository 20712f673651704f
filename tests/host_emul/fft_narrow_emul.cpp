// Host emulation of the 8-channel two-pass FFT kernels (lama_b200/csrc/fft.cu, lengths 448..1024), compiled with g++
// against lama_b200/csrc/fft_core.cuh.  One CTA's shared-memory tile is data[point * 8 + lane]: every pass runs for
// all workers and all 8 lanes (lanes >= C are dead and carry zeros, as in the kernels), rows two at a time
// (two-for-one), the column pass over the half spectrum, the C2R rule on a NON-Hermitian spectrum.  Axes shorter
// than 448 points run the 32-channel orchestration (lane stride 32).  Each live lane is checked against a float64
// DFT.  Also checks the runtime radix planner for every length 321..1024.
// Usage: fft_narrow_emul [verbose]; exit code 0 = every plane within 2e-6 of max |ref|.
#include <algorithm>
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
    float a = 2.0f * (float)t / (float)n;       // device: sincospif(2t/n) in float
    tw[t] = make_float2((float)cos(M_PI * (double)a), (float)-sin(M_PI * (double)a));
  }
  return tw;
}

static int lanes_for(int n) { return 8 * (n + 64 * n) <= 227 * 1024 ? 32 : 8; }      // fft.cu: make_plan
static int workers_for_rt(int n, int lanes) {
  if (lanes == 8) return std::min((n + 7) / 8, 1024 / 8);
  return n > 64 ? std::min((n + 7) / 8, 32) : 8;
}

// fft.cu: fft_dispatch<0, LS, INV> over every lane and worker of one CTA.  Returns the buffer holding the result.
template <bool INV, int LS>
static float2* run_tile(int n, float2* a, float2* b, const float2* tw) {
  const RtPlan rp = make_rt_plan(n);
  const int nw = workers_for_rt(n, LS);
  int ns = 1;
  for (int p = 0; p < rp.np; ++p) {
    for (int w = 0; w < nw; ++w)
      for (int lane = 0; lane < LS; ++lane) generic_pass<INV, LS>(a, b, tw, n, rp.radix[p], ns, lane, w, nw);
    ns *= rp.radix[p];          // __syncthreads()
    std::swap(a, b);
  }
  return a;
}

template <bool INV>
static float2* run_axis(int n, int ls, float2* a, float2* b, const float2* tw) {
  return ls == 8 ? run_tile<INV, 8>(n, a, b, tw) : run_tile<INV, 32>(n, a, b, tw);
}

// One CTA per row pair / column, C live lanes.  x[c][y][w] real; returns max over lanes of the relative errors.
static double check(int H, int W, int C, bool verbose) {
  const int wf = W / 2 + 1, lw = lanes_for(W), lh = lanes_for(H);
  std::vector<float> x((size_t)C * H * W);
  for (auto& v : x) v = (float)(rand() / (double)RAND_MAX * 2.0 - 1.0);
  auto tww = twiddles(W), twh = twiddles(H);
  const int nmax = std::max(H, W);
  std::vector<float2> a((size_t)nmax * 32), b((size_t)nmax * 32);
  // ---- forward: rfft_rows_kernel<0, lw> then fft_cols_fwd_kernel<0, lh>;  ws[c][y][k]
  std::vector<float2> ws((size_t)C * H * wf), spec((size_t)C * H * wf);
  for (int y0 = 0; y0 < H; y0 += 2) {
    const bool row1 = y0 + 1 < H;
    for (int xx = 0; xx < W; ++xx)
      for (int lane = 0; lane < lw; ++lane) {
        float2 z = make_float2(0.f, 0.f);
        if (lane < C) z = make_float2(x[((size_t)lane * H + y0) * W + xx], row1 ? x[((size_t)lane * H + y0 + 1) * W + xx] : 0.f);
        a[(size_t)xx * lw + lane] = z;
      }
    const float2* r = run_axis<false>(W, lw, a.data(), b.data(), tww.data());
    for (int lane = 0; lane < C; ++lane)
      for (int k = 0; k < wf; ++k) {
        float2 p, q;
        if (lw == 8) r2c_pair_post<8>(r, W, k, lane, p, q); else r2c_pair_post<32>(r, W, k, lane, p, q);
        ws[((size_t)lane * H + y0) * wf + k] = p;
        if (row1) ws[((size_t)lane * H + y0 + 1) * wf + k] = q;
      }
  }
  const float scale = (float)(1.0 / std::sqrt((double)H * W));
  for (int k = 0; k < wf; ++k) {
    for (int y = 0; y < H; ++y)
      for (int lane = 0; lane < lh; ++lane)
        a[(size_t)y * lh + lane] = lane < C ? ws[((size_t)lane * H + y) * wf + k] : make_float2(0.f, 0.f);
    const float2* r = run_axis<false>(H, lh, a.data(), b.data(), twh.data());
    for (int lane = 0; lane < C; ++lane)
      for (int y = 0; y < H; ++y) {
        const float2 z = r[(size_t)y * lh + lane];
        spec[((size_t)lane * H + y) * wf + k] = make_float2(z.x * scale, z.y * scale);
      }
  }
  // ---- inverse of a NON-Hermitian (post-ReLU like) spectrum: fft_cols_inv_kernel<0, lh> then irfft_rows_kernel<0, lw>
  std::vector<float2> z((size_t)C * H * wf);
  for (auto& v : z) v = make_float2(std::max(0.f, (float)(rand() / (double)RAND_MAX * 2 - 1)),
                                    std::max(0.f, (float)(rand() / (double)RAND_MAX * 2 - 1)));
  for (int k = 0; k < wf; ++k) {
    for (int y = 0; y < H; ++y)
      for (int lane = 0; lane < lh; ++lane)
        a[(size_t)y * lh + lane] = lane < C ? z[((size_t)lane * H + y) * wf + k] : make_float2(0.f, 0.f);
    const float2* r = run_axis<true>(H, lh, a.data(), b.data(), twh.data());
    for (int lane = 0; lane < C; ++lane)
      for (int y = 0; y < H; ++y) ws[((size_t)lane * H + y) * wf + k] = r[(size_t)y * lh + lane];
  }
  std::vector<float> out((size_t)C * H * W);
  for (int y0 = 0; y0 < H; y0 += 2) {
    const bool row1 = y0 + 1 < H;
    for (int k = 0; k < wf; ++k)
      for (int lane = 0; lane < lw; ++lane) {
        float2 x1 = make_float2(0.f, 0.f), x2 = make_float2(0.f, 0.f);
        if (lane < C) {
          x1 = ws[((size_t)lane * H + y0) * wf + k];
          if (row1) x2 = ws[((size_t)lane * H + y0 + 1) * wf + k];
        }
        if (lw == 8) c2r_pair_pre<8>(a.data(), W, k, lane, x1, x2); else c2r_pair_pre<32>(a.data(), W, k, lane, x1, x2);
      }
    const float2* r = run_axis<true>(W, lw, a.data(), b.data(), tww.data());
    for (int lane = 0; lane < C; ++lane)
      for (int xx = 0; xx < W; ++xx) {
        const float2 q = r[(size_t)xx * lw + lane];
        out[((size_t)lane * H + y0) * W + xx] = q.x * scale;
        if (row1) out[((size_t)lane * H + y0 + 1) * W + xx] = q.y * scale;
      }
  }
  // ---- float64 references, separable with tabulated roots of unity
  std::vector<cd> rw(W), rh(H);
  for (int t = 0; t < W; ++t) rw[t] = std::polar(1.0, -2 * M_PI * t / W);
  for (int t = 0; t < H; ++t) rh[t] = std::polar(1.0, -2 * M_PI * t / H);
  double worst = 0, ef_all = 0, ei_all = 0;
  for (int c = 0; c < C; ++c) {
    const float* xc = x.data() + (size_t)c * H * W;
    std::vector<cd> rowdft((size_t)H * wf);
    for (int y = 0; y < H; ++y)
      for (int kx = 0; kx < wf; ++kx) {
        cd acc = 0;
        for (int xx = 0; xx < W; ++xx) acc += (double)xc[(size_t)y * W + xx] * rw[((size_t)kx * xx) % W];
        rowdft[(size_t)y * wf + kx] = acc;
      }
    double err_f = 0, mag = 0;
    std::vector<cd> col(H);
    for (int kx = 0; kx < wf; ++kx) {
      for (int y = 0; y < H; ++y) col[y] = rowdft[(size_t)y * wf + kx];
      for (int ky = 0; ky < H; ++ky) {
        cd acc = 0;
        for (int y = 0; y < H; ++y) acc += col[y] * rh[((size_t)ky * y) % H];
        acc /= std::sqrt((double)H * W);
        const float2 g = spec[((size_t)c * H + ky) * wf + kx];
        err_f = std::max(err_f, std::abs(acc - cd(g.x, g.y)));
        mag = std::max(mag, std::abs(acc));
      }
    }
    // inverse along H (all columns), then C2R along W dropping Im of bins 0 and W/2
    std::vector<cd> t((size_t)H * wf);
    for (int k = 0; k < wf; ++k) {
      for (int q = 0; q < H; ++q) { const float2 v = z[((size_t)c * H + q) * wf + k]; col[q] = cd(v.x, v.y); }
      for (int y = 0; y < H; ++y) {
        cd acc = 0;
        for (int q = 0; q < H; ++q) acc += col[q] * std::conj(rh[((size_t)q * y) % H]);
        t[(size_t)y * wf + k] = acc / std::sqrt((double)H);
      }
    }
    double err_i = 0, mag_i = 0;
    const int last = (W % 2 == 0) ? wf - 1 : wf;
    for (int y = 0; y < H; ++y)
      for (int n = 0; n < W; ++n) {
        double acc = t[(size_t)y * wf].real();
        for (int k = 1; k < last; ++k) acc += 2.0 * (t[(size_t)y * wf + k] * std::conj(rw[((size_t)k * n) % W])).real();
        if (W % 2 == 0) acc += t[(size_t)y * wf + wf - 1].real() * ((n % 2) ? -1.0 : 1.0);
        acc /= std::sqrt((double)W);
        err_i = std::max(err_i, std::abs(acc - (double)out[((size_t)c * H + y) * W + n]));
        mag_i = std::max(mag_i, std::abs(acc));
      }
    ef_all = std::max(ef_all, err_f / mag);
    ei_all = std::max(ei_all, err_i / mag_i);
  }
  worst = std::max(ef_all, ei_all);
  if (verbose)
    printf("H=%4d W=%4d C=%d (lanes %2d x %2d)  fwd %.2e  inv %.2e  (relative to max |ref|)\n", H, W, C, lh, lw, ef_all,
           ei_all);
  return worst;
}

int main(int argc, char** argv) {
  const bool verbose = argc > 1;
  for (int n = 2; n <= 1024; ++n) {          // every plan multiplies back to n with at most kMaxRtPasses radices >= 2
    const RtPlan rp = make_rt_plan(n);
    int prod = 1;
    for (int p = 0; p < rp.np; ++p) {
      if (rp.radix[p] < 2) { printf("plan(%d): radix %d\n", n, rp.radix[p]); return 3; }
      prod *= rp.radix[p];
    }
    if (prod != n || rp.np < 1 || rp.np > kMaxRtPasses) { printf("plan(%d) broken\n", n); return 3; }
    if (verbose && n > 320 && (n % 32 == 0 || n == 479 || n == 1021)) {
      printf("plan(%4d) =", n);
      for (int p = 0; p < rp.np; ++p) printf(" %d", rp.radix[p]);
      printf("\n");
    }
  }
  double worst = 0;
  // every length both as the row axis and as the column axis; primes run the direct DFT (a single radix-n pass)
  const int lens[] = {448, 480, 500, 512, 540, 750, 960, 1000, 1024, 449, 479, 1021};
  for (int n : lens) {
    worst = std::max(worst, check(7, n, 5, verbose));
    worst = std::max(worst, check(n, 10, 8, verbose));
  }
  // mixed planes: bottlenecks of 3840x2160, 4000x3000 photos, a 32-channel column axis beside an 8-channel row axis
  const int planes[][3] = {{270, 480, 3}, {375, 500, 2}, {448, 96, 4}, {479, 270, 2}};
  for (auto& p : planes) worst = std::max(worst, check(p[0], p[1], p[2], verbose));
  printf("worst relative error %.3e\n", worst);
  return worst < 2e-6 ? 0 : 1;
}
