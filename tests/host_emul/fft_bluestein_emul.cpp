// Host emulation of the Bluestein (chirp-z) mode of the two-pass FFT kernels (lama_b200/csrc/fft.cu, setup_tile and
// fft_dispatch<0, L, INV, true>), compiled with g++ against lama_b200/csrc/fft_core.cuh.  For every length 2..1024 that
// make_bluestein_plan routes to Bluestein, one CTA is emulated phase by phase (every worker of a phase runs before the
// next phase, as the barriers order them): the per-CTA filter spectrum over all threads, then per lane the chirp and
// zero pad, the m-point forward passes (compile-time Stockham, m = 512 / 1024 / 2048), the filter product, the m-point
// inverse passes and the final chirp.  Checked
// against a float64 DFT, relative to max |ref| of each lane:
//   * the row pass forward (two rows per lane, two-for-one split into half spectra),
//   * the row pass inverse (C2R rule on a NON-Hermitian half spectrum, two rows per lane),
//   * the column pass forward and inverse (complex),
// with 3 live lanes; the other lanes of the CTA are dead and carry zeros, as in the kernels.
// Usage: fft_bluestein_emul [verbose]      exit code 0 = every length within 2e-6 of max |ref|
//        fft_bluestein_emul plans          prints "n m lanes bluestein_cost direct_cost | radices of the runtime plan"
//                                          for n = 2..1024 (m = 0: the runtime plan runs; costs of the planner's model)
#include <algorithm>
#include <cmath>
#include <complex>
#include <cstdio>
#include <cstdlib>
#include <cstring>
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

// compile-time Stockham passes PASS.. of length N over `lanes` lanes and nw workers (fft.cu: stockham_passes)
template <int N, int PASS, bool INV, int LS>
static float2* stockham_passes(float2* x, float2* y, const float2* tw, int lanes, int nw) {
  if constexpr (PASS == Plan<N>::P) {
    return x;
  } else {
    for (int w = 0; w < nw; ++w)
      for (int lane = 0; lane < lanes; ++lane) stockham_pass<N, PASS, INV, LS>(x, y, tw, lane, w, nw);
    return stockham_passes<N, PASS + 1, INV, LS>(y, x, tw, lanes, nw);      // __syncthreads()
  }
}

// One CTA of the Bluestein mode: L lanes, `workers` workers per lane (fft.cu: make_plan), convolution length M.
template <int L, int M>
struct Cta {
  int n, m, workers;
  std::vector<float2> tw, chirp_f, chirp_i, filt_f, filt_i, a, b;

  Cta(int n_, const BluesteinPlan& bp) : n(n_), m(M) {
    workers = std::min((m + 7) / 8, 1024 / L);
    tw = twiddles(m);
    a.assign((size_t)m * L, make_float2(0.f, 0.f));
    b = a;
    setup<false>(chirp_f, filt_f);
    setup<true>(chirp_i, filt_i);
  }

  // m-point passes on every lane (LS lanes, nw workers); returns the buffer with the result
  template <bool INV, int LS>
  float2* passes(float2* x, float2* y, int lanes, int nw) {
    return stockham_passes<M, 0, INV, LS>(x, y, tw.data(), lanes, nw);
  }

  // fft.cu setup_tile<.., INV, true>: chirp table and filter spectrum / m, all L * workers threads on one transform
  template <bool INV>
  void setup(std::vector<float2>& chirp, std::vector<float2>& filt) {
    const int nthreads = L * workers;
    chirp.resize(n);
    filt.resize(m);
    for (int j = 0; j < n; ++j) chirp[j] = bluestein_chirp<INV>(j, n);
    for (int j = 0; j < m; ++j) filt[j] = bluestein_filter<INV>(j, n, m);
    const float2* f = passes<false, 1>(filt.data(), a.data(), 1, nthreads);
    const float inv_m = 1.0f / (float)m;
    std::vector<float2> s(m);
    for (int j = 0; j < m; ++j) s[j] = cscale(f[j], inv_m);
    filt = s;
  }

  // fft_dispatch<0, L, INV, true> on a.data() (points 0..n-1 staged); returns the buffer with the n results
  template <bool INV>
  const float2* transform() {
    const float2* chirp = INV ? chirp_i.data() : chirp_f.data();
    const float2* filt = INV ? filt_i.data() : filt_f.data();
    for (int w = 0; w < workers; ++w)
      for (int lane = 0; lane < L; ++lane) bluestein_pre<L>(a.data(), chirp, n, m, lane, w, workers);
    float2* f = passes<false, L>(a.data(), b.data(), L, workers);
    for (int w = 0; w < workers; ++w)
      for (int lane = 0; lane < L; ++lane) bluestein_mul<L>(f, filt, m, lane, w, workers);
    float2* g = passes<true, L>(f, f == a.data() ? b.data() : a.data(), L, workers);
    for (int w = 0; w < workers; ++w)
      for (int lane = 0; lane < L; ++lane) bluestein_post<L>(g, chirp, n, lane, w, workers);
    return g;
  }
};

static double rnd() { return rand() / (double)RAND_MAX * 2.0 - 1.0; }

// max over live lanes of max |got - ref| / max |ref|
struct Err {
  double e = 0, mag = 0;
  void add(cd ref, cd got) { e = std::max(e, std::abs(ref - got)); mag = std::max(mag, std::abs(ref)); }
  double rel() const { return e / (mag > 0 ? mag : 1.0); }
};

template <int L, int M>
static double check(int n, const BluesteinPlan& bp, bool verbose) {
  constexpr int kLive = 3;
  Cta<L, M> cta(n, bp);
  std::vector<cd> rw(n);
  for (int t = 0; t < n; ++t) rw[t] = std::polar(1.0, -2 * M_PI * t / n);
  auto dft = [&](const std::vector<cd>& x, bool inv) {
    std::vector<cd> y(n);
    for (int k = 0; k < n; ++k) {
      cd acc = 0;
      for (int j = 0; j < n; ++j) {
        const cd w = rw[((size_t)j * k) % n];
        acc += x[j] * (inv ? std::conj(w) : w);
      }
      y[k] = acc;
    }
    return y;
  };
  auto stage = [&](const std::vector<std::vector<cd>>& x) {      // kernels' staging: live lanes, dead lanes zero
    std::fill(cta.a.begin(), cta.a.end(), make_float2(0.f, 0.f));
    std::fill(cta.b.begin(), cta.b.end(), make_float2(1e30f, 1e30f));   // stale scratch must never be read
    for (int lane = 0; lane < kLive; ++lane)
      for (int j = 0; j < n; ++j) cta.a[(size_t)j * L + lane] = make_float2((float)x[lane][j].real(), (float)x[lane][j].imag());
  };
  const int wf = n / 2 + 1;
  double worst = 0;
  double errs[4];
  // ---- columns, forward and inverse: complex input per lane
  for (int dir = 0; dir < 2; ++dir) {
    std::vector<std::vector<cd>> x(kLive, std::vector<cd>(n));
    for (auto& v : x)
      for (auto& z : v) z = cd((float)rnd(), (float)rnd());
    stage(x);
    const float2* r = dir ? cta.template transform<true>() : cta.template transform<false>();
    Err e;
    for (int lane = 0; lane < kLive; ++lane) {
      const auto ref = dft(x[lane], dir == 1);
      for (int k = 0; k < n; ++k) e.add(ref[k], cd(r[(size_t)k * L + lane].x, r[(size_t)k * L + lane].y));
    }
    for (int lane = kLive; lane < L; ++lane)
      for (int k = 0; k < n; ++k) e.add(0.0, cd(r[(size_t)k * L + lane].x, r[(size_t)k * L + lane].y));
    errs[dir] = e.rel();
  }
  // ---- rows forward: z = row_a + i row_b, two-for-one split into the half spectra of both rows
  {
    std::vector<std::vector<cd>> ra(kLive, std::vector<cd>(n)), rb = ra, z = ra;
    for (int lane = 0; lane < kLive; ++lane)
      for (int j = 0; j < n; ++j) {
        ra[lane][j] = (float)rnd();
        rb[lane][j] = lane == 2 ? 0.0 : (float)rnd();     // lane 2: a last, unpaired row (row1 false)
        z[lane][j] = cd(ra[lane][j].real(), rb[lane][j].real());
      }
    stage(z);
    const float2* r = cta.template transform<false>();
    Err e;
    for (int lane = 0; lane < kLive; ++lane) {
      const auto A = dft(ra[lane], false), B = dft(rb[lane], false);
      for (int k = 0; k < wf; ++k) {
        float2 p, q;
        r2c_pair_post<L>(r, n, k, lane, p, q);
        e.add(A[k], cd(p.x, p.y));
        e.add(B[k], cd(q.x, q.y));
      }
    }
    errs[2] = e.rel();
  }
  // ---- rows inverse: C2R rule (Im of bin 0 and of the Nyquist bin ignored) on non-Hermitian half spectra
  {
    std::fill(cta.a.begin(), cta.a.end(), make_float2(0.f, 0.f));
    std::vector<std::vector<cd>> x1(kLive, std::vector<cd>(wf)), x2 = x1;
    for (int lane = 0; lane < kLive; ++lane)
      for (int k = 0; k < wf; ++k) {
        x1[lane][k] = cd(std::max(0.f, (float)rnd()), std::max(0.f, (float)rnd()));
        x2[lane][k] = cd(std::max(0.f, (float)rnd()), std::max(0.f, (float)rnd()));
      }
    for (int k = 0; k < wf; ++k)
      for (int lane = 0; lane < L; ++lane) {
        float2 p = make_float2(0.f, 0.f), q = p;
        if (lane < kLive) {
          p = make_float2((float)x1[lane][k].real(), (float)x1[lane][k].imag());
          q = make_float2((float)x2[lane][k].real(), (float)x2[lane][k].imag());
        }
        c2r_pair_pre<L>(cta.a.data(), n, k, lane, p, q);
      }
    const float2* r = cta.template transform<true>();
    Err e;
    const int last = (n % 2 == 0) ? wf - 1 : wf;
    for (int lane = 0; lane < kLive; ++lane)
      for (int j = 0; j < n; ++j) {
        double ya = x1[lane][0].real(), yb = x2[lane][0].real();
        for (int k = 1; k < last; ++k) {
          const cd w = std::conj(rw[((size_t)k * j) % n]);
          ya += 2.0 * (x1[lane][k] * w).real();
          yb += 2.0 * (x2[lane][k] * w).real();
        }
        if (n % 2 == 0) {
          ya += x1[lane][wf - 1].real() * ((j % 2) ? -1.0 : 1.0);
          yb += x2[lane][wf - 1].real() * ((j % 2) ? -1.0 : 1.0);
        }
        e.add(ya, r[(size_t)j * L + lane].x);
        e.add(yb, r[(size_t)j * L + lane].y);
      }
    errs[3] = e.rel();
  }
  for (double v : errs) worst = std::max(worst, v);
  if (verbose)
    printf("n=%4d m=%4d lanes %d workers %3d: cols fwd %.2e inv %.2e  rows fwd %.2e inv %.2e\n", n, cta.m, L,
           cta.workers, errs[0], errs[1], errs[2], errs[3]);
  return worst;
}

int main(int argc, char** argv) {
  if (argc > 1 && !strcmp(argv[1], "plans")) {
    for (int n = 2; n <= 1024; ++n) {
      const BluesteinPlan bp = make_bluestein_plan(n);
      const RtPlan rp = make_rt_plan(n);
      printf("%d %d %d %.0f %d |", n, bp.m, bp.lanes, bp.cost, bp.direct);
      for (int p = 0; p < rp.np; ++p) printf(" %d", rp.radix[p]);
      printf("\n");
    }
    return 0;
  }
  const bool verbose = argc > 1;
  double worst = 0;
  int count = 0, worst_n = 0;
  for (int n = 2; n <= 1024; ++n) {
    const BluesteinPlan bp = make_bluestein_plan(n);
    if (!bp.m) continue;
    if (bp.m < 2 * n - 1 || (bp.m != 512 && bp.m != 1024 && bp.m != 2048) || bp.m >= 4 * n - 2 || bluestein_smem(n, bp.m, bp.lanes) > kBluesteinSmemLimit ||
        bp.lanes != bluestein_lanes(n, bp.m)) {
      printf("bluestein plan(%d): m %d, %d lanes\n", n, bp.m, bp.lanes);
      return 3;
    }
    const double e = bp.m == 512 ? check<8, 512>(n, bp, verbose)
                     : bp.m == 1024 ? check<8, 1024>(n, bp, verbose) : check<4, 2048>(n, bp, verbose);
    if (e > worst) { worst = e; worst_n = n; }
    ++count;
  }
  printf("%d Bluestein lengths, worst relative error %.3e (n = %d)\n", count, worst, worst_n);
  return count > 0 && worst < 2e-6 ? 0 : 1;
}
