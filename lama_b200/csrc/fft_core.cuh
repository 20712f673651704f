// FFT arithmetic shared by the CUDA kernels (fft.cu) and the host emulation test
// (tests/host_emul/fft_emul.cpp compiles this header with g++ and checks every size against a
// double-precision DFT — the kernels' index algebra is verified on the CPU-only build box).
//
// Data layout: data[point * LS + lane], LS = lane stride (32 on the device: lane == channel).
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdlib.h>
#include <vector_functions.h>
#include <vector_types.h>

#if defined(__CUDACC__)
#define FFCB_HD __host__ __device__ __forceinline__
#else
#define FFCB_HD inline
#endif

namespace ffcb {
namespace fftc {

// Complex arithmetic: IEEE round-to-nearest fp32 add / mul / fma.  The multiply rounds a.x*b first and fuses the
// a.y term into it, so every build (and the host emulation in tests/host_emul) rounds the same way.
FFCB_HD float2 cmul(float2 a, float2 b) {
  return make_float2(fmaf(-a.y, b.y, a.x * b.x), fmaf(a.y, b.x, a.x * b.y));
}
FFCB_HD float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
FFCB_HD float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
FFCB_HD float2 cscale(float2 a, float s) { return make_float2(a.x * s, a.y * s); }

// multiply by -i (forward transform) or +i (inverse)
template <bool INV>
FFCB_HD float2 mul_mi(float2 a) {
  return INV ? make_float2(-a.y, a.x) : make_float2(a.y, -a.x);
}

template <bool INV>
FFCB_HD void fft2(float2& a, float2& b) {
  float2 t = a;
  a = cadd(t, b);
  b = csub(t, b);
}

template <bool INV>
FFCB_HD void fft4(float2& v0, float2& v1, float2& v2, float2& v3) {
  float2 t0 = cadd(v0, v2), t1 = csub(v0, v2), t2 = cadd(v1, v3), t3 = mul_mi<INV>(csub(v1, v3));
  v0 = cadd(t0, t2);
  v2 = csub(t0, t2);
  v1 = cadd(t1, t3);
  v3 = csub(t1, t3);
}

template <bool INV>
FFCB_HD void fft8(float2* v) {
  fft4<INV>(v[0], v[2], v[4], v[6]);  // E[0..3] -> v[0], v[2], v[4], v[6]
  fft4<INV>(v[1], v[3], v[5], v[7]);  // O[0..3] -> v[1], v[3], v[5], v[7]
  const float h = 0.70710678118654752440f;
  float2 o1, o2, o3;  // w^q * O[q], w = exp(-+ 2 pi i / 8):  w^1 z = h (z -+ i z),  w^2 z = -+ i z,  w^3 z = h (-z -+ i z)
  if (INV) {
    o1 = cscale(cadd(v[3], make_float2(-v[3].y, v[3].x)), h);        // h (z + i z)
    o2 = make_float2(-v[5].y, v[5].x);                               // i z
    o3 = cscale(csub(make_float2(-v[7].y, v[7].x), v[7]), h);        // h (i z - z)
  } else {
    o1 = cscale(cadd(v[3], make_float2(v[3].y, -v[3].x)), h);        // h (z - i z)
    o2 = make_float2(v[5].y, -v[5].x);                               // -i z
    o3 = cscale(csub(make_float2(v[7].y, -v[7].x), v[7]), h);        // h (-i z - z)
  }
  const float2 e0 = v[0], e1 = v[2], e2 = v[4], e3 = v[6], o0 = v[1];
  v[0] = cadd(e0, o0); v[4] = csub(e0, o0);
  v[1] = cadd(e1, o1); v[5] = csub(e1, o1);
  v[2] = cadd(e2, o2); v[6] = csub(e2, o2);
  v[3] = cadd(e3, o3); v[7] = csub(e3, o3);
}

// Radix plan of the mixed-radix Stockham autosort, per power-of-two length.
template <int N> struct Plan;
template <> struct Plan<4>   { static constexpr int P = 1; static constexpr int R[3] = {4, 1, 1}; };
template <> struct Plan<8>   { static constexpr int P = 1; static constexpr int R[3] = {8, 1, 1}; };
template <> struct Plan<16>  { static constexpr int P = 2; static constexpr int R[3] = {4, 4, 1}; };
template <> struct Plan<32>  { static constexpr int P = 2; static constexpr int R[3] = {8, 4, 1}; };
template <> struct Plan<64>  { static constexpr int P = 2; static constexpr int R[3] = {8, 8, 1}; };
template <> struct Plan<128> { static constexpr int P = 3; static constexpr int R[3] = {8, 4, 4}; };
template <> struct Plan<256> { static constexpr int P = 3; static constexpr int R[3] = {8, 8, 4}; };
// convolution lengths of the Bluestein transforms (below)
template <> struct Plan<512>  { static constexpr int P = 3; static constexpr int R[3] = {8, 8, 8}; };
template <> struct Plan<1024> { static constexpr int P = 4; static constexpr int R[4] = {8, 8, 4, 4}; };
template <> struct Plan<2048> { static constexpr int P = 4; static constexpr int R[4] = {8, 8, 8, 4}; };

template <int N, int PASS> constexpr int plan_radix() { return Plan<N>::R[PASS]; }
template <int N, int PASS> constexpr int plan_ns() {
  int ns = 1;
  for (int i = 0; i < PASS; ++i) ns *= Plan<N>::R[i];
  return ns;
}
// worker threads per transform the kernels launch with
constexpr int workers_for(int n) { return n >= 8 ? n / 8 : 1; }

// One out-of-place Stockham pass (src -> dst) for one lane, butterflies j = worker, worker+nw, ...
// tw[t] = exp(-2 pi i t / N), t in [0, N).
template <int N, int PASS, bool INV, int LS>
FFCB_HD void stockham_pass(const float2* src, float2* dst, const float2* tw, int lane, int worker, int nworkers) {
  constexpr int R = plan_radix<N, PASS>();
  constexpr int NS = plan_ns<N, PASS>();
  constexpr int NB = N / R;
  for (int j = worker; j < NB; j += nworkers) {
    const int k = j % NS;
    float2 v[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float2 x = src[(j + r * NB) * LS + lane];
      if (NS > 1 && r > 0) {
        float2 w = tw[r * k * (N / (NS * R))];
        if (INV) w.y = -w.y;
        x = cmul(x, w);
      }
      v[r] = x;
    }
    if (R == 8) fft8<INV>(v);
    else if (R == 4) fft4<INV>(v[0], v[1], v[2], v[3]);
    else fft2<INV>(v[0], v[1]);
    const int j0 = (j - k) * R + k;
#pragma unroll
    for (int r = 0; r < R; ++r) dst[(j0 + r * NS) * LS + lane] = v[r];
  }
}

// Direct DFT of runtime length n (src -> dst), output bins k = worker, worker+nw, ...
template <bool INV, int LS>
FFCB_HD void dft_pass(const float2* src, float2* dst, const float2* tw, int n, int lane, int worker, int nworkers) {
  for (int k = worker; k < n; k += nworkers) {
    float2 acc = make_float2(0.f, 0.f);
    int t = 0;  // (k * m) mod n
    for (int m = 0; m < n; ++m) {
      float2 w = tw[t];
      if (INV) w.y = -w.y;
      const float2 x = src[m * LS + lane];
      acc.x += x.x * w.x - x.y * w.y;
      acc.y += x.x * w.y + x.y * w.x;
      t += k;
      if (t >= n) t -= n;
    }
    dst[k * LS + lane] = acc;
  }
}

// ---------------------------------------------------------------------------------------------
// Lengths without a compile-time plan (SURVEY.md row f2: bin/predict.py pads images to multiples of 8 only, so the
// bottleneck planes are e.g. 96x128, 135x240, 125x188): a runtime mixed-radix Stockham autosort.  The length is
// split into factors R_0 * R_1 * ... (any integers >= 2); pass p is the textbook radix-R_p Stockham step with the
// R-point butterfly evaluated directly, one output per iteration:
//   dst[j0 + q*NS] = sum_r src[j + r*n/R] * w_n^{ r * (k * n/(NS*R) + q * n/R) },  k = j mod NS, j0 = (j-k)*R + k
// so one transform costs n * sum_p R_p complex MACs instead of n^2 (a prime length degenerates to the direct DFT).
constexpr int kMaxRtPasses = 8;
struct RtPlan {
  int np;                    // number of passes; < 0: use dft_pass (single direct DFT)
  int radix[kMaxRtPasses];
};

// Factorisation minimising sum_p (R_p + 3) (the +3 prices a pass: barrier, index set-up, one smem round trip).
// Host only.
inline RtPlan make_rt_plan(int n) {
  RtPlan p;
  p.np = 0;
  for (int i = 0; i < kMaxRtPasses; ++i) p.radix[i] = 1;
  constexpr int kMaxN = 1024;
  if (n < 2) return p;
  if (n > kMaxN) { p.np = 1; p.radix[0] = n; return p; }
  static_assert(kMaxN <= 1024, "cost tables live on the stack");
  int cost[kMaxN + 1], pick[kMaxN + 1];
  cost[1] = 0; pick[1] = 1;
  for (int m = 2; m <= n; ++m) {
    if (n % m) continue;
    cost[m] = m + 3; pick[m] = m;
    for (int d = 2; d * 2 <= m; ++d) {
      if (m % d || n % (m / d)) continue;
      const int c = d + 3 + cost[m / d];
      if (c < cost[m]) { cost[m] = c; pick[m] = d; }
    }
  }
  int m = n, radices[32], cnt = 0;
  while (m > 1 && cnt < 32) { radices[cnt++] = pick[m]; m /= pick[m]; }
  // more factors than slots (cannot happen for n <= 1024, where at most 5 are chosen): merge the tail
  while (cnt > kMaxRtPasses) { radices[cnt - 2] *= radices[cnt - 1]; --cnt; }
  // largest radix first: the early passes (NS small) need no twiddle beyond the butterfly's own
  for (int i = 0; i < cnt; ++i)
    for (int j = i + 1; j < cnt; ++j)
      if (radices[j] > radices[i]) { const int t = radices[i]; radices[i] = radices[j]; radices[j] = t; }
  p.np = cnt;
  for (int i = 0; i < cnt; ++i) p.radix[i] = radices[i];
  return p;
}

// One runtime-radix Stockham pass (src -> dst) for one lane; outputs o = worker, worker+nw, ...
template <bool INV, int LS>
FFCB_HD void generic_pass(const float2* src, float2* dst, const float2* tw, int n, int R, int NS, int lane, int worker,
                          int nworkers) {
  const int NB = n / R;              // butterflies
  const int tws = n / (NS * R);      // twiddle exponent per unit of k
  for (int o = worker; o < n; o += nworkers) {
    const int q = o / NB, j = o - q * NB;
    const int k = j % NS;
    const int step = (k * tws + q * NB) % n;
    float2 acc = make_float2(0.f, 0.f);
    int t = 0;                       // (r * step) mod n
    const float2* s = src + j * LS + lane;
    for (int r = 0; r < R; ++r) {
      float2 w = tw[t];
      if (INV) w.y = -w.y;
      const float2 x = s[r * NB * LS];
      acc.x += x.x * w.x - x.y * w.y;
      acc.y += x.x * w.y + x.y * w.x;
      t += step;
      if (t >= n) t -= n;
    }
    dst[((j - k) * R + k + q * NS) * LS + lane] = acc;
  }
}

// Two-for-one real transforms.  z = row_a + i * row_b, Z = FFT(z) (length W, unnormalised):
//   A[k] = (Z[k] + conj(Z[-k])) / 2,  B[k] = (Z[k] - conj(Z[-k])) / (2i),  k = 0 .. W/2
template <int LS>
FFCB_HD void r2c_pair_post(const float2* z, int W, int k, int lane, float2& a, float2& b) {
  const float2 zk = z[k * LS + lane];
  const float2 zm = z[((W - k) % W) * LS + lane];
  a = make_float2(0.5f * (zk.x + zm.x), 0.5f * (zk.y - zm.y));
  b = make_float2(0.5f * (zk.y + zm.y), -0.5f * (zk.x - zm.x));
}

// Inverse: given half-spectra X1[k], X2[k] (k = 0..W/2) build Z with z = IFFT(Z) = row_a + i*row_b.
// Implements the C2R rule: Im of bin 0 and of the Nyquist bin (even W) is ignored.
template <int LS>
FFCB_HD void c2r_pair_pre(float2* z, int W, int k, int lane, float2 x1, float2 x2) {
  if (k == 0 || 2 * k == W) {
    z[k * LS + lane] = make_float2(x1.x, x2.x);
  } else {
    z[k * LS + lane] = make_float2(x1.x - x2.y, x1.y + x2.x);          // X1 + i X2
    z[(W - k) * LS + lane] = make_float2(x1.x + x2.y, x2.x - x1.y);    // conj(X1) + i conj(X2)
  }
}

// ---------------------------------------------------------------------------------------------
// Bluestein (chirp-z) transforms for runtime lengths with a large prime factor, where the runtime plan above costs
// nearly n^2.  With c[j] = exp(-+ i pi j^2 / n) (forward / inverse) and jk = (j^2 + k^2 - (k-j)^2) / 2:
//   X[k] = c[k] * sum_j (x[j] c[j]) conj(c[k-j])
// a cyclic convolution of the zero-padded chirped input with h[d] = conj(c[|d|]), evaluated at the power of two
// m >= 2n - 1 (512, 1024 or 2048) as IFFT_m(FFT_m(x c) * FFT_m(h)) / m.  Both m-point transforms run the compile-time
// radix-8/4 Stockham passes (stockham_pass, Plan<m>): register butterflies with no per-output index arithmetic, which
// is what makes Bluestein pay off against the runtime plans; a smooth m closer to 2n - 1 would run the generic passes,
// measured 2-3x slower per point.  The filter spectrum FFT_m(h) / m is the same for every lane: a CTA computes it once.
struct BluesteinPlan {
  int m;       // convolution length; 0: the runtime plan of n is cheaper
  int lanes;   // channels per CTA (bluestein_lanes)
  float cost;  // modelled cost of the Bluestein transform (0 for lengths it cannot serve)
  int direct;  // modelled cost of the runtime plan of n
};

// make_rt_plan's cost model: sum over passes of (R_p + 3) per point
inline int rt_plan_cost(int n, const RtPlan& p) {
  if (p.np < 0) return n * (n + 3);
  int s = 0;
  for (int i = 0; i < p.np; ++i) s += p.radix[i] + 3;
  return n * s;
}

// Shared memory of a Bluestein CTA: [twiddles m][chirp n][filter spectrum m][ping m * lanes | pong m * lanes] float2.
// 8 channels fit the 227 KB a CTA may hold for m = 512 and 1024 (152 KB at n = 512); m = 2048 takes 4 channels
// (172 KB at n = 1024), the widest layout that keeps the two m-long buffers per lane the out-of-place passes need.
constexpr int kBluesteinSmemLimit = 227 * 1024;
inline int bluestein_smem(int n, int m, int lanes) { return (int)sizeof(float2) * (2 * m + n + 2 * lanes * m); }
inline int bluestein_lanes(int n, int m) { return bluestein_smem(n, m, 8) <= kBluesteinSmemLimit ? 8 : 4; }

// Bluestein is taken when its modelled cost, times this factor, is below the runtime plan's.  The model prices a
// compile-time radix-R pass like a runtime one (R + 3 per point), which overstates it; the factor is the measured
// correction.  tools/fft_lengths_bench.py on an H100 timed every length this factor selects (311 of 129..1024, n x n
// planes of 192 channels, DESIGN §6): each ran the FFT pair 1.28x to 8.9x faster than its runtime plan.
constexpr float kBluesteinCostFactor = 0.5f;

// Plan for n: m = 0 when the runtime plan of n stays cheaper.  The model counts two m-point transforms, three
// point-wise passes (chirp + zero pad over m, filter over m, chirp over n; 4 per point, like a radix-1 pass) and the
// lane's share of the per-CTA filter transform.  Host only; no search, so it is cheap on every call.
inline BluesteinPlan make_bluestein_plan(int n) {
  BluesteinPlan b;
  b.m = 0;
  b.lanes = 0;
  b.cost = 0.f;
  b.direct = 0;
  if (n < 129 || n > 1024) return b;                    // m = 512 .. 2048
  b.direct = rt_plan_cost(n, make_rt_plan(n));
  int m = 512;
  while (m < 2 * n - 1) m *= 2;
  const int per_point = m == 512 ? 3 * (8 + 3) : (m == 1024 ? 2 * (8 + 3) + 2 * (4 + 3) : 3 * (8 + 3) + (4 + 3));
  const int lanes = bluestein_lanes(n, m);
  const float tm = (float)m * per_point;
  b.cost = 2.f * tm + 4.f * (2 * m + n) + tm / lanes;
  if (kBluesteinCostFactor * b.cost < (float)b.direct) { b.m = m; b.lanes = lanes; }
  return b;
}

// ---------------------------------------------------------------------------------------------
// Launch plan of one axis of the two-pass kernels (fft.cu), host only; tests/host_emul/fft_plan_emul.cpp prints it.
constexpr int kLanes = 32;        // channels per CTA of every length whose buffers fit
constexpr int kNarrowLanes = 8;   // channels per CTA of lengths 448..1024, and of Bluestein lengths up to n = 512

struct LaunchPlan {
  int N;       // template length (0 = runtime length)
  int n;       // runtime length
  int m;       // Bluestein convolution length: 512, 1024 or 2048 (n otherwise)
  bool bluestein;
  int lanes;   // channels per CTA: kLanes, or kNarrowLanes (N == 0 only); Bluestein: bluestein_lanes
  dim3 block;  // (lanes, workers, groups)
  size_t smem;
  RtPlan rp;   // N == 0 without Bluestein: runtime radix plan (np < 0: direct DFT)
};

// Lengths without a compile-time plan: runtime mixed-radix Stockham (FFCB_FFT_MIXED_RADIX=0 selects the O(n^2)
// direct DFT they ran in the first revision — same results to round-off, kept as the cross-check; it turns Bluestein
// off too).
inline bool mixed_radix_enabled() {
  const char* e = getenv("FFCB_FFT_MIXED_RADIX");
  return e ? atoi(e) != 0 : true;
}

// Lengths with a large prime factor: Bluestein when the planner prices it below the runtime plan
// (FFCB_FFT_BLUESTEIN=0 restores the runtime plans, kept as the cross-check).
inline bool bluestein_enabled() {
  const char* e = getenv("FFCB_FFT_BLUESTEIN");
  return e ? atoi(e) != 0 : true;
}

inline bool is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

inline size_t two_pass_smem(int n, int lanes, int groups) {
  return sizeof(float2) * ((size_t)n + (size_t)groups * 2 * n * lanes);
}

inline LaunchPlan make_plan(int n) {
  LaunchPlan p;
  p.n = n;
  p.m = n;
  p.bluestein = false;
  p.lanes = kLanes;
  p.rp.np = -1;
  for (int i = 0; i < kMaxRtPasses; ++i) p.rp.radix[i] = 1;
  BluesteinPlan bp;
  bp.m = 0;
  if (!(is_pow2(n) && n >= 4 && n <= 256) && mixed_radix_enabled() && bluestein_enabled())
    bp = make_bluestein_plan(n);
  if (bp.m > 0) {
    // Bluestein: one group of 8 (m = 512, 1024) or 4 (m = 2048) channels, m / 8 workers: one radix-8 butterfly per
    // worker and pass, up to a full 1024-thread CTA (bluestein_lanes)
    p.N = 0;
    p.m = bp.m;
    p.bluestein = true;
    p.lanes = bp.lanes;
    const int workers = (bp.m + 7) / 8 < 1024 / bp.lanes ? (bp.m + 7) / 8 : 1024 / bp.lanes;
    p.block = dim3(bp.lanes, workers, 1);
    p.smem = (size_t)bluestein_smem(n, bp.m, bp.lanes);
  } else if (is_pow2(n) && n >= 4 && n <= 256) {
    p.N = n;
    const int workers = workers_for(n);
    const int groups = workers >= 8 ? 1 : 8 / workers;
    p.block = dim3(kLanes, workers, groups);
    p.smem = two_pass_smem(n, kLanes, groups);
  } else if (two_pass_smem(n, kLanes, 1) <= (size_t)kBluesteinSmemLimit) {
    p.N = 0;
    int workers = n >= 8 ? 8 : (n >= 4 ? 4 : 1);
    if (mixed_radix_enabled()) {
      p.rp = make_rt_plan(n);
      // one output per worker-iteration: ~8 outputs per worker and pass, up to a full 1024-thread CTA
      if (n > 64) workers = (n + 7) / 8 < 32 ? (n + 7) / 8 : 32;
    }
    const int groups = n <= 32 ? (8 / workers > 0 ? 8 / workers : 1) : 1;
    p.block = dim3(kLanes, workers, groups);
    p.smem = two_pass_smem(n, kLanes, groups);
  } else {
    // 448..1024 (longer lengths are rejected by check_fft_shapes): 8 channels per CTA, ~8 outputs per worker and
    // pass, up to a full 1024-thread CTA
    p.N = 0;
    p.lanes = kNarrowLanes;
    if (mixed_radix_enabled()) p.rp = make_rt_plan(n);
    const int workers = (n + 7) / 8 < 1024 / kNarrowLanes ? (n + 7) / 8 : 1024 / kNarrowLanes;
    p.block = dim3(kNarrowLanes, workers, 1);
    p.smem = two_pass_smem(n, kNarrowLanes, 1);
  }
  return p;
}

// The two passes of an H x W plane, in either direction: the row passes transform along W, the column passes along H.
struct PlanePlans {
  LaunchPlan rows, cols;
};
inline PlanePlans make_plane_plans(int H, int W) { return PlanePlans{make_plan(W), make_plan(H)}; }

// c[j] = exp(-+ i pi j^2 / n).  The phase is reduced exactly in integers (j^2 mod 2n) first: j^2 / n in float loses
// it at n ~ 1000.
template <bool INV>
FFCB_HD float2 bluestein_chirp(int j, int n) {
  const int r = (int)(((long long)j * j) % (2 * n));
  float s, c;
#if defined(__CUDA_ARCH__)
  sincospif((float)r / (float)n, &s, &c);
#else
  const double a = M_PI * (double)((float)r / (float)n);
  s = (float)sin(a);
  c = (float)cos(a);
#endif
  return make_float2(c, INV ? s : -s);
}

// time-domain filter h[t] = conj(c[t]) for t < n, conj(c[m - t]) for t > m - n, 0 between (m >= 2n - 1)
template <bool INV>
FFCB_HD float2 bluestein_filter(int t, int n, int m) {
  const int d = t < n ? t : (t > m - n ? m - t : -1);
  if (d < 0) return make_float2(0.f, 0.f);
  const float2 c = bluestein_chirp<INV>(d, n);
  return make_float2(c.x, -c.y);
}

// step 1: a[j] *= c[j] for j < n, zero for n <= j < m (the caller stored points 0..n-1)
template <int LS>
FFCB_HD void bluestein_pre(float2* a, const float2* chirp, int n, int m, int lane, int worker, int nworkers) {
  for (int j = worker; j < m; j += nworkers)
    a[j * LS + lane] = j < n ? cmul(a[j * LS + lane], chirp[j]) : make_float2(0.f, 0.f);
}

// step 3: a[k] *= filt[k] (filter spectrum, 1/m folded in), k < m
template <int LS>
FFCB_HD void bluestein_mul(float2* a, const float2* filt, int m, int lane, int worker, int nworkers) {
  for (int k = worker; k < m; k += nworkers) a[k * LS + lane] = cmul(a[k * LS + lane], filt[k]);
}

// step 5: a[k] *= c[k], k < n: the n results in natural order
template <int LS>
FFCB_HD void bluestein_post(float2* a, const float2* chirp, int n, int lane, int worker, int nworkers) {
  for (int k = worker; k < n; k += nworkers) a[k * LS + lane] = cmul(a[k * LS + lane], chirp[k]);
}


// ------------------------------------------------------------------------------------------------
// 64-point complex FFT held entirely in registers (fully unrolled 8 x 8 Cooley-Tukey, compile-time
// twiddles): n = 8a + b, k = c + 8d;  step 1: FFT8 over a (stride 8), step 2: * w64^(b c), step 3: FFT8 over b.
// In/out in place; OUTPUT ORDER IS TRANSPOSED: X[k] is left in v[8*(k%8) + k/8]  (see fft64_at()).
FFCB_HD int fft64_at(int k) { return 8 * (k & 7) + (k >> 3); }

// w64^t = exp(-2 pi i t / 64), t = 0..63
FFCB_HD float2 tw64(int t) {
  constexpr float c[17] = {1.0f, 0.99518472667219688624f, 0.98078528040323044913f, 0.95694033573220886494f,
                           0.92387953251128675613f, 0.88192126434835502971f, 0.83146961230254523708f,
                           0.77301045336273696081f, 0.70710678118654752440f, 0.63439328416364549822f,
                           0.55557023301960222474f, 0.47139673682599764856f, 0.38268343236508977173f,
                           0.29028467725446236764f, 0.19509032201612826785f, 0.09801714032956060199f, 0.0f};
  // cos(2 pi t/64), sin(2 pi t/64) from the first-quadrant table
  const int q = (t >> 4) & 3, r = t & 15;
  const float cr = c[r], sr = c[16 - r];
  float co, si;
  if (q == 0) { co = cr; si = sr; }
  else if (q == 1) { co = -sr; si = cr; }
  else if (q == 2) { co = -cr; si = -sr; }
  else { co = sr; si = -cr; }
  return make_float2(co, -si);
}

template <bool INV>
FFCB_HD void fft64_regs(float2* v) {
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    float2 t[8];
#pragma unroll
    for (int a = 0; a < 8; ++a) t[a] = v[8 * a + b];
    fft8<INV>(t);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      float2 y = t[c];
      if (b * c != 0) {
        float2 w = tw64((b * c) & 63);
        if (INV) w.y = -w.y;
        y = cmul(y, w);
      }
      v[8 * c + b] = y;
    }
  }
#pragma unroll
  for (int c = 0; c < 8; ++c) fft8<INV>(v + 8 * c);
}


// 32-point complex FFT in registers, same construction: n = 8a + b (a < 4, b < 8); FFT4 over a, twiddle w32^(b c), FFT8
// over b.  X[k], k = c + 4d, is left in v[8c + d]  (fft32_at()).
FFCB_HD int fft32_at(int k) { return 8 * (k & 3) + (k >> 2); }

template <bool INV>
FFCB_HD void fft32_regs(float2* v) {
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    float2 t0 = v[b], t1 = v[8 + b], t2 = v[16 + b], t3 = v[24 + b];
    fft4<INV>(t0, t1, t2, t3);
    const float2 t[4] = {t0, t1, t2, t3};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float2 y = t[c];
      if (b * c != 0) {
        float2 w = tw64((2 * b * c) & 63);      // w32^(bc) = w64^(2bc)
        if (INV) w.y = -w.y;
        y = cmul(y, w);
      }
      v[8 * c + b] = y;
    }
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) fft8<INV>(v + 8 * c);
}

// length-generic access to the register transforms (N = 32 or 64)
template <int N> struct RegFft;
template <> struct RegFft<64> {
  template <bool INV> static FFCB_HD void run(float2* v) { fft64_regs<INV>(v); }
  static FFCB_HD int at(int k) { return fft64_at(k); }
};
template <> struct RegFft<32> {
  template <bool INV> static FFCB_HD void run(float2* v) { fft32_regs<INV>(v); }
  static FFCB_HD int at(int k) { return fft32_at(k); }
};

// Per-thread steps of the fused 64x64 plane kernels (fft_plane.cu); functors keep them host-testable.
//   rows forward : z[n] = (row_a[n], row_b[n]) -> half spectra A[k], B[k], k = 0..32 (two-for-one)
//   columns      : 64-point complex transform of one (kx, channel) column, natural order in and out
//   rows inverse : half spectra X1[k], X2[k] (C2R rule) -> (row_a[n], row_b[n])
template <class Load, class Store>
FFCB_HD void plane64_rows_fwd(Load&& ld, Store&& st) {
  float2 v[64];
#pragma unroll
  for (int n = 0; n < 64; ++n) v[n] = ld(n);
  fft64_regs<false>(v);
#pragma unroll
  for (int k = 0; k <= 32; ++k) {
    const float2 zk = v[fft64_at(k)], zm = v[fft64_at((64 - k) & 63)];
    st(k, make_float2(0.5f * (zk.x + zm.x), 0.5f * (zk.y - zm.y)),
       make_float2(0.5f * (zk.y + zm.y), -0.5f * (zk.x - zm.x)));
  }
}

template <bool INV, class Load, class Store>
FFCB_HD void plane64_col(Load&& ld, Store&& st) {
  float2 v[64];
#pragma unroll
  for (int n = 0; n < 64; ++n) v[n] = ld(n);
  fft64_regs<INV>(v);
#pragma unroll
  for (int k = 0; k < 64; ++k) st(k, v[fft64_at(k)]);
}

template <class Load, class Store>
FFCB_HD void plane64_rows_inv(Load&& ld, Store&& st) {
  float2 v[64];
#pragma unroll
  for (int k = 0; k <= 32; ++k) {
    float2 x1, x2;
    ld(k, x1, x2);
    if (k == 0 || k == 32) {
      v[k] = make_float2(x1.x, x2.x);                      // Im of DC / Nyquist ignored (C2R rule)
    } else {
      v[k] = make_float2(x1.x - x2.y, x1.y + x2.x);        // X1 + i X2
      v[64 - k] = make_float2(x1.x + x2.y, x2.x - x1.y);   // conj(X1) + i conj(X2)
    }
  }
  fft64_regs<true>(v);
  // hand the results over 16 pixels at a time so that the caller can put its 32 residual loads in
  // flight before the dependent adds / stores (registers are full of v[]: no room to hoist all 128)
#pragma unroll
  for (int n0 = 0; n0 < 64; n0 += 16) {
    float2 zb[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) zb[j] = v[fft64_at(n0 + j)];
    st(n0, zb);
  }
}

// Inverse plane kernel (fft_plane.cu: irfft2_plane64_v2_kernel): after the C2R row transforms the
// real results of row r are staged IN PLACE of that row's half spectrum (S row = 268 float2 = 536 floats >= 64 px x
// 8 channels), channels-last, so that the epilogue moves whole pixels (8 channels = 32 bytes) with vector accesses.
constexpr int kP64Pitch = 33 * 8 + 4;        // float2 per S row of the 8-channel plane kernels
FFCB_HD int p64_stage_index(int row, int x, int c) { return row * (2 * kP64Pitch) + x * 8 + c; }   // float index
// epilogue slot i (0..15) of a lane: warp w owns rows 8w .. 8w+7 (its four row-pair groups), 64 pixels each
FFCB_HD void p64_store_slot(int warp, int lane, int i, int& row, int& x) {
  const int s = i * 32 + lane;
  row = 8 * warp + (s >> 6);
  x = s & 63;
}

}  // namespace fftc
}  // namespace ffcb
