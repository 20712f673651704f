// Batched real 2-D FFT pair over channels-last tensors (norm='ortho').
//
// Replaces torch.fft.rfftn / irfftn and the stack/permute/view shuffles around them
// (reference ffc.py:86-89, 103-108) — no cuFFT.
//
// Mapping: lane == channel.  In NHWC the 32 lanes of a warp read 32 consecutive channels of one
// pixel (one 128-byte line), every lane owns one independent 1-D transform, and the transform's
// points live in shared memory as data[point][lane] (float2), so shared-memory accesses are
// conflict-free and twiddles are warp-uniform broadcasts.  A 2-D transform is a row pass and a
// column pass with the half-spectrum intermediate in a caller workspace (L2-resident at the
// sizes of the path); rows are transformed two at a time ("two-for-one": z = row_a + i*row_b).
//
// Sizes: power-of-two lengths 4..256 run a mixed-radix (8/4) Stockham autosort (ping-pong buffers);
// every other length runs the runtime mixed-radix Stockham (a direct DFT for primes), so odd /
// non-power-of-two planes (bin/predict.py pads images to multiples of 8 only -> e.g. 125x188
// bottlenecks) stay native.  Lengths with a large prime factor (e.g. 479), where that plan costs
// nearly n^2, run a Bluestein chirp-z transform through compile-time radix-8/4 passes of the power of
// two m >= 2n - 1 (fft_core.cuh: make_bluestein_plan), 8 or 4 channels per CTA (setup_tile).
//
// Channels per CTA (template L): 32, or 8 for lengths 448..1024, whose 32-channel ping-pong buffers
// (8 * (n + 64 n) bytes) exceed the 227 KB of shared memory a CTA may hold; the 8-channel CTA needs
// 8 * (n + 16 n) bytes (139 KB at 1024).  With L = 8 a warp covers 8 channels x 4 workers, so every
// global access still moves whole 32-byte sectors.  These lengths are the bottlenecks of 4K and
// larger photos (3840x2160 -> 480x270, 4000x3000 -> 500x375, 4096^2 -> 512^2).
#include <math.h>
#include <stdlib.h>

#include "common.cuh"
#include "fft_core.cuh"

namespace ffcb {
namespace {

constexpr int kBsWideLanes = 4;   // channels per CTA of Bluestein lengths 513..1024 (2048-long buffers: fft_core.cuh)
constexpr int kMaxLen = 1024;     // longest axis (make_rt_plan factors every length up to 1024)
using namespace fftc;

// Runtime mixed-radix Stockham (row f2) of length n for this lane: `a` holds the input (already synchronised), `b`
// is scratch of the same size; returns the buffer holding the result.  Ends with a barrier.
template <bool INV, int LS>
__device__ __forceinline__ float2* rt_passes(float2* a, float2* b, const float2* tw, int n, const RtPlan& rp, int lane,
                                             int worker, int nworkers) {
  int ns = 1;
  for (int p = 0; p < rp.np; ++p) {
    const int R = rp.radix[p];
    generic_pass<INV, LS>(a, b, tw, n, R, ns, lane, worker, nworkers);
    __syncthreads();
    ns *= R;
    float2* t = a; a = b; b = t;
  }
  return a;
}

// Compile-time Stockham passes PASS.. of length N (a Bluestein convolution length) from `a`, scratch `b`; returns the
// buffer holding the result.  Each pass ends with a barrier.
template <int N, int PASS, bool INV, int LS>
__device__ __forceinline__ float2* stockham_passes(float2* a, float2* b, const float2* tw, int lane, int worker,
                                                   int nworkers) {
  if constexpr (PASS == Plan<N>::P) {
    return a;
  } else {
    stockham_pass<N, PASS, INV, LS>(a, b, tw, lane, worker, nworkers);
    __syncthreads();
    return stockham_passes<N, PASS + 1, INV, LS>(b, a, tw, lane, worker, nworkers);
  }
}

// Shared-memory tile of one CTA.  Two-pass: [twiddles n][group g: ping n*L | pong n*L].
// Bluestein: [twiddles m][chirp n][filter spectrum m][ping m*L | pong m*L] (one group).
struct Tile {
  float2* tw;
  float2* data;    // the kernel stages its n input points here
  float2* tmp;
  float2* chirp;   // Bluestein only
  float2* filt;    // Bluestein only
};

// Complex FFT of length N (compile-time power of two, or runtime n when N == 0) for this lane on t.data (already
// synchronised); returns the buffer holding the n results in natural order.  BM > 0: Bluestein through BM-point
// compile-time transforms (fft_core.cuh); otherwise rp is the plan of n.  Ends with a barrier.
template <int N, int L, bool INV, int BM>
__device__ __forceinline__ float2* fft_dispatch(const Tile& t, int n, int lane, int worker, int nworkers,
                                                const RtPlan& rp) {
  float2 *a = t.data, *b = t.tmp;
  if constexpr (BM > 0) {                  // Bluestein (chirp-z)
    bluestein_pre<L>(a, t.chirp, n, BM, lane, worker, nworkers);
    __syncthreads();
    float2* f = stockham_passes<BM, 0, false, L>(a, b, t.tw, lane, worker, nworkers);
    bluestein_mul<L>(f, t.filt, BM, lane, worker, nworkers);
    __syncthreads();
    float2* g = stockham_passes<BM, 0, true, L>(f, f == a ? b : a, t.tw, lane, worker, nworkers);
    bluestein_post<L>(g, t.chirp, n, lane, worker, nworkers);
    __syncthreads();
    return g;
  } else if constexpr (N == 0) {
    if (rp.np < 0) {                       // direct DFT
      dft_pass<INV, L>(a, b, t.tw, n, lane, worker, nworkers);
      __syncthreads();
      return b;
    }
    return rt_passes<INV, L>(a, b, t.tw, n, rp, lane, worker, nworkers);   // runtime mixed-radix Stockham
  } else {
    const float2* tw = t.tw;
    stockham_pass<N, 0, INV, L>(a, b, tw, lane, worker, nworkers);
    __syncthreads();
    if constexpr (Plan<N>::P == 1) return b;
    else {
      stockham_pass<N, 1, INV, L>(b, a, tw, lane, worker, nworkers);
      __syncthreads();
      if constexpr (Plan<N>::P == 2) return a;
      else {
        stockham_pass<N, 2, INV, L>(a, b, tw, lane, worker, nworkers);
        __syncthreads();
        return b;
      }
    }
  }
}

__device__ __forceinline__ void make_twiddles(float2* tw, int n) {
  const int tid = threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z);
  const int nthreads = blockDim.x * blockDim.y * blockDim.z;
  for (int t = tid; t < n; t += nthreads) {
    float s, c;
    sincospif(2.0f * (float)t / (float)n, &s, &c);
    tw[t] = make_float2(c, -s);  // exp(-2 pi i t / n)
  }
}

// Carves this group's tile out of shared memory and fills the tables: twiddles of the transform length (m for
// Bluestein), and for Bluestein the chirp of direction INV and the filter spectrum FFT_m(h) / m, which every thread of
// the CTA computes together with the m-point passes, using the ping buffer as scratch (the caller stages its input
// only afterwards).  Ends with a barrier when it wrote more than the twiddles (the kernels' staging loops end with one).
template <int N, int L, bool INV, int BM>
__device__ __forceinline__ Tile setup_tile(float2* smem, int n, int group) {
  Tile t;
  if constexpr (BM > 0) {
    constexpr int m = BM;
    t.tw = smem;
    t.chirp = smem + m;
    t.filt = t.chirp + n;
    t.data = t.filt + m;
    t.tmp = t.data + (size_t)m * L;
    make_twiddles(t.tw, m);
    const int tid = threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z);
    const int nthreads = blockDim.x * blockDim.y * blockDim.z;
    for (int j = tid; j < n; j += nthreads) t.chirp[j] = bluestein_chirp<INV>(j, n);
    for (int j = tid; j < m; j += nthreads) t.filt[j] = bluestein_filter<INV>(j, n, m);
    __syncthreads();
    const float2* f = stockham_passes<m, 0, false, 1>(t.filt, t.data, t.tw, 0, tid, nthreads);
    const float inv_m = 1.0f / (float)m;
    for (int j = tid; j < m; j += nthreads) t.filt[j] = cscale(f[j], inv_m);
    __syncthreads();
  } else {
    t.tw = smem;
    t.data = smem + n + (size_t)group * 2 * n * L;
    t.tmp = t.data + n * L;
    t.chirp = t.filt = nullptr;
    make_twiddles(t.tw, n);
  }
  return t;
}

// ---------------------------------------------------------------------------------------------
// Row pass, forward.  grid.x = ceil(B*ceil(H/2) / G), grid.y = ceil(C/L).
// in (B,H,W,C) real  ->  ws[b][y][k][c] complex, k = 0..W/2   (unscaled)
template <int N, int L, int BM>
__global__ void __launch_bounds__(1024) rfft_rows_kernel(View in, float2* __restrict__ ws, int n, RtPlan rp) {
  extern __shared__ float2 smem_f2[];
  const int W = (N > 0) ? N : n;
  const int lane = threadIdx.x, worker = threadIdx.y, nworkers = blockDim.y, group = threadIdx.z;
  const Tile t = setup_tile<N, L, false, BM>(smem_f2, W, group);
  float2* data = t.data;

  const int hp = (in.H + 1) / 2;
  const int pair = blockIdx.x * blockDim.z + group;       // (b, y-pair)
  const bool live = pair < in.B * hp;
  const int b = live ? pair / hp : 0;
  const int y0 = live ? (pair % hp) * 2 : 0;
  const int c = blockIdx.y * L + lane;
  const bool cok = live && c < in.C;
  const bool row1 = (y0 + 1) < in.H;

  for (int x = worker; x < W; x += nworkers) {
    float2 z = make_float2(0.f, 0.f);
    if (cok) {
      z.x = load1(in, pix_off(in, b, y0, x) + c);
      if (row1) z.y = load1(in, pix_off(in, b, y0 + 1, x) + c);
    }
    data[x * L + lane] = z;
  }
  __syncthreads();
  const float2* res = fft_dispatch<N, L, false, BM>(t, W, lane, worker, nworkers, rp);

  const int wf = W / 2 + 1;
  if (cok) {
    for (int k = worker; k < wf; k += nworkers) {
      float2 a, bb;
      r2c_pair_post<L>(res, W, k, lane, a, bb);
      const size_t o = (((size_t)b * in.H + y0) * wf + k) * in.C + c;
      ws[o] = a;
      if (row1) ws[o + (size_t)wf * in.C] = bb;
    }
  }
}

// Column pass, forward.  grid.x = ceil(B*Wf / G), grid.y = ceil(C/L).
// ws[b][y][k][c] complex -> spec (B,H,Wf,2C): channel 2c = Re, 2c+1 = Im, scaled by `scale`.
template <int N, int L, int BM>
__global__ void __launch_bounds__(1024) fft_cols_fwd_kernel(const float2* __restrict__ ws, View spec, int n,
                                                            int C, float scale, RtPlan rp) {
  extern __shared__ float2 smem_f2[];
  const int H = (N > 0) ? N : n;
  const int lane = threadIdx.x, worker = threadIdx.y, nworkers = blockDim.y, group = threadIdx.z;
  const Tile t = setup_tile<N, L, false, BM>(smem_f2, H, group);
  float2* data = t.data;

  const int wf = spec.W;
  const int col = blockIdx.x * blockDim.z + group;  // (b, k)
  const bool live = col < spec.B * wf;
  const int b = live ? col / wf : 0;
  const int k = live ? col % wf : 0;
  const int c = blockIdx.y * L + lane;
  const bool cok = live && c < C;

  for (int y = worker; y < H; y += nworkers) {
    float2 z = make_float2(0.f, 0.f);
    if (cok) z = ws[(((size_t)b * H + y) * wf + k) * C + c];
    data[y * L + lane] = z;
  }
  __syncthreads();
  const float2* res = fft_dispatch<N, L, false, BM>(t, H, lane, worker, nworkers, rp);

  if (cok) {
    for (int y = worker; y < H; y += nworkers) {
      const float2 z = res[y * L + lane];
      const long long o = pix_off(spec, b, y, k) + 2 * c;
      if (spec.fmt == FFCB_F32) {
        *reinterpret_cast<float2*>(reinterpret_cast<float*>(spec.ptr) + o) = make_float2(z.x * scale, z.y * scale);
      } else {
        __nv_bfloat16 h0, l0, h1, l1;
        split_bf16(z.x * scale, h0, l0);
        split_bf16(z.y * scale, h1, l1);
        unsigned* p = reinterpret_cast<unsigned*>(reinterpret_cast<unsigned short*>(spec.ptr) + o);
        p[0] = pack_bf16(h0, h1);
        *reinterpret_cast<unsigned*>(reinterpret_cast<unsigned short*>(spec.ptr) + o + spec.lo_off) =
            pack_bf16(l0, l1);
      }
    }
  }
}

// Column pass, inverse: spec (B,H,Wf,2C) -> ws[b][y][k][c] complex (unscaled inverse along H).
template <int N, int L, int BM>
__global__ void __launch_bounds__(N > 0 && N <= 64 ? 256 : 1024, N > 0 && N <= 64 ? 6 : 1) fft_cols_inv_kernel(View spec, float2* __restrict__ ws, int n, int C, RtPlan rp) {
  extern __shared__ float2 smem_f2[];
  const int H = (N > 0) ? N : n;
  const int lane = threadIdx.x, worker = threadIdx.y, nworkers = blockDim.y, group = threadIdx.z;
  const Tile t = setup_tile<N, L, true, BM>(smem_f2, H, group);
  float2* data = t.data;

  const int wf = spec.W;
  const int col = blockIdx.x * blockDim.z + group;
  const bool live = col < spec.B * wf;
  const int b = live ? col / wf : 0;
  const int k = live ? col % wf : 0;
  const int c = blockIdx.y * L + lane;
  const bool cok = live && c < C;

  for (int y = worker; y < H; y += nworkers) {
    float2 z = make_float2(0.f, 0.f);
    if (cok) {
      const long long o = pix_off(spec, b, y, k) + 2 * c;
      if (spec.fmt == FFCB_F32) {
        z = __ldg(reinterpret_cast<const float2*>(reinterpret_cast<const float*>(spec.ptr) + o));
      } else {
        z.x = load1(spec, o);
        z.y = load1(spec, o + 1);
      }
    }
    data[y * L + lane] = z;
  }
  __syncthreads();
  const float2* res = fft_dispatch<N, L, true, BM>(t, H, lane, worker, nworkers, rp);

  if (cok) {
    for (int y = worker; y < H; y += nworkers)
      ws[(((size_t)b * H + y) * wf + k) * C + c] = res[y * L + lane];
  }
}

// Row pass, inverse (C2R, two rows at a time): ws[b][y][k][c] -> out (B,H,W,C) real,
// out = residual + scale * c2r(ws).  Im of bins 0 and (even W) W/2 is ignored.
template <int N, int L, int BM>
__global__ void __launch_bounds__(N > 0 && N <= 64 ? 256 : 1024, N > 0 && N <= 64 ? 6 : 1) irfft_rows_kernel(const float2* __restrict__ ws, View res, View out, int n,
                                                          float scale, RtPlan rp) {
  extern __shared__ float2 smem_f2[];
  const int W = (N > 0) ? N : n;
  const int lane = threadIdx.x, worker = threadIdx.y, nworkers = blockDim.y, group = threadIdx.z;
  const Tile t = setup_tile<N, L, true, BM>(smem_f2, W, group);
  float2* data = t.data;

  const int hp = (out.H + 1) / 2;
  const int pair = blockIdx.x * blockDim.z + group;
  const bool live = pair < out.B * hp;
  const int b = live ? pair / hp : 0;
  const int y0 = live ? (pair % hp) * 2 : 0;
  const int c = blockIdx.y * L + lane;
  const bool cok = live && c < out.C;
  const bool row1 = (y0 + 1) < out.H;
  const int wf = W / 2 + 1;

  for (int k = worker; k < wf; k += nworkers) {
    float2 x1 = make_float2(0.f, 0.f), x2 = make_float2(0.f, 0.f);
    if (cok) {
      const size_t o = (((size_t)b * out.H + y0) * wf + k) * out.C + c;
      x1 = ws[o];
      if (row1) x2 = ws[o + (size_t)wf * out.C];
    }
    c2r_pair_pre<L>(data, W, k, lane, x1, x2);
  }
  __syncthreads();
  const float2* fin = fft_dispatch<N, L, true, BM>(t, W, lane, worker, nworkers, rp);

  if (cok) {
    if (N > 0) {
      // power-of-two lengths: every worker owns exactly 8 pixels.  Put all residual loads in flight first —
      // the compiler cannot hoist them above the stores itself (res / out may alias as far as it knows).
      float ra[8], rb[8];
      const long long q0 = res.ptr ? pix_off(res, b, y0, 0) + c : 0, o0 = pix_off(out, b, y0, 0) + c;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int x = worker + i * nworkers;
        ra[i] = (res.ptr != nullptr && x < W) ? load1(res, q0 + x * res.sx) : 0.f;
        rb[i] = (res.ptr != nullptr && x < W && row1) ? load1(res, q0 + res.sy + x * res.sx) : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int x = worker + i * nworkers;
        if (x < W) {
          const float2 z = fin[x * L + lane];
          store1(out, o0 + x * out.sx, fmaf(z.x, scale, ra[i]));
          if (row1) store1(out, o0 + out.sy + x * out.sx, fmaf(z.y, scale, rb[i]));
        }
      }
    } else {
      for (int x = worker; x < W; x += nworkers) {
        const float2 z = fin[x * L + lane];
        float r0 = z.x * scale, r1 = z.y * scale;
        if (res.ptr != nullptr) {
          r0 += load1(res, pix_off(res, b, y0, x) + c);
          if (row1) r1 += load1(res, pix_off(res, b, y0 + 1, x) + c);
        }
        store1(out, pix_off(out, b, y0, x) + c, r0);
        if (row1) store1(out, pix_off(out, b, y0 + 1, x) + c, r1);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Launch plans of the two passes: fft_core.cuh (make_plan, make_plane_plans).
template <typename K>
int set_smem(K kernel, size_t bytes) {
  if (bytes > 48 * 1024) FFCB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return FFCB_OK;
}

// NN: template length, LL: channels per CTA, BM: Bluestein convolution length (0: none)
#define FFCB_DISPATCH_N(PLAN, ...)                                                            \
  if ((PLAN).bluestein) {                                                                     \
    switch ((PLAN).m) {                                                                       \
      case 512: { constexpr int NN = 0, LL = kNarrowLanes, BM = 512; __VA_ARGS__; } break;    \
      case 1024: { constexpr int NN = 0, LL = kNarrowLanes, BM = 1024; __VA_ARGS__; } break;  \
      case 2048: { constexpr int NN = 0, LL = kBsWideLanes, BM = 2048; __VA_ARGS__; } break;  \
      default: set_error("fft: internal plan error"); return FFCB_EINVAL;                     \
    }                                                                                         \
  } else if ((PLAN).lanes == kNarrowLanes) {                                                  \
    constexpr int NN = 0, LL = kNarrowLanes, BM = 0; __VA_ARGS__;                             \
  } else switch ((PLAN).N) {                                                                  \
    case 0: { constexpr int NN = 0, LL = kLanes, BM = 0; __VA_ARGS__; } break;                \
    case 4: { constexpr int NN = 4, LL = kLanes, BM = 0; __VA_ARGS__; } break;                \
    case 8: { constexpr int NN = 8, LL = kLanes, BM = 0; __VA_ARGS__; } break;                \
    case 16: { constexpr int NN = 16, LL = kLanes, BM = 0; __VA_ARGS__; } break;              \
    case 32: { constexpr int NN = 32, LL = kLanes, BM = 0; __VA_ARGS__; } break;              \
    case 64: { constexpr int NN = 64, LL = kLanes, BM = 0; __VA_ARGS__; } break;              \
    case 128: { constexpr int NN = 128, LL = kLanes, BM = 0; __VA_ARGS__; } break;            \
    case 256: { constexpr int NN = 256, LL = kLanes, BM = 0; __VA_ARGS__; } break;            \
    default: set_error("fft: internal plan error"); return FFCB_EINVAL;                       \
  }

int check_fft_shapes(const ffcb_tensor* real, const ffcb_tensor* spec, const char* who) {
  FFCB_REQUIRE(real->H >= 1 && real->W >= 2, "%s: plane %dx%d too small", who, real->H, real->W);
  FFCB_REQUIRE(spec->B == real->B && spec->H == real->H && spec->W == real->W / 2 + 1 && spec->C == 2 * real->C,
               "%s: spectrum view must be (B,H,W/2+1,2C) = (%d,%d,%d,%d), got (%d,%d,%d,%d)", who, real->B, real->H,
               real->W / 2 + 1, 2 * real->C, spec->B, spec->H, spec->W, spec->C);
  FFCB_REQUIRE(real->H <= kMaxLen && real->W <= kMaxLen, "%s: plane %dx%d exceeds the %d-point FFT limit", who,
               real->H, real->W, kMaxLen);
  return FFCB_OK;
}

}  // namespace

// fused whole-plane path (fft_plane.cu)
bool plane64_eligible(const ffcb_tensor* real);
bool plane64_inv_eligible(const ffcb_tensor* spec, const ffcb_tensor* residual, const ffcb_tensor* out);
int rfft2_plane64(const ffcb_tensor* in, const ffcb_tensor* spec, cudaStream_t stream);
int irfft2_plane64(const ffcb_tensor* spec, const ffcb_tensor* residual, const ffcb_tensor* out, cudaStream_t stream);
// channel-group planar plane kernels (fft_plane_cg.cu)
bool plane64_cg_fwd_eligible(const ffcb_tensor* in, const ffcb_tensor* spec);
bool plane64_cg_inv_eligible(const ffcb_tensor* spec, const ffcb_tensor* residual, const ffcb_tensor* out);
int rfft2_plane64_cg(const ffcb_tensor* in, const ffcb_tensor* spec, cudaStream_t stream);
int irfft2_plane64_cg(const ffcb_tensor* spec, const ffcb_tensor* residual, const ffcb_tensor* out, cudaStream_t stream);

size_t fft2_workspace_bytes(int B, int H, int W, int C) {
  return sizeof(float2) * (size_t)B * H * (W / 2 + 1) * C;
}

int rfft2(const ffcb_tensor* in, const ffcb_tensor* spec, void* ws, size_t ws_bytes, cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(in, "rfft2.in", true)) || (rc = check_tensor(spec, "rfft2.spec", true))) return rc;
  if ((rc = check_fft_shapes(in, spec, "rfft2"))) return rc;
  if (ws_bytes < fft2_workspace_bytes(in->B, in->H, in->W, in->C)) {
    set_error("rfft2: workspace %zu < %zu bytes", ws_bytes, fft2_workspace_bytes(in->B, in->H, in->W, in->C));
    return FFCB_ENOMEM;
  }
  if (in->B == 0 || in->C == 0) return FFCB_OK;
  if (in->cg != 0 || spec->cg != 0) {
    FFCB_REQUIRE(plane64_cg_fwd_eligible(in, spec),
                 "rfft2: channel-group planar views need a 64x64 / 32x32 float32 cg=4 input and a split-bf16 cg=8 spectrum");
    return rfft2_plane64_cg(in, spec, stream);
  }
  if (plane64_eligible(in) && !getenv("FFCB_FFT_TWO_PASS")) return rfft2_plane64(in, spec, stream);
  const View vin = make_view(*in), vspec = make_view(*spec);
  float2* w2 = reinterpret_cast<float2*>(ws);
  const int C = in->C;
  const float scale = (float)(1.0 / sqrt((double)in->H * (double)in->W));
  {
    const LaunchPlan p = make_plane_plans(in->H, in->W).rows;
    const int pairs = in->B * ((in->H + 1) / 2);
    dim3 grid((pairs + p.block.z - 1) / p.block.z, (C + p.lanes - 1) / p.lanes);
    FFCB_DISPATCH_N(p, {
      if ((rc = set_smem(rfft_rows_kernel<NN, LL, BM>, p.smem))) return rc;
      rfft_rows_kernel<NN, LL, BM><<<grid, p.block, p.smem, stream>>>(vin, w2, p.n, p.rp);
    });
    FFCB_LAUNCH_CHECK("rfft_rows_kernel");
  }
  {
    const LaunchPlan p = make_plane_plans(in->H, in->W).cols;
    const int cols = in->B * spec->W;
    dim3 grid((cols + p.block.z - 1) / p.block.z, (C + p.lanes - 1) / p.lanes);
    FFCB_DISPATCH_N(p, {
      if ((rc = set_smem(fft_cols_fwd_kernel<NN, LL, BM>, p.smem))) return rc;
      fft_cols_fwd_kernel<NN, LL, BM><<<grid, p.block, p.smem, stream>>>(w2, vspec, p.n, in->C, scale, p.rp);
    });
    FFCB_LAUNCH_CHECK("fft_cols_fwd_kernel");
  }
  return FFCB_OK;
}

int irfft2(const ffcb_tensor* spec, const ffcb_tensor* residual, const ffcb_tensor* out, void* ws, size_t ws_bytes,
           cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(spec, "irfft2.spec", true)) || (rc = check_tensor(out, "irfft2.out", true))) return rc;
  if ((rc = check_fft_shapes(out, spec, "irfft2"))) return rc;
  View vres = null_view();
  if (residual != nullptr && residual->ptr != nullptr) {
    if ((rc = check_tensor(residual, "irfft2.residual", true))) return rc;
    FFCB_REQUIRE(residual->B == out->B && residual->H == out->H && residual->W == out->W && residual->C == out->C,
                 "irfft2: residual shape differs from output");
    vres = make_view(*residual);
  }
  if (ws_bytes < fft2_workspace_bytes(out->B, out->H, out->W, out->C)) {
    set_error("irfft2: workspace %zu < %zu bytes", ws_bytes, fft2_workspace_bytes(out->B, out->H, out->W, out->C));
    return FFCB_ENOMEM;
  }
  if (out->B == 0 || out->C == 0) return FFCB_OK;
  if (spec->cg != 0 || out->cg != 0 || (residual && residual->ptr && residual->cg != 0)) {
    FFCB_REQUIRE(plane64_cg_inv_eligible(spec, residual, out),
                 "irfft2: channel-group planar views need a 64x64 / 32x32 plane, a float32 cg=8 spectrum, a float32 cg=4 "
                 "residual and a split-bf16 cg=8 or float32 cg=4 output");
    return irfft2_plane64_cg(spec, residual, out, stream);
  }
  // views the plane kernel cannot take with 16-byte vector accesses run the two-pass kernels below
  if (plane64_eligible(out) && plane64_inv_eligible(spec, residual, out) && !getenv("FFCB_FFT_TWO_PASS"))
    return irfft2_plane64(spec, residual, out, stream);
  const View vspec = make_view(*spec), vout = make_view(*out);
  float2* w2 = reinterpret_cast<float2*>(ws);
  const int C = out->C;
  const float scale = (float)(1.0 / sqrt((double)out->H * (double)out->W));
  {
    const LaunchPlan p = make_plane_plans(out->H, out->W).cols;
    const int cols = out->B * spec->W;
    dim3 grid((cols + p.block.z - 1) / p.block.z, (C + p.lanes - 1) / p.lanes);
    FFCB_DISPATCH_N(p, {
      if ((rc = set_smem(fft_cols_inv_kernel<NN, LL, BM>, p.smem))) return rc;
      fft_cols_inv_kernel<NN, LL, BM><<<grid, p.block, p.smem, stream>>>(vspec, w2, p.n, out->C, p.rp);
    });
    FFCB_LAUNCH_CHECK("fft_cols_inv_kernel");
  }
  {
    const LaunchPlan p = make_plane_plans(out->H, out->W).rows;
    const int pairs = out->B * ((out->H + 1) / 2);
    dim3 grid((pairs + p.block.z - 1) / p.block.z, (C + p.lanes - 1) / p.lanes);
    FFCB_DISPATCH_N(p, {
      if ((rc = set_smem(irfft_rows_kernel<NN, LL, BM>, p.smem))) return rc;
      irfft_rows_kernel<NN, LL, BM><<<grid, p.block, p.smem, stream>>>(w2, vres, vout, p.n, scale, p.rp);
    });
    FFCB_LAUNCH_CHECK("irfft_rows_kernel");
  }
  return FFCB_OK;
}

}  // namespace ffcb
