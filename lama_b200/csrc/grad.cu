// Input-gradient helpers of the FFC block (SURVEY.md row f3: the reference's refinement optimises the feature maps
// entering the residual blocks, evaluation/refinement.py:137-167, 266-289 — it needs dL/dx_l, dL/dx_g through
// FFCResnetBlock, not weight gradients).
//
// With eval-mode BatchNorm folded into the weights every backward step of the block is one of the forward's own
// operations on transposed weights (lama_b200/engine.py: emit_block_backward) — ffcb_conv with flipped 3x3 taps on a
// zero border, ffcb_rfft2 / ffcb_irfft2 (the adjoint of the ortho R2C / C2R pair is the pair itself: the per-column
// weights 2 and 1/2 of the half spectrum cancel around the channel-mixing GEMM) — plus the two elementwise kernels
// here:
//   ffcb_relu_bwd             dx = dy * [y > 0]                      (y = the forward activation, ffc.py:101,133,253-254)
//   ffcb_fold_reflect_border  adjoint of ReflectionPad(1): the gradient w.r.t. the padded plane folded back onto the
//                             interior (+ up to two addends: the 1x1 branch's gradient, the residual path's gradient)
//   ffcb_relu_mask_pack       bits = [y > 0], one bit per element, so that the refinement step program can drop the
//   ffcb_relu_bwd_bits        full-width forward activations after the forward; dx = dy * bit is ffcb_relu_bwd
// and, for the generator's rear (residual blocks + up-sampling tail + head, lama_b200/engine.py:
// build_rear_grad_program):
//   ffcb_add                  out = a + b over the padded extent (the block identity X + Y2, ffc.py:288, with Y2 kept)
//   ffcb_head_bwd7            adjoint of ReflectionPad2d(3) + Conv2d 7x7 + act (ffc.py:360-363), fused with the ReLU
//                             mask of the last up-sampling stage (ffc.py:350-354); ffcb_head_bwd7_bits reads that mask
//                             as bits and may write a row band of the plane (the banded up-sampling tail)
#include <stdint.h>

#include "common.cuh"

namespace ffcb {
namespace {

// generic 4-channel access that also understands channel-group planar views
__device__ __forceinline__ float4 load4g(const View& v, int b, int y, int x, int c) {
  return load4(v, elem_off(v, b, y, x, c));
}
__device__ __forceinline__ void store4g(const View& v, int b, int y, int x, int c, float4 r) {
  store4(v, elem_off(v, b, y, x, c), r);
}

__global__ void relu_bwd_kernel(View dy, View y, View out) {
  const int c4 = out.C / 4;
  const long long total = (long long)out.B * out.H * out.W * c4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    // planar views: channels of one group are contiguous per pixel, pixels contiguous per group -> iterate pixels
    // fastest inside a 4-channel quad so that both layouts are read in whole lines
    const int q = out.cg ? (int)(i / ((long long)out.B * out.H * out.W)) : (int)(i % c4);
    const long long p = out.cg ? i % ((long long)out.B * out.H * out.W) : i / c4;
    const int x = (int)(p % out.W);
    const int yy = (int)((p / out.W) % out.H);
    const int b = (int)(p / ((long long)out.W * out.H));
    const float4 g = load4g(dy, b, yy, x, 4 * q), a = load4g(y, b, yy, x, 4 * q);
    store4g(out, b, yy, x, 4 * q,
            make_float4(a.x > 0.f ? g.x : 0.f, a.y > 0.f ? g.y : 0.f, a.z > 0.f ? g.z : 0.f, a.w > 0.f ? g.w : 0.f));
  }
}

// ---- bit-packed ReLU masks: word ((b*H + y)*W + x)*nw + c/32 of a view holds bit c%32 = [y(b,y,x,c) > 0] ----------
// The comparison reads the value exactly as relu_bwd_kernel does (load1 / load4 decode split bf16 as hi + lo in the
// same float addition), so relu_bwd_bits_kernel with these words writes what relu_bwd_kernel writes with the values.

// channels-last views: one warp per (pixel, 32-channel word), lane l tests channel 32w + l and __ballot_sync builds
// the word (a warp reads 32 adjacent channels: 128 contiguous bytes per fp32 plane, 64 per bf16 plane)
// Row bands: the words of a view of rows [row0, row0 + y.H) of a plane of hb rows live at
// ((b*hb + row0 + y)*W + x)*nw + c/32 — a band of a whole-plane mask buffer; hb = y.H, row0 = 0 is the whole plane.
__device__ __forceinline__ long long band_word(long long p, int W, int H, int hb, int row0, int nw) {
  const long long row = p / W, b = row / H;
  return ((b * hb + row0 + (row - b * H)) * W + p % W) * nw;
}

__global__ void relu_mask_pack_cl_kernel(View y, uint32_t* __restrict__ bits, int nw, int hb, int row0) {
  const long long total = (long long)y.B * y.H * y.W * nw;
  const int lane = threadIdx.x & 31;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  // every lane of a warp has the same i, so the whole warp takes part in each ballot
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < total; i += nwarps) {
    const int w = (int)(i % nw);
    const long long p = i / nw;
    const int x = (int)(p % y.W), yy = (int)((p / y.W) % y.H), b = (int)(p / ((long long)y.W * y.H));
    const int c = 32 * w + lane;
    const bool on = c < y.C && load1(y, pix_off(y, b, yy, x) + c) > 0.f;
    const unsigned word = __ballot_sync(0xffffffffu, on);
    if (lane == 0) bits[band_word(p, y.W, y.H, hb, row0, nw) + w] = word;
  }
}

// channel-group planar / tile-blocked views: one thread per (pixel, word), pixels fastest so that neighbouring threads
// read neighbouring pixels of one group plane; 4-channel loads never straddle a group (C % 4 == 0, cg in {4, 8})
__global__ void relu_mask_pack_cg_kernel(View y, uint32_t* __restrict__ bits, int nw, int hb, int row0) {
  const long long npix = (long long)y.B * y.H * y.W;
  const long long total = npix * nw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int w = (int)(i / npix);
    const long long p = i % npix;
    const int x = (int)(p % y.W), yy = (int)((p / y.W) % y.H), b = (int)(p / ((long long)y.W * y.H));
    unsigned word = 0;
    for (int k = 0; k < 32 && 32 * w + k < y.C; k += 4) {
      const float4 a = load4g(y, b, yy, x, 32 * w + k);
      word |= ((unsigned)(a.x > 0.f) | (unsigned)(a.y > 0.f) << 1 | (unsigned)(a.z > 0.f) << 2 |
               (unsigned)(a.w > 0.f) << 3) << k;
    }
    bits[band_word(p, y.W, y.H, hb, row0, nw) + w] = word;
  }
}

// relu_bwd_kernel with the mask read from the packed words: the same loop order, loads and stores
__global__ void relu_bwd_bits_kernel(View dy, const uint32_t* __restrict__ bits, int nw, int hb, int row0, View out) {
  const int c4 = out.C / 4;
  const long long total = (long long)out.B * out.H * out.W * c4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int q = out.cg ? (int)(i / ((long long)out.B * out.H * out.W)) : (int)(i % c4);
    const long long p = out.cg ? i % ((long long)out.B * out.H * out.W) : i / c4;
    const int x = (int)(p % out.W);
    const int yy = (int)((p / out.W) % out.H);
    const int b = (int)(p / ((long long)out.W * out.H));
    const float4 g = load4g(dy, b, yy, x, 4 * q);
    const unsigned m = __ldg(bits + band_word(p, out.W, out.H, hb, row0, nw) + (q >> 3)) >> (4 * (q & 7));  // 4q..4q+3
    store4g(out, b, yy, x, 4 * q,
            make_float4((m & 1u) ? g.x : 0.f, (m & 2u) ? g.y : 0.f, (m & 4u) ? g.z : 0.f, (m & 8u) ? g.w : 0.f));
  }
}

__global__ void fold_reflect_kernel(View gp, View add0, View add1, View out) {
  const int H = out.H, W = out.W, c4 = out.C / 4;
  const long long total = (long long)out.B * H * W * c4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(i % c4);
    const long long p = i / c4;
    const int x = (int)(p % W), y = (int)((p / W) % H), b = (int)(p / ((long long)W * H));
    // padded coordinates (1-pixel ring: gp is (H+2) x (W+2)) whose reflection lands on (y, x)
    int ys[3], xs[3], ny = 0, nx = 0;
    ys[ny++] = y + 1;
    if (y == 1) ys[ny++] = 0;
    if (y == H - 2) ys[ny++] = H + 1;
    xs[nx++] = x + 1;
    if (x == 1) xs[nx++] = 0;
    if (x == W - 2) xs[nx++] = W + 1;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int a = 0; a < ny; ++a)
      for (int e = 0; e < nx; ++e) {
        const float4 v = load4g(gp, b, ys[a], xs[e], 4 * q);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    if (add0.ptr != nullptr && 4 * q >= add0.pad && 4 * q < add0.pad + add0.C) {   // .pad re-used as channel offset
      const float4 v = load4g(add0, b, y, x, 4 * q - add0.pad);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (add1.ptr != nullptr && 4 * q >= add1.pad && 4 * q < add1.pad + add1.C) {
      const float4 v = load4g(add1, b, y, x, 4 * q - add1.pad);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    store4g(out, b, y, x, 4 * q, acc);
  }
}

int grid_for(long long total) {
  const long long blocks = (total + 255) / 256;
  return (int)(blocks < 132 * 16 ? blocks : 132 * 16);
}

// out = a + b over the whole padded extent (interior and ring) of three views of one geometry
__global__ void add_kernel(View a, View b, View out) {
  const int P = out.pad, Hp = out.H + 2 * P, Wp = out.W + 2 * P, c4 = out.C / 4;
  const long long total = (long long)out.B * Hp * Wp * c4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(i % c4);
    const long long p = i / c4;
    const int x = (int)(p % Wp) - P, y = (int)((p / Wp) % Hp) - P, bb = (int)(p / ((long long)Wp * Hp));
    const float4 u = load4g(a, bb, y, x, 4 * q), v = load4g(b, bb, y, x, 4 * q);
    store4g(out, bb, y, x, 4 * q, make_float4(u.x + v.x, u.y + v.y, u.z + v.z, u.w + v.w));
  }
}

// ---- head backward: [mask > 0] * Fold3(Conv7^T(act'(y) * dy)) --------------------------------------------------
// One CTA: HB_TH x HB_TW interior pixels x HB_CC channels of one image.  g = act'(y) * dy of the output rows / columns
// the tile's 7x7 windows reach ([y0-3, y0+TH+3) x [x0-3, x0+TW+3), zero outside the plane) and the tile's weights
// stay in shared memory.  A thread owns 4 adjacent pixels x 4 channels: per (n, ky) it reads 10 g values and 7
// weight quads for 112 FMA.
//
// Padded position (py, px) of the (H+6) x (W+6) plane receives  sum_{ky,kx} g[py-ky][px-kx] w[ky][kx]  and interior
// pixel (y, x) collects every padded position ReflectionPad2d(3) copied from it: row y+3, row 3-y (1 <= y <= 3) and
// row 2H+1-y (H-4 <= y <= H-2), the same for columns.  The main term (y+3, x+3) runs vectorised; the reflected
// terms exist only for pixels within 4 of an edge and run per pixel.  Every g they read lies inside the tile's window
// or outside the plane (the tiles are at least 4 rows / columns, so the first tile starts at 0 and the tile holding
// row H-2 reaches row H-1).
constexpr int HB_TH = 8, HB_TW = 32, HB_CC = 32, HB_GR = HB_TH + 6, HB_GC = HB_TW + 6;
constexpr int HB_THREADS = (HB_CC / 4) * (HB_TW / 4) * HB_TH;

__device__ __forceinline__ void fma4(float4& a, float g, const float4& w) {
  a.x = __fmaf_rn(g, w.x, a.x); a.y = __fmaf_rn(g, w.y, a.y); a.z = __fmaf_rn(g, w.z, a.z); a.w = __fmaf_rn(g, w.w, a.w);
}

__global__ void __launch_bounds__(HB_THREADS) head_bwd7_kernel(const float* __restrict__ y, const float* __restrict__ dy,
                                                               int N, int H, int W, int Cin,
                                                               const float* __restrict__ w, int act, View mask,
                                                               const uint32_t* __restrict__ mbits, int row0, int hout,
                                                               View out, int nchunk) {
  __shared__ float g_s[4][HB_GR][HB_GC];
  __shared__ __align__(16) float w_s[4 * 49 * HB_CC];
  const int b = blockIdx.z / nchunk, c0 = (blockIdx.z % nchunk) * HB_CC;
  const int cc = min(HB_CC, Cin - c0);
  const int y0 = row0 + blockIdx.y * HB_TH, x0 = blockIdx.x * HB_TW;     // plane rows; out holds [row0, row0+hout)
  const int tid = threadIdx.x;
  for (int i = tid; i < N * 49 * HB_CC; i += HB_THREADS) {           // w: [N][49][Cin] -> [N][49][HB_CC]
    const int c = i % HB_CC, nt = i / HB_CC;
    w_s[i] = c < cc ? w[(long long)nt * Cin + c0 + c] : 0.f;
  }
  for (int i = tid; i < N * HB_GR * HB_GC; i += HB_THREADS) {
    const int cx = i % HB_GC, r = (i / HB_GC) % HB_GR, n = i / (HB_GC * HB_GR);
    const int oy = y0 - 3 + r, ox = x0 - 3 + cx;
    float v = 0.f;
    if (oy >= 0 && oy < H && ox >= 0 && ox < W) {
      const long long o = (((long long)b * N + n) * H + oy) * W + ox;
      const float yv = y[o], d = dy[o];
      v = act == FFCB_ACT_SIGMOID ? d * (yv * (1.f - yv)) : (act == FFCB_ACT_TANH ? d * (1.f - yv * yv) : d);
    }
    g_s[n][r][cx] = v;
  }
  __syncthreads();
  const int q = tid % (HB_CC / 4), xg = (tid / (HB_CC / 4)) % (HB_TW / 4), ty = tid / ((HB_CC / 4) * (HB_TW / 4));
  float4 acc[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int n = 0; n < N; ++n) {
#pragma unroll 1
    for (int ky = 0; ky < 7; ++ky) {
      float gv[10];
#pragma unroll
      for (int j = 0; j < 10; ++j) gv[j] = g_s[n][ty + 6 - ky][xg * 4 + j];
      const float4* wr = reinterpret_cast<const float4*>(w_s + (n * 49 + ky * 7) * HB_CC) + q;
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        const float4 wv = wr[kx * (HB_CC / 4)];
#pragma unroll
        for (int j = 0; j < 4; ++j) fma4(acc[j], gv[j + 6 - kx], wv);
      }
    }
  }
  if (4 * q >= cc) return;
  const int yy = y0 + ty;
  if (yy >= row0 + hout) return;
  int rows[3], nr = 1;
  rows[0] = yy + 3;
  if (yy >= 1 && yy <= 3) rows[nr++] = 3 - yy;
  if (yy >= H - 4 && yy <= H - 2) rows[nr++] = 2 * H + 1 - yy;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int xx = x0 + xg * 4 + j;
    if (xx >= W) break;
    int cols[3], nc = 1;
    cols[0] = xx + 3;
    if (xx >= 1 && xx <= 3) cols[nc++] = 3 - xx;
    if (xx >= W - 4 && xx <= W - 2) cols[nc++] = 2 * W + 1 - xx;
    float4 r = acc[j];
    for (int a = 0; a < nr; ++a)
      for (int e = 0; e < nc; ++e) {
        if (a == 0 && e == 0) continue;                          // the main term, done above
        for (int n = 0; n < N; ++n)
          for (int ky = 0; ky < 7; ++ky) {
            const int lr = rows[a] - ky - y0 + 3;              // local row of g[py - ky]
            if (lr < 0 || lr >= HB_GR) continue;
            for (int kx = 0; kx < 7; ++kx) {
              const int lc = cols[e] - kx - x0 + 3;
              if (lc < 0 || lc >= HB_GC) continue;
              fma4(r, g_s[n][lr][lc], reinterpret_cast<const float4*>(w_s + (n * 49 + ky * 7 + kx) * HB_CC)[q]);
            }
          }
      }
    bool on[4];
    if (mbits != nullptr) {          // words of the whole plane; channels c0+4q .. +3 share one word (c0 % 32 == 0)
      const unsigned m = __ldg(mbits + (((long long)b * H + yy) * W + xx) * ((Cin + 31) / 32) + (c0 >> 5)) >> (4 * q);
      on[0] = m & 1u; on[1] = m & 2u; on[2] = m & 4u; on[3] = m & 8u;
    } else {
      const float4 m = load4g(mask, b, yy - row0, xx, c0 + 4 * q);
      on[0] = m.x > 0.f; on[1] = m.y > 0.f; on[2] = m.z > 0.f; on[3] = m.w > 0.f;
    }
    store4g(out, b, yy - row0, xx, c0 + 4 * q,
            make_float4(on[0] ? r.x : 0.f, on[1] ? r.y : 0.f, on[2] ? r.z : 0.f, on[3] ? r.w : 0.f));
  }
}

// ---- stem backward: dx = Fold3(Conv7^T(g)) ------------------------------------------------------------------------
// The adjoint of ReflectionPad2d(3) + the 7x7 stem conv (ffc.py:314-316, pix2pixhd.py:365-366) w.r.t. the generator's
// NCHW input.  Cin <= 16 outputs over K = N*49 is far too narrow for wgmma, so it runs on CUDA cores in the structure
// of head_bwd7_kernel: one CTA holds SB_TH x SB_TW interior pixels of one image, every Cin; per chunk of SB_NC gradient
// channels it stages g over the tile plus a 3-pixel apron (zero outside the plane) and that chunk's weights in shared
// memory.  A thread owns 2 pixels 16 columns apart, all CP (Cin rounded up to 4, 8 or 16) outputs.  The reflected
// terms (padded rows 3-y and 2H+1-y, columns likewise) exist for pixels within 4 of an edge and run per pixel, from
// the same shared tile (see head_bwd7_kernel for why they never leave it).  Each pixel's sum runs in one fixed order
// — per chunk the main term over (ky, kx, n), then its reflected terms — whatever the tile or the batch.
constexpr int SB_TH = 16, SB_TW = 32, SB_GR = SB_TH + 6, SB_GC = SB_TW + 6, SB_THREADS = 256;

template <int CP, int NC>
__global__ void __launch_bounds__(SB_THREADS) stem_bwd7_kernel(View g, const float* __restrict__ w, int Cin,
                                                                float* __restrict__ dx) {
  __shared__ float g_s[NC][SB_GR][SB_GC];
  __shared__ __align__(16) float w_s[49 * NC * CP];      // [tap][n][c]
  const int H = g.H, W = g.W, N = g.C;
  const int b = blockIdx.z, y0 = blockIdx.y * SB_TH, x0 = blockIdx.x * SB_TW;
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int yy = y0 + ty;
  float acc[2][CP];
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int c = 0; c < CP; ++c) acc[j][c] = 0.f;
  // padded rows / columns ReflectionPad2d(3) copied from each owned pixel: the main one first
  int rows[3], nr = 1;
  rows[0] = yy + 3;
  if (yy >= 1 && yy <= 3) rows[nr++] = 3 - yy;
  if (yy >= H - 4 && yy <= H - 2) rows[nr++] = 2 * H + 1 - yy;
  for (int n0 = 0; n0 < N; n0 += NC) {
    const int nc = min(NC, N - n0);
    __syncthreads();
    for (int i = tid; i < 49 * NC * CP; i += SB_THREADS) {       // w: [N][49][Cin] -> [49][NC][CP], zero-padded
      const int c = i % CP, nl = (i / CP) % NC, tap = i / (CP * NC);
      w_s[i] = (c < Cin && nl < nc) ? w[((long long)(n0 + nl) * 49 + tap) * Cin + c] : 0.f;
    }
    for (int i = tid; i < NC * SB_GR * SB_GC; i += SB_THREADS) {  // channels fastest: runs of NC channels per pixel
      const int nl = i % NC, cx = (i / NC) % SB_GC, r = i / (NC * SB_GC);
      const int oy = y0 - 3 + r, ox = x0 - 3 + cx;
      float v = 0.f;
      if (nl < nc && oy >= 0 && oy < H && ox >= 0 && ox < W) v = load1(g, pix_off(g, b, oy, ox) + n0 + nl);
      g_s[nl][r][cx] = v;
    }
    __syncthreads();
    // main term: padded position (y+3, x+3) receives g[y+3-ky][x+3-kx] w[ky][kx], local row ty + 6 - ky
#pragma unroll 1
    for (int ky = 0; ky < 7; ++ky)
#pragma unroll 1
      for (int kx = 0; kx < 7; ++kx)
#pragma unroll 2
        for (int nl = 0; nl < NC; ++nl) {
          const float ga = g_s[nl][ty + 6 - ky][tx + 6 - kx], gb = g_s[nl][ty + 6 - ky][tx + 22 - kx];
          const float4* wr = reinterpret_cast<const float4*>(w_s + ((ky * 7 + kx) * NC + nl) * CP);
#pragma unroll
          for (int q = 0; q < CP / 4; ++q) {
            const float4 wv = wr[q];
            acc[0][4 * q] = __fmaf_rn(ga, wv.x, acc[0][4 * q]);
            acc[0][4 * q + 1] = __fmaf_rn(ga, wv.y, acc[0][4 * q + 1]);
            acc[0][4 * q + 2] = __fmaf_rn(ga, wv.z, acc[0][4 * q + 2]);
            acc[0][4 * q + 3] = __fmaf_rn(ga, wv.w, acc[0][4 * q + 3]);
            acc[1][4 * q] = __fmaf_rn(gb, wv.x, acc[1][4 * q]);
            acc[1][4 * q + 1] = __fmaf_rn(gb, wv.y, acc[1][4 * q + 1]);
            acc[1][4 * q + 2] = __fmaf_rn(gb, wv.z, acc[1][4 * q + 2]);
            acc[1][4 * q + 3] = __fmaf_rn(gb, wv.w, acc[1][4 * q + 3]);
          }
        }
    if (yy >= H) continue;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int xx = x0 + tx + 16 * j;
      if (xx >= W) continue;
      int cols[3], ncol = 1;
      cols[0] = xx + 3;
      if (xx >= 1 && xx <= 3) cols[ncol++] = 3 - xx;
      if (xx >= W - 4 && xx <= W - 2) cols[ncol++] = 2 * W + 1 - xx;
      if (nr == 1 && ncol == 1) continue;
      for (int a = 0; a < nr; ++a)
        for (int e = 0; e < ncol; ++e) {
          if (a == 0 && e == 0) continue;                          // the main term, done above
          for (int ky = 0; ky < 7; ++ky) {
            const int lr = rows[a] - ky - y0 + 3;                  // local row of g[py - ky]
            if (lr < 0 || lr >= SB_GR) continue;
            for (int kx = 0; kx < 7; ++kx) {
              const int lc = cols[e] - kx - x0 + 3;
              if (lc < 0 || lc >= SB_GC) continue;
              for (int nl = 0; nl < NC; ++nl) {
                const float gv = g_s[nl][lr][lc];
                const float* wr = w_s + ((ky * 7 + kx) * NC + nl) * CP;
#pragma unroll
                for (int c = 0; c < CP; ++c) acc[j][c] = __fmaf_rn(gv, wr[c], acc[j][c]);
              }
            }
          }
        }
    }
  }
  if (yy >= H) return;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int xx = x0 + tx + 16 * j;
    if (xx >= W) continue;
#pragma unroll
    for (int c = 0; c < CP; ++c)
      if (c < Cin) dx[(((long long)b * Cin + c) * H + yy) * W + xx] = acc[j][c];
  }
}

}  // namespace

int stem_bwd7(const ffcb_tensor* g, const float* w, int Cin, float* dx, cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(g, "stem_bwd7.g"))) return rc;
  FFCB_REQUIRE(Cin >= 1 && Cin <= 16, "stem_bwd7: Cin=%d outside [1,16]", Cin);
  FFCB_REQUIRE(g->H >= 4 && g->W >= 4, "stem_bwd7: ReflectionPad2d(3) needs H, W >= 4 (got %dx%d)", g->H, g->W);
  FFCB_REQUIRE(!g->window, "stem_bwd7: window views are not accepted");
  FFCB_REQUIRE(w != nullptr && dx != nullptr, "stem_bwd7: null pointer");
  if ((long long)g->B * g->H * g->W * g->C == 0) return FFCB_OK;
  FFCB_REQUIRE(g->B <= 65535, "stem_bwd7: batch %d too large", g->B);
  dim3 grid((g->W + SB_TW - 1) / SB_TW, (g->H + SB_TH - 1) / SB_TH, g->B);
  const View v = make_view(*g);
  if (Cin <= 4)
    stem_bwd7_kernel<4, 8><<<grid, SB_THREADS, 0, stream>>>(v, w, Cin, dx);
  else if (Cin <= 8)
    stem_bwd7_kernel<8, 8><<<grid, SB_THREADS, 0, stream>>>(v, w, Cin, dx);
  else
    stem_bwd7_kernel<16, 4><<<grid, SB_THREADS, 0, stream>>>(v, w, Cin, dx);
  FFCB_LAUNCH_CHECK("stem_bwd7_kernel");
  return FFCB_OK;
}

int relu_bwd(const ffcb_tensor* dy, const ffcb_tensor* y, const ffcb_tensor* out, cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(dy, "relu_bwd.dy", true)) || (rc = check_tensor(y, "relu_bwd.y", true)) ||
      (rc = check_tensor(out, "relu_bwd.out", true)))
    return rc;
  FFCB_REQUIRE(dy->B == out->B && dy->H == out->H && dy->W == out->W && dy->C == out->C && y->B == out->B &&
                   y->H == out->H && y->W == out->W && y->C == out->C,
               "relu_bwd: shapes differ");
  const long long total = (long long)out->B * out->H * out->W * (out->C / 4);
  if (total == 0) return FFCB_OK;
  relu_bwd_kernel<<<grid_for(total), 256, 0, stream>>>(make_view(*dy), make_view(*y), make_view(*out));
  FFCB_LAUNCH_CHECK("relu_bwd_kernel");
  return FFCB_OK;
}

int relu_mask_pack_rows(const ffcb_tensor* y, uint32_t* bits, int hb, int row0, cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(y, "relu_mask_pack.y", true))) return rc;
  FFCB_REQUIRE(row0 >= 0 && row0 + y->H <= hb, "relu_mask_pack: rows [%d, %d) outside a plane of %d rows", row0,
               row0 + y->H, hb);
  const long long npix = (long long)y->B * y->H * y->W;
  if (npix * y->C == 0) return FFCB_OK;
  FFCB_REQUIRE(bits != nullptr && ((uintptr_t)bits % 4) == 0, "relu_mask_pack: bits must be a 4-byte aligned pointer");
  const int nw = (y->C + 31) / 32;
  const View v = make_view(*y);
  if (v.cg) {
    relu_mask_pack_cg_kernel<<<grid_for(npix * nw), 256, 0, stream>>>(v, bits, nw, hb, row0);
    FFCB_LAUNCH_CHECK("relu_mask_pack_cg_kernel");
  } else {
    relu_mask_pack_cl_kernel<<<grid_for(npix * nw * 32), 256, 0, stream>>>(v, bits, nw, hb, row0);
    FFCB_LAUNCH_CHECK("relu_mask_pack_cl_kernel");
  }
  return FFCB_OK;
}

int relu_mask_pack(const ffcb_tensor* y, uint32_t* bits, cudaStream_t stream) {
  return relu_mask_pack_rows(y, bits, y == nullptr ? 0 : y->H, 0, stream);
}

int relu_bwd_bits_rows(const ffcb_tensor* dy, const uint32_t* bits, int hb, int row0, const ffcb_tensor* out,
                       cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(dy, "relu_bwd_bits.dy", true)) || (rc = check_tensor(out, "relu_bwd_bits.out", true)))
    return rc;
  FFCB_REQUIRE(row0 >= 0 && row0 + out->H <= hb, "relu_bwd_bits: rows [%d, %d) outside a plane of %d rows", row0,
               row0 + out->H, hb);
  FFCB_REQUIRE(dy->B == out->B && dy->H == out->H && dy->W == out->W && dy->C == out->C,
               "relu_bwd_bits: shapes differ");
  const long long total = (long long)out->B * out->H * out->W * (out->C / 4);
  if (total == 0) return FFCB_OK;
  FFCB_REQUIRE(bits != nullptr && ((uintptr_t)bits % 4) == 0, "relu_bwd_bits: bits must be a 4-byte aligned pointer");
  relu_bwd_bits_kernel<<<grid_for(total), 256, 0, stream>>>(make_view(*dy), bits, (out->C + 31) / 32, hb, row0,
                                                            make_view(*out));
  FFCB_LAUNCH_CHECK("relu_bwd_bits_kernel");
  return FFCB_OK;
}

int relu_bwd_bits(const ffcb_tensor* dy, const uint32_t* bits, const ffcb_tensor* out, cudaStream_t stream) {
  return relu_bwd_bits_rows(dy, bits, out == nullptr ? 0 : out->H, 0, out, stream);
}

int fold_reflect_border(const ffcb_tensor* gpad, const ffcb_tensor* add0, int add0_c0, const ffcb_tensor* add1,
                        int add1_c0, const ffcb_tensor* out, cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(gpad, "fold.gpad")) || (rc = check_tensor(out, "fold.out"))) return rc;
  FFCB_REQUIRE(gpad->B == out->B && gpad->H == out->H + 2 && gpad->W == out->W + 2 && gpad->C == out->C,
               "fold: gpad must be (B, H+2, W+2, C) for an out of (B, H, W, C)");
  FFCB_REQUIRE(out->H >= 2 && out->W >= 2, "fold: reflect padding needs H, W >= 2");
  View va = null_view(), vb = null_view();
  const ffcb_tensor* adds[2] = {add0, add1};
  const int offs[2] = {add0_c0, add1_c0};
  View* vs[2] = {&va, &vb};
  for (int i = 0; i < 2; ++i) {
    if (adds[i] == nullptr || adds[i]->ptr == nullptr) continue;
    if ((rc = check_tensor(adds[i], "fold.addend"))) return rc;
    FFCB_REQUIRE(adds[i]->B == out->B && adds[i]->H == out->H && adds[i]->W == out->W && offs[i] % 4 == 0 &&
                     offs[i] >= 0 && offs[i] + adds[i]->C <= out->C,
                 "fold: addend %d does not fit the output (channel offset %d)", i, offs[i]);
    *vs[i] = make_view(*adds[i]);
    vs[i]->pad = offs[i];                      // the kernel reads .pad as the addend's first output channel
  }
  const long long total = (long long)out->B * out->H * out->W * (out->C / 4);
  if (total == 0) return FFCB_OK;
  fold_reflect_kernel<<<grid_for(total), 256, 0, stream>>>(make_view(*gpad), va, vb, make_view(*out));
  FFCB_LAUNCH_CHECK("fold_reflect_kernel");
  return FFCB_OK;
}

int add(const ffcb_tensor* a, const ffcb_tensor* b, const ffcb_tensor* out, cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(a, "add.a")) || (rc = check_tensor(b, "add.b")) || (rc = check_tensor(out, "add.out")))
    return rc;
  for (const ffcb_tensor* t : {a, b})
    FFCB_REQUIRE(t->B == out->B && t->H == out->H && t->W == out->W && t->C == out->C && t->pad == out->pad &&
                     !t->window,
                 "add: the three views must have one geometry (B, H, W, C, ring)");
  FFCB_REQUIRE(!out->window, "add: window views are not accepted");
  const long long total = (long long)out->B * (out->H + 2 * out->pad) * (out->W + 2 * out->pad) * (out->C / 4);
  if (total == 0) return FFCB_OK;
  add_kernel<<<grid_for(total), 256, 0, stream>>>(make_view(*a), make_view(*b), make_view(*out));
  FFCB_LAUNCH_CHECK("add_kernel");
  return FFCB_OK;
}

int head_bwd7(const float* y, const float* dy, int B, int N, int H, int W, const float* w, int act,
              const ffcb_tensor* mask, const ffcb_tensor* out, cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(mask, "head_bwd7.mask")) || (rc = check_tensor(out, "head_bwd7.out"))) return rc;
  FFCB_REQUIRE(N >= 1 && N <= 4, "head_bwd7: N=%d outside [1,4]", N);
  FFCB_REQUIRE(act == FFCB_ACT_NONE || act == FFCB_ACT_SIGMOID || act == FFCB_ACT_TANH,
               "head_bwd7: activation %d is not none / sigmoid / tanh", act);
  FFCB_REQUIRE(H >= 4 && W >= 4, "head_bwd7: ReflectionPad2d(3) needs H, W >= 4 (got %dx%d)", H, W);
  FFCB_REQUIRE(out->B == B && out->H == H && out->W == W && mask->B == B && mask->H == H && mask->W == W &&
                   mask->C == out->C && !out->window && !mask->window,
               "head_bwd7: out / mask must be (B, H, W, Cin) views of the output's plane");
  FFCB_REQUIRE(y != nullptr && dy != nullptr && w != nullptr, "head_bwd7: null pointer");
  if ((long long)B * H * W * out->C == 0) return FFCB_OK;
  const int nchunk = (out->C + HB_CC - 1) / HB_CC;
  FFCB_REQUIRE((long long)B * nchunk <= 65535, "head_bwd7: batch %d too large", B);
  dim3 grid((W + HB_TW - 1) / HB_TW, (H + HB_TH - 1) / HB_TH, B * nchunk);
  head_bwd7_kernel<<<grid, HB_THREADS, 0, stream>>>(y, dy, N, H, W, out->C, w, act, make_view(*mask), nullptr, 0, H,
                                                     make_view(*out), nchunk);
  FFCB_LAUNCH_CHECK("head_bwd7_kernel");
  return FFCB_OK;
}

int head_bwd7_bits(const float* y, const float* dy, int B, int N, int H, int W, const float* w, int act,
                   const uint32_t* mask_bits, int row0, const ffcb_tensor* out, cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(out, "head_bwd7_bits.out"))) return rc;
  FFCB_REQUIRE(N >= 1 && N <= 4, "head_bwd7_bits: N=%d outside [1,4]", N);
  FFCB_REQUIRE(act == FFCB_ACT_NONE || act == FFCB_ACT_SIGMOID || act == FFCB_ACT_TANH,
               "head_bwd7_bits: activation %d is not none / sigmoid / tanh", act);
  FFCB_REQUIRE(H >= 4 && W >= 4, "head_bwd7_bits: ReflectionPad2d(3) needs H, W >= 4 (got %dx%d)", H, W);
  FFCB_REQUIRE(out->B == B && out->W == W && row0 >= 0 && row0 + out->H <= H && !out->window,
               "head_bwd7_bits: out must be a (B, rows, W, Cin) view of rows [row0, row0+rows) of the %dx%d plane",
               H, W);
  FFCB_REQUIRE(y != nullptr && dy != nullptr && w != nullptr && mask_bits != nullptr &&
                   ((uintptr_t)mask_bits % 4) == 0,
               "head_bwd7_bits: null or misaligned pointer");
  if ((long long)B * out->H * W * out->C == 0) return FFCB_OK;
  const int nchunk = (out->C + HB_CC - 1) / HB_CC;
  FFCB_REQUIRE((long long)B * nchunk <= 65535, "head_bwd7_bits: batch %d too large", B);
  dim3 grid((W + HB_TW - 1) / HB_TW, (out->H + HB_TH - 1) / HB_TH, B * nchunk);
  head_bwd7_kernel<<<grid, HB_THREADS, 0, stream>>>(y, dy, N, H, W, out->C, w, act, null_view(), mask_bits, row0,
                                                     out->H, make_view(*out), nchunk);
  FFCB_LAUNCH_CHECK("head_bwd7_kernel");
  return FFCB_OK;
}

}  // namespace ffcb
