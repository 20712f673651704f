// Generator shell kernels and layout adapters:
//   stem_conv7  : ReflectionPad2d(3) + Conv2d(Cin->N, 7x7) + folded BN + ReLU, NCHW float in -> NHWC out
//                 (reference ffc.py:315-317, 253)
//   head_conv7  : ReflectionPad2d(3) + Conv2d(C->N<=4, 7x7, bias) + activation, NHWC in -> NCHW float out
//                 (reference ffc.py:360-363)
//   nchw<->nhwc : module-boundary layout conversion (the reference's tensors are NCHW float)
//   reflect ring: (re)build the 1-pixel reflected border of a padded view
#include "common.cuh"

namespace ffcb {
namespace {

constexpr int HALO = 3;            // 7x7
constexpr int TX = 32, TY = 16;    // output tile per CTA: 32 columns (lane == column) x 16 rows
constexpr int PW = TX + 2 * HALO;  // 38
constexpr int PH = TY + 2 * HALO;  // 22
constexpr int kShellThreads = 128; // 4 warps: warp w owns rows {w, w+4, w+8, w+12} (stem) / {4w..4w+3} (head)

// ---------------------------------------------------------------------------------------- stem
// Register tile: 4 pixels (same column, rows w + 4r) x 16 output channels per thread; blockIdx.z walks
// the output channels 16 at a time.  Per (tap, input channel): 4 conflict-free scalar patch reads +
// 4 broadcast float4 weight reads feed 64 FMAs, so the kernel is FMA-issue bound rather than
// shared-memory bound.  smem: patch[Cin][22][38], w[49*Cin][16].
constexpr int SN = 16;
__global__ void __launch_bounds__(kShellThreads) stem_conv7_kernel(const float* __restrict__ x, int B, int Cin, int H,
                                                                   int W, const float* __restrict__ w,
                                                                   const float* __restrict__ shift, int N, View out) {
  extern __shared__ __align__(16) float smem[];
  float* patch = smem;
  float* ws = smem + ((Cin * PH * PW + 3) & ~3);
  const int tx = threadIdx.x & 31, wy = threadIdx.x >> 5;
  const int tiles_x = (W + TX - 1) / TX;
  const int x0 = (blockIdx.x % tiles_x) * TX, y0 = (blockIdx.x / tiles_x) * TY;
  const int b = blockIdx.y;
  const int n0 = blockIdx.z * SN;
  const int K = 49 * Cin;

  for (int i = threadIdx.x; i < Cin * PH * PW; i += blockDim.x) {
    const int c = i / (PH * PW), r = i % (PH * PW);
    // reflect, then clamp for tiles hanging over the image edge (those values feed no in-range pixel)
    const int yy = min(max(reflect_idx(y0 + r / PW - HALO, H), 0), H - 1);
    const int xx = min(max(reflect_idx(x0 + r % PW - HALO, W), 0), W - 1);
    patch[i] = __ldg(x + (((long long)b * Cin + c) * H + yy) * W + xx);
  }
  for (int i = threadIdx.x; i < K * SN; i += blockDim.x) {
    const int k = i / SN, j = i % SN;
    ws[i] = (n0 + j < N) ? __ldg(w + (long long)k * N + n0 + j) : 0.f;
  }
  __syncthreads();

  // accumulators as channel pairs (ffma2: one rounding per lane)
  float2 acc[4][SN / 2];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int j = 0; j < SN / 2; ++j) acc[r][j] = make_float2(0.f, 0.f);

  for (int ky = 0; ky < 7; ++ky) {
    for (int c = 0; c < Cin; ++c) {
      const float* prow = patch + (c * PH + wy + ky) * PW + tx;
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        const float4* wr = reinterpret_cast<const float4*>(ws + ((ky * 7 + kx) * Cin + c) * SN);
        const float4 w0 = wr[0], w1 = wr[1], w2 = wr[2], w3 = wr[3];
        const float2 wv[SN / 2] = {make_float2(w0.x, w0.y), make_float2(w0.z, w0.w), make_float2(w1.x, w1.y),
                                   make_float2(w1.z, w1.w), make_float2(w2.x, w2.y), make_float2(w2.z, w2.w),
                                   make_float2(w3.x, w3.y), make_float2(w3.z, w3.w)};
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const float a = prow[4 * r * PW + kx];
          const float2 aa = make_float2(a, a);
#pragma unroll
          for (int j = 0; j < SN / 2; ++j) acc[r][j] = ffma2(aa, wv[j], acc[r][j]);
        }
      }
    }
  }

  const int xo = x0 + tx;
  if (xo >= W) return;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int y = y0 + wy + 4 * r;
    if (y >= H) continue;
    const long long o = pix_off(out, b, y, xo);
#pragma unroll
    for (int q = 0; q < SN / 4; ++q) {
      const int n = n0 + 4 * q;
      if (n >= N) break;
      float4 v = make_float4(acc[r][2 * q].x, acc[r][2 * q].y, acc[r][2 * q + 1].x, acc[r][2 * q + 1].y);
      if (shift != nullptr) {
        const float4 sh = __ldg(reinterpret_cast<const float4*>(shift + n));
        v.x += sh.x; v.y += sh.y; v.z += sh.z; v.w += sh.w;
      }
      v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
      store4(out, o + n, v);
    }
  }
}

// ---------------------------------------------------------------------------------------- stem pack
// NCHW float -> reflect-padded NHWC8 (split bf16 or fp32): one thread per padded pixel, 8 channels = one
// 16-byte (bf16) store per plane.  Feeds the tensor-core stem through a sliding-window view.
// Cin <= 4 ("two-row" packing): channels 4..7 of padded pixel (yp, xp) hold channels 0..3 of pixel (yp+1, xp), so one
// 64-element window (8 taps x 8 channels) covers TWO kernel rows and the 7x7 stem is four K-segments instead of seven.
__global__ void stem_pack_kernel(const float* __restrict__ x, int Cin, int H, int W, View out) {
  const int Wp = out.W, Hp = out.H;           // W + 8, H + 6
  const long long total = (long long)out.B * Hp * Wp;
  const bool two_rows = Cin <= 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int xp = (int)(i % Wp);
    const int yp = (int)((i / Wp) % Hp);
    const int b = (int)(i / ((long long)Wp * Hp));
    float v[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] = 0.f;
    if (xp < W + 6) {
      const int yy = reflect_idx(yp - HALO, H), xx = reflect_idx(xp - HALO, W);
      const int y2 = reflect_idx(yp + 1 - HALO, H);
      const bool row2 = two_rows && yp + 1 < Hp;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        if (c < Cin) v[c] = __ldg(x + (((long long)b * Cin + c) * H + yy) * W + xx);
        else if (row2 && c >= 4 && c - 4 < Cin) v[c] = __ldg(x + (((long long)b * Cin + (c - 4)) * H + y2) * W + xx);
      }
    }
    const long long o = pix_off(out, b, yp, xp);
    store4(out, o, make_float4(v[0], v[1], v[2], v[3]));
    store4(out, o + 4, make_float4(v[4], v[5], v[6], v[7]));
  }
}

// uint8 front end of the predict path (SURVEY.md row f1): decode + pad_img_to_modulo('symmetric') + mask
// binarisation + mask multiply + channel concat + ReflectionPad2d(3), written straight into the packed stem image.
//   reference: evaluation/data.py:11-19 (u8 / 255, float32), :32-36 (np.pad symmetric to a multiple of 8),
//              bin/predict.py:83 (mask > 0), trainers/default.py:59 (img * (1 - mask)), :68 (cat mask)
// image: [B][H0][W0][3] (decoded RGB), mask: [B][H0][W0]; the padded size (H, W) comes from the packed view.
__device__ __forceinline__ int symmetric_idx(int i, int n0) { return i < n0 ? i : 2 * n0 - 1 - i; }

__global__ void stem_pack_u8_kernel(const uint8_t* __restrict__ img, const uint8_t* __restrict__ mask, int H0, int W0,
                                    View out) {
  const int Wp = out.W, Hp = out.H, H = Hp - 2 * HALO, W = Wp - 8;
  const long long total = (long long)out.B * Hp * Wp;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int xp = (int)(i % Wp);
    const int yp = (int)((i / Wp) % Hp);
    const int b = (int)(i / ((long long)Wp * Hp));
    // decoded + masked pixel at padded coordinates (yq, xp): (img * (1 - mask), mask)
    auto fetch = [&](int yq) {
      float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
      const int ys = symmetric_idx(reflect_idx(yq - HALO, H), H0), xs = symmetric_idx(reflect_idx(xp - HALO, W), W0);
      const long long p = ((long long)b * H0 + ys) * W0 + xs;
      if (__ldg(mask + p) > 0) {
        r.w = 1.f;                                   // img * (1 - 1) = +0, mask channel = 1
      } else {                                       // img * (1 - 0) = img exactly
        r.x = __fdiv_rn((float)__ldg(img + 3 * p + 0), 255.f);
        r.y = __fdiv_rn((float)__ldg(img + 3 * p + 1), 255.f);
        r.z = __fdiv_rn((float)__ldg(img + 3 * p + 2), 255.f);
      }
      return r;
    };
    float4 lo = make_float4(0.f, 0.f, 0.f, 0.f), hi = lo;      // hi: the pixel one row below (two-row packing)
    if (xp < W + 2 * HALO) {
      lo = fetch(yp);
      if (yp + 1 < Hp) hi = fetch(yp + 1);
    }
    const long long o = pix_off(out, b, yp, xp);
    store4(out, o, lo);
    store4(out, o + 4, hi);
  }
}

// ---------------------------------------------------------------------------------------- head
// Register tile: 4 vertically adjacent pixels x (N <= 4) outputs per thread.  For one (kx, channel quad)
// the 10 patch rows a thread needs are loaded once (float4, conflict-free: pixel pitch 20 floats) and
// reused by the 4 pixels x 7 ky taps; weights are broadcast float4 reads.  Channels are staged 16 at a time:
// patch[22][38][PSTR] floats, w[4][49][16].
constexpr int HC = 16, PSTR = 20;

__global__ void __launch_bounds__(kShellThreads) head_conv7_kernel(View in, const float* __restrict__ w,
                                                                   const float* __restrict__ bias, int N, int act,
                                                                   float* __restrict__ y_out) {
  extern __shared__ __align__(16) float smem[];
  float* patch = smem;                  // [PH*PW][PSTR]
  float* ws = smem + PH * PW * PSTR;    // [4][49][HC]
  const int tx = threadIdx.x & 31, wy = threadIdx.x >> 5;
  const int H = in.H, W = in.W, C = in.C;
  const int tiles_x = (W + TX - 1) / TX;
  const int x0 = (blockIdx.x % tiles_x) * TX, y0 = (blockIdx.x / tiles_x) * TY;
  const int b = blockIdx.y;

  // two partial sums per output (even / odd channels), accumulated as float2 pairs
  float2 acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int n = 0; n < 4; ++n) acc[r][n] = make_float2(0.f, 0.f);

  for (int c0 = 0; c0 < C; c0 += HC) {
    for (int i = threadIdx.x; i < PH * PW * (HC / 4); i += blockDim.x) {
      const int pix = i / (HC / 4), q = i % (HC / 4);
      const int yy = min(max(reflect_idx(y0 + pix / PW - HALO, H), 0), H - 1);
      const int xx = min(max(reflect_idx(x0 + pix % PW - HALO, W), 0), W - 1);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c0 + 4 * q < C) v = load4(in, pix_off(in, b, yy, xx) + c0 + 4 * q);
      *reinterpret_cast<float4*>(patch + pix * PSTR + 4 * q) = v;
    }
    for (int i = threadIdx.x; i < 4 * 49 * HC; i += blockDim.x) {
      const int n = i / (49 * HC), r = i % (49 * HC), t = r / HC, c = r % HC;
      ws[i] = (n < N && c0 + c < C) ? __ldg(w + ((long long)n * 49 + t) * C + c0 + c) : 0.f;
    }
    __syncthreads();
    for (int kx = 0; kx < 7; ++kx) {
#pragma unroll
      for (int q = 0; q < HC / 4; ++q) {
        float4 a[10];
        const float* pp = patch + ((4 * wy) * PW + tx + kx) * PSTR + 4 * q;
#pragma unroll
        for (int j = 0; j < 10; ++j) a[j] = *reinterpret_cast<const float4*>(pp + j * PW * PSTR);
#pragma unroll
        for (int ky = 0; ky < 7; ++ky) {
#pragma unroll
          for (int n = 0; n < 3; ++n) {
            const float4 wv = *reinterpret_cast<const float4*>(ws + (n * 49 + ky * 7 + kx) * HC + 4 * q);
            const float2 wlo = make_float2(wv.x, wv.y), whi = make_float2(wv.z, wv.w);
#pragma unroll
            for (int r = 0; r < 4; ++r) {
              acc[r][n] = ffma2(make_float2(a[r + ky].x, a[r + ky].y), wlo, acc[r][n]);
              acc[r][n] = ffma2(make_float2(a[r + ky].z, a[r + ky].w), whi, acc[r][n]);
            }
          }
          if (N == 4) {
            const float4 wv = *reinterpret_cast<const float4*>(ws + (3 * 49 + ky * 7 + kx) * HC + 4 * q);
            const float2 wlo = make_float2(wv.x, wv.y), whi = make_float2(wv.z, wv.w);
#pragma unroll
            for (int r = 0; r < 4; ++r) {
              acc[r][3] = ffma2(make_float2(a[r + ky].x, a[r + ky].y), wlo, acc[r][3]);
              acc[r][3] = ffma2(make_float2(a[r + ky].z, a[r + ky].w), whi, acc[r][3]);
            }
          }
        }
      }
    }
    __syncthreads();
  }
  const int xo = x0 + tx;
  if (xo >= W) return;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int y = y0 + 4 * wy + r;
    if (y >= H) continue;
#pragma unroll
    for (int n = 0; n < 4; ++n) {       // static indices keep acc[][] in registers
      if (n < N) {
        const float v = apply_act(acc[r][n].x + acc[r][n].y + (bias ? __ldg(bias + n) : 0.f), act);
        y_out[(((long long)b * N + n) * H + y) * W + xo] = v;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------- layout
// [C][W] <-> [W][C] transposes per (b, y) row through a 32x33 shared tile.
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, int C, int H, int W, View out) {
  __shared__ float tile[32][33];
  const int c0 = blockIdx.y * 32, x0 = blockIdx.x * 32;
  for (int z = blockIdx.z; z < out.B * H; z += gridDim.z) {      // (image, row) pairs: grid.z is capped at 65535
    const int b = z / H, y = z % H;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
      const int c = c0 + i, xx = x0 + threadIdx.x;
      tile[i][threadIdx.x] = (c < C && xx < W) ? __ldg(x + (((long long)b * C + c) * H + y) * W + xx) : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
      const int xx = x0 + i, c = c0 + threadIdx.x;
      if (xx < W && c < C) store1(out, elem_off(out, b, y, xx, c), tile[threadIdx.x][i]);
    }
    __syncthreads();
  }
}

__global__ void nhwc_to_nchw_kernel(View in, float* __restrict__ yo) {
  __shared__ float tile[32][33];
  const int H = in.H, W = in.W, C = in.C;
  const int c0 = blockIdx.y * 32, x0 = blockIdx.x * 32;
  for (int z = blockIdx.z; z < in.B * H; z += gridDim.z) {
    const int b = z / H, y = z % H;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
      const int xx = x0 + i, c = c0 + threadIdx.x;
      tile[i][threadIdx.x] = (xx < W && c < C) ? load1(in, elem_off(in, b, y, xx, c)) : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
      const int c = c0 + i, xx = x0 + threadIdx.x;
      if (c < C && xx < W) yo[(((long long)b * C + c) * H + y) * W + xx] = tile[threadIdx.x][i];
    }
    __syncthreads();
  }
}

// Reflected ring of a padded view (pad = 1..3): every pixel of the padded plane outside the interior copies
// interior pixel (reflect(y), reflect(x)).
__global__ void reflect_ring_kernel(View t) {
  const int p = t.pad, Wp = t.W + 2 * p;
  const int band = p * Wp;                       // pixels of the top (and of the bottom) band
  const int ring = 2 * band + 2 * p * t.H;       // ring pixels per image
  const int c4 = t.C / 4;
  const long long total = (long long)t.B * ring * c4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(i % c4);
    const long long pi = i / c4;
    int r = (int)(pi % ring);
    const int b = (int)(pi / ring);
    int y, x;
    if (r < band) { y = r / Wp - p; x = r % Wp - p; }
    else if (r < 2 * band) { r -= band; y = t.H + r / Wp; x = r % Wp - p; }
    else { r -= 2 * band; y = r / (2 * p); const int j = r % (2 * p); x = j < p ? j - p : t.W + (j - p); }
    const float4 v = load4(t, pix_off(t, b, reflect_idx(y, t.H), reflect_idx(x, t.W)) + 4 * q);
    store4(t, pix_off(t, b, y, x) + 4 * q, v);
  }
}

// Head gather: y[b,n,y,x] = act(bias[n] + sum_kx q[b,y,reflect(x+kx-3),n*7+kx]).  One CTA = 128 consecutive
// pixels of a row; the (128+6) x 7N partial sums are staged through shared memory (row pitch 7N+1: conflict-free).
constexpr int GT = 128;
// Output rows [row0, row0 + q.H) of an NCHW plane of hout rows (hout = q.H, row0 = 0: the whole plane).
__global__ void __launch_bounds__(GT) head_gather7_kernel(View q, const float* __restrict__ bias, int N, int act,
                                                          float* __restrict__ y_out, int hout, int row0) {
  extern __shared__ float tile[];
  const int nq = 7 * N, pitch = nq + 1;
  const int tiles_x = (q.W + GT - 1) / GT;
  const int x0 = (blockIdx.x % tiles_x) * GT, y = blockIdx.x / tiles_x, b = blockIdx.y;
  for (int i = threadIdx.x; i < (GT + 6) * nq; i += GT) {
    const int px = i / nq, j = i % nq;
    const int xx = min(max(reflect_idx(x0 + px - 3, q.W), 0), q.W - 1);
    tile[px * pitch + j] = load1(q, pix_off(q, b, y, xx) + j);
  }
  __syncthreads();
  const int x = x0 + threadIdx.x;
  if (x >= q.W) return;
  for (int n = 0; n < N; ++n) {
    float acc = bias ? __ldg(bias + n) : 0.f;
#pragma unroll
    for (int kx = 0; kx < 7; ++kx) acc += tile[(threadIdx.x + kx) * pitch + n * 7 + kx];
    y_out[(((long long)b * N + n) * hout + row0 + y) * q.W + x] = apply_act(acc, act);
  }
}

// uint8 back end of the predict path (row f1): head gather + output activation + blend with the input image +
// crop to the unpadded size + x255 / clip / truncate, RGB bytes out.
//   reference: trainers/default.py:71 (mask * predicted + (1 - mask) * image — an exact select for mask in {0,1}),
//              bin/predict.py:86-91 (unpad_to_size crop), :93 (np.clip(res * 255, 0, 255).astype('uint8'))
// q is over the padded image (reflection about the padded width); out: [B][H0][W0][3].
__global__ void __launch_bounds__(GT) head_gather7_blend_u8_kernel(View q, const float* __restrict__ bias, int act,
                                                                   const uint8_t* __restrict__ img,
                                                                   const uint8_t* __restrict__ mask, int H0, int W0,
                                                                   uint8_t* __restrict__ out) {
  extern __shared__ float tile[];
  constexpr int nq = 21, pitch = nq + 1;
  const int tiles_x = (W0 + GT - 1) / GT;
  const int x0 = (blockIdx.x % tiles_x) * GT, y = blockIdx.x / tiles_x, b = blockIdx.y;
  for (int i = threadIdx.x; i < (GT + 6) * nq; i += GT) {
    const int px = i / nq, j = i % nq;
    const int xx = min(max(reflect_idx(x0 + px - 3, q.W), 0), q.W - 1);
    tile[px * pitch + j] = load1(q, pix_off(q, b, y, xx) + j);
  }
  __syncthreads();
  const int x = x0 + threadIdx.x;
  if (x >= W0) return;
  const long long p = ((long long)b * H0 + y) * W0 + x;
  const bool hole = __ldg(mask + p) > 0;
#pragma unroll
  for (int n = 0; n < 3; ++n) {
    float v;
    if (hole) {
      float acc = bias ? __ldg(bias + n) : 0.f;
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) acc += tile[(threadIdx.x + kx) * pitch + n * 7 + kx];
      v = apply_act(acc, act);
    } else {
      v = __fdiv_rn((float)__ldg(img + 3 * p + n), 255.f);
    }
    v = fminf(fmaxf(__fmul_rn(v, 255.f), 0.f), 255.f);
    out[3 * p + n] = (uint8_t)(int)v;            // float -> int truncates toward zero like astype('uint8')
  }
}

}  // namespace

int stem_conv7(const float* x, int B, int Cin, int H, int W, const float* w, const float* shift, int N,
               const ffcb_tensor* out, cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(out, "stem_conv7.out"))) return rc;
  FFCB_REQUIRE(x && w, "stem_conv7: null pointer");
  FFCB_REQUIRE(Cin >= 1 && Cin <= 16, "stem_conv7: Cin=%d outside [1,16]", Cin);
  FFCB_REQUIRE(H >= 4 && W >= 4, "stem_conv7: reflect pad 3 needs H,W >= 4 (got %dx%d)", H, W);
  FFCB_REQUIRE(N % 4 == 0 && N >= 4, "stem_conv7: N=%d must be a positive multiple of 4", N);
  FFCB_REQUIRE(out->B == B && out->H == H && out->W == W && out->C == N, "stem_conv7: out view shape mismatch");
  FFCB_REQUIRE(B <= 65535, "stem_conv7: batch exceeds grid.y");
  if (B == 0) return FFCB_OK;
  const size_t smem = sizeof(float) * (((size_t)Cin * PH * PW + 3) / 4 * 4 + (size_t)49 * Cin * SN);
  if (smem > 48 * 1024)
    FFCB_CUDA(cudaFuncSetAttribute(stem_conv7_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(((W + TX - 1) / TX) * ((H + TY - 1) / TY), B, (N + SN - 1) / SN);
  stem_conv7_kernel<<<grid, kShellThreads, smem, stream>>>(x, B, Cin, H, W, w, shift, N, make_view(*out));
  FFCB_LAUNCH_CHECK("stem_conv7_kernel");
  return FFCB_OK;
}

int stem_pack(const float* x, int B, int Cin, int H, int W, const ffcb_tensor* packed, cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(packed, "stem_pack.packed"))) return rc;
  FFCB_REQUIRE(x != nullptr, "stem_pack: null input");
  FFCB_REQUIRE(Cin >= 1 && Cin <= 8, "stem_pack: Cin=%d outside [1,8]", Cin);
  FFCB_REQUIRE(H >= 4 && W >= 4, "stem_pack: reflect pad 3 needs H,W >= 4");
  FFCB_REQUIRE(packed->B == B && packed->H == H + 6 && packed->W == W + 8 && packed->C == 8 && !packed->window,
               "stem_pack: packed view must be (B, H+6, W+8, 8)");
  const long long total = (long long)B * (H + 6) * (W + 8);
  if (total == 0) return FFCB_OK;
  const int blocks = (int)((total + 255) / 256 < 132 * 16 ? (total + 255) / 256 : 132 * 16);
  stem_pack_kernel<<<blocks, 256, 0, stream>>>(x, Cin, H, W, make_view(*packed));
  FFCB_LAUNCH_CHECK("stem_pack_kernel");
  return FFCB_OK;
}

int stem_pack_u8(const uint8_t* img, const uint8_t* mask, int B, int H0, int W0, const ffcb_tensor* packed,
                 cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(packed, "stem_pack_u8.packed"))) return rc;
  FFCB_REQUIRE(img != nullptr && mask != nullptr, "stem_pack_u8: null input");
  const int H = packed->H - 6, W = packed->W - 8;
  FFCB_REQUIRE(packed->B == B && packed->C == 8 && !packed->window && H >= 4 && W >= 4,
               "stem_pack_u8: packed view must be (B, H+6, W+8, 8) with H, W >= 4");
  FFCB_REQUIRE(H0 >= 1 && W0 >= 1 && H0 <= H && W0 <= W && H - H0 <= H0 && W - W0 <= W0,
               "stem_pack_u8: %dx%d cannot be symmetric-padded to %dx%d", H0, W0, H, W);
  const long long total = (long long)B * (H + 6) * (W + 8);
  if (total == 0) return FFCB_OK;
  const int blocks = (int)((total + 255) / 256 < 132 * 16 ? (total + 255) / 256 : 132 * 16);
  stem_pack_u8_kernel<<<blocks, 256, 0, stream>>>(img, mask, H0, W0, make_view(*packed));
  FFCB_LAUNCH_CHECK("stem_pack_u8_kernel");
  return FFCB_OK;
}

int head_gather7_blend_u8(const ffcb_tensor* q, const float* bias, int act, const uint8_t* img, const uint8_t* mask,
                          int H0, int W0, uint8_t* out, cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(q, "head_gather7_blend_u8.q"))) return rc;
  FFCB_REQUIRE(img && mask && out, "head_gather7_blend_u8: null pointer");
  FFCB_REQUIRE(q->C >= 21, "head_gather7_blend_u8: q.C=%d < 21 (three outputs x seven taps)", q->C);
  FFCB_REQUIRE(q->W >= 4 && q->B <= 65535, "head_gather7_blend_u8: W >= 4 and B <= 65535 required");
  FFCB_REQUIRE(H0 >= 1 && W0 >= 1 && H0 <= q->H && W0 <= q->W, "head_gather7_blend_u8: crop %dx%d outside %dx%d", H0,
               W0, q->H, q->W);
  if (q->B == 0) return FFCB_OK;
  dim3 grid(((W0 + GT - 1) / GT) * H0, q->B);
  const size_t smem = sizeof(float) * (GT + 6) * 22;
  head_gather7_blend_u8_kernel<<<grid, GT, smem, stream>>>(make_view(*q), bias, act, img, mask, H0, W0, out);
  FFCB_LAUNCH_CHECK("head_gather7_blend_u8_kernel");
  return FFCB_OK;
}

int head_gather7_rows(const ffcb_tensor* q, const float* bias, int N, int act, float* y, int hout, int row0,
                      cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(q, "head_gather7.q"))) return rc;
  FFCB_REQUIRE(row0 >= 0 && row0 + q->H <= hout, "head_gather7: rows [%d, %d) outside an output of %d rows", row0,
               row0 + q->H, hout);
  FFCB_REQUIRE(y != nullptr, "head_gather7: null output");
  FFCB_REQUIRE(N >= 1 && N <= 4 && q->C >= 7 * N, "head_gather7: need 1 <= N <= 4 and q.C >= 7N (N=%d, C=%d)", N, q->C);
  FFCB_REQUIRE(q->W >= 4 && q->B <= 65535, "head_gather7: W >= 4 and B <= 65535 required");
  if (q->B == 0) return FFCB_OK;
  dim3 grid(((q->W + GT - 1) / GT) * q->H, q->B);
  const size_t smem = sizeof(float) * (GT + 6) * (7 * N + 1);
  head_gather7_kernel<<<grid, GT, smem, stream>>>(make_view(*q), bias, N, act, y, hout, row0);
  FFCB_LAUNCH_CHECK("head_gather7_kernel");
  return FFCB_OK;
}

int head_gather7(const ffcb_tensor* q, const float* bias, int N, int act, float* y, cudaStream_t stream) {
  return head_gather7_rows(q, bias, N, act, y, q == nullptr ? 0 : q->H, 0, stream);
}

int head_conv7(const ffcb_tensor* in, const float* w, const float* bias, int N, int act, float* y,
               cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(in, "head_conv7.in"))) return rc;
  FFCB_REQUIRE(w && y, "head_conv7: null pointer");
  FFCB_REQUIRE(N >= 1 && N <= 4, "head_conv7: N=%d outside [1,4]", N);
  FFCB_REQUIRE(in->H >= 4 && in->W >= 4, "head_conv7: reflect pad 3 needs H,W >= 4");
  if (in->B == 0) return FFCB_OK;
  FFCB_REQUIRE(in->B <= 65535, "head_conv7: batch exceeds grid.y");
  dim3 grid(((in->W + TX - 1) / TX) * ((in->H + TY - 1) / TY), in->B);
  constexpr size_t smem = sizeof(float) * (PH * PW * PSTR + 4 * 49 * HC);
  FFCB_CUDA(cudaFuncSetAttribute(head_conv7_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  head_conv7_kernel<<<grid, kShellThreads, smem, stream>>>(make_view(*in), w, bias, N, act, y);
  FFCB_LAUNCH_CHECK("head_conv7_kernel");
  return FFCB_OK;
}

int nchw_to_nhwc(const float* x, int B, int C, int H, int W, const ffcb_tensor* out, cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(out, "nchw_to_nhwc.out", true))) return rc;
  FFCB_REQUIRE(out->B == B && out->C == C && out->H == H && out->W == W, "nchw_to_nhwc: shape mismatch");
  if ((long long)B * C * H * W == 0) return FFCB_OK;
  const long long rows = (long long)B * H;
  dim3 grid((W + 31) / 32, (C + 31) / 32, (unsigned)(rows < 65535 ? rows : 65535)), block(32, 8);
  nchw_to_nhwc_kernel<<<grid, block, 0, stream>>>(x, C, H, W, make_view(*out));
  FFCB_LAUNCH_CHECK("nchw_to_nhwc_kernel");
  return FFCB_OK;
}

int nhwc_to_nchw(const ffcb_tensor* in, float* y, cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(in, "nhwc_to_nchw.in", true))) return rc;
  if ((long long)in->B * in->C * in->H * in->W == 0) return FFCB_OK;
  const long long rows = (long long)in->B * in->H;
  dim3 grid((in->W + 31) / 32, (in->C + 31) / 32, (unsigned)(rows < 65535 ? rows : 65535)), block(32, 8);
  nhwc_to_nchw_kernel<<<grid, block, 0, stream>>>(make_view(*in), y);
  FFCB_LAUNCH_CHECK("nhwc_to_nchw_kernel");
  return FFCB_OK;
}

int fill_reflect_border(const ffcb_tensor* t, cudaStream_t stream) {
  int rc;
  if ((rc = check_tensor(t, "fill_reflect_border"))) return rc;
  FFCB_REQUIRE(t->pad >= 1, "fill_reflect_border: view has no border ring (pad=%d)", t->pad);
  FFCB_REQUIRE(t->H > t->pad && t->W > t->pad, "fill_reflect_border: reflect needs H,W > pad");
  const long long total = (long long)t->B * (2 * t->pad * (t->W + 2 * t->pad) + 2 * t->pad * t->H) * (t->C / 4);
  if (total == 0) return FFCB_OK;
  const int blocks = (int)((total + 255) / 256 < 132 * 8 ? (total + 255) / 256 : 132 * 8);
  reflect_ring_kernel<<<blocks, 256, 0, stream>>>(make_view(*t));
  FFCB_LAUNCH_CHECK("reflect_ring_kernel");
  return FFCB_OK;
}

}  // namespace ffcb
