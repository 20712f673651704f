// Gradient of the refinement loss w.r.t. the prediction (SURVEY.md row f3; evaluation/refinement.py:75-84, 19-26,
// 151-158): the per-iteration image-space work of the refinement loop that is not the generator's rear, so that one
// Adam step (rear forward | this | rear backward | Adam) runs on the device without a host synchronisation.
//
// Per image b (NCHW float32; pred / image / grad (B,C,Hp,Wp), mask (B,1,Hp,Wp), ref (B,C,h,w), md (B,1,h,w),
// h = H0 / 2, w = W0 / 2):
//   L_b = mean_{c,p: mask < 1e-8} |pred - image| + mean_{c,q: md >= 1e-8} |D(pred[:, :, :H0, :W0]) - ref|
//   D   = bilinear(align_corners=False) to (h, w)  o  5x5 separable Gaussian with reflect-101 padding
// D is separable: D = My (x) Mx with the 1-D operator M[d][y] = l0(d) B(i0(d), y) + l1(d) B(i1(d), y), where (i0, i1,
// l0, l1) are the bilinear taps of destination d as torch's float64 interpolate computes them (src = max(scale (d + 0.5)
// - 0.5, 0), scale = in / out, in double; the weights then rounded to float — torch's float32 interpolate, the loop of
// refine_predict, computes them in float) and B(p, y) = sum_a k[a] [reflect101(p + a - 2) == y] is the weight of input
// y in blur row p.
//
// Passes (no atomics in the gradient; every output is one fixed-order gather, so image b's gradient does not depend on
// which other images share the batch):
//   init   loss[b][t] = 0, or NaN where the selection of term t is empty (torch's mean of nothing)
//   down   r[b][c][i][j] = sign(D pred - ref) [md >= 1e-8] / n_down                  (+ the second loss term)
//   full   grad = sign(pred - image) [mask < 1e-8] / n_out  +  sum_{i,j} My[i][y] Mx[j][x] r[i][j]  (inside the crop)
//                                                                                     (+ the first loss term)
// 1 / n comes from a device array (B, 2) so that a captured CUDA graph replays with the counts of the current batch.
#include <math.h>
#include <stdint.h>

#include "common.cuh"

namespace ffcb {
namespace {

constexpr int RL_THREADS = 256;
constexpr int RL_MAXT = 8;          // nonzero entries of one column of M (scale = in / (in / 2) >= 2 -> at most 4)

struct Axis {
  int in, out;
  double scale;   // the source index in double: a float one is off by ~1e-5 at d ~ 100, which the weights inherit
};

__device__ __forceinline__ int reflect101(int p, int n) {
  p = p < 0 ? -p : p;
  return p >= n ? 2 * n - 2 - p : p;
}

__device__ __forceinline__ void bilinear_taps(const Axis& a, int d, int& i0, int& i1, float& l0, float& l1) {
  double src = a.scale * ((double)d + 0.5) - 0.5;
  src = src < 0.0 ? 0.0 : src;
  i0 = (int)src;
  i1 = i0 + (i0 < a.in - 1 ? 1 : 0);
  l1 = (float)(src - (double)i0);
  l0 = (float)(1.0 - (src - (double)i0));
}

__device__ __forceinline__ float blur_weight(const float* k, int p, int y, int n) {
  float s = 0.f;
#pragma unroll
  for (int a = 0; a < 5; ++a)
    if (reflect101(p + a - 2, n) == y) s += k[a];
  return s;
}

// the nonzero M[d][y] over d for one input index y, in ascending d
__device__ __forceinline__ int adjoint_taps(const Axis& a, const float* k, int y, int* idx, float* wt) {
  // blur rows reading y lie in [y-2, y+2] (the reflection of a 2-pixel pad stays there too); i0 in [y-3, y+2]
  const int lo = max(0, (int)floor((y - 2.5) / a.scale - 0.5) - 1);
  const int hi = min(a.out - 1, (int)floor((y + 3.5) / a.scale - 0.5) + 1);
  int n = 0;
  for (int d = lo; d <= hi && n < RL_MAXT; ++d) {
    int i0, i1;
    float l0, l1;
    bilinear_taps(a, d, i0, i1, l0, l1);
    const float m = l0 * blur_weight(k, i0, y, a.in) + l1 * blur_weight(k, i1, y, a.in);
    if (m != 0.f) {
      idx[n] = d;
      wt[n] = m;
      ++n;
    }
  }
  return n;
}

__device__ __forceinline__ float sgn(float v) { return (float)((v > 0.f) - (v < 0.f)); }

// one plane's sum of v over the CTA -> one atomic per CTA (loss values only)
__device__ __forceinline__ void block_add(float v, float* dst) {
  __shared__ float part[RL_THREADS / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < RL_THREADS / 32; ++i) s += part[i];
    if (s != 0.f) atomicAdd(dst, s);
  }
}

__global__ void loss_init_kernel(const float* __restrict__ inv, float* __restrict__ loss, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) loss[i] = inv[i] > 0.f ? 0.f : __int_as_float(0x7fc00000);
}

// grid: (x blocks, B*C); one thread per low-resolution pixel of plane (b, c)
__global__ void __launch_bounds__(RL_THREADS) refine_down_kernel(const float* __restrict__ pred, int C, int Hp, int Wp,
                                                                 Axis ay, Axis ax, const float* __restrict__ ref,
                                                                 const float* __restrict__ md,
                                                                 const float* __restrict__ inv,
                                                                 const float* __restrict__ taps, float* __restrict__ r,
                                                                 float* __restrict__ loss) {
  float k[5];
#pragma unroll
  for (int a = 0; a < 5; ++a) k[a] = taps[a];
  const int plane = blockIdx.y, b = plane / C;
  const int h = ay.out, w = ax.out, H0 = ay.in, W0 = ax.in;
  const float inv_n = inv[2 * b + 1];
  const float* x = pred + (long long)plane * Hp * Wp;
  float lsum = 0.f;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < h * w; p += gridDim.x * blockDim.x) {
    const int i = p / w, j = p % w;
    float v = 0.f;
    const long long q = (long long)plane * h * w + p;
    if (md[(long long)b * h * w + p] >= 1e-8f && inv_n > 0.f) {
      int r0, r1, c0, c1;
      float ly0, ly1, lx0, lx1;
      bilinear_taps(ay, i, r0, r1, ly0, ly1);
      bilinear_taps(ax, j, c0, c1, lx0, lx1);
      float bl[2][2];
      const int rows[2] = {r0, r1}, cols[2] = {c0, c1};
#pragma unroll
      for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          // horizontal pass, then vertical (refine.gaussian_blur2d)
          float s = 0.f;
#pragma unroll
          for (int a = 0; a < 5; ++a) {
            const float* row = x + (long long)reflect101(rows[u] + a - 2, H0) * Wp;
            float t = 0.f;
#pragma unroll
            for (int bb = 0; bb < 5; ++bb) t = fmaf(k[bb], row[reflect101(cols[e] + bb - 2, W0)], t);
            s = fmaf(k[a], t, s);
          }
          bl[u][e] = s;
        }
      const float d = ly0 * (lx0 * bl[0][0] + lx1 * bl[0][1]) + ly1 * (lx0 * bl[1][0] + lx1 * bl[1][1]) - ref[q];
      v = sgn(d) * inv_n;
      lsum += fabsf(d) * inv_n;
    }
    r[q] = v;
  }
  block_add(lsum, loss + 2 * b + 1);
}

// grid: (x blocks, B*C); one thread per full-resolution pixel of plane (b, c)
__global__ void __launch_bounds__(RL_THREADS) refine_full_kernel(const float* __restrict__ pred,
                                                                 const float* __restrict__ image,
                                                                 const float* __restrict__ mask, int C, int Hp, int Wp,
                                                                 Axis ay, Axis ax, const float* __restrict__ inv,
                                                                 const float* __restrict__ taps,
                                                                 const float* __restrict__ r,
                                                                 float* __restrict__ grad, float* __restrict__ loss) {
  float k[5];
#pragma unroll
  for (int a = 0; a < 5; ++a) k[a] = taps[a];
  const int plane = blockIdx.y, b = plane / C;
  const int h = ay.out, w = ax.out;
  const float inv_out = inv[2 * b], inv_down = inv[2 * b + 1];
  const float* rp = r + (long long)plane * h * w;
  float lsum = 0.f;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < Hp * Wp; p += gridDim.x * blockDim.x) {
    const int y = p / Wp, x = p % Wp;
    const long long o = (long long)plane * Hp * Wp + p;
    float g = 0.f;
    if (mask[(long long)b * Hp * Wp + p] < 1e-8f && inv_out > 0.f) {
      const float d = pred[o] - image[o];
      g = sgn(d) * inv_out;
      lsum += fabsf(d) * inv_out;
    }
    if (y < ay.in && x < ax.in && inv_down > 0.f) {
      int iy[RL_MAXT], ix[RL_MAXT];
      float wy[RL_MAXT], wx[RL_MAXT];
      const int ny = adjoint_taps(ay, k, y, iy, wy), nx = adjoint_taps(ax, k, x, ix, wx);
      float acc = 0.f;
      for (int u = 0; u < ny; ++u) {
        const float* row = rp + (long long)iy[u] * w;
        float s = 0.f;
        for (int e = 0; e < nx; ++e) s = fmaf(wx[e], row[ix[e]], s);
        acc = fmaf(wy[u], s, acc);
      }
      g += acc;
    }
    grad[o] = g;
  }
  block_add(lsum, loss + 2 * b);
}

int plane_blocks(long long n) {
  const long long blocks = (n + RL_THREADS - 1) / RL_THREADS;
  return (int)(blocks < 64 ? blocks : 64);
}

}  // namespace

int refine_l1_grad(const float* pred, const float* image, const float* mask, int B, int C, int Hp, int Wp, int H0,
                   int W0, const float* ref, const float* md, const float* inv_n, const float* taps, float* work,
                   float* grad, float* loss, cudaStream_t stream) {
  FFCB_REQUIRE(pred && image && mask && ref && md && inv_n && taps && work && grad && loss,
               "refine_l1_grad: null pointer");
  FFCB_REQUIRE(B >= 1 && (long long)B * C <= 65535, "refine_l1_grad: batch %d out of range", B);
  FFCB_REQUIRE(C >= 1 && C <= 4, "refine_l1_grad: C=%d outside [1,4]", C);
  FFCB_REQUIRE(H0 >= 3 && W0 >= 3 && H0 <= Hp && W0 <= Wp,
               "refine_l1_grad: crop %dx%d must be >= 3x3 and inside the %dx%d plane", H0, W0, Hp, Wp);
  const Axis ay{H0, H0 / 2, (double)H0 / (H0 / 2)}, ax{W0, W0 / 2, (double)W0 / (W0 / 2)};
  loss_init_kernel<<<(2 * B + 127) / 128, 128, 0, stream>>>(inv_n, loss, 2 * B);
  FFCB_LAUNCH_CHECK("refine_loss_init_kernel");
  refine_down_kernel<<<dim3(plane_blocks((long long)ay.out * ax.out), B * C), RL_THREADS, 0, stream>>>(
      pred, C, Hp, Wp, ay, ax, ref, md, inv_n, taps, work, loss);
  FFCB_LAUNCH_CHECK("refine_down_kernel");
  refine_full_kernel<<<dim3(plane_blocks((long long)Hp * Wp), B * C), RL_THREADS, 0, stream>>>(
      pred, image, mask, C, Hp, Wp, ay, ax, inv_n, taps, work, grad, loss);
  FFCB_LAUNCH_CHECK("refine_full_kernel");
  return FFCB_OK;
}

}  // namespace ffcb
