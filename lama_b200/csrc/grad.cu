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

}  // namespace

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

}  // namespace ffcb
