// FP32 CUDA-core implicit-GEMM convolution over channels-last tensors (FFCB_MATH_FP32).
//
// Reference-grade arm of ffcb_conv(): fp32 operands, FFMA, fp32 accumulate — same arithmetic as
// the reference's fp32 convolutions (ffc.py:189-196, 129, 139, 57-59) with BatchNorm folded into
// weights/shift and bias/residual/activation fused into the epilogue.  The tensor-core arm
// (conv_tc.cu) implements the same ffcb_conv_desc contract and is checked against this one.
//
// Tiling: 128 output pixels x 64 output channels per CTA, K stepped 16 channels at a time through
// the K-segment list (tap, channel range); 256 threads, 8x4 register tile, register prefetch of
// the next K step while the current one is multiplied.
#include "common.cuh"

namespace ffcb {
namespace {

constexpr int BM = 128, BN = 64, BK = 16, NT = 256;
constexpr int AS = BM + 4;  // padded row length of the A tile

struct SimtParams {
  View in[2];
  View out;
  View addend;
  const float* w;      // [Ktot][N]
  const float* shift;  // [N] or null
  int N, stride, border, act, nseg, addend_post;
  ffcb_kseg seg[FFCB_MAX_KSEG];
};

struct PixelSrc {  // per (thread, pixel): where the current segment's tap lands
  long long off;   // element offset of channel c0 at the tap, valid only if ok
  bool ok;
};

__global__ void __launch_bounds__(NT) conv_simt_kernel(const __grid_constant__ SimtParams p) {
  __shared__ __align__(16) float As[BK * AS];
  __shared__ __align__(16) float Bs[BK * BN];

  const int tid = threadIdx.x;
  const int HW = p.out.H * p.out.W;
  const long long M = (long long)p.out.B * HW;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // ---- A-load role: two (pixel, channel-quad) slots per thread
  const int a_kq = tid & 3;
  int a_m[2] = {tid >> 2, (tid >> 2) + 64};
  int pb[2], py[2], px[2];
  bool pvalid[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const long long m = m0 + a_m[i];
    pvalid[i] = m < M;
    const long long mm = pvalid[i] ? m : 0;
    pb[i] = (int)(mm / HW);
    const int r = (int)(mm - (long long)pb[i] * HW);
    py[i] = r / p.out.W;
    px[i] = r - py[i] * p.out.W;
  }
  // ---- B-load role
  const int b_k = tid >> 4;          // 0..15
  const int b_n = n0 + (tid & 15) * 4;

  // ---- compute role
  const int tx = tid & 15, ty = tid >> 4;
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  // K iterator over (segment, 16-channel chunk)
  int seg = 0, cin = 0, kglob = 0;  // cin: channel offset inside the segment; kglob: row of W
  PixelSrc src[2];
  auto locate = [&](int s) {
    const ffcb_kseg g = p.seg[s];
    const View& v = p.in[g.src];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      int yi = py[i] * p.stride + g.dy, xi = px[i] * p.stride + g.dx;
      bool ok = pvalid[i];
      if (p.border == FFCB_BORDER_REFLECT) {
        yi = reflect_idx(yi, v.H);
        xi = reflect_idx(xi, v.W);
      } else {
        ok = ok && yi >= 0 && yi < v.H && xi >= 0 && xi < v.W;
      }
      src[i].ok = ok;
      src[i].off = ok ? pix_off(v, pb[i], yi, xi) + g.c0 : 0;
    }
  };

  float4 ra[2], rb;
  auto fetch = [&]() {  // global -> registers for the current (seg, cin)
    const ffcb_kseg g = p.seg[seg];
    const View& v = p.in[g.src];
    const int c = cin + a_kq * 4;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      ra[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (src[i].ok && c < g.nch) ra[i] = load4(v, src[i].off + c);
    }
    rb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (cin + b_k < g.nch && b_n < p.N)
      rb = __ldg(reinterpret_cast<const float4*>(p.w + (long long)(kglob + b_k) * p.N + b_n));
  };
  auto advance = [&]() -> bool {  // move to the next K step; false when exhausted
    const int nch = p.seg[seg].nch;
    const int step = min(BK, nch - cin);
    cin += step;
    kglob += step;
    if (cin >= nch) {
      ++seg;
      cin = 0;
      if (seg >= p.nseg) return false;
      locate(seg);
    }
    return true;
  };

  bool more = p.nseg > 0;
  if (more) {
    locate(0);
    fetch();
  }
  while (more) {
    // registers -> shared
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float* a = As + (a_kq * 4) * AS + a_m[i];
      a[0 * AS] = ra[i].x; a[1 * AS] = ra[i].y; a[2 * AS] = ra[i].z; a[3 * AS] = ra[i].w;
    }
    *reinterpret_cast<float4*>(Bs + b_k * BN + (tid & 15) * 4) = rb;
    __syncthreads();
    more = advance();
    if (more) fetch();  // prefetch next step while computing this one
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(As + k * AS + ty * 8);
      const float4 a1 = *reinterpret_cast<const float4*>(As + k * AS + ty * 8 + 4);
      const float4 b = *reinterpret_cast<const float4*>(Bs + k * BN + tx * 4);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }

  // ---- epilogue
  const int n = n0 + tx * 4;
  if (n >= p.N) return;
  float4 sh = make_float4(0.f, 0.f, 0.f, 0.f);
  if (p.shift != nullptr) sh = __ldg(reinterpret_cast<const float4*>(p.shift + n));
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long long m = m0 + ty * 8 + i;
    if (m >= M) break;
    const int b = (int)(m / HW);
    const int r = (int)(m - (long long)b * HW);
    const int y = r / p.out.W, x = r - y * p.out.W;
    float4 v = make_float4(acc[i][0] + sh.x, acc[i][1] + sh.y, acc[i][2] + sh.z, acc[i][3] + sh.w);
    float4 ad = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.addend.ptr != nullptr) ad = load4(p.addend, pix_off(p.addend, b, y, x) + n);
    if (!p.addend_post) { v.x += ad.x; v.y += ad.y; v.z += ad.z; v.w += ad.w; }
    v.x = apply_act(v.x, p.act); v.y = apply_act(v.y, p.act);
    v.z = apply_act(v.z, p.act); v.w = apply_act(v.w, p.act);
    if (p.addend_post) { v.x += ad.x; v.y += ad.y; v.z += ad.z; v.w += ad.w; }
    store4(p.out, pix_off(p.out, b, y, x) + n, v);
  }
}

}  // namespace

int conv_simt(const ffcb_conv_desc* d, cudaStream_t stream) {
  SimtParams p;
  p.in[0] = make_view(d->in[0]);
  p.in[1] = d->in[1].ptr ? make_view(d->in[1]) : null_view();
  p.out = make_view(d->out);
  p.addend = d->addend.ptr ? make_view(d->addend) : null_view();
  p.w = reinterpret_cast<const float*>(d->weight);
  p.shift = d->shift;
  p.N = d->n_out; p.stride = d->stride; p.border = d->border; p.act = d->act; p.nseg = d->nseg; p.addend_post = d->addend_post;
  for (int i = 0; i < d->nseg; ++i) p.seg[i] = d->seg[i];
  const long long M = (long long)d->out.B * d->out.H * d->out.W;
  if (M == 0 || d->n_out == 0) return FFCB_OK;
  dim3 grid((unsigned)((M + BM - 1) / BM), (unsigned)((d->n_out + BN - 1) / BN));
  conv_simt_kernel<<<grid, NT, 0, stream>>>(p);
  FFCB_LAUNCH_CHECK("conv_simt_kernel");
  return FFCB_OK;
}

}  // namespace ffcb
