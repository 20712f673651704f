// extern "C" surface of libffc_b200.so (see include/ffc_b200.h) + error / launch bookkeeping.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace ffcb {

static thread_local char g_err[512] = "";
static thread_local long long g_launches = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return FFCB_ECUDA;
}

void count_launch(int n) { g_launches += n; }

bool l2_hints_enabled() {
  const char* e = getenv("FFCB_L2_HINTS");
  return e ? atoi(e) != 0 : true;
}

int check_tensor(const ffcb_tensor* t, const char* name, bool allow_cg) {
  FFCB_REQUIRE(t != nullptr, "%s: null tensor descriptor", name);
  FFCB_REQUIRE(t->B >= 0 && t->H >= 0 && t->W >= 0 && t->C >= 0, "%s: negative extent", name);
  if ((long long)t->B * t->H * t->W * t->C == 0) return FFCB_OK;
  FFCB_REQUIRE(t->ptr != nullptr, "%s: null data pointer", name);
  FFCB_REQUIRE(t->fmt == FFCB_F32 || t->fmt == FFCB_BF16X2, "%s: unknown storage format %d", name, t->fmt);
  FFCB_REQUIRE(t->C % 4 == 0, "%s: channel count %d is not a multiple of 4", name, t->C);
  const int esz = t->fmt == FFCB_F32 ? 4 : 2;
  // 4-channel vector access: 16 B (float) / 8 B (bf16 planes)
  const uintptr_t align = t->fmt == FFCB_F32 ? 16 : 8;
  FFCB_REQUIRE(((uintptr_t)t->ptr % align) == 0, "%s: pointer %p not %zu-byte aligned", name, t->ptr, (size_t)align);
  FFCB_REQUIRE(t->sx % 4 == 0 && t->sy % 4 == 0 && t->sb % 4 == 0, "%s: strides must be multiples of 4 elements",
               name);
  FFCB_REQUIRE(t->sx >= t->C || t->window || t->cg, "%s: pixel stride %lld < C=%d (only window views may overlap)",
               name, (long long)t->sx, t->C);
  if (t->fmt == FFCB_BF16X2)
    FFCB_REQUIRE(t->lo_off % 4 == 0 && t->lo_off != 0, "%s: lo_off must be a non-zero multiple of 4", name);
  FFCB_REQUIRE(t->pad >= 0 && t->pad <= 3, "%s: pad must be in [0,3]", name);
  if (t->cg != 0) {
    FFCB_REQUIRE(allow_cg, "%s: channel-group planar views (cg=%d) are not accepted by this entry point", name, t->cg);
    FFCB_REQUIRE((t->cg == 4 || t->cg == 8) && t->C % t->cg == 0, "%s: cg=%d must be 4 or 8 and divide C=%d", name,
                 t->cg, t->C);
    FFCB_REQUIRE(t->sx >= t->cg && t->sg % 4 == 0 && t->sg > 0 && !t->window && t->pad == 0,
                 "%s: bad channel-group strides (sx=%lld, sg=%lld)", name, (long long)t->sx, (long long)t->sg);
    FFCB_REQUIRE(t->tile == 0 || (t->tile == 128 && t->cg == 8 && t->sg % 1024 == 0 && t->sg >= (long long)(t->C / 8) * 1024),
                 "%s: tile-blocked views need tile=128, cg=8 and sg = a whole number of 1024-element group slabs", name);
  } else {
    FFCB_REQUIRE(t->tile == 0, "%s: tile != 0 needs cg == 8", name);
  }
  (void)esz;
  return FFCB_OK;
}

// implemented in the other translation units
int conv_simt(const ffcb_conv_desc* d, cudaStream_t stream);
int conv_tc(const ffcb_conv_desc* d, cudaStream_t stream);
int conv_tc_plan(const ffcb_conv_desc* d, ffcb_conv_plan_info* info);
int stem_conv7(const float*, int, int, int, int, const float*, const float*, int, const ffcb_tensor*, cudaStream_t);
int head_conv7(const ffcb_tensor*, const float*, const float*, int, int, float*, cudaStream_t);
size_t fft2_workspace_bytes(int B, int H, int W, int C);
int rfft2(const ffcb_tensor*, const ffcb_tensor*, void*, size_t, cudaStream_t);
int irfft2(const ffcb_tensor*, const ffcb_tensor*, const ffcb_tensor*, void*, size_t, cudaStream_t);
int nchw_to_nhwc(const float*, int, int, int, int, const ffcb_tensor*, cudaStream_t);
int nhwc_to_nchw(const ffcb_tensor*, float*, cudaStream_t);
int fill_reflect_border(const ffcb_tensor*, cudaStream_t);
int stem_pack(const float*, int, int, int, int, const ffcb_tensor*, cudaStream_t);
int head_gather7(const ffcb_tensor*, const float*, int, int, float*, cudaStream_t);
int head_gather7_rows(const ffcb_tensor*, const float*, int, int, float*, int, int, cudaStream_t);
int stem_pack_u8(const uint8_t*, const uint8_t*, int, int, int, const ffcb_tensor*, cudaStream_t);
int head_gather7_blend_u8(const ffcb_tensor*, const float*, int, const uint8_t*, const uint8_t*, int, int, uint8_t*,
                          cudaStream_t);
int relu_bwd(const ffcb_tensor*, const ffcb_tensor*, const ffcb_tensor*, cudaStream_t);
int relu_mask_pack(const ffcb_tensor*, uint32_t*, cudaStream_t);
int relu_bwd_bits(const ffcb_tensor*, const uint32_t*, const ffcb_tensor*, cudaStream_t);
int relu_mask_pack_rows(const ffcb_tensor*, uint32_t*, int, int, cudaStream_t);
int relu_bwd_bits_rows(const ffcb_tensor*, const uint32_t*, int, int, const ffcb_tensor*, cudaStream_t);
int fold_reflect_border(const ffcb_tensor*, const ffcb_tensor*, int, const ffcb_tensor*, int, const ffcb_tensor*,
                        cudaStream_t);
int add(const ffcb_tensor*, const ffcb_tensor*, const ffcb_tensor*, cudaStream_t);
int head_bwd7(const float*, const float*, int, int, int, int, const float*, int, const ffcb_tensor*, const ffcb_tensor*,
              cudaStream_t);
int head_bwd7_bits(const float*, const float*, int, int, int, int, const float*, int, const uint32_t*, int,
                   const ffcb_tensor*, cudaStream_t);
int stem_bwd7(const ffcb_tensor*, const float*, int, float*, cudaStream_t);
int refine_l1_grad(const float*, const float*, const float*, int, int, int, int, int, int, const float*, const float*,
                   const float*, const float*, float*, float*, float*, cudaStream_t);

static int check_conv(const ffcb_conv_desc* d) {
  FFCB_REQUIRE(d != nullptr, "conv: null descriptor");
  int rc;
  const bool tc = d->math == FFCB_MATH_BF16X3;     // only the tensor-core arm understands channel-group planar views
  if ((rc = check_tensor(&d->in[0], "conv.in[0]", tc))) return rc;
  if ((rc = check_tensor(&d->out, "conv.out", tc))) return rc;
  FFCB_REQUIRE(d->weight != nullptr, "conv: null weight");
  FFCB_REQUIRE(d->n_out > 0 && d->n_out % 4 == 0, "conv: n_out=%d must be a positive multiple of 4", d->n_out);
  FFCB_REQUIRE(d->out.C == d->n_out, "conv: out view has C=%d, n_out=%d", d->out.C, d->n_out);
  FFCB_REQUIRE(d->stride == 1 || d->stride == 2, "conv: stride %d unsupported", d->stride);
  FFCB_REQUIRE(d->nseg >= 1 && d->nseg <= FFCB_MAX_KSEG, "conv: nseg=%d outside [1,%d]", d->nseg, FFCB_MAX_KSEG);
  FFCB_REQUIRE(d->border == FFCB_BORDER_ZERO || d->border == FFCB_BORDER_REFLECT, "conv: bad border mode");
  FFCB_REQUIRE(d->act >= FFCB_ACT_NONE && d->act <= FFCB_ACT_TANH, "conv: bad activation");
  bool uses1 = false;
  for (int i = 0; i < d->nseg; ++i) {
    const ffcb_kseg& s = d->seg[i];
    FFCB_REQUIRE(s.src == 0 || s.src == 1, "conv: seg %d has src=%d", i, s.src);
    uses1 |= s.src == 1;
    const ffcb_tensor& t = d->in[s.src];
    FFCB_REQUIRE(s.nch > 0 && s.nch % 4 == 0 && s.c0 % 4 == 0 && s.c0 >= 0 && s.c0 + s.nch <= t.C,
                 "conv: seg %d channel range [%d,%d) invalid for C=%d", i, s.c0, s.c0 + s.nch, t.C);
    FFCB_REQUIRE(t.B == d->out.B, "conv: batch mismatch between in[%d] and out", s.src);
    if (d->border == FFCB_BORDER_REFLECT) {
      // reflect needs every sampled coordinate within one reflection of the interior
      const int ymin = s.dy, ymax = (d->out.H - 1) * d->stride + s.dy;
      const int xmin = s.dx, xmax = (d->out.W - 1) * d->stride + s.dx;
      FFCB_REQUIRE(ymin > -t.H && ymax < 2 * t.H - 1 && xmin > -t.W && xmax < 2 * t.W - 1 && t.H >= 1 && t.W >= 1,
                   "conv: seg %d tap (%d,%d) reaches beyond one reflection of a %dx%d input", i, s.dy, s.dx, t.H, t.W);
    }
  }
  if (uses1 && (rc = check_tensor(&d->in[1], "conv.in[1]", tc))) return rc;
  if (d->addend.ptr != nullptr) {
    if ((rc = check_tensor(&d->addend, "conv.addend"))) return rc;
    FFCB_REQUIRE(d->addend.B == d->out.B && d->addend.H == d->out.H && d->addend.W == d->out.W &&
                     d->addend.C == d->n_out, "conv: addend shape differs from out");
  }
  return FFCB_OK;
}

}  // namespace ffcb

using namespace ffcb;

extern "C" {

int ffcb_version(void) { return FFCB_VERSION; }
const char* ffcb_last_error(void) { return g_err; }

int ffcb_check_device(int device) {
  cudaDeviceProp prop;
  FFCB_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("device %d is sm_%d%d; libffc_b200 is built for sm_90a only", device, prop.major, prop.minor);
    return FFCB_EARCH;
  }
  return FFCB_OK;
}

void ffcb_shutdown(void) {}

int ffcb_conv(const ffcb_conv_desc* d, ffcb_stream_t stream) {
  int rc = check_conv(d);
  if (rc) return rc;
  if (d->math == FFCB_MATH_FP32) return conv_simt(d, (cudaStream_t)stream);
  if (d->math == FFCB_MATH_BF16X3) return conv_tc(d, (cudaStream_t)stream);
  set_error("conv: unknown math mode %d", d->math);
  return FFCB_EINVAL;
}

int ffcb_conv_plan(const ffcb_conv_desc* d, ffcb_conv_plan_info* info) {
  int rc = check_conv(d);
  if (rc) return rc;
  FFCB_REQUIRE(info != nullptr, "conv_plan: null result");
  FFCB_REQUIRE(d->math == FFCB_MATH_BF16X3, "conv_plan: only the tensor-core arm (FFCB_MATH_BF16X3) has a plan");
  return conv_tc_plan(d, info);
}

int ffcb_stem_conv7(const float* x, int B, int Cin, int H, int W, const float* w, const float* shift, int N,
                    const ffcb_tensor* out, ffcb_stream_t stream) {
  return stem_conv7(x, B, Cin, H, W, w, shift, N, out, (cudaStream_t)stream);
}

int ffcb_stem_pack(const float* x, int B, int Cin, int H, int W, const ffcb_tensor* packed, ffcb_stream_t stream) {
  return stem_pack(x, B, Cin, H, W, packed, (cudaStream_t)stream);
}

int ffcb_stem_pack_u8(const uint8_t* image_hwc, const uint8_t* mask_hw, int B, int H0, int W0,
                      const ffcb_tensor* packed, ffcb_stream_t stream) {
  return stem_pack_u8(image_hwc, mask_hw, B, H0, W0, packed, (cudaStream_t)stream);
}

int ffcb_head_gather7_blend_u8(const ffcb_tensor* q, const float* bias, int act, const uint8_t* image_hwc,
                               const uint8_t* mask_hw, int H0, int W0, uint8_t* out_hwc, ffcb_stream_t stream) {
  return head_gather7_blend_u8(q, bias, act, image_hwc, mask_hw, H0, W0, out_hwc, (cudaStream_t)stream);
}

int ffcb_head_gather7(const ffcb_tensor* q, const float* bias, int N, int act, float* y, ffcb_stream_t stream) {
  return head_gather7(q, bias, N, act, y, (cudaStream_t)stream);
}

int ffcb_head_conv7(const ffcb_tensor* in, const float* w, const float* bias, int N, int act, float* y,
                    ffcb_stream_t stream) {
  return head_conv7(in, w, bias, N, act, y, (cudaStream_t)stream);
}

size_t ffcb_fft2_workspace_bytes(int B, int H, int W, int C) { return fft2_workspace_bytes(B, H, W, C); }

int ffcb_rfft2(const ffcb_tensor* in, const ffcb_tensor* spec, void* ws, size_t ws_bytes, ffcb_stream_t stream) {
  return rfft2(in, spec, ws, ws_bytes, (cudaStream_t)stream);
}

int ffcb_irfft2(const ffcb_tensor* spec, const ffcb_tensor* residual, const ffcb_tensor* out, void* ws,
                size_t ws_bytes, ffcb_stream_t stream) {
  return irfft2(spec, residual, out, ws, ws_bytes, (cudaStream_t)stream);
}

int ffcb_nchw_to_nhwc(const float* x, int B, int C, int H, int W, const ffcb_tensor* out, ffcb_stream_t stream) {
  return nchw_to_nhwc(x, B, C, H, W, out, (cudaStream_t)stream);
}

int ffcb_nhwc_to_nchw(const ffcb_tensor* in, float* y, ffcb_stream_t stream) {
  return nhwc_to_nchw(in, y, (cudaStream_t)stream);
}

int ffcb_fill_reflect_border(const ffcb_tensor* t, ffcb_stream_t stream) {
  return fill_reflect_border(t, (cudaStream_t)stream);
}

int ffcb_relu_bwd(const ffcb_tensor* dy, const ffcb_tensor* y, const ffcb_tensor* out, ffcb_stream_t stream) {
  return relu_bwd(dy, y, out, (cudaStream_t)stream);
}

int ffcb_relu_mask_pack(const ffcb_tensor* y, uint32_t* bits, ffcb_stream_t stream) {
  return relu_mask_pack(y, bits, (cudaStream_t)stream);
}

int ffcb_relu_bwd_bits(const ffcb_tensor* dy, const uint32_t* bits, const ffcb_tensor* out, ffcb_stream_t stream) {
  return relu_bwd_bits(dy, bits, out, (cudaStream_t)stream);
}

int ffcb_fold_reflect_border(const ffcb_tensor* gpad, const ffcb_tensor* add0, int add0_c0, const ffcb_tensor* add1,
                             int add1_c0, const ffcb_tensor* out, ffcb_stream_t stream) {
  return fold_reflect_border(gpad, add0, add0_c0, add1, add1_c0, out, (cudaStream_t)stream);
}

int ffcb_add(const ffcb_tensor* a, const ffcb_tensor* b, const ffcb_tensor* out, ffcb_stream_t stream) {
  return add(a, b, out, (cudaStream_t)stream);
}

int ffcb_head_bwd7(const float* y_nchw, const float* dy_nchw, int B, int N, int H, int W, const float* w, int act,
                   const ffcb_tensor* mask, const ffcb_tensor* out, ffcb_stream_t stream) {
  return head_bwd7(y_nchw, dy_nchw, B, N, H, W, w, act, mask, out, (cudaStream_t)stream);
}

int ffcb_stem_bwd7(const ffcb_tensor* g, const float* w, int Cin, float* dx_nchw, ffcb_stream_t stream) {
  return stem_bwd7(g, w, Cin, dx_nchw, (cudaStream_t)stream);
}

int ffcb_head_bwd7_bits(const float* y_nchw, const float* dy_nchw, int B, int N, int H, int W, const float* w,
                        int act, const uint32_t* mask_bits, int row0, const ffcb_tensor* out, ffcb_stream_t stream) {
  return head_bwd7_bits(y_nchw, dy_nchw, B, N, H, W, w, act, mask_bits, row0, out, (cudaStream_t)stream);
}

int ffcb_relu_mask_pack_rows(const ffcb_tensor* y, uint32_t* bits, int H, int row0, ffcb_stream_t stream) {
  return relu_mask_pack_rows(y, bits, H, row0, (cudaStream_t)stream);
}

int ffcb_relu_bwd_bits_rows(const ffcb_tensor* dy, const uint32_t* bits, int H, int row0, const ffcb_tensor* out,
                            ffcb_stream_t stream) {
  return relu_bwd_bits_rows(dy, bits, H, row0, out, (cudaStream_t)stream);
}

int ffcb_head_gather7_rows(const ffcb_tensor* q, const float* bias, int N, int act, float* y_nchw, int H, int row0,
                           ffcb_stream_t stream) {
  return head_gather7_rows(q, bias, N, act, y_nchw, H, row0, (cudaStream_t)stream);
}

int ffcb_refine_l1_grad(const float* pred, const float* image, const float* mask, int B, int C, int Hp, int Wp, int H0,
                        int W0, const float* ref, const float* md, const float* inv_n, const float* taps, float* work,
                        float* grad, float* loss, ffcb_stream_t stream) {
  return refine_l1_grad(pred, image, mask, B, C, Hp, Wp, H0, W0, ref, md, inv_n, taps, work, grad, loss,
                        (cudaStream_t)stream);
}

long long ffcb_launch_count(void) { return g_launches; }
void ffcb_reset_launch_count(void) { g_launches = 0; }

}  // extern "C"
