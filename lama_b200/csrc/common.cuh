// Shared device/host helpers for libffc_b200 (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ffc_b200.h"

namespace ffcb {

// ---------------------------------------------------------------- error plumbing (api.cu)
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);
void count_launch(int n = 1);
bool l2_hints_enabled();     // FFCB_L2_HINTS (default on)

#define FFCB_REQUIRE(cond, ...)                 \
  do {                                          \
    if (!(cond)) {                              \
      ::ffcb::set_error(__VA_ARGS__);           \
      return FFCB_EINVAL;                       \
    }                                           \
  } while (0)

#define FFCB_CUDA(call)                                           \
  do {                                                            \
    cudaError_t _e = (call);                                      \
    if (_e != cudaSuccess) return ::ffcb::cuda_fail(_e, #call);   \
  } while (0)

#define FFCB_LAUNCH_CHECK(name)                                   \
  do {                                                            \
    ::ffcb::count_launch();                                       \
    cudaError_t _e = cudaGetLastError();                          \
    if (_e != cudaSuccess) return ::ffcb::cuda_fail(_e, name);    \
  } while (0)

// ---------------------------------------------------------------- device view of ffcb_tensor
struct View {
  char* ptr;
  long long sb, sy, sx, lo_off, sg;
  int B, H, W, C;
  int fmt, pad, reflect_border, cg, tile;
};

inline View make_view(const ffcb_tensor& t) {
  View v;
  v.ptr = (char*)t.ptr;
  v.sb = t.sb; v.sy = t.sy; v.sx = t.sx; v.lo_off = t.lo_off;
  v.B = t.B; v.H = t.H; v.W = t.W; v.C = t.C;
  v.fmt = t.fmt; v.pad = t.pad; v.reflect_border = t.reflect_border;
  v.cg = t.cg; v.sg = t.cg ? t.sg : 0;
  v.tile = t.cg ? t.tile : 0;
  return v;
}

inline View null_view() {
  View v{};
  v.ptr = nullptr;
  return v;
}

// Validation shared by entry points: 4-channel vector access everywhere.  Channel-group planar views (cg != 0) are
// only accepted where `allow_cg` says so (the FourierUnit chain: ffcb_conv's tensor-core arm and the plane FFT kernels).
int check_tensor(const ffcb_tensor* t, const char* name, bool allow_cg = false);

__host__ __device__ __forceinline__ long long pix_off(const View& v, int b, int y, int x) {
  return (long long)b * v.sb + (long long)y * v.sy + (long long)x * v.sx;
}

// element offset of channel c inside a pixel: c for channels-last views, (c / cg) * sg + c % cg for channel-group planar
__host__ __device__ __forceinline__ long long chan_off(const View& v, int c) {
  return v.cg ? (long long)(c / v.cg) * v.sg + (c % v.cg) : (long long)c;
}

// element offset of (b, y, x, c) for every layout: channels-last, channel-group planar, tile-blocked
__host__ __device__ __forceinline__ long long elem_off(const View& v, int b, int y, int x, int c) {
  if (v.tile) {
    const long long m = ((long long)b * v.H + y) * v.W + x;
    return (m >> 7) * v.sg + (long long)(c >> 3) * 1024 + (m & 127) * 8 + (c & 7);
  }
  return pix_off(v, b, y, x) + chan_off(v, c);
}

// reflect without edge repeat: -1 -> 1, n -> n-2 (valid for |overshoot| < n)
__host__ __device__ __forceinline__ int reflect_idx(int i, int n) {
  i = i < 0 ? -i : i;
  return i >= n ? 2 * n - 2 - i : i;
}

#ifdef __CUDACC__
// split-bf16 encode/decode: v ~= hi + lo, |v - (hi+lo)| <= 2^-17 |v|
__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// hi / lo bf16 pairs of two values (round to nearest even, lo = bf16(v - hi)): the packed conversion (F2FP.PACK_AB)
// instead of two scalar F2F — same bits, but F2F issues at 1/8 of the packed instruction's rate
__device__ __forceinline__ void split_pair(float a, float b, unsigned& hi, unsigned& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const float2 hf = __bfloat1622float2(h);
  const __nv_bfloat162 l = __floats2bfloat162_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<const unsigned*>(&h);
  lo = *reinterpret_cast<const unsigned*>(&l);
}

// element-wise a * b + c of a float2 with one rounding per lane (the sm_90 form of __ffma2_rn: two FFMA)
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

__device__ __forceinline__ float bf16_bits_to_float(unsigned short u) {
  return __uint_as_float(((unsigned)u) << 16);
}

// 4 consecutive channels at element offset `off` (multiple of 4) of a view
__device__ __forceinline__ float4 load4(const View& v, long long off) {
  if (v.fmt == FFCB_F32) {
    return __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(v.ptr) + off));
  }
  const unsigned short* p = reinterpret_cast<const unsigned short*>(v.ptr);
  uint2 h = __ldg(reinterpret_cast<const uint2*>(p + off));
  uint2 l = __ldg(reinterpret_cast<const uint2*>(p + off + v.lo_off));
  float4 r;
  r.x = __uint_as_float(h.x << 16) + __uint_as_float(l.x << 16);
  r.y = __uint_as_float(h.x & 0xffff0000u) + __uint_as_float(l.x & 0xffff0000u);
  r.z = __uint_as_float(h.y << 16) + __uint_as_float(l.y << 16);
  r.w = __uint_as_float(h.y & 0xffff0000u) + __uint_as_float(l.y & 0xffff0000u);
  return r;
}

__device__ __forceinline__ unsigned pack_bf16(__nv_bfloat16 a, __nv_bfloat16 b) {
  return (unsigned)__bfloat16_as_ushort(a) | ((unsigned)__bfloat16_as_ushort(b) << 16);
}

__device__ __forceinline__ void store4(const View& v, long long off, float4 r) {
  if (v.fmt == FFCB_F32) {
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(v.ptr) + off) = r;
    return;
  }
  unsigned h0, l0, h1, l1;
  split_pair(r.x, r.y, h0, l0);
  split_pair(r.z, r.w, h1, l1);
  unsigned short* p = reinterpret_cast<unsigned short*>(v.ptr);
  *reinterpret_cast<uint2*>(p + off) = make_uint2(h0, h1);
  *reinterpret_cast<uint2*>(p + off + v.lo_off) = make_uint2(l0, l1);
}

// scalar access (tails, odd layouts)
__device__ __forceinline__ float load1(const View& v, long long off) {
  if (v.fmt == FFCB_F32) return __ldg(reinterpret_cast<const float*>(v.ptr) + off);
  const unsigned short* p = reinterpret_cast<const unsigned short*>(v.ptr);
  return bf16_bits_to_float(__ldg(p + off)) + bf16_bits_to_float(__ldg(p + off + v.lo_off));
}

__device__ __forceinline__ void store1(const View& v, long long off, float r) {
  if (v.fmt == FFCB_F32) { reinterpret_cast<float*>(v.ptr)[off] = r; return; }
  __nv_bfloat16 h, l;
  split_bf16(r, h, l);
  __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(v.ptr);
  p[off] = h;
  p[off + v.lo_off] = l;
}

__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case FFCB_ACT_RELU: return fmaxf(v, 0.f);
    case FFCB_ACT_SIGMOID: return __fdividef(1.f, 1.f + __expf(-v));   // explicit fast intrinsics: ~2 ulp
    case FFCB_ACT_TANH: return tanhf(v);                              // precise (no --use_fast_math)
    default: return v;
  }
}

// ---- L2 residency hints (createpolicy + .L2::cache_hint accesses).  The FourierUnit chain hands two spectra from
// kernel to kernel (rfft2 -> spectral GEMM -> irfft2); they should stay in the 50 MB L2 while the planes that are
// only streamed through (t in, u out) should not push them out: producers store intermediates with evict_last,
// consumers read them (and everything read once) with evict_first.  FFCB_L2_HINTS=0 makes every policy "normal".
__device__ __forceinline__ uint64_t l2_policy(int kind) {     // 0 normal, 1 evict_first, 2 evict_last
  uint64_t p;
  if (kind == 1) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  else if (kind == 2) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  else asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void st_hint_b32(void* p, unsigned v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.b32 [%0], %1, %2;" ::"l"(p), "r"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_hint_v2(void* p, uint2 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v2.b32 [%0], {%1, %2}, %3;" ::"l"(p), "r"(v.x), "r"(v.y), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_hint_u4(void* p, uint4 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_hint_f4(void* p, float4 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w), "l"(pol) : "memory");
}
__device__ __forceinline__ float2 ld_hint_f2(const void* p, uint64_t pol) {
  float2 v;
  asm volatile("ld.global.nc.L2::cache_hint.v2.f32 {%0, %1}, [%2], %3;" : "=f"(v.x), "=f"(v.y) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ float4 ld_hint_f4(const void* p, uint64_t pol) {
  float4 v;
  asm volatile("ld.global.nc.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol));
  return v;
}

// Mirror targets of an interior pixel in the reflected border ring of a pad==1 view (H, W >= 4):
// row 1 also lands on row -1, row H-2 on row H, likewise columns; corners follow from both.
// Returns false for the ~94% of pixels that have no mirror image.
__device__ __forceinline__ bool ring_mirrors(const View& v, int y, int x, int& my, int& mx) {
  my = (y == 1) ? -1 : ((y == v.H - 2) ? v.H : -2);   // -2: none
  mx = (x == 1) ? -1 : ((x == v.W - 2) ? v.W : -2);
  return (my != -2) | (mx != -2);
}

static __device__ __noinline__ float slow_act(float v, int act) {
  return act == FFCB_ACT_SIGMOID ? __fdividef(1.f, 1.f + __expf(-v)) : tanhf(v);
}
#endif  // __CUDACC__

}  // namespace ffcb
