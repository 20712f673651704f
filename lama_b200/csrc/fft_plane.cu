// Fused 2-D real FFT pair for 64x64 planes (the bottleneck of 512x512 images): one CTA transforms the
// whole plane of 8 channels, so the half-spectrum intermediate lives in shared memory instead of a
// global workspace (halves the HBM traffic of ffcb_rfft2 / ffcb_irfft2 and removes two launches).
//
// Every 64-point transform is held in the registers of ONE thread (fft64_regs: unrolled 8x8 Cooley-Tukey
// with compile-time twiddles) — no shuffles, no shared-memory butterflies, one barrier per plane:
//   forward : 256 threads = 8 channels x 32 row pairs (two-for-one real rows)  -> S[y][kx][c] -> barrier ->
//             8 channels x (31 complex columns + 1 packed DC/Nyquist pair) -> spectrum (Re/Im interleaved, scaled)
//   inverse : columns first (all 33, complex), barrier, then C2R rows (+ residual).
// smem: S[64][P] float2 with row pitch P = 33*8 + 4 (the +4 spreads the four row-pair groups of a warp
// over both halves of the banks).  Lanes: 8 consecutive channels (32 B of a pixel) x 4 rows/columns.
#include <stdint.h>
#include <stdlib.h>

#include "common.cuh"
#include "fft_core.cuh"

namespace ffcb {
int inv_plane_variant();   // FFCB_FFT_INV_PLANE (defined with the dispatchers at the end of this file)
namespace {

using namespace fftc;
constexpr int PN = 64, PWF = 33;
// Channels per CTA (PCH): 8 = one CTA per SM (137 KB of shared memory), lanes cover one full 32-byte sector of a
// pixel; 4 = 69 KB, two CTAs per SM so that one CTA's load / store phases overlap the other's transforms
// (FFCB_FFT_PLANE_CH=4, an experiment of round 1 — half-sector accesses, the sibling CTA picks up the other half
// from L2).  The row pitch keeps the row-phase stores of a half-warp on 32 distinct banks: 4*P mod 32 = 128 / PCH.
template <int PCH> struct PlaneCfg {
  static constexpr int pitch = PWF * PCH + (PCH == 8 ? 4 : 2);
  static constexpr int row_threads = 32 * PCH;                       // PCH channels x 32 row pairs
  static constexpr int col_threads = (PWF * PCH + 31) / 32 * 32;     // PCH channels x 33 columns, whole warps
  static constexpr size_t smem = sizeof(float2) * PN * pitch;
  static constexpr int ctas_per_sm = PCH == 8 ? 1 : 2;
};

// Forward: rows by the first 32*PCH threads, the 33 x PCH column tasks by the first 33*PCH (for PCH = 8 chosen
// over the packed 256-thread variant: fewer registers per thread, and one more warp to hide latency).
template <int PCH, int OCC>
__global__ void __launch_bounds__(PlaneCfg<PCH>::col_threads, OCC)
rfft2_plane64_kernel(View in, View spec, float scale) {
  extern __shared__ float2 S[];
  constexpr int PPITCH = PlaneCfg<PCH>::pitch;
  const int tid = threadIdx.x, c = tid % PCH, g = tid / PCH;
  const int ch = blockIdx.x * PCH + c, b = blockIdx.y;
  if (tid < PlaneCfg<PCH>::row_threads) {   // g = row pair
    const long long r0 = pix_off(in, b, 2 * g, 0) + ch, r1 = r0 + in.sy;
    plane64_rows_fwd(
        [&](int n) { return make_float2(load1(in, r0 + n * in.sx), load1(in, r1 + n * in.sx)); },
        [&](int k, float2 a, float2 bb) {
          S[(2 * g) * PPITCH + k * PCH + c] = a;
          S[(2 * g + 1) * PPITCH + k * PCH + c] = bb;
        });
  }
  __syncthreads();
  if (tid < PWF * PCH) {   // g = kx
    const long long o0 = pix_off(spec, b, 0, g) + 2 * ch;
    plane64_col<false>(
        [&](int y) { return S[y * PPITCH + g * PCH + c]; },
        [&](int ky, float2 z) {
          const long long o = o0 + ky * spec.sy;
          z.x *= scale; z.y *= scale;
          if (spec.fmt == FFCB_F32) {
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(spec.ptr) + o) = z;
          } else {
            __nv_bfloat16 h0, l0, h1, l1;
            split_bf16(z.x, h0, l0);
            split_bf16(z.y, h1, l1);
            unsigned short* p = reinterpret_cast<unsigned short*>(spec.ptr);
            *reinterpret_cast<unsigned*>(p + o) = pack_bf16(h0, h1);
            *reinterpret_cast<unsigned*>(p + o + spec.lo_off) = pack_bf16(l0, l1);
          }
        });
  }
}

// Forward, second revision (default for float32 inputs).  Same algorithm and thread mapping; the differences are in
// what surrounds the arithmetic (a third of the first revision's instruction body is 64-bit address arithmetic and
// every access carries both format branches):
//   * the spectrum format is a template parameter (one store path compiled in, no branch per store),
//   * the CTA's base pointers are uniform (blockIdx-only) and every thread addresses with 32-bit offsets.
template <int PCH, bool SPLIT>
__global__ void __launch_bounds__(PlaneCfg<PCH>::col_threads, 1)
rfft2_plane64_v2_kernel(const float* __restrict__ in_ptr, long long in_sb, unsigned in_sy, unsigned in_sx,
                        void* __restrict__ spec_ptr, long long spec_sb, unsigned spec_sy, unsigned spec_sx,
                        long long spec_lo, float scale) {
  extern __shared__ float2 S[];
  constexpr int PPITCH = PlaneCfg<PCH>::pitch;
  const int tid = threadIdx.x, c = tid % PCH, g = tid / PCH;
  if (tid < PlaneCfg<PCH>::row_threads) {   // g = row pair
    const float* __restrict__ inb = in_ptr + (long long)blockIdx.y * in_sb + blockIdx.x * PCH;
    const unsigned o0 = 2u * g * in_sy + c;
    plane64_rows_fwd(
        [&](int n) {
          const unsigned o = o0 + (unsigned)n * in_sx;
          return make_float2(__ldg(inb + o), __ldg(inb + o + in_sy));
        },
        [&](int k, float2 a, float2 bb) {
          S[(2 * g) * PPITCH + k * PCH + c] = a;
          S[(2 * g + 1) * PPITCH + k * PCH + c] = bb;
        });
  }
  __syncthreads();
  if (tid < PWF * PCH) {   // g = kx
    const unsigned o0 = (unsigned)g * spec_sx + 2u * c;
    const long long cta = (long long)blockIdx.y * spec_sb + 2 * blockIdx.x * PCH;
    if constexpr (SPLIT) {
      unsigned short* __restrict__ hi = reinterpret_cast<unsigned short*>(spec_ptr) + cta;
      unsigned short* __restrict__ lo = hi + spec_lo;
      plane64_col<false>(
          [&](int y) { return S[y * PPITCH + g * PCH + c]; },
          [&](int ky, float2 z) {
            const unsigned o = o0 + (unsigned)ky * spec_sy;
            __nv_bfloat16 h0, l0, h1, l1;
            split_bf16(z.x * scale, h0, l0);
            split_bf16(z.y * scale, h1, l1);
            *reinterpret_cast<unsigned*>(hi + o) = pack_bf16(h0, h1);
            *reinterpret_cast<unsigned*>(lo + o) = pack_bf16(l0, l1);
          });
    } else {
      float* __restrict__ sp = reinterpret_cast<float*>(spec_ptr) + cta;
      plane64_col<false>(
          [&](int y) { return S[y * PPITCH + g * PCH + c]; },
          [&](int ky, float2 z) {
            const unsigned o = o0 + (unsigned)ky * spec_sy;
            *reinterpret_cast<float2*>(sp + o) = make_float2(z.x * scale, z.y * scale);
          });
    }
  }
}

template <int PCH>
__global__ void __launch_bounds__(PlaneCfg<PCH>::row_threads, PlaneCfg<PCH>::ctas_per_sm)
irfft2_plane64_kernel(View spec, View res, View out, float scale) {
  extern __shared__ float2 S[];
  constexpr int PPITCH = PlaneCfg<PCH>::pitch;
  const int tid = threadIdx.x, c = tid % PCH, g = tid / PCH;
  const int ch = blockIdx.x * PCH + c, b = blockIdx.y;
  auto get = [&](long long o) {
    if (spec.fmt == FFCB_F32) return __ldg(reinterpret_cast<const float2*>(reinterpret_cast<const float*>(spec.ptr) + o));
    return make_float2(load1(spec, o), load1(spec, o + 1));
  };
  const long long o0 = pix_off(spec, b, 0, 0) + 2 * ch;
  const bool packed = g == 0;
  plane64_col_inv_any(
      packed, [&](int ky) { return get(o0 + ky * spec.sy + g * spec.sx); },
      [&](int ky) { return get(o0 + ky * spec.sy + 32 * spec.sx); },
      [&](int y, float2 z) { S[y * PPITCH + g * PCH + c] = z; },
      [&](int y, float2 z) { S[y * PPITCH + 32 * PCH + c] = z; });
  __syncthreads();
  {   // g = row pair: C2R along W
    const long long r0 = pix_off(out, b, 2 * g, 0) + ch, r1 = r0 + out.sy;
    const bool has_res = res.ptr != nullptr;
    const long long q0 = has_res ? pix_off(res, b, 2 * g, 0) + ch : 0, q1 = q0 + res.sy;
    plane64_rows_inv(
        [&](int k, float2& x1, float2& x2) {
          x1 = S[(2 * g) * PPITCH + k * PCH + c];
          x2 = S[(2 * g + 1) * PPITCH + k * PCH + c];
        },
        [&](int n0, const float2* zb) {
          float ra[16], rb[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            ra[j] = has_res ? load1(res, q0 + (n0 + j) * res.sx) : 0.f;
            rb[j] = has_res ? load1(res, q1 + (n0 + j) * res.sx) : 0.f;
          }
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            store1(out, r0 + (n0 + j) * out.sx, fmaf(zb[j].x, scale, ra[j]));
            store1(out, r1 + (n0 + j) * out.sx, fmaf(zb[j].y, scale, rb[j]));
          }
        });
  }
}

// Inverse, second revision (FFCB_FFT_INV_PLANE=3): the one-task-per-column variant below with
//   * formats as template parameters (float32 spectrum / residual in; float32 or split-bf16 out),
//   * uniform CTA base pointers + 32-bit in-plane offsets,
//   * a channels-last epilogue: row results are staged in place of the row's half spectrum and leave the SM as
//     whole pixels (2 x LDS.128 + 2 x LDG.128 residual + 2 x STG.128 per pixel) instead of 64 x (LDG.32 +
//     2 x STG.16) per thread — a quarter of the memory instructions and none of their 64-bit address arithmetic.
struct PlaneInvArgs {
  const float* spec; long long spec_sb; unsigned spec_sy, spec_sx;
  const float* res;  long long res_sb;  unsigned res_sy, res_sx;
  void* out;         long long out_sb;  unsigned out_sy, out_sx; long long out_lo;
  float scale;
};

template <bool HAS_RES, bool OUT_SPLIT>
__global__ void __launch_bounds__(PlaneCfg<8>::col_threads, 1) irfft2_plane64_v2_kernel(PlaneInvArgs a) {
  extern __shared__ float2 S[];
  constexpr int PPITCH = PlaneCfg<8>::pitch;
  static_assert(PPITCH == kP64Pitch, "staging indices assume the 8-channel pitch");
  const int tid = threadIdx.x, c = tid & 7, g = tid >> 3;
  if (tid < PWF * 8) {   // g = kx: inverse transform along H of one (column, channel)
    const float* __restrict__ sp = a.spec + (long long)blockIdx.y * a.spec_sb + 2 * blockIdx.x * 8;
    const unsigned o0 = (unsigned)g * a.spec_sx + 2u * c;
    plane64_col<true>(
        [&](int ky) { return __ldg(reinterpret_cast<const float2*>(sp + (o0 + (unsigned)ky * a.spec_sy))); },
        [&](int y, float2 z) { S[y * PPITCH + g * 8 + c] = z; });
  }
  __syncthreads();
  if (tid < 256) {       // g = row pair: C2R along W, results staged channels-last in place of rows 2g, 2g+1
    float* R = reinterpret_cast<float*>(S);
    plane64_rows_inv(
        [&](int k, float2& x1, float2& x2) {
          x1 = S[(2 * g) * PPITCH + k * 8 + c];
          x2 = S[(2 * g + 1) * PPITCH + k * 8 + c];
        },
        [&](int n0, const float2* zb) {
          // rows 2g, 2g+1 are read and written by the eight threads of group g only (one warp): once every lane
          // holds its inputs in registers the rows may be overwritten
          if (n0 == 0) __syncwarp();
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            R[p64_stage_index(2 * g, n0 + j, c)] = zb[j].x;
            R[p64_stage_index(2 * g + 1, n0 + j, c)] = zb[j].y;
          }
        });
    __syncwarp();
    const int warp = tid >> 5, lane = tid & 31;
    const long long res_cta = (long long)blockIdx.y * a.res_sb + blockIdx.x * 8;
    const long long out_cta = (long long)blockIdx.y * a.out_sb + blockIdx.x * 8;
#pragma unroll 4
    for (int i = 0; i < 16; ++i) {
      int row, x;
      p64_store_slot(warp, lane, i, row, x);
      const float4* r4 = reinterpret_cast<const float4*>(R + p64_stage_index(row, x, 0));
      float4 v0 = r4[0], v1 = r4[1];
      float4 q0 = make_float4(0.f, 0.f, 0.f, 0.f), q1 = q0;
      if constexpr (HAS_RES) {
        const float4* q = reinterpret_cast<const float4*>(a.res + res_cta + ((unsigned)row * a.res_sy + (unsigned)x * a.res_sx));
        q0 = __ldg(q);
        q1 = __ldg(q + 1);
      }
      v0 = make_float4(fmaf(v0.x, a.scale, q0.x), fmaf(v0.y, a.scale, q0.y), fmaf(v0.z, a.scale, q0.z), fmaf(v0.w, a.scale, q0.w));
      v1 = make_float4(fmaf(v1.x, a.scale, q1.x), fmaf(v1.y, a.scale, q1.y), fmaf(v1.z, a.scale, q1.z), fmaf(v1.w, a.scale, q1.w));
      const unsigned o = (unsigned)row * a.out_sy + (unsigned)x * a.out_sx;
      if constexpr (OUT_SPLIT) {
        __nv_bfloat16 h[8], l[8];
        split_bf16(v0.x, h[0], l[0]); split_bf16(v0.y, h[1], l[1]); split_bf16(v0.z, h[2], l[2]); split_bf16(v0.w, h[3], l[3]);
        split_bf16(v1.x, h[4], l[4]); split_bf16(v1.y, h[5], l[5]); split_bf16(v1.z, h[6], l[6]); split_bf16(v1.w, h[7], l[7]);
        unsigned short* hi = reinterpret_cast<unsigned short*>(a.out) + out_cta;
        *reinterpret_cast<uint4*>(hi + o) =
            make_uint4(pack_bf16(h[0], h[1]), pack_bf16(h[2], h[3]), pack_bf16(h[4], h[5]), pack_bf16(h[6], h[7]));
        *reinterpret_cast<uint4*>(hi + a.out_lo + o) =
            make_uint4(pack_bf16(l[0], l[1]), pack_bf16(l[2], l[3]), pack_bf16(l[4], l[5]), pack_bf16(l[6], l[7]));
      } else {
        float4* op = reinterpret_cast<float4*>(reinterpret_cast<float*>(a.out) + out_cta + o);
        op[0] = v0;
        op[1] = v1;
      }
    }
  }
}

// Inverse, 9-warp variant (FFCB_FFT_INV_PLANE=2): 264 independent column tasks (no packing), then 256 row tasks.
template <int PCH>
__global__ void __launch_bounds__(PlaneCfg<PCH>::col_threads, PlaneCfg<PCH>::ctas_per_sm)
irfft2_plane64_9w_kernel(View spec, View res, View out, float scale) {
  extern __shared__ float2 S[];
  constexpr int PPITCH = PlaneCfg<PCH>::pitch;
  const int tid = threadIdx.x, c = tid % PCH, g = tid / PCH;
  const int ch = blockIdx.x * PCH + c, b = blockIdx.y;
  if (tid < PWF * PCH) {   // g = kx
    const long long o0 = pix_off(spec, b, 0, g) + 2 * ch;
    plane64_col<true>(
        [&](int ky) {
          const long long o = o0 + ky * spec.sy;
          if (spec.fmt == FFCB_F32) return __ldg(reinterpret_cast<const float2*>(reinterpret_cast<const float*>(spec.ptr) + o));
          return make_float2(load1(spec, o), load1(spec, o + 1));
        },
        [&](int y, float2 z) { S[y * PPITCH + g * PCH + c] = z; });
  }
  __syncthreads();
  if (tid < PlaneCfg<PCH>::row_threads) {   // g = row pair
    const long long r0 = pix_off(out, b, 2 * g, 0) + ch, r1 = r0 + out.sy;
    const bool has_res = res.ptr != nullptr;
    const long long q0 = has_res ? pix_off(res, b, 2 * g, 0) + ch : 0, q1 = q0 + res.sy;
    plane64_rows_inv(
        [&](int k, float2& x1, float2& x2) {
          x1 = S[(2 * g) * PPITCH + k * PCH + c];
          x2 = S[(2 * g + 1) * PPITCH + k * PCH + c];
        },
        [&](int n0, const float2* zb) {
          float ra[16], rb[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            ra[j] = has_res ? load1(res, q0 + (n0 + j) * res.sx) : 0.f;
            rb[j] = has_res ? load1(res, q1 + (n0 + j) * res.sx) : 0.f;
          }
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            store1(out, r0 + (n0 + j) * out.sx, fmaf(zb[j].x, scale, ra[j]));
            store1(out, r1 + (n0 + j) * out.sx, fmaf(zb[j].y, scale, rb[j]));
          }
        });
  }
}

int plane_channels() {
  const char* e = getenv("FFCB_FFT_PLANE_CH");
  return (e && atoi(e) == 4) ? 4 : 8;
}

template <int PCH, int OCC>
int launch_fwd(const ffcb_tensor* in, const ffcb_tensor* spec, cudaStream_t stream) {
  using Cfg = PlaneCfg<PCH>;
  FFCB_CUDA(cudaFuncSetAttribute(rfft2_plane64_kernel<PCH, OCC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::smem));
  dim3 grid(in->C / PCH, in->B);
  rfft2_plane64_kernel<PCH, OCC><<<grid, Cfg::col_threads, Cfg::smem, stream>>>(make_view(*in), make_view(*spec), 1.0f / 64.0f);
  FFCB_LAUNCH_CHECK("rfft2_plane64_kernel");
  return FFCB_OK;
}

template <int PCH>
int launch_inv(const ffcb_tensor* spec, const ffcb_tensor* residual, const ffcb_tensor* out, cudaStream_t stream) {
  using Cfg = PlaneCfg<PCH>;
  dim3 grid(out->C / PCH, out->B);
  const View vres = (residual && residual->ptr) ? make_view(*residual) : null_view();
  if (inv_plane_variant() == 2) {
    FFCB_CUDA(cudaFuncSetAttribute(irfft2_plane64_9w_kernel<PCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::smem));
    irfft2_plane64_9w_kernel<PCH><<<grid, Cfg::col_threads, Cfg::smem, stream>>>(make_view(*spec), vres, make_view(*out), 1.0f / 64.0f);
    FFCB_LAUNCH_CHECK("irfft2_plane64_9w_kernel");
    return FFCB_OK;
  }
  FFCB_CUDA(cudaFuncSetAttribute(irfft2_plane64_kernel<PCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::smem));
  irfft2_plane64_kernel<PCH><<<grid, Cfg::row_threads, Cfg::smem, stream>>>(make_view(*spec), vres, make_view(*out), 1.0f / 64.0f);
  FFCB_LAUNCH_CHECK("irfft2_plane64_kernel");
  return FFCB_OK;
}

}  // namespace

bool plane64_eligible(const ffcb_tensor* real) {
  return real->H == PN && real->W == PN && real->C % 8 == 0 && real->B <= 65535;
}

template <bool SPLIT>
int launch_fwd_v2(const ffcb_tensor* in, const ffcb_tensor* spec, cudaStream_t stream) {
  using Cfg = PlaneCfg<8>;
  FFCB_CUDA(cudaFuncSetAttribute(rfft2_plane64_v2_kernel<8, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::smem));
  dim3 grid(in->C / 8, in->B);
  rfft2_plane64_v2_kernel<8, SPLIT><<<grid, Cfg::col_threads, Cfg::smem, stream>>>(
      reinterpret_cast<const float*>(in->ptr), in->sb, (unsigned)in->sy, (unsigned)in->sx, spec->ptr, spec->sb,
      (unsigned)spec->sy, (unsigned)spec->sx, spec->lo_off, 1.0f / 64.0f);
  FFCB_LAUNCH_CHECK("rfft2_plane64_v2_kernel");
  return FFCB_OK;
}

constexpr int kDefaultFwdPlaneRevision = 1;      // until revision 2 has been validated / measured on the GPU

// 32-bit in-plane offsets: 64 rows of either tensor must span fewer than 2^31 elements (always true on this path:
// 64 x 64 pixels x at most a few thousand channels)
bool fwd_v2_eligible(const ffcb_tensor* in, const ffcb_tensor* spec) {
  const char* e = getenv("FFCB_FFT_PLANE_FWD");   // 1 = first revision, 2 = second
  if ((e ? atoi(e) : kDefaultFwdPlaneRevision) != 2) return false;
  return in->fmt == FFCB_F32 && plane_channels() == 8 && in->sy > 0 && in->sx > 0 && spec->sy > 0 && spec->sx > 0 &&
         64 * in->sy < (1LL << 31) && 64 * spec->sy < (1LL << 31);
}

int rfft2_plane64(const ffcb_tensor* in, const ffcb_tensor* spec, cudaStream_t stream) {
  if (fwd_v2_eligible(in, spec))
    return spec->fmt == FFCB_BF16X2 ? launch_fwd_v2<true>(in, spec, stream) : launch_fwd_v2<false>(in, spec, stream);
  if (plane_channels() == 4) {
    const char* occ = getenv("FFCB_FFT_PLANE_OCC");      // 3: cap registers at 136 so that three CTAs share an SM
    return (occ && atoi(occ) == 3) ? launch_fwd<4, 3>(in, spec, stream) : launch_fwd<4, 2>(in, spec, stream);
  }
  return launch_fwd<8, 1>(in, spec, stream);
}

template <bool HAS_RES, bool OUT_SPLIT>
int launch_inv_v2(const PlaneInvArgs& a, dim3 grid, cudaStream_t stream) {
  using Cfg = PlaneCfg<8>;
  FFCB_CUDA(cudaFuncSetAttribute(irfft2_plane64_v2_kernel<HAS_RES, OUT_SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::smem));
  irfft2_plane64_v2_kernel<HAS_RES, OUT_SPLIT><<<grid, Cfg::col_threads, Cfg::smem, stream>>>(a);
  FFCB_LAUNCH_CHECK("irfft2_plane64_v2_kernel");
  return FFCB_OK;
}

bool vec_ok(const ffcb_tensor* t, int elems_per_16b) {   // 16-byte vector access to 8-channel pixels, 32-bit offsets
  return ((uintptr_t)t->ptr % 16 == 0) && t->sb % elems_per_16b == 0 && t->sy % elems_per_16b == 0 &&
         t->sx % elems_per_16b == 0 && t->lo_off % elems_per_16b == 0 && t->sy > 0 && t->sx > 0 &&
         64 * t->sy < (1LL << 31);
}

bool inv_v2_eligible(const ffcb_tensor* spec, const ffcb_tensor* residual, const ffcb_tensor* out) {
  if (plane_channels() != 8 || spec->fmt != FFCB_F32 || !vec_ok(spec, 2)) return false;
  if (residual && residual->ptr && (residual->fmt != FFCB_F32 || !vec_ok(residual, 4))) return false;
  return vec_ok(out, out->fmt == FFCB_F32 ? 4 : 8);
}

// default: the second-revision plane kernel; 0 selects the two-pass kernels, which also take every view it cannot
// handle
constexpr int kDefaultInvPlaneVariant = 3;
int inv_plane_variant() {
  const char* e = getenv("FFCB_FFT_INV_PLANE");
  if (!e || e[0] < '0' || e[0] > '3') return kDefaultInvPlaneVariant;
  return e[0] - '0';
}

// returns FFCB_OK / a negative error, or 1 when the selected variant cannot handle these views (caller falls back)
int irfft2_plane64(const ffcb_tensor* spec, const ffcb_tensor* residual, const ffcb_tensor* out, cudaStream_t stream) {
  const int variant_id = inv_plane_variant();
  if (variant_id == 3) {
    if (!inv_v2_eligible(spec, residual, out)) return 1;
    const bool has_res = residual && residual->ptr;
    PlaneInvArgs a;
    a.spec = reinterpret_cast<const float*>(spec->ptr); a.spec_sb = spec->sb; a.spec_sy = (unsigned)spec->sy; a.spec_sx = (unsigned)spec->sx;
    a.res = has_res ? reinterpret_cast<const float*>(residual->ptr) : nullptr;
    a.res_sb = has_res ? residual->sb : 0; a.res_sy = has_res ? (unsigned)residual->sy : 0; a.res_sx = has_res ? (unsigned)residual->sx : 0;
    a.out = out->ptr; a.out_sb = out->sb; a.out_sy = (unsigned)out->sy; a.out_sx = (unsigned)out->sx; a.out_lo = out->lo_off;
    a.scale = 1.0f / 64.0f;
    dim3 grid(out->C / 8, out->B);
    const bool split = out->fmt == FFCB_BF16X2;
    if (has_res) return split ? launch_inv_v2<true, true>(a, grid, stream) : launch_inv_v2<true, false>(a, grid, stream);
    return split ? launch_inv_v2<false, true>(a, grid, stream) : launch_inv_v2<false, false>(a, grid, stream);
  }
  return plane_channels() == 4 ? launch_inv<4>(spec, residual, out, stream) : launch_inv<8>(spec, residual, out, stream);
}

}  // namespace ffcb
