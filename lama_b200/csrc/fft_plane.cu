// Fused 2-D real FFT pair for 64x64 channels-last planes (the bottleneck of 512x512 images): one CTA transforms the
// whole plane of 8 channels, so the half-spectrum intermediate lives in shared memory instead of a global workspace
// (halves the HBM traffic of ffcb_rfft2 / ffcb_irfft2 and removes two launches).
//
// Every 64-point transform is held in the registers of ONE thread (fft64_regs: unrolled 8x8 Cooley-Tukey with
// compile-time twiddles) — no shuffles, no shared-memory butterflies, one barrier per plane.  288 threads:
//   forward : 256 threads = 8 channels x 32 row pairs (two-for-one real rows) -> S[y][kx][c] -> barrier ->
//             264 threads = 8 channels x 33 complex columns -> spectrum (Re/Im interleaved, scaled; float32 or split
//             bf16, chosen per store)
//   inverse : 264 column tasks (complex, along H) -> S -> barrier -> 256 row-pair tasks (C2R along W), results staged
//             channels-last in place of their rows -> whole-pixel vector epilogue (+ residual).  It takes a float32
//             spectrum and residual and 16-byte aligned views (plane64_inv_eligible); fft.cu sends every other view
//             to the two-pass kernels.
// smem: S[64][kP64Pitch] float2, row pitch 33*8 + 4 (the +4 spreads the four row-pair groups of a warp over both
// halves of the banks), 137 KB: one CTA per SM.  Lanes: 8 consecutive channels (32 B of a pixel) x 4 rows/columns.
#include <stdint.h>

#include "common.cuh"
#include "fft_core.cuh"

namespace ffcb {
namespace {

using namespace fftc;
constexpr int PN = 64, PWF = 33;
constexpr int PCH = 8;                                       // channels per CTA
constexpr int kThreads = (PWF * PCH + 31) / 32 * 32;         // 33 x 8 column tasks, whole warps
constexpr size_t kSmem = sizeof(float2) * PN * kP64Pitch;

// Rows by the first 32*PCH threads, the 33 x PCH column tasks by the first 33*PCH (chosen over packing the DC and
// Nyquist columns into one transform on 256 threads: fewer registers per thread, and one more warp to hide latency).
__global__ void __launch_bounds__(kThreads, 1) rfft2_plane64_kernel(View in, View spec, float scale) {
  extern __shared__ float2 S[];
  constexpr int PPITCH = kP64Pitch;
  const int tid = threadIdx.x, c = tid % PCH, g = tid / PCH;
  const int ch = blockIdx.x * PCH + c, b = blockIdx.y;
  if (tid < 32 * PCH) {   // g = row pair
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

// Inverse: one task per column, then C2R rows, with
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
__global__ void __launch_bounds__(kThreads, 1) irfft2_plane64_v2_kernel(PlaneInvArgs a) {
  extern __shared__ float2 S[];
  constexpr int PPITCH = kP64Pitch;
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

template <bool HAS_RES, bool OUT_SPLIT>
int launch_inv(const PlaneInvArgs& a, dim3 grid, cudaStream_t stream) {
  FFCB_CUDA(cudaFuncSetAttribute(irfft2_plane64_v2_kernel<HAS_RES, OUT_SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem));
  irfft2_plane64_v2_kernel<HAS_RES, OUT_SPLIT><<<grid, kThreads, kSmem, stream>>>(a);
  FFCB_LAUNCH_CHECK("irfft2_plane64_v2_kernel");
  return FFCB_OK;
}

bool vec_ok(const ffcb_tensor* t, int elems_per_16b) {   // 16-byte vector access to 8-channel pixels, 32-bit offsets
  return ((uintptr_t)t->ptr % 16 == 0) && t->sb % elems_per_16b == 0 && t->sy % elems_per_16b == 0 &&
         t->sx % elems_per_16b == 0 && t->lo_off % elems_per_16b == 0 && t->sy > 0 && t->sx > 0 &&
         64 * t->sy < (1LL << 31);
}

}  // namespace

bool plane64_eligible(const ffcb_tensor* real) {
  return real->H == PN && real->W == PN && real->C % 8 == 0 && real->B <= 65535;
}

bool plane64_inv_eligible(const ffcb_tensor* spec, const ffcb_tensor* residual, const ffcb_tensor* out) {
  if (spec->fmt != FFCB_F32 || !vec_ok(spec, 2)) return false;
  if (residual && residual->ptr && (residual->fmt != FFCB_F32 || !vec_ok(residual, 4))) return false;
  return vec_ok(out, out->fmt == FFCB_F32 ? 4 : 8);
}

int rfft2_plane64(const ffcb_tensor* in, const ffcb_tensor* spec, cudaStream_t stream) {
  FFCB_CUDA(cudaFuncSetAttribute(rfft2_plane64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem));
  dim3 grid(in->C / PCH, in->B);
  rfft2_plane64_kernel<<<grid, kThreads, kSmem, stream>>>(make_view(*in), make_view(*spec), 1.0f / 64.0f);
  FFCB_LAUNCH_CHECK("rfft2_plane64_kernel");
  return FFCB_OK;
}

// views as plane64_eligible(out) && plane64_inv_eligible(spec, residual, out) accept
int irfft2_plane64(const ffcb_tensor* spec, const ffcb_tensor* residual, const ffcb_tensor* out, cudaStream_t stream) {
  const bool has_res = residual && residual->ptr;
  PlaneInvArgs a;
  a.spec = reinterpret_cast<const float*>(spec->ptr); a.spec_sb = spec->sb; a.spec_sy = (unsigned)spec->sy; a.spec_sx = (unsigned)spec->sx;
  a.res = has_res ? reinterpret_cast<const float*>(residual->ptr) : nullptr;
  a.res_sb = has_res ? residual->sb : 0; a.res_sy = has_res ? (unsigned)residual->sy : 0; a.res_sx = has_res ? (unsigned)residual->sx : 0;
  a.out = out->ptr; a.out_sb = out->sb; a.out_sy = (unsigned)out->sy; a.out_sx = (unsigned)out->sx; a.out_lo = out->lo_off;
  a.scale = 1.0f / 64.0f;
  dim3 grid(out->C / PCH, out->B);
  const bool split = out->fmt == FFCB_BF16X2;
  if (has_res) return split ? launch_inv<true, true>(a, grid, stream) : launch_inv<true, false>(a, grid, stream);
  return split ? launch_inv<false, true>(a, grid, stream) : launch_inv<false, false>(a, grid, stream);
}

}  // namespace ffcb
