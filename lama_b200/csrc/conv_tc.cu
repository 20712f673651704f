// Tensor-core arm of ffcb_conv() (FFCB_MATH_BF16X3): implicit-GEMM convolution with the warpgroup MMA
// (wgmma) of sm_90a.
//
//   D[128 pixels x BN] (fp32, registers)  +=  A_hi*W_hi + A_lo*W_hi + A_hi*W_lo        per 64-channel K block
//
// Operands are "split bf16" (value = hi + lo, include/ffc_b200.h): three bf16 products with fp32
// accumulation carry ~16 mantissa bits per operand (vs 8 for plain bf16, 11 for tf32) with the same
// operand bytes as fp32.
//
// Data movement: every operand tile is one TMA box (cp.async.bulk.tensor, 128-byte swizzle) —
//   activations: 5-D map (C, W+2p, H+2p, B, plane) over the reflect-ring-padded NHWC buffer; the tile of
//                tap (dy,dx) is the same box shifted by (dx,dy); stride-2 convs use elementStrides=2;
//                zero-border convs map the interior only and let TMA zero-fill out-of-bounds;
//                dense 1x1 inputs (spectra, W/2+1 columns) use a flat 3-D map (C, B*H*W, plane);
//                tile-blocked inputs (ffcb_tensor.tile, the FourierUnit chain) need no map: the "interleaved"
//                K-major operand tile [K/8][pixel][8] is one contiguous 16 KB run, fetched with a 1-D bulk copy;
//   weights    : 3-D map (Kpad, N, plane), K-major.
// Warp roles (384 threads, persistent CTAs, one per SM): warp 0 = TMA producer (warp-uniform control flow, one lane
// chosen by elect.sync issues); warpgroups 1 and 2 = consumers.  Consumer g owns pixel rows [64g, 64g+64) of the
// 128-pixel tile: per K block it issues the three products as m64nBNk16 wgmmas straight from the shared-memory stage
// (both operands through matrix descriptors), keeps one K block of wgmmas in flight while it releases the stage
// before, and after the last K block runs the epilogue from its registers (shift / addend / activation -> split-bf16
// or fp32 channels-last stores, or planar float32 stores; the reflected ring of a whole-plane output is written here
// too).  The producer runs up to `stages` K blocks ahead, so the loads of the next tile overlap the epilogue.
// Template parameters select the operand / output kinds (IL, PO), the rows-resident mode of the 7x7 shell layers
// (RR: one halo load per M tile, resident weight tiles) and the column-halo mode of stride-1 3x3 contractions (HALO:
// per M tile, 64-channel block and column shift one box serves the three taps of that column; see
// TcParams::seg_taps).
#include <cuda.h>
#include <stdlib.h>

#include <type_traits>

#include "common.cuh"

namespace ffcb {
namespace {

constexpr int BM = 128;          // pixels per tile (two m64 wgmma row blocks)
constexpr int BK = 64;           // bf16 channels per K block = one 128-byte swizzle row
constexpr int WG_K = 16;         // K of one bf16 wgmma
constexpr int kThreads = 384;    // producer warpgroup + 2 consumer warpgroups
constexpr int kConsumers = 256;
constexpr int kTileABytes = BM * BK * 2;   // 16 KB per plane
constexpr int kMaxStages = 8;
constexpr int kBarBytes = 1024;  // mbarriers, padded so that the stages stay 1024-byte aligned
constexpr int kSmemLimit = 227 * 1024;     // opt-in dynamic shared memory per block on sm_90

struct TcParams {
  View out, addend;
  const float* shift;
  int N, act, addend_post;
  int BN, num_n_tiles;
  long long num_m_tiles;
  int stages;
  int flat;                  // 1: M = B*H*W flattened (dense 1x1), 0: spatial TW x TH tiles
  int TW, TH, tiles_x, tiles_y;
  int stride;
  int coord_off[2];          // +1 when in[src] is mapped with its border ring
  int nseg;
  // Tile-blocked "interleaved" A operands (ffcb_tensor.tile == 128, cg == 8; the FourierUnit chain): the operand tile
  // [8 groups][128 pixels][8 channels] of one 64-channel K block of one M tile is ONE contiguous 16 KB run per plane,
  // fetched with a single 1-D bulk copy and multiplied through a no-swizzle K-major descriptor (core matrix = 8
  // pixels x 16 B; SBO 128 B, LBO 2048 B).
  int a_il[2];
  const unsigned short* a_ptr[2];
  long long a_sg[2], a_lo[2];     // elements per 128-pixel block, hi -> lo plane offset
  int a_tiles_per_image[2];       // spatial mode: 128-pixel blocks per image (H * W / 128)
  int out_planar;                 // out is channel-group planar float32
  int ring;                       // out has a 1-pixel reflected ring: the epilogue also writes the mirrored copies
  int hints;                      // L2 residency hints for the planar (FourierUnit chain) outputs
  // Rows-resident mode (template RR; the 7x7 head's row contraction and the windowed 7x7 stem): every K segment is the
  // SAME 64-channel block of one source shifted by dy only, so the activation tile is loaded ONCE per M tile as a
  // (TH + R) x TW halo (a dy shift is a whole number of 1024-byte swizzle atoms, the wgmma descriptor just starts
  // (dy - dy0) * TW rows further down) and the (small) weight tiles of all segments stay resident in shared memory
  // for the whole kernel.
  int rr_dy0, rr_a_bytes, rr_w_bytes;
  // Column-halo mode (template HALO; stride-1 3x3 reflect contractions over ring-padded channels-last sources, 64 x 2
  // tiles).  The K order is channel-block-major, then dx, then dy: per M tile, 64-channel block of a complete 3x3 group
  // (nine consecutive segments, same src / c0 / nch, every (dy,dx) in {-1,0,1}^2) and column shift dx, ONE TMA box of
  // (64 ch, TW, TH+2) pixels per plane lands in an A buffer, and the three taps of that column read it dy * TW rows
  // further down — whole 1024-byte swizzle atoms, as in RR — so 3 boxes of 4 rows replace 9 boxes of 2 rows (a third
  // fewer activation bytes into shared memory).  Every other segment is a one-tap group over the same kind of box.
  // Shared memory: 2 A buffers x (hi | lo) x halo_a_bytes (2 x 2 x 32 KB at 64 x 2), then a ring of one-tap weight
  // stages: 64 channels x BN x (hi | lo) = 32 KB at BN = 128, 3 of them in 227 KB.
  // seg_taps[s]: 9 = segment s starts a 3x3 group, 0 = inside one, 1 = a one-tap group.
  int halo_a_bytes;
  signed char seg_taps[FFCB_MAX_KSEG];
  ffcb_kseg seg[FFCB_MAX_KSEG];
};

// ------------------------------------------------------------------------------------------ PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}

__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// 1-D bulk copy global -> shared, completion on an mbarrier (bytes: multiple of 16, both addresses 16-byte aligned)
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// wgmma shared-memory matrix descriptors, as (lo, hi) 32-bit words: lo = start address >> 4 (bits [0,14)) | LBO >> 4
// (bits [16,30)); hi = SBO >> 4 (bits [32,46)) | layout type (bits [62,64): 1 = 128-byte swizzle, 0 = none).
// Advancing along K only touches the start-address field of the low word.
//   128-byte swizzle, K-major: rows 128 B apart, 8-row groups 1024 B apart (SBO); LBO unused (1).
//   no swizzle ("interleaved") K-major: the tile is [K/8][128 rows][8 bf16]; a core matrix is 8 rows x 16 B = 128
//   contiguous bytes, 8-row groups follow each other every 128 B (SBO) and the two 16-byte K chunks of one K = 16
//   step are one slab = 2048 B apart (LBO).
constexpr uint32_t kLoSw = 1u << 16;
constexpr uint32_t kHiSw = (uint32_t)(1024 >> 4) | (1u << 30);
constexpr uint32_t kLoIl = (uint32_t)(2048 >> 4) << 16;
constexpr uint32_t kHiIl = (uint32_t)(128 >> 4);

__device__ __forceinline__ uint32_t desc_addr(uint32_t saddr) { return (saddr & 0x3FFFF) >> 4; }

__device__ __forceinline__ uint64_t desc64(uint32_t lo, uint32_t hi) {
  uint64_t d;
  asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "r"(lo), "r"(hi));
  return d;
}
// one lane of the (converged) warp
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of the accumulator registers across a wgmma fence / wait
template <int BN>
__device__ __forceinline__ void fence_acc(float* d) {
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, bf16 in, fp32 accumulators: d[4j + 2h + c] = D[row 16w + lane/4 + 8h]
// [col 8j + 2(lane%4) + c] for warp w of the warpgroup.
__device__ __forceinline__ void wgmma_n32(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
      "}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_n64(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_n96(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
      "}, %48, %49, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_n128(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <int BN>
__device__ __forceinline__ void wgmma_bn(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
  static_assert(BN == 32 || BN == 64 || BN == 96 || BN == 128, "N tile");
  if constexpr (BN == 32) wgmma_n32(d, da, db, scale_d);
  else if constexpr (BN == 64) wgmma_n64(d, da, db, scale_d);
  else if constexpr (BN == 96) wgmma_n96(d, da, db, scale_d);
  else wgmma_n128(d, da, db, scale_d);
}

// ------------------------------------------------------------------------------------------ kernel
struct TileCoord {
  int b, y0, x0;       // spatial: first output pixel of the tile
  long long m0;        // flat: first flattened pixel
};

__device__ __forceinline__ TileCoord tile_coord(const TcParams& p, long long m_tile) {
  TileCoord t;
  if (p.flat) {
    t.m0 = m_tile * BM;
    t.b = 0; t.y0 = 0; t.x0 = 0;
  } else {
    const int per_img = p.tiles_x * p.tiles_y;
    t.b = (int)(m_tile / per_img);
    const int r = (int)(m_tile - (long long)t.b * per_img);
    t.y0 = (r / p.tiles_x) * p.TH;
    t.x0 = (r % p.tiles_x) * p.TW;
    t.m0 = 0;
  }
  return t;
}

// IL: some K segment reads a channel-group planar ("interleaved") operand.  The instantiation without them walks the
// whole contraction with one descriptor kind.
// PO: the output is channel-group planar float32.
// BN: the N tile (TcParams::BN), a compile-time wgmma shape.
template <bool IL, bool PO, bool RR, bool HALO, int BN>
__global__ void __launch_bounds__(kThreads, 1)
conv_tc_kernel(const __grid_constant__ TcParams p, const __grid_constant__ CUtensorMap map_in0,
               const __grid_constant__ CUtensorMap map_in1, const __grid_constant__ CUtensorMap map_w) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [RR: resident weights | HALO: 2 A buffers of (hi | lo)] stages of [A_hi | A_lo | W_hi | W_lo] (HALO: one-tap
  // weight stages [W_hi | W_lo]), then barriers
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int w_bytes = p.BN * BK * 2;
  const int stage_bytes = RR ? 2 * p.rr_a_bytes : HALO ? 2 * w_bytes : 2 * kTileABytes + 2 * w_bytes;
  uint8_t* w_res = smem;                                   // RR: resident weight tiles [seg][hi | lo]
  uint8_t* a_buf = smem;                                   // HALO: A buffers [2][hi | lo]
  if constexpr (RR) smem += p.rr_w_bytes;
  if constexpr (HALO) smem += (size_t)4 * p.halo_a_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * stage_bytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + kMaxStages;
  uint64_t* w_bar = bars + 2 * kMaxStages;                 // RR: the resident weights have landed
  uint64_t* a_full = bars + 2 * kMaxStages + 1;            // HALO: A buffer landed / released (2 each)
  uint64_t* a_empty = a_full + 2;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&map_in0);
    prefetch_tmap(&map_in1);
    prefetch_tmap(&map_w);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kConsumers); }
    if constexpr (RR) mbar_init(w_bar, 1);
    if constexpr (HALO)
      for (int s = 0; s < 2; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], kConsumers); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // K blocks of the whole contraction
  int total_kblocks = 0;
  for (int s = 0; s < p.nseg; ++s) total_kblocks += (p.seg[s].nch + BK - 1) / BK;
  const long long num_tiles = p.num_m_tiles * p.num_n_tiles;

  if (warp == 0) {
    // ================================================================ TMA producer (uniform control flow, one elected lane issues)
    if constexpr (HALO) {
      // per group, 64-channel block and column shift dx: the A buffer (the column box shifted by dx), then one weight
      // stage per tap of that column (weight K of tap t, block j = kofs + (t * nblk + j) * 64, kofs = the group's
      // first K)
      int stage = 0, ast = 0;
      uint32_t phase = 0, aph = 0;
      for (long long t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int n_tile = (int)(t % p.num_n_tiles);
        const TileCoord tc = tile_coord(p, t / p.num_n_tiles);
        int kofs = 0;
        for (int s = 0; s < p.nseg;) {
          const int ntap = p.seg_taps[s];
          const ffcb_kseg g = p.seg[s];
          const CUtensorMap* map = g.src ? &map_in1 : &map_in0;
          const int nblk = (g.nch + BK - 1) / BK;
          for (int j = 0; j < nblk; ++j) {
            for (int u = 0; u < (ntap == 9 ? 3 : 1); ++u) {
              const int dxu = ntap == 9 ? u - 1 : g.dx;
              mbar_wait(&a_empty[ast], aph ^ 1);
              if (elect_one()) {
                uint8_t* ab = a_buf + (size_t)ast * 2 * p.halo_a_bytes;
                mbar_expect_tx(&a_full[ast], 2u * p.TW * (p.TH + 2) * BK * 2);
                const int cx = tc.x0 + dxu + p.coord_off[g.src], cy = tc.y0 - 1 + p.coord_off[g.src];
                tma_load_5d(ab, map, &a_full[ast], g.c0 + j * BK, cx, cy, tc.b, 0);
                tma_load_5d(ab + p.halo_a_bytes, map, &a_full[ast], g.c0 + j * BK, cx, cy, tc.b, 1);
              }
              __syncwarp();
              if (++ast == 2) { ast = 0; aph ^= 1; }
              for (int tap = 0; tap < ntap; ++tap) {
                if (p.seg[s + tap].dx != dxu) continue;
                mbar_wait(&empty[stage], phase ^ 1);
                if (elect_one()) {
                  uint8_t* st = smem + (size_t)stage * stage_bytes;
                  mbar_expect_tx(&full[stage], (uint32_t)stage_bytes);
                  const int k = kofs + (tap * nblk + j) * BK;
                  tma_load_3d(st, &map_w, &full[stage], k, n_tile * p.BN, 0);
                  tma_load_3d(st + w_bytes, &map_w, &full[stage], k, n_tile * p.BN, 1);
                }
                __syncwarp();
                if (++stage == p.stages) { stage = 0; phase ^= 1; }
              }
            }
          }
          kofs += ntap * nblk * BK;
          s += ntap;
        }
      }
    } else if constexpr (RR) {
      const ffcb_kseg g0 = p.seg[0];
      const CUtensorMap* map = g0.src ? &map_in1 : &map_in0;
      if (elect_one()) {
        mbar_expect_tx(w_bar, (uint32_t)p.rr_w_bytes);
        for (int s = 0; s < p.nseg; ++s) {
          tma_load_3d(w_res + (size_t)s * 2 * w_bytes, &map_w, w_bar, s * BK, 0, 0);
          tma_load_3d(w_res + (size_t)s * 2 * w_bytes + w_bytes, &map_w, w_bar, s * BK, 0, 1);
        }
      }
      __syncwarp();
      int stage = 0;
      uint32_t phase = 0;
      for (long long t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const TileCoord tc = tile_coord(p, t);
        mbar_wait(&empty[stage], phase ^ 1);
        if (elect_one()) {
          uint8_t* st = smem + (size_t)stage * stage_bytes;
          mbar_expect_tx(&full[stage], (uint32_t)stage_bytes);
          const int cx = tc.x0 + g0.dx + p.coord_off[g0.src], cy = tc.y0 + p.rr_dy0 + p.coord_off[g0.src];
          tma_load_5d(st, map, &full[stage], g0.c0, cx, cy, tc.b, 0);
          tma_load_5d(st + p.rr_a_bytes, map, &full[stage], g0.c0, cx, cy, tc.b, 1);
        }
        __syncwarp();
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
    } else {
      int stage = 0;
      uint32_t phase = 0;
      for (long long t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        // tile order: N tiles of one pixel tile are adjacent, so the CTAs working on them run
        // concurrently and share the activation tile through L2 (one DRAM read instead of num_n_tiles)
        const int n_tile = (int)(t % p.num_n_tiles);
        const TileCoord tc = tile_coord(p, t / p.num_n_tiles);
        int kb = 0;
        for (int s = 0; s < p.nseg; ++s) {
          const ffcb_kseg g = p.seg[s];
          const CUtensorMap* map = g.src ? &map_in1 : &map_in0;
          const int nblk = (g.nch + BK - 1) / BK;
          const int cx = tc.x0 * p.stride + g.dx + p.coord_off[g.src];
          const int cy = tc.y0 * p.stride + g.dy + p.coord_off[g.src];
          const int il = IL ? p.a_il[g.src] : 0;
          for (int j = 0; j < nblk; ++j, ++kb) {
            mbar_wait(&empty[stage], phase ^ 1);
            if (elect_one()) {
              uint8_t* st = smem + (size_t)stage * stage_bytes;
              mbar_expect_tx(&full[stage], (uint32_t)stage_bytes);
              const int cc = g.c0 + j * BK;
              if (IL && il) {
                // one contiguous 16 KB run per plane: block of this M tile, groups cc/8 .. cc/8+7
                const long long blk = p.flat ? (tc.m0 >> 7)
                                             : (long long)tc.b * p.a_tiles_per_image[g.src] + ((tc.y0 * p.out.W) >> 7);
                const unsigned short* src = p.a_ptr[g.src] + blk * p.a_sg[g.src] + (long long)(cc >> 3) * 1024;
                bulk_load(st, src, kTileABytes, &full[stage]);
                bulk_load(st + kTileABytes, src + p.a_lo[g.src], kTileABytes, &full[stage]);
              } else if (p.flat) {
                tma_load_3d(st, map, &full[stage], cc, (int)tc.m0, 0);
                tma_load_3d(st + kTileABytes, map, &full[stage], cc, (int)tc.m0, 1);
              } else {
                tma_load_5d(st, map, &full[stage], cc, cx, cy, tc.b, 0);
                tma_load_5d(st + kTileABytes, map, &full[stage], cc, cx, cy, tc.b, 1);
              }
              tma_load_3d(st + 2 * kTileABytes, &map_w, &full[stage], kb * BK, n_tile * p.BN, 0);
              tma_load_3d(st + 2 * kTileABytes + w_bytes, &map_w, &full[stage], kb * BK, n_tile * p.BN, 1);
            }
            __syncwarp();
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ================================================================ consumers (2 warpgroups)
    const int g = (warp >> 2) - 1;                 // row block: pixels [64g, 64g + 64) of the tile
    const int w = warp & 3, q = lane & 3;
    // after the pair exchange below, this thread owns ONE pixel row of the tile and 4 consecutive channels of every
    // 8-column group of the accumulator: even lanes row 16w + lane/4, odd lanes the row 8 below
    const int row = g * 64 + w * 16 + (lane >> 2) + 8 * (q & 1);
    const int cb = 4 * (q >> 1);
    const bool odd = (q & 1) != 0;
    const uint32_t a_row_sw = (uint32_t)(g * 64 * BK * 2) >> 4;     // 64 rows of 128 B down the swizzled tile
    const uint32_t a_row_il = (uint32_t)(g * 64 * 16) >> 4;         // 64 rows of 16 B down one interleaved slab
    const int HW = p.out.H * p.out.W;
    const bool has_add = p.addend.ptr != nullptr;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0, ast = 0;
    uint32_t phase = 0, aph = 0;
    // HALO: row of the column box holding this warpgroup's first pixel at dy = 0 (tile row g, below the top halo row)
    const int a_row0 = (g + 1) * p.TW;
    if constexpr (RR) mbar_wait(w_bar, 0);
    for (long long t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const int n_tile = (int)(t % p.num_n_tiles);
      const TileCoord tc = tile_coord(p, t / p.num_n_tiles);
      fence_acc<BN>(acc);
      if constexpr (HALO) {
        // Release protocol (one tap of wgmmas in flight, wait<1>).  A weight stage goes back after the wait of the next
        // tap: its wgmmas have retired then.  An A buffer is read by every tap of its column, so it goes back only
        // after the wait of the FIRST tap of the next column, which retires the column's last wgmmas.  The end of the
        // tile (wait<0>) releases the last of each.
        int prev = -1, a_prev = -1, nt = 0;
        for (int s = 0; s < p.nseg;) {
          const int ntap = p.seg_taps[s];
          const int nblk = (p.seg[s].nch + BK - 1) / BK;
          for (int j = 0; j < nblk; ++j) {
            for (int u = 0; u < (ntap == 9 ? 3 : 1); ++u) {
              const int dxu = ntap == 9 ? u - 1 : p.seg[s].dx;
              mbar_wait(&a_full[ast], aph);
              const uint32_t ab = smem_u32(a_buf + (size_t)ast * 2 * p.halo_a_bytes);
              for (int tap = 0; tap < ntap; ++tap) {
                const int dy = p.seg[s + tap].dy;
                if (p.seg[s + tap].dx != dxu) continue;
                // this warpgroup's 64 pixels shifted by dy: 64 rows of 128 B further down per row of the column box,
                // whole 1024-byte swizzle atoms
                const uint32_t a_off = (uint32_t)((a_row0 + dy * p.TW) * (BK * 2)) >> 4;
                const uint32_t a_hi = desc_addr(ab) + a_off;
                const uint32_t a_lo = desc_addr(ab + (uint32_t)p.halo_a_bytes) + a_off;
                mbar_wait(&full[stage], phase);
                wgmma_fence();
                const uint32_t st = smem_u32(smem + (size_t)stage * stage_bytes);
                const uint32_t w_hi = desc_addr(st), w_lo = desc_addr(st + (uint32_t)w_bytes);
#pragma unroll
                for (int k = 0; k < BK / WG_K; ++k) {
                  const uint32_t adv = (uint32_t)((k * WG_K * 2) >> 4);     // +32 B per K = 16 inside the swizzle row
                  wgmma_bn<BN>(acc, desc64((a_hi + adv) | kLoSw, kHiSw), desc64((w_hi + adv) | kLoSw, kHiSw),
                               (nt | k) != 0);
                  wgmma_bn<BN>(acc, desc64((a_lo + adv) | kLoSw, kHiSw), desc64((w_hi + adv) | kLoSw, kHiSw), 1);
                  wgmma_bn<BN>(acc, desc64((a_hi + adv) | kLoSw, kHiSw), desc64((w_lo + adv) | kLoSw, kHiSw), 1);
                }
                wgmma_commit();
                wgmma_wait<1>();
                if (prev >= 0) mbar_arrive(&empty[prev]);
                prev = stage;
                if (++stage == p.stages) { stage = 0; phase ^= 1; }
                if (a_prev >= 0) { mbar_arrive(&a_empty[a_prev]); a_prev = -1; }
                ++nt;
              }
              a_prev = ast;
              if (++ast == 2) { ast = 0; aph ^= 1; }
            }
          }
          s += ntap;
        }
        wgmma_wait<0>();
        fence_acc<BN>(acc);
        mbar_arrive(&empty[prev]);
        mbar_arrive(&a_empty[a_prev]);
      } else if constexpr (RR) {
        mbar_wait(&full[stage], phase);
        const uint32_t st = smem_u32(smem + (size_t)stage * stage_bytes);
        const uint32_t wr = smem_u32(w_res);
        for (int sgi = 0; sgi < p.nseg; ++sgi) {
          wgmma_fence();
          const uint32_t a_off = (uint32_t)((p.seg[sgi].dy - p.rr_dy0) * p.TW * (BK * 2));
          const uint32_t a_hi = desc_addr(st + a_off) + a_row_sw;
          const uint32_t a_lo = desc_addr(st + a_off + (uint32_t)p.rr_a_bytes) + a_row_sw;
          const uint32_t w_hi = desc_addr(wr + (uint32_t)(sgi * 2 * w_bytes));
          const uint32_t w_lo = desc_addr(wr + (uint32_t)(sgi * 2 * w_bytes + w_bytes));
#pragma unroll
          for (int k = 0; k < BK / WG_K; ++k) {
            const uint32_t adv = (uint32_t)((k * WG_K * 2) >> 4);
            wgmma_bn<BN>(acc, desc64((a_hi + adv) | kLoSw, kHiSw), desc64((w_hi + adv) | kLoSw, kHiSw), (sgi | k) != 0);
            wgmma_bn<BN>(acc, desc64((a_lo + adv) | kLoSw, kHiSw), desc64((w_hi + adv) | kLoSw, kHiSw), 1);
            wgmma_bn<BN>(acc, desc64((a_hi + adv) | kLoSw, kHiSw), desc64((w_lo + adv) | kLoSw, kHiSw), 1);
          }
          wgmma_commit();
          wgmma_wait<1>();
        }
        wgmma_wait<0>();
        fence_acc<BN>(acc);
        mbar_arrive(&empty[stage]);
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      } else {
        // one loop over the K blocks of the whole contraction; IL: the segment (and with it the descriptor kind of
        // the A operand) is tracked alongside
        int prev = -1, sgi = 0, j = 0;
        for (int kb = 0; kb < total_kblocks; ++kb) {
          const bool il = IL && p.a_il[p.seg[sgi].src] != 0;
          const uint32_t a_lodesc = il ? kLoIl : kLoSw, a_hidesc = il ? kHiIl : kHiSw;
          const uint32_t a_row = il ? a_row_il : a_row_sw;
          const uint32_t a_step = il ? (uint32_t)(4096 >> 4) : (uint32_t)((WG_K * 2) >> 4);   // 2 slabs / +32 B
          if (IL && ++j == (p.seg[sgi].nch + BK - 1) / BK) { ++sgi; j = 0; }
          mbar_wait(&full[stage], phase);
          wgmma_fence();
          const uint32_t st = smem_u32(smem + (size_t)stage * stage_bytes);
          const uint32_t a_hi = desc_addr(st) + a_row;
          const uint32_t a_lo = desc_addr(st + kTileABytes) + a_row;
          const uint32_t w_hi = desc_addr(st + 2 * kTileABytes);
          const uint32_t w_lo = desc_addr(st + 2 * kTileABytes + w_bytes);
#pragma unroll
          for (int k = 0; k < BK / WG_K; ++k) {
            const uint32_t wadv = (uint32_t)((k * WG_K * 2) >> 4);     // +32 B per K = 16 inside the swizzle row
            const uint32_t aadv = (uint32_t)k * a_step;
            wgmma_bn<BN>(acc, desc64((a_hi + aadv) | a_lodesc, a_hidesc), desc64((w_hi + wadv) | kLoSw, kHiSw),
                         (kb | k) != 0);
            wgmma_bn<BN>(acc, desc64((a_lo + aadv) | a_lodesc, a_hidesc), desc64((w_hi + wadv) | kLoSw, kHiSw), 1);
            wgmma_bn<BN>(acc, desc64((a_hi + aadv) | a_lodesc, a_hidesc), desc64((w_lo + wadv) | kLoSw, kHiSw), 1);
          }
          wgmma_commit();
          // the wgmmas of the previous K block have retired: its stage goes back to the producer
          wgmma_wait<1>();
          if (prev >= 0) mbar_arrive(&empty[prev]);
          prev = stage;
          if (++stage == p.stages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_acc<BN>(acc);
        mbar_arrive(&empty[prev]);
      }

      // ---- epilogue: this thread's pixel
      int b, y, x;
      bool valid;
      if (p.flat) {
        const unsigned m = (unsigned)tc.m0 + (unsigned)row;            // host guarantees B*H*W < 2^31
        valid = m < (unsigned)(p.out.B * HW);
        const unsigned mm = valid ? m : 0u;
        b = (int)(mm / (unsigned)HW);
        const unsigned r = mm - (unsigned)b * (unsigned)HW;
        y = (int)(r / (unsigned)p.out.W);
        x = (int)(r - (unsigned)y * (unsigned)p.out.W);
      } else {
        b = tc.b;
        y = tc.y0 + row / p.TW;
        x = tc.x0 + row % p.TW;
        valid = y < p.out.H && x < p.out.W;
      }
      const long long o_out = valid ? pix_off(p.out, b, y, x) : 0;
      const long long o_add = (has_add && valid) ? pix_off(p.addend, b, y, x) : 0;
      // this pixel's mirror images in the output's reflected ring, as element offsets from the pixel itself (0: none):
      // pixels of rows 1 / H-2 and columns 1 / W-2 also land on the ring (<= 3 copies) — no separate ring kernel
      int mir_dy = 0, mir_dx = 0;
      if (!PO && p.ring && valid) {
        int my, mx;
        if (ring_mirrors(p.out, y, x, my, mx)) {
          if (my != -2) mir_dy = (my - y) * (int)p.out.sy;
          if (mx != -2) mir_dx = (mx - x) * (int)p.out.sx;
        }
      }
      const uint64_t pol = l2_policy(PO && p.hints ? 2 : 0);      // planar outputs: consumed by the next kernel
      // Shift and addend of EB column groups are loaded before any of their stores: the stores may alias the addend
      // (an in-place residual), so loads placed after them would each wait a full global-memory round trip.
      constexpr int EB = (BN / 8) % 8 == 0 ? 8 : 4;
      static_assert((BN / 8) % EB == 0, "whole batches of column groups");
#pragma unroll
      for (int j0 = 0; j0 < BN / 8; j0 += EB) {
        float4 shv[EB], adv[EB];
#pragma unroll
        for (int i = 0; i < EB; ++i) {
          const int n = n_tile * p.BN + 8 * (j0 + i) + cb;
          const bool ok = valid && n < p.N;
          shv[i] = (ok && p.shift != nullptr) ? __ldg(reinterpret_cast<const float4*>(p.shift + n))
                                               : make_float4(0.f, 0.f, 0.f, 0.f);
          adv[i] = (ok && has_add) ? load4(p.addend, o_add + n) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int i = 0; i < EB; ++i) {
          const int j = j0 + i;
          // lane pairs swap half of their 8-column group: even lanes keep row r, odd lanes row r + 8
          const float s0 = odd ? acc[4 * j] : acc[4 * j + 2], s1 = odd ? acc[4 * j + 1] : acc[4 * j + 3];
          const float r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
          float4 v = odd ? make_float4(r0, r1, acc[4 * j + 2], acc[4 * j + 3])
                         : make_float4(acc[4 * j], acc[4 * j + 1], r0, r1);
          const int n = n_tile * p.BN + 8 * j + cb;
          if (!valid || n >= p.N) continue;
          const float4 sh = shv[i], ad = adv[i];
          v.x += sh.x; v.y += sh.y; v.z += sh.z; v.w += sh.w;
          if (!p.addend_post) { v.x += ad.x; v.y += ad.y; v.z += ad.z; v.w += ad.w; }
          if (p.act == FFCB_ACT_RELU) {
            v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
          } else if (p.act != FFCB_ACT_NONE) {
            v.x = slow_act(v.x, p.act); v.y = slow_act(v.y, p.act); v.z = slow_act(v.z, p.act); v.w = slow_act(v.w, p.act);
          }
          if (p.addend_post) { v.x += ad.x; v.y += ad.y; v.z += ad.z; v.w += ad.w; }
          if constexpr (PO) {
            st_hint_f4(reinterpret_cast<float*>(p.out.ptr) + o_out + chan_off(p.out, n), v, pol);
          } else {
            store4(p.out, o_out + n, v);
            if (mir_dy) store4(p.out, o_out + mir_dy + n, v);
            if (mir_dx) store4(p.out, o_out + mir_dx + n, v);
            if (mir_dy && mir_dx) store4(p.out, o_out + mir_dy + mir_dx + n, v);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int encode_typed(CUtensorMap* map, void* base, CUtensorMapDataType dt, CUtensorMapSwizzle sw, int rank,
                 const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box, const cuuint32_t* estr,
                 const char* what) {
  EncodeTiledFn fn = get_encode();
  if (fn == nullptr) {
    set_error("conv(tc): cuTensorMapEncodeTiled entry point unavailable");
    return FFCB_ECUDA;
  }
  CUresult r = fn(map, dt, (cuuint32_t)rank, base, dims, strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("conv(tc): cuTensorMapEncodeTiled(%s) failed with CUresult %d (rank %d, dims %llu %llu %llu, box %u %u %u)",
              what, (int)r, rank, (unsigned long long)dims[0], (unsigned long long)dims[1],
              (unsigned long long)(rank > 2 ? dims[2] : 0), box[0], box[1], rank > 2 ? box[2] : 0);
    return FFCB_ECUDA;
  }
  return FFCB_OK;
}

int encode(CUtensorMap* map, void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
           const cuuint32_t* box, const cuuint32_t* estr, const char* what) {
  return encode_typed(map, base, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, CU_TENSOR_MAP_SWIZZLE_128B, rank, dims, strides_bytes,
                      box, estr, what);
}

// N-tile width (one wgmma N, at most 128).  Pipeline depth matters more than tile area here: every stage carries 32 KB
// of activations (hi+lo) plus 256 B per output column, so BN=128 leaves 3 stages in flight in 227 KB, BN>=192 only 2.
int pick_bn(int n) {
  if (const char* e = getenv("FFCB_TC_BN")) {          // tuning knob: force the N tile (multiple of 32, <= 128)
    const int v = atoi(e);
    if (v >= 32 && v <= 128 && v % 32 == 0) return v < n ? v : (n + 31) / 32 * 32;
  }
  if (n <= 128) return (n + 31) / 32 * 32;
  if (n == 192) return 96;
  return 128;
}

// Everything a launch needs except the tensor maps, decided on the host from the descriptor (and the FFCB_TC_*
// variables) alone: conv_tc() launches what plan_tc() decides, ffcb_conv_plan() reports it.
struct TcPlan {
  TcParams p;
  bool used[2], taps[2];
  int kind;                  // FFCB_PLAN_*
  bool il, po;               // template parameters IL / PO of the instantiation
  int rr_span;               // RR: rows of halo below the tile (largest minus smallest dy)
  int kpad;                  // K of the weight matrix: every segment padded to whole 64-channel blocks
  int stage_bytes, bar_bytes;
  size_t smem;
};

int plan_tc(const ffcb_conv_desc* d, TcPlan& pl) {
  TcParams& p = pl.p;
  bool* used = pl.used;
  bool* taps = pl.taps;
  // ---- requirements of this arm (the fp32 arm has none of them)
  FFCB_REQUIRE(d->out.B > 0, "conv(tc): empty batch");
  FFCB_REQUIRE((long long)d->out.B * d->out.H * d->out.W < (1ll << 31), "conv(tc): more than 2^31 output pixels");
  used[0] = used[1] = taps[0] = taps[1] = false;
  int reach[2] = {0, 0};       // furthest tap offset per source: the ring must be at least that wide
  for (int i = 0; i < d->nseg; ++i) {
    used[d->seg[i].src] = true;
    if (d->seg[i].dx != 0 || d->seg[i].dy != 0) taps[d->seg[i].src] = true;
    const int ax = d->seg[i].dx < 0 ? -d->seg[i].dx : d->seg[i].dx, ay = d->seg[i].dy < 0 ? -d->seg[i].dy : d->seg[i].dy;
    if (ax > reach[d->seg[i].src]) reach[d->seg[i].src] = ax;
    if (ay > reach[d->seg[i].src]) reach[d->seg[i].src] = ay;
    FFCB_REQUIRE(d->seg[i].c0 % 8 == 0, "conv(tc): segment %d starts at channel %d (must be a multiple of 8)", i,
                 d->seg[i].c0);
  }
  for (int s = 0; s < 2; ++s) {
    if (!used[s]) continue;
    const ffcb_tensor& t = d->in[s];
    FFCB_REQUIRE(t.fmt == FFCB_BF16X2, "conv(tc): in[%d] must be split bf16 (FFCB_BF16X2)", s);
    if (t.cg != 0) {
      // interleaved operand: 1x1 taps at unit stride only, whole 64-channel K blocks, dense group images
      FFCB_REQUIRE(t.cg == 8 && t.tile == 128 && !taps[s] && d->stride == 1 && t.H == d->out.H && t.W == d->out.W,
                   "conv(tc): a channel-group planar in[%d] must be tile-blocked (tile=128, cg=8) with 1x1 taps, stride 1",
                   s);
      for (int i = 0; i < d->nseg; ++i)
        if (d->seg[i].src == s)
          FFCB_REQUIRE(d->seg[i].nch % 64 == 0 && d->seg[i].c0 % 8 == 0,
                       "conv(tc): segment %d of a channel-group planar input must cover whole 64-channel blocks", i);
    }
    FFCB_REQUIRE(t.sx % 8 == 0 && t.sy % 8 == 0 && t.sb % 8 == 0 && t.lo_off % 8 == 0 && ((uintptr_t)t.ptr % 16) == 0,
                 "conv(tc): in[%d] strides / pointer not 16-byte aligned", s);
    if (taps[s] && d->border == FFCB_BORDER_REFLECT)
      FFCB_REQUIRE(t.pad >= reach[s] && t.reflect_border, "conv(tc): in[%d] needs a reflected border ring of %d pixels",
                   s, reach[s]);
  }

  p.out = make_view(d->out);
  p.out_planar = d->out.cg != 0 ? 1 : 0;
  p.ring = (d->out.reflect_border && d->out.pad == 1 && d->out.cg == 0 && d->out.fmt == FFCB_BF16X2 && d->out.H >= 4 &&
            d->out.W >= 4) ? 1 : 0;
  if (d->out.cg != 0)
    FFCB_REQUIRE(d->out.fmt == FFCB_F32 && d->out.sx % 4 == 0 && d->out.sy % 4 == 0 && d->out.sb % 4 == 0,
                 "conv(tc): channel-group planar outputs are float32");
  if (d->out.cg != 0)     // 16-byte stores
    FFCB_REQUIRE(d->out.sg % 4 == 0 && (reinterpret_cast<uintptr_t>(d->out.ptr) & 15) == 0,
                 "conv(tc): planar output needs 16-byte aligned channel groups");
  p.hints = l2_hints_enabled() ? 1 : 0;
  p.addend = d->addend.ptr ? make_view(d->addend) : null_view();
  p.shift = d->shift;
  p.N = d->n_out; p.act = d->act; p.addend_post = d->addend_post;
  p.BN = pick_bn(d->n_out);
  p.num_n_tiles = (d->n_out + p.BN - 1) / p.BN;
  p.stride = d->stride;
  p.nseg = d->nseg;
  int kpad = 0;
  for (int i = 0; i < d->nseg; ++i) {
    p.seg[i] = d->seg[i];
    kpad += (d->seg[i].nch + BK - 1) / BK * BK;
  }

  // ---- tiling: flat when every tap is (0,0) on dense unit-stride inputs, else spatial TW x TH
  const int H = d->out.H, W = d->out.W;
  bool flat = d->stride == 1 && !taps[0] && !taps[1];
  for (int s = 0; s < 2 && flat; ++s) {
    if (!used[s]) continue;
    const ffcb_tensor& t = d->in[s];
    flat = t.H == H && t.W == W && (t.tile != 0 || (t.sy == (int64_t)W * t.sx && t.sb == (int64_t)H * t.sy));
  }
  for (int s = 0; s < 2; ++s) {
    p.a_il[s] = 0; p.a_ptr[s] = nullptr; p.a_sg[s] = p.a_lo[s] = 0; p.a_tiles_per_image[s] = 0;
    if (!used[s] || d->in[s].cg == 0) continue;
    const ffcb_tensor& t = d->in[s];
    p.a_il[s] = 1;
    p.a_ptr[s] = reinterpret_cast<const unsigned short*>(t.ptr);
    p.a_sg[s] = t.sg; p.a_lo[s] = t.lo_off;
    p.a_tiles_per_image[s] = (t.H * t.W) >> 7;
    FFCB_REQUIRE(t.lo_off % 8 == 0, "conv(tc): tile-blocked in[%d]: lo plane not 16-byte aligned", s);
  }
  p.flat = flat ? 1 : 0;
  // rows-resident mode (TcParams::rr_*): every segment = the same 64-channel block of one channels-last source, shifted
  // by dy only (the 7x7 head's row contraction, the windowed 7x7 stem), into a channels-last output (the RR
  // instantiation has no planar epilogue), with the resident weights and two halo stages fitting in shared memory;
  // FFCB_TC_ROWS=0 disables it
  bool rr = false;
  int rr_dy_min = 0, rr_dy_max = 0, rr_tw = 8;
  p.rr_dy0 = p.rr_a_bytes = p.rr_w_bytes = 0;
  {
    const char* e = getenv("FFCB_TC_ROWS");
    rr = !flat && d->stride == 1 && d->nseg >= 3 && p.num_n_tiles == 1 && (e ? atoi(e) != 0 : true) &&
         d->in[d->seg[0].src].cg == 0 && d->out.cg == 0;
    rr_dy_min = rr_dy_max = d->seg[0].dy;
    for (int i = 0; i < d->nseg && rr; ++i) {
      const ffcb_kseg& g = d->seg[i];
      rr = g.src == d->seg[0].src && g.c0 == d->seg[0].c0 && g.nch == BK && g.dx == d->seg[0].dx;
      for (int j = 0; j < i && rr; ++j) rr = d->seg[j].dy != g.dy;
      if (g.dy < rr_dy_min) rr_dy_min = g.dy;
      if (g.dy > rr_dy_max) rr_dy_max = g.dy;
    }
    rr = rr && (rr_dy_max - rr_dy_min) <= 8;
    // a dy shift = TW rows of 128 B must be whole 1024-byte swizzle atoms: TW = 8 (tall tiles: the smallest halo,
    // 22 rows x 8 pixels = 44 KB per stage for a 7-tap column) or 16; FFCB_TC_ROWS_TW overrides
    const char* etw = getenv("FFCB_TC_ROWS_TW");
    rr_tw = (etw && atoi(etw) == 16) ? 16 : 8;
    if (rr) {
      const int w_res = d->nseg * 2 * p.BN * BK * 2;
      const int halo_stage = 2 * (BM / rr_tw + rr_dy_max - rr_dy_min) * rr_tw * BK * 2;
      rr = (kSmemLimit - 1024 - kBarBytes - w_res) / halo_stage >= 2;
    }
  }
  // column-halo mode (TcParams::seg_taps): spatial, stride 1, planes wider than 32 (the current tiling's TW >= 64),
  // and channels-last outputs; every segment reads a reflect-ring-padded channels-last source within one pixel
  // (coord_off >= 1); at least one complete 3x3 group.  Contractions with a tile-blocked segment (the global one:
  // convl2g + st.conv2) keep the per-tap path: on big-lama's 64-wide planes the column-halo mode measured 1-4 % slower
  // for them, even with two tile-blocked K blocks per A buffer (DESIGN.md §9).
  bool halo = !flat && !rr && d->stride == 1 && W > 32 && d->out.cg == 0;
  int ngroups = 0;
  for (int i = 0; i < d->nseg && halo;) {
    const ffcb_kseg& g = d->seg[i];
    const ffcb_tensor& t = d->in[g.src];
    halo = t.cg == 0 && d->border == FFCB_BORDER_REFLECT && taps[g.src] && t.pad >= 1 && t.window == 0;
    unsigned mask = 0;
    int n = 0;
    for (; n < 9 && i + n < d->nseg; ++n) {
      const ffcb_kseg& q = d->seg[i + n];
      if (q.src != g.src || q.c0 != g.c0 || q.nch != g.nch || q.dy < -1 || q.dy > 1 || q.dx < -1 || q.dx > 1) break;
      mask |= 1u << ((q.dy + 1) * 3 + q.dx + 1);
    }
    if (n == 9 && mask == 0x1FFu) {
      p.seg_taps[i] = 9;
      for (int k = 1; k < 9; ++k) p.seg_taps[i + k] = 0;
      i += 9;
      ++ngroups;
    } else {
      halo = halo && g.dy >= -1 && g.dy <= 1 && g.dx >= -1 && g.dx <= 1;
      p.seg_taps[i++] = 1;
    }
  }
  halo = halo && ngroups > 0;
  p.halo_a_bytes = 0;
  if (flat) {
    p.TW = BM; p.TH = 1; p.tiles_x = p.tiles_y = 1;
    p.num_m_tiles = ((long long)d->out.B * H * W + BM - 1) / BM;
  } else if (rr) {
    p.TW = rr_tw;
    p.TH = BM / p.TW;
    p.tiles_x = (W + p.TW - 1) / p.TW;
    p.tiles_y = (H + p.TH - 1) / p.TH;
    p.num_m_tiles = (long long)d->out.B * p.tiles_x * p.tiles_y;
    p.rr_dy0 = rr_dy_min;
    p.rr_a_bytes = (p.TH + rr_dy_max - rr_dy_min) * p.TW * BK * 2;
    p.rr_w_bytes = d->nseg * 2 * p.BN * BK * 2;
  } else if (halo) {
    // 64 x 2 tiles for every plane width (column tiles beyond 64): each warpgroup's 64 pixels are one image row of the
    // column box, so a dy shift is 64 rows = 8 swizzle atoms; the box is 4 x 64 pixel rows (32 KB per plane; a 128 x 1
    // tile would need 3 x 128 rows, and two A buffers of those leave no room for weight stages)
    p.TW = 64; p.TH = 2;
    p.tiles_x = (W + p.TW - 1) / p.TW;
    p.tiles_y = (H + p.TH - 1) / p.TH;
    p.num_m_tiles = (long long)d->out.B * p.tiles_x * p.tiles_y;
    p.halo_a_bytes = p.TW * (p.TH + 2) * BK * 2;
  } else {
    int tw = 1;
    while (tw < W && tw < BM) tw <<= 1;      // smallest power of two >= W, capped at 128
    p.TW = tw; p.TH = BM / tw;
    p.tiles_x = (W + p.TW - 1) / p.TW;
    p.tiles_y = (H + p.TH - 1) / p.TH;
    p.num_m_tiles = (long long)d->out.B * p.tiles_x * p.tiles_y;
    FFCB_REQUIRE(p.TW * d->stride <= 256 && p.TH * d->stride <= 256, "conv(tc): tile exceeds the TMA box limit");
  }

  for (int s = 0; s < 2; ++s)
    if (p.a_il[s] && !flat)
      FFCB_REQUIRE(p.TW == W && p.TW * p.TH == BM && H % p.TH == 0 && (H * W) % BM == 0,
                   "conv(tc): tile-blocked in[%d] in a spatial contraction needs M tiles of whole rows (W a power of two "
                   "<= 128 dividing 128, H*W a multiple of 128); got %dx%d", s, H, W);
  // activation coordinates: +pad when the source is mapped with its reflected ring
  for (int s = 0; s < 2; ++s)
    p.coord_off[s] = (used[s] && !p.a_il[s] && !flat && taps[s] && d->border == FFCB_BORDER_REFLECT) ? d->in[s].pad : 0;
  FFCB_REQUIRE(((uintptr_t)d->weight % 16) == 0, "conv(tc): weight pointer not 16-byte aligned");
  if (d->out.cg == 0) {
    const ffcb_tensor& t = d->out;
    const int64_t esz = t.fmt == FFCB_BF16X2 ? 2 : 4;
    FFCB_REQUIRE(((uintptr_t)t.ptr % 16) == 0 && (t.sx * esz) % 16 == 0 && (t.sy * esz) % 16 == 0 &&
                     (t.sb * esz) % 16 == 0 && (esz == 4 || (t.lo_off * esz) % 16 == 0),
                 "conv(tc): out strides / pointer not 16-byte aligned (C must be a multiple of %d)", esz == 2 ? 8 : 4);
  }

  // stage: RR the halo (hi | lo), HALO one tap's weight tile (hi | lo), else one K block of A and W (hi | lo each);
  // the resident weights (RR) / the two A buffers (HALO) are carved next to the barriers
  pl.stage_bytes = rr ? 2 * p.rr_a_bytes : halo ? 2 * p.BN * BK * 2 : 2 * kTileABytes + 2 * p.BN * BK * 2;
  pl.bar_bytes = kBarBytes + (rr ? p.rr_w_bytes : 0) + (halo ? 4 * p.halo_a_bytes : 0);
  int stages = (kSmemLimit - 1024 - pl.bar_bytes) / pl.stage_bytes;
  if (stages > kMaxStages) stages = kMaxStages;
  FFCB_REQUIRE(stages >= 2, "conv(tc): BN=%d leaves fewer than 2 pipeline stages", p.BN);
  p.stages = stages;
  pl.smem = (size_t)stages * pl.stage_bytes + pl.bar_bytes + 1024;

  pl.kind = flat ? FFCB_PLAN_FLAT : rr ? FFCB_PLAN_ROWS : halo ? FFCB_PLAN_HALO : FFCB_PLAN_SPATIAL;
  pl.il = !rr && !halo && (p.a_il[0] || p.a_il[1]);
  pl.po = p.out_planar != 0;
  pl.rr_span = rr ? rr_dy_max - rr_dy_min : 0;
  pl.kpad = kpad;
  return FFCB_OK;
}

}  // namespace

int conv_tc_plan(const ffcb_conv_desc* d, ffcb_conv_plan_info* info) {
  TcPlan pl;
  const int rc = plan_tc(d, pl);
  if (rc) return rc;
  info->kind = pl.kind;
  info->il = pl.il;
  info->po = pl.po;
  info->ring = pl.p.ring;
  info->bn = pl.p.BN;
  info->tw = pl.p.TW;
  info->th = pl.p.TH;
  info->stages = pl.p.stages;
  info->m_tiles = pl.p.num_m_tiles;
  info->n_tiles = pl.p.num_n_tiles;
  info->_reserved = 0;
  return FFCB_OK;
}

int conv_tc(const ffcb_conv_desc* d, cudaStream_t stream) {
  TcPlan pl;
  int rc = plan_tc(d, pl);
  if (rc) return rc;
  TcParams& p = pl.p;
  const bool rr = pl.kind == FFCB_PLAN_ROWS, halo = pl.kind == FFCB_PLAN_HALO, flat = pl.kind == FFCB_PLAN_FLAT;

  // ---- tensor maps
  alignas(64) CUtensorMap maps[3];
  for (int s = 0; s < 2; ++s) {
    if (!pl.used[s] || p.a_il[s]) continue;     // no tensor map (bulk copies / unused): patched with a valid one below
    const ffcb_tensor& t = d->in[s];
    const cuuint64_t esz = 2;
    if (flat) {
      cuuint64_t dims[3] = {(cuuint64_t)t.C, (cuuint64_t)t.B * t.H * t.W, 2};
      cuuint64_t str[2] = {(cuuint64_t)t.sx * esz, (cuuint64_t)t.lo_off * esz};
      cuuint32_t box[3] = {BK, BM, 1}, es[3] = {1, 1, 1};
      if ((rc = encode(&maps[s], t.ptr, 3, dims, str, box, es, "flat activations"))) return rc;
    } else {
      const int off = p.coord_off[s];
      char* base = (char*)t.ptr - (int64_t)off * ((int64_t)t.sy + t.sx) * (int64_t)esz;
      cuuint64_t dims[5] = {(cuuint64_t)t.C, (cuuint64_t)(t.W + 2 * off), (cuuint64_t)(t.H + 2 * off),
                            (cuuint64_t)t.B, 2};
      cuuint64_t str[4] = {(cuuint64_t)t.sx * esz, (cuuint64_t)t.sy * esz, (cuuint64_t)t.sb * esz,
                           (cuuint64_t)t.lo_off * esz};
      cuuint32_t box[5] = {BK, (cuuint32_t)(p.TW * d->stride), (cuuint32_t)(p.TH * d->stride), 1, 1};
      if (rr) box[2] = (cuuint32_t)(p.TH + pl.rr_span);      // the whole halo of the tile in one box
      if (halo) box[2] = (cuuint32_t)(p.TH + 2);            // the tile's rows and one above / below
      cuuint32_t es[5] = {1, (cuuint32_t)d->stride, (cuuint32_t)d->stride, 1, 1};
      if ((rc = encode(&maps[s], base, 5, dims, str, box, es, "spatial activations"))) return rc;
    }
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)pl.kpad, (cuuint64_t)d->n_out, 2};
    cuuint64_t str[2] = {(cuuint64_t)pl.kpad * 2, (cuuint64_t)pl.kpad * d->n_out * 2};
    cuuint32_t box[3] = {BK, (cuuint32_t)p.BN, 1}, es[3] = {1, 1, 1};
    if ((rc = encode(&maps[2], const_cast<void*>(d->weight), 3, dims, str, box, es, "weights"))) return rc;
  }
  for (int s = 0; s < 2; ++s)
    if (!pl.used[s] || p.a_il[s]) maps[s] = maps[2];      // never dereferenced by the kernel, but prefetched

  // ---- launch: the instantiation of the plan
  int dev = 0, sms = 132;
  FFCB_CUDA(cudaGetDevice(&dev));
  FFCB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const long long tiles = p.num_m_tiles * p.num_n_tiles;
  const int grid = (int)(tiles < sms ? tiles : sms);
  const size_t smem = pl.smem;
  auto launch = [&](auto kernel) -> int {
    FFCB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    kernel<<<grid, kThreads, smem, stream>>>(p, maps[0], maps[1], maps[2]);
    return FFCB_OK;
  };
  auto launch_bn = [&](auto bn) -> int {
    constexpr int N = decltype(bn)::value;
    if (rr) return launch(conv_tc_kernel<false, false, true, false, N>);      // plan_tc: never il / po
    if (halo) return launch(conv_tc_kernel<false, false, false, true, N>);
    if (pl.il)
      return pl.po ? launch(conv_tc_kernel<true, true, false, false, N>)
                   : launch(conv_tc_kernel<true, false, false, false, N>);
    return pl.po ? launch(conv_tc_kernel<false, true, false, false, N>)
                 : launch(conv_tc_kernel<false, false, false, false, N>);
  };
  switch (p.BN) {
    case 32: rc = launch_bn(std::integral_constant<int, 32>()); break;
    case 64: rc = launch_bn(std::integral_constant<int, 64>()); break;
    case 96: rc = launch_bn(std::integral_constant<int, 96>()); break;
    default: rc = launch_bn(std::integral_constant<int, 128>()); break;
  }
  if (rc) return rc;
  FFCB_LAUNCH_CHECK("conv_tc_kernel");
  return FFCB_OK;
}

}  // namespace ffcb
