/*
 * ffc_b200.h — C ABI of libffc_b200.so: the H100 (sm_90a) kernels behind the drop-in
 * replacements for advimman/lama's FFC inference path
 * (reference: saicinpainting/training/modules/ffc.py).
 *
 * The reference has no FFI: its seam is the Python nn.Module surface, and every FLOP runs
 * inside torch (cuFFT / cuDNN / ATen).  This library is what a maintainer binds *instead of*
 * those torch calls; each entry point names the reference lines it replaces.  The binding
 * itself (ctypes) is lama_b200/_lib.py and is documented in INTEGRATION.md.
 *
 * Conventions
 *  - extern "C", plain pointers and sizes, no C++/torch types, no exceptions.
 *  - every function returns 0 (FFCB_OK) or a negative FFCB_E* code; the message of the last
 *    failure on the calling thread is ffcb_last_error().
 *  - all device pointers are owned by the caller (torch's caching allocator in the Python
 *    binding) and must stay alive until the stream work completes.  The library allocates
 *    nothing (FFT twiddles are generated in shared memory by the kernels themselves).
 *  - every launch goes to the caller's stream; no call synchronises or allocates, so all
 *    entry points are CUDA-graph capturable (run each op once eagerly first: kernels that need
 *    more than 48 KB of shared memory set their function attribute on first use).
 *  - activations inside the path are channels-last ("NHWC"): element (b, y, x, c) of a tensor
 *    lives at ptr + b*sb + y*sy + x*sx + c.  Strides let one allocation hold a reflect-padded
 *    plane ([B][H+2][W+2][C], ptr at the interior origin) or a channel slice of a wider tensor
 *    (the local|global halves of an FFC feature map share one 512-channel buffer).
 *    Tensors of the FourierUnit chain may instead be "channel-group planar" (ffcb_tensor.cg / .sg below).
 *  - storage formats: FFCB_F32 (float) and FFCB_BF16X2 ("split" bfloat16: value = hi + lo with
 *    hi = bf16(v), lo = bf16(v - hi); hi plane at ptr, lo plane at ptr + lo_off elements).
 *    The split format is what the wgmma path multiplies (3 bf16 products, fp32 accumulate:
 *    hi*hi + lo*hi + hi*lo, relative error ~2^-16, see DESIGN.md "precision").
 */
#ifndef FFC_B200_H_
#define FFC_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FFCB_VERSION 117 /* 0.1.7: ffcb_stem_bwd7 (0.1.6: ffcb_conv_plan; 0.1.5: ffcb_head_bwd7_bits, ffcb_relu_mask_pack_rows, ffcb_relu_bwd_bits_rows,
                            ffcb_head_gather7_rows (0.1.4: ffcb_relu_mask_pack, ffcb_relu_bwd_bits; 0.1.3:
                            ffcb_refine_l1_grad; 0.1.2: ffcb_add, ffcb_head_bwd7; 0.1.1: ffcb_tensor gained cg / tile / sg)) */

enum {
  FFCB_OK = 0,
  FFCB_EINVAL = -1,  /* bad shape / alignment / unsupported combination */
  FFCB_EARCH = -2,   /* device is not sm_90 */
  FFCB_ECUDA = -3,   /* CUDA runtime / driver error (text in ffcb_last_error) */
  FFCB_ENOMEM = -4   /* caller-provided workspace too small */
};

enum { FFCB_F32 = 0, FFCB_BF16X2 = 1 };
enum { FFCB_ACT_NONE = 0, FFCB_ACT_RELU = 1, FFCB_ACT_SIGMOID = 2, FFCB_ACT_TANH = 3 };
enum { FFCB_BORDER_ZERO = 0, FFCB_BORDER_REFLECT = 1 };
/* arithmetic of the contraction kernels */
enum {
  FFCB_MATH_FP32 = 0,   /* CUDA-core FFMA, fp32 operands (reference-grade path) */
  FFCB_MATH_BF16X3 = 1  /* wgmma (bf16) on split-bf16 operands, fp32 accumulators in registers */
};

typedef void* ffcb_stream_t; /* cudaStream_t */

/* Channels-last tensor view.  Strides are in elements of the storage type. */
typedef struct {
  void* ptr;       /* element (0,0,0,0); for FFCB_BF16X2 the hi plane */
  int64_t sb, sy, sx;
  int64_t lo_off;  /* FFCB_BF16X2: offset (elements) from the hi to the lo plane */
  int32_t B, H, W, C;
  int32_t fmt;     /* FFCB_F32 | FFCB_BF16X2 */
  int32_t pad;     /* physical border pixels around the interior (0..3).  With reflect_border != 0 the ring holds
                      the reflected image (ffcb_fill_reflect_border), so that the TMA tile of tap (dy,dx),
                      |dy|,|dx| <= pad, is the output tile shifted by (dx,dy) — no index math. */
  int32_t reflect_border;
  int32_t window;  /* != 0: "sliding window" view — consecutive pixels overlap (sx < C): pixel x exposes the C
                      contiguous elements starting at x*sx.  Used to feed the 7x7 stem to ffcb_conv as 7 K-segments
                      of (8 taps x 8 channels) read straight out of a packed NHWC8 image (see ffcb_stem_pack). */
  int32_t cg;      /* 0: plain channels-last.  > 0: "channel-group planar" — channels are stored in groups of cg
                      (4 or 8): element (b,y,x,c) lives at ptr + (c/cg)*sg + b*sb + y*sy + x*sx + (c%cg), i.e. every
                      group of cg channels is its own dense little channels-last image.  This is the layout of the
                      FourierUnit chain (SpectralTransform.conv1 -> rfft2 -> spectral conv -> irfft2 -> conv2,
                      ffc.py:145-161): one (image, group) plane set is ONE contiguous block for the plane FFT kernels
                      and the [K/8][pixel][8] "interleaved" (no-swizzle, K-major) operand tile of wgmma. */
  int32_t tile;    /* 0, or 128 with cg == 8: "tile-blocked" variant for wgmma operands — pixels are flattened
                      (m = (b*H + y)*W + x over the view) and stored in blocks of 128:
                        element (m, c) at ptr + (m/128)*sg + (c/8)*1024 + (m%128)*8 + c%8
                      so the [8 groups][128 pixels][8] operand tile of one 64-channel K block of one 128-pixel M tile is
                      ONE contiguous 16 KB run (a single cp.async.bulk per plane); sg = elements per 128-pixel block
                      (all groups of the allocation), sb / sy / sx are ignored.  Written by the plane FFT kernels,
                      read by ffcb_conv (tensor-core arm; 1x1 taps; M tiles that coincide with the blocks). */
  int64_t sg;      /* cg > 0: stride between channel groups (elements), or between 128-pixel blocks when tile != 0 */
} ffcb_tensor;

/* One K-segment of an implicit-GEMM convolution: `nch` input channels starting at channel
 * `c0` of input tensor `src`, sampled at input pixel (y*stride + dy, x*stride + dx). */
typedef struct {
  int32_t src, dy, dx, c0, nch;
} ffcb_kseg;

#define FFCB_MAX_KSEG 64

/*
 * v            = sum_seg sum_k in[seg.src][b, y*stride+dy, x*stride+dx, c0+k] * W[n][koff(seg)+k] + shift[n]
 * out[b,y,x,n] = addend_post ? act(v) + addend[b,y,x,n]      (residual: id + act(bn(conv)), ffc.py:288)
 *                            : act(v + addend[b,y,x,n])
 *
 * Replaces, with BatchNorm folded into W/shift by the caller (lama_b200/packing.py):
 *   nn.Conv2d k in {1,3} of FFC.convl2l/convl2g/convg2l            ffc.py:189-196, 221, 223
 *   SpectralTransform.conv1 (1x1 + BN + ReLU) and .conv2 (1x1)     ffc.py:128-133, 139-140, 145, 161
 *   FourierUnit.conv_layer + bn + relu on the interleaved spectrum ffc.py:57-61, 100-101
 *   FFC_BN_ACT.bn_l/bn_g + act                                     ffc.py:243-249, 253-254
 *   the residual add of FFCResnetBlock                             ffc.py:288
 *   nn.ConvTranspose2d(k3,s2,p1,op1)+BN+ReLU as four sub-pixel phases  ffc.py:350-354
 * The out view's H,W are the output grid; input coordinates outside the input's interior are
 * zero (FFCB_BORDER_ZERO) or reflected without edge repeat (FFCB_BORDER_REFLECT, ffc.py:189
 * padding_mode='reflect').
 * Output ring (FFCB_MATH_BF16X3): when `out` is a whole split-bf16 plane with a 1-pixel reflected ring
 * (out.reflect_border != 0, out.pad == 1, H, W >= 4) the kernel also writes the mirrored copies of rows 1 / H-2 and columns 1 / W-2 into the
 * ring, so the result can feed the next 3x3 reflect contraction without ffcb_fill_reflect_border.  The FP32 arm and
 * every other producer leave the ring to ffcb_fill_reflect_border.
 *
 * weight: FFCB_MATH_FP32  -> float  [Ktot][N]           (N contiguous), Ktot = sum nch
 *         FFCB_MATH_BF16X3 -> bf16  [2][N][Kpad] hi|lo   (K contiguous), Kpad = sum of nch rounded up to 64 each,
 *                                                         the padding columns zero
 * Reads of the tensor-core arm: it multiplies whole 64-channel blocks, so a segment whose nch is not a multiple of 64
 * also reads channels [c0 + nch, c0 + 64 * ceil(nch / 64)) of its source that lie inside the view (C) and multiplies
 * them by the zero padding weights: they must be finite (a NaN or Inf there makes the outputs NaN).  Channels beyond
 * the view's C and, under FFCB_BORDER_ZERO, everything outside the interior are never read.
 */
typedef struct {
  ffcb_tensor in[2];
  ffcb_tensor out;
  ffcb_tensor addend;   /* addend.ptr == NULL: none */
  const void* weight;
  const float* shift;   /* [N] or NULL */
  int32_t n_out;        /* N */
  int32_t stride;       /* 1 or 2 */
  int32_t border;       /* FFCB_BORDER_* */
  int32_t act;          /* FFCB_ACT_* */
  int32_t nseg;
  int32_t math;         /* FFCB_MATH_* */
  int32_t addend_post;  /* 0: addend joins the pre-activation sum; 1: added after the activation */
  int32_t _reserved;
  ffcb_kseg seg[FFCB_MAX_KSEG];
} ffcb_conv_desc;

int ffcb_version(void);
const char* ffcb_last_error(void);
/* 0 if `device` is an sm_90 part this library can run on */
int ffcb_check_device(int device);
void ffcb_shutdown(void);

/* Generic fused convolution / pointwise contraction (see ffcb_conv_desc). */
int ffcb_conv(const ffcb_conv_desc* desc, ffcb_stream_t stream);

/*
 * Dispatch of the tensor-core arm (FFCB_MATH_BF16X3), from the planning step ffcb_conv itself runs before it encodes
 * the tensor maps and launches: which kernel instantiation and tiling ffcb_conv would use for `desc` under the current
 * FFCB_TC_BN / FFCB_TC_ROWS / FFCB_TC_ROWS_TW (read on every call).  Host only: no device call, no tensor map, so it
 * also answers without a GPU.  A descriptor the arm refuses returns FFCB_EINVAL with the message of ffcb_conv (the
 * tensor-map encoding at launch can still refuse a descriptor with FFCB_ECUDA).
 *   kind     FFCB_PLAN_FLAT     dense 1x1 contraction, 128 flattened pixels per M tile
 *            FFCB_PLAN_SPATIAL  one TMA box per tap and 64-channel block, TW x TH pixel tiles
 *            FFCB_PLAN_ROWS     rows-resident: one (TH + dy span) x TW halo per M tile, resident weights
 *            FFCB_PLAN_HALO     column-halo: one (64 ch, TW, TH + 2) box per column shift serves three 3x3 taps
 *   il, po   tile-blocked A operands / channel-group planar float32 output (template IL / PO)
 *   ring     the epilogue also writes the output's reflected 1-pixel ring
 *   bn       N tile (32, 64, 96 or 128); m_tiles x n_tiles tiles over persistent CTAs; stages: pipeline depth
 */
enum { FFCB_PLAN_FLAT = 0, FFCB_PLAN_SPATIAL = 1, FFCB_PLAN_ROWS = 2, FFCB_PLAN_HALO = 3 };
typedef struct {
  int32_t kind;
  int32_t il, po, ring;
  int32_t bn, tw, th, stages;
  int64_t m_tiles;
  int32_t n_tiles;
  int32_t _reserved;
} ffcb_conv_plan_info;
int ffcb_conv_plan(const ffcb_conv_desc* desc, ffcb_conv_plan_info* info);

/*
 * Stem: ReflectionPad2d(3) + Conv2d(Cin -> N, k7, no bias) + folded BN + ReLU.
 * ffc.py:315-317 (FFC_BN_ACT with ratio 0/0 -> convl2l only) and :253.
 * x: NCHW float [B][Cin][H][W] contiguous (what the caller of the generator passes);
 * w: float [7*7*Cin][N] (k index = (ky*7+kx)*Cin + c); out: channels-last view.
 */
int ffcb_stem_conv7(const float* x_nchw, int B, int Cin, int H, int W, const float* w, const float* shift,
                    int N, const ffcb_tensor* out, ffcb_stream_t stream);

/*
 * Stem, tensor-core form.  ffcb_stem_pack writes the generator input as a reflect-padded (3 pixels) channels-last
 * image with 8 channels per pixel (Cin real + zeros), rows of W+8 pixels (the tail is zero), in split bf16:
 *     packed[b][yp][xp][c],  yp in [0,H+6), xp in [0,W+8),  = x[b][c][reflect(yp-3)][reflect(xp-3)]      (c < Cin)
 * and, when Cin <= 4 ("two-row" packing), packed[b][yp][xp][4+c] = packed[b][yp+1][xp][c] (zero below the last row).
 * A window view of it (C = 64, sx = 8, window = 1) exposes, at pixel x, the 8 taps x 8 channels of one kernel
 * row (two kernel rows with the two-row packing) as ONE contiguous 128-byte K block, so ReflectionPad2d(3) +
 * Conv2d(k7) (ffc.py:315-317) becomes an ffcb_conv with seven K-segments (dy = 0..6, dx = 0) and zero-padded
 * weights [N][7][8 taps][8 channels] — or four K-segments (dy = 0, 2, 4, 6) with weights
 * [N][4][8 taps][row dy | row dy+1][4 channels] when Cin <= 4 (43 % fewer tensor-core MACs).
 */
int ffcb_stem_pack(const float* x_nchw, int B, int Cin, int H, int W, const ffcb_tensor* packed, ffcb_stream_t stream);

/*
 * Head: ReflectionPad2d(3) + Conv2d(C -> N<=4, k7, bias) + activation, NCHW float output.
 * ffc.py:360-363.  w: float [N][7*7][C]; bias [N]; y: [B][N][H][W].
 */
int ffcb_head_conv7(const ffcb_tensor* in, const float* w, const float* bias, int N, int act, float* y_nchw,
                    ffcb_stream_t stream);

/*
 * Real 2-D FFT pair, norm='ortho', over the (H, W) axes of a channels-last tensor.
 *   ffcb_rfft2 : torch.fft.rfftn(x, dim=(-2,-1), norm='ortho') + the stack/permute/view that
 *                interleaves Re/Im as channels 2k / 2k+1                       ffc.py:86-89
 *                in (B,H,W,C) real -> spec (B,H,W/2+1,2C)
 *   ffcb_irfft2: the inverse view/permute/complex + torch.fft.irfftn(s=(H,W), norm='ortho'),
 *                with the residual of SpectralTransform fused: out = residual + irfft2(spec)
 *                                                                     ffc.py:103-108, 161
 *                spec (B,H,W/2+1,2C) float -> out (B,H,W,C)
 * The inverse transforms along H first (all W/2+1 columns, complex) and then C2R along W,
 * ignoring Im of the k_w=0 and (even W) k_w=W/2 bins — exactly what torch/cuFFT/MKL do for the
 * non-Hermitian post-ReLU spectrum (SURVEY.md Appendix A).
 * H and W may be any length from 1 to 1024 (W >= 2); longer axes return FFCB_EINVAL.  Most 64x64
 * planes take a fused whole-plane kernel; every other plane takes a row and a column kernel with
 * the transform in shared memory: power-of-two lengths 4..256 a compile-time Stockham plan,
 * every other length a runtime mixed-radix Stockham plan (a direct DFT for primes), with 32
 * channels per CTA up to 447 points and 8 channels per CTA for 448..1024.
 * ws: caller workspace of ffcb_fft2_workspace_bytes(B,H,W,C) bytes (row-pass intermediate).
 */
size_t ffcb_fft2_workspace_bytes(int B, int H, int W, int C);
int ffcb_rfft2(const ffcb_tensor* in, const ffcb_tensor* spec, void* ws, size_t ws_bytes, ffcb_stream_t stream);
int ffcb_irfft2(const ffcb_tensor* spec, const ffcb_tensor* residual /* nullable */, const ffcb_tensor* out,
                void* ws, size_t ws_bytes, ffcb_stream_t stream);

/*
 * Head, tensor-core form (ffc.py:360-363).  The 7x7 convolution to N <= 3 outputs is split into
 *   (1) an ffcb_conv over the kernel ROWS only — seven K-segments (dy = -3..3, dx = 0) producing, for every input
 *       column, the 7*N partial sums q[b,y,x',n*7+kx] = sum_ky sum_c in[b,y+ky-3,x',c] * w[n,c,ky,kx], and
 *   (2) this gather: y[b,n,y,x] = act(bias[n] + sum_kx q[b,y,reflect(x+kx-3),n*7+kx])   (NCHW float output).
 * q: float view (B,H,W,>=7N).
 */
int ffcb_head_gather7(const ffcb_tensor* q, const float* bias, int N, int act, float* y_nchw, ffcb_stream_t stream);

/*
 * uint8 image I/O of the predict path (SURVEY.md row f1) — the elementwise work the reference does around the
 * generator, fused into the two kernels that touch the full-resolution image anyway.
 *
 * ffcb_stem_pack_u8 replaces, for a batch of decoded RGB images [B][H0][W0][3] and masks [B][H0][W0]:
 *     load_image: u8 -> float32 / 255                         saicinpainting/evaluation/data.py:11-19
 *     pad_img_to_modulo(mode='symmetric') to (H, W)           evaluation/data.py:32-36 (bottom / right only)
 *     mask = (mask > 0) * 1                                   bin/predict.py:83
 *     masked_img = img * (1 - mask); cat([masked_img, mask])  training/trainers/default.py:59, 68
 *     ReflectionPad2d(3) of the stem                          ffc.py:315
 * and writes the packed stem image of ffcb_stem_pack (view (B, H+6, W+8, 8); H, W = padded size, H-H0 <= H0).
 *
 * ffcb_head_gather7_blend_u8 is ffcb_head_gather7 (N = 3) followed by
 *     inpainted = mask * predicted + (1 - mask) * image       training/trainers/default.py:71
 *     crop to unpad_to_size (H0, W0)                          bin/predict.py:86-91
 *     np.clip(res * 255, 0, 255).astype('uint8')              bin/predict.py:93   (truncation)
 * writing RGB bytes [B][H0][W0][3].  Pixels outside the hole reproduce the reference's u8 -> /255 -> *255 -> u8
 * round trip bit for bit (IEEE float32 division and product).
 */
int ffcb_stem_pack_u8(const uint8_t* image_hwc, const uint8_t* mask_hw, int B, int H0, int W0,
                      const ffcb_tensor* packed, ffcb_stream_t stream);
int ffcb_head_gather7_blend_u8(const ffcb_tensor* q, const float* bias, int act, const uint8_t* image_hwc,
                               const uint8_t* mask_hw, int H0, int W0, uint8_t* out_hwc, ffcb_stream_t stream);

/* Layout/format conversion at the module boundary (the reference's tensors are NCHW float):
 * ffc.py has no counterpart — these replace nothing, they adapt torch's layout to the path's. */
int ffcb_nchw_to_nhwc(const float* x_nchw, int B, int C, int H, int W, const ffcb_tensor* out, ffcb_stream_t stream);
int ffcb_nhwc_to_nchw(const ffcb_tensor* in, float* y_nchw, ffcb_stream_t stream);
/* (re)write the reflected 1-pixel border ring of a pad==1 view from its interior */
int ffcb_fill_reflect_border(const ffcb_tensor* t, ffcb_stream_t stream);

/*
 * Input gradients through FFCResnetBlock (SURVEY.md row f3; reference: evaluation/refinement.py:137-167 optimises the
 * block inputs by back-propagation).  With eval-mode BN folded, the backward pass of the block re-uses ffcb_conv (3x3
 * taps flipped, zero border, transposed weights) and the ffcb_rfft2 / ffcb_irfft2 pair itself; these two elementwise
 * steps complete it:
 *   ffcb_relu_bwd:            out = dy * [y > 0]   — nn.ReLU backward with the forward activation y (ffc.py:101,
 *                             133, 253-254); any storage format / layout on each of the three views
 *   ffcb_fold_reflect_border: adjoint of the reflect padding of ffc.py:189 (padding_mode='reflect', pad 1):
 *                             out[b,y,x,c] = sum of gpad over the padded positions that reflect onto (y,x)
 *                                           (+ add0[b,y,x,c-add0_c0] + add1[b,y,x,c-add1_c0] where defined);
 *                             gpad is (B,H+2,W+2,C); addends are optional (NULL) channel slices of the output
 */
int ffcb_relu_bwd(const ffcb_tensor* dy, const ffcb_tensor* y, const ffcb_tensor* out, ffcb_stream_t stream);
int ffcb_fold_reflect_border(const ffcb_tensor* gpad, const ffcb_tensor* add0, int add0_c0, const ffcb_tensor* add1,
                             int add1_c0, const ffcb_tensor* out, ffcb_stream_t stream);

/*
 * ReLU masks kept as bits (ffc.py:101, 133, 253-254, 354: the nn.ReLU backwards of the FourierUnit, the
 * SpectralTransform's conv1, FFC_BN_ACT and the up-sampling stages only test the forward activation for sign), so that
 * a forward+backward program can release the activation itself after the forward:
 *   ffcb_relu_mask_pack: bits[((b*H + y)*W + x)*nw + c/32] bit c%32 = [y(b,y,x,c) > 0], nw = ceil(C/32), over the
 *                        interior of the view (B, H, W, C of `y`); the nw*32 - C unused high bits of a pixel's last word
 *                        are 0.  The value compared is the one ffcb_relu_bwd reads (hi + lo for FFCB_BF16X2).
 *   ffcb_relu_bwd_bits:  out = dy * bit — ffcb_relu_bwd with the mask of `y` packed by ffcb_relu_mask_pack (bits
 *                        sized by out's B, H, W, C), bit-identical to it.
 * Both take every view ffcb_relu_bwd takes: either storage format, rings, channel slices, channel-group planar and
 * tile-blocked views.  bits: device memory of B*H*W*nw uint32, 4-byte aligned.
 */
int ffcb_relu_mask_pack(const ffcb_tensor* y, uint32_t* bits, ffcb_stream_t stream);
int ffcb_relu_bwd_bits(const ffcb_tensor* dy, const uint32_t* bits, const ffcb_tensor* out, ffcb_stream_t stream);

/*
 * Row bands of a bit mask (the banded up-sampling tail of the refinement step, lama_b200/banded.py): `bits` is the mask
 * of a whole plane of H rows, B*H*W*nw words laid out as above, and the view (`y`, resp. `dy` / `out`) holds its rows
 * [row0, row0 + view.H) (view.W = the plane's W).  With H = view.H and row0 = 0 these are ffcb_relu_mask_pack and
 * ffcb_relu_bwd_bits.  For B > 1 a band's words are not contiguous: image b's rows start at word b*H*W*nw.
 */
int ffcb_relu_mask_pack_rows(const ffcb_tensor* y, uint32_t* bits, int H, int row0, ffcb_stream_t stream);
int ffcb_relu_bwd_bits_rows(const ffcb_tensor* dy, const uint32_t* bits, int H, int row0, const ffcb_tensor* out,
                            ffcb_stream_t stream);

/*
 * Input gradients through the generator's rear (residual blocks -> ConcatTupleLayer -> up-sampling tail -> head,
 * ffc.py:345-363; what evaluation/refinement.py:137-167 back-propagates through on every Adam step) as one program:
 *   ffcb_add:       out = a + b elementwise over the whole padded extent (interior and ring) of three views of one
 *                   geometry (B, H, W, C, pad); any storage format on each; `out` may alias `a`.  Replaces the block
 *                   identity add `x_l + y_l, x_g + y_g` (ffc.py:288) where the backward needs y (= Y2, the conv2 ReLU
 *                   output) kept apart.  Summing the reflected rings keeps out's ring a reflection of its interior.
 *   ffcb_head_bwd7: adjoint of ReflectionPad2d(3) -> Conv2d(Cin -> N <= 4, k7) -> act (ffc.py:360-363), fused with
 *                   the ReLU of the last up-sampling stage (ffc.py:354):
 *                     out = [mask > 0] * Fold3(Conv7^T(act'(y) * dy))
 *                   y, dy: the forward output and its gradient, NCHW float [B][N][H][W]; act' = y(1-y) (sigmoid),
 *                   1-y^2 (tanh), 1 (none); w: float [N][7*7][Cin] (the layout of ffcb_head_conv7); Conv7^T scatters
 *                   every output pixel's gradient over its 7x7 window of the (H+6)x(W+6) padded plane and Fold3 adds
 *                   each padded position onto the interior pixel the reflection copied it from.  mask, out: (B, H, W,
 *                   Cin) views (mask = the last up-sampling output, any ring width).  H, W >= 4.
 */
int ffcb_add(const ffcb_tensor* a, const ffcb_tensor* b, const ffcb_tensor* out, ffcb_stream_t stream);
int ffcb_head_bwd7(const float* y_nchw, const float* dy_nchw, int B, int N, int H, int W, const float* w, int act,
                   const ffcb_tensor* mask, const ffcb_tensor* out, ffcb_stream_t stream);
/*
 * ffcb_head_bwd7_bits: ffcb_head_bwd7 with the mask read as bits (ffcb_relu_mask_pack of the last up-sampling output,
 * B*H*W*ceil(Cin/32) words of the whole plane), writing rows [row0, row0 + out.H) of the result into out (B, rows, W,
 * Cin).  y, dy are the whole NCHW planes: a band reads the gradient rows its 7x7 windows reach and folds the
 * reflection only at the plane's own top and bottom rows, so every pixel gets the operands, and the summation order,
 * of ffcb_head_bwd7 — the two are equal bit for bit.
 * ffcb_head_gather7_rows: ffcb_head_gather7 writing rows [row0, row0 + q.H) of an NCHW output of H rows.
 */
int ffcb_head_bwd7_bits(const float* y_nchw, const float* dy_nchw, int B, int N, int H, int W, const float* w, int act,
                        const uint32_t* mask_bits, int row0, const ffcb_tensor* out, ffcb_stream_t stream);
int ffcb_head_gather7_rows(const ffcb_tensor* q, const float* bias, int N, int act, float* y_nchw, int H, int row0,
                           ffcb_stream_t stream);

/*
 * Input gradient through the whole generator (lama_b200/generator_grad.py): the adjoint of the stem's
 * ReflectionPad2d(3) -> Conv2d(Cin -> N, k7) (ffc.py:314-316, pix2pixhd.py:365-366) w.r.t. the NCHW input:
 *   ffcb_stem_bwd7: dx = Fold3(Conv7^T(g))
 *                   g: (B, H, W, N) view of the gradient w.r.t. the stem's pre-activation (its ReLU mask applied),
 *                   either storage format, any ring; w: float [N][7*7][Cin] (the stem weight with the BN scale
 *                   folded along N); dx: float NCHW [B][Cin][H][W], overwritten.  Conv7^T scatters every pixel's
 *                   gradient over its 7x7 window of the (H+6)x(W+6) padded plane, Fold3 adds each padded position onto
 *                   the interior pixel the reflection copied it from.  1 <= Cin <= 16, H, W >= 4.  No atomics: each
 *                   pixel sums its terms in one order, independent of the batch and the tiling.
 */
int ffcb_stem_bwd7(const ffcb_tensor* g, const float* w, int Cin, float* dx_nchw, ffcb_stream_t stream);

/*
 * Gradient of the refinement loss w.r.t. the prediction (evaluation/refinement.py:75-84 _l1_loss, 19-26 _pyrdown,
 * 151-158 the loss of one Adam step), per image b of NCHW float32 tensors:
 *   L_b = mean_{c,p: mask < 1e-8} |pred - image|                      over the padded plane (B, C, Hp, Wp)
 *       + mean_{c,q: md >= 1e-8} |D(pred[:, :, :H0, :W0]) - ref|       ref (B, C, H0/2, W0/2), md (B, 1, H0/2, W0/2)
 *   D   = bilinear (align_corners=False, source max(scale (d + 0.5) - 0.5, 0), scale = in / out) to (H0/2, W0/2)
 *         with the source index and weights computed as torch's double-precision interpolate does (then rounded
 *         to float); torch's float32 interpolate computes them in float, which differs by up to ~1e-5 at d ~ 100
 *         o 5x5 separable Gaussian with reflect-101 padding (kornia's gaussian_blur2d, border 'reflect')
 *   grad = dL_b / dpred = sign(pred - image) [mask < 1e-8] inv_n[b][0]
 *                         + D^T(sign(D pred - ref) [md >= 1e-8] inv_n[b][1])        (zero outside the crop)
 * mask (B, 1, Hp, Wp); inv_n (B, 2) device floats 1 / n_out, 1 / n_down with n = C x the selected pixel count, 0 for
 * an empty selection (that term then adds no gradient and its loss is NaN, as torch.mean of nothing); taps: the 5
 * float Gaussian taps; work: B*C*(H0/2)*(W0/2) floats of scratch.  loss (B, 2): the two terms (reported only, summed
 * with atomics).  sign(0) = 0.  The gradient is a fixed-order gather per element: no atomics, batch-independent.
 * C in [1, 4], 3 <= H0 <= Hp, 3 <= W0 <= Wp.
 */
int ffcb_refine_l1_grad(const float* pred, const float* image, const float* mask, int B, int C, int Hp, int Wp, int H0,
                        int W0, const float* ref, const float* md, const float* inv_n, const float* taps, float* work,
                        float* grad, float* loss, ffcb_stream_t stream);

/* number of kernel launches issued by this library on the calling thread since the last
 * ffcb_reset_launch_count() — bench.py reports it as "gpu_launches" */
long long ffcb_launch_count(void);
void ffcb_reset_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* FFC_B200_H_ */
