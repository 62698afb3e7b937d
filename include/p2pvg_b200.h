/* p2pvg_b200 — C ABI of the sm_90a kernels behind the p2pvg training hot path.
 *
 * The reference (yccyenchicheng/p2pvg) has no FFI of its own: its boundary for this path is the Python
 * module API (models/p2p_model.py, models/lstm.py, models/dcgan_64.py, models/dcgan_128.py,
 * misc/criterion.py).  The drop-in Python modules in p2pvg_b200/ keep that API and call the entry
 * points below through ctypes.  Each entry point cites the reference lines whose arithmetic it
 * replaces.  Conventions:
 *   - plain pointers and sizes only; all pointers are DEVICE pointers unless stated otherwise;
 *   - the caller (PyTorch) owns every buffer; the library allocates nothing persistent;
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*);
 *   - return 0 on success, a negative P2PVG_ERR_* code otherwise; p2pvg_last_error() gives the text
 *     (thread-local).  There is no CPU fallback: unsupported shapes are errors.
 *   - dtype: 0 = fp32, 1 = bf16 ("act dtype" of the conv stacks); statistics/LSTM/optimizer are fp32.
 *   - activations are NHWC, flattened to [rows, C]; a "group" is one encoder/decoder call of the
 *     reference (BatchNorm statistics are per group, SURVEY.md §3.3).
 */
#ifndef P2PVG_B200_H
#define P2PVG_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
struct p2pvg_conv_fusion;

#define P2PVG_OK 0
#define P2PVG_ERR_BAD_ARG -1
#define P2PVG_ERR_UNSUPPORTED -2
#define P2PVG_ERR_CUDA -3
#define P2PVG_ERR_WORKSPACE -4

#define P2PVG_F32 0
#define P2PVG_BF16 1
#define P2PVG_F64 2 /* p2pvg_histograms segments only */

#define P2PVG_ACT_NONE 0
#define P2PVG_ACT_LRELU 1 /* LeakyReLU(0.2): models/dcgan_64.py:10,22 */
#define P2PVG_ACT_TANH 2  /* models/dcgan_64.py:45, models/lstm.py:18 */
#define P2PVG_ACT_RELU 4   /* models/h36m_mlp.py:33-41 */
#define P2PVG_ACT_SIGMOID 3 /* models/dcgan_64.py:77 (stand-alone decoder forward) */

/* 200: the sm_90a library (wgmma tensor-core kernels); p2pvg_has_tcgen05 of version 100 is now p2pvg_has_tc_gemm.
 * 201: p2pvg_conv_fusion lost its reserved backward-BatchNorm members (bwd_raw ... bwd_stat_partial, rows_per_group), and
 *      p2pvg_conv_thin_in, p2pvg_convT_thin_out, p2pvg_bn_bwd_finalize_tiles and p2pvg_bn_bwd_apply were removed. */
int p2pvg_version(void);
const char* p2pvg_last_error(void);
/* 1 when the wgmma/TMA GEMM can be used on this process' device (driver entry points resolved). */
int p2pvg_has_tc_gemm(void);
/* 0 = pick automatically (wgmma for bf16 operands), 1 = force the CUDA-core GEMM, 2 = force wgmma */
int p2pvg_set_gemm_impl(int impl);
/* p2pvg_gemm `flags` (per call; there is no process-global precision state):
 *   P2PVG_GEMM_TF32          fp32 operands MAY run on wgmma .tf32 (LSTM GEMMs of the bf16 training mode).  The
 *                            tensor-core kernel needs both operands K-major, K >= 32, 16-byte aligned bases and row
 *                            pitches (TMA); any other fp32 GEMM of such a call runs on the exact CUDA-core kernel --
 *                            a documented, precision-INCREASING dispatch between two kernels of this library (never a
 *                            CPU or vendor-library fallback).
 *   P2PVG_GEMM_TF32_REQUIRE  with P2PVG_GEMM_TF32: return P2PVG_ERR_UNSUPPORTED instead of dispatching to the
 *                            CUDA-core kernel when the operands are not TMA-compatible. */
#define P2PVG_GEMM_TF32 1
#define P2PVG_GEMM_TF32_REQUIRE 2

/* C[M,N] = (accumulate ? C : 0) + opA(A)*opB(B) + bias[n] + addend[m,n]
 *   a_mn=0: A[m*lda+k] (K-major), a_mn=1: A[k*lda+m];  b_mn=0: B[n*ldb+k], b_mn=1: B[k*ldb+n].
 * Replaces the library GEMMs behind nn.Conv2d / nn.ConvTranspose2d (models/dcgan_64.py:8,20,43,64,76 after
 * lowering), nn.Linear and nn.LSTMCell (models/lstm.py:13-17,54-57) and their autograd backward.
 * bf16 operands run on the tensor cores (wgmma, fp32 accumulation in registers); fp32 operands on CUDA cores (exact) unless
 * `flags` allows TF32 (see above).  Documented dispatch between two kernels of this library: bf16 operands whose base
 * address or row pitch is not 16-byte aligned (not expressible as a TMA tensor map) run on the CUDA-core kernel with the
 * same arithmetic contract; p2pvg_set_gemm_impl(2) turns that case into P2PVG_ERR_UNSUPPORTED.
 * workspace: split-K partials for the tensor-core path (may be NULL when ws_bytes == 0). */
int p2pvg_gemm(const void* A, int in_dtype, int a_mn, int64_t lda, const void* B, int b_mn, int64_t ldb, void* C, int c_dtype,
               int64_t ldc, int M, int N, int K, int accumulate, const float* bias, const void* addend, int64_t ldd,
               void* workspace, size_t ws_bytes, int flags, void* stream);

/* Implicit-GEMM 4x4 / stride-2 / pad-1 convolution family on NHWC bf16 tensors (TMA 4-D pixel-box loads feeding wgmma;
 * no im2col / col2im buffers).  H, W = size of the SMALL map (the big map is 2H x 2W).
 *   kind 0: c_small[N,H,W,Cn] = conv_s2(a_big[N,2H,2W,Ck]) . b[Cn,(kh,kw,Ck)] + bias       nn.Conv2d(.,.,4,2,1) forward
 *           (models/dcgan_64.py:8) and the data-gradient of nn.ConvTranspose2d(.,.,4,2,1) (models/dcgan_64.py:20)
 *   kind 1: c[Cm,(kh,kw,Cn)] = sum_pix a_small[pix,Cm]^T . gather_s2(b_big[N,2H,2W,Cn])    the weight gradients of both (fp32)
 *   kind 2: c_big[N,2H,2W,Cn] = convT_s2(a_small[N,H,W,Ck]) . b[Ck,(kh,kw,Cn)] + bias + addend[src]   ConvTranspose2d forward
 *           and the Conv2d data-gradient; `addend` (fp32, big-map layout) is the skip half of torch.cat([d, skip], 1)
 *           (models/dcgan_64.py:84-87) computed once per distinct source call; image n adds addend image
 *           grp_src[n / imgs_per_group] * imgs_per_group + n % imgs_per_group.
 * 3x3 / stride-1 / pad-1 variants for the vgg_64 layers (models/vgg_64.py:8-13), both maps H x W:
 *   kind 3: c[N,H,W,Cn] = conv3x3(a[N,H,W,Ck]) . b[Cn,(kh,kw,Ck)] + bias + addend[src]       forward; `addend` (fp32 [.,H,W,Cn])
 *           is the skip half of torch.cat([up(d), skip], 1) (models/vgg_64.py:97-104), indexed like kind 2
 *   kind 4: c[Cm,(kh,kw,Cn)] = sum_pix a[pix,Cm]^T . gather_3x3(b[N,H,W,Cn])                  weight gradient (fp32)
 *   kind 5: kind 3 with mirrored tap offsets, b = [Cin,(kh,kw,Cout)]                          data gradient
 * Returns P2PVG_ERR_UNSUPPORTED for shapes outside the pixel-box tiling (channels not a multiple of 64, ...). */
int p2pvg_conv_gemm(int kind, const void* a, const void* b, int64_t ldb, void* c, int c_dtype, int64_t ldc, int N, int H, int W, int Ck,
                    int Cn, int Cm, const float* bias, const void* addend, const int* grp_src, int imgs_per_group, int accumulate,
                    void* workspace, size_t ws_bytes, const struct p2pvg_conv_fusion* fusion, void* stream);

/* Optional epilogue fusions of p2pvg_conv_gemm (kinds 0, 2, 3, 5; `fusion` may be NULL, every member may be NULL).
 * nn.BatchNorm2d in training mode sits between every pair of convolutions (models/dcgan_64.py:9,21, models/vgg_64.py:9): its
 * batch statistics need the whole convolution output, so the producing GEMM emits them from its accumulator registers
 * instead of a separate pass over the stored tensor.
 *   fwd_stat_partial  out, float2 [pixel tile of 128 output rows x phase (kind 2: 4 output parities, else 1)][Cn]:
 *                     (sum y, sum y^2) of the tile's rows, y as stored (bf16-rounded for a bf16 output).  The tile of GEMM
 *                     row block mt and phase ph is row mt*phases + ph; reduce per group with p2pvg_bn_fwd_finalize_tiles
 *                     (rows of one BatchNorm group must be a multiple of 128).
 *   addend_dtype      the skip-half addend may be stored in bf16 (it is the output of another p2pvg_conv_gemm call).
 *   eval_scale/shift  kinds 0, 2 and 3: nn.BatchNorm2d in eval mode + activation applied in the epilogue (generation,
 *                     models/p2p_model.py:80-183 with running statistics): the stored output is
 *                     y = act(eval_scale[c] * (acc + bias[c] + addend) + eval_shift[c]), act = P2PVG_ACT_LRELU | P2PVG_ACT_TANH,
 *                     coefficients as p2pvg_bn_eval_coeffs writes them.  NULL: no such epilogue.  Not combinable with
 *                     fwd_stat_partial or accumulate (P2PVG_ERR_BAD_ARG). */
typedef struct p2pvg_conv_fusion {
  void* fwd_stat_partial;
  int addend_dtype; /* dtype of `addend`: P2PVG_F32 (default, also without a fusion struct) or P2PVG_BF16 (half the epilogue read traffic) */
  const float* eval_scale;
  const float* eval_shift;
  int act;
} p2pvg_conv_fusion_t;

/* vgg_64 data movement (models/vgg_64.py), NHWC, dtype f32 | bf16.
 *   im2col3  : col[(n,y,x), tap*C + c] = x[n, y + sgn*(kh-1), x + sgn*(kw-1), c], row pitch ld >= 9C (pad columns zeroed);
 *              explicit lowering of nn.Conv2d(.,.,3,1,1) (models/vgg_64.py:9) for the fp32 path and the 3-channel ends
 *   col2im3  : y[(n,y,x), c] = bias[c] + sum_tap col[(n, y-(kh-1), x-(kw-1)), tap*C + c]   nn.ConvTranspose2d(64,nc,3,1,1)
 *              (models/vgg_64.py:88) after the [pix,64] x [64,9*nc] GEMM
 *   maxpool2 : nn.MaxPool2d(2,2) (models/vgg_64.py:47) forward / backward (first maximum in row-major order takes the gradient)
 *   upsample2: nn.UpsamplingNearest2d(scale_factor=2) (models/vgg_64.py:91) forward / backward
 *   gather_add: dst[g] += src_f32[grp_src[g]] over chunks of n elements (skip-half addend, explicit path). */
int p2pvg_im2col3(const void* x, void* col, int dtype, int N, int H, int W, int C, int ld, int sgn, void* stream);
int p2pvg_col2im3(const void* col, void* y, int dtype, int N, int H, int W, int C, int ld, const float* bias, void* stream);
int p2pvg_maxpool2_fwd(const void* x, void* y, int dtype, int N, int H, int W, int C, void* stream);
int p2pvg_maxpool2_bwd(const void* x, const void* dy, void* dx, int dtype, int N, int H, int W, int C, void* stream);
int p2pvg_upsample2_fwd(const void* x, void* y, int dtype, int N, int H, int W, int C, void* stream);
int p2pvg_upsample2_bwd(const void* dy, void* dx, int dtype, int N, int H, int W, int C, void* stream);
int p2pvg_gather_add(void* dst, int dtype, const float* src, const int* grp_src, int G, int64_t n, void* stream);

/* The two thin ends of the vgg stacks in eval mode (generation), each one launch on the CUDA cores.  Both read the fp32
 * parameters in PyTorch's own layout, in place, and accumulate in fp32 FFMA in a fixed order (first: input channel, kh, kw;
 * last: kh, kw, input channel); the activations are stored in `dtype` (f32 | bf16), rounded once.  nc = 1..4 image channels (else P2PVG_ERR_UNSUPPORTED).
 *   vgg_first_eval: the first encoder layer vgg_layer(nc, 64) (models/vgg_64.py:22) with BatchNorm on running statistics:
 *                   y[N,H,W,64] (NHWC) = LeakyReLU_0.2(scale[c] * (conv3x3_p1(x)[c] + bias[c]) + shift[c]) from fp32 NCHW frames
 *                   x[N,nc,H,W]; w = Conv2d weight [64][nc][3][3], scale / shift as p2pvg_bn_eval_coeffs writes them.
 *   vgg_last_eval:  the closing ConvTranspose2d(64, nc, 3, 1, 1) + Sigmoid (models/vgg_64.py:87-90):
 *                   out[n,c,y,x] (fp32 NCHW) = sigmoid(bias[c] + sum_{ci,kh,kw} d[n, y+1-kh, x+1-kw, ci] * w[ci][c][kh][kw]) from
 *                   d[N,H,W,64] (NHWC); w = ConvTranspose2d weight [64][nc][3][3].
 * P2PVG_ERR_BAD_ARG: NULL pointers, N < 0, H or W < 1, a y / d base that is not 16-byte aligned. */
int p2pvg_vgg_first_eval(const float* x, int nc, const float* w, const float* bias, const float* scale, const float* shift, void* y,
                         int y_dtype, int N, int H, int W, void* stream);
int p2pvg_vgg_last_eval(const void* d, int d_dtype, const float* w, const float* bias, float* out, int nc, int N, int H, int W,
                        void* stream);

/* 4x4 / stride 2 / pad 1 lowering (nn.Conv2d(nin,nout,4,2,1), models/dcgan_64.py:8; and the data-gradient of
 * nn.ConvTranspose2d(nin,nout,4,2,1), models/dcgan_64.py:20): x [N,H,W,C] -> col [N*H/2*W/2, 16*C], K order (kh,kw,c). */
int p2pvg_im2col_k4s2p1(const void* x, void* col, int dtype, int N, int H, int W, int C, void* stream);
/* Inverse gather (ConvTranspose2d forward after the GEMM, Conv2d data-gradient): y [N,2Hi,2Wi,C] from
 * col [N*Hi*Wi,16*C]; optional second operand col2 holds the skip-connection half of torch.cat([d, skip], 1)
 * (models/dcgan_64.py:84-87) computed once per distinct source call: image n reads col2 image
 * grp_src[n / imgs_per_group]*imgs_per_group + n % imgs_per_group. */
int p2pvg_col2im_k4s2p1(const void* col, const void* col2, const int* grp_src, int imgs_per_group, void* y, int dtype, int N,
                        int Hi, int Wi, int C, const float* bias, int accumulate, void* stream);
/* dst (contiguous, dims[4]) = src gathered with per-destination-dimension strides (weight packing, NCHW->NHWC, casts). */
int p2pvg_permute4(const void* src, int src_dtype, void* dst, int dst_dtype, const int* dims /*host*/,
                   const int64_t* src_strides /*host*/, int accumulate, void* stream);
/* Frames x [N, C, H*W] fp32 (the layout the data loaders hand to P2PModel.forward, models/p2p_model.py:185-197) -> channels-last
 * [N, H*W, C], written once in fp32 (dst_f32: the MSE target, may be NULL) and once in the activation dtype (dst_act: input
 * of the first convolution, may be NULL) from a single read.  C in {2,3,4}, H*W % 4 == 0; one-channel frames need no
 * conversion (NCHW == NHWC). */
int p2pvg_nchw_to_nhwc_dual(const float* src, float* dst_f32, void* dst_act, int act_dtype, int64_t N, int hw, int C, void* stream);
int p2pvg_add_indexed(void* dst, const void* src, int dtype, const int* dst_idx, int F, int64_t n, void* stream);
int p2pvg_group_sum(const void* in, void* out, int dtype, const int* grp_src, int G, int F, int64_t n, void* stream);
/* dst[a][q][p] = src[a][p][q] for a < A (tiled, coalesced both ways): nn.Conv2d / nn.ConvTranspose2d weights
 * [A][B][kh*kw] -> the GEMM layout [A][(kh,kw)][B] (models/dcgan_64.py:8,20) and the weight gradients back. */
int p2pvg_transpose_batched(const void* src, int src_dtype, void* dst, int dst_dtype, int A, int P, int Q, void* stream);
/* dst[g*R, g*C] = blockdiag(src[R, C], ..., src[R, C]): lets the 1/3-channel ends of the conv stacks (K = 16*nc or N = 16*nc,
 * models/dcgan_64.py:34,76) run as [M/g, g*C] GEMMs whose TMA boxes are never out of bounds. */
int p2pvg_blockdiag(const void* src, int src_dtype, void* dst, int dst_dtype, int R, int C, int g, void* stream);

/* nn.BatchNorm2d in training mode (models/dcgan_64.py:9,21,44,65), statistics per group. */
size_t p2pvg_bn_workspace_bytes(int G, int C);
int p2pvg_bn_fwd_stats(const void* x, int dtype, int G, int64_t R, int C, const float* gamma, const float* beta, float eps,
                       void* ws, size_t ws_bytes, float* mean, float* invstd, float* var_unbiased, float* scale, float* shift,
                       void* stream);
int p2pvg_bn_act(const void* x, void* y, int dtype, const float* scale, const float* shift, int G, int64_t R, int C, int act,
                 void* stream);
/* y may be NULL for LeakyReLU: the activation derivative is then recomputed from sign(x*scale+shift) (saves one read of y). */
int p2pvg_bn_bwd(const void* dy, const void* x, const void* y, int dtype, const float* mean, const float* invstd,
                 const float* gamma, int G, int64_t R, int C, int act, void* ws, size_t ws_bytes, void* dx, float* sum_dz,
                 float* sum_dzx, const float* scale, const float* shift, void* stream);
/* p2pvg_bn_bwd for bf16 activations and LeakyReLU (y omitted: the slope comes from sign(x*scale+shift)), whose apply pass
 * also writes dx_sum[f] = sum over the groups g with grp_src[g] == f of dx[g] (f < F; R*C bf16 elements each), summed in
 * fp32 in increasing g and rounded once: bit-identical to p2pvg_group_sum of the dx that p2pvg_bn_bwd writes.  A source
 * no group maps to comes out as zeros; a group whose grp_src is outside [0, F) is left untouched.  dx may alias dy.
 * dout != NULL (C = 64): the layer's output y = bf16(lrelu(x*scale+shift)) feeds a 4x4 / stride-2 / pad-1 ConvTranspose2d(64,
 * 1) whose output-map gradient is dout [G * R / Ho^2][2 Ho][2 Ho] (bf16, Ho a power of two); the reduce pass then also writes that
 * convolution's weight gradient dw[c][kh * 4 + kw] = sum over rows of y[c] * dout[tap] (the [64][tap] packed layout),
 * through wpart as p2pvg_bn_bwd_wgrad_c1 does.  dout == NULL: Ho, wpart, wpart_bytes and dw are ignored. */
int p2pvg_bn_bwd_group_sum(const void* dy, const void* x, const float* mean, const float* invstd, const float* gamma, int G,
                           int64_t R, int C, void* ws, size_t ws_bytes, void* dx, float* sum_dz, float* sum_dzx,
                           const float* scale, const float* shift, const int* grp_src, int F, void* dx_sum, const void* dout,
                           int Ho, float* wpart, size_t wpart_bytes, float* dw, void* stream);
/* p2pvg_bn_bwd for bf16 activations, LeakyReLU (y omitted) and C = 64, where x is the output of a 4x4 / stride-2 / pad-1
 * convolution of the 1-channel bf16 map cin [G * R / Ho^2][2 Ho][2 Ho] (R = rows per group = images per group * Ho^2,
 * Ho a power of two).
 * dx is not stored: its weight gradient dw[c][kh * 4 + kw] = sum over rows of bf16(dx[c]) * cin[tap] (PyTorch's
 * [64][1][4][4] layout) is written instead, accumulated in fp32 per block into wpart (p2pvg_bn_wgrad_c1_partial_bytes(G)
 * bytes) and combined in fp64 in a fixed order (deterministic). */
size_t p2pvg_bn_wgrad_c1_partial_bytes(int G);
int p2pvg_bn_bwd_wgrad_c1(const void* dy, const void* x, const float* mean, const float* invstd, const float* gamma, int G,
                          int64_t R, void* ws, size_t ws_bytes, float* sum_dz, float* sum_dzx, const float* scale,
                          const float* shift, const void* cin, int Ho, float* wpart, size_t wpart_bytes, float* dw,
                          void* stream);
/* The forward statistics when their per-tile column sums were produced by a GEMM epilogue (p2pvg_conv_fusion):
 * partial is float2 [G * parts_per_group][ldp]; channel c of group g sums the group's partial rows over the `fold` column
 * groups f*C + c (a GEMM row may hold several pixels / filter taps of one channel).  R = elements per (group, channel).
 * fp64 combine in a fixed order (deterministic).  Replaces the statistics pass of nn.BatchNorm2d (models/dcgan_64.py:9). */
int p2pvg_bn_fwd_finalize_tiles(const void* partial, int parts_per_group, int ldp, int fold, int G, int64_t R, int C,
                                const float* gamma, const float* beta, float eps, float* mean, float* invstd, float* var_unbiased,
                                float* scale, float* shift, void* stream);
/* eval-mode BatchNorm (running statistics; generate.py / p2p_generate): scale = gamma/sqrt(rvar+eps), shift = beta-rmean*scale */
int p2pvg_bn_eval_coeffs(const float* gamma, const float* beta, const float* rmean, const float* rvar, float eps, int C,
                         float* scale, float* shift, void* stream);
int p2pvg_bn_param_grad(const float* sum_dz, const float* sum_dzx, int G, int C, float* dgamma, float* dbeta, void* stream);
/* running_mean / running_var EMA applied call by call in the reference's call order (SURVEY.md A.3 item 7). */
int p2pvg_bn_ema(float* rmean, float* rvar, const float* mean, const float* var_unbiased, const int* order, int ncalls, int C,
                 float momentum, void* stream);

/* nn.LSTMCell pointwise part (models/lstm.py:41,89): gates [B,4R] in: pre-activations (i,f,g,o), out: activations. */
int p2pvg_lstm_pointwise_fwd(float* gates, const float* c_prev, float* c_out, float* h_out, int B, int R, void* stream);
int p2pvg_lstm_pointwise_bwd(const float* dh, const float* dc_next, const float* gates, const float* c_prev, const float* c,
                             float* dgates, float* dc_prev, int B, int R, void* stream);
/* Whole-sequence recurrence of one nn.LSTMCell layer in ONE persistent launch (the W_hh slice of a CTA stays on chip for all
 * timesteps).  tf32 = 1 dispatches by hidden size: R in {64,128,256}: thread-block clusters of 8 CTAs, slabs of 16 batch rows per
 * cluster (32 above 128 rows), hardware cluster barrier per timestep; R = 512: clusters of 16 CTAs (non-portable size), forward slabs of 16 / 32 / 48 batch rows per cluster chosen so that
 * the resident clusters cover the batch in as few waves as possible, backward in 16-row slabs with the reduction scattered through
 * distributed shared memory; the part of the weight slice that does not fit the registers lives in shared memory.  tf32 = 0:
 * cooperative grid with a grid barrier per timestep, exact fp32 FFMA products.
 *   forward : gates_s = pre_s + b_hh + h_{s-1}.W_hh^T -> (i,f,g,o) -> c_s, h_s       pre [S,B,4R] = x-part incl. b_ih
 *             gates [S,B,4R] out (activations), hs / cs [S+1,B,R] with slot 0 = initial state (zeros, models/lstm.py:21-27)
 *   backward: dh_s = dhtop_s + dG_{s+1}.W_hh, cell backward -> dG [S,B,4R] (gradient w.r.t. the gate pre-activations)
 * `counter` is a zero-initialised uint32 in device memory (the grid barrier of the cooperative variant); R %% 64 == 0, R <= 256, or
 * R = 512 (tf32 = 1: any batch; tf32 = 0: as long as the cooperative grid fits).  Unsupported shapes return P2PVG_ERR_UNSUPPORTED.
 * tf32 = 1: the recurrent products on the tensor cores (mma.sync m16n8k8 tf32, fp32 accumulation). */
int p2pvg_lstm_scan_fwd(const float* pre, const float* whh, const float* bhh, float* gates, float* hs, float* cs, int S, int B, int R,
                        int tf32, unsigned* counter, void* stream);
int p2pvg_lstm_scan_bwd(const float* dhtop, const float* whh, const float* gates, const float* cs, float* dG, int S, int B, int R,
                        int tf32, unsigned* counter, void* stream);
/* diagnostics: cudaOccupancyMaxActiveClusters of the hidden-size-512 scans (clusters of 16 CTAs): which = 0 / 1 / 3 forward with
 * 16- / 32- / 48-row slabs; any other value the backward scan (its only instance, 16-row slabs); -1 on error */
int p2pvg_lstm_cluster512_max_clusters(int which);
/* the same for the hidden-size-256 scans (clusters of 8 CTAs): which = 0 / 1 forward with 16- / 32-row slabs, 2 / 3 backward */
int p2pvg_lstm_cluster_max_clusters(int which);
/* One timestep of one or two stand-alone LSTM modules in ONE launch (models/lstm.py:29-44 `lstm`, :83-94 `gaussian_lstm`):
 * embed Linear -> `layers` x nn.LSTMCell -> head.  Generation runs posterior + prior as one launch and the frame predictor as a
 * second.  Clusters of 8 CTAs, each CTA owning R/8 hidden units of every layer, one cluster per slab of 8 batch rows; stage
 * outputs are exchanged through distributed shared memory; weights stream from L2; exact fp32 FFMA.  R in 64..512 (multiple
 * of 8), any layer count, any row count.
 *   input row b  = [ seg_a[idx_a[0]*rows + b, 0:ga] | seg_b[idx_b[0]*rows + b, 0:gb] | tuc[0] | dt[0] ]  (the torch.cat of
 *                  models/p2p_model.py:150-179, never materialised; idx_a / idx_b / tuc / dt are device pointers read at run time)
 *   layer_w      device array [layers][4] of device pointers: weight_ih [4R][R], bias_ih [4R], weight_hh [4R][R], bias_hh [4R]
 *   state        device array [layers][4] of device pointers: h_in, c_in, h_out, c_out, each [rows][R] fp32 (h_out == h_in and
 *                c_out == c_in is allowed: the state may be updated in place)
 *   head         P2PVG_LSTM_HEAD_LINEAR_TANH: out[rows][out_dim] = tanh(h W_out^T + b_out)
 *                P2PVG_LSTM_HEAD_GAUSSIAN:    mu = h W_out^T + b_out, logvar = h W_out2^T + b_out2, out = eps * exp(logvar / 2) + mu
 *                                             (mu / logvar written when non-NULL)
 *   counter_rows 0: tuc[0] and dt[0] are the time counters of every row; > 0: row b reads tuc[b / counter_rows] and
 *                dt[b / counter_rows] (groups of counter_rows rows, e.g. one output length each); negative: P2PVG_ERR_BAD_ARG  */
#define P2PVG_LSTM_HEAD_LINEAR_TANH 0
#define P2PVG_LSTM_HEAD_GAUSSIAN 1
typedef struct p2pvg_lstm_step_module {
  const float* seg_a;
  const int* idx_a;
  int ga;
  const float* seg_b;
  const int* idx_b;
  int gb;
  const float* tuc;
  const float* dt;
  const float* w_embed;
  const float* b_embed;
  int layers;
  const float* const* layer_w;
  float* const* state;
  int head;
  int out_dim;
  const float* w_out;
  const float* b_out;
  const float* w_out2;
  const float* b_out2;
  const float* eps;
  float* out;
  float* mu;
  float* logvar;
  int counter_rows;
} p2pvg_lstm_step_module;
int p2pvg_lstm_step(const p2pvg_lstm_step_module* modules /*host array*/, int n_modules, int rows, int R, void* stream);
/* One whole call of the h36m pose encoder or decoder (models/h36m_mlp.py:28-95; no BatchNorm, so eval == train) in ONE launch.
 *   residual_linear(nin, nout):  LayerNorm(relu(shortcut(x)) + relu(L3(relu(L2(relu(L1(x))))))), long-path width nin / 2,
 *                                LayerNorm eps 1e-5 (the nn.LayerNorm default)
 *   encoder (decoder = 0): fc1 = residual_linear(51, g), fc2 = residual_linear(g, g), out = tanh(fc3(h2)) [rows][g];
 *                          h1 / h2 [rows][g] (the skips) written when non-NULL
 *   decoder (decoder = 1): d1 = fc1(x) with fc1 = residual_linear(g, g), d2 = fc2([d1 | skip2]) with residual_linear(2g, g),
 *                          out = fc3([d2 | skip1]) [rows][51] (Linear 2g -> 51, no activation); output row r reads skip row
 *                          r % nsrc of skip1 / skip2 [nsrc][g] (skips encoded at B rows shared by nsample * B rows)
 *   input row b = src[(src_idx[0] * rows + b) * in_dim + 0 : in_dim] (in_dim 51 / g; src_idx is a device pointer read at run time,
 *                 NULL = frame 0)
 * Clusters of 8 CTAs per slab of 8 rows, each CTA owning 1/8 of every Linear's output units (uneven for 25 / 51); stage outputs
 * are pushed to every CTA of the cluster through distributed shared memory; weights stream from L2; exact fp32 FFMA.
 * P2PVG_ERR_BAD_ARG: NULL pointers, g < 8, nsrc < 1.  P2PVG_ERR_UNSUPPORTED: the slab does not fit in shared memory. */
typedef struct p2pvg_pose_residual {
  const float* w_sc;   /* shortcut Linear [nout][nin], bias [nout] */
  const float* b_sc;
  const float* w1;     /* long path: [nin/2][nin], [nin/2][nin/2], [nout][nin/2] and their biases */
  const float* b1;
  const float* w2;
  const float* b2;
  const float* w3;
  const float* b3;
  const float* gamma;  /* LayerNorm(nout) */
  const float* beta;
} p2pvg_pose_residual;
typedef struct p2pvg_pose_mlp_args {
  int decoder;
  int g;
  const float* src;
  const int* src_idx;
  p2pvg_pose_residual fc1;
  p2pvg_pose_residual fc2;
  const float* w3;     /* fc3: encoder [g][g], decoder [51][2g] */
  const float* b3;
  const float* skip1;  /* decoder only */
  const float* skip2;
  int nsrc;
  float* out;
  float* h1;           /* encoder only */
  float* h2;
} p2pvg_pose_mlp_args;
int p2pvg_pose_mlp(const p2pvg_pose_mlp_args* args /*host*/, int rows, void* stream);
/* gaussian_lstm.reparameterize (models/lstm.py:76-81) for posterior and prior + KLCriterion.forward
 * (misc/criterion.py:10-15) summed over all elements (division by opt.batch_size happens in finalize_losses). */
int p2pvg_reparam_kl_fwd(const float* mu, const float* lv, const float* mu_p, const float* lv_p, const float* eps,
                         const float* eps_p, float* z, float* z_p, int n, float* kl_sum, void* stream);
int p2pvg_reparam_kl_bwd(const float* mu, const float* lv, const float* mu_p, const float* lv_p, const float* eps,
                         const float* eps_p, const float* dz, const float* dz_p, float kl_coef, float* dmu, float* dlv,
                         float* dmu_p, float* dlv_p, int n, void* stream);
/* torch.cat([h, global_z | z, time_until_cp, delta_time], 1) (models/p2p_model.py:241-242,247,252) for all steps. */
int p2pvg_build_concat(float* dst, const float* A, const int* ia, int ga, const float* Bm, const int* ib, int gb,
                       const float* tuc, const float* dt, int S, int B, int ld /* row pitch >= ga+gb+2, zero padded */, void* stream);
int p2pvg_gather_add_cols(float* dst, const float* src, const int* idx, int S, int T, int B, int g, int W, int col0, int init,
                          void* stream);
/* align_loss += MSE(h[0], h_pred) with h[0] = batch row 0 broadcast (models/p2p_model.py:224-225), value + gradients. */
int p2pvg_align(const float* H, const int* in_idx, const float* h_pred, int P, int B, int g, float coef, float* loss_partial,
                float* d_hpred, float* dH, void* stream);
/* out[c] (+)= sum_r x[r*ld + c] — bias gradients. */
int p2pvg_colsum(const void* x, int dtype, int64_t rows, int cols, int64_t ld, float* out, int accumulate, void* ws /* >= 1024*cols floats */,
                 size_t ws_bytes, void* stream);
int p2pvg_act_fwd(float* x, int64_t n, int act, void* stream);
/* dx = dy * act'(x), the derivative taken from the forward output y = act(x) (in place: x == y). */
int p2pvg_act_bwd(const float* dy, const float* y, float* dx, int64_t n, int act, void* stream);

/* nn.Sigmoid (models/dcgan_64.py:77) + nn.MSELoss (models/p2p_model.py:254,256): per-group sum of squared error
 * partials [G, p2pvg_mse_chunks()] and d(loss)/d(raw) = coef[g]*2*(s-x)*s*(1-s). */
int p2pvg_mse_chunks(void);
int p2pvg_sigmoid_mse(const void* raw, int dtype, const float* x, const int* tgt, const float* coef, int G, int64_t E,
                      void* pred, void* d_raw, float* partial, void* stream);
/* The last decoder layer of the dcgan stacks (C = 1 or 3 image channels) fused with its loss: ConvTranspose2d(2*64, C, 4, 2, 1) +
 * nn.Sigmoid (models/dcgan_64.py:75-79, models/dcgan_128.py:82-84) + nn.MSELoss against frame tgt[g] (models/p2p_model.py:254,256).
 * col [G*B*Hi*Wi, 16*C] / col2 [nsrc*B*Hi*Wi, 16*C]: the 16 tap products (x C channels) of every input pixel of the decoder half /
 * of the shared skip half (group g uses skip source grp_src[g]), as produced by p2pvg_gemm.  Writes d(loss)/d(raw)
 * [G, B*2Hi*2Wi*C] (NHWC) and the squared-error partials [G, p2pvg_mse_chunks()]; the raw output is never materialised. */
int p2pvg_convt_c1_loss(const void* col, const void* col2, int dtype, const int* grp_src, const float* bias, const float* x, const int* tgt,
                        const float* coef, int G, int B, int Hi, int Wi, int C, void* d_raw, float* partial, void* stream);
/* h36m pose backbone (models/h36m_mlp.py): nn.LayerNorm of residual_linear (:43,46) forward / backward (fp32, row-wise; dx may alias
 * dy; dgamma == NULL skips the parameter gradients) and the plain nn.MSELoss on [B,17,3] poses (models/p2p_model.py:254,256) with
 * the same partial-sum layout as p2pvg_sigmoid_mse. */
int p2pvg_layernorm_fwd(const float* x, const float* gamma, const float* beta, float* y, float* mean, float* rstd, int64_t rows, int C,
                        float eps, void* stream);
int p2pvg_layernorm_bwd(const float* dy, const float* x, const float* mean, const float* rstd, const float* gamma, float* dx,
                        float* dgamma, float* dbeta, int64_t rows, int C, void* ws, size_t ws_bytes, void* stream);
int p2pvg_mse_plain(const float* pred, const float* x, const int* tgt, const float* coef, int G, int64_t E, float* d_pred, float* partial,
                    void* stream);
/* the four scalars returned by P2PModel.forward (models/p2p_model.py:271): out[0..3] = mse,kld,cpc,align (/seq_len). */
int p2pvg_finalize_losses(const float* mse_partial, int n_recon, int has_cpc, double E, const float* kl_sum, float batch_size,
                          const float* align_partial, int n_align, float seq_len, float* out, void* stream);
/* Held-out scoring (P2PModel.p2p_losses): the four terms of P2PModel.forward's objective (models/p2p_model.py:224-257, /seq_len)
 * split by batch row, from the buffers of an eval-mode forward with S executed steps and G = S + 1 decodes.
 *   rec        [G][B][E] decoded frames (dtype P2PVG_F32 / P2PVG_BF16; pre-sigmoid when sigmoid != 0), decode S = the CPC decode
 *   x          [T][B][E] fp32 targets in the same element order; decode s is scored against x[tgt[s]] (tgt[S] = T - 1)
 *   mu, lv, mu_p, lv_p  [S][B][z] fp32 posterior / prior heads;  H [T][B][g] fp32 latents;  h_pred [G][B][g] fp32
 *   in_idx     [>= S - 1]: step s < S - 1 adds MSE(H[in_idx[s]][0] broadcast, h_pred[s]) (the reference's h[0] quirk)
 *   partial    [G * B][3] fp64 workspace;  counter: one uint32, zero before the first launch and left zero by every launch
 *   per_seq    [4][B] fp64: row b's mse, kld, cpc, align -- element means over row b (kld: its KL sum / batch_size), / seq_len
 *   out        [4] fp64: mse, cpc, align = the row means of per_seq, kld = its row sum (the values forward returns)
 * Fixed-order fp64 sums, no float atomics: repeated launches on the same data are bit-identical.  E: 1..4 image channels
 * at any size, or 51 for [17, 3] poses.  One launch; streams rec and the scored frames of x once. */
int p2pvg_seq_losses(const void* rec, int dtype, int sigmoid, const float* x, const int* tgt, int S, int B, int64_t E,
                     const float* mu, const float* lv, const float* mu_p, const float* lv_p, int z, const float* H,
                     const int* in_idx, const float* h_pred, int g, int has_cpc, double batch_size, double seq_len,
                     double* partial, uint32_t* counter, double* per_seq, double* out, void* stream);
/* Early read-back of the step's scalars (models/p2p_model.py:271 returns them as host numbers: `mse.data.cpu().numpy()`): the
 * kernel stores src[0..n) and then *seq into page-locked, device-mapped host memory host_mapped[0..n] (n floats + one int);
 * the host polls host_mapped[n] for the sequence number it wrote to *seq before launching.  The values are final once the
 * forward pass is done, so the caller gets them while the backward passes and the optimiser of the same step still run;
 * everything else stays stream-ordered.  n <= 64. */
int p2pvg_publish_scalars(const float* src, int n, float* host_mapped, const int* seq, void* stream);
/* optim.Adam.step of PyTorch 1.0 (README.md:62; models/p2p_model.py:273-280) on a flat parameter arena. */
int p2pvg_adam_legacy(float* p, const float* g, float* m, float* v, int64_t n, double lr, double beta1, double beta2,
                      double eps, const int* step_ptr, void* stream);
int p2pvg_scale(float* x, int64_t n, float a, void* stream);

/* Moving MNIST training batches (DynamicLengthMovingMNIST.__getitem__, data/moving_mnist.py:51-105) rendered on the device.
 *   digits [n_digits][32][32] uint8 (MNIST resized to 32 x 32), converted to fp32 as u / 255 (ToTensor)
 *   draws  [B][num_digits][draw_stride] int32: the values every np.random.randint(lo, hi) call of (sequence b, digit n) returns,
 *          in the reference's call order (digit index, sx, sy, dx, dy, then up to four per step at the wall bounces), taken as
 *          lo + r % (hi - lo); draw_stride >= 5 + 4T
 *   out    [T][B][1][S][S] fp32, time-major (the generator's permute(1, 0, 2, 3, 4)[:T]); 16-byte aligned
 * Each frame is the fp32 sum of the digits in digit order, clipped at 1 (x[x > 1] = 1): bit-identical to the reference for the
 * same draws.  T frames of a max_seq_len sequence are its first T frames (later draws do not change earlier frames).
 * P2PVG_ERR_BAD_ARG: S < 33 or S % 4 != 0, num_digits outside 1..4, draw_stride < 5 + 4T, NULL pointers, n_digits < 1.
 * P2PVG_ERR_UNSUPPORTED: num_digits * (1024 + 5 + 4T) * 4 bytes of draws and digits exceed 48 KB of shared memory. */
int p2pvg_moving_mnist(const uint8_t* digits, int n_digits, const int32_t* draws, int draw_stride, float* out, int T, int B, int S,
                       int num_digits, int deterministic, void* stream);

/* Video training batches cut from a device-resident uint8 clip store: the windows WeizmannDataset.__getitem__
 * (data/weizmann.py:103-114) and BairRobotPush.get_seq (data/bair.py:51-75) return, time-major and truncated to T frames.
 *   frames     [F][C][H][W] uint8, 4-byte aligned; clip c is frames[clip_first[c] .. clip_first[c] + clip_len[c])
 *   entries    [B] int32: paired_flips = 1: entry e is clip e >> 1, mirrored left-right when e is odd (the reference appends
 *              each clip, then its RandomHorizontalFlip(p=1) copy); paired_flips = 0: entry e is clip e, never mirrored
 *   draws      [B] int32 or NULL: row b's window starts at (unsigned)draws[b] % (clip_len - L + 1), i.e.
 *              np.random.randint(0, n_frames - L + 1) as lo + r % (hi - lo); NULL: every window starts at frame 0
 *   out        [T][B][C][H][W] fp32, 16-byte aligned: out[t, b, c, y, x] = frames[first + start + t][c][y][x'] / 255 (ToTensor,
 *              correctly rounded), x' = W - 1 - x for a mirrored entry.  T <= L: the first T frames of the L-frame window.
 * Precondition (not checked on the device): every entry lies in [0, n_clips * (paired_flips ? 2 : 1)) and every clip an entry
 * names has clip_len >= L; p2pvg_b200.data.ClipBatches builds entries and draws that way.
 * P2PVG_ERR_BAD_ARG: NULL frames / clip tables / entries / out, misaligned frames or out, n_clips < 1, B < 0, T < 0, T > L,
 * L < 1, C < 1, H < 1, W % 4 != 0 or W < 4.  P2PVG_ERR_UNSUPPORTED: C * H * W > 2^30 or T * B >= 2^31. */
int p2pvg_video_windows(const uint8_t* frames, const int64_t* clip_first, const int32_t* clip_len, int n_clips,
                        const int32_t* entries, const int32_t* draws, int paired_flips, int B, int L, int T, int C, int H, int W,
                        float* out, void* stream);

/* Human3.6M training batches gathered from device-resident pose stores: the windows Human36mDataset.__getitem__
 * (data/human36m/human36m.py:67-107, constant-speed branch) returns, time-major and truncated to T frames, for both outputs in
 * one launch.
 *   pose2d     [F][J][2] fp32, pose3d [F][J][3] fp32: sequence s is frames seq_first[s] .. seq_first[s] + seq_len[s) of both
 *   entries    [B] int32: the sequence of batch row b
 *   draws      [2][B] int32: row b starts at start = (unsigned)draws[b] % (seq_len[e] - speed_hi * L + 1) and steps by
 *              speed = speed_lo + (unsigned)draws[B + b] % (speed_hi - speed_lo + 1), i.e. the reference's
 *              np.random.randint(lo, hi) calls as lo + r % (hi - lo)
 *   out2d      [T][B][J][2] fp32, out3d [T][B][J][3] fp32: out[t, b] = pose[seq_first[e] + start + t * speed], a copy of the
 *              store's values.  T <= L: the first T frames of the L-frame window.
 * Precondition (not checked on the device): every entry lies in [0, n_seq) and every sequence an entry names has
 * seq_len >= speed_hi * L; p2pvg_b200.data.PoseClips and PoseBatches build stores, entries and draws that way.
 * P2PVG_ERR_BAD_ARG: NULL or misaligned pointers (fp32 / int32 4-byte, seq_first 8-byte), n_seq < 1, J < 1, B < 0, T < 0,
 * T > L, L < 1, speed_lo < 1, speed_lo > speed_hi.  P2PVG_ERR_UNSUPPORTED: speed_hi * L >= 2^31 or T * B * J * 5 >= 2^31. */
int p2pvg_pose_windows(const float* pose2d, const float* pose3d, int J, const int64_t* seq_first, const int32_t* seq_len, int n_seq,
                       const int32_t* entries, const int32_t* draws, int B, int speed_lo, int speed_hi, int L, int T, float* out2d,
                       float* out3d, void* stream);

/* Scores of generated frames against ground-truth frames, one result row per pair.
 *   pred       [N][C][H][W] fp32, 16-byte aligned; gt [M][C][H][W] fp32, 16-byte aligned
 *   pairs      [n_pairs][2] int32, 4-byte aligned: pair p scores pred frame pairs[p][0] against gt frame pairs[p][1]
 *   out        [n_pairs][3] fp64, 8-byte aligned: mse, psnr, ssim of each pair, with R = data_range:
 *              mse  = sum (P - G)^2 / (C H W)
 *              psnr = 10 log10(R^2 / mse), +inf when mse == 0
 *              ssim = the mean over channels of the mean of S over the (H - 6)(W - 6) 7x7 windows inside the frame, with
 *                     window means ux, uy, sample (ddof 1) variances vx, vy and covariance vxy,
 *                     S = (2 ux uy + C1)(2 vxy + C2) / ((ux^2 + uy^2 + C1)(vx + vy + C2)), C1 = (0.01 R)^2, C2 = (0.03 R)^2
 *                     (skimage.metrics.structural_similarity at its defaults, data_range = R, channels averaged)
 * One pass: each element of a pair's two frames is read once; per-pixel arithmetic is fp32, the per-pair sums fp64 in a
 * fixed order, so a pair's row is bit-identical whichever other pairs share the launch.  Pairs that share a gt frame are
 * best placed next to each other: the repeats of that frame are then served from L2.
 * Precondition (not checked on the device): 0 <= pairs[p][0] < N and 0 <= pairs[p][1] < M; p2pvg_b200.metrics checks it.
 * n_pairs == 0 returns P2PVG_OK without a launch (pairs and out may then be NULL, as empty arrays' storage often is).
 * P2PVG_ERR_BAD_ARG: NULL or misaligned pointers, C < 1, H < 7, W < 8, W % 4 != 0, n_pairs < 0, data_range not finite and
 * positive.  P2PVG_ERR_UNSUPPORTED: W > 128 (the width the shared-memory tiles cover) or C * H * W >= 2^31. */
int p2pvg_frame_metrics(const float* pred, const float* gt, const int32_t* pairs, int n_pairs, int C, int H, int W,
                        float data_range, double* out, void* stream);

/* Scores of generated poses against ground-truth poses, one result row per pair.
 *   pred [N][J][3] fp32, gt [M][J][3] fp32 (4-byte aligned); pairs [n_pairs][2] int32 (4-byte aligned) as for
 *   p2pvg_frame_metrics; out [n_pairs][2] fp64 (8-byte aligned): mse = the mean of the 3J squared differences,
 *   mpjpe = (1/J) sum_j ||P_j - G_j||_2.  fp64 throughout, a fixed summation order.
 * Precondition (not checked on the device): pair indices in range.  n_pairs == 0 returns P2PVG_OK without a launch (pairs
 * and out may then be NULL).
 * P2PVG_ERR_BAD_ARG: NULL or misaligned pointers, J < 1, n_pairs < 0. */
int p2pvg_pose_metrics(const float* pred, const float* gt, const int32_t* pairs, int n_pairs, int J, double* out, void* stream);

/* One batch's scores folded into split-level totals (p2pvg_b200.evaluate.evaluate_split), in one launch.
 *   scores     [n_pairs][n_metrics] fp64: what p2pvg_frame_metrics / p2pvg_pose_metrics wrote for the pairs of the segments
 *   higher_mask bit m set: a higher value of metric m is better (psnr, ssim); clear: lower is better (mse, mpjpe)
 *   segs       [n_seg][3] int32, device: per segment (one output length of the batch) its first pair off, its first column c0
 *              and its scored frame count F; pair (frame j, row b, sample s) of the segment is off + (j * B + b) * nsample + s
 *              and frame j is column c0 + j
 *   col_bin    [n_cols] int32, device: the bin of every column; a bin is one (output length, scored frame) of the split
 *   part_v     [n_cols][B][n_metrics][2] fp64 and part_c [n_cols][B][n_metrics][2] int32: workspace
 *   counter    one uint32, zero before the first launch and left zero by every launch
 *   sums       [n_bins][n_metrics][3] fp64, += per bin: the sum over rows of the best sample's finite value, the sum of its
 *              squares, and the sum over rows and samples of the finite values
 *   counts     [n_bins][n_metrics][4] uint64, += per bin: the best sample's +-inf values, its NaN values, and the +-inf and
 *              NaN values over all samples (none of them is in sums)
 *   rows       [n_bins] uint64, += the rows folded into each bin
 * Best sample, per segment, row and metric: the best mean over the segment's F frames (frames summed in order, then / F),
 * the first sample on ties, and the first NaN mean if there is one (torch's argmax / argmin).  Every sum is fp64 in a fixed
 * order (columns of a bin in column order, rows in row order) with no float atomics, so the totals are bit-identical from
 * run to run and do not depend on which other bins share the launch.
 * Preconditions (not checked on the device): segs name pairs below n_pairs and columns below n_cols; a bin outside
 * [0, n_bins) is skipped.  P2PVG_ERR_BAD_ARG: NULL or misaligned pointers, n_metrics outside 1..8, B, nsample, n_seg or
 * n_bins < 1, n_cols < n_seg.  P2PVG_ERR_UNSUPPORTED: n_cols * B * n_metrics >= 2^31. */
int p2pvg_metrics_fold(const double* scores, int n_metrics, int higher_mask, int B, int nsample, const int32_t* segs, int n_seg,
                       const int32_t* col_bin, int n_cols, int n_bins, double* part_v, int32_t* part_c, uint32_t* counter,
                       double* sums, uint64_t* counts, uint64_t* rows, void* stream);

/* The pictures of the reference's misc/visualize.py vis_seq (:176-261) from generated frames, in one launch.
 *   store0 [n0][C][H][H], store1 [n1][C][H][H] fp32 frame stores (a generation graph's input and output buffers, or any
 *              stacked store); C = 1 (replicated to 3 channels) or 3; square frames, 1 <= H <= 128
 *   tiles_host [r_len][n_block][6][3] int32, HOST memory: per tile (frame t, row block i, row j) the store (0 / 1), the frame
 *              in it (-1: an all-zero frame) and the border (0 none, 1 orange (1, 165/255, 0), 2 red (1, 0, 0), 3 pixels
 *              wide); checked, then copied to tiles_dev (device, same size) on the stream before the launch
 *   canvas     [3][n_block * 6 * H][r_len * H] fp32: tile (t, i, j) at rows (6 i + j) H, columns t H (the PNG)
 *   video      [r_len][3][n_block * H][6 * H] fp32: tile (t, i, j) in frame t at rows i H, columns j H (add_video)
 *   gif        [r_len][n_block * H][6 * H][3] uint8: video frame t, channels last, (uint8)truncf(v * 255.f) (the GIF frames,
 *              the reference's (frame * 255).astype(np.uint8) for frames in [0, 1])
 * Every output value is a copy of a frame value, a border constant or that truncation, so all three are bit-identical to
 * the reference's composition of the same frames.
 * P2PVG_ERR_BAD_ARG: NULL pointers, C not 1 or 3, H outside 1..128, r_len < 1, n_block < 1, a tile whose store is not 0 / 1,
 * whose frame is not -1 .. n_store - 1 or whose border is not 0..2.  P2PVG_ERR_UNSUPPORTED: outputs of 2^31 values or more. */
int p2pvg_vis_canvas(const float* store0, int n0, const float* store1, int n1, int C, int H, const int32_t* tiles_host,
                     int32_t* tiles_dev, int r_len, int n_block, float* canvas, float* video, uint8_t* gif, void* stream);

/* The pictures of the reference's generate.py (:117-163) for every output length, in one launch: tiles of frames, each with
 * its control-point border, written into destination images.
 *   store0 [n0][C][H][H], store1 [n1][C][H][H] fp32 frame stores; C = 1 (replicated to 3 channels) or 3; 1 <= H <= 128
 *   images_host [n_images][4] int64, HOST memory: per destination image (offset, kind, h, w): kind 0 is fp32 [3][h][w] at
 *              out_f + offset, kind 1 uint8 [h][w][3] at out_u8 + offset
 *   tiles_host [n_tiles][6] int32, HOST memory: (store 0 / 1, frame or -1 for zeros, border 0 none / 1 orange / 2 red,
 *              image, y, x): the H x H frame written at rows y.., columns x.. of the image, channels c -> c (C = 3) or 0
 *              (C = 1); border pixels (3 wide) are (1, 165 / 255, 0) or (1, 0, 0); uint8 values are (uint8)truncf(v * 255.f)
 *   tables_dev device workspace, 8-byte aligned, of 32 n_images + 24 n_tiles bytes: the checked tables are copied there on
 *              the stream before the launch
 *   out_f      n_f fp32 values, out_u8 n_u8 bytes (either may be NULL when its count is 0)
 * P2PVG_ERR_BAD_ARG: NULL or misaligned tables, C not 1 or 3, H outside 1..128, n_images < 1, an image of 2^20 rows or
 * columns or more, or one that does not fit its output, a tile whose store, frame, border or image is out of range or which does not fit its image.  Nothing is copied or
 * launched then.  n_tiles == 0 returns P2PVG_OK without a launch. */
int p2pvg_vis_tiles(const float* store0, int n0, const float* store1, int n1, int C, int H, const int32_t* tiles_host,
                    int n_tiles, const int64_t* images_host, int n_images, void* tables_dev, float* out_f, long long n_f,
                    uint8_t* out_u8, long long n_u8, void* stream);

/* TensorBoard histograms (the reference's train.py:225-233 add_histogram calls) of many device ranges in one launch.
 *   segs       [n_seg][3] int64, HOST memory: per segment the device address of a contiguous range, its element count
 *              (>= 1) and its dtype (P2PVG_F32 or P2PVG_F64); the address is aligned to the element size
 *   edges      [n_edges] fp64, HOST memory: strictly increasing finite bin edges, 2 <= n_edges <= 4096 (p2pvg_b200.tboard
 *              DEFAULT_BINS holds TensorBoard's 1549 default edges)
 *   workspace  p2pvg_histograms_workspace_bytes(segs, n_seg, n_edges) bytes, 16-byte aligned: the edge and segment tables
 *              (staged on the host and copied on the stream before the launch) and fp64 partials of every chunk of
 *              P2PVG_HIST_CHUNK elements, i.e. 32 * sum_s ceil(count_s / 16384) bytes plus the tables
 *   counts     [n_seg][n_edges - 1] int64 (8-byte aligned): np.histogram(values.astype(np.float64), bins=edges) -- bins
 *              [e_k, e_k+1), the last one closed; values below e_0 or above e_last and NaN are not counted; -0.0 counts
 *              as 0.0.  fp32 values are widened to fp64 exactly (the library is built without -ftz or fast math).
 *   stats      [n_seg][5] fp64 (8-byte aligned): min, max (numpy's: NaN if any value is NaN, +-inf kept), num (the element
 *              count), sum and sum of squares of the fp64 values
 * sum and sum of squares are summed in a fixed order of fixed-size chunks of the segment, so each segment's results are
 * bit-identical whatever else shares the launch and from run to run; the order is not numpy's, so they match
 * values.sum() / values.dot(values) to rounding, and exactly when every partial sum is representable.
 * n_seg == 0 returns P2PVG_OK without a launch (every pointer may then be NULL).
 * P2PVG_ERR_BAD_ARG: NULL or misaligned pointers, n_seg < 0, n_edges < 2, an edge not finite or not above the previous one,
 * a segment dtype other than F32 / F64, a count < 1.  P2PVG_ERR_UNSUPPORTED: n_edges > 4096, a count >= 2^40.
 * P2PVG_ERR_WORKSPACE: workspace smaller than the query. */
#define P2PVG_HIST_CHUNK 16384
size_t p2pvg_histograms_workspace_bytes(const int64_t* segs, int n_seg, int n_edges);
int p2pvg_histograms(const int64_t* segs, int n_seg, const double* edges, int n_edges, void* workspace, size_t ws_bytes,
                     int64_t* counts, double* stats, void* stream);

/* PNG files (8-bit RGB, colour type 2) of n images in one call, every stage on the device: quantisation, per-row filter
 * choice, deflate in segments of P2PVG_PNG_SEGMENT filtered bytes (one IDAT chunk each), zlib framing, chunk CRCs and the
 * packing of every file into one buffer.
 *   images     [n][5] int64, HOST memory: per image the device address of a contiguous [C][H][W] array, its dtype
 *              (P2PVG_F32, 4-byte aligned, or P2PVG_PNG_U8), C (1: the channel is replicated to RGB, or 3), H and W
 *              (1 .. 2^24 - 1 each)
 *   rule       P2PVG_PNG_SAVE_IMAGE: u8 = trunc(clamp((x * 255) + 0.5, 0, 255)), each operation one fp32 rounding
 *              (torchvision.utils.save_image); P2PVG_PNG_TENSORBOARD: u8 = trunc(clamp(x * 255, 0, 255))
 *              (torch.utils.tensorboard.summary.image for float input).  uint8 images are taken as they are.  NaN is
 *              outside the contract.
 *   workspace  p2pvg_png_workspace_bytes(images, n) bytes, 256-byte aligned (tables, filtered streams, LZ77 scratch)
 *   out        at least p2pvg_png_out_bytes(images, n) bytes: the files, back to back in image order
 *   files      [n][2] int64 (8-byte aligned): offset in out and size of each file
 * Each segment is deflated by one CTA (matches reach up to 32 KB back, into earlier segments of the same image but never
 * before its first byte); every segment but an image's last ends with an empty stored block.  The Adler-32 of an image's
 * stream is combined from its segments' (sum of bytes, sum of (bytes to the segment's end) * byte) parts:
 * a = 1 + sum S_k, b = N + sum (W_k + (bytes after segment k) * S_k), mod 65521.  The bytes of a file depend on its image
 * and the rule alone, not on the other images of the call.
 * n == 0 returns P2PVG_OK without a launch.  P2PVG_ERR_BAD_ARG: a malformed table row, rule or pointer;
 * P2PVG_ERR_UNSUPPORTED: an image of 2^24 rows or columns or more; P2PVG_ERR_WORKSPACE: workspace or out too small.
 * The size queries return 0 for a table the encoder rejects. */
#define P2PVG_PNG_U8 3
#define P2PVG_PNG_SAVE_IMAGE 0
#define P2PVG_PNG_TENSORBOARD 1
#define P2PVG_PNG_SEGMENT 65536
size_t p2pvg_png_workspace_bytes(const int64_t* images, int n);
size_t p2pvg_png_out_bytes(const int64_t* images, int n);
int p2pvg_png_encode(const int64_t* images, int n, int rule, void* workspace, size_t ws_bytes, uint8_t* out, size_t out_bytes,
                     int64_t* files, void* stream);

/* GIF89a animations of n frame sequences in one call, every per-pixel stage on the device: quantisation, each frame's
 * colour set and palette, the index map, LZW in independent segments of P2PVG_GIF_SEGMENT pixels, the bit packing, the
 * data sub-blocks and the packing of every file into one buffer.
 *   anims      [n][7] int64, HOST memory: per animation the device address of contiguous frames -- P2PVG_PNG_U8
 *              [T][H][W][3] or P2PVG_F32 [T][3][H][W] (4-byte aligned) --, T, H and W (1..65535 each), the delay of every
 *              frame in centiseconds and the NETSCAPE2.0 loop count (0: forever; 0..65535 each)
 *   rule       the quantisation of fp32 frames, as p2pvg_png_encode's (P2PVG_PNG_SAVE_IMAGE or P2PVG_PNG_TENSORBOARD)
 *   workspace  p2pvg_gif_workspace_bytes(anims, n) bytes, 256-byte aligned
 *   out        at least p2pvg_gif_out_bytes(anims, n) bytes: the files, back to back in animation order
 *   files      [n][2] int64 (8-byte aligned): offset in out and size of each file
 * A file: the header and a logical screen descriptor without a global colour table, a NETSCAPE2.0 loop block, per frame a
 * graphic control extension (the delay, no transparency), an image descriptor of the whole frame with a local table of 256
 * entries, LZW minimum code size 8 and the data sub-blocks; then the trailer.  The palette: a frame of at most 256 distinct
 * colours lists exactly those, sorted by 24-bit key (0xRRGGBB), and is lossless; otherwise median cut (split the box of
 * largest count-weighted squared error along its widest channel at the count-weighted median) to 256 boxes, their rounded
 * means, then 3 Lloyd iterations over the distinct colours.  Each pixel takes its nearest entry (squared RGB distance,
 * lowest index on ties).  LZW: each segment starts from the post-clear state and ends with a CLEAR at its final code width
 * (the frame's last with an EOI); the stream opens with a CLEAR; a table of 4096 codes emits a CLEAR at 12 bits.  The bytes
 * of a file depend on its frames, rule, delay and loop alone, not on the other animations of the call.
 * n == 0 returns P2PVG_OK without a launch.  P2PVG_ERR_BAD_ARG: a malformed table row, rule or pointer;
 * P2PVG_ERR_UNSUPPORTED: 2^40 pixels or 2^24 frames in all or more; P2PVG_ERR_WORKSPACE: workspace or out too small.
 * The size queries return 0 for a table the encoder rejects. */
#define P2PVG_GIF_SEGMENT 65536
size_t p2pvg_gif_workspace_bytes(const int64_t* anims, int n);
size_t p2pvg_gif_out_bytes(const int64_t* anims, int n);
int p2pvg_gif_encode(const int64_t* anims, int n, int rule, void* workspace, size_t ws_bytes, uint8_t* out, size_t out_bytes,
                     int64_t* files, void* stream);

/* CRC-32C (Castagnoli) of n host bytes, continuing from crc (0 to start): crc32c(a + b) = p2pvg_crc32c(b, crc32c(a)).
 * Host code (no device, no stream); data may be NULL when n == 0. */
uint32_t p2pvg_crc32c(const void* data, size_t n, uint32_t crc);

/* Human3.6M skeletons as the reference's Skeleton3DVisualizer draws them (data/human36m/human36m.py:290-388), n images in
 * one launch; the camera, stroke and blend rules are those of p2pvg_b200/skeleton.py's module docstring.
 *   poses       [n][J][3] fp32 device poses (x, y, z), plotted at (x, z, y)
 *   views       [n] int32 device camera view per image, 0..3; an image whose view is outside 0..3 is left white
 *   J           joints, 2..32; limb l = 0..J-2 joins joint l + 1 to parents_host[l + 1], drawn in that order
 *   parents_host [J] int32, HOST memory: parents[0] = -1 and 0 <= parents[j] < j
 *   colors_host [J - 1][3] fp32, HOST memory: limb RGB in 0..1
 *   matrices_host [4][3][4] fp32, HOST memory: per view rows 0, 1 and 3 of M = P . View . W (the plot limits are in W)
 *   out_f       [n][3][98][98] fp32 or NULL: float32(q / 255.) of the quantised value q
 *   out_u8      [n][98][98][3] uint8 or NULL: q = min(255, floor(255 c + 0.5)) of the blended fp32 colour c
 * Projection and coverage are fp64 with one rounding per operation; blend and quantisation fp32, likewise.  A limb shorter
 * than 1e-6 px or with a non-finite projected end draws nothing.
 * n == 0 returns P2PVG_OK without a launch.  P2PVG_ERR_BAD_ARG (nothing launched): n < 0, J outside 2..32, a null table,
 * null poses / views or both outputs when n > 0, misaligned device pointers, bad parents, a colour outside 0..1, a
 * non-finite matrix value. */
int p2pvg_skeleton_render(const float* poses, const int32_t* views, int n, int J, const int32_t* parents_host,
                          const float* colors_host, const float* matrices_host, float* out_f, uint8_t* out_u8, void* stream);

#ifdef __cplusplus
}
#endif
#endif
