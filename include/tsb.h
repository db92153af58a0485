/*
 * libtsb — C ABI of the H100-native (sm_90a) semantic-segmentation training hot path.
 *
 * Drop-in boundary for the training step of yu-changqian/TorchSeg ("furnace"): every entry point
 * replaces one lowering that the reference obtains from torch.nn / ATen / cuDNN / apex on the path
 *   model/bisenet/cityscapes.bisenet.R18/train.py:116-142  (zero_grad → forward(loss) → backward → step).
 * The reference itself has no C ABI (its two pybind11 extensions are dead code, SURVEY.md §2.1); the
 * symbols below are what a ctypes / cffi / pybind binding on the reference side would bind
 * (see INTEGRATION.md for the stub).
 *
 * Conventions (all functions):
 *   - plain pointers + sizes, no torch types; the CALLER owns every buffer including workspaces;
 *   - no allocation, no host synchronisation, no global mutable state inside (except a cached
 *     driver entry point and SM count);
 *   - work is enqueued on the cudaStream_t passed in (pass 0 for the legacy default stream);
 *   - entry points that sum per-CTA partials (conv statistics and weight gradients, BN reductions, channel-attention
 *     gradient, adaptive pooling, bias gradient) take `float* ws, long long ws_floats`: a caller-owned fp32
 *     workspace that holds one slot per CTA; the slots are summed in a fixed order, so results are identical from run
 *     to run. A workspace may only be used by one call at a time: give each stream its own, or order the calls.
 *     24 Mi floats (96 MB) covers every shape of the shipped networks; a too-small workspace is an error (the
 *     weight-gradient kernels instead fall back to one split, which needs none);
 *   - the device is the calling thread's current device;
 *   - return 0 on success, a negative TSB_ERR_* on failure; tsb_last_error() returns a thread-local
 *     human-readable message;
 *   - activations are NHWC ("channels-last") with an explicit channel stride `cs` (elements between
 *     consecutive pixels), so channel slices of a wider buffer (concat-free FFM/PPM) are addressable;
 *     pixel (n,h,w) of a tensor with height H, width W lives at ((n*H + h)*W + w)*cs;
 *   - dtype tags: TSB_F32 / TSB_BF16.
 */
#ifndef TSB_H_
#define TSB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* tsb_stream_t; /* == cudaStream_t */

enum { TSB_F32 = 0, TSB_BF16 = 1 };
enum { TSB_OK = 0, TSB_ERR_ARG = -1, TSB_ERR_CUDA = -2, TSB_ERR_UNSUPPORTED = -3 };

/* ---- library ---------------------------------------------------------------------------------- */
const char* tsb_last_error(void);
int tsb_version(void);          /* 10000*major + 100*minor + patch */
/* number of kernels launched by this library from the calling process since load (all threads) */
long long tsb_launch_count(void);

/* ================================================================================================
 * OHEM cross-entropy — replaces ProbOhemCrossEntropy2d.forward, furnace/seg_opr/loss_opr.py:68-98
 * (softmax :75, gather :82-83, torch.sort :86, threshold :87-89, kept mask :90-92, CE :98).
 *
 * Workspace `state` is TSB_OHEM_STATE_WORDS 32-bit words (device), zeroed by tsb_ohem_begin.
 * Pipeline (no host sync anywhere):
 *   tsb_ohem_begin → tsb_ohem_ptarget[_up] → tsb_ohem_select → tsb_ohem_loss  (forward)
 *   tsb_ohem_grad[_up]                                                       (backward)
 * ============================================================================================== */
#define TSB_OHEM_STATE_WORDS 8192
/* word offsets inside `state` that callers may read back (after a stream sync) */
#define TSB_OHEM_ST_NUM_VALID 4096   /* uint32: #pixels with label != ignore                     */
#define TSB_OHEM_ST_COUNT_LE 4097    /* uint32: #pixels (incl. ignored, p:=1) with p <= thresh    */
#define TSB_OHEM_ST_ACTIVE 4098      /* uint32: 1 if the kept mask is applied (loss_opr.py:80,85) */
#define TSB_OHEM_ST_THRESH 4099      /* float : final threshold T                                 */
#define TSB_OHEM_ST_KEPT 4100        /* uint32: #kept pixels (written by tsb_ohem_loss)           */
#define TSB_OHEM_ST_LOSS 4101        /* float : mean loss (written by tsb_ohem_loss)              */
#define TSB_OHEM_ST_INVDEN 4102      /* float : 1/denominator used for the gradient               */

int tsb_ohem_begin(uint32_t* state, tsb_stream_t stream);

/* p_target from MATERIALISED logits (the reference boundary). logits: dtype F32/BF16, element
 * (n,c,y,x) at n*sn + c*sc + y*sy + x*sx (element strides; NCHW contiguous: sc=H*W, sy=W, sx=1).
 * labels int64 [N,H,W] contiguous. Writes p[N*H*W] (ignored pixels := 1.0f, loss_opr.py:81) and
 * nll[N*H*W] = -log_softmax(logits)[label] (0 for ignored); accumulates num_valid and count(p<=thresh)
 * into state (the radix histograms are built lazily by tsb_ohem_select, only when the k-th value is needed). */
int tsb_ohem_ptarget(const void* logits, int dtype, long long sn, long long sc, long long sy, long long sx,
                     const int64_t* labels, int N, int C, int H, int W, int ignore_label, float thresh,
                     float* p, float* nll, uint32_t* state, tsb_stream_t stream);

/* Fused-upsample form: logits are the LOW-resolution fp32 NHWC head output [N,h,w,cs] and are
 * bilinearly interpolated (align_corners=True, network.py:163-166) to [H,W] on the fly. */
int tsb_ohem_ptarget_up(const float* logits_lo, int cs, int h, int w, const int64_t* labels, int N, int C, int H,
                        int W, int ignore_label, float thresh, float* p, float* nll, uint32_t* state,
                        tsb_stream_t stream);

/* k-th-smallest selection (exact, 12+12+8-bit radix select over the bit patterns of p) replacing the
 * full torch.sort (loss_opr.py:86-89). n = N*H*W. */
int tsb_ohem_select(const float* p, long long n, long long min_kept, float thresh, uint32_t* state,
                    tsb_stream_t stream);

/* kept = valid && (!active || p <= T); loss = sum(w[label]*nll)/sum(w[label]) over kept (w==NULL → 1).
 * Writes *loss_out (device float) and state[KEPT|LOSS|INVDEN]. */
int tsb_ohem_loss(const float* p, const float* nll, const int64_t* labels, long long n, int ignore_label,
                  const float* class_weight, uint32_t* state, float* loss_out, tsb_stream_t stream);

/* d(logits) for materialised logits, same strides/dtype as the logits:
 * (softmax - onehot) * w[label] * invden * (*gscale) for kept pixels, 0 elsewhere. gscale: device float. */
int tsb_ohem_grad(const void* logits, int dtype, long long sn, long long sc, long long sy, long long sx,
                  const int64_t* labels, const float* p, int N, int C, int H, int W, int ignore_label,
                  const float* class_weight, const uint32_t* state, const float* gscale, void* dlogits,
                  tsb_stream_t stream);

/* d(low-res logits) through the transposed bilinear stencil. dlogits_lo fp32 [N,h,w,cs] must be
 * zeroed by the caller (accumulated with red.global.add.f32). */
int tsb_ohem_grad_up(const float* logits_lo, int cs, int h, int w, const int64_t* labels, const float* p, int N,
                     int C, int H, int W, int ignore_label, const float* class_weight, const uint32_t* state,
                     const float* gscale, float* dlogits_lo, tsb_stream_t stream);

/* ================================================================================================
 * Bilinear resize, align_corners=True — replaces F.interpolate(mode='bilinear', align_corners=True)
 * call sites model/bisenet/cityscapes.bisenet.R18/network.py:82-84,93-94,164-166 (SURVEY §8 a10).
 * NHWC, C channels, channel strides ics/ocs >= C. Backward is the deterministic gather-form transpose.
 * The forward takes 16-byte vectors when C, ics and ocs are multiples of 8 and both pointers are 16-byte aligned, and
 * a scalar path otherwise; the backward requires exactly that (C, ics, ocs multiples of 8; dout, din 16-byte aligned).
 * ============================================================================================== */
int tsb_bilinear_fwd(const void* in, int idtype, int ics, void* out, int odtype, int ocs, int N, int C, int Hi,
                     int Wi, int Ho, int Wo, tsb_stream_t stream);
int tsb_bilinear_bwd(const void* dout, int odtype, int ocs, void* din, int idtype, int ics, int N, int C, int Hi,
                     int Wi, int Ho, int Wo, int accumulate, tsb_stream_t stream);
/* NCHW fp32 variant used at the reference boundary (BiSeNetHead returns NCHW fp32 full-res logits). */
int tsb_bilinear_fwd_nhwc_to_nchw(const void* in, int idtype, int ics, float* out, int N, int C, int Hi, int Wi,
                                  int Ho, int Wo, tsb_stream_t stream);

/* ================================================================================================
 * Pooling — nn.AdaptiveAvgPool2d (furnace/seg_opr/seg_oprs.py:113,200,223; pspnet network.py:83)
 * and nn.MaxPool2d(3,2,1) (furnace/base_model/resnet.py:132). NHWC bf16; C and every channel stride are multiples of
 * 8 with stride >= C; activations and the fp32 adaptive-pool gradient dout are 16-byte aligned, argmax 8-byte aligned.
 * ============================================================================================== */
/* out fp32 [N, S, S, C] (bins [floor(i*H/S), ceil((i+1)*H/S)) ), S==1 is the global pool */
int tsb_adaptive_avgpool_fwd(const void* in, int ics, int N, int C, int H, int W, int S, float* out, float* ws,
                             long long ws_floats, tsb_stream_t stream);
/* din(bf16) (+)= dout[n, bin(h), bin(w), c] / bin_area  (S==1 → broadcast of dout/(H*W)) */
int tsb_adaptive_avgpool_bwd(const float* dout, int N, int C, int H, int W, int S, void* din, int ics,
                             int accumulate, tsb_stream_t stream);
/* argmax (optional): uint8 [N,P,Q,C] window position r*3+s of the FIRST maximum in scan order (ATen
 * max_pool2d tie semantics); the backward is a gather over it. */
int tsb_maxpool3x3s2_fwd(const void* in, int ics, void* out, int ocs, void* argmax, int N, int C, int H, int W,
                         tsb_stream_t stream);
int tsb_maxpool3x3s2_bwd(const void* argmax, const void* dout, int ocs, void* din, int dcs, int N, int C, int H,
                         int W, tsb_stream_t stream);

/* ================================================================================================
 * BatchNorm (training) — replaces norm_layer(...) inside ConvBnRelu (seg_oprs.py:34,42), resnet
 * bn1/bn2 (resnet.py:24-51) and apex SyncBatchNorm (train.py:54-55). Statistics come from the conv
 * epilogue (tsb_conv2d sum/sumsq) or tsb_bn_stats; cross-GPU reduction of {sum,sumsq} happens between
 * stats and finalize (NCCL, outside this library).
 * x, y, dy, dx, residual, dres: bf16 NHWC, C and channel strides multiples of 8, strides >= C, 16-byte aligned. The fp32
 * per-channel vectors (scale, shift, mean, invstd, gamma, sum_dz, sum_dz_xhat) and the workspace are 16-byte aligned.
 * ============================================================================================== */
/* per-channel sum and sum of squares of x (bf16 NHWC), accumulated into fp32 sum[C], sumsq[C] (caller zeroes) */
int tsb_bn_stats(const void* x, int cs, long long npix, int C, float* sum, float* sumsq, float* ws, long long ws_floats,
                 tsb_stream_t stream);
/* mean/invstd from (sum,sumsq,count); scale=gamma*invstd, shift=beta-mean*scale; running stats update
 * (momentum, unbiased variance — SURVEY App. A3). running_* may be NULL. */
int tsb_bn_finalize(const float* sum, const float* sumsq, double count, int C, const float* gamma,
                    const float* beta, float eps, float momentum, float* mean, float* invstd, float* scale,
                    float* shift, float* running_mean, float* running_var, tsb_stream_t stream);
/* y = act(x*scale[c] + shift[c] + residual); act = ReLU if relu. x,y,residual bf16 NHWC (own strides) */
int tsb_bn_apply(const void* x, int xcs, const float* scale, const float* shift, const void* residual, int rcs,
                 int relu, void* y, int ycs, long long npix, int C, tsb_stream_t stream);
/* backward pass 1: dz = dy * (relu ? y>0 : 1); sum_dz[c] += Σ dz ; sum_dz_xhat[c] += Σ dz * (x-mean)*invstd.
 * With relu and y == NULL the mask is recomputed as fma(x, scale[c], shift[c]) > 0 (exact for layers WITHOUT a
 * residual input) and the read of y is saved; scale/shift are then required. */
int tsb_bn_bwd_reduce(const void* dy, int dycs, const void* y, int ycs, const void* x, int xcs, const float* mean,
                      const float* invstd, int relu, long long npix, int C, float* sum_dz, float* sum_dz_xhat,
                      const float* scale, const float* shift, float* ws, long long ws_floats, tsb_stream_t stream);
/* backward pass 2: dx = gamma*invstd*(dz - sum_dz/cnt - xhat*sum_dz_xhat/cnt); optional dres = dz;
 * optional dgamma_acc[c] += sum_dz_xhat[c], dbeta_acc[c] += sum_dz[c] (parameter gradients, folded into this pass);
 * y == NULL with relu: mask recomputed from scale/shift as in tsb_bn_bwd_reduce */
int tsb_bn_bwd_apply(const void* dy, int dycs, const void* y, int ycs, const void* x, int xcs, const float* mean,
                     const float* invstd, const float* gamma, const float* sum_dz, const float* sum_dz_xhat,
                     double count, int relu, void* dx, int dxcs, void* dres, int drcs, long long npix, int C,
                     float* dgamma_acc, float* dbeta_acc, const float* scale, const float* shift,
                     tsb_stream_t stream);
/* tsb_bn_bwd_apply, ADDING into dx: dx = bf16(float(dx) + r), rounded once, with r the fp32 value tsb_bn_bwd_apply
 * would round and store (same arguments, same dgamma_acc / dbeta_acc folding and mask rules). The input gradients of
 * several BatchNorms over channel slices of one concatenated tensor (DenseASPP's pre-activation blocks) land in one
 * gradient buffer this way. */
int tsb_bn_bwd_apply_add(const void* dy, int dycs, const void* y, int ycs, const void* x, int xcs, const float* mean,
                         const float* invstd, const float* gamma, const float* sum_dz, const float* sum_dz_xhat,
                         double count, int relu, void* dx, int dxcs, void* dres, int drcs, long long npix, int C,
                         float* dgamma_acc, float* dbeta_acc, const float* scale, const float* shift,
                         tsb_stream_t stream);
/* out/argmax = tsb_maxpool3x3s2_fwd of tsb_bn_apply(x, scale, shift, no residual, relu = 1), bit for bit and in the
 * same layouts, in one pass that never writes the normalised map (the context stem of BiSeNet-R18). */
int tsb_bn_apply_maxpool3x3s2(const void* x, int xcs, const float* scale, const float* shift, void* out, int ocs,
                              void* argmax, int N, int C, int H, int W, tsb_stream_t stream);

/* ================================================================================================
 * Channel-attention fusions — AttentionRefinement.forward seg_oprs.py:207-212 (fm*sigmoid(se) and the
 * caller's `fm += last_fm`, bisenet network.py:91-92) and FeatureFusion.forward seg_oprs.py:233-238
 * (fm + fm*sigmoid(se)).  a[n,c] is the PRE-sigmoid attention logit (fp32 [N,C]).
 *   y = x * (base + sigmoid(a[n,c])) + add          base=0 (ARM) / 1 (FFM); add may be NULL
 * bf16 NHWC operands: C and channel strides multiples of 8, strides >= C, 16-byte aligned; a is 16-byte aligned.
 * ============================================================================================== */
int tsb_chan_scale_fwd(const void* x, int xcs, const float* a, float base, const void* add, int acs, void* y,
                       int ycs, int N, int HW, int C, tsb_stream_t stream);
/* dx = dy*(base+sig); da[n,c] += Σ_hw dy*x*sig*(1-sig)  (da fp32 [N,C], caller zeroes); dadd == dy */
int tsb_chan_scale_bwd(const void* dy, int dycs, const void* x, int xcs, const float* a, float base, void* dx,
                       int dxcs, float* da, int N, int HW, int C, float* ws, long long ws_floats, tsb_stream_t stream);

/* ================================================================================================
 * Layout / precision packing
 * ============================================================================================== */
/* NCHW fp32 image [N,3,H,W] → 2x2 space-to-depth, column-padded, NHWC16 bf16 [N, H/2, W/2+4, 16]
 * (channel = (py*2+px)*3 + c, 12..15 zero; 2 zero pixels of left padding) — operand of the 7x7/2 stems
 * resnet.py:126, bisenet network.py:118. */
int tsb_pack_image_s2d(const float* img, int N, int H, int W, void* out, tsb_stream_t stream);
/* fp32 [K,R,S,C] weights (KRSC == channels_last OIHW) → bf16 copy and bf16 flipped-transposed
 * [C,R,S,K] copy for dgrad (either output may be NULL) */
int tsb_pack_weight(const float* w, int K, int R, int S, int C, void* w_bf16, void* wt_bf16, tsb_stream_t stream);
/* RxRx3 stride-2 stem weights [K,R,R,3] fp32 (R = 7 pad 3: resnet.py:126 / bisenet network.py:118; R = 3 pad 1:
 * the v1c deep stem resnet.py:111-112) → s2d-packed bf16 [K,4,4,16]; and the reverse for gradients
 * (dW[K,R,R,3] += unpack(dWp[K,4,4,16] fp32)) */
int tsb_pack_stem_weight(const float* w, int K, int R, void* wp_bf16, tsb_stream_t stream);
int tsb_unpack_stem_wgrad(const float* dwp, int K, int R, float* dw, tsb_stream_t stream);
/* elementwise: dst = (dtype)src * (*scale_dev or 1) ; strided NHWC channel slices, C multiple of 8.
 * For cast_scale, add, add_relu and relu_bwd: C and channel strides multiples of 8, strides >= C, 16-byte aligned. */
int tsb_cast_scale(const void* src, int sdtype, int scs, void* dst, int ddtype, int dcs, long long npix, int C,
                   const float* scale_dev, tsb_stream_t stream);
/* dst[pix, 0..Kp) = (bf16) src[pix, 0..K) zero-extended (any K, any source channel stride): the gradient of a K-class
 * head into the 64-multiple GEMM-K layout tsb_conv2d_dgrad / wgrad read */
int tsb_cast_pad(const void* src, int sdtype, int scs, int K, void* dst_bf16, int dcs, int Kp, long long npix,
                 tsb_stream_t stream);
/* y = a + b (bf16 NHWC) */
int tsb_add(const void* a, int acs, const void* b, int bcs, void* y, int ycs, long long npix, int C,
            tsb_stream_t stream);
/* y = relu(a + b): the `self.relu(t + x)` tail of RefineResidual / BNRefine (seg_oprs.py:158-162,184-188);
 * dx = (y > 0) ? dy : 0 is its backward (the same dx goes to both addends) */
int tsb_add_relu(const void* a, int acs, const void* b, int bcs, void* y, int ycs, long long npix, int C,
                 tsb_stream_t stream);
int tsb_relu_bwd(const void* dy, int dycs, const void* y, int ycs, void* dx, int dxcs, long long npix, int C,
                 tsb_stream_t stream);

/* ---- point-wise spatial attention (PSANet: model/psanet/ade.psanet.R101_v1c/network.py:119-138) ----
 * `torch.softmax(att.view(b, c, -1), dim=1)`: in NHWC the softmax runs over the C (=3600) contiguous channels of each
 * of the `rows` pixels; channels [C, Cp) of the output are written as zeros so the matrix can be the GEMM-K operand
 * of a 64-channel-tiled 1x1 convolution (input bf16 or fp32 logits: the reference keeps them in fp32 and a peaky
 * soft-max amplifies bf16 logit rounding). bwd: dA = S * (dS - Σ_c S·dS).
 * `torch.bmm(reduce_x.view(b,512,-1), S)` itself runs per image on tsb_conv2d_{fprop,dgrad,wgrad} with the image's
 * feature map as the weight operand; tsb_transpose_pad builds that operand: out[c, r] = in[r, c] (bf16 out, rows of
 * length ocs, columns [R, Rp) zero-filled). */
int tsb_softmax_rows_fwd(const void* in, int idtype, int ics, void* out_bf16, int ocs, long long rows, int C, int Cp,
                         tsb_stream_t stream);
int tsb_softmax_rows_bwd(const void* S_bf16, int scs, const void* dS_bf16, int dscs, void* dA_bf16, int dacs,
                         long long rows, int C, int Cp, tsb_stream_t stream);
int tsb_transpose_pad(const void* in, int idtype, int ics, void* out_bf16, int ocs, int R, int Cc, int Rp,
                      tsb_stream_t stream);

/* ================================================================================================
 * Convolution as im2col-free implicit GEMM on Hopper tensor cores (TMA → 128B-swizzled smem →
 * wgmma, fp32 accumulators in registers) — replaces nn.Conv2d inside ConvBnRelu (seg_oprs.py:29-31),
 * conv3x3 (resnet.py:11-14), the 1x1 heads (bisenet network.py:156-161) and their cuDNN
 * dgrad / wgrad. bf16 operands, fp32 accumulation.
 *
 * x : bf16 NHWC [N,H,W,C] (channel stride xcs >= C, C % 64 == 0)
 * w : bf16 [K,R,S,C] (tsb_pack_weight)   — fprop;  wt: bf16 [C,R,S,K] flipped — dgrad
 * y : NHWC [N,P,Q,*] with channel stride ycs >= K; dtype BF16 or F32; K_store = ceil8(K) channels written, those
 *     past K as zeros
 * Every activation may be a channel slice of a wider buffer: its pointer 16-byte aligned (a multiple of 8 bf16
 * channels), its channel stride a multiple of 8. Channels past C (past K for dy) are never read.
 * ============================================================================================== */
typedef struct {
    int N, H, W, C;          /* input  */
    int K, R, S;             /* filter */
    int stride, pad, dil;    /* same in both spatial dims */
    int P, Q;                /* output spatial size */
} tsb_conv_shape;

/* fprop: y = conv(x, w) (+bias[k]) ; optional per-channel batch statistics of the ROUNDED output
 * accumulated into sum[K], sumsq[K] (fp32, caller zeroes) — the BN-statistics epilogue. */
int tsb_conv2d_fprop(const tsb_conv_shape* s, const void* x, int xcs, const void* w, const float* bias, void* y,
                     int ydtype, int ycs, float* sum, float* sumsq, float* ws, long long ws_floats, tsb_stream_t stream);
/* inference form with the BatchNorm FOLDED into the weights (evaluator path, furnace/engine/evaluator.py:255-275 runs the
 * network in eval mode): y = relu?(conv(x, w_folded) + bias (+ res)) in the conv epilogue — no raw tensor, no BN pass.
 * res (optional, bf16) must be laid out exactly like y (rescs == ycs): the shortcut of a residual block. */
int tsb_conv2d_fprop_fused(const tsb_conv_shape* s, const void* x, int xcs, const void* w, const float* bias,
                           const void* res, int rescs, int relu, void* y, int ydtype, int ycs, tsb_stream_t stream);
/* dgrad: dx = conv_transpose(dy, w). wt is the flipped-transposed pack. K % 64 == 0, dycs >= K; C % 8 == 0, dx bf16
 * (channel stride dxcs >= C; channels [C, dxcs) are not written). If accumulate != 0, dx += result (residual /
 * multi-consumer gradient accumulation in the epilogue); a stride-2 1x1 leaves the positions no tap reaches as they
 * were, and writes zeros there when accumulate == 0. */
int tsb_conv2d_dgrad(const tsb_conv_shape* s, const void* dy, int dycs, const void* wt, void* dx, int dxcs,
                     int accumulate, tsb_stream_t stream);
/* transposed convolution — replaces the nn.ConvTranspose2d of DeConvBnRelu (furnace/seg_opr/seg_oprs.py:49-73).
 * ConvTranspose2d(Ci, Co, k, stride s, padding p, output_padding op, dilation d) maps x[N,Ci,H,W] to y[N,Co,Ho,Wo] with
 * Ho = (H-1)*s - 2p + d(k-1) + op + 1. `s` describes the ADJOINT conv, whose dgrad this is: {N, H = Ho, W = Wo, C = Co,
 * K = Ci, R = S = k, stride s, pad p, dil d, P = H, Q = W}. Its weight [K = Ci][C = Co][R][S] is the deconv weight
 * W[Ci][Co][k][k] itself, so a channels_last ConvTranspose2d weight is the adjoint conv's KRSC, and
 *   y       = tsb_conv_transpose2d_fprop(x, wt)       wt = flipped [Co][k][k][Ci] pack (tsb_pack_weight's second output)
 *   dx      = tsb_conv2d_fprop(dy)                     with the [Ci][k][k][Co] pack
 *   dW      = tsb_conv2d_wgrad(x := dy, dy := x)       straight into W's KRSC storage
 *   dbias   = tsb_bias_grad(dy)
 * The geometry limits follow: s in {1, 2}, k <= 4 (16 taps), square kernel / stride / pad / dilation, groups 1, and
 * op < s (otherwise the adjoint conv's output is not H x W and P, Q are rejected as inconsistent). Ci % 64 == 0,
 * Co % 8 == 0 (xcs >= Ci, ycs >= Co, multiples of 8). Epilogue as tsb_conv2d_fprop plus ReLU: y = relu?(acc + bias), bf16
 * or fp32; optional statistics of the rounded bf16 outputs added into sum[Co], sumsq[Co] (caller zeroes). Stride 2 runs
 * one launch per output parity class; positions no tap reaches (k = 1) hold relu?(bias) (0 without bias) and count in
 * the statistics, and the slots of all classes are summed in a fixed order. */
int tsb_conv_transpose2d_fprop(const tsb_conv_shape* s, const void* x, int xcs, const void* wt, const float* bias, int relu,
                               void* y, int ydtype, int ycs, float* sum, float* sumsq, float* ws, long long ws_floats,
                               tsb_stream_t stream);
/* wgrad: dw[K,R,S,C] (fp32, KRSC) += Σ_pixels dy ⊗ x (caller zeroes or accumulates); xcs >= C, dycs >= K (any K).
 * The per-split partial sums go to ws and are added in a fixed order, so the result is bit-reproducible; without a
 * workspace large enough for two splits the kernel adds into dw in place. */
int tsb_conv2d_wgrad(const tsb_conv_shape* s, const void* x, int xcs, const void* dy, int dycs, float* dw, float* ws,
                     long long ws_floats, tsb_stream_t stream);
/* 1x1 convolution of a pre-activation input (BatchNorm → ReLU → 1x1 conv, DenseASPP's blocks): the conv reads
 *   x̂ = bf16(relu(fmaf(x, in_scale[c], in_shift[c])))
 * (the arithmetic of tsb_bn_apply with relu, rounded once) instead of x. The kernels normalise each landed activation
 * tile in shared memory between the TMA load and the wgmma, so x̂ never reaches HBM; rows past the last pixel stay
 * zero. R = S = 1, stride 1, pad 0 only (anything else: TSB_ERR_UNSUPPORTED); C % 64 == 0; in_scale / in_shift fp32 [C],
 * 16-byte aligned.
 * fprop: y = relu?(conv(x̂, w) + bias), the rest as tsb_conv2d_fprop: training passes sum/sumsq (the BN-statistics
 *        epilogue over the rounded output) and no ReLU; eval passes the next BatchNorm folded into w / bias, relu = 1.
 *        Bit for bit tsb_bn_apply(relu) followed by tsb_conv2d_fprop (tsb_conv2d_fprop_fused in eval form).
 * wgrad: dw += Σ_pixels dy ⊗ x̂, the split plan and workspace rules of tsb_conv2d_wgrad; bit for bit tsb_bn_apply(relu)
 *        followed by tsb_conv2d_wgrad. */
int tsb_conv1x1_bnrelu_fprop(const tsb_conv_shape* s, const void* x, int xcs, const float* in_scale, const float* in_shift,
                             const void* w, const float* bias, int relu, void* y, int ydtype, int ycs, float* sum,
                             float* sumsq, float* ws, long long ws_floats, tsb_stream_t stream);
int tsb_conv1x1_bnrelu_wgrad(const tsb_conv_shape* s, const void* x, int xcs, const float* in_scale, const float* in_shift,
                             const void* dy, int dycs, float* dw, float* ws, long long ws_floats, tsb_stream_t stream);
/* stride-2 C_in=3 stem (7x7 pad 3 or 3x3 pad 1, same packed weight format) on the s2d-packed image (tsb_pack_image_s2d / tsb_pack_stem_weight):
 * xs2d [N,H/2,W/2+4,16] bf16, wp [K,4,4,16] bf16 → y [N,H/2,W/2,K] (K % 8 == 0, channel stride ycs >= K, exactly K
 * channels written). wgrad: dy with channel stride dycs >= K → dwp [K,4,64] fp32 (+=; tsb_unpack_stem_wgrad). */
int tsb_conv_stem_fprop(const void* xs2d, int N, int H, int W, const void* wp, int K, void* y, int ycs, float* sum,
                        float* sumsq, float* ws, long long ws_floats, tsb_stream_t stream);
int tsb_conv_stem_fprop_fused(const void* xs2d, int N, int H, int W, const void* wp, int K, const float* bias, int relu,
                              void* y, int ycs, tsb_stream_t stream);
int tsb_conv_stem_wgrad(const void* xs2d, int N, int H, int W, const void* dy, int dycs, int K, float* dwp, float* ws,
                        long long ws_floats, tsb_stream_t stream);
/* column sums: db[k] += Σ_pixels dy[pix,k] (bias gradient of the 1x1 classifier heads); any K, dycs >= K */
int tsb_bias_grad(const void* dy, int dycs, long long npix, int K, float* db, float* ws, long long ws_floats,
                  tsb_stream_t stream);

/* ================================================================================================
 * Depthwise 3x3 convolution (groups = C) — replaces the `groups=in_channels` nn.Conv2d of SeparableConvBnRelu
 * (furnace/base_model/xception.py:14-16; furnace/seg_opr/seg_oprs.py:76-94 with padding = dilation) and its cuDNN
 * dgrad / wgrad. Geometry: stride 1 with padding = dilation >= 1, or stride 2 with padding 1 and dilation 1; anything
 * else is an error. x, y, dy, dx: bf16 NHWC with channel strides (multiples of 8, >= C; 16-byte aligned), so channel
 * slices of wider (e.g. 64-padded) buffers are read and written in place; C % 8 == 0, C <= 4096. H, W: INPUT size; the
 * output is P = (H - 1) / stride + 1 by Q = (W - 1) / stride + 1. w: the fp32 [C][3][3] master weight, rounded to bf16
 * on load. All sums are fp32, taps in a fixed (r, s) order, rounded to bf16 once; taps outside the map add nothing.
 * ============================================================================================== */
/* y[n,p,q,c] = Σ_{r,s} x[n, p·stride+(r−1)·dilation, q·stride+(s−1)·dilation, c] · w[c,r,s] */
int tsb_dwconv2d_fprop(const void* x, int xcs, const float* w, void* y, int ycs, int N, int H, int W, int C, int stride,
                       int dilation, tsb_stream_t stream);
/* dx = the gather-form transpose of fprop (no atomics); accumulate != 0: dx = bf16(dx + result) */
int tsb_dwconv2d_dgrad(const void* dy, int dycs, const float* w, void* dx, int dxcs, int N, int H, int W, int C,
                       int stride, int dilation, int accumulate, tsb_stream_t stream);
/* dw[c,r,s] (fp32 [C][3][3]) += Σ_{n,p,q} dy[n,p,q,c] · x[n, p·stride+(r−1)·dilation, q·stride+(s−1)·dilation, c]: one
 * [C·9] workspace slot per CTA, summed in slot order (a too-small workspace is an error) */
int tsb_dwconv2d_wgrad(const void* x, int xcs, const void* dy, int dycs, float* dw, int N, int H, int W, int C,
                       int stride, int dilation, float* ws, long long ws_floats, tsb_stream_t stream);
/* the same three at dilation 1 (padding 1) */
int tsb_dwconv_fprop(const void* x, int xcs, const float* w, void* y, int ycs, int N, int H, int W, int C, int stride,
                     tsb_stream_t stream);
int tsb_dwconv_dgrad(const void* dy, int dycs, const float* w, void* dx, int dxcs, int N, int H, int W, int C, int stride,
                     int accumulate, tsb_stream_t stream);
int tsb_dwconv_wgrad(const void* x, int xcs, const void* dy, int dycs, float* dw, int N, int H, int W, int C, int stride,
                     float* ws, long long ws_floats, tsb_stream_t stream);

/* ================================================================================================
 * Context Encoding (EncNet's Encoding layer, Zhang et al., CVPR 2018) and the SE-loss. For the N pixels x_i (bf16 NHWC,
 * channel stride xcs) of each of B images, K codewords c_k (fp32 [K][D]) and smoothing factors s_k (fp32 [K]):
 *   d²_ik = ‖x_i − c_k‖² (direct differences), a_ik = softmax_k(s_k d²_ik), E_bk = Σ_i a_ik (x_i − c_k).
 * K is a multiple of 8 and at most 32 (one warp lane per codeword), D a multiple of 64 and at most 1024 with K·D <= 16384
 * (the codewords sit in shared memory); anything else is TSB_ERR_UNSUPPORTED. xcs, dxcs: multiples of 8, >= D; x, dx
 * 16-byte aligned. Arithmetic is fp32. Each CTA sums its pixels into its own workspace slot (16 slots per image, so
 * B·16·(K·D + K) floats forward and B·16·(K·D + 2K) backward, independent of N) and the slots are added in a fixed order.
 * ============================================================================================== */
/* E: bf16 [B·D rows][K channels] (row b·D + d), an NHWC tensor with C = K that the BN entry points normalise as is.
 * a, d2: fp32 [B·N][K], saved for the backward (both NULL in inference). sum_a: fp32 [B][K] = Σ_i a_ik. */
int tsb_encoding_fwd(const void* x, int xcs, int B, int N, int D, const float* codewords, const float* scale, int K,
                     float* a, float* d2, float* sum_a, void* E, float* ws, long long ws_floats, tsb_stream_t stream);
/* dE bf16 [B·D][K] like E. With t_ik = dE_k·(x_i − c_k) and g_ik = a_ik (t_ik − Σ_j a_ij t_ij):
 *   dx_i = Σ_k a_ik dE_k + 2 Σ_k g_ik s_k (x_i − c_k)                        (bf16, written)
 *   dcodewords_k += −Σ_b (Σ_i a_ik) dE_bk − 2 s_k Σ_b Σ_i g_ik (x_i − c_k)    (fp32 [K][D], accumulated)
 *   dscale_k     += Σ_b Σ_i g_ik d²_ik                                        (fp32 [K], accumulated) */
int tsb_encoding_bwd(const void* dE, const void* x, int xcs, int B, int N, int D, const float* codewords,
                     const float* scale, int K, const float* a, const float* d2, const float* sum_a, void* dx, int dxcs,
                     float* dcodewords, float* dscale, float* ws, long long ws_floats, tsb_stream_t stream);
/* y[p] = (1/C) Σ_c x[p, c] summed in channel order (bf16 in, bf16 y[npix] out): EncNet's mean over the codewords.
 * bwd: dx[p, c] = dy[p] / C (dy dense bf16 [npix], dx channel stride dxcs >= C). */
int tsb_chan_mean_fwd(const void* x, int xcs, long long npix, int C, void* y, tsb_stream_t stream);
int tsb_chan_mean_bwd(const void* dy, long long npix, int C, void* dx, int dxcs, tsb_stream_t stream);
/* SE-loss: nn.BCELoss(sigmoid(z), presence) with presence[b, c] = any(labels[b] == c) for c in [0, C) (other label values
 * count for nothing). labels int64 [B][HW]; z fp32 [B][C] with row stride zs. presence: uint32 [B][ceil(C/32)] bit words,
 * written (per-CTA shared-memory bitmaps ORed together, so deterministic). *loss: the mean with torch's −100 clamp on
 * the logs; dz_unit (row stride dzs): d loss / d z for a unit upstream gradient. C <= 4096. No host synchronisation. */
int tsb_se_loss_fwd_bwd(const int64_t* labels, int B, long long HW, const float* z, int zs, int C, uint32_t* presence,
                        float* loss, float* dz_unit, int dzs, tsb_stream_t stream);

/* ---- OCNet: fused self-attention over the pixels of each image ------------------------------------------------------
 *   o[b,i,:] = Σ_j softmax_j(scale · q[b,i,:]·k[b,j,:]) · v[b,j,:]     b < B, i, j < N
 * q, k, v, o, dout and the gradients are bf16 rows [B·N][d] (row b·N + i) with channel stride *cs: multiples of 8, every
 * pointer 16-byte aligned; q, k, dq and dk have d = d_k (stride >= d_k), v, o, dout and dv have d = d_v (stride >= d_v).
 * Two (d_k, d_v) pairs are implemented: (256, 256) (OCNet) and (64, 512) (DANet's position attention, whose value side
 * runs in two 256-channel slices); anything else is TSB_ERR_UNSUPPORTED. B·N < 2^31, B <= 65535, 0 < scale < inf.
 * S = q·kᵀ and its softmax are never written to global memory; every output element has one writer, so results are
 * bit-identical from run to run. */
/* lse: fp32 [B·N], m_i + log Σ_j exp(scale·s_ij − m_i) per query row (the softmax normaliser), or NULL (inference). */
int tsb_attention_fwd(const void* q, int qcs, const void* k, int kcs, const void* v, int vcs, void* o, int ocs, float* lse,
                      int B, int N, int dim_k, int dim_v, float scale, tsb_stream_t stream);
/* The gradient from the forward's o and lse. delta_ws: fp32 [B·N] scratch (δ_i = Σ_c dout_ic·o_ic). dk and dv are
 * written; dq is written, or, with dq_accumulate, added to (dq += dQ, rounded once): with dq == dk the shared query/key
 * gradient dQ + dK comes out of one call, since dK is finished before dQ is added. */
int tsb_attention_bwd(const void* q, int qcs, const void* k, int kcs, const void* v, int vcs, const void* o, int ocs,
                      const void* dout, int docs, const float* lse, float* delta_ws, void* dq, int dqcs, void* dk,
                      int dkcs, void* dv, int dvcs, int dq_accumulate, int B, int N, int dim_k, int dim_v, float scale,
                      tsb_stream_t stream);
/* Cross attention (OCRNet's pixel-region relation): Nq queries and Nk keys / values per image,
 *   o[b,i,:] = Σ_j softmax_j(scale · q[b,i,:]·k[b,j,:]) · v[b,j,:]     b < B, i < Nq, j < Nk
 * on the (256, 256) kernels of tsb_attention_*, with their conventions: q, o, dout, dq, lse and delta_ws have B·Nq rows
 * (row b·Nq + i), k, v, dk and dv B·Nk rows (row b·Nk + j). Only (d_k, d_v) = (256, 256); anything else is
 * TSB_ERR_UNSUPPORTED. B·Nq, B·Nk < 2^31, B <= 65535. dq is written (there is no shared query / key form). With
 * Nq = Nk = N the results are those of tsb_attention_* bit for bit. */
int tsb_cross_attention_fwd(const void* q, int qcs, const void* k, int kcs, const void* v, int vcs, void* o, int ocs,
                            float* lse, int B, int Nq, int Nk, int dim_k, int dim_v, float scale, tsb_stream_t stream);
int tsb_cross_attention_bwd(const void* q, int qcs, const void* k, int kcs, const void* v, int vcs, const void* o,
                            int ocs, const void* dout, int docs, const float* lse, float* delta_ws, void* dq, int dqcs,
                            void* dk, int dkcs, void* dv, int dvcs, int B, int Nq, int Nk, int dim_k, int dim_v,
                            float scale, tsb_stream_t stream);

/* ---- OCRNet: soft-max over the pixels of each image (the soft object regions of the SpatialGather module) -------------
 * logits: fp32 NHWC rows [B·N][lcs] (row b·N + n), K valid channels, 1 <= K <= 256, lcs a multiple of 8 and >= K
 * rounded up to 8, 16-byte aligned; channels K..lcs−1 are never used. B·N < 2^31, B <= 65535.
 * fwd: per (b, k) M = max_n l and S = Σ_n exp(l − M) in fp32, into stats (fp32 [B][2][K]: M, then S); P = exp(l − M) / S
 *      rounded once into bf16 P [B·N][Kp] (dense, Kp = K rounded up to 64, channels K..Kp−1 written as exact zeros), an
 *      operand of the per-image tsb_conv2d_* products.
 * bwd: dl[n, k] = P[n, k] · (dP[n, k] − Σ_n' P[n', k] · dP[n', k]) with P recomputed in fp32 from the logits and stats;
 *      dP fp32 [B·N][dpcs], dl fp32 [B·N][dlcs] (channels < K written), strides multiples of 8 and >= K rounded up to 8.
 * Sums over the pixels run over fixed pixel ranges set by N and K whose partials (ws, ws_floats: B · ranges · 2K floats,
 * at most 64 ranges per image until N exceeds 64 · 4 · 256 / ceil(K/8) pixels) are added in a fixed order: bit-identical
 * from run to run and independent of the other images. */
int tsb_spatial_softmax_fwd(const float* logits, int lcs, void* P, float* stats, int B, int N, int K, float* ws,
                            long long ws_floats, tsb_stream_t stream);
int tsb_spatial_softmax_bwd(const float* logits, int lcs, const float* stats, const float* dP, int dpcs, float* dl,
                            int dlcs, int B, int N, int K, float* ws, long long ws_floats, tsb_stream_t stream);

/* ---- DANet: channel attention (CAM) and the learnable-gamma residual --------------------------------------------------
 * CAM per image b with C channels: E = X Xᵀ (fp32 [C][C], tsb_conv2d_wgrad with dy = x), A = softmax_row(rowmax(E) − E),
 * out = A X (a 1x1 tsb_conv2d_fprop with A as the weight). E, dA: fp32 [B][C][C]; A, G: bf16 [B][C][C], row-major.
 * fwd: A from E; t_ij = rowmax_i − E_ij in fp32 as written, exp(t_ij − max_j t_ij) normalised over the row, rounded once.
 * bwd: G = −(dẼ + dẼᵀ), dẼ = A ∘ (dA − Σ_j A_ij dA_ij) (the gradient through rowmax, zero in exact arithmetic, is
 *      dropped). G is exactly symmetric; dX += G·X is then a tsb_conv2d_dgrad with accumulate = 1 and G as the pack.
 *      rowdot_ws: fp32 [B·C] scratch. B <= 65535, C·C <= 2^30. */
int tsb_chan_attn_softmax_fwd(const float* E, void* A, int B, int C, tsb_stream_t stream);
int tsb_chan_attn_softmax_bwd(const void* A, const float* dA, float* rowdot_ws, void* G, int B, int C,
                              tsb_stream_t stream);
/* y = bf16(fmaf(gamma, o, x)) over npix pixels of C channels (DANet's `gamma * out + x`), gamma read on the device from
 * the fp32 parameter (no host synchronisation). bwd: dout = bf16(gamma · dy), and dgamma (fp32 [1]) += Σ dy·o, the
 * per-CTA partials summed in slot order through the workspace (ws, ws_floats). C % 8 == 0; x, o, y, dy, dout bf16 NHWC,
 * 16-byte aligned, channel strides multiples of 8 and >= C. */
int tsb_gamma_residual_fwd(const void* x, int xcs, const void* o, int ocs, const float* gamma, void* y, int ycs,
                           long long npix, int C, tsb_stream_t stream);
int tsb_gamma_residual_bwd(const void* dy, int dycs, const void* o, int ocs, const float* gamma, void* dout, int docs,
                           float* dgamma, long long npix, int C, float* ws, long long ws_floats, tsb_stream_t stream);

/* ================================================================================================
 * Optimiser — fused flat-buffer momentum SGD replacing torch.optim.SGD.step (train.py:86-89,142) with
 * the group semantics of furnace/utils/init_func.py:34-57 (decay / no-decay, 1x / 10x LR):
 *   g = grad*gscale + wd*p ; buf = first ? g : mom*buf + g ; p -= lr*buf      (torch SGD, dampening 0)
 * Segments: seg_end[i] = exclusive end offset (elements) of segment i, with seg_lr[i], seg_wd[i]
 * (device arrays, updated every iteration by the host without sync).
 * ============================================================================================== */
int tsb_sgd_flat(float* param, const float* grad, float* mom_buf, long long n, const long long* seg_end,
                 const float* seg_lr, const float* seg_wd, int nseg, float momentum, float gscale, int first_step,
                 tsb_stream_t stream);
/* same update, and additionally param_bf16[i] = bf16(param[i]) for the whole flat buffer: conv weights are stored
 * KRSC, so the bf16 copy IS the fprop/wgrad weight operand of every layer (no per-layer pack launches next step) */
int tsb_sgd_flat_pack(float* param, const float* grad, float* mom_buf, long long n, const long long* seg_end,
                      const float* seg_lr, const float* seg_wd, int nseg, float momentum, float gscale, int first_step,
                      void* param_bf16, tsb_stream_t stream);
/* all dgrad weight operands in one launch: for tensor t (descriptor {int64 off; int32 K, RS, C, tiles_k, tiles_c, pad}
 * = 32 bytes, tiles_* = ceil(./32)), wt_flat[off + ((c*RS + RS-1-rs)*K + k)] = wb_flat[off + ((k*RS + rs)*C + c)].
 * block_start[t] = first block of tensor t (blocks per tensor = RS * tiles_k * tiles_c), nblocks = their sum. */
int tsb_pack_wt_multi(const void* wb_flat_bf16, void* wt_flat_bf16, const void* desc, const int* block_start,
                      int ntensors, int nblocks, tsb_stream_t stream);

/* ================================================================================================
 * Fused bilinear up-sampling (align_corners=True, to H x W) + cross-entropy(mean over valid pixels, ignore index) for many
 * classes (1 <= C <= 152) — replaces F.interpolate → log_softmax → nn.CrossEntropyLoss of the PSPNet / PSANet heads
 * (model/pspnet/ade.pspnet.R101_v1c/network.py:46-57, model/psanet/.../network.py:46-55); the [N,C,H,W] logits are never written.
 * logits_lo: fp32 NHWC [N,h,w,cs]; lse: fp32 [N*H*W] (log-sum-exp per pixel, kept for the backward); state: 8 words
 * (zeroed inside): {double Σ loss, valid count, loss, 1/count}. backward: dlogits_lo (fp32 NHWC, caller-zeroed) +=
 * d loss / d logits_lo · *gscale.
 * ============================================================================================== */
int tsb_ce_up_fwd(const float* logits_lo, int cs, int h, int w, const int64_t* labels, int N, int C, int H, int W,
                  int ignore_label, float* lse, uint32_t* state, float* loss_out, tsb_stream_t stream);
int tsb_ce_up_bwd(const float* logits_lo, int cs, int h, int w, const int64_t* labels, const float* lse, int N, int C,
                  int H, int W, int ignore_label, const uint32_t* state, const float* gscale, float* dlogits_lo,
                  tsb_stream_t stream);

/* ================================================================================================
 * Sigmoid focal loss (DFN border branch) — SigmoidFocalLoss.forward loss_opr.py:23-45, reproduced
 * as is (incl. the sigmoid-inside-logsumexp quirk, SURVEY App. A2). pred fp32/bf16 [n], target int64.
 * ============================================================================================== */
int tsb_sigmoid_focal_fwd_bwd(const void* pred, int dtype, const int64_t* target, long long n, int ignore_label,
                              float gamma, float alpha, float* loss_mean, void* dpred_unit, tsb_stream_t stream);

/* ================================================================================================
 * Device-initiated all-reduce of small fp32 vectors over NVLink peer memory — the SyncBatchNorm statistics exchange
 * (replaces the per-layer all-reduce inside apex.parallel.SyncBatchNorm, model/bisenet/cityscapes.bisenet.R18/
 * train.py:54-55). The caller owns ONE symmetric buffer per rank of tsb_p2p_buffer_bytes() bytes, zero-filled before
 * the first exchange ({value, sequence} pairs: no fences, no flag resets), and passes the peer-mapped base address of every rank's buffer (host array `peer_bases[world]`).
 * `seq` = 1, 2, 3, ... must be the same on all ranks for the same exchange; alternatively `seq_dev` points at a device
 * counter (zero-initialised, private to this buffer) that the kernel pre-increments — the form a captured CUDA graph can
 * replay. vals[n] (n % 4 == 0, n <= slot_floats) is
 * replaced by the sum over ranks (rank order: identical bits everywhere). Optional acc_hi/acc_lo[n/2]: the LOCAL
 * halves are accumulated first (acc_lo += vals[0:n/2], acc_hi += vals[n/2:n]) — dbeta / dgamma of the BN backward.
 * ============================================================================================== */
#define TSB_P2P_MAX_WORLD 16
size_t tsb_p2p_buffer_bytes(int world, int nslots, int slot_floats);
int tsb_p2p_allreduce_sum(float* vals, int n, const unsigned long long* peer_bases, int rank, int world,
                          unsigned int seq, unsigned int* seq_dev, int nslots, int slot_floats, float* acc_hi,
                          float* acc_lo, tsb_stream_t stream);

/* ================================================================================================
 * Training-time input pipeline (SURVEY §8 f4) — replaces TrainPre.__call__, model/bisenet/cityscapes.bisenet.R18/
 * dataloader.py:16-33 (random_mirror, random_scale = cv2.resize INTER_LINEAR / INTER_NEAREST, normalize,
 * random_crop_pad_to_shape, transpose; furnace/utils/img_utils.py:24-78,118-125,140-145,181-187), one fused pass from the
 * decoded uint8 frames to the fp32 [n,3,crop_h,crop_w] batch and the int64 [n,crop_h,crop_w] labels. Bit-exact with the
 * cv2 path (fixed-point 8-bit INTER_LINEAR). The random draws are the caller's (host).
 * samples_dev: device array of n rows x 10 int64: {img ptr (uint8 [H,W,3]), gt ptr (uint8 [H,W]), H, W, flip (0/1),
 * sh, sw (size after random_scale), pos_h, pos_w (crop origin in the scaled image), 0}. reverse_channels: the frame is
 * BGR as decoded and the output planes are RGB (BaseDataset.py:45). lut: [3][256] normalised values per output plane.
 * ============================================================================================== */
int tsb_train_preprocess(const long long* samples_dev, int n, int crop_h, int crop_w, int reverse_channels,
                         const float* lut, float img_pad, int gt_pad, float* out_img, long long* out_gt,
                         tsb_stream_t stream);

/* DFN border labels ('aux_label', model/dfn/cityscapes.dfn.R101_v1c/dataloader.py:15-29,38-42): cv2.Canny(apertureSize=7,
 * thresholds 5, 5) of the scaled label map with 255 → 0, cv2.dilate(7x7 rect), 255 → 1, cropped / padded (255) like the label.
 * Same sample descriptors as tsb_train_preprocess; integer arithmetic throughout (bit-exact vs cv2). The workspace is the
 * caller's (tsb_edge_labels_workspace_bytes, 256-byte aligned). */
size_t tsb_edge_labels_workspace_bytes(int n, int crop_h, int crop_w);
int tsb_edge_labels(const long long* samples_dev, int n, int crop_h, int crop_w, int gt_pad, void* workspace,
                    size_t workspace_bytes, long long* out_aux, tsb_stream_t stream);

/* ================================================================================================
 * Evaluator (SURVEY §8 f2) — what Evaluator.sliding_eval / scale_process / whole_eval (torchseg_b200/engine/evaluator.py,
 * TorchSeg furnace/engine/evaluator.py:163-251) do around the network forward, bit-identical to their cv2 / numpy / torch
 * host path: one frame, one scale per call.
 *
 * tsb_eval_windows: uint8 HWC frame src[H][W][cin] (cin 1 = grey, replicated to 3 planes, or 3) → cv2.resize(src, None,
 * fx, fx, INTER_LINEAR) of size (sh, sw) = (rint(H*fx), rint(W*fx)) — fixed point with coefficient scale 1/fx, INTER_AREA
 * when 1/fx == 2, a copy when (sh, sw) == (H, W) (fx is then ignored) — placed at (top, left) of a padded canvas, then
 * normalised through lut[3][256] (utils.gpu_pipeline.normalize_lut). Canvas pixels outside the frame are lut[c][0]
 * (pad_zero = 0: the uint8 frame is padded, then normalised) or 0.0f (pad_zero = 1: normalised, then padded).
 * out[n][3][wh][ww] fp32 = the canvas windows whose top-left corners are corners[n][2] = {y, x} (int32, device), mirrored
 * left-right when `mirror`.
 *
 * tsb_eval_accumulate: lp[n][C][wh][ww] fp32 network log-probs of those windows and optionally lp_flip, the log-probs of
 * the mirrored windows → acc[C][acc_h][acc_w] += exp(lp + mirror(lp_flip)) per window (accurate expf, fp32). Overlapping
 * windows are SUMMED in window order (no atomics); pixels covered by no window are not touched.
 *
 * tsb_eval_resize_add: src = a strided fp32 [C][h][w] view (element (c, y, x) at c*plane_stride + y*row_stride + x)
 * → cv2.resize(src as HWC, (W, H), INTER_LINEAR) in fp32 (a copy at the same size, INTER_AREA at an exact 2x down-scale)
 * → total[C][H][W] (fp64) += resized. With pred != NULL the total is not stored; pred[H][W] (int64) receives the first
 * index of the maximum of the updated total over C (numpy argmax). Bit-exact with cv2 for C not in {1, 3, 4}.
 * ============================================================================================== */
int tsb_eval_windows(const uint8_t* src, int H, int W, int cin, double fx, int sh, int sw, int top, int left,
                     const float* lut, int pad_zero, const int* corners, int n, int wh, int ww, int mirror, float* out,
                     tsb_stream_t stream);
int tsb_eval_accumulate(const float* lp, const float* lp_flip, const int* corners, int n, int C, int wh, int ww,
                        float* acc, int acc_h, int acc_w, tsb_stream_t stream);
int tsb_eval_resize_add(const float* src, int C, int h, int w, long long plane_stride, long long row_stride,
                        double* total, int H, int W, int64_t* pred, tsb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* TSB_H_ */
