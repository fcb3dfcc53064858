/* effdet_b200 -- C ABI of the H100-native (sm_90a) EfficientDet forward/backward hot path.
 *
 * The reference (toandaominh1997/EfficientDet.Pytorch @ fbe56e5) is 100% Python and has NO
 * native boundary of its own: every entry point below replaces a chain of ATen/cuDNN/torchvision
 * calls made by the cited reference lines.  The reference-side binding is the ctypes stub in
 * INTEGRATION.md (a Python reference binds through ctypes/`torch.autograd.Function`).
 *
 * Conventions
 *   - all tensors are fp32, dense, NHWC ("[B,H,W,C]") unless a comment says otherwise;
 *     pointers are device pointers owned by the caller (PyTorch's caching allocator);
 *   - nothing here allocates, frees, retains a pointer after return, or synchronises the device;
 *   - every call takes the CUDA device ordinal and the cudaStream_t to launch on;
 *   - return value 0 = launched; negative = error, text via effdet_last_error() (thread-local);
 *   - "+=" in a comment means the kernel ACCUMULATES into a caller-initialised buffer.
 */
#ifndef EFFDET_B200_H
#define EFFDET_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EFFDET_OK 0
#define EFFDET_ERR_ARG (-1)
#define EFFDET_ERR_LAUNCH (-2)
#define EFFDET_ERR_DEVICE (-3)
#define EFFDET_ERR_UNSUPPORTED (-4)

#define EFFDET_ACT_NONE 0
#define EFFDET_ACT_RELU 1
#define EFFDET_ACT_SWISH 2
#define EFFDET_ACT_SIGMOID 3

#define EFFDET_FUSE_UP 0   /* second input is the coarser map, nearest x2 (models/bifpn.py:189) */
#define EFFDET_FUSE_POOL 1 /* second input is the finer map, 2x2/2 max-pool (models/bifpn.py:195,200) */

typedef void* effdet_stream_t; /* cudaStream_t */

int effdet_version(void);
const char* effdet_last_error(void);
uint64_t effdet_launch_count(void); /* kernels launched by this library in this process */
void effdet_reset_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Dense convolution, k in {1,3}, stride 1, "same" zero padding, as an implicit GEMM
 *   y[b,p,n] = epilogue( sum_{tap,c} x[b, p+tap, c] * a_scale[b,c] * w[tap,c,n] )
 * Replaces F.conv2d + bias + BatchNorm(eval) + activation + residual in
 *   ConvModule.forward           models/module.py:507-515   (neck 1x1/3x3, head 3x3 + ReLU)
 *   RetinaHead.forward_single    models/retinahead.py:109-129 (retina_cls + sigmoid, retina_reg)
 *   MBConvBlock.forward          models/efficientnet.py:85,96-104 (expand / project 1x1)
 * and, with the flipped/transposed weight pack, the data gradient of each of them.
 * Epilogue order: v = acc + bias;  z = v (optional save);  v = v*scale + shift;  v = act(v);
 *                 v *= row_scale[b];  v += residual;  v = mask_src > 0 ? v : 0;  y = v.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    const float* x;        int64_t x_bstride; /* [B,H,W,Cin]; elements between consecutive images */
    const float* w;                            /* packed [k*k][Cin][Cout] (effdet_pack_conv_weight) */
    float* y;              int64_t y_bstride; /* [B,H,W,Cout]; stride lets the head write straight
                                                  into the concatenated [B, sum(HWA), K] buffer
                                                  (kills torch.cat, models/efficientdet.py:64-65) */
    float* z;                                  /* optional raw (pre-affine) output, y's layout */
    const float* bias;                         /* [Cout] or NULL */
    const float* scale;    const float* shift; /* [Cout] eval-BN affine, or both NULL */
    const float* a_scale;                      /* [B,Cin] squeeze-excite gate on the input, or NULL */
    const float* row_scale;                    /* [B] drop-connect keep/keep_prob, or NULL */
    const float* residual; int64_t r_bstride;  /* [B,H,W,Cout] added last, or NULL */
    const float* mask_src; int64_t m_bstride;  /* [B,H,W,Cout]: ReLU-backward mask source, or NULL */
    int32_t B, H, W, Cin, Cout, ksize, act;
    const void* w_tc;      /* optional bf16 hi/lo planes from effdet_pack_conv_weight_tc: when set (and the
                              epilogue needs only bias/act/residual/mask) the layer runs on the wgmma
                              tensor cores as a bf16x3 split-precision implicit GEMM (~2^-16 per product; see tc_single) */
    const float* in_scale; const float* in_shift; /* [Cin] or both NULL: the input is a RAW conv output and the
                              operand is swish(x*in_scale+in_shift) (eval-BN + swish applied while the tile is
                              staged, so the activated tensor never exists in HBM: MemoryEfficientSwish keeps
                              only the pre-activation too, models/utils.py:31-42); applied before a_scale */
    const void* x_planes;  /* optional (1x1 convs, tensor-core path): the input PRE-SPLIT into bf16 planes
                              [2][B*H*W][Cin] (plane 0 = hi, plane 1 = lo, x ~= hi + lo; Cin % 8 == 0), as written by
                              effdet_dwconv_bwd_fused; x may then be NULL */
    int32_t tc_single;     /* 1: when this call runs on the tensor cores, one bf16 product per multiply-add (hi(x)*hi(w),
                              fp32 accumulation) instead of bf16x3; 3x3 convolutions only (ksize 1 -> EFFDET_ERR_ARG).
                              0 keeps the bf16x3 split precision. Needs w_tc (else EFFDET_ERR_ARG); every level of a
                              multi-level call must pass the same value */
} effdet_conv_args;
int effdet_conv2d(const effdet_conv_args* a, int device, effdet_stream_t stream);
/* The same convolution (shared w / w_tc / bias / act, channels, ksize) applied to `nlevels` (<= 8) feature maps of
 * different sizes in ONE launch -- RetinaHead.forward runs every layer on P3..P7 with the same weights
 * (models/retinahead.py:131-132).  Falls back to one launch per level in exact-fp32 mode. */
int effdet_conv2d_multi(const effdet_conv_args* levels, int nlevels, int device, effdet_stream_t stream);

/* Weight gradient (and optional bias gradient) of the convolution above.
 *   dw[n,c,ky,kx] += sum_{b,p} x[b,p+tap,c]*a_scale[b,c] * dy[b,p,n]     (OIHW, as .grad)
 *   dbias[n]      += sum_{b,p} dy[b,p,n]
 * Replaces cuDNN bwd-filter reached through autograd (SURVEY.md K13). */
typedef struct {
    const float* x;   int64_t x_bstride;
    const float* dy;  int64_t dy_bstride;
    float* dw;        /* [Cout,Cin,k,k]  += */
    float* dbias;     /* [Cout] += , or NULL */
    const float* a_scale;
    int32_t B, H, W, Cin, Cout, ksize;
    int32_t precision;     /* 0: exact fp32 on the CUDA cores; 1: bf16x3 on the wgmma tensor cores */
    void* ws_x;            /* precision 1: bf16 workspaces for the pre-split operands, */
    void* ws_dy;           /*   2*B*H*W*kpad(Cin) resp. 2*B*H*W*kpad(Cout) elements (TMA-fed kernel);
                              NULL -> the gather-producer tensor-core kernel is used instead */
    const float* in_scale; const float* in_shift; /* [Cin] or both NULL: x is a raw conv output, the operand is
                              swish(x*in_scale+in_shift)*a_scale (see effdet_conv_args) */
    const void* dy_planes; /* optional (precision 1): dy PRE-SPLIT into bf16 planes [2][B*H*W][pitch(Cout)], as written
                              by effdet_dwconv_bwd_fused / effdet_conv_planes_multi: no split pass over dy, ws_dy unused,
                              dy may be NULL (dbias must be NULL) */
    const void* x_planes;  /* optional, likewise for x ([2][B*H*W][pitch(Cin)]; no a_scale / in_scale): ws_x unused */
    int32_t tc_single;     /* 1: when this call runs on the tensor cores, one bf16 product per multiply-add (hi(x)*hi(w),
                              fp32 accumulation) instead of bf16x3; 3x3 convolutions only (ksize 1 -> EFFDET_ERR_ARG).
                              0 keeps the bf16x3 split precision. Needs precision 1 (else EFFDET_ERR_ARG); every
                              level of a multi-level call must pass the same value */
    void* ws_dw;           /* fp32 workspace of 4*9*Cout*Cin bytes, 16-byte aligned, that the tensor-core kernels of a 3x3
                              weight gradient reduce into (tap-major [9][Cout][Cin]) before one fold adds it to dw; needed
                              when a 3x3 call takes a tensor-core route, else unused.  A multi-level call uses the first
                              level's.  1x1 tensor-core weight gradients reduce straight into dw */
} effdet_wgrad_args;
int effdet_conv2d_wgrad(const effdet_wgrad_args* a, int device, effdet_stream_t stream);
/* Weight gradient of one shared-weight layer accumulated over `nlevels` feature maps in one launch (all levels
 * must name the same dw / dbias); falls back to one launch per level when a level cannot use the TMA path. */
int effdet_conv2d_wgrad_multi(const effdet_wgrad_args* levels, int nlevels, int device, effdet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * The same dense convolution with activations kept in HBM as bf16 hi/lo PLANES [2][B][H][W][pitch] (x ~= hi + lo, the
 * tensor-core operand format; pitch = channels rounded up to 8): the RetinaHead towers end to end
 * (models/retinahead.py:67-132).  The im2col gather is a TMA load (5-D tensor map, tap = coordinate offset, hardware
 * zero fill = padding), the epilogue writes the next layer's planes (and / or fp32), so no layer re-splits its input and
 * no weight gradient needs a split pass.  All levels of one call share weights / bias (RetinaHead.forward).
 *   epilogue: v = acc + bias; v = act(v); v += residual; v = mask > 0 ? v : 0; store planes and / or fp32;
 *             colsum[n] += sum over pixels of v   (the bias gradient of the layer that produced this layer's input
 *             gradient -- a data-gradient launch hands it over for free)
 * The mask is given either as the forward's planes (mask_planes) or as the bits a ReLU forward wrote (mask_bits), not
 * both.  y_mask / mask_bits: uint32 [B][H][W][(Cout + 31) / 32], bit c % 32 of word c / 32 set <=> the value stored in
 * the planes for channel c is > 0 (words past Cout's last channel are zero).
 * Needs effdet_wgrad_tc_geometry_ok(B,H,W) for every level; with colsum, 4 * Cout bytes of shared memory beyond the
 * kernel's own (Cout up to about 3200).
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    const void* x_planes;                       /* [2][B][H][W][pitch(Cin)] bf16 */
    const void* w_tc;                           /* effdet_pack_conv_weight_tc pack (forward or data-gradient) */
    const float* bias;                          /* [Cout] or NULL */
    float* y;              int64_t y_bstride;   /* fp32 output [B][H*W][Cout] (image stride y_bstride) or NULL */
    void* y_planes;                             /* planes output [2][B][H][W][pitch(Cout)] or NULL */
    const void* mask_planes;                    /* ReLU-backward mask source, planes of pitch(Cout), or NULL */
    const float* residual; int64_t r_bstride;   /* fp32 [B][H*W][Cout] added before the mask, or NULL */
    float* colsum;                              /* [Cout] += or NULL */
    int32_t B, H, W, Cin, Cout, ksize, act;
    int32_t tc_single;                          /* 1: one bf16 product per multiply-add (hi planes only), as in
                                                   effdet_conv_args; 3x3 only, the same on every level */
    void* y_mask;                               /* ReLU bits of the stored planes (act RELU with y_planes) or NULL */
    const void* mask_bits;                      /* ReLU-backward mask as y_mask wrote it, or NULL */
} effdet_conv_planes_args;
int effdet_conv_planes_multi(const effdet_conv_planes_args* levels, int nlevels, int device, effdet_stream_t stream);
/* fp32 [B][HW][C] (image stride x_bstride) -> planes [2][B*HW][pitch(C)]; with prob != NULL the value is first
 * multiplied by p*(1-p) (sigmoid backward of the classification head, models/retinahead.py:121); with colsum != NULL
 * the per-channel sums of what was written are accumulated (bias gradient) in the same pass */
int effdet_to_planes(const float* x, int64_t x_bstride, const float* prob, int64_t p_bstride, void* planes, float* colsum,
                     int B, int HW, int C, int device, effdet_stream_t stream);

/* OIHW -> [k*k][Cin][Cout] (forward) and, if w_dgrad != NULL, the 180-degree-rotated transpose
 * [k*k][Cout][Cin] that turns the data gradient into the same implicit GEMM. */
int effdet_pack_conv_weight(const float* w_oihw, float* w_fwd, float* w_dgrad, int Cout, int Cin, int ksize,
                            int device, effdet_stream_t stream);

/* OIHW fp32 -> pre-split bf16 planes for the tensor-core path, K-major and zero padded:
 *   w_fwd   [2][Cout][k*k][kpad(Cin)]   (plane 0 = hi, plane 1 = lo, w ~= hi + lo)
 *   w_dgrad [2][Cin][k*k][kpad(Cout)]   (rotated 180 degrees and transposed), may be NULL
 * kpad(c) = effdet_conv_tc_kpad(c) = c rounded up to a multiple of 64. */
int effdet_conv_tc_kpad(int channels);
/* 1 when the TMA-fed tensor-core weight-gradient kernel can tile a [B,H,W,*] map into pixel boxes (required before
 * handing it pre-split operands, effdet_wgrad_args.dy_planes); no device work */
int effdet_wgrad_tc_geometry_ok(int B, int H, int W);
int effdet_pack_conv_weight_tc(const float* w_oihw, void* w_fwd, void* w_dgrad, int Cout, int Cin, int ksize,
                               int device, effdet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Stem: 3x3 stride-2 conv on the NCHW image with TF-"SAME" pad (0,1,0,1), eval-BN, swish.
 * Replaces EfficientNet.extract_features stem, models/efficientnet.py:193 (+ utils.py:126-155).
 *   x [B,3,H,W] NCHW  ->  z (raw conv) and y = swish(z*scale+shift), both [B,H/2,W/2,C0] NHWC
 *   (y may be NULL: the consumer applies BN+swish while staging z)
 * ------------------------------------------------------------------------------------------ */
int effdet_stem_fwd(const float* x_nchw, const float* w_oihw, const float* scale, const float* shift, float* z,
                    float* y, int B, int H, int W, int C0, int device, effdet_stream_t stream);
/* dw[C0,3,3,3] += sum x * dz   (the image needs no data gradient) */
int effdet_stem_wgrad(const float* x_nchw, const float* dz, float* dw_oihw, int B, int H, int W, int C0,
                      int device, effdet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Depthwise phase of MBConvBlock.forward with only PRE-activations in HBM (the reference's
 * MemoryEfficientSwish saves the pre-activation only, models/utils.py:31-42; block: models/efficientnet.py:85-94).
 * Depthwise k x k (k in {3,5}), stride in {1,2}, w_kkc = [k][k][C] (effdet_pack_dw_weight).
 * Pads must be the reference's static ones (models/utils.py:126-149): k3s1 1, k5s1 2, k3s2 0, k5s2 1 (top/left).
 *   fwd: a0 = in_scale ? swish(x*in_scale+in_shift) : x        (BN0+swish applied while the tile is staged)
 *        z  = depthwise(a0)                                    raw output, the only tensor written
 *        se_sum[b,c] += se_alpha * sum_pixels swish(z*scale+shift)   (squeeze-excite mean, an epilogue by-product)
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    const float* x;                                /* [B,H,W,C] raw expand-conv output z0, or the block input */
    const float* in_scale; const float* in_shift;  /* [C] folded BN0, or both NULL (x used as is) */
    const float* w_kkc;                            /* [k][k][C] */
    const float* scale;    const float* shift;     /* [C] folded BN1 */
    float* z;                                      /* [B,Ho,Wo,C] */
    float* se_sum;                                 /* [B,C] += se_alpha * sum  (se_alpha = 1/(Ho*Wo) makes it the SE mean) */
    int32_t B, H, W, C, k, stride, pad_t, pad_l, Ho, Wo;
    float se_alpha;
} effdet_dw_fwd_args;
int effdet_dwconv_fwd_fused(const effdet_dw_fwd_args* a, int device, effdet_stream_t stream);
/*   bwd, one pass over the expanded tensor (replaces BN1-swish backward + depthwise weight/data gradient + BN0-swish
 *   backward, models/utils.py:38-42 through autograd):
 *        du1 = (dq*gate + dmean*inv_hw) * swish'(z1*scale1+shift1);  dgamma1 += sum du1*(z1-mean1)*rstd1;  dbeta1 += sum du1
 *        dz1 = du1*scale1  (kept on chip);  da0 = depthwise^T(dz1);  dw[c,ky,kx] += sum a0 * dz1
 *        scale0 ? { du0 = da0*swish'(x*scale0+shift0); dgamma0, dbeta0 += ...; dx = du0*scale0 } : dx = da0 */
typedef struct {
    const float* dq;       /* [B,Ho,Wo,C] gradient w.r.t. (a1*gate), i.e. the project conv's data gradient */
    const float* z1;       /* [B,Ho,Wo,C] raw depthwise output */
    const float* gate;     const float* dmean;   /* [B,C] SE gate, gradient w.r.t. the SE mean */
    const float* scale1;   const float* shift1;  const float* mean1;  const float* rstd1;   /* [C] BN1 */
    const float* x;        /* [B,H,W,C] raw z0 (scale0 != NULL) or the block input */
    const float* scale0;   const float* shift0;  const float* mean0;  const float* rstd0;   /* [C] BN0 or all NULL */
    const float* w_kkc;    /* [k][k][C] */
    float* dx;             /* [B,H,W,C] */
    float* dw;             /* [C,1,k,k] += */
    float* dgamma1; float* dbeta1; float* dgamma0; float* dbeta0;   /* [C] += (BN0 ones may be NULL without BN0) */
    float inv_hw;          /* 1/(Ho*Wo) */
    int32_t B, H, W, C, k, stride, pad_t, pad_l, Ho, Wo;
    void* dx_planes;       /* optional: write dx as bf16 hi/lo planes [2][B*H*W][C] (dx ~= hi + lo) INSTEAD of fp32 dx
                              (dx may then be NULL): the form the tensor-core data / weight gradients of the expand conv
                              consume directly (effdet_conv_args.x_planes, effdet_wgrad_args.dy_planes); C % 8 == 0 */
} effdet_dw_bwd_args;
int effdet_dwconv_bwd_fused(const effdet_dw_bwd_args* a, int device, effdet_stream_t stream);
/* depthwise weight [C,1,k,k] -> w_kkc [k][k][C] */
int effdet_pack_dw_weight(const float* w_c1kk, float* w_kkc, int C, int k, int device, effdet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Backward of  y = act(BN_eval(z)) [* row_scale]  with frozen statistics but trainable affine
 * (models/efficientdet.py:88-92; swish backward models/utils.py:38-42):
 *   g  = dy*row_scale[b]            (or, SE mode:  g = dy*gate[b,c] + dmean[b,c]*inv_hw)
 *   du = g * act'(z*scale+shift);  dgamma += sum du*(z-mean)*rstd;  dbeta += sum du;  dz = du*scale
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    const float* dy;    /* [B,HW,C] */
    const float* z;     /* [B,HW,C] raw conv output */
    float* dz;          /* [B,HW,C] */
    const float* scale; const float* shift; const float* mean; const float* rstd; /* [C] */
    float* dgamma;      float* dbeta;   /* [C] += */
    const float* row_scale; /* [B] or NULL */
    const float* gate;      /* [B,C] or NULL */
    const float* dmean;     /* [B,C] or NULL */
    float inv_hw;
    int32_t B, HW, C, act;  /* act: EFFDET_ACT_NONE or EFFDET_ACT_SWISH */
} effdet_bnact_bwd_args;
int effdet_bnact_bwd(const effdet_bnact_bwd_args* a, int device, effdet_stream_t stream);

/* Frozen BatchNorm2d (eval mode even while training, models/efficientdet.py:88-92) folded to a
 * per-channel affine: rstd = 1/sqrt(var+eps), scale = gamma*rstd, shift = beta - mean*scale. */
int effdet_bn_fold(const float* gamma, const float* beta, const float* mean, const float* var, float eps, float* scale,
                   float* shift, float* rstd, int C, int device, effdet_stream_t stream);
/* out = a + b (skip-connection gradient join) ;  dz = y > 0 ? dy : 0 (stand-alone ReLU backward) */
int effdet_add(const float* a, const float* b, float* out, int64_t n, int device, effdet_stream_t stream);
int effdet_relu_bwd(const float* dy, const float* y, float* dz, int64_t n, int device, effdet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Squeeze-excite (models/efficientnet.py:90-94).
 *   effdet_spatial_reduce_act : out[b,c] += alpha * sum_hw a[b,hw,c] * swish(z[b,hw,c]*scale[c]+shift[c])
 *                               (gradient w.r.t. the SE gate from the raw depthwise output: the activated tensor is
 *                               recomputed, not stored)
 *   effdet_se_gate_fwd        : s_pre = W1*mean+b1 ; gate = sigmoid(W2*swish(s_pre)+b2)
 *   effdet_se_gate_bwd        : given dgate -> dmean, and += into dW1,db1,dW2,db2
 * W1 = _se_reduce.weight [S,C], W2 = _se_expand.weight [C,S].
 * ------------------------------------------------------------------------------------------ */
int effdet_spatial_reduce_act(const float* a, const float* z, const float* scale, const float* shift, float* out,
                              float alpha, int B, int HW, int C, int device, effdet_stream_t stream);
int effdet_se_gate_fwd(const float* mean, const float* w1, const float* b1, const float* w2, const float* b2,
                       float* s_pre, float* gate, int B, int C, int S, int device, effdet_stream_t stream);
int effdet_se_gate_bwd(const float* dgate, const float* mean, const float* s_pre, const float* gate,
                       const float* w1, const float* w2, float* dmean, float* dw1, float* db1, float* dw2,
                       float* db2, float* ws /* B*(C+S) floats of scratch */, int B, int C, int S, int device,
                       effdet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * BiFPN fast-normalised fusion node input (BiFPNModule.forward, models/bifpn.py:177-201):
 *   r = relu(w_col); n = r/(sum r + eps); out = sum_j n_j*in_j / (sum_j n_j + eps)
 *   in_0 = a; in_1 = up2(b) or maxpool2(b); in_2 = c (3-input nodes only)
 * The raw weight column is read as w[j*w_stride], j < (c ? 3 : 2).
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    const float* a; const float* b; const float* c;
    const float* w; int32_t w_stride; float eps;
    float* out;
    int32_t B, H, W, C, mode; /* H,W = resolution of a/out */
    void* out_planes;         /* optional: the fused map as bf16 hi/lo planes [2][B*H*W][pitch(C)] (the node conv's TMA
                                 operand, effdet_conv_planes_multi); `out` may then be NULL */
} effdet_fuse_args;
int effdet_bifpn_fuse_fwd(const effdet_fuse_args* a, int device, effdet_stream_t stream);

typedef struct {
    const float* dout;
    const float* a; const float* b; const float* c;
    const float* w; int32_t w_stride; float eps;
    float* da; float* db; float* dc;  /* input gradients (dc NULL for 2-input nodes) */
    int32_t acc_a, acc_b, acc_c;      /* 0: overwrite, 1: += */
    float* dw;                        /* gradient of the raw weights, indexed like w, += */
    float* scratch;                   /* [4] floats, zero on entry */
    int32_t B, H, W, C, mode;
} effdet_fuse_bwd_args;
int effdet_bifpn_fuse_bwd(const effdet_fuse_bwd_args* a, int device, effdet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * FocalLoss.forward (models/losses.py:32-152): IoU assignment + focal BCE + smooth-L1, no host
 * sync, no per-image Python loop.
 *   cls [B,A,K] probabilities, reg [B,A,4], anchors [A,4] (x1,y1,x2,y2), annots [B,G,5] (-1 pad)
 *   fwd: losses[0] = mean_b cls_loss_b, losses[1] = mean_b reg_loss_b;
 *        assign_ws [B,A] int32 (>=0 matched annotation row, -1 background, -2 ignored, -3 image
 *        without boxes) and stats_ws [B,4] float (npos, cls_sum, reg_sum, -) are kept for bwd.
 *   bwd: dcls = gout[0] * d losses[0]/d cls ; dreg = gout[1] * d losses[1]/d reg
 *        (gout: the two upstream gradients, read from DEVICE memory -> no sync).
 * ------------------------------------------------------------------------------------------ */
int effdet_focal_loss_fwd(const float* cls, const float* reg, const float* anchors, const float* annots,
                          float* losses, int32_t* assign_ws, float* stats_ws, int B, int A, int K, int G,
                          float alpha, float gamma, int device, effdet_stream_t stream);
int effdet_focal_loss_bwd(const float* cls, const float* reg, const float* anchors, const float* annots,
                          const float* gout, const int32_t* assign_ws, const float* stats_ws, float* dcls,
                          float* dreg, int B, int A, int K, int G, float alpha, float gamma, int device,
                          effdet_stream_t stream);
/* The same loss with the image and annotation counts in DEVICE memory, for any G >= 1 (the table is staged in
 * chunks of 256 rows; an anchor's first maximum holds across chunks).
 *   counts [1+B] int32: counts[0] = n_img (1..B), counts[1+b] = rows of image b that are read (0..G); values outside
 *          those ranges are clamped.  Rows at or past counts[1+b] are never read, rows labelled -1 before it are skipped.
 *   Images b >= n_img read nothing of cls, reg or annots: assign_ws -3, zero stats, dcls and dreg exactly 0.
 *   losses and gradient scales average over n_img instead of B: gout[0] / (max(npos,1) * n_img), gout[1] / (4 npos n_img).
 *   Refused before any launch: null pointers, B outside 1..65535, G < 1 (or G * 5 beyond int). */
int effdet_focal_loss_counted_fwd(const float* cls, const float* reg, const float* anchors, const float* annots,
                                  const int32_t* counts, float* losses, int32_t* assign_ws, float* stats_ws, int B, int A,
                                  int K, int G, float alpha, float gamma, int device, effdet_stream_t stream);
int effdet_focal_loss_counted_bwd(const float* cls, const float* reg, const float* anchors, const float* annots,
                                  const int32_t* counts, const float* gout, const int32_t* assign_ws, const float* stats_ws,
                                  float* dcls, float* dreg, int B, int A, int K, int G, float alpha, float gamma, int device,
                                  effdet_stream_t stream);
/* A ragged collated batch annots [B,G,5] (-1 padded) into a static table out [Bcap,Gcap,5] and its counts [1+Bcap]:
 * per image the rows whose label is not -1, in their order, then -1 rows; counts[1+b] = rows kept (0 for b >= B),
 * counts[0] = B.  No host read.  Refused before the launch: B outside 1..Bcap, G outside 1..Gcap, Bcap > 65535. */
int effdet_pack_annots(const float* annots, int B, int G, float* out, int32_t* counts, int Bcap, int Gcap, int device,
                       effdet_stream_t stream);
/* y = g * p*(1-p) (sigmoid backward) ; y may alias g */
int effdet_sigmoid_bwd(const float* g, const float* p, float* y, int64_t n, int device, effdet_stream_t stream);
/* ------------------------------------------------------------------------------------------
 * Inference post-processing (models/efficientdet.py:70-86, models/module.py:24-67, torchvision.ops.nms):
 * decode + clip + class max + threshold + sort + greedy NMS for a batch of B images in one set of
 * launches, all on the device.  The per-image counts stay in device memory and no launch's grid
 * depends on them, so the three calls can be captured in a CUDA graph.
 *   cls [B,A,K], reg [B,A,4] (16-byte aligned), anchors [A,4] shared by all images (16-byte aligned)
 *   boxes [B,A,4] (16-byte aligned), scores [B,A], classes [B,A] int32: every anchor, decoded and clipped
 *   keys [B,npad] (npad = pow2 >= A): image b's segment sorted ascending, so that entry j < count[b]
 *        is its j-th best candidate (score desc, anchor index asc); the rest are ~0 sentinels
 *   count [B] int32: candidates of image b above the threshold
 * ------------------------------------------------------------------------------------------ */
int effdet_detect_candidates_batch(const float* cls, const float* reg, const float* anchors, float* boxes, float* scores,
                                   int32_t* classes, uint64_t* keys, int32_t* count, int B, int A, int K, int npad,
                                   float img_w, float img_h, float threshold, int device, effdet_stream_t stream);
/* Greedy NMS of at most `cap` candidates per image (1 <= cap <= A, ceil(cap/64)*8 <= 200 KiB of scan bitmap).
 *   boxes [B,A,4], keys [B,npad] and count [B] as written by effdet_detect_candidates_batch
 *   mask_ws [B][cap][ceil(cap/64)] uint64 workspace
 *   keep_idx [B][cap] int32: anchor indices of image b's kept boxes, best first, in its first nkeep[b] entries
 *   nkeep [B] int32: boxes kept in image b, or -1 when count[b] > cap (overflow: nothing else is written for it) */
int effdet_nms_batch(const float* boxes, const uint64_t* keys, const int32_t* count, int B, int A, int npad, int cap,
                     double iou_threshold, uint64_t* mask_ws, int32_t* keep_idx, int32_t* nkeep, int device,
                     effdet_stream_t stream);
/* The same greedy NMS in column chunks of `chunk` sorted candidates, in a workspace linear in cap: for each chunk, a
 * cross step tests its candidates against the boxes kept so far (through keep_idx), then the upper-triangle mask and
 * the greedy scan run inside the chunk.  The keep sets, their order and nkeep equal effdet_nms_batch's for every chunk;
 * chunk == cap is effdet_nms_batch itself.  The launch sequence depends on B, cap and chunk only (capturable).
 *   1 <= B <= 65535; 1 <= cap <= A (any cap: only the chunk's bitmap lives in shared memory);
 *   chunk a multiple of 64 in [64, cap], or chunk == cap
 *   workspace: effdet_nms_chunked_workspace(B, cap, chunk) bytes, 16-byte aligned (-1 when the arguments are refused)
 *   keep_idx, nkeep: as effdet_nms_batch */
int64_t effdet_nms_chunked_workspace(int B, int cap, int chunk);
int effdet_nms_batch_chunked(const float* boxes, const uint64_t* keys, const int32_t* count, int B, int A, int npad,
                             int cap, int chunk, double iou_threshold, void* workspace, int64_t workspace_bytes,
                             int32_t* keep_idx, int32_t* nkeep, int device, effdet_stream_t stream);
/* Padded detections: row i < nkeep[b] of image b is its i-th kept box, every later row is zero (all rows when
 * nkeep[b] == -1).  out_scores [B][cap] float, out_classes [B][cap] int64, out_boxes [B][cap][4] float (16-byte aligned). */
int effdet_gather_detections_batch(const float* boxes, const float* scores, const int32_t* classes,
                                   const int32_t* keep_idx, const int32_t* nkeep, int B, int A, int cap, float* out_scores,
                                   int64_t* out_classes, float* out_boxes, int device, effdet_stream_t stream);
/* Soft-NMS (Bodla et al., ICCV 2017, Algorithm 1) of the same candidates, written directly as padded detections in
 * effdet_gather_detections_batch's layout.  Each pick emits the live candidate with the highest current score (ties:
 * lower anchor index) and rescales every other live score s by a weight of its IoU ov with the pick (fp32 IoU as the
 * greedy NMS computes it; 0 when the intersection is 0):
 *   EFFDET_SOFT_NMS_LINEAR  : w = (double)ov > iou_threshold ? 1 - ov : 1                  (iou_threshold in [0, 1])
 *   EFFDET_SOFT_NMS_GAUSSIAN: w = (float)exp(-((double)ov * ov) / sigma), in fp64           (iou_threshold unused)
 *   s = s * w in fp32; a candidate with !(s > threshold) leaves the live set.
 * Row i of image b is its i-th pick: the score at the moment of the pick (non-increasing down the rows), the
 * candidate's class and box.  Rows from out_count[b] on are zero; out_count[b] = -1 (all rows zero) when count[b] > cap.
 *   boxes, scores, classes [B,A], keys [B,npad], count [B]: as effdet_detect_candidates_batch writes them
 *   1 <= B <= 65535, 1 <= cap <= A, sigma finite and > 0 (checked for either method)
 *   workspace: effdet_soft_nms_workspace(B, cap) bytes (B*cap*24 rounded up to a multiple of 16), 16-byte aligned;
 *              0 bytes (null allowed) unless cap > 32768
 *   threshold: candidates whose score is not above it are never picked (effdet_detect_candidates_batch leaves none)
 *   out_scores [B][cap], out_classes [B][cap] int64, out_boxes [B][cap][4] (16-byte aligned), out_count [B] int32
 * One launch whose grid depends on B and cap only (capturable); no host read. */
#define EFFDET_SOFT_NMS_LINEAR 1
#define EFFDET_SOFT_NMS_GAUSSIAN 2
int64_t effdet_soft_nms_workspace(int B, int cap);
int effdet_soft_nms_batch(const float* boxes, const float* scores, const int32_t* classes, const uint64_t* keys,
                          const int32_t* count, int B, int A, int npad, int cap, int method, double iou_threshold,
                          double sigma, float threshold, void* workspace, int64_t workspace_bytes, float* out_scores,
                          int64_t* out_classes, float* out_boxes, int32_t* out_count, int device,
                          effdet_stream_t stream);
/* Class-aware NMS.  Per-class greedy NMS: effdet_nms_batch_chunked's arguments and workspace plus classes [B,A] int32
 * (as effdet_detect_candidates_batch writes them); a pair of candidates counts only when their classes are equal.  The
 * candidates of one class, taken in the global (score desc, anchor asc) order, are that class's own sorted list, so
 * keep_idx holds torchvision's per-class keep sets (_batched_nms_vanilla) merged in (score desc, anchor asc) order. */
int effdet_nms_batch_chunked_classes(const float* boxes, const uint64_t* keys, const int32_t* count,
                                     const int32_t* classes, int B, int A, int npad, int cap, int chunk,
                                     double iou_threshold, void* workspace, int64_t workspace_bytes, int32_t* keep_idx,
                                     int32_t* nkeep, int device, effdet_stream_t stream);
/* Per-class Soft-NMS: effdet_soft_nms_batch's arguments, refusals and workspace.  Picks go in the global order; a pick
 * decays only the live candidates of its own class (classes [B,A]), the others stay live and unchanged. */
int effdet_soft_nms_batch_classes(const float* boxes, const float* scores, const int32_t* classes,
                                  const uint64_t* keys, const int32_t* count, int B, int A, int npad, int cap,
                                  int method, double iou_threshold, double sigma, float threshold, void* workspace,
                                  int64_t workspace_bytes, float* out_scores, int64_t* out_classes, float* out_boxes,
                                  int32_t* out_count, int device, effdet_stream_t stream);
/* Multi-label candidates: every (anchor a, class k) pair with cls[b,a,k] > threshold, numbered p = a*K + k, and the
 * best k' = min(top_k, A*K) of them in (score desc, p asc) order, selected exactly by a radix select on the unique
 * 64-bit key (~order(score) << 32) | p.  Written in effdet_detect_candidates_batch's format with the k' slots in place
 * of the anchors, so the NMS entries run on it with A := k' and npad := kpad:
 *   boxes [B,k',4] (16-byte aligned): slot i's pair's anchor box, decoded and clipped bit for bit as the candidates
 *        entry decodes it; scores [B,k'] its cls value; classes [B,k'] int32 its k; slots >= count[b] are zero
 *   keys [B,kpad] (kpad = pow2 >= k'): (~order(score) << 32) | slot, sorted; ~0 sentinels from count[b] on
 *   count [B] int32: min(pairs above threshold, k')
 *   1 <= B <= 65535, A*K < 2^32, top_k >= 1; cls [B,A,K], reg [B,A,4] and anchors [A,4] as for the candidates entry
 *   workspace: effdet_detect_topk_workspace(B, A, K, top_k) bytes, 16-byte aligned (-1 when the arguments are refused)
 * The launch sequence depends on B, A, K and top_k only and there is no host read (capturable).  cls is read once per
 * histogram pass an image still takes part in (one to six; one when it has at most k' pairs above the threshold) and
 * once by the compaction. */
int64_t effdet_detect_topk_workspace(int B, int A, int K, int top_k);
int effdet_detect_topk_batch(const float* cls, const float* reg, const float* anchors, int B, int A, int K, float img_w,
                             float img_h, float threshold, int top_k, int kpad, void* workspace,
                             int64_t workspace_bytes, float* boxes, float* scores, int32_t* classes, uint64_t* keys,
                             int32_t* count, int device, effdet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * SURVEY.md 8(f) rank 1: the optimizer step that follows backward in the reference loop,
 *   clip_grad_norm_(parameters, max_norm) + AdamW.step()        (train.py:115-118, train.py:268)
 * as two multi-tensor launches.  The tables live in DEVICE memory: per tensor t its fp32 data pointers and
 * element count, per chunk c the tensor it belongs to and its element offset; one CTA per chunk.
 *   effdet_multi_sumsq      : norm_sq[0] += sum_t sum_i g_t[i]^2
 *   effdet_multi_clip_adamw : g *= min(1, max_norm/(sqrt(norm_sq)+1e-6)) (max_norm <= 0: no clipping);
 *                             p *= 1 - lr*wd;  m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;
 *                             p -= lr/bias_c1 * m / (sqrt(v)/sqrt(bias_c2) + eps)     (torch.optim.AdamW)
 * ------------------------------------------------------------------------------------------ */
int effdet_multi_sumsq(const uint64_t* g_ptrs, const int64_t* numels, const int32_t* chunk_tensor,
                       const int64_t* chunk_off, int nchunks, int chunk, float* norm_sq, int device,
                       effdet_stream_t stream);
int effdet_multi_clip_adamw(const uint64_t* p_ptrs, const uint64_t* g_ptrs, const uint64_t* m_ptrs,
                            const uint64_t* v_ptrs, const int64_t* numels, const int32_t* chunk_tensor,
                            const int64_t* chunk_off, int nchunks, int chunk, const float* norm_sq, float max_norm,
                            float lr, float beta1, float beta2, float eps, float weight_decay, float bias_c1,
                            float bias_c2, int write_clipped_grad, int device, effdet_stream_t stream);
/* The same step replayed from a CUDA graph, with gradient accumulation (train.py:107-118 with
 * --grad_accumulation_steps k): every value that changes between steps is read from device memory.
 *   effdet_multi_accumulate     : acc_t[i] += g_t[i] for every tensor, unless loss[0] == 0.0f exactly (the reference's
 *                                 `if bool(loss == 0): continue`), in which case nothing is written.  With gate given
 *                                 (update_requested then too): gate[0] = update_requested[0] != 0 && loss[0] != 0.
 *   effdet_multi_clip_adamw_dev : gate[0] == 0: returns without touching p, m, v, acc or the counter.  Otherwise the
 *                                 update of effdet_multi_clip_adamw on g_ptrs = the accumulators, with lr = lr[0],
 *                                 bias_c = (float)(1 - beta^(step[0] + 1)) in fp64 and 1 - beta rounded from fp64
 *                                 (torch.optim.AdamW's rounding), then acc = 0 and step[0] += 1.
 *                                 ticket: one zero-initialised uint32 that the launch returns to zero (it orders the
 *                                 counter's advance after every CTA's read); launches sharing it must be stream-ordered.
 * norm_sq for the update comes from effdet_multi_sumsq over the accumulators, zeroed before it. */
int effdet_multi_accumulate(const uint64_t* acc_ptrs, const uint64_t* g_ptrs, const int64_t* numels,
                            const int32_t* chunk_tensor, const int64_t* chunk_off, int nchunks, int chunk,
                            const float* loss, const int32_t* update_requested, int32_t* gate, int device,
                            effdet_stream_t stream);
int effdet_multi_clip_adamw_dev(const uint64_t* p_ptrs, const uint64_t* g_ptrs, const uint64_t* m_ptrs,
                                const uint64_t* v_ptrs, const int64_t* numels, const int32_t* chunk_tensor,
                                const int64_t* chunk_off, int nchunks, int chunk, const float* norm_sq, float max_norm,
                                const float* lr, int64_t* step, const int32_t* gate, uint32_t* ticket, double beta1,
                                double beta2, float eps, float weight_decay, int device, effdet_stream_t stream);
/* Exponential moving average of the weights (Tan et al., EfficientDet section 5.1), over the same chunk tables:
 * ema_ptrs[t] the averaged fp32 tensors, src_ptrs[t] the model's, one CTA per chunk.
 *   gate      : gate[0] == 0 (the gate effdet_multi_accumulate writes): returns and writes nothing, not even the
 *               counter.  gate NULL: every launch updates.
 *   updates   : int64 counter; this launch is update k = updates[0] + 1, and advances updates[0] by exactly one.
 *   ticket    : one zero-initialised uint32 that the launch returns to zero (every CTA reads the counter before it
 *               takes a ticket; the last one advances it); launches sharing it must be stream-ordered.
 *   decay     : d = ramp ? min(decay, (1 + k) / (10 + k)) : decay in fp64 -- TF's ExponentialMovingAverage(decay,
 *               num_updates=k) -- then w = (float)(1 - d), rounded once.
 *   element   : e = e - w * (e - s) in fp32, each operation rounded on its own (__fsub_rn / __fmul_rn, no FMA):
 *               TF's assign_moving_average, variable - (variable - value) * (1 - decay).
 * Refused (-1, message naming multi_ema): a NULL table, counter or ticket, nchunks < 1, chunk < 1, decay outside
 * [0, 1]. */
int effdet_multi_ema(const uint64_t* ema_ptrs, const uint64_t* src_ptrs, const int64_t* numels,
                     const int32_t* chunk_tensor, const int64_t* chunk_off, int nchunks, int chunk, double decay,
                     int ramp, int64_t* updates, const int32_t* gate, uint32_t* ticket, int device,
                     effdet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * SURVEY.md 8(f) rank 2: the step BEFORE the hot path, on the device.  Normalizer + Augmenter (horizontal flip) + zero pad
 * to the common size + collater + `.cuda().float()` (datasets/augmentation.py:69-91,111-150, train.py:105-106), bit-identical
 * to NumPy: (float32(u8) - mean) / std evaluated in float64, then cast to float32.  effdet_normalize_pad takes images at
 * their final resolution (h, w <= S); effdet_resize_normalize_pad below also runs Resizer's cv2.resize.
 *   pixels  : uint8 HWC images back to back, image b starts at byte offsets[b] and is hw[2b] x hw[2b+1] x 3
 *   flip    : [B] or NULL;  out_nchw : float32 [B,3,S,S];  mean3 / std3 : 3 host doubles
 *   annotations: rows [sum n_b, 5] float64, image b owns rows row_off[b] .. row_off[b+1]; out float32 [B,G,5], -1 padded;
 *   scale [B] float64 or NULL (Resizer's box scale), width [B] = image widths (needed with flip)
 * ------------------------------------------------------------------------------------------ */
int effdet_normalize_pad(const uint8_t* pixels, const int64_t* offsets, const int32_t* hw, const uint8_t* flip,
                         float* out_nchw, int B, int S, const double* mean3, const double* std3, int device,
                         effdet_stream_t stream);
int effdet_collate_annots(const double* rows, const int32_t* row_off, const double* scale, const uint8_t* flip,
                          const int32_t* width, float* out, int B, int G, int device, effdet_stream_t stream);
/* effdet_collate_annots followed by effdet_pack_annots, bit for bit, in one launch and with no host read, for a raw batch
 * (models/pipeline.py RawBatch) in device memory: B = header[0] (1..Bcap) images, image b owns rows row_off[b] ..
 * row_off[b+1] (at most Gcap of them), flip [Bcap], hw [Bcap,2] (the width is the flip's `cols`), scale [Bcap] float64.
 * out [Bcap,Gcap,5] float32: per image its rows whose float32 label is not -1, flipped and scaled, in order, then -1
 * rows; counts [1+Bcap]: counts[0] = B, counts[1+b] = rows kept, 0 for b >= B.  Refused before the launch: a null
 * pointer, Bcap outside 1..65535, Gcap < 1.  Whether a batch fits is the caller's check (RawBatch holds the counts). */
int effdet_collate_pack_annots(const int64_t* header, const double* rows, const int32_t* row_off, const double* scale,
                               const uint8_t* flip, const int32_t* hw, float* out, int32_t* counts, int Bcap, int Gcap,
                               int device, effdet_stream_t stream);
/* The same input step with Resizer's cv2.resize (datasets/augmentation.py:94-115,118-150): images of any size h, w >= 1,
 * image b resized (after the flip) to resized_hw[2b] x resized_hw[2b+1] (1 .. S each) by OpenCV's generic INTER_LINEAR
 * for CV_64FC3 on the float64 normalized image, zero padded to S x S, cast to float32 once.  pixel_scale selects the
 * Normalizer's input: 1 = float32(u8) (COCO), 255 = float32(u8) / 255.f (VOC, datasets/voc0712.py:109).  Offsets, hw
 * and flip as effdet_normalize_pad; the annotations go through effdet_collate_annots with Resizer's scale. */
int effdet_resize_normalize_pad(const uint8_t* pixels, const int64_t* offsets, const int32_t* hw, const int32_t* resized_hw,
                                const uint8_t* flip, float* out_nchw, int B, int S, int pixel_scale, const double* mean3,
                                const double* std3, int device, effdet_stream_t stream);
/* Scale jitter (models/pipeline.py RawCollater(scale_jitter=...)): the siblings above plus crops int32 [B,2] (Bcap for
 * the pack) = (y0, x0) per image.
 * effdet_resize_crop_normalize_pad: image b is resized to resized_hw[b] (Resizer at the drawn common size L, so up to
 * L >= S per side) and out[b] is the S x S window at (y0, x0) of it: out[y, x] = R[y + y0, x + x0] where that lies
 * inside the resized image, 0 elsewhere (a negative offset writes a zero image).
 * effdet_collate_pack_annots_crop: after the flip and the scale, x1/x2 -= x0 and y1/y2 -= y0, each coordinate clamped
 * to [0, S] with S = header[4], in float64, then cast to float32 once; a row is kept only if its float32 label is not
 * -1, x2 > x1 and y2 > y1.  Refusals as the siblings'. */
int effdet_resize_crop_normalize_pad(const uint8_t* pixels, const int64_t* offsets, const int32_t* hw,
                                     const int32_t* resized_hw, const int32_t* crops, const uint8_t* flip, float* out_nchw,
                                     int B, int S, int pixel_scale, const double* mean3, const double* std3, int device,
                                     effdet_stream_t stream);
int effdet_collate_pack_annots_crop(const int64_t* header, const double* rows, const int32_t* row_off, const double* scale,
                                    const uint8_t* flip, const int32_t* hw, const int32_t* crops, float* out,
                                    int32_t* counts, int Bcap, int Gcap, int device, effdet_stream_t stream);
/* demo.py's per-frame path (Detect.process, demo.py:71-104) for a batch of frames.
 * effdet_frame_transform replaces get_augumentation(phase='test') + `.to(device).unsqueeze(0)` (demo.py:75-78,
 * datasets/augmentation.py:38-48, albumentations 0.5.2): cv2.resize(frame, (W, H), INTER_LINEAR) of the uint8 frame in
 * OpenCV's fixed-point CV_8U arithmetic, then Normalize ((float32(u8) - mean * 255) * float32(1 / (std * 255)), float32
 * steps) and ToTensor, bit-identical to OpenCV 4.13.0 and NumPy.  Channels keep the frame's byte order (BGR).
 *   pixels  : uint8 HWC frames back to back, frame b starts at byte offsets[b] and is hw[2b] x hw[2b+1] x 3 (any size
 *             >= 1 x 1); hw[2b] == 0 marks a padding frame, whose output is zero
 *   out_nchw: float32 [B,3,H,W];  mean3 / std3: 3 host floats (Normalize's mean and std, in [0, 1])
 * effdet_frame_boxes replaces demo.py's per-box loop (demo.py:86-104) on the padded detections of the batch:
 *   scores [B,C], classes [B,C] int64, boxes [B,C,4] (16-byte aligned), count [B] as GraphedDetect / detect_batch(cap=C)
 *   write them; hw [2B] the frames' (h, w); H, W the network input's size (demo's size_image)
 *   rows [B,C,6] int32: row k < out_count[b] of frame b is (int(x1 * w / W), int(y1 * h / H), int(x2 * w / W),
 *        int(y2 * h / H), label, int(np.around(score, 2) * 100)), float32 arithmetic (NumPy >= 2); later rows are not
 *        written.  out_count [B] int32: count[b], 0 for a padding frame, -1 when the frame overflowed the cap.
 * Neither reads device memory on the host: both can be captured in a CUDA graph. */
int effdet_frame_transform(const uint8_t* pixels, const int64_t* offsets, const int32_t* hw, float* out_nchw, int B, int H,
                           int W, const float* mean3, const float* std3, int device, effdet_stream_t stream);
int effdet_frame_boxes(const float* scores, const int64_t* classes, const float* boxes, const int32_t* count,
                       const int32_t* hw, int B, int C, int H, int W, int32_t* rows, int32_t* out_count, int device,
                       effdet_stream_t stream);
/* SURVEY.md 8(f) rank 3: the step AFTER NMS (eval.py:105-128) for one image: boxes /= scale, score > threshold,
 * top-max_det by score (ties: lower input index), split per label.  out_dets [max_det,5] (x1,y1,x2,y2,score) grouped by
 * label ascending and in score order inside a label, out_labels [max_det], class_offsets [num_classes+1] (rows of label c
 * are class_offsets[c] .. class_offsets[c+1]), count[0] = selected rows. */
int effdet_eval_select(const float* scores, const int64_t* labels, const float* boxes, int n, float scale,
                       float score_threshold, int max_det, int num_classes, float* out_dets, int32_t* out_labels,
                       int32_t* class_offsets, int32_t* count, int device, effdet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * VOC mean average precision on the device (eval.py::evaluate, eval.py:165-257), for a whole test set without a host
 * read until the end.  A record is one detection slot: image i owns records i*max_det .. (i+1)*max_det - 1.
 *
 * effdet_eval_select_batch: effdet_eval_select for B images at once, on the padded output of the batched detection
 *   (scores [B,C], labels [B,C] int64, boxes [B,C,4] 16-byte aligned, count [B] int32 kept rows, -1 = NMS overflow),
 *   with per-image scales scale [B] float on the device.  Image b's rows equal effdet_eval_select(..., count[b],
 *   scale[b], ...) bit for bit and go to out_dets [B][max_det][5], out_labels [B][max_det] (-1: empty slot) and
 *   class_offsets [B][num_classes+1].  count[b] == -1: every label -1 and overflow[b] = 1 (else 0).
 *   score_threshold >= 0 (the AP key below relies on positive scores).
 * effdet_voc_match: eval.py:199-224 for the B images of one effdet_eval_select_batch call.  Ground truth: gt [num_gt,5]
 *   fp64 rows (x1,y1,x2,y2,label) in original image coordinates, image b owns rows gt_offsets[b] .. gt_offsets[b+1]
 *   ([B+1] int32 on the device).  Per (image, class) the detections are taken in slot order (score descending) and
 *   matched greedily: IoU as compute_overlap computes it (fp64, no FMA contraction), the first maximum wins, TP iff
 *   IoU >= iou_threshold and that ground truth is not taken yet.  tp [B][max_det] uint8 = 1 (TP) / 0 (FP) for every
 *   filled slot; gt_count [num_classes] int64 += ground-truth rows per class.
 * effdet_voc_ap: eval.py:226-248 for every class over num_records records (dets [R][5], labels [R], tp [R] as written
 *   above, gt_count as accumulated above) -> ap [num_classes] fp64, num_annotations [num_classes] fp64 (both 0 for a
 *   class without ground truth).  Records of one class are ordered by score descending, ties by record index (image,
 *   then rank inside the image): the order a stable sort of the reference's append order gives.  Sums follow NumPy's
 *   pairwise summation, so the results equal the reference's float64 values.  The sort key packs class (8 bits),
 *   score (31 bits) and record index (25 bits): num_classes <= 255 and num_records <= 2^25 (33,554,432).
 *   workspace: effdet_voc_ap_workspace(num_records, num_classes) bytes, 16-byte aligned (-1 when over the limits).
 * ------------------------------------------------------------------------------------------ */
int effdet_eval_select_batch(const float* scores, const int64_t* labels, const float* boxes, const int32_t* count,
                             const float* scale, int B, int C, float score_threshold, int max_det, int num_classes,
                             float* out_dets, int32_t* out_labels, int32_t* class_offsets, int32_t* overflow, int device,
                             effdet_stream_t stream);
int effdet_voc_match(const float* dets, const int32_t* class_offsets, const double* gt, const int32_t* gt_offsets,
                     int num_gt, int B, int max_det, int num_classes, double iou_threshold, uint8_t* tp,
                     int64_t* gt_count, int device, effdet_stream_t stream);
int64_t effdet_voc_ap_workspace(int num_records, int num_classes);
int effdet_voc_ap(const float* dets, const int32_t* labels, const uint8_t* tp, const int64_t* gt_count, int num_records,
                  int num_classes, double* ap, double* num_annotations, void* workspace, int64_t workspace_bytes,
                  int device, effdet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * COCO box mAP on the device (eval.py::evaluate_coco, eval.py:260-338, with pycocotools' COCOeval for iouType 'bbox'
 * and default Params), for a whole test set without a host read until the end.  Images are identified by their rank
 * among the sorted image ids (COCOeval's imgIds), categories by their index among the sorted category ids (catIds).
 * Records live in a buffer of `capacity` slots: rec_box [capacity] float4 (x, y, w, h after boxes /= scale, in
 * float32), rec_score [capacity] float, rec_meta [capacity] int4 (model label, category index or -1, image rank, rank
 * inside (image, category) after a stable sort by score descending), rec_meta initialised to -1 by the caller.
 * Limits: num_categories <= 255, num_images <= 2^18, capacity <= 2^25, max_gt <= 256 ground truths per (image,
 * category).
 *
 * effdet_coco_select_batch: eval.py:280-311 for B images of the padded detection output (scores [B,C], labels [B,C]
 *   int64, boxes [B,C,4] 16-byte aligned, count [B] int32 kept rows, -1 = NMS overflow) with per-image scale [B]
 *   float and image_rank [B] int32 on the device.  Image b records its rows in NMS order up to the first with
 *   (double)score < score_threshold; label l maps to category label_category[l] (-1 when l is outside
 *   [0, num_labels) or maps to no ground-truth category).  The rows go to the slots at the device-side cursor (int64,
 *   records asked for so far, also past capacity), in batch order; image_offset / image_count [num_images] (indexed by
 *   rank) and batch_offset / batch_count [B] receive each image's slots.  status [B]: 0 recorded, 1 NMS overflow
 *   (nothing recorded), 2 out of capacity (nothing recorded).
 * effdet_coco_match: COCOeval.computeIoU + evaluateImg for the images of one effdet_coco_select_batch call (the same
 *   image_rank, batch_offset, batch_count).  Ground truth gt [n,6] fp64 (x, y, w, h, area, iscrowd) grouped by
 *   (image rank, category) in annotation order: group q*num_categories + k owns rows gt_offsets[..] ..
 *   gt_offsets[..+1] (int32 [num_images*num_categories+1]); max_gt = the largest group.  iou_thrs: the 10 fp64 values
 *   of Params.iouThrs on the device; iou_type must be EFFDET_COCO_BBOX.  flags [capacity][4] uint32 per record of rank
 *   < 100 and area range (all, small, medium, large): bit t = matched at threshold t, bit 16+t = ignored.
 *   npig [num_categories][4] int64 += non-ignored ground truths.
 * effdet_coco_accumulate: COCOeval.accumulate -> precision [10][101][num_categories][4][3] and recall
 *   [10][num_categories][4][3] fp64 (-1 where a (category, area range) has no non-ignored ground truth).  rec_thrs: the
 *   101 fp64 values of Params.recThrs on the device; max_dets must be (1, 10, 100).  Records of one category are
 *   ordered by score descending, then image rank, then rank inside (image, category), with one 64-bit key sort over
 *   category (8 bits), score (31) and the record's position in image-rank order (25).  workspace:
 *   effdet_coco_accumulate_workspace(capacity, num_images, num_categories) bytes, 16-byte aligned.
 * ------------------------------------------------------------------------------------------ */
#define EFFDET_COCO_BBOX 1
int effdet_coco_select_batch(const float* scores, const int64_t* labels, const float* boxes, const int32_t* count,
                             const float* scale, const int32_t* image_rank, int B, int C, double score_threshold,
                             const int32_t* label_category, int num_labels, int num_categories, int num_images,
                             int capacity, float* rec_box, float* rec_score, int32_t* rec_meta, int64_t* cursor,
                             int32_t* image_offset, int32_t* image_count, int32_t* status, int32_t* batch_offset,
                             int32_t* batch_count, int device, effdet_stream_t stream);
int effdet_coco_match(const float* rec_box, const int32_t* rec_meta, const int32_t* batch_offset,
                      const int32_t* batch_count, const int32_t* image_rank, int B, const double* gt,
                      const int32_t* gt_offsets, int num_images, int num_categories, int max_gt, const double* iou_thrs,
                      int num_iou_thrs, int iou_type, uint32_t* flags, int64_t* npig, int device,
                      effdet_stream_t stream);
int64_t effdet_coco_accumulate_workspace(int capacity, int num_images, int num_categories);
int effdet_coco_accumulate(const float* rec_score, const int32_t* rec_meta, const uint32_t* flags,
                           const int64_t* cursor, const int32_t* image_offset, const int32_t* image_count,
                           const int64_t* npig, const double* rec_thrs, int num_rec_thrs, int max_det0, int max_det1,
                           int max_det2, int capacity, int num_images, int num_categories, double* precision,
                           double* recall, void* workspace, int64_t workspace_bytes, int device,
                           effdet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Layout plumbing at the module boundary (callers see logical NCHW, kernels are NHWC).
 * ------------------------------------------------------------------------------------------ */
int effdet_nchw_to_nhwc(const float* x, float* y, int B, int C, int H, int W, int device, effdet_stream_t stream);
int effdet_nhwc_to_nchw(const float* x, float* y, int B, int C, int H, int W, int device, effdet_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* EFFDET_B200_H */
