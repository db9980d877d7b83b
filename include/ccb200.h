/* ccb200.h - C ABI of libccb200.so: the H100 (sm_90a) implementation of the Competitive-Collaboration
 * training step's dense per-pixel path (anuragranj/cc @ 2b4e362).
 *
 * Conventions (SURVEY.md 8b):
 *   - every pointer is a DEVICE pointer to contiguous fp32 NCHW data unless a comment says "host";
 *   - the caller (torch.empty on the Python side) owns every buffer, including workspaces and the
 *     buffers saved for backward; the library owns no tensors and keeps no state between calls (the only process-wide
 *     variables are the launch counter and the bring-up switches of ccb200_debug.h; a weight cache is an explicit handle
 *     the caller creates, passes in ccb_conv_desc and destroys)
 *     (the reference caches a module-global pixel grid, inverse_warp.py:10 - we do not);
 *   - every entry point is asynchronous on `stream` (a cudaStream_t), never synchronises the host,
 *     never throws, and returns CCB_OK or a negative ccb_status; ccb_last_error_string() explains it;
 *   - shape errors that the reference reports as Python AssertionError (inverse_warp.py:23-28) are
 *     raised by the Python mirror (cc_b200/*.py) before the call; the ABI re-checks what it needs;
 *   - every scratch buffer (a parameter or descriptor field named work, partials or *_partials) is followed by its size
 *     in the unit of its pointer type: float* -> *_floats, unsigned long long* -> *_words, void* -> *_bytes.  The size
 *     needed is what the entry point's size query returns for the same arguments (the warps' fixed-point scatter buffer
 *     has no query: it needs the image gradient's element count + 1 words).  A smaller size returns CCB_ERR_ARG, naming
 *     the entry point and the buffer, and launches nothing; a larger one changes nothing.  NULL with size 0 is allowed
 *     exactly where the need is 0.  A size query returns -1 for invalid sizes.  void* workspaces must be 8-byte aligned.
 *
 * Each entry point names the reference interface it replaces (file:line relative to the reference).
 */
#ifndef CCB200_H
#define CCB200_H

#ifdef __cplusplus
extern "C" {
#endif

#define CCB_MAX_LEVELS 8
#define CCB_MAX_REFS 4
#define CCB_SSIM_TAPS 13

typedef void* ccb_stream_t; /* cudaStream_t */

typedef enum ccb_status {
    CCB_OK = 0,
    CCB_ERR_ARG = -1,         /* bad size / null pointer / unsupported combination */
    CCB_ERR_LAUNCH = -2,      /* CUDA launch or runtime error */
    CCB_ERR_UNSUPPORTED = -3
} ccb_status;

const char* ccb_last_error_string(void);
int ccb_version(void);
/* 1 only for the CPU execution-model simulator build used by the GPU-less unit tests (tests/sim). */
int ccb_is_simulator(void);

/* ------------------------------------------------------------------------------------------------
 * Image pyramid: level l = exact 2^l x 2^l box mean of the full-resolution planes.
 * Replaces the 15 adaptive_avg_pool2d calls per level per step (loss_functions.py:36-37,89-90,
 * 163-165,315).  out_levels: HOST array of nlevels-1 device pointers (levels 1..nlevels-1),
 * each [planes, H>>l, W>>l].  H and W must be divisible by 2^(nlevels-1).
 * ---------------------------------------------------------------------------------------------- */
int ccb_image_pyramid(const float* img, int planes, int H, int W, int nlevels,
                      float* const* out_levels, ccb_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Fused multi-scale photometric loss (one launch covers every pyramid level).
 *   mode CCB_PHOTO_RIGID : photometric_reconstruction_loss  (loss_functions.py:80-128)
 *        = pixel2cam -> pose_vec2mat -> cam2pixel -> bilinear sample (inverse_warp.py:250-283)
 *          + depth_occlusion_masks (loss_functions.py:132-137,343-352) + SSIM 13x13 (ssim.py:19-36)
 *          + robust L1 (loss_functions.py:18-21) + oob normalisation.
 *   mode CCB_PHOTO_FLOW  : photometric_flow_loss             (loss_functions.py:27-77)
 *        = flow_warp (inverse_warp.py:164-192) + occlusion_masks + SSIM + robust L1.
 *   mode CCB_PHOTO_CONSENSUS : consensus_exp_masks targets   (loss_functions.py:160-202), R = 3
 *        "refs": (ref_fwd,cam_flow_fwd) (ref_bwd,cam_flow_bwd) (ref_fwd,flow_fwd); no gradient.
 * ---------------------------------------------------------------------------------------------- */
enum { CCB_PHOTO_RIGID = 0, CCB_PHOTO_FLOW = 1, CCB_PHOTO_CONSENSUS = 2 };
enum { CCB_ROT_EULER = 0, CCB_ROT_QUAT = 1 };
enum { CCB_PAD_ZEROS = 0, CCB_PAD_BORDER = 1, CCB_PAD_NONE = 2 };

typedef struct ccb_photo_desc {
    int mode;
    int B, R;                 /* batch, number of reference frames (<= CCB_MAX_REFS) */
    int H, W;                 /* full-resolution size: downscale_l = H / h[l] (loss_functions.py:87) */
    int nlevels;
    int h[CCB_MAX_LEVELS], w[CCB_MAX_LEVELS];
    int has_mask;             /* explainability mask given (mask[l] != NULL for all l) */
    int has_occ;              /* apply occlusion masks (always 1 in the reference paths) */
    int rotation_mode;        /* CCB_ROT_* (rigid) */
    int padding_mode;         /* CCB_PAD_ZEROS | CCB_PAD_BORDER (rigid) */
    float wssim, qch, lambda_oob, wrig;
    float one_minus_wssim;    /* (1 - wssim) evaluated in double by the caller, as the reference does */
    float taps[CCB_SSIM_TAPS]; /* fp32 Gaussian taps exactly as ssim.py:9-11 builds them */
    /* inputs */
    const float* tgt[CCB_MAX_LEVELS];                 /* [B,3,h,w] pooled target frame */
    const float* ref[CCB_MAX_LEVELS][CCB_MAX_REFS];   /* [B,3,h,w] pooled reference frames */
    const float* depth[CCB_MAX_LEVELS];               /* rigid: [B,1,h,w] */
    const float* flow[CCB_MAX_LEVELS][CCB_MAX_REFS];  /* flow/consensus: [B,2,h,w] */
    const float* mask[CCB_MAX_LEVELS];                /* [B,R,h,w] or NULL */
    const float* pose;                                /* rigid: [B,R,6] */
    const float* K;                                   /* rigid: [B,3,3] full-res intrinsics */
    const float* Kinv;                                /* rigid: [B,3,3] */
    /* saved for backward (written by fwd, read by bwd).  Forward with vo[0] == NULL: value-only (no backward will run;
     * dmaps / vo / gmask all NULL, none written).  gmask[0] == NULL with has_mask: the mask needs no gradient (not
     * computed); then the backward takes d_mask == NULL.  The loss value is the same in every case. */
    float* dmaps[CCB_MAX_LEVELS];    /* [B,R,9,h,w] gamma * dS/d(mu2,Eyy,Exy); unused when wssim == 0 */
    float* gmask[CCB_MAX_LEVELS];    /* [B,R,h,w]  unscaled d loss / d mask (has_mask only) */
    float* vo[CCB_MAX_LEVELS];       /* [B,R,h,w]  valid * (1 - occ) */
    float* scal;                     /* [nlevels,R,4] : c_l, oob, sum_valid, level-ref loss */
    /* forward outputs / workspace */
    float* partials;                 /* ccb_photo_partials_floats() */
    long long partials_floats;
    float* loss;                     /* [1] */
    float* target[CCB_MAX_LEVELS];   /* consensus: [B,1,h,w] 0/1 */
    /* backward inputs / outputs / workspace */
    const float* grad_out;           /* [1] d L / d loss */
    float* d_depth[CCB_MAX_LEVELS];                 /* rigid: [B,1,h,w] */
    float* d_flow[CCB_MAX_LEVELS][CCB_MAX_REFS];    /* flow:  [B,2,h,w] */
    float* d_mask[CCB_MAX_LEVELS];                  /* [B,R,h,w] (has_mask) */
    float* d_pose;                                  /* rigid: [B,R,6] */
    float* pose_partials;            /* rigid: ccb_photo_pose_partials_floats() */
    long long pose_partials_floats;
} ccb_photo_desc;

long long ccb_photo_partials_floats(const ccb_photo_desc* d);
long long ccb_photo_pose_partials_floats(const ccb_photo_desc* d);
int ccb_photo_loss_fwd(const ccb_photo_desc* d, ccb_stream_t stream);
int ccb_photo_loss_bwd(const ccb_photo_desc* d, ccb_stream_t stream);
int ccb_consensus_targets(const ccb_photo_desc* d, ccb_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Stand-alone warp layer (the functions train.py:22 imports by name).
 * ---------------------------------------------------------------------------------------------- */
/* inverse_warp (inverse_warp.py:250-283): img [B,3,h,w], depth [B,h,w], pose [B,6] with row stride
 * pose_stride floats, K/Kinv [B,3,3] (already scaled by the caller) -> out [B,3,h,w]. */
int ccb_inverse_warp_fwd(const float* img, const float* depth, const float* pose, int pose_stride,
                         const float* K, const float* Kinv, int B, int h, int w, int rotation_mode,
                         int padding_mode, float* out, ccb_stream_t stream);
/* grads wrt depth [B,h,w] and pose [B,6] (contiguous); pose_partials: ccb_warp_pose_partials_floats(B, h, w). */
int ccb_inverse_warp_bwd(const float* img, const float* depth, const float* pose, int pose_stride,
                         const float* K, const float* Kinv, int B, int h, int w, int rotation_mode,
                         int padding_mode, const float* grad_out, float* d_depth, float* d_pose,
                         float* pose_partials, long long pose_partials_floats, ccb_stream_t stream);
long long ccb_warp_pose_partials_floats(int B, int h, int w);
/* flow_warp (inverse_warp.py:164-192): img [B,C,h,w], flow [B,2,h,w]; padding zeros|border. */
int ccb_flow_warp_fwd(const float* img, const float* flow, int B, int C, int h, int w,
                      int padding_mode, float* out, ccb_stream_t stream);
/* d_flow [B,2,h,w] (may be NULL), d_img [B,C,h,w] (may be NULL; the gradient is ADDED to it).  With d_img, work holds
 * B*C*h*w + 1 words (0 without): the image gradient is a scatter, summed in fixed point so that it is the same on every
 * run. */
int ccb_flow_warp_bwd(const float* img, const float* flow, int B, int C, int h, int w,
                      int padding_mode, const float* grad_out, float* d_flow, float* d_img,
                      unsigned long long* work, long long work_words, ccb_stream_t stream);
/* pose2flow (inverse_warp.py:195-220): -> flow [B,2,h,w]; padding_mode CCB_PAD_NONE | CCB_PAD_ZEROS. */
int ccb_pose2flow_fwd(const float* depth, const float* pose, int pose_stride, const float* K,
                      const float* Kinv, int B, int h, int w, int rotation_mode, int padding_mode,
                      float* flow, ccb_stream_t stream);
int ccb_pose2flow_bwd(const float* depth, const float* pose, int pose_stride, const float* K,
                      const float* Kinv, int B, int h, int w, int rotation_mode, int padding_mode,
                      const float* grad_flow, float* d_depth, float* d_pose, float* pose_partials,
                      long long pose_partials_floats, ccb_stream_t stream);

/* ssim map (ssim.py:68-76, window 13, sigma 1.5, zero padding): img1,img2,out [planes,h,w]. */
int ccb_ssim_fwd(const float* img1, const float* img2, int planes, int h, int w, const float* taps_host,
                 float* out, ccb_stream_t stream);
/* d_img1/d_img2 may be NULL. */
long long ccb_ssim_bwd_workspace_floats(int planes, int h, int w);
int ccb_ssim_bwd(const float* img1, const float* img2, int planes, int h, int w, const float* taps_host,
                 const float* grad_out, float* d_img1, float* d_img2, float* work, long long work_floats,
                 ccb_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Smoothness (loss_functions.py:287-341) for a list of predictions [B,C,h_l,w_l].
 *   kind CCB_SMOOTH_EDGE   : edge_aware_smoothness_loss(img, pred): needs img[l] = pooled tgt [B,3,h,w]
 *   kind CCB_SMOOTH_SECOND : smooth_loss(pred), level weight 1/2.3^l
 * ---------------------------------------------------------------------------------------------- */
enum { CCB_SMOOTH_EDGE = 0, CCB_SMOOTH_SECOND = 1 };
typedef struct ccb_smooth_desc {
    int kind, B, C, nlevels;
    int h[CCB_MAX_LEVELS], w[CCB_MAX_LEVELS];
    const float* img[CCB_MAX_LEVELS];
    const float* pred[CCB_MAX_LEVELS];
    float* partials;          /* ccb_smooth_partials_floats() */
    long long partials_floats;
    float* loss;              /* [1] */
    const float* grad_out;    /* [1] */
    float* d_pred[CCB_MAX_LEVELS];
} ccb_smooth_desc;
long long ccb_smooth_partials_floats(const ccb_smooth_desc* d);
int ccb_smooth_fwd(const ccb_smooth_desc* d, ccb_stream_t stream);
int ccb_smooth_bwd(const ccb_smooth_desc* d, ccb_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Mask cross-entropies.
 *   kind CCB_BCE_ONES     : explainability_loss (loss_functions.py:148-155): BCE(mask, 1) per level
 *   kind CCB_BCE_CONSENSUS: consensus_depth_flow_mask + weighted_binary_cross_entropy
 *                           (loss_functions.py:221-261)
 * ---------------------------------------------------------------------------------------------- */
enum { CCB_BCE_ONES = 0, CCB_BCE_CONSENSUS = 1 };
typedef struct ccb_bce_desc {
    int kind, B, C, nlevels;  /* C = mask channels (4) */
    int h[CCB_MAX_LEVELS], w[CCB_MAX_LEVELS];
    float thresh, wbce;
    const float* mask[CCB_MAX_LEVELS];        /* [B,C,h,w] */
    const float* census_bwd[CCB_MAX_LEVELS];  /* [B,2,h,w] |cam_flow_bwd - flow_bwd| */
    const float* census_fwd[CCB_MAX_LEVELS];  /* [B,2,h,w] */
    const float* target_bwd[CCB_MAX_LEVELS];  /* [B,1,h,w] */
    const float* target_fwd[CCB_MAX_LEVELS];  /* [B,1,h,w] */
    float* partials;          /* ccb_bce_partials_floats() */
    long long partials_floats;
    float* loss;
    const float* grad_out;
    float* d_mask[CCB_MAX_LEVELS];
} ccb_bce_desc;
long long ccb_bce_partials_floats(const ccb_bce_desc* d);
int ccb_bce_fwd(const ccb_bce_desc* d, ccb_stream_t stream);
int ccb_bce_bwd(const ccb_bce_desc* d, ccb_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Convolutions of the four networks (replace the cuDNN calls behind nn.Conv2d / nn.ConvTranspose2d /
 * nn.BatchNorm2d in models/DispResNet6.py:9-94, PoseNetB6.py:10-21, MaskNet6.py:5-16,
 * back2future.py:27-48).  NCHW fp32, weights [Co,Ci,kh,kw], square stride/pad.
 *   y = act(conv(x, w) + bias + res)                               ccb_conv2d_fprop
 *   dx = act(conv_transpose(dy, w) + bias + res)                   ccb_conv2d_dgrad
 *        (plain data-gradient when bias/res are NULL and act is NONE; with them it is the
 *         nn.ConvTranspose2d forward of a layer whose torch weight [Cin_t,Cout_t,k,k] is this w)
 *   dw = d/dw                                                      ccb_conv2d_wgrad
 *        (the bias gradient comes with the activation backward: ccb_act_bwd_bias)
 * impl: CCB_CONV_IMPL_AUTO picks the wgmma tensor-core kernels (3xTF32: fp32 parity) where they pay off
 *       and the FFMA kernels otherwise; _FFMA / _TC force one (tests).
 * ---------------------------------------------------------------------------------------------- */
enum { CCB_ACT_NONE = 0, CCB_ACT_RELU = 1, CCB_ACT_LEAKY = 2, CCB_ACT_SIGMOID = 3 };
enum { CCB_CONV_FPROP = 0, CCB_CONV_DGRAD = 1, CCB_CONV_WGRAD = 2 };
enum { CCB_CONV_IMPL_AUTO = 0, CCB_CONV_IMPL_FFMA = 1, CCB_CONV_IMPL_TC = 2 };
typedef struct ccb_conv_desc {
    int B, Ci, Hi, Wi;      /* input  [B,Ci,Hi,Wi] */
    int Co, Ho, Wo;         /* output [B,Co,Ho,Wo]; Ho = (Hi + 2 pad - kh) / stride + 1 */
    int kh, kw, stride, pad;
    int act;                /* CCB_ACT_* fused into the epilogue */
    float slope;            /* LeakyReLU negative slope */
    int impl;               /* CCB_CONV_IMPL_* */
    void* wcache;           /* weight cache handle (ccb_wcache_create) or NULL: prepared weight copies are then made per call */
} ccb_conv_desc;
/* Weight cache.  The tensor-core kernels read weights from a prepared copy (tf32 hi | lo split, K order of the kernel).
 * Without a cache every conv call prepares its copy into `work`.  With one (a trainer owns it; the weights then only
 * change in the optimiser step): while the cache is RECORDING, conv calls note which prepared layouts they need (and still
 * prepare on the spot); ccb_wcache_plan_floats / ccb_wcache_table_bytes size the caller-allocated persistent buffer and
 * device table, ccb_wcache_commit binds them, ccb_wcache_refresh re-prepares EVERY copy in one launch (call it after each
 * weight update), and conv calls whose (weights, layout) are recorded skip their preparation launch.
 * The caller must refresh after ANY change of the weights (optimizer step, load_state_dict). */
void* ccb_wcache_create(void);
void ccb_wcache_destroy(void* cache);
long long ccb_wcache_plan_floats(void* cache);
long long ccb_wcache_table_bytes(void* cache);
int ccb_wcache_commit(void* cache, float* buf, long long buf_floats, void* table, long long table_bytes, ccb_stream_t stream);
int ccb_wcache_refresh(void* cache, ccb_stream_t stream);
/* out4 = {recorded layouts, cache hits, misses after commit, state (0 recording, 1 committed)} */
void ccb_wcache_stats(void* cache, long long* out4);
/* Each call is planned from the descriptor alone (kernels, split-K, hence the summation order): `work` must hold at least
 * ccb_conv_workspace_floats() floats (else CCB_ERR_ARG, nothing launched); a larger one changes nothing.  -1: bad descriptor. */
long long ccb_conv_workspace_floats(const ccb_conv_desc* d, int op);
int ccb_conv2d_fprop(const ccb_conv_desc* d, const float* x, const float* w, const float* bias,
                     const float* res, float* y, float* work, long long work_floats, ccb_stream_t stream);
int ccb_conv2d_dgrad(const ccb_conv_desc* d, const float* dy, const float* w, const float* bias,
                     const float* res, float* dx, float* work, long long work_floats, ccb_stream_t stream);
int ccb_conv2d_wgrad(const ccb_conv_desc* d, const float* x, const float* dy, float* dw,
                     float* work, long long work_floats, ccb_stream_t stream);
/* fused: dz = dy * act'(y) (not touched when act == CCB_ACT_NONE; in place allowed) and, when db != NULL,
 * db[c] = sum over (b, pixel) of dz - one pass over the gradient.  work: ccb_act_bwd_bias_workspace_floats() with db,
 * 0 without. */
long long ccb_act_bwd_bias_workspace_floats(int B, int C, int plane);
int ccb_act_bwd_bias(const float* dy, const float* y, float* dz, float* db, int B, int C, int plane, int act, float slope,
                     float* work, long long work_floats, ccb_stream_t stream);
/* bring-up / diagnostic entry points (ccb_debug_*): include/ccb200_debug.h - not part of the drop-in boundary */

/* Back2Future operators (models/back2future.py).
 * corr81: cost volume of correlate() :15-25 (third-party spatial_correlation_sample, kernel 1, patch 9,
 * zero padded, divided by C) with the reference's channel permutation baked in (reversed=0: idx_fwd,
 * 1: idx_bwd, :56-59).  f1,f2 [B,C,h,w] -> out [B,81,h,w].   d_f1 / d_f2 may be NULL.
 * featwarp: Model.warp :287-321 = grid_sample(x, grid+flow, padding border, align_corners False). */
/* work: per-channel-chunk partial sums (0 when one CTA per tile sums all channels) */
long long ccb_corr81_fwd_workspace_floats(int B, int C, int h, int w);
int ccb_corr81_fwd(const float* f1, const float* f2, float* out, int B, int C, int h, int w, int reversed,
                   float* work, long long work_floats, ccb_stream_t stream);
/* work: the mirrored gradient planes with d_f2, 0 without */
long long ccb_corr81_bwd_workspace_floats(int B, int C, int h, int w);
int ccb_corr81_bwd(const float* f1, const float* f2, const float* grad_out, float* d_f1, float* d_f2, int B,
                   int C, int h, int w, int reversed, float* work, long long work_floats, ccb_stream_t stream);
/* FlowNetC6 operator (models/FlowNetC6.py).
 * corr441d: correlate() :18-30 (third-party spatial_correlation_sample, kernel 1, patch 21, stride 1, padding 0,
 * dilation_patch 2, divided by C) with corr_activation LeakyReLU(0.1) :54,112 fused:
 *   out[b, 21 i + j, y, x] = leaky((1/C) sum_c f1[b,c,y,x] f2[b,c,y + 2(i-10), x + 2(j-10)]), zero outside the map.
 * f1,f2 [B,C,h,w] -> out [B,441,h,w].  Backward takes the forward's `out` (the activation derivative comes from its sign);
 * d_f1 / d_f2 may be NULL (not both).  No workspace: every element is summed in a fixed order by one thread. */
int ccb_corr441d_fwd(const float* f1, const float* f2, float* out, int B, int C, int h, int w, ccb_stream_t stream);
int ccb_corr441d_bwd(const float* f1, const float* f2, const float* out, const float* grad_out, float* d_f1, float* d_f2,
                     int B, int C, int h, int w, ccb_stream_t stream);
int ccb_featwarp_fwd(const float* x, const float* flow, int B, int C, int h, int w, float* out,
                     ccb_stream_t stream);
/* d_flow / d_x may be NULL; the gradient is ADDED to d_x; with d_x, work holds B*C*h*w + 1 words (as flow_warp_bwd) */
int ccb_featwarp_bwd(const float* x, const float* flow, int B, int C, int h, int w, const float* grad_out,
                     float* d_flow, float* d_x, unsigned long long* work, long long work_words, ccb_stream_t stream);

/* BatchNorm2d over [B,C,plane] (DispResNet6.py:45-52).  training: batch statistics, stats[C][2] =
 * {mean, invstd} saved for backward, running stats updated in place (momentum, unbiased var). */
long long ccb_bn_workspace_floats(int B, int C, int plane);   /* `work` of both calls; bn_fwd needs 0 in eval mode */
int ccb_bn_fwd(const float* x, const float* gamma, const float* beta, float* y, float* stats,
               float* running_mean, float* running_var, int B, int C, int plane, float eps, float momentum,
               int training, float* work, long long work_floats, ccb_stream_t stream);
int ccb_bn_bwd(const float* x, const float* dy, const float* gamma, const float* stats, float* dx,
               float* dgamma, float* dbeta, int B, int C, int plane, float* work, long long work_floats,
               ccb_stream_t stream);
/* bilinear x2 upsample, align_corners=False (DispResNet6.py:174; back2future.py:60): [planes,h,w] -> [planes,2h,2w] */
int ccb_upsample2x_fwd(const float* x, float* y, int planes, int h, int w, ccb_stream_t stream);
int ccb_upsample2x_bwd(const float* dy, float* dx, int planes, int h, int w, ccb_stream_t stream);
/* torch.optim.Adam step (train.py:307-310,568) over listed ranges of flat fp32 buffers (params, grads, exp_avg,
 * exp_avg_sq), each range belonging to one parameter group with its own step counter (torch.optim.Adam keeps one per
 * parameter; a network that is fixed for a phase of training, train.py --fix-*, keeps its count).  grad_scale
 * pre-multiplies the gradient (1/world_size after the NCCL all-reduce sum).  ranges: device table of nranges entries
 * {offset, count, group, first_block}, where first_block is the number of 256-element blocks of the entries before it;
 * nblocks is that number over all entries.  Elements outside the listed ranges are neither read nor written.
 * group_state: 4*ngroups device floats, group g at [4g, 4g+4) = {step count, 1-b1^t, sqrt(1-b2^t), unused},
 * zero-initialised by the caller; group_active: ngroups device ints, the prep step advances the counter and bias
 * corrections of the groups that are non-zero there (NULL: all).  The counters are incremented on the device, so a
 * captured CUDA graph of the training step replays correctly.  One flat buffer of n elements trained as one group is
 * the table {0, n, 0, 0}. */
int ccb_adam_step_ranges(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, const long long* ranges,
                         int nranges, long long nblocks, const int* group_active, int ngroups, float* group_state,
                         float lr, float beta1, float beta2, float eps, float grad_scale, ccb_stream_t stream);
/* ---- callers either side of the step (SURVEY.md 8f N2 / N1) -------------------------------------------------------
 * Validation metrics, reference loss_functions.py:355-467, as fused masked reductions (deterministic, no host sync).
 * ccb_flow_metrics: gt [B,nc,Hg,Wg] (nc 3: third channel = valid mask; nc 2: plain mean), predictions [B,2,hp,wp]
 *   bilinearly resized to the ground truth (F.upsample(size=gt) = align_corners False) and rescaled by Wg/wp, Hg/hp.
 *   pred_nonrigid / rigidity_mask NULL: out4 = {compute_epe :368-387, -, -, outlier_err :389-407 with tau = (tau0, tau1)}.
 *   Otherwise compute_all_epes :409-427 (mask [B,1,hm,wm], composite by mask > thresh at prediction resolution,
 *   ground truth split at its own): out4 = {all, rigid, non-rigid EPE, outliers}.
 *   epe_map (optional, [B,Hg,Wg]) receives flow_diff :355-365 of the (composited) prediction.
 * ccb_depth_errors: compute_errors :430-467 on gt, pred [B,H,W]: valid = 0 < gt < 80 (inside the Garg crop when
 *   crop != 0), pred clamped to [1e-3, 80] and scaled by median(gt)/median(pred) per sample (lower medians, by radix
 *   select on the device), out6 = batch means of {abs_diff, abs_rel, sq_rel, a1, a2, a3}. */
long long ccb_flow_metrics_workspace_bytes(int B, int Hg, int Wg);
int ccb_flow_metrics(const float* gt, const float* pred_rigid, const float* pred_nonrigid, const float* rigidity_mask,
                     int B, int nc, int Hg, int Wg, int hp, int wp, int hm, int wm, float thresh, float tau0,
                     float tau1, float* epe_map, void* work, long long work_bytes, float* out4, ccb_stream_t stream);
long long ccb_depth_errors_workspace_bytes(int B, int H, int W);
int ccb_depth_errors(const float* gt, const float* pred, int B, int H, int W, int crop, void* work, long long work_bytes,
                     float* out6, ccb_stream_t stream);
/* Motion segmentation scores of one sample each (test_mask.py:129-156, mask_error :224-262), no host sync.  emask
 * [B,C,h,w] is the mask net's eval output (C >= 3; channels 1 and 2 are read), flow_cam and flow [B,2,h,w], obj_map and
 * semantic_map [B,Hg,Wg] hold label values as floats.  Three rigidity masks at h x w:
 *   bare = 1 - (1-e1)(1-e2) > 0.5;  census = soft > thresh with soft = 1 - d/max(d), d = |flow_cam - flow|_2 and the
 *   maximum taken per sample (the reference runs batch 1);  combined = bare or census.
 * d, the division and the subtraction are single correctly rounded fp32 operations (no contraction, no approximate
 * division or root), so the counts are those of an IEEE evaluation of the expressions operation by operation;
 * max(d) = 0 gives NaN and an empty census as in the reference.
 * counts [B,3,4]: per sample and mask {combined, census, bare} the confusion matrix n[pred][gt] = {n00, n01, n10, n11}
 * over the ground-truth pixels with semantic_map == car_label, where gt = (obj_map != 0), pred = 0 where the mask is 1
 * (argmax([mask, 1-mask])), and the mask is read at the pixel scipy.ndimage.zoom(order=0) reads: index
 * floor(o (n_in-1)/(n_out-1) + 0.5) per axis, in fp64.  mask_error's six numbers are tp0 = n00, fp0 = fn1 = n01,
 * fn0 = fp1 = n10, tp1 = n11.  The counts are summed with 64-bit integer atomics: integer addition is associative, so
 * every run gives the same counts.
 * masks (optional, [B,4,h,w]) receives combined, census, bare as 0/1 and soft. */
long long ccb_mask_iou_workspace_bytes(int B, int h, int w, int Hg, int Wg);
int ccb_mask_iou(const float* emask, const float* flow_cam, const float* flow, const float* obj_map,
                 const float* semantic_map, int B, int C, int h, int w, int Hg, int Wg, float thresh, int car_label,
                 float* masks, void* work, long long work_bytes, long long* counts, ccb_stream_t stream);
/* The KITTI-2015 flow submission of one sample each (submit_flow.py:119-156), no host sync.  emask [B,C,h,w] (C >= 3),
 * flow_cam and flow_fwd [B,2,h,w] at the nets' resolution:
 *   combined = bare or census, bare = 1 - (1-e1)(1-e2) > 0.5, census = |cam - fwd| < thresh in u and in v  -> mask [B,1,h,w]
 *   total = (combined <= thresh) * fwd + (combined > thresh) * cam
 * total, fwd and cam resized bilinearly to Hg x Wg as torch's CPU interpolate(align_corners=False) computes it when
 * both axes change size and Wg >= 16 (fma source index, fma per axis, x inside y; see io_ops.cu), u times (float)(Wg/w) and v times (float)(Hg/h):
 *   full  (optional) [B,3,2,Hg,Wg]  cam, fwd, total, fp32
 *   png   [B,Hg,Wg,3] uint16        KITTI triplet of total: (uint16)(u*64.0 + 2^15) in fp64 with numpy's x86-64 cast
 *                                   (truncate to int32, keep the low 16 bits: flows past +-512 px wrap), valid = 1
 *   flo   [B,Hg,Wg,2] fp32          the .flo payload of total (u, v interleaved) */
int ccb_flow_submit(const float* emask, const float* flow_cam, const float* flow_fwd, int B, int C, int h, int w, int Hg,
                    int Wg, float thresh, float* mask, float* full, unsigned short* png, float* flo, ccb_stream_t stream);
/* The KITTI-2015 flow scores of one sample each (test_flow.py:112-140, test_back2future.py), no host sync.  emask
 * [B,C,h,w] (C >= 3; channels 1 and 2 are read), flow_cam and flow_fwd [B,2,h,w] at the nets' resolution, flow_gt
 * [B,3,Hg,Wg] (u, v, valid), obj_map [B,Hg,Wg] (labels as floats):
 *   combined = bare or census, bare = 1 - (1-e1)(1-e2) > 0.5, census = |cam - fwd| < thresh in u and in v, each step
 *   one rounded fp32 operation (0 or 1; written to combined [B,1,h,w] when it is not NULL)
 *   out [B,8] = compute_all_epes(gt, cam, fwd, combined) and compute_all_epes(gt, cam, fwd, 1 - obj), each {all, rigid,
 *   non-rigid EPE, Fl} with compute_all_epes' own THRESH epe_thresh (kept apart from thresh) and tau = (tau0, tau1),
 *   with ccb_flow_metrics' semantics per sample (batch 1).
 * emask and flow_cam NULL: test_back2future.py's compute_all_epes(gt, fwd, fwd, 1 - obj) alone, in out[:, 4:8]; out[:, 0:4]
 * is not written.  fp64 block partials per sample with a fixed-order finalize: the same bits on every run and at any B. */
long long ccb_flow_eval_workspace_bytes(int B, int h, int w, int Hg, int Wg);
int ccb_flow_eval(const float* emask, const float* flow_cam, const float* flow_fwd, const float* flow_gt,
                  const float* obj_map, int B, int C, int h, int w, int Hg, int Wg, float thresh, float epe_thresh,
                  float tau0, float tau1, float* combined, void* work, long long work_bytes, float* out, ccb_stream_t stream);
/* Middlebury flow colours (flowlib.py flow_to_image / compute_color), no host sync.  flow [B,P,2,H,W]: per image P
 * panels stacked along H as np.hstack stacks CHW arrays, normalised by ONE maximum radius -> out [B,3,P*H,W] uint8
 * levels (the reference's float image times 255).  |u| or |v| > 1e7 is unknown (black, left out of the maximum); NaN
 * pixels are black and make the maximum -1, as python's max(-1, nan) does; the colour pass runs in fp64. */
long long ccb_flow_color_workspace_bytes(int B, int P, int H, int W);
int ccb_flow_color(const float* flow, int B, int P, int H, int W, void* work, long long work_bytes, unsigned char* out,
                   ccb_stream_t stream);
/* Colormaps of utils.py tensor2array as run_inference.py saves them, (255 * tensor2array(x, max, colormap)).astype(uint8),
 * no host sync.  maps [B,H,W] fp32 (1/x first, in fp32, when invert != 0) -> out [B,H,W,3] uint8 through lut [N,3] uint8
 * (device): t = (x / max) * N, each rounded in fp32; NaN is black, t < 0 takes lut[0], t >= N lut[N-1], else lut[trunc(t)].
 * max is max_value, or each image's own maximum (any NaN makes it NaN, as torch.max) when per_image_max != 0; only then
 * is a workspace needed. */
long long ccb_colorize_workspace_bytes(int B, int H, int W, int per_image_max);
int ccb_colorize(const float* maps, int B, int H, int W, const unsigned char* lut, int N, int invert, int per_image_max,
                 float max_value, void* work, long long work_bytes, unsigned char* out, ccb_stream_t stream);
/* KITTI flow scores of two 16-bit triplets each (evaluate_flow.py compute_err :44-53 on flow_read_png's decoding), no host
 * sync.  gt and pred [B,H,W,3] uint16 -> out [B,2] fp64 (aepe, Fl) and optionally counts [B,2] (outliers weighted by
 * valid_gt, sum of valid_gt).  fp64 block partials with a fixed-order finalize: the same bits on every run. */
long long ccb_kitti_flow_errors_workspace_bytes(int B, int H, int W);
int ccb_kitti_flow_errors(const unsigned short* gt, const unsigned short* pred, int B, int H, int W, void* work,
                          long long work_bytes, double* out, long long* counts, ccb_stream_t stream);
/* Depth evaluation of test_disp.py on the device, no host sync.
 * ccb_velo_depth: KITTI ground truth of B velodyne sweeps (kitti_eval/depth_evaluation_utils.py generate_depth_map
 *   :148-191).  points [total,4] fp32 (column 3 is not read), offsets [B+1] int64 (sample b owns points
 *   offsets[b] .. offsets[b+1]-1; malformed offsets give the sample no point), P_velo2im [B,3,4] fp64 -> depth [B,H,W] fp64.
 *   Points with x >= 0 are projected in fp64, u = round(X/Z) - 1 and v = round(Y/Z) - 1 half to even, kept inside the
 *   frame; each pixel takes the Z of its last point; for every sub2ind key v*(W-1) + u - 1 shared by several points the
 *   pixel of the first of them takes their least Z; negative depths become 0.  Integer atomics: the same bits every run.
 * ccb_spline_zoom: scipy.ndimage.zoom(order=3) of src [N,h,w] fp32 to dst [N,H,W] fp32 (mirror-initialised cubic
 *   B-spline prefilter along rows then columns, evaluation at o*(n-1)/(m-1), all in fp64), then clip(lo, hi) in fp32.
 * ccb_eigen_depth_errors: the errors of one sample each (test_disp.py:124-141, compute_errors :171-187) of gt [B,H,W] fp64
 *   and the zoomed, clipped prediction pred [B,H,W] fp32 over mask = min_depth < gt < max_depth inside the crop
 *   crop (host, 4 fractions in [0,1]: rows [int(crop[0]*H), int(crop[1]*H)), columns [int(crop[2]*W), int(crop[3]*W))).
 *   out [B,2,7] fp64 = abs_rel sq_rel rms log_rms a1 a2 a3; row 1 scales pred by median(gt)/median(pred) (numpy medians),
 *   row 0 by the mean of displacements/|poses[:3]| over the displacements > 0 (0 if none; poses [B,R,6] fp32,
 *   displacements [B,R] fp64), zeros when poses is NULL.  a1..a3 are exact counts; the other sums are fp64 block partials
 *   with a fixed-order finalize. */
long long ccb_velo_depth_workspace_bytes(int B, int H, int W);
int ccb_velo_depth(const float* points, const long long* offsets, const double* P_velo2im, long long total, int B, int H, int W,
                   void* work, long long work_bytes, double* depth, ccb_stream_t stream);
long long ccb_spline_zoom_workspace_bytes(int N, int h, int w);
int ccb_spline_zoom(const float* src, int N, int h, int w, int H, int W, float lo, float hi, void* work, long long work_bytes,
                    float* dst, ccb_stream_t stream);
long long ccb_eigen_depth_errors_workspace_bytes(int B, int H, int W);
int ccb_eigen_depth_errors(const double* gt, const float* pred, int B, int H, int W, double min_depth, double max_depth,
                           const double* crop, const float* poses, const double* displacements, int R, void* work,
                           long long work_bytes, double* out, ccb_stream_t stream);
/* Make3D depth evaluation of test_make3d.py on the device, no host sync.
 * ccb_bytescale_u8: the contrast stretch scipy.misc.imresize (scipy 1.1: toimage -> bytescale) applies to a float32 image
 *   before Pillow resizes it (test_make3d.py:100-102), of src [N,H,W,3] uint8 (the float32 frame holds integers) into
 *   dst [N,H,W,3] uint8: over each whole image cmin, cmax, cscale = cmax - cmin (1 when 0), scale = 255 / cscale and
 *   dst = trunc(clip((src - cmin) * scale, 0, 255) + 0.5), every operation rounded in float32 on its own (no fused
 *   multiply-add).  The range is taken with integer atomics: the same bytes every run.
 * ccb_make3d_depth_errors: the errors of one sample each (test_make3d.py:139-148, compute_errors :174-190) of gt [B,H,W]
 *   fp64 and the zoomed, clipped prediction pred [B,H,W] fp32 over mask = min_depth < gt < max_depth (no crop).
 *   out [B,2,7] fp64: row 0 zeros (the script never writes it), row 1 = abs_rel sq_rel rms log_rms a1 a2 a3 of
 *   min(pred * median(gt)/median(pred), max_depth) with numpy's medians, the product in fp64, and log_rms of log10.
 *   An empty mask gives a NaN row.  The workspace and the reductions are those of ccb_eigen_depth_errors. */
long long ccb_bytescale_u8_workspace_bytes(int N, int H, int W);
int ccb_bytescale_u8(const unsigned char* src, int N, int H, int W, void* work, long long work_bytes, unsigned char* dst,
                     ccb_stream_t stream);
long long ccb_make3d_depth_errors_workspace_bytes(int B, int H, int W);
int ccb_make3d_depth_errors(const double* gt, const float* pred, int B, int H, int W, double min_depth, double max_depth,
                            void* work, long long work_bytes, double* out, ccb_stream_t stream);
/* Pose evaluation of test_pose.py / test_sintel_pose.py on the device, no host sync, no workspace: one thread per snippet.
 * ccb_pose_errors: poses [S,L-1,6] fp32 is the pose net's output for S snippets of L frames (L odd, 3 <= L <= 15).  Per
 *   snippet (test_pose.py:74-92): a zero six-vector inserted at mid = L/2; each six-vector -> [R_i|t_i] in fp32 with
 *   pose_vec2mat's arithmetic (rot_mode CCB_ROT_EULER / CCB_ROT_QUAT), cast to fp64; rot_i = inv(R_i) (a true inverse,
 *   not a transpose); final_i = R_0 [rot_i | -rot_i t_i], final_i[:, 3] += t_0, written to final_poses [S,L,3,4] fp64
 *   when it is not NULL.  gt [S,L,3,4] fp64 is the compensated ground truth the framework yields (Sintel's float32 gt
 *   upcast exactly); with it out [S,2] fp64 = compute_pose_error (:107-122):
 *     ATE = ||gt_t - k pred_t|| / L with k = sum(gt_t pred_t) / sum(pred_t^2) (NaN when every pred_t is zero, as numpy),
 *     RE = sum_i atan2(||(R01-R10, R12-R21, R02-R20)||, tr R - 1) / L with R = gt_i[:, :3] inv(final_i[:, :3]).
 *   gt and out come together; at least one of out and final_poses is written.  Every run gives the same bits. */
int ccb_pose_errors(const float* poses, int S, int L, int rot_mode, const double* gt, double* final_poses, double* out,
                    ccb_stream_t stream);
/* Input pipeline on the device (train.py:448-451 H2D + custom_transforms.py:21-30,47-118): uint8 HWC frames
 * src [B,F,Hs,Ws,3] -> F normalised fp32 NCHW tensors dst[f] [B,3,H,W] = (v/255 - .5)/.5, per sample horizontally
 * flipped (params[b][0] != 0) and scale-cropped: resized by (params[b][1], params[b][2]) = (scaled_w/Ws, scaled_h/Hs)
 * with a half-pixel-centre bilinear lookup, then cropped at offs[b] = (x0, y0).  params [B,4] floats, offs [B,2] ints,
 * device memory; dst = host array of F device pointers. */
int ccb_prep_frames(const unsigned char* src_u8, float* const* dst, const float* params, const int* offs, int B, int F,
                    int Hs, int Ws, int H, int W, ccb_stream_t stream);
/* The same lookup writing v/255 only (ArrayToTensor without Normalize), for ccb_normalize_local to follow. */
int ccb_prep_frames_unit(const unsigned char* src_u8, float* const* dst, const float* params, const int* offs, int B, int F,
                         int Hs, int Ws, int H, int W, ccb_stream_t stream);
/* The same lookup writing run_inference.py's (v/255 - .5)/.2. */
int ccb_prep_frames_inference(const unsigned char* src_u8, float* const* dst, const float* params, const int* offs, int B,
                              int F, int Hs, int Ws, int H, int W, ccb_stream_t stream);
/* RandomRotate (custom_transforms.py:75-85) = scipy.misc.imrotate = Pillow Image.rotate(angle, BILINEAR), bit-exact:
 * src, dst [B,F,H,W,3] uint8 (not in place); affine [B,6] fp64 maps an output pixel centre (x+.5, y+.5) to the input point
 * (a0 x + a1 y + a2, a3 x + a4 y + a5), as Pillow builds it (cc_b200.input_pipeline.pil_rotate_affine); the identity
 * leaves a sample's frames unchanged.  Points outside the frame give 0. */
int ccb_rotate_frames_u8(const unsigned char* src, const double* affine, unsigned char* dst, int B, int F, int H, int W,
                         ccb_stream_t stream);
/* Scale (custom_transforms.py:120-137) = scipy.misc.imresize = Pillow resize((W, H), BILINEAR), bit-exact (8-bit
 * ImagingResample: antialiased on a downscale, 22-bit fixed-point weights, horizontal pass first, each pass rounded to
 * uint8): src [N,Hs,Ws,3] -> dst [N,H,W,3] uint8.  The weights are computed on the device into `work`, so the call is
 * asynchronous and can be captured in a graph. */
long long ccb_resize_u8_workspace_bytes(int N, int Hs, int Ws, int H, int W);
int ccb_resize_u8(const unsigned char* src, unsigned char* dst, int N, int Hs, int Ws, int H, int W, void* work,
                  long long work_bytes, ccb_stream_t stream);
/* NormalizeLocally (custom_transforms.py:33-44) in place on F frames[f] [B,3,H,W]: per sample and channel, the mean and
 * unbiased std over all F*H*W values (fp64, deterministic), rounded to fp32, then x = (x - m) / s in fp32.  stats
 * ([B,3,2] = {mean, std}) may be NULL.  A zero std gives inf / nan, as in the reference. */
long long ccb_normalize_local_workspace_bytes(int B, int H, int W);
int ccb_normalize_local(float* const* frames, int B, int F, int H, int W, float* stats, void* work, long long work_bytes,
                        ccb_stream_t stream);
/* number of kernel launches issued through this library by the calling process so far */
long long ccb_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* CCB200_H */
