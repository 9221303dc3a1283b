/*
 * council_b200.h -- C ABI of libcouncil_b200.so: the sm_90a kernels behind the Council-GAN
 * training step (dis_update / dis_council_update / gen_update).
 *
 * The reference (Onr/Council-GAN) has no FFI: every device op on this path is a PyTorch library
 * call made from networks.py / trainer_council.py.  Each entry point below replaces one of those
 * call sites (cited per function, paths relative to the reference tree) so that a maintainer can
 * bind it with ctypes (see INTEGRATION.md) from the same Python code.
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless named host_*;
 *   - all tensors are dense fp32; activations are channels-last, stacked over the council:
 *         act[G][B][H][W][C]      G = council members in the launch ("groups"), C % 4 == 0
 *     a source with `x_groups == 1` is shared (broadcast) by all G members;
 *   - convolution weights are stacked OHWI:  w[G][Cout][KH][KW][Cin]   (reference: OIHW per member);
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*), never allocates,
 *     and returns 0 on success or a negative cg_status; cg_last_error() describes the last failure
 *     of the calling thread;
 *   - `ws` / `ws_bytes` is caller-provided scratch; if it is too small the call fails with
 *     CG_ERR_WORKSPACE and cg_last_error() reports the size needed.
 */
#ifndef COUNCIL_B200_H
#define COUNCIL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    CG_OK = 0,
    CG_ERR_ARG = -1,        /* unsupported shape / argument */
    CG_ERR_WORKSPACE = -2,  /* workspace too small */
    CG_ERR_CUDA = -3,       /* CUDA runtime / driver error */
    CG_ERR_NO_DEVICE = -4   /* no CUDA device */
} cg_status;

/* activation codes (Conv2dBlock activations, networks.py:494-507) */
enum { CG_ACT_NONE = 0, CG_ACT_RELU = 1, CG_ACT_LRELU = 2, CG_ACT_TANH = 3 };

/* Geometry of one grouped convolution.  Spatial sizes are those of the STORED input tensor;
 * with `ups` the convolution sees nearest-upsample-x2 of it (nn.Upsample(scale_factor=2),
 * networks.py:385, folded into the gather).  Ho/Wo are the output sizes. */
typedef struct {
    int32_t G, x_groups;         /* groups in w / y; groups in x (1 = shared input) */
    int32_t B, H, W, Cin;        /* stored input  [x_groups][B][H][W][Cin]  */
    int32_t Ho, Wo, Cout;        /* output        [G][B][Ho][Wo][Cout]      */
    int32_t KH, KW, stride, pad; /* zero padding (nn.ZeroPad2d, networks.py:473-474) */
    int32_t ups;                 /* 0/1 */
} cg_conv_geom;

const char* cg_last_error(void);
/* Library / device introspection: returns the SM count of the current device (>0) or a cg_status. */
int cg_device_info(int* sm_count, int* cc_major, int* cc_minor);
/* 0 = SIMT fp32 kernels only; 1 (default) = TF32 tensor-core kernels (wgmma / mma.sync) wherever a layer qualifies;
 * other values are a bit mask for bring-up: 2 = data gradient only, 4 = weight gradient only, ...
 * (internally 1 forward | 2 dgrad | 4 wgrad).  Switches on top of the mask: 1<<22 = programmatic dependent launch between this
 * library's kernels (every kernel carries the griddepcontrol pair; the trainer turns it on for small maps only),
 * 1<<23 = keep the widest N tile on small maps
 * (default: narrower tiles when a launch has fewer tiles than SMs), 1<<25 = weight gradients of stride-1 and stride-2 KxK layers
 * on the previous tensor-core kernel, which transposes both operands in the MMA warps, for comparisons in one process (default:
 * the TMA-fed kernel that reads one operand from a channel-major copy), 1<<26 = the previous epilogue and tile walk of the
 * forward / data-gradient tensor-core kernel, which load the addend and mask one column group at a time and walk the parity
 * classes outermost, for comparisons in one process (same results), 1<<27 = every forward / data-gradient tensor-core launch on
 * the register epilogue (default: the shared-memory epilogue, TMA-loaded addend and mask and TMA-stored results, wherever the
 * tile geometry allows it), for comparisons in one process (same results).  Other bits are accepted and ignored.
 * The switches are per calling thread (like cg_last_error), not process-global.  Returns the previous mask. */
int cg_set_tensor_core_mode(int mode);
/* number of kernels launched by this library since load (bench.py reports it as gpu_launches) */
uint64_t cg_launch_count(void);
/* TMA descriptors are cached by (device pointer, geometry): hits / misses since load (bench.py reports them) */
void cg_tensor_map_cache_stats(uint64_t* hits, uint64_t* misses);

/* ---- convolution (Conv2dBlock conv + bias + activation, networks.py:513-520; nn.Linear with
 *      H=W=KH=KW=1, networks.py:531,563) ------------------------------------------------------- */
/* y = act(conv(x, w) + bias).  bias may be NULL. */
int cg_conv_fwd(const cg_conv_geom* g, const float* x, const float* w, const float* bias, float* y,
                int act, float slope, void* ws, size_t ws_bytes, void* stream);
/* y = conv(x, w) (no bias, no activation) and the instance-norm statistics of y in one call (Conv2d followed by
 * InstanceNorm2d / AdaIN, networks.py:516-518): mean, rstd [G][B][Cout].  On the tensor path the per-channel sums come
 * out of the convolution epilogue, saving a pass over y. */
int cg_conv_fwd_stats(const cg_conv_geom* g, const float* x, const float* w, float* y, float* mean, float* rstd,
                      float eps, void* ws, size_t ws_bytes, void* stream);
size_t cg_conv_fwd_stats_workspace_bytes(const cg_conv_geom* g);
/* dx = (conv_transpose(dy, w) [+ addend]) * act'(mask_src)      (autograd of the call above)
 * dx has the STORED input shape; with g->ups the 2x2 upsample fan-in is summed.
 * addend / mask_src (same shape as dx) may be NULL; act' = mask_src > 0 ? 1 : mask_slope. */
int cg_conv_dgrad(const cg_conv_geom* g, const float* dy, const float* w, float* dx,
                  const float* addend, const float* mask_src, float mask_slope,
                  void* ws, size_t ws_bytes, void* stream);
/* dw[G][Cout][KH][KW][Cin] = sum over pixels dy (x) im2col(x);  db[G][Cout] = sum dy (NULL: skip).
 * Deterministic (fixed split-K order). */
int cg_conv_wgrad(const cg_conv_geom* g, const float* x, const float* dy, float* dw, float* db,
                  void* ws, size_t ws_bytes, void* stream);
size_t cg_conv_workspace_bytes(const cg_conv_geom* g, int which /*0 fwd, 1 dgrad, 2 wgrad*/);

/* ---- instance norm / AdaIN (nn.InstanceNorm2d networks.py:483; AdaptiveInstanceNorm2d :640-653) */
/* mean, rstd [G][B][C] over H*W (biased variance, rstd = 1/sqrt(var+eps)). */
int cg_in_stats(const float* y, float* mean, float* rstd, int G, int B, int HW, int C, float eps,
                void* ws, size_t ws_bytes, void* stream);
/* z = act(gamma * (y-mean)*rstd + beta) [+ res];  AdaIN parameters come straight from the MLP
 * output adain[G][B][P]: beta = adain[.., off : off+C], gamma = adain[.., off+C : off+2C]
 * (assign_adain_params, networks.py:303-312).  adain == NULL: plain instance norm.
 * ups: z is written nearest-upsampled x2 ([G][B][2H][2W][C]).  res (shape of y) may be NULL. */
int cg_norm_act_fwd(const float* y, const float* mean, const float* rstd, const float* adain, int P,
                    int off, const float* res, float* z, int G, int B, int H, int W, int C, int act,
                    int ups, void* stream);
/* backward of the above w.r.t. y and the AdaIN parameters (d_adain[..][off:off+2C] is overwritten).
 * dz has the shape of z (upsampled if ups).  The residual branch gradient is dz itself. */
int cg_norm_act_bwd(const float* dz, const float* y, const float* mean, const float* rstd,
                    const float* adain, int P, int off, float* dy, float* d_adain, int G, int B,
                    int H, int W, int C, int act, int ups, void* ws, size_t ws_bytes, void* stream);

/* act may also be CG_ACT_LRELU (slope 0.2, as Conv2dBlock fixes it: the discriminators' dis.norm in). */

/* ---- layer norm (LayerNorm networks.py:659-686: the discriminators' dis.norm ln) ------------------------------------ */
/* mean[G][B] and the UNBIASED std[G][B] (torch.std) of each sample over C*H*W; fp64 fixed-order fold of fp32 partials of
 * 128 pixels, so the result is deterministic.  Needs C*H*W > 1.  Workspace: cg_ln_workspace_bytes. */
size_t cg_ln_workspace_bytes(int G, int B, int HW, int C);
int cg_ln_stats(const float* y, float* mean, float* std, int G, int B, int HW, int C, void* ws, size_t ws_bytes, void* stream);
/* z = act((y - mean) / (std + eps) * gamma[g][c] + beta[g][c]); gamma, beta [G][C] (one row per member). */
int cg_ln_act_fwd(const float* y, const float* mean, const float* std, const float* gamma, const float* beta, float eps,
                  float* z, int G, int B, int H, int W, int C, int act, void* stream);
/* backward of the above (the autograd of (y - mean) / (std + eps) with the unbiased std, statistics included; at std 0 the
 * term through the std is taken as 0): dy, and dgamma / dbeta [G][C] summed over each member's samples (overwritten, like
 * cg_conv_wgrad's db). */
int cg_ln_act_bwd(const float* dz, const float* y, const float* mean, const float* std, const float* gamma,
                  const float* beta, float eps, float* dy, float* dgamma, float* dbeta, int G, int B, int H, int W, int C,
                  int act, void* ws, size_t ws_bytes, void* stream);

/* backward of nn.Upsample(scale_factor=2) (networks.py:385): dx[N][H][W][C] = 2x2 fan-in sum of d_up[N][2H][2W][C] */
int cg_upsample2x_bwd(const float* d_up, float* dx, int N, int H, int W, int C, void* stream);

/* ---- attention-mask head (Decoder_V2_atten.forward networks.py:398-407) ----------------------- */
/* h[G][B][HW][12] = tanh output of dec.model.9; x_in[B][HW][4] (shared); outputs padded to 4 ch. */
int cg_mask_head_fwd(const float* h, const float* x_in, float* x_fake, float* mask, int G, int B,
                     int HW, void* stream);
/* dh_pre[G][B][HW][12] = gradient w.r.t. the PRE-tanh output of dec.model.9. d_mask may be NULL. */
int cg_mask_head_bwd(const float* h, const float* x_in, const float* d_xfake, const float* d_mask,
                     float* dh_pre, int G, int B, int HW, void* stream);

/* The decoder tail of a no-grad pass in ONE launch (csrc/head_fused.cu): y[G][B][HW][64] = raw output of the last 3x3 block;
 * z = relu(AdaIN(y)) -> 1x1 64->64 + relu (w1, b1) -> 1x1 64->64 + relu (w2, b2) -> 1x1 64->12 + tanh (w3, b3) -> mask
 * compositing with x_in (cg_mask_head_fwd).  Weights [G][Cout][64], HW % 128 == 0.  Replaces cg_norm_act_fwd + 3 x cg_conv_fwd +
 * cg_mask_head_fwd (Decoder_V2_atten, networks.py:391-407) when nothing has to be kept for a backward pass. */
int cg_head_fused(const float* y, const float* mean, const float* rstd, const float* adain, int P, int off, const float* w1,
                  const float* b1, const float* w2, const float* b2, const float* w3, const float* b3, const float* x_in,
                  float* x_fake, float* mask, int G, int B, int HW, void* stream);

/* ---- image-space helpers ---------------------------------------------------------------------- */
/* nn.AvgPool2d(3, 2, padding=1, count_include_pad=False), networks.py:32,129 */
int cg_avgpool_fwd(const float* x, float* y, int N, int H, int W, int C, void* stream);
/* global average pool of the style encoder (networks.py:348): y[N][C] = mean over HW of h[N][HW][C] (pixel-order float sum / HW);
 * backward: dh[N][HW][C] = dy[N][C] / HW, zeroed where h <= 0 when relu_gate (h: the ReLU output that was pooled); C % 4 == 0 */
int cg_global_avgpool_fwd(const float* h, float* y, int N, int HW, int C, void* stream);
int cg_global_avgpool_bwd(const float* dy, const float* h, float* dh, int N, int HW, int C, int relu_gate, void* stream);
/* dx[N][H][W][Cx] (first nch lanes) = or += avgpool^T(dy[N][H/2][W/2][Cy] first nch lanes) */
int cg_avgpool_bwd(const float* dy, float* dx, int N, int H, int W, int Cy, int Cx, int nch,
                   int accumulate, void* stream);
/* dst[n][..][0:nch] += src[n][..][0:nch]  (pixel counts equal) */
int cg_acc_slice(float* dst, const float* src, long npix, int Cd, int Cs, int nch, void* stream);
/* y[g][n] = slot(idx[g*Bt+n]) (4 lanes) ++ x_in[n % B] (4 lanes, if x_in != NULL -> 8-lane output), where
 * slot(k) = k < n0 ? pool0[k] : pool1[k - n0]  (pool1 may be NULL when every index is < n0):
 * builds discriminator minibatches without materialising torch.cat((fake, real)) (networks.py:56-64) or
 * torch.cat((x, x_input), 1) (networks.py:152). */
int cg_gather_images(const float* pool0, int n0, const float* pool1, const int32_t* idx, const float* x_in, float* y,
                     int G, int Bt, int B, int HW, void* stream);
/* do_Dis_only_gray (trainer_council.py:736-737, 761, 765, 504, 510): the slots of cg_gather_images (same arguments; x_in must be
 * NULL) converted to gray scale, y[g][n] = {m, m, m, 0} with m = (x0 + x1 + x2) / 3 (summed in that order, then a true division):
 * torch.sum(x, 1).unsqueeze(1).repeat(1, input_dim, 1, 1) / input_dim with input_dim = 3. */
int cg_gather_images_gray(const float* pool0, int n0, const float* pool1, const int32_t* idx, const float* x_in, float* y,
                          int G, int Bt, int B, int HW, void* stream);
/* the data gradient through that conversion, in place on d_x[npix][4]: lanes 0..2 = g0/3 + g1/3 + g2/3 (autograd's order);
 * lane 3 keeps its value */
int cg_gray_fold(float* d_x, long npix, void* stream);
/* useRandomDis (trainer_council.py:499-501): a parameter bank with members drawn from another, dst[g] = src[host_map[g]] in each
 * member-major segment s (floats [host_off[s], host_off[s] + G*host_n[s]) of both buffers, host_off[s] % 4 == 0).  host_map[G]
 * (host memory, passed by value) may repeat members and map a member to itself: G <= CG_LOSS_MAX_G, 0 <= host_map[g] < G,
 * nseg <= CG_GATHER_MAX_SEG.  Floats outside the segments are not written. */
#define CG_GATHER_MAX_SEG 64
int cg_gather_members(const float* src, float* dst, const int64_t* host_off, const int64_t* host_n, int nseg,
                      const int32_t* host_map, int G, void* stream);
/* NCHW [N][C][HW] <-> channels-last [N][HW][Cp] (Cp >= C, pad lanes zeroed) */
int cg_nchw_to_nhwc(const float* x, float* y, int N, int C, int HW, int Cp, void* stream);
int cg_nhwc_to_nchw(const float* x, float* y, int N, int C, int HW, int Cp, void* stream);

/* ---- losses ----------------------------------------------------------------------------------- */
/* LSGAN (networks.py:64,90,166,194).  out[G][nseg][n_per_seg]; sums[G][nseg] = sum (out-target[seg])^2;
 * loss[g] (+)= sum_seg weights[g][seg] * mean_seg((out-target[seg])^2).  targets: device [nseg]; weights: device [G][nseg]. */
int cg_lsgan_fwd(const float* out, const float* targets, const float* weights, float* sums, float* loss,
                 int G, int nseg, int n_per_seg, int accumulate, void* stream);
/* dout = coef[g][seg] * (out - target[seg])   (coef device pointer, [G][nseg]) */
int cg_lsgan_bwd(const float* out, const float* targets, const float* coef, float* dout, int G,
                 int nseg, int n_per_seg, void* stream);
/* focus-loss sums over a mask [G][B][H][W][4] (3 live lanes), trainer_council.py:230-250:
 * sums[G][4] = { sum 1/(|m-c|+eps), sum m, sum |m[h+1]-m[h]|, sum |m[w+1]-m[w]| } */
int cg_focus_fwd(const float* mask, float* sums, int G, int B, int H, int W, float center, float eps,
                 void* ws, size_t ws_bytes, void* stream);
/* dmask = coef[g][0]*d(zero_one term) + coef[g][1]*d(sum m) + coef[g][2]*d(TV sums) */
int cg_focus_bwd(const float* mask, const float* coef, float* dmask, int G, int B, int H, int W,
                 float center, float eps, void* stream);

/* ---- fused losses (one launch per discriminator update and direction; two per gen_update and direction, two more each with
 *      abs_beginning_end or council_abs_w on) -------------------------------------------------------------------------
 * These replace the four calls above on the training path: the loss of EVERY discriminator scale, the focus terms, the
 * loss-history matching and all their gradients, with no host round trip (trainer_council.py:518-524,576-586 run on the
 * device).  `ws`: >= cg_loss_workspace_bytes() bytes, ZERO-INITIALISED once by the caller, not shared between streams;
 * every call leaves its first 16 bytes (a ticket counter) zero again. */
#define CG_LOSS_MAX_MAPS 4
#define CG_LOSS_MAX_G 8
#define CG_LOSS_MAX_SEG 8
typedef struct {
    int32_t nmaps, G, nseg, _pad;             /* patch maps (discriminator scales), members, segments per member */
    const float* out[CG_LOSS_MAX_MAPS];       /* out[m][G][nseg][n_per_seg[m]]                                      */
    float* dout[CG_LOSS_MAX_MAPS];            /* gradient of the same shape (NULL: not wanted)                      */
    int32_t n_per_seg[CG_LOSS_MAX_MAPS];
    float target[CG_LOSS_MAX_SEG];            /* 0 for generated, 1 for real / less-style segments                  */
    float weight[CG_LOSS_MAX_G][CG_LOSS_MAX_SEG];
    float loss_scale, grad_scale;             /* 1/world under data parallelism                                     */
} cg_lsgan_desc;
/* loss_total[g] (+)= loss_scale * sum_m sum_s weight[g][s] * mean((out-target[s])^2);   loss_plain[g] (NULL: skip) = the
 * same with unit weights;   dout = grad_scale * weight[g][s] * 2/n_per_seg * (out - target[s]).
 * calc_dis_loss networks.py:56-64,158-166 for all scales at once, with its autograd. */
int cg_lsgan_fused(const cg_lsgan_desc* d, float* loss_total, int accumulate, float* loss_plain, void* ws,
                   size_t ws_bytes, void* stream);

typedef struct {
    int32_t G, B, H, W;                       /* mask[G][B][H][W][4]; B = this rank's batch                         */
    int32_t n_adv, n_cl;                      /* scales of MsImageDis / MsImageDisCouncil evaluated on x_fake (0..2) */
    const float* adv_out[2]; float* adv_dout[2];   /* [G][adv_n]; gradient written by pass 1 (constant coefficient)  */
    const float* cl_out[2];  float* cl_dout[2];    /* [G][cl_n];  gradient written by pass 2 (needs w_match)         */
    int32_t adv_n[2], cl_n[2];
    const float* mask;                        /* NULL: no focus terms                                               */
    float center, eps, adv_grad_scale, _pad;  /* d adv_out = adv_grad_scale * 2/adv_n * (out-1): gan_w / world       */
} cg_gen_loss_desc;
typedef struct {
    int32_t world, hist_size, head_gan, head_council;   /* history rings double[G][hist_size+1], window starts at head */
    int32_t gan_on, council_on, focus_on, matching, small_abs, small_square;
    double gan_w, council_w, w01, wtot, wtv;  /* loss weights (0 = term off)                                        */
    double numel;                             /* mask.numel() of the GLOBAL minibatch                               */
    /* do_w_loss_matching_focus (trainer_council.py:398-410, 433-445); all zero = off.  While focus_on, each focus term is
     * scaled by mean(GAN history BEFORE this call's append) / mean(its own history after the append), the ratio rounded to
     * float32: the zero-one term (w01 != 0) through hist_focus01, the mask-total term (wtot != 0) through hist_focus.      */
    int32_t focus_matching, head_focus, head_focus01, _pad;
    double* hist_focus;                       /* double[G][hist_size+1]: appends the unscaled float32 mask-total term  */
    double* hist_focus01;                     /* double[G][hist_size+1]: appends the unscaled float32 zero-one term    */
    const float* focus_src;                   /* NULL, or the pub[G][8] of the a2b call: the b2a history then appends   *
                                               * its column 3, a2b's SCALED mask-total term (:441)                      */
    float* focus_w;                           /* NULL, or [G][2] = { zero-one ratio, mask-total ratio } (1: not scaled)  */
} cg_gen_loss_hp;
/* pass 1: scal[G][6] = { sum_scales mean (D(x)-1)^2, sum_scales mean (DC(x)-1)^2, sum 1/(|m-c|+eps), sum m,
 * sum |dh m|, sum |dw m| } for this rank, and the gradient of the adversarial maps (calc_gen_loss networks.py:84-90,188-194;
 * focus criteria trainer_council.py:230-250). */
int cg_gen_loss_fwd(const cg_gen_loss_desc* d, float* scal, void* ws, size_t ws_bytes, void* stream);
/* pass 2 (scal summed over ranks): assembles the generator loss of every member (trainer_council.py:392-451,497-529,
 * 559-634), appends to the loss histories and derives w_match (:518-524,576-586), publishes
 * pub[G][8] = { total of this direction, adv, zero_one, mask_total, TV, council loss, w_match, raw council },
 * total[g] (+)= direction total, and writes the council-map and mask gradients.  The caller advances head_gan /
 * head_council by one after a call that appended (gan_on && matching / council_on && matching), and head_focus01 /
 * head_focus after a call that appended to those (focus_on && focus_matching, with w01 != 0 / wtot != 0).  With
 * focus_matching, zero_one and mask_total in pub are the scaled values. */
int cg_gen_loss_bwd(const cg_gen_loss_desc* d, const cg_gen_loss_hp* hp, const float* scal, double* hist_gan,
                    double* hist_council, float* total, int accumulate, float* pub, float* d_mask, void* ws,
                    size_t ws_bytes, void* stream);
/* abs_beginning_end: recon_criterion_v2_color(x_fake, x) (trainer_council.py:210-215, 477-495) with d = x_fake - x over the 3 live
 * lanes of x_fake[G][B][H][W][4] and the shared x[1][B][H][W][4] (the generator's input); loss = L1 = mean |d| if L1 > L2 = mean d^2,
 * else L2 (a tie picks L2).
 * pass 1: sums[G][2] = { sum |d|, sum d^2 } for this rank (float partials per block, added in double; fixed order). */
int cg_abs_beginning_end_fwd(const float* x_fake, const float* x, float* sums, int G, int B, int H, int W, void* ws,
                             size_t ws_bytes, void* stream);
/* pass 2 (sums summed over ranks; numel = 3*H*W*B of the GLOBAL minibatch): the branch is chosen from the sums on the device;
 * pub[g] = unweighted loss; d_x (+)= host_weight[g] * (sign(d) / numel  or  2d / numel) on lanes 0..2 (sign(0) = 0);
 * total[g] (+)= host_weight[g] * loss through the double accumulator cg_gen_loss_bwd keeps in the same workspace, so it must
 * follow the cg_gen_loss_bwd call of the same direction on the same workspace and stream.  host_weight[G] (host memory) is
 * passed to the kernel by value; 0 leaves total and d_x of that member untouched. */
int cg_abs_beginning_end_bwd(const float* x_fake, const float* x, const float* sums, double numel, const double* host_weight,
                             float* total, float* pub, float* d_x, int G, int B, int H, int W, void* ws, size_t ws_bytes,
                             void* stream);
/* council abs loss, council_abs_w (trainer_council.py:224-228, 595-619): member g's translation x_fake[g] against the detached
 * translation of its peer x_fake[host_peer[g]], x_fake[G][B][H][W][4]; colour: |d| on the 3 live lanes, gray: |sum_c x_g - sum_c x_p|
 * per pixel.  host_peer[G] (host memory, passed by value) must name another member: G <= CG_LOSS_MAX_G, 0 <= peer < G, peer != g.
 * pass 1: sums[g] = the sum of those over member g on this rank (float partials per block, added in double; fixed order). */
int cg_council_abs_fwd(const float* x_fake, const int32_t* host_peer, int gray, float* sums, int G, int B, int H, int W, void* ws,
                       size_t ws_bytes, void* stream);
/* pass 2 (sums summed over ranks; numel = (gray ? 1 : 3)*H*W*B of the GLOBAL minibatch): pub[g] = w * sums[g] / numel (the weighted
 * term); total[g] += pub[g] through the double accumulator cg_gen_loss_bwd keeps in the same workspace, so it must follow the
 * cg_gen_loss_bwd call of the same direction on the same workspace and stream; d_x[g] += w / numel * sign(d) on lanes 0..2 (gray: the
 * sign of the channel-sum difference on all three; sign(0) = 0).  Lane 3 keeps its value; the peer takes no gradient. */
int cg_council_abs_bwd(const float* x_fake, const int32_t* host_peer, int gray, const float* sums, double numel, double w, float* total,
                       float* pub, float* d_x, int G, int B, int H, int W, void* ws, size_t ws_bytes, void* stream);
/* latent reconstruction, recon_c_w / recon_s_w (trainer_council.py:359-369, 460-469): recon_criterion(a, b) = mean |a - b| of a
 * re-encoded code a[G][n] against its target b ([G][n], or [n] shared by all members when b_shared).
 * sums[g] = sum |a - b| over member g on this rank (float partials per block, added in double; fixed order), and in the same pass
 * da (+)= coef * sign(a - b), db (+)= -coef * sign(a - b) (sign(0) = 0; NULL: not wanted; accumulate 0 writes, 1 adds) with
 * coef = w / numel of the GLOBAL minibatch.  db needs a per-member b. */
int cg_latent_l1(const float* a, const float* b, int b_shared, float* da, float* db, float coef, int accumulate, float* sums,
                 int G, long n, void* ws, size_t ws_bytes, void* stream);
#define CG_RECON_MAX_TERMS 8
/* after the all-reduce of sums[nterm][G]: pub[k][g] = sums[k][g] / host_numel[k]; total[g] += sum_k host_weight[k] * pub[k][g]
 * through the double accumulator cg_gen_loss_bwd keeps in the same workspace (so it must follow the cg_gen_loss_bwd calls of
 * this update on that workspace and stream).  host_numel / host_weight (host memory) are passed by value. */
int cg_recon_finalize(const float* sums, const double* host_numel, const double* host_weight, int nterm, int G, float* total,
                      float* pub, void* ws, size_t ws_bytes, void* stream);
/* image reconstruction (recon_x_w, trainer_council.py:339-345, 455-459): h[G][B][HW][12] = tanh output of the last head layer of
 * the other direction's decoder, x[B][HW][4] the shared source image; x_recon = the cg_mask_head_fwd composite, never written.
 * fwd: sums[g] = sum |x_recon - x| over the 3 live lanes of member g on this rank (float per block of 2048 pixels, blocks added in
 * double in a fixed order).  bwd: dh_pre[G][B][HW][12] = cg_mask_head_bwd's result for d_xfake = coef * sign(x_recon - x)
 * (sign(0) = 0) and d_mask = 0, the composite recomputed bit for bit. */
int cg_recon_head_fwd(const float* h, const float* x, float* sums, int G, int B, int HW, void* ws, size_t ws_bytes, void* stream);
int cg_recon_head_bwd(const float* h, const float* x, float coef, float* dh_pre, int G, int B, int HW, void* stream);
size_t cg_loss_workspace_bytes(int G, int B, int H, int W);

/* ---- perceptual loss, vgg_w (trainer_council.py:199-205, 531-538, 636-641): the frozen Vgg16 (networks.py:573-622) runs on
 *      cg_conv_fwd (CG_ACT_RELU) / cg_conv_dgrad (mask_src = the previous ReLU output, slope 0); these are the other pieces ---------- */
/* vgg_preprocess (utils.py:380-390) on channels-last pixels x[npix][4] (lanes 0..2 RGB): y[npix][4] = {B', G', R', 0} with
 * c' = (x_c + 1) * 255 * 0.5 - {103.939, 116.779, 123.680}[BGR lane], each operation rounded as torch rounds it */
int cg_vgg_preprocess(const float* x, float* y, long npix, void* stream);
/* its data gradient: d_x[p][c] (+)= 127.5 * dy[p][2 - c] for c = 0..2; lane 3 is written 0 (accumulate 0) or kept (accumulate 1) */
int cg_vgg_preprocess_bwd(const float* dy, float* d_x, long npix, int accumulate, void* stream);
/* F.max_pool2d(x, 2, 2) (networks.py:598, 603, 609), floor size: x[N][H][W][C] -> y[N][H/2][W/2][C], C % 4 == 0 */
int cg_maxpool2x2_fwd(const float* x, float* y, int N, int H, int W, int C, void* stream);
/* backward of max_pool2d(relu(pre)) w.r.t. pre, without an index tensor: x = the saved ReLU output [N][H][W][C]; each window's first
 * maximum in row-major order (a later value must be strictly greater, as max_pool2d picks it) takes dy[N][H/2][W/2][C] where x > 0;
 * every other position of dx[N][H][W][C], and the last row / column an odd size leaves uncovered, is written 0 */
int cg_maxpool2x2_bwd(const float* dy, const float* x, float* dx, int N, int H, int W, int C, void* stream);
/* compute_vgg_loss (trainer_council.py:636-641) over R stacked image rows f_img[R][HW][C] (relu5_3) against the target rows
 * f_tgt[.][HW][C], image row r paired with target row (r / per_dir) * B + r % B; mean / rstd [rows][C] from cg_in_stats (eps 1e-5),
 * IN(f) = (f - mean) * rstd (nn.InstanceNorm2d(512, affine=False), :121).
 * sums[k] (k < R / B) = sum of (IN(f_img) - IN(f_tgt))^2 over rows [k B, k B + B) on this rank (float partials per block, added in
 * double in a fixed order); d_pre[R][HW][C] = the instance-norm backward (statistics included) of 2 coef (IN(f_img) - IN(f_tgt)), times
 * relu5_3's mask f_img > 0: the gradient w.r.t. conv5_3's pre-activation for a loss coef * sum, coef = vgg_w / numel of the GLOBAL
 * minibatch.  The targets take no gradient.  ws: the loss workspace (16 + 64 + 4 R C / 32 bytes at least). */
int cg_vgg_loss(const float* f_img, const float* mean_img, const float* rstd_img, const float* f_tgt, const float* mean_tgt,
                const float* rstd_tgt, int R, int B, int per_dir, int HW, int C, float coef, float* sums, float* d_pre, void* ws,
                size_t ws_bytes, void* stream);

/* ---- reflection padding, pad_type: reflect (Conv2dBlock networks.py:470-471: nn.ReflectionPad2d(padding), then an nn.Conv2d with
 *      padding 0).  The convolutions above pad with zeros only; a reflect layer runs cg_conv_* with pad 0 on the padded copy -------- */
/* xp[N][Hs+2p][Ws+2p][C] = ReflectionPad2d(p) of x[N][H][W][C] (N = G*B), seen at Hs x Ws = H x W, or with ups = 1 at 2H x 2W
 * nearest-upsampled first (nn.Upsample(scale_factor=2) networks.py:385, then the padding: one pass).  Index -i above the first row and
 * 2 (Hs - 1) - i below the last: the edge pixel is not repeated.  C % 4 == 0; 1 <= p < Hs and p < Ws, as ReflectionPad2d requires. */
int cg_reflect_pad(const float* x, float* xp, int N, int H, int W, int C, int p, int ups, void* stream);
/* its backward: dx[N][H][W][C] = (fold(dxp) + addend) * act'(mask_src), fold(dxp) = the sum of every position of dxp[N][H+2p][W+2p][C]
 * that the padding copied the pixel to (up to 9; 4 at the corners of a map larger than 2p), in padded row-major order.  addend /
 * mask_src (shape of dx) may be NULL and mean what they mean in cg_conv_dgrad: act' = mask_src > 0 ? 1 : mask_slope.  No upsample:
 * the x2 fan-in of an upsampled input is summed by cg_norm_act_bwd (ups) / cg_upsample2x_bwd.  1 <= p < H, p < W. */
int cg_reflect_pad_bwd(const float* dxp, float* dx, const float* addend, const float* mask_src, float mask_slope, int N, int H, int W,
                       int C, int p, void* stream);

/* plumbing: p[0:bytes] = 0 on `stream` (cudaMemsetAsync; keeps framework fill kernels out of the launch list) */
int cg_zero(void* p, size_t bytes, void* stream);

/* ---- input pipeline (the reference's per-image torchvision / Pillow transforms, utils.py:122-181, on a batch of decoded
 *      uint8 RGB images in device memory; bit-exact with Pillow 12 / torchvision 0.26, see csrc/augment.cu) ------------------ */
enum { CG_AUG_NONE = 0, CG_AUG_GRAY = 1, CG_AUG_BRIGHTNESS = 2, CG_AUG_CONTRAST = 3, CG_AUG_SATURATION = 4, CG_AUG_HUE = 5 };
/* One colour phase, in place: image b (desc[b] = {byte offset into imgs, H, W, 0}, RGB interleaved) gets opcode[b] with param[b]:
 * GRAY = RandomGrayscale; BRIGHTNESS / CONTRAST / SATURATION = ImageEnhance with factor param[b]; HUE = hue shift of
 * (int)param[b] steps of 1/255 (pass float(int(hue_factor * 255))).  lsum: B x uint64 scratch.  transforms.ColorJitter applies its
 * four ops in a random per-image order: call once per position of the permutation. */
int cg_aug_color(uint8_t* imgs, const int32_t* desc, const int32_t* opcode, const float* param, unsigned long long* lsum,
                 int B, int max_pixels, int any_contrast, void* stream);
/* n images of ONE source size H x W (src_off[i] = byte offset): optional horizontal flip, Pillow bilinear resize to oh x ow
 * (tables from Resample.c precompute_coeffs: bounds[out][2] = {first tap, count}, kk[out][ksize] 22-bit fixed point), crop window
 * crop[i] = {top, left} of size ch x cw, ToTensor + Normalize(0.5, 0.5): image i is written to batch slot slot[i] of
 * out_nhwc[.][ch][cw][4] (fp32, lane 3 = 0) and, if not NULL, of out_nchw[.][3][ch][cw].  tmp: n * H * ow * 3 bytes. */
int cg_aug_resize_crop(const uint8_t* imgs, const int32_t* src_off, const int32_t* flip, const int32_t* slot,
                       const int32_t* crop, int n, int H, int W, int oh, int ow, int ch, int cw, const int32_t* bounds_h,
                       const int32_t* kk_h, int ksize_h, const int32_t* bounds_v, const int32_t* kk_v, int ksize_v,
                       uint8_t* tmp, float* out_nhwc, float* out_nchw, void* stream);

/* ---- optimiser (torch.optim.Adam as used at trainer_council.py:170-179) ----------------------- */
int cg_adam_step(float* p, const float* g, float* m, float* v, long n, float lr, float beta1,
                 float beta2, float eps, float weight_decay, int step, float grad_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* COUNCIL_B200_H */
