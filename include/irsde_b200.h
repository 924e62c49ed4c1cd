/*
 * irsde_b200 - C ABI of the H100-native IR-SDE / Denoising-SDE reverse-diffusion sampler.
 *
 * The reference (Algolzw/image-restoration-sde @ 2598d73) is pure Python and has no FFI; the
 * calls below are what a binding for its hot path would bind.  Each entry point cites the
 * reference interface it replaces (paths relative to the reference checkout).
 *
 * Conventions
 *   - every function returns 0 on success or a negative irsde_status; the message for the last
 *     failure is available from irsde_last_error(ctx) (ctx may be NULL for create failures);
 *   - nothing throws across the ABI; one context per device; a context is not thread-safe;
 *   - image tensors are raw DEVICE pointers to dense fp32 NCHW data ([B,C,H,W], the layout
 *     the reference's torch tensors have); `stream` is a cudaStream_t passed as void*
 *     (torch.cuda.current_stream().cuda_stream);
 *   - weights are copied/repacked by the library; the caller keeps ownership of its buffers.
 *
 * Streams
 *   - every entry with a `stream` argument reads its device inputs and writes its outputs in that stream's order (work
 *     enqueued on the stream before the call is seen, work enqueued after it sees the outputs), on blocking and
 *     non-blocking streams alike, and never uses the legacy default stream for it;
 *   - these synchronize the device: irsde_set_schedule, irsde_set_coeffs, irsde_load_tensor (it waits for all earlier
 *     device work before its copy and returns once the copy is complete, so `data` may come from any stream and may be
 *     reused at once), irsde_finalize_weights, irsde_broadcast_weights, irsde_trim, irsde_destroy, irsde_profile_end*;
 *     the standalone operator entries (irsde_conv2d*, irsde_layernorm, irsde_attention, irsde_linattn_block,
 *     irsde_nafnet_op, irsde_time_embedding, irsde_prep_input) synchronize their stream and free their scratch memory,
 *     which waits for the device;
 *   - the first use of a (B, H, W) by a context (building its launch plan, including irsde_plan_num_ops /
 *     irsde_plan_op_info) synchronizes the device, and the first graph capture of a mode may block the host; every
 *     later call only enqueues work;
 *   - calls on one context from different streams are serialized: a call that uses the context's plans, tables or uid
 *     buffer (irsde_noise_fn, irsde_reverse, irsde_trace_forward, irsde_latent_encode / _decode, irsde_set_image_uids,
 *     irsde_noise_state_images, irsde_step_philox) on another stream than the previous such call first makes its stream
 *     wait for the work that call enqueued.
 */
#ifndef IRSDE_B200_H
#define IRSDE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct irsde_ctx irsde_ctx;

typedef enum {
  IRSDE_OK = 0,
  IRSDE_ERR_INVALID = -1,     /* bad argument / shape */
  IRSDE_ERR_CUDA = -2,        /* CUDA runtime / driver error */
  IRSDE_ERR_STATE = -3,       /* call order (weights / schedule missing) */
  IRSDE_ERR_UNSUPPORTED = -4  /* configuration this build cannot run */
} irsde_status;

/* score-network variant */
#define IRSDE_NET_CONDITIONAL 0 /* codes/config/deraining/models/modules/DenoisingUNet_arch.py:19-134 */
#define IRSDE_NET_DENOISING 1   /* codes/config/denoising-sde/models/modules/DenoisingUNet_arch.py:19-133 */

/* numerics mode */
#define IRSDE_PREC_FP32 0 /* parity mode: fp32 storage + fp32 FMA everywhere                     */
#define IRSDE_PREC_BF16 1 /* perf mode: bf16 activations/weights, wgmma MMA, fp32 accumulate,  */
                          /* fp32 sampler state                                                   */
#define IRSDE_PREC_FP32X3 2 /* fp32-accurate tensor-core mode: fp32 storage; every conv is three   */
                            /* tf32 wgmma passes over hi/lo split operands            */
                            /* (hi*hi + lo*hi + hi*lo, fp32 accumulate): meets the 1e-3    */
                            /* bound of the fp32 mode on the tensor cores                          */

/* sampler */
#define IRSDE_MODE_SDE 0       /* IRSDE.reverse_sde        codes/utils/sde_utils.py:252-266 */
#define IRSDE_MODE_ODE 1       /* IRSDE.reverse_ode        codes/utils/sde_utils.py:268-282 */
#define IRSDE_MODE_POSTERIOR 2 /* IRSDE.reverse_posterior  codes/utils/sde_utils.py:284-299 */
#define IRSDE_MODE_DSDE_SDE 3  /* DenoisingSDE.reverse_sde codes/utils/sde_utils.py:483-500 */
#define IRSDE_MODE_DSDE_ODE 4  /* DenoisingSDE.reverse_ode codes/utils/sde_utils.py:502-522 */
#define IRSDE_NUM_MODES 5
#define IRSDE_NUM_COEF 8 /* floats per timestep in a coefficient table */

typedef struct {
  int32_t in_nc;     /* image channels (ConditionalUNet in_nc)  */
  int32_t out_nc;    /* output channels                          */
  int32_t nf;        /* base width                               */
  int32_t depth;     /* number of levels                         */
  int32_t variant;   /* IRSDE_NET_*                              */
  int32_t precision; /* IRSDE_PREC_*                             */
  int32_t device;    /* CUDA device ordinal                      */
  int32_t flags;     /* IRSDE_FLAG_* (0 = defaults)              */
} irsde_config;
/* flags (all three config structs): bf16 storage through the fp32-FMA SIMT conv engine instead of the tensor cores - a debugging
 * aid that separates storage rounding from tensor-core issues; never the product path. */
#define IRSDE_FLAG_FORCE_SIMT 1

/* Refusion score network: ConditionalNAFNet(img_channel, width, middle_blk_num, enc_blk_nums, dec_blk_nums)
 * (codes/config/deraining/models/modules/DenoisingNAFNet_arch.py:87-143); latent != 0 selects the latent
 * variant whose last conv sees x + intro(x) (codes/config/latent-dehazing/models/modules/DenoisingNAFNet_arch.py:176). */
typedef struct {
  int32_t img_channel;
  int32_t width;
  int32_t middle_blk_num;
  int32_t n_levels;          /* len(enc_blk_nums) == len(dec_blk_nums), <= 8 */
  int32_t enc_blk_nums[8];
  int32_t dec_blk_nums[8];
  int32_t latent;
  int32_t precision;         /* IRSDE_PREC_* */
  int32_t device;
  int32_t flags;             /* IRSDE_FLAG_* */
} irsde_nafnet_config;

/* Refusion latent autoencoder: UNet(in_ch, out_ch, ch, ch_mult, embed_dim)
 * (codes/config/latent-dehazing/models/modules/UNet_arch.py:17-57). */
typedef struct {
  int32_t in_ch, out_ch, ch;
  int32_t n_levels;      /* len(ch_mult) <= 8 */
  int32_t ch_mult[8];
  int32_t embed_dim;
  int32_t precision;     /* IRSDE_PREC_* */
  int32_t device;
  int32_t flags;         /* IRSDE_FLAG_* */
} irsde_latent_unet_config;

/* Replaces `ConditionalUNet(in_nc,out_nc,nf,depth)` + `.to(device)`
 * (DenoisingUNet_arch.py:20, models/denoising_model.py:36).  nf <= 2456: the time MLP keeps 20 nf bytes in shared memory. */
int irsde_create(const irsde_config* cfg, irsde_ctx** out);
/* The latent-task variant `ConditionalUNet(in_nc, out_nc, nf, ch_mult=[1,2,4,4])`
 * (codes/config/latent-dehazing/models/modules/DenoisingUNet_arch.py:17-20,51-56,70): level i has nf*[1,ch_mult...][i]
 * channels and depth = len(ch_mult) (cfg->depth is ignored). */
int irsde_create_ch_mult(const irsde_config* cfg, const int32_t* ch_mult, int32_t n_levels, irsde_ctx** out);
/* Same context type, ConditionalNAFNet architecture; every other entry point (load_tensor, noise_fn, reverse, ...)
 * is shared.  Replaces `ConditionalNAFNet(...)` + `.to(device)` (DenoisingNAFNet_arch.py:89).  width <= 944 and
 * width << n_levels <= 12288: the time MLP (52 width bytes) and the SCA mat-vec (4 bytes per channel) fit in 48 KB of
 * shared memory. */
int irsde_create_nafnet(const irsde_nafnet_config* cfg, irsde_ctx** out);
/* irsde_create_nafnet with the network variant: IRSDE_NET_CONDITIONAL is irsde_create_nafnet; IRSDE_NET_DENOISING is the
 * denoising-sde task's ConditionalNAFNet, whose intro conv reads the img_channel channels of x and whose forward takes
 * no condition (codes/config/denoising-sde/models/modules/DenoisingNAFNet_arch.py:89-103,147).  That context drives the
 * DenoisingSDE modes and takes mu == NULL; cfg->latent must be 0 with it. */
int irsde_create_nafnet_variant(const irsde_nafnet_config* cfg, int32_t variant, irsde_ctx** out);
void irsde_destroy(irsde_ctx* ctx);
const char* irsde_last_error(const irsde_ctx* ctx);
/* "irsde_b200 <version> sm_90a" */
const char* irsde_version(void);

/* Latent autoencoder context (same weight-loading entry points).  encode replaces `UNet.encode(x) -> (z, h)`
 * (UNet_arch.py:59-76): z is fp32 [B, embed_dim, lat_h, lat_w] (irsde_latent_shape); the skip list h stays inside the
 * context.  decode replaces `UNet.decode(z, h)` (UNet_arch.py:78-91) and uses the skips of the last encode with the
 * same (B, H, W); out is fp32 [B, out_ch, H, W]. */
int irsde_create_latent_unet(const irsde_latent_unet_config* cfg, irsde_ctx** out);
int irsde_latent_shape(irsde_ctx* ctx, int32_t H, int32_t W, int32_t* lat_h, int32_t* lat_w);
int irsde_latent_encode(irsde_ctx* ctx, const float* x, float* z, int32_t B, int32_t H, int32_t W, void* stream);
int irsde_latent_decode(irsde_ctx* ctx, const float* z, float* out, int32_t B, int32_t H, int32_t W, void* stream);

/* Replaces `load_state_dict` (models/base_model.py:92-105): one call per state-dict entry,
 * `name` and `shape` exactly as in the reference state dict; `data` is fp32, host or device. */
int irsde_load_tensor(irsde_ctx* ctx, const char* name, const void* data, int32_t ndim, const int64_t* shape);
/* Check that every tensor of the architecture was loaded and repack for the kernels. */
int irsde_finalize_weights(irsde_ctx* ctx);

/* Replaces `IRSDE.__init__/_initialize` / `DenoisingSDE._initialize` results
 * (sde_utils.py:132-149, :419-426): host arrays of length T+1, index 0 unused. */
int irsde_set_schedule(irsde_ctx* ctx, const float* thetas, const float* sigmas, const float* thetas_cumsum,
                       const float* sigma_bars, float dt, float max_sigma, int32_t T);
/* Optional: override the per-timestep scalars of one mode ([T+1][IRSDE_NUM_COEF] host floats)
 * with values computed by the caller in the reference's own op order (see DESIGN.md). */
int irsde_set_coeffs(irsde_ctx* ctx, int32_t mode, const float* table, int32_t T);

/* Replaces `IRSDE.noise_fn` -> `ConditionalUNet.forward(xt, cond, time)`
 * (sde_utils.py:192-194, DenoisingUNet_arch.py:85-134).  `times` is a HOST array of n_times
 * values (1 = shared by the batch, B = per image); `mu` is ignored for IRSDE_NET_DENOISING. */
int irsde_noise_fn(irsde_ctx* ctx, const float* x, const float* mu, const float* times, int32_t n_times, float* out,
                   int32_t B, int32_t H, int32_t W, void* stream);

/* Replaces `reverse_sde_step / reverse_ode_step / reverse_posterior_step`
 * (sde_utils.py:44-48,219-223,450-462): one fused elementwise update over n floats.
 * z may be NULL for the ODE modes.  out may alias x. */
int irsde_step(irsde_ctx* ctx, int32_t mode, const float* x, const float* mu, const float* noise, const float* z,
               int32_t t, float* out, int64_t n, void* stream);

/* Replaces the whole loop `for t in reversed(range(1, T+1))` of reverse_sde/ode/posterior
 * (sde_utils.py:252-299, :483-522): network forward + update for t = T..1.
 * z: [T][B*C*H*W] pre-drawn N(0,1) in loop order (first slice used at t=T), or NULL to draw
 * in-kernel (Philox4x32-10, seeded with `seed`).  use_graph != 0 replays one captured step graph. */
int irsde_reverse(irsde_ctx* ctx, int32_t mode, const float* xT, const float* mu, const float* z, float* x0,
                  int32_t B, int32_t H, int32_t W, int32_t T, uint64_t seed, int32_t use_graph, void* stream);

/* x_T = mu + N(0,1)*max_sigma on the device (sde_utils.py:360-361) with the library's Philox; the n floats are
 * treated as ONE image (uid = the ctx's image base). */
int irsde_noise_state(irsde_ctx* ctx, const float* mu, float* out, int64_t n, uint64_t seed, void* stream);
/* Same for a batch [B][image_elems]: image b is drawn with uid = image base + b. */
int irsde_noise_state_images(irsde_ctx* ctx, const float* mu, float* out, int32_t B, int64_t image_elems, uint64_t seed,
                             void* stream);
/* Training-time state sampler `IRSDE.generate_random_states` (sde_utils.py:343-358; train.py:236): one fused pass
 * x_t = noise * sigma_bar[t_b] + (mu + (x0 - mu) * w[b]) with per-image scalars w[b] = exp(-thetas_cumsum[t_b] dt) and
 * sigma_bar[b] (device arrays of B floats); bit-identical to the reference's torch expression.  Stateless (no ctx). */
int irsde_random_states(const float* x0, const float* mu, const float* noise, const float* w, const float* sigma_bar, float* out,
                        int32_t B, int64_t image_elems, void* stream);

/* The in-kernel Philox (irsde_reverse with z == NULL, irsde_noise_state*) is keyed by
 * (seed, image uid, timestep, element index inside the image), uid = image base + position in the batch.
 * An image's noise therefore does not depend on the batch it is processed in, its position, or the rank that
 * owns it: set the base to the global index of the shard's / batch's first image (default 0) and batched,
 * sharded and one-at-a-time runs give bit-identical images (SURVEY.md 8 a-16 xi, e, f-2). */
int irsde_set_image_base(irsde_ctx* ctx, uint64_t first_image_uid);
/* Explicit uids for the next batch (n host values, n == B of the following calls), e.g. when a batch is assembled from
 * same-sized images that are not consecutive in the dataset.  irsde_set_image_base() returns to base + position. */
int irsde_set_image_uids(irsde_ctx* ctx, const uint64_t* uids, int32_t n, void* stream);

/* Instrumented pass: between begin/end every op of the launch plan is bracketed by CUDA events on the
 * launching stream (graph replay is bypassed).  end() synchronises and returns, per op category
 * (0 tensor-core conv, 1 SIMT conv, 2 LayerNorm, 3 attention, 4 misc, 5 update), the summed device time in
 * ms, the executed conv flops and the number of ops.  ncat must be >= 6. */
int irsde_profile_begin(irsde_ctx* ctx);
int irsde_profile_end(irsde_ctx* ctx, double* ms, double* flops, int64_t* launches, int32_t ncat);
/* Same, plus bytes[cat] = the ops' ALGORITHMIC HBM bytes (each op's inputs + outputs + its weights once; DESIGN.md 4):
 * the numerator of the HBM roofline of the memory-bound kernels. */
int irsde_profile_end_bytes(irsde_ctx* ctx, double* ms, double* flops, int64_t* launches, double* bytes, int32_t ncat);

/* Kernel launches issued by this context since creation (for bench.py's gpu_launches). */
int64_t irsde_launch_count(const irsde_ctx* ctx);
/* Bytes of device memory held by the context (weights + workspaces). */
int64_t irsde_device_bytes(const irsde_ctx* ctx);

/* ---- standalone operator entry points (unit-test / micro-benchmark surface) -------------- */
/* Generic NHWC convolution through the engine selected by `engine` (0 = fp32 SIMT implicit
 * GEMM, 1 = wgmma bf16 tap-GEMM, 2 = wgmma fp32x3 tap-GEMM: fp32 in/out, 3 x tf32 MMA).  Input/weights/output are fp32 device buffers:
 * x [B,Cin,H,W], w [Cout,Cin,KH,KW] (nn.Conv2d layout, module_util.py:96,101,105), y
 * [B,Cout,Ho,Wo]; the call repacks to the engine's layout, runs, and unpacks. */
int irsde_conv2d(irsde_ctx* ctx, int32_t engine, const float* x, const float* w, const float* bias, float* y,
                 int32_t B, int32_t Cin, int32_t H, int32_t W, int32_t Cout, int32_t KH, int32_t KW, int32_t stride,
                 int32_t pad, int32_t upsample, int32_t silu, void* stream);

/* Same with the tensor-core engine's fused epilogues (engine must be 1 when any is used):
 *   residual  fp32 [B,Cout,Ho,Wo] added after the activation (ResBlock `h + res_conv(x)`, module_util.py:146), or NULL;
 *   IRSDE_CONV_QSOFTMAX     1x1 conv whose first 128 output channels are LinearAttention's q: softmax over each
 *                           32-channel head times 32^-0.5 (module_util.py:168,171);
 *   IRSDE_CONV_W_PER_IMAGE  w is [B,Cout,Cin]: image b is multiplied by its own matrix (LinearAttention's second einsum
 *                           + to_out re-associated, module_util.py:176-178). */
#define IRSDE_CONV_QSOFTMAX 1
#define IRSDE_CONV_W_PER_IMAGE 2
int irsde_conv2d_ex(irsde_ctx* ctx, int32_t engine, const float* x, const float* w, const float* bias, const float* residual,
                    float* y, int32_t B, int32_t Cin, int32_t H, int32_t W, int32_t Cout, int32_t KH, int32_t KW,
                    int32_t stride, int32_t pad, int32_t upsample, int32_t silu, int32_t flags, void* stream);

/* The fused epilogue of one network conv, with the views the launch plan gives it.  All pointers are device pointers. */
typedef struct {
  const float* bias;     /* [Cout] or NULL */
  const float* mult_vec; /* [Cout] or NULL: (acc + bias) * mult_vec (NAFBlock beta / gamma); not allowed together with ss */
  const float* ss;       /* time-modulation table [ss_rows][ss_S] or NULL: image b uses row t_row + b * ss_img_stride, */
                         /* scale = row[ss_off + n], shift = row[ss_off + Cout + n]: (acc + bias) * (scale + 1) + shift  */
  const float* res;      /* residual added last, fp32 NHWC [B][Ho][Wo][res_pitch] read at channels res_off.., or NULL */
  int32_t silu;          /* SiLU after the modulation, before the residual */
  int32_t flags;         /* IRSDE_CONV_QSOFTMAX (engine 1, 1x1) */
  int32_t ss_rows, ss_S, ss_off, ss_img_stride, t_row;
  int32_t res_pitch, res_off;
  int32_t in_pitch, in_off;   /* x is fp32 NHWC [B][H][W][in_pitch]; the conv reads channels in_off .. in_off+Cin-1 */
  int32_t out_pitch, out_off; /* y is fp32 NHWC [B][Ho][Wo][out_pitch]; the conv writes channels out_off .. out_off+Cout-1 */
  int32_t crop_h, crop_w;     /* > 0 (3x3 head only): y is fp32 NCHW [B][Cout][crop_h][crop_w] instead, the output's */
                              /* top-left crop_h x crop_w pixels; out_pitch / out_off are then ignored */
} irsde_conv_epilogue;

/* One conv of the launch plan with its fused epilogue, through the same descriptor and launch calls the plan builder uses
 * (engine 0 = fp32 SIMT, 1 = bf16 wgmma, 2 = fp32x3 wgmma; KxK/stride/pad/upsample as in irsde_conv2d, 3x3/1, 1x1 and 4x4/2).
 * y is read and written: the whole buffer is converted to the engine's storage type (bf16 for engine 1), the conv writes its
 * slice, and the whole buffer is converted back, so an element outside the slice comes back unchanged when it is
 * representable in that type.  Every view, table row and crop is checked on the host before anything is launched; offsets
 * and pitches must be multiples of 16 bytes of the engine's storage type.
 * info (or NULL) receives {BN, MODE, EKT, number of output tiles} of the conv_tc_persist_kernel instantiation that ran
 * (engines 1 and 2), or zeros (engine 0). */
int irsde_conv2d_fused(irsde_ctx* ctx, int32_t engine, const float* x, const float* w, const irsde_conv_epilogue* ep, float* y,
                       int32_t B, int32_t Cin, int32_t H, int32_t W, int32_t Cout, int32_t KH, int32_t KW, int32_t stride,
                       int32_t pad, int32_t upsample, int32_t* info, void* stream);

/* One channel LayerNorm of the network (module_util.py:70-79; biased variance, eps 1e-5), with the optional NAFBlock time
 * modulation (DenoisingNAFNet_arch.py:62-63,75-76) and residual: y = ln(x) * g [* (scale + 1) + shift] [+ res].
 * x, res and y are fp32 NHWC buffers of B*N pixels, each read or written through a (pitch, channel offset) view; views need
 * not be 16-byte aligned. */
typedef struct {
  const float* g;          /* gain [C] */
  const float* res;        /* residual buffer [B*N][res_pitch] read at channels res_off.., or NULL */
  const float* ss;         /* time-modulation table [ss_rows][ss_S] or NULL: image b uses row t_row + b * ss_img_stride, */
                           /* scale = row[off_scale + c], shift = row[off_shift + c] */
  int32_t in_pitch, in_off;
  int32_t res_pitch, res_off;
  int32_t out_pitch, out_off;
  int32_t ss_rows, ss_S, off_scale, off_shift, ss_img_stride, t_row;
} irsde_ln_args;

/* precision 0 (fp32; IRSDE_PREC_FP32X3 runs the same kernels) or 1 (bf16).  y is read and written: for bf16 the whole x, res
 * and y buffers are converted to bf16, the kernel writes y's slice, and y is converted back, so an element outside the slice
 * comes back unchanged when bf16 represents it.  Every view, table row and size is checked on the host before anything is
 * allocated or launched.  info (or NULL) receives {kind, MAXV, LPP, PP} of the kernel that ran: kind 0 =
 * layernorm_scalar_kernel (MAXV = LPP = PP = 0), 1 = layernorm_vec_kernel<MAXV> (LPP lanes per pixel, PP = 1),
 * 2 = layernorm_geo_kernel<MAXV, LPP, PP>. */
int irsde_layernorm(irsde_ctx* ctx, int32_t precision, const float* x, const irsde_ln_args* args, float* y, int32_t B, int32_t N,
                    int32_t C, int32_t* info, void* stream);

/* One attention core of the network on qkv = to_qkv's output, an fp32 NHWC buffer [B*N][qkv_pitch] whose channels
 * qkv_off .. qkv_off+383 are q | k | v (4 heads of 32).
 *   IRSDE_ATTN_LINEAR       LinearAttention (module_util.py:163-177): ctx_out = fp32 [B][4][32][32] context
 *                           (ctx[b][h][d][e] = sum_n softmax_n(k)[d,n] v[e,n] / N), out = the 128 hidden channels, written
 *                           through the view (out_pitch, out_off) of an fp32 [B*N][out_pitch] buffer;
 *   IRSDE_ATTN_LINEAR_FOLD  (bf16 only) the same context, folded into the to_out weights wout fp32 [Cout][128]:
 *                           out = fp32 [B][Cout][128], Mb[b][c][h*32+d] = sum_e wout[c][h*32+e] ctx[b][h][d][e]
 *                           (module_util.py:176-178 re-associated); out_pitch / out_off are ignored;
 *   IRSDE_ATTN_FULL         softmax Attention (module_util.py:192-204): out = hidden through (out_pitch, out_off); ctx_out
 *                           is not used.
 * Buffers are converted as in irsde_layernorm.  The linear kinds need views that start on 16 bytes of the storage type and
 * pitches that are multiples of 16 bytes of it.  info (or NULL) receives {kernel, nblk, nchunks, 0}: kernel 1 =
 * la_kv_kernel<float>, 2 = la_kv_mma_kernel, 3 = fullattn_kernel, 4 = fullattn_mma_kernel; nblk blocks per image
 * share nchunks chunks of 64 pixels in the k,v pass (0 for IRSDE_ATTN_FULL). */
#define IRSDE_ATTN_LINEAR 0
#define IRSDE_ATTN_LINEAR_FOLD 1
#define IRSDE_ATTN_FULL 2
int irsde_attention(irsde_ctx* ctx, int32_t precision, int32_t kind, const float* qkv, int32_t qkv_pitch, int32_t qkv_off,
                    float* out, int32_t out_pitch, int32_t out_off, const float* wout, int32_t Cout, float* ctx_out, int32_t B,
                    int32_t N, int32_t* info, void* stream);

/* One whole Residual(PreNorm(LinearAttention)) block (module_util.py:150-178) on the bf16 path, C = 64 or 128, as the
 * launch plan runs it: two fused passes over x (LayerNorm + k,v projection + the context partials; LayerNorm + q projection
 * + q softmax + to_out with the folded context + LayerNorm + residual) around the combine and the fold.
 *   x     fp32 [B*N][x_pitch], the block input at channels x_off .. x_off+C-1 (x_pitch, x_off multiples of 8);
 *   out   fp32 [B*N][out_pitch], the block output written at channels out_off .. out_off+C-1 (even pitch and offset);
 *   g1    fn.norm.g [C]; wqkv fn.fn.to_qkv.weight [384][C]; wout fn.fn.to_out.0.weight [C][128]; bout its bias [C];
 *   g2    fn.fn.to_out.1.g [C] (g1, g2, bout and wout start on 16 bytes);
 *   xn_out NULL, or fp32 [B*N][C]: the bf16 LayerNorm(x) the first pass computes.
 * Buffers are converted as in irsde_layernorm. */
int irsde_linattn_block(irsde_ctx* ctx, const float* x, int32_t x_pitch, int32_t x_off, float* out, int32_t out_pitch,
                        int32_t out_off, const float* g1, const float* wqkv, const float* wout, const float* bout, const float* g2,
                        float* xn_out, int32_t B, int32_t N, int32_t C, void* stream);

/* One NAFBlock op of the launch plan (DenoisingNAFNet_arch.py:9-12,29-33,65-67; the decoder's PixelShuffle + skip, :172-174;
 * the latent variant's x + intro(x)).  x, y and out are fp32 NHWC buffers read or written through (pitch, channel offset)
 * views; views need not be aligned.  Pixel counts: x and (for ADD) y hold B*H*W pixels; for PIXEL_SHUFFLE_ADD, H x W is the
 * input's size and y (the skip) and out hold B*2H*2W pixels.
 *   IRSDE_NAF_DWGATE_SCA      gate = dw3x3(x)[0..c) * dw3x3(x)[c..2c) (depthwise, zero padding 1, bias), then
 *                             sca[b] = sca_w @ mean_HW(gate[b]) + sca_b and out = gate * sca: x holds 2c channels, w is
 *                             [2c][9], bias [2c], sca_w [c][c], sca_b [c], sca fp32 [B][c] (written);
 *   IRSDE_NAF_SIMPLE_GATE     out = x[0..c) * x[c..2c);
 *   IRSDE_NAF_PIXEL_SHUFFLE_ADD  out[b, 2h+i, 2w+j, q] = x[b, h, w, 4q + 2i + j] + y[b, 2h+i, 2w+j, q] (c = q);
 *   IRSDE_NAF_ADD             out = x + y (c channels each). */
#define IRSDE_NAF_DWGATE_SCA 0
#define IRSDE_NAF_SIMPLE_GATE 1
#define IRSDE_NAF_PIXEL_SHUFFLE_ADD 2
#define IRSDE_NAF_ADD 3
typedef struct {
  const float* x;
  const float* y;         /* PIXEL_SHUFFLE_ADD, ADD; else ignored */
  float* out;
  const float* w;         /* DWGATE_SCA only: conv2 weight [2c][9] and bias [2c] */
  const float* bias;
  const float* sca_w;     /* DWGATE_SCA only: sca.1 weight [c][c] and bias [c] */
  const float* sca_b;
  float* sca;             /* DWGATE_SCA only: fp32 [B][c] output */
  int32_t x_pitch, x_off;
  int32_t y_pitch, y_off;
  int32_t out_pitch, out_off;
} irsde_nafnet_args;

/* Buffers are converted as in irsde_layernorm (sca stays fp32).  Every view and size is checked on the host before anything is
 * allocated or launched.  info (or NULL) receives, for DWGATE_SCA, {pixels per pooling chunk, chunks per image, launches of
 * the SCA stage (1: sca_kernel scales the gate in place, 2: a scale_channels_kernel pass follows), 0}; zeros otherwise. */
int irsde_nafnet_op(irsde_ctx* ctx, int32_t precision, int32_t kind, const irsde_nafnet_args* args, int32_t B, int32_t H,
                    int32_t W, int32_t c, int32_t* info, void* stream);

/* The time-embedding MLP and the per-block (scale, shift) table the plan builds (stateless: no ctx; device pointers).
 *   family 0 (ConditionalUNet, DenoisingUNet_arch.py:42-47, module_util.py:29-41,128-141): temb [rows][4 width] =
 *            SiLU(Linear(GELU(Linear(pos(t))))), w1 [4w][w], w2 [4w][4w], wall [S][4w];
 *   family 1 (NAFNet, DenoisingNAFNet_arch.py:18-20,51-54,96-101): temb [rows][2 width] = SimpleGate(Linear(SimpleGate(
 *            Linear(pos(t))))), w1 [8w][w], w2 [4w][4w], wall [S][2w];
 * table [rows][S] = temb @ wall^T + ball.  times: [rows] device floats.  width must be even and >= 4, and the MLP's shared
 * memory (20 width or 52 width bytes) must fit in 48 KB. */
int irsde_time_embedding(int32_t family, const float* times, int32_t rows, int32_t width, const float* w1, const float* b1,
                         const float* w2, const float* b2, const float* wall, const float* ball, int32_t S, float* temb,
                         float* table, void* stream);

/* irsde_step for the stochastic modes with z drawn in-kernel, as irsde_reverse(z = NULL) draws it at step t: keyed by (seed,
 * image uid, t, element index inside the image) with the uids of irsde_set_image_base / irsde_set_image_uids; x, mu, noise and
 * out hold B images of image_elems floats. */
int irsde_step_philox(irsde_ctx* ctx, int32_t mode, const float* x, const float* mu, const float* noise, int32_t t, float* out,
                      int32_t B, int64_t image_elems, uint64_t seed, void* stream);

/* The network's input packing (stateless): out [B][img_rows][row_pix][pitch] (row_pix = img_rows = 0: [B][Hp][Wp][pitch]) gets,
 * at pixel (pad_top + hp, pad_left + wp), cat(xt - cond, cond) (conditional) or xt, of the image padded at the bottom / right
 * to Hp x Wp by reflection (zero_pad = 0; Hp - H < H and Wp - W < W) or with zeros; channels 2C (C) .. pitch-1 are set to zero.
 * Pixels outside the padded image (the border) are not written.  xt, cond: fp32 NCHW [B][C][H][W].  out is converted as in
 * irsde_layernorm for precision 1. */
int irsde_prep_input(int32_t precision, const float* xt, const float* cond, float* out, int32_t B, int32_t C, int32_t H, int32_t W,
                     int32_t Hp, int32_t Wp, int32_t pitch, int32_t conditional, int32_t zero_pad, int32_t pad_top, int32_t pad_left,
                     int32_t row_pix, int32_t img_rows, void* stream);

/* ---- launch-plan introspection (parity instrumentation: per-layer comparison with the oracle) ----
 * The network forward for a (B,H,W) input is a fixed list of ops.  irsde_plan_num_ops returns its length (or a negative
 * irsde_status); irsde_plan_op_info gives op `op`'s label (the state-dict name of the weight it applies, e.g.
 * "downs.0.0.block1.proj.weight 256x256 k3 ...") and dims = {C, H, W of the NHWC view it writes (C == 0: none),
 * category as in irsde_profile_end}; irsde_trace_forward runs ops 0..op of `irsde_noise_fn(x, mu, times)` and writes
 * op `op`'s output as fp32 [B,C,H,W] to `dump` (device). */
int32_t irsde_plan_num_ops(irsde_ctx* ctx, int32_t B, int32_t H, int32_t W);
int irsde_plan_op_info(irsde_ctx* ctx, int32_t B, int32_t H, int32_t W, int32_t op, char* label, int32_t label_cap,
                       int32_t* dims /* [4] */);
int irsde_trace_forward(irsde_ctx* ctx, const float* x, const float* mu, const float* times, int32_t n_times, int32_t B,
                        int32_t H, int32_t W, int32_t op, float* dump, void* stream);

/* Drop every cached (B,H,W) launch plan (activation workspaces, TMA descriptors, step graphs).  The cache is also
 * bounded on its own: least-recently-used plans are evicted beyond IRSDE_PLAN_CACHE_MB (default 24576) megabytes or
 * IRSDE_PLAN_CACHE_MAX (default 8) entries, so looping over variable-size images (codes/config/<task>/test.py:96-130,
 * batch 1 at native resolution) does not grow device memory without limit. */
int irsde_trim(irsde_ctx* ctx);

/* ---- multi-GPU plumbing (one process per GPU; SURVEY.md 8 b, e) ------------------------------------------------
 * Replaces DataParallel's per-step replicate / scatter / gather (models/denoising_model.py:41-42) with the two
 * collectives the path needs.  NCCL is dlopen()ed on first use (IRSDE_NCCL_LIB overrides the soname) so single-GPU users
 * keep a library without an NCCL dependency; ranks exchange the 128-byte id out of band (rank 0 creates it).
 * irsde_broadcast_weights: every rank has loaded a state dict of the same names/shapes; the fp32 tensors are replaced
 * by rank `src`'s in one NCCL group and repacked (irsde_finalize_weights is called inside).
 * irsde_gather: rank r contributes counts[r] floats (its slice of x0 in the contiguous batch partition, which may be
 * ragged); x_all receives all slices in rank order = batch order, on every rank. */
int irsde_comm_unique_id(void* id128);
int irsde_comm_init(irsde_ctx* ctx, const void* id128, int32_t rank, int32_t nranks);
int irsde_broadcast_weights(irsde_ctx* ctx, int32_t src, void* stream);
int irsde_gather(irsde_ctx* ctx, const float* x_local, float* x_all, const int64_t* counts /* [nranks] */, void* stream);

/* ---- image conversion and full-reference metrics on the device (SURVEY.md section 8 f-3) -------------------
 * Stateless (no ctx): errors are reported through the return code and irsde_last_error(NULL).
 * Replaces util.tensor2img (codes/utils/img_utils.py:136-163), img2tensor / read_img's "/255." (:171-180,
 * codes/data/util.py:72), calculate_psnr (:182-190) and ssim / calculate_ssim (:193-234).  All pointers are
 * device pointers.  Images are uint8 [B][H][W][C] (BGR when C == 3, the cv2 order), tensors fp32 [B][C][H][W] RGB. */
int irsde_tensor2img_u8(const float* chw, uint8_t* hwc, int32_t B, int32_t C, int32_t H, int32_t W, double lo, double hi,
                        void* stream);
int irsde_img2tensor_u8(const uint8_t* hwc, float* chw, int32_t B, int32_t C, int32_t H, int32_t W, void* stream);
/* sums[b] = sum over the crop-bordered region of (a - b)^2, exact; PSNR = 20 log10(255 / sqrt(sums / n)). */
int irsde_sqerr_u8(const uint8_t* a, const uint8_t* b, int32_t B, int32_t H, int32_t W, int32_t C, int32_t crop,
                   uint64_t* sums, void* stream);
/* number of doubles irsde_ssim_u8 needs as workspace */
int64_t irsde_ssim_workspace(int32_t B, int32_t H, int32_t W, int32_t C, int32_t crop);
/* ssim[b] = mean SSIM of the crop-bordered images (11x11 Gaussian window, valid region), fp64 */
int irsde_ssim_u8(const uint8_t* a, const uint8_t* b, int32_t B, int32_t H, int32_t W, int32_t C, int32_t crop,
                  double* workspace, double* ssim, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* IRSDE_B200_H */
