// Shared declarations for the irsde_b200 native library (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <string>

namespace irsde {

typedef __nv_bfloat16 bf16;

// ---- small device helpers -------------------------------------------------------------------
__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(bf16 v) { return __bfloat162float(v); }
template <typename T>
__device__ __forceinline__ T from_f(float v);
template <>
__device__ __forceinline__ float from_f<float>(float v) { return v; }
template <>
__device__ __forceinline__ bf16 from_f<bf16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float silu_f(float v) { return v / (1.0f + expf(-v)); }

// ---- programmatic dependent launch (PDL) -----------------------------------------------------------
// Every kernel of the sampler step starts with PDL_ENTRY(): it lets the NEXT kernel of the stream be scheduled
// right away (its CTAs become resident and run their own prologue as SM resources free up) and then blocks until
// the PREVIOUS kernel has completed and flushed - so all global-memory accesses keep plain stream-order semantics,
// but the launch latency and the tail of one kernel overlap the ramp of the next.  pdl_launch() attaches the launch
// attribute (also inside stream capture: the step graph gets programmatic edges).  OPT-IN (IRSDE_PDL=1): the
// captured step graph uses plain edges by default; early-resident CTAs parked in griddepcontrol.wait can cost more
// than the launch gap they hide.
// Without the attribute the device instructions are no-ops.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#define PDL_ENTRY() \
  do {              \
    pdl_trigger();  \
    pdl_wait();     \
  } while (0)
extern bool g_pdl;
template <typename... KArgs, typename... Args>
inline cudaError_t pdl_launch(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = g_pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// A strided NHWC view: element (b,h,w,c) lives at p[((b*H + h)*W + w)*pitch + c].
struct View {
  void* p;
  int pitch;  // channel pitch of the underlying buffer (elements)
  int C;      // channels visible through the view
};

// ---- epilogue description shared by both conv engines ---------------------------------------
struct Epilogue {
  const float* bias;      // [Cout] or null
  const float* ss;        // time-modulation table base ([rows][ss_S]) or null
  const int* t_ptr;       // device int: current table row (null => row 0)
  int ss_S;               // row length of the table
  int ss_off;             // offset of this block's (scale[Cout], shift[Cout]) inside a row
  int ss_img_stride;      // rows per image (0 = shared time, 1 = per-image time)
  // per-output-channel multiplier (NAFBlock beta / gamma) or null: out = (acc + bias) * mult_vec.  Never combined with the
  // time table (tc_conv_create and the plan builder refuse it), so the engines need no common order for the two.
  const float* mult_vec;
  int silu;               // apply SiLU after modulation
  const void* res;        // residual view (same dtype as output) or null
  int res_pitch;
};

// ---- launch bookkeeping ------------------------------------------------------------------------
struct LaunchCounter {
  long long n = 0;
};

// ---- SIMT conv (conv_simt.cu) -----------------------------------------------------------------
struct ConvGeom {
  int B, Hin, Win, Cin;  // Hin/Win are the stored input size (before nearest upsample)
  int up;                // 1 or 2: nearest-neighbour upsample folded into the gather
  int KH, KW, stride, pad;
  int Hout, Wout, Cout;
};
// in/out dtype T (float or bf16), weights fp32 [KH*KW][Cin][Cout]; out_nchw != null writes fp32
// NCHW cropped to (cropH, cropW) instead of the NHWC view.
template <typename T>
void launch_conv_simt(const ConvGeom& g, const T* in, int in_pitch, const float* w, const Epilogue& ep, T* out,
                      int out_pitch, float* out_nchw, int cropH, int cropW, cudaStream_t st);
// The code path launch_conv_simt takes for these operands: {vecA (4-wide input gather), vecB (4-wide weight load), vecO
// (4-wide NHWC store), blocks}.
template <typename T>
void conv_simt_path(const ConvGeom& g, const T* in, int in_pitch, const float* w, const T* out, int out_pitch, int32_t path[4]);

// ---- elementwise / reduction kernels (elementwise.cu) -----------------------------------------
template <typename T>
void launch_prep_input(const float* xt, const float* cond, T* out, int B, int C, int H, int W, int Hp, int Wp,
                       int out_pitch, int conditional, cudaStream_t st, int pad_top = 0, int pad_left = 0, int row_pix = 0,
                       int img_rows = 0, int zero_pad = 0);
template <typename T>
void launch_nchw_to_nhwc(const float* in, T* out, int B, int C, int H, int W, int out_pitch, cudaStream_t st);
template <typename T>
void launch_nhwc_to_nchw(const T* in, int in_pitch, float* out, int B, int C, int H, int W, cudaStream_t st);
// channel LayerNorm (eps 1e-5) * g [* (scale+1) + shift from the time table] (+ residual)
struct LnMod {
  const float* ss;     // time table base or null
  const int* t_ptr;    // device row index (null => 0)
  int S, off_scale, off_shift, img_stride, pix_per_img;
};
template <typename T>
void launch_layernorm(const T* x, int x_pitch, const float* g, const T* res, int res_pitch, T* out, int out_pitch,
                      long long npix, int C, cudaStream_t st, const LnMod* mod = nullptr);
// the kernel launch_layernorm runs: layernorm_scalar_kernel, layernorm_vec_kernel<MAXV> (lpp lanes per pixel) or
// layernorm_geo_kernel<MAXV, LPP, PP>; res may be null
enum { LN_SCALAR = 0, LN_VEC = 1, LN_GEO = 2 };
struct LnPick {
  int kind, maxv, lpp, pp;
};
template <typename T>
LnPick ln_pick(int C, long long npix, int x_pitch, int res_pitch, int out_pitch, const void* x, const float* g, const void* res,
               const void* out);
// ---- NAFNet kernels (nafnet.cu)
// pixels per pooling chunk of an N-pixel image, and the chunks of an H x W image
int dw_pix(int N);
int dwgate_chunks(int H, int W);
template <typename T>
void launch_dwgate(const T* x, int x_pitch, const float* w, const float* bias, T* gate, int g_pitch, float* partial, int B,
                   int H, int W, int c, cudaStream_t st);
// true: sca_kernel scales the gate in place (one launch); false: a scale_channels_kernel pass follows (two launches)
bool sca_fused(int N);
template <typename T>
void launch_sca_scale(const float* partial, const float* w, const float* bias, float* sca, T* g, int g_pitch, int B, int c,
                      int nchunks, int N, int* launches, cudaStream_t st);
template <typename T>
void launch_scale_channels(T* x, int pitch, const float* sca, int B, int N, int c, cudaStream_t st);
template <typename T>
void launch_simple_gate(const T* x, int x_pitch, T* out, int o_pitch, long long npix, int c, cudaStream_t st);
template <typename T>
void launch_pixel_shuffle_add(const T* in, int in_pitch, const T* skip, int s_pitch, T* out, int o_pitch, int B, int h, int w, int q,
                              cudaStream_t st);
template <typename T>
void launch_add(const T* a, int a_pitch, const T* b, int b_pitch, T* out, int o_pitch, long long npix, int c, cudaStream_t st);
// dynamic shared memory of naf_time_mlp_kernel / time_mlp_kernel (bytes)
size_t naf_time_mlp_smem(int width);
size_t time_mlp_smem(int nf);
void launch_naf_time_gate(const float* times, int rows, int width, const float* w1, const float* b1, const float* w2,
                          const float* b2, float* tgate, cudaStream_t st);
// table[r][j] = dot(wall[j][0..td), tvec[r][0..td)) + ball[j]
void launch_time_rows(const float* tvec, int rows, int td, const float* wall, const float* ball, int S, float* table, cudaStream_t st);
// linear attention: qkv [B,N,384] -> ctx [B,4,32,32] (fp32) -> hidden [B,N,128].  The launchers launch nothing and return
// false when linattn_views_ok rejects the views (elem = sizeof(T); hidden may be null).
bool linattn_views_ok(const void* qkv, int qkv_pitch, const void* hidden, int hid_pitch, size_t elem);
template <typename T>
bool launch_linattn(const T* qkv, int qkv_pitch, float* partial, float* ctx, T* hidden, int hid_pitch, int B, int N,
                    cudaStream_t st);
size_t linattn_partial_floats(int B, int N);
// pass A's partition: nchunks chunks of 64 pixels per image, spread over nblk blocks per image (independent of B)
void linattn_partition(int B, int N, int* nblk, int* nchunks);
// passes A+B only (k,v -> ctx); and the fold of ctx into the to_out weights:
//   Mb[b][c][h*32+d] = sum_e Wout[c][h*32+e] * ctx[b][h][d][e]   (bf16, K-major rows of 128)
template <typename T>
bool launch_linattn_ctx(const T* qkv, int qkv_pitch, float* partial, float* ctx, int B, int N, cudaStream_t st);
void launch_la_fold(const float* ctx, const float* wout, bf16* Mb, int B, int C, cudaStream_t st);
// pass B alone: merge pass A's partial records into ctx [B][4][32][32]
void launch_la_combine(const float* partial, float* ctx, int B, int N, cudaStream_t st);
// Residual(PreNorm(LinearAttention)) in two fused passes over x (linattn_fused.cu, bf16, C = 64 or 128):
//   launch_la_kv_ln: LayerNorm(x; g1), k|v = W_kv xn (W_kv = rows 128..383 of the packed to_qkv weight, [256][C]), pass A's
//                    partial records (then launch_la_combine, launch_la_fold); xn_dump (tests; null in the plan) gets xn
//   launch_la_out_ln: out = LayerNorm(Mb[b] softmax_h(W_q xn) + bias; g2) + x  (W_q = rows 0..127, [128][C])
// linattn_fused_ok: C and the views the fused passes take (x: 16-byte vectors, out: bf16 pairs)
bool linattn_fused_ok(int C, const void* x, int x_pitch, const void* out, int out_pitch);
void launch_la_kv_ln(const bf16* x, int x_pitch, const float* g1, const bf16* wkv, float* partial, int B, int N, int C,
                     bf16* xn_dump, cudaStream_t st);
void launch_la_out_ln(const bf16* x, int x_pitch, const float* g1, const bf16* wq, const bf16* Mb, const float* bias,
                      const float* g2, bf16* out, int out_pitch, int B, int N, int C, cudaStream_t st);
// full softmax attention (denoising-sde mid_attn): qkv [B,N,384] -> hidden [B,N,128]; fullattn_pick is the kernel
// launch_fullattn runs (FA_MMA: bf16 only)
enum FullAttnKernel { FA_SCALAR = 0, FA_MMA = 1 };
template <typename T>
FullAttnKernel fullattn_pick(const T* qkv, int qkv_pitch, const T* hidden, int hid_pitch);
template <typename T>
void launch_fullattn(const T* qkv, int qkv_pitch, T* hidden, int hid_pitch, int B, int N, cudaStream_t st);
// time embedding: times[rows] -> table[rows][S]
void launch_time_table(const float* times, int rows, int nf, const float* w1, const float* b1, const float* w2,
                       const float* b2, const float* wall, const float* ball, int S, float* temb_ws, float* table,
                       cudaStream_t st);
// sampler update.  z == null draws z in-kernel, keyed by seed, uid_base / uids and t: from *st_dev in the chain, from the
// arguments (t_host) otherwise
struct StepState {
  int t;               // current timestep (table row)
  int i;               // executed-step index (z slice)
  const float* z;      // pre-drawn noise [T][n] or null (in-kernel Philox)
  unsigned long long seed;
  unsigned long long uid_base;  // uid of the batch's first image (Philox is keyed per image)
  const unsigned long long* uids;  // explicit per-image uids [B] or null (uid = uid_base + b)
};
void launch_sde_update(int mode, const float* x, const float* mu, const float* noise, const float* z, long long z_stride,
                       const float* coef, const StepState* st_dev, int t_host, float* out, long long n, uint64_t seed,
                       long long img_elems, uint64_t uid_base, const unsigned long long* uids, cudaStream_t st);
void launch_advance_step(StepState* st_dev, cudaStream_t st);
void launch_set_step(StepState* st_dev, int t, int i, const float* z, unsigned long long seed, unsigned long long uid_base,
                     const unsigned long long* uids, cudaStream_t st);
void launch_noise_state(const float* mu, float* out, long long n, float max_sigma, uint64_t seed, long long img_elems,
                        uint64_t uid_base, const unsigned long long* uids, cudaStream_t st);
void launch_random_states(const float* x0, const float* mu, const float* noise, const float* w, const float* sb, float* out,
                          int B, long long img_elems, cudaStream_t st);
// layout helpers for the tensor-core path
template <typename T>
void launch_space_to_depth(const T* in, int in_pitch, T* out, int B, int H, int W, int C, cudaStream_t st);

// ---- tensor-core (wgmma) tap-GEMM conv (conv_tc.cu) ---------------------------------------------------------
struct TcTap {
  int dh, dw;   // pixel offset of this tap in the A tensor
  int plane;    // 5th coordinate of the A tensor map (space-to-depth plane), 0 otherwise
};
struct TcConvDesc;  // opaque: tensor maps + tap table + tile config
// S = bf16, or float for fp32x3 (3 x tf32 wgmma on hi/lo split fp32 operands, fp32 output; see conv_tc.cu MODE 3).
// in: [planes][B][Hin][Win] pixels of in_pitch elements; fp32x3: the launch_split_tf32 output [2][planes][B][H][W][Cin]
// (in_pitch = Cin); the 7x7 stem (bf16, planes < 0): its padded [B][Hin+6][Win+8][8] layout (in_pitch = 8; the creator
// takes Cin = 64, whatever is passed).  w: [phase][tap][Cout_w][Cin] (bf16 per-image weights: [B][Cout_w][Cin]); fp32x3: [phase*tap][2][Cout_w][Cin].
// nphases: 1 or 4 (upsample phases).  out == nullptr: fp32 NCHW output, set at launch (tc_conv_set_out_nchw).
template <typename S>
TcConvDesc* tc_conv_create(const S* in, int in_pitch, int B, int Hin, int Win, int Cin, int planes, const S* w, int Cout, int ntaps,
                           const TcTap* taps, int nphases, const Epilogue& ep, S* out, int out_pitch, int Hout, int Wout,
                           std::string* err, int flags = 0);
enum { TC_FLAG_QSOFTMAX = 1, TC_FLAG_W_PER_IMAGE = 2 };  // bf16 only
// hi = rn_tf32(x), lo = rn_tf32(x - hi) of a pitched NHWC fp32 view -> dense out[0][npix][C] (hi), out[1][npix][C] (lo)
void launch_split_tf32(const float* in, int in_pitch, float* out, long long npix, int C, cudaStream_t st);
void tc_conv_destroy(TcConvDesc*);
void tc_conv_set_runtime(TcConvDesc*, const float* ss, const int* t_ptr, int ss_img_stride);
void tc_conv_set_out_nchw(TcConvDesc*, float* out, int cropH, int cropW);  // out==nullptr at create => fp32 NCHW output
int tc_conv_launch(TcConvDesc*, cudaStream_t st);  // returns number of launches (1), <0 on error
// the kernel tc_conv_launch would run now (call after tc_conv_set_runtime): {BN, MODE, EKT, number of output tiles}
void tc_conv_query(const TcConvDesc*, int info[4]);
bool tc_init(std::string* err);                    // resolves cuTensorMapEncodeTiled

// ---- image conversion / metrics (imaging.cu) ---------------------------------------------------
void launch_tensor2img(const float* in, unsigned char* out, int B, int C, int H, int W, double lo, double hi, cudaStream_t st);
void launch_img2tensor(const unsigned char* in, float* out, int B, int C, int H, int W, cudaStream_t st);
void launch_sqerr_u8(const unsigned char* a, const unsigned char* b, int B, int H, int W, int C, int crop, unsigned long long* out,
                     cudaStream_t st);
long long ssim_partial_count(int H, int W, int C, int crop);
void launch_ssim_u8(const unsigned char* a, const unsigned char* b, int B, int H, int W, int C, int crop, double* partial, double* out,
                    cudaStream_t st);

}  // namespace irsde
