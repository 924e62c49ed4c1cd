// irsde_b200 engine: context, weight store/repack, ConditionalUNet launch plan, sampler chain
// (CUDA-graph replay of one captured step) and the C ABI declared in include/irsde_b200.h.
//
// Data layout in HBM: activations are NHWC (channels-last) so that the skip concatenations of the
// UNet (DenoisingUNet_arch.py:118,121,127) are channel-offset views into one pre-allocated buffer
// (producers write at their channel offset: no torch.cat copies) and so that a 64-channel slab of a
// pixel row is one 128-byte line (the TMA / UMMA swizzle atom of the tensor-core engine).
#include <dlfcn.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <functional>
#include <map>
#include <string>
#include <tuple>
#include <type_traits>
#include <vector>

#include "../../include/irsde_b200.h"
#include "common.cuh"

using namespace irsde;

namespace irsde {
bool g_pdl = false;  // IRSDE_PDL=1 enables programmatic dependent launch (read in tc_init)
}

namespace {
thread_local std::string g_last_error;

struct RawTensor {
  std::vector<int64_t> shape;
  float* dev = nullptr;
  long long numel = 0;
};

struct RunCfg {  // per-invocation pointers read by the op closures at launch time
  const float* x = nullptr;
  const float* mu = nullptr;
  float* out = nullptr;
  const float* ss = nullptr;  // time-modulation table
  const int* t_ptr = nullptr;
  int ss_img_stride = 0;
};

struct Plan;
typedef std::function<int(Plan*, cudaStream_t)> Op;  // enqueues the op's kernels, returns how many it launched
enum { CAT_TC = 0, CAT_SIMT, CAT_LN, CAT_ATTN, CAT_MISC, CAT_UPDATE, CAT_COUNT };
struct OpRec {
  int cat;
  double flops;  // executed multiply-add flops (2*MAC) of this op, 0 for memory-bound ops
  Op fn;
  std::string label;   // for IRSDE_PROFILE_DUMP
  double bytes = 0.0;  // algorithmic HBM bytes (inputs + outputs + weights once)
  // NHWC view this op writes (irsde_trace_forward reads it back right after the op ran); null for fp32-NCHW outputs
  const void* out_p = nullptr;
  int out_pitch = 0, out_C = 0, out_H = 0, out_W = 0;
};

struct Plan {
  int B, H, W, Hp, Wp;
  std::vector<void*> allocs;
  std::vector<OpRec> ops;
  std::vector<OpRec> ops_dec;  // latent UNet: decode half (ops = encode half)
  int lat_h = 0, lat_w = 0;     // latent spatial size
  std::vector<TcConvDesc*> tc_descs;
  RunCfg cur;
  // chain state
  float *x_state = nullptr, *mu_buf = nullptr, *eps_buf = nullptr;
  StepState* d_step = nullptr;
  int* d_zero = nullptr;
  float *fwd_times = nullptr, *fwd_temb = nullptr, *fwd_table = nullptr;        // module-forward table (B rows)
  float *chain_times = nullptr, *chain_temb = nullptr, *chain_table = nullptr;  // chain table rows 0..cap-1
  int chain_cap = 0;
  cudaGraphExec_t graph[IRSDE_NUM_MODES] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  long long step_launches[IRSDE_NUM_MODES] = {0, 0, 0, 0, 0};
  long long bytes = 0;               // device memory owned by this plan (plan cache accounting)
  unsigned long long last_use = 0;   // LRU stamp
};
}  // namespace

struct NafCfg {
  bool on = false;
  int img_channel = 0, width = 0, middle = 0, n_enc = 0, n_dec = 0;
  int enc[8] = {0}, dec[8] = {0};
  bool latent = false;
};

// Refusion latent autoencoder UNet (codes/config/latent-dehazing/models/modules/UNet_arch.py:17-97)
struct LatCfg {
  bool on = false;
  int in_ch = 0, out_ch = 0, ch = 0, depth = 0, embed = 0;
  int mult[9] = {1, 0, 0, 0, 0, 0, 0, 0, 0};  // [1] + ch_mult
};

struct irsde_ctx {
  irsde_config cfg;
  NafCfg naf;
  LatCfg lat;
  mutable std::string err;
  std::map<std::string, RawTensor> raw;
  bool finalized = false;
  std::map<std::string, float*> w_simt;  // [KH*KW][Cin][Cout] fp32
  std::map<std::string, bf16*> w_tc;     // [phase][tap][Cout][Cin] bf16
  std::map<std::string, float*> w_tc3;   // fp32x3: [phase][tap][2 (hi,lo)][Cout_pad][Cin] fp32 (tf32-rounded parts)
  bool use_tc3 = false;                  // fp32x3 mode: fp32 storage, convs through 3 x tf32 wgmma
  std::map<std::string, int> ss_off;
  float *wall = nullptr, *ball = nullptr;
  int S = 0;
  // schedule
  bool have_sched = false;
  int T = 0;
  float dt = 0, max_sigma = 0;
  std::vector<float> thetas, sigmas, cumsum, sbars;
  float* coef_dev[IRSDE_NUM_MODES] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  std::map<std::tuple<int, int, int>, Plan*> plans;  // LRU-bounded cache, see build_plan()
  unsigned long long use_clock = 0;
  long long plan_bytes = 0;
  long long launches = 0;
  unsigned long long image_base = 0;  // uid of the first image of the next batch (Philox key; irsde_set_image_base)
  void* nccl_comm = nullptr;             // ncclComm_t (irsde_comm_init)
  int comm_rank = 0, comm_nranks = 1;
  unsigned long long* d_uids = nullptr;  // explicit per-image uids (irsde_set_image_uids), capacity MAX_UIDS
  int n_uids = 0;                        // 0: uid = image_base + b
  long long dev_bytes = 0;
  std::vector<void*> allocs;
  bool tc_ok = false;
  bool prof = false;
  struct ProfEv { int cat; double flops; cudaEvent_t e0, e1; const OpRec* op; };
  std::vector<ProfEv> prof_events;
  bool use_tc = false;  // bf16 mode: route eligible convs through the wgmma tap-GEMM engine
  std::vector<int> udim;  // UNet channels per level: nf * [1, ch_mult...] (DenoisingUNet_arch.py:51-56)
  cudaEvent_t order_ev = nullptr;    // end of the work the last stream-ordered call enqueued (StreamOrder)
  cudaStream_t order_st = nullptr;   // the stream that call ran on
};

namespace {

#define CUDA_TRY(ctx, expr)                                                                      \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      char _b[512];                                                                              \
      snprintf(_b, sizeof(_b), "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      (ctx)->err = _b;                                                                           \
      g_last_error = _b;                                                                         \
      return IRSDE_ERR_CUDA;                                                                     \
    }                                                                                            \
  } while (0)

int fail(const irsde_ctx* ctx, int code, const std::string& msg) {
  if (ctx) ctx->err = msg;
  g_last_error = msg;
  return code;
}

// the time MLPs run with the default dynamic shared memory limit (no cudaFuncSetAttribute opt-in)
constexpr size_t kTimeMlpSmemMax = 48 * 1024;
// sca_kernel keeps the c channel means in dynamic shared memory, under the same limit
constexpr int kScaMaxC = 48 * 1024 / 4;

// The shape limits of the kernels' launches and index arithmetic (include/irsde_b200.h "Shape limits"), checked on the host
// before anything is allocated or launched, by the plan builder and by every standalone entry:
//   - a grid's y and z dimensions take at most 65535: the kernels put B there (the LinearAttention passes, dwgate / sca,
//     the time table's rows, tensor2img / img2tensor / sqerr / ssim) and 4 B for full attention (one row per image and head);
//   - the network kernels (dwgate / sca, LinearAttention, full attention, the tap-GEMM conv) hold the pixel count of one image
//     (N = H * W, a pixel index inside it) in int: H * W <= 2^30.  The image entries index in long long and pass 1 x 1.
// grid_rows is the largest value the caller's launches put in y or z, named by `what`; H, W is the largest image they see.
constexpr long long kMaxGridYZ = 65535, kMaxImagePixels = 1LL << 30;
int check_shape_limits(const irsde_ctx* ctx, long long grid_rows, const char* what, long long H, long long W) {
  char b[256];
  if (grid_rows > kMaxGridYZ) {
    snprintf(b, sizeof b, "%s = %lld exceeds 65535, the CUDA grid y / z limit of the launches that index it", what, grid_rows);
    return fail(ctx, IRSDE_ERR_INVALID, b);
  }
  if (H * W > kMaxImagePixels) {
    snprintf(b, sizeof b, "an image of %lld x %lld pixels exceeds 2^30 pixels, the int pixel count of the kernels", H, W);
    return fail(ctx, IRSDE_ERR_INVALID, b);
  }
  return IRSDE_OK;
}

// The calls that use a context's plans, time tables or uid buffer (noise_fn, reverse, trace_forward, latent encode /
// decode, set_image_uids, noise_state_images, step_philox) share those buffers whatever stream they run on.  One event
// per context serializes them: every such call records it on its stream when it returns, and a call on another stream
// than the previous one first makes its stream wait for it.  No launch is added.
struct StreamOrder {
  irsde_ctx* ctx;
  cudaStream_t st;
  StreamOrder(irsde_ctx* c, cudaStream_t s) : ctx(c), st(s) {
    if (!ctx->order_ev) cudaEventCreateWithFlags(&ctx->order_ev, cudaEventDisableTiming);
    else if (ctx->order_st != st) cudaStreamWaitEvent(st, ctx->order_ev, 0);
  }
  ~StreamOrder() {
    if (!ctx->order_ev) return;
    cudaEventRecord(ctx->order_ev, st);
    ctx->order_st = st;
  }
};

// ctx may be null (the entries that take no context): nothing is counted
void* dev_alloc(irsde_ctx* ctx, size_t bytes, std::vector<void*>* owner) {
  void* p = nullptr;
  if (bytes == 0) bytes = 16;
  if (cudaMalloc(&p, bytes) != cudaSuccess) return nullptr;
  if (ctx) ctx->dev_bytes += (long long)bytes;
  owner->push_back(p);
  return p;
}

// ---- weight repack kernels ---------------------------------------------------------------------
__global__ void pack_simt_kernel(const float* __restrict__ w, float* __restrict__ o, int Cout, int Cin, int KH, int KW) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)Cout * Cin * KH * KW;
  if (idx >= total) return;
  int co = idx % Cout;
  int c = (idx / Cout) % Cin;
  int tap = idx / ((long long)Cout * Cin);
  int r = tap / KW, s = tap % KW;
  o[idx] = w[(((long long)co * Cin + c) * KH + r) * KW + s];
}
// 7x7 stem as 7 row-taps with K=64 = 8 pixels x 8 channels (see conv_tc.cu): [r][Cout][s*8+c]
__global__ void pack_tc_stem_kernel(const float* __restrict__ w, bf16* __restrict__ o, int Cout, int Cin) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)7 * Cout * 64;
  if (idx >= total) return;
  int j = idx % 64;
  int co = (idx / 64) % Cout;
  int r = idx / ((long long)64 * Cout);
  int s = j >> 3, c = j & 7;
  float v = (s < 7 && c < Cin) ? w[(((long long)co * Cin + c) * 7 + r) * 7 + s] : 0.f;
  o[idx] = __float2bfloat16_rn(v);
}

// Tap-GEMM weight element (tap, co, c) of a [tap][Cout_pad][Cin] layout.  bf16: one value.  fp32x3: [tap][2 (hi, lo)]
// [Cout_pad][Cin] fp32, hi = rn_tf32(w), lo = rn_tf32(w - hi).
__device__ __forceinline__ float rn_tf32_w(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
__device__ __forceinline__ void store_tc_w(bf16* o, int tap, int co, int c, int Cout_pad, int Cin, float v) {
  o[((long long)tap * Cout_pad + co) * Cin + c] = __float2bfloat16_rn(v);
}
__device__ __forceinline__ void store_tc_w(float* o, int tap, int co, int c, int Cout_pad, int Cin, float v) {
  const float hi = rn_tf32_w(v);
  const long long base = ((long long)tap * 2 * Cout_pad + co) * Cin + c;
  o[base] = hi;
  o[base + (long long)Cout_pad * Cin] = rn_tf32_w(v - hi);
}
// [tap][Cout_pad][Cin] with zero rows for co >= Cout (head conv, Cout=3)
template <typename S>
__global__ void pack_tc_taps_kernel(const float* __restrict__ w, S* __restrict__ o, int Cout, int Cout_pad, int Cin, int KH, int KW) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)Cout_pad * Cin * KH * KW;
  if (idx >= total) return;
  int c = idx % Cin;
  int co = (idx / Cin) % Cout_pad;
  int tap = idx / ((long long)Cout_pad * Cin);
  int r = tap / KW, s = tap % KW;
  store_tc_w(o, tap, co, c, Cout_pad, Cin, co < Cout ? w[(((long long)co * Cin + c) * KH + r) * KW + s] : 0.f);
}
// nearest-x2 upsample followed by 3x3/pad1 == four 2x2 phase convolutions on the low-res input with
// pre-summed weights: [phase=(py,px)][tap=(a,b)][Cout_pad][Cin]
template <typename S>
__global__ void pack_tc_up_kernel(const float* __restrict__ w, S* __restrict__ o, int Cout, int Cout_pad, int Cin) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)16 * Cout_pad * Cin;
  if (idx >= total) return;
  int c = idx % Cin;
  int co = (idx / Cin) % Cout_pad;
  int tap = (idx / ((long long)Cout_pad * Cin)) % 4;
  int phase = idx / ((long long)4 * Cout_pad * Cin);
  int py = phase >> 1, px = phase & 1, a = tap >> 1, b = tap & 1;
  // rows of the 3x3 kernel that fall on low-res offset a for phase py
  int r0, r1, s0, s1;
  if (py == 0) { if (a == 0) { r0 = 0; r1 = 0; } else { r0 = 1; r1 = 2; } }
  else         { if (a == 0) { r0 = 0; r1 = 1; } else { r0 = 2; r1 = 2; } }
  if (px == 0) { if (b == 0) { s0 = 0; s1 = 0; } else { s0 = 1; s1 = 2; } }
  else         { if (b == 0) { s0 = 0; s1 = 1; } else { s0 = 2; s1 = 2; } }
  float acc = 0.f;  // fp32 sum in this order, then one rounding
  if (co < Cout)
    for (int r = r0; r <= r1; ++r)
      for (int s = s0; s <= s1; ++s) acc += w[(((long long)co * Cin + c) * 3 + r) * 3 + s];
  store_tc_w(o, phase * 4 + tap, co, c, Cout_pad, Cin, acc);
}

// Packed conv weight layouts.  SIMT: [KH*KW][Cin][Cout] fp32.  Tap-GEMM (stored as S: bf16, or float for the fp32x3 engine's
// tf32 hi/lo pairs): plain taps [KH*KW][Cout_pad][Cin]; upsample phases (nearest x2 + 3x3) [4][4][Cout_pad][Cin]; the bf16
// 7x7 stem [7][Cout][64]; per-image 1x1 weights [B*Cout][Cin] from a raw [B][Cout][Cin].
enum WLayout { WL_SIMT, WL_TAPS, WL_UP, WL_STEM, WL_PER_IMAGE };
// rows per tap of a tap-GEMM layout: Cout padded to 8, except the bf16 upsample layout (Cout rows) and per-image weights
template <typename S>
int packed_rows(WLayout l, int Cout, int B) {
  if (l == WL_PER_IMAGE) return B * Cout;
  return l == WL_UP && std::is_same<S, bf16>::value ? Cout : (Cout + 7) / 8 * 8;
}
template <typename S>
long long packed_weight_elems(WLayout l, int Cout, int Cin, int KH, int KW, int B = 1) {
  const long long parts = std::is_same<S, float>::value ? 2 : 1, rows = packed_rows<S>(l, Cout, B);
  switch (l) {
    case WL_SIMT: return (long long)Cout * Cin * KH * KW;
    case WL_STEM: return 7LL * Cout * 64;
    case WL_UP: return 16 * parts * rows * Cin;
    default: return parts * rows * Cin * KH * KW;
  }
}
template <typename S>
void pack_weight(WLayout l, const float* w, S* o, int Cout, int Cin, int KH, int KW, int B, cudaStream_t st) {
  const long long n = packed_weight_elems<S>(l, Cout, Cin, KH, KW, B);
  const int rows = packed_rows<S>(l, Cout, B);
  if constexpr (std::is_same<S, float>::value) {
    if (l == WL_SIMT) { pack_simt_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(w, o, Cout, Cin, KH, KW); return; }
  } else {
    if (l == WL_STEM) { pack_tc_stem_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(w, o, Cout, Cin); return; }
  }
  const long long nt = n / (std::is_same<S, float>::value ? 2 : 1);  // one thread per (hi, lo) pair
  if (l == WL_UP) pack_tc_up_kernel<S><<<(unsigned)((nt + 255) / 256), 256, 0, st>>>(w, o, Cout, rows, Cin);
  else pack_tc_taps_kernel<S><<<(unsigned)((nt + 255) / 256), 256, 0, st>>>(w, o, l == WL_PER_IMAGE ? rows : Cout, rows, Cin, KH, KW);
}

// How the tap-GEMM runs a conv shape (callers have checked stride and padding): 3x3/1, nearest x2 + 3x3/1 (four 2x2 phase
// convolutions), 1x1, 4x4/2 and 2x2/2 (over space-to-depth planes), and the 7x7 stem (7 row taps over its padded layout).
struct TapTable {
  TcTap taps[16];
  int ntaps = 0;
  int nph = 1;     // upsample phases
  int planes = 1;  // A planes: 4 after the space-to-depth pass, -1 for the stem
  bool s2d() const { return planes == 4; }
};
TapTable tap_table(int K, int up) {
  TapTable t;
  if (K == 7) {
    for (int r = 0; r < 7; ++r) t.taps[t.ntaps++] = TcTap{r, 0, 0};
    t.planes = -1;
  } else if (K == 3 && up == 1) {
    for (int r = 0; r < 3; ++r) for (int q = 0; q < 3; ++q) t.taps[t.ntaps++] = TcTap{r - 1, q - 1, 0};
  } else if (K == 3) {
    t.nph = 4;
    for (int a = 0; a < 2; ++a) for (int q = 0; q < 2; ++q) t.taps[t.ntaps++] = TcTap{a - 1, q - 1, 0};
  } else if (K == 1) {
    t.taps[t.ntaps++] = TcTap{0, 0, 0};
  } else {  // stride 2 over space-to-depth planes: 4x4 pad 1 (UNet Downsample) or 2x2 pad 0 (NAFNet downs)
    static const int PY[4] = {1, 0, 1, 0}, DH[4] = {-1, 0, 0, 1};
    if (K == 4) {
      for (int r = 0; r < 4; ++r) for (int q = 0; q < 4; ++q) t.taps[t.ntaps++] = TcTap{DH[r], DH[q], PY[r] * 2 + PY[q]};
    } else {
      for (int r = 0; r < 2; ++r) for (int q = 0; q < 2; ++q) t.taps[t.ntaps++] = TcTap{0, 0, r * 2 + q};
    }
    t.planes = 4;
  }
  return t;
}

// ---- architecture description --------------------------------------------------------------------
struct ResBlockInfo {
  std::string pre;
  int cin, cout;
};
// D[i] = channels of level i: nf * [1, ch_mult...][i] (nf * 2^i for the plain depth constructor)
std::vector<ResBlockInfo> resblocks(const irsde_config& c, const std::vector<int>& D) {
  std::vector<ResBlockInfo> v;
  char b[64];
  for (int i = 0; i < c.depth; ++i) {
    int di = D[i];
    snprintf(b, sizeof b, "downs.%d.0.", i); v.push_back({b, di, di});
    snprintf(b, sizeof b, "downs.%d.1.", i); v.push_back({b, di, di});
  }
  int mid = D[c.depth];
  v.push_back({"mid_block1.", mid, mid});
  v.push_back({"mid_block2.", mid, mid});
  for (int j = 0; j < c.depth; ++j) {
    int i = c.depth - 1 - j, di = D[i], dout = D[i + 1];
    snprintf(b, sizeof b, "ups.%d.0.", j); v.push_back({b, dout + di, dout});
    snprintf(b, sizeof b, "ups.%d.1.", j); v.push_back({b, dout + di, dout});
  }
  v.push_back({"final_res_block.", 2 * c.nf, c.nf});
  return v;
}

// How irsde_finalize_weights packs a parameter: RAW stays fp32 as loaded (vectors, Linear matrices, gains, and the NAFBlock's
// beta / gamma, depthwise and SCA weights, which their kernels read raw); TAPS is a conv weight over its own taps; UP is the
// 3x3 conv of an Upsample, run as four 2x2 phases over the low-resolution input (nearest x2 + 3x3).
enum Pack { PACK_RAW, PACK_TAPS, PACK_UP };
struct ParamSpec {
  std::string name;
  std::vector<int64_t> shape;
  Pack pack = PACK_RAW;
};

// NAFBlocks of ConditionalNAFNet in a fixed order (prefix, channels)   DenoisingNAFNet_arch.py:111-141
struct NafBlockInfo {
  std::string pre;
  int c;
};
std::vector<NafBlockInfo> naf_blocks(const NafCfg& n) {
  std::vector<NafBlockInfo> v;
  char b[64];
  int chan = n.width;
  for (int i = 0; i < n.n_enc; ++i) {
    for (int j = 0; j < n.enc[i]; ++j) { snprintf(b, sizeof b, "encoders.%d.%d.", i, j); v.push_back({b, chan}); }
    chan *= 2;
  }
  for (int j = 0; j < n.middle; ++j) { snprintf(b, sizeof b, "middle_blks.%d.", j); v.push_back({b, chan}); }
  for (int i = 0; i < n.n_dec; ++i) {
    chan /= 2;
    for (int j = 0; j < n.dec[i]; ++j) { snprintf(b, sizeof b, "decoders.%d.%d.", i, j); v.push_back({b, chan}); }
  }
  return v;
}
// variant: IRSDE_NET_CONDITIONAL reads cat(x - cond, cond); the denoising-sde task's network reads x alone
// (codes/config/denoising-sde/models/modules/DenoisingNAFNet_arch.py:103)
std::vector<ParamSpec> naf_param_specs(const NafCfg& n, int variant) {
  std::vector<ParamSpec> v;
  int64_t w = n.width, td = 4 * w, ic = n.img_channel;
  v.push_back({"time_mlp.1.weight", {2 * td, w}});
  v.push_back({"time_mlp.1.bias", {2 * td}});
  v.push_back({"time_mlp.3.weight", {td, td}});
  v.push_back({"time_mlp.3.bias", {td}});
  v.push_back({"intro.weight", {w, variant == IRSDE_NET_CONDITIONAL ? 2 * ic : ic, 3, 3}, PACK_TAPS});
  v.push_back({"intro.bias", {w}});
  v.push_back({"ending.weight", {ic, w, 3, 3}, PACK_TAPS});
  v.push_back({"ending.bias", {ic}});
  for (auto& blk : naf_blocks(n)) {
    int64_t c = blk.c;
    const std::string& p = blk.pre;
    v.push_back({p + "beta", {1, c, 1, 1}});
    v.push_back({p + "gamma", {1, c, 1, 1}});
    v.push_back({p + "mlp.1.weight", {4 * c, td / 2}});
    v.push_back({p + "mlp.1.bias", {4 * c}});
    v.push_back({p + "conv1.weight", {2 * c, c, 1, 1}, PACK_TAPS});
    v.push_back({p + "conv1.bias", {2 * c}});
    v.push_back({p + "conv2.weight", {2 * c, 1, 3, 3}});
    v.push_back({p + "conv2.bias", {2 * c}});
    v.push_back({p + "conv3.weight", {c, c, 1, 1}, PACK_TAPS});
    v.push_back({p + "conv3.bias", {c}});
    v.push_back({p + "sca.1.weight", {c, c, 1, 1}});
    v.push_back({p + "sca.1.bias", {c}});
    v.push_back({p + "conv4.weight", {2 * c, c, 1, 1}, PACK_TAPS});
    v.push_back({p + "conv4.bias", {2 * c}});
    v.push_back({p + "conv5.weight", {c, c, 1, 1}, PACK_TAPS});
    v.push_back({p + "conv5.bias", {c}});
    v.push_back({p + "norm1.g", {1, c, 1, 1}});
    v.push_back({p + "norm2.g", {1, c, 1, 1}});
  }
  char b[64];
  int64_t chan = w << n.n_enc;
  for (int i = 0; i < n.n_dec; ++i) {
    snprintf(b, sizeof b, "ups.%d.0.weight", i);
    v.push_back({b, {chan * 2, chan, 1, 1}, PACK_TAPS});
    chan /= 2;
  }
  chan = w;
  for (int i = 0; i < n.n_enc; ++i) {
    snprintf(b, sizeof b, "downs.%d.", i);
    v.push_back({std::string(b) + "weight", {chan * 2, chan, 2, 2}, PACK_TAPS});
    v.push_back({std::string(b) + "bias", {chan * 2}});
    chan *= 2;
  }
  return v;
}
std::vector<ParamSpec> param_specs(const irsde_config& c, const std::vector<int>& D) {
  std::vector<ParamSpec> v;
  int64_t nf = c.nf, td = 4 * nf;
  int64_t cin0 = c.variant == IRSDE_NET_CONDITIONAL ? 2 * c.in_nc : c.in_nc;
  v.push_back({"init_conv.weight", {nf, cin0, 7, 7}, PACK_TAPS});
  v.push_back({"time_mlp.1.weight", {td, nf}});
  v.push_back({"time_mlp.1.bias", {td}});
  v.push_back({"time_mlp.3.weight", {td, td}});
  v.push_back({"time_mlp.3.bias", {td}});
  for (auto& rb : resblocks(c, D)) {
    v.push_back({rb.pre + "mlp.1.weight", {2 * rb.cout, td}});
    v.push_back({rb.pre + "mlp.1.bias", {2 * rb.cout}});
    v.push_back({rb.pre + "block1.proj.weight", {rb.cout, rb.cin, 3, 3}, PACK_TAPS});
    v.push_back({rb.pre + "block2.proj.weight", {rb.cout, rb.cout, 3, 3}, PACK_TAPS});
    if (rb.cin != rb.cout) v.push_back({rb.pre + "res_conv.weight", {rb.cout, rb.cin, 1, 1}, PACK_TAPS});
  }
  auto attn = [&](const std::string& pre, int64_t C, bool full) {
    v.push_back({pre + "fn.fn.to_qkv.weight", {384, C, 1, 1}, PACK_TAPS});
    if (full) {
      v.push_back({pre + "fn.fn.to_out.weight", {C, 128, 1, 1}, PACK_TAPS});
      v.push_back({pre + "fn.fn.to_out.bias", {C}});
    } else {
      v.push_back({pre + "fn.fn.to_out.0.weight", {C, 128, 1, 1}, PACK_TAPS});
      v.push_back({pre + "fn.fn.to_out.0.bias", {C}});
      v.push_back({pre + "fn.fn.to_out.1.g", {1, C, 1, 1}});
    }
    v.push_back({pre + "fn.norm.g", {1, C, 1, 1}});
  };
  char b[64];
  for (int i = 0; i < c.depth; ++i) {
    int64_t di = D[i], dout = D[i + 1];
    snprintf(b, sizeof b, "downs.%d.2.", i);
    attn(b, di, false);
    snprintf(b, sizeof b, "downs.%d.3.", i);
    if (i != c.depth - 1) {
      v.push_back({std::string(b) + "weight", {dout, di, 4, 4}, PACK_TAPS});
      v.push_back({std::string(b) + "bias", {dout}});
    } else {
      v.push_back({std::string(b) + "weight", {dout, di, 3, 3}, PACK_TAPS});
    }
  }
  attn("mid_attn.", D[c.depth], c.variant == IRSDE_NET_DENOISING);
  for (int j = 0; j < c.depth; ++j) {
    int i = c.depth - 1 - j;
    int64_t di = D[i], dout = D[i + 1];
    snprintf(b, sizeof b, "ups.%d.2.", j);
    attn(b, dout, false);
    if (i != 0) {
      snprintf(b, sizeof b, "ups.%d.3.1.", j);
      v.push_back({std::string(b) + "weight", {di, dout, 3, 3}, PACK_UP});
      v.push_back({std::string(b) + "bias", {di}});
    } else {
      snprintf(b, sizeof b, "ups.%d.3.", j);
      v.push_back({std::string(b) + "weight", {di, dout, 3, 3}, PACK_TAPS});
    }
  }
  v.push_back({"final_conv.weight", {c.out_nc, nf, 3, 3}, PACK_TAPS});
  v.push_back({"final_conv.bias", {c.out_nc}});
  return v;
}

std::vector<ParamSpec> lat_param_specs(const LatCfg& L) {
  std::vector<ParamSpec> v;
  char b[64];
  v.push_back({"init_conv.weight", {L.ch, L.in_ch, 3, 3}, PACK_TAPS});
  auto rb = [&](const std::string& pre, int64_t ci, int64_t co) {
    v.push_back({pre + "block1.proj.weight", {co, ci, 3, 3}, PACK_TAPS});
    v.push_back({pre + "block2.proj.weight", {co, co, 3, 3}, PACK_TAPS});
    if (ci != co) v.push_back({pre + "res_conv.weight", {co, ci, 1, 1}, PACK_TAPS});
  };
  auto la = [&](const std::string& pre, int64_t C) {
    v.push_back({pre + "fn.fn.to_qkv.weight", {384, C, 1, 1}, PACK_TAPS});
    v.push_back({pre + "fn.fn.to_out.0.weight", {C, 128, 1, 1}, PACK_TAPS});
    v.push_back({pre + "fn.fn.to_out.0.bias", {C}});
    v.push_back({pre + "fn.fn.to_out.1.g", {1, C, 1, 1}});
    v.push_back({pre + "fn.norm.g", {1, C, 1, 1}});
  };
  for (int i = 0; i < L.depth; ++i) {
    int64_t di = (int64_t)L.ch * L.mult[i], dout = (int64_t)L.ch * L.mult[i + 1];
    snprintf(b, sizeof b, "encoder.%d.", i);
    std::string pre = b;
    rb(pre + "0.", di, di);
    rb(pre + "1.", di, di);
    if (i == L.depth - 1) la(pre + "2.", di);
    if (i != L.depth - 1) {
      v.push_back({pre + "3.weight", {dout, di, 4, 4}, PACK_TAPS});
      v.push_back({pre + "3.bias", {dout}});
    } else {
      v.push_back({pre + "3.weight", {dout, di, 3, 3}, PACK_TAPS});
    }
  }
  for (int j = 0; j < L.depth; ++j) {
    int i = L.depth - 1 - j;
    int64_t di = (int64_t)L.ch * L.mult[i], dout = (int64_t)L.ch * L.mult[i + 1];
    snprintf(b, sizeof b, "decoder.%d.", j);
    std::string pre = b;
    rb(pre + "0.", dout + di, dout);
    rb(pre + "1.", dout + di, dout);
    if (i == L.depth - 1) la(pre + "2.", dout);
    if (i != 0) {
      v.push_back({pre + "3.1.weight", {di, dout, 3, 3}, PACK_UP});
      v.push_back({pre + "3.1.bias", {di}});
    } else {
      v.push_back({pre + "3.weight", {di, dout, 3, 3}, PACK_TAPS});
    }
  }
  int64_t mid = (int64_t)L.ch * L.mult[L.depth];
  v.push_back({"latent_conv.weight", {L.embed, mid, 1, 1}, PACK_TAPS});
  v.push_back({"post_latent_conv.weight", {mid, L.embed, 1, 1}, PACK_TAPS});
  v.push_back({"final_conv.weight", {L.out_ch, L.ch, 3, 3}, PACK_TAPS});
  v.push_back({"final_conv.bias", {L.out_ch}});
  return v;
}

// Which of the tap-GEMM's conv shapes (tap_table) a conv is: 3x3/1 pad 1 (also after nearest x2), 1x1, 4x4/2 pad 1 or 2x2/2
// pad 0 over an even H x W, or the 7x7/1 pad 3 stem.  The plan builder and each standalone entry apply their own engine
// rules on top.
struct ConvShape {
  bool k3, k1, k4, k2, k7;
};
ConvShape conv_shape(int KH, int KW, int stride, int pad, int up, int H, int W) {
  const bool even = up == 1 && H % 2 == 0 && W % 2 == 0;
  return ConvShape{KH == 3 && KW == 3 && stride == 1 && pad == 1, KH == 1 && KW == 1 && stride == 1 && pad == 0 && up == 1,
                   KH == 4 && KW == 4 && stride == 2 && pad == 1 && even, KH == 2 && KW == 2 && stride == 2 && pad == 0 && even,
                   KH == 7 && KW == 7 && stride == 1 && pad == 3 && up == 1};
}
ConvGeom conv_geom(int B, int Cin, int H, int W, int Cout, int KH, int KW, int stride, int pad, int up) {
  return ConvGeom{B, H, W, Cin, up, KH, KW, stride, pad, (H * up + 2 * pad - KH) / stride + 1, (W * up + 2 * pad - KW) / stride + 1,
                  Cout};
}

// The three networks run every level on the image padded to a multiple of 2^levels: level i is (Hp >> i) x (Wp >> i).  The
// padded size is held in long long so that build_plan can check it against the kernels' limits for any int H, W.
struct Levels {
  long long Hp, Wp;
  int h(int i) const { return (int)(Hp >> i); }
  int w(int i) const { return (int)(Wp >> i); }
};
Levels level_sizes(long long H, long long W, int levels) {
  const long long s = 1LL << levels;
  return Levels{(H + s - 1) / s * s, (W + s - 1) / s * s};
}

// ---- plan builder ----------------------------------------------------------------------------------
template <typename T>
struct Builder {
  irsde_ctx* ctx;
  Plan* plan;
  bool ok = true;
  std::string err;
  std::multimap<size_t, void*> free_tmp;
  std::map<void*, size_t> tmp_size;

  T* alloc(long long elems) {
    void* p = dev_alloc(ctx, (size_t)elems * sizeof(T), &plan->allocs);
    if (!p) { ok = false; err = "cudaMalloc failed in plan builder"; }
    return (T*)p;
  }
  T* tmp(long long elems) {
    size_t bytes = (size_t)elems * sizeof(T);
    auto it = free_tmp.lower_bound(bytes);
    if (it != free_tmp.end() && it->first <= bytes * 2 + 4096) {
      void* p = it->second;
      free_tmp.erase(it);
      return (T*)p;
    }
    void* p = alloc(elems);
    tmp_size[p] = bytes;
    return (T*)p;
  }
  void release(void* p) { free_tmp.insert({tmp_size[p], p}); }

  float* fw(const std::string& n) {  // fp32 raw parameter (bias / gain vectors)
    auto it = ctx->raw.find(n);
    if (it == ctx->raw.end()) { ok = false; err = "missing tensor " + n; return nullptr; }
    return it->second.dev;
  }

  struct V { T* p; int pitch; int C; };  // channel-offset NHWC view
  static V view(T* base, int pitch, int off, int C) { return V{base + off, pitch, C}; }
  // appends an op to the plan; label and bytes are what IRSDE_PROFILE_DUMP and irsde_profile_end_bytes report
  void push_op(int cat, double flops, std::string label, double bytes, Op fn) {
    plan->ops.push_back(OpRec{cat, flops, std::move(fn), std::move(label), bytes});
  }
  void mark_out(V out, int H, int W) {  // the op just pushed writes this view (irsde_trace_forward)
    OpRec& r = plan->ops.back();
    r.out_p = out.p; r.out_pitch = out.pitch; r.out_C = out.C; r.out_H = H; r.out_W = W;
  }

  // One conv of a network.  Every conv here pads to keep the size at stride 1 and to halve it exactly at stride 2, so its
  // padding is (K - stride) / 2.
  struct ConvSpec {
    std::string w;              // weight name
    V in;
    int H = 0, W = 0;           // input size (before the nearest x2 upsample)
    int K = 0, stride = 1, up = 1;
    std::string bias;           // bias name, "" = none
    std::string ss;             // ResBlock / NAFBlock prefix whose (scale, shift) modulate the output, "" = none
    int silu = 0;
    std::string mult;           // per-output-channel multiplier name (NAFBlock beta / gamma), "" = none
    V res{};                    // residual added to the output (res.p == nullptr: none)
    V out{};                    // output view; out.C is Cout
    bool nchw = false;          // write fp32 NCHW to the run's output pointer instead of `out` (out.p null)
    int crop_h = 0, crop_w = 0;  // crop of the NCHW output, 0 = the image size
    bool stem_layout = false;   // `in` is the zero-bordered [B][Hp+6][Wp+8][8] layout of the tensor-core stem
    int tc_flags = 0;           // TC_FLAG_* epilogues of the tap-GEMM (bf16 only)
    const bf16* w_override = nullptr;  // tap-GEMM weights other than the packed `w` (per-image weights)
  };
  void conv(const ConvSpec& s) {
    const V in = s.in, out = s.out;
    const int K = s.K, stride = s.stride, up = s.up, Hin = s.H, Win = s.W, Cout = out.C, pad = (K - stride) / 2;
    const ConvGeom g = conv_geom(plan->B, in.C, Hin, Win, Cout, K, K, stride, pad, up);
    char b[160];
    snprintf(b, sizeof b, "%s %dx%d k%d s%d up%d Cin%d Cout%d", s.w.c_str(), Hin, Win, K, stride, up, in.C, Cout);
    const std::string label = b;
    const double esz = sizeof(T);
    const double bytes = (double)plan->B * Hin * Win * in.C * esz + (double)plan->B * g.Hout * g.Wout * Cout * (s.nchw ? 4.0 : esz) +
                         (double)K * K * in.C * Cout * esz + (s.res.p ? (double)plan->B * g.Hout * g.Wout * Cout * esz : 0.0);
    double simt_flops = 2.0 * plan->B * g.Hout * g.Wout * (double)Cout * in.C * K * K;
    // the tensor-core engine runs nearest-x2 + 3x3 as four 2x2 phase convolutions (4 taps per output pixel) and the 7x7 stem
    // as 7 row taps of 8 pixels x 8 channels
    double tc_flops = (K == 3 && up == 2) ? simt_flops * 4.0 / 9.0
                      : K == 7            ? 2.0 * plan->B * g.Hout * g.Wout * (double)Cout * 448
                                          : simt_flops;
    Epilogue ep;
    memset(&ep, 0, sizeof ep);
    ep.bias = s.bias.empty() ? nullptr : fw(s.bias);
    ep.mult_vec = s.mult.empty() ? nullptr : fw(s.mult);
    ep.silu = s.silu;
    ep.ss_S = ctx->S;
    const bool use_ss = !s.ss.empty();
    if (use_ss && ep.mult_vec) { ok = false; err = "time modulation and mult_vec cannot be combined: " + s.w; return; }
    ep.ss_off = use_ss ? ctx->ss_off[s.ss] : 0;
    if (s.res.p) { ep.res = s.res.p; ep.res_pitch = s.res.pitch; }
    const bool nchw = s.nchw;
    const int cH = s.crop_h ? s.crop_h : plan->H, cW = s.crop_w ? s.crop_w : plan->W;
    constexpr bool f32 = std::is_same<T, float>::value;  // fp32x3 engine: tf32 hi/lo split operands
    constexpr int al = f32 ? 4 : 8;                       // elements per 16 bytes
    const ConvShape cs = conv_shape(K, K, stride, pad, up, Hin, Win);
    const bool out_aligned = Cout % al == 0 && out.pitch % al == 0;
    const bool stem = !f32 && s.stem_layout && cs.k7 && out_aligned;
    const bool taps = (cs.k3 || cs.k1 || cs.k4 || cs.k2) && in.C % al == 0 && in.pitch % al == 0 &&
                      (nchw ? cs.k3 && up == 1 : out_aligned);
    // fused-attention flags and per-image weights are bf16-only epilogues
    const bool engine_on =
        f32 ? ctx->use_tc3 && !s.tc_flags && !s.w_override && (((uintptr_t)in.p) & 15) == 0 : ctx->use_tc;
    if (engine_on && (stem || taps)) {
      const T* wt;
      if constexpr (f32) wt = ctx->w_tc3[s.w];
      else wt = s.w_override ? s.w_override : ctx->w_tc[s.w];
      if (!wt) { ok = false; err = (f32 ? "unpacked fp32x3 weight " : "unpacked tc weight ") + s.w; return; }
      const TapTable t = tap_table(K, up);
      const int Ha = t.s2d() ? Hin / 2 : Hin, Wa = t.s2d() ? Win / 2 : Win;
      const T* a = in.p;
      int a_pitch = in.pitch;
      if (t.s2d()) {
        T* s2d = tmp((long long)plan->B * Hin * Win * in.C);
        int Bc = plan->B, Cc = in.C;
        push_op(CAT_MISC, 0.0, "", 0.0, [=](Plan*, cudaStream_t st) {
          launch_space_to_depth<T>(in.p, in.pitch, s2d, Bc, Hin, Win, Cc, st);
          return 1;
        });
        a = s2d; a_pitch = in.C;
        release(s2d);  // safe: stream order; the next tmp user runs after this conv
      }
      if constexpr (f32) {
        // operand split (hi, lo) of the conv input: [2][planes][B][Ha][Wa][C]
        const long long npix_a = (long long)t.planes * plan->B * Ha * Wa;
        float* split = tmp(2 * npix_a * in.C);
        int Cc = in.C;
        push_op(CAT_MISC, 0.0, s.w + " tf32 hi/lo split of the input", 3.0 * npix_a * in.C * 4.0, [=](Plan*, cudaStream_t st) {
          launch_split_tf32(a, a_pitch, split, npix_a, Cc, st);
          return 1;
        });
        a = split; a_pitch = in.C;
        release(split);  // safe: stream order, as for s2d
      }
      std::string terr;
      TcConvDesc* d = tc_conv_create(a, a_pitch, plan->B, Ha, Wa, in.C, t.planes, wt, Cout, t.ntaps, t.taps, t.nph, ep, out.p,
                                     out.pitch, g.Hout, g.Wout, &terr, s.tc_flags);
      if (!d) { ok = false; err = "tc_conv_create(" + s.w + "): " + terr; return; }
      plan->tc_descs.push_back(d);
      push_op(CAT_TC, tc_flops, label, bytes, [=](Plan* p, cudaStream_t st) {
        if (use_ss) tc_conv_set_runtime(d, p->cur.ss, p->cur.t_ptr, p->cur.ss_img_stride);
        if (nchw) tc_conv_set_out_nchw(d, p->cur.out, cH, cW);
        tc_conv_launch(d, st);
        return 1;
      });
    } else {
      if (s.tc_flags || s.w_override) { ok = false; err = "fused attention conv needs the tensor-core engine: " + s.w; return; }
      const float* w = ctx->w_simt[s.w];
      if (!w) { ok = false; err = "unpacked weight " + s.w; return; }
      push_op(CAT_SIMT, simt_flops, label, bytes, [=](Plan* p, cudaStream_t st) {
        Epilogue e = ep;
        if (use_ss) { e.ss = p->cur.ss; e.t_ptr = p->cur.t_ptr; e.ss_img_stride = p->cur.ss_img_stride; }
        launch_conv_simt<T>(g, in.p, in.pitch, w, e, out.p, out.pitch, nchw ? p->cur.out : nullptr, cH, cW, st);
        return 1;
      });
    }
    if (!nchw) mark_out(out, g.Hout, g.Wout);
  }

  void resblock(const std::string& pre, V in, int Cout, V out, int H, int W, bool time_mod = true) {
    long long npix = (long long)plan->B * H * W;
    T* h1 = tmp(npix * Cout);
    V vh1{h1, Cout, Cout};
    conv({.w = pre + "block1.proj.weight", .in = in, .H = H, .W = W, .K = 3, .ss = time_mod ? pre : "", .silu = 1, .out = vh1});
    V res = in;
    T* r = nullptr;
    if (in.C != Cout) {
      r = tmp(npix * Cout);
      res = V{r, Cout, Cout};
      conv({.w = pre + "res_conv.weight", .in = in, .H = H, .W = W, .K = 1, .out = res});
    }
    conv({.w = pre + "block2.proj.weight", .in = vh1, .H = H, .W = W, .K = 3, .silu = 1, .res = res, .out = out});
    release(h1);
    if (r) release(r);
  }

  // Residual(PreNorm(LinearAttention)) or Residual(PreNorm(Attention)); pre = "...2." / "mid_attn."
  void attention(const std::string& pre, V in, V out, int H, int W, bool full, float* la_partial, float* la_ctx) {
    int C = in.C, B = plan->B, N = H * W;
    long long npix = (long long)B * N;
    if constexpr (std::is_same<T, bf16>::value) {
      if (!full && ctx->use_tc && linattn_fused_ok(C, in.p, in.pitch, out.p, out.pitch)) {
        linattn_fused(pre, in, out, H, W, la_partial, la_ctx);
        return;
      }
    }
    T* xn = tmp(npix * C);
    float* g1 = fw(pre + "fn.norm.g");
    push_op(CAT_LN, 0.0, pre + "norm", 2.0 * npix * C * sizeof(T), [=](Plan*, cudaStream_t st) {
      launch_layernorm<T>(in.p, in.pitch, g1, nullptr, 0, xn, C, npix, C, st);
      return 1;
    });
    mark_out(V{xn, C, C}, H, W);
    T* qkv = tmp(npix * 384);
    if constexpr (std::is_same<T, bf16>::value) {
      if (!full && ctx->use_tc && C % 8 == 0) {
        // Fused LinearAttention: (1) the to_qkv GEMM epilogue applies softmax_d(q)*32^-.5 per head, (2) k,v -> ctx,
        // (3) ctx is folded into the to_out weights per image, (4) ONE per-image-weight 1x1 GEMM on q gives to_out's
        // output (module_util.py:163-178 with the two einsums + to_out conv re-associated), (5) LayerNorm + residual.
        conv({.w = pre + "fn.fn.to_qkv.weight", .in = V{xn, C, C}, .H = H, .W = W, .K = 1, .out = V{qkv, 384, 384},
              .tc_flags = TC_FLAG_QSOFTMAX});
        release(xn);
        if (!linattn_views_ok(qkv, 384, nullptr, 0, sizeof(T))) { ok = false; err = "linear attention: qkv view not 16-byte aligned"; }
        push_op(CAT_ATTN, 0.0, pre + "linattn kv->ctx (2 kernels)", (double)npix * 256 * sizeof(T), [=](Plan*, cudaStream_t st) {
          launch_linattn_ctx<T>(qkv, 384, la_partial, la_ctx, B, N, st);
          return 2;
        });
        bf16* Mb = tmp((long long)B * C * 128);
        float* wout = fw(pre + "fn.fn.to_out.0.weight");
        // (combine + fold in ONE kernel gives 8-64 blocks of latency-bound work instead of 32 + 256..4096: kept as two launches)
        push_op(CAT_ATTN, 0.0, pre + "fold ctx into to_out", 0.0, [=](Plan*, cudaStream_t st) {
          launch_la_fold(la_ctx, wout, Mb, B, C, st);
          return 1;
        });
        T* y = tmp(npix * C);
        conv({.w = pre + "fn.fn.to_out.0.weight", .in = V{qkv, 384, 128}, .H = H, .W = W, .K = 1, .bias = pre + "fn.fn.to_out.0.bias",
              .out = V{y, C, C}, .tc_flags = TC_FLAG_W_PER_IMAGE, .w_override = Mb});
        float* g2 = fw(pre + "fn.fn.to_out.1.g");
        push_op(CAT_LN, 0.0, pre + "to_out.norm+res", 3.0 * npix * C * sizeof(T), [=](Plan*, cudaStream_t st) {
          launch_layernorm<T>(y, C, g2, in.p, in.pitch, out.p, out.pitch, npix, C, st);
          return 1;
        });
        mark_out(out, H, W);
        release(y);
        release(Mb);
        release(qkv);
        return;
      }
    }
    conv({.w = pre + "fn.fn.to_qkv.weight", .in = V{xn, C, C}, .H = H, .W = W, .K = 1, .out = V{qkv, 384, 384}});
    release(xn);
    T* hid = tmp(npix * 128);
    if (full) {
      push_op(CAT_ATTN, 0.0, pre + "full attention", 0.0, [=](Plan*, cudaStream_t st) {
        launch_fullattn<T>(qkv, 384, hid, 128, B, N, st);
        return 1;
      });
      mark_out(V{hid, 128, 128}, H, W);
      conv({.w = pre + "fn.fn.to_out.weight", .in = V{hid, 128, 128}, .H = H, .W = W, .K = 1, .bias = pre + "fn.fn.to_out.bias",
            .res = in, .out = out});
    } else {
      if (!linattn_views_ok(qkv, 384, hid, 128, sizeof(T))) { ok = false; err = "linear attention: views not 16-byte aligned"; }
      push_op(CAT_ATTN, 0.0, pre + "linattn(3 kernels)", (double)npix * (384 + 128) * sizeof(T), [=](Plan*, cudaStream_t st) {
        launch_linattn<T>(qkv, 384, la_partial, la_ctx, hid, 128, B, N, st);
        return 3;
      });
      T* y = tmp(npix * C);
      conv({.w = pre + "fn.fn.to_out.0.weight", .in = V{hid, 128, 128}, .H = H, .W = W, .K = 1, .bias = pre + "fn.fn.to_out.0.bias",
            .out = V{y, C, C}});
      float* g2 = fw(pre + "fn.fn.to_out.1.g");
      push_op(CAT_LN, 0.0, pre + "to_out.norm+res", 3.0 * npix * C * sizeof(T), [=](Plan*, cudaStream_t st) {
        launch_layernorm<T>(y, C, g2, in.p, in.pitch, out.p, out.pitch, npix, C, st);
        return 1;
      });
      mark_out(out, H, W);
      release(y);
    }
    release(qkv);
    release(hid);
  }

  // Residual(PreNorm(LinearAttention)) for C = 64 / 128 (bf16): two fused passes over x (linattn_fused.cu) around the combine
  // and the fold, four launches instead of seven, and none of the xn, qkv and y tensors.  W_q and W_kv are rows 0..127 and
  // 128..383 of the packed to_qkv weight ([384][C], irsde_finalize_weights).
  void linattn_fused(const std::string& pre, V in, V out, int H, int W, float* la_partial, float* la_ctx) {
    const int C = in.C, B = plan->B, N = H * W;
    const long long npix = (long long)B * N;
    const bf16* wqkv = ctx->w_tc[pre + "fn.fn.to_qkv.weight"];
    if (!wqkv) { ok = false; err = "unpacked tc weight " + pre + "fn.fn.to_qkv.weight"; return; }
    float* g1 = fw(pre + "fn.norm.g");
    push_op(CAT_ATTN, 0.0, pre + "norm+to_qkv k,v+linattn kv (fused)", (double)npix * C * sizeof(T), [=](Plan*, cudaStream_t st) {
      launch_la_kv_ln(in.p, in.pitch, g1, wqkv + 128 * C, la_partial, B, N, C, nullptr, st);
      return 1;
    });
    push_op(CAT_ATTN, 0.0, pre + "linattn combine", 0.0, [=](Plan*, cudaStream_t st) {
      launch_la_combine(la_partial, la_ctx, B, N, st);
      return 1;
    });
    bf16* Mb = tmp((long long)B * C * 128);
    float* wout = fw(pre + "fn.fn.to_out.0.weight");
    push_op(CAT_ATTN, 0.0, pre + "fold ctx into to_out", 0.0, [=](Plan*, cudaStream_t st) {
      launch_la_fold(la_ctx, wout, Mb, B, C, st);
      return 1;
    });
    float* bout = fw(pre + "fn.fn.to_out.0.bias");
    float* g2 = fw(pre + "fn.fn.to_out.1.g");
    push_op(CAT_ATTN, 0.0, pre + "to_out.norm+res", 2.0 * npix * C * sizeof(T), [=](Plan*, cudaStream_t st) {
      launch_la_out_ln(in.p, in.pitch, g1, wqkv, Mb, bout, g2, out.p, out.pitch, B, N, C, st);
      return 1;
    });
    mark_out(out, H, W);
    release(Mb);
  }

  // ---- latent autoencoder UNet.encode / UNet.decode (UNet_arch.py:59-91) --------------------------------------
  // plan->ops = encode (image -> z, skips stay in the decoder's concat buffers), plan->ops_dec = decode (z -> image).
  void build_latent() {
    const LatCfg& L = ctx->lat;
    const int B = plan->B, depth = L.depth;
    const Levels lv = level_sizes(plan->H, plan->W, depth);
    plan->Hp = lv.h(0);
    plan->Wp = lv.w(0);
    plan->lat_h = lv.h(depth - 1); plan->lat_w = lv.w(depth - 1);
    float* la_partial = (float*)dev_alloc(ctx, linattn_partial_floats(B, plan->lat_h * plan->lat_w) * sizeof(float), &plan->allocs);
    float* la_ctx = (float*)dev_alloc(ctx, (size_t)B * 4096 * sizeof(float), &plan->allocs);
    if (!la_partial || !la_ctx) { ok = false; err = "cudaMalloc failed"; return; }
    const int C0 = L.in_ch, pitch0 = (C0 + 7) / 8 * 8;
    const long long np0 = (long long)B * plan->Hp * plan->Wp;
    T* X0 = alloc(np0 * pitch0);
    T* H0 = alloc(np0 * L.ch);  // h[0] = init_conv output, added back before final_conv
    int in_ch = L.in_ch, Hh = plan->H, Ww = plan->W, Hp = plan->Hp, Wp = plan->Wp;
    push_op(CAT_MISC, 0.0, "", 0.0, [=](Plan* p, cudaStream_t st) {
      launch_prep_input<T>(p->cur.x, nullptr, X0, B, in_ch, Hh, Ww, Hp, Wp, pitch0, 0, st);  // reflect pad, no condition
      return 1;
    });
    conv({.w = "init_conv.weight", .in = V{X0, pitch0, C0}, .H = Hp, .W = Wp, .K = 3, .out = V{H0, L.ch, L.ch}});
    V cur{H0, L.ch, L.ch};
    std::vector<T*> U1(depth), U2(depth);
    char nb[64];
    for (int i = 0; i < depth; ++i) {
      const int di = L.ch * L.mult[i], dout = L.ch * L.mult[i + 1], H = lv.h(i), W = lv.w(i);
      const long long npix = (long long)B * H * W;
      U1[i] = alloc(npix * (dout + di));
      U2[i] = alloc(npix * (dout + di));
      snprintf(nb, sizeof nb, "encoder.%d.", i);
      std::string pre = nb;
      V s2 = view(U2[i], dout + di, dout, di), s1 = view(U1[i], dout + di, dout, di);
      resblock(pre + "0.", cur, di, s2, H, W, false);
      if (i == depth - 1) {
        T* ta = tmp(npix * di);
        resblock(pre + "1.", s2, di, V{ta, di, di}, H, W, false);
        attention(pre + "2.", V{ta, di, di}, s1, H, W, false, la_partial, la_ctx);
        release(ta);
        T* xm = alloc(npix * dout);
        conv({.w = pre + "3.weight", .in = s1, .H = H, .W = W, .K = 3, .out = V{xm, dout, dout}});
        cur = V{xm, dout, dout};
      } else {
        resblock(pre + "1.", s2, di, s1, H, W, false);  // Identity attention: the skip is b2's output
        T* xn = alloc((long long)B * lv.h(i + 1) * lv.w(i + 1) * dout);
        conv({.w = pre + "3.weight", .in = s1, .H = H, .W = W, .K = 4, .stride = 2, .bias = pre + "3.bias", .out = V{xn, dout, dout}});
        cur = V{xn, dout, dout};
      }
    }
    // z = latent_conv(x): fp32 NCHW [B, embed, lat_h, lat_w] straight from the epilogue
    conv({.w = "latent_conv.weight", .in = cur, .H = plan->lat_h, .W = plan->lat_w, .K = 1, .out = V{nullptr, 0, L.embed},
          .nchw = true, .crop_h = plan->lat_h, .crop_w = plan->lat_w});
    // ----- decode half
    std::vector<OpRec> enc_ops;
    enc_ops.swap(plan->ops);
    const int mid = L.ch * L.mult[depth];
    const long long npl = (long long)B * plan->lat_h * plan->lat_w;
    const int zp = (L.embed + 7) / 8 * 8;
    T* Z = alloc(npl * zp);
    int embed = L.embed, lh = plan->lat_h, lw = plan->lat_w;
    push_op(CAT_MISC, 0.0, "", 0.0, [=](Plan* p, cudaStream_t st) {
      launch_nchw_to_nhwc<T>(p->cur.x, Z, B, embed, lh, lw, zp, st);
      return 1;
    });
    {
      const int i = depth - 1, di = L.ch * L.mult[i];
      conv({.w = "post_latent_conv.weight", .in = V{Z, zp, L.embed}, .H = lh, .W = lw, .K = 1, .out = view(U1[i], mid + di, 0, mid)});
    }
    for (int j = 0; j < depth; ++j) {
      const int i = depth - 1 - j, di = L.ch * L.mult[i], dout = L.ch * L.mult[i + 1], H = lv.h(i), W = lv.w(i);
      const long long npix = (long long)B * H * W;
      snprintf(nb, sizeof nb, "decoder.%d.", j);
      std::string pre = nb;
      resblock(pre + "0.", V{U1[i], dout + di, dout + di}, dout, view(U2[i], dout + di, 0, dout), H, W, false);
      T* tb = tmp(npix * dout);
      resblock(pre + "1.", V{U2[i], dout + di, dout + di}, dout, V{tb, dout, dout}, H, W, false);
      V xo{tb, dout, dout};
      T* tc = nullptr;
      if (i == depth - 1) {
        tc = tmp(npix * dout);
        attention(pre + "2.", V{tb, dout, dout}, V{tc, dout, dout}, H, W, false, la_partial, la_ctx);
        xo = V{tc, dout, dout};
      }
      if (i != 0) {
        const int dprev_total = L.ch * L.mult[i] + L.ch * L.mult[i - 1];  // concat width of level i-1: dout_{i-1} + di_{i-1}
        conv({.w = pre + "3.1.weight", .in = xo, .H = H, .W = W, .K = 3, .up = 2, .bias = pre + "3.1.bias",
              .out = view(U1[i - 1], dprev_total, 0, di)});
      } else {
        T* xf = tmp(np0 * L.ch);
        conv({.w = pre + "3.weight", .in = xo, .H = H, .W = W, .K = 3, .out = V{xf, L.ch, L.ch}});
        T* xs = tmp(np0 * L.ch);
        int chn = L.ch;
        push_op(CAT_MISC, 0.0, "", 0.0, [=](Plan*, cudaStream_t st) {
          launch_add<T>(xf, chn, H0, chn, xs, chn, np0, chn, st);   // x + h[0]
          return 1;
        });
        conv({.w = "final_conv.weight", .in = V{xs, L.ch, L.ch}, .H = Hp, .W = Wp, .K = 3, .bias = "final_conv.bias",
              .out = V{nullptr, 0, L.out_ch}, .nchw = true});
        release(xf);
        release(xs);
      }
      release(tb);
      if (tc) release(tc);
    }
    plan->ops_dec.swap(plan->ops);
    plan->ops.swap(enc_ops);
  }

  // ---- ConditionalNAFNet (DenoisingNAFNet_arch.py:87-188) -------------------------------------------------
  float* naf_partial = nullptr;
  float* naf_sca = nullptr;

  void ln_mod(const std::string& gname, const std::string& blk, int off_scale, int off_shift, V in, V out, int H, int W) {
    int C = in.C, B = plan->B;
    long long npix = (long long)B * H * W;
    float* g = fw(gname);
    int base = ctx->ss_off[blk], S = ctx->S, ppi = H * W;
    push_op(CAT_LN, 0.0, gname + " (LN+mod)", 2.0 * npix * C * sizeof(T), [=](Plan* p, cudaStream_t st) {
      LnMod m;
      m.ss = p->cur.ss; m.t_ptr = p->cur.t_ptr; m.S = S; m.off_scale = base + off_scale; m.off_shift = base + off_shift;
      m.img_stride = p->cur.ss_img_stride; m.pix_per_img = ppi;
      launch_layernorm<T>(in.p, in.pitch, g, nullptr, 0, out.p, out.pitch, npix, C, st, &m);
      return 1;
    });
  }

  void nafblock(const std::string& pre, V x, V out, int H, int W) {
    const int c = x.C, B = plan->B, N = H * W;
    const long long npix = (long long)B * N;
    T* t1 = tmp(npix * c);
    ln_mod(pre + "norm1.g", pre, c, 0, x, V{t1, c, c}, H, W);            // x * (scale_att + 1) + shift_att
    T* t2 = tmp(npix * 2 * c);
    conv({.w = pre + "conv1.weight", .in = V{t1, c, c}, .H = H, .W = W, .K = 1, .bias = pre + "conv1.bias", .out = V{t2, 2 * c, 2 * c}});
    release(t1);
    T* g = tmp(npix * c);
    {
      float* w2 = fw(pre + "conv2.weight"); float* bb2 = fw(pre + "conv2.bias");
      float* ws = fw(pre + "sca.1.weight"); float* bs = fw(pre + "sca.1.bias");
      float* partial = naf_partial; float* sca = naf_sca;
      const int nch = dwgate_chunks(H, W);
      push_op(CAT_MISC, 0.0, pre + "dw3x3+gate+sca", (double)npix * (2 * c + c + 2 * c) * sizeof(T), [=](Plan*, cudaStream_t st) {
        launch_dwgate<T>(t2, 2 * c, w2, bb2, g, c, partial, B, H, W, c, st);
        int nl = 0;
        launch_sca_scale<T>(partial, ws, bs, sca, g, c, B, c, nch, N, &nl, st);
        return 1 + nl;
      });
    }
    release(t2);
    T* y = tmp(npix * c);
    conv({.w = pre + "conv3.weight", .in = V{g, c, c}, .H = H, .W = W, .K = 1, .bias = pre + "conv3.bias", .mult = pre + "beta",
          .res = x, .out = V{y, c, c}});                                     // y = inp + conv3(.)*beta
    release(g);
    t1 = tmp(npix * c);
    ln_mod(pre + "norm2.g", pre, 3 * c, 2 * c, V{y, c, c}, V{t1, c, c}, H, W);  // * (scale_ffn+1) + shift_ffn
    t2 = tmp(npix * 2 * c);
    conv({.w = pre + "conv4.weight", .in = V{t1, c, c}, .H = H, .W = W, .K = 1, .bias = pre + "conv4.bias", .out = V{t2, 2 * c, 2 * c}});
    release(t1);
    g = tmp(npix * c);
    push_op(CAT_MISC, 0.0, pre + "simple_gate", 0.0, [=](Plan*, cudaStream_t st) {
      launch_simple_gate<T>(t2, 2 * c, g, c, npix, c, st);
      return 1;
    });
    release(t2);
    conv({.w = pre + "conv5.weight", .in = V{g, c, c}, .H = H, .W = W, .K = 1, .bias = pre + "conv5.bias", .mult = pre + "gamma",
          .res = V{y, c, c}, .out = out});                                   // out = y + conv5(.)*gamma
    release(g);
    release(y);
  }

  void build_naf() {
    const NafCfg& n = ctx->naf;
    const int B = plan->B, w = n.width, ic = n.img_channel;
    const Levels lv = level_sizes(plan->H, plan->W, n.n_enc);
    plan->Hp = lv.h(0);
    plan->Wp = lv.w(0);
    size_t pmax = 0, cmax = 0;
    for (int i = 0; i <= n.n_enc; ++i) {
      size_t cc = (size_t)w << i;
      pmax = std::max(pmax, (size_t)B * dwgate_chunks(lv.h(i), lv.w(i)) * cc);
      cmax = std::max(cmax, cc);
    }
    naf_partial = (float*)dev_alloc(ctx, pmax * sizeof(float), &plan->allocs);
    naf_sca = (float*)dev_alloc(ctx, (size_t)B * cmax * sizeof(float), &plan->allocs);
    if (!naf_partial || !naf_sca) { ok = false; err = "cudaMalloc failed"; return; }
    // conditional: intro reads cat(x - cond, cond); denoising-sde: x alone (DenoisingNAFNet_arch.py:103,147-150)
    const int cond = ctx->cfg.variant == IRSDE_NET_CONDITIONAL ? 1 : 0;
    const int C0 = cond ? 2 * ic : ic, pitch0 = (C0 + 7) / 8 * 8;
    const long long np0 = (long long)B * plan->Hp * plan->Wp;
    T* X0 = alloc(np0 * pitch0);
    int Hh = plan->H, Ww = plan->W, Hp = plan->Hp, Wp = plan->Wp;
    push_op(CAT_MISC, 0.0, "", 0.0, [=](Plan* p, cudaStream_t st) {
      launch_prep_input<T>(p->cur.x, p->cur.mu, X0, B, ic, Hh, Ww, Hp, Wp, pitch0, cond, st, 0, 0, 0, 0, 1);  // zero pad
      return 1;
    });
    T* xin = alloc(np0 * w);
    conv({.w = "intro.weight", .in = V{X0, pitch0, C0}, .H = Hp, .W = Wp, .K = 3, .bias = "intro.bias", .out = V{xin, w, w}});
    V cur{xin, w, w};
    std::vector<V> encs;
    char nb[64];
    for (int i = 0; i < n.n_enc; ++i) {
      const int c = w << i;
      const long long npix = (long long)B * lv.h(i) * lv.w(i);
      for (int j = 0; j < n.enc[i]; ++j) {
        T* o = alloc(npix * c);
        snprintf(nb, sizeof nb, "encoders.%d.%d.", i, j);
        nafblock(nb, cur, V{o, c, c}, lv.h(i), lv.w(i));
        cur = V{o, c, c};
      }
      encs.push_back(cur);
      T* d = alloc((long long)B * lv.h(i + 1) * lv.w(i + 1) * 2 * c);
      snprintf(nb, sizeof nb, "downs.%d.", i);
      conv({.w = std::string(nb) + "weight", .in = cur, .H = lv.h(i), .W = lv.w(i), .K = 2, .stride = 2,
            .bias = std::string(nb) + "bias", .out = V{d, 2 * c, 2 * c}});
      cur = V{d, 2 * c, 2 * c};
    }
    {
      const int c = w << n.n_enc;
      const long long npix = (long long)B * lv.h(n.n_enc) * lv.w(n.n_enc);
      for (int j = 0; j < n.middle; ++j) {
        T* o = alloc(npix * c);
        snprintf(nb, sizeof nb, "middle_blks.%d.", j);
        nafblock(nb, cur, V{o, c, c}, lv.h(n.n_enc), lv.w(n.n_enc));
        cur = V{o, c, c};
      }
    }
    for (int i = 0; i < n.n_dec; ++i) {
      const int l = n.n_enc - 1 - i;           // level after upsampling
      const int chan = w << (l + 1), q = chan / 2;
      const int hl = lv.h(l + 1), wl = lv.w(l + 1);
      const long long np_lo = (long long)B * hl * wl, np_hi = (long long)B * lv.h(l) * lv.w(l);
      T* u = tmp(np_lo * 2 * chan);
      snprintf(nb, sizeof nb, "ups.%d.0.weight", i);
      conv({.w = nb, .in = cur, .H = hl, .W = wl, .K = 1, .out = V{u, 2 * chan, 2 * chan}});
      T* v = alloc(np_hi * q);
      V skip = encs[l];
      push_op(CAT_MISC, 0.0, std::string(nb) + " pixel_shuffle+skip", 0.0, [=](Plan*, cudaStream_t st) {
        launch_pixel_shuffle_add<T>(u, 2 * chan, skip.p, skip.pitch, v, q, B, hl, wl, q, st);
        return 1;
      });
      release(u);
      cur = V{v, q, q};
      for (int j = 0; j < n.dec[i]; ++j) {
        T* o = alloc(np_hi * q);
        snprintf(nb, sizeof nb, "decoders.%d.%d.", i, j);
        nafblock(nb, cur, V{o, q, q}, lv.h(l), lv.w(l));
        cur = V{o, q, q};
      }
    }
    if (n.latent) {  // latent variant: ending(x + encs[0]) with encs[0] = intro output
      T* e = alloc(np0 * w);
      V a = cur;
      push_op(CAT_MISC, 0.0, "", 0.0, [=](Plan*, cudaStream_t st) {
        launch_add<T>(a.p, a.pitch, xin, w, e, w, np0, w, st);
        return 1;
      });
      cur = V{e, w, w};
    }
    conv({.w = "ending.weight", .in = cur, .H = Hp, .W = Wp, .K = 3, .bias = "ending.bias", .out = V{nullptr, 0, ic}, .nchw = true});
  }

  void build() {
    const irsde_config& c = ctx->cfg;
    int B = plan->B, nf = c.nf, depth = c.depth;
    const std::vector<int>& D = ctx->udim;
    const Levels lv = level_sizes(plan->H, plan->W, depth);
    plan->Hp = lv.h(0);
    plan->Wp = lv.w(0);
    bool cond = c.variant == IRSDE_NET_CONDITIONAL;
    int C0 = cond ? 2 * c.in_nc : c.in_nc;
    int pitch0 = (C0 + 7) / 8 * 8;
    long long np0 = (long long)B * plan->Hp * plan->Wp;
    // linear-attention scratch sized for the largest level
    float* la_partial = (float*)dev_alloc(ctx, linattn_partial_floats(B, plan->Hp * plan->Wp) * sizeof(float), &plan->allocs);
    float* la_ctx = (float*)dev_alloc(ctx, (size_t)B * 4096 * sizeof(float), &plan->allocs);
    if (!la_partial || !la_ctx) { ok = false; err = "cudaMalloc failed"; return; }

    int in_nc = c.in_nc, Hh = plan->H, Ww = plan->W, Hp = plan->Hp, Wp = plan->Wp;
    // X0 lives in the zero-bordered [B][Hp+6][Wp+8][8] layout of the tensor-core stem
    const bool sp = std::is_same<T, bf16>::value && ctx->use_tc && pitch0 == 8 && nf % 8 == 0;
    long long x0_elems = sp ? (long long)B * (Hp + 6) * (Wp + 8) * 8 + 64 : np0 * pitch0;
    T* X0 = alloc(x0_elems);
    if (X0 && sp) cudaMemset(X0, 0, (size_t)x0_elems * sizeof(T));  // borders stay zero forever
    T* F = alloc(np0 * 2 * nf);
    push_op(CAT_MISC, 0.0, "", 0.0, [=](Plan* p, cudaStream_t st) {
      if (sp) launch_prep_input<T>(p->cur.x, p->cur.mu, X0, B, in_nc, Hh, Ww, Hp, Wp, pitch0, cond ? 1 : 0, st, 3, 3, Wp + 8, Hp + 6);
      else launch_prep_input<T>(p->cur.x, p->cur.mu, X0, B, in_nc, Hh, Ww, Hp, Wp, pitch0, cond ? 1 : 0, st);
      return 1;
    });
    conv({.w = "init_conv.weight", .in = V{X0, pitch0, C0}, .H = Hp, .W = Wp, .K = 7, .out = view(F, 2 * nf, nf, nf),
          .stem_layout = sp});
    V cur = view(F, 2 * nf, nf, nf);
    std::vector<T*> U1(depth), U2(depth);
    char nb[64];
    for (int i = 0; i < depth; ++i) {
      int di = D[i], dout = D[i + 1], H = lv.h(i), W = lv.w(i);
      long long npix = (long long)B * H * W;
      U1[i] = alloc(npix * (dout + di));
      U2[i] = alloc(npix * (dout + di));
      snprintf(nb, sizeof nb, "downs.%d.", i);
      std::string pre = nb;
      V s2 = view(U2[i], dout + di, dout, di), s1 = view(U1[i], dout + di, dout, di);
      resblock(pre + "0.", cur, di, s2, H, W);
      T* ta = tmp(npix * di);
      resblock(pre + "1.", s2, di, V{ta, di, di}, H, W);
      attention(pre + "2.", V{ta, di, di}, s1, H, W, false, la_partial, la_ctx);
      release(ta);
      if (i != depth - 1) {
        T* xn = alloc((long long)B * lv.h(i + 1) * lv.w(i + 1) * dout);
        conv({.w = pre + "3.weight", .in = s1, .H = H, .W = W, .K = 4, .stride = 2, .bias = pre + "3.bias", .out = V{xn, dout, dout}});
        cur = V{xn, dout, dout};
      } else {
        T* xn = alloc(npix * dout);
        conv({.w = pre + "3.weight", .in = s1, .H = H, .W = W, .K = 3, .out = V{xn, dout, dout}});
        cur = V{xn, dout, dout};
      }
    }
    {
      int i = depth - 1, di = D[i], mid = D[depth], H = lv.h(i), W = lv.w(i);
      long long npix = (long long)B * H * W;
      T* m1 = tmp(npix * mid);
      T* m2 = tmp(npix * mid);
      resblock("mid_block1.", cur, mid, V{m1, mid, mid}, H, W);
      attention("mid_attn.", V{m1, mid, mid}, V{m2, mid, mid}, H, W, c.variant == IRSDE_NET_DENOISING, la_partial, la_ctx);
      resblock("mid_block2.", V{m2, mid, mid}, mid, view(U1[i], mid + di, 0, mid), H, W);
      release(m1);
      release(m2);
    }
    for (int j = 0; j < depth; ++j) {
      int i = depth - 1 - j, di = D[i], dout = D[i + 1], H = lv.h(i), W = lv.w(i);
      long long npix = (long long)B * H * W;
      snprintf(nb, sizeof nb, "ups.%d.", j);
      std::string pre = nb;
      resblock(pre + "0.", V{U1[i], dout + di, dout + di}, dout, view(U2[i], dout + di, 0, dout), H, W);
      T* tb = tmp(npix * dout);
      resblock(pre + "1.", V{U2[i], dout + di, dout + di}, dout, V{tb, dout, dout}, H, W);
      T* tc = tmp(npix * dout);
      attention(pre + "2.", V{tb, dout, dout}, V{tc, dout, dout}, H, W, false, la_partial, la_ctx);
      release(tb);
      if (i != 0) {
        int dprev = D[i];  // == dout of level i-1
        conv({.w = pre + "3.1.weight", .in = V{tc, dout, dout}, .H = H, .W = W, .K = 3, .up = 2, .bias = pre + "3.1.bias",
              .out = view(U1[i - 1], dprev + D[i - 1], 0, dprev)});
      } else {
        conv({.w = pre + "3.weight", .in = V{tc, dout, dout}, .H = H, .W = W, .K = 3, .out = view(F, 2 * nf, 0, nf)});
      }
      release(tc);
    }
    T* G = tmp(np0 * nf);
    resblock("final_res_block.", V{F, 2 * nf, 2 * nf}, nf, V{G, nf, nf}, Hp, Wp);
    conv({.w = "final_conv.weight", .in = V{G, nf, nf}, .H = Hp, .W = Wp, .K = 3, .bias = "final_conv.bias",
          .out = V{nullptr, 0, c.out_nc}, .nchw = true});
  }
};

void free_plan(irsde_ctx* ctx, Plan* p) {
  for (int m = 0; m < IRSDE_NUM_MODES; ++m)
    if (p->graph[m]) cudaGraphExecDestroy(p->graph[m]);
  for (auto* d : p->tc_descs) tc_conv_destroy(d);
  for (void* q : p->allocs) cudaFree(q);  // cudaFree waits for in-flight work that may still use the buffer
  ctx->dev_bytes -= p->bytes;
  ctx->plan_bytes -= p->bytes;
  delete p;
}

// The plan cache is bounded: every (B,H,W) plan owns its activation workspace, TMA descriptors and step graphs, so a
// loop over a dataset of variable-size images (test.py runs batch 1 at native size) would otherwise grow without limit.
// Least-recently-used plans are dropped while the cache holds more than IRSDE_PLAN_CACHE_MB (default 24576) or
// IRSDE_PLAN_CACHE_MAX (default 8) entries; `keep` is never evicted.
void evict_plans(irsde_ctx* ctx, Plan* keep, bool all) {
  static long long budget = -1, maxn = -1;
  if (budget < 0) {
    const char* e = getenv("IRSDE_PLAN_CACHE_MB");
    budget = (e && atoll(e) > 0 ? atoll(e) : 24576LL) << 20;
    e = getenv("IRSDE_PLAN_CACHE_MAX");
    maxn = e && atoll(e) > 0 ? atoll(e) : 8;
  }
  for (;;) {
    const bool over = all || ctx->plan_bytes > budget || (long long)ctx->plans.size() > maxn;
    if (!over) return;
    auto victim = ctx->plans.end();
    for (auto it = ctx->plans.begin(); it != ctx->plans.end(); ++it)
      if (it->second != keep && (victim == ctx->plans.end() || it->second->last_use < victim->second->last_use)) victim = it;
    if (victim == ctx->plans.end()) return;
    free_plan(ctx, victim->second);
    ctx->plans.erase(victim);
  }
}

int build_plan(irsde_ctx* ctx, int B, int H, int W, Plan** out) {
  auto key = std::make_tuple(B, H, W);
  auto it = ctx->plans.find(key);
  if (it != ctx->plans.end()) { it->second->last_use = ++ctx->use_clock; *out = it->second; return IRSDE_OK; }
  if (B <= 0 || H <= 0 || W <= 0) return fail(ctx, IRSDE_ERR_INVALID, "bad image shape");
  // the denoising UNet's mid_attn is full attention
  const Levels lv = level_sizes(H, W, ctx->lat.on ? ctx->lat.depth : ctx->naf.on ? ctx->naf.n_enc : ctx->cfg.depth);
  const bool full = !ctx->lat.on && !ctx->naf.on && ctx->cfg.variant == IRSDE_NET_DENOISING;
  if (int rc = check_shape_limits(ctx, full ? 4LL * B : B, full ? "4 B (full-attention grid rows)" : "B", lv.Hp, lv.Wp)) return rc;
  const long long bytes_before = ctx->dev_bytes;
  // reflect pad needs pad < size (F.pad 'reflect' raises otherwise, DenoisingUNet_arch.py:82)
  if (!ctx->naf.on && (lv.Hp - H >= H || lv.Wp - W >= W)) return fail(ctx, IRSDE_ERR_INVALID, "image too small for reflect padding");
  Plan* p = new Plan();
  p->B = B; p->H = H; p->W = W;
  std::string err;
  bool ok;
  if (ctx->cfg.precision != IRSDE_PREC_BF16) {
    Builder<float> b{ctx, p};
    if (ctx->lat.on) b.build_latent(); else if (ctx->naf.on) b.build_naf(); else b.build();
    ok = b.ok; err = b.err;
  } else {
    Builder<bf16> b{ctx, p};
    if (ctx->lat.on) b.build_latent(); else if (ctx->naf.on) b.build_naf(); else b.build();
    ok = b.ok; err = b.err;
  }
  long long n = (long long)B * ctx->cfg.in_nc * H * W;
  long long no = (long long)B * ctx->cfg.out_nc * H * W;
  p->x_state = (float*)dev_alloc(ctx, n * 4, &p->allocs);
  p->mu_buf = (float*)dev_alloc(ctx, n * 4, &p->allocs);
  p->eps_buf = (float*)dev_alloc(ctx, no * 4, &p->allocs);
  p->d_step = (StepState*)dev_alloc(ctx, sizeof(StepState), &p->allocs);
  p->d_zero = (int*)dev_alloc(ctx, sizeof(int), &p->allocs);
  int td = ctx->cfg.nf * 4;
  p->fwd_times = (float*)dev_alloc(ctx, (size_t)B * 4, &p->allocs);
  p->fwd_temb = (float*)dev_alloc(ctx, (size_t)B * td * 4, &p->allocs);
  p->fwd_table = (float*)dev_alloc(ctx, (size_t)B * ctx->S * 4, &p->allocs);
  if (ok && p->x_state && p->mu_buf && p->eps_buf && p->d_step && p->d_zero && p->fwd_table) {
    cudaMemset(p->d_zero, 0, sizeof(int));
    // The stem's zero border and d_zero are set on the legacy stream, which non-blocking streams do not wait for: the
    // plan is complete on the device before any of its work is enqueued, whatever stream runs it.
    cudaError_t se = cudaDeviceSynchronize();
    if (se != cudaSuccess) { ok = false; err = std::string("plan setup failed: ") + cudaGetErrorString(se); }
  }
  if (!ok || !p->x_state || !p->mu_buf || !p->eps_buf || !p->d_step || !p->d_zero || !p->fwd_table) {
    for (auto* d : p->tc_descs) tc_conv_destroy(d);
    for (void* q : p->allocs) cudaFree(q);
    ctx->dev_bytes = bytes_before;
    delete p;
    return fail(ctx, IRSDE_ERR_CUDA, err.empty() ? "plan allocation failed" : err);
  }
  p->bytes = ctx->dev_bytes - bytes_before;
  p->last_use = ++ctx->use_clock;
  ctx->plan_bytes += p->bytes;
  ctx->plans[key] = p;
  evict_plans(ctx, p, false);
  *out = p;
  return IRSDE_OK;
}

void run_ops(irsde_ctx* ctx, Plan* p, std::vector<OpRec>& ops, cudaStream_t st) {
  if (!ctx->prof) {
    for (auto& op : ops) ctx->launches += op.fn(p, st);
    return;
  }
  for (auto& op : ops) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    cudaEventRecord(e0, st);
    ctx->launches += op.fn(p, st);
    cudaEventRecord(e1, st);
    ctx->prof_events.push_back({op.cat, op.flops, e0, e1, &op});
  }
}
void run_forward(irsde_ctx* ctx, Plan* p, cudaStream_t st) { run_ops(ctx, p, p->ops, st); }

// default per-timestep scalars in fp32, same op order as the reference's 0-dim tensor math
void fill_default_coeffs(irsde_ctx* c, int mode, std::vector<float>& tab) {
  int T = c->T;
  tab.assign((size_t)(T + 1) * IRSDE_NUM_COEF, 0.f);
  float dt = c->dt, sqdt = (float)sqrt((double)dt);
  for (int t = 1; t <= T; ++t) {
    float* r = &tab[(size_t)t * IRSDE_NUM_COEF];
    float th = c->thetas[t], sg = c->sigmas[t], cs = c->cumsum[t], cs1 = c->cumsum[t - 1], sb = c->sbars[t];
    float sg2 = sg * sg;
    switch (mode) {
      case IRSDE_MODE_SDE: r[0] = th; r[1] = sg2; r[2] = sb; r[3] = dt; r[4] = sg; r[5] = sqdt; break;
      case IRSDE_MODE_ODE: r[0] = th; r[1] = 0.5f * sg2; r[2] = sb; r[3] = dt; break;
      case IRSDE_MODE_POSTERIOR: {
        float A0 = expf(cs * dt);
        float A = expf(-th * dt), Bv = expf(-cs * dt), Cv = expf(-cs1 * dt);
        float term1 = A * (1.f - Cv * Cv) / (1.f - Bv * Bv);
        float term2 = Cv * (1.f - A * A) / (1.f - Bv * Bv);
        float A2 = expf(-2.f * th * dt), B2 = expf(-2.f * cs * dt), C2 = expf(-2.f * cs1 * dt);
        float var = (1.f - A2) * (1.f - C2) / (1.f - B2);
        float mn = 1e-20f * dt;
        float lv = logf(var < mn ? mn : var);
        float sd = expf(0.5f * lv) * c->max_sigma;
        r[0] = A0; r[1] = sb; r[2] = term1; r[3] = term2; r[4] = sd;
        break;
      }
      case IRSDE_MODE_DSDE_SDE: {
        float A = expf(-2.f * cs * dt);
        r[0] = -0.5f * sg2 * (1.f + A); r[1] = sb; r[2] = dt; r[3] = sg; r[4] = sqdt;
        break;
      }
      default: {
        float A = expf(-2.f * cs * dt);
        r[0] = -0.5f * sg2 * A; r[1] = sb; r[2] = dt;
        break;
      }
    }
  }
}

int upload_coeffs(irsde_ctx* ctx, int mode, const float* tab, int T) {
  size_t bytes = (size_t)(T + 1) * IRSDE_NUM_COEF * sizeof(float);
  if (ctx->coef_dev[mode]) {
    // keep pointer stable across re-uploads of the same T (captured graphs reference it)
  } else {
    ctx->coef_dev[mode] = (float*)dev_alloc(ctx, (size_t)(4096 + 1) * IRSDE_NUM_COEF * sizeof(float), &ctx->allocs);
    if (!ctx->coef_dev[mode]) return fail(ctx, IRSDE_ERR_CUDA, "cudaMalloc coef failed");
  }
  if (T > 4096) return fail(ctx, IRSDE_ERR_UNSUPPORTED, "T > 4096 not supported");
  CUDA_TRY(ctx, cudaDeviceSynchronize());  // chains in flight on non-blocking streams still read the old table
  CUDA_TRY(ctx, cudaMemcpy(ctx->coef_dev[mode], tab, bytes, cudaMemcpyHostToDevice));
  // a pageable copy returns once staged; its DMA runs on the legacy stream, which later chains do not wait for
  CUDA_TRY(ctx, cudaDeviceSynchronize());
  return IRSDE_OK;
}

// times[rows] -> table[rows][S] for either network family
void time_rows(irsde_ctx* ctx, const float* times, int rows, float* temb_ws, float* table, cudaStream_t st) {
  if (ctx->naf.on) {
    launch_naf_time_gate(times, rows, ctx->naf.width, ctx->raw["time_mlp.1.weight"].dev, ctx->raw["time_mlp.1.bias"].dev,
                         ctx->raw["time_mlp.3.weight"].dev, ctx->raw["time_mlp.3.bias"].dev, temb_ws, st);
    launch_time_rows(temb_ws, rows, 2 * ctx->naf.width, ctx->wall, ctx->ball, ctx->S, table, st);
  } else {
    launch_time_table(times, rows, ctx->cfg.nf, ctx->raw["time_mlp.1.weight"].dev, ctx->raw["time_mlp.1.bias"].dev,
                      ctx->raw["time_mlp.3.weight"].dev, ctx->raw["time_mlp.3.bias"].dev, ctx->wall, ctx->ball, ctx->S, temb_ws,
                      table, st);
  }
  ctx->launches += 2;
}

int ensure_chain_table(irsde_ctx* ctx, Plan* p, int T, cudaStream_t st) {
  int rows = T + 1;
  if (rows > p->chain_cap) {
    int cap = rows < 128 ? 128 : rows;
    int td = ctx->cfg.nf * 4;
    p->chain_times = (float*)dev_alloc(ctx, (size_t)cap * 4, &p->allocs);
    p->chain_temb = (float*)dev_alloc(ctx, (size_t)cap * td * 4, &p->allocs);
    p->chain_table = (float*)dev_alloc(ctx, (size_t)cap * ctx->S * 4, &p->allocs);
    if (!p->chain_times || !p->chain_temb || !p->chain_table) return fail(ctx, IRSDE_ERR_CUDA, "cudaMalloc chain table failed");
    { const long long add = ((long long)cap * 4 + (long long)cap * td * 4 + (long long)cap * ctx->S * 4); p->bytes += add; ctx->plan_bytes += add; }
    std::vector<float> tv(cap);
    for (int i = 0; i < cap; ++i) tv[i] = (float)i;
    // pageable source: staged before the call returns, copied in the caller's stream order ahead of time_rows below
    CUDA_TRY(ctx, cudaMemcpyAsync(p->chain_times, tv.data(), (size_t)cap * 4, cudaMemcpyHostToDevice, st));
    p->chain_cap = cap;
    for (int m = 0; m < IRSDE_NUM_MODES; ++m)
      if (p->graph[m]) { cudaGraphExecDestroy(p->graph[m]); p->graph[m] = nullptr; }
  }
  time_rows(ctx, p->chain_times, rows, p->chain_temb, p->chain_table, st);
  return IRSDE_OK;
}

// ---- the standalone entries' scratch and conv body (irsde_conv2d_ex ... irsde_prep_input) ---------------------------------
__global__ void cast_f32_bf16_kernel(const float* __restrict__ in, bf16* __restrict__ out, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = __float2bfloat16_rn(in[i]);
}
__global__ void cast_bf16_f32_kernel(const bf16* __restrict__ in, float* __restrict__ out, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = __bfloat162float(in[i]);
}

// The device scratch of one standalone entry call.  The bf16 paths run on bf16 copies of the caller's fp32 buffers: a
// staged buffer is converted whole, the kernels work on views into the copy, and finish() converts the outputs back.
// Memory comes from dev_alloc (counted in the context's bytes, for the entries that take a context), and every launch goes
// to the entry's stream.  Nothing is freed before that stream has drained: finish() waits for it, and so
// does the destructor when an early return skipped finish().
class Scratch {
 public:
  irsde_ctx* const ctx;
  const cudaStream_t st;

  Scratch(irsde_ctx* c, cudaStream_t s) : ctx(c), st(s) {}
  ~Scratch() {
    if (!bufs_.empty()) release();
  }
  template <typename T>
  T* alloc(long long n) {
    return (T*)dev_alloc(ctx, n * sizeof(T), &bufs_);
  }
  // bf16 copies of the caller's buffers: of one the call reads, of one it only writes (converted back by finish()), and of
  // one it updates or writes a view of (both)
  const bf16* in(const float* src, long long n) { return stage(src, nullptr, n); }
  bf16* out(float* dst, long long n) { return stage(nullptr, dst, n); }
  bf16* inout(float* buf, long long n) { return stage(buf, buf, n); }
  // a device copy of v (the time-table row of a modulated epilogue)
  const int* upload(int v) {
    int* p = alloc<int>(1);
    if (p) cudaMemcpyAsync(p, &v, sizeof v, cudaMemcpyHostToDevice, st);
    return p;
  }
  int oom() const { return fail(ctx, IRSDE_ERR_CUDA, "cudaMalloc failed"); }
  // With rc == IRSDE_OK, converts the staged outputs back.  Then waits for the stream, turns a launch error into
  // IRSDE_ERR_CUDA ("what: <CUDA error>") and frees the scratch.
  int finish(int rc, const char* what) {
    if (!rc)
      for (const Back& b : back_) cast_bf16_f32_kernel<<<blocks(b.n), 256, 0, st>>>(b.src, b.dst, b.n);
    const cudaError_t ce = release();
    if (!rc && ce != cudaSuccess) rc = fail(ctx, IRSDE_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(ce));
    return rc;
  }

 private:
  struct Back { const bf16* src; float* dst; long long n; };
  std::vector<void*> bufs_;
  std::vector<Back> back_;
  static unsigned blocks(long long n) { return (unsigned)std::min<long long>((n + 255) / 256, 65536); }
  bf16* stage(const float* from, float* to, long long n) {
    bf16* b = alloc<bf16>(n);
    if (!b) return nullptr;
    if (from) cast_f32_bf16_kernel<<<blocks(n), 256, 0, st>>>(from, b, n);
    if (to) back_.push_back({b, to, n});
    return b;
  }
  cudaError_t release() {
    cudaError_t ce = cudaStreamSynchronize(st);
    if (ce == cudaSuccess) ce = cudaGetLastError();
    for (void* p : bufs_) cudaFree(p);
    bufs_.clear();
    back_.clear();
    return ce;
  }
};

// A channel view [off, off + width) of rows `pitch` elements apart; off and pitch also multiples of `align`.
bool view_ok(int pitch, int off, long long width, int align = 1) {
  return off >= 0 && off + width <= pitch && off % align == 0 && pitch % align == 0;
}

// An entry's info[4]: the caller's, or `local` when it passes none; zeroed.
int32_t* zeroed_info(int32_t* info, int32_t* local) {
  if (!info) info = local;
  info[0] = info[1] = info[2] = info[3] = 0;
  return info;
}

// Runs the conv the plan builder would make of this shape on the tap-GEMM (S = bf16, or fp32 for the fp32x3 engine), with
// the operands of run_conv.  As in a plan, the time table of `ep` (ss, t_ptr, ss_img_stride) is attached after the
// descriptor is created.
template <typename S>
int run_tc_conv(Scratch& sc, const ConvGeom& g, const S* in, int in_pitch, const S* w, const Epilogue& ep, S* out, int out_pitch,
                float* out_nchw, int crop_h, int crop_w, int flags, int32_t* info) {
  constexpr bool f32 = std::is_same<S, float>::value;
  const TapTable t = tap_table(g.KH, g.up);
  const int Ha = t.s2d() ? g.Hin / 2 : g.Hin, Wa = t.s2d() ? g.Win / 2 : g.Win;
  const long long npix = (long long)g.B * g.Hin * g.Win;  // A pixels, also after the space-to-depth pass (4 planes of Ha x Wa)
  S* s2d = t.s2d() ? sc.alloc<S>(npix * g.Cin) : nullptr;
  float* split = f32 ? sc.alloc<float>(2 * npix * g.Cin) : nullptr;
  if ((t.s2d() && !s2d) || (f32 && !split)) return sc.oom();
  if (s2d) {
    launch_space_to_depth<S>(in, in_pitch, s2d, g.B, g.Hin, g.Win, g.Cin, sc.st);
    in = s2d;
    in_pitch = g.Cin;
  }
  if constexpr (f32) {
    launch_split_tf32(in, in_pitch, split, npix, g.Cin, sc.st);
    in = split;
    in_pitch = g.Cin;
  }
  Epilogue e0 = ep;
  e0.ss = nullptr; e0.t_ptr = nullptr; e0.ss_img_stride = 0;
  std::string terr;
  TcConvDesc* d = tc_conv_create(in, in_pitch, g.B, Ha, Wa, g.Cin, t.planes, w, g.Cout, t.ntaps, t.taps, t.nph, e0, out, out_pitch,
                                 g.Hout, g.Wout, &terr, flags);
  if (!d) return fail(sc.ctx, IRSDE_ERR_INVALID, "tc_conv_create: " + terr);
  if (ep.ss) tc_conv_set_runtime(d, ep.ss, ep.t_ptr, ep.ss_img_stride);
  if (!out) tc_conv_set_out_nchw(d, out_nchw, crop_h, crop_w);
  if (info) tc_conv_query(d, info);
  tc_conv_launch(d, sc.st);
  tc_conv_destroy(d);
  return IRSDE_OK;
}

// One conv outside a plan in storage type S: packs w into the scratch in layout wl and runs it, on the SIMT kernel for
// WL_SIMT (fp32 weights, as in a plan) and on the tap-GEMM otherwise.  in and ep.res are NHWC views in S (the stem's
// padded layout for K = 7).  The output is the NHWC view (out, out_pitch), or with out == nullptr fp32 NCHW at out_nchw
// cropped to crop_h x crop_w.  flags are the tap-GEMM's TC_FLAG_*; info (may be null) receives the SIMT kernel's
// conv_simt_path or the tap-GEMM's tc_conv_query.
template <typename S>
int run_conv(Scratch& sc, const ConvGeom& g, const S* in, int in_pitch, WLayout wl, const float* w, const Epilogue& ep, S* out,
             int out_pitch, float* out_nchw, int crop_h, int crop_w, int flags, int32_t* info) {
  if (wl == WL_SIMT) {
    float* wp = sc.alloc<float>(packed_weight_elems<float>(wl, g.Cout, g.Cin, g.KH, g.KW));
    if (!wp) return sc.oom();
    pack_weight<float>(wl, w, wp, g.Cout, g.Cin, g.KH, g.KW, g.B, sc.st);
    if (info) conv_simt_path<S>(g, in, in_pitch, wp, out, out_pitch, info);
    launch_conv_simt<S>(g, in, in_pitch, wp, ep, out, out_pitch, out_nchw, crop_h, crop_w, sc.st);
    return IRSDE_OK;
  }
  S* wp = sc.alloc<S>(packed_weight_elems<S>(wl, g.Cout, g.Cin, g.KH, g.KW, g.B));
  if (!wp) return sc.oom();
  pack_weight<S>(wl, w, wp, g.Cout, g.Cin, g.KH, g.KW, g.B, sc.st);
  return run_tc_conv<S>(sc, g, in, in_pitch, wp, ep, out, out_pitch, out_nchw, crop_h, crop_w, flags, info);
}

}  // namespace

// =====================================================================================================
// C ABI
// =====================================================================================================
extern "C" {

const char* irsde_version(void) { return "irsde_b200 0.1 sm_90a"; }

const char* irsde_last_error(const irsde_ctx* ctx) { return ctx ? ctx->err.c_str() : g_last_error.c_str(); }

int irsde_create(const irsde_config* cfg, irsde_ctx** out) {
  if (!cfg || !out) return fail(nullptr, IRSDE_ERR_INVALID, "null argument");
  if (cfg->nf < 4 || cfg->nf % 2 || cfg->depth < 1 || cfg->depth > 6 || cfg->in_nc < 1 || cfg->out_nc < 1)
    return fail(nullptr, IRSDE_ERR_INVALID, "bad network configuration");
  if (cfg->variant != IRSDE_NET_CONDITIONAL && cfg->variant != IRSDE_NET_DENOISING)
    return fail(nullptr, IRSDE_ERR_INVALID, "bad variant");
  if (time_mlp_smem(cfg->nf) > kTimeMlpSmemMax)
    return fail(nullptr, IRSDE_ERR_UNSUPPORTED, "nf > 2457: the time MLP needs more than 48 KB of shared memory");
  if (cfg->precision != IRSDE_PREC_FP32 && cfg->precision != IRSDE_PREC_BF16 && cfg->precision != IRSDE_PREC_FP32X3)
    return fail(nullptr, IRSDE_ERR_INVALID, "bad precision");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) return fail(nullptr, IRSDE_ERR_CUDA, "no CUDA device available (this library has no CPU path)");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, IRSDE_ERR_INVALID, "bad device ordinal");
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, cfg->device);
  if (prop.major != 9 || prop.minor != 0)
    return fail(nullptr, IRSDE_ERR_UNSUPPORTED, "irsde_b200 is built for sm_90a (H100) only");
  irsde_ctx* c = new irsde_ctx();
  c->cfg = *cfg;
  if (cudaSetDevice(cfg->device) != cudaSuccess) { delete c; return fail(nullptr, IRSDE_ERR_CUDA, "cudaSetDevice failed"); }
  std::string terr;
  c->tc_ok = tc_init(&terr);
  if (cfg->precision != IRSDE_PREC_FP32 && !c->tc_ok) {
    delete c;
    return fail(nullptr, IRSDE_ERR_CUDA, "tensor-core engine init failed: " + terr);
  }
  c->use_tc = cfg->precision == IRSDE_PREC_BF16 && !(cfg->flags & IRSDE_FLAG_FORCE_SIMT);
  c->use_tc3 = cfg->precision == IRSDE_PREC_FP32X3 && !(cfg->flags & IRSDE_FLAG_FORCE_SIMT);
  for (int i = 0; i <= cfg->depth; ++i) c->udim.push_back(cfg->nf * (1 << i));
  *out = c;
  return IRSDE_OK;
}

int irsde_create_ch_mult(const irsde_config* cfg, const int32_t* ch_mult, int32_t n_levels, irsde_ctx** out) {
  if (!cfg || !ch_mult || !out || n_levels < 1 || n_levels > 6) return fail(nullptr, IRSDE_ERR_INVALID, "bad ch_mult");
  for (int i = 0; i < n_levels; ++i)
    if (ch_mult[i] < 1 || (long long)ch_mult[i] * cfg->nf > 65536) return fail(nullptr, IRSDE_ERR_INVALID, "bad ch_mult entry");
  irsde_config c2 = *cfg;
  c2.depth = n_levels;
  int rc = irsde_create(&c2, out);
  if (rc) return rc;
  (*out)->udim.assign(1, cfg->nf);
  for (int i = 0; i < n_levels; ++i) (*out)->udim.push_back(cfg->nf * ch_mult[i]);
  return IRSDE_OK;
}

int irsde_create_latent_unet(const irsde_latent_unet_config* lcfg, irsde_ctx** out) {
  if (!lcfg || !out) return fail(nullptr, IRSDE_ERR_INVALID, "null argument");
  if (lcfg->ch < 1 || lcfg->in_ch < 1 || lcfg->out_ch < 1 || lcfg->n_levels < 1 || lcfg->n_levels > 8 || lcfg->embed_dim < 1)
    return fail(nullptr, IRSDE_ERR_INVALID, "bad latent UNet configuration");
  irsde_config cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.in_nc = lcfg->in_ch; cfg.out_nc = lcfg->out_ch; cfg.nf = 8; cfg.depth = lcfg->n_levels;
  cfg.variant = IRSDE_NET_CONDITIONAL; cfg.precision = lcfg->precision; cfg.device = lcfg->device; cfg.flags = lcfg->flags;
  int rc = irsde_create(&cfg, out);
  if (rc) return rc;
  irsde_ctx* c = *out;
  c->lat.on = true;
  c->lat.in_ch = lcfg->in_ch; c->lat.out_ch = lcfg->out_ch; c->lat.ch = lcfg->ch; c->lat.depth = lcfg->n_levels;
  c->lat.embed = lcfg->embed_dim;
  c->lat.mult[0] = 1;
  for (int i = 0; i < lcfg->n_levels; ++i) c->lat.mult[i + 1] = lcfg->ch_mult[i];
  return IRSDE_OK;
}

static int latent_run(irsde_ctx* ctx, bool decode, const float* in, float* out, int32_t B, int32_t H, int32_t W, void* stream) {
  if (!ctx || !in || !out) return fail(ctx, IRSDE_ERR_INVALID, "null argument");
  if (!ctx->lat.on) return fail(ctx, IRSDE_ERR_STATE, "not a latent UNet context");
  if (!ctx->finalized) return fail(ctx, IRSDE_ERR_STATE, "weights not finalized");
  cudaSetDevice(ctx->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  StreamOrder order(ctx, st);
  Plan* p;
  auto key = std::make_tuple(B, H, W);
  bool existed = ctx->plans.find(key) != ctx->plans.end();
  if (decode && !existed) return fail(ctx, IRSDE_ERR_STATE, "decode needs a preceding encode of the same shape (skip features)");
  int rc = build_plan(ctx, B, H, W, &p);
  if (rc) return rc;
  p->cur.x = in; p->cur.mu = nullptr; p->cur.out = out;
  p->cur.ss = nullptr; p->cur.t_ptr = p->d_zero; p->cur.ss_img_stride = 0;
  run_ops(ctx, p, decode ? p->ops_dec : p->ops, st);
  CUDA_TRY(ctx, cudaGetLastError());
  return IRSDE_OK;
}

int irsde_latent_encode(irsde_ctx* ctx, const float* x, float* z, int32_t B, int32_t H, int32_t W, void* stream) {
  return latent_run(ctx, false, x, z, B, H, W, stream);
}
int irsde_latent_decode(irsde_ctx* ctx, const float* z, float* out, int32_t B, int32_t H, int32_t W, void* stream) {
  return latent_run(ctx, true, z, out, B, H, W, stream);
}
int irsde_latent_shape(irsde_ctx* ctx, int32_t H, int32_t W, int32_t* lat_h, int32_t* lat_w) {
  if (!ctx || !ctx->lat.on || !lat_h || !lat_w) return fail(ctx, IRSDE_ERR_INVALID, "bad argument");
  const Levels lv = level_sizes(H, W, ctx->lat.depth);
  *lat_h = lv.h(ctx->lat.depth - 1);
  *lat_w = lv.w(ctx->lat.depth - 1);
  return IRSDE_OK;
}

int irsde_create_nafnet(const irsde_nafnet_config* ncfg, irsde_ctx** out) {
  return irsde_create_nafnet_variant(ncfg, IRSDE_NET_CONDITIONAL, out);
}

int irsde_create_nafnet_variant(const irsde_nafnet_config* ncfg, int32_t variant, irsde_ctx** out) {
  if (!ncfg || !out) return fail(nullptr, IRSDE_ERR_INVALID, "null argument");
  if (variant != IRSDE_NET_CONDITIONAL && variant != IRSDE_NET_DENOISING) return fail(nullptr, IRSDE_ERR_INVALID, "bad variant");
  if (variant == IRSDE_NET_DENOISING && ncfg->latent)
    return fail(nullptr, IRSDE_ERR_INVALID, "the latent NAFNet has no denoising variant");
  if (ncfg->width < 4 || ncfg->width % 2 || ncfg->img_channel < 1 || ncfg->n_levels < 0 || ncfg->n_levels > 8 ||
      ncfg->middle_blk_num < 0)
    return fail(nullptr, IRSDE_ERR_INVALID, "bad NAFNet configuration");
  if (naf_time_mlp_smem(ncfg->width) > kTimeMlpSmemMax)
    return fail(nullptr, IRSDE_ERR_UNSUPPORTED, "width > 945: the time MLP needs more than 48 KB of shared memory");
  if (((long long)ncfg->width << ncfg->n_levels) > kScaMaxC)
    return fail(nullptr, IRSDE_ERR_UNSUPPORTED, "width << n_levels > 12288: the SCA mat-vec needs more than 48 KB of shared memory");
  irsde_config cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.in_nc = cfg.out_nc = ncfg->img_channel;
  cfg.nf = ncfg->width;
  cfg.depth = ncfg->n_levels > 0 ? ncfg->n_levels : 1;
  // the entry points that take mu (noise_fn, reverse, trace_forward) check it against this variant
  cfg.variant = variant;
  cfg.precision = ncfg->precision;
  cfg.device = ncfg->device;
  cfg.flags = ncfg->flags;
  int rc = irsde_create(&cfg, out);
  if (rc) return rc;
  irsde_ctx* c = *out;
  c->cfg.depth = ncfg->n_levels;
  c->naf.on = true;
  c->naf.img_channel = ncfg->img_channel;
  c->naf.width = ncfg->width;
  c->naf.middle = ncfg->middle_blk_num;
  c->naf.n_enc = c->naf.n_dec = ncfg->n_levels;
  for (int i = 0; i < ncfg->n_levels; ++i) { c->naf.enc[i] = ncfg->enc_blk_nums[i]; c->naf.dec[i] = ncfg->dec_blk_nums[i]; }
  c->naf.latent = ncfg->latent != 0;
  return IRSDE_OK;
}

// ---- NCCL behind the C ABI (SURVEY 8 b): dlopen()ed on first use so that single-GPU users keep a library without
// an NCCL dependency.  Only the two collectives of the path: one weight broadcast, one gather of x0. ----------------
struct NcclId { char internal[128]; };  // ncclUniqueId (NCCL_UNIQUE_ID_BYTES = 128), passed by value like the original
namespace {
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, NcclId, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*Broadcast)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
}  // namespace
namespace {
NcclApi g_nccl;
const int kNcclFloat = 7;  // ncclFloat32
bool nccl_load(std::string* err) {
  if (g_nccl.lib) return true;
  const char* names[] = {getenv("IRSDE_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
  void* h = nullptr;
  for (const char* n : names)
    if (n && n[0] && (h = dlopen(n, RTLD_NOW | RTLD_GLOBAL))) break;
  if (!h) { *err = "libnccl.so.2 not found (set IRSDE_NCCL_LIB)"; return false; }
  NcclApi a;
  a.lib = h;
  a.GetUniqueId = (int (*)(void*))dlsym(h, "ncclGetUniqueId");
  a.CommInitRank = (int (*)(void**, int, NcclId, int))dlsym(h, "ncclCommInitRank");
  a.CommDestroy = (int (*)(void*))dlsym(h, "ncclCommDestroy");
  a.Broadcast = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(h, "ncclBroadcast");
  a.GroupStart = (int (*)())dlsym(h, "ncclGroupStart");
  a.GroupEnd = (int (*)())dlsym(h, "ncclGroupEnd");
  a.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
  if (!a.GetUniqueId || !a.CommInitRank || !a.CommDestroy || !a.Broadcast || !a.GroupStart || !a.GroupEnd) { *err = "incomplete NCCL library"; return false; }
  g_nccl = a;
  return true;
}
int nccl_fail(irsde_ctx* ctx, const char* what, int rc) {
  return fail(ctx, IRSDE_ERR_CUDA, std::string(what) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "NCCL error"));
}
}  // namespace

int irsde_comm_unique_id(void* id128) {
  std::string err;
  if (!id128) return fail(nullptr, IRSDE_ERR_INVALID, "null id buffer");
  if (!nccl_load(&err)) return fail(nullptr, IRSDE_ERR_UNSUPPORTED, err);
  int rc = g_nccl.GetUniqueId(id128);
  return rc ? nccl_fail(nullptr, "ncclGetUniqueId", rc) : IRSDE_OK;
}

int irsde_comm_init(irsde_ctx* ctx, const void* id128, int32_t rank, int32_t nranks) {
  if (!ctx || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return fail(ctx, IRSDE_ERR_INVALID, "bad argument");
  if (ctx->nccl_comm) return fail(ctx, IRSDE_ERR_STATE, "communicator already initialised");
  std::string err;
  if (!nccl_load(&err)) return fail(ctx, IRSDE_ERR_UNSUPPORTED, err);
  cudaSetDevice(ctx->cfg.device);
  NcclId id;
  memcpy(id.internal, id128, sizeof id.internal);
  int rc = g_nccl.CommInitRank(&ctx->nccl_comm, nranks, id, rank);
  if (rc) { ctx->nccl_comm = nullptr; return nccl_fail(ctx, "ncclCommInitRank", rc); }
  ctx->comm_rank = rank; ctx->comm_nranks = nranks;
  return IRSDE_OK;
}

int irsde_broadcast_weights(irsde_ctx* ctx, int32_t src, void* stream) {
  if (!ctx || !ctx->nccl_comm) return fail(ctx, IRSDE_ERR_STATE, "irsde_comm_init first");
  if (src < 0 || src >= ctx->comm_nranks) return fail(ctx, IRSDE_ERR_INVALID, "bad source rank");
  if (ctx->raw.empty()) return fail(ctx, IRSDE_ERR_STATE, "load a state dict of the architecture on every rank first");
  cudaSetDevice(ctx->cfg.device);
  // every rank has loaded a state dict of the same names/shapes (std::map: same iteration order on every rank); the raw
  // fp32 tensors are overwritten in place inside ONE NCCL group (a single fused launch), then repacked for the kernels
  CUDA_TRY(ctx, cudaDeviceSynchronize());  // chains in flight still read the packed weights
  int rc = g_nccl.GroupStart();
  if (rc) return nccl_fail(ctx, "ncclGroupStart", rc);
  for (auto& kv : ctx->raw) {
    rc = g_nccl.Broadcast(kv.second.dev, kv.second.dev, (size_t)kv.second.numel, kNcclFloat, src, ctx->nccl_comm, (cudaStream_t)stream);
    if (rc) { g_nccl.GroupEnd(); return nccl_fail(ctx, "ncclBroadcast", rc); }
  }
  rc = g_nccl.GroupEnd();
  if (rc) return nccl_fail(ctx, "ncclGroupEnd", rc);
  CUDA_TRY(ctx, cudaStreamSynchronize((cudaStream_t)stream));
  ctx->finalized = false;
  return irsde_finalize_weights(ctx);
}

int irsde_gather(irsde_ctx* ctx, const float* x_local, float* x_all, const int64_t* counts, void* stream) {
  if (!ctx || !ctx->nccl_comm) return fail(ctx, IRSDE_ERR_STATE, "irsde_comm_init first");
  if (!x_all || !counts) return fail(ctx, IRSDE_ERR_INVALID, "bad argument");
  cudaSetDevice(ctx->cfg.device);
  // rank r's slice (counts[r] floats; the contiguous batch partition may be ragged) lands at the running offset in
  // x_all on EVERY rank: one broadcast per root inside a single group = an all-gather with per-rank counts
  int rc = g_nccl.GroupStart();
  if (rc) return nccl_fail(ctx, "ncclGroupStart", rc);
  int64_t off = 0;
  for (int r = 0; r < ctx->comm_nranks; ++r) {
    if (counts[r] < 0 || (r == ctx->comm_rank && counts[r] > 0 && !x_local)) { g_nccl.GroupEnd(); return fail(ctx, IRSDE_ERR_INVALID, "bad counts"); }
    if (counts[r] > 0) {
      rc = g_nccl.Broadcast(r == ctx->comm_rank ? (const void*)x_local : (const void*)(x_all + off), x_all + off, (size_t)counts[r],
                            kNcclFloat, r, ctx->nccl_comm, (cudaStream_t)stream);
      if (rc) { g_nccl.GroupEnd(); return nccl_fail(ctx, "ncclBroadcast", rc); }
    }
    off += counts[r];
  }
  rc = g_nccl.GroupEnd();
  return rc ? nccl_fail(ctx, "ncclGroupEnd", rc) : IRSDE_OK;
}

void irsde_destroy(irsde_ctx* ctx) {
  if (!ctx) return;
  if (ctx->nccl_comm && g_nccl.CommDestroy) g_nccl.CommDestroy(ctx->nccl_comm);
  cudaSetDevice(ctx->cfg.device);
  cudaDeviceSynchronize();
  if (ctx->order_ev) cudaEventDestroy(ctx->order_ev);
  for (auto& kv : ctx->plans) free_plan(ctx, kv.second);
  ctx->plans.clear();
  for (void* q : ctx->allocs) cudaFree(q);
  delete ctx;
}

int irsde_load_tensor(irsde_ctx* ctx, const char* name, const void* data, int32_t ndim, const int64_t* shape) {
  if (!ctx || !name || !data || ndim < 0 || ndim > 4) return fail(ctx, IRSDE_ERR_INVALID, "bad argument to irsde_load_tensor");
  cudaSetDevice(ctx->cfg.device);
  // Weights are pointer-stable buffers that captured step graphs read: a re-upload (load_state_dict, broadcast) must not
  // overtake chains still in flight on the caller's (possibly non-blocking) streams, and `data` may be a device tensor
  // that such a stream is still writing.  A device-to-device cudaMemcpy orders itself against neither, so every copy
  // waits for all earlier device work, and the call returns only once its copy is complete (the caller may free or
  // reuse `data` at once).
  CUDA_TRY(ctx, cudaDeviceSynchronize());
  long long n = 1;
  std::vector<int64_t> sh(shape, shape + ndim);
  for (auto d : sh) n *= d;
  RawTensor& t = ctx->raw[name];
  if (t.dev && t.numel != n) return fail(ctx, IRSDE_ERR_INVALID, std::string("shape change for ") + name);
  if (!t.dev) {
    t.dev = (float*)dev_alloc(ctx, (size_t)n * 4, &ctx->allocs);
    if (!t.dev) return fail(ctx, IRSDE_ERR_CUDA, "cudaMalloc failed");
  }
  t.shape = sh;
  t.numel = n;
  CUDA_TRY(ctx, cudaMemcpy(t.dev, data, (size_t)n * 4, cudaMemcpyDefault));
  CUDA_TRY(ctx, cudaDeviceSynchronize());
  ctx->finalized = false;
  return IRSDE_OK;
}

int irsde_finalize_weights(irsde_ctx* ctx) {
  if (!ctx) return fail(nullptr, IRSDE_ERR_INVALID, "null ctx");
  cudaSetDevice(ctx->cfg.device);
  auto specs = ctx->lat.on ? lat_param_specs(ctx->lat)
                           : (ctx->naf.on ? naf_param_specs(ctx->naf, ctx->cfg.variant) : param_specs(ctx->cfg, ctx->udim));
  for (auto& s : specs) {
    auto it = ctx->raw.find(s.name);
    if (it == ctx->raw.end()) return fail(ctx, IRSDE_ERR_STATE, "missing state-dict entry " + s.name);
    if (it->second.shape != s.shape) return fail(ctx, IRSDE_ERR_INVALID, "shape mismatch for " + s.name);
  }
  if (ctx->raw.size() != specs.size()) return fail(ctx, IRSDE_ERR_INVALID, "unexpected extra state-dict entries");
  // conv weights -> engine layouts (buffers are allocated once; reload keeps pointers stable)
  for (auto& s : specs) {
    if (s.pack == PACK_RAW) continue;
    const int Cout = (int)s.shape[0], Cin = (int)s.shape[1], KH = (int)s.shape[2], KW = (int)s.shape[3];
    const float* raw = ctx->raw[s.name].dev;
    auto pack_into = [&](auto*& buf, WLayout l) {
      using S = std::remove_reference_t<decltype(*buf)>;
      if (!buf) buf = (S*)dev_alloc(ctx, (size_t)packed_weight_elems<S>(l, Cout, Cin, KH, KW) * sizeof(S), &ctx->allocs);
      if (buf) pack_weight<S>(l, raw, buf, Cout, Cin, KH, KW, 1, 0);
      return buf != nullptr;
    };
    if (!pack_into(ctx->w_simt[s.name], WL_SIMT)) return fail(ctx, IRSDE_ERR_CUDA, "cudaMalloc failed");
    // the tap-GEMM runs a 7x7 conv only as the bf16 stem over at most 8 input channels
    const bool bf = ctx->cfg.precision == IRSDE_PREC_BF16;
    if (ctx->cfg.precision == IRSDE_PREC_FP32 || (KH == 7 && !(bf && Cin <= 8))) continue;
    const WLayout l = KH == 7 ? WL_STEM : s.pack == PACK_UP ? WL_UP : WL_TAPS;
    if (!(bf ? pack_into(ctx->w_tc[s.name], l) : pack_into(ctx->w_tc3[s.name], l))) return fail(ctx, IRSDE_ERR_CUDA, "cudaMalloc failed");
  }
  // time-modulation: concatenate every block's mlp.1 into one [S][td_in] matrix
  // (UNet ResBlock: Linear(4nf -> 2*Cout); NAFBlock: Linear(2w -> 4c))
  struct TB { std::string pre; int rows; };
  std::vector<TB> tbs;
  int td = 0;
  if (ctx->lat.on) {
    td = 1;  // no time conditioning in the autoencoder
  } else if (ctx->naf.on) {
    td = 2 * ctx->naf.width;
    for (auto& b : naf_blocks(ctx->naf)) tbs.push_back({b.pre, 4 * b.c});
  } else {
    td = ctx->cfg.nf * 4;
    for (auto& rb : resblocks(ctx->cfg, ctx->udim)) tbs.push_back({rb.pre, 2 * rb.cout});
  }
  int S = 0;
  for (auto& t : tbs) { ctx->ss_off[t.pre] = S; S += t.rows; }
  if (!ctx->wall) {
    ctx->wall = (float*)dev_alloc(ctx, (size_t)S * td * 4, &ctx->allocs);
    ctx->ball = (float*)dev_alloc(ctx, (size_t)S * 4, &ctx->allocs);
    if (!ctx->wall || !ctx->ball) return fail(ctx, IRSDE_ERR_CUDA, "cudaMalloc failed");
  }
  ctx->S = S;
  for (auto& t : tbs) {
    int off = ctx->ss_off[t.pre];
    CUDA_TRY(ctx, cudaMemcpy(ctx->wall + (size_t)off * td, ctx->raw[t.pre + "mlp.1.weight"].dev, (size_t)t.rows * td * 4,
                             cudaMemcpyDeviceToDevice));
    CUDA_TRY(ctx, cudaMemcpy(ctx->ball + off, ctx->raw[t.pre + "mlp.1.bias"].dev, (size_t)t.rows * 4, cudaMemcpyDeviceToDevice));
  }
  CUDA_TRY(ctx, cudaDeviceSynchronize());
  ctx->finalized = true;
  return IRSDE_OK;
}

int irsde_set_schedule(irsde_ctx* ctx, const float* thetas, const float* sigmas, const float* thetas_cumsum,
                       const float* sigma_bars, float dt, float max_sigma, int32_t T) {
  if (!ctx || !thetas || !sigmas || !thetas_cumsum || !sigma_bars || T < 1) return fail(ctx, IRSDE_ERR_INVALID, "bad schedule");
  cudaSetDevice(ctx->cfg.device);
  ctx->T = T; ctx->dt = dt; ctx->max_sigma = max_sigma;
  ctx->thetas.assign(thetas, thetas + T + 1);
  ctx->sigmas.assign(sigmas, sigmas + T + 1);
  ctx->cumsum.assign(thetas_cumsum, thetas_cumsum + T + 1);
  ctx->sbars.assign(sigma_bars, sigma_bars + T + 1);
  std::vector<float> tab;
  for (int m = 0; m < IRSDE_NUM_MODES; ++m) {
    fill_default_coeffs(ctx, m, tab);
    int rc = upload_coeffs(ctx, m, tab.data(), T);
    if (rc) return rc;
  }
  ctx->have_sched = true;
  return IRSDE_OK;
}

int irsde_set_coeffs(irsde_ctx* ctx, int32_t mode, const float* table, int32_t T) {
  if (!ctx || !table || mode < 0 || mode >= IRSDE_NUM_MODES) return fail(ctx, IRSDE_ERR_INVALID, "bad argument");
  if (!ctx->have_sched || T != ctx->T) return fail(ctx, IRSDE_ERR_STATE, "irsde_set_schedule must be called first with the same T");
  cudaSetDevice(ctx->cfg.device);
  return upload_coeffs(ctx, mode, table, T);
}

int irsde_noise_fn(irsde_ctx* ctx, const float* x, const float* mu, const float* times, int32_t n_times, float* out,
                   int32_t B, int32_t H, int32_t W, void* stream) {
  if (!ctx || !x || !times || !out) return fail(ctx, IRSDE_ERR_INVALID, "null argument");
  if (!ctx->finalized) return fail(ctx, IRSDE_ERR_STATE, "weights not finalized");
  if (ctx->cfg.variant == IRSDE_NET_CONDITIONAL && !mu) return fail(ctx, IRSDE_ERR_INVALID, "mu required for the conditional network");
  if (n_times != 1 && n_times != B) return fail(ctx, IRSDE_ERR_INVALID, "n_times must be 1 or B");
  cudaSetDevice(ctx->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  StreamOrder order(ctx, st);
  Plan* p;
  int rc = build_plan(ctx, B, H, W, &p);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaMemcpyAsync(p->fwd_times, times, (size_t)n_times * 4, cudaMemcpyHostToDevice, st));
  time_rows(ctx, p->fwd_times, n_times, p->fwd_temb, p->fwd_table, st);
  p->cur.x = x; p->cur.mu = mu; p->cur.out = out;
  p->cur.ss = p->fwd_table; p->cur.t_ptr = p->d_zero; p->cur.ss_img_stride = (n_times > 1) ? 1 : 0;
  run_forward(ctx, p, st);
  CUDA_TRY(ctx, cudaGetLastError());
  return IRSDE_OK;
}

int irsde_step(irsde_ctx* ctx, int32_t mode, const float* x, const float* mu, const float* noise, const float* z,
               int32_t t, float* out, int64_t n, void* stream) {
  if (!ctx || !x || !noise || !out || mode < 0 || mode >= IRSDE_NUM_MODES) return fail(ctx, IRSDE_ERR_INVALID, "bad argument");
  if (!ctx->have_sched) return fail(ctx, IRSDE_ERR_STATE, "schedule not set");
  if (t < 1 || t > ctx->T) return fail(ctx, IRSDE_ERR_INVALID, "t out of range [1,T]");
  bool need_z = mode == IRSDE_MODE_SDE || mode == IRSDE_MODE_POSTERIOR || mode == IRSDE_MODE_DSDE_SDE;
  if (need_z && !z) return fail(ctx, IRSDE_ERR_INVALID, "z required for stochastic modes");
  if (mode <= IRSDE_MODE_POSTERIOR && !mu) return fail(ctx, IRSDE_ERR_INVALID, "mu required for IRSDE modes");
  cudaSetDevice(ctx->cfg.device);
  launch_sde_update(mode, x, mu, noise, z, 0, ctx->coef_dev[mode], nullptr, t, out, n, 0, 0, 0, nullptr, (cudaStream_t)stream);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  return IRSDE_OK;
}

int irsde_reverse(irsde_ctx* ctx, int32_t mode, const float* xT, const float* mu, const float* z, float* x0, int32_t B,
                  int32_t H, int32_t W, int32_t T, uint64_t seed, int32_t use_graph, void* stream) {
  if (!ctx || !xT || !x0 || mode < 0 || mode >= IRSDE_NUM_MODES) return fail(ctx, IRSDE_ERR_INVALID, "bad argument");
  if (!ctx->finalized) return fail(ctx, IRSDE_ERR_STATE, "weights not finalized");
  if (!ctx->have_sched) return fail(ctx, IRSDE_ERR_STATE, "schedule not set");
  if (T < 0) T = ctx->T;
  if (T > ctx->T) return fail(ctx, IRSDE_ERR_INVALID, "T exceeds the schedule length");
  bool irs = mode <= IRSDE_MODE_POSTERIOR;
  if (irs != (ctx->cfg.variant == IRSDE_NET_CONDITIONAL))
    return fail(ctx, IRSDE_ERR_INVALID, "sampler mode does not match the network variant");
  if (irs && !mu) return fail(ctx, IRSDE_ERR_INVALID, "mu required");
  if (ctx->cfg.in_nc != ctx->cfg.out_nc) return fail(ctx, IRSDE_ERR_INVALID, "chain needs in_nc == out_nc");
  cudaSetDevice(ctx->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  StreamOrder order(ctx, st);
  Plan* p;
  int rc = build_plan(ctx, B, H, W, &p);
  if (rc) return rc;
  long long n = (long long)B * ctx->cfg.in_nc * H * W;
  CUDA_TRY(ctx, cudaMemcpyAsync(p->x_state, xT, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
  if (mu) CUDA_TRY(ctx, cudaMemcpyAsync(p->mu_buf, mu, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
  if (T == 0) {
    CUDA_TRY(ctx, cudaMemcpyAsync(x0, p->x_state, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    return IRSDE_OK;
  }
  rc = ensure_chain_table(ctx, p, ctx->T, st);
  if (rc) return rc;
  if (ctx->n_uids && ctx->n_uids != B) return fail(ctx, IRSDE_ERR_INVALID, "irsde_set_image_uids count does not match the batch");
  launch_set_step(p->d_step, T, 0, z, seed, ctx->image_base, ctx->n_uids ? ctx->d_uids : nullptr, st);
  ctx->launches++;
  p->cur.x = p->x_state; p->cur.mu = p->mu_buf; p->cur.out = p->eps_buf;
  p->cur.ss = p->chain_table; p->cur.t_ptr = &p->d_step->t; p->cur.ss_img_stride = 0;
  const float* mu_arg = irs ? p->mu_buf : nullptr;
  auto one_step = [&](cudaStream_t s) {
    run_forward(ctx, p, s);
    launch_sde_update(mode, p->x_state, mu_arg, p->eps_buf, nullptr, n, ctx->coef_dev[mode], p->d_step, 0, p->x_state, n, 0,
                      n / B, 0, nullptr, s);
    launch_advance_step(p->d_step, s);
    ctx->launches += 2;
  };
  if (use_graph && !ctx->prof) {
    if (!p->graph[mode]) {
      cudaStream_t cs;
      CUDA_TRY(ctx, cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
      long long before = ctx->launches;
      cudaGraph_t g;
      cudaError_t e = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
      if (e == cudaSuccess) {
        one_step(cs);
        e = cudaStreamEndCapture(cs, &g);
      }
      p->step_launches[mode] = ctx->launches - before;  // kernels in one captured step
      ctx->launches = before;                            // capture does not execute
      if (e != cudaSuccess) {
        cudaStreamDestroy(cs);
        return fail(ctx, IRSDE_ERR_CUDA, std::string("graph capture failed: ") + cudaGetErrorString(e));
      }
      e = cudaGraphInstantiate(&p->graph[mode], g, 0);
      cudaGraphDestroy(g);
      cudaStreamDestroy(cs);
      if (e != cudaSuccess) return fail(ctx, IRSDE_ERR_CUDA, std::string("graph instantiate failed: ") + cudaGetErrorString(e));
    }
    for (int i = 0; i < T; ++i) CUDA_TRY(ctx, cudaGraphLaunch(p->graph[mode], st));
    ctx->launches += (long long)T * p->step_launches[mode];
  } else {
    for (int i = 0; i < T; ++i) one_step(st);
  }
  CUDA_TRY(ctx, cudaMemcpyAsync(x0, p->x_state, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
  CUDA_TRY(ctx, cudaGetLastError());
  return IRSDE_OK;
}

int irsde_noise_state(irsde_ctx* ctx, const float* mu, float* out, int64_t n, uint64_t seed, void* stream) {
  if (!ctx || !mu || !out) return fail(ctx, IRSDE_ERR_INVALID, "null argument");
  if (!ctx->have_sched) return fail(ctx, IRSDE_ERR_STATE, "schedule not set");
  cudaSetDevice(ctx->cfg.device);
  launch_noise_state(mu, out, n, ctx->max_sigma, seed, n, ctx->image_base, nullptr, (cudaStream_t)stream);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  return IRSDE_OK;
}

int irsde_noise_state_images(irsde_ctx* ctx, const float* mu, float* out, int32_t B, int64_t image_elems, uint64_t seed,
                             void* stream) {
  if (!ctx || !mu || !out || B < 1 || image_elems < 1) return fail(ctx, IRSDE_ERR_INVALID, "bad argument");
  if (!ctx->have_sched) return fail(ctx, IRSDE_ERR_STATE, "schedule not set");
  cudaSetDevice(ctx->cfg.device);
  if (ctx->n_uids && ctx->n_uids != B) return fail(ctx, IRSDE_ERR_INVALID, "irsde_set_image_uids count does not match the batch");
  StreamOrder order(ctx, (cudaStream_t)stream);
  launch_noise_state(mu, out, (long long)B * image_elems, ctx->max_sigma, seed, image_elems, ctx->image_base,
                     ctx->n_uids ? ctx->d_uids : nullptr, (cudaStream_t)stream);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  return IRSDE_OK;
}

int irsde_random_states(const float* x0, const float* mu, const float* noise, const float* w, const float* sigma_bar, float* out,
                        int32_t B, int64_t image_elems, void* stream) {
  if (!x0 || !mu || !noise || !w || !sigma_bar || !out || B < 1 || image_elems < 1)
    return fail(nullptr, IRSDE_ERR_INVALID, "bad argument to irsde_random_states");
  launch_random_states(x0, mu, noise, w, sigma_bar, out, B, image_elems, (cudaStream_t)stream);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(nullptr, IRSDE_ERR_CUDA, std::string("random_states: ") + cudaGetErrorString(e));
  return IRSDE_OK;
}

int irsde_set_image_base(irsde_ctx* ctx, uint64_t first_image_uid) {
  if (!ctx) return fail(ctx, IRSDE_ERR_INVALID, "null ctx");
  ctx->image_base = first_image_uid;
  ctx->n_uids = 0;
  return IRSDE_OK;
}

int irsde_set_image_uids(irsde_ctx* ctx, const uint64_t* uids, int32_t n, void* stream) {
  const int MAX_UIDS = 4096;
  if (!ctx || !uids || n < 1 || n > MAX_UIDS) return fail(ctx, IRSDE_ERR_INVALID, "uids: need 1..4096 host values");
  cudaSetDevice(ctx->cfg.device);
  if (!ctx->d_uids) {
    ctx->d_uids = (unsigned long long*)dev_alloc(ctx, sizeof(unsigned long long) * MAX_UIDS, &ctx->allocs);
    if (!ctx->d_uids) return fail(ctx, IRSDE_ERR_CUDA, "cudaMalloc failed");
  }
  StreamOrder order(ctx, (cudaStream_t)stream);
  // pageable host source: the copy is staged before the call returns, so the caller may reuse `uids` at once
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_uids, uids, sizeof(uint64_t) * n, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  ctx->n_uids = n;
  return IRSDE_OK;
}

int irsde_profile_begin(irsde_ctx* ctx) {
  if (!ctx) return fail(nullptr, IRSDE_ERR_INVALID, "null ctx");
  for (auto& e : ctx->prof_events) { cudaEventDestroy(e.e0); cudaEventDestroy(e.e1); }
  ctx->prof_events.clear();
  ctx->prof = true;
  return IRSDE_OK;
}

int irsde_profile_end(irsde_ctx* ctx, double* ms, double* flops, int64_t* launches, int32_t ncat) {
  return irsde_profile_end_bytes(ctx, ms, flops, launches, nullptr, ncat);
}

int irsde_profile_end_bytes(irsde_ctx* ctx, double* ms, double* flops, int64_t* launches, double* bytes, int32_t ncat) {
  if (!ctx || !ms || !flops || !launches || ncat < CAT_COUNT) return fail(ctx, IRSDE_ERR_INVALID, "bad argument");
  cudaSetDevice(ctx->cfg.device);
  ctx->prof = false;
  CUDA_TRY(ctx, cudaDeviceSynchronize());
  for (int i = 0; i < ncat; ++i) { ms[i] = 0; flops[i] = 0; launches[i] = 0; if (bytes) bytes[i] = 0; }
  const char* dump = getenv("IRSDE_PROFILE_DUMP");
  for (auto& e : ctx->prof_events) {
    float t = 0.f;
    cudaEventElapsedTime(&t, e.e0, e.e1);
    if (dump && dump[0] == '1' && e.op)
      fprintf(stderr, "PROF\t%d\t%.4f\t%.1f\t%.1f\t%s\n", e.cat, t, e.op->flops > 0 ? e.op->flops / (t * 1e-3) / 1e12 : 0.0,
              e.op->bytes > 0 ? e.op->bytes / (t * 1e-3) / 1e9 : 0.0, e.op->label.c_str());
    ms[e.cat] += t;
    if (bytes && e.op) bytes[e.cat] += e.op->bytes;
    flops[e.cat] += e.flops;
    launches[e.cat] += 1;
    cudaEventDestroy(e.e0);
    cudaEventDestroy(e.e1);
  }
  ctx->prof_events.clear();
  return IRSDE_OK;
}

int irsde_trim(irsde_ctx* ctx) {
  if (!ctx) return fail(nullptr, IRSDE_ERR_INVALID, "null ctx");
  cudaSetDevice(ctx->cfg.device);
  evict_plans(ctx, nullptr, true);
  return IRSDE_OK;
}

int32_t irsde_plan_num_ops(irsde_ctx* ctx, int32_t B, int32_t H, int32_t W) {
  if (!ctx) return fail(nullptr, IRSDE_ERR_INVALID, "null ctx");
  if (!ctx->finalized) return fail(ctx, IRSDE_ERR_STATE, "weights not finalized");
  cudaSetDevice(ctx->cfg.device);
  Plan* p;
  int rc = build_plan(ctx, B, H, W, &p);
  return rc ? rc : (int32_t)p->ops.size();
}

int irsde_plan_op_info(irsde_ctx* ctx, int32_t B, int32_t H, int32_t W, int32_t op, char* label, int32_t label_cap,
                       int32_t* dims) {
  if (!ctx || !label || label_cap < 1 || !dims) return fail(ctx, IRSDE_ERR_INVALID, "bad argument");
  if (!ctx->finalized) return fail(ctx, IRSDE_ERR_STATE, "weights not finalized");
  cudaSetDevice(ctx->cfg.device);
  Plan* p;
  int rc = build_plan(ctx, B, H, W, &p);
  if (rc) return rc;
  if (op < 0 || op >= (int)p->ops.size()) return fail(ctx, IRSDE_ERR_INVALID, "op index out of range");
  const OpRec& r = p->ops[op];
  snprintf(label, (size_t)label_cap, "%s", r.label.c_str());
  dims[0] = r.out_p ? r.out_C : 0; dims[1] = r.out_H; dims[2] = r.out_W; dims[3] = r.cat;
  return IRSDE_OK;
}

int irsde_trace_forward(irsde_ctx* ctx, const float* x, const float* mu, const float* times, int32_t n_times, int32_t B,
                        int32_t H, int32_t W, int32_t op, float* dump, void* stream) {
  if (!ctx || !x || !times || !dump) return fail(ctx, IRSDE_ERR_INVALID, "null argument");
  if (!ctx->finalized) return fail(ctx, IRSDE_ERR_STATE, "weights not finalized");
  if (ctx->cfg.variant == IRSDE_NET_CONDITIONAL && !ctx->lat.on && !mu) return fail(ctx, IRSDE_ERR_INVALID, "mu required");
  if (n_times != 1 && n_times != B) return fail(ctx, IRSDE_ERR_INVALID, "n_times must be 1 or B");
  cudaSetDevice(ctx->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  StreamOrder order(ctx, st);
  Plan* p;
  int rc = build_plan(ctx, B, H, W, &p);
  if (rc) return rc;
  if (op < 0 || op >= (int)p->ops.size()) return fail(ctx, IRSDE_ERR_INVALID, "op index out of range");
  const OpRec& r = p->ops[op];
  if (!r.out_p) return fail(ctx, IRSDE_ERR_UNSUPPORTED, "this op has no NHWC output view to read back");
  CUDA_TRY(ctx, cudaMemcpyAsync(p->fwd_times, times, (size_t)n_times * 4, cudaMemcpyHostToDevice, st));
  time_rows(ctx, p->fwd_times, n_times, p->fwd_temb, p->fwd_table, st);
  p->cur.x = x; p->cur.mu = mu; p->cur.out = p->eps_buf;
  p->cur.ss = p->fwd_table; p->cur.t_ptr = p->d_zero; p->cur.ss_img_stride = (n_times > 1) ? 1 : 0;
  for (int i = 0; i <= op; ++i) ctx->launches += p->ops[i].fn(p, st);
  if (ctx->cfg.precision != IRSDE_PREC_BF16)
    launch_nhwc_to_nchw<float>((const float*)r.out_p, r.out_pitch, dump, B, r.out_C, r.out_H, r.out_W, st);
  else
    launch_nhwc_to_nchw<bf16>((const bf16*)r.out_p, r.out_pitch, dump, B, r.out_C, r.out_H, r.out_W, st);
  CUDA_TRY(ctx, cudaGetLastError());
  return IRSDE_OK;
}

int64_t irsde_launch_count(const irsde_ctx* ctx) { return ctx ? ctx->launches : 0; }
int64_t irsde_device_bytes(const irsde_ctx* ctx) { return ctx ? ctx->dev_bytes : 0; }

int irsde_conv2d(irsde_ctx* ctx, int32_t engine, const float* x, const float* w, const float* bias, float* y, int32_t B,
                 int32_t Cin, int32_t H, int32_t W, int32_t Cout, int32_t KH, int32_t KW, int32_t stride, int32_t pad,
                 int32_t upsample, int32_t silu, void* stream) {
  return irsde_conv2d_ex(ctx, engine, x, w, bias, nullptr, y, B, Cin, H, W, Cout, KH, KW, stride, pad, upsample, silu, 0, stream);
}

int irsde_conv2d_ex(irsde_ctx* ctx, int32_t engine, const float* x, const float* w, const float* bias, const float* residual,
                    float* y, int32_t B, int32_t Cin, int32_t H, int32_t W, int32_t Cout, int32_t KH, int32_t KW, int32_t stride,
                    int32_t pad, int32_t upsample, int32_t silu, int32_t flags, void* stream) {
  if (!ctx || !x || !w || !y) return fail(ctx, IRSDE_ERR_INVALID, "null argument");
  const bool f_qsm = (flags & IRSDE_CONV_QSOFTMAX) != 0, f_wimg = (flags & IRSDE_CONV_W_PER_IMAGE) != 0;
  if ((f_qsm || f_wimg) && engine != 1) return fail(ctx, IRSDE_ERR_UNSUPPORTED, "q-softmax / per-image weights are bf16 tensor-core epilogues");
  if (residual && engine == 0) return fail(ctx, IRSDE_ERR_UNSUPPORTED, "residual is an epilogue of the tensor-core engines");
  if ((f_qsm || f_wimg) && !(KH == 1 && KW == 1 && stride == 1 && pad == 0 && !upsample && Cout % 8 == 0))
    return fail(ctx, IRSDE_ERR_INVALID, "q-softmax / per-image weights need a 1x1 conv with Cout % 8 == 0");
  if (f_qsm && Cout < 128) return fail(ctx, IRSDE_ERR_INVALID, "q-softmax needs Cout >= 128 (4 heads x 32)");
  cudaSetDevice(ctx->cfg.device);
  if (engine < 0 || engine > 2) return fail(ctx, IRSDE_ERR_INVALID, "unknown engine");
  std::string terr;
  if (engine != 0 && !tc_init(&terr)) return fail(ctx, IRSDE_ERR_CUDA, "tc_init: " + terr);
  const int up = upsample ? 2 : 1;
  const ConvShape s = conv_shape(KH, KW, stride, pad, up, H, W);
  bool k7 = false, nchw = false;  // nchw: head-style output, fp32 NCHW straight from the epilogue
  if (engine == 1) {  // bf16 tap-GEMM: the plan builder's shapes, the stem included
    k7 = s.k7 && Cin <= 8 && Cout % 8 == 0;
    nchw = Cout % 8 != 0;
    if (!(s.k3 || s.k1 || s.k4 || k7) || (!k7 && Cin % 8) || (nchw && !(s.k3 && up == 1)))
      return fail(ctx, IRSDE_ERR_UNSUPPORTED, "shape not supported by the tensor-core engine");
    if (residual && nchw) return fail(ctx, IRSDE_ERR_UNSUPPORTED, "residual needs Cout % 8 == 0");
  } else if (engine == 2) {  // fp32x3: fp32 NHWC, hi/lo split, 3 x tf32 wgmma (conv_tc.cu MODE 3)
    nchw = Cout % 4 != 0;
    if (!(s.k3 || s.k1 || s.k4) || Cin % 4 || (nchw && !(s.k3 && up == 1)) || residual && nchw)
      return fail(ctx, IRSDE_ERR_UNSUPPORTED, "shape not supported by the fp32x3 engine");
  }
  const ConvGeom g = conv_geom(B, Cin, H, W, Cout, KH, KW, stride, pad, up);
  const int Ho = g.Hout, Wo = g.Wout;
  // per-image: w is [B][Cout][Cin]
  const WLayout wl = engine == 0 ? WL_SIMT : k7 ? WL_STEM : f_wimg ? WL_PER_IMAGE : (s.k3 && up == 2) ? WL_UP : WL_TAPS;
  const int tc_flags = (f_qsm ? TC_FLAG_QSOFTMAX : 0) | (f_wimg ? TC_FLAG_W_PER_IMAGE : 0);
  Scratch sc(ctx, (cudaStream_t)stream);
  // NCHW -> NHWC staging in the engine's storage type; bf16 output rows padded to 8 channels, the fp32x3 output with slack
  auto run = [&](auto* type) {
    using S = std::remove_pointer_t<decltype(type)>;
    const long long nin = k7 ? (long long)B * (H + 6) * (W + 8) * 8 + 64 : (long long)B * H * W * Cin;
    const long long nout = (long long)B * Ho * Wo * (engine == 1 ? (Cout + 7) / 8 * 8 : Cout);
    S* res = residual ? sc.alloc<S>(nout) : nullptr;
    S* xin = sc.alloc<S>(nin);
    S* yo = sc.alloc<S>(engine == 2 ? nout + 16 : nout);
    if ((residual && !res) || !xin || !yo) return sc.oom();
    if (res) launch_nchw_to_nhwc<S>(residual, res, B, Cout, Ho, Wo, Cout, sc.st);
    if (k7) {
      cudaMemsetAsync(xin, 0, nin * sizeof(S), sc.st);
      launch_prep_input<S>(x, nullptr, xin, B, Cin, H, W, H, W, 8, 0, sc.st, 3, 3, W + 8, H + 6);
    } else {
      launch_nchw_to_nhwc<S>(x, xin, B, Cin, H, W, Cin, sc.st);
    }
    Epilogue ep;
    memset(&ep, 0, sizeof ep);
    ep.bias = bias;
    ep.silu = silu;
    if (res) { ep.res = res; ep.res_pitch = Cout; }
    const int rc = run_conv<S>(sc, g, xin, k7 ? 8 : Cin, wl, w, ep, nchw ? nullptr : yo, Cout, nchw ? y : nullptr, Ho, Wo, tc_flags,
                               nullptr);
    if (!rc && !nchw) launch_nhwc_to_nchw<S>(yo, Cout, y, B, Cout, Ho, Wo, sc.st);
    return rc;
  };
  const int rc = engine == 1 ? run((bf16*)nullptr) : run((float*)nullptr);
  if (!rc) ctx->launches += engine == 2 ? 5 : 4;
  return sc.finish(rc, engine == 1 ? "tensor-core conv2d failed" : engine == 2 ? "fp32x3 conv2d failed" : "conv2d failed");
}

int irsde_conv2d_fused(irsde_ctx* ctx, int32_t engine, const float* x, const float* w, const irsde_conv_epilogue* epi, float* y,
                       int32_t B, int32_t Cin, int32_t H, int32_t W, int32_t Cout, int32_t KH, int32_t KW, int32_t stride,
                       int32_t pad, int32_t upsample, int32_t* info, void* stream) {
  // ---- everything is validated here, before the first launch: no argument may make a kernel index out of bounds
  if (!ctx || !x || !w || !y || !epi) return fail(ctx, IRSDE_ERR_INVALID, "null argument");
  const irsde_conv_epilogue& e = *epi;
  if (engine < 0 || engine > 3) return fail(ctx, IRSDE_ERR_INVALID, "unknown engine");
  if (B < 1 || Cin < 1 || H < 1 || W < 1 || Cout < 1) return fail(ctx, IRSDE_ERR_INVALID, "bad shape");
  const bool simt = engine == 0 || engine == 3, bf = engine == 1 || engine == 3;
  const int up = upsample ? 2 : 1;
  const ConvShape s = conv_shape(KH, KW, stride, pad, up, H, W);
  const bool k7 = engine == 1 && s.k7;  // the bf16 tensor-core stem
  if (simt) {  // the SIMT kernel takes any kernel size, stride and padding
    if (KH < 1 || KW < 1 || KH > 16 || KW > 16 || stride < 1 || pad < 0 || pad >= KH || pad >= KW ||
        H * up + 2 * pad < KH || W * up + 2 * pad < KW)
      return fail(ctx, IRSDE_ERR_INVALID, "SIMT conv: bad kernel size, stride or padding");
  } else if (!(s.k3 || s.k1 || s.k4 || s.k2 || k7)) {
    return fail(ctx, IRSDE_ERR_UNSUPPORTED,
                "tensor-core conv: 3x3/1 (optionally after nearest x2), 1x1, 4x4/2 or 2x2/2 over an even H x W, or the bf16 7x7 stem");
  }
  const ConvGeom g = conv_geom(B, Cin, H, W, Cout, KH, KW, stride, pad, up);
  const int Ho = g.Hout, Wo = g.Wout;
  const bool nchw = e.crop_h != 0 || e.crop_w != 0;
  const bool qsm = (e.flags & IRSDE_CONV_QSOFTMAX) != 0;
  if (e.flags & ~IRSDE_CONV_QSOFTMAX) return fail(ctx, IRSDE_ERR_UNSUPPORTED, "fused conv: flags other than IRSDE_CONV_QSOFTMAX");
  if (qsm && (engine != 1 || !s.k1 || Cout < 128 || nchw))
    return fail(ctx, IRSDE_ERR_INVALID, "q-softmax is the bf16 epilogue of a 1x1 conv with Cout >= 128");
  // views: offsets and pitches in 16 bytes of the tap-GEMM's storage type, or in the SIMT kernel's 4-element vectors
  const int al = engine == 1 ? 8 : 4;
  if (!simt && ((k7 ? Cin > 8 : Cin % al) || (!nchw && Cout % al)))
    return fail(ctx, IRSDE_ERR_INVALID, "tensor-core engines: Cin and Cout must be multiples of 16 bytes (the stem: Cin <= 8)");
  if (!view_ok(e.in_pitch, e.in_off, Cin, al)) return fail(ctx, IRSDE_ERR_INVALID, "input view outside its pitch or not aligned");
  if (nchw) {
    if (!simt && (!s.k3 || up != 1))
      return fail(ctx, IRSDE_ERR_UNSUPPORTED, "the tensor-core engines' cropped fp32 NCHW output is the 3x3 head's epilogue");
    if (e.crop_h < 1 || e.crop_w < 1 || e.crop_h > Ho || e.crop_w > Wo) return fail(ctx, IRSDE_ERR_INVALID, "crop larger than the output");
    if (e.res) return fail(ctx, IRSDE_ERR_UNSUPPORTED, "no residual with the NCHW output");
  } else if (!view_ok(e.out_pitch, e.out_off, Cout, al)) {
    return fail(ctx, IRSDE_ERR_INVALID, "output view outside its pitch or not aligned");
  }
  if (e.res && !view_ok(e.res_pitch, e.res_off, Cout, al))
    return fail(ctx, IRSDE_ERR_INVALID, "residual view outside its pitch or not aligned");
  if (e.ss) {
    if (e.mult_vec) return fail(ctx, IRSDE_ERR_INVALID, "the time-modulation table and mult_vec cannot be combined");
    if (e.t_row < 0 || e.ss_img_stride < 0 || (long long)e.t_row + (long long)(B - 1) * e.ss_img_stride >= e.ss_rows)
      return fail(ctx, IRSDE_ERR_INVALID, "time-modulation row outside the table");
    if (e.ss_off < 0 || (long long)e.ss_off + 2LL * Cout > e.ss_S)
      return fail(ctx, IRSDE_ERR_INVALID, "scale / shift columns outside the table row");
  }
  const float* ptrs[] = {x, y, e.res, e.bias, e.mult_vec, e.ss};
  for (const float* q : ptrs)
    if ((uintptr_t)q & 15) return fail(ctx, IRSDE_ERR_INVALID, "device buffers must be 16-byte aligned");
  int32_t info_local[4];
  info = zeroed_info(info, info_local);

  cudaSetDevice(ctx->cfg.device);
  std::string terr;
  if (!simt && !tc_init(&terr)) return fail(ctx, IRSDE_ERR_CUDA, "tc_init: " + terr);
  Scratch sc(ctx, (cudaStream_t)stream);
  const int* t_dev = sc.upload(e.t_row);
  if (!t_dev) return sc.oom();
  Epilogue ep;
  memset(&ep, 0, sizeof ep);
  ep.bias = e.bias;
  ep.mult_vec = e.mult_vec;
  ep.silu = e.silu;
  ep.ss_S = e.ss_S;
  ep.ss_off = e.ss_off;
  if (e.ss) { ep.ss = e.ss; ep.t_ptr = t_dev; ep.ss_img_stride = e.ss_img_stride; }
  ep.res_pitch = e.res_pitch;
  const WLayout wl = simt ? WL_SIMT : k7 ? WL_STEM : (s.k3 && up == 2) ? WL_UP : WL_TAPS;
  float* out_nchw = nchw ? y : nullptr;
  int rc;
  if (bf) {  // bf16 copies of the whole of x, res and y
    const long long npix_out = (long long)B * Ho * Wo;
    const bf16* xb;
    int in_pitch = e.in_pitch;
    if (k7) {  // the stem reads its input view from the zero-bordered [B][H+6][W+8][8] layout, as a plan stages it
      const long long nin = (long long)B * (H + 6) * (W + 8) * 8 + 64;
      float* xn = sc.alloc<float>((long long)B * Cin * H * W);
      bf16* xp = sc.alloc<bf16>(nin);
      if (!xn || !xp) return sc.oom();
      cudaMemsetAsync(xp, 0, nin * sizeof(bf16), sc.st);
      launch_nhwc_to_nchw<float>(x + e.in_off, e.in_pitch, xn, B, Cin, H, W, sc.st);
      launch_prep_input<bf16>(xn, nullptr, xp, B, Cin, H, W, H, W, 8, 0, sc.st, 3, 3, W + 8, H + 6);
      xb = xp;
      in_pitch = 8;
    } else {
      xb = sc.in(x, (long long)B * H * W * e.in_pitch);
      if (xb) xb += e.in_off;
    }
    const bf16* rb = e.res ? sc.in(e.res, npix_out * e.res_pitch) : nullptr;
    bf16* yb = nchw ? nullptr : sc.inout(y, npix_out * e.out_pitch);
    if (!xb || (e.res && !rb) || (!nchw && !yb)) return sc.oom();
    if (rb) ep.res = rb + e.res_off;
    rc = run_conv<bf16>(sc, g, xb, in_pitch, wl, w, ep, yb ? yb + e.out_off : nullptr, e.out_pitch, out_nchw, e.crop_h, e.crop_w,
                        qsm ? TC_FLAG_QSOFTMAX : 0, info);
  } else {
    if (e.res) ep.res = e.res + e.res_off;
    rc = run_conv<float>(sc, g, x + e.in_off, e.in_pitch, wl, w, ep, nchw ? nullptr : y + e.out_off, e.out_pitch, out_nchw,
                         e.crop_h, e.crop_w, 0, info);
  }
  if (!rc) ctx->launches += 4;
  return sc.finish(rc, "fused conv2d failed");
}

// ---- one LayerNorm / attention op outside a plan ------------------------------------------------------------------
int irsde_layernorm(irsde_ctx* ctx, int32_t precision, const float* x, const irsde_ln_args* args, float* y, int32_t B, int32_t N,
                    int32_t C, int32_t* info, void* stream) {
  // ---- everything is validated here, before the first allocation or launch
  if (!ctx || !x || !y || !args || !args->g) return fail(ctx, IRSDE_ERR_INVALID, "null argument");
  const irsde_ln_args& a = *args;
  if (precision < IRSDE_PREC_FP32 || precision > IRSDE_PREC_FP32X3) return fail(ctx, IRSDE_ERR_INVALID, "bad precision");
  if (B < 1 || N < 1 || C < 1) return fail(ctx, IRSDE_ERR_INVALID, "bad shape");
  if (!view_ok(a.in_pitch, a.in_off, C)) return fail(ctx, IRSDE_ERR_INVALID, "input view outside its pitch");
  if (!view_ok(a.out_pitch, a.out_off, C)) return fail(ctx, IRSDE_ERR_INVALID, "output view outside its pitch");
  if (a.res && !view_ok(a.res_pitch, a.res_off, C)) return fail(ctx, IRSDE_ERR_INVALID, "residual view outside its pitch");
  if (a.ss) {
    if (a.t_row < 0 || a.ss_img_stride < 0 || (long long)a.t_row + (long long)(B - 1) * a.ss_img_stride >= a.ss_rows)
      return fail(ctx, IRSDE_ERR_INVALID, "time-modulation row outside the table");
    if (a.off_scale < 0 || a.off_shift < 0 || (long long)a.off_scale + C > a.ss_S || (long long)a.off_shift + C > a.ss_S)
      return fail(ctx, IRSDE_ERR_INVALID, "scale / shift columns outside the table row");
  }
  int32_t info_local[4];
  info = zeroed_info(info, info_local);

  cudaSetDevice(ctx->cfg.device);
  const long long npix = (long long)B * N;
  Scratch sc(ctx, (cudaStream_t)stream);
  const int* t_dev = sc.upload(a.t_row);
  if (!t_dev) return sc.oom();
  LnMod m;
  memset(&m, 0, sizeof m);
  if (a.ss) {
    m.ss = a.ss; m.t_ptr = t_dev; m.S = a.ss_S; m.off_scale = a.off_scale; m.off_shift = a.off_shift;
    m.img_stride = a.ss_img_stride;
  }
  m.pix_per_img = N;
  LnPick k{};
  auto run = [&](auto* xs, auto* rs, auto* ys) {
    using S = std::remove_pointer_t<decltype(ys)>;
    const S *xv = xs + a.in_off, *rv = rs ? rs + a.res_off : nullptr;
    S* yv = ys + a.out_off;
    k = ln_pick<S>(C, npix, a.in_pitch, a.res_pitch, a.out_pitch, xv, a.g, rv, yv);
    launch_layernorm<S>(xv, a.in_pitch, a.g, rv, a.res_pitch, yv, a.out_pitch, npix, C, sc.st, &m);
  };
  if (precision == IRSDE_PREC_BF16) {
    const bf16* xb = sc.in(x, npix * a.in_pitch);
    bf16* yb = sc.inout(y, npix * a.out_pitch);
    const bf16* rb = a.res ? sc.in(a.res, npix * a.res_pitch) : nullptr;
    if (!xb || !yb || (a.res && !rb)) return sc.oom();
    run(xb, rb, yb);
  } else {
    run(x, a.res, y);
  }
  info[0] = k.kind; info[1] = k.maxv; info[2] = k.lpp; info[3] = k.pp;
  ctx->launches++;
  return sc.finish(IRSDE_OK, "layernorm failed");
}

int irsde_attention(irsde_ctx* ctx, int32_t precision, int32_t kind, const float* qkv, int32_t qkv_pitch, int32_t qkv_off,
                    float* out, int32_t out_pitch, int32_t out_off, const float* wout, int32_t Cout, float* ctx_out, int32_t B,
                    int32_t N, int32_t* info, void* stream) {
  // ---- everything is validated here, before the first allocation or launch
  if (!ctx || !qkv || !out) return fail(ctx, IRSDE_ERR_INVALID, "null argument");
  if (precision < IRSDE_PREC_FP32 || precision > IRSDE_PREC_FP32X3) return fail(ctx, IRSDE_ERR_INVALID, "bad precision");
  if (kind < IRSDE_ATTN_LINEAR || kind > IRSDE_ATTN_FULL) return fail(ctx, IRSDE_ERR_INVALID, "unknown attention kind");
  const bool bf = precision == IRSDE_PREC_BF16, lin = kind != IRSDE_ATTN_FULL, fold = kind == IRSDE_ATTN_LINEAR_FOLD;
  if (fold && !bf) return fail(ctx, IRSDE_ERR_UNSUPPORTED, "the folded linear attention is the bf16 path");
  if (B < 1 || N < 1) return fail(ctx, IRSDE_ERR_INVALID, "bad shape");
  if (int rc = check_shape_limits(ctx, lin ? B : 4LL * B, lin ? "B" : "4 B (full-attention grid rows)", N, 1)) return rc;
  if (lin && !ctx_out) return fail(ctx, IRSDE_ERR_INVALID, "linear attention needs ctx_out");
  if (fold && (!wout || Cout < 1 || ((uintptr_t)wout & 15)))
    return fail(ctx, IRSDE_ERR_INVALID, "the fold needs 16-byte aligned to_out weights [Cout][128], Cout >= 1");
  if (!view_ok(qkv_pitch, qkv_off, 384)) return fail(ctx, IRSDE_ERR_INVALID, "qkv view outside its pitch");
  if (!fold && !view_ok(out_pitch, out_off, 128)) return fail(ctx, IRSDE_ERR_INVALID, "hidden view outside its pitch");
  // the views the launchers get: the caller's buffers (fp32), or bf16 copies that start on 256 bytes
  const size_t elem = bf ? 2 : 4;
  auto at = [&](const float* base, int off) { return (const void*)((bf ? 0 : (uintptr_t)base) + (uintptr_t)off * elem); };
  if (lin && !linattn_views_ok(at(qkv, qkv_off), qkv_pitch, fold ? nullptr : at(out, out_off), out_pitch, elem))
    return fail(ctx, IRSDE_ERR_INVALID, "linear attention: views must start on 16 bytes and pitches be multiples of 16 bytes");
  int32_t info_local[4];
  info = zeroed_info(info, info_local);

  cudaSetDevice(ctx->cfg.device);
  const long long npix = (long long)B * N;
  Scratch sc(ctx, (cudaStream_t)stream);
  float* part = lin ? sc.alloc<float>(linattn_partial_floats(B, N)) : nullptr;
  float* cx = lin ? sc.alloc<float>((long long)B * 4096) : nullptr;
  if (lin && (!part || !cx)) return sc.oom();
  int kern = 0;
  // kern: 1 / 2 the fp32 / bf16 linear attention, 3 the scalar and 4 the MMA full attention
  auto run = [&](auto* qs, auto* os) -> bool {
    using S = std::remove_pointer_t<decltype(os)>;
    const S* qv = qs + qkv_off;
    if (lin) kern = bf ? 2 : 1;
    if constexpr (std::is_same<S, bf16>::value) {
      if (fold) {
        if (!launch_linattn_ctx<bf16>(qv, qkv_pitch, part, cx, B, N, sc.st)) return false;
        launch_la_fold(cx, wout, os, B, Cout, sc.st);
        return true;
      }
    }
    if (lin) return launch_linattn<S>(qv, qkv_pitch, part, cx, os + out_off, out_pitch, B, N, sc.st);
    kern = fullattn_pick<S>(qv, qkv_pitch, os + out_off, out_pitch) == FA_MMA ? 4 : 3;
    launch_fullattn<S>(qv, qkv_pitch, os + out_off, out_pitch, B, N, sc.st);
    return true;
  };
  bool launched;
  if (bf) {
    const long long no = fold ? (long long)B * Cout * 128 : npix * out_pitch;
    const bf16* qb = sc.in(qkv, npix * qkv_pitch);
    bf16* ob = fold ? sc.out(out, no) : sc.inout(out, no);
    if (!qb || !ob) return sc.oom();
    launched = run(qb, ob);
  } else {
    launched = run(qkv, out);
  }
  if (!launched) return fail(ctx, IRSDE_ERR_INVALID, "the linear-attention launcher refused the views");
  if (lin) {
    int nblk, nchunks;
    linattn_partition(B, N, &nblk, &nchunks);
    info[1] = nblk; info[2] = nchunks;
    cudaMemcpyAsync(ctx_out, cx, (size_t)B * 4096 * sizeof(float), cudaMemcpyDeviceToDevice, sc.st);
  }
  info[0] = kern;
  ctx->launches += lin ? 3 : 1;
  return sc.finish(IRSDE_OK, "attention failed");
}

int irsde_linattn_block(irsde_ctx* ctx, const float* x, int32_t x_pitch, int32_t x_off, float* out, int32_t out_pitch,
                        int32_t out_off, const float* g1, const float* wqkv, const float* wout, const float* bout, const float* g2,
                        float* xn_out, int32_t B, int32_t N, int32_t C, void* stream) {
  // ---- everything is validated here, before the first allocation or launch
  if (!ctx || !x || !out || !g1 || !wqkv || !wout || !bout || !g2) return fail(ctx, IRSDE_ERR_INVALID, "null argument");
  if (B < 1 || N < 1) return fail(ctx, IRSDE_ERR_INVALID, "bad shape");
  if (int rc = check_shape_limits(ctx, B, "B", N, 1)) return rc;
  if (C != 64 && C != 128) return fail(ctx, IRSDE_ERR_UNSUPPORTED, "the fused linear-attention block takes C = 64 or 128");
  if (!view_ok(x_pitch, x_off, C)) return fail(ctx, IRSDE_ERR_INVALID, "input view outside its pitch");
  if (!view_ok(out_pitch, out_off, C)) return fail(ctx, IRSDE_ERR_INVALID, "output view outside its pitch");
  if (x_pitch % 8 || x_off % 8 || out_pitch % 2 || out_off % 2)
    return fail(ctx, IRSDE_ERR_INVALID, "input view: pitch and offset multiples of 8; output view: multiples of 2");
  if (((uintptr_t)g1 | (uintptr_t)g2 | (uintptr_t)bout | (uintptr_t)wout) & 15)
    return fail(ctx, IRSDE_ERR_INVALID, "g1, g2, bout and wout must start on 16 bytes");
  cudaSetDevice(ctx->cfg.device);
  const long long npix = (long long)B * N;
  Scratch sc(ctx, (cudaStream_t)stream);
  float* part = sc.alloc<float>(linattn_partial_floats(B, N));
  float* cx = sc.alloc<float>((long long)B * 4096);
  const bf16* xb = sc.in(x, npix * x_pitch);
  bf16* ob = sc.inout(out, npix * out_pitch);
  bf16* wp = sc.alloc<bf16>(384LL * C);
  bf16* Mb = sc.alloc<bf16>((long long)B * C * 128);
  bf16* xnb = xn_out ? sc.out(xn_out, npix * C) : nullptr;
  if (!part || !cx || !xb || !ob || !wp || !Mb || (xn_out && !xnb)) return sc.oom();
  if (!linattn_fused_ok(C, xb + x_off, x_pitch, ob + out_off, out_pitch))
    return fail(ctx, IRSDE_ERR_INVALID, "the fused linear-attention passes refused the views");
  pack_weight<bf16>(WL_TAPS, wqkv, wp, 384, C, 1, 1, 1, sc.st);  // the layout irsde_finalize_weights gives to_qkv
  launch_la_kv_ln(xb + x_off, x_pitch, g1, wp + 128 * C, part, B, N, C, xnb, sc.st);
  launch_la_combine(part, cx, B, N, sc.st);
  launch_la_fold(cx, wout, Mb, B, C, sc.st);
  launch_la_out_ln(xb + x_off, x_pitch, g1, wp, Mb, bout, g2, ob + out_off, out_pitch, B, N, C, sc.st);
  ctx->launches += 4;
  return sc.finish(IRSDE_OK, "linear-attention block failed");
}

// ---- one NAFNet op, time embedding, sampler step or input packing outside a plan ----------------------------------
int irsde_nafnet_op(irsde_ctx* ctx, int32_t precision, int32_t kind, const irsde_nafnet_args* args, int32_t B, int32_t H,
                    int32_t W, int32_t c, int32_t* info, void* stream) {
  // ---- everything is validated here, before the first allocation or launch
  if (!ctx || !args || !args->x || !args->out) return fail(ctx, IRSDE_ERR_INVALID, "null argument");
  const irsde_nafnet_args& a = *args;
  if (precision < IRSDE_PREC_FP32 || precision > IRSDE_PREC_FP32X3) return fail(ctx, IRSDE_ERR_INVALID, "bad precision");
  if (kind < IRSDE_NAF_DWGATE_SCA || kind > IRSDE_NAF_ADD) return fail(ctx, IRSDE_ERR_INVALID, "unknown NAFNet op");
  const bool dw = kind == IRSDE_NAF_DWGATE_SCA, ps = kind == IRSDE_NAF_PIXEL_SHUFFLE_ADD;
  if (B < 1 || H < 1 || W < 1 || c < 1) return fail(ctx, IRSDE_ERR_INVALID, "bad shape");
  if (int rc = check_shape_limits(ctx, B, "B", ps ? 2LL * H : H, ps ? 2LL * W : W)) return rc;
  if (dw && c > kScaMaxC) return fail(ctx, IRSDE_ERR_UNSUPPORTED, "c > 12288: the SCA mat-vec needs more than 48 KB of shared memory");
  if (dw && (!a.w || !a.bias || !a.sca_w || !a.sca_b || !a.sca)) return fail(ctx, IRSDE_ERR_INVALID, "DWGATE_SCA needs w, bias, sca_w, sca_b and sca");
  if ((ps || kind == IRSDE_NAF_ADD) && !a.y) return fail(ctx, IRSDE_ERR_INVALID, "PIXEL_SHUFFLE_ADD and ADD need y");
  const long long xw = ps ? 4LL * c : kind == IRSDE_NAF_ADD ? c : 2LL * c;
  if (!view_ok(a.x_pitch, a.x_off, xw)) return fail(ctx, IRSDE_ERR_INVALID, "x view outside its pitch");
  if (a.y && (ps || kind == IRSDE_NAF_ADD) && !view_ok(a.y_pitch, a.y_off, c)) return fail(ctx, IRSDE_ERR_INVALID, "y view outside its pitch");
  if (!view_ok(a.out_pitch, a.out_off, c)) return fail(ctx, IRSDE_ERR_INVALID, "out view outside its pitch");
  int32_t info_local[4];
  info = zeroed_info(info, info_local);

  cudaSetDevice(ctx->cfg.device);
  const int N = H * W;
  const long long npix_in = (long long)B * N, npix_out = ps ? 4 * npix_in : npix_in;  // PIXEL_SHUFFLE_ADD: H x W is the input
  const int nchunks = dw ? dwgate_chunks(H, W) : 0;
  Scratch sc(ctx, (cudaStream_t)stream);
  float* partial = dw ? sc.alloc<float>((long long)B * nchunks * c) : nullptr;
  if (dw && !partial) return sc.oom();
  int sca_launches = 0;
  // one launch path for both storage types: S = float views of the caller's buffers, or bf16 copies of them
  auto run = [&](auto* xs, auto* ys, auto* os) {
    using S = std::remove_pointer_t<decltype(os)>;
    const S* xv = xs + a.x_off;
    const S* yv = ys ? ys + a.y_off : nullptr;
    S* ov = os + a.out_off;
    if (dw) {
      launch_dwgate<S>(xv, a.x_pitch, a.w, a.bias, ov, a.out_pitch, partial, B, H, W, c, sc.st);
      launch_sca_scale<S>(partial, a.sca_w, a.sca_b, a.sca, ov, a.out_pitch, B, c, nchunks, N, &sca_launches, sc.st);
    } else if (kind == IRSDE_NAF_SIMPLE_GATE) {
      launch_simple_gate<S>(xv, a.x_pitch, ov, a.out_pitch, npix_in, c, sc.st);
    } else if (ps) {
      launch_pixel_shuffle_add<S>(xv, a.x_pitch, yv, a.y_pitch, ov, a.out_pitch, B, H, W, c, sc.st);
    } else {
      launch_add<S>(xv, a.x_pitch, yv, a.y_pitch, ov, a.out_pitch, npix_in, c, sc.st);
    }
  };
  const bool has_y = ps || kind == IRSDE_NAF_ADD;
  if (precision == IRSDE_PREC_BF16) {
    const bf16* xb = sc.in(a.x, npix_in * a.x_pitch);
    const bf16* yb = has_y ? sc.in(a.y, npix_out * a.y_pitch) : nullptr;
    bf16* ob = sc.inout(a.out, npix_out * a.out_pitch);
    if (!xb || !ob || (has_y && !yb)) return sc.oom();
    run(xb, yb, ob);
  } else {
    run(a.x, has_y ? a.y : (const float*)nullptr, a.out);
  }
  if (dw) {
    info[0] = dw_pix(N); info[1] = nchunks; info[2] = sca_launches;
    ctx->launches += 1 + sca_launches;
  } else {
    ctx->launches++;
  }
  return sc.finish(IRSDE_OK, "NAFNet op failed");
}

int irsde_step_philox(irsde_ctx* ctx, int32_t mode, const float* x, const float* mu, const float* noise, int32_t t, float* out,
                      int32_t B, int64_t image_elems, uint64_t seed, void* stream) {
  if (!ctx || !x || !noise || !out || mode < 0 || mode >= IRSDE_NUM_MODES) return fail(ctx, IRSDE_ERR_INVALID, "bad argument");
  if (mode != IRSDE_MODE_SDE && mode != IRSDE_MODE_POSTERIOR && mode != IRSDE_MODE_DSDE_SDE)
    return fail(ctx, IRSDE_ERR_INVALID, "the ODE modes draw no noise");
  if (!ctx->have_sched) return fail(ctx, IRSDE_ERR_STATE, "schedule not set");
  if (t < 1 || t > ctx->T) return fail(ctx, IRSDE_ERR_INVALID, "t out of range [1,T]");
  if (mode <= IRSDE_MODE_POSTERIOR && !mu) return fail(ctx, IRSDE_ERR_INVALID, "mu required for IRSDE modes");
  if (B < 1 || image_elems < 1) return fail(ctx, IRSDE_ERR_INVALID, "bad shape");
  if (ctx->n_uids && ctx->n_uids != B) return fail(ctx, IRSDE_ERR_INVALID, "irsde_set_image_uids count does not match the batch");
  cudaSetDevice(ctx->cfg.device);
  StreamOrder order(ctx, (cudaStream_t)stream);
  launch_sde_update(mode, x, mu, noise, nullptr, 0, ctx->coef_dev[mode], nullptr, t, out, (long long)B * image_elems, seed,
                    image_elems, ctx->image_base, ctx->n_uids ? ctx->d_uids : nullptr, (cudaStream_t)stream);
  ctx->launches++;
  CUDA_TRY(ctx, cudaGetLastError());
  return IRSDE_OK;
}

int irsde_time_embedding(int32_t family, const float* times, int32_t rows, int32_t width, const float* w1, const float* b1,
                         const float* w2, const float* b2, const float* wall, const float* ball, int32_t S, float* temb,
                         float* table, void* stream) {
  if (!times || !w1 || !b1 || !w2 || !b2 || !wall || !ball || !temb || !table) return fail(nullptr, IRSDE_ERR_INVALID, "null argument");
  if (family != 0 && family != 1) return fail(nullptr, IRSDE_ERR_INVALID, "family must be 0 (ConditionalUNet) or 1 (NAFNet)");
  if (rows < 1 || S < 1 || width < 4 || width % 2) return fail(nullptr, IRSDE_ERR_INVALID, "bad shape");
  if (int rc = check_shape_limits(nullptr, rows, "rows", 1, 1)) return rc;
  if ((family == 0 ? time_mlp_smem(width) : naf_time_mlp_smem(width)) > kTimeMlpSmemMax)
    return fail(nullptr, IRSDE_ERR_UNSUPPORTED, "the time MLP of this width needs more than 48 KB of shared memory");
  Scratch sc(nullptr, (cudaStream_t)stream);
  if (family == 0) {
    launch_time_table(times, rows, width, w1, b1, w2, b2, wall, ball, S, temb, table, sc.st);
  } else {
    launch_naf_time_gate(times, rows, width, w1, b1, w2, b2, temb, sc.st);
    launch_time_rows(temb, rows, 2 * width, wall, ball, S, table, sc.st);
  }
  return sc.finish(IRSDE_OK, "time embedding failed");
}

int irsde_prep_input(int32_t precision, const float* xt, const float* cond, float* out, int32_t B, int32_t C, int32_t H, int32_t W,
                     int32_t Hp, int32_t Wp, int32_t pitch, int32_t conditional, int32_t zero_pad, int32_t pad_top, int32_t pad_left,
                     int32_t row_pix, int32_t img_rows, void* stream) {
  if (!xt || !out || (conditional && !cond)) return fail(nullptr, IRSDE_ERR_INVALID, "null argument");
  if (precision < IRSDE_PREC_FP32 || precision > IRSDE_PREC_FP32X3) return fail(nullptr, IRSDE_ERR_INVALID, "bad precision");
  if (B < 1 || C < 1 || H < 1 || W < 1 || Hp < H || Wp < W) return fail(nullptr, IRSDE_ERR_INVALID, "bad shape");
  if (!zero_pad && (Hp - H >= H || Wp - W >= W))
    return fail(nullptr, IRSDE_ERR_INVALID, "reflect padding of H - 1 or more rows / columns would read outside the image");
  if (pitch < C * (conditional ? 2 : 1)) return fail(nullptr, IRSDE_ERR_INVALID, "pitch below the packed channels");
  if (row_pix == 0 && (img_rows || pad_top || pad_left)) return fail(nullptr, IRSDE_ERR_INVALID, "a border needs row_pix and img_rows");
  if (row_pix != 0 && (pad_top < 0 || pad_left < 0 || (long long)pad_top + Hp > img_rows || (long long)pad_left + Wp > row_pix))
    return fail(nullptr, IRSDE_ERR_INVALID, "the padded image does not fit inside its border");
  const long long n = (long long)B * (row_pix ? (long long)img_rows * row_pix : (long long)Hp * Wp) * pitch;
  Scratch sc(nullptr, (cudaStream_t)stream);
  auto run = [&](auto* o) {
    launch_prep_input(xt, cond, o, B, C, H, W, Hp, Wp, pitch, conditional ? 1 : 0, sc.st, pad_top, pad_left, row_pix, img_rows,
                      zero_pad ? 1 : 0);
  };
  if (precision == IRSDE_PREC_BF16) {
    bf16* ob = sc.inout(out, n);
    if (!ob) return sc.oom();
    run(ob);
  } else {
    run(out);
  }
  return sc.finish(IRSDE_OK, "prep_input failed");
}

// ---- image conversion / metrics (stateless) ----------------------------------------------------------------
static int img_args_ok(const void* a, const void* b, int B, int C, int H, int W) {
  if (!a || !b || B < 1 || H < 1 || W < 1 || (C != 1 && C != 3)) return fail(nullptr, IRSDE_ERR_INVALID, "bad image argument");
  return check_shape_limits(nullptr, B, "B", 1, 1);  // the image kernels index pixels in long long: only B is limited
}
static int img_launch_status(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(nullptr, IRSDE_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
  return IRSDE_OK;
}
int irsde_tensor2img_u8(const float* chw, uint8_t* hwc, int32_t B, int32_t C, int32_t H, int32_t W, double lo, double hi,
                        void* stream) {
  if (int rc = img_args_ok(chw, hwc, B, C, H, W)) return rc;
  if (!(hi > lo)) return fail(nullptr, IRSDE_ERR_INVALID, "min_max must be increasing");
  launch_tensor2img(chw, hwc, B, C, H, W, lo, hi, (cudaStream_t)stream);
  return img_launch_status("tensor2img");
}
int irsde_img2tensor_u8(const uint8_t* hwc, float* chw, int32_t B, int32_t C, int32_t H, int32_t W, void* stream) {
  if (int rc = img_args_ok(hwc, chw, B, C, H, W)) return rc;
  launch_img2tensor(hwc, chw, B, C, H, W, (cudaStream_t)stream);
  return img_launch_status("img2tensor");
}
int irsde_sqerr_u8(const uint8_t* a, const uint8_t* b, int32_t B, int32_t H, int32_t W, int32_t C, int32_t crop, uint64_t* sums,
                   void* stream) {
  if (int rc = img_args_ok(a, b, B, C, H, W)) return rc;
  if (!sums || crop < 0 || H - 2 * crop < 1 || W - 2 * crop < 1) return fail(nullptr, IRSDE_ERR_INVALID, "bad crop / output");
  launch_sqerr_u8(a, b, B, H, W, C, crop, (unsigned long long*)sums, (cudaStream_t)stream);
  return img_launch_status("sqerr_u8");
}
int64_t irsde_ssim_workspace(int32_t B, int32_t H, int32_t W, int32_t C, int32_t crop) {
  if (B < 1 || crop < 0 || H - 2 * crop < 11 || W - 2 * crop < 11) return 0;
  return (int64_t)B * ssim_partial_count(H, W, C, crop);
}
int irsde_ssim_u8(const uint8_t* a, const uint8_t* b, int32_t B, int32_t H, int32_t W, int32_t C, int32_t crop, double* workspace,
                  double* ssim, void* stream) {
  if (int rc = img_args_ok(a, b, B, C, H, W)) return rc;
  if (!workspace || !ssim || crop < 0 || H - 2 * crop < 11 || W - 2 * crop < 11)
    return fail(nullptr, IRSDE_ERR_INVALID, "SSIM needs at least 11x11 pixels after cropping");
  launch_ssim_u8(a, b, B, H, W, C, crop, workspace, ssim, (cudaStream_t)stream);
  return img_launch_status("ssim_u8");
}

}  // extern "C"
