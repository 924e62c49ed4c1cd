// HBM-bound kernels around the attention sites of the UNet: channel LayerNorm, LinearAttention
// (module_util.py:150-178) and the full softmax Attention of the denoising-sde variant (:182-204).
// All loads/stores are 128-bit vectors over the NHWC channel dimension; math is fp32.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace irsde {

// Newer kernels of this file, one bit each (IRSDE_HBM_NEW; 0 = the previous kernels, kept for A/B runs and as the reference
// the newer ones are compared against).  IRSDE_HBM_DEFAULT is the default setting.
//   1 = LayerNorm with compile-time lane geometry     2 = la_combine with 128-bit record loads
//   4 = la_fold with 16 output rows per block          8 = k/v pass with warp-shuffle, branch-free softmax statistics
//  16 = la_combine with the records spread over 8 warps (takes precedence over 2)
#define IRSDE_HBM_DEFAULT 31
#define IRSDE_LN_PP_DEFAULT 2
static int hbm_mask_from_env() {
  const char* e = getenv("IRSDE_HBM_NEW");
  return e && *e ? atoi(e) : IRSDE_HBM_DEFAULT;
}
static const int g_hbm_new = hbm_mask_from_env();
static int ln_pp_from_env() {  // pixels per lane group of layernorm_geo_kernel (rows of <= 2 vectors per lane)
  const char* e = getenv("IRSDE_LN_PP");
  return e && *e ? (*e == '1' ? 1 : 2) : IRSDE_LN_PP_DEFAULT;
}
static const int g_ln_pp = ln_pp_from_env();

// accurate exp in parity (fp32) mode, fast exp in perf (bf16) mode
template <typename T>
__device__ __forceinline__ float fexp(float x);
template <>
__device__ __forceinline__ float fexp<float>(float x) { return expf(x); }
template <>
__device__ __forceinline__ float fexp<bf16>(float x) { return __expf(x); }

// ---- 16-byte vector access over float / bf16 ----------------------------------------------------
template <typename T>
struct VecIO;
template <>
struct VecIO<float> {
  static constexpr int N = 4;
  typedef float4 Raw;  // a vector as loaded (unpacked late to keep registers down)
  static __device__ __forceinline__ Raw load_raw(const float* p) { return *reinterpret_cast<const float4*>(p); }
  static __device__ __forceinline__ void unpack(const Raw& t, float* v) { v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
  static __device__ __forceinline__ void load(const float* p, float* v) {
    float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
  static __device__ __forceinline__ void store(float* p, const float* v) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
};
template <>
struct VecIO<bf16> {
  static constexpr int N = 8;
  typedef uint4 Raw;
  static __device__ __forceinline__ Raw load_raw(const bf16* p) { return *reinterpret_cast<const uint4*>(p); }
  static __device__ __forceinline__ void unpack(const Raw& t, float* v) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) { v[2 * i] = __low2float(h[i]); v[2 * i + 1] = __high2float(h[i]); }
  }
  static __device__ __forceinline__ void load(const bf16* p, float* v) {
    uint4 t = *reinterpret_cast<const uint4*>(p);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) { v[2 * i] = __low2float(h[i]); v[2 * i + 1] = __high2float(h[i]); }
  }
  static __device__ __forceinline__ void store(bf16* p, const float* v) {
    uint4 t;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = t;
  }
};

// =============================================================================================
// channel LayerNorm: (x-mean)*rsqrt(var_biased+1e-5)*g (+ residual)   module_util.py:70-79,20-26
// `lpp` lanes cooperate on one pixel (lpp = 32 for wide C, fewer for narrow C so a warp covers
// several pixels with full 16-byte loads); the row is held in registers between the two passes.
// =============================================================================================
template <typename T, int MAXV>
__global__ void __launch_bounds__(256) layernorm_vec_kernel(const T* __restrict__ x, int x_pitch,
                                                            const float* __restrict__ g, const T* __restrict__ res,
                                                            int res_pitch, T* __restrict__ out, int out_pitch,
                                                            long long npix, int C, int lpp, LnMod mod) {
  PDL_ENTRY();
  constexpr int N = VecIO<T>::N;
  const int lane = threadIdx.x & 31;
  const int ppw = 32 / lpp;
  const long long warp_g = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long pix = warp_g * ppw + lane / lpp;
  const int sub = lane % lpp;
  const int nvec = C / N;
  const bool valid = pix < npix;
  float v[MAXV][N];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int i = sub + k * lpp;
    if (valid && i < nvec) {
      VecIO<T>::load(x + pix * x_pitch + i * N, v[k]);
#pragma unroll
      for (int j = 0; j < N; ++j) s += v[k][j];
    } else {
#pragma unroll
      for (int j = 0; j < N; ++j) v[k][j] = 0.f;
    }
  }
  for (int o = lpp >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)C;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int i = sub + k * lpp;
    if (i < nvec) {
#pragma unroll
      for (int j = 0; j < N; ++j) { float d = v[k][j] - mean; q += d * d; }
    }
  }
  for (int o = lpp >> 1; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = 1.0f / sqrtf(q / (float)C + 1e-5f);
  if (!valid) return;
  const float* mrow = nullptr;  // NAFBlock time modulation: y * (scale + 1) + shift  (DenoisingNAFNet_arch.py:62-63,75-76)
  if (mod.ss) mrow = mod.ss + (long long)((mod.t_ptr ? *mod.t_ptr : 0) + (int)(pix / mod.pix_per_img) * mod.img_stride) * mod.S;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int i = sub + k * lpp;
    if (i < nvec) {
      float y[N], r[N];
#pragma unroll
      for (int j = 0; j < N; j += 4) {
        float4 gg = *reinterpret_cast<const float4*>(g + i * N + j);
        y[j] = (v[k][j] - mean) * rstd * gg.x;
        y[j + 1] = (v[k][j + 1] - mean) * rstd * gg.y;
        y[j + 2] = (v[k][j + 2] - mean) * rstd * gg.z;
        y[j + 3] = (v[k][j + 3] - mean) * rstd * gg.w;
      }
      if (mrow) {
#pragma unroll
        for (int j = 0; j < N; ++j) y[j] = y[j] * (mrow[mod.off_scale + i * N + j] + 1.0f) + mrow[mod.off_shift + i * N + j];
      }
      if (res) {
        VecIO<T>::load(res + pix * res_pitch + i * N, r);
#pragma unroll
        for (int j = 0; j < N; ++j) y[j] += r[j];
      }
      VecIO<T>::store(out + pix * out_pitch + i * N, y);
    }
  }
}

// LayerNorm with compile-time geometry.  The kernel above is bound by the instructions it ISSUES per 16-byte vector (run-time lane geometry: integer divisions, shuffle loops
// with branches, per-vector bounds checks, IEEE divide / sqrt slow-path scaffolding), not by bytes in flight.  Here the
// geometry is a template parameter (C == N * LPP * MAXV exactly, lane / LPP are shifts, shuffle trees unrolled), a lane
// group owns PP pixels so the gain row and the address set-up are shared, the residual row is requested together with x,
// out-of-range pixels are clamped to the last valid one (loads stay unpredicated, only the store is guarded), and the bf16
// (perf) instantiation uses mean = s * (1/C) and rsqrtf.  The fp32 instantiations keep the IEEE forms and the operation
// order of the kernel above, so fp32 / fp32x3 results are unchanged bit for bit.
template <typename T, int MAXV, int LPP, int PP>
__global__ void __launch_bounds__(256, (MAXV * PP <= 2 ? 4 : (MAXV * PP <= 4 ? 2 : 1))) layernorm_geo_kernel(const T* __restrict__ x, int x_pitch, const float* __restrict__ g,
                                                            const T* __restrict__ res, int res_pitch, T* __restrict__ out,
                                                            int out_pitch, long long npix, int C, float inv_C, LnMod mod) {
  PDL_ENTRY();
  constexpr int N = VecIO<T>::N;
  constexpr int PPW = 32 / LPP;               // pixels per warp and pass
  constexpr bool FAST = sizeof(T) == 2;
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPP;
  const long long pix0 = ((long long)blockIdx.x * PP * 8 + (threadIdx.x >> 5)) * PPW + lane / LPP;
  float v[PP][MAXV][N];
  typename VecIO<T>::Raw r[PP][MAXV];
  long long pixc[PP];
  bool valid[PP];
#pragma unroll
  for (int p = 0; p < PP; ++p) {
    const long long pix = pix0 + (long long)p * 8 * PPW;
    valid[p] = pix < npix;
    pixc[p] = valid[p] ? pix : npix - 1;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) VecIO<T>::load(x + pixc[p] * x_pitch + (sub + k * LPP) * N, v[p][k]);
  }
  if (res) {
#pragma unroll
    for (int p = 0; p < PP; ++p)
#pragma unroll
      for (int k = 0; k < MAXV; ++k) r[p][k] = VecIO<T>::load_raw(res + pixc[p] * res_pitch + (sub + k * LPP) * N);
  }
  float gg[MAXV][N];
#pragma unroll
  for (int k = 0; k < MAXV; ++k)
#pragma unroll
    for (int j = 0; j < N; j += 4) {
      const float4 t = *reinterpret_cast<const float4*>(g + (sub + k * LPP) * N + j);
      gg[k][j] = t.x; gg[k][j + 1] = t.y; gg[k][j + 2] = t.z; gg[k][j + 3] = t.w;
    }
  float rstd[PP];
#pragma unroll
  for (int p = 0; p < PP; ++p) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k)
#pragma unroll
      for (int j = 0; j < N; ++j) s += v[p][k][j];
#pragma unroll
    for (int o = LPP >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = FAST ? s * inv_C : s / (float)C;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k)
#pragma unroll
      for (int j = 0; j < N; ++j) { v[p][k][j] -= mean; q += v[p][k][j] * v[p][k][j]; }
#pragma unroll
    for (int o = LPP >> 1; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    rstd[p] = FAST ? rsqrtf(q * inv_C + 1e-5f) : 1.0f / sqrtf(q / (float)C + 1e-5f);
  }
#pragma unroll
  for (int p = 0; p < PP; ++p) {
    const float* mrow = nullptr;  // NAFBlock time modulation: y * (scale + 1) + shift  (DenoisingNAFNet_arch.py:62-63,75-76)
    if (mod.ss) mrow = mod.ss + (long long)((mod.t_ptr ? *mod.t_ptr : 0) + (int)(pixc[p] / mod.pix_per_img) * mod.img_stride) * mod.S;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      const int c0 = (sub + k * LPP) * N;
      float y[N];
#pragma unroll
      for (int j = 0; j < N; ++j) y[j] = v[p][k][j] * rstd[p] * gg[k][j];
      if (mrow) {
#pragma unroll
        for (int j = 0; j < N; ++j) y[j] = y[j] * (mrow[mod.off_scale + c0 + j] + 1.0f) + mrow[mod.off_shift + c0 + j];
      }
      if (res) {
        float rr[N];
        VecIO<T>::unpack(r[p][k], rr);
#pragma unroll
        for (int j = 0; j < N; ++j) y[j] += rr[j];
      }
      if (valid[p]) VecIO<T>::store(out + pixc[p] * out_pitch + c0, y);
    }
  }
}

// scalar fallback (any C / alignment): one warp per pixel, three cached passes
template <typename T>
__global__ void layernorm_scalar_kernel(const T* __restrict__ x, int x_pitch, const float* __restrict__ g,
                                        const T* __restrict__ res, int res_pitch, T* __restrict__ out, int out_pitch,
                                        long long npix, int C, LnMod mod) {
  PDL_ENTRY();
  int lane = threadIdx.x & 31;
  long long pix = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (pix >= npix) return;
  const T* xr = x + pix * x_pitch;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += to_f(xr[c]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  float mean = s / (float)C;
  float v = 0.f;
  for (int c = lane; c < C; c += 32) { float d = to_f(xr[c]) - mean; v += d * d; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  float rstd = 1.0f / sqrtf(v / (float)C + 1e-5f);
  T* orow = out + pix * out_pitch;
  const T* rr = res ? res + pix * res_pitch : nullptr;
  const float* mrow = nullptr;
  if (mod.ss) mrow = mod.ss + (long long)((mod.t_ptr ? *mod.t_ptr : 0) + (int)(pix / mod.pix_per_img) * mod.img_stride) * mod.S;
  for (int c = lane; c < C; c += 32) {
    float y = (to_f(xr[c]) - mean) * rstd * g[c];
    if (mrow) y = y * (mrow[mod.off_scale + c] + 1.0f) + mrow[mod.off_shift + c];
    if (rr) y += to_f(rr[c]);
    orow[c] = from_f<T>(y);
  }
}

template <typename T>
void launch_layernorm(const T* x, int x_pitch, const float* g, const T* res, int res_pitch, T* out, int out_pitch,
                      long long npix, int C, cudaStream_t st, const LnMod* modp) {
  LnMod mod;
  memset(&mod, 0, sizeof mod);
  if (modp) mod = *modp;
  if (mod.pix_per_img <= 0) mod.pix_per_img = 1;
  constexpr int N = VecIO<T>::N;
  bool vec_ok = C % N == 0 && x_pitch % N == 0 && out_pitch % N == 0 && ((uintptr_t)x % 16 == 0) &&
                ((uintptr_t)out % 16 == 0) && ((uintptr_t)g % 16 == 0) &&
                (!res || (res_pitch % N == 0 && (uintptr_t)res % 16 == 0));
  int nvec = C / N;
  int lpp = 1;
  while (lpp * 2 <= 32 && lpp * 2 <= nvec) lpp *= 2;
  int per_lane = vec_ok ? (nvec + lpp - 1) / lpp : 999;
  if (!vec_ok || per_lane > 16) {
    const int warps = 8;
    pdl_launch(layernorm_scalar_kernel<T>, (unsigned)((npix + warps - 1) / warps), warps * 32, 0, st, x, x_pitch, g, res, res_pitch,
                                                                                            out, out_pitch, npix, C, mod);
    return;
  }
  const int warps = 8;
  long long pix_per_block = (long long)warps * (32 / lpp);
  if ((g_hbm_new & 1) && nvec == lpp * per_lane && (per_lane & (per_lane - 1)) == 0 && lpp >= 8 && npix > 0) {
    // exact geometry: C == N * LPP * MAXV.  PP pixels per lane group (IRSDE_LN_PP, default 2) while the row fits 2 vectors per lane.
#define LN_GEO(MV, LP, PPX)                                                                                              \
  pdl_launch(layernorm_geo_kernel<T, MV, LP, PPX>, (unsigned)((npix + pix_per_block * PPX - 1) / (pix_per_block * PPX)),   \
             warps * 32, 0, st, x, x_pitch, g, res, res_pitch, out, out_pitch, npix, C, 1.0f / (float)C, mod)
#define LN_GEO_PP(MV, LP)                \
  do {                                   \
    if (g_ln_pp == 2) LN_GEO(MV, LP, 2); \
    else LN_GEO(MV, LP, 1);              \
    return;                              \
  } while (0)
    if (lpp == 8 && per_lane == 1) LN_GEO_PP(1, 8);
    if (lpp == 16 && per_lane == 1) LN_GEO_PP(1, 16);
    if (lpp == 32 && per_lane == 1) LN_GEO_PP(1, 32);
    if (lpp == 32 && per_lane == 2) LN_GEO_PP(2, 32);
    if (lpp == 32 && per_lane == 4) { LN_GEO(4, 32, 1); return; }
    if (lpp == 32 && per_lane == 8 && sizeof(T) == 4) { LN_GEO(8, 32, 1); return; }
#undef LN_GEO_PP
#undef LN_GEO
  }
  unsigned grid = (unsigned)((npix + pix_per_block - 1) / pix_per_block);
#define LN_LAUNCH(MV) \
  pdl_launch(layernorm_vec_kernel<T, MV>, grid, warps * 32, 0, st, x, x_pitch, g, res, res_pitch, out, out_pitch, npix, C, lpp, mod)
  if (per_lane <= 1) LN_LAUNCH(1);
  else if (per_lane <= 2) LN_LAUNCH(2);
  else if (per_lane <= 4) LN_LAUNCH(4);
  else if (per_lane <= 8) LN_LAUNCH(8);
  else LN_LAUNCH(16);
#undef LN_LAUNCH
}
template void launch_layernorm<float>(const float*, int, const float*, const float*, int, float*, int, long long, int,
                                      cudaStream_t, const LnMod*);
template void launch_layernorm<bf16>(const bf16*, int, const float*, const bf16*, int, bf16*, int, long long, int,
                                     cudaStream_t, const LnMod*);

// =============================================================================================
// LinearAttention core (module_util.py:163-177).  heads=4, dim_head=32 (fixed by the reference).
// qkv channel layout: [q(4x32) | k(4x32) | v(4x32)], head h = channels h*32..h*32+31 of each third.
//   pass A (la_kv): each block streams chunks of 64 pixels of ONE image, all 4 heads, keeping running
//           (max, sum, ctx[32x32]) per head with the online-softmax rescale; one partial per block
//   pass B (la_combine): merge the per-block partials: ctx[d][e] = sum_n softmax_n(k)[d,n] v[e,n] / N
//   pass C (la_out): per pixel/head: q = softmax_d(q) * 32^-.5 ; out[e] = sum_d ctx[d][e] q[d]
// =============================================================================================
static const int LA_PIX = 64;               // pixels per chunk
static const int LA_REC = 4 * (64 + 1024);  // floats per partial record (4 heads x (m[32], s[32], ctx[32][32]))
static const int LA_MAXBLK = 64;            // partial records per image

static int la_blocks_per_image(int B, int N) {
  int nchunks = (N + LA_PIX - 1) / LA_PIX;
  // The partition must not depend on the batch size: a batch-sharded run has to reproduce the unsharded one bit for
  // bit (fp32 summation order).  37 blocks per image = one full wave of 2 resident blocks/SM at 8 images per GPU.
  (void)B;
  int nblk = 37;
  if (nblk > LA_MAXBLK) nblk = LA_MAXBLK;
  if (nblk > nchunks) nblk = nchunks;
  return nblk < 1 ? 1 : nblk;
}
size_t linattn_partial_floats(int B, int N) { return (size_t)B * LA_MAXBLK * LA_REC; }

template <typename T>
__global__ void __launch_bounds__(256) la_kv_kernel(const T* __restrict__ qkv, int pitch, float* __restrict__ part,
                                                    int N, int nchunks, int nblk) {
  PDL_ENTRY();
  extern __shared__ __align__(16) float la_sm[];
  float (*ks)[128] = reinterpret_cast<float (*)[128]>(la_sm);               // [64][128] k -> p
  float (*vs)[128] = reinterpret_cast<float (*)[128]>(la_sm + LA_PIX * 128);  // [64][128]
  float* m_run = la_sm + 2 * LA_PIX * 128;  // [128]
  float* s_run = m_run + 128;               // [128]
  float* alpha_s = s_run + 128;             // [128]
  float* red = alpha_s + 128;               // [2][128] scratch
  constexpr int NV = VecIO<T>::N;
  const int tid = threadIdx.x, b = blockIdx.y, blk = blockIdx.x;
  if (tid < 128) { m_run[tid] = -INFINITY; s_run[tid] = 0.f; }
  const int h = tid >> 6, d = (tid & 63) >> 1, e0 = (tid & 1) * 16;
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = 0.f;
  const int c = tid & 127, half = tid >> 7;
  const int c0 = (int)(((long long)nchunks * blk) / nblk), c1 = (int)(((long long)nchunks * (blk + 1)) / nblk);
  for (int ch = c0; ch < c1; ++ch) {
    const int n0 = ch * LA_PIX;
    __syncthreads();  // previous chunk fully consumed
    // ---- load k,v (256 contiguous channels per pixel) with 16-byte vectors
    constexpr int VPP = 256 / NV;  // vectors per pixel
    for (int i = tid; i < LA_PIX * VPP; i += 256) {
      const int n = i / VPP, j = i - n * VPP;
      float tmp[NV];
      const bool ok = n0 + n < N;
      if (ok) VecIO<T>::load(qkv + ((long long)b * N + n0 + n) * pitch + 128 + j * NV, tmp);
      const int cc = j * NV;  // 0..255 : [0,128) = k, [128,256) = v
#pragma unroll
      for (int q = 0; q < NV; ++q) {
        if (cc < 128) ks[n][cc + q] = ok ? tmp[q] : -INFINITY;
        else vs[n][cc - 128 + q] = ok ? tmp[q] : 0.f;
      }
    }
    __syncthreads();
    // ---- per-channel running max / exp / sum (online softmax over the pixel axis)
    float mx = -INFINITY;
#pragma unroll 8
    for (int n = half * 32; n < half * 32 + 32; ++n) mx = fmaxf(mx, ks[n][c]);
    red[half * 128 + c] = mx;
    __syncthreads();
    const float m_old = m_run[c];
    const float m_new = fmaxf(m_old, fmaxf(red[c], red[128 + c]));
    float ps = 0.f;
#pragma unroll 8
    for (int n = half * 32; n < half * 32 + 32; ++n) {
      float p = fexp<T>(ks[n][c] - m_new);
      ks[n][c] = p;
      ps += p;
    }
    __syncthreads();  // everyone has read red[] / m_run
    red[half * 128 + c] = ps;
    __syncthreads();
    if (half == 0) {
      const float al = fexp<T>(m_old - m_new);  // exp(-inf) = 0 on the first chunk
      alpha_s[c] = al;
      s_run[c] = s_run[c] * al + red[c] + red[128 + c];
      m_run[c] = m_new;
    }
    __syncthreads();
    // ---- ctx[h][d][e0..e0+15] += sum_n p[n][h*32+d] * v[n][h*32+e]
    const float al = alpha_s[h * 32 + d];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] *= al;
#pragma unroll 4
    for (int n = 0; n < LA_PIX; ++n) {
      const float p = ks[n][h * 32 + d];
      const float4* vp = reinterpret_cast<const float4*>(&vs[n][h * 32 + e0]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float4 vv = vp[j];
        acc[4 * j] += p * vv.x;
        acc[4 * j + 1] += p * vv.y;
        acc[4 * j + 2] += p * vv.z;
        acc[4 * j + 3] += p * vv.w;
      }
    }
  }
  __syncthreads();
  float* rec = part + ((long long)b * LA_MAXBLK + blk) * LA_REC;
  if (tid < 128) {
    const int hh = tid >> 5, dd = tid & 31;
    rec[hh * 1088 + dd] = m_run[tid];
    rec[hh * 1088 + 32 + dd] = s_run[tid];
  }
  float* cp = rec + h * 1088 + 64 + d * 32 + e0;
#pragma unroll
  for (int j = 0; j < 16; j += 4) *reinterpret_cast<float4*>(cp + j) = make_float4(acc[j], acc[j + 1], acc[j + 2], acc[j + 3]);
}

// One block = 256 ctx entries (8 d-rows x 32 e) of one (image, head); the loops over the <= 64 partial records are fully
// unrolled so that all their loads are in flight at once: the kernel is pure dependent-load latency.  Same arithmetic and summation order per entry as before (bit-identical ctx).
__global__ void __launch_bounds__(256) la_combine_kernel(const float* __restrict__ part, float* __restrict__ ctx,
                                                         int N, int nblk) {
  PDL_ENTRY();
  const int bh = blockIdx.x >> 2, b = bh >> 2, h = bh & 3, tid = (blockIdx.x & 3) * 256 + threadIdx.x;
  const int d = tid >> 5;
  const float* base = part + (long long)b * LA_MAXBLK * LA_REC + h * 1088;
  float mk[LA_MAXBLK];
#pragma unroll
  for (int k = 0; k < LA_MAXBLK; ++k) mk[k] = k < nblk ? base[(long long)k * LA_REC + d] : -INFINITY;
  float M = -INFINITY;
#pragma unroll
  for (int k = 0; k < LA_MAXBLK; ++k) M = fmaxf(M, mk[k]);
  float S = 0.f, acc = 0.f;
#pragma unroll
  for (int k0 = 0; k0 < LA_MAXBLK; k0 += 16) {   // 16 records (32 loads) in flight per batch
    float sk[16], ck[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float* rec = base + (long long)(k0 + j) * LA_REC;
      sk[j] = (k0 + j) < nblk ? rec[32 + d] : 0.f;
      ck[j] = (k0 + j) < nblk ? rec[64 + tid] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      if (k0 + j < nblk) {
        const float w = expf(mk[k0 + j] - M);
        S += sk[j] * w;
        acc += ck[j] * w;
      }
    }
  }
  ctx[(long long)bh * 1024 + tid] = acc / S / (float)N;
}

// Wide-load merge.  la_combine_kernel above issues 192 scalar requests per thread (1 536 per block / SM): its time is the
// SM's outstanding-request limit, not latency of a single chain.  Here one WARP owns 4 d-rows of one
// (image, head) = 128 ctx entries as one float4 per lane: the 64 records' (m, s) for those rows come in as two float4 loads
// per lane and are shared through shared memory, and each record's ctx slice is ONE 128-bit request per lane, 32 records
// in flight.  Per entry the arithmetic and its order are those of la_combine_kernel (bit-identical ctx).
__global__ void __launch_bounds__(32) la_combine4_kernel(const float* __restrict__ part, float* __restrict__ ctx, int N, int nblk) {
  PDL_ENTRY();
  __shared__ __align__(16) float ms[LA_MAXBLK][4], ss[LA_MAXBLK][4];
  const int bh = blockIdx.x >> 3, b = bh >> 2, h = bh & 3, d0 = (blockIdx.x & 7) * 4;
  const int lane = threadIdx.x, dd = lane >> 3, e4 = (lane & 7) * 4;
  const float* base = part + (long long)b * LA_MAXBLK * LA_REC + h * 1088;
#pragma unroll
  for (int k = lane; k < LA_MAXBLK; k += 32) {
    float4 m4 = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY), s4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k < nblk) {
      m4 = *reinterpret_cast<const float4*>(base + (long long)k * LA_REC + d0);
      s4 = *reinterpret_cast<const float4*>(base + (long long)k * LA_REC + 32 + d0);
    }
    *reinterpret_cast<float4*>(ms[k]) = m4;
    *reinterpret_cast<float4*>(ss[k]) = s4;
  }
  __syncwarp();
  float M = -INFINITY;
#pragma unroll
  for (int k = 0; k < LA_MAXBLK; ++k) M = fmaxf(M, ms[k][dd]);
  const float* cbase = base + 64 + (d0 + dd) * 32 + e4;
  float S = 0.f;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int k0 = 0; k0 < LA_MAXBLK; k0 += 32) {
    float4 ck[32];
#pragma unroll
    for (int j = 0; j < 32; ++j)
      ck[j] = (k0 + j) < nblk ? *reinterpret_cast<const float4*>(cbase + (long long)(k0 + j) * LA_REC) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if (k0 + j < nblk) {
        const float w = expf(ms[k0 + j][dd] - M);
        S += ss[k0 + j][dd] * w;
        acc.x += ck[j].x * w;
        acc.y += ck[j].y * w;
        acc.z += ck[j].z * w;
        acc.w += ck[j].w * w;
      }
    }
  }
  const float fN = (float)N;
  *reinterpret_cast<float4*>(ctx + (long long)bh * 1024 + (d0 + dd) * 32 + e4) =
      make_float4(acc.x / S / fN, acc.y / S / fN, acc.z / S / fN, acc.w / S / fN);
}

// Merge with the records spread over warps.  la_combine4_kernel turned the request storm into 40 wide loads per lane, but
// what remains is ONE warp walking the <= 64 records in sequence (expf + 5 dependent FMAs each).
// Here the 8 warps of a block take records w, w + 8, ... (<= 8 each, all loads in flight at once), and warp 0 adds the 8
// partial (S, ctx) pairs in a fixed order.  The record partition does not depend on the batch, so batch-sharded runs stay
// bit-identical; the summation order differs from la_combine_kernel (fp32 rounding only).
__global__ void __launch_bounds__(256) la_combine8_kernel(const float* __restrict__ part, float* __restrict__ ctx, int N, int nblk) {
  PDL_ENTRY();
  __shared__ __align__(16) float ms[LA_MAXBLK][4], ss[LA_MAXBLK][4];
  __shared__ __align__(16) float4 pacc[8][32];
  __shared__ float pS[8][32];
  const int bh = blockIdx.x >> 3, b = bh >> 2, h = bh & 3, d0 = (blockIdx.x & 7) * 4;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, dd = lane >> 3, e4 = (lane & 7) * 4;
  const float* base = part + (long long)b * LA_MAXBLK * LA_REC + h * 1088;
  const float* cbase = base + 64 + (d0 + dd) * 32 + e4;
  float4 ck[LA_MAXBLK / 8];
#pragma unroll
  for (int j = 0; j < LA_MAXBLK / 8; ++j) {
    const int k = warp + 8 * j;
    ck[j] = k < nblk ? *reinterpret_cast<const float4*>(cbase + (long long)k * LA_REC) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (tid < LA_MAXBLK) {
    float4 m4 = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY), s4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (tid < nblk) {
      m4 = *reinterpret_cast<const float4*>(base + (long long)tid * LA_REC + d0);
      s4 = *reinterpret_cast<const float4*>(base + (long long)tid * LA_REC + 32 + d0);
    }
    *reinterpret_cast<float4*>(ms[tid]) = m4;
    *reinterpret_cast<float4*>(ss[tid]) = s4;
  }
  __syncthreads();
  float M = -INFINITY;
#pragma unroll
  for (int k = 0; k < LA_MAXBLK; ++k) M = fmaxf(M, ms[k][dd]);
  float S = 0.f;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int j = 0; j < LA_MAXBLK / 8; ++j) {
    const int k = warp + 8 * j;
    if (k < nblk) {
      const float w = expf(ms[k][dd] - M);
      S += ss[k][dd] * w;
      acc.x += ck[j].x * w;
      acc.y += ck[j].y * w;
      acc.z += ck[j].z * w;
      acc.w += ck[j].w * w;
    }
  }
  pacc[warp][lane] = acc;
  pS[warp][lane] = S;
  __syncthreads();
  if (warp == 0) {
    float St = pS[0][lane];
    float4 a = pacc[0][lane];
#pragma unroll
    for (int w = 1; w < 8; ++w) {
      const float4 t = pacc[w][lane];
      St += pS[w][lane];
      a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w;
    }
    const float fN = (float)N;
    *reinterpret_cast<float4*>(ctx + (long long)bh * 1024 + (d0 + dd) * 32 + e4) = make_float4(a.x / St / fN, a.y / St / fN, a.z / St / fN, a.w / St / fN);
  }
}

template <typename T>
__global__ void __launch_bounds__(256) la_out_kernel(const T* __restrict__ qkv, int pitch, const float* __restrict__ ctx,
                                                     T* __restrict__ hidden, int hid_pitch, int N) {
  PDL_ENTRY();
  __shared__ __align__(16) float cs[4][32][32];
  constexpr int NV = VecIO<T>::N;
  const int b = blockIdx.y, tid = threadIdx.x;
  for (int i = tid; i < 1024; i += 256)
    reinterpret_cast<float4*>(&cs[0][0][0])[i] = reinterpret_cast<const float4*>(ctx + (long long)b * 4096)[i];
  __syncthreads();
  const int h = tid >> 6;
  const int n = blockIdx.x * 64 + (tid & 63);
  if (n >= N) return;
  const T* row = qkv + ((long long)b * N + n) * pitch + h * 32;
  float q[32];
#pragma unroll
  for (int j = 0; j < 32; j += NV) VecIO<T>::load(row + j, q + j);
  float m = q[0];
#pragma unroll
  for (int dd = 1; dd < 32; ++dd) m = fmaxf(m, q[dd]);
  float s = 0.f;
#pragma unroll
  for (int dd = 0; dd < 32; ++dd) { q[dd] = fexp<T>(q[dd] - m); s += q[dd]; }
  const float sc = 0.17677669529663687f / s;  // softmax normaliser * 32^-0.5
  float o[32];
#pragma unroll
  for (int e = 0; e < 32; ++e) o[e] = 0.f;
#pragma unroll
  for (int dd = 0; dd < 32; ++dd) {
    const float qd = q[dd] * sc;
#pragma unroll
    for (int e = 0; e < 32; e += 4) {
      float4 cc = *reinterpret_cast<const float4*>(&cs[h][dd][e]);
      o[e] += cc.x * qd;
      o[e + 1] += cc.y * qd;
      o[e + 2] += cc.z * qd;
      o[e + 3] += cc.w * qd;
    }
  }
  T* orow = hidden + ((long long)b * N + n) * hid_pitch + h * 32;
#pragma unroll
  for (int j = 0; j < 32; j += NV) VecIO<T>::store(orow + j, o + j);
}

// ---------------------------------------------------------------------------------------------
// bf16 perf-mode version of pass A.  Same partial-record format, but the [64 px x 256 ch] k|v tile is
// streamed with double-buffered cp.async and the 32x32 context of every head is accumulated with
// warp-level mma.sync (m16n8k16, bf16 x bf16 -> fp32): ctx_h += P_h^T (32 x 64px) * V_h (64px x 32).
// Both operands are pixel-major in shared memory, so fragments come from ldmatrix.trans.
// Warp w owns head w/2 and d-rows 16*(w%2)..+15 (4 n-tiles of 8 e's => 16 fp32 accumulators / thread).
// ---------------------------------------------------------------------------------------------
static const int LAM_TP = 264;  // tile row pitch (bf16): 256 + 8 pad -> conflict-free ldmatrix
static const int LAM_PP = 136;  // P row pitch (bf16): 128 + 8 pad
static const size_t LAM_SMEM = (size_t)2 * LA_PIX * LAM_TP * 2 + (size_t)LA_PIX * LAM_PP * 2 + (128 * 3 + 4 * 128) * 4;

__device__ __forceinline__ void ldsm_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ float ex2_approx(float x) {  // 2^x, one MUFU (rel. error 2^-22; -inf -> +0)
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ void mma_bf16_16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                               uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// SHFL: the softmax statistics of a chunk stay inside a warp.  Lane (qtr = lane / 4, cpl = lane % 4) of warp w
// owns channel pairs w*4+cpl and 32+w*4+cpl on the 8 pixels px == qtr (mod 8): the running max / sum live in registers
// (replicated over the 8 qtr lanes), the cross-pixel max and sum are three xor-shuffles each, and the bf16x2 accesses
// (word = 4*px + pair mod 32) are bank-conflict free.  One chunk then needs TWO block barriers (tile landed / P and alpha
// visible to the MMA warps) instead of five: in the <false> form the per-chunk barrier chain, not memory, is the bound.
template <bool SHFL>
__global__ void __launch_bounds__(256) la_kv_mma_kernel(const bf16* __restrict__ qkv, int pitch, float* __restrict__ part,
                                                        int N, int nchunks, int nblk) {
  PDL_ENTRY();
  extern __shared__ __align__(16) uint8_t lam_sm[];
  bf16* tile = reinterpret_cast<bf16*>(lam_sm);                          // [2][64][LAM_TP]  (k | v)
  bf16* Ps = tile + 2 * LA_PIX * LAM_TP;                                 // [64][LAM_PP]
  float* m_run = reinterpret_cast<float*>(Ps + LA_PIX * LAM_PP);         // [128]
  float* s_run = m_run + 128;
  float* alpha_s = s_run + 128;
  float* red = alpha_s + 128;                                            // [4][128]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.y, blk = blockIdx.x;
  if (tid < 128) { m_run[tid] = -INFINITY; s_run[tid] = 0.f; }
  const int c0 = (int)(((long long)nchunks * blk) / nblk), c1 = (int)(((long long)nchunks * (blk + 1)) / nblk);
  const int h = warp >> 1, dbase = h * 32 + (warp & 1) * 16;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  auto issue_load = [&](int ch, int buf) {
    const int n0 = ch * LA_PIX;
    bf16* dst = tile + buf * LA_PIX * LAM_TP;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int v = tid + i * 256;      // 2048 16-byte vectors: 32 per pixel
      const int px = v >> 5, j = v & 31;
      bf16* d = dst + px * LAM_TP + j * 8;
      if (n0 + px < N) {
        const bf16* src = qkv + ((long long)b * N + n0 + px) * pitch + 128 + j * 8;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(d)), "l"(src));
      } else {
        *reinterpret_cast<uint4*>(d) = make_uint4(0, 0, 0, 0);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  // SHFL loader: the same 8 vectors per thread, but the 64-bit source address and the shared-memory address are set up ONCE
  // (vector i of a thread is pixel (tid / 32) + 8 i, channel vector tid % 32: a fixed pitch apart), and the k channels
  // (vector index < 16) of a pixel past the image get -1e30 (bf16 0xF14A) instead of 0: their exp is 0 and the max is
  // unaffected, so the statistics loops need no per-pixel bounds checks.  v rows past the image are zero as before.
  const int lpx0 = tid >> 5, lj = tid & 31;
  const bf16* const gsrc0 = qkv + ((long long)b * N + lpx0) * pitch + 128 + lj * 8;
  const long long gstep = (long long)8 * pitch;
  const uint32_t sdst0 = (uint32_t)__cvta_generic_to_shared(tile) + (uint32_t)((lpx0 * LAM_TP + lj * 8) * 2);
  const uint32_t kfill = lj < 16 ? 0xF14AF14Au : 0u;
  auto issue_load_lean = [&](int ch, int buf) {
    const int n0 = ch * LA_PIX;
    const bf16* src = gsrc0 + (long long)n0 * pitch;
    const uint32_t dst = sdst0 + (uint32_t)(buf * LA_PIX * LAM_TP * 2);
    if (n0 + LA_PIX <= N) {  // whole chunk inside the image (block-uniform): eight plain copies
#pragma unroll
      for (int i = 0; i < 8; ++i)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + (uint32_t)(i * 8 * LAM_TP * 2)), "l"(src + i * gstep));
    } else {
      const int left = N - n0 - lpx0;  // pixels lpx0 + 8 i with 8 i < left are inside the image
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (8 * i < left) {
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + (uint32_t)(i * 8 * LAM_TP * 2)), "l"(src + i * gstep));
        } else {
          asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(dst + (uint32_t)(i * 8 * LAM_TP * 2)), "r"(kfill) : "memory");
        }
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  if (c0 < c1) {
    if constexpr (SHFL) issue_load_lean(c0, 0);
    else issue_load(c0, 0);
  }
  const int cp2 = (tid & 63) * 2, qtr = tid >> 6;  // stats mapping: 2 channels x 16 pixels per thread
  const float LOG2E = 1.4426950408889634f;
  // SHFL mapping and register-resident running statistics: [0,1] = pair A (lo, hi channel), [2,3] = pair B
  const int sq = lane >> 2, pA = warp * 4 + (lane & 3), pB = 32 + pA;
  float mr[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY}, sr[4] = {0.f, 0.f, 0.f, 0.f};
  for (int ch = c0; ch < c1; ++ch) {
    const int buf = (ch - c0) & 1;
    const bf16* T0 = tile + buf * LA_PIX * LAM_TP;
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();  // tile[buf] landed; everyone is done with tile[buf^1] and Ps of the previous chunk
    if (ch + 1 < c1) {
      if constexpr (SHFL) issue_load_lean(ch + 1, buf ^ 1);
      else issue_load(ch + 1, buf ^ 1);
    }
    const int nvalid = min(LA_PIX, N - ch * LA_PIX);
    if constexpr (SHFL) {
      // branch-free: rows past the image hold k = -1e30 (see issue_load); ~13 instructions per bf16 pair
      float k[16][2];
      float mx[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const bf16* row = T0 + (i * 8 + sq) * LAM_TP;
        const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(row + 2 * pA);
        const __nv_bfloat162 c = *reinterpret_cast<const __nv_bfloat162*>(row + 2 * pB);
        k[i][0] = __low2float(a); k[i][1] = __high2float(a);
        k[8 + i][0] = __low2float(c); k[8 + i][1] = __high2float(c);
        mx[0] = fmaxf(mx[0], k[i][0]); mx[1] = fmaxf(mx[1], k[i][1]);
        mx[2] = fmaxf(mx[2], k[8 + i][0]); mx[3] = fmaxf(mx[3], k[8 + i][1]);
      }
      float mn[4], mnl[4], ps[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) mx[c] = fmaxf(mx[c], __shfl_xor_sync(0xffffffffu, mx[c], o));
        mn[c] = fmaxf(mr[c], mx[c]);
        mnl[c] = mn[c] * LOG2E;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        bf16* prow = Ps + (i * 8 + sq) * LAM_PP;
        const __nv_bfloat162 qa = __floats2bfloat162_rn(ex2_approx(fmaf(k[i][0], LOG2E, -mnl[0])), ex2_approx(fmaf(k[i][1], LOG2E, -mnl[1])));
        const __nv_bfloat162 qb = __floats2bfloat162_rn(ex2_approx(fmaf(k[8 + i][0], LOG2E, -mnl[2])), ex2_approx(fmaf(k[8 + i][1], LOG2E, -mnl[3])));
        ps[0] += __low2float(qa);   // sum the rounded values the MMA will actually use
        ps[1] += __high2float(qa);
        ps[2] += __low2float(qb);
        ps[3] += __high2float(qb);
        *reinterpret_cast<__nv_bfloat162*>(prow + 2 * pA) = qa;
        *reinterpret_cast<__nv_bfloat162*>(prow + 2 * pB) = qb;
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) {
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) ps[c] += __shfl_xor_sync(0xffffffffu, ps[c], o);
        const float a = ex2_approx((mr[c] - mn[c]) * LOG2E);  // 0 on the first chunk (mr = -inf)
        sr[c] = sr[c] * a + ps[c];
        mr[c] = mn[c];
        if (sq == 0) alpha_s[2 * (c < 2 ? pA : pB) + (c & 1)] = a;
      }
      __syncthreads();  // P and alpha visible to the MMA warps
    } else {
    // ---- per-channel max over the chunk
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int px = qtr * 16 + i;
      if (px < nvalid) {
        __nv_bfloat162 kk = *reinterpret_cast<const __nv_bfloat162*>(T0 + px * LAM_TP + cp2);
        mx0 = fmaxf(mx0, __low2float(kk));
        mx1 = fmaxf(mx1, __high2float(kk));
      }
    }
    red[qtr * 128 + cp2] = mx0;
    red[qtr * 128 + cp2 + 1] = mx1;
    __syncthreads();
    const float mo0 = m_run[cp2], mo1 = m_run[cp2 + 1];
    float mn0 = mo0, mn1 = mo1;
#pragma unroll
    for (int q = 0; q < 4; ++q) { mn0 = fmaxf(mn0, red[q * 128 + cp2]); mn1 = fmaxf(mn1, red[q * 128 + cp2 + 1]); }
    float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int px = qtr * 16 + i;
      __nv_bfloat162 pp = __floats2bfloat162_rn(0.f, 0.f);
      if (px < nvalid) {
        __nv_bfloat162 kk = *reinterpret_cast<const __nv_bfloat162*>(T0 + px * LAM_TP + cp2);
        pp = __floats2bfloat162_rn(exp2f((__low2float(kk) - mn0) * LOG2E), exp2f((__high2float(kk) - mn1) * LOG2E));
        ps0 += __low2float(pp);   // sum the rounded values the MMA will actually use
        ps1 += __high2float(pp);
      }
      *reinterpret_cast<__nv_bfloat162*>(Ps + px * LAM_PP + cp2) = pp;
    }
    __syncthreads();  // all reads of red (max) done
    red[qtr * 128 + cp2] = ps0;
    red[qtr * 128 + cp2 + 1] = ps1;
    __syncthreads();
    if (qtr == 0) {
      const float a0 = exp2f((mo0 - mn0) * LOG2E), a1 = exp2f((mo1 - mn1) * LOG2E);  // 0 on the first chunk
      alpha_s[cp2] = a0;
      alpha_s[cp2 + 1] = a1;
      s_run[cp2] = s_run[cp2] * a0 + red[cp2] + red[128 + cp2] + red[256 + cp2] + red[384 + cp2];
      s_run[cp2 + 1] = s_run[cp2 + 1] * a1 + red[cp2 + 1] + red[128 + cp2 + 1] + red[256 + cp2 + 1] + red[384 + cp2 + 1];
      m_run[cp2] = mn0;
      m_run[cp2 + 1] = mn1;
    }
    __syncthreads();
    }  // !SHFL
    // ---- rescale and accumulate: rows g / g+8 of this warp's 16 d-rows
    {
      const float al_lo = alpha_s[dbase + (lane >> 2)], al_hi = alpha_s[dbase + (lane >> 2) + 8];
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) { acc[nt][0] *= al_lo; acc[nt][1] *= al_lo; acc[nt][2] *= al_hi; acc[nt][3] *= al_hi; }
    }
    const uint32_t Pbase = (uint32_t)__cvta_generic_to_shared(Ps);
    const uint32_t Vbase = (uint32_t)__cvta_generic_to_shared(T0);
    const int mi = lane >> 3, r8 = lane & 7;  // ldmatrix: lane supplies row r8 of matrix mi
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const int k0 = ks * 16;
      uint32_t a0, a1, a2, a3;
      // A = P^T: matrices (k0-7,m0-7) (k0-7,m8-15) (k8-15,m0-7) (k8-15,m8-15) -> a0,a1,a2,a3 after transpose
      ldsm_x4_trans(Pbase + (uint32_t)(((k0 + (mi >> 1) * 8 + r8) * LAM_PP + dbase + (mi & 1) * 8) * 2), a0, a1, a2, a3);
#pragma unroll
      for (int np = 0; np < 2; ++np) {  // two pairs of n-tiles (16 e's each)
        uint32_t b0, b1, b2, b3;
        // B = V: matrices (k0-7,n0-7) (k8-15,n0-7) (k0-7,n8-15) (k8-15,n8-15)
        ldsm_x4_trans(Vbase + (uint32_t)(((k0 + (mi & 1) * 8 + r8) * LAM_TP + 128 + h * 32 + np * 16 + (mi >> 1) * 8) * 2), b0,
                      b1, b2, b3);
        mma_bf16_16816(acc[np * 2], a0, a1, a2, a3, b0, b1);
        mma_bf16_16816(acc[np * 2 + 1], a0, a1, a2, a3, b2, b3);
      }
    }
  }
  __syncthreads();
  float* rec = part + ((long long)b * LA_MAXBLK + blk) * LA_REC;
  if constexpr (SHFL) {
    if (sq == 0) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int chn = 2 * (c < 2 ? pA : pB) + (c & 1);
        rec[(chn >> 5) * 1088 + (chn & 31)] = mr[c];
        rec[(chn >> 5) * 1088 + 32 + (chn & 31)] = sr[c];
      }
    }
  } else if (tid < 128) {
    const int hh = tid >> 5, dd = tid & 31;
    rec[hh * 1088 + dd] = m_run[tid];
    rec[hh * 1088 + 32 + dd] = s_run[tid];
  }
  {
    const int g = lane >> 2, t4 = lane & 3, drow = (warp & 1) * 16 + g;
    float* cp = rec + h * 1088 + 64;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const int e = nt * 8 + t4 * 2;
      *reinterpret_cast<float2*>(cp + drow * 32 + e) = make_float2(acc[nt][0], acc[nt][1]);
      *reinterpret_cast<float2*>(cp + (drow + 8) * 32 + e) = make_float2(acc[nt][2], acc[nt][3]);
    }
  }
}

static bool g_la_attr_done = false;

template <typename T>
static void launch_la_kv(const T* qkv, int qkv_pitch, float* partial, int B, int N, int nchunks, int nblk, size_t smem,
                         cudaStream_t st);
template <>
void launch_la_kv<float>(const float* qkv, int qkv_pitch, float* partial, int B, int N, int nchunks, int nblk, size_t smem,
                         cudaStream_t st) {
  pdl_launch(la_kv_kernel<float>, dim3(nblk, B), 256, smem, st, qkv, qkv_pitch, partial, N, nchunks, nblk);
}
template <>
void launch_la_kv<bf16>(const bf16* qkv, int qkv_pitch, float* partial, int B, int N, int nchunks, int nblk, size_t smem,
                        cudaStream_t st) {
  if (qkv_pitch % 8 == 0 && ((uintptr_t)qkv % 16) == 0)
    if (g_hbm_new & 8) pdl_launch(la_kv_mma_kernel<true>, dim3(nblk, B), 256, LAM_SMEM, st, qkv, qkv_pitch, partial, N, nchunks, nblk);
    else pdl_launch(la_kv_mma_kernel<false>, dim3(nblk, B), 256, LAM_SMEM, st, qkv, qkv_pitch, partial, N, nchunks, nblk);
  else
    pdl_launch(la_kv_kernel<bf16>, dim3(nblk, B), 256, smem, st, qkv, qkv_pitch, partial, N, nchunks, nblk);
}

template <typename T>
void launch_linattn_ctx(const T* qkv, int qkv_pitch, float* partial, float* ctx, int B, int N, cudaStream_t st) {
  const int nchunks = (N + LA_PIX - 1) / LA_PIX;
  const int nblk = la_blocks_per_image(B, N);
  const size_t smem = (size_t)(2 * LA_PIX * 128 + 128 * 5) * sizeof(float);
  if (!g_la_attr_done) {
    cudaFuncSetAttribute(la_kv_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(la_kv_kernel<bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(la_kv_mma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LAM_SMEM);
    cudaFuncSetAttribute(la_kv_mma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LAM_SMEM);
    g_la_attr_done = true;
  }
  launch_la_kv<T>(qkv, qkv_pitch, partial, B, N, nchunks, nblk, smem, st);
  if (g_hbm_new & 16) pdl_launch(la_combine8_kernel, B * 4 * 8, 256, 0, st, partial, ctx, N, nblk);
  else if (g_hbm_new & 2) pdl_launch(la_combine4_kernel, B * 4 * 8, 32, 0, st, partial, ctx, N, nblk);
  else pdl_launch(la_combine_kernel, B * 4 * 4, 256, 0, st, partial, ctx, N, nblk);
}
template void launch_linattn_ctx<float>(const float*, int, float*, float*, int, int, cudaStream_t);
template void launch_linattn_ctx<bf16>(const bf16*, int, float*, float*, int, int, cudaStream_t);

template <typename T>
void launch_linattn(const T* qkv, int qkv_pitch, float* partial, float* ctx, T* hidden, int hid_pitch, int B, int N,
                    cudaStream_t st) {
  launch_linattn_ctx<T>(qkv, qkv_pitch, partial, ctx, B, N, st);
  pdl_launch(la_out_kernel<T>, dim3((N + 63) / 64, B), 256, 0, st, qkv, qkv_pitch, ctx, hidden, hid_pitch, N);
}
template void launch_linattn<float>(const float*, int, float*, float*, float*, int, int, int, cudaStream_t);
template void launch_linattn<bf16>(const bf16*, int, float*, float*, bf16*, int, int, int, cudaStream_t);

// Fold the per-image context into the to_out 1x1 weights so that pass C and the to_out conv become ONE
// per-image-weight GEMM on the (head-softmaxed) q:  y[px][c] = sum_k qs[px][k] * Mb[b][c][k],
// Mb[b][c][h*32+d] = sum_e Wout[c][h*32+e] * ctx[b][h][d][e]   (module_util.py:176-178 re-associated).
__global__ void la_fold_kernel(const float* __restrict__ ctx, const float* __restrict__ wout, bf16* __restrict__ Mb, int C) {
  PDL_ENTRY();
  __shared__ float cs[4][32][33];
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < 4096; i += blockDim.x) cs[i >> 10][(i >> 5) & 31][i & 31] = ctx[(long long)b * 4096 + i];
  __syncthreads();
  const int c = blockIdx.x * 2 + (threadIdx.x >> 7), k = threadIdx.x & 127;
  if (c >= C) return;
  const int h = k >> 5, d = k & 31;
  const float* w = wout + (long long)c * 128 + h * 32;
  float acc = 0.f;
#pragma unroll
  for (int e = 0; e < 32; ++e) acc += w[e] * cs[h][d][e];
  Mb[((long long)b * C + c) * 128 + k] = __float2bfloat16_rn(acc);
}
// 16-row fold: la_fold_kernel stages the image's whole 16 KB context in shared memory for TWO output rows (2 048 blocks x
// 16 KB of L2 reads at C = 512).  Here a block owns 16 output rows: a thread keeps ITS context row (h, d, 0..31) in
// registers (eight 128-bit loads, no staging), the 16 weight rows go through shared memory once, and all loads of the block
// are one round trip.  Same per-entry sum order as above (bit-identical Mb).
__global__ void __launch_bounds__(256) la_fold16_kernel(const float* __restrict__ ctx, const float* __restrict__ wout,
                                                        bf16* __restrict__ Mb, int C) {
  PDL_ENTRY();
  __shared__ __align__(16) float ws[16][128];
  const int b = blockIdx.y, cbase = blockIdx.x * 16, tid = threadIdx.x;
  const int k = tid & 127, h = k >> 5, cc = tid >> 7;
  float cr[32];
  const float4* cp = reinterpret_cast<const float4*>(ctx + (long long)b * 4096 + k * 32);  // ctx[b][h][d][0..31], k = h*32+d
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 t = cp[j];
    cr[4 * j] = t.x; cr[4 * j + 1] = t.y; cr[4 * j + 2] = t.z; cr[4 * j + 3] = t.w;
  }
#pragma unroll
  for (int i = tid; i < 16 * 32; i += 256) {   // 16 rows x 32 float4
    const int row = i >> 5, c = cbase + row;
    reinterpret_cast<float4*>(&ws[row][0])[i & 31] =
        c < C ? reinterpret_cast<const float4*>(wout + (long long)c * 128)[i & 31] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int row = i * 2 + cc, c = cbase + row;
    if (c >= C) continue;
    const float* w = &ws[row][h * 32];
    float acc = 0.f;
#pragma unroll
    for (int e = 0; e < 32; ++e) acc += w[e] * cr[e];
    Mb[((long long)b * C + c) * 128 + k] = __float2bfloat16_rn(acc);
  }
}
void launch_la_fold(const float* ctx, const float* wout, bf16* Mb, int B, int C, cudaStream_t st) {
  if (g_hbm_new & 4) pdl_launch(la_fold16_kernel, dim3((C + 15) / 16, B), 256, 0, st, ctx, wout, Mb, C);
  else pdl_launch(la_fold_kernel, dim3((C + 1) / 2, B), 256, 0, st, ctx, wout, Mb, C);
}

// =============================================================================================
// full softmax attention (module_util.py:192-204) - denoising-sde mid_attn only.
// thread per query, keys/values staged through shared memory, online softmax.
// =============================================================================================
template <typename T>
__global__ void __launch_bounds__(128) fullattn_kernel(const T* __restrict__ qkv, int pitch, T* __restrict__ hidden,
                                                       int hid_pitch, int N) {
  PDL_ENTRY();
  __shared__ __align__(16) float ks[64][32];
  __shared__ __align__(16) float vs[64][32];
  int bh = blockIdx.y, b = bh >> 2, h = bh & 3;
  int tid = threadIdx.x;
  int i = blockIdx.x * 128 + tid;
  bool valid = i < N;
  float q[32], acc[32];
  const float scale = 0.17677669529663687f;
  if (valid) {
    const T* row = qkv + ((long long)b * N + i) * pitch + h * 32;
#pragma unroll
    for (int d = 0; d < 32; ++d) q[d] = to_f(row[d]) * scale;
  } else {
#pragma unroll
    for (int d = 0; d < 32; ++d) q[d] = 0.f;
  }
#pragma unroll
  for (int d = 0; d < 32; ++d) acc[d] = 0.f;
  float m = -INFINITY, l = 0.f;
  for (int j0 = 0; j0 < N; j0 += 64) {
    __syncthreads();
    for (int t = tid; t < 64 * 32; t += 128) {
      int j = t >> 5, d = t & 31;
      float kv = 0.f, vv = 0.f;
      if (j0 + j < N) {
        const T* row = qkv + ((long long)b * N + j0 + j) * pitch;
        kv = to_f(row[128 + h * 32 + d]);
        vv = to_f(row[256 + h * 32 + d]);
      }
      ks[j][d] = kv;
      vs[j][d] = vv;
    }
    __syncthreads();
    int jmax = min(64, N - j0);
    for (int j = 0; j < jmax; ++j) {
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < 32; d += 4) {
        float4 k4 = *reinterpret_cast<const float4*>(&ks[j][d]);
        s += q[d] * k4.x + q[d + 1] * k4.y + q[d + 2] * k4.z + q[d + 3] * k4.w;
      }
      float mn = fmaxf(m, s);
      float alpha = expf(m - mn);
      float p = expf(s - mn);
      l = l * alpha + p;
#pragma unroll
      for (int d = 0; d < 32; d += 4) {
        float4 v4 = *reinterpret_cast<const float4*>(&vs[j][d]);
        acc[d] = acc[d] * alpha + p * v4.x;
        acc[d + 1] = acc[d + 1] * alpha + p * v4.y;
        acc[d + 2] = acc[d + 2] * alpha + p * v4.z;
        acc[d + 3] = acc[d + 3] * alpha + p * v4.w;
      }
      m = mn;
    }
  }
  if (valid) {
    T* orow = hidden + ((long long)b * N + i) * hid_pitch + h * 32;
#pragma unroll
    for (int d = 0; d < 32; ++d) orow[d] = from_f<T>(acc[d] / l);
  }
}
// ---------------------------------------------------------------------------------------------
// bf16 perf-mode version: flash attention on the tensor cores (module_util.py:192-204: q*32^-.5, sim = q^T k,
// softmax_j, out = attn v).  One CTA = 64 queries of one (image, head); warp w owns query rows 16w..16w+15.
// Per 64-key block: S = Q K^T by mma.sync m16n8k16 (bf16 x bf16 -> fp32; K rows are the natural col-major B operand),
// online softmax on the accumulator fragments (row max / sum across the 4 lanes of a quad by shuffles), P re-packed in
// registers as the bf16 A operand of the second product (the FlashAttention-2 register reuse, no smem round trip),
// O += P V with V fragments from ldmatrix.trans.  K and V tiles stream through a double-buffered cp.async ring.
// With d = 32 every mma.sync is surrounded by ~6 softmax / re-pack instructions, so the issue slots fill before the tensor
// pipe does.  It stays on mma.sync, whose operands come straight from registers.
// ---------------------------------------------------------------------------------------------
static const int FA_Q = 64, FA_K = 64, FA_P = 40;  // queries / keys per block; smem row pitch (32 + 8 pad, bf16)
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__global__ void __launch_bounds__(128) fullattn_mma_kernel(const bf16* __restrict__ qkv, int pitch, bf16* __restrict__ hidden,
                                                           int hid_pitch, int N) {
  PDL_ENTRY();
  __shared__ __align__(16) bf16 Qs[FA_Q * FA_P];
  __shared__ __align__(16) bf16 Ks[2][FA_K * FA_P];
  __shared__ __align__(16) bf16 Vs[2][FA_K * FA_P];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int bh = blockIdx.y, b = bh >> 2, h = bh & 3;
  const int q0 = blockIdx.x * FA_Q;
  const bf16* base = qkv + (long long)b * N * pitch + h * 32;

  auto load_kv = [&](int j0, int buf) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int v = tid + i * 128;  // 512 16-byte vectors: 64 keys x (4 of K + 4 of V)
      const int key = v >> 3, part = v & 7, isv = part >> 2, j = part & 3;
      bf16* d = (isv ? Vs[buf] : Ks[buf]) + key * FA_P + j * 8;
      if (j0 + key < N) {
        const bf16* src = base + (long long)(j0 + key) * pitch + (isv ? 256 : 128) + j * 8;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(d)), "l"(src));
      } else {
        *reinterpret_cast<uint4*>(d) = make_uint4(0, 0, 0, 0);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  // Q tile (zero rows past N)
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int v = tid + i * 128, row = v >> 2, j = v & 3;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (q0 + row < N) val = *reinterpret_cast<const uint4*>(base + (long long)(q0 + row) * pitch + j * 8);
    *reinterpret_cast<uint4*>(Qs + row * FA_P + j * 8) = val;
  }
  load_kv(0, 0);
  __syncthreads();
  // A fragments of Q: rows warp*16 + (0..15), two k-steps of 16 d's
  uint32_t qa[2][4];
  {
    const int mi = lane >> 3, r8 = lane & 7;  // matrices: (rows 0-7, d 0-7) (rows 8-15, d 0-7) (rows 0-7, d 8-15) (rows 8-15, d 8-15)
    const uint32_t qb = (uint32_t)__cvta_generic_to_shared(Qs);
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
      ldsm_x4(qb + (uint32_t)(((warp * 16 + (mi & 1) * 8 + r8) * FA_P + ks * 16 + (mi >> 1) * 8) * 2), qa[ks][0], qa[ks][1], qa[ks][2],
              qa[ks][3]);
  }
  float o[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
  const float SC = 0.17677669529663687f * 1.4426950408889634f;  // 32^-0.5 * log2(e): softmax in base 2
  const int nblk = (N + FA_K - 1) / FA_K;
  for (int kb = 0; kb < nblk; ++kb) {
    const int buf = kb & 1, j0 = kb * FA_K;
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();  // tile[buf] landed; everyone finished with tile[buf^1]
    if (kb + 1 < nblk) load_kv(j0 + FA_K, buf ^ 1);
    const uint32_t kbase = (uint32_t)__cvta_generic_to_shared(Ks[buf]);
    const uint32_t vbase = (uint32_t)__cvta_generic_to_shared(Vs[buf]);
    const int mi = lane >> 3, r8 = lane & 7;
    // ---- S = Q K^T: 8 n-tiles of 8 keys
    float sc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
      uint32_t b0, b1, b2, b3;  // (keys, d 0-7) (keys, d 8-15) (keys, d 16-23) (keys, d 24-31)
      ldsm_x4(kbase + (uint32_t)(((nt * 8 + r8) * FA_P + mi * 8) * 2), b0, b1, b2, b3);
      mma_bf16_16816(sc[nt], qa[0][0], qa[0][1], qa[0][2], qa[0][3], b0, b1);
      mma_bf16_16816(sc[nt], qa[1][0], qa[1][1], qa[1][2], qa[1][3], b2, b3);
    }
    // ---- mask keys past N, scale, row max
    const int g = lane >> 2, t4 = lane & 3;
    float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int key = j0 + nt * 8 + t4 * 2;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const bool ok = key + (e & 1) < N;
        sc[nt][e] = ok ? sc[nt][e] * SC : -INFINITY;
      }
      mx_lo = fmaxf(mx_lo, fmaxf(sc[nt][0], sc[nt][1]));
      mx_hi = fmaxf(mx_hi, fmaxf(sc[nt][2], sc[nt][3]));
    }
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
    const float mn_lo = fmaxf(m_lo, mx_lo), mn_hi = fmaxf(m_hi, mx_hi);   // finite: every block holds >= 1 valid key
    const float al_lo = exp2f(m_lo - mn_lo), al_hi = exp2f(m_hi - mn_hi); // 0 on the first block
    m_lo = mn_lo; m_hi = mn_hi;
    // ---- P = exp2(S - m) as bf16 A fragments; row sums of the ROUNDED values the MMA consumes
    uint32_t pa[4][4];
    float ps_lo = 0.f, ps_hi = 0.f;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int nt = kk * 2 + half;
        const float p0 = exp2f(sc[nt][0] - mn_lo), p1 = exp2f(sc[nt][1] - mn_lo);
        const float p2 = exp2f(sc[nt][2] - mn_hi), p3 = exp2f(sc[nt][3] - mn_hi);
        const uint32_t lo2 = pack_bf16x2(p0, p1), hi2 = pack_bf16x2(p2, p3);
        pa[kk][half * 2 + 0] = lo2;
        pa[kk][half * 2 + 1] = hi2;
        const __nv_bfloat162 l2 = *reinterpret_cast<const __nv_bfloat162*>(&lo2), h2 = *reinterpret_cast<const __nv_bfloat162*>(&hi2);
        ps_lo += __low2float(l2) + __high2float(l2);
        ps_hi += __low2float(h2) + __high2float(h2);
      }
    }
    ps_lo += __shfl_xor_sync(0xffffffffu, ps_lo, 1);
    ps_lo += __shfl_xor_sync(0xffffffffu, ps_lo, 2);
    ps_hi += __shfl_xor_sync(0xffffffffu, ps_hi, 1);
    ps_hi += __shfl_xor_sync(0xffffffffu, ps_hi, 2);
    l_lo = l_lo * al_lo + ps_lo;
    l_hi = l_hi * al_hi + ps_hi;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) { o[nt][0] *= al_lo; o[nt][1] *= al_lo; o[nt][2] *= al_hi; o[nt][3] *= al_hi; }
    // ---- O += P V: 4 k-steps of 16 keys, 4 n-tiles of 8 d's
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int np = 0; np < 2; ++np) {
        uint32_t b0, b1, b2, b3;  // (k 0-7, n 0-7) (k 8-15, n 0-7) (k 0-7, n 8-15) (k 8-15, n 8-15) after transpose
        ldsm_x4_trans(vbase + (uint32_t)(((kk * 16 + (mi & 1) * 8 + r8) * FA_P + np * 16 + (mi >> 1) * 8) * 2), b0, b1, b2, b3);
        mma_bf16_16816(o[np * 2], pa[kk][0], pa[kk][1], pa[kk][2], pa[kk][3], b0, b1);
        mma_bf16_16816(o[np * 2 + 1], pa[kk][0], pa[kk][1], pa[kk][2], pa[kk][3], b2, b3);
      }
    }
  }
  // ---- normalise and store rows g / g+8
  const int g = lane >> 2, t4 = lane & 3;
  const float inv_lo = 1.0f / l_lo, inv_hi = 1.0f / l_hi;
  const int r_lo = q0 + warp * 16 + g, r_hi = r_lo + 8;
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const int col = h * 32 + nt * 8 + t4 * 2;
    if (r_lo < N)
      *reinterpret_cast<__nv_bfloat162*>(hidden + ((long long)b * N + r_lo) * hid_pitch + col) = __floats2bfloat162_rn(o[nt][0] * inv_lo, o[nt][1] * inv_lo);
    if (r_hi < N)
      *reinterpret_cast<__nv_bfloat162*>(hidden + ((long long)b * N + r_hi) * hid_pitch + col) = __floats2bfloat162_rn(o[nt][2] * inv_hi, o[nt][3] * inv_hi);
  }
}

template <typename T>
void launch_fullattn(const T* qkv, int qkv_pitch, T* hidden, int hid_pitch, int B, int N, cudaStream_t st) {
  pdl_launch(fullattn_kernel<T>, dim3((N + 127) / 128, B * 4), 128, 0, st, qkv, qkv_pitch, hidden, hid_pitch, N);
}
template <>
void launch_fullattn<bf16>(const bf16* qkv, int qkv_pitch, bf16* hidden, int hid_pitch, int B, int N, cudaStream_t st) {
  static const bool force_scalar = getenv("IRSDE_FULLATTN_SCALAR") && getenv("IRSDE_FULLATTN_SCALAR")[0] == '1';
  if (!force_scalar && qkv_pitch % 8 == 0 && hid_pitch % 2 == 0 && ((uintptr_t)qkv % 16) == 0 && ((uintptr_t)hidden % 4) == 0)
    pdl_launch(fullattn_mma_kernel, dim3((N + FA_Q - 1) / FA_Q, B * 4), 128, 0, st, qkv, qkv_pitch, hidden, hid_pitch, N);
  else
    pdl_launch(fullattn_kernel<bf16>, dim3((N + 127) / 128, B * 4), 128, 0, st, qkv, qkv_pitch, hidden, hid_pitch, N);
}
template void launch_fullattn<float>(const float*, int, float*, int, int, int, cudaStream_t);
template void launch_fullattn<bf16>(const bf16*, int, bf16*, int, int, int, cudaStream_t);

}  // namespace irsde
