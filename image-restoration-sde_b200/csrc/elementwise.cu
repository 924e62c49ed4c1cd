// Memory-bound kernels of the IR-SDE hot path: input packing, timestep-embedding table, the fused
// sampler update and layout helpers (LayerNorm / attention live in attention.cu).  All fp32 math; activations
// are float (parity mode) or bf16 (perf mode).
#include <math.h>

#include "common.cuh"

namespace irsde {

// =============================================================================================
// input packing: x = cat(xt - cond, cond) with reflect pad (bottom/right) -> NHWC
// reference: DenoisingUNet_arch.py:78-83 (check_image_size), :90-94
// =============================================================================================
template <typename T>
__global__ void prep_input_kernel(const float* __restrict__ xt, const float* __restrict__ cond, T* __restrict__ out,
                                  int B, int C, int H, int W, int Hp, int Wp, int pitch, int conditional,
                                  int pad_top, int pad_left, int row_pix, int img_rows, int zero_pad) {
  PDL_ENTRY();
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)B * Hp * Wp;
  if (idx >= total) return;
  int wp = idx % Wp;
  int hp = (idx / Wp) % Hp;
  int b = idx / ((long long)Wp * Hp);
  int h = hp < H ? hp : 2 * (H - 1) - hp;  // reflect (no edge repeat)
  int w = wp < W ? wp : 2 * (W - 1) - wp;
  // destination pixel inside an optionally zero-bordered buffer [B][img_rows][row_pix][pitch]
  T* o = out + (((long long)b * img_rows + hp + pad_top) * row_pix + wp + pad_left) * pitch;
  const bool zp = zero_pad && (hp >= H || wp >= W);  // NAFNet pads with zeros (DenoisingNAFNet_arch.py:183-188)
  for (int c = 0; c < C; ++c) {
    long long s = (((long long)b * C + c) * H + h) * W + w;
    float xv = zp ? 0.f : xt[s];
    if (conditional) {
      float cv = zp ? 0.f : cond[s];
      o[c] = from_f<T>(__fsub_rn(xv, cv));
      o[C + c] = from_f<T>(cv);
    } else {
      o[c] = from_f<T>(xv);
    }
  }
  for (int c = conditional ? 2 * C : C; c < pitch; ++c) o[c] = from_f<T>(0.f);
}

template <typename T>
void launch_prep_input(const float* xt, const float* cond, T* out, int B, int C, int H, int W, int Hp, int Wp,
                       int out_pitch, int conditional, cudaStream_t st, int pad_top, int pad_left, int row_pix,
                       int img_rows, int zero_pad) {
  long long total = (long long)B * Hp * Wp;
  if (row_pix == 0) { row_pix = Wp; img_rows = Hp; }
  pdl_launch(prep_input_kernel<T>, (unsigned)((total + 255) / 256), 256, 0, st, xt, cond, out, B, C, H, W, Hp, Wp, out_pitch,
                                                                         conditional, pad_top, pad_left, row_pix, img_rows, zero_pad);
}
template void launch_prep_input<float>(const float*, const float*, float*, int, int, int, int, int, int, int, int,
                                       cudaStream_t, int, int, int, int, int);
template void launch_prep_input<bf16>(const float*, const float*, bf16*, int, int, int, int, int, int, int, int,
                                      cudaStream_t, int, int, int, int, int);

template <typename T>
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, T* __restrict__ out, int B, int C, int H, int W,
                                    int pitch) {
  PDL_ENTRY();
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)B * H * W;
  if (idx >= total) return;
  long long hw = idx % ((long long)H * W);
  int b = idx / ((long long)H * W);
  for (int c = 0; c < C; ++c) out[idx * pitch + c] = from_f<T>(in[((long long)b * C + c) * H * W + hw]);
  for (int c = C; c < pitch; ++c) out[idx * pitch + c] = from_f<T>(0.f);
}
template <typename T>
void launch_nchw_to_nhwc(const float* in, T* out, int B, int C, int H, int W, int out_pitch, cudaStream_t st) {
  long long total = (long long)B * H * W;
  pdl_launch(nchw_to_nhwc_kernel<T>, (unsigned)((total + 255) / 256), 256, 0, st, in, out, B, C, H, W, out_pitch);
}
template void launch_nchw_to_nhwc<float>(const float*, float*, int, int, int, int, int, cudaStream_t);
template void launch_nchw_to_nhwc<bf16>(const float*, bf16*, int, int, int, int, int, cudaStream_t);

template <typename T>
__global__ void nhwc_to_nchw_kernel(const T* __restrict__ in, int pitch, float* __restrict__ out, int B, int C, int H,
                                    int W) {
  PDL_ENTRY();
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)B * H * W;
  if (idx >= total) return;
  long long hw = idx % ((long long)H * W);
  int b = idx / ((long long)H * W);
  for (int c = 0; c < C; ++c) out[((long long)b * C + c) * H * W + hw] = to_f(in[idx * pitch + c]);
}
template <typename T>
void launch_nhwc_to_nchw(const T* in, int in_pitch, float* out, int B, int C, int H, int W, cudaStream_t st) {
  long long total = (long long)B * H * W;
  pdl_launch(nhwc_to_nchw_kernel<T>, (unsigned)((total + 255) / 256), 256, 0, st, in, in_pitch, out, B, C, H, W);
}
template void launch_nhwc_to_nchw<float>(const float*, int, float*, int, int, int, int, cudaStream_t);
template void launch_nhwc_to_nchw<bf16>(const bf16*, int, float*, int, int, int, int, cudaStream_t);

// =============================================================================================
// timestep embedding -> per-ResBlock (scale, shift) table
// SinusoidalPosEmb (module_util.py:29-41) -> Linear -> GELU -> Linear (DenoisingUNet_arch.py:42-47)
// then for every ResBlock: SiLU -> Linear(4nf -> 2*Cout) (module_util.py:128-130,138-141).
// Batch independent, so it is evaluated once per distinct t (a [rows][S] table).
// =============================================================================================
__global__ void time_mlp_kernel(const float* __restrict__ times, int nf, const float* __restrict__ w1,
                                const float* __restrict__ b1, const float* __restrict__ w2,
                                const float* __restrict__ b2, float* __restrict__ temb_silu) {
  extern __shared__ float sm[];
  int td = nf * 4, half = nf / 2;
  float* emb = sm;        // [nf]
  float* h1 = sm + nf;    // [td]
  int row = blockIdx.x;
  float t = times[row];
  float e = logf(10000.0f) / (float)(half - 1);
  for (int i = threadIdx.x; i < half; i += blockDim.x) {
    float f = expf((float)i * -e);
    float a = t * f;
    emb[i] = sinf(a);
    emb[half + i] = cosf(a);
  }
  __syncthreads();
  for (int o = threadIdx.x; o < td; o += blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < nf; ++k) s += w1[o * nf + k] * emb[k];
    s += b1[o];
    h1[o] = 0.5f * s * (1.0f + erff(s * 0.70710678118654752440f));  // exact GELU
  }
  __syncthreads();
  for (int o = threadIdx.x; o < td; o += blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < td; ++k) s += w2[o * td + k] * h1[k];
    s += b2[o];
    temb_silu[(long long)row * td + o] = silu_f(s);
  }
}

__global__ void time_table_kernel(const float* __restrict__ temb_silu, int td, const float* __restrict__ wall,
                                  const float* __restrict__ ball, int S, float* __restrict__ table) {
  int row = blockIdx.y;
  int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (j >= S) return;
  const float* w = wall + (long long)j * td;
  const float* x = temb_silu + (long long)row * td;
  float s = 0.f;
  for (int k = lane; k < td; k += 32) s += w[k] * x[k];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) table[(long long)row * S + j] = s + ball[j];
}

void launch_time_rows(const float* tvec, int rows, int td, const float* wall, const float* ball, int S, float* table, cudaStream_t st) {
  time_table_kernel<<<dim3((S + 7) / 8, rows), 256, 0, st>>>(tvec, td, wall, ball, S, table);
}

// emb [nf] + h1 [4nf] floats
size_t time_mlp_smem(int nf) { return (size_t)nf * 5 * sizeof(float); }

void launch_time_table(const float* times, int rows, int nf, const float* w1, const float* b1, const float* w2,
                       const float* b2, const float* wall, const float* ball, int S, float* temb_ws, float* table,
                       cudaStream_t st) {
  int td = nf * 4;
  time_mlp_kernel<<<rows, 256, time_mlp_smem(nf), st>>>(times, nf, w1, b1, w2, b2, temb_ws);
  time_table_kernel<<<dim3((S + 7) / 8, rows), 256, 0, st>>>(temb_ws, td, wall, ball, S, table);
}

// =============================================================================================
// sampler update (one fused kernel per step).  Op order follows the reference exactly, with
// explicit round-to-nearest intrinsics so ptxas cannot contract to FMA:
//   sde_utils.py:44-48,175-185 (IRSDE sde/ode), :197-223,237-239 (posterior),
//   :450-462 (DenoisingSDE).
// coef row layout (IRSDE_NUM_COEF floats per t), see engine.cu fill_default_coeffs():
//   SDE      : theta, sigma^2, sigma_bar, dt, sigma, sqrt(dt)
//   ODE      : theta, 0.5*sigma^2, sigma_bar, dt
//   POSTERIOR: exp(Theta_t dt), sigma_bar, term1, term2, std
//   DSDE_SDE : -0.5 sigma^2 (1+A), sigma_bar, dt, sigma, sqrt(dt)
//   DSDE_ODE : -0.5 sigma^2 A, sigma_bar, dt
// =============================================================================================
__device__ __forceinline__ uint32_t mulhilo(uint32_t a, uint32_t b, uint32_t* hi) {
  unsigned long long p = (unsigned long long)a * b;
  *hi = (uint32_t)(p >> 32);
  return (uint32_t)p;
}
__device__ __forceinline__ void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0, hi1;
    uint32_t lo0 = mulhilo(0xD2511F53u, c[0], &hi0);
    uint32_t lo1 = mulhilo(0xCD9E8D57u, c[2], &hi1);
    uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
    c[0] = n0;
    c[1] = n1;
    c[2] = n2;
    c[3] = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
}
// Four N(0,1) draws of Philox block `blk` of image `uid` at stream `stream` (= timestep; 0xffffffff for noise_state).
// The counter is (block within the image, image uid, stream): what an image receives depends only on (seed, uid, t,
// element index inside the image) - not on the batch it travels in, its position in it, or the rank that owns it.
__device__ __forceinline__ void normal4(uint64_t seed, uint64_t uid, uint32_t blk, uint32_t stream, float out[4]) {
  uint32_t c[4] = {blk, (uint32_t)uid, stream, 0x1234567u ^ (uint32_t)(uid >> 32)};
  philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  const float two_pow_m32 = 2.3283064365386963e-10f;
  float u0 = ((float)c[0] + 0.5f) * two_pow_m32, u1 = ((float)c[1] + 0.5f) * two_pow_m32;
  float u2 = ((float)c[2] + 0.5f) * two_pow_m32, u3 = ((float)c[3] + 0.5f) * two_pow_m32;
  u0 = fminf(fmaxf(u0, 1e-12f), 1.0f);
  u2 = fminf(fmaxf(u2, 1e-12f), 1.0f);
  float r0 = sqrtf(-2.0f * logf(u0)), r1 = sqrtf(-2.0f * logf(u2));
  float s0, c0, s1, c1;
  sincosf(6.283185307179586f * u1, &s0, &c0);
  sincosf(6.283185307179586f * u3, &s1, &c1);
  out[0] = r0 * c0;
  out[1] = r0 * s0;
  out[2] = r1 * c1;
  out[3] = r1 * s1;
}

// z for the 4 consecutive elements i0..i0+3 of a [B][img_elems] buffer (a group may straddle two images or two
// Philox blocks when img_elems % 4 != 0; it is one block otherwise).
__device__ __forceinline__ void image_normals(uint64_t seed, uint64_t uid_base, const unsigned long long* __restrict__ uids,
                                              long long i0, long long img_elems, uint32_t stream, float zr[4]) {
  long long b = i0 / img_elems, j = i0 - b * img_elems;
  float blk[4];
  long long cur_b = -1, cur_blk = -1;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (j == img_elems) { j = 0; ++b; }
    const long long q = j >> 2;
    if (b != cur_b || q != cur_blk) {
      normal4(seed, uids ? (uint64_t)uids[b] : uid_base + (uint64_t)b, (uint32_t)q, stream, blk);
      cur_b = b; cur_blk = q;
    }
    zr[k] = blk[j & 3];
    ++j;
  }
}

__device__ __forceinline__ float sde_update_one(int mode, const float* c, float x, float mu, float eps, float z) {
  switch (mode) {
    case 0: {  // IRSDE sde
      float score = __fdiv_rn(-eps, c[2]);
      float drift = __fmul_rn(__fsub_rn(__fmul_rn(c[0], __fsub_rn(mu, x)), __fmul_rn(c[1], score)), c[3]);
      float disp = __fmul_rn(c[4], __fmul_rn(z, c[5]));
      return __fsub_rn(__fsub_rn(x, drift), disp);
    }
    case 1: {  // IRSDE ode
      float score = __fdiv_rn(-eps, c[2]);
      float drift = __fmul_rn(__fsub_rn(__fmul_rn(c[0], __fsub_rn(mu, x)), __fmul_rn(c[1], score)), c[3]);
      return __fsub_rn(x, drift);
    }
    case 2: {  // IRSDE posterior
      float xm = __fsub_rn(x, mu);
      float x0 = __fadd_rn(__fmul_rn(__fsub_rn(xm, __fmul_rn(c[1], eps)), c[0]), mu);
      float mean = __fadd_rn(__fadd_rn(__fmul_rn(c[2], xm), __fmul_rn(c[3], __fsub_rn(x0, mu))), mu);
      return __fadd_rn(mean, __fmul_rn(c[4], z));
    }
    case 3: {  // DenoisingSDE sde
      float score = __fdiv_rn(-eps, c[1]);
      float drift = __fmul_rn(__fmul_rn(c[0], score), c[2]);
      float disp = __fmul_rn(c[3], __fmul_rn(z, c[4]));
      return __fsub_rn(__fsub_rn(x, drift), disp);
    }
    default: {  // DenoisingSDE ode
      float score = __fdiv_rn(-eps, c[1]);
      float drift = __fmul_rn(__fmul_rn(c[0], score), c[2]);
      return __fsub_rn(x, drift);
    }
  }
}

__global__ void sde_update_kernel(int mode, const float* __restrict__ x, const float* __restrict__ mu,
                                  const float* __restrict__ noise, const float* __restrict__ z, long long z_stride,
                                  const float* __restrict__ coef, const StepState* __restrict__ stp, int t_host,
                                  float* __restrict__ out, long long n, uint64_t seed, long long img_elems,
                                  uint64_t uid_base, const unsigned long long* __restrict__ uids) {
  PDL_ENTRY();
  int t = stp ? stp->t : t_host;
  int si = stp ? stp->i : 0;
  float c[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) c[k] = coef[t * 8 + k];
  bool need_z = (mode == 0 || mode == 2 || mode == 3);
  if (stp) { z = stp->z; seed = stp->seed; uid_base = stp->uid_base; uids = stp->uids; }
  const float* zz = z ? z + (long long)si * z_stride : nullptr;
  const bool vec4 = (((uintptr_t)x | (uintptr_t)noise | (uintptr_t)out | (uintptr_t)mu | (uintptr_t)zz) & 15) == 0;
  long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // group of 4 elements
  long long i0 = q * 4;
  if (i0 >= n) return;
  float zr[4] = {0.f, 0.f, 0.f, 0.f};
  if (need_z && !zz) image_normals(seed, uid_base, uids, i0, img_elems, (uint32_t)t, zr);
  if (vec4 && i0 + 3 < n) {  // 128-bit loads/stores: every operand is 16-byte aligned and the group is complete
    const float4 xv = *reinterpret_cast<const float4*>(x + i0);
    const float4 ev = *reinterpret_cast<const float4*>(noise + i0);
    const float4 mv = mu ? *reinterpret_cast<const float4*>(mu + i0) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (need_z && zz) {
      const float4 zv = *reinterpret_cast<const float4*>(zz + i0);
      zr[0] = zv.x; zr[1] = zv.y; zr[2] = zv.z; zr[3] = zv.w;
    }
    float4 o;
    o.x = sde_update_one(mode, c, xv.x, mv.x, ev.x, zr[0]);
    o.y = sde_update_one(mode, c, xv.y, mv.y, ev.y, zr[1]);
    o.z = sde_update_one(mode, c, xv.z, mv.z, ev.z, zr[2]);
    o.w = sde_update_one(mode, c, xv.w, mv.w, ev.w, zr[3]);
    *reinterpret_cast<float4*>(out + i0) = o;
    return;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    long long i = i0 + k;
    if (i < n) {
      float zv = need_z ? (zz ? zz[i] : zr[k]) : 0.f;
      float mv = mu ? mu[i] : 0.f;
      out[i] = sde_update_one(mode, c, x[i], mv, noise[i], zv);
    }
  }
}

void launch_sde_update(int mode, const float* x, const float* mu, const float* noise, const float* z, long long z_stride,
                       const float* coef, const StepState* st_dev, int t_host, float* out, long long n, uint64_t seed,
                       long long img_elems, uint64_t uid_base, const unsigned long long* uids, cudaStream_t st) {
  long long groups = (n + 3) / 4;
  pdl_launch(sde_update_kernel, (unsigned)((groups + 255) / 256), 256, 0, st, mode, x, mu, noise, z, z_stride, coef, st_dev,
                                                                      t_host, out, n, seed, img_elems > 0 ? img_elems : n,
                                                                      uid_base, uids);
}

__global__ void advance_step_kernel(StepState* s) {
  PDL_ENTRY();
  s->t -= 1;
  s->i += 1;
}
__global__ void set_step_kernel(StepState* s, int t, int i, const float* z, unsigned long long seed, unsigned long long uid_base,
                                const unsigned long long* uids) {
  s->t = t;
  s->i = i;
  s->z = z;
  s->seed = seed;
  s->uid_base = uid_base;
  s->uids = uids;
}
void launch_advance_step(StepState* st_dev, cudaStream_t st) { pdl_launch(advance_step_kernel, 1, 1, 0, st, st_dev); }
void launch_set_step(StepState* st_dev, int t, int i, const float* z, unsigned long long seed, unsigned long long uid_base,
                     const unsigned long long* uids, cudaStream_t st) {
  set_step_kernel<<<1, 1, 0, st>>>(st_dev, t, i, z, seed, uid_base, uids);
}

__global__ void noise_state_kernel(const float* __restrict__ mu, float* __restrict__ out, long long n, float max_sigma,
                                   uint64_t seed, long long img_elems, uint64_t uid_base,
                                   const unsigned long long* __restrict__ uids) {
  long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long i0 = q * 4;
  if (i0 >= n) return;
  float zr[4];
  image_normals(seed, uid_base, uids, i0, img_elems, 0xffffffffu, zr);
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (i0 + k < n) out[i0 + k] = mu[i0 + k] + zr[k] * max_sigma;
}
void launch_noise_state(const float* mu, float* out, long long n, float max_sigma, uint64_t seed, long long img_elems,
                        uint64_t uid_base, const unsigned long long* uids, cudaStream_t st) {
  long long groups = (n + 3) / 4;
  noise_state_kernel<<<(unsigned)((groups + 255) / 256), 256, 0, st>>>(mu, out, n, max_sigma, seed, img_elems > 0 ? img_elems : n,
                                                                       uid_base, uids);
}

// =============================================================================================
// space-to-depth (stride-2 phase planes) for the 4x4/s2 downsample on the tensor-core path:
// out[plane=(h&1)*2+(w&1)][b][h/2][w/2][c] = in[b][h][w][c]
// =============================================================================================
template <typename T>
__global__ void s2d_kernel(const T* __restrict__ in, int pitch, T* __restrict__ out, int B, int H, int W, int C) {
  PDL_ENTRY();
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over B*H*W*(C/8) 16-byte groups
  int vec = 16 / sizeof(T);
  int cg = C / vec;
  long long total = (long long)B * H * W * cg;
  if (idx >= total) return;
  int g = idx % cg;
  long long pix = idx / cg;
  int w = pix % W;
  int h = (pix / W) % H;
  int b = pix / ((long long)W * H);
  int plane = (h & 1) * 2 + (w & 1);
  long long o = ((((long long)plane * B + b) * (H / 2) + (h >> 1)) * (W / 2) + (w >> 1)) * C + g * vec;
  *reinterpret_cast<uint4*>(out + o) = *reinterpret_cast<const uint4*>(in + pix * pitch + g * vec);
}
template <typename T>
void launch_space_to_depth(const T* in, int in_pitch, T* out, int B, int H, int W, int C, cudaStream_t st) {
  int vec = 16 / sizeof(T);
  long long total = (long long)B * H * W * (C / vec);
  pdl_launch(s2d_kernel<T>, (unsigned)((total + 255) / 256), 256, 0, st, in, in_pitch, out, B, H, W, C);
}
// =============================================================================================
// training-time state sampler (sde_utils.py:343-358): x_t = noise * sigma_bar[t_b] + (mu + (x0 - mu) * exp(-Theta[t_b] dt)),
// one timestep per image; w[b] / sb[b] are the per-image scalars, the arithmetic follows the reference's op order with
// round-to-nearest intrinsics (no FMA contraction), so the result is bit-identical to the torch expression.
// =============================================================================================
__global__ void random_states_kernel(const float* __restrict__ x0, const float* __restrict__ mu, const float* __restrict__ noise,
                                     const float* __restrict__ w, const float* __restrict__ sb, float* __restrict__ out,
                                     long long n, long long img_elems) {
  long long i0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i0 >= n) return;
  const bool vec = ((((uintptr_t)x0 | (uintptr_t)mu | (uintptr_t)noise | (uintptr_t)out) & 15) == 0) && (img_elems % 4 == 0) && i0 + 3 < n;
  if (vec) {
    const int b = (int)(i0 / img_elems);
    const float wb = w[b], sbb = sb[b];
    const float4 a = *reinterpret_cast<const float4*>(x0 + i0), m = *reinterpret_cast<const float4*>(mu + i0);
    const float4 z = *reinterpret_cast<const float4*>(noise + i0);
    float4 o;
    o.x = __fadd_rn(__fmul_rn(z.x, sbb), __fadd_rn(m.x, __fmul_rn(__fsub_rn(a.x, m.x), wb)));
    o.y = __fadd_rn(__fmul_rn(z.y, sbb), __fadd_rn(m.y, __fmul_rn(__fsub_rn(a.y, m.y), wb)));
    o.z = __fadd_rn(__fmul_rn(z.z, sbb), __fadd_rn(m.z, __fmul_rn(__fsub_rn(a.z, m.z), wb)));
    o.w = __fadd_rn(__fmul_rn(z.w, sbb), __fadd_rn(m.w, __fmul_rn(__fsub_rn(a.w, m.w), wb)));
    *reinterpret_cast<float4*>(out + i0) = o;
    return;
  }
  for (long long i = i0; i < n && i < i0 + 4; ++i) {
    const int b = (int)(i / img_elems);
    out[i] = __fadd_rn(__fmul_rn(noise[i], sb[b]), __fadd_rn(mu[i], __fmul_rn(__fsub_rn(x0[i], mu[i]), w[b])));
  }
}
void launch_random_states(const float* x0, const float* mu, const float* noise, const float* w, const float* sb, float* out,
                          int B, long long img_elems, cudaStream_t st) {
  const long long n = (long long)B * img_elems, groups = (n + 3) / 4;
  random_states_kernel<<<(unsigned)((groups + 255) / 256), 256, 0, st>>>(x0, mu, noise, w, sb, out, n, img_elems);
}

// =============================================================================================
// fp32x3 operand split: hi = rn_tf32(x) (10-bit mantissa, low 13 bits zero), lo = rn_tf32(x - hi).  x - hi is exact in
// fp32, so x = hi + lo + r with |r| <= 2^-22 |x|: three tf32 MMAs (hi*hi + lo*hi + hi*lo) reproduce the fp32 product to
// 2^-21 relative.  Both parts carry explicit zero low bits, so the result does not depend on how the tensor core
// treats the 13 bits kind::tf32 ignores.
// =============================================================================================
__device__ __forceinline__ float rn_tf32(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
__global__ void split_tf32_kernel(const float* __restrict__ in, int pitch, float* __restrict__ out, long long npix, int C) {
  PDL_ENTRY();
  const int cg = C >> 2;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= npix * cg) return;
  const long long pix = idx / cg;
  const int g = (int)(idx - pix * cg);
  const float4 v = *reinterpret_cast<const float4*>(in + pix * pitch + g * 4);
  float4 h, l;
  h.x = rn_tf32(v.x); h.y = rn_tf32(v.y); h.z = rn_tf32(v.z); h.w = rn_tf32(v.w);
  l.x = rn_tf32(v.x - h.x); l.y = rn_tf32(v.y - h.y); l.z = rn_tf32(v.z - h.z); l.w = rn_tf32(v.w - h.w);
  *reinterpret_cast<float4*>(out + pix * C + g * 4) = h;
  *reinterpret_cast<float4*>(out + (npix + pix) * C + g * 4) = l;
}
void launch_split_tf32(const float* in, int in_pitch, float* out, long long npix, int C, cudaStream_t st) {
  long long total = npix * (C >> 2);
  pdl_launch(split_tf32_kernel, (unsigned)((total + 255) / 256), 256, 0, st, in, in_pitch, out, npix, C);
}

template void launch_space_to_depth<bf16>(const bf16*, int, bf16*, int, int, int, int, cudaStream_t);
template void launch_space_to_depth<float>(const float*, int, float*, int, int, int, int, cudaStream_t);

}  // namespace irsde
