// Residual(PreNorm(LinearAttention)) (module_util.py:150-178) as two fused passes over the block input x, bf16, for
// C = 64 and 128 channels:
//   pass 1 (la_kv_ln_kernel): LayerNorm(x) -> k|v = W_kv xn on the tensor cores -> the online softmax over pixels and
//           P^T V of pass A (la_chunk_softmax_pv), one partial record per block in pass A's format and partition; the
//           records then go through la_combine8 and la_fold16 unchanged (ctx, then Mb[b] = Wout ctx_b).
//   pass 2 (la_out_ln_kernel): LayerNorm(x) -> q = W_q xn -> per-head softmax(q) * 32^-.5 -> y = Mb[b] q + bias ->
//           LayerNorm(y) * g2 + x.
// Neither the 384-channel qkv tensor, nor xn, nor y ever reaches global memory: the block reads x twice and writes its
// output once.  Both passes compute xn with the arithmetic of layernorm_geo_kernel<bf16, 1, C/8, 2>, so the bf16 xn tile
// equals launch_layernorm's output bit for bit.  Wider rows (C >= 256) keep the unfused path: W_kv (256 x C bf16) must
// stay resident in shared memory next to the tiles.
#include <string.h>

#include "la_mma.cuh"

namespace irsde {

// LayerNorm of one pixel row of C = 8 * LPP channels, one 16-byte vector per lane on LPP consecutive lanes (every lane of
// the warp calls it), with layernorm_geo_kernel's bf16 operation order: s = sum of the lane's 8 values, xor-tree over the
// lane group, mean = s * inv_C, q likewise over (v - mean)^2, rstd = rsqrtf(q * inv_C + 1e-5), y = (v - mean) * rstd * g.
template <int LPP>
__device__ __forceinline__ uint4 ln_row_vec8(uint4 raw, const float (&gg)[8], float inv_C) {
  float v[8];
  const __nv_bfloat162* hx = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
  for (int i = 0; i < 4; ++i) { v[2 * i] = __low2float(hx[i]); v[2 * i + 1] = __high2float(hx[i]); }
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) s += v[j];
#pragma unroll
  for (int o = LPP >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s * inv_C;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) { v[j] -= mean; q += v[j] * v[j]; }
#pragma unroll
  for (int o = LPP >> 1; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q * inv_C + 1e-5f);
  uint4 t;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&t);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i] * rstd * gg[2 * i], v[2 * i + 1] * rstd * gg[2 * i + 1]);
  return t;
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src));
}
__device__ __forceinline__ void st_shared_zero16(uint32_t dst) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(dst), "r"(0u) : "memory");
}

template <int C>
struct LaFused {
  static constexpr int XP = C + 8;  // x / xn / weight row pitch (bf16): 16 bytes of pad -> conflict-free ldmatrix
  static constexpr int LPP = C / 8;
  // pass 2: warps per block and blocks per SM.  Pass 2 is bound by latency, so it runs as many warps as the registers allow
  // without spills: 2 x 8 warps at C = 64 (<= 128 registers), 12 warps (<= 168 registers: 3 per SM sub-partition) at C = 128.
  static constexpr int NW2 = C == 64 ? 8 : 12, BPS2 = C == 64 ? 2 : 1;
  // pass 1: W_kv [256][XP], x [2][64][XP], k|v tile [64][LAM_TP], P [64][LAM_PP], alpha [128]
  static constexpr size_t SMEM1 = ((size_t)256 * XP + 2 * LA_PIX * XP + LA_PIX * LAM_TP + LA_PIX * LAM_PP) * 2 + 128 * 4;
  // pass 2: W_q [128][XP], Mb[b] [C][136], per warp x [2][16][XP] and xn [16][XP] (226 304 B at C = 128)
  static constexpr size_t SMEM2 = ((size_t)128 * XP + C * 136 + NW2 * 3 * 16 * XP) * 2;
};

// ---- pass 1 ---------------------------------------------------------------------------------------------------------
// Per 64-pixel chunk, four block barriers: x landed (the previous chunk's P^T V is done with the tile), xn written,
// k|v written, P visible (inside la_chunk_softmax_pv).  The projection: warp w computes k|v columns 32w..32w+31 of all 64
// pixels (4 m-tiles x 4 n-tiles, A = xn and B = W_kv rows through ldmatrix).  k of a pixel past the image is -1e30 and
// its v 0, as pass A's loader fills them.  xn_dump (tests) receives the bf16 xn rows.
template <int C>
__global__ void __launch_bounds__(256) la_kv_ln_kernel(const bf16* __restrict__ x, int x_pitch, const float* __restrict__ g,
                                                       float inv_C, const bf16* __restrict__ wkv, float* __restrict__ part,
                                                       int N, int nchunks, int nblk, bf16* __restrict__ xn_dump) {
  using F = LaFused<C>;
  constexpr int XP = F::XP, LPP = F::LPP, VPR = C / 8;  // 16-byte vectors per row
  PDL_ENTRY();
  extern __shared__ __align__(16) uint8_t lf_sm[];
  bf16* Ws = reinterpret_cast<bf16*>(lf_sm);  // [256][XP]
  bf16* Xs = Ws + 256 * XP;                   // [2][64][XP]
  bf16* tile = Xs + 2 * LA_PIX * XP;          // [64][LAM_TP]
  bf16* Ps = tile + LA_PIX * LAM_TP;          // [64][LAM_PP]
  float* alpha_s = reinterpret_cast<float*>(Ps + LA_PIX * LAM_PP);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.y, blk = blockIdx.x;
  const int c0 = (int)(((long long)nchunks * blk) / nblk), c1 = (int)(((long long)nchunks * (blk + 1)) / nblk);
  const bf16* xb = x + (long long)b * N * x_pitch;
  const uint32_t xs_base = (uint32_t)__cvta_generic_to_shared(Xs);
  auto issue_x = [&](int ch, int buf) {
    const int n0 = ch * LA_PIX;
#pragma unroll
    for (int i = 0; i < LA_PIX * VPR / 256; ++i) {
      const int v = tid + i * 256, px = v / VPR, j = v % VPR;
      const uint32_t dst = xs_base + (uint32_t)(((buf * LA_PIX + px) * XP + j * 8) * 2);
      if (n0 + px < N) cp_async16(dst, xb + (long long)(n0 + px) * x_pitch + j * 8);
      else st_shared_zero16(dst);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  {
    const uint32_t ws_base = (uint32_t)__cvta_generic_to_shared(Ws);
    for (int v = tid; v < 256 * VPR; v += 256) cp_async16(ws_base + (uint32_t)(((v / VPR) * XP + (v % VPR) * 8) * 2), wkv + (long long)v * 8);
  }
  if (c0 < c1) issue_x(c0, 0);  // one group with the weights
  float gg[8];
  {
    const int sub = tid % LPP;
#pragma unroll
    for (int j = 0; j < 8; ++j) gg[j] = g[sub * 8 + j];
  }
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  float mr[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY}, sr[4] = {0.f, 0.f, 0.f, 0.f};
  const int mi = lane >> 3, r8 = lane & 7, gq = lane >> 2, t4 = lane & 3;
  for (int ch = c0; ch < c1; ++ch) {
    const int buf = (ch - c0) & 1, n0 = ch * LA_PIX;
    bf16* X0 = Xs + buf * LA_PIX * XP;
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();  // x[buf] landed; the previous chunk is done with x[buf^1], the k|v tile, P and alpha
    if (ch + 1 < c1) issue_x(ch + 1, buf ^ 1);
    // ---- LayerNorm in place: LPP lanes per pixel
#pragma unroll
    for (int p = 0; p < LA_PIX * LPP / 256; ++p) {
      const int px = p * (256 / LPP) + tid / LPP, sub = tid % LPP;
      uint4* cell = reinterpret_cast<uint4*>(X0 + px * XP + sub * 8);
      const uint4 y = ln_row_vec8<LPP>(*cell, gg, inv_C);
      *cell = y;
      if (xn_dump && n0 + px < N) *reinterpret_cast<uint4*>(xn_dump + ((long long)b * N + n0 + px) * C + sub * 8) = y;
    }
    __syncthreads();
    // ---- k|v = xn W_kv^T: warp w -> columns 32w..32w+31
    {
      float kv[4][4][4];
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) kv[mt][nt][0] = kv[mt][nt][1] = kv[mt][nt][2] = kv[mt][nt][3] = 0.f;
      const uint32_t xbase = (uint32_t)__cvta_generic_to_shared(X0), wbase = (uint32_t)__cvta_generic_to_shared(Ws);
#pragma unroll
      for (int k2 = 0; k2 < C / 32; ++k2) {
        uint32_t a[2][4][4];
#pragma unroll
        for (int kh = 0; kh < 2; ++kh)
#pragma unroll
          for (int mt = 0; mt < 4; ++mt)
            ldsm_x4(xbase + (uint32_t)(((mt * 16 + (mi & 1) * 8 + r8) * XP + k2 * 32 + kh * 16 + (mi >> 1) * 8) * 2), a[kh][mt][0],
                    a[kh][mt][1], a[kh][mt][2], a[kh][mt][3]);
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          uint32_t b0, b1, b2, b3;  // n-tile rows of W_kv, k 0-7 / 8-15 / 16-23 / 24-31 of this 32-step
          ldsm_x4(wbase + (uint32_t)(((warp * 32 + nt * 8 + r8) * XP + k2 * 32 + mi * 8) * 2), b0, b1, b2, b3);
#pragma unroll
          for (int mt = 0; mt < 4; ++mt) {
            mma_bf16_16816(kv[mt][nt], a[0][mt][0], a[0][mt][1], a[0][mt][2], a[0][mt][3], b0, b1);
            mma_bf16_16816(kv[mt][nt], a[1][mt][0], a[1][mt][1], a[1][mt][2], a[1][mt][3], b2, b3);
          }
        }
      }
      const uint32_t fill = warp < 4 ? 0xF14AF14Au : 0u;  // k = -1e30, v = 0 past the image
#pragma unroll
      for (int mt = 0; mt < 4; ++mt) {
        const int r_lo = mt * 16 + gq, r_hi = r_lo + 8;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int col = warp * 32 + nt * 8 + t4 * 2;
          *reinterpret_cast<uint32_t*>(tile + r_lo * LAM_TP + col) = n0 + r_lo < N ? pack_bf16x2(kv[mt][nt][0], kv[mt][nt][1]) : fill;
          *reinterpret_cast<uint32_t*>(tile + r_hi * LAM_TP + col) = n0 + r_hi < N ? pack_bf16x2(kv[mt][nt][2], kv[mt][nt][3]) : fill;
        }
      }
    }
    __syncthreads();
    la_chunk_softmax_pv(tile, Ps, alpha_s, mr, sr, acc);
  }
  __syncthreads();
  la_store_record(part + ((long long)b * LA_MAXBLK + blk) * LA_REC, mr, sr, acc);
}

// ---- pass 2 ---------------------------------------------------------------------------------------------------------
// The block holds W_q and Mb[b] in shared memory; its NW2 warps then work independently, each on 16-pixel chunks of image b
// with its own double-buffered x tile (no block barriers in the loop).  Per chunk, a warp: LayerNorm -> xn (its own tile);
// then head by head
// q_h = xn W_q,h^T (4 n-tiles, fp32 fragments), softmax over the head's 32 channels on the fragments (row max / sum across
// the quad) with the to_qkv epilogue's arithmetic (__expf, __fdividef(32^-.5, sum)), q_h re-packed in registers as the bf16
// A operand (the FlashAttention-2 register reuse) and y += q_h Mb[b][:, head]^T; then y + bias, LayerNorm of y in fp32
// (two-pass, rows across the quad) * g2 + x; bf16 pairs into the output view.  Working head by head keeps the live
// fragments to y plus one head, so 12 - 16 warps fit on an SM: the pass is bound by latency, and the extra warps hide it.
template <int C>
__global__ void __launch_bounds__(LaFused<C>::NW2 * 32, LaFused<C>::BPS2) la_out_ln_kernel(const bf16* __restrict__ x, int x_pitch, const float* __restrict__ g1,
                                                           float inv_C, const bf16* __restrict__ wq, const bf16* __restrict__ Mb,
                                                           const float* __restrict__ bias, const float* __restrict__ g2,
                                                           bf16* __restrict__ out, int out_pitch, int N, int nblk) {
  using F = LaFused<C>;
  constexpr int XP = F::XP, LPP = F::LPP, VPR = C / 8, MP = 136, NT = C / 8, NW = F::NW2, NTH = NW * 32;
  PDL_ENTRY();
  extern __shared__ __align__(16) uint8_t lf_sm[];
  bf16* Wq = reinterpret_cast<bf16*>(lf_sm);  // [128][XP]
  bf16* Ms = Wq + 128 * XP;                   // [C][MP]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  bf16* Xw = Ms + C * MP + warp * 3 * 16 * XP;  // [2][16][XP] x, then [16][XP] xn
  bf16* XNw = Xw + 2 * 16 * XP;
  const int b = blockIdx.y, blk = blockIdx.x;
  const int n16 = (N + 15) / 16;
  const int j0 = (int)(((long long)n16 * blk) / nblk), j1 = (int)(((long long)n16 * (blk + 1)) / nblk);
  const bf16* xb = x + (long long)b * N * x_pitch;
  {
    const uint32_t wb = (uint32_t)__cvta_generic_to_shared(Wq), mb = (uint32_t)__cvta_generic_to_shared(Ms);
    for (int v = tid; v < 128 * VPR; v += NTH) cp_async16(wb + (uint32_t)(((v / VPR) * XP + (v % VPR) * 8) * 2), wq + (long long)v * 8);
    const bf16* Mbb = Mb + (long long)b * C * 128;
    for (int v = tid; v < C * 16; v += NTH) cp_async16(mb + (uint32_t)(((v >> 4) * MP + (v & 15) * 8) * 2), Mbb + (long long)v * 8);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  const uint32_t xw_base = (uint32_t)__cvta_generic_to_shared(Xw), xnb = (uint32_t)__cvta_generic_to_shared(XNw);
  auto issue_x = [&](int j, int buf) {
    const int n0 = j * 16;
#pragma unroll
    for (int i = 0; i < 16 * VPR / 32; ++i) {
      const int v = lane + i * 32, px = v / VPR, jj = v % VPR;
      const uint32_t dst = xw_base + (uint32_t)(((buf * 16 + px) * XP + jj * 8) * 2);
      if (n0 + px < N) cp_async16(dst, xb + (long long)(n0 + px) * x_pitch + jj * 8);
      else st_shared_zero16(dst);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  if (j0 + warp < j1) issue_x(j0 + warp, 0);
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();  // W_q and Mb[b] resident (and this warp's first x tile)
  const int mi = lane >> 3, r8 = lane & 7, gq = lane >> 2, t4 = lane & 3;
  const uint32_t wqb = (uint32_t)__cvta_generic_to_shared(Wq), msb = (uint32_t)__cvta_generic_to_shared(Ms);
  int buf = 0;
  for (int j = j0 + warp; j < j1; j += NW, buf ^= 1) {
    const int n0 = j * 16;
    __syncwarp();  // every lane is done with x[buf^1] (the previous chunk's residual)
    if (j + NW < j1) {
      issue_x(j + NW, buf ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncwarp();
    const bf16* X0 = Xw + buf * 16 * XP;
    // ---- LayerNorm -> xn (the gain is re-read per chunk from L1: registers are what limits the warps per SM)
    float gg[8];
#pragma unroll
    for (int q4 = 0; q4 < 2; ++q4) {
      const float4 t = *reinterpret_cast<const float4*>(g1 + (lane % LPP) * 8 + q4 * 4);
      gg[4 * q4] = t.x; gg[4 * q4 + 1] = t.y; gg[4 * q4 + 2] = t.z; gg[4 * q4 + 3] = t.w;
    }
#pragma unroll
    for (int p = 0; p < 16 * LPP / 32; ++p) {
      const int px = p * (32 / LPP) + lane / LPP, sub = lane % LPP;
      *reinterpret_cast<uint4*>(XNw + px * XP + sub * 8) =
          ln_row_vec8<LPP>(*reinterpret_cast<const uint4*>(X0 + px * XP + sub * 8), gg, inv_C);
    }
    __syncwarp();
    float y[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) y[nt][0] = y[nt][1] = y[nt][2] = y[nt][3] = 0.f;
#pragma unroll 1
    for (int h = 0; h < 4; ++h) {  // not unrolled: the fragments of one head at a time stay live
      // ---- q_h = xn W_q,h^T: 16 rows x 32 channels (n-tiles 4h..4h+3)
      float q[4][4];
#pragma unroll
      for (int t = 0; t < 4; ++t) q[t][0] = q[t][1] = q[t][2] = q[t][3] = 0.f;
#pragma unroll
      for (int k2 = 0; k2 < C / 32; ++k2) {
        uint32_t a[2][4];
#pragma unroll
        for (int kh = 0; kh < 2; ++kh)
          ldsm_x4(xnb + (uint32_t)((((mi & 1) * 8 + r8) * XP + k2 * 32 + kh * 16 + (mi >> 1) * 8) * 2), a[kh][0], a[kh][1],
                  a[kh][2], a[kh][3]);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          uint32_t b0, b1, b2, b3;
          ldsm_x4(wqb + (uint32_t)((((4 * h + t) * 8 + r8) * XP + k2 * 32 + mi * 8) * 2), b0, b1, b2, b3);
          mma_bf16_16816(q[t], a[0][0], a[0][1], a[0][2], a[0][3], b0, b1);
          mma_bf16_16816(q[t], a[1][0], a[1][1], a[1][2], a[1][3], b2, b3);
        }
      }
      // ---- softmax over the head's 32 channels, rows g (elements 0, 1) and g+8 (2, 3)
      float m_lo = q[0][0], m_hi = q[0][2];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        m_lo = fmaxf(m_lo, fmaxf(q[t][0], q[t][1]));
        m_hi = fmaxf(m_hi, fmaxf(q[t][2], q[t][3]));
      }
      m_lo = fmaxf(m_lo, __shfl_xor_sync(0xffffffffu, m_lo, 1));
      m_lo = fmaxf(m_lo, __shfl_xor_sync(0xffffffffu, m_lo, 2));
      m_hi = fmaxf(m_hi, __shfl_xor_sync(0xffffffffu, m_hi, 1));
      m_hi = fmaxf(m_hi, __shfl_xor_sync(0xffffffffu, m_hi, 2));
      float s_lo = 0.f, s_hi = 0.f;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        q[t][0] = __expf(q[t][0] - m_lo); q[t][1] = __expf(q[t][1] - m_lo);
        q[t][2] = __expf(q[t][2] - m_hi); q[t][3] = __expf(q[t][3] - m_hi);
        s_lo += q[t][0] + q[t][1];
        s_hi += q[t][2] + q[t][3];
      }
      s_lo += __shfl_xor_sync(0xffffffffu, s_lo, 1);
      s_lo += __shfl_xor_sync(0xffffffffu, s_lo, 2);
      s_hi += __shfl_xor_sync(0xffffffffu, s_hi, 1);
      s_hi += __shfl_xor_sync(0xffffffffu, s_hi, 2);
      const float i_lo = __fdividef(0.17677669529663687f, s_lo), i_hi = __fdividef(0.17677669529663687f, s_hi);
      uint32_t qa[2][4];  // k-step kk = n-tiles 2kk (a0, a1) and 2kk+1 (a2, a3) of the head
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        qa[kk][0] = pack_bf16x2(q[2 * kk][0] * i_lo, q[2 * kk][1] * i_lo);
        qa[kk][1] = pack_bf16x2(q[2 * kk][2] * i_hi, q[2 * kk][3] * i_hi);
        qa[kk][2] = pack_bf16x2(q[2 * kk + 1][0] * i_lo, q[2 * kk + 1][1] * i_lo);
        qa[kk][3] = pack_bf16x2(q[2 * kk + 1][2] * i_hi, q[2 * kk + 1][3] * i_hi);
      }
      // ---- y += q_h Mb[b][:, 32h..32h+31]^T
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4(msb + (uint32_t)(((nt * 8 + r8) * MP + h * 32 + mi * 8) * 2), b0, b1, b2, b3);
        mma_bf16_16816(y[nt], qa[0][0], qa[0][1], qa[0][2], qa[0][3], b0, b1);
        mma_bf16_16816(y[nt], qa[1][0], qa[1][1], qa[1][2], qa[1][3], b2, b3);
      }
    }
    // ---- LayerNorm(y + bias) * g2 + x
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const float2 bb = *reinterpret_cast<const float2*>(bias + nt * 8 + t4 * 2);
      y[nt][0] += bb.x; y[nt][1] += bb.y; y[nt][2] += bb.x; y[nt][3] += bb.y;
    }
    float s_lo = 0.f, s_hi = 0.f;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) { s_lo += y[nt][0] + y[nt][1]; s_hi += y[nt][2] + y[nt][3]; }
    s_lo += __shfl_xor_sync(0xffffffffu, s_lo, 1);
    s_lo += __shfl_xor_sync(0xffffffffu, s_lo, 2);
    s_hi += __shfl_xor_sync(0xffffffffu, s_hi, 1);
    s_hi += __shfl_xor_sync(0xffffffffu, s_hi, 2);
    const float mean_lo = s_lo * inv_C, mean_hi = s_hi * inv_C;
    float v_lo = 0.f, v_hi = 0.f;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      y[nt][0] -= mean_lo; y[nt][1] -= mean_lo; y[nt][2] -= mean_hi; y[nt][3] -= mean_hi;
      v_lo += y[nt][0] * y[nt][0] + y[nt][1] * y[nt][1];
      v_hi += y[nt][2] * y[nt][2] + y[nt][3] * y[nt][3];
    }
    v_lo += __shfl_xor_sync(0xffffffffu, v_lo, 1);
    v_lo += __shfl_xor_sync(0xffffffffu, v_lo, 2);
    v_hi += __shfl_xor_sync(0xffffffffu, v_hi, 1);
    v_hi += __shfl_xor_sync(0xffffffffu, v_hi, 2);
    const float r_lo = rsqrtf(v_lo * inv_C + 1e-5f), r_hi = rsqrtf(v_hi * inv_C + 1e-5f);
    const bool ok_lo = n0 + gq < N, ok_hi = n0 + gq + 8 < N;
    bf16* o_lo = out + ((long long)b * N + n0 + gq) * out_pitch;
    bf16* o_hi = o_lo + (long long)8 * out_pitch;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const int col = nt * 8 + t4 * 2;
      const float2 gv = *reinterpret_cast<const float2*>(g2 + col);
      const __nv_bfloat162 x_lo = *reinterpret_cast<const __nv_bfloat162*>(X0 + gq * XP + col);
      const __nv_bfloat162 x_hi = *reinterpret_cast<const __nv_bfloat162*>(X0 + (gq + 8) * XP + col);
      if (ok_lo)
        *reinterpret_cast<__nv_bfloat162*>(o_lo + col) = __floats2bfloat162_rn(y[nt][0] * r_lo * gv.x + __low2float(x_lo),
                                                                               y[nt][1] * r_lo * gv.y + __high2float(x_lo));
      if (ok_hi)
        *reinterpret_cast<__nv_bfloat162*>(o_hi + col) = __floats2bfloat162_rn(y[nt][2] * r_hi * gv.x + __low2float(x_hi),
                                                                               y[nt][3] * r_hi * gv.y + __high2float(x_hi));
    }
  }
}

// ---- launchers --------------------------------------------------------------------------------------------------------
bool linattn_fused_ok(int C, const void* x, int x_pitch, const void* out, int out_pitch) {
  return (C == 64 || C == 128) && (uintptr_t)x % 16 == 0 && x_pitch % 8 == 0 && (uintptr_t)out % 4 == 0 && out_pitch % 2 == 0;
}

template <int C>
static void set_smem_attrs() {
  static bool done = false;
  if (done) return;
  cudaFuncSetAttribute(la_kv_ln_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LaFused<C>::SMEM1);
  cudaFuncSetAttribute(la_out_ln_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LaFused<C>::SMEM2);
  done = true;
}

void launch_la_kv_ln(const bf16* x, int x_pitch, const float* g1, const bf16* wkv, float* partial, int B, int N, int C,
                     bf16* xn_dump, cudaStream_t st) {
  int nblk, nchunks;
  linattn_partition(B, N, &nblk, &nchunks);
  const float inv_C = 1.0f / (float)C;
  if (C == 64) {
    set_smem_attrs<64>();
    pdl_launch(la_kv_ln_kernel<64>, dim3(nblk, B), 256, LaFused<64>::SMEM1, st, x, x_pitch, g1, inv_C, wkv, partial, N, nchunks, nblk, xn_dump);
  } else {
    set_smem_attrs<128>();
    pdl_launch(la_kv_ln_kernel<128>, dim3(nblk, B), 256, LaFused<128>::SMEM1, st, x, x_pitch, g1, inv_C, wkv, partial, N, nchunks, nblk, xn_dump);
  }
}

// Blocks per image of pass 2: one resident wave over the device for the whole batch (every pixel is computed the same way
// whatever block owns it), at least one 16-pixel chunk per warp.
template <int C>
static int la_out_blocks(int B, int N) {
  static int resident = 0;  // blocks of la_out_ln_kernel<C> the device holds at once
  if (!resident) {
    int dev = 0, sms = 1, per_sm = 1;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    set_smem_attrs<C>();
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, la_out_ln_kernel<C>, LaFused<C>::NW2 * 32, LaFused<C>::SMEM2);
    resident = (sms > 0 ? sms : 1) * (per_sm > 0 ? per_sm : 1);
  }
  const int n16 = (N + 15) / 16;
  int nblk = (resident + B - 1) / B;
  if (nblk > (n16 + LaFused<C>::NW2 - 1) / LaFused<C>::NW2) nblk = (n16 + LaFused<C>::NW2 - 1) / LaFused<C>::NW2;
  return nblk < 1 ? 1 : nblk;
}

void launch_la_out_ln(const bf16* x, int x_pitch, const float* g1, const bf16* wq, const bf16* Mb, const float* bias,
                      const float* g2, bf16* out, int out_pitch, int B, int N, int C, cudaStream_t st) {
  const float inv_C = 1.0f / (float)C;
  if (C == 64) {
    const int nblk = la_out_blocks<64>(B, N);
    pdl_launch(la_out_ln_kernel<64>, dim3(nblk, B), LaFused<64>::NW2 * 32, LaFused<64>::SMEM2, st, x, x_pitch, g1, inv_C, wq, Mb, bias, g2, out, out_pitch, N, nblk);
  } else {
    const int nblk = la_out_blocks<128>(B, N);
    pdl_launch(la_out_ln_kernel<128>, dim3(nblk, B), LaFused<128>::NW2 * 32, LaFused<128>::SMEM2, st, x, x_pitch, g1, inv_C, wq, Mb, bias, g2, out, out_pitch, N, nblk);
  }
}

}  // namespace irsde
