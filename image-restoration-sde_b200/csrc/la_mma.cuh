// Warp-level tensor-core pieces of the bf16 LinearAttention kernels (attention.cu, linattn_fused.cu): the mma.sync /
// ldmatrix wrappers, the partial-record format of pass A and the per-chunk online softmax + P^T V step it runs on a
// [64 px][k | v] tile in shared memory.
#pragma once
#include <math.h>

#include "common.cuh"

namespace irsde {

static const int LA_PIX = 64;               // pixels per chunk
static const int LA_REC = 4 * (64 + 1024);  // floats per partial record (4 heads x (m[32], s[32], ctx[32][32]))
static const int LA_MAXBLK = 64;            // partial records per image
static const int LAM_TP = 264;              // k|v tile row pitch (bf16): 256 + 8 pad -> conflict-free ldmatrix
static const int LAM_PP = 136;              // P row pitch (bf16): 128 + 8 pad

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
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
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// One 64-pixel chunk of pass A on the k|v tile T0 ([64][LAM_TP]; k rows of pixels past the image hold -1e30, v rows 0),
// for a block of 8 warps.  The softmax statistics of a chunk stay inside a warp: lane (qtr = lane / 4, cpl = lane % 4) of
// warp w owns channel pairs w*4+cpl and 32+w*4+cpl on the 8 pixels px == qtr (mod 8): the running max mr / sum sr live in
// registers (replicated over the 8 qtr lanes), the cross-pixel max and sum are three xor-shuffles each, and the bf16x2
// accesses (word = 4*px + pair mod 32) are bank-conflict free.  P goes to Ps ([64][LAM_PP]) and the rescale factors to
// alpha_s[128]; one block barrier makes them visible, then warp w adds P_h^T V_h for head w/2 and d-rows 16*(w%2)..+15 to
// acc (4 n-tiles of 8 e's) with mma.sync, operands from ldmatrix.trans.  The caller's next barrier must come before T0,
// Ps or alpha_s are written again.
__device__ __forceinline__ void la_chunk_softmax_pv(const bf16* T0, bf16* Ps, float* alpha_s, float (&mr)[4], float (&sr)[4],
                                                    float (&acc)[4][4]) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int h = warp >> 1, dbase = h * 32 + (warp & 1) * 16;
  const float LOG2E = 1.4426950408889634f;
  const int sq = lane >> 2, pA = warp * 4 + (lane & 3), pB = 32 + pA;
  // ---- softmax statistics, branch-free: rows past the image hold k = -1e30; ~13 instructions per bf16 pair
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

// The block's partial record: (m, s) of the 128 k channels and the 4 heads' 32x32 contexts, from the state
// la_chunk_softmax_pv left in registers.
__device__ __forceinline__ void la_store_record(float* rec, const float (&mr)[4], const float (&sr)[4], const float (&acc)[4][4]) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int h = warp >> 1, sq = lane >> 2, pA = warp * 4 + (lane & 3), pB = 32 + pA;
  if (sq == 0) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int chn = 2 * (c < 2 ? pA : pB) + (c & 1);
      rec[(chn >> 5) * 1088 + (chn & 31)] = mr[c];
      rec[(chn >> 5) * 1088 + 32 + (chn & 31)] = sr[c];
    }
  }
  const int g = lane >> 2, t4 = lane & 3, drow = (warp & 1) * 16 + g;
  float* cp = rec + h * 1088 + 64;
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const int e = nt * 8 + t4 * 2;
    *reinterpret_cast<float2*>(cp + drow * 32 + e) = make_float2(acc[nt][0], acc[nt][1]);
    *reinterpret_cast<float2*>(cp + (drow + 8) * 32 + e) = make_float2(acc[nt][2], acc[nt][3]);
  }
}

}  // namespace irsde
