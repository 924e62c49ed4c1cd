// Hopper (sm_90a) "tap-GEMM" convolution: bf16 NHWC activations, bf16 weights, fp32 accumulate in registers (wgmma).
//
//   D[pixel, n] = sum_{tap} sum_{c} A[pixel + (dh,dw)_tap, c] * Wt[phase][tap][n][c]
//
// One CTA computes a 128-pixel x BN-channel tile.  The 128 pixels are a BW x BH patch of one image
// (BW*BH = 128), so that for every tap the A operand is ONE TMA box {64 ch, BW, BH} of the NHWC
// tensor shifted by (dw,dh): zero padding is the TMA out-of-bounds fill, im2col never exists in
// memory.  The box lands in shared memory as 128 rows x 128 B with the 128B swizzle, which is exactly
// the canonical K-major wgmma operand layout; the weights tile ({64 ch, BN} of [tap][Cout][Cin]) likewise.
// This one kernel serves: 3x3 (9 taps), 1x1 (1 tap), 4x4/s2 (16 taps over 4 space-to-depth planes),
// nearest-x2-upsample + 3x3 (4 output phases x 4 taps with pre-summed weights).
//
// One persistent kernel (conv_tc_persist_kernel<BN, MODE, EKT>), 384 threads: warps 0..7 = two consumer warpgroups (each
// issues wgmma.m64nBNk16 into its registers, then runs the epilogue on them: q-softmax / bias / (scale+1)*x+shift / SiLU /
// +residual (TMA-loaded into the warp's store tile) -> bf16 -> stmatrix into that tile -> TMA bulk store at the channel
// offset of the destination concat buffer), warp 8 = TMA producer (warps 9..11 only give their registers to the consumers: setmaxnreg
// 40 / 232).  Schedule: bf16 BN = 64 / 128 PING-PONG (a warpgroup computes all 128 rows of every other tile, so its
// epilogue overlaps the other warpgroup's MMAs), otherwise COOPERATIVE (each warpgroup 64 rows of every tile).
// Pipeline: STAGES-deep smem ring with full/empty mbarriers.  Each consumer warpgroup issues a stage's MMAs as one wgmma
// group and keeps it in flight while it waits for the next stage's bytes and issues that stage's group; wgmma.wait_group 1
// then shows the older group done and the warpgroup releases its slot.  The producer runs ahead into the next tile.
// No function call may sit inside the wgmma window (see mbar_wait), or ptxas serializes every wgmma; the kernel makes no
// external call at all.  (The fp32x3 epilogue keeps calls to the IEEE-division slow path, a subroutine of the kernel
// itself that runs after the K loop's final wait.)
// Variants: MODE 0 per-tap boxes, MODE 2 ROWS (3x3, row-window reuse), MODE 3 fp32x3 (3 x tf32 wgmma on split fp32
// operands), EKT = epilogue features compiled in.
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>

#include <memory>
#include <type_traits>

#include "common.cuh"

namespace irsde {

namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

struct TcParams {
  int B, H, W;          // pixel grid enumerated by the tiles (== A tensor spatial size)
  int Cin, Cout;
  int ntaps, kchunks;
  int BW, BH, logBW;
  int tilesW, tilesH;
  int nphases;
  int Hout, Wout, os;   // output spatial size and output stride (2 for the upsample phases)
  bf16* out;
  int out_pitch;
  float* out_nchw;      // if set: write fp32 NCHW cropped to (cropH, cropW) instead of the NHWC view
  int cropH, cropW;
  int qsm;              // LinearAttention q: softmax over each 32-channel head * 32^-0.5 for output channels < 128
  int w_per_image;      // weights tensor is [B][Cout][Cin]: third TMA coordinate = image index
  float* out_f32;       // MODE 3 (fp32x3): fp32 NHWC output view (channel offset applied), pitch = out_pitch
  const float* res_f32; // MODE 3: fp32 residual view
  int lo_plane_off;     // MODE 3: plane offset of the "lo" split of the A tensor ([hi planes][lo planes])
  // tile decode without integer divisions (they cost ~25 instructions + a MUFU.RCP each, five per tile and warp: on layers
  // with one k-iteration per tile the kernel is ISSUE-bound on them): q = umulhi(x, mg) with mg = ceil(2^32 / d)
  unsigned mg_tiles_m, mg_tiles_n, mg_tilesW, mg_tilesH, mg_B;  // 0: divisor is 1 (or fast path not provable): see fdiv
  int epi_kind;         // host-only (no kernel reads it): the EKT of the instantiation tc_conv_launch runs, set there
  int n_fast;           // tile order: N tiles of one M tile are consecutive (1x1 convs with several N tiles, see tc_conv_create)
  int tiles_n;
  int rows_a_bytes;     // ROWS mode: bytes of one A box ((BH+2) x BW x 128)
  unsigned long long* dbg;  // optional [grid][8] cycle counters (IRSDE_TC_DEBUG=1)
  const bf16* res;
  int res_pitch;
  const float* bias;
  const float* mult_vec;
  const float* ss;
  const int* t_ptr;
  int ss_S, ss_off, ss_img_stride, silu;
  TcTap taps[16];
};

// ---- PTX wrappers ------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (fails the launch) instead of hanging the GPU.  No message is printed: printf
// compiles to a call of vprintf, and ptxas serializes every wgmma of a kernel whose wgmma window contains a function call
// (warning C7510: each HGMMA is then followed by a wait for zero groups in flight).  The consumers wait here while their
// previous stage's MMAs are still running, so the call must not exist; tests/test_conv_tc_sass.py checks that it does not.
// The launch is failed by a store to address 0 rather than by `trap`: a reachable trap makes ptxas hold the consumer
// warpgroups to the launch's 168 registers even after setmaxnreg has raised them to 232, and the ping-pong tiles spill.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  long long t0 = 0;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0xfffu) == 0) {
      long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000LL) asm volatile("st.global.u32 [%0], 0;" ::"l"(0ull) : "memory");  // ~2 s: fault
    }
  }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_5d(void* smem, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_u32(smem)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// sm_90 wgmma shared-memory matrix descriptor: K-major operand, 128B swizzle, rows of 128 bytes, 8-row core groups
// 1024 B apart (SBO).  Stepping K by 16 bf16 (or 8 tf32) inside the swizzle atom = +32 B on the start address (+2).
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);  // start address
  d |= (uint64_t)1 << 16;                       // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;             // stride byte offset between 8-row groups
  d |= (uint64_t)1 << 62;                       // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Pins the accumulator registers: no read of them is scheduled above a preceding wgmma.wait_group.
template <int N>
__device__ __forceinline__ void acc_fence(float* d) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, both K-major in shared memory, fp32 accumulator in registers; tf32: K = 8.
template <int N>
__device__ void wgmma_bf16(float* d, uint64_t a, uint64_t b);
template <int N>
__device__ void wgmma_tf32(float* d, uint64_t a, uint64_t b);
template <> __device__ __forceinline__ void wgmma_bf16<32>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_bf16<64>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_bf16<128>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_bf16<256>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a), "l"(b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_tf32<32>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_tf32<64>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_tf32<128>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(1));
}

constexpr int A_STAGE_BYTES = 128 * 128;  // 128 pixel rows x 64 bf16

// =====================================================================================================
// Persistent kernel: one CTA per SM loops over output tiles.  The smem ring is as deep as the 227 KB of shared memory
// allows (at most 8 stages) to cover TMA latency, and the prologue (barrier init, descriptor prefetch) is paid once per SM.
// =====================================================================================================
//
// ROWS mode (default for 3x3 stride-1 convs with BN <= 128): a stage is ONE TMA box of (BH+2) image rows x BW pixels
// for a given horizontal shift dw, plus the three weight tiles of the taps (dh=-1,0,1; dw).  The three vertical taps
// read 1024-byte-ALIGNED row windows of the same box (window dh starts (dh+1)*BW pixel rows in), so the A operand
// is fetched 3x instead of 9x per 64-channel chunk with ordinary aligned wgmma descriptors, and one full/empty
// barrier round covers 12 MMAs per warpgroup.
constexpr int TF3_SEG = 2;  // fp32x3: k-iterations (of 32 channels, 12 MMAs each) accumulated from zero before a fp32 sum
constexpr int ROWS_A_SLOT = 20 * 1024;  // (8+2) rows x 16 px x 128 B (or 18 x 8 px for narrow images)
constexpr int SMEM_LIMIT = 232448;      // 227 KB: the opt-in shared memory per block of sm_90

// MODE 3 "fp32x3" (the fp32-accurate tensor-core mode, SURVEY 7 "Parity vs precision"): operands are fp32 tensors that were
// split into hi = rn_tf32(x) and lo = rn_tf32(x - hi) (|x - hi - lo| <= 2^-22 |x|); a K chunk is 32 fp32 channels = the same
// 128-byte swizzled row as 64 bf16 channels; per chunk each warpgroup issues A_hi*W_hi + A_lo*W_hi + A_hi*W_lo as three
// groups of four tf32 wgmma (K=8) into the SAME fp32 accumulator (the dropped lo*lo term is 2^-22 relative).
// The epilogue keeps everything in fp32 (IEEE SiLU, fp32 residual, fp32 NHWC / NCHW stores).
template <int BN, int MODE>
struct TcCfgP {
  static constexpr bool ROWS = MODE == 2;
  static constexpr bool TF3 = MODE == 3;
  static constexpr int B_STAGE_BYTES = BN * 128;
  // PING-PONG schedule (bf16, BN = 64 / 128): a CTA's tiles alternate between the two consumer warpgroups, each computing
  // all 128 rows of its tile, so one warpgroup's epilogue runs while the other issues its MMAs.  BN = 256 (128 accumulator
  // registers per 64 rows), BN = 32 and fp32x3 keep the COOPERATIVE schedule: both warpgroups on one tile, 64 rows each.
  static constexpr bool PP = !TF3 && (BN == 64 || BN == 128);
  static constexpr int BSUB = ROWS ? 3 : (TF3 ? 2 : 1);  // weight tiles per stage
  static constexpr int A_SLOT = TF3 ? 2 * A_STAGE_BYTES : (ROWS ? ROWS_A_SLOT : A_STAGE_BYTES);
  static constexpr int STAGE_BYTES = A_SLOT + BSUB * B_STAGE_BYTES;
  static constexpr int EPI_FLOATS = 2 * 2 * BN;  // one (mult, add) table per consumer warpgroup
  // fp32x3 only: the accumulators pass through fp32 staging rows, 64 rows x 64 (+4: conflict-free 16-byte row reads)
  // columns per warpgroup.  The bf16 epilogue works on the accumulator registers.
  static constexpr int ACC_PITCH = 68;
  static constexpr int ACC_BYTES = TF3 ? 2 * 64 * ACC_PITCH * 4 : 0;
  // bf16: STG_BUFS store tiles per consumer warp, each 16 pixel rows x 32 channels (1 KB, 64B swizzle).  The ring takes
  // as many stages as fit next to two tiles, the tiles then take what the ring leaves (at most four).  Stages / tiles:
  // per-tap BN=256 / 128 / 64 / 32: 4/3, 6/3, 8/4, 8/4; ROWS BN=128 / 64 / 32: 3/2, 4/4, 6/4; fp32x3 BN=128 / 64 / 32: 2, 3, 4.
  static constexpr int STG_TILE = 1024;
  static constexpr int BAR_BYTES = 512;  // full and empty barriers of the ring, one residual barrier per store tile
  static constexpr int OTHER_BYTES = 1024 + ACC_BYTES + EPI_FLOATS * 4 + BAR_BYTES;
  static constexpr int STG_MIN = TF3 ? 0 : 2;
  static constexpr int STAGES_FIT = (SMEM_LIMIT - OTHER_BYTES - STG_MIN * 8 * STG_TILE) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 8 ? 8 : STAGES_FIT;
  static constexpr int STG_FIT = (SMEM_LIMIT - OTHER_BYTES - STAGES * STAGE_BYTES) / (8 * STG_TILE);
  static constexpr int STG_BUFS = TF3 ? 0 : (STG_FIT > 4 ? 4 : STG_FIT);
  static constexpr int STG_BYTES = STG_BUFS * 8 * STG_TILE;
  static constexpr int FIXED_BYTES = OTHER_BYTES + STG_BYTES;
  static constexpr int A_BYTES = STAGES * A_SLOT;
  static constexpr int SMEM_BYTES = FIXED_BYTES + STAGES * STAGE_BYTES;
  static_assert(STAGES >= 2, "shared memory holds fewer than two pipeline stages");
  static_assert(TF3 || STG_BUFS >= 2, "the bf16 epilogue needs two store tiles per warp");
  static_assert(2 * 8 + 8 * 4 <= BAR_BYTES / 8, "barrier area too small");
  static_assert(SMEM_BYTES <= SMEM_LIMIT, "over the 227 KB per-CTA shared memory limit");
  static_assert(!(BN == 256 && MODE == 0) || STAGES == 4, "per-tap BN=256 is meant to run a 4-stage ring");
  static_assert(!(BN == 128 && MODE == 2) || STAGES == 3, "ROWS BN=128 is meant to run a 3-stage ring");
};

// One elected lane of a converged warp (the compiler recognises elect.sync and emits straight-line uniform
// datapath code for the UTMA / UTCHMMA instructions under it, instead of per-active-thread ELECT loops).
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
      "elect.sync rx|px, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, px;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

struct OutMaps {
  CUtensorMap m[4];  // one per upsample phase (only m[0] otherwise)
};
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* smem, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(map),
               "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_4d(const CUtensorMap* map, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];" ::"l"(map), "r"(c0), "r"(c1), "r"(c2),
               "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the bulk stores this thread committed, except the N most recent, have finished reading shared memory
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// four 8 x 8 bf16 matrices in the mma fragment layout (lane l: row l / 4, columns 2 (l % 4), +1); lane l addresses row
// l % 8 of matrix l / 8
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, const uint32_t* r) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]),
               "r"(r[3])
               : "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t* r) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}

struct TileCoord {
  int b, phase, py, px, h0, w0, n0;
};
// x / d for 0 <= x with x * d < 2^32 (host-checked in tc_fill_magic; mg == 0 selects the plain division)
__device__ __forceinline__ int fdiv(int x, int d, unsigned mg) { return mg ? (int)__umulhi((unsigned)x, mg) : x / d; }
enum { EK_QSM = 1, EK_AFF = 2, EK_SILU = 4, EK_RES = 8, EK_GENERIC = 16 };

__device__ __forceinline__ void decode_m(const TcParams& P, int m_idx, TileCoord& t) {
  int q = fdiv(m_idx, P.tilesW, P.mg_tilesW);
  const int tw_i = m_idx - q * P.tilesW; m_idx = q;
  q = fdiv(m_idx, P.tilesH, P.mg_tilesH);
  const int th_i = m_idx - q * P.tilesH; m_idx = q;
  q = fdiv(m_idx, P.B, P.mg_B);
  t.b = m_idx - q * P.B;
  t.phase = q;
  t.py = t.phase >> 1; t.px = t.phase & 1;
  t.h0 = th_i * P.BH; t.w0 = tw_i * P.BW;
}
__device__ __forceinline__ TileCoord decode_tile(const TcParams& P, int tile, int tiles_m, int BN) {
  TileCoord t;
  int m_idx;
  if (P.n_fast) { m_idx = fdiv(tile, P.tiles_n, P.mg_tiles_n); t.n0 = (tile - m_idx * P.tiles_n) * BN; }
  else { const int q = fdiv(tile, tiles_m, P.mg_tiles_m); m_idx = tile - q * tiles_m; t.n0 = q * BN; }
  decode_m(P, m_idx, t);
  return t;
}

#define DBG_WAIT(ctr, bar, par)                 \
  do {                                          \
    if (P.dbg) {                                \
      long long _t0 = clock64();                \
      mbar_wait(bar, par);                      \
      ctr += (unsigned)(clock64() - _t0);       \
    } else {                                    \
      mbar_wait(bar, par);                      \
    }                                           \
  } while (0)


// EKT: EK_* features the epilogue is compiled for.  Only the per-tap and ROWS instantiations that serve the common layer kinds
// (res_conv: 0, to_qkv: EK_QSM, to_out: EK_AFF, ResBlock convs: EK_AFF|EK_SILU, EK_SILU|EK_RES) are specialised - there the
// kernel is issue-bound on epilogue instructions; everything else runs EK_GENERIC (every feature checked at run time).
constexpr int TC_THREADS = 384;  // consumer warpgroups 0 and 1, producer warpgroup 2 (warp 8 issues the TMA loads)
constexpr int TC_DBG_SLOTS = 16;  // IRSDE_TC_DEBUG counters per CTA

template <int BN, int MODE, int EKT = 16 /* EK_GENERIC */>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_persist_kernel(const __grid_constant__ CUtensorMap map_a,
                                                                 const __grid_constant__ CUtensorMap map_b,
                                                                 const __grid_constant__ OutMaps map_o,
                                                                 const __grid_constant__ OutMaps map_r,
                                                                 const __grid_constant__ TcParams P, int tiles_m,
                                                                 int num_tiles) {
  using Cfg = TcCfgP<BN, MODE>;
  constexpr bool ROWS = Cfg::ROWS;
  constexpr bool TF3 = Cfg::TF3;
  constexpr int STAGES = Cfg::STAGES;
  constexpr bool PP = Cfg::PP;
  constexpr int NACC = BN / 2;  // accumulator registers per thread for one m64 x BN block
  constexpr int MH = PP ? 2 : 1;  // 64-row halves of a tile held by one warpgroup
  pdl_trigger();  // the next kernel may be scheduled; this one's prologue below touches no global memory
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* smem_a = smem;                       // A ring
  uint8_t* smem_b = smem + Cfg::A_BYTES;
  uint8_t* smem_stg = smem_b + STAGES * Cfg::BSUB * Cfg::B_STAGE_BYTES;  // 1024-aligned: bf16 store tiles
  float* s_acc = reinterpret_cast<float*>(smem_stg + Cfg::STG_BYTES);       // fp32x3 staging rows
  float* s_epi = s_acc + Cfg::ACC_BYTES / 4;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_epi + Cfg::EPI_FLOATS);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int KI = P.ntaps * P.kchunks;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], PP ? 1 : 2);  // one arrive per warpgroup that reads the stage
    }
    for (int i = 0; i < 8 * Cfg::STG_BUFS; ++i) mbar_init(&bars[2 * STAGES + i], 1);  // residual loads into store tiles
    fence_barrier_init();
  }
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
  }
  __syncthreads();
  // barriers and descriptors are ready: from here on global memory written by the previous kernel is read
  // (activations, the device step counter behind P.t_ptr) and buffers it may still be reading are overwritten
  pdl_wait();

  // Register split (128 x 40 + 256 x 232 <= 64 K): the launch gives every thread 168, the producer warpgroup hands its
  // surplus to the consumers, whose ping-pong tiles keep 2 x BN / 2 accumulators per thread.
  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp != 8) return;
    // ================= TMA producer (whole warp loops; one elected lane issues) =================
    int it = 0;
    long long w_prod = 0, t_start = clock64();
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(P, tile, tiles_m, BN);
      if constexpr (TF3) {
        for (int ki = 0; ki < KI; ++ki, ++it) {
          const int s = it % STAGES;
          if (it >= STAGES) DBG_WAIT(w_prod, &empty_bar[s], ((it / STAGES) - 1) & 1);
          if (elect_one()) {
            const int tap = ki / P.kchunks, kc = ki - tap * P.kchunks;
            const int dh = P.taps[tap].dh + (P.nphases == 4 ? t.py : 0);
            const int dw = P.taps[tap].dw + (P.nphases == 4 ? t.px : 0);
            const int wt = (t.phase * P.ntaps + tap) * 2;
            mbar_expect_tx(&full_bar[s], 2 * A_STAGE_BYTES + 2 * Cfg::B_STAGE_BYTES);
            tma_load_5d(smem_a + (s * 2 + 0) * A_STAGE_BYTES, &map_a, &full_bar[s], kc * 32, t.w0 + dw, t.h0 + dh, t.b, P.taps[tap].plane);
            tma_load_5d(smem_a + (s * 2 + 1) * A_STAGE_BYTES, &map_a, &full_bar[s], kc * 32, t.w0 + dw, t.h0 + dh, t.b,
                        P.taps[tap].plane + P.lo_plane_off);
            tma_load_3d(smem_b + (s * 2 + 0) * Cfg::B_STAGE_BYTES, &map_b, &full_bar[s], kc * 32, t.n0, wt);
            tma_load_3d(smem_b + (s * 2 + 1) * Cfg::B_STAGE_BYTES, &map_b, &full_bar[s], kc * 32, t.n0, wt + 1);
          }
          __syncwarp();
        }
      } else if constexpr (ROWS) {
        for (int kc = 0; kc < P.kchunks; ++kc) {
          for (int dwi = 0; dwi < 3; ++dwi, ++it) {
            const int s = it % STAGES;
            if (it >= STAGES) DBG_WAIT(w_prod, &empty_bar[s], ((it / STAGES) - 1) & 1);
            if (elect_one()) {
              mbar_expect_tx(&full_bar[s], P.rows_a_bytes + 3 * Cfg::B_STAGE_BYTES);
              tma_load_5d(smem_a + s * ROWS_A_SLOT, &map_a, &full_bar[s], kc * 64, t.w0 + dwi - 1, t.h0 - 1, t.b, 0);
#pragma unroll
              for (int j = 0; j < 3; ++j)  // taps (dh = j-1, dw = dwi-1): index (dh+1)*3 + (dw+1)
                tma_load_3d(smem_b + (s * 3 + j) * Cfg::B_STAGE_BYTES, &map_b, &full_bar[s], kc * 64, t.n0, j * 3 + dwi);
            }
            __syncwarp();
          }
        }
      } else {
        for (int ki = 0; ki < KI; ++ki, ++it) {
          const int s = it % STAGES;
          if (it >= STAGES) DBG_WAIT(w_prod, &empty_bar[s], ((it / STAGES) - 1) & 1);
          if (elect_one()) {
            const int tap = ki / P.kchunks, kc = ki - tap * P.kchunks;
            const int dh = P.taps[tap].dh + (P.nphases == 4 ? t.py : 0);
            const int dw = P.taps[tap].dw + (P.nphases == 4 ? t.px : 0);
            mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
            tma_load_5d(smem_a + s * A_STAGE_BYTES, &map_a, &full_bar[s], kc * 64, t.w0 + dw, t.h0 + dh, t.b, P.taps[tap].plane);
            tma_load_3d(smem_b + s * Cfg::B_STAGE_BYTES, &map_b, &full_bar[s], kc * 64, t.n0,
                        t.phase * P.ntaps + tap + (P.w_per_image ? t.b : 0));
          }
          __syncwarp();
        }
      }
    }
    if (P.dbg && lane == 0) {
      P.dbg[blockIdx.x * TC_DBG_SLOTS + 0] = (unsigned long long)w_prod;
      P.dbg[blockIdx.x * TC_DBG_SLOTS + 1] = (unsigned long long)(clock64() - t_start);
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");

  // ================= consumers =================
  // COOPERATIVE: warpgroup wg owns pixel rows 64*wg .. 64*wg+63 of every tile.  PING-PONG: warpgroup wg owns every row of
  // the CTA's tiles lt with lt & 1 == wg; their turns at the tensor cores alternate through named barriers 4 + wg (below).
  const int wg = warp >> 2;
  const int wq = warp & 3;               // wgmma layout: this warp holds accumulator rows 16*wq + lane/4 (+8)
  const int et = threadIdx.x & 127;
  const int trow = P.t_ptr ? *P.t_ptr : 0;
  const bool affine = (P.ss != nullptr) || (P.bias != nullptr) || (P.mult_vec != nullptr);
  float* const epi = s_epi + wg * 2 * BN;  // this warpgroup's (mult, add) table
  const uint32_t a_off = PP ? 0u : (uint32_t)(wg * 64 * 128);  // cooperative: this warpgroup's 64 pixel rows of every A box
  const int NST = ROWS ? 3 * P.kchunks : KI;  // ring stages per tile
  const bool signaller = (threadIdx.x & 127) == 0;
  unsigned w_full = 0, w_turn = 0, c_epi = 0;  // debug cycle counts: 32 bits span a launch many times over
  const unsigned t_start = (unsigned)clock();
  // bf16 epilogue: the warp's output goes out in blocks of its 16 accumulator rows x 32 channels, block q of the launch
  // through store tile q % NBUF, whose barrier res_bar[q % NBUF] signals the block's residual (TMA-loaded into that tile)
  constexpr int NBUF = TF3 ? 1 : Cfg::STG_BUFS;  // (fp32x3 has no store tiles)
  constexpr bool GEN = EKT == EK_GENERIC;
  uint8_t* const stg = smem_stg + warp * NBUF * Cfg::STG_TILE;
  uint64_t* const res_bar = bars + 2 * STAGES + warp * NBUF;
  const bool has_res = !TF3 && (GEN ? (P.res != nullptr && P.out_nchw == nullptr) : (EKT & EK_RES) != 0);
  // stmatrix / ldmatrix address of this lane in a store tile: row lane % 8 of 16-byte chunk lane / 8, 64B swizzle
  const uint32_t frag_off = (uint32_t)((lane & 7) * 64 + (((lane >> 3) ^ ((lane >> 1) & 3)) << 4));
  unsigned blk = 0;
  int it = 0, lt = 0, epi_n0 = -1, epi_b = -1;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++lt) {
    if (PP && (lt & 1) != wg) continue;
    it = lt * NST;  // the ring position of the tile's first stage (the other warpgroup consumed the stages in between)
    const TileCoord t = decode_tile(P, tile, tiles_m, BN);
    // this warp's output blocks of the tile: nblk 32-channel blocks (those below Cout) per 64-row half, halves in order
    const int nblk = (P.Cout - t.n0 + 31) / 32 < BN / 32 ? (P.Cout - t.n0 + 31) / 32 : BN / 32;
    const int NB = MH * nblk;
    // TMA coordinates of block i (c: channel, x, y: image column and row of its first pixel)
    auto blk_coord = [&](int i, int& c, int& x, int& y) __attribute__((always_inline)) {
      const int h = (MH == 2 && i >= nblk) ? 1 : 0;
      const int m0 = (PP ? h : wg) * 64 + wq * 16;
      c = t.n0 + (i - h * nblk) * 32;
      x = t.w0 + (m0 & (P.BW - 1));
      y = t.h0 + (m0 >> P.logBW);
    };
    auto res_load = [&](int i) __attribute__((always_inline)) {  // lane 0: block i's residual into its store tile
      int c, x, y;
      blk_coord(i, c, x, y);
      const unsigned q = blk + (unsigned)i;
      mbar_expect_tx(&res_bar[q % NBUF], Cfg::STG_TILE);
      tma_load_4d(stg + (q % NBUF) * Cfg::STG_TILE, &map_r.m[t.phase], &res_bar[q % NBUF], c, x, y, t.b);
    };
    // Residual fetched ahead, before the main loop: the first NBUF - 1 blocks into the (idle) store tiles, the rest of
    // the tile's residual into L2.  Block i + NBUF - 1 is loaded once block i is stored.
    if constexpr (!TF3) {
      if (has_res && lane == 0) {
        bulk_wait_read<0>();
        for (int i = 0; i < NB; ++i) {
          if (i < NBUF - 1) {
            res_load(i);
          } else {
            int c, x, y;
            blk_coord(i, c, x, y);
            tma_prefetch_4d(&map_r.m[t.phase], c, x, y, t.b);
          }
        }
      }
    }
    float acc[MH][NACC];
    float sum[TF3 ? NACC : 1];  // fp32x3: the tile's K segments summed with round-to-nearest adds
#pragma unroll
    for (int h = 0; h < MH; ++h)
#pragma unroll
      for (int r = 0; r < NACC; ++r) acc[h][r] = 0.f;
#pragma unroll
    for (int r = 0; r < (TF3 ? NACC : 1); ++r) sum[r] = 0.f;
    // Ping-pong turn: wait until the other warpgroup has waited on every full barrier of the previous tile.  Besides
    // ordering the MMAs, this is what makes the parity waits exact: a warpgroup that ran ahead could otherwise wait on
    // a slot whose previous fill (the other warpgroup's stage it - STAGES) has not landed yet, and the phase bit of that
    // barrier would already read as "this fill complete".
    if constexpr (PP) {
      if (lt > 0) {
        const unsigned t0 = (unsigned)clock();
        asm volatile("bar.sync %0, 256;" ::"r"(4 + wg) : "memory");
        w_turn += (unsigned)clock() - t0;
      }
    }
    auto pass_turn = [&]() __attribute__((always_inline)) {  // after the tile's last full-barrier wait
      if constexpr (PP)
        if (tile + (int)gridDim.x < num_tiles) asm volatile("bar.arrive %0, 256;" ::"r"(4 + (wg ^ 1)) : "memory");
    };
    // one stage: wait for its bytes, issue this warpgroup's MMAs on it, then release the PREVIOUS stage once its MMAs have
    // finished reading shared memory (one wgmma group stays in flight)
    int prev_s = -1;
    auto stage_begin = [&](int s) __attribute__((always_inline)) {
      DBG_WAIT(w_full, &full_bar[s], (it / STAGES) & 1);
      wgmma_fence();
    };
    auto stage_end = [&](int s) __attribute__((always_inline)) {
      wgmma_commit();
      wgmma_wait<1>();
      if (prev_s >= 0 && signaller) mbar_arrive(&empty_bar[prev_s]);
      prev_s = s;
      ++it;
    };
    auto drain = [&]() __attribute__((always_inline)) {
      wgmma_wait<0>();
#pragma unroll
      for (int h = 0; h < MH; ++h) acc_fence<NACC>(acc[h]);
      if (prev_s >= 0 && signaller) mbar_arrive(&empty_bar[prev_s]);
      prev_s = -1;
    };
    if constexpr (TF3) {
      // fp32x3: the K loop of a tile is cut into SEGMENTS of TF3_SEG k-iterations; each segment accumulates from zero and is
      // added to `sum` with round-to-nearest adds.  Reason: the tensor core's accumulator update truncates, so a single
      // accumulation over n MMAs drifts by ~n * 2^-26 relative (3e-5 per layer at K = 13 824); 24 MMAs per segment keep
      // it at the fp32 FMA path's own level.
      for (int k0 = 0; k0 < KI; k0 += TF3_SEG) {
        const int k1 = k0 + TF3_SEG < KI ? k0 + TF3_SEG : KI;
        for (int ki = k0; ki < k1; ++ki) {
          const int s = it % STAGES;
          stage_begin(s);
          const uint64_t a_hi = make_sw128_desc(smem_u32(smem_a + (s * 2 + 0) * A_STAGE_BYTES) + a_off);
          const uint64_t a_lo = make_sw128_desc(smem_u32(smem_a + (s * 2 + 1) * A_STAGE_BYTES) + a_off);
          const uint64_t b_hi = make_sw128_desc(smem_u32(smem_b + (s * 2 + 0) * Cfg::B_STAGE_BYTES));
          const uint64_t b_lo = make_sw128_desc(smem_u32(smem_b + (s * 2 + 1) * Cfg::B_STAGE_BYTES));
          // the two small cross terms first, the dominant hi*hi product last
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_tf32<BN>(acc[0], a_lo + (uint64_t)(k * 2), b_hi + (uint64_t)(k * 2));
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_tf32<BN>(acc[0], a_hi + (uint64_t)(k * 2), b_lo + (uint64_t)(k * 2));
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_tf32<BN>(acc[0], a_hi + (uint64_t)(k * 2), b_hi + (uint64_t)(k * 2));
          stage_end(s);
        }
        drain();
#pragma unroll
        for (int r = 0; r < NACC; ++r) {
          sum[(TF3 ? r : 0)] = __fadd_rn(sum[(TF3 ? r : 0)], acc[0][r]);
          acc[0][r] = 0.f;
        }
      }
    } else if constexpr (ROWS) {
      for (int si = 0; si < NST; ++si) {
        const int s = it % STAGES;
        stage_begin(s);
        const uint32_t a0 = smem_u32(smem_a + s * ROWS_A_SLOT) + a_off;
#pragma unroll
        for (int j = 0; j < 3; ++j) {  // vertical tap dh = j-1: row window starting j*BW pixel rows into the box
          const uint64_t bdesc = make_sw128_desc(smem_u32(smem_b + (s * 3 + j) * Cfg::B_STAGE_BYTES));
#pragma unroll
          for (int h = 0; h < MH; ++h) {
            const uint64_t adesc = make_sw128_desc(a0 + (uint32_t)(j * P.BW * 128 + h * 64 * 128));
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_bf16<BN>(acc[h], adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2));
          }
        }
        stage_end(s);
      }
      pass_turn();
      drain();
    } else {
      for (int ki = 0; ki < KI; ++ki) {
        const int s = it % STAGES;
        stage_begin(s);
        const uint64_t bdesc = make_sw128_desc(smem_u32(smem_b + s * Cfg::B_STAGE_BYTES));
#pragma unroll
        for (int h = 0; h < MH; ++h) {
          const uint64_t adesc = make_sw128_desc(smem_u32(smem_a + s * A_STAGE_BYTES) + a_off + (uint32_t)(h * 64 * 128));
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_bf16<BN>(acc[h], adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2));
        }
        stage_end(s);
      }
      pass_turn();
      drain();
    }

    // ---- epilogue
    const unsigned t_epi = (unsigned)clock();
    // The per-channel (mult, add) table depends on the N tile (and on the image only with per-image timesteps):
    // rebuild it - two warpgroup barriers and a dependent global load - only when that changes.
    const int key_b = P.ss_img_stride ? t.b : 0;
    if (affine && (t.n0 != epi_n0 || key_b != epi_b)) {
      epi_n0 = t.n0; epi_b = key_b;
      asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");  // previous tile's reads of the table are done
      const float* ssrow = P.ss ? P.ss + (long long)(trow + t.b * P.ss_img_stride) * P.ss_S + P.ss_off : nullptr;
      for (int j = et; j < BN; j += 128) {
        const int n = t.n0 + j;
        float mult = 1.f, add = 0.f, bias = 0.f;
        if (n < P.Cout) {
          if (ssrow) { mult = ssrow[n] + 1.0f; add = ssrow[P.Cout + n]; }
          if (P.mult_vec) mult *= P.mult_vec[n];
          if (P.bias) bias = P.bias[n];
        }
        epi[j] = mult; epi[BN + j] = bias * mult + add;  // (x + bias) * mult + add == x * mult + (bias * mult + add)
      }
      asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
    }
    if constexpr (TF3) {
      // fp32 in, fp32 out, IEEE arithmetic: one 64-row half of the tile per pass through this warpgroup's staging rows,
      // then per lane one pixel x 32 channels
      constexpr int ACC_PITCH = Cfg::ACC_PITCH;
      float* const acc_stg = s_acc + wg * 64 * ACC_PITCH;
      const int half = wq >> 1;  // 32-channel chunks alternate by `half`
      const int m = (wg * 2 + (wq & 1)) * 32 + lane;  // pixel of the tile
      const int hh = t.h0 + (m >> P.logBW), ww = t.w0 + (m & (P.BW - 1));
      const bool pvalid = hh < P.H && ww < P.W;
      const long long opix = ((long long)t.b * P.Hout + (hh * P.os + t.py)) * P.Wout + (ww * P.os + t.px);
      auto process = [&](uint32_t* v, const int c0) __attribute__((always_inline)) {
        if (affine) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = __float_as_uint(fmaf(__uint_as_float(v[j]), epi[c0 + j], epi[BN + c0 + j]));
        }
        if (P.silu) {
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const float x = __uint_as_float(v[j]);
            v[j] = __float_as_uint(x / (1.0f + expf(-x)));
          }
        }
        if (P.out_nchw) {
          if (pvalid && hh < P.cropH && ww < P.cropW) {
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              const int n = t.n0 + c0 + j;
              if (n < P.Cout) P.out_nchw[(((long long)t.b * P.Cout + n) * P.cropH + hh) * P.cropW + ww] = __uint_as_float(v[j]);
            }
          }
          return;
        }
        if (!pvalid) return;
        float* of = P.out_f32 + opix * P.out_pitch + t.n0 + c0;
        const float* rf = P.res_f32 ? P.res_f32 + opix * P.res_pitch + t.n0 + c0 : nullptr;
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          if (t.n0 + c0 + g * 4 < P.Cout) {
            float4 o = make_float4(__uint_as_float(v[g * 4]), __uint_as_float(v[g * 4 + 1]), __uint_as_float(v[g * 4 + 2]),
                                   __uint_as_float(v[g * 4 + 3]));
            if (rf) {
              const float4 r = *reinterpret_cast<const float4*>(rf + g * 4);
              o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
            }
            *reinterpret_cast<float4*>(of + g * 4) = o;
          }
        }
      };
      constexpr int NR = (BN + 63) / 64;
#pragma unroll
      for (int i = 0; i < NR; ++i) {
        asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");  // this warpgroup's previous reads of the staging rows are done
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = i * 8 + jj;  // n8 block of the accumulator: registers 4j .. 4j+3
          if (j * 8 < BN) {
            const int row = wq * 16 + (lane >> 2), col = jj * 8 + 2 * (lane & 3);
            *reinterpret_cast<float2*>(acc_stg + row * ACC_PITCH + col) = make_float2(sum[4 * j], sum[4 * j + 1]);
            *reinterpret_cast<float2*>(acc_stg + (row + 8) * ACC_PITCH + col) = make_float2(sum[4 * j + 2], sum[4 * j + 3]);
          }
        }
        asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
        const int c0 = i * 64 + half * 32;
        if (c0 < BN && t.n0 + c0 < P.Cout) {  // chunks entirely past Cout carry no output
          uint32_t v[32];
          const float* src = acc_stg + ((wq & 1) * 32 + lane) * ACC_PITCH + half * 32;
#pragma unroll
          for (int g = 0; g < 8; ++g) {
            const float4 f = *reinterpret_cast<const float4*>(src + 4 * g);
            v[4 * g] = __float_as_uint(f.x); v[4 * g + 1] = __float_as_uint(f.y);
            v[4 * g + 2] = __float_as_uint(f.z); v[4 * g + 3] = __float_as_uint(f.w);
          }
          process(v, c0);
        }
      }
    } else {
      // bf16: on the accumulator registers.  Thread (wq, lane) holds rows 16 wq + lane / 4 + 8 i (i = 0, 1) of each 64-row
      // half and, per n8 block j, the channel pair 8 j + 2 (lane % 4) + e: register 4 j + 2 i + e.  Block (h, cb) is the
      // 16 rows x channels 32 cb .. 32 cb + 31 of half h.  EKT: the EK_* features compiled in (feature blocks outside it
      // do not exist in the instantiation); EK_GENERIC keeps every run-time check and the fp32 NCHW output.
      const int cq = 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < MH; ++h) {
#pragma unroll
        for (int cb = 0; cb < BN / 32; ++cb) {
          if (cb >= nblk) continue;  // blocks entirely past Cout carry no output
          float* const v = &acc[h][cb * 16];
          const int c0 = cb * 32;
          const int i = h * nblk + cb;
          const unsigned q = blk + (unsigned)i;
          if constexpr (GEN || (EKT & EK_QSM)) if ((!GEN || P.qsm) && t.n0 + c0 < 128) {
            // one block row == one attention head of a pixel's q (module_util.py:168,171), spread over four lanes; its
            // sum is taken in channel order 0 .. 31 by each of them
#pragma unroll
            for (int r = 0; r < 2; ++r) {
              float mx = v[2 * r];
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) mx = fmaxf(fmaxf(mx, v[4 * jj + 2 * r]), v[4 * jj + 2 * r + 1]);
              mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
              mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
#pragma unroll
              for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                for (int e = 0; e < 2; ++e) v[4 * jj + 2 * r + e] = __expf(v[4 * jj + 2 * r + e] - mx);
              float sm = 0.f;
#pragma unroll
              for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                for (int l4 = 0; l4 < 4; ++l4)
#pragma unroll
                  for (int e = 0; e < 2; ++e) sm += __shfl_sync(0xffffffffu, v[4 * jj + 2 * r + e], (lane & ~3) | l4);
              const float inv = __fdividef(0.17677669529663687f, sm);
#pragma unroll
              for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                for (int e = 0; e < 2; ++e) v[4 * jj + 2 * r + e] = v[4 * jj + 2 * r + e] * inv;
            }
          }
          if constexpr (GEN || (EKT & EK_AFF)) if (!GEN || affine) {
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const float2 mu = *reinterpret_cast<const float2*>(epi + c0 + 8 * jj + cq);
              const float2 ad = *reinterpret_cast<const float2*>(epi + BN + c0 + 8 * jj + cq);
#pragma unroll
              for (int r = 0; r < 2; ++r) {
                v[4 * jj + 2 * r] = fmaf(v[4 * jj + 2 * r], mu.x, ad.x);
                v[4 * jj + 2 * r + 1] = fmaf(v[4 * jj + 2 * r + 1], mu.y, ad.y);
              }
            }
          }
          if constexpr (GEN || (EKT & EK_SILU)) if (!GEN || P.silu) {
#pragma unroll
            for (int k = 0; k < 16; ++k) {
              // SiLU(x) = x * (0.5 + 0.5 tanh(x/2)): one MUFU op (tanh.approx, rel. error 2^-11 << bf16 rounding) instead of
              // ex2 + rcp; on the narrow layers the epilogue is MUFU-bound (128 x BN outputs per tile, 16 MUFU/clk/SM)
              const float x = v[k];
              float th;
              asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(0.5f * x));
              v[k] = x * fmaf(th, 0.5f, 0.5f);
            }
          }
          if constexpr (GEN) if (P.out_nchw) {  // fp32 NCHW, cropped
#pragma unroll
            for (int r = 0; r < 2; ++r) {
              const int m = (PP ? h : wg) * 64 + wq * 16 + (lane >> 2) + 8 * r;
              const int hh = t.h0 + (m >> P.logBW), ww = t.w0 + (m & (P.BW - 1));
              if (hh < P.H && ww < P.W && hh < P.cropH && ww < P.cropW) {
#pragma unroll
                for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                  for (int e = 0; e < 2; ++e) {
                    const int n = t.n0 + c0 + 8 * jj + cq + e;
                    if (n < P.Cout) P.out_nchw[(((long long)t.b * P.Cout + n) * P.cropH + hh) * P.cropW + ww] = v[4 * jj + 2 * r + e];
                  }
              }
            }
            continue;
          }
          uint8_t* const tile_s = stg + (q % NBUF) * Cfg::STG_TILE;
          const uint32_t fa = smem_u32(tile_s) + frag_off;
          uint32_t rv[8];  // residual, bf16 pairs: [4 r + jj]
          if constexpr (GEN || (EKT & EK_RES)) if (has_res) {
            mbar_wait(&res_bar[q % NBUF], (q / NBUF) & 1);
            ldmatrix_x4(fa, rv);
            ldmatrix_x4(fa + 512, rv + 4);
#pragma unroll
            for (int jj = 0; jj < 4; ++jj)
#pragma unroll
              for (int r = 0; r < 2; ++r) {
                const __nv_bfloat162 r2 = *reinterpret_cast<const __nv_bfloat162*>(&rv[4 * r + jj]);
                v[4 * jj + 2 * r] += __low2float(r2);
                v[4 * jj + 2 * r + 1] += __high2float(r2);
              }
          }
          uint32_t ov[8];  // [4 r + jj]: matrix jj of rows 8 r .. 8 r + 7
#pragma unroll
          for (int jj = 0; jj < 4; ++jj)
#pragma unroll
            for (int r = 0; r < 2; ++r) {
              const __nv_bfloat162 o2 = __floats2bfloat162_rn(v[4 * jj + 2 * r], v[4 * jj + 2 * r + 1]);
              ov[4 * r + jj] = *reinterpret_cast<const uint32_t*>(&o2);
            }
          if (!has_res) {  // with a residual, its load into the tile already waited for the tile's previous store
            if (lane == 0) bulk_wait_read<NBUF - 1>();  // the store of block q - NBUF has read the tile
            __syncwarp();
          }
          stmatrix_x4(fa, ov);
          stmatrix_x4(fa + 512, ov + 4);
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) {
            int c, x, y;
            blk_coord(i, c, x, y);
            tma_store_4d(&map_o.m[t.phase], tile_s, c, x, y, t.b);
            bulk_commit();
            if (has_res && i + NBUF - 1 < NB) {
              bulk_wait_read<1>();  // the store of block q - 1 has read tile (q + NBUF - 1) % NBUF
              res_load(i + NBUF - 1);
            }
          }
        }
      }
      blk += (unsigned)NB;
    }
    if (P.dbg) c_epi += (unsigned)clock() - t_epi;
  }
  if (lane == 0) bulk_wait_all();  // staging smem must stay valid until the last bulk store has read it
  if (P.dbg && signaller) {
    unsigned long long* dbg = P.dbg + blockIdx.x * TC_DBG_SLOTS;
    dbg[2 + wg] = (unsigned long long)w_full;
    dbg[4 + wg] = (unsigned long long)c_epi;
    dbg[6 + wg] = (unsigned long long)w_turn;
    dbg[8 + wg] = (unsigned long long)((unsigned)clock() - t_start);
    dbg[10 + wg] = (unsigned long long)(PP ? (lt + 1 - wg) / 2 : lt);  // this warpgroup's tiles
  }
}

int g_num_sms = 132;

}  // namespace

struct TcConvDesc {
  CUtensorMap map_a, map_b;
  OutMaps map_o, map_r;  // bf16 output and residual views, one map per upsample phase
  TcParams P;
  int BN;
  dim3 grid;
  int tiles_m, num_tiles;
  int mode;  // 0 per-tap boxes, 2 ROWS (row-window reuse), 3 fp32x3
};

// One row per compiled conv_tc_persist_kernel instantiation: tc_init sets each row's shared memory, tc_pick chooses the row
// a descriptor runs.  An instantiation is added or removed here and nowhere else; tests/test_conv_tc_sass.py checks that
// tests/test_gpu_conv_epilogues.py has a case for each.
struct TcKernel {
  int BN, mode, ekt;
  void (*fn)(CUtensorMap, CUtensorMap, OutMaps, OutMaps, TcParams, int, int);
  int smem;
};
template <int BN, int MODE, int EKT = EK_GENERIC>
static TcKernel tc_kernel() {
  return TcKernel{BN, MODE, EKT, conv_tc_persist_kernel<BN, MODE, EKT>, TcCfgP<BN, MODE>::SMEM_BYTES};
}
static const TcKernel TC_KERNELS[] = {
    tc_kernel<32, 0>(),
    tc_kernel<64, 0>(),  tc_kernel<64, 0, 0>(),  tc_kernel<64, 0, EK_AFF>(),
    tc_kernel<128, 0>(), tc_kernel<128, 0, 0>(), tc_kernel<128, 0, EK_AFF>(), tc_kernel<128, 0, EK_QSM>(),
    tc_kernel<256, 0>(), tc_kernel<256, 0, 0>(), tc_kernel<256, 0, EK_AFF>(),  // deep res_conv; downsample / to_out (bias)
    tc_kernel<32, 2>(),
    tc_kernel<64, 2>(),  tc_kernel<64, 2, EK_AFF | EK_SILU>(),  tc_kernel<64, 2, EK_SILU | EK_RES>(),
    tc_kernel<128, 2>(), tc_kernel<128, 2, EK_AFF | EK_SILU>(), tc_kernel<128, 2, EK_SILU | EK_RES>(),
    tc_kernel<32, 3>(),  tc_kernel<64, 3>(),  tc_kernel<128, 3>(),
};

// The row that runs d now: the one compiled for exactly the epilogue features d uses, else the EK_GENERIC row of its
// (BN, mode).  fp32x3 and the fp32 NCHW output always run EK_GENERIC.  The time-modulation table (EK_AFF) usually arrives
// after create, through tc_conv_set_runtime, so this is decided at launch; tc_conv_query asks the same function.
static const TcKernel* tc_pick(const TcConvDesc* d) {
  const TcParams& P = d->P;
  int ek = EK_GENERIC;
  if (d->mode != 3 && P.out)
    ek = (P.qsm ? EK_QSM : 0) | (P.ss || P.bias || P.mult_vec ? EK_AFF : 0) | (P.silu ? EK_SILU : 0) | (P.res ? EK_RES : 0);
  const TcKernel* generic = nullptr;
  for (const TcKernel& k : TC_KERNELS) {
    if (k.BN != d->BN || k.mode != d->mode) continue;
    if (k.ekt == ek) return &k;
    if (k.ekt == EK_GENERIC) generic = &k;
  }
  return generic;
}

bool tc_init(std::string* err) {
  if (g_encode) return true;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
    if (err) *err = "cuTensorMapEncodeTiled not available from the driver";
    return false;
  }
  g_encode = (EncodeTiledFn)fn;
  for (const TcKernel& k : TC_KERNELS) cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, k.smem);
  {
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) g_num_sms = n;
    const char* e = getenv("IRSDE_PDL");
    g_pdl = (e && e[0] == '1');  // opt-in (see common.cuh)
  }
  cudaError_t le = cudaGetLastError();
  if (le != cudaSuccess) {
    if (err) *err = std::string("cudaFuncSetAttribute failed: ") + cudaGetErrorString(le);
    g_encode = nullptr;
    return false;
  }
  return true;
}

// tile-decode multipliers of a finished descriptor
static void tc_fill_magic(TcConvDesc* d) {
  TcParams& P = d->P;
  const unsigned long long max_x = (unsigned long long)d->num_tiles + 2;
  auto mg = [&](int dv) -> unsigned {
    if (dv <= 1) return 0u;                                       // x / 1: fdiv falls back to the (free) plain division
    if (max_x * (unsigned long long)dv >= (1ull << 32)) return 0u;  // exactness not provable: plain division
    return (unsigned)(((1ull << 32) + (unsigned)dv - 1) / (unsigned)dv);
  };
  P.mg_tiles_m = mg(d->tiles_m);
  P.mg_tiles_n = mg(P.tiles_n);
  P.mg_tilesW = mg(P.tilesW);
  P.mg_tilesH = mg(P.tilesH);
  P.mg_B = mg(P.B);
}

// cuTensorMapEncodeTiled with unit element strides, no interleave and zero out-of-bounds fill; on failure *err names `what`
static bool tc_encode(CUtensorMap* map, CUtensorMapDataType type, cuuint32_t rank, const void* base, const cuuint64_t* dims,
                      const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2,
                      const char* what, std::string* err) {
  const cuuint32_t es[5] = {1, 1, 1, 1, 1};
  const CUresult r = g_encode(map, type, rank, (void*)base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_SUCCESS) return true;
  if (err) { char b[96]; snprintf(b, sizeof b, "cuTensorMapEncodeTiled(%s) failed: %d", what, (int)r); *err = b; }
  return false;
}

// Both storage types share every step; what depends on the element size follows from S (a K chunk is one 128-byte swizzled
// row: 64 bf16 or 32 fp32 channels; 16 bytes are 8 or 4 elements), and what only bf16 has is marked so.
template <typename S>
TcConvDesc* tc_conv_create(const S* in, int in_pitch, int B, int Hin, int Win, int Cin, int planes, const S* w, int Cout, int ntaps,
                           const TcTap* taps, int nphases, const Epilogue& ep, S* out, int out_pitch, int Hout, int Wout,
                           std::string* err, int flags) {
  constexpr bool f32 = std::is_same<S, float>::value;
  constexpr int es = sizeof(S), al = 16 / es, kc = 128 / es;  // element bytes, elements per 16 bytes, channels per K chunk
  constexpr CUtensorMapDataType dtype = f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  auto bad = [&](const char* m) -> TcConvDesc* {
    if (err) *err = m;
    return nullptr;
  };
  if (!g_encode) return bad("tc_init not called");
  if (ntaps < 1 || ntaps > 16) return bad("ntaps out of range");
  if (f32 && planes < 1) return bad("planes must be >= 1");  // the 7x7 stem is bf16 only
  if (f32 && flags) return bad("the q-softmax and per-image weights are bf16 only");
  if ((flags & TC_FLAG_W_PER_IMAGE) && (ntaps != 1 || nphases != 1)) return bad("per-image weights need a 1x1 conv");
  // 7x7 stem "row trick" (planes < 0): the input is a zero-bordered [B][H+6][W+8][8ch] buffer; one GEMM K-chunk of 64
  // elements = 8 consecutive pixels x 8 channels of one input row (overlapping pixel stride of 16 B), so kernel row r is a
  // single tap (dh=r) and K = 7 x 64.
  if (planes < 0) Cin = 64;
  const bool nchw_out = (out == nullptr);  // caller sets the fp32 NCHW pointer at launch (tc_conv_set_out_nchw)
  const int Cout_w = (Cout + 7) / 8 * 8;   // rows of the packed weight tensor (zero padded)
  if (Cin % al || in_pitch % al) return bad("input channel count / pitch must be multiples of 16 bytes");
  if (!nchw_out && (Cout % al || out_pitch % al)) return bad("output channel count / pitch must be multiples of 16 bytes");
  if (((uintptr_t)in & 15) || ((uintptr_t)w & 15) || ((uintptr_t)out & 15)) return bad("operands must be 16-byte aligned");
  if (ep.res && (((uintptr_t)ep.res & 15) || ep.res_pitch % al)) return bad("residual must be 16-byte aligned");
  if (ep.ss && ep.mult_vec) return bad("the time-modulation table and mult_vec cannot be combined");
  std::unique_ptr<TcConvDesc> d(new TcConvDesc());  // value-initialised: every parameter and map starts zero
  TcParams& P = d->P;
  P.B = B; P.H = Hin; P.W = Win; P.Cin = Cin; P.Cout = Cout;
  P.ntaps = ntaps; P.kchunks = (Cin + kc - 1) / kc;
  P.nphases = nphases;
  P.Hout = Hout; P.Wout = Wout; P.os = nphases == 4 ? 2 : 1;
  P.out_pitch = out_pitch; P.res_pitch = ep.res_pitch;
  if constexpr (f32) {
    P.out_f32 = out; P.res_f32 = (const float*)ep.res;
    P.lo_plane_off = planes;
  } else {
    P.out = out; P.res = (const bf16*)ep.res;
  }
  P.bias = ep.bias; P.mult_vec = ep.mult_vec; P.ss = ep.ss; P.t_ptr = ep.t_ptr; P.ss_S = ep.ss_S; P.ss_off = ep.ss_off;
  P.ss_img_stride = ep.ss_img_stride; P.silu = ep.silu;
  for (int i = 0; i < ntaps; ++i) P.taps[i] = taps[i];
  P.qsm = (flags & TC_FLAG_QSOFTMAX) ? 1 : 0;
  P.w_per_image = (flags & TC_FLAG_W_PER_IMAGE) ? 1 : 0;
  int BN = Cout > 64 ? 128 : (Cout > 32 ? 64 : 32);
  // bf16 only: BN = 256, except where Cout is a multiple of 128 but not of 256 (to_qkv, 384: no half-empty N tile)
  if (!f32 && Cout >= 256 && !(Cout % 256 != 0 && Cout % 128 == 0)) BN = 256;
  bool rows = false;  // bf16 only
  if (!f32 && nphases == 1 && planes == 1 && ntaps == 9 && BN <= 128) {
    rows = true;
    for (int i = 0; rows && i < 9; ++i) rows = taps[i].dh == i / 3 - 1 && taps[i].dw == i % 3 - 1 && taps[i].plane == 0;
  }
  d->mode = f32 ? 3 : rows ? 2 : 0;
  // tile shape: BW x BH = 128 pixels, minimise padded work
  long long best = -1;
  for (int bw = 128; bw >= 8; bw >>= 1) {
    int bh = 128 / bw;
    long long cost = (long long)((Win + bw - 1) / bw) * bw * ((Hin + bh - 1) / bh) * bh;
    if (best < 0 || cost < best) { best = cost; P.BW = bw; P.BH = bh; }
  }
  if (rows) {  // (BH+2) x BW box must fit the 20 KB slot: BW <= 16
    if (Win >= 16) { P.BW = 16; P.BH = 8; } else { P.BW = 8; P.BH = 16; }
    P.rows_a_bytes = (P.BH + 2) * P.BW * 128;
  }
  P.logBW = 0;
  while ((1 << P.logBW) < P.BW) P.logBW++;
  P.tilesW = (Win + P.BW - 1) / P.BW;
  P.tilesH = (Hin + P.BH - 1) / P.BH;
  // Small problems (NAFNet's 16x16 levels, sharded deep UNet levels): fewer tiles than half the SMs means a handful
  // of CTAs stream all the weights; narrower N tiles spread that over more SMs.  Tap mode 0 accumulates in the same
  // K order for every BN, so results do not depend on this choice (and hence not on the batch size).  bf16 keeps BN for
  // ROWS, the q-softmax and the NCHW output, and goes no lower than 64; fp32x3 always halves, down to 32.
  if (f32 || (!rows && !P.qsm && !nchw_out)) {
    const int tm = P.tilesW * P.tilesH * B * nphases, bn_min = f32 ? 32 : 64;
    while (BN > bn_min && Cout % (BN / 2) == 0 && (long long)tm * ((Cout + BN - 1) / BN) < g_num_sms / 2) BN >>= 1;
  }
  d->BN = BN;
  d->grid = dim3((unsigned)(P.tilesW * P.tilesH * B * nphases), (unsigned)((Cout + BN - 1) / BN));
  d->tiles_m = P.tilesW * P.tilesH * B * nphases;
  d->num_tiles = d->tiles_m * ((Cout + BN - 1) / BN);
  // Tile order.  Default: M fastest - the CTAs of a wave share one N tile, i.e. one set of weight tiles (3x3 layers: the
  // weights of an N tile are MBs, the A tensor of the deep levels fits in L2).  1x1 convs with several N tiles (to_qkv:
  // 384 outputs = 3 tiles) invert that: their weights are a few KB but the A tensor of the 256^2 / 128^2 levels is larger
  // than L2, and M-fastest re-read it from DRAM once per N tile (about 3x the input's bytes for to_qkv).  N fastest
  // makes the N tiles of one pixel tile run back to back in the same wave, so the second and third read hit L2.
  P.tiles_n = (Cout + BN - 1) / BN;
  // (bf16 only, and only where the input is too large to stay in L2 anyway; small inputs keep M-fastest and its
  // once-per-N-tile epilogue table)
  const long long a_bytes = (long long)B * Hin * Win * in_pitch * es;
  P.n_fast = (!f32 && ntaps == 1 && P.tiles_n > 1 && !P.w_per_image && a_bytes > (24ll << 20)) ? 1 : 0;
  // A: [planes][B][H][W][C] (C contiguous, pixel pitch in_pitch); fp32x3: 2 x planes dense planes, hi then lo
  {
    cuuint64_t dims[5] = {(cuuint64_t)Cin, (cuuint64_t)Win, (cuuint64_t)Hin, (cuuint64_t)B, (cuuint64_t)(f32 ? 2 * planes : planes)};
    cuuint64_t strides[4] = {(cuuint64_t)in_pitch * es, (cuuint64_t)Win * in_pitch * es, (cuuint64_t)Hin * Win * in_pitch * es,
                             (cuuint64_t)B * Hin * Win * in_pitch * es};
    if (planes < 0) {  // the stem's overlapping 8-pixel rows (see above)
      dims[2] = (cuuint64_t)(Hin + 6); dims[4] = 1;
      strides[0] = 16; strides[1] = (cuuint64_t)(Win + 8) * 16; strides[2] = (cuuint64_t)(Hin + 6) * (Win + 8) * 16;
      strides[3] = strides[2] * B;
    }
    const cuuint32_t box[5] = {(cuuint32_t)kc, (cuuint32_t)P.BW, (cuuint32_t)(rows ? P.BH + 2 : P.BH), 1, 1};
    if (!tc_encode(&d->map_a, dtype, 5, in, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   "A", err))
      return nullptr;
  }
  // B: [phase*ntaps][Cout_w][Cin]; bf16 per-image weights: [B][Cout_w][Cin]; fp32x3: [phase*ntaps][2 (hi, lo)][Cout_w][Cin]
  {
    const cuuint64_t dims[3] = {(cuuint64_t)Cin, (cuuint64_t)Cout_w,
                                (cuuint64_t)(P.w_per_image ? B : nphases * ntaps * (f32 ? 2 : 1))};
    const cuuint64_t strides[2] = {(cuuint64_t)Cin * es, (cuuint64_t)Cout_w * Cin * es};
    const cuuint32_t box[3] = {(cuuint32_t)kc, (cuuint32_t)BN, 1};
    if (!tc_encode(&d->map_b, dtype, 3, w, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   "B", err))
      return nullptr;
  }
  // bf16 only: maps of the epilogue's store tiles (16 pixel rows of the tile = one box of 32 channels, 64B swizzle): the
  // TMA stores into the destination and the TMA loads of the residual.  [B][H][W][C] view of the tensor (channel offset
  // already in the pointer), pixel stride os*pitch; one map per upsample phase (base shifted by (py,px)).
  auto tile_maps = [&](OutMaps& maps, const S* t, int pitch, CUtensorMapL2promotion l2, const char* what) -> bool {
    const int bw = P.BW < 16 ? P.BW : 16, bh = 16 / bw;
    for (int ph = 0; ph < nphases; ++ph) {
      const int py = ph >> 1, px = ph & 1;
      const cuuint64_t dims[4] = {(cuuint64_t)Cout, (cuuint64_t)Win, (cuuint64_t)Hin, (cuuint64_t)B};
      const cuuint64_t strides[3] = {(cuuint64_t)P.os * pitch * es, (cuuint64_t)P.os * Wout * pitch * es,
                                     (cuuint64_t)Hout * Wout * pitch * es};
      const cuuint32_t box[4] = {32, (cuuint32_t)bw, (cuuint32_t)bh, 1};
      if (!tc_encode(&maps.m[ph], dtype, 4, t + ((long long)py * Wout + px) * pitch, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B,
                     l2, what, err))
        return false;
    }
    return true;
  };
  if (!f32 && !nchw_out) {
    if (!tile_maps(d->map_o, out, out_pitch, CU_TENSOR_MAP_L2_PROMOTION_NONE, "out")) return nullptr;
    if (ep.res && !tile_maps(d->map_r, (const S*)ep.res, ep.res_pitch, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "residual"))
      return nullptr;
  }
  tc_fill_magic(d.get());
  if (!tc_pick(d.get())) return bad("no conv_tc_persist_kernel instantiation for this BN and mode");
  return d.release();
}
template TcConvDesc* tc_conv_create(const bf16*, int, int, int, int, int, int, const bf16*, int, int, const TcTap*, int,
                                    const Epilogue&, bf16*, int, int, int, std::string*, int);
template TcConvDesc* tc_conv_create(const float*, int, int, int, int, int, int, const float*, int, int, const TcTap*, int,
                                    const Epilogue&, float*, int, int, int, std::string*, int);

void tc_conv_destroy(TcConvDesc* d) { delete d; }

void tc_conv_set_out_nchw(TcConvDesc* d, float* out, int cropH, int cropW) {
  d->P.out_nchw = out;
  d->P.cropH = cropH;
  d->P.cropW = cropW;
}

void tc_conv_set_runtime(TcConvDesc* d, const float* ss, const int* t_ptr, int ss_img_stride) {
  d->P.ss = ss;
  d->P.t_ptr = t_ptr;
  d->P.ss_img_stride = ss_img_stride;
}

void tc_conv_query(const TcConvDesc* d, int info[4]) {
  info[0] = d->BN;
  info[1] = d->mode;
  info[2] = tc_pick(d)->ekt;
  info[3] = d->num_tiles;
}

int tc_conv_launch(TcConvDesc* d, cudaStream_t st) {
  const TcKernel& k = *tc_pick(d);
  const unsigned g = (unsigned)(d->num_tiles < g_num_sms ? d->num_tiles : g_num_sms);
  static unsigned long long* dbg_dev = nullptr;
  const char* dbg_env = getenv("IRSDE_TC_DEBUG");
  const bool dbg = dbg_env && dbg_env[0] == '1';
  if (dbg) {
    if (!dbg_dev) cudaMalloc(&dbg_dev, 256 * TC_DBG_SLOTS * sizeof(unsigned long long));
    cudaMemsetAsync(dbg_dev, 0, 256 * TC_DBG_SLOTS * sizeof(unsigned long long), st);
  }
  d->P.dbg = dbg ? dbg_dev : nullptr;
  d->P.epi_kind = k.ekt;
  const auto kernel = k.fn;
  pdl_launch(kernel, g, TC_THREADS, k.smem, st, d->map_a, d->map_b, d->map_o, d->map_r, d->P, d->tiles_m, d->num_tiles);
  if (dbg) {
    // per CTA: [0] producer cycles waiting on empty barriers, [1] producer cycles; per consumer warpgroup w: [2+w] cycles
    // waiting on full barriers, [4+w] in the epilogue, [6+w] waiting for its ping-pong turn, [8+w] in all, [10+w] tiles
    unsigned long long h[256 * TC_DBG_SLOTS];
    cudaStreamSynchronize(st);
    cudaMemcpy(h, dbg_dev, sizeof h, cudaMemcpyDeviceToHost);
    double a[TC_DBG_SLOTS] = {0};
    for (unsigned i = 0; i < g; ++i) for (int j = 0; j < TC_DBG_SLOTS; ++j) a[j] += (double)h[i * TC_DBG_SLOTS + j] / g;
    fprintf(stderr,
            "TCDBG BN=%d mode=%d ekt=%d grid=%u tiles=%d ntaps=%d kch=%d | prod wait %.0f / %.0f | wg0 full %.0f epi %.0f turn %.0f"
            " / %.0f (tiles/cta %.1f) | wg1 full %.0f epi %.0f turn %.0f / %.0f (tiles/cta %.1f)\n",
            d->BN, d->mode, k.ekt, g, d->num_tiles, d->P.ntaps, d->P.kchunks, a[0], a[1], a[2], a[4], a[6], a[8], a[10], a[3], a[5],
            a[7], a[9], a[11]);
  }
  return 1;
}

}  // namespace irsde
