// fp32 SIMT implicit-GEMM convolution over NHWC activations (parity mode, and the few layers the
// tensor-core engine does not take: Cin=6 stem, Cout=3 head).  One generic kernel:
//   any KHxKW, stride, zero pad, optional nearest x2 upsample folded into the gather
//   (module_util.py:93-97: src = dst >> 1), epilogue = bias -> (scale+1)*x+shift -> SiLU -> +res
//   (module_util.py:114-122,136-146), output NHWC (channel-offset view) or cropped fp32 NCHW
//   (DenoisingUNet_arch.py:132).
// Tile 64 pixels x 64 channels x 16 k, 256 threads, 4x4 outputs / thread, register prefetch.
#include "common.cuh"

namespace irsde {

namespace {
constexpr int BM = 64, BN = 64, BK = 16;

template <typename T>
struct Vec4 {};
template <>
struct Vec4<float> {
  static __device__ __forceinline__ void load(const float* p, float v[4]) {
    float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
  static __device__ __forceinline__ void store(float* p, const float v[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
};
template <>
struct Vec4<bf16> {
  static __device__ __forceinline__ void load(const bf16* p, float v[4]) {
    uint2 t = *reinterpret_cast<const uint2*>(p);
    __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&t.x), b = *reinterpret_cast<__nv_bfloat162*>(&t.y);
    v[0] = __low2float(a); v[1] = __high2float(a); v[2] = __low2float(b); v[3] = __high2float(b);
  }
  static __device__ __forceinline__ void store(bf16* p, const float v[4]) {
    __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], v[3]);
    uint2 t;
    t.x = *reinterpret_cast<uint32_t*>(&a);
    t.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(p) = t;
  }
};

template <typename T>
__global__ void __launch_bounds__(256) conv_simt_kernel(ConvGeom g, const T* __restrict__ in, int in_pitch,
                                                        const float* __restrict__ w, Epilogue ep, T* __restrict__ out,
                                                        int out_pitch, float* __restrict__ out_nchw, int cropH,
                                                        int cropW, int vecA, int vecB, int vecO) {
  PDL_ENTRY();
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN];
  const int tid = threadIdx.x;
  const long long M = (long long)g.B * g.Hout * g.Wout;
  const int Ktot = g.KH * g.KW * g.Cin;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // --- A loader coordinates: this thread always loads pixel a_row, k offsets a_k..a_k+3
  const int a_row = tid >> 2, a_k = (tid & 3) * 4;
  long long am = m0 + a_row;
  bool a_valid = am < M;
  int ab = 0, aho = 0, awo = 0;
  if (a_valid) {
    awo = am % g.Wout;
    aho = (am / g.Wout) % g.Hout;
    ab = am / ((long long)g.Wout * g.Hout);
  }
  const int Hup = g.Hin * g.up, Wup = g.Win * g.up;
  const int b_k = tid >> 4, b_n = (tid & 15) * 4;

  float ra[4], rb[4];
  auto load_tile = [&](int k0) {
    // A
    int k = k0 + a_k;
#pragma unroll
    for (int j = 0; j < 4; ++j) ra[j] = 0.f;
    if (a_valid && k < Ktot) {
      if (vecA) {  // Cin % 4 == 0: the 4 k's share one tap and are contiguous
        int tap = k / g.Cin, c = k - tap * g.Cin;
        int r = tap / g.KW, s = tap - r * g.KW;
        int hi = aho * g.stride - g.pad + r, wi = awo * g.stride - g.pad + s;
        if (hi >= 0 && hi < Hup && wi >= 0 && wi < Wup) {
          if (g.up == 2) { hi >>= 1; wi >>= 1; }
          Vec4<T>::load(in + (((long long)ab * g.Hin + hi) * g.Win + wi) * in_pitch + c, ra);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          int kk = k + j;
          if (kk < Ktot) {
            int tap = kk / g.Cin, c = kk - tap * g.Cin;
            int r = tap / g.KW, s = tap - r * g.KW;
            int hi = aho * g.stride - g.pad + r, wi = awo * g.stride - g.pad + s;
            if (hi >= 0 && hi < Hup && wi >= 0 && wi < Wup) {
              if (g.up == 2) { hi >>= 1; wi >>= 1; }
              ra[j] = to_f(in[(((long long)ab * g.Hin + hi) * g.Win + wi) * in_pitch + c]);
            }
          }
        }
      }
    }
    // B
    int kb = k0 + b_k;
#pragma unroll
    for (int j = 0; j < 4; ++j) rb[j] = 0.f;
    if (kb < Ktot) {
      const float* wr = w + (long long)kb * g.Cout + n0 + b_n;
      if (vecB && n0 + b_n + 3 < g.Cout) {
        float4 t = *reinterpret_cast<const float4*>(wr);
        rb[0] = t.x; rb[1] = t.y; rb[2] = t.z; rb[3] = t.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (n0 + b_n + j < g.Cout) rb[j] = wr[j];
      }
    }
  };

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int ty = tid >> 4, tx = tid & 15;
  const int nkt = (Ktot + BK - 1) / BK;
  load_tile(0);
  for (int kt = 0; kt < nkt; ++kt) {
#pragma unroll
    for (int j = 0; j < 4; ++j) As[a_k + j][a_row] = ra[j];
    *reinterpret_cast<float4*>(&Bs[b_k][b_n]) = make_float4(rb[0], rb[1], rb[2], rb[3]);
    __syncthreads();
    if (kt + 1 < nkt) load_tile((kt + 1) * BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }

  // --- epilogue
  const int trow = ep.t_ptr ? *ep.t_ptr : 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    long long m = m0 + ty * 4 + i;
    if (m >= M) continue;
    int wo = m % g.Wout;
    int ho = (m / g.Wout) % g.Hout;
    int b = m / ((long long)g.Wout * g.Hout);
    int nbase = n0 + tx * 4;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int n = nbase + j;
      float x = acc[i][j];
      if (n < g.Cout) {
        if (ep.bias) x += ep.bias[n];
        if (ep.ss) {
          const float* row = ep.ss + (long long)(trow + b * ep.ss_img_stride) * ep.ss_S + ep.ss_off;
          x = x * (row[n] + 1.0f) + row[g.Cout + n];
        }
        if (ep.mult_vec) x *= ep.mult_vec[n];
        if (ep.silu) x = silu_f(x);
      }
      v[j] = x;
    }
    if (out_nchw) {
      if (ho < cropH && wo < cropW) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (nbase + j < g.Cout)
            out_nchw[(((long long)b * g.Cout + nbase + j) * cropH + ho) * cropW + wo] = v[j];
      }
    } else {
      if (ep.res) {
        const T* rr = reinterpret_cast<const T*>(ep.res) + m * ep.res_pitch + nbase;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (nbase + j < g.Cout) v[j] += to_f(rr[j]);
      }
      T* o = out + m * out_pitch + nbase;
      if (vecO && nbase + 3 < g.Cout) {
        Vec4<T>::store(o, v);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (nbase + j < g.Cout) o[j] = from_f<T>(v[j]);
      }
    }
  }
}
}  // namespace

template <typename T>
void conv_simt_path(const ConvGeom& g, const T* in, int in_pitch, const float* w, const T* out, int out_pitch, int32_t path[4]) {
  const long long M = (long long)g.B * g.Hout * g.Wout;
  const int vw = 4 * sizeof(T);  // bytes of a 4-element vector
  path[0] = (g.Cin % 4 == 0) && (in_pitch % 4 == 0) && (((uintptr_t)in) % vw == 0);
  path[1] = (g.Cout % 4 == 0) && (((uintptr_t)w) % 16 == 0);
  path[2] = out && (out_pitch % 4 == 0) && (((uintptr_t)out) % vw == 0);
  path[3] = (int32_t)((M + BM - 1) / BM * ((g.Cout + BN - 1) / BN));
}

template <typename T>
void launch_conv_simt(const ConvGeom& g, const T* in, int in_pitch, const float* w, const Epilogue& ep, T* out,
                      int out_pitch, float* out_nchw, int cropH, int cropW, cudaStream_t st) {
  long long M = (long long)g.B * g.Hout * g.Wout;
  dim3 grid((unsigned)((M + BM - 1) / BM), (unsigned)((g.Cout + BN - 1) / BN));
  int32_t path[4];
  conv_simt_path<T>(g, in, in_pitch, w, out, out_pitch, path);
  pdl_launch(conv_simt_kernel<T>, grid, 256, 0, st, g, in, in_pitch, w, ep, out, out_pitch, out_nchw, cropH, cropW, (int)path[0],
             (int)path[1], (int)path[2]);
}
template void conv_simt_path<float>(const ConvGeom&, const float*, int, const float*, const float*, int, int32_t*);
template void conv_simt_path<bf16>(const ConvGeom&, const bf16*, int, const float*, const bf16*, int, int32_t*);
template void launch_conv_simt<float>(const ConvGeom&, const float*, int, const float*, const Epilogue&, float*, int,
                                      float*, int, int, cudaStream_t);
template void launch_conv_simt<bf16>(const ConvGeom&, const bf16*, int, const float*, const Epilogue&, bf16*, int,
                                     float*, int, int, cudaStream_t);

}  // namespace irsde
