// Shared declarations for the convolution kernels (wgmma implicit GEMM + SIMT debug path).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace kgb {

// One fused convolution launch:  out = conv(A, W) [+ ncbias[n]] [+ residual];  raw_out = out;
// act_out = mask * act(out * bn_scale + bn_bias)  (the NEXT layer's BN+activation, applied by the producer so that
// the consumer's A operand can go TMA -> smem -> wgmma untouched).
//
// Replaces, per reference call site, the sequence
//   applyCScaleBias*Kernel (cudahelpers.cu:1370-2101) -> cudnnConvolutionForward / cublas*gemm
//   (cudabackend.cpp:788-841) [beta=1 residual accumulate]  [-> addNCBiasInplace* (cudahelpers.cu:1250-1364)]
// i.e. NormActConv::apply / ConvLayer::apply of the Eigen path (eigenbackend.cpp:448-701, 1065-1077).
//
// Data layout ("padded rows"): activations are 2-D row-major [M = n*P rows][C_p channels], C_p a multiple of 64,
// where every image owns P = (Y+pad)*(X+pad) rows: `pad` zero rows on top and `pad` zero columns at the right of each
// board row (pad = largest conv radius of the net).  A (dy,dx) filter tap is then the same matrix shifted by
// dy*(X+pad)+dx rows, the zero padding of the convolution is physically present (or supplied by TMA out-of-bounds
// fill at the two ends), and boards smaller than (X,Y) are handled by the same mask that zeroes the pad rows.
struct ConvParams {
  int M;            // valid rows (= batch * P)
  int P;            // rows per image
  int Wp;           // X + pad (row pitch of the board inside an image)
  int ky, kx;       // filter size
  int cin_p;        // padded input channels (multiple of 64)
  int cout_p;       // padded output channels (multiple of 64)
  int n_tile;       // wgmma N (cout_p / num_n_tiles), multiple of 32, <= 256
  int num_m_tiles, num_n_tiles;
  int split;        // 0: fp16 operands; 1: 3-term split-fp16 ("fp32-equivalent") - A and W carry [hi | lo] halves
  // epilogue
  const void* residual;   // [M][cout_p] or null
  int residual_fp32;
  const float* ncbias;    // [batch][cout_p] or null
  void* raw_out;          // [M][cout_p] or null
  int raw_fp32;
  __half* act_out;        // [M][cout_p * (split ? 2 : 1)] or null
  const float* bn_scale;  // [cout_p] (zero in padded channels)
  const float* bn_bias;   // [cout_p]
  int act;                // kgb::Activation
  const float* mask;      // [M] 1.0 on-board, 0.0 pad/off-board
};

// fp32 activation functions shared by every epilogue (reference: eigenbackend.cpp:780-809, cudahelpers.cu mish/silu).
// mish(x) = x * tanh(softplus(x)) = x * n / (n + 2),  n = e^x (e^x + 2)   (exact identity; x clamped at 20 like the
// reference so that e^2x cannot overflow).
__device__ __forceinline__ float kgb_ex2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float kgb_rcp(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float kgb_activate(float x, int act) {
  if(act == 1) return fmaxf(x, 0.0f);
  if(act == 2) {
    float e = kgb_ex2(fminf(x, 20.0f) * 1.4426950408889634f);
    float n = fmaf(e, e, e + e);
    return x * (n * kgb_rcp(n + 2.0f));
  }
  if(act == 3) return x * kgb_rcp(1.0f + kgb_ex2(x * -1.4426950408889634f));
  return x;
}

// ------------------------------------------------------------------------------------------------------------
// Epilogue for one 16-column chunk of one accumulator row
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void epilogue_chunk(const ConvParams& p, const uint32_t (&acc)[16], int row, int col, float maskv, int img,
                                               const float* sc, const float* bi) {
  float v[16];
#pragma unroll
  for(int j = 0; j < 16; j++) v[j] = __uint_as_float(acc[j]);
  if(p.ncbias != nullptr) {
    const float4* b = reinterpret_cast<const float4*>(p.ncbias + (size_t)img * p.cout_p + col);
#pragma unroll
    for(int q = 0; q < 4; q++) {
      float4 t = __ldg(b + q);
      v[4 * q] += t.x; v[4 * q + 1] += t.y; v[4 * q + 2] += t.z; v[4 * q + 3] += t.w;
    }
  }
  size_t off = (size_t)row * p.cout_p + col;
  if(p.residual != nullptr) {
    if(p.residual_fp32) {
      const float4* r = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.residual) + off);
#pragma unroll
      for(int q = 0; q < 4; q++) {
        float4 t = r[q];
        v[4 * q] += t.x; v[4 * q + 1] += t.y; v[4 * q + 2] += t.z; v[4 * q + 3] += t.w;
      }
    }
    else {
      const uint4* r = reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(p.residual) + off);
#pragma unroll
      for(int q = 0; q < 2; q++) {
        uint4 t = r[q];
        const __half2* h = reinterpret_cast<const __half2*>(&t);
#pragma unroll
        for(int e = 0; e < 4; e++) {
          float2 f = __half22float2(h[e]);
          v[8 * q + 2 * e] += f.x; v[8 * q + 2 * e + 1] += f.y;
        }
      }
    }
  }
  if(p.raw_out != nullptr) {
    if(p.raw_fp32) {
      float4* o = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.raw_out) + off);
#pragma unroll
      for(int q = 0; q < 4; q++) o[q] = make_float4(v[4 * q] * maskv, v[4 * q + 1] * maskv, v[4 * q + 2] * maskv, v[4 * q + 3] * maskv);
    }
    else {
      uint4* o = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(p.raw_out) + off);
#pragma unroll
      for(int q = 0; q < 2; q++) {
        uint4 t;
        __half2* h = reinterpret_cast<__half2*>(&t);
#pragma unroll
        for(int e = 0; e < 4; e++) h[e] = __floats2half2_rn(v[8 * q + 2 * e] * maskv, v[8 * q + 2 * e + 1] * maskv);
        o[q] = t;
      }
    }
  }
  if(p.act_out != nullptr) {
    float a[16];
    const float4* s4 = reinterpret_cast<const float4*>(sc);
    const float4* b4 = reinterpret_cast<const float4*>(bi);
#pragma unroll
    for(int q = 0; q < 4; q++) {
      float4 s = s4[q], b = b4[q];
      a[4 * q] = kgb_activate(fmaf(v[4 * q], s.x, b.x), p.act) * maskv;
      a[4 * q + 1] = kgb_activate(fmaf(v[4 * q + 1], s.y, b.y), p.act) * maskv;
      a[4 * q + 2] = kgb_activate(fmaf(v[4 * q + 2], s.z, b.z), p.act) * maskv;
      a[4 * q + 3] = kgb_activate(fmaf(v[4 * q + 3], s.w, b.w), p.act) * maskv;
    }
    if(maskv == 0.0f) {
#pragma unroll
      for(int j = 0; j < 16; j++) a[j] = 0.0f;  // guards NaN/inf garbage at pad rows
    }
    int ldo = p.split ? 2 * p.cout_p : p.cout_p;
    __half* dst = p.act_out + (size_t)row * ldo + col;
    uint4 hi[2], lo[2];
    __half2* hh = reinterpret_cast<__half2*>(hi);
    __half2* hl = reinterpret_cast<__half2*>(lo);
#pragma unroll
    for(int e = 0; e < 8; e++) {
      __half2 h = __floats2half2_rn(a[2 * e], a[2 * e + 1]);
      hh[e] = h;
      if(p.split) {
        float2 hf = __half22float2(h);
        hl[e] = __floats2half2_rn(a[2 * e] - hf.x, a[2 * e + 1] - hf.y);
      }
    }
    reinterpret_cast<uint4*>(dst)[0] = hi[0];
    reinterpret_cast<uint4*>(dst)[1] = hi[1];
    if(p.split) {
      reinterpret_cast<uint4*>(dst + p.cout_p)[0] = lo[0];
      reinterpret_cast<uint4*>(dst + p.cout_p)[1] = lo[1];
    }
  }
}

// Launchers (defined in kgb_conv_wg.cu / kgb_kernels.cu)
// tmapA: [M][cin_p (* 2)] fp16, box {64, convABoxRows}; tmapB: packed weights, box {64, n_tile}; both 128B swizzle.
// tmapR (read only when p.residual is set): the residual [M][cout_p], box {32, 128}, 128B swizzle when fp32, 64B when fp16.
// The residual may alias raw_out (each element is read and written by the CTA of its own tile); A must alias neither raw_out nor
// act_out, since a tile's halo rows belong to the neighbouring tiles.
cudaError_t launchConvWG(const CUtensorMap& tmapA, const CUtensorMap& tmapB, const CUtensorMap& tmapR, const ConvParams& p,
                         cudaStream_t stream);
cudaError_t launchConvSimt(const __half* A, int lda, const __half* W, const ConvParams& p, cudaStream_t stream);
inline int convABoxRows(int ky, int kx, int Wp) { return 128 + 2 * ((ky / 2) * Wp + (kx / 2)); }  // TMA box rows of the A halo tile
cudaError_t convWGInit();  // per device, before the first launch

}  // namespace kgb
