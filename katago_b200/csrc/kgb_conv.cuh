// Shared declarations for the wgmma implicit-GEMM convolution (kgb_conv_wg.cu) and the small kernels around it.
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

// fp32 activation functions of the small kernels, and of the convolution epilogue except its mish, which epilogue_store
// computes in a form of its own (reference: eigenbackend.cpp:780-809, cudahelpers.cu mish/silu).
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

// Launcher (defined in kgb_conv_wg.cu)
// tmapA: [M][cin_p (* 2)] fp16, box {64, convABoxRows}; tmapB: packed weights, box {64, n_tile}; both 128B swizzle.
// tmapR (read only when p.residual is set): the residual [M][cout_p], box {32, 128}, 128B swizzle when fp32, 64B when fp16.
// The residual may alias raw_out (each element is read and written by the CTA of its own tile); A must alias neither raw_out nor
// act_out, since a tile's halo rows belong to the neighbouring tiles.
cudaError_t launchConvWG(const CUtensorMap& tmapA, const CUtensorMap& tmapB, const CUtensorMap& tmapR, const ConvParams& p,
                         cudaStream_t stream);
inline int convABoxRows(int ky, int kx, int Wp) { return 128 + 2 * ((ky / 2) * Wp + (kx / 2)); }  // TMA box rows of the A halo tile
cudaError_t convWGInit();  // per device, before the first launch

}  // namespace kgb
