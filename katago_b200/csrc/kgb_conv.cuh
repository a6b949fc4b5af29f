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
// Data layout ("padded rows"): activations are 2-D row-major [M rows][C_p channels], C_p a multiple of 64, where every image
// owns (h+pad)*(w+pad) rows for its board box w x h: `pad` zero rows on top and `pad` zero columns at the right of each board
// row (pad = largest conv radius of the net), pitch w+pad.  A (dy,dx) filter tap is then the same matrix shifted by
// dy*(w+pad)+dx rows, and the zero padding of the convolution is physically present (or supplied by TMA out-of-bounds fill at
// the two ends).  Images of one width are laid out back to back in segments of whole 128-row tiles (RowPlan, kgb_kernels.cuh),
// so each tile has one pitch; points of the box that are off the board are handled by the same mask that zeroes the pad rows.
// The frame layout is the case where every box is the full X x Y frame: image i at row i*(Y+pad)*(X+pad).
struct ConvParams {
  int M;            // rows the buffers hold (at least the plan's rows)
  int Wp;           // X + pad, the frame's pitch: the A halo box is sized for it, the widest pitch a tile can have
  const int* tile_wp;     // [num_m_tiles] row pitch of each 128-row tile
  const int* row_img;     // [M] image of each board row, read for ncbias (other rows are masked: -1 or any image)
  const int* m_tiles;     // the number of 128-row tiles the plan uses (device), at most num_m_tiles
  int ky, kx;       // filter size
  int cin_p;        // padded input channels (multiple of 64)
  int cout_p;       // padded output channels (multiple of 64)
  int n_tile;       // wgmma N (cout_p / num_n_tiles), multiple of 32, <= 256
  int num_m_tiles, num_n_tiles;   // num_m_tiles: the most tiles a plan can use (sizes the persistent grid)
  int split;        // 0: fp16 operands; 1: 3-term split-fp16 ("fp32-equivalent") - A and W carry [hi | lo] halves
  // epilogue
  const void* residual;   // [M][cout_p] or null
  int residual_fp32;
  const float* ncbias;    // [batch][cout_p] or null, by row_img
  void* raw_out;          // [M][cout_p] or null
  int raw_fp32;
  __half* act_out;        // [M][cout_p * (split ? 2 : 1)] or null
  const float* bn_scale;  // [cout_p] (zero in padded channels)
  const float* bn_bias;   // [cout_p]
  int act;                // kgb::Activation
  const float* mask;      // [M] 1.0 on-board, 0.0 pad/off-board
  // chaining (launchConvWG / launchConvPair)
  int* tile_flags;        // [num_m_tiles] this launch's tile flags, zero before the launch when a chained launch reads them
  const int* pred_flags;  // the previous launch's tile_flags when this launch is chained to it, else null
  int pred_parts;         // the value a tile flag of the previous launch has once the tile is written (convChainParts)
  int epi_wg;             // launchConvWG may take the epilogue-warpgroup kernel (convEpilogueWG); 0 keeps kgb_conv_wg_kernel
  int pair_epi_wg;        // launchConvPair may take the exit-epilogue-warpgroup kernel (convPairEpilogueWG); 0 keeps kgb_conv_pair_kernel
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

// Tensor maps of one launch.  A: [M][cin_p (* 2)] fp16, box {64, convABoxRows}; B: packed weights, box {64, n_tile}; both 128B
// swizzle.  residual, raw, act: box {32, 64} (convSliceBoxRows), 128B swizzle when fp32 and 64B when fp16.  residual = the
// residual [M][cout_p] (read only when p.residual is set), raw = raw_out [M][cout_p] and act = act_out [M][cout_p * (split ? 2 : 1)]
// (written only when set).
struct ConvTmaps {
  CUtensorMap A, B, residual, raw, act;
};

// Launcher (defined in kgb_conv_wg.cu).  A persistent grid of at most one CTA per SM walks the output tiles; the epilogue stages
// its outputs in shared memory and writes them with TMA stores.  When both the residual and raw_out are set they must have the
// same dtype: the raw output is written back over the residual slice in shared memory.  The residual may alias raw_out (each
// element is read and written by the CTA of its own tile); A must alias neither raw_out nor act_out, since a tile's halo rows
// belong to the neighbouring tiles.
//
// Chaining.  Every launch adds 1 to p.tile_flags[m] per (n-group, consumer warpgroup) once that part's TMA stores of 128-row tile m
// are complete (2 per n-group at once from the epilogue warpgroup of kgb_conv_wg_epi_kernel), so a tile is written when its flag
// reaches convChainParts(p) if the flags were zero before the launch.  With
// p.pred_flags set, the launch is a programmatic dependent launch of the previous kernel on the stream, which must be a
// convolution launch whose tile_flags these are, with pred_parts = convChainParts of it.  Its CTAs may then start while that
// kernel's last tiles still run: before a tile loads its operand rows or its residual it waits until the previous launch's tiles
// m-1, m and m+1 are written.  A CTA does not exit before the previous launch has completed, so a launch that follows a chained
// one in the ordinary way still sees every launch of the chain complete.  Data written inside a chain is read through TMA only.
// A flag wait that lasts longer than ~4 s gives up and sets the sticky word that convChainStatus reports.  The word is one for the
// process (mapped host memory, shared by every device and handle) and is never reset: after one wait has given up, the outputs of
// that forward are wrong and every later synchronising call of every handle reports the error.
cudaError_t launchConvWG(const ConvTmaps& tm, const ConvParams& p, cudaStream_t stream);
// Whether launchConvWG runs these parameters with kgb_conv_wg_epi_kernel (a dedicated epilogue warpgroup fed through a shared-memory
// accumulator tile, so the MMAs of the next tile run under each tile's epilogue) rather than kgb_conv_wg_kernel: p.epi_wg set, fp16
// operands, a filter wider than 1x1, n_tile 96 to 192, an fp16 stream or none (or only a raw fp32 output), and rings that fit.
// Both kernels give the same bits.
bool convEpilogueWG(const ConvParams& p);
inline int convChainParts(const ConvParams& p) { return 2 * p.num_n_tiles; }
cudaError_t convChainStatus();  // cudaErrorLaunchTimeout once a flag wait of this process has given up
inline int convABoxRows(int ky, int kx, int Wp) { return 128 + 2 * ((ky / 2) * Wp + (kx / 2)); }  // TMA box rows of the A halo tile
inline int convSliceBoxRows() { return 64; }  // TMA box rows of the epilogue's slices: one consumer warpgroup's half of a tile
cudaError_t convWGInit();  // per device, before the first launch (sets the kernels' shared-memory limit, reads the SM count)

// A block boundary in one launch: p1 = a nested block's exit 1x1 (inner -> trunk channels, + residual, raw stream written in
// place, p1.act_out unused), p2 = the next nested block's entry 1x1 (trunk -> inner channels, raw stream + activated operand).  The
// activated trunk operand that p1 would write and p2 would read stays in shared memory, 64 columns at a time, each chunk an entry
// k-block.  Every output element is summed in the same order and goes through the same epilogue as with two launchConvWG calls,
// so the results are bit-identical.  p2.act_out may be the same buffer as p1's A (a tile reads all of its rows of A before its
// epilogue writes them, and there is no halo).  Tensor maps: A = p1's operand, box {64, 128}; W1 = the exit's packed weights, box
// {64, 64}; W2 = the entry's, box {64, p2.n_tile}; stream1 = p1's residual and raw stream, stream2 = p2.raw_out, act2 = p2.act_out
// (slice boxes as in ConvTmaps).  Chaining as launchConvWG, with p1's chain fields; a tile is written (all of p1's and p2's outputs)
// when its flag reaches convPairChainParts.
// When convPairEpilogueWG(p1, p2), the exit is made in chunks of kConvPairEpiChunk columns instead: W1 has box {64,
// kConvPairEpiChunk}, and W2 box {kConvPairEpiChunk, p2.n_tile} with the 64B swizzle (makeTmapK32 in kgb_api.cu).
struct ConvPairTmaps {
  CUtensorMap A, W1, W2, stream1, stream2, act2;
};
static constexpr int kConvPairChunk = 64;      // box rows of W1
static constexpr int kConvPairEpiChunk = 32;   // box rows of W1 and box columns of W2 for kgb_conv_pair_epi_kernel
static constexpr int kConvPairParts = 2;       // one per consumer warpgroup
// Whether launchConvPair takes these launches: fp16 operands, mish at both ends, 1x1 filters, (inner, trunk) widths the kernel is
// compiled for, and rings that fit in shared memory.
bool convPairSupported(const ConvParams& p1, const ConvParams& p2);
// Whether launchConvPair runs them with kgb_conv_pair_epi_kernel (the exit's epilogue in a warpgroup of its own, fed through
// shared-memory accumulator slots) rather than kgb_conv_pair_kernel: p1.pair_epi_wg set, fp16 streams, (inner, trunk) = (192, 384).
// Both kernels give the same bits.
bool convPairEpilogueWG(const ConvParams& p1, const ConvParams& p2);
// The value a tile flag of the launch reaches once the tile is written: kConvPairParts, or 3 with the exit-epilogue warpgroup
// (each MMA warpgroup publishes its half of the entry's outputs, the epilogue warpgroup the exit's).
int convPairChainParts(const ConvParams& p1, const ConvParams& p2);
cudaError_t launchConvPair(const ConvPairTmaps& tm, const ConvParams& p1, const ConvParams& p2, cudaStream_t stream);

}  // namespace kgb
