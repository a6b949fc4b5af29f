// Small fp32 kernels around the wgmma convolution: input packing, pooling, tiny matmuls, head outputs.
#pragma once
#include <algorithm>

#include "kgb_conv.cuh"

namespace kgb {

// The evaluator's frame: X x Y positions, the inputs' and outputs' index space.  P = (Y+pad)*(X+pad) rows is what one image
// takes when it is laid out at the full frame; row of (y,x) inside such an image = (y+pad)*Wp + x.
struct Layout {
  int X, Y, pad, Wp, P;
};

// The row layout of one forward ("ragged rows", planned on the device by launchPlanRows).  Image i is the bounding box
// (x0, y0, w, h) of its non-zero mask positions, taken after its symmetry, laid out from row base[i] as (h+pad) rows of pitch
// w+pad like a frame of its own.  Images of one box width form a segment, back to back in image order; a segment ends with at
// least pad*(w+pad)+pad zero rows and is rounded up to a multiple of 128 rows, so that every 128-row tile has one pitch and no
// tap of a board row reaches another segment.  Segments follow each other by increasing width.  With `ragged` off every box is
// the full frame: one segment, image i at row i*P, the frame layout.
struct RowPlan {
  int4* box;      // [n] x0, y0, w, h (w = h = 0: the mask is empty, the image has no rows)
  int* base;      // [n] first row of the image (its top pad row); -1 when it has no rows
  int* tileWp;    // [tiles] row pitch of each 128-row tile
  int* rowImg;    // [rows] image of each row that holds a board position (other rows: some image index, or -1; they are masked)
  int* stats;     // [3] rows, 128-row tiles and segments the forward uses
  int ragged;
};

// Rows the row buffers need at batch n: every image at its largest (P rows), and per possible segment (one per box width) the
// gap that ends it and the remainder up to the next 128 rows.
inline size_t planRowCapacity(const Layout& L, int n) {
  const size_t segs = (size_t)std::min(n, L.X);
  return ((size_t)n * L.P + segs * ((size_t)L.pad * L.Wp + L.pad + 127) + 127) / 128 * 128;
}

// Row of frame position (y, x) of an image with box b and first row base, or -1 when the position lies outside the box: a mask-0
// position, which contributes exactly what a mask-0 row of the frame layout contributes.
__device__ __forceinline__ int planRow(int4 b, int base, int pad, int y, int x) {
  const int yy = y - b.y, xx = x - b.x;
  if(yy < 0 || xx < 0 || yy >= b.w || xx >= b.z) return -1;
  return base + (yy + pad) * (b.z + pad) + xx;
}
__device__ __forceinline__ int planRow(const RowPlan& rp, int pad, int img, int y, int x) { return planRow(rp.box[img], rp.base[img], pad, y, x); }

// Plans the rows of a batch from its inputs (the boxes, then the layout), on `s`.  spatial/symmetry as for launchPackInput.
cudaError_t launchPlanRows(const float* spatial, int n, int C, bool nhwc, const int* symmetry, Layout L, const RowPlan& rp, cudaStream_t s);

// Inputs (reference: NeuralNet::getOutput eigenbackend.cpp:2467-2486 + SymmetryHelpers::copyInputsWithSymmetry
// nninputs.cpp:529-590; mask = input channel 0, eigenbackend.cpp:2181; computeMaskSum :124).
// spatial: [n][C][Y][X] (NCHW) or [n][Y][X][C] (NHWC) fp32 as written by NNInputs::fillRowV7.  Positions outside an image's
// box are not written: their features must be zero, as fillRowV7 leaves every point off the board.  act and mask are cleared
// over all M rows first.
cudaError_t launchPackInput(const float* spatial, int n, int C, bool nhwc, const int* symmetry, Layout L, const RowPlan& rp, size_t M,
                            __half* act, int cin_p, int split, float* mask, float* maskSum, cudaStream_t s);

// out[n][co] = act( sum_k in[n][k] * W[k][co] + bias[co] )   (MatMulLayer / MatBiasLayer / ActivationLayer,
// eigenbackend.cpp:811-862); out has leading dimension ldo and is zero-filled in [cout, ldo).  accumulate: out = out + that instead
// (the metadata encoder's output added to the global inputs' bias, eigenbackend.cpp:1927-1932).
cudaError_t launchMatMulNC(const float* in, int ldi, const float* W, const float* bias, int n, int cin, int cout, int act,
                           float* out, int ldo, cudaStream_t s, bool accumulate = false);

// Global pooling of act(BN(raw[:, c0:c0+C])) * mask  ->  pooled [n][3C]
//   valueHead == 0: mean, mean*(sqrt(area)-14)/10, max       (poolRowsGPool, eigenbackend.cpp:152-177)
//   valueHead == 1: mean, mean*(sqrt(area)-14)/10, mean*((sqrt(area)-14)^2/100 - 0.1)   (poolRowsValueHead :179-197)
// The sums run over the frame's positions in frame order whatever the row layout, so that they do not depend on it.
cudaError_t launchGPool(const void* raw, int rawFp32, int ldr, int c0, int C, const float* bnScale, const float* bnBias, int act,
                        const float* mask, const float* maskSum, int n, Layout L, const RowPlan& rp, int valueHead, float* pooled,
                        cudaStream_t s);

// act_out[m][c] = mask * act( (raw[m][c] + ncbias[img][c]) * scale[c] + bias[c] )  for c < C, zero for c in [C, cp)
// (addNCBiasInplace + BatchNormLayer::apply, eigenbackend.cpp:137-148,739-762), for the rows the plan uses (of at most M).
cudaError_t launchBiasAct(const void* raw, int rawFp32, int ldr, int C, const float* ncbias, int ldb, const float* bnScale,
                          const float* bnBias, int act, const float* mask, int M, const RowPlan& rp, __half* actOut, int cp, int split,
                          cudaStream_t s);

// Policy head tail (PolicyHead::apply eigenbackend.cpp:2022-2025 + getOutput :2539-2565):
//   h = mask*act(BN_p1(raw[m][c0+c] + g1bias[img][c])), logits_k = sum_c h_c * Wp2[c][k], k < cp2
//   policy[img][inverse_symmetry(y,x)] = l0 + (l1 - l0) * optimism   (cp2 >= 2) or l0 (cp2 == 1)
cudaError_t launchPolicyOut(const float* raw, int ldr, int c0, int C, const float* g1bias, int ldb, const float* bnScale,
                            const float* bnBias, int act, const float* Wp2, int cp2, const float* mask, const int* symmetry,
                            const float* optimism, int n, Layout L, const RowPlan& rp, float* policy /*[n][X*Y+1]*/,
                            cudaStream_t s);

// Ownership (ValueHead::apply eigenbackend.cpp:2113): own[img][inv_sym(y,x)] = sum_c mask*act(BN_v1(raw[m][c0+c])) * Wown[c]
cudaError_t launchOwnershipOut(const float* raw, int ldr, int c0, int C, const float* bnScale, const float* bnBias, int act,
                               const float* Wown, const float* mask, const int* symmetry, int n, Layout L, const RowPlan& rp,
                               float* ownership /*[n][X*Y]*/, cudaStream_t s);

// pass logit + value/score packing (getOutput eigenbackend.cpp:2563-2626):
//   policy[n][X*Y] = pp0 + (pp1-pp0)*optimism (or pp0), value[n][3], score[n][6] by model version.
cudaError_t launchFinalize(const float* passLogits, int ldp, int cp2, const float* optimism, const float* value, const float* sv,
                           int numSV, int version, int n, int policyStride, float* policy, float* valueOut, float* scoreOut,
                           cudaStream_t s);

}  // namespace kgb
