// Small fp32 kernels around the wgmma convolution: input packing, pooling, tiny matmuls, head outputs.
#pragma once
#include "kgb_conv.cuh"

namespace kgb {

struct Layout {
  int X, Y, pad, Wp, P;  // P = (Y+pad)*(X+pad) rows per image; row of (y,x) = (y+pad)*Wp + x
};

// Inputs (reference: NeuralNet::getOutput eigenbackend.cpp:2467-2486 + SymmetryHelpers::copyInputsWithSymmetry
// nninputs.cpp:529-590; mask = input channel 0, eigenbackend.cpp:2181; computeMaskSum :124).
// spatial: [n][C][Y][X] (NCHW) or [n][Y][X][C] (NHWC) fp32 as written by NNInputs::fillRowV7.
cudaError_t launchPackInput(const float* spatial, int n, int C, bool nhwc, const int* symmetry, Layout L,
                            __half* act, int cin_p, int split, float* mask, float* maskSum, cudaStream_t s);

// out[n][co] = act( sum_k in[n][k] * W[k][co] + bias[co] )   (MatMulLayer / MatBiasLayer / ActivationLayer,
// eigenbackend.cpp:811-862); out has leading dimension ldo and is zero-filled in [cout, ldo).
cudaError_t launchMatMulNC(const float* in, int ldi, const float* W, const float* bias, int n, int cin, int cout, int act,
                           float* out, int ldo, cudaStream_t s);

// Global pooling of act(BN(raw[:, c0:c0+C])) * mask  ->  pooled [n][3C]
//   valueHead == 0: mean, mean*(sqrt(area)-14)/10, max       (poolRowsGPool, eigenbackend.cpp:152-177)
//   valueHead == 1: mean, mean*(sqrt(area)-14)/10, mean*((sqrt(area)-14)^2/100 - 0.1)   (poolRowsValueHead :179-197)
cudaError_t launchGPool(const void* raw, int rawFp32, int ldr, int c0, int C, const float* bnScale, const float* bnBias, int act,
                        const float* mask, const float* maskSum, int n, Layout L, int valueHead, float* pooled, cudaStream_t s);

// act_out[m][c] = mask * act( (raw[m][c] + ncbias[img][c]) * scale[c] + bias[c] )  for c < C, zero for c in [C, cp)
// (addNCBiasInplace + BatchNormLayer::apply, eigenbackend.cpp:137-148,739-762).
cudaError_t launchBiasAct(const void* raw, int rawFp32, int ldr, int C, const float* ncbias, int ldb, const float* bnScale,
                          const float* bnBias, int act, const float* mask, int M, int P, __half* actOut, int cp, int split,
                          cudaStream_t s);

// Policy head tail (PolicyHead::apply eigenbackend.cpp:2022-2025 + getOutput :2539-2565):
//   h = mask*act(BN_p1(raw[m][c0+c] + g1bias[img][c])), logits_k = sum_c h_c * Wp2[c][k], k < cp2
//   policy[img][inverse_symmetry(y,x)] = l0 + (l1 - l0) * optimism   (cp2 >= 2) or l0 (cp2 == 1)
cudaError_t launchPolicyOut(const float* raw, int ldr, int c0, int C, const float* g1bias, int ldb, const float* bnScale,
                            const float* bnBias, int act, const float* Wp2, int cp2, const float* mask, const int* symmetry,
                            const float* optimism, int n, Layout L, float* policy /*[n][X*Y+1]*/, cudaStream_t s);

// Ownership (ValueHead::apply eigenbackend.cpp:2113): own[img][inv_sym(y,x)] = sum_c mask*act(BN_v1(raw[m][c0+c])) * Wown[c]
cudaError_t launchOwnershipOut(const float* raw, int ldr, int c0, int C, const float* bnScale, const float* bnBias, int act,
                               const float* Wown, const float* mask, const int* symmetry, int n, Layout L,
                               float* ownership /*[n][X*Y]*/, cudaStream_t s);

// pass logit + value/score packing (getOutput eigenbackend.cpp:2563-2626):
//   policy[n][X*Y] = pp0 + (pp1-pp0)*optimism (or pp0), value[n][3], score[n][6] by model version.
cudaError_t launchFinalize(const float* passLogits, int ldp, int cp2, const float* optimism, const float* value, const float* sv,
                           int numSV, int version, int n, int policyStride, float* policy, float* valueOut, float* scoreOut,
                           cudaStream_t s);

}  // namespace kgb
