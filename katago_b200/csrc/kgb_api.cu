// C-ABI of libkgb200.so (include/kgb200.h) and the forward-pass engine behind it.
//
// The engine turns a ModelDesc into a flat list of launches ("ops") at handle creation:
//   pack-input -> initial conv(+global matmul bias) -> residual / gpool / nested-bottleneck blocks -> fused head conv
//   -> pooling, tiny matmuls, policy / ownership / value outputs.
// Every convolution is one launch of the wgmma kernel with the NEXT layer's BN+activation+mask fused into its
// epilogue (kgb_conv.cuh), so a trunk layer is exactly one kernel.  Per batch size the whole list is captured once into
// a CUDA graph (no tracing compiler: the op list is static).  Reference structure mirrored: Model/Trunk/heads
// eigenbackend.cpp:1909-2216, getOutput :2445-2628 (and cudabackend.cpp:3649-3888 for the host<->device traffic).
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>      // types only: the library is looked up at run time (ncclApi below), libkgb200.so does not link against it

#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/kgb200.h"
#include "kgb_conv.cuh"
#include "kgb_handle.h"
#include "kgb_kernels.cuh"
#include "kgb_model.h"
#include "kgb_scorevalue.h"
#include "kgb_rand.h"

using namespace kgb;

// ------------------------------------------------------------------------------------------------------------
// Driver entry point for cuTensorMapEncodeTiled (no link-time dependency on libcuda)
// ------------------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled getEncodeTiled() {
  static PFN_encodeTiled fn = nullptr;
  if(fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres));
    if(p == nullptr || qres != cudaDriverEntryPointSuccess) throw CudaFailure("cuTensorMapEncodeTiled is not available from this driver");
    fn = (PFN_encodeTiled)p;
  }
  return fn;
}

// 2-D fp16 row-major tensor [rows][cols], box {64 cols, boxRows}, 128B swizzle, zero OOB fill.
static CUtensorMap makeTmap2D(const void* ptr, uint64_t rows, uint64_t cols, uint32_t boxRows) {
  CUtensorMap m;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {cols * sizeof(__half)};
  cuuint32_t box[2] = {64, boxRows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = getEncodeTiled()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if(r != CUDA_SUCCESS) throw CudaFailure("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
  return m;
}

// 2-D fp16 row-major tensor [rows][cols], box {32 cols, boxRows}, 64B swizzle, zero OOB fill: one 32-column k-chunk of a packed
// weight matrix, K-major, for kgb_conv_pair_epi_kernel's entry MMAs.
static CUtensorMap makeTmapK32(const void* ptr, uint64_t rows, uint64_t cols, uint32_t boxRows) {
  CUtensorMap m;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {cols * sizeof(__half)};
  cuuint32_t box[2] = {(cuuint32_t)kConvPairEpiChunk, boxRows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = getEncodeTiled()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if(r != CUDA_SUCCESS) throw CudaFailure("cuTensorMapEncodeTiled (k32) failed with CUresult " + std::to_string((int)r));
  return m;
}

// Epilogue slices of a stream or operand [rows][cols], fp32 or fp16, box {32 cols, convSliceBoxRows() rows}: the residual the
// convolution's epilogue reads into shared memory and the raw and activated outputs it stores from there, 128B-swizzled for fp32
// (128 B rows) and 64B-swizzled for fp16 (64 B rows), zero OOB fill (rows past the end are clipped on store).
static CUtensorMap makeTmapSlices(const void* ptr, uint64_t rows, uint64_t cols, bool fp32) {
  CUtensorMap m;
  const uint64_t esize = fp32 ? sizeof(float) : sizeof(__half);
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {cols * esize};
  cuuint32_t box[2] = {32, (cuuint32_t)convSliceBoxRows()};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = getEncodeTiled()(&m, fp32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), gdim,
                                gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, fp32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if(r != CUDA_SUCCESS) throw CudaFailure("cuTensorMapEncodeTiled (slices) failed with CUresult " + std::to_string((int)r));
  return m;
}

// ------------------------------------------------------------------------------------------------------------
// Opaque handles
// ------------------------------------------------------------------------------------------------------------
struct kgb_model {
  std::unique_ptr<ModelDesc> desc;
};

struct kgb_context {
  std::vector<int> gpuIdxs;
  int X = 0, Y = 0;
  int fp16 = 1;
  const kgb_model* model = nullptr;
};

static inline int cpad(int c) { return (c + 63) / 64 * 64; }

struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
};

struct ConvWeights {
  __half* w = nullptr;     // packed [taps][cout_p][cin_p * (split ? 2 : 1)]
  int ky = 0, kx = 0, cin_p = 0, cout_p = 0, n_tile = 0, num_n_tiles = 0;
  CUtensorMap tmapB;       // box {64, n_tile}
};

// ------------------------------------------------------------------------------------------------------------
// Graph builder
// ------------------------------------------------------------------------------------------------------------
namespace {

struct Builder {
  kgb_handle& h;
  const ModelDesc& m;
  size_t Mmax;
  int actMul;  // 2 in split mode ([hi | lo])
  Builder(kgb_handle& hh) : h(hh), m(*hh.model), Mmax(hh.planRows(hh.maxBatch)), actMul(hh.split ? 2 : 1) {}

  // Chaining (kgb_conv.cuh, launchConvWG): in a forward (build), a convolution op that directly follows another convolution op is
  // launched as a programmatic dependent of it, with the previous op's flag slot as its predecessor.  The single-layer hooks emit
  // ops that run one at a time, without a predecessor; nothing reads their flags, so these are never zeroed.
  bool chain = false;
  int lastConvOp = -1, lastConvSlot = -1, lastConvParts = 0;
  // The flag slot of the next convolution op, and the slot and flag target of its predecessor (-1: none)
  struct ChainLink {
    int slot, pred, predParts;
  };
  ChainLink nextLink() {
    const bool linked = chain && lastConvOp >= 0 && (size_t)lastConvOp + 1 == h.ops.size();
    h.chainedLaunches += linked ? 1 : 0;
    return ChainLink{h.chainSlots++, linked ? lastConvSlot : -1, linked ? lastConvParts : 0};
  }
  void linkConvOp(const ChainLink& l, int parts) {
    lastConvOp = (int)h.ops.size() - 1;
    lastConvSlot = l.slot;
    lastConvParts = parts;
  }
  static void applyLink(const kgb_handle& hh, const ChainLink& l, ConvParams& p) {
    p.tile_flags = hh.chainFlags(l.slot);
    p.pred_flags = l.pred >= 0 ? hh.chainFlags(l.pred) : nullptr;
    p.pred_parts = l.predParts;
  }

  struct Level {
    int C = 0, cp = 0;
    bool fp32 = false;
    void* S = nullptr;       // raw stream [M][cp]
    __half* A = nullptr;     // act(preBN(S)) for the next consumer
    __half* T = nullptr;     // mid activations inside residual units
    float* G = nullptr;      // fp32 raw output of the gpool unit's first conv
    int gcp = 0;
  };

  // Levels with the same channel count share their buffers (all nested blocks of a net reuse one set): a line that is
  // overwritten while still in L2 never costs an HBM write-back, and the footprint stays ~0.5 GB at batch 256.
  std::map<int, Level> levelCache;

  Level makeLevel(int C, bool fp32, const std::vector<BlockDesc>& blocks) {
    Level& lv = levelCache[C * 2 + (fp32 ? 1 : 0)];
    if(lv.S == nullptr) {
      lv.C = C; lv.cp = cpad(C); lv.fp32 = fp32;
      lv.S = fp32 ? (void*)h.dalloc<float>(Mmax * lv.cp) : (void*)h.dalloc<__half>(Mmax * lv.cp);
      lv.A = h.dalloc<__half>(Mmax * lv.cp * actMul);
    }
    bool needT = false;
    int gcp = 0;
    for(const auto& b : blocks) {
      if(b.kind != BLOCK_NESTED) needT = true;
      if(b.kind == BLOCK_GPOOL) gcp = std::max(gcp, cpad(b.conv1.cout + b.gpoolConv.cout));
    }
    if(needT && lv.T == nullptr) lv.T = h.dalloc<__half>(Mmax * lv.cp * actMul);
    if(gcp > lv.gcp) { lv.G = h.dalloc<float>(Mmax * gcp); lv.gcp = gcp; }
    return lv;
  }

  // Pack one or more convs (concatenated along cout) as fp16 [tap][cout_p][cin_p (* 2)]
  ConvWeights packConv(const std::vector<const ConvDesc*>& convs) {
    const ConvDesc& c0 = *convs[0];
    ConvWeights cw;
    cw.ky = c0.ky; cw.kx = c0.kx;
    cw.cin_p = cpad(c0.cin);
    int cout = 0;
    for(auto c : convs) {
      if(c->ky != c0.ky || c->kx != c0.kx || c->cin != c0.cin) throw std::invalid_argument("cannot fuse convolutions of different shapes");
      cout += c->cout;
    }
    cw.cout_p = cpad(cout);
    int nt = (cw.cout_p + 255) / 256;
    while(cw.cout_p % nt != 0 || (cw.cout_p / nt) % 32 != 0) nt++;
    cw.num_n_tiles = nt;
    cw.n_tile = cw.cout_p / nt;
    int taps = cw.ky * cw.kx;
    int ldw = cw.cin_p * actMul;
    h.wSignature += "conv" + std::to_string(cw.ky) + "x" + std::to_string(cw.kx) + ":" + std::to_string(c0.cin) + ">" + std::to_string(cout) + ";";
    const size_t count = (size_t)taps * cw.cout_p * ldw;
    void* hostDst = nullptr;
    cw.w = (__half*)h.walloc(count * sizeof(__half), &hostDst);
    if(h.wMode == kgb_handle::W_SIZE) return cw;
    std::vector<__half> host(count, __float2half(0.0f));
    int coBase = 0;
    for(auto c : convs) {
      for(int t = 0; t < taps; t++)
        for(int ci = 0; ci < c->cin; ci++)
          for(int co = 0; co < c->cout; co++) {
            float w = c->w[((size_t)t * c->cin + ci) * c->cout + co];
            __half hi = __float2half_rn(w);
            size_t o = ((size_t)t * cw.cout_p + coBase + co) * ldw + ci;
            host[o] = hi;
            if(h.split) host[o + cw.cin_p] = __float2half_rn(w - __half2float(hi));
          }
      coBase += c->cout;
    }
    memcpy(hostDst, host.data(), count * sizeof(__half));
    cw.tmapB = makeTmap2D(cw.w, (uint64_t)taps * cw.cout_p, (uint64_t)ldw, (uint32_t)cw.n_tile);
    return cw;
  }

  struct BNDev {
    const float* scale = nullptr;
    const float* bias = nullptr;
    int act = ACT_IDENTITY;
  };
  BNDev uploadBN(const BNDesc& bn, int act, int cp) {
    BNDev d;
    h.wSignature += "bn" + std::to_string(act) + "," + std::to_string(cp) + ";";
    d.scale = h.upload(bn.scale, cp);
    d.bias = h.upload(bn.bias, cp);
    d.act = act;
    return d;
  }

  // The launch parameters of one convolution at batch n
  static ConvParams convParams(const kgb_handle& hh, int n, const ConvWeights& cw, const void* residual, bool residualFp32, const float* ncbias,
                               void* rawOut, bool rawFp32, __half* actOut, BNDev bn) {
    ConvParams p;
    memset(&p, 0, sizeof(p));
    p.M = (int)hh.planRows(n);
    p.Wp = hh.L.Wp;
    p.tile_wp = hh.plan.tileWp;
    p.row_img = hh.plan.rowImg;
    p.m_tiles = hh.plan.stats + 1;
    p.ky = cw.ky; p.kx = cw.kx;
    p.cin_p = cw.cin_p; p.cout_p = cw.cout_p;
    p.n_tile = cw.n_tile;
    p.num_m_tiles = (p.M + 127) / 128;
    p.num_n_tiles = cw.num_n_tiles;
    p.split = hh.split;
    p.residual = residual; p.residual_fp32 = residualFp32 ? 1 : 0;
    p.ncbias = ncbias;
    p.raw_out = rawOut; p.raw_fp32 = rawFp32 ? 1 : 0;
    p.act_out = actOut;
    p.bn_scale = bn.scale; p.bn_bias = bn.bias; p.act = bn.act;
    p.mask = hh.dMask;
    p.epi_wg = hh.epilogueWG ? 1 : 0;
    p.pair_epi_wg = hh.pairEpilogueWG ? 1 : 0;
    return p;
  }

  // Emit a block boundary as one op (launchConvPair): the exit conv `wpost` of a nested block (operand innerA, residual stream S
  // updated in place, the next block's preBN `bn1`) and the entry conv `wpre` of the next nested block (raw stream innerS, activated
  // operand innerAOut, its first inner block's preBN `bn2`).  The trunk operand between them never leaves the kernel.  innerAOut may
  // be innerA: levels of one width share their buffers, and the kernel reads each tile's operand rows before it writes them.
  // Returns false, emitting nothing, when the kernel does not take these shapes or epilogues.
  bool emitConvPair(const ConvWeights& wpost, const __half* innerA, void* S, bool sFp32, BNDev bn1, const ConvWeights& wpre, void* innerS,
                    bool innerFp32, __half* innerAOut, BNDev bn2) {
    const ConvParams q1 = convParams(h, h.maxBatch, wpost, S, sFp32, nullptr, S, sFp32, nullptr, bn1);
    const ConvParams q2 = convParams(h, h.maxBatch, wpre, nullptr, false, nullptr, innerS, innerFp32, innerAOut, bn2);
    if(!convPairSupported(q1, q2)) return false;
    // the kernel choice depends on the shapes and streams only, which do not change with the batch
    const bool epi = convPairEpilogueWG(q1, q2);
    kgb_handle* hp = &h;
    const ChainLink link = nextLink();
    h.ops.push_back([=](int n, cudaStream_t s) {
      ConvParams p1 = convParams(*hp, n, wpost, S, sFp32, nullptr, S, sFp32, nullptr, bn1);
      const ConvParams p2 = convParams(*hp, n, wpre, nullptr, false, nullptr, innerS, innerFp32, innerAOut, bn2);
      applyLink(*hp, link, p1);
      ConvPairTmaps tm;
      memset(&tm, 0, sizeof(tm));
      tm.A = makeTmap2D(innerA, (uint64_t)p1.M, (uint64_t)wpost.cin_p, (uint32_t)convABoxRows(1, 1, p1.Wp));
      tm.W1 = makeTmap2D(wpost.w, (uint64_t)wpost.cout_p, (uint64_t)wpost.cin_p, (uint32_t)(epi ? kConvPairEpiChunk : kConvPairChunk));
      tm.W2 = epi ? makeTmapK32(wpre.w, (uint64_t)wpre.cout_p, (uint64_t)wpre.cin_p, (uint32_t)wpre.n_tile) : wpre.tmapB;
      tm.stream1 = makeTmapSlices(S, (uint64_t)p1.M, (uint64_t)wpost.cout_p, sFp32);
      tm.stream2 = makeTmapSlices(innerS, (uint64_t)p1.M, (uint64_t)wpre.cout_p, innerFp32);
      tm.act2 = makeTmapSlices(innerAOut, (uint64_t)p1.M, (uint64_t)wpre.cout_p, false);
      CK(launchConvPair(tm, p1, p2, s));
    });
    linkConvOp(link, convPairChainParts(q1, q2));
    h.launchesPerForward++;
    h.pairEpilogueWGLaunches += epi ? 1 : 0;
    return true;
  }

  // Emit one convolution op.  residual/rawOut may alias (in-place residual update).
  void emitConv(const ConvWeights& cw, const __half* A, const void* residual, bool residualFp32, const float* ncbias, void* rawOut,
                bool rawFp32, __half* actOut, BNDev bn) {
    // the kernel reads a tile's halo rows of A while the neighbouring tiles write their outputs (the scratch passes have no buffers)
    if(h.wMode == kgb_handle::W_BUILD && ((const void*)A == (const void*)actOut || (const void*)A == rawOut))
      throw std::logic_error("emitConv: the operand aliases an output");
    // the epilogue writes the raw output over the residual slice it read
    if(residual != nullptr && rawOut != nullptr && residualFp32 != rawFp32)
      throw std::logic_error("emitConv: the residual and the raw output differ in dtype");
    kgb_handle* hp = &h;
    const int actMulL = actMul;
    const ChainLink link = nextLink();
    h.ops.push_back([=](int n, cudaStream_t s) {
      ConvParams p = convParams(*hp, n, cw, residual, residualFp32, ncbias, rawOut, rawFp32, actOut, bn);
      applyLink(*hp, link, p);
      ConvTmaps tm;
      memset(&tm, 0, sizeof(tm));
      tm.A = makeTmap2D(A, (uint64_t)p.M, (uint64_t)cw.cin_p * actMulL, (uint32_t)convABoxRows(cw.ky, cw.kx, p.Wp));
      tm.B = cw.tmapB;
      if(residual != nullptr) tm.residual = makeTmapSlices(residual, (uint64_t)p.M, (uint64_t)cw.cout_p, residualFp32);
      if(rawOut != nullptr) tm.raw = makeTmapSlices(rawOut, (uint64_t)p.M, (uint64_t)cw.cout_p, rawFp32);
      if(actOut != nullptr) tm.act = makeTmapSlices(actOut, (uint64_t)p.M, (uint64_t)cw.cout_p * actMulL, false);
      CK(launchConvWG(tm, p, s));
    });
    linkConvOp(link, 2 * cw.num_n_tiles);
    h.launchesPerForward++;
    h.epilogueWGLaunches += convEpilogueWG(convParams(h, h.maxBatch, cw, residual, residualFp32, ncbias, rawOut, rawFp32, actOut, bn)) ? 1 : 0;
  }

  // blocks operate on stream lv.S, with lv.A = act(preBN_0(S)) on entry and = act(finalBN(S_out)) on exit.
  void emitBlocks(const std::vector<BlockDesc>& blocks, Level& lv, const BNDesc& finalBN, int finalAct, bool keepFinalRaw) {
    // A nested block followed by another nested block holds its exit conv back: the next block's entry conv goes out with it as
    // one launch when emitConvPair takes the pair, else the two go out as before.  Either way the weights are packed in the same
    // order, so the arena layout does not depend on the choice.
    bool exitPending = false;
    ConvWeights pendingW;
    __half* pendingA = nullptr;
    BNDev pendingBN;
    for(size_t i = 0; i < blocks.size(); i++) {
      const BlockDesc& b = blocks[i];
      bool last = i + 1 == blocks.size();
      const BNDesc& nextBNd = last ? finalBN : blocks[i + 1].preBN;
      int nextAct = last ? finalAct : blocks[i + 1].preAct;
      BNDev nextBN = uploadBN(nextBNd, nextAct, lv.cp);
      void* rawOut = (last && !keepFinalRaw) ? nullptr : lv.S;
      if(b.kind == BLOCK_ORDINARY) {
        ConvWeights w1 = packConv({&b.conv1});
        ConvWeights w2 = packConv({&b.conv2});
        BNDev mid = uploadBN(b.midBN, b.midAct, w1.cout_p);
        emitConv(w1, lv.A, nullptr, false, nullptr, nullptr, false, lv.T, mid);
        emitConv(w2, lv.T, lv.S, lv.fp32, nullptr, rawOut, lv.fp32, lv.A, nextBN);
      }
      else if(b.kind == BLOCK_GPOOL) {
        ConvWeights w1 = packConv({&b.conv1, &b.gpoolConv});
        ConvWeights w2 = packConv({&b.conv2});
        const int regC = b.conv1.cout, gC = b.gpoolConv.cout;
        BNDev none;
        emitConv(w1, lv.A, nullptr, false, nullptr, lv.G, true, nullptr, none);
        BNDev gbn = uploadBN(b.gpoolBN, b.gpoolAct, gC);
        float* pooled = h.dalloc<float>((size_t)h.maxBatch * 3 * gC);
        float* bias = h.dalloc<float>((size_t)h.maxBatch * regC);
        const float* Wg = h.upload(b.gpoolToBias.w);
        BNDev mid = uploadBN(b.midBN, b.midAct, regC);
        kgb_handle* hp = &h;
        float* G = lv.G; __half* T = lv.T;
        const int gld = w1.cout_p, tcp = w2.cin_p, split = h.split;
        h.ops.push_back([=](int n, cudaStream_t s) {
          CK(launchGPool(G, 1, gld, regC, gC, gbn.scale, gbn.bias, gbn.act, hp->dMask, hp->dMaskSum, n, hp->L, hp->plan, 0, pooled, s));
          CK(launchMatMulNC(pooled, 3 * gC, Wg, nullptr, n, 3 * gC, regC, ACT_IDENTITY, bias, regC, s));
          CK(launchBiasAct(G, 1, gld, regC, bias, regC, mid.scale, mid.bias, mid.act, hp->dMask, (int)hp->planRows(n), hp->plan, T, tcp, split, s));
        });
        h.launchesPerForward += 3;
        emitConv(w2, lv.T, lv.S, lv.fp32, nullptr, rawOut, lv.fp32, lv.A, nextBN);
      }
      else {
        ConvWeights wpre = packConv({&b.conv1});
        ConvWeights wpost = packConv({&b.conv2});
        Level inner = makeLevel(b.conv1.cout, h.streamInnerFp32, b.blocks);
        BNDev innerPre = uploadBN(b.blocks[0].preBN, b.blocks[0].preAct, inner.cp);
        if(!exitPending || !emitConvPair(pendingW, pendingA, lv.S, lv.fp32, pendingBN, wpre, inner.S, inner.fp32, inner.A, innerPre)) {
          if(exitPending) emitConv(pendingW, pendingA, lv.S, lv.fp32, nullptr, lv.S, lv.fp32, lv.A, pendingBN);
          emitConv(wpre, lv.A, nullptr, false, nullptr, inner.S, inner.fp32, inner.A, innerPre);
        }
        exitPending = false;
        emitBlocks(b.blocks, inner, b.midBN, b.midAct, false);
        if(h.fuseBoundaries && !last && blocks[i + 1].kind == BLOCK_NESTED) {
          exitPending = true;
          pendingW = wpost; pendingA = inner.A; pendingBN = nextBN;
        }
        else emitConv(wpost, inner.A, lv.S, lv.fp32, nullptr, rawOut, lv.fp32, lv.A, nextBN);
      }
    }
  }

  void build() {
    const Layout& L = h.L;
    const int XY = L.X * L.Y;
    const int cinP = cpad(m.numInputChannels);
    // inputs / outputs
    h.dSpatial = h.dalloc<float>((size_t)h.maxBatch * m.numInputChannels * XY);
    h.dGlobal = h.dalloc<float>((size_t)h.maxBatch * m.numInputGlobalChannels);
    h.dOptimism = h.dalloc<float>(h.maxBatch);
    h.dSymmetry = h.dalloc<int>(h.maxBatch);
    h.dPolicy = h.dalloc<float>((size_t)h.maxBatch * (XY + 1));
    h.dValue = h.dalloc<float>((size_t)h.maxBatch * 3);
    h.dScore = h.dalloc<float>((size_t)h.maxBatch * 6);
    h.dOwnership = h.dalloc<float>((size_t)h.maxBatch * XY);
    h.dMask = h.dalloc<float>(Mmax + 128);
    h.dMaskSum = h.dalloc<float>(h.maxBatch);
    h.plan.box = h.dalloc<int4>(h.maxBatch);
    h.plan.base = h.dalloc<int>(h.maxBatch);
    h.plan.tileWp = h.dalloc<int>(Mmax / 128);
    h.plan.rowImg = h.dalloc<int>(Mmax);
    h.plan.stats = h.dalloc<int>(3);
    __half* inAct = h.dalloc<__half>(Mmax * cinP * actMul);
    kgb_handle* hp = &h;
    const int C = m.numInputChannels, split = h.split;
    chain = true;
    h.ops.push_back([=](int n, cudaStream_t s) {
      CK(cudaMemsetAsync(hp->chain, 0, (size_t)hp->chainSlots * hp->chainStride() * sizeof(int), s));
      CK(launchPlanRows(hp->dSpatial, n, C, hp->nhwc, hp->dSymmetry, hp->L, hp->plan, s));
      CK(launchPackInput(hp->dSpatial, n, C, hp->nhwc, hp->dSymmetry, hp->L, hp->plan, hp->planRows(n), inAct, cinP, split, hp->dMask,
                         hp->dMaskSum, s));
    });
    h.launchesPerForward += 6;
    // trunk
    Level trunk = makeLevel(m.trunkC, h.streamTrunkFp32, m.blocks);
    float* initBias = h.dalloc<float>((size_t)h.maxBatch * trunk.cp);
    const float* Wglob = h.upload(m.initialMatMul.w);
    const int G = m.numInputGlobalChannels, trunkC = m.trunkC, trunkCp = trunk.cp;
    h.ops.push_back([=](int n, cudaStream_t s) {
      CK(launchMatMulNC(hp->dGlobal, G, Wglob, nullptr, n, G, trunkC, ACT_IDENTITY, initBias, trunkCp, s));
    });
    h.launchesPerForward++;
    if(m.numInputMetaChannels > 0) {
      // the SGF-metadata encoder in fp32 in both modes; its output joins the global inputs' bias (eigenbackend.cpp:1839-1857, 1927-1932)
      const MetaEncoderDesc& e = m.metaEncoder;
      h.dMeta = h.dalloc<float>((size_t)h.maxBatch * m.numInputMetaChannels);
      const float *W1 = h.upload(e.mul1.w), *b1 = h.upload(e.bias1.w), *W2 = h.upload(e.mul2.w), *b2 = h.upload(e.bias2.w), *W3 = h.upload(e.mul3.w);
      const int cm = m.numInputMetaChannels, c1 = e.mul1.cout, c2 = e.mul2.cout, act1 = e.act1, act2 = e.act2;
      float* mid1 = h.dalloc<float>((size_t)h.maxBatch * c1);
      float* mid2 = h.dalloc<float>((size_t)h.maxBatch * c2);
      h.ops.push_back([=](int n, cudaStream_t s) {
        CK(launchMatMulNC(hp->dMeta, cm, W1, b1, n, cm, c1, act1, mid1, c1, s));
        CK(launchMatMulNC(mid1, c1, W2, b2, n, c1, c2, act2, mid2, c2, s));
        CK(launchMatMulNC(mid2, c2, W3, nullptr, n, c2, trunkC, ACT_IDENTITY, initBias, trunkCp, s, true));
      });
      h.launchesPerForward += 3;
      h.wSignature += "meta" + std::to_string(cm) + ":" + std::to_string(c1) + "," + std::to_string(c2) + "," + std::to_string(act1) + "," +
                      std::to_string(act2) + ";";
    }
    ConvWeights winit = packConv({&m.initialConv});
    BNDev firstPre = uploadBN(m.blocks[0].preBN, m.blocks[0].preAct, trunk.cp);
    emitConv(winit, inAct, nullptr, false, initBias, trunk.S, trunk.fp32, trunk.A, firstPre);
    emitBlocks(m.blocks, trunk, m.tipBN, m.tipAct, false);
    // heads: one fused 1x1 conv [p1 | g1 | v1] -> fp32 raw H
    ConvWeights wheads = packConv({&m.p1Conv, &m.g1Conv, &m.v1Conv});
    float* H = h.dalloc<float>(Mmax * wheads.cout_p);
    BNDev none;
    emitConv(wheads, trunk.A, nullptr, false, nullptr, H, true, nullptr, none);
    const int p1C = m.p1Conv.cout, g1C = m.g1Conv.cout, v1C = m.v1Conv.cout, hld = wheads.cout_p;
    BNDev g1bn = uploadBN(m.g1BN, m.g1Act, g1C);
    BNDev p1bn = uploadBN(m.p1BN, m.p1Act, p1C);
    BNDev v1bn = uploadBN(m.v1BN, m.v1Act, v1C);
    float* g1pool = h.dalloc<float>((size_t)h.maxBatch * 3 * g1C);
    float* g1bias = h.dalloc<float>((size_t)h.maxBatch * p1C);
    const float* Wg2b = h.upload(m.gpoolToBias.w);
    const float* Wp2 = h.upload(m.p2Conv.w);
    const int cp2 = m.policyOutChannels;
    const float* Wpass = h.upload(m.gpoolToPass.w);
    const int passMid = m.gpoolToPass.cout;
    const float* passBias = m.version >= 15 ? h.upload(m.gpoolToPassBias.w) : nullptr;
    const float* Wpass2 = m.version >= 15 ? h.upload(m.gpoolToPass2.w) : nullptr;
    const int passAct = m.passAct, version = m.version;
    float* passH = h.dalloc<float>((size_t)h.maxBatch * std::max(passMid, 4));
    float* passLogits = h.dalloc<float>((size_t)h.maxBatch * 4);
    float* v1pool = h.dalloc<float>((size_t)h.maxBatch * 3 * v1C);
    const int v2C = m.v2Mul.cout;
    float* v2 = h.dalloc<float>((size_t)h.maxBatch * v2C);
    const float* Wv2 = h.upload(m.v2Mul.w); const float* bv2 = h.upload(m.v2Bias.w); const int v2Act = m.v2Act;
    const float* Wv3 = h.upload(m.v3Mul.w); const float* bv3 = h.upload(m.v3Bias.w);
    const float* Wsv3 = h.upload(m.sv3Mul.w); const float* bsv3 = h.upload(m.sv3Bias.w);
    const int numSV = m.sv3Mul.cout;
    float* value = h.dalloc<float>((size_t)h.maxBatch * 3);
    float* sv = h.dalloc<float>((size_t)h.maxBatch * 8);
    const float* Wown = h.upload(m.ownershipConv.w);
    h.ops.push_back([=](int n, cudaStream_t s) {
      // policy head
      CK(launchGPool(H, 1, hld, p1C, g1C, g1bn.scale, g1bn.bias, g1bn.act, hp->dMask, hp->dMaskSum, n, hp->L, hp->plan, 0, g1pool, s));
      CK(launchMatMulNC(g1pool, 3 * g1C, Wg2b, nullptr, n, 3 * g1C, p1C, ACT_IDENTITY, g1bias, p1C, s));
      CK(launchPolicyOut(H, hld, 0, p1C, g1bias, p1C, p1bn.scale, p1bn.bias, p1bn.act, Wp2, cp2, hp->dMask, hp->dSymmetry,
                         hp->dOptimism, n, hp->L, hp->plan, hp->dPolicy, s));
      if(version >= 15) {
        CK(launchMatMulNC(g1pool, 3 * g1C, Wpass, passBias, n, 3 * g1C, passMid, passAct, passH, passMid, s));
        CK(launchMatMulNC(passH, passMid, Wpass2, nullptr, n, passMid, cp2, ACT_IDENTITY, passLogits, 4, s));
      }
      else {
        CK(launchMatMulNC(g1pool, 3 * g1C, Wpass, nullptr, n, 3 * g1C, cp2, ACT_IDENTITY, passLogits, 4, s));
      }
      // value head
      CK(launchGPool(H, 1, hld, p1C + g1C, v1C, v1bn.scale, v1bn.bias, v1bn.act, hp->dMask, hp->dMaskSum, n, hp->L, hp->plan, 1, v1pool, s));
      CK(launchMatMulNC(v1pool, 3 * v1C, Wv2, bv2, n, 3 * v1C, v2C, v2Act, v2, v2C, s));
      CK(launchMatMulNC(v2, v2C, Wv3, bv3, n, v2C, 3, ACT_IDENTITY, value, 3, s));
      CK(launchMatMulNC(v2, v2C, Wsv3, bsv3, n, v2C, numSV, ACT_IDENTITY, sv, numSV, s));
      CK(launchOwnershipOut(H, hld, p1C + g1C, v1C, v1bn.scale, v1bn.bias, v1bn.act, Wown, hp->dMask, hp->dSymmetry, n, hp->L, hp->plan,
                            hp->dOwnership, s));
      CK(launchFinalize(passLogits, 4, cp2, hp->dOptimism, value, sv, numSV, version, n, hp->L.X * hp->L.Y + 1, hp->dPolicy,
                        hp->dValue, hp->dScore, s));
    });
    h.launchesPerForward += (version >= 15 ? 11 : 10);
    h.allocChain();
    // constants the ops above captured by value, and the post-processing constants callers read from the model: a staged model
    // (kgb_handle_stage_weights) must agree on all of them
    char buf[512];
    snprintf(buf, sizeof(buf), "v%d in%d,%d trunk%d heads%d,%d,%d pol%d pass%d,%d v2:%d,%d sv%d own%d mult%.9g,%.9g,%.9g,%.9g,%.9g,%.9g,%.9g", version,
             m.numInputChannels, m.numInputGlobalChannels, m.trunkC, p1C, g1C, v1C, cp2, passMid, passAct, v2C, v2Act, numSV, m.ownershipConv.cout,
             (double)m.tdScoreMultiplier, (double)m.scoreMeanMultiplier, (double)m.scoreStdevMultiplier, (double)m.leadMultiplier,
             (double)m.varianceTimeMultiplier, (double)m.shorttermValueErrorMultiplier, (double)m.shorttermScoreErrorMultiplier);
    h.wSignature += buf;
  }
};

// serial: the ops one at a time, outside a graph, each followed by a stream synchronise - the reference the chained graph is
// tested against (kgb_test_forward_serial)
void runOps(kgb_handle* h, int n, bool serial = false) {
  if(serial) {
    for(auto& op : h->ops) {
      op(n, h->stream);
      CK(cudaStreamSynchronize(h->stream));
    }
    return;
  }
  auto it = h->graphs.find(n);
  if(it == h->graphs.end())
    it = h->graphs.emplace(n, captureGraph(h->stream, [&] { for(auto& op : h->ops) op(n, h->stream); })).first;
  CK(cudaGraphLaunch(it->second, h->stream));
}

}  // namespace

cudaGraphExec_t captureGraph(cudaStream_t s, const std::function<void()>& launches) {
  cudaGraph_t graph = nullptr;
  CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
  try {
    launches();
  }
  catch(...) {
    cudaStreamEndCapture(s, &graph);
    if(graph) cudaGraphDestroy(graph);
    throw;
  }
  CK(cudaStreamEndCapture(s, &graph));
  cudaGraphExec_t exec = nullptr;
  const cudaError_t e = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  CK(e);
  return exec;
}

// ------------------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------------------
extern "C" {

KGB_API int kgb_global_init(void) { return KGB_OK; }
KGB_API int kgb_global_cleanup(void) { return KGB_OK; }
KGB_API const char* kgb_last_error(void) { return g_lastError.c_str(); }

KGB_API int kgb_device_count(int* count) {
  return guarded([&] {
    if(!count) throw std::invalid_argument("kgb_device_count: count is NULL");
    int c = 0;
    cudaError_t e = cudaGetDeviceCount(&c);
    if(e != cudaSuccess) { cudaGetLastError(); c = 0; }
    *count = c;
  });
}

KGB_API int kgb_device_name(int device, char* buf, int buf_len, int* cc_major, int* cc_minor) {
  return guarded([&] {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    if(buf && buf_len > 0) { strncpy(buf, prop.name, buf_len - 1); buf[buf_len - 1] = 0; }
    if(cc_major) *cc_major = prop.major;
    if(cc_minor) *cc_minor = prop.minor;
  });
}

KGB_API int kgb_model_load_file(const char* path, const char* expected_sha256, kgb_model** out) {
  return guarded([&] {
    if(!path || !out) throw std::invalid_argument("kgb_model_load_file: NULL argument");
    std::unique_ptr<kgb_model> m(new kgb_model());
    m->desc = loadModelFile(path, expected_sha256 ? expected_sha256 : "");
    *out = m.release();
  });
}

KGB_API void kgb_model_free(kgb_model* model) { delete model; }

KGB_API int kgb_model_get_info(const kgb_model* model, kgb_model_info* out) {
  return guarded([&] {
    if(!model || !out) throw std::invalid_argument("kgb_model_get_info: NULL argument");
    const ModelDesc& d = *model->desc;
    memset(out, 0, sizeof(*out));
    strncpy(out->name, d.name.c_str(), sizeof(out->name) - 1);
    strncpy(out->sha256, d.sha256.c_str(), sizeof(out->sha256) - 1);
    out->model_version = d.version;
    out->num_input_channels = d.numInputChannels;
    out->num_input_global_channels = d.numInputGlobalChannels;
    out->num_policy_channels = d.policyOutChannels;
    out->num_value_channels = d.v3Mul.cout;
    out->num_score_value_channels = d.sv3Mul.cout;
    out->num_ownership_channels = d.ownershipConv.cout;
    out->trunk_num_channels = d.trunkC;
    out->num_blocks = (int)d.blocks.size();
    out->prefer_pass_alive_under_suicide_rules = d.preferPassAliveUnderSuicideRules;
    out->td_score_multiplier = d.tdScoreMultiplier;
    out->score_mean_multiplier = d.scoreMeanMultiplier;
    out->score_stdev_multiplier = d.scoreStdevMultiplier;
    out->lead_multiplier = d.leadMultiplier;
    out->variance_time_multiplier = d.varianceTimeMultiplier;
    out->shortterm_value_error_multiplier = d.shorttermValueErrorMultiplier;
    out->shortterm_score_error_multiplier = d.shorttermScoreErrorMultiplier;
    out->conv_macs_per_position = d.convMacsPerPosition();
    out->num_input_meta_channels = d.numInputMetaChannels;
  });
}

KGB_API int kgb_context_create(const int* gpu_idxs, int num_gpu_idxs, int nn_x_len, int nn_y_len, int fp16_mode, const kgb_model* model,
                       kgb_context** out) {
  return guarded([&] {
    if(!model || !out) throw std::invalid_argument("kgb_context_create: NULL argument");
    if(nn_x_len < 2 || nn_y_len < 2 || nn_x_len > 37 || nn_y_len > 37) throw std::invalid_argument("kgb_context_create: nnXLen/nnYLen out of range");
    std::unique_ptr<kgb_context> c(new kgb_context());
    for(int i = 0; i < num_gpu_idxs; i++) c->gpuIdxs.push_back(gpu_idxs[i]);
    c->X = nn_x_len; c->Y = nn_y_len;
    c->fp16 = (fp16_mode == 0) ? 0 : 1;
    c->model = model;
    *out = c.release();
  });
}

KGB_API void kgb_context_free(kgb_context* ctx) { delete ctx; }

// NCCL, bound at run time: a single-GPU process never needs it, and a process that has torch loaded shares torch's copy
// (the same communicator library that torch.distributed uses over NVLink / NVSwitch).
struct NcclApi {
  ncclResult_t (*getUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*commInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*commDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*getErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
  std::string why;
};
static NcclApi& ncclApi() {
  static NcclApi api;
  static bool tried = false;
  if(tried) return api;
  tried = true;
  void* lib = nullptr;
  const char* override_ = getenv("KGB_NCCL_LIB");
  for(const char* name : {override_, "libnccl.so.2", "libnccl.so"}) {
    if(name && (lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL)) != nullptr) break;
  }
  if(!lib) { api.why = std::string("libnccl.so.2 cannot be loaded (") + (dlerror() ? dlerror() : "not found") + "); set KGB_NCCL_LIB"; return api; }
  api.getUniqueId = (decltype(api.getUniqueId))dlsym(lib, "ncclGetUniqueId");
  api.commInitRank = (decltype(api.commInitRank))dlsym(lib, "ncclCommInitRank");
  api.commDestroy = (decltype(api.commDestroy))dlsym(lib, "ncclCommDestroy");
  api.broadcast = (decltype(api.broadcast))dlsym(lib, "ncclBroadcast");
  api.getErrorString = (decltype(api.getErrorString))dlsym(lib, "ncclGetErrorString");
  api.ok = api.getUniqueId && api.commInitRank && api.commDestroy && api.broadcast && api.getErrorString;
  if(!api.ok) api.why = "the NCCL library lacks an expected symbol";
  return api;
}
static void ncclCheck(ncclResult_t r, const char* what) {
  if(r != ncclSuccess) throw CudaFailure(std::string(what) + ": " + ncclApi().getErrorString(r));
}

// KGB_EPILOGUE_WG=0 keeps every convolution on kgb_conv_wg_kernel (same-build A/B runs and tests; the results are the same).  Read
// where a handle is made: kgb_handle_create and the single-layer test hooks.
static bool epilogueWGFromEnv() {
  const char* e = getenv("KGB_EPILOGUE_WG");
  return !(e && std::string(e) == "0");
}
// KGB_PAIR_EPILOGUE_WG=0 keeps every fused block boundary on kgb_conv_pair_kernel, in the same way
static bool pairEpilogueWGFromEnv() {
  const char* e = getenv("KGB_PAIR_EPILOGUE_WG");
  return !(e && std::string(e) == "0");
}

// The settings that decide how the graph builder lays the weights out
static void copyBuildSettings(kgb_handle& dst, const kgb_handle& src) {
  dst.device = src.device; dst.model = src.model; dst.L = src.L; dst.maxBatch = src.maxBatch; dst.split = src.split;
  dst.nhwc = src.nhwc; dst.streamTrunkFp32 = src.streamTrunkFp32; dst.streamInnerFp32 = src.streamInnerFp32;
  dst.fuseBoundaries = src.fuseBoundaries; dst.epilogueWG = src.epilogueWG;
  dst.pairEpilogueWG = src.pairEpilogueWG;
}

// Makes device `dev` (-1: the current device) current, after checking that it exists and is the sm_90a device the kernels are
// built for.  Returns its index.
static int selectDevice(int dev) {
  int count = 0;
  if(cudaGetDeviceCount(&count) != cudaSuccess || count == 0)
    throw CudaFailure("libkgb200: no CUDA device is visible; the backend has no CPU fallback");
  if(dev < 0) CK(cudaGetDevice(&dev));
  if(dev >= count) throw std::invalid_argument("libkgb200: gpu index " + std::to_string(dev) + " >= device count");
  CK(cudaSetDevice(dev));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, dev));
  if(prop.major != 9 || prop.minor != 0)
    throw CudaFailure(std::string("libkgb200 is built for sm_90a (H100) only; device ") + prop.name + " is sm_" +
                      std::to_string(prop.major) + std::to_string(prop.minor));
  return dev;
}

// Padded rows of an X x Y board with `pad` zero rows on top and `pad` zero columns at the right (kgb_conv.cuh)
static Layout boardLayout(int X, int Y, int pad) { return Layout{X, Y, pad, X + pad, (Y + pad) * (X + pad)}; }

// The weight arena is laid out by two passes over the same code: pack(handle) runs on a scratch handle that only adds up the
// spans, then on h for real, where walloc checks every span against that list.  The packed bytes reach the device in one copy.
static void buildWeights(kgb_handle& h, const std::function<void(kgb_handle&)>& pack) {
  kgb_handle sizing;
  copyBuildSettings(sizing, h);
  sizing.wMode = kgb_handle::W_SIZE;
  pack(sizing);
  h.wSizes = sizing.wSizes;
  h.wAllocArena(sizing.wCursor);
  pack(h);
  if(h.wCursor != h.wBytes || h.wSignature != sizing.wSignature) throw std::logic_error("libkgb200: the two builder passes disagree");
  h.wFlushLive();
}

static void destroyHandle(kgb_handle* h) {
  if(!h) return;
  cudaSetDevice(h->device);
  for(auto& g : h->graphs) cudaGraphExecDestroy(g.second);
  for(void* p : h->allocs) cudaFree(p);
  if(h->wShadow) cudaFree(h->wShadow);
  if(h->wHost) cudaFreeHost(h->wHost);
  if(h->ncclComm && ncclApi().ok) ncclApi().commDestroy((ncclComm_t)h->ncclComm);
  for(cudaEvent_t e : {h->stagedEvent, h->bcastStart, h->bcastStop}) if(e) cudaEventDestroy(e);
  if(h->copyStream) cudaStreamDestroy(h->copyStream);
  for(void* p : {(void*)h->hSpatial, (void*)h->hGlobal, (void*)h->hMeta, (void*)h->hOptimism, (void*)h->hPolicy, (void*)h->hValue, (void*)h->hScore,
                 (void*)h->hOwnership, (void*)h->hSymmetry})
    if(p) cudaFreeHost(p);
  if(h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

KGB_API int kgb_handle_create(kgb_context* ctx, const kgb_model* model, int max_batch_size, int require_exact_nn_len, int inputs_nhwc,
                      int gpu_idx, kgb_handle** out) {
  (void)require_exact_nn_len;  // masking is always on: it is what zeroes our pad rows
  kgb_handle* raw = nullptr;
  int rc = guarded([&] {
    if(!ctx || !model || !out) throw std::invalid_argument("kgb_handle_create: NULL argument");
    if(max_batch_size < 1 || max_batch_size > 65536) throw std::invalid_argument("kgb_handle_create: maxBatchSize out of range");
    int dev = gpu_idx;
    if(dev < 0) dev = (!ctx->gpuIdxs.empty() && ctx->gpuIdxs[0] >= 0) ? ctx->gpuIdxs[0] : 0;
    dev = selectDevice(dev);
    raw = new kgb_handle();
    kgb_handle& h = *raw;
    h.device = dev;
    h.model = model->desc.get();
    h.maxBatch = max_batch_size;
    h.split = ctx->fp16 ? 0 : 1;
    h.nhwc = inputs_nhwc != 0;
    h.L = boardLayout(ctx->X, ctx->Y, h.model->maxConvRadius());
    // Residual streams: fp32-equivalent mode keeps all of them in fp32; fp16 mode keeps all of them in fp16, like the reference's
    // FP16 CUDA path keeps its trunk in half (cudabackend.cpp: useFP16 buffers).  KGB_STREAM_FP32 = all | trunk | none overrides
    // fp16 mode only.
    const char* env = getenv("KGB_STREAM_FP32");
    std::string streams = h.split ? "all" : (env ? env : "none");
    h.streamTrunkFp32 = streams != "none";
    h.streamInnerFp32 = streams == "all";
    // KGB_FUSE_BOUNDARY=0 keeps every nested block boundary as two launches (same-build A/B runs and tests; the results are the same)
    const char* fuse = getenv("KGB_FUSE_BOUNDARY");
    h.fuseBoundaries = !h.split && !(fuse && std::string(fuse) == "0");
    // KGB_RAGGED_ROWS=0 lays every image out at the full frame (the reference plan of the tests and same-build A/B runs; the
    // results are the same)
    const char* ragged = getenv("KGB_RAGGED_ROWS");
    h.plan.ragged = !(ragged && std::string(ragged) == "0");
    h.epilogueWG = epilogueWGFromEnv();
    h.pairEpilogueWG = pairEpilogueWGFromEnv();
    CK(cudaStreamCreateWithFlags(&h.stream, cudaStreamNonBlocking));
    CK(convWGInit());
    CK(cudaStreamCreateWithFlags(&h.copyStream, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&h.stagedEvent, cudaEventDisableTiming));
    CK(cudaEventCreate(&h.bcastStart));
    CK(cudaEventCreate(&h.bcastStop));
    buildWeights(h, [](kgb_handle& hh) { Builder(hh).build(); });
    const int XY = h.L.X * h.L.Y;
    const ModelDesc& m = *h.model;
    CK(cudaMallocHost((void**)&h.hSpatial, (size_t)h.maxBatch * m.numInputChannels * XY * sizeof(float)));
    CK(cudaMallocHost((void**)&h.hGlobal, (size_t)h.maxBatch * m.numInputGlobalChannels * sizeof(float)));
    if(m.numInputMetaChannels > 0) CK(cudaMallocHost((void**)&h.hMeta, (size_t)h.maxBatch * m.numInputMetaChannels * sizeof(float)));
    CK(cudaMallocHost((void**)&h.hOptimism, (size_t)h.maxBatch * sizeof(float)));
    CK(cudaMallocHost((void**)&h.hSymmetry, (size_t)h.maxBatch * sizeof(int)));
    CK(cudaMallocHost((void**)&h.hPolicy, (size_t)h.maxBatch * (XY + 1) * sizeof(float)));
    CK(cudaMallocHost((void**)&h.hValue, (size_t)h.maxBatch * 3 * sizeof(float)));
    CK(cudaMallocHost((void**)&h.hScore, (size_t)h.maxBatch * 6 * sizeof(float)));
    CK(cudaMallocHost((void**)&h.hOwnership, (size_t)h.maxBatch * XY * sizeof(float)));
    CK(cudaStreamSynchronize(h.stream));
    *out = raw;
    raw = nullptr;
  });
  if(raw) destroyHandle(raw);
  return rc;
}

KGB_API void kgb_handle_free(kgb_handle* handle) { destroyHandle(handle); }

// ---- new weights into a live handle (the reference: a new NNEvaluator per polled model file, command/selfplay.cpp:142-231,336-352) ----

KGB_API int kgb_handle_weights_bytes(const kgb_handle* handle, uint64_t* bytes) {
  return guarded([&] {
    if(!handle || !bytes) throw std::invalid_argument("kgb_handle_weights_bytes: NULL argument");
    *bytes = handle->wBytes;
  });
}

static void ensureShadow(kgb_handle* h) {
  if(h->wShadow) return;
  CK(cudaMalloc((void**)&h->wShadow, std::max<size_t>(h->wBytes, 256)));
  CK(cudaMemsetAsync(h->wShadow, 0, std::max<size_t>(h->wBytes, 256), h->copyStream));
}

KGB_API int kgb_handle_stage_weights(kgb_handle* handle, const kgb_model* model) {
  return guarded([&] {
    if(!handle || !model) throw std::invalid_argument("kgb_handle_stage_weights: NULL argument");
    CK(cudaSetDevice(handle->device));
    ensureShadow(handle);
    CK(cudaStreamSynchronize(handle->copyStream));        // an earlier staging copy may still be reading the host mirror
    kgb_handle pack;
    copyBuildSettings(pack, *handle);
    pack.model = model->desc.get();
    if(pack.model->maxConvRadius() != handle->L.pad) throw std::invalid_argument("kgb_handle_stage_weights: the model's largest convolution differs");
    pack.wMode = kgb_handle::W_REPACK;
    pack.wHost = handle->wHost; pack.wShadow = handle->wShadow; pack.wBytes = handle->wBytes; pack.wSizes = handle->wSizes;
    Builder(pack).build();
    if(pack.wCursor != handle->wBytes || pack.wIndex != handle->wSizes.size() || pack.wSignature != handle->wSignature)
      throw std::invalid_argument("kgb_handle_stage_weights: the model is not of the architecture this handle was built for");
    CK(cudaMemcpyAsync(handle->wShadow, handle->wHost, handle->wBytes, cudaMemcpyHostToDevice, handle->copyStream));
    CK(cudaEventRecord(handle->stagedEvent, handle->copyStream));
    handle->staged = true;
  });
}

KGB_API int kgb_handle_wait_staged(kgb_handle* handle) {
  return guarded([&] {
    if(!handle) throw std::invalid_argument("kgb_handle_wait_staged: NULL handle");
    CK(cudaSetDevice(handle->device));
    CK(cudaStreamSynchronize(handle->copyStream));
  });
}

KGB_API int kgb_handle_commit_weights(kgb_handle* handle) {
  return guarded([&] {
    if(!handle) throw std::invalid_argument("kgb_handle_commit_weights: NULL handle");
    if(!handle->staged) throw std::invalid_argument("kgb_handle_commit_weights: nothing is staged (kgb_handle_stage_weights or kgb_handle_broadcast_staged_weights first)");
    CK(cudaSetDevice(handle->device));
    // ordered on the evaluation stream: every forward pass (and every self-play wave) enqueued after this call sees the new net whole
    CK(cudaStreamWaitEvent(handle->stream, handle->stagedEvent, 0));
    CK(cudaMemcpyAsync(handle->wLive, handle->wShadow, handle->wBytes, cudaMemcpyDeviceToDevice, handle->stream));
    handle->staged = false;
  });
}

KGB_API int kgb_nccl_unique_id(void* id_out_128_bytes) {
  return guarded([&] {
    if(!id_out_128_bytes) throw std::invalid_argument("kgb_nccl_unique_id: NULL argument");
    NcclApi& api = ncclApi();
    if(!api.ok) throw CudaFailure("kgb_nccl_unique_id: " + api.why);
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    ncclUniqueId id;
    ncclCheck(api.getUniqueId(&id), "ncclGetUniqueId");
    memcpy(id_out_128_bytes, &id, sizeof(id));
  });
}

KGB_API int kgb_handle_comm_init(kgb_handle* handle, const void* id_128_bytes, int rank, int num_ranks) {
  return guarded([&] {
    if(!handle || !id_128_bytes) throw std::invalid_argument("kgb_handle_comm_init: NULL argument");
    if(num_ranks < 1 || rank < 0 || rank >= num_ranks) throw std::invalid_argument("kgb_handle_comm_init: rank out of range");
    if(handle->ncclComm) throw std::invalid_argument("kgb_handle_comm_init: the handle already has a communicator");
    NcclApi& api = ncclApi();
    if(!api.ok) throw CudaFailure("kgb_handle_comm_init: " + api.why);
    CK(cudaSetDevice(handle->device));
    ncclUniqueId id;
    memcpy(&id, id_128_bytes, sizeof(id));
    ncclComm_t comm = nullptr;
    ncclCheck(api.commInitRank(&comm, num_ranks, id, rank), "ncclCommInitRank");
    handle->ncclComm = comm; handle->ncclRank = rank; handle->ncclRanks = num_ranks;
  });
}

KGB_API int kgb_handle_broadcast_staged_weights(kgb_handle* handle, int root, float* ms_out) {
  return guarded([&] {
    if(!handle) throw std::invalid_argument("kgb_handle_broadcast_staged_weights: NULL handle");
    if(!handle->ncclComm) throw std::invalid_argument("kgb_handle_broadcast_staged_weights: kgb_handle_comm_init first");
    if(root < 0 || root >= handle->ncclRanks) throw std::invalid_argument("kgb_handle_broadcast_staged_weights: root out of range");
    if(handle->ncclRank == root && !handle->staged) throw std::invalid_argument("kgb_handle_broadcast_staged_weights: the root has nothing staged");
    CK(cudaSetDevice(handle->device));
    ensureShadow(handle);
    // the packed arena (fp16 conv weights, fp32 scales / biases / head matrices), device to device, in place in the shadow arena;
    // the copy stream orders it behind the root's own host-to-device staging copy
    CK(cudaEventRecord(handle->bcastStart, handle->copyStream));
    ncclCheck(ncclApi().broadcast(handle->wShadow, handle->wShadow, handle->wBytes, ncclChar, root, (ncclComm_t)handle->ncclComm, handle->copyStream),
              "ncclBroadcast");
    CK(cudaEventRecord(handle->bcastStop, handle->copyStream));
    CK(cudaEventRecord(handle->stagedEvent, handle->copyStream));
    CK(cudaStreamSynchronize(handle->copyStream));
    float ms = 0.0f;
    CK(cudaEventElapsedTime(&ms, handle->bcastStart, handle->bcastStop));
    if(ms_out) *ms_out = ms;
    handle->staged = true;
  });
}

KGB_API int kgb_handle_is_fp16(const kgb_handle* handle) { return handle && !handle->split ? 1 : 0; }
KGB_API uint64_t kgb_handle_stream(kgb_handle* handle) { return handle ? (uint64_t)(uintptr_t)handle->stream : 0; }
KGB_API int kgb_handle_launches_per_forward(const kgb_handle* handle) { return handle ? handle->launchesPerForward : 0; }
KGB_API int kgb_handle_chained_launches_per_forward(const kgb_handle* handle) { return handle ? handle->chainedLaunches : 0; }
KGB_API int kgb_handle_epilogue_wg_launches_per_forward(const kgb_handle* handle) { return handle ? handle->epilogueWGLaunches : 0; }
KGB_API int kgb_handle_pair_epilogue_wg_launches_per_forward(const kgb_handle* handle) { return handle ? handle->pairEpilogueWGLaunches : 0; }

KGB_API int kgb_handle_get_layout_stats(kgb_handle* handle, int64_t* rows, int64_t* m_tiles, int64_t* segments) {
  return guarded([&] {
    if(!handle || !rows || !m_tiles || !segments) throw std::invalid_argument("kgb_handle_get_layout_stats: NULL argument");
    CK(cudaSetDevice(handle->device));
    int st[3] = {0, 0, 0};
    CK(cudaMemcpyAsync(st, handle->plan.stats, sizeof(st), cudaMemcpyDeviceToHost, handle->stream));
    CK(cudaStreamSynchronize(handle->stream));
    *rows = st[0]; *m_tiles = st[1]; *segments = st[2];
  });
}

KGB_API int kgb_handle_sync(kgb_handle* handle) {
  return guarded([&] {
    if(!handle) throw std::invalid_argument("kgb_handle_sync: NULL handle");
    CK(cudaSetDevice(handle->device));
    CK(cudaStreamSynchronize(handle->stream));
    CK(convChainStatus());
  });
}

static void checkForwardArgs(kgb_handle* h, int n, const void* a, const void* b, const void* c, const void* d, const void* e) {
  if(!h) throw std::invalid_argument("kgb_forward: NULL handle");
  if(n < 1 || n > h->maxBatch) throw std::invalid_argument("kgb_forward: batch size " + std::to_string(n) + " not in [1, maxBatchSize]");
  if(!a || !b || !c || !d || !e) throw std::invalid_argument("kgb_forward: NULL buffer");
}

// A metadata net needs its rows (the reference's fatalError when they are missing, nneval.cpp:471-474), and rows need a metadata net
static void checkMetaArgs(const kgb_handle* h, const void* meta, const char* fn) {
  const bool hasEncoder = h->model->numInputMetaChannels > 0;
  if(hasEncoder && !meta)
    throw std::invalid_argument(std::string(fn) + ": the net has an SGF-metadata encoder and needs a metadata row per image (kgb_forward_meta / kgb_forward_device_meta)");
  if(!hasEncoder && meta) throw std::invalid_argument(std::string(fn) + ": metadata rows given for a net without an SGF-metadata encoder");
}

static void forwardHost(kgb_handle* h, int n, const float* spatial, const float* global, const float* meta, const int32_t* symmetry,
                        const float* policy_optimism, float* policy, float* value, float* score_value, float* ownership) {
  CK(cudaSetDevice(h->device));
  const ModelDesc& m = *h->model;
  const int XY = h->L.X * h->L.Y;
  const size_t spB = (size_t)n * m.numInputChannels * XY * sizeof(float);
  const size_t glB = (size_t)n * m.numInputGlobalChannels * sizeof(float);
  const size_t metaB = (size_t)n * m.numInputMetaChannels * sizeof(float);
  memcpy(h->hSpatial, spatial, spB);
  memcpy(h->hGlobal, global, glB);
  if(meta) memcpy(h->hMeta, meta, metaB);
  for(int i = 0; i < n; i++) {
    h->hSymmetry[i] = symmetry ? symmetry[i] : 0;
    h->hOptimism[i] = policy_optimism ? policy_optimism[i] : 0.0f;
    if(h->hSymmetry[i] < 0 || h->hSymmetry[i] > 7) throw std::invalid_argument("kgb_forward: symmetry must be in 0..7");
  }
  cudaStream_t s = h->stream;
  CK(cudaMemcpyAsync(h->dSpatial, h->hSpatial, spB, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(h->dGlobal, h->hGlobal, glB, cudaMemcpyHostToDevice, s));
  if(meta) CK(cudaMemcpyAsync(h->dMeta, h->hMeta, metaB, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(h->dSymmetry, h->hSymmetry, n * sizeof(int), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(h->dOptimism, h->hOptimism, n * sizeof(float), cudaMemcpyHostToDevice, s));
  runOps(h, n);
  CK(cudaMemcpyAsync(h->hPolicy, h->dPolicy, (size_t)n * (XY + 1) * sizeof(float), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(h->hValue, h->dValue, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(h->hScore, h->dScore, (size_t)n * 6 * sizeof(float), cudaMemcpyDeviceToHost, s));
  if(ownership) CK(cudaMemcpyAsync(h->hOwnership, h->dOwnership, (size_t)n * XY * sizeof(float), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(convChainStatus());
  memcpy(policy, h->hPolicy, (size_t)n * (XY + 1) * sizeof(float));
  memcpy(value, h->hValue, (size_t)n * 3 * sizeof(float));
  memcpy(score_value, h->hScore, (size_t)n * 6 * sizeof(float));
  if(ownership) memcpy(ownership, h->hOwnership, (size_t)n * XY * sizeof(float));
}

static void forwardDevice(kgb_handle* h, int n, const float* d_spatial, const float* d_global, const float* d_meta, const int32_t* d_symmetry,
                          const float* d_policy_optimism, float* d_policy, float* d_value, float* d_score_value, float* d_ownership,
                          bool serial = false) {
  CK(cudaSetDevice(h->device));
  const ModelDesc& m = *h->model;
  const int XY = h->L.X * h->L.Y;
  cudaStream_t s = h->stream;
  if(d_spatial != h->dSpatial)
    CK(cudaMemcpyAsync(h->dSpatial, d_spatial, (size_t)n * m.numInputChannels * XY * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if(d_global != h->dGlobal)
    CK(cudaMemcpyAsync(h->dGlobal, d_global, (size_t)n * m.numInputGlobalChannels * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if(d_meta && d_meta != h->dMeta)
    CK(cudaMemcpyAsync(h->dMeta, d_meta, (size_t)n * m.numInputMetaChannels * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if(d_symmetry) CK(cudaMemcpyAsync(h->dSymmetry, d_symmetry, n * sizeof(int), cudaMemcpyDeviceToDevice, s));
  else CK(cudaMemsetAsync(h->dSymmetry, 0, n * sizeof(int), s));
  if(d_policy_optimism) CK(cudaMemcpyAsync(h->dOptimism, d_policy_optimism, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
  else CK(cudaMemsetAsync(h->dOptimism, 0, n * sizeof(float), s));
  runOps(h, n, serial);
  CK(cudaMemcpyAsync(d_policy, h->dPolicy, (size_t)n * (XY + 1) * sizeof(float), cudaMemcpyDeviceToDevice, s));
  CK(cudaMemcpyAsync(d_value, h->dValue, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToDevice, s));
  CK(cudaMemcpyAsync(d_score_value, h->dScore, (size_t)n * 6 * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if(d_ownership) CK(cudaMemcpyAsync(d_ownership, h->dOwnership, (size_t)n * XY * sizeof(float), cudaMemcpyDeviceToDevice, s));
}

KGB_API int kgb_forward(kgb_handle* h, int n, const float* spatial, const float* global, const int32_t* symmetry, const float* policy_optimism,
                float* policy, float* value, float* score_value, float* ownership) {
  return guarded([&] {
    checkForwardArgs(h, n, spatial, global, policy, value, score_value);
    checkMetaArgs(h, nullptr, "kgb_forward");
    forwardHost(h, n, spatial, global, nullptr, symmetry, policy_optimism, policy, value, score_value, ownership);
  });
}

KGB_API int kgb_forward_meta(kgb_handle* h, int n, const float* spatial, const float* global, const float* meta, const int32_t* symmetry,
                             const float* policy_optimism, float* policy, float* value, float* score_value, float* ownership) {
  return guarded([&] {
    checkForwardArgs(h, n, spatial, global, policy, value, score_value);
    checkMetaArgs(h, meta, "kgb_forward_meta");
    forwardHost(h, n, spatial, global, meta, symmetry, policy_optimism, policy, value, score_value, ownership);
  });
}

KGB_API int kgb_forward_device(kgb_handle* h, int n, const float* d_spatial, const float* d_global, const int32_t* d_symmetry,
                       const float* d_policy_optimism, float* d_policy, float* d_value, float* d_score_value, float* d_ownership) {
  return guarded([&] {
    checkForwardArgs(h, n, d_spatial, d_global, d_policy, d_value, d_score_value);
    checkMetaArgs(h, nullptr, "kgb_forward_device");
    forwardDevice(h, n, d_spatial, d_global, nullptr, d_symmetry, d_policy_optimism, d_policy, d_value, d_score_value, d_ownership);
  });
}

KGB_API int kgb_test_forward_serial(kgb_handle* h, int n, const float* d_spatial, const float* d_global, const int32_t* d_symmetry,
                                    const float* d_policy_optimism, float* d_policy, float* d_value, float* d_score_value, float* d_ownership) {
  return guarded([&] {
    checkForwardArgs(h, n, d_spatial, d_global, d_policy, d_value, d_score_value);
    checkMetaArgs(h, nullptr, "kgb_test_forward_serial");
    forwardDevice(h, n, d_spatial, d_global, nullptr, d_symmetry, d_policy_optimism, d_policy, d_value, d_score_value, d_ownership, true);
    CK(cudaStreamSynchronize(h->stream));
  });
}

KGB_API int kgb_conv_chain_error(int* out) {
  return guarded([&] {
    if(!out) throw std::invalid_argument("kgb_conv_chain_error: NULL argument");
    *out = convChainStatus() == cudaSuccess ? 0 : 1;
  });
}

KGB_API int kgb_forward_device_meta(kgb_handle* h, int n, const float* d_spatial, const float* d_global, const float* d_meta,
                                    const int32_t* d_symmetry, const float* d_policy_optimism, float* d_policy, float* d_value,
                                    float* d_score_value, float* d_ownership) {
  return guarded([&] {
    checkForwardArgs(h, n, d_spatial, d_global, d_policy, d_value, d_score_value);
    checkMetaArgs(h, d_meta, "kgb_forward_device_meta");
    forwardDevice(h, n, d_spatial, d_global, d_meta, d_symmetry, d_policy_optimism, d_policy, d_value, d_score_value, d_ownership);
  });
}

}  // extern "C" (part 1)

// Stand-alone single convolution (testEvaluateConv / kernel-level roofline timing).
namespace {
// The frame layout as a fixed plan for h.maxBatch images: image i at row i*P, no gap rows (the single-layer hooks lay out and
// mask their rows on the host).
void uploadFramePlan(kgb_handle& h) {
  const int n = h.maxBatch, P = h.L.P;
  h.fixedPlan = true;
  const size_t M = h.planRows(n), tiles = (M + 127) / 128;
  std::vector<int4> box(n, make_int4(0, 0, h.L.X, h.L.Y));
  std::vector<int> base(n), tileWp(tiles, h.L.Wp), rowImg(M), stats = {(int)M, (int)tiles, 1};
  for(int i = 0; i < n; i++) base[i] = i * P;
  for(size_t r = 0; r < M; r++) rowImg[r] = (int)(r / P);
  h.plan.box = h.dalloc<int4>(n);
  h.plan.base = h.dalloc<int>(n);
  h.plan.tileWp = h.dalloc<int>(tiles);
  h.plan.rowImg = h.dalloc<int>(M);
  h.plan.stats = h.dalloc<int>(3);
  CK(cudaMemcpyAsync(h.plan.box, box.data(), n * sizeof(int4), cudaMemcpyHostToDevice, h.stream));
  CK(cudaMemcpyAsync(h.plan.base, base.data(), n * sizeof(int), cudaMemcpyHostToDevice, h.stream));
  CK(cudaMemcpyAsync(h.plan.tileWp, tileWp.data(), tiles * sizeof(int), cudaMemcpyHostToDevice, h.stream));
  CK(cudaMemcpyAsync(h.plan.rowImg, rowImg.data(), M * sizeof(int), cudaMemcpyHostToDevice, h.stream));
  CK(cudaMemcpyAsync(h.plan.stats, stats.data(), 3 * sizeof(int), cudaMemcpyHostToDevice, h.stream));
  CK(cudaStreamSynchronize(h.stream));
}

// Plan mode of the test hooks: the row plan the evaluator makes at the start of a forward, for boards given by size.
// The plan's buffers for h.maxBatch images, sized as Builder::build sizes them.
void allocPlan(kgb_handle& h) {
  const size_t Mmax = h.planRows(h.maxBatch);
  h.dMask = h.dalloc<float>(Mmax + 128);
  h.dMaskSum = h.dalloc<float>(h.maxBatch);
  h.plan.box = h.dalloc<int4>(h.maxBatch);
  h.plan.base = h.dalloc<int>(h.maxBatch);
  h.plan.tileWp = h.dalloc<int>(Mmax / 128);
  h.plan.rowImg = h.dalloc<int>(Mmax);
  h.plan.stats = h.dalloc<int>(3);
  h.dSymmetry = h.dalloc<int>(h.maxBatch);
}

// A plan as the device holds it after launchPlanRows + launchPackInput.
struct HostPlan {
  std::vector<int4> box;
  std::vector<int> base;
  std::vector<float> mask;   // [M]
  int stats[3] = {0, 0, 0};
  // row of frame position (y, x) of image i, or -1 outside its box (planRow)
  long row(const Layout& L, int i, int y, int x) const {
    const int4 b = box[i];
    const int yy = y - b.y, xx = x - b.x;
    if(yy < 0 || xx < 0 || yy >= b.w || xx >= b.z) return -1;
    return (long)base[i] + (long)(yy + L.pad) * (b.z + L.pad) + xx;
  }
  void copyOut(int n, int64_t* statsOut, int32_t* planOut) const {
    if(statsOut) for(int k = 0; k < 3; k++) statsOut[k] = stats[k];
    if(planOut)
      for(int i = 0; i < n; i++) {
        const int4 b = box[i];
        const int32_t v[5] = {b.x, b.y, b.z, b.w, base[i]};
        memcpy(planOut + 5 * i, v, sizeof(v));
      }
  }
};

void checkBoards(const char* fn, int n, int X, int Y, const int32_t* board_xy, const int32_t* symmetry, bool allowEmpty) {
  for(int i = 0; board_xy && i < n; i++) {
    const int bx = board_xy[2 * i], by = board_xy[2 * i + 1];
    if(!(allowEmpty && bx == 0 && by == 0) && (bx < 1 || bx > X || by < 1 || by > Y))
      throw std::invalid_argument(std::string(fn) + ": board size of image " + std::to_string(i) + " not in the frame");
  }
  for(int i = 0; symmetry && i < n; i++)
    if(symmetry[i] < 0 || symmetry[i] > 7) throw std::invalid_argument(std::string(fn) + ": symmetry must be in 0..7");
}

// Step 1: the mask of image i is 1 on the top-left board_xy[i] of the frame (0 x 0: an empty mask), as fillRowV7 places boards,
// before symmetry[i]; launchPlanRows plans the rows from it (h.plan.ragged chooses the plan).  Returns the mask input (NHWC, 1 channel).
float* planBoards(kgb_handle& h, int n, const int32_t* board_xy, const int32_t* symmetry) {
  const Layout& L = h.L;
  std::vector<float> m((size_t)n * L.X * L.Y, 0.0f);
  std::vector<int> sym(n, 0);
  for(int i = 0; i < n; i++) {
    const int bx = board_xy ? board_xy[2 * i] : L.X, by = board_xy ? board_xy[2 * i + 1] : L.Y;
    for(int y = 0; y < by; y++)
      for(int x = 0; x < bx; x++) m[((size_t)i * L.Y + y) * L.X + x] = 1.0f;
    if(symmetry) sym[i] = symmetry[i];
  }
  float* dm = h.dalloc<float>(m.size());
  CK(cudaMemcpyAsync(dm, m.data(), m.size() * sizeof(float), cudaMemcpyHostToDevice, h.stream));
  CK(cudaMemcpyAsync(h.dSymmetry, sym.data(), n * sizeof(int), cudaMemcpyHostToDevice, h.stream));
  CK(launchPlanRows(dm, n, 1, true, h.dSymmetry, L, h.plan, h.stream));
  return dm;
}

// Step 2 (after the caller packed its own features, which sets the mask from their channel 0): the mask packed as the mask,
// with its sums and the row -> image table, and the plan read back.
HostPlan readPlan(kgb_handle& h, int n);
HostPlan finishPlan(kgb_handle& h, int n, const float* dMaskIn) {
  const size_t M = h.planRows(n);
  __half* scratch = h.dalloc<__half>(M * 64);
  CK(launchPackInput(dMaskIn, n, 1, true, h.dSymmetry, h.L, h.plan, M, scratch, 64, 0, h.dMask, h.dMaskSum, h.stream));
  return readPlan(h, n);
}
HostPlan readPlan(kgb_handle& h, int n) {
  const size_t M = h.planRows(n);
  HostPlan hp;
  hp.box.resize(n); hp.base.resize(n); hp.mask.resize(M);
  CK(cudaMemcpyAsync(hp.box.data(), h.plan.box, n * sizeof(int4), cudaMemcpyDeviceToHost, h.stream));
  CK(cudaMemcpyAsync(hp.base.data(), h.plan.base, n * sizeof(int), cudaMemcpyDeviceToHost, h.stream));
  CK(cudaMemcpyAsync(hp.mask.data(), h.dMask, M * sizeof(float), cudaMemcpyDeviceToHost, h.stream));
  CK(cudaMemcpyAsync(hp.stats, h.plan.stats, sizeof(hp.stats), cudaMemcpyDeviceToHost, h.stream));
  CK(cudaStreamSynchronize(h.stream));
  if(hp.stats[0] < 0 || (size_t)hp.stats[0] > M || hp.stats[0] % 128 != 0 || hp.stats[1] * 128 != hp.stats[0])
    throw std::runtime_error("the plan's rows " + std::to_string(hp.stats[0]) + " do not fit its buffers of " + std::to_string(M) + " rows");
  return hp;
}

// Rows at or past the plan's end are filled with all-ones bytes (a NaN in fp16 and fp32) before a launch; no launch may write them.
void poisonTail(kgb_handle& h, void* buf, size_t rowBytes, size_t fromRow, size_t M) {
  if(buf && fromRow < M) CK(cudaMemsetAsync((uint8_t*)buf + fromRow * rowBytes, 0xFF, (M - fromRow) * rowBytes, h.stream));
}
size_t countTouchedTail(const std::vector<uint8_t>& v, size_t rowBytes, size_t fromRow) {
  size_t k = 0;
  for(size_t b = fromRow * rowBytes; b < v.size(); b++) k += v[b] != 0xFF;
  return k;
}

// The kernel the last convolution test hook launched (kgb_test_last_conv_kernel), as convEpilogueWG and convPairEpilogueWG chose
// it; -1 until a hook has run, and after one that failed before its launch
enum { TEST_KERNEL_WG = 0, TEST_KERNEL_WG_EPI = 1, TEST_KERNEL_PAIR = 2, TEST_KERNEL_PAIR_EPI = 3 };
int g_lastConvKernel = -1;

struct SingleConv {
  kgb_handle h;
  ModelDesc dummy;
  ConvWeights cw;
  int n, X, Y, cin, cout;
  size_t M;
  // one entry per buffer set: the operand, the activated output (kinds 1-4) and the raw output (kind 0) or raw stream (kinds 2-4)
  std::vector<__half*> As, acts;
  std::vector<void*> raws;
  float* ncbias = nullptr;   // [n][cout_p], the initial conv's per-image bias, when asked for
  std::vector<float> mask;   // [M], as setInput uploaded it
  bool rawF32 = true;   // the raw output of kind 0 is fp32; the stream of kinds 2-6 is fp32 for kinds 4 and 6 and in fp32-equivalent mode
  int rotate, next = 0;
  // kind: 0 = fp32 raw output only; 1 = the first conv of a residual unit (BN + mish + mask -> fp16 operand of the next conv);
  // 2 = the second conv of a unit (+ fp16 residual stream, updated in place, and the next unit's BN + mish operand); 3 = a nested
  // block's pre conv (fp16 raw stream + activated operand); 4 = kind 2 with an fp32 residual stream, as the trunk runs in fp16 mode
  // with KGB_STREAM_FP32=trunk; 5 and 6 = kinds 2 and 4 without the raw output (the residual is read, the stream is not written),
  // as the last block of a level runs.  In fp32-equivalent mode every stream is fp32.  `rotate` independent buffer sets are cycled
  // through by run() so that a timing loop does not live in L2.
  SingleConv(int ky, int kx, int in_c, int out_c, const float* weights, int n_, int X_, int Y_, int use_fp16, int kind, int rotate_ = 1,
             const float* bnScale = nullptr, const float* bnBias = nullptr, int actKind = ACT_MISH, bool withNcbias = false,
             int ragged = -1)
      : n(n_), X(X_), Y(Y_), cin(in_c), cout(out_c), rotate(rotate_ < 1 ? 1 : rotate_) {
    h.device = selectDevice(-1);
    h.model = &dummy;
    h.maxBatch = n;
    h.split = use_fp16 ? 0 : 1;
    h.epilogueWG = epilogueWGFromEnv();
    h.L = boardLayout(X, Y, std::max(1, std::max(ky / 2, kx / 2)));
    h.streamTrunkFp32 = h.streamInnerFp32 = h.split != 0;
    CK(cudaStreamCreateWithFlags(&h.stream, cudaStreamNonBlocking));
    CK(convWGInit());
    // ragged < 0: the fixed frame layout, masked on the host (setInput); else plan mode (setInputPlanned)
    if(ragged < 0) uploadFramePlan(h);
    else {
      h.plan.ragged = ragged;
      allocPlan(h);
    }
    ConvDesc cd;
    cd.ky = ky; cd.kx = kx; cd.cin = in_c; cd.cout = out_c;
    cd.w.assign(weights, weights + (size_t)ky * kx * in_c * out_c);
    BNDesc bn;
    bn.c = out_c; bn.scale.assign(out_c, 1.0f); bn.bias.assign(out_c, 0.0f);
    if(bnScale) bn.scale.assign(bnScale, bnScale + out_c);
    if(bnBias) bn.bias.assign(bnBias, bnBias + out_c);
    Builder::BNDev dev;
    buildWeights(h, [&](kgb_handle& hh) {
      Builder b(hh);
      cw = b.packConv({&cd});
      dev = b.uploadBN(bn, actKind, cw.cout_p);
    });
    Builder b(h);
    M = h.planRows(n);
    if(ragged < 0) {
      h.dMask = h.dalloc<float>(M + 128);
      h.dMaskSum = h.dalloc<float>(n);
    }
    rawF32 = kind == 0 || kind == 4 || kind == 6 || h.split != 0;
    const bool residual = kind == 2 || kind == 4 || kind == 5 || kind == 6, rawOut = kind != 1 && kind != 5 && kind != 6;
    if(withNcbias) ncbias = h.dalloc<float>((size_t)n * cw.cout_p);
    for(int r = 0; r < rotate; r++) {
      __half* A = h.dalloc<__half>(M * cw.cin_p * b.actMul);
      __half* act = kind == 0 ? nullptr : h.dalloc<__half>(M * cw.cout_p * b.actMul);
      void* raw = kind == 1 ? nullptr : rawF32 ? (void*)h.dalloc<float>(M * cw.cout_p) : (void*)h.dalloc<__half>(M * cw.cout_p);
      As.push_back(A);
      if(act) acts.push_back(act);
      if(raw) raws.push_back(raw);
      b.emitConv(cw, A, residual ? raw : nullptr, rawF32, ncbias, rawOut ? raw : nullptr, rawF32, act, kind == 0 ? Builder::BNDev() : dev);
    }
    h.allocChain();
  }
  ~SingleConv() {
    for(void* p : h.allocs) cudaFree(p);
    if(h.wHost) cudaFreeHost(h.wHost);
    if(h.stream) cudaStreamDestroy(h.stream);
  }
  // boardXY [n][2] (or null = the whole frame): image i's board is its top-left X_i x Y_i, as the self-play loop places boards
  void setInput(const float* input /* NHWC */, const int32_t* boardXY = nullptr) {
    float* dIn = h.dalloc<float>((size_t)n * X * Y * cin);
    CK(cudaMemcpyAsync(dIn, input, (size_t)n * X * Y * cin * sizeof(float), cudaMemcpyHostToDevice, h.stream));
    CK(launchPackInput(dIn, n, cin, true, nullptr, h.L, h.plan, M, As[0], cw.cin_p, h.split, h.dMask, h.dMaskSum, h.stream));
    for(size_t r = 1; r < As.size(); r++)
      CK(cudaMemcpyAsync(As[r], As[0], M * cw.cin_p * (h.split ? 2 : 1) * sizeof(__half), cudaMemcpyDeviceToDevice, h.stream));
    // the mask of a bare convolution is "every point of the image's board", not input channel 0
    std::vector<float> hm(M, 0.0f);
    for(int i = 0; i < n; i++) {
      const int bx = boardXY ? boardXY[2 * i] : X, by = boardXY ? boardXY[2 * i + 1] : Y;
      for(int y = 0; y < by; y++)
        for(int x = 0; x < bx; x++) hm[(size_t)i * h.L.P + (size_t)(y + h.L.pad) * h.L.Wp + x] = 1.0f;
    }
    mask = hm;
    CK(cudaMemcpyAsync(h.dMask, hm.data(), M * sizeof(float), cudaMemcpyHostToDevice, h.stream));
  }
  // Plan mode: the real launchPlanRows and launchPackInput for boards board_xy moved by `symmetry`.  The input is given before
  // the symmetry and must be zero off the board, as fillRowV7 leaves it.  Rows of the operand at or past the plan's end hold
  // finite garbage (fp16 1024), as an earlier, larger forward can leave them: a board row whose tap reached them would be wrong.
  HostPlan setInputPlanned(const float* input /* NHWC */, const int32_t* boardXY, const int32_t* symmetry) {
    float* dIn = h.dalloc<float>((size_t)n * X * Y * cin);
    CK(cudaMemcpyAsync(dIn, input, (size_t)n * X * Y * cin * sizeof(float), cudaMemcpyHostToDevice, h.stream));
    const float* dMaskIn = planBoards(h, n, boardXY, symmetry);
    CK(launchPackInput(dIn, n, cin, true, h.dSymmetry, h.L, h.plan, M, As[0], cw.cin_p, h.split, h.dMask, h.dMaskSum, h.stream));
    HostPlan hp = finishPlan(h, n, dMaskIn);
    const size_t ld = (size_t)cw.cin_p * (h.split ? 2 : 1);
    const std::vector<__half> tail((M - hp.stats[0]) * ld, __float2half(1024.0f));
    if(!tail.empty()) CK(cudaMemcpyAsync(As[0] + hp.stats[0] * ld, tail.data(), tail.size() * sizeof(__half), cudaMemcpyHostToDevice, h.stream));
    mask = hp.mask;
    return hp;
  }
  void run() { h.ops[next](n, h.stream); next = (next + 1) % rotate; }
};

// The seeded boundary's host arrays, from one generator: the exit's and the entry's weights, the trunk's and the inner BN
// constants, then (BoundaryConv::seedInputs) the inputs of every board row in row order
struct BoundarySeed {
  uint32_t st;
  explicit BoundarySeed(uint32_t seed) : st(seed * 2654435761u + 12345u) {}
  float uni() { st = st * 1664525u + 1013904223u; return (st >> 8) * (1.0f / 16777216.0f); }
  ConvDesc conv(int cin, int cout) {
    ConvDesc c;
    c.ky = c.kx = 1; c.cin = cin; c.cout = cout;
    c.w.resize((size_t)cin * cout);
    for(auto& v : c.w) v = (uni() - 0.5f) * 4.0f / std::sqrt((float)cin);
    return c;
  }
  BNDesc bn(int c) {
    BNDesc b;
    b.c = c;
    for(int i = 0; i < c; i++) { b.scale.push_back(0.5f + uni()); b.bias.push_back(uni() - 0.5f); }
    return b;
  }
};

// A nested-block boundary on its own: the exit 1x1 `post` (inner_c -> trunk_c, + the trunk stream, then the trunk BN and mish) of
// one block and the entry 1x1 `pre` (trunk_c -> inner_c, then the inner BN and mish) of the next.  Buffer set 2r runs it as one fused
// launch (launchConvPair), set 2r + 1 as the two launches of the unfused path, on the same inputs (setInputs); `rotate` pairs of sets
// are cycled through by run() so that a timing loop does not live in L2.
struct BoundaryConv {
  kgb_handle h;
  ModelDesc dummy;
  ConvWeights wpost, wpre;
  int n, innerC, trunkC, innerCp = 0, trunkCp = 0, rotate, next = 0;
  int fusedKernel = TEST_KERNEL_PAIR;   // the kernel of the fused op, as emitConvPair counted convPairEpilogueWG's choice
  bool trunkF32, innerF32, planned;
  size_t M;
  struct Set {
    __half *innerA = nullptr, *trunkA = nullptr;
    void *trunkS = nullptr, *innerS = nullptr;
  };
  std::vector<Set> sets;
  std::vector<float> mask;
  HostPlan hp;   // plan mode: the plan; every buffer's rows from hp.stats[0] on hold all-ones bytes before the launches
  // ragged < 0: the fixed frame layout; else plan mode, boards moved by `symmetry` (planBoards)
  BoundaryConv(int inner_c, int trunk_c, int n_, int X, int Y, const int32_t* boardXY, bool trunkFp32, bool innerFp32, const ConvDesc& post,
               const ConvDesc& pre, const BNDesc& bnTrunk, const BNDesc& bnInner, int rotate_, const int32_t* symmetry = nullptr, int ragged = -1)
      : n(n_), innerC(inner_c), trunkC(trunk_c), rotate(rotate_ < 1 ? 1 : rotate_), trunkF32(trunkFp32), innerF32(innerFp32),
        planned(ragged >= 0) {
    h.device = selectDevice(-1);
    h.model = &dummy;
    h.maxBatch = n;
    h.pairEpilogueWG = pairEpilogueWGFromEnv();
    h.L = boardLayout(X, Y, 1);
    CK(cudaStreamCreateWithFlags(&h.stream, cudaStreamNonBlocking));
    CK(convWGInit());
    if(ragged < 0) uploadFramePlan(h);
    else {
      h.plan.ragged = ragged;
      allocPlan(h);
      hp = finishPlan(h, n, planBoards(h, n, boardXY, symmetry));
    }
    Builder::BNDev bn1, bn2;
    buildWeights(h, [&](kgb_handle& hh) {
      Builder b(hh);
      wpost = b.packConv({&post});
      wpre = b.packConv({&pre});
      bn1 = b.uploadBN(bnTrunk, ACT_MISH, wpost.cout_p);
      bn2 = b.uploadBN(bnInner, ACT_MISH, wpre.cout_p);
    });
    innerCp = wpost.cin_p; trunkCp = wpost.cout_p;
    M = h.planRows(n);
    if(ragged < 0) {
      h.dMask = h.dalloc<float>(M + 128);
      mask.assign(M, 0.0f);
      for(int i = 0; i < n; i++) {
        const int bx = boardXY ? boardXY[2 * i] : X, by = boardXY ? boardXY[2 * i + 1] : Y;
        for(int y = 0; y < by; y++)
          for(int x = 0; x < bx; x++) mask[(size_t)i * h.L.P + (size_t)(y + h.L.pad) * h.L.Wp + x] = 1.0f;
      }
      CK(cudaMemcpyAsync(h.dMask, mask.data(), M * sizeof(float), cudaMemcpyHostToDevice, h.stream));
    }
    else mask = hp.mask;
    Builder b(h);
    for(int k = 0; k < 2 * rotate; k++) {
      Set s;
      s.innerA = h.dalloc<__half>(M * innerCp);
      s.trunkA = h.dalloc<__half>(M * trunkCp);
      s.trunkS = trunkF32 ? (void*)h.dalloc<float>(M * trunkCp) : (void*)h.dalloc<__half>(M * trunkCp);
      s.innerS = innerF32 ? (void*)h.dalloc<float>(M * innerCp) : (void*)h.dalloc<__half>(M * innerCp);
      sets.push_back(s);
      if(k % 2 == 0) {
        if(!b.emitConvPair(wpost, s.innerA, s.trunkS, trunkF32, bn1, wpre, s.innerS, innerF32, s.innerA, bn2))
          throw std::invalid_argument("the fused boundary kernel does not take " + std::to_string(inner_c) + " / " + std::to_string(trunk_c) +
                                      " channels with these streams");
      }
      else {
        // one op per launch, as emitBlocks emits an unfused boundary
        b.emitConv(wpost, s.innerA, s.trunkS, trunkF32, nullptr, s.trunkS, trunkF32, s.trunkA, bn1);
        b.emitConv(wpre, s.trunkA, nullptr, false, nullptr, s.innerS, innerF32, s.innerA, bn2);
      }
    }
    fusedKernel = h.pairEpilogueWGLaunches > 0 ? TEST_KERNEL_PAIR_EPI : TEST_KERNEL_PAIR;
    h.allocChain();
    CK(cudaStreamSynchronize(h.stream));
  }
  ~BoundaryConv() {
    for(void* p : h.allocs) cudaFree(p);
    if(h.wHost) cudaFreeHost(h.wHost);
    if(h.stream) cudaStreamDestroy(h.stream);
  }
  // The inputs of every set, as the previous layers leave them: the inner operand hA [M][innerCp] and the trunk stream hS
  // [M][trunkCp], zero in masked rows and padded channels
  void setInputs(const std::vector<__half>& hA, const std::vector<float>& hS) {
    std::vector<__half> hS16(hS.size());
    for(size_t k = 0; k < hS.size(); k++) hS16[k] = __float2half_rn(hS[k]);
    for(const Set& s : sets) {
      CK(cudaMemcpyAsync(s.innerA, hA.data(), hA.size() * sizeof(__half), cudaMemcpyHostToDevice, h.stream));
      if(trunkF32) CK(cudaMemcpyAsync(s.trunkS, hS.data(), hS.size() * sizeof(float), cudaMemcpyHostToDevice, h.stream));
      else CK(cudaMemcpyAsync(s.trunkS, hS16.data(), hS16.size() * sizeof(__half), cudaMemcpyHostToDevice, h.stream));
      if(planned) {   // 1x1 convolutions: no tap reaches past a tile's own rows, so every buffer can hold NaN there
        poisonTail(h, s.innerA, (size_t)innerCp * 2, hp.stats[0], M);
        poisonTail(h, s.trunkA, (size_t)trunkCp * 2, hp.stats[0], M);
        poisonTail(h, s.trunkS, (size_t)trunkCp * (trunkF32 ? 4 : 2), hp.stats[0], M);
        poisonTail(h, s.innerS, (size_t)innerCp * (innerF32 ? 4 : 2), hp.stats[0], M);
      }
    }
    CK(cudaStreamSynchronize(h.stream));
  }
  void seedInputs(BoundarySeed& g) {
    std::vector<__half> hA(M * innerCp, __float2half(0.0f));
    std::vector<float> hS(M * trunkCp, 0.0f);
    for(size_t r = 0; r < M; r++) {
      if(mask[r] == 0.0f) continue;
      for(int c = 0; c < innerC; c++) hA[r * innerCp + c] = __float2half_rn(g.uni() * 2.0f);
      for(int c = 0; c < trunkC; c++) hS[r * trunkCp + c] = (g.uni() - 0.5f) * 8.0f;
    }
    setInputs(hA, hS);
  }
  // ops: set 2r's fused op is op 3r, set 2r + 1's two launches ops 3r + 1 and 3r + 2
  void run(bool fused) {
    if(fused) h.ops[3 * next](n, h.stream);
    else { h.ops[3 * next + 1](n, h.stream); h.ops[3 * next + 2](n, h.stream); }
    next = (next + 1) % rotate;
  }
};

// kgb_test_conv_ex and its two narrower forms kgb_test_conv (kind 0) and kgb_test_conv_epilogue (kinds 1-4): one launch, NHWC in
// and out.  act_lo_out is written in split mode only.
//
// ragged >= 0 is plan mode (kgb_test_conv_plan): the plan is made on the device for boards board_xy moved by `symmetry`, every input
// but `input` and every output is in the coordinates after the symmetry, and rows at or past the plan's end must come back as the
// all-ones bytes they were filled with.  stats_out [3] and plan_out [n][5] (x0, y0, w, h, first row) report the plan.
void testConv(const char* fn, int ky, int kx, int in_c, int out_c, const float* weights, int n, int nn_x_len, int nn_y_len, int use_fp16, int kind,
              const float* input, const int32_t* board_xy, const float* ncbias, const float* residual_in, const float* bn_scale,
              const float* bn_bias, int activation, float* raw_out, float* act_hi_out, float* act_lo_out, const int32_t* symmetry = nullptr,
              int ragged = -1, int64_t* stats_out = nullptr, int32_t* plan_out = nullptr) {
  const bool hasResidual = kind == 2 || kind == 4 || kind == 5 || kind == 6;
  const bool hasRaw = kind == 0 || (kind >= 2 && kind <= 4);
  const bool planned = ragged >= 0;
  g_lastConvKernel = -1;
  if(!weights || !input || n < 1 || kind < 0 || kind > 6 || activation < ACT_IDENTITY || activation > ACT_SILU ||
     (kind == 0 ? !raw_out : !act_hi_out))
    throw std::invalid_argument(std::string(fn) + ": bad argument");
  if(hasResidual && !residual_in) throw std::invalid_argument(std::string(fn) + ": kinds 2, 4, 5 and 6 need residual_in");
  if(kind >= 2 && kind <= 4 && !raw_out) throw std::invalid_argument(std::string(fn) + ": kinds 2 to 4 need raw_out");
  checkBoards(fn, n, nn_x_len, nn_y_len, board_xy, symmetry, planned);
  SingleConv sc(ky, kx, in_c, out_c, weights, n, nn_x_len, nn_y_len, use_fp16, kind, 1, bn_scale, bn_bias, activation, ncbias != nullptr,
                planned ? (ragged != 0) : -1);
  // emitConv counted convEpilogueWG's choice for the op, as launchConvWG makes it
  const int kernel = sc.h.epilogueWGLaunches > 0 ? TEST_KERNEL_WG_EPI : TEST_KERNEL_WG;
  HostPlan hp;
  if(planned) {
    hp = sc.setInputPlanned(input, board_xy, symmetry);
    hp.copyOut(n, stats_out, plan_out);
  }
  else sc.setInput(input, board_xy);
  const size_t used = planned ? (size_t)hp.stats[0] : sc.M;   // rows the launch may write
  const int cp = sc.cw.cout_p;
  const bool f32 = sc.rawF32;
  const bool split = sc.h.split != 0;
  const cudaStream_t s = sc.h.stream;
  if(split && kind != 0 && !act_lo_out) throw std::invalid_argument(std::string(fn) + ": split mode needs act_lo_out");
  auto rowOf = [&](int i, int y, int x) -> long {
    return planned ? hp.row(sc.h.L, i, y, x) : (long)((size_t)i * sc.h.L.P + (size_t)(y + sc.h.L.pad) * sc.h.L.Wp + x);
  };
  if(ncbias) {
    std::vector<float> hb((size_t)n * cp, 0.0f);
    for(int i = 0; i < n; i++) for(int c = 0; c < out_c; c++) hb[(size_t)i * cp + c] = ncbias[(size_t)i * out_c + c];
    CK(cudaMemcpyAsync(sc.ncbias, hb.data(), hb.size() * sizeof(float), cudaMemcpyHostToDevice, s));
  }
  const int am = split ? 2 : 1;
  const size_t rawRowBytes = (size_t)cp * (f32 ? 4 : 2), actRowBytes = (size_t)cp * am * 2;
  std::vector<uint8_t> streamIn;   // the stream's bytes as uploaded
  if(hasResidual) {
    // given as fp32; an fp16 stream holds it rounded to nearest
    std::vector<float> hf(sc.M * cp, 0.0f);
    for(int i = 0; i < n; i++) for(int y = 0; y < nn_y_len; y++) for(int x = 0; x < nn_x_len; x++) {
      const long row = rowOf(i, y, x);
      if(row < 0) continue;
      for(int c = 0; c < out_c; c++) hf[row * cp + c] = residual_in[(((size_t)i * nn_y_len + y) * nn_x_len + x) * out_c + c];
    }
    streamIn.resize(sc.M * rawRowBytes);
    if(f32) memcpy(streamIn.data(), hf.data(), streamIn.size());
    else
      for(size_t k = 0; k < hf.size(); k++) {
        const __half v = __float2half_rn(hf[k]);
        memcpy(&streamIn[2 * k], &v, 2);
      }
    CK(cudaMemcpyAsync(sc.raws[0], streamIn.data(), streamIn.size(), cudaMemcpyHostToDevice, s));
  }
  if(planned) {
    if(!sc.raws.empty()) poisonTail(sc.h, sc.raws[0], rawRowBytes, used, sc.M);
    if(!sc.acts.empty()) poisonTail(sc.h, sc.acts[0], actRowBytes, used, sc.M);
  }
  sc.run();
  g_lastConvKernel = kernel;
  auto download = [&](void* dst, const void* src, size_t bytes) {
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  };
  std::vector<__half> ha;
  if(!sc.acts.empty()) {
    ha.resize(sc.M * cp * am);
    download(ha.data(), sc.acts[0], ha.size() * sizeof(__half));
  }
  if(hasResidual && !hasRaw) {
    // kinds 5 and 6 read the stream and must leave it as it was (rows past the plan's end are checked below with the others)
    std::vector<uint8_t> v(streamIn.size());
    download(v.data(), sc.raws[0], v.size());
    if(memcmp(v.data(), streamIn.data(), used * rawRowBytes) != 0) throw std::runtime_error(std::string(fn) + ": the residual stream was written");
    if(planned) {
      if(const size_t k = countTouchedTail(v, rawRowBytes, used))
        throw std::runtime_error(std::string(fn) + ": the residual stream was written past the plan's end (" + std::to_string(k) + " bytes)");
    }
  }
  std::vector<float> hr;
  if(hasRaw) {
    hr.resize(sc.M * cp);
    if(f32) download(hr.data(), sc.raws[0], hr.size() * sizeof(float));
    else {
      std::vector<__half> hh(hr.size());
      download(hh.data(), sc.raws[0], hh.size() * sizeof(__half));
      for(size_t k = 0; k < hr.size(); k++) hr[k] = __half2float(hh[k]);
    }
  }
  if(planned) {
    // the rows past the plan: the bytes they were filled with (no tile writes there)
    auto tail = [&](const char* what, const void* p, size_t rowBytes) {
      std::vector<uint8_t> v(sc.M * rowBytes);
      memcpy(v.data(), p, v.size());
      if(const size_t k = countTouchedTail(v, rowBytes, used))
        throw std::runtime_error(std::string(fn) + ": " + what + " was written past the plan's " + std::to_string(used) + " rows (" +
                                 std::to_string(k) + " bytes)");
    };
    if(hasRaw && f32) tail("the raw output", hr.data(), rawRowBytes);
    if(hasRaw && !f32) {
      std::vector<__half> hh(sc.M * cp);
      download(hh.data(), sc.raws[0], hh.size() * sizeof(__half));
      tail("the raw output", hh.data(), rawRowBytes);
    }
    if(!ha.empty()) tail("the activated operand", ha.data(), actRowBytes);
  }
  // Exact zeros where the next layer relies on them: every column of a row the mask zeroes (pad rows and columns, and points off
  // a smaller board; in plan mode also the gap rows that end a segment and the rows up to the next 128), which the next conv's halo
  // reads as its zero padding; and the padded channels cout..cout_p of every row, which the next conv reads as part of K (0 x NaN is
  // not 0).  The raw output is checked too, and in split mode the lo half.
  auto check = [&](const char* what, int ld, int col0, auto value) {
    for(size_t r = 0; r < used; r++) {
      const bool off = sc.mask[r] == 0.0f;
      for(int c = off ? 0 : out_c; c < cp; c++)
        if(value(r * ld + col0 + c) != 0.0f)
          throw std::runtime_error(std::string(fn) + ": " + what + " is not zero at row " + std::to_string(r) + (off ? " (masked)" : "") +
                                   ", channel " + std::to_string(c));
    }
  };
  if(!hr.empty()) check("the raw output", cp, 0, [&](size_t k) { return hr[k]; });
  if(!ha.empty()) {
    check("the activated operand", cp * am, 0, [&](size_t k) { return __half2float(ha[k]); });
    if(split) check("the activated operand's lo half", cp * am, cp, [&](size_t k) { return __half2float(ha[k]); });
  }
  for(int i = 0; i < n; i++) for(int y = 0; y < nn_y_len; y++) for(int x = 0; x < nn_x_len; x++) for(int c = 0; c < out_c; c++) {
    const long prow = rowOf(i, y, x);
    const size_t row = (size_t)prow, o = (((size_t)i * nn_y_len + y) * nn_x_len + x) * out_c + c;
    if(prow < 0) {   // outside the image's box: a mask-0 position, whose outputs are zero
      if(!ha.empty()) { act_hi_out[o] = 0.0f; if(split) act_lo_out[o] = 0.0f; }
      if(!hr.empty()) raw_out[o] = 0.0f;
      continue;
    }
    if(!ha.empty()) {
      act_hi_out[o] = __half2float(ha[row * cp * am + c]);
      if(split) act_lo_out[o] = __half2float(ha[row * cp * am + cp + c]);
    }
    if(!hr.empty()) raw_out[o] = hr[row * cp + c];
  }
}

// kgb_test_conv_boundary (ragged < 0, the frame layout) and kgb_test_conv_boundary_plan.  out[0..2]: elements of trunk.S, inner.S,
// inner.A whose bits differ between the fused launch and the two launches; out[3..5]: nonzero elements of the fused outputs in masked
// rows or padded channels.  Plan mode, over the rows below the plan's end, and out[6..8]: NaN elements of the fused outputs there;
// out[9..11]: bytes at or past the plan's end that either path changed.
void testBoundary(const char* fn, int inner_c, int trunk_c, int n, int nn_x_len, int nn_y_len, const int32_t* board_xy, const int32_t* symmetry,
                  int ragged, int trunk_fp32, int inner_fp32, uint32_t seed, int64_t* out, int64_t* stats_out) {
  const bool planned = ragged >= 0;
  g_lastConvKernel = -1;
  if(!out || n < 1 || inner_c < 1 || trunk_c < 1 || nn_x_len < 2 || nn_y_len < 2 || (inner_fp32 && !trunk_fp32))
    throw std::invalid_argument(std::string(fn) + ": bad argument");
  checkBoards(fn, n, nn_x_len, nn_y_len, board_xy, symmetry, planned);
  BoundarySeed g(seed);
  const ConvDesc post = g.conv(inner_c, trunk_c), pre = g.conv(trunk_c, inner_c);
  const BNDesc bnTrunk = g.bn(trunk_c), bnInner = g.bn(inner_c);
  BoundaryConv bc(inner_c, trunk_c, n, nn_x_len, nn_y_len, board_xy, trunk_fp32 != 0, inner_fp32 != 0, post, pre, bnTrunk, bnInner, 1, symmetry,
                  planned ? (ragged != 0) : -1);
  bc.seedInputs(g);
  if(planned) bc.hp.copyOut(n, stats_out, nullptr);
  const size_t used = planned ? (size_t)bc.hp.stats[0] : bc.M;
  bc.run(true);
  bc.run(false);
  g_lastConvKernel = bc.fusedKernel;
  const cudaStream_t s = bc.h.stream;
  auto download = [&](const void* src, size_t bytes) {
    std::vector<uint8_t> v(bytes);
    CK(cudaMemcpyAsync(v.data(), src, bytes, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return v;
  };
  struct Out { size_t off; int cp, c, esize; };
  const Out outs[3] = {{offsetof(BoundaryConv::Set, trunkS), bc.trunkCp, trunk_c, trunk_fp32 ? 4 : 2},
                       {offsetof(BoundaryConv::Set, innerS), bc.innerCp, inner_c, inner_fp32 ? 4 : 2},
                       {offsetof(BoundaryConv::Set, innerA), bc.innerCp, inner_c, 2}};
  for(int k = 0; k < 3; k++) {
    const Out& o = outs[k];
    auto ptr = [&](const BoundaryConv::Set& st) { return *reinterpret_cast<void* const*>(reinterpret_cast<const uint8_t*>(&st) + o.off); };
    const size_t bytes = bc.M * o.cp * o.esize;
    const std::vector<uint8_t> f = download(ptr(bc.sets[0]), bytes), u = download(ptr(bc.sets[1]), bytes);
    int64_t diff = 0, nonzero = 0, nan = 0;
    for(size_t r = 0; r < used; r++)
      for(int c = 0; c < o.cp; c++) {
        const size_t e = (r * o.cp + c) * o.esize;
        if(memcmp(&f[e], &u[e], o.esize) != 0) diff++;
        float v;
        if(o.esize == 4) memcpy(&v, &f[e], 4);
        else { __half hv; memcpy(&hv, &f[e], 2); v = __half2float(hv); }
        if(std::isnan(v)) nan++;
        if((bc.mask[r] == 0.0f || c >= o.c) && v != 0.0f) nonzero++;
      }
    out[k] = diff;
    out[3 + k] = nonzero;
    if(planned) {
      out[6 + k] = nan;
      out[9 + k] = (int64_t)(countTouchedTail(f, (size_t)o.cp * o.esize, used) + countTouchedTail(u, (size_t)o.cp * o.esize, used));
    }
  }
}

// kgb_test_conv_boundary_ex: the boundary on the caller's operand, stream, weights and BN constants, one path (fused or the two
// launches).  Inputs and outputs are NHWC in the coordinates after the symmetry; only board positions are read.
void testBoundaryEx(int inner_c, int trunk_c, int n, int nn_x_len, int nn_y_len, const float* inner_a, const float* exit_w, const float* trunk_s,
                    const float* trunk_scale, const float* trunk_bias, const float* entry_w, const float* inner_scale, const float* inner_bias,
                    const int32_t* board_xy, const int32_t* symmetry, int ragged, int trunk_fp32, int inner_fp32, int fused, float* trunk_s_out,
                    float* inner_s_out, float* inner_a_out, int64_t* stats_out) {
  const char* fn = "kgb_test_conv_boundary_ex";
  const bool planned = ragged >= 0;
  g_lastConvKernel = -1;
  if(n < 1 || inner_c < 1 || trunk_c < 1 || nn_x_len < 2 || nn_y_len < 2 || (inner_fp32 && !trunk_fp32) || (symmetry && !planned) ||
     !inner_a || !exit_w || !trunk_s || !trunk_scale || !trunk_bias || !entry_w || !inner_scale || !inner_bias || !trunk_s_out ||
     !inner_s_out || !inner_a_out)
    throw std::invalid_argument(std::string(fn) + ": bad argument");
  checkBoards(fn, n, nn_x_len, nn_y_len, board_xy, symmetry, planned);
  auto conv = [](int cin, int cout, const float* w) {
    ConvDesc c;
    c.ky = c.kx = 1; c.cin = cin; c.cout = cout;
    c.w.assign(w, w + (size_t)cin * cout);
    return c;
  };
  auto bn = [](int c, const float* scale, const float* bias) {
    BNDesc b;
    b.c = c; b.scale.assign(scale, scale + c); b.bias.assign(bias, bias + c);
    return b;
  };
  BoundaryConv bc(inner_c, trunk_c, n, nn_x_len, nn_y_len, board_xy, trunk_fp32 != 0, inner_fp32 != 0, conv(inner_c, trunk_c, exit_w),
                  conv(trunk_c, inner_c, entry_w), bn(trunk_c, trunk_scale, trunk_bias), bn(inner_c, inner_scale, inner_bias), 1, symmetry,
                  planned ? (ragged != 0) : -1);
  if(planned) bc.hp.copyOut(n, stats_out, nullptr);
  const size_t used = planned ? (size_t)bc.hp.stats[0] : bc.M;
  const Layout& L = bc.h.L;
  auto rowOf = [&](int i, int y, int x) -> long {
    const long r = planned ? bc.hp.row(L, i, y, x) : (long)((size_t)i * L.P + (size_t)(y + L.pad) * L.Wp + x);
    return r >= 0 && bc.mask[r] != 0.0f ? r : -1;
  };
  std::vector<__half> hA(bc.M * bc.innerCp, __float2half(0.0f));
  std::vector<float> hS(bc.M * bc.trunkCp, 0.0f);
  for(int i = 0; i < n; i++) for(int y = 0; y < nn_y_len; y++) for(int x = 0; x < nn_x_len; x++) {
    const long r = rowOf(i, y, x);
    if(r < 0) continue;
    const size_t o = ((size_t)i * nn_y_len + y) * nn_x_len + x;
    for(int c = 0; c < inner_c; c++) hA[r * bc.innerCp + c] = __float2half_rn(inner_a[o * inner_c + c]);
    for(int c = 0; c < trunk_c; c++) hS[r * bc.trunkCp + c] = trunk_s[o * trunk_c + c];
  }
  bc.setInputs(hA, hS);
  bc.run(fused != 0);
  g_lastConvKernel = fused ? bc.fusedKernel : bc.h.epilogueWGLaunches > 0 ? TEST_KERNEL_WG_EPI : TEST_KERNEL_WG;
  // the set the path ran on: its outputs, with exact zeros in every row the mask zeroes and every padded channel, and in plan mode
  // nothing written at or past the plan's end
  const BoundaryConv::Set& st = bc.sets[fused ? 0 : 1];
  struct Out { const void* p; int cp, c, esize; float* dst; const char* what; };
  const Out outs[3] = {{st.trunkS, bc.trunkCp, trunk_c, trunk_fp32 ? 4 : 2, trunk_s_out, "the trunk stream"},
                       {st.innerS, bc.innerCp, inner_c, inner_fp32 ? 4 : 2, inner_s_out, "the inner stream"},
                       {st.innerA, bc.innerCp, inner_c, 2, inner_a_out, "the inner operand"}};
  for(const Out& o : outs) {
    std::vector<uint8_t> v(bc.M * o.cp * o.esize);
    CK(cudaMemcpyAsync(v.data(), o.p, v.size(), cudaMemcpyDeviceToHost, bc.h.stream));
    CK(cudaStreamSynchronize(bc.h.stream));
    auto value = [&](size_t e) {
      float f;
      if(o.esize == 4) memcpy(&f, &v[e * 4], 4);
      else { __half hv; memcpy(&hv, &v[e * 2], 2); f = __half2float(hv); }
      return f;
    };
    for(size_t r = 0; r < used; r++) {
      const bool off = bc.mask[r] == 0.0f;
      for(int c = off ? 0 : o.c; c < o.cp; c++)
        if(value(r * o.cp + c) != 0.0f)
          throw std::runtime_error(std::string(fn) + ": " + o.what + " is not zero at row " + std::to_string(r) + (off ? " (masked)" : "") +
                                   ", channel " + std::to_string(c));
    }
    if(planned)
      if(const size_t k = countTouchedTail(v, (size_t)o.cp * o.esize, used))
        throw std::runtime_error(std::string(fn) + ": " + o.what + " was written past the plan's end (" + std::to_string(k) + " bytes)");
    for(int i = 0; i < n; i++) for(int y = 0; y < nn_y_len; y++) for(int x = 0; x < nn_x_len; x++) {
      const long r = rowOf(i, y, x);
      const size_t q = ((size_t)i * nn_y_len + y) * nn_x_len + x;
      for(int c = 0; c < o.c; c++) o.dst[q * o.c + c] = r < 0 ? 0.0f : value(r * o.cp + c);
    }
  }
}

// kgb_test_head_kernel (include/kgb200.h): one launch of one of the evaluator's fp32 kernels on the caller's tensors.
enum { HK_PACK = 0, HK_GPOOL = 1, HK_BIASACT = 2, HK_MATMUL = 3, HK_POLICY = 4, HK_OWNERSHIP = 5, HK_FINALIZE = 6 };

void testHead(int which, int n, int X, int Y, int pad, const int32_t* board_xy, const int32_t* symmetry, int ragged, const int32_t* ip, int nip,
              const float* const* in, int nin, float* const* out, int nout, int64_t* stats_out, int32_t* plan_out) {
  static const int needIp[7] = {3, 6, 4, 5, 5, 4, 4}, needIn[7] = {1, 3, 4, 3, 6, 4, 4}, needOut[7] = {4, 1, 2, 1, 1, 1, 3};
  const char* fn = "kgb_test_head_kernel";
  if(which < 0 || which > 6 || n < 1 || X < 2 || Y < 2 || X > 37 || Y > 37 || pad < 1 || pad > 2 || (ragged != 0 && ragged != 1) || !ip ||
     nip != needIp[which] || !in || nin != needIn[which] || !out || nout != needOut[which])
    throw std::invalid_argument(std::string(fn) + ": bad argument");
  checkBoards(fn, n, X, Y, board_xy, symmetry, true);
  kgb_handle h;
  struct Release {
    kgb_handle& h;
    ~Release() { for(void* p : h.allocs) cudaFree(p); if(h.stream) cudaStreamDestroy(h.stream); }
  } release{h};
  ModelDesc dummy;
  h.device = selectDevice(-1);
  h.model = &dummy;
  h.maxBatch = n;
  h.L = boardLayout(X, Y, pad);
  h.plan.ragged = ragged;
  CK(cudaStreamCreateWithFlags(&h.stream, cudaStreamNonBlocking));
  const cudaStream_t s = h.stream;
  const Layout L = h.L;
  const int XY = X * Y;
  auto up = [&](const float* p, size_t count) -> float* {
    if(!p) return nullptr;
    float* d = h.dalloc<float>(count);
    CK(cudaMemcpyAsync(d, p, count * sizeof(float), cudaMemcpyHostToDevice, s));
    return d;
  };
  auto down = [&](void* dst, const void* src, size_t bytes) {
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  };
  auto poisoned = [&](size_t count) {   // an fp32 output, all-ones bytes (NaN) where the kernel does not write
    float* d = h.dalloc<float>(count);
    CK(cudaMemsetAsync(d, 0xFF, count * sizeof(float), s));
    return d;
  };
  auto need = [&](bool ok) { if(!ok) throw std::invalid_argument(std::string(fn) + ": bad argument for kernel " + std::to_string(which)); };
  auto isOnes = [](const void* p, size_t bytes) {
    for(size_t b = 0; b < bytes; b++) if(((const uint8_t*)p)[b] != 0xFF) return false;
    return true;
  };

  if(which == HK_MATMUL) {
    const int cin = ip[0], cout = ip[1], act = ip[2], ldi = ip[3], ldo = ip[4];
    need(cin >= 1 && cin <= ldi && cin <= 8192 && cout >= 1 && cout <= ldo && act >= ACT_IDENTITY && act <= ACT_SILU && in[0] && in[1]);
    float* o = poisoned((size_t)n * ldo);
    CK(launchMatMulNC(up(in[0], (size_t)n * ldi), ldi, up(in[1], (size_t)cin * cout), up(in[2], cout), n, cin, cout, act, o, ldo, s));
    down(out[0], o, (size_t)n * ldo * sizeof(float));
    return;
  }
  if(which == HK_FINALIZE) {
    const int cp2 = ip[0], numSV = ip[1], version = ip[2], ldp = ip[3];
    need(cp2 >= 1 && cp2 <= ldp && numSV >= (version >= 9 ? 6 : version >= 8 ? 4 : version >= 4 ? 2 : 1) && in[0] && in[2] && in[3] &&
         out[0] && out[1] && out[2]);
    float *pol = poisoned((size_t)n * (XY + 1)), *val = poisoned((size_t)n * 3), *score = poisoned((size_t)n * 6);
    CK(launchFinalize(up(in[0], (size_t)n * ldp), ldp, cp2, up(in[1], n), up(in[2], (size_t)n * 3), up(in[3], (size_t)n * numSV), numSV, version,
                      n, XY + 1, pol, val, score, s));
    down(out[0], pol, (size_t)n * (XY + 1) * sizeof(float));
    down(out[1], val, (size_t)n * 3 * sizeof(float));
    down(out[2], score, (size_t)n * 6 * sizeof(float));
    return;
  }

  allocPlan(h);
  const size_t M = h.planRows(n);
  HostPlan hp;
  if(which == HK_PACK) {
    // the plan from the input itself (its channel 0 is the mask), as a forward plans it
    const int C = ip[0], split = ip[1], nhwc = ip[2];
    need(C >= 1 && C <= 64 && (split == 0 || split == 1) && in[0] && out[0] && out[2] && out[3] && (!split || out[1]));
    const float* sp = up(in[0], (size_t)n * C * XY);
    std::vector<int> sym(n, 0);
    for(int i = 0; symmetry && i < n; i++) sym[i] = symmetry[i];
    CK(cudaMemcpyAsync(h.dSymmetry, sym.data(), n * sizeof(int), cudaMemcpyHostToDevice, s));
    const int cinP = cpad(C), ld = cinP * (split ? 2 : 1);
    __half* act = h.dalloc<__half>(M * ld);
    CK(launchPlanRows(sp, n, C, nhwc != 0, h.dSymmetry, L, h.plan, s));
    CK(launchPackInput(sp, n, C, nhwc != 0, h.dSymmetry, L, h.plan, M, act, cinP, split, h.dMask, h.dMaskSum, s));
    hp = readPlan(h, n);
    std::vector<__half> ha(M * ld);
    down(ha.data(), act, ha.size() * sizeof(__half));
    down(out[2], h.dMaskSum, n * sizeof(float));
    // a row that is not a board position is zero in every channel, and so is every padded channel
    for(size_t r = 0; r < (size_t)hp.stats[0]; r++)
      for(int c = 0; c < ld; c++)
        if((hp.mask[r] == 0.0f || c % cinP >= C) && __half2float(ha[r * ld + c]) != 0.0f)
          throw std::runtime_error(std::string(fn) + ": the packed input is not zero at row " + std::to_string(r) + ", column " + std::to_string(c));
    for(int i = 0; i < n; i++)
      for(int y = 0; y < Y; y++)
        for(int x = 0; x < X; x++) {
          const long row = hp.row(L, i, y, x);
          const size_t o = ((size_t)i * Y + y) * X + x;
          out[3][o] = row < 0 ? 0.0f : hp.mask[row];
          for(int c = 0; c < C; c++) {
            out[0][o * C + c] = row < 0 ? 0.0f : __half2float(ha[row * ld + c]);
            if(split) out[1][o * C + c] = row < 0 ? 0.0f : __half2float(ha[row * ld + cinP + c]);
          }
        }
    hp.copyOut(n, stats_out, plan_out);
    return;
  }
  hp = finishPlan(h, n, planBoards(h, n, board_xy, symmetry));
  hp.copyOut(n, stats_out, plan_out);
  // t [n][Y][X][C] (the coordinates after the symmetry) into rows of ld columns from column c0: every other element, and every row
  // that is not a board position, NaN; the kernels must read neither
  auto placeRows = [&](const float* t, int C, int ld, int c0, bool fp16) -> void* {
    std::vector<float> v(M * ld, NAN);
    for(int i = 0; i < n; i++)
      for(int y = 0; y < Y; y++)
        for(int x = 0; x < X; x++) {
          const long row = hp.row(L, i, y, x);
          if(row < 0 || hp.mask[row] != 1.0f) continue;
          for(int c = 0; c < C; c++) v[row * ld + c0 + c] = t[(((size_t)i * Y + y) * X + x) * C + c];
        }
    if(!fp16) return up(v.data(), v.size());
    std::vector<__half> hv(v.size());
    for(size_t k = 0; k < v.size(); k++) hv[k] = __float2half_rn(v[k]);
    __half* d = h.dalloc<__half>(hv.size());
    CK(cudaMemcpyAsync(d, hv.data(), hv.size() * sizeof(__half), cudaMemcpyHostToDevice, s));
    return d;
  };
  if(which == HK_GPOOL) {
    const int C = ip[0], act = ip[1], valueHead = ip[2], rawFp32 = ip[3], c0 = ip[4], ldr = ip[5];
    need(C >= 1 && c0 >= 0 && c0 + C <= ldr && act >= ACT_IDENTITY && act <= ACT_SILU && in[0] && in[1] && in[2]);
    float* pooled = poisoned((size_t)n * 3 * C);
    CK(launchGPool(placeRows(in[0], C, ldr, c0, !rawFp32), rawFp32 ? 1 : 0, ldr, c0, C, up(in[1], C), up(in[2], C), act, h.dMask, h.dMaskSum, n, L,
                   h.plan, valueHead ? 1 : 0, pooled, s));
    down(out[0], pooled, (size_t)n * 3 * C * sizeof(float));
  }
  else if(which == HK_BIASACT) {
    const int C = ip[0], act = ip[1], split = ip[2], rawFp32 = ip[3];
    need(C >= 1 && (split == 0 || split == 1) && act >= ACT_IDENTITY && act <= ACT_SILU && in[0] && in[2] && in[3] && out[0] && (!split || out[1]));
    const int cp = cpad(C), ld = cp * (split ? 2 : 1);
    __half* actOut = h.dalloc<__half>(M * ld);
    CK(cudaMemsetAsync(actOut, 0xFF, M * ld * sizeof(__half), s));
    CK(launchBiasAct(placeRows(in[0], C, cp, 0, !rawFp32), rawFp32 ? 1 : 0, cp, C, up(in[1], (size_t)n * C), C, up(in[2], C), up(in[3], C), act,
                     h.dMask, (int)M, h.plan, actOut, cp, split, s));
    std::vector<__half> ha(M * ld);
    down(ha.data(), actOut, ha.size() * sizeof(__half));
    const size_t used = hp.stats[0];
    if(!isOnes(ha.data() + used * ld, (M - used) * ld * sizeof(__half)))
      throw std::runtime_error(std::string(fn) + ": biasAct wrote past the plan's " + std::to_string(used) + " rows");
    for(size_t r = 0; r < used; r++)
      for(int c = 0; c < ld; c++)
        if((hp.mask[r] == 0.0f || c % cp >= C) && __half2float(ha[r * ld + c]) != 0.0f)
          throw std::runtime_error(std::string(fn) + ": biasAct's output is not zero at row " + std::to_string(r) + ", column " + std::to_string(c));
    for(int i = 0; i < n; i++)
      for(int y = 0; y < Y; y++)
        for(int x = 0; x < X; x++) {
          const long row = hp.row(L, i, y, x);
          const size_t o = (((size_t)i * Y + y) * X + x) * C;
          for(int c = 0; c < C; c++) {
            out[0][o + c] = row < 0 ? 0.0f : __half2float(ha[row * ld + c]);
            if(split) out[1][o + c] = row < 0 ? 0.0f : __half2float(ha[row * ld + cp + c]);
          }
        }
  }
  else if(which == HK_POLICY) {
    const int C = ip[0], act = ip[1], cp2 = ip[2], c0 = ip[3], ldr = ip[4];
    need(C >= 1 && cp2 >= 1 && cp2 <= 4 && c0 >= 0 && c0 + C <= ldr && act >= ACT_IDENTITY && act <= ACT_SILU && in[0] && in[1] && in[2] && in[3] && in[4]);
    float* pol = poisoned((size_t)n * (XY + 1));
    CK(launchPolicyOut((const float*)placeRows(in[0], C, ldr, c0, false), ldr, c0, C, up(in[1], (size_t)n * C), C, up(in[2], C), up(in[3], C), act,
                       up(in[4], (size_t)C * cp2), cp2, h.dMask, h.dSymmetry, up(in[5], n), n, L, h.plan, pol, s));
    down(out[0], pol, (size_t)n * (XY + 1) * sizeof(float));
  }
  else {   // HK_OWNERSHIP
    const int C = ip[0], act = ip[1], c0 = ip[2], ldr = ip[3];
    need(C >= 1 && c0 >= 0 && c0 + C <= ldr && act >= ACT_IDENTITY && act <= ACT_SILU && in[0] && in[1] && in[2] && in[3]);
    float* own = poisoned((size_t)n * XY);
    CK(launchOwnershipOut((const float*)placeRows(in[0], C, ldr, c0, false), ldr, c0, C, up(in[1], C), up(in[2], C), act, up(in[3], C), h.dMask,
                          h.dSymmetry, n, L, h.plan, own, s));
    down(out[0], own, (size_t)n * XY * sizeof(float));
  }
}
}  // namespace

extern "C" {

KGB_API int kgb_test_conv(int ky, int kx, int in_c, int out_c, const float* weights, int n, int nn_x_len, int nn_y_len, int use_fp16,
                  const float* input, float* output) {
  return guarded([&] {
    testConv("kgb_test_conv", ky, kx, in_c, out_c, weights, n, nn_x_len, nn_y_len, use_fp16, 0, input, nullptr, nullptr, nullptr, nullptr, nullptr,
             ACT_IDENTITY, output, nullptr, nullptr);
  });
}

KGB_API int kgb_test_conv_epilogue(int ky, int kx, int in_c, int out_c, const float* weights, int n, int nn_x_len, int nn_y_len, int use_fp16,
                           int epilogue_kind, const float* input, const float* residual_in, const float* bn_scale, const float* bn_bias,
                           int activation, float* raw_out, float* act_out) {
  return guarded([&] {
    if(epilogue_kind < 1 || epilogue_kind > 4) throw std::invalid_argument("kgb_test_conv_epilogue: bad argument");
    // the activated operand as the next layer sees it: hi + lo in split mode
    std::vector<float> lo(use_fp16 || !act_out ? 0 : (size_t)n * nn_x_len * nn_y_len * out_c);
    testConv("kgb_test_conv_epilogue", ky, kx, in_c, out_c, weights, n, nn_x_len, nn_y_len, use_fp16, epilogue_kind, input, nullptr, nullptr,
             residual_in, bn_scale, bn_bias, activation, raw_out, act_out, lo.empty() ? nullptr : lo.data());
    for(size_t k = 0; k < lo.size(); k++) act_out[k] += lo[k];
  });
}

KGB_API int kgb_test_conv_ex(int ky, int kx, int in_c, int out_c, const float* weights, int n, int nn_x_len, int nn_y_len, int use_fp16,
                             int epilogue_kind, const float* input, const int32_t* board_xy, const float* ncbias, const float* residual_in,
                             const float* bn_scale, const float* bn_bias, int activation, float* raw_out, float* act_hi_out,
                             float* act_lo_out) {
  return guarded([&] {
    testConv("kgb_test_conv_ex", ky, kx, in_c, out_c, weights, n, nn_x_len, nn_y_len, use_fp16, epilogue_kind, input, board_xy, ncbias,
             residual_in, bn_scale, bn_bias, activation, raw_out, act_hi_out, act_lo_out);
  });
}

KGB_API int kgb_test_conv_plan(int ky, int kx, int in_c, int out_c, const float* weights, int n, int nn_x_len, int nn_y_len, int use_fp16,
                               int epilogue_kind, const float* input, const int32_t* board_xy, const int32_t* symmetry, int ragged,
                               const float* ncbias, const float* residual_in, const float* bn_scale, const float* bn_bias, int activation,
                               float* raw_out, float* act_hi_out, float* act_lo_out, int64_t* layout_stats, int32_t* plan_out) {
  return guarded([&] {
    if(ragged < 0) throw std::invalid_argument("kgb_test_conv_plan: ragged must be 0 or 1");
    testConv("kgb_test_conv_plan", ky, kx, in_c, out_c, weights, n, nn_x_len, nn_y_len, use_fp16, epilogue_kind, input, board_xy, ncbias,
             residual_in, bn_scale, bn_bias, activation, raw_out, act_hi_out, act_lo_out, symmetry, ragged, layout_stats, plan_out);
  });
}

KGB_API int kgb_bench_conv_ex(int ky, int kx, int in_c, int out_c, int n, int nn_x_len, int nn_y_len, int use_fp16, int epilogue_kind, int rotate,
                      int warmup, int iters, float* ms_per_launch) {
  return guarded([&] {
    if(!ms_per_launch || n < 1 || iters < 1 || epilogue_kind < 0 || epilogue_kind > 4) throw std::invalid_argument("kgb_bench_conv_ex: bad argument");
    std::vector<float> w((size_t)ky * kx * in_c * out_c);
    uint32_t st = 12345u;
    for(auto& v : w) { st = st * 1664525u + 1013904223u; v = ((st >> 8) * (1.0f / 16777216.0f) - 0.5f) * 0.1f; }
    SingleConv sc(ky, kx, in_c, out_c, w.data(), n, nn_x_len, nn_y_len, use_fp16, epilogue_kind, rotate);
    std::vector<float> in((size_t)n * nn_x_len * nn_y_len * in_c);
    for(auto& v : in) { st = st * 1664525u + 1013904223u; v = (st >> 8) * (1.0f / 16777216.0f); }
    sc.setInput(in.data());
    for(int i = 0; i < warmup; i++) sc.run();
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    CK(cudaStreamSynchronize(sc.h.stream));
    CK(cudaEventRecord(e0, sc.h.stream));
    for(int i = 0; i < iters; i++) sc.run();
    CK(cudaEventRecord(e1, sc.h.stream));
    CK(cudaStreamSynchronize(sc.h.stream));
    float ms = 0.0f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    *ms_per_launch = ms / iters;
  });
}

KGB_API int kgb_test_conv_boundary(int inner_c, int trunk_c, int n, int nn_x_len, int nn_y_len, const int32_t* board_xy, int trunk_fp32,
                                   int inner_fp32, uint32_t seed, int64_t* out) {
  return guarded([&] { testBoundary("kgb_test_conv_boundary", inner_c, trunk_c, n, nn_x_len, nn_y_len, board_xy, nullptr, -1, trunk_fp32,
                                    inner_fp32, seed, out, nullptr); });
}

KGB_API int kgb_test_conv_boundary_plan(int inner_c, int trunk_c, int n, int nn_x_len, int nn_y_len, const int32_t* board_xy,
                                        const int32_t* symmetry, int ragged, int trunk_fp32, int inner_fp32, uint32_t seed, int64_t* out,
                                        int64_t* layout_stats) {
  return guarded([&] {
    if(ragged < 0) throw std::invalid_argument("kgb_test_conv_boundary_plan: ragged must be 0 or 1");
    testBoundary("kgb_test_conv_boundary_plan", inner_c, trunk_c, n, nn_x_len, nn_y_len, board_xy, symmetry, ragged, trunk_fp32, inner_fp32,
                 seed, out, layout_stats);
  });
}

KGB_API int kgb_test_conv_boundary_ex(int inner_c, int trunk_c, int n, int nn_x_len, int nn_y_len, const float* inner_a, const float* exit_w,
                                      const float* trunk_s, const float* trunk_scale, const float* trunk_bias, const float* entry_w,
                                      const float* inner_scale, const float* inner_bias, const int32_t* board_xy, const int32_t* symmetry,
                                      int ragged, int trunk_fp32, int inner_fp32, int fused, float* trunk_s_out, float* inner_s_out,
                                      float* inner_a_out, int64_t* layout_stats) {
  return guarded([&] {
    testBoundaryEx(inner_c, trunk_c, n, nn_x_len, nn_y_len, inner_a, exit_w, trunk_s, trunk_scale, trunk_bias, entry_w, inner_scale, inner_bias,
                   board_xy, symmetry, ragged, trunk_fp32, inner_fp32, fused, trunk_s_out, inner_s_out, inner_a_out, layout_stats);
  });
}

KGB_API int kgb_test_last_conv_kernel(int* out) {
  return guarded([&] {
    if(!out) throw std::invalid_argument("kgb_test_last_conv_kernel: bad argument");
    if(g_lastConvKernel < 0) throw std::runtime_error("kgb_test_last_conv_kernel: no convolution test hook has launched since the last failure");
    *out = g_lastConvKernel;
  });
}

KGB_API int kgb_test_head_kernel(int which, int n, int nn_x_len, int nn_y_len, int pad, const int32_t* board_xy, const int32_t* symmetry,
                                 int ragged, const int32_t* iparams, int num_iparams, const float* const* inputs, int num_inputs,
                                 float* const* outputs, int num_outputs, int64_t* layout_stats, int32_t* plan_out) {
  return guarded([&] {
    testHead(which, n, nn_x_len, nn_y_len, pad, board_xy, symmetry, ragged, iparams, num_iparams, inputs, num_inputs, outputs, num_outputs,
             layout_stats, plan_out);
  });
}

KGB_API int kgb_bench_conv_boundary(int inner_c, int trunk_c, int n, int nn_x_len, int nn_y_len, int trunk_fp32, int inner_fp32, int fused,
                                    int rotate, int warmup, int iters, float* ms_per_boundary) {
  return guarded([&] {
    if(!ms_per_boundary || n < 1 || iters < 1 || (inner_fp32 && !trunk_fp32)) throw std::invalid_argument("kgb_bench_conv_boundary: bad argument");
    BoundarySeed g(1);
    const ConvDesc post = g.conv(inner_c, trunk_c), pre = g.conv(trunk_c, inner_c);
    const BNDesc bnTrunk = g.bn(trunk_c), bnInner = g.bn(inner_c);
    BoundaryConv bc(inner_c, trunk_c, n, nn_x_len, nn_y_len, nullptr, trunk_fp32 != 0, inner_fp32 != 0, post, pre, bnTrunk, bnInner, rotate);
    bc.seedInputs(g);
    for(int i = 0; i < warmup; i++) bc.run(fused != 0);
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    CK(cudaStreamSynchronize(bc.h.stream));
    CK(cudaEventRecord(e0, bc.h.stream));
    for(int i = 0; i < iters; i++) bc.run(fused != 0);
    CK(cudaEventRecord(e1, bc.h.stream));
    CK(cudaStreamSynchronize(bc.h.stream));
    float ms = 0.0f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    *ms_per_boundary = ms / iters;
  });
}

// ---- Host-side tables and generators of the self-play loop (the loop itself is in kgb_selfplay.cu) ----------------------
KGB_API int kgb_expected_white_score_value(int n, const double* mean, const double* stdev, const double* center, const double* scale,
                                           const double* sqrt_board_area, double* out) {
  return guarded([&] {
    if(n < 0 || !mean || !stdev || !center || !scale || !sqrt_board_area || !out) throw std::invalid_argument("kgb_expected_white_score_value: bad argument");
    static const std::vector<double> table = makeExpectedSVTable();
    for(int i = 0; i < n; i++) out[i] = svExpectedWhiteScoreValue(table.data(), mean[i], stdev[i], center[i], scale[i], sqrt_board_area[i]);
  });
}

KGB_API int kgb_rand_uint32_stream(const char* seed_string, int n, uint32_t* out) {
  return guarded([&] {
    if(!seed_string || !out || n < 0) throw std::invalid_argument("kgb_rand_uint32_stream: bad argument");
    RefRand r(seed_string);
    for(int i = 0; i < n; i++) out[i] = r.nextUInt();
  });
}

KGB_API int kgb_value_weight_cdf_table(double* out, int n) {
  return guarded([&] {
    if(!out || n != VW_TABLE_SIZE) throw std::invalid_argument("kgb_value_weight_cdf_table: out must hold 2000 doubles");
    const std::vector<double> t = makeValueWeightCdfTable();
    std::copy(t.begin(), t.end(), out);
  });
}

KGB_API int kgb_zobrist_tables(int x_size, int y_size, uint64_t* board_hash, uint64_t* size_hash) {
  return guarded([&] {
    if(!board_hash || !size_hash || x_size < 2 || y_size < 2 || x_size > 19 || y_size > 19) throw std::invalid_argument("kgb_zobrist_tables: bad argument");
    ZobristTables z = makeZobristTables(x_size, y_size);
    for(int y = 0; y < y_size; y++)
      for(int x = 0; x < x_size; x++)
        for(int c = 0; c < 2; c++) {
          const Hash128& h = z.board[(y * 32 + x) * 2 + c];
          uint64_t* o = board_hash + (((size_t)y * x_size + x) * 2 + c) * 2;
          o[0] = h.h0; o[1] = h.h1;
        }
    size_hash[0] = z.sizeHash.h0; size_hash[1] = z.sizeHash.h1;
  });
}

}  // extern "C"
