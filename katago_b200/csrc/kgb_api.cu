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
#include "kgb_kernels.cuh"
#include "kgb_model.h"
#include "kgb_selfplay.h"
#include "kgb_scorevalue.h"
#include "kgb_rand.h"

using namespace kgb;

// ------------------------------------------------------------------------------------------------------------
// Error plumbing
// ------------------------------------------------------------------------------------------------------------
static thread_local std::string g_lastError;

struct CudaFailure : std::runtime_error {
  using std::runtime_error::runtime_error;
};

#define CK(expr)                                                                                                       \
  do {                                                                                                                 \
    cudaError_t _e = (expr);                                                                                           \
    if(_e != cudaSuccess)                                                                                              \
      throw CudaFailure(std::string("CUDA error ") + cudaGetErrorName(_e) + " (" + cudaGetErrorString(_e) + ") at " + \
                        __FILE__ + ":" + std::to_string(__LINE__) + ": " #expr);                                       \
  } while(0)

template <class F>
static int guarded(F&& f) {
  try {
    f();
    return KGB_OK;
  }
  catch(const CudaFailure& e) { g_lastError = e.what(); return KGB_ERR_CUDA; }
  catch(const std::invalid_argument& e) { g_lastError = e.what(); return KGB_ERR_INVALID; }
  catch(const std::exception& e) { g_lastError = e.what(); return KGB_ERR_IO; }
}

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

// Residual stream [rows][cols], fp32 or fp16, box {32 cols, 128 rows}: the slices the convolution's epilogue reads from shared
// memory, 128B-swizzled for fp32 (128 B rows) and 64B-swizzled for fp16 (64 B rows), zero OOB fill.
static CUtensorMap makeTmapResidual(const void* ptr, uint64_t rows, uint64_t cols, bool fp32) {
  CUtensorMap m;
  const uint64_t esize = fp32 ? sizeof(float) : sizeof(__half);
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {cols * esize};
  cuuint32_t box[2] = {32, 128};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = getEncodeTiled()(&m, fp32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), gdim,
                                gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, fp32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if(r != CUDA_SUCCESS) throw CudaFailure("cuTensorMapEncodeTiled (residual) failed with CUresult " + std::to_string((int)r));
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

struct kgb_handle {
  int device = 0;
  cudaStream_t stream = nullptr;
  const ModelDesc* model = nullptr;
  Layout L{};
  int maxBatch = 0;
  int split = 0;          // fp32-equivalent mode
  bool nhwc = true;
  bool streamTrunkFp32 = true, streamInnerFp32 = false;
  std::vector<void*> allocs;
  // inputs / outputs (device, fixed addresses so graphs can be replayed)
  float *dSpatial = nullptr, *dGlobal = nullptr, *dOptimism = nullptr;
  int* dSymmetry = nullptr;
  float *dPolicy = nullptr, *dValue = nullptr, *dScore = nullptr, *dOwnership = nullptr;
  // pinned staging
  float *hSpatial = nullptr, *hGlobal = nullptr, *hOptimism = nullptr, *hPolicy = nullptr, *hValue = nullptr, *hScore = nullptr,
        *hOwnership = nullptr;
  int* hSymmetry = nullptr;
  float *dMask = nullptr, *dMaskSum = nullptr;
  std::vector<std::function<void(int, cudaStream_t)>> ops;
  int launchesPerForward = 0;
  std::map<int, cudaGraphExec_t> graphs;

  // Weights live in ONE arena: a net of the same architecture is swapped in between two waves by one device copy
  // (kgb_handle_stage_weights / kgb_handle_commit_weights) and travels between the GPUs of a node as one ncclBroadcast
  // (kgb_handle_broadcast_staged_weights).  The graph builder runs in three modes over the same code:
  //   W_SIZE   on a scratch handle: only adds up the arena (nothing is allocated, no op is kept)
  //   W_BUILD  the real build: device addresses from wLive, bytes packed into the pinned mirror wHost, one H2D copy at the end
  //   W_REPACK on a scratch handle: packs ANOTHER model's weights into wHost at the same offsets, destined for wShadow
  enum { W_BUILD = 0, W_SIZE = 1, W_REPACK = 2 };
  int wMode = W_BUILD;
  char *wLive = nullptr, *wShadow = nullptr, *wHost = nullptr;
  size_t wBytes = 0, wCursor = 0, wIndex = 0;
  std::vector<size_t> wSizes;     // the arena's spans in build order: a staged model must produce the same sequence
  std::string wSignature;         // shapes, activations and head constants that ops capture by value (must match as well)
  cudaStream_t copyStream = nullptr;
  cudaEvent_t stagedEvent = nullptr, bcastStart = nullptr, bcastStop = nullptr;
  bool staged = false;
  void* ncclComm = nullptr;
  int ncclRank = 0, ncclRanks = 0;

  template <class T>
  T* dalloc(size_t count) {
    if(wMode != W_BUILD) return (T*)(uintptr_t)256;      // scratch pass: activations are never touched
    void* p = nullptr;
    CK(cudaMalloc(&p, count * sizeof(T)));
    CK(cudaMemset(p, 0, count * sizeof(T)));
    allocs.push_back(p);
    return (T*)p;
  }
  // One span of the weight arena: returns its device address and (except in W_SIZE) where to pack its bytes on the host
  void* walloc(size_t bytes, void** host) {
    const size_t b = (bytes + 255) & ~(size_t)255;
    const size_t o = wCursor;
    wCursor += b;
    if(wMode == W_SIZE) {
      wSizes.push_back(b);
      *host = nullptr;
      return (void*)(uintptr_t)(256 + o);
    }
    if(wIndex >= wSizes.size() || wSizes[wIndex] != b || o + b > wBytes)
      throw std::invalid_argument("the model's weights do not have the layout this handle was built for (different architecture)");
    wIndex++;
    *host = wHost + o;
    return (wMode == W_BUILD ? wLive : wShadow) + o;
  }
  void wAllocArena(size_t bytes) {
    wBytes = bytes;
    CK(cudaMalloc((void**)&wLive, std::max<size_t>(bytes, 256)));
    CK(cudaMemset(wLive, 0, std::max<size_t>(bytes, 256)));
    allocs.push_back(wLive);
    CK(cudaMallocHost((void**)&wHost, std::max<size_t>(bytes, 256)));
    memset(wHost, 0, std::max<size_t>(bytes, 256));
  }
  void wFlushLive() {       // the packed bytes reach the device in one copy
    CK(cudaMemcpy(wLive, wHost, wCursor, cudaMemcpyHostToDevice));
    CK(cudaDeviceSynchronize());
  }
  float* upload(const std::vector<float>& v, size_t padTo = 0) {
    size_t n = std::max(v.size(), padTo);
    void* hp = nullptr;
    float* d = (float*)walloc(n * sizeof(float), &hp);
    if(hp) {
      memset(hp, 0, n * sizeof(float));
      if(!v.empty()) memcpy(hp, v.data(), v.size() * sizeof(float));
    }
    return d;
  }
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
  Builder(kgb_handle& hh) : h(hh), m(*hh.model), Mmax((size_t)hh.maxBatch * hh.L.P), actMul(hh.split ? 2 : 1) {}

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

  // Emit one convolution op.  residual/rawOut may alias (in-place residual update).
  void emitConv(const ConvWeights& cw, const __half* A, const void* residual, bool residualFp32, const float* ncbias, void* rawOut,
                bool rawFp32, __half* actOut, BNDev bn) {
    // the kernel reads a tile's halo rows of A while the neighbouring tiles write their outputs (the scratch passes have no buffers)
    if(h.wMode == kgb_handle::W_BUILD && ((const void*)A == (const void*)actOut || (const void*)A == rawOut))
      throw std::logic_error("emitConv: the operand aliases an output");
    kgb_handle* hp = &h;
    const int actMulL = actMul;
    h.ops.push_back([=](int n, cudaStream_t s) {
      ConvParams p;
      memset(&p, 0, sizeof(p));
      p.M = n * hp->L.P;
      p.P = hp->L.P;
      p.Wp = hp->L.Wp;
      p.ky = cw.ky; p.kx = cw.kx;
      p.cin_p = cw.cin_p; p.cout_p = cw.cout_p;
      p.n_tile = cw.n_tile;
      p.num_m_tiles = (p.M + 127) / 128;
      p.num_n_tiles = cw.num_n_tiles;
      p.split = hp->split;
      p.residual = residual; p.residual_fp32 = residualFp32 ? 1 : 0;
      p.ncbias = ncbias;
      p.raw_out = rawOut; p.raw_fp32 = rawFp32 ? 1 : 0;
      p.act_out = actOut;
      p.bn_scale = bn.scale; p.bn_bias = bn.bias; p.act = bn.act;
      p.mask = hp->dMask;
      CUtensorMap tmA = makeTmap2D(A, (uint64_t)p.M, (uint64_t)cw.cin_p * actMulL, (uint32_t)convABoxRows(cw.ky, cw.kx, p.Wp));
      CUtensorMap tmR;
      memset(&tmR, 0, sizeof(tmR));
      if(residual != nullptr) tmR = makeTmapResidual(residual, (uint64_t)p.M, (uint64_t)cw.cout_p, residualFp32);
      CK(launchConvWG(tmA, cw.tmapB, tmR, p, s));
    });
    h.launchesPerForward++;
  }

  // blocks operate on stream lv.S, with lv.A = act(preBN_0(S)) on entry and = act(finalBN(S_out)) on exit.
  void emitBlocks(const std::vector<BlockDesc>& blocks, Level& lv, const BNDesc& finalBN, int finalAct, bool keepFinalRaw) {
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
          CK(launchGPool(G, 1, gld, regC, gC, gbn.scale, gbn.bias, gbn.act, hp->dMask, hp->dMaskSum, n, hp->L, 0, pooled, s));
          CK(launchMatMulNC(pooled, 3 * gC, Wg, nullptr, n, 3 * gC, regC, ACT_IDENTITY, bias, regC, s));
          CK(launchBiasAct(G, 1, gld, regC, bias, regC, mid.scale, mid.bias, mid.act, hp->dMask, n * hp->L.P, hp->L.P, T, tcp, split, s));
        });
        h.launchesPerForward += 3;
        emitConv(w2, lv.T, lv.S, lv.fp32, nullptr, rawOut, lv.fp32, lv.A, nextBN);
      }
      else {
        ConvWeights wpre = packConv({&b.conv1});
        ConvWeights wpost = packConv({&b.conv2});
        Level inner = makeLevel(b.conv1.cout, h.streamInnerFp32, b.blocks);
        BNDev innerPre = uploadBN(b.blocks[0].preBN, b.blocks[0].preAct, inner.cp);
        emitConv(wpre, lv.A, nullptr, false, nullptr, inner.S, inner.fp32, inner.A, innerPre);
        emitBlocks(b.blocks, inner, b.midBN, b.midAct, false);
        emitConv(wpost, inner.A, lv.S, lv.fp32, nullptr, rawOut, lv.fp32, lv.A, nextBN);
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
    __half* inAct = h.dalloc<__half>(Mmax * cinP * actMul);
    kgb_handle* hp = &h;
    const int C = m.numInputChannels, split = h.split;
    h.ops.push_back([=](int n, cudaStream_t s) {
      CK(launchPackInput(hp->dSpatial, n, C, hp->nhwc, hp->dSymmetry, hp->L, inAct, cinP, split, hp->dMask, hp->dMaskSum, s));
    });
    h.launchesPerForward += 4;
    // trunk
    Level trunk = makeLevel(m.trunkC, h.streamTrunkFp32, m.blocks);
    float* initBias = h.dalloc<float>((size_t)h.maxBatch * trunk.cp);
    const float* Wglob = h.upload(m.initialMatMul.w);
    const int G = m.numInputGlobalChannels, trunkC = m.trunkC, trunkCp = trunk.cp;
    h.ops.push_back([=](int n, cudaStream_t s) {
      CK(launchMatMulNC(hp->dGlobal, G, Wglob, nullptr, n, G, trunkC, ACT_IDENTITY, initBias, trunkCp, s));
    });
    h.launchesPerForward++;
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
      CK(launchGPool(H, 1, hld, p1C, g1C, g1bn.scale, g1bn.bias, g1bn.act, hp->dMask, hp->dMaskSum, n, hp->L, 0, g1pool, s));
      CK(launchMatMulNC(g1pool, 3 * g1C, Wg2b, nullptr, n, 3 * g1C, p1C, ACT_IDENTITY, g1bias, p1C, s));
      CK(launchPolicyOut(H, hld, 0, p1C, g1bias, p1C, p1bn.scale, p1bn.bias, p1bn.act, Wp2, cp2, hp->dMask, hp->dSymmetry,
                         hp->dOptimism, n, hp->L, hp->dPolicy, s));
      if(version >= 15) {
        CK(launchMatMulNC(g1pool, 3 * g1C, Wpass, passBias, n, 3 * g1C, passMid, passAct, passH, passMid, s));
        CK(launchMatMulNC(passH, passMid, Wpass2, nullptr, n, passMid, cp2, ACT_IDENTITY, passLogits, 4, s));
      }
      else {
        CK(launchMatMulNC(g1pool, 3 * g1C, Wpass, nullptr, n, 3 * g1C, cp2, ACT_IDENTITY, passLogits, 4, s));
      }
      // value head
      CK(launchGPool(H, 1, hld, p1C + g1C, v1C, v1bn.scale, v1bn.bias, v1bn.act, hp->dMask, hp->dMaskSum, n, hp->L, 1, v1pool, s));
      CK(launchMatMulNC(v1pool, 3 * v1C, Wv2, bv2, n, 3 * v1C, v2C, v2Act, v2, v2C, s));
      CK(launchMatMulNC(v2, v2C, Wv3, bv3, n, v2C, 3, ACT_IDENTITY, value, 3, s));
      CK(launchMatMulNC(v2, v2C, Wsv3, bsv3, n, v2C, numSV, ACT_IDENTITY, sv, numSV, s));
      CK(launchOwnershipOut(H, hld, p1C + g1C, v1C, v1bn.scale, v1bn.bias, v1bn.act, Wown, hp->dMask, hp->dSymmetry, n, hp->L,
                            hp->dOwnership, s));
      CK(launchFinalize(passLogits, 4, cp2, hp->dOptimism, value, sv, numSV, version, n, hp->L.X * hp->L.Y + 1, hp->dPolicy,
                        hp->dValue, hp->dScore, s));
    });
    h.launchesPerForward += (version >= 15 ? 11 : 10);
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

void runOps(kgb_handle* h, int n) {
  auto it = h->graphs.find(n);
  if(it == h->graphs.end()) {
    cudaGraph_t graph = nullptr;
    CK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
    try {
      for(auto& op : h->ops) op(n, h->stream);
    }
    catch(...) {
      cudaStreamEndCapture(h->stream, &graph);
      if(graph) cudaGraphDestroy(graph);
      throw;
    }
    CK(cudaStreamEndCapture(h->stream, &graph));
    cudaGraphExec_t exec = nullptr;
    CK(cudaGraphInstantiate(&exec, graph, 0));
    CK(cudaGraphDestroy(graph));
    it = h->graphs.emplace(n, exec).first;
  }
  CK(cudaGraphLaunch(it->second, h->stream));
}

}  // namespace

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

// The settings that decide how the graph builder lays the weights out
static void copyBuildSettings(kgb_handle& dst, const kgb_handle& src) {
  dst.device = src.device; dst.model = src.model; dst.L = src.L; dst.maxBatch = src.maxBatch; dst.split = src.split;
  dst.nhwc = src.nhwc; dst.streamTrunkFp32 = src.streamTrunkFp32; dst.streamInnerFp32 = src.streamInnerFp32;
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
  for(void* p : {(void*)h->hSpatial, (void*)h->hGlobal, (void*)h->hOptimism, (void*)h->hPolicy, (void*)h->hValue, (void*)h->hScore,
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
    CK(cudaMallocHost((void**)&h.hOptimism, (size_t)h.maxBatch * sizeof(float)));
    CK(cudaMallocHost((void**)&h.hSymmetry, (size_t)h.maxBatch * sizeof(int)));
    CK(cudaMallocHost((void**)&h.hPolicy, (size_t)h.maxBatch * (XY + 1) * sizeof(float)));
    CK(cudaMallocHost((void**)&h.hValue, (size_t)h.maxBatch * 3 * sizeof(float)));
    CK(cudaMallocHost((void**)&h.hScore, (size_t)h.maxBatch * 6 * sizeof(float)));
    CK(cudaMallocHost((void**)&h.hOwnership, (size_t)h.maxBatch * XY * sizeof(float)));
    CK(cudaDeviceSynchronize());
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
  CK(cudaMemset(h->wShadow, 0, std::max<size_t>(h->wBytes, 256)));
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

KGB_API int kgb_handle_sync(kgb_handle* handle) {
  return guarded([&] {
    if(!handle) throw std::invalid_argument("kgb_handle_sync: NULL handle");
    CK(cudaSetDevice(handle->device));
    CK(cudaStreamSynchronize(handle->stream));
  });
}

static void checkForwardArgs(kgb_handle* h, int n, const void* a, const void* b, const void* c, const void* d, const void* e) {
  if(!h) throw std::invalid_argument("kgb_forward: NULL handle");
  if(n < 1 || n > h->maxBatch) throw std::invalid_argument("kgb_forward: batch size " + std::to_string(n) + " not in [1, maxBatchSize]");
  if(!a || !b || !c || !d || !e) throw std::invalid_argument("kgb_forward: NULL buffer");
}

KGB_API int kgb_forward(kgb_handle* h, int n, const float* spatial, const float* global, const int32_t* symmetry, const float* policy_optimism,
                float* policy, float* value, float* score_value, float* ownership) {
  return guarded([&] {
    checkForwardArgs(h, n, spatial, global, policy, value, score_value);
    CK(cudaSetDevice(h->device));
    const ModelDesc& m = *h->model;
    const int XY = h->L.X * h->L.Y;
    const size_t spB = (size_t)n * m.numInputChannels * XY * sizeof(float);
    const size_t glB = (size_t)n * m.numInputGlobalChannels * sizeof(float);
    memcpy(h->hSpatial, spatial, spB);
    memcpy(h->hGlobal, global, glB);
    for(int i = 0; i < n; i++) {
      h->hSymmetry[i] = symmetry ? symmetry[i] : 0;
      h->hOptimism[i] = policy_optimism ? policy_optimism[i] : 0.0f;
      if(h->hSymmetry[i] < 0 || h->hSymmetry[i] > 7) throw std::invalid_argument("kgb_forward: symmetry must be in 0..7");
    }
    cudaStream_t s = h->stream;
    CK(cudaMemcpyAsync(h->dSpatial, h->hSpatial, spB, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(h->dGlobal, h->hGlobal, glB, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(h->dSymmetry, h->hSymmetry, n * sizeof(int), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(h->dOptimism, h->hOptimism, n * sizeof(float), cudaMemcpyHostToDevice, s));
    runOps(h, n);
    CK(cudaMemcpyAsync(h->hPolicy, h->dPolicy, (size_t)n * (XY + 1) * sizeof(float), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(h->hValue, h->dValue, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(h->hScore, h->dScore, (size_t)n * 6 * sizeof(float), cudaMemcpyDeviceToHost, s));
    if(ownership) CK(cudaMemcpyAsync(h->hOwnership, h->dOwnership, (size_t)n * XY * sizeof(float), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    memcpy(policy, h->hPolicy, (size_t)n * (XY + 1) * sizeof(float));
    memcpy(value, h->hValue, (size_t)n * 3 * sizeof(float));
    memcpy(score_value, h->hScore, (size_t)n * 6 * sizeof(float));
    if(ownership) memcpy(ownership, h->hOwnership, (size_t)n * XY * sizeof(float));
  });
}

KGB_API int kgb_forward_device(kgb_handle* h, int n, const float* d_spatial, const float* d_global, const int32_t* d_symmetry,
                       const float* d_policy_optimism, float* d_policy, float* d_value, float* d_score_value, float* d_ownership) {
  return guarded([&] {
    checkForwardArgs(h, n, d_spatial, d_global, d_policy, d_value, d_score_value);
    CK(cudaSetDevice(h->device));
    const ModelDesc& m = *h->model;
    const int XY = h->L.X * h->L.Y;
    cudaStream_t s = h->stream;
    if(d_spatial != h->dSpatial)
      CK(cudaMemcpyAsync(h->dSpatial, d_spatial, (size_t)n * m.numInputChannels * XY * sizeof(float), cudaMemcpyDeviceToDevice, s));
    if(d_global != h->dGlobal)
      CK(cudaMemcpyAsync(h->dGlobal, d_global, (size_t)n * m.numInputGlobalChannels * sizeof(float), cudaMemcpyDeviceToDevice, s));
    if(d_symmetry) CK(cudaMemcpyAsync(h->dSymmetry, d_symmetry, n * sizeof(int), cudaMemcpyDeviceToDevice, s));
    else CK(cudaMemsetAsync(h->dSymmetry, 0, n * sizeof(int), s));
    if(d_policy_optimism) CK(cudaMemcpyAsync(h->dOptimism, d_policy_optimism, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
    else CK(cudaMemsetAsync(h->dOptimism, 0, n * sizeof(float), s));
    runOps(h, n);
    CK(cudaMemcpyAsync(d_policy, h->dPolicy, (size_t)n * (XY + 1) * sizeof(float), cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(d_value, h->dValue, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(d_score_value, h->dScore, (size_t)n * 6 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    if(d_ownership) CK(cudaMemcpyAsync(d_ownership, h->dOwnership, (size_t)n * XY * sizeof(float), cudaMemcpyDeviceToDevice, s));
  });
}

}  // extern "C" (part 1)

// Stand-alone single convolution (testEvaluateConv / kernel-level roofline timing).
namespace {
struct SingleConv {
  kgb_handle h;
  ModelDesc dummy;
  ConvWeights cw;
  int n, X, Y, cin, cout;
  size_t M;
  // one entry per buffer set: the operand, the activated output (kinds 1-4) and the raw output (kind 0) or raw stream (kinds 2-4)
  std::vector<__half*> As, acts;
  std::vector<void*> raws;
  bool rawF32 = true;   // the raw output of kind 0 is fp32; the stream of kinds 2-4 is fp32 for kind 4 and in fp32-equivalent mode
  int rotate, next = 0;
  // kind: 0 = fp32 raw output only; 1 = the first conv of a residual unit (BN + mish + mask -> fp16 operand of the next conv);
  // 2 = the second conv of a unit (+ fp16 residual stream, updated in place, and the next unit's BN + mish operand); 3 = a nested
  // block's pre conv (fp16 raw stream + activated operand); 4 = kind 2 with an fp32 residual stream, as the trunk runs in fp16 mode
  // with KGB_STREAM_FP32=trunk.  In fp32-equivalent mode every stream is fp32.  `rotate` independent buffer sets are cycled through
  // by run() so that a timing loop does not live in L2.
  SingleConv(int ky, int kx, int in_c, int out_c, const float* weights, int n_, int X_, int Y_, int use_fp16, int kind, int rotate_ = 1,
             const float* bnScale = nullptr, const float* bnBias = nullptr, int actKind = ACT_MISH)
      : n(n_), X(X_), Y(Y_), cin(in_c), cout(out_c), rotate(rotate_ < 1 ? 1 : rotate_) {
    h.device = selectDevice(-1);
    h.model = &dummy;
    h.maxBatch = n;
    h.split = use_fp16 ? 0 : 1;
    h.L = boardLayout(X, Y, std::max(1, std::max(ky / 2, kx / 2)));
    h.streamTrunkFp32 = h.streamInnerFp32 = h.split != 0;
    CK(cudaStreamCreateWithFlags(&h.stream, cudaStreamNonBlocking));
    CK(convWGInit());
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
    M = (size_t)n * h.L.P;
    h.dMask = h.dalloc<float>(M + 128);
    h.dMaskSum = h.dalloc<float>(n);
    rawF32 = kind == 0 || kind == 4 || h.split != 0;
    for(int r = 0; r < rotate; r++) {
      __half* A = h.dalloc<__half>(M * cw.cin_p * b.actMul);
      __half* act = kind == 0 ? nullptr : h.dalloc<__half>(M * cw.cout_p * b.actMul);
      void* raw = kind == 1 ? nullptr : rawF32 ? (void*)h.dalloc<float>(M * cw.cout_p) : (void*)h.dalloc<__half>(M * cw.cout_p);
      As.push_back(A);
      if(act) acts.push_back(act);
      if(raw) raws.push_back(raw);
      b.emitConv(cw, A, kind == 2 || kind == 4 ? raw : nullptr, rawF32, nullptr, raw, rawF32, act, kind == 0 ? Builder::BNDev() : dev);
    }
  }
  ~SingleConv() {
    for(void* p : h.allocs) cudaFree(p);
    if(h.wHost) cudaFreeHost(h.wHost);
    if(h.stream) cudaStreamDestroy(h.stream);
  }
  void setInput(const float* input /* NHWC */) {
    float* dIn = h.dalloc<float>((size_t)n * X * Y * cin);
    CK(cudaMemcpy(dIn, input, (size_t)n * X * Y * cin * sizeof(float), cudaMemcpyHostToDevice));
    CK(cudaDeviceSynchronize());   // see below: the pack kernel runs on a non-blocking stream
    CK(launchPackInput(dIn, n, cin, true, nullptr, h.L, As[0], cw.cin_p, h.split, h.dMask, h.dMaskSum, h.stream));
    CK(cudaStreamSynchronize(h.stream));
    for(size_t r = 1; r < As.size(); r++) CK(cudaMemcpy(As[r], As[0], M * cw.cin_p * (h.split ? 2 : 1) * sizeof(__half), cudaMemcpyDeviceToDevice));
    // the mask of a bare convolution is "every board point", not input channel 0
    std::vector<float> hm(M, 0.0f);
    for(int i = 0; i < n; i++)
      for(int y = 0; y < Y; y++)
        for(int x = 0; x < X; x++) hm[(size_t)i * h.L.P + (size_t)(y + h.L.pad) * h.L.Wp + x] = 1.0f;
    CK(cudaMemcpy(h.dMask, hm.data(), M * sizeof(float), cudaMemcpyHostToDevice));
    // cudaMemcpy from pageable memory may return before the DMA has landed, and h.stream is non-blocking:
    // nothing else orders these uploads before the kernels launched on it.
    CK(cudaDeviceSynchronize());
  }
  void run() { h.ops[next](n, h.stream); next = (next + 1) % rotate; }
};

// kgb_test_conv (kind 0) and kgb_test_conv_epilogue (kinds 1-4): one launch, NHWC in and out
void testConv(const char* fn, int ky, int kx, int in_c, int out_c, const float* weights, int n, int nn_x_len, int nn_y_len, int use_fp16, int kind,
              const float* input, const float* residual_in, const float* bn_scale, const float* bn_bias, int activation, float* raw_out,
              float* act_out) {
  const bool hasResidual = kind == 2 || kind == 4;
  if(!weights || !input || n < 1 || (kind == 0 ? !raw_out : !act_out)) throw std::invalid_argument(std::string(fn) + ": bad argument");
  if(hasResidual && !residual_in) throw std::invalid_argument(std::string(fn) + ": kinds 2 and 4 need residual_in");
  if(kind >= 2 && !raw_out) throw std::invalid_argument(std::string(fn) + ": kinds 2 to 4 need raw_out");
  SingleConv sc(ky, kx, in_c, out_c, weights, n, nn_x_len, nn_y_len, use_fp16, kind, 1, bn_scale, bn_bias, activation);
  sc.setInput(input);
  const int cp = sc.cw.cout_p;
  const bool f32 = sc.rawF32;
  auto rowOf = [&](int i, int y, int x) { return (size_t)i * sc.h.L.P + (size_t)(y + sc.h.L.pad) * sc.h.L.Wp + x; };
  if(hasResidual) {
    std::vector<float> hf(sc.M * cp, 0.0f);
    for(int i = 0; i < n; i++) for(int y = 0; y < nn_y_len; y++) for(int x = 0; x < nn_x_len; x++) for(int c = 0; c < out_c; c++)
      hf[rowOf(i, y, x) * cp + c] = residual_in[(((size_t)i * nn_y_len + y) * nn_x_len + x) * out_c + c];
    if(f32) CK(cudaMemcpy(sc.raws[0], hf.data(), hf.size() * sizeof(float), cudaMemcpyHostToDevice));
    else {
      std::vector<__half> hh(hf.size());
      for(size_t k = 0; k < hf.size(); k++) hh[k] = __float2half_rn(hf[k]);
      CK(cudaMemcpy(sc.raws[0], hh.data(), hh.size() * sizeof(__half), cudaMemcpyHostToDevice));
    }
    CK(cudaDeviceSynchronize());
  }
  sc.run();
  CK(cudaStreamSynchronize(sc.h.stream));
  const int am = sc.h.split ? 2 : 1;
  std::vector<__half> ha;
  if(!sc.acts.empty()) {
    ha.resize(sc.M * cp * am);
    CK(cudaMemcpy(ha.data(), sc.acts[0], ha.size() * sizeof(__half), cudaMemcpyDeviceToHost));
  }
  std::vector<float> hr;
  if(!sc.raws.empty()) {
    hr.resize(sc.M * cp);
    if(f32) CK(cudaMemcpy(hr.data(), sc.raws[0], hr.size() * sizeof(float), cudaMemcpyDeviceToHost));
    else {
      std::vector<__half> hh(hr.size());
      CK(cudaMemcpy(hh.data(), sc.raws[0], hh.size() * sizeof(__half), cudaMemcpyDeviceToHost));
      for(size_t k = 0; k < hr.size(); k++) hr[k] = __half2float(hh[k]);
    }
  }
  if(!ha.empty()) {
    // every row that is not a board point (pad rows / columns) must have been written as zero: the next conv's halo reads them
    std::vector<char> onBoard(sc.M, 0);
    for(int i = 0; i < n; i++) for(int y = 0; y < nn_y_len; y++) for(int x = 0; x < nn_x_len; x++) onBoard[rowOf(i, y, x)] = 1;
    for(size_t r = 0; r < sc.M; r++)
      if(!onBoard[r])
        for(int c = 0; c < cp * am; c++)
          if(__half2float(ha[r * cp * am + c]) != 0.0f) throw std::runtime_error(std::string(fn) + ": pad row " + std::to_string(r) + " of the activation output is not zero");
  }
  for(int i = 0; i < n; i++) for(int y = 0; y < nn_y_len; y++) for(int x = 0; x < nn_x_len; x++) for(int c = 0; c < out_c; c++) {
    const size_t row = rowOf(i, y, x), o = (((size_t)i * nn_y_len + y) * nn_x_len + x) * out_c + c;
    if(!ha.empty()) act_out[o] = __half2float(ha[row * cp * am + c]) + (am == 2 ? __half2float(ha[row * cp * am + cp + c]) : 0.0f);
    if(!hr.empty()) raw_out[o] = hr[row * cp + c];
  }
}
}  // namespace

extern "C" {

KGB_API int kgb_test_conv(int ky, int kx, int in_c, int out_c, const float* weights, int n, int nn_x_len, int nn_y_len, int use_fp16,
                  const float* input, float* output) {
  return guarded([&] {
    testConv("kgb_test_conv", ky, kx, in_c, out_c, weights, n, nn_x_len, nn_y_len, use_fp16, 0, input, nullptr, nullptr, nullptr, ACT_IDENTITY, output,
             nullptr);
  });
}

KGB_API int kgb_test_conv_epilogue(int ky, int kx, int in_c, int out_c, const float* weights, int n, int nn_x_len, int nn_y_len, int use_fp16,
                           int epilogue_kind, const float* input, const float* residual_in, const float* bn_scale, const float* bn_bias,
                           int activation, float* raw_out, float* act_out) {
  return guarded([&] {
    if(epilogue_kind < 1 || epilogue_kind > 4) throw std::invalid_argument("kgb_test_conv_epilogue: bad argument");
    testConv("kgb_test_conv_epilogue", ky, kx, in_c, out_c, weights, n, nn_x_len, nn_y_len, use_fp16, epilogue_kind, input, residual_in, bn_scale,
             bn_bias, activation, raw_out, act_out);
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

// ---- Boundary 2: device-resident self-play ------------------------------------------------------------------
struct kgb_selfplay {
  kgb_handle* h = nullptr;
  SelfplayImpl* impl = nullptr;
  int n = 0;
  bool fakeNN = false;
  cudaGraphExec_t stepGraph = nullptr;
};

static void selfplayStepLaunches(kgb_selfplay* sp, cudaStream_t s) {
  selfplayLaunchSelect(sp->impl, s);
  if(sp->fakeNN) selfplayLaunchFakeNN(sp->impl, sp->h->dPolicy, sp->h->dValue, sp->h->dScore, sp->h->dOwnership, s);
  else for(auto& op : sp->h->ops) op(sp->n, s);
  selfplayLaunchBackup(sp->impl, s);
}

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

KGB_API int kgb_selfplay_get_play_selection_values(kgb_selfplay* sp, int game, double* values) {
  return guarded([&] {
    if(!sp || !values) throw std::invalid_argument("kgb_selfplay_get_play_selection_values: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadPlaySelection(sp->impl, game, values);
  });
}

KGB_API int kgb_test_choose_index_with_temperature(const char* seed_string, const double* relative_probs, int n, double temperature,
                                                   double only_below_prob, int count, int32_t* chosen) {
  return guarded([&] {
    if(!seed_string || !relative_probs || !chosen || n < 1 || count < 1) throw std::invalid_argument("kgb_test_choose_index_with_temperature: bad argument");
    chooseIndexTest(seed_string, relative_probs, n, temperature, only_below_prob, count, chosen);
  });
}

KGB_API int kgb_test_history_replay(int x_len, int y_len, int ko_rule, int multi_stone_suicide_legal, int num_games, int max_moves, const int8_t* moves_xy,
                                    uint8_t* flags, uint8_t* legal_next, uint8_t* super_ko_banned) {
  return guarded([&] {
    if(!moves_xy || !flags || !legal_next || !super_ko_banned || num_games < 1 || max_moves < 1 || ko_rule < 0 || ko_rule > 3)
      throw std::invalid_argument("kgb_test_history_replay: bad argument");
    historyReplay(x_len, y_len, ko_rule, multi_stone_suicide_legal, num_games, max_moves, moves_xy, flags, legal_next, super_ko_banned);
  });
}

KGB_API int kgb_test_repetition_bound(int x_len, int y_len, int num_moves, int bound, const int8_t* moves_xyp, uint8_t* out) {
  return guarded([&] {
    if(!moves_xyp || !out || num_moves < 1) throw std::invalid_argument("kgb_test_repetition_bound: bad argument");
    repBoundTest(x_len, y_len, num_moves, bound, moves_xyp, out);
  });
}

KGB_API int kgb_test_root_policy_noise(const char* seed_string, int x_len, int y_len, int policy_size, int turn_number, int noise_enabled,
                                       double concentration, double weight, double temperature, double temperature_early, double halflife,
                                       const float* policy_in, float* policy_out) {
  return guarded([&] {
    if(!seed_string || !policy_in || !policy_out || policy_size < 1 || policy_size > 362) throw std::invalid_argument("kgb_test_root_policy_noise: bad argument");
    rootNoiseTest(seed_string, x_len, y_len, policy_size, turn_number, noise_enabled, concentration, weight, temperature, temperature_early, halflife,
                  policy_in, policy_out);
  });
}

KGB_API int kgb_selfplay_create(kgb_handle* handle, const kgb_selfplay_config* config, kgb_selfplay** out) {
  return guarded([&] {
    if(!handle || !config || !out) throw std::invalid_argument("kgb_selfplay_create: NULL argument");
    if(config->num_games > handle->maxBatch) throw std::invalid_argument("kgb_selfplay_create: num_games exceeds the handle's max_batch_size");
    if(!handle->nhwc) throw std::invalid_argument("kgb_selfplay_create: the handle must be created with inputs_nhwc = 1");
    if(handle->model->numInputChannels != 22 || handle->model->numInputGlobalChannels != 19)
      throw std::invalid_argument("kgb_selfplay_create: the device loop writes V7 features (22 spatial, 19 global)");
    CK(cudaSetDevice(handle->device));
    std::unique_ptr<kgb_selfplay> sp(new kgb_selfplay());
    sp->h = handle;
    sp->n = config->num_games;
    sp->fakeNN = config->debug_fake_nn != 0;
    SelfplayNNBuffers nn{handle->dSpatial, handle->dGlobal, handle->dOptimism, handle->dSymmetry, handle->dPolicy, handle->dValue, handle->dScore, handle->dOwnership,
                         (double)handle->model->scoreMeanMultiplier, (double)handle->model->scoreStdevMultiplier, (double)handle->model->leadMultiplier};
    sp->impl = selfplayCreate(*config, handle->L.X, handle->L.Y, nn, handle->stream);
    *out = sp.release();
  });
}

KGB_API void kgb_selfplay_free(kgb_selfplay* sp) {
  if(!sp) return;
  if(sp->stepGraph) cudaGraphExecDestroy(sp->stepGraph);
  selfplayDestroy(sp->impl);
  delete sp;
}

KGB_API int kgb_selfplay_run(kgb_selfplay* sp, int steps) {
  return guarded([&] {
    if(!sp || steps < 0) throw std::invalid_argument("kgb_selfplay_run: bad argument");
    kgb_handle* h = sp->h;
    CK(cudaSetDevice(h->device));
    if(!sp->stepGraph) {
      cudaGraph_t graph = nullptr;
      CK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
      try { selfplayStepLaunches(sp, h->stream); }
      catch(...) { cudaStreamEndCapture(h->stream, &graph); if(graph) cudaGraphDestroy(graph); throw; }
      CK(cudaStreamEndCapture(h->stream, &graph));
      CK(cudaGraphInstantiate(&sp->stepGraph, graph, 0));
      CK(cudaGraphDestroy(graph));
    }
    for(int i = 0; i < steps; i++) CK(cudaGraphLaunch(sp->stepGraph, h->stream));
  });
}

KGB_API int kgb_selfplay_set_search_rand(kgb_selfplay* sp, const char* seed_string) {
  return guarded([&] {
    if(!sp || !seed_string) throw std::invalid_argument("kgb_selfplay_set_search_rand: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplaySetSearchRand(sp->impl, seed_string);
  });
}

KGB_API int kgb_selfplay_random_openings(kgb_selfplay* sp, int max_moves) {
  return guarded([&] {
    if(!sp || max_moves < 0) throw std::invalid_argument("kgb_selfplay_random_openings: bad argument");
    CK(cudaSetDevice(sp->h->device));
    selfplayRandomOpenings(sp->impl, max_moves, sp->h->stream);
  });
}

KGB_API int kgb_selfplay_get_stats(kgb_selfplay* sp, kgb_selfplay_stats* out) {
  return guarded([&] {
    if(!sp || !out) throw std::invalid_argument("kgb_selfplay_get_stats: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadStats(sp->impl, out);
  });
}

KGB_API int kgb_selfplay_get_game(kgb_selfplay* sp, int game, uint8_t* colors, int32_t* info) {
  return guarded([&] {
    if(!sp || !colors || !info) throw std::invalid_argument("kgb_selfplay_get_game: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadGame(sp->impl, game, colors, info);
  });
}

KGB_API int kgb_selfplay_get_root_children(kgb_selfplay* sp, int game, int32_t* visits, float* policy, double* util_sum) {
  return guarded([&] {
    if(!sp || !visits || !policy || !util_sum) throw std::invalid_argument("kgb_selfplay_get_root_children: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadRootChildren(sp->impl, game, visits, policy, util_sum);
  });
}

KGB_API int kgb_selfplay_get_root_value_stats(kgb_selfplay* sp, int game, double* child_stats, double* root_stats) {
  return guarded([&] {
    if(!sp || !child_stats || !root_stats) throw std::invalid_argument("kgb_selfplay_get_root_value_stats: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadRootMoments(sp->impl, game, child_stats, root_stats);
  });
}

KGB_API int kgb_selfplay_set_komi(kgb_selfplay* sp, const float* komi, int also_current_games) {
  return guarded([&] {
    if(!sp || !komi) throw std::invalid_argument("kgb_selfplay_set_komi: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplaySetKomi(sp->impl, komi, also_current_games != 0);
  });
}

KGB_API int kgb_selfplay_set_game_setup(kgb_selfplay* sp, const int32_t* setup, int also_current_games) {
  return guarded([&] {
    if(!sp || !setup) throw std::invalid_argument("kgb_selfplay_set_game_setup: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplaySetGameSetup(sp->impl, setup, also_current_games != 0, sp->h->stream);
  });
}

KGB_API int kgb_selfplay_set_next_search_limits(kgb_selfplay* sp, const int32_t* visits, const uint8_t* plain_root, int also_current_roots) {
  return guarded([&] {
    if(!sp || !visits) throw std::invalid_argument("kgb_selfplay_set_next_search_limits: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplaySetNextSearchLimits(sp->impl, visits, plain_root, also_current_roots != 0, sp->h->stream);
  });
}

KGB_API int kgb_selfplay_get_search_limits(kgb_selfplay* sp, int32_t* visits, uint8_t* plain_root) {
  return guarded([&] {
    if(!sp) throw std::invalid_argument("kgb_selfplay_get_search_limits: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadSearchLimits(sp->impl, visits, plain_root);
  });
}

KGB_API int kgb_selfplay_set_policy_init(kgb_selfplay* sp, const int32_t* num_moves, double temperature, int also_current_games) {
  return guarded([&] {
    if(!sp || !num_moves) throw std::invalid_argument("kgb_selfplay_set_policy_init: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplaySetPolicyInit(sp->impl, num_moves, temperature, also_current_games != 0, sp->h->stream);
  });
}

KGB_API int kgb_selfplay_get_policy_init(kgb_selfplay* sp, int32_t* moves_left, int32_t* count, int16_t* moves, int max_moves) {
  return guarded([&] {
    if(!sp) throw std::invalid_argument("kgb_selfplay_get_policy_init: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadPolicyInit(sp->impl, moves_left, count, moves, max_moves);
  });
}

KGB_API int kgb_selfplay_get_nn_symmetries(kgb_selfplay* sp, int32_t* symmetries) {
  return guarded([&] {
    if(!sp || !symmetries) throw std::invalid_argument("kgb_selfplay_get_nn_symmetries: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadSymmetries(sp->impl, symmetries);
  });
}

KGB_API int kgb_selfplay_get_root_raw_policy_entropy(kgb_selfplay* sp, double* entropy) {
  return guarded([&] {
    if(!sp || !entropy) throw std::invalid_argument("kgb_selfplay_get_root_raw_policy_entropy: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadRootRawEntropy(sp->impl, entropy);
  });
}

KGB_API int kgb_selfplay_get_game_setup(kgb_selfplay* sp, int32_t* current, int32_t* last_finished) {
  return guarded([&] {
    if(!sp) throw std::invalid_argument("kgb_selfplay_get_game_setup: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadGameSetup(sp->impl, current, last_finished);
  });
}

KGB_API int kgb_selfplay_get_komi(kgb_selfplay* sp, float* current, float* last_finished) {
  return guarded([&] {
    if(!sp) throw std::invalid_argument("kgb_selfplay_get_komi: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadKomi(sp->impl, current, last_finished);
  });
}

KGB_API int kgb_selfplay_get_leaf_cache_key(kgb_selfplay* sp, int game, uint64_t* key2) {
  return guarded([&] {
    if(!sp || !key2) throw std::invalid_argument("kgb_selfplay_get_leaf_cache_key: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    unsigned long long k[2];
    selfplayReadLeafKey(sp->impl, game, k);
    key2[0] = k[0]; key2[1] = k[1];
  });
}

KGB_API int kgb_selfplay_clear_nn_cache(kgb_selfplay* sp) {
  return guarded([&] {
    if(!sp) throw std::invalid_argument("kgb_selfplay_clear_nn_cache: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    selfplayClearNNCache(sp->impl, sp->h->stream);
  });
}

KGB_API int kgb_selfplay_release(kgb_selfplay* sp, const uint8_t* games_mask) {
  return guarded([&] {
    if(!sp) throw std::invalid_argument("kgb_selfplay_release: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayRelease(sp->impl, games_mask);
  });
}

KGB_API int kgb_selfplay_get_root_visits(kgb_selfplay* sp, int32_t* visits) {
  return guarded([&] {
    if(!sp || !visits) throw std::invalid_argument("kgb_selfplay_get_root_visits: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadRootVisitsAll(sp->impl, visits);
  });
}

KGB_API int kgb_selfplay_get_root_extra(kgb_selfplay* sp, int game, int32_t* child_node_visits, double* root_nn_stats) {
  return guarded([&] {
    if(!sp || !child_node_visits || !root_nn_stats) throw std::invalid_argument("kgb_selfplay_get_root_extra: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadRootExtra(sp->impl, game, child_node_visits, root_nn_stats);
  });
}

KGB_API int kgb_selfplay_get_last_move(kgb_selfplay* sp, int game, int32_t* info, float* final_score, uint8_t* final_colors, uint8_t* final_area) {
  return guarded([&] {
    if(!sp || !info || !final_score || !final_colors || !final_area) throw std::invalid_argument("kgb_selfplay_get_last_move: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadLastMove(sp->impl, game, info, final_score, final_colors, final_area);
  });
}

KGB_API int kgb_selfplay_get_nn_row(kgb_selfplay* sp, int game, float* spatial, float* global) {
  return guarded([&] {
    if(!sp || !spatial || !global || game < 0 || game >= sp->n) throw std::invalid_argument("kgb_selfplay_get_nn_row: bad argument");
    kgb_handle* h = sp->h;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    const size_t XY = (size_t)h->L.X * h->L.Y;
    CK(cudaMemcpy(spatial, h->dSpatial + (size_t)game * XY * 22, XY * 22 * sizeof(float), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(global, h->dGlobal + (size_t)game * 19, 19 * sizeof(float), cudaMemcpyDeviceToHost));
  });
}

KGB_API int kgb_selfplay_get_root_row(kgb_selfplay* sp, int game, float* spatial, float* global) {
  return guarded([&] {
    if(!sp || !spatial || !global || game < 0 || game >= sp->n) throw std::invalid_argument("kgb_selfplay_get_root_row: bad argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadRootRow(sp->impl, game, spatial, global);
  });
}

KGB_API int kgb_selfplay_get_leaf_path(kgb_selfplay* sp, int game, int32_t* moves_xy, int32_t max_len, int32_t* len_out, int32_t* valid_out) {
  return guarded([&] {
    if(!sp || !moves_xy || !len_out || !valid_out || max_len < 0) throw std::invalid_argument("kgb_selfplay_get_leaf_path: bad argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    *len_out = selfplayReadLeafPath(sp->impl, game, moves_xy, max_len, valid_out);
  });
}

KGB_API int kgb_selfplay_play_moves(kgb_selfplay* sp, const int8_t* moves_xy, int num_moves) {
  return guarded([&] {
    if(!sp || (!moves_xy && num_moves > 0) || num_moves < 0) throw std::invalid_argument("kgb_selfplay_play_moves: bad argument");
    CK(cudaSetDevice(sp->h->device));
    selfplayPlayMoves(sp->impl, moves_xy, num_moves, sp->h->stream);
  });
}

KGB_API int kgb_selfplay_play_moves_game(kgb_selfplay* sp, int game, const int8_t* moves_xy, int num_moves) {
  return guarded([&] {
    if(!sp || game < 0 || (!moves_xy && num_moves > 0) || num_moves < 0) throw std::invalid_argument("kgb_selfplay_play_moves_game: bad argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayPlayMoves(sp->impl, moves_xy, num_moves, sp->h->stream, game);
  });
}

KGB_API int kgb_selfplay_time_tree_kernels(kgb_selfplay* sp, int iters, float* ms_select, float* ms_backup) {
  return guarded([&] {
    if(!sp || iters < 1 || !ms_select || !ms_backup) throw std::invalid_argument("kgb_selfplay_time_tree_kernels: bad argument");
    kgb_handle* h = sp->h;
    CK(cudaSetDevice(h->device));
    cudaEvent_t e0, e1, e2;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1)); CK(cudaEventCreate(&e2));
    float accS = 0.f, accB = 0.f;
    CK(cudaStreamSynchronize(h->stream));
    for(int i = 0; i < iters; i++) {   // the evaluator outputs of the last wave are reused: the trees keep growing normally
      CK(cudaEventRecord(e0, h->stream));
      selfplayLaunchSelect(sp->impl, h->stream);
      CK(cudaEventRecord(e1, h->stream));
      selfplayLaunchBackup(sp->impl, h->stream);
      CK(cudaEventRecord(e2, h->stream));
      CK(cudaStreamSynchronize(h->stream));
      float a = 0.f, b = 0.f;
      CK(cudaEventElapsedTime(&a, e0, e1)); CK(cudaEventElapsedTime(&b, e1, e2));
      accS += a; accB += b;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaEventDestroy(e2);
    *ms_select = accS / iters; *ms_backup = accB / iters;
  });
}

KGB_API int kgb_selfplay_debug_cycles(kgb_selfplay* sp, int64_t* cycles, int clear) {
  return guarded([&] {
    if(!sp || !cycles) throw std::invalid_argument("kgb_selfplay_debug_cycles: NULL argument");
    CK(cudaSetDevice(sp->h->device));
    CK(cudaStreamSynchronize(sp->h->stream));
    selfplayReadDebugCycles(sp->impl, (long long*)cycles, clear != 0);
  });
}

KGB_API int kgb_selfplay_launches_per_step(const kgb_selfplay* sp) { return sp ? sp->h->launchesPerForward + 2 : 0; }

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

KGB_API int kgb_test_board_replay(int x_size, int y_size, int num_boards, int num_moves, int multi_stone_suicide_legal, const int8_t* moves,
                          uint8_t* colors, int8_t* ko, int16_t* caps, uint8_t* lib_class, uint8_t* legal_next, uint64_t* pos_hash, uint8_t* area) {
  return guarded([&] {
    if(!moves || !colors || !ko || !caps || !lib_class || !legal_next || !pos_hash || !area || num_boards < 1 || num_moves < 1)
      throw std::invalid_argument("kgb_test_board_replay: bad argument");
    int count = 0;
    if(cudaGetDeviceCount(&count) != cudaSuccess || count == 0) throw CudaFailure("libkgb200: no CUDA device is visible");
    boardReplay(x_size, y_size, num_boards, num_moves, multi_stone_suicide_legal, moves, colors, ko, caps, lib_class, legal_next, pos_hash, area);
  });
}

}  // extern "C"
