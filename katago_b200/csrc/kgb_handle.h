// The evaluator handle and the error path of the C ABI, shared by the evaluator (kgb_api.cu) and the device self-play loop
// (kgb_selfplay.cu).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <functional>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/kgb200.h"
#include "kgb_kernels.cuh"
#include "kgb_model.h"

// ------------------------------------------------------------------------------------------------------------
// Error plumbing: every C-ABI function runs its body through guarded(), which turns the exception into the return code
// ------------------------------------------------------------------------------------------------------------
inline thread_local std::string g_lastError;

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
int guarded(F&& f) {
  try {
    f();
    return KGB_OK;
  }
  catch(const CudaFailure& e) { g_lastError = e.what(); return KGB_ERR_CUDA; }
  catch(const std::invalid_argument& e) { g_lastError = e.what(); return KGB_ERR_INVALID; }
  catch(const std::exception& e) { g_lastError = e.what(); return KGB_ERR_IO; }
}

// Captures the launches `launches` enqueues on `s` into a CUDA graph and instantiates it.
cudaGraphExec_t captureGraph(cudaStream_t s, const std::function<void()>& launches);

// ------------------------------------------------------------------------------------------------------------
// The evaluator handle.  Everything it does on the device is ordered on `stream` (weight staging excepted: `copyStream`).
// ------------------------------------------------------------------------------------------------------------
struct kgb_handle {
  int device = 0;
  cudaStream_t stream = nullptr;
  const kgb::ModelDesc* model = nullptr;
  kgb::Layout L{};
  int maxBatch = 0;
  int split = 0;          // fp32-equivalent mode
  bool nhwc = true;
  bool streamTrunkFp32 = true, streamInnerFp32 = false;
  bool fuseBoundaries = false;   // consecutive nested blocks' exit + entry 1x1 as one launch (launchConvPair)
  bool epilogueWG = true;        // launchConvWG may take the epilogue-warpgroup kernel (convEpilogueWG); KGB_EPILOGUE_WG=0 keeps the other
  bool pairEpilogueWG = true;    // launchConvPair may take the exit-epilogue-warpgroup kernel (convPairEpilogueWG); KGB_PAIR_EPILOGUE_WG=0 keeps the other
  std::vector<void*> allocs;
  // inputs / outputs (device, fixed addresses so graphs can be replayed)
  float *dSpatial = nullptr, *dGlobal = nullptr, *dMeta = nullptr, *dOptimism = nullptr;   // dMeta: SGF-metadata nets only
  int* dSymmetry = nullptr;
  float *dPolicy = nullptr, *dValue = nullptr, *dScore = nullptr, *dOwnership = nullptr;
  // pinned staging
  float *hSpatial = nullptr, *hGlobal = nullptr, *hMeta = nullptr, *hOptimism = nullptr, *hPolicy = nullptr, *hValue = nullptr, *hScore = nullptr,
        *hOwnership = nullptr;
  int* hSymmetry = nullptr;
  float *dMask = nullptr, *dMaskSum = nullptr;
  // The rows of the current forward (kgb_kernels.cuh RowPlan), planned on the device at the start of every forward; plan.ragged
  // is off with KGB_RAGGED_ROWS=0 (every image at the full frame).  The single-layer test hooks upload the frame layout once
  // instead (fixedPlan): n*P rows, no gap.
  kgb::RowPlan plan{};
  bool fixedPlan = false;
  size_t planRows(int n) const { return fixedPlan ? (size_t)n * L.P : kgb::planRowCapacity(L, n); }   // rows the row buffers hold
  std::vector<std::function<void(int, cudaStream_t)>> ops;
  int launchesPerForward = 0;
  // Tile flags of the convolution launches (kgb_conv.cuh, launchConvWG): one slot of chainStride() ints per launch, allocated
  // once the ops are emitted.  A forward zeroes them all at its head.
  int* chain = nullptr;
  int chainSlots = 0;
  int chainedLaunches = 0;   // convolution launches per forward that are programmatic dependents of the one before
  int epilogueWGLaunches = 0;   // convolution launches per forward that run with the epilogue warpgroup (convEpilogueWG)
  int pairEpilogueWGLaunches = 0;   // fused block boundaries per forward that run with the exit-epilogue warpgroup (convPairEpilogueWG)
  size_t chainStride() const { return (planRows(maxBatch) + 127) / 128; }
  int* chainFlags(int slot) const { return chain + (size_t)slot * chainStride(); }
  void allocChain() { chain = dalloc<int>((size_t)std::max(chainSlots, 1) * chainStride()); }
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
    CK(cudaMemsetAsync(p, 0, count * sizeof(T), stream));
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
    CK(cudaMemsetAsync(wLive, 0, std::max<size_t>(bytes, 256), stream));
    allocs.push_back(wLive);
    CK(cudaMallocHost((void**)&wHost, std::max<size_t>(bytes, 256)));
    memset(wHost, 0, std::max<size_t>(bytes, 256));
  }
  void wFlushLive() {       // the packed bytes reach the device in one copy
    CK(cudaMemcpyAsync(wLive, wHost, wCursor, cudaMemcpyHostToDevice, stream));
    CK(cudaStreamSynchronize(stream));
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
