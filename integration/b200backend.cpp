// neuralnet/b200backend.cpp - the translation unit a KataGo maintainer adds to select the H100 backend
// (one TU defining `namespace NeuralNet`, cpp/neuralnet/nninterface.h:32-182; template: neuralnet/dummybackend.cpp;
// selected like the others in cpp/CMakeLists.txt:60-172).  Everything forwards 1:1 to the C ABI of libkgb200.so
// (include/kgb200.h); no CUDA, no torch and no weights logic lives on this side of the boundary.
//
// Built for tests/benchmarks by oracle/Makefile.drivers into oracle/_ref/katago_b200 (the UNMODIFIED reference sources
// + this file), see INTEGRATION.md.
#include "../neuralnet/nninterface.h"
#include "../neuralnet/nneval.h"
#include "../neuralnet/nninputs.h"
#include "../neuralnet/modelversion.h"

#include "kgb200.h"

using namespace std;

static void kgbCheck(int rc, const char* what) {
  if(rc != KGB_OK)
    throw StringError(string("H100 backend: ") + what + ": " + kgb_last_error());
}

struct LoadedModel {
  ModelDesc modelDesc;   // parsed by the reference's own loader: NNEvaluator reads it through getModelDesc()
  kgb_model* km;
  LoadedModel(const string& file, const string& expectedSha256) : km(NULL) {
    ModelDesc::loadFromFileMaybeGZipped(file, modelDesc, expectedSha256);
    kgbCheck(kgb_model_load_file(file.c_str(), expectedSha256.c_str(), &km), "loadModelFile");
  }
  ~LoadedModel() { kgb_model_free(km); }
  LoadedModel() = delete;
  LoadedModel(const LoadedModel&) = delete;
  LoadedModel& operator=(const LoadedModel&) = delete;
};

struct ComputeContext {
  kgb_context* kc;
  int nnXLen, nnYLen;
};

struct ComputeHandle {
  kgb_handle* kh;
  int nnXLen, nnYLen, maxBatchSize, modelVersion;
  int numSpatial, numGlobal, numMeta;   // numMeta: 192 for an SGF-metadata (human SL) net, else 0
  bool inputsUseNHWC;
  // contiguous host staging (the C ABI takes plain row-major arrays)
  vector<float> spatial, global, meta, optimism, policy, value, score, ownership;
  vector<int32_t> symmetry;
};

struct InputBuffers {
  int maxBatchSize;
};

void NeuralNet::globalInitialize() { kgbCheck(kgb_global_init(), "globalInitialize"); }
void NeuralNet::globalCleanup() { kgb_global_cleanup(); }

void NeuralNet::printDevices() {
  int n = 0;
  kgbCheck(kgb_device_count(&n), "printDevices");
  for(int i = 0; i < n; i++) {
    char name[256]; int ma = 0, mi = 0;
    kgbCheck(kgb_device_name(i, name, sizeof(name), &ma, &mi), "printDevices");
    cout << "Found CUDA device " << i << ": " << name << " (sm_" << ma << mi << ")" << endl;
  }
}

LoadedModel* NeuralNet::loadModelFile(const string& file, const string& expectedSha256) { return new LoadedModel(file, expectedSha256); }
void NeuralNet::freeLoadedModel(LoadedModel* loadedModel) { delete loadedModel; }
const ModelDesc& NeuralNet::getModelDesc(const LoadedModel* loadedModel) { return loadedModel->modelDesc; }

ComputeContext* NeuralNet::createComputeContext(
  const std::vector<int>& gpuIdxs, Logger* logger, int nnXLen, int nnYLen, const string& homeDataDirOverride,
  enabled_t useFP16Mode, const LoadedModel* loadedModel, ConfigParser& cfg
) {
  (void)logger; (void)homeDataDirOverride; (void)cfg;
  ComputeContext* c = new ComputeContext();
  c->nnXLen = nnXLen; c->nnYLen = nnYLen;
  int fp16 = useFP16Mode == enabled_t::False ? 0 : useFP16Mode == enabled_t::True ? 1 : -1;
  int rc = kgb_context_create(gpuIdxs.data(), (int)gpuIdxs.size(), nnXLen, nnYLen, fp16, loadedModel->km, &c->kc);
  if(rc != KGB_OK) { delete c; kgbCheck(rc, "createComputeContext"); }
  return c;
}
void NeuralNet::freeComputeContext(ComputeContext* computeContext) {
  if(computeContext) { kgb_context_free(computeContext->kc); delete computeContext; }
}

ComputeHandle* NeuralNet::createComputeHandle(
  ComputeContext* context, const LoadedModel* loadedModel, Logger* logger, int maxBatchSize, bool requireExactNNLen,
  bool inputsUseNHWC, int gpuIdxForThisThread, int serverThreadIdx
) {
  ComputeHandle* h = new ComputeHandle();
  int rc = kgb_handle_create(context->kc, loadedModel->km, maxBatchSize, requireExactNNLen ? 1 : 0, inputsUseNHWC ? 1 : 0,
                             gpuIdxForThisThread, &h->kh);
  if(rc != KGB_OK) { delete h; kgbCheck(rc, "createComputeHandle"); }
  h->nnXLen = context->nnXLen; h->nnYLen = context->nnYLen;
  h->maxBatchSize = maxBatchSize;
  h->modelVersion = loadedModel->modelDesc.modelVersion;
  h->numSpatial = NNModelVersion::getNumSpatialFeatures(h->modelVersion);
  h->numGlobal = NNModelVersion::getNumGlobalFeatures(h->modelVersion);
  h->numMeta = loadedModel->modelDesc.numInputMetaChannels;
  h->inputsUseNHWC = inputsUseNHWC;
  const size_t xy = (size_t)h->nnXLen * h->nnYLen;
  h->spatial.resize((size_t)maxBatchSize * h->numSpatial * xy);
  h->global.resize((size_t)maxBatchSize * h->numGlobal);
  h->meta.resize((size_t)maxBatchSize * h->numMeta);
  h->optimism.resize(maxBatchSize);
  h->symmetry.resize(maxBatchSize);
  h->policy.resize((size_t)maxBatchSize * (xy + 1));
  h->value.resize((size_t)maxBatchSize * 3);
  h->score.resize((size_t)maxBatchSize * 6);
  h->ownership.resize((size_t)maxBatchSize * xy);
  if(logger != NULL)
    logger->write("H100 backend thread " + Global::intToString(serverThreadIdx) + ": Model version " + Global::intToString(h->modelVersion) +
                  " useFP16 = " + string(kgb_handle_is_fp16(h->kh) ? "true" : "false (3-term split fp16, fp32-equivalent)"));
  return h;
}
void NeuralNet::freeComputeHandle(ComputeHandle* computeHandle) {
  if(computeHandle) { kgb_handle_free(computeHandle->kh); delete computeHandle; }
}
bool NeuralNet::isUsingFP16(const ComputeHandle* computeHandle) { return kgb_handle_is_fp16(computeHandle->kh) != 0; }
bool NeuralNet::setIsWarmup(const ComputeHandle* computeHandle, bool isWarmup) { (void)computeHandle; (void)isWarmup; return false; }

InputBuffers* NeuralNet::createInputBuffers(const LoadedModel* loadedModel, int maxBatchSize, int nnXLen, int nnYLen) {
  (void)loadedModel; (void)nnXLen; (void)nnYLen;
  InputBuffers* b = new InputBuffers();
  b->maxBatchSize = maxBatchSize;
  return b;
}
void NeuralNet::freeInputBuffers(InputBuffers* buffers) { delete buffers; }

void NeuralNet::getOutput(
  ComputeHandle* h, InputBuffers* buffers, int numBatchEltsFilled, NNResultBuf** inputBufs, vector<NNOutput*>& outputs
) {
  const int n = numBatchEltsFilled;
  if(n <= 0 || n > h->maxBatchSize || n > buffers->maxBatchSize) throw StringError("H100 backend: getOutput batch size out of range");
  const size_t xy = (size_t)h->nnXLen * h->nnYLen;
  const size_t spElts = (size_t)h->numSpatial * xy;
  bool anyOwner = false;
  for(int i = 0; i < n; i++) {
    const NNResultBuf* rb = inputBufs[i];
    if(rb->rowSpatialBuf.size() < spElts || rb->rowGlobalBuf.size() < (size_t)h->numGlobal) throw StringError("H100 backend: row buffers too small");
    // NNEvaluator fills rowMetaBuf (SGFMetadata::fillMetadataRow) exactly when the net has an encoder (nneval.cpp:466-484)
    if(rb->hasRowMeta != (h->numMeta > 0) || rb->rowMetaBuf.size() < (size_t)h->numMeta) throw StringError("H100 backend: metadata row does not match the net");
    std::copy(rb->rowSpatialBuf.begin(), rb->rowSpatialBuf.begin() + spElts, h->spatial.begin() + i * spElts);
    std::copy(rb->rowGlobalBuf.begin(), rb->rowGlobalBuf.begin() + h->numGlobal, h->global.begin() + (size_t)i * h->numGlobal);
    std::copy(rb->rowMetaBuf.begin(), rb->rowMetaBuf.begin() + h->numMeta, h->meta.begin() + (size_t)i * h->numMeta);
    h->symmetry[i] = rb->symmetry;
    h->optimism[i] = (float)rb->policyOptimism;
    anyOwner = anyOwner || outputs[i]->whiteOwnerMap != NULL;
  }
  if(h->numMeta > 0)
    kgbCheck(kgb_forward_meta(h->kh, n, h->spatial.data(), h->global.data(), h->meta.data(), h->symmetry.data(), h->optimism.data(),
                              h->policy.data(), h->value.data(), h->score.data(), anyOwner ? h->ownership.data() : NULL), "getOutput");
  else
    kgbCheck(kgb_forward(h->kh, n, h->spatial.data(), h->global.data(), h->symmetry.data(), h->optimism.data(), h->policy.data(),
                         h->value.data(), h->score.data(), anyOwner ? h->ownership.data() : NULL), "getOutput");
  for(int i = 0; i < n; i++) {
    NNOutput* o = outputs[i];
    std::copy(h->policy.begin() + i * (xy + 1), h->policy.begin() + (i + 1) * (xy + 1), o->policyProbs);
    o->whiteWinProb = h->value[i * 3]; o->whiteLossProb = h->value[i * 3 + 1]; o->whiteNoResultProb = h->value[i * 3 + 2];
    const float* s = &h->score[(size_t)i * 6];
    o->whiteScoreMean = s[0]; o->whiteScoreMeanSq = s[1]; o->whiteLead = s[2]; o->varTimeLeft = s[3];
    o->shorttermWinlossError = s[4]; o->shorttermScoreError = s[5];
    if(o->whiteOwnerMap != NULL) std::copy(h->ownership.begin() + i * xy, h->ownership.begin() + (i + 1) * xy, o->whiteOwnerMap);
  }
}

// FOR TESTING ---------------------------------------------------------------------------------------------------------
bool NeuralNet::testEvaluateConv(
  const ConvLayerDesc* desc, int batchSize, int nnXLen, int nnYLen, bool useFP16, bool useNHWC,
  const std::vector<float>& inputBuffer, std::vector<float>& outputBuffer
) {
  if(desc->dilationX != 1 || desc->dilationY != 1) return false;
  const int ky = desc->convYSize, kx = desc->convXSize, ic = desc->inChannels, oc = desc->outChannels;
  const size_t xy = (size_t)nnXLen * nnYLen;
  // ConvLayerDesc::weights is (oc,ic,y,x) (desc.cpp:110-155); the C ABI takes the model-file order (y,x,ic,oc)
  vector<float> w((size_t)ky * kx * ic * oc);
  for(int o = 0; o < oc; o++) for(int i = 0; i < ic; i++) for(int y = 0; y < ky; y++) for(int x = 0; x < kx; x++)
    w[(((size_t)y * kx + x) * ic + i) * oc + o] = desc->weights[(((size_t)o * ic + i) * ky + y) * kx + x];
  vector<float> in(inputBuffer.size());
  if(useNHWC) in = inputBuffer;
  else for(int n = 0; n < batchSize; n++) for(int c = 0; c < ic; c++) for(size_t p = 0; p < xy; p++)
    in[((size_t)n * xy + p) * ic + c] = inputBuffer[((size_t)n * ic + c) * xy + p];
  vector<float> out((size_t)batchSize * xy * oc);
  kgbCheck(kgb_test_conv(ky, kx, ic, oc, w.data(), batchSize, nnXLen, nnYLen, useFP16 ? 1 : 0, in.data(), out.data()), "testEvaluateConv");
  outputBuffer.resize(out.size());
  if(useNHWC) outputBuffer = out;
  else for(int n = 0; n < batchSize; n++) for(int c = 0; c < oc; c++) for(size_t p = 0; p < xy; p++)
    outputBuffer[((size_t)n * oc + c) * xy + p] = out[((size_t)n * xy + p) * oc + c];
  return true;
}

// Layer-level hooks the H100 backend does not expose (the whole-net and conv hooks are covered): report "unsupported".
bool NeuralNet::testEvaluateBatchNorm(const BatchNormLayerDesc*, int, int, int, bool, bool, const std::vector<float>&, const std::vector<float>&, std::vector<float>&) { return false; }
bool NeuralNet::testEvaluateResidualBlock(const ResidualBlockDesc*, int, int, int, bool, bool, const std::vector<float>&, const std::vector<float>&, std::vector<float>&) { return false; }
bool NeuralNet::testEvaluateGlobalPoolingResidualBlock(const GlobalPoolingResidualBlockDesc*, int, int, int, bool, bool, const std::vector<float>&, const std::vector<float>&, std::vector<float>&) { return false; }
