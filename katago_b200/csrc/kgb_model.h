// Host-side model description for the H100 NN evaluator (product code; does NOT depend on oracle/).
//
// Parses KataGo model files (.bin/.txt, optionally .gz) into plain structs and applies the same load-time weight
// folding as the reference: BN merge (cpp/neuralnet/desc.cpp:282-289) and transformToReduceActivations
// (desc.cpp:627-632, 745-758, 944-1001, 1911-1972, applied at :2810).  The grammar is SURVEY.md Appendix A
// (desc.cpp:110-155, 208-289, 382-403, 451-535, 566-576, 652-666, 783-801, 1444-1562, 1669-1764, 2051-2103,
// 2242-2272, 2441-2574, and the SGF-metadata encoder 1571-1617, 1729-1746).  Transformer nets and RMSNorm trunk tips are rejected
// (out of scope, SURVEY.md §2).
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

namespace kgb {

enum Activation : int { ACT_IDENTITY = 0, ACT_RELU = 1, ACT_MISH = 2, ACT_SILU = 3 };

struct ConvDesc {
  std::string name;
  int ky = 0, kx = 0, cin = 0, cout = 0;
  std::vector<float> w;  // [ky][kx][cin][cout]  (file order)
  void scaleOutputChannels(const std::vector<float>& f);
};

struct BNDesc {
  std::string name;
  int c = 0;
  std::vector<float> scale, bias;  // merged
  void scaleInputChannels(const std::vector<float>& f);
  void extractFactorsAbsLtOne(std::vector<float>& f);
  void extractFactorsAbsLtOneWithInverses(std::vector<float>& f, std::vector<float>& inv);
};

struct MatMulDesc {
  std::string name;
  int cin = 0, cout = 0;
  std::vector<float> w;  // [cin][cout]
  void scaleOutputChannels(const std::vector<float>& f);
};

struct MatBiasDesc {
  std::string name;
  int c = 0;
  std::vector<float> w;
};

// SGF-metadata encoder of human-SL nets (desc.cpp:1571-1617): 192 metadata inputs -> mul1 + bias1, act1 -> mul2 + bias2, act2 -> mul3
// (trunk channels), added to the initial convolution's per-image bias (eigenbackend.cpp:1839-1857, 1927-1932)
struct MetaEncoderDesc {
  std::string name;
  MatMulDesc mul1; MatBiasDesc bias1; int act1 = ACT_RELU;
  MatMulDesc mul2; MatBiasDesc bias2; int act2 = ACT_RELU;
  MatMulDesc mul3;
};

enum BlockKind : int { BLOCK_ORDINARY = 0, BLOCK_GPOOL = 1, BLOCK_NESTED = 2 };

struct BlockDesc {
  BlockKind kind = BLOCK_ORDINARY;
  std::string name;
  // ordinary: preBN/preAct/conv1(regular)/midBN/midAct/conv2(final)
  // gpool:    preBN/preAct/conv1(regular)/gpoolConv/gpoolBN/gpoolAct/gpoolToBias/midBN/midAct/conv2(final)
  // nested:   preBN/preAct/conv1(pre 1x1)/blocks/midBN(post)/midAct(post)/conv2(post 1x1)
  BNDesc preBN; int preAct = ACT_RELU;
  ConvDesc conv1;
  ConvDesc gpoolConv; BNDesc gpoolBN; int gpoolAct = ACT_RELU; MatMulDesc gpoolToBias;
  BNDesc midBN; int midAct = ACT_RELU;
  ConvDesc conv2;
  std::vector<BlockDesc> blocks;
  void transformToReduceActivations();
};

struct ModelDesc {
  std::string name;
  std::string sha256;
  int version = 0;
  int numInputChannels = 0, numInputGlobalChannels = 0;
  // ModelPostProcessParams (desc.cpp:2412-2420 / :2477-2513)
  float tdScoreMultiplier = 20.f, scoreMeanMultiplier = 20.f, scoreStdevMultiplier = 20.f, leadMultiplier = 20.f,
        varianceTimeMultiplier = 40.f, shorttermValueErrorMultiplier = 0.25f, shorttermScoreErrorMultiplier = 30.f;
  int preferPassAliveUnderSuicideRules = 0;
  int numInputMetaChannels = 0;   // 192 when the net has an SGF-metadata encoder (metaEncoderVersion 1), else 0
  // trunk
  int trunkC = 0, midC = 0, regularC = 0, gpoolC = 0;
  ConvDesc initialConv; MatMulDesc initialMatMul;
  MetaEncoderDesc metaEncoder;    // only when numInputMetaChannels > 0
  std::vector<BlockDesc> blocks;
  BNDesc tipBN; int tipAct = ACT_RELU;
  // policy head
  int policyOutChannels = 1;
  ConvDesc p1Conv, g1Conv; BNDesc g1BN; int g1Act = ACT_RELU; MatMulDesc gpoolToBias; BNDesc p1BN; int p1Act = ACT_RELU;
  ConvDesc p2Conv; MatMulDesc gpoolToPass; MatBiasDesc gpoolToPassBias; int passAct = ACT_RELU; MatMulDesc gpoolToPass2;
  // value head
  ConvDesc v1Conv; BNDesc v1BN; int v1Act = ACT_RELU; MatMulDesc v2Mul; MatBiasDesc v2Bias; int v2Act = ACT_RELU;
  MatMulDesc v3Mul; MatBiasDesc v3Bias; MatMulDesc sv3Mul; MatBiasDesc sv3Bias; ConvDesc ownershipConv;

  int numScoreValueChannels() const { return sv3Mul.cout; }
  int64_t convMacsPerPosition() const;  // direct-convolution MACs (SURVEY.md §8d), = sum ky*kx*cin*cout
  int maxConvRadius() const;
  void transformToReduceActivations();
};

// Throws std::runtime_error on malformed input or sha256 mismatch (mirrors StringError in the reference).
std::unique_ptr<ModelDesc> loadModelFile(const std::string& path, const std::string& expectedSha256);
std::unique_ptr<ModelDesc> parseModel(const std::string& data, bool binaryFloats);

std::string sha256Hex(const void* data, size_t len);

}  // namespace kgb
