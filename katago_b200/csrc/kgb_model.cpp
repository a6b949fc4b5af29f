// Model-file loader for the H100 NN evaluator.  See kgb_model.h for the reference lines this mirrors.
#include "kgb_model.h"

#include <zlib.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <stdexcept>

namespace kgb {

// ------------------------------------------------------------------------------------------------------------
// SHA-256 (FIPS 180-4), used for the optional expectedSha256 check of loadModelFile
// (reference: NeuralNet::loadModelFile -> FileUtils::loadFileIntoString with expectedSha256).
// ------------------------------------------------------------------------------------------------------------
namespace {
inline uint32_t rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
const uint32_t K256[64] = {
  0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01,
  0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc,
  0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147,
  0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
  0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08,
  0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
  0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
void sha256Block(uint32_t st[8], const uint8_t* p) {
  uint32_t w[64];
  for(int i = 0; i < 16; i++)
    w[i] = ((uint32_t)p[4 * i] << 24) | ((uint32_t)p[4 * i + 1] << 16) | ((uint32_t)p[4 * i + 2] << 8) | p[4 * i + 3];
  for(int i = 16; i < 64; i++) {
    uint32_t s0 = rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3);
    uint32_t s1 = rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
    w[i] = w[i - 16] + s0 + w[i - 7] + s1;
  }
  uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
  for(int i = 0; i < 64; i++) {
    uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25);
    uint32_t ch = (e & f) ^ (~e & g);
    uint32_t t1 = h + S1 + ch + K256[i] + w[i];
    uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22);
    uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
    uint32_t t2 = S0 + mj;
    h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
  }
  st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}
}  // namespace

std::string sha256Hex(const void* data, size_t len) {
  uint32_t st[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
  const uint8_t* p = (const uint8_t*)data;
  size_t n = len;
  while(n >= 64) { sha256Block(st, p); p += 64; n -= 64; }
  uint8_t tail[128];
  memset(tail, 0, sizeof(tail));
  memcpy(tail, p, n);
  tail[n] = 0x80;
  size_t tl = (n < 56) ? 64 : 128;
  uint64_t bits = (uint64_t)len * 8;
  for(int i = 0; i < 8; i++) tail[tl - 1 - i] = (uint8_t)(bits >> (8 * i));
  sha256Block(st, tail);
  if(tl == 128) sha256Block(st, tail + 64);
  char buf[65];
  for(int i = 0; i < 8; i++) snprintf(buf + 8 * i, 9, "%08x", st[i]);
  return std::string(buf, 64);
}

// ------------------------------------------------------------------------------------------------------------
// Token reader (desc.cpp:28-90)
// ------------------------------------------------------------------------------------------------------------
namespace {
struct Reader {
  const std::string& d;
  size_t p = 0;
  bool binary;
  Reader(const std::string& data, bool bin) : d(data), binary(bin) {}

  static bool isWs(char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '\v' || c == '\f'; }

  std::string tok(const char* what) {
    size_t n = d.size();
    while(p < n && isWs(d[p])) p++;
    size_t s = p;
    while(p < n && !isWs(d[p])) p++;
    if(s == p) throw std::runtime_error(std::string("model file ended while reading ") + what);
    return d.substr(s, p - s);
  }
  int readInt(const char* what) {
    std::string t = tok(what);
    char* end = nullptr;
    long v = strtol(t.c_str(), &end, 10);
    if(end == t.c_str()) throw std::runtime_error(std::string("failed to parse integer for ") + what + ": '" + t + "'");
    return (int)v;
  }
  float readFloat(const char* what) {
    std::string t = tok(what);
    char* end = nullptr;
    float v = strtof(t.c_str(), &end);
    if(end == t.c_str()) throw std::runtime_error(std::string("failed to parse float for ") + what + ": '" + t + "'");
    return v;
  }
  void readFloats(size_t n, const std::string& name, std::vector<float>& buf) {
    // A malformed or hostile file must not drive the allocation: a binary block cannot hold more floats than bytes remain / 4, a
    // text block needs at least two bytes ("0 ") per float.  Checked BEFORE the resize (and before p + 4 * n could wrap).
    const size_t remaining = p <= d.size() ? d.size() - p : 0;
    if(n > remaining / (binary ? 4 : 2))
      throw std::runtime_error(name + ": the file is too short for the " + std::to_string(n) + " floats its header announces");
    buf.resize(n);
    if(!binary) {
      for(size_t i = 0; i < n; i++) {
        buf[i] = readFloat(name.c_str());
        if(!std::isfinite(buf[i])) throw std::runtime_error(name + ": non-finite weight");
      }
      return;
    }
    // "@BIN@" + n little-endian fp32 (desc.cpp:52-89)
    int skipped = 0;
    while(p < d.size() && d[p] != '@') {
      p++;
      if(++skipped > 100) throw std::runtime_error(name + ": could not read float weights (not a .bin model?)");
    }
    if(p + 5 > d.size() || d.compare(p, 5, "@BIN@") != 0)
      throw std::runtime_error(name + ": did not find expected header for binary float block");
    p += 5;
    if(n > (d.size() - p) / 4) throw std::runtime_error(name + ": did not find the expected number of floats in binary float block");
    memcpy(buf.data(), d.data() + p, 4 * n);  // host is little-endian (x86-64 / aarch64)
    p += 4 * n;
    for(size_t i = 0; i < n; i++)
      if(!std::isfinite(buf[i])) throw std::runtime_error(name + ": non-finite weight");
  }
};

ConvDesc parseConv(Reader& r) {
  ConvDesc c;
  c.name = r.tok("conv name");
  c.ky = r.readInt("convYSize"); c.kx = r.readInt("convXSize");
  c.cin = r.readInt("inChannels"); c.cout = r.readInt("outChannels");
  int dy = r.readInt("dilationY"), dx = r.readInt("dilationX");
  if(c.ky <= 0 || c.kx <= 0 || c.ky % 2 != 1 || c.kx % 2 != 1) throw std::runtime_error(c.name + ": convolution filter sizes must be positive and odd");
  if(c.cin <= 0 || c.cout <= 0) throw std::runtime_error(c.name + ": number of in and out channels must be positive");
  // sane limits before the sizes are multiplied (the product below cannot wrap a size_t once these hold)
  if(c.ky > 15 || c.kx > 15 || c.cin > 16384 || c.cout > 16384) throw std::runtime_error(c.name + ": convolution of unreasonable size (" + std::to_string(c.ky) + "x" + std::to_string(c.kx) + ", " + std::to_string(c.cin) + " -> " + std::to_string(c.cout) + " channels)");
  if(dy != 1 || dx != 1) throw std::runtime_error(c.name + ": dilated convolutions are not supported by the H100 backend");
  r.readFloats((size_t)c.ky * c.kx * c.cin * c.cout, c.name, c.w);
  return c;
}

BNDesc parseBN(Reader& r) {
  BNDesc b;
  b.name = r.tok("bn name");
  b.c = r.readInt("bn numChannels");
  float eps = r.readFloat("bn epsilon");
  int hasScale = r.readInt("bn hasScale"), hasBias = r.readInt("bn hasBias");
  if(b.c < 1) throw std::runtime_error(b.name + ": numChannels < 1");
  if(!(eps > 0) || !std::isfinite(eps)) throw std::runtime_error(b.name + ": epsilon is not positive and finite");
  std::vector<float> mean, var, scale, bias;
  r.readFloats(b.c, b.name, mean);
  r.readFloats(b.c, b.name, var);
  if(hasScale) r.readFloats(b.c, b.name, scale); else scale.assign(b.c, 1.0f);
  if(hasBias) r.readFloats(b.c, b.name, bias); else bias.assign(b.c, 0.0f);
  b.scale.resize(b.c); b.bias.resize(b.c);
  for(int i = 0; i < b.c; i++) {  // desc.cpp:282-289
    b.scale[i] = scale[i] / sqrtf(var[i] + eps);
    b.bias[i] = bias[i] - b.scale[i] * mean[i];
  }
  return b;
}

int parseAct(Reader& r, int version) {  // desc.cpp:382-403
  r.tok("activation name");
  if(version < 11) return ACT_RELU;
  std::string k = r.tok("activation kind");
  if(k == "ACTIVATION_IDENTITY") return ACT_IDENTITY;
  if(k == "ACTIVATION_RELU") return ACT_RELU;
  if(k == "ACTIVATION_MISH") return ACT_MISH;
  if(k == "ACTIVATION_SILU") return ACT_SILU;
  throw std::runtime_error("unknown activation " + k);
}

MatMulDesc parseMatMul(Reader& r) {
  MatMulDesc m;
  m.name = r.tok("matmul name");
  m.cin = r.readInt("matmul inChannels"); m.cout = r.readInt("matmul outChannels");
  if(m.cin <= 0 || m.cout <= 0) throw std::runtime_error(m.name + ": number of in and out channels must be positive");
  if(m.cin > (1 << 20) || m.cout > (1 << 20)) throw std::runtime_error(m.name + ": matrix of unreasonable size");
  r.readFloats((size_t)m.cin * m.cout, m.name, m.w);
  return m;
}

MatBiasDesc parseMatBias(Reader& r) {
  MatBiasDesc m;
  m.name = r.tok("matbias name");
  m.c = r.readInt("matbias numChannels");
  if(m.c <= 0) throw std::runtime_error(m.name + ": numChannels must be positive");
  r.readFloats(m.c, m.name, m.w);
  return m;
}

void parseBlockStack(Reader& r, int version, int n, int expectC, std::vector<BlockDesc>& out);

MetaEncoderDesc parseMetaEncoder(Reader& r, int version, int expectInputs) {  // desc.cpp:1571-1617
  MetaEncoderDesc e;
  e.name = r.tok("sgf metadata encoder name");
  const int numInputs = r.readInt("sgf metadata encoder num input channels");
  if(numInputs != expectInputs)
    throw std::runtime_error(e.name + ": number of in channels (" + std::to_string(numInputs) + ") did not match expected (" +
                             std::to_string(expectInputs) + ")");
  e.mul1 = parseMatMul(r); e.bias1 = parseMatBias(r); e.act1 = parseAct(r, version);
  e.mul2 = parseMatMul(r); e.bias2 = parseMatBias(r); e.act2 = parseAct(r, version);
  e.mul3 = parseMatMul(r);
  if(e.mul1.cout != e.bias1.c)
    throw std::runtime_error(e.name + ": mul1.outChannels (" + std::to_string(e.mul1.cout) + ") != bias1.numChannels (" + std::to_string(e.bias1.c) + ")");
  if(e.mul2.cin != e.mul1.cout)
    throw std::runtime_error(e.name + ": mul2.inChannels (" + std::to_string(e.mul2.cin) + ") != mul1.outChannels (" + std::to_string(e.mul1.cout) + ")");
  if(e.mul2.cout != e.bias2.c)
    throw std::runtime_error(e.name + ": mul2.outChannels (" + std::to_string(e.mul2.cout) + ") != bias2.numChannels (" + std::to_string(e.bias2.c) + ")");
  if(e.mul2.cout != e.mul3.cin)
    throw std::runtime_error(e.name + ": mul2.outChannels (" + std::to_string(e.mul2.cout) + ") != mul3.inChannels (" + std::to_string(e.mul3.cin) + ")");
  return e;
}

BlockDesc parseBlock(Reader& r, int version, const std::string& kind) {
  BlockDesc b;
  b.name = r.tok("block name");
  if(kind == "ordinary_block") {  // desc.cpp:566-576
    b.kind = BLOCK_ORDINARY;
    b.preBN = parseBN(r); b.preAct = parseAct(r, version);
    b.conv1 = parseConv(r);
    b.midBN = parseBN(r); b.midAct = parseAct(r, version);
    b.conv2 = parseConv(r);
    if(b.preBN.c != b.conv1.cin || b.midBN.c != b.conv1.cout || b.midBN.c != b.conv2.cin)
      throw std::runtime_error(b.name + ": residual block channel mismatch");
  }
  else if(kind == "gpool_block") {  // desc.cpp:652-666
    b.kind = BLOCK_GPOOL;
    b.preBN = parseBN(r); b.preAct = parseAct(r, version);
    b.conv1 = parseConv(r);
    b.gpoolConv = parseConv(r);
    b.gpoolBN = parseBN(r); b.gpoolAct = parseAct(r, version);
    b.gpoolToBias = parseMatMul(r);
    b.midBN = parseBN(r); b.midAct = parseAct(r, version);
    b.conv2 = parseConv(r);
    if(b.preBN.c != b.conv1.cin || b.preBN.c != b.gpoolConv.cin || b.gpoolBN.c != b.gpoolConv.cout ||
       b.gpoolToBias.cin != 3 * b.gpoolBN.c || b.gpoolToBias.cout != b.conv1.cout || b.midBN.c != b.conv1.cout ||
       b.midBN.c != b.conv2.cin)
      throw std::runtime_error(b.name + ": gpool block channel mismatch");
  }
  else if(kind == "nested_bottleneck_block") {  // desc.cpp:783-801
    b.kind = BLOCK_NESTED;
    int nInner = r.readInt("nested numBlocks");
    if(nInner < 1) throw std::runtime_error(b.name + ": nested bottleneck block needs >= 1 inner block");
    b.preBN = parseBN(r); b.preAct = parseAct(r, version);
    b.conv1 = parseConv(r);
    parseBlockStack(r, version, nInner, b.conv1.cout, b.blocks);
    b.midBN = parseBN(r); b.midAct = parseAct(r, version);
    b.conv2 = parseConv(r);
    if(b.preBN.c != b.conv1.cin || b.midBN.c != b.conv1.cout || b.midBN.c != b.conv2.cin)
      throw std::runtime_error(b.name + ": nested block channel mismatch");
  }
  else
    throw std::runtime_error("block kind '" + kind + "' is not supported by the H100 backend (transformer nets are out of scope)");
  return b;
}

void parseBlockStack(Reader& r, int version, int n, int expectC, std::vector<BlockDesc>& out) {
  for(int i = 0; i < n; i++) {
    std::string kind = r.tok("block kind");
    out.push_back(parseBlock(r, version, kind));
    const BlockDesc& b = out.back();
    if(b.preBN.c != expectC || b.conv2.cout != expectC)
      throw std::runtime_error(b.name + ": block channels do not match its trunk");
  }
}

void expectZeros(Reader& r, int n, const char* what) {
  for(int i = 0; i < n; i++)
    if(r.readInt(what) != 0) throw std::runtime_error(std::string("unknown/unsupported ") + what);
}

void scaleVec(std::vector<float>& v, const std::vector<float>& f) {
  for(size_t i = 0; i < v.size(); i++) v[i] *= f[i];
}
}  // namespace

// ------------------------------------------------------------------------------------------------------------
// Weight folding (transformToReduceActivations)
// ------------------------------------------------------------------------------------------------------------
void ConvDesc::scaleOutputChannels(const std::vector<float>& f) {
  size_t rows = (size_t)ky * kx * cin;
  for(size_t i = 0; i < rows; i++)
    for(int oc = 0; oc < cout; oc++) w[i * cout + oc] *= f[oc];
}
void MatMulDesc::scaleOutputChannels(const std::vector<float>& f) {
  for(int ic = 0; ic < cin; ic++)
    for(int oc = 0; oc < cout; oc++) w[(size_t)ic * cout + oc] *= f[oc];
}
void BNDesc::scaleInputChannels(const std::vector<float>& f) { scaleVec(scale, f); }  // desc.cpp:291-305
void BNDesc::extractFactorsAbsLtOne(std::vector<float>& f) {                          // desc.cpp:307-325
  f.assign(c, 1.0f);
  for(int i = 0; i < c; i++)
    if(fabsf(scale[i]) < 1.0f) { f[i] = scale[i]; scale[i] = 1.0f; }
}
void BNDesc::extractFactorsAbsLtOneWithInverses(std::vector<float>& f, std::vector<float>& inv) {  // desc.cpp:326-353
  f.assign(c, 1.0f); inv.assign(c, 1.0f);
  for(int i = 0; i < c; i++) {
    if(fabsf(scale[i]) < 0.5f) { f[i] = 0.5f; inv[i] = 2.0f; scale[i] *= 2.0f; }
    else if(fabsf(scale[i]) < 1.0f) { f[i] = scale[i]; inv[i] = 1.0f / scale[i]; scale[i] = 1.0f; }
  }
}

void BlockDesc::transformToReduceActivations() {
  std::vector<float> f, inv;
  if(kind == BLOCK_ORDINARY) {  // desc.cpp:627-632
    midBN.extractFactorsAbsLtOne(f);
    conv1.scaleOutputChannels(f);
  }
  else if(kind == BLOCK_GPOOL) {  // desc.cpp:745-758
    midBN.extractFactorsAbsLtOne(f);
    conv1.scaleOutputChannels(f);
    gpoolToBias.scaleOutputChannels(f);
    gpoolBN.extractFactorsAbsLtOne(f);
    gpoolConv.scaleOutputChannels(f);
  }
  else {  // desc.cpp:944-1001
    midBN.extractFactorsAbsLtOneWithInverses(f, inv);
    conv1.scaleOutputChannels(f);
    for(auto& b : blocks) { b.preBN.scaleInputChannels(inv); b.conv2.scaleOutputChannels(f); }
    for(auto& b : blocks) b.transformToReduceActivations();
  }
}

void ModelDesc::transformToReduceActivations() {  // desc.cpp:1911-1972
  std::vector<float> f, inv;
  tipBN.extractFactorsAbsLtOneWithInverses(f, inv);
  initialConv.scaleOutputChannels(f);
  initialMatMul.scaleOutputChannels(f);
  if(numInputMetaChannels > 0) metaEncoder.mul3.scaleOutputChannels(f);
  for(auto& b : blocks) { b.preBN.scaleInputChannels(inv); b.conv2.scaleOutputChannels(f); }
  for(auto& b : blocks) b.transformToReduceActivations();
}

static void accumulateConvs(const std::vector<BlockDesc>& blocks, int64_t& macs, int& radius) {
  auto add = [&](const ConvDesc& c) {
    macs += (int64_t)c.ky * c.kx * c.cin * c.cout;
    radius = std::max(radius, std::max(c.ky / 2, c.kx / 2));
  };
  for(const auto& b : blocks) {
    add(b.conv1);
    if(b.kind == BLOCK_GPOOL) add(b.gpoolConv);
    if(b.kind == BLOCK_NESTED) accumulateConvs(b.blocks, macs, radius);
    add(b.conv2);
  }
}

int64_t ModelDesc::convMacsPerPosition() const {
  int64_t macs = 0; int radius = 0;
  accumulateConvs(blocks, macs, radius);
  for(const ConvDesc* c : {&initialConv, &p1Conv, &g1Conv, &p2Conv, &v1Conv, &ownershipConv})
    macs += (int64_t)c->ky * c->kx * c->cin * c->cout;
  return macs;
}

int ModelDesc::maxConvRadius() const {
  int64_t macs = 0; int radius = 0;
  accumulateConvs(blocks, macs, radius);
  for(const ConvDesc* c : {&initialConv, &p1Conv, &g1Conv, &p2Conv, &v1Conv, &ownershipConv})
    radius = std::max(radius, std::max(c->ky / 2, c->kx / 2));
  return radius;
}

// ------------------------------------------------------------------------------------------------------------
// Model parse (desc.cpp:2441-2574) and file loading (desc.cpp:2753-2815)
// ------------------------------------------------------------------------------------------------------------
std::unique_ptr<ModelDesc> parseModel(const std::string& data, bool binaryFloats) {
  Reader r(data, binaryFloats);
  std::unique_ptr<ModelDesc> mp(new ModelDesc());
  ModelDesc& m = *mp;
  m.name = r.tok("model name");
  m.version = r.readInt("model version");
  if(m.version < 3) throw std::runtime_error("This neural net is from an extremely old version of KataGo and is not supported. Model version: " + std::to_string(m.version));
  if(m.version > 17) throw std::runtime_error("This neural net requires a newer implementation. Model version: " + std::to_string(m.version));
  const int v = m.version;
  m.numInputChannels = r.readInt("numInputChannels");
  m.numInputGlobalChannels = r.readInt("numInputGlobalChannels");
  if(m.numInputChannels <= 0 || m.numInputGlobalChannels <= 0) throw std::runtime_error(m.name + ": input channel counts must be positive");
  if(v >= 13) {
    float* dst[7] = {&m.tdScoreMultiplier, &m.scoreMeanMultiplier, &m.scoreStdevMultiplier, &m.leadMultiplier,
                     &m.varianceTimeMultiplier, &m.shorttermValueErrorMultiplier, &m.shorttermScoreErrorMultiplier};
    for(int i = 0; i < 7; i++) {
      *dst[i] = r.readFloat("postprocess multiplier");
      if(!(*dst[i] > 0) || !std::isfinite(*dst[i])) throw std::runtime_error(m.name + ": postprocess multipliers must be positive");
    }
  }
  if(v >= 15) {
    int metaEncoderVersion = r.readInt("metaEncoderVersion");   // desc.cpp:2519-2533, modelversion.cpp:83-89
    if(metaEncoderVersion < 0) throw std::runtime_error(m.name + ": model metaEncoderVersion unexpected value: " + std::to_string(metaEncoderVersion));
    if(metaEncoderVersion > 1)
      throw std::runtime_error(m.name + ": model metaEncoderVersion not implemented, you may need a newer KataGo version, value was: " +
                               std::to_string(metaEncoderVersion));
    m.numInputMetaChannels = metaEncoderVersion == 1 ? 192 : 0;
    m.preferPassAliveUnderSuicideRules = r.readInt("preferPassAliveUnderSuicideRules");
    if(m.preferPassAliveUnderSuicideRules != 0 && m.preferPassAliveUnderSuicideRules != 1)
      throw std::runtime_error(m.name + ": model preferPassAliveUnderSuicideRules unexpected value");
    expectZeros(r, 6, "model option");
  }
  // Trunk
  const std::string trunkName = r.tok("trunk name");
  int numBlocks = r.readInt("trunk numBlocks");
  m.trunkC = r.readInt("trunkNumChannels"); m.midC = r.readInt("midNumChannels"); m.regularC = r.readInt("regularNumChannels");
  r.readInt("dilatedNumChannels");
  m.gpoolC = r.readInt("gpoolNumChannels");
  if(v >= 15) {
    int trunkNormKind = r.readInt("trunkNormKind");
    if(trunkNormKind != 0) throw std::runtime_error(m.name + ": RMSNorm trunk tips are not supported by the H100 backend");
    expectZeros(r, 5, "trunk option");
  }
  if(numBlocks < 1) throw std::runtime_error(m.name + ": trunk num blocks must be positive");
  if(m.trunkC <= 0 || m.midC <= 0 || m.regularC <= 0 || m.gpoolC <= 0) throw std::runtime_error(m.name + ": all numbers of channels must be positive");
  m.initialConv = parseConv(r);
  m.initialMatMul = parseMatMul(r);
  if(m.initialConv.cout != m.trunkC || m.initialMatMul.cout != m.trunkC) throw std::runtime_error(m.name + ": initial conv/matmul outChannels != trunkNumChannels");
  if(m.initialConv.cin != m.numInputChannels || m.initialMatMul.cin != m.numInputGlobalChannels) throw std::runtime_error(m.name + ": initial conv/matmul inChannels mismatch");
  if(m.numInputMetaChannels > 0) {
    m.metaEncoder = parseMetaEncoder(r, v, m.numInputMetaChannels);
    const MetaEncoderDesc& e = m.metaEncoder;
    if(e.mul1.cin != m.numInputMetaChannels)  // desc.cpp:1729-1746
      throw std::runtime_error(trunkName + ": " + e.name + " sgfMetadataEncoder.mul1.inChannels (" + std::to_string(e.mul1.cin) +
                               ") != numInputMetaChannels (" + std::to_string(m.numInputMetaChannels) + ")");
    if(e.mul3.cout != m.trunkC)
      throw std::runtime_error(trunkName + ": " + e.name + " sgfMetadataEncoder.mul3.outChannels (" + std::to_string(e.mul3.cout) +
                               ") != trunkNumChannels (" + std::to_string(m.trunkC) + ")");
  }
  parseBlockStack(r, v, numBlocks, m.trunkC, m.blocks);
  m.tipBN = parseBN(r);
  m.tipAct = parseAct(r, v);
  if(m.tipBN.c != m.trunkC) throw std::runtime_error(m.name + ": trunkTipBN.numChannels != trunkNumChannels");
  // Policy head
  r.tok("policy head name");
  if(v >= 17) {
    m.policyOutChannels = r.readInt("policyOutChannels");
    if(m.policyOutChannels != 2 && m.policyOutChannels != 4) throw std::runtime_error(m.name + ": policy head got invalid policyOutChannels");
    expectZeros(r, 3, "policy option");
  }
  else if(v == 16) m.policyOutChannels = 4;
  else if(v >= 12) m.policyOutChannels = 2;
  else m.policyOutChannels = 1;
  m.p1Conv = parseConv(r);
  m.g1Conv = parseConv(r);
  m.g1BN = parseBN(r); m.g1Act = parseAct(r, v);
  m.gpoolToBias = parseMatMul(r);
  m.p1BN = parseBN(r); m.p1Act = parseAct(r, v);
  m.p2Conv = parseConv(r);
  m.gpoolToPass = parseMatMul(r);
  if(v >= 15) {
    m.gpoolToPassBias = parseMatBias(r);
    m.passAct = parseAct(r, v);
    m.gpoolToPass2 = parseMatMul(r);
  }
  if(m.p1Conv.cin != m.trunkC || m.g1Conv.cin != m.trunkC || m.p1Conv.cout != m.p1BN.c || m.g1Conv.cout != m.g1BN.c ||
     m.gpoolToBias.cin != 3 * m.g1BN.c || m.gpoolToBias.cout != m.p1BN.c || m.p2Conv.cin != m.p1BN.c ||
     m.p2Conv.cout != m.policyOutChannels || m.gpoolToPass.cin != 3 * m.g1BN.c)
    throw std::runtime_error(m.name + ": policy head channel mismatch");
  // Value head
  r.tok("value head name");
  if(v >= 17) expectZeros(r, 3, "value option");
  m.v1Conv = parseConv(r);
  m.v1BN = parseBN(r); m.v1Act = parseAct(r, v);
  m.v2Mul = parseMatMul(r); m.v2Bias = parseMatBias(r); m.v2Act = parseAct(r, v);
  m.v3Mul = parseMatMul(r); m.v3Bias = parseMatBias(r);
  m.sv3Mul = parseMatMul(r); m.sv3Bias = parseMatBias(r);
  m.ownershipConv = parseConv(r);
  if(m.v1Conv.cin != m.trunkC || m.v1Conv.cout != m.v1BN.c || m.v2Mul.cin != 3 * m.v1BN.c || m.v2Mul.cout != m.v2Bias.c ||
     m.v3Mul.cin != m.v2Mul.cout || m.v3Mul.cout != 3 || m.v3Bias.c != 3 || m.sv3Mul.cin != m.v2Mul.cout ||
     m.sv3Bias.c != m.sv3Mul.cout || m.ownershipConv.cin != m.v1Conv.cout || m.ownershipConv.cout != 1)
    throw std::runtime_error(m.name + ": value head channel mismatch");
  int expectSV = v >= 9 ? 6 : v >= 8 ? 4 : v >= 4 ? 2 : 1;
  if(m.sv3Mul.cout != expectSV) throw std::runtime_error(m.name + ": sv3Mul.outChannels unexpected for this model version");
  return mp;
}

static bool hasSuffix(const std::string& s, const char* suf) {
  size_t n = strlen(suf);
  return s.size() >= n && s.compare(s.size() - n, n, suf) == 0;
}

std::unique_ptr<ModelDesc> loadModelFile(const std::string& path, const std::string& expectedSha256) {
  try {
    std::ifstream in(path, std::ios::binary);
    if(!in.good()) throw std::runtime_error("could not open file");
    std::string raw((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
    std::string sha = sha256Hex(raw.data(), raw.size());
    if(!expectedSha256.empty()) {
      std::string lowerExp = expectedSha256;
      for(auto& c : lowerExp) c = (char)tolower(c);
      if(lowerExp != sha) throw std::runtime_error("file " + path + " sha256 was " + sha + " which does not match the expected sha256 " + expectedSha256);
    }
    std::string lower = path;
    for(auto& c : lower) c = (char)tolower(c);
    std::unique_ptr<ModelDesc> m;
    if(hasSuffix(lower, ".txt")) m = parseModel(raw, false);
    else if(hasSuffix(lower, ".bin")) m = parseModel(raw, true);
    else if(hasSuffix(lower, ".gz")) {
      // gunzip via zlib
      std::string un;
      z_stream zs;
      memset(&zs, 0, sizeof(zs));
      if(inflateInit2(&zs, 15 + 32) != Z_OK) throw std::runtime_error("zlib init failed");
      zs.next_in = (Bytef*)raw.data();
      zs.avail_in = (uInt)raw.size();
      std::vector<char> chunk(1 << 20);
      int rc;
      do {
        zs.next_out = (Bytef*)chunk.data();
        zs.avail_out = (uInt)chunk.size();
        rc = inflate(&zs, Z_NO_FLUSH);
        if(rc != Z_OK && rc != Z_STREAM_END) { inflateEnd(&zs); throw std::runtime_error("zlib inflate failed (corrupt .gz?)"); }
        un.append(chunk.data(), chunk.size() - zs.avail_out);
      } while(rc != Z_STREAM_END);
      inflateEnd(&zs);
      bool binaryFloats = !hasSuffix(lower, ".txt.gz");
      try { m = parseModel(un, binaryFloats); }
      catch(const std::exception& e) {
        if(!(binaryFloats && !hasSuffix(lower, ".bin.gz"))) throw;
        m = parseModel(un, false);
      }
    }
    else
      throw std::runtime_error("Model file should end with .txt, .bin, .txt.gz, .bin.gz, or possibly just .gz.");
    m->sha256 = sha;
    m->transformToReduceActivations();  // desc.cpp:2810
    return m;
  }
  catch(const std::exception& e) {
    throw std::runtime_error("Error loading or parsing model file " + path + ": " + e.what());
  }
}

}  // namespace kgb
