// fp32 support kernels of the NN evaluator (everything that is not the wgmma convolution).  HBM/latency-bound byte
// shuffling and small reductions: coalesced along channels, one pass over the data each.
#include "kgb_kernels.cuh"

namespace kgb {

// SymmetryHelpers copyWithSymmetry index map (nninputs.cpp:529-575): destination flat index (pitch W) of source (y,x).
__device__ __forceinline__ int symIndex(int y, int x, int H, int W, int sym, bool reverse) {
  bool transpose = (sym & 4) != 0 && H == W;
  bool flipX = (sym & 2) != 0, flipY = (sym & 1) != 0;
  if(transpose && !reverse) { bool t = flipX; flipX = flipY; flipY = t; }
  int hs = W, ws = 1, hb = 0, wb = 0;
  if(flipY) { hb = (H - 1) * hs; hs = -hs; }
  if(flipX) { wb = (W - 1) * ws; ws = -ws; }
  if(transpose) { int t = hs; hs = ws; ws = t; }
  return hb + y * hs + wb + x * ws;
}

// ------------------------------------------------------------------------------------------------------------
// The row plan (RowPlan, kgb_kernels.cuh): the boxes, one warp per image, then the layout in one block
// ------------------------------------------------------------------------------------------------------------
__global__ void planBoxKernel(const float* __restrict__ spatial, int n, int C, int nhwc, const int* __restrict__ symmetry, Layout L,
                              RowPlan rp) {
  const int img = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if(img >= n) return;
  int4 b = make_int4(0, 0, L.X, L.Y);
  if(rp.ragged) {
    // the box of the mask's non-zero positions where packInputKernel puts them, i.e. after the symmetry
    const int XY = L.X * L.Y, sym = symmetry ? symmetry[img] : 0;
    const float* src = spatial + (size_t)img * C * XY;
    int x0 = L.X, y0 = L.Y, x1 = -1, y1 = -1;
    for(int pos = lane; pos < XY; pos += 32) {
      if((nhwc ? src[(size_t)pos * C] : src[pos]) == 0.0f) continue;
      const int d = symIndex(pos / L.X, pos % L.X, L.Y, L.X, sym, false);
      const int yd = d / L.X, xd = d % L.X;
      x0 = min(x0, xd); x1 = max(x1, xd); y0 = min(y0, yd); y1 = max(y1, yd);
    }
    x0 = __reduce_min_sync(0xffffffffu, x0); y0 = __reduce_min_sync(0xffffffffu, y0);
    x1 = __reduce_max_sync(0xffffffffu, x1); y1 = __reduce_max_sync(0xffffffffu, y1);
    b = x1 < 0 ? make_int4(0, 0, 0, 0) : make_int4(x0, y0, x1 - x0 + 1, y1 - y0 + 1);
  }
  if(lane == 0) rp.box[img] = b;
}

static constexpr int PLAN_THREADS = 1024, PLAN_CHUNK = 2048, PLAN_MAX_W = 64;

__global__ void __launch_bounds__(PLAN_THREADS) planLayoutKernel(int n, Layout L, RowPlan rp) {
  __shared__ int sWidth[PLAN_CHUNK], sRows[PLAN_CHUNK];
  __shared__ int sTotal[PLAN_MAX_W], sSize[PLAN_MAX_W], sStart[PLAN_MAX_W];   // per box width: image rows, segment rows, first row
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, pad = L.pad;
  if(threadIdx.x < PLAN_MAX_W) sTotal[threadIdx.x] = 0;
  // 1. a stable counting sort by width: the warp of width w scans the images in order and gives each of its images the rows of
  //    the earlier ones as its offset in the segment (parked in base until the segments' first rows are known)
  for(int c0 = 0; c0 < n; c0 += PLAN_CHUNK) {
    const int cn = min(PLAN_CHUNK, n - c0);
    __syncthreads();
    for(int k = threadIdx.x; k < cn; k += PLAN_THREADS) {
      const int4 b = rp.box[c0 + k];
      sWidth[k] = b.z;
      sRows[k] = (b.w + pad) * (b.z + pad);
    }
    __syncthreads();
    for(int w = 1 + warp; w <= L.X; w += PLAN_THREADS / 32) {
      int total = sTotal[w];
      for(int k0 = 0; k0 < cn; k0 += 32) {
        const int k = k0 + lane;
        const int rows = k < cn && sWidth[k] == w ? sRows[k] : 0;
        int incl = rows;
#pragma unroll
        for(int o = 1; o < 32; o <<= 1) {
          const int v = __shfl_up_sync(0xffffffffu, incl, o);
          if(lane >= o) incl += v;
        }
        if(rows != 0) rp.base[c0 + k] = total + incl - rows;
        total += __shfl_sync(0xffffffffu, incl, 31);
      }
      if(lane == 0) sTotal[w] = total;
    }
  }
  __syncthreads();
  if(threadIdx.x == 0) {
    int start = 0, segments = 0;
    for(int w = 1; w <= L.X; w++) {
      const int t = sTotal[w];
      sSize[w] = t == 0 ? 0 : (t + pad * (w + pad) + pad + 127) / 128 * 128;
      sStart[w] = start;
      start += sSize[w];
      segments += t != 0;
    }
    rp.stats[0] = start;
    rp.stats[1] = start / 128;
    rp.stats[2] = segments;
  }
  __syncthreads();
  // 2. each segment's tile pitches, each image's first row (packInputKernel fills the row -> image table for the board positions)
  for(int w = 1 + warp; w <= L.X; w += PLAN_THREADS / 32)
    for(int t = sStart[w] / 128 + lane; t < (sStart[w] + sSize[w]) / 128; t += 32) rp.tileWp[t] = w + pad;
  for(int i = threadIdx.x; i < n; i += PLAN_THREADS) {
    const int w = rp.box[i].z;
    rp.base[i] = w > 0 ? sStart[w] + rp.base[i] : -1;
  }
}

cudaError_t launchPlanRows(const float* spatial, int n, int C, bool nhwc, const int* symmetry, Layout L, const RowPlan& rp, cudaStream_t s) {
  if(L.X >= PLAN_MAX_W) return cudaErrorInvalidValue;
  planBoxKernel<<<(n + 7) / 8, 256, 0, s>>>(spatial, n, C, nhwc ? 1 : 0, symmetry, L, rp);
  planLayoutKernel<<<1, PLAN_THREADS, 0, s>>>(n, L, rp);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------
__global__ void packInputKernel(const float* __restrict__ spatial, int n, int C, int nhwc, const int* __restrict__ symmetry,
                                Layout L, RowPlan rp, __half* __restrict__ act, int cin_p, int split, float* __restrict__ mask) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  int XY = L.X * L.Y;
  if(idx >= n * XY) return;
  int img = idx / XY, pos = idx % XY;
  int y = pos / L.X, x = pos % L.X;
  int sym = symmetry ? symmetry[img] : 0;
  int d = symIndex(y, x, L.Y, L.X, sym, false);
  const int r = planRow(rp, L.pad, img, d / L.X, d % L.X);
  if(r < 0) return;   // outside the box: mask 0, and no features to carry
  size_t row = (size_t)r;
  rp.rowImg[row] = img;
  int ld = split ? 2 * cin_p : cin_p;
  __half* dst = act + row * ld;
  const float* src = spatial + (size_t)img * C * XY;
  for(int c = 0; c < cin_p; c++) {
    float v = 0.0f;
    if(c < C) v = nhwc ? src[(size_t)pos * C + c] : src[(size_t)c * XY + pos];
    __half h = __float2half_rn(v);
    dst[c] = h;
    if(split) dst[cin_p + c] = __float2half_rn(v - __half2float(h));
    if(c == 0) mask[row] = v;
  }
}

// The mask's sum over the frame's rows, in the frame layout's order: a position outside the box, like a pad row, adds 0.
__global__ void maskSumKernel(const float* __restrict__ mask, Layout L, RowPlan rp, float* __restrict__ maskSum) {
  int img = blockIdx.x;
  const int4 box = rp.box[img];
  const int base = rp.base[img];
  float s = 0.0f;
  for(int r = threadIdx.x; r < L.P; r += 32) {
    const int yy = r / L.Wp - L.pad, xx = r % L.Wp;
    const int row = yy < 0 || xx >= L.X ? -1 : planRow(box, base, L.pad, yy, xx);
    s += row < 0 ? 0.0f : mask[row];
  }
  for(int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if(threadIdx.x == 0) maskSum[img] = s;
}

cudaError_t launchPackInput(const float* spatial, int n, int C, bool nhwc, const int* symmetry, Layout L, const RowPlan& rp, size_t M,
                            __half* act, int cin_p, int split, float* mask, float* maskSum, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(act, 0, M * cin_p * (split ? 2 : 1) * sizeof(__half), s);
  if(e != cudaSuccess) return e;
  e = cudaMemsetAsync(mask, 0, M * sizeof(float), s);
  if(e != cudaSuccess) return e;
  int total = n * L.X * L.Y;
  packInputKernel<<<(total + 127) / 128, 128, 0, s>>>(spatial, n, C, nhwc ? 1 : 0, symmetry, L, rp, act, cin_p, split, mask);
  maskSumKernel<<<n, 32, 0, s>>>(mask, L, rp, maskSum);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------
__global__ void matMulNCKernel(const float* __restrict__ in, int ldi, const float* __restrict__ W, const float* __restrict__ bias,
                               int cin, int cout, int act, float* __restrict__ out, int ldo, bool accumulate) {
  extern __shared__ float sIn[];
  int img = blockIdx.x;
  for(int k = threadIdx.x; k < cin; k += blockDim.x) sIn[k] = in[(size_t)img * ldi + k];
  __syncthreads();
  for(int co = threadIdx.x; co < ldo; co += blockDim.x) {
    float v = 0.0f;
    if(co < cout) {
      for(int k = 0; k < cin; k++) v = fmaf(sIn[k], W[(size_t)k * cout + co], v);
      if(bias) v += bias[co];
      v = kgb_activate(v, act);
      if(accumulate) v = out[(size_t)img * ldo + co] + v;
    }
    out[(size_t)img * ldo + co] = v;
  }
}

cudaError_t launchMatMulNC(const float* in, int ldi, const float* W, const float* bias, int n, int cin, int cout, int act, float* out,
                           int ldo, cudaStream_t s, bool accumulate) {
  matMulNCKernel<<<n, 128, cin * sizeof(float), s>>>(in, ldi, W, bias, cin, cout, act, out, ldo, accumulate);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------
// block = (32 channels, 8 row groups); grid = (n, ceil(C/32))
__global__ void gpoolKernel(const void* __restrict__ raw, int rawFp32, int ldr, int c0, int C, const float* __restrict__ bnScale,
                            const float* __restrict__ bnBias, int act, const float* __restrict__ mask,
                            const float* __restrict__ maskSum, Layout L, RowPlan rp, int valueHead, float* __restrict__ pooled) {
  __shared__ float sSum[8][33];
  __shared__ float sMax[8][33];
  int img = blockIdx.x;
  int c = blockIdx.y * 32 + threadIdx.x;
  int rg = threadIdx.y;
  float sum = 0.0f, mx = -1.0f;
  if(c < C) {
    float sc = bnScale[c], bi = bnBias[c];
    const int4 box = rp.box[img];
    const int base = rp.base[img];
    // the frame's positions in the frame layout's row order, whatever the plan
    for(int r = rg; r < L.P; r += 8) {
      // Positions inside the (X,Y) grid but off the actual board contribute 0 to the sum and -1 to the max, as in the
      // reference; pad rows/columns of the layout are not positions at all and are skipped.
      int yy = r / L.Wp - L.pad, xx = r % L.Wp;
      if(yy < 0 || xx >= L.X) continue;
      const int pr = planRow(box, base, L.pad, yy, xx);
      const size_t row = (size_t)(pr < 0 ? 0 : pr);
      const float m = pr < 0 ? 0.0f : mask[row];
      float v = 0.0f;
      if(m == 1.0f) {
        float x = rawFp32 ? reinterpret_cast<const float*>(raw)[row * ldr + c0 + c]
                          : __half2float(reinterpret_cast<const __half*>(raw)[row * ldr + c0 + c]);
        v = kgb_activate(fmaf(x, sc, bi), act);
      }
      sum += v;
      mx = fmaxf(mx, v + (m - 1.0f));
    }
  }
  sSum[rg][threadIdx.x] = sum;
  sMax[rg][threadIdx.x] = mx;
  __syncthreads();
  if(rg == 0 && c < C) {
    for(int i = 1; i < 8; i++) { sum += sSum[i][threadIdx.x]; mx = fmaxf(mx, sMax[i][threadIdx.x]); }
    float div = maskSum[img];
    float sq = sqrtf(div);
    float mean = sum / div;
    float* o = pooled + (size_t)img * 3 * C;
    o[c] = mean;
    o[C + c] = mean * (sq - 14.0f) * 0.1f;
    o[2 * C + c] = valueHead ? mean * ((sq - 14.0f) * (sq - 14.0f) * 0.01f - 0.1f) : mx;
  }
}

cudaError_t launchGPool(const void* raw, int rawFp32, int ldr, int c0, int C, const float* bnScale, const float* bnBias, int act,
                        const float* mask, const float* maskSum, int n, Layout L, const RowPlan& rp, int valueHead, float* pooled,
                        cudaStream_t s) {
  dim3 grid(n, (C + 31) / 32), block(32, 8);
  gpoolKernel<<<grid, block, 0, s>>>(raw, rawFp32, ldr, c0, C, bnScale, bnBias, act, mask, maskSum, L, rp, valueHead, pooled);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------
__global__ void biasActKernel(const void* __restrict__ raw, int rawFp32, int ldr, int C, const float* __restrict__ ncbias, int ldb,
                              const float* __restrict__ bnScale, const float* __restrict__ bnBias, int act,
                              const float* __restrict__ mask, int M, RowPlan rp, __half* __restrict__ actOut, int cp, int split) {
  int groups = cp / 8;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if(idx >= (size_t)M * groups) return;
  int row = (int)(idx / groups);
  if(row >= rp.stats[0]) return;   // past the plan's rows: no tile reads them as its own
  int cb = (int)(idx % groups) * 8;
  float m = mask[row];
  int ld = split ? 2 * cp : cp;
  __align__(16) __half hi[8];
  __align__(16) __half lo[8];
#pragma unroll
  for(int j = 0; j < 8; j++) {
    int c = cb + j;
    float a = 0.0f;
    if(c < C && m == 1.0f) {
      float x = rawFp32 ? reinterpret_cast<const float*>(raw)[(size_t)row * ldr + c]
                        : __half2float(reinterpret_cast<const __half*>(raw)[(size_t)row * ldr + c]);
      if(ncbias) x += ncbias[(size_t)rp.rowImg[row] * ldb + c];
      a = kgb_activate(fmaf(x, bnScale[c], bnBias[c]), act);
    }
    hi[j] = __float2half_rn(a);
    lo[j] = __float2half_rn(a - __half2float(hi[j]));
  }
  *reinterpret_cast<uint4*>(actOut + (size_t)row * ld + cb) = *reinterpret_cast<const uint4*>(hi);
  if(split) *reinterpret_cast<uint4*>(actOut + (size_t)row * ld + cp + cb) = *reinterpret_cast<const uint4*>(lo);
}

cudaError_t launchBiasAct(const void* raw, int rawFp32, int ldr, int C, const float* ncbias, int ldb, const float* bnScale,
                          const float* bnBias, int act, const float* mask, int M, const RowPlan& rp, __half* actOut, int cp, int split,
                          cudaStream_t s) {
  size_t total = (size_t)M * (cp / 8);
  biasActKernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(raw, rawFp32, ldr, C, ncbias, ldb, bnScale, bnBias, act, mask, M, rp,
                                                                actOut, cp, split);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------
__global__ void policyOutKernel(const float* __restrict__ raw, int ldr, int c0, int C, const float* __restrict__ g1bias, int ldb,
                                const float* __restrict__ bnScale, const float* __restrict__ bnBias, int act,
                                const float* __restrict__ Wp2, int cp2, const float* __restrict__ mask,
                                const int* __restrict__ symmetry, const float* __restrict__ optimism, int n, Layout L,
                                RowPlan rp, float* __restrict__ policy) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  int XY = L.X * L.Y;
  if(idx >= n * XY) return;
  int img = idx / XY, pos = idx % XY;
  int y = pos / L.X, x = pos % L.X;
  const int pr = planRow(rp, L.pad, img, y, x);
  const size_t row = (size_t)(pr < 0 ? 0 : pr);
  float m = pr < 0 ? 0.0f : mask[row];
  float l[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  if(m == 1.0f) {
    const float* r = raw + row * ldr + c0;
    const float* b = g1bias + (size_t)img * ldb;
    for(int c = 0; c < C; c++) {
      float h = kgb_activate(fmaf(r[c] + b[c], bnScale[c], bnBias[c]), act);
      for(int k = 0; k < cp2; k++) l[k] = fmaf(h, Wp2[c * cp2 + k], l[k]);
    }
  }
  float p = l[0];
  if(cp2 >= 2) p = l[0] + (l[1] - l[0]) * (optimism ? optimism[img] : 0.0f);
  int sym = symmetry ? symmetry[img] : 0;
  int d = symIndex(y, x, L.Y, L.X, sym, true);
  policy[(size_t)img * (XY + 1) + d] = p;
}

cudaError_t launchPolicyOut(const float* raw, int ldr, int c0, int C, const float* g1bias, int ldb, const float* bnScale,
                            const float* bnBias, int act, const float* Wp2, int cp2, const float* mask, const int* symmetry,
                            const float* optimism, int n, Layout L, const RowPlan& rp, float* policy, cudaStream_t s) {
  int total = n * L.X * L.Y;
  policyOutKernel<<<(total + 127) / 128, 128, 0, s>>>(raw, ldr, c0, C, g1bias, ldb, bnScale, bnBias, act, Wp2, cp2, mask, symmetry,
                                                      optimism, n, L, rp, policy);
  return cudaGetLastError();
}

__global__ void ownershipOutKernel(const float* __restrict__ raw, int ldr, int c0, int C, const float* __restrict__ bnScale,
                                   const float* __restrict__ bnBias, int act, const float* __restrict__ Wown,
                                   const float* __restrict__ mask, const int* __restrict__ symmetry, int n, Layout L,
                                   RowPlan rp, float* __restrict__ ownership) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  int XY = L.X * L.Y;
  if(idx >= n * XY) return;
  int img = idx / XY, pos = idx % XY;
  int y = pos / L.X, x = pos % L.X;
  const int pr = planRow(rp, L.pad, img, y, x);
  const size_t row = (size_t)(pr < 0 ? 0 : pr);
  float o = 0.0f;
  if(pr >= 0 && mask[row] == 1.0f) {
    const float* r = raw + row * ldr + c0;
    for(int c = 0; c < C; c++) o = fmaf(kgb_activate(fmaf(r[c], bnScale[c], bnBias[c]), act), Wown[c], o);
  }
  int sym = symmetry ? symmetry[img] : 0;
  ownership[(size_t)img * XY + symIndex(y, x, L.Y, L.X, sym, true)] = o;
}

cudaError_t launchOwnershipOut(const float* raw, int ldr, int c0, int C, const float* bnScale, const float* bnBias, int act,
                               const float* Wown, const float* mask, const int* symmetry, int n, Layout L, const RowPlan& rp,
                               float* ownership, cudaStream_t s) {
  int total = n * L.X * L.Y;
  ownershipOutKernel<<<(total + 127) / 128, 128, 0, s>>>(raw, ldr, c0, C, bnScale, bnBias, act, Wown, mask, symmetry, n, L, rp, ownership);
  return cudaGetLastError();
}

__global__ void finalizeKernel(const float* __restrict__ passLogits, int ldp, int cp2, const float* __restrict__ optimism,
                               const float* __restrict__ value, const float* __restrict__ sv, int numSV, int version, int n,
                               int policyStride, float* __restrict__ policy, float* __restrict__ valueOut,
                               float* __restrict__ scoreOut) {
  int img = blockIdx.x * blockDim.x + threadIdx.x;
  if(img >= n) return;
  const float* pp = passLogits + (size_t)img * ldp;
  float p = pp[0];
  if(cp2 >= 2) p = pp[0] + (pp[1] - pp[0]) * (optimism ? optimism[img] : 0.0f);
  policy[(size_t)img * policyStride + policyStride - 1] = p;
  for(int k = 0; k < 3; k++) valueOut[img * 3 + k] = value[img * 3 + k];
  const float* s = sv + (size_t)img * numSV;
  float o[6] = {0, 0, 0, 0, 0, 0};
  if(version >= 9) { for(int k = 0; k < 6; k++) o[k] = s[k]; }
  else if(version >= 8) { for(int k = 0; k < 4; k++) o[k] = s[k]; }
  else if(version >= 4) { o[0] = s[0]; o[1] = s[1]; o[2] = s[0]; }
  else { o[0] = s[0]; o[1] = s[0] * s[0]; o[2] = s[0]; }
  for(int k = 0; k < 6; k++) scoreOut[img * 6 + k] = o[k];
}

cudaError_t launchFinalize(const float* passLogits, int ldp, int cp2, const float* optimism, const float* value, const float* sv,
                           int numSV, int version, int n, int policyStride, float* policy, float* valueOut, float* scoreOut,
                           cudaStream_t s) {
  finalizeKernel<<<(n + 63) / 64, 64, 0, s>>>(passLogits, ldp, cp2, optimism, value, sv, numSV, version, n, policyStride, policy,
                                               valueOut, scoreOut);
  return cudaGetLastError();
}

}  // namespace kgb
