// TMA / wgmma implicit-GEMM convolution for sm_90a: the trunk hot op of the NN evaluator
// (reference call sites: ConvLayer::apply eigenbackend.cpp:448-701, cudnnConvolutionForward / cublasHgemm
// cudabackend.cpp:788-841, BN+act+mask cudahelpers.cu:1370-2101).
//
// GEMM view:  D[M = batch*P rows, N = cout]  =  sum over k-blocks kb, taps t of  A_t[M, 64] * W_t[64, N]
//   A_t = the activation matrix shifted by the tap's row offset (see kgb_conv.cuh "padded rows").  All taps of one k-block
//         read the SAME rows of A, only shifted: the producer loads ONE halo tile {64 channels, 128 + 2*halo rows}
//         (halo = ry*(X+pad)+rx, 128B swizzle, out-of-range rows zero-filled by TMA) and the consumers read tap t's rows
//         `halo + dy*(X+pad)+dx` onwards out of it with ldmatrix, so A is fetched from L2 once instead of once per tap.  The
//         shift is any number of rows, so A goes to the tensor core from registers: ldmatrix applies the 128B swizzle
//         per row, which a shared-memory descriptor can only do from an 8-row boundary.
//   W   = packed [tap][cout_p][cin_p] fp16 (K-major), box {64, n_tile}, one TMA box per (k-block, tap), read by wgmma
//         through a shared-memory descriptor.
//   D   = fp32 in registers: warpgroup g of the two consumer warpgroups owns rows 64g..64g+63 of the 128-row tile.
//
// One CTA per (128-row, n_tile) tile, 384 threads:
//   warpgroup 0   TMA producer (one lane): A halo tiles into a 2-deep ring, one weight tile per tap into a deeper ring, and the
//                 tile's residual in 32-column slices into a 4-slot ring (the first slices at the start, so they land during the
//                 main loop; the rest as the epilogue frees slots)
//   warpgroups 1-2  ldmatrix + wgmma.mma_async m64 x n_tile x 16, then the fused epilogue straight from the accumulators
// The A fragments are double-buffered in registers: step t+1's ldmatrix runs while step t's wgmma group is still in flight,
// and a consumer waits only for the group before the one it just issued (wait_group 1).  The epilogue reads the residual, the
// mask and the BN constants from shared memory, so no global load sits between its stores.
//
// "split" mode computes a*w ~= ah*wh + al*wh + ah*wl with a = ah + al, w = wh + wl in fp16 (fp32 accumulate):
// fp32-grade accuracy on the fp16 tensor pipe at 3x the MMA count (the backend's useFP16=false mode).
#include "kgb_conv.cuh"
#include "kgb_wgmma.cuh"

namespace kgb {

static constexpr int BLOCK_M = 128;
static constexpr int BLOCK_K = 64;      // fp16 elements = one 128B swizzle row
static constexpr int MAX_STAGES = 8;
static constexpr int SMEM_LIMIT = 227 * 1024;
static constexpr int THREADS = 384;
static constexpr int CONSUMER_WARPS = 8;
static constexpr int RES_COLS = 32;     // columns of one residual slice (every n_tile is a multiple of 32)
static constexpr int RES_SLOTS = 4;     // residual ring: 4 x 16 KB for an fp32 stream, 4 x 8 KB for fp16

// ------------------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  } while(!done);
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
    "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
    ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
template <int N>
__device__ __forceinline__ void fence_acc(float (&d)[N]) {
#pragma unroll
  for(int i = 0; i < N; i++) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }   // the two consumer warpgroups

// wgmma shared-memory descriptor, K-major, 128B swizzle:
//   [0,14) start>>4 | [16,30) LBO>>4 (1, unused for swizzled K-major) | [32,46) SBO>>4 (1024 B = 8 rows x 128 B) | [62,64) 1 = 128B swizzle
// Weight tiles start 1024-aligned, so the base offset [49,52) is 0; +32 bytes (+2 units) steps 16 fp16 along K inside the row.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

struct __align__(8) Bars {
  uint64_t full[MAX_STAGES];    // weight tile landed
  uint64_t empty[MAX_STAGES];   // weight tile consumed by every consumer warp
  uint64_t a_full[2];           // A halo tile landed
  uint64_t a_empty[2];          // A halo tile consumed by all of its taps
  uint64_t r_full[RES_SLOTS];   // residual slice landed
  uint64_t r_empty[RES_SLOTS];  // residual slice consumed by every consumer warp
};

// dynamic smem: [<=1023 B slack][2 x A halo tile][RES_SLOTS x residual slice][stages x weight tile][Bars][mask 128][BN scale N][BN bias N]
static inline int aBufBytes(int a_box_rows) { return (a_box_rows * BLOCK_K * 2 + 1023) / 1024 * 1024; }
// One residual slice = one TMA box of 128 rows x 32 columns.  fp32 rows are 128 B with the 128B swizzle (16-byte chunk c of row r
// at c ^ (r & 7)), fp16 rows 64 B with the 64B swizzle (chunk c at c ^ ((r >> 1) & 3)): either way the 8 rows one warp reads per
// fragment column fall into distinct banks.
__host__ __device__ inline int resSlotBytes(const ConvParams& p) {
  return p.residual != nullptr ? BLOCK_M * RES_COLS * (p.residual_fp32 ? 4 : 2) : 0;
}
__device__ __forceinline__ float2 load_residual(const uint8_t* slot, int r, int c, bool fp32) {
  if(fp32) return *reinterpret_cast<const float2*>(slot + r * 128 + ((((c >> 2) ^ (r & 7)) << 4) | ((c & 3) << 2)));
  return __half22float2(*reinterpret_cast<const __half2*>(slot + r * 64 + ((((c >> 3) ^ ((r >> 1) & 3)) << 4) | ((c & 7) << 1))));
}

// Epilogue of two adjacent columns (col, col+1) of one accumulator row: r = the residual (used when p.residual is set), sc / bi =
// the BN constants of col in shared memory.
__device__ __forceinline__ void epilogue_store(const ConvParams& p, int row, int col, float v0, float v1, float maskv, float2 r,
                                               const float* sc, const float* bi) {
  if(p.ncbias != nullptr) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(p.ncbias + (size_t)(row / p.P) * p.cout_p + col));
    v0 += b.x; v1 += b.y;
  }
  const size_t off = (size_t)row * p.cout_p + col;
  if(p.residual != nullptr) { v0 += r.x; v1 += r.y; }
  if(p.raw_out != nullptr) {
    if(p.raw_fp32) *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.raw_out) + off) = make_float2(v0 * maskv, v1 * maskv);
    else *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(p.raw_out) + off) = __floats2half2_rn(v0 * maskv, v1 * maskv);
  }
  if(p.act_out != nullptr) {
    float a0 = fmaf(v0, sc[0], bi[0]);
    float a1 = fmaf(v1, sc[1], bi[1]);
    if(p.act == 2) {   // mish(x) = x - 2x / (e^x (e^x + 2) + 2): overflow of e gives x, underflow gives 0, no clamps needed
      const float e0 = kgb_ex2(a0 * 1.4426950408889634f), e1 = kgb_ex2(a1 * 1.4426950408889634f);
      a0 = fmaf(-2.0f, a0 * kgb_rcp(fmaf(e0, e0 + 2.0f, 2.0f)), a0);
      a1 = fmaf(-2.0f, a1 * kgb_rcp(fmaf(e1, e1 + 2.0f, 2.0f)), a1);
    }
    else {
      a0 = kgb_activate(a0, p.act);
      a1 = kgb_activate(a1, p.act);
    }
    if(maskv == 0.0f) { a0 = 0.0f; a1 = 0.0f; }   // pad and off-board rows (also guards NaN/inf garbage there)
    const int ldo = p.split ? 2 * p.cout_p : p.cout_p;
    __half* dst = p.act_out + (size_t)row * ldo + col;
    const __half2 h = __floats2half2_rn(a0, a1);
    *reinterpret_cast<__half2*>(dst) = h;
    if(p.split) {
      const float2 hf = __half22float2(h);
      *reinterpret_cast<__half2*>(dst + p.cout_p) = __floats2half2_rn(a0 - hf.x, a1 - hf.y);
    }
  }
}

template <int N>
__global__ void __launch_bounds__(THREADS, 1)
kgb_conv_wg_kernel(const __grid_constant__ CUtensorMap tmapA, const __grid_constant__ CUtensorMap tmapB,
                   const __grid_constant__ CUtensorMap tmapR, const __grid_constant__ ConvParams p, int stages) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr int b_tile_bytes = N * BLOCK_K * 2;               // one tap's weight tile
  const int halo = (p.ky / 2) * p.Wp + (p.kx / 2);            // rows of A above / below the tile that the taps reach
  const int a_tx_bytes = (BLOCK_M + 2 * halo) * BLOCK_K * 2;
  const int a_buf_bytes = (a_tx_bytes + 1023) / 1024 * 1024;
  constexpr int slices = N / RES_COLS;
  const int r_slot_bytes = resSlotBytes(p);
  const uint32_t smem_r = smem_base + 2 * a_buf_bytes;
  const uint32_t smem_b = smem_r + RES_SLOTS * r_slot_bytes;
  uint8_t* const smem = smem_raw + (smem_base - smem_u32(smem_raw));
  Bars* bars = reinterpret_cast<Bars*>(smem + (smem_b - smem_base) + (size_t)stages * b_tile_bytes);
  float* const s_mask = reinterpret_cast<float*>(bars + 1);
  float* const s_scale = s_mask + BLOCK_M;
  float* const s_bias = s_scale + N;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int m0 = (blockIdx.x / p.num_n_tiles) * BLOCK_M;
  const int n0 = (blockIdx.x % p.num_n_tiles) * N;
  const int taps = p.ky * p.kx;
  const int parts = p.split ? 3 : 1;
  const int phases = (p.cin_p / BLOCK_K) * parts;             // one A halo tile per (k-block, split part)

  if(threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmapA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmapB) : "memory");
    if(p.residual != nullptr) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmapR) : "memory");
    for(int s = 0; s < stages; s++) {
      mbar_init(smem_u32(&bars->full[s]), 1);
      mbar_init(smem_u32(&bars->empty[s]), CONSUMER_WARPS);
    }
    for(int s = 0; s < 2; s++) {
      mbar_init(smem_u32(&bars->a_full[s]), 1);
      mbar_init(smem_u32(&bars->a_empty[s]), CONSUMER_WARPS);
    }
    for(int s = 0; s < RES_SLOTS; s++) {
      mbar_init(smem_u32(&bars->r_full[s]), 1);
      mbar_init(smem_u32(&bars->r_empty[s]), CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if(warp < 4) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if(warp == 0 && lane == 0) {
      auto load_residual_slice = [&](int s) {
        const uint32_t rfull = smem_u32(&bars->r_full[s % RES_SLOTS]);
        mbar_arrive_expect_tx(rfull, (uint32_t)r_slot_bytes);
        tma_load_2d(smem_r + (s % RES_SLOTS) * r_slot_bytes, &tmapR, rfull, n0 + s * RES_COLS, m0);
      };
      if(p.residual != nullptr)
        for(int s = 0; s < slices && s < RES_SLOTS; s++) load_residual_slice(s);
      int stage = 0; uint32_t phase = 0;
      for(int ph = 0; ph < phases; ph++) {
        const int kb = ph / parts, part = ph - kb * parts;
        const int colA = kb * BLOCK_K + (part == 1 ? p.cin_p : 0);
        const int colB = kb * BLOCK_K + (part == 2 ? p.cin_p : 0);
        const int abuf = ph & 1;
        mbar_wait(smem_u32(&bars->a_empty[abuf]), ((ph >> 1) & 1) ^ 1);
        const uint32_t afull = smem_u32(&bars->a_full[abuf]);
        mbar_arrive_expect_tx(afull, (uint32_t)a_tx_bytes);
        tma_load_2d(smem_base + abuf * a_buf_bytes, &tmapA, afull, colA, m0 - halo);
        for(int t = 0; t < taps; t++) {
          mbar_wait(smem_u32(&bars->empty[stage]), phase ^ 1);
          const uint32_t full = smem_u32(&bars->full[stage]);
          mbar_arrive_expect_tx(full, (uint32_t)b_tile_bytes);
          tma_load_2d(smem_b + stage * b_tile_bytes, &tmapB, full, colB, t * p.cout_p + n0);
          if(++stage == stages) { stage = 0; phase ^= 1; }
        }
      }
      // slice s reuses the slot of slice s - RES_SLOTS once every consumer warp has read that one
      if(p.residual != nullptr)
        for(int s = RES_SLOTS; s < slices; s++) {
          mbar_wait(smem_u32(&bars->r_empty[s % RES_SLOTS]), (uint32_t)(s / RES_SLOTS - 1) & 1);
          load_residual_slice(s);
        }
    }
    return;
  }

  // ===================== consumers: warpgroup g owns tile rows 64g..64g+63, warp q of it rows 16q..16q+15 =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int g = (warp - 4) >> 2, q = warp & 3;
  const int ry = p.ky / 2, rx = p.kx / 2;
  // ldmatrix.x4 lane roles: matrix j = lane / 8 supplies (rows +0 / +8) x (k 0-7 / 8-15) of a 16 x 16 A fragment
  const int lrow = g * 64 + q * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
  const uint32_t lchunk = (uint32_t)(lane >> 4);
  // the tile's mask and BN constants into shared memory; the epilogue reads them after the consumer barrier below
  {
    const int ct = threadIdx.x - 128;
    if(ct < BLOCK_M) s_mask[ct] = m0 + ct < p.M ? __ldg(p.mask + m0 + ct) : 0.0f;
    if(p.act_out != nullptr)
      for(int i = ct; i < N; i += 32 * CONSUMER_WARPS) { s_scale[i] = __ldg(p.bn_scale + n0 + i); s_bias[i] = __ldg(p.bn_bias + n0 + i); }
  }
  float acc[N / 2];
#pragma unroll
  for(int i = 0; i < N / 2; i++) acc[i] = 0.0f;
  fence_acc(acc);
  // One step = one (k-block, tap): ldmatrix the tap's A fragments into `af` and issue its 4 wgmma as one group.  Steps alternate
  // between two fragment buffers; wait_group 1 after issuing step i means step i-1's group has finished, so its weight stage can be
  // released and its fragment buffer is free for step i+1.  The MMAs reach the accumulators in k-block, tap, k16 order as before.
  int stage = 0, prev_stage = -1, ph = 0, t = 0, dy = -ry, dx = -rx;
  uint32_t phase = 0;
  auto step = [&](uint32_t (&af)[4][4]) {
    const int abuf = ph & 1;
    if(t == 0) mbar_wait(smem_u32(&bars->a_full[abuf]), (ph >> 1) & 1);
    const uint32_t a_base = smem_base + abuf * a_buf_bytes;
    // tap (dy,dx) = the tile's rows shifted by `halo + dy*Wp + dx`; the 128B swizzle puts 16-byte chunk c of row r at c ^ (r & 7)
    const uint32_t r = (uint32_t)(lrow + halo + dy * p.Wp + dx);
#pragma unroll
    for(int k = 0; k < 4; k++) ldmatrix_x4(a_base + r * 128u + (((2u * k + lchunk) ^ (r & 7u)) << 4), af[k]);
    mbar_wait(smem_u32(&bars->full[stage]), phase);
    const uint64_t db = make_smem_desc(smem_b + stage * b_tile_bytes);
    wgmma_fence();
#pragma unroll
    for(int k = 0; k < 4; k++) Wgmma<N>::mma(acc, af[k], db + 2 * k);
    wgmma_commit();
    // the wgmma issue above consumed the fragments of the k-block's last tap, so its A halo tile may be refilled
    if(t == taps - 1) {
      __syncwarp();
      if(lane == 0) mbar_arrive(smem_u32(&bars->a_empty[abuf]));
    }
    wgmma_wait1();
    if(prev_stage >= 0) {
      __syncwarp();
      if(lane == 0) mbar_arrive(smem_u32(&bars->empty[prev_stage]));
    }
    prev_stage = stage;
    if(++stage == stages) { stage = 0; phase ^= 1; }
    if(++dx > rx) { dx = -rx; dy++; }
    if(++t == taps) { t = 0; dy = -ry; ph++; }
  };
  const int steps = phases * taps;
  uint32_t af0[4][4], af1[4][4];
  for(int i = 0; i + 1 < steps; i += 2) {
    step(af0);
    step(af1);
  }
  if(steps & 1) step(af0);
  wgmma_wait0();   // the last group; the producer loads no further weight tile, so its stage is not released
  fence_acc(acc);
  consumer_sync();   // s_mask / s_scale / s_bias written

  // ===================== epilogue straight from the accumulator fragments, one 32-column residual slice at a time =====================
  // acc[4j + 2h + e]: row 16q + lane/4 + 8h of the warpgroup's 64, column 8j + 2*(lane%4) + e
  const int rloc = g * 64 + q * 16 + (lane >> 2);
  const uint8_t* const ring = smem + (smem_r - smem_base);
#pragma unroll
  for(int s = 0; s < slices; s++) {
    const uint8_t* const slot = ring + (s % RES_SLOTS) * r_slot_bytes;
    if(p.residual != nullptr) mbar_wait(smem_u32(&bars->r_full[s % RES_SLOTS]), (uint32_t)(s / RES_SLOTS) & 1);
#pragma unroll
    for(int h = 0; h < 2; h++) {
      const int rl = rloc + 8 * h, row = m0 + rl;
      if(row >= p.M) continue;
      const float maskv = s_mask[rl];
#pragma unroll
      for(int jj = 0; jj < RES_COLS / 8; jj++) {
        const int j = s * (RES_COLS / 8) + jj, lc = 8 * j + 2 * (lane & 3);
        const float2 r = p.residual != nullptr ? load_residual(slot, rl, lc - s * RES_COLS, p.residual_fp32 != 0) : make_float2(0.0f, 0.0f);
        epilogue_store(p, row, n0 + lc, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], maskv, r, s_scale + lc, s_bias + lc);
      }
    }
    if(p.residual != nullptr && s + RES_SLOTS < slices) {
      __syncwarp();
      if(lane == 0) mbar_arrive(smem_u32(&bars->r_empty[s % RES_SLOTS]));
    }
  }
}

cudaError_t convWGInit() {
  for(cudaError_t e : {cudaFuncSetAttribute(kgb_conv_wg_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT),
                       cudaFuncSetAttribute(kgb_conv_wg_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT),
                       cudaFuncSetAttribute(kgb_conv_wg_kernel<96>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT),
                       cudaFuncSetAttribute(kgb_conv_wg_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT),
                       cudaFuncSetAttribute(kgb_conv_wg_kernel<160>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT),
                       cudaFuncSetAttribute(kgb_conv_wg_kernel<192>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT),
                       cudaFuncSetAttribute(kgb_conv_wg_kernel<224>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT),
                       cudaFuncSetAttribute(kgb_conv_wg_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT)})
    if(e != cudaSuccess) return e;
  return cudaSuccess;
}

template <int N>
static cudaError_t launchN(const CUtensorMap& tmapA, const CUtensorMap& tmapB, const CUtensorMap& tmapR, const ConvParams& p, int stages,
                           int smem, cudaStream_t stream) {
  kgb_conv_wg_kernel<N><<<p.num_m_tiles * p.num_n_tiles, THREADS, smem, stream>>>(tmapA, tmapB, tmapR, p, stages);
  return cudaGetLastError();
}

cudaError_t launchConvWG(const CUtensorMap& tmapA, const CUtensorMap& tmapB, const CUtensorMap& tmapR, const ConvParams& p,
                         cudaStream_t stream) {
  const int halo = (p.ky / 2) * p.Wp + (p.kx / 2);
  if(BLOCK_M + 2 * halo > 256) return cudaErrorInvalidValue;  // TMA box limit
  if(p.n_tile % RES_COLS != 0) return cudaErrorInvalidValue;
  const int bTile = p.n_tile * BLOCK_K * 2;
  // the residual ring and the epilogue's mask / BN copies come first; the weight ring gets what is left
  const int fixed = 1024 + 2 * aBufBytes(BLOCK_M + 2 * halo) + RES_SLOTS * resSlotBytes(p) + (int)sizeof(Bars) +
                    (BLOCK_M + 2 * p.n_tile) * (int)sizeof(float);
  int stages = (SMEM_LIMIT - fixed) / bTile;
  if(stages > MAX_STAGES) stages = MAX_STAGES;
  if(stages < 2) return cudaErrorInvalidValue;
  const int smem = fixed + stages * bTile;
  switch(p.n_tile) {
    case 32: return launchN<32>(tmapA, tmapB, tmapR, p, stages, smem, stream);
    case 64: return launchN<64>(tmapA, tmapB, tmapR, p, stages, smem, stream);
    case 96: return launchN<96>(tmapA, tmapB, tmapR, p, stages, smem, stream);
    case 128: return launchN<128>(tmapA, tmapB, tmapR, p, stages, smem, stream);
    case 160: return launchN<160>(tmapA, tmapB, tmapR, p, stages, smem, stream);
    case 192: return launchN<192>(tmapA, tmapB, tmapR, p, stages, smem, stream);
    case 224: return launchN<224>(tmapA, tmapB, tmapR, p, stages, smem, stream);
    case 256: return launchN<256>(tmapA, tmapB, tmapR, p, stages, smem, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace kgb
