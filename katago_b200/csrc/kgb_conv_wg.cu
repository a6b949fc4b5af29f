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
// Persistent CTAs, 384 threads: min(tiles, SMs) CTAs (rounded down to a multiple of num_n_tiles, so that a CTA keeps one n0)
// walk the (128-row, n_tile) tiles blockIdx.x, blockIdx.x + gridDim.x, ... in m-major order.
//   warpgroup 0   TMA producers.  Lane 0 of warp 0: A halo tiles into a 2-deep ring and one weight tile per tap into a deeper
//                 ring.  Lane 0 of warp 1: the residual in 32-column slices into a ring of up to 4 slots.  Every ring keeps its
//                 stage and phase across tiles, so tile i+1's A halo, first weight stages and first residual slices land while
//                 the consumers are still in tile i's epilogue.
//   warpgroups 1-2  ldmatrix + wgmma.mma_async m64 x n_tile x 16, then the fused epilogue from the accumulators into shared
//                 memory, written out by TMA stores that overlap the next tile's main loop.
// The A fragments are double-buffered in registers: step t+1's ldmatrix runs while step t's wgmma group is still in flight,
// and a consumer waits only for the group before the one it just issued (wait_group 1).  The epilogue reads the residual and the
// BN constants from shared memory and the tile's mask from registers, so no global load sits in it.  It writes the raw stream back
// into the residual slice it read (a staging slot when there is no residual) and the activated operand into a 2-slot ring of
// 128 x 32 fp16 slices; each warpgroup stores its 64-row half of a slice with one TMA store per output.
//
// "split" mode computes a*w ~= ah*wh + al*wh + ah*wl with a = ah + al, w = wh + wl in fp16 (fp32 accumulate):
// fp32-grade accuracy on the fp16 tensor pipe at 3x the MMA count (the backend's useFP16=false mode).
#include <algorithm>

#include "kgb_conv.cuh"
#include "kgb_wgmma.cuh"

namespace kgb {

static constexpr int BLOCK_M = 128;
static constexpr int BLOCK_K = 64;      // fp16 elements = one 128B swizzle row
static constexpr int MAX_STAGES = 8;
static constexpr int SMEM_LIMIT = 227 * 1024;
static constexpr int THREADS = 384;
static constexpr int CONSUMER_WARPS = 8;
static constexpr int RES_COLS = 32;     // columns of one epilogue slice (every n_tile is a multiple of 32)
static constexpr int RES_SLOTS = 4;     // stream ring with a residual: 4 x 16 KB for an fp32 stream, 4 x 8 KB for fp16
static constexpr int STAGE_SLOTS = 2;   // stream ring without one (raw output staging only)
static constexpr int ACT_SLOTS = 2;     // activated-operand ring: 128 x 32 fp16 slices (hi and lo in split mode)
static constexpr int ACT_SLICE_BYTES = BLOCK_M * RES_COLS * 2;

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
__device__ __forceinline__ void warpgroup_sync(int g) { asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory"); }
// TMA stores: the generic-proxy writes of every thread are made visible to the async proxy before the barrier that precedes the store
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(map), "r"(src), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------------------
// Chained launches (kgb_conv.cuh, launchConvWG).  The ordering argument, in terms of the PTX memory consistency model
// (PTX ISA, "Memory Consistency Model"):
//   writer  the leader thread that issued a tile part's TMA stores waits for their completion (cp.async.bulk.wait_group 0: the
//           writes are performed), then fence.proxy.async orders those async-proxy writes before its later generic-proxy
//           operations ("Proxies", "Proxy fences"), and red.release.gpu adds to the tile's flag: a release pattern at gpu scope.
//   reader  the producer / residual lane reads the flags with ld.acquire.gpu.  An acquire that observes the value of the writers'
//           releases synchronizes with them ("Release and acquire patterns", "Causality order"), so the stores are visible to
//           the reader's later operations; fence.proxy.async then extends that to the TMA loads it issues next, which run in the
//           async proxy.  What the consumers do with the loaded rows follows the loads through the mbarriers.
// Both RAW (a tile's operand and residual rows) and WAR (a launch overwriting rows that an earlier launch still reads through its
// halo, in place or in a buffer that levels share) are covered by waiting on the previous launch's tiles m-1..m+1 only: that
// launch's tile m' was written after it had waited on tiles m'-1..m'+1 of the launch before it, so by induction a launch k steps
// back has finished every tile within k tiles of m.  A halo is at most 64 rows (BLOCK_M + 2 * halo <= 256), so every reader of
// tile m's rows is one of tiles m-1..m+1 of its launch.  1x1 launches wait on the same three tiles, so that the induction does
// not depend on which launches have a halo.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_add(int* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ int* g_chainError;   // host-mapped sticky word (convWGInit), set when a flag wait gives up

// Leader of a consumer warpgroup: its TMA stores of tile m_tile are all issued; publish them.  Out of line, so that it adds nothing
// to the register pressure of the consumers' accumulators.
__device__ __noinline__ void chain_publish(int* flags, int m_tile) {
  bulk_wait0();
  fence_proxy_async_global();
  red_release_gpu_add(flags + m_tile, 1);
}

// The same for the tile whose stores are all but the last 4 bulk groups the thread has committed
__device__ __noinline__ void chain_publish_before4(int* flags, int m_tile) {
  asm volatile("cp.async.bulk.wait_group 4;" ::: "memory");
  fence_proxy_async_global();
  red_release_gpu_add(flags + m_tile, 1);
}

// Producer lanes, before a tile's loads: the previous launch's tiles m_tile-1..m_tile+1 (of the plan's m_tiles) are written.  The
// wait sleeps between polls, so that a waiter sharing an SM with the previous launch's CTA does not take its issue slots.
__device__ __noinline__ void chain_wait(const int* pred, int parts, int m_tile, int m_tiles) {
  if(pred == nullptr) return;
  for(int t = max(m_tile - 1, 0); t <= min(m_tile + 1, m_tiles - 1); t++) {
    if(ld_acquire_gpu(pred + t) >= parts) continue;
    const uint64_t t0 = globaltimer_ns();
    uint32_t ns = 64;
    while(ld_acquire_gpu(pred + t) < parts) {
      __nanosleep(ns);
      if(ns < 2048) ns *= 2;
      if(globaltimer_ns() - t0 > 4000000000ull) {   // never in a correct chain: record it and go on rather than hang the device
        atomicExch_system(g_chainError, 1);
        break;
      }
    }
  }
  fence_proxy_async_global();
}

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

// The operand rings of kgb_conv_wg_kernel and kgb_conv_wg_epi_kernel
struct __align__(8) RingBars {
  uint64_t full[MAX_STAGES];    // weight tile landed
  uint64_t empty[MAX_STAGES];   // weight tile consumed by every consumer warp
  uint64_t a_full[2];           // A halo tile landed
  uint64_t a_empty[2];          // A halo tile consumed by all of its taps
  int a_wp[2];                  // row pitch of the tile whose A halo tile is in the slot (written before the slot's a_full arrive)
};

struct __align__(8) Bars {
  RingBars ring;
  uint64_t r_full[RES_SLOTS];   // residual slice landed
  uint64_t r_empty[RES_SLOTS];  // residual slice read, and the raw stream written over it stored, by both consumer warpgroups
};

// Rows of A above / below the tile that the widest pitch's taps reach
__host__ __device__ inline int convHalo(const ConvParams& p) { return (p.ky / 2) * p.Wp + (p.kx / 2); }
// dynamic smem: [<=1023 B slack][2 x A halo tile][stream ring][ACT_SLOTS x act slice (x 2 split)][stages x weight tile][Bars]
//               [BN scale N][BN bias N]
__host__ __device__ inline int aBufBytes(int a_box_rows) { return (a_box_rows * BLOCK_K * 2 + 1023) / 1024 * 1024; }

__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) { asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory"); }

// A weight ring of `stages` stages, each filled by one TMA transaction count and emptied by every consumer warp
__device__ __forceinline__ void init_weight_ring(uint64_t* full, uint64_t* empty, int stages) {
  for(int s = 0; s < stages; s++) {
    mbar_init(smem_u32(&full[s]), 1);
    mbar_init(smem_u32(&empty[s]), CONSUMER_WARPS);
  }
}

// Thread 0 of kgb_conv_wg_kernel and kgb_conv_wg_epi_kernel: the tensor maps the launch uses, and the operand rings' barriers
__device__ __forceinline__ void init_operand_rings(RingBars& b, int stages, const ConvParams& p, const CUtensorMap& tmapA,
                                                   const CUtensorMap& tmapB, const CUtensorMap& tmapR, const CUtensorMap& tmapRaw,
                                                   const CUtensorMap& tmapAct) {
  prefetch_tmap(&tmapA);
  prefetch_tmap(&tmapB);
  if(p.residual != nullptr) prefetch_tmap(&tmapR);
  if(p.raw_out != nullptr) prefetch_tmap(&tmapRaw);
  if(p.act_out != nullptr) prefetch_tmap(&tmapAct);
  init_weight_ring(b.full, b.empty, stages);
  for(int s = 0; s < 2; s++) {
    mbar_init(smem_u32(&b.a_full[s]), 1);
    mbar_init(smem_u32(&b.a_empty[s]), CONSUMER_WARPS);
  }
}

// One arrival of the warp on `bar`, once all of its lanes are done with what the barrier guards
__device__ __forceinline__ void warp_arrive(uint32_t bar, int lane) {
  __syncwarp();
  if(lane == 0) mbar_arrive(bar);
}

// Lane 0 of warp 0 of kgb_conv_wg_kernel and kgb_conv_wg_epi_kernel: the A halo tiles into a 2-deep ring at smem_a and one weight
// tile per tap into a ring of `stages` at smem_b, running ahead across tiles as far as the two rings allow.  One A halo tile per
// (k-block, split part): `parts` is 3 in split mode, whose part 1 reads A's lo half and part 2 W's (columns cin_p on), else 1.
template <int N>
__device__ __forceinline__ void produce_operands(const ConvParams& p, RingBars& bars, const CUtensorMap& tmapA, const CUtensorMap& tmapB,
                                                 uint32_t smem_a, uint32_t smem_b, int stages, int tiles, int n0, int parts) {
  constexpr int b_tile_bytes = N * BLOCK_K * 2;   // one tap's weight tile
  const int halo = convHalo(p), taps = p.ky * p.kx, phases = (p.cin_p / BLOCK_K) * parts;
  const int a_tx_bytes = (BLOCK_M + 2 * halo) * BLOCK_K * 2, a_buf_bytes = aBufBytes(BLOCK_M + 2 * halo);
  int stage = 0, ac = 0;
  uint32_t phase = 0;
  for(int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int m0 = (tile / p.num_n_tiles) * BLOCK_M;
    const int wp = __ldg(p.tile_wp + m0 / BLOCK_M);       // loaded here, ahead of the consumers, who read it from the A slot
    chain_wait(p.pred_flags, p.pred_parts, m0 / BLOCK_M, tiles / p.num_n_tiles);
    for(int ph = 0; ph < phases; ph++, ac++) {
      const int kb = ph / parts, part = ph - kb * parts;
      const int colA = kb * BLOCK_K + (part == 1 ? p.cin_p : 0);
      const int colB = kb * BLOCK_K + (part == 2 ? p.cin_p : 0);
      const int abuf = ac & 1;
      mbar_wait(smem_u32(&bars.a_empty[abuf]), ((ac >> 1) & 1) ^ 1);
      const uint32_t afull = smem_u32(&bars.a_full[abuf]);
      bars.a_wp[abuf] = wp;
      mbar_arrive_expect_tx(afull, (uint32_t)a_tx_bytes);
      tma_load_2d(smem_a + abuf * a_buf_bytes, &tmapA, afull, colA, m0 - halo);
      for(int t = 0; t < taps; t++) {
        mbar_wait(smem_u32(&bars.empty[stage]), phase ^ 1);
        const uint32_t full = smem_u32(&bars.full[stage]);
        mbar_arrive_expect_tx(full, (uint32_t)b_tile_bytes);
        tma_load_2d(smem_b + stage * b_tile_bytes, &tmapB, full, colB, t * p.cout_p + n0);
        if(++stage == stages) { stage = 0; phase ^= 1; }
      }
    }
  }
}

// Lane 0 of warp 1: the residual stream's slices, `slices` of RES_COLS columns per tile from column col0, into a ring of `slots`
// slots of `slot_bytes` at smem_r, each slice as two TMA boxes of 64 rows.  In a lane of its own, so that one waiting on a slot
// does not hold up the next tile's operands.  The tiles are m-major, `n_tiles` per 128-row m-tile.
__device__ __forceinline__ void produce_residual(const ConvParams& p, uint64_t* r_full, uint64_t* r_empty, const CUtensorMap& tmapR,
                                                 uint32_t smem_r, int slots, int slot_bytes, int col0, int slices, int tiles, int n_tiles) {
  int rs = 0;
  uint32_t rphase = 0;
  for(int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int m0 = (tile / n_tiles) * BLOCK_M;
    chain_wait(p.pred_flags, p.pred_parts, m0 / BLOCK_M, tiles / n_tiles);
    for(int s = 0; s < slices; s++) {
      mbar_wait(smem_u32(&r_empty[rs]), rphase ^ 1);
      const uint32_t rfull = smem_u32(&r_full[rs]), dst = smem_r + rs * slot_bytes;
      mbar_arrive_expect_tx(rfull, (uint32_t)slot_bytes);
      tma_load_2d(dst, &tmapR, rfull, col0 + s * RES_COLS, m0);
      tma_load_2d(dst + slot_bytes / 2, &tmapR, rfull, col0 + s * RES_COLS, m0 + BLOCK_M / 2);
      if(++rs == slots) { rs = 0; rphase ^= 1; }
    }
  }
}

// A consumer warp's positions in the operand rings, carried across tiles like the producer's
struct RingPos {
  int stage = 0;        // the weight stage of the next step
  uint32_t phase = 0;   // its parity
  int ph = 0;           // A halo tiles taken: the next one is in slot ph & 1 with parity (ph >> 1) & 1
};

// The main loop of one 128-row x N tile for a consumer warp: acc = the sum over the tile's `phases` A halo tiles and the taps.
// ldmatrix.x4 lane roles: matrix j = lane / 8 supplies (rows +0 / +8) x (k 0-7 / 8-15) of a 16 x 16 A fragment, lrow being this
// lane's row of the tile.  One step = one (k-block, tap): ldmatrix the tap's A fragments into `af` and issue its 4 wgmma as one
// group.  Steps alternate between two fragment buffers; wait_group 1 after issuing step i means step i-1's group has finished, so
// its weight stage can be released and its fragment buffer is free for step i+1.  The MMAs reach the accumulators in k-block,
// tap, k16 order.  Returns with the MMAs complete and every stage of the tile released.
template <int N>
__device__ __forceinline__ void conv_main_loop(float (&acc)[N / 2], RingPos& rp, RingBars& bars, const ConvParams& p, uint32_t smem_a,
                                               uint32_t smem_b, int stages, int phases, int lrow, int lane, int halo, int a_buf_bytes) {
  constexpr int b_tile_bytes = N * BLOCK_K * 2;
  const int ry = p.ky / 2, rx = p.kx / 2;
  const uint32_t lchunk = (uint32_t)(lane >> 4);
#pragma unroll
  for(int i = 0; i < N / 2; i++) acc[i] = 0.0f;
  fence_acc(acc);
  // the tap is (dy, dx); the k-block's first tap is (-ry, -rx), its last (ry, rx)
  int wp = 0, prev_stage = -1, dy = -ry, dx = -rx;
  auto step = [&](uint32_t (&af)[4][4]) {
    const int abuf = rp.ph & 1;
    if(dy == -ry && dx == -rx) {
      mbar_wait(smem_u32(&bars.a_full[abuf]), (rp.ph >> 1) & 1);
      wp = bars.a_wp[abuf];
    }
    const uint32_t a_base = smem_a + abuf * a_buf_bytes;
    // tap (dy,dx) = the tile's rows shifted by `halo + dy*wp + dx`; the 128B swizzle puts 16-byte chunk c of row r at c ^ (r & 7)
    const uint32_t r = (uint32_t)(lrow + halo + dy * wp + dx);
#pragma unroll
    for(int k = 0; k < 4; k++) ldmatrix_x4(a_base + r * 128u + (((2u * k + lchunk) ^ (r & 7u)) << 4), af[k]);
    mbar_wait(smem_u32(&bars.full[rp.stage]), rp.phase);
    const uint64_t db = make_smem_desc(smem_b + rp.stage * b_tile_bytes);
    wgmma_fence();
#pragma unroll
    for(int k = 0; k < 4; k++) Wgmma<N>::mma(acc, af[k], db + 2 * k);
    wgmma_commit();
    // the wgmma issue above consumed the fragments of the k-block's last tap, so its A halo tile may be refilled
    if(dy == ry && dx == rx) warp_arrive(smem_u32(&bars.a_empty[abuf]), lane);
    wgmma_wait1();
    if(prev_stage >= 0) warp_arrive(smem_u32(&bars.empty[prev_stage]), lane);
    prev_stage = rp.stage;
    if(++rp.stage == stages) { rp.stage = 0; rp.phase ^= 1; }
    if(++dx > rx) {
      dx = -rx;
      if(++dy > ry) { dy = -ry; rp.ph++; }
    }
  };
  const int steps = phases * (p.ky * p.kx);
  uint32_t af0[4][4], af1[4][4];
  for(int i = 0; i + 1 < steps; i += 2) {
    step(af0);
    step(af1);
  }
  if(steps & 1) step(af0);
  wgmma_wait0();
  fence_acc(acc);
  warp_arrive(smem_u32(&bars.empty[prev_stage]), lane);   // the tile's last stage: the producer is already on the next tile
}
// The stream ring holds the residual, and the raw output written back over it; without a residual it only stages the raw output.
// When both exist they have the same dtype (the launcher checks it).
__host__ __device__ inline bool streamFp32(const ConvParams& p) { return p.residual != nullptr ? p.residual_fp32 != 0 : p.raw_fp32 != 0; }
__host__ __device__ inline int streamSlots(const ConvParams& p) {
  return p.residual != nullptr ? RES_SLOTS : p.raw_out != nullptr ? STAGE_SLOTS : 0;
}
__host__ __device__ inline int streamSlotBytes(const ConvParams& p) { return BLOCK_M * RES_COLS * (streamFp32(p) ? 4 : 2); }
__host__ __device__ inline int actSlotBytes(const ConvParams& p) {
  return p.act_out != nullptr ? ACT_SLICE_BYTES * (p.split ? 2 : 1) : 0;
}
// One slice = 128 rows x 32 columns, moved as two TMA boxes of 64 rows (one per consumer warpgroup).  fp32 rows are 128 B with the
// 128B swizzle (16-byte chunk c of row r at c ^ (r & 7)), fp16 rows 64 B with the 64B swizzle (chunk c at c ^ ((r >> 1) & 3)):
// either way the 8 rows one warp touches per fragment column fall into distinct banks.
__device__ __forceinline__ int slice_offset(int r, int c, bool fp32) {
  if(fp32) return r * 128 + ((((c >> 2) ^ (r & 7)) << 4) | ((c & 3) << 2));
  return r * 64 + ((((c >> 3) ^ ((r >> 1) & 3)) << 4) | ((c & 7) << 1));
}

// What an epilogue does, as bits.  The kernel has one straight-line copy of the slice epilogue for every combination the nets
// launch (epiDispatch below), with these choices made at compile time: a thread's 8 column pairs of a slice then form one run of
// instructions whose shared-memory loads, ex2 and rcp overlap each other.  With the choices read from ConvParams per pair, each
// pair is a chain of branches that waits out its own latencies, with two warps per scheduler to hide them.  Everything else (an
// activation other than mish, in practice test launches) takes the EPI_RUNTIME copy.  Same arithmetic in every copy.
enum EpiFlags {
  EPI_RES = 1,       // + residual, read from the stream slice
  EPI_RAW = 2,       // raw output written to the stream slice
  EPI_FP32 = 4,      // the stream is fp32 (else fp16)
  EPI_MISH = 8,      // BN + mish + mask -> fp16 operand
  EPI_SPLIT = 16,    // the operand also gets its lo half
  EPI_NCBIAS = 32,   // + per-image bias
  EPI_RUNTIME = -1   // every choice read from ConvParams
};
__host__ __device__ inline int epiFlags(const ConvParams& p) {
  if(p.act_out != nullptr && p.act != 2) return EPI_RUNTIME;
  const bool stream = p.residual != nullptr || p.raw_out != nullptr;
  return (p.residual != nullptr ? EPI_RES : 0) | (p.raw_out != nullptr ? EPI_RAW : 0) | (stream && streamFp32(p) ? EPI_FP32 : 0) |
         (p.act_out != nullptr ? EPI_MISH | (p.split ? EPI_SPLIT : 0) : 0) | (p.ncbias != nullptr ? EPI_NCBIAS : 0);
}

// Epilogue of two adjacent columns (col, col+1) of one accumulator row: r = the residual (used when there is one), sc / bi =
// the BN constants of col in shared memory.  raw goes to `raw_dst` in the stream slice, the activated operand to `act_dst` (and
// its lo half to `act_lo_dst` in split mode).
template <int F>
__device__ __forceinline__ void epilogue_store(const ConvParams& p, int row, int col, float v0, float v1, float maskv, float2 r,
                                               const float* sc, const float* bi, uint8_t* raw_dst, uint8_t* act_dst,
                                               uint8_t* act_lo_dst) {
  constexpr bool rt = F == EPI_RUNTIME;
  const bool has_ncbias = rt ? p.ncbias != nullptr : (F & EPI_NCBIAS) != 0;
  const bool has_res = rt ? p.residual != nullptr : (F & EPI_RES) != 0;
  const bool has_raw = rt ? p.raw_out != nullptr : (F & EPI_RAW) != 0;
  const bool raw_fp32 = rt ? p.raw_fp32 != 0 : (F & EPI_FP32) != 0;
  const bool has_act = rt ? p.act_out != nullptr : (F & EPI_MISH) != 0;
  const bool mish = rt ? p.act == 2 : true;
  const bool split = rt ? p.split != 0 : (F & EPI_SPLIT) != 0;
  if(has_ncbias) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(p.ncbias + (size_t)max(__ldg(p.row_img + row), 0) * p.cout_p + col));   // off-board rows are masked
    v0 += b.x; v1 += b.y;
  }
  if(has_res) { v0 += r.x; v1 += r.y; }
  if(has_raw) {
    if(raw_fp32) *reinterpret_cast<float2*>(raw_dst) = make_float2(v0 * maskv, v1 * maskv);
    else *reinterpret_cast<__half2*>(raw_dst) = __floats2half2_rn(v0 * maskv, v1 * maskv);
  }
  if(has_act) {
    float a0 = fmaf(v0, sc[0], bi[0]);
    float a1 = fmaf(v1, sc[1], bi[1]);
    if(mish) {   // mish(x) = x - 2x / (e^x (e^x + 2) + 2): overflow of e gives x, underflow gives 0, no clamps needed
      const float e0 = kgb_ex2(a0 * 1.4426950408889634f), e1 = kgb_ex2(a1 * 1.4426950408889634f);
      a0 = fmaf(-2.0f, a0 * kgb_rcp(fmaf(e0, e0 + 2.0f, 2.0f)), a0);
      a1 = fmaf(-2.0f, a1 * kgb_rcp(fmaf(e1, e1 + 2.0f, 2.0f)), a1);
    }
    else {
      a0 = kgb_activate(a0, p.act);
      a1 = kgb_activate(a1, p.act);
    }
    if(maskv == 0.0f) { a0 = 0.0f; a1 = 0.0f; }   // pad and off-board rows (also guards NaN/inf garbage there)
    const __half2 h = __floats2half2_rn(a0, a1);
    *reinterpret_cast<__half2*>(act_dst) = h;
    if(split) {
      const float2 hf = __half22float2(h);
      *reinterpret_cast<__half2*>(act_lo_dst) = __floats2half2_rn(a0 - hf.x, a1 - hf.y);
    }
  }
}

// One thread's part of slice s of a tile: 2 rows (rloc, rloc + 8) x 4 column pairs out of the accumulators into the slice's
// stream and act slots.
template <int F, int N>
__device__ __forceinline__ void epilogue_slice(const ConvParams& p, const float (&acc)[N / 2], int s, int m0, int n0, int rloc, int lane,
                                               float mask0, float mask1, const float* s_scale, const float* s_bias, uint8_t* slot,
                                               uint8_t* aslot) {
  constexpr bool rt = F == EPI_RUNTIME;
  const bool has_res = rt ? p.residual != nullptr : (F & EPI_RES) != 0;
  const bool s_fp32 = rt ? streamFp32(p) : (F & EPI_FP32) != 0;
#pragma unroll
  for(int h = 0; h < 2; h++) {
    const int rl = rloc + 8 * h, row = m0 + rl;
    if(row >= p.M) continue;   // no ncbias entry for rows past the batch; the TMA stores clip them
    const float maskv = h ? mask1 : mask0;
#pragma unroll
    for(int jj = 0; jj < RES_COLS / 8; jj++) {
      const int j = s * (RES_COLS / 8) + jj, lc = 8 * j + 2 * (lane & 3), c = lc - s * RES_COLS;
      uint8_t* const rp = slot + slice_offset(rl, c, s_fp32);
      uint8_t* const ap = aslot + slice_offset(rl, c, false);
      const float2 r = has_res ? (s_fp32 ? *reinterpret_cast<const float2*>(rp) : __half22float2(*reinterpret_cast<const __half2*>(rp)))
                               : make_float2(0.0f, 0.0f);
      epilogue_store<F>(p, row, n0 + lc, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], maskv, r, s_scale + lc, s_bias + lc, rp, ap,
                        ap + ACT_SLICE_BYTES);
    }
  }
}

// The compile-time copies: what the evaluator launches in fp16 mode (fp16 or fp32 streams) and in fp32-equivalent mode (split
// operands, fp32 streams).  `flags` is the same for every thread of the launch.
template <int N>
__device__ __forceinline__ void epiDispatch(int flags, const ConvParams& p, const float (&acc)[N / 2], int s, int m0, int n0, int rloc,
                                            int lane, float mask0, float mask1, const float* s_scale, const float* s_bias, uint8_t* slot,
                                            uint8_t* aslot) {
#define KGB_EPI(F) case (F): epilogue_slice<(F), N>(p, acc, s, m0, n0, rloc, lane, mask0, mask1, s_scale, s_bias, slot, aslot); break;
  switch(flags) {
    KGB_EPI(EPI_RAW | EPI_FP32)                                     // raw fp32 only: the gpool unit's first conv, the heads' 1x1
    KGB_EPI(EPI_MISH)                                               // the first conv of a residual unit
    KGB_EPI(EPI_RES | EPI_RAW | EPI_MISH)                           // the second conv of a unit, a nested block's post conv
    KGB_EPI(EPI_RES | EPI_RAW | EPI_FP32 | EPI_MISH)
    KGB_EPI(EPI_RES | EPI_MISH)                                     // the trunk's last block: the stream is not kept
    KGB_EPI(EPI_RES | EPI_FP32 | EPI_MISH)
    KGB_EPI(EPI_RAW | EPI_MISH)                                     // a nested block's pre conv
    KGB_EPI(EPI_RAW | EPI_FP32 | EPI_MISH)
    KGB_EPI(EPI_RAW | EPI_MISH | EPI_NCBIAS)                        // the initial conv
    KGB_EPI(EPI_RAW | EPI_FP32 | EPI_MISH | EPI_NCBIAS)
    KGB_EPI(EPI_MISH | EPI_SPLIT)                                   // fp32-equivalent mode
    KGB_EPI(EPI_RES | EPI_RAW | EPI_FP32 | EPI_MISH | EPI_SPLIT)
    KGB_EPI(EPI_RES | EPI_FP32 | EPI_MISH | EPI_SPLIT)
    KGB_EPI(EPI_RAW | EPI_FP32 | EPI_MISH | EPI_SPLIT)
    KGB_EPI(EPI_RAW | EPI_FP32 | EPI_MISH | EPI_SPLIT | EPI_NCBIAS)
    default: epilogue_slice<EPI_RUNTIME, N>(p, acc, s, m0, n0, rloc, lane, mask0, mask1, s_scale, s_bias, slot, aslot);
  }
#undef KGB_EPI
}

template <int N>
__global__ void __launch_bounds__(THREADS, 1)
kgb_conv_wg_kernel(const __grid_constant__ CUtensorMap tmapA, const __grid_constant__ CUtensorMap tmapB,
                   const __grid_constant__ CUtensorMap tmapR, const __grid_constant__ CUtensorMap tmapRaw,
                   const __grid_constant__ CUtensorMap tmapAct, const __grid_constant__ ConvParams p, int stages) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr int b_tile_bytes = N * BLOCK_K * 2;
  constexpr int slices = N / RES_COLS;
  const int r_slots = streamSlots(p), r_slot_bytes = streamSlotBytes(p), act_slot_bytes = actSlotBytes(p);
  const bool s_fp32 = streamFp32(p);
  const int flags = epiFlags(p);
  const int halo = convHalo(p), a_buf_bytes = aBufBytes(BLOCK_M + 2 * halo);
  const uint32_t smem_r = smem_base + 2 * a_buf_bytes;
  const uint32_t smem_act = smem_r + r_slots * r_slot_bytes;
  const uint32_t smem_b = smem_act + ACT_SLOTS * act_slot_bytes;
  uint8_t* const smem = smem_raw + (smem_base - smem_u32(smem_raw));
  Bars* bars = reinterpret_cast<Bars*>(smem + (smem_b - smem_base) + (size_t)stages * b_tile_bytes);
  float* const s_scale = reinterpret_cast<float*>(bars + 1);
  float* const s_bias = s_scale + N;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int tiles = __ldg(p.m_tiles) * p.num_n_tiles;        // the plan's tiles; a CTA past them has nothing to do
  const int n0 = (blockIdx.x % p.num_n_tiles) * N;            // gridDim.x is a multiple of num_n_tiles: one n0 per CTA
  const int parts = p.split ? 3 : 1;

  pdl_launch_dependents();   // the next launch's CTAs take the SMs this grid leaves (they need all of shared memory)
  if(threadIdx.x == 0) {
    init_operand_rings(bars->ring, stages, p, tmapA, tmapB, tmapR, tmapRaw, tmapAct);
    for(int s = 0; s < RES_SLOTS; s++) {
      mbar_init(smem_u32(&bars->r_full[s]), 1);
      mbar_init(smem_u32(&bars->r_empty[s]), 2);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if(warp < 4) {
    // ===================== TMA producers =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if(warp == 0 && lane == 0) produce_operands<N>(p, bars->ring, tmapA, tmapB, smem_base, smem_b, stages, tiles, n0, parts);
    else if(warp == 1 && lane == 0 && p.residual != nullptr)
      produce_residual(p, bars->r_full, bars->r_empty, tmapR, smem_r, RES_SLOTS, r_slot_bytes, n0, slices, tiles, p.num_n_tiles);
    return;
  }

  // ===================== consumers: warpgroup g owns tile rows 64g..64g+63, warp q of it rows 16q..16q+15 =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int g = (warp - 4) >> 2, q = warp & 3;
  const bool leader = q == 0 && lane == 0;    // issues the warpgroup's TMA stores
  const int lrow = g * 64 + q * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
  // acc[4j + 2h + e]: row 16q + lane/4 + 8h of the warpgroup's 64, column 8j + 2*(lane%4) + e
  const int rloc = g * 64 + q * 16 + (lane >> 2);
  // the CTA's BN constants into shared memory, once: every tile of the CTA has the same n0
  if(p.act_out != nullptr)
    for(int i = threadIdx.x - 128; i < N; i += 32 * CONSUMER_WARPS) { s_scale[i] = __ldg(p.bn_scale + n0 + i); s_bias[i] = __ldg(p.bn_bias + n0 + i); }
  consumer_sync();

  RingPos rp;
  int rs = 0, prev_rs = -1, as = 0;
  uint32_t rphase = 0;
  uint8_t* const ring = smem + (smem_r - smem_base);
  uint8_t* const act_ring = smem + (smem_act - smem_base);
  int pending = -1;   // the m-tile whose stores this warpgroup issued last and has not published yet
  for(int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int m0 = (tile / p.num_n_tiles) * BLOCK_M;
    // this thread's two epilogue rows' mask values; the loads complete during the main loop
    const float mask0 = m0 + rloc < p.M ? __ldg(p.mask + m0 + rloc) : 0.0f;
    const float mask1 = m0 + rloc + 8 < p.M ? __ldg(p.mask + m0 + rloc + 8) : 0.0f;
    float acc[N / 2];
    conv_main_loop<N>(acc, rp, bars->ring, p, smem_base, smem_b, stages, (p.cin_p / BLOCK_K) * parts, lrow, lane, halo, a_buf_bytes);
    // the previous tile's stores were issued a whole main loop ago
    if(leader && pending >= 0) chain_publish(p.tile_flags, pending);

    // ===================== epilogue: one 32-column slice at a time, into shared memory, out by TMA stores =====================
#pragma unroll
    for(int s = 0; s < slices; s++) {
      uint8_t* const slot = ring + rs * r_slot_bytes;
      uint8_t* const aslot = act_ring + as * act_slot_bytes;
      if(p.residual != nullptr) mbar_wait(smem_u32(&bars->r_full[rs]), rphase);
      epiDispatch<N>(flags, p, acc, s, m0, n0, rloc, lane, mask0, mask1, s_scale, s_bias, slot, aslot);
      fence_proxy_async();
      if(leader) {
        // the previous slice's stores have read their slots: its act slot (the next slice's) and its stream slot are free again
        bulk_wait_read0();
        if(p.residual != nullptr && prev_rs >= 0) mbar_arrive(smem_u32(&bars->r_empty[prev_rs]));
      }
      warpgroup_sync(g);
      if(leader) {
        const int c0 = n0 + s * RES_COLS, r0 = m0 + g * (BLOCK_M / 2);
        if(p.raw_out != nullptr) tma_store_2d(&tmapRaw, smem_u32(slot + g * (r_slot_bytes / 2)), c0, r0);
        if(p.act_out != nullptr) {
          tma_store_2d(&tmapAct, smem_u32(aslot + g * (ACT_SLICE_BYTES / 2)), c0, r0);
          if(p.split) tma_store_2d(&tmapAct, smem_u32(aslot + ACT_SLICE_BYTES + g * (ACT_SLICE_BYTES / 2)), p.cout_p + c0, r0);
        }
        bulk_commit();
      }
      prev_rs = rs;
      if(++rs >= r_slots) { rs = 0; rphase ^= 1; }   // r_slots is 0 when there is no stream
      as ^= 1;
    }
    pending = m0 / BLOCK_M;
  }
  if(leader && pending >= 0) chain_publish(p.tile_flags, pending);
  if(leader) bulk_wait0();
  pdl_wait();   // this grid completes after the previous one
}

// The widths it is compiled for
#define KGB_WG_SHAPES(X) X(32) X(64) X(96) X(128) X(160) X(192) X(224) X(256)

// ------------------------------------------------------------------------------------------------------------
// Epilogue warpgroup (kgb_conv_wg_epi_kernel, launchConvWG when convEpilogueWG)
// ------------------------------------------------------------------------------------------------------------
// In kgb_conv_wg_kernel both consumer warpgroups leave the main loop together and run the epilogue arithmetic with the tensor
// pipe idle.  Here a fourth warpgroup runs it, 512 threads:
//   warpgroup 0     produce_operands and produce_residual, with one residual slot instead of a ring of four.
//   warpgroups 1-2  conv_main_loop, so every accumulator holds the same bits.  At the end of a tile they wait until the
//                   accumulator tile in shared memory is empty, write their fp32 accumulators into it (N/32 slices of 128 x 32 in
//                   slice_offset's fp32 layout), arrive on t_full and start the next tile at once.
//   warpgroup 3     the epilogue, one thread per tile row: slice by slice it reads its row's 32 accumulators (and the residual),
//                   applies epilogue_store<F> to each column pair exactly as the other kernel does, and writes the raw output
//                   and the activated operand back into the slice it read (raw fp16 in the first 8 KB, the operand in the
//                   second; a raw fp32 output over the whole slice), out by TMA stores.  Once the last stores have read shared
//                   memory it arrives on t_empty, and once they are complete it publishes the tile for the chain.
// Shared memory for N = 192 at the 19x19 pitch: 2 x 22 KB A halo tiles, 96 KB accumulator tile, 8 KB residual slot, 3 x 24 KB
// weight stages.  Registers after setmaxnreg: producers 40, consumers 184 (96 accumulators, 2 x 16 fragments), epilogue 104.
static constexpr int EPI_WG_THREADS = 512;
static constexpr int EPI_WG_MIN_STAGES = 3;
static constexpr int ACC_SLICE_BYTES = BLOCK_M * RES_COLS * 4;

// The epilogues it has a copy of: fp16 mode's 3x3 layers (kgb_conv_wg_kernel's epiDispatch without fp32 streams or split mode),
// and the gpool unit's raw fp32 output, which is written over the accumulator slice it came from.
#define KGB_EPI_WG_FLAGS(X) X(EPI_RAW | EPI_FP32) X(EPI_MISH) X(EPI_RES | EPI_RAW | EPI_MISH) X(EPI_RES | EPI_MISH) \
  X(EPI_RAW | EPI_MISH) X(EPI_RAW | EPI_MISH | EPI_NCBIAS)
// The widths it is compiled for: b28's 256-column tiles would need 128 KB of accumulator tile, and the 64-column copy spills
#define KGB_EPI_WG_SHAPES(X) X(96) X(128) X(160) X(192)

struct __align__(8) EpiBars {
  RingBars ring;
  uint64_t r_full, r_empty;     // residual slice landed / read by the epilogue warpgroup
  uint64_t t_full, t_empty;     // accumulator tile written by every consumer warp / read, and its stores' reads done
};

// Epilogue warpgroup: tile m_tile's stores are all issued; publish it for both halves of the parts count (convChainParts).
__device__ __noinline__ void chain_publish_tile(int* flags, int m_tile) {
  bulk_wait0();
  fence_proxy_async_global();
  red_release_gpu_add(flags + m_tile, 2);
}
// The epilogue warpgroup.  bar.sync is .aligned: a warp reaches it converged, so after an mbarrier wait loop (which its lanes may
// leave in different iterations) the epilogue brings the warp together with __syncwarp.
__device__ __forceinline__ void epi_wg_sync() { asm volatile("bar.sync 4, 128;" ::: "memory"); }

// Epilogue warpgroups: row rl of an fp32 accumulator slice (slice_offset's fp32 layout)
__device__ __forceinline__ void load_acc_row(const uint8_t* slice, int rl, float (&v)[RES_COLS]) {
#pragma unroll
  for(int k = 0; k < RES_COLS / 4; k++) {
    const float4 f = *reinterpret_cast<const float4*>(slice + slice_offset(rl, 4 * k, true));
    v[4 * k] = f.x; v[4 * k + 1] = f.y; v[4 * k + 2] = f.z; v[4 * k + 3] = f.w;
  }
}
// Row rl of an fp16 stream slice, as half2
__device__ __forceinline__ void load_half_row(const uint8_t* slice, int rl, uint32_t (&res)[RES_COLS / 2]) {
#pragma unroll
  for(int k = 0; k < RES_COLS / 8; k++) {
    const uint4 u = *reinterpret_cast<const uint4*>(slice + slice_offset(rl, 8 * k, false));
    res[4 * k] = u.x; res[4 * k + 1] = u.y; res[4 * k + 2] = u.z; res[4 * k + 3] = u.w;
  }
}
// Consumer warps: the accumulator fragments of N columns (rows rloc and rloc + 8, as in epilogue_slice) into N / 32 fp32 slices
// from `dst`, for an epilogue warpgroup to read by rows
template <int N>
__device__ __forceinline__ void store_acc_slices(uint8_t* dst, const float (&acc)[N / 2], int rloc, int lane) {
#pragma unroll
  for(int j = 0; j < N / 8; j++)
#pragma unroll
    for(int h = 0; h < 2; h++)
      *reinterpret_cast<float2*>(dst + (j / 4) * ACC_SLICE_BYTES + slice_offset(rloc + 8 * h, 8 * (j % 4) + 2 * (lane & 3), true)) =
        make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
}

// One row's part of slice s: its 16 column pairs through epilogue_store<F>, the outputs gathered in registers and written as
// 16-byte chunks, the raw output into `region` (the slice it was read from: every row of the slice has been read by then) and
// the activated operand into `act_region`.
template <int F>
__device__ __forceinline__ void epilogue_row(const ConvParams& p, int row, int rl, int col0, const float (&v)[RES_COLS],
                                             const uint32_t (&res)[RES_COLS / 2], float maskv, const float* sc, const float* bi,
                                             uint8_t* region, uint8_t* act_region) {
  constexpr bool raw32 = (F & EPI_FP32) != 0;
  float2 rawf[RES_COLS / 2];
  uint32_t rawh[RES_COLS / 2], act[RES_COLS / 2];
#pragma unroll
  for(int k = 0; k < RES_COLS / 2; k++) {
    const float2 r = (F & EPI_RES) ? __half22float2(*reinterpret_cast<const __half2*>(&res[k])) : make_float2(0.0f, 0.0f);
    epilogue_store<F>(p, row, col0 + 2 * k, v[2 * k], v[2 * k + 1], maskv, r, sc + 2 * k, bi + 2 * k,
                      raw32 ? reinterpret_cast<uint8_t*>(&rawf[k]) : reinterpret_cast<uint8_t*>(&rawh[k]),
                      reinterpret_cast<uint8_t*>(&act[k]), nullptr);
  }
  if(F & EPI_RAW) {
    if(raw32) {
#pragma unroll
      for(int k = 0; k < RES_COLS / 4; k++)
        *reinterpret_cast<float4*>(region + slice_offset(rl, 4 * k, true)) =
          make_float4(rawf[2 * k].x, rawf[2 * k].y, rawf[2 * k + 1].x, rawf[2 * k + 1].y);
    }
    else {
#pragma unroll
      for(int k = 0; k < RES_COLS / 8; k++)
        *reinterpret_cast<uint4*>(region + slice_offset(rl, 8 * k, false)) = make_uint4(rawh[4 * k], rawh[4 * k + 1], rawh[4 * k + 2], rawh[4 * k + 3]);
    }
  }
  if(F & EPI_MISH) {
#pragma unroll
    for(int k = 0; k < RES_COLS / 8; k++)
      *reinterpret_cast<uint4*>(act_region + slice_offset(rl, 8 * k, false)) =
        make_uint4(act[4 * k], act[4 * k + 1], act[4 * k + 2], act[4 * k + 3]);
  }
}

template <int N>
__global__ void __launch_bounds__(EPI_WG_THREADS, 1)
kgb_conv_wg_epi_kernel(const __grid_constant__ CUtensorMap tmapA, const __grid_constant__ CUtensorMap tmapB,
                       const __grid_constant__ CUtensorMap tmapR, const __grid_constant__ CUtensorMap tmapRaw,
                       const __grid_constant__ CUtensorMap tmapAct, const __grid_constant__ ConvParams p, int stages) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr int b_tile_bytes = N * BLOCK_K * 2;
  constexpr int slices = N / RES_COLS;
  const int flags = epiFlags(p);
  // [<=1023 B slack][2 x A halo tile][accumulator tile: slices x 16 KB][residual slot, 8 KB][stages x weight tile][EpiBars][BN]
  const int halo = convHalo(p), a_buf_bytes = aBufBytes(BLOCK_M + 2 * halo);
  const uint32_t smem_acc = smem_base + 2 * a_buf_bytes;
  const uint32_t smem_r = smem_acc + slices * ACC_SLICE_BYTES;
  const uint32_t smem_b = smem_r + (p.residual != nullptr ? ACT_SLICE_BYTES : 0);
  uint8_t* const smem = smem_raw + (smem_base - smem_u32(smem_raw));
  EpiBars* bars = reinterpret_cast<EpiBars*>(smem + (smem_b - smem_base) + (size_t)stages * b_tile_bytes);
  float* const s_scale = reinterpret_cast<float*>(bars + 1);
  float* const s_bias = s_scale + N;
  uint8_t* const acc_tile = smem + (smem_acc - smem_base);

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int tiles = __ldg(p.m_tiles) * p.num_n_tiles;
  const int n0 = (blockIdx.x % p.num_n_tiles) * N;

  pdl_launch_dependents();
  if(threadIdx.x == 0) {
    init_operand_rings(bars->ring, stages, p, tmapA, tmapB, tmapR, tmapRaw, tmapAct);
    mbar_init(smem_u32(&bars->r_full), 1);
    mbar_init(smem_u32(&bars->r_empty), 1);
    mbar_init(smem_u32(&bars->t_full), CONSUMER_WARPS);
    mbar_init(smem_u32(&bars->t_empty), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if(warp < 4) {
    // ===================== TMA producers =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    // no split mode here: one A halo tile per k-block
    if(warp == 0 && lane == 0) produce_operands<N>(p, bars->ring, tmapA, tmapB, smem_base, smem_b, stages, tiles, n0, 1);
    else if(warp == 1 && lane == 0 && p.residual != nullptr)   // each slice as soon as the epilogue warpgroup has read the one before
      produce_residual(p, &bars->r_full, &bars->r_empty, tmapR, smem_r, 1, ACT_SLICE_BYTES, n0, slices, tiles, p.num_n_tiles);
    return;
  }

  if(warp >= 12) {
    // ===================== epilogue warpgroup: thread rl finishes row rl of every tile =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 104;");
    const int rl = threadIdx.x - 384;
    const bool leader = rl == 0;    // issues the TMA stores and publishes the tiles
    if(p.act_out != nullptr)
      for(int i = rl; i < N; i += 128) { s_scale[i] = __ldg(p.bn_scale + n0 + i); s_bias[i] = __ldg(p.bn_bias + n0 + i); }
    epi_wg_sync();
    uint32_t tphase = 0, rphase = 0;
    for(int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
      const int m0 = (tile / p.num_n_tiles) * BLOCK_M, row = m0 + rl;
      const float maskv = row < p.M ? __ldg(p.mask + row) : 0.0f;
      mbar_wait(smem_u32(&bars->t_full), tphase);
      __syncwarp();
#pragma unroll 1
      for(int s = 0; s < slices; s++) {
        uint8_t* const region = acc_tile + s * ACC_SLICE_BYTES;
        float v[RES_COLS];
        load_acc_row(region, rl, v);
        uint32_t res[RES_COLS / 2];
        if(p.residual != nullptr) {
          mbar_wait(smem_u32(&bars->r_full), rphase);
          __syncwarp();
          rphase ^= 1;
          load_half_row(smem + (smem_r - smem_base), rl, res);
          // the slot's next TMA load (async proxy) follows these reads through the barrier below and r_empty: without the proxy
          // fence it may land before a read has returned its value
          fence_proxy_async();
        }
        else {
#pragma unroll
          for(int k = 0; k < RES_COLS / 2; k++) res[k] = 0;
        }
        epi_wg_sync();   // every row of the slice and the residual slot are read: the slot refills, the slice takes the outputs
        if(leader && p.residual != nullptr) mbar_arrive(smem_u32(&bars->r_empty));
        if(row < p.M) {   // no ncbias entry for rows past the batch; the TMA stores clip them
          const int lc = s * RES_COLS;
          switch(flags) {
#define KGB_EPI_ROW(F) case (F): epilogue_row<(F)>(p, row, rl, n0 + lc, v, res, maskv, s_scale + lc, s_bias + lc, region, region + ACT_SLICE_BYTES); break;
            KGB_EPI_WG_FLAGS(KGB_EPI_ROW)
#undef KGB_EPI_ROW
            default: break;   // launchConvWG launches no other
          }
        }
        fence_proxy_async();
        epi_wg_sync();
        if(leader) {
          const int c0 = n0 + s * RES_COLS;
          const bool raw32 = (flags & EPI_FP32) != 0;
          for(int h = 0; h < 2; h++) {
            const int r0 = m0 + h * (BLOCK_M / 2);
            if(p.raw_out != nullptr) tma_store_2d(&tmapRaw, smem_u32(region + h * (raw32 ? ACC_SLICE_BYTES : ACT_SLICE_BYTES) / 2), c0, r0);
            if(p.act_out != nullptr) tma_store_2d(&tmapAct, smem_u32(region + ACT_SLICE_BYTES + h * (ACT_SLICE_BYTES / 2)), c0, r0);
          }
          bulk_commit();
        }
      }
      tphase ^= 1;
      if(leader) {
        bulk_wait_read0();   // the stores have read the tile: the consumers may write the next one
        mbar_arrive(smem_u32(&bars->t_empty));
        chain_publish_tile(p.tile_flags, m0 / BLOCK_M);
      }
    }
    pdl_wait();
    return;
  }

  // ===================== consumers: warpgroup g owns tile rows 64g..64g+63, warp q of it rows 16q..16q+15 =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 184;");
  const int g = (warp - 4) >> 2, q = warp & 3;
  const int lrow = g * 64 + q * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
  // acc[4j + 2h + e]: row 16q + lane/4 + 8h of the warpgroup's 64, column 8j + 2*(lane%4) + e
  const int rloc = g * 64 + q * 16 + (lane >> 2);
  RingPos rp;
  uint32_t tphase = 0;
  for(int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    float acc[N / 2];
    conv_main_loop<N>(acc, rp, bars->ring, p, smem_base, smem_b, stages, p.cin_p / BLOCK_K, lrow, lane, halo, a_buf_bytes);
    // hand the accumulators to the epilogue warpgroup once it has read the previous tile out of the accumulator tile
    mbar_wait(smem_u32(&bars->t_empty), tphase ^ 1);
    tphase ^= 1;
    store_acc_slices<N>(acc_tile, acc, rloc, lane);
    warp_arrive(smem_u32(&bars->t_full), lane);
  }
  pdl_wait();
}

static int g_smCount[64];   // per device ordinal, read by convWGInit
static int* g_chainErrorHost;   // the sticky word chain_wait sets, in mapped host memory shared by every device
static cudaError_t convPairInit();

cudaError_t convChainStatus() {
  return g_chainErrorHost != nullptr && *(volatile int*)g_chainErrorHost != 0 ? cudaErrorLaunchTimeout : cudaSuccess;
}

cudaError_t convWGInit() {
  int dev = 0;
  cudaError_t e0 = cudaGetDevice(&dev);
  if(e0 != cudaSuccess) return e0;
  if(dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  e0 = cudaDeviceGetAttribute(&g_smCount[dev], cudaDevAttrMultiProcessorCount, dev);
  if(e0 != cudaSuccess) return e0;
  static int* word = [] {
    int* w = nullptr;
    if(cudaHostAlloc((void**)&w, sizeof(int), cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) return (int*)nullptr;
    *w = 0;
    return w;
  }();
  if(word == nullptr) return cudaErrorMemoryAllocation;
  g_chainErrorHost = word;
  int* devWord = nullptr;
  e0 = cudaHostGetDevicePointer((void**)&devWord, word, 0);
  if(e0 != cudaSuccess) return e0;
  e0 = cudaMemcpyToSymbol(g_chainError, &devWord, sizeof(devWord));
  if(e0 != cudaSuccess) return e0;
#define KGB_WG_ATTR(N) cudaFuncSetAttribute(kgb_conv_wg_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT),
#define KGB_EPI_WG_ATTR(N) cudaFuncSetAttribute(kgb_conv_wg_epi_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT),
  for(cudaError_t e : {KGB_WG_SHAPES(KGB_WG_ATTR) KGB_EPI_WG_SHAPES(KGB_EPI_WG_ATTR) convPairInit()})
    if(e != cudaSuccess) return e;
#undef KGB_EPI_WG_ATTR
#undef KGB_WG_ATTR
  return cudaSuccess;
}

// The SM count convWGInit recorded for the current device: the persistent grids' CTA limit
static cudaError_t smCount(int* n) {
  int dev = 0;
  const cudaError_t e = cudaGetDevice(&dev);
  if(e != cudaSuccess) return e;
  if(dev < 0 || dev >= 64 || g_smCount[dev] < 1) return cudaErrorInitializationError;   // convWGInit not run on this device
  *n = g_smCount[dev];
  return cudaSuccess;
}

// A chained launch (p.pred_flags set) may start while the previous kernel on the stream still runs
template <class... Args>
static cudaError_t launchChained(void (*kernel)(Args...), const ConvParams& p, int grid, int threads, int smem, cudaStream_t stream,
                                 Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = p.pred_flags != nullptr ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}

// A kernel's shared memory: its fixed bytes first, then as many weight stages as fit
struct SmemLayout {
  int stages = 0, smem = 0;
  int r_slots = 0;   // the fused boundary's residual ring
};
static SmemLayout fitStages(int fixed, int stage_bytes, int r_slots = 0) {
  SmemLayout l;
  l.stages = std::min(MAX_STAGES, (SMEM_LIMIT - fixed) / stage_bytes);
  l.smem = fixed + l.stages * stage_bytes;
  l.r_slots = r_slots;
  return l;
}

// kgb_conv_wg_kernel: the stream and act rings and the BN copies are fixed
static SmemLayout wgLayout(const ConvParams& p) {
  return fitStages(1024 + 2 * aBufBytes(BLOCK_M + 2 * convHalo(p)) + streamSlots(p) * streamSlotBytes(p) + ACT_SLOTS * actSlotBytes(p) +
                   (int)sizeof(Bars) + 2 * p.n_tile * (int)sizeof(float), p.n_tile * BLOCK_K * 2);
}

// kgb_conv_wg_epi_kernel: the accumulator tile, the residual slot and the BN copies are fixed
static SmemLayout epiLayout(const ConvParams& p) {
  return fitStages(1024 + 2 * aBufBytes(BLOCK_M + 2 * convHalo(p)) + p.n_tile / RES_COLS * ACC_SLICE_BYTES +
                   (p.residual != nullptr ? ACT_SLICE_BYTES : 0) + (int)sizeof(EpiBars) + 2 * p.n_tile * (int)sizeof(float),
                   p.n_tile * BLOCK_K * 2);
}

bool convEpilogueWG(const ConvParams& p) {
  if(!p.epi_wg || p.split || p.ky * p.kx == 1) return false;
  const int f = epiFlags(p), halo = convHalo(p);
  bool shape = false, epi = false;
#define KGB_EPI_WG_IS(N) shape = shape || p.n_tile == N;
  KGB_EPI_WG_SHAPES(KGB_EPI_WG_IS)
#undef KGB_EPI_WG_IS
#define KGB_EPI_WG_IS(F) epi = epi || f == (F);
  KGB_EPI_WG_FLAGS(KGB_EPI_WG_IS)
#undef KGB_EPI_WG_IS
  return shape && epi && BLOCK_M + 2 * halo <= 256 && epiLayout(p).stages >= EPI_WG_MIN_STAGES;
}

cudaError_t launchConvWG(const ConvTmaps& tm, const ConvParams& p, cudaStream_t stream) {
  if(BLOCK_M + 2 * convHalo(p) > 256) return cudaErrorInvalidValue;  // TMA box limit
  if(p.n_tile % RES_COLS != 0) return cudaErrorInvalidValue;
  // the raw output is written over the residual slice it was read from
  if(p.residual != nullptr && p.raw_out != nullptr && (p.residual_fp32 != 0) != (p.raw_fp32 != 0)) return cudaErrorInvalidValue;
  if(p.tile_flags == nullptr) return cudaErrorInvalidValue;
  int sms = 0;
  const cudaError_t e = smCount(&sms);
  if(e != cudaSuccess) return e;
  // persistent grid: at most one CTA per SM (the rings take all of shared memory), a multiple of num_n_tiles
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  int grid = std::min(tiles, sms) / p.num_n_tiles * p.num_n_tiles;
  if(grid < p.num_n_tiles) grid = p.num_n_tiles;
  if(convEpilogueWG(p)) {
    const SmemLayout l = epiLayout(p);
#define KGB_EPI_WG_LAUNCH(N) \
    if(p.n_tile == N)        \
      return launchChained(kgb_conv_wg_epi_kernel<N>, p, grid, EPI_WG_THREADS, l.smem, stream, tm.A, tm.B, tm.residual, tm.raw, tm.act, p, l.stages);
    KGB_EPI_WG_SHAPES(KGB_EPI_WG_LAUNCH)
#undef KGB_EPI_WG_LAUNCH
  }
  const SmemLayout l = wgLayout(p);
  if(l.stages < 2) return cudaErrorInvalidValue;
#define KGB_WG_LAUNCH(N) \
  if(p.n_tile == N)      \
    return launchChained(kgb_conv_wg_kernel<N>, p, grid, THREADS, l.smem, stream, tm.A, tm.B, tm.residual, tm.raw, tm.act, p, l.stages);
  KGB_WG_SHAPES(KGB_WG_LAUNCH)
#undef KGB_WG_LAUNCH
  return cudaErrorInvalidValue;
}

// ------------------------------------------------------------------------------------------------------------
// Fused block boundary (launchConvPair): exit 1x1 of nested block i + entry 1x1 of nested block i+1
// ------------------------------------------------------------------------------------------------------------
// Both layers are bound by HBM bytes; in two launches the activated trunk operand (fp16, trunk channels) is written by the exit
// and read straight back by the entry.  Here one persistent CTA per SM walks 128-row tiles; for one tile:
//   phase 1  the exit's output in chunks of PAIR_NC columns: acc1[128 x 64] = A[128 x K1] * W1[chunk], the inner operand A resident
//            in shared memory for the whole tile (1x1: no halo).  Its epilogue is the exit's (residual slice in, raw stream out by
//            TMA store), except that the activated operand goes into a shared-memory chunk slot T, 64B-swizzled 32-column slices.
//   phase 2  each finished chunk is one k-block of the entry: acc2[128 x N2] += T * W2[chunk], both operands by shared-memory
//            descriptor.  After the last chunk, the entry's epilogue writes the inner raw stream and activated operand.
// The loop per chunk c issues P1(c+1) and P2(c) together and waits for P1(c+1) only, so P2(c) runs under chunk c+1's epilogue;
// T has two slots for that.  Weight stages hold one chunk of W1 (K1/64 boxes {64, 64}) or of W2 (one box {64, N2}), both
// N2 * 128 bytes, in the order the consumers take them: W1(0), then W1(c+1), W2(c) for each c.  acc2 sums over K in the order of
// the entry's own launch (chunk = k-block, then k16), acc1 in that of the exit's, and the epilogues are the same code.
static constexpr int PAIR_NC = kConvPairChunk;
static constexpr int PAIR_T_BYTES = BLOCK_M * PAIR_NC * 2;   // one chunk slot: PAIR_NC / 32 act slices

struct __align__(8) PairBars {
  uint64_t full[MAX_STAGES];
  uint64_t empty[MAX_STAGES];
  uint64_t a_full, a_empty;     // the inner operand tile of the current tile
  uint64_t r_full[RES_SLOTS];
  uint64_t r_empty[RES_SLOTS];
};

// 64B-swizzled K-major operand (the act slices, slice_offset's fp16 layout): 64 B rows, 8-row groups 512 B apart
__device__ __forceinline__ uint64_t make_smem_desc_sw64(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(512 >> 4) << 32;
  d |= (uint64_t)2 << 62;
  return d;
}

// Lane 0 of warp 0 of the fused boundary: the inner operand tile (K1/64 boxes {64, 128}), then the weight chunks of NC columns in the
// order the consumers take them: W1(0), then W1(c+1), W2(c) for each chunk c.  A W1 chunk is K1/64 boxes {64, NC} and a W2 chunk
// NC/64 boxes {64, N2} or one box {32, N2}, either way one stage of N2 * NC * 2 bytes.
template <int N2, int N1, int NC, class PB>
__device__ __forceinline__ void produce_pair_operands(const ConvParams& p1, PB& bars, const CUtensorMap& tmapA, const CUtensorMap& tmapW1,
                                                      const CUtensorMap& tmapW2, uint32_t smem_a, uint32_t smem_w, int stages, int tiles) {
  constexpr int K1 = N2, A_BYTES = BLOCK_M * K1 * 2, W_BYTES = N2 * NC * 2, chunks = N1 / NC;
  int stage = 0;
  uint32_t phase = 0, aphase = 0;
  auto loadW = [&](bool entry, int c) {
    mbar_wait(smem_u32(&bars.empty[stage]), phase ^ 1);
    const uint32_t full = smem_u32(&bars.full[stage]), dst = smem_w + stage * W_BYTES;
    mbar_arrive_expect_tx(full, (uint32_t)W_BYTES);
    if(entry) {
      for(int j = 0; j < (NC + BLOCK_K - 1) / BLOCK_K; j++) tma_load_2d(dst + j * N2 * 128, &tmapW2, full, c * NC + j * BLOCK_K, 0);
    }
    else {
      for(int kb = 0; kb < K1 / BLOCK_K; kb++) tma_load_2d(dst + kb * NC * 128, &tmapW1, full, kb * BLOCK_K, c * NC);
    }
    if(++stage == stages) { stage = 0; phase ^= 1; }
  };
  // the first tile's first exit chunk goes out before its chain wait (weights do not depend on the previous launch)
  bool pre = (int)blockIdx.x < tiles;
  if(pre) loadW(false, 0);
  for(int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int m0 = tile * BLOCK_M;
    chain_wait(p1.pred_flags, p1.pred_parts, tile, tiles);
    mbar_wait(smem_u32(&bars.a_empty), aphase ^ 1);
    const uint32_t afull = smem_u32(&bars.a_full);
    mbar_arrive_expect_tx(afull, (uint32_t)A_BYTES);
    for(int kb = 0; kb < K1 / BLOCK_K; kb++) tma_load_2d(smem_a + kb * BLOCK_M * 128, &tmapA, afull, kb * BLOCK_K, m0);
    aphase ^= 1;
    if(!pre) loadW(false, 0);
    pre = false;
    for(int c = 0; c < chunks; c++) {
      if(c + 1 < chunks) loadW(false, c + 1);
      loadW(true, c);
    }
  }
}

// Fused-boundary consumers: wait for the next weight stage and return it
__device__ __forceinline__ int take_stage(uint64_t* full, int stages, int& stage, uint32_t& phase) {
  const int st = stage;
  mbar_wait(smem_u32(&full[st]), phase);
  if(++stage == stages) { stage = 0; phase ^= 1; }
  return st;
}

// The entry's epilogue for consumer warpgroup g: the inner raw stream and the activated inner operand out of acc2, one 32-column
// slice at a time through the staging ring at stg_ring (slot ps) and the act ring at act_ring (slot as), out by TMA stores.  Once
// the first slice's bulk_wait_read0 shows that the stores before it have read their slots, the leader also releases the exit's
// residual slot `release_rs` (-1: none).
template <int F2, int N2, int R2_BYTES>
__device__ __forceinline__ void pair_entry_epilogue(const ConvParams& p2, const float (&acc2)[N2 / 2], int m0, int g, int rloc, int lane,
                                                    bool leader, float mask0, float mask1, const float* s_scale2, const float* s_bias2,
                                                    uint8_t* stg_ring, uint8_t* act_ring, int& ps, int& as, const CUtensorMap& tmapS2,
                                                    const CUtensorMap& tmapA2, uint64_t* r_empty, int release_rs) {
#pragma unroll
  for(int s = 0; s < N2 / RES_COLS; s++) {
    uint8_t* const slot = stg_ring + ps * R2_BYTES;
    uint8_t* const aslot = act_ring + as * ACT_SLICE_BYTES;
    epilogue_slice<F2, N2>(p2, acc2, s, m0, 0, rloc, lane, mask0, mask1, s_scale2, s_bias2, slot, aslot);
    fence_proxy_async();
    if(leader) {
      bulk_wait_read0();
      if(s == 0 && release_rs >= 0) mbar_arrive(smem_u32(&r_empty[release_rs]));
    }
    warpgroup_sync(g);
    if(leader) {
      const int c0 = s * RES_COLS, r0 = m0 + g * (BLOCK_M / 2);
      tma_store_2d(&tmapS2, smem_u32(slot + g * (R2_BYTES / 2)), c0, r0);
      tma_store_2d(&tmapA2, smem_u32(aslot + g * (ACT_SLICE_BYTES / 2)), c0, r0);
      bulk_commit();
    }
    ps ^= 1;
    as ^= 1;
  }
}

// dynamic smem: [<=1023 B slack][A tile: K1/64 x 16 KB][2 x T slot][residual ring][2 x raw staging][2 x act slice][stages x weights]
//               [PairBars][BN scale / bias: exit N1, entry N2]
static SmemLayout pairLayout(const ConvParams& p1, const ConvParams& p2) {
  const int n2 = p2.cout_p, n1 = p1.cout_p;
  const int r1 = BLOCK_M * RES_COLS * (p1.residual_fp32 ? 4 : 2), r2 = BLOCK_M * RES_COLS * (p2.raw_fp32 ? 4 : 2);
  // a full residual ring when it leaves room for three weight stages, else half of one
  for(int rs : {RES_SLOTS, 2}) {
    const SmemLayout l = fitStages(1024 + BLOCK_M * n2 * 2 + 2 * PAIR_T_BYTES + rs * r1 + STAGE_SLOTS * r2 + ACT_SLOTS * ACT_SLICE_BYTES +
                                   (int)sizeof(PairBars) + 2 * (n1 + n2) * (int)sizeof(float), n2 * PAIR_NC * 2, rs);
    if(l.stages >= 3 || (rs == 2 && l.stages >= 2)) return l;
  }
  return SmemLayout();
}

template <int N2, int N1, bool S1_FP32, bool S2_FP32>
__global__ void __launch_bounds__(THREADS, 1)
kgb_conv_pair_kernel(const __grid_constant__ CUtensorMap tmapA, const __grid_constant__ CUtensorMap tmapW1,
                     const __grid_constant__ CUtensorMap tmapW2, const __grid_constant__ CUtensorMap tmapS1,
                     const __grid_constant__ CUtensorMap tmapS2, const __grid_constant__ CUtensorMap tmapA2,
                     const __grid_constant__ ConvParams p1, const __grid_constant__ ConvParams p2, int stages, int r_slots) {
  constexpr int F1 = EPI_RES | EPI_RAW | EPI_MISH | (S1_FP32 ? EPI_FP32 : 0);
  constexpr int F2 = EPI_RAW | EPI_MISH | (S2_FP32 ? EPI_FP32 : 0);
  constexpr int K1 = N2;                             // the exit's K = the entry's N = the inner channels
  constexpr int A_BYTES = BLOCK_M * K1 * 2;          // K1 / 64 boxes {64, 128}
  constexpr int W_BYTES = N2 * PAIR_NC * 2;
  constexpr int R1_BYTES = BLOCK_M * RES_COLS * (S1_FP32 ? 4 : 2), R2_BYTES = BLOCK_M * RES_COLS * (S2_FP32 ? 4 : 2);
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_t = smem_base + A_BYTES;
  const uint32_t smem_r = smem_t + 2 * PAIR_T_BYTES;
  const uint32_t smem_stg = smem_r + r_slots * R1_BYTES;
  const uint32_t smem_act = smem_stg + STAGE_SLOTS * R2_BYTES;
  const uint32_t smem_w = smem_act + ACT_SLOTS * ACT_SLICE_BYTES;
  uint8_t* const smem = smem_raw + (smem_base - smem_u32(smem_raw));
  PairBars* bars = reinterpret_cast<PairBars*>(smem + (smem_w - smem_base) + (size_t)stages * W_BYTES);
  constexpr int chunks = N1 / PAIR_NC;
  float* const s_scale1 = reinterpret_cast<float*>(bars + 1);
  float* const s_bias1 = s_scale1 + N1;
  float* const s_scale2 = s_bias1 + N1;
  float* const s_bias2 = s_scale2 + N2;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int tiles = __ldg(p1.m_tiles);

  pdl_launch_dependents();
  if(threadIdx.x == 0) {
    for(const CUtensorMap* m : {&tmapA, &tmapW1, &tmapW2, &tmapS1, &tmapS2, &tmapA2}) prefetch_tmap(m);
    init_weight_ring(bars->full, bars->empty, stages);
    mbar_init(smem_u32(&bars->a_full), 1);
    mbar_init(smem_u32(&bars->a_empty), CONSUMER_WARPS);
    for(int s = 0; s < RES_SLOTS; s++) {
      mbar_init(smem_u32(&bars->r_full[s]), 1);
      mbar_init(smem_u32(&bars->r_empty[s]), 2);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if(warp < 4) {
    // ===================== TMA producers =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if(warp == 0 && lane == 0) produce_pair_operands<N2, N1, PAIR_NC>(p1, *bars, tmapA, tmapW1, tmapW2, smem_base, smem_w, stages, tiles);
    else if(warp == 1 && lane == 0)   // the exit's residual slices
      produce_residual(p1, bars->r_full, bars->r_empty, tmapS1, smem_r, r_slots, R1_BYTES, 0, N1 / RES_COLS, tiles, 1);
    return;
  }

  // ===================== consumers: warpgroup g owns tile rows 64g..64g+63 =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int g = (warp - 4) >> 2, q = warp & 3;
  const bool leader = q == 0 && lane == 0;
  const int rloc = g * 64 + q * 16 + (lane >> 2);
  for(int i = threadIdx.x - 128; i < N1; i += 32 * CONSUMER_WARPS) { s_scale1[i] = __ldg(p1.bn_scale + i); s_bias1[i] = __ldg(p1.bn_bias + i); }
  for(int i = threadIdx.x - 128; i < N2; i += 32 * CONSUMER_WARPS) { s_scale2[i] = __ldg(p2.bn_scale + i); s_bias2[i] = __ldg(p2.bn_bias + i); }
  consumer_sync();

  int stage = 0, rs = 0, prev_rs = -1, ps = 0, as = 0;
  uint32_t phase = 0, rphase = 0, aphase = 0;
  uint8_t* const ring = smem + (smem_r - smem_base);
  uint8_t* const t_ring = smem + (smem_t - smem_base);
  uint8_t* const stg_ring = smem + (smem_stg - smem_base);
  uint8_t* const act_ring = smem + (smem_act - smem_base);
  int pending = -1;   // the tile whose stores this warpgroup issued last and has not published yet
  for(int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int m0 = tile * BLOCK_M;
    const float mask0 = m0 + rloc < p1.M ? __ldg(p1.mask + m0 + rloc) : 0.0f;
    const float mask1 = m0 + rloc + 8 < p1.M ? __ldg(p1.mask + m0 + rloc + 8) : 0.0f;
    float acc1[PAIR_NC / 2], acc2[N2 / 2];
#pragma unroll
    for(int i = 0; i < N2 / 2; i++) acc2[i] = 0.0f;
    // P1: acc1 = A rows 64g.. x W1 chunk in stage st (K1 / 64 k-blocks of 4 k16 steps, as the exit's launch sums them)
    auto issueP1 = [&](int st) {
      const uint32_t w = smem_w + st * W_BYTES, a = smem_base + g * 64 * 128;
#pragma unroll
      for(int kb = 0; kb < K1 / BLOCK_K; kb++)
#pragma unroll
        for(int k = 0; k < 4; k++)
          WgmmaSS<PAIR_NC>::mma(acc1, make_smem_desc(a + kb * BLOCK_M * 128) + 2 * k, make_smem_desc(w + kb * PAIR_NC * 128) + 2 * k);
      wgmma_commit();
    };
    // P2: acc2 += T slot rows 64g.. x W2 chunk in stage st (the chunk's k16 steps in order)
    auto issueP2 = [&](int st, int slot) {
      const uint32_t w = smem_w + st * W_BYTES, t = smem_t + slot * PAIR_T_BYTES + g * 64 * 64;
#pragma unroll
      for(int k = 0; k < PAIR_NC / 16; k++)
        WgmmaSS<N2>::mma(acc2, make_smem_desc_sw64(t + (k / 2) * ACT_SLICE_BYTES) + 2 * (k & 1),
                         make_smem_desc(w + (k / 4) * N2 * 128) + 2 * (k & 3));
      wgmma_commit();
    };
    auto zeroAcc1 = [&]() {
#pragma unroll
      for(int i = 0; i < PAIR_NC / 2; i++) acc1[i] = 0.0f;
    };

    mbar_wait(smem_u32(&bars->a_full), aphase);
    aphase ^= 1;
    zeroAcc1();
    fence_acc(acc1);
    fence_acc(acc2);
    int st1 = take_stage(bars->full, stages, stage, phase), st2 = -1;
    wgmma_fence();
    issueP1(st1);
    wgmma_wait0();
    fence_acc(acc1);
    warp_arrive(smem_u32(&bars->empty[st1]), lane);
    if(chunks == 1) warp_arrive(smem_u32(&bars->a_empty), lane);
    if(leader && pending >= 0) chain_publish(p1.tile_flags, pending);
#pragma unroll
    for(int c = 0; c < chunks; c++) {
      // ---- the exit's epilogue of chunk c: residual in, raw stream out, activated operand into T slot c & 1 ----
#pragma unroll
      for(int s = 0; s < PAIR_NC / RES_COLS; s++) {
        uint8_t* const slot = ring + rs * R1_BYTES;
        mbar_wait(smem_u32(&bars->r_full[rs]), rphase);
        epilogue_slice<F1, PAIR_NC>(p1, acc1, s, m0, c * PAIR_NC, rloc, lane, mask0, mask1, s_scale1 + c * PAIR_NC, s_bias1 + c * PAIR_NC,
                                    slot, t_ring + (c & 1) * PAIR_T_BYTES + s * ACT_SLICE_BYTES);
        fence_proxy_async();   // the raw slice for its TMA store, the T slice for the wgmma that reads it
        if(leader) {
          bulk_wait_read0();
          if(prev_rs >= 0) mbar_arrive(smem_u32(&bars->r_empty[prev_rs]));
        }
        warpgroup_sync(g);
        if(leader) {
          tma_store_2d(&tmapS1, smem_u32(slot + g * (R1_BYTES / 2)), c * PAIR_NC + s * RES_COLS, m0 + g * (BLOCK_M / 2));
          bulk_commit();
        }
        prev_rs = rs;
        if(++rs == r_slots) { rs = 0; rphase ^= 1; }
      }
      // P2(c - 1) has read T slot (c - 1) & 1 and its weight stage
      if(c > 0) {
        wgmma_wait0();
        warp_arrive(smem_u32(&bars->empty[st2]), lane);
      }
      zeroAcc1();
      fence_acc(acc1);
      fence_acc(acc2);
      wgmma_fence();
      if(c + 1 < chunks) {
        st1 = take_stage(bars->full, stages, stage, phase);
        issueP1(st1);
      }
      st2 = take_stage(bars->full, stages, stage, phase);
      issueP2(st2, c & 1);
      if(c + 1 < chunks) {
        wgmma_wait1();   // P1(c + 1) done, P2(c) may still run under the next chunk's epilogue
        fence_acc(acc1);
        warp_arrive(smem_u32(&bars->empty[st1]), lane);
        if(c + 2 == chunks) warp_arrive(smem_u32(&bars->a_empty), lane);   // the tile's last P1: the next tile's A may land
      }
    }
    wgmma_wait0();
    fence_acc(acc2);
    warp_arrive(smem_u32(&bars->empty[st2]), lane);

    pair_entry_epilogue<F2, N2, R2_BYTES>(p2, acc2, m0, g, rloc, lane, leader, mask0, mask1, s_scale2, s_bias2, stg_ring, act_ring, ps, as,
                                          tmapS2, tmapA2, bars->r_empty, prev_rs);
    prev_rs = -1;
    pending = tile;
  }
  if(leader && pending >= 0) chain_publish(p1.tile_flags, pending);
  if(leader) bulk_wait0();
  pdl_wait();
}

// ------------------------------------------------------------------------------------------------------------
// Fused block boundary with an exit-epilogue warpgroup (kgb_conv_pair_epi_kernel, launchConvPair when convPairEpilogueWG)
// ------------------------------------------------------------------------------------------------------------
// In kgb_conv_pair_kernel the two consumer warpgroups run each exit chunk's epilogue themselves, so only one chunk of entry MMAs
// overlaps it and the loads and stores in flight wait on their arithmetic.  Here a fourth warpgroup runs the exit's epilogue,
// 512 threads, with exit chunks of PAIR_EPI_NC = 32 columns:
//   warpgroup 0     TMA producers: the inner operand tile, the weight chunks in consumption order (W1(0), then W1(c+1), W2(c)),
//                   the exit's residual slices into a ring.
//   warpgroups 1-2  MMA, 64 rows each.  Step c issues P1(c) (acc1 = A x W1 chunk c), writes acc1 as fp32 into accumulator slot
//                   c & 1 (slice_offset's fp32 layout) and arrives on acc_full, then issues P2(c-1) (acc2 += T x W2 chunk c-1) once
//                   T slot (c-1) & 1 is full: P1(c+1) is handed over while the epilogue warpgroup works on chunk c.  After the
//                   tile's last P2 they hand over the next tile's chunk 0, then run the entry's epilogue from acc2 as
//                   kgb_conv_pair_kernel does, and publish their halves of it 3 chunks into the next tile.
//   warpgroup 3     the exit's epilogue, one thread per row: for chunk c it reads its row of accumulator slot c & 1 and of the
//                   residual slice, applies epilogue_store<F1> (epilogue_row), writes the raw trunk stream back over the residual
//                   slice for its TMA store and the activated operand into T slot c & 1, and arrives on t_full.  It publishes the
//                   tile's exit part once its stores are complete, 3 chunks into the next tile, so a tile is written when its flag
//                   reaches 3 (convPairChainParts).
// Every exit column is still summed over K1 in k-block, k16 order and every entry output over the trunk channels in k16 order (12
// chunks of 2 k16 steps instead of 6 of 4): the same bits as kgb_conv_pair_kernel and the two launches.
// Shared memory for (192, 384) with fp16 streams: A tile 48 KB, 2 accumulator slots of 16 KB, 2 T slots of 8 KB, a 4-slot residual
// ring of 8 KB, entry staging 2 x 8 KB raw + 2 x 8 KB act, 5 weight stages of 12 KB (W1 chunk: K1/64 boxes {64, 32}, 128B swizzle;
// W2 chunk: one box {32, N2}, 64B swizzle), PairEpiBars and the BN constants: 231,184 B of the 232,448.  A 64-column chunk would need
// 32 KB accumulator slots and 24 KB weight stages, 64 KB more than fits.  Registers after setmaxnreg: producers 40, MMA 184 (acc2 96,
// acc1 16), epilogue 104.
static constexpr int PAIR_EPI_NC = RES_COLS;
static constexpr int PAIR_EPI_THREADS = 512;

struct __align__(8) PairEpiBars {
  uint64_t full[MAX_STAGES];
  uint64_t empty[MAX_STAGES];
  uint64_t a_full, a_empty;     // the inner operand tile of the current tile
  uint64_t r_full[RES_SLOTS];   // residual slice landed
  uint64_t r_empty[RES_SLOTS];  // residual slice read and the raw stream written over it stored
  uint64_t acc_full[2];         // accumulator slot written by every MMA warp
  uint64_t acc_empty[2];        // accumulator slot read by every epilogue warp
  uint64_t t_full[2];           // T slot written by the epilogue warpgroup
  uint64_t t_empty[2];          // T slot read by every MMA warp's P2
};

// dynamic smem: [<=1023 B slack][A tile][2 x accumulator slot][2 x T slot][residual ring][2 x raw staging][2 x act slice]
//               [stages x weights][PairEpiBars][BN scale / bias: exit N1, entry N2]
static SmemLayout pairEpiLayout(const ConvParams& p1, const ConvParams& p2) {
  const int n2 = p2.cout_p, n1 = p1.cout_p;
  return fitStages(1024 + BLOCK_M * n2 * 2 + 2 * ACC_SLICE_BYTES + 2 * ACT_SLICE_BYTES + RES_SLOTS * ACT_SLICE_BYTES +
                   STAGE_SLOTS * ACT_SLICE_BYTES + ACT_SLOTS * ACT_SLICE_BYTES + (int)sizeof(PairEpiBars) + 2 * (n1 + n2) * (int)sizeof(float),
                   n2 * PAIR_EPI_NC * 2, RES_SLOTS);
}

template <int N2, int N1>
__global__ void __launch_bounds__(PAIR_EPI_THREADS, 1)
kgb_conv_pair_epi_kernel(const __grid_constant__ CUtensorMap tmapA, const __grid_constant__ CUtensorMap tmapW1,
                         const __grid_constant__ CUtensorMap tmapW2, const __grid_constant__ CUtensorMap tmapS1,
                         const __grid_constant__ CUtensorMap tmapS2, const __grid_constant__ CUtensorMap tmapA2,
                         const __grid_constant__ ConvParams p1, const __grid_constant__ ConvParams p2, int stages) {
  constexpr int F1 = EPI_RES | EPI_RAW | EPI_MISH;
  constexpr int F2 = EPI_RAW | EPI_MISH;
  constexpr int NC = PAIR_EPI_NC;
  constexpr int K1 = N2;
  constexpr int A_BYTES = BLOCK_M * K1 * 2;
  constexpr int W_BYTES = N2 * NC * 2;
  constexpr int chunks = N1 / NC;
  static_assert(chunks >= 4, "the MMA loop keeps the P2 of two chunks in flight; tiles are published 3 chunks into the next");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_acc = smem_base + A_BYTES;
  const uint32_t smem_t = smem_acc + 2 * ACC_SLICE_BYTES;
  const uint32_t smem_r = smem_t + 2 * ACT_SLICE_BYTES;
  const uint32_t smem_stg = smem_r + RES_SLOTS * ACT_SLICE_BYTES;
  const uint32_t smem_act = smem_stg + STAGE_SLOTS * ACT_SLICE_BYTES;
  const uint32_t smem_w = smem_act + ACT_SLOTS * ACT_SLICE_BYTES;
  uint8_t* const smem = smem_raw + (smem_base - smem_u32(smem_raw));
  PairEpiBars* bars = reinterpret_cast<PairEpiBars*>(smem + (smem_w - smem_base) + (size_t)stages * W_BYTES);
  float* const s_scale1 = reinterpret_cast<float*>(bars + 1);
  float* const s_bias1 = s_scale1 + N1;
  float* const s_scale2 = s_bias1 + N1;
  float* const s_bias2 = s_scale2 + N2;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int tiles = __ldg(p1.m_tiles);

  pdl_launch_dependents();
  if(threadIdx.x == 0) {
    for(const CUtensorMap* m : {&tmapA, &tmapW1, &tmapW2, &tmapS1, &tmapS2, &tmapA2}) prefetch_tmap(m);
    init_weight_ring(bars->full, bars->empty, stages);
    mbar_init(smem_u32(&bars->a_full), 1);
    mbar_init(smem_u32(&bars->a_empty), CONSUMER_WARPS);
    for(int s = 0; s < RES_SLOTS; s++) {
      mbar_init(smem_u32(&bars->r_full[s]), 1);
      mbar_init(smem_u32(&bars->r_empty[s]), 1);
    }
    for(int s = 0; s < 2; s++) {
      mbar_init(smem_u32(&bars->acc_full[s]), CONSUMER_WARPS);
      mbar_init(smem_u32(&bars->acc_empty[s]), 4);
      mbar_init(smem_u32(&bars->t_full[s]), 1);
      mbar_init(smem_u32(&bars->t_empty[s]), CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if(warp < 4) {
    // ===================== TMA producers =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if(warp == 0 && lane == 0) produce_pair_operands<N2, N1, NC>(p1, *bars, tmapA, tmapW1, tmapW2, smem_base, smem_w, stages, tiles);
    else if(warp == 1 && lane == 0)
      produce_residual(p1, bars->r_full, bars->r_empty, tmapS1, smem_r, RES_SLOTS, ACT_SLICE_BYTES, 0, chunks, tiles, 1);
    return;
  }

  if(warp >= 12) {
    // ===================== exit epilogue: thread rl finishes row rl of every chunk =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 104;");
    const int rl = threadIdx.x - 384;
    const bool leader = rl == 0;    // issues the TMA stores and publishes the tiles' exit part
    for(int i = rl; i < N1; i += 128) { s_scale1[i] = __ldg(p1.bn_scale + i); s_bias1[i] = __ldg(p1.bn_bias + i); }
    epi_wg_sync();
    int rs = 0, prev_rs = -1, k = 0;   // k: chunks finished by this CTA, whose parity picks the accumulator and T slot
    uint32_t rphase = 0;
    int pending = -1;   // the tile whose exit stores were issued last and are not published yet
    for(int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
      const int m0 = tile * BLOCK_M, row = m0 + rl;
      const float maskv = row < p1.M ? __ldg(p1.mask + row) : 0.0f;
#pragma unroll 1
      for(int c = 0; c < chunks; c++, k++) {
        const int slot = k & 1;
        const uint32_t par = (k >> 1) & 1;
        uint8_t* const rslot = smem + (smem_r - smem_base) + rs * ACT_SLICE_BYTES;
        mbar_wait(smem_u32(&bars->acc_full[slot]), par);
        __syncwarp();
        float v[RES_COLS];
        load_acc_row(smem + (smem_acc - smem_base) + slot * ACC_SLICE_BYTES, rl, v);
        mbar_wait(smem_u32(&bars->r_full[rs]), rphase);
        __syncwarp();
        uint32_t res[RES_COLS / 2];
        load_half_row(rslot, rl, res);
        // the warp's rows of the accumulator slot are read: the MMA warpgroups may write chunk k + 2 into it
        warp_arrive(smem_u32(&bars->acc_empty[slot]), lane);
        mbar_wait(smem_u32(&bars->t_empty[slot]), par ^ 1);   // P2 of chunk k - 2 has read the T slot
        __syncwarp();
        uint8_t* const tslot = smem + (smem_t - smem_base) + slot * ACT_SLICE_BYTES;
        if(row < p1.M) epilogue_row<F1>(p1, row, rl, c * NC, v, res, maskv, s_scale1 + c * NC, s_bias1 + c * NC, rslot, tslot);
        fence_proxy_async();   // the raw slice for its TMA store, the T slot for the wgmma that reads it
        epi_wg_sync();
        if(leader) {
          mbar_arrive(smem_u32(&bars->t_full[slot]));
          for(int h = 0; h < 2; h++)
            tma_store_2d(&tmapS1, smem_u32(rslot + h * (ACT_SLICE_BYTES / 2)), c * NC, m0 + h * (BLOCK_M / 2));
          bulk_commit();
          // the previous chunk's store has read its residual slot: the slot may be refilled (only warp 0 waits for that)
          bulk_wait_read1();
          if(prev_rs >= 0) mbar_arrive(smem_u32(&bars->r_empty[prev_rs]));
          // the previous tile's exit part, once the stores of this tile's first 4 chunks are the only ones that may be in flight:
          // publishing at the end of a tile would hold the warpgroup until its last stores are complete
          if(c == 3 && pending >= 0) chain_publish_before4(p1.tile_flags, pending);
        }
        prev_rs = rs;
        if(++rs == RES_SLOTS) { rs = 0; rphase ^= 1; }
      }
      pending = tile;
    }
    if(leader && pending >= 0) chain_publish(p1.tile_flags, pending);
    if(leader) bulk_wait0();
    pdl_wait();
    return;
  }

  // ===================== MMA warpgroups: warpgroup g owns tile rows 64g..64g+63 =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 184;");
  const int g = (warp - 4) >> 2, q = warp & 3;
  const bool leader = q == 0 && lane == 0;
  const int rloc = g * 64 + q * 16 + (lane >> 2);
  for(int i = threadIdx.x - 128; i < N2; i += 32 * CONSUMER_WARPS) { s_scale2[i] = __ldg(p2.bn_scale + i); s_bias2[i] = __ldg(p2.bn_bias + i); }
  consumer_sync();

  int stage = 0, ps = 0, as = 0, k = 0;   // k: as the epilogue warpgroup's
  uint32_t phase = 0, aphase = 0;
  uint8_t* const acc_ring = smem + (smem_acc - smem_base);
  uint8_t* const stg_ring = smem + (smem_stg - smem_base);
  uint8_t* const act_ring = smem + (smem_act - smem_base);
  int pending = -1;   // the tile whose stores this warpgroup issued last and has not published yet
  float acc1[NC / 2];
  // P1 of the chunk with index kc (acc1 = A rows 64g.. x the W1 chunk of the next weight stage, K1 / 64 k-blocks of 4 k16 steps, as
  // the exit's launch sums them), handed to the epilogue warpgroup through accumulator slot kc & 1 once it has read chunk kc - 2
  // out of it.  The wait for P1 also completes every P2 issued before it.
  auto handChunk = [&](int kc, bool last) {
#pragma unroll
    for(int i = 0; i < NC / 2; i++) acc1[i] = 0.0f;
    fence_acc(acc1);
    wgmma_fence();
    const int st1 = take_stage(bars->full, stages, stage, phase);
    const uint32_t w = smem_w + st1 * W_BYTES, a = smem_base + g * 64 * 128;
#pragma unroll
    for(int kb = 0; kb < K1 / BLOCK_K; kb++)
#pragma unroll
      for(int j = 0; j < 4; j++)
        WgmmaSS<NC>::mma(acc1, make_smem_desc(a + kb * BLOCK_M * 128) + 2 * j, make_smem_desc(w + kb * NC * 128) + 2 * j);
    wgmma_commit();
    wgmma_wait0();
    fence_acc(acc1);
    warp_arrive(smem_u32(&bars->empty[st1]), lane);
    if(last) warp_arrive(smem_u32(&bars->a_empty), lane);   // the tile's last P1: the next tile's A may land
    const int slot = kc & 1;
    mbar_wait(smem_u32(&bars->acc_empty[slot]), ((kc >> 1) & 1) ^ 1);
    store_acc_slices<NC>(acc_ring + slot * ACC_SLICE_BYTES, acc1, rloc, lane);
    warp_arrive(smem_u32(&bars->acc_full[slot]), lane);
  };
  bool have0 = false;   // the tile's chunk 0 was handed over before the previous tile's entry epilogue
  for(int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int m0 = tile * BLOCK_M;
    const float mask0 = m0 + rloc < p1.M ? __ldg(p1.mask + m0 + rloc) : 0.0f;
    const float mask1 = m0 + rloc + 8 < p1.M ? __ldg(p1.mask + m0 + rloc + 8) : 0.0f;
    float acc2[N2 / 2];
#pragma unroll
    for(int i = 0; i < N2 / 2; i++) acc2[i] = 0.0f;
    fence_acc(acc2);   // no access to acc2 from here to the tile's last wait: P2(c - 1) runs on while P1(c) is handed off
    if(!have0) {
      mbar_wait(smem_u32(&bars->a_full), aphase);
      aphase ^= 1;
    }
    // P2(c): acc2 += T slot rows 64g.. x W2 chunk c (its k16 steps in order), once the epilogue warpgroup has filled the slot;
    // returns the weight stage, released with the T slot once the MMAs are complete (releaseP2)
    auto issueP2 = [&](int c) {
      const int tslot = (k + c) & 1;
      mbar_wait(smem_u32(&bars->t_full[tslot]), ((k + c) >> 1) & 1);
      const int st = take_stage(bars->full, stages, stage, phase);
      const uint32_t w = smem_w + st * W_BYTES, t = smem_t + tslot * ACT_SLICE_BYTES + g * 64 * 64;
#pragma unroll
      for(int j = 0; j < NC / 16; j++) WgmmaSS<N2>::mma(acc2, make_smem_desc_sw64(t) + 2 * j, make_smem_desc_sw64(w) + 2 * j);
      wgmma_commit();
      return st;
    };
    auto releaseP2 = [&](int c, int st) {
      warp_arrive(smem_u32(&bars->empty[st]), lane);
      warp_arrive(smem_u32(&bars->t_empty[(k + c) & 1]), lane);
    };
    // Chunk c: P1(c), handed to the epilogue warpgroup as soon as it is complete; then P2(c - 1) once the epilogue warpgroup has
    // made T slot (c - 1) & 1 out of chunk c - 1.  So the epilogue warpgroup finds chunk c ready when it finishes chunk c - 1, and
    // runs it while the MMA warpgroups issue P2(c - 1) and P1(c + 1).
    int st2 = -1;   // the weight stage of the P2 in flight
#pragma unroll 1
    for(int c = have0 ? 1 : 0; c < chunks; c++) {
      handChunk(k + c, c + 1 == chunks);   // P1(c) and P2(c - 2) are complete
      if(st2 >= 0) releaseP2(c - 2, st2);
      // the previous tile's entry stores were issued 3 chunks ago
      if(c == 3 && leader && pending >= 0) chain_publish(p1.tile_flags, pending);
      st2 = c > 0 ? issueP2(c - 1) : -1;
    }
    const int st2_last = issueP2(chunks - 1);
    wgmma_wait0();
    fence_acc(acc2);
    releaseP2(chunks - 2, st2);
    releaseP2(chunks - 1, st2_last);
    k += chunks;
    // the next tile's chunk 0 goes to the epilogue warpgroup now, so that it does not idle through this tile's entry epilogue
    have0 = tile + (int)gridDim.x < tiles;
    if(have0) {
      mbar_wait(smem_u32(&bars->a_full), aphase);
      aphase ^= 1;
      handChunk(k, false);
    }

    pair_entry_epilogue<F2, N2, ACT_SLICE_BYTES>(p2, acc2, m0, g, rloc, lane, leader, mask0, mask1, s_scale2, s_bias2, stg_ring, act_ring,
                                                 ps, as, tmapS2, tmapA2, bars->r_empty, -1);
    pending = tile;
  }
  if(leader && pending >= 0) chain_publish(p1.tile_flags, pending);
  if(leader) bulk_wait0();
  pdl_wait();
}

template <int N2, int N1>
static cudaError_t pairFuncAttrs() {
  for(cudaError_t e : {cudaFuncSetAttribute(kgb_conv_pair_kernel<N2, N1, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT),
                       cudaFuncSetAttribute(kgb_conv_pair_kernel<N2, N1, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT),
                       cudaFuncSetAttribute(kgb_conv_pair_kernel<N2, N1, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT)})
    if(e != cudaSuccess) return e;
  return cudaSuccess;
}

// The (inner, trunk) widths of the nested-bottleneck nets: tiny_nbt, mid_nbt, b18c384nbt.  b28c512nbt's (256, 512) spills with fp32
// streams (256-column acc2 next to acc1), so its boundaries keep two launches.
#define KGB_PAIR_SHAPES(X) X(64, 64) X(64, 128) X(192, 384)

// The (inner, trunk) widths kgb_conv_pair_epi_kernel is compiled for: b18c384nbt's
#define KGB_PAIR_EPI_SHAPES(X) X(192, 384)

static cudaError_t convPairInit() {
#define KGB_PAIR_ATTR(N2, N1) pairFuncAttrs<N2, N1>(),
#define KGB_PAIR_EPI_ATTR(N2, N1) cudaFuncSetAttribute(kgb_conv_pair_epi_kernel<N2, N1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT),
  for(cudaError_t e : {KGB_PAIR_SHAPES(KGB_PAIR_ATTR) KGB_PAIR_EPI_SHAPES(KGB_PAIR_EPI_ATTR)})
    if(e != cudaSuccess) return e;
#undef KGB_PAIR_EPI_ATTR
#undef KGB_PAIR_ATTR
  return cudaSuccess;
}

static bool pairShapeCompiled(int n2, int n1) {
#define KGB_PAIR_IS(N2, N1) (n2 == N2 && n1 == N1) ||
  return KGB_PAIR_SHAPES(KGB_PAIR_IS) false;
#undef KGB_PAIR_IS
}

bool convPairSupported(const ConvParams& p1, const ConvParams& p2) {
  const int n2 = p2.cout_p;
  return p1.ky == 1 && p1.kx == 1 && p2.ky == 1 && p2.kx == 1 && !p1.split && !p2.split && p1.cin_p == n2 && p2.cin_p == p1.cout_p &&
         pairShapeCompiled(n2, p1.cout_p) && p2.n_tile == n2 && p1.M == p2.M &&
         p1.residual != nullptr && p1.raw_out != nullptr && p1.ncbias == nullptr && p1.act == 2 && p2.residual == nullptr &&
         p2.raw_out != nullptr && p2.act_out != nullptr && p2.ncbias == nullptr && p2.act == 2 &&
         (p1.residual_fp32 != 0) == (p1.raw_fp32 != 0) && !(p2.raw_fp32 && !p1.raw_fp32) && pairLayout(p1, p2).stages >= 2;
}

bool convPairEpilogueWG(const ConvParams& p1, const ConvParams& p2) {
  if(!p1.pair_epi_wg || p1.residual_fp32 || p1.raw_fp32 || p2.raw_fp32 || !convPairSupported(p1, p2)) return false;
  bool shape = false;
#define KGB_PAIR_EPI_IS(N2, N1) shape = shape || (p2.cout_p == N2 && p1.cout_p == N1);
  KGB_PAIR_EPI_SHAPES(KGB_PAIR_EPI_IS)
#undef KGB_PAIR_EPI_IS
  return shape && pairEpiLayout(p1, p2).stages >= 4;
}

int convPairChainParts(const ConvParams& p1, const ConvParams& p2) { return convPairEpilogueWG(p1, p2) ? 3 : kConvPairParts; }

template <int N2, int N1>
static cudaError_t launchPairN(const ConvPairTmaps& tm, const ConvParams& p1, const ConvParams& p2, int grid, const SmemLayout& l,
                               cudaStream_t stream) {
  auto k = p1.raw_fp32 ? (p2.raw_fp32 ? kgb_conv_pair_kernel<N2, N1, true, true> : kgb_conv_pair_kernel<N2, N1, true, false>)
                       : kgb_conv_pair_kernel<N2, N1, false, false>;
  return launchChained(k, p1, grid, THREADS, l.smem, stream, tm.A, tm.W1, tm.W2, tm.stream1, tm.stream2, tm.act2, p1, p2, l.stages, l.r_slots);
}

cudaError_t launchConvPair(const ConvPairTmaps& tm, const ConvParams& p1, const ConvParams& p2, cudaStream_t stream) {
  if(!convPairSupported(p1, p2) || p1.tile_flags == nullptr) return cudaErrorInvalidValue;
  int sms = 0;
  const cudaError_t e = smCount(&sms);
  if(e != cudaSuccess) return e;
  const int grid = std::min(p1.num_m_tiles, sms);
  if(convPairEpilogueWG(p1, p2)) {
    const SmemLayout l = pairEpiLayout(p1, p2);
#define KGB_PAIR_EPI_LAUNCH(N2, N1)                                                                                                         \
    if(p2.cout_p == N2 && p1.cout_p == N1)                                                                                                   \
      return launchChained(kgb_conv_pair_epi_kernel<N2, N1>, p1, grid, PAIR_EPI_THREADS, l.smem, stream, tm.A, tm.W1, tm.W2, tm.stream1, \
                           tm.stream2, tm.act2, p1, p2, l.stages);
    KGB_PAIR_EPI_SHAPES(KGB_PAIR_EPI_LAUNCH)
#undef KGB_PAIR_EPI_LAUNCH
  }
  const SmemLayout l = pairLayout(p1, p2);
#define KGB_PAIR_LAUNCH(N2, N1) if(p2.cout_p == N2 && p1.cout_p == N1) return launchPairN<N2, N1>(tm, p1, p2, grid, l, stream);
  KGB_PAIR_SHAPES(KGB_PAIR_LAUNCH)
#undef KGB_PAIR_LAUNCH
  return cudaErrorInvalidValue;
}

}  // namespace kgb
