// Tensor-core implicit-GEMM convolution for sm_90a: TMA-staged channels-last tiles -> shared memory (128B swizzle) ->
// wgmma (m64 x Nt x k16 per warpgroup, fp16 in, fp32 accumulators in registers) -> epilogue with folded-BN scale/shift,
// residual and ReLU staged in shared memory: the residual tile arrives and the output tile leaves by TMA (plain conv,
// stride-phase transposed conv, grouped outputs).
//
// GEMM view:  M = output positions (tile = a bw x bh x bd x bn box of 128 positions),
//             N = output channels (tile Nt = 16 / 32 / 64 / 128), K = taps x Cin.
// For every filter tap the A tile is ONE TMA box load of the input tensor shifted by the tap
// offset; out-of-range coordinates are zero-filled by TMA, which implements the padding.
//
// Precision: activations and weights travel as split-fp16 rows [32 hi | 32 lo] (x = hi + lo, see common.cuh).  Per 16-wide K
// slice the kernel accumulates hi*hi into D1 and hi*lo + lo*hi into D2 and the epilogue forms D1 + D2 (~22 significand bits per
// operand, the dropped lo*lo term is 2^-22 relative: fp32-grade results from the fp16 pipe); keeping the small cross products out
// of the big accumulator limits the rounding of the accumulation steps.  LT_CONV_TC1 (fast mode) issues hi*hi only.
//
// Weights: [tap][Cin/32][CoutP rows][32 hi | 32 lo] fp16 (128-byte rows), so the K slices of both operands are descriptor offsets
// (+0, +2 hi; +4, +6 lo, in 16-byte units).
//
// Warp roles (384 threads): warpgroup 0 = TMA producers (warp 0 fills the operand ring, warp 1 owns the epilogue buffers),
// warpgroups 1 and 2 = MMA + epilogue for rows 0-63 and 64-127 of the M tile.  The operand ring is released per stage by one
// arrival of each consumer warpgroup once its MMAs that read the stage have completed (wgmma.wait_group 1 keeps one chunk of MMAs
// in flight behind the issue).
//
// Epilogue: stored straight from the accumulators, each residual load of a 128-channel tile would wait behind the previous store
// (the output may alias the residual): 32 dependent memory round trips per unit with the tensor cores idle.  So warp 1 TMA-loads
// the unit's residual tile into a shared-memory buffer while the K loop runs, the consumers turn it into the output tile in place
// with shared-memory accesses only, and warp 1 TMA-stores it while the next unit's K loop runs.  Warp 0 never waits on that
// buffer.  Launches with short K loops (tc_layout) keep two such buffers and alternate between them, so the next unit's residual
// load does not wait for this unit's epilogue and store.  16-channel tiles (half a 32-channel slab) keep the register store.
//
// Persistent grid: min(work units, SMs) CTAs stride over the work units (M tile x N tile x K split, N tile fastest).  Producer and
// consumers keep one ring across unit boundaries, so the next unit's first boxes load while the consumers run the epilogue; on the
// 1x1 layers of the backbone (2-8 K chunks per tile) the fill was most of a one-tile CTA's time.  The K split count comes from a
// launch-time model (tc_plan, exported as lt_conv_tc_plan); split units write fp32 partial tiles that splitk_reduce_kernel sums in
// a fixed order.
#include "tc_common.cuh"
#include "conv_tc_params.cuh"
#include <stdlib.h>
#include <string.h>

namespace lt {

// ------------------------------------------------------------------------------------------------
// Kernel
// ------------------------------------------------------------------------------------------------
constexpr int kTcThreads = 384;

// Work unit u of the persistent grid: N tile fastest, so the N tiles of one M tile (which read the same A boxes) run side by side
// in time and the A boxes are L2 hits for all but the first; then M tile; the K split z outermost.
struct TcUnit {
  int m, n0, z, q_begin, nchunks;
  int k, c;   // chain mode: block and layer class (0 otherwise)
};
__device__ __forceinline__ TcUnit tc_unit(const TcParams& p, int u, int m_tiles, int nchunks_all) {
  TcUnit w;
  const int n = u % p.n_tiles;
  u /= p.n_tiles;
  w.m = u % m_tiles;
  w.z = u / m_tiles;
  w.n0 = n * p.Nt;
  w.q_begin = (int)(((long)w.z * nchunks_all) / p.splits);
  w.nchunks = (int)(((long)(w.z + 1) * nchunks_all) / p.splits) - w.q_begin;
  w.k = w.c = 0;
  return w;
}
__device__ __forceinline__ void tc_tile_origin(const TcParams& p, int t, int& ow0, int& oh0, int& od0, int& nb0) {
  ow0 = (t % p.tw) * p.bw; t /= p.tw;
  oh0 = (t % p.th) * p.bh; t /= p.th;
  od0 = (t % p.td) * p.bd;
  nb0 = (t / p.td) * p.bn;
}

// The epilogue tile buffer: per 32 output channels one 16 KB slab of 128 rows (M-tile positions) x 128 bytes, [32 hi | 32 lo]
// fp16 or 32 fp32, 128-byte swizzled like the A box.  Units of a launch without K split and with whole slabs use it.
constexpr int kSlabBytes = 128 * 128;
__host__ __device__ constexpr int tc_epi_bytes(int nt, int splits) { return (nt >= 32 && splits == 1) ? nt / 32 * kSlabBytes : 0; }

// map index and box channel coordinate of the slab that starts at GEMM column co (a multiple of 32)
__device__ __forceinline__ void epi_slab(const TcParams& p, int co, int& g, int& c) {
  g = p.n_maps > 1 ? co / p.oc : 0;
  const int ch = co - g * p.oc;
  c = p.out_format == LT_FMT_F32 ? ch : 2 * ch;
}

// byte offset of byte b of row `row` in a 128-byte-swizzled slab (16-byte chunk j of row r sits at chunk j ^ (r % 8))
__device__ __forceinline__ uint32_t sw128(int row, int b) {
  return (uint32_t)(row * 128 + ((((b >> 4) ^ row) & 7) << 4) + (b & 15));
}

// ---- chain mode (lt_conv_tc_chain_fwd): one persistent launch over a run of identical bottleneck blocks ----
// Layer c of block k (c = 0: 1x1 reduce, 1: the 3x3, 2: 1x1 expansion + residual) is layer 3k + c of the chain.  All layers share
// the output grid and the M-tile box of the launch's TcParams; what differs per layer class is below, per block the filter and the
// folded scale / shift.  Units are numbered layer-major, then M tile, then N tile, so every unit's inputs come from units with
// smaller numbers: CTAs take units in that order from one global counter and start each once the tiles it reads are stored.
constexpr int kChainMaxBlocks = 36;
constexpr int kChainRing = 4;   // unit ids in flight between a CTA's dispatching warp and its other roles
struct TcChainGeom {
  int blocks, m_tiles, units_per_block;
  int tw, th, td, tn, bw, bh, bd, bn, OW, OH, OD;
  int n_tiles[3], chunks[3], CB[3], KW[3], KH[3], KD[3], pw[3], ph[3], pd[3], CoutP[3], FC[3], residual[3], relu[3];
};
struct TcChain {
  CUtensorMap a[3][2];     // [class][block parity]: the A operand (block input X, Y1, Y2)
  CUtensorMap out[3][2];   // [class][block parity]: the output (Y1, Y2, X); the expansion writes its residual X in place
  CUtensorMap res;         // the expansion's residual: X
  CUtensorMap b[kChainMaxBlocks][3];
  const float* scale[kChainMaxBlocks][3];
  const float* shift[kChainMaxBlocks][3];
  unsigned* counters;      // [0]: next unit to take; [1 + layer * m_tiles + m]: N tiles of (layer, M tile m) stored
  TcChainGeom g;
};

__host__ __device__ inline void chain_unit(const TcChainGeom& g, int u, int& k, int& c, int& m, int& n) {
  k = u / g.units_per_block;
  int r = u - k * g.units_per_block;
  c = 0;
  while (c < 2 && r >= g.m_tiles * g.n_tiles[c]) { r -= g.m_tiles * g.n_tiles[c]; ++c; }
  m = r / g.n_tiles[c];
  n = r - m * g.n_tiles[c];
}

// The tiles unit (block k, class c, M tile m) reads: tiles lo..hi per axis (w, h, d, batch) of layer `src` = 3k + c - 1, the one
// that writes its input, each complete once `need` (that layer's N tiles) units have stored it.  The receptive field of the tile
// is clipped to the grid: what lies outside is padding, which TMA zero-fills.  false: the chain's first layer reads the input X.
__host__ __device__ inline bool chain_deps(const TcChainGeom& g, int k, int c, int m, int& src, int& need, int lo[4], int hi[4]) {
  if (k == 0 && c == 0) return false;
  src = 3 * k + c - 1;
  need = g.n_tiles[(c + 2) % 3];
  const int tile[3] = {m % g.tw, (m / g.tw) % g.th, (m / (g.tw * g.th)) % g.td};
  const int box[3] = {g.bw, g.bh, g.bd}, ext[3] = {g.OW, g.OH, g.OD};
  const int kk[3] = {g.KW[c], g.KH[c], g.KD[c]}, pad[3] = {g.pw[c], g.ph[c], g.pd[c]};
  for (int a = 0; a < 3; ++a) {
    int p0 = tile[a] * box[a] - pad[a], p1 = tile[a] * box[a] + box[a] - 1 - pad[a] + kk[a] - 1;
    p0 = p0 < 0 ? 0 : p0;
    p1 = p1 > ext[a] - 1 ? ext[a] - 1 : p1;
    lo[a] = p0 / box[a];
    hi[a] = p1 / box[a];
  }
  lo[3] = hi[3] = m / (g.tw * g.th * g.td);
  return true;
}

__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* a) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_add(unsigned* a, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(a), "r"(v) : "memory");
}
// orders generic-proxy accesses to global memory against the async proxy (TMA) of this thread
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
// Bounded like mbar_wait: a protocol bug traps instead of hanging the GPU.
__device__ __forceinline__ void wait_count(const unsigned* a, unsigned need) {
  if (ld_acquire_gpu(a) >= need) return;
  const long long t0 = clock64();
  while (ld_acquire_gpu(a) < need) {
    __nanosleep(100);
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}

template <int NT, bool CHAIN>
__device__ __forceinline__ void conv_tc_body(const CUtensorMap* tmA, const CUtensorMap* tmB, const TcEpiMaps* tmE, const TcParams& p,
                                             const TcChain* cp) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int kStage = kATileBytes + NT * 128;
  const int epi_bytes = tc_epi_bytes(NT, p.splits);
  const bool staged = epi_bytes > 0;
  uint8_t* ebuf = smem + (size_t)p.stages * kStage;   // p.epi_buffers tile buffers of epi_bytes
  uint64_t* full = reinterpret_cast<uint64_t*>(ebuf + p.epi_buffers * epi_bytes);
  uint64_t* empty = full + p.stages;
  uint64_t* efull = empty + p.stages;   // [b]: tile buffer b is free and holds its unit's residual
  uint64_t* edone = efull + 2;          // [b]: both consumer warpgroups wrote their unit's output into tile buffer b
  // chain: ring slot i holds the id of a unit taken by warp 0 (ufull) until warp 1's lane and the 8 consumer warps read it (uempty)
  uint64_t* ufull = edone + 2;
  uint64_t* uempty = ufull + kChainRing;
  volatile int* uid = reinterpret_cast<volatile int*>(uempty + kChainRing);

  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int lane = threadIdx.x & 31;
  const int m_tiles = p.tw * p.th * p.td * p.tn;
  int units = m_tiles * p.n_tiles * p.splits;
  if constexpr (CHAIN) units = cp->g.blocks * cp->g.units_per_block;
  const int nchunks_all = p.KD * p.KH * p.KW * p.CB;
  auto unit_of = [&](int u) {
    if constexpr (CHAIN) {
      TcUnit w;
      int n;
      chain_unit(cp->g, u, w.k, w.c, w.m, n);
      w.n0 = n * NT;
      w.z = 0;
      w.q_begin = 0;
      w.nchunks = cp->g.chunks[w.c];
      return w;
    } else {
      return tc_unit(p, u, m_tiles, nchunks_all);
    }
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    for (int b = 0; b < 2; ++b) { mbar_init(&efull[b], 1); mbar_init(&edone[b], 256); }
    if constexpr (CHAIN) {
      for (int i = 0; i < kChainRing; ++i) { mbar_init(&ufull[i], 1); mbar_init(&uempty[i], 9); }
    }
    fence_barrier_init();
    if constexpr (CHAIN) {
      for (int c = 0; c < 3; ++c)
        for (int q = 0; q < 2; ++q) { prefetch_tmap(&cp->a[c][q]); prefetch_tmap(&cp->out[c][q]); }
      prefetch_tmap(&cp->res);
    } else {
      prefetch_tmap(tmA);
      prefetch_tmap(tmB);
    }
  }
  __syncthreads();

  if (wg == 0) {
    regs_release_producer();
    if (staged && threadIdx.x == 32) {
      // ================= epilogue buffers (warp 1, one lane): residual tiles in, output tiles out =================
      // The k-th unit of this CTA uses buffer k % epi_buffers.  With two buffers the next unit's residual load is issued as soon
      // as the previous unit's store has read the other buffer, ahead of this unit's epilogue: it overlaps this unit's K loop,
      // epilogue and store and the next unit's K loop, so the consumers find it there when they finish that K loop.  With one
      // buffer it waits until this unit's store has read the buffer.  A unit's store overlaps the next unit's K loop either way.
      const int nbuf = p.epi_buffers;
      auto load_residual = [&](int u, int b) {
        uint8_t* buf = ebuf + b * epi_bytes;
        const TcUnit w = unit_of(u);
        int res_mode = p.residual;
        if constexpr (CHAIN) res_mode = cp->g.residual[w.c];
        if (res_mode == LT_RES_NONE) {
          mbar_arrive_local(&efull[b]);
          return;
        }
        int ow0, oh0, od0, nb0;
        tc_tile_origin(p, w.m, ow0, oh0, od0, nb0);
        if constexpr (CHAIN) fence_proxy_async_global();   // the tiles were stored by other CTAs (warp 0 acquired them)
        mbar_expect_tx(&efull[b], (uint32_t)epi_bytes);   // out-of-range positions and channels arrive as zeros
        for (int sl = 0; sl < NT / 32; ++sl) {
          int g, c;
          epi_slab(p, w.n0 + 32 * sl, g, c);
          tma_load_5d(buf + sl * kSlabBytes, CHAIN ? &cp->res : &tmE->res[g], &efull[b], c, ow0, oh0, od0, nb0);
        }
      };
      uint32_t eph = 0;   // bit b: phase of edone[b]
      if constexpr (CHAIN) {
        // One buffer.  A unit counts as stored once its TMA store has completed (not only read shared memory); its (layer, M tile)
        // counter is raised before this lane waits for the next unit id, which may be a unit that depends on this one.
        int rs = 0;
        uint32_t rph = 0;
        auto take = [&]() {
          mbar_wait(&ufull[rs], rph);
          const int v = uid[rs];
          mbar_arrive_local(&uempty[rs]);
          if (++rs == kChainRing) { rs = 0; rph ^= 1u; }
          return v;
        };
        int u = take();
        if (u < units) load_residual(u, 0);
        while (u < units) {
          const TcUnit w = unit_of(u);
          int ow0, oh0, od0, nb0;
          tc_tile_origin(p, w.m, ow0, oh0, od0, nb0);
          mbar_wait(&edone[0], eph & 1u);
          eph ^= 1u;
          for (int sl = 0; sl < NT / 32; ++sl) {
            int g, c;
            epi_slab(p, w.n0 + 32 * sl, g, c);
            tma_store_5d(&cp->out[w.c][w.k & 1], ebuf + sl * kSlabBytes, c, ow0, oh0, od0, nb0);
          }
          bulk_commit();
          bulk_wait0();
          fence_proxy_async_global();
          red_release_gpu_add(cp->counters + 1 + (size_t)(3 * w.k + w.c) * m_tiles + w.m, 1u);
          u = take();
          if (u < units) load_residual(u, 0);
        }
      } else {
        int b = 0;
        if (blockIdx.x < units) load_residual(blockIdx.x, 0);
        for (int u = blockIdx.x; u < units; u += gridDim.x) {
          const int un = u + gridDim.x, bn = b ^ (nbuf - 1);
          if (nbuf == 2 && un < units) {
            bulk_wait_read0();                    // the previous unit's store has read buffer bn
            load_residual(un, bn);
          }
          const TcUnit w = tc_unit(p, u, m_tiles, nchunks_all);
          int ow0, oh0, od0, nb0;
          tc_tile_origin(p, w.m, ow0, oh0, od0, nb0);
          mbar_wait(&edone[b], (eph >> b) & 1u);
          eph ^= 1u << b;
          for (int sl = 0; sl < NT / 32; ++sl) {  // clipped at the edges of the output grid and at FC
            int g, c;
            epi_slab(p, w.n0 + 32 * sl, g, c);
            tma_store_5d(&tmE->out[g], ebuf + b * epi_bytes + sl * kSlabBytes, c, ow0, oh0, od0, nb0);
          }
          bulk_commit();
          if (nbuf == 1 && un < units) {
            bulk_wait_read0();                    // this unit's store has read the buffer
            load_residual(un, 0);
          }
          b = bn;
        }
        bulk_wait0();
      }
    }
    // ================= TMA producer (warp 0 runs the loop; one elected lane issues) =================
    // The ring slot / phase run on across units: the next unit's boxes load while the consumers run the previous epilogue.
    if (threadIdx.x < 32) {
      int s = 0;
      uint32_t ph = 0;
      int rs = 0;
      uint32_t rph = 0;
      // chain: take the next unit, wait until the tiles it reads are stored, then hand its id to the other roles
      auto take = [&]() {
        mbar_wait(&uempty[rs], rph ^ 1u);
        int u = 0;
        if (lane == 0) u = (int)atomicAdd(cp->counters, 1u);
        u = __shfl_sync(0xffffffffu, u, 0);
        u = u < units ? u : units;
        if (u < units) {
          int k, c, m, n, src, need, lo[4], hi[4];
          chain_unit(cp->g, u, k, c, m, n);
          if (chain_deps(cp->g, k, c, m, src, need, lo, hi)) {
            const int nw = hi[0] - lo[0] + 1, nh = hi[1] - lo[1] + 1, nd = hi[2] - lo[2] + 1;
            for (int i = lane; i < nw * nh * nd; i += 32) {
              const int t = ((hi[3] * cp->g.td + lo[2] + i / (nw * nh)) * cp->g.th + lo[1] + (i / nw) % nh) * cp->g.tw + lo[0] + i % nw;
              wait_count(cp->counters + 1 + (size_t)src * m_tiles + t, (unsigned)need);
            }
            __syncwarp();
            fence_proxy_async_global();   // the TMA loads below read what the acquired stores wrote
          }
        }
        if (lane == 0) {
          uid[rs] = u;
          mbar_arrive_local(&ufull[rs]);
        }
        __syncwarp();
        if (++rs == kChainRing) { rs = 0; rph ^= 1u; }
        return u;
      };
      int u;
      if constexpr (CHAIN) u = take();
      else u = blockIdx.x;
      while (u < units) {
        const TcUnit w = unit_of(u);
        int ow0, oh0, od0, nb0;
        tc_tile_origin(p, w.m, ow0, oh0, od0, nb0);
        int CB = p.CB, KW = p.KW, KH = p.KH, pw = p.pw, ph_ = p.ph, pd = p.pd, b_step1 = p.b_step1;
        const CUtensorMap* mA = tmA;
        const CUtensorMap* mB = tmB;
        if constexpr (CHAIN) {
          const TcChainGeom& g = cp->g;
          CB = g.CB[w.c]; KW = g.KW[w.c]; KH = g.KH[w.c]; pw = g.pw[w.c]; ph_ = g.ph[w.c]; pd = g.pd[w.c]; b_step1 = g.CoutP[w.c];
          mA = &cp->a[w.c][w.k & 1];
          mB = &cp->b[w.k][w.c];
        }
        // chunk -> (tap, channel block) advanced incrementally: no integer division in the loop
        int tap = w.q_begin / CB, cb = w.q_begin - tap * CB;
        int kw = tap % KW, kh = (tap / KW) % KH, kd = tap / (KW * KH);
        const int ax = ow0 * p.sw - pw, ay = oh0 * p.sh - ph_, az = od0 * p.sd - pd, bn0 = w.n0 * p.b_nmul;
        for (int q = 0, qa = w.q_begin; q < w.nchunks; ++q, ++qa) {
          mbar_wait(&empty[s], ph ^ 1u);
          uint8_t* a_dst = smem + (size_t)s * kStage;
          if (elect_one()) {
            mbar_expect_tx(&full[s], (uint32_t)kStage);
            tma_load_5d(a_dst, mA, &full[s], cb * 64, ax + kw, ay + kh, az + kd, nb0);
            tma_load_2d(a_dst + kATileBytes, mB, &full[s], qa * p.b_step0, qa * b_step1 + bn0);
          }
          __syncwarp();
          if (++cb == CB) { cb = 0; if (++kw == KW) { kw = 0; if (++kh == KH) { kh = 0; ++kd; } } }
          if (++s == p.stages) { s = 0; ph ^= 1u; }
        }
        if constexpr (CHAIN) u = take();
        else u += gridDim.x;
      }
    }
    return;
  }

  // ================= MMA + epilogue (warpgroups 1, 2: rows 64 (wg - 1) .. +63 of the M tile) =================
  regs_claim_consumer();
  const int g = wg - 1;
  float d1[NT / 2], d2[NT / 2];
#pragma unroll
  for (int i = 0; i < NT / 2; ++i) { d1[i] = 0.f; d2[i] = 0.f; }
  // this thread holds rows r0 and r0 + 8, columns 8i + c2 (+1) of the 64 x NT warpgroup tile
  const int r0 = g * 64 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
  const int c2 = 2 * (lane & 3);
  const uint32_t ring0 = smem_u32(smem);
  int s = 0;
  uint32_t ph = 0;
  int eb = 0;          // tile buffer of this unit (staged epilogue)
  uint32_t eph = 0;    // bit b: phase of efull[b]
  int rs = 0;
  uint32_t rph = 0;
  auto take = [&]() {  // chain: every thread reads the id, one arrival per warp
    mbar_wait(&ufull[rs], rph);
    const int v = uid[rs];
    __syncwarp();
    if (lane == 0) mbar_arrive_local(&uempty[rs]);
    if (++rs == kChainRing) { rs = 0; rph ^= 1u; }
    return v;
  };
  int u;
  if constexpr (CHAIN) u = take();
  else u = blockIdx.x;
  for (; u < units; u = CHAIN ? take() : u + (int)gridDim.x) {
    const TcUnit w = unit_of(u);
    int prev = -1;
    for (int q = 0; q < w.nchunks; ++q) {
      mbar_wait(&full[s], ph);
      const uint32_t a_addr = ring0 + (uint32_t)(s * kStage) + (uint32_t)(g * 64 * 128);
      const uint32_t b_addr = ring0 + (uint32_t)(s * kStage) + kATileBytes;
      const uint64_t ad = make_sw128_desc(a_addr), bd = make_sw128_desc(b_addr);
      const uint32_t acc = (q == 0) ? 0u : 1u;
      wg_fence();
      if (p.terms == 3) {
        wgmma_f16<NT>(d1, ad, bd, acc);              // hi * hi
        wgmma_f16<NT>(d1, ad + 2, bd + 2, 1u);
        wgmma_f16<NT>(d2, ad, bd + 4, acc);          // hi * lo
        wgmma_f16<NT>(d2, ad + 2, bd + 6, 1u);
        wgmma_f16<NT>(d2, ad + 4, bd, 1u);           // lo * hi
        wgmma_f16<NT>(d2, ad + 6, bd + 2, 1u);
      } else if (p.terms == 1) {
        wgmma_f16<NT>(d1, ad, bd, acc);              // high parts only
        wgmma_f16<NT>(d1, ad + 2, bd + 2, 1u);
      } else {
        // plain fp16 rows (self test): 4 slices of 16
        wgmma_f16<NT>(d1, ad, bd, acc);
        wgmma_f16<NT>(d1, ad + 2, bd + 2, 1u);
        wgmma_f16<NT>(d1, ad + 4, bd + 4, 1u);
        wgmma_f16<NT>(d1, ad + 6, bd + 6, 1u);
      }
      wg_commit();
      wg_wait<1>();                                   // the MMAs of chunk q - 1 have completed: release its stage
      if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive_local(&empty[prev]);
      prev = s;
      if (++s == p.stages) { s = 0; ph ^= 1u; }
    }
    wg_wait<0>();
    if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive_local(&empty[prev]);   // the producer refills it during the epilogue
    wg_fence_regs(d1);
    wg_fence_regs(d2);

    // ---- epilogue ----
    if (p.splits > 1) {
      // ---- split-K: raw accumulators to the workspace, epilogue deferred to splitk_reduce_kernel ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float* wrow = p.ws + (((size_t)w.z * m_tiles + w.m) * 128 + r0 + 8 * h) * p.ws_ld + w.n0;
#pragma unroll
        for (int i = 0; i < NT / 8; ++i) {
          const int k = 4 * i + 2 * h;
          const float v0 = (p.terms == 3) ? fmaf(d2[k], kLoInv, d1[k]) : d1[k];
          const float v1 = (p.terms == 3) ? fmaf(d2[k + 1], kLoInv, d1[k + 1]) : d1[k + 1];
          *reinterpret_cast<float2*>(wrow + 8 * i + c2) = make_float2(v0, v1);
        }
      }
      continue;
    }
    if constexpr (NT >= 32) {
      // ---- staged: the residual comes from and the output goes to tile buffer eb; warp 1 moves both with TMA ----
      // The arithmetic is conv_epilogue_row's.  A thread's residual and output elements share their addresses.
      int FC = p.FC, res_mode = p.residual, relu = p.relu;
      const float* scale = p.scale;
      const float* shift = p.shift;
      if constexpr (CHAIN) {
        FC = cp->g.FC[w.c]; res_mode = cp->g.residual[w.c]; relu = cp->g.relu[w.c];
        scale = cp->scale[w.k][w.c];
        shift = cp->shift[w.k][w.c];
      }
      mbar_wait(&efull[eb], (eph >> eb) & 1u);
      eph ^= 1u << eb;
      const uint32_t e0 = smem_u32(ebuf + eb * epi_bytes);
      // Column group i + 1's scale and shift load while group i is processed: the compiler does not move loads across the
      // shared-memory accesses (volatile asm), so a load issued in its own iteration would wait a full L1 round trip.
      auto fc_ok = [&](int co) {
        int ch;
        long pix;
        epilogue_target(p, co, 0, ch, pix);
        return ch < FC;
      };
      float2 sc = make_float2(0.f, 0.f), sh = sc;
      if (fc_ok(w.n0 + c2)) {
        sc = __ldg(reinterpret_cast<const float2*>(scale + w.n0 + c2));
        sh = __ldg(reinterpret_cast<const float2*>(shift + w.n0 + c2));
      }
#pragma unroll
      for (int i = 0; i < NT / 8; ++i) {
        const int co = w.n0 + 8 * i + c2;
        const bool ok = fc_ok(co);
        float2 sc_next = sc, sh_next = sh;
        if (i + 1 < NT / 8 && fc_ok(co + 8)) {
          sc_next = __ldg(reinterpret_cast<const float2*>(scale + co + 8));
          sh_next = __ldg(reinterpret_cast<const float2*>(shift + co + 8));
        }
        const uint32_t slab = e0 + (uint32_t)((i >> 2) * kSlabBytes);
        const int cc = 8 * (i & 3) + c2;   // column in the slab
#pragma unroll
        for (int h = 0; h < 2 && ok; ++h) {
          const int row = r0 + 8 * h;
          const int k = 4 * i + 2 * h;
          float v0 = (p.terms == 3) ? fmaf(d2[k], kLoInv, d1[k]) : d1[k];
          float v1 = (p.terms == 3) ? fmaf(d2[k + 1], kLoInv, d1[k + 1]) : d1[k + 1];
          v0 = fmaf(v0, sc.x, sh.x);
          v1 = fmaf(v1, sc.y, sh.y);
          if (p.out_format == LT_FMT_F32) {
            const uint32_t a = slab + sw128(row, 4 * cc);
            float2 r = make_float2(0.f, 0.f);
            if (res_mode != LT_RES_NONE) r = lds_f2(a);
            if (res_mode == LT_RES_BEFORE_RELU) { v0 += r.x; v1 += r.y; }
            if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            if (res_mode == LT_RES_AFTER_RELU) { v0 += r.x; v1 += r.y; }
            sts_f2(a, make_float2(v0, v1));
          } else {
            const uint32_t ahi = slab + sw128(row, 2 * cc), alo = slab + sw128(row, 64 + 2 * cc);
            float2 r = make_float2(0.f, 0.f);
            if (res_mode != LT_RES_NONE) {
              const uint32_t rh = lds32(ahi), rl = lds32(alo);
              const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&rh));
              const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&rl));
              r = make_float2(fmaf(b.x, kLoInv, a.x), fmaf(b.y, kLoInv, a.y));
            }
            if (res_mode == LT_RES_BEFORE_RELU) { v0 += r.x; v1 += r.y; }
            if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            if (res_mode == LT_RES_AFTER_RELU) { v0 += r.x; v1 += r.y; }
            uint32_t hi2, lo2;
            split_s32x2(v0, v1, hi2, lo2);
            sts32(ahi, hi2);
            sts32(alo, lo2);
          }
        }
        sc = sc_next;
        sh = sh_next;
      }
      fence_proxy_async();   // the generic-proxy writes become visible to the TMA store
      mbar_arrive_local(&edone[eb]);
      eb ^= p.epi_buffers - 1;
    } else {
      // ---- 16-channel tiles (half a slab): fused epilogue straight from the accumulator registers ----
      int ow0, oh0, od0, nb0;
      tc_tile_origin(p, w.m, ow0, oh0, od0, nb0);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        int r_ = r0 + 8 * h;
        const int dw = r_ % p.bw; r_ /= p.bw;
        const int dh = r_ % p.bh; r_ /= p.bh;
        const int dd = r_ % p.bd; r_ /= p.bd;
        const int ow = ow0 + dw, oh = oh0 + dh, od = od0 + dd, nb = nb0 + r_;
        if (!(ow < p.OW && oh < p.OH && od < p.OD && nb < p.N)) continue;
        const long opix = (((long)nb * p.FD + (od * p.osd + p.ood)) * p.FH + (oh * p.osh + p.ooh)) * p.FW + (ow * p.osw + p.oow);
        conv_epilogue_row<NT>(p, d1, d2, h, opix, w.n0, c2);
      }
    }
  }
}

template <int NT>
__global__ void __launch_bounds__(kTcThreads, 1) conv_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                const __grid_constant__ CUtensorMap tmB,
                                                                const __grid_constant__ TcEpiMaps tmE, const TcParams p) {
  conv_tc_body<NT, false>(&tmA, &tmB, &tmE, p, nullptr);
}

// Chain mode of conv_tc_kernel<128>: the K loop, products, epilogue and tile box are the per-layer kernel's, so every unit computes
// the bits its per-layer launch computes.  `p` holds what the chain's layers share (box, grid, format, terms, ring depth).
__global__ void __launch_bounds__(kTcThreads, 1) conv_tc_chain_kernel(const __grid_constant__ TcChain chain, const TcParams p) {
  conv_tc_body<128, true>(nullptr, nullptr, nullptr, p, &chain);
}

// ------------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// Encoded tensor maps are cached per host thread by their full argument list (base pointer, dims, strides, box, element strides,
// swizzle, type): an eager forward re-encodes the same ~300 maps every step otherwise (cuTensorMapEncodeTiled costs ~1-2 us each;
// graph replays never come here).  256-entry direct-mapped table, 64-bit FNV-1a key with full-argument verification.
struct MapKey {
  const void* base;
  int rank, swizzle, f32;
  uint64_t dims[5], strides[4];
  uint32_t box[5], es[5];
};
struct MapSlot {
  bool used = false;
  MapKey key;
  CUtensorMap map;
};

int make_map(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
             const uint32_t* box, const uint32_t* estrides, int swizzle128, int f32) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return fail(LT_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  MapKey key;
  memset(&key, 0, sizeof(key));
  key.base = base; key.rank = rank; key.swizzle = swizzle128; key.f32 = f32;
  for (int i = 0; i < rank; ++i) { key.dims[i] = dims[i]; key.box[i] = box[i]; key.es[i] = estrides ? estrides[i] : 1; }
  for (int i = 0; i + 1 < rank; ++i) key.strides[i] = strides_bytes[i];
  uint64_t h = 1469598103934665603ull;
  const unsigned char* kb = reinterpret_cast<const unsigned char*>(&key);
  for (size_t i = 0; i < sizeof(key); ++i) { h ^= kb[i]; h *= 1099511628211ull; }
  static thread_local MapSlot cache[256];
  MapSlot& slot = cache[(h ^ (h >> 29)) & 255];
  if (slot.used && memcmp(&slot.key, &key, sizeof(key)) == 0) {
    *map = slot.map;
    return LT_OK;
  }
  cuuint64_t gd[5], gs[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = estrides ? estrides[i] : 1; }
  for (int i = 0; i + 1 < rank; ++i) gs[i] = strides_bytes[i];
  CUresult r = fn(map, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle128 == 1 ? CU_TENSOR_MAP_SWIZZLE_128B : (swizzle128 == 2 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE),
                  CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(LT_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  slot.used = true;
  slot.key = key;
  slot.map = *map;
  return LT_OK;
}

static int pow2_ceil(int v) { int p = 1; while (p < v) p <<= 1; return p; }

// pick the (bw, bh, bd, bn) power-of-two box with product 128 that wastes the fewest positions
static void pick_box(int OW, int OH, int OD, int N, int* box) {
  double best = 1e300;
  for (int bw = 1; bw <= 128; bw <<= 1)
    for (int bh = 1; bw * bh <= 128; bh <<= 1)
      for (int bd = 1; bw * bh * bd <= 128; bd <<= 1) {
        const int bn = 128 / (bw * bh * bd);
        if (bw > pow2_ceil(OW) || bh > pow2_ceil(OH) || bd > pow2_ceil(OD) || bn > pow2_ceil(N)) continue;
        const double padded = (double)ceil_div(OW, bw) * bw * ceil_div(OH, bh) * bh * (double)ceil_div(OD, bd) * bd * ceil_div(N, bn) * bn;
        const double score = padded * (1.0 + 1e-3 / bw);  // tie-break: wider rows
        if (score < best) { best = score; box[0] = bw; box[1] = bh; box[2] = bd; box[3] = bn; }
      }
  if (best == 1e300) { box[0] = pow2_ceil(OW) > 128 ? 128 : pow2_ceil(OW); box[1] = box[2] = 1; box[3] = 128 / box[0]; }
}

// Split-K second pass: sums the per-split accumulator tiles in a fixed order (deterministic) and applies the fused
// epilogue (scale/shift, residual, ReLU, output format).  One thread per (tile row, 4 channels).
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const TcParams p, long m_tiles, int coutp) {
  const int c4 = coutp >> 2;
  const long total = m_tiles * 128 * c4;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int co = (int)(i % c4) * 4;
    const long tr = i / c4;
    const int row = (int)(tr % 128);
    long t = tr / 128;
    const int twi = (int)(t % p.tw); t /= p.tw;
    const int thi = (int)(t % p.th); t /= p.th;
    const int tdi = (int)(t % p.td); t /= p.td;
    const int tni = (int)t;
    int r_ = row;
    const int dw = r_ % p.bw; r_ /= p.bw;
    const int dh = r_ % p.bh; r_ /= p.bh;
    const int dd = r_ % p.bd; r_ /= p.bd;
    const int ow = twi * p.bw + dw, oh = thi * p.bh + dh, od = tdi * p.bd + dd, nb = tni * p.bn + r_;
    if (!(ow < p.OW && oh < p.OH && od < p.OD && nb < p.N) || co >= p.FC) continue;
    const long opix = (((long)nb * p.FD + (od * p.osd + p.ood)) * p.FH + (oh * p.osh + p.ooh)) * p.FW + (ow * p.osw + p.oow);
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int z = 0; z < p.splits; ++z) {
      const float4 v = *reinterpret_cast<const float4*>(p.ws + ((size_t)z * m_tiles * 128 + tr) * p.ws_ld + co);
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
    a.x *= p.ws_gain; a.y *= p.ws_gain; a.z *= p.ws_gain; a.w *= p.ws_gain;
    const float4 sc = __ldg(reinterpret_cast<const float4*>(p.scale + co));
    const float4 sh = __ldg(reinterpret_cast<const float4*>(p.shift + co));
    float4 o = make_float4(fmaf(a.x, sc.x, sh.x), fmaf(a.y, sc.y, sh.y), fmaf(a.z, sc.z, sh.z), fmaf(a.w, sc.w, sh.w));
    float4 rr = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.residual != LT_RES_NONE) {
      if (p.out_format == LT_FMT_F32) rr = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.res) + opix * p.FC + co);
      else rr = load_s32x4(reinterpret_cast<const sh_t*>(p.res) + opix * 2 * p.FC, co);
    }
    if (p.residual == LT_RES_BEFORE_RELU) { o.x += rr.x; o.y += rr.y; o.z += rr.z; o.w += rr.w; }
    if (p.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
    if (p.residual == LT_RES_AFTER_RELU) { o.x += rr.x; o.y += rr.y; o.z += rr.z; o.w += rr.w; }
    if (p.out_format == LT_FMT_F32) *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + opix * p.FC + co) = o;
    else store_s32x4(reinterpret_cast<sh_t*>(p.out) + opix * 2 * p.FC, co, o);
  }
}

static int out_groups(const lt_conv_desc* d) {
  const int g = (d->ogd > 1 ? d->ogd : 1) * (d->ogh > 1 ? d->ogh : 1) * (d->ogw > 1 ? d->ogw : 1);
  return g;
}

// largest N tile of {128, 64, 32, 16} that divides the padded channel count (a multiple of 16)
static int pick_nt(int CoutP) {
  for (int nt = 128; nt > 16; nt >>= 1)
    if (CoutP % nt == 0) return nt;
  return 16;
}

template <int NT>
static int launch_nt(const CUtensorMap& tmA, const CUtensorMap& tmB, const TcEpiMaps& tmE, const TcParams& p, dim3 grid, size_t smem,
                     cudaStream_t st) {
  static DeviceOnce configured;
  if (configured.first()) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e != cudaSuccess) return fail(LT_ERR_CUDA, "conv_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  }
  conv_tc_kernel<NT><<<grid, kTcThreads, smem, st>>>(tmA, tmB, tmE, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(LT_ERR_CUDA, "conv_tc_kernel: %s", cudaGetErrorString(e));
  return LT_OK;
}

// Modelled time of one conv_tc launch (SM clocks) with the K loop split `splits` ways: every CTA of the persistent grid runs
// ceil(units / grid) work units, each its share of the K chunks plus one epilogue; a split adds the fp32 partial tiles, which
// splitk_reduce_kernel reads back.  Per K chunk the SM takes the larger of its MMA time (3 products: 12 m64 x Nt x k16 wgmma of
// 64 * Nt / 128 clocks) and its operand feed from L2 (16 KB of A and Nt * 128 bytes of B at ~30 B/clk per SM).  The epilogue
// moves 128 x Nt x 4 bytes from one SM at the same rate; the reduce pass streams its bytes over the whole GPU at ~1.5 KB/clk
// (2.5 TB/s at 1.7 GHz) after a ~7000-clock launch.  Only the ranking of split counts matters, not the absolute values.
static double tc_model_clocks(long tiles, int chunks, int nt, int splits, int sm) {
  const long units = tiles * splits;
  const long grid = units < sm ? units : sm;
  const long waves = (units + grid - 1) / grid;
  const double chunk = fmax(12.0 * 64.0 * nt / 128.0, (kATileBytes + nt * 128.0) / 30.0);
  const double epilogue = 128.0 * nt * 4.0 / 30.0;
  double t = (double)waves * ((double)ceil_div(chunks, splits) * chunk + epilogue);
  if (splits > 1) t += 7000.0 + (double)tiles * 128 * nt * 4.0 * (splits + 2) / 1500.0;
  return t;
}

// Work decomposition of one conv_tc launch: tiles, K split and persistent grid size (host only, no device access).  A split is
// taken when the model above says it is faster and its partial tiles fit the workspace; `terms` 0 (plain-fp16 self test) and
// grouped outputs never split.
static void tc_plan(long m_tiles, int n_tiles, int nt, int chunks, int terms, int n_maps, int splitk, size_t ws_bytes, int sm,
                    int* splits_out, int* grid_out) {
  const long tiles = m_tiles * n_tiles;
  int best = 1;
  if (splitk && terms != 0 && n_maps == 1) {
    const size_t per_split = (size_t)tiles * 128 * nt * sizeof(float);
    double best_t = tc_model_clocks(tiles, chunks, nt, 1, sm);
    for (int s = 2; s <= chunks / 4 && (size_t)s * per_split <= ws_bytes; ++s) {
      const double t = tc_model_clocks(tiles, chunks, nt, s, sm);
      if (t < best_t) { best_t = t; best = s; }
    }
  }
  const long units = tiles * best;
  *splits_out = best;
  *grid_out = (int)(units < sm ? units : sm);
}

// Positions of one output axis that group phase `ph` of a launch writes: those of its sub-lattice off + ph + o os (o < n) that
// lie inside the tensor's extent F, at most the launch's n.  A stride-2 data gradient of an odd-sized input has one position fewer
// in its odd phase than in its even one; every other launch writes exactly n.
static int group_extent(int n, int F, int off, int ph, int os) {
  const int e = (F - off - ph + os - 1) / os;
  return e < n ? e : n;
}

// Tensor maps of the staged epilogue.  Output position (ow, oh, od, nb) of group g is row ((nb FD + od osd + ood) FH + oh osh + ooh)
// FW + ow osw + oow of the channels-last tensor plus the group's phase offset, so every output is a plain map over the group's
// share of the launch's OW x OH x OD x N grid (group_extent): base at the (phase) origin, position strides scaled by osw / osh / osd,
// so the TMA store clips what falls outside the tensor.  Rows are FC x 4 bytes in both formats (the C ABI requires FC % 4 == 0,
// so they are 16-byte multiples).
static int make_epi_maps(const TcParams& p, TcEpiMaps* m) {
  const int f32 = p.out_format == LT_FMT_F32;
  const uint64_t rowb = (uint64_t)p.FC * 4;
  const uint64_t str[4] = {rowb * p.osw, rowb * p.FW * p.osh, rowb * p.FW * p.FH * p.osd, rowb * p.FW * p.FH * p.FD};
  const uint32_t bx[5] = {f32 ? 32u : 64u, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bd, (uint32_t)p.bn};
  for (int g = 0; g < p.n_maps; ++g) {
    const int ga = g / (p.gh * p.gw), gb = (g / p.gw) % p.gh, gc = g % p.gw;
    const int ew = group_extent(p.OW, p.FW, p.oow, gc, p.osw), eh = group_extent(p.OH, p.FH, p.ooh, gb, p.osh),
              ed = group_extent(p.OD, p.FD, p.ood, ga, p.osd);
    LT_REQUIRE(ew > 0 && eh > 0 && ed > 0, "conv_tc: output group %d lies outside the %dx%dx%d output tensor", g, p.FD, p.FH, p.FW);
    const uint64_t dims[5] = {(uint64_t)(f32 ? p.FC : 2 * p.FC), (uint64_t)ew, (uint64_t)eh, (uint64_t)ed, (uint64_t)p.N};
    const long pix0 = ((long)(p.ood + ga) * p.FH + p.ooh + gb) * p.FW + p.oow + gc;
    int rc = make_map(&m->out[g], static_cast<const uint8_t*>(p.out) + pix0 * rowb, 5, dims, str, bx, nullptr, 1, f32);
    if (rc) return rc;
    if (p.residual == LT_RES_NONE) continue;
    rc = make_map(&m->res[g], static_cast<const uint8_t*>(p.res) + pix0 * rowb, 5, dims, str, bx, nullptr, 1, f32);
    if (rc) return rc;
  }
  return LT_OK;
}

// one CTA per SM (the two consumer warpgroups hold up to 128 fp32 accumulators per thread): the shared memory beside the epilogue
// tile buffers is pipeline depth
constexpr int kTcSmemBudget = 224 * 1024;

// Shared-memory layout of one conv_tc launch (host only; launch_tc and lt_conv_tc_plan).  A second epilogue tile buffer lets the
// next unit's residual tile load while this unit's output tile waits for its epilogue and store, but it takes ring stages: at N
// tile 128 two 64 KB buffers leave 3 stages where one leaves 5.  Measured per layer class on an H100 80GB HBM3 (700 W), two
// buffers win on the backbone's 1x1 expansions with 2 and 4 K chunks per unit (96^2 64 -> 256: 1.40 -> 1.04 ms, 48^2 128 -> 512:
// 1.60 -> 1.39 ms per step) and lose from 8 chunks up, where the K loop needs the deeper ring (24^2 256 -> 1024, 8 chunks:
// 4.18 -> 4.76 ms; 3x3 256 -> 256, 72 chunks: 4.49 -> 5.15 ms).  So staged launches of at most kTcShortK chunks per unit take
// two buffers, longer ones one, and the ring gets the rest of the budget (N tile 128: 3 / 5 stages, 64: 6 / 8, 32: 8 / 8).
constexpr int kTcShortK = 4;
static void tc_layout(int nt, int splits, int chunks, int* stages, int* epi_buffers) {
  const int epi_bytes = tc_epi_bytes(nt, splits);
  *epi_buffers = epi_bytes == 0 ? 0 : (chunks <= kTcShortK ? 2 : 1);
  const int s = (kTcSmemBudget - *epi_buffers * epi_bytes) / (kATileBytes + nt * 128);
  *stages = s > 8 ? 8 : s;
}

static int launch_tc(const CUtensorMap& tmA, const CUtensorMap& tmB, TcParams& p, int n_tiles, cudaStream_t st, void* ws = nullptr,
                     size_t ws_bytes = 0) {
  const long m_tiles = (long)p.tw * p.th * p.td * p.tn;
  int splits, grid;
  tc_plan(m_tiles, n_tiles, p.Nt, p.KD * p.KH * p.KW * p.CB, p.terms, p.n_maps, ws ? opts().tc_splitk : 0, ws_bytes, sm_count(),
          &splits, &grid);
  p.splits = splits;
  // The folded scale compensates the truncation of all 2 x chunks k16 steps (engine.pack_filter); each split's partial accumulator
  // takes 1 / splits of them, so the reduce pass scales the sum back to that gain.
  const double steps = 2.0 * p.KD * p.KH * p.KW * p.CB;
  p.ws_gain = (float)(accum_gain(steps / splits) / accum_gain(steps));
  p.ws = reinterpret_cast<float*>(ws);
  p.ws_ld = n_tiles * p.Nt;
  p.n_tiles = n_tiles;
  const int stage_bytes = kATileBytes + p.Nt * 128;
  const int epi_bytes = tc_epi_bytes(p.Nt, splits);
  tc_layout(p.Nt, splits, p.KD * p.KH * p.KW * p.CB, &p.stages, &p.epi_buffers);
  const size_t smem = (size_t)p.stages * stage_bytes + (size_t)p.epi_buffers * epi_bytes + (2 * p.stages + 4) * 8 + 1024;
  TcEpiMaps tmE{};
  int rc;
  if (epi_bytes) {
    rc = make_epi_maps(p, &tmE);
    if (rc) return rc;
  }
  switch (p.Nt) {
    case 128: rc = launch_nt<128>(tmA, tmB, tmE, p, dim3(grid), smem, st); break;
    case 64: rc = launch_nt<64>(tmA, tmB, tmE, p, dim3(grid), smem, st); break;
    case 32: rc = launch_nt<32>(tmA, tmB, tmE, p, dim3(grid), smem, st); break;
    case 16: rc = launch_nt<16>(tmA, tmB, tmE, p, dim3(grid), smem, st); break;
    default: return fail(LT_ERR_INVALID, "conv_tc: unsupported N tile %d", p.Nt);
  }
  if (rc) return rc;
  if (splits > 1) {
    const long total = m_tiles * 128 * (p.ws_ld / 4);
    long blocks = (total + 255) / 256;
    if (blocks > 4L * sm_count()) blocks = 4L * sm_count();
    splitk_reduce_kernel<<<(unsigned)blocks, 256, 0, st>>>(p, m_tiles, p.ws_ld);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(LT_ERR_CUDA, "splitk_reduce_kernel: %s", cudaGetErrorString(e));
  }
  return LT_OK;
}

// fills the geometry / epilogue part of the launch parameters (M-tile box, taps, output mapping)
void fill_params(const lt_conv_desc* d, TcParams& p, int CB, int CoutP, int Nt, int terms, const float* scale, const float* shift,
                        const void* residual, void* out) {
  p.OW = d->OW; p.OH = d->OH; p.OD = d->OD; p.N = d->N;
  int box[4];
  pick_box(d->OW, d->OH, d->OD, d->N, box);
  p.bw = box[0]; p.bh = box[1]; p.bd = box[2]; p.bn = box[3];
  p.tw = ceil_div(d->OW, p.bw); p.th = ceil_div(d->OH, p.bh); p.td = ceil_div(d->OD, p.bd); p.tn = ceil_div(d->N, p.bn);
  p.KW = d->KW; p.KH = d->KH; p.KD = d->KD; p.pw = d->pw; p.ph = d->ph; p.pd = d->pd;
  p.sw = d->sw; p.sh = d->sh; p.sd = d->sd;
  p.CB = CB; p.b_step0 = 0; p.b_step1 = CoutP; p.b_nmul = 1; p.Nt = Nt; p.terms = terms;
  p.FC = d->FC; p.FD = d->FD; p.FH = d->FH; p.FW = d->FW;
  p.osd = d->osd; p.osh = d->osh; p.osw = d->osw; p.ood = d->ood; p.ooh = d->ooh; p.oow = d->oow;
  p.relu = d->relu; p.residual = d->residual; p.out_format = d->out_format;
  p.scale = scale; p.shift = shift; p.res = residual; p.out = out;
  p.splits = 1; p.ws = nullptr; p.ws_ld = 0; p.ws_gain = 1.0f; p.stages = 0; p.n_tiles = 1; p.epi_buffers = 0;
  p.n_maps = out_groups(d);
  p.oc = p.n_maps > 1 ? d->Cout / p.n_maps : CoutP;
  p.gh = d->ogh > 1 ? d->ogh : 1; p.gw = d->ogw > 1 ? d->ogw : 1;
}

int make_in_map(CUtensorMap* tmA, const lt_conv_desc* d, int bw, int bh, int bd, int bn, const void* in) {
  const uint64_t rowb = (uint64_t)d->Cin * 2 * 2;  // 2*Cin fp16 per position
  const uint64_t dims[5] = {(uint64_t)d->Cin * 2, (uint64_t)d->IW, (uint64_t)d->IH, (uint64_t)d->ID, (uint64_t)d->N};
  const uint64_t str[4] = {rowb, rowb * d->IW, rowb * d->IW * d->IH, rowb * d->IW * d->IH * d->ID};
  // strided convs: TMA traversal strides; the box spans (b-1)*s+1 input positions and delivers b of them
  const uint32_t es[5] = {1, (uint32_t)d->sw, (uint32_t)d->sh, (uint32_t)d->sd, 1};
  uint32_t bx[5] = {64, (uint32_t)bw, (uint32_t)bh, (uint32_t)bd, (uint32_t)bn};
  for (int i = 1; i <= 3; ++i) bx[i] = (bx[i] - 1) * es[i] + 1;
  LT_REQUIRE(bx[1] <= 256 && bx[2] <= 256 && bx[3] <= 256, "conv_tc: strided box exceeds 256");
  return make_map(tmA, in, 5, dims, str, bx, es, 1);
}

// grouped output (k2 s2 transposed conv, stride-2 data gradient: one GEMM, one output phase per channel block): every channel of the
// GEMM belongs to exactly one group, and a group fills the output's channels exactly.  Split-fp16 or float32: the staged epilogue
// stores whole 32-channel slabs of either format.
static bool groups_ok(const lt_conv_desc* d, int CoutP) {
  const int G = out_groups(d);
  return d->Cout % G == 0 && (d->Cout / G) % 32 == 0 && d->Cout / G == d->FC && CoutP == d->Cout && G <= kMaxOutMaps;
}

// LT_CONV_TC (terms = 3) and LT_CONV_TC1 (terms = 1): weights packed as [tap][Cin/32][CoutP rows][32 hi | 32 lo] fp16,
// CoutP = round_up(Cout, 16) (lt_conv_tc_pack_weights).
int conv_tc_fwd_terms(const lt_conv_desc* d, const void* in, const void* weight, const float* scale, const float* shift,
                      const void* residual, void* out, int terms, void* stream) {
  LT_REQUIRE(d->in_format == LT_FMT_S32, "conv_tc: input must be split-fp16");
  LT_REQUIRE(d->Cin % 32 == 0, "conv_tc: Cin=%d must be a multiple of 32", d->Cin);
  LT_REQUIRE(d->FC % 4 == 0 && (d->out_format == LT_FMT_F32 || d->FC % 32 == 0), "conv_tc: bad output channel stride %d", d->FC);
  LT_REQUIRE((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(residual)) % 16 == 0,
             "conv_tc: out and residual must be 16-byte aligned (TMA global addresses)");
  const int CoutP = (d->Cout + 15) & ~15;
  const int CB = d->Cin / 32;
  const int taps = d->KD * d->KH * d->KW;
  const int Nt = pick_nt(CoutP);
  TcParams p;
  fill_params(d, p, CB, CoutP, Nt, terms, scale, shift, residual, out);
  if (p.n_maps > 1)
    LT_REQUIRE(groups_ok(d, CoutP), "conv_tc: grouped output needs Cout / groups == FC, a multiple of 32");
  CUtensorMap tmA, tmB;
  int rc = make_in_map(&tmA, d, p.bw, p.bh, p.bd, p.bn, in);
  if (rc) return rc;
  {
    const uint64_t dims[2] = {64, (uint64_t)taps * CB * CoutP};
    const uint64_t str[1] = {128};
    const uint32_t bx[2] = {64, (uint32_t)Nt};
    rc = make_map(&tmB, weight, 2, dims, str, bx, nullptr, 1);
    if (rc) return rc;
  }
  return launch_tc(tmA, tmB, p, CoutP / Nt, (cudaStream_t)stream, d->workspace, d->workspace_bytes);
}

// ---- chain mode (lt_conv_tc_chain_fwd) ----
// Geometry of a chain of `blocks` bottleneck blocks whose three launches `d` describes (host only): what the kernel and the
// planner need to number the units and find their dependencies.
static int chain_geom(const lt_conv_desc* d, int blocks, TcChainGeom* g) {
  LT_REQUIRE(d && g, "conv_tc_chain: null pointer");
  LT_REQUIRE(blocks >= 1 && blocks <= kChainMaxBlocks, "conv_tc_chain: %d blocks, 1 to %d per launch", blocks, kChainMaxBlocks);
  for (int c = 0; c < 3; ++c) {
    const lt_conv_desc& e = d[c];
    LT_REQUIRE(e.in_format == LT_FMT_S32 && e.out_format == LT_FMT_S32, "conv_tc_chain: layer %d must be split-fp16 in and out", c);
    LT_REQUIRE(e.N == d[0].N && e.OD == d[0].OD && e.OH == d[0].OH && e.OW == d[0].OW && e.ID == e.OD && e.IH == e.OH && e.IW == e.OW &&
                   e.FD == e.OD && e.FH == e.OH && e.FW == e.OW && e.N > 0 && e.OD > 0 && e.OH > 0 && e.OW > 0,
               "conv_tc_chain: layer %d must map the chain's output grid onto itself", c);
    LT_REQUIRE(e.sd == 1 && e.sh == 1 && e.sw == 1 && e.osd == 1 && e.osh == 1 && e.osw == 1 && e.ood == 0 && e.ooh == 0 && e.oow == 0 &&
                   out_groups(&e) == 1,
               "conv_tc_chain: layer %d must be a stride-1 conv with a plain output", c);
    LT_REQUIRE(e.KD > 0 && e.KH > 0 && e.KW > 0 && 2 * e.pd == e.KD - 1 && 2 * e.ph == e.KH - 1 && 2 * e.pw == e.KW - 1,
               "conv_tc_chain: layer %d must pad to its own output size", c);
    LT_REQUIRE(e.Cin % 32 == 0 && e.Cout % 128 == 0 && e.FC == e.Cout && e.Cin == d[(c + 2) % 3].Cout,
               "conv_tc_chain: layer %d channels %d -> %d (FC %d) do not chain at N tile 128", c, e.Cin, e.Cout, e.FC);
    LT_REQUIRE(c == 2 ? (e.residual == LT_RES_BEFORE_RELU || e.residual == LT_RES_AFTER_RELU) : e.residual == LT_RES_NONE,
               "conv_tc_chain: only the expansion (layer 2) adds the residual");
  }
  int box[4];
  pick_box(d[0].OW, d[0].OH, d[0].OD, d[0].N, box);
  g->blocks = blocks;
  g->bw = box[0]; g->bh = box[1]; g->bd = box[2]; g->bn = box[3];
  g->OW = d[0].OW; g->OH = d[0].OH; g->OD = d[0].OD;
  g->tw = ceil_div(g->OW, g->bw); g->th = ceil_div(g->OH, g->bh); g->td = ceil_div(g->OD, g->bd); g->tn = ceil_div(d[0].N, g->bn);
  g->m_tiles = g->tw * g->th * g->td * g->tn;
  g->units_per_block = 0;
  for (int c = 0; c < 3; ++c) {
    const lt_conv_desc& e = d[c];
    g->n_tiles[c] = e.Cout / 128;
    g->CB[c] = e.Cin / 32;
    g->KW[c] = e.KW; g->KH[c] = e.KH; g->KD[c] = e.KD;
    g->pw[c] = e.pw; g->ph[c] = e.ph; g->pd[c] = e.pd;
    g->chunks[c] = e.KD * e.KH * e.KW * g->CB[c];
    g->CoutP[c] = e.Cout;
    g->FC[c] = e.FC;
    g->residual[c] = e.residual;
    g->relu[c] = e.relu;
    g->units_per_block += g->m_tiles * g->n_tiles[c];
  }
  LT_REQUIRE((long)g->units_per_block * blocks < (1L << 30), "conv_tc_chain: too many work units");
  return LT_OK;
}

// one launch's parameters: the chain's kernel parameter block, beside TcParams, must stay within the 32764 bytes a launch takes
static_assert(sizeof(TcChain) + sizeof(TcParams) + 64 <= 32764, "conv_tc_chain_kernel parameters exceed the launch limit");

static int launch_chain(const lt_conv_desc* d, int blocks, void* x, void* const* bufs, const void* const* weights,
                        const float* const* scales, const float* const* shifts, void* counters, size_t counters_bytes, int terms,
                        cudaStream_t st) {
  static thread_local TcChain ch;   // ~17 KB: kept off the stack
  memset(&ch, 0, sizeof(ch));
  int rc = chain_geom(d, blocks, &ch.g);
  if (rc) return rc;
  const TcChainGeom& g = ch.g;
  LT_REQUIRE(x && bufs && weights && scales && shifts && counters, "conv_tc_chain: null pointer");
  const size_t ncount = 1 + (size_t)3 * blocks * g.m_tiles;
  LT_REQUIRE(counters_bytes >= ncount * sizeof(unsigned), "conv_tc_chain: counters need %zu bytes", ncount * sizeof(unsigned));
  void* in_of[3][2] = {{x, x}, {bufs[0], bufs[1]}, {bufs[2], bufs[3]}};
  void* out_of[3][2] = {{bufs[0], bufs[1]}, {bufs[2], bufs[3]}, {x, x}};
  for (int i = 0; i < 4; ++i) LT_REQUIRE(bufs[i] && reinterpret_cast<uintptr_t>(bufs[i]) % 16 == 0, "conv_tc_chain: buffer %d", i);
  LT_REQUIRE(reinterpret_cast<uintptr_t>(x) % 16 == 0, "conv_tc_chain: x must be 16-byte aligned (TMA global addresses)");
  TcParams p;
  fill_params(&d[0], p, g.CB[0], g.CoutP[0], 128, terms, nullptr, nullptr, nullptr, x);
  tc_layout(128, 1, kTcShortK + 1, &p.stages, &p.epi_buffers);   // one tile buffer, the deep ring: every chained layer has > 4 chunks
  for (int c = 0; c < 3; ++c) {
    for (int q = 0; q < 2; ++q) {
      rc = make_in_map(&ch.a[c][q], &d[c], p.bw, p.bh, p.bd, p.bn, in_of[c][q]);
      if (rc) return rc;
      TcParams lp;
      fill_params(&d[c], lp, g.CB[c], g.CoutP[c], 128, terms, nullptr, nullptr, c == 2 ? x : nullptr, out_of[c][q]);
      TcEpiMaps em;
      rc = make_epi_maps(lp, &em);
      if (rc) return rc;
      ch.out[c][q] = em.out[0];
      if (c == 2) ch.res = em.res[0];
    }
  }
  for (int k = 0; k < blocks; ++k)
    for (int c = 0; c < 3; ++c) {
      const int l = 3 * k + c;
      LT_REQUIRE(weights[l] && scales[l] && shifts[l], "conv_tc_chain: null filter, scale or shift of layer %d", l);
      const uint64_t dims[2] = {64, (uint64_t)g.chunks[c] * g.CoutP[c]};
      const uint64_t str[1] = {128};
      const uint32_t bx[2] = {64, 128};
      rc = make_map(&ch.b[k][c], weights[l], 2, dims, str, bx, nullptr, 1);
      if (rc) return rc;
      ch.scale[k][c] = scales[l];
      ch.shift[k][c] = shifts[l];
    }
  ch.counters = static_cast<unsigned*>(counters);
  cudaError_t e = cudaMemsetAsync(counters, 0, ncount * sizeof(unsigned), st);
  if (e != cudaSuccess) return fail(LT_ERR_CUDA, "conv_tc_chain: cudaMemsetAsync: %s", cudaGetErrorString(e));
  const long units = (long)g.units_per_block * blocks;
  const int grid = (int)(units < sm_count() ? units : sm_count());
  const size_t smem = (size_t)p.stages * (kATileBytes + 128 * 128) + (size_t)p.epi_buffers * tc_epi_bytes(128, 1) + (2 * p.stages + 4) * 8 +
                      kChainRing * (2 * 8 + 4) + 1024;
  static DeviceOnce configured;
  if (configured.first()) {
    e = cudaFuncSetAttribute(conv_tc_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e != cudaSuccess) return fail(LT_ERR_CUDA, "conv_tc_chain: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  }
  conv_tc_chain_kernel<<<grid, kTcThreads, smem, st>>>(ch, p);
  e = cudaGetLastError();
  if (e != cudaSuccess) return fail(LT_ERR_CUDA, "conv_tc_chain_kernel: %s", cudaGetErrorString(e));
  return LT_OK;
}

// ---- weight packing: fp32 [taps][Cin][Cout] -> fp16 [taps][Cin/32][CoutP][32 hi | 32 lo] (128-byte rows) ----------
__global__ void __launch_bounds__(256) pack_weights_kernel(const float* __restrict__ w, sh_t* __restrict__ out,
                                                           int taps, int Cin, int Cout, int CoutP) {
  const int CB = Cin / 32;
  const long total = (long)taps * CB * CoutP * 32;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int j = (int)(i % 32);
    long r = i / 32;
    const int n = (int)(r % CoutP); r /= CoutP;
    const int cb = (int)(r % CB);
    const int tap = (int)(r / CB);
    const float v = (n < Cout) ? w[((long)tap * Cin + cb * 32 + j) * Cout + n] : 0.0f;
    sh_t hi, lo;
    split_s32(v, hi, lo);
    sh_t* rowp = out + ((((long)tap * CB + cb) * CoutP + n) << 6);
    rowp[j] = hi;
    rowp[32 + j] = lo;
  }
}

__global__ void ones_zeros_kernel(float* ones, float* zeros, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { ones[i] = 1.0f; zeros[i] = 0.0f; }
}

}  // namespace lt

using namespace lt;

extern "C" int lt_conv_tc_plan(const lt_conv_desc* d, int sm_count, int splitk, lt_conv_tc_launch_plan* plan) {
  LT_REQUIRE(d && plan && sm_count > 0, "conv_tc_plan: bad arguments");
  LT_REQUIRE(d->Cin % 32 == 0 && d->Cout > 0, "conv_tc_plan: Cin=%d must be a multiple of 32", d->Cin);
  const int CoutP = (d->Cout + 15) & ~15;
  int box[4];
  pick_box(d->OW, d->OH, d->OD, d->N, box);
  plan->nt = pick_nt(CoutP);
  plan->m_tiles = ceil_div(d->OW, box[0]) * ceil_div(d->OH, box[1]) * ceil_div(d->OD, box[2]) * ceil_div(d->N, box[3]);
  plan->n_tiles = CoutP / plan->nt;
  plan->chunks = d->KD * d->KH * d->KW * (d->Cin / 32);
  tc_plan(plan->m_tiles, plan->n_tiles, plan->nt, plan->chunks, 3, out_groups(d), d->workspace ? splitk : 0, d->workspace_bytes,
          sm_count, &plan->splits, &plan->grid);
  tc_layout(plan->nt, plan->splits, plan->chunks, &plan->stages, &plan->epi_buffers);
  return LT_OK;
}

extern "C" int lt_conv_tc_chain_plan(const lt_conv_desc* descs, int blocks, int sm_count, lt_conv_tc_chain_launch_plan* plan) {
  LT_REQUIRE(plan && sm_count > 0, "conv_tc_chain_plan: bad arguments");
  TcChainGeom g;
  const int rc = chain_geom(descs, blocks, &g);
  if (rc) return rc;
  plan->m_tiles = g.m_tiles;
  for (int c = 0; c < 3; ++c) plan->n_tiles[c] = g.n_tiles[c];
  plan->units = g.units_per_block * blocks;
  plan->grid = plan->units < sm_count ? plan->units : sm_count;
  plan->counters = 1 + 3 * blocks * g.m_tiles;
  return LT_OK;
}

extern "C" int lt_conv_tc_chain_deps(const lt_conv_desc* descs, int blocks, int unit, lt_conv_tc_chain_unit* info, int* tiles, int cap) {
  LT_REQUIRE(info && (tiles || cap == 0), "conv_tc_chain_deps: bad arguments");
  TcChainGeom g;
  const int rc = chain_geom(descs, blocks, &g);
  if (rc) return rc;
  LT_REQUIRE(unit >= 0 && unit < g.units_per_block * blocks, "conv_tc_chain_deps: unit %d out of range", unit);
  int k, c, m, n, src, need, lo[4], hi[4];
  chain_unit(g, unit, k, c, m, n);
  info->layer = 3 * k + c;
  info->m_tile = m;
  info->n_tile = n;
  info->src_layer = -1;
  info->need = 0;
  info->n_deps = 0;
  if (!chain_deps(g, k, c, m, src, need, lo, hi)) return LT_OK;
  info->src_layer = src;
  info->need = need;
  for (int tn = lo[3]; tn <= hi[3]; ++tn)
    for (int td = lo[2]; td <= hi[2]; ++td)
      for (int th = lo[1]; th <= hi[1]; ++th)
        for (int tw = lo[0]; tw <= hi[0]; ++tw) {
          LT_REQUIRE(info->n_deps < cap, "conv_tc_chain_deps: more than %d tiles", cap);
          tiles[info->n_deps++] = ((tn * g.td + td) * g.th + th) * g.tw + tw;
        }
  return LT_OK;
}

extern "C" int lt_conv_tc_chain_fwd(const lt_conv_desc* descs, int blocks, void* x, void* const* bufs, const void* const* weights,
                                    const float* const* scales, const float* const* shifts, void* counters, size_t counters_bytes, int impl,
                                    void* stream) {
  LT_REQUIRE(impl == LT_CONV_TC || impl == LT_CONV_TC1, "conv_tc_chain: impl %d is not a tensor-core conv", impl);
  return launch_chain(descs, blocks, x, bufs, weights, scales, shifts, counters, counters_bytes, impl == LT_CONV_TC ? 3 : 1,
                      (cudaStream_t)stream);
}

extern "C" size_t lt_conv_tc_weight_bytes(int taps, int Cin, int Cout) {
  const int CoutP = (Cout + 15) & ~15;
  return (size_t)taps * (Cin / 32) * CoutP * 128;
}

extern "C" int lt_conv_tc_pack_weights(const float* w, void* packed, int taps, int Cin, int Cout, void* stream) {
  LT_REQUIRE(w && packed, "conv_tc_pack_weights: null pointer");
  LT_REQUIRE(Cin % 32 == 0 && taps > 0 && Cout > 0, "conv_tc_pack_weights: bad sizes");
  const int CoutP = (Cout + 15) & ~15;
  const long total = (long)taps * (Cin / 32) * CoutP * 32;
  long blocks = (total + 255) / 256;
  if (blocks > 65535) blocks = 65535;
  pack_weights_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(w, reinterpret_cast<sh_t*>(packed), taps, Cin, Cout, CoutP);
  LT_CHECK_LAUNCH("pack_weights_kernel");
  return LT_OK;
}

// D[M][N] (fp32) = A[M][K] * B[N][K]^T, plain fp16 row-major operands; exercises the exact TMA /
// descriptor / wgmma / epilogue code of the conv kernel (terms = 0 selects plain rows).
// `d` must hold M*N floats followed by 2*N floats of scratch (scale/shift).
extern "C" int lt_tc_gemm_selftest(const void* a, const void* b, float* d, int M, int N, int K, int variant, void* stream) {
  LT_REQUIRE(a && b && d, "tc_gemm_selftest: null pointer");
  LT_REQUIRE(M > 0 && N % 16 == 0 && N >= 16 && K % 64 == 0, "tc_gemm_selftest: need N %% 16 == 0, K %% 64 == 0");
  (void)variant;
  const int Nt = pick_nt(N);
  float* ones = d + (size_t)M * N;
  float* zeros = ones + N;
  ones_zeros_kernel<<<ceil_div(N, 256), 256, 0, (cudaStream_t)stream>>>(ones, zeros, N);
  TcParams p;
  p.OW = M; p.OH = 1; p.OD = 1; p.N = 1;
  p.bw = 128; p.bh = 1; p.bd = 1; p.bn = 1;
  p.tw = ceil_div(M, 128); p.th = 1; p.td = 1; p.tn = 1;
  p.KW = p.KH = p.KD = 1; p.pw = p.ph = p.pd = 0; p.sw = p.sh = p.sd = 1;
  p.CB = K / 64; p.b_step0 = 64; p.b_step1 = 0; p.b_nmul = 1; p.Nt = Nt; p.terms = 0;
  p.FC = N; p.FD = 1; p.FH = 1; p.FW = M; p.osd = p.osh = p.osw = 1; p.ood = p.ooh = p.oow = 0;
  p.relu = 0; p.residual = LT_RES_NONE; p.out_format = LT_FMT_F32;
  p.scale = ones; p.shift = zeros; p.res = nullptr; p.out = d;
  p.n_maps = 1; p.oc = N; p.gh = p.gw = 1;
  p.splits = 1; p.ws = nullptr; p.ws_ld = 0; p.ws_gain = 1.0f; p.n_tiles = 1; p.epi_buffers = 0;
  CUtensorMap tmA, tmB;
  {
    const uint64_t dims[5] = {(uint64_t)K, (uint64_t)M, 1, 1, 1};
    const uint64_t str[4] = {(uint64_t)K * 2, (uint64_t)K * 2 * M, (uint64_t)K * 2 * M, (uint64_t)K * 2 * M};
    const uint32_t bx[5] = {64, 128, 1, 1, 1};
    int rc = make_map(&tmA, a, 5, dims, str, bx, nullptr, 1);
    if (rc) return rc;
  }
  {
    const uint64_t dims[2] = {(uint64_t)K, (uint64_t)N};
    const uint64_t str[1] = {(uint64_t)K * 2};
    const uint32_t bx[2] = {64, (uint32_t)Nt};
    int rc = make_map(&tmB, b, 2, dims, str, bx, nullptr, 1);
    if (rc) return rc;
  }
  return launch_tc(tmA, tmB, p, N / Nt, (cudaStream_t)stream);
}
