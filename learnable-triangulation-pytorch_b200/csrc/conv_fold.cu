// Halo-reusing wgmma convolution for the full-resolution V2V layers (LT_CONV_TC_FOLD): Cin = 32, cubic K = 3 or 7, stride 1,
// "same" padding, Cout <= 32.  Same arithmetic and epilogue as conv_tc_kernel (conv_tc.cu), different operand staging.
//
// The generic kernel loads one 128-position A tile per filter tap, so every input row is fetched K^3 times and each byte brought
// into the SM feeds only ~39 FLOP at these narrow N.  Here the output tile is 8 (w) x BH (h) x BD (d) positions whose 64-row m64
// blocks are whole 8-wide W lines at 8 consecutive h of one d plane, and an A pipeline stage holds ONE input halo box
//   {64 channels, 8 + K - 1 (w), BH + K - 1 (h), BD + KDS - 1 (d)}   at input offset (-K/2, -K/2, kd0 - K/2)
// that serves every kw, every kh and KDS consecutive kd.  TMA zero fill supplies the padding.
//
// The A operand comes from registers (wgmma RS): each warp owns 16 rows of an m64 block, i.e. the W lines 2 w' and 2 w' + 1 of
// the block (w' = warp in the warpgroup), and loads them with ldmatrix from the 128B-swizzled box (chunk j of box row R sits at
// j ^ (R % 8), the box starting on a 1024-byte boundary).  A tap may therefore start at any box row: the kw shift is a one-row
// offset.  Eight consecutive rows of a line hit eight distinct 16-byte chunks, so the loads are conflict-free.  Along kh the
// fragments of the second line are the first line of the next tap, so each kh step loads one new line per warp.
//
//   K = 3: tile 8 x 8 x 2 (box 10 x 10 x 4, one A stage per tile); the whole packed filter (27 taps) stays resident in shared
//          memory, loaded once per CTA, and each consumer warpgroup owns whole tiles (alternating), so one warpgroup's epilogue
//          overlaps the other's MMAs.  Products in (kw, kd, kh) order, as in the previous staging: results are unchanged.
//   K = 7: tile 8 x 16 x 2 (box 14 x 22 x 2, one A stage per kd), both consumer warpgroups on the same tile (two m64 blocks
//          each); the filter streams through its own ring, one slice per (kd, kw) = the 7 kh taps.  Products in (kd, kw, kh) order.
//
// Weights: lt_conv_fold_pack_weights, [kw][kd][kh][NC rows][32 hi | 32 lo] fp16, NC = round_up(Cout, 16); a (kw, kd) slice is
// K consecutive taps.  The N tile is NC: the 7^3 layer (Cout 16) multiplies no padding; output channels NC .. FC-1 go through the
// same epilogue with zero accumulators (scale 0, shift 0 for the padding channels: written as zeros).
//
// Per 16-wide K slice hi*hi accumulates into D1 and hi*lo + lo*hi into D2, as in conv_tc_kernel: D1 takes K^3 x Cin / 16
// accumulation steps per output (the accum_steps of the folded scale, engine._pack).
//
// Persistent grid: one CTA per SM strides over the tiles; the producer warp runs its rings across tile boundaries, so the next
// tile's boxes load while the consumers run the epilogue of the previous one.  An A stage is released as soon as the consumers'
// ldmatrix reads of it have completed; a weight slice once the MMAs reading it have.
#include "tc_common.cuh"
#include "conv_tc_params.cuh"

namespace lt {

constexpr int kFoldThreads = 384;
constexpr int kFoldSmem = 227 * 1024;

template <int K>
struct FoldTile;
template <>
struct FoldTile<3> { static constexpr int BH = 8, BD = 2, KDS = 3; static constexpr bool RES = true; };
template <>
struct FoldTile<7> { static constexpr int BH = 16, BD = 2, KDS = 1; static constexpr bool RES = false; };

template <int K, int NC>
struct FoldCfg {
  static constexpr int BW = 8, BH = FoldTile<K>::BH, BD = FoldTile<K>::BD, KDS = FoldTile<K>::KDS;
  // RES: filter resident, each consumer warpgroup owns whole tiles; else both warpgroups share a tile, weights ringed
  static constexpr bool RES = FoldTile<K>::RES;
  static constexpr int WBOX = BW + K - 1, HBOX = BH + K - 1, DBOX = BD + KDS - 1;
  static constexpr int A_BYTES = WBOX * HBOX * DBOX * 128;
  static constexpr int ASTAGES = K / KDS;             // A boxes per tile
  static constexpr int TAP = NC * 128;                 // one packed weight tap
  static constexpr int B_SLICE = RES ? K * K * K * TAP : KDS * K * TAP;
  static constexpr int BLOCKS = BH * BD / 8;           // m64 blocks per tile
  static constexpr int MB = RES ? BLOCKS : BLOCKS / 2; // m64 blocks per consumer warpgroup
  static constexpr int AVAIL = kFoldSmem - 1024 - 256;
  static constexpr int ARING_FIT = RES ? (AVAIL - B_SLICE) / A_BYTES : 2;
  static constexpr int ARING = ARING_FIT > 4 ? 4 : ARING_FIT;
  static constexpr int BRING_FIT = RES ? 1 : (AVAIL - ARING * A_BYTES) / B_SLICE;
  static constexpr int BRING = BRING_FIT > 4 ? 4 : BRING_FIT;
  static constexpr int A_OFF = BRING * B_SLICE;
  static constexpr int BAR_OFF = A_OFF + ARING * A_BYTES;
  static constexpr size_t SMEM = (size_t)BAR_OFF + 256 + 1024;
  static_assert(BW * BH * BD == (RES ? 128 : 256) && BH % 8 == 0 && MB == 2, "two m64 blocks of whole 8-wide lines per warpgroup");
  static_assert(A_BYTES % 1024 == 0 && B_SLICE % 1024 == 0, "boxes must start on 1024-byte swizzle atoms");
  static_assert(ARING >= 2 && BRING >= (RES ? 1 : 2) && 2 * (ARING + BRING) * 8 <= 256 && SMEM <= (size_t)kFoldSmem, "shared memory");
};

__device__ __forceinline__ void fold_tile_origin(const TcParams& p, int t, int& ow0, int& oh0, int& od0, int& nb) {
  ow0 = (t % p.tw) * p.bw; t /= p.tw;
  oh0 = (t % p.th) * p.bh; t /= p.th;
  od0 = (t % p.td) * p.bd;
  nb = t / p.td;
}

// One 8-row W line of the box, all 64 fp16 of each row: f[q][m] = 8x8 matrix of 16-byte chunk 4 q + m.  `row` is this lane's box
// row (the line's first row + lane % 8); lanes 8 m .. 8 m + 7 address chunk 4 q + m.
__device__ __forceinline__ void fold_load_line(uint32_t (&f)[2][4], uint32_t box, uint32_t row, uint32_t m) {
  const uint32_t a = box + row * 128u, sw = row & 7u;
  ldmatrix_x4(f[0], a + ((m ^ sw) << 4));
  ldmatrix_x4(f[1], a + (((m + 4u) ^ sw) << 4));
}

// The six products of one tap for one m64 block: rows 0-7 of each warp's 16 from line l0, rows 8-15 from line l1.
template <int NC>
__device__ __forceinline__ void fold_tap(float (&d1)[NC / 2], float (&d2)[NC / 2], const uint32_t (&l0)[2][4],
                                         const uint32_t (&l1)[2][4], uint64_t bd, uint32_t acc) {
  uint32_t a[4][4];   // K slice s = chunks 2 s, 2 s + 1 (s = 0, 1: hi; 2, 3: lo)
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    const int q = s >> 1, c = 2 * (s & 1);
    a[s][0] = l0[q][c]; a[s][1] = l1[q][c]; a[s][2] = l0[q][c + 1]; a[s][3] = l1[q][c + 1];
  }
  wgmma_f16_rs<NC>(d1, a[0], bd, acc);        // hi * hi
  wgmma_f16_rs<NC>(d1, a[1], bd + 2, 1u);
  wgmma_f16_rs<NC>(d2, a[0], bd + 4, acc);    // hi * lo
  wgmma_f16_rs<NC>(d2, a[1], bd + 6, 1u);
  wgmma_f16_rs<NC>(d2, a[2], bd, 1u);         // lo * hi
  wgmma_f16_rs<NC>(d2, a[3], bd + 2, 1u);
}

template <int K, int NC>
__global__ void __launch_bounds__(kFoldThreads, 1) conv_fold_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                    const __grid_constant__ CUtensorMap tmB, const TcParams p) {
  using C = FoldCfg<K, NC>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* bsm = smem;
  uint8_t* asm_ = smem + C::A_OFF;
  uint64_t* afull = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);
  uint64_t* aempty = afull + C::ARING;
  uint64_t* bfull = aempty + C::ARING;
  uint64_t* bempty = bfull + C::BRING;

  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int lane = threadIdx.x & 31;
  const int ntiles = p.tw * p.th * p.td * p.tn;

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::ARING; ++s) { mbar_init(&afull[s], 1); mbar_init(&aempty[s], C::RES ? 128 : 256); }
    for (int s = 0; s < C::BRING; ++s) { mbar_init(&bfull[s], 1); mbar_init(&bempty[s], 2); }
    fence_barrier_init();
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
  }
  __syncthreads();

  if (wg == 0) {
    // ================= TMA producer (warp 0; one elected lane issues) =================
    regs_release_producer();
    if (threadIdx.x < 32) {
      if (C::RES && elect_one()) {
        mbar_expect_tx(&bfull[0], (uint32_t)C::B_SLICE);
        tma_load_3d(bsm, &tmB, &bfull[0], 0, 0, 0);
      }
      int sa = 0, sb = 0;
      uint32_t pa = 0, pb = 0;
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        int ow0, oh0, od0, nb;
        fold_tile_origin(p, t, ow0, oh0, od0, nb);
        for (int as = 0; as < C::ASTAGES; ++as) {
          mbar_wait(&aempty[sa], pa ^ 1u);
          if (elect_one()) {
            mbar_expect_tx(&afull[sa], (uint32_t)C::A_BYTES);
            tma_load_5d(asm_ + (size_t)sa * C::A_BYTES, &tmA, &afull[sa], 0, ow0 - K / 2, oh0 - K / 2, od0 + as * C::KDS - K / 2, nb);
          }
          __syncwarp();
          if (++sa == C::ARING) { sa = 0; pa ^= 1u; }
          if constexpr (!C::RES) {
            for (int kw = 0; kw < K; ++kw) {
              mbar_wait(&bempty[sb], pb ^ 1u);
              if (elect_one()) {
                mbar_expect_tx(&bfull[sb], (uint32_t)C::B_SLICE);
                tma_load_3d(bsm + (size_t)sb * C::B_SLICE, &tmB, &bfull[sb], 0, 0, (kw * K + as * C::KDS) * K);
              }
              __syncwarp();
              if (++sb == C::BRING) { sb = 0; pb ^= 1u; }
            }
          }
        }
      }
    }
    return;
  }

  // ================= MMA + epilogue (warpgroups 1, 2) =================
  regs_claim_consumer();
  const int g = wg - 1, warp = (threadIdx.x >> 5) & 3;
  float d1[C::MB][NC / 2], d2[C::MB][NC / 2];
#pragma unroll
  for (int b = 0; b < C::MB; ++b)
#pragma unroll
    for (int i = 0; i < NC / 2; ++i) { d1[b][i] = 0.f; d2[b][i] = 0.f; }
  // m64 block b of this warpgroup: d plane dd and 8-line h block hb of the tile; this lane's box row for kw = kh = kdl = 0
  int blk_dd[C::MB], blk_hb[C::MB];
  uint32_t row0[C::MB];
#pragma unroll
  for (int b = 0; b < C::MB; ++b) {
    const int blk = C::RES ? b : C::MB * g + b;
    blk_dd[b] = blk / (C::BH / 8);
    blk_hb[b] = blk % (C::BH / 8);
    row0[b] = (uint32_t)((blk_dd[b] * C::HBOX + blk_hb[b] * 8 + 2 * warp) * C::WBOX + (lane & 7));
  }
  const uint32_t mlane = (uint32_t)(lane >> 3);
  const int r_lo = warp * 16 + (lane >> 2);   // this thread's accumulator rows r_lo, r_lo + 8 of an m64 block
  const int c2 = 2 * (lane & 3);
  const uint32_t bsm0 = smem_u32(bsm), asm0 = smem_u32(asm_);
  const bool wg_lead = (threadIdx.x & 127) == 0;
  if (C::RES) mbar_wait(&bfull[0], 0);
  // CTA-local tile kt: tile blockIdx.x + kt gridDim.x; with RES warpgroup g takes kt = g, g + 2, ...
  const int kt0 = C::RES ? g : 0, kstep = C::RES ? 2 : 1;
  int bprev = -1;
  for (int kt = kt0;; kt += kstep) {
    const int t = blockIdx.x + kt * gridDim.x;
    if (t >= ntiles) break;
#pragma unroll 1
    for (int as = 0; as < C::ASTAGES; ++as) {
      const int na = kt * C::ASTAGES + as;
      const int sa = na % C::ARING;
      mbar_wait(&afull[sa], (uint32_t)(na / C::ARING) & 1u);
      const uint32_t box = asm0 + (uint32_t)(sa * C::A_BYTES);
#pragma unroll 1
      for (int kw = 0; kw < K; ++kw) {
        const int nbs = na * K + kw;
        const int sb = C::RES ? 0 : nbs % C::BRING;
        if (!C::RES) mbar_wait(&bfull[sb], (uint32_t)(nbs / C::BRING) & 1u);
        const uint32_t bslice = bsm0 + (uint32_t)(sb * C::B_SLICE);
#pragma unroll
        for (int kdl = 0; kdl < C::KDS; ++kdl) {
          const int kd = as * C::KDS + kdl;
          const uint32_t roff = (uint32_t)(kdl * C::HBOX * C::WBOX + kw);
          uint32_t ln[K + 1][C::MB][2][4];
#pragma unroll
          for (int b = 0; b < C::MB; ++b) fold_load_line(ln[0][b], box, row0[b] + roff, mlane);
#pragma unroll
          for (int kh = 0; kh < K; ++kh) {
#pragma unroll
            for (int b = 0; b < C::MB; ++b) fold_load_line(ln[kh + 1][b], box, row0[b] + roff + (uint32_t)((kh + 1) * C::WBOX), mlane);
            wg_fence();
            const int tap = C::RES ? (kw * K + kd) * K + kh : kdl * K + kh;
            const uint64_t bd = make_sw128_desc(bslice + (uint32_t)(tap * C::TAP));
            const uint32_t acc = (as == 0 && kw == 0 && kdl == 0 && kh == 0) ? 0u : 1u;
#pragma unroll
            for (int b = 0; b < C::MB; ++b) fold_tap<NC>(d1[b], d2[b], ln[kh][b], ln[kh + 1][b], bd, acc);
            wg_commit();
            wg_wait<1>();
            if (!C::RES && kh == 0 && bprev >= 0) {   // every MMA of the previous weight slice has completed
              if (wg_lead) mbar_arrive_local(&bempty[bprev]);
              bprev = -1;
            }
          }
        }
        if (!C::RES) bprev = sb;
      }
      mbar_arrive_local(&aempty[sa]);   // this thread's ldmatrix reads of the box have completed
    }
    wg_wait<0>();
    if (!C::RES) {
      if (wg_lead) mbar_arrive_local(&bempty[bprev]);
      bprev = -1;
    }
#pragma unroll
    for (int b = 0; b < C::MB; ++b) { wg_fence_regs(d1[b]); wg_fence_regs(d2[b]); }

    // ---- epilogue ----
    int ow0, oh0, od0, nb;
    fold_tile_origin(p, t, ow0, oh0, od0, nb);
#pragma unroll
    for (int b = 0; b < C::MB; ++b) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r_lo + 8 * h;
        const int ow = ow0 + (r & 7), oh = oh0 + blk_hb[b] * 8 + (r >> 3), od = od0 + blk_dd[b];
        if (!(ow < p.OW && oh < p.OH && od < p.OD)) continue;
        const long opix = (((long)nb * p.FD + od) * p.FH + oh) * p.FW + ow;
        conv_epilogue_row<NC>(p, d1[b], d2[b], h, opix, 0, c2);
        if constexpr (NC == 16) {   // output channels 16..31: no weights
          const float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          conv_epilogue_row<16>(p, z, z, h, opix, 16, c2);
        }
      }
    }
  }
}

template <int K, int NC>
static int launch_fold(const CUtensorMap& tmA, const CUtensorMap& tmB, const TcParams& p, cudaStream_t st) {
  using C = FoldCfg<K, NC>;
  static DeviceOnce configured;
  if (configured.first()) {
    cudaError_t e = cudaFuncSetAttribute(conv_fold_kernel<K, NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFoldSmem);
    if (e != cudaSuccess) return fail(LT_ERR_CUDA, "conv_fold: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  }
  const long ntiles = (long)p.tw * p.th * p.td * p.tn;
  const int grid = (int)(ntiles < sm_count() ? ntiles : sm_count());
  conv_fold_kernel<K, NC><<<grid, kFoldThreads, C::SMEM, st>>>(tmA, tmB, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(LT_ERR_CUDA, "conv_fold_kernel: %s", cudaGetErrorString(e));
  return LT_OK;
}

template <int K, int NC>
static int conv_fold_run(const lt_conv_desc* d, const void* in, const void* weight, const float* scale, const float* shift,
                         const void* residual, void* out, cudaStream_t st) {
  using C = FoldCfg<K, NC>;
  TcParams p;
  fill_params(d, p, 1, NC, NC, 3, scale, shift, residual, out);
  p.bw = C::BW; p.bh = C::BH; p.bd = C::BD; p.bn = 1;
  p.tw = ceil_div(d->OW, p.bw); p.th = ceil_div(d->OH, p.bh); p.td = ceil_div(d->OD, p.bd); p.tn = d->N;
  p.stages = C::ARING;
  CUtensorMap tmA, tmB;
  int rc = make_in_map(&tmA, d, C::WBOX, C::HBOX, C::DBOX, 1, in);
  if (rc) return rc;
  const uint64_t dims[3] = {64, (uint64_t)NC, (uint64_t)K * K * K};
  const uint64_t str[2] = {128, (uint64_t)NC * 128};
  const uint32_t bx[3] = {64, (uint32_t)NC, (uint32_t)(C::B_SLICE / C::TAP)};
  rc = make_map(&tmB, weight, 3, dims, str, bx, nullptr, 1);
  if (rc) return rc;
  return launch_fold<K, NC>(tmA, tmB, p, st);
}

int conv_fold_supported(const lt_conv_desc* d) {
  const bool cubic = d->KD == d->KH && d->KH == d->KW && (d->KW == 3 || d->KW == 7);
  const int pd = d->KW / 2;
  return cubic && d->Cin == 32 && d->Cout <= 32 && d->sd == 1 && d->sh == 1 && d->sw == 1 && d->pd == pd && d->ph == pd &&
         d->pw == pd && d->OD == d->ID && d->OH == d->IH && d->OW == d->IW && d->osd == 1 && d->osh == 1 && d->osw == 1 &&
         d->ood == 0 && d->ooh == 0 && d->oow == 0 && d->FD == d->OD && d->FH == d->OH && d->FW == d->OW && d->FC == 32 &&
         d->in_format == LT_FMT_S32 && d->IW >= 16;
}

// desc->Cout = real output channel count; weights from lt_conv_fold_pack_weights with the same K and Cout
int conv_fold_fwd(const lt_conv_desc* d, const void* in, const void* weight, const float* scale, const float* shift,
                  const void* residual, void* out, void* stream) {
  LT_REQUIRE(conv_fold_supported(d), "conv_fold: unsupported layer shape");
  const cudaStream_t st = (cudaStream_t)stream;
  const bool narrow = d->Cout <= 16;
  if (d->KW == 3)
    return narrow ? conv_fold_run<3, 16>(d, in, weight, scale, shift, residual, out, st)
                  : conv_fold_run<3, 32>(d, in, weight, scale, shift, residual, out, st);
  return narrow ? conv_fold_run<7, 16>(d, in, weight, scale, shift, residual, out, st)
                : conv_fold_run<7, 32>(d, in, weight, scale, shift, residual, out, st);
}

// fp32 [K^3 taps (kd, kh, kw)][32][Cout] -> fp16 [kw][kd][kh][NC][32 hi | 32 lo] (128-byte rows), zero rows for Cout .. NC-1
__global__ void __launch_bounds__(256) fold_pack_weights_kernel(const float* __restrict__ w, sh_t* __restrict__ out, int K, int Cout,
                                                                int NC) {
  const int total = K * K * K * NC * 32;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int ci = i % 32;
    int r = i / 32;
    const int co = r % NC; r /= NC;
    const int kh = r % K; r /= K;
    const int kd = r % K;
    const int kw = r / K;
    const int tap = (kd * K + kh) * K + kw;
    const float v = co < Cout ? w[((long)tap * 32 + ci) * Cout + co] : 0.0f;
    sh_t hi, lo;
    split_s32(v, hi, lo);
    sh_t* rowp = out + ((long)((kw * K + kd) * K + kh) * NC + co) * 64;
    rowp[ci] = hi;
    rowp[32 + ci] = lo;
  }
}

}  // namespace lt

using namespace lt;

extern "C" size_t lt_conv_fold_weight_bytes(int K, int Cout) {
  const int NC = (Cout + 15) & ~15;
  return (size_t)K * K * K * NC * 128;
}

extern "C" int lt_conv_fold_pack_weights(const float* w_tap_ci_co, void* packed, int K, int Cout, void* stream) {
  LT_REQUIRE(w_tap_ci_co && packed && (K == 3 || K == 7) && Cout > 0 && Cout <= 32, "conv_fold_pack_weights: bad arguments");
  const int NC = (Cout + 15) & ~15;
  const int total = K * K * K * NC * 32;
  fold_pack_weights_kernel<<<ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(w_tap_ci_co, reinterpret_cast<sh_t*>(packed), K,
                                                                                   Cout, NC);
  LT_CHECK_LAUNCH("fold_pack_weights_kernel");
  return LT_OK;
}
