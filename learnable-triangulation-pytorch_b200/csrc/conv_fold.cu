// Halo-reusing wgmma convolution for the full-resolution V2V layers (LT_CONV_TC_FOLD): Cin = 32, cubic K = 3 or 7, stride 1,
// "same" padding, Cout <= 32.  Same arithmetic and epilogue as conv_tc_kernel (conv_tc.cu), different operand staging.
//
// The generic kernel loads one 128-position A tile per filter tap, so every input row is fetched K^3 times and each byte brought
// into the SM feeds only ~39 FLOP at these narrow N.  Here the output tile is 8 (w) x BH (h) x BD (d) positions whose 64-row m64
// blocks are whole 8-wide W lines at 8 consecutive h of one d plane, and a pipeline stage holds ONE input halo box
//   {64 channels, 8 (w), BH + K - 1 (h), BD + KDS - 1 (d)}   at input offset (kw - K/2, -K/2, kd0 - K/2)
// plus the KDS x K weight taps (kd0 .. kd0 + KDS - 1, all kh) of that kw.  The A operand of tap (kd0 + kdl, kh) for the m64 block at
// (d plane dd, h block hb) is the box at line (hb * 8 + kh) + (BH + K - 1) (dd + kdl): a whole number of 1024-byte swizzle atoms,
// i.e. a plain 128B-swizzle descriptor.  TMA zero fill supplies the padding.  Per tile and kw the input halo is read once instead
// of KDS x K times.
//
//   K = 3: tile 8 x 8 x 4 (KDS = 3: one stage per kw, box 8 x 10 x 6), 3 stages per tile
//   K = 7: tile 8 x 16 x 2 (KDS = 1: one stage per (kw, kd), box 8 x 22 x 2), 49 stages per tile
//
// Weights: lt_conv_fold_pack_weights, [kw][kd][kh][NC rows][32 hi | 32 lo] fp16, NC = round_up(Cout, 16), so the taps of one stage
// are one 3-D TMA box {64, NC, KDS * K}.  The N tile is NC: the 7^3 layer (Cout 16) multiplies no padding; output channels
// NC .. FC-1 go through the same epilogue with zero accumulators (scale 0, shift 0 for the padding channels: written as zeros).
//
// Each tile has 256 positions = 4 m64 blocks; consumer warpgroup g (1, 2) owns blocks 2 (g - 1) and 2 (g - 1) + 1, so every weight
// byte in shared memory feeds two MMAs.  Per 16-wide K slice hi*hi accumulates into D1 and hi*lo + lo*hi into D2, as in
// conv_tc_kernel: D1 takes K^3 x Cin / 16 accumulation steps per output (the accum_steps of the folded scale, engine._pack).
//
// Persistent grid: one CTA per SM strides over the tiles; the producer warp runs its ring across tile boundaries, so the next
// tile's first boxes load while the consumers run the epilogue of the previous one.
#include "tc_common.cuh"
#include "conv_tc_params.cuh"

namespace lt {

constexpr int kFoldThreads = 384;
constexpr int kFoldSmem = 227 * 1024;

template <int K>
struct FoldTile;
template <>
struct FoldTile<3> { static constexpr int BH = 8, BD = 4, KDS = 3; };
template <>
struct FoldTile<7> { static constexpr int BH = 16, BD = 2, KDS = 1; };

template <int K, int NC>
struct FoldCfg {
  static constexpr int BW = 8, BH = FoldTile<K>::BH, BD = FoldTile<K>::BD, KDS = FoldTile<K>::KDS;
  static constexpr int HBOX = BH + K - 1, DBOX = BD + KDS - 1;
  static constexpr int A_BYTES = BW * HBOX * DBOX * 128;
  static constexpr int B_BYTES = KDS * K * NC * 128;
  static constexpr int STAGE = A_BYTES + B_BYTES;
  static constexpr int KDG = K / KDS;         // stages per kw
  static constexpr int STAGES = K * KDG;      // stages per tile
  static constexpr int RING_MAX = (kFoldSmem - 1024 - 256) / STAGE;
  static constexpr int RING = RING_MAX > 4 ? 4 : RING_MAX;
  static constexpr size_t SMEM = (size_t)RING * STAGE + 2 * RING * 8 + 1024;
  static_assert(BW * BH * BD == 256 && BH % 8 == 0, "four m64 blocks of whole 8-wide lines per tile");
  static_assert(A_BYTES % 1024 == 0 && B_BYTES % 1024 == 0, "boxes must start on 1024-byte swizzle atoms");
  static_assert(RING >= 2 && SMEM <= (size_t)kFoldSmem, "shared memory");
};

__device__ __forceinline__ void fold_tile_origin(const TcParams& p, int t, int& ow0, int& oh0, int& od0, int& nb) {
  ow0 = (t % p.tw) * p.bw; t /= p.tw;
  oh0 = (t % p.th) * p.bh; t /= p.th;
  od0 = (t % p.td) * p.bd;
  nb = t / p.td;
}

template <int K, int NC>
__global__ void __launch_bounds__(kFoldThreads, 1) conv_fold_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                    const __grid_constant__ CUtensorMap tmB, const TcParams p) {
  using C = FoldCfg<K, NC>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)C::RING * C::STAGE);
  uint64_t* empty = full + C::RING;

  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int lane = threadIdx.x & 31;
  const int ntiles = p.tw * p.th * p.td * p.tn;

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::RING; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    fence_barrier_init();
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
  }
  __syncthreads();

  if (wg == 0) {
    // ================= TMA producer (warp 0; one elected lane issues) =================
    regs_release_producer();
    if (threadIdx.x < 32) {
      int s = 0;
      uint32_t ph = 0;
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        int ow0, oh0, od0, nb;
        fold_tile_origin(p, t, ow0, oh0, od0, nb);
        for (int j = 0; j < C::STAGES; ++j) {
          const int kw = j / C::KDG, kd0 = (j - kw * C::KDG) * C::KDS;
          mbar_wait(&empty[s], ph ^ 1u);
          uint8_t* dst = smem + (size_t)s * C::STAGE;
          if (elect_one()) {
            mbar_expect_tx(&full[s], (uint32_t)C::STAGE);
            tma_load_5d(dst, &tmA, &full[s], 0, ow0 + kw - K / 2, oh0 - K / 2, od0 + kd0 - K / 2, nb);
            tma_load_3d(dst + C::A_BYTES, &tmB, &full[s], 0, 0, (kw * K + kd0) * K);
          }
          __syncwarp();
          if (++s == C::RING) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }

  // ================= MMA + epilogue (warpgroups 1, 2: m64 blocks 2 g, 2 g + 1 of the tile) =================
  regs_claim_consumer();
  const int g = wg - 1;
  float d1[2][NC / 2], d2[2][NC / 2];
#pragma unroll
  for (int b = 0; b < 2; ++b)
#pragma unroll
    for (int i = 0; i < NC / 2; ++i) { d1[b][i] = 0.f; d2[b][i] = 0.f; }
  // m64 block b of this warpgroup: d plane dd and 8-line h block hb of the tile -> first box line it reads (kh = kdl = 0)
  uint32_t line0[2];
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const int blk = 2 * g + b, dd = blk / (C::BH / 8), hb = blk % (C::BH / 8);
    line0[b] = (uint32_t)(hb * 8 + C::HBOX * dd);
  }
  const int r_lo = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);   // this thread's rows r_lo, r_lo + 8 of an m64 block
  const int c2 = 2 * (lane & 3);
  const uint32_t ring0 = smem_u32(smem);
  int s = 0;
  uint32_t ph = 0;
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    int prev = -1;
    for (int j = 0; j < C::STAGES; ++j) {
      mbar_wait(&full[s], ph);
      const uint32_t a_base = ring0 + (uint32_t)(s * C::STAGE), b_base = a_base + C::A_BYTES;
      wg_fence();
#pragma unroll
      for (int kdl = 0; kdl < C::KDS; ++kdl) {
#pragma unroll
        for (int kh = 0; kh < K; ++kh) {
          const uint32_t acc = (j == 0 && kdl == 0 && kh == 0) ? 0u : 1u;
          const uint64_t bd = make_sw128_desc(b_base + (uint32_t)((kdl * K + kh) * NC * 128));
#pragma unroll
          for (int b = 0; b < 2; ++b) {
            const uint64_t ad = make_sw128_desc(a_base + (line0[b] + (uint32_t)(kh + C::HBOX * kdl)) * 1024u);
            wgmma_f16<NC>(d1[b], ad, bd, acc);              // hi * hi
            wgmma_f16<NC>(d1[b], ad + 2, bd + 2, 1u);
            wgmma_f16<NC>(d2[b], ad, bd + 4, acc);          // hi * lo
            wgmma_f16<NC>(d2[b], ad + 2, bd + 6, 1u);
            wgmma_f16<NC>(d2[b], ad + 4, bd, 1u);           // lo * hi
            wgmma_f16<NC>(d2[b], ad + 6, bd + 2, 1u);
          }
        }
      }
      wg_commit();
      wg_wait<1>();                                          // the MMAs of the previous stage have completed: release it
      if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive_local(&empty[prev]);
      prev = s;
      if (++s == C::RING) { s = 0; ph ^= 1u; }
    }
    wg_wait<0>();
    if ((threadIdx.x & 127) == 0) mbar_arrive_local(&empty[prev]);   // the producer refills it during the epilogue
#pragma unroll
    for (int b = 0; b < 2; ++b) { wg_fence_regs(d1[b]); wg_fence_regs(d2[b]); }

    // ---- epilogue ----
    int ow0, oh0, od0, nb;
    fold_tile_origin(p, t, ow0, oh0, od0, nb);
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int blk = 2 * g + b, dd = blk / (C::BH / 8), hb = blk % (C::BH / 8);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r_lo + 8 * h;
        const int ow = ow0 + (r & 7), oh = oh0 + hb * 8 + (r >> 3), od = od0 + dd;
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
  p.stages = C::RING;
  CUtensorMap tmA, tmB;
  int rc = make_in_map(&tmA, d, C::BW, C::HBOX, C::DBOX, 1, in);
  if (rc) return rc;
  const uint64_t dims[3] = {64, (uint64_t)NC, (uint64_t)K * K * K};
  const uint64_t str[2] = {128, (uint64_t)NC * 128};
  const uint32_t bx[3] = {64, (uint32_t)NC, (uint32_t)(C::KDS * K)};
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
