// Fused tail of the V2V network (reference v2v.py:154-160, 168-169): back_layers[1] (1x1x1 conv 32->32 + BN + ReLU),
// back_layers[2] (same) and output_layer (1x1x1 conv 32->J, bias) as ONE kernel.
//
// Unfused, each of the three point-wise layers reads and writes the whole 64^3 x 32-channel volume (2 x 268 MB per layer at
// B = 8): pure HBM round trips for 5 GFLOP.  Here a CTA streams 128-voxel tiles of the input once (TMA, 16 KB), chains the
// three 128 x 32 x 32 GEMMs on the tensor cores (wgmma, 3-term split-fp16 products, fp32 accumulators in registers) with the
// two hidden activations going registers (scale / shift / ReLU / split) -> a swizzled shared-memory tile that is the next
// GEMM's A operand, and writes only the logits (float32, `FC` floats per voxel: 17 joints rounded up to 20).
// HBM traffic: 128 B in + 80 B out per voxel instead of 3 x 256 B.
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (weights once, then the input tiles through a two-stage ring),
// warpgroups 1 and 2 = GEMM chain + activations for rows 0-63 / 64-127 of a tile, each with its own hidden tile.  Two CTAs
// per SM overlap one CTA's serial chain with the other's.
#include "conv_tc_params.cuh"
#include "softargmax_common.cuh"

namespace lt {

struct TailParams {
  const float* scale1; const float* shift1;   // [32] folded BN of back_layers[1]
  const float* scale2; const float* shift2;   // [32] back_layers[2]
  const float* scale3; const float* bias3;    // [FC] output layer: 1 / (filter pre-scale) and bias (zero padded)
  float* logits;                              // [rows][FC]
  long rows;
  long tiles;
  int FC;
  // fused statistics pass of the volumetric soft-argmax (op.py:84-96; null coord = off): rows = B x nvox, nvox % 128 == 0
  const float* coord;                         // [rows][3]
  float* partial;                             // [B][gridDim.x][J][5] online-softmax partials (max, sum e, sum e x, sum e y, sum e z)
  int B, J, tiles_per_sample, softmax;
  float mult;
};

constexpr int kTailThreads = 384;
constexpr int kTailStages = 2;
constexpr int kTailWBytes = 32 * 128;        // one 32 x [32 hi | 32 lo] weight tile
constexpr int kTailHBytes = 64 * 128;        // hidden tile of one consumer warpgroup: 64 rows x [32 hi | 32 lo]
// smem: A ring | H tiles [2] | W1 W2 W3 | barriers
constexpr int kTailOffH = kTailStages * kATileBytes;
constexpr int kTailOffW = kTailOffH + 2 * kTailHBytes;
constexpr int kTailOffBar = kTailOffW + 3 * kTailWBytes;
// fused statistics: per consumer warp a [16 rows][FC <= 20 floats] logit tile + [16][4] coordinates, then the [8][32][5] merge scratch
constexpr int kTailStatMaxFC = 20;
constexpr int kTailOffStat = kTailOffBar + 128;
constexpr int kTailStatWarpBytes = 16 * kTailStatMaxFC * 4 + 16 * 16;
constexpr int kTailOffMerge = kTailOffStat + 8 * kTailStatWarpBytes;
constexpr int kTailSmem = kTailOffBar + 128 + 1024;
constexpr int kTailSmemStats = kTailOffMerge + 8 * 32 * 5 * 4 + 1024;

__device__ __forceinline__ void tail_wg_sync(int g) {   // the 128 threads of consumer warpgroup g
  if (g == 0) asm volatile("bar.sync 1, 128;" ::: "memory");
  else asm volatile("bar.sync 2, 128;" ::: "memory");
}
__device__ __forceinline__ void tail_consumers_sync() { asm volatile("bar.sync 3, 256;" ::: "memory"); }

// 64 x 32 x 32 GEMM of one warpgroup on split-fp16 rows [32 hi | 32 lo]: K slices hi0 +0, hi1 +2, lo0 +4, lo1 +6 (16-byte units);
// hi*hi, hi*lo and lo*hi into one accumulator; returns once the MMAs have completed
__device__ __forceinline__ void gemm32(float (&d)[16], uint64_t ad, uint64_t bd) {
  wg_fence();
  wgmma_f16<32>(d, ad, bd, 0u);
  wgmma_f16<32>(d, ad + 2, bd + 2, 1u);
  wgmma_f16<32>(d, ad, bd + 4, 1u);
  wgmma_f16<32>(d, ad + 2, bd + 6, 1u);
  wgmma_f16<32>(d, ad + 4, bd, 1u);
  wgmma_f16<32>(d, ad + 6, bd + 2, 1u);
  wg_commit();
  wg_wait<0>();
  wg_fence_regs(d);
}

// scale / shift / ReLU of a hidden layer and its split-fp16 store into the warpgroup's swizzled hidden tile (the next A operand):
// this thread's accumulator elements are rows rl + 8 (k / 2 & 1), channels 8 (k / 4) + c2 + (k & 1)
__device__ __forceinline__ void hidden_store(const float (&d)[16], const float* __restrict__ scale, const float* __restrict__ shift,
                                             uint32_t hbase, int rl, int c2) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = 8 * i + c2;
    const float2 sc = __ldg(reinterpret_cast<const float2*>(scale + c));
    const float2 sh = __ldg(reinterpret_cast<const float2*>(shift + c));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = rl + 8 * h;
      const float v0 = fmaxf(fmaf(d[4 * i + 2 * h], sc.x, sh.x), 0.f), v1 = fmaxf(fmaf(d[4 * i + 2 * h + 1], sc.y, sh.y), 0.f);
      uint32_t hi2, lo2;
      split_s32x2(v0, v1, hi2, lo2);
      // hi halves of channels 8i..8i+7 = 16-byte chunk i of the row, lo halves = chunk 4 + i; 128-byte swizzle
      const uint32_t sw = (uint32_t)(r & 7);
      asm volatile("st.shared.u32 [%0], %1;" ::"r"(hbase + r * 128 + (((uint32_t)i ^ sw) << 4) + c2 * 2), "r"(hi2) : "memory");
      asm volatile("st.shared.u32 [%0], %1;" ::"r"(hbase + r * 128 + (((uint32_t)(4 + i) ^ sw) << 4) + c2 * 2), "r"(lo2) : "memory");
    }
  }
}

// STATS: 0 = logits only, 1 = + softmax statistics, 2 = + ReLU ("volume_softmax: false") statistics.  The logits a warp has just
// produced (16 voxel rows x J joints) are transposed through a warp-private shared-memory tile so that lane j folds joint j of the
// 16 rows into its online-softmax state (4 rows per step: one rescale + four ex2); the state lives in five registers per lane for
// the whole kernel and is written per (sample, CTA) -- the logits are never re-read for the statistics.
template <int STATS>
__global__ void __launch_bounds__(kTailThreads, 2) v2v_tail_kernel(const __grid_constant__ CUtensorMap tmX,
                                                                    const __grid_constant__ CUtensorMap tmW1,
                                                                    const __grid_constant__ CUtensorMap tmW2,
                                                                    const __grid_constant__ CUtensorMap tmW3, const TailParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* w_tiles = smem + kTailOffW;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + kTailOffBar);   // [2]
  uint64_t* a_empty = a_full + kTailStages;                             // [2]
  uint64_t* w_full = a_empty + kTailStages;                             // [1]

  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kTailStages; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 2); }
    mbar_init(w_full, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ================= producer: weights once, then the input tiles =================
    if (threadIdx.x < 32) {
      if (elect_one()) {
        prefetch_tmap(&tmX);
        mbar_expect_tx(w_full, 3u * kTailWBytes);
        tma_load_2d(w_tiles, &tmW1, w_full, 0, 0);
        tma_load_2d(w_tiles + kTailWBytes, &tmW2, w_full, 0, 0);
        tma_load_2d(w_tiles + 2 * kTailWBytes, &tmW3, w_full, 0, 0);
      }
      __syncwarp();
      uint32_t s = 0, ph = 0;
      for (long t = blockIdx.x; t < p.tiles; t += gridDim.x) {
        mbar_wait(&a_empty[s], ph ^ 1u);
        if (elect_one()) {
          mbar_expect_tx(&a_full[s], (uint32_t)kATileBytes);
          tma_load_2d(smem + s * kATileBytes, &tmX, &a_full[s], 0, (int)(t * 128));
        }
        __syncwarp();
        if (++s == kTailStages) { s = 0; ph ^= 1u; }
      }
    }
    return;
  }

  // ================= consumers: warpgroup g owns rows 64 g .. 64 g + 63 of every tile =================
  const int g = wg - 1;
  const int wq = (threadIdx.x >> 5) & 3;
  const int rl = wq * 16 + (lane >> 2);          // this thread's rows rl and rl + 8 of the warpgroup's 64
  const int c2 = 2 * (lane & 3);
  const uint32_t hbase = smem_u32(smem + kTailOffH + g * kTailHBytes);
  const uint64_t hd = make_sw128_desc(hbase);
  const uint64_t w1 = make_sw128_desc(smem_u32(w_tiles)), w2 = make_sw128_desc(smem_u32(w_tiles + kTailWBytes)),
                 w3 = make_sw128_desc(smem_u32(w_tiles + 2 * kTailWBytes));
  // fused statistics state
  constexpr bool SM = STATS == 1;
  const int aw = g * 4 + wq;                     // consumer warp 0..7
  float* lg_s = reinterpret_cast<float*>(smem + kTailOffStat + aw * kTailStatWarpBytes);     // [16][FC]
  float4* cd_s = reinterpret_cast<float4*>(lg_s + 16 * kTailStatMaxFC);                      // [16] (x, y, z, -)
  float* merge_s = reinterpret_cast<float*>(smem + kTailOffMerge);                          // [8][32][5]
  SoftState st;
  st_init(st, SM);
  int cur_b = -1;
  auto flush = [&](int b) {      // CTA merge of the eight warps' states -> partial[b][blockIdx.x][j], then reset (CTA-uniform call sites)
    float* my = merge_s + (aw * 32 + lane) * 5;
    my[0] = st.m; my[1] = st.d; my[2] = st.sx; my[3] = st.sy; my[4] = st.sz;
    st_init(st, SM);
    tail_consumers_sync();
    if (aw == 0 && lane < p.J) {
      SoftState a{merge_s[lane * 5], merge_s[lane * 5 + 1], merge_s[lane * 5 + 2], merge_s[lane * 5 + 3], merge_s[lane * 5 + 4]};
#pragma unroll
      for (int w = 1; w < 8; ++w) {
        const float* o = merge_s + (w * 32 + lane) * 5;
        SoftState t{o[0], o[1], o[2], o[3], o[4]};
        st_merge(a, t, SM);
      }
      float* dst = p.partial + (((long)b * gridDim.x + blockIdx.x) * p.J + lane) * 5;
      dst[0] = a.m; dst[1] = a.d; dst[2] = a.sx; dst[3] = a.sy; dst[4] = a.sz;
    }
    tail_consumers_sync();
  };
  if (STATS) {
    // samples in which this CTA owns no tile still need an (identity) partial for the merge
    for (int i = threadIdx.x - 128; i < p.B * p.J; i += 256) {
      const int b = i / p.J, j = i % p.J;
      const long lo = (long)b * p.tiles_per_sample, G = gridDim.x;
      const long f0 = lo + (((long)blockIdx.x - lo) % G + G) % G;     // first tile >= lo owned by this CTA
      if (!(f0 < lo + p.tiles_per_sample)) {
        float* dst = p.partial + (((long)b * G + blockIdx.x) * p.J + j) * 5;
        dst[0] = SM ? -INFINITY : 0.0f; dst[1] = 0.f; dst[2] = 0.f; dst[3] = 0.f; dst[4] = 0.f;
      }
    }
  }

  mbar_wait(w_full, 0);
  uint32_t s = 0, ph = 0;
  for (long t = blockIdx.x; t < p.tiles; t += gridDim.x) {
    if (STATS) {
      // rows = B x nvox with nvox % 128 == 0: every tile is full and lies inside one sample; a sample boundary closes the
      // previous sample's partial (CTA-uniform)
      const int b = (int)(t / p.tiles_per_sample);
      if (b != cur_b) {
        if (cur_b >= 0) flush(cur_b);
        cur_b = b;
      }
    }
    float d[16];
    mbar_wait(&a_full[s], ph);
    gemm32(d, make_sw128_desc(smem_u32(smem + s * kATileBytes + g * kTailHBytes)), w1);
    if ((threadIdx.x & 127) == 0) mbar_arrive_local(&a_empty[s]);
    if (++s == kTailStages) { s = 0; ph ^= 1u; }
#pragma unroll
    for (int layer = 0; layer < 2; ++layer) {
      tail_wg_sync(g);           // the previous MMA that read the hidden tile has completed in every warp
      hidden_store(d, layer == 0 ? p.scale1 : p.scale2, layer == 0 ? p.shift1 : p.shift2, hbase, rl, c2);
      fence_proxy_async();       // generic-proxy stores -> visible to the MMA's operand reads
      tail_wg_sync(g);
      gemm32(d, hd, layer == 0 ? w2 : w3);
    }
    // ---- logits (and their statistics) ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int rw = (lane >> 2) + 8 * h;        // row within this warp's 16
      const long vox = t * 128 + g * 64 + rl + 8 * h;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = 8 * i + c2;
        if (c < p.FC) {
          const float2 a = __ldg(reinterpret_cast<const float2*>(p.scale3 + c));
          const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias3 + c));
          const float2 o = make_float2(fmaf(d[4 * i + 2 * h], a.x, bb.x), fmaf(d[4 * i + 2 * h + 1], a.y, bb.y));
          if (vox < p.rows) *reinterpret_cast<float2*>(p.logits + vox * p.FC + c) = o;
          if (STATS) *reinterpret_cast<float2*>(lg_s + rw * p.FC + c) = o;
        }
      }
    }
    if (STATS) {
      if (lane < 16) {
        const long vox = t * 128 + g * 64 + wq * 16 + lane;
        const float* cp = p.coord + vox * 3;
        cd_s[lane] = make_float4(__ldg(cp), __ldg(cp + 1), __ldg(cp + 2), 0.f);
      }
      __syncwarp();
      if (lane < p.J) {
        for (int r0 = 0; r0 < 16; r0 += 4) {
          float l[4], x[4], y[4], z[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            l[k] = lg_s[(r0 + k) * p.FC + lane] * p.mult;
            const float4 c = cd_s[r0 + k];
            x[k] = c.x; y[k] = c.y; z[k] = c.z;
          }
          st_push4<SM>(st, l, x, y, z);
        }
      }
      __syncwarp();
    }
  }
  if (STATS && cur_b >= 0) flush(cur_b);
}

}  // namespace lt

using namespace lt;

// shared launcher: stats = 0 (logits only), 1 (softmax statistics), 2 (ReLU statistics); returns the grid size through *grid_out
static int launch_tail(const void* x, const void* w1, const void* w2, const void* w3, lt::TailParams& p, int stats, int* grid_out, void* stream) {
  using namespace lt;
  CUtensorMap tmX, tmW[3];
  {
    const uint64_t dims[2] = {64, (uint64_t)p.rows};
    const uint64_t str[1] = {128};
    const uint32_t bx[2] = {64, 128};
    int rc = make_map(&tmX, x, 2, dims, str, bx, nullptr, 1);
    if (rc) return rc;
  }
  // each map spans the rows the buffer holds; the 32-row box reads past the 16 rows of a w3 with J <= 16 as zeros (TMA fill)
  const void* ws[3] = {w1, w2, w3};
  const uint64_t wrows[3] = {32, 32, (uint64_t)((p.FC + 15) & ~15)};
  for (int i = 0; i < 3; ++i) {
    const uint64_t dims[2] = {64, wrows[i]};
    const uint64_t str[1] = {128};
    const uint32_t bx[2] = {64, 32};
    int rc = make_map(&tmW[i], ws[i], 2, dims, str, bx, nullptr, 1);
    if (rc) return rc;
  }
  p.tiles = (p.rows + 127) / 128;
  static DeviceOnce configured;
  if (configured.first()) {
    cudaError_t e = cudaFuncSetAttribute(v2v_tail_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTailSmem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(v2v_tail_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTailSmemStats);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(v2v_tail_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTailSmemStats);
    if (e != cudaSuccess) return fail(LT_ERR_CUDA, "v2v_tail: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  }
  long grid = 2L * sm_count();
  if (grid > p.tiles) grid = p.tiles;
  if (grid_out) *grid_out = (int)grid;
  cudaStream_t st = (cudaStream_t)stream;
  if (stats == 1) v2v_tail_kernel<1><<<(unsigned)grid, kTailThreads, kTailSmemStats, st>>>(tmX, tmW[0], tmW[1], tmW[2], p);
  else if (stats == 2) v2v_tail_kernel<2><<<(unsigned)grid, kTailThreads, kTailSmemStats, st>>>(tmX, tmW[0], tmW[1], tmW[2], p);
  else v2v_tail_kernel<0><<<(unsigned)grid, kTailThreads, kTailSmem, st>>>(tmX, tmW[0], tmW[1], tmW[2], p);
  LT_CHECK_LAUNCH("v2v_tail_kernel");
  return LT_OK;
}

// x: split-fp16 rows [rows][32 hi | 32 lo]; w1/w2/w3: lt_conv_tc_pack_weights(taps = 1, Cin = 32, Cout = 32 / 32 / J) buffers
// (32, 32 and round_up(FC, 16) rows); scale/shift: folded BN of the two hidden layers; scale3 / bias3 [FC]: output affine
// (scale3 = 1 / filter pre-scale, bias zero padded);
// logits float32 [rows][FC], FC % 4 == 0, J <= FC <= 32.
extern "C" int lt_v2v_tail_fwd(const void* x, const void* w1, const void* w2, const void* w3, const float* scale1, const float* shift1,
                               const float* scale2, const float* shift2, const float* scale3, const float* bias3, float* logits, long rows,
                               int FC, void* stream) {
  LT_REQUIRE(x && w1 && w2 && w3 && scale1 && shift1 && scale2 && shift2 && scale3 && bias3 && logits, "v2v_tail: null pointer");
  LT_REQUIRE(rows > 0 && rows < (1L << 31) && FC % 4 == 0 && FC >= 4 && FC <= 32, "v2v_tail: bad sizes (rows=%ld FC=%d)", rows, FC);
  TailParams p;
  p.scale1 = scale1; p.shift1 = shift1; p.scale2 = scale2; p.shift2 = shift2; p.scale3 = scale3; p.bias3 = bias3;
  p.logits = logits; p.rows = rows; p.FC = FC;
  p.coord = nullptr; p.partial = nullptr; p.B = 0; p.J = 0; p.tiles_per_sample = 1; p.softmax = 0; p.mult = 1.0f;
  return launch_tail(x, w1, w2, w3, p, 0, nullptr, stream);
}

// Same kernel with the statistics pass of the volumetric soft-argmax (op.py:84-96) fused into the epilogue that produces the logits:
// rows = B x nvox (nvox % 128 == 0, nvox >= 16384, FC == 20: the statistics tile holds at most 20 floats per voxel and the finish
// streams no narrower rows, stream_layout_ok), coord [B][nvox][3]; `workspace` (lt_softargmax3d_workspace_bytes) receives the
// online-softmax partials [B][*n_partials][J][5]; lt_softargmax3d_finish_fwd(..., G = *n_partials, ...) then merges them into the key
// points and writes the normalised volumes.  softmax: 1 = softmax, 0 = ReLU ("volume_softmax: false").
extern "C" int lt_v2v_tail_stats_fwd(const void* x, const void* w1, const void* w2, const void* w3, const float* scale1, const float* shift1,
                                     const float* scale2, const float* shift2, const float* scale3, const float* bias3, float* logits, int B,
                                     long nvox, int FC, const float* coord, int J, float multiplier, int softmax, void* workspace,
                                     size_t workspace_bytes, int* n_partials, void* stream) {
  LT_REQUIRE(x && w1 && w2 && w3 && scale1 && shift1 && scale2 && shift2 && scale3 && bias3 && logits && coord && workspace && n_partials,
             "v2v_tail_stats: null pointer");
  LT_REQUIRE(B > 0 && nvox > 0 && nvox % 128 == 0 && (long)B * nvox < (1L << 31), "v2v_tail_stats: bad sizes (B=%d nvox=%ld)", B, nvox);
  LT_REQUIRE(FC % 4 == 0 && FC >= 4 && FC <= kTailStatMaxFC && J > 0 && J <= FC, "v2v_tail_stats: need J <= FC <= %d, FC %% 4 == 0", kTailStatMaxFC);
  // only partials that lt_softargmax3d_finish_fwd can merge: with FC <= 20 that is FC == 20 (J 17..20) and nvox >= 16384
  LT_REQUIRE(stream_layout_ok(FC, J, nvox), "v2v_tail_stats: logits of width FC=%d (J=%d, nvox=%ld) are not covered by the streaming finish",
             FC, J, nvox);
  LT_REQUIRE(softmax == 0 || softmax == 1, "v2v_tail_stats: mode must be 0 (ReLU) or 1 (softmax)");
  LT_REQUIRE(workspace_bytes >= lt_softargmax3d_workspace_bytes(B, J, nvox), "v2v_tail_stats: workspace too small");
  TailParams p;
  p.scale1 = scale1; p.shift1 = shift1; p.scale2 = scale2; p.shift2 = shift2; p.scale3 = scale3; p.bias3 = bias3;
  p.logits = logits; p.rows = (long)B * nvox; p.FC = FC;
  p.coord = coord; p.partial = reinterpret_cast<float*>(workspace); p.B = B; p.J = J; p.tiles_per_sample = (int)(nvox / 128);
  p.softmax = softmax; p.mult = multiplier;
  return launch_tail(x, w1, w2, w3, p, softmax ? 1 : 2, n_partials, stream);
}
