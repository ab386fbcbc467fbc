// Weight gradient of lt_conv_nd_fwd on the tensor cores (sm_90a), the training counterpart of conv_tc_kernel:
//   dW[t][ci][co] = sum_{n, o} in[n, o s - p + t][ci] * dout[n, o os + oo][co]
// GEMM view: M = taps x Cin, N = Cout, K = output positions.  Both operands are the split-fp16 channels-last rows the forward
// stages, TMA-loaded into 128B-swizzled shared memory: per M tile of 128 positions (the forward's box) one box of `in` at the
// tap-shifted coordinates and one box of `dout` per 32-channel output block.  A box row (one position, [32 hi | 32 lo]) runs
// along M (or N) and the rows run along K, so both are MN-major wgmma operands as they land: one m64n64k16 MMA per 16 positions
// yields hi*hi, hi*lo, lo*hi and lo*lo in the four 32 x 32 quadrants of its accumulator, which the epilogue adds (four-term
// products: fp32-grade, and the small cross products never enter the big sum).
//
// Precision: every M tile (8 MMAs) starts a fresh tensor-core accumulator that is then added into an fp32 register sum with
// round-to-nearest, so the truncating tensor-core accumulation never runs longer than 128 positions.  `dout` is expected
// pre-scaled by a power of two (lt_f32_to_s32_scaled) so that gradients far below fp16's normal range keep their bits; the
// reduce pass divides the scale out exactly.  Per element, |dW - float64| <= 2 (8 + ceil(m_tiles / splits) + 3 + splits) 2^-24
// sum|x||g| / S + 2^-24 |dW| (8 truncating k16 steps per tile, one rounded add per tile of a split, three quadrant adds, the split
// reduce): tests/test_gpu_conv_bwd.py holds every instantiation, split and ring depth to it (worst err/bar 0.16 on an H100 80GB
// HBM3 at 700 W) and measures the systematic gain on a 4096-tile layer at -1.55e-7 (the 8-step truncation model: -1.34e-7), small
// enough to leave uncompensated.  lt_conv_wgrad_plan exposes the launch plan to the host (tests/test_conv_bwd_cpu.py).
//
// Determinism: the K loop (M tiles) is split over CTAs in fixed contiguous ranges; each writes an fp32 partial tile and
// wgrad_reduce_kernel sums the partials in split order.  No atomics.
//
// CTA = (tap, 32-channel input block, group of <= 4 output blocks, K split); one consumer warpgroup per output block; thread 0
// issues the TMA loads `stages` M tiles ahead.
#include "tc_common.cuh"
#include "conv_tc_params.cuh"
#include <string.h>

namespace lt {

constexpr int kWgBox = 128 * 128;   // one TMA box: 128 positions x 64 fp16

struct WgParams {
  TcParams g;         // geometry of the forward launch (fill_params): M-tile box, taps, strides, padding, output mapping
  int ncb;            // 32-channel GEMM column blocks (N / 32)
  int ngroups;        // CTAs along N: ceil(ncb / warpgroups per CTA)
  int m_tiles, splits, stages;
  float* ws;          // fp32 partials [splits][taps][32 CB][32 ncb]
};

// ---- index mapping (shared with the CPU test hook) ----
// Box origins of M tile m for filter tap `tap`: the input box at the tap-shifted coordinates (the TMA traversal strides of the
// input map step it by the conv stride), the output-gradient box at the tile's output positions.
struct WgBoxes {
  int ax, ay, az;       // input box origin (w, h, d)
  int ow0, oh0, od0;    // output positions of the tile
  int nb0;              // first sample
};
__host__ __device__ inline WgBoxes wgrad_boxes(const TcParams& p, int m, int tap) {
  WgBoxes b;
  int t = m;
  b.ow0 = (t % p.tw) * p.bw; t /= p.tw;
  b.oh0 = (t % p.th) * p.bh; t /= p.th;
  b.od0 = (t % p.td) * p.bd;
  b.nb0 = (t / p.td) * p.bn;
  const int kw = tap % p.KW, kh = (tap / p.KW) % p.KH, kd = tap / (p.KW * p.KH);
  b.ax = b.ow0 * p.sw - p.pw + kw;
  b.ay = b.oh0 * p.sh - p.ph + kh;
  b.az = b.od0 * p.sd - p.pd + kd;
  return b;
}
// GEMM column block j (32 channels) -> output group g (its phase of the output lattice) and first channel c inside the group
__host__ __device__ inline void wgrad_col_block(const TcParams& p, int j, int& g, int& c) {
  g = p.n_maps > 1 ? 32 * j / p.oc : 0;
  c = 32 * j - g * p.oc;
}
// Row r of the boxes of M tile b: input position (or false where TMA zero-fills it) and output-gradient pixel (or false outside
// the launch's output grid).  Group g lands at output offset (ood + a, ooh + b, oow + c) as in the forward's epilogue.
__host__ __device__ inline bool wgrad_in_row(const TcParams& p, const WgBoxes& b, int r, int ID, int IH, int IW, long& pix) {
  const int dw = r % p.bw, dh = (r / p.bw) % p.bh, dd = (r / (p.bw * p.bh)) % p.bd, dn = r / (p.bw * p.bh * p.bd);
  const int x = b.ax + dw * p.sw, y = b.ay + dh * p.sh, z = b.az + dd * p.sd, n = b.nb0 + dn;
  if (x < 0 || y < 0 || z < 0 || x >= IW || y >= IH || z >= ID || n >= p.N) return false;
  pix = (((long)n * ID + z) * IH + y) * IW + x;
  return true;
}
__host__ __device__ inline bool wgrad_out_row(const TcParams& p, const WgBoxes& b, int r, int g, long& pix) {
  const int dw = r % p.bw, dh = (r / p.bw) % p.bh, dd = (r / (p.bw * p.bh)) % p.bd, dn = r / (p.bw * p.bh * p.bd);
  const int ow = b.ow0 + dw, oh = b.oh0 + dh, od = b.od0 + dd, n = b.nb0 + dn;
  if (ow >= p.OW || oh >= p.OH || od >= p.OD || n >= p.N) return false;
  const int ga = g / (p.gh * p.gw), gb = (g / p.gw) % p.gh, gc = g % p.gw;
  pix = (((long)n * p.FD + od * p.osd + p.ood + ga) * p.FH + oh * p.osh + p.ooh + gb) * p.FW + ow * p.osw + p.oow + gc;
  return true;
}

// m64n64k16 with both operands MN-major (transposed): A rows and B rows run along K in shared memory
__device__ __forceinline__ void wgmma_f16_mn64(float (&d)[32], uint64_t ad, uint64_t bd, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(ad), "l"(bd), "r"(scale_d));
}

template <int NWG>
__global__ void __launch_bounds__(128 * NWG, 1) conv_wgrad_kernel(const __grid_constant__ CUtensorMap tmIn,
                                                                  const __grid_constant__ TcEpiMaps tmG, const WgParams P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int kStage = kWgBox * (1 + NWG);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)P.stages * kStage);
  const TcParams& p = P.g;

  int u = blockIdx.x;
  const int z = u % P.splits; u /= P.splits;
  const int ng = u % P.ngroups; u /= P.ngroups;
  const int cb = u % p.CB;
  const int tap = u / p.CB;
  const int taps = p.KD * p.KH * p.KW;
  const int j0 = ng * NWG;
  const int nj = min(NWG, P.ncb - j0);
  const int m_begin = (int)((long)z * P.m_tiles / P.splits);
  const int n = (int)((long)(z + 1) * P.m_tiles / P.splits) - m_begin;
  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < P.stages; ++s) mbar_init(&full[s], 1);
    fence_barrier_init();
    prefetch_tmap(&tmIn);
  }
  __syncthreads();

  auto issue = [&](int i, int s) {
    const WgBoxes b = wgrad_boxes(p, m_begin + i, tap);
    uint8_t* dst = smem + (size_t)s * kStage;
    mbar_expect_tx(&full[s], (uint32_t)(kWgBox * (1 + nj)));   // out-of-range rows arrive as zeros
    tma_load_5d(dst, &tmIn, &full[s], cb * 64, b.ax, b.ay, b.az, b.nb0);
    for (int jj = 0; jj < nj; ++jj) {
      int g, c;
      wgrad_col_block(p, j0 + jj, g, c);
      tma_load_5d(dst + kWgBox * (1 + jj), &tmG.out[g], &full[s], 2 * c, b.ow0, b.oh0, b.od0, b.nb0);
    }
  };
  if (threadIdx.x == 0)
    for (int s = 0; s < P.stages && s < n; ++s) issue(s, s);

  float acc[32], sum[32];
#pragma unroll
  for (int r = 0; r < 32; ++r) { acc[r] = 0.f; sum[r] = 0.f; }
  const bool active = wg < nj;
  const uint32_t ring0 = smem_u32(smem);
  for (int i = 0; i < n; ++i) {
    const int s = i % P.stages;
    mbar_wait(&full[s], (uint32_t)((i / P.stages) & 1));
    if (active) {
      const uint32_t a = ring0 + (uint32_t)(s * kStage);
      const uint64_t ad = make_sw128_desc(a), bd = make_sw128_desc(a + (uint32_t)(kWgBox * (1 + wg)));
      wg_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k)   // 16 positions (two 8-row swizzle atoms, 2048 bytes) per MMA
        wgmma_f16_mn64(acc, ad + 128 * k, bd + 128 * k, k > 0 ? 1u : 0u);
      wg_commit();
      wg_wait<0>();
      wg_fence_regs(acc);
#pragma unroll
      for (int r = 0; r < 32; ++r) sum[r] += acc[r];
    }
    __syncthreads();   // every warpgroup's MMAs that read stage s have completed
    if (threadIdx.x == 0 && i + P.stages < n) issue(i + P.stages, s);
  }

  // ---- epilogue: quadrants through shared memory, hi*hi + ((hi*lo + lo*hi) + lo*lo) -> fp32 partial tile ----
  // Thread (warp w, lane l) of a warpgroup holds rows 16 w + l / 4 (+8) and columns 8 i + 2 (l % 4) (+1) of its 64 x 64 tile;
  // rows 0-31 / 32-63 are the hi / lo parts of the input channels, columns likewise for the output channels.
  float* buf = reinterpret_cast<float*>(smem);   // [NWG][64][65]
  if (active) {
    float* t = buf + wg * 64 * 65;
    const int r0 = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      t[r0 * 65 + 8 * i + c0] = sum[4 * i];
      t[r0 * 65 + 8 * i + c0 + 1] = sum[4 * i + 1];
      t[(r0 + 8) * 65 + 8 * i + c0] = sum[4 * i + 2];
      t[(r0 + 8) * 65 + 8 * i + c0 + 1] = sum[4 * i + 3];
    }
  }
  __syncthreads();
  const int ld = P.ncb * 32;
  float* out = P.ws + (((size_t)z * taps + tap) * p.CB * 32 + cb * 32) * ld + j0 * 32;
  for (int idx = threadIdx.x; idx < nj * 1024; idx += blockDim.x) {
    const int jj = idx >> 10, ci = (idx >> 5) & 31, co = idx & 31;
    const float* t = buf + jj * 64 * 65;
    const float v = t[ci * 65 + co] + ((t[ci * 65 + co + 32] + t[(ci + 32) * 65 + co]) + t[(ci + 32) * 65 + co + 32]);
    out[(size_t)ci * ld + jj * 32 + co] = v;
  }
}

// Second pass: grad_w[tap][ci][g Cout + c] = (sum over splits, in split order) / S for the real channels only.
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float* __restrict__ ws, int splits, int taps, int CinP, int ld, int Cin,
                                                           int Cout, int G, int oc, const unsigned* __restrict__ absmax_bits,
                                                           float* __restrict__ grad_w) {
  const float inv = 1.0f / weight_pow2_scale(absmax_bits);   // a power of two: exact
  const long total = (long)taps * Cin * G * Cout;
  const size_t zstride = (size_t)taps * CinP * ld;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int col = (int)(i % (G * Cout));
    long r = i / (G * Cout);
    const int ci = (int)(r % Cin);
    const int tap = (int)(r / Cin);
    const int g = col / Cout, c = col - g * Cout;
    const float* src = ws + ((size_t)tap * CinP + ci) * ld + g * oc + c;
    float a = 0.f;
    for (int z = 0; z < splits; ++z) a += src[(size_t)z * zstride];
    grad_w[i] = a * inv;
  }
}

// ---- host side ----
struct WgPlan {
  TcParams g;
  int ncb, nwg, ngroups, m_tiles, splits, stages, G, oc;
};

// sm: the SM count the K split is planned for (the launch passes the device's; lt_conv_wgrad_plan any)
static int wgrad_plan(const lt_conv_desc* d, int sm, WgPlan* pl) {
  LT_REQUIRE(d->in_format == LT_FMT_S32 && d->out_format == LT_FMT_S32, "conv_wgrad: input and output gradient must be split-fp16");
  LT_REQUIRE(d->Cin % 32 == 0 && d->Cout % 32 == 0 && d->Cout > 0, "conv_wgrad: Cin=%d and Cout=%d must be multiples of 32", d->Cin, d->Cout);
  TcParams& p = pl->g;
  fill_params(d, p, d->Cin / 32, d->Cout, 32, 3, nullptr, nullptr, nullptr, nullptr);
  pl->G = p.n_maps;
  pl->oc = p.oc;
  LT_REQUIRE(p.n_maps <= kMaxOutMaps && d->Cout % p.n_maps == 0 && p.oc % 32 == 0 && p.oc == d->FC,
             "conv_wgrad: grouped output needs Cout / groups == FC, a multiple of 32");
  LT_REQUIRE(p.n_maps > 1 || d->FC == d->Cout, "conv_wgrad: FC=%d must equal Cout=%d", d->FC, d->Cout);
  pl->ncb = d->Cout / 32;
  pl->nwg = pl->ncb >= 3 ? 4 : pl->ncb;
  pl->ngroups = ceil_div(pl->ncb, pl->nwg);
  pl->m_tiles = p.tw * p.th * p.td * p.tn;
  // K split: the count (at most one per 16 M tiles) whose CTAs fill the SMs' waves best; ties go to the smaller count
  const long base = (long)d->KD * d->KH * d->KW * p.CB * pl->ngroups;
  int best = 1;
  double best_eff = 0.0;
  const int smax = pl->m_tiles / 16 > 1 ? pl->m_tiles / 16 : 1;
  for (int s = 1; s <= smax && base * s <= 16L * sm; ++s) {
    const long ctas = base * s;
    const double eff = (double)ctas / ((double)((ctas + sm - 1) / sm) * sm);
    if (eff > best_eff + 1e-3) { best_eff = eff; best = s; }
  }
  pl->splits = best;
  // TMA ring: as many M tiles (one input box + one output-gradient box per warpgroup) as fit 200 KiB, at most 6
  pl->stages = (200 * 1024) / (kWgBox * (1 + pl->nwg));
  if (pl->stages > 6) pl->stages = 6;
  return LT_OK;
}

static int device_sms() { return sm_count() > 0 ? sm_count() : 132; }

static size_t wgrad_ws_bytes(const lt_conv_desc* d, const WgPlan& pl) {
  return (size_t)pl.splits * d->KD * d->KH * d->KW * d->Cin * d->Cout * sizeof(float);
}

template <int NWG>
static int launch_wgrad(const CUtensorMap& tmIn, const TcEpiMaps& tmG, const WgParams& P, unsigned grid, cudaStream_t st) {
  constexpr int kStage = kWgBox * (1 + NWG);
  const size_t smem = (size_t)P.stages * kStage + P.stages * 8 + 1024;
  static DeviceOnce configured;
  if (configured.first()) {
    cudaError_t e = cudaFuncSetAttribute(conv_wgrad_kernel<NWG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e != cudaSuccess) return fail(LT_ERR_CUDA, "conv_wgrad: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  }
  conv_wgrad_kernel<NWG><<<grid, 128 * NWG, smem, st>>>(tmIn, tmG, P);
  LT_CHECK_LAUNCH("conv_wgrad_kernel");
  return LT_OK;
}

}  // namespace lt

using namespace lt;

extern "C" size_t lt_conv_wgrad_workspace_bytes(const lt_conv_desc* d) {
  WgPlan pl;
  if (!d || wgrad_plan(d, device_sms(), &pl) != LT_OK) return 0;
  return wgrad_ws_bytes(d, pl);
}

extern "C" int lt_conv_wgrad_plan(const lt_conv_desc* d, int sm_count, lt_conv_wgrad_launch_plan* plan) {
  LT_REQUIRE(d && plan && sm_count > 0, "conv_wgrad_plan: bad arguments");
  WgPlan pl;
  const int rc = wgrad_plan(d, sm_count, &pl);
  if (rc) return rc;
  plan->nwg = pl.nwg;
  plan->ngroups = pl.ngroups;
  plan->m_tiles = pl.m_tiles;
  plan->splits = pl.splits;
  plan->stages = pl.stages;
  return LT_OK;
}

extern "C" int lt_conv_wgrad_fwd(const lt_conv_desc* d, const void* in, const void* grad_out, const unsigned int* grad_absmax_bits,
                                 int Cin, int Cout, float* grad_w, void* workspace, size_t workspace_bytes, void* stream) {
  LT_REQUIRE(d && in && grad_out && grad_w && workspace, "conv_wgrad: null pointer");
  WgPlan pl;
  int rc = wgrad_plan(d, device_sms(), &pl);
  if (rc) return rc;
  LT_REQUIRE(Cin > 0 && Cin <= d->Cin && Cout > 0 && Cout <= pl.oc, "conv_wgrad: real channel counts Cin=%d Cout=%d exceed the padded %d / %d",
             Cin, Cout, d->Cin, pl.oc);
  LT_REQUIRE(workspace_bytes >= wgrad_ws_bytes(d, pl), "conv_wgrad: workspace of %zu bytes, %zu needed", workspace_bytes,
             wgrad_ws_bytes(d, pl));
  WgParams P;
  P.g = pl.g;
  P.ncb = pl.ncb;
  P.ngroups = pl.ngroups;
  P.m_tiles = pl.m_tiles;
  P.splits = pl.splits;
  P.ws = reinterpret_cast<float*>(workspace);
  P.stages = pl.stages;
  CUtensorMap tmIn;
  rc = make_in_map(&tmIn, d, P.g.bw, P.g.bh, P.g.bd, P.g.bn, in);
  if (rc) return rc;
  // output-gradient maps: the forward's epilogue maps (one per output group) over split-fp16 rows, 32-channel boxes
  TcEpiMaps tmG;
  memset(&tmG, 0, sizeof(tmG));
  {
    const TcParams& p = P.g;
    const uint64_t rowb = (uint64_t)p.FC * 4;
    const uint64_t dims[5] = {(uint64_t)(2 * p.FC), (uint64_t)p.OW, (uint64_t)p.OH, (uint64_t)p.OD, (uint64_t)p.N};
    const uint64_t str[4] = {rowb * p.osw, rowb * p.FW * p.osh, rowb * p.FW * p.FH * p.osd, rowb * p.FW * p.FH * p.FD};
    const uint32_t bx[5] = {64u, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bd, (uint32_t)p.bn};
    for (int g = 0; g < p.n_maps; ++g) {
      const long pix0 = ((long)(p.ood + g / (p.gh * p.gw)) * p.FH + p.ooh + (g / p.gw) % p.gh) * p.FW + p.oow + g % p.gw;
      rc = make_map(&tmG.out[g], static_cast<const uint8_t*>(grad_out) + pix0 * rowb, 5, dims, str, bx, nullptr, 1, 0);
      if (rc) return rc;
    }
  }
  const int taps = d->KD * d->KH * d->KW;
  const unsigned grid = (unsigned)((long)taps * P.g.CB * P.ngroups * P.splits);
  const cudaStream_t st = (cudaStream_t)stream;
  switch (pl.nwg) {
    case 1: rc = launch_wgrad<1>(tmIn, tmG, P, grid, st); break;
    case 2: rc = launch_wgrad<2>(tmIn, tmG, P, grid, st); break;
    default: rc = launch_wgrad<4>(tmIn, tmG, P, grid, st); break;
  }
  if (rc) return rc;
  const long total = (long)taps * Cin * pl.G * Cout;
  long blocks = (total + 255) / 256;
  if (blocks > 4L * sm_count()) blocks = 4L * sm_count();
  if (blocks < 1) blocks = 1;
  wgrad_reduce_kernel<<<(unsigned)blocks, 256, 0, st>>>(P.ws, P.splits, taps, d->Cin, d->Cout, Cin, Cout, pl.G, pl.oc, grad_absmax_bits,
                                                       grad_w);
  LT_CHECK_LAUNCH("wgrad_reduce_kernel");
  return LT_OK;
}

// CPU test hook: the kernel's index mapping (wgrad_boxes / wgrad_col_block / wgrad_in_row / wgrad_out_row) over plain float32
// channels-last tensors, summed in double: in [N][ID][IH][IW][desc->Cin], grad_out [N][FD][FH][FW][FC] -> grad_w [taps][Cin][G Cout].
extern "C" int lt_test_conv_wgrad_host(const lt_conv_desc* d, const float* in, const float* grad_out, int Cin, int Cout, float* grad_w) {
  LT_REQUIRE(d && in && grad_out && grad_w, "test_conv_wgrad_host: null pointer");
  WgPlan pl;
  int rc = wgrad_plan(d, device_sms(), &pl);
  if (rc) return rc;
  LT_REQUIRE(Cin > 0 && Cin <= d->Cin && Cout > 0 && Cout <= pl.oc, "test_conv_wgrad_host: bad channel counts");
  const TcParams& p = pl.g;
  const int taps = d->KD * d->KH * d->KW, ncol = pl.G * Cout;
  double* acc = new double[(size_t)taps * Cin * ncol]();
  for (int tap = 0; tap < taps; ++tap)
    for (int m = 0; m < pl.m_tiles; ++m) {
      const WgBoxes b = wgrad_boxes(p, m, tap);
      for (int r = 0; r < 128; ++r) {
        long ipix;
        if (!wgrad_in_row(p, b, r, d->ID, d->IH, d->IW, ipix)) continue;
        const float* x = in + ipix * d->Cin;
        for (int j = 0; j < pl.ncb; ++j) {
          int g, c0;
          wgrad_col_block(p, j, g, c0);
          long opix;
          if (!wgrad_out_row(p, b, r, g, opix)) continue;
          const float* dy = grad_out + opix * d->FC + c0;
          for (int ci = 0; ci < Cin; ++ci) {
            double* a = acc + ((size_t)tap * Cin + ci) * ncol + g * Cout;
            for (int c = 0; c < 32 && c0 + c < Cout; ++c) a[c0 + c] += (double)x[ci] * (double)dy[c];
          }
        }
      }
    }
  for (size_t i = 0; i < (size_t)taps * Cin * ncol; ++i) grad_w[i] = (float)acc[i];
  delete[] acc;
  return LT_OK;
}
