// wgmma convolutions for the full-resolution V2V layers (LT_CONV_TC_FOLD): Cin = 32, cubic K = 3 or 7, stride 1, "same" padding,
// Cout <= 32.  Same split-fp16 products and epilogue arithmetic as conv_tc_kernel (conv_tc.cu), different operand staging.  Both
// kernels take the A operand from registers (wgmma RS), loaded with ldmatrix from 128B-swizzled TMA boxes (chunk j of box row R
// sits at j ^ (R % 8), every box starting on a 1024-byte boundary), so an m64 block may start at any box row.
//
// conv_lines_kernel (K = 3, 16 <= W <= 64): kw is part of the GEMM's N instead of its K.  For a stride-1 "same" 3^3 conv
//   out[w] = sum_kw P_kw[w + kw - 1],   P_kw[w] = sum_{kd, kh, ci} x[d + kd - 1, h + kh - 1, w, ci] W[kd, kh, kw, ci, :],
// so per (kd, kh) a warpgroup issues six m64 x (3 NC) x k16 products (N = 96 for Cout 32) whose A is the input line itself: read
// once per (kd, kh) instead of once per (kd, kh, kw), with no W halo (the zero padding along W is the line end).  An m64 block is
// LPB = floor(64 / W) whole W lines stacked (spare rows masked); a CTA owns 2 LPB adjacent h lines, LPB per consumer warpgroup,
// and walks along d.  Each input plane arrives as one TMA box of 2 LPB + 2 lines x W positions in a ring of three planes, consumed
// kd = 0, 1, 2, so the oldest plane is released after the first third of an output plane and the next needs one new box.  The
// whole packed filter stays resident.  The epilogue forms v_kw = D1 + D2 / S per row and out[w] = v_0[w - 1] + v_1[w] + v_2[w + 1]
// in fp32 (zero past the line ends): rows w +- 1 sit in lanes +- 4 or the thread's other accumulator half, and only the first and
// last row of each warp cross to the neighbour warp, through shared memory.  The epilogue is staged: the TMA loads each warpgroup's
// residual rows into its 8 KB slab while the products run, the output rows are written over them and leave by one TMA store,
// which the warpgroup does not wait for (the slab is released after the next plane's first products are issued).  Work: the (n, h block, d) output planes in order, cut into one contiguous range per CTA (one
// CTA per SM), so every SM computes the same number of planes to within one.  3^3 layers with W > 64 run on conv_tc_kernel.
//
// conv_fold_kernel (K = 7): tile 8 (w) x 16 (h) x BD = 64 / NC (d) outputs; consumer warpgroup g owns the 8-line h half g in all
// BD output planes (m64 rows = whole 8-wide W lines at 8 consecutive h).  An A stage holds ONE input plane's halo box
//   {64 channels, 8 + 6 (w), 16 + 6 (h), 1 (d)}
// that serves every kw and kh of every output plane that reads it: the BD + 6 input planes of a tile are each loaded once.  TMA
// zero fill supplies the padding.  Each warp owns 16 rows, i.e. the W lines 2 w' and 2 w' + 1 of its h half (w' = warp in the
// warpgroup): the kw shift is a one-row offset, and along kh the fragments of the second line are the first line of the next tap,
// so each kh step loads one new line per warp.  The output planes share these A fragments, so one m64 x 64 wgmma per K slice
// computes all of them: N = the BD planes' NC columns, B = the taps kd = plane - b of one (kw, kh), one B stage per (plane, kw)
// read as [kh][kd][NC] from the [kw][kd][kh] packing, zero-filled where kd falls outside the filter.  Every output still sees its
// products in (kd, kw, kh) order.
//
// Weights: lt_conv_fold_pack_weights, rows of [32 hi | 32 lo] fp16, NC = round_up(Cout, 16) rows per tap: 3^3 as
// [kd][kh][kw][NC] (a (kd, kh) slice is the 3 NC-row B operand of the kw-wide products), 7^3 as [kw][kd][kh][NC] (a (kd, kw) slice
// is 7 consecutive taps).  The N tile is NC: the 7^3 layer (Cout 16) multiplies no padding; output channels NC .. FC-1 go through
// the same epilogue with zero accumulators (scale 0, shift 0 for the padding channels: written as zeros).
//
// Per 16-wide K slice hi*hi accumulates into D1 and hi*lo + lo*hi into D2, as in conv_tc_kernel: D1 takes 9 Cin / 16 (3^3: one
// column per kw) or K^3 Cin / 16 (7^3) accumulation steps per output (the accum_steps of the folded scale: ConvPack.scale_fold,
// engine.pack_filter).
//
// Persistent grids: one CTA per SM; the producer warp runs its rings across tile (piece) boundaries.  An A stage is released as
// soon as the consumers' ldmatrix reads of it have completed; a weight slice once the MMAs reading it have.
#include "tc_common.cuh"
#include "conv_tc_params.cuh"

namespace lt {

constexpr int kFoldThreads = 384;
constexpr int kFoldSmem = 227 * 1024;

// ------------------------------------------------------------------------------------------------------------------------------
// 3^3: conv_lines_kernel
// ------------------------------------------------------------------------------------------------------------------------------
template <int NC>
struct LinesCfg {
  static constexpr int N = 3 * NC;                    // (kw, Cout) columns of one product
  static constexpr int SLICE = N * 128;               // one (kd, kh) B operand
  static constexpr int B_BYTES = 9 * SLICE;           // the whole filter, resident
  static constexpr int PLANE = 32 * 1024;             // ring slot: (2 LPB + 2) lines x W rows x 128 B <= 32 KB for 16 <= W <= 64
  static constexpr int RING = 3;
  static constexpr int XCH = 2 * 2 * 4 * 2 * 4 * (NC / 4) * 4;   // [plane parity][warpgroup][warp][v0 row 15 | v2 row 0][4 lanes][NC/4]
  static constexpr int SLAB = 8 * 1024;               // one warpgroup's residual / output rows: LPB lines x W x 128 B <= 8 KB
  static constexpr int A_OFF = B_BYTES;
  static constexpr int S_OFF = A_OFF + RING * PLANE;
  static constexpr int X_OFF = S_OFF + 2 * SLAB;
  static constexpr int BAR_OFF = X_OFF + XCH;
  static constexpr size_t SMEM = (size_t)BAR_OFF + 128 + 1024;
  static_assert(SLICE % 1024 == 0 && B_BYTES % 1024 == 0, "B slices must start on 1024-byte swizzle atoms");
  static_assert(SMEM <= (size_t)kFoldSmem, "shared memory");
};

// Walk the output planes [q0, q1) of the (n, h block, d) order in pieces of consecutive d of one (n, h block) column.
struct LinesPiece {
  int n, h0, dA, dB;
};
__device__ __forceinline__ bool lines_next_piece(const TcParams& p, long& q, long q1, LinesPiece& pc) {
  if (q >= q1) return false;
  const long col = q / p.OD;
  pc.dA = (int)(q - col * p.OD);
  pc.dB = (int)((q1 - q) < (long)(p.OD - pc.dA) ? pc.dA + (q1 - q) : p.OD);
  pc.h0 = (int)(col % p.th) * p.bh;
  pc.n = (int)(col / p.th);
  q += pc.dB - pc.dA;
  return true;
}

// Staged epilogue of output channels co, co + 1 of slab row `row` (128 bytes, 128B-swizzled: 32 float32 or 32 hi | 32 lo fp16):
// conv_epilogue_row's arithmetic, the residual read from the row and the output written over it.
// scale / shift: loaded where they are used (volatile), not hoisted out of the plane loop beside the accumulators
__device__ __forceinline__ float2 ldg_f2_here(const float* a) {
  float2 v;
  asm volatile("ld.global.nc.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(a));
  return v;
}
__device__ __forceinline__ void lines_epilogue_pair(const TcParams& p, uint32_t slab, int row, int co, float v0, float v1) {
  const float2 sc = ldg_f2_here(p.scale + co);
  const float2 sh = ldg_f2_here(p.shift + co);
  v0 = fmaf(v0, sc.x, sh.x);
  v1 = fmaf(v1, sc.y, sh.y);
  const uint32_t rb = slab + (uint32_t)row * 128u, sw = (uint32_t)row & 7u;
  if (p.out_format == LT_FMT_F32) {
    const uint32_t a = rb + (((((uint32_t)co >> 2) ^ sw)) << 4) + ((uint32_t)co & 3u) * 4u;
    const float2 r = p.residual == LT_RES_NONE ? make_float2(0.f, 0.f) : lds_f2(a);
    if (p.residual == LT_RES_BEFORE_RELU) { v0 += r.x; v1 += r.y; }
    if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
    if (p.residual == LT_RES_AFTER_RELU) { v0 += r.x; v1 += r.y; }
    sts_f2(a, make_float2(v0, v1));
  } else {
    const uint32_t ah = rb + ((((uint32_t)co >> 3) ^ sw) << 4) + ((uint32_t)co & 7u) * 2u;
    const uint32_t al = rb + (((((uint32_t)co >> 3) + 4u) ^ sw) << 4) + ((uint32_t)co & 7u) * 2u;
    float2 r = make_float2(0.f, 0.f);
    if (p.residual != LT_RES_NONE) {
      const uint32_t hi = lds32(ah), lo = lds32(al);
      const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&hi));
      const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&lo));
      r = make_float2(fmaf(b.x, kLoInv, a.x), fmaf(b.y, kLoInv, a.y));
    }
    if (p.residual == LT_RES_BEFORE_RELU) { v0 += r.x; v1 += r.y; }
    if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
    if (p.residual == LT_RES_AFTER_RELU) { v0 += r.x; v1 += r.y; }
    uint32_t hi2, lo2;
    split_s32x2(v0, v1, hi2, lo2);
    sts32(ah, hi2);
    sts32(al, lo2);
  }
}

// p.bw = W, p.bh = 2 LPB output lines per CTA, p.th = h blocks.  tmO / tmR: the output / residual, boxes of LPB lines (one
// warpgroup's m64 block), 128B-swizzled 128-byte rows
template <int NC>
__global__ void __launch_bounds__(kFoldThreads, 1) conv_lines_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                     const __grid_constant__ CUtensorMap tmB,
                                                                     const __grid_constant__ CUtensorMap tmO,
                                                                     const __grid_constant__ CUtensorMap tmR, const TcParams p) {
  using C = LinesCfg<NC>;
  constexpr int NR = C::N / 2;     // accumulator registers per thread
  constexpr int NI = NC / 8;       // 8-column groups per kw
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* bsm = smem;
  uint8_t* asm_ = smem + C::A_OFF;
  uint8_t* ssm = smem + C::S_OFF;
  float* xch = reinterpret_cast<float*>(smem + C::X_OFF);
  uint64_t* afull = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);
  uint64_t* aempty = afull + C::RING;
  uint64_t* bfull = aempty + C::RING;
  uint64_t* rfull = bfull + 1;     // [warpgroup]: the residual rows of its next output plane are in its slab
  uint64_t* rempty = rfull + 2;    // [warpgroup]: the TMA store of its previous output plane has read the slab

  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int lane = threadIdx.x & 31;
  const int W = p.bw, LPB = p.bh / 2;
  const long total = (long)p.N * p.th * p.OD;
  const long q0 = (long)blockIdx.x * total / gridDim.x, q1 = (long)(blockIdx.x + 1) * total / gridDim.x;

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::RING; ++s) { mbar_init(&afull[s], 1); mbar_init(&aempty[s], 256); }
    mbar_init(&bfull[0], 1);
    for (int s = 0; s < 2; ++s) { mbar_init(&rfull[s], 1); mbar_init(&rempty[s], 1); }
    fence_barrier_init();
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    prefetch_tmap(&tmO);
    if (p.residual != LT_RES_NONE) prefetch_tmap(&tmR);
  }
  __syncthreads();

  if (wg == 0) {
    // ================= TMA producer (warp 0; one elected lane issues) =================
    regs_release_producer();
    if (threadIdx.x < 32) {
      if (elect_one()) {
        mbar_expect_tx(&bfull[0], (uint32_t)C::B_BYTES);
        tma_load_3d(bsm, &tmB, &bfull[0], 0, 0, 0);
      }
      const uint32_t box_bytes = (uint32_t)((p.bh + 2) * W * 128), res_bytes = (uint32_t)(LPB * W * 128);
      int s = 0;
      uint32_t ph = 0, rph = 0;
      long q = q0;
      LinesPiece pc;
      while (lines_next_piece(p, q, q1, pc)) {
        for (int dd = pc.dA - 1; dd <= pc.dB; ++dd) {
          mbar_wait(&aempty[s], ph ^ 1u);
          if (elect_one()) {
            mbar_expect_tx(&afull[s], box_bytes);
            tma_load_5d(asm_ + (size_t)s * C::PLANE, &tmA, &afull[s], 0, 0, pc.h0 - 1, dd, pc.n);
          }
          __syncwarp();
          if (++s == C::RING) { s = 0; ph ^= 1u; }
          if (dd > pc.dA) {   // every input plane of output plane dd - 1 is on its way: its residual rows next
            for (int r = 0; r < 2; ++r) {
              mbar_wait(&rempty[r], rph ^ 1u);
              if (elect_one()) {
                if (p.residual != LT_RES_NONE) {
                  mbar_expect_tx(&rfull[r], res_bytes);
                  tma_load_5d(ssm + (size_t)r * C::SLAB, &tmR, &rfull[r], 0, 0, pc.h0 + r * LPB, dd - 1, pc.n);
                } else {
                  mbar_arrive_local(&rfull[r]);
                }
              }
              __syncwarp();
            }
            rph ^= 1u;
          }
        }
      }
    }
    return;
  }

  // ================= MMA + epilogue (warpgroups 1, 2) =================
  regs_claim_consumer();
  const int g = wg - 1, warp = (threadIdx.x >> 5) & 3;
  // this lane's ldmatrix row: matrix m = lane / 8 covers rows 8 (m % 2) .. +7 of the warp's 16 and chunk 2 s + m / 2 of K slice s
  int lrow = 16 * warp + 8 * ((lane >> 3) & 1) + (lane & 7);
  int lline = lrow / W;
  if (lline >= LPB) lline = LPB - 1;   // masked rows read a valid line; their results are never stored
  const uint32_t abase = (uint32_t)((g * LPB + lline) * W + lrow % W);   // box row of tap kh = 0
  const uint32_t cbit = (uint32_t)(lane >> 4);
  // this thread's accumulator rows r_lo + 8 h: line and position in the line
  const int r_lo = warp * 16 + (lane >> 2);
  const int c2 = 2 * (lane & 3);
  const uint32_t bsm0 = smem_u32(bsm), asm0 = smem_u32(asm_);
  const uint32_t slab = smem_u32(ssm) + (uint32_t)(g * C::SLAB);
  const bool wg_lead = (threadIdx.x & 127) == 0;
  const uint32_t bar_id = 1u + (uint32_t)g;
  mbar_wait(&bfull[0], 0);

  float d1[NR], d2[NR];
  uint32_t a[2][4][4];
  int seq = 0;   // plane loads of this CTA so far (the producer's order)
  uint32_t xpar = 0;   // parity of this CTA's output planes so far
  long q = q0;
  LinesPiece pc;
  while (lines_next_piece(p, q, q1, pc)) {
    const int P = pc.dB - pc.dA;
    for (int j = 0; j < P; ++j) {
      const int od = pc.dA + j;
      auto plane = [&](int kd) -> uint32_t {
        const int pq = seq + j + kd;
        const int sl = (int)(pq % C::RING);
        mbar_wait(&afull[sl], (uint32_t)(pq / C::RING) & 1u);
        return asm0 + (uint32_t)(sl * C::PLANE);
      };
      auto release = [&](int kd) {   // this thread's ldmatrix reads of plane kd have completed
        if (kd == 0 || j == P - 1) mbar_arrive_local(&aempty[(int)((seq + j + kd) % C::RING)]);
      };
      auto load = [&](uint32_t box, int kh, uint32_t (&f)[4][4]) {
        const uint32_t row = abase + (uint32_t)(kh * W), sw = row & 7u;
        const uint32_t ra = box + row * 128u;
#pragma unroll
        for (int s = 0; s < 4; ++s) ldmatrix_x4(f[s], ra + (((2u * s + cbit) ^ sw) << 4));
      };
      uint32_t box = plane(0);
      load(box, 0, a[0]);
#pragma unroll
      for (int st = 0; st < 9; ++st) {
        const int kd = st / 3;
        const uint64_t bd = make_sw128_desc(bsm0 + (uint32_t)(st * C::SLICE));
        const uint32_t acc = st == 0 ? 0u : 1u;
        uint32_t (&f)[4][4] = a[st & 1];
        wg_fence();
        wgmma_f16_rs<C::N>(d1, f[0], bd, acc);        // hi * hi
        wgmma_f16_rs<C::N>(d1, f[1], bd + 2, 1u);
        wgmma_f16_rs<C::N>(d2, f[0], bd + 4, acc);    // hi * lo
        wgmma_f16_rs<C::N>(d2, f[1], bd + 6, 1u);
        wgmma_f16_rs<C::N>(d2, f[2], bd, 1u);         // lo * hi
        wgmma_f16_rs<C::N>(d2, f[3], bd + 2, 1u);
        wg_commit();
        if (st == 0 && (seq > 0 || j > 0) && wg_lead) {   // free the slab for this plane's residual once the previous store has read it
          bulk_wait_read0();
          mbar_arrive_local(&rempty[g]);
        }
        wg_wait<1>();   // the products of step st - 1 have completed: its A registers may be reloaded
        if (st + 1 < 9) {
          if ((st + 1) % 3 == 0) {
            release(kd);
            box = plane(kd + 1);
          }
          load(box, (st + 1) % 3, a[(st + 1) & 1]);
        }
      }
      release(2);
      wg_wait<0>();
      wg_fence_regs(d1);
      wg_fence_regs(d2);

      // ---- epilogue: v_kw = D1 + D2 / S, out[w] = v_0[w - 1] + v_1[w] + v_2[w + 1] ----
      auto v = [&](int kw, int h, int i, int e) {
        const int k = 4 * (kw * NI + i) + 2 * h + e;
        return fmaf(d2[k], kLoInv, d1[k]);
      };
      // rows 16 w - 1 (v_0 of the previous warp's row 15) and 16 w + 16 (v_2 of the next warp's row 0) through shared memory
      float* xw = xch + (size_t)((xpar * 2 + g) * 4) * (2 * 4 * 2 * NI);
      if (lane >= 28) {
#pragma unroll
        for (int i = 0; i < NI; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e) xw[((warp * 2 + 0) * 4 + (lane - 28)) * 2 * NI + 2 * i + e] = v(0, 1, i, e);
      }
      if (lane < 4) {
#pragma unroll
        for (int i = 0; i < NI; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e) xw[((warp * 2 + 1) * 4 + lane) * 2 * NI + 2 * i + e] = v(2, 0, i, e);
      }
      asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
      xpar ^= 1u;
      // the output rows replace the residual rows in the slab; one TMA store per warpgroup (rows past OH are clipped)
      mbar_wait(&rfull[g], xpar ^ 1u);
      int rl[2], rw[2];   // line and position of this thread's rows r_lo + 8 h
#pragma unroll
      for (int h = 0; h < 2; ++h) { rl[h] = (r_lo + 8 * h) / W; rw[h] = (r_lo + 8 * h) % W; }
#pragma unroll
      for (int i = 0; i < NI; ++i) {
        float o[2][2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float t0 = __shfl_sync(0xffffffffu, v(0, 0, i, e), (lane + 28) & 31);
          const float t1 = __shfl_sync(0xffffffffu, v(0, 1, i, e), (lane + 28) & 31);
          const float u0 = __shfl_sync(0xffffffffu, v(2, 0, i, e), (lane + 4) & 31);
          const float u1 = __shfl_sync(0xffffffffu, v(2, 1, i, e), (lane + 4) & 31);
          float prev0 = t0, prev1 = t1, next0 = u0, next1 = u1;
          if (lane < 4) {
            prev1 = t0;
            prev0 = warp > 0 ? xw[(((warp - 1) * 2 + 0) * 4 + lane) * 2 * NI + 2 * i + e] : 0.f;
          }
          if (lane >= 28) {
            next0 = u1;
            next1 = warp < 3 ? xw[(((warp + 1) * 2 + 1) * 4 + (lane - 28)) * 2 * NI + 2 * i + e] : 0.f;
          }
          const float pv[2] = {prev0, prev1}, nx[2] = {next0, next1};
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float sum = (rw[h] > 0 ? pv[h] : 0.f) + v(1, h, i, e);
            sum += rw[h] < W - 1 ? nx[h] : 0.f;
            o[h][e] = sum;
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (rl[h] < LPB) lines_epilogue_pair(p, slab, r_lo + 8 * h, 8 * i + c2, o[h][0], o[h][1]);
      }
#pragma unroll
      for (int i = NI; i < 4; ++i)   // output channels NC .. 31 (Cout 16): zero accumulators, scale 0, shift 0
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (rl[h] < LPB) lines_epilogue_pair(p, slab, r_lo + 8 * h, 8 * i + c2, 0.f, 0.f);
      fence_proxy_async();
      asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
      if (wg_lead) {
        tma_store_5d(&tmO, ssm + (size_t)g * C::SLAB, 0, 0, pc.h0 + g * LPB, od, pc.n);
        bulk_commit();
      }
    }
    seq += P + 2;
  }
  if (wg_lead) bulk_wait0();
}

template <int NC>
static int conv_lines_run(const lt_conv_desc* d, const void* in, const void* weight, const float* scale, const float* shift,
                          const void* residual, void* out, cudaStream_t st) {
  using C = LinesCfg<NC>;
  TcParams p;
  fill_params(d, p, 1, NC, NC, 1, scale, shift, residual, out);
  LT_REQUIRE((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(residual)) % 16 == 0,
             "conv_fold: out and residual must be 16-byte aligned (TMA global addresses)");
  const int lpb = 64 / d->OW;
  p.bw = d->OW; p.bh = 2 * lpb; p.bd = 1; p.bn = 1;
  p.tw = 1; p.th = ceil_div(d->OH, p.bh); p.td = d->OD; p.tn = d->N;
  p.stages = C::RING;
  CUtensorMap tmA, tmB;
  int rc = make_in_map(&tmA, d, p.bw, p.bh + 2, 1, 1, in);
  if (rc) return rc;
  const uint64_t dims[3] = {64, (uint64_t)C::N, 9};
  const uint64_t str[2] = {128, (uint64_t)C::SLICE};
  const uint32_t bx[3] = {64, (uint32_t)C::N, 9};
  rc = make_map(&tmB, weight, 3, dims, str, bx, nullptr, 1);
  if (rc) return rc;
  // output / residual: 128-byte rows (32 float32 or 32 hi | 32 lo fp16), boxes of one warpgroup's LPB lines
  CUtensorMap tmO, tmR;
  const int f32 = d->out_format == LT_FMT_F32;
  const uint64_t odims[5] = {(uint64_t)(f32 ? 32 : 64), (uint64_t)d->OW, (uint64_t)d->OH, (uint64_t)d->OD, (uint64_t)d->N};
  const uint64_t ostr[4] = {128, 128ull * d->OW, 128ull * d->OW * d->OH, 128ull * d->OW * d->OH * d->OD};
  const uint32_t obx[5] = {(uint32_t)(f32 ? 32 : 64), (uint32_t)d->OW, (uint32_t)(p.bh / 2), 1, 1};
  rc = make_map(&tmO, out, 5, odims, ostr, obx, nullptr, 1, f32);
  if (rc) return rc;
  rc = make_map(&tmR, residual ? residual : out, 5, odims, ostr, obx, nullptr, 1, f32);
  if (rc) return rc;
  static DeviceOnce configured;
  if (configured.first()) {
    cudaError_t e = cudaFuncSetAttribute(conv_lines_kernel<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFoldSmem);
    if (e != cudaSuccess) return fail(LT_ERR_CUDA, "conv_lines: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  }
  const long planes = (long)p.N * p.th * p.OD;
  const int grid = (int)(planes < sm_count() ? planes : sm_count());
  conv_lines_kernel<NC><<<grid, kFoldThreads, C::SMEM, st>>>(tmA, tmB, tmO, tmR, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(LT_ERR_CUDA, "conv_lines_kernel: %s", cudaGetErrorString(e));
  return LT_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------
// 7^3: conv_fold_kernel
// ------------------------------------------------------------------------------------------------------------------------------
template <int K, int NC>
struct FoldCfg {
  static_assert(K == 7, "the 3^3 layers run on conv_lines_kernel");
  static constexpr int BW = 8, BH = 16;
  static constexpr int BD = 64 / NC;                   // output planes per tile: N = BD NC = 64 per wgmma
  static constexpr int WBOX = BW + K - 1, HBOX = BH + K - 1;
  static constexpr int A_BYTES = WBOX * HBOX * 128;    // one input plane's halo box
  static constexpr int A_STAGE = (A_BYTES + 1023) / 1024 * 1024;
  static constexpr int TAP = NC * 128;                 // one packed weight tap
  static constexpr int B_KH = BD * TAP;                // one kh of a B stage: the taps of BD consecutive kd, the wide B operand
  static constexpr int B_STAGE = K * B_KH;             // one (plane, kw) step: [kh][kd][NC]
  static constexpr int AVAIL = kFoldSmem - 1024 - 256;
  static constexpr int ARING = 2;
  static constexpr int BRING = (AVAIL - ARING * A_STAGE) / B_STAGE;
  static constexpr int A_OFF = BRING * B_STAGE;
  static constexpr int BAR_OFF = A_OFF + ARING * A_STAGE;
  static constexpr size_t SMEM = (size_t)BAR_OFF + 256 + 1024;
  static_assert(BD * NC == 64 && BH == 16, "one 8-line h half of BD planes per consumer warpgroup, N <= 64 per wgmma");
  static_assert(B_KH % 1024 == 0, "B operands must start on 1024-byte swizzle atoms");
  static_assert(BRING >= 2 && 2 * (ARING + BRING) * 8 <= 256 && SMEM <= (size_t)kFoldSmem, "shared memory");
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

// The products of one input plane for every output block of the tile, kw by kw.  The blocks share their A fragments, so one
// m64 x (BD NC) wgmma per K slice serves all of them: its B operand is the taps kd = pl - BD + 1 .. pl of one (kw, kh), adjacent
// in the B stage (zero where kd is outside 0 .. K - 1, so a block only ever adds its own taps), and its accumulator columns are
// the blocks' accumulators, stored in descending block order (slot BD - 1 - b) so that kd ascends with the column.  Each kh step
// loads one new W line per warp.  The B stage of the previous (plane, kw) step is released once its MMAs have completed.
template <int K, int NC>
__device__ __forceinline__ void fold_plane(float (&d1)[FoldCfg<K, NC>::BD * NC / 2], float (&d2)[FoldCfg<K, NC>::BD * NC / 2],
                                           uint32_t box, uint32_t row0, uint32_t mlane, uint32_t bsm0, uint64_t* bfull, uint64_t* bempty,
                                           int& nbs, int& held, bool wg_lead) {
  using C = FoldCfg<K, NC>;
#pragma unroll 1
  for (int kw = 0; kw < K; ++kw, ++nbs) {
    const int sb = nbs % C::BRING;
    mbar_wait(&bfull[sb], (uint32_t)(nbs / C::BRING) & 1u);
    const uint32_t bstage = bsm0 + (uint32_t)(sb * C::B_STAGE);
    uint32_t ln[K + 1][2][4];
    fold_load_line(ln[0], box, row0 + kw, mlane);
#pragma unroll
    for (int kh = 0; kh < K; ++kh) {
      fold_load_line(ln[kh + 1], box, row0 + kw + (uint32_t)((kh + 1) * C::WBOX), mlane);
      wg_fence();
      fold_tap<C::BD * NC>(d1, d2, ln[kh], ln[kh + 1], make_sw128_desc(bstage + (uint32_t)(kh * C::B_KH)), 1u);
      wg_commit();
      wg_wait<1>();
      if (kh == 0 && held >= 0) {   // every MMA of the previous step has completed
        if (wg_lead) mbar_arrive_local(&bempty[held % C::BRING]);
        held = -1;
      }
    }
    held = nbs;
  }
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
    for (int s = 0; s < C::ARING; ++s) { mbar_init(&afull[s], 1); mbar_init(&aempty[s], 256); }
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
      int sa = 0, sb = 0;
      uint32_t pa = 0, pb = 0;
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        int ow0, oh0, od0, nb;
        fold_tile_origin(p, t, ow0, oh0, od0, nb);
        const int nvb = p.OD - od0 < C::BD ? p.OD - od0 : C::BD;
        for (int pl = 0; pl < nvb + K - 1; ++pl) {
          mbar_wait(&aempty[sa], pa ^ 1u);
          if (elect_one()) {
            mbar_expect_tx(&afull[sa], (uint32_t)C::A_BYTES);
            tma_load_5d(asm_ + (size_t)sa * C::A_STAGE, &tmA, &afull[sa], 0, ow0 - K / 2, oh0 - K / 2, od0 + pl - K / 2, nb);
          }
          __syncwarp();
          if (++sa == C::ARING) { sa = 0; pa ^= 1u; }
          for (int kw = 0; kw < K; ++kw) {   // taps kd = pl - BD + 1 .. pl of (kw, every kh); zero fill outside 0 .. K - 1
            mbar_wait(&bempty[sb], pb ^ 1u);
            if (elect_one()) {
              mbar_expect_tx(&bfull[sb], (uint32_t)C::B_STAGE);
              tma_load_5d(bsm + (size_t)sb * C::B_STAGE, &tmB, &bfull[sb], 0, 0, pl - C::BD + 1, 0, kw);
            }
            __syncwarp();
            if (++sb == C::BRING) { sb = 0; pb ^= 1u; }
          }
        }
      }
    }
    return;
  }

  // ================= MMA + epilogue (warpgroups 1, 2) =================
  // warpgroup g owns the 8-line h half g of the tile in all BD output planes (m64 block b = output plane od0 + b); each input
  // plane's box and weight slices are shared by both warpgroups
  regs_claim_consumer();
  const int g = wg - 1, warp = (threadIdx.x >> 5) & 3;
  float d1[C::BD * NC / 2], d2[C::BD * NC / 2];   // output block b: the NC / 2 registers of slot BD - 1 - b
  const uint32_t row0 = (uint32_t)((g * 8 + 2 * warp) * C::WBOX + (lane & 7));   // this lane's box row for kw = kh = 0
  const uint32_t mlane = (uint32_t)(lane >> 3);
  const int r_lo = warp * 16 + (lane >> 2);   // this thread's accumulator rows r_lo, r_lo + 8 of an m64 block
  const int c2 = 2 * (lane & 3);
  const uint32_t bsm0 = smem_u32(bsm), asm0 = smem_u32(asm_);
  const bool wg_lead = (threadIdx.x & 127) == 0;
  int na = 0, nbs = 0;   // input planes and B stages of this CTA so far (the producer's order)
  int held = -1;         // the B stage of the previous (plane, kw) step until its MMAs have completed
  for (int kt = 0;; ++kt) {
    const int t = blockIdx.x + kt * gridDim.x;
    if (t >= ntiles) break;
    int ow0, oh0, od0, nb;
    fold_tile_origin(p, t, ow0, oh0, od0, nb);
    const int nvb = p.OD - od0 < C::BD ? p.OD - od0 : C::BD;
#pragma unroll
    for (int i = 0; i < C::BD * NC / 2; ++i) { d1[i] = 0.f; d2[i] = 0.f; }   // the blocks of a tile start at different planes
#pragma unroll 1
    for (int pl = 0; pl < nvb + K - 1; ++pl, ++na) {
      const int sa = na % C::ARING;
      mbar_wait(&afull[sa], (uint32_t)(na / C::ARING) & 1u);
      const uint32_t box = asm0 + (uint32_t)(sa * C::A_STAGE);
      fold_plane<K, NC>(d1, d2, box, row0, mlane, bsm0, bfull, bempty, nbs, held, wg_lead);
      mbar_arrive_local(&aempty[sa]);   // this thread's ldmatrix reads of the box have completed
    }
    wg_wait<0>();
    if (wg_lead) mbar_arrive_local(&bempty[held % C::BRING]);
    held = -1;
    wg_fence_regs(d1);
    wg_fence_regs(d2);

    // ---- epilogue ----
#pragma unroll
    for (int b = 0; b < C::BD; ++b) {
      if (b >= nvb) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r_lo + 8 * h;
        const int ow = ow0 + (r & 7), oh = oh0 + g * 8 + (r >> 3), od = od0 + b;
        if (!(ow < p.OW && oh < p.OH)) continue;
        const long opix = (((long)nb * p.FD + od) * p.FH + oh) * p.FW + ow;
        const int slot = (C::BD - 1 - b) * (NC / 2);
        conv_epilogue_row<NC>(p, *reinterpret_cast<const float(*)[NC / 2]>(&d1[slot]), *reinterpret_cast<const float(*)[NC / 2]>(&d2[slot]),
                              h, opix, 0, c2);
        if constexpr (NC == 16) {   // output channels 16..31: no weights
          const float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          conv_epilogue_row<16>(p, z, z, h, opix, 16, c2);
        }
      }
    }
  }
}

template <int NC>
static int conv_fold_run(const lt_conv_desc* d, const void* in, const void* weight, const float* scale, const float* shift,
                         const void* residual, void* out, cudaStream_t st) {
  constexpr int K = 7;
  using C = FoldCfg<K, NC>;
  TcParams p;
  fill_params(d, p, 1, NC, NC, 3, scale, shift, residual, out);
  p.bw = C::BW; p.bh = C::BH; p.bd = C::BD; p.bn = 1;
  p.tw = ceil_div(d->OW, p.bw); p.th = ceil_div(d->OH, p.bh); p.td = ceil_div(d->OD, p.bd); p.tn = d->N;
  p.stages = C::ARING;
  CUtensorMap tmA, tmB;
  int rc = make_in_map(&tmA, d, C::WBOX, C::HBOX, 1, 1, in);
  if (rc) return rc;
  // packed [kw][kd][kh][NC] taps read as [kh][kd][NC] per kw: the BD kd of one kh are the N rows of one wide B operand
  const uint64_t dims[5] = {64, (uint64_t)NC, (uint64_t)K, (uint64_t)K, (uint64_t)K};
  const uint64_t str[4] = {128, (uint64_t)C::TAP * K, (uint64_t)C::TAP, (uint64_t)C::TAP * K * K};
  const uint32_t bx[5] = {64, (uint32_t)NC, (uint32_t)C::BD, (uint32_t)K, 1};
  rc = make_map(&tmB, weight, 5, dims, str, bx, nullptr, 1);
  if (rc) return rc;
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

// 3^3 layers are taken up to W = 64 (one W line per m64 block); wider ones run on conv_tc_kernel
int conv_fold_supported(const lt_conv_desc* d) {
  const bool cubic = d->KD == d->KH && d->KH == d->KW && (d->KW == 3 || d->KW == 7);
  const int pd = d->KW / 2;
  return cubic && d->Cin == 32 && d->Cout <= 32 && d->sd == 1 && d->sh == 1 && d->sw == 1 && d->pd == pd && d->ph == pd &&
         d->pw == pd && d->OD == d->ID && d->OH == d->IH && d->OW == d->IW && d->osd == 1 && d->osh == 1 && d->osw == 1 &&
         d->ood == 0 && d->ooh == 0 && d->oow == 0 && d->FD == d->OD && d->FH == d->OH && d->FW == d->OW && d->FC == 32 &&
         d->in_format == LT_FMT_S32 && d->IW >= 16 && (d->KW == 7 || d->IW <= 64);
}

// desc->Cout = real output channel count; weights from lt_conv_fold_pack_weights with the same K and Cout
int conv_fold_fwd(const lt_conv_desc* d, const void* in, const void* weight, const float* scale, const float* shift,
                  const void* residual, void* out, void* stream) {
  LT_REQUIRE(conv_fold_supported(d), "conv_fold: unsupported layer shape");
  const cudaStream_t st = (cudaStream_t)stream;
  const bool narrow = d->Cout <= 16;
  if (d->KW == 3)
    return narrow ? conv_lines_run<16>(d, in, weight, scale, shift, residual, out, st)
                  : conv_lines_run<32>(d, in, weight, scale, shift, residual, out, st);
  return narrow ? conv_fold_run<16>(d, in, weight, scale, shift, residual, out, st)
                : conv_fold_run<32>(d, in, weight, scale, shift, residual, out, st);
}

// fp32 [K^3 taps (kd, kh, kw)][32][Cout] -> fp16 [NC][32 hi | 32 lo] (128-byte rows) per tap, zero rows for Cout .. NC-1; taps in
// (kd, kh, kw) order for K = 3 (conv_lines_kernel), (kw, kd, kh) for K = 7 (conv_fold_kernel)
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
    const int slot = K == 3 ? tap : (kw * K + kd) * K + kh;
    sh_t* rowp = out + ((long)slot * NC + co) * 64;
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
