// Tensor-core implicit-GEMM convolution for sm_90a: TMA-staged channels-last tiles -> shared memory (128B swizzle) ->
// wgmma (m64 x Nt x k16 per warpgroup, fp16 in, fp32 accumulators in registers) -> epilogue with folded-BN scale/shift,
// residual, ReLU and strided channels-last store straight from the accumulator registers (plain conv, stride-phase
// transposed conv, grouped outputs).
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
// Warp roles (384 threads): warpgroup 0 = TMA producer (one warp issues), warpgroups 1 and 2 = MMA + epilogue for rows 0-63 and
// 64-127 of the M tile.  The operand ring is released per stage by one arrival of each consumer warpgroup once its MMAs that read
// the stage have completed (wgmma.wait_group 1 keeps one chunk of MMAs in flight behind the issue).
#include "tc_common.cuh"
#include "conv_tc_params.cuh"
#include <stdlib.h>
#include <string.h>

namespace lt {

// ------------------------------------------------------------------------------------------------
// Kernel
// ------------------------------------------------------------------------------------------------
constexpr int kTcThreads = 384;

__device__ __forceinline__ void regs_release_producer() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void regs_claim_consumer() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }

template <int NT>
__global__ void __launch_bounds__(kTcThreads, 1) conv_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                const __grid_constant__ CUtensorMap tmB, const TcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int kStage = kATileBytes + NT * 128;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * kStage);
  uint64_t* empty = full + p.stages;

  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int lane = threadIdx.x & 31;

  // tile coordinates
  int t = blockIdx.x;
  const int twi = t % p.tw; t /= p.tw;
  const int thi = t % p.th; t /= p.th;
  const int tdi = t % p.td; t /= p.td;
  const int tni = t;
  const int ow0 = twi * p.bw, oh0 = thi * p.bh, od0 = tdi * p.bd, nb0 = tni * p.bn;
  const int n0 = blockIdx.y * NT;
  const int nchunks_all = p.KD * p.KH * p.KW * p.CB;
  const int q_begin = (int)(((long)blockIdx.z * nchunks_all) / p.splits);
  const int nchunks = (int)(((long)(blockIdx.z + 1) * nchunks_all) / p.splits) - q_begin;   // chunks of this split

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    fence_barrier_init();
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
  }
  __syncthreads();

  if (wg == 0) {
    // ================= TMA producer (warp 0 runs the loop; one elected lane issues) =================
    regs_release_producer();
    if (threadIdx.x < 32) {
      // chunk -> (tap, channel block) and ring slot / phase are advanced incrementally: no integer division in the loop
      int tap = q_begin / p.CB, cb = q_begin - tap * p.CB;
      int kw = tap % p.KW, kh = (tap / p.KW) % p.KH, kd = tap / (p.KW * p.KH);
      int s = 0;
      uint32_t ph = 0;
      const int ax = ow0 * p.sw - p.pw, ay = oh0 * p.sh - p.ph, az = od0 * p.sd - p.pd, bn0 = n0 * p.b_nmul;
      for (int q = 0, qa = q_begin; q < nchunks; ++q, ++qa) {
        mbar_wait(&empty[s], ph ^ 1u);
        uint8_t* a_dst = smem + (size_t)s * kStage;
        if (elect_one()) {
          mbar_expect_tx(&full[s], (uint32_t)kStage);
          tma_load_5d(a_dst, &tmA, &full[s], cb * 64, ax + kw, ay + kh, az + kd, nb0);
          tma_load_2d(a_dst + kATileBytes, &tmB, &full[s], qa * p.b_step0, qa * p.b_step1 + bn0);
        }
        __syncwarp();
        if (++cb == p.CB) { cb = 0; if (++kw == p.KW) { kw = 0; if (++kh == p.KH) { kh = 0; ++kd; } } }
        if (++s == p.stages) { s = 0; ph ^= 1u; }
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
  {
    int s = 0, prev = -1;
    uint32_t ph = 0;
    const uint32_t ring0 = smem_u32(smem);
    for (int q = 0; q < nchunks; ++q) {
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
    wg_fence_regs(d1);
    wg_fence_regs(d2);
  }

  // ---- epilogue: this thread holds rows r0 and r0 + 8, columns 8i + c2 (+1) of the 64 x NT warpgroup tile ----
  const int r0 = g * 64 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
  const int c2 = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = r0 + 8 * h;
    if (p.splits > 1) {
      // ---- split-K: raw accumulators to the workspace, epilogue deferred to splitk_reduce_kernel ----
      float* wrow = p.ws + (((size_t)blockIdx.z * gridDim.x + blockIdx.x) * 128 + row) * p.ws_ld + n0;
#pragma unroll
      for (int i = 0; i < NT / 8; ++i) {
        const int k = 4 * i + 2 * h;
        const float v0 = (p.terms == 3) ? fmaf(d2[k], kLoInv, d1[k]) : d1[k];
        const float v1 = (p.terms == 3) ? fmaf(d2[k + 1], kLoInv, d1[k + 1]) : d1[k + 1];
        *reinterpret_cast<float2*>(wrow + 8 * i + c2) = make_float2(v0, v1);
      }
      continue;
    }
    int r_ = row;
    const int dw = r_ % p.bw; r_ /= p.bw;
    const int dh = r_ % p.bh; r_ /= p.bh;
    const int dd = r_ % p.bd; r_ /= p.bd;
    const int ow = ow0 + dw, oh = oh0 + dh, od = od0 + dd, nb = nb0 + r_;
    if (!(ow < p.OW && oh < p.OH && od < p.OD && nb < p.N)) continue;
    const long opix = (((long)nb * p.FD + (od * p.osd + p.ood)) * p.FH + (oh * p.osh + p.ooh)) * p.FW + (ow * p.osw + p.oow);
#pragma unroll
    for (int i = 0; i < NT / 8; ++i) {
      const int k = 4 * i + 2 * h;
      const int co = n0 + 8 * i + c2;
      int ch = co;
      long pix = opix;
      if (p.n_maps > 1) {   // grouped output: channel block of group mi goes to output phase (mi / (gh gw), (mi / gw) % gh, mi % gw)
        const int mi = ch / p.oc;
        ch -= mi * p.oc;
        pix += ((long)(mi / (p.gh * p.gw)) * p.FH + (mi / p.gw) % p.gh) * p.FW + mi % p.gw;
      }
      if (ch >= p.FC) continue;
      float v0 = (p.terms == 3) ? fmaf(d2[k], kLoInv, d1[k]) : d1[k];
      float v1 = (p.terms == 3) ? fmaf(d2[k + 1], kLoInv, d1[k + 1]) : d1[k + 1];
      const float2 sc = __ldg(reinterpret_cast<const float2*>(p.scale + co));
      const float2 sh = __ldg(reinterpret_cast<const float2*>(p.shift + co));
      v0 = fmaf(v0, sc.x, sh.x);
      v1 = fmaf(v1, sc.y, sh.y);
      float2 rr = make_float2(0.f, 0.f);
      if (p.residual != LT_RES_NONE) {
        if (p.out_format == LT_FMT_F32) {
          rr = *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(p.res) + pix * p.FC + ch);
        } else {
          const sh_t* rp = reinterpret_cast<const sh_t*>(p.res) + pix * 2 * p.FC + s32_off(ch);
          const float2 a = __half22float2(*reinterpret_cast<const __half2*>(rp));
          const float2 b = __half22float2(*reinterpret_cast<const __half2*>(rp + 32));
          rr = make_float2(fmaf(b.x, kLoInv, a.x), fmaf(b.y, kLoInv, a.y));
        }
      }
      if (p.residual == LT_RES_BEFORE_RELU) { v0 += rr.x; v1 += rr.y; }
      if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
      if (p.residual == LT_RES_AFTER_RELU) { v0 += rr.x; v1 += rr.y; }
      if (p.out_format == LT_FMT_F32) {
        *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + pix * p.FC + ch) = make_float2(v0, v1);
      } else {
        uint32_t hi2, lo2;
        split_s32x2(v0, v1, hi2, lo2);
        sh_t* op = reinterpret_cast<sh_t*>(p.out) + pix * 2 * p.FC + s32_off(ch);
        *reinterpret_cast<uint32_t*>(op) = hi2;
        *reinterpret_cast<uint32_t*>(op + 32) = lo2;
      }
    }
  }
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
static int launch_nt(const CUtensorMap& tmA, const CUtensorMap& tmB, const TcParams& p, dim3 grid, size_t smem, cudaStream_t st) {
  static DeviceOnce configured;
  if (configured.first()) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e != cudaSuccess) return fail(LT_ERR_CUDA, "conv_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  }
  conv_tc_kernel<NT><<<grid, kTcThreads, smem, st>>>(tmA, tmB, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(LT_ERR_CUDA, "conv_tc_kernel: %s", cudaGetErrorString(e));
  return LT_OK;
}

static int launch_tc(const CUtensorMap& tmA, const CUtensorMap& tmB, TcParams& p, int n_tiles, cudaStream_t st, void* ws = nullptr,
                     size_t ws_bytes = 0) {
  const int stage_bytes = kATileBytes + p.Nt * 128;
  // one CTA per SM (the two consumer warpgroups hold up to 128 fp32 accumulators per thread): the whole shared memory is
  // pipeline depth
  int stages = (200 * 1024) / stage_bytes;
  if (stages > 8) stages = 8;
  p.stages = stages;
  const size_t smem = (size_t)stages * stage_bytes + 2 * stages * 8 + 1024;
  const long m_tiles = (long)p.tw * p.th * p.td * p.tn;
  const int nchunks_total = p.KD * p.KH * p.KW * p.CB;
  // split-K: a grid that cannot fill half the SMs is bound by the serial K loop of each CTA (27 taps x Cin/32 chunks of
  // weights streamed from HBM by ONE SM); spread the chunks over blockIdx.z instead
  int splits = 1;
  const long grid_ctas = m_tiles * n_tiles;
  if (opts().tc_splitk && ws && p.terms != 0 && p.n_maps == 1 && grid_ctas * 2 <= (long)sm_count() && nchunks_total >= 16) {
    splits = (int)((long)sm_count() / grid_ctas);
    if (splits > nchunks_total / 4) splits = nchunks_total / 4;
    const size_t per_split = (size_t)m_tiles * 128 * (size_t)n_tiles * p.Nt * sizeof(float);
    if ((size_t)splits * per_split > ws_bytes) splits = (int)(ws_bytes / per_split);
    if (splits < 2) splits = 1;
  }
  p.splits = splits;
  p.ws = reinterpret_cast<float*>(ws);
  p.ws_ld = n_tiles * p.Nt;
  dim3 grid((unsigned)m_tiles, (unsigned)n_tiles, (unsigned)splits);
  int rc;
  switch (p.Nt) {
    case 128: rc = launch_nt<128>(tmA, tmB, p, grid, smem, st); break;
    case 64: rc = launch_nt<64>(tmA, tmB, p, grid, smem, st); break;
    case 32: rc = launch_nt<32>(tmA, tmB, p, grid, smem, st); break;
    case 16: rc = launch_nt<16>(tmA, tmB, p, grid, smem, st); break;
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
static void fill_params(const lt_conv_desc* d, TcParams& p, int CB, int CoutP, int Nt, int terms, const float* scale, const float* shift,
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
  p.splits = 1; p.ws = nullptr; p.ws_ld = 0; p.stages = 0;
  p.n_maps = out_groups(d);
  p.oc = p.n_maps > 1 ? d->Cout / p.n_maps : CoutP;
  p.gh = d->ogh > 1 ? d->ogh : 1; p.gw = d->ogw > 1 ? d->ogw : 1;
}

static int make_in_map(CUtensorMap* tmA, const lt_conv_desc* d, const TcParams& p, const void* in) {
  const uint64_t rowb = (uint64_t)d->Cin * 2 * 2;  // 2*Cin fp16 per position
  const uint64_t dims[5] = {(uint64_t)d->Cin * 2, (uint64_t)d->IW, (uint64_t)d->IH, (uint64_t)d->ID, (uint64_t)d->N};
  const uint64_t str[4] = {rowb, rowb * d->IW, rowb * d->IW * d->IH, rowb * d->IW * d->IH * d->ID};
  // strided convs: TMA traversal strides; the box spans (b-1)*s+1 input positions and delivers b of them
  const uint32_t es[5] = {1, (uint32_t)d->sw, (uint32_t)d->sh, (uint32_t)d->sd, 1};
  uint32_t bx[5] = {64, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bd, (uint32_t)p.bn};
  for (int i = 1; i <= 3; ++i) bx[i] = (bx[i] - 1) * es[i] + 1;
  LT_REQUIRE(bx[1] <= 256 && bx[2] <= 256 && bx[3] <= 256, "conv_tc: strided box exceeds 256");
  return make_map(tmA, in, 5, dims, str, bx, es, 1);
}

// grouped output (k2 s2 transposed conv as one GEMM): every channel of the GEMM belongs to exactly one group, and a group fills the
// output's channels exactly
static bool groups_ok(const lt_conv_desc* d, int CoutP) {
  const int G = out_groups(d);
  return d->Cout % G == 0 && (d->Cout / G) % 32 == 0 && d->Cout / G == d->FC && CoutP == d->Cout && G <= kMaxOutMaps &&
         d->out_format == LT_FMT_S32;
}

// Shared by every tensor-core entry point: weights packed as [tap][Cin/32][CoutP rows][32 hi | 32 lo] fp16.
static int conv_wg_fwd(const lt_conv_desc* d, const void* in, const void* weight, int CoutP, const float* scale, const float* shift,
                       const void* residual, void* out, int terms, void* stream) {
  LT_REQUIRE(d->in_format == LT_FMT_S32, "conv_tc: input must be split-fp16");
  LT_REQUIRE(d->Cin % 32 == 0, "conv_tc: Cin=%d must be a multiple of 32", d->Cin);
  LT_REQUIRE(d->FC % 4 == 0 && (d->out_format == LT_FMT_F32 || d->FC % 32 == 0), "conv_tc: bad output channel stride %d", d->FC);
  const int CB = d->Cin / 32;
  const int taps = d->KD * d->KH * d->KW;
  const int Nt = pick_nt(CoutP);
  TcParams p;
  fill_params(d, p, CB, CoutP, Nt, terms, scale, shift, residual, out);
  if (p.n_maps > 1)
    LT_REQUIRE(groups_ok(d, CoutP), "conv_tc: grouped output needs split-fp16 output, Cout / groups == FC, a multiple of 32");
  CUtensorMap tmA, tmB;
  int rc = make_in_map(&tmA, d, p, in);
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

// 128-padded weights (lt_conv_pair_pack_weights): the layers with Cout % 128 == 0
int conv_pair_fwd(const lt_conv_desc* d, const void* in, const void* weight, const float* scale, const float* shift,
                  const void* residual, void* out, void* stream, int probe_only) {
  const int CoutP = (d->Cout + 127) & ~127;
  const int G = out_groups(d);
  const bool ok = d->in_format == LT_FMT_S32 && d->Cin % 32 == 0 && d->Cout % 128 == 0 &&
                  (G > 1 ? groups_ok(d, CoutP) : (d->FC % 32 == 0 && CoutP <= d->FC));
  if (probe_only) return ok ? 0 : 1;
  if (!ok) return fail(LT_ERR_INVALID, "conv_pair: shape not covered (Cout=%d FC=%d)", d->Cout, d->FC);
  return conv_wg_fwd(d, in, weight, CoutP, scale, shift, residual, out, 3, stream);
}

int conv_tc_fwd_terms(const lt_conv_desc* d, const void* in, const void* weight, const float* scale, const float* shift,
                      const void* residual, void* out, int terms, void* stream) {
  return conv_wg_fwd(d, in, weight, (d->Cout + 15) & ~15, scale, shift, residual, out, terms, stream);
}

// kw-fold entry point (LT_CONV_TC_FOLD: Cin = 32 cubic stride-1 layers): the same kernel over weights packed by
// lt_conv_fold_pack_weights as [tap][1][32 rows][32 hi | 32 lo], i.e. all 32 output channels (the padding ones are zero)
int conv_fold_supported(const lt_conv_desc* d) {
  const bool cubic = d->KD == d->KH && d->KH == d->KW && (d->KW == 3 || d->KW == 7);
  const int pd = d->KW / 2;
  return cubic && d->Cin == 32 && d->Cout <= 32 && d->sd == 1 && d->sh == 1 && d->sw == 1 && d->pd == pd && d->ph == pd &&
         d->pw == pd && d->OD == d->ID && d->OH == d->IH && d->OW == d->IW && d->osd == 1 && d->osh == 1 && d->osw == 1 &&
         d->ood == 0 && d->ooh == 0 && d->oow == 0 && d->FD == d->OD && d->FH == d->OH && d->FW == d->OW && d->FC == 32 &&
         d->in_format == LT_FMT_S32 && d->IW >= 16;
}

int conv_fold_fwd(const lt_conv_desc* d, const void* in, const void* weight, const float* scale, const float* shift,
                  const void* residual, void* out, void* stream) {
  LT_REQUIRE(conv_fold_supported(d), "conv_fold: unsupported layer shape");
  lt_conv_desc dg = *d;
  dg.Cout = 32;
  return conv_wg_fwd(&dg, in, weight, 32, scale, shift, residual, out, 3, stream);
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

static int pack_weights(const float* w, void* packed, int taps, int Cin, int Cout, int CoutP, void* stream) {
  const long total = (long)taps * (Cin / 32) * CoutP * 32;
  long blocks = (total + 255) / 256;
  if (blocks > 65535) blocks = 65535;
  pack_weights_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(w, reinterpret_cast<sh_t*>(packed), taps, Cin, Cout, CoutP);
  LT_CHECK_LAUNCH("pack_weights_kernel");
  return LT_OK;
}

__global__ void ones_zeros_kernel(float* ones, float* zeros, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { ones[i] = 1.0f; zeros[i] = 0.0f; }
}

}  // namespace lt

using namespace lt;

extern "C" size_t lt_conv_tc_weight_bytes(int taps, int Cin, int Cout) {
  const int CoutP = (Cout + 15) & ~15;
  return (size_t)taps * (Cin / 32) * CoutP * 128;
}

extern "C" int lt_conv_tc_pack_weights(const float* w, void* packed, int taps, int Cin, int Cout, void* stream) {
  LT_REQUIRE(w && packed, "conv_tc_pack_weights: null pointer");
  LT_REQUIRE(Cin % 32 == 0 && taps > 0 && Cout > 0, "conv_tc_pack_weights: bad sizes");
  return pack_weights(w, packed, taps, Cin, Cout, (Cout + 15) & ~15, stream);
}

extern "C" size_t lt_conv_pair_weight_bytes(int taps, int Cin, int Cout) {
  const int CoutP = (Cout + 127) & ~127;
  return (size_t)taps * (Cin / 32) * CoutP * 128;
}

extern "C" int lt_conv_pair_pack_weights(const float* w, void* packed, int taps, int Cin, int Cout, void* stream) {
  LT_REQUIRE(w && packed, "conv_pair_pack_weights: null pointer");
  LT_REQUIRE(Cin % 32 == 0 && taps > 0 && Cout > 0, "conv_pair_pack_weights: bad sizes");
  return pack_weights(w, packed, taps, Cin, Cout, (Cout + 127) & ~127, stream);
}

extern "C" size_t lt_conv_fold_weight_bytes(int K, int Cout) {
  (void)Cout;
  return (size_t)K * K * K * 32 * 128;
}

// w_tap_ci_co: fp32 [K^3 taps (kd, kh, kw)][32][Cout]
extern "C" int lt_conv_fold_pack_weights(const float* w_tap_ci_co, void* packed, int K, int Cout, void* stream) {
  LT_REQUIRE(w_tap_ci_co && packed && (K == 3 || K == 7) && Cout > 0 && Cout <= 32, "conv_fold_pack_weights: bad arguments");
  return pack_weights(w_tap_ci_co, packed, K * K * K, 32, Cout, 32, stream);
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
