// Launch parameters of the wgmma implicit-GEMM conv kernel (conv_tc.cu).
#pragma once
#include "tc_common.cuh"

namespace lt {

struct TcParams {
  int OW, OH, OD, N;       // output grid computed by this launch
  int bw, bh, bd, bn;      // M-tile box, product 128
  int tw, th, td, tn;      // tiles per dim
  int KW, KH, KD, pw, ph, pd;
  int sw, sh, sd;          // input stride (TMA element strides)
  int CB;                  // 64-element K chunks per tap
  int b_step0, b_step1;    // B-map coordinates of chunk q: (q*b_step0, q*b_step1 + n0*b_nmul)
  int b_nmul;
  int Nt, stages, terms;   // N tile, pipeline depth, 0 (plain fp16 rows), 1 or 3 product terms
  // epilogue
  int FC, FD, FH, FW, osd, osh, osw, ood, ooh, oow, relu, residual, out_format;
  const float* scale;
  const float* shift;
  const void* res;
  void* out;
  // split-K (latency-bound layers with fewer CTAs than SMs): blockIdx.z owns a contiguous range of the K chunks and
  // writes its raw fp32 accumulator tile to ws[z][m tile][128][ws_ld]; splitk_reduce_kernel sums and applies the epilogue
  int splits, ws_ld;
  float* ws;
  float ws_gain;   // splitk_reduce_kernel: accum_gain(steps of one split) / accum_gain(steps of the whole K loop), see launch_tc
  int n_tiles;   // N tiles of Nt channels (conv_tc_kernel work units: n_tiles x M tiles x splits)
  // grouped output (lt_conv_desc.ogd/ogh/ogw): output channel block g of `oc` channels goes to output map g (its own phase offset)
  int oc, n_maps;
  int gh, gw;    // output group grid (group g -> offset (g / (gh*gw), (g / gw) % gh, g % gw)); 1, 1 without groups
  int epi_buffers;   // conv_tc_kernel's staged epilogue tile buffers: 2 (unit k uses buffer k & 1), 1, or 0 when not staged
};

// grouped output (lt_conv_desc.ogd/ogh/ogw): a k2 s2 transposed conv as ONE GEMM with N = 8 x Cout, group g = phase (a, b, c) of
// the output lattice
constexpr int kMaxOutMaps = 8;

// Tensor maps of conv_tc_kernel's staged epilogue, one per output group (only [0] without groups): the output and the residual
// over the launch's OW x OH x OD x N output grid (stride-phase outputs: the phase's sub-lattice), boxes of 32 channels x the M tile.
struct TcEpiMaps {
  CUtensorMap out[kMaxOutMaps];
  CUtensorMap res[kMaxOutMaps];
};

constexpr int kATileBytes = 128 * 128;  // 128 rows x 64 fp16

// Output pixel and channel of accumulator column 8i + c2 of a tile whose first output channel is n0: grouped outputs send channel
// block mi to output phase (mi / (gh gw), (mi / gw) % gh, mi % gw).
__device__ __forceinline__ void epilogue_target(const TcParams& p, int co, long opix, int& ch, long& pix) {
  ch = co;
  pix = opix;
  if (p.n_maps > 1) {
    const int mi = ch / p.oc;
    ch -= mi * p.oc;
    pix += ((long)(mi / (p.gh * p.gw)) * p.FH + (mi / p.gw) % p.gh) * p.FW + mi % p.gw;
  }
}

// Fused epilogue of one row of a 64 x NT wgmma accumulator tile (conv_tc.cu, conv_fold.cu): this thread holds columns 8i + c2 (+1)
// of row 16 w + l / 4 (h = 0) or the row 8 below it (h = 1), which belongs to output pixel `opix`; n0 is the tile's first output
// channel.  Forms D1 + D2 / S (3-term products) and applies the folded scale / shift, the residual, ReLU and the store (float32 or
// split-fp16; grouped outputs go to their phase of the output lattice).
template <int NT>
__device__ __forceinline__ float2 epilogue_residual(const TcParams& p, int ch, long pix) {
  if (p.residual == LT_RES_NONE || ch >= p.FC) return make_float2(0.f, 0.f);
  if (p.out_format == LT_FMT_F32) return *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(p.res) + pix * p.FC + ch);
  const sh_t* rp = reinterpret_cast<const sh_t*>(p.res) + pix * 2 * p.FC + s32_off(ch);
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(rp));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(rp + 32));
  return make_float2(fmaf(b.x, kLoInv, a.x), fmaf(b.y, kLoInv, a.y));
}

// The residual of the whole row is loaded before the first store: the output may alias the residual as far as the compiler knows,
// so loads interleaved with the stores would each wait for a full memory round trip.  Used for tiles of up to 32 channels only
// (conv_fold_kernel, and conv_tc_kernel's 16-channel tiles); wider conv_tc tiles stage their epilogue in shared memory.
template <int NT>
__device__ __forceinline__ void conv_epilogue_row(const TcParams& p, const float (&d1)[NT / 2], const float (&d2)[NT / 2], int h,
                                                  long opix, int n0, int c2) {
  static_assert(NT <= 32, "wider tiles would not hold the hoisted residual beside their accumulators");
  float2 rr[NT / 8];
#pragma unroll
  for (int i = 0; i < NT / 8; ++i) {
    int ch;
    long pix;
    epilogue_target(p, n0 + 8 * i + c2, opix, ch, pix);
    rr[i] = epilogue_residual<NT>(p, ch, pix);
  }
#pragma unroll
  for (int i = 0; i < NT / 8; ++i) {
    const int k = 4 * i + 2 * h;
    const int co = n0 + 8 * i + c2;
    int ch;
    long pix;
    epilogue_target(p, co, opix, ch, pix);
    if (ch >= p.FC) continue;
    float v0 = (p.terms == 3) ? fmaf(d2[k], kLoInv, d1[k]) : d1[k];
    float v1 = (p.terms == 3) ? fmaf(d2[k + 1], kLoInv, d1[k + 1]) : d1[k + 1];
    const float2 sc = __ldg(reinterpret_cast<const float2*>(p.scale + co));
    const float2 sh = __ldg(reinterpret_cast<const float2*>(p.shift + co));
    v0 = fmaf(v0, sc.x, sh.x);
    v1 = fmaf(v1, sc.y, sh.y);
    const float2 r = rr[i];
    if (p.residual == LT_RES_BEFORE_RELU) { v0 += r.x; v1 += r.y; }
    if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
    if (p.residual == LT_RES_AFTER_RELU) { v0 += r.x; v1 += r.y; }
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

// ---- host helpers (conv_tc.cu) ----
// geometry / epilogue part of the launch parameters for `CB` 32-channel input blocks, CoutP padded output channels and N tile Nt
void fill_params(const lt_conv_desc* d, TcParams& p, int CB, int CoutP, int Nt, int terms, const float* scale, const float* shift,
                 const void* residual, void* out);
// input tensor map: split-fp16 channels-last rows [64 fp16], box of bw x bh x bd x bn positions (before the traversal strides)
int make_in_map(CUtensorMap* tmA, const lt_conv_desc* d, int bw, int bh, int bd, int bn, const void* in);

}  // namespace lt
