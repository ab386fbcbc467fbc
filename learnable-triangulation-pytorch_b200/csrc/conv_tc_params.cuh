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
  // grouped output (lt_conv_desc.ogd/ogh/ogw): output channel block g of `oc` channels goes to output map g (its own phase offset)
  int oc, n_maps;
  int gh, gw;    // output group grid (group g -> offset (g / (gh*gw), (g / gw) % gh, g % gw)); 1, 1 without groups
};

// grouped output (lt_conv_desc.ogd/ogh/ogw): a k2 s2 transposed conv as ONE GEMM with N = 8 x Cout, group g = phase (a, b, c) of
// the output lattice
constexpr int kMaxOutMaps = 8;

constexpr int kATileBytes = 128 * 128;  // 128 rows x 64 fp16

}  // namespace lt
