// Exact-fp32 implicit-GEMM convolution on CUDA cores (FFMA), channels-last, any filter size /
// stride / padding in up to three spatial dims, with the folded-BN scale/shift, residual and
// ReLU epilogue and the strided output mapping used for transposed-conv phases.
//
// Role: (1) "parity mode" of the conv path -- plain fp32 accumulation, so the whole network can
// be checked against the fp32 oracle at ~1e-6; (2) on-GPU checker for the tensor-core path
// (conv_tc.cu) at sizes the CPU oracle cannot reach; (3) executor for layers the tensor-core
// kernel does not cover (Cin not a multiple of 32: the 7x7 stem).
// Replaces the cuDNN/ATen convs behind pose_resnet.py:62-95,205-209,266-291 and v2v.py:7-66.
#include "common.cuh"

namespace lt {

constexpr int BK = 16;

struct ConvSimtParams {
  lt_conv_desc d;
  const float* in;
  const float* w;      // [taps][Cin][CoutW]
  const float* scale;  // [CoutW]
  const float* shift;  // [CoutW]
  const void* res;
  void* out;
  int CoutW, taps, K;
  long M;              // N*OD*OH*OW
};

__device__ __forceinline__ void decode_pixel(const lt_conv_desc& d, long m, int& n, int& od, int& oh, int& ow) {
  ow = (int)(m % d.OW); m /= d.OW;
  oh = (int)(m % d.OH); m /= d.OH;
  od = (int)(m % d.OD);
  n = (int)(m / d.OD);
}

template <int BM, int BN, int TM, int TN, bool VECA>
__global__ void __launch_bounds__(256) conv_simt_kernel(const ConvSimtParams p) {
  static_assert((BM / TM) * (BN / TN) == 256, "thread tiling must cover the block tile with 256 threads");
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN];
  const lt_conv_desc& d = p.d;
  const int tid = threadIdx.x;
  const long m0 = (long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // ---- per-thread A-load assignment (fixed pixels for the whole K loop) ----
  constexpr int A_LOADS = VECA ? (BM * 4 / 256) : (BM * BK / 256);
  int a_m[VECA ? A_LOADS : 1];
  long a_base[VECA ? A_LOADS : 1];
  int a_d[VECA ? A_LOADS : 1], a_h[VECA ? A_LOADS : 1], a_w[VECA ? A_LOADS : 1];
  if constexpr (VECA) {
#pragma unroll
    for (int i = 0; i < A_LOADS; ++i) {
      const int idx = tid + i * 256;
      const int m = idx >> 2;
      a_m[i] = m;
      const long gm = m0 + m;
      if (gm < p.M) {
        int n, od, oh, ow;
        decode_pixel(d, gm, n, od, oh, ow);
        a_base[i] = (long)n * d.ID * d.IH * d.IW;
        a_d[i] = od * d.sd - d.pd; a_h[i] = oh * d.sh - d.ph; a_w[i] = ow * d.sw - d.pw;
      } else {
        a_base[i] = 0; a_d[i] = -(1 << 28); a_h[i] = 0; a_w[i] = 0;  // forces out-of-bounds -> zeros
      }
    }
  } else {
    const int m = tid % BM;
    a_m[0] = m;
    const long gm = m0 + m;
    if (gm < p.M) {
      int n, od, oh, ow;
      decode_pixel(d, gm, n, od, oh, ow);
      a_base[0] = (long)n * d.ID * d.IH * d.IW;
      a_d[0] = od * d.sd - d.pd; a_h[0] = oh * d.sh - d.ph; a_w[0] = ow * d.sw - d.pw;
    } else {
      a_base[0] = 0; a_d[0] = -(1 << 28); a_h[0] = 0; a_w[0] = 0;
    }
  }

  const int ty = tid / (BN / TN), tx = tid % (BN / TN);
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.0f;

  for (int k0 = 0; k0 < p.K; k0 += BK) {
    // ---- A tile: BM pixels x 16 reduction elements ----
    if constexpr (VECA) {
      const int tap = k0 / d.Cin, ci0 = k0 % d.Cin;
      const int kw = tap % d.KW, kh = (tap / d.KW) % d.KH, kd = tap / (d.KW * d.KH);
#pragma unroll
      for (int i = 0; i < A_LOADS; ++i) {
        const int q = (tid + i * 256) & 3;
        const int id = a_d[i] + kd, ih = a_h[i] + kh, iw = a_w[i] + kw;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (id >= 0 && id < d.ID && ih >= 0 && ih < d.IH && iw >= 0 && iw < d.IW)
          v = __ldg(reinterpret_cast<const float4*>(p.in + (a_base[i] + ((long)id * d.IH + ih) * d.IW + iw) * d.Cin + ci0 + q * 4));
        As[q * 4 + 0][a_m[i]] = v.x; As[q * 4 + 1][a_m[i]] = v.y;
        As[q * 4 + 2][a_m[i]] = v.z; As[q * 4 + 3][a_m[i]] = v.w;
      }
    } else {
#pragma unroll
      for (int i = 0; i < A_LOADS; ++i) {
        const int kk = (tid + i * 256) / BM;
        const int k = k0 + kk;
        float v = 0.0f;
        if (k < p.K) {
          const int tap = k / d.Cin, ci = k % d.Cin;
          const int kw = tap % d.KW, kh = (tap / d.KW) % d.KH, kd = tap / (d.KW * d.KH);
          const int id = a_d[0] + kd, ih = a_h[0] + kh, iw = a_w[0] + kw;
          if (id >= 0 && id < d.ID && ih >= 0 && ih < d.IH && iw >= 0 && iw < d.IW)
            v = __ldg(p.in + (a_base[0] + ((long)id * d.IH + ih) * d.IW + iw) * d.Cin + ci);
        }
        As[kk][a_m[0]] = v;
      }
    }
    // ---- B tile: 16 reduction elements x BN output channels ----
    for (int idx = tid; idx < BK * BN / 4; idx += 256) {
      const int kk = idx / (BN / 4), c4 = (idx % (BN / 4)) * 4;
      const int k = k0 + kk, co = n0 + c4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k < p.K && co < p.CoutW) v = __ldg(reinterpret_cast<const float4*>(p.w + (long)k * p.CoutW + co));
      *reinterpret_cast<float4*>(&Bs[kk][c4]) = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i += 4) *reinterpret_cast<float4*>(&a[i]) = *reinterpret_cast<const float4*>(&As[kk][ty * TM + i]);
#pragma unroll
      for (int j = 0; j < TN; j += 4) *reinterpret_cast<float4*>(&b[j]) = *reinterpret_cast<const float4*>(&Bs[kk][tx * TN + j]);
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

  // ---- epilogue: scale/shift (+residual) (+ReLU) and strided channels-last store ----
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const long gm = m0 + ty * TM + i;
    if (gm >= p.M) continue;
    int n, od, oh, ow;
    decode_pixel(d, gm, n, od, oh, ow);
    const long opix = (((long)n * d.FD + (od * d.osd + d.ood)) * d.FH + (oh * d.osh + d.ooh)) * d.FW + (ow * d.osw + d.oow);
#pragma unroll
    for (int j = 0; j < TN; j += 4) {
      const int co = n0 + tx * TN + j;
      if (co >= p.CoutW || co >= d.FC) continue;
      const float4 sc = __ldg(reinterpret_cast<const float4*>(p.scale + co));
      const float4 sh = __ldg(reinterpret_cast<const float4*>(p.shift + co));
      float4 v = make_float4(fmaf(acc[i][j], sc.x, sh.x), fmaf(acc[i][j + 1], sc.y, sh.y),
                             fmaf(acc[i][j + 2], sc.z, sh.z), fmaf(acc[i][j + 3], sc.w, sh.w));
      float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
      if (d.residual != LT_RES_NONE) {
        if (d.out_format == LT_FMT_F32) r = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.res) + opix * d.FC + co);
        else r = load_s32x4(reinterpret_cast<const sh_t*>(p.res) + opix * 2 * d.FC, co);
      }
      if (d.residual == LT_RES_BEFORE_RELU) { v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w; }
      if (d.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
      if (d.residual == LT_RES_AFTER_RELU) { v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w; }
      if (d.out_format == LT_FMT_F32) *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + opix * d.FC + co) = v;
      else store_s32x4(reinterpret_cast<sh_t*>(p.out) + opix * 2 * d.FC, co, v);
    }
  }
}

template <int BM, int BN, int TM, int TN>
static int launch_simt(const ConvSimtParams& p, cudaStream_t st) {
  const long gx = (p.M + BM - 1) / BM;
  const int gy = (p.CoutW + BN - 1) / BN;
  if (gx > 2147483647L) return fail(LT_ERR_INVALID, "conv_simt: too many output positions");
  dim3 grid((unsigned)gx, (unsigned)gy);
  if (p.d.Cin % BK == 0) conv_simt_kernel<BM, BN, TM, TN, true><<<grid, 256, 0, st>>>(p);
  else conv_simt_kernel<BM, BN, TM, TN, false><<<grid, 256, 0, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(LT_ERR_CUDA, "conv_simt_kernel: %s", cudaGetErrorString(e));
  return LT_OK;
}

int conv_simt_fwd(const lt_conv_desc* d, const void* in, const void* weight, const float* scale, const float* shift,
                  const void* residual, void* out, void* stream) {
  LT_REQUIRE(d->in_format == LT_FMT_F32, "conv_simt: input must be float32 channels-last");
  LT_REQUIRE(d->FC % 4 == 0, "conv_simt: output channel stride FC=%d must be a multiple of 4", d->FC);
  LT_REQUIRE(d->out_format == LT_FMT_F32 || d->FC % 32 == 0, "conv_simt: split-fp16 output needs FC %% 32 == 0");
  ConvSimtParams p;
  p.d = *d;
  p.in = reinterpret_cast<const float*>(in);
  p.w = reinterpret_cast<const float*>(weight);
  p.scale = scale; p.shift = shift; p.res = residual; p.out = out;
  p.CoutW = (d->Cout + 3) & ~3;
  p.taps = d->KD * d->KH * d->KW;
  p.K = p.taps * d->Cin;
  p.M = (long)d->N * d->OD * d->OH * d->OW;
  cudaStream_t st = (cudaStream_t)stream;
  if (p.CoutW <= 16) return launch_simt<256, 16, 4, 4>(p, st);
  if (p.CoutW <= 32) return launch_simt<128, 32, 4, 4>(p, st);
  return launch_simt<128, 64, 8, 4>(p, st);
}

}  // namespace lt
