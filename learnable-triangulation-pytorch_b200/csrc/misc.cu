// Small bandwidth-bound helpers: coordinate volume, max pooling, layout / format conversion.
#include "common.cuh"

namespace lt {

// ---- coordinate volume -------------------------------------------------------------------------
// triangulation.py:306-333: grid index -> mm (position + step * index, float32), minus centre,
// rotation (volumetric.py:102-114, R @ v), plus centre; optional CMU->H36M transfer (:336-339):
// out[a][b][c] = base[a][c][n-1-b].  __fmul_rn/__fadd_rn keep the reference's unfused op order.
__global__ void __launch_bounds__(256) coord_volume_kernel(const float* __restrict__ position, const float* __restrict__ center,
                                                           const float* __restrict__ step, const float* __restrict__ rot,
                                                           float* __restrict__ out, int B, int n, int transfer_cmu) {
  const long nvox = (long)n * n * n;
  const long total = (long)B * nvox;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int b = (int)(i / nvox);
    const long r = i % nvox;
    int a = (int)(r / ((long)n * n)), bb = (int)((r / n) % n), c = (int)(r % n);
    int gi = a, gj = bb, gk = c;
    if (transfer_cmu) { gj = c; gk = n - 1 - bb; }
    const float* pos = position + b * 3;
    const float* cen = center + b * 3;
    const float* R = rot + b * 9;
    float x = __fadd_rn(pos[0], __fmul_rn(step[0], (float)gi));
    float y = __fadd_rn(pos[1], __fmul_rn(step[1], (float)gj));
    float z = __fadd_rn(pos[2], __fmul_rn(step[2], (float)gk));
    x = __fadd_rn(x, -cen[0]); y = __fadd_rn(y, -cen[1]); z = __fadd_rn(z, -cen[2]);
    const float rx = fmaf(R[2], z, fmaf(R[1], y, __fmul_rn(R[0], x)));
    const float ry = fmaf(R[5], z, fmaf(R[4], y, __fmul_rn(R[3], x)));
    const float rz = fmaf(R[8], z, fmaf(R[7], y, __fmul_rn(R[6], x)));
    float* o = out + i * 3;
    o[0] = __fadd_rn(rx, cen[0]);
    o[1] = __fadd_rn(ry, cen[1]);
    o[2] = __fadd_rn(rz, cen[2]);
  }
}

// ---- cuboid placement from predicted key points ------------------------------------------------------
// One thread per (sample, axis): the values _base_points / _host_geometry compute on the host from the key points as float32
// numpy rows.  The coco hip midpoint is the float32 sum halved in float32, as numpy's / 2 on a float32 array (x * 0.5 rounds to
// the same float as x / 2); position = base - side / 2 is formed in float64 and rounded to float32 last.  Explicit _rn
// intrinsics: nothing is contracted into an FMA.  Not a hot path: a few threads per batch between the algebraic and the
// volumetric stage.
__global__ void cuboid_from_keypoints_kernel(const float* __restrict__ keypoints, int B, int J, int kind, double side,
                                             float* __restrict__ center, float* __restrict__ position) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * 3) return;
  const int b = i / 3, c = i - b * 3;
  const float* kp = keypoints + (long)b * J * 3;
  const float base = kind == LT_KIND_COCO ? __fmul_rn(__fadd_rn(kp[11 * 3 + c], kp[12 * 3 + c]), 0.5f) : kp[6 * 3 + c];
  center[i] = base;
  position[i] = __double2float_rn(__dsub_rn((double)base, __ddiv_rn(side, 2.0)));
}

// ---- max pooling, channels-last, 4 channels per thread ----------------------------------------------
// torch's max_pool rule per lane, in window order: a value replaces the running maximum if it is greater or NaN, so a NaN in the
// window gives NaN (fmaxf would drop it); taps in the padding are skipped, i.e. they count as -inf.
__device__ __forceinline__ float pool_max(float m, float v) { return (v > m || isnan(v)) ? v : m; }

struct PoolParams {
  const void* in; void* out; int format;
  int N, ID, IH, IW, C, kd, kh, kw, sd, sh, sw, pd, ph, pw, OD, OH, OW;
};

__global__ void __launch_bounds__(256) maxpool_kernel(const PoolParams p) {
  const int c4n = p.C / 4;
  const long total = (long)p.N * p.OD * p.OH * p.OW * c4n;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % c4n) * 4;
    long r = i / c4n;
    const int ow = (int)(r % p.OW); r /= p.OW;
    const int oh = (int)(r % p.OH); r /= p.OH;
    const int od = (int)(r % p.OD);
    const int n = (int)(r / p.OD);
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int a = 0; a < p.kd; ++a) {
      const int id = od * p.sd - p.pd + a;
      if (id < 0 || id >= p.ID) continue;
      for (int b = 0; b < p.kh; ++b) {
        const int ih = oh * p.sh - p.ph + b;
        if (ih < 0 || ih >= p.IH) continue;
        for (int e = 0; e < p.kw; ++e) {
          const int iw = ow * p.sw - p.pw + e;
          if (iw < 0 || iw >= p.IW) continue;
          const long pix = (((long)n * p.ID + id) * p.IH + ih) * p.IW + iw;
          float4 v;
          if (p.format == LT_FMT_F32) v = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.in) + pix * p.C + c));
          else v = load_s32x4(reinterpret_cast<const sh_t*>(p.in) + pix * 2 * p.C, c);
          m.x = pool_max(m.x, v.x); m.y = pool_max(m.y, v.y); m.z = pool_max(m.z, v.z); m.w = pool_max(m.w, v.w);
        }
      }
    }
    const long opix = (((long)n * p.OD + od) * p.OH + oh) * p.OW + ow;
    if (p.format == LT_FMT_F32) *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + opix * p.C + c) = m;
    else store_s32x4(reinterpret_cast<sh_t*>(p.out) + opix * 2 * p.C, c, m);
  }
}


// ---- max-pool backward, non-overlapping windows (kernel == stride, no padding), float32, any element strides ----------
// The gather form of torch's max_pool3d backward: one thread per input element re-finds its window's arg-max with torch's rule
// (scan d, h, w; a value is taken if greater than the running maximum or NaN, the window's first element if none is), and writes
// 0 + grad_y there (torch adds into a zeroed gradient) and 0 elsewhere, including the tail floor mode drops.  No atomics.
struct Pool3dBwdParams {
  const float* x; const float* gy; float* gx;
  int N, C, D, H, W, k;
  long xs[5], gs[5];    // element strides (n, c, d, h, w) of x and grad_x, and of grad_y
};

__host__ __device__ __forceinline__ void pool3d_bwd_item(const Pool3dBwdParams& p, long i) {
  int n, c, d, h, w;
  long r = i;
  if (p.xs[1] == 1 && p.C > 1) {   // channels-last: walk memory order, c fastest
    c = (int)(r % p.C); r /= p.C; w = (int)(r % p.W); r /= p.W; h = (int)(r % p.H); r /= p.H; d = (int)(r % p.D); n = (int)(r / p.D);
  } else {
    w = (int)(r % p.W); r /= p.W; h = (int)(r % p.H); r /= p.H; d = (int)(r % p.D); r /= p.D; c = (int)(r % p.C); n = (int)(r / p.C);
  }
  const int k = p.k, od = d / k, oh = h / k, ow = w / k;
  float out = 0.0f;
  if (od < p.D / k && oh < p.H / k && ow < p.W / k) {
    const float* xb = p.x + n * p.xs[0] + c * p.xs[1];
    const int d0 = od * k, h0 = oh * k, w0 = ow * k;
    float m = -INFINITY;
    int best = 0;
    for (int a = 0; a < k; ++a)
      for (int b = 0; b < k; ++b)
        for (int e = 0; e < k; ++e) {
          const float v = xb[(d0 + a) * p.xs[2] + (h0 + b) * p.xs[3] + (w0 + e) * p.xs[4]];
          if (v > m || v != v) { m = v; best = (a * k + b) * k + e; }
        }
    if (best == ((d - d0) * k + (h - h0)) * k + (w - w0))
      out = 0.0f + p.gy[n * p.gs[0] + c * p.gs[1] + od * p.gs[2] + oh * p.gs[3] + ow * p.gs[4]];
  }
  p.gx[n * p.xs[0] + c * p.xs[1] + d * p.xs[2] + h * p.xs[3] + w * p.xs[4]] = out;
}

__global__ void __launch_bounds__(256) pool3d_bwd_kernel(const Pool3dBwdParams p, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) pool3d_bwd_item(p, i);
}

static int pool3d_bwd_check(const float* x, const float* grad_y, float* grad_x, int N, int C, int D, int H, int W, int k) {
  LT_REQUIRE(x && grad_y && grad_x, "maxpool3d_bwd: null pointer");
  LT_REQUIRE(N > 0 && C > 0 && D > 0 && H > 0 && W > 0, "maxpool3d_bwd: non-positive size");
  LT_REQUIRE(k >= 1 && k <= D && k <= H && k <= W, "maxpool3d_bwd: window %d must fit in the input (%d, %d, %d)", k, D, H, W);
  return LT_OK;
}


// ---- batch image ingest ---------------------------------------------------------------------------
// Host batches arrive as the dataset leaves them: [N][H][W][C] (HWC) uint8 / float32 / float64 (datasets/utils.py:24).
// The reference transposes to CHW and casts on the CPU (image_batch_to_torch, img.py:96-99) after normalising per image
// on the CPU as well (normalize_image, img.py:102-110).  Here the raw HWC buffer is uploaded once and this kernel does
// transpose + cast (+ per-channel 256-entry table for uint8: the table is built on the host in float64 with the
// reference's formula and rounded once, so the result equals normalize_image(...).astype(float32) bit for bit).
template <typename T>
__global__ void __launch_bounds__(256) images_hwc_to_nchw_kernel(const T* __restrict__ in, const float* __restrict__ lut,
                                                                 float* __restrict__ out, long N, int C, long hw) {
  __shared__ float s_lut[4 * 256];
  const bool use_lut = lut != nullptr && sizeof(T) == 1;
  if (use_lut) {
    for (int i = threadIdx.x; i < C * 256; i += blockDim.x) s_lut[i] = lut[i];
    __syncthreads();
  }
  const long total = N * hw;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long n = i / hw, r = i % hw;
    const T* src = in + i * C;
    for (int c = 0; c < C; ++c) {
      float v;
      if (sizeof(T) == 1) {
        const unsigned u = (unsigned)src[c];
        v = use_lut ? s_lut[c * 256 + u] : (float)u;
      } else {
        v = (float)src[c];     // float64 -> float32 round-to-nearest, as ndarray.astype / Tensor.float()
      }
      out[(n * C + c) * hw + r] = v;
    }
  }
}

// ---- layout / format conversion -------------------------------------------------------------------
__global__ void __launch_bounds__(256) nchw_to_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                           int N, int C, int H, int W, int Cp) {
  const long hw = (long)H * W;
  const long total = (long)N * hw;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long n = i / hw, r = i % hw;
    float* o = out + i * Cp;
    for (int c = 0; c < Cp; ++c) o[c] = (c < C) ? __ldg(in + (n * C + c) * hw + r) : 0.0f;
  }
}

// Stem input packing: images [N][3][H][W] fp32 -> 2x2 space-to-depth, channels-last split-fp16 [N][H/2][W/2][32]
// with channel (r*2 + s)*3 + c = in[c][2y + r][2x + s] (12 used, 20 zero), so that the 7x7 stride-2 stem conv
// (pose_resnet.py:205) becomes a 4x4 stride-1 conv with 32 input channels on the tensor-core kernel.
__global__ void __launch_bounds__(256) stem_s2d_kernel(const float* __restrict__ in, sh_t* __restrict__ out, int N, int C, int H, int W) {
  const int H2 = H / 2, W2 = W / 2;
  const long total = (long)N * H2 * W2;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int x = (int)(i % W2);
    const int y = (int)((i / W2) % H2);
    const long n = i / ((long)W2 * H2);
    sh_t hi[32], lo[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) { hi[k] = __float2half_rn(0.f); lo[k] = hi[k]; }
    for (int r = 0; r < 2; ++r)
      for (int s = 0; s < 2; ++s)
        for (int c = 0; c < C; ++c) {
          const float v = __ldg(in + ((n * C + c) * H + (2 * y + r)) * W + (2 * x + s));
          split_s32(v, hi[(r * 2 + s) * C + c], lo[(r * 2 + s) * C + c]);
        }
    uint4* dst = reinterpret_cast<uint4*>(out + i * 64);
    const uint4* h4 = reinterpret_cast<const uint4*>(hi);
    const uint4* l4 = reinterpret_cast<const uint4*>(lo);
#pragma unroll
    for (int k = 0; k < 4; ++k) { dst[k] = h4[k]; dst[4 + k] = l4[k]; }
  }
}

__global__ void __launch_bounds__(256) f32_to_s32_kernel(const float* __restrict__ in, sh_t* __restrict__ out, long pixels, int C) {
  const int c4n = C / 4;
  const long total = pixels * c4n;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long pix = i / c4n;
    const int c = (int)(i % c4n) * 4;
    store_s32x4(out + pix * 2 * C, c, __ldg(reinterpret_cast<const float4*>(in + pix * C + c)));
  }
}

// [P][C] float32 (any C) -> [P][CP] split-fp16 of S * x, S = weight_pow2_scale(absmax_bits) (1 without bits), channels C..CP-1 zero;
// inv_scale (optional) receives 1 / S
__global__ void __launch_bounds__(256) f32_to_s32_scaled_kernel(const float* __restrict__ in, sh_t* __restrict__ out, long pixels, int C,
                                                                int CP, const unsigned* __restrict__ absmax_bits, float* __restrict__ inv_scale) {
  const float S = weight_pow2_scale(absmax_bits);
  if (inv_scale && blockIdx.x == 0 && threadIdx.x == 0) *inv_scale = 1.0f / S;
  const int c4n = CP / 4;
  const long total = pixels * c4n;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long pix = i / c4n;
    const int c = (int)(i % c4n) * 4;
    const float* src = in + pix * C;
    float4 v;
    v.x = c < C ? __ldg(src + c) * S : 0.0f;
    v.y = c + 1 < C ? __ldg(src + c + 1) * S : 0.0f;
    v.z = c + 2 < C ? __ldg(src + c + 2) * S : 0.0f;
    v.w = c + 3 < C ? __ldg(src + c + 3) * S : 0.0f;
    store_s32x4(out + pix * 2 * CP, c, v);
  }
}

__global__ void __launch_bounds__(256) s32_to_f32_kernel(const sh_t* __restrict__ in, float* __restrict__ out, long pixels, int C) {
  const int c4n = C / 4;
  const long total = pixels * c4n;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long pix = i / c4n;
    const int c = (int)(i % c4n) * 4;
    *reinterpret_cast<float4*>(out + pix * C + c) = load_s32x4(in + pix * 2 * C, c);
  }
}

// [N][P][Cs] -> [N][C][P], 32x32 tiles through shared memory
__global__ void __launch_bounds__(256) cl_to_cf_kernel(const float* __restrict__ in, float* __restrict__ out, long P, int Cs, int C) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const long p0 = (long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int r = ty; r < 32; r += 8) {
    const long pp = p0 + r;
    const int c = c0 + tx;
    tile[r][tx] = (pp < P && c < C) ? __ldg(in + ((long)n * P + pp) * Cs + c) : 0.0f;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r;
    const long pp = p0 + tx;
    if (c < C && pp < P) out[((long)n * C + c) * P + pp] = tile[tx][r];
  }
}

static inline unsigned grid_for(long total, int per_block = 256) {
  long b = (total + per_block - 1) / per_block;
  const long cap = (long)sm_count() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}

// ---- weight preparation (engine.prepare): framework-layout filters -> canonical [tap][CinP][CoutP] float32, BN folding ----------
// Element (td, th, tw, ci, co) of the source filter sits at w[base + td*s_td + th*s_th + tw*s_tw + ci*s_ci + co*s_co]: plain convs
// (Cout, Cin, KD, KH, KW), transposed convs (Cin, Cout, ...) and their stride phases (a sub-lattice of taps walked with negative
// strides) are all affine maps, so ONE kernel replaces the permute / slice / pad / contiguous chain.
__global__ void __launch_bounds__(256) absmax_kernel(const float* __restrict__ w, long n, unsigned* __restrict__ out_bits) {
  // max |w| over the finite elements only: each non-finite element is skipped on its own, so an Inf does not hide the finite
  // values its warp read (fmaxf already drops NaN)
  float m = 0.0f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const float a = fabsf(w[i]);
    if (a < INFINITY) m = fmaxf(m, a);
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0 && m > 0.0f) atomicMax(out_bits, __float_as_uint(m));   // non-negative floats order like their bits
}

__global__ void __launch_bounds__(256) gather_weights_kernel(const float* __restrict__ w, long base, long s_td, long s_th, long s_tw, long s_ci,
                                                             long s_co, int KH, int KW, int Cin, int CinP, int Cout, int CoutP, long total,
                                                             const unsigned* __restrict__ absmax_bits, float* __restrict__ out, int out_ld,
                                                             int out_col0) {
  const float S = weight_pow2_scale(absmax_bits);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int co = (int)(i % CoutP);
    long r = i / CoutP;
    const int ci = (int)(r % CinP);
    const int tap = (int)(r / CinP);
    const int tw = tap % KW, th = (tap / KW) % KH, td = tap / (KW * KH);
    out[((long)tap * CinP + ci) * out_ld + out_col0 + co] =
        (ci < Cin && co < Cout) ? w[base + td * s_td + th * s_th + tw * s_tw + ci * s_ci + co * s_co] * S : 0.0f;
  }
}

// y = acc * scale + shift with scale = gamma / sqrt(var + eps), shift = beta - mean * scale (+ conv_bias * scale); double arithmetic,
// rounded once.  Any of gamma / beta / bias may be null; mean == null means "no BatchNorm" (scale 1, shift = bias).
// accum_gain(steps) (common.cuh): compensates the expected shrinkage of a sum accumulated by `steps` truncating tensor-core additions;
// 1 for the exact-fp32 kernels.
__global__ void fold_bn_kernel(const float* gamma, const float* beta, const float* mean, const float* var, const float* bias, double eps,
                               int C, int CP, const unsigned* absmax_bits, double accum_gain, float* scale, float* shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= CP) return;
  const double inv_s = 1.0 / (double)weight_pow2_scale(absmax_bits);   // the packed filter carries S: acc = S * sum x w
  double sc = 0.0, sh = 0.0;
  if (c < C) {
    if (mean) {
      sc = (gamma ? (double)gamma[c] : 1.0) / sqrt((double)var[c] + eps);
      sh = (beta ? (double)beta[c] : 0.0) - (double)mean[c] * sc;
      if (bias) sh += (double)bias[c] * sc;
    } else {
      sc = 1.0;
      sh = bias ? (double)bias[c] : 0.0;
    }
  }
  scale[c] = (float)(sc * inv_s * accum_gain);
  shift[c] = (float)sh;
}

// ---- multi-GPU feature exchange: this rank's feature maps -> the owner ranks' buffers (peer memory over NVLink) ----------
// src [B][Vl][row] (row = h*w*C floats); sample b belongs to rank b / per; dst buffer of owner o: [per][V][row], this rank's local
// view j is global view view_rank + j*G.  One CTA column per (sample, local view); float4 stores straight into peer memory.
struct PeerPtrs { float* p[8]; };
__global__ void __launch_bounds__(256) feature_scatter_kernel(const float* __restrict__ src, PeerPtrs peers, int Vl, int V, int G,
                                                              int view_rank, int per, long row4) {
  const int bv = blockIdx.y;
  const int b = bv / Vl, j = bv - b * Vl;
  const int owner = b / per, bl = b - owner * per, v = view_rank + j * G;
  const float4* s4 = reinterpret_cast<const float4*>(src) + (long)bv * row4;
  float4* d4 = reinterpret_cast<float4*>(peers.p[owner]) + ((long)bl * V + v) * row4;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < row4; i += (long)gridDim.x * blockDim.x) d4[i] = s4[i];
}

}  // namespace lt

extern "C" int lt_absmax_fwd(const float* w, long n, unsigned int* out_bits, void* stream) {
  using namespace lt;
  LT_REQUIRE(w && out_bits && n > 0, "absmax: bad arguments");
  cudaError_t e = cudaMemsetAsync(out_bits, 0, sizeof(unsigned int), (cudaStream_t)stream);
  if (e != cudaSuccess) return fail(LT_ERR_CUDA, "absmax: cudaMemsetAsync: %s", cudaGetErrorString(e));
  long blocks = (n + 255) / 256;
  if (blocks > 1024) blocks = 1024;
  absmax_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(w, n, out_bits);
  LT_CHECK_LAUNCH("absmax_kernel");
  return LT_OK;
}

extern "C" int lt_conv_gather_weights_fwd(const float* w, long base, long s_td, long s_th, long s_tw, long s_ci, long s_co, int KD, int KH,
                                          int KW, int Cin, int CinP, int Cout, int CoutP, const unsigned int* absmax_bits, float* out,
                                          int out_ld, int out_col0, void* stream) {
  using namespace lt;
  LT_REQUIRE(w && out && KD > 0 && KH > 0 && KW > 0 && Cin > 0 && Cout > 0 && CinP >= Cin && CoutP >= Cout, "conv_gather_weights: bad arguments");
  if (out_ld <= 0) out_ld = CoutP;
  LT_REQUIRE(out_col0 >= 0 && out_col0 + CoutP <= out_ld, "conv_gather_weights: column block [%d, %d) exceeds the row length %d", out_col0, out_col0 + CoutP, out_ld);
  const long total = (long)KD * KH * KW * CinP * CoutP;
  long blocks = (total + 255) / 256;
  if (blocks > 4096) blocks = 4096;
  gather_weights_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(w, base, s_td, s_th, s_tw, s_ci, s_co, KH, KW, Cin, CinP, Cout, CoutP,
                                                                              total, absmax_bits, out, out_ld, out_col0);
  LT_CHECK_LAUNCH("gather_weights_kernel");
  return LT_OK;
}

extern "C" int lt_fold_bn_fwd(const float* gamma, const float* beta, const float* mean, const float* var, const float* conv_bias, float eps,
                              int C, int CP, const unsigned int* absmax_bits, int accum_steps, float* scale, float* shift, void* stream) {
  using namespace lt;
  LT_REQUIRE(scale && shift && C > 0 && CP >= C && (!mean || var) && accum_steps >= 0, "fold_bn: bad arguments");
  fold_bn_kernel<<<ceil_div(CP, 128), 128, 0, (cudaStream_t)stream>>>(gamma, beta, mean, var, conv_bias, (double)eps, C, CP, absmax_bits,
                                                                   accum_gain((double)accum_steps), scale, shift);
  LT_CHECK_LAUNCH("fold_bn_kernel");
  return LT_OK;
}

extern "C" int lt_feature_scatter_fwd(const float* feats, float* const* peer_buffers, int n_peers, int view_rank, int B, int V_local,
                                      int V, long row_elems, void* stream) {
  using namespace lt;
  LT_REQUIRE(feats && peer_buffers && n_peers >= 1 && n_peers <= 8, "feature_scatter: need 1..8 peer buffers");
  LT_REQUIRE(B % n_peers == 0 && row_elems % 4 == 0 && V_local * n_peers == V, "feature_scatter: bad sizes (B=%d G=%d Vl=%d V=%d)", B, n_peers, V_local, V);
  PeerPtrs pp;
  for (int i = 0; i < 8; ++i) pp.p[i] = i < n_peers ? peer_buffers[i] : nullptr;
  const long row4 = row_elems / 4;
  int gx = (int)((row4 + 255) / 256);
  if (gx > 64) gx = 64;
  dim3 grid((unsigned)gx, (unsigned)(B * V_local));
  feature_scatter_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(feats, pp, V_local, V, n_peers, view_rank, B / n_peers, row4);
  LT_CHECK_LAUNCH("feature_scatter_kernel");
  return LT_OK;
}

namespace lt {
}  // namespace lt

using namespace lt;

extern "C" int lt_coord_volume_fwd(const float* position, const float* center, const float* step, const float* rot,
                                   float* out, int B, int n, int transfer_cmu, void* stream) {
  LT_REQUIRE(position && center && step && rot && out, "coord_volume: null pointer");
  LT_REQUIRE(B > 0 && n > 1, "coord_volume: bad size B=%d n=%d", B, n);
  coord_volume_kernel<<<grid_for((long)B * n * n * n), 256, 0, (cudaStream_t)stream>>>(position, center, step, rot, out, B, n, transfer_cmu);
  LT_CHECK_LAUNCH("coord_volume_kernel");
  return LT_OK;
}

extern "C" int lt_cuboid_from_keypoints_fwd(const float* keypoints_3d, int B, int J, int kind, double cuboid_side, float* center,
                                            float* position, void* stream) {
  LT_REQUIRE(keypoints_3d && center && position, "cuboid_from_keypoints: null pointer");
  LT_REQUIRE(kind == LT_KIND_MPII || kind == LT_KIND_COCO, "cuboid_from_keypoints: unknown skeleton kind %d", kind);
  LT_REQUIRE(B > 0 && J > (kind == LT_KIND_COCO ? 12 : 6), "cuboid_from_keypoints: bad size B=%d J=%d for skeleton kind %d", B, J, kind);
  cuboid_from_keypoints_kernel<<<ceil_div(B * 3, 128), 128, 0, (cudaStream_t)stream>>>(keypoints_3d, B, J, kind, cuboid_side, center,
                                                                                      position);
  LT_CHECK_LAUNCH("cuboid_from_keypoints_kernel");
  return LT_OK;
}

extern "C" int lt_maxpool_fwd(const void* in, void* out, int format, int N, int ID, int IH, int IW, int C, int kd, int kh,
                              int kw, int sd, int sh, int sw, int pd, int ph, int pw, int OD, int OH, int OW, void* stream) {
  LT_REQUIRE(in && out, "maxpool: null pointer");
  LT_REQUIRE(C % 4 == 0, "maxpool: C %% 4 != 0");
  LT_REQUIRE(format == LT_FMT_F32 || C % 32 == 0, "maxpool: split-fp16 needs C %% 32 == 0");
  PoolParams p{in, out, format, N, ID, IH, IW, C, kd, kh, kw, sd, sh, sw, pd, ph, pw, OD, OH, OW};
  maxpool_kernel<<<grid_for((long)N * OD * OH * OW * (C / 4)), 256, 0, (cudaStream_t)stream>>>(p);
  LT_CHECK_LAUNCH("maxpool_kernel");
  return LT_OK;
}

extern "C" int lt_maxpool3d_bwd(const float* x, const float* grad_y, float* grad_x, int N, int C, int D, int H, int W, long xs_n, long xs_c,
                                long xs_d, long xs_h, long xs_w, long gs_n, long gs_c, long gs_d, long gs_h, long gs_w, int k, void* stream) {
  const int rc = pool3d_bwd_check(x, grad_y, grad_x, N, C, D, H, W, k);
  if (rc != LT_OK) return rc;
  const Pool3dBwdParams p{x, grad_y, grad_x, N, C, D, H, W, k, {xs_n, xs_c, xs_d, xs_h, xs_w}, {gs_n, gs_c, gs_d, gs_h, gs_w}};
  const long total = (long)N * C * D * H * W;
  pool3d_bwd_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>(p, total);
  LT_CHECK_LAUNCH("pool3d_bwd_kernel");
  return LT_OK;
}

extern "C" int lt_test_maxpool3d_bwd_host(const float* x, const float* grad_y, float* grad_x, int N, int C, int D, int H, int W, long xs_n,
                                          long xs_c, long xs_d, long xs_h, long xs_w, long gs_n, long gs_c, long gs_d, long gs_h, long gs_w, int k) {
  const int rc = pool3d_bwd_check(x, grad_y, grad_x, N, C, D, H, W, k);
  if (rc != LT_OK) return rc;
  const Pool3dBwdParams p{x, grad_y, grad_x, N, C, D, H, W, k, {xs_n, xs_c, xs_d, xs_h, xs_w}, {gs_n, gs_c, gs_d, gs_h, gs_w}};
  const long total = (long)N * C * D * H * W;
  for (long i = 0; i < total; ++i) pool3d_bwd_item(p, i);
  return LT_OK;
}

extern "C" int lt_nchw_to_nhwc_f32(const float* in, float* out, int N, int C, int H, int W, int Cp, void* stream) {
  LT_REQUIRE(in && out && Cp >= C, "nchw_to_nhwc: bad arguments");
  nchw_to_nhwc_kernel<<<grid_for((long)N * H * W), 256, 0, (cudaStream_t)stream>>>(in, out, N, C, H, W, Cp);
  LT_CHECK_LAUNCH("nchw_to_nhwc_kernel");
  return LT_OK;
}

extern "C" int lt_images_hwc_to_nchw_fwd(const void* in, int in_dtype, const float* lut, float* out, int N, int C, int H, int W,
                                         void* stream) {
  LT_REQUIRE(in && out && N > 0 && C > 0 && C <= 4 && H > 0 && W > 0, "images_hwc_to_nchw: bad arguments");
  LT_REQUIRE(in_dtype >= LT_IMG_U8 && in_dtype <= LT_IMG_F64, "images_hwc_to_nchw: unknown input dtype %d", in_dtype);
  LT_REQUIRE(lut == nullptr || in_dtype == LT_IMG_U8, "images_hwc_to_nchw: the table applies to uint8 input only");
  const long hw = (long)H * W;
  const unsigned grid = grid_for((long)N * hw);
  cudaStream_t st = (cudaStream_t)stream;
  if (in_dtype == LT_IMG_U8) images_hwc_to_nchw_kernel<unsigned char><<<grid, 256, 0, st>>>(reinterpret_cast<const unsigned char*>(in), lut, out, N, C, hw);
  else if (in_dtype == LT_IMG_F32) images_hwc_to_nchw_kernel<float><<<grid, 256, 0, st>>>(reinterpret_cast<const float*>(in), nullptr, out, N, C, hw);
  else images_hwc_to_nchw_kernel<double><<<grid, 256, 0, st>>>(reinterpret_cast<const double*>(in), nullptr, out, N, C, hw);
  LT_CHECK_LAUNCH("images_hwc_to_nchw_kernel");
  return LT_OK;
}

extern "C" int lt_stem_s2d_fwd(const float* in, void* out, int N, int C, int H, int W, void* stream) {
  LT_REQUIRE(in && out && C * 4 <= 32 && H % 2 == 0 && W % 2 == 0, "stem_s2d: need C <= 8 and even H, W");
  stem_s2d_kernel<<<grid_for((long)N * (H / 2) * (W / 2)), 256, 0, (cudaStream_t)stream>>>(in, reinterpret_cast<sh_t*>(out), N, C, H, W);
  LT_CHECK_LAUNCH("stem_s2d_kernel");
  return LT_OK;
}

extern "C" int lt_f32_to_s32(const float* in, void* out, long pixels, int C, void* stream) {
  LT_REQUIRE(in && out && C % 32 == 0, "f32_to_s32: C %% 32 != 0");
  f32_to_s32_kernel<<<grid_for(pixels * (C / 4)), 256, 0, (cudaStream_t)stream>>>(in, reinterpret_cast<sh_t*>(out), pixels, C);
  LT_CHECK_LAUNCH("f32_to_s32_kernel");
  return LT_OK;
}

extern "C" int lt_f32_to_s32_scaled(const float* in, void* out, long pixels, int C, int CP, const unsigned int* absmax_bits,
                                    float* inv_scale, void* stream) {
  LT_REQUIRE(in && out && C > 0 && CP >= C && CP % 32 == 0, "f32_to_s32_scaled: need C <= CP, CP %% 32 == 0");
  f32_to_s32_scaled_kernel<<<grid_for(pixels * (CP / 4)), 256, 0, (cudaStream_t)stream>>>(in, reinterpret_cast<sh_t*>(out), pixels, C, CP,
                                                                                         absmax_bits, inv_scale);
  LT_CHECK_LAUNCH("f32_to_s32_scaled_kernel");
  return LT_OK;
}

extern "C" int lt_s32_to_f32(const void* in, float* out, long pixels, int C, void* stream) {
  LT_REQUIRE(in && out && C % 32 == 0, "s32_to_f32: C %% 32 != 0");
  s32_to_f32_kernel<<<grid_for(pixels * (C / 4)), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const sh_t*>(in), out, pixels, C);
  LT_CHECK_LAUNCH("s32_to_f32_kernel");
  return LT_OK;
}

extern "C" int lt_cl_to_cf_f32(const float* in, float* out, int N, long P, int Cs, int C, void* stream) {
  LT_REQUIRE(in && out && C <= Cs && N <= 65535, "cl_to_cf: bad arguments");
  dim3 grid((unsigned)((P + 31) / 32), (unsigned)((C + 31) / 32), (unsigned)N);
  cl_to_cf_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, out, P, Cs, C);
  LT_CHECK_LAUNCH("cl_to_cf_kernel");
  return LT_OK;
}
