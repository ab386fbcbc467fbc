// BatchNorm for training (nn.BatchNorm2d / BatchNorm3d in train and eval mode, pose_resnet.py and v2v.py) fused with the ReLU after
// it and the residual add of a residual unit: y = act(gamma (x - mean) invstd + beta [+ r]), and its backward.
//
// Every map is float32 channels-last [M][C], M = N*D*H*W, C % 4 == 0 (float4 accesses along C).  A CTA of kBnThreads threads is a
// (tc, ry) grid: tc threads over float4 columns of one channel block (tc = min(C/4, 32)), ry = kBnThreads / tc rows at a time.
//   bn_reduce_kernel<0>     forward statistics: per (row split, channel) the sums of d = x - x[0][c] and d^2 (shifted sums: no
//                           cancellation when |mean| >> std), accumulated in fp64 and summed over the CTA's rows in a fixed order;
//   bn_finalize_fwd_kernel  per channel: the splits merged in a fixed order (8 lanes, then the lanes in order) -> mean,
//                           invstd = 1 / sqrt(var_biased + eps) (0 when both are 0, as in torch), the running statistics (unbiased
//                           variance) and the apply coefficients; in eval mode the running statistics instead;
//   bn_apply_fwd_kernel     y = act(a (x - mean) + beta [+ r]), a = gamma invstd, act(NaN) = NaN as in torch.relu.  (x - mean) is
//                           formed first, as torch does: the folded form a x + (beta - a mean) loses ~log2(|mean| / std) bits of y;
//   bn_reduce_kernel<1>     backward: per (row split, channel) the sums of g' and g' (x - mean), g' = g [!(y <= 0)] under ReLU
//                           (torch's threshold_backward: a NaN output passes its gradient), in fp64;
//   bn_finalize_bwd_kernel  dbeta = sum g', dgamma = invstd sum g' (x - mean) and the apply coefficients;
//   bn_apply_bwd_kernel     dx = a (g' - sum g' / M - xhat sum g' xhat / M) (train) or a g' (eval); dr = g' when asked for.
// No floating-point atomics and no host synchronisation: the launch plan (bn_plan, lt_batch_norm_plan) depends on M, C and the SM
// count only, so results repeat bit for bit on one device.
#include "common.cuh"
#include <math.h>

namespace lt {

constexpr int kBnThreads = 256;
constexpr int kBnUnroll = 4;        // rows a thread loads before it uses any of them (memory-level parallelism)
constexpr int kBnCtasPerSm = 4;     // reduce / apply CTAs per SM and wave
constexpr int kBnMinSteps = 16;     // a row split covers at least 16 row steps of its CTA
constexpr int kBnMaxCtas = 1024;    // channel blocks x row splits of a reduce pass: one wave on up to 256 SMs
constexpr int kBnLanes = 8;         // finalize: lanes per channel that merge the splits (then merged in lane order)

struct BnGeom {
  int C4, tc, ry, cblocks;
};

static inline BnGeom bn_geom(int C) {
  BnGeom g;
  g.C4 = C / 4;
  g.tc = g.C4 < 32 ? g.C4 : 32;
  g.ry = kBnThreads / g.tc;
  g.cblocks = ceil_div(g.C4, g.tc);
  return g;
}

// Upper bound of the row splits (what the workspace holds): device independent.
static inline int bn_max_splits(long M, int C) {
  const BnGeom g = bn_geom(C);
  const long by_rows = (M + (long)g.ry * kBnMinSteps - 1) / ((long)g.ry * kBnMinSteps);
  const long by_ctas = (kBnMaxCtas + g.cblocks - 1) / g.cblocks;
  const long s = by_rows < by_ctas ? by_rows : by_ctas;
  return s < 1 ? 1 : (int)s;
}

// The launch plan of both directions for `sms` SMs: reduce passes of one wave of kBnCtasPerSm CTAs per SM within bn_max_splits,
// each split then taking ceil(M / splits) rows (which can leave fewer splits); apply passes of about two waves along M.
static inline lt_batch_norm_launch_plan bn_plan(long M, int C, int sms) {
  const BnGeom g = bn_geom(C);
  if (sms <= 0) sms = 132;
  lt_batch_norm_launch_plan p;
  p.tc = g.tc;
  p.ry = g.ry;
  p.cblocks = g.cblocks;
  p.want_splits = ceil_div((long)sms * kBnCtasPerSm, g.cblocks);
  if (p.want_splits < 1) p.want_splits = 1;
  p.max_splits = bn_max_splits(M, C);
  const int s = p.want_splits < p.max_splits ? p.want_splits : p.max_splits;
  p.rows_per_split = (M + s - 1) / s;
  p.splits = (int)((M + p.rows_per_split - 1) / p.rows_per_split);
  const long by_rows = (M + (long)g.ry * kBnUnroll - 1) / ((long)g.ry * kBnUnroll);
  long rb = ((long)sms * kBnCtasPerSm * 2 + g.cblocks - 1) / g.cblocks;   // two waves
  if (rb > by_rows) rb = by_rows;
  if (rb > 65535) rb = 65535;
  p.row_blocks = rb < 1 ? 1 : (int)rb;
  return p;
}

// workspace: fp64 partials [splits][2][C], then float coefficients [5][C]
static inline size_t bn_partial_bytes(long M, int C) { return (size_t)bn_max_splits(M, C) * 2 * C * sizeof(double); }

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float f4(const float4& v, int k) { return k == 0 ? v.x : k == 1 ? v.y : k == 2 ? v.z : v.w; }

// grid (cblocks, splits), block (tc, ry).  MODE 0: sums of x - x[0][c] and its square.  MODE 1: sums of g' and g' (x - mean).
// part[split][0|1][C] receives the CTA's sums.
template <int MODE, bool RELU>
__global__ void __launch_bounds__(kBnThreads) bn_reduce_kernel(const float* __restrict__ x, const float* __restrict__ gy,
                                                               const float* __restrict__ y, const float* __restrict__ mean, long M,
                                                               int C, long rows_per_split, double* __restrict__ part) {
  __shared__ double s[2][kBnThreads * 4];
  const int tc = blockDim.x, ry = blockDim.y, tx = threadIdx.x, ty = threadIdx.y;
  const int c4 = blockIdx.x * tc + tx;
  const bool on = c4 < (C >> 2);
  const long r0 = (long)blockIdx.y * rows_per_split;
  const long r1 = r0 + rows_per_split < M ? r0 + rows_per_split : M;
  double a0[4] = {0.0, 0.0, 0.0, 0.0}, a1[4] = {0.0, 0.0, 0.0, 0.0};
  if (on) {
    double ref[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) ref[k] = (double)(MODE == 0 ? __ldg(x + 4 * c4 + k) : __ldg(mean + 4 * c4 + k));
    for (long rb = r0 + ty; rb < r1; rb += (long)ry * kBnUnroll) {
      float4 xv[kBnUnroll], gv[kBnUnroll], yv[kBnUnroll];
#pragma unroll
      for (int u = 0; u < kBnUnroll; ++u) {
        const long r = rb + (long)u * ry;
        const float4 one = make_float4(1.0f, 1.0f, 1.0f, 1.0f);
        xv[u] = gv[u] = yv[u] = one;
        if (r < r1) {
          const long off = r * C + 4 * c4;
          xv[u] = ld4(x + off);
          if (MODE == 1) gv[u] = ld4(gy + off);
          if (MODE == 1 && RELU) yv[u] = ld4(y + off);
        }
      }
#pragma unroll
      for (int u = 0; u < kBnUnroll; ++u) {
        if (rb + (long)u * ry >= r1) break;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const double dx = (double)f4(xv[u], k) - ref[k];      // exact: the difference of two floats
          if (MODE == 0) {
            a0[k] += dx;
            a1[k] = fma(dx, dx, a1[k]);
          } else {
            const double g = !(f4(yv[u], k) <= 0.0f) ? (double)f4(gv[u], k) : 0.0;
            a0[k] += g;
            a1[k] = fma(g, dx, a1[k]);
          }
        }
      }
    }
  }
  const int slot = (ty * tc + tx) * 4;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    s[0][slot + k] = a0[k];
    s[1][slot + k] = a1[k];
  }
  __syncthreads();
  // the ry row groups of each (sum, channel) added in row-group order
  for (int t = ty * tc + tx; t < 2 * tc * 4; t += tc * ry) {
    const int which = t / (tc * 4), col = t % (tc * 4);
    double acc = 0.0;
    for (int j = 0; j < ry; ++j) acc += s[which][j * tc * 4 + col];
    const int c = blockIdx.x * tc * 4 + col;
    if (c < C) part[((long)blockIdx.y * 2 + which) * C + c] = acc;
  }
}

// Sums of the two partials of channel c over the splits: lane l of kBnLanes takes splits l, l + kBnLanes, ...; the lanes are then added in
// lane order.  block (32, kBnLanes); returns false for the threads that stop here (lanes > 0, channels >= C).
__device__ __forceinline__ bool bn_merge_splits(const double* __restrict__ part, int splits, int C, int c, double& s1, double& s2) {
  __shared__ double sh[2][kBnLanes][32];
  s1 = s2 = 0.0;
  if (c < C)
    for (int sp = threadIdx.y; sp < splits; sp += kBnLanes) {
      s1 += part[((long)sp * 2) * C + c];
      s2 += part[((long)sp * 2 + 1) * C + c];
    }
  sh[0][threadIdx.y][threadIdx.x] = s1;
  sh[1][threadIdx.y][threadIdx.x] = s2;
  __syncthreads();
  if (threadIdx.y != 0 || c >= C) return false;
  s1 = s2 = 0.0;
#pragma unroll
  for (int l = 0; l < kBnLanes; ++l) {
    s1 += sh[0][l][threadIdx.x];
    s2 += sh[1][l][threadIdx.x];
  }
  return true;
}

// block (32, kBnLanes) per 32 channels.  Training: merge the splits (fixed order) -> save_mean / save_invstd, running statistics,
// coefficients.  Eval: the running statistics.  coef[0..2][C] = mean, a = gamma invstd, beta.
__global__ void __launch_bounds__(32 * kBnLanes) bn_finalize_fwd_kernel(
    const double* __restrict__ part, int splits, const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
    float* __restrict__ running_mean, float* __restrict__ running_var, float* __restrict__ save_mean, float* __restrict__ save_invstd,
    float* __restrict__ coef, long M, int C, float eps, float momentum, int training) {
  const int c = blockIdx.x * 32 + threadIdx.x;
  double s1, s2;
  if (!bn_merge_splits(part, training ? splits : 0, C, c, s1, s2)) return;
  float mean_f, invstd_f;
  if (training) {
    const double dm = s1 / (double)M;
    double var = s2 / (double)M - dm * dm;
    if (var < 0.0) var = 0.0;
    const double mean = (double)x[c] + dm;
    mean_f = (float)mean;
    // a constant channel with eps = 0 normalises with invstd 0, as torch's batch statistics do (y = beta, dx = dgamma = 0)
    invstd_f = var == 0.0 && eps == 0.0f ? 0.0f : (float)(1.0 / sqrt(var + (double)eps));
    const float var_unbiased = (float)(var * ((double)M / (double)(M - 1)));
    running_mean[c] = momentum * mean_f + (1.0f - momentum) * running_mean[c];
    running_var[c] = momentum * var_unbiased + (1.0f - momentum) * running_var[c];
  } else {
    mean_f = running_mean[c];
    invstd_f = (float)(1.0 / sqrt((double)running_var[c] + (double)eps));
  }
  save_mean[c] = mean_f;
  save_invstd[c] = invstd_f;
  coef[c] = mean_f;
  coef[C + c] = gamma[c] * invstd_f;
  coef[2 * C + c] = beta[c];
}

// grid (cblocks, row blocks), block (tc, ry): y = act(a (x - mean) + beta [+ r])
template <bool RES, bool RELU>
__global__ void __launch_bounds__(kBnThreads) bn_apply_fwd_kernel(const float* __restrict__ x, const float* __restrict__ r,
                                                                  const float* __restrict__ coef, float* __restrict__ y, long M, int C) {
  const int c4 = blockIdx.x * blockDim.x + threadIdx.x;
  if (c4 >= (C >> 2)) return;
  float mu[4], a[4], b[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    mu[k] = coef[4 * c4 + k];
    a[k] = coef[C + 4 * c4 + k];
    b[k] = coef[2 * C + 4 * c4 + k];
  }
  const long step = (long)gridDim.y * blockDim.y;
  for (long rb = (long)blockIdx.y * blockDim.y + threadIdx.y; rb < M; rb += step * kBnUnroll) {
    float4 v[kBnUnroll], rv[kBnUnroll];
#pragma unroll
    for (int u = 0; u < kBnUnroll; ++u) {
      const long row = rb + u * step;
      v[u] = rv[u] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      if (row < M) {
        v[u] = ld4(x + row * C + 4 * c4);
        if (RES) rv[u] = ld4(r + row * C + 4 * c4);
      }
    }
#pragma unroll
    for (int u = 0; u < kBnUnroll; ++u) {
      const long row = rb + u * step;
      if (row >= M) break;
      float o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        o[k] = fmaf(a[k], f4(v[u], k) - mu[k], b[k]);
        if (RES) o[k] += f4(rv[u], k);
        if (RELU) o[k] = o[k] < 0.0f ? 0.0f : o[k];    // NaN stays NaN, as torch.relu
      }
      st4(y + row * C + 4 * c4, make_float4(o[0], o[1], o[2], o[3]));
    }
  }
}

// block (32, kBnLanes) per 32 channels: dbeta, dgamma and coef[0..4][C] = mean, invstd, a, sum g' / M, dgamma / M (the last two 0 in eval mode).
__global__ void __launch_bounds__(32 * kBnLanes) bn_finalize_bwd_kernel(
    const double* __restrict__ part, int splits, const float* __restrict__ gamma, const float* __restrict__ save_mean,
    const float* __restrict__ save_invstd, float* __restrict__ grad_gamma, float* __restrict__ grad_beta, float* __restrict__ coef, long M,
    int C, int training) {
  const int c = blockIdx.x * 32 + threadIdx.x;
  double s1, s2;
  if (!bn_merge_splits(part, splits, C, c, s1, s2)) return;
  const float invstd = save_invstd[c];
  const double dg = s2 * (double)invstd;
  if (grad_beta) grad_beta[c] = (float)s1;
  if (grad_gamma) grad_gamma[c] = (float)dg;
  coef[c] = save_mean[c];
  coef[C + c] = invstd;
  coef[2 * C + c] = gamma[c] * invstd;
  coef[3 * C + c] = training ? (float)(s1 / (double)M) : 0.0f;
  coef[4 * C + c] = training ? (float)(dg / (double)M) : 0.0f;
}

// grid (cblocks, row blocks), block (tc, ry): dx = a (g' - k1 - xhat k2), xhat = (x - mean) invstd (training) or a g' (eval);
// dr = g' (DRES)
template <bool RELU, bool DRES>
__global__ void __launch_bounds__(kBnThreads) bn_apply_bwd_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                                                  const float* __restrict__ gy, const float* __restrict__ coef,
                                                                  float* __restrict__ gx, float* __restrict__ gr, long M, int C,
                                                                  int training) {
  const int c4 = blockIdx.x * blockDim.x + threadIdx.x;
  if (c4 >= (C >> 2)) return;
  float mu[4], is[4], a[4], k1[4], k2[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    mu[k] = coef[4 * c4 + k];
    is[k] = coef[C + 4 * c4 + k];
    a[k] = coef[2 * C + 4 * c4 + k];
    k1[k] = coef[3 * C + 4 * c4 + k];
    k2[k] = coef[4 * C + 4 * c4 + k];
  }
  const long step = (long)gridDim.y * blockDim.y;
  for (long rb = (long)blockIdx.y * blockDim.y + threadIdx.y; rb < M; rb += step * kBnUnroll) {
    float4 v[kBnUnroll], gv[kBnUnroll], yv[kBnUnroll];
#pragma unroll
    for (int u = 0; u < kBnUnroll; ++u) {
      const long row = rb + u * step;
      v[u] = gv[u] = yv[u] = make_float4(1.0f, 1.0f, 1.0f, 1.0f);
      if (row < M) {
        v[u] = ld4(x + row * C + 4 * c4);
        gv[u] = ld4(gy + row * C + 4 * c4);
        if (RELU) yv[u] = ld4(y + row * C + 4 * c4);
      }
    }
#pragma unroll
    for (int u = 0; u < kBnUnroll; ++u) {
      const long row = rb + u * step;
      if (row >= M) break;
      const float4 g = make_float4(!(yv[u].x <= 0.0f) ? gv[u].x : 0.0f, !(yv[u].y <= 0.0f) ? gv[u].y : 0.0f,
                                   !(yv[u].z <= 0.0f) ? gv[u].z : 0.0f, !(yv[u].w <= 0.0f) ? gv[u].w : 0.0f);
      if (DRES) st4(gr + row * C + 4 * c4, g);
      float o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float xhat = (f4(v[u], k) - mu[k]) * is[k];
        o[k] = training ? a[k] * (f4(g, k) - k1[k] - xhat * k2[k]) : a[k] * f4(g, k);   // eval: no x term, so a non-finite x stays local
      }
      st4(gx + row * C + 4 * c4, make_float4(o[0], o[1], o[2], o[3]));
    }
  }
}

static bool aligned16(const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static int bn_check_sizes(const char* fn, long M, int C, int training) {
  LT_REQUIRE(M > 0 && C > 0, "%s: bad sizes (M %ld, C %d)", fn, M, C);
  LT_REQUIRE(C % 4 == 0, "%s: C %% 4 != 0 (C %d)", fn, C);
  LT_REQUIRE(!training || M >= 2, "%s: training needs M >= 2 values per channel (M %ld)", fn, M);
  return LT_OK;
}

}  // namespace lt

using namespace lt;

extern "C" size_t lt_batch_norm_workspace_bytes(long M, int C) {
  if (M <= 0 || C <= 0 || C % 4) return 0;
  return bn_partial_bytes(M, C) + (size_t)5 * C * sizeof(float);
}

extern "C" int lt_batch_norm_plan(long M, int C, int sm_count, lt_batch_norm_launch_plan* plan) {
  LT_REQUIRE(plan && sm_count > 0, "batch_norm_plan: bad arguments");
  const int rc = bn_check_sizes("batch_norm_plan", M, C, 0);
  if (rc != LT_OK) return rc;
  *plan = bn_plan(M, C, sm_count);
  return LT_OK;
}

extern "C" int lt_batch_norm_fwd(const float* x, const float* residual, const float* gamma, const float* beta, float* running_mean,
                                 float* running_var, float* save_mean, float* save_invstd, float* y, long M, int C, float eps,
                                 float momentum, int training, int relu, void* workspace, size_t workspace_bytes, void* stream) {
  const int rc = bn_check_sizes("batch_norm_fwd", M, C, training);
  if (rc != LT_OK) return rc;
  LT_REQUIRE(x && gamma && beta && running_mean && running_var && save_mean && save_invstd && y && workspace,
             "batch_norm_fwd: null pointer");
  LT_REQUIRE(workspace_bytes >= lt_batch_norm_workspace_bytes(M, C), "batch_norm_fwd: workspace too small");
  LT_REQUIRE(aligned16(x) && aligned16(residual) && aligned16(y) && aligned16(workspace), "batch_norm_fwd: maps must be 16-byte aligned");
  LT_REQUIRE(eps >= 0.0f, "batch_norm_fwd: eps must be >= 0");
  const cudaStream_t s = (cudaStream_t)stream;
  const lt_batch_norm_launch_plan p = bn_plan(M, C, sm_count());
  double* part = reinterpret_cast<double*>(workspace);
  float* coef = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + bn_partial_bytes(M, C));
  const dim3 block(p.tc, p.ry);
  if (training) {
    bn_reduce_kernel<0, false><<<dim3(p.cblocks, p.splits), block, 0, s>>>(x, nullptr, nullptr, nullptr, M, C, p.rows_per_split, part);
    LT_CHECK_LAUNCH("bn_reduce_kernel");
  }
  bn_finalize_fwd_kernel<<<ceil_div(C, 32), dim3(32, kBnLanes), 0, s>>>(part, training ? p.splits : 0, x, gamma, beta, running_mean, running_var,
                                                           save_mean, save_invstd, coef, M, C, eps, momentum, training);
  LT_CHECK_LAUNCH("bn_finalize_fwd_kernel");
  const dim3 grid(p.cblocks, p.row_blocks);
  if (residual) {
    if (relu) bn_apply_fwd_kernel<true, true><<<grid, block, 0, s>>>(x, residual, coef, y, M, C);
    else bn_apply_fwd_kernel<true, false><<<grid, block, 0, s>>>(x, residual, coef, y, M, C);
  } else {
    if (relu) bn_apply_fwd_kernel<false, true><<<grid, block, 0, s>>>(x, nullptr, coef, y, M, C);
    else bn_apply_fwd_kernel<false, false><<<grid, block, 0, s>>>(x, nullptr, coef, y, M, C);
  }
  LT_CHECK_LAUNCH("bn_apply_fwd_kernel");
  return LT_OK;
}

extern "C" int lt_batch_norm_bwd(const float* x, const float* y, const float* grad_y, const float* gamma, const float* save_mean,
                                 const float* save_invstd, float* grad_x, float* grad_residual, float* grad_gamma, float* grad_beta, long M,
                                 int C, int training, int relu, void* workspace, size_t workspace_bytes, void* stream) {
  const int rc = bn_check_sizes("batch_norm_bwd", M, C, training);
  if (rc != LT_OK) return rc;
  LT_REQUIRE(x && grad_y && gamma && save_mean && save_invstd && grad_x && workspace, "batch_norm_bwd: null pointer");
  LT_REQUIRE(!relu || y, "batch_norm_bwd: null pointer (y is needed with relu)");
  LT_REQUIRE(workspace_bytes >= lt_batch_norm_workspace_bytes(M, C), "batch_norm_bwd: workspace too small");
  LT_REQUIRE(aligned16(x) && aligned16(y) && aligned16(grad_y) && aligned16(grad_x) && aligned16(grad_residual) && aligned16(workspace),
             "batch_norm_bwd: maps must be 16-byte aligned");
  const cudaStream_t s = (cudaStream_t)stream;
  const lt_batch_norm_launch_plan p = bn_plan(M, C, sm_count());
  double* part = reinterpret_cast<double*>(workspace);
  float* coef = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + bn_partial_bytes(M, C));
  const dim3 block(p.tc, p.ry);
  const dim3 rgrid(p.cblocks, p.splits);
  if (relu) bn_reduce_kernel<1, true><<<rgrid, block, 0, s>>>(x, grad_y, y, save_mean, M, C, p.rows_per_split, part);
  else bn_reduce_kernel<1, false><<<rgrid, block, 0, s>>>(x, grad_y, nullptr, save_mean, M, C, p.rows_per_split, part);
  LT_CHECK_LAUNCH("bn_reduce_kernel");
  bn_finalize_bwd_kernel<<<ceil_div(C, 32), dim3(32, kBnLanes), 0, s>>>(part, p.splits, gamma, save_mean, save_invstd, grad_gamma, grad_beta, coef,
                                                           M, C, training);
  LT_CHECK_LAUNCH("bn_finalize_bwd_kernel");
  const dim3 grid(p.cblocks, p.row_blocks);
  if (relu) {
    if (grad_residual) bn_apply_bwd_kernel<true, true><<<grid, block, 0, s>>>(x, y, grad_y, coef, grad_x, grad_residual, M, C, training);
    else bn_apply_bwd_kernel<true, false><<<grid, block, 0, s>>>(x, y, grad_y, coef, grad_x, nullptr, M, C, training);
  } else {
    if (grad_residual) bn_apply_bwd_kernel<false, true><<<grid, block, 0, s>>>(x, nullptr, grad_y, coef, grad_x, grad_residual, M, C, training);
    else bn_apply_bwd_kernel<false, false><<<grid, block, 0, s>>>(x, nullptr, grad_y, coef, grad_x, nullptr, M, C, training);
  }
  LT_CHECK_LAUNCH("bn_apply_bwd_kernel");
  return LT_OK;
}
