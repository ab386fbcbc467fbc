// Kernels of the RANSAC triangulation baseline (RANSACTriangulationNet, triangulation.py:17-128):
//   - heat-map arg-max: the final conv's channels-last logits -> the raw (N, J, h, w) heat maps and the int64 key points of
//     torch.max's first maximal index, scaled to the image and truncated (triangulation.py:44-52); one read and one write of the maps
//   - RANSAC triangulation over host-drawn view pairs, then the inlier DLT and the optional Huber refinement of the reprojection
//     error (triangulation.py:72-128), one thread per (sample, joint), all in float64.
// This file is compiled with -fmad=false (build.py): no multiply-add is contracted, so the device code and the host test hook
// (lt_test_triangulate_ransac_host) run the same sequence of IEEE operations.
#include "common.cuh"
#include "dlt_common.cuh"
#include <math.h>

namespace lt {

// ---- heat-map arg-max ------------------------------------------------------------------------------------------------------

constexpr int kArgmaxWarps = 8;
constexpr int kArgmaxTilesPerWarp = 4;
constexpr int kArgmaxSlice = kArgmaxWarps * kArgmaxTilesPerWarp * 32;   // pixels per CTA

// torch.max's order on (value, index) (ATen GreaterOrNan): a NaN beats every number and the lower index wins between NaNs and
// between equal values.  `better(v, i, bv, bi)`: does (v, i) replace the current best (bv, bi); bi < 0 marks "none yet".
__host__ __device__ __forceinline__ bool argmax_better(float v, int i, float bv, int bi) {
  if (bi < 0) return true;
  if (isnan(bv)) return isnan(v) && i < bi;
  if (isnan(v)) return true;
  return v > bv || (v == bv && i < bi);
}

// grid (slices, N, channel groups of 32); lane = channel.  Each warp walks its 32-pixel tiles in pixel order: one coalesced
// 128-byte load per pixel, the lane's running best, and the tile transposed through shared memory into coalesced rows of the
// (N, J, h, w) heat maps.  The CTA's best per channel goes to part_val / part_idx [(n J + j) slices + slice].
__global__ void __launch_bounds__(kArgmaxWarps * 32) heatmap_argmax_kernel(const float* __restrict__ logits, int C,
                                                                           float* __restrict__ heat, float* __restrict__ part_val,
                                                                           int* __restrict__ part_idx, int J, int hw, int slices) {
  __shared__ float tile[kArgmaxWarps][32][33];
  __shared__ float best_v[kArgmaxWarps][32];
  __shared__ int best_i[kArgmaxWarps][32];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int n = blockIdx.y, ch0 = blockIdx.z * 32, ch = ch0 + lane;
  const bool live = ch < C;
  float bv = 0.0f;
  int bi = -1;
  for (int t = 0; t < kArgmaxTilesPerWarp; ++t) {
    const int p0 = blockIdx.x * kArgmaxSlice + (t * kArgmaxWarps + warp) * 32;
    if (p0 >= hw) break;
#pragma unroll 8
    for (int i = 0; i < 32; ++i) {
      const int q = p0 + i;
      float v = 0.0f;
      if (q < hw && live) {
        v = logits[((long)n * hw + q) * C + ch];
        if (argmax_better(v, q, bv, bi)) { bv = v; bi = q; }
      }
      tile[warp][i][lane] = v;
    }
    __syncwarp();
    const int q = p0 + lane;
    for (int c = 0; c < 32 && ch0 + c < J; ++c)
      if (q < hw) heat[((long)n * J + ch0 + c) * hw + q] = tile[warp][lane][c];
    __syncwarp();
  }
  best_v[warp][lane] = bv;
  best_i[warp][lane] = bi;
  __syncthreads();
  if (warp == 0 && ch < J) {
    for (int k = 1; k < kArgmaxWarps; ++k)
      if (best_i[k][lane] >= 0 && argmax_better(best_v[k][lane], best_i[k][lane], bv, bi)) { bv = best_v[k][lane]; bi = best_i[k][lane]; }
    const long o = ((long)n * J + ch) * slices + blockIdx.x;
    part_val[o] = bv;
    part_idx[o] = bi;
  }
}

// One thread per (n, j): the slices' bests merged in slice order, then x = trunc(float32(idx % w) * sx), y = trunc(float32(idx / w) * sy)
// (the float32 product the reference assigns into an int64 tensor, triangulation.py:49-52).
__global__ void __launch_bounds__(128) heatmap_argmax_finish_kernel(const float* __restrict__ part_val, const int* __restrict__ part_idx,
                                                                    long long* __restrict__ kp, int NJ, int slices, int w, float sx, float sy) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= NJ) return;
  float bv = 0.0f;
  int bi = -1;
  for (int s = 0; s < slices; ++s) {
    const long o = (long)t * slices + s;
    if (argmax_better(part_val[o], part_idx[o], bv, bi)) { bv = part_val[o]; bi = part_idx[o]; }
  }
  kp[(long)t * 2] = (long long)truncf(__fmul_rn((float)(bi % w), sx));
  kp[(long)t * 2 + 1] = (long long)truncf(__fmul_rn((float)(bi / w), sy));
}

// ---- RANSAC triangulation --------------------------------------------------------------------------------------------------

constexpr int kRefineIters = 1000;     // cap of the Levenberg-Marquardt iterations of the refinement
constexpr double kRefineStep = 1e-12;  // stop once an accepted step is below this fraction of |X|

__host__ __device__ __forceinline__ int popcount64(unsigned long long m) {
#ifdef __CUDA_ARCH__
  return __popcll(m);
#else
  return __builtin_popcountll(m);
#endif
}

struct RansacItem {
  const float* P;          // [V][3][4] of the sample
  const long long* kp;     // key point (x, y) of view v: kp[v * kp_stride], kp[v * kp_stride + 1]
  long kp_stride;
  int V;
};

// The two unweighted DLT rows of view v in float64 from the float32 matrix and the integer point, as numpy forms them
// (multiview.py:130-131): x * P[2] - P[0], y * P[2] - P[1].
__host__ __device__ __forceinline__ void ransac_rows(const RansacItem& it, int v, double r0[4], double r1[4]) {
  const float* P = it.P + v * 12;
  const double x = (double)it.kp[v * it.kp_stride], y = (double)it.kp[v * it.kp_stride + 1];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    r0[c] = x * (double)P[8 + c] - (double)P[c];
    r1[c] = y * (double)P[8 + c] - (double)P[4 + c];
  }
}

// DLT (multiview.py:113-138) on the views of `mask`, accumulated in ascending view order: X = u[0:3] / u[3] of the smallest
// eigenvector of A^T A.
__host__ __device__ __forceinline__ void ransac_dlt(const RansacItem& it, unsigned long long mask, double X[3]) {
  double M[4][4], E[4][4], u[4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) M[r][c] = 0.0;
  for (int v = 0; v < it.V; ++v) {
    if (!((mask >> v) & 1ull)) continue;
    double r0[4], r1[4];
    ransac_rows(it, v, r0, r1);
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) M[r][c] += r0[r] * r0[c] + r1[r] * r1[c];
  }
  dlt_column(E, dlt_jacobi(M, E), u);
  X[0] = u[0] / u[3];
  X[1] = u[1] / u[3];
  X[2] = u[2] / u[3];
}

// pi(X) of view v in float64 (multiview.py:89-110): (u / w, v / w) of P [X, 1]; returns w
__host__ __device__ __forceinline__ double ransac_project(const RansacItem& it, int v, const double X[3], double& pu, double& pv) {
  const float* P = it.P + v * 12;
  double p[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) p[r] = X[0] * (double)P[4 * r] + X[1] * (double)P[4 * r + 1] + X[2] * (double)P[4 * r + 2] + (double)P[4 * r + 3];
  pu = p[0] / p[2];
  pv = p[1] / p[2];
  return p[2];
}

// f_v^2 = (0.5 |p_v - pi(X)|)^2, the square of view v's reprojection error (multiview.py:186-193)
__host__ __device__ __forceinline__ double ransac_error2(const RansacItem& it, int v, const double X[3]) {
  double pu, pv;
  ransac_project(it, v, X, pu, pv);
  const double dx = (double)it.kp[v * it.kp_stride] - pu, dy = (double)it.kp[v * it.kp_stride + 1] - pv;
  return 0.25 * (dx * dx + dy * dy);
}

// The reference's refinement cost (least_squares(loss='huber', f_scale=1)): 1/2 sum over the inliers of rho(f_v^2), rho(z) = z for
// z <= 1, 2 sqrt(z) - 1 above.
__host__ __device__ __forceinline__ double ransac_cost(const RansacItem& it, unsigned long long mask, const double X[3]) {
  double s = 0.0;
  for (int v = 0; v < it.V; ++v) {
    if (!((mask >> v) & 1ull)) continue;
    const double z = ransac_error2(it, v, X);
    s += z <= 1.0 ? z : 2.0 * sqrt(z) - 1.0;
  }
  return 0.5 * s;
}

// Minimise ransac_cost from X by Levenberg-Marquardt on the 2 n_inliers residual components r_v = 0.5 (pi_v(X) - p_v), reweighted
// per iteration: weight 1 where f_v <= 1, 1 / f_v above, so that the weighted gradient sum w_v J_v^T r_v is the cost's own
// gradient.  The curvature of a view above f_v = 1 is the Gauss-Newton one of f_v itself, J^T (I - r r^T / f^2) J / f: plain
// reweighting (J^T J / f) overstates it along r and crawls where a view sits far out in the Huber branch.  Steps are accepted only where they lower the cost; the loop ends after kRefineIters iterations, on an accepted
// step below kRefineStep |X|, or when the damping cannot find a lower cost.  Deterministic: fixed order, no data-dependent
// precision.
__host__ __device__ __forceinline__ void ransac_refine(const RansacItem& it, unsigned long long mask, double X[3]) {
  double c = ransac_cost(it, mask, X);
  if (!isfinite(c)) return;
  double lambda = 1e-3, H[3][3], g[3];
  bool fresh = true;
  for (int iter = 0; iter < kRefineIters; ++iter) {
    if (fresh) {
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        g[r] = 0.0;
#pragma unroll
        for (int k = 0; k < 3; ++k) H[r][k] = 0.0;
      }
      for (int v = 0; v < it.V; ++v) {
        if (!((mask >> v) & 1ull)) continue;
        const float* P = it.P + v * 12;
        double pu, pv;
        const double w = ransac_project(it, v, X, pu, pv);
        const double ru = 0.5 * (pu - (double)it.kp[v * it.kp_stride]), rv = 0.5 * (pv - (double)it.kp[v * it.kp_stride + 1]);
        const double f = sqrt(ru * ru + rv * rv);
        const bool outer = f > 1.0;
        const double wt = outer ? 1.0 / f : 1.0;
        double ju[3], jv[3], jr[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          ju[k] = 0.5 * ((double)P[k] - pu * (double)P[8 + k]) / w;
          jv[k] = 0.5 * ((double)P[4 + k] - pv * (double)P[8 + k]) / w;
          jr[k] = outer ? (ju[k] * ru + jv[k] * rv) / f : 0.0;     // J^T r / f: the radial direction of the Huber branch
        }
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          g[r] += wt * (ju[r] * ru + jv[r] * rv);
#pragma unroll
          for (int k = 0; k < 3; ++k) H[r][k] += wt * (ju[r] * ju[k] + jv[r] * jv[k] - jr[r] * jr[k]);
        }
      }
      fresh = false;
    }
    // (H + lambda diag(H)) d = -g by the adjugate
    double A[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int k = 0; k < 3; ++k) A[r][k] = H[r][k] + (r == k ? lambda * H[r][k] : 0.0);
    const double c00 = A[1][1] * A[2][2] - A[1][2] * A[2][1], c01 = A[1][2] * A[2][0] - A[1][0] * A[2][2],
                 c02 = A[1][0] * A[2][1] - A[1][1] * A[2][0];
    const double det = A[0][0] * c00 + A[0][1] * c01 + A[0][2] * c02;
    const double c10 = A[0][2] * A[2][1] - A[0][1] * A[2][2], c11 = A[0][0] * A[2][2] - A[0][2] * A[2][0],
                 c12 = A[0][1] * A[2][0] - A[0][0] * A[2][1];
    const double c20 = A[0][1] * A[1][2] - A[0][2] * A[1][1], c21 = A[0][2] * A[1][0] - A[0][0] * A[1][2],
                 c22 = A[0][0] * A[1][1] - A[0][1] * A[1][0];
    const double d[3] = {-(c00 * g[0] + c10 * g[1] + c20 * g[2]) / det, -(c01 * g[0] + c11 * g[1] + c21 * g[2]) / det,
                         -(c02 * g[0] + c12 * g[1] + c22 * g[2]) / det};
    const double Xn[3] = {X[0] + d[0], X[1] + d[1], X[2] + d[2]};
    const double cn = ransac_cost(it, mask, Xn);
    if (cn < c) {           // false for a NaN cost (singular system)
      X[0] = Xn[0]; X[1] = Xn[1]; X[2] = Xn[2];
      c = cn;
      lambda = fmax(lambda * 0.1, 1e-12);
      fresh = true;
      if (sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]) <= kRefineStep * sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2])) break;
    } else {
      lambda *= 10.0;
      if (lambda > 1e16) break;
    }
  }
}

// Item (b, j) of triangulate_ransac (triangulation.py:72-128) with the drawn pairs pairs[((b J + j) n_iters + i) 2 + {0, 1}]:
//   per pair, the 2-view DLT and the inlier set {pair} + {v : f_v < eps} (strict); the first of the largest sets wins; the DLT on
//   the inliers (all views if none, as the reference falls back); with `direct`, ransac_refine.  A pair outside [0, V) or of one
//   view twice is skipped.  inliers[b J + j] (optional) gets the set as a bit mask.
__host__ __device__ __forceinline__ void ransac_item(const float* __restrict__ proj, const long long* __restrict__ kp2d,
                                                     const int* __restrict__ pairs, int B, int V, int J, int n_iters, double eps,
                                                     int direct, float* __restrict__ out, unsigned long long* __restrict__ inliers,
                                                     int b, int j) {
  const RansacItem it{proj + (long)b * V * 12, kp2d + ((long)b * V * J + j) * 2, (long)J * 2, V};
  unsigned long long best = 0;
  int best_n = 0;
  for (int i = 0; i < n_iters; ++i) {
    const int* pr = pairs + (((long)b * J + j) * n_iters + i) * 2;
    const int va = pr[0], vb = pr[1];
    if (va < 0 || vb < 0 || va >= V || vb >= V || va == vb) continue;
    unsigned long long mask = (1ull << va) | (1ull << vb);
    double X[3];
    ransac_dlt(it, mask, X);
    for (int v = 0; v < V; ++v)
      if (sqrt(ransac_error2(it, v, X)) < eps) mask |= 1ull << v;     // sqrt(f^2) = 0.5 |p - pi(X)| exactly
    const int n = popcount64(mask);
    if (n > best_n) { best = mask; best_n = n; }
  }
  if (best == 0) best = V == 64 ? ~0ull : (1ull << V) - 1;
  double X[3];
  ransac_dlt(it, best, X);
  if (direct) ransac_refine(it, best, X);
  const long bj = (long)b * J + j;
  out[bj * 3] = (float)X[0];
  out[bj * 3 + 1] = (float)X[1];
  out[bj * 3 + 2] = (float)X[2];
  if (inliers) inliers[bj] = best;
}

__global__ void __launch_bounds__(128) triangulate_ransac_kernel(const float* __restrict__ proj, const long long* __restrict__ kp2d,
                                                                 const int* __restrict__ pairs, int B, int V, int J, int n_iters,
                                                                 double eps, int direct, float* __restrict__ out,
                                                                 unsigned long long* __restrict__ inliers) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * J) return;
  ransac_item(proj, kp2d, pairs, B, V, J, n_iters, eps, direct, out, inliers, idx / J, idx % J);
}

}  // namespace lt

using namespace lt;

extern "C" size_t lt_heatmap_argmax_workspace_bytes(int N, int J, int h, int w) {
  if (N <= 0 || J <= 0 || h <= 0 || w <= 0) return 0;
  const long slices = ceil_div((long)h * w, kArgmaxSlice);
  return (size_t)N * J * slices * (sizeof(float) + sizeof(int));
}

extern "C" int lt_heatmap_argmax_fwd(const float* logits, int C, float* heatmaps, long long* keypoints_2d, void* workspace,
                                     size_t workspace_bytes, int N, int J, int h, int w, float scale_x, float scale_y, void* stream) {
  LT_REQUIRE(logits && heatmaps && keypoints_2d && workspace, "heatmap_argmax: null pointer");
  LT_REQUIRE(N > 0 && J > 0 && h > 0 && w > 0 && C >= J && N <= 65535, "heatmap_argmax: bad sizes");
  LT_REQUIRE((long)h * w < (1l << 24), "heatmap_argmax: maps of %d x %d pixels, at most 2^24 supported", h, w);
  LT_REQUIRE(workspace_bytes >= lt_heatmap_argmax_workspace_bytes(N, J, h, w), "heatmap_argmax: workspace of %zu bytes, %zu needed",
             workspace_bytes, lt_heatmap_argmax_workspace_bytes(N, J, h, w));
  const int hw = h * w, slices = ceil_div(hw, kArgmaxSlice);
  float* part_val = static_cast<float*>(workspace);
  int* part_idx = reinterpret_cast<int*>(part_val + (long)N * J * slices);
  cudaStream_t st = (cudaStream_t)stream;
  heatmap_argmax_kernel<<<dim3(slices, N, ceil_div(J, 32)), kArgmaxWarps * 32, 0, st>>>(logits, C, heatmaps, part_val, part_idx, J,
                                                                                         hw, slices);
  LT_CHECK_LAUNCH("heatmap_argmax_kernel");
  heatmap_argmax_finish_kernel<<<ceil_div((long)N * J, 128), 128, 0, st>>>(part_val, part_idx, keypoints_2d, N * J, slices, w, scale_x,
                                                                           scale_y);
  LT_CHECK_LAUNCH("heatmap_argmax_finish_kernel");
  return LT_OK;
}

extern "C" int lt_triangulate_ransac_fwd(const float* proj, const long long* keypoints_2d, const int* pairs, int B, int V, int J,
                                         int n_iters, double eps, int direct, float* keypoints_3d, unsigned long long* inliers,
                                         void* stream) {
  LT_REQUIRE(proj && keypoints_2d && pairs && keypoints_3d, "triangulate_ransac: null pointer");
  LT_REQUIRE(B > 0 && J > 0 && n_iters >= 0 && V >= 2, "triangulate_ransac: bad sizes");
  LT_REQUIRE(V <= 64, "triangulate_ransac: %d views, at most 64 supported (inlier sets are 64-bit masks)", V);
  triangulate_ransac_kernel<<<ceil_div((long)B * J, 128), 128, 0, (cudaStream_t)stream>>>(proj, keypoints_2d, pairs, B, V, J, n_iters,
                                                                                          eps, direct, keypoints_3d, inliers);
  LT_CHECK_LAUNCH("triangulate_ransac_kernel");
  return LT_OK;
}

// test hook: the kernel's per-item code on host pointers, for the `-m "not gpu"` tests
extern "C" int lt_test_triangulate_ransac_host(const float* proj, const long long* keypoints_2d, const int* pairs, int B, int V, int J,
                                               int n_iters, double eps, int direct, float* keypoints_3d, unsigned long long* inliers) {
  LT_REQUIRE(proj && keypoints_2d && pairs && keypoints_3d, "test_triangulate_ransac_host: null pointer");
  LT_REQUIRE(B > 0 && J > 0 && n_iters >= 0 && V >= 2, "test_triangulate_ransac_host: bad sizes");
  LT_REQUIRE(V <= 64, "test_triangulate_ransac_host: %d views, at most 64 supported (inlier sets are 64-bit masks)", V);
  for (int b = 0; b < B; ++b)
    for (int j = 0; j < J; ++j) ransac_item(proj, keypoints_2d, pairs, B, V, J, n_iters, eps, direct, keypoints_3d, inliers, b, j);
  return LT_OK;
}
