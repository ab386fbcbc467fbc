// Small kernels of the algebraic-triangulation path and the confidence heads (SURVEY section 8f rows 2 and 4):
//   - global-average-pool + 3-layer MLP + sigmoid tail of GlobalAveragePoolingHead (pose_resnet.py:163-174)
//   - normalisation of per-view confidences (triangulation.py:173-174, :268-269)
//   - confidence-weighted DLT triangulation (multiview.py:141-183) and its backward, one thread per (sample, joint); the
//     projection-matrix gradient as per-(sample, joint) partials summed over the joints in a fixed order
#include "common.cuh"
#include "dlt_common.cuh"
#include <math.h>
#include <stdlib.h>

namespace lt {

// One CTA per image: mean over P positions of C0 channels, then Linear(C0,H1)+ReLU, Linear(H1,H2)+ReLU,
// Linear(H2,NO)+Sigmoid.  Weights are row-major [out][in] float32 (nn.Linear layout).  Dynamic smem: C0+H1+H2 floats.
__global__ void __launch_bounds__(256) gap_mlp3_kernel(const void* __restrict__ in, int format, int P, int C0, int H1, int H2, int NO,
                                                       const float* __restrict__ w1, const float* __restrict__ b1,
                                                       const float* __restrict__ w2, const float* __restrict__ b2,
                                                       const float* __restrict__ w3, const float* __restrict__ b3,
                                                       float* __restrict__ out) {
  extern __shared__ float sm[];
  float* x0 = sm;
  float* x1 = x0 + C0;
  float* x2 = x1 + H1;
  const int n = blockIdx.x;
  for (int c = threadIdx.x; c < C0; c += blockDim.x) {
    float acc = 0.0f;
    for (int q = 0; q < P; ++q) {
      const long pix = (long)n * P + q;
      if (format == LT_FMT_F32) acc += reinterpret_cast<const float*>(in)[pix * C0 + c];
      else {
        const sh_t* row = reinterpret_cast<const sh_t*>(in) + pix * 2 * C0;
        acc += join_s32(row[s32_off(c)], row[s32_off(c) + 32]);
      }
    }
    x0[c] = acc / (float)P;
  }
  __syncthreads();
  for (int o = threadIdx.x; o < H1; o += blockDim.x) {
    float acc = b1[o];
    for (int i = 0; i < C0; ++i) acc = fmaf(w1[(long)o * C0 + i], x0[i], acc);
    x1[o] = fmaxf(acc, 0.0f);
  }
  __syncthreads();
  for (int o = threadIdx.x; o < H2; o += blockDim.x) {
    float acc = b2[o];
    for (int i = 0; i < H1; ++i) acc = fmaf(w2[(long)o * H1 + i], x1[i], acc);
    x2[o] = fmaxf(acc, 0.0f);
  }
  __syncthreads();
  for (int o = threadIdx.x; o < NO; o += blockDim.x) {
    float acc = b3[o];
    for (int i = 0; i < H2; ++i) acc = fmaf(w3[(long)o * H2 + i], x2[i], acc);
    out[(long)n * NO + o] = 1.0f / (1.0f + expf(-acc));
  }
}

// conf[B][V][C] /= sum over views; += eps
__global__ void view_normalize_kernel(float* __restrict__ conf, int B, int V, int C, float eps) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  const int b = i / C, c = i % C;
  float s = 0.0f;
  for (int v = 0; v < V; ++v) s += conf[((long)b * V + v) * C + c];
  for (int v = 0; v < V; ++v) conf[((long)b * V + v) * C + c] = conf[((long)b * V + v) * C + c] / s + eps;
}

// Weighted DLT (Hartley & Zisserman 12.2): rows c*(x*P[2] - P[0]), c*(y*P[2] - P[1]); the solution is the right singular
// vector of the smallest singular value of A (2V x 4) = eigenvector of A^T A for its smallest eigenvalue.  A^T A and a cyclic
// Jacobi eigen-solve run in float64 (forming A^T A squares the condition number, fp32 would not do); the reference's
// `-vh[:, 3]` sign cancels in the dehomogenisation.

// (p2 * x - p0) * cf with one float32 rounding per operation, as the reference rounds it: on the device __fmul_rn / __fsub_rn
// keep nvcc from contracting the subtraction into an FFMA; the host compiler is not asked for FMA, so the plain operators match.
__host__ __device__ __forceinline__ float dlt_entry(float p2, float x, float p0, float cf) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(__fsub_rn(__fmul_rn(p2, x), p0), cf);
#else
  return (p2 * x - p0) * cf;
#endif
}

// the two DLT rows of view v, as the forward rounds them: formed in float32 like the reference (multiview.py:159-161), then
// widened; bit-identical on the device and the host.  cf = 1 gives the unweighted rows x*P[2] - P[0], y*P[2] - P[1].
__host__ __device__ __forceinline__ void dlt_rows(const float* P, float x, float y, float cf, double r0[4], double r1[4]) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    r0[c] = (double)dlt_entry(P[8 + c], x, P[c], cf);
    r1[c] = (double)dlt_entry(P[8 + c], y, P[4 + c], cf);
  }
}

// A^T A of item (b, j) accumulated in float64, then diagonalised by dlt_jacobi (dlt_common.cuh): on return M's diagonal holds the
// eigenvalues, the columns of E the eigenvectors, and the result is the index of the smallest eigenvalue (the first one on a
// tie).  Shared by the forward and the backward kernel (and the host test hook): one sequence of operations.
__host__ __device__ __forceinline__ int dlt_eigen(const float* __restrict__ proj, const float* __restrict__ kp2d,
                                                  const float* __restrict__ conf, int b, int j, int V, int J, double M[4][4],
                                                  double E[4][4]) {
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) M[r][c] = 0.0;
  for (int v = 0; v < V; ++v) {
    const float* P = proj + ((long)b * V + v) * 12;
    const float x = kp2d[(((long)b * V + v) * J + j) * 2], y = kp2d[(((long)b * V + v) * J + j) * 2 + 1];
    const float cf = conf ? conf[((long)b * V + v) * J + j] : 1.0f;
    double r0[4], r1[4];
    dlt_rows(P, x, y, cf, r0, r1);
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) M[r][c] += r0[r] * r0[c] + r1[r] * r1[c];
  }
  return dlt_jacobi(M, E);
}

// Forward of the weighted DLT for item (b, j): out[b][j] = u[0:3] / u[3].  A point at infinity (u[3] = 0) gives the IEEE
// quotients (inf or nan), as the reference's division does.
__host__ __device__ __forceinline__ void dlt_fwd_item(const float* __restrict__ proj, const float* __restrict__ kp2d,
                                                      const float* __restrict__ conf, float* __restrict__ out, int b, int j, int V,
                                                      int J) {
  double M[4][4], E[4][4], u[4];
  dlt_column(E, dlt_eigen(proj, kp2d, conf, b, j, V, J, M, E), u);
  const double w = u[3];
  const long bj = (long)b * J + j;
  out[bj * 3 + 0] = (float)(u[0] / w);
  out[bj * 3 + 1] = (float)(u[1] / w);
  out[bj * 3 + 2] = (float)(u[2] / w);
}

__global__ void __launch_bounds__(128) triangulate_dlt_kernel(const float* __restrict__ proj, const float* __restrict__ kp2d,
                                                              const float* __restrict__ conf, float* __restrict__ out, int B, int V, int J) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * J) return;
  dlt_fwd_item(proj, kp2d, conf, out, idx / J, idx % J, V, J);
}

// Tie rule of dlt_bwd_item: a gap |lambda_0 - lambda_k| at or below kDltTieTol of the larger of the two eigenvalues, or below
// kDltGapFloor of the largest one, counts as a tie.  The relative test, not one against the largest eigenvalue, is what keeps
// graded systems: the fourth column of A is ~1e3x the others, so with confidences of (1, 1e-4, 1e-4, 1e-4) the two smallest
// eigenvalues are ~1e-17 and ~1e-14 of the largest, yet the float64 Jacobi solve resolves them and their gap carries the main
// term of the gradient.  The floor only bounds 1 / gap; confidence ratios down to 1e-6 give gaps of ~1e-18 of the largest
// eigenvalue and are kept.
constexpr double kDltTieTol = 1e-12;
constexpr double kDltGapFloor = 1e-30;

// Backward of the weighted DLT for item (b, j).  With (lambda_k, e_k) the eigenpairs of M = A^T A, u = e_0 the smallest:
//   X = u[0:3] / u[3]  ->  g_u = [g_X / u[3], -(g_X . u[0:3]) / u[3]^2]
//   w = sum_{k != 0} (g_u . e_k) / (lambda_0 - lambda_k) e_k          (first-order perturbation of the eigenvector)
//   G_A = A (w u^T + u w^T): row r of A gets (a_r . w) u + (a_r . u) w
//   d x = c (G_A[r0] . P[2]),  d y = c (G_A[r1] . P[2]),  d c = G_A[r0] . (x P[2] - P[0]) + G_A[r1] . (y P[2] - P[1]),
//   d P[0] = -c G_A[r0],  d P[1] = -c G_A[r1],  d P[2] = c (x G_A[r0] + y G_A[r1])   (the float32 rounding of the rows as identity).
// Independent of the sign of u.  A term whose gap is a tie by the rule above (kDltTieTol) is dropped: on an exact tie the
// derivative does not exist (torch's SVD backward returns non-finite values there); dropping keeps it finite.
// dlt_perturbation gives u and w of item (b, j); dlt_row_grads the rows G_A[r0], G_A[r1] of view v.  Both item functions below
// use them, so the key-point, confidence and projection gradients follow one derivation.
__host__ __device__ __forceinline__ void dlt_perturbation(const float* __restrict__ proj, const float* __restrict__ kp2d,
                                                          const float* __restrict__ conf, const float* __restrict__ grad_out, int b, int j,
                                                          int V, int J, double u[4], double w[4]) {
  double M[4][4], E[4][4];
  const int m = dlt_eigen(proj, kp2d, conf, b, j, V, J, M, E);
  dlt_column(E, m, u);
  double lam0 = M[0][0], lmax = fabs(M[0][0]);
#pragma unroll
  for (int k = 1; k < 4; ++k) {
    if (k == m) lam0 = M[k][k];
    lmax = fmax(lmax, fabs(M[k][k]));
  }
  const long bj = (long)b * J + j;
  const double gx = grad_out[bj * 3], gy = grad_out[bj * 3 + 1], gz = grad_out[bj * 3 + 2];
  const double iw = 1.0 / u[3];
  const double gu[4] = {gx * iw, gy * iw, gz * iw, -(gx * u[0] + gy * u[1] + gz * u[2]) * iw * iw};
#pragma unroll
  for (int r = 0; r < 4; ++r) w[r] = 0.0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double gap = lam0 - M[k][k];
    if (k == m || !(fabs(gap) > kDltTieTol * fmax(fabs(lam0), fabs(M[k][k])) + kDltGapFloor * lmax)) continue;
    const double s = (gu[0] * E[0][k] + gu[1] * E[1][k] + gu[2] * E[2][k] + gu[3] * E[3][k]) / gap;
#pragma unroll
    for (int r = 0; r < 4; ++r) w[r] += s * E[r][k];
  }
}

// G_A rows g0 (from x) and g1 (from y) of view P with key point (x, y) and confidence cf
__host__ __device__ __forceinline__ void dlt_row_grads(const float* P, float x, float y, float cf, const double u[4], const double w[4],
                                                       double g0[4], double g1[4]) {
  double a0[4], a1[4];
  dlt_rows(P, x, y, cf, a0, a1);
  double aw0 = 0.0, au0 = 0.0, aw1 = 0.0, au1 = 0.0;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    aw0 += a0[c] * w[c]; au0 += a0[c] * u[c];
    aw1 += a1[c] * w[c]; au1 += a1[c] * u[c];
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    g0[c] = aw0 * u[c] + au0 * w[c];
    g1[c] = aw1 * u[c] + au1 * w[c];
  }
}

// grad_kp / grad_conf are WRITTEN (every (v, j) of the item), grad_conf may be null.
__host__ __device__ __forceinline__ void dlt_bwd_item(const float* __restrict__ proj, const float* __restrict__ kp2d,
                                                      const float* __restrict__ conf, const float* __restrict__ grad_out,
                                                      float* __restrict__ grad_kp, float* __restrict__ grad_conf, int b, int j,
                                                      int V, int J) {
  double u[4], w[4];
  dlt_perturbation(proj, kp2d, conf, grad_out, b, j, V, J, u, w);
  for (int v = 0; v < V; ++v) {
    const float* P = proj + ((long)b * V + v) * 12;
    const long vj = ((long)b * V + v) * J + j;
    const float x = kp2d[vj * 2], y = kp2d[vj * 2 + 1];
    const float cf = conf ? conf[vj] : 1.0f;
    double g0[4], g1[4], dx = 0.0, dy = 0.0;
    dlt_row_grads(P, x, y, cf, u, w, g0, g1);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      dx += g0[c] * (double)P[8 + c];
      dy += g1[c] * (double)P[8 + c];
    }
    grad_kp[vj * 2] = (float)(cf * dx);
    grad_kp[vj * 2 + 1] = (float)(cf * dy);
    if (grad_conf) {
      double a0[4], a1[4];
      dlt_rows(P, x, y, 1.0f, a0, a1);
      double dc = 0.0;
#pragma unroll
      for (int c = 0; c < 4; ++c) dc += g0[c] * a0[c] + g1[c] * a1[c];
      grad_conf[vj] = (float)dc;
    }
  }
}

// d P of item (b, j), float64, WRITTEN to partial[((b J + j) V + v) 12 + e] for every view
__host__ __device__ __forceinline__ void dlt_proj_bwd_item(const float* __restrict__ proj, const float* __restrict__ kp2d,
                                                           const float* __restrict__ conf, const float* __restrict__ grad_out,
                                                           double* __restrict__ partial, int b, int j, int V, int J) {
  double u[4], w[4];
  dlt_perturbation(proj, kp2d, conf, grad_out, b, j, V, J, u, w);
  for (int v = 0; v < V; ++v) {
    const float* P = proj + ((long)b * V + v) * 12;
    const long vj = ((long)b * V + v) * J + j;
    const double x = kp2d[vj * 2], y = kp2d[vj * 2 + 1];
    const float cf = conf ? conf[vj] : 1.0f;
    double g0[4], g1[4];
    dlt_row_grads(P, (float)x, (float)y, cf, u, w, g0, g1);
    double* d = partial + (((long)b * J + j) * V + v) * 12;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      d[c] = -(double)cf * g0[c];
      d[4 + c] = -(double)cf * g1[c];
      d[8 + c] = (double)cf * (x * g0[c] + y * g1[c]);
    }
  }
}

// d P[b][v][e] = sum_j partial (joints in order)
__host__ __device__ __forceinline__ void dlt_proj_merge_item(const double* __restrict__ partial, float* __restrict__ grad_proj, int V, int J,
                                                             int b, int v, int e) {
  double s = 0.0;
  for (int j = 0; j < J; ++j) s += partial[(((long)b * J + j) * V + v) * 12 + e];
  grad_proj[((long)b * V + v) * 12 + e] = (float)s;
}

__global__ void __launch_bounds__(128) triangulate_dlt_bwd_kernel(const float* __restrict__ proj, const float* __restrict__ kp2d,
                                                                  const float* __restrict__ conf, const float* __restrict__ grad_out,
                                                                  float* __restrict__ grad_kp, float* __restrict__ grad_conf, int B,
                                                                  int V, int J) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * J) return;
  dlt_bwd_item(proj, kp2d, conf, grad_out, grad_kp, grad_conf, idx / J, idx % J, V, J);
}

__global__ void __launch_bounds__(128) triangulate_dlt_proj_bwd_kernel(const float* __restrict__ proj, const float* __restrict__ kp2d,
                                                                       const float* __restrict__ conf, const float* __restrict__ grad_out,
                                                                       double* __restrict__ partial, int B, int V, int J) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * J) return;
  dlt_proj_bwd_item(proj, kp2d, conf, grad_out, partial, idx / J, idx % J, V, J);
}

__global__ void __launch_bounds__(128) triangulate_dlt_proj_merge_kernel(const double* __restrict__ partial, float* __restrict__ grad_proj,
                                                                         int B, int V, int J) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * V * 12) return;
  dlt_proj_merge_item(partial, grad_proj, V, J, idx / (V * 12), (idx / 12) % V, idx % 12);
}

}  // namespace lt

using namespace lt;

extern "C" int lt_gap_mlp3_fwd(const void* in, int format, int N, int P, int C0, int H1, int H2, int NO, const float* w1,
                               const float* b1, const float* w2, const float* b2, const float* w3, const float* b3, float* out,
                               void* stream) {
  LT_REQUIRE(in && w1 && b1 && w2 && b2 && w3 && b3 && out, "gap_mlp3: null pointer");
  LT_REQUIRE(N > 0 && P > 0 && C0 > 0 && H1 > 0 && H2 > 0 && NO > 0, "gap_mlp3: bad sizes");
  LT_REQUIRE(format == LT_FMT_F32 || C0 % 32 == 0, "gap_mlp3: split-fp16 input needs C0 %% 32 == 0");
  const size_t smem = (size_t)(C0 + H1 + H2) * sizeof(float);
  LT_REQUIRE(smem <= 48 * 1024, "gap_mlp3: hidden sizes too large");
  gap_mlp3_kernel<<<N, 256, smem, (cudaStream_t)stream>>>(in, format, P, C0, H1, H2, NO, w1, b1, w2, b2, w3, b3, out);
  LT_CHECK_LAUNCH("gap_mlp3_kernel");
  return LT_OK;
}

extern "C" int lt_view_normalize_fwd(float* conf, int B, int V, int C, float eps, void* stream) {
  LT_REQUIRE(conf && B > 0 && V > 0 && C > 0, "view_normalize: bad arguments");
  view_normalize_kernel<<<ceil_div((long)B * C, 128), 128, 0, (cudaStream_t)stream>>>(conf, B, V, C, eps);
  LT_CHECK_LAUNCH("view_normalize_kernel");
  return LT_OK;
}

extern "C" int lt_triangulate_dlt_fwd(const float* proj, const float* keypoints_2d, const float* confidences, float* out, int B,
                                      int V, int J, void* stream) {
  LT_REQUIRE(proj && keypoints_2d && out && B > 0 && V > 0 && J > 0, "triangulate_dlt: bad arguments");
  triangulate_dlt_kernel<<<ceil_div((long)B * J, 128), 128, 0, (cudaStream_t)stream>>>(proj, keypoints_2d, confidences, out, B, V, J);
  LT_CHECK_LAUNCH("triangulate_dlt_kernel");
  return LT_OK;
}

extern "C" int lt_triangulate_dlt_bwd(const float* proj, const float* keypoints_2d, const float* confidences, const float* grad_out,
                                      float* grad_keypoints_2d, float* grad_confidences, int B, int V, int J, void* stream) {
  LT_REQUIRE(proj && keypoints_2d && grad_out && grad_keypoints_2d && B > 0 && V > 0 && J > 0, "triangulate_dlt_bwd: bad arguments");
  triangulate_dlt_bwd_kernel<<<ceil_div((long)B * J, 128), 128, 0, (cudaStream_t)stream>>>(proj, keypoints_2d, confidences, grad_out,
                                                                                           grad_keypoints_2d, grad_confidences, B, V, J);
  LT_CHECK_LAUNCH("triangulate_dlt_bwd_kernel");
  return LT_OK;
}

extern "C" size_t lt_triangulate_dlt_proj_bwd_workspace_bytes(int B, int V, int J) {
  return (B > 0 && V > 0 && J > 0) ? (size_t)B * J * V * 12 * sizeof(double) : 0;
}

extern "C" int lt_triangulate_dlt_proj_bwd(const float* proj, const float* keypoints_2d, const float* confidences, const float* grad_out,
                                           float* grad_proj, void* workspace, size_t workspace_bytes, int B, int V, int J, void* stream) {
  LT_REQUIRE(proj && keypoints_2d && grad_out && grad_proj && workspace && B > 0 && V > 0 && J > 0, "triangulate_dlt_proj_bwd: bad arguments");
  LT_REQUIRE(workspace_bytes >= lt_triangulate_dlt_proj_bwd_workspace_bytes(B, V, J), "triangulate_dlt_proj_bwd: workspace of %zu bytes, %zu needed",
             workspace_bytes, lt_triangulate_dlt_proj_bwd_workspace_bytes(B, V, J));
  double* partial = static_cast<double*>(workspace);
  cudaStream_t st = (cudaStream_t)stream;
  triangulate_dlt_proj_bwd_kernel<<<ceil_div((long)B * J, 128), 128, 0, st>>>(proj, keypoints_2d, confidences, grad_out, partial, B, V, J);
  LT_CHECK_LAUNCH("triangulate_dlt_proj_bwd_kernel");
  triangulate_dlt_proj_merge_kernel<<<ceil_div((long)B * V * 12, 128), 128, 0, st>>>(partial, grad_proj, B, V, J);
  LT_CHECK_LAUNCH("triangulate_dlt_proj_merge_kernel");
  return LT_OK;
}

// test hooks: the forward's and the backward's per-item code on the CPU (host pointers), for the `-m "not gpu"` tests
extern "C" int lt_test_triangulate_dlt_fwd_host(const float* proj, const float* keypoints_2d, const float* confidences, float* out,
                                                int B, int V, int J) {
  LT_REQUIRE(proj && keypoints_2d && out && B > 0 && V > 0 && J > 0, "test_triangulate_dlt_fwd_host: bad arguments");
  for (int b = 0; b < B; ++b)
    for (int j = 0; j < J; ++j) dlt_fwd_item(proj, keypoints_2d, confidences, out, b, j, V, J);
  return LT_OK;
}

extern "C" int lt_test_triangulate_dlt_bwd_host(const float* proj, const float* keypoints_2d, const float* confidences,
                                                const float* grad_out, float* grad_keypoints_2d, float* grad_confidences, int B, int V,
                                                int J) {
  LT_REQUIRE(proj && keypoints_2d && grad_out && grad_keypoints_2d && B > 0 && V > 0 && J > 0,
             "test_triangulate_dlt_bwd_host: bad arguments");
  for (int b = 0; b < B; ++b)
    for (int j = 0; j < J; ++j) dlt_bwd_item(proj, keypoints_2d, confidences, grad_out, grad_keypoints_2d, grad_confidences, b, j, V, J);
  return LT_OK;
}

extern "C" int lt_test_triangulate_dlt_proj_bwd_host(const float* proj, const float* keypoints_2d, const float* confidences,
                                                     const float* grad_out, float* grad_proj, int B, int V, int J) {
  LT_REQUIRE(proj && keypoints_2d && grad_out && grad_proj && B > 0 && V > 0 && J > 0, "test_triangulate_dlt_proj_bwd_host: bad arguments");
  double* partial = static_cast<double*>(malloc(lt_triangulate_dlt_proj_bwd_workspace_bytes(B, V, J)));
  LT_REQUIRE(partial, "test_triangulate_dlt_proj_bwd_host: out of memory");
  for (int b = 0; b < B; ++b)
    for (int j = 0; j < J; ++j) dlt_proj_bwd_item(proj, keypoints_2d, confidences, grad_out, partial, b, j, V, J);
  for (int b = 0; b < B; ++b)
    for (int v = 0; v < V; ++v)
      for (int e = 0; e < 12; ++e) dlt_proj_merge_item(partial, grad_proj, V, J, b, v, e);
  free(partial);
  return LT_OK;
}
