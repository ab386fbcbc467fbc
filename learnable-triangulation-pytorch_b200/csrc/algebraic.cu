// Small kernels of the algebraic-triangulation path and the confidence heads (SURVEY section 8f rows 2 and 4):
//   - global-average-pool + 3-layer MLP + sigmoid tail of GlobalAveragePoolingHead (pose_resnet.py:163-174)
//   - the same tail for training (head_backend="native"): the second 2x2 max pool, ReLU, mean and MLP forward, saving what the
//     backward reads, and its backward (weight, bias and input-map gradients), every sum in a fixed order without atomics
//   - normalisation of per-view confidences (triangulation.py:173-174, :268-269) and its backward
//   - confidence-weighted DLT triangulation (multiview.py:141-183) and its backward, one thread per (sample, joint); the
//     projection-matrix gradient as per-(sample, joint) partials summed over the joints in a fixed order
#include "common.cuh"
#include "dlt_common.cuh"
#include <math.h>
#include <stdlib.h>

namespace lt {

// ---- the confidence heads' MLP tail: Linear(C0,H1)+ReLU, Linear(H1,H2)+ReLU, Linear(H2,NO)+Sigmoid on one row --------------------
// Weights are row-major [out][in] float32 (nn.Linear layout).  Every output is b[o] followed by one fmaf per input in input order, so
// the inference tail (gap_mlp3_kernel), the training tail (conf_head_fwd_kernel) and the host test hook compute the same floats.
__host__ __device__ __forceinline__ float linear_item(const float* __restrict__ w, const float* __restrict__ b, const float* x, int in,
                                                      int o) {
  float acc = b[o];
  for (int i = 0; i < in; ++i) acc = fmaf(w[(long)o * in + i], x[i], acc);
  return acc;
}

__host__ __device__ __forceinline__ float sigmoid_f(float v) { return 1.0f / (1.0f + expf(-v)); }
// dL/dv of y = sigmoid(v) from y and g = dL/dy, as autograd's sigmoid backward: g y (1 - y)
__host__ __device__ __forceinline__ float sigmoid_bwd(float g, float y) { return g * y * (1.0f - y); }

// The ReLU of the hidden layers.  kTorchRelu: torch's rule (a NaN stays NaN), which training follows so that its forward and the
// backward's masks are autograd's; otherwise fmaxf, which maps NaN to 0, as the inference tail always has.
template <bool kTorchRelu>
__host__ __device__ __forceinline__ float hidden_relu(float v) { return kTorchRelu ? (v <= 0.0f ? 0.0f : v) : fmaxf(v, 0.0f); }

// The three layers of row x0 (C0 floats) by the CTA: x1 (H1) and x2 (H2) are the post-ReLU activations, in shared memory, complete on
// return; out (NO) is the sigmoid.  x0 must be complete (after a barrier) on entry.
template <bool kTorchRelu>
__device__ __forceinline__ void mlp3_row(const float* x0, float* x1, float* x2, int C0, int H1, int H2, int NO,
                                         const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ w2,
                                         const float* __restrict__ b2, const float* __restrict__ w3, const float* __restrict__ b3,
                                         float* __restrict__ out) {
  for (int o = threadIdx.x; o < H1; o += blockDim.x) x1[o] = hidden_relu<kTorchRelu>(linear_item(w1, b1, x0, C0, o));
  __syncthreads();
  for (int o = threadIdx.x; o < H2; o += blockDim.x) x2[o] = hidden_relu<kTorchRelu>(linear_item(w2, b2, x1, H1, o));
  __syncthreads();
  for (int o = threadIdx.x; o < NO; o += blockDim.x) out[o] = sigmoid_f(linear_item(w3, b3, x2, H2, o));
}

// One CTA per image: mean over P positions of C0 channels, then the MLP tail (mlp3_row).  Dynamic smem: C0+H1+H2 floats.
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
  mlp3_row<false>(x0, x1, x2, C0, H1, H2, NO, w1, b1, w2, b2, w3, b3, out + (long)n * NO);
}

// ---- training tail of ConfidenceHead (pose_resnet.py): from the second BatchNorm's output x (N, C0, H, W), float32, any element
// strides, through MaxPool2d(2) -> ReLU -> mean over the P = (H/2)(W/2) pooled positions -> the MLP tail, and its backward.
//   forward  conf_head_fwd_kernel, one CTA per row: x0 = mean(relu(pool(x))) with torch's pooling rule (pool_max of misc.cu: a value
//            replaces the running maximum if greater or NaN; floor mode) and a NaN-keeping ReLU, then mlp3_row<true>.  x0, h1, h2
//            are saved for the backward.
//   backward conf_head_bwd_rows_kernel, one CTA per row: d3 = g y (1 - y), d2 = [!(h2 <= 0)] W3^T d3, d1 = [!(h1 <= 0)] W2^T d2,
//            dx0 = W1^T d1 (torch's threshold_backward masks: a NaN activation passes its gradient), into the workspace;
//            conf_head_wgrad_kernel, one thread per weight or bias: the sum over the rows n = 0..N-1 in order;
//            conf_head_dx_kernel, one thread per element of x: dx0 / P at its window's arg-max when !(pooled <= 0), 0 elsewhere
//            (including the last row / column floor mode drops).  No atomics: every sum has one fixed order.
struct HeadMap {
  const float* x; int N, C, H, W; long xs[4];   // element strides (n, c, h, w)
};

// the window of pooled position (ph, pw) of row n, channel c: its maximum under torch's rule and the index (2 a + b) of the element
// holding it (the first one; 0 if no element is taken)
__host__ __device__ __forceinline__ float head_window_max(const HeadMap& m, int n, int c, int ph, int pw, int* arg) {
  const float* xb = m.x + n * m.xs[0] + c * m.xs[1] + (2 * ph) * m.xs[2] + (2 * pw) * m.xs[3];
  float mx = -INFINITY;
  int best = 0;
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b) {
      const float v = xb[a * m.xs[2] + b * m.xs[3]];
      if (v > mx || v != v) { mx = v; best = 2 * a + b; }
    }
  *arg = best;
  return mx;
}

// x0[n][c]: the pooled, rectified values summed in row-major pooled order, over P
__host__ __device__ __forceinline__ float head_gap_item(const HeadMap& m, int n, int c) {
  const int OH = m.H / 2, OW = m.W / 2;
  float acc = 0.0f;
  for (int ph = 0; ph < OH; ++ph)
    for (int pw = 0; pw < OW; ++pw) {
      int arg;
      const float v = head_window_max(m, n, c, ph, pw, &arg);
      acc += v <= 0.0f ? 0.0f : v;
    }
  return acc / (float)(OH * OW);
}

// sum_o w[o][i] d[o] over the `out` rows of an [out][in] weight, o in order
__host__ __device__ __forceinline__ float linear_bwd_item(const float* __restrict__ w, const float* d, int out, int in, int i) {
  float acc = 0.0f;
  for (int o = 0; o < out; ++o) acc = fmaf(w[(long)o * in + i], d[o], acc);
  return acc;
}

// Workspace of the backward: per row d3 (NO), d2 (H2), d1 (H1) and dx0 (C0), float32
__host__ __device__ __forceinline__ long head_ws_row(int C0, int H1, int H2, int NO) { return (long)NO + H2 + H1 + C0; }

// one weight or bias gradient: element e of the flattened [dW1 | db1 | dW2 | db2 | dW3 | db3], summed over the rows in order
__host__ __device__ __forceinline__ void head_wgrad_item(const float* __restrict__ ws, const float* __restrict__ x0,
                                                         const float* __restrict__ h1, const float* __restrict__ h2, int N, int C0, int H1,
                                                         int H2, int NO, long e, float* __restrict__ dw1, float* __restrict__ db1,
                                                         float* __restrict__ dw2, float* __restrict__ db2, float* __restrict__ dw3,
                                                         float* __restrict__ db3) {
  const long row = head_ws_row(C0, H1, H2, NO);
  // the gradient's array, the layer's deltas (offset in a workspace row), its input activations (nullptr for a bias) and their width
  float* dst;
  const float* act = nullptr;
  long doff;
  int in = 1;
  if (e < (long)H1 * C0) { dst = dw1; act = x0; in = C0; doff = (long)NO + H2; }
  else if ((e -= (long)H1 * C0) < H1) { dst = db1; doff = (long)NO + H2; }
  else if ((e -= H1) < (long)H2 * H1) { dst = dw2; act = h1; in = H1; doff = NO; }
  else if ((e -= (long)H2 * H1) < H2) { dst = db2; doff = NO; }
  else if ((e -= H2) < (long)NO * H2) { dst = dw3; act = h2; in = H2; doff = 0; }
  else { e -= (long)NO * H2; dst = db3; doff = 0; }
  const long o = act ? e / in : e, i = act ? e % in : 0;
  float acc = 0.0f;
  for (int n = 0; n < N; ++n) {
    const float d = ws[n * row + doff + o];
    acc = act ? fmaf(d, act[(long)n * in + i], acc) : acc + d;
  }
  dst[e] = acc;
}

// grad_x at element i of the map, walked in the memory order of grad_x (channels fastest when its channel stride is 1)
__host__ __device__ __forceinline__ void head_dx_item(const HeadMap& m, const long gs[4], const float* __restrict__ ws, int C0, int H1,
                                                      int H2, int NO, float* __restrict__ gx, long i) {
  int n, c, h, w;
  long r = i;
  if (gs[1] == 1 && m.C > 1) {
    c = (int)(r % m.C); r /= m.C; w = (int)(r % m.W); r /= m.W; h = (int)(r % m.H); n = (int)(r / m.H);
  } else {
    w = (int)(r % m.W); r /= m.W; h = (int)(r % m.H); r /= m.H; c = (int)(r % m.C); n = (int)(r / m.C);
  }
  const int OH = m.H / 2, OW = m.W / 2, ph = h / 2, pw = w / 2;
  float out = 0.0f;
  if (ph < OH && pw < OW) {
    int arg;
    const float mx = head_window_max(m, n, c, ph, pw, &arg);
    if (arg == 2 * (h - 2 * ph) + (w - 2 * pw) && !(mx <= 0.0f))
      out = ws[n * head_ws_row(C0, H1, H2, NO) + (long)NO + H2 + H1 + c] / (float)(OH * OW);
  }
  gx[n * gs[0] + c * gs[1] + h * gs[2] + w * gs[3]] = out;
}

__global__ void __launch_bounds__(256) conf_head_fwd_kernel(const HeadMap m, int H1, int H2, int NO, const float* __restrict__ w1,
                                                            const float* __restrict__ b1, const float* __restrict__ w2,
                                                            const float* __restrict__ b2, const float* __restrict__ w3,
                                                            const float* __restrict__ b3, float* __restrict__ out,
                                                            float* __restrict__ x0_out, float* __restrict__ h1_out,
                                                            float* __restrict__ h2_out) {
  extern __shared__ float sm[];
  const int C0 = m.C, n = blockIdx.x;
  float* x0 = sm;
  float* x1 = x0 + C0;
  float* x2 = x1 + H1;
  for (int c = threadIdx.x; c < C0; c += blockDim.x) x0_out[(long)n * C0 + c] = x0[c] = head_gap_item(m, n, c);
  __syncthreads();
  mlp3_row<true>(x0, x1, x2, C0, H1, H2, NO, w1, b1, w2, b2, w3, b3, out + (long)n * NO);
  for (int o = threadIdx.x; o < H1; o += blockDim.x) h1_out[(long)n * H1 + o] = x1[o];
  for (int o = threadIdx.x; o < H2; o += blockDim.x) h2_out[(long)n * H2 + o] = x2[o];
}

// Dynamic smem: NO + H2 + H1 floats (the row's deltas, also written to its workspace row)
__global__ void __launch_bounds__(256) conf_head_bwd_rows_kernel(int C0, int H1, int H2, int NO, const float* __restrict__ w1,
                                                                 const float* __restrict__ w2, const float* __restrict__ w3,
                                                                 const float* __restrict__ h1, const float* __restrict__ h2,
                                                                 const float* __restrict__ y, const float* __restrict__ g,
                                                                 float* __restrict__ ws) {
  extern __shared__ float sm[];
  float* d3 = sm;
  float* d2 = d3 + NO;
  float* d1 = d2 + H2;
  const int n = blockIdx.x;
  float* wrow = ws + n * head_ws_row(C0, H1, H2, NO);
  for (int o = threadIdx.x; o < NO; o += blockDim.x) {
    wrow[o] = d3[o] = sigmoid_bwd(g[(long)n * NO + o], y[(long)n * NO + o]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < H2; i += blockDim.x)
    wrow[NO + i] = d2[i] = !(h2[(long)n * H2 + i] <= 0.0f) ? linear_bwd_item(w3, d3, NO, H2, i) : 0.0f;
  __syncthreads();
  for (int i = threadIdx.x; i < H1; i += blockDim.x)
    wrow[NO + H2 + i] = d1[i] = !(h1[(long)n * H1 + i] <= 0.0f) ? linear_bwd_item(w2, d2, H2, H1, i) : 0.0f;
  __syncthreads();
  for (int i = threadIdx.x; i < C0; i += blockDim.x) wrow[NO + H2 + H1 + i] = linear_bwd_item(w1, d1, H1, C0, i);
}

__global__ void __launch_bounds__(256) conf_head_wgrad_kernel(const float* __restrict__ ws, const float* __restrict__ x0,
                                                              const float* __restrict__ h1, const float* __restrict__ h2, int N, int C0,
                                                              int H1, int H2, int NO, long total, float* __restrict__ dw1,
                                                              float* __restrict__ db1, float* __restrict__ dw2, float* __restrict__ db2,
                                                              float* __restrict__ dw3, float* __restrict__ db3) {
  for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x)
    head_wgrad_item(ws, x0, h1, h2, N, C0, H1, H2, NO, e, dw1, db1, dw2, db2, dw3, db3);
}

__global__ void __launch_bounds__(256) conf_head_dx_kernel(const HeadMap m, const long4 gs4, const float* __restrict__ ws, int H1, int H2,
                                                           int NO, float* __restrict__ gx, long total) {
  const long gs[4] = {gs4.x, gs4.y, gs4.z, gs4.w};
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x)
    head_dx_item(m, gs, ws, m.C, H1, H2, NO, gx, i);
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

// Backward of y_v = c_v / S + eps, S = sum_u c_u, for one (b, c): dc_v = g_v / S - (sum_u g_u c_u) / S^2, the sums over the views in
// order, in float64, rounded once.
__host__ __device__ __forceinline__ void view_normalize_bwd_item(const float* __restrict__ conf, const float* __restrict__ grad,
                                                                 float* __restrict__ grad_conf, int V, int C, int b, int c) {
  double s = 0.0, t = 0.0;
  for (int v = 0; v < V; ++v) {
    const long k = ((long)b * V + v) * C + c;
    s += (double)conf[k];
    t += (double)grad[k] * (double)conf[k];
  }
  for (int v = 0; v < V; ++v) {
    const long k = ((long)b * V + v) * C + c;
    grad_conf[k] = (float)((double)grad[k] / s - t / (s * s));
  }
}

__global__ void view_normalize_bwd_kernel(const float* __restrict__ conf, const float* __restrict__ grad, float* __restrict__ grad_conf,
                                          int B, int V, int C) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  view_normalize_bwd_item(conf, grad, grad_conf, V, C, i / C, i % C);
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

static int conf_head_check(const float* x, int N, int C0, int H, int W, int H1, int H2, int NO) {
  LT_REQUIRE(x, "conf_head_tail: null input map");
  LT_REQUIRE(N > 0 && C0 > 0 && H > 0 && W > 0 && H1 > 0 && H2 > 0 && NO > 0, "conf_head_tail: non-positive size");
  LT_REQUIRE(H >= 2 && W >= 2, "conf_head_tail: a %dx%d map is too small for the 2x2 max pool", H, W);
  LT_REQUIRE((size_t)(C0 + H1 + H2) * sizeof(float) <= 48 * 1024, "conf_head_tail: layer widths too large");
  return LT_OK;
}

extern "C" int lt_conf_head_tail_fwd(const float* x, int N, int C0, int H, int W, long xs_n, long xs_c, long xs_h, long xs_w, int H1,
                                     int H2, int NO, const float* w1, const float* b1, const float* w2, const float* b2, const float* w3,
                                     const float* b3, float* out, float* x0, float* h1, float* h2, void* stream) {
  const int rc = conf_head_check(x, N, C0, H, W, H1, H2, NO);
  if (rc != LT_OK) return rc;
  LT_REQUIRE(w1 && b1 && w2 && b2 && w3 && b3 && out && x0 && h1 && h2, "conf_head_tail_fwd: null pointer");
  const HeadMap m{x, N, C0, H, W, {xs_n, xs_c, xs_h, xs_w}};
  conf_head_fwd_kernel<<<N, 256, (size_t)(C0 + H1 + H2) * sizeof(float), (cudaStream_t)stream>>>(m, H1, H2, NO, w1, b1, w2, b2, w3, b3,
                                                                                                 out, x0, h1, h2);
  LT_CHECK_LAUNCH("conf_head_fwd_kernel");
  return LT_OK;
}

extern "C" size_t lt_conf_head_tail_bwd_workspace_bytes(int N, int C0, int H1, int H2, int NO) {
  return (N > 0 && C0 > 0 && H1 > 0 && H2 > 0 && NO > 0) ? (size_t)N * head_ws_row(C0, H1, H2, NO) * sizeof(float) : 0;
}

extern "C" int lt_conf_head_tail_bwd(const float* x, int N, int C0, int H, int W, long xs_n, long xs_c, long xs_h, long xs_w, long gs_n,
                                     long gs_c, long gs_h, long gs_w, int H1, int H2, int NO, const float* w1, const float* w2,
                                     const float* w3, const float* x0, const float* h1, const float* h2, const float* y,
                                     const float* grad_y, float* grad_x, float* dw1, float* db1, float* dw2, float* db2, float* dw3,
                                     float* db3, void* workspace, size_t workspace_bytes, void* stream) {
  const int rc = conf_head_check(x, N, C0, H, W, H1, H2, NO);
  if (rc != LT_OK) return rc;
  LT_REQUIRE(w1 && w2 && w3 && x0 && h1 && h2 && y && grad_y && grad_x && dw1 && db1 && dw2 && db2 && dw3 && db3 && workspace,
             "conf_head_tail_bwd: null pointer");
  const size_t need = lt_conf_head_tail_bwd_workspace_bytes(N, C0, H1, H2, NO);
  LT_REQUIRE(workspace_bytes >= need, "conf_head_tail_bwd: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = static_cast<float*>(workspace);
  conf_head_bwd_rows_kernel<<<N, 256, (size_t)(NO + H2 + H1) * sizeof(float), st>>>(C0, H1, H2, NO, w1, w2, w3, h1, h2, y, grad_y, ws);
  LT_CHECK_LAUNCH("conf_head_bwd_rows_kernel");
  const long nw = (long)H1 * C0 + H1 + (long)H2 * H1 + H2 + (long)NO * H2 + NO;
  conf_head_wgrad_kernel<<<ceil_div(nw, 256), 256, 0, st>>>(ws, x0, h1, h2, N, C0, H1, H2, NO, nw, dw1, db1, dw2, db2, dw3, db3);
  LT_CHECK_LAUNCH("conf_head_wgrad_kernel");
  const HeadMap m{x, N, C0, H, W, {xs_n, xs_c, xs_h, xs_w}};
  const long total = (long)N * C0 * H * W;
  conf_head_dx_kernel<<<ceil_div(total, 256), 256, 0, st>>>(m, make_long4(gs_n, gs_c, gs_h, gs_w), ws, H1, H2, NO, grad_x, total);
  LT_CHECK_LAUNCH("conf_head_dx_kernel");
  return LT_OK;
}

extern "C" int lt_view_normalize_bwd(const float* conf, const float* grad, float* grad_conf, int B, int V, int C, void* stream) {
  LT_REQUIRE(conf && grad && grad_conf && B > 0 && V > 0 && C > 0, "view_normalize_bwd: bad arguments");
  view_normalize_bwd_kernel<<<ceil_div((long)B * C, 128), 128, 0, (cudaStream_t)stream>>>(conf, grad, grad_conf, B, V, C);
  LT_CHECK_LAUNCH("view_normalize_bwd_kernel");
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

// The forward kernel's and (grad_y not null) the backward kernels' per-item code on host pointers, row by row as the CTAs run it.
extern "C" int lt_test_conf_head_tail_host(const float* x, int N, int C0, int H, int W, long xs_n, long xs_c, long xs_h, long xs_w,
                                           long gs_n, long gs_c, long gs_h, long gs_w, int H1, int H2, int NO, const float* w1,
                                           const float* b1, const float* w2, const float* b2, const float* w3, const float* b3, float* out,
                                           float* x0, float* h1, float* h2, const float* grad_y, float* grad_x, float* dw1, float* db1,
                                           float* dw2, float* db2, float* dw3, float* db3) {
  const int rc = conf_head_check(x, N, C0, H, W, H1, H2, NO);
  if (rc != LT_OK) return rc;
  LT_REQUIRE(w1 && b1 && w2 && b2 && w3 && b3 && out && x0 && h1 && h2, "test_conf_head_tail_host: null pointer");
  LT_REQUIRE(!grad_y || (grad_x && dw1 && db1 && dw2 && db2 && dw3 && db3), "test_conf_head_tail_host: null gradient pointer");
  const HeadMap m{x, N, C0, H, W, {xs_n, xs_c, xs_h, xs_w}};
  for (int n = 0; n < N; ++n) {
    float* r0 = x0 + (long)n * C0;
    float* r1 = h1 + (long)n * H1;
    float* r2 = h2 + (long)n * H2;
    for (int c = 0; c < C0; ++c) r0[c] = head_gap_item(m, n, c);
    for (int o = 0; o < H1; ++o) r1[o] = hidden_relu<true>(linear_item(w1, b1, r0, C0, o));
    for (int o = 0; o < H2; ++o) r2[o] = hidden_relu<true>(linear_item(w2, b2, r1, H1, o));
    for (int o = 0; o < NO; ++o) out[(long)n * NO + o] = sigmoid_f(linear_item(w3, b3, r2, H2, o));
  }
  if (!grad_y) return LT_OK;
  const long row = head_ws_row(C0, H1, H2, NO);
  float* ws = static_cast<float*>(malloc((size_t)N * row * sizeof(float)));
  LT_REQUIRE(ws, "test_conf_head_tail_host: out of memory");
  for (int n = 0; n < N; ++n) {
    float* d3 = ws + n * row;
    float* d2 = d3 + NO;
    float* d1 = d2 + H2;
    for (int o = 0; o < NO; ++o) d3[o] = sigmoid_bwd(grad_y[(long)n * NO + o], out[(long)n * NO + o]);
    for (int i = 0; i < H2; ++i) d2[i] = !(h2[(long)n * H2 + i] <= 0.0f) ? linear_bwd_item(w3, d3, NO, H2, i) : 0.0f;
    for (int i = 0; i < H1; ++i) d1[i] = !(h1[(long)n * H1 + i] <= 0.0f) ? linear_bwd_item(w2, d2, H2, H1, i) : 0.0f;
    for (int i = 0; i < C0; ++i) d1[H1 + i] = linear_bwd_item(w1, d1, H1, C0, i);
  }
  const long nw = (long)H1 * C0 + H1 + (long)H2 * H1 + H2 + (long)NO * H2 + NO;
  for (long e = 0; e < nw; ++e) head_wgrad_item(ws, x0, h1, h2, N, C0, H1, H2, NO, e, dw1, db1, dw2, db2, dw3, db3);
  const long gs[4] = {gs_n, gs_c, gs_h, gs_w};
  for (long i = 0; i < (long)N * C0 * H * W; ++i) head_dx_item(m, gs, ws, C0, H1, H2, NO, grad_x, i);
  free(ws);
  return LT_OK;
}

extern "C" int lt_test_view_normalize_bwd_host(const float* conf, const float* grad, float* grad_conf, int B, int V, int C) {
  LT_REQUIRE(conf && grad && grad_conf && B > 0 && V > 0 && C > 0, "test_view_normalize_bwd_host: bad arguments");
  for (int b = 0; b < B; ++b)
    for (int c = 0; c < C; ++c) view_normalize_bwd_item(conf, grad, grad_conf, V, C, b, c);
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
