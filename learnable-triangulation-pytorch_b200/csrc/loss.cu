// Volumetric cross-entropy loss of the training recipe (VolumetricCELoss, loss.py:52-80; train.py:222-230) and its backward.
//
// Per (sample b, joint j) the reference takes the voxel nearest to the ground-truth point -- torch.argmin over the rounded fp32
// distances sqrt((dx*dx + dy*dy) + dz*dz) of every voxel of the coordinate volume -- and adds v * -log(p + 1e-6) of the softmaxed
// volume there.  Here:
//   ce_search_kernel  one pass over the coordinate volume per sample: each thread keeps VPT voxels' coordinates in registers across
//                     all J joints (joint groups of JG) and folds every distance into a 64-bit key (distance key << 32 | voxel);
//                     the per-block minimum per joint goes to workspace[b][j] by atomicMin (a minimum is independent of the order
//                     in which it is taken: deterministic);
//   ce_finish_kernel  one CTA: index / picked probability / term per (b, j), then the terms summed in the reference's order;
//   ce_bwd_kernel     writes the whole gradient in one pass: zeros, and the autograd value at the picked voxel.
// The distance, the key, the term and the gradient value are __host__ __device__ helpers that the host test hook runs as well.
#include "common.cuh"
#include <math.h>
#include <string.h>

namespace lt {

constexpr int kCeThreads = 256;
constexpr int kCeVpt = 4;                        // voxels per thread
constexpr int kCeChunk = kCeThreads * kCeVpt;    // voxels per CTA
constexpr int kCeJg = 8;                         // joints per group (keys held in registers)

// fp32 arithmetic of the reference, one rounding per operation (no FMA contraction on the device; the host compiler is not asked
// for FMA either: these are the plain operators there).
__host__ __device__ __forceinline__ float ce_add(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ float ce_sub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ __forceinline__ float ce_mul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ float ce_div(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
__host__ __device__ __forceinline__ float ce_sqrt(float a) {
#ifdef __CUDA_ARCH__
  return __fsqrt_rn(a);
#else
  return sqrtf(a);
#endif
}
__host__ __device__ __forceinline__ unsigned ce_float_bits(float a) {
#ifdef __CUDA_ARCH__
  return __float_as_uint(a);
#else
  unsigned u;
  memcpy(&u, &a, sizeof u);
  return u;
#endif
}

// loss.py:68: sqrt(((coord - kp) ** 2).sum(-1)), the three squares summed left to right
__host__ __device__ __forceinline__ float ce_distance(float cx, float cy, float cz, float kx, float ky, float kz) {
  const float dx = ce_sub(cx, kx), dy = ce_sub(cy, ky), dz = ce_sub(cz, kz);
  return ce_sqrt(ce_add(ce_add(ce_mul(dx, dx), ce_mul(dy, dy)), ce_mul(dz, dz)));
}

// torch.argmin order (loss.py:71) as one unsigned 64-bit key, smaller = better: a NaN distance beats every number, distances
// (>= 0, so their bit patterns order like the values, +inf included) order by value, and ties -- equal distances or two NaNs --
// go to the smaller flat voxel index.  ~0ull is larger than every key.
__host__ __device__ __forceinline__ unsigned long long ce_key(float d, unsigned voxel) {
  const unsigned k = d != d ? 0u : ce_float_bits(d) + 1u;
  return ((unsigned long long)k << 32) | voxel;
}

// loss.py:76: validity[0] * (-torch.log(p + 1e-6)), computed whatever v is (0 * NaN stays NaN, as in the reference)
__host__ __device__ __forceinline__ float ce_term(float p, float v) { return ce_mul(v, -logf(ce_add(p, 1e-6f))); }

// What autograd hands the picked voxel in the reference (loss.py:76,80 backward): Div by n, Mul by v, Neg, Log.
__host__ __device__ __forceinline__ float ce_grad(float g, float p, float v, float n) {
  return ce_div(-ce_mul(ce_div(g, n), v), ce_add(p, 1e-6f));
}

__device__ __forceinline__ unsigned long long ce_min(unsigned long long a, unsigned long long b) { return b < a ? b : a; }

// grid (ceil(nvox / kCeChunk), B); best[B][J] holds ~0 on entry (cudaMemsetAsync) and the minimum key on exit
__global__ void __launch_bounds__(kCeThreads) ce_search_kernel(const float* __restrict__ coord, const float* __restrict__ kp, int J,
                                                               long nvox, unsigned long long* __restrict__ best) {
  __shared__ unsigned long long s_key[kCeJg][kCeThreads / 32];
  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long base = (long)blockIdx.x * kCeChunk + threadIdx.x;
  const float* cb = coord + (long)b * nvox * 3;
  float cx[kCeVpt], cy[kCeVpt], cz[kCeVpt];
#pragma unroll
  for (int k = 0; k < kCeVpt; ++k) {
    const long v = base + (long)k * kCeThreads;
    const bool ok = v < nvox;
    cx[k] = ok ? cb[v * 3] : 0.0f;
    cy[k] = ok ? cb[v * 3 + 1] : 0.0f;
    cz[k] = ok ? cb[v * 3 + 2] : 0.0f;
  }
  const float* kb = kp + (long)b * J * 3;
  for (int j0 = 0; j0 < J; j0 += kCeJg) {
    unsigned long long key[kCeJg];
#pragma unroll
    for (int g = 0; g < kCeJg; ++g) {
      key[g] = ~0ull;
      const int j = j0 + g;
      if (j >= J) continue;
      const float kx = kb[j * 3], ky = kb[j * 3 + 1], kz = kb[j * 3 + 2];
#pragma unroll
      for (int k = 0; k < kCeVpt; ++k) {
        const long v = base + (long)k * kCeThreads;
        if (v < nvox) key[g] = ce_min(key[g], ce_key(ce_distance(cx[k], cy[k], cz[k], kx, ky, kz), (unsigned)v));
      }
    }
#pragma unroll
    for (int g = 0; g < kCeJg; ++g) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) key[g] = ce_min(key[g], __shfl_xor_sync(0xffffffffu, key[g], o));
      if (lane == 0) s_key[g][warp] = key[g];
    }
    __syncthreads();
    if (threadIdx.x < kCeJg && j0 + threadIdx.x < J) {
      unsigned long long m = s_key[threadIdx.x][0];
#pragma unroll
      for (int w = 1; w < kCeThreads / 32; ++w) m = ce_min(m, s_key[threadIdx.x][w]);
      atomicMin(best + (long)b * J + j0 + threadIdx.x, m);
    }
    __syncthreads();
  }
}

// One CTA: per (b, j) the chosen voxel, its probability and the term; thread 0 sums the terms sample by sample, joint by joint,
// from 0 in fp32 (the reference's `loss +=` loop, loss.py:61-77) and divides by B * J (:80).
__global__ void __launch_bounds__(kCeThreads) ce_finish_kernel(const float* __restrict__ probs, const float* __restrict__ validity,
                                                               const unsigned long long* __restrict__ best, int rows, long nvox,
                                                               float* __restrict__ loss, int* __restrict__ index,
                                                               float* __restrict__ picked) {
  __shared__ float s_term[kCeThreads];
  float acc = 0.0f;
  for (int r0 = 0; r0 < rows; r0 += kCeThreads) {
    const int r = r0 + threadIdx.x;
    if (r < rows) {
      const unsigned idx = (unsigned)(best[r] & 0xffffffffull);
      const float p = probs[(long)r * nvox + idx];
      index[r] = (int)idx;
      picked[r] = p;
      s_term[threadIdx.x] = ce_term(p, validity[r]);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const int n = min(kCeThreads, rows - r0);
      for (int t = 0; t < n; ++t) acc = ce_add(acc, s_term[t]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss = ce_div(acc, (float)rows);
}

// grid (column blocks, rows): row r = (b, j) of grad_probs gets zeros and, at index[r], ce_grad.  VEC: nvox % 4 == 0 (float4 stores).
template <bool VEC>
__global__ void __launch_bounds__(kCeThreads) ce_bwd_kernel(const float* __restrict__ grad_loss, const int* __restrict__ index,
                                                            const float* __restrict__ picked, const float* __restrict__ validity,
                                                            float* __restrict__ grad, int rows, long nvox) {
  const float g = *grad_loss;
  for (int r = blockIdx.y; r < rows; r += gridDim.y) {
    const long idx = index[r];
    const float val = ce_grad(g, picked[r], validity[r], (float)rows);
    float* row = grad + (long)r * nvox;
    if (VEC) {
      const long n4 = nvox >> 2;
      for (long q = (long)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (long)gridDim.x * blockDim.x) {
        float4 o = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        const long d = idx - q * 4;
        if (d == 0) o.x = val;
        if (d == 1) o.y = val;
        if (d == 2) o.z = val;
        if (d == 3) o.w = val;
        reinterpret_cast<float4*>(row)[q] = o;
      }
    } else {
      for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < nvox; e += (long)gridDim.x * blockDim.x)
        row[e] = e == idx ? val : 0.0f;
    }
  }
}

}  // namespace lt

using namespace lt;

extern "C" size_t lt_volumetric_ce_workspace_bytes(int B, int J, long nvox) {
  (void)nvox;
  return B > 0 && J > 0 ? (size_t)B * J * sizeof(unsigned long long) : 0;
}

static int ce_check(const float* probs, const float* coord, const float* kp, const float* validity, int B, int J, long nvox) {
  LT_REQUIRE(probs && coord && kp && validity, "volumetric_ce: null pointer");
  LT_REQUIRE(B > 0 && J > 0 && nvox > 0, "volumetric_ce: bad sizes");
  LT_REQUIRE(nvox < 0x7fffffffL, "volumetric_ce: nvox must be < 2^31");
  return LT_OK;
}

extern "C" int lt_volumetric_ce_fwd(const float* probs, const float* coord, const float* keypoints_gt, const float* validity,
                                    float* loss, int* index, float* picked, void* workspace, size_t workspace_bytes, int B, int J,
                                    long nvox, void* stream) {
  const int rc = ce_check(probs, coord, keypoints_gt, validity, B, J, nvox);
  if (rc != LT_OK) return rc;
  LT_REQUIRE(loss && index && picked && workspace, "volumetric_ce: null pointer");
  LT_REQUIRE(workspace_bytes >= lt_volumetric_ce_workspace_bytes(B, J, nvox), "volumetric_ce: workspace too small");
  LT_REQUIRE(B <= 65535, "volumetric_ce: B must be <= 65535");
  const cudaStream_t s = (cudaStream_t)stream;
  unsigned long long* best = reinterpret_cast<unsigned long long*>(workspace);
  if (cudaMemsetAsync(best, 0xff, (size_t)B * J * sizeof(unsigned long long), s) != cudaSuccess)
    return fail(LT_ERR_CUDA, "volumetric_ce: cudaMemsetAsync failed");
  ce_search_kernel<<<dim3(ceil_div(nvox, kCeChunk), B), kCeThreads, 0, s>>>(coord, keypoints_gt, J, nvox, best);
  LT_CHECK_LAUNCH("ce_search_kernel");
  ce_finish_kernel<<<1, kCeThreads, 0, s>>>(probs, validity, best, B * J, nvox, loss, index, picked);
  LT_CHECK_LAUNCH("ce_finish_kernel");
  return LT_OK;
}

extern "C" int lt_volumetric_ce_bwd(const float* grad_loss, const int* index, const float* picked, const float* validity,
                                    float* grad_probs, int B, int J, long nvox, void* stream) {
  LT_REQUIRE(grad_loss && index && picked && validity && grad_probs, "volumetric_ce_bwd: null pointer");
  LT_REQUIRE(B > 0 && J > 0 && nvox > 0, "volumetric_ce_bwd: bad sizes");
  const int rows = B * J;
  const bool vec = nvox % 4 == 0 && (reinterpret_cast<uintptr_t>(grad_probs) & 15) == 0;
  const long per_row = vec ? nvox / 4 : nvox;
  // ~4 stores per thread; rows beyond 65535 are walked by the grid-stride loop
  const dim3 grid(ceil_div(per_row, kCeThreads * 4), rows < 65535 ? rows : 65535);
  if (vec) ce_bwd_kernel<true><<<grid, kCeThreads, 0, (cudaStream_t)stream>>>(grad_loss, index, picked, validity, grad_probs, rows, nvox);
  else ce_bwd_kernel<false><<<grid, kCeThreads, 0, (cudaStream_t)stream>>>(grad_loss, index, picked, validity, grad_probs, rows, nvox);
  LT_CHECK_LAUNCH("ce_bwd_kernel");
  return LT_OK;
}

// test hook: the same distance / key / term / gradient code on the CPU (host pointers)
extern "C" int lt_test_volumetric_ce_host(const float* probs, const float* coord, const float* keypoints_gt, const float* validity,
                                          float* loss, int* index, float* picked, const float* grad_loss, float* grad_probs, int B,
                                          int J, long nvox) {
  const int rc = ce_check(probs, coord, keypoints_gt, validity, B, J, nvox);
  if (rc != LT_OK) return rc;
  LT_REQUIRE(loss && index && picked, "test_volumetric_ce_host: null pointer");
  LT_REQUIRE(!grad_probs || grad_loss, "test_volumetric_ce_host: grad_probs needs grad_loss");
  float acc = 0.0f;
  for (int b = 0; b < B; ++b) {
    for (int j = 0; j < J; ++j) {
      const float* k = keypoints_gt + ((long)b * J + j) * 3;
      unsigned long long m = ~0ull;
      for (long v = 0; v < nvox; ++v) {
        const float* c = coord + ((long)b * nvox + v) * 3;
        const unsigned long long key = ce_key(ce_distance(c[0], c[1], c[2], k[0], k[1], k[2]), (unsigned)v);
        if (key < m) m = key;
      }
      const long r = (long)b * J + j;
      index[r] = (int)(m & 0xffffffffull);
      picked[r] = probs[r * nvox + index[r]];
      acc = ce_add(acc, ce_term(picked[r], validity[r]));
    }
  }
  *loss = ce_div(acc, (float)(B * J));
  if (grad_probs) {
    for (long r = 0; r < (long)B * J; ++r)
      for (long v = 0; v < nvox; ++v)
        grad_probs[r * nvox + v] = v == index[r] ? ce_grad(*grad_loss, picked[r], validity[r], (float)(B * J)) : 0.0f;
  }
  return LT_OK;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Keypoint criteria of the training recipe (KeypointsMSELoss, KeypointsMSESmoothLoss, KeypointsMAELoss, KeypointsL2Loss,
// loss.py:7-49) and their backward.  pred, gt [n][dim], validity [n]; every term is formed in float64 from the float32 inputs and
// multiplied by v whatever v is (a non-finite residual at v = 0 gives NaN, as in the reference).
//   kp_loss_fwd_kernel  one CTA: thread t sums the terms (and v) of points t, t + kKpThreads, ... in float64, then a fixed tree
//                       over the threads: the same sum on every call.  The divisor dim * max(1, sum v) (L2: max(1, sum v)) stays
//                       on the device for the backward; the loss is the float64 quotient rounded to float32.
//   kp_loss_bwd_kernel  one thread per element: g / divisor times the derivative autograd takes through the reference formula.
// The term, the derivative and the summation order are shared with the host test hook.
namespace lt {

constexpr int kKpThreads = 256;
enum { kKpMse = 0, kKpMseSmooth = 1, kKpMae = 2, kKpL2 = 3 };

// one point's term: MSE sum_d (gt - pred)^2 v; MSE_SMOOTH the same with each d = (gt - pred)^2 v > t replaced by d^0.1 t^0.9
// (t09 = t^0.9); MAE sum_d |gt - pred| v; L2 sqrt(sum_d (gt - pred)^2 v)
__host__ __device__ __forceinline__ double kp_term(const float* pred, const float* gt, double v, int dim, int kind, double t,
                                                   double t09) {
  double acc = 0.0;
  for (int k = 0; k < dim; ++k) {
    const double r = (double)gt[k] - (double)pred[k];
    if (kind == kKpMae) {
      acc += fabs(r) * v;
    } else {
      double d = r * r * v;
      if (kind == kKpMseSmooth && d > t) d = pow(d, 0.1) * t09;
      acc += d;
    }
  }
  return kind == kKpL2 ? sqrt(acc) : acc;
}

// d loss / d pred[k] times g, where g = grad_loss / divisor: autograd's chain through the reference formula (sub, pow 2 or abs,
// mul by v; MSE_SMOOTH's pow 0.1 on the replaced branch; L2's sum over d and sqrt, whose backward g / (2 sqrt(s)) is inf at s = 0,
// so a zero-length residual gives NaN as in torch)
__host__ __device__ __forceinline__ double kp_grad(const float* pred, const float* gt, double v, int k, int dim, int kind, double t,
                                                   double t09, double g) {
  const double r = (double)gt[k] - (double)pred[k];
  if (kind == kKpMae) return -(g * v * (double)((r > 0.0) - (r < 0.0)));      // torch's sgn: 0 at 0 and at NaN
  double gd = g;
  if (kind == kKpMseSmooth) {
    const double d = r * r * v;
    if (d > t) gd = g * t09 * (0.1 * pow(d, -0.9));
  } else if (kind == kKpL2) {
    double s = 0.0;
    for (int q = 0; q < dim; ++q) {
      const double rq = (double)gt[q] - (double)pred[q];
      s += rq * rq * v;
    }
    gd = g / (2.0 * sqrt(s));
  }
  return -(gd * v * (2.0 * r));
}

__host__ __device__ __forceinline__ double kp_divisor(double sum_v, int dim, int kind) {
  const double m = sum_v > 1.0 ? sum_v : 1.0;          // python's max(1, x): 1 for a NaN sum as well
  return kind == kKpL2 ? m : (double)dim * m;
}

__global__ void __launch_bounds__(kKpThreads) kp_loss_fwd_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                                                 const float* __restrict__ validity, int n, int dim, int kind,
                                                                 double t, double t09, float* __restrict__ loss,
                                                                 double* __restrict__ norm) {
  __shared__ double s_term[kKpThreads], s_v[kKpThreads];
  double acc = 0.0, acc_v = 0.0;
  for (int p = threadIdx.x; p < n; p += kKpThreads) {
    const double v = validity[p];
    acc += kp_term(pred + (long)p * dim, gt + (long)p * dim, v, dim, kind, t, t09);
    acc_v += v;
  }
  s_term[threadIdx.x] = acc;
  s_v[threadIdx.x] = acc_v;
  __syncthreads();
  for (int s = kKpThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      s_term[threadIdx.x] += s_term[threadIdx.x + s];
      s_v[threadIdx.x] += s_v[threadIdx.x + s];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double d = kp_divisor(s_v[0], dim, kind);
    *norm = d;
    *loss = (float)(s_term[0] / d);
  }
}

__global__ void __launch_bounds__(kKpThreads) kp_loss_bwd_kernel(const float* __restrict__ grad_loss, const float* __restrict__ pred,
                                                                 const float* __restrict__ gt, const float* __restrict__ validity,
                                                                 const double* __restrict__ norm, float* __restrict__ grad_pred,
                                                                 int n, int dim, int kind, double t, double t09) {
  const long i = (long)blockIdx.x * kKpThreads + threadIdx.x;
  if (i >= (long)n * dim) return;
  const long p = i / dim;
  const double g = (double)*grad_loss / *norm;
  grad_pred[i] = (float)kp_grad(pred + p * dim, gt + p * dim, validity[p], (int)(i - p * dim), dim, kind, t, t09, g);
}

}  // namespace lt

static int kp_check(const float* pred, const float* gt, const float* validity, int kind, int n_points, int dim) {
  LT_REQUIRE(pred && gt && validity, "keypoints_loss: null pointer");
  LT_REQUIRE(n_points > 0 && dim > 0, "keypoints_loss: bad sizes");
  LT_REQUIRE((long)n_points * dim < 0x7fffffffL, "keypoints_loss: n_points * dim must be < 2^31");
  LT_REQUIRE(kind >= kKpMse && kind <= kKpL2, "keypoints_loss: unknown kind %d", kind);
  return LT_OK;
}

extern "C" int lt_keypoints_loss_fwd(const float* pred, const float* gt, const float* validity, float* loss, double* norm, int kind,
                                     double threshold, int n_points, int dim, void* stream) {
  const int rc = kp_check(pred, gt, validity, kind, n_points, dim);
  if (rc != LT_OK) return rc;
  LT_REQUIRE(loss && norm, "keypoints_loss: null pointer");
  kp_loss_fwd_kernel<<<1, kKpThreads, 0, (cudaStream_t)stream>>>(pred, gt, validity, n_points, dim, kind, threshold,
                                                                 pow(threshold, 0.9), loss, norm);
  LT_CHECK_LAUNCH("kp_loss_fwd_kernel");
  return LT_OK;
}

extern "C" int lt_keypoints_loss_bwd(const float* grad_loss, const float* pred, const float* gt, const float* validity,
                                     const double* norm, float* grad_pred, int kind, double threshold, int n_points, int dim,
                                     void* stream) {
  const int rc = kp_check(pred, gt, validity, kind, n_points, dim);
  if (rc != LT_OK) return rc;
  LT_REQUIRE(grad_loss && norm && grad_pred, "keypoints_loss_bwd: null pointer");
  kp_loss_bwd_kernel<<<ceil_div((long)n_points * dim, kKpThreads), kKpThreads, 0, (cudaStream_t)stream>>>(
      grad_loss, pred, gt, validity, norm, grad_pred, n_points, dim, kind, threshold, pow(threshold, 0.9));
  LT_CHECK_LAUNCH("kp_loss_bwd_kernel");
  return LT_OK;
}

// test hook: the kernels' term, derivative and summation order on the CPU (host pointers)
extern "C" int lt_test_keypoints_loss_host(const float* pred, const float* gt, const float* validity, float* loss, double* norm,
                                           const float* grad_loss, float* grad_pred, int kind, double threshold, int n_points,
                                           int dim) {
  const int rc = kp_check(pred, gt, validity, kind, n_points, dim);
  if (rc != LT_OK) return rc;
  LT_REQUIRE(loss && norm, "test_keypoints_loss_host: null pointer");
  LT_REQUIRE(!grad_pred || grad_loss, "test_keypoints_loss_host: grad_pred needs grad_loss");
  const double t09 = pow(threshold, 0.9);
  double term[kKpThreads], sv[kKpThreads];
  for (int tid = 0; tid < kKpThreads; ++tid) {
    term[tid] = sv[tid] = 0.0;
    for (int p = tid; p < n_points; p += kKpThreads) {
      const double v = validity[p];
      term[tid] += kp_term(pred + (long)p * dim, gt + (long)p * dim, v, dim, kind, threshold, t09);
      sv[tid] += v;
    }
  }
  for (int s = kKpThreads / 2; s > 0; s >>= 1) {
    for (int tid = 0; tid < s; ++tid) {
      term[tid] += term[tid + s];
      sv[tid] += sv[tid + s];
    }
  }
  *norm = kp_divisor(sv[0], dim, kind);
  *loss = (float)(term[0] / *norm);
  if (grad_pred) {
    const double g = (double)*grad_loss / *norm;
    for (long i = 0; i < (long)n_points * dim; ++i) {
      const long p = i / dim;
      grad_pred[i] = (float)kp_grad(pred + p * dim, gt + p * dim, validity[p], (int)(i - p * dim), dim, kind, threshold, t09, g);
    }
  }
  return LT_OK;
}
