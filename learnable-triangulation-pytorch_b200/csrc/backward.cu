// Backward passes of the two custom ops of the volumetric path (SURVEY section 8f row 1, first stage): what
// `total_loss.backward()` (train.py:236) needs from op.unproject_heatmaps (op.py:99-166) and
// op.integrate_tensor_3d_with_coordinates (op.py:84-96) when they run on the native kernels inside the torch training
// graph (`backend="hybrid"`: torch convolutions, native custom ops).  Gradients flow to the feature maps (and to the
// per-view confidences of the `conf` aggregation) and to the V2V logits; projection matrices and coordinate volumes carry
// no gradient in the reference either (they are built from numpy inputs).
//
// Unprojection backward (HBM / atomics bound): one thread per (voxel, 4 channels) recomputes the four bilinear taps of every
// view exactly as the forward does, re-aggregates, forms the per-view sample gradient
//     sum:      g                      conf:   g * conf_v   (and d conf_v += g * s_v)
//     max:      g on the arg-max view  softmax: g * p_v * (1 + s_v - out),  p = softmax_v(s)
// and scatters it with 16-byte vector atomics (red.global.add.v4.f32) into the channels-last feature gradient.
// Soft-argmax backward (HBM bound, NCDHW like the op-level API): with t_i = g_vol_i + <g_kp, x_i>,
//     softmax: d logit_i = mult * p_i * (t_i - sum_k p_k t_k)      ReLU: d logit_i = mult * [mult * logit_i > 0] * t_i
#include "common.cuh"
#include <math.h>

// The per-item bodies are __host__ __device__: the kernels run them on the GPU, and lt_test_*_bwd_host (bottom of the file)
// runs the SAME code on the CPU so that `-m "not gpu"` tests can check the gradient arithmetic against torch autograd
// without a GPU (test hook only: nothing on the product path calls it).
#ifdef __CUDA_ARCH__
#define LT_LD(p) __ldg(p)
#else
#define LT_LD(p) (*(p))
#endif

namespace lt {

struct BwdTaps {
  int o[4];
  float w[4];     // bilinear weight, 0 where the tap is outside the map or the depth test failed
};

// identical arithmetic to make_taps() in unproject.cu (op.py:116-135, multiview.py:89-110)
__host__ __device__ __forceinline__ BwdTaps bwd_taps(const float* __restrict__ P, float X, float Y, float Z, int h, int w) {
  BwdTaps t;
  float px = fmaf(Z, P[2], fmaf(Y, P[1], X * P[0])) + P[3];
  float py = fmaf(Z, P[6], fmaf(Y, P[5], X * P[4])) + P[7];
  float pz = fmaf(Z, P[10], fmaf(Y, P[9], X * P[8])) + P[11];
  const bool depth_ok = !(pz <= 0.0f);
  if (pz == 0.0f) pz = 1.0f;
  const float x = px / pz, y = py / pz;
  const float gx = 2.0f * (x / (float)h - 0.5f);      // op.py:128-129: x by the map HEIGHT, y by the WIDTH
  const float gy = 2.0f * (y / (float)w - 0.5f);
  const float ix = ((gx + 1.0f) / 2.0f) * (float)(w - 1);
  const float iy = ((gy + 1.0f) / 2.0f) * (float)(h - 1);
  const float x0 = floorf(ix), y0 = floorf(iy);
  const float x1 = x0 + 1.0f, y1 = y0 + 1.0f;
  const float wm = (float)(w - 1), hm = (float)(h - 1);
  const bool vx0 = (x0 >= 0.0f) && (x0 <= wm), vx1 = (x1 >= 0.0f) && (x1 <= wm);
  const bool vy0 = (y0 >= 0.0f) && (y0 <= hm), vy1 = (y1 >= 0.0f) && (y1 <= hm);
  const int xi = (int)fminf(fmaxf(x0, -2.0f), wm + 1.0f), yi = (int)fminf(fmaxf(y0, -2.0f), hm + 1.0f);
  const int xa = xi < 0 ? 0 : (xi > w - 1 ? w - 1 : xi), xb = xi + 1 < 0 ? 0 : (xi + 1 > w - 1 ? w - 1 : xi + 1);
  const int ya = yi < 0 ? 0 : (yi > h - 1 ? h - 1 : yi), yb = yi + 1 < 0 ? 0 : (yi + 1 > h - 1 ? h - 1 : yi + 1);
  t.o[0] = ya * w + xa; t.o[1] = ya * w + xb; t.o[2] = yb * w + xa; t.o[3] = yb * w + xb;
  t.w[0] = (depth_ok && vx0 && vy0) ? (x1 - ix) * (y1 - iy) : 0.0f;
  t.w[1] = (depth_ok && vx1 && vy0) ? (ix - x0) * (y1 - iy) : 0.0f;
  t.w[2] = (depth_ok && vx0 && vy1) ? (x1 - ix) * (iy - y0) : 0.0f;
  t.w[3] = (depth_ok && vx1 && vy1) ? (ix - x0) * (iy - y0) : 0.0f;
  return t;
}

__host__ __device__ __forceinline__ float4 sample4(const float* __restrict__ fmap, int C, int c0, const BwdTaps& t) {
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (t.w[k] != 0.0f) {
      const float4 q = LT_LD(reinterpret_cast<const float4*>(fmap + (long)t.o[k] * C + c0));
      s.x = fmaf(q.x, t.w[k], s.x); s.y = fmaf(q.y, t.w[k], s.y); s.z = fmaf(q.z, t.w[k], s.z); s.w = fmaf(q.w, t.w[k], s.w);
    }
  return s;
}

__host__ __device__ __forceinline__ void red_add_v4(float* addr, float4 v) {
#ifdef __CUDA_ARCH__
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
#else
  addr[0] += v.x; addr[1] += v.y; addr[2] += v.z; addr[3] += v.w;
#endif
}
__host__ __device__ __forceinline__ void acc_add(float* addr, float v) {
#ifdef __CUDA_ARCH__
  atomicAdd(addr, v);
#else
  *addr += v;
#endif
}

__host__ __device__ __forceinline__ void scatter4(float* __restrict__ gmap, int C, int c0, const BwdTaps& t, float4 gs) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (t.w[k] != 0.0f)
      red_add_v4(gmap + (long)t.o[k] * C + c0, make_float4(gs.x * t.w[k], gs.y * t.w[k], gs.z * t.w[k], gs.w * t.w[k]));
}

struct UnprojBwdParams {
  const float* features;   // [B][V][h][w][C]
  const float* proj;       // [B][V][12]
  const float* coord;      // [B][nvox][3]
  const float* conf;       // [B][V][C] or null
  const float* grad_out;   // [B][nvox][C]
  float* grad_features;    // [B][V][h][w][C], accumulated into (caller zero-fills)
  float* grad_conf;        // [B][V][C] or null, accumulated into
  int B, V, C, h, w, agg;
  long nvox;
};

constexpr int kBwdSmemViews = 64;

// one (voxel, 4-channel quad) of sample b.  projs: the sample's first kBwdSmemViews projection matrices (shared memory on
// the GPU) or null; gconf_acc: [V][C] accumulator of d conf (shared memory on the GPU, the output itself on the host) or null
__host__ __device__ __forceinline__ void unproject_bwd_item(const UnprojBwdParams& p, int b, long it, const float* projs, float* gconf_acc) {
  const int quads = p.C >> 2;
  const long map_elems = (long)p.h * p.w * p.C;
  const bool want_gconf = gconf_acc != nullptr && p.agg == LT_AGG_CONF;
  {
    const long vox = it / quads;
    const int c0 = (int)(it % quads) * 4;
    const float* cp = p.coord + ((long)b * p.nvox + vox) * 3;
    const float X = LT_LD(cp), Y = LT_LD(cp + 1), Z = LT_LD(cp + 2);
    const float4 g = LT_LD(reinterpret_cast<const float4*>(p.grad_out + ((long)b * p.nvox + vox) * p.C + c0));
    const float* fb = p.features + (long)b * p.V * map_elems;
    float* gb = p.grad_features + (long)b * p.V * map_elems;
    auto view_proj = [&](int v) { return (projs != nullptr && v < kBwdSmemViews) ? projs + v * 12 : p.proj + ((long)b * p.V + v) * 12; };

    if (p.agg == LT_AGG_SUM || p.agg == LT_AGG_CONF) {
      for (int v = 0; v < p.V; ++v) {
        const BwdTaps t = bwd_taps(view_proj(v), X, Y, Z, p.h, p.w);
        float4 gs = g;
        if (p.agg == LT_AGG_CONF) {
          const float4 cf = LT_LD(reinterpret_cast<const float4*>(p.conf + ((long)b * p.V + v) * p.C + c0));
          if (want_gconf) {
            const float4 s = sample4(fb + v * map_elems, p.C, c0, t);
            float* a = gconf_acc + v * p.C + c0;
            acc_add(a, g.x * s.x); acc_add(a + 1, g.y * s.y); acc_add(a + 2, g.z * s.z); acc_add(a + 3, g.w * s.w);
          }
          gs = make_float4(g.x * cf.x, g.y * cf.y, g.z * cf.z, g.w * cf.w);
        }
        scatter4(gb + v * map_elems, p.C, c0, t, gs);
      }
    } else if (p.agg == LT_AGG_MAX) {
      // torch.max(dim=0) routes the gradient to the first view that attains the maximum
      float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
      int ax = 0, ay = 0, az = 0, aw = 0;
      for (int v = 0; v < p.V; ++v) {
        const float4 s = sample4(fb + v * map_elems, p.C, c0, bwd_taps(view_proj(v), X, Y, Z, p.h, p.w));
        if (s.x > m.x) { m.x = s.x; ax = v; }
        if (s.y > m.y) { m.y = s.y; ay = v; }
        if (s.z > m.z) { m.z = s.z; az = v; }
        if (s.w > m.w) { m.w = s.w; aw = v; }
      }
      for (int v = 0; v < p.V; ++v) {
        const float4 gs = make_float4(v == ax ? g.x : 0.f, v == ay ? g.y : 0.f, v == az ? g.z : 0.f, v == aw ? g.w : 0.f);
        if (gs.x != 0.f || gs.y != 0.f || gs.z != 0.f || gs.w != 0.f)
          scatter4(gb + v * map_elems, p.C, c0, bwd_taps(view_proj(v), X, Y, Z, p.h, p.w), gs);
      }
    } else {
      // softmax over views: out = sum_v s_v p_v;  d out / d s_v = p_v (1 + s_v - out).  Three passes over the views
      // (max, normaliser + out, scatter), each re-gathering the sample: no per-view register arrays, any V.
      float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
      for (int v = 0; v < p.V; ++v) {
        const float4 s = sample4(fb + v * map_elems, p.C, c0, bwd_taps(view_proj(v), X, Y, Z, p.h, p.w));
        m.x = fmaxf(m.x, s.x); m.y = fmaxf(m.y, s.y); m.z = fmaxf(m.z, s.z); m.w = fmaxf(m.w, s.w);
      }
      float4 den = make_float4(0.f, 0.f, 0.f, 0.f), num = den;
      for (int v = 0; v < p.V; ++v) {
        const float4 s = sample4(fb + v * map_elems, p.C, c0, bwd_taps(view_proj(v), X, Y, Z, p.h, p.w));
        const float ex = expf(s.x - m.x), ey = expf(s.y - m.y), ez = expf(s.z - m.z), ew = expf(s.w - m.w);
        den.x += ex; den.y += ey; den.z += ez; den.w += ew;
        num.x = fmaf(s.x, ex, num.x); num.y = fmaf(s.y, ey, num.y); num.z = fmaf(s.z, ez, num.z); num.w = fmaf(s.w, ew, num.w);
      }
      const float4 out = make_float4(num.x / den.x, num.y / den.y, num.z / den.z, num.w / den.w);
      for (int v = 0; v < p.V; ++v) {
        const BwdTaps t = bwd_taps(view_proj(v), X, Y, Z, p.h, p.w);
        const float4 s = sample4(fb + v * map_elems, p.C, c0, t);
        const float4 gs = make_float4(g.x * (expf(s.x - m.x) / den.x) * (1.0f + s.x - out.x), g.y * (expf(s.y - m.y) / den.y) * (1.0f + s.y - out.y),
                                      g.z * (expf(s.z - m.z) / den.z) * (1.0f + s.z - out.z), g.w * (expf(s.w - m.w) / den.w) * (1.0f + s.w - out.w));
        scatter4(gb + v * map_elems, p.C, c0, t, gs);
      }
    }
  }
}

__global__ void __launch_bounds__(256) unproject_bwd_kernel(const UnprojBwdParams p) {
  __shared__ float sP[kBwdSmemViews * 12];
  extern __shared__ float sConf[];          // [V][C] block-level accumulator of d conf (only with grad_conf)
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < min(p.V, kBwdSmemViews) * 12; i += blockDim.x) sP[i] = p.proj[(long)b * p.V * 12 + i];
  const bool want_gconf = p.grad_conf != nullptr && p.agg == LT_AGG_CONF;
  if (want_gconf)
    for (int i = threadIdx.x; i < p.V * p.C; i += blockDim.x) sConf[i] = 0.0f;
  __syncthreads();
  const long items = p.nvox * (p.C >> 2);
  for (long it = (long)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (long)gridDim.x * blockDim.x)
    unproject_bwd_item(p, b, it, sP, want_gconf ? sConf : nullptr);
  if (want_gconf) {
    __syncthreads();
    for (int i = threadIdx.x; i < p.V * p.C; i += blockDim.x) atomicAdd(p.grad_conf + (long)b * p.V * p.C + i, sConf[i]);
  }
}

// ---- soft-argmax backward, NCDHW: volumes / logits / grads are [B][J][nvox] ----
struct SoftBwdParams {
  const float* probs;      // forward output: softmax(mult * logits) (softmax) or relu(mult * logits) (ReLU)
  const float* coord;      // [B][nvox][3]
  const float* g_kp;       // [B][J][3]
  const float* g_vol;      // [B][J][nvox] or null
  float* dots;             // [B][J] scratch: sum_k p_k t_k
  float* grad_logits;      // [B][J][nvox]
  int B, J, softmax;
  long nvox;
  float mult;
};

__host__ __device__ __forceinline__ float soft_t(const SoftBwdParams& p, int b, int j, long i, float gx, float gy, float gz) {
  const float* c = p.coord + ((long)b * p.nvox + i) * 3;
  float t = fmaf(gx, LT_LD(c), fmaf(gy, LT_LD(c + 1), gz * LT_LD(c + 2)));
  if (p.g_vol) t += LT_LD(p.g_vol + ((long)b * p.J + j) * p.nvox + i);
  return t;
}
__host__ __device__ __forceinline__ float soft_grad(const SoftBwdParams& p, float pi, float t, float S) {
  // ReLU: probs = relu(mult * logit) > 0 exactly where the gradient passes
  return p.softmax ? p.mult * pi * (t - S) : (pi > 0.0f ? p.mult * t : 0.0f);
}

// one CTA per (b, j): S = sum_i p_i t_i
__global__ void __launch_bounds__(512) softargmax_bwd_dot_kernel(const SoftBwdParams p) {
  const int bj = blockIdx.x, b = bj / p.J, j = bj % p.J;
  const float gx = p.g_kp[bj * 3], gy = p.g_kp[bj * 3 + 1], gz = p.g_kp[bj * 3 + 2];
  const float* pr = p.probs + (long)bj * p.nvox;
  float acc = 0.f;
  for (long i = threadIdx.x; i < p.nvox; i += blockDim.x) acc = fmaf(__ldg(pr + i), soft_t(p, b, j, i, gx, gy, gz), acc);
  acc = warp_sum(acc);
  __shared__ float sh[16];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) p.dots[bj] = v;
  }
}

__global__ void __launch_bounds__(256) softargmax_bwd_apply_kernel(const SoftBwdParams p) {
  const int bj = blockIdx.y, b = bj / p.J, j = bj % p.J;
  const float gx = p.g_kp[bj * 3], gy = p.g_kp[bj * 3 + 1], gz = p.g_kp[bj * 3 + 2];
  const float S = p.softmax ? p.dots[bj] : 0.f;
  const float* pr = p.probs + (long)bj * p.nvox;
  float* out = p.grad_logits + (long)bj * p.nvox;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < p.nvox; i += (long)gridDim.x * blockDim.x) {
    out[i] = soft_grad(p, __ldg(pr + i), soft_t(p, b, j, i, gx, gy, gz), S);
  }
}

}  // namespace lt

using namespace lt;

extern "C" int lt_unproject_aggregate_bwd(const float* features, const float* proj, const float* coord, const float* conf,
                                          const float* grad_out, float* grad_features, float* grad_conf, int B, int V, int C, int h, int w,
                                          long nvox, int agg, void* stream) {
  LT_REQUIRE(features && proj && coord && grad_out && grad_features, "unproject_bwd: null pointer");
  LT_REQUIRE(B > 0 && V > 0 && C > 0 && h > 0 && w > 0 && nvox > 0, "unproject_bwd: non-positive size");
  LT_REQUIRE(C % 4 == 0, "unproject_bwd: C %% 4 != 0 (C=%d)", C);
  LT_REQUIRE(agg >= LT_AGG_SUM && agg <= LT_AGG_CONF, "unproject_bwd: unknown aggregation %d", agg);
  LT_REQUIRE(agg != LT_AGG_CONF || conf, "unproject_bwd: LT_AGG_CONF needs confidences");
  LT_REQUIRE(B <= 65535, "unproject_bwd: batch too large");
  UnprojBwdParams p{features, proj, coord, conf, grad_out, grad_features, grad_conf, B, V, C, h, w, agg, nvox};
  const long items = nvox * (C / 4);
  long blocks = (items + 255) / 256;
  const long cap = (long)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  const size_t smem = (grad_conf && agg == LT_AGG_CONF) ? (size_t)V * C * sizeof(float) : 0;
  LT_REQUIRE(smem <= 40 * 1024, "unproject_bwd: V * C too large for the confidence-gradient accumulator");
  unproject_bwd_kernel<<<dim3((unsigned)blocks, (unsigned)B), 256, smem, (cudaStream_t)stream>>>(p);
  LT_CHECK_LAUNCH("unproject_bwd_kernel");
  return LT_OK;
}

extern "C" int lt_softargmax3d_bwd(const float* probs, const float* coord, const float* grad_keypoints, const float* grad_volumes,
                                   float* grad_logits, float* scratch, int B, int J, long nvox, float multiplier, int softmax, void* stream) {
  LT_REQUIRE(probs && coord && grad_keypoints && grad_logits && scratch, "softargmax3d_bwd: null pointer");
  LT_REQUIRE(B > 0 && J > 0 && nvox > 0 && (long)B * J <= 65535, "softargmax3d_bwd: bad sizes");
  SoftBwdParams p{probs, coord, grad_keypoints, grad_volumes, scratch, grad_logits, B, J, softmax, nvox, multiplier};
  cudaStream_t st = (cudaStream_t)stream;
  if (softmax) {
    softargmax_bwd_dot_kernel<<<B * J, 512, 0, st>>>(p);
    LT_CHECK_LAUNCH("softargmax_bwd_dot_kernel");
  }
  long bx = (nvox + 255) / 256;
  if (bx > 64) bx = 64;
  softargmax_bwd_apply_kernel<<<dim3((unsigned)bx, (unsigned)(B * J)), 256, 0, st>>>(p);
  LT_CHECK_LAUNCH("softargmax_bwd_apply_kernel");
  return LT_OK;
}

// ---- test hooks: the same per-item code on the CPU (host pointers), for the `-m "not gpu"` gradient tests -------------
extern "C" int lt_test_unproject_aggregate_bwd_host(const float* features, const float* proj, const float* coord, const float* conf,
                                                    const float* grad_out, float* grad_features, float* grad_conf, int B, int V, int C, int h,
                                                    int w, long nvox, int agg) {
  LT_REQUIRE(features && proj && coord && grad_out && grad_features && C % 4 == 0, "test_unproject_bwd_host: bad arguments");
  LT_REQUIRE(agg >= LT_AGG_SUM && agg <= LT_AGG_CONF && (agg != LT_AGG_CONF || conf), "test_unproject_bwd_host: bad aggregation");
  UnprojBwdParams p{features, proj, coord, conf, grad_out, grad_features, grad_conf, B, V, C, h, w, agg, nvox};
  const long items = nvox * (C / 4);
  for (int b = 0; b < B; ++b)
    for (long it = 0; it < items; ++it)
      unproject_bwd_item(p, b, it, nullptr, (grad_conf && agg == LT_AGG_CONF) ? grad_conf + (long)b * V * C : nullptr);
  return LT_OK;
}

extern "C" int lt_test_softargmax3d_bwd_host(const float* probs, const float* coord, const float* grad_keypoints, const float* grad_volumes,
                                             float* grad_logits, int B, int J, long nvox, float multiplier, int softmax) {
  LT_REQUIRE(probs && coord && grad_keypoints && grad_logits, "test_softargmax3d_bwd_host: null pointer");
  SoftBwdParams p{probs, coord, grad_keypoints, grad_volumes, nullptr, grad_logits, B, J, softmax, nvox, multiplier};
  for (int bj = 0; bj < B * J; ++bj) {
    const int b = bj / J, j = bj % J;
    const float gx = grad_keypoints[bj * 3], gy = grad_keypoints[bj * 3 + 1], gz = grad_keypoints[bj * 3 + 2];
    const float* pr = probs + (long)bj * nvox;
    double S = 0.0;
    if (softmax)
      for (long i = 0; i < nvox; ++i) S += (double)pr[i] * soft_t(p, b, j, i, gx, gy, gz);
    for (long i = 0; i < nvox; ++i) grad_logits[(long)bj * nvox + i] = soft_grad(p, pr[i], soft_t(p, b, j, i, gx, gy, gz), (float)S);
  }
  return LT_OK;
}
