// Backward passes of the two custom ops of the volumetric path (SURVEY section 8f row 1, first stage), the soft-argmax one
// also serving the 2-D soft-argmax of the algebraic model: what
// `total_loss.backward()` (train.py:236) needs from op.unproject_heatmaps (op.py:99-166) and
// op.integrate_tensor_3d_with_coordinates (op.py:84-96) when they run on the native kernels inside the torch training
// graph (`backend="hybrid"`: torch convolutions, native custom ops).  Gradients flow to the feature maps (and to the
// per-view confidences of the `conf` aggregation) and to the V2V logits.  The models build their geometry from numpy, but the
// op-level drop-ins differentiate projection matrices and coordinate volumes like the reference's torch graph does, so the
// geometry variant below (lt_unproject_aggregate_bwd_geom) and lt_softargmax3d_coord_bwd give those gradients too.
//
// Unprojection backward (HBM / atomics bound): one thread per (voxel, 4 channels) recomputes the four bilinear taps of every
// view exactly as the forward does, re-aggregates, forms the per-view sample gradient
//     sum:      g                      conf:   g * conf_v   (and d conf_v += g * s_v)
//     max:      g on the arg-max view  softmax: g * p_v * (1 + s_v - out),  p = softmax_v(s)
// and scatters it with 16-byte vector atomics (red.global.add.v4.f32) into the channels-last feature gradient.
// Soft-argmax backward (HBM bound, NCDHW like the op-level API): with t_i = g_vol_i + <g_kp, x_i>,
//     softmax: d logit_i = mult * p_i * (t_i - sum_k p_k t_k)      ReLU: d logit_i = mult * [mult * logit_i > 0] * t_i
// and for mode 2, the ReLU branch of the 2-D op (op.integrate_tensor_2d, op.py:25-41: kp = sum p_i x_i / M, M = sum p_i), which
// the algebraic model (triangulation.py:131-200) trains through with the pixel grid (x, y, 0) as coordinates:
//     mass:    d logit_i = mult * [p_i > 0] * (g_vol_i + (<g_kp, x_i> - <g_kp, kp>) / M)
// The DLT backward of the algebraic model is in algebraic.cu (it shares the forward's eigen-solve).
//
// Fixed-order unprojection backward (lt_unproject_aggregate_bwd_det, selected by torch.use_deterministic_algorithms): no float
// atomics.  Pass 1 runs the same per-item code but stores each (sample, view, voxel) sample gradient and the voxel's floor cell
// instead of scattering; pass 2 sorts the voxels of every (sample, view) by cell, stably (voxel order within a cell); pass 3 gathers
// per (pixel, channel quad) the terms gs * w_k of the four cells that have the pixel as a tap, in a fixed cell order and voxel order.
// d conf sums fixed voxel chunks and merges them in chunk order.  Every sum depends only on the inputs of its own sample.
#include "common.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <math.h>
#include <stdlib.h>
#include <vector>

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

// What the geometry gradient needs of one (voxel, view) beyond the taps: the tap validity (a tap with weight 0 can still carry
// a derivative), d w_k / d ix and d w_k / d iy of the taps inside the map (torch's grid_sampler_2d_backward convention: the same
// floor cell, also at integer positions and at border taps), the projected position and the depth.
struct GeomTaps {
  float dx[4], dy[4];   // 0 where the tap is outside the map or the depth test failed
  float x, y, pz;       // pz after the 0 -> 1 replacement
  bool live;            // depth test passed and at least one tap is inside the map
};

// identical arithmetic to make_taps() in unproject.cu (op.py:116-135, multiview.py:89-110); kGeom also fills *gt
template <bool kGeom>
__host__ __device__ __forceinline__ BwdTaps bwd_taps_impl(const float* __restrict__ P, float X, float Y, float Z, int h, int w, GeomTaps* gt) {
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
  if (kGeom) {
    const bool in[4] = {depth_ok && vx0 && vy0, depth_ok && vx1 && vy0, depth_ok && vx0 && vy1, depth_ok && vx1 && vy1};
    const float ddx[4] = {-(y1 - iy), y1 - iy, -(iy - y0), iy - y0};
    const float ddy[4] = {-(x1 - ix), -(ix - x0), x1 - ix, ix - x0};
#pragma unroll
    for (int k = 0; k < 4; ++k) { gt->dx[k] = in[k] ? ddx[k] : 0.0f; gt->dy[k] = in[k] ? ddy[k] : 0.0f; }
    gt->x = x; gt->y = y; gt->pz = pz;
    gt->live = in[0] || in[1] || in[2] || in[3];
  }
  return t;
}

__host__ __device__ __forceinline__ BwdTaps bwd_taps(const float* __restrict__ P, float X, float Y, float Z, int h, int w) {
  return bwd_taps_impl<false>(P, X, Y, Z, h, w, nullptr);
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

// (G_ix, G_iy) of one 4-channel quad: sum_c gs_c d s_c / d ix and d s_c / d iy over the taps inside the map
__host__ __device__ __forceinline__ float2 geom_partial(const float* __restrict__ fmap, int C, int c0, const BwdTaps& t, const GeomTaps& gt,
                                                        float4 gs) {
  float gix = 0.0f, giy = 0.0f;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (gt.dx[k] != 0.0f || gt.dy[k] != 0.0f) {
      const float4 q = LT_LD(reinterpret_cast<const float4*>(fmap + (long)t.o[k] * C + c0));
      const float d = fmaf(gs.w, q.w, fmaf(gs.z, q.z, fmaf(gs.y, q.y, gs.x * q.x)));
      gix = fmaf(gt.dx[k], d, gix);
      giy = fmaf(gt.dy[k], d, giy);
    }
  return make_float2(gix, giy);
}

// q = dL/dp of p = P [X, 1] from the voxel's (G_ix, G_iy) summed over all channels: G_x = G_ix (w - 1) / h, G_y = G_iy (h - 1) / w
// (ix = x / h (w - 1), iy = y / w (h - 1)), then through x = px / pz, y = py / pz.  Exactly 0 for a voxel that fails the depth test
// or has no tap inside the map (pz may be 2^-60 there: no inf * 0).
__host__ __device__ __forceinline__ void geom_q(const GeomTaps& gt, float gix, float giy, int h, int w, float q[3]) {
  if (!gt.live) { q[0] = q[1] = q[2] = 0.0f; return; }
  const float gx = gix * ((float)(w - 1) / (float)h), gy = giy * ((float)(h - 1) / (float)w);
  q[0] = gx / gt.pz;
  q[1] = gy / gt.pz;
  q[2] = -fmaf(gx, gt.x, gy * gt.y) / gt.pz;
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
  float* geom_q;           // geometry variant: [B][V][nvox][3] q per (sample, view, voxel), written (the host hook accumulates
                           // (G_ix, G_iy) into its first two slots instead and forms q afterwards)
  float* stage_gs;         // fixed-order pass 1: [B][V][nvox][C] sample gradient per (sample, view, voxel), written
  unsigned* stage_key;     //   [B][V][nvox] sort key (b V + v) (cells + 1) + floor cell (det_cell), written
  unsigned* stage_vox;     //   [B][V][nvox] the voxel index (the sort's values), written
};

// The (h + 1) x (w + 1) floor cells (xi, yi) of bwd_taps_impl whose taps can lie inside the map, xi, yi in [-1, size - 1], as
// (yi + 1) (w + 1) + xi + 1, read off the first tap with a weight (such a tap is not clamped); (h + 1) (w + 1) when no tap has a
// weight, i.e. the voxel adds nothing to this view.
__host__ __device__ __forceinline__ unsigned det_cell(const BwdTaps& t, int h, int w) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (t.w[k] != 0.0f) {
      const int y = t.o[k] / w - (k >> 1), x = t.o[k] % w - (k & 1);
      return (unsigned)((y + 1) * (w + 1) + x + 1);
    }
  return (unsigned)((h + 1) * (w + 1));
}
__host__ __device__ __forceinline__ long det_keys_per_view(int h, int w) { return (long)(h + 1) * (w + 1) + 1; }

// pass 1 sink: what scatter4 would add for (b, v, vox, quad), stored; the voxel's first quad also stores its key and index
__host__ __device__ __forceinline__ void det_stage(const UnprojBwdParams& p, int b, int v, long vox, int c0, const BwdTaps& t, float4 gs) {
  const long row = ((long)b * p.V + v) * p.nvox + vox;
  *reinterpret_cast<float4*>(p.stage_gs + row * p.C + c0) = gs;
  if (c0 == 0) {
    p.stage_key[row] = (unsigned)(((long)b * p.V + v) * det_keys_per_view(p.h, p.w) + det_cell(t, p.h, p.w));
    p.stage_vox[row] = (unsigned)vox;
  }
}

constexpr int kBwdSmemViews = 64;

// The quad's (G_ix, G_iy) of view v, summed over the C / 4 quads of the voxel.  GPU: those are C / 4 adjacent lanes of one warp
// (C / 4 is a power of two <= 32, the grid stride a multiple of 32 and the item count a multiple of C / 4), summed by a fixed
// butterfly; the voxel's first quad forms q and writes it.  Host: items run in order, so (G_ix, G_iy) accumulates in place.
__host__ __device__ __forceinline__ void geom_emit(const UnprojBwdParams& p, int b, int v, long vox, int quad, const GeomTaps& gt, float2 G) {
  float* dst = p.geom_q + (((long)b * p.V + v) * p.nvox + vox) * 3;
#ifdef __CUDA_ARCH__
  const int quads = p.C >> 2;
  const unsigned lane = threadIdx.x & 31;
  const unsigned mask = quads == 32 ? 0xffffffffu : (((1u << quads) - 1u) << (lane & ~(unsigned)(quads - 1)));
  for (int o = 1; o < quads; o <<= 1) {
    G.x += __shfl_xor_sync(mask, G.x, o);
    G.y += __shfl_xor_sync(mask, G.y, o);
  }
  if (quad == 0) {
    float q[3];
    geom_q(gt, G.x, G.y, p.h, p.w, q);
    dst[0] = q[0]; dst[1] = q[1]; dst[2] = q[2];
  }
#else
  (void)gt; (void)quad;
  dst[0] += G.x; dst[1] += G.y;
#endif
}

// one (voxel, 4-channel quad) of sample b.  projs: the sample's first kBwdSmemViews projection matrices (shared memory on
// the GPU) or null; gconf_acc: [V][C] accumulator of d conf (shared memory on the GPU, the output itself on the host) or null.
// kGeom also hands every view's (G_ix, G_iy) to geom_emit, once per view on every path (the GPU lanes of a voxel meet there).
// kStage (the fixed-order path) stores every view's sample gradient with det_stage instead of scattering it.
template <bool kGeom, bool kStage = false>
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
        GeomTaps gt;
        const BwdTaps t = bwd_taps_impl<kGeom>(view_proj(v), X, Y, Z, p.h, p.w, &gt);
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
        if (kStage) det_stage(p, b, v, vox, c0, t, gs);
        else scatter4(gb + v * map_elems, p.C, c0, t, gs);
        if (kGeom) geom_emit(p, b, v, vox, c0 >> 2, gt, geom_partial(fb + v * map_elems, p.C, c0, t, gt, gs));
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
        if (kGeom) {
          GeomTaps gt;
          const BwdTaps t = bwd_taps_impl<true>(view_proj(v), X, Y, Z, p.h, p.w, &gt);
          if (kStage) det_stage(p, b, v, vox, c0, t, gs);
          else if (gs.x != 0.f || gs.y != 0.f || gs.z != 0.f || gs.w != 0.f) scatter4(gb + v * map_elems, p.C, c0, t, gs);
          geom_emit(p, b, v, vox, c0 >> 2, gt, geom_partial(fb + v * map_elems, p.C, c0, t, gt, gs));
        } else if (kStage) {
          det_stage(p, b, v, vox, c0, bwd_taps(view_proj(v), X, Y, Z, p.h, p.w), gs);
        } else if (gs.x != 0.f || gs.y != 0.f || gs.z != 0.f || gs.w != 0.f) {
          scatter4(gb + v * map_elems, p.C, c0, bwd_taps(view_proj(v), X, Y, Z, p.h, p.w), gs);
        }
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
        GeomTaps gt;
        const BwdTaps t = bwd_taps_impl<kGeom>(view_proj(v), X, Y, Z, p.h, p.w, &gt);
        const float4 s = sample4(fb + v * map_elems, p.C, c0, t);
        const float4 gs = make_float4(g.x * (expf(s.x - m.x) / den.x) * (1.0f + s.x - out.x), g.y * (expf(s.y - m.y) / den.y) * (1.0f + s.y - out.y),
                                      g.z * (expf(s.z - m.z) / den.z) * (1.0f + s.z - out.z), g.w * (expf(s.w - m.w) / den.w) * (1.0f + s.w - out.w));
        if (kStage) det_stage(p, b, v, vox, c0, t, gs);
        else scatter4(gb + v * map_elems, p.C, c0, t, gs);
        if (kGeom) geom_emit(p, b, v, vox, c0 >> 2, gt, geom_partial(fb + v * map_elems, p.C, c0, t, gt, gs));
      }
    }
  }
}

// the body of unproject_bwd_kernel (kGeom = false) and unproject_bwd_geom_kernel (true)
template <bool kGeom>
__device__ __forceinline__ void unproject_bwd_body(const UnprojBwdParams& p) {
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
    unproject_bwd_item<kGeom>(p, b, it, sP, want_gconf ? sConf : nullptr);
  if (want_gconf) {
    __syncthreads();
    for (int i = threadIdx.x; i < p.V * p.C; i += blockDim.x) atomicAdd(p.grad_conf + (long)b * p.V * p.C + i, sConf[i]);
  }
}

__global__ void __launch_bounds__(256) unproject_bwd_kernel(const UnprojBwdParams p) { unproject_bwd_body<false>(p); }
__global__ void __launch_bounds__(256) unproject_bwd_geom_kernel(const UnprojBwdParams p) { unproject_bwd_body<true>(p); }

// ---- second pass of the geometry gradient: deterministic sums of q (no float atomics) ----
// dP_v[r][:] = sum_voxels q_r [X, Y, Z, 1]: fixed voxel chunks per CTA summed in float64 (fixed butterfly, warps in order), the
// chunks merged in order.  dX = sum_v sum_r q_r P_v[r][0:3] per voxel, views in order.
constexpr int kGeomChunk = 8192;        // voxels per dP partial
constexpr int kGeomThreads = 256;

__host__ __device__ __forceinline__ int geom_chunks(long nvox) { return (int)((nvox + kGeomChunk - 1) / kGeomChunk); }

// the 12 float64 terms voxel `vox` adds to dP of (b, v)
__host__ __device__ __forceinline__ void geom_dp_terms(const float* __restrict__ coord, const float* __restrict__ q, long nvox, int b,
                                                       int bv, long vox, double t[12]) {
  const float* cp = coord + ((long)b * nvox + vox) * 3;
  const float* qp = q + ((long)bv * nvox + vox) * 3;
  const double X4[4] = {(double)LT_LD(cp), (double)LT_LD(cp + 1), (double)LT_LD(cp + 2), 1.0};
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double qr = (double)LT_LD(qp + r);
#pragma unroll
    for (int c = 0; c < 4; ++c) t[r * 4 + c] = qr * X4[c];
  }
}

__host__ __device__ __forceinline__ void geom_dx_item(const float* __restrict__ proj, const float* __restrict__ q, float* __restrict__ grad_coord,
                                                      int V, long nvox, int b, long vox) {
  float d[3] = {0.0f, 0.0f, 0.0f};
  for (int v = 0; v < V; ++v) {
    const float* P = proj + ((long)b * V + v) * 12;
    const float* qp = q + (((long)b * V + v) * nvox + vox) * 3;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float qr = LT_LD(qp + r);
#pragma unroll
      for (int k = 0; k < 3; ++k) d[k] = fmaf(qr, LT_LD(P + r * 4 + k), d[k]);
    }
  }
  float* out = grad_coord + ((long)b * nvox + vox) * 3;
  out[0] = d[0]; out[1] = d[1]; out[2] = d[2];
}

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// grid (chunks, B * V): partial[(bv * chunks + chunk) * 12 + e]
__global__ void __launch_bounds__(kGeomThreads) unproject_geom_dp_partial_kernel(const float* __restrict__ coord, const float* __restrict__ q,
                                                                                 double* __restrict__ partial, int V, long nvox) {
  const int bv = blockIdx.y, b = bv / V, chunk = blockIdx.x;
  const long v0 = (long)chunk * kGeomChunk, v1 = min(nvox, v0 + kGeomChunk);
  double acc[12];
#pragma unroll
  for (int e = 0; e < 12; ++e) acc[e] = 0.0;
  for (long vox = v0 + threadIdx.x; vox < v1; vox += kGeomThreads) {
    double t[12];
    geom_dp_terms(coord, q, nvox, b, bv, vox, t);
#pragma unroll
    for (int e = 0; e < 12; ++e) acc[e] += t[e];
  }
  __shared__ double sh[kGeomThreads / 32][12];
#pragma unroll
  for (int e = 0; e < 12; ++e) {
    const double s = warp_sum_f64(acc[e]);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5][e] = s;
  }
  __syncthreads();
  if (threadIdx.x < 12) {
    double s = 0.0;
    for (int k = 0; k < kGeomThreads / 32; ++k) s += sh[k][threadIdx.x];
    partial[((long)bv * gridDim.x + chunk) * 12 + threadIdx.x] = s;
  }
}

// one thread per (b, v, e): the chunks in order
__global__ void unproject_geom_dp_merge_kernel(const double* __restrict__ partial, float* __restrict__ grad_proj, int BV, int chunks) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= BV * 12) return;
  const int bv = i / 12, e = i % 12;
  double s = 0.0;
  for (int k = 0; k < chunks; ++k) s += partial[((long)bv * chunks + k) * 12 + e];
  grad_proj[i] = (float)s;
}

__global__ void __launch_bounds__(256) unproject_geom_dx_kernel(const float* __restrict__ proj, const float* __restrict__ q,
                                                                float* __restrict__ grad_coord, int B, int V, long nvox) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * nvox) return;
  geom_dx_item(proj, q, grad_coord, V, nvox, (int)(i / nvox), i % nvox);
}

// ---- fixed-order unprojection backward: passes 1 and 3 and the confidence gradient (see the top of the file) ----
#ifdef __CUDA_ARCH__
#define LT_ADD_PROD(acc, a, b) __fadd_rn((acc), __fmul_rn((a), (b)))    // the product rounded as the atomic kernel rounds it, then added
#else
#define LT_ADD_PROD(acc, a, b) ((acc) + (a) * (b))
#endif

__host__ __device__ __forceinline__ void add_prod4(float4& acc, float4 a, float b) {
  acc.x = LT_ADD_PROD(acc.x, a.x, b); acc.y = LT_ADD_PROD(acc.y, a.y, b); acc.z = LT_ADD_PROD(acc.z, a.z, b); acc.w = LT_ADD_PROD(acc.w, a.w, b);
}

// d features of (b v, pixel pix, quad c0): the terms gs * w_k of the cells (y - 1, x - 1), (y - 1, x), (y, x - 1), (y, x) in that
// order (the pixel is their tap k = 3, 2, 1, 0), each cell's voxels in ascending order (seg_begin / seg_end: the cell's range of
// sorted_vox).  The taps are recomputed with bwd_taps, so w_k is the weight pass 1 and the atomic kernel use.
__host__ __device__ __forceinline__ float4 det_gather_item(const UnprojBwdParams& p, const unsigned* __restrict__ seg_begin,
                                                           const unsigned* __restrict__ seg_end, const unsigned* __restrict__ sorted_vox,
                                                           int bv, int pix, int c0) {
  const int b = bv / p.V, y = pix / p.w, x = pix % p.w;
  const float* P = p.proj + (long)bv * 12;
  const long kbase = (long)bv * det_keys_per_view(p.h, p.w);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int k = 3; k >= 0; --k) {
    const long key = kbase + (long)(y - (k >> 1) + 1) * (p.w + 1) + (x - (k & 1) + 1);
    const unsigned e = LT_LD(seg_end + key);
    for (unsigned i = LT_LD(seg_begin + key); i < e; ++i) {
      const long vox = LT_LD(sorted_vox + i);
      const float* cp = p.coord + ((long)b * p.nvox + vox) * 3;
      const float wk = bwd_taps(P, LT_LD(cp), LT_LD(cp + 1), LT_LD(cp + 2), p.h, p.w).w[k];
      if (wk != 0.0f) add_prod4(acc, LT_LD(reinterpret_cast<const float4*>(p.stage_gs + ((long)bv * p.nvox + vox) * p.C + c0)), wk);
    }
  }
  return acc;
}

// d conf of (b v, quad c0) over one chunk of kDetConfChunk voxels: the terms g * s, voxels in order (the atomic kernel's terms)
constexpr int kDetConfChunk = 256;
__host__ __device__ __forceinline__ long det_conf_chunks(long nvox) { return (nvox + kDetConfChunk - 1) / kDetConfChunk; }

__host__ __device__ __forceinline__ float4 det_conf_partial(const UnprojBwdParams& p, int bv, long chunk, int c0) {
  const int b = bv / p.V;
  const float* P = p.proj + (long)bv * 12;
  const float* fmap = p.features + (long)bv * p.h * p.w * p.C;
  const long v0 = chunk * kDetConfChunk, v1 = v0 + kDetConfChunk < p.nvox ? v0 + kDetConfChunk : p.nvox;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long vox = v0; vox < v1; ++vox) {
    const float* cp = p.coord + ((long)b * p.nvox + vox) * 3;
    const float4 s = sample4(fmap, p.C, c0, bwd_taps(P, LT_LD(cp), LT_LD(cp + 1), LT_LD(cp + 2), p.h, p.w));
    const float4 g = LT_LD(reinterpret_cast<const float4*>(p.grad_out + ((long)b * p.nvox + vox) * p.C + c0));
    acc.x = LT_ADD_PROD(acc.x, g.x, s.x); acc.y = LT_ADD_PROD(acc.y, g.y, s.y);
    acc.z = LT_ADD_PROD(acc.z, g.z, s.z); acc.w = LT_ADD_PROD(acc.w, g.w, s.w);
  }
  return acc;
}

// grad_conf[bv][c] += the chunk partials [bv][chunk][c] in chunk order
__host__ __device__ __forceinline__ void det_conf_merge_item(const float* __restrict__ partial, float* __restrict__ grad_conf, int C, long chunks,
                                                             long i) {
  const long bv = i / C, c = i % C;
  float s = 0.0f;
  for (long k = 0; k < chunks; ++k) s += LT_LD(partial + (bv * chunks + k) * C + c);
  grad_conf[i] += s;
}

template <bool kGeom>
__global__ void __launch_bounds__(256) fo_unproj_bwd_stage_kernel(const UnprojBwdParams p) {
  const long items = p.nvox * (p.C >> 2);
  for (long it = (long)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (long)gridDim.x * blockDim.x)
    unproject_bwd_item<kGeom, true>(p, blockIdx.y, it, nullptr, nullptr);
}

// each sorted key's segment [begin, end) of the sorted order; keys of no voxel keep the empty [0, 0)
__global__ void __launch_bounds__(256) fo_unproj_bwd_bounds_kernel(const unsigned* __restrict__ keys, unsigned* __restrict__ seg_begin,
                                                                    unsigned* __restrict__ seg_end, long n) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned k = keys[i];
  if (i == 0 || keys[i - 1] != k) seg_begin[k] = (unsigned)i;
  if (i == n - 1 || keys[i + 1] != k) seg_end[k] = (unsigned)(i + 1);
}

// grid (pixel quads / 256, B V): grad_features, which the caller zero-fills, gets each total added once
__global__ void __launch_bounds__(256) fo_unproj_bwd_gather_kernel(const UnprojBwdParams p, const unsigned* __restrict__ seg_begin,
                                                                    const unsigned* __restrict__ seg_end, const unsigned* __restrict__ sorted_vox) {
  const int quads = p.C >> 2, bv = blockIdx.y;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)p.h * p.w * quads) return;
  const int pix = (int)(i / quads), c0 = (int)(i % quads) * 4;
  const float4 a = det_gather_item(p, seg_begin, seg_end, sorted_vox, bv, pix, c0);
  float4* dst = reinterpret_cast<float4*>(p.grad_features + ((long)bv * p.h * p.w + pix) * p.C + c0);
  float4 d = *dst;
  d.x += a.x; d.y += a.y; d.z += a.z; d.w += a.w;
  *dst = d;
}

// grid (chunks x quads / 128, B V): partial[bv][chunk][C]
__global__ void __launch_bounds__(128) fo_unproj_bwd_conf_partial_kernel(const UnprojBwdParams p, float* __restrict__ partial) {
  const int quads = p.C >> 2, bv = blockIdx.y;
  const long chunks = det_conf_chunks(p.nvox);
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= chunks * quads) return;
  const long chunk = i / quads;
  const int c0 = (int)(i % quads) * 4;
  *reinterpret_cast<float4*>(partial + ((long)bv * chunks + chunk) * p.C + c0) = det_conf_partial(p, bv, chunk, c0);
}

__global__ void __launch_bounds__(128) fo_unproj_bwd_conf_merge_kernel(const float* __restrict__ partial, float* __restrict__ grad_conf, int C,
                                                                        long chunks, long n) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) det_conf_merge_item(partial, grad_conf, C, chunks, i);
}

// ---- soft-argmax backward, NCDHW: volumes / logits / grads are [B][J][nvox] ----
struct SoftBwdParams {
  const float* probs;      // forward output: softmax(mult * logits) (softmax) or relu(mult * logits) (ReLU)
  const float* coord;      // [B][nvox][3]
  const float* g_kp;       // [B][J][3]
  const float* g_vol;      // [B][J][nvox] or null
  float* dots;             // scratch: mode 1 [B][J] sum_k p_k t_k; mode 2 [2][B][J] (S, M) below
  float* grad_logits;      // [B][J][nvox]
  int B, J, softmax;       // mode: 0 ReLU, 1 softmax, 2 ReLU with mass-normalised coordinates
  long nvox;
  float mult;
};

// <g_kp, x_i>
__host__ __device__ __forceinline__ float soft_tk(const SoftBwdParams& p, int b, long i, float gx, float gy, float gz) {
  const float* c = p.coord + ((long)b * p.nvox + i) * 3;
  return fmaf(gx, LT_LD(c), fmaf(gy, LT_LD(c + 1), gz * LT_LD(c + 2)));
}
__host__ __device__ __forceinline__ float soft_gvol(const SoftBwdParams& p, int b, int j, long i) {
  return p.g_vol ? LT_LD(p.g_vol + ((long)b * p.J + j) * p.nvox + i) : 0.0f;
}
// t_i = g_vol_i + <g_kp, x_i>
__host__ __device__ __forceinline__ float soft_t(const SoftBwdParams& p, int b, int j, long i, float gx, float gy, float gz) {
  float t = soft_tk(p, b, i, gx, gy, gz);
  if (p.g_vol) t += soft_gvol(p, b, j, i);
  return t;
}
// modes 0 and 1; ReLU: probs = relu(mult * logit) > 0 exactly where the gradient passes
__host__ __device__ __forceinline__ float soft_grad(const SoftBwdParams& p, float pi, float t, float S) {
  return p.softmax ? p.mult * pi * (t - S) : (pi > 0.0f ? p.mult * t : 0.0f);
}
// mode 2: kp = sum p_i x_i / M with M = sum p_i, S = <g_kp, kp>:  d logit_i = mult [p_i > 0] (g_vol_i + (<g_kp, x_i> - S) / M)
__host__ __device__ __forceinline__ float soft_grad_mass(const SoftBwdParams& p, float pi, float tk, float gv, float S, float M) {
  return pi > 0.0f ? p.mult * (gv + (tk - S) / M) : 0.0f;
}

// one CTA per (b, j), one pass over the voxels.  Mode 1: dots[bj] = sum_i p_i t_i.  Mode 2: dots[bj] = S = sum_i p_i tk_i / M and
// dots[B*J + bj] = M = sum_i p_i.
__global__ void __launch_bounds__(512) softargmax_bwd_dot_kernel(const SoftBwdParams p) {
  const int bj = blockIdx.x, b = bj / p.J, j = bj % p.J;
  const bool mass = p.softmax == 2;
  const float gx = p.g_kp[bj * 3], gy = p.g_kp[bj * 3 + 1], gz = p.g_kp[bj * 3 + 2];
  const float* pr = p.probs + (long)bj * p.nvox;
  float acc = 0.f, m = 0.f;
  if (mass) {
    for (long i = threadIdx.x; i < p.nvox; i += blockDim.x) {
      const float pi = __ldg(pr + i);
      acc = fmaf(pi, soft_tk(p, b, i, gx, gy, gz), acc);
      m += pi;
    }
  } else {
    for (long i = threadIdx.x; i < p.nvox; i += blockDim.x) acc = fmaf(__ldg(pr + i), soft_t(p, b, j, i, gx, gy, gz), acc);
  }
  acc = warp_sum(acc);
  if (mass) m = warp_sum(m);
  __shared__ float sh[2][16];
  if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = acc; sh[1][threadIdx.x >> 5] = m; }
  __syncthreads();
  if (threadIdx.x < 32) {
    const bool lane_ok = threadIdx.x < (blockDim.x >> 5);
    float v = lane_ok ? sh[0][threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (mass) {
      float mv = lane_ok ? sh[1][threadIdx.x] : 0.f;
      mv = warp_sum(mv);
      if (threadIdx.x == 0) { p.dots[bj] = v / mv; p.dots[p.B * p.J + bj] = mv; }
    } else if (threadIdx.x == 0) {
      p.dots[bj] = v;
    }
  }
}

__global__ void __launch_bounds__(256) softargmax_bwd_apply_kernel(const SoftBwdParams p) {
  const int bj = blockIdx.y, b = bj / p.J, j = bj % p.J;
  const float gx = p.g_kp[bj * 3], gy = p.g_kp[bj * 3 + 1], gz = p.g_kp[bj * 3 + 2];
  const float* pr = p.probs + (long)bj * p.nvox;
  float* out = p.grad_logits + (long)bj * p.nvox;
  if (p.softmax == 2) {
    const float S = p.dots[bj], M = p.dots[p.B * p.J + bj];
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < p.nvox; i += (long)gridDim.x * blockDim.x)
      out[i] = soft_grad_mass(p, __ldg(pr + i), soft_tk(p, b, i, gx, gy, gz), soft_gvol(p, b, j, i), S, M);
    return;
  }
  const float S = p.softmax ? p.dots[bj] : 0.f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < p.nvox; i += (long)gridDim.x * blockDim.x) {
    out[i] = soft_grad(p, __ldg(pr + i), soft_t(p, b, j, i, gx, gy, gz), S);
  }
}

// d coord[b][i] = sum_j probs[b][j][i] g_kp[b][j] (kp = sum_i p_i x_i in modes 0 and 1), joints in order
__host__ __device__ __forceinline__ void softargmax_coord_bwd_item(const float* __restrict__ probs, const float* __restrict__ g_kp,
                                                                   float* __restrict__ grad_coord, int J, long nvox, int b, long i) {
  float d[3] = {0.0f, 0.0f, 0.0f};
  for (int j = 0; j < J; ++j) {
    const float pi = LT_LD(probs + ((long)b * J + j) * nvox + i);
    const float* g = g_kp + ((long)b * J + j) * 3;
    d[0] = fmaf(pi, LT_LD(g), d[0]);
    d[1] = fmaf(pi, LT_LD(g + 1), d[1]);
    d[2] = fmaf(pi, LT_LD(g + 2), d[2]);
  }
  float* out = grad_coord + ((long)b * nvox + i) * 3;
  out[0] = d[0]; out[1] = d[1]; out[2] = d[2];
}

__global__ void __launch_bounds__(256) softargmax_coord_bwd_kernel(const float* __restrict__ probs, const float* __restrict__ g_kp,
                                                                   float* __restrict__ grad_coord, int J, long nvox) {
  const int b = blockIdx.y;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nvox; i += (long)gridDim.x * blockDim.x)
    softargmax_coord_bwd_item(probs, g_kp, grad_coord, J, nvox, b, i);
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

static size_t geom_q_bytes(int B, int V, long nvox) { return ((size_t)B * V * nvox * 3 * sizeof(float) + 255) & ~(size_t)255; }

extern "C" size_t lt_unproject_aggregate_bwd_geom_workspace_bytes(int B, int V, long nvox) {
  if (B <= 0 || V <= 0 || nvox <= 0) return 0;
  return geom_q_bytes(B, V, nvox) + (size_t)B * V * geom_chunks(nvox) * 12 * sizeof(double);
}

// dP (when grad_proj) and dX (when grad_coord) from the q of every (sample, view, voxel)
static int geom_tail(const float* proj, const float* coord, const float* q, double* partial, float* grad_proj, float* grad_coord, int B, int V,
                     long nvox, cudaStream_t st) {
  if (grad_proj) {
    const int chunks = geom_chunks(nvox);
    unproject_geom_dp_partial_kernel<<<dim3((unsigned)chunks, (unsigned)(B * V)), kGeomThreads, 0, st>>>(coord, q, partial, V, nvox);
    LT_CHECK_LAUNCH("unproject_geom_dp_partial_kernel");
    unproject_geom_dp_merge_kernel<<<ceil_div((long)B * V * 12, 128), 128, 0, st>>>(partial, grad_proj, B * V, chunks);
    LT_CHECK_LAUNCH("unproject_geom_dp_merge_kernel");
  }
  if (grad_coord) {
    unproject_geom_dx_kernel<<<ceil_div((long)B * nvox, 256), 256, 0, st>>>(proj, q, grad_coord, B, V, nvox);
    LT_CHECK_LAUNCH("unproject_geom_dx_kernel");
  }
  return LT_OK;
}

extern "C" int lt_unproject_aggregate_bwd_geom(const float* features, const float* proj, const float* coord, const float* conf,
                                               const float* grad_out, float* grad_features, float* grad_conf, float* grad_proj,
                                               float* grad_coord, void* workspace, size_t workspace_bytes, int B, int V, int C, int h,
                                               int w, long nvox, int agg, void* stream) {
  LT_REQUIRE(features && proj && coord && grad_out && grad_features && workspace, "unproject_bwd_geom: null pointer");
  LT_REQUIRE(B > 0 && V > 0 && C > 0 && h > 0 && w > 0 && nvox > 0, "unproject_bwd_geom: non-positive size");
  LT_REQUIRE(C % 4 == 0 && C <= 128 && ((C / 4) & (C / 4 - 1)) == 0,
             "unproject_bwd_geom: C / 4 must be a power of two <= 32 (the voxel's channel quads are summed within a warp), C=%d", C);
  LT_REQUIRE(agg >= LT_AGG_SUM && agg <= LT_AGG_CONF, "unproject_bwd_geom: unknown aggregation %d", agg);
  LT_REQUIRE(agg != LT_AGG_CONF || conf, "unproject_bwd_geom: LT_AGG_CONF needs confidences");
  LT_REQUIRE(B <= 65535 && (long)B * V <= 65535, "unproject_bwd_geom: batch too large");
  LT_REQUIRE(workspace_bytes >= lt_unproject_aggregate_bwd_geom_workspace_bytes(B, V, nvox),
             "unproject_bwd_geom: workspace of %zu bytes, %zu needed", workspace_bytes, lt_unproject_aggregate_bwd_geom_workspace_bytes(B, V, nvox));
  float* q = reinterpret_cast<float*>(workspace);
  double* partial = reinterpret_cast<double*>(reinterpret_cast<char*>(workspace) + geom_q_bytes(B, V, nvox));
  UnprojBwdParams p{features, proj, coord, conf, grad_out, grad_features, grad_conf, B, V, C, h, w, agg, nvox, q};
  const long items = nvox * (C / 4);
  long blocks = (items + 255) / 256;
  const long cap = (long)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  const size_t smem = (grad_conf && agg == LT_AGG_CONF) ? (size_t)V * C * sizeof(float) : 0;
  LT_REQUIRE(smem <= 40 * 1024, "unproject_bwd_geom: V * C too large for the confidence-gradient accumulator");
  cudaStream_t st = (cudaStream_t)stream;
  unproject_bwd_geom_kernel<<<dim3((unsigned)blocks, (unsigned)B), 256, smem, st>>>(p);
  LT_CHECK_LAUNCH("unproject_bwd_geom_kernel");
  return geom_tail(proj, coord, q, partial, grad_proj, grad_coord, B, V, nvox, st);
}

// ---- fixed-order unprojection backward: workspace layout and launches ----
struct DetLayout {
  size_t gs, key0, key1, vox0, vox1, seg_begin, seg_end, conf, geom, sort, sort_bytes, total;
  int key_bits;
};

static size_t det_align(size_t n) { return (n + 255) & ~(size_t)255; }

// the sort's scratch is what cub::DeviceRadixSort asks for on the current device (0 with no device: the layout is then unusable)
static DetLayout det_layout(int B, int V, int C, int h, int w, long nvox, bool want_conf, bool geom) {
  DetLayout L{};
  const long n = (long)B * V * nvox, nkeys = (long)B * V * det_keys_per_view(h, w);
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += det_align(bytes); return o; };
  L.gs = take((size_t)n * C * sizeof(float));
  L.key0 = take((size_t)n * 4); L.key1 = take((size_t)n * 4); L.vox0 = take((size_t)n * 4); L.vox1 = take((size_t)n * 4);
  L.seg_begin = take((size_t)nkeys * 4); L.seg_end = take((size_t)nkeys * 4);
  L.conf = take(want_conf ? (size_t)B * V * det_conf_chunks(nvox) * C * sizeof(float) : 0);
  L.geom = take(geom ? lt_unproject_aggregate_bwd_geom_workspace_bytes(B, V, nvox) : 0);
  L.key_bits = 1;
  while (L.key_bits < 32 && (1L << L.key_bits) < nkeys) ++L.key_bits;
  size_t sort_bytes = 0;
  if (cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const unsigned*)nullptr, (unsigned*)nullptr, (const unsigned*)nullptr,
                                      (unsigned*)nullptr, (int)n, 0, L.key_bits) != cudaSuccess) {
    cudaGetLastError();
    return DetLayout{};
  }
  L.sort = take(sort_bytes);
  L.sort_bytes = sort_bytes;
  L.total = off;
  return L;
}

static bool det_sizes_ok(int B, int V, int h, int w, long nvox) {
  return B > 0 && V > 0 && h > 0 && w > 0 && nvox > 0 && (long)B * V <= 65535 && (long)B * V * nvox <= 0x7fffffffL &&
         (long)B * V * det_keys_per_view(h, w) <= 0x7fffffffL;
}

extern "C" size_t lt_unproject_aggregate_bwd_det_workspace_bytes(int B, int V, int C, int h, int w, long nvox, int agg, int geom) {
  if (!det_sizes_ok(B, V, h, w, nvox) || C <= 0) return 0;
  return det_layout(B, V, C, h, w, nvox, agg == LT_AGG_CONF, geom != 0).total;
}

extern "C" int lt_unproject_aggregate_bwd_det(const float* features, const float* proj, const float* coord, const float* conf,
                                              const float* grad_out, float* grad_features, float* grad_conf, float* grad_proj, float* grad_coord,
                                              void* workspace, size_t workspace_bytes, int B, int V, int C, int h, int w, long nvox, int agg,
                                              void* stream) {
  LT_REQUIRE(features && proj && coord && grad_out && grad_features && workspace, "unproject_bwd_det: null pointer");
  LT_REQUIRE(B > 0 && V > 0 && C > 0 && h > 0 && w > 0 && nvox > 0, "unproject_bwd_det: non-positive size");
  LT_REQUIRE(det_sizes_ok(B, V, h, w, nvox), "unproject_bwd_det: too large (B V <= 65535, B V nvox and B V (h + 1) (w + 1) below 2^31)");
  const bool geom = grad_proj != nullptr || grad_coord != nullptr;
  LT_REQUIRE(C % 4 == 0 && (!geom || (C <= 128 && ((C / 4) & (C / 4 - 1)) == 0)),
             "unproject_bwd_det: C %% 4 != 0, or with geometry outputs C / 4 not a power of two <= 32 (C=%d)", C);
  LT_REQUIRE(agg >= LT_AGG_SUM && agg <= LT_AGG_CONF, "unproject_bwd_det: unknown aggregation %d", agg);
  LT_REQUIRE(agg != LT_AGG_CONF || conf, "unproject_bwd_det: LT_AGG_CONF needs confidences");
  const bool want_conf = grad_conf != nullptr && agg == LT_AGG_CONF;
  const DetLayout L = det_layout(B, V, C, h, w, nvox, want_conf, geom);
  LT_REQUIRE(L.total > 0 && workspace_bytes >= L.total, "unproject_bwd_det: workspace of %zu bytes, %zu needed", workspace_bytes, L.total);
  char* ws = reinterpret_cast<char*>(workspace);
  unsigned* key0 = reinterpret_cast<unsigned*>(ws + L.key0);
  unsigned* key1 = reinterpret_cast<unsigned*>(ws + L.key1);
  unsigned* vox0 = reinterpret_cast<unsigned*>(ws + L.vox0);
  unsigned* vox1 = reinterpret_cast<unsigned*>(ws + L.vox1);
  unsigned* seg_begin = reinterpret_cast<unsigned*>(ws + L.seg_begin);
  unsigned* seg_end = reinterpret_cast<unsigned*>(ws + L.seg_end);
  float* q = reinterpret_cast<float*>(ws + L.geom);
  UnprojBwdParams p{features, proj, coord, conf, grad_out, grad_features, nullptr, B, V, C, h, w, agg, nvox, q,
                    reinterpret_cast<float*>(ws + L.gs), key0, vox0};
  cudaStream_t st = (cudaStream_t)stream;
  const long n = (long)B * V * nvox, nkeys = (long)B * V * det_keys_per_view(h, w);
  long blocks = (nvox * (C / 4) + 255) / 256;
  const long cap = (long)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (geom) fo_unproj_bwd_stage_kernel<true><<<dim3((unsigned)blocks, (unsigned)B), 256, 0, st>>>(p);
  else fo_unproj_bwd_stage_kernel<false><<<dim3((unsigned)blocks, (unsigned)B), 256, 0, st>>>(p);
  LT_CHECK_LAUNCH("fo_unproj_bwd_stage_kernel");
  size_t sort_bytes = L.sort_bytes;
  const cudaError_t se = cub::DeviceRadixSort::SortPairs(ws + L.sort, sort_bytes, key0, key1, vox0, vox1, (int)n, 0, L.key_bits, st);
  LT_REQUIRE(se == cudaSuccess, "unproject_bwd_det: radix sort failed: %s", cudaGetErrorString(se));
  LT_REQUIRE(cudaMemsetAsync(seg_begin, 0, (size_t)nkeys * 4, st) == cudaSuccess && cudaMemsetAsync(seg_end, 0, (size_t)nkeys * 4, st) == cudaSuccess,
             "unproject_bwd_det: memset failed");
  fo_unproj_bwd_bounds_kernel<<<ceil_div(n, 256), 256, 0, st>>>(key1, seg_begin, seg_end, n);
  LT_CHECK_LAUNCH("fo_unproj_bwd_bounds_kernel");
  fo_unproj_bwd_gather_kernel<<<dim3((unsigned)ceil_div((long)h * w * (C / 4), 256), (unsigned)(B * V)), 256, 0, st>>>(p, seg_begin, seg_end, vox1);
  LT_CHECK_LAUNCH("fo_unproj_bwd_gather_kernel");
  if (want_conf) {
    float* partial = reinterpret_cast<float*>(ws + L.conf);
    const long chunks = det_conf_chunks(nvox);
    fo_unproj_bwd_conf_partial_kernel<<<dim3((unsigned)ceil_div(chunks * (C / 4), 128), (unsigned)(B * V)), 128, 0, st>>>(p, partial);
    LT_CHECK_LAUNCH("fo_unproj_bwd_conf_partial_kernel");
    fo_unproj_bwd_conf_merge_kernel<<<ceil_div((long)B * V * C, 128), 128, 0, st>>>(partial, grad_conf, C, chunks, (long)B * V * C);
    LT_CHECK_LAUNCH("fo_unproj_bwd_conf_merge_kernel");
  }
  if (geom) {
    double* partial = reinterpret_cast<double*>(reinterpret_cast<char*>(q) + geom_q_bytes(B, V, nvox));
    return geom_tail(proj, coord, q, partial, grad_proj, grad_coord, B, V, nvox, st);
  }
  return LT_OK;
}

extern "C" int lt_softargmax3d_coord_bwd(const float* probs, const float* grad_keypoints, float* grad_coord, int B, int J, long nvox,
                                         int softmax, void* stream) {
  LT_REQUIRE(probs && grad_keypoints && grad_coord, "softargmax3d_coord_bwd: null pointer");
  LT_REQUIRE(B > 0 && J > 0 && nvox > 0 && B <= 65535, "softargmax3d_coord_bwd: bad sizes");
  LT_REQUIRE(softmax == 0 || softmax == 1,
             "softargmax3d_coord_bwd: mode must be 0 (ReLU) or 1 (softmax), got %d (mode 2, the 2-D op, has no coordinate input)", softmax);
  long bx = (nvox + 255) / 256;
  const long cap = (long)sm_count() * 8;
  if (bx > cap) bx = cap;
  softargmax_coord_bwd_kernel<<<dim3((unsigned)bx, (unsigned)B), 256, 0, (cudaStream_t)stream>>>(probs, grad_keypoints, grad_coord, J, nvox);
  LT_CHECK_LAUNCH("softargmax_coord_bwd_kernel");
  return LT_OK;
}

extern "C" int lt_softargmax3d_bwd(const float* probs, const float* coord, const float* grad_keypoints, const float* grad_volumes,
                                   float* grad_logits, float* scratch, int B, int J, long nvox, float multiplier, int softmax, void* stream) {
  LT_REQUIRE(probs && coord && grad_keypoints && grad_logits && scratch, "softargmax3d_bwd: null pointer");
  LT_REQUIRE(B > 0 && J > 0 && nvox > 0 && (long)B * J <= 65535, "softargmax3d_bwd: bad sizes");
  LT_REQUIRE(softmax >= 0 && softmax <= 2, "softargmax3d_bwd: mode must be 0 (ReLU), 1 (softmax) or 2 (ReLU, mass-normalised coordinates), got %d",
             softmax);
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
      unproject_bwd_item<false>(p, b, it, nullptr, (grad_conf && agg == LT_AGG_CONF) ? grad_conf + (long)b * V * C : nullptr);
  return LT_OK;
}

static void geom_host_tail(const float* proj, const float* coord, float* q, float* grad_proj, float* grad_coord, int B, int V, int h, int w,
                           long nvox);

extern "C" int lt_test_unproject_aggregate_bwd_geom_host(const float* features, const float* proj, const float* coord, const float* conf,
                                                         const float* grad_out, float* grad_features, float* grad_conf, float* grad_proj,
                                                         float* grad_coord, int B, int V, int C, int h, int w, long nvox, int agg) {
  LT_REQUIRE(features && proj && coord && grad_out && grad_features && C % 4 == 0 && B > 0 && V > 0 && nvox > 0,
             "test_unproject_bwd_geom_host: bad arguments");
  LT_REQUIRE(agg >= LT_AGG_SUM && agg <= LT_AGG_CONF && (agg != LT_AGG_CONF || conf), "test_unproject_bwd_geom_host: bad aggregation");
  float* q = static_cast<float*>(calloc((size_t)B * V * nvox * 3, sizeof(float)));
  LT_REQUIRE(q, "test_unproject_bwd_geom_host: out of memory");
  UnprojBwdParams p{features, proj, coord, conf, grad_out, grad_features, grad_conf, B, V, C, h, w, agg, nvox, q};
  const long items = nvox * (C / 4);
  for (int b = 0; b < B; ++b)
    for (long it = 0; it < items; ++it)
      unproject_bwd_item<true>(p, b, it, nullptr, (grad_conf && agg == LT_AGG_CONF) ? grad_conf + (long)b * V * C : nullptr);
  geom_host_tail(proj, coord, q, grad_proj, grad_coord, B, V, h, w, nvox);
  free(q);
  return LT_OK;
}

// (G_ix, G_iy) accumulated in q's first two slots -> q, then dP and dX, as the GPU's geometry passes form them
static void geom_host_tail(const float* proj, const float* coord, float* q, float* grad_proj, float* grad_coord, int B, int V, int h, int w,
                           long nvox) {
  for (int b = 0; b < B; ++b)       // (G_ix, G_iy) -> q, as the voxel's first lane forms it on the GPU
    for (int v = 0; v < V; ++v)
      for (long vox = 0; vox < nvox; ++vox) {
        const float* cp = coord + ((long)b * nvox + vox) * 3;
        GeomTaps gt;
        bwd_taps_impl<true>(proj + ((long)b * V + v) * 12, cp[0], cp[1], cp[2], h, w, &gt);
        float* qp = q + (((long)b * V + v) * nvox + vox) * 3;
        geom_q(gt, qp[0], qp[1], h, w, qp);
      }
  for (int bv = 0; grad_proj && bv < B * V; ++bv) {
    double acc[12] = {0.0};
    for (long vox = 0; vox < nvox; ++vox) {
      double t[12];
      geom_dp_terms(coord, q, nvox, bv / V, bv, vox, t);
      for (int e = 0; e < 12; ++e) acc[e] += t[e];
    }
    for (int e = 0; e < 12; ++e) grad_proj[(long)bv * 12 + e] = (float)acc[e];
  }
  for (int b = 0; grad_coord && b < B; ++b)
    for (long vox = 0; vox < nvox; ++vox) geom_dx_item(proj, q, grad_coord, V, nvox, b, vox);
}

// the fixed-order path on the CPU: pass 1 and the gather / confidence items of the GPU, with a host counting sort (stable: voxels in
// order within a cell, the order cub's stable radix sort gives)
extern "C" int lt_test_unproject_aggregate_bwd_det_host(const float* features, const float* proj, const float* coord, const float* conf,
                                                        const float* grad_out, float* grad_features, float* grad_conf, float* grad_proj,
                                                        float* grad_coord, int B, int V, int C, int h, int w, long nvox, int agg) {
  LT_REQUIRE(features && proj && coord && grad_out && grad_features && C % 4 == 0 && det_sizes_ok(B, V, h, w, nvox),
             "test_unproject_bwd_det_host: bad arguments");
  LT_REQUIRE(agg >= LT_AGG_SUM && agg <= LT_AGG_CONF && (agg != LT_AGG_CONF || conf), "test_unproject_bwd_det_host: bad aggregation");
  const bool geom = grad_proj != nullptr || grad_coord != nullptr;
  const long n = (long)B * V * nvox, nkeys = (long)B * V * det_keys_per_view(h, w);
  std::vector<float> gs((size_t)n * C + 4), q(geom ? (size_t)n * 3 : 0, 0.0f);
  std::vector<unsigned> key(n), vox(n), sorted(n), seg_begin(nkeys, 0), seg_end(nkeys, 0);
  UnprojBwdParams p{features, proj, coord, conf, grad_out, grad_features, nullptr, B, V, C, h, w, agg, nvox, geom ? q.data() : nullptr,
                    gs.data(), key.data(), vox.data()};
  const long items = nvox * (C / 4);
  for (int b = 0; b < B; ++b)
    for (long it = 0; it < items; ++it) {
      if (geom) unproject_bwd_item<true, true>(p, b, it, nullptr, nullptr);
      else unproject_bwd_item<false, true>(p, b, it, nullptr, nullptr);
    }
  for (long i = 0; i < n; ++i) ++seg_end[key[i]];
  for (long k = 0, off = 0; k < nkeys; ++k) { seg_begin[k] = (unsigned)off; off += seg_end[k]; seg_end[k] = seg_begin[k]; }
  for (long i = 0; i < n; ++i) sorted[seg_end[key[i]]++] = vox[i];
  for (int bv = 0; bv < B * V; ++bv)
    for (int pix = 0; pix < h * w; ++pix)
      for (int c0 = 0; c0 < C; c0 += 4) {
        const float4 a = det_gather_item(p, seg_begin.data(), seg_end.data(), sorted.data(), bv, pix, c0);
        float* d = grad_features + ((long)bv * h * w + pix) * C + c0;
        d[0] += a.x; d[1] += a.y; d[2] += a.z; d[3] += a.w;
      }
  if (grad_conf && agg == LT_AGG_CONF) {
    const long chunks = det_conf_chunks(nvox);
    std::vector<float> partial((size_t)B * V * chunks * C);
    for (int bv = 0; bv < B * V; ++bv)
      for (long ch = 0; ch < chunks; ++ch)
        for (int c0 = 0; c0 < C; c0 += 4) {
          const float4 a = det_conf_partial(p, bv, ch, c0);
          float* d = partial.data() + ((long)bv * chunks + ch) * C + c0;
          d[0] = a.x; d[1] = a.y; d[2] = a.z; d[3] = a.w;
        }
    for (long i = 0; i < (long)B * V * C; ++i) det_conf_merge_item(partial.data(), grad_conf, C, chunks, i);
  }
  if (geom) geom_host_tail(proj, coord, q.data(), grad_proj, grad_coord, B, V, h, w, nvox);
  return LT_OK;
}

extern "C" int lt_test_softargmax3d_coord_bwd_host(const float* probs, const float* grad_keypoints, float* grad_coord, int B, int J,
                                                   long nvox) {
  LT_REQUIRE(probs && grad_keypoints && grad_coord && B > 0 && J > 0 && nvox > 0, "test_softargmax3d_coord_bwd_host: bad arguments");
  for (int b = 0; b < B; ++b)
    for (long i = 0; i < nvox; ++i) softargmax_coord_bwd_item(probs, grad_keypoints, grad_coord, J, nvox, b, i);
  return LT_OK;
}

extern "C" int lt_test_softargmax3d_bwd_host(const float* probs, const float* coord, const float* grad_keypoints, const float* grad_volumes,
                                             float* grad_logits, int B, int J, long nvox, float multiplier, int softmax) {
  LT_REQUIRE(probs && coord && grad_keypoints && grad_logits, "test_softargmax3d_bwd_host: null pointer");
  LT_REQUIRE(softmax >= 0 && softmax <= 2, "test_softargmax3d_bwd_host: mode must be 0, 1 or 2, got %d", softmax);
  SoftBwdParams p{probs, coord, grad_keypoints, grad_volumes, nullptr, grad_logits, B, J, softmax, nvox, multiplier};
  for (int bj = 0; bj < B * J; ++bj) {
    const int b = bj / J, j = bj % J;
    const float gx = grad_keypoints[bj * 3], gy = grad_keypoints[bj * 3 + 1], gz = grad_keypoints[bj * 3 + 2];
    const float* pr = probs + (long)bj * nvox;
    if (softmax == 2) {
      double num = 0.0, M = 0.0;
      for (long i = 0; i < nvox; ++i) {
        num += (double)pr[i] * soft_tk(p, b, i, gx, gy, gz);
        M += pr[i];
      }
      const float S = (float)(num / M);
      for (long i = 0; i < nvox; ++i)
        grad_logits[(long)bj * nvox + i] = soft_grad_mass(p, pr[i], soft_tk(p, b, i, gx, gy, gz), soft_gvol(p, b, j, i), S, (float)M);
      continue;
    }
    double S = 0.0;
    if (softmax)
      for (long i = 0; i < nvox; ++i) S += (double)pr[i] * soft_t(p, b, j, i, gx, gy, gz);
    for (long i = 0; i < nvox; ++i) grad_logits[(long)bj * nvox + i] = soft_grad(p, pr[i], soft_t(p, b, j, i, gx, gy, gz), (float)S);
  }
  return LT_OK;
}
