// Fused unprojection + cross-view aggregation (HBM-bound).
//
// Replaces mvn/utils/op.py:99-166 (unproject_heatmaps): the reference loops over B*V pairs,
// launches ~15 ATen kernels per pair, materialises a (V, C, N^3) staging tensor per sample and
// makes >= 5 more passes over it for the softmax aggregation.  Here one launch does everything:
// a group of G = C/4 lanes owns one voxel; per view the group builds the projection ray
// (3x4 matvec, depth test, perspective divide), derives the four bilinear taps with
// grid_sample(align_corners=True, padding zeros) semantics -- including the reference's
// normalisation quirk (x divided by the map HEIGHT, y by the WIDTH, op.py:128-129) -- fetches
// each tap as one coalesced 16-byte load per lane (C=32 -> one 128-byte line per tap per voxel
// from the channels-last feature map), keeps the V per-view samples in registers, aggregates
// (softmax / sum / max / conf) and writes the voxel's C channels once, channels-last, either as
// float32 or directly in the split-fp16 operand format of the V2V tensor-core convs.
//
// Algorithmic bytes per sample (V=4, C=32, 96x96 maps, 64^3 voxels, fp32 out):
//   33.55 MB volume write + 4.72 MB feature read (compulsory) + 3.15 MB coordinate read = 41.42 MB.
#include "common.cuh"
#include <stdlib.h>

namespace lt {

constexpr int kMaxStoredViews = 8;
constexpr int kMaxSmemViews = 64;

struct UnprojParams {
  const float* features;  // [B][V][h][w][C]
  const float* proj;      // [B][V][12]
  const float* coord;     // [B][nvox][3]
  const float* conf;      // [B][V][C] or null
  void* out;              // full: [B][nvox][C] (fmt); partial: float [B][P][nvox][C]
  int B, V, C, h, w;
  long nvox;
  int agg, out_format, G, partial;
  // partial == 2 ("push"): sample b's partial goes to peer[b / samples_per_owner] (P2P store over NVLink) at slot src_rank
  float* peer[8];
  int samples_per_owner, src_rank;
  // v2 kernel: cubic volumes (nvox = n^3, n % brick == 0) are walked brick by brick (brick^3 voxels at a time per CTA) so that
  // the 2x2 tap cells of a CTA's consecutive voxels overlap in every view and are served by L1 instead of the 64 B/clk L2 port
  int brick_n, brick;
  int brick_order;   // voxel order inside a brick: 0 = z fastest, 1 = x fastest, 2 = 2 x 2 (x, y) tiles fastest (see brick_decode)
};

// Voxel w of a brick^3 block -> (dx, dy, dz).  Which voxels share a warp decides how many DISTINCT 128-byte feature rows one tap
// instruction touches (the L1 serves one row per wavefront, whatever the number of lanes reading it): a camera moves the projection by
// ~0.37 px per voxel along its viewing direction and ~1.1 px across it (cuboid 2.5 m / 64, heat-maps 96 x 96), and cameras look
// horizontally, so vertical (z) neighbours never share a bilinear cell while neighbours along the viewing axis mostly do.
//   0: z fastest (4 z-neighbours per warp: no sharing); 1: x fastest; 2: 2 x 2 tiles in (x, y) fastest: every horizontal camera
//   direction gets one close pair per warp.
__device__ __forceinline__ void brick_decode(int w, int bs, int order, int& dx, int& dy, int& dz) {
  if (order == 1) { dx = w % bs; dy = (w / bs) % bs; dz = w / (bs * bs); }
  else if (order == 2) {
    const int q = w & 3, r = w >> 2, hb = bs >> 1;
    dx = 2 * (r % hb) + (q & 1); dy = 2 * ((r / hb) % hb) + (q >> 1); dz = r / (hb * hb);
  } else { dz = w % bs; dy = (w / bs) % bs; dx = w / (bs * bs); }
}


struct Taps {
  int o00, o01, o10, o11;  // pixel offsets (y*w + x), valid only when the matching weight flag is set
  float w00, w01, w10, w11;
  float fx, fy;            // fractional position inside the cell (exact: ix - floor(ix))
  int xi, yi;              // integer cell coordinates (clamped to [-2, size])
  unsigned mask;           // bit i set -> tap i inside the map; 0 when depth <= 0
};

__device__ __forceinline__ Taps make_taps(const float* __restrict__ P, float X, float Y, float Z, int h, int w) {
  Taps t;
  // [X Y Z 1] . P^T (multiview.py:104), k-sequential accumulation like sgemm
  float px = fmaf(Z, P[2], fmaf(Y, P[1], X * P[0])) + P[3];
  float py = fmaf(Z, P[6], fmaf(Y, P[5], X * P[4])) + P[7];
  float pz = fmaf(Z, P[10], fmaf(Y, P[9], X * P[8])) + P[11];
  const bool depth_ok = !(pz <= 0.0f);      // op.py:121
  if (pz == 0.0f) pz = 1.0f;                // op.py:123
  const float x = px / pz, y = py / pz;     // multiview.py:84
  // op.py:128-129: x normalised by heatmap_shape[0] (= h), y by heatmap_shape[1] (= w)
  const float gx = 2.0f * (x / (float)h - 0.5f);
  const float gy = 2.0f * (y / (float)w - 0.5f);
  // grid_sample unnormalise, align_corners=True
  const float ix = ((gx + 1.0f) / 2.0f) * (float)(w - 1);
  const float iy = ((gy + 1.0f) / 2.0f) * (float)(h - 1);
  const float x0 = floorf(ix), y0 = floorf(iy);
  const float x1 = x0 + 1.0f, y1 = y0 + 1.0f;
  t.fx = ix - x0;
  t.fy = iy - y0;
  t.w00 = (x1 - ix) * (y1 - iy);  // nw
  t.w01 = (ix - x0) * (y1 - iy);  // ne
  t.w10 = (x1 - ix) * (iy - y0);  // sw
  t.w11 = (ix - x0) * (iy - y0);  // se
  const float wm = (float)(w - 1), hm = (float)(h - 1);
  const bool vx0 = (x0 >= 0.0f) && (x0 <= wm), vx1 = (x1 >= 0.0f) && (x1 <= wm);
  const bool vy0 = (y0 >= 0.0f) && (y0 <= hm), vy1 = (y1 >= 0.0f) && (y1 <= hm);
  // NaN/inf-safe integer conversion (comparisons above are false for NaN)
  const int xi = (int)fminf(fmaxf(x0, -2.0f), wm + 1.0f);
  const int yi = (int)fminf(fmaxf(y0, -2.0f), hm + 1.0f);
  t.xi = xi; t.yi = yi;
  t.o00 = yi * w + xi;
  t.o01 = t.o00 + 1;
  t.o10 = t.o00 + w;
  t.o11 = t.o10 + 1;
  t.mask = depth_ok ? ((vx0 && vy0 ? 1u : 0u) | (vx1 && vy0 ? 2u : 0u) | (vx0 && vy1 ? 4u : 0u) | (vx1 && vy1 ? 8u : 0u)) : 0u;
  return t;
}

template <int VEC>
__device__ __forceinline__ void load_vec(const float* p, float (&v)[VEC]) {
  if constexpr (VEC == 4) {
    const float4 q = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  } else {
    v[0] = __ldg(p);
  }
}

template <int VEC>
__device__ __forceinline__ void sample(const float* __restrict__ fmap, int C, int c0, const Taps& t, float (&s)[VEC]) {
#pragma unroll
  for (int i = 0; i < VEC; ++i) s[i] = 0.0f;
  float v[VEC];
  if (t.mask & 1u) { load_vec<VEC>(fmap + (long)t.o00 * C + c0, v);
#pragma unroll
    for (int i = 0; i < VEC; ++i) s[i] = fmaf(v[i], t.w00, s[i]); }
  if (t.mask & 2u) { load_vec<VEC>(fmap + (long)t.o01 * C + c0, v);
#pragma unroll
    for (int i = 0; i < VEC; ++i) s[i] = fmaf(v[i], t.w01, s[i]); }
  if (t.mask & 4u) { load_vec<VEC>(fmap + (long)t.o10 * C + c0, v);
#pragma unroll
    for (int i = 0; i < VEC; ++i) s[i] = fmaf(v[i], t.w10, s[i]); }
  if (t.mask & 8u) { load_vec<VEC>(fmap + (long)t.o11 * C + c0, v);
#pragma unroll
    for (int i = 0; i < VEC; ++i) s[i] = fmaf(v[i], t.w11, s[i]); }
}

template <int VEC>
__device__ __forceinline__ void store_out(const UnprojParams& p, long b, long vox, int c0, const float (&o)[VEC]) {
  if (p.out_format == LT_FMT_F32) {
    float* dst = reinterpret_cast<float*>(p.out) + ((long)b * p.nvox + vox) * p.C + c0;
    if constexpr (VEC == 4) *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
    else dst[0] = o[0];
  } else {
    sh_t* row = reinterpret_cast<sh_t*>(p.out) + ((long)b * p.nvox + vox) * 2 * p.C;
    if constexpr (VEC == 4) store_s32x4(row, c0, make_float4(o[0], o[1], o[2], o[3]));
    else {
      sh_t hi, lo;
      split_s32(o[0], hi, lo);
      row[s32_off(c0)] = hi;
      row[s32_off(c0) + 32] = lo;
    }
  }
}

// STORED: V <= kMaxStoredViews, per-view samples kept in registers (two-pass softmax with the
// max subtracted, like torch.softmax); otherwise a streaming (online) softmax is used.
template <int VEC, bool STORED>
__global__ void __launch_bounds__(256) unproject_kernel(const UnprojParams p) {
  __shared__ float sP[kMaxSmemViews * 12];
  const int b = blockIdx.y;
  const int nP = min(p.V, kMaxSmemViews) * 12;
  for (int i = threadIdx.x; i < nP; i += blockDim.x) sP[i] = p.proj[(long)b * p.V * 12 + i];
  __syncthreads();

  const int G = p.G;
  const int slot = threadIdx.x / G, sub = threadIdx.x % G;
  const int vpb = blockDim.x / G;
  const long map_elems = (long)p.h * p.w * p.C;

  for (long vox = (long)blockIdx.x * vpb + slot; vox < p.nvox; vox += (long)gridDim.x * vpb) {
    const float* cp = p.coord + ((long)b * p.nvox + vox) * 3;
    const float X = __ldg(cp), Y = __ldg(cp + 1), Z = __ldg(cp + 2);

    for (int c0 = sub * VEC; c0 < p.C; c0 += G * VEC) {
      float acc[VEC], aux[VEC], run_max[VEC];
      float st[STORED ? kMaxStoredViews : 1][VEC];
#pragma unroll
      for (int i = 0; i < VEC; ++i) { acc[i] = 0.0f; aux[i] = 0.0f; run_max[i] = -INFINITY; }

      const int vend = STORED ? kMaxStoredViews : p.V;
#pragma unroll
      for (int v = 0; v < vend; ++v) {
        if (STORED && v >= p.V) break;
        const float* Pm = (v < kMaxSmemViews) ? (sP + v * 12) : (p.proj + ((long)b * p.V + v) * 12);
        const Taps t = make_taps(Pm, X, Y, Z, p.h, p.w);
        float s[VEC];
        sample<VEC>(p.features + ((long)b * p.V + v) * map_elems, p.C, c0, t, s);

        if (p.partial) {
          if (p.agg == LT_AGG_SOFTMAX) {
#pragma unroll
            for (int i = 0; i < VEC; ++i) { const float e = expf(s[i]); acc[i] = fmaf(s[i], e, acc[i]); aux[i] += e; }
          } else if (p.agg == LT_AGG_MAX) {
#pragma unroll
            for (int i = 0; i < VEC; ++i) run_max[i] = fmaxf(run_max[i], s[i]);
          } else if (p.agg == LT_AGG_CONF) {
            float cf[VEC];
            load_vec<VEC>(p.conf + ((long)b * p.V + v) * p.C + c0, cf);
#pragma unroll
            for (int i = 0; i < VEC; ++i) acc[i] = fmaf(s[i], cf[i], acc[i]);
          } else {
#pragma unroll
            for (int i = 0; i < VEC; ++i) acc[i] += s[i];
          }
        } else if (p.agg == LT_AGG_SOFTMAX) {
          if constexpr (STORED) {
#pragma unroll
            for (int i = 0; i < VEC; ++i) { st[v][i] = s[i]; run_max[i] = fmaxf(run_max[i], s[i]); }
          } else {
#pragma unroll
            for (int i = 0; i < VEC; ++i) {
              const float m = fmaxf(run_max[i], s[i]);
              const float r = expf(run_max[i] - m), e = expf(s[i] - m);
              acc[i] = fmaf(acc[i], r, s[i] * e);
              aux[i] = fmaf(aux[i], r, e);
              run_max[i] = m;
            }
          }
        } else if (p.agg == LT_AGG_MAX) {
#pragma unroll
          for (int i = 0; i < VEC; ++i) run_max[i] = fmaxf(run_max[i], s[i]);
        } else if (p.agg == LT_AGG_CONF) {
          float cf[VEC];
          load_vec<VEC>(p.conf + ((long)b * p.V + v) * p.C + c0, cf);
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[i] = fmaf(s[i], cf[i], acc[i]);
        } else {
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[i] += s[i];
        }
      }

      if (p.partial) {
        float* base = reinterpret_cast<float*>(p.out);
        const int planes = (p.agg == LT_AGG_SOFTMAX) ? 2 : 1;
        float* d0 = base + (((long)b * planes + 0) * p.nvox + vox) * p.C + c0;
        const float* src = (p.agg == LT_AGG_MAX) ? run_max : acc;
        if constexpr (VEC == 4) *reinterpret_cast<float4*>(d0) = make_float4(src[0], src[1], src[2], src[3]);
        else d0[0] = src[0];
        if (planes == 2) {
          float* d1 = d0 + p.nvox * p.C;
          if constexpr (VEC == 4) *reinterpret_cast<float4*>(d1) = make_float4(aux[0], aux[1], aux[2], aux[3]);
          else d1[0] = aux[0];
        }
        continue;
      }

      float o[VEC];
      if (p.agg == LT_AGG_SOFTMAX) {
        if constexpr (STORED) {
          float den[VEC];
#pragma unroll
          for (int i = 0; i < VEC; ++i) den[i] = 0.0f;
#pragma unroll
          for (int v = 0; v < kMaxStoredViews; ++v) {
            if (v >= p.V) break;
#pragma unroll
            for (int i = 0; i < VEC; ++i) den[i] += expf(st[v][i] - run_max[i]);
          }
#pragma unroll
          for (int i = 0; i < VEC; ++i) o[i] = 0.0f;
#pragma unroll
          for (int v = 0; v < kMaxStoredViews; ++v) {
            if (v >= p.V) break;
#pragma unroll
            for (int i = 0; i < VEC; ++i) {
              const float pr = expf(st[v][i] - run_max[i]) / den[i];   // softmax over views (op.py:158)
              o[i] = fmaf(st[v][i], pr, o[i]);                          // (vol * softmax).sum(0) (op.py:162)
            }
          }
        } else {
#pragma unroll
          for (int i = 0; i < VEC; ++i) o[i] = acc[i] / aux[i];
        }
      } else if (p.agg == LT_AGG_MAX) {
#pragma unroll
        for (int i = 0; i < VEC; ++i) o[i] = run_max[i];
      } else {
#pragma unroll
        for (int i = 0; i < VEC; ++i) o[i] = acc[i];
      }
      store_out<VEC>(p, b, vox, c0, o);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Fast path (C = 4*G channels, V <= 8): the G lanes of a voxel group split the per-view ray setup
// (lane j builds the taps of view j and the group shares them with width-G shuffles), per-view samples
// stay in registers and the view softmax is one pass (max, then exp once: num = sum s*e, den = sum e).
// ------------------------------------------------------------------------------------------------
template <int G, int MAXV, int CPL>   // CPL channels per lane (4 or 8): C = CPL * G
__global__ void __launch_bounds__(256) unproject_fast_kernel(const UnprojParams p) {
  __shared__ float sP[kMaxStoredViews * 12];
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < p.V * 12; i += blockDim.x) sP[i] = p.proj[(long)b * p.V * 12 + i];
  __syncthreads();

  constexpr int C = CPL * G;
  constexpr int NQ = CPL / 4;
  const int sub = threadIdx.x % G;
  const int slot = threadIdx.x / G;
  constexpr int VPB = 256 / G;
  const long map_elems = (long)p.h * p.w * C;
  const float* fbase = p.features + (long)b * p.V * map_elems + sub * CPL;
  const int c0 = sub * CPL;
  const int wm = p.w - 1, hm = p.h - 1;

  // block-uniform trip count: the width-G shuffles below need every lane of the warp present
  // work items: VPB consecutive voxels (linear order), or -- brick mode -- VPB voxels of one brick^3 block (z fastest)
  const int bs = p.brick, bpd = p.brick_n > 0 ? p.brick_n / bs : 0;            // brick side, bricks per dimension
  const int bvol = bs * bs * bs;
  const int ipb = p.brick_n > 0 ? bvol / VPB : 1;             // items per brick: a CTA finishes a brick before taking the next
  const long n_outer = p.brick_n > 0 ? (long)bpd * bpd * bpd : (p.nvox + VPB - 1) / VPB;
  for (long outer = blockIdx.x; outer < n_outer; outer += gridDim.x)
  for (int inner = 0; inner < ipb; ++inner) {
    const long item = outer * ipb + inner;
    long vox;
    bool live;
    if (p.brick_n > 0) {
      const long brick = outer;
      const int w = inner * VPB + slot;                        // voxel inside the brick
      const int bz = (int)(brick % bpd), by = (int)((brick / bpd) % bpd), bx = (int)(brick / ((long)bpd * bpd));
      int dx, dy, dz;
      brick_decode(w, bs, p.brick_order, dx, dy, dz);
      vox = ((long)(bx * bs + dx) * p.brick_n + (by * bs + dy)) * p.brick_n + (bz * bs + dz);
      live = true;
    } else {
      live = item * VPB + slot < p.nvox;
      vox = live ? item * VPB + slot : p.nvox - 1;
    }
    const float* cp = p.coord + ((long)b * p.nvox + vox) * 3;
    const float X = __ldg(cp), Y = __ldg(cp + 1), Z = __ldg(cp + 2);
    float s[MAXV][CPL];
#pragma unroll
    for (int v0 = 0; v0 < MAXV; v0 += G) {
      if (v0 >= p.V) break;
      // my share of the ray setup: view v0 + sub
      int xi_m = 0, yi_m = 0; float fx_m = 0.f, fy_m = 0.f; unsigned mask_m = 0u;
      if (v0 + sub < p.V) {
        const Taps t = make_taps(sP + (v0 + sub) * 12, X, Y, Z, p.h, p.w);
        xi_m = t.xi; yi_m = t.yi; mask_m = t.mask;
        fx_m = t.fx; fy_m = t.fy;
      }
#pragma unroll
      for (int j = 0; j < G; ++j) {
        const int v = v0 + j;
        if (v >= MAXV) break;
        if (v < p.V) {
          const int xi = __shfl_sync(0xffffffffu, xi_m, j, G);
          const int yi = __shfl_sync(0xffffffffu, yi_m, j, G);
          const float fx = __shfl_sync(0xffffffffu, fx_m, j, G);
          const float fy = __shfl_sync(0xffffffffu, fy_m, j, G);
          const unsigned mask = __shfl_sync(0xffffffffu, mask_m, j, G);
          // unconditional, clamped loads (independent -> all taps of all views in flight); invalid taps get weight 0
          const int x0 = min(max(xi, 0), wm), x1 = min(max(xi + 1, 0), wm);
          const int y0 = min(max(yi, 0), hm), y1 = min(max(yi + 1, 0), hm);
          const float* f = fbase + (long)v * map_elems;
          const float* f00 = f + (long)(y0 * p.w + x0) * C;
          const float* f01 = f + (long)(y0 * p.w + x1) * C;
          const float* f10 = f + (long)(y1 * p.w + x0) * C;
          const float* f11 = f + (long)(y1 * p.w + x1) * C;
          float4 q00[NQ], q01[NQ], q10[NQ], q11[NQ];
#pragma unroll
          for (int qd = 0; qd < NQ; ++qd) {
            q00[qd] = __ldg(reinterpret_cast<const float4*>(f00) + qd);
            q01[qd] = __ldg(reinterpret_cast<const float4*>(f01) + qd);
            q10[qd] = __ldg(reinterpret_cast<const float4*>(f10) + qd);
            q11[qd] = __ldg(reinterpret_cast<const float4*>(f11) + qd);
          }
          const float gx = 1.0f - fx, gy = 1.0f - fy;
          const float w00 = (mask & 1u) ? gx * gy : 0.0f, w01 = (mask & 2u) ? fx * gy : 0.0f;
          const float w10 = (mask & 4u) ? gx * fy : 0.0f, w11 = (mask & 8u) ? fx * fy : 0.0f;
#pragma unroll
          for (int qd = 0; qd < NQ; ++qd) {
            s[v][qd * 4 + 0] = fmaf(q11[qd].x, w11, fmaf(q10[qd].x, w10, fmaf(q01[qd].x, w01, q00[qd].x * w00)));
            s[v][qd * 4 + 1] = fmaf(q11[qd].y, w11, fmaf(q10[qd].y, w10, fmaf(q01[qd].y, w01, q00[qd].y * w00)));
            s[v][qd * 4 + 2] = fmaf(q11[qd].z, w11, fmaf(q10[qd].z, w10, fmaf(q01[qd].z, w01, q00[qd].z * w00)));
            s[v][qd * 4 + 3] = fmaf(q11[qd].w, w11, fmaf(q10[qd].w, w10, fmaf(q01[qd].w, w01, q00[qd].w * w00)));
          }
        }
      }
    }

    float o[CPL], o2[CPL];
    if (p.agg == LT_AGG_SOFTMAX) {
      if (p.partial) {
#pragma unroll
        for (int i = 0; i < CPL; ++i) { o[i] = 0.f; o2[i] = 0.f; }
#pragma unroll
        for (int v = 0; v < MAXV; ++v)
          if (v < p.V) {
#pragma unroll
            for (int i = 0; i < CPL; ++i) { const float e = __expf(s[v][i]); o[i] = fmaf(s[v][i], e, o[i]); o2[i] += e; }
          }
      } else {
#pragma unroll
        for (int i = 0; i < CPL; ++i) {
          float m = -INFINITY;
#pragma unroll
          for (int v = 0; v < MAXV; ++v) if (v < p.V) m = fmaxf(m, s[v][i]);
          float num = 0.f, den = 0.f;
#pragma unroll
          for (int v = 0; v < MAXV; ++v)
            if (v < p.V) { const float e = __expf(s[v][i] - m); num = fmaf(s[v][i], e, num); den += e; }
          o[i] = num / den;
        }
      }
    } else if (p.agg == LT_AGG_MAX) {
#pragma unroll
      for (int i = 0; i < CPL; ++i) o[i] = -INFINITY;
#pragma unroll
      for (int v = 0; v < MAXV; ++v)
        if (v < p.V) {
#pragma unroll
          for (int i = 0; i < CPL; ++i) o[i] = fmaxf(o[i], s[v][i]);
        }
    } else {
#pragma unroll
      for (int i = 0; i < CPL; ++i) o[i] = 0.f;
#pragma unroll
      for (int v = 0; v < MAXV; ++v)
        if (v < p.V) {
#pragma unroll
          for (int qd = 0; qd < NQ; ++qd) {
            float cf[4] = {1.f, 1.f, 1.f, 1.f};
            if (p.agg == LT_AGG_CONF) load_vec<4>(p.conf + ((long)b * p.V + v) * C + c0 + qd * 4, cf);
#pragma unroll
            for (int i = 0; i < 4; ++i) o[qd * 4 + i] = fmaf(s[v][qd * 4 + i], cf[i], o[qd * 4 + i]);
          }
        }
    }

    if (!live) continue;
    if (p.partial) {
      const int planes = (p.agg == LT_AGG_SOFTMAX) ? 2 : 1;
      float* d0;
      if (p.partial == 2) {   // fused exchange: write straight into the owner rank's reduction buffer (peer memory)
        const int owner = b / p.samples_per_owner, bl = b % p.samples_per_owner;
        d0 = p.peer[owner] + ((((long)p.src_rank * p.samples_per_owner + bl) * planes) * p.nvox + vox) * C + c0;
      } else {
        d0 = reinterpret_cast<float*>(p.out) + (((long)b * planes) * p.nvox + vox) * C + c0;
      }
#pragma unroll
      for (int qd = 0; qd < NQ; ++qd) {
        reinterpret_cast<float4*>(d0)[qd] = make_float4(o[qd * 4], o[qd * 4 + 1], o[qd * 4 + 2], o[qd * 4 + 3]);
        if (planes == 2) reinterpret_cast<float4*>(d0 + p.nvox * C)[qd] = make_float4(o2[qd * 4], o2[qd * 4 + 1], o2[qd * 4 + 2], o2[qd * 4 + 3]);
      }
    } else {
#pragma unroll
      for (int qd = 0; qd < NQ; ++qd) {
        const float oq[4] = {o[qd * 4], o[qd * 4 + 1], o[qd * 4 + 2], o[qd * 4 + 3]};
        store_out<4>(p, b, vox, c0 + qd * 4, oq);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Production-shape specialisation (C = 32, softmax aggregation, full output, V <= MAXV): same lane layout as the
// fast kernel (8 lanes x float4 per voxel), but the lane that builds view j's ray also finishes the tap set -- four
// clamped pixel offsets and four weights with the validity mask folded in -- so the seven consuming lanes only
// shuffle, add and load; divisions use the reciprocal unit (the bilinear sample is continuous in the pixel
// coordinate, so a 2-ulp coordinate difference moves the sample by ~1e-6 of the feature scale); all control flow on
// V / aggregation / output format is resolved at compile time.  ~35 % fewer issued instructions per voxel.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

__device__ __forceinline__ float ex2_approx(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
// base + idx (float4 units) as ONE 64-bit multiply-add
__device__ __forceinline__ const float4* q_at(const float4* base, unsigned idx) {
  unsigned long long r;
  asm("mad.wide.u32 %0, %1, 16, %2;" : "=l"(r) : "r"(idx), "l"(reinterpret_cast<unsigned long long>(base)));
  return reinterpret_cast<const float4*>(r);
}

// two adjacent float4 of a channels-last pixel row through the read-only path (sm_90 has no 256-bit load: two 128-bit requests)
__device__ __forceinline__ void ldg256(const float4* p, float4& a, float4& b) {
  a = __ldg(p);
  b = __ldg(p + 1);
}

template <int MAXV, int FMT, bool EXACT, int MINB, int CPL>   // EXACT: V == MAXV (no per-view predicates); MINB: min CTAs / SM; CPL: channels per lane (4 or 8)
__global__ void __launch_bounds__(256, MINB) unproject_v2_kernel(const UnprojParams p) {
  __shared__ float sP[MAXV * 12];
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < p.V * 12; i += blockDim.x) sP[i] = p.proj[(long)b * p.V * 12 + i];
  __syncthreads();
  constexpr int C = 32, G = C / CPL, NQ = CPL / 4, VPB = 256 / G;
  const int sub = threadIdx.x & (G - 1);
  const int slot = threadIdx.x / G;
  const int V = EXACT ? MAXV : p.V;
  const unsigned map_q = (unsigned)(p.h * p.w * (C / 4));   // float4 units per view map
  // this lane's CPL channels of pixel 0 of view 0; tap offsets are 32-bit counts of float4 (one IMAD.WIDE per address)
  const float4* fbase = reinterpret_cast<const float4*>(p.features + (long)b * V * p.h * p.w * C) + sub * NQ;
  const float inv_h = 1.0f / (float)p.h, inv_w = 1.0f / (float)p.w;
  const float wm = (float)(p.w - 1), hm = (float)(p.h - 1);
  const int wi = p.w - 1, hi = p.h - 1;

  // work items: VPB consecutive voxels (linear order), or -- brick mode -- VPB voxels of one brick^3 block (z fastest)
  const int bs = p.brick, bpd = p.brick_n > 0 ? p.brick_n / bs : 0;            // brick side, bricks per dimension
  const int bvol = bs * bs * bs;
  const int ipb = p.brick_n > 0 ? bvol / VPB : 1;             // items per brick: a CTA finishes a brick before taking the next
  const long n_outer = p.brick_n > 0 ? (long)bpd * bpd * bpd : (p.nvox + VPB - 1) / VPB;
  for (long outer = blockIdx.x; outer < n_outer; outer += gridDim.x)
  for (int inner = 0; inner < ipb; ++inner) {
    const long item = outer * ipb + inner;
    long vox;
    bool live;
    if (p.brick_n > 0) {
      const long brick = outer;
      const int w = inner * VPB + slot;                        // voxel inside the brick
      const int bz = (int)(brick % bpd), by = (int)((brick / bpd) % bpd), bx = (int)(brick / ((long)bpd * bpd));
      int dx, dy, dz;
      brick_decode(w, bs, p.brick_order, dx, dy, dz);
      vox = ((long)(bx * bs + dx) * p.brick_n + (by * bs + dy)) * p.brick_n + (bz * bs + dz);
      live = true;
    } else {
      live = item * VPB + slot < p.nvox;
      vox = live ? item * VPB + slot : p.nvox - 1;
    }
    const float* cp = p.coord + ((long)b * p.nvox + vox) * 3;
    const float X = __ldg(cp), Y = __ldg(cp + 1), Z = __ldg(cp + 2);
    float s[MAXV][CPL];
#pragma unroll
    for (int v0 = 0; v0 < MAXV; v0 += G) {
      // my share of the ray setup: view v0 + sub -> four clamped tap offsets and four weights with the mask folded in
      unsigned o0 = 0, o1 = 0, o2 = 0, o3 = 0;
      float w0 = 0.f, w1 = 0.f, w2 = 0.f, w3 = 0.f;
      if (v0 + sub < V) {
        const float* P = sP + (v0 + sub) * 12;
        const float px = fmaf(Z, P[2], fmaf(Y, P[1], X * P[0])) + P[3];
        const float py = fmaf(Z, P[6], fmaf(Y, P[5], X * P[4])) + P[7];
        float pz = fmaf(Z, P[10], fmaf(Y, P[9], X * P[8])) + P[11];
        const bool depth_ok = !(pz <= 0.0f);            // op.py:121
        if (pz == 0.0f) pz = 1.0f;                      // op.py:123
        const float rz = rcp_approx(pz);
        const float x = px * rz, y = py * rz;
        const float gx = 2.0f * (x * inv_h - 0.5f);     // op.py:128-129 (x by the map HEIGHT, y by the WIDTH)
        const float gy = 2.0f * (y * inv_w - 0.5f);
        const float ix = ((gx + 1.0f) * 0.5f) * wm, iy = ((gy + 1.0f) * 0.5f) * hm;
        const float x0 = floorf(ix), y0 = floorf(iy);
        const float fx = ix - x0, fy = iy - y0;
        const float ex = 1.0f - fx, ey = 1.0f - fy;
        const bool vx0 = (x0 >= 0.0f) && (x0 <= wm), vx1 = (x0 + 1.0f >= 0.0f) && (x0 + 1.0f <= wm);
        const bool vy0 = (y0 >= 0.0f) && (y0 <= hm), vy1 = (y0 + 1.0f >= 0.0f) && (y0 + 1.0f <= hm);
        const int xi = (int)fminf(fmaxf(x0, -2.0f), wm + 1.0f), yi = (int)fminf(fmaxf(y0, -2.0f), hm + 1.0f);
        const int xa = min(max(xi, 0), wi), xb = min(max(xi + 1, 0), wi);
        const int ya = min(max(yi, 0), hi), yb = min(max(yi + 1, 0), hi);
        const unsigned vb = (unsigned)(v0 + sub) * map_q;
        o0 = vb + (unsigned)(ya * p.w + xa) * (C / 4); o1 = vb + (unsigned)(ya * p.w + xb) * (C / 4);
        o2 = vb + (unsigned)(yb * p.w + xa) * (C / 4); o3 = vb + (unsigned)(yb * p.w + xb) * (C / 4);
        w0 = (depth_ok && vx0 && vy0) ? ex * ey : 0.0f;
        w1 = (depth_ok && vx1 && vy0) ? fx * ey : 0.0f;
        w2 = (depth_ok && vx0 && vy1) ? ex * fy : 0.0f;
        w3 = (depth_ok && vx1 && vy1) ? fx * fy : 0.0f;
      }
#pragma unroll
      for (int j = 0; j < G; ++j) {
        const int v = v0 + j;
        if (v >= MAXV) break;
        const unsigned a0 = __shfl_sync(0xffffffffu, o0, j, G), a1 = __shfl_sync(0xffffffffu, o1, j, G);
        const unsigned a2 = __shfl_sync(0xffffffffu, o2, j, G), a3 = __shfl_sync(0xffffffffu, o3, j, G);
        const float c0 = __shfl_sync(0xffffffffu, w0, j, G), c1 = __shfl_sync(0xffffffffu, w1, j, G);
        const float c2 = __shfl_sync(0xffffffffu, w2, j, G), c3 = __shfl_sync(0xffffffffu, w3, j, G);
        // views >= V carry offset 0 / weight 0: harmless loads of pixel 0
        const float4* t0 = q_at(fbase, a0);
        const float4* t1 = q_at(fbase, a1);
        const float4* t2 = q_at(fbase, a2);
        const float4* t3 = q_at(fbase, a3);
        if constexpr (NQ == 2) {
          float4 q0, q1, q2, q3, r0, r1, r2, r3;
          ldg256(t0, q0, r0); ldg256(t1, q1, r1); ldg256(t2, q2, r2); ldg256(t3, q3, r3);
          s[v][0] = fmaf(q3.x, c3, fmaf(q2.x, c2, fmaf(q1.x, c1, q0.x * c0)));
          s[v][1] = fmaf(q3.y, c3, fmaf(q2.y, c2, fmaf(q1.y, c1, q0.y * c0)));
          s[v][2] = fmaf(q3.z, c3, fmaf(q2.z, c2, fmaf(q1.z, c1, q0.z * c0)));
          s[v][3] = fmaf(q3.w, c3, fmaf(q2.w, c2, fmaf(q1.w, c1, q0.w * c0)));
          s[v][4] = fmaf(r3.x, c3, fmaf(r2.x, c2, fmaf(r1.x, c1, r0.x * c0)));
          s[v][5] = fmaf(r3.y, c3, fmaf(r2.y, c2, fmaf(r1.y, c1, r0.y * c0)));
          s[v][6] = fmaf(r3.z, c3, fmaf(r2.z, c2, fmaf(r1.z, c1, r0.z * c0)));
          s[v][7] = fmaf(r3.w, c3, fmaf(r2.w, c2, fmaf(r1.w, c1, r0.w * c0)));
        } else {
          const float4 q0 = __ldg(t0), q1 = __ldg(t1), q2 = __ldg(t2), q3 = __ldg(t3);
          s[v][0] = fmaf(q3.x, c3, fmaf(q2.x, c2, fmaf(q1.x, c1, q0.x * c0)));
          s[v][1] = fmaf(q3.y, c3, fmaf(q2.y, c2, fmaf(q1.y, c1, q0.y * c0)));
          s[v][2] = fmaf(q3.z, c3, fmaf(q2.z, c2, fmaf(q1.z, c1, q0.z * c0)));
          s[v][3] = fmaf(q3.w, c3, fmaf(q2.w, c2, fmaf(q1.w, c1, q0.w * c0)));
        }
      }
    }
    if constexpr (!EXACT) {
      // absent views must not take part in the view softmax: a large negative FINITE score (exp -> 0, s * 0 = -0)
#pragma unroll
      for (int v = 0; v < MAXV; ++v)
        if (v >= V) {
#pragma unroll
          for (int i = 0; i < CPL; ++i) s[v][i] = -1.0e30f;
        }
    }
    float o[CPL];
#pragma unroll
    for (int i = 0; i < CPL; ++i) {
      float m = s[0][i];
#pragma unroll
      for (int v = 1; v < MAXV; ++v) m = fmaxf(m, s[v][i]);
      const float ml = -m * 1.4426950408889634f;     // exp(s - m) = 2^(s * log2(e) - m * log2(e))
      float num = 0.f, den = 0.f;
#pragma unroll
      for (int v = 0; v < MAXV; ++v) { const float e = ex2_approx(fmaf(s[v][i], 1.4426950408889634f, ml)); num = fmaf(s[v][i], e, num); den += e; }
      o[i] = num * rcp_approx(den);                  // den in [1, V]: no range scaling needed
    }
    if (!live) continue;
#pragma unroll
    for (int qd = 0; qd < NQ; ++qd) {
      const float4 ov = make_float4(o[qd * 4], o[qd * 4 + 1], o[qd * 4 + 2], o[qd * 4 + 3]);
      if constexpr (FMT == LT_FMT_F32) {
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + ((long)b * p.nvox + vox) * C + sub * CPL + qd * 4) = ov;
      } else {
        store_s32x4(reinterpret_cast<sh_t*>(p.out) + ((long)b * p.nvox + vox) * 2 * C, sub * CPL + qd * 4, ov);
      }
    }
  }
}

// partial[B][P][nvox][C] -> out[B][nvox][C] (divide numerator by denominator for softmax)
// nslots > 1: partial is [slot][B][P][nvox][C] (one slot per source rank, filled by P2P stores) and is reduced here.
__global__ void __launch_bounds__(256) unproject_finalize_kernel(const float* __restrict__ partial, void* out, int out_format,
                                                                 int B, int C, long nvox, int agg, int nslots) {
  const long per_b = nvox * C;
  const long total4 = (long)B * per_b / 4;
  const int planes = (agg == LT_AGG_SOFTMAX) ? 2 : 1;
  const long slot_stride = (long)B * planes * per_b;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (long)gridDim.x * blockDim.x) {
    const long e = i * 4;
    const long b = e / per_b, r = e % per_b;
    float4 n = *reinterpret_cast<const float4*>(partial + (b * planes) * per_b + r);
    for (int s = 1; s < nslots; ++s) {
      const float4 t = *reinterpret_cast<const float4*>(partial + s * slot_stride + (b * planes) * per_b + r);
      if (agg == LT_AGG_MAX) { n.x = fmaxf(n.x, t.x); n.y = fmaxf(n.y, t.y); n.z = fmaxf(n.z, t.z); n.w = fmaxf(n.w, t.w); }
      else { n.x += t.x; n.y += t.y; n.z += t.z; n.w += t.w; }
    }
    float4 o = n;
    if (planes == 2) {
      float4 d = *reinterpret_cast<const float4*>(partial + (b * planes + 1) * per_b + r);
      for (int s = 1; s < nslots; ++s) {
        const float4 t = *reinterpret_cast<const float4*>(partial + s * slot_stride + (b * planes + 1) * per_b + r);
        d.x += t.x; d.y += t.y; d.z += t.z; d.w += t.w;
      }
      o = make_float4(n.x / d.x, n.y / d.y, n.z / d.z, n.w / d.w);
    }
    if (out_format == LT_FMT_F32) {
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + e) = o;
    } else {
      const long pix = e / C;
      const int c = (int)(e % C);
      store_s32x4(reinterpret_cast<sh_t*>(out) + pix * 2 * C, c, o);
    }
  }
}

static int launch_unproject(const float* features, const float* proj, const float* coord, const float* conf, void* out,
                            int out_format, int B, int V, int C, int h, int w, long nvox, int agg, int partial,
                            void* stream, float* const* peers = nullptr, int n_peers = 0, int src_rank = 0) {
  LT_REQUIRE(features && proj && coord && out, "unproject: null pointer");
  LT_REQUIRE(B > 0 && V > 0 && C > 0 && h > 0 && w > 0 && nvox > 0, "unproject: non-positive size");
  LT_REQUIRE(agg >= LT_AGG_SUM && agg <= LT_AGG_CONF, "unproject: unknown aggregation %d", agg);
  LT_REQUIRE(agg != LT_AGG_CONF || conf, "unproject: LT_AGG_CONF needs confidences");
  LT_REQUIRE(out_format == LT_FMT_F32 || (out_format == LT_FMT_S32 && C % 32 == 0),
             "unproject: split-fp16 output needs C %% 32 == 0 (C=%d)", C);
  LT_REQUIRE(B <= 65535, "unproject: batch too large");
  UnprojParams p{features, proj, coord, conf, out, B, V, C, h, w, nvox, agg, out_format, 1, partial};
  p.samples_per_owner = 1; p.src_rank = src_rank;
  p.brick_n = 0; p.brick = 8; p.brick_order = 0;
  for (int i = 0; i < 8; ++i) p.peer[i] = (peers && i < n_peers) ? peers[i] : nullptr;
  if (partial == 2) {
    LT_REQUIRE(peers && n_peers >= 1 && n_peers <= 8 && B % n_peers == 0, "unproject_push: need 1..8 peers dividing the batch");
    LT_REQUIRE(C % 4 == 0 && C <= 128 && ((C / 4) & (C / 4 - 1)) == 0 && V <= kMaxStoredViews, "unproject_push: unsupported shape");
    p.samples_per_owner = B / n_peers;
  }
  const bool vec4 = (C % 4 == 0);
  const int units = vec4 ? C / 4 : C;   // lanes wanted per voxel
  int G = 1;
  while (G < units && G < 32) G <<= 1;
  p.G = G;
  const int vpb = 256 / G;
  long blocks = (nvox + vpb - 1) / vpb;
  const long cap = (long)sm_count() * 8;    // 8 resident 256-thread CTAs per SM, grid-stride beyond
  if (blocks > cap) blocks = cap;
  dim3 grid((unsigned)blocks, (unsigned)B);
  cudaStream_t st = (cudaStream_t)stream;
  const bool stored = V <= kMaxStoredViews;
  const bool pow2q = (units & (units - 1)) == 0;
  const int v2_mode = opts().unproject_v2;
  if (v2_mode && C == 32 && agg == LT_AGG_SOFTMAX && partial == 0 && V <= 8 && (long)V * h * w * C < (1L << 30)) {
    // variants: 8 lanes x 4 channels per voxel at 4 CTAs/SM (default); 4 lanes x 8 channels halves the per-voxel ray / shuffle /
    // address overhead
    const int cpl = opts().unproject_cpl, lb = opts().unproject_lb;
    {
      // brick walk for cubic volumes (the coordinate volume of the reference is n x n x n, triangulation.py:306-311)
      long n = (long)llround(cbrt((double)nvox));
      const int bs = opts().unproject_brick;
      if (bs > 0 && n * n * n == nvox && n % bs == 0 && (bs * bs * bs) % (256 / (32 / cpl)) == 0) {
        p.brick_n = (int)n; p.brick = bs; p.brick_order = opts().unproject_brick_order;
        const long nbricks = (n / bs) * (n / bs) * (n / bs);
        grid.x = (unsigned)(nbricks < (long)sm_count() * 8 ? nbricks : (long)sm_count() * 8);
      }
    }
    if (cpl == 8 && p.brick_n == 0) {
      const int vpb8 = 64;
      long blocks8 = (nvox + vpb8 - 1) / vpb8;
      if (blocks8 > (long)sm_count() * 8) blocks8 = (long)sm_count() * 8;
      grid.x = (unsigned)blocks8;
    }
#define LT_UNPROJ_V2(FMT)                                                                   \
    if (cpl == 8 && V == 4 && lb == 3) unproject_v2_kernel<4, FMT, true, 3, 8><<<grid, 256, 0, st>>>(p); \
    else if (cpl == 8 && V == 4) unproject_v2_kernel<4, FMT, true, 2, 8><<<grid, 256, 0, st>>>(p); \
    else if (cpl == 8 && V == 8) unproject_v2_kernel<8, FMT, true, 1, 8><<<grid, 256, 0, st>>>(p); \
    else if (cpl == 8 && V < 4) unproject_v2_kernel<4, FMT, false, 2, 8><<<grid, 256, 0, st>>>(p); \
    else if (cpl == 8) unproject_v2_kernel<8, FMT, false, 1, 8><<<grid, 256, 0, st>>>(p); \
    else if (V == 4 && lb == 5) unproject_v2_kernel<4, FMT, true, 5, 4><<<grid, 256, 0, st>>>(p); \
    else if (V == 4) unproject_v2_kernel<4, FMT, true, 4, 4><<<grid, 256, 0, st>>>(p);        \
    else if (V == 8) unproject_v2_kernel<8, FMT, true, 3, 4><<<grid, 256, 0, st>>>(p);        \
    else if (V < 4) unproject_v2_kernel<4, FMT, false, 5, 4><<<grid, 256, 0, st>>>(p);        \
    else unproject_v2_kernel<8, FMT, false, 3, 4><<<grid, 256, 0, st>>>(p)
    if (out_format == LT_FMT_F32) { LT_UNPROJ_V2(LT_FMT_F32); } else { LT_UNPROJ_V2(LT_FMT_S32); }
#undef LT_UNPROJ_V2
  } else if (vec4 && stored && pow2q && C <= 128) {
    // C = 8*G' (two float4 per lane per tap: half the per-lane ray/weight overhead) when possible, else C = 4*G
#define LT_UNPROJ_FAST(GG, CPL)                                                             \
    if (V <= 2) unproject_fast_kernel<GG, 2, CPL><<<grid, 256, 0, st>>>(p);                 \
    else if (V <= 4) unproject_fast_kernel<GG, 4, CPL><<<grid, 256, 0, st>>>(p);            \
    else unproject_fast_kernel<GG, 8, CPL><<<grid, 256, 0, st>>>(p)
    {
      switch (G) {
        case 1: LT_UNPROJ_FAST(1, 4); break;
        case 2: LT_UNPROJ_FAST(2, 4); break;
        case 4: LT_UNPROJ_FAST(4, 4); break;
        case 8: LT_UNPROJ_FAST(8, 4); break;
        case 16: LT_UNPROJ_FAST(16, 4); break;
        default: LT_UNPROJ_FAST(32, 4); break;
      }
    }
#undef LT_UNPROJ_FAST
  } else if (vec4) {
    if (stored) unproject_kernel<4, true><<<grid, 256, 0, st>>>(p);
    else unproject_kernel<4, false><<<grid, 256, 0, st>>>(p);
  } else {
    if (stored) unproject_kernel<1, true><<<grid, 256, 0, st>>>(p);
    else unproject_kernel<1, false><<<grid, 256, 0, st>>>(p);
  }
  LT_CHECK_LAUNCH("unproject_kernel");
  return LT_OK;
}

}  // namespace lt

extern "C" int lt_unproject_aggregate_fwd(const float* features, const float* proj, const float* coord, const float* conf,
                                          void* out, int out_format, int B, int V, int C, int h, int w, long nvox,
                                          int agg, void* stream) {
  return lt::launch_unproject(features, proj, coord, conf, out, out_format, B, V, C, h, w, nvox, agg, 0, stream);
}

extern "C" int lt_unproject_partial_fwd(const float* features, const float* proj, const float* coord, const float* conf,
                                        float* partial, int B, int V_local, int C, int h, int w, long nvox, int agg,
                                        void* stream) {
  return lt::launch_unproject(features, proj, coord, conf, partial, LT_FMT_F32, B, V_local, C, h, w, nvox, agg, 1, stream);
}

extern "C" int lt_unproject_push_fwd(const float* features, const float* proj, const float* coord, const float* conf,
                                     float* const* peer_buffers, int n_peers, int src_rank, int B, int V_local, int C, int h,
                                     int w, long nvox, int agg, void* stream) {
  return lt::launch_unproject(features, proj, coord, conf, (void*)peer_buffers[src_rank], LT_FMT_F32, B, V_local, C, h, w, nvox, agg, 2,
                              stream, peer_buffers, n_peers, src_rank);
}

extern "C" int lt_unproject_reduce_finalize_fwd(const float* slots, int nslots, void* out, int out_format, int B, int C, long nvox,
                                                int agg, void* stream) {
  using namespace lt;
  LT_REQUIRE(slots && out && nslots >= 1 && C % 4 == 0, "unproject_reduce_finalize: bad arguments");
  LT_REQUIRE(out_format == LT_FMT_F32 || C % 32 == 0, "unproject_reduce_finalize: split-fp16 output needs C %% 32 == 0");
  const long total4 = (long)B * nvox * C / 4;
  long blocks = (total4 + 255) / 256;
  const long cap = (long)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  unproject_finalize_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(slots, out, out_format, B, C, nvox, agg, nslots);
  LT_CHECK_LAUNCH("unproject_finalize_kernel");
  return LT_OK;
}

extern "C" int lt_unproject_finalize_fwd(const float* partial, void* out, int out_format, int B, int C, long nvox, int agg,
                                         void* stream) {
  using namespace lt;
  LT_REQUIRE(partial && out, "unproject_finalize: null pointer");
  LT_REQUIRE(C % 4 == 0, "unproject_finalize: C %% 4 != 0");
  LT_REQUIRE(out_format == LT_FMT_F32 || C % 32 == 0, "unproject_finalize: split-fp16 output needs C %% 32 == 0");
  const long total4 = (long)B * nvox * C / 4;
  long blocks = (total4 + 255) / 256;
  const long cap = (long)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  unproject_finalize_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(partial, out, out_format, B, C, nvox, agg, 1);
  LT_CHECK_LAUNCH("unproject_finalize_kernel");
  return LT_OK;
}
