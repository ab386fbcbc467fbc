// Online-softmax state of the volumetric soft-argmax (op.py:84-96), shared by the streaming kernels (softargmax.cu) and the fused V2V
// tail (conv_tail.cu: the statistics pass runs in the epilogue that produces the logits).
#pragma once
#include "common.cuh"

namespace lt {

constexpr float kLog2e = 1.4426950408889634f;

struct SoftState {
  float m, d, sx, sy, sz;
};

__device__ __forceinline__ void st_init(SoftState& s, bool softmax) {
  s.m = softmax ? -INFINITY : 0.0f;
  s.d = s.sx = s.sy = s.sz = 0.0f;
}
// add one element with logit l and coordinate (x, y, z)
__device__ __forceinline__ void st_push(SoftState& s, float l, float x, float y, float z, bool softmax) {
  if (softmax) {
    const float mn = fmaxf(s.m, l);
    const float r = __expf(s.m - mn);   // rescale of the running sums (exp(-inf) = 0 on first element)
    const float e = __expf(l - mn);
    s.d = fmaf(s.d, r, e);
    s.sx = fmaf(s.sx, r, e * x);
    s.sy = fmaf(s.sy, r, e * y);
    s.sz = fmaf(s.sz, r, e * z);
    s.m = mn;
  } else {
    const float e = fmaxf(l, 0.0f);     // op.py:90-91: ReLU, no normalisation (d = mass, only used by mode 2, op.py:25-41)
    s.d += e;
    s.sx = fmaf(e, x, s.sx);
    s.sy = fmaf(e, y, s.sy);
    s.sz = fmaf(e, z, s.sz);
  }
}
__device__ __forceinline__ void st_merge(SoftState& a, const SoftState& b, bool softmax) {
  if (softmax) {
    const float mn = fmaxf(a.m, b.m);
    const float ra = (a.m == -INFINITY) ? 0.0f : __expf(a.m - mn);
    const float rb = (b.m == -INFINITY) ? 0.0f : __expf(b.m - mn);
    a.d = a.d * ra + b.d * rb;
    a.sx = a.sx * ra + b.sx * rb;
    a.sy = a.sy * ra + b.sy * rb;
    a.sz = a.sz * ra + b.sz * rb;
    a.m = mn;
  } else {
    a.d += b.d; a.sx += b.sx; a.sy += b.sy; a.sz += b.sz;
  }
}
__device__ __forceinline__ SoftState st_shfl_xor(const SoftState& s, int o) {
  SoftState r;
  r.m = __shfl_xor_sync(0xffffffffu, s.m, o);
  r.d = __shfl_xor_sync(0xffffffffu, s.d, o);
  r.sx = __shfl_xor_sync(0xffffffffu, s.sx, o);
  r.sy = __shfl_xor_sync(0xffffffffu, s.sy, o);
  r.sz = __shfl_xor_sync(0xffffffffu, s.sz, o);
  return r;
}

__device__ __forceinline__ float ex2f(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// fold four (logit, coordinate) pairs into one online-softmax state: one rescale + four exponentials.  The exponents are formed as
// (l - m) * log2(e), not as fma(l, log2(e), -m * log2(e)): the rounding of m * log2(e) grows with |m| and differs between running
// maxima, which put up to ~2e-8 x |m| of relative error into the weights (4e-5 of scale at |m| = 1024); l - m is exact for the logits
// that matter (Sterbenz), so the weights are as accurate at any offset as at m = 0.
template <bool SM>
__device__ __forceinline__ void st_push4(SoftState& s, const float (&l)[4], const float (&x)[4], const float (&y)[4], const float (&z)[4]) {
  if (SM) {
    const float mn = fmaxf(fmaxf(fmaxf(l[0], l[1]), fmaxf(l[2], l[3])), s.m);
    if (mn == -INFINITY) return;                 // nothing but padding so far
    const float r = ex2f((s.m - mn) * kLog2e);   // exp(m_old - m_new); 0 for the first batch (m_old = -inf)
    const float e0 = ex2f((l[0] - mn) * kLog2e), e1 = ex2f((l[1] - mn) * kLog2e);
    const float e2 = ex2f((l[2] - mn) * kLog2e), e3 = ex2f((l[3] - mn) * kLog2e);
    s.d = fmaf(s.d, r, (e0 + e1) + (e2 + e3));
    s.sx = fmaf(s.sx, r, fmaf(e0, x[0], fmaf(e1, x[1], fmaf(e2, x[2], e3 * x[3]))));
    s.sy = fmaf(s.sy, r, fmaf(e0, y[0], fmaf(e1, y[1], fmaf(e2, y[2], e3 * y[3]))));
    s.sz = fmaf(s.sz, r, fmaf(e0, z[0], fmaf(e1, z[1], fmaf(e2, z[2], e3 * z[3]))));
    s.m = mn;
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float e = fmaxf(l[k], 0.0f);         // op.py:90-91: ReLU, no normalisation
      s.sx = fmaf(e, x[k], s.sx); s.sy = fmaf(e, y[k], s.sy); s.sz = fmaf(e, z[k], s.sz);
    }
  }
}


// Logits layout the streaming kernels read (softargmax.cu): channels-last rows of vs floats with vs % 4 == 0, 20 <= vs <= 32 and
// J <= vs, nvox % 8 == 0 and at least kStreamMinVoxels voxels.  lt_softargmax3d_fwd streams such logits (given aligned pointers),
// lt_softargmax3d_finish_fwd accepts only them, and lt_v2v_tail_stats_fwd produces partials only for them, so every set of fused
// partials can be merged.  engine.NativeEngine.v2v mirrors this test (_stream_layout_ok) when it decides to fuse.
constexpr long kStreamMinVoxels = 16384;
__host__ __device__ inline bool stream_layout_ok(long vs, int J, long nvox) {
  return vs % 4 == 0 && vs >= 20 && vs <= 32 && J <= vs && nvox % 8 == 0 && nvox >= kStreamMinVoxels;
}

// Workspace layout shared by lt_softargmax3d_fwd (streaming path), lt_v2v_tail_stats_fwd and lt_softargmax3d_finish_fwd:
// partial [B][G][J][5] floats, then (16-byte aligned) stats [B][J][2] = (max, 1 / sum)
__host__ __device__ inline size_t stream_stats_offset(int B, int G, int J) { return ((size_t)B * G * J * 5 + 3) & ~(size_t)3; }

}  // namespace lt
