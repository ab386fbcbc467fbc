// Volumetric soft-argmax (HBM-bound).
//
// Replaces mvn/utils/op.py:84-96 (integrate_tensor_3d_with_coordinates): softmax over the N^3
// voxels of every (sample, joint) followed by the expectation of the voxel coordinates
// (einsum "bnxyz,bxyzc->bnc"), returning the keypoints and the normalised volumes.
//
// Pass 1 streams the logits once with an online (running max) softmax that carries the three
// coordinate-weighted sums along, warp-reduced per chunk; pass 2 merges the per-chunk partials of
// each (b, j) in one warp; pass 3 (only when the normalised volumes are requested -- the API
// default) re-reads the logits (L2-resident per sample) and writes exp(l - max)/sum in NCDHW,
// transposing channels-last tiles through shared memory so both sides stay coalesced.
//
// Algorithmic bytes per sample (J=17, 64^3): 17.83 MB logits + 3.15 MB coords (+17.83 MB volume
// write) = 20.97 MB keypoints-only / 38.80 MB with volumes.
#include "tc_common.cuh"
#include "softargmax_common.cuh"
#include <stdlib.h>

namespace lt {

constexpr int kChunk = 2048;  // voxels per pass-1 CTA

struct SoftParams {
  const float* logits;
  long bs, vs, cs;        // batch / voxel / channel strides (floats)
  const float* coord;     // [B][nvox][3]
  float* volumes;         // [B][J][nvox] or null
  float* keypoints;       // [B][J][3]
  float* partial;         // [B][J][nch][5]
  float* stats;           // [B][J][2] = (max, sum)
  int B, J, nch;
  long nvox;
  float mult;
  int softmax;
};

// Pass 1, channels-last logits (cs == 1, J <= 32): lane = joint, warps stride over voxels.
__global__ void __launch_bounds__(256) softargmax_partial_cl(const SoftParams p) {
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long v0 = (long)chunk * kChunk;
  const long v1 = min(v0 + kChunk, p.nvox);
  const bool sm = p.softmax == 1;
  const bool active = lane < p.J;
  const float* lg = p.logits + (long)b * p.bs + lane;
  const float* cd = p.coord + (long)b * p.nvox * 3;
  SoftState s;
  st_init(s, sm);
  // 4 voxels in flight per warp iteration
  for (long v = v0 + warp * 4; v < v1; v += 32) {
    float l[4], x[4], y[4], z[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long vv = v + u;
      const bool ok = vv < v1;
      l[u] = (ok && active) ? __ldg(lg + vv * p.vs) : 0.0f;
      x[u] = ok ? __ldg(cd + vv * 3) : 0.0f;
      y[u] = ok ? __ldg(cd + vv * 3 + 1) : 0.0f;
      z[u] = ok ? __ldg(cd + vv * 3 + 2) : 0.0f;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (v + u < v1) st_push(s, l[u] * p.mult, x[u], y[u], z[u], sm);
  }
  __shared__ SoftState sh[8][32];
  sh[warp][lane] = s;
  __syncthreads();
  if (warp == 0 && active) {
    SoftState a = sh[0][lane];
#pragma unroll
    for (int w = 1; w < 8; ++w) st_merge(a, sh[w][lane], sm);
    float* o = p.partial + (((long)b * p.J + lane) * p.nch + chunk) * 5;
    o[0] = a.m; o[1] = a.d; o[2] = a.sx; o[3] = a.sy; o[4] = a.sz;
  }
}

// Pass 1, generic strides: one CTA per (chunk, joint, sample), threads stride over voxels.
__global__ void __launch_bounds__(256) softargmax_partial_generic(const SoftParams p) {
  const int chunk = blockIdx.x, j = blockIdx.y, b = blockIdx.z;
  const long v0 = (long)chunk * kChunk;
  const long v1 = min(v0 + kChunk, p.nvox);
  const bool sm = p.softmax == 1;
  const float* lg = p.logits + (long)b * p.bs + (long)j * p.cs;
  const float* cd = p.coord + (long)b * p.nvox * 3;
  SoftState s;
  st_init(s, sm);
  for (long v = v0 + threadIdx.x; v < v1; v += blockDim.x)
    st_push(s, __ldg(lg + v * p.vs) * p.mult, __ldg(cd + v * 3), __ldg(cd + v * 3 + 1), __ldg(cd + v * 3 + 2), sm);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const SoftState t = st_shfl_xor(s, o); st_merge(s, t, sm); }
  __shared__ SoftState sh[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) sh[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    SoftState a = sh[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) st_merge(a, sh[w], sm);
    float* o = p.partial + (((long)b * p.J + j) * p.nch + chunk) * 5;
    o[0] = a.m; o[1] = a.d; o[2] = a.sx; o[3] = a.sy; o[4] = a.sz;
  }
}

// Pass 2: one warp per (b, j) merges the chunk partials.
__global__ void __launch_bounds__(128) softargmax_finalize(const SoftParams p) {
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= p.B * p.J) return;
  const bool sm = p.softmax == 1;
  SoftState s;
  st_init(s, sm);
  const float* src = p.partial + (long)gw * p.nch * 5;
  for (int c = lane; c < p.nch; c += 32) {
    SoftState t{src[c * 5], src[c * 5 + 1], src[c * 5 + 2], src[c * 5 + 3], src[c * 5 + 4]};
    st_merge(s, t, sm);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const SoftState t = st_shfl_xor(s, o); st_merge(s, t, sm); }
  if (lane == 0) {
    float* k = p.keypoints + (long)gw * 3;
    if (sm || p.softmax == 2) { k[0] = s.sx / s.d; k[1] = s.sy / s.d; k[2] = s.sz / s.d; }   // mode 2: ReLU mass-normalised
    else { k[0] = s.sx; k[1] = s.sy; k[2] = s.sz; }
    p.stats[gw * 2] = s.m;
    p.stats[gw * 2 + 1] = s.d;
  }
}

// Pass 3, channels-last logits: each warp transposes a 32-voxel x 32-channel tile.
__global__ void __launch_bounds__(256) softargmax_normalize_cl(const SoftParams p) {
  __shared__ float tile[8][32][33];
  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool sm = p.softmax == 1;
  const float* st = p.stats + (long)b * p.J * 2;
  for (long v0 = ((long)blockIdx.x * 8 + warp) * 32; v0 < p.nvox; v0 += (long)gridDim.x * 256) {
    const float* lg = p.logits + (long)b * p.bs + lane;
#pragma unroll 8
    for (int r = 0; r < 32; ++r) {
      const long v = v0 + r;
      tile[warp][r][lane] = (v < p.nvox && lane < p.J) ? __ldg(lg + v * p.vs) : 0.0f;
    }
    __syncwarp();
    const long v = v0 + lane;
    if (v < p.nvox) {
      for (int j = 0; j < p.J; ++j) {
        const float l = tile[warp][lane][j] * p.mult;
        const float o = sm ? __expf(l - st[j * 2]) / st[j * 2 + 1] : fmaxf(l, 0.0f);
        p.volumes[((long)b * p.J + j) * p.nvox + v] = o;
      }
    }
    __syncwarp();
  }
}

__global__ void __launch_bounds__(256) softargmax_normalize_generic(const SoftParams p) {
  const int j = blockIdx.y, b = blockIdx.z;
  const bool sm = p.softmax == 1;
  const float mx = p.stats[((long)b * p.J + j) * 2], dn = p.stats[((long)b * p.J + j) * 2 + 1];
  const float* lg = p.logits + (long)b * p.bs + (long)j * p.cs;
  float* o = p.volumes + ((long)b * p.J + j) * p.nvox;
  for (long v = (long)blockIdx.x * blockDim.x + threadIdx.x; v < p.nvox; v += (long)gridDim.x * blockDim.x) {
    const float l = __ldg(lg + v * p.vs) * p.mult;
    o[v] = sm ? __expf(l - mx) / dn : fmaxf(l, 0.0f);
  }
}


// ------------------------------------------------------------------------------------------------
// Streaming path (channels-last logits with a compact voxel stride: vs % 4 == 0, 20 <= vs <= 32, J <= vs).
//
// Two persistent kernels + a tiny merge, each CTA owning the flat tiles f = g, g + G, ... of the whole batch
// (f -> sample f / tiles, tile f % tiles; ~35 tiles per CTA, balanced to 1 %).  In both kernels a producer warp
// streams 16 KB logit tiles (stats pass: + the matching coordinate rows) into a 4-stage shared-memory ring with 1-D
// TMA bulk copies (cp.async.bulk -> mbarrier complete_tx): up to 128 KB of reads in flight per SM, no register staging.
//
//   stream_stats_kernel      8 consumer warps read the tile as a flat float4 array (conflict-free: thread = (row, 4-joint
//                            chunk)) and fold 4 rows x 4 joints per step into an online-softmax state (one rescale + four
//                            ex2 per joint per step); per (sample, CTA) partials -> global memory.
//   softargmax_stream_merge  one warp per (sample, joint): merges the G partials -> keypoints, (max, 1/sum).
//   stream_normalize_kernel  same ring, samples in REVERSE order (the tail of the stats pass is still in the 126 MB L2);
//                            a warp reads 8 rows x 4 joints per instruction (bank-conflict free for 80- and 112-byte rows) and
//                            writes exp(l - max) / sum in NCDHW as four full 32-byte sectors (streaming stores).
// ------------------------------------------------------------------------------------------------
constexpr int kStreamConsumers = 256;
constexpr int kStreamThreads = kStreamConsumers + 32;   // + producer warp
constexpr int kStreamStages = 4;
constexpr int kStreamLogitBytes = 16384;
constexpr int kStreamCoordBytes = 2560;
constexpr int kStreamStageBytes = kStreamLogitBytes + kStreamCoordBytes;
constexpr int kStreamScratchBytes = 20480;             // CTA merge scratch [256][20] floats (stats kernel)
constexpr int kStreamSmemBytes = kStreamStages * kStreamStageBytes + kStreamScratchBytes + 128 + 128;
constexpr int kMaxStreamCtas = 640;
constexpr int kMaxPartials = 1024;      // partial slots per sample the workspace is sized for (fused tail: 3 CTAs per SM)

struct StreamParams {
  const float* logits;    // [B][nvox][vs]
  const float* coord;     // [B][nvox][3]
  float* volumes;         // [B][J][nvox]
  float* keypoints;       // [B][J][3]
  float* partial;         // [B][G][J][5]
  float* stats;           // [B][J][2] = (max, 1 / sum)
  long bs, nvox, total_tiles;
  int vs, B, J, Q, RPI, T, tiles, G;
  float mult;
  int softmax;
};

__device__ __forceinline__ void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
// producer warp: stream the CTA's tiles in order; reverse = samples from last to first
__device__ __forceinline__ void stream_producer(const StreamParams& p, uint8_t* smem, uint64_t* full, uint64_t* empty, bool with_coord,
                                                bool reverse) {
  const int lane = threadIdx.x & 31;
  uint32_t it = 0;
  const unsigned total = (unsigned)p.total_tiles, tiles = (unsigned)p.tiles;
  for (unsigned f = blockIdx.x; f < total; f += gridDim.x, ++it) {
    const uint32_t s = it % kStreamStages;
    mbar_wait(&empty[s], ((it / kStreamStages) & 1u) ^ 1u);
    if (lane == 0) {
      int b = (int)(f / tiles);
      const int t = (int)(f - (unsigned)b * tiles);
      if (reverse) b = p.B - 1 - b;
      const long v0 = (long)t * p.T;
      const int rows = (int)min((long)p.T, p.nvox - v0);
      const uint32_t lb = (uint32_t)rows * (uint32_t)p.vs * 4u, cb = with_coord ? (uint32_t)rows * 12u : 0u;
      uint8_t* dst = smem + (size_t)s * kStreamStageBytes;
      mbar_expect_tx(&full[s], lb + cb);
      bulk_load_1d(dst, p.logits + (long)b * p.bs + v0 * p.vs, lb, &full[s]);
      if (with_coord) bulk_load_1d(dst + kStreamLogitBytes, p.coord + ((long)b * p.nvox + v0) * 3, cb, &full[s]);
    }
    __syncwarp();
  }
}

template <bool SM>
__global__ void __launch_bounds__(kStreamThreads, 2) stream_stats_kernel(const StreamParams p) {
  extern __shared__ uint8_t fsm_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(fsm_raw) + 127) & ~(uintptr_t)127);
  float* scratch = reinterpret_cast<float*>(smem + kStreamStages * kStreamStageBytes);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStreamStages * kStreamStageBytes + kStreamScratchBytes);
  uint64_t* empty = full + kStreamStages;
  const int g = blockIdx.x, G = gridDim.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStreamStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kStreamConsumers / 32); }
    fence_barrier_init();
  }
  __syncthreads();
  if (warp == kStreamConsumers / 32) { stream_producer(p, smem, full, empty, true, false); return; }

  const int tid = threadIdx.x;
  const int row_l = tid / p.Q, c = tid % p.Q;
  const bool active = (tid < p.RPI * p.Q) && (4 * c < p.J);
  SoftState st[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) st_init(st[i], SM);

  // samples in which this CTA owns no tile still need an (identity) partial for the merge
  for (int i = tid; i < p.B * p.J; i += kStreamConsumers) {
    const int b = i / p.J, j = i % p.J;
    const long lo = (long)b * p.tiles;
    const long f0 = lo + (((long)g - lo) % G + G) % G;     // first flat tile >= lo owned by this CTA
    if (!(f0 < lo + p.tiles)) {
      float* dst = p.partial + (((long)b * G + g) * p.J + j) * 5;
      dst[0] = SM ? -INFINITY : 0.0f; dst[1] = 0.f; dst[2] = 0.f; dst[3] = 0.f; dst[4] = 0.f;
    }
  }

  auto flush = [&](int b) {   // CTA merge of the per-thread states -> partial[b][g][*], then reset
    consumer_bar();
    float* my = scratch + tid * 20;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      SoftState z;
      st_init(z, SM);
      const SoftState& a = active ? st[i] : z;
      my[i * 5] = a.m; my[i * 5 + 1] = a.d; my[i * 5 + 2] = a.sx; my[i * 5 + 3] = a.sy; my[i * 5 + 4] = a.sz;
      st_init(st[i], SM);
    }
    consumer_bar();
    for (int j = warp; j < p.J; j += kStreamConsumers / 32) {
      const int cj = j >> 2, ij = j & 3;
      SoftState a;
      st_init(a, SM);
      for (int r = lane; r < p.RPI; r += 32) {
        const float* src = scratch + (r * p.Q + cj) * 20 + ij * 5;
        SoftState t{src[0], src[1], src[2], src[3], src[4]};
        st_merge(a, t, SM);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) { const SoftState t = st_shfl_xor(a, o); st_merge(a, t, SM); }
      if (lane == 0) {
        float* dst = p.partial + (((long)b * G + g) * p.J + j) * 5;
        dst[0] = a.m; dst[1] = a.d; dst[2] = a.sx; dst[3] = a.sy; dst[4] = a.sz;
      }
    }
  };

  uint32_t it = 0;
  int cur_b = -1;
  const unsigned total = (unsigned)p.total_tiles, tiles = (unsigned)p.tiles;
  for (unsigned f = g; f < total; f += G, ++it) {
    const int b = (int)(f / tiles), t = (int)(f - (unsigned)b * tiles);
    if (b != cur_b) {
      if (cur_b >= 0) flush(cur_b);
      cur_b = b;
    }
    const uint32_t s = it % kStreamStages;
    const int rows = (int)min((long)p.T, p.nvox - (long)t * p.T);
    mbar_wait(&full[s], (it / kStreamStages) & 1u);
    const uint32_t lbase = smem_u32(smem + (size_t)s * kStreamStageBytes);
    const float* cd = reinterpret_cast<const float*>(smem + (size_t)s * kStreamStageBytes + kStreamLogitBytes);
    if (active) {
      float l[4][4], x[4], y[4], z[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int row = k * p.RPI + row_l;
        if (row < rows) {
          const uint4 q = lds128(lbase + (uint32_t)(row * p.Q + c) * 16u);
          l[0][k] = __uint_as_float(q.x) * p.mult; l[1][k] = __uint_as_float(q.y) * p.mult;
          l[2][k] = __uint_as_float(q.z) * p.mult; l[3][k] = __uint_as_float(q.w) * p.mult;
          x[k] = cd[row * 3]; y[k] = cd[row * 3 + 1]; z[k] = cd[row * 3 + 2];
        } else {   // rows past the end of a sample's last tile: no weight, finite coordinates
          l[0][k] = l[1][k] = l[2][k] = l[3][k] = SM ? -INFINITY : 0.0f;
          x[k] = y[k] = z[k] = 0.0f;
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) st_push4<SM>(st[i], l[i], x, y, z);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive_local(&empty[s]);
  }
  if (cur_b >= 0) flush(cur_b);
}

// one warp per (sample, joint): merge the G partials -> keypoints, (max, 1 / sum)
__global__ void __launch_bounds__(128) softargmax_stream_merge(const StreamParams p) {
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= p.B * p.J) return;
  const int b = gw / p.J, j = gw % p.J;
  const bool sm = p.softmax == 1;
  SoftState a;
  st_init(a, sm);
  for (int gg = lane; gg < p.G; gg += 32) {
    const float* src = p.partial + (((long)b * p.G + gg) * p.J + j) * 5;
    SoftState t{src[0], src[1], src[2], src[3], src[4]};
    st_merge(a, t, sm);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const SoftState t = st_shfl_xor(a, o); st_merge(a, t, sm); }
  if (lane == 0) {
    float* k = p.keypoints + (long)gw * 3;
    if (sm) { k[0] = a.sx / a.d; k[1] = a.sy / a.d; k[2] = a.sz / a.d; }
    else { k[0] = a.sx; k[1] = a.sy; k[2] = a.sz; }
    p.stats[gw * 2] = a.m;
    p.stats[gw * 2 + 1] = 1.0f / a.d;
  }
}

template <bool SM>
__global__ void __launch_bounds__(kStreamThreads, 2) stream_normalize_kernel(const StreamParams p) {
  extern __shared__ uint8_t fsm_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(fsm_raw) + 127) & ~(uintptr_t)127);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStreamStages * kStreamStageBytes + kStreamScratchBytes);
  uint64_t* empty = full + kStreamStages;
  const int g = blockIdx.x, G = gridDim.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStreamStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kStreamConsumers / 32); }
    fence_barrier_init();
  }
  __syncthreads();
  if (warp == kStreamConsumers / 32) { stream_producer(p, smem, full, empty, false, true); return; }

  // lane = (row within an 8-row group, joint within a 4-joint group): one LDS covers 8 rows x 4 joints -- 32 distinct banks
  // for a row stride of 20 or 28 words (the compact 17/21..28-joint layouts) --, one STG writes four aligned 32-byte sectors (T and the tile origins are multiples of 8 rows)
  const int ji = lane & 3, rr = lane >> 2;
  const int jgroups = (p.J + 3) >> 2;
  uint32_t it = 0;
  const unsigned total = (unsigned)p.total_tiles, tiles = (unsigned)p.tiles;
  for (unsigned f = g; f < total; f += G, ++it) {
    const int bf = (int)(f / tiles), t = (int)(f - (unsigned)bf * tiles);
    const int b = p.B - 1 - bf;
    const uint32_t s = it % kStreamStages;
    const long v0 = (long)t * p.T;
    const int rows = (int)min((long)p.T, p.nvox - v0);
    const int rgroups = (rows + 7) >> 3;
    mbar_wait(&full[s], (it / kStreamStages) & 1u);
    const float* tile = reinterpret_cast<const float*>(smem + (size_t)s * kStreamStageBytes);
    for (int jg = 0; jg < jgroups; ++jg) {
      const int j = jg * 4 + ji;
      const bool jok = j < p.J;
      const float2 ms = jok ? __ldg(reinterpret_cast<const float2*>(p.stats + ((long)b * p.J + j) * 2)) : make_float2(0.f, 0.f);
      float* dst = p.volumes + ((long)b * p.J + (jok ? j : 0)) * p.nvox + v0;
      for (int rg = warp; rg < rgroups; rg += kStreamConsumers / 32) {
        const int r = rg * 8 + rr;
        if (jok && r < rows) {
          const float v = tile[r * p.vs + j] * p.mult;          // same rounding as the statistics pass
          const float o = SM ? ex2f((v - ms.x) * kLog2e) * ms.y : fmaxf(v, 0.0f);   // l - max first, as in st_push4
          __stcs(dst + r, o);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive_local(&empty[s]);
  }
}

static bool stream_shape_ok(const float* logits, long batch_stride, long voxel_stride, const float* coord, const float* volumes_out, int J,
                            long nvox) {
  return stream_layout_ok(voxel_stride, J, nvox) && batch_stride % 4 == 0 && ((uintptr_t)logits & 15) == 0 && ((uintptr_t)coord & 15) == 0 &&
         (!volumes_out || ((uintptr_t)volumes_out & 31) == 0);
}

// tile geometry of the streaming kernels for one problem (everything but the partial / stats pointers and G)
static int stream_setup(StreamParams& f, const float* logits, long batch_stride, int vs, const float* coord, float* volumes_out, float* keypoints_out,
                        int B, int J, long nvox, float multiplier, int softmax) {
  f.logits = logits; f.coord = coord; f.volumes = volumes_out; f.keypoints = keypoints_out;
  f.bs = batch_stride; f.nvox = nvox; f.vs = vs; f.B = B; f.J = J;
  f.Q = f.vs / 4;
  f.RPI = (kStreamConsumers / f.Q) & ~1;      // rows per pass, even -> T = 4 * RPI is a multiple of 8 rows
  f.T = 4 * f.RPI;
  f.tiles = (int)((nvox + f.T - 1) / f.T);
  f.total_tiles = (long)f.tiles * B;
  f.mult = multiplier; f.softmax = softmax;
  LT_REQUIRE(f.T * f.vs * 4 <= kStreamLogitBytes && f.T * 12 <= kStreamCoordBytes, "softargmax stream: tile does not fit (vs=%d)", f.vs);
  LT_REQUIRE(f.total_tiles < (1L << 31), "softargmax stream: too many tiles");
  static DeviceOnce configured;
  if (configured.first()) {
    cudaError_t e = cudaFuncSetAttribute(stream_stats_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kStreamSmemBytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(stream_stats_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kStreamSmemBytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(stream_normalize_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kStreamSmemBytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(stream_normalize_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kStreamSmemBytes);
    if (e != cudaSuccess) return fail(LT_ERR_CUDA, "softargmax stream: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  }
  return LT_OK;
}

// merge of the f.G partials per (sample, joint) -> key points, (max, 1 / sum); then the normalisation pass (if volumes are requested)
static int stream_finish(const StreamParams& f, cudaStream_t st) {
  softargmax_stream_merge<<<ceil_div((long)f.B * f.J * 32, 128), 128, 0, st>>>(f);
  LT_CHECK_LAUNCH("softargmax_stream_merge");
  if (f.volumes) {
    int G = 2 * sm_count();
    if (G > kMaxStreamCtas) G = kMaxStreamCtas;
    if ((long)G > f.total_tiles) G = (int)f.total_tiles;
    if (f.softmax) stream_normalize_kernel<true><<<G, kStreamThreads, kStreamSmemBytes, st>>>(f);
    else stream_normalize_kernel<false><<<G, kStreamThreads, kStreamSmemBytes, st>>>(f);
    LT_CHECK_LAUNCH("stream_normalize_kernel");
  }
  return LT_OK;
}

static inline int n_chunks(long nvox) { return (int)((nvox + kChunk - 1) / kChunk); }

}  // namespace lt

extern "C" size_t lt_softargmax3d_workspace_bytes(int B, int J, long nvox) {
  const size_t classic = (size_t)B * J * ((size_t)lt::n_chunks(nvox) * 5 + 2) * sizeof(float);
  // streaming path: partial [B][G <= kMaxStreamCtas][J][5] + stats [B][J][2]
  const size_t stream = (size_t)B * ((size_t)lt::kMaxPartials * J * 5 + (size_t)J * 2) * sizeof(float) + 64;
  return classic > stream ? classic : stream;
}

extern "C" int lt_softargmax3d_fwd(const float* logits, long batch_stride, long voxel_stride, long chan_stride,
                                   const float* coord, float* volumes_out, float* keypoints_out, void* workspace,
                                   size_t workspace_bytes, int B, int J, long nvox, float multiplier, int softmax,
                                   void* stream) {
  using namespace lt;
  LT_REQUIRE(logits && coord && keypoints_out && workspace, "softargmax3d: null pointer");
  LT_REQUIRE(B > 0 && J > 0 && nvox > 0, "softargmax3d: non-positive size");
  LT_REQUIRE(B <= 65535 && J <= 65535, "softargmax3d: B/J too large");
  LT_REQUIRE(workspace_bytes >= lt_softargmax3d_workspace_bytes(B, J, nvox), "softargmax3d: workspace too small");
  SoftParams p;
  p.logits = logits; p.bs = batch_stride; p.vs = voxel_stride; p.cs = chan_stride;
  p.coord = coord; p.volumes = volumes_out; p.keypoints = keypoints_out;
  p.nch = n_chunks(nvox);
  p.partial = reinterpret_cast<float*>(workspace);
  p.stats = p.partial + (size_t)B * J * p.nch * 5;
  p.B = B; p.J = J; p.nvox = nvox; p.mult = multiplier; p.softmax = softmax;
  cudaStream_t st = (cudaStream_t)stream;
  const bool cl = (chan_stride == 1 && J <= 32 && voxel_stride >= J);
  LT_REQUIRE(softmax >= 0 && softmax <= 2, "softargmax3d: mode must be 0 (ReLU), 1 (softmax) or 2 (ReLU, mass-normalised coordinates)");
  // ---- streaming path ----
  const int stream_mode = opts().softargmax_stream;
  if (stream_mode && softmax != 2 && cl && stream_shape_ok(logits, batch_stride, voxel_stride, coord, volumes_out, J, nvox)) {
    StreamParams f;
    int rc = stream_setup(f, logits, batch_stride, (int)voxel_stride, coord, volumes_out, keypoints_out, B, J, nvox, multiplier, softmax);
    if (rc) return rc;
    int max_ctas = 2 * sm_count();
    if (max_ctas > kMaxStreamCtas) max_ctas = kMaxStreamCtas;
    const int G = f.total_tiles < max_ctas ? (int)f.total_tiles : max_ctas;
    f.G = G;
    float* w = reinterpret_cast<float*>(workspace);
    f.partial = w;
    f.stats = w + stream_stats_offset(B, G, J);
    if (softmax) stream_stats_kernel<true><<<G, kStreamThreads, kStreamSmemBytes, st>>>(f);
    else stream_stats_kernel<false><<<G, kStreamThreads, kStreamSmemBytes, st>>>(f);
    LT_CHECK_LAUNCH("stream_stats_kernel");
    return stream_finish(f, st);
  }
  if (cl) softargmax_partial_cl<<<dim3(p.nch, B), 256, 0, st>>>(p);
  else softargmax_partial_generic<<<dim3(p.nch, J, B), 256, 0, st>>>(p);
  LT_CHECK_LAUNCH("softargmax_partial");
  softargmax_finalize<<<ceil_div((long)B * J * 32, 128), 128, 0, st>>>(p);
  LT_CHECK_LAUNCH("softargmax_finalize");
  if (volumes_out) {
    if (cl) {
      long blocks = (nvox + 255) / 256;
      const long cap = (long)sm_count() * 8;
      if (blocks > cap) blocks = cap;
      softargmax_normalize_cl<<<dim3((unsigned)blocks, B), 256, 0, st>>>(p);
    } else {
      long blocks = (nvox + 255) / 256;
      if (blocks > 1024) blocks = 1024;
      softargmax_normalize_generic<<<dim3((unsigned)blocks, J, B), 256, 0, st>>>(p);
    }
    LT_CHECK_LAUNCH("softargmax_normalize");
  }
  return LT_OK;
}

// Second half of the streaming soft-argmax for logits whose statistics pass ran inside the kernel that produced them
// (lt_v2v_tail_stats_fwd): workspace holds partial [B][G][J][5]; merges them -> key points, then writes the normalised volumes.
extern "C" int lt_softargmax3d_finish_fwd(const float* logits, long batch_stride, long voxel_stride, const float* coord, float* volumes_out,
                                          float* keypoints_out, void* workspace, size_t workspace_bytes, int B, int J, long nvox, int G,
                                          float multiplier, int softmax, void* stream) {
  using namespace lt;
  LT_REQUIRE(logits && coord && keypoints_out && workspace, "softargmax3d_finish: null pointer");
  LT_REQUIRE(B > 0 && J > 0 && nvox > 0 && G > 0 && G <= kMaxPartials, "softargmax3d_finish: bad sizes (G=%d)", G);
  LT_REQUIRE(softmax == 0 || softmax == 1, "softargmax3d_finish: mode must be 0 (ReLU) or 1 (softmax)");
  LT_REQUIRE(workspace_bytes >= lt_softargmax3d_workspace_bytes(B, J, nvox), "softargmax3d_finish: workspace too small");
  LT_REQUIRE(stream_shape_ok(logits, batch_stride, voxel_stride, coord, volumes_out, J, nvox), "softargmax3d_finish: logits layout not covered by the streaming kernels");
  StreamParams f;
  int rc = stream_setup(f, logits, batch_stride, (int)voxel_stride, coord, volumes_out, keypoints_out, B, J, nvox, multiplier, softmax);
  if (rc) return rc;
  f.G = G;
  float* w = reinterpret_cast<float*>(workspace);
  f.partial = w;
  f.stats = w + stream_stats_offset(B, G, J);
  return stream_finish(f, (cudaStream_t)stream);
}
