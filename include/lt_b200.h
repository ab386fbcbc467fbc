/*
 * lt_b200.h -- C ABI of liblt_b200.so: the H100 (sm_90a) kernels behind the volumetric
 * triangulation hot path of karfly/learnable-triangulation-pytorch.
 *
 * The reference is 100% Python/PyTorch: it has no FFI for this path.  Each entry point
 * below replaces the PyTorch library calls of one reference call site (cited per function);
 * the Python host code in learnable-triangulation-pytorch_b200/ binds them with ctypes and
 * INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless said otherwise;
 *   - the caller owns all memory (incl. workspaces); nothing here allocates device memory;
 *   - every launch goes to `stream` (a cudaStream_t passed as void*), nothing synchronises;
 *   - return value: 0 on success, negative lt_status on failure; lt_last_error_string()
 *     returns a thread-local description of the last failure;
 *   - activation tensors are channels-last: [N][D][H][W][C] (2-D maps have D = 1);
 *   - LT_FMT_F32 is plain float; LT_FMT_S32 is "split-fp16": channels in blocks of 32, each
 *     block stored as 32 fp16 high parts followed by 32 fp16 low parts (x = hi + lo/2048, 128
 *     bytes per block, same footprint as fp32, ~22 significand bits) -- the tensor-core operand
 *     format (see DESIGN.md).
 */
#ifndef LT_B200_H
#define LT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum lt_status {
  LT_OK = 0,
  LT_ERR_INVALID = -1,     /* bad argument */
  LT_ERR_CUDA = -2,        /* CUDA runtime/driver error at launch */
  LT_ERR_UNSUPPORTED = -3  /* shape/format combination not implemented */
};

enum lt_format { LT_FMT_F32 = 0, LT_FMT_S32 = 1 };

/* view aggregation of the unprojection, reference mvn/utils/op.py:150-164 */
enum lt_agg { LT_AGG_SUM = 0, LT_AGG_MAX = 1, LT_AGG_SOFTMAX = 2, LT_AGG_CONF = 3 };

/* conv implementation selector */
enum lt_conv_impl {
  LT_CONV_SIMT = 0, /* fp32 FFMA implicit GEMM (exact, any shape) */
  LT_CONV_TC = 1,   /* wgmma, split-fp16 3-term products (fp32-grade) */
  LT_CONV_TC1 = 2,  /* wgmma, high parts only (plain fp16 precision, fast mode) */
  LT_CONV_TC_FOLD = 3, /* wgmma, 3-term products, one input halo box per pipeline stage serving all kh (and kd) taps of a kw
                         (Cin = 32 cubic 3^3 / 7^3 stride-1 "same" layers; weights from lt_conv_fold_pack_weights; desc->Cout = real
                         channel count <= 32, N tile round_up(Cout, 16), FC = 32 with channels Cout .. 31 written as zeros) */
};

/* residual placement in the conv epilogue */
enum lt_residual { LT_RES_NONE = 0, LT_RES_BEFORE_RELU = 1, LT_RES_AFTER_RELU = 2 };

/* Kernel-selection options: the ONLY mutable process-wide state of the library besides its caches (encoded tensor maps,
 * per-device function attributes).  Set once before launching (lt_set_options is not synchronised against concurrent launches);
 * no entry point reads the environment. */
typedef struct lt_options {
  /* sm_90a: the variants of the first (tensor-memory) kernels that these fields selected are one wgmma kernel; the fields
     marked "no effect" are kept for ABI compatibility and ignored */
  int tc_persist;          /* no effect */
  int tc_splitk;           /* conv_tc: split the K loop where the launch model says it pays (lt_conv_tc_plan; default 1) */
  int tc_bres;             /* no effect */
  int tc_direct_epilogue;  /* no effect */
  int fold_fast_issue;     /* no effect */
  int fold_debug;          /* no effect */
  int softargmax_stream;   /* soft-argmax: streaming TMA kernels for compact channels-last logits (default 1) */
  int unproject_v2;        /* unprojection: production-shape kernel (default 1) */
  int unproject_cpl;       /* unprojection v2: channels per lane, 4 (default) or 8 */
  int unproject_lb;        /* unprojection v2: min CTAs / SM override (0 = per-variant default) */
  int unproject_brick;     /* unprojection v2: side of the voxel bricks a CTA walks (0 = linear order, default) */
  int unproject_brick_order; /* voxel order inside a brick: 0 = z fastest, 1 = x fastest, 2 = 2 x 2 (x, y) tiles (voxels of a warp share taps) */
  int pair_nt, pair_stages; /* no effect */
  int pair_prof;           /* no effect */
  int pair_direct_out;     /* no effect */
  int pair_two_acc;        /* no effect: the hi*lo + lo*hi products always accumulate in their own accumulator */
  int fold_pair;           /* no effect */
  int fold_direct;         /* no effect */
  int fold_fullw;          /* no effect */
} lt_options;
void lt_default_options(lt_options* o);
int lt_get_options(lt_options* o);
int lt_set_options(const lt_options* o);

int lt_version(void);
const char* lt_last_error_string(void);

/* Number of SMs / compute capability of the current device (host-side query; -1 if no device). */
int lt_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ------------------------------------------------------------------------------------------
 * Coordinate volume.  Replaces triangulation.py:306-341 (meshgrid, affine to mm, rotation
 * about the base point, optional CMU->H36M axis transfer), all samples in one launch.
 *   position[B*3], center[B*3] : float32 casts of (base - side/2) and base
 *   step[3]                    : float32 cast of side / (n - 1)
 *   rot[B*9]                   : float32 row-major rotation per sample (identity in eval)
 *   out[B][n][n][n][3]
 * ---------------------------------------------------------------------------------------- */
int lt_coord_volume_fwd(const float* position, const float* center, const float* step, const float* rot,
                        float* out, int B, int n, int transfer_cmu, void* stream);

/* ------------------------------------------------------------------------------------------
 * Cuboid placement from predicted key points (TwoStageTriangulationNet).  Replaces the host
 * hand-off of the reference's two-stage protocol: the algebraic model's evaluation writes
 * results.pkl, the volumetric run reloads it as batch['pred_keypoints_3d'] (pred_results_path)
 * and places each cuboid around its pelvis on the host, triangulation.py:284-296.
 *   keypoints_3d[B][J][3] : float32 key points (the algebraic model's output)
 *   kind                  : LT_KIND_MPII (joint 6, J >= 7) or LT_KIND_COCO (mean of joints 11
 *                           and 12, J >= 13)
 *   center[B][3]          : the base point, float32; the coco mean is the float32 sum halved in
 *                           float32, as numpy computes it on the float32 array
 *   position[B][3]        : float32((double)center - cuboid_side / 2), formed in float64
 * No FMA contraction: the values equal what the host path uploads for the same key points bit
 * for bit.  It writes the buffers lt_coord_volume_fwd reads.  A few threads per batch, not a hot
 * path: what it saves is the device-to-host copy and synchronisation between the two stages.
 * ---------------------------------------------------------------------------------------- */
enum lt_skeleton_kind { LT_KIND_MPII = 0, LT_KIND_COCO = 1 };
int lt_cuboid_from_keypoints_fwd(const float* keypoints_3d, int B, int J, int kind, double cuboid_side, float* center,
                                 float* position, void* stream);

/* ------------------------------------------------------------------------------------------
 * Fused unprojection + view aggregation.  Replaces op.unproject_heatmaps (op.py:99-166):
 * per voxel, per view: project with proj (3x4), depth mask, bilinear sample of the feature map
 * (grid_sample align_corners=True, zero padding, incl. the reference's x/H, y/W normalisation
 * quirk op.py:128-129), then aggregate across views in registers.
 *   features [B][V][h][w][C] channels-last float32
 *   proj     [B][V][3][4]
 *   coord    [B][nvox][3]
 *   conf     [B][V][C] (LT_AGG_CONF) or NULL
 *   out      [B][nvox][C] in out_format (LT_FMT_S32 needs C % 32 == 0)
 * ---------------------------------------------------------------------------------------- */
int lt_unproject_aggregate_fwd(const float* features, const float* proj, const float* coord, const float* conf,
                               void* out, int out_format, int B, int V, int C, int h, int w, long nvox,
                               int agg, void* stream);

/* View-sharded variant (multi-GPU): this rank holds V_local views.  Writes float32 partials
 *   LT_AGG_SOFTMAX: partial[B][2][nvox][C] = (sum_v s*exp(s), sum_v exp(s))   (unshifted)
 *   LT_AGG_SUM/CONF: partial[B][1][nvox][C] = sum_v s (*conf);  LT_AGG_MAX: max_v s
 * which one all-reduce (sum / max) over ranks completes; lt_unproject_finalize_fwd then divides
 * (softmax) and converts to out_format.
 * Known limit of the unshifted softmax partials: exp(s) overflows above s ~ 88, and the result is 0/0 when every view's
 * sample is below ~ -87 (fast kernel: __expf flushes to zero) or ~ -104 (generic kernel). */
int lt_unproject_partial_fwd(const float* features, const float* proj, const float* coord, const float* conf,
                             float* partial, int B, int V_local, int C, int h, int w, long nvox,
                             int agg, void* stream);
int lt_unproject_finalize_fwd(const float* partial, void* out, int out_format, int B, int C, long nvox,
                              int agg, void* stream);

/* Fused unprojection + exchange over NVLink peer memory (no NCCL on the data path).  peer_buffers[r] is rank r's
 * reduction buffer [n_peers slots][B/n_peers][P][nvox][C] float32, mapped into this process (CUDA IPC / symmetric
 * memory).  The kernel computes this rank's partials for all B samples and STORES sample b's partial directly into
 * peer_buffers[b / (B/n_peers)] at slot src_rank, so the transfer overlaps the gather/softmax math voxel by voxel.
 * After a cross-rank barrier, lt_unproject_reduce_finalize_fwd on each owner sums its n_peers slots (max for
 * LT_AGG_MAX), divides (softmax) and converts.  C = 4*2^k <= 128, V_local <= 8. */
int lt_unproject_push_fwd(const float* features, const float* proj, const float* coord, const float* conf,
                          float* const* peer_buffers /* HOST array of n_peers device pointers */, int n_peers, int src_rank,
                          int B, int V_local, int C, int h, int w, long nvox, int agg, void* stream);
int lt_unproject_reduce_finalize_fwd(const float* slots, int nslots, void* out, int out_format, int B, int C, long nvox,
                                     int agg, void* stream);

/* Feature-map exchange of the view-sharded path (alternative to the voxel-partial exchanges): rank `view_rank` of an n_peers-rank
 * view group stores its feature maps [B][V_local][row_elems] (float32) into the owner ranks' peer-mapped buffers
 * ([B/n_peers][V][row_elems] each; local view j = global view view_rank + j*n_peers); a cross-rank barrier orders the stores,
 * then each owner runs lt_unproject_aggregate_fwd on its buffer -- exactly the single-GPU arithmetic. */
int lt_feature_scatter_fwd(const float* feats, float* const* peer_buffers, int n_peers, int view_rank, int B, int V_local,
                           int V, long row_elems, void* stream);

/* Backward of lt_unproject_aggregate_fwd for the training loop (train.py:236 total_loss.backward(); the reference gets it
 * from autograd through F.grid_sample and the aggregation ops of op.py:131-162).  grad_out [B][nvox][C] float32;
 * grad_features [B][V][h][w][C] and grad_conf [B][V][C] (LT_AGG_CONF, may be NULL) are ACCUMULATED into (zero them first).
 * Projection matrices and coordinate volumes get no gradient here: lt_unproject_aggregate_bwd_geom adds them.  C % 4 == 0. */
int lt_unproject_aggregate_bwd(const float* features, const float* proj, const float* coord, const float* conf,
                               const float* grad_out, float* grad_features, float* grad_conf, int B, int V, int C, int h, int w,
                               long nvox, int agg, void* stream);
/* lt_unproject_aggregate_bwd plus the gradients the reference's torch graph gives the geometry (the matmul, the division by depth
 * and F.grid_sample with respect to the grid, op.py:113-147): grad_proj [B][V][12] and grad_coord [B][nvox][3], either may be NULL;
 * both are WRITTEN, not accumulated into.  grad_features / grad_conf are accumulated into by the same per-item code as
 * lt_unproject_aggregate_bwd.  The sample derivative is torch's grid_sampler_2d_backward convention (weight derivatives of the taps
 * inside the map, the same floor cell); a voxel that fails the depth test or has no tap inside the map contributes exactly 0.
 * Deterministic: no float atomics in the geometry sums (dP accumulates in float64 in a fixed order).  No host synchronisation.
 * C / 4 must be a power of two <= 32.  workspace: lt_unproject_aggregate_bwd_geom_workspace_bytes(B, V, nvox) bytes. */
size_t lt_unproject_aggregate_bwd_geom_workspace_bytes(int B, int V, long nvox);
int lt_unproject_aggregate_bwd_geom(const float* features, const float* proj, const float* coord, const float* conf,
                                    const float* grad_out, float* grad_features, float* grad_conf, float* grad_proj, float* grad_coord,
                                    void* workspace, size_t workspace_bytes, int B, int V, int C, int h, int w, long nvox, int agg,
                                    void* stream);
/* The fixed-order variant of lt_unproject_aggregate_bwd / lt_unproject_aggregate_bwd_geom (what training under
 * torch.use_deterministic_algorithms runs): no float atomics.  Every element of grad_features is the sum of the same terms gs * w_k the
 * atomic kernel adds, in one order fixed by the inputs (the four cells that have the pixel as a tap in a fixed order, each cell's
 * voxels ascending); grad_conf sums fixed chunks of voxels in chunk order.  The result depends on no launch geometry, SM count or
 * stream, and sample b's on no other sample.  grad_features / grad_conf are accumulated into (zero them first); grad_proj and
 * grad_coord (either may be NULL, both NULL for no geometry gradient) are written, bit-identical to lt_unproject_aggregate_bwd_geom's.
 * C % 4 == 0; with a geometry output C / 4 must be a power of two <= 32.  No host synchronisation.  workspace:
 * lt_unproject_aggregate_bwd_det_workspace_bytes(B, V, C, h, w, nvox, agg, geom) bytes on the current device (geom: 1 if grad_proj or
 * grad_coord will be given), about B V nvox (C + 16) * 4 bytes; 0 when the sizes are out of range or no device is present. */
size_t lt_unproject_aggregate_bwd_det_workspace_bytes(int B, int V, int C, int h, int w, long nvox, int agg, int geom);
int lt_unproject_aggregate_bwd_det(const float* features, const float* proj, const float* coord, const float* conf,
                                   const float* grad_out, float* grad_features, float* grad_conf, float* grad_proj, float* grad_coord,
                                   void* workspace, size_t workspace_bytes, int B, int V, int C, int h, int w, long nvox, int agg,
                                   void* stream);

/* ------------------------------------------------------------------------------------------
 * Volumetric soft-argmax.  Replaces op.integrate_tensor_3d_with_coordinates (op.py:84-96).
 *   logits: element (b, j, vox) at logits[b*batch_stride + vox*voxel_stride + j*chan_stride]
 *           (channels-last: voxel_stride = Cpad, chan_stride = 1; NCDHW: voxel_stride = 1,
 *           chan_stride = nvox)
 *   coord [B][nvox][3]; multiplier is applied to the logits first (triangulation.py:353)
 *   volumes_out [B][J][nvox] (may be NULL to skip the normalised-volume write)
 *   keypoints_out [B][J][3]
 *   workspace: lt_softargmax3d_workspace_bytes(B, J, nvox) bytes
 *   softmax = 1: softmax over the voxels (op.py:88-89); 0: the ReLU variant (op.py:90-91: no normalisation);
 *   2: ReLU with mass-normalised coordinates, the non-softmax branch of the 2-D op (integrate_tensor_2d, op.py:25-41:
 *   volumes_out = relu(logits), keypoints = sum(relu * coord) / sum(relu)).
 * ---------------------------------------------------------------------------------------- */
/* Backward of the soft-argmax in the op-level (NCDHW) layout: probs = the forward's volumes_out [B][J][nvox],
 * grad_keypoints [B][J][3], grad_volumes [B][J][nvox] or NULL -> grad_logits [B][J][nvox] (written).  softmax = the forward's
 * mode: 0 and 1 are op.py:84-96; 2 is the ReLU branch of the 2-D op (op.py:11-47, run with the pixel grid (x, y, 0) as coord):
 * d logit_i = multiplier * [probs_i > 0] * (grad_volumes_i + (<g_kp, x_i> - <g_kp, kp>) / sum probs).  Other modes are rejected.
 * scratch: >= B*J floats in mode 1, >= 2*B*J floats in mode 2, unused in mode 0. */
int lt_softargmax3d_bwd(const float* probs, const float* coord, const float* grad_keypoints, const float* grad_volumes,
                        float* grad_logits, float* scratch, int B, int J, long nvox, float multiplier, int softmax, void* stream);
/* Coordinate gradient of the soft-argmax (modes 0 and 1, where kp = sum_i probs_i x_i): grad_coord[b][i] = sum_j probs[b][j][i]
 * grad_keypoints[b][j], joints summed in order, WRITTEN.  Mode 2 (the 2-D op, whose pixel grid is no input) is rejected. */
int lt_softargmax3d_coord_bwd(const float* probs, const float* grad_keypoints, float* grad_coord, int B, int J, long nvox, int softmax,
                              void* stream);
size_t lt_softargmax3d_workspace_bytes(int B, int J, long nvox);
int lt_softargmax3d_fwd(const float* logits, long batch_stride, long voxel_stride, long chan_stride,
                        const float* coord, float* volumes_out, float* keypoints_out,
                        void* workspace, size_t workspace_bytes,
                        int B, int J, long nvox, float multiplier, int softmax, void* stream);
/* Second half of lt_softargmax3d_fwd for compact channels-last logits (chan_stride 1, voxel_stride % 4 == 0, 20 <= voxel_stride <= 32,
 * J <= voxel_stride, nvox % 8 == 0, nvox >= 16384; the layout lt_softargmax3d_fwd streams) whose statistics were produced by
 * lt_v2v_tail_stats_fwd: merge of the G partials per (sample, joint) -> keypoints_out, then volumes_out (may be NULL). */
int lt_softargmax3d_finish_fwd(const float* logits, long batch_stride, long voxel_stride, const float* coord, float* volumes_out,
                               float* keypoints_out, void* workspace, size_t workspace_bytes, int B, int J, long nvox, int G,
                               float multiplier, int softmax, void* stream);

/* ------------------------------------------------------------------------------------------
 * N-d convolution as implicit GEMM with fused epilogue.  Replaces nn.Conv2d/Conv3d (+ folded
 * BatchNorm, + residual add, + ReLU) call sites of pose_resnet.py:75-95,293-318 and
 * v2v.py:7-42,146-160; transposed convs (pose_resnet.py:266-291 k4s2p1, v2v.py:54-66 k2s2)
 * are issued as stride-phase sub-convolutions through the output mapping fields.
 *   out[n, od*osd+ood, oh*osh+ooh, ow*osw+oow, co] =
 *       act( scale[co] * sum_{kd,kh,kw,ci} in[n, od*sd-pd+kd, oh*sh-ph+kh, ow*sw-pw+kw, ci]
 *                                          * W[kd,kh,kw,ci,co]  + shift[co]  (+ residual) )
 * ---------------------------------------------------------------------------------------- */
typedef struct lt_conv_desc {
  int N, ID, IH, IW, Cin;    /* input tensor dims (channels-last) */
  int OD, OH, OW, Cout;      /* output positions computed by this call, output channels */
  int KD, KH, KW;            /* filter taps */
  int sd, sh, sw;            /* input stride */
  int pd, ph, pw;            /* front zero padding */
  int FD, FH, FW, FC;        /* full output tensor dims ([N][FD][FH][FW][FC]) */
  int osd, osh, osw;         /* output coordinate scale (1 for plain conv, 2 for deconv phases) */
  int ood, ooh, oow;         /* output coordinate offset */
  int relu;                  /* apply max(x,0) */
  int residual;              /* lt_residual; residual tensor has the output tensor's shape/format */
  int in_format, out_format; /* lt_format */
  int ogd, ogh, ogw;         /* output groups (0 or 1 = none): with G = ogd*ogh*ogw > 1 the Cout output channels are G blocks of
                                Cout/G channels, block g = (a*ogh + b)*ogw + c being written (and its residual read) at the output
                                offset (ood + a, ooh + b, oow + c) with channel index 0..Cout/G-1 (FC == Cout/G).  A k2 s2
                                transposed conv (v2v.py:54-66) is ONE 1x1x1 GEMM this way: N = 8 x Cout, osd=osh=osw=2, ogd=ogh=ogw=2;
                                scale/shift carry Cout entries (the per-channel values repeated G times).  A stride-2 data gradient
                                writes all input phases this way (fp32 or split-fp16 output); group g stores only the positions of
                                its phase inside the FD x FH x FW tensor.  LT_CONV_TC / TC1 only */
  int reserved0;             /* set to 0 (keeps the pointer below 8-byte aligned without implicit padding) */
  void* workspace;           /* optional device scratch for split-K (LT_CONV_TC / TC1 layers whose tiles fill the SMs
                                unevenly: the K loop is spread over more CTAs and summed in a fixed order, see
                                lt_conv_tc_plan); NULL = never split */
  size_t workspace_bytes;    /* size of workspace; a split is only used when its partial tiles fit */
} lt_conv_desc;

/* SIMT weights: float32 [KD*KH*KW][Cin][CoutW], CoutW = round_up(Cout, 4), zero padded.
 * TC weights: see lt_conv_tc_pack_weights.
 * LT_CONV_TC / TC1: `out` and `residual` must be 16-byte aligned and FC % 4 == 0 (the epilogue reads and writes them with TMA);
 * LT_ERR_INVALID otherwise. */
int lt_conv_nd_fwd(const lt_conv_desc* desc, const void* in, const void* weight, const float* scale,
                   const float* shift, const void* residual, void* out, int impl, void* stream);

/* Tensor-core weight packing: float32 [taps][Cin][Cout] (host or device? -> DEVICE)
 * to fp16 [taps][Cin/32][n tile][hi|lo][Nt][32] (64-byte rows; Nt = min(CoutP, 128), CoutP = round_up(Cout, 16));
 * Cin % 32 == 0. */
size_t lt_conv_tc_weight_bytes(int taps, int Cin, int Cout);

/* Work decomposition of one LT_CONV_TC / TC1 launch of lt_conv_nd_fwd on a GPU with `sm_count` SMs, computed on the host without
 * touching the device.  The persistent kernel runs `grid` CTAs (one per SM at most) over m_tiles x n_tiles x splits work units.
 * splits > 1 spreads each tile's K chunks over that many units whose fp32 partial tiles are summed in a fixed order by a second
 * launch; it is chosen by a model of the launch time (waves x per-unit K work + epilogue, plus the reduce pass) when `splitk` is
 * non-zero, desc->workspace is not NULL and the partial tiles fit desc->workspace_bytes.  Grouped outputs never split. */
typedef struct lt_conv_tc_launch_plan {
  int nt;                    /* N tile: 16, 32, 64 or 128 output channels */
  int m_tiles, n_tiles;      /* output tiles: 128 positions x nt channels */
  int chunks;                /* K chunks of a tile: taps x Cin / 32 */
  int splits;                /* K split count, 1 = none */
  int grid;                  /* CTAs launched: min(m_tiles x n_tiles x splits, sm_count) */
  int stages;                /* operand ring depth in shared memory */
  int epi_buffers;           /* shared-memory epilogue tile buffers: 2 for at most 4 chunks, else 1; 0 for split launches and
                                16-channel tiles, which keep no tile buffer */
} lt_conv_tc_launch_plan;
int lt_conv_tc_plan(const lt_conv_desc* desc, int sm_count, int splitk, lt_conv_tc_launch_plan* plan);

/* Chain mode of the LT_CONV_TC / TC1 kernel: `blocks` identical bottleneck blocks in ONE persistent launch.  descs[0..2] are the
 * lt_conv_nd_fwd descriptors of a block's 1x1 reduce, its 3x3 and its 1x1 expansion (residual BEFORE or AFTER ReLU): stride 1, split-
 * fp16 in and out, one output grid for all three, every Cout a multiple of 128 (N tile 128, never split along K).  The chain runs in
 * place on x (the first block's input, the last block's output); bufs = {Y1 even, Y1 odd, Y2 even, Y2 odd} hold the reduce and 3x3
 * outputs of even / odd blocks.  weights / scales / shifts: 3 x blocks entries, layer 3 k + c.  Every unit (layer, M tile, N tile)
 * computes the bits its own lt_conv_nd_fwd launch would.  counters: lt_conv_tc_chain_plan.counters unsigned ints of device scratch,
 * zeroed in the stream by the call.  At most 36 blocks per call. */
typedef struct lt_conv_tc_chain_launch_plan {
  int m_tiles;               /* output tiles of 128 positions, shared by every layer */
  int n_tiles[3];            /* N tiles of 128 channels of the reduce, the 3x3 and the expansion */
  int units;                 /* work units of the launch, numbered layer-major, then M tile, then N tile */
  int grid;                  /* CTAs launched: min(units, sm_count) */
  int counters;              /* unsigned ints of the counter scratch: the unit dispenser + one per (layer, M tile) */
} lt_conv_tc_chain_launch_plan;
int lt_conv_tc_chain_plan(const lt_conv_desc* descs, int blocks, int sm_count, lt_conv_tc_chain_launch_plan* plan);
/* What unit `unit` of that chain waits for before it loads: all of tiles[0..n_deps) of layer src_layer (-1: nothing, the first
 * layer) must have `need` N tiles stored.  At most `cap` tiles are written. */
typedef struct lt_conv_tc_chain_unit {
  int layer, m_tile, n_tile;
  int src_layer, need, n_deps;
} lt_conv_tc_chain_unit;
int lt_conv_tc_chain_deps(const lt_conv_desc* descs, int blocks, int unit, lt_conv_tc_chain_unit* info, int* tiles, int cap);
int lt_conv_tc_chain_fwd(const lt_conv_desc* descs, int blocks, void* x, void* const* bufs, const void* const* weights,
                         const float* const* scales, const float* const* shifts, void* counters, size_t counters_bytes, int impl,
                         void* stream);
int lt_conv_tc_pack_weights(const float* w_tap_ci_co, void* packed, int taps, int Cin, int Cout, void* stream);

/* Weight preparation (once per parameter version, engine.prepare()).
 * lt_conv_gather_weights_fwd: any framework filter layout -> canonical float32 [KD*KH*KW][CinP][CoutP] (zero padded); element
 *   (td, th, tw, ci, co) is read from w[base + td*s_td + th*s_th + tw*s_tw + ci*s_ci + co*s_co] (nn.Conv: (Cout, Cin, k...);
 *   nn.ConvTranspose: (Cin, Cout, k...); stride phases of a transposed conv: a tap sub-lattice walked with negative strides).
 * lt_fold_bn_fwd: eval-mode BatchNorm (pose_resnet.py:30-31, v2v.py:12) + conv bias -> per-channel scale / shift [CP] (double
 *   arithmetic, rounded once); mean == NULL: no BatchNorm.  accum_steps: tensor-core MMA steps that accumulate into the main fp32
 *   accumulator of the kernel that will consume this scale (taps x Cin / 16 for conv_tc_kernel, whose split-K reduce rescales to one
 *   split's share, and conv_fold_kernel; 9 x Cin / 16 for conv_lines_kernel; 0 for the exact-fp32 kernels).  The tensor core adds
 *   with truncation, which shrinks a sum by an expected 0.28 x steps x 2^-24 (wgmma on an H100 80GB HBM3 at 700 W: 0.25 - 0.33,
 *   tests/test_gpu_conv.py); the scale is multiplied by 1 + that, which halves the rms accumulation error.
 * lt_absmax_fwd: float bit pattern of max|w| over n elements.  Passed (optionally, else NULL) to the two calls above it selects the
 *   power-of-two filter pre-scale S = 2^(9 - floor(log2 max|w|)) of the tensor-core path: the gathered filter is multiplied by S,
 *   the folded scale by 1 / S (exact), so that the unscaled low halves of the split-fp16 weights stay normal numbers. */
int lt_absmax_fwd(const float* w, long n, unsigned int* out_bits, void* stream);
int lt_conv_gather_weights_fwd(const float* w, long base, long s_td, long s_th, long s_tw, long s_ci, long s_co, int KD, int KH, int KW,
                               int Cin, int CinP, int Cout, int CoutP, const unsigned int* absmax_bits, float* out, int out_ld,
                               int out_col0, void* stream);   /* out row length (0 = CoutP) and first column: column blocks of a wider filter */
int lt_fold_bn_fwd(const float* gamma, const float* beta, const float* mean, const float* var, const float* conv_bias, float eps,
                   int C, int CP, const unsigned int* absmax_bits, int accum_steps, float* scale, float* shift, void* stream);

/* Fused tail of the V2V network (v2v.py:154-160,168-169): back_layers[1], back_layers[2] (1x1x1 conv 32->32 + BN + ReLU each) and
 * output_layer (1x1x1 conv 32->J + bias) as one kernel: x split-fp16 [rows][32 hi | 32 lo] -> logits float32 [rows][FC]
 * (J <= FC <= 32, FC % 4 == 0; channels J..FC-1 are written as bias3 = 0).  w1/w2/w3: lt_conv_tc_pack_weights(taps 1, Cin 32)
 * buffers with Cout = 32, 32 and J; w3 must hold round_up(FC, 16) rows (it does for FC = round_up(J, 4)).  scale/shift: folded
 * BatchNorm ([32] each); scale3 / bias3 [FC]: output affine (lt_fold_bn_fwd without BatchNorm: the inverse filter pre-scale and
 * the bias, zero padded). */
int lt_v2v_tail_fwd(const void* x, const void* w1, const void* w2, const void* w3, const float* scale1, const float* shift1,
                    const float* scale2, const float* shift2, const float* scale3, const float* bias3, float* logits, long rows, int FC,
                    void* stream);
/* The same kernel with the STATISTICS PASS of the volumetric soft-argmax (op.py:84-96: integrate_tensor_3d_with_coordinates) fused into
 * the epilogue that produces the logits (v2v.py:168-169 -> op.py:88-89): x [B * nvox][64], nvox % 128 == 0, nvox >= 16384, FC == 20
 * (J 17..20; the statistics tile holds at most 20 floats per voxel, and lt_softargmax3d_finish_fwd streams no narrower rows, so any
 * other width is refused rather than producing partials nothing can merge; J <= 16 takes lt_v2v_tail_fwd + lt_softargmax3d_fwd), coord
 * [B][nvox][3].  `workspace` (lt_softargmax3d_workspace_bytes(B, J, nvox)) receives the per-CTA online-softmax partials
 * [B][*n_partials][J][5]; lt_softargmax3d_finish_fwd with G = *n_partials (a host value known at launch time, safe under stream
 * capture) merges them into the key points and writes the normalised volumes.  softmax: 1 = softmax, 0 = ReLU (volume_softmax:false). */
int lt_v2v_tail_stats_fwd(const void* x, const void* w1, const void* w2, const void* w3, const float* scale1, const float* shift1,
                          const float* scale2, const float* shift2, const float* scale3, const float* bias3, float* logits, int B,
                          long nvox, int FC, const float* coord, int J, float multiplier, int softmax, void* workspace,
                          size_t workspace_bytes, int* n_partials, void* stream);

/* Weight gradient of the lt_conv_nd_fwd call that `desc` describes (training backward of nn.Conv3d / nn.ConvTranspose3d, v2v.py):
 *   grad_w[t][ci][g*Cout + co] = sum_{n,o} in[n, o*s - p + t][ci] * grad_out[n, o*os + oo (+ group g's offset)][g*(desc->Cout/G) + co]
 * for ci < Cin, co < Cout (the real channel counts; padded channels never reach grad_w), with the output-mapping fields
 * (osd/ood, ogd/ogh/ogw) read as the forward reads them: a k2 s2 transposed conv is the one 1x1x1 grouped GEMM of the forward.
 * `in` and `grad_out` are split-fp16 (in_format = out_format = LT_FMT_S32) with desc->Cin and desc->Cout multiples of 32 and
 * FC == desc->Cout / G.  grad_out carries the power-of-two scale of lt_f32_to_s32_scaled with the same grad_absmax_bits (NULL: none),
 * which is divided out exactly.  wgmma with four-term products (fp32-grade).  Deterministic: the K split over positions writes
 * fp32 partial tiles into `workspace` (lt_conv_wgrad_workspace_bytes(desc) bytes) that a second pass sums in a fixed order. */
size_t lt_conv_wgrad_workspace_bytes(const lt_conv_desc* desc);
/* Work decomposition of one lt_conv_wgrad_fwd launch on a GPU with `sm_count` SMs, computed on the host without touching the
 * device.  The grid is taps x desc->Cin / 32 x ngroups x splits CTAs of nwg consumer warpgroups, one per 32-channel output block
 * (conv_wgrad_kernel<1 / 2 / 4>; the last group may have fewer active ones); each CTA runs its share of the m_tiles M tiles of 128
 * output positions (split z takes tiles [z m_tiles / splits, (z + 1) m_tiles / splits)) through a TMA ring of `stages` tiles. */
typedef struct lt_conv_wgrad_launch_plan {
  int nwg;                   /* warpgroups per CTA: 1, 2 or 4 */
  int ngroups;               /* CTAs along the output channels: ceil(Cout / 32 / nwg) */
  int m_tiles;               /* M tiles of 128 output positions (the K of the GEMM) */
  int splits;                /* K split count, 1 = none */
  int stages;                /* TMA ring depth in M tiles */
} lt_conv_wgrad_launch_plan;
int lt_conv_wgrad_plan(const lt_conv_desc* desc, int sm_count, lt_conv_wgrad_launch_plan* plan);
int lt_conv_wgrad_fwd(const lt_conv_desc* desc, const void* in, const void* grad_out, const unsigned int* grad_absmax_bits, int Cin,
                      int Cout, float* grad_w, void* workspace, size_t workspace_bytes, void* stream);

/* LT_CONV_TC_FOLD weight packing: float32 [K^3 taps (kd, kh, kw)][32][Cout] (DEVICE) -> split-fp16 [kw][kd][kh][NC][32 hi | 32 lo]
 * (128-byte rows), NC = round_up(Cout, 16), rows Cout .. NC-1 zero; lt_conv_fold_weight_bytes = K^3 * NC * 128. */
size_t lt_conv_fold_weight_bytes(int K, int Cout);
int lt_conv_fold_pack_weights(const float* w_tap_ci_co, void* packed, int K, int Cout, void* stream);

/* ------------------------------------------------------------------------------------------
 * Max pooling, channels-last (pose_resnet.py:208 3x3 s2 p1; v2v.py:51 2x2x2 s2).
 * ---------------------------------------------------------------------------------------- */
int lt_maxpool_fwd(const void* in, void* out, int format, int N, int ID, int IH, int IW, int C,
                   int kd, int kh, int kw, int sd, int sh, int sw, int pd, int ph, int pw,
                   int OD, int OH, int OW, void* stream);
/* Backward of a float32 max pool with kernel == stride == k on all three axes and no padding (floor mode), as
 * F.max_pool3d(x, k, k) computes it: grad_x[i] = 0 + grad_y[window] where x[i] is the window's arg-max by torch's rule (d, h, w
 * scan order; greater or NaN replaces; the first element if none does), 0 elsewhere and in the dropped tail.  Written, not
 * accumulated into.  x and grad_x share the element strides xs_* of (n, c, d, h, w); grad_y has gs_*.  No atomics. */
int lt_maxpool3d_bwd(const float* x, const float* grad_y, float* grad_x, int N, int C, int D, int H, int W, long xs_n, long xs_c,
                     long xs_d, long xs_h, long xs_w, long gs_n, long gs_c, long gs_d, long gs_h, long gs_w, int k, void* stream);

/* ------------------------------------------------------------------------------------------
 * Algebraic-triangulation path and confidence heads (config #5; SURVEY 8f rows 2 and 4).
 * ---------------------------------------------------------------------------------------- */
/* tail of GlobalAveragePoolingHead (pose_resnet.py:163-174): mean over the P positions of a channels-last map
 * [N][P][C0] (either format), Linear(C0,H1)+ReLU, Linear(H1,H2)+ReLU, Linear(H2,NO)+Sigmoid; nn.Linear weight layout. */
int lt_gap_mlp3_fwd(const void* in, int format, int N, int P, int C0, int H1, int H2, int NO, const float* w1,
                    const float* b1, const float* w2, const float* b2, const float* w3, const float* b3, float* out,
                    void* stream);
/* conf[B][V][C] <- conf / sum_v conf + eps   (triangulation.py:173-174 with eps = 1e-5; :268-269 with eps = 0) */
int lt_view_normalize_fwd(float* conf, int B, int V, int C, float eps, void* stream);
/* Training tail of ConfidenceHead (head_backend="native"): x is the second head BatchNorm's output (N, C0, H, W), float32, element
 * strides xs_* of (n, c, h, w) (NCHW and channels_last alike).  Per row n: 2x2 stride-2 max pool in floor mode (torch's rule: greater
 * or NaN replaces), ReLU keeping NaN, mean over the P = (H/2)(W/2) pooled positions -> x0 (N, C0); Linear(C0,H1)+ReLU -> h1 (N, H1),
 * Linear(H1,H2)+ReLU -> h2 (N, H2), Linear(H2,NO)+Sigmoid -> out (N, NO), the hidden ReLUs keeping NaN.  Fails for P = 0. */
int lt_conf_head_tail_fwd(const float* x, int N, int C0, int H, int W, long xs_n, long xs_c, long xs_h, long xs_w, int H1, int H2, int NO,
                          const float* w1, const float* b1, const float* w2, const float* b2, const float* w3, const float* b3, float* out,
                          float* x0, float* h1, float* h2, void* stream);
size_t lt_conf_head_tail_bwd_workspace_bytes(int N, int C0, int H1, int H2, int NO);
/* Backward of lt_conf_head_tail_fwd from grad_y = dL/d(out) and the saved x, x0, h1, h2, out (= y): autograd's derivative of the torch
 * formula (sigmoid backward g y (1 - y); ReLU masks !(h <= 0), so a NaN passes its gradient).  dW1..3, db1..3 (nn.Linear layouts)
 * are sums over the N rows in order; grad_x (element strides gs_*) is written in one pass, dx0 / P at each window's arg-max when
 * !(pooled <= 0), 0 elsewhere and in the tail floor mode drops.  No atomics; the caller passes the workspace. */
int lt_conf_head_tail_bwd(const float* x, int N, int C0, int H, int W, long xs_n, long xs_c, long xs_h, long xs_w, long gs_n, long gs_c,
                          long gs_h, long gs_w, int H1, int H2, int NO, const float* w1, const float* w2, const float* w3, const float* x0,
                          const float* h1, const float* h2, const float* y, const float* grad_y, float* grad_x, float* dw1, float* db1,
                          float* dw2, float* db2, float* dw3, float* db3, void* workspace, size_t workspace_bytes, void* stream);
/* Backward of y_v = c_v / S + eps, S = sum_u c_u over the views: grad_conf[b][v][c] = g_v / S - (sum_u g_u c_u) / S^2, from the
 * un-normalised conf [B][V][C]; float64 sums over the views in order. */
int lt_view_normalize_bwd(const float* conf, const float* grad, float* grad_conf, int B, int V, int C, void* stream);
/* confidence-weighted DLT (multiview.py:141-183): proj [B][V][3][4], keypoints_2d [B][V][J][2], confidences [B][V][J] or
 * NULL -> out [B][J][3]; float64 A^T A + Jacobi eigen-solve per (sample, joint). */
int lt_triangulate_dlt_fwd(const float* proj, const float* keypoints_2d, const float* confidences, float* out, int B,
                           int V, int J, void* stream);
/* Backward of lt_triangulate_dlt_fwd for the training loop: what autograd derives through the reference's per-(sample, joint)
 * torch.svd (multiview.py:141-183).  grad_out [B][J][3] -> grad_keypoints_2d [B][V][J][2] and grad_confidences [B][V][J] (may
 * be NULL; confidences NULL means all ones).  Both are WRITTEN, not accumulated into (unlike lt_unproject_aggregate_bwd).
 * Projection matrices get no gradient here: lt_triangulate_dlt_proj_bwd gives it.  One thread per (sample, joint)
 * redoes the forward's float64 eigen-solve (same code, same order of operations) and applies the first-order eigenvector
 * perturbation.  Where the smallest eigenvalue of A^T A is tied with another (gap <= 1e-12 of the larger of the two, or below
 * 1e-30 of the largest eigenvalue) the derivative does not exist; the tied term is dropped, so the gradient stays finite (torch's
 * SVD backward is not finite there). */
int lt_triangulate_dlt_bwd(const float* proj, const float* keypoints_2d, const float* confidences, const float* grad_out,
                           float* grad_keypoints_2d, float* grad_confidences, int B, int V, int J, void* stream);
/* Projection-matrix gradient of lt_triangulate_dlt_fwd (the reference's torch.svd backward through A = c (x P[2] - P[0]),
 * c (y P[2] - P[1]), multiview.py:159-163): grad_proj [B][V][3][4], WRITTEN.  The same eigen-solve, perturbation and tie rule as
 * lt_triangulate_dlt_bwd; per-(sample, joint) float64 partials in `workspace` (lt_triangulate_dlt_proj_bwd_workspace_bytes(B, V, J)
 * bytes), then summed over the joints in a fixed order: deterministic. */
size_t lt_triangulate_dlt_proj_bwd_workspace_bytes(int B, int V, int J);
int lt_triangulate_dlt_proj_bwd(const float* proj, const float* keypoints_2d, const float* confidences, const float* grad_out,
                                float* grad_proj, void* workspace, size_t workspace_bytes, int B, int V, int J, void* stream);
/* RANSAC triangulation baseline (RANSACTriangulationNet, triangulation.py:17-128).
 * Heat-map arg-max: logits channels-last float32 [N][h][w][C] (C >= J, the final conv's padded output) -> heatmaps [N][J][h][w]
 * (the raw logits) and keypoints_2d int64 [N][J][2] of torch.max's first maximal index (a NaN counts as the maximum):
 * x = trunc(float32(idx % w) * scale_x), y = trunc(float32(idx / w) * scale_y) with scale = float32(image side / map side).
 * One read and one write of the maps; per-slice bests in `workspace` (lt_heatmap_argmax_workspace_bytes(N, J, h, w) bytes),
 * merged in a fixed order by a second small kernel. */
size_t lt_heatmap_argmax_workspace_bytes(int N, int J, int h, int w);
int lt_heatmap_argmax_fwd(const float* logits, int C, float* heatmaps, long long* keypoints_2d, void* workspace, size_t workspace_bytes,
                          int N, int J, int h, int w, float scale_x, float scale_y, void* stream);
/* RANSAC triangulation: proj [B][V][3][4] float32, keypoints_2d int64 [B][V][J][2], the drawn view pairs int32
 * [B][J][n_iters][2] -> keypoints_3d [B][J][3] float32 and, if not NULL, inliers [B][J] uint64 (bit v = view v is an inlier).
 * One thread per (sample, joint), float64 throughout: per pair the 2-view DLT (rows x P[2] - P[0], y P[2] - P[1] formed in
 * float64) and the views with 0.5 |p - pi(X)| < eps; the first largest set wins; the DLT on it; with `direct`, the Huber
 * (f_scale 1) reprojection cost minimised by iteratively reweighted Levenberg-Marquardt.  2 <= V <= 64; no atomics, no host
 * synchronisation; the same result as lt_test_triangulate_ransac_host bit for bit. */
int lt_triangulate_ransac_fwd(const float* proj, const long long* keypoints_2d, const int* pairs, int B, int V, int J, int n_iters,
                              double eps, int direct, float* keypoints_3d, unsigned long long* inliers, void* stream);

/* ------------------------------------------------------------------------------------------
 * Volumetric cross-entropy loss of the volumetric training recipe.  Replaces VolumetricCELoss (mvn/models/loss.py:52-80, called
 * from train.py:222-230): per (sample, joint) the voxel nearest to the ground-truth point, loss.py:68-72 (per-sample difference
 * and distance tensors, torch.argmin, copy of the indices to the host), and v * -log(p + 1e-6) there, loss.py:74-77 (one chain
 * of selects per (sample, joint), each of whose backward zero-fills a volume-sized gradient).
 *   probs [B][J][nvox] (the softmaxed volumes), coord [B][nvox][3], keypoints_gt [B][J][3], validity [B][J] (element 0 of the
 *   reference's validity vector)
 *   loss: one float; index [B][J]: flat voxel index chosen; picked [B][J]: probs at that index (kept for the backward)
 *   workspace: lt_volumetric_ce_workspace_bytes(B, J, nvox) bytes
 * Exactly the reference's choice: the distance is sqrt((dx*dx + dy*dy) + dz*dz) rounded per fp32 operation (no FMA), and the
 * rounded square roots are compared over every voxel (any coordinate volume: rotated, permuted, flipped); ties go to the smallest
 * index, a NaN distance wins and the first NaN wins (torch.argmin).  loss = (sum over b, then j, of v * -log(p + 1e-6)) / (B * J),
 * summed from 0 in fp32 in that order; the term is computed when v == 0 as well (a NaN propagates as in the reference).
 * Deterministic, no host synchronisation.  nvox < 2^31. */
size_t lt_volumetric_ce_workspace_bytes(int B, int J, long nvox);
int lt_volumetric_ce_fwd(const float* probs, const float* coord, const float* keypoints_gt, const float* validity, float* loss,
                         int* index, float* picked, void* workspace, size_t workspace_bytes, int B, int J, long nvox, void* stream);
/* Backward of lt_volumetric_ce_fwd, what autograd derives through loss.py:76,80: grad_loss is a DEVICE pointer to dL/dloss;
 * grad_probs [B][J][nvox] is WRITTEN in full: -((g / (B * J)) * v) / (p + 1e-6) at index[b][j], 0 everywhere else.  Coordinates,
 * ground truth and validity get no gradient (the reference's argmin is detached; they are data). */
int lt_volumetric_ce_bwd(const float* grad_loss, const int* index, const float* picked, const float* validity, float* grad_probs,
                         int B, int J, long nvox, void* stream);

/* ------------------------------------------------------------------------------------------
 * Keypoint criteria of the training recipe.  Replace KeypointsMSELoss, KeypointsMSESmoothLoss, KeypointsMAELoss and
 * KeypointsL2Loss (mvn/models/loss.py:7-49), whose divisor max(1, sum v) is read to the host with .item() (and MSESmooth's
 * boolean-mask index synchronises once more).  pred, gt [n_points][dim] float32 (n_points = B * J), validity [n_points]:
 *   LT_KP_MSE         sum (gt - pred)^2 v / (dim * max(1, sum v))
 *   LT_KP_MSE_SMOOTH  the same with every d = (gt - pred)^2 v > threshold (strictly) replaced by d^0.1 * threshold^0.9
 *   LT_KP_MAE         sum |gt - pred| v / (dim * max(1, sum v))
 *   LT_KP_L2          sum over points of sqrt(sum_d (gt - pred)^2 v) / max(1, sum v)
 * Every term is formed in float64 and multiplied by v whatever v is (a non-finite residual at v = 0 gives NaN, as in the
 * reference); the terms and sum v are summed in float64 in a fixed order inside one CTA (bitwise-equal repeats).  loss: one float
 * (the float64 quotient rounded); norm: one double, the divisor, kept on the device for the backward.  No host synchronisation. */
enum lt_keypoints_loss_kind { LT_KP_MSE = 0, LT_KP_MSE_SMOOTH = 1, LT_KP_MAE = 2, LT_KP_L2 = 3 };
int lt_keypoints_loss_fwd(const float* pred, const float* gt, const float* validity, float* loss, double* norm, int kind,
                          double threshold, int n_points, int dim, void* stream);
/* Backward: grad_loss (DEVICE pointer, one float) and norm (lt_keypoints_loss_fwd's) -> grad_pred [n_points][dim] WRITTEN in full:
 * g / norm times the derivative autograd takes through the reference formula, in float64, rounded once.  MSE_SMOOTH's replaced
 * branch has 0.1 d^-0.9 threshold^0.9 dd/dpred; L2's is -(g / (2 sqrt(s))) v 2 (gt - pred), NaN where s = 0, as in torch.  The
 * ground truth and the validity get no gradient. */
int lt_keypoints_loss_bwd(const float* grad_loss, const float* pred, const float* gt, const float* validity, const double* norm,
                          float* grad_pred, int kind, double threshold, int n_points, int dim, void* stream);

/* ------------------------------------------------------------------------------------------
 * Batch-statistics BatchNorm for training, fused with the ReLU after it and the residual add of a residual unit.  Replaces
 * nn.BatchNorm2d / nn.BatchNorm3d in train and eval mode with the nn.ReLU and the `+ shortcut` that follow them (pose_resnet.py:25-137
 * residual units, stem and deconv stack; v2v.py:7-66 Basic3DBlock, Res3DBlock, Upsample3DBlock).
 *   x, residual, y, grad_* maps: float32 channels-last [M][C], M = N*D*H*W, C % 4 == 0, 16-byte aligned; residual may be NULL
 *   per-channel vectors [C]: gamma, beta, running_mean, running_var, save_mean, save_invstd
 * Forward: y = act(gamma * (x - mean) * invstd + beta (+ residual)), act = ReLU when relu != 0.  training != 0: mean and the biased
 * variance of the batch (M >= 2), save_invstd = 1 / sqrt(var + eps) (0 when var = eps = 0, as torch does), and the running statistics updated in place as nn.BatchNorm does
 * (running = (1 - momentum) * running + momentum * batch value, the variance unbiased by M / (M - 1)); training == 0: the running
 * statistics are used and left alone (save_mean / save_invstd still receive the values used).
 * Backward (the same relu / training; y is read only with relu, for its mask): g' = grad_y [!(y <= 0)], torch's threshold_backward,
 * so a NaN output passes its gradient; the forward's ReLU keeps NaN, as torch.relu does;
 *   grad_beta = sum g', grad_gamma = sum g' * xhat, xhat = (x - save_mean) * save_invstd;
 *   grad_x = gamma * save_invstd * (g' - sum g' / M - xhat * sum g' xhat / M) (training) or gamma * save_invstd * g' (eval);
 *   grad_residual = g' (NULL: not written); grad_gamma / grad_beta may be NULL.
 * Per-channel sums are accumulated in float64 and merged in a fixed order (no atomics): bitwise repeatable, no host synchronisation.
 * workspace: lt_batch_norm_workspace_bytes(M, C) bytes, for either direction.
 * ---------------------------------------------------------------------------------------- */
size_t lt_batch_norm_workspace_bytes(long M, int C);
/* Host-only launch plan of lt_batch_norm_fwd / _bwd for `sm_count` SMs (both launch from it with the device's count).  A CTA is tc x ry
 * = up to 256 threads: tc threads over float4 columns of one channel block, ry rows at a time.  Reduce passes run cblocks x splits
 * CTAs; split z takes rows [z rows_per_split, min((z + 1) rows_per_split, M)). */
typedef struct lt_batch_norm_launch_plan {
  int tc;                /* float4 columns per CTA: min(C / 4, 32) */
  int ry;                /* rows per CTA step: 256 / tc */
  int cblocks;           /* CTAs along the channels: ceil(C / 4 / tc) */
  int want_splits;       /* row splits of one wave of 4 CTAs per SM: ceil(4 sm_count / cblocks) */
  int max_splits;        /* row splits the workspace holds, independent of the device: min(ceil(M / (16 ry)), ceil(1024 / cblocks)) */
  int splits;            /* row splits launched: ceil(M / rows_per_split) <= min(want_splits, max_splits) */
  long rows_per_split;   /* ceil(M / min(want_splits, max_splits)) */
  int row_blocks;        /* CTAs along M of an apply pass: about two waves, at most ceil(M / (4 ry)) */
} lt_batch_norm_launch_plan;
int lt_batch_norm_plan(long M, int C, int sm_count, lt_batch_norm_launch_plan* plan);
int lt_batch_norm_fwd(const float* x, const float* residual, const float* gamma, const float* beta, float* running_mean, float* running_var,
                      float* save_mean, float* save_invstd, float* y, long M, int C, float eps, float momentum, int training, int relu,
                      void* workspace, size_t workspace_bytes, void* stream);
int lt_batch_norm_bwd(const float* x, const float* y, const float* grad_y, const float* gamma, const float* save_mean, const float* save_invstd,
                      float* grad_x, float* grad_residual, float* grad_gamma, float* grad_beta, long M, int C, int training, int relu,
                      void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Layout / format helpers.
 * ---------------------------------------------------------------------------------------- */
/* images [N][C][H][W] float32 -> [N][H][W][Cp] float32, channels >= C zero filled */
int lt_nchw_to_nhwc_f32(const float* in, float* out, int N, int C, int H, int W, int Cp, void* stream);
/* Batch image ingest.  Replaces image_batch_to_torch (mvn/utils/img.py:96-99, called from prepare_batch,
 * mvn/datasets/utils.py:45-52) and, for uint8 input with a table, normalize_image (img.py:102-110):
 *   in  [N][H][W][C] as collated by the dataset (datasets/utils.py:24), dtype lt_image_dtype, C <= 4
 *   lut NULL, or float32 [C][256] applied to uint8 input (out = lut[c][in]); NULL = plain cast
 *   out [N][C][H][W] float32 */
enum lt_image_dtype { LT_IMG_U8 = 0, LT_IMG_F32 = 1, LT_IMG_F64 = 2 };
int lt_images_hwc_to_nchw_fwd(const void* in, int in_dtype, const float* lut, float* out, int N, int C, int H, int W,
                              void* stream);
/* stem input packing: images [N][C<=8][H][W] float32 -> 2x2 space-to-depth split-fp16 [N][H/2][W/2][32],
 * channel (r*2+s)*C + c = in[c][2y+r][2x+s]; turns the 7x7 stride-2 stem conv (pose_resnet.py:205) into a 4x4 stride-1 conv */
int lt_stem_s2d_fwd(const float* in, void* out, int N, int C, int H, int W, void* stream);
/* channels-last [P][C] float32 <-> split-fp16 (C % 32 == 0) */
int lt_f32_to_s32(const float* in, void* out, long pixels, int C, void* stream);
int lt_s32_to_f32(const void* in, float* out, long pixels, int C, void* stream);
/* [P][C] float32 (any C) -> [P][CP] split-fp16 of S * x (CP % 32 == 0, channels C .. CP-1 zero), S the power-of-two pre-scale
 * that lt_absmax_fwd bits select (the filters' rule: max|S x| in [512, 1024)), 1 for absmax_bits NULL; inv_scale (NULL or one
 * float) receives 1 / S.  Output gradients lie far below fp16's normal range; scaled, they keep ~22 significand bits. */
int lt_f32_to_s32_scaled(const float* in, void* out, long pixels, int C, int CP, const unsigned int* absmax_bits, float* inv_scale,
                         void* stream);
/* channels-last [N][P][Cs] (first C channels) -> channels-first [N][C][P] float32 */
int lt_cl_to_cf_f32(const float* in, float* out, int N, long P, int Cs, int C, void* stream);

/* Self test of the wgmma/TMA GEMM core: D[M][N] = A[M][K] * B[N][K]^T with fp16 inputs
 * (row-major, K contiguous), float32 output.  variant selects descriptor conventions
 * (bring-up aid; 0 is the shipped one). */
int lt_tc_gemm_selftest(const void* a_fp16, const void* b_fp16, float* d, int M, int N, int K,
                        int variant, void* stream);

/* ------------------------------------------------------------------------------------------
 * Test hooks (NOT part of the product path): the per-item code of the backward kernels (and of the DLT forward) executed on
 * the CPU with HOST pointers, so that the `-m "not gpu"` suite can check the arithmetic against references without a GPU.
 * Same arguments as the device entry points minus scratch / stream (softmax: modes 0, 1 and 2 as in lt_softargmax3d_bwd).
 * ---------------------------------------------------------------------------------------- */
int lt_test_unproject_aggregate_bwd_host(const float* features, const float* proj, const float* coord, const float* conf,
                                         const float* grad_out, float* grad_features, float* grad_conf, int B, int V, int C, int h, int w,
                                         long nvox, int agg);
int lt_test_unproject_aggregate_bwd_det_host(const float* features, const float* proj, const float* coord, const float* conf,
                                             const float* grad_out, float* grad_features, float* grad_conf, float* grad_proj,
                                             float* grad_coord, int B, int V, int C, int h, int w, long nvox, int agg);
int lt_test_maxpool3d_bwd_host(const float* x, const float* grad_y, float* grad_x, int N, int C, int D, int H, int W, long xs_n,
                               long xs_c, long xs_d, long xs_h, long xs_w, long gs_n, long gs_c, long gs_d, long gs_h, long gs_w, int k);
int lt_test_softargmax3d_bwd_host(const float* probs, const float* coord, const float* grad_keypoints, const float* grad_volumes,
                                  float* grad_logits, int B, int J, long nvox, float multiplier, int softmax);
int lt_test_triangulate_dlt_fwd_host(const float* proj, const float* keypoints_2d, const float* confidences, float* out, int B,
                                     int V, int J);
int lt_test_triangulate_dlt_bwd_host(const float* proj, const float* keypoints_2d, const float* confidences, const float* grad_out,
                                     float* grad_keypoints_2d, float* grad_confidences, int B, int V, int J);
int lt_test_unproject_aggregate_bwd_geom_host(const float* features, const float* proj, const float* coord, const float* conf,
                                              const float* grad_out, float* grad_features, float* grad_conf, float* grad_proj,
                                              float* grad_coord, int B, int V, int C, int h, int w, long nvox, int agg);
int lt_test_softargmax3d_coord_bwd_host(const float* probs, const float* grad_keypoints, float* grad_coord, int B, int J, long nvox);
/* lt_conf_head_tail_fwd (+ lt_conf_head_tail_bwd when grad_y is not NULL) on host pointers, with the kernels' per-item code. */
int lt_test_conf_head_tail_host(const float* x, int N, int C0, int H, int W, long xs_n, long xs_c, long xs_h, long xs_w, long gs_n,
                                long gs_c, long gs_h, long gs_w, int H1, int H2, int NO, const float* w1, const float* b1, const float* w2,
                                const float* b2, const float* w3, const float* b3, float* out, float* x0, float* h1, float* h2,
                                const float* grad_y, float* grad_x, float* dw1, float* db1, float* dw2, float* db2, float* dw3, float* db3);
int lt_test_view_normalize_bwd_host(const float* conf, const float* grad, float* grad_conf, int B, int V, int C);
int lt_test_triangulate_dlt_proj_bwd_host(const float* proj, const float* keypoints_2d, const float* confidences, const float* grad_out,
                                          float* grad_proj, int B, int V, int J);
/* lt_volumetric_ce_fwd (+ lt_volumetric_ce_bwd when grad_probs is not NULL, grad_loss then a HOST pointer) on host pointers, with
 * the kernels' distance, argmin key, term and gradient code: loss.py:52-80. */
int lt_test_volumetric_ce_host(const float* probs, const float* coord, const float* keypoints_gt, const float* validity, float* loss,
                               int* index, float* picked, const float* grad_loss, float* grad_probs, int B, int J, long nvox);
/* lt_keypoints_loss_fwd (+ lt_keypoints_loss_bwd when grad_pred is not NULL, grad_loss then a HOST pointer) on host pointers, with
 * the kernels' term, derivative and summation order: loss.py:7-49. */
int lt_test_keypoints_loss_host(const float* pred, const float* gt, const float* validity, float* loss, double* norm,
                                const float* grad_loss, float* grad_pred, int kind, double threshold, int n_points, int dim);
/* lt_conv_wgrad_fwd's index mapping (which input row and which output-gradient row meet for a tap, M tile, row and output group) on
 * host pointers, summed in double over plain float32 channels-last tensors: in [N][ID][IH][IW][desc->Cin], grad_out [N][FD][FH][FW][FC]
 * -> grad_w [taps][Cin][G * Cout]. */
int lt_test_conv_wgrad_host(const lt_conv_desc* desc, const float* in, const float* grad_out, int Cin, int Cout, float* grad_w);
/* lt_triangulate_ransac_fwd's per-item code on host pointers. */
int lt_test_triangulate_ransac_host(const float* proj, const long long* keypoints_2d, const int* pairs, int B, int V, int J, int n_iters,
                                    double eps, int direct, float* keypoints_3d, unsigned long long* inliers);

#ifdef __cplusplus
}
#endif
#endif /* LT_B200_H */
