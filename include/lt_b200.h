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
  LT_CONV_TC_FOLD = 3, /* wgmma over all 32 output channels (Cin = 32 cubic 3^3 / 7^3 stride-1 layers; weights from
                         lt_conv_fold_pack_weights; desc->Cout = real channel count <= 32, FC = 32) */
  LT_CONV_TC_PAIR = 4  /* wgmma, 3-term products, weights padded to 128 output channels (layers with Cout % 128 == 0 that
                         lt_conv_pair_eligible accepts; weights from lt_conv_pair_pack_weights) */
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
  int tc_splitk;           /* conv_tc: split-K for grids below half the SMs (default 1) */
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
 * (softmax) and converts to out_format. */
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
 * Projection matrices and coordinate volumes carry no gradient (they do not in the reference either).  C % 4 == 0. */
int lt_unproject_aggregate_bwd(const float* features, const float* proj, const float* coord, const float* conf,
                               const float* grad_out, float* grad_features, float* grad_conf, int B, int V, int C, int h, int w,
                               long nvox, int agg, void* stream);

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
 * grad_keypoints [B][J][3], grad_volumes [B][J][nvox] or NULL, scratch >= B*J floats -> grad_logits [B][J][nvox]. */
int lt_softargmax3d_bwd(const float* probs, const float* coord, const float* grad_keypoints, const float* grad_volumes,
                        float* grad_logits, float* scratch, int B, int J, long nvox, float multiplier, int softmax, void* stream);
size_t lt_softargmax3d_workspace_bytes(int B, int J, long nvox);
int lt_softargmax3d_fwd(const float* logits, long batch_stride, long voxel_stride, long chan_stride,
                        const float* coord, float* volumes_out, float* keypoints_out,
                        void* workspace, size_t workspace_bytes,
                        int B, int J, long nvox, float multiplier, int softmax, void* stream);
/* Second half of lt_softargmax3d_fwd for compact channels-last logits (chan_stride 1, 20 <= voxel_stride <= 32) whose statistics were
 * produced by lt_v2v_tail_stats_fwd: merge of the G partials per (sample, joint) -> keypoints_out, then volumes_out (may be NULL). */
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
                                scale/shift carry Cout entries (the per-channel values repeated G times).  LT_CONV_TC / _PAIR only */
  int reserved0;             /* set to 0 (keeps the pointer below 8-byte aligned without implicit padding) */
  void* workspace;           /* optional device scratch for split-K (layers with fewer M x N tiles than half the SMs:
                                the K loop is spread over more CTAs and summed in a fixed order); NULL = never split */
  size_t workspace_bytes;    /* size of workspace; a split is only used when its partial tiles fit */
} lt_conv_desc;

/* SIMT weights: float32 [KD*KH*KW][Cin][CoutW], CoutW = round_up(Cout, 4), zero padded.
 * TC weights: see lt_conv_tc_pack_weights. */
int lt_conv_nd_fwd(const lt_conv_desc* desc, const void* in, const void* weight, const float* scale,
                   const float* shift, const void* residual, void* out, int impl, void* stream);

/* Tensor-core weight packing: float32 [taps][Cin][Cout] (host or device? -> DEVICE)
 * to fp16 [taps][Cin/32][n tile][hi|lo][Nt][32] (64-byte rows; Nt = min(CoutP, 128), CoutP = round_up(Cout, 16));
 * Cin % 32 == 0. */
size_t lt_conv_tc_weight_bytes(int taps, int Cin, int Cout);
int lt_conv_tc_pack_weights(const float* w_tap_ci_co, void* packed, int taps, int Cin, int Cout, void* stream);

/* Weight preparation (once per parameter version, engine.prepare()).
 * lt_conv_gather_weights_fwd: any framework filter layout -> canonical float32 [KD*KH*KW][CinP][CoutP] (zero padded); element
 *   (td, th, tw, ci, co) is read from w[base + td*s_td + th*s_th + tw*s_tw + ci*s_ci + co*s_co] (nn.Conv: (Cout, Cin, k...);
 *   nn.ConvTranspose: (Cin, Cout, k...); stride phases of a transposed conv: a tap sub-lattice walked with negative strides).
 * lt_fold_bn_fwd: eval-mode BatchNorm (pose_resnet.py:30-31, v2v.py:12) + conv bias -> per-channel scale / shift [CP] (double
 *   arithmetic, rounded once); mean == NULL: no BatchNorm.  accum_steps: tensor-core MMA steps that accumulate into the main fp32
 *   accumulator of the kernel that will consume this scale (taps x Cin / 16; 0 for the exact-fp32 kernels).  The tensor core adds
 *   with truncation, which shrinks a sum by an expected 0.28 x steps x 2^-24 (rate measured on the tensor-memory MMA of the kernels' first target, not re-measured for wgmma);
 *   the scale is multiplied by 1 + that, which halves the rms accumulation error.
 * lt_absmax_fwd: float bit pattern of max|w| over n elements.  Passed (optionally, else NULL) to the two calls above it selects the
 *   power-of-two filter pre-scale S = 2^(9 - floor(log2 max|w|)) of the tensor-core path: the gathered filter is multiplied by S,
 *   the folded scale by 1 / S (exact), so that the unscaled low halves of the split-fp16 weights stay normal numbers. */
int lt_absmax_fwd(const float* w, long n, unsigned int* out_bits, void* stream);
int lt_conv_gather_weights_fwd(const float* w, long base, long s_td, long s_th, long s_tw, long s_ci, long s_co, int KD, int KH, int KW,
                               int Cin, int CinP, int Cout, int CoutP, const unsigned int* absmax_bits, float* out, int out_ld,
                               int out_col0, void* stream);   /* out row length (0 = CoutP) and first column: column blocks of a wider filter */
int lt_fold_bn_fwd(const float* gamma, const float* beta, const float* mean, const float* var, const float* conv_bias, float eps,
                   int C, int CP, const unsigned int* absmax_bits, int accum_steps, float* scale, float* shift, void* stream);

/* CTA-pair weight packing: float32 [taps][Cin][Cout] (DEVICE) -> fp16 [taps][Cin/32][CoutP][32 hi | 32 lo] (128-byte rows),
 * CoutP = round_up(Cout, 128).  lt_conv_pair_eligible: 1 if LT_CONV_TC_PAIR covers this launch (shape / tiling heuristics),
 * else 0 (use LT_CONV_TC). */
size_t lt_conv_pair_weight_bytes(int taps, int Cin, int Cout);
int lt_conv_pair_pack_weights(const float* w_tap_ci_co, void* packed, int taps, int Cin, int Cout, void* stream);
int lt_conv_pair_eligible(const lt_conv_desc* desc);

/* Fused tail of the V2V network (v2v.py:154-160,168-169): back_layers[1], back_layers[2] (1x1x1 conv 32->32 + BN + ReLU each) and
 * output_layer (1x1x1 conv 32->J + bias) as one kernel: x split-fp16 [rows][32 hi | 32 lo] -> logits float32 [rows][FC]
 * (J <= FC <= 32, FC % 4 == 0; channels J..FC-1 are written as bias3 = 0).  w1/w2/w3: lt_conv_pair_pack_weights(taps 1, Cin 32)
 * buffers; scale/shift: folded BatchNorm ([32] each); scale3 / bias3 [32]: output affine (lt_fold_bn_fwd without BatchNorm: the
 * inverse filter pre-scale and the bias, zero padded). */
int lt_v2v_tail_fwd(const void* x, const void* w1, const void* w2, const void* w3, const float* scale1, const float* shift1,
                    const float* scale2, const float* shift2, const float* scale3, const float* bias3, float* logits, long rows, int FC,
                    void* stream);
/* The same kernel with the STATISTICS PASS of the volumetric soft-argmax (op.py:84-96: integrate_tensor_3d_with_coordinates) fused into
 * the epilogue that produces the logits (v2v.py:168-169 -> op.py:88-89): x [B * nvox][64], nvox % 128 == 0, FC <= 20, coord
 * [B][nvox][3].  `workspace` (lt_softargmax3d_workspace_bytes(B, J, nvox)) receives the per-CTA online-softmax partials
 * [B][*n_partials][J][5]; lt_softargmax3d_finish_fwd with G = *n_partials (a host value known at launch time, safe under stream
 * capture) merges them into the key points and writes the normalised volumes.  softmax: 1 = softmax, 0 = ReLU (volume_softmax:false). */
int lt_v2v_tail_stats_fwd(const void* x, const void* w1, const void* w2, const void* w3, const float* scale1, const float* shift1,
                          const float* scale2, const float* shift2, const float* scale3, const float* bias3, float* logits, int B,
                          long nvox, int FC, const float* coord, int J, float multiplier, int softmax, void* workspace,
                          size_t workspace_bytes, int* n_partials, void* stream);

/* kw-folded weight packing: float32 [K^3][32][Cout] (DEVICE) -> split-fp16 [kd][kh][kw*NC + co][64], NC = round_up(Cout, 16). */
size_t lt_conv_fold_weight_bytes(int K, int Cout);
int lt_conv_fold_pack_weights(const float* w_tap_ci_co, void* packed, int K, int Cout, void* stream);

/* ------------------------------------------------------------------------------------------
 * Max pooling, channels-last (pose_resnet.py:208 3x3 s2 p1; v2v.py:51 2x2x2 s2).
 * ---------------------------------------------------------------------------------------- */
int lt_maxpool_fwd(const void* in, void* out, int format, int N, int ID, int IH, int IW, int C,
                   int kd, int kh, int kw, int sd, int sh, int sw, int pd, int ph, int pw,
                   int OD, int OH, int OW, void* stream);

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
/* confidence-weighted DLT (multiview.py:141-183): proj [B][V][3][4], keypoints_2d [B][V][J][2], confidences [B][V][J] or
 * NULL -> out [B][J][3]; float64 A^T A + Jacobi eigen-solve per (sample, joint). */
int lt_triangulate_dlt_fwd(const float* proj, const float* keypoints_2d, const float* confidences, float* out, int B,
                           int V, int J, void* stream);

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
/* channels-last [N][P][Cs] (first C channels) -> channels-first [N][C][P] float32 */
int lt_cl_to_cf_f32(const float* in, float* out, int N, long P, int Cs, int C, void* stream);

/* Self test of the wgmma/TMA GEMM core: D[M][N] = A[M][K] * B[N][K]^T with fp16 inputs
 * (row-major, K contiguous), float32 output.  variant selects descriptor conventions
 * (bring-up aid; 0 is the shipped one). */
int lt_tc_gemm_selftest(const void* a_fp16, const void* b_fp16, float* d, int M, int N, int K,
                        int variant, void* stream);

/* ------------------------------------------------------------------------------------------
 * Test hooks (NOT part of the product path): the per-item code of the two backward kernels executed on the CPU with HOST
 * pointers, so that the `-m "not gpu"` suite can check the gradient arithmetic against torch autograd without a GPU.
 * Same arguments as the device entry points minus scratch / stream.
 * ---------------------------------------------------------------------------------------- */
int lt_test_unproject_aggregate_bwd_host(const float* features, const float* proj, const float* coord, const float* conf,
                                         const float* grad_out, float* grad_features, float* grad_conf, int B, int V, int C, int h, int w,
                                         long nvox, int agg);
int lt_test_softargmax3d_bwd_host(const float* probs, const float* coord, const float* grad_keypoints, const float* grad_volumes,
                                  float* grad_logits, int B, int J, long nvox, float multiplier, int softmax);

#ifdef __cplusplus
}
#endif
#endif /* LT_B200_H */
