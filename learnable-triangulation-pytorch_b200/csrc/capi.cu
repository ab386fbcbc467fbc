// C-ABI glue: error state, device queries and the conv dispatcher (include/lt_b200.h).
#include "common.cuh"
#include <string.h>

namespace lt {

char* err_buf() {
  static thread_local char buf[512] = {0};
  return buf;
}

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(err_buf(), 512, fmt, ap);
  va_end(ap);
  return code;
}

static lt_options make_default_options() {
  lt_options o;
  o.tc_persist = 1; o.tc_splitk = 1; o.tc_bres = 1; o.tc_direct_epilogue = 0;
  o.fold_fast_issue = 1; o.fold_debug = 0;
  o.softargmax_stream = 1;
  o.unproject_v2 = 1; o.unproject_cpl = 4; o.unproject_lb = 0;     // 8 lanes x 4 channels, 4 CTAs/SM (the 4 x 8 variant measured 4 % faster, r02l,
  // but the view-sharded all_reduce path stopped matching the single-GPU forward on the seed-100 batches while it was the default)
  o.unproject_brick = 0; o.unproject_brick_order = 2;
  o.pair_nt = 0; o.pair_stages = 0;
  o.pair_prof = 0;
  o.pair_direct_out = 1;
  o.pair_two_acc = 1;
  o.fold_pair = 1;
  o.fold_direct = 0;
  o.fold_fullw = 1;
  return o;
}
static lt_options g_options = make_default_options();
const lt_options& opts() { return g_options; }

int sm_count() {
  static thread_local int cached_dev = -1, cached = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev != cached_dev) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached = n;
    cached_dev = dev;
  }
  return cached;
}

int conv_simt_fwd(const lt_conv_desc* d, const void* in, const void* weight, const float* scale, const float* shift,
                  const void* residual, void* out, void* stream);
int conv_tc_fwd_terms(const lt_conv_desc* d, const void* in, const void* weight, const float* scale, const float* shift,
                      const void* residual, void* out, int terms, void* stream);

int conv_pair_fwd(const lt_conv_desc* d, const void* in, const void* weight, const float* scale, const float* shift,
                  const void* residual, void* out, void* stream, int probe_only);

int conv_fold_fwd(const lt_conv_desc* d, const void* in, const void* weight, const float* scale, const float* shift,
                  const void* residual, void* out, void* stream);

}  // namespace lt

extern "C" int lt_version(void) { return 200; }

extern "C" void lt_default_options(lt_options* o) {
  if (o) *o = lt::make_default_options();
}
extern "C" int lt_get_options(lt_options* o) {
  if (!o) return lt::fail(LT_ERR_INVALID, "lt_get_options: null pointer");
  *o = lt::g_options;
  return LT_OK;
}
extern "C" int lt_set_options(const lt_options* o) {
  using namespace lt;
  LT_REQUIRE(o, "lt_set_options: null pointer");
  LT_REQUIRE(o->unproject_cpl == 4 || o->unproject_cpl == 8, "lt_set_options: unproject_cpl must be 4 or 8");
  LT_REQUIRE(o->tc_persist >= 0 && o->tc_persist <= 2, "lt_set_options: tc_persist must be 0, 1 or 2");
  g_options = *o;
  return LT_OK;
}

extern "C" const char* lt_last_error_string(void) { return lt::err_buf(); }

extern "C" int lt_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return lt::fail(LT_ERR_CUDA, "no CUDA device");
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return lt::fail(LT_ERR_CUDA, "cudaGetDeviceProperties failed");
  if (sm_count) *sm_count = prop.multiProcessorCount;
  if (cc_major) *cc_major = prop.major;
  if (cc_minor) *cc_minor = prop.minor;
  return LT_OK;
}

extern "C" int lt_conv_nd_fwd(const lt_conv_desc* d, const void* in, const void* weight, const float* scale,
                              const float* shift, const void* residual, void* out, int impl, void* stream) {
  using namespace lt;
  LT_REQUIRE(d && in && weight && scale && shift && out, "conv_nd: null pointer");
  LT_REQUIRE(d->N > 0 && d->ID > 0 && d->IH > 0 && d->IW > 0 && d->Cin > 0, "conv_nd: bad input dims");
  LT_REQUIRE(d->OD > 0 && d->OH > 0 && d->OW > 0 && d->Cout > 0, "conv_nd: bad output dims");
  LT_REQUIRE(d->KD > 0 && d->KH > 0 && d->KW > 0 && d->sd > 0 && d->sh > 0 && d->sw > 0, "conv_nd: bad filter/stride");
  LT_REQUIRE(d->osd > 0 && d->osh > 0 && d->osw > 0, "conv_nd: bad output scale");
  const int gd = d->ogd > 1 ? d->ogd : 1, gh = d->ogh > 1 ? d->ogh : 1, gw = d->ogw > 1 ? d->ogw : 1;
  LT_REQUIRE((d->OD - 1) * d->osd + d->ood + gd - 1 < d->FD && (d->OH - 1) * d->osh + d->ooh + gh - 1 < d->FH &&
                 (d->OW - 1) * d->osw + d->oow + gw - 1 < d->FW && d->ood >= 0 && d->ooh >= 0 && d->oow >= 0,
             "conv_nd: output mapping exceeds the output tensor");
  LT_REQUIRE(gd * gh * gw == 1 || impl == LT_CONV_TC || impl == LT_CONV_TC1 || impl == LT_CONV_TC_PAIR,
             "conv_nd: grouped output (ogd/ogh/ogw) is only implemented by the tensor-core kernels");
  LT_REQUIRE(d->residual == LT_RES_NONE || residual, "conv_nd: residual requested but pointer is null");
  LT_REQUIRE(d->residual >= LT_RES_NONE && d->residual <= LT_RES_AFTER_RELU, "conv_nd: bad residual mode");
  if (impl == LT_CONV_SIMT) return conv_simt_fwd(d, in, weight, scale, shift, residual, out, stream);
  if (impl == LT_CONV_TC) return conv_tc_fwd_terms(d, in, weight, scale, shift, residual, out, 3, stream);
  if (impl == LT_CONV_TC_FOLD) return conv_fold_fwd(d, in, weight, scale, shift, residual, out, stream);
  if (impl == LT_CONV_TC1) return conv_tc_fwd_terms(d, in, weight, scale, shift, residual, out, 1, stream);
  if (impl == LT_CONV_TC_PAIR) return conv_pair_fwd(d, in, weight, scale, shift, residual, out, stream, 0);
  return fail(LT_ERR_INVALID, "conv_nd: unknown impl %d", impl);
}

extern "C" int lt_conv_pair_eligible(const lt_conv_desc* d) {
  if (!d || d->in_format != LT_FMT_S32 || d->Cin % 32 != 0) return 0;
  return lt::conv_pair_fwd(d, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 1) == 0 ? 1 : 0;
}
