// api.cu — C-ABI entry points (include/atomai_b200.h): error plumbing, validation and dispatch
// between the math modes.  No CPU path exists: every function launches CUDA work or fails.
#include <stdarg.h>
#include <string.h>

#include <map>
#include <mutex>
#include <utility>

#include "common.cuh"

// implemented in conv_tc.cu / conv_simt.cu / wgrad_tc.cu
int ab_conv_tc_supported(const ab_conv_t* d);
int64_t ab_pack_weights_tc_elems(int Cout, int Cin, int th, int tw, int mode, int x3);
int ab_pack_weights_tc(const float* w, int Cout, int Cin, int th, int tw, int mode, int x3,
                       float* out, cudaStream_t stream);
int ab_conv_tc_fwd(const ab_conv_t* d, const float* wblob, const float* bias, float* y, int ld_y,
                   double* stats, cudaStream_t stream);
int ab_conv_tc_info(const ab_conv_t* d, int* grid, int* block, int* smem_bytes);
int ab_pack_weights_simt(const float* w, int Cout, int Cin, int th, int tw, int mode, float* out,
                         cudaStream_t stream);
int ab_conv_simt_fwd(const ab_conv_t* d, const float* w, const float* bias, float* y, int ld_y,
                     double* stats, cudaStream_t stream);
int ab_conv_simt_wgrad(const ab_conv_t* d, const float* dy, int ld_dy, float* dw,
                       cudaStream_t stream);
int ab_wgrad_tc_supported(const ab_conv_t* d);
int ab_conv_tc_wgrad(const ab_conv_t* d, const float* dy, int ld_dy, float* dw,
                     cudaStream_t stream);

static thread_local char g_err[512] = "";

void ab_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int ab_optin_smem(const void* func, int bytes, unsigned char* done) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = -1;
  if (dev >= 0 && done[dev]) return 0;
  if (cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess) {
    ab_set_error("cudaFuncSetAttribute(MaxDynamicSharedMemorySize=%d) failed", bytes);
    return 1;
  }
  if (dev >= 0) done[dev] = 1;
  return 0;
}

int ab_num_sms() {
  static int sms[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (sms[dev] == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0)
      v = 132;
    sms[dev] = v;
  }
  return sms[dev];
}

// One workspace per (device, stream): launches on one stream run in order, so the slots and
// tickets of consecutive launches never overlap; launches on different streams get different
// workspaces and may run concurrently.
int ab_ordered_ws(cudaStream_t stream, int64_t n_doubles, int groups, Ordered* out) {
  constexpr int kMaxGroups = 4096;
  struct Ws {
    double* slots = nullptr;
    int64_t cap = 0;
    unsigned* tickets = nullptr;
  };
  static std::mutex mu;
  static std::map<std::pair<int, cudaStream_t>, Ws> table;
  int dev = 0;
  AB_CUDA(cudaGetDevice(&dev));
  AB_CHECK(groups >= 1 && groups <= kMaxGroups && n_doubles >= 0,
           "ordered-sum workspace: %d groups", groups);
  std::lock_guard<std::mutex> lock(mu);
  Ws& w = table[std::make_pair(dev, stream)];
  if (!w.tickets) {
    AB_CUDA(cudaMalloc(&w.tickets, kMaxGroups * sizeof(unsigned)));
    AB_CUDA(cudaMemsetAsync(w.tickets, 0, kMaxGroups * sizeof(unsigned), stream));
  }
  if (n_doubles > w.cap) {
    // cudaFree waits for the device, so no launch still reads the old buffer
    const int64_t want = n_doubles > 2 * w.cap ? n_doubles : 2 * w.cap;
    if (w.slots) AB_CUDA(cudaFree(w.slots));
    w.slots = nullptr;
    w.cap = 0;
    AB_CUDA(cudaMalloc(&w.slots, want * sizeof(double)));
    w.cap = want;
  }
  out->slots = w.slots;
  out->ticket = w.tickets;
  return 0;
}

int ab_make_srcset(const ab_conv_t* d, SrcSet* out) {
  AB_CHECK(d != nullptr, "null conv descriptor");
  AB_CHECK(d->nsrc == 1 || d->nsrc == 2, "conv: nsrc=%d (must be 1 or 2)", d->nsrc);
  AB_CHECK(d->N >= 0 && d->H > 0 && d->W > 0 && d->Cout > 0, "conv: bad shape N=%d H=%d W=%d Cout=%d",
           d->N, d->H, d->W, d->Cout);
  AB_CHECK((d->ks_h == 1 || d->ks_h == 3) && (d->ks_w == 1 || d->ks_w == 3),
           "conv: kernel %dx%d unsupported (1 or 3 per axis)", d->ks_h, d->ks_w);
  AB_CHECK(d->dil >= 1, "conv: dilation %d", d->dil);
  out->nsrc = d->nsrc;
  out->Ctot = 0;
  for (int i = 0; i < 2; ++i) {
    SrcDev& s = out->s[i];
    if (i < d->nsrc) {
      const ab_src_t& a = d->src[i];
      AB_CHECK(a.ptr != nullptr && a.C > 0 && a.ld >= a.C, "conv: source %d invalid (C=%d ld=%d)", i,
               a.C, a.ld);
      AB_CHECK((a.scale == nullptr) == (a.shift == nullptr), "conv: source %d scale/shift mismatch",
               i);
      AB_CHECK(a.pool >= 0 && a.pool <= 3, "conv: source %d transform code %d", i, a.pool);
      AB_CHECK(a.pool < 2 || (d->H % 2 == 0 && d->W % 2 == 0),
               "conv: upsample-on-load needs even H, W (got %d x %d)", d->H, d->W);
      s.ptr = a.ptr; s.scale = a.scale; s.shift = a.shift; s.C = a.C; s.ld = a.ld; s.pool = a.pool;
      out->Ctot += a.C;
    } else {
      s.ptr = nullptr; s.scale = nullptr; s.shift = nullptr; s.C = 0; s.ld = 0; s.pool = 0;
    }
  }
  return 0;
}

extern "C" {

const char* atomai_b200_version(void) { return "atomai_b200 0.1.0 (sm_90a)"; }
const char* atomai_b200_last_error(void) { return g_err; }

int atomai_b200_device_ok(int device) {
  int major = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device) != cudaSuccess) {
    ab_set_error("cannot query device %d", device);
    return 0;
  }
  return major == 9 ? 1 : 0;
}

int64_t atomai_b200_prep_weights_elems(int Cout, int Cin, int ks_h, int ks_w, int mode, int math) {
  if (math == AB_MATH_TF32 || math == AB_MATH_TF32X3)
    return ab_pack_weights_tc_elems(Cout, Cin, ks_h, ks_w, mode, math == AB_MATH_TF32X3);
  return (int64_t)Cout * Cin * ks_h * ks_w;
}

int atomai_b200_prep_weights(const float* w_oihw, int Cout, int Cin, int ks_h, int ks_w, int mode,
                             int math, float* out, void* stream) {
  AB_CHECK(w_oihw && out, "prep_weights: null pointer");
  AB_CHECK(mode == AB_WMODE_FWD || mode == AB_WMODE_DGRAD, "prep_weights: mode=%d", mode);
  if (math == AB_MATH_TF32 || math == AB_MATH_TF32X3)
    return ab_pack_weights_tc(w_oihw, Cout, Cin, ks_h, ks_w, mode, math == AB_MATH_TF32X3, out,
                              (cudaStream_t)stream);
  return ab_pack_weights_simt(w_oihw, Cout, Cin, ks_h, ks_w, mode, out, (cudaStream_t)stream);
}

int atomai_b200_conv_fwd(const ab_conv_t* d, const float* w_prepped, const float* bias, float* y,
                         int ld_y, double* stats, void* stream) {
  AB_CHECK(d && w_prepped && y, "conv_fwd: null pointer");
  AB_CHECK(d->out_nchw || ld_y >= d->Cout, "conv_fwd: ld_y=%d < Cout=%d", ld_y, d->Cout);
  if (d->math == AB_MATH_TF32 || d->math == AB_MATH_TF32X3) {
    AB_CHECK(ab_conv_tc_supported(d),
             "conv_fwd: shape not supported by the tensor-core path (need C%%8==0, Cout%%16==0, "
             "16<=Cout<=256, 16B-aligned sources); use AB_MATH_FP32");
    return ab_conv_tc_fwd(d, w_prepped, bias, y, ld_y, stats, (cudaStream_t)stream);
  }
  AB_CHECK(d->math == AB_MATH_FP32, "conv_fwd: math=%d", d->math);
  return ab_conv_simt_fwd(d, w_prepped, bias, y, ld_y, stats, (cudaStream_t)stream);
}

int atomai_b200_conv_supported(const ab_conv_t* d, int which) {
  if (!d) return 0;
  return which == 0 ? ab_conv_tc_supported(d) : ab_wgrad_tc_supported(d);
}

int atomai_b200_conv_info(const ab_conv_t* d, int* grid, int* block, int* smem_bytes) {
  AB_CHECK(d && grid && block && smem_bytes, "conv_info: null pointer");
  AB_CHECK((d->math == AB_MATH_TF32 || d->math == AB_MATH_TF32X3) && ab_conv_tc_supported(d),
           "conv_info: tensor-core path only");
  return ab_conv_tc_info(d, grid, block, smem_bytes);
}

int atomai_b200_conv_wgrad(const ab_conv_t* d, const float* dy, int ld_dy, float* dw_oihw,
                           void* stream) {
  AB_CHECK(d && dy && dw_oihw, "conv_wgrad: null pointer");
  AB_CHECK(ld_dy >= d->Cout, "conv_wgrad: ld_dy=%d < Cout=%d", ld_dy, d->Cout);
  if (d->math == AB_MATH_TF32 || d->math == AB_MATH_TF32X3) {
    AB_CHECK(ab_wgrad_tc_supported(d), "conv_wgrad: shape not supported by the tensor-core path");
    return ab_conv_tc_wgrad(d, dy, ld_dy, dw_oihw, (cudaStream_t)stream);
  }
  AB_CHECK(d->math == AB_MATH_FP32, "conv_wgrad: math=%d", d->math);
  return ab_conv_simt_wgrad(d, dy, ld_dy, dw_oihw, (cudaStream_t)stream);
}

}  // extern "C"
