// seg_api.cu — C-ABI glue: error reporting, device check, launch accounting and the convolution dispatcher
// (wgmma path where the shape allows it, CUDA-core implicit GEMM otherwise).  No CPU fallback anywhere.
#include <stdarg.h>
#include "seg_common.cuh"
#include "seg_sync.cuh"

namespace seg {

static thread_local char g_err[1024] = "";
std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

namespace tc {
bool supported(const seg_conv_desc* d);
int conv_fwd(const seg_conv_desc* d, const void* x, const void* w, void* y, int y_dtype, const float* bias, float beta,
             double* stats, unsigned* stat_ticket, const seg_sync_desc* sync, cudaStream_t stream);
int conv_dgrad(const seg_conv_desc* d, const void* dy, const void* w, void* dx, float beta, cudaStream_t stream);
int conv_wgrad(const seg_conv_desc* d, const void* dy, const void* x, float* dw, float* ws, cudaStream_t stream);
int64_t wgrad_workspace_floats(const seg_conv_desc* d);
}  // namespace tc
namespace simt {
int conv_fwd(const seg_conv_desc* d, const void* x, const void* w, void* y, int y_dtype, const float* bias, float beta,
             double* stats, unsigned* stat_ticket, const seg_sync_desc* sync, cudaStream_t stream);
int conv_dgrad(const seg_conv_desc* d, const void* dy, const void* w, void* dx, float beta, cudaStream_t stream);
int conv_wgrad(const seg_conv_desc* d, const void* dy, const void* x, float* dw, cudaStream_t stream);
}  // namespace simt

static int check_desc(const seg_conv_desc* d) {
  SEG_REQUIRE(d != nullptr, "null conv descriptor");
  SEG_REQUIRE(d->N > 0 && d->H > 0 && d->W > 0 && d->C > 0 && d->K > 0 && d->R > 0 && d->S > 0, "bad conv dims");
  SEG_REQUIRE(d->stride >= 1 && d->dil >= 1 && d->pad >= 0, "bad conv stride/dil/pad");
  const int P = (d->H + 2 * d->pad - d->dil * (d->R - 1) - 1) / d->stride + 1;
  const int Q = (d->W + 2 * d->pad - d->dil * (d->S - 1) - 1) / d->stride + 1;
  SEG_REQUIRE(P == d->P && Q == d->Q, "conv output size mismatch: expected %dx%d got %dx%d", P, Q, d->P, d->Q);
  SEG_REQUIRE(d->ldx >= d->C && d->ldy >= d->K, "conv pitch smaller than channel count");
  return 0;
}

// The wgmma path reads its operands through TMA tensor maps, whose base addresses must be 16-byte aligned.  A channel
// slice at an offset that is not a multiple of 8 bf16 elements is not; AUTO sends such a call to the CUDA-core kernel.
static bool tma_base_ok(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace seg

using namespace seg;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

const char* seg_last_error(void) { return g_err; }
int seg_version(void) { return 100; }
int64_t seg_launch_count(void) { return (int64_t)g_launches.load(); }
void seg_launch_count_reset(void) { g_launches.store(0); }

int seg_device_ok(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    set_error("cudaGetDevice: %s", cudaGetErrorString(e));
    return 1;
  }
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0) {
    set_error("seg_b200 kernels are built for sm_90a (H100) only; device is sm_%d%d", major, minor);
    return 1;
  }
  return 0;
}

int seg_conv2d_fwd(const seg_conv_desc* d, const void* x, const void* w_packed, void* y, int y_dtype, const float* bias,
                   float beta, double* stats, const seg_sync_desc* sync, void* sync_ticket, int impl, void* stream) {
  if (check_desc(d)) return 1;
  SEG_REQUIRE(!sync || (stats && sync_ticket), "seg_conv2d_fwd: SyncBN needs stats and a zeroed ticket word");
  if (sync && sync_check_desc(sync, 4ll * d->K, "seg_conv2d_fwd")) return 1;  // 2K fp64 statistics
  SEG_REQUIRE(!stats || beta == 0.f, "seg_conv2d_fwd: BatchNorm statistics need beta = 0 (got beta = %g)", (double)beta);
  const bool tc_ok = tc::supported(d) && tma_base_ok(x) && tma_base_ok(w_packed);
  unsigned* tk = reinterpret_cast<unsigned*>(sync_ticket);
  if (impl == SEG_IMPL_TC || (impl == SEG_IMPL_AUTO && tc_ok))
    return tc::conv_fwd(d, x, w_packed, y, y_dtype, bias, beta, stats, tk, sync, ST(stream));
  return simt::conv_fwd(d, x, w_packed, y, y_dtype, bias, beta, stats, tk, sync, ST(stream));
}

int seg_conv2d_dgrad(const seg_conv_desc* d, const void* dy, const void* w_packed, void* dx, float beta, int impl,
                     void* stream) {
  if (check_desc(d)) return 1;
  const bool tc_ok = tc::supported(d) && d->ldy % 8 == 0 && tma_base_ok(dy) && tma_base_ok(w_packed);
  if (impl == SEG_IMPL_TC || (impl == SEG_IMPL_AUTO && tc_ok))
    return tc::conv_dgrad(d, dy, w_packed, dx, beta, ST(stream));
  return simt::conv_dgrad(d, dy, w_packed, dx, beta, ST(stream));
}

static bool wgrad_on_tc(const seg_conv_desc* d, int impl) {
  return impl == SEG_IMPL_TC || (impl == SEG_IMPL_AUTO && tc::supported(d) && d->ldy % 8 == 0);
}

int64_t seg_conv2d_wgrad_workspace_floats(const seg_conv_desc* d, int impl) {
  if (check_desc(d)) return -1;
  return wgrad_on_tc(d, impl) ? tc::wgrad_workspace_floats(d) : 0;
}

int seg_conv2d_wgrad(const seg_conv_desc* d, const void* dy, const void* x, float* dw_packed, float* workspace, int impl,
                     void* stream) {
  if (check_desc(d)) return 1;
  // the workspace query sees no pointers: a call it sized for the wgmma path may still run on the CUDA cores, which
  // leave the workspace unused
  if (wgrad_on_tc(d, impl) && (impl == SEG_IMPL_TC || (tma_base_ok(dy) && tma_base_ok(x))))
    return tc::conv_wgrad(d, dy, x, dw_packed, workspace, ST(stream));
  return simt::conv_wgrad(d, dy, x, dw_packed, ST(stream));
}

}  // extern "C"
