// seg_dwconv.cu — depthwise 3x3 (atrous) convolution, the HBM-bound half of the Aligned-Xception backbone
// (SeparableConv2d.conv1, models/deeplabv3_plus.py:77-78: groups = C, stride 1|2, dilation 1|2|4, "same" padding).
// 0.75 % of the network's FLOPs but 348 M activation elements per image (SURVEY.md §2.3): pure bandwidth work, so
// these are vectorised streaming kernels (8 channels = 16 bytes per thread, channel-group-stationary: each thread
// keeps its 9 x 8 filter taps in registers while it strides over pixels) — not GEMMs.
//   fwd       : y = dw(x)            (+ per-channel sum / sum-of-squares of y for the BatchNorm that follows)
//   bwd_data  : dx (+)= dw^T(dy)     (gather form, no atomics)
//   bwd_weight: dw[9][C] += sum_pixels dy * x_shifted   (72 register accumulators per thread, slotted atomics)
// Packed depthwise weights: fp32 [9][C] (tap-major).
#include "seg_common.cuh"
#include "seg_sync.cuh"

namespace seg {


struct DwMap {
  int g, rl, rows_par;
  bool active;
};
__device__ __forceinline__ DwMap dw_map(int C) {
  const int G = C >> 3;
  const int GB = min(G, 256);
  DwMap r;
  r.rows_par = 256 / GB;
  r.rl = threadIdx.x / GB;
  r.g = blockIdx.y * GB + (threadIdx.x % GB);
  r.active = r.g < G && r.rl < r.rows_par;
  return r;
}

__device__ __forceinline__ void load_taps(const float* __restrict__ w9, int C, int co, float (*w)[8]) {
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    *reinterpret_cast<float4*>(w[t]) = __ldg(reinterpret_cast<const float4*>(w9 + (size_t)t * C + co));
    *reinterpret_cast<float4*>(w[t] + 4) = __ldg(reinterpret_cast<const float4*>(w9 + (size_t)t * C + co + 4));
  }
}

// block-level reduction of NACC x 8 per-thread sums over the row lanes (fixed order), then ONE fp64 atomic per channel into
// acc[NACC][C] (zero at launch): exact accumulation of fp32 partials -> order-independent, bit-reproducible totals
template <int NACC>
__device__ __forceinline__ void dw_block_reduce(const DwMap& m, int C, float (*acc)[8], double* __restrict__ acc_out) {
  __shared__ float red[256 * 8];
  const int GB = min(C >> 3, 256);
  const int gl = threadIdx.x % GB;
  for (int a = 0; a < NACC; ++a) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 8; ++i) red[threadIdx.x * 8 + i] = m.active ? acc[a][i] : 0.f;
    __syncthreads();
    if (m.rl == 0 && m.g < (C >> 3)) {
      float s[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) s[i] = 0.f;
      for (int r = 0; r < m.rows_par; ++r)
#pragma unroll
        for (int i = 0; i < 8; ++i) s[i] += red[(r * GB + gl) * 8 + i];
#pragma unroll
      for (int i = 0; i < 8; ++i) atomicAdd(acc_out + (size_t)a * C + m.g * 8 + i, (double)s[i]);
    }
  }
}

__global__ void __launch_bounds__(256)
    dwconv_fwd_kernel(const __nv_bfloat16* __restrict__ x, int ldx, const float* __restrict__ w9, __nv_bfloat16* __restrict__ y,
                      int ldy, int N, int H, int W, int C, int P, int Q, int stride, int pad, int dil,
                      double* __restrict__ stats, const SyncDesc sync, unsigned* sync_ticket) {
  const DwMap m = dw_map(C);
  float w[9][8];
  float acc[2][8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[0][i] = acc[1][i] = 0.f;
  if (m.active) {
    const int co = m.g * 8;
    load_taps(w9, C, co, w);
    const int64_t M = (int64_t)N * P * Q;
    const int64_t step = (int64_t)gridDim.x * m.rows_par;
    for (int64_t row = (int64_t)blockIdx.x * m.rows_par + m.rl; row < M; row += step) {
      const int n = (int)(row / (P * Q));
      const int rem = (int)(row - (int64_t)n * P * Q);
      const int p = rem / Q, q = rem - p * Q;
      float o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = 0.f;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const int ih = p * stride - pad + r * dil;
        if (ih < 0 || ih >= H) continue;
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const int iw = q * stride - pad + s * dil;
          if (iw < 0 || iw >= W) continue;
          float f[8];
          unpack8(*reinterpret_cast<const bf16x8*>(x + (((int64_t)n * H + ih) * W + iw) * ldx + co), f);
#pragma unroll
          for (int i = 0; i < 8; ++i) o[i] = fmaf(f[i], w[r * 3 + s][i], o[i]);
        }
      }
      const bf16x8 v = pack8(o);
      *reinterpret_cast<bf16x8*>(y + row * ldy + co) = v;
      if (stats) {
        unpack8(v, o);  // the statistics are of y as stored (bf16-rounded): the values bn_apply normalises
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          acc[0][i] += o[i];
          acc[1][i] += o[i] * o[i];
        }
      }
    }
  }
  if (stats) {
    dw_block_reduce<2>(m, C, acc, stats);
    if (sync.world > 0) {  // SyncBN: the last block pushes the finished totals to the peers
      __shared__ int sm_flag;
      sync_push_when_last(sync, stats, 2 * C, sync_ticket, gridDim.x * gridDim.y, (int)threadIdx.x, 256, [] { __syncthreads(); }, &sm_flag);
    }
  }
}

__global__ void __launch_bounds__(256)
    dwconv_bwd_data_kernel(const __nv_bfloat16* __restrict__ dy, int lddy, const float* __restrict__ w9,
                           __nv_bfloat16* __restrict__ dx, int lddx, int N, int H, int W, int C, int P, int Q, int stride,
                           int pad, int dil, float beta) {
  const DwMap m = dw_map(C);
  if (!m.active) return;
  const int co = m.g * 8;
  float w[9][8];
  load_taps(w9, C, co, w);
  const int64_t M = (int64_t)N * H * W;
  const int64_t step = (int64_t)gridDim.x * m.rows_par;
  for (int64_t row = (int64_t)blockIdx.x * m.rows_par + m.rl; row < M; row += step) {
    const int n = (int)(row / (H * W));
    const int rem = (int)(row - (int64_t)n * H * W);
    const int ih = rem / W, iw = rem - ih * W;
    float o[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int th = ih + pad - r * dil;
      if (th < 0 || (th % stride) != 0) continue;
      const int p = th / stride;
      if (p >= P) continue;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int tw = iw + pad - s * dil;
        if (tw < 0 || (tw % stride) != 0) continue;
        const int q = tw / stride;
        if (q >= Q) continue;
        float f[8];
        unpack8(*reinterpret_cast<const bf16x8*>(dy + (((int64_t)n * P + p) * Q + q) * lddy + co), f);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = fmaf(f[i], w[r * 3 + s][i], o[i]);
      }
    }
    __nv_bfloat16* dst = dx + row * lddx + co;
    if (beta != 0.f) {
      float f[8];
      unpack8(*reinterpret_cast<const bf16x8*>(dst), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] += beta * f[i];
    }
    *reinterpret_cast<bf16x8*>(dst) = pack8(o);
  }
}

__global__ void __launch_bounds__(256)
    dwconv_bwd_weight_kernel(const __nv_bfloat16* __restrict__ dy, int lddy, const __nv_bfloat16* __restrict__ x, int ldx,
                             int N, int H, int W, int C, int P, int Q, int stride, int pad, int dil,
                             double* acc9 /*[9][C] fp64, zero at launch*/, unsigned* ticket, float* __restrict__ dw9, float beta) {
  const DwMap m = dw_map(C);
  float acc[9][8];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[t][i] = 0.f;
  if (m.active) {
    const int co = m.g * 8;
    const int64_t M = (int64_t)N * P * Q;
    const int64_t step = (int64_t)gridDim.x * m.rows_par;
    for (int64_t row = (int64_t)blockIdx.x * m.rows_par + m.rl; row < M; row += step) {
      const int n = (int)(row / (P * Q));
      const int rem = (int)(row - (int64_t)n * P * Q);
      const int p = rem / Q, q = rem - p * Q;
      float g[8];
      unpack8(*reinterpret_cast<const bf16x8*>(dy + row * lddy + co), g);
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const int ih = p * stride - pad + r * dil;
        if (ih < 0 || ih >= H) continue;
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const int iw = q * stride - pad + s * dil;
          if (iw < 0 || iw >= W) continue;
          float f[8];
          unpack8(*reinterpret_cast<const bf16x8*>(x + (((int64_t)n * H + ih) * W + iw) * ldx + co), f);
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[r * 3 + s][i] = fmaf(f[i], g[i], acc[r * 3 + s][i]);
        }
      }
    }
  }
  dw_block_reduce<9>(m, C, acc, acc9);
  // the last block rounds the fp64 totals: dw9 = beta*dw9 + total
  __shared__ int last_flag;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last_flag = (atomicAdd(ticket, 1u) == gridDim.x * gridDim.y - 1u);
  __syncthreads();
  if (!last_flag) return;
  __threadfence();
  for (int i = threadIdx.x; i < 9 * C; i += blockDim.x) {
    const float v = (float)__ldcg(acc9 + i);
    dw9[i] = (beta != 0.f) ? beta * dw9[i] + v : v;
  }
}

// depthwise master weight [C][1][3][3] fp32 <-> packed [9][C] fp32
__global__ void dw_pack_kernel(const float* __restrict__ w, float* __restrict__ w9, int C) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 9 * C) return;
  const int t = i / C, c = i - t * C;
  w9[i] = w[(size_t)c * 9 + t];
}
__global__ void dw_unpack_kernel(const float* __restrict__ g9, float* __restrict__ g, int C, float beta) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 9 * C) return;
  const int c = i / 9, t = i - c * 9;
  const float v = g9[(size_t)t * C + c];
  g[i] = (beta != 0.f) ? beta * g[i] + v : v;
}

constexpr int DW_WGRAD_BLOCKS_PER_SM = 4;  // every block ends with 72*C/8 fp64 atomics: fewer, fatter blocks
static dim3 dw_grid(int64_t M, int C, int blocks_per_sm = 6) {
  const int G = C / 8;
  const int GB = G < 256 ? G : 256;
  const int rows_par = 256 / GB;
  const int gy = ceil_div(G, GB);
  int64_t gx = ceil_div64(M, (int64_t)rows_par * 2);
  const int64_t cap = ((int64_t)num_sms() * blocks_per_sm + gy - 1) / gy;
  if (gx > cap) gx = cap;
  if (gx < 1) gx = 1;
  return dim3((unsigned)gx, (unsigned)gy, 1);
}
}  // namespace seg

using namespace seg;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define BF(p) reinterpret_cast<__nv_bfloat16*>(p)
#define CBF(p) reinterpret_cast<const __nv_bfloat16*>(p)

extern "C" {

// scratch of seg_dwconv3x3_bwd_weight: fp64 accumulators [9][C] + a ticket, as floats
int64_t seg_dwconv_scratch_floats(int C) { return (int64_t)2 * 9 * C + 32; }

// xs: the x-side tensor (x or dx), ys: the y-side tensor (y or dy).  Every load and store is a 16-byte bf16x8, so besides
// C and the pitches the base pointers must be 16-byte aligned (a channel slice must start at a multiple of 8 channels).
static int dw_check(const seg_conv_desc* d, const void* xs, const void* ys) {
  SEG_REQUIRE(d && d->R == 3 && d->S == 3 && d->K == d->C, "dwconv: 3x3 depthwise (K == C) only");
  SEG_REQUIRE(d->C % 8 == 0 && d->ldx % 8 == 0 && d->ldy % 8 == 0, "dwconv: C / pitches must be multiples of 8");
  SEG_REQUIRE((reinterpret_cast<uintptr_t>(xs) & 15) == 0 && (reinterpret_cast<uintptr_t>(ys) & 15) == 0,
              "dwconv: x / y / dy / dx base pointers must be 16-byte aligned (channel offset a multiple of 8)");
  const int P = (d->H + 2 * d->pad - d->dil * 2 - 1) / d->stride + 1, Q = (d->W + 2 * d->pad - d->dil * 2 - 1) / d->stride + 1;
  SEG_REQUIRE(P == d->P && Q == d->Q, "dwconv: output size mismatch");
  return 0;
}

int seg_dwconv3x3_fwd(const seg_conv_desc* d, const void* x, const float* w9, void* y, double* stats,
                      const seg_sync_desc* sync, void* sync_ticket, void* stream) {
  if (dw_check(d, x, y)) return 1;
  SEG_REQUIRE(!sync || (stats && sync_ticket), "dwconv fwd: SyncBN needs stats and a zeroed ticket word");
  if (sync && sync_check_desc(sync, 4ll * d->C, "dwconv fwd")) return 1;  // 2C fp64 statistics
  const int64_t M = (int64_t)d->N * d->P * d->Q;
  dwconv_fwd_kernel<<<dw_grid(M, d->C), 256, 0, ST(stream)>>>(CBF(x), d->ldx, w9, BF(y), d->ldy, d->N, d->H, d->W, d->C, d->P, d->Q,
                                                              d->stride, d->pad, d->dil, stats, sync ? *sync : SyncDesc{},
                                                              reinterpret_cast<unsigned*>(sync_ticket));
  return check_launch("dwconv_fwd");
}

int seg_dwconv3x3_bwd_data(const seg_conv_desc* d, const void* dy, const float* w9, void* dx, float beta, void* stream) {
  if (dw_check(d, dx, dy)) return 1;
  const int64_t M = (int64_t)d->N * d->H * d->W;
  dwconv_bwd_data_kernel<<<dw_grid(M, d->C), 256, 0, ST(stream)>>>(CBF(dy), d->ldy, w9, BF(dx), d->ldx, d->N, d->H, d->W, d->C,
                                                                   d->P, d->Q, d->stride, d->pad, d->dil, beta);
  return check_launch("dwconv_bwd_data");
}

int seg_dwconv3x3_bwd_weight(const seg_conv_desc* d, const void* dy, const void* x, float* dw9, float beta, float* scratch,
                             void* stream) {
  if (dw_check(d, x, dy)) return 1;
  SEG_REQUIRE(scratch != nullptr && (reinterpret_cast<uintptr_t>(scratch) & 7) == 0,
              "dwconv bwd_weight: 8-byte aligned scratch of seg_dwconv_scratch_floats(C) floats required");
  const int64_t M = (int64_t)d->N * d->P * d->Q;
  const size_t acc_bytes = (size_t)9 * d->C * sizeof(double);
  cudaMemsetAsync(scratch, 0, acc_bytes + 64, ST(stream));
  double* acc9 = reinterpret_cast<double*>(scratch);
  unsigned* ticket = reinterpret_cast<unsigned*>(reinterpret_cast<char*>(scratch) + acc_bytes);
  dwconv_bwd_weight_kernel<<<dw_grid(M, d->C, DW_WGRAD_BLOCKS_PER_SM), 256, 0, ST(stream)>>>(
      CBF(dy), d->ldy, CBF(x), d->ldx, d->N, d->H, d->W, d->C, d->P, d->Q, d->stride, d->pad, d->dil, acc9, ticket, dw9, beta);
  return check_launch("dwconv_bwd_weight");
}

int seg_dw_pack_weight(const float* w_c133, float* w9, int C, void* stream) {
  dw_pack_kernel<<<ceil_div(9 * C, 128), 128, 0, ST(stream)>>>(w_c133, w9, C);
  return check_launch("dw_pack");
}
int seg_dw_unpack_wgrad(const float* g9, float* g_c133, int C, float beta, void* stream) {
  dw_unpack_kernel<<<ceil_div(9 * C, 128), 128, 0, ST(stream)>>>(g9, g_c133, C, beta);
  return check_launch("dw_unpack");
}

}  // extern "C"
