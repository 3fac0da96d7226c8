// seg_conv_simt.cu — CUDA-core implicit-GEMM convolution (forward / dgrad / wgrad) for every shape the
// wgmma path does not take (stride-2 data gradients, channel counts that are not a multiple of 8) and as an
// on-device cross-check of the tensor-core kernels.  64x64 tiles, 16-deep k-slices staged in shared memory,
// 256 threads x (4x4) fp32 accumulators.  Same semantics as seg_conv_tc.cu (reference: nn.Conv2d call sites listed there).
#include "seg_common.cuh"

namespace seg {
int bn_stats_launch(const void* x, int64_t M, int C, int ldx, double* stats, const seg_sync_desc* sync, unsigned* ticket,
                    cudaStream_t stream);  // seg_elementwise.cu
namespace simt {

constexpr int TM = 64, TN = 64, TK = 16;

struct P {
  seg_conv_desc d;
  const __nv_bfloat16* a;  // fwd: x ; dgrad: dy ; wgrad: dy
  const __nv_bfloat16* b;  // fwd/dgrad: packed w ; wgrad: x
  void* out;
  int out_dtype;
  float beta;
  const float* bias;
  float* stats;
  int64_t M;     // GEMM rows
  int Ncols;     // GEMM cols
  int64_t Kdim;  // GEMM depth
  int splits;
};

enum { FWD = 0, DGRAD = 1, WGRAD = 2 };

// A[m][k]
template <int MODE>
__device__ __forceinline__ float load_a(const P& p, int64_t m, int64_t k) {
  const seg_conv_desc& d = p.d;
  if (MODE == FWD) {
    // m = (n, op, oq) ; k = (tap, c)
    const int tap = (int)(k / d.C), c = (int)(k - (int64_t)tap * d.C);
    const int r = tap / d.S, s = tap - r * d.S;
    const int n = (int)(m / (d.P * d.Q));
    const int rem = (int)(m - (int64_t)n * d.P * d.Q);
    const int op = rem / d.Q, oq = rem - op * d.Q;
    const int ih = op * d.stride - d.pad + r * d.dil, iw = oq * d.stride - d.pad + s * d.dil;
    if (ih < 0 || ih >= d.H || iw < 0 || iw >= d.W) return 0.f;
    return bf2f(p.a[(((int64_t)n * d.H + ih) * d.W + iw) * d.ldx + c]);
  } else if (MODE == DGRAD) {
    // m = (n, ih, iw) ; k = (tap, ko)
    const int tap = (int)(k / d.K), ko = (int)(k - (int64_t)tap * d.K);
    const int r = tap / d.S, s = tap - r * d.S;
    const int n = (int)(m / (d.H * d.W));
    const int rem = (int)(m - (int64_t)n * d.H * d.W);
    const int ih = rem / d.W, iw = rem - ih * d.W;
    const int th = ih + d.pad - r * d.dil, tw = iw + d.pad - s * d.dil;
    if (th < 0 || tw < 0 || (th % d.stride) != 0 || (tw % d.stride) != 0) return 0.f;
    const int op = th / d.stride, oq = tw / d.stride;
    if (op >= d.P || oq >= d.Q) return 0.f;
    return bf2f(p.a[(((int64_t)n * d.P + op) * d.Q + oq) * d.ldy + ko]);
  } else {
    // m = ko ; k = pixel (n, op, oq)
    return bf2f(p.a[k * d.ldy + m]);
  }
}
// B[k][n]
template <int MODE>
__device__ __forceinline__ float load_b(const P& p, int64_t k, int n) {
  const seg_conv_desc& d = p.d;
  if (MODE == FWD) {
    const int tap = (int)(k / d.C), c = (int)(k - (int64_t)tap * d.C);
    return bf2f(p.b[((int64_t)tap * d.K + n) * d.C + c]);
  } else if (MODE == DGRAD) {
    const int tap = (int)(k / d.K), ko = (int)(k - (int64_t)tap * d.K);
    return bf2f(p.b[((int64_t)tap * d.K + ko) * d.C + n]);
  } else {
    // n = (tap, c) ; k = pixel
    const int tap = n / d.C, c = n - tap * d.C;
    const int r = tap / d.S, s = tap - r * d.S;
    const int img = (int)(k / (d.P * d.Q));
    const int rem = (int)(k - (int64_t)img * d.P * d.Q);
    const int op = rem / d.Q, oq = rem - op * d.Q;
    const int ih = op * d.stride - d.pad + r * d.dil, iw = oq * d.stride - d.pad + s * d.dil;
    if (ih < 0 || ih >= d.H || iw < 0 || iw >= d.W) return 0.f;
    return bf2f(p.b[(((int64_t)img * d.H + ih) * d.W + iw) * d.ldx + c]);
  }
}

template <int MODE>
__global__ void __launch_bounds__(256) igemm_simt(const P p) {
  __shared__ float As[TK][TM + 4];
  __shared__ float Bs[TK][TN + 4];
  const int tid = threadIdx.x;
  const int64_t m0 = (int64_t)blockIdx.x * TM;
  const int n0 = blockIdx.y * TN;
  const int tx = tid & 15, ty = tid >> 4;  // 16 x 16 threads, each 4 x 4
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  int64_t kbeg = 0, kend = p.Kdim;
  if (MODE == WGRAD) {
    const int64_t per = ceil_div64(ceil_div64(p.Kdim, p.splits), TK) * TK;
    kbeg = (int64_t)blockIdx.z * per;
    kend = min(kbeg + per, p.Kdim);
  }
  for (int64_t k0 = kbeg; k0 < kend; k0 += TK) {
    // cooperative loads: 64*16 = 1024 elements each, 4 per thread
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int idx = tid + e * 256;
      {
        // A tile: pick the fast index to follow memory contiguity (k for FWD/DGRAD, m for WGRAD)
        int mi, ki;
        if (MODE == WGRAD) { mi = idx & 63; ki = idx >> 6; } else { ki = idx & 15; mi = idx >> 4; }
        const int64_t m = m0 + mi, k = k0 + ki;
        As[ki][mi] = (m < p.M && k < kend) ? load_a<MODE>(p, m, k) : 0.f;
      }
      {
        int ni, ki;
        if (MODE == FWD) { ki = idx & 15; ni = idx >> 4; } else { ni = idx & 63; ki = idx >> 6; }
        const int n = n0 + ni;
        const int64_t k = k0 + ki;
        Bs[ki][ni] = (n < p.Ncols && k < kend) ? load_b<MODE>(p, k, n) : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < TK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  // epilogue
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t m = m0 + ty * 4 + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= p.Ncols) continue;
      float v = acc[i][j];
      if (MODE == WGRAD) {
        // out = dw[tap][ko][c] fp32, n = tap*C + c, m = ko
        const int tap = n / p.d.C, c = n - tap * p.d.C;
        atomicAdd(reinterpret_cast<float*>(p.out) + ((int64_t)tap * p.d.K + m) * p.d.C + c, v);
      } else {
        if (p.bias) v += p.bias[n];
        const int64_t ld = (MODE == FWD) ? p.d.ldy : p.d.ldx;
        if (p.out_dtype == SEG_DT_BF16) {
          __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + m * ld + n;
          if (p.beta != 0.f) v += p.beta * bf2f(*o);
          *o = f2bf(v);
        } else {
          float* o = reinterpret_cast<float*>(p.out) + m * ld + n;
          if (p.beta != 0.f) v += p.beta * (*o);
          *o = v;
        }
      }
    }
  }
}

int conv_fwd(const seg_conv_desc* d, const void* x, const void* w, void* y, int y_dtype, const float* bias, float beta,
             double* stats, unsigned* stat_ticket, const seg_sync_desc* sync, cudaStream_t stream) {
  SEG_REQUIRE(!stats || (y_dtype == SEG_DT_BF16 && d->K % 8 == 0 && d->ldy % 8 == 0),
              "CUDA-core conv: BatchNorm statistics need a bf16 output with K, ldy multiples of 8");
  P p;
  p.d = *d;
  p.a = (const __nv_bfloat16*)x;
  p.b = (const __nv_bfloat16*)w;
  p.out = y;
  p.out_dtype = y_dtype;
  p.beta = beta;
  p.bias = bias;
  p.stats = nullptr;
  p.M = (int64_t)d->N * d->P * d->Q;
  p.Ncols = d->K;
  p.Kdim = (int64_t)d->R * d->S * d->C;
  p.splits = 1;
  dim3 grid((unsigned)ceil_div64(p.M, TM), (unsigned)ceil_div(p.Ncols, TN), 1);
  igemm_simt<FWD><<<grid, 256, 0, stream>>>(p);
  if (check_launch("igemm_simt<FWD>")) return 1;
  // statistics of the output AS STORED, by the deterministic column reduction (same workspace contract as the wgmma path)
  if (stats) return bn_stats_launch(y, p.M, d->K, d->ldy, stats, sync, stat_ticket, stream);
  return 0;
}

int conv_dgrad(const seg_conv_desc* d, const void* dy, const void* w, void* dx, float beta, cudaStream_t stream) {
  P p;
  p.d = *d;
  p.a = (const __nv_bfloat16*)dy;
  p.b = (const __nv_bfloat16*)w;
  p.out = dx;
  p.out_dtype = SEG_DT_BF16;
  p.beta = beta;
  p.bias = nullptr;
  p.stats = nullptr;
  p.M = (int64_t)d->N * d->H * d->W;
  p.Ncols = d->C;
  p.Kdim = (int64_t)d->R * d->S * d->K;
  p.splits = 1;
  dim3 grid((unsigned)ceil_div64(p.M, TM), (unsigned)ceil_div(p.Ncols, TN), 1);
  igemm_simt<DGRAD><<<grid, 256, 0, stream>>>(p);
  return check_launch("igemm_simt<DGRAD>");
}

int conv_wgrad(const seg_conv_desc* d, const void* dy, const void* x, float* dw, cudaStream_t stream) {
  P p;
  p.d = *d;
  p.a = (const __nv_bfloat16*)dy;
  p.b = (const __nv_bfloat16*)x;
  p.out = dw;
  p.out_dtype = SEG_DT_F32;
  p.beta = 0.f;
  p.bias = nullptr;
  p.stats = nullptr;
  p.M = d->K;
  p.Ncols = d->R * d->S * d->C;
  p.Kdim = (int64_t)d->N * d->P * d->Q;
  const int tiles = ceil_div((int)p.M, TM) * ceil_div(p.Ncols, TN);
  int splits = max(1, (4 * num_sms() + tiles - 1) / tiles);
  { const int64_t kb = ceil_div64(p.Kdim, TK); if ((int64_t)splits > kb) splits = (int)kb; }
  splits = min(splits, 65535);
  p.splits = splits;
  dim3 grid((unsigned)ceil_div64(p.M, TM), (unsigned)ceil_div(p.Ncols, TN), (unsigned)splits);
  igemm_simt<WGRAD><<<grid, 256, 0, stream>>>(p);
  return check_launch("igemm_simt<WGRAD>");
}

}  // namespace simt
}  // namespace seg
