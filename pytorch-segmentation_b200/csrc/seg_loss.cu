// seg_loss.cu — per-pixel loss kernels.
//   * CrossEntropyLoss2d on the full-resolution NCHW fp32 logits the reference model returns
//     (utils/losses.py:24-31 -> nn.CrossEntropyLoss(ignore_index, reduction='mean')).
//   * the fused path: bilinear upsample (align_corners as in deeplabv3_plus.py:361 / pspnet.py:86) + log-softmax + NLL
//     (+ arg-max label map) straight from the low-resolution NHWC fp32 logits, so the 20 MB/img full-resolution logit
//     tensor never exists in HBM; backward accumulates into low-res tiles in shared memory.
#include "seg_common.cuh"

namespace seg {

__device__ __forceinline__ void block_accum2(double a, double b, double* out) {
  a = warp_sum_d(a);
  b = warp_sum_d(b);
  __shared__ double sa[32], sb[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    sa[warp] = a;
    sb[warp] = b;
  }
  __syncthreads();
  if (warp == 0) {
    const int nw = (blockDim.x + 31) >> 5;
    a = lane < nw ? sa[lane] : 0.0;
    b = lane < nw ? sb[lane] : 0.0;
    a = warp_sum_d(a);
    b = warp_sum_d(b);
    if (lane == 0) {
      atomicAdd(out, a);
      atomicAdd(out + 1, b);
    }
  }
}

__global__ void __launch_bounds__(256) ce_nchw_fwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target,
                                                          int N, int C, int H, int W, int64_t ignore, double* accum) {
  const int64_t HW = (int64_t)H * W, total = (int64_t)N * HW;
  double loss = 0.0, cnt = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = target[i];
    if (t == ignore) continue;
    const int n = (int)(i / HW);
    const float* l = logits + (int64_t)n * C * HW + (i - (int64_t)n * HW);
    float mx = -INFINITY;
    for (int c = 0; c < C; ++c) mx = fmaxf(mx, l[(int64_t)c * HW]);
    float se = 0.f;
    for (int c = 0; c < C; ++c) se += expf(l[(int64_t)c * HW] - mx);
    const float lt = (t >= 0 && t < C) ? l[t * HW] : 0.f;
    loss += (double)(mx + logf(se) - lt);
    cnt += 1.0;
  }
  block_accum2(loss, cnt, accum);
}

__global__ void __launch_bounds__(256) ce_nchw_bwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target,
                                                          int N, int C, int H, int W, int64_t ignore,
                                                          const double* __restrict__ accum, const float* __restrict__ gscale,
                                                          float* __restrict__ dl) {
  const int64_t HW = (int64_t)H * W, total = (int64_t)N * HW;
  const float g = (gscale ? *gscale : 1.f) / (float)fmax(accum[1], 1.0);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = target[i];
    const int n = (int)(i / HW);
    const int64_t off = (int64_t)n * C * HW + (i - (int64_t)n * HW);
    const float* l = logits + off;
    float* d = dl + off;
    if (t == ignore) {
      for (int c = 0; c < C; ++c) d[(int64_t)c * HW] = 0.f;
      continue;
    }
    float mx = -INFINITY;
    for (int c = 0; c < C; ++c) mx = fmaxf(mx, l[(int64_t)c * HW]);
    float se = 0.f;
    for (int c = 0; c < C; ++c) se += expf(l[(int64_t)c * HW] - mx);
    const float inv = 1.f / se;
    for (int c = 0; c < C; ++c) {
      const float p = expf(l[(int64_t)c * HW] - mx) * inv;
      d[(int64_t)c * HW] = (p - (c == t ? 1.f : 0.f)) * g;
    }
  }
}

// ---------------------------------------------------------------- Dice (utils/losses.py:33-50)
// loss = 1 - (2*I + smooth) / (sum(softmax) + sum(onehot) + smooth),  I = sum_pixels softmax[target].
// accum[0] += I, accum[1] += sum(softmax) (== #pixels up to rounding), accum[2] += #pixels (sum of the one-hot tensor).
__global__ void __launch_bounds__(256) dice_nchw_fwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target,
                                                            int N, int C, int H, int W, double* accum) {
  const int64_t HW = (int64_t)H * W, total = (int64_t)N * HW;
  double inter = 0.0, psum = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = target[i];
    const int n = (int)(i / HW);
    const float* l = logits + (int64_t)n * C * HW + (i - (int64_t)n * HW);
    float mx = -INFINITY;
    for (int c = 0; c < C; ++c) mx = fmaxf(mx, l[(int64_t)c * HW]);
    float se = 0.f, et = 0.f;
    for (int c = 0; c < C; ++c) {
      const float e = expf(l[(int64_t)c * HW] - mx);
      se += e;
      if (c == t) et = e;
    }
    inter += (double)(et / se);
    psum += 1.0;
  }
  block_accum2(inter, psum, accum);
}

// d loss / d logit_c = -(2 / D) * p_t * (delta_ct - p_c),  D = accum[1] + accum[2] + smooth
__global__ void __launch_bounds__(256) dice_nchw_bwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target,
                                                            int N, int C, int H, int W, const double* __restrict__ accum,
                                                            float smooth, const float* __restrict__ gscale,
                                                            float* __restrict__ dl, float beta) {
  const int64_t HW = (int64_t)H * W, total = (int64_t)N * HW;
  const double I = accum[0], P = accum[1], T = accum[1];
  const double D = P + T + (double)smooth;
  // d/dp_t of -(2I+s)/D with D depending on sum(p): the sum(p) term has zero gradient through softmax (rows sum to 1)
  const float g = (gscale ? *gscale : 1.f) * (float)(-2.0 / D);
  (void)I;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = target[i];
    const int n = (int)(i / HW);
    const int64_t off = (int64_t)n * C * HW + (i - (int64_t)n * HW);
    const float* l = logits + off;
    float* d = dl + off;
    float mx = -INFINITY;
    for (int c = 0; c < C; ++c) mx = fmaxf(mx, l[(int64_t)c * HW]);
    float se = 0.f;
    for (int c = 0; c < C; ++c) se += expf(l[(int64_t)c * HW] - mx);
    const float inv = 1.f / se;
    const float pt = (t >= 0 && t < C) ? expf(l[t * HW] - mx) * inv : 0.f;
    for (int c = 0; c < C; ++c) {
      const float pc = expf(l[(int64_t)c * HW] - mx) * inv;
      const float v = g * pt * ((c == t ? 1.f : 0.f) - pc);
      d[(int64_t)c * HW] = (beta != 0.f) ? beta * d[(int64_t)c * HW] + v : v;
    }
  }
}

__global__ void dice_finalize_kernel(const double* accum, float smooth, float* loss) {
  if (threadIdx.x == 0 && blockIdx.x == 0)
    *loss = (float)(1.0 - (2.0 * accum[0] + smooth) / (accum[1] + accum[1] + smooth));
}

__global__ void ce_finalize_kernel(const double* accum, float* loss) {
  if (threadIdx.x == 0 && blockIdx.x == 0) *loss = (float)(accum[0] / fmax(accum[1], 1.0));
}

// ---------------------------------------------------------------- fused upsample + CE
struct Lerp2 {
  int i0, i1;
  float l1;
};
__device__ __forceinline__ Lerp2 src_idx(int dst, float scale, int in_size, int ac) {
  float s;
  if (ac) {
    s = scale * (float)dst;
  } else {
    s = scale * ((float)dst + 0.5f) - 0.5f;
    if (s < 0.f) s = 0.f;
  }
  Lerp2 r;
  r.i0 = (int)s;
  if (r.i0 > in_size - 1) r.i0 = in_size - 1;
  r.i1 = r.i0 + ((r.i0 < in_size - 1) ? 1 : 0);
  r.l1 = s - (float)r.i0;
  return r;
}
static inline float rscale(int in_size, int out_size, int ac) {
  if (ac) return out_size > 1 ? (float)(in_size - 1) / (float)(out_size - 1) : 0.f;
  return (float)in_size / (float)out_size;
}

constexpr int MAXC = 160;  // classes supported by the fused kernel (19 / 21 / 150 on the configs)
constexpr int TILE = 32;   // output tile edge (the backward halves it when the 32 x 32 tile's patch does not fit in shared memory)

// The backward accumulates the logits gradient in 64-bit fixed point: integer additions are associative, so the result
// does not depend on the order in which threads and blocks add their contributions (fp32 atomics did).  Every contribution
// is at most |g| in magnitude and the interpolation weights reaching one low-res element sum to less than
// (2/sh + 2)(2/sw + 2), so with that bound below 2^e the scale 2^(61-e) cannot overflow; a contribution is rounded to
// |bound| * 2^-62, far below the fp32 rounding of the result.
__device__ __forceinline__ double ce_grad_scale(float g, float sh, float sw, int Ho, int Wo) {
  const double ry = sh > 0.f ? 2.0 / sh : (double)Ho, rx = sw > 0.f ? 2.0 / sw : (double)Wo;
  int e;
  frexp(fabs((double)g) * (ry + 2.0) * (rx + 2.0), &e);
  return ldexp(1.0, 61 - e);
}
__device__ __forceinline__ float ce_grad_g(const float* gscale, const double* accum) {
  return (gscale ? *gscale : 1.f) / (float)fmax(accum[1], 1.0);
}
__device__ __forceinline__ unsigned long long to_fixed(float v, double scale) {
  return (unsigned long long)__double2ll_rn((double)v * scale);
}

// one block = one 32x32 output tile; the low-res source patch (<= PATCH x PATCH pixels x C) is staged in smem
template <bool BWD>
__global__ void __launch_bounds__(256) upsample_ce_kernel(const float* __restrict__ lo, const int64_t* __restrict__ target,
                                                          int N, int Hi, int Wi, int Ho, int Wo, int C, int ac, float sh,
                                                          float sw, int64_t ignore, double* accum, int32_t* argmax,
                                                          const float* __restrict__ gscale,
                                                          unsigned long long* __restrict__ dlo_fixed, int patch, int tile) {
  extern __shared__ unsigned long long sm64[];
  unsigned long long* dst = BWD ? sm64 : nullptr;  // [patch*patch][C] fixed-point grad accumulators
  float* src = reinterpret_cast<float*>(BWD ? sm64 + patch * patch * C : sm64);  // [patch*patch][C]
  const int tiles_x = (Wo + tile - 1) / tile, tiles_y = (Ho + tile - 1) / tile;
  int t = blockIdx.x;
  const int tx = t % tiles_x;
  t /= tiles_x;
  const int ty = t % tiles_y;
  const int n = t / tiles_y;
  const int oy0 = ty * tile, ox0 = tx * tile;
  const int oy1 = min(oy0 + tile, Ho) - 1, ox1 = min(ox0 + tile, Wo) - 1;
  const int sy0 = src_idx(oy0, sh, Hi, ac).i0, sx0 = src_idx(ox0, sw, Wi, ac).i0;
  const int sy1 = src_idx(oy1, sh, Hi, ac).i1, sx1 = src_idx(ox1, sw, Wi, ac).i1;
  const int ph = sy1 - sy0 + 1, pw = sx1 - sx0 + 1;  // <= patch by construction (checked on host)
  for (int i = threadIdx.x; i < ph * pw * C; i += blockDim.x) {
    const int c = i % C;
    const int pp = i / C;
    const int py = pp / pw, px = pp - py * pw;
    src[i] = lo[(((int64_t)n * Hi + sy0 + py) * Wi + sx0 + px) * C + c];
    if (BWD) dst[i] = 0ull;
  }
  __syncthreads();
  double loss = 0.0, cnt = 0.0;
  float g = 0.f;
  double scale = 0.0;
  if (BWD) {
    g = ce_grad_g(gscale, accum);
    scale = ce_grad_scale(g, sh, sw, Ho, Wo);
  }
  for (int e = threadIdx.x; e < tile * tile; e += blockDim.x) {
    const int oy = oy0 + e / tile, ox = ox0 + e % tile;
    if (oy >= Ho || ox >= Wo) continue;
    const int64_t tg = target[((int64_t)n * Ho + oy) * Wo + ox];
    const bool valid = tg != ignore;
    if (!valid && (BWD || argmax == nullptr)) continue;
    const Lerp2 ly = src_idx(oy, sh, Hi, ac), lx = src_idx(ox, sw, Wi, ac);
    const float h1 = ly.l1, h0 = 1.f - h1, w1 = lx.l1, w0 = 1.f - w1;
    const float* pa = src + ((ly.i0 - sy0) * pw + (lx.i0 - sx0)) * C;
    const float* pb = src + ((ly.i0 - sy0) * pw + (lx.i1 - sx0)) * C;
    const float* pc = src + ((ly.i1 - sy0) * pw + (lx.i0 - sx0)) * C;
    const float* pd = src + ((ly.i1 - sy0) * pw + (lx.i1 - sx0)) * C;
    float mx = -INFINITY;
    int am = 0;
    for (int c = 0; c < C; ++c) {
      const float v = h0 * (w0 * pa[c] + w1 * pb[c]) + h1 * (w0 * pc[c] + w1 * pd[c]);
      if (v > mx) {
        mx = v;
        am = c;
      }
    }
    float se = 0.f, lt = 0.f;
    for (int c = 0; c < C; ++c) {
      const float v = h0 * (w0 * pa[c] + w1 * pb[c]) + h1 * (w0 * pc[c] + w1 * pd[c]);
      se += expf(v - mx);
      if (c == tg) lt = v;
    }
    if (!BWD) {
      if (argmax) argmax[((int64_t)n * Ho + oy) * Wo + ox] = am;
      if (valid) {
        loss += (double)(mx + logf(se) - lt);
        cnt += 1.0;
      }
    } else {
      const float inv = 1.f / se;
      unsigned long long* da = dst + ((ly.i0 - sy0) * pw + (lx.i0 - sx0)) * C;
      unsigned long long* db = dst + ((ly.i0 - sy0) * pw + (lx.i1 - sx0)) * C;
      unsigned long long* dc = dst + ((ly.i1 - sy0) * pw + (lx.i0 - sx0)) * C;
      unsigned long long* dd = dst + ((ly.i1 - sy0) * pw + (lx.i1 - sx0)) * C;
      for (int c = 0; c < C; ++c) {
        const float v = h0 * (w0 * pa[c] + w1 * pb[c]) + h1 * (w0 * pc[c] + w1 * pd[c]);
        const float gr = (expf(v - mx) * inv - (c == tg ? 1.f : 0.f)) * g;
        atomicAdd(da + c, to_fixed(h0 * w0 * gr, scale));
        atomicAdd(db + c, to_fixed(h0 * w1 * gr, scale));
        atomicAdd(dc + c, to_fixed(h1 * w0 * gr, scale));
        atomicAdd(dd + c, to_fixed(h1 * w1 * gr, scale));
      }
    }
  }
  if (!BWD) {
    block_accum2(loss, cnt, accum);
  } else {
    __syncthreads();
    for (int i = threadIdx.x; i < ph * pw * C; i += blockDim.x) {
      const unsigned long long v = dst[i];
      if (v != 0ull) {
        const int c = i % C;
        const int pp = i / C;
        const int py = pp / pw, px = pp - py * pw;
        atomicAdd(dlo_fixed + (((int64_t)n * Hi + sy0 + py) * Wi + sx0 + px) * C + c, v);
      }
    }
  }
}

// fixed-point accumulators -> fp32 gradient (the scale is recomputed exactly as the accumulating kernel did)
__global__ void ce_grad_from_fixed_kernel(const unsigned long long* __restrict__ acc, int64_t n, const float* gscale,
                                          const double* accum, float sh, float sw, int Ho, int Wo, float* __restrict__ dlo) {
  const double inv = 1.0 / ce_grad_scale(ce_grad_g(gscale, accum), sh, sw, Ho, Wo);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dlo[i] = (float)((double)(long long)acc[i] * inv);
}

__global__ void cast_pad_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, int64_t M, int C, int ld) {
  const int64_t total = M * ld;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % ld);
    const int64_t r = i / ld;
    y[i] = f2bf(c < C ? x[r * C + c] : 0.f);
  }
}

static int patch_for(int in_size, int out_size, int ac, int tile) {
  // upper bound on low-res rows touched by `tile` consecutive output rows
  const float sc = rscale(in_size, out_size, ac);
  int p = (int)ceilf(sc * (tile - 1)) + 3;
  return p < in_size + 1 ? p : in_size + 1;
}

}  // namespace seg

using namespace seg;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int seg_ce_nchw_fwd(const float* logits, const int64_t* target, int N, int C, int H, int W, int64_t ignore_index,
                    double* accum, void* stream) {
  const int64_t total = (int64_t)N * H * W;
  int blocks = (int)std::min<int64_t>(ceil_div64(total, 256), (int64_t)num_sms() * 8);
  ce_nchw_fwd_kernel<<<blocks, 256, 0, ST(stream)>>>(logits, target, N, C, H, W, ignore_index, accum);
  return check_launch("ce_nchw_fwd");
}
int seg_ce_nchw_bwd(const float* logits, const int64_t* target, int N, int C, int H, int W, int64_t ignore_index,
                    const double* accum, const float* gscale, float* dlogits, void* stream) {
  const int64_t total = (int64_t)N * H * W;
  int blocks = (int)std::min<int64_t>(ceil_div64(total, 256), (int64_t)num_sms() * 8);
  ce_nchw_bwd_kernel<<<blocks, 256, 0, ST(stream)>>>(logits, target, N, C, H, W, ignore_index, accum, gscale, dlogits);
  return check_launch("ce_nchw_bwd");
}
int seg_dice_nchw_fwd(const float* logits, const int64_t* target, int N, int C, int H, int W, float smooth, double* accum,
                      float* loss, void* stream) {
  const int64_t total = (int64_t)N * H * W;
  int blocks = (int)std::min<int64_t>(ceil_div64(total, 256), (int64_t)num_sms() * 8);
  dice_nchw_fwd_kernel<<<blocks, 256, 0, ST(stream)>>>(logits, target, N, C, H, W, accum);
  if (check_launch("dice_nchw_fwd")) return 1;
  dice_finalize_kernel<<<1, 32, 0, ST(stream)>>>(accum, smooth, loss);
  return check_launch("dice_finalize");
}
int seg_dice_nchw_bwd(const float* logits, const int64_t* target, int N, int C, int H, int W, const double* accum,
                      float smooth, const float* gscale, float* dlogits, float beta, void* stream) {
  const int64_t total = (int64_t)N * H * W;
  int blocks = (int)std::min<int64_t>(ceil_div64(total, 256), (int64_t)num_sms() * 8);
  dice_nchw_bwd_kernel<<<blocks, 256, 0, ST(stream)>>>(logits, target, N, C, H, W, accum, smooth, gscale, dlogits, beta);
  return check_launch("dice_nchw_bwd");
}
int seg_ce_finalize(const double* accum, float* loss, void* stream) {
  ce_finalize_kernel<<<1, 32, 0, ST(stream)>>>(accum, loss);
  return check_launch("ce_finalize");
}

int seg_upsample_ce_fwd(const float* logits_lo, const int64_t* target, int N, int Hi, int Wi, int Ho, int Wo, int C,
                        int align_corners, int64_t ignore_index, double* accum, int32_t* argmax, void* stream) {
  SEG_REQUIRE(C <= MAXC, "upsample_ce: C=%d > %d", C, MAXC);
  const int patch = std::max(patch_for(Hi, Ho, align_corners, TILE), patch_for(Wi, Wo, align_corners, TILE));
  const size_t smem = (size_t)patch * patch * C * sizeof(float);
  SEG_REQUIRE(smem <= 200 * 1024, "upsample_ce: patch too large (%zu B)", smem);
  static size_t set_smem = 0;
  if (smem > set_smem) {
    cudaFuncSetAttribute(upsample_ce_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    set_smem = smem;
  }
  const int blocks = N * ceil_div(Ho, TILE) * ceil_div(Wo, TILE);
  upsample_ce_kernel<false><<<blocks, 256, smem, ST(stream)>>>(
      logits_lo, target, N, Hi, Wi, Ho, Wo, C, align_corners, rscale(Hi, Ho, align_corners), rscale(Wi, Wo, align_corners),
      ignore_index, accum, argmax, nullptr, nullptr, patch, TILE);
  return check_launch("upsample_ce_fwd");
}

// dlo_f32: fp32 [N,Hi,Wi,C]; dlo_fixed: int64 scratch [N,Hi,Wi,C] (zeroed here); dx: bf16 [N*Hi*Wi][lddx] or NULL
int seg_upsample_ce_bwd(const float* logits_lo, const int64_t* target, int N, int Hi, int Wi, int Ho, int Wo, int C,
                        int align_corners, int64_t ignore_index, const double* accum, const float* gscale,
                        float* dlo_f32, void* dlo_fixed, void* dx, int lddx, void* stream) {
  SEG_REQUIRE(C <= MAXC, "upsample_ce: C=%d > %d", C, MAXC);
  // fixed-point accumulators (8 B) + the fp32 source patch per (patch pixel, class)
  auto bwd_patch = [&](int t) { return std::max(patch_for(Hi, Ho, align_corners, t), patch_for(Wi, Wo, align_corners, t)); };
  auto bwd_smem = [&](int t) { return (size_t)bwd_patch(t) * bwd_patch(t) * C * (sizeof(unsigned long long) + sizeof(float)); };
  const int tile = bwd_smem(TILE) <= 227 * 1024 ? TILE : TILE / 2;
  const int patch = bwd_patch(tile);
  const size_t smem = bwd_smem(tile);
  SEG_REQUIRE(smem <= 227 * 1024, "upsample_ce: patch too large (%zu B)", smem);
  static size_t set_smem = 0;
  if (smem > set_smem) {
    cudaFuncSetAttribute(upsample_ce_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    set_smem = smem;
  }
  const int64_t M = (int64_t)N * Hi * Wi;
  unsigned long long* fixed = reinterpret_cast<unsigned long long*>(dlo_fixed);
  cudaMemsetAsync(fixed, 0, (size_t)M * C * sizeof(unsigned long long), ST(stream));
  const int blocks = N * ceil_div(Ho, tile) * ceil_div(Wo, tile);
  const float sh = rscale(Hi, Ho, align_corners), sw = rscale(Wi, Wo, align_corners);
  upsample_ce_kernel<true><<<blocks, 256, smem, ST(stream)>>>(
      logits_lo, target, N, Hi, Wi, Ho, Wo, C, align_corners, sh, sw, ignore_index, const_cast<double*>(accum), nullptr, gscale,
      fixed, patch, tile);
  if (check_launch("upsample_ce_bwd")) return 1;
  const int64_t n = M * C;
  ce_grad_from_fixed_kernel<<<(unsigned)std::min<int64_t>(ceil_div64(n, 256), (int64_t)num_sms() * 8), 256, 0, ST(stream)>>>(
      fixed, n, gscale, accum, sh, sw, Ho, Wo, dlo_f32);
  if (check_launch("ce_grad_from_fixed")) return 1;
  if (dx) {
    int blocks2 = (int)std::min<int64_t>(ceil_div64(M * lddx, 256), (int64_t)num_sms() * 8);
    cast_pad_kernel<<<blocks2, 256, 0, ST(stream)>>>(dlo_f32, reinterpret_cast<__nv_bfloat16*>(dx), M, C, lddx);
    return check_launch("cast_pad");
  }
  return 0;
}

}  // extern "C"

// ------------------------------------------------------------------ eval_metrics (utils/metrics.py:42-67)
// One pass over the NCHW fp32 logits: per-pixel argmax, pixel accuracy and the per-class histograms the reference gets
// from three torch.histc calls — integer counters, bit-exact.  out (int64, pre-zeroed by the entry point):
//   [0] correct  [1] labeled  [2 .. 2+K) area_inter  [2+K .. 2+2K) area_pred  [2+2K .. 2+3K) area_lab      (K = num_class)
namespace seg {
__global__ void __launch_bounds__(256)
    eval_metrics_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target, int N, int C, int64_t HW, int K,
                        unsigned long long* __restrict__ out) {
  extern __shared__ unsigned int hist[];  // [3][K] + correct + labeled
  for (int i = threadIdx.x; i < 3 * K + 2; i += blockDim.x) hist[i] = 0u;
  __syncthreads();
  const int64_t total = (int64_t)N * HW;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = target[i];
    if (t < 0 || t >= K) continue;  // labeled = (target+1 > 0) & (target+1 <= num_class)
    const int n = (int)(i / HW);
    const float* l = logits + (int64_t)n * C * HW + (i - (int64_t)n * HW);
    float best = l[0];
    int arg = 0;
    for (int c = 1; c < C; ++c) {
      const float v = l[(int64_t)c * HW];
      if (v > best) {  // first maximum wins, like torch.max
        best = v;
        arg = c;
      }
    }
    atomicAdd(&hist[3 * K + 1], 1u);
    if (arg < K) atomicAdd(&hist[K + arg], 1u);  // area_pred (histc range [1, K] on predict+1)
    atomicAdd(&hist[2 * K + (int)t], 1u);         // area_lab
    if (arg == (int)t) {
      atomicAdd(&hist[3 * K], 1u);
      atomicAdd(&hist[(int)t], 1u);  // area_inter
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * K + 2; i += blockDim.x) {
    const unsigned int v = hist[i];
    if (v == 0u) continue;
    const int dst = (i == 3 * K) ? 0 : (i == 3 * K + 1) ? 1 : 2 + i;
    atomicAdd(out + dst, (unsigned long long)v);
  }
}
}  // namespace seg

extern "C" int seg_eval_metrics_nchw(const float* logits, const int64_t* target, int N, int C, int H, int W, int num_class,
                                     int64_t* out, void* stream) {
  using namespace seg;
  SEG_REQUIRE(N > 0 && C > 0 && num_class > 0 && num_class <= 4096, "eval_metrics: bad sizes (C=%d num_class=%d)", C, num_class);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  cudaMemsetAsync(out, 0, (size_t)(2 + 3 * num_class) * sizeof(int64_t), st);
  const int64_t HW = (int64_t)H * W, total = (int64_t)N * HW;
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = (int64_t)num_sms() * 8;
  if (blocks > cap) blocks = cap;
  eval_metrics_kernel<<<(unsigned)blocks, 256, (size_t)(3 * num_class + 2) * sizeof(unsigned int), st>>>(
      logits, target, N, C, HW, num_class, reinterpret_cast<unsigned long long*>(out));
  return check_launch("eval_metrics");
}
