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

// Per-pixel loss variants (utils/losses.py:24-31,52-65,67-77).  With nll = lse(z) - z_t at a pixel labelled t:
//   LOSS_CE     nll                       denominator: valid pixels      (unweighted mean CE)
//   LOSS_WCE    L = w_t * nll             denominator: sum of valid w_t  (nn.CrossEntropyLoss(weight); w = 1 without one)
//   LOSS_FOCAL  (1 - pt)^gamma * L, pt = exp(-L)   denominator: every pixel, ignored ones included (FocalLoss's .mean())
// accum[1] holds the denominator; the 'sum' reductions ignore it.  dL/dz_c = w_t (p_c - delta_ct) F'(L) with the focal
// factor F'(L) = u^gamma (1 + gamma r), u = -expm1(-L), r = L / expm1(L) (r = 1 at L = 0): u and r lie in [0, 1], so
// 0 <= F' <= 1 + gamma, and no 0 * inf is formed where pt rounds to 1 (F' -> 0 there for gamma > 0).
enum LossKind { LOSS_CE = SEG_LOSS_CE, LOSS_WCE = SEG_LOSS_WCE, LOSS_FOCAL = SEG_LOSS_FOCAL };
struct LossArgs {
  const float* weight;  // fp32 [C] (finite, >= 0) or NULL = all ones; unused by LOSS_CE
  float gamma;          // LOSS_FOCAL only
  int mean;             // 1: divide by accum[1]; 0: 'sum' / size_average=False
};

__device__ __forceinline__ float class_weight(const LossArgs& a, int64_t t, int C) {
  return a.weight ? ((t >= 0 && t < C) ? a.weight[t] : 0.f) : 1.f;
}
template <int K>
__device__ __forceinline__ float pixel_loss(float nll, float w, float gamma) {
  if (K == LOSS_CE) return nll;
  const float L = w * nll;
  if (K == LOSS_WCE) return L;
  return powf(-expm1f(-L), gamma) * L;
}
// the factor w_t F'(L) the softmax gradient (p - onehot) of a pixel is multiplied by
template <int K>
__device__ __forceinline__ float pixel_grad_factor(float nll, float w, float gamma) {
  if (K != LOSS_FOCAL) return w;
  const float L = w * nll;
  const float r = L > 0.f ? L / expm1f(L) : 1.f;
  return w * powf(-expm1f(-L), gamma) * (1.f + gamma * r);
}
// d loss / d (per-pixel loss sum): gscale / accum[1] for a mean.  A weighted or focal mean with accum[1] == 0 (nothing
// valid, or only zero-weight classes present) has loss 0 and gradient 0; accum[1] < 1 is legitimate there.
template <int K>
__device__ __forceinline__ float loss_grad_g(const float* gscale, const double* accum, int mean) {
  const float gs = gscale ? *gscale : 1.f;
  if (K == LOSS_CE) return gs / (float)fmax(accum[1], 1.0);
  if (!mean) return gs;
  return accum[1] > 0.0 ? (float)((double)gs / accum[1]) : 0.f;
}

template <int K>
__global__ void __launch_bounds__(256) ce_nchw_fwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target,
                                                          int N, int C, int H, int W, int64_t ignore, LossArgs la, double* accum) {
  const int64_t HW = (int64_t)H * W, total = (int64_t)N * HW;
  double loss = 0.0, cnt = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = target[i];
    if (K == LOSS_FOCAL) cnt += 1.0;
    if (t == ignore) continue;
    const int n = (int)(i / HW);
    const float* l = logits + (int64_t)n * C * HW + (i - (int64_t)n * HW);
    float mx = -INFINITY;
    for (int c = 0; c < C; ++c) mx = fmaxf(mx, l[(int64_t)c * HW]);
    float se = 0.f;
    for (int c = 0; c < C; ++c) se += expf(l[(int64_t)c * HW] - mx);
    const float lt = (t >= 0 && t < C) ? l[t * HW] : 0.f;
    const float w = K == LOSS_CE ? 1.f : class_weight(la, t, C);
    loss += (double)pixel_loss<K>(mx + logf(se) - lt, w, la.gamma);
    if (K == LOSS_CE) cnt += 1.0;
    if (K == LOSS_WCE) cnt += (double)w;
  }
  block_accum2(loss, cnt, accum);
}

template <int K>
__global__ void __launch_bounds__(256) ce_nchw_bwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target,
                                                          int N, int C, int H, int W, int64_t ignore, LossArgs la,
                                                          const double* __restrict__ accum, const float* __restrict__ gscale,
                                                          float* __restrict__ dl) {
  const int64_t HW = (int64_t)H * W, total = (int64_t)N * HW;
  const float g = loss_grad_g<K>(gscale, accum, la.mean);
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
    float gp = g;
    if (K != LOSS_CE) {
      const float lt = (t >= 0 && t < C) ? l[t * HW] : 0.f;
      gp = g * pixel_grad_factor<K>(mx + logf(se) - lt, class_weight(la, t, C), la.gamma);
    }
    for (int c = 0; c < C; ++c) {
      const float p = expf(l[(int64_t)c * HW] - mx) * inv;
      d[(int64_t)c * HW] = (p - (c == t ? 1.f : 0.f)) * gp;
    }
  }
}

// ---------------------------------------------------------------- Dice (utils/losses.py:33-50)
// loss = 1 - (2*I + smooth) / (sum(softmax) + sum(onehot) + smooth),  I = sum_pixels softmax[target].
// accum[0] += I, accum[1] += #pixels.  Every softmax row sums to 1 and every pixel carries one label after the target
// fix-up, so sum(softmax) and sum(onehot) both equal #pixels and D = 2 accum[1] + smooth (to within the softmax rounding).
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

// d loss / d logit_c = -(2 / D) * p_t * (delta_ct - p_c),  D = 2 accum[1] + smooth (see dice_nchw_fwd_kernel)
__global__ void __launch_bounds__(256) dice_nchw_bwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target,
                                                            int N, int C, int H, int W, const double* __restrict__ accum,
                                                            float smooth, const float* __restrict__ gscale,
                                                            float* __restrict__ dl, float beta) {
  const int64_t HW = (int64_t)H * W, total = (int64_t)N * HW;
  const double D = accum[1] + accum[1] + (double)smooth;
  // d/dp_t of -(2I+s)/D with D depending on sum(p): the sum(p) term has zero gradient through softmax (rows sum to 1)
  const float g = (gscale ? *gscale : 1.f) * (float)(-2.0 / D);
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

// a mean with a zero denominator is 0 (see loss_grad_g); a sum is accum[0]
// LOSS_CE (mean): accum[1] is an integer count and accum[0] is +0.0 when it is 0, so this equals accum[0] / fmax(accum[1], 1)
__global__ void loss_finalize_kernel(const double* accum, int mean, float* loss) {
  if (threadIdx.x == 0 && blockIdx.x == 0) *loss = (float)(!mean ? accum[0] : accum[1] > 0.0 ? accum[0] / accum[1] : 0.0);
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
// is at most gmax = |g| * max(w) * (1 + gamma) in magnitude (|p_c - delta_ct| <= 1, w_t <= max(w), 0 <= F' <= 1 + gamma;
// unweighted CE: gmax = |g|) and the interpolation weights reaching one low-res element sum to less than
// (2/sh + 2)(2/sw + 2), so with that bound below 2^e the scale 2^(61-e) cannot overflow; a contribution is rounded to
// |bound| * 2^-62, far below the fp32 rounding of the result.
__device__ __forceinline__ double ce_grad_scale(double gmax, float sh, float sw, int Ho, int Wo) {
  const double ry = sh > 0.f ? 2.0 / sh : (double)Ho, rx = sw > 0.f ? 2.0 / sw : (double)Wo;
  int e;
  frexp(fabs(gmax) * (ry + 2.0) * (rx + 2.0), &e);
  return ldexp(1.0, 61 - e);
}
// max over the class weights (1 without weights), on every lane of the calling warp (all 32 lanes must be active)
__device__ __forceinline__ float warp_weight_max(const float* w, int C) {
  float m = w ? 0.f : 1.f;
  if (w)
    for (int c = threadIdx.x & 31; c < C; c += 32) m = fmaxf(m, w[c]);
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  return m;
}
template <int K>
__device__ __forceinline__ double loss_grad_bound(float g, const LossArgs& la, int C) {
  if (K == LOSS_CE) return (double)g;
  return (double)g * (double)warp_weight_max(la.weight, C) * (K == LOSS_FOCAL ? 1.0 + (double)la.gamma : 1.0);
}
__device__ __forceinline__ unsigned long long to_fixed(float v, double scale) {
  return (unsigned long long)__double2ll_rn((double)v * scale);
}

// one block = one 32x32 output tile; the low-res source patch (<= PATCH x PATCH pixels x C) is staged in smem.
// MET (forward only): also add the eval_metrics counters of the tile (utils/metrics.py:42-67, as eval_metrics_kernel
// counts them) into counters = int64 [2 + 3C]: correct, labeled, inter[C], pred[C], lab[C].  "Labeled" is 0 <= t < C,
// whatever the loss's ignore_index; the prediction is the arg-max of the same interpolated fp32 values the loss uses
// (first maximum wins).  The block counts into a shared-memory histogram behind the source patch and flushes it with one
// global atomic per non-zero bin: integer sums, so the counters do not depend on the order of the blocks.
template <bool BWD, int K, bool MET = false>
__global__ void __launch_bounds__(256) upsample_ce_kernel(const float* __restrict__ lo, const int64_t* __restrict__ target,
                                                          int N, int Hi, int Wi, int Ho, int Wo, int C, int ac, float sh,
                                                          float sw, int64_t ignore, LossArgs la, double* accum, int32_t* argmax,
                                                          const float* __restrict__ gscale,
                                                          unsigned long long* __restrict__ dlo_fixed, int patch, int tile,
                                                          unsigned long long* __restrict__ counters) {
  extern __shared__ unsigned long long sm64[];
  unsigned long long* dst = BWD ? sm64 : nullptr;  // [patch*patch][C] fixed-point grad accumulators
  float* src = reinterpret_cast<float*>(BWD ? sm64 + patch * patch * C : sm64);  // [patch*patch][C]
  unsigned int* hist = MET ? reinterpret_cast<unsigned int*>(src + patch * patch * C) : nullptr;  // [2 + 3C], as counters
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
  if (MET)
    for (int i = threadIdx.x; i < 3 * C + 2; i += blockDim.x) hist[i] = 0u;
  __syncthreads();
  double loss = 0.0, cnt = 0.0;
  unsigned int n_correct = 0u, n_labeled = 0u;
  float g = 0.f;
  double scale = 0.0;
  if (BWD) {
    g = loss_grad_g<K>(gscale, accum, la.mean);
    scale = ce_grad_scale(loss_grad_bound<K>(g, la, C), sh, sw, Ho, Wo);
  }
  for (int e = threadIdx.x; e < tile * tile; e += blockDim.x) {
    const int oy = oy0 + e / tile, ox = ox0 + e % tile;
    if (oy >= Ho || ox >= Wo) continue;
    const int64_t tg = target[((int64_t)n * Ho + oy) * Wo + ox];
    const bool valid = tg != ignore;
    const bool labeled = MET && tg >= 0 && tg < C;
    if (K == LOSS_FOCAL && !BWD) cnt += 1.0;
    if (!valid && (BWD || (argmax == nullptr && !labeled))) continue;
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
      if (MET && labeled) {
        ++n_labeled;
        atomicAdd(&hist[2 + C + am], 1u);          // area_pred
        atomicAdd(&hist[2 + 2 * C + (int)tg], 1u);  // area_lab
        if (am == (int)tg) {
          ++n_correct;
          atomicAdd(&hist[2 + (int)tg], 1u);  // area_inter
        }
      }
      if (valid) {
        const float w = K == LOSS_CE ? 1.f : class_weight(la, tg, C);
        loss += (double)pixel_loss<K>(mx + logf(se) - lt, w, la.gamma);
        if (K == LOSS_CE) cnt += 1.0;
        if (K == LOSS_WCE) cnt += (double)w;
      }
    } else {
      const float inv = 1.f / se;
      const float gp = K == LOSS_CE ? g : g * pixel_grad_factor<K>(mx + logf(se) - lt, class_weight(la, tg, C), la.gamma);
      unsigned long long* da = dst + ((ly.i0 - sy0) * pw + (lx.i0 - sx0)) * C;
      unsigned long long* db = dst + ((ly.i0 - sy0) * pw + (lx.i1 - sx0)) * C;
      unsigned long long* dc = dst + ((ly.i1 - sy0) * pw + (lx.i0 - sx0)) * C;
      unsigned long long* dd = dst + ((ly.i1 - sy0) * pw + (lx.i1 - sx0)) * C;
      for (int c = 0; c < C; ++c) {
        const float v = h0 * (w0 * pa[c] + w1 * pb[c]) + h1 * (w0 * pc[c] + w1 * pd[c]);
        const float gr = (expf(v - mx) * inv - (c == tg ? 1.f : 0.f)) * gp;
        atomicAdd(da + c, to_fixed(h0 * w0 * gr, scale));
        atomicAdd(db + c, to_fixed(h0 * w1 * gr, scale));
        atomicAdd(dc + c, to_fixed(h1 * w0 * gr, scale));
        atomicAdd(dd + c, to_fixed(h1 * w1 * gr, scale));
      }
    }
  }
  if (!BWD) {
    block_accum2(loss, cnt, accum);
    if (MET) {
      n_correct = __reduce_add_sync(0xffffffffu, n_correct);
      n_labeled = __reduce_add_sync(0xffffffffu, n_labeled);
      if ((threadIdx.x & 31) == 0) {
        atomicAdd(&hist[0], n_correct);
        atomicAdd(&hist[1], n_labeled);
      }
      __syncthreads();
      for (int i = threadIdx.x; i < 3 * C + 2; i += blockDim.x) {
        const unsigned int v = hist[i];
        if (v != 0u) atomicAdd(counters + i, (unsigned long long)v);
      }
    }
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
template <int K>
__global__ void ce_grad_from_fixed_kernel(const unsigned long long* __restrict__ acc, int64_t n, const float* gscale,
                                          const double* accum, LossArgs la, int C, float sh, float sw, int Ho, int Wo,
                                          float* __restrict__ dlo) {
  const double inv = 1.0 / ce_grad_scale(loss_grad_bound<K>(loss_grad_g<K>(gscale, accum, la.mean), la, C), sh, sw, Ho, Wo);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dlo[i] = (float)((double)(long long)acc[i] * inv);
}

// ---------------------------------------------------------------- fused pixel shuffle + loss (duc_hdc.py:30,233)
// The logits of full-resolution pixel (oy, ox) are read in place from the low-resolution bf16 map as its nn.PixelShuffle(r)
// view: class c sits at channel c*r*r + (oy % r)*r + ox % r of low-res pixel (oy / r, ox / r).  One thread per pixel.  Every
// low-res element belongs to exactly one pixel, so the backward writes each gradient element once (no accumulation: the
// result does not depend on the thread order) and zeroes the pad lanes r*r*C .. lddx-1.  MET: the eval_metrics counters,
// counted as upsample_ce_kernel counts them (shared-memory histogram, one global atomic per non-zero bin).
// T: the storage type of the map — bf16 for DUC_HDC's shuffle; fp32 at r = 1 for full-resolution NHWC logits (UNetResnet).
__device__ __forceinline__ float logit_f(__nv_bfloat16 v) { return bf2f(v); }
__device__ __forceinline__ float logit_f(float v) { return v; }
template <bool BWD, int K, bool MET = false, typename T = __nv_bfloat16>
__global__ void __launch_bounds__(256) shuffle_ce_kernel(const T* __restrict__ lo, int ldlo,
                                                         const int64_t* __restrict__ target, int N, int h, int w, int C, int r,
                                                         int64_t ignore, LossArgs la, double* accum,
                                                         const float* __restrict__ gscale, __nv_bfloat16* __restrict__ dx,
                                                         int lddx, unsigned long long* __restrict__ counters) {
  extern __shared__ unsigned int hist[];  // MET: [2 + 3C], as counters
  if (MET) {
    for (int i = threadIdx.x; i < 3 * C + 2; i += blockDim.x) hist[i] = 0u;
    __syncthreads();
  }
  const int Ho = h * r, Wo = w * r, rr = r * r;
  const int64_t total = (int64_t)N * Ho * Wo;
  double loss = 0.0, cnt = 0.0;
  unsigned int n_correct = 0u, n_labeled = 0u;
  const float g = BWD ? loss_grad_g<K>(gscale, accum, la.mean) : 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ox = (int)(i % Wo);
    const int64_t t = i / Wo;
    const int oy = (int)(t % Ho);
    const int n = (int)(t / Ho);
    const int64_t tg = target[i];
    const bool valid = tg != ignore;
    const bool labeled = MET && tg >= 0 && tg < C;
    if (K == LOSS_FOCAL && !BWD) cnt += 1.0;
    const int64_t px = ((int64_t)n * h + oy / r) * w + ox / r;
    const int sub = (oy % r) * r + ox % r;
    const T* z = lo + px * ldlo + sub;  // class c at z[c * rr]
    __nv_bfloat16* d = BWD ? dx + px * lddx + sub : nullptr;
    if (BWD) {
      if (sub == 0)
        for (int c = C * rr; c < lddx; ++c) d[c] = f2bf(0.f);
      if (!valid) {
        for (int c = 0; c < C; ++c) d[c * rr] = f2bf(0.f);
        continue;
      }
    } else if (!valid && !labeled) {
      continue;
    }
    float mx = -INFINITY;
    int am = 0;
    for (int c = 0; c < C; ++c) {
      const float v = logit_f(z[c * rr]);
      if (v > mx) {
        mx = v;
        am = c;
      }
    }
    float se = 0.f, lt = 0.f;
    for (int c = 0; c < C; ++c) {
      const float v = logit_f(z[c * rr]);
      se += expf(v - mx);
      if (c == tg) lt = v;
    }
    if (!BWD) {
      if (MET && labeled) {
        ++n_labeled;
        atomicAdd(&hist[2 + C + am], 1u);          // area_pred
        atomicAdd(&hist[2 + 2 * C + (int)tg], 1u);  // area_lab
        if (am == (int)tg) {
          ++n_correct;
          atomicAdd(&hist[2 + (int)tg], 1u);  // area_inter
        }
      }
      if (valid) {
        const float wt = K == LOSS_CE ? 1.f : class_weight(la, tg, C);
        loss += (double)pixel_loss<K>(mx + logf(se) - lt, wt, la.gamma);
        if (K == LOSS_CE) cnt += 1.0;
        if (K == LOSS_WCE) cnt += (double)wt;
      }
    } else {
      const float inv = 1.f / se;
      const float gp = K == LOSS_CE ? g : g * pixel_grad_factor<K>(mx + logf(se) - lt, class_weight(la, tg, C), la.gamma);
      for (int c = 0; c < C; ++c) {
        const float v = logit_f(z[c * rr]);
        d[c * rr] = f2bf((expf(v - mx) * inv - (c == tg ? 1.f : 0.f)) * gp);
      }
    }
  }
  if (!BWD) {
    block_accum2(loss, cnt, accum);
    if (MET) {
      n_correct = __reduce_add_sync(0xffffffffu, n_correct);
      n_labeled = __reduce_add_sync(0xffffffffu, n_labeled);
      if ((threadIdx.x & 31) == 0) {
        atomicAdd(&hist[0], n_correct);
        atomicAdd(&hist[1], n_labeled);
      }
      __syncthreads();
      for (int i = threadIdx.x; i < 3 * C + 2; i += blockDim.x) {
        const unsigned int v = hist[i];
        if (v != 0u) atomicAdd(counters + i, (unsigned long long)v);
      }
    }
  }
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

namespace seg {
template <int K>
static int ce_nchw_fwd(const float* logits, const int64_t* target, int N, int C, int H, int W, int64_t ignore_index,
                       LossArgs la, double* accum, cudaStream_t stream) {
  const int64_t total = (int64_t)N * H * W;
  int blocks = (int)std::min<int64_t>(ceil_div64(total, 256), (int64_t)num_sms() * 8);
  ce_nchw_fwd_kernel<K><<<blocks, 256, 0, stream>>>(logits, target, N, C, H, W, ignore_index, la, accum);
  return check_launch("ce_nchw_fwd");
}
template <int K>
static int ce_nchw_bwd(const float* logits, const int64_t* target, int N, int C, int H, int W, int64_t ignore_index,
                       LossArgs la, const double* accum, const float* gscale, float* dlogits, cudaStream_t stream) {
  const int64_t total = (int64_t)N * H * W;
  int blocks = (int)std::min<int64_t>(ceil_div64(total, 256), (int64_t)num_sms() * 8);
  ce_nchw_bwd_kernel<K><<<blocks, 256, 0, stream>>>(logits, target, N, C, H, W, ignore_index, la, accum, gscale, dlogits);
  return check_launch("ce_nchw_bwd");
}

// counters != NULL: counters (int64 [2 + 3C]) += the eval_metrics counters of the batch (the MET instantiation)
template <int K>
static int upsample_ce_fwd(const float* logits_lo, const int64_t* target, int N, int Hi, int Wi, int Ho, int Wo, int C,
                           int align_corners, int64_t ignore_index, LossArgs la, double* accum, int32_t* argmax,
                           int64_t* counters, cudaStream_t stream) {
  SEG_REQUIRE(C <= MAXC, "upsample_ce: C=%d > %d", C, MAXC);
  const bool met = counters != nullptr;
  const auto kernel = met ? upsample_ce_kernel<false, K, true> : upsample_ce_kernel<false, K, false>;
  const int patch = std::max(patch_for(Hi, Ho, align_corners, TILE), patch_for(Wi, Wo, align_corners, TILE));
  const size_t smem = (size_t)patch * patch * C * sizeof(float) + (met ? (size_t)(3 * C + 2) * sizeof(unsigned int) : 0);
  SEG_REQUIRE(smem <= 200 * 1024, "upsample_ce: patch too large (%zu B)", smem);
  static size_t set_smem[2] = {0, 0};  // per instantiation
  if (smem > set_smem[met]) {
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    set_smem[met] = smem;
  }
  const int blocks = N * ceil_div(Ho, TILE) * ceil_div(Wo, TILE);
  kernel<<<blocks, 256, smem, stream>>>(
      logits_lo, target, N, Hi, Wi, Ho, Wo, C, align_corners, rscale(Hi, Ho, align_corners), rscale(Wi, Wo, align_corners),
      ignore_index, la, accum, argmax, nullptr, nullptr, patch, TILE, reinterpret_cast<unsigned long long*>(counters));
  return check_launch(met ? "upsample_ce_fwd_metrics" : "upsample_ce_fwd");
}

template <int K>
static int upsample_ce_bwd(const float* logits_lo, const int64_t* target, int N, int Hi, int Wi, int Ho, int Wo, int C,
                           int align_corners, int64_t ignore_index, LossArgs la, const double* accum, const float* gscale,
                           float* dlo_f32, void* dlo_fixed, void* dx, int lddx, cudaStream_t stream) {
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
    cudaFuncSetAttribute(upsample_ce_kernel<true, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    set_smem = smem;
  }
  const int64_t M = (int64_t)N * Hi * Wi;
  unsigned long long* fixed = reinterpret_cast<unsigned long long*>(dlo_fixed);
  cudaMemsetAsync(fixed, 0, (size_t)M * C * sizeof(unsigned long long), stream);
  const int blocks = N * ceil_div(Ho, tile) * ceil_div(Wo, tile);
  const float sh = rscale(Hi, Ho, align_corners), sw = rscale(Wi, Wo, align_corners);
  upsample_ce_kernel<true, K><<<blocks, 256, smem, stream>>>(
      logits_lo, target, N, Hi, Wi, Ho, Wo, C, align_corners, sh, sw, ignore_index, la, const_cast<double*>(accum), nullptr,
      gscale, fixed, patch, tile, nullptr);
  if (check_launch("upsample_ce_bwd")) return 1;
  const int64_t n = M * C;
  ce_grad_from_fixed_kernel<K><<<(unsigned)std::min<int64_t>(ceil_div64(n, 256), (int64_t)num_sms() * 8), 256, 0, stream>>>(
      fixed, n, gscale, accum, la, C, sh, sw, Ho, Wo, dlo_f32);
  if (check_launch("ce_grad_from_fixed")) return 1;
  if (dx) {
    int blocks2 = (int)std::min<int64_t>(ceil_div64(M * lddx, 256), (int64_t)num_sms() * 8);
    cast_pad_kernel<<<blocks2, 256, 0, stream>>>(dlo_f32, reinterpret_cast<__nv_bfloat16*>(dx), M, C, lddx);
    return check_launch("cast_pad");
  }
  return 0;
}

static int shuffle_ce_check(int N, int h, int w, int C, int r, int ld) {
  SEG_REQUIRE(C <= MAXC, "shuffle_loss: C=%d > %d", C, MAXC);
  SEG_REQUIRE(N > 0 && h > 0 && w > 0 && r >= 1, "shuffle_loss: bad sizes");
  SEG_REQUIRE(ld >= C * r * r, "shuffle_loss: pitch %d < r*r*C = %d", ld, C * r * r);
  return 0;
}
static unsigned shuffle_ce_blocks(int N, int h, int w, int r) {
  return (unsigned)std::min<int64_t>(ceil_div64((int64_t)N * h * w * r * r, 256), (int64_t)num_sms() * 8);
}
template <int K, typename T = __nv_bfloat16>
static int shuffle_ce_fwd(const void* lo, int ldlo, const int64_t* target, int N, int h, int w, int C, int r, int64_t ignore_index,
                          LossArgs la, double* accum, int64_t* counters, cudaStream_t stream) {
  if (shuffle_ce_check(N, h, w, C, r, ldlo)) return 1;
  const bool met = counters != nullptr;
  const auto kernel = met ? shuffle_ce_kernel<false, K, true, T> : shuffle_ce_kernel<false, K, false, T>;
  kernel<<<shuffle_ce_blocks(N, h, w, r), 256, met ? (size_t)(3 * C + 2) * sizeof(unsigned int) : 0, stream>>>(
      reinterpret_cast<const T*>(lo), ldlo, target, N, h, w, C, r, ignore_index, la, accum, nullptr, nullptr, 0,
      reinterpret_cast<unsigned long long*>(counters));
  return check_launch(met ? "shuffle_ce_fwd_metrics" : "shuffle_ce_fwd");
}
template <int K, typename T = __nv_bfloat16>
static int shuffle_ce_bwd(const void* lo, int ldlo, const int64_t* target, int N, int h, int w, int C, int r, int64_t ignore_index,
                          LossArgs la, const double* accum, const float* gscale, void* dx, int lddx, cudaStream_t stream) {
  if (shuffle_ce_check(N, h, w, C, r, ldlo) || shuffle_ce_check(N, h, w, C, r, lddx)) return 1;
  shuffle_ce_kernel<true, K, false, T><<<shuffle_ce_blocks(N, h, w, r), 256, 0, stream>>>(
      reinterpret_cast<const T*>(lo), ldlo, target, N, h, w, C, r, ignore_index, la, const_cast<double*>(accum),
      gscale, reinterpret_cast<__nv_bfloat16*>(dx), lddx, nullptr);
  return check_launch("shuffle_ce_bwd");
}
// full-resolution NHWC fp32 logits: the shuffle loss at r = 1 over an fp32 map
template <int K>
static int nhwc_ce_fwd(const float* logits, int ld, const int64_t* target, int N, int H, int W, int C, int64_t ignore_index,
                       LossArgs la, double* accum, int64_t* counters, cudaStream_t stream) {
  return shuffle_ce_fwd<K, float>(logits, ld, target, N, H, W, C, 1, ignore_index, la, accum, counters, stream);
}
template <int K>
static int nhwc_ce_bwd(const float* logits, int ld, const int64_t* target, int N, int H, int W, int C, int64_t ignore_index,
                       LossArgs la, const double* accum, const float* gscale, void* dx, int lddx, cudaStream_t stream) {
  return shuffle_ce_bwd<K, float>(logits, ld, target, N, H, W, C, 1, ignore_index, la, accum, gscale, dx, lddx, stream);
}

// kind: LOSS_CE (weight NULL, a mean), LOSS_WCE (NULL weight = ones) or LOSS_FOCAL (weight optional)
static int loss_args(const float* weight, int kind, float gamma, int mean, int C, LossArgs* la) {
  SEG_REQUIRE(C > 0, "loss: C=%d", C);
  SEG_REQUIRE(kind == LOSS_CE || kind == LOSS_WCE || kind == LOSS_FOCAL, "loss: unknown kind %d", kind);
  SEG_REQUIRE(kind != LOSS_CE || (weight == nullptr && mean), "loss: SEG_LOSS_CE takes no class weight and is a mean");
  SEG_REQUIRE(kind != LOSS_FOCAL || (gamma >= 0.f && isfinite(gamma)), "loss: focal gamma must be finite and >= 0 (got %g)",
              (double)gamma);
  *la = LossArgs{weight, gamma, mean ? 1 : 0};
  return 0;
}
#define SEG_LOSS_DISPATCH(kind, fn, ...)                   \
  ((kind) == LOSS_CE    ? fn<LOSS_CE>(__VA_ARGS__)         \
   : (kind) == LOSS_WCE ? fn<LOSS_WCE>(__VA_ARGS__)        \
                        : fn<LOSS_FOCAL>(__VA_ARGS__))
}  // namespace seg

extern "C" {

int seg_loss_nchw_fwd(const float* logits, const int64_t* target, int N, int C, int H, int W, int64_t ignore_index,
                      const float* weight, int kind, float gamma, double* accum, void* stream) {
  LossArgs la;
  if (loss_args(weight, kind, gamma, 1, C, &la)) return 1;
  return SEG_LOSS_DISPATCH(kind, ce_nchw_fwd, logits, target, N, C, H, W, ignore_index, la, accum, ST(stream));
}
int seg_loss_nchw_bwd(const float* logits, const int64_t* target, int N, int C, int H, int W, int64_t ignore_index,
                      const float* weight, int kind, float gamma, int mean, const double* accum, const float* gscale,
                      float* dlogits, void* stream) {
  LossArgs la;
  if (loss_args(weight, kind, gamma, mean, C, &la)) return 1;
  return SEG_LOSS_DISPATCH(kind, ce_nchw_bwd, logits, target, N, C, H, W, ignore_index, la, accum, gscale, dlogits, ST(stream));
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
int seg_loss_finalize(const double* accum, int mean, float* loss, void* stream) {
  loss_finalize_kernel<<<1, 32, 0, ST(stream)>>>(accum, mean, loss);
  return check_launch("loss_finalize");
}

int seg_upsample_loss_fwd(const float* logits_lo, const int64_t* target, int N, int Hi, int Wi, int Ho, int Wo, int C,
                          int align_corners, int64_t ignore_index, const float* weight, int kind, float gamma, double* accum,
                          int32_t* argmax, int64_t* counters, void* stream) {
  LossArgs la;
  if (loss_args(weight, kind, gamma, 1, C, &la)) return 1;
  return SEG_LOSS_DISPATCH(kind, upsample_ce_fwd, logits_lo, target, N, Hi, Wi, Ho, Wo, C, align_corners, ignore_index, la, accum,
                           argmax, counters, ST(stream));
}
// dlo_f32: fp32 [N,Hi,Wi,C]; dlo_fixed: int64 scratch [N,Hi,Wi,C] (zeroed here); dx: bf16 [N*Hi*Wi][lddx] or NULL
int seg_upsample_loss_bwd(const float* logits_lo, const int64_t* target, int N, int Hi, int Wi, int Ho, int Wo, int C,
                          int align_corners, int64_t ignore_index, const float* weight, int kind, float gamma, int mean,
                          const double* accum, const float* gscale, float* dlo_f32, void* dlo_fixed, void* dx, int lddx,
                          void* stream) {
  LossArgs la;
  if (loss_args(weight, kind, gamma, mean, C, &la)) return 1;
  return SEG_LOSS_DISPATCH(kind, upsample_ce_bwd, logits_lo, target, N, Hi, Wi, Ho, Wo, C, align_corners, ignore_index, la, accum,
                           gscale, dlo_f32, dlo_fixed, dx, lddx, ST(stream));
}

int seg_shuffle_loss_fwd(const void* logits_lo, int ldlo, const int64_t* target, int N, int h, int w, int C, int r,
                         int64_t ignore_index, const float* weight, int kind, float gamma, double* accum, int64_t* counters,
                         void* stream) {
  LossArgs la;
  if (loss_args(weight, kind, gamma, 1, C, &la)) return 1;
  return SEG_LOSS_DISPATCH(kind, shuffle_ce_fwd, logits_lo, ldlo, target, N, h, w, C, r, ignore_index, la, accum, counters,
                           ST(stream));
}
int seg_shuffle_loss_bwd(const void* logits_lo, int ldlo, const int64_t* target, int N, int h, int w, int C, int r,
                         int64_t ignore_index, const float* weight, int kind, float gamma, int mean, const double* accum,
                         const float* gscale, void* dx, int lddx, void* stream) {
  LossArgs la;
  if (loss_args(weight, kind, gamma, mean, C, &la)) return 1;
  return SEG_LOSS_DISPATCH(kind, shuffle_ce_bwd, logits_lo, ldlo, target, N, h, w, C, r, ignore_index, la, accum, gscale, dx, lddx,
                           ST(stream));
}

int seg_nhwc_loss_fwd(const float* logits, int ld, const int64_t* target, int N, int H, int W, int C, int64_t ignore_index,
                      const float* weight, int kind, float gamma, double* accum, int64_t* counters, void* stream) {
  LossArgs la;
  if (loss_args(weight, kind, gamma, 1, C, &la)) return 1;
  return SEG_LOSS_DISPATCH(kind, nhwc_ce_fwd, logits, ld, target, N, H, W, C, ignore_index, la, accum, counters, ST(stream));
}
int seg_nhwc_loss_bwd(const float* logits, int ld, const int64_t* target, int N, int H, int W, int C, int64_t ignore_index,
                      const float* weight, int kind, float gamma, int mean, const double* accum, const float* gscale, void* dx,
                      int lddx, void* stream) {
  LossArgs la;
  if (loss_args(weight, kind, gamma, mean, C, &la)) return 1;
  return SEG_LOSS_DISPATCH(kind, nhwc_ce_bwd, logits, ld, target, N, H, W, C, ignore_index, la, accum, gscale, dx, lddx,
                           ST(stream));
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
