// seg_elementwise.cu — the HBM-bound kernels of the hot path: weight packing, explicit im2col (stem only),
// BatchNorm statistics / finalize / apply(+residual+ReLU+dropout) / backward, max-pool, adaptive average pool,
// bilinear resize (both align_corners modes) and layout conversion.  All activation kernels are NHWC bf16 and move
// 16-byte (8-channel) vectors per thread; reductions use warp shuffles + one atomic per block-column.
// Reference call sites are cited next to each entry point in include/seg_b200.h.
#include "seg_common.cuh"
#include "seg_sync.cuh"

namespace seg {

static inline int grid_for(int64_t work_items, int threads, int max_blocks_per_sm = 8) {
  int64_t b = ceil_div64(work_items, threads);
  int64_t cap = (int64_t)num_sms() * max_blocks_per_sm;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

// ------------------------------------------------------------------ weights
__global__ void pack_weight_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int K, int C, int R,
                                   int S, int Cpad) {
  const int64_t total = (int64_t)R * S * K * Cpad;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cpad);
    const int64_t t1 = i / Cpad;
    const int k = (int)(t1 % K);
    const int tap = (int)(t1 / K);
    const int r = tap / S, s = tap - r * S;
    float v = 0.f;
    if (c < C) v = w[(((int64_t)k * C + c) * R + r) * S + s];
    out[i] = f2bf(v);
  }
}

// ---- batched variants: ONE launch packs every conv weight of the model / unpacks every weight gradient ----
struct PackEntry {
  const float* oihw;      // fp32 master weight (pack: source) / fp32 OIHW grad (unpack: destination, as float*)
  void* packed;           // bf16 packed weight (pack: destination) / fp32 packed grad (unpack: source)
  int K, C, R, S, Cpad;
  int explicit_rsc;       // 1: stem-style [K][(r,s,c) padded to Cpad] single-tap matrix
  long long start;        // prefix sum of work items
};

__device__ __forceinline__ int find_entry(const PackEntry* __restrict__ tab, int n, long long i) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tab[mid].start <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(256) pack_weights_batched_kernel(const PackEntry* __restrict__ tab, int n, long long total) {
  const PackEntry e = tab[blockIdx.y];  // one block row per conv: no per-element table search
  const long long count = (blockIdx.y + 1 < n ? tab[blockIdx.y + 1].start : total) - e.start;
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < count; j += (long long)gridDim.x * blockDim.x) {
    __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(e.packed);
    float v = 0.f;
    if (e.explicit_rsc) {
      const int kk = (int)(j % e.Cpad);
      const int k = (int)(j / e.Cpad);
      if (kk < e.R * e.S * e.C) {
        const int c = kk % e.C, tap = kk / e.C;
        const int r = tap / e.S, s = tap - r * e.S;
        v = e.oihw[(((long long)k * e.C + c) * e.R + r) * e.S + s];
      }
    } else {
      const int c = (int)(j % e.Cpad);
      const long long t1 = j / e.Cpad;
      const int k = (int)(t1 % e.K);
      const int tap = (int)(t1 / e.K);
      const int r = tap / e.S, s = tap - r * e.S;
      if (c < e.C) v = e.oihw[(((long long)k * e.C + c) * e.R + r) * e.S + s];
    }
    out[j] = f2bf(v);
  }
}

// OIHW fp32 grad (+)= packed fp32 grad.  Work items index the OIHW tensor.
__global__ void __launch_bounds__(256) unpack_wgrads_batched_kernel(const PackEntry* __restrict__ tab, int n, long long total,
                                                                    float beta) {
  const PackEntry e = tab[blockIdx.y];
  const long long count = (blockIdx.y + 1 < n ? tab[blockIdx.y + 1].start : total) - e.start;
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < count; j += (long long)gridDim.x * blockDim.x) {
    const int s = (int)(j % e.S);
    long long t = j / e.S;
    const int r = (int)(t % e.R);
    t /= e.R;
    const int c = (int)(t % e.C);
    const int k = (int)(t / e.C);
    const float* src = reinterpret_cast<const float*>(e.packed);
    float v;
    if (e.explicit_rsc)
      v = src[(long long)k * e.Cpad + (r * e.S + s) * e.C + c];
    else
      v = src[((long long)(r * e.S + s) * e.K + k) * e.Cpad + c];
    float* g = const_cast<float*>(e.oihw);
    g[j] = (beta != 0.f) ? beta * g[j] + v : v;
  }
}

__global__ void unpack_wgrad_kernel(const float* __restrict__ dw, float* __restrict__ g, int K, int C, int R, int S,
                                    int Cpad, float beta) {
  const int64_t total = (int64_t)K * C * R * S;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int s = (int)(i % S);
    int64_t t = i / S;
    const int r = (int)(t % R);
    t /= R;
    const int c = (int)(t % C);
    const int k = (int)(t / C);
    const float v = dw[((int64_t)(r * S + s) * K + k) * Cpad + c];
    g[i] = (beta != 0.f) ? beta * g[i] + v : v;
  }
}

__global__ void __launch_bounds__(256) im2col_kernel(seg_conv_desc d, const void* __restrict__ x, int x_nchw_f32,
                                                     __nv_bfloat16* __restrict__ col, int Kpad) {
  // one thread = 8 consecutive columns of one output pixel -> a single 16-byte store
  const int64_t M = (int64_t)d.N * d.P * d.Q;
  const int KV = Kpad >> 3;
  const int64_t total = M * KV;
  const int Kreal = d.R * d.S * d.C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int kv = (int)(i % KV);
    const int64_t m = i / KV;
    const int n = (int)(m / (d.P * d.Q));
    const int rem = (int)(m - (int64_t)n * d.P * d.Q);
    const int op = rem / d.Q, oq = rem - op * d.Q;
    const int ih0 = op * d.stride - d.pad, iw0 = oq * d.stride - d.pad;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int kk = kv * 8 + j;
      float val = 0.f;
      if (kk < Kreal) {
        const int tap = kk / d.C;
        const int c = kk - tap * d.C;
        const int r = tap / d.S, s = tap - r * d.S;
        const int ih = ih0 + r * d.dil, iw = iw0 + s * d.dil;
        if (ih >= 0 && ih < d.H && iw >= 0 && iw < d.W) {
          if (x_nchw_f32)
            val = __ldg(reinterpret_cast<const float*>(x) + (((int64_t)n * d.C + c) * d.H + ih) * d.W + iw);
          else
            val = bf2f(reinterpret_cast<const __nv_bfloat16*>(x)[(((int64_t)n * d.H + ih) * d.W + iw) * d.ldx + c]);
        }
      }
      v[j] = val;
    }
    *reinterpret_cast<bf16x8*>(col + m * Kpad + kv * 8) = pack8(v);
  }
}

// ------------------------------------------------------------------ BatchNorm
// Column-reduction skeleton shared by bn_stats and bn_bwd_reduce: a 256-thread block owns GB = min(G,256) channel
// groups (8 channels each) and 256/GB row lanes; rows are grid-strided.  The block's sums (fixed order inside the block)
// are added to acc[NACC][C] (fp64, ZERO at launch) with one fp64 atomic per channel: exact accumulation of fp32 partials,
// hence order-independent and bit-reproducible (see conv_gemm_pp's statistics epilogue for the argument).
constexpr int RED_SLOTS = 8;  // accumulator copies the blocks spread their atomics over (contention: blocks / 8 per address)
template <int NACC, int SLOTS = 1, class F>
__device__ __forceinline__ void column_reduce(int64_t M, int C, double* acc_out /*[SLOTS][NACC][C]*/, F f) {
  const int G = C >> 3;
  const int GB = min(G, 256);
  const int rows_par = 256 / GB;
  const int gl = threadIdx.x % GB;
  const int rl = threadIdx.x / GB;
  const int g = blockIdx.y * GB + gl;
  float acc[NACC][8];
#pragma unroll
  for (int a = 0; a < NACC; ++a)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[a][i] = 0.f;
  if (g < G && rl < rows_par) {
#pragma unroll 2
    for (int64_t row = (int64_t)blockIdx.x * rows_par + rl; row < M; row += (int64_t)gridDim.x * rows_par)
      f(row, g, acc);
  }
  __shared__ float red[256 * 8];
  for (int a = 0; a < NACC; ++a) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 8; ++i) red[threadIdx.x * 8 + i] = acc[a][i];
    __syncthreads();
    if (rl == 0 && g < G) {
      float s[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) s[i] = 0.f;
      for (int r = 0; r < rows_par; ++r)
#pragma unroll
        for (int i = 0; i < 8; ++i) s[i] += red[(r * GB + gl) * 8 + i];
      double* o = acc_out + ((size_t)(blockIdx.x % SLOTS) * NACC + a) * C + g * 8;
#pragma unroll
      for (int i = 0; i < 8; ++i) atomicAdd(o + i, (double)s[i]);
    }
  }
}

// `ticket` pattern shared by the reductions: true in every thread of the LAST of gridDim.x*gridDim.y blocks to arrive
__device__ __forceinline__ bool last_block_arrived(unsigned* ticket) {
  __shared__ int last_flag;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last_flag = (atomicAdd(ticket, 1u) == gridDim.x * gridDim.y - 1u);
  __syncthreads();
  if (last_flag) __threadfence();
  return last_flag != 0;
}

// stats[2C] fp64 (zero at launch) += (sum x, sum x^2); SyncBN: the last block pushes the totals to the peers
__global__ void __launch_bounds__(256, 4) bn_stats_kernel(const __nv_bfloat16* __restrict__ x, int64_t M, int C, int ldx,
                                                          double* __restrict__ stats, const SyncDesc sync, unsigned* ticket) {
  column_reduce<2>(M, C, stats, [&](int64_t row, int g, float(*acc)[8]) {
    const bf16x8 v = *reinterpret_cast<const bf16x8*>(x + row * ldx + g * 8);
    float f[8];
    unpack8(v, f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      acc[0][i] += f[i];
      acc[1][i] += f[i] * f[i];
    }
  });
  if (sync.world > 0) {
    __shared__ int sm_flag;
    sync_push_when_last(sync, stats, 2 * C, ticket, gridDim.x * gridDim.y, (int)threadIdx.x, 256, [] { __syncthreads(); }, &sm_flag);
  }
}

__global__ void bn_finalize_kernel(const double* __restrict__ stats, double count, int C, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float eps, float momentum, int clamp_eps,
                                   float* running_mean, float* running_var, float* __restrict__ scale_shift,
                                   float* __restrict__ save) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double mean = stats[c] / count;
  double var = stats[C + c] / count - mean * mean;
  if (var < 0) var = 0;
  const double istd = clamp_eps ? 1.0 / sqrt(var < (double)eps ? (double)eps : var) : 1.0 / sqrt(var + (double)eps);
  if (running_mean) {
    const double unbiased = count > 1 ? var * count / (count - 1) : var;
    running_mean[c] = (float)((1.0 - momentum) * running_mean[c] + momentum * mean);
    running_var[c] = (float)((1.0 - momentum) * running_var[c] + momentum * unbiased);
  }
  const float sc = (float)(gamma[c] * istd);
  scale_shift[c] = sc;
  scale_shift[C + c] = (float)(beta[c] - mean * gamma[c] * istd);
  save[c] = (float)mean;
  save[C + c] = (float)istd;
}

__global__ void bn_eval_kernel(int C, const float* gamma, const float* beta, const float* rm, const float* rv, float eps,
                               float* scale_shift, float* save) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float istd = rsqrtf(rv[c] + eps);
  const float sc = gamma[c] * istd;
  scale_shift[c] = sc;
  scale_shift[C + c] = beta[c] - rm[c] * sc;
  if (save) {
    save[c] = rm[c];
    save[C + c] = istd;
  }
}

// Channel-group-stationary mapping shared by the three streaming BN kernels: a 256-thread block owns GB = min(G,256)
// channel groups (8 channels = one 16-byte vector each) x 256/GB row lanes, so every thread keeps its per-channel
// coefficients in registers for the whole grid-stride loop over rows (no per-element coefficient loads, no division).
struct RowMap {
  int g, rl, rows_par;
  bool active;
};
__device__ __forceinline__ RowMap row_map(int C) {
  const int G = C >> 3;
  const int GB = min(G, 256);
  RowMap r;
  r.rows_par = 256 / GB;
  r.rl = threadIdx.x / GB;
  r.g = blockIdx.y * GB + (threadIdx.x % GB);
  r.active = r.g < G && r.rl < r.rows_par;
  return r;
}
__device__ __forceinline__ void ld8(const float* p, float* v) {
  *reinterpret_cast<float4*>(v) = __ldg(reinterpret_cast<const float4*>(p));
  *reinterpret_cast<float4*>(v + 4) = __ldg(reinterpret_cast<const float4*>(p + 4));
}

// Training-mode coefficients computed in the consumer (no separate finalize launch): every thread derives scale/shift of
// its 8 channels from the batch sums; the threads of block row 0 also record (mean, 1/std) for the backward pass and
// update the running statistics (nn.BatchNorm2d semantics: momentum, unbiased variance).
struct BnTrain {
  const double* stats;  // [2C] fp64 sum, sum of squares over `count` elements (null: use the precomputed scale_shift)
  double count;
  const float *gamma, *beta;
  float eps, momentum;
  int clamp_eps;
  float *running_mean, *running_var, *save;
  // growth > 0: `stats` is a dense block's statistics table — records [sum(w), sum^2(w)] back to back in channel order,
  // the block input's (w = c0) first, then one per layer (w = growth); channel c's sums are read from its record
  int c0, growth;
};

// TABLE: tr.stats is a dense block's statistics table (BnTrain::c0 / growth); the launch without it compiles as before
template <bool TABLE = false>
__global__ void __launch_bounds__(256, 4) bn_apply_kernel(const __nv_bfloat16* __restrict__ x, int ldx,
                                                       const float* __restrict__ ss, const __nv_bfloat16* __restrict__ res,
                                                       int ldr, __nv_bfloat16* __restrict__ out, int ldo, int64_t M, int C,
                                                       int relu, float drop_p, uint64_t seed,
                                                       const uint64_t* __restrict__ step_ctr, int drop_hw, const BnTrain tr,
                                                       uint8_t* __restrict__ mask /*[M][C/8] or null*/) {
  pdl_wait();
  const RowMap rm = row_map(C);
  if (step_ctr) seed += (*step_ctr) * 0x9E3779B97F4A7C15ull;  // device-side step counter keeps CUDA-graph replays fresh
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  float sc[8], sh[8];
  if (rm.active) {
    if (tr.stats) {
      float gm[8], bt[8];
      ld8(tr.gamma + rm.g * 8, gm);
      ld8(tr.beta + rm.g * 8, bt);
      const bool writer = blockIdx.x == 0 && rm.rl == 0;
      const double inv_count = 1.0 / tr.count;  // one division; the per-channel math below is multiply-add + fp32 rsqrt
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        // fp64 totals, one channel at a time (no register arrays of doubles); under SyncBN the producer's exchange has
        // already turned them into the world's
        const int cj = rm.g * 8 + j;
        int rec = 0, w = C, k = cj;
        if constexpr (TABLE) {
          if (cj < tr.c0) {
            w = tr.c0;
          } else {
            const int l = (cj - tr.c0) / tr.growth;
            w = tr.growth;
            k = cj - tr.c0 - l * tr.growth;
            rec = 2 * tr.c0 + 2 * l * tr.growth;
          }
        }
        const double s1 = __ldg(tr.stats + rec + k);
        const double s2 = __ldg(tr.stats + rec + w + k);
        const double mean = s1 * inv_count;
        double var = fma(s2, inv_count, -mean * mean);
        if (var < 0) var = 0;
        const float vf = tr.clamp_eps ? fmaxf((float)var, tr.eps) : (float)(var + (double)tr.eps);
        float istd = rsqrtf(vf);
        istd = istd * (1.5f - 0.5f * vf * istd * istd);  // one Newton step: fp32-exact 1/sqrt
        sc[j] = gm[j] * istd;
        sh[j] = fmaf(-(float)mean, sc[j], bt[j]);
        if (writer) {
          const int c = rm.g * 8 + j;
          tr.save[c] = (float)mean;
          tr.save[C + c] = istd;
          if (tr.running_mean) {
            const double unbiased = tr.count > 1 ? var * tr.count / (tr.count - 1) : var;
            tr.running_mean[c] = (float)((1.0 - tr.momentum) * tr.running_mean[c] + tr.momentum * mean);
            tr.running_var[c] = (float)((1.0 - tr.momentum) * tr.running_var[c] + tr.momentum * unbiased);
          }
        }
      }
    } else {
      ld8(ss + rm.g * 8, sc);
      ld8(ss + C + rm.g * 8, sh);
    }
    const int64_t step = (int64_t)gridDim.x * rm.rows_par;
    const int co = rm.g * 8;
    for (int64_t row = (int64_t)blockIdx.x * rm.rows_par + rm.rl; row < M; row += 2 * step) {
      const int64_t row2 = row + step;
      const bool has2 = row2 < M;
      bf16x8 xa = *reinterpret_cast<const bf16x8*>(x + row * ldx + co), xb, ra, rb;
      if (has2) xb = *reinterpret_cast<const bf16x8*>(x + row2 * ldx + co);
      if (res) {
        ra = *reinterpret_cast<const bf16x8*>(res + row * ldr + co);
        if (has2) rb = *reinterpret_cast<const bf16x8*>(res + row2 * ldr + co);
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        if (u == 1 && !has2) break;
        const int64_t r = u ? row2 : row;
        float f[8];
        unpack8(u ? xb : xa, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = fmaf(f[j], sc[j], sh[j]);
        if (res) {
          float q[8];
          unpack8(u ? rb : ra, q);
#pragma unroll
          for (int j = 0; j < 8; ++j) f[j] += q[j];
        }
        if (relu) {
#pragma unroll
          for (int j = 0; j < 8; ++j) f[j] = fmaxf(f[j], 0.f);
        }
        if (drop_p > 0.f) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            // nn.Dropout: one draw per element; nn.Dropout2d (drop_hw = H*W > 0): one draw per (image, channel)
            const float uu = hash_uniform(seed, (uint64_t)((drop_hw > 0 ? r / drop_hw : r) * C + co + j));
            f[j] = (uu >= drop_p) ? f[j] * keep_scale : 0.f;
          }
        }
        const bf16x8 a = pack8(f);
        *reinterpret_cast<bf16x8*>(out + r * ldo + co) = a;
        if (mask) {
          // bit j = (stored bf16 A > 0): the predicate the activation-reading backward evaluates, on the same values
          float o[8];
          unpack8(a, o);
          unsigned b = 0;
#pragma unroll
          for (int j = 0; j < 8; ++j) b |= (o[j] > 0.f ? 1u : 0u) << j;
          mask[r * (C >> 3) + rm.g] = (uint8_t)b;
        }
      }
    }
  }
  pdl_trigger();
}

// Where the backward passes take the ReLU (and dropout keep) mask from:
//   ACT        the stored activation A (out > 0)
//   RECOMPUTE  x with the forward's own coefficients (BN -> ReLU with nothing in between, batch statistics, no dropout)
//   BITS       the bit mask bn_apply wrote in the forward: one byte per (row, 8-channel group), bit j = A[8g+j] > 0 —
//              1/16 of the bytes of A
enum class MaskSrc { ACT, RECOMPUTE, BITS };
// mask source of a backward call: the bit mask when given, else the stored activation, else (relu, out == NULL) recomputed
static MaskSrc mask_src(int relu, const void* out, const uint8_t* mask) {
  if (!relu) return MaskSrc::ACT;  // no mask at all (the ACT variants test relu at run time)
  return mask ? MaskSrc::BITS : out ? MaskSrc::ACT : MaskSrc::RECOMPUTE;
}
template <class K>
static K by_mask_src(MaskSrc ms, K act, K recompute, K bits) {
  return ms == MaskSrc::BITS ? bits : ms == MaskSrc::RECOMPUTE ? recompute : act;
}
__device__ __forceinline__ void apply_mask_bits(unsigned b, float keep_scale, float* dz) {
#pragma unroll
  for (int j = 0; j < 8; ++j) dz[j] = ((b >> j) & 1u) ? dz[j] * keep_scale : 0.f;
}

__device__ __noinline__ void bn_bwd_reduce_finalize(const double* acc, float* final_sums, float* dgamma, float* dbeta, int accumulate,
                                                    int C, const SyncDesc sync) {
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) {
    double t = 0.0;  // the copies' totals are exact sums; so is their sum
#pragma unroll
    for (int sl = 0; sl < RED_SLOTS; ++sl) t += __ldcg(acc + (size_t)sl * 2 * C + c);
    const float v = (float)t;
    final_sums[c] = v;
    float* pg = c < C ? dbeta : dgamma;
    const int ch = c < C ? c : c - C;
    if (pg) pg[ch] = accumulate ? pg[ch] + v : v;
  }
  if (sync.world > 0) {  // whole exchange here: final_sums becomes the world's sums (bn_bwd_apply then needs no SyncBN logic)
    __threadfence();
    __syncthreads();
    sync_exchange_block_f(sync, final_sums, 2 * C, (int)threadIdx.x, (int)blockDim.x, [] { __syncthreads(); });
  }
}

template <MaskSrc MS>
__global__ void __launch_bounds__(256, 4)
    bn_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ dout, int lddo, const __nv_bfloat16* __restrict__ out, int ldo,
                         const uint8_t* __restrict__ mask, const __nv_bfloat16* __restrict__ x, int ldx,
                         const float* __restrict__ save, int64_t M, int C,
                         int relu, float drop_p, double* acc /*[RED_SLOTS][2C] fp64, zero at launch*/, unsigned* ticket, float* final_sums,
                         float* dgamma, float* dbeta, int accumulate, const float* __restrict__ gamma,
                         const float* __restrict__ beta, const SyncDesc sync) {
  constexpr bool REMASK = MS == MaskSrc::RECOMPUTE;
  pdl_wait();
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const RowMap rm = row_map(C);
  // ReLU mask (MaskSrc): RECOMPUTE derives it from x with exactly the forward's coefficients  sc = gamma*istd,
  // sh = fma(-mean, sc, beta)
  float mean[8], wi[8], sc[REMASK ? 8 : 1], sh[REMASK ? 8 : 1];
  if (rm.active) {
    ld8(save + rm.g * 8, mean);
    ld8(save + C + rm.g * 8, wi);
    if constexpr (REMASK) {
      float gm[8], bt[8];
      ld8(gamma + rm.g * 8, gm);
      ld8(beta + rm.g * 8, bt);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        sc[i] = gm[i] * wi[i];
        sh[i] = fmaf(-mean[i], sc[i], bt[i]);
      }
    }
  }
  column_reduce<2, RED_SLOTS>(M, C, acc, [&](int64_t row, int g, float(*a)[8]) {
    float dz[8], xv[8];
    const bf16x8 dv = *reinterpret_cast<const bf16x8*>(dout + row * lddo + g * 8);
    const bf16x8 xx = *reinterpret_cast<const bf16x8*>(x + row * ldx + g * 8);
    unpack8(dv, dz);
    unpack8(xx, xv);
    if constexpr (REMASK) {
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] = (fmaf(xv[i], sc[i], sh[i]) > 0.f) ? dz[i] : 0.f;
    } else if constexpr (MS == MaskSrc::BITS) {
      apply_mask_bits(mask[row * (C >> 3) + g], keep_scale, dz);
    } else if (relu) {
      float o[8];
      unpack8(*reinterpret_cast<const bf16x8*>(out + row * ldo + g * 8), o);
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] = (o[i] > 0.f) ? dz[i] * keep_scale : 0.f;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      a[0][i] += dz[i];
      a[1][i] += dz[i] * (xv[i] - mean[i]) * wi[i];
    }
  });
  pdl_trigger();
  // the last block to finish rounds the fp64 totals to fp32, writes the parameter gradients (dbeta = sum dz, dgamma = sum
  // dz*xhat) and, under SyncBN, exchanges the sums with the peers — a cold path kept out of line so that its registers do not
  // push the streaming loop above 64 (4 blocks per SM)
  if (!last_block_arrived(ticket)) return;
  bn_bwd_reduce_finalize(acc, final_sums, dgamma, dbeta, accumulate, C, sync);
}

// dx = A*dz + B*x + Cc with A = gamma*istd, B = -gamma*istd^2*s1/count, Cc = -gamma*istd*s0/count + gamma*istd^2*mean*s1/count
// ACC: dx += (the same), summed in fp32 and rounded to bf16 once (pre-activation BN adding into a concat's gradient)
template <MaskSrc MS, bool ACC = false>
__global__ void __launch_bounds__(256, 4)
    bn_bwd_apply_kernel(const __nv_bfloat16* __restrict__ dout, int lddo, const __nv_bfloat16* __restrict__ out, int ldo,
                        const uint8_t* __restrict__ mask, const __nv_bfloat16* __restrict__ x, int ldx,
                        const float* __restrict__ save,
                        const float* __restrict__ gamma, const float* __restrict__ sums, float inv_count, int64_t M, int C,
                        int relu, float drop_p, __nv_bfloat16* __restrict__ dx, int lddx, __nv_bfloat16* dres, int lddres,
                        float beta_res, const float* __restrict__ beta) {
  constexpr bool REMASK = MS == MaskSrc::RECOMPUTE;
  pdl_wait();
  const RowMap rm = row_map(C);
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const int co = rm.g * 8;
  float cA[8], cB[8], cC[8], sh[REMASK ? 8 : 1];
  if (rm.active) {
    float mean[8], istd[8], gm[8], s0[8], s1[8];
    ld8(save + co, mean);
    ld8(save + C + co, istd);
    ld8(gamma + co, gm);
    ld8(sums + co, s0);
    ld8(sums + C + co, s1);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float a = gm[j] * istd[j];
      cA[j] = a;
      cB[j] = -a * istd[j] * s1[j] * inv_count;
      cC[j] = -a * s0[j] * inv_count - cB[j] * mean[j];
    }
    if constexpr (REMASK) {
      float bt[8];
      ld8(beta + co, bt);
#pragma unroll
      for (int j = 0; j < 8; ++j) sh[j] = fmaf(-mean[j], cA[j], bt[j]);  // forward: sc = gamma*istd (= cA), sh = fma(-mean, sc, beta)
    }
  }
  const int64_t step = (int64_t)gridDim.x * rm.rows_par;
  const int64_t row_end = rm.active ? M : 0;
  for (int64_t row = (int64_t)blockIdx.x * rm.rows_par + rm.rl; row < row_end; row += step) {
    float dz[8], xv[8];
    const bf16x8 dv = *reinterpret_cast<const bf16x8*>(dout + row * lddo + co);
    const bf16x8 xx = *reinterpret_cast<const bf16x8*>(x + row * ldx + co);
    unpack8(dv, dz);
    unpack8(xx, xv);
    if constexpr (REMASK) {
#pragma unroll
      for (int j = 0; j < 8; ++j) dz[j] = (fmaf(xv[j], cA[j], sh[j]) > 0.f) ? dz[j] : 0.f;
    } else if constexpr (MS == MaskSrc::BITS) {
      apply_mask_bits(mask[row * (C >> 3) + rm.g], keep_scale, dz);
    } else if (relu) {
      float o[8];
      unpack8(*reinterpret_cast<const bf16x8*>(out + row * ldo + co), o);
#pragma unroll
      for (int j = 0; j < 8; ++j) dz[j] = (o[j] > 0.f) ? dz[j] * keep_scale : 0.f;
    }
    if (dres) {
      float r[8];
      if (beta_res != 0.f) {
        unpack8(*reinterpret_cast<const bf16x8*>(dres + row * lddres + co), r);
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = beta_res * r[j] + dz[j];
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = dz[j];
      }
      *reinterpret_cast<bf16x8*>(dres + row * lddres + co) = pack8(r);
    }
    float o8[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o8[j] = fmaf(cA[j], dz[j], fmaf(cB[j], xv[j], cC[j]));
    if constexpr (ACC) {
      float old[8];
      unpack8(*reinterpret_cast<const bf16x8*>(dx + row * lddx + co), old);
#pragma unroll
      for (int j = 0; j < 8; ++j) o8[j] += old[j];
    }
    *reinterpret_cast<bf16x8*>(dx + row * lddx + co) = pack8(o8);
  }
  pdl_trigger();
}

// ------------------------------------------------------------------------------------------------------------------
// BatchNorm backward in ONE cooperative launch (replaces bn_bwd_reduce + bn_bwd_apply on the engine's path; the two-launch
// forms stay for callers that need the sums separately).
//   phase 1   every block streams its rows once: per-channel partial sums (sum dz, sum dz*xhat) -> its own workspace row
//   barrier   all blocks are co-resident (the host sizes the grid from the occupancy of THIS kernel), so a grid-wide
//             barrier is an atomic counter + spin
//   phase 1b  the cross-block sum is spread over ALL blocks: block b adds its few columns over every row, in row order ->
//             bit-reproducible totals with no atomics at all; the same threads write dgamma / dbeta
//   barrier   (+ SyncBN: block 0 exchanges the totals with the peers (seg_sync.cuh), leaving the world's; barrier)
//   phase 2   dx = A*dz + B*x + Cc (and the residual branch's gradient); the second read of dz / x hits L2 for the small maps
// Same arithmetic as the two-launch path.
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void grid_barrier(unsigned* ctr, unsigned target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(ctr, 1u);
    const long long t0 = clock64();
    while (ld_acquire_gpu(ctr) < target) {
      if (clock64() - t0 > 8000000000ll) {  // ~4 s: the blocks were not co-resident; trap instead of hanging the box
        printf("seg_b200: grid barrier timeout (block %d,%d target %u)\n", blockIdx.x, blockIdx.y, target);
        __trap();
      }
    }
    __threadfence();
  }
  __syncthreads();
}

struct BnBwdFused {
  const __nv_bfloat16 *dout, *out, *x;
  const uint8_t* mask;  // [M][C/8] ReLU bits (MaskSrc::BITS)
  int lddo, ldo, ldx;
  const float *save, *gamma, *beta;
  int64_t M;
  int C, relu;
  float drop_p, inv_count;  // inv_count = 1 / (rows summed over the WORLD)
  float* rows;              // [gridDim.y][gridDim.x][2][W] partial sums (W = channels of a slab)
  float* totals;            // [2C] totals (always written): the LOCAL ones, the world's after a SyncBN exchange
  unsigned* ctr;            // grid-barrier counter, zero at launch
  float *dgamma, *dbeta;
  int accumulate, zero_sums;  // zero_sums: frozen BatchNorm (eval statistics): dx = gamma*istd*dz
  __nv_bfloat16 *dx, *dres;
  int lddx, lddres;
  float beta_res;
  SyncDesc sync;
};

template <MaskSrc MS, bool ACC = false>
__global__ void __launch_bounds__(256, 3) bn_bwd_fused_kernel(const BnBwdFused p) {
  constexpr bool REMASK = MS == MaskSrc::RECOMPUTE;
  const RowMap rm = row_map(p.C);
  const int C = p.C;
  const int co = rm.g * 8;
  const float keep_scale = p.drop_p > 0.f ? 1.f / (1.f - p.drop_p) : 1.f;
  const int GB = min(C >> 3, 256);
  const int W = GB * 8;
  const unsigned nblocks = gridDim.x * gridDim.y;
  __shared__ float red[256 * 8];
  // forward coefficients of this thread's 8 channels (mask recomputation / xhat)
  float mean[8], istd[8], gm[8], sh[REMASK ? 8 : 1];
  if (rm.active) {
    ld8(p.save + co, mean);
    ld8(p.save + C + co, istd);
    ld8(p.gamma + co, gm);
    if constexpr (REMASK) {
      float bt[8];
      ld8(p.beta + co, bt);
#pragma unroll
      for (int j = 0; j < 8; ++j) sh[j] = fmaf(-mean[j], gm[j] * istd[j], bt[j]);
    }
  }
  const int64_t step = (int64_t)gridDim.x * rm.rows_par;
  // ------------------------------------------------ phase 1: partial sums
  {
    float a0[8], a1[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a0[j] = a1[j] = 0.f;
    if (rm.active) {
#pragma unroll 2
      for (int64_t row = (int64_t)blockIdx.x * rm.rows_par + rm.rl; row < p.M; row += step) {
        float dz[8], xv[8];
        unpack8(*reinterpret_cast<const bf16x8*>(p.dout + row * p.lddo + co), dz);
        unpack8(*reinterpret_cast<const bf16x8*>(p.x + row * p.ldx + co), xv);
        if constexpr (REMASK) {
#pragma unroll
          for (int j = 0; j < 8; ++j) dz[j] = (fmaf(xv[j], gm[j] * istd[j], sh[j]) > 0.f) ? dz[j] : 0.f;
        } else if constexpr (MS == MaskSrc::BITS) {
          apply_mask_bits(p.mask[row * (C >> 3) + rm.g], keep_scale, dz);
        } else if (p.relu) {
          float o[8];
          unpack8(*reinterpret_cast<const bf16x8*>(p.out + row * p.ldo + co), o);
#pragma unroll
          for (int j = 0; j < 8; ++j) dz[j] = (o[j] > 0.f) ? dz[j] * keep_scale : 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          a0[j] += dz[j];
          a1[j] += dz[j] * (xv[j] - mean[j]) * istd[j];
        }
      }
    }
    float* myrow = p.rows + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * (2 * W);
    const int gl = threadIdx.x % GB;
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      __syncthreads();
#pragma unroll
      for (int j = 0; j < 8; ++j) red[threadIdx.x * 8 + j] = a ? a1[j] : a0[j];
      __syncthreads();
      if (rm.rl == 0) {
        float s[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j] = 0.f;
        if (rm.g < (C >> 3)) {
          for (int r = 0; r < rm.rows_par; ++r)
#pragma unroll
            for (int j = 0; j < 8; ++j) s[j] += red[(r * GB + gl) * 8 + j];
        }
        *reinterpret_cast<float4*>(myrow + a * W + gl * 8) = make_float4(s[0], s[1], s[2], s[3]);
        *reinterpret_cast<float4*>(myrow + a * W + gl * 8 + 4) = make_float4(s[4], s[5], s[6], s[7]);
      }
    }
  }
  grid_barrier(p.ctr, nblocks);
  // ------------------------------------------------ phase 1b: distributed fixed-order fold of this slab's 2W columns
  {
    const int nb = gridDim.x;
    const int ncol = 2 * W;
    const int cpb = (ncol + nb - 1) / nb;  // columns per block
    const int c0 = blockIdx.x * cpb, c1 = min(c0 + cpb, ncol);
    const int TC = min(cpb, 256), RL = 256 / TC;
    const int tc = threadIdx.x % TC, rl = threadIdx.x / TC;
    const float* base = p.rows + (size_t)blockIdx.y * nb * ncol;
    for (int cb = c0; cb < c1; cb += TC) {  // uniform trip count over the block
      const int col = cb + tc;
      float part = 0.f;
      if (col < c1 && rl < RL) {
#pragma unroll 8
        for (int r = rl; r < nb; r += RL) part += __ldcg(base + (size_t)r * ncol + col);
      }
      __syncthreads();
      red[threadIdx.x] = part;
      __syncthreads();
      if (rl == 0 && col < c1) {
        float tot = 0.f;
        for (int q = 0; q < RL; ++q) tot += red[q * TC + tc];
        const int a = col / W, ch = blockIdx.y * W + (col - a * W);
        if (ch < C) {
          p.totals[(size_t)a * C + ch] = tot;
          float* pg = a == 0 ? p.dbeta : p.dgamma;
          if (pg) pg[ch] = p.accumulate ? pg[ch] + tot : tot;
        }
      }
    }
    if (p.sync.world > 0) __threadfence_system();
  }
  grid_barrier(p.ctr, 2u * nblocks);
  // ------------------------------------------------ SyncBN: ONE block exchanges the finished local totals with the world and
  // leaves the world's in p.totals
  float s0[8], s1[8];
  if (p.sync.world > 0) {
    if (blockIdx.x == 0 && blockIdx.y == 0)
      sync_exchange_block_f(p.sync, p.totals, 2 * C, (int)threadIdx.x, 256, [] { __syncthreads(); });
    grid_barrier(p.ctr, 3u * nblocks);
  }
  if (rm.active) {
    *reinterpret_cast<float4*>(s0) = __ldcg(reinterpret_cast<const float4*>(p.totals + co));
    *reinterpret_cast<float4*>(s0 + 4) = __ldcg(reinterpret_cast<const float4*>(p.totals + co + 4));
    *reinterpret_cast<float4*>(s1) = __ldcg(reinterpret_cast<const float4*>(p.totals + C + co));
    *reinterpret_cast<float4*>(s1 + 4) = __ldcg(reinterpret_cast<const float4*>(p.totals + C + co + 4));
  }
  // ------------------------------------------------ phase 2: apply
  if (rm.active) {
    float cA[8], cB[8], cC[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float a = gm[j] * istd[j];
      const float t0 = p.zero_sums ? 0.f : s0[j], t1 = p.zero_sums ? 0.f : s1[j];
      cA[j] = a;
      cB[j] = -a * istd[j] * t1 * p.inv_count;
      cC[j] = -a * t0 * p.inv_count - cB[j] * mean[j];
    }
#pragma unroll 2
    for (int64_t row = (int64_t)blockIdx.x * rm.rows_par + rm.rl; row < p.M; row += step) {
      float dz[8], xv[8];
      unpack8(*reinterpret_cast<const bf16x8*>(p.dout + row * p.lddo + co), dz);
      unpack8(*reinterpret_cast<const bf16x8*>(p.x + row * p.ldx + co), xv);
      if constexpr (REMASK) {
#pragma unroll
        for (int j = 0; j < 8; ++j) dz[j] = (fmaf(xv[j], cA[j], sh[j]) > 0.f) ? dz[j] : 0.f;
      } else if constexpr (MS == MaskSrc::BITS) {
        apply_mask_bits(p.mask[row * (C >> 3) + rm.g], keep_scale, dz);
      } else if (p.relu) {
        float o[8];
        unpack8(*reinterpret_cast<const bf16x8*>(p.out + row * p.ldo + co), o);
#pragma unroll
        for (int j = 0; j < 8; ++j) dz[j] = (o[j] > 0.f) ? dz[j] * keep_scale : 0.f;
      }
      if (p.dres) {
        float r[8];
        if (p.beta_res != 0.f) {
          unpack8(*reinterpret_cast<const bf16x8*>(p.dres + row * p.lddres + co), r);
#pragma unroll
          for (int j = 0; j < 8; ++j) r[j] = p.beta_res * r[j] + dz[j];
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) r[j] = dz[j];
        }
        *reinterpret_cast<bf16x8*>(p.dres + row * p.lddres + co) = pack8(r);
      }
      float o8[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o8[j] = fmaf(cA[j], dz[j], fmaf(cB[j], xv[j], cC[j]));
      if constexpr (ACC) {  // as bn_bwd_apply_kernel<MS, true>
        float old[8];
        unpack8(*reinterpret_cast<const bf16x8*>(p.dx + row * p.lddx + co), old);
#pragma unroll
        for (int j = 0; j < 8; ++j) o8[j] += old[j];
      }
      *reinterpret_cast<bf16x8*>(p.dx + row * p.lddx + co) = pack8(o8);
    }
  }
}

__global__ void bn_param_grad_kernel(const float* __restrict__ sums, int C, float* dgamma, float* dbeta, int accumulate) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (dbeta) dbeta[c] = accumulate ? dbeta[c] + sums[c] : sums[c];
  if (dgamma) dgamma[c] = accumulate ? dgamma[c] + sums[C + c] : sums[C + c];
}

// ------------------------------------------------------------------ pooling
__global__ void __launch_bounds__(256) maxpool_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                          uint8_t* __restrict__ idx, int N, int H, int W, int C, int P, int Q) {
  const int G = C >> 3;
  const int64_t total = (int64_t)N * P * Q * G;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    int64_t t = i / G;
    const int q = (int)(t % Q);
    t /= Q;
    const int p = (int)(t % P);
    const int n = (int)(t / P);
    float best[8];
    int bi[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      best[j] = -INFINITY;
      bi[j] = 0;
    }
    bool first = true;
    for (int r = 0; r < 3; ++r) {
      const int ih = 2 * p - 1 + r;
      if (ih < 0 || ih >= H) continue;
      for (int s = 0; s < 3; ++s) {
        const int iw = 2 * q - 1 + s;
        if (iw < 0 || iw >= W) continue;
        float f[8];
        unpack8(*reinterpret_cast<const bf16x8*>(x + (((int64_t)n * H + ih) * W + iw) * C + g * 8), f);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (first || f[j] > best[j]) {  // first maximum wins (matches ATen max_pool2d index selection)
            best[j] = f[j];
            bi[j] = r * 3 + s;
          }
        first = false;
      }
    }
    const int64_t o = (((int64_t)n * P + p) * Q + q) * C + g * 8;
    *reinterpret_cast<bf16x8*>(y + o) = pack8(best);
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      lo |= (uint32_t)bi[j] << (8 * j);
      hi |= (uint32_t)bi[j + 4] << (8 * j);
    }
    *reinterpret_cast<uint2*>(idx + o) = make_uint2(lo, hi);
  }
}

__global__ void __launch_bounds__(256) maxpool_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ idx,
                                                          __nv_bfloat16* __restrict__ dx, int N, int H, int W, int C, int P,
                                                          int Q) {
  const int G = C >> 3;
  const int64_t total = (int64_t)N * H * W * G;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    int64_t t = i / G;
    const int w = (int)(t % W);
    t /= W;
    const int h = (int)(t % H);
    const int n = (int)(t / H);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int r = 0; r < 3; ++r) {
      const int th = h + 1 - r;
      if (th < 0 || (th & 1)) continue;
      const int p = th >> 1;
      if (p >= P) continue;
      for (int s = 0; s < 3; ++s) {
        const int tw = w + 1 - s;
        if (tw < 0 || (tw & 1)) continue;
        const int q = tw >> 1;
        if (q >= Q) continue;
        const int64_t o = (((int64_t)n * P + p) * Q + q) * C + g * 8;
        const uint2 id = *reinterpret_cast<const uint2*>(idx + o);
        float f[8];
        unpack8(*reinterpret_cast<const bf16x8*>(dy + o), f);
        const int code = r * 3 + s;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if ((int)((id.x >> (8 * j)) & 0xff) == code) acc[j] += f[j];
          if ((int)((id.y >> (8 * j)) & 0xff) == code) acc[j + 4] += f[j + 4];
        }
      }
    }
    *reinterpret_cast<bf16x8*>(dx + (((int64_t)n * H + h) * W + w) * C + g * 8) = pack8(acc);
  }
}

// ---- 2x2 / stride-2 max pool with indices and max unpool (SegNet).  Floor mode, no padding: the windows never overlap,
// so all four ops are selections and move raw bf16 bits.  One uint8 code per pooled element, code = 2r + s.  Pointers
// are in 16-byte vectors (8 channels); G = C / 8.
union Raw8 {
  uint4 u;
  unsigned short h[8];
};

__device__ __forceinline__ float bf16_bits_to_float(unsigned short b) { return __uint_as_float((uint32_t)b << 16); }

// ATen's rule (max_pool2d_with_indices): scan the window in row-major order from -inf, take v > best || isnan(v); the
// index starts at the window's first element.  Starting from that element instead gives the same value and index.
// CEIL_RELU (FCN8's VGG trunk: conv -> ReLU -> MaxPool2d(2, 2, ceil_mode=True), fcn.py:20-22): P = ceil(H/2), Q = ceil(W/2),
// the last row / column windows of an odd H / W hold only their in-range elements, and the output is relu(window max).  The
// window max is > 0 or NaN exactly when the pool of the ReLU'd map picks a positive / NaN element, and then both rules pick
// the same element, so the code is ATen's on relu(x) there.  A window whose max is <= 0 pools to 0 and gets code bit 2 (4 +
// its raw 2r + s): the ReLU's backward zeroes its gradient, and the scatter, which matches codes 0-3 only, writes 0 for it.
template <bool CEIL_RELU>
__global__ void __launch_bounds__(256) maxpool2x2_fwd_kernel(const uint4* __restrict__ x, uint4* __restrict__ y,
                                                             uint2* __restrict__ code, int N, int H, int W, int G, int P, int Q) {
  const int64_t total = (int64_t)N * P * Q * G;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    int64_t t = i / G;
    const int q = (int)(t % Q);
    t /= Q;
    const int p = (int)(t % P);
    const int n = (int)(t / P);
    const int64_t b = (((int64_t)n * H + 2 * p) * W + 2 * q) * G + g;
    const bool s1 = !CEIL_RELU || 2 * q + 1 < W, r1 = !CEIL_RELU || 2 * p + 1 < H;
    const bool valid[4] = {true, s1, r1, r1 && s1};
    Raw8 v[4], o;
    v[0].u = x[b];
    v[1].u = s1 ? x[b + G] : v[0].u;
    v[2].u = r1 ? x[b + (int64_t)W * G] : v[0].u;
    v[3].u = (r1 && s1) ? x[b + (int64_t)W * G + G] : v[0].u;
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      unsigned short bits = v[0].h[j];
      float best = bf16_bits_to_float(bits);
      uint32_t c = 0;
#pragma unroll
      for (int k = 1; k < 4; ++k) {
        const float f = bf16_bits_to_float(v[k].h[j]);
        if (valid[k] && (f > best || isnan(f))) {
          best = f;
          bits = v[k].h[j];
          c = k;
        }
      }
      if (CEIL_RELU && !(best > 0.f) && !isnan(best)) {
        bits = 0;
        c |= 4u;
      }
      o.h[j] = bits;
      if (j < 4) lo |= c << (8 * j);
      else hi |= c << (8 * (j - 4));
    }
    y[i] = o.u;
    code[i] = make_uint2(lo, hi);
  }
}

// pooled [N,P,Q] -> full [N,H,W]: the value at its coded position of each window, zeros in the other three and on the row /
// column that floor mode dropped (H or W odd).  Writes every output element once.  The max-pool backward (dy -> dx) and
// the max-unpool forward (x -> y) are both this scatter.
__global__ void __launch_bounds__(256) unpool2x2_scatter_kernel(const uint4* __restrict__ src, const uint2* __restrict__ code,
                                                                uint4* __restrict__ dst, int N, int H, int W, int G, int P, int Q) {
  const int P2 = (H + 1) >> 1, Q2 = (W + 1) >> 1;
  const int64_t total = (int64_t)N * P2 * Q2 * G;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    int64_t t = i / G;
    const int q = (int)(t % Q2);
    t /= Q2;
    const int p = (int)(t % P2);
    const int n = (int)(t / P2);
    Raw8 o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k].u = make_uint4(0u, 0u, 0u, 0u);
    if (p < P && q < Q) {
      const int64_t pi = (((int64_t)n * P + p) * Q + q) * G + g;
      Raw8 v;
      v.u = src[pi];
      const uint2 c = code[pi];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t cj = ((j < 4 ? c.x : c.y) >> (8 * (j & 3))) & 0xffu;
#pragma unroll
        for (int k = 0; k < 4; ++k) o[k].h[j] = (cj == (uint32_t)k) ? v.h[j] : (unsigned short)0;
      }
    }
    const int64_t b = (((int64_t)n * H + 2 * p) * W + 2 * q) * G + g;
    const bool r1 = 2 * p + 1 < H, s1 = 2 * q + 1 < W;
    dst[b] = o[0].u;
    if (s1) dst[b + G] = o[1].u;
    if (r1) dst[b + (int64_t)W * G] = o[2].u;
    if (r1 && s1) dst[b + (int64_t)W * G + G] = o[3].u;
  }
}

// full [N,H,W] -> pooled [N,P,Q]: each pooled element takes the value at its coded position (the max-unpool backward).
__global__ void __launch_bounds__(256) unpool2x2_gather_kernel(const uint4* __restrict__ src, const uint2* __restrict__ code,
                                                               uint4* __restrict__ dst, int N, int H, int W, int G, int P, int Q) {
  const int64_t total = (int64_t)N * P * Q * G;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    int64_t t = i / G;
    const int q = (int)(t % Q);
    t /= Q;
    const int p = (int)(t % P);
    const int n = (int)(t / P);
    const int64_t b = (((int64_t)n * H + 2 * p) * W + 2 * q) * G + g;
    Raw8 v[4], o;
    v[0].u = src[b];
    v[1].u = src[b + G];
    v[2].u = src[b + (int64_t)W * G];
    v[3].u = src[b + (int64_t)W * G + G];
    const uint2 c = code[i];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t cj = ((j < 4 ? c.x : c.y) >> (8 * (j & 3))) & 0xffu;
      o.h[j] = cj == 0 ? v[0].h[j] : cj == 1 ? v[1].h[j] : cj == 2 ? v[2].h[j] : v[3].h[j];
    }
    dst[i] = o.u;
  }
}

__device__ __forceinline__ int bin_lo(int i, int L, int b) { return (i * L) / b; }
__device__ __forceinline__ int bin_hi(int i, int L, int b) { return ((i + 1) * L + b - 1) / b; }

// grid (N*bins*bins, ceil(G/32)); block 256 = 32 channel groups x 8 pixel lanes
__global__ void __launch_bounds__(256) adaptive_avgpool_fwd_kernel(const __nv_bfloat16* __restrict__ x, int ldx,
                                                                   __nv_bfloat16* __restrict__ y, int N, int H, int W, int C,
                                                                   int bins) {
  const int G = C >> 3;
  const int gl = threadIdx.x & 31, pl = threadIdx.x >> 5;
  const int g = blockIdx.y * 32 + gl;
  int t = blockIdx.x;
  const int j = t % bins;
  t /= bins;
  const int i = t % bins;
  const int n = t / bins;
  const int h0 = bin_lo(i, H, bins), h1 = bin_hi(i, H, bins), w0 = bin_lo(j, W, bins), w1 = bin_hi(j, W, bins);
  const int bw = w1 - w0, cnt = (h1 - h0) * bw;
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = 0.f;
  if (g < G) {
    for (int e = pl; e < cnt; e += 8) {
      const int h = h0 + e / bw, w = w0 + e % bw;
      float f[8];
      unpack8(*reinterpret_cast<const bf16x8*>(x + (((int64_t)n * H + h) * W + w) * ldx + g * 8), f);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += f[k];
    }
  }
  __shared__ float red[8][32][8];
#pragma unroll
  for (int k = 0; k < 8; ++k) red[pl][gl][k] = acc[k];
  __syncthreads();
  if (pl == 0 && g < G) {
    float s[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      s[k] = 0.f;
      for (int l = 0; l < 8; ++l) s[k] += red[l][gl][k];
      s[k] /= (float)cnt;
    }
    *reinterpret_cast<bf16x8*>(y + (((int64_t)n * bins + i) * bins + j) * C + g * 8) = pack8(s);
  }
}

// nn.AvgPool2d(2, 2), floor mode (DenseNet's transition1): y[n][p][q] = mean of the 2x2 window at (2p, 2q); a trailing odd
// row / column is dropped.  The fp32 sum of the four bf16 values is rounded to bf16 once.  ldx / ldy: channel pitches (y may
// be a channel slice of a concat buffer).
__global__ void __launch_bounds__(256) avgpool2x2_fwd_kernel(const __nv_bfloat16* __restrict__ x, int ldx,
                                                             __nv_bfloat16* __restrict__ y, int ldy, int N, int H, int W, int C) {
  const int G = C >> 3, P = H >> 1, Q = W >> 1;
  const int64_t total = (int64_t)N * P * Q * G;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    int64_t t = i / G;
    const int q = (int)(t % Q);
    t /= Q;
    const int pp = (int)(t % P);
    const int n = (int)(t / P);
    const int64_t r0 = ((int64_t)n * H + 2 * pp) * W + 2 * q;
    float a[8], b[8], c[8], d[8], o[8];
    unpack8(*reinterpret_cast<const bf16x8*>(x + r0 * ldx + g * 8), a);
    unpack8(*reinterpret_cast<const bf16x8*>(x + (r0 + 1) * ldx + g * 8), b);
    unpack8(*reinterpret_cast<const bf16x8*>(x + (r0 + W) * ldx + g * 8), c);
    unpack8(*reinterpret_cast<const bf16x8*>(x + (r0 + W + 1) * ldx + g * 8), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = ((a[j] + b[j]) + (c[j] + d[j])) * 0.25f;
    *reinterpret_cast<bf16x8*>(y + (((int64_t)n * P + pp) * Q + q) * ldy + g * 8) = pack8(o);
  }
}

// its backward: dx = beta * dx + dy / 4 over every element of dx (0 for a dropped row / column), in fp32, rounded once
__global__ void __launch_bounds__(256) avgpool2x2_bwd_kernel(const __nv_bfloat16* __restrict__ dy, int lddy,
                                                             __nv_bfloat16* __restrict__ dx, int lddx, int N, int H, int W, int C,
                                                             float beta) {
  const int G = C >> 3, P = H >> 1, Q = W >> 1;
  const int64_t total = (int64_t)N * H * W * G;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    const int64_t r = i / G;
    const int w = (int)(r % W);
    const int h = (int)((r / W) % H);
    const int n = (int)(r / ((int64_t)W * H));
    float v[8];
    if (h < 2 * P && w < 2 * Q) {
      unpack8(*reinterpret_cast<const bf16x8*>(dy + (((int64_t)n * P + (h >> 1)) * Q + (w >> 1)) * lddy + g * 8), v);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] *= 0.25f;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.f;
    }
    __nv_bfloat16* o = dx + r * lddx + g * 8;
    if (beta != 0.f) {
      float old[8];
      unpack8(*reinterpret_cast<const bf16x8*>(o), old);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = fmaf(beta, old[j], v[j]);
    }
    *reinterpret_cast<bf16x8*>(o) = pack8(v);
  }
}

__global__ void __launch_bounds__(256) adaptive_avgpool_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                                   __nv_bfloat16* __restrict__ dx, int lddx, int N, int H,
                                                                   int W, int C, int bins, float beta) {
  const int G = C >> 3;
  const int64_t total = (int64_t)N * H * W * G;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(idx % G);
    int64_t t = idx / G;
    const int w = (int)(t % W);
    t /= W;
    const int h = (int)(t % H);
    const int n = (int)(t / H);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int i = 0; i < bins; ++i) {
      const int h0 = bin_lo(i, H, bins), h1 = bin_hi(i, H, bins);
      if (h < h0 || h >= h1) continue;
      for (int j = 0; j < bins; ++j) {
        const int w0 = bin_lo(j, W, bins), w1 = bin_hi(j, W, bins);
        if (w < w0 || w >= w1) continue;
        float f[8];
        unpack8(*reinterpret_cast<const bf16x8*>(dy + (((int64_t)n * bins + i) * bins + j) * C + g * 8), f);
        const float inv = 1.f / (float)((h1 - h0) * (w1 - w0));
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] += f[k] * inv;
      }
    }
    __nv_bfloat16* o = dx + (((int64_t)n * H + h) * W + w) * lddx + g * 8;
    if (beta != 0.f) {
      float f[8];
      unpack8(*reinterpret_cast<const bf16x8*>(o), f);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += beta * f[k];
    }
    *reinterpret_cast<bf16x8*>(o) = pack8(acc);
  }
}

// ------------------------------------------------------------------ bilinear
// Source index exactly as ATen's area_pixel_compute_source_index (float arithmetic).
struct Lerp {
  int i0, i1;
  float l1;
};
__device__ __forceinline__ Lerp src_index(int dst, float scale, int in_size, int align_corners) {
  float s;
  if (align_corners) {
    s = scale * (float)dst;
  } else {
    s = scale * ((float)dst + 0.5f) - 0.5f;
    if (s < 0.f) s = 0.f;
  }
  Lerp r;
  r.i0 = (int)s;
  if (r.i0 > in_size - 1) r.i0 = in_size - 1;
  r.i1 = r.i0 + ((r.i0 < in_size - 1) ? 1 : 0);
  r.l1 = s - (float)r.i0;
  return r;
}
static inline float resize_scale(int in_size, int out_size, int align_corners) {
  if (align_corners) return out_size > 1 ? (float)(in_size - 1) / (float)(out_size - 1) : 0.f;
  return (float)in_size / (float)out_size;
}
// candidate output range whose source support may touch input index y
__device__ __forceinline__ void dst_range(int y, float scale, int out_size, int align_corners, int& lo, int& hi) {
  if (scale <= 0.f) {
    lo = 0;
    hi = out_size - 1;
    return;
  }
  float a, b;
  if (align_corners) {
    a = ((float)y - 1.f) / scale;
    b = ((float)y + 1.f) / scale;
  } else {
    a = ((float)y - 0.5f) / scale - 0.5f;
    b = ((float)y + 1.5f) / scale - 0.5f;
  }
  lo = max(0, (int)floorf(a) - 1);
  hi = min(out_size - 1, (int)ceilf(b) + 1);
}

__global__ void __launch_bounds__(256) bilinear_fwd_kernel(const __nv_bfloat16* __restrict__ x, int ldx,
                                                           __nv_bfloat16* __restrict__ y, int ldy, int N, int Hi, int Wi,
                                                           int Ho, int Wo, int C, int ac, float sh, float sw) {
  const int G = C >> 3;
  const int64_t total = (int64_t)N * Ho * Wo * G;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    int64_t t = i / G;
    const int ox = (int)(t % Wo);
    t /= Wo;
    const int oy = (int)(t % Ho);
    const int n = (int)(t / Ho);
    const Lerp ly = src_index(oy, sh, Hi, ac), lx = src_index(ox, sw, Wi, ac);
    const __nv_bfloat16* base = x + (int64_t)n * Hi * Wi * ldx + g * 8;
    float a[8], b[8], c[8], d[8], o[8];
    unpack8(*reinterpret_cast<const bf16x8*>(base + ((int64_t)ly.i0 * Wi + lx.i0) * ldx), a);
    unpack8(*reinterpret_cast<const bf16x8*>(base + ((int64_t)ly.i0 * Wi + lx.i1) * ldx), b);
    unpack8(*reinterpret_cast<const bf16x8*>(base + ((int64_t)ly.i1 * Wi + lx.i0) * ldx), c);
    unpack8(*reinterpret_cast<const bf16x8*>(base + ((int64_t)ly.i1 * Wi + lx.i1) * ldx), d);
    const float h1 = ly.l1, h0 = 1.f - h1, w1 = lx.l1, w0 = 1.f - w1;
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = h0 * (w0 * a[k] + w1 * b[k]) + h1 * (w0 * c[k] + w1 * d[k]);
    *reinterpret_cast<bf16x8*>(y + (((int64_t)n * Ho + oy) * Wo + ox) * ldy + g * 8) = pack8(o);
  }
}

// weights of input index `y` in every output index of [lo, hi]: w[k] for output lo+k (0 when y is not a source of it)
__device__ __forceinline__ int lerp_weights(int y, float scale, int in_size, int out_size, int ac, float* w, int maxn, int& lo) {
  int hi;
  dst_range(y, scale, out_size, ac, lo, hi);
  // trim the conservative range to the outputs that really reference y
  int n = 0, first = -1, last = -1;
  for (int o = lo; o <= hi; ++o) {
    const Lerp l = src_index(o, scale, in_size, ac);
    float wy = 0.f;
    if (l.i0 == y) wy += 1.f - l.l1;
    if (l.i1 == y) wy += l.l1;
    if (wy != 0.f) {
      if (first < 0) first = o;
      last = o;
    }
  }
  if (first < 0) return 0;
  n = last - first + 1;
  if (n > maxn) return -1;
  for (int k = 0; k < n; ++k) {
    const Lerp l = src_index(first + k, scale, in_size, ac);
    float wy = 0.f;
    if (l.i0 == y) wy += 1.f - l.l1;
    if (l.i1 == y) wy += l.l1;
    w[k] = wy;
  }
  lo = first;
  return n;
}

__global__ void __launch_bounds__(256) bilinear_bwd_kernel(const __nv_bfloat16* __restrict__ dy, int lddy,
                                                           __nv_bfloat16* __restrict__ dx, int lddx, int N, int Hi, int Wi,
                                                           int Ho, int Wo, int C, int ac, float sh, float sw, float beta) {
  const int G = C >> 3;
  const int64_t total = (int64_t)N * Hi * Wi * G;
  constexpr int MAXN = 24;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    int64_t t = i / G;
    const int x = (int)(t % Wi);
    t /= Wi;
    const int y = (int)(t % Hi);
    const int n = (int)(t / Hi);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    float wy[MAXN], wx[MAXN];
    int oy0, ox0;
    const int ny = lerp_weights(y, sh, Hi, Ho, ac, wy, MAXN, oy0);
    const int nx = lerp_weights(x, sw, Wi, Wo, ac, wx, MAXN, ox0);
    if (ny >= 0 && nx >= 0) {
      for (int a = 0; a < ny; ++a) {
        if (wy[a] == 0.f) continue;
        const __nv_bfloat16* rowp = dy + (((int64_t)n * Ho + oy0 + a) * Wo + ox0) * lddy + g * 8;
        for (int b = 0; b < nx; ++b) {
          if (wx[b] == 0.f) continue;
          float f[8];
          unpack8(*reinterpret_cast<const bf16x8*>(rowp + (int64_t)b * lddy), f);
          const float wgt = wy[a] * wx[b];
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[k] = fmaf(wgt, f[k], acc[k]);
        }
      }
    } else {
      // very large magnification (e.g. the 1x1 global-pool branch): generic loop over the conservative range
      int oy1, ox1;
      dst_range(y, sh, Ho, ac, oy0, oy1);
      dst_range(x, sw, Wo, ac, ox0, ox1);
      for (int oy = oy0; oy <= oy1; ++oy) {
        const Lerp ly = src_index(oy, sh, Hi, ac);
        float wyy = 0.f;
        if (ly.i0 == y) wyy += 1.f - ly.l1;
        if (ly.i1 == y) wyy += ly.l1;
        if (wyy == 0.f) continue;
        for (int ox = ox0; ox <= ox1; ++ox) {
          const Lerp lx = src_index(ox, sw, Wi, ac);
          float wxx = 0.f;
          if (lx.i0 == x) wxx += 1.f - lx.l1;
          if (lx.i1 == x) wxx += lx.l1;
          if (wxx == 0.f) continue;
          float f[8];
          unpack8(*reinterpret_cast<const bf16x8*>(dy + (((int64_t)n * Ho + oy) * Wo + ox) * lddy + g * 8), f);
          const float wgt = wyy * wxx;
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[k] = fmaf(wgt, f[k], acc[k]);
        }
      }
    }
    __nv_bfloat16* o = dx + (((int64_t)n * Hi + y) * Wi + x) * lddx + g * 8;
    if (beta != 0.f) {
      float f[8];
      unpack8(*reinterpret_cast<const bf16x8*>(o), f);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += beta * f[k];
    }
    *reinterpret_cast<bf16x8*>(o) = pack8(acc);
  }
}

// low-res NHWC fp32 logits -> full-res NCHW fp32 logits; threads run along ox for coalesced NCHW stores
__global__ void __launch_bounds__(256) bilinear_logits_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int N,
                                                                  int Hi, int Wi, int Ho, int Wo, int C, int ac, float sh,
                                                                  float sw) {
  const int64_t total = (int64_t)N * Ho * Wo;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ox = (int)(i % Wo);
    int64_t t = i / Wo;
    const int oy = (int)(t % Ho);
    const int n = (int)(t / Ho);
    const Lerp ly = src_index(oy, sh, Hi, ac), lx = src_index(ox, sw, Wi, ac);
    const float* base = x + (int64_t)n * Hi * Wi * C;
    const float* pa = base + ((int64_t)ly.i0 * Wi + lx.i0) * C;
    const float* pb = base + ((int64_t)ly.i0 * Wi + lx.i1) * C;
    const float* pc = base + ((int64_t)ly.i1 * Wi + lx.i0) * C;
    const float* pd = base + ((int64_t)ly.i1 * Wi + lx.i1) * C;
    const float h1 = ly.l1, h0 = 1.f - h1, w1 = lx.l1, w0 = 1.f - w1;
    float* o = y + (int64_t)n * C * Ho * Wo + (int64_t)oy * Wo + ox;
    for (int c = 0; c < C; ++c)
      o[(int64_t)c * Ho * Wo] = h0 * (w0 * pa[c] + w1 * pb[c]) + h1 * (w0 * pc[c] + w1 * pd[c]);
  }
}

// NCHW fp32 grad -> low-res NHWC bf16 grad (pitch lddx, channels >= C zero-filled up to lddx)
__global__ void __launch_bounds__(128) bilinear_logits_bwd_kernel(const float* __restrict__ dy, __nv_bfloat16* __restrict__ dx,
                                                                  int lddx, int N, int Hi, int Wi, int Ho, int Wo, int C,
                                                                  int ac, float sh, float sw) {
  const int64_t total = (int64_t)N * Hi * Wi;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % Wi);
    int64_t t = i / Wi;
    const int y = (int)(t % Hi);
    const int n = (int)(t / Hi);
    int oy0, oy1, ox0, ox1;
    dst_range(y, sh, Ho, ac, oy0, oy1);
    dst_range(x, sw, Wo, ac, ox0, ox1);
    __nv_bfloat16* o = dx + (((int64_t)n * Hi + y) * Wi + x) * lddx;
    for (int c = 0; c < C; ++c) {
      const float* src = dy + ((int64_t)n * C + c) * Ho * Wo;
      float acc = 0.f;
      for (int oy = oy0; oy <= oy1; ++oy) {
        const Lerp ly = src_index(oy, sh, Hi, ac);
        float wy = 0.f;
        if (ly.i0 == y) wy += 1.f - ly.l1;
        if (ly.i1 == y) wy += ly.l1;
        if (wy == 0.f) continue;
        for (int ox = ox0; ox <= ox1; ++ox) {
          const Lerp lx = src_index(ox, sw, Wi, ac);
          float wx = 0.f;
          if (lx.i0 == x) wx += 1.f - lx.l1;
          if (lx.i1 == x) wx += lx.l1;
          if (wx != 0.f) acc += wy * wx * src[(int64_t)oy * Wo + ox];
        }
      }
      o[c] = f2bf(acc);
    }
    for (int c = C; c < lddx; ++c) o[c] = f2bf(0.f);
  }
}

// ------------------------------------------------------------------ pixel shuffle (nn.PixelShuffle, duc_hdc.py:22,30)
// Source channel of output (c, oy, ox) is c*r*r + (oy % r)*r + (ox % r) at source pixel (oy / r, ox / r).  Pure
// permutations: every output is one input element, so the results are exact.
__global__ void __launch_bounds__(256) pixel_shuffle_fwd_kernel(const __nv_bfloat16* __restrict__ x, int ldx,
                                                                __nv_bfloat16* __restrict__ y, int ldy, int N, int H, int W,
                                                                int C, int r, int Ho, int Wo) {
  const int64_t total = (int64_t)N * Ho * Wo * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    int64_t t = i / C;
    const int ox = (int)(t % Wo);
    t /= Wo;
    const int oy = (int)(t % Ho);
    const int n = (int)(t / Ho);
    const int sc = (c * r + oy % r) * r + ox % r;
    y[(((int64_t)n * Ho + oy) * Wo + ox) * ldy + c] = x[(((int64_t)n * H + oy / r) * W + ox / r) * ldx + sc];
  }
}

// dx = beta*dx + shuffle^T(dy); source positions the crop dropped get a zero gradient
__global__ void __launch_bounds__(256) pixel_shuffle_bwd_kernel(const __nv_bfloat16* __restrict__ dy, int lddy,
                                                                __nv_bfloat16* __restrict__ dx, int lddx, int N, int H, int W,
                                                                int C, int r, int Ho, int Wo, float beta) {
  const int Cr = C * r * r;
  const int64_t total = (int64_t)N * H * W * Cr;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int sc = (int)(i % Cr);
    int64_t t = i / Cr;
    const int w = (int)(t % W);
    t /= W;
    const int h = (int)(t % H);
    const int n = (int)(t / H);
    const int c = sc / (r * r), oy = h * r + (sc / r) % r, ox = w * r + sc % r;
    float v = 0.f;
    if (oy < Ho && ox < Wo) v = bf2f(dy[(((int64_t)n * Ho + oy) * Wo + ox) * lddy + c]);
    __nv_bfloat16* o = dx + (((int64_t)n * H + h) * W + w) * lddx + sc;
    if (beta != 0.f) v += beta * bf2f(*o);
    *o = f2bf(v);
  }
}

// low-res NHWC bf16 [N,h,w,r*r*C] -> full-res NCHW fp32 [N,C,r*h,r*w]; threads run along ox for coalesced NCHW stores
__global__ void __launch_bounds__(256) pixel_shuffle_logits_fwd_kernel(const __nv_bfloat16* __restrict__ x, int ldx,
                                                                       float* __restrict__ y, int N, int h, int w, int C,
                                                                       int r) {
  const int Ho = h * r, Wo = w * r;
  const int64_t total = (int64_t)N * C * Ho * Wo;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ox = (int)(i % Wo);
    int64_t t = i / Wo;
    const int oy = (int)(t % Ho);
    t /= Ho;
    const int c = (int)(t % C);
    const int n = (int)(t / C);
    y[i] = bf2f(x[(((int64_t)n * h + oy / r) * w + ox / r) * ldx + (c * r + oy % r) * r + ox % r]);
  }
}

// NCHW fp32 grad -> low-res NHWC bf16 grad (pitch lddx, channels >= r*r*C zero-filled up to lddx)
__global__ void __launch_bounds__(256) pixel_shuffle_logits_bwd_kernel(const float* __restrict__ dy,
                                                                       __nv_bfloat16* __restrict__ dx, int lddx, int N, int h,
                                                                       int w, int C, int r) {
  const int Cr = C * r * r, Ho = h * r, Wo = w * r;
  const int64_t total = (int64_t)N * h * w * lddx;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int sc = (int)(i % lddx);
    int64_t t = i / lddx;
    const int x0 = (int)(t % w);
    t /= w;
    const int y0 = (int)(t % h);
    const int n = (int)(t / h);
    float v = 0.f;
    if (sc < Cr) {
      const int c = sc / (r * r), oy = y0 * r + (sc / r) % r, ox = x0 * r + sc % r;
      v = dy[(((int64_t)n * C + c) * Ho + oy) * Wo + ox];
    }
    dx[i] = f2bf(v);
  }
}

// ------------------------------------------------------------------ misc
__global__ void nhwc_to_nchw_kernel(const void* __restrict__ x, int ldx, int x_dtype, float* __restrict__ y, int N, int H,
                                    int W, int C) {
  const int64_t total = (int64_t)N * C * H * W;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int w = (int)(i % W);
    int64_t t = i / W;
    const int h = (int)(t % H);
    t /= H;
    const int c = (int)(t % C);
    const int n = (int)(t / C);
    const int64_t src = (((int64_t)n * H + h) * W + w) * ldx + c;
    y[i] = x_dtype == SEG_DT_BF16 ? bf2f(reinterpret_cast<const __nv_bfloat16*>(x)[src])
                                  : reinterpret_cast<const float*>(x)[src];
  }
}

__global__ void axpby_kernel(const __nv_bfloat16* __restrict__ x, int ldx, __nv_bfloat16* __restrict__ y, int ldy, int64_t M,
                             int C, float beta) {
  const int G = C >> 3;
  const int64_t total = M * G;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    const int64_t row = i / G;
    float a[8];
    unpack8(*reinterpret_cast<const bf16x8*>(x + row * ldx + g * 8), a);
    if (beta != 0.f) {
      float b[8];
      unpack8(*reinterpret_cast<const bf16x8*>(y + row * ldy + g * 8), b);
#pragma unroll
      for (int k = 0; k < 8; ++k) a[k] += beta * b[k];
    }
    *reinterpret_cast<bf16x8*>(y + row * ldy + g * 8) = pack8(a);
  }
}

// ReLU + nn.Dropout(p) (FCN8's conv6 / conv7, fcn.py:49-51): the element index r * C + c and the seed (+ the device step
// counter) feed hash_uniform exactly as in bn_apply's dropout, so graph replays draw fresh masks.  The backward reads the
// keep mask from out > 0 (a kept element of a positive input is positive, a dropped or ReLU'd one is 0).
__global__ void relu_dropout_fwd_kernel(const __nv_bfloat16* __restrict__ x, int ldx, __nv_bfloat16* __restrict__ y, int ldy,
                                        int64_t M, int C, float drop_p, uint64_t seed, const uint64_t* __restrict__ step_ctr) {
  if (step_ctr) seed += (*step_ctr) * 0x9E3779B97F4A7C15ull;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const int G = C >> 3;
  const int64_t total = M * G;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    const int64_t row = i / G;
    float a[8];
    unpack8(*reinterpret_cast<const bf16x8*>(x + row * ldx + g * 8), a);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      a[k] = fmaxf(a[k], 0.f);
      if (drop_p > 0.f) a[k] = hash_uniform(seed, (uint64_t)(row * C + g * 8 + k)) >= drop_p ? a[k] * keep_scale : 0.f;
    }
    *reinterpret_cast<bf16x8*>(y + row * ldy + g * 8) = pack8(a);
  }
}
__global__ void relu_dropout_bwd_kernel(const __nv_bfloat16* __restrict__ dy, int lddy, const __nv_bfloat16* __restrict__ y, int ldy,
                                        __nv_bfloat16* __restrict__ dx, int lddx, int64_t M, int C, float drop_p, float beta) {
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const int G = C >> 3;
  const int64_t total = M * G;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    const int64_t row = i / G;
    float d[8], o[8];
    unpack8(*reinterpret_cast<const bf16x8*>(dy + row * lddy + g * 8), d);
    unpack8(*reinterpret_cast<const bf16x8*>(y + row * ldy + g * 8), o);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = o[k] > 0.f ? d[k] * keep_scale : 0.f;
    if (beta != 0.f) {
      float b[8];
      unpack8(*reinterpret_cast<const bf16x8*>(dx + row * lddx + g * 8), b);
#pragma unroll
      for (int k = 0; k < 8; ++k) d[k] += beta * b[k];
    }
    *reinterpret_cast<bf16x8*>(dx + row * lddx + g * 8) = pack8(d);
  }
}

__global__ void counter_add_kernel(uint64_t* ctr, uint64_t inc) {
  if (threadIdx.x == 0 && blockIdx.x == 0) *ctr += inc;
}

// standalone ReLU (Xception: F.relu(low_level) before block2, deeplabv3_plus.py:210)
__global__ void relu_fwd_kernel(const __nv_bfloat16* __restrict__ x, int ldx, __nv_bfloat16* __restrict__ y, int ldy, int64_t M, int C) {
  const int G = C >> 3;
  const int64_t total = M * G;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    const int64_t row = i / G;
    float a[8];
    unpack8(*reinterpret_cast<const bf16x8*>(x + row * ldx + g * 8), a);
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] = fmaxf(a[k], 0.f);
    *reinterpret_cast<bf16x8*>(y + row * ldy + g * 8) = pack8(a);
  }
}
__global__ void relu_bwd_kernel(const __nv_bfloat16* __restrict__ dy, int lddy, const __nv_bfloat16* __restrict__ y, int ldy,
                                __nv_bfloat16* __restrict__ dx, int lddx, int64_t M, int C, float beta) {
  const int G = C >> 3;
  const int64_t total = M * G;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    const int64_t row = i / G;
    float d[8], o[8];
    unpack8(*reinterpret_cast<const bf16x8*>(dy + row * lddy + g * 8), d);
    unpack8(*reinterpret_cast<const bf16x8*>(y + row * ldy + g * 8), o);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = o[k] > 0.f ? d[k] : 0.f;
    if (beta != 0.f) {
      float b[8];
      unpack8(*reinterpret_cast<const bf16x8*>(dx + row * lddx + g * 8), b);
#pragma unroll
      for (int k = 0; k < 8; ++k) d[k] += beta * b[k];
    }
    *reinterpret_cast<bf16x8*>(dx + row * lddx + g * 8) = pack8(d);
  }
}

struct SgdChunkArgs {
  float* const* params;
  float* const* grads;
  float* const* bufs;
  const int64_t* sizes;
  const float* lrs;
};
// one block-row (blockIdx.y) per tensor, grid-stride inside
// hyper != nullptr: (momentum, weight decay) are read from device memory, so a schedule that changes the momentum every
// iteration (OneCycle, utils/lr_scheduler.py:24-59) also works when the step is replayed from a CUDA graph
__global__ void sgd_kernel(SgdChunkArgs a, float momentum, float wd, int first_step, float grad_scale,
                           const float* __restrict__ hyper) {
  if (hyper != nullptr) {
    momentum = hyper[0];
    wd = hyper[1];
  }
  const int t = blockIdx.y;
  float* p = a.params[t];
  const float* g = a.grads[t];
  float* b = a.bufs[t];
  const int64_t n = a.sizes[t];
  const float lr = a.lrs[t];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float d = g[i] * grad_scale + wd * p[i];
    if (momentum != 0.f) {
      const float m = first_step ? d : momentum * b[i] + d;
      b[i] = m;
      d = m;
    }
    p[i] -= lr * d;
  }
}

}  // namespace seg

// =================================================================== C ABI
using namespace seg;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define BF(p) reinterpret_cast<__nv_bfloat16*>(p)
#define CBF(p) reinterpret_cast<const __nv_bfloat16*>(p)

extern "C" {

int seg_pack_weight(const float* w, void* out, int K, int C, int R, int S, int Cpad, void* stream) {
  const int64_t total = (int64_t)R * S * K * Cpad;
  pack_weight_kernel<<<grid_for(total, 256), 256, 0, ST(stream)>>>(w, BF(out), K, C, R, S, Cpad);
  return check_launch("pack_weight");
}
int seg_unpack_wgrad(const float* dw, float* g, int K, int C, int R, int S, int Cpad, float beta, void* stream) {
  const int64_t total = (int64_t)K * C * R * S;
  unpack_wgrad_kernel<<<grid_for(total, 256), 256, 0, ST(stream)>>>(dw, g, K, C, R, S, Cpad, beta);
  return check_launch("unpack_wgrad");
}
int seg_pack_weights_batched(const void* table, int n, int64_t total, void* stream) {
  if (n <= 0) return 0;
  SEG_REQUIRE(n <= 65535, "too many convs");
  pack_weights_batched_kernel<<<dim3(48, (unsigned)n, 1), 256, 0, ST(stream)>>>(reinterpret_cast<const PackEntry*>(table), n, total);
  return check_launch("pack_weights_batched");
}
int seg_unpack_wgrads_batched(const void* table, int n, int64_t total, float beta, void* stream) {
  if (n <= 0) return 0;
  SEG_REQUIRE(n <= 65535, "too many convs");
  unpack_wgrads_batched_kernel<<<dim3(48, (unsigned)n, 1), 256, 0, ST(stream)>>>(reinterpret_cast<const PackEntry*>(table), n,
                                                                                 total, beta);
  return check_launch("unpack_wgrads_batched");
}
int seg_pack_entry_bytes(void) { return (int)sizeof(PackEntry); }
int seg_im2col(const seg_conv_desc* d, const void* x, int x_nchw_f32, void* col, int Kpad, void* stream) {
  SEG_REQUIRE(Kpad >= d->R * d->S * d->C, "im2col: Kpad too small");
  SEG_REQUIRE(Kpad % 8 == 0, "im2col: Kpad must be a multiple of 8");
  const int64_t total = (int64_t)d->N * d->P * d->Q * (Kpad / 8);
  im2col_kernel<<<grid_for(total, 256), 256, 0, ST(stream)>>>(*d, x, x_nchw_f32, BF(col), Kpad);
  return check_launch("im2col");
}

// grid for the channel-group-stationary streaming kernels: full occupancy (8 blocks of 256 threads per SM)
// Grid of the channel-group-stationary streaming kernels.  Every thread pays a fixed prologue (per-channel coefficients,
// and for the reductions a block-level fold + atomics), so small maps get FEWER, fatter blocks: aim at >= 8 rows per
// thread, but never fewer than two blocks per SM (or one row group per block), and at most eight blocks per SM.
static dim3 rowmap_grid(int64_t M, int C, int rows_per_thread = 8) {
  const int G = C / 8;
  const int GB = G < 256 ? G : 256;
  const int rows_par = 256 / GB;
  const int gy = ceil_div(G, GB);
  const int64_t groups = ceil_div64(M, rows_par);  // block-iterations needed to cover all rows
  int64_t gx = ceil_div64(groups, rows_per_thread);
  const int64_t floor_blocks = ((int64_t)num_sms() * 2 + gy - 1) / gy;
  if (gx < floor_blocks) gx = floor_blocks < groups ? floor_blocks : groups;
  const int64_t cap = ((int64_t)num_sms() * 8 + gy - 1) / gy;
  if (gx > cap) gx = cap;
  if (gx < 1) gx = 1;
  return dim3((unsigned)gx, (unsigned)gy, 1);
}

static dim3 colreduce_grid(int64_t M, int C) {
  const int G = C / 8;
  const int GB = G < 256 ? G : 256;
  const int rows_par = 256 / GB;
  const int gy = ceil_div(G, GB);
  int64_t gx = ceil_div64(M, (int64_t)rows_par * 4);
  const int64_t cap = (int64_t)num_sms() * 8 / gy + 1;
  if (gx > cap) gx = cap;
  if (gx < 1) gx = 1;
  return dim3((unsigned)gx, (unsigned)gy, 1);
}

static SyncDesc to_sync(const seg_sync_desc* sync) { return sync ? *sync : SyncDesc{}; }
}  // extern "C"
namespace seg {
// also used by the CUDA-core conv path (seg_conv_simt.cu) for its BatchNorm statistics
int bn_stats_launch(const void* x, int64_t M, int C, int ldx, double* stats, const seg_sync_desc* sync, unsigned* ticket,
                    cudaStream_t stream) {
  SEG_REQUIRE(C % 8 == 0 && ldx % 8 == 0, "bn_stats: C/ldx must be multiples of 8 (C=%d ldx=%d)", C, ldx);
  SEG_REQUIRE(!sync || ticket, "bn_stats: SyncBN needs a zeroed ticket word");
  if (sync && sync_check_desc(sync, 4ll * C, "bn_stats")) return 1;  // 2C fp64 totals
  bn_stats_kernel<<<colreduce_grid(M, C), 256, 0, stream>>>(CBF(x), M, C, ldx, stats, to_sync(sync), ticket);
  return check_launch("bn_stats");
}
}  // namespace seg
extern "C" {
int seg_bn_stats(const void* x, int64_t M, int C, int ldx, double* stats, const seg_sync_desc* sync, void* sync_ticket, void* stream) {
  return bn_stats_launch(x, M, C, ldx, stats, sync, reinterpret_cast<unsigned*>(sync_ticket), ST(stream));
}
int seg_bn_finalize(const double* stats, double count, int C, const float* gamma, const float* beta, float eps,
                    float momentum, int clamp_eps, float* running_mean, float* running_var, float* scale_shift,
                    float* save, void* stream) {
  bn_finalize_kernel<<<ceil_div(C, 128), 128, 0, ST(stream)>>>(stats, count, C, gamma, beta, eps, momentum, clamp_eps,
                                                                running_mean, running_var, scale_shift, save);
  return check_launch("bn_finalize");
}
int seg_bn_eval_scale_shift(int C, const float* gamma, const float* beta, const float* rm, const float* rv, float eps,
                            float* scale_shift, float* save_mean_istd, void* stream) {
  bn_eval_kernel<<<ceil_div(C, 128), 128, 0, ST(stream)>>>(C, gamma, beta, rm, rv, eps, scale_shift, save_mean_istd);
  return check_launch("bn_eval");
}
int seg_bn_apply(const void* x, int ldx, const float* ss, const void* res, int ldr, void* out, int ldo, int64_t M, int C,
                 int relu, float drop_p, uint64_t seed, const uint64_t* step_ctr, int drop_hw, void* stream) {
  SEG_REQUIRE(C % 8 == 0 && ldx % 8 == 0 && ldo % 8 == 0 && (!res || ldr % 8 == 0), "bn_apply: alignment");
  BnTrain tr;
  memset(&tr, 0, sizeof(tr));
  launch_pdl(bn_apply_kernel<false>, rowmap_grid(M, C), dim3(256), 0, ST(stream), CBF(x), ldx, ss, CBF(res), ldr, BF(out), ldo, M, C, relu,
             drop_p, seed, step_ctr, drop_hw, tr, (uint8_t*)nullptr);
  return check_launch("bn_apply");
}
int seg_bn_apply_train(const void* x, int ldx, const double* stats, double count, const float* gamma, const float* beta,
                       float eps, float momentum, int clamp_eps, float* running_mean, float* running_var, float* save,
                       const void* res, int ldr, void* out, int ldo, uint8_t* mask, int64_t M, int C, int relu, float drop_p,
                       uint64_t seed, const uint64_t* step_ctr, int drop_hw, int c0, int growth, void* stream) {
  SEG_REQUIRE(C % 8 == 0 && ldx % 8 == 0 && ldo % 8 == 0 && (!res || ldr % 8 == 0), "bn_apply_train: alignment");
  SEG_REQUIRE(stats && gamma && beta && save && count > 0, "bn_apply_train: stats, gamma, beta, save required");
  SEG_REQUIRE(!mask || relu, "bn_apply_train: the ReLU bit mask needs relu");
  SEG_REQUIRE(growth >= 0 && (growth == 0 || (c0 > 0 && c0 <= C)),
              "bn_apply_train: statistics table needs 0 < c0 <= C and growth > 0 (c0=%d growth=%d C=%d)", c0, growth, C);
  BnTrain tr = {stats, count, gamma, beta, eps, momentum, clamp_eps, running_mean, running_var, save, c0, growth};
  launch_pdl(growth > 0 ? bn_apply_kernel<true> : bn_apply_kernel<false>, rowmap_grid(M, C), dim3(256), 0, ST(stream), CBF(x), ldx,
             (const float*)nullptr, CBF(res), ldr, BF(out),
             ldo, M, C, relu, drop_p, seed, step_ctr, drop_hw, tr, mask);
  return check_launch("bn_apply_train");
}
// reductions end with a block fold + 2C atomics per block: fewer, fatter blocks (>= 32 rows per thread)
static dim3 reduce2_grid(int64_t M, int C) { return rowmap_grid(M, C, 32); }

int seg_bn_bwd_reduce_slots(void) { return RED_SLOTS; }
int seg_bn_bwd_reduce(const void* dout, int lddo, const void* out, int ldo, const uint8_t* mask, const void* x, int ldx,
                      const float* save, int64_t M, int C, int relu, float drop_p, float* sums, double* acc, void* ticket,
                      float* dgamma, float* dbeta, int accumulate, const float* gamma, const float* beta,
                      const seg_sync_desc* sync, void* stream) {
  const MaskSrc ms = mask_src(relu, out, mask);
  SEG_REQUIRE(C % 8 == 0 && lddo % 8 == 0 && ldx % 8 == 0 && (ms != MaskSrc::ACT || !relu || ldo % 8 == 0), "bn_bwd_reduce: alignment");
  SEG_REQUIRE(ms != MaskSrc::RECOMPUTE || (gamma && beta && drop_p == 0.f), "bn_bwd_reduce: out == NULL (mask recomputed from x) needs gamma, beta and no dropout");
  SEG_REQUIRE(relu || drop_p == 0.f, "bn_bwd_reduce: dropout (drop_p > 0) needs relu: the keep mask is read from out > 0");
  SEG_REQUIRE(acc && ticket, "bn_bwd_reduce: zeroed fp64 accumulators [seg_bn_bwd_reduce_slots()][2C] and ticket word required");
  if (sync && sync_check_desc(sync, 2ll * C, "bn_bwd_reduce")) return 1;
  const dim3 grid = reduce2_grid(M, C);
  launch_pdl(by_mask_src(ms, bn_bwd_reduce_kernel<MaskSrc::ACT>, bn_bwd_reduce_kernel<MaskSrc::RECOMPUTE>,
                         bn_bwd_reduce_kernel<MaskSrc::BITS>),
             grid, dim3(256), 0, ST(stream), CBF(dout), lddo, CBF(out), ldo, mask, CBF(x), ldx, save, M, C, relu, drop_p, acc,
             reinterpret_cast<unsigned*>(ticket), sums, dgamma, dbeta, accumulate, gamma, beta, to_sync(sync));
  return check_launch("bn_bwd_reduce");
}
int seg_bn_bwd_apply(const void* dout, int lddo, const void* out, int ldo, const uint8_t* mask, const void* x, int ldx,
                     const float* save, const float* gamma, const float* sums, double count, int64_t M, int C, int relu,
                     float drop_p, void* dx, int lddx, void* dres, int lddres, float beta_res, const float* beta, float beta_dx,
                     void* stream) {
  const MaskSrc ms = mask_src(relu, out, mask);
  SEG_REQUIRE(C % 8 == 0 && lddo % 8 == 0 && ldx % 8 == 0 && lddx % 8 == 0, "bn_bwd_apply: alignment");
  SEG_REQUIRE(ms != MaskSrc::RECOMPUTE || (beta && drop_p == 0.f), "bn_bwd_apply: out == NULL (mask recomputed from x) needs beta and no dropout");
  SEG_REQUIRE(relu || drop_p == 0.f, "bn_bwd_apply: dropout (drop_p > 0) needs relu: the keep mask is read from out > 0");
  SEG_REQUIRE(beta_dx == 0.f || beta_dx == 1.f, "bn_bwd_apply: beta_dx must be 0 or 1 (got %g)", (double)beta_dx);
  launch_pdl(beta_dx != 0.f ? by_mask_src(ms, bn_bwd_apply_kernel<MaskSrc::ACT, true>, bn_bwd_apply_kernel<MaskSrc::RECOMPUTE, true>,
                                          bn_bwd_apply_kernel<MaskSrc::BITS, true>)
                            : by_mask_src(ms, bn_bwd_apply_kernel<MaskSrc::ACT>, bn_bwd_apply_kernel<MaskSrc::RECOMPUTE>,
                                          bn_bwd_apply_kernel<MaskSrc::BITS>),
             rowmap_grid(M, C), dim3(256), 0, ST(stream), CBF(dout), lddo, CBF(out), ldo, mask, CBF(x), ldx, save,
             gamma, sums, (float)(1.0 / count), M, C, relu, drop_p, BF(dx), lddx, BF(dres), lddres, beta_res, beta);
  return check_launch("bn_bwd_apply");
}
}  // extern "C"
// co-resident grid of the cooperative kernel: blocks per SM from the occupancy of the instantiation actually launched
template <MaskSrc MS, bool ACC = false>
static int fused_blocks_per_sm() {
  static int v = 0;
  if (v == 0) {
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, bn_bwd_fused_kernel<MS, ACC>, 256, 0) != cudaSuccess || n < 1) n = 1;
    v = n;
  }
  return v;
}
// The grid fixes which rows each block sums, and so the rounding of the fp32 partial sums: the BITS variant runs on the
// ACT variant's grid (when it fits), so that its sums and dx are bit-identical to those read from the activation
static int fused_bps(MaskSrc ms) {
  if (ms == MaskSrc::RECOMPUTE) return fused_blocks_per_sm<MaskSrc::RECOMPUTE>();
  const int act = fused_blocks_per_sm<MaskSrc::ACT>();
  if (ms == MaskSrc::ACT) return act;
  const int bits = fused_blocks_per_sm<MaskSrc::BITS>();
  return bits < act ? bits : act;
}
// the accumulating variant: never more blocks than it can keep co-resident (the grid barrier needs every block resident)
static int fused_bps(MaskSrc ms, bool acc) {
  const int b = fused_bps(ms);
  if (!acc) return b;
  const int a = ms == MaskSrc::RECOMPUTE ? fused_blocks_per_sm<MaskSrc::RECOMPUTE, true>()
                : ms == MaskSrc::BITS   ? fused_blocks_per_sm<MaskSrc::BITS, true>()
                                        : fused_blocks_per_sm<MaskSrc::ACT, true>();
  return a < b ? a : b;
}
extern "C" {
static dim3 fused_grid(int64_t M, int C, int blocks_per_sm) {
  dim3 g = rowmap_grid(M, C, 16);
  const int64_t cap = (int64_t)num_sms() * blocks_per_sm / g.y;
  if ((int64_t)g.x > cap) g.x = (unsigned)(cap < 1 ? 1 : cap);
  return g;
}
int seg_bn_bwd_fused_workspace(int64_t M, int C, int64_t* rows_floats, int64_t* tickets) {
  SEG_REQUIRE(C % 8 == 0 && rows_floats && tickets, "seg_bn_bwd_fused_workspace: bad arguments");
  const int b0 = fused_bps(MaskSrc::ACT), b1 = fused_bps(MaskSrc::RECOMPUTE), b2 = fused_bps(MaskSrc::BITS);
  const int bps = b0 > b1 ? (b0 > b2 ? b0 : b2) : (b1 > b2 ? b1 : b2);
  const dim3 g = fused_grid(M, C, bps);
  const int G = C / 8, GB = G < 256 ? G : 256;
  *rows_floats = (int64_t)g.y * g.x * 2 * GB * 8;
  *tickets = 1;
  return 0;
}
int seg_bn_bwd_fused(const void* dout, int lddo, const void* out, int ldo, const uint8_t* mask, const void* x, int ldx,
                     const float* save, const float* gamma, const float* beta, double count_total, int64_t M, int C, int relu,
                     float drop_p, float* sums, float* rows, void* tickets, float* dgamma, float* dbeta, int accumulate, void* dx,
                     int lddx, void* dres, int lddres, float beta_res, int zero_sums, const seg_sync_desc* sync, float beta_dx,
                     void* stream) {
  const MaskSrc ms = mask_src(relu, out, mask);
  SEG_REQUIRE(beta_dx == 0.f || beta_dx == 1.f, "bn_bwd_fused: beta_dx must be 0 or 1 (got %g)", (double)beta_dx);
  const bool acc = beta_dx != 0.f;
  SEG_REQUIRE(C % 8 == 0 && lddo % 8 == 0 && ldx % 8 == 0 && lddx % 8 == 0 && (!out || ldo % 8 == 0) && (!dres || lddres % 8 == 0),
              "bn_bwd_fused: alignment");
  SEG_REQUIRE(ms != MaskSrc::RECOMPUTE || (beta && drop_p == 0.f), "bn_bwd_fused: out == NULL (mask recomputed from x) needs beta and no dropout");
  SEG_REQUIRE(relu || drop_p == 0.f, "bn_bwd_fused: dropout (drop_p > 0) needs relu: the keep mask is read from out > 0");
  SEG_REQUIRE(sums && rows && tickets && gamma && save && dx && count_total > 0, "bn_bwd_fused: missing buffer");
  BnBwdFused p;
  memset(&p, 0, sizeof(p));
  p.dout = CBF(dout); p.out = CBF(out); p.x = CBF(x); p.mask = mask;
  p.lddo = lddo; p.ldo = ldo; p.ldx = ldx;
  p.save = save; p.gamma = gamma; p.beta = beta;
  p.M = M; p.C = C; p.relu = relu; p.drop_p = drop_p; p.inv_count = (float)(1.0 / count_total);
  p.rows = rows; p.totals = sums; p.ctr = reinterpret_cast<unsigned*>(tickets);
  p.dgamma = dgamma; p.dbeta = dbeta; p.accumulate = accumulate; p.zero_sums = zero_sums;
  p.dx = BF(dx); p.dres = BF(dres); p.lddx = lddx; p.lddres = lddres; p.beta_res = beta_res;
  if (sync) {
    if (sync_check_desc(sync, 2ll * C, "bn_bwd_fused")) return 1;
    p.sync = *sync;
  }
  // multi-GPU: leave one block slot per SM free — a concurrently running NCCL kernel (bucketed gradient all-reduce on the side
  // stream) must not keep part of this grid from becoming resident, or every block would sit at the barrier until it finishes
  int bps = fused_bps(ms, acc);
  if (sync && bps > 1) bps -= 1;
  const dim3 grid = fused_grid(M, C, bps);
  (acc ? by_mask_src(ms, bn_bwd_fused_kernel<MaskSrc::ACT, true>, bn_bwd_fused_kernel<MaskSrc::RECOMPUTE, true>,
                     bn_bwd_fused_kernel<MaskSrc::BITS, true>)
       : by_mask_src(ms, bn_bwd_fused_kernel<MaskSrc::ACT>, bn_bwd_fused_kernel<MaskSrc::RECOMPUTE>,
                     bn_bwd_fused_kernel<MaskSrc::BITS>))<<<grid, 256, 0, ST(stream)>>>(p);
  return check_launch("bn_bwd_fused");
}
int seg_bn_param_grad(const float* sums, int C, float* dgamma, float* dbeta, int accumulate, void* stream) {
  bn_param_grad_kernel<<<ceil_div(C, 128), 128, 0, ST(stream)>>>(sums, C, dgamma, dbeta, accumulate);
  return check_launch("bn_param_grad");
}

int seg_maxpool3x3s2_fwd(const void* x, void* y, uint8_t* idx, int N, int H, int W, int C, int P, int Q, void* stream) {
  SEG_REQUIRE(C % 8 == 0, "maxpool: C %% 8");
  maxpool_fwd_kernel<<<grid_for((int64_t)N * P * Q * (C / 8), 256), 256, 0, ST(stream)>>>(CBF(x), BF(y), idx, N, H, W, C, P, Q);
  return check_launch("maxpool_fwd");
}
int seg_maxpool3x3s2_bwd(const void* dy, const uint8_t* idx, void* dx, int N, int H, int W, int C, int P, int Q,
                         void* stream) {
  SEG_REQUIRE(C % 8 == 0, "maxpool: C %% 8");
  maxpool_bwd_kernel<<<grid_for((int64_t)N * H * W * (C / 8), 256), 256, 0, ST(stream)>>>(CBF(dy), idx, BF(dx), N, H, W, C, P, Q);
  return check_launch("maxpool_bwd");
}

static int check_pool2x2(const char* what, const void* a, const void* b, const void* code, int N, int H, int W, int C,
                         int min_hw = 2) {
  SEG_REQUIRE(N > 0 && H >= min_hw && W >= min_hw, "%s: needs N >= 1 and H, W >= %d (got %d x %d x %d)", what, min_hw, N, H, W);
  SEG_REQUIRE(C > 0 && C % 8 == 0, "%s: C = %d is not a positive multiple of 8", what, C);
  SEG_REQUIRE(((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(code) & 7) == 0,
              "%s: activations must be 16-byte and codes 8-byte aligned", what);
  return 0;
}
int seg_maxpool2x2_fwd(const void* x, void* y, uint8_t* code, int N, int H, int W, int C, void* stream) {
  if (check_pool2x2("maxpool2x2_fwd", x, y, code, N, H, W, C)) return 1;
  const int P = H / 2, Q = W / 2;
  maxpool2x2_fwd_kernel<false><<<grid_for((int64_t)N * P * Q * (C / 8), 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(y), reinterpret_cast<uint2*>(code), N, H, W, C / 8, P, Q);
  return check_launch("maxpool2x2_fwd");
}
static int launch_unpool2x2_scatter(const char* what, const void* src, const uint8_t* code, void* dst, int N, int H, int W,
                                    int C, void* stream) {
  if (check_pool2x2(what, src, dst, code, N, H, W, C)) return 1;
  unpool2x2_scatter_kernel<<<grid_for((int64_t)N * ((H + 1) / 2) * ((W + 1) / 2) * (C / 8), 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const uint4*>(src), reinterpret_cast<const uint2*>(code), reinterpret_cast<uint4*>(dst), N, H, W, C / 8,
      H / 2, W / 2);
  return check_launch(what);
}
int seg_maxpool2x2_bwd(const void* dy, const uint8_t* code, void* dx, int N, int H, int W, int C, void* stream) {
  return launch_unpool2x2_scatter("maxpool2x2_bwd", dy, code, dx, N, H, W, C, stream);
}
int seg_maxunpool2x2_fwd(const void* x, const uint8_t* code, void* y, int N, int H, int W, int C, void* stream) {
  return launch_unpool2x2_scatter("maxunpool2x2_fwd", x, code, y, N, H, W, C, stream);
}
int seg_maxunpool2x2_bwd(const void* dy, const uint8_t* code, void* dx, int N, int H, int W, int C, void* stream) {
  if (check_pool2x2("maxunpool2x2_bwd", dy, dx, code, N, H, W, C)) return 1;
  const int P = H / 2, Q = W / 2;
  unpool2x2_gather_kernel<<<grid_for((int64_t)N * P * Q * (C / 8), 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const uint4*>(dy), reinterpret_cast<const uint2*>(code), reinterpret_cast<uint4*>(dx), N, H, W, C / 8, P, Q);
  return check_launch("maxunpool2x2_bwd");
}
int seg_relu_maxpool2x2_ceil_fwd(const void* x, void* y, uint8_t* code, int N, int H, int W, int C, void* stream) {
  if (check_pool2x2("relu_maxpool2x2_ceil_fwd", x, y, code, N, H, W, C, 1)) return 1;
  const int P = (H + 1) / 2, Q = (W + 1) / 2;
  maxpool2x2_fwd_kernel<true><<<grid_for((int64_t)N * P * Q * (C / 8), 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(y), reinterpret_cast<uint2*>(code), N, H, W, C / 8, P, Q);
  return check_launch("relu_maxpool2x2_ceil_fwd");
}
int seg_relu_maxpool2x2_ceil_bwd(const void* dy, const uint8_t* code, void* dx, int N, int H, int W, int C, void* stream) {
  if (check_pool2x2("relu_maxpool2x2_ceil_bwd", dy, dx, code, N, H, W, C, 1)) return 1;
  // the floor-mode scatter with every window read: codes 4-7 (max <= 0) match no position, so the whole window gets 0
  unpool2x2_scatter_kernel<<<grid_for((int64_t)N * ((H + 1) / 2) * ((W + 1) / 2) * (C / 8), 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const uint4*>(dy), reinterpret_cast<const uint2*>(code), reinterpret_cast<uint4*>(dx), N, H, W, C / 8,
      (H + 1) / 2, (W + 1) / 2);
  return check_launch("relu_maxpool2x2_ceil_bwd");
}
int seg_adaptive_avgpool_fwd(const void* x, int ldx, void* y, int N, int H, int W, int C, int bins, void* stream) {
  SEG_REQUIRE(C % 8 == 0 && ldx % 8 == 0, "avgpool: alignment");
  dim3 grid((unsigned)(N * bins * bins), (unsigned)ceil_div(C / 8, 32), 1);
  adaptive_avgpool_fwd_kernel<<<grid, 256, 0, ST(stream)>>>(CBF(x), ldx, BF(y), N, H, W, C, bins);
  return check_launch("adaptive_avgpool_fwd");
}
int seg_adaptive_avgpool_bwd(const void* dy, void* dx, int lddx, int N, int H, int W, int C, int bins, float beta,
                             void* stream) {
  SEG_REQUIRE(C % 8 == 0 && lddx % 8 == 0, "avgpool: alignment");
  adaptive_avgpool_bwd_kernel<<<grid_for((int64_t)N * H * W * (C / 8), 256), 256, 0, ST(stream)>>>(CBF(dy), BF(dx), lddx, N, H,
                                                                                                   W, C, bins, beta);
  return check_launch("adaptive_avgpool_bwd");
}

int seg_avgpool2x2_fwd(const void* x, int ldx, void* y, int ldy, int N, int H, int W, int C, void* stream) {
  SEG_REQUIRE(C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && ldx >= C && ldy >= C, "avgpool2x2: alignment");
  SEG_REQUIRE(N > 0 && H >= 2 && W >= 2, "avgpool2x2: needs H, W >= 2 (got %dx%d)", H, W);
  avgpool2x2_fwd_kernel<<<grid_for((int64_t)N * (H / 2) * (W / 2) * (C / 8), 256), 256, 0, ST(stream)>>>(CBF(x), ldx, BF(y), ldy, N,
                                                                                                         H, W, C);
  return check_launch("avgpool2x2_fwd");
}
int seg_avgpool2x2_bwd(const void* dy, int lddy, void* dx, int lddx, int N, int H, int W, int C, float beta, void* stream) {
  SEG_REQUIRE(C % 8 == 0 && lddy % 8 == 0 && lddx % 8 == 0 && lddy >= C && lddx >= C, "avgpool2x2_bwd: alignment");
  SEG_REQUIRE(N > 0 && H >= 2 && W >= 2, "avgpool2x2_bwd: needs H, W >= 2 (got %dx%d)", H, W);
  avgpool2x2_bwd_kernel<<<grid_for((int64_t)N * H * W * (C / 8), 256), 256, 0, ST(stream)>>>(CBF(dy), lddy, BF(dx), lddx, N, H, W,
                                                                                             C, beta);
  return check_launch("avgpool2x2_bwd");
}

int seg_bilinear_fwd(const void* x, int ldx, void* y, int ldy, int N, int Hi, int Wi, int Ho, int Wo, int C,
                     int align_corners, void* stream) {
  SEG_REQUIRE(C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0, "bilinear: alignment");
  bilinear_fwd_kernel<<<grid_for((int64_t)N * Ho * Wo * (C / 8), 256), 256, 0, ST(stream)>>>(
      CBF(x), ldx, BF(y), ldy, N, Hi, Wi, Ho, Wo, C, align_corners, resize_scale(Hi, Ho, align_corners),
      resize_scale(Wi, Wo, align_corners));
  return check_launch("bilinear_fwd");
}
int seg_bilinear_bwd(const void* dy, int lddy, void* dx, int lddx, int N, int Hi, int Wi, int Ho, int Wo, int C,
                     int align_corners, float beta, void* stream) {
  SEG_REQUIRE(C % 8 == 0 && lddx % 8 == 0 && lddy % 8 == 0, "bilinear: alignment");
  bilinear_bwd_kernel<<<grid_for((int64_t)N * Hi * Wi * (C / 8), 256), 256, 0, ST(stream)>>>(
      CBF(dy), lddy, BF(dx), lddx, N, Hi, Wi, Ho, Wo, C, align_corners, resize_scale(Hi, Ho, align_corners),
      resize_scale(Wi, Wo, align_corners), beta);
  return check_launch("bilinear_bwd");
}
int seg_bilinear_logits_fwd(const float* x, float* y, int N, int Hi, int Wi, int Ho, int Wo, int C, int align_corners,
                            void* stream) {
  bilinear_logits_fwd_kernel<<<grid_for((int64_t)N * Ho * Wo, 256), 256, 0, ST(stream)>>>(
      x, y, N, Hi, Wi, Ho, Wo, C, align_corners, resize_scale(Hi, Ho, align_corners), resize_scale(Wi, Wo, align_corners));
  return check_launch("bilinear_logits_fwd");
}
int seg_bilinear_logits_bwd(const float* dy, void* dx, int lddx, int N, int Hi, int Wi, int Ho, int Wo, int C,
                            int align_corners, void* stream) {
  bilinear_logits_bwd_kernel<<<grid_for((int64_t)N * Hi * Wi, 128, 16), 128, 0, ST(stream)>>>(
      dy, BF(dx), lddx, N, Hi, Wi, Ho, Wo, C, align_corners, resize_scale(Hi, Ho, align_corners),
      resize_scale(Wi, Wo, align_corners));
  return check_launch("bilinear_logits_bwd");
}

int seg_pixel_shuffle_fwd(const void* x, int ldx, void* y, int ldy, int N, int H, int W, int C, int r, int Ho, int Wo,
                          void* stream) {
  SEG_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && r >= 1, "pixel_shuffle: bad sizes");
  SEG_REQUIRE(Ho >= 1 && Ho <= r * H && Wo >= 1 && Wo <= r * W, "pixel_shuffle: crop %dx%d outside %dx%d", Ho, Wo, r * H, r * W);
  SEG_REQUIRE(ldx >= C * r * r && ldy >= C, "pixel_shuffle: pitch smaller than channel count");
  pixel_shuffle_fwd_kernel<<<grid_for((int64_t)N * Ho * Wo * C, 256), 256, 0, ST(stream)>>>(CBF(x), ldx, BF(y), ldy, N, H, W, C,
                                                                                              r, Ho, Wo);
  return check_launch("pixel_shuffle_fwd");
}
int seg_pixel_shuffle_bwd(const void* dy, int lddy, void* dx, int lddx, int N, int H, int W, int C, int r, int Ho, int Wo,
                          float beta, void* stream) {
  SEG_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && r >= 1, "pixel_shuffle: bad sizes");
  SEG_REQUIRE(Ho >= 1 && Ho <= r * H && Wo >= 1 && Wo <= r * W, "pixel_shuffle: crop %dx%d outside %dx%d", Ho, Wo, r * H, r * W);
  SEG_REQUIRE(lddx >= C * r * r && lddy >= C, "pixel_shuffle: pitch smaller than channel count");
  pixel_shuffle_bwd_kernel<<<grid_for((int64_t)N * H * W * C * r * r, 256), 256, 0, ST(stream)>>>(CBF(dy), lddy, BF(dx), lddx, N,
                                                                                                   H, W, C, r, Ho, Wo, beta);
  return check_launch("pixel_shuffle_bwd");
}
int seg_pixel_shuffle_logits_fwd(const void* x, int ldx, float* y_nchw, int N, int h, int w, int C, int r, void* stream) {
  SEG_REQUIRE(N > 0 && h > 0 && w > 0 && C > 0 && r >= 1 && ldx >= C * r * r, "pixel_shuffle_logits: bad sizes");
  pixel_shuffle_logits_fwd_kernel<<<grid_for((int64_t)N * C * h * w * r * r, 256), 256, 0, ST(stream)>>>(CBF(x), ldx, y_nchw, N, h,
                                                                                                          w, C, r);
  return check_launch("pixel_shuffle_logits_fwd");
}
int seg_pixel_shuffle_logits_bwd(const float* dy_nchw, void* dx, int lddx, int N, int h, int w, int C, int r, void* stream) {
  SEG_REQUIRE(N > 0 && h > 0 && w > 0 && C > 0 && r >= 1 && lddx >= C * r * r, "pixel_shuffle_logits: bad sizes");
  pixel_shuffle_logits_bwd_kernel<<<grid_for((int64_t)N * h * w * lddx, 256), 256, 0, ST(stream)>>>(dy_nchw, BF(dx), lddx, N, h,
                                                                                                     w, C, r);
  return check_launch("pixel_shuffle_logits_bwd");
}

int seg_nhwc_to_nchw_f32(const void* x, int ldx, int x_dtype, float* y, int N, int H, int W, int C, void* stream) {
  nhwc_to_nchw_kernel<<<grid_for((int64_t)N * C * H * W, 256), 256, 0, ST(stream)>>>(x, ldx, x_dtype, y, N, H, W, C);
  return check_launch("nhwc_to_nchw");
}
int seg_axpby_bf16(const void* x, int ldx, void* y, int ldy, int64_t M, int C, float beta, void* stream) {
  SEG_REQUIRE(C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0, "axpby: alignment");
  axpby_kernel<<<grid_for(M * (C / 8), 256), 256, 0, ST(stream)>>>(CBF(x), ldx, BF(y), ldy, M, C, beta);
  return check_launch("axpby");
}
int seg_relu_fwd(const void* x, int ldx, void* y, int ldy, int64_t M, int C, void* stream) {
  SEG_REQUIRE(C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0, "relu: alignment");
  relu_fwd_kernel<<<grid_for(M * (C / 8), 256), 256, 0, ST(stream)>>>(CBF(x), ldx, BF(y), ldy, M, C);
  return check_launch("relu_fwd");
}
int seg_relu_dropout_fwd(const void* x, int ldx, void* y, int ldy, int64_t M, int C, float drop_p, uint64_t seed,
                         const uint64_t* step_ctr, void* stream) {
  SEG_REQUIRE(C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0, "relu_dropout_fwd: C and pitches must be multiples of 8");
  SEG_REQUIRE(drop_p >= 0.f && drop_p < 1.f, "relu_dropout_fwd: drop_p = %g is not in [0, 1)", (double)drop_p);
  relu_dropout_fwd_kernel<<<grid_for(M * (C / 8), 256), 256, 0, ST(stream)>>>(CBF(x), ldx, BF(y), ldy, M, C, drop_p, seed, step_ctr);
  return check_launch("relu_dropout_fwd");
}
int seg_relu_dropout_bwd(const void* dy, int lddy, const void* y, int ldy, void* dx, int lddx, int64_t M, int C, float drop_p,
                         float beta, void* stream) {
  SEG_REQUIRE(C % 8 == 0 && lddy % 8 == 0 && ldy % 8 == 0 && lddx % 8 == 0, "relu_dropout_bwd: C and pitches must be multiples of 8");
  SEG_REQUIRE(drop_p >= 0.f && drop_p < 1.f, "relu_dropout_bwd: drop_p = %g is not in [0, 1)", (double)drop_p);
  relu_dropout_bwd_kernel<<<grid_for(M * (C / 8), 256), 256, 0, ST(stream)>>>(CBF(dy), lddy, CBF(y), ldy, BF(dx), lddx, M, C, drop_p,
                                                                           beta);
  return check_launch("relu_dropout_bwd");
}
int seg_relu_bwd(const void* dy, int lddy, const void* y, int ldy, void* dx, int lddx, int64_t M, int C, float beta,
                 void* stream) {
  SEG_REQUIRE(C % 8 == 0 && lddy % 8 == 0 && ldy % 8 == 0 && lddx % 8 == 0, "relu: alignment");
  relu_bwd_kernel<<<grid_for(M * (C / 8), 256), 256, 0, ST(stream)>>>(CBF(dy), lddy, CBF(y), ldy, BF(dx), lddx, M, C, beta);
  return check_launch("relu_bwd");
}
int seg_counter_add(uint64_t* ctr, uint64_t inc, void* stream) {
  counter_add_kernel<<<1, 32, 0, ST(stream)>>>(ctr, inc);
  return check_launch("counter_add");
}
int seg_sgd_step(float* const* params, float* const* grads, float* const* bufs, const int64_t* sizes, const float* lrs,
                 int n, float momentum, float weight_decay, int first_step, float grad_scale, void* stream) {
  if (n <= 0) return 0;
  SEG_REQUIRE(n <= 65535, "sgd_step: at most 65535 tensors per launch (one block row per tensor)");
  SgdChunkArgs a{params, grads, bufs, sizes, lrs};
  dim3 grid(64, (unsigned)n, 1);
  sgd_kernel<<<grid, 256, 0, ST(stream)>>>(a, momentum, weight_decay, first_step, grad_scale, nullptr);
  return check_launch("sgd_step");
}
int seg_sgd_step_dev(float* const* params, float* const* grads, float* const* bufs, const int64_t* sizes, const float* lrs,
                     int n, const float* hyper, int first_step, float grad_scale, void* stream) {
  if (n <= 0) return 0;
  SEG_REQUIRE(hyper != nullptr, "sgd_step_dev: hyper (device [momentum, weight_decay]) is required");
  SEG_REQUIRE(n <= 65535, "sgd_step_dev: at most 65535 tensors per launch (one block row per tensor)");
  SgdChunkArgs a{params, grads, bufs, sizes, lrs};
  dim3 grid(64, (unsigned)n, 1);
  sgd_kernel<<<grid, 256, 0, ST(stream)>>>(a, 0.f, 0.f, first_step, grad_scale, hyper);
  return check_launch("sgd_step_dev");
}

}  // extern "C"
