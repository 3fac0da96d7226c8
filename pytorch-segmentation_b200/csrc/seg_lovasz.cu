// seg_lovasz.cu — Lovász-softmax loss (LovaszSoftmax.forward, utils/losses.py:79-89 -> lovasz_softmax /
// lovasz_softmax_flat / lovasz_grad, utils/lovasz_losses.py:153-199,19-31; classes='present', per_image=False).
//
// The reference loops over classes on the host: per class an ATen sort of P floats, two cumsums, a dot product and a
// host sync (`fg.sum() == 0`).  Here every present class is handled at once, on the device:
//   1. emit   : per valid pixel, softmax, then one 64-bit key per PRESENT class
//                 [class rank : 8][~bits(|fg - p_c|) : 32][fg : 1][pixel index : 23]
//               written to segment `rank` of a [n_present][P] array at slot = number of valid pixels before the pixel
//               (per-chunk valid counts, an exclusive scan, a block-local rank), so every segment is in pixel order.
//   2. sort   : one global LSD radix sort over bits 24..63 (5 passes x 8 bits: histogram, per-digit scan, stable
//               scatter) -> each class segment sorted by error, descending; segments stay [rank*P, (rank+1)*P).
//   3. jaccard: per class a tiled inclusive scan of the fg flags gives intersection / union at every rank, hence the
//               Lovász gradient  d_i = J_i - J_{i-1};  loss_c = sum_i e_i d_i (fp64 per-tile partials), and
//               dLoss/dp[pixel, c] = d_i * sign scattered into an NCHW scratch tensor.
//   4. finish : loss = mean_c loss_c, folded from the tile partials in a fixed order; the softmax Jacobian turns dLoss/dp
//               into dLoss/dlogits in place.
// Pure HBM-bound integer/byte work (no GEMM).  Tie order: exactly tied errors take ranks in flat pixel order (the order a
// stable sort of the reference's flattened error vector gives).  The loss value does not depend on it (the sum
// telescopes) but the per-pixel gradient d_i does; a stable sort of pixel-ordered segments makes both reproducible.
#include "seg_common.cuh"

namespace seg {

constexpr int LV_THREADS = 256;
constexpr int LV_ITEMS = 32;                      // keys per thread per radix tile
constexpr int LV_TILE = LV_THREADS * LV_ITEMS;    // 8192 keys per block
constexpr int LV_MAXC = 256;

// ---------------------------------------------------------------- 0. class presence
__global__ void lv_count_kernel(const int64_t* __restrict__ target, int64_t npix, int C, int64_t ignore, int* __restrict__ counts) {
  __shared__ int sh[LV_MAXC + 1];
  for (int i = threadIdx.x; i <= LV_MAXC; i += blockDim.x) sh[i] = 0;
  __syncthreads();
  int valid = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < npix; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = target[i];
    if (t == ignore) continue;
    ++valid;
    if (t >= 0 && t < C) atomicAdd(&sh[(int)t], 1);
  }
  if (valid) atomicAdd(&sh[LV_MAXC], valid);       // number of valid pixels
  __syncthreads();
  for (int i = threadIdx.x; i < C; i += blockDim.x)
    if (sh[i]) atomicAdd(counts + i, sh[i]);
  if (threadIdx.x == 0 && sh[LV_MAXC]) atomicAdd(counts + C, sh[LV_MAXC]);
}

// rank[c] = index of class c among the present classes (or -1)
__global__ void lv_rank_kernel(const int* __restrict__ counts, int C, int* __restrict__ rank) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    int r = 0;
    for (int c = 0; c < C; ++c) rank[c] = counts[c] > 0 ? r++ : -1;
  }
}

// ---------------------------------------------------------------- 1. softmax + key emission
// Pixels are processed in chunks of LV_THREADS consecutive pixels, one chunk per block iteration (chunk j = pixels
// [j*256, (j+1)*256)).  chunk_valid[j] = valid pixels of chunk j; lv_emit reads its exclusive scan.
__global__ void __launch_bounds__(LV_THREADS)
    lv_chunk_count_kernel(const int64_t* __restrict__ target, int64_t total, int64_t ignore, unsigned int* __restrict__ chunk_valid) {
  const int64_t nchunks = ceil_div64(total, LV_THREADS);
  for (int64_t ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
    const int64_t i = ch * LV_THREADS + threadIdx.x;
    const int n = __syncthreads_count(i < total && target[i] != ignore);
    if (threadIdx.x == 0) chunk_valid[ch] = (unsigned int)n;
  }
}

__global__ void __launch_bounds__(LV_THREADS)
    lv_emit_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target, int N, int C, int H, int W,
                   int64_t ignore, const int* __restrict__ rank, long long P, unsigned long long* __restrict__ keys,
                   const unsigned int* __restrict__ chunk_off) {
  const int64_t HW = (int64_t)H * W, total = (int64_t)N * HW;
  const int64_t nchunks = ceil_div64(total, LV_THREADS);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __shared__ unsigned int wvalid[LV_THREADS / 32];
  for (int64_t ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
    const int64_t i = ch * LV_THREADS + threadIdx.x;
    const int64_t t = i < total ? target[i] : ignore;
    const bool ok = t != ignore;
    // slot = valid pixels before chunk ch + valid pixels of this chunk before pixel i
    const unsigned int ballot = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) wvalid[warp] = __popc(ballot);
    __syncthreads();
    unsigned int slot = chunk_off[ch] + __popc(ballot & ((1u << lane) - 1u));
    for (int w = 0; w < warp; ++w) slot += wvalid[w];
    __syncthreads();  // wvalid is rewritten by the next chunk
    if (!ok) continue;
    const int n = (int)(i / HW);
    const float* l = logits + (int64_t)n * C * HW + (i - (int64_t)n * HW);
    float mx = -INFINITY;
    for (int c = 0; c < C; ++c) mx = fmaxf(mx, l[(int64_t)c * HW]);
    float se = 0.f;
    for (int c = 0; c < C; ++c) se += expf(l[(int64_t)c * HW] - mx);
    const float inv = 1.f / se;
    for (int c = 0; c < C; ++c) {
      const int r = rank[c];
      if (r < 0) continue;
      const float p = expf(l[(int64_t)c * HW] - mx) * inv;
      const unsigned int fg = (c == t) ? 1u : 0u;
      const float err = fabsf((float)fg - p);
      const unsigned long long key = ((unsigned long long)r << 56) | ((unsigned long long)(~__float_as_uint(err)) << 24) |
                                     ((unsigned long long)fg << 23) | (unsigned long long)i;
      keys[(long long)r * P + slot] = key;
    }
  }
}

// ---------------------------------------------------------------- 2. LSD radix sort (8-bit digits)
__global__ void __launch_bounds__(LV_THREADS)
    lv_radix_hist_kernel(const unsigned long long* __restrict__ keys, long long n, int shift, unsigned int* __restrict__ table,
                         int nblocks) {
  __shared__ unsigned int h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const long long base = (long long)blockIdx.x * LV_TILE;
  for (int k = 0; k < LV_ITEMS; ++k) {
    const long long i = base + (long long)k * LV_THREADS + threadIdx.x;
    if (i < n) atomicAdd(&h[(unsigned int)(keys[i] >> shift) & 255u], 1u);
  }
  __syncthreads();
  table[(size_t)threadIdx.x * nblocks + blockIdx.x] = h[threadIdx.x];  // digit-major
}

// one block per digit: exclusive scan of its row of block counts (in place); total[d] = row sum
__global__ void __launch_bounds__(1024) lv_radix_scan_rows_kernel(unsigned int* __restrict__ table, int nblocks,
                                                                  unsigned int* __restrict__ total) {
  __shared__ unsigned int part[1024];
  unsigned int* row = table + (size_t)blockIdx.x * nblocks;
  const int per = (nblocks + 1023) / 1024;
  const int b0 = threadIdx.x * per, b1 = min(b0 + per, nblocks);
  unsigned int s = 0;
  for (int b = b0; b < b1; ++b) s += row[b];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {  // Hillis-Steele inclusive scan
    unsigned int v = threadIdx.x >= off ? part[threadIdx.x - off] : 0u;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  unsigned int run = part[threadIdx.x] - s;  // exclusive prefix of this thread's chunk
  for (int b = b0; b < b1; ++b) {
    const unsigned int v = row[b];
    row[b] = run;
    run += v;
  }
  if (threadIdx.x == 1023) total[blockIdx.x] = part[1023];
}

__global__ void lv_radix_scan_digits_kernel(const unsigned int* __restrict__ total, unsigned int* __restrict__ digit_base) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    unsigned int run = 0;
    for (int d = 0; d < 256; ++d) {
      digit_base[d] = run;
      run += total[d];
    }
  }
}

// stable scatter: rank inside the block by rounds of 256 keys (warp match + per-warp digit counts)
__global__ void __launch_bounds__(LV_THREADS)
    lv_radix_scatter_kernel(const unsigned long long* __restrict__ in, unsigned long long* __restrict__ out, long long n, int shift,
                            const unsigned int* __restrict__ table, const unsigned int* __restrict__ digit_base, int nblocks) {
  __shared__ unsigned int run[256];            // next output offset per digit for this block
  __shared__ unsigned int wcnt[8][256];        // per-warp digit counts of the current round
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  run[threadIdx.x] = digit_base[threadIdx.x] + table[(size_t)threadIdx.x * nblocks + blockIdx.x];
#pragma unroll
  for (int w = 0; w < 8; ++w) wcnt[w][threadIdx.x] = 0;
  __syncthreads();
  const long long base = (long long)blockIdx.x * LV_TILE;
  for (int k = 0; k < LV_ITEMS; ++k) {
    const long long i = base + (long long)k * LV_THREADS + threadIdx.x;
    const bool ok = i < n;
    unsigned long long key = 0;
    unsigned int d = 256;  // sentinel digit for out-of-range lanes (never matches a real digit)
    if (ok) {
      key = in[i];
      d = (unsigned int)(key >> shift) & 255u;
    }
    const unsigned int peers = __match_any_sync(0xffffffffu, d);
    const unsigned int rank_in_warp = __popc(peers & ((1u << lane) - 1u));
    if (ok && rank_in_warp == 0) wcnt[warp][d] = __popc(peers);
    __syncthreads();
    if (ok) {
      unsigned int off = run[d] + rank_in_warp;
      for (int w = 0; w < warp; ++w) off += wcnt[w][d];
      out[off] = key;
    }
    __syncthreads();
    {
      unsigned int s = 0;
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        s += wcnt[w][threadIdx.x];
        wcnt[w][threadIdx.x] = 0;
      }
      run[threadIdx.x] += s;
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- 3. per-class scan of fg + Lovász gradient
constexpr int LV_JT = 4096;  // keys per block in the jaccard stage (256 threads x 16)

__global__ void __launch_bounds__(256) lv_tile_sums_kernel(const unsigned long long* __restrict__ keys, long long P, int tiles,
                                                           unsigned int* __restrict__ tile_sum) {
  const int r = blockIdx.y, t = blockIdx.x;
  const long long base = (long long)r * P + (long long)t * LV_JT;
  const long long end = min((long long)r * P + P, base + LV_JT);
  unsigned int s = 0;
  for (long long i = base + threadIdx.x; i < end; i += 256) s += (unsigned int)(keys[i] >> 23) & 1u;
  __shared__ unsigned int red[256];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if (threadIdx.x < off) red[threadIdx.x] += red[threadIdx.x + off];
    __syncthreads();
  }
  if (threadIdx.x == 0) tile_sum[(size_t)r * tiles + t] = red[0];
}

// one block per class: exclusive scan of its tile sums (in place) and gts[r] = number of foreground pixels
__global__ void __launch_bounds__(1024) lv_class_scan_kernel(unsigned int* __restrict__ tile_sum, int tiles, unsigned int* __restrict__ gts) {
  __shared__ unsigned int part[1024];
  unsigned int* row = tile_sum + (size_t)blockIdx.x * tiles;
  const int per = (tiles + 1023) / 1024;
  const int b0 = threadIdx.x * per, b1 = min(b0 + per, tiles);
  unsigned int s = 0;
  for (int b = b0; b < b1; ++b) s += row[b];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    unsigned int v = threadIdx.x >= off ? part[threadIdx.x - off] : 0u;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  unsigned int run = part[threadIdx.x] - s;
  for (int b = b0; b < b1; ++b) {
    const unsigned int v = row[b];
    row[b] = run;
    run += v;
  }
  if (threadIdx.x == 1023) gts[blockIdx.x] = part[1023];
}

__device__ __forceinline__ float lv_jaccard(float gts, float cumfg, float cumbg) {
  const float inter = gts - cumfg;
  const float uni = gts + cumbg;
  return 1.f - inter / uni;  // lovasz_losses.py:26-28
}

__global__ void __launch_bounds__(256)
    lv_jaccard_kernel(const unsigned long long* __restrict__ keys, long long P, int tiles, const unsigned int* __restrict__ tile_off,
                      const unsigned int* __restrict__ gts_arr, const int* __restrict__ class_of_rank, int C, long long HW,
                      double* __restrict__ loss_part /*[n_present][tiles]*/, float* __restrict__ gprob /*NCHW scratch*/) {
  const int r = blockIdx.y, t = blockIdx.x;
  const long long cbase = (long long)r * P;
  const long long base = cbase + (long long)t * LV_JT;
  const long long end = min(cbase + P, base + LV_JT);
  const float gts = (float)gts_arr[r];
  const int cls = class_of_rank[r];
  // each thread owns 16 CONSECUTIVE keys -> local serial scan, then a block scan of the per-thread sums
  const long long my0 = base + (long long)threadIdx.x * 16;
  unsigned long long k[16];
  unsigned int mysum = 0;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const long long i = my0 + j;
    k[j] = i < end ? keys[i] : 0ull;
    mysum += (unsigned int)(k[j] >> 23) & 1u;
  }
  __shared__ unsigned int part[256];
  part[threadIdx.x] = mysum;
  __syncthreads();
  for (int off = 1; off < 256; off <<= 1) {
    unsigned int v = threadIdx.x >= off ? part[threadIdx.x - off] : 0u;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  unsigned int cum = tile_off[(size_t)r * tiles + t] + part[threadIdx.x] - mysum;  // fg count strictly before my first key
  double acc = 0.0;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const long long i = my0 + j;
    if (i >= end) break;
    const unsigned int fg = (unsigned int)(k[j] >> 23) & 1u;
    const long long pos = i - cbase;  // 0-based rank inside the class
    const float cumfg_prev = (float)cum, cumbg_prev = (float)(pos - (long long)cum);
    cum += fg;
    const float cumfg = (float)cum, cumbg = (float)(pos + 1 - (long long)cum);
    const float j_now = lv_jaccard(gts, cumfg, cumbg);
    const float j_prev = pos > 0 ? lv_jaccard(gts, cumfg_prev, cumbg_prev) : 0.f;
    const float d = j_now - j_prev;  // lovasz_grad, lovasz_losses.py:29-30
    const float err = __uint_as_float(~(unsigned int)(k[j] >> 24));
    acc += (double)err * (double)d;
    const long long pix = (long long)(k[j] & 0x7FFFFFull);
    const long long n = pix / HW;
    // d|fg - p| / dp = -1 for foreground, +1 for background
    gprob[(n * C + cls) * HW + (pix - n * HW)] = fg ? -d : d;
  }
  acc = warp_sum_d(acc);
  __shared__ double wsum[8];
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += wsum[w];
    loss_part[(size_t)r * tiles + t] = s;
  }
}

__global__ void lv_class_of_rank_kernel(const int* __restrict__ rank, int C, int* __restrict__ class_of_rank) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C && rank[c] >= 0) class_of_rank[rank[c]] = c;
}

// one block: loss_c = the tile partials of class c folded in a fixed order (strided per thread, then the warp and block
// trees), loss = mean over the present classes; no atomics, so the value does not depend on the block schedule
__global__ void __launch_bounds__(256) lv_loss_kernel(const double* __restrict__ loss_part, int n_present, int tiles,
                                                      float* __restrict__ loss) {
  __shared__ double wsum[8];
  double total = 0.0;
  for (int r = 0; r < n_present; ++r) {
    double s = 0.0;
    for (int t = threadIdx.x; t < tiles; t += 256) s += loss_part[(size_t)r * tiles + t];
    s = warp_sum_d(s);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      double c = 0.0;
      for (int w = 0; w < 8; ++w) c += wsum[w];
      total += c;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss = n_present > 0 ? (float)(total / n_present) : 0.f;
}

// ---------------------------------------------------------------- 4. softmax Jacobian, in place on the NCHW scratch
__global__ void __launch_bounds__(256)
    lv_softmax_bwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target, int N, int C, int H, int W,
                          int64_t ignore, const int* __restrict__ rank, float inv_present, float* __restrict__ g) {
  const int64_t HW = (int64_t)H * W, total = (int64_t)N * HW;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / HW);
    const int64_t off = (int64_t)n * C * HW + (i - (int64_t)n * HW);
    float* gp = g + off;
    if (target[i] == ignore) {
      for (int c = 0; c < C; ++c) gp[(int64_t)c * HW] = 0.f;
      continue;
    }
    const float* l = logits + off;
    float mx = -INFINITY;
    for (int c = 0; c < C; ++c) mx = fmaxf(mx, l[(int64_t)c * HW]);
    float se = 0.f;
    for (int c = 0; c < C; ++c) se += expf(l[(int64_t)c * HW] - mx);
    const float inv = 1.f / se;
    float dot = 0.f;
    for (int c = 0; c < C; ++c) {
      if (rank[c] < 0) continue;
      dot += gp[(int64_t)c * HW] * expf(l[(int64_t)c * HW] - mx) * inv;
    }
    for (int c = 0; c < C; ++c) {
      const float p = expf(l[(int64_t)c * HW] - mx) * inv;
      const float gc = rank[c] >= 0 ? gp[(int64_t)c * HW] : 0.f;
      gp[(int64_t)c * HW] = p * (gc - dot) * inv_present;
    }
  }
}

}  // namespace seg

using namespace seg;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

// counts: int32 [C + 1], zeroed here; counts[c] = valid pixels of class c, counts[C] = all valid pixels
int seg_lovasz_count(const int64_t* target, int64_t npix, int C, int64_t ignore_index, int32_t* counts, void* stream) {
  SEG_REQUIRE(C <= LV_MAXC, "lovasz: at most %d classes", LV_MAXC);
  cudaMemsetAsync(counts, 0, (size_t)(C + 1) * sizeof(int32_t), ST(stream));
  int blocks = (int)std::min<int64_t>(ceil_div64(npix, 256 * 8), (int64_t)num_sms() * 4);
  lv_count_kernel<<<blocks < 1 ? 1 : blocks, 256, 0, ST(stream)>>>(target, npix, C, ignore_index, counts);
  return check_launch("lv_count");
}

// bytes of the workspace for P valid pixels and n_present classes (radix table + totals + tile sums + ...)
int64_t seg_lovasz_workspace_bytes(int64_t P, int n_present, int C) {
  const int64_t nkeys = P * n_present;
  const int64_t nblocks = ceil_div64(nkeys, LV_TILE);
  const int64_t tiles = ceil_div64(P, LV_JT);
  int64_t b = 0;
  b += 256 * nblocks * 4;                 // radix table
  b += 256 * 4 * 2;                       // totals + digit bases
  b += (int64_t)n_present * tiles * 4;    // tile sums / offsets
  b += (int64_t)n_present * 4;            // gts
  b += (int64_t)n_present * tiles * 8;    // loss per class and tile (fp64)
  b += (int64_t)C * 4 * 2;                // rank, class_of_rank
  b += 16 * 16;                           // alignment slack
  return b;
}

// loss (fp32 scalar) and dlogits = d loss / d logits (NCHW fp32, also used as scratch).  keys0/keys1: uint64 [n_present*P].
int seg_lovasz_softmax_nchw(const float* logits, const int64_t* target, int N, int C, int H, int W, int64_t ignore_index,
                            const int32_t* counts, int64_t P, int n_present, void* keys0, void* keys1, void* workspace,
                            float* loss, float* dlogits, void* stream) {
  SEG_REQUIRE(C <= LV_MAXC && n_present >= 0 && n_present <= C, "lovasz: bad class counts");
  const int64_t npix = (int64_t)N * H * W;
  SEG_REQUIRE(npix < (1ll << 23), "lovasz: more than 2^23 pixels per batch are not supported by the key layout");
  cudaStream_t st = ST(stream);
  const int64_t HW = (int64_t)H * W;
  if (P == 0 || n_present == 0) {  // only void pixels: loss 0, gradient 0 (lovasz_losses.py:178-180)
    cudaMemsetAsync(loss, 0, sizeof(float), st);
    cudaMemsetAsync(dlogits, 0, (size_t)npix * C * sizeof(float), st);
    return 0;
  }
  const int64_t nkeys = P * n_present;
  SEG_REQUIRE(nkeys < (1ll << 32), "lovasz: too many keys");
  const int nblocks = (int)ceil_div64(nkeys, LV_TILE);
  const int tiles = (int)ceil_div64(P, LV_JT);
  // carve the workspace
  uint8_t* w = reinterpret_cast<uint8_t*>(workspace);
  auto take = [&](size_t bytes) { uint8_t* p = w; w += (bytes + 15) & ~(size_t)15; return p; };
  unsigned int* table = reinterpret_cast<unsigned int*>(take((size_t)256 * nblocks * 4));
  unsigned int* total = reinterpret_cast<unsigned int*>(take(256 * 4));
  unsigned int* dbase = reinterpret_cast<unsigned int*>(take(256 * 4));
  unsigned int* tsum = reinterpret_cast<unsigned int*>(take((size_t)n_present * tiles * 4));
  unsigned int* gts = reinterpret_cast<unsigned int*>(take((size_t)n_present * 4));
  double* lpart = reinterpret_cast<double*>(take((size_t)n_present * tiles * 8));
  int* rank = reinterpret_cast<int*>(take((size_t)C * 4));
  int* cor = reinterpret_cast<int*>(take((size_t)C * 4));

  lv_rank_kernel<<<1, 32, 0, st>>>(counts, C, rank);
  if (check_launch("lv_rank")) return 1;
  lv_class_of_rank_kernel<<<ceil_div(C, 128), 128, 0, st>>>(rank, C, cor);
  if (check_launch("lv_class_of_rank")) return 1;
  // key slots: per-chunk valid counts and their exclusive scan, kept in dlogits (npix * C floats >= one word per chunk)
  // until the emission has read them; dlogits is zeroed after it
  const int64_t nchunks = ceil_div64(npix, LV_THREADS);
  unsigned int* chunk_off = reinterpret_cast<unsigned int*>(dlogits);
  const int eb = (int)std::min<int64_t>(nchunks, (int64_t)num_sms() * 8);
  lv_chunk_count_kernel<<<eb, LV_THREADS, 0, st>>>(target, npix, ignore_index, chunk_off);
  if (check_launch("lv_chunk_count")) return 1;
  lv_radix_scan_rows_kernel<<<1, 1024, 0, st>>>(chunk_off, (int)nchunks, total);
  if (check_launch("lv_chunk_scan")) return 1;
  unsigned long long* ka = reinterpret_cast<unsigned long long*>(keys0);
  unsigned long long* kb = reinterpret_cast<unsigned long long*>(keys1);
  lv_emit_kernel<<<eb, LV_THREADS, 0, st>>>(logits, target, N, C, H, W, ignore_index, rank, (long long)P, ka, chunk_off);
  if (check_launch("lv_emit")) return 1;
  cudaMemsetAsync(dlogits, 0, (size_t)npix * C * sizeof(float), st);
  for (int pass = 0; pass < 5; ++pass) {
    const int shift = 24 + 8 * pass;
    lv_radix_hist_kernel<<<nblocks, LV_THREADS, 0, st>>>(ka, nkeys, shift, table, nblocks);
    if (check_launch("lv_radix_hist")) return 1;
    lv_radix_scan_rows_kernel<<<256, 1024, 0, st>>>(table, nblocks, total);
    if (check_launch("lv_radix_scan_rows")) return 1;
    lv_radix_scan_digits_kernel<<<1, 32, 0, st>>>(total, dbase);
    if (check_launch("lv_radix_scan_digits")) return 1;
    lv_radix_scatter_kernel<<<nblocks, LV_THREADS, 0, st>>>(ka, kb, nkeys, shift, table, dbase, nblocks);
    if (check_launch("lv_radix_scatter")) return 1;
    unsigned long long* tmp = ka;
    ka = kb;
    kb = tmp;
  }
  dim3 jg((unsigned)tiles, (unsigned)n_present, 1);
  lv_tile_sums_kernel<<<jg, 256, 0, st>>>(ka, (long long)P, tiles, tsum);
  if (check_launch("lv_tile_sums")) return 1;
  lv_class_scan_kernel<<<n_present, 1024, 0, st>>>(tsum, tiles, gts);
  if (check_launch("lv_class_scan")) return 1;
  lv_jaccard_kernel<<<jg, 256, 0, st>>>(ka, (long long)P, tiles, tsum, gts, cor, C, HW, lpart, dlogits);
  if (check_launch("lv_jaccard")) return 1;
  lv_loss_kernel<<<1, 256, 0, st>>>(lpart, n_present, tiles, loss);
  if (check_launch("lv_loss")) return 1;
  lv_softmax_bwd_kernel<<<eb, 256, 0, st>>>(logits, target, N, C, H, W, ignore_index, rank, 1.f / (float)n_present, dlogits);
  return check_launch("lv_softmax_bwd");
}

}  // extern "C"
