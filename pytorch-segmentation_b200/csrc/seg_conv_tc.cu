// seg_conv_tc.cu — wgmma + TMA implicit-GEMM convolution for sm_90a (forward, data-gradient, weight-gradient).
//
// Replaces what the reference dispatches to cuDNN for every nn.Conv2d on the hot path (dense 3x3 / dilated 3x3 /
// 1x1; SURVEY.md §2.3): models/deeplabv3_plus.py:256 (ASPP d=6/12/18), :312-315 (decoder 3x3), torchvision
// Bottleneck conv1/conv2/conv3 (layer4 conv2 dilated at deeplabv3_plus.py:47-53), models/resnet.py:43-48.
//
// Two kernels share one pipeline: a TMA producer warpgroup feeding an mbarrier ring, wgmma consumer warpgroups with fp32
// accumulators in registers.  The activation operand is fetched with an IM2COL-mode tensor map: one instruction brings 128
// output pixels x 64 channels of one filter tap (tap displacement passed as the im2col offset, padding = the bounding-box
// corners, out-of-image taps zero-filled by the TMA unit) straight into the 128B-swizzled K-major layout wgmma consumes —
// the im2col gather happens in the copy engine, never in HBM.  Weights come through a tiled 2-D map over the packed
// [tap][K][C] matrix.
//
// conv_gemm_pp<BN, KIND> — fprop (KK) and dgrad (KM): persistent, warp-specialised "ping-pong" kernel.  One CTA per SM walks
// the 128 x BN output tiles t = blockIdx.x, blockIdx.x + gridDim.x, ...  (384 threads):
//   warpgroup 0   : TMA producer (one thread) — loads the k-blocks of the CTA's tiles into the ring, tile after tile.
//   warpgroups 1-2: consumers that take alternate tiles; each owns a whole 128 x BN tile (two m64 wgmma row blocks).  An
//                   ordered pair of named barriers lets one warpgroup issue MMAs at a time while the other runs the epilogue
//                   of its previous tile: accumulators (+ bias) -> its private XOR-swizzled staging tile -> per-channel sum /
//                   sum of squares of the values as stored (BatchNorm statistics, fixed order, one fp64 atomic per channel
//                   per tile) -> fully coalesced 16-byte global stores (optionally beta-accumulate, optionally onto a strided
//                   sub-grid of the output).  The epilogue of tile i thus hides under the main loop of tile i + 1.
//   KK (fprop) : A = activations (K-major),  B = weights  [tap*K + k][c]   (K-major)
//   KM (dgrad) : A = dY im2col  (K-major),  B = weights  [tap*K + k][c]   (MN-major: c contiguous).  Stride 1: taps
//                flipped.  Stride s > 1: the input pixels are split into s*s parity classes; each class is a stride-1
//                gather over dY with only the taps whose parity matches, written to its strided sub-grid of dX —
//                no wasted MACs on inserted zeros.
// conv_gemm_wgrad<BN> — wgrad (MM): one 128 x BN tile per CTA, the two consumer warpgroups splitting its rows.
//   A = dY [pixel][k] (MN-major), B = X im2col [pixel][c] (MN-major), contraction over pixels, split-K over pixel blocks
//   sized to one wave: each split stores its partial tile to a workspace [split][tap][k][c] and a second kernel adds the
//   splits to dW[tap][k][c] in split order — bit-reproducible, unlike atomics.
#include <cuda.h>
#include <mutex>
#include <stdlib.h>
#include "seg_common.cuh"
#include "seg_ptx.cuh"
#include "seg_sync.cuh"

namespace seg {
namespace tc {

using namespace ptx;

constexpr int BM = 128;
constexpr int BK = 64;  // elements per k-block = 128 bytes of bf16
constexpr int A_BYTES = BM * 128;
constexpr int KIND_KK = 0, KIND_KM = 1;
constexpr int NTHREADS = 384;
constexpr int NCONS = 256;  // consumer threads (warpgroups 1 and 2)
constexpr int MAXT = 49;

// named barriers (0 is __syncthreads)
constexpr int BAR_CONSUMERS = 1;  // both consumer warpgroups (256 threads)
constexpr int BAR_ORDER = 2;      // 2 + c: consumer c may issue its MMAs (ping-pong kernel)
constexpr int BAR_WG = 4;         // 4 + c: the 128 threads of consumer c (ping-pong kernel)

struct TcParams {
  CUtensorMap mapA;  // KK/KM: activation-side operand ; MM: dY 2-D
  CUtensorMap mapB;  // KK/KM: packed weights 2-D      ; MM: X (im2col or 2-D)
  int M;             // valid output rows
  int Ncols;         // valid output cols
  int taps;          // entries of the tap table
  int kchunks;       // KK/KM: 64-wide channel chunks per tap
  int stride;        // traversal stride of the im2col map (row -> base coordinate)
  int lower_h, lower_w;
  int PQ, Q;         // row index -> (n, p, q)
  int x_im2col;      // activation operand uses the im2col map
  int brows_per_tap; // weight-matrix rows per tap
  short tap_wt[MAXT];  // weight tap index
  short tap_oh[MAXT];  // im2col offset (h)
  short tap_ow[MAXT];  // im2col offset (w)
  void* out;
  long long ldo;
  int out_dtype;
  float beta;
  const float* bias;
  double* stats;     // [2*Ncols] or null, ZERO at launch: per-channel sum / sum of squares of the output (BatchNorm batch
                     // statistics), accumulated with fp64 atomics (see the epilogue)
  int stat_rows;     // rows per group of the statistics fold (32, 64 or 128; see stat_rows_for)
  unsigned* stat_ticket;   // SyncBN only: one zeroed word counting finished CTAs
  SyncDesc sync;           // world > 0: SyncBN — the last CTA pushes the finished totals to every peer (seg_sync.cuh)
  // strided sub-grid output (stride>1 dgrad): row (n,i,j) -> pixel (n, i*osy+opy, j*osx+opx) of an out_H x out_W map
  int out_strided, out_H, out_W, osy, osx, opy, opx;
  // KK/KM: tile t covers rows (t / n_tiles) * BM and columns (t % n_tiles) * BN — the column block runs fastest, so the
  // CTAs working at the same time share their activation rows in L2 and each row block comes from HBM once, however many
  // column blocks the layer has (with the row block fastest, every column block would stream the whole activation
  // operand again — 71 MB for layer 4's 2048-channel 1x1 convs, more than the 50 MB L2)
  int n_tiles, tiles;
  // MM only
  int kblocks_total, kblocks_per_split;
  float* dw;
  int dw_K, dw_C;
  float* ws;  // split-K partials [split][tap][dw_K][dw_C]; null with one split (the tile is added to dW directly)
};

__device__ __forceinline__ void row_to_coords(int m, int PQ, int Q, int stride, int lower_h, int lower_w, int& n, int& h,
                                              int& w) {
  n = m / PQ;
  int rem = m - n * PQ;
  int pp = rem / Q;
  int qq = rem - pp * Q;
  h = lower_h + pp * stride;
  w = lower_w + qq * stride;
}

template <int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_tile(float* acc, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if constexpr (BN == 64) wgmma_m64n64k16<TA, TB>(acc, adesc, bdesc, accumulate);
  else if constexpr (BN == 128) wgmma_m64n128k16<TA, TB>(acc, adesc, bdesc, accumulate);
  else wgmma_m64n256k16<TA, TB>(acc, adesc, bdesc, accumulate);
}

// The TMA loads of one k-block (ring stage `st`) of a KK / KM tile.
template <int BN, int KIND>
__device__ __forceinline__ void load_kblock(const TcParams& p, uint32_t a_dst, uint32_t bar, int kc, int wtap, uint16_t oh,
                                            uint16_t ow, int n_img, int h0, int w0, int m0, int n0) {
  const uint32_t b_dst = a_dst + A_BYTES;
  if (p.x_im2col)
    tma_load_im2col_4d(a_dst, &p.mapA, bar, kc * BK, w0, h0, n_img, ow, oh);
  else
    tma_load_2d(a_dst, &p.mapA, bar, kc * BK, m0);
  if (KIND == KIND_KK) {
    tma_load_2d(b_dst, &p.mapB, bar, kc * BK, wtap * p.brows_per_tap + n0);  // box [BN][64]
  } else {
#pragma unroll
    for (int j = 0; j < BN / 64; ++j)  // boxes [64 k-rows][64 cols]
      tma_load_2d(b_dst + j * 8192, &p.mapB, bar, n0 + j * 64, wtap * p.brows_per_tap + kc * BK);
  }
}

// The accumulators of one m64 x BN wgmma row block (+ bias) -> rows rbase.. of the XOR-swizzled staging tile
// [128 rows][BN * esize bytes]; with acc1, also those of the row block below it (rows rbase + 64..).  `bias`: the tile's BN
// bias values in shared memory, zero past the layer's last column (or null).
template <int BN>
__device__ __forceinline__ void stage_acc(const float* acc, const float* acc1, uint8_t* stage, int rbase, int warp, int lane,
                                          const float* bias, bool out_f32) {
  const int esize = out_f32 ? 4 : 2;
  const int CPR = BN * esize / 16;  // 16-byte chunks per staged row
  const int swz = (CPR >= 32 ? 31 : CPR - 1);
  const int r0 = rbase + warp * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = j * 8 + 2 * (lane & 3);
    float b0 = 0.f, b1 = 0.f;
    if (bias) {
      b0 = bias[col];
      b1 = bias[col + 1];
    }
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      if (h >= 2 && !acc1) break;
      const float* a = h < 2 ? acc : acc1;
      const int r = r0 + 8 * (h & 1) + 32 * (h & 2);
      const float x0 = a[4 * j + 2 * (h & 1)] + b0, x1 = a[4 * j + 2 * (h & 1) + 1] + b1;
      const int byte = col * esize;
      uint8_t* dst = stage + (size_t)r * (BN * esize) + ((((byte >> 4) ^ (r & swz))) << 4) + (byte & 15);
      if (out_f32)
        *reinterpret_cast<float2*>(dst) = make_float2(x0, x1);
      else
        *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(x0, x1);
    }
  }
}

// ================================ fprop / dgrad: persistent ping-pong kernel ================================

// Ring depth per tile width.  Each consumer has a private staging tile of 128 rows x 256 B (BN * esize <= 256: fp32 outputs
// take BN = 64) and a private statistics scratch, because the ring never idles and cannot double as the staging area.
template <int BN>
struct PPCfg {
  static_assert(BN == 64 || BN == 128, "ping-pong tile width");
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = BN == 64 ? 6 : 4;
  static constexpr int RING = STAGES * STAGE_BYTES;
  static constexpr int STG_BYTES = BM * 256;
  static constexpr int MAXG = BM / 32;                  // statistics row groups per tile (stat_rows >= 32)
  static constexpr int STAT_BYTES = MAXG * 2 * BN * 4 + BN * 4;  // [group][sum, sum of squares][column] fp32 + [column] bias
  static constexpr int SMEM = RING + 2 * (STG_BYTES + STAT_BYTES) + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(16 * STAGES + 8 <= 256, "barrier area");
  static_assert(SMEM <= 227 * 1024, "shared memory per block");
};

template <int BN, int KIND>
__global__ void __launch_bounds__(NTHREADS, 1) conv_gemm_pp(const __grid_constant__ TcParams p) {
  using C = PPCfg<BN>;
  constexpr int STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t smem0 = (raw_addr + 1023u) & ~1023u;  // 1024-B alignment for SWIZZLE_128B atoms
  uint8_t* smem_gen = smem_raw + (smem0 - raw_addr);
  const uint32_t bar0 = smem0 + C::RING + 2 * (C::STG_BYTES + C::STAT_BYTES);
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (STAGES + s); };
  volatile int* flag_sm = reinterpret_cast<volatile int*>(smem_gen + (bar0 - smem0) + 16 * STAGES);

  const int num_iters = p.taps * p.kchunks;  // k-blocks per tile (0: a parity class no tap reaches — zeros are written)
  const int grid = gridDim.x;
  const int ntiles = (p.tiles - (int)blockIdx.x + grid - 1) / grid;  // this CTA's tiles: blockIdx.x + j * grid

  if (threadIdx.x == 0) {
    prefetch_tmap(&p.mapA);
    prefetch_tmap(&p.mapB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 4);  // each stage is consumed by one warpgroup: one arrival per warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // setup above overlapped the previous kernel's tail; global memory is touched only from here on

  if (threadIdx.x < 128) {
    // =============================== TMA producer ===============================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0 && num_iters > 0) {
      int it = 0;
      for (int j = 0; j < ntiles; ++j) {
        const int t = blockIdx.x + j * grid;
        const int m0 = (t / p.n_tiles) * BM, n0 = (t % p.n_tiles) * BN;
        int n_img = 0, h0 = 0, w0 = 0;
        if (p.x_im2col) row_to_coords(m0, p.PQ, p.Q, p.stride, p.lower_h, p.lower_w, n_img, h0, w0);
        for (int tap = 0; tap < p.taps; ++tap) {
          const int wtap = p.tap_wt[tap];
          const uint16_t oh = (uint16_t)p.tap_oh[tap], ow = (uint16_t)p.tap_ow[tap];
          for (int kc = 0; kc < p.kchunks; ++kc, ++it) {
            const int st = it % STAGES;
            mbar_wait_nocall(empty_bar(st), ((it / STAGES) & 1) ^ 1u);
            mbar_arrive_expect_tx(full_bar(st), C::STAGE_BYTES);
            load_kblock<BN, KIND>(p, smem0 + st * C::STAGE_BYTES, full_bar(st), kc, wtap, oh, ow, n_img, h0, w0, m0, n0);
          }
        }
      }
    }
    return;
  }

  // =============================== wgmma consumers ===============================
  setmaxnreg_inc<232>();
  const int cw = (threadIdx.x - 128) >> 7;  // consumer warpgroup: local tiles j = cw, cw + 2, ...
  const int tid = threadIdx.x & 127;
  const int warp = tid >> 5, lane = tid & 31;
  uint8_t* stage = smem_gen + C::RING + cw * C::STG_BYTES;
  float* stat_sm = reinterpret_cast<float*>(smem_gen + C::RING + 2 * C::STG_BYTES + cw * C::STAT_BYTES);
  float* bias_sm = stat_sm + C::MAXG * 2 * BN;
  const bool out_f32 = p.out_dtype != SEG_DT_BF16;
  const int esize = out_f32 ? 4 : 2;
  const int CPR = BN * esize / 16;  // 16-byte chunks per staged row
  const int swz = (CPR >= 32 ? 31 : CPR - 1);
  auto wg_sync = [&] { named_sync(BAR_WG + cw, 128); };

  for (int j = cw; j < ntiles; j += 2) {
    const int t = blockIdx.x + j * grid;
    const int m0 = (t / p.n_tiles) * BM, n0 = (t % p.n_tiles) * BN;
    float acc0[BN / 2], acc1[BN / 2];  // rows 0..63 and 64..127 of the tile
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc0[i] = acc1[i] = 0.f;

    // ---- main loop: only after the other consumer has issued every MMA of local tile j - 1 ----
    if (j > 0) named_sync(BAR_ORDER + cw, NCONS);
    {
      constexpr int TB = (KIND == KIND_KK) ? 0 : 1;
      const int it0 = j * num_iters;  // ring position of this tile's first k-block: the producer loads tiles in order
      for (int i = 0; i < num_iters; ++i) {
        const int it = it0 + i;
        const int st = it % STAGES;
        mbar_wait_nocall(full_bar(st), (it / STAGES) & 1);
        const uint32_t a_addr = smem0 + st * C::STAGE_BYTES;  // K-major: 128 rows x 128 B, rows 64.. at +8192
        const uint32_t b_addr = a_addr + A_BYTES;
        // K-major: 8-row atoms 1024 B apart, K advance = 32 B inside the swizzle atom.
        // MN-major: 64-wide MN blocks one box (8192 B) apart, 8-row K groups 1024 B apart, K advance = 16 rows.
        const uint64_t adesc0 = make_smem_desc_sw128(a_addr, 16, 1024);
        const uint64_t adesc1 = make_smem_desc_sw128(a_addr + 8192, 16, 1024);
        const uint64_t bdesc0 = make_smem_desc_sw128(b_addr, TB ? 8192 : 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t bdesc = bdesc0 + (uint64_t)(TB ? (k * 2048 >> 4) : (k * 32 >> 4));
          wgmma_tile<BN, 0, TB>(acc0, adesc0 + (uint64_t)(k * 32 >> 4), bdesc, 1u);
          wgmma_tile<BN, 0, TB>(acc1, adesc1 + (uint64_t)(k * 32 >> 4), bdesc, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs have retired: its stage goes back to the producer
        __syncwarp();
        if (i > 0 && lane == 0) mbar_arrive(empty_bar((it - 1) % STAGES));
      }
      if (j + 1 < ntiles) named_arrive(BAR_ORDER + (cw ^ 1), NCONS);  // the other consumer may start its main loop
      wgmma_wait<0>();
      __syncwarp();
      if (num_iters > 0 && lane == 0) mbar_arrive(empty_bar((it0 + num_iters - 1) % STAGES));
    }

    // -------- phase 1: registers -> (bias) -> swizzled staging tile --------
    const int ncols_tile = min(BN, p.Ncols - n0);
    if (p.bias && tid < BN) bias_sm[tid] = tid < ncols_tile ? __ldg(p.bias + n0 + tid) : 0.f;  // read in phase 1 only
    wg_sync();  // the previous tile's epilogue is done with the staging tile and the statistics scratch
    stage_acc<BN>(acc0, acc1, stage, 0, warp, lane, p.bias ? bias_sm : nullptr, out_f32);
    wg_sync();

    // -------- phase 2: BN statistics of the tile AS STORED (bf16-rounded for bf16 outputs — exactly what bn_apply
    //          normalises): per column, fp32 sums over groups of stat_rows rows, the groups added in order in phase 4.
    //          The grouping depends on the layer (stat_rows), never on the tile width, and a column's groups are shared
    //          by up to 128 / BN threads. --------
    const int ngroups = BM / p.stat_rows;
    if (p.stats) {
      const int parts = min(128 / BN, ngroups);  // threads per column
      const int rpp = BM / parts;                // rows per thread
      const int c = tid % BN, part = tid / BN;
      const int rvalid = min(BM, p.M - m0);
      if (part < parts) {
        const int byte = c * esize;
        int g = part * rpp / p.stat_rows;
        for (int rg = part * rpp; rg < (part + 1) * rpp; rg += p.stat_rows, ++g) {
          float s1 = 0.f, s2 = 0.f;
          const int rend = min(rg + p.stat_rows, rvalid);
          for (int r = rg; r < rend; ++r) {
            const uint8_t* src = stage + (size_t)r * (BN * esize) + ((((byte >> 4) ^ (r & swz))) << 4) + (byte & 15);
            const float x = out_f32 ? *reinterpret_cast<const float*>(src) : bf2f(*reinterpret_cast<const __nv_bfloat16*>(src));
            s1 += x;
            s2 = fmaf(x, x, s2);
          }
          stat_sm[(g * 2 + 0) * BN + c] = s1;
          stat_sm[(g * 2 + 1) * BN + c] = s2;
        }
      }
    }

    // -------- phase 3: coalesced 16-byte stores of the staged tile --------
    {
      const int nchunks = (ncols_tile * esize + 15) >> 4;  // 16-byte chunks that hold valid data
      const bool vec_ok = ((p.ldo * esize) & 15) == 0 && ((reinterpret_cast<uintptr_t>(p.out) + (size_t)n0 * esize) & 15) == 0;
      for (int idx = tid; idx < BM * CPR; idx += 128) {
        const int tr = idx / CPR;
        const int c16 = idx - tr * CPR;
        if (c16 >= nchunks) continue;
        const int grow = m0 + tr;
        if (grow >= p.M) continue;
        long long pixel = grow;
        if (p.out_strided) {
          const int n = grow / p.PQ;
          const int rem = grow - n * p.PQ;
          const int i = rem / p.Q, jj = rem - i * p.Q;
          pixel = ((long long)n * p.out_H + (i * p.osy + p.opy)) * p.out_W + (jj * p.osx + p.opx);
        }
        const uint8_t* src = stage + (size_t)tr * (BN * esize) + ((c16 ^ (tr & swz)) << 4);
        uint8_t* dst = reinterpret_cast<uint8_t*>(p.out) + ((size_t)pixel * p.ldo + n0) * esize + ((size_t)c16 << 4);
        const int first_col = (c16 << 4) / esize;
        const bool full = first_col + 16 / esize <= ncols_tile;
        if (!out_f32) {
          bf16x8 val = *reinterpret_cast<const bf16x8*>(src);
          if (vec_ok && full) {
            if (p.beta != 0.f) {
              float a[8], b[8];
              unpack8(val, a);
              unpack8(*reinterpret_cast<const bf16x8*>(dst), b);
#pragma unroll
              for (int k = 0; k < 8; ++k) a[k] += p.beta * b[k];
              val = pack8(a);
            }
            *reinterpret_cast<bf16x8*>(dst) = val;
          } else {
            float a[8];
            unpack8(val, a);
            __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(dst);
            for (int k = 0; k < 8; ++k)
              if (first_col + k < ncols_tile) {
                float o = a[k];
                if (p.beta != 0.f) o += p.beta * bf2f(d[k]);
                d[k] = f2bf(o);
              }
          }
        } else {
          const float4 val = *reinterpret_cast<const float4*>(src);
          const float a[4] = {val.x, val.y, val.z, val.w};
          float* d = reinterpret_cast<float*>(dst);
          if (vec_ok && full && p.beta == 0.f) {
            *reinterpret_cast<float4*>(d) = val;
          } else {
            for (int k = 0; k < 4; ++k)
              if (first_col + k < ncols_tile) d[k] = (p.beta != 0.f) ? a[k] + p.beta * d[k] : a[k];
          }
        }
      }
    }
    if (j == ntiles - 1 && tid == 0) pdl_trigger();  // the CTA's last tile is stored

    // -------- phase 4: this tile's column sums are added to the layer's totals with fp64 atomics.  Each contribution is an
    //          fp32 value, so the fp64 sum of the <= few thousand partials of a channel is EXACT (no rounding at all) whenever
    //          their exponents span less than 2^17 — then the order of the atomics cannot matter and the statistics are
    //          bit-reproducible (fp32 atomics were not, and the batch-2 image-pooling BatchNorm amplified that into 3-5 %
    //          logit differences between runs).  (Beyond that span the order can move the fp64 sum by one fp64 ulp —
    //          invisible after the rounding to fp32.) --------
    if (p.stats) {
      wg_sync();
      if (tid < ncols_tile) {
        float a = 0.f, b = 0.f;
        for (int g = 0; g < ngroups; ++g) {
          a += stat_sm[(g * 2 + 0) * BN + tid];
          b += stat_sm[(g * 2 + 1) * BN + tid];
        }
        atomicAdd(p.stats + n0 + tid, (double)a);
        atomicAdd(p.stats + p.Ncols + n0 + tid, (double)b);
      }
    }
  }

  // SyncBN: one ticket per CTA, taken after both consumers' atomics of every tile of the CTA
  if (p.stats && p.sync.world > 0)
    sync_push_when_last<false>(p.sync, p.stats, 2 * p.Ncols, p.stat_ticket, gridDim.x, threadIdx.x - 128, NCONS,
                               [] { named_sync(BAR_CONSUMERS, NCONS); }, flag_sm);
}

// ================================ wgrad: one tile per CTA ================================

// Pipeline stages per tile width: one CTA per SM (384 threads, up to 128 accumulator registers per consumer thread), so
// the ring takes most of the 227 KB; the fp32 staging tile of the epilogue (128 x BN x 4 B) reuses it.
template <int BN>
struct Cfg {
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = BN == 64 ? 6 : (BN == 128 ? 5 : 4);
  static constexpr int SMEM = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(STAGES * STAGE_BYTES >= BM * BN * 4, "staging tile must fit in the pipeline ring");
  static_assert(SMEM <= 227 * 1024, "shared memory per block");
};

template <int BN>
__global__ void __launch_bounds__(NTHREADS, 1) conv_gemm_wgrad(const __grid_constant__ TcParams p) {
  using C = Cfg<BN>;
  constexpr int STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t smem0 = (raw_addr + 1023u) & ~1023u;  // 1024-B alignment for SWIZZLE_128B atoms
  uint8_t* smem_gen = smem_raw + (smem0 - raw_addr);
  const uint32_t bar0 = smem0 + STAGES * C::STAGE_BYTES;
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (STAGES + s); };

  const int m0 = blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // ---- iteration space of the k loop ----
  const int tap_mm = blockIdx.z % p.taps;
  const int split = blockIdx.z / p.taps;
  const int kb_begin = split * p.kblocks_per_split;
  const int kb_end = min(kb_begin + p.kblocks_per_split, p.kblocks_total);
  const int num_iters = max(kb_end - kb_begin, 0);

  if (threadIdx.x == 0) {
    prefetch_tmap(&p.mapA);
    prefetch_tmap(&p.mapB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // setup above overlapped the previous kernel's tail; global memory is touched only from here on

  if (threadIdx.x < 128) {
    // =============================== TMA producer ===============================
    if (threadIdx.x == 0 && num_iters > 0) {
      const uint16_t oh = (uint16_t)p.tap_oh[tap_mm], ow = (uint16_t)p.tap_ow[tap_mm];
      int it = 0;
      for (int kb = kb_begin; kb < kb_end; ++kb, ++it) {
        const int st = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        mbar_wait_nocall(empty_bar(st), ph ^ 1u);
        const uint32_t a_dst = smem0 + st * C::STAGE_BYTES;
        const uint32_t b_dst = a_dst + A_BYTES;
        const int pix0 = kb * BK;
        mbar_arrive_expect_tx(full_bar(st), C::STAGE_BYTES);
        tma_load_2d(a_dst, &p.mapA, full_bar(st), m0, pix0);  // dY box [64 pixels][64 k]
        tma_load_2d(a_dst + 8192, &p.mapA, full_bar(st), m0 + 64, pix0);
        if (p.x_im2col) {
          int n_img, h0, w0;
          row_to_coords(pix0, p.PQ, p.Q, p.stride, p.lower_h, p.lower_w, n_img, h0, w0);
#pragma unroll
          for (int j = 0; j < BN / 64; ++j)
            tma_load_im2col_4d(b_dst + j * 8192, &p.mapB, full_bar(st), n0 + j * 64, w0, h0, n_img, ow, oh);
        } else {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) tma_load_2d(b_dst + j * 8192, &p.mapB, full_bar(st), n0 + j * 64, pix0);
        }
      }
    }
    return;
  }

  // =============================== wgmma consumers ===============================
  if (num_iters == 0) return;  // an empty split adds nothing (uniform across the consumers)
  const int ctid = threadIdx.x - 128;  // 0..255
  const int cw = ctid >> 7;            // consumer warpgroup: rows 64*cw.. of the tile
  const int warp = (ctid >> 5) & 3, lane = ctid & 31;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  for (int it = 0; it < num_iters; ++it) {
    const int st = it % STAGES;
    mbar_wait_nocall(full_bar(st), (it / STAGES) & 1);
    const uint32_t a_addr = smem0 + st * C::STAGE_BYTES + cw * 8192;  // MN-major: box cw
    const uint32_t b_addr = smem0 + st * C::STAGE_BYTES + A_BYTES;
    // MN-major: 64-wide MN blocks one box (8192 B) apart, 8-row K groups 1024 B apart, K advance = 16 rows.
    const uint64_t adesc0 = make_smem_desc_sw128(a_addr, 8192, 1024);
    const uint64_t bdesc0 = make_smem_desc_sw128(b_addr, 8192, 1024);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)
      wgmma_tile<BN, 1, 1>(acc, adesc0 + (uint64_t)(k * 2048 >> 4), bdesc0 + (uint64_t)(k * 2048 >> 4), 1u);
    wgmma_commit();
    wgmma_wait<1>();  // the previous k-block's MMAs have retired: its stage goes back to the producer
    __syncwarp();
    if (it > 0 && lane == 0) mbar_arrive(empty_bar((it - 1) % STAGES));
  }
  wgmma_wait<0>();
  named_sync(BAR_CONSUMERS, NCONS);  // both warpgroups are done reading the ring: it becomes the staging tile

  // -------- registers -> swizzled fp32 staging tile [128 rows][BN * 4 bytes] --------
  uint8_t* stage = smem_gen;
  const int ncols_tile = min(BN, p.Ncols - n0);
  stage_acc<BN>(acc, nullptr, stage, cw * 64, warp, lane, nullptr, true);
  named_sync(BAR_CONSUMERS, NCONS);

  // -------- wgrad tile: with one split, added to dW[tap][k][c] (once per element: order-free); with several, stored
  //          to this split's slice of the workspace for the fixed-order reduction --------
  const int CPR = BN * 4 / 16;
  const int swz = (CPR >= 32 ? 31 : CPR - 1);
  float* base = p.ws ? p.ws + (size_t)split * p.taps * p.dw_K * p.dw_C : p.dw;
  for (int idx = ctid; idx < BM * CPR; idx += NCONS) {
    const int tr = idx / CPR, c16 = idx - tr * CPR;
    const int row = m0 + tr, col0 = c16 * 4;
    if (row >= p.M || col0 >= ncols_tile) continue;
    const float4 v = *reinterpret_cast<const float4*>(stage + (size_t)tr * (BN * 4) + ((c16 ^ (tr & swz)) << 4));
    float* dst = base + ((size_t)tap_mm * p.dw_K + row) * p.dw_C + n0 + col0;
    const bool vec = col0 + 4 <= ncols_tile && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0);
    const float a[4] = {v.x, v.y, v.z, v.w};
    if (p.ws) {
      if (vec)
        *reinterpret_cast<float4*>(dst) = v;
      else
        for (int i = 0; i < 4; ++i)
          if (col0 + i < ncols_tile) dst[i] = a[i];
    } else if (vec) {
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                   : "memory");
    } else {
      for (int i = 0; i < 4; ++i)
        if (col0 + i < ncols_tile) atomicAdd(dst + i, a[i]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side: tensor-map construction (driver entry points resolved at run time; no -lcuda link dependency)
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode_tiled = nullptr;
static EncodeIm2colFn g_encode_im2col = nullptr;
static int g_driver_version = 0;

static int resolve_driver() {
  static std::once_flag once;
  static int status = 0;
  std::call_once(once, [] {
    void* f1 = nullptr;
    void* f2 = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f1, cudaEnableDefault, &q) != cudaSuccess || !f1) status = 1;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &f2, cudaEnableDefault, &q) != cudaSuccess || !f2) status = 1;
    g_encode_tiled = (EncodeTiledFn)f1;
    g_encode_im2col = (EncodeIm2colFn)f2;
    cudaDriverGetVersion(&g_driver_version);
  });
  if (status) set_error("cannot resolve cuTensorMapEncode* driver entry points");
  return status;
}

// 2-D bf16 matrix [rows][cols] with row pitch ld (elements); box = [box_rows][64 cols], 128B swizzle
static int make_map_2d(CUtensorMap* m, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  if (resolve_driver()) return 1;
  SEG_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "TMA: base pointer not 16-byte aligned");
  SEG_REQUIRE(ld % 8 == 0, "TMA: row pitch %lld not a multiple of 8 elements", (long long)ld);
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = g_encode_tiled(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, es,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SEG_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld box_rows=%d", (int)r,
              (long long)rows, (long long)cols, (long long)ld, box_rows);
  return 0;
}

// NHWC bf16 tensor, im2col mode: `pixels` base positions x 64 channels per load.  Corners per dimension (w, h).
static int make_map_im2col(CUtensorMap* m, const void* ptr, int N, int H, int W, int C, int64_t ld, int lower_w,
                           int lower_h, int upper_w, int upper_h, int stride, int pixels) {
  if (resolve_driver()) return 1;
  SEG_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "TMA: base pointer not 16-byte aligned");
  SEG_REQUIRE(ld % 8 == 0, "TMA: channel pitch %lld not a multiple of 8", (long long)ld);
  SEG_REQUIRE(lower_w >= -128 && upper_w >= -128 && lower_w <= 127 && upper_w <= 127 && lower_h >= -128 &&
                  upper_h >= -128 && lower_h <= 127 && upper_h <= 127,
              "im2col corner out of range");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)W * ld * 2, (cuuint64_t)H * W * ld * 2};
  int lo[2] = {lower_w, lower_h};
  int up[2] = {upper_w, upper_h};
  cuuint32_t es[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  CUresult r = g_encode_im2col(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, lo, up,
                               64, (cuuint32_t)pixels, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SEG_REQUIRE(r == CUDA_SUCCESS,
              "cuTensorMapEncodeIm2col failed (%d) N=%d H=%d W=%d C=%d ld=%lld lo=(%d,%d) up=(%d,%d) s=%d", (int)r, N, H,
              W, C, (long long)ld, lower_w, lower_h, upper_w, upper_h, stride);
  // Same workaround CUTLASS applies for drivers <= 13.1: small tensors (< 128 KiB) must clear bit 21 of word 1.
  if (g_driver_version <= 13010) {
    const uint64_t bytes = (uint64_t)N * H * W * ld * 2;
    if (bytes < 131072) reinterpret_cast<uint64_t*>(m)[1] &= ~(1ull << 21);
  }
  return 0;
}

// fprop / dgrad: the persistent grid, one CTA per SM (one per tile when there are fewer tiles).  Fills p.n_tiles / p.tiles.
template <int BN, int KIND>
static int launch_pp(TcParams& p, cudaStream_t stream) {
  static bool attr_set = false;
  auto kfn = conv_gemm_pp<BN, KIND>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, PPCfg<BN>::SMEM);
    SEG_REQUIRE(e == cudaSuccess, "cudaFuncSetAttribute(smem=%d): %s", PPCfg<BN>::SMEM, cudaGetErrorString(e));
    attr_set = true;
  }
  const int n_tiles = ceil_div(p.Ncols, BN);
  const int64_t tiles = ceil_div64(p.M, BM) * n_tiles;
  SEG_REQUIRE(tiles < (1ll << 31), "too many output tiles");
  p.n_tiles = n_tiles;
  p.tiles = (int)tiles;
  const dim3 grid((unsigned)std::min<int64_t>(tiles, num_sms()));
  launch_pdl(kfn, grid, dim3(NTHREADS), (size_t)PPCfg<BN>::SMEM, stream, p);
  return check_launch("conv_gemm_pp");
}

template <int KIND>
static int launch_pp_bn(int bn, TcParams& p, cudaStream_t stream) {
  switch (bn) {
    case 64: return launch_pp<64, KIND>(p, stream);
    case 128: return launch_pp<128, KIND>(p, stream);
  }
  set_error("bad BN %d", bn);
  return 1;
}

template <int BN>
static int launch_wgrad(const TcParams& p, dim3 grid, cudaStream_t stream) {
  static bool attr_set = false;
  auto kfn = conv_gemm_wgrad<BN>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::SMEM);
    SEG_REQUIRE(e == cudaSuccess, "cudaFuncSetAttribute(smem=%d): %s", Cfg<BN>::SMEM, cudaGetErrorString(e));
    attr_set = true;
  }
  launch_pdl(kfn, grid, dim3(NTHREADS), (size_t)Cfg<BN>::SMEM, stream, p);
  return check_launch("conv_gemm_wgrad");
}

static int launch_wgrad_bn(int bn, const TcParams& p, dim3 grid, cudaStream_t stream) {
  switch (bn) {
    case 64: return launch_wgrad<64>(p, grid, stream);
    case 128: return launch_wgrad<128>(p, grid, stream);
    case 256: return launch_wgrad<256>(p, grid, stream);
  }
  set_error("bad BN %d", bn);
  return 1;
}

// Tile width of fprop / dgrad: a consumer warpgroup holds a whole 128 x BN tile in registers (BN / 2 fp32 accumulators per
// thread and m64 row block), so BN <= 128; fp32 outputs take 64 (the staging tile is 128 rows x 256 B).
static int pick_bn(int ncols, bool out_f32) { return (ncols <= 64 || out_f32) ? 64 : 128; }

// Rows per group of the statistics fold of a layer with `ncols` output channels: 32 up to 64 channels, 128 from 256 channels
// on where the last 256-column block is not mostly padding, 64 otherwise.  A function of the layer only, never of the tile
// width, so the statistics do not depend on the picker.  These are the groups of the earlier one-tile-per-CTA kernel (its
// 128-row tile summed in 256 / BN groups, BN in {64, 128, 256} chosen by this rule), so its statistics are reproduced bit for bit.
static int stat_rows_for(int ncols) {
  if (ncols <= 64) return 32;
  if (ncols < 256) return 64;
  return ceil_div(ncols, 256) * 256 - ncols < 128 ? 128 : 64;
}

bool supported(const seg_conv_desc* d) {
  if (d->C % 8 != 0 || d->ldx % 8 != 0) return false;
  if (d->R != d->S) return false;
  if (d->R * d->S > MAXT) return false;
  if (d->pad > 127 || d->dil * (d->R - 1) - d->pad > 127 || d->dil * (d->R - 1) - d->pad < -127) return false;
  if (d->stride > 8) return false;
  return true;
}

static bool is_pointwise(const seg_conv_desc* d) { return d->R == 1 && d->S == 1 && d->stride == 1 && d->pad == 0; }

int conv_fwd(const seg_conv_desc* d, const void* x, const void* w, void* y, int y_dtype, const float* bias, float beta,
             double* stats, unsigned* stat_ticket, const SyncDesc* sync, cudaStream_t stream) {
  SEG_REQUIRE(supported(d), "wgmma conv fwd: unsupported shape (C=%d ldx=%d R=%d pad=%d dil=%d)", d->C, d->ldx, d->R,
              d->pad, d->dil);
  TcParams p;
  memset(&p, 0, sizeof(p));
  const int64_t M = (int64_t)d->N * d->P * d->Q;
  SEG_REQUIRE(M < (1ll << 31), "M too large");
  p.M = (int)M;
  p.Ncols = d->K;
  p.taps = d->R * d->S;
  for (int t = 0; t < p.taps; ++t) {
    p.tap_wt[t] = (short)t;
    p.tap_oh[t] = (short)((t / d->S) * d->dil);
    p.tap_ow[t] = (short)((t % d->S) * d->dil);
  }
  p.kchunks = ceil_div(d->C, BK);
  p.stride = d->stride;
  p.lower_h = p.lower_w = -d->pad;
  p.PQ = d->P * d->Q;
  p.Q = d->Q;
  p.brows_per_tap = d->K;
  p.out = y;
  p.ldo = d->ldy;
  p.out_dtype = y_dtype;
  p.beta = beta;
  p.bias = bias;
  p.stats = stats;
  p.stat_ticket = stat_ticket;
  if (sync && stats) {
    SEG_REQUIRE(stat_ticket != nullptr, "conv fwd: SyncBN needs a zeroed ticket word");
    SEG_REQUIRE(4 * d->K <= sync->n_max, "conv fwd: 2*K = %d fp64 statistics exceed the SyncBN buffer (%d floats)", 2 * d->K, sync->n_max);
    p.sync = *sync;
  }
  const int bn = pick_bn(d->K, y_dtype != SEG_DT_BF16);
  p.stat_rows = stat_rows_for(d->K);
  if (is_pointwise(d)) {
    p.x_im2col = 0;
    if (make_map_2d(&p.mapA, x, M, d->C, d->ldx, BM)) return 1;
  } else {
    p.x_im2col = 1;
    const int upper = d->pad - (d->R - 1) * d->dil;
    if (make_map_im2col(&p.mapA, x, d->N, d->H, d->W, d->C, d->ldx, -d->pad, -d->pad, upper, upper, d->stride, BM)) return 1;
  }
  if (make_map_2d(&p.mapB, w, (int64_t)p.taps * d->K, d->C, d->C, bn)) return 1;
  return launch_pp_bn<KIND_KK>(bn, p, stream);
}

static int floordiv(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }

int conv_dgrad(const seg_conv_desc* d, const void* dy, const void* w, void* dx, float beta, cudaStream_t stream) {
  SEG_REQUIRE(supported(d) && d->ldy % 8 == 0, "wgmma conv dgrad: unsupported shape (stride=%d K=%d ldy=%d)", d->stride,
              d->K, d->ldy);
  const int s = d->stride;
  const int bn = pick_bn(d->C, false);
  // One launch per parity class (py, px) of the input pixels; stride 1 has the single class (0, 0).
  for (int py = 0; py < s; ++py) {
    for (int px = 0; px < s; ++px) {
      const int Hs = (d->H - py + s - 1) / s, Ws = (d->W - px + s - 1) / s;
      if (Hs <= 0 || Ws <= 0) continue;
      TcParams p;
      memset(&p, 0, sizeof(p));
      // taps whose parity matches: y*1 + pad - r*dil must be a multiple of the stride; offset = that / stride
      int rh[8], oh[8], nh = 0, rw[8], ow[8], nw = 0;
      for (int r = 0; r < d->R; ++r) {
        const int num = py + d->pad - r * d->dil;
        if (((num % s) + s) % s == 0) { rh[nh] = r; oh[nh] = floordiv(num, s); ++nh; }
      }
      for (int q = 0; q < d->S; ++q) {
        const int num = px + d->pad - q * d->dil;
        if (((num % s) + s) % s == 0) { rw[nw] = q; ow[nw] = floordiv(num, s); ++nw; }
      }
      int min_oh = 0, min_ow = 0;
      for (int i = 0; i < nh; ++i) min_oh = (i == 0) ? oh[i] : min(min_oh, oh[i]);
      for (int i = 0; i < nw; ++i) min_ow = (i == 0) ? ow[i] : min(min_ow, ow[i]);
      p.taps = nh * nw;
      for (int i = 0; i < nh; ++i)
        for (int j = 0; j < nw; ++j) {
          const int t = i * nw + j;
          p.tap_wt[t] = (short)(rh[i] * d->S + rw[j]);
          p.tap_oh[t] = (short)(oh[i] - min_oh);
          p.tap_ow[t] = (short)(ow[j] - min_ow);
        }
      const int64_t M = (int64_t)d->N * Hs * Ws;
      SEG_REQUIRE(M < (1ll << 31), "M too large");
      p.M = (int)M;
      p.Ncols = d->C;
      p.kchunks = ceil_div(d->K, BK);
      p.stride = 1;
      p.lower_h = min_oh;
      p.lower_w = min_ow;
      p.PQ = Hs * Ws;
      p.Q = Ws;
      p.brows_per_tap = d->K;
      p.out = dx;
      p.ldo = d->ldx;
      p.out_dtype = SEG_DT_BF16;
      p.beta = beta;
      if (s > 1) {
        p.out_strided = 1;
        p.out_H = d->H;
        p.out_W = d->W;
        p.osy = p.osx = s;
        p.opy = py;
        p.opx = px;
      }
      p.stat_rows = BM;  // no statistics
      if (p.taps > 0) {
        const bool plain = (s == 1 && is_pointwise(d));
        if (plain) {
          p.x_im2col = 0;
          if (make_map_2d(&p.mapA, dy, M, d->K, d->ldy, BM)) return 1;
        } else {
          p.x_im2col = 1;
          // base positions per dimension must number Hs (Ws): box = [lower, dim + upper - 1]
          const int upper_h = Hs - d->P + min_oh, upper_w = Ws - d->Q + min_ow;
          if (make_map_im2col(&p.mapA, dy, d->N, d->P, d->Q, d->K, d->ldy, min_ow, min_oh, upper_w, upper_h, 1, BM)) return 1;
        }
        if (make_map_2d(&p.mapB, w, (int64_t)d->R * d->S * d->K, d->C, d->C, 64)) return 1;
      } else {
        if (beta == 1.f) continue;  // dx = 1 * dx + 0: the class keeps its values
        // no tap reaches this class: the kernel (num_iters == 0) writes 0 + beta * dx, i.e. zeros for beta = 0 and the
        // scaled old values otherwise; maps unused but must be valid objects
        if (make_map_2d(&p.mapA, w, (int64_t)d->R * d->S * d->K, d->C, d->C, BM)) return 1;
        if (make_map_2d(&p.mapB, w, (int64_t)d->R * d->S * d->K, d->C, d->C, 64)) return 1;
      }
      if (launch_pp_bn<KIND_KM>(bn, p, stream)) return 1;
    }
  }
  return 0;
}

// dW[i] += sum over splits s (in order) of ws[s][i]
__global__ void wgrad_split_reduce_kernel(const float* __restrict__ ws, int splits, int64_t n, float* __restrict__ dw) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float acc = ws[i];
    for (int s = 1; s < splits; ++s) acc += ws[(size_t)s * n + i];
    dw[i] += acc;
  }
}

// tile width and number of k-splits of the wgrad of `d` (one wave: tiles * splits <= resident CTAs, one per SM)
static void wgrad_plan(const seg_conv_desc* d, int& bn, int& splits, int& kblocks_per_split) {
  // 256-wide tiles for the 3x3 convs with C a multiple of 256; the 1x1s keep 128-wide tiles (twice as many tiles for the
  // one-wave split-K)
  const bool wide = d->R * d->S >= 9 && d->C >= 256 && d->C % 256 == 0;
  bn = (d->C <= 64) ? 64 : (wide ? 256 : 128);
  const int kblocks_total = (int)ceil_div64((int64_t)d->N * d->P * d->Q, BK);
  const int tiles = ceil_div(d->K, BM) * ceil_div(d->C, bn) * d->R * d->S;
  splits = max(1, num_sms() / tiles);
  splits = min(splits, kblocks_total);
  splits = min(splits, 1024);
  kblocks_per_split = ceil_div(kblocks_total, splits);
  // recounted so that every split owns at least one k-block: the split-order reduction reads every split's workspace slice,
  // and a split without k-blocks would leave its slice unwritten (conv_wgrad checks this)
  splits = ceil_div(kblocks_total, kblocks_per_split);
}

int64_t wgrad_workspace_floats(const seg_conv_desc* d) {
  if (!supported(d)) return 0;
  int bn, splits, kps;
  wgrad_plan(d, bn, splits, kps);
  return splits > 1 ? (int64_t)splits * d->R * d->S * d->K * d->C : 0;
}

int conv_wgrad(const seg_conv_desc* d, const void* dy, const void* x, float* dw, float* ws, cudaStream_t stream) {
  SEG_REQUIRE(supported(d) && d->ldy % 8 == 0, "wgmma conv wgrad: unsupported shape");
  TcParams p;
  memset(&p, 0, sizeof(p));
  const int64_t npix = (int64_t)d->N * d->P * d->Q;
  SEG_REQUIRE(npix < (1ll << 31), "too many pixels");
  p.M = d->K;
  p.Ncols = d->C;
  p.taps = d->R * d->S;
  for (int t = 0; t < p.taps; ++t) {
    p.tap_wt[t] = (short)t;
    p.tap_oh[t] = (short)((t / d->S) * d->dil);
    p.tap_ow[t] = (short)((t % d->S) * d->dil);
  }
  p.stride = d->stride;
  p.lower_h = p.lower_w = -d->pad;
  p.PQ = d->P * d->Q;
  p.Q = d->Q;
  p.dw = dw;
  p.dw_K = d->K;
  p.dw_C = d->C;
  p.kblocks_total = (int)ceil_div64(npix, BK);
  int bn, splits;
  wgrad_plan(d, bn, splits, p.kblocks_per_split);
  SEG_REQUIRE(splits == 1 || ws != nullptr, "wgmma conv wgrad: %d k-splits need the workspace (seg_conv2d_wgrad_workspace_floats)", splits);
  SEG_REQUIRE((int64_t)(splits - 1) * p.kblocks_per_split < p.kblocks_total, "wgmma conv wgrad: split %d has no k-blocks", splits - 1);
  if (splits > 1) p.ws = ws;
  if (make_map_2d(&p.mapA, dy, npix, d->K, d->ldy, 64)) return 1;
  if (is_pointwise(d)) {
    p.x_im2col = 0;
    if (make_map_2d(&p.mapB, x, npix, d->C, d->ldx, 64)) return 1;
  } else {
    p.x_im2col = 1;
    const int upper = d->pad - (d->R - 1) * d->dil;
    if (make_map_im2col(&p.mapB, x, d->N, d->H, d->W, d->C, d->ldx, -d->pad, -d->pad, upper, upper, d->stride, 64)) return 1;
  }
  SEG_REQUIRE((unsigned)(p.taps * splits) <= 65535u, "wgrad grid.z too large");
  dim3 grid((unsigned)ceil_div(d->K, BM), (unsigned)ceil_div(d->C, bn), (unsigned)(p.taps * splits));
  if (launch_wgrad_bn(bn, p, grid, stream)) return 1;
  if (splits == 1) return 0;
  const int64_t n = (int64_t)p.taps * d->K * d->C;
  wgrad_split_reduce_kernel<<<(unsigned)std::min<int64_t>(ceil_div64(n, 256), (int64_t)num_sms() * 8), 256, 0, stream>>>(ws, splits, n, dw);
  return check_launch("wgrad_split_reduce");
}

}  // namespace tc
}  // namespace seg
