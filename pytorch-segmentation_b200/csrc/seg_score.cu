// seg_score.cu — FCN8's frozen score upsamplers (models/fcn.py:57-97): ConvTranspose2d(C, C, k = 2s, stride s, padding 0) over
// a class map, computed only over a requested output window, with the skip branch's alpha * skip + bias added in the same
// pass.  Tensor cores through mma.sync.m16n8k16 (bf16 operands, fp32 accumulation).
//
// Forward.  Output row oy = y0 + i takes input rows qy = oy / s and qy - 1 with kernel rows oy % s and oy % s + s, so the
// output pixels of one parity class (oy % s, ox % s) = (ry, rx) share four taps: a dense GEMM [pixels] x [4 * CP] x [C].
// Data gradient.  dx[iy, ix] sums dy over the k x k window at (iy * s - y0, ix * s - x0): a GEMM [pixels] x [k*k * CP] x [C],
// the taps that fall outside the computed window contributing zero.
// CP = C rounded up to 16 (one k-step never straddles two taps).  The weight is packed once per call into mma.sync B-fragment
// order: packed[cls][kstep][ntile][lane] = the lane's two 32-bit registers, so a warp reads one n8 x k16 tile as 256
// contiguous bytes.  A fragments are read straight from the NHWC activations (two bf16 lanes per 32-bit load).
// Every output element is one thread's sum in a fixed order: no atomics, bit-identical reruns.
#include "seg_common.cuh"

namespace seg {
namespace {

constexpr int WARPS = 4;   // 128 threads
constexpr int MT = 2;      // m16 tiles per warp: 32 pixels
constexpr int NT = 4;      // n8 tiles per CTA: 32 output channels (grid.y covers the rest)
constexpr int MAX_C = 160;

__host__ __device__ inline int cpad16(int C) { return (C + 15) / 16 * 16; }
__host__ __device__ inline int ntiles(int C) { return (C + 31) / 32 * NT; }  // n8 tiles, padded to whole CTA column blocks

__device__ __forceinline__ void mma16816(float* c, const uint32_t* a, uint2 b) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b.x), "r"(b.y));
}

// channels ci, ci + 1 (ci even) of one NHWC row as a bf16x2 register; lanes >= C are never read and give 0
__device__ __forceinline__ uint32_t ld_pair(const unsigned short* row, int ci, int C) {
  if (row == nullptr || ci >= C) return 0u;
  if (ci + 1 < C) return __ldg(reinterpret_cast<const unsigned int*>(row + ci));
  return (uint32_t)__ldg(row + ci);
}

__device__ __forceinline__ unsigned short f2bf_bits(float f) {
  return __bfloat16_as_ushort(__float2bfloat16_rn(f));
}

// one bf16 element of the packed B operand: GEMM row kidx, column n, of parity class cls (forward) or of the data gradient
__device__ __forceinline__ float packed_value(const float* w, int C, int s, int bwd, int cls, int kidx, int n) {
  const int CP = cpad16(C), k = 2 * s;
  const int tap = kidx / CP, c = kidx % CP;
  int ci, co, ky, kx;
  if (!bwd) {  // rows (tap = 2 dy + dx, input channel), columns = output channels
    ci = c;
    co = n;
    ky = cls / s + s * (tap >> 1);
    kx = cls % s + s * (tap & 1);
  } else {     // rows (tap = ky * k + kx, output channel), columns = input channels
    co = c;
    ci = n;
    ky = tap / k;
    kx = tap % k;
  }
  if (ci >= C || co >= C) return 0.f;
  return w[(((int64_t)ci * C + co) * k + ky) * k + kx];  // ConvTranspose2d weight [in][out][k][k]
}

__global__ void score_pack_kernel(const float* __restrict__ w, uint2* __restrict__ out, int C, int s, int bwd) {
  const int KS = (bwd ? 4 * s * s : 4) * (cpad16(C) / 16);  // k-steps per class: four taps, or all k * k
  const int NTP = ntiles(C);
  const int classes = bwd ? 1 : s * s;
  const int64_t total = (int64_t)classes * KS * NTP * 32;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int lane = (int)(i % 32);
    int64_t t = i / 32;
    const int nt = (int)(t % NTP);
    t /= NTP;
    const int ks = (int)(t % KS);
    const int cls = (int)(t / KS);
    const int g = lane >> 2, q = lane & 3;
    const int n = nt * 8 + g, k0 = ks * 16 + 2 * q;
    const uint32_t r0 = (uint32_t)f2bf_bits(packed_value(w, C, s, bwd, cls, k0, n)) |
                        ((uint32_t)f2bf_bits(packed_value(w, C, s, bwd, cls, k0 + 1, n)) << 16);
    const uint32_t r1 = (uint32_t)f2bf_bits(packed_value(w, C, s, bwd, cls, k0 + 8, n)) |
                        ((uint32_t)f2bf_bits(packed_value(w, C, s, bwd, cls, k0 + 9, n)) << 16);
    out[i] = make_uint2(r0, r1);
  }
}

struct FwdArgs {
  const unsigned short* x;
  int ldx, N, h, w, C, s;
  const uint2* wp;
  void* y;
  int ldy, y_f32, y0, x0, Ho, Wo;
  const unsigned short* skip;
  int lds, Hs, Ws, sy0, sx0;
  float alpha;
  const float* bias;
};

__global__ void __launch_bounds__(WARPS * 32) score_fwd_kernel(const FwdArgs a) {
  const int s = a.s, cls = blockIdx.z, ry = cls / s, rx = cls % s;
  const int i0 = ((ry - a.y0) % s + s) % s, j0 = ((rx - a.x0) % s + s) % s;
  const int ny = i0 < a.Ho ? (a.Ho - i0 + s - 1) / s : 0, nx = j0 < a.Wo ? (a.Wo - j0 + s - 1) / s : 0;
  const int64_t M = (int64_t)a.N * ny * nx;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int64_t mbase = ((int64_t)blockIdx.x * WARPS + warp) * (MT * 16);
  if (mbase >= M) return;
  // this lane's four pixel rows (m-tile r / 2, rows g and g + 8): image, and input row / column of tap (0, 0); -1 = no pixel
  int rn[2 * MT], qy[2 * MT], qx[2 * MT];
#pragma unroll
  for (int r = 0; r < 2 * MT; ++r) {
    const int64_t m = mbase + (r >> 1) * 16 + (r & 1) * 8 + g;
    const int64_t mm = m < M ? m : 0;
    rn[r] = m < M ? (int)(mm / ((int64_t)ny * nx)) : -1;
    const int rem = (int)(mm % ((int64_t)ny * nx));
    qy[r] = (a.y0 + i0 + (rem / nx) * s) / s;
    qx[r] = (a.x0 + j0 + (rem % nx) * s) / s;
  }
  const int KC = cpad16(a.C) / 16, KS = 4 * KC, NTP = ntiles(a.C);
  float acc[MT][NT][4];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[mt][j][e] = 0.f;
  for (int tap = 0; tap < 4; ++tap) {
    const unsigned short* rp[2 * MT];
    bool any = false;
#pragma unroll
    for (int r = 0; r < 2 * MT; ++r) {
      const int iy = qy[r] - (tap >> 1), ix = qx[r] - (tap & 1);
      const bool ok = rn[r] >= 0 && iy >= 0 && iy < a.h && ix >= 0 && ix < a.w;
      rp[r] = ok ? a.x + (((int64_t)rn[r] * a.h + iy) * a.w + ix) * a.ldx : nullptr;
      any |= ok;
    }
    if (!__any_sync(0xffffffffu, any)) continue;  // warp-uniform: the whole tap is outside the input
    const uint2* bp = a.wp + (((int64_t)cls * KS + tap * KC) * NTP + blockIdx.y * NT) * 32 + lane;
    for (int kc = 0; kc < KC; ++kc, bp += (int64_t)NTP * 32) {
      const int ci = kc * 16 + 2 * q;
      uint32_t af[MT][4];
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        af[mt][0] = ld_pair(rp[2 * mt], ci, a.C);
        af[mt][1] = ld_pair(rp[2 * mt + 1], ci, a.C);
        af[mt][2] = ld_pair(rp[2 * mt], ci + 8, a.C);
        af[mt][3] = ld_pair(rp[2 * mt + 1], ci + 8, a.C);
      }
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        const uint2 b = __ldg(bp + j * 32);
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) mma16816(acc[mt][j], af[mt], b);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 2 * MT; ++r) {
    if (rn[r] < 0) continue;
    const int ri = qy[r] * s + ry - a.y0, rj = qx[r] * s + rx - a.x0;  // window row / column
    const int64_t orow = ((int64_t)rn[r] * a.Ho + ri) * a.Wo + rj;
    const int64_t srow = a.skip ? ((int64_t)rn[r] * a.Hs + a.sy0 + ri) * a.Ws + a.sx0 + rj : 0;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = (blockIdx.y * NT + j) * 8 + 2 * q + e;
        if (c >= a.C) continue;
        float v = acc[r >> 1][j][(r & 1) * 2 + e];
        if (a.skip) {
          // adj_poolN(alpha * pool) = alpha * (W pool) + b, cropped, then + the upsampled scores (fcn.py:86-94)
          float sk = a.alpha * __uint_as_float((uint32_t)a.skip[srow * a.lds + c] << 16);
          if (a.bias) sk += a.bias[c];
          v = sk + v;
        }
        if (a.y_f32) reinterpret_cast<float*>(a.y)[orow * a.ldy + c] = v;
        else reinterpret_cast<unsigned short*>(a.y)[orow * a.ldy + c] = f2bf_bits(v);
      }
    }
  }
}

struct BwdArgs {
  const unsigned short* dy;
  int lddy, N, h, w, C, s;
  const uint2* wp;
  unsigned short* dx;
  int ldx, y0, x0, Ho, Wo;
};

__global__ void __launch_bounds__(WARPS * 32) score_bwd_kernel(const BwdArgs a) {
  const int s = a.s, k = 2 * s;
  const int64_t M = (int64_t)a.N * a.h * a.w;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int64_t mbase = ((int64_t)blockIdx.x * WARPS + warp) * (MT * 16);
  if (mbase >= M) return;
  int rn[2 * MT], oy0[2 * MT], ox0[2 * MT];
  bool rv[2 * MT];
#pragma unroll
  for (int r = 0; r < 2 * MT; ++r) {
    const int64_t m = mbase + (r >> 1) * 16 + (r & 1) * 8 + g;
    rv[r] = m < M;
    const int64_t mm = rv[r] ? m : 0;
    rn[r] = (int)(mm / ((int64_t)a.h * a.w));
    const int rem = (int)(mm % ((int64_t)a.h * a.w));
    oy0[r] = (rem / a.w) * s - a.y0;  // window row of kernel row 0
    ox0[r] = (rem % a.w) * s - a.x0;
  }
  const int KC = cpad16(a.C) / 16, NTP = ntiles(a.C);
  float acc[MT][NT][4];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[mt][j][e] = 0.f;
  for (int tap = 0; tap < k * k; ++tap) {
    const int ky = tap / k, kx = tap % k;
    const unsigned short* rp[2 * MT];
    bool any = false;
#pragma unroll
    for (int r = 0; r < 2 * MT; ++r) {
      const int oy = oy0[r] + ky, ox = ox0[r] + kx;
      const bool ok = rv[r] && oy >= 0 && oy < a.Ho && ox >= 0 && ox < a.Wo;
      rp[r] = ok ? a.dy + (((int64_t)rn[r] * a.Ho + oy) * a.Wo + ox) * a.lddy : nullptr;
      any |= ok;
    }
    if (!__any_sync(0xffffffffu, any)) continue;  // warp-uniform: the tap lies outside the window for all 32 pixels
    const uint2* bp = a.wp + ((int64_t)tap * KC * NTP + blockIdx.y * NT) * 32 + lane;
    for (int kc = 0; kc < KC; ++kc, bp += (int64_t)NTP * 32) {
      const int co = kc * 16 + 2 * q;
      uint32_t af[MT][4];
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        af[mt][0] = ld_pair(rp[2 * mt], co, a.C);
        af[mt][1] = ld_pair(rp[2 * mt + 1], co, a.C);
        af[mt][2] = ld_pair(rp[2 * mt], co + 8, a.C);
        af[mt][3] = ld_pair(rp[2 * mt + 1], co + 8, a.C);
      }
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        const uint2 b = __ldg(bp + j * 32);
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) mma16816(acc[mt][j], af[mt], b);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 2 * MT; ++r) {
    if (!rv[r]) continue;
    const int64_t row = mbase + (r >> 1) * 16 + (r & 1) * 8 + g;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = (blockIdx.y * NT + j) * 8 + 2 * q + e;
        if (c < a.C) a.dx[row * a.ldx + c] = f2bf_bits(acc[r >> 1][j][(r & 1) * 2 + e]);
      }
    }
  }
}

__global__ void score_skip_bwd_kernel(const unsigned short* __restrict__ dy, int lddy, int Ho, int Wo, unsigned short* __restrict__ ds,
                                      int ldd, int N, int Hs, int Ws, int C, int sy0, int sx0, float alpha) {
  const int64_t total = (int64_t)N * Hs * Ws * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    int64_t t = i / C;
    const int b = (int)(t % Ws);
    t /= Ws;
    const int r = (int)(t % Hs);
    const int n = (int)(t / Hs);
    const int oy = r - sy0, ox = b - sx0;
    float v = 0.f;
    if (oy >= 0 && oy < Ho && ox >= 0 && ox < Wo)
      v = alpha * __uint_as_float((uint32_t)dy[(((int64_t)n * Ho + oy) * Wo + ox) * lddy + c] << 16);
    ds[(((int64_t)n * Hs + r) * Ws + b) * ldd + c] = f2bf_bits(v);
  }
}

int grid_cap(int64_t blocks) {
  const int64_t cap = (int64_t)num_sms() * 8;
  return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

bool al4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) == 0; }

int check_common(const char* what, int N, int h, int w, int C, int s, int y0, int x0, int Ho, int Wo) {
  SEG_REQUIRE(C >= 1 && C <= MAX_C, "%s: C = %d classes; the score kernels take 1 <= C <= %d", what, C, MAX_C);
  SEG_REQUIRE(s >= 1 && s <= 8, "%s: stride %d not in 1..8 (kernel 2s)", what, s);
  SEG_REQUIRE(N >= 1 && h >= 1 && w >= 1 && Ho >= 1 && Wo >= 1, "%s: empty input or window", what);
  SEG_REQUIRE(y0 >= 0 && x0 >= 0 && y0 + Ho <= (h + 1) * s && x0 + Wo <= (w + 1) * s,
              "%s: window [%d, %d) x [%d, %d) outside the %d x %d output", what, y0, y0 + Ho, x0, x0 + Wo, (h + 1) * s, (w + 1) * s);
  return 0;
}

}  // namespace
}  // namespace seg

using namespace seg;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int64_t seg_score_packed_elems(int C, int s) {
  if (C < 1 || C > MAX_C || s < 1 || s > 8) return -1;
  return (int64_t)4 * s * s * (cpad16(C) / 16) * ntiles(C) * 32 * 4;
}

int seg_score_pack(const float* w, void* packed, int C, int s, int bwd, void* stream) {
  SEG_REQUIRE(C >= 1 && C <= MAX_C && s >= 1 && s <= 8, "score_pack: C = %d, s = %d (need 1 <= C <= %d, 1 <= s <= 8)", C, s, MAX_C);
  SEG_REQUIRE(w && packed && (reinterpret_cast<uintptr_t>(packed) & 7) == 0, "score_pack: null or misaligned operand");
  const int64_t n = seg_score_packed_elems(C, s) / 4;
  score_pack_kernel<<<grid_cap(ceil_div64(n, 256)), 256, 0, ST(stream)>>>(w, reinterpret_cast<uint2*>(packed), C, s, bwd ? 1 : 0);
  return check_launch("score_pack");
}

int seg_score_upsample_fwd(const void* x, int ldx, int N, int h, int w, int C, int s, const void* packed, void* y, int ldy,
                           int y_dtype, int y0, int x0, int Ho, int Wo, const void* skip, int lds, int Hs, int Ws, int sy0, int sx0,
                           float alpha, const float* bias, void* stream) {
  if (check_common("score_upsample_fwd", N, h, w, C, s, y0, x0, Ho, Wo)) return 1;
  SEG_REQUIRE(x && packed && y && al4(x) && ldx >= C && ldx % 2 == 0 && ldy >= C && (reinterpret_cast<uintptr_t>(packed) & 7) == 0,
              "score_upsample_fwd: operands must be non-null, bf16 pitches even and >= C, bases 4-byte aligned");
  SEG_REQUIRE(y_dtype == SEG_DT_BF16 || y_dtype == SEG_DT_F32, "score_upsample_fwd: bad output dtype %d", y_dtype);
  if (skip) {
    SEG_REQUIRE(al4(skip) && lds >= C && lds % 2 == 0, "score_upsample_fwd: skip pitch / alignment");
    SEG_REQUIRE(sy0 >= 0 && sx0 >= 0 && sy0 + Ho <= Hs && sx0 + Wo <= Ws, "score_upsample_fwd: skip window [%d, %d) x [%d, %d) "
                "outside the %d x %d skip map", sy0, sy0 + Ho, sx0, sx0 + Wo, Hs, Ws);
  }
  FwdArgs a;
  a.x = static_cast<const unsigned short*>(x);
  a.ldx = ldx; a.N = N; a.h = h; a.w = w; a.C = C; a.s = s;
  a.wp = static_cast<const uint2*>(packed);
  a.y = y; a.ldy = ldy; a.y_f32 = y_dtype == SEG_DT_F32; a.y0 = y0; a.x0 = x0; a.Ho = Ho; a.Wo = Wo;
  a.skip = static_cast<const unsigned short*>(skip);
  a.lds = lds; a.Hs = Hs; a.Ws = Ws; a.sy0 = sy0; a.sx0 = sx0; a.alpha = alpha; a.bias = bias;
  const int64_t maxM = (int64_t)N * ceil_div(Ho, s) * ceil_div(Wo, s);  // the largest parity class
  const int64_t bx = ceil_div64(maxM, WARPS * MT * 16);
  SEG_REQUIRE(bx < (1ll << 31), "score_upsample_fwd: too many pixels");
  dim3 grid((unsigned)bx, (unsigned)(ntiles(C) / NT), (unsigned)(s * s));
  score_fwd_kernel<<<grid, WARPS * 32, 0, ST(stream)>>>(a);
  return check_launch("score_upsample_fwd");
}

int seg_score_upsample_bwd(const void* dy, int lddy, int N, int h, int w, int C, int s, const void* packed_bwd, void* dx, int ldx,
                           int y0, int x0, int Ho, int Wo, void* stream) {
  if (check_common("score_upsample_bwd", N, h, w, C, s, y0, x0, Ho, Wo)) return 1;
  SEG_REQUIRE(dy && packed_bwd && dx && al4(dy) && lddy >= C && lddy % 2 == 0 && ldx >= C &&
                  (reinterpret_cast<uintptr_t>(packed_bwd) & 7) == 0,
              "score_upsample_bwd: operands must be non-null, dy's pitch even and >= C, bases aligned");
  BwdArgs a;
  a.dy = static_cast<const unsigned short*>(dy);
  a.lddy = lddy; a.N = N; a.h = h; a.w = w; a.C = C; a.s = s;
  a.wp = static_cast<const uint2*>(packed_bwd);
  a.dx = static_cast<unsigned short*>(dx);
  a.ldx = ldx; a.y0 = y0; a.x0 = x0; a.Ho = Ho; a.Wo = Wo;
  const int64_t bx = ceil_div64((int64_t)N * h * w, WARPS * MT * 16);
  SEG_REQUIRE(bx < (1ll << 31), "score_upsample_bwd: too many pixels");
  dim3 grid((unsigned)bx, (unsigned)(ntiles(C) / NT), 1);
  score_bwd_kernel<<<grid, WARPS * 32, 0, ST(stream)>>>(a);
  return check_launch("score_upsample_bwd");
}

int seg_score_skip_bwd(const void* dy, int lddy, int Ho, int Wo, void* dskip, int ldd, int N, int Hs, int Ws, int C, int sy0,
                       int sx0, float alpha, void* stream) {
  SEG_REQUIRE(dy && dskip && N >= 1 && Hs >= 1 && Ws >= 1 && C >= 1 && lddy >= C && ldd >= C, "score_skip_bwd: bad operands");
  SEG_REQUIRE(sy0 >= 0 && sx0 >= 0 && sy0 + Ho <= Hs && sx0 + Wo <= Ws, "score_skip_bwd: window outside the skip map");
  score_skip_bwd_kernel<<<grid_cap(ceil_div64((int64_t)N * Hs * Ws * C, 256)), 256, 0, ST(stream)>>>(
      static_cast<const unsigned short*>(dy), lddy, Ho, Wo, static_cast<unsigned short*>(dskip), ldd, N, Hs, Ws, C, sy0, sx0, alpha);
  return check_launch("score_skip_bwd");
}

}  // extern "C"
