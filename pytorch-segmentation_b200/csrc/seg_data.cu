// seg_data.cu — the two callers either side of the train step that SURVEY.md §8(f) ranks next:
//   * the tail of the input pipeline (base/base_dataset.py:88-136: pad -> crop -> horizontal flip -> ToTensor ->
//     Normalize) on uint8 images that crossed PCIe as bytes (4x fewer than the reference's fp32 batches), and
//   * the resampling / accumulation arithmetic of inference.py:26-79 (multi-scale + flip, sliding window) on fp32 NCHW
//     score maps that never leave the device.
// All kernels are HBM streaming kernels: one thread per output element along x (coalesced fp32 stores), grid-stride.
#include "seg_common.cuh"

namespace seg {

static inline int grid_for(int64_t work_items, int threads, int max_blocks_per_sm = 8) {
  int64_t b = ceil_div64(work_items, threads);
  int64_t cap = (int64_t)num_sms() * max_blocks_per_sm;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

// ------------------------------------------------------------------ pad + crop + flip + ToTensor + Normalize
// out[b][c][y][x] = ((float)u8 / 255 - mean[c]) / std[c], u8 = pixel (y + y0, xs + x0) of image b (xs = x, or
// crop_w-1-x when the image is flipped AFTER cropping as base_dataset.py:119-123 does); positions outside the h x w image
// are the zero padding of cv2.copyMakeBorder(value=0) (base_dataset.py:93-105) — for the label too.
// Division (not reciprocal multiplication) in fp32, the order torchvision's to_tensor / normalize use: bit-exact.
struct AugParams {
  float mean[3];
  float stdv[3];
};

// Label maps (SEG_AUG_LABEL_MAP in a record's lbl_bytes): a raw uint8 label map of n pixels is followed, at the next
// 4-byte boundary, by 256 int32 entries, and the label read at index k is map[raw[k]] (a dataset's id -> train-id table,
// cityscapes.py:53-54, applied where the reference applies it: in _load_data, before any resize, rotation or padding).
// Fill values (the zero padding, the rotation's constant border) are post-map values and never go through the map.
// LabelMap = false instantiates exactly the reads the kernels had before label maps existed.
template <bool LabelMap>
__device__ __forceinline__ const int32_t* label_map_of(const uint8_t* lbl, int lbl_bytes, int64_t n) {
  if constexpr (LabelMap)
    return (lbl != nullptr && (lbl_bytes & SEG_AUG_LABEL_MAP)) ? reinterpret_cast<const int32_t*>(lbl + (n + 3) / 4 * 4) : nullptr;
  return nullptr;
}
template <bool LabelMap>
__device__ __forceinline__ int read_label(const uint8_t* lbl, const int32_t* lmap, int lbl_bytes, int64_t k) {
  if constexpr (LabelMap)
    if (lmap != nullptr) return __ldg(lmap + lbl[k]);
  return lbl_bytes == 1 ? (int)lbl[k] : reinterpret_cast<const int32_t*>(lbl)[k];
}
template <bool LabelMap>
__global__ void __launch_bounds__(256) augment_u8_kernel(const uint8_t* __restrict__ arena, const seg_aug_entry* __restrict__ table,
                                                         int crop_h, int crop_w, AugParams prm, float* __restrict__ out,
                                                         int64_t* __restrict__ labels) {
  // A uint8 channel has 256 possible values: the block evaluates the exact fp32 formula once per (channel, value) into
  // shared memory and every pixel becomes three table look-ups.  (First version: six IEEE divisions per pixel — ncu showed
  // the kernel instruction-bound, 220 instructions per pixel, 0.37 of the HBM roofline.)
  __shared__ float lut[3][256];
  for (int t = threadIdx.x; t < 768; t += blockDim.x) {
    const int c = t >> 8, v = t & 255;
    lut[c][v] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)v, 255.f), prm.mean[c]), prm.stdv[c]);
  }
  __syncthreads();
  const int b = blockIdx.y;
  const seg_aug_entry e = table[b];
  const uint8_t* img = arena + e.img_off;
  const uint8_t* lbl = (e.lbl_off >= 0 && labels != nullptr) ? arena + e.lbl_off : nullptr;
  const int32_t* lmap = label_map_of<LabelMap>(lbl, e.lbl_bytes, (int64_t)e.h * e.w);
  const int plane = crop_h * crop_w;  // < 2^31 (checked on the host)
  float* o = out + (int64_t)b * 3 * plane;
  int64_t* lo = labels != nullptr ? labels + (int64_t)b * plane : nullptr;
  // four pixels per thread and iteration, all loads issued before the stores: 4x the bytes in flight
  constexpr int U = 4;
  const int stride = gridDim.x * blockDim.x;
  for (int i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < plane; i0 += stride * U) {
    unsigned r[U], g[U], bl[U];
    int lab[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * stride;
      r[u] = g[u] = bl[u] = 0;
      lab[u] = 0;
      if (i < plane) {
        const int y = i / crop_w, x = i - y * crop_w;
        const int xs = e.flip ? crop_w - 1 - x : x;
        const int sy = y + e.y0, sx = xs + e.x0;
        if (sy < e.h && sx < e.w) {
          const int64_t k = (int64_t)sy * e.w + sx;
          const uint8_t* p = img + k * 3;
          r[u] = p[0];
          g[u] = p[1];
          bl[u] = p[2];
          if (lbl != nullptr) lab[u] = read_label<LabelMap>(lbl, lmap, e.lbl_bytes, k);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * stride;
      if (i < plane) {
        o[i] = lut[0][r[u]];
        o[plane + i] = lut[1][g[u]];
        o[2 * (int64_t)plane + i] = lut[2][bl[u]];
        if (lo != nullptr) lo[i] = (int64_t)lab[u];
      }
    }
  }
}

// ------------------------------------------------------------------ random-scale resize fused in front of the tail
// base_dataset.py:66-75 resizes the sample (cv2.resize: INTER_LINEAR on the float32 image, INTER_NEAREST on the label)
// before the pad / crop / flip / np.uint8 / ToTensor / Normalize tail.  Here the RAW uint8 sample crosses PCIe and each
// output pixel of the crop interpolates its value straight from the raw image: no resized intermediate exists.
// Arithmetic = OpenCV's own float path (modules/imgproc/src/resize.cpp, resizeGeneric_ / HResizeLinear / VResizeLinear):
//   f = (float)((d + 0.5) * scale - 0.5) with scale = 1 / (dst / src) in float64;  s = floor(f);  f -= s;
//   x: s < 0 -> (0, f = 0);  s >= src-1 -> (src-1, f = 0);      y: coefficient kept, ROW indices clipped to [0, src-1]
//   H = S[s]*(1-fx) + S[s+1]*fx   (fp32, no fma);   V = H0*(1-fy) + H1*fy   (fp32, no fma);   u8 = (uint8)V  (np.uint8 truncates)
//   label: src index = min(floor(d * scale), src-1)
// (opencv-python wheels route float32 resize through Intel IPP, whose closed-source arithmetic differs from the above by
// <= 3e-3 before the uint8 truncation: against the reference AS RUN the images agree except ~0.1 % of the pixels by one
// level; against OpenCV's own code path — cv2.ipp.setUseIPP(False) — and the oracle restatement they are bit-exact.)
__device__ __forceinline__ void cv_linear_coord(int d, double scale, int src, bool clamp, int& s, float& f) {
  const float fv = (float)__dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5);
  const float fl = floorf(fv);
  s = (int)fl;
  f = __fsub_rn(fv, fl);
  if (clamp) {
    if (s < 0) {
      s = 0;
      f = 0.f;
    }
    if (s >= src - 1) {
      s = src - 1;
      f = 0.f;
    }
  }
}

// PilLabels = false: the training tail's label rule above (cv2.resize INTER_NEAREST).
// PilLabels = true: the validation tail's (base_dataset.py:40-61), which resizes the label with PIL's Image.resize(NEAREST).
// Pillow walks the destination with a float64 source coordinate that it ACCUMULATES (xo = a/2, then xo += a per pixel,
// a = src / dst; Geometry.c ImagingScaleAffine) and truncates, so the index is not a closed-form function of d: for about
// half of the size pairs some index differs from floor((d + 0.5) * a).  The host runs the same additions and appends the
// two int32 index tables (x: w entries, then y: h entries) to the label map in the arena, 4-byte aligned; the kernel looks
// them up.  The image arithmetic is the same in both instantiations.
template <bool PilLabels, bool LabelMap>
__global__ void __launch_bounds__(256) augment_scale_u8_kernel(const uint8_t* __restrict__ arena,
                                                               const seg_aug_scale_entry* __restrict__ table, int crop_h, int crop_w,
                                                               AugParams prm, float* __restrict__ out, int64_t* __restrict__ labels) {
  __shared__ float lut[3][256];
  for (int t = threadIdx.x; t < 768; t += blockDim.x) {
    const int c = t >> 8, v = t & 255;
    lut[c][v] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)v, 255.f), prm.mean[c]), prm.stdv[c]);
  }
  __syncthreads();
  const int b = blockIdx.y;
  const seg_aug_scale_entry e = table[b];
  const uint8_t* img = arena + e.img_off;
  const uint8_t* lbl = (e.lbl_off >= 0 && labels != nullptr) ? arena + e.lbl_off : nullptr;
  const int32_t* lmap = label_map_of<LabelMap>(lbl, e.lbl_bytes, (int64_t)e.src_h * e.src_w);
  const int plane = crop_h * crop_w;
  float* o = out + (int64_t)b * 3 * plane;
  int64_t* lo = labels != nullptr ? labels + (int64_t)b * plane : nullptr;
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < plane; i += stride) {
    const int y = i / crop_w, x = i - y * crop_w;
    const int xs = e.flip ? crop_w - 1 - x : x;
    const int dy = y + e.y0, dx = xs + e.x0;  // position in the RESIZED (h x w) image; outside = zero padding
    unsigned r = 0, g = 0, bl = 0;
    int lab = 0;
    if (dy < e.h && dx < e.w) {
      int sx, sy;
      float fx, fy;
      cv_linear_coord(dx, e.scale_x, e.src_w, true, sx, fx);
      cv_linear_coord(dy, e.scale_y, e.src_h, false, sy, fy);
      const int sx1 = sx + 1 < e.src_w ? sx + 1 : e.src_w - 1;
      const int y0c = min(max(sy, 0), e.src_h - 1), y1c = min(max(sy + 1, 0), e.src_h - 1);
      const float ax0 = __fsub_rn(1.f, fx), ay0 = __fsub_rn(1.f, fy);
      const uint8_t* r0 = img + (int64_t)y0c * e.src_w * 3;
      const uint8_t* r1 = img + (int64_t)y1c * e.src_w * 3;
      unsigned res[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float h0 = __fadd_rn(__fmul_rn((float)r0[sx * 3 + c], ax0), __fmul_rn((float)r0[sx1 * 3 + c], fx));
        const float h1 = __fadd_rn(__fmul_rn((float)r1[sx * 3 + c], ax0), __fmul_rn((float)r1[sx1 * 3 + c], fx));
        const float v = __fadd_rn(__fmul_rn(h0, ay0), __fmul_rn(h1, fy));
        res[c] = (unsigned)v;  // np.uint8(float): truncation; v is a convex combination of [0, 255] values
        if (res[c] > 255u) res[c] = 255u;
      }
      r = res[0];
      g = res[1];
      bl = res[2];
      if (lbl != nullptr) {
        int lx, ly;
        if constexpr (PilLabels) {
          // the index tables follow the label map, and its 256-entry id table when there is one
          const int32_t* tab = (LabelMap && lmap != nullptr) ? lmap + 256
                                                             : reinterpret_cast<const int32_t*>(lbl + ((int64_t)e.src_h * e.src_w * e.lbl_bytes + 3) / 4 * 4);
          lx = tab[dx];
          ly = tab[e.w + dy];
        } else {
          lx = (int)floor(__dmul_rn((double)dx, e.scale_x));
          ly = (int)floor(__dmul_rn((double)dy, e.scale_y));
          lx = lx < e.src_w - 1 ? lx : e.src_w - 1;
          ly = ly < e.src_h - 1 ? ly : e.src_h - 1;
        }
        const int64_t k = (int64_t)ly * e.src_w + lx;
        lab = read_label<LabelMap>(lbl, lmap, e.lbl_bytes, k);
      }
    }
    o[i] = lut[0][r];
    o[plane + i] = lut[1][g];
    o[2 * (int64_t)plane + i] = lut[2][bl];
    if (lo != nullptr) lo[i] = (int64_t)lab;
  }
}

// ------------------------------------------------------------------ scale + ROTATE + tail
// base_dataset.py:77-83 rotates the resized float image (cv2.warpAffine INTER_LINEAR) and label (INTER_NEAREST) about the
// centre by a drawn angle, constant-0 border.  OpenCV's walk, restated bit-exactly in oracle/data.py::cv_warp_affine: the
// inverse matrix (float64, from the host) gives fixed-point source coordinates with 10 fractional bits,
//   X = rint((A12*y + b1) * 1024) + delta + rint(A11*x * 1024),  Y likewise,   delta = 16 (linear) / 512 (nearest);
// INTER_LINEAR keeps 5 fractional bits (a 1/32-pixel grid) and blends the four taps with float32 weight products; taps
// outside the resized image are 0.  Each tap of the RESIZED image is itself the cv2.resize interpolation of the raw image
// (augment_scale_u8_kernel's arithmetic, NOT truncated: the rotation consumes the float image), so an output pixel costs up
// to 16 raw taps and no intermediate image exists.  Reached through DeviceBatcher.stage_full.
__device__ __forceinline__ void resized_pixel_f32(const uint8_t* __restrict__ img, const seg_aug_full_entry& e, int ry, int rx, float* out3) {
  if (ry < 0 || ry >= e.h || rx < 0 || rx >= e.w) {
    out3[0] = out3[1] = out3[2] = 0.f;
    return;
  }
  int sx, sy;
  float fx, fy;
  cv_linear_coord(rx, e.scale_x, e.src_w, true, sx, fx);
  cv_linear_coord(ry, e.scale_y, e.src_h, false, sy, fy);
  const int sx1 = sx + 1 < e.src_w ? sx + 1 : e.src_w - 1;
  const int y0c = min(max(sy, 0), e.src_h - 1), y1c = min(max(sy + 1, 0), e.src_h - 1);
  const float ax0 = __fsub_rn(1.f, fx), ay0 = __fsub_rn(1.f, fy);
  const uint8_t* r0 = img + (int64_t)y0c * e.src_w * 3;
  const uint8_t* r1 = img + (int64_t)y1c * e.src_w * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float h0 = __fadd_rn(__fmul_rn((float)r0[sx * 3 + c], ax0), __fmul_rn((float)r0[sx1 * 3 + c], fx));
    const float h1 = __fadd_rn(__fmul_rn((float)r1[sx * 3 + c], ax0), __fmul_rn((float)r1[sx1 * 3 + c], fx));
    out3[c] = __fadd_rn(__fmul_rn(h0, ay0), __fmul_rn(h1, fy));
  }
}

template <bool LabelMap>
__device__ __forceinline__ int resized_label(const uint8_t* __restrict__ lbl, const int32_t* lmap, const seg_aug_full_entry& e, int ry,
                                             int rx) {
  if (ry < 0 || ry >= e.h || rx < 0 || rx >= e.w) return 0;
  int lx = (int)floor(__dmul_rn((double)rx, e.scale_x)), ly = (int)floor(__dmul_rn((double)ry, e.scale_y));
  lx = lx < e.src_w - 1 ? lx : e.src_w - 1;
  ly = ly < e.src_h - 1 ? ly : e.src_h - 1;
  const int64_t k = (int64_t)ly * e.src_w + lx;
  return read_label<LabelMap>(lbl, lmap, e.lbl_bytes, k);
}

// INTER_NEAREST uses delta = AB_SCALE / 2 on the same rounded row / column terms
__device__ __forceinline__ long long rowX_nearest_fix(long long row_term, long long col_term) { return row_term + 512 + col_term; }

// Fixed-point source coordinates in the resized image of rotated pixel (dy, dx): the two rounded terms are added as
// integers, as OpenCV does.
struct RotCoords {
  long long colX, colY, rowX, rowY;
};
__device__ __forceinline__ RotCoords rot_coords(const seg_aug_full_entry& e, int dy, int dx) {
  RotCoords q;
  q.colX = __double2ll_rn(__dmul_rn(__dmul_rn(e.a11, (double)dx), 1024.0));
  q.colY = __double2ll_rn(__dmul_rn(__dmul_rn(e.a21, (double)dx), 1024.0));
  q.rowX = __double2ll_rn(__dmul_rn(__dadd_rn(__dmul_rn(e.a12, (double)dy), e.b1), 1024.0));
  q.rowY = __double2ll_rn(__dmul_rn(__dadd_rn(__dmul_rn(e.a22, (double)dy), e.b2), 1024.0));
  return q;
}

// The float (pre-np.uint8) value of rotated pixel (dy, dx), inside the h x w image: INTER_LINEAR over four resized taps.
__device__ __forceinline__ void rotated_pixel_f32(const uint8_t* __restrict__ img, const seg_aug_full_entry& e, const RotCoords& q,
                                                  float* v3) {
  const long long X = q.rowX + 16 + q.colX, Y = q.rowY + 16 + q.colY;  // delta = AB_SCALE / INTER_TAB_SIZE / 2
  const long long Xf = X >> 5, Yf = Y >> 5;                            // 5 fractional bits left
  const int xi = (int)(Xf >> 5), yi = (int)(Yf >> 5);
  const float fx = __fdiv_rn((float)(int)(Xf & 31), 32.f), fy = __fdiv_rn((float)(int)(Yf & 31), 32.f);
  const float one_fx = __fsub_rn(1.f, fx), one_fy = __fsub_rn(1.f, fy);
  const float w00 = __fmul_rn(one_fy, one_fx), w01 = __fmul_rn(one_fy, fx), w10 = __fmul_rn(fy, one_fx), w11 = __fmul_rn(fy, fx);
  float p00[3], p01[3], p10[3], p11[3];
  resized_pixel_f32(img, e, yi, xi, p00);
  resized_pixel_f32(img, e, yi, xi + 1, p01);
  resized_pixel_f32(img, e, yi + 1, xi, p10);
  resized_pixel_f32(img, e, yi + 1, xi + 1, p11);
#pragma unroll
  for (int c = 0; c < 3; ++c)
    v3[c] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p00[c], w00), __fmul_rn(p01[c], w01)), __fmul_rn(p10[c], w10)), __fmul_rn(p11[c], w11));
}

__device__ __forceinline__ unsigned trunc_u8(float v) {
  unsigned r = v > 0.f ? (unsigned)v : 0u;  // np.uint8(float) truncates
  return r > 255u ? 255u : r;
}

template <bool LabelMap>
__device__ __forceinline__ int rotated_label(const uint8_t* __restrict__ lbl, const int32_t* lmap, const seg_aug_full_entry& e,
                                             const RotCoords& q) {
  const long long X = rowX_nearest_fix(q.rowX, q.colX), Y = rowX_nearest_fix(q.rowY, q.colY);
  return resized_label<LabelMap>(lbl, lmap, e, (int)(Y >> 10), (int)(X >> 10));
}

template <bool LabelMap>
__global__ void __launch_bounds__(256) augment_full_u8_kernel(const uint8_t* __restrict__ arena, const seg_aug_full_entry* __restrict__ table,
                                                              int crop_h, int crop_w, AugParams prm, float* __restrict__ out,
                                                              int64_t* __restrict__ labels) {
  __shared__ float lut[3][256];
  for (int t = threadIdx.x; t < 768; t += blockDim.x) {
    const int c = t >> 8, v = t & 255;
    lut[c][v] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)v, 255.f), prm.mean[c]), prm.stdv[c]);
  }
  __syncthreads();
  const int b = blockIdx.y;
  const seg_aug_full_entry e = table[b];
  const uint8_t* img = arena + e.img_off;
  const uint8_t* lbl = (e.lbl_off >= 0 && labels != nullptr) ? arena + e.lbl_off : nullptr;
  const int32_t* lmap = label_map_of<LabelMap>(lbl, e.lbl_bytes, (int64_t)e.src_h * e.src_w);
  const int plane = crop_h * crop_w;
  float* o = out + (int64_t)b * 3 * plane;
  int64_t* lo = labels != nullptr ? labels + (int64_t)b * plane : nullptr;
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < plane; i += stride) {
    const int y = i / crop_w, x = i - y * crop_w;
    const int xs = e.flip ? crop_w - 1 - x : x;
    const int dy = y + e.y0, dx = xs + e.x0;  // position in the rotated h x w image; outside = zero padding
    unsigned r = 0, g = 0, bl = 0;
    int lab = 0;
    if (dy < e.h && dx < e.w) {
      const RotCoords q = rot_coords(e, dy, dx);
      float v[3];
      rotated_pixel_f32(img, e, q, v);
      r = trunc_u8(v[0]);
      g = trunc_u8(v[1]);
      bl = trunc_u8(v[2]);
      if (lbl != nullptr) lab = rotated_label<LabelMap>(lbl, lmap, e, q);
    }
    o[i] = lut[0][r];
    o[plane + i] = lut[1][g];
    o[2 * (int64_t)plane + i] = lut[2][bl];
    if (lo != nullptr) lo[i] = (int64_t)lab;
  }
}

// ------------------------------------------------------------------ scale + rotate + tail + GAUSSIAN BLUR
// base_dataset.py:114-119 blurs the float32 crop AFTER the flip, BEFORE np.uint8: cv2.GaussianBlur(image, (k, k), sigma,
// sigma, BORDER_REFLECT_101) with k = 1 (a copy) or 3.  OpenCV's float path for k = 3 (smooth.dispatch.cpp -> sepFilter2D,
// filter.simd.hpp SymmRowSmallFilter / SymmColumnSmallFilter), restated bit-exactly in the tests' blur oracle:
//   taps  k0 (centre), k1 (side): getGaussianKernel in float64 rounded to float32 — computed by the HOST, passed per sample;
//   row   R = C*k0 + (C[x-1] + C[x+1])*k1    then    column   B = (R[y-1] + R[y+1])*k1 + R*k0    (fp32, no fma);
//   reflect-101 at the CROP's border (index -1 -> 1, n -> n-2);  an axis of length 1 is not filtered (OpenCV's kernel
//   size drops to 1 there);  taps (1, 0) are an exact identity (C*1 + (..)*0 == C for the finite values here).
// The 3-tap kernel is symmetric and a + b == b + a in IEEE arithmetic, so blurring the unflipped crop and flipping the
// result is bit-identical to the reference's flip-then-blur.  Each block stages a TY x TX tile of the pre-truncation crop
// values plus a one-pixel halo (recomputed from the raw image: 16 raw taps per staged pixel, 1.2x the tile) in shared
// memory, runs the row pass into a second buffer, then the column pass, np.uint8, ToTensor and Normalize.
constexpr int BLUR_TY = 16, BLUR_TX = 32;

__device__ __forceinline__ int reflect101(int i, int n) { return n == 1 ? 0 : (i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i)); }

template <bool LabelMap>
__global__ void __launch_bounds__(256) augment_full_blur_u8_kernel(const uint8_t* __restrict__ arena,
                                                                   const seg_aug_full_entry* __restrict__ table,
                                                                   const float* __restrict__ blur_taps, int crop_h, int crop_w,
                                                                   int tiles_x, AugParams prm, float* __restrict__ out,
                                                                   int64_t* __restrict__ labels) {
  __shared__ float lut[3][256];
  __shared__ float cs[3][BLUR_TY + 2][BLUR_TX + 2];  // crop values, halo included
  __shared__ float rs[3][BLUR_TY + 2][BLUR_TX];      // after the row pass
  for (int t = threadIdx.x; t < 768; t += blockDim.x) {
    const int c = t >> 8, v = t & 255;
    lut[c][v] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)v, 255.f), prm.mean[c]), prm.stdv[c]);
  }
  const int b = blockIdx.y;
  const seg_aug_full_entry e = table[b];
  const uint8_t* img = arena + e.img_off;
  const int ty0 = (int)(blockIdx.x / tiles_x) * BLUR_TY, tx0 = (int)(blockIdx.x % tiles_x) * BLUR_TX;
  // the unflipped crop at (y, xs): rotated-image pixel (y + y0, xs + x0), zero padding outside h x w
  for (int t = threadIdx.x; t < (BLUR_TY + 2) * (BLUR_TX + 2); t += blockDim.x) {
    const int hy = t / (BLUR_TX + 2), hx = t - hy * (BLUR_TX + 2);
    const int y = ty0 + hy - 1, xs = tx0 + hx - 1;
    float v[3] = {0.f, 0.f, 0.f};
    if (y <= crop_h && xs <= crop_w) {  // beyond that only pixels outside the crop would read the value
      const int dy = reflect101(y, crop_h) + e.y0, dx = reflect101(xs, crop_w) + e.x0;
      if (dy < e.h && dx < e.w) rotated_pixel_f32(img, e, rot_coords(e, dy, dx), v);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) cs[c][hy][hx] = v[c];
  }
  __syncthreads();
  const float k0 = blur_taps[2 * b], k1 = blur_taps[2 * b + 1];
  const float kx0 = crop_w > 1 ? k0 : 1.f, kx1 = crop_w > 1 ? k1 : 0.f;
  const float ky0 = crop_h > 1 ? k0 : 1.f, ky1 = crop_h > 1 ? k1 : 0.f;
  for (int t = threadIdx.x; t < (BLUR_TY + 2) * BLUR_TX; t += blockDim.x) {
    const int hy = t / BLUR_TX, x = t - hy * BLUR_TX;
#pragma unroll
    for (int c = 0; c < 3; ++c)
      rs[c][hy][x] = __fadd_rn(__fmul_rn(cs[c][hy][x + 1], kx0), __fmul_rn(__fadd_rn(cs[c][hy][x], cs[c][hy][x + 2]), kx1));
  }
  __syncthreads();
  const uint8_t* lbl = (e.lbl_off >= 0 && labels != nullptr) ? arena + e.lbl_off : nullptr;
  const int32_t* lmap = label_map_of<LabelMap>(lbl, e.lbl_bytes, (int64_t)e.src_h * e.src_w);
  const int plane = crop_h * crop_w;
  float* o = out + (int64_t)b * 3 * plane;
  int64_t* lo = labels != nullptr ? labels + (int64_t)b * plane : nullptr;
  for (int t = threadIdx.x; t < BLUR_TY * BLUR_TX; t += blockDim.x) {
    const int ty = t / BLUR_TX, tx = t - ty * BLUR_TX;
    const int y = ty0 + ty, xs = tx0 + tx;
    if (y >= crop_h || xs >= crop_w) continue;
    unsigned u[3];
#pragma unroll
    for (int c = 0; c < 3; ++c)
      u[c] = trunc_u8(__fadd_rn(__fmul_rn(__fadd_rn(rs[c][ty][tx], rs[c][ty + 2][tx]), ky1), __fmul_rn(rs[c][ty + 1][tx], ky0)));
    const int i = y * crop_w + (e.flip ? crop_w - 1 - xs : xs);
    o[i] = lut[0][u[0]];
    o[plane + i] = lut[1][u[1]];
    o[2 * (int64_t)plane + i] = lut[2][u[2]];
    if (lo != nullptr) {
      const int dy = y + e.y0, dx = xs + e.x0;
      lo[i] = (dy < e.h && dx < e.w && lbl != nullptr) ? (int64_t)rotated_label<LabelMap>(lbl, lmap, e, rot_coords(e, dy, dx)) : 0;
    }
  }
}

// ------------------------------------------------------------------ bilinear resize of fp32 NCHW planes
// Source index exactly as ATen's area_pixel_compute_source_index (float arithmetic) — same helper as seg_elementwise.cu.
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

// dst[p][oy][ox] = beta * dst + alpha * R[p][oy][flip_x ? Wd-1-ox : ox],  R = bilinear resize of src plane p to Hd x Wd.
// mode 0 / 1 = ATen's bilinear with align_corners False / True (float source index, as F.interpolate / nn.Upsample);
// mode 2 = scipy.ndimage.zoom(order=1, prefilter=False) as inference.py:65 calls it: float64 coordinate o * (in-1)/(out-1),
// and — the library's mode='constant' rule — an output whose coordinate rounds to MORE than in-1 is the fill value 0
// (for some size pairs the last row / column of the zoomed image is black in the reference; reproduced, not fixed).
__global__ void __launch_bounds__(256) resize_nchw_kernel(const float* __restrict__ src, int64_t planes, int Hs, int Ws,
                                                          float* __restrict__ dst, int Hd, int Wd, int mode, float sh, float sw,
                                                          double zh, double zw, int flip_x, float alpha, float beta) {
  const int64_t total = planes * Hd * Wd;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ox = (int)(i % Wd);
    const int64_t t = i / Wd;
    const int oy = (int)(t % Hd);
    const int64_t p = t / Hd;
    const int sx = flip_x ? Wd - 1 - ox : ox;
    const float* base = src + p * Hs * Ws;
    float r;
    if (mode == 2) {
      const double cy = (double)oy * zh, cx = (double)sx * zw;
      if (cy > (double)(Hs - 1) || cx > (double)(Ws - 1)) {
        r = 0.f;
      } else {
        const int y0 = (int)cy, x0 = (int)cx;  // cy, cx >= 0
        const int y1 = y0 + (y0 < Hs - 1 ? 1 : 0), x1 = x0 + (x0 < Ws - 1 ? 1 : 0);
        const double ty = cy - (double)y0, tx = cx - (double)x0;
        const double a = base[(int64_t)y0 * Ws + x0], b = base[(int64_t)y0 * Ws + x1];
        const double c = base[(int64_t)y1 * Ws + x0], d = base[(int64_t)y1 * Ws + x1];
        r = (float)((1.0 - ty) * ((1.0 - tx) * a + tx * b) + ty * ((1.0 - tx) * c + tx * d));
      }
    } else {
      const Lerp ly = src_index(oy, sh, Hs, mode), lx = src_index(sx, sw, Ws, mode);
      const float a = base[(int64_t)ly.i0 * Ws + lx.i0], b = base[(int64_t)ly.i0 * Ws + lx.i1];
      const float c = base[(int64_t)ly.i1 * Ws + lx.i0], d = base[(int64_t)ly.i1 * Ws + lx.i1];
      const float h1 = ly.l1, h0 = 1.f - h1, w1 = lx.l1, w0 = 1.f - w1;
      r = h0 * (w0 * a + w1 * b) + h1 * (w0 * c + w1 * d);
    }
    const float v = alpha * r;
    dst[i] = beta != 0.f ? beta * dst[i] + v : v;
  }
}

// dst[p][y0 + y][x0 + x] += alpha * src[p][y][flip_x ? Ws-1-x : x]   for y < h, x < w   (sliding-window accumulation)
__global__ void __launch_bounds__(256) window_add_kernel(const float* __restrict__ src, int64_t planes, int Hs, int Ws,
                                                         float* __restrict__ dst, int Hd, int Wd, int y0, int x0, int h, int w,
                                                         int flip_x, float alpha) {
  const int64_t total = planes * h * w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % w);
    const int64_t t = i / w;
    const int y = (int)(t % h);
    const int64_t p = t / h;
    const float v = src[(p * Hs + y) * Ws + (flip_x ? Ws - 1 - x : x)];
    float* o = dst + (p * Hd + y0 + y) * Wd + x0 + x;
    *o += alpha * v;
  }
}

// x[p][y][x] /= count[y][x]  (sliding-window average, inference.py:55)
__global__ void __launch_bounds__(256) div_by_count_kernel(float* __restrict__ x, int64_t planes, int64_t hw,
                                                           const float* __restrict__ count) {
  const int64_t total = planes * hw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    x[i] = __fdiv_rn(x[i], count[i % hw]);
}

// labels[n][y][x] = `F.softmax(prediction, dim=0).argmax(0)` of inference.py:156 without the softmax pass:
//   * a pixel whose scores hold a NaN or a +inf has label 0 (its float64 softmax column is all NaN, and argmax returns the
//     first NaN);
//   * otherwise the first index of the maximum score (the softmax is monotone on finite and -inf scores, and argmax keeps
//     the first of equal values).
// One class of finite inputs differs: two top scores that differ by less than a float64 softmax resolves (both under about
// 2e-9 in magnitude) can round to equal probabilities, where the reference keeps the first; here the larger score wins.
__global__ void __launch_bounds__(256) argmax_nchw_kernel(const float* __restrict__ s, int N, int C, int64_t hw,
                                                          int64_t* __restrict__ labels) {
  const int64_t total = (int64_t)N * hw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / hw, q = i - n * hw;
    const float* p = s + n * C * hw + q;
    float best = p[0];
    int arg = 0;
    bool nonfinite = !(best < INFINITY);  // NaN or +inf
    for (int c = 1; c < C; ++c) {
      const float v = p[(int64_t)c * hw];
      nonfinite |= !(v < INFINITY);
      if (v > best) {
        best = v;
        arg = c;
      }
    }
    labels[i] = nonfinite ? 0 : arg;
  }
}

}  // namespace seg

using namespace seg;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int seg_aug_entry_bytes(void) { return (int)sizeof(seg_aug_entry); }
int seg_aug_scale_entry_bytes(void) { return (int)sizeof(seg_aug_scale_entry); }
int seg_aug_full_entry_bytes(void) { return (int)sizeof(seg_aug_full_entry); }

}  // extern "C"

namespace {

// Kernel launches of the augmentation entry points; LabelMap = true only for the *_mapped twins.
enum AugKind { AUG_PLAIN, AUG_SCALE, AUG_VAL, AUG_FULL, AUG_FULL_BLUR };

template <bool LabelMap>
int launch_augment(AugKind kind, const char* name, const uint8_t* arena, const void* table, const float* blur_taps, int B, int crop_h,
                   int crop_w, const float* mean3, const float* std3, float* out_nchw, int64_t* out_labels, void* stream) {
  SEG_REQUIRE(arena != nullptr && table != nullptr && out_nchw != nullptr && mean3 != nullptr && std3 != nullptr &&
                  (kind != AUG_FULL_BLUR || blur_taps != nullptr),
              "%s: null pointer", name);
  SEG_REQUIRE(B > 0 && B <= 65535 && crop_h > 0 && crop_w > 0 && (int64_t)crop_h * crop_w < (1ll << 30), "%s: bad batch / crop size", name);
  AugParams prm;
  for (int c = 0; c < 3; ++c) {
    prm.mean[c] = mean3[c];  // host pointers: six floats by value into the kernel arguments
    prm.stdv[c] = std3[c];
    SEG_REQUIRE(std3[c] != 0.f, "%s: std must be non-zero", name);
  }
  if (kind == AUG_FULL_BLUR) {
    const int64_t tiles_x = ceil_div64(crop_w, BLUR_TX), tiles = tiles_x * ceil_div64(crop_h, BLUR_TY);  // < 2^31 for crop_h * crop_w < 2^30
    dim3 grid((unsigned)tiles, (unsigned)B, 1);
    augment_full_blur_u8_kernel<LabelMap><<<grid, 256, 0, ST(stream)>>>(arena, static_cast<const seg_aug_full_entry*>(table), blur_taps,
                                                                        crop_h, crop_w, (int)tiles_x, prm, out_nchw, out_labels);
    return check_launch(name);
  }
  // blockIdx.y = image; the B images share ~8 blocks per SM between them
  int64_t per_image = ((int64_t)num_sms() * 8 + B - 1) / B;
  const int64_t need = ceil_div64((int64_t)crop_h * crop_w, 256);
  if (per_image > need) per_image = need;
  if (per_image < 1) per_image = 1;
  dim3 grid((unsigned)per_image, (unsigned)B, 1);
  switch (kind) {
    case AUG_PLAIN:
      augment_u8_kernel<LabelMap><<<grid, 256, 0, ST(stream)>>>(arena, static_cast<const seg_aug_entry*>(table), crop_h, crop_w, prm,
                                                                out_nchw, out_labels);
      break;
    case AUG_SCALE:
      augment_scale_u8_kernel<false, LabelMap><<<grid, 256, 0, ST(stream)>>>(arena, static_cast<const seg_aug_scale_entry*>(table), crop_h,
                                                                             crop_w, prm, out_nchw, out_labels);
      break;
    case AUG_VAL:
      augment_scale_u8_kernel<true, LabelMap><<<grid, 256, 0, ST(stream)>>>(arena, static_cast<const seg_aug_scale_entry*>(table), crop_h,
                                                                            crop_w, prm, out_nchw, out_labels);
      break;
    default:
      augment_full_u8_kernel<LabelMap><<<grid, 256, 0, ST(stream)>>>(arena, static_cast<const seg_aug_full_entry*>(table), crop_h, crop_w,
                                                                     prm, out_nchw, out_labels);
  }
  return check_launch(name);
}

}  // namespace

extern "C" {

#define SEG_AUG_ENTRY(fn, kind, rec, mapped)                                                                                       \
  int fn(const uint8_t* arena, const rec* table, int B, int crop_h, int crop_w, const float* mean3, const float* std3, float* out_nchw, \
         int64_t* out_labels, void* stream) {                                                                                         \
    return launch_augment<mapped>(kind, #fn, arena, table, nullptr, B, crop_h, crop_w, mean3, std3, out_nchw, out_labels, stream);   \
  }
SEG_AUG_ENTRY(seg_augment_batch_u8, AUG_PLAIN, seg_aug_entry, false)
SEG_AUG_ENTRY(seg_augment_scale_batch_u8, AUG_SCALE, seg_aug_scale_entry, false)
SEG_AUG_ENTRY(seg_augment_val_batch_u8, AUG_VAL, seg_aug_scale_entry, false)
SEG_AUG_ENTRY(seg_augment_full_batch_u8, AUG_FULL, seg_aug_full_entry, false)
SEG_AUG_ENTRY(seg_augment_mapped_batch_u8, AUG_PLAIN, seg_aug_entry, true)
SEG_AUG_ENTRY(seg_augment_scale_mapped_batch_u8, AUG_SCALE, seg_aug_scale_entry, true)
SEG_AUG_ENTRY(seg_augment_val_mapped_batch_u8, AUG_VAL, seg_aug_scale_entry, true)
SEG_AUG_ENTRY(seg_augment_full_mapped_batch_u8, AUG_FULL, seg_aug_full_entry, true)
#undef SEG_AUG_ENTRY

int seg_augment_full_blur_batch_u8(const uint8_t* arena, const seg_aug_full_entry* table, const float* blur_taps, int B, int crop_h,
                                   int crop_w, const float* mean3, const float* std3, float* out_nchw, int64_t* out_labels,
                                   void* stream) {
  return launch_augment<false>(AUG_FULL_BLUR, "seg_augment_full_blur_batch_u8", arena, table, blur_taps, B, crop_h, crop_w, mean3, std3,
                               out_nchw, out_labels, stream);
}

int seg_augment_full_blur_mapped_batch_u8(const uint8_t* arena, const seg_aug_full_entry* table, const float* blur_taps, int B,
                                          int crop_h, int crop_w, const float* mean3, const float* std3, float* out_nchw,
                                          int64_t* out_labels, void* stream) {
  return launch_augment<true>(AUG_FULL_BLUR, "seg_augment_full_blur_mapped_batch_u8", arena, table, blur_taps, B, crop_h, crop_w, mean3,
                              std3, out_nchw, out_labels, stream);
}

int seg_resize_nchw_f32(const float* src, int64_t planes, int Hs, int Ws, float* dst, int Hd, int Wd, int mode, int flip_x,
                        float alpha, float beta, void* stream) {
  SEG_REQUIRE(planes > 0 && Hs > 0 && Ws > 0 && Hd > 0 && Wd > 0, "resize: bad size");
  SEG_REQUIRE(src != dst, "resize: in-place is not supported");
  SEG_REQUIRE(mode >= 0 && mode <= 2, "resize: mode must be 0 (align_corners=False), 1 (True) or 2 (ndimage.zoom)");
  const int ac = mode == 0 ? 0 : 1;
  // ndimage.zoom: zoom = (in - 1) / (out - 1) per axis in float64, 1 where out == 1 (scipy/ndimage/_interpolation.py)
  const double zh = Hd > 1 ? (double)(Hs - 1) / (double)(Hd - 1) : 1.0, zw = Wd > 1 ? (double)(Ws - 1) / (double)(Wd - 1) : 1.0;
  resize_nchw_kernel<<<grid_for(planes * Hd * Wd, 256), 256, 0, ST(stream)>>>(
      src, planes, Hs, Ws, dst, Hd, Wd, mode, resize_scale(Hs, Hd, ac), resize_scale(Ws, Wd, ac), zh, zw, flip_x, alpha, beta);
  return check_launch("resize_nchw_f32");
}

int seg_window_add_nchw_f32(const float* src, int64_t planes, int Hs, int Ws, float* dst, int Hd, int Wd, int y0, int x0, int h,
                            int w, int flip_x, float alpha, void* stream) {
  SEG_REQUIRE(planes > 0 && h > 0 && w > 0 && h <= Hs && w <= Ws && y0 >= 0 && x0 >= 0 && y0 + h <= Hd && x0 + w <= Wd,
              "window_add: window (%d,%d)+(%dx%d) does not fit src %dx%d / dst %dx%d", y0, x0, h, w, Hs, Ws, Hd, Wd);
  window_add_kernel<<<grid_for(planes * h * w, 256), 256, 0, ST(stream)>>>(src, planes, Hs, Ws, dst, Hd, Wd, y0, x0, h, w, flip_x, alpha);
  return check_launch("window_add_nchw_f32");
}

int seg_div_by_count_nchw_f32(float* x, int64_t planes, int H, int W, const float* count_hw, void* stream) {
  SEG_REQUIRE(planes > 0 && H > 0 && W > 0, "div_by_count: bad size");
  div_by_count_kernel<<<grid_for(planes * H * W, 256), 256, 0, ST(stream)>>>(x, planes, (int64_t)H * W, count_hw);
  return check_launch("div_by_count_nchw_f32");
}

int seg_argmax_nchw_f32(const float* scores, int N, int C, int H, int W, int64_t* labels, void* stream) {
  SEG_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0, "argmax: bad size");
  argmax_nchw_kernel<<<grid_for((int64_t)N * H * W, 256), 256, 0, ST(stream)>>>(scores, N, C, (int64_t)H * W, labels);
  return check_launch("argmax_nchw_f32");
}

}  // extern "C"
