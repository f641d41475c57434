// ImageAug3D + ImageNormalize of the camera pipeline (transforms_3d.py:98-192, 992-1006) on the device, bit-exact
// to Pillow + torchvision:
//
//   TF.normalize(TF.to_tensor(img.resize(dims).crop(box)[.transpose(FLIP_LEFT_RIGHT)].rotate(deg)), mean, std)
//
// Three launches per call, all draw parameters read from device memory (CUDA-graph capturable):
//   1. image_aug_setup_kernel    one CTA per camera: validates the draw, builds Pillow's BICUBIC coefficient tables
//                                for the crop window's columns and rows only (precompute_coeffs +
//                                normalize_coeffs_8bpc: double filter weights in Pillow's order, then 22-bit fixed
//                                point), the source-row band the vertical filters read, Image.rotate's inverse matrix
//                                (round(cos, 15) included) and the reference's fp32 img_aug_matrix.
//   2. image_aug_hpass_kernel    horizontal pass (ImagingResampleHorizontal_8bpc) over the band rows and the crop
//                                columns: uint8 RGBx rows into the workspace.
//   3. image_aug_vpass_kernel    one thread per output pixel: Pillow's rotate rule picks the crop pixel, the flip
//                                and the crop map it into the resized image (outside it is 0), the vertical pass
//                                (ImagingResampleVertical_8bpc) makes its three uint8 channels, and u8 / 255 then
//                                (x - mean) / std in fp32 gives the planar output; the stores are coalesced per plane.
//
// Every double and float expression that Pillow, CPython or torch evaluate is written with explicit _rn intrinsics
// so that nvcc cannot contract it into an FMA: the host code being matched has none.
#include <math.h>

#include "common.cuh"

namespace bevb200 {
namespace {

constexpr int kPrecisionBits = 22;        // Resample.c PRECISION_BITS (32 - 8 - 2)
constexpr int kMaxFrame = 16384;          // output sides: keeps every rotate coordinate in the 16.16 fixed range
constexpr int kMaxSource = 1 << 19;       // input and resized sides (grid rows, exact float box)
constexpr int kSetupThreads = 256;
constexpr int kHpassCols = 128;
constexpr int kHpassRows = 8;
constexpr int kVpassCols = 128;
constexpr int kMaxGridY = 65535;          // CUDA's grid.y and grid.z limit: hpass row blocks, cameras

enum RotateKind { kCopy = 0, kRot180 = 1, kRot90 = 2, kRot270 = 3, kScale = 4, kAffine = 5 };

struct CamParams {
  int valid;                     // 0: the draw was rejected; the camera's outputs are NaN
  int resize_w, resize_h, crop_x, crop_y, flip;
  int band_first, band_rows;     // source rows [band_first, band_first + band_rows) feed the vertical pass
  int kind;                      // RotateKind
  int a0, a1, a2, a3, a4, a5;    // 16.16 fixed-point affine (kAffine)
  double xo, yo, sx, sy;         // scaling path (kScale)
};

// ---- Pillow's coefficient arithmetic -------------------------------------------------------------

__device__ __forceinline__ double bicubic_filter(double x) {
  // ((a + 2) x - (a + 3)) x x + 1 and (((x - 5) x + 8) x - 4) a with a = -0.5, evaluated as Resample.c does
  if (x < 0.0) x = -x;
  if (x < 1.0) return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(1.5, x), 2.5), x), x), 1.0);
  if (x < 2.0) return __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(x, 5.0), x), 8.0), x), 4.0), -0.5);
  return 0.0;
}

struct FilterGeom {
  double scale, filterscale, support, ss;
  int ksize;
};

__device__ __forceinline__ FilterGeom filter_geom(int in_size, int out_size) {
  FilterGeom g;
  g.scale = __ddiv_rn((double)((float)in_size - 0.0f), (double)out_size);
  g.filterscale = g.scale < 1.0 ? 1.0 : g.scale;
  g.support = __dmul_rn(2.0, g.filterscale);
  g.ksize = (int)ceil(g.support) * 2 + 1;
  g.ss = __ddiv_rn(1.0, g.filterscale);
  return g;
}

// precompute_coeffs for output index xx, then normalize_coeffs_8bpc: writes k[0, count) and returns (xmin, count)
__device__ int2 pillow_coeffs(const FilterGeom &g, int in_size, int xx, int32_t *k) {
  const double center = __dadd_rn(0.0, __dmul_rn((double)xx + 0.5, g.scale));
  int xmin = (int)__dadd_rn(__dsub_rn(center, g.support), 0.5);
  if (xmin < 0) xmin = 0;
  int xmax = (int)__dadd_rn(__dadd_rn(center, g.support), 0.5);
  if (xmax > in_size) xmax = in_size;
  xmax -= xmin;
  double ww = 0.0;
  for (int x = 0; x < xmax; ++x)
    ww = __dadd_rn(ww, bicubic_filter(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), g.ss)));
  for (int x = 0; x < xmax; ++x) {
    double w = bicubic_filter(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), g.ss));
    if (ww != 0.0) w = __ddiv_rn(w, ww);
    const double s = __dmul_rn(w, (double)(1 << kPrecisionBits));
    k[x] = w < 0 ? (int)__dadd_rn(-0.5, s) : (int)__dadd_rn(0.5, s);
  }
  return make_int2(xmin, xmax);
}

__device__ __forceinline__ int clip8(int ss) {
  ss >>= kPrecisionBits;
  return ss < 0 ? 0 : (ss > 255 ? 255 : ss);
}

// ---- Image.rotate's matrix -------------------------------------------------------------------------

// CPython's round(v, 15): the exact binary value rounded half-to-even at the 15th decimal, then the nearest double
// (half-to-even is symmetric: the magnitude is rounded and the sign put back, -0.0 included)
__device__ double round15(double v) {
  const bool neg = signbit(v);
  v = fabs(v);
  const double p = __dmul_rn(v, 1e15);
  const double e = __fma_rn(v, 1e15, -p);   // v * 1e15 == p + e exactly
  double n;
  if (p < 0.5) {
    n = 0.0;
  } else if (p == 0.5) {
    n = e > 0.0 ? 1.0 : 0.0;
  } else {
    const double fl = floor(p);
    const double d = __dsub_rn(__dsub_rn(p, fl), 0.5);   // exact: p >= 0.5 carries at most 52 fraction bits
    if (d > -e) n = fl + 1.0;
    else if (d < -e) n = fl;
    else n = fmod(fl, 2.0) == 0.0 ? fl : fl + 1.0;
  }
  const double r = __ddiv_rn(n, 1e15);
  return neg ? -r : r;
}

__device__ __forceinline__ int fix16(double v) { return (int)floor(__dadd_rn(__dmul_rn(v, 65536.0), 0.5)); }

// Image.rotate(angle) of a w x h image, NEAREST, no expand, no centre or translate
__device__ void rotate_setup(double angle, int w, int h, CamParams &p) {
  double a = fmod(angle, 360.0);                           // CPython float %
  if (a != 0.0) {
    if (a < 0.0) a = __dadd_rn(a, 360.0);
  } else {
    a = 0.0;
  }
  if (a == 0.0) { p.kind = kCopy; return; }
  if (a == 180.0) { p.kind = kRot180; return; }
  if ((a == 90.0 || a == 270.0) && w == h) { p.kind = a == 90.0 ? kRot90 : kRot270; return; }
  const double t = -__dmul_rn(a, 3.141592653589793 / 180.0);  // -math.radians(angle)
  const double c = cos(t), s = sin(t);
  const double m0 = round15(c), m1 = round15(s), m3 = round15(-s), m4 = round15(c);
  const double cx = w / 2.0, cy = h / 2.0;
  double m2 = __dadd_rn(__dadd_rn(__dmul_rn(m0, -cx), __dmul_rn(m1, -cy)), 0.0);
  double m5 = __dadd_rn(__dadd_rn(__dmul_rn(m3, -cx), __dmul_rn(m4, -cy)), 0.0);
  m2 = __dadd_rn(m2, cx);
  m5 = __dadd_rn(m5, cy);
  if (m1 == 0.0 && m3 == 0.0) {
    // ImagingScaleAffine: here |m0| == |m4| == 1, so its running sums are exact and equal the closed form
    p.kind = kScale;
    p.xo = __dadd_rn(m2, __dmul_rn(m0, 0.5));
    p.yo = __dadd_rn(m5, __dmul_rn(m4, 0.5));
    p.sx = m0;
    p.sy = m4;
    return;
  }
  // affine_fixed: 16.16 integer sums, exact in closed form (every corner of a kMaxFrame frame is within +-32768)
  p.kind = kAffine;
  p.a0 = fix16(m0);
  p.a1 = fix16(m1);
  p.a3 = fix16(m3);
  p.a4 = fix16(m4);
  p.a2 = fix16(__dadd_rn(__dadd_rn(m2, __dmul_rn(m0, 0.5)), __dmul_rn(m1, 0.5)));
  p.a5 = fix16(__dadd_rn(__dadd_rn(m5, __dmul_rn(m3, 0.5)), __dmul_rn(m4, 0.5)));
}

__device__ __forceinline__ float dot2(float a0, float b0, float a1, float b1) {
  return __fadd_rn(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}

// img_transform's post-homography (transforms_3d.py:145-162) in the reference's torch fp32 arithmetic
__device__ void img_aug_matrix(double resize, int crop_x, int crop_y, int flip, double rotate, int fW, int fH,
                           float *M) {
  const float r = __double2float_rn(resize);
  float R[2][2] = {{r, 0.0f}, {0.0f, r}};
  float t[2] = {__fsub_rn(0.0f, (float)crop_x), __fsub_rn(0.0f, (float)crop_y)};
  if (flip) {
    const float A[2][2] = {{-1.0f, 0.0f}, {0.0f, 1.0f}};
    float R2[2][2];
    for (int i = 0; i < 2; ++i)
      for (int j = 0; j < 2; ++j) R2[i][j] = dot2(A[i][0], R[0][j], A[i][1], R[1][j]);
    const float t0 = __fadd_rn(dot2(A[0][0], t[0], A[0][1], t[1]), (float)fW);
    const float t1 = __fadd_rn(dot2(A[1][0], t[0], A[1][1], t[1]), 0.0f);
    for (int i = 0; i < 2; ++i)
      for (int j = 0; j < 2; ++j) R[i][j] = R2[i][j];
    t[0] = t0;
    t[1] = t1;
  }
  const double theta = __dmul_rn(__ddiv_rn(rotate, 180.0), 3.141592653589793);
  const double c = cos(theta), s = sin(theta);
  const float A[2][2] = {{__double2float_rn(c), __double2float_rn(s)}, {__double2float_rn(-s), __double2float_rn(c)}};
  const float cx = __fdiv_rn((float)fW, 2.0f), cy = __fdiv_rn((float)fH, 2.0f);
  const float b0 = __fadd_rn(dot2(A[0][0], -cx, A[0][1], -cy), cx);
  const float b1 = __fadd_rn(dot2(A[1][0], -cx, A[1][1], -cy), cy);
  for (int i = 0; i < 16; ++i) M[i] = (i % 5 == 0) ? 1.0f : 0.0f;
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j) M[i * 4 + j] = dot2(A[i][0], R[0][j], A[i][1], R[1][j]);
  M[3] = __fadd_rn(dot2(A[0][0], t[0], A[0][1], t[1]), b0);
  M[7] = __fadd_rn(dot2(A[1][0], t[0], A[1][1], t[1]), b1);
}

__device__ __forceinline__ bool is_int_in(double v, double lo, double hi) {
  return v == floor(v) && v >= lo && v <= hi;   // false for NaN
}

// ---- kernels -----------------------------------------------------------------------------------------

struct Tables {
  CamParams *params;
  int2 *hbounds;      // [cams, fW] (xmin, count) per crop column; count 0: the column is outside the resized image
  int32_t *hcoef;     // [cams, fW, kcap_w]
  int2 *vbounds;      // [cams, fH]
  int32_t *vcoef;     // [cams, fH, kcap_h]
  uchar4 *band;       // [cams, H, fW] horizontally resampled rows (RGB + pad)
};

__global__ void __launch_bounds__(kSetupThreads)
image_aug_setup_kernel(const double *__restrict__ draws, int H, int W, int fH, int fW, int kcap_w, int kcap_h,
                       Tables T, float *__restrict__ aug_matrix, int32_t *__restrict__ status) {
  const int cam = blockIdx.x;
  __shared__ CamParams sp;
  __shared__ int band_lo, band_hi;
  const double *d = draws + (size_t)cam * BEVB200_IMAGE_AUG_DRAW_FIELDS;
  if (threadIdx.x == 0) {
    const double resize = d[0], rw = d[1], rh = d[2], cxd = d[3], cyd = d[4], fl = d[5], rot = d[6];
    int bad = 0;
    if (!(isfinite(resize) && isfinite(rot)) || !is_int_in(rw, 1.0, kMaxSource - 1) ||
        !is_int_in(rh, 1.0, kMaxSource - 1) || !is_int_in(cxd, -1073741824.0, 1073741824.0) ||
        !is_int_in(cyd, -1073741824.0, 1073741824.0) || !(fl == 0.0 || fl == 1.0))
      bad |= BEVB200_IMAGE_AUG_BAD_DRAW;
    CamParams p = {};
    if (!bad) {
      p.resize_w = (int)rw;
      p.resize_h = (int)rh;
      p.crop_x = (int)cxd;
      p.crop_y = (int)cyd;
      p.flip = (int)fl;
      if (filter_geom(W, p.resize_w).ksize > kcap_w || filter_geom(H, p.resize_h).ksize > kcap_h)
        bad |= BEVB200_IMAGE_AUG_OVER_CAPACITY;
    }
    float *M = aug_matrix + (size_t)cam * 16;
    if (bad) {
      atomicOr(status, bad);
      for (int i = 0; i < 16; ++i) M[i] = __int_as_float(0x7fc00000);
    } else {
      p.valid = 1;
      rotate_setup(rot, fW, fH, p);
      img_aug_matrix(resize, p.crop_x, p.crop_y, p.flip, rot, fW, fH, M);
    }
    sp = p;
    band_lo = 0x7fffffff;
    band_hi = 0;
  }
  __syncthreads();
  if (!sp.valid) {
    if (threadIdx.x == 0) T.params[cam] = sp;
    return;
  }
  const FilterGeom gw = filter_geom(W, sp.resize_w), gh = filter_geom(H, sp.resize_h);
  for (int j = threadIdx.x; j < fW; j += blockDim.x) {
    const int xr = sp.crop_x + j;
    int2 b = make_int2(0, 0);
    if (xr >= 0 && xr < sp.resize_w) b = pillow_coeffs(gw, W, xr, T.hcoef + ((size_t)cam * fW + j) * kcap_w);
    T.hbounds[(size_t)cam * fW + j] = b;
  }
  for (int i = threadIdx.x; i < fH; i += blockDim.x) {
    const int yr = sp.crop_y + i;
    int2 b = make_int2(0, 0);
    if (yr >= 0 && yr < sp.resize_h) {
      b = pillow_coeffs(gh, H, yr, T.vcoef + ((size_t)cam * fH + i) * kcap_h);
      atomicMin(&band_lo, b.x);
      atomicMax(&band_hi, b.x + b.y);
    }
    T.vbounds[(size_t)cam * fH + i] = b;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    CamParams p = sp;
    p.band_first = band_hi > band_lo ? band_lo : 0;
    p.band_rows = band_hi > band_lo ? band_hi - band_lo : 0;
    T.params[cam] = p;
  }
}

__global__ void __launch_bounds__(kHpassCols)
image_aug_hpass_kernel(const uint8_t *__restrict__ images, int H, int W, int fW, int kcap_w, Tables T) {
  const int cam = blockIdx.z;
  const int j = blockIdx.x * kHpassCols + threadIdx.x;
  const CamParams &p = T.params[cam];
  if (!p.valid || j >= fW) return;
  const int row0 = blockIdx.y * kHpassRows;
  if (row0 >= p.band_rows) return;
  const int2 b = T.hbounds[(size_t)cam * fW + j];
  if (b.y == 0) return;
  const int32_t *k = T.hcoef + ((size_t)cam * fW + j) * kcap_w;
  // a band taller than gridDim.y row blocks (in_h > 65535 * kHpassRows) is covered in gridDim.y strides
  for (int first = row0; first < p.band_rows; first += gridDim.y * kHpassRows) {
    const int rows = min(kHpassRows, p.band_rows - first);
    for (int r = 0; r < rows; ++r) {
      const int y = p.band_first + first + r;
      const uint8_t *src = images + (((size_t)cam * H + y) * W + b.x) * 3;
      int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
      for (int x = 0; x < b.y; ++x) {
        const int kx = __ldg(k + x);
        s0 += (int)__ldg(src + 3 * x + 0) * kx;
        s1 += (int)__ldg(src + 3 * x + 1) * kx;
        s2 += (int)__ldg(src + 3 * x + 2) * kx;
      }
      T.band[((size_t)cam * H + first + r) * fW + j] =
          make_uchar4((unsigned char)clip8(s0), (unsigned char)clip8(s1), (unsigned char)clip8(s2), 0);
    }
  }
}

__global__ void __launch_bounds__(kVpassCols)
image_aug_vpass_kernel(int H, int fH, int fW, int kcap_h, Tables T, float m0, float m1, float m2, float s0, float s1,
                       float s2, float *__restrict__ out) {
  const int cam = blockIdx.z, y = blockIdx.y;
  const int x = blockIdx.x * kVpassCols + threadIdx.x;
  if (x >= fW) return;
  const CamParams &p = T.params[cam];
  const size_t plane = (size_t)fH * fW;
  float *o = out + (size_t)cam * 3 * plane + (size_t)y * fW + x;
  if (!p.valid) {
    const float nan = __int_as_float(0x7fc00000);
    o[0] = nan;
    o[plane] = nan;
    o[2 * plane] = nan;
    return;
  }
  // Image.rotate: which pixel (xc, yc) of the cropped (and flipped) image lands at (x, y)
  int xc, yc;
  switch (p.kind) {
    case kCopy: xc = x; yc = y; break;
    case kRot180: xc = fW - 1 - x; yc = fH - 1 - y; break;
    case kRot90: xc = fH - 1 - y; yc = x; break;
    case kRot270: xc = y; yc = fW - 1 - x; break;
    case kScale: {
      const double vx = __dadd_rn(p.xo, __dmul_rn((double)x, p.sx));
      const double vy = __dadd_rn(p.yo, __dmul_rn((double)y, p.sy));
      xc = vx < 0.0 ? -1 : (int)vx;
      yc = vy < 0.0 ? -1 : (int)vy;
      break;
    }
    default:
      xc = (p.a2 + y * p.a1 + x * p.a0) >> 16;
      yc = (p.a5 + y * p.a4 + x * p.a3) >> 16;
  }
  int c0 = 0, c1 = 0, c2 = 0;
  if (xc >= 0 && xc < fW && yc >= 0 && yc < fH) {
    const int xs = p.flip ? fW - 1 - xc : xc;        // FLIP_LEFT_RIGHT of the crop
    const int2 b = T.vbounds[(size_t)cam * fH + yc];
    const int2 h = T.hbounds[(size_t)cam * fW + xs];
    if (b.y > 0 && h.y > 0) {                          // inside the resized image; else the crop's fill 0
      const int32_t *k = T.vcoef + ((size_t)cam * fH + yc) * kcap_h;
      const uchar4 *col = T.band + ((size_t)cam * H + (b.x - p.band_first)) * fW + xs;
      int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
      for (int r = 0; r < b.y; ++r) {
        const uchar4 v = col[(size_t)r * fW];
        const int kr = __ldg(k + r);
        a0 += (int)v.x * kr;
        a1 += (int)v.y * kr;
        a2 += (int)v.z * kr;
      }
      c0 = clip8(a0);
      c1 = clip8(a1);
      c2 = clip8(a2);
    }
  }
  o[0] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)c0, 255.0f), m0), s0);
  o[plane] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)c1, 255.0f), m1), s1);
  o[2 * plane] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)c2, 255.0f), m2), s2);
}

// ksize of Pillow's BICUBIC filter for in_size -> out_size (filter_geom on the host)
int ksize_for(int in_size, int out_size) {
  const double scale = (double)((float)in_size - 0.0f) / (double)out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  return (int)ceil(2.0 * filterscale) * 2 + 1;
}

Tables carve(void *ws, int cams, int H, int fH, int fW, int kcap_w, int kcap_h, size_t *bytes) {
  Arena a(ws, 0);
  Tables T;
  T.params = a.take<CamParams>(cams);
  T.hbounds = a.take<int2>((size_t)cams * fW);
  T.hcoef = a.take<int32_t>((size_t)cams * fW * kcap_w);
  T.vbounds = a.take<int2>((size_t)cams * fH);
  T.vcoef = a.take<int32_t>((size_t)cams * fH * kcap_h);
  T.band = a.take<uchar4>((size_t)cams * H * fW);
  *bytes = a.off;
  return T;
}

bool sizes_ok(int cams, int H, int W, int fH, int fW, int min_w, int min_h) {
  return cams >= 0 && cams <= kMaxGridY && H >= 1 && W >= 1 && H < kMaxSource && W < kMaxSource && fH >= 1 &&
         fW >= 1 && fH <= kMaxFrame && fW <= kMaxFrame && min_w >= 1 && min_h >= 1 && min_w < kMaxSource &&
         min_h < kMaxSource;
}

}  // namespace
}  // namespace bevb200

using namespace bevb200;

extern "C" {

size_t bevb200_image_aug_workspace_bytes(int cams, int in_h, int in_w, int out_h, int out_w, int min_resize_w,
                                         int min_resize_h) {
  if (!sizes_ok(cams, in_h, in_w, out_h, out_w, min_resize_w, min_resize_h)) return 0;
  size_t bytes = 0;
  carve(nullptr, cams, in_h, out_h, out_w, ksize_for(in_w, min_resize_w), ksize_for(in_h, min_resize_h), &bytes);
  return bytes;
}

int bevb200_image_aug(const uint8_t *images, int cams, int in_h, int in_w, const double *draws, int out_h, int out_w,
                      int min_resize_w, int min_resize_h, float mean0, float mean1, float mean2, float std0,
                      float std1, float std2, float *out, float *aug_matrix, int32_t *status, void *workspace,
                      size_t workspace_bytes, void *stream) {
  BEVB200_REQUIRE(sizes_ok(cams, in_h, in_w, out_h, out_w, min_resize_w, min_resize_h),
                  "sizes out of range (cams <= 65535; 1 <= out_h, out_w <= 16384; 1 <= in_h, in_w, min_resize_* < 2^19)");
  if (cams == 0) return BEVB200_OK;
  BEVB200_REQUIRE(images && draws && out && aug_matrix && status, "null pointer");
  const int kcap_w = ksize_for(in_w, min_resize_w), kcap_h = ksize_for(in_h, min_resize_h);
  size_t need = 0;
  carve(nullptr, cams, in_h, out_h, out_w, kcap_w, kcap_h, &need);
  if (!workspace || workspace_bytes < need) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace of %zu bytes, need %zu", __func__, workspace_bytes,
             need);
    return BEVB200_EWORKSPACE;
  }
  Tables T = carve(workspace, cams, in_h, out_h, out_w, kcap_w, kcap_h, &need);
  cudaStream_t st = (cudaStream_t)stream;
  BEVB200_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
  BEVB200_LAUNCH(image_aug_setup_kernel, cams, kSetupThreads, 0, st, draws, in_h, in_w, out_h, out_w, kcap_w, kcap_h,
                 T, aug_matrix, status);
  const int row_blocks = min((in_h + kHpassRows - 1) / kHpassRows, kMaxGridY);   // the kernel strides past 65535
  const dim3 hgrid((out_w + kHpassCols - 1) / kHpassCols, row_blocks, cams);
  BEVB200_LAUNCH(image_aug_hpass_kernel, hgrid, kHpassCols, 0, st, images, in_h, in_w, out_w, kcap_w, T);
  const dim3 vgrid((out_w + kVpassCols - 1) / kVpassCols, out_h, cams);
  BEVB200_LAUNCH(image_aug_vpass_kernel, vgrid, kVpassCols, 0, st, in_h, out_h, out_w, kcap_h, T, mean0, mean1, mean2,
                 std0, std1, std2, out);
  return BEVB200_OK;
}

}  // extern "C"
