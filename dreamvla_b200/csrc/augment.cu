// Device-side pieces of the reference's collator (SURVEY.md 8f-2): the random-shift augmentation and the depth resize, which
// the reference runs on CPU data-loader workers (utils/data_utils.py:326-383 `RandomShiftsAug`, :3588-3603 `depth_image_fn`,
// applied in `collator` :1337-1354).
//
// RandomShiftsAug: replicate-pad by `pad`, then grid_sample (bilinear, align_corners=False) on a grid of the padded image's
// own pixel centres moved by an INTEGER number of pixels (sx, sy) in [0, 2*pad] -- every sample point is a pixel centre, the
// bilinear weights are (1, 0, 0, 0), and the op is a shifted crop with clamped indices:
//     out[n, c, y, x] = in[n, c, clamp(y + sy - pad, 0, H-1), clamp(x + sx - pad, 0, W-1)]
// (exact; the reference's fp32 grid arithmetic lands within ~1e-5 pixels of the centres, oracle/augment_oracle.py measures the
// difference).  One pass: 4 B read (fp32 from the loader) + 2 B written (bf16 for the model) per element, HBM-bound.
//
// depth resize: torchvision `Resize(NEAREST)` on a tensor = F.interpolate(mode="nearest"): src = min(floor(dst * in/out), in-1),
// the scale computed in fp32 as torch does.
//
// image_fn: CLIP's `_transform(224)` (Resize(224, BICUBIC) on the short side, CenterCrop(224), ToTensor, Normalize) of uint8 HWC
// frames, the reference's `image_processor` (collator :175-179, :1311-1312; rollouts eval_utils_calvin.py:82-90,
// eval_utils_libero.py:94-106).  Pillow resizes 8-bit images in two separable integer passes (horizontal, then vertical) with
// 22-bit fixed-point coefficients and rounds to uint8 between them, so the crop is reproduced bit for bit: the coefficients are
// Pillow's own computation (dvla_bicubic_coeffs below, host double arithmetic), the passes its integer sums.  Normalize is a
// [3, 256] table the caller fills with torch's own arithmetic.
#include <math.h>

#include "common.cuh"
#include "host.cuh"
#include "../../include/dvla.h"

namespace dvla {

template <typename T> __device__ __forceinline__ float ld_as_float(const T* p);
template <> __device__ __forceinline__ float ld_as_float<float>(const float* p) { return __ldg(p); }
template <> __device__ __forceinline__ float ld_as_float<bf16>(const bf16* p) { return __bfloat162float(*p); }
template <typename T> __device__ __forceinline__ void st_from_float(T* p, float v);
template <> __device__ __forceinline__ void st_from_float<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void st_from_float<bf16>(bf16* p, float v) { *p = __float2bfloat16(v); }

// warp = one output row (img, channel, y) at a time, lanes stride x: the index arithmetic (two divisions, the clamp of y) is done
// once per row, reads of a row are contiguous (shifted by sx) except at the clamped borders, writes are contiguous
template <typename Tin, typename Tout>
__global__ void __launch_bounds__(256) shift_crop_kernel(const Tin* __restrict__ x, Tout* __restrict__ out,
                                                         const int* __restrict__ shifts, long long n, int c, int h, int w, int pad) {
  const int lane = threadIdx.x & 31;
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long rows = n * c * h;
  for (long long r = warp; r < rows; r += nwarps) {
    const long long img = r / (static_cast<long long>(c) * h);
    const int y = static_cast<int>(r % h);
    const int sx = __ldg(shifts + 2 * img), sy = __ldg(shifts + 2 * img + 1);
    const int ys = min(max(y + sy - pad, 0), h - 1);
    const Tin* src = x + (r - y + ys) * w;            // same image and channel, source row ys
    Tout* dst = out + r * w;
    for (int xx = lane; xx < w; xx += 32) st_from_float(dst + xx, ld_as_float(src + min(max(xx + sx - pad, 0), w - 1)));
  }
}

template <typename Tout>
__global__ void __launch_bounds__(256) resize_nearest_kernel(const float* __restrict__ x, Tout* __restrict__ out, long long n,
                                                             int hin, int win, int hout, int wout, float sh, float sw) {
  const long long plane = static_cast<long long>(hout) * wout;
  const long long total = n * plane;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long img = i / plane;
    const int yx = static_cast<int>(i - img * plane);
    const int y = yx / wout, xx = yx - y * wout;
    const int ys = min(static_cast<int>(floorf(y * sh)), hin - 1), xs = min(static_cast<int>(floorf(xx * sw)), win - 1);
    st_from_float(out + i, __ldg(x + img * hin * win + static_cast<long long>(ys) * win + xs));
  }
}

// ---- image_fn ----------------------------------------------------------------------------------------------------------------
constexpr int kCrop = 224;                 // CLIP ViT input side
constexpr int kPrecisionBits = 22;         // Pillow Resample.c PRECISION_BITS = 32 - 8 - 2
constexpr int kImageFnMaxSide = 16 * kCrop;  // a downscale of at most 16x keeps one output row's input rows within 48 KB of smem
constexpr int kImageFnSmemCap = 48 * 1024;

// Pillow's bicubic filter (a = -0.5) and the bounds of output pixel xx of a line resized from in_size to out_size
// (Resample.c precompute_coeffs): double arithmetic in Pillow's order.
static double bicubic_filter(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

struct BicubicLine {
  double scale, filterscale, support;
  int taps;
  BicubicLine(int64_t in_size, int64_t out_size) {
    scale = filterscale = static_cast<double>(in_size) / static_cast<double>(out_size);
    if (filterscale < 1.0) filterscale = 1.0;
    support = 2.0 * filterscale;
    taps = static_cast<int>(ceil(support)) * 2 + 1;
  }
  // first input pixel and number of taps of output pixel xx
  void bounds(int64_t in_size, int64_t xx, int* xmin, int* count, double* center) const {
    *center = (xx + 0.5) * scale;
    int lo = static_cast<int>(*center - support + 0.5);
    if (lo < 0) lo = 0;
    int hi = static_cast<int>(*center + support + 0.5);
    if (hi > in_size) hi = static_cast<int>(in_size);
    *xmin = lo;
    *count = hi - lo;
  }
};

// torchvision Resize(224) on the short side + CenterCrop(224): resized size and crop offsets (Python's round, half to even)
static void image_fn_geometry(int64_t h, int64_t w, int64_t* rh, int64_t* rw, int64_t* top, int64_t* left) {
  const int64_t shrt = w <= h ? w : h, lng = w <= h ? h : w;
  const int64_t new_long = static_cast<int64_t>(static_cast<double>(kCrop * lng) / static_cast<double>(shrt));
  *rw = w <= h ? kCrop : new_long;
  *rh = w <= h ? new_long : kCrop;
  auto offset = [](int64_t d) { const int64_t k = d / 2; return (d % 2 == 0 || k % 2 == 0) ? k : k + 1; };
  *top = offset(*rh - kCrop);
  *left = offset(*rw - kCrop);
}

__device__ __forceinline__ uint8_t clip8(int v) {          // Pillow clip8: >> 22 with saturation
  return v <= 0 ? 0 : (v >= (1 << (kPrecisionBits + 8)) ? 255 : static_cast<uint8_t>(v >> kPrecisionBits));
}

template <typename T> struct Vec4;
template <> struct Vec4<float> {
  static __device__ __forceinline__ void store(float* p, float a, float b, float c, float d) {
    *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d);
  }
};
template <> struct Vec4<bf16> {
  static __device__ __forceinline__ void store(bf16* p, float a, float b, float c, float d) {
    __nv_bfloat162 lo = __floats2bfloat162_rn(a, b), hi = __floats2bfloat162_rn(c, d);
    uint2 v;
    v.x = *reinterpret_cast<uint32_t*>(&lo);
    v.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(p) = v;
  }
};

// One CTA = one frame x one band of `band` output rows of the crop.  Horizontal pass: the input rows the band's vertical taps
// reach, only the 224 crop columns, all three channels, rounded to uint8 into shared memory ([3][rows][224]).  Vertical pass:
// four adjacent output columns per thread (uchar4 reads of the staged rows), Normalize through the [3, 256] table, CHW rows
// written as float4 / 4 x bf16.  Table entries are clamped to the frame and the staged rows, so inconsistent tables cannot
// read or write out of bounds.
template <typename Tout>
__global__ void __launch_bounds__(256) image_fn_kernel(const uint8_t* __restrict__ frames, Tout* __restrict__ out, int h, int w,
                                                       const int* __restrict__ xb, const int* __restrict__ xc, int kx,
                                                       const int* __restrict__ yb, const int* __restrict__ yc, int ky,
                                                       const float* __restrict__ lut, int flip, int band, int rows_cap) {
  extern __shared__ __align__(16) unsigned char smem[];
  float* s_lut = reinterpret_cast<float*>(smem);                    // [3][256]
  uint8_t* tmp = smem + 3 * 256 * sizeof(float);                    // [3][rows_cap][224]
  const int bands = kCrop / band;
  const long long img = blockIdx.x / bands;
  const int y0 = static_cast<int>(blockIdx.x % bands) * band, y1 = y0 + band - 1;
  const int r0 = __ldg(yb + 2 * y0);
  const int nrows = max(1, min(__ldg(yb + 2 * y1) + __ldg(yb + 2 * y1 + 1) - r0, rows_cap));
  for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) s_lut[i] = __ldg(lut + i);
  const uint8_t* src = frames + img * h * w * 3;
  const int plane = rows_cap * kCrop;

  for (int i = threadIdx.x; i < nrows * kCrop; i += blockDim.x) {
    const int r = i / kCrop, x = i - r * kCrop;
    const int row = min(max(r0 + r, 0), h - 1);
    const uint8_t* p = src + static_cast<long long>(flip ? h - 1 - row : row) * w * 3;
    const int x0 = __ldg(xb + 2 * x), cnt = __ldg(xb + 2 * x + 1);
    const int* k = xc + x * kx;
    int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
    for (int t = 0; t < min(cnt, kx); ++t) {
      const int c = __ldg(k + t);
      const uint8_t* q = p + min(max(x0 + t, 0), w - 1) * 3;
      s0 += q[0] * c;
      s1 += q[1] * c;
      s2 += q[2] * c;
    }
    tmp[r * kCrop + x] = clip8(s0);
    tmp[plane + r * kCrop + x] = clip8(s1);
    tmp[2 * plane + r * kCrop + x] = clip8(s2);
  }
  __syncthreads();

  constexpr int kQuads = kCrop / 4;
  for (int i = threadIdx.x; i < 3 * band * kQuads; i += blockDim.x) {
    const int q = i % kQuads, cy = i / kQuads;
    const int yy = cy % band, ch = cy / band;
    const int y = y0 + yy;
    const int ys = __ldg(yb + 2 * y) - r0, cnt = __ldg(yb + 2 * y + 1);
    const int* k = yc + y * ky;
    const uint8_t* col = tmp + ch * plane + 4 * q;
    int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0, s3 = s0;
    for (int t = 0; t < min(cnt, ky); ++t) {
      const int c = __ldg(k + t);
      const uchar4 v = *reinterpret_cast<const uchar4*>(col + min(max(ys + t, 0), nrows - 1) * kCrop);
      s0 += v.x * c;
      s1 += v.y * c;
      s2 += v.z * c;
      s3 += v.w * c;
    }
    const float* l = s_lut + ch * 256;
    Vec4<Tout>::store(out + ((img * 3 + ch) * kCrop + y) * kCrop + 4 * q, l[clip8(s0)], l[clip8(s1)], l[clip8(s2)], l[clip8(s3)]);
  }
}

}  // namespace dvla

using namespace dvla;

// dtype codes: 0 = fp32, 1 = bf16
extern "C" int dvla_shift_crop(const void* x, void* out, const int32_t* shifts, int64_t n, int64_t c, int64_t h, int64_t w,
                               int32_t pad, int32_t in_dtype, int32_t out_dtype, void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (n == 0) return DVLA_OK;
  if (!x || !out || !shifts) { set_error("shift_crop: null pointer"); return DVLA_ERR_INVALID; }
  if (n < 0 || c <= 0 || h <= 0 || w <= 0 || pad < 0 || h > 32768 || w > 32768 || c > 65535) { set_error("shift_crop: bad dims"); return DVLA_ERR_INVALID; }
  if ((in_dtype | out_dtype) & ~1) { set_error("shift_crop: dtype codes are 0 (fp32) / 1 (bf16)"); return DVLA_ERR_INVALID; }
  const unsigned g = grid_for(n * c * h * 32, 256, 32);   // one warp per row
#define SC(TI, TO) shift_crop_kernel<TI, TO><<<g, 256, 0, s>>>((const TI*)x, (TO*)out, shifts, n, (int)c, (int)h, (int)w, pad)
  switch (in_dtype * 2 + out_dtype) {
    case 0: SC(float, float); break;
    case 1: SC(float, bf16); break;
    case 2: SC(bf16, float); break;
    default: SC(bf16, bf16); break;
  }
#undef SC
  DVLA_CHECK_LAUNCH("shift_crop");
  return DVLA_OK;
}

extern "C" int dvla_resize_nearest(const float* x, void* out, int64_t n, int64_t hin, int64_t win, int64_t hout, int64_t wout,
                                   int32_t out_dtype, void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (n == 0) return DVLA_OK;
  if (!x || !out) { set_error("resize_nearest: null pointer"); return DVLA_ERR_INVALID; }
  if (n < 0 || hin <= 0 || win <= 0 || hout <= 0 || wout <= 0 || hin > 32768 || win > 32768 || hout > 32768 || wout > 32768) {
    set_error("resize_nearest: bad dims"); return DVLA_ERR_INVALID;
  }
  if (out_dtype & ~1) { set_error("resize_nearest: dtype codes are 0 (fp32) / 1 (bf16)"); return DVLA_ERR_INVALID; }
  if (n == 0) return DVLA_OK;
  const float sh = static_cast<float>(hin) / static_cast<float>(hout), sw = static_cast<float>(win) / static_cast<float>(wout);
  const unsigned g = grid_for(n * hout * wout, 256, 32);
  if (out_dtype == 0) resize_nearest_kernel<float><<<g, 256, 0, s>>>(x, (float*)out, n, (int)hin, (int)win, (int)hout, (int)wout, sh, sw);
  else                resize_nearest_kernel<bf16><<<g, 256, 0, s>>>(x, (bf16*)out, n, (int)hin, (int)win, (int)hout, (int)wout, sh, sw);
  DVLA_CHECK_LAUNCH("resize_nearest");
  return DVLA_OK;
}

extern "C" int32_t dvla_bicubic_taps(int64_t in_size, int64_t out_size) {
  if (in_size <= 0 || out_size <= 0 || in_size > (1 << 20) || out_size > (1 << 20)) {
    set_error("bicubic_taps: sizes must be in [1, 2^20]"); return DVLA_ERR_INVALID;
  }
  return in_size == out_size ? 1 : BicubicLine(in_size, out_size).taps;
}

extern "C" int dvla_bicubic_coeffs(int64_t in_size, int64_t out_size, int64_t first, int64_t count, int32_t* bounds,
                                   int32_t* coeffs) {
  const int taps = dvla_bicubic_taps(in_size, out_size);
  if (taps < 0) return taps;
  if (!bounds || !coeffs) { set_error("bicubic_coeffs: null pointer"); return DVLA_ERR_INVALID; }
  if (first < 0 || count < 0 || first + count > out_size) { set_error("bicubic_coeffs: outputs out of range"); return DVLA_ERR_INVALID; }
  const BicubicLine line(in_size, out_size);
  const double ss = 1.0 / line.filterscale;
  for (int64_t i = 0; i < count; ++i) {
    int32_t* c = coeffs + i * taps;
    for (int t = 0; t < taps; ++t) c[t] = 0;
    if (in_size == out_size) {                             // Pillow skips the pass: the identity
      bounds[2 * i] = static_cast<int32_t>(first + i);
      bounds[2 * i + 1] = 1;
      c[0] = 1 << kPrecisionBits;
      continue;
    }
    int xmin, n;
    double center;
    line.bounds(in_size, first + i, &xmin, &n, &center);
    double ww = 0.0;
    for (int x = 0; x < n; ++x) ww += bicubic_filter((x + xmin - center + 0.5) * ss);
    for (int x = 0; x < n; ++x) {
      const double f = bicubic_filter((x + xmin - center + 0.5) * ss);     // the same value again: no scratch buffer
      const double v = ww != 0.0 ? f / ww : f;
      c[x] = static_cast<int32_t>(v < 0 ? -0.5 + v * (1 << kPrecisionBits) : 0.5 + v * (1 << kPrecisionBits));
    }
    bounds[2 * i] = xmin;
    bounds[2 * i + 1] = n;
  }
  return DVLA_OK;
}

extern "C" int dvla_image_fn(const dvla_image_fn_args* a, void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!a) { set_error("image_fn: null args"); return DVLA_ERR_INVALID; }
  if (a->n == 0) return DVLA_OK;
  if (!a->frames || !a->out || !a->xbounds || !a->xcoeffs || !a->ybounds || !a->ycoeffs || !a->lut) {
    set_error("image_fn: null pointer"); return DVLA_ERR_INVALID;
  }
  if (a->c != 3) { set_error("image_fn: frames must have 3 channels (8-bit RGB), got %lld", (long long)a->c); return DVLA_ERR_INVALID; }
  if (a->n < 0 || a->n > (1LL << 24) || a->h <= 0 || a->w <= 0 || a->h > kImageFnMaxSide || a->w > kImageFnMaxSide) {
    set_error("image_fn: bad dims (n=%lld, h=%lld, w=%lld; sides must be in [1, %d])", (long long)a->n, (long long)a->h,
              (long long)a->w, kImageFnMaxSide);
    return DVLA_ERR_INVALID;
  }
  if (a->out_dtype & ~1) { set_error("image_fn: dtype codes are 0 (fp32) / 1 (bf16)"); return DVLA_ERR_INVALID; }
  if (!aligned16(a->out)) { set_error("image_fn: out must be 16-byte aligned"); return DVLA_ERR_INVALID; }
  int64_t rh, rw, top, left;
  image_fn_geometry(a->h, a->w, &rh, &rw, &top, &left);
  const int kx = dvla_bicubic_taps(a->w, rw), ky = dvla_bicubic_taps(a->h, rh);
  // the largest band of output rows whose staged input rows fit the shared-memory budget (bounds as dvla_bicubic_coeffs gives them)
  const BicubicLine line(a->h, rh);
  auto row_bound = [&](int y, bool end) {                    // first input row output row y reads, or (end) one past its last
    if (a->h == rh) return static_cast<int>(top + y) + (end ? 1 : 0);
    int lo, n; double c;
    line.bounds(a->h, top + y, &lo, &n, &c);
    return end ? lo + n : lo;
  };
  int band = 0, rows_cap = 0;
  for (int cand = 32; cand >= 1 && !band; cand /= 2) {
    int need = 0;
    for (int y0 = 0; y0 < kCrop; y0 += cand) need = max(need, row_bound(y0 + cand - 1, true) - row_bound(y0, false));
    if (3 * 256 * 4 + 3 * need * kCrop <= kImageFnSmemCap) band = cand, rows_cap = need;
  }
  if (!band) { set_error("image_fn: %lldx%lld frames need more shared memory than supported", (long long)a->h, (long long)a->w); return DVLA_ERR_UNSUPPORTED; }
  const long long grid = a->n * (kCrop / band);
  const size_t smem = 3 * 256 * 4 + 3 * static_cast<size_t>(rows_cap) * kCrop;
#define IF(T) image_fn_kernel<T><<<static_cast<unsigned>(grid), 256, smem, s>>>(a->frames, (T*)a->out, (int)a->h, (int)a->w, a->xbounds, \
      a->xcoeffs, kx, a->ybounds, a->ycoeffs, ky, a->lut, a->flip_vertical ? 1 : 0, band, rows_cap)
  if (a->out_dtype == 0) IF(float);
  else                   IF(bf16);
#undef IF
  DVLA_CHECK_LAUNCH("image_fn");
  return DVLA_OK;
}
