// ingest.cu -- raw frames -> encoder input in one pass: bilinear resize (align_corners=True) of a strided uint8 or fp32
// clip [T,3,H,W] to [T,3,oh,ow] fp32, then [0,255] -> [-1,1] (reference predictor.py:60-64 + cotracker3_offline.py:63).
//
// The result is bit-identical to
//     2.0 * (F.interpolate(src.float(), (oh, ow), mode="bilinear", align_corners=True) / 255.0) - 1.0
// on the GPU, so the arithmetic is ATen's, step by step (every rounding made explicit with __f*_rn intrinsics, so
// nvcc cannot contract differently):
//   - scale (float)(in - 1) / (out - 1) (0 when out == 1), computed on the host (area_pixel_compute_scale);
//   - source index scale * dst, i0 = (int)src, neighbour offset i0 < in - 1, l1 = src - i0, l0 = 1 - l1;
//   - the blend as upsample_bilinear2d_out_frame<float, float> is compiled for sm_90 (its SASS):
//         fma(h0, fma(w0, a, w1 * b), h1 * fma(w0, c, w1 * d))
//     With 3 channels ATen always runs that kernel (the NHWC one needs more channels), whatever the input strides;
//   - a same-size resize is ATen's plain copy;
//   - x / 255.0 with a CPU scalar divisor is x * (1.0f / 255.0f) in ATen (div_true_kernel_cuda multiplies by the
//     reciprocal), then * 2 (exact) and - 1.
//
// The kernel is templated on how it reads one source pixel's three channels (a "fetch"): the strided RGB read, or a
// YUV read that loads the pixel's Y and its shared chroma (semi-planar, planar or packed, 8- or 16-bit samples) and
// applies the integer conversion of ct3_prepare_frames_yuv_fmt (cv2's BT.601 constants by default).  The resize, copy
// and normalisation are this one piece of code for all of them, so a YUV clip gives exactly the floats its uint8 RGB
// conversion would.
//
// The kernel optionally reads a crop_h x crop_w window of each frame at a per-frame (top, left) from the device
// (kCrop, ct3_prepare_frames_crop / ct3_prepare_frames_yuv_crop): the resize is that of a crop_h x crop_w frame and the
// offset moves only the integer sample indices, so the output is the un-cropped kernel's on the materialised window.
// Without kCrop the template makes exactly the code it made before windows existed.
#include "../../include/ct3_b200.h"
#include "kernels.cuh"

namespace ct3 {
namespace {

constexpr int kPrepThreads = 256;
constexpr int kMaxGridY = 65535;

template <typename Tin>
__device__ __forceinline__ float px(const Tin* p) { return static_cast<float>(__ldg(p)); }

// A fetch is how the kernel reads a source pixel's three channels from frame f: pixel() for the same-size copy, quad()
// for the bilinear 2x2 neighbourhood, whose at(c, k) gives channel c of corner k in the order the blend uses them.
// With the RGB fetch the kernel makes the loads and arithmetic of the strided RGB kernel it replaced, in that order.
//
// RgbFetch: [T,3,H,W] frames of Tin at element strides (st, sc, sh, sw).
template <typename Tin>
struct RgbFetch {
  using Src = Tin;
  int64_t sc, sh, sw;

  __device__ __forceinline__ void pixel(const Tin* f, int y, int x, float (&v)[3]) const {
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = px(f + c * sc + y * sh + x * sw);
  }
  // corners (y, x), (y, x + dx), (y + dy, x), (y + dy, x + dx); at(c, k) loads when the blend asks for it
  struct Quad {
    const Tin* f;
    int64_t sc, o[4];
    __device__ __forceinline__ float at(int c, int k) const { return px(f + c * sc + o[k]); }
  };
  __device__ __forceinline__ Quad quad(const Tin* f, int y, int x, int dy, int dx) const {
    const int64_t o00 = y * sh + x * sw, o01 = o00 + dx * sw, o10 = o00 + dy * sh, o11 = o10 + dx * sw;
    return {f, sc, {o00, o01, o10, o11}};
  }
};

// A YUV fetch is a read family (how a pixel's Y and its shared U, V are found in a frame) and a colour (how they
// become RGB).  Strides and offsets are in samples of the family's type S (uint8_t or uint16_t).
//
// SemiPlanarRead: NV12, P010, P016: H luma rows, then H/2 rows of interleaved U,V, at row stride sr; uv = H * sr.
template <typename S>
struct SemiPlanarRead {
  using Src = S;
  int64_t sr, uv;
  __device__ __forceinline__ void load(const S* f, int y, int x, int& Y, int& U, int& V) const {
    Y = __ldg(f + y * sr + x);
    const S* c = f + uv + (y >> 1) * sr + (x & ~1);
    U = __ldg(c);
    V = __ldg(c + 1);
  }
};

// PlanarRead<S, XS, YS>: I420 (1, 1), YUV422P (1, 0), YUV444P (0, 0) and their 10-bit forms: the Y plane (rows dense,
// sr == W), then the U plane at uv = H * W and the V plane cplane further, chroma rows of W >> XS samples; a chroma
// sample covers 2^XS x 2^YS pixels.  The shifts are compile-time, so I420 makes the loads and index arithmetic of the
// I420 read this replaced.
template <typename S, int XS, int YS>
struct PlanarRead {
  using Src = S;
  int64_t sr, uv, cplane;
  __device__ __forceinline__ void load(const S* f, int y, int x, int& Y, int& U, int& V) const {
    Y = __ldg(f + y * sr + x);
    const int64_t c = uv + (y >> YS) * (sr >> XS) + (x >> XS);
    U = __ldg(f + c);
    V = __ldg(f + c + cplane);
  }
};

// PackedRead: YUYV, H rows of W/2 pixel pairs Y0 U Y1 V at row stride sr.
template <typename S>
struct PackedRead {
  using Src = S;
  int64_t sr;
  __device__ __forceinline__ void load(const S* f, int y, int x, int& Y, int& U, int& V) const {
    const S* p = f + y * sr + 2 * (x & ~1);
    Y = __ldg(p + 2 * (x & 1));
    U = __ldg(p + 1);
    V = __ldg(p + 3);
  }
};

__device__ __forceinline__ float clamp255(long long x) { return (float)(int)min(max(x, 0ll), 255ll); }

// Cv2Bt601: cv2's BT.601 limited-range conversion of 8-bit samples, the default colour, with its Q20 constants
// compiled in (every term fits int32).
struct Cv2Bt601 {
  __device__ __forceinline__ void rgb(int Y, int U, int V, float (&v)[3]) const {
    const int yy = max(Y - 16, 0) * 1220542, u = U - 128, w = V - 128;
    v[0] = (float)min(max((yy + 1673527 * w + (1 << 19)) >> 20, 0), 255);
    v[1] = (float)min(max((yy - 852492 * w - 409993 * u + (1 << 19)) >> 20, 0), 255);
    v[2] = (float)min(max((yy + 2116026 * u + (1 << 19)) >> 20, 0), 255);
  }
};

// YuvCoeffs: any layout and colour, the formula of ct3_prepare_frames_yuv_fmt in int64 (yuv_coeffs() below).  A
// container value c holds the sample (c >> rshift) & mask.
struct YuvCoeffs {
  int rshift, mask, yoff, ylo, coff, shift;
  long long cy, crv, cgv, cgu, cbu;
  __device__ __forceinline__ void rgb(int Y, int U, int V, float (&v)[3]) const {
    Y = (Y >> rshift) & mask;
    U = (U >> rshift) & mask;
    V = (V >> rshift) & mask;
    const long long yy = max(Y - yoff, ylo) * cy, u = U - coff, w = V - coff, h = 1ll << (shift - 1);
    v[0] = clamp255((yy + crv * w + h) >> shift);
    v[1] = clamp255((yy - cgv * w - cgu * u + h) >> shift);
    v[2] = clamp255((yy + cbu * u + h) >> shift);
  }
};

template <class Read, class Color>
struct YuvFetch {
  using Src = typename Read::Src;
  Read read;
  Color color;

  __device__ __forceinline__ void pixel(const Src* f, int y, int x, float (&v)[3]) const {
    int Y, U, V;
    read.load(f, y, x, Y, U, V);
    color.rgb(Y, U, V, v);
  }
  // the 2x2 neighbourhood, converted up front: a pixel's three channels come from the same loads
  struct Quad {
    float p[4][3];
    __device__ __forceinline__ float at(int c, int k) const { return p[k][c]; }
  };
  __device__ __forceinline__ Quad quad(const Src* f, int y, int x, int dy, int dx) const {
    Quad q;
    pixel(f, y, x, q.p[0]);
    pixel(f, y, x + dx, q.p[1]);
    pixel(f, y + dy, x, q.p[2]);
    pixel(f, y + dy, x + dx, q.p[3]);
    return q;
  }
};

// The window of a launch: frames H x W, resized from a window ch x cw whose top-left corner in frame t is
// (offsets[2t], offsets[2t + 1]) (kCrop), or from the whole frame (ch = H, cw = W, no offsets).
struct Geom {
  int T, H, W, ch, cw, oh, ow;
  const int32_t* offsets;   // device [T,2] (top, left), or null for the whole frame
};

// A window sample index: r + o, clamped into [0, n - 1] so that an offset the host did not check never reads outside
// the frame (int64: o is any int32).
__device__ __forceinline__ int clamp_index(int r, int o, int n) {
  return (int)min(max((long long)r + o, 0ll), (long long)n - 1);
}

template <class Fetch, bool kCrop>
__global__ void __launch_bounds__(kPrepThreads) prepare_frames_kernel(const typename Fetch::Src* __restrict__ src,
                                                                      int64_t st, const Fetch fetch,
                                                                      const int32_t* __restrict__ offsets, int H, int W,
                                                                      int ch, int cw, int oh, int ow, float rh,
                                                                      float rw, int copy, float inv255,
                                                                      float* __restrict__ out) {
  const int64_t p = (int64_t)blockIdx.x * kPrepThreads + threadIdx.x;
  const int64_t plane = (int64_t)oh * ow;   // <= INT32_MAX (ct3_prepare_frames*), so y and x fit in int
  if (p >= plane) return;
  const int t = blockIdx.y;
  const int y = (int)(p / ow), x = (int)(p - (int64_t)y * ow);
  const typename Fetch::Src* f = src + (int64_t)t * st;
  int top = 0, left = 0;
  if constexpr (kCrop) {
    top = __ldg(offsets + 2 * t);
    left = __ldg(offsets + 2 * t + 1);
  }
  float v[3];
  if (copy) {
    if constexpr (kCrop)
      fetch.pixel(f, clamp_index(y, top, H), clamp_index(x, left, W), v);
    else
      fetch.pixel(f, y, x, v);
  } else {
    // ATen's source indices of a ch x cw frame; the window's offset moves the integer samples only
    const float h1r = __fmul_rn(rh, (float)y);
    const int h1 = (int)h1r;
    const int h1p = h1 < ch - 1 ? 1 : 0;
    const float h1l = __fsub_rn(h1r, (float)h1);
    const float h0l = __fsub_rn(1.0f, h1l);
    const float w1r = __fmul_rn(rw, (float)x);
    const int w1 = (int)w1r;
    const int w1p = w1 < cw - 1 ? 1 : 0;
    const float w1l = __fsub_rn(w1r, (float)w1);
    const float w0l = __fsub_rn(1.0f, w1l);
    typename Fetch::Quad q;
    if constexpr (kCrop) {
      const int y0 = clamp_index(h1, top, H), x0 = clamp_index(w1, left, W);
      q = fetch.quad(f, y0, x0, clamp_index(h1 + h1p, top, H) - y0, clamp_index(w1 + w1p, left, W) - x0);
    } else {
      q = fetch.quad(f, h1, w1, h1p, w1p);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float row0 = __fmaf_rn(w0l, q.at(c, 0), __fmul_rn(w1l, q.at(c, 1)));
      const float row1 = __fmaf_rn(w0l, q.at(c, 2), __fmul_rn(w1l, q.at(c, 3)));
      v[c] = __fmaf_rn(h0l, row0, __fmul_rn(h1l, row1));
    }
  }
  float* o = out + (int64_t)t * 3 * plane + p;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c * plane] = __fsub_rn(__fmul_rn(2.0f, __fmul_rn(v[c], inv255)), 1.0f);
}

template <class Fetch>
cudaError_t launch_fetch(const typename Fetch::Src* src, int64_t st, const Fetch& fetch, const Geom& g, float* out,
                         cudaStream_t s) {
  // area_pixel_compute_scale<float>(in, out, align_corners=true): float / int in float, in = the window
  const float rh = g.oh > 1 ? (float)(g.ch - 1) / (g.oh - 1) : 0.0f;
  const float rw = g.ow > 1 ? (float)(g.cw - 1) / (g.ow - 1) : 0.0f;
  const int copy = (g.ch == g.oh && g.cw == g.ow) ? 1 : 0;
  const float inv255 = 1.0f / 255.0f;
  const int64_t plane = (int64_t)g.oh * g.ow;
  const unsigned gx = (unsigned)((plane + kPrepThreads - 1) / kPrepThreads);
  for (int t0 = 0; t0 < g.T; t0 += kMaxGridY) {
    const int tc = (g.T - t0) < kMaxGridY ? (g.T - t0) : kMaxGridY;
    const dim3 grid(gx, tc);
    const auto* s0 = src + (int64_t)t0 * st;
    float* o0 = out + (int64_t)t0 * 3 * plane;
    if (g.offsets)
      prepare_frames_kernel<Fetch, true><<<grid, kPrepThreads, 0, s>>>(s0, st, fetch, g.offsets + 2 * (int64_t)t0, g.H,
                                                                       g.W, g.ch, g.cw, g.oh, g.ow, rh, rw, copy,
                                                                       inv255, o0);
    else
      prepare_frames_kernel<Fetch, false><<<grid, kPrepThreads, 0, s>>>(s0, st, fetch, nullptr, g.H, g.W, g.ch, g.cw,
                                                                        g.oh, g.ow, rh, rw, copy, inv255, o0);
  }
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_prepare_frames(const void* src, int dtype, int T, int H, int W, int64_t st, int64_t sc, int64_t sh,
                                  int64_t sw, const int32_t* offsets, int ch, int cw, int oh, int ow, float* out,
                                  cudaStream_t s) {
  const Geom g{T, H, W, ch, cw, oh, ow, offsets};
  if (dtype == CT3_FRAMES_U8)
    return launch_fetch(static_cast<const uint8_t*>(src), st, RgbFetch<uint8_t>{sc, sh, sw}, g, out, s);
  return launch_fetch(static_cast<const float*>(src), st, RgbFetch<float>{sc, sh, sw}, g, out, s);
}

namespace {

// The coefficients of ct3_prepare_frames_yuv_fmt (include/ct3_b200.h) for one layout and colour: cv2's constants for
// BT.601 limited range, otherwise each derived exactly from Kr, Kb (in 1e-4) and rounded half up at Q = 48.
YuvCoeffs yuv_coeffs(const YuvFormat& f, int matrix, int full_range) {
  constexpr int kQ = 48;
  const int n = f.bits, s = 1 << (n - 8);
  YuvCoeffs k;
  k.rshift = f.msb ? 16 - n : 0;
  k.mask = (1 << n) - 1;
  if (matrix == CT3_MATRIX_BT601 && !full_range) {
    k.yoff = 16 * s, k.ylo = 0, k.coff = 128 * s, k.shift = 20 + n - 8;
    k.cy = 1220542, k.crv = 1673527, k.cgv = 852492, k.cgu = 409993, k.cbu = 2116026;
    return k;
  }
  static const long long kKrKb[3][2] = {{2990, 1140}, {2126, 722}, {2627, 593}};
  const long long kr = kKrKb[matrix][0], kb = kKrKb[matrix][1], kg = 10000 - kr - kb;
  long long dy, dc;
  if (full_range) {
    k.yoff = 0, k.coff = 1 << (n - 1), dy = dc = (1ll << n) - 1;
  } else {
    k.yoff = 16 * s, k.coff = 128 * s, dy = 219ll * s, dc = 224ll * s;
  }
  k.ylo = -k.yoff, k.shift = kQ;
  // num / den * 2^Q rounded half up: num < 2^37 and den < 2^47, so num * 2^(Q+1) + den fits 128 bits
  auto q = [](long long num, long long den) {
    using u128 = unsigned __int128;
    return (long long)((((u128)num << (kQ + 1)) + (u128)den) / (2 * (u128)den));
  };
  k.cy = q(255, dy);
  k.crv = q(510 * (10000 - kr), 10000 * dc);
  k.cgv = q(510 * kr * (10000 - kr), 10000 * kg * dc);
  k.cgu = q(510 * kb * (10000 - kb), 10000 * kg * dc);
  k.cbu = q(510 * (10000 - kb), 10000 * dc);
  return k;
}

// Launch the fetch of one read family: 8-bit samples in cv2's BT.601 limited range take the compiled-in constants,
// everything else the runtime coefficients.
template <class Read>
cudaError_t launch_read(const void* src, int64_t st, const Read& read, const YuvFormat& f, int matrix, int full_range,
                        const Geom& g, float* out, cudaStream_t s) {
  using S = typename Read::Src;
  const S* p = static_cast<const S*>(src);
  if constexpr (sizeof(S) == 1) {
    if (matrix == CT3_MATRIX_BT601 && !full_range)
      return launch_fetch(p, st, YuvFetch<Read, Cv2Bt601>{read, {}}, g, out, s);
  }
  return launch_fetch(p, st, YuvFetch<Read, YuvCoeffs>{read, yuv_coeffs(f, matrix, full_range)}, g, out, s);
}

template <typename S>
cudaError_t launch_family(const void* src, const YuvFormat& f, int matrix, int full_range, const Geom& g, int64_t st,
                          int64_t sr, float* out, cudaStream_t s) {
  st /= (int64_t)sizeof(S), sr /= (int64_t)sizeof(S);   // byte strides -> sample strides (validated multiples)
  if (f.family == YuvFormat::kSemiPlanar)
    return launch_read(src, st, SemiPlanarRead<S>{sr, (int64_t)g.H * sr}, f, matrix, full_range, g, out, s);
  if (f.family == YuvFormat::kPlanar) {
    const int64_t uv = (int64_t)g.H * g.W, cplane = (int64_t)(g.H >> f.ys) * (g.W >> f.xs);
    if (f.ys) return launch_read(src, st, PlanarRead<S, 1, 1>{sr, uv, cplane}, f, matrix, full_range, g, out, s);
    if (f.xs) return launch_read(src, st, PlanarRead<S, 1, 0>{sr, uv, cplane}, f, matrix, full_range, g, out, s);
    return launch_read(src, st, PlanarRead<S, 0, 0>{sr, uv, cplane}, f, matrix, full_range, g, out, s);
  }
  if constexpr (sizeof(S) == 1)   // YUYV is the only packed layout
    return launch_read(src, st, PackedRead<S>{sr}, f, matrix, full_range, g, out, s);
  return cudaErrorInvalidValue;
}

}  // namespace

cudaError_t launch_prepare_frames_yuv(const void* src, int layout, int matrix, int full_range, int T, int H, int W,
                                      int64_t st, int64_t sr, const int32_t* offsets, int ch, int cw, int oh, int ow,
                                      float* out, cudaStream_t s) {
  const YuvFormat& f = *yuv_format(layout);
  const Geom g{T, H, W, ch, cw, oh, ow, offsets};
  if (f.bytes == 1) return launch_family<uint8_t>(src, f, matrix, full_range, g, st, sr, out, s);
  return launch_family<uint16_t>(src, f, matrix, full_range, g, st, sr, out, s);
}

}  // namespace ct3
