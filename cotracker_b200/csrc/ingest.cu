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
// YUV read (NV12, I420, YUYV) that loads the pixel's Y and its shared chroma and applies cv2's integer BT.601
// conversion (ct3_prepare_frames_yuv).  The resize, copy and normalisation are this one piece of code for both, so a
// YUV clip gives exactly the floats its uint8 RGB conversion would.
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

// YuvFetch<L>: uint8 YUV frames of layout L (CT3_YUV_*) at byte strides st (frame) and sr (row), converted to RGB as
// cv2.cvtColor(COLOR_YUV2RGB_*) does (BT.601 limited range, Q20 integers; the formula is in include/ct3_b200.h).
// uv: the byte offset of the chroma in a frame (NV12: H rows; I420: the U plane at H*W, V a quarter plane further).
template <int L>
struct YuvFetch {
  using Src = uint8_t;
  int64_t sr, uv, quarter;

  __device__ __forceinline__ void pixel(const uint8_t* f, int y, int x, float (&v)[3]) const {
    int Y, U, V;
    if (L == CT3_YUV_NV12) {
      Y = __ldg(f + y * sr + x);
      const uint8_t* c = f + uv + (y >> 1) * sr + (x & ~1);
      U = __ldg(c);
      V = __ldg(c + 1);
    } else if (L == CT3_YUV_I420) {   // rows are dense: sr == W
      Y = __ldg(f + y * sr + x);
      const int64_t c = uv + (y >> 1) * (sr >> 1) + (x >> 1);
      U = __ldg(f + c);
      V = __ldg(f + c + quarter);
    } else {   // YUYV: Y0 U Y1 V per pixel pair
      const uint8_t* p = f + y * sr + 2 * (x & ~1);
      Y = __ldg(p + 2 * (x & 1));
      U = __ldg(p + 1);
      V = __ldg(p + 3);
    }
    const int yy = max(Y - 16, 0) * 1220542, u = U - 128, w = V - 128;
    v[0] = (float)min(max((yy + 1673527 * w + (1 << 19)) >> 20, 0), 255);
    v[1] = (float)min(max((yy - 852492 * w - 409993 * u + (1 << 19)) >> 20, 0), 255);
    v[2] = (float)min(max((yy + 2116026 * u + (1 << 19)) >> 20, 0), 255);
  }
  // the 2x2 neighbourhood, converted up front: a pixel's three channels come from the same loads
  struct Quad {
    float p[4][3];
    __device__ __forceinline__ float at(int c, int k) const { return p[k][c]; }
  };
  __device__ __forceinline__ Quad quad(const uint8_t* f, int y, int x, int dy, int dx) const {
    Quad q;
    pixel(f, y, x, q.p[0]);
    pixel(f, y, x + dx, q.p[1]);
    pixel(f, y + dy, x, q.p[2]);
    pixel(f, y + dy, x + dx, q.p[3]);
    return q;
  }
};

template <class Fetch>
__global__ void __launch_bounds__(kPrepThreads) prepare_frames_kernel(const typename Fetch::Src* __restrict__ src,
                                                                      int64_t st, const Fetch fetch, int H, int W,
                                                                      int oh, int ow, float rh, float rw, int copy,
                                                                      float inv255, float* __restrict__ out) {
  const int64_t p = (int64_t)blockIdx.x * kPrepThreads + threadIdx.x;
  const int64_t plane = (int64_t)oh * ow;   // <= INT32_MAX (ct3_prepare_frames*), so y and x fit in int
  if (p >= plane) return;
  const int t = blockIdx.y;
  const int y = (int)(p / ow), x = (int)(p - (int64_t)y * ow);
  const typename Fetch::Src* f = src + (int64_t)t * st;
  float v[3];
  if (copy) {
    fetch.pixel(f, y, x, v);
  } else {
    const float h1r = __fmul_rn(rh, (float)y);
    const int h1 = (int)h1r;
    const int h1p = h1 < H - 1 ? 1 : 0;
    const float h1l = __fsub_rn(h1r, (float)h1);
    const float h0l = __fsub_rn(1.0f, h1l);
    const float w1r = __fmul_rn(rw, (float)x);
    const int w1 = (int)w1r;
    const int w1p = w1 < W - 1 ? 1 : 0;
    const float w1l = __fsub_rn(w1r, (float)w1);
    const float w0l = __fsub_rn(1.0f, w1l);
    const auto q = fetch.quad(f, h1, w1, h1p, w1p);
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
cudaError_t launch_fetch(const typename Fetch::Src* src, int64_t st, const Fetch& fetch, int T, int H, int W, int oh,
                         int ow, float* out, cudaStream_t s) {
  // area_pixel_compute_scale<float>(in, out, align_corners=true): float / int in float
  const float rh = oh > 1 ? (float)(H - 1) / (oh - 1) : 0.0f;
  const float rw = ow > 1 ? (float)(W - 1) / (ow - 1) : 0.0f;
  const int copy = (H == oh && W == ow) ? 1 : 0;
  const float inv255 = 1.0f / 255.0f;
  const int64_t plane = (int64_t)oh * ow;
  const unsigned gx = (unsigned)((plane + kPrepThreads - 1) / kPrepThreads);
  for (int t0 = 0; t0 < T; t0 += kMaxGridY) {
    const int tc = (T - t0) < kMaxGridY ? (T - t0) : kMaxGridY;
    prepare_frames_kernel<Fetch><<<dim3(gx, tc), kPrepThreads, 0, s>>>(src + (int64_t)t0 * st, st, fetch, H, W, oh, ow,
                                                                      rh, rw, copy, inv255,
                                                                      out + (int64_t)t0 * 3 * plane);
  }
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_prepare_frames(const void* src, int dtype, int T, int H, int W, int64_t st, int64_t sc, int64_t sh,
                                  int64_t sw, int oh, int ow, float* out, cudaStream_t s) {
  if (dtype == CT3_FRAMES_U8)
    return launch_fetch(static_cast<const uint8_t*>(src), st, RgbFetch<uint8_t>{sc, sh, sw}, T, H, W, oh, ow, out, s);
  return launch_fetch(static_cast<const float*>(src), st, RgbFetch<float>{sc, sh, sw}, T, H, W, oh, ow, out, s);
}

cudaError_t launch_prepare_frames_yuv(const uint8_t* src, int layout, int T, int H, int W, int64_t st, int64_t sr,
                                      int oh, int ow, float* out, cudaStream_t s) {
  if (layout == CT3_YUV_NV12)
    return launch_fetch(src, st, YuvFetch<CT3_YUV_NV12>{sr, (int64_t)H * sr, 0}, T, H, W, oh, ow, out, s);
  if (layout == CT3_YUV_I420) {
    const int64_t quarter = (int64_t)(H / 2) * (W / 2);
    return launch_fetch(src, st, YuvFetch<CT3_YUV_I420>{sr, (int64_t)H * W, quarter}, T, H, W, oh, ow, out, s);
  }
  return launch_fetch(src, st, YuvFetch<CT3_YUV_YUYV>{sr, 0, 0}, T, H, W, oh, ow, out, s);
}

}  // namespace ct3
