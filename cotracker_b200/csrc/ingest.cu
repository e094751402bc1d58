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
#include "../../include/ct3_b200.h"
#include "kernels.cuh"

namespace ct3 {
namespace {

constexpr int kPrepThreads = 256;
constexpr int kMaxGridY = 65535;

template <typename Tin>
__device__ __forceinline__ float px(const Tin* p) { return static_cast<float>(__ldg(p)); }

template <typename Tin>
__global__ void __launch_bounds__(kPrepThreads) prepare_frames_kernel(const Tin* __restrict__ src, int64_t st,
                                                                      int64_t sc, int64_t sh, int64_t sw, int H, int W,
                                                                      int oh, int ow, float rh, float rw, int copy,
                                                                      float inv255, float* __restrict__ out) {
  const int64_t p = (int64_t)blockIdx.x * kPrepThreads + threadIdx.x;
  const int64_t plane = (int64_t)oh * ow;   // <= INT32_MAX (ct3_prepare_frames), so y and x fit in int
  if (p >= plane) return;
  const int t = blockIdx.y;
  const int y = (int)(p / ow), x = (int)(p - (int64_t)y * ow);
  const Tin* f = src + (int64_t)t * st;
  float v[3];
  if (copy) {
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = px(f + c * sc + y * sh + x * sw);
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
    const int64_t o00 = h1 * sh + w1 * sw, o01 = o00 + w1p * sw, o10 = o00 + h1p * sh, o11 = o10 + w1p * sw;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const Tin* fc = f + c * sc;
      const float row0 = __fmaf_rn(w0l, px(fc + o00), __fmul_rn(w1l, px(fc + o01)));
      const float row1 = __fmaf_rn(w0l, px(fc + o10), __fmul_rn(w1l, px(fc + o11)));
      v[c] = __fmaf_rn(h0l, row0, __fmul_rn(h1l, row1));
    }
  }
  float* o = out + (int64_t)t * 3 * plane + p;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c * plane] = __fsub_rn(__fmul_rn(2.0f, __fmul_rn(v[c], inv255)), 1.0f);
}

template <typename Tin>
cudaError_t launch_typed(const Tin* src, int T, int H, int W, int64_t st, int64_t sc, int64_t sh, int64_t sw, int oh,
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
    prepare_frames_kernel<Tin><<<dim3(gx, tc), kPrepThreads, 0, s>>>(src + (int64_t)t0 * st, st, sc, sh, sw, H, W, oh,
                                                                     ow, rh, rw, copy, inv255,
                                                                     out + (int64_t)t0 * 3 * plane);
  }
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_prepare_frames(const void* src, int dtype, int T, int H, int W, int64_t st, int64_t sc, int64_t sh,
                                  int64_t sw, int oh, int ow, float* out, cudaStream_t s) {
  if (dtype == CT3_FRAMES_U8)
    return launch_typed(static_cast<const uint8_t*>(src), T, H, W, st, sc, sh, sw, oh, ow, out, s);
  return launch_typed(static_cast<const float*>(src), T, H, W, st, sc, sh, sw, oh, ow, out, s);
}

}  // namespace ct3
