// prep.cu -- per-clip preparation around the hot loop:
//   * prepare_pyramid : L2-normalise fnet output over channels, re-lay channels-last, 3x 2x2 average pool
//                       (cotracker3_offline.py:92-117)
//   * sample_support  : 7x7 bilinear support features of every track at its query frame, all levels
//                       (get_track_feat, cotracker3_online.py:113-128 -> sample_features5d, model_utils.py:293-323)
// Layout decision: the reference keeps feature maps channel-planar [T,128,H,W] -- the worst case for the
// per-track gathers of the hot loop.  Here a texel is 128 contiguous floats (one 512-byte line), so every
// bilinear tap is one fully coalesced warp-wide float4 load.
#include "kernels.cuh"

namespace ct3 {

PyramidLayout pyramid_layout(int T, int H4, int W4) {
  PyramidLayout p;
  int h = H4, w = W4;
  int64_t off = 0;
  for (int l = 0; l < kL; ++l) {
    p.off[l] = off;
    p.h[l] = h;
    p.w[l] = w;
    off += (int64_t)T * h * w * kD;
    h /= 2;  // F.avg_pool2d(kernel 2, stride 2) floors odd sizes
    w /= 2;
  }
  p.total = off;
  return p;
}

namespace {

// block: 32 consecutive x of one (t,y) row, all 128 channels.  256 threads.
__global__ void __launch_bounds__(256)
normalize_to_channels_last_kernel(const float* __restrict__ in, float* __restrict__ out, int T, int H, int W) {
  __shared__ float tile[kD][33];
  const int x0 = blockIdx.x * 32, y = blockIdx.y, t = blockIdx.z;
  for (int i = threadIdx.x; i < kD * 32; i += 256) {
    const int c = i >> 5, xi = i & 31;
    const int x = x0 + xi;
    tile[c][xi] = (x < W) ? in[(((int64_t)t * kD + c) * H + y) * W + x] : 0.f;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int px = warp; px < 32; px += 8) {
    const int x = x0 + px;
    float v[4], ss = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      v[k] = tile[lane * 4 + k][px];
      ss += v[k] * v[k];
    }
    ss = warp_sum(ss);
    const float denom = sqrtf(fmaxf(ss, 1e-12f));
    if (x < W) {
      float4 o = make_float4(v[0] / denom, v[1] / denom, v[2] / denom, v[3] / denom);
      reinterpret_cast<float4*>(out + (((int64_t)t * H + y) * W + x) * kD)[lane] = o;
    }
  }
}

// channels-last 2x2 average pool; one thread = one float4 of one output texel
__global__ void avgpool2_channels_last_kernel(const float* __restrict__ in, float* __restrict__ out, int T, int Hi,
                                              int Wi, int Ho, int Wo) {
  const int64_t total = (int64_t)T * Ho * Wo * (kD / 4);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % (kD / 4));
    int64_t r = i / (kD / 4);
    const int x = (int)(r % Wo);
    r /= Wo;
    const int y = (int)(r % Ho);
    const int t = (int)(r / Ho);
    const float4* p = reinterpret_cast<const float4*>(in + (((int64_t)t * Hi + 2 * y) * Wi + 2 * x) * kD) + c4;
    const float4 a = p[0], b = p[kD / 4], c = p[(int64_t)Wi * (kD / 4)], d = p[(int64_t)Wi * (kD / 4) + kD / 4];
    float4 o;
    o.x = (a.x + b.x + c.x + d.x) * 0.25f;
    o.y = (a.y + b.y + c.y + d.y) * 0.25f;
    o.z = (a.z + b.z + c.z + d.z) * 0.25f;
    o.w = (a.w + b.w + c.w + d.w) * 0.25f;
    reinterpret_cast<float4*>(out)[i] = o;
  }
}

// block = (track n, level l), 128 threads = channels
__global__ void __launch_bounds__(128)
sample_support_kernel(const float* __restrict__ pyr, PyramidLayout lay, int T, const int32_t* __restrict__ qframes,
                      const float* __restrict__ qcoords, int N, const uint8_t* __restrict__ acc_mask,
                      float* __restrict__ support) {
  const int n = blockIdx.x, l = blockIdx.y, c = threadIdx.x;
  if (acc_mask && !acc_mask[n]) return;
  const int H = lay.h[l], W = lay.w[l];
  int f = qframes[n];
  f = f < 0 ? 0 : (f > T - 1 ? T - 1 : f);
  const float inv = 1.0f / (float)(1 << l);
  const float cx = qcoords[2 * n] * inv, cy = qcoords[2 * n + 1] * inv;
  const float* fm = pyr + lay.off[l] + (int64_t)f * H * W * kD;
  float* dst = support + (int64_t)l * kP * N * kD;
  for (int p = 0; p < kP; ++p) {
    const int a = p / 7, b = p % 7;  // a: x offset index, b: y offset index (cotracker3_online.py:99-104)
    float x = fminf(fmaxf(cx + (float)(a - kR), 0.f), (float)(W - 1));
    float y = fminf(fmaxf(cy + (float)(b - kR), 0.f), (float)(H - 1));
    const float xf = floorf(x), yf = floorf(y);
    const int x0 = (int)xf, y0 = (int)yf;
    const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
    const float wx = x - xf, wy = y - yf;
    const float v00 = fm[((int64_t)y0 * W + x0) * kD + c], v01 = fm[((int64_t)y0 * W + x1) * kD + c];
    const float v10 = fm[((int64_t)y1 * W + x0) * kD + c], v11 = fm[((int64_t)y1 * W + x1) * kD + c];
    const float v = (1.f - wy) * ((1.f - wx) * v00 + wx * v01) + wy * ((1.f - wx) * v10 + wx * v11);
    float* o = dst + ((int64_t)p * N + n) * kD + c;
    if (acc_mask) *o += v; else *o = v;
  }
}

}  // namespace

cudaError_t launch_pyramid_pools(int T, int H4, int W4, float* pyr, cudaStream_t s) {
  const PyramidLayout lay = pyramid_layout(T, H4, W4);
  for (int l = 1; l < kL; ++l) {
    const int64_t total = (int64_t)T * lay.h[l] * lay.w[l] * (kD / 4);
    if (total == 0) continue;
    const int blocks = (int)((total + 255) / 256 > 132 * 16 ? 132 * 16 : (total + 255) / 256);
    avgpool2_channels_last_kernel<<<blocks, 256, 0, s>>>(pyr + lay.off[l - 1], pyr + lay.off[l], T, lay.h[l - 1],
                                                        lay.w[l - 1], lay.h[l], lay.w[l]);
  }
  return cudaGetLastError();
}

cudaError_t launch_prepare_pyramid(const float* fmaps, int T, int H4, int W4, float* pyr, cudaStream_t s) {
  const PyramidLayout lay = pyramid_layout(T, H4, W4);
  dim3 g((W4 + 31) / 32, H4, T);
  normalize_to_channels_last_kernel<<<g, 256, 0, s>>>(fmaps, pyr + lay.off[0], T, H4, W4);
  for (int l = 1; l < kL; ++l) {
    const int64_t total = (int64_t)T * lay.h[l] * lay.w[l] * (kD / 4);
    if (total == 0) continue;
    const int blocks = (int)((total + 255) / 256 > 132 * 16 ? 132 * 16 : (total + 255) / 256);
    avgpool2_channels_last_kernel<<<blocks, 256, 0, s>>>(pyr + lay.off[l - 1], pyr + lay.off[l], T, lay.h[l - 1],
                                                        lay.w[l - 1], lay.h[l], lay.w[l]);
  }
  return cudaGetLastError();
}

cudaError_t launch_sample_support(const float* pyr, int T, int H4, int W4, const int32_t* qframes,
                                  const float* qcoords, int N, const uint8_t* acc_mask, float* support,
                                  cudaStream_t s) {
  const PyramidLayout lay = pyramid_layout(T, H4, W4);
  dim3 g(N, kL);
  sample_support_kernel<<<g, 128, 0, s>>>(pyr, lay, T, qframes, qcoords, N, acc_mask, support);
  return cudaGetLastError();
}

}  // namespace ct3
