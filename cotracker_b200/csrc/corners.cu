// corners.cu -- Shi-Tomasi corners (cv2.goodFeaturesToTrack with useHarrisDetector=False) in K prepared frames at once
// (ct3_detect_corners).  The result is bit-identical to a float64 restatement (tests/corner_cases.py), so every
// rounding is explicit: __f*_rn / __d*_rn intrinsics keep nvcc from contracting products into FMAs, which numpy never
// does.  Per frame:
//   1. response: gray g = 0.299 R + 0.587 G + 0.114 B (fp32); 3x3 Sobel dx, dy (fp64, reflect-101); box sums of dx^2,
//      dx dy, dy^2 over block x block (reflect-101, row-major accumulation); lambda = a + c - sqrt((a - c)^2 + b^2) with
//      a = Sxx / 2, b = Sxy, c = Syy / 2.  The frame's max lambda is reduced with an order-preserving u64 key.
//   2. candidates: interior pixels (1 <= x < W-1, 1 <= y < H-1) with lambda > quality * max, lambda equal to its 3x3
//      maximum and outside every exclusion disc, compacted to (lambda bits, raster index).
//   3. rank: each candidate's position in (lambda desc, index desc) order, counted by comparison against every other
//      candidate in 256 x 256 tiles.  The order is total (indices are distinct), so the ranks are a permutation.  This
//      is O(n^2) in a frame's candidates: a few thousand in a textured frame, microseconds; a frame where every pixel
//      is a candidate is correct and slow.
//   4. greedy: one warp per frame walks the sorted candidates 32 at a time and keeps one unless a kept corner lies at
//      dx^2 + dy^2 < min_distance^2, up to max_corners.  Kept corners live in a grid of floor(min_distance)-pixel cells
//      (at most 4 per cell, and a conflict is never more than one cell away); the conflicts inside a batch of 32 are
//      resolved in rank order with warp shuffles, so the result is the sequential walk's.
// With a region mask (ct3_detect_corners_masked; kMasked = true) step 1 takes the maximum over the mask's pixels only
// and step 2 also drops candidates outside the mask; the 3x3 maximum still reads every pixel, as cv2 dilates the whole
// thresholded map.  ct3_detect_corners runs the kMasked = false instantiations, which are the kernels without the mask.
// ct3_prepare_masks resizes masks to the detector's frames: ATen's nearest rule, one thread per output pixel.
#include <math.h>

#include "../../include/ct3_b200.h"
#include "kernels.cuh"

namespace ct3 {
namespace {

constexpr int kTX = 32, kTY = 16;          // response tile
constexpr int kMaxR = 4;                   // Sobel radius 1 + box radius <= 3
constexpr int kThreads = 256;

__device__ __forceinline__ int refl101(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

// fp64 -> u64 with the same order (negative values included)
__device__ __forceinline__ unsigned long long order_key(double v) {
  const long long b = __double_as_longlong(v);
  return b >= 0 ? (unsigned long long)b | 0x8000000000000000ull : ~(unsigned long long)b;
}
__device__ __forceinline__ double order_value(unsigned long long k) {
  return __longlong_as_double((long long)((k & 0x8000000000000000ull) ? (k & 0x7fffffffffffffffull) : ~k));
}

template <bool kMasked>
__global__ void __launch_bounds__(kTX * kTY)
corner_response_kernel(const float* __restrict__ frames, int64_t frame_stride, int H, int W,
                       const CornerFrame* __restrict__ fp, const uint8_t* __restrict__ mask, int64_t mask_stride,
                       double* __restrict__ lam, unsigned long long* __restrict__ maxkey) {
  __shared__ float g[kTY + 2 * kMaxR][kTX + 2 * kMaxR];
  __shared__ double sdx[kTY + 2 * kMaxR - 2][kTX + 2 * kMaxR - 2];
  __shared__ double sdy[kTY + 2 * kMaxR - 2][kTX + 2 * kMaxR - 2];
  const int k = blockIdx.z;
  const int r = fp[k].block / 2, R = r + 1;
  const int x0 = blockIdx.x * kTX, y0 = blockIdx.y * kTY;
  const int tid = threadIdx.y * kTX + threadIdx.x;
  const int64_t HW = (int64_t)H * W;
  const float* f = frames + (int64_t)k * frame_stride;
  // gray at frame rows [y0 - R, y0 + kTY + R), columns likewise (cells outside the frame are never read)
  for (int c = tid; c < (kTY + 2 * R) * (kTX + 2 * R); c += kTX * kTY) {
    const int i = c / (kTX + 2 * R), j = c % (kTX + 2 * R);
    const int gy = y0 - R + i, gx = x0 - R + j;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
      const int64_t o = (int64_t)gy * W + gx;
      g[i][j] = __fadd_rn(__fadd_rn(__fmul_rn(0.299f, f[o]), __fmul_rn(0.587f, f[HW + o])), __fmul_rn(0.114f, f[2 * HW + o]));
    }
  }
  __syncthreads();
  // dx, dy at the (reflected) positions [y0 - r, min(y0 + kTY, H) + r) x [x0 - r, min(x0 + kTX, W) + r): their gray
  // neighbours, reflected, lie in the rows and columns loaded above
  const int ye = min(y0 + kTY, H) + r, xe = min(x0 + kTX, W) + r;
  const int dw = kTX + 2 * r;
  for (int c = tid; c < (kTY + 2 * r) * dw; c += kTX * kTY) {
    const int i = c / dw, j = c % dw;
    const int yy = y0 - r + i, xx = x0 - r + j;
    if (yy >= ye || xx >= xe) continue;
    const int ry = refl101(yy, H), rx = refl101(xx, W);
    const int ym = refl101(ry - 1, H) - (y0 - R), yc = ry - (y0 - R), yp = refl101(ry + 1, H) - (y0 - R);
    const int xm = refl101(rx - 1, W) - (x0 - R), xc = rx - (x0 - R), xp = refl101(rx + 1, W) - (x0 - R);
    const double t0 = __dsub_rn((double)g[ym][xp], (double)g[ym][xm]);
    const double t1 = __dsub_rn((double)g[yc][xp], (double)g[yc][xm]);
    const double t2 = __dsub_rn((double)g[yp][xp], (double)g[yp][xm]);
    const double s0 = __dsub_rn((double)g[yp][xm], (double)g[ym][xm]);
    const double s1 = __dsub_rn((double)g[yp][xc], (double)g[ym][xc]);
    const double s2 = __dsub_rn((double)g[yp][xp], (double)g[ym][xp]);
    sdx[i][j] = __dadd_rn(__dadd_rn(t0, __dmul_rn(2.0, t1)), t2);
    sdy[i][j] = __dadd_rn(__dadd_rn(s0, __dmul_rn(2.0, s1)), s2);
  }
  __syncthreads();
  const int y = y0 + threadIdx.y, x = x0 + threadIdx.x;
  unsigned long long key = 0;
  if (y < H && x < W) {
    const int b = 2 * r + 1;
    double sxx = 0.0, sxy = 0.0, syy = 0.0;
    for (int i = 0; i < b; ++i)
      for (int j = 0; j < b; ++j) {
        const double u = sdx[threadIdx.y + i][threadIdx.x + j], v = sdy[threadIdx.y + i][threadIdx.x + j];
        sxx = __dadd_rn(sxx, __dmul_rn(u, u));
        sxy = __dadd_rn(sxy, __dmul_rn(u, v));
        syy = __dadd_rn(syy, __dmul_rn(v, v));
      }
    const double a = __dmul_rn(sxx, 0.5), c = __dmul_rn(syy, 0.5), d = __dsub_rn(a, c);
    const double l = __dsub_rn(__dadd_rn(a, c), __dsqrt_rn(__dadd_rn(__dmul_rn(d, d), __dmul_rn(sxy, sxy))));
    lam[(int64_t)k * HW + (int64_t)y * W + x] = l;
    if constexpr (kMasked) {
      if (mask[(int64_t)k * mask_stride + (int64_t)y * W + x]) key = order_key(l);   // minMaxLoc(eig, ..., mask)
    } else {
      key = order_key(l);
    }
  }
  for (int o = 16; o; o >>= 1) key = max(key, __shfl_xor_sync(0xffffffffu, key, o));
  if ((tid & 31) == 0 && key) atomicMax(maxkey + k, key);
}

// frame k's candidate region: keys u64 [HW], then idx i32 [HW], then rank i32 [HW]; the greedy step reuses it as the
// cell grid (int4 per cell, at most HW cells)
__device__ __forceinline__ unsigned long long* cand_keys(uint8_t* cand, int k, int64_t HW) {
  return reinterpret_cast<unsigned long long*>(cand + (size_t)k * HW * 16);
}

template <bool kMasked>
__global__ void __launch_bounds__(kThreads)
corner_candidates_kernel(int H, int W, const CornerFrame* __restrict__ fp, const double* __restrict__ lam,
                         const unsigned long long* __restrict__ maxkey, const float* __restrict__ exclude, int E_max,
                         const uint8_t* __restrict__ mask, int64_t mask_stride, int* __restrict__ count,
                         uint8_t* __restrict__ cand) {
  const int k = blockIdx.y;
  const int64_t HW = (int64_t)H * W;
  const int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (p >= HW) return;
  const int y = (int)(p / W), x = (int)(p - (int64_t)y * W);
  if (x < 1 || x >= W - 1 || y < 1 || y >= H - 1) return;
  if constexpr (kMasked) {
    if (!mask[(int64_t)k * mask_stride + p]) return;
  }
  const double* L = lam + (size_t)k * HW;
  const double l = L[p];
  const CornerFrame P = fp[k];
  if (!(l > __dmul_rn(P.quality, order_value(maxkey[k])))) return;
  for (int dy = -1; dy <= 1; ++dy)
    for (int dx = -1; dx <= 1; ++dx)
      if (L[p + (int64_t)dy * W + dx] > l) return;
  if (P.r2 > 0.0) {
    const float* e = exclude + (size_t)k * E_max * 2;
    for (int i = 0; i < P.E; ++i) {
      const double ex = __dsub_rn((double)x, (double)e[2 * i]), ey = __dsub_rn((double)y, (double)e[2 * i + 1]);
      if (__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)) < P.r2) return;
    }
  }
  const int slot = atomicAdd(count + k, 1);
  unsigned long long* keys = cand_keys(cand, k, HW);
  int* idx = reinterpret_cast<int*>(keys + HW);
  keys[slot] = (unsigned long long)__double_as_longlong(l);   // l > 0: the bits order as the values
  idx[slot] = (int)p;
  idx[HW + slot] = 0;                                          // rank
}

__global__ void __launch_bounds__(kThreads)
corner_rank_kernel(int H, int W, const int* __restrict__ count, uint8_t* __restrict__ cand) {
  __shared__ unsigned long long sk[kThreads];
  __shared__ int si[kThreads];
  const int k = blockIdx.y;
  const int64_t HW = (int64_t)H * W;
  const int n = count[k];
  const unsigned long long* keys = cand_keys(cand, k, HW);
  const int* idx = reinterpret_cast<const int*>(keys + HW);
  int* rank = const_cast<int*>(idx) + HW;
  const long long tiles = (n + kThreads - 1) / kThreads;
  for (long long pp = blockIdx.x; pp < tiles * tiles; pp += gridDim.x) {
    const int it = (int)(pp / tiles), j0 = (int)(pp % tiles) * kThreads;
    const int m = min(kThreads, n - j0);
    if ((int)threadIdx.x < m) { sk[threadIdx.x] = keys[j0 + threadIdx.x]; si[threadIdx.x] = idx[j0 + threadIdx.x]; }
    __syncthreads();
    const int i = it * kThreads + threadIdx.x;
    if (i < n) {
      const unsigned long long ki = keys[i];
      const int ii = idx[i];
      int c = 0;
      for (int t = 0; t < m; ++t) c += (sk[t] > ki) | ((sk[t] == ki) & (si[t] > ii));
      if (c) atomicAdd(rank + i, c);
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kThreads)
corner_greedy_kernel(int H, int W, const CornerFrame* __restrict__ fp, const int* __restrict__ count,
                     uint8_t* __restrict__ cand, int* __restrict__ sorted_all, int M, float* __restrict__ corners,
                     int32_t* __restrict__ counts) {
  __shared__ int s_kept;
  const int k = blockIdx.x;
  const int64_t HW = (int64_t)H * W;
  const int n = count[k];
  const CornerFrame P = fp[k];
  unsigned long long* keys = cand_keys(cand, k, HW);
  const int* idx = reinterpret_cast<const int*>(keys + HW);
  const int* rank = idx + HW;
  int* sorted = sorted_all + (size_t)k * HW;
  for (int i = threadIdx.x; i < n; i += kThreads) sorted[rank[i]] = idx[i];
  __syncthreads();
  // md^2 <= 1: distinct pixels are never closer than that, so nothing conflicts
  const bool check = P.md2 > 1.0;
  int4* grid = reinterpret_cast<int4*>(keys);
  if (check)
    for (int c = threadIdx.x; c < P.gw * P.gh; c += kThreads) grid[c] = make_int4(-1, -1, -1, -1);
  __syncthreads();
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    const unsigned below = (1u << lane) - 1u;
    int kept = 0;
    for (int base = 0; base < n && kept < P.max_corners; base += 32) {
      const bool have = base + lane < n;
      const int p = have ? sorted[base + lane] : 0;
      const int y = p / W, x = p - y * W;
      const int cx = check ? x / P.cs : 0, cy = check ? y / P.cs : 0;
      bool alive = have;
      unsigned conf = 0;
      if (check) {
        for (int gy = max(cy - 1, 0); alive && gy <= min(cy + 1, P.gh - 1); ++gy)
          for (int gx = max(cx - 1, 0); gx <= min(cx + 1, P.gw - 1); ++gx) {
            const int4 c = __ldcg(grid + gy * P.gw + gx);
            const int s[4] = {c.x, c.y, c.z, c.w};
            for (int q = 0; q < 4; ++q) {
              if (s[q] < 0) continue;
              const int64_t qy = s[q] / W, qx = s[q] - qy * W;
              const int64_t d2 = (qx - x) * (qx - x) + (qy - y) * (qy - y);
              if ((double)d2 < P.md2) alive = false;
            }
          }
        for (int j = 0; j < 32; ++j) {
          const int xj = __shfl_sync(0xffffffffu, x, j), yj = __shfl_sync(0xffffffffu, y, j);
          const int64_t d2 = (int64_t)(xj - x) * (xj - x) + (int64_t)(yj - y) * (yj - y);
          if (j < lane && (double)d2 < P.md2) conf |= 1u << j;
        }
      }
      const unsigned alive_mask = __ballot_sync(0xffffffffu, alive);
      unsigned keep = 0;
      int total = kept;
      for (int j = 0; j < 32; ++j) {
        const unsigned cj = __shfl_sync(0xffffffffu, conf, j);
        if (((alive_mask >> j) & 1u) && !(cj & keep) && total < P.max_corners) { keep |= 1u << j; ++total; }
      }
      if ((keep >> lane) & 1u) {
        const int o = kept + __popc(keep & below);
        corners[((size_t)k * M + o) * 2] = (float)x;
        corners[((size_t)k * M + o) * 2 + 1] = (float)y;
        if (check) {
          int* slot = reinterpret_cast<int*>(grid + cy * P.gw + cx);
          for (int q = 0; q < 4 && atomicCAS(slot + q, -1, p) != -1; ++q) {}
        }
      }
      kept = total;
      __syncwarp();
    }
    if (lane == 0) { counts[k] = kept; s_kept = kept; }
  }
  __syncthreads();
  for (int j = s_kept + threadIdx.x; j < M; j += kThreads) {
    corners[((size_t)k * M + j) * 2] = 0.f;
    corners[((size_t)k * M + j) * 2 + 1] = 0.f;
  }
}

// out[k][y][x] = src[k][sy][sx] != 0 with s = min(floor(d * (in / out)), in - 1) in fp32, ATen's nearest index
template <typename T>
__global__ void __launch_bounds__(kThreads)
prepare_masks_kernel(const T* __restrict__ src, int H, int W, int64_t stride_k, int64_t stride_h, int64_t stride_w,
                     int oh, int ow, float scale_h, float scale_w, uint8_t* __restrict__ out) {
  const int k = blockIdx.y;
  const int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (p >= (int64_t)oh * ow) return;
  const int y = (int)(p / ow), x = (int)(p - (int64_t)y * ow);
  const int sy = min((int)floorf(__fmul_rn((float)y, scale_h)), H - 1);
  const int sx = min((int)floorf(__fmul_rn((float)x, scale_w)), W - 1);
  const T v = src[(int64_t)k * stride_k + (int64_t)sy * stride_h + (int64_t)sx * stride_w];
  out[(int64_t)k * oh * ow + p] = v != T(0) ? 1 : 0;
}

}  // namespace

cudaError_t launch_prepare_masks(const void* src, bool f32, int K, int H, int W, int64_t stride_k, int64_t stride_h,
                                 int64_t stride_w, int oh, int ow, uint8_t* out, cudaStream_t s) {
  const dim3 grid((unsigned)(((int64_t)oh * ow + kThreads - 1) / kThreads), K);
  // area_pixel_compute_scale without align_corners or a scale factor: (float)in / out
  const float sh = (float)H / (float)oh, sw = (float)W / (float)ow;
  if (f32)
    prepare_masks_kernel<float><<<grid, kThreads, 0, s>>>(static_cast<const float*>(src), H, W, stride_k, stride_h,
                                                          stride_w, oh, ow, sh, sw, out);
  else
    prepare_masks_kernel<uint8_t><<<grid, kThreads, 0, s>>>(static_cast<const uint8_t*>(src), H, W, stride_k, stride_h,
                                                            stride_w, oh, ow, sh, sw, out);
  return cudaGetLastError();
}

cudaError_t launch_detect_corners(const float* frames, int64_t frame_stride, int K, int H, int W,
                                  const CornerFrame* fp_dev, const float* exclude, int E_max, const uint8_t* mask,
                                  int64_t mask_stride, int M, float* corners, int32_t* counts,
                                  const CornerWorkspace& ws, int num_sms, cudaStream_t s) {
  const int64_t HW = (int64_t)H * W;
  cudaError_t e = cudaMemsetAsync(ws.maxkey, 0, (size_t)K * (sizeof(unsigned long long) + sizeof(int)), s);
  if (e != cudaSuccess) return e;
  int* count = reinterpret_cast<int*>(ws.maxkey + K);
  const dim3 rgrid((W + kTX - 1) / kTX, (H + kTY - 1) / kTY, K), cgrid((unsigned)((HW + kThreads - 1) / kThreads), K);
  if (mask) {
    corner_response_kernel<true><<<rgrid, dim3(kTX, kTY), 0, s>>>(frames, frame_stride, H, W, fp_dev, mask, mask_stride,
                                                                  ws.lam, ws.maxkey);
    corner_candidates_kernel<true><<<cgrid, kThreads, 0, s>>>(H, W, fp_dev, ws.lam, ws.maxkey, exclude, E_max, mask,
                                                              mask_stride, count, ws.cand);
  } else {
    corner_response_kernel<false><<<rgrid, dim3(kTX, kTY), 0, s>>>(frames, frame_stride, H, W, fp_dev, nullptr, 0,
                                                                   ws.lam, ws.maxkey);
    corner_candidates_kernel<false><<<cgrid, kThreads, 0, s>>>(H, W, fp_dev, ws.lam, ws.maxkey, exclude, E_max,
                                                               nullptr, 0, count, ws.cand);
  }
  const int per_frame = max(1, min(4096, (4 * num_sms + K - 1) / K));
  corner_rank_kernel<<<dim3(per_frame, K), kThreads, 0, s>>>(H, W, count, ws.cand);
  corner_greedy_kernel<<<K, kThreads, 0, s>>>(H, W, fp_dev, count, ws.cand, ws.sorted, M, corners, counts);
  return cudaGetLastError();
}

}  // namespace ct3
