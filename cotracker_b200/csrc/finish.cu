// finish.cu -- the tail of CoTrackerPredictor in one pass (reference predictor.py:161-209): merge the backward pass in
// before each query frame, drop the support-grid tracks, threshold the visibility, pin every query point to where it
// was asked for and scale the tracks from the model's resolution to the input's.
//
// Per output element this is a select, a compare and one fp32 multiply, so the result is bit-identical to the ATen
// sequence it replaces:
//     before = arange(T)[None, :, None] < queries[:, None, :, 0]          (int64 < fp32: compared in fp32)
//     tracks = where(before[..., None], bwd_tracks.flip(1), fwd_tracks);  vis likewise
//     vis = vis[:, :, :n_keep] > threshold                                (fp32 compare)
//     tracks[b, int64(queries[b, i, 0]), i] = queries[b, i, 1:];  vis[...] = True
//     tracks *= (scale_x, scale_y)
#include "../../include/ct3_b200.h"
#include "kernels.cuh"

namespace ct3 {
namespace {

constexpr int kFinishThreads = 256;

__global__ void __launch_bounds__(kFinishThreads) finish_tracks_kernel(
    const float2* __restrict__ fwd_tracks, const float* __restrict__ fwd_vis, const float2* __restrict__ bwd_tracks,
    const float* __restrict__ bwd_vis, const float* __restrict__ queries, int T, int N, int n_keep, float threshold,
    float scale_x, float scale_y, int64_t total, float2* __restrict__ tracks, uint8_t* __restrict__ visibility) {
  const int64_t e = (int64_t)blockIdx.x * kFinishThreads + threadIdx.x;   // element (b, t, i) of the output
  if (e >= total) return;
  const int i = (int)(e % n_keep);
  const int64_t bt = e / n_keep;
  const int t = (int)(bt % T);
  const int64_t b = bt / T;
  const float* q = queries + (b * N + i) * 3;
  const float qt = __ldg(q);
  float2 p;
  bool vis;
  if (t == (int64_t)qt) {   // the query point itself: .to(int64) truncates toward zero
    p = make_float2(__ldg(q + 1), __ldg(q + 2));
    vis = true;
  } else {
    // the backward pass is in reversed-clip time: its frame T-1-t is frame t
    const bool back = bwd_tracks != nullptr && (float)t < qt;
    const int64_t src = (b * T + (back ? T - 1 - t : t)) * N + i;
    p = __ldg((back ? bwd_tracks : fwd_tracks) + src);
    vis = __ldg((back ? bwd_vis : fwd_vis) + src) > threshold;
  }
  tracks[e] = make_float2(__fmul_rn(p.x, scale_x), __fmul_rn(p.y, scale_y));
  visibility[e] = vis ? 1 : 0;
}

}  // namespace

cudaError_t launch_finish_tracks(const float* fwd_tracks, const float* fwd_vis, const float* bwd_tracks,
                                 const float* bwd_vis, const float* queries, int B, int T, int N, int n_keep,
                                 float threshold, float scale_x, float scale_y, float* tracks, uint8_t* visibility,
                                 cudaStream_t s) {
  const int64_t total = (int64_t)B * T * n_keep;   // < 2^31 * kFinishThreads (ct3_finish_tracks)
  const unsigned grid = (unsigned)((total + kFinishThreads - 1) / kFinishThreads);
  finish_tracks_kernel<<<grid, kFinishThreads, 0, s>>>(
      reinterpret_cast<const float2*>(fwd_tracks), fwd_vis, reinterpret_cast<const float2*>(bwd_tracks), bwd_vis,
      queries, T, N, n_keep, threshold, scale_x, scale_y, total, reinterpret_cast<float2*>(tracks), visibility);
  return cudaGetLastError();
}

}  // namespace ct3
