// online.cu -- the per-window work of the streaming model around one update-loop pass, for K streams at once, each at
// its own window start (reference cotracker3_online.py:457-541 and the online predictor's tail, predictor.py:276-309).
//
// Every output element is a copy, a select, an integer compare, one fp32 multiply or torch.sigmoid of fp32
// (1 / (1 + expf(-x)), IEEE division, no fast-math), so the results are bit-identical to the ATen expressions they
// replace (include/ct3_b200.h).  Division by the stride is a multiply by the fp32 reciprocal, as ATen evaluates a
// division by a scalar.  Block (x, k) strides over the elements of stream k; the grid's y dimension is the stream.
// With scores (ct3_online_window_end_scores) the two sigmoids of the visibility compare are stored as well.
// A ring history (ring = 1) holds frame f at row f mod cap; the host checks guarantee that every frame a launch reads
// is still held and that no row is both read and written by one window_end launch.  A preview entry (preview = 1)
// takes the same loads and arithmetic and skips the three history stores, so its output is that of the same entry
// with preview = 0 and its history is left as it was.
#include "../../include/ct3_b200.h"
#include "kernels.cuh"

namespace ct3 {
namespace {

constexpr int kOnlineThreads = 256;
constexpr int kOnlineMaxBlocksX = 1024;

// the history row of stream frame f
__device__ __forceinline__ int64_t history_row(const ct3_online_stream& st, int64_t f) {
  return st.ring ? f % st.cap : f;
}

__global__ void __launch_bounds__(kOnlineThreads) online_window_begin_kernel(
    const ct3_online_stream* __restrict__ streams, int S, int step, float inv_stride, const int32_t* __restrict__ qframes,
    const float2* __restrict__ qcoords, int N, uint8_t* __restrict__ valid, uint8_t* __restrict__ entering,
    int32_t* __restrict__ rel, float2* __restrict__ coords_init, float* __restrict__ vis_init,
    float* __restrict__ conf_init) {
  const ct3_online_stream& st = streams[blockIdx.y];
  const int n = st.n, first = st.first, ind = st.ind, frame0 = st.frame0;
  const int overlap = S - step;
  const float2* __restrict__ hc = reinterpret_cast<const float2*>(st.coords);
  const float* __restrict__ hv = st.vis;
  const float* __restrict__ hq = st.conf;
  const int64_t total = (int64_t)S * n;
  for (int64_t e = (int64_t)blockIdx.x * kOnlineThreads + threadIdx.x; e < total;
       e += (int64_t)gridDim.x * kOnlineThreads) {
    const int t = (int)(e / n), j = (int)(e % n), i = first + j;
    const int qf = __ldg(qframes + i);   // |qf| <= 2^30 and ind + S <= 2^30: no int32 overflow below
    if (t == 0) {
      const int left = ind == 0 ? 0 : ind + step;
      valid[i] = qf < ind + S ? 1 : 0;
      entering[i] = (qf >= left && qf < ind + S) ? 1 : 0;
      rel[i] = min(max(qf - ind, 0), S - 1) + frame0;
    }
    float2 c;
    float v = 0.f, q = 0.f;
    if (ind > 0 && qf < ind + overlap) {   // warm start: the previous window's overlap, its last frame repeated
      const int64_t src = history_row(st, ind + min(t, overlap - 1)) * n + j;
      const float2 h = hc[src];
      c = make_float2(__fmul_rn(h.x, inv_stride), __fmul_rn(h.y, inv_stride));
      v = hv[src];
      q = hq[src];
    } else {
      c = __ldg(qcoords + i);
    }
    const int64_t o = (int64_t)t * N + i;
    coords_init[o] = c;
    vis_init[o] = v;
    conf_init[o] = q;
  }
}

// kScores: also write the two probabilities of each output element where the stream's scores entry is set.
// 8 blocks per SM: with the preview branch the kScores instantiation would otherwise take 40 registers (6 blocks);
// with the bound both take 32 with no spills, as before the branch.
template <bool kScores>
__global__ void __launch_bounds__(kOnlineThreads, 8) online_window_end_kernel(
    const ct3_online_stream* __restrict__ streams, const ct3_online_scores* __restrict__ scores, float stride,
    const float2* __restrict__ coords, const float* __restrict__ vis, const float* __restrict__ conf, int N,
    float threshold) {
  const ct3_online_stream& st = streams[blockIdx.y];
  float* __restrict__ score_vis = kScores ? scores[blockIdx.y].vis : nullptr;
  float* __restrict__ score_conf = kScores ? scores[blockIdx.y].conf : nullptr;
  const int n = st.n, first = st.first, ind = st.ind, n_keep = st.n_keep;
  const bool preview = st.preview != 0;   // read the history, never write it
  float2* __restrict__ hc = reinterpret_cast<float2*>(st.coords);
  float* __restrict__ hv = st.vis;
  float* __restrict__ hq = st.conf;
  float2* __restrict__ tracks = reinterpret_cast<float2*>(st.tracks);
  uint8_t* __restrict__ visibility = st.visibility;
  // frames [lo, ind + T): the window's frames, and before them those of the output (frames before lo are not touched)
  const int64_t out_first = st.out_first;
  const int64_t lo = tracks != nullptr && out_first < ind ? out_first : ind;
  const int64_t total = ((int64_t)ind + st.T - lo) * n;
  for (int64_t e = (int64_t)blockIdx.x * kOnlineThreads + threadIdx.x; e < total;
       e += (int64_t)gridDim.x * kOnlineThreads) {
    const int64_t t = lo + e / n;
    const int j = (int)(e % n);
    const bool out = tracks != nullptr && j < n_keep && t >= out_first;
    const int64_t h = history_row(st, t) * n + j;
    float2 p;
    float v, q;
    if (t >= ind) {   // a frame of this window: the loop's result, written back (frames ind + T.. are padding)
      const int64_t src = (t - ind) * N + first + j;
      const float2 c = __ldg(coords + src);
      p = make_float2(__fmul_rn(c.x, stride), __fmul_rn(c.y, stride));
      v = __ldg(vis + src);
      q = __ldg(conf + src);
      if (!preview) {
        hc[h] = p;
        hv[h] = v;
        hq[h] = q;
      }
    } else if (out) {   // an earlier frame: the history as it stands
      p = hc[h];
      v = hv[h];
      q = hq[h];
    } else {
      continue;
    }
    if (out) {
      const int64_t o = (t - out_first) * n_keep + j;
      tracks[o] = make_float2(__fmul_rn(p.x, st.scale_x), __fmul_rn(p.y, st.scale_y));
      const float pv = sigmoid_aten(v), pq = sigmoid_aten(q);
      visibility[o] = __fmul_rn(pv, pq) > threshold ? 1 : 0;
      if constexpr (kScores) {
        if (score_vis != nullptr) {
          score_vis[o] = pv;
          score_conf[o] = pq;
        }
      }
    }
  }
}

dim3 online_grid(int K, int64_t max_elems) {
  const int64_t bx = (max_elems + kOnlineThreads - 1) / kOnlineThreads;
  return dim3((unsigned)(bx < 1 ? 1 : bx > kOnlineMaxBlocksX ? kOnlineMaxBlocksX : bx), (unsigned)K);
}

}  // namespace

cudaError_t launch_online_window_begin(const ct3_online_stream* streams, int K, int64_t max_elems, int S, int step,
                                       float inv_stride, const int32_t* qframes, const float* qcoords, int N,
                                       uint8_t* valid, uint8_t* entering, int32_t* rel, float* coords_init,
                                       float* vis_init, float* conf_init, cudaStream_t s) {
  online_window_begin_kernel<<<online_grid(K, max_elems), kOnlineThreads, 0, s>>>(
      streams, S, step, inv_stride, qframes, reinterpret_cast<const float2*>(qcoords), N, valid, entering, rel,
      reinterpret_cast<float2*>(coords_init), vis_init, conf_init);
  return cudaGetLastError();
}

cudaError_t launch_online_window_end(const ct3_online_stream* streams, int K, int64_t max_elems, float stride,
                                     const float* coords, const float* vis, const float* conf, int N, float threshold,
                                     cudaStream_t s) {
  online_window_end_kernel<false><<<online_grid(K, max_elems), kOnlineThreads, 0, s>>>(
      streams, nullptr, stride, reinterpret_cast<const float2*>(coords), vis, conf, N, threshold);
  return cudaGetLastError();
}

cudaError_t launch_online_window_end_scores(const ct3_online_stream* streams, const ct3_online_scores* scores, int K,
                                            int64_t max_elems, float stride, const float* coords, const float* vis,
                                            const float* conf, int N, float threshold, cudaStream_t s) {
  online_window_end_kernel<true><<<online_grid(K, max_elems), kOnlineThreads, 0, s>>>(
      streams, scores, stride, reinterpret_cast<const float2*>(coords), vis, conf, N, threshold);
  return cudaGetLastError();
}

}  // namespace ct3
