// api.cu -- C ABI of libct3_b200.so (see include/ct3_b200.h): the library-wide state (errors, options, profiler) and the
// small entry points (pyramid, support sampling, frame ingest, track rendering, split rows).  The update loop and its
// weight packing are in api_loop.cu, the encoder in api_encoder.cu.
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <vector>

#include "abi.cuh"

namespace ct3 {

thread_local char g_err[512] = "";
// Options and the profiler are PER HOST THREAD (thread_local): a thread that drives its own GPU/stream never sees
// another thread's verification switches or profile records.
struct OptDef { const char* name; int lo, hi; };
constexpr int kDefPrecCorr = 2, kDefPrecFc1 = 3;   // DESIGN.md section 2
constexpr OptDef kOptDefs[OPT_COUNT] = {
    {"gemm", 0, 1},   // 0 wgmma, 1 SIMT verification
    {"corr", 0, 2},   // 0 wgmma correlate-then-interpolate (corr_tc3.cu / corr_tc2.cu), 1 exact-fp32 SIMT, 2 corr_tc.cu
    {"attn", 0, 1},   // 0 tensor-core kernels (wgmma point<-virtual, mma.sync elsewhere), 1 exact-fp32 SIMT verification
    // tensor-core products per FLOP of a GEMM group (DESIGN.md section 2): 3 = split x split (hi*hi + lo*hi + hi*lo),
    // 2 = fp16 activation plane x split fp16 weights, 1 = single fp16 product.  Only the correlation branch has the
    // switch: SURVEY 7.3 measured that every transformer GEMM breaks the 1e-3 px budget with fewer than 3 products.
    {"prec.corr", 1, 3},   // the 49x128x49 correlation contraction (corr_tc2.cu)
    {"prec.fc1", 1, 3},    // corr_mlp.fc1 (K = 2401): 1|2 also make the correlation volume a single fp16 plane
    // time blocks: 0 = separate q|k|v projection and attention kernels (what T > 128 always runs; the tests'
    // cross-check), 1 = both in one kernel (gemm_qkv_time_attn_kernel)
    {"fuse", 0, 1},
};
thread_local int g_opt[OPT_COUNT] = {0, 0, 0, kDefPrecCorr, kDefPrecFc1, 1};

int fail(int code, const char* fmt, const char* detail) {
  snprintf(g_err, sizeof(g_err), fmt, detail);
  return code;
}
int fail_cuda(cudaError_t e, const char* where) {
  snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
  return CT3_ECUDA;
}
int fail_launch(int rc, const char* what, const char* detail) {
  snprintf(g_err, sizeof(g_err), "%s: %s (%s)", what, cudaGetErrorString((cudaError_t)rc), detail ? detail : "");
  return CT3_ECUDA;
}

int num_sms() {
  static std::atomic<int> cache[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev >= 0 && dev < 64) {
    const int c = cache[dev].load(std::memory_order_relaxed);
    if (c > 0) return c;
  }
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  if (dev >= 0 && dev < 64) cache[dev].store(n, std::memory_order_relaxed);
  return n;
}

struct ProfRec { int cat; cudaEvent_t a, b; double flops; int launches; };
thread_local bool g_prof_on = false;
thread_local std::vector<ProfRec> g_prof;
ProfScope::ProfScope(cudaStream_t s_, int cat_, double flops_, int launches_)
    : s(s_), cat(cat_), flops(flops_), launches(launches_) {
  if (g_prof_on && cat_ >= 0) { cudaEventCreate(&a); cudaEventCreate(&b); cudaEventRecord(a, s); }
}
ProfScope::~ProfScope() {
  if (a) { cudaEventRecord(b, s); g_prof.push_back({cat, a, b, flops, launches}); }
}

GemmProblem linear_problem(const void* x_split, const void* w_split, const void* bias, int64_t M, int N, int Kpad,
                           float* y) {
  GemmProblem p;
  p.x_split = static_cast<const __nv_bfloat16*>(x_split);
  p.w_split = static_cast<const __nv_bfloat16*>(w_split);
  p.M = (int)M; p.N = N; p.Kpad = Kpad;
  p.epi.bias = static_cast<const float*>(bias);
  p.epi.out_f32 = y; p.epi.ld_f32 = N;
  return p;
}
int run_gemm(const GemmProblem& p, int impl, cudaStream_t s, const char* what) {
  if (const char* bad = gemm_check(p)) {
    snprintf(g_err, sizeof(g_err), "%s: %s", what, bad);
    return CT3_EINVAL;
  }
  const char* gerr = nullptr;
  const int rc = gemm_launch(p, impl, num_sms(), s, &gerr);
  return rc ? fail_launch(rc, what, gerr) : 0;
}

// every source offset sum |stride| * index of a [T,3,H,W] frame tensor must fit in int64, in bytes
static bool frame_extent_fits(int dtype, int T, int H, int W, int64_t stride_t, int64_t stride_c, int64_t stride_h,
                              int64_t stride_w) {
  const int64_t sizes[4] = {T, 3, H, W}, strides[4] = {stride_t, stride_c, stride_h, stride_w};
  const int64_t esize = dtype == CT3_FRAMES_U8 ? 1 : 4;
  int64_t extent = 0;
  for (int i = 0; i < 4; ++i) {
    if (strides[i] == INT64_MIN) return false;
    const int64_t a = strides[i] < 0 ? -strides[i] : strides[i], m = sizes[i] - 1;
    if (m > 0 && a > (INT64_MAX - extent) / m) return false;
    extent += a * m;
  }
  return extent <= INT64_MAX / esize;
}

}  // namespace ct3

using namespace ct3;

// ================================================================================================
extern "C" {

int ct3_version(void) { return 102; }
const char* ct3_last_error(void) { return g_err; }

int ct3_set_option(const char* name, int value) {
  if (!name) return fail(CT3_EINVAL, "null option name%s");
  for (int i = 0; i < OPT_COUNT; ++i)
    if (!strcmp(name, kOptDefs[i].name)) {
      if (value < kOptDefs[i].lo || value > kOptDefs[i].hi) return fail(CT3_EINVAL, "option value out of range: %s", name);
      g_opt[i] = value;
      return 0;
    }
  return fail(CT3_EINVAL, "unknown option %s", name);
}
int ct3_get_option(const char* name, int* value) {
  if (!name || !value) return fail(CT3_EINVAL, "null argument%s");
  for (int i = 0; i < OPT_COUNT; ++i)
    if (!strcmp(name, kOptDefs[i].name)) { *value = g_opt[i]; return 0; }
  return fail(CT3_EINVAL, "unknown option %s", name);
}

int ct3_profile_enable(int on) {
  for (auto& r : g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  g_prof.clear();
  g_prof_on = on != 0;
  return 0;
}
// ms[7], launches[7], gemm_flops (plain linear layers only; category 6 = the fused q|k|v + time-attention kernel): sums since ct3_profile_enable(1); synchronises the recorded events
int ct3_profile_read(double* ms, int* launches, double* gemm_flops) {
  if (!ms || !launches || !gemm_flops) return fail(CT3_EINVAL, "null argument%s");
  for (int i = 0; i < CAT_COUNT; ++i) { ms[i] = 0.0; launches[i] = 0; }
  *gemm_flops = 0.0;
  for (auto& r : g_prof) {
    CK(cudaEventSynchronize(r.b), "profile sync");
    float t = 0.f;
    CK(cudaEventElapsedTime(&t, r.a, r.b), "profile elapsed");
    ms[r.cat] += t;
    launches[r.cat] += r.launches;
    if (r.cat == CAT_GEMM) *gemm_flops += r.flops;
  }
  return 0;
}

int ct3_pyramid_layout(int T, int H4, int W4, int64_t level_off[4], int level_h[4], int level_w[4],
                       int64_t* total_floats) {
  if (T < 1 || H4 < 1 || W4 < 1) return fail(CT3_EINVAL, "bad pyramid shape%s");
  const PyramidLayout p = pyramid_layout(T, H4, W4);
  for (int l = 0; l < kL; ++l) {
    if (p.h[l] < 1 || p.w[l] < 1) return fail(CT3_EINVAL, "feature map too small for 4 pyramid levels%s");
    if (level_off) level_off[l] = p.off[l];
    if (level_h) level_h[l] = p.h[l];
    if (level_w) level_w[l] = p.w[l];
  }
  if (total_floats) *total_floats = p.total;
  return 0;
}

int ct3_prepare_pyramid(const float* fmaps, int T, int H4, int W4, float* pyr, ct3_stream_t stream) {
  if (!fmaps || !pyr) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = check_pyramid(T, H4, W4)) return rc;
  CK(launch_prepare_pyramid(fmaps, T, H4, W4, pyr, (cudaStream_t)stream), "prepare_pyramid");
  return 0;
}

int ct3_pyramid_pools(int T, int H4, int W4, float* pyr, ct3_stream_t stream) {
  if (!pyr) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = check_pyramid(T, H4, W4)) return rc;
  CK(launch_pyramid_pools(T, H4, W4, pyr, (cudaStream_t)stream), "pyramid_pools");
  return 0;
}

int ct3_sample_support(const float* pyr, int T, int H4, int W4, const int32_t* queried_frames,
                       const float* queried_coords, int N, const uint8_t* accumulate_mask, float* support,
                       ct3_stream_t stream) {
  if (!pyr || !queried_frames || !queried_coords || !support) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = check_pyramid(T, H4, W4)) return rc;
  if (N < 1) return fail(CT3_EINVAL, "N must be >= 1%s");
  CK(launch_sample_support(pyr, T, H4, W4, queried_frames, queried_coords, N, accumulate_mask, support,
                           (cudaStream_t)stream), "sample_support");
  return 0;
}

namespace {
// the checks of ct3_prepare_frames and ct3_prepare_frames_crop
int check_frames(const void* src, int dtype, int T, int H, int W, int64_t stride_t, int64_t stride_c, int64_t stride_h,
                 int64_t stride_w, int out_h, int out_w, const float* out) {
  if (!src || !out) return fail(CT3_EINVAL, "null argument%s");
  if (T < 1 || H < 1 || W < 1 || out_h < 1 || out_w < 1) return fail(CT3_EINVAL, "T, H, W, out_h and out_w must be >= 1%s");
  if (dtype != CT3_FRAMES_U8 && dtype != CT3_FRAMES_F32) return fail(CT3_EINVAL, "unknown frame dtype%s");
  if (!frame_extent_fits(dtype, T, H, W, stride_t, stride_c, stride_h, stride_w))
    return fail(CT3_EINVAL, "stride extent overflows int64%s");
  // the kernel indexes the pixels of one output plane with int
  if ((int64_t)out_h * out_w > INT32_MAX) return fail(CT3_EINVAL, "output plane too large%s");
  if ((int64_t)out_h * out_w > INT64_MAX / 12 / T) return fail(CT3_EINVAL, "output too large%s");
  return 0;
}

int check_window(const int32_t* offsets, int H, int W, int crop_h, int crop_w) {
  if (!offsets) return fail(CT3_EINVAL, "null offsets%s");
  if (crop_h < 1 || crop_h > H || crop_w < 1 || crop_w > W)
    return fail(CT3_EINVAL, "crop_h and crop_w must lie in [1, H] and [1, W]%s");
  return 0;
}
}  // namespace

int ct3_prepare_frames(const void* src, int dtype, int T, int H, int W, int64_t stride_t, int64_t stride_c,
                       int64_t stride_h, int64_t stride_w, int out_h, int out_w, float* out, ct3_stream_t stream) {
  if (int rc = check_frames(src, dtype, T, H, W, stride_t, stride_c, stride_h, stride_w, out_h, out_w, out)) return rc;
  CK(launch_prepare_frames(src, dtype, T, H, W, stride_t, stride_c, stride_h, stride_w, nullptr, H, W, out_h, out_w,
                           out, (cudaStream_t)stream),
     "prepare_frames");
  return 0;
}

int ct3_prepare_frames_crop(const void* src, int dtype, int T, int H, int W, int64_t stride_t, int64_t stride_c,
                            int64_t stride_h, int64_t stride_w, const int32_t* offsets, int crop_h, int crop_w,
                            int out_h, int out_w, float* out, ct3_stream_t stream) {
  if (int rc = check_frames(src, dtype, T, H, W, stride_t, stride_c, stride_h, stride_w, out_h, out_w, out)) return rc;
  if (int rc = check_window(offsets, H, W, crop_h, crop_w)) return rc;
  CK(launch_prepare_frames(src, dtype, T, H, W, stride_t, stride_c, stride_h, stride_w, offsets, crop_h, crop_w, out_h,
                           out_w, out, (cudaStream_t)stream),
     "prepare_frames_crop");
  return 0;
}

int ct3_prepare_frames_yuv(const uint8_t* src, int layout, int T, int H, int W, int64_t stride_t, int64_t stride_row,
                           int out_h, int out_w, float* out, ct3_stream_t stream) {
  if (!src || !out) return fail(CT3_EINVAL, "null argument%s");
  if (layout != CT3_YUV_NV12 && layout != CT3_YUV_I420 && layout != CT3_YUV_YUYV)
    return fail(CT3_EINVAL, "unknown YUV layout%s");
  return ct3_prepare_frames_yuv_fmt(src, layout, CT3_MATRIX_BT601, 0, T, H, W, stride_t, stride_row, out_h, out_w, out,
                                    stream);
}

namespace {
// the checks of ct3_prepare_frames_yuv_fmt and ct3_prepare_frames_yuv_crop
int check_frames_yuv(const void* src, int layout, int matrix, int full_range, int T, int H, int W, int64_t stride_t,
                     int64_t stride_row, int out_h, int out_w, const float* out) {
  if (!src || !out) return fail(CT3_EINVAL, "null argument%s");
  const YuvFormat* f = yuv_format(layout);
  if (!f) return fail(CT3_EINVAL, "unknown YUV layout%s");
  if (matrix != CT3_MATRIX_BT601 && matrix != CT3_MATRIX_BT709 && matrix != CT3_MATRIX_BT2020)
    return fail(CT3_EINVAL, "unknown colour matrix%s");
  if (full_range != 0 && full_range != 1) return fail(CT3_EINVAL, "full_range must be 0 or 1%s");
  if (T < 1 || H < 1 || W < 1 || out_h < 1 || out_w < 1) return fail(CT3_EINVAL, "T, H, W, out_h and out_w must be >= 1%s");
  if ((f->ys && (H & 1)) || (f->xs && (W & 1)))
    return fail(CT3_EINVAL, f->ys ? "%s frames must have an even width and height" : "%s frames must have an even width",
                f->name);
  if (f->bytes == 2 && ((stride_t | stride_row) & 1))
    return fail(CT3_EINVAL, "%s strides must be even (16-bit samples)", f->name);
  const int64_t row_bytes = (int64_t)W * f->bytes * (f->family == YuvFormat::kPacked ? 2 : 1);
  if (stride_row < row_bytes) return fail(CT3_EINVAL, "the row stride is below the bytes of a row%s");
  if (f->family == YuvFormat::kPlanar && stride_row != row_bytes)
    return fail(CT3_EINVAL, "%s rows must be dense (stride_row == W * sample bytes)", f->name);
  // the last byte of the last frame: |stride_t| * (T - 1) + stride_row * (rows - 1) + row_bytes - 1 fits int64
  const int64_t rows = yuv_rows(*f, H);
  if (stride_t == INT64_MIN || stride_row > (INT64_MAX - row_bytes) / rows)
    return fail(CT3_EINVAL, "stride extent overflows int64%s");
  const int64_t frame = stride_row * (rows - 1) + row_bytes, at = stride_t < 0 ? -stride_t : stride_t;
  if (T > 1 && at > (INT64_MAX - frame) / (T - 1)) return fail(CT3_EINVAL, "stride extent overflows int64%s");
  if ((int64_t)out_h * out_w > INT32_MAX) return fail(CT3_EINVAL, "output plane too large%s");
  if ((int64_t)out_h * out_w > INT64_MAX / 12 / T) return fail(CT3_EINVAL, "output too large%s");
  return 0;
}
}  // namespace

int ct3_prepare_frames_yuv_fmt(const void* src, int layout, int matrix, int full_range, int T, int H, int W,
                               int64_t stride_t, int64_t stride_row, int out_h, int out_w, float* out,
                               ct3_stream_t stream) {
  if (int rc = check_frames_yuv(src, layout, matrix, full_range, T, H, W, stride_t, stride_row, out_h, out_w, out))
    return rc;
  CK(launch_prepare_frames_yuv(src, layout, matrix, full_range, T, H, W, stride_t, stride_row, nullptr, H, W, out_h,
                               out_w, out, (cudaStream_t)stream),
     "prepare_frames_yuv");
  return 0;
}

int ct3_prepare_frames_yuv_crop(const void* src, int layout, int matrix, int full_range, int T, int H, int W,
                                int64_t stride_t, int64_t stride_row, const int32_t* offsets, int crop_h, int crop_w,
                                int out_h, int out_w, float* out, ct3_stream_t stream) {
  if (int rc = check_frames_yuv(src, layout, matrix, full_range, T, H, W, stride_t, stride_row, out_h, out_w, out))
    return rc;
  if (int rc = check_window(offsets, H, W, crop_h, crop_w)) return rc;
  CK(launch_prepare_frames_yuv(src, layout, matrix, full_range, T, H, W, stride_t, stride_row, offsets, crop_h, crop_w,
                               out_h, out_w, out, (cudaStream_t)stream),
     "prepare_frames_yuv_crop");
  return 0;
}

// ---- the predictor's tail (finish.cu) ----------------------------------------------------------------------------
namespace {
// the checks ct3_finish_tracks and ct3_finish_tracks_scores share
int check_finish(const float* fwd_tracks, const float* fwd_vis, const float* bwd_tracks, const float* bwd_vis,
                 const float* queries, int B, int T, int N, int n_keep, const float* tracks, const uint8_t* visibility) {
  if (!fwd_tracks || !fwd_vis || !queries || !tracks || !visibility) return fail(CT3_EINVAL, "null argument%s");
  if ((bwd_tracks == nullptr) != (bwd_vis == nullptr))
    return fail(CT3_EINVAL, "bwd_tracks and bwd_vis must be given together%s");
  if (B < 1 || T < 1 || N < 1) return fail(CT3_EINVAL, "B, T and N must be >= 1%s");
  if (n_keep < 1 || n_keep > N) return fail(CT3_EINVAL, "n_keep must be in [1, N]%s");
  if (((uintptr_t)fwd_tracks | (uintptr_t)bwd_tracks | (uintptr_t)tracks) & 7)
    return fail(CT3_EINVAL, "tracks must be 8-byte aligned%s");
  // one thread per output element, one-dimensional grid
  if ((int64_t)B * T > (INT64_MAX >> 12) / N || (int64_t)B * T * N > (int64_t)INT32_MAX * 256)
    return fail(CT3_EINVAL, "problem too large%s");
  return 0;
}
}  // namespace

int ct3_finish_tracks(const float* fwd_tracks, const float* fwd_vis, const float* bwd_tracks, const float* bwd_vis,
                      const float* queries, int B, int T, int N, int n_keep, float threshold, float scale_x,
                      float scale_y, float* tracks, uint8_t* visibility, ct3_stream_t stream) {
  if (int rc = check_finish(fwd_tracks, fwd_vis, bwd_tracks, bwd_vis, queries, B, T, N, n_keep, tracks, visibility))
    return rc;
  CK(launch_finish_tracks(fwd_tracks, fwd_vis, bwd_tracks, bwd_vis, queries, B, T, N, n_keep, threshold, scale_x,
                          scale_y, tracks, visibility, (cudaStream_t)stream), "finish_tracks");
  return 0;
}

int ct3_finish_tracks_scores(const float* fwd_tracks, const float* fwd_vis, const float* fwd_conf,
                             const float* bwd_tracks, const float* bwd_vis, const float* bwd_conf, const float* queries,
                             int B, int T, int N, int n_keep, float threshold, float scale_x, float scale_y,
                             float* tracks, uint8_t* visibility, float* score_vis, float* score_conf,
                             ct3_stream_t stream) {
  if (int rc = check_finish(fwd_tracks, fwd_vis, bwd_tracks, bwd_vis, queries, B, T, N, n_keep, tracks, visibility))
    return rc;
  if (!fwd_conf || !score_vis || !score_conf) return fail(CT3_EINVAL, "null argument%s");
  if ((bwd_conf == nullptr) != (bwd_vis == nullptr))
    return fail(CT3_EINVAL, "bwd_conf must be given with the backward pair, and only with it%s");
  CK(launch_finish_tracks_scores(fwd_tracks, fwd_vis, fwd_conf, bwd_tracks, bwd_vis, bwd_conf, queries, B, T, N, n_keep,
                                 threshold, scale_x, scale_y, tracks, visibility, score_vis, score_conf,
                                 (cudaStream_t)stream),
     "finish_tracks_scores");
  return 0;
}

// ---- streaming windows (online.cu) -----------------------------------------------------------------------------
namespace {
constexpr int kOnlineMaxInd = 1 << 30;   // ind + S and |query frame| stay below this: int32 arithmetic in the kernels

// the checks both ct3_online_window_* share; end = window_end's extra conditions.  max_elems: the largest per-stream
// element count of the kernel (S * n for begin, (ind + T - first frame touched) * n for end).  A ring history (ring =
// 1) holds frames [len - cap, len): every frame a kernel reads must lie there.
int check_online(const ct3_online_stream* st, int K, int S, int step, int stride, int N, bool end, int64_t* max_elems,
                 const void* workspace, size_t workspace_bytes) {
  if (!st || !workspace) return fail(CT3_EINVAL, "null argument%s");
  if (K < 1 || K > 65535) return fail(CT3_EINVAL, "K must be in [1, 65535]%s");
  if (S < 2 || stride < 1 || N < 1) return fail(CT3_EINVAL, "S must be >= 2, stride and N >= 1%s");
  if (!end && (step < 1 || step >= S)) return fail(CT3_EINVAL, "step must be in [1, S)%s");
  if (((uintptr_t)workspace & 15)) return fail(CT3_EINVAL, "workspace must be 16-byte aligned%s");
  if (workspace_bytes < (size_t)K * sizeof(ct3_online_stream)) return fail(CT3_ENOSPC, "workspace too small%s");
  int64_t next = 0;
  *max_elems = 0;
  for (int k = 0; k < K; ++k) {
    const ct3_online_stream& s = st[k];
    if (s.n < 1 || s.first != next || (int64_t)s.first + s.n > N)
      return fail(CT3_EINVAL, "the streams' tracks must tile [0, N) in order%s");
    next += s.n;
    if (s.T < 1 || s.T > S) return fail(CT3_EINVAL, "a stream's T must be in [1, S]%s");
    if (s.ind < 0 || (int64_t)s.ind + S > kOnlineMaxInd) return fail(CT3_EINVAL, "a stream's ind must be in [0, 2^30 - S]%s");
    if (s.ring != 0 && s.ring != 1) return fail(CT3_EINVAL, "a stream's ring must be 0 or 1%s");
    if (s.len < 0 || (!s.ring && s.cap < s.len))
      return fail(CT3_EINVAL, "a stream's history must have 0 <= len <= cap%s");
    if (s.ring && s.cap < S) return fail(CT3_EINVAL, "a ring history must hold at least S frames%s");
    const int64_t held = s.ring ? s.len - s.cap : 0;   // the first frame the history still holds
    // a preview (window_end only) writes no history: at ind = 0 it reads none either, so it may have none
    const bool preview = end && s.preview;
    if (end && s.preview != 0 && s.preview != 1) return fail(CT3_EINVAL, "a stream's preview must be 0 or 1%s");
    if (preview && !s.tracks) return fail(CT3_EINVAL, "a preview entry needs an output (tracks)%s");
    const bool no_history = !s.coords && !s.vis && !s.conf && s.cap == 0 && s.len == 0 && !s.ring;
    const bool reads = (end || s.ind > 0) && !(preview && s.ind == 0 && no_history);
    if (reads && (!s.coords || !s.vis || !s.conf)) return fail(CT3_EINVAL, "a stream's history is null%s");
    if (reads && ((uintptr_t)s.coords & 7)) return fail(CT3_EINVAL, "history coords must be 8-byte aligned%s");
    int64_t elems = (int64_t)S * s.n;
    if (!end) {
      if (s.ind > 0 && s.len < (int64_t)s.ind + (S - step))
        return fail(CT3_EINVAL, "a stream's history must hold the window's overlap frames%s");
      if (s.ind > 0 && s.ind < held) return fail(CT3_EINVAL, "the ring no longer holds the window's overlap frames%s");
    } else {
      const int64_t rows = (int64_t)s.ind + s.T;
      if (!s.ring && !preview && s.cap < rows) return fail(CT3_EINVAL, "a stream's history must hold ind + T frames%s");
      if (s.len < s.ind) return fail(CT3_EINVAL, "a stream's history must hold the frames before its window%s");
      int64_t lo = s.ind;   // the first frame the kernel touches
      if (s.tracks) {
        if (!s.visibility || s.n_keep < 1 || s.n_keep > s.n)
          return fail(CT3_EINVAL, "a stream's output needs visibility and n_keep in [1, n]%s");
        if ((uintptr_t)s.tracks & 7) return fail(CT3_EINVAL, "output tracks must be 8-byte aligned%s");
        if (s.out_first < 0 || s.out_first >= rows)
          return fail(CT3_EINVAL, "a stream's out_first must be in [0, ind + T)%s");
        if (s.ring && rows - s.out_first > s.cap)
          return fail(CT3_EINVAL, "a ring stream's output must fit in the ring (ind + T - out_first <= cap)%s");
        if (s.out_first < s.ind && s.out_first < held)
          return fail(CT3_EINVAL, "the ring no longer holds the output's frames before the window%s");
        if (s.out_first < lo) lo = s.out_first;
      }
      elems = (rows - lo) * s.n;
    }
    if (elems > *max_elems) *max_elems = elems;
  }
  if (next != N) return fail(CT3_EINVAL, "the streams' tracks must tile [0, N) in order%s");
  return 0;
}
}  // namespace

int ct3_online_window_begin(const ct3_online_stream* streams_host, int K, int S, int step, int stride, int T_pyr,
                            const int32_t* qframes, const float* qcoords, int N, uint8_t* valid, uint8_t* entering,
                            int32_t* rel, float* coords_init, float* vis_init, float* conf_init, void* workspace,
                            size_t workspace_bytes, ct3_stream_t stream) {
  if (!qframes || !qcoords || !valid || !entering || !rel || !coords_init || !vis_init || !conf_init)
    return fail(CT3_EINVAL, "null argument%s");
  if (((uintptr_t)qcoords | (uintptr_t)coords_init) & 7) return fail(CT3_EINVAL, "coords must be 8-byte aligned%s");
  int64_t max_elems = 0;
  if (int rc = check_online(streams_host, K, S, step, stride, N, false, &max_elems, workspace, workspace_bytes)) return rc;
  for (int k = 0; k < K; ++k)
    if (streams_host[k].frame0 < 0 || (int64_t)streams_host[k].frame0 + S > T_pyr)
      return fail(CT3_EINVAL, "a stream's window must lie in the T_pyr pyramid frames%s");
  cudaStream_t s = (cudaStream_t)stream;
  auto* dev = reinterpret_cast<ct3_online_stream*>(workspace);
  CK(cudaMemcpyAsync(dev, streams_host, (size_t)K * sizeof(ct3_online_stream), cudaMemcpyHostToDevice, s),
     "online_window_begin");
  CK(launch_online_window_begin(dev, K, max_elems, S, step, 1.0f / (float)stride, qframes, qcoords, N, valid, entering,
                                rel, coords_init, vis_init, conf_init, s),
     "online_window_begin");
  return 0;
}

int ct3_online_window_end(const ct3_online_stream* streams_host, int K, int S, int stride, const float* coords,
                          const float* vis, const float* conf, int N, float threshold, void* workspace,
                          size_t workspace_bytes, ct3_stream_t stream) {
  if (!coords || !vis || !conf) return fail(CT3_EINVAL, "null argument%s");
  if ((uintptr_t)coords & 7) return fail(CT3_EINVAL, "coords must be 8-byte aligned%s");
  int64_t max_elems = 0;
  if (int rc = check_online(streams_host, K, S, 1, stride, N, true, &max_elems, workspace, workspace_bytes)) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  auto* dev = reinterpret_cast<ct3_online_stream*>(workspace);
  CK(cudaMemcpyAsync(dev, streams_host, (size_t)K * sizeof(ct3_online_stream), cudaMemcpyHostToDevice, s),
     "online_window_end");
  CK(launch_online_window_end(dev, K, max_elems, (float)stride, coords, vis, conf, N, threshold, s), "online_window_end");
  return 0;
}

int ct3_online_window_end_scores(const ct3_online_stream* streams_host, int K, int S, int stride, const float* coords,
                                 const float* vis, const float* conf, int N, float threshold,
                                 const ct3_online_scores* scores_host, void* workspace, size_t workspace_bytes,
                                 ct3_stream_t stream) {
  if (!coords || !vis || !conf || !scores_host) return fail(CT3_EINVAL, "null argument%s");
  if ((uintptr_t)coords & 7) return fail(CT3_EINVAL, "coords must be 8-byte aligned%s");
  int64_t max_elems = 0;
  if (int rc = check_online(streams_host, K, S, 1, stride, N, true, &max_elems, workspace, workspace_bytes)) return rc;
  // the scores follow the streams in the workspace
  static_assert(sizeof(ct3_online_stream) % alignof(ct3_online_scores) == 0, "scores table misaligned");
  const size_t table = (size_t)K * sizeof(ct3_online_stream);
  if (workspace_bytes < table + (size_t)K * sizeof(ct3_online_scores)) return fail(CT3_ENOSPC, "workspace too small%s");
  for (int k = 0; k < K; ++k) {
    const ct3_online_scores& sc = scores_host[k];
    if ((sc.vis == nullptr) != (sc.conf == nullptr))
      return fail(CT3_EINVAL, "a stream's scores need both vis and conf, or neither%s");
    if (sc.vis && !streams_host[k].tracks)
      return fail(CT3_EINVAL, "a stream's scores need its output (tracks and visibility)%s");
    if (((uintptr_t)sc.vis | (uintptr_t)sc.conf) & 3) return fail(CT3_EINVAL, "scores must be 4-byte aligned%s");
  }
  cudaStream_t s = (cudaStream_t)stream;
  auto* dev = reinterpret_cast<ct3_online_stream*>(workspace);
  auto* dev_scores = reinterpret_cast<ct3_online_scores*>(static_cast<char*>(workspace) + table);
  CK(cudaMemcpyAsync(dev, streams_host, table, cudaMemcpyHostToDevice, s), "online_window_end_scores");
  CK(cudaMemcpyAsync(dev_scores, scores_host, (size_t)K * sizeof(ct3_online_scores), cudaMemcpyHostToDevice, s),
     "online_window_end_scores");
  CK(launch_online_window_end_scores(dev, dev_scores, K, max_elems, (float)stride, coords, vis, conf, N, threshold, s),
     "online_window_end_scores");
  return 0;
}

// ---- track visualiser (render.cu) ------------------------------------------------------------------------------
int ct3_render_prepare(const void* src, int dtype, int T, int H, int W, int64_t stride_t, int64_t stride_c,
                       int64_t stride_h, int64_t stride_w, int pad, int grayscale, uint8_t* out, ct3_stream_t stream) {
  if (!src || !out) return fail(CT3_EINVAL, "null argument%s");
  if (T < 1 || H < 1 || W < 1) return fail(CT3_EINVAL, "T, H and W must be >= 1%s");
  if (T > 65535) return fail(CT3_EINVAL, "T must be <= 65535%s");
  if (pad < 0) return fail(CT3_EINVAL, "pad must be >= 0%s");
  if (grayscale != 0 && grayscale != 1) return fail(CT3_EINVAL, "grayscale must be 0 or 1%s");
  if (dtype != CT3_FRAMES_U8 && dtype != CT3_FRAMES_F32) return fail(CT3_EINVAL, "unknown frame dtype%s");
  if (!frame_extent_fits(dtype, T, H, W, stride_t, stride_c, stride_h, stride_w))
    return fail(CT3_EINVAL, "stride extent overflows int64%s");
  const int64_t ho = (int64_t)H + 2 * (int64_t)pad, wo = (int64_t)W + 2 * (int64_t)pad;
  if (ho > INT32_MAX || wo > INT32_MAX || ho * wo > INT32_MAX) return fail(CT3_EINVAL, "output plane too large%s");
  CK(launch_render_prepare(src, dtype, T, H, W, stride_t, stride_c, stride_h, stride_w, pad, grayscale, out,
                           (cudaStream_t)stream), "render_prepare");
  return 0;
}

int ct3_render_workspace_bytes(int T, int H, int W, int N, int trail, size_t* out_bytes) {
  if (!out_bytes) return fail(CT3_EINVAL, "null argument%s");
  if (T < 1 || H < 1 || W < 1 || N < 1) return fail(CT3_EINVAL, "T, H, W and N must be >= 1%s");
  if (T > 65535) return fail(CT3_EINVAL, "T must be <= 65535%s");
  if (trail < -1) return fail(CT3_EINVAL, "trail must be >= -1%s");
  if ((int64_t)H * W > INT32_MAX) return fail(CT3_EINVAL, "frame plane too large%s");
  if ((int64_t)T * N > INT32_MAX) return fail(CT3_EINVAL, "T * N too large%s");   // draw-order keys u * N + i
  *out_bytes = align_up((size_t)T * H * W * sizeof(int32_t));
  return 0;
}

int ct3_render_tracks(uint8_t* frames, int T, int H, int W, const float* pts, const uint8_t* visible,
                      const uint8_t* colors, const uint8_t* draw_mask, int N, int radius, int linewidth, int trail,
                      int query_frame, const double* alphas, const double* diff, void* workspace,
                      size_t workspace_bytes, ct3_stream_t stream) {
  if (!frames || !pts || !colors || !workspace) return fail(CT3_EINVAL, "null argument%s");
  size_t need = 0;
  if (int rc = ct3_render_workspace_bytes(T, H, W, N, trail, &need)) return rc;
  if (radius < 0 || radius > kRenderMaxRadius) return fail(CT3_EINVAL, "radius must be in [0, 255]%s");
  if (linewidth < 0) return fail(CT3_EINVAL, "linewidth must be >= 0%s");
  if (query_frame < 0 || query_frame >= T) return fail(CT3_EINVAL, "query_frame must be in [0, T)%s");
  if (trail > 0 && !alphas) return fail(CT3_EINVAL, "trail > 0 needs the blend weights (alphas)%s");
  if (int rc = check_space(workspace_bytes, need, "workspace")) return rc;
  CK(launch_render_tracks(frames, T, H, W, pts, visible, colors, draw_mask, N, radius, linewidth, trail, query_frame,
                          alphas, diff, static_cast<int*>(workspace), (cudaStream_t)stream),
     "render_tracks");
  return 0;
}

int ct3_render_flow_workspace_bytes(int T, int N, size_t* out_bytes) {
  if (!out_bytes) return fail(CT3_EINVAL, "null argument%s");
  if (T < 1 || N < 1) return fail(CT3_EINVAL, "T and N must be >= 1%s");
  if ((int64_t)T * N > INT32_MAX) return fail(CT3_EINVAL, "T * N too large%s");
  *out_bytes = align_up(sizeof(unsigned long long));
  return 0;
}

int ct3_render_flow_colors(const float* pts, int T, int N, int query_frame, uint8_t* colors, void* workspace,
                           size_t workspace_bytes, ct3_stream_t stream) {
  if (!pts || !colors || !workspace) return fail(CT3_EINVAL, "null argument%s");
  size_t need = 0;
  if (int rc = ct3_render_flow_workspace_bytes(T, N, &need)) return rc;
  if (query_frame < 0 || query_frame >= T) return fail(CT3_EINVAL, "query_frame must be in [0, T)%s");
  if (workspace_bytes < need) return fail(CT3_EINVAL, "workspace too small%s");
  CK(launch_render_flow_colors(pts, T, N, query_frame, colors, workspace, (cudaStream_t)stream), "render_flow_colors");
  return 0;
}

// ---- Shi-Tomasi corners (corners.cu) -----------------------------------------------------------------------------
namespace {
// the workspace's buffers (lam first: ct3_detect_corners documents it); a null base only measures
CornerWorkspace corner_workspace(void* base, int K, int64_t HW, CornerFrame** fp, size_t* total) {
  Carver c(base);
  CornerWorkspace w;
  w.lam = static_cast<double*>(c.take((size_t)K * HW * sizeof(double)));
  w.cand = static_cast<uint8_t*>(c.take((size_t)K * HW * 16));
  w.sorted = static_cast<int*>(c.take((size_t)K * HW * sizeof(int)));
  w.maxkey = static_cast<unsigned long long*>(c.take((size_t)K * (sizeof(unsigned long long) + sizeof(int))));
  *fp = static_cast<CornerFrame*>(c.take((size_t)K * sizeof(CornerFrame)));
  *total = c.off;
  return w;
}
int check_corner_shape(int K, int H, int W) {
  if (K < 1 || K > 65535) return fail(CT3_EINVAL, "K must be in [1, 65535]%s");
  if (H < 1 || W < 1) return fail(CT3_EINVAL, "H and W must be >= 1%s");
  if ((int64_t)H * W > INT32_MAX) return fail(CT3_EINVAL, "frame plane too large%s");
  if (H > 65535 * 16) return fail(CT3_EINVAL, "H must be <= 1048560%s");
  return 0;
}
}  // namespace

int ct3_corners_workspace_bytes(int K, int H, int W, size_t* bytes) {
  if (!bytes) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = check_corner_shape(K, H, W)) return rc;
  CornerFrame* fp = nullptr;
  corner_workspace(nullptr, K, (int64_t)H * W, &fp, bytes);
  return 0;
}

namespace {
// ct3_detect_corners and ct3_detect_corners_masked: mask null runs the kernels without a mask
int detect_corners(const float* frames, int64_t frame_stride, int K, int H, int W, const ct3_corner_params* params,
                   const float* exclude, const int32_t* exclude_counts, int E_max, const uint8_t* mask,
                   int64_t mask_stride, float* corners, int32_t* counts, void* workspace, size_t workspace_bytes,
                   ct3_stream_t stream) {
  if (!frames || !params || !corners || !counts || !workspace) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = check_corner_shape(K, H, W)) return rc;
  if (int rc = check_aligned(workspace, "workspace")) return rc;
  const int64_t HW = (int64_t)H * W;
  if (frame_stride < 0) return fail(CT3_EINVAL, "frame_stride must be >= 0%s");
  if (K > 1 && frame_stride > (INT64_MAX / 4 - 3 * HW) / (K - 1)) return fail(CT3_EINVAL, "stride extent overflows int64%s");
  if (mask) {
    if (mask_stride < 0) return fail(CT3_EINVAL, "mask_stride must be >= 0%s");
    if (K > 1 && mask_stride > (INT64_MAX - HW) / (K - 1)) return fail(CT3_EINVAL, "mask stride extent overflows int64%s");
  }
  if (E_max < 0 || E_max > INT32_MAX / 2) return fail(CT3_EINVAL, "E_max must be in [0, 2^30)%s");
  std::vector<CornerFrame> fp(K);
  int M = 0;
  for (int k = 0; k < K; ++k) {
    const ct3_corner_params& p = params[k];
    if (p.block_size != 3 && p.block_size != 5 && p.block_size != 7) return fail(CT3_EINVAL, "block_size must be 3, 5 or 7%s");
    if (H < p.block_size || W < p.block_size) return fail(CT3_EINVAL, "H and W must be >= block_size%s");
    if (!(p.quality_level > 0.0 && p.quality_level <= 1.0)) return fail(CT3_EINVAL, "quality_level must be in (0, 1]%s");
    if (p.max_corners < 1) return fail(CT3_EINVAL, "max_corners must be >= 1%s");
    if (!(p.min_distance >= 0.0 && p.min_distance < 1e300)) return fail(CT3_EINVAL, "min_distance must be finite and >= 0%s");
    if (!(p.exclude_radius >= 0.0 && p.exclude_radius < 1e300))
      return fail(CT3_EINVAL, "exclude_radius must be finite and >= 0%s");
    const int E = exclude_counts ? exclude_counts[k] : 0;
    if (E < 0 || E > E_max) return fail(CT3_EINVAL, "exclude_counts must be in [0, E_max]%s");
    if (E > 0 && !exclude) return fail(CT3_EINVAL, "exclusion points given without the exclude buffer%s");
    CornerFrame& f = fp[k];
    f.max_corners = p.max_corners;
    f.block = p.block_size;
    f.E = p.exclude_radius > 0.0 ? E : 0;
    f.quality = p.quality_level;
    f.md2 = p.min_distance * p.min_distance;
    f.r2 = p.exclude_radius * p.exclude_radius;
    const double side = std::floor(p.min_distance);
    f.cs = side < 1.0 ? 1 : side > (double)std::max(H, W) ? std::max(H, W) : (int)side;
    f.gw = (W + f.cs - 1) / f.cs;
    f.gh = (H + f.cs - 1) / f.cs;
    M = std::max(M, p.max_corners);
  }
  if ((int64_t)K * M > INT32_MAX) return fail(CT3_EINVAL, "K * max(max_corners) too large%s");
  CornerFrame* fp_dev = nullptr;
  size_t need = 0;
  const CornerWorkspace ws = corner_workspace(workspace, K, HW, &fp_dev, &need);
  if (int rc = check_space(workspace_bytes, need, "workspace")) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaMemcpyAsync(fp_dev, fp.data(), (size_t)K * sizeof(CornerFrame), cudaMemcpyHostToDevice, s), "detect_corners");
  CK(launch_detect_corners(frames, frame_stride, K, H, W, fp_dev, exclude, E_max, mask, mask_stride, M, corners, counts,
                           ws, num_sms(), s),
     mask ? "detect_corners_masked" : "detect_corners");
  return 0;
}
}  // namespace

int ct3_detect_corners(const float* frames, int64_t frame_stride, int K, int H, int W, const ct3_corner_params* params,
                       const float* exclude, const int32_t* exclude_counts, int E_max, float* corners, int32_t* counts,
                       void* workspace, size_t workspace_bytes, ct3_stream_t stream) {
  return detect_corners(frames, frame_stride, K, H, W, params, exclude, exclude_counts, E_max, nullptr, 0, corners,
                        counts, workspace, workspace_bytes, stream);
}

int ct3_detect_corners_masked(const float* frames, int64_t frame_stride, int K, int H, int W,
                              const ct3_corner_params* params, const float* exclude, const int32_t* exclude_counts,
                              int E_max, const uint8_t* mask, int64_t mask_stride, float* corners, int32_t* counts,
                              void* workspace, size_t workspace_bytes, ct3_stream_t stream) {
  if (!mask) return fail(CT3_EINVAL, "null argument%s");
  return detect_corners(frames, frame_stride, K, H, W, params, exclude, exclude_counts, E_max, mask, mask_stride,
                        corners, counts, workspace, workspace_bytes, stream);
}

int ct3_prepare_masks(const void* src, int dtype, int K, int H, int W, int64_t stride_k, int64_t stride_h,
                      int64_t stride_w, int out_h, int out_w, uint8_t* out, ct3_stream_t stream) {
  if (!src || !out) return fail(CT3_EINVAL, "null argument%s");
  if (dtype != CT3_MASK_U8 && dtype != CT3_MASK_BOOL && dtype != CT3_MASK_F32) return fail(CT3_EINVAL, "unknown mask dtype%s");
  if (K < 1 || K > 65535) return fail(CT3_EINVAL, "K must be in [1, 65535]%s");
  if (H < 1 || W < 1 || out_h < 1 || out_w < 1) return fail(CT3_EINVAL, "H, W, out_h and out_w must be >= 1%s");
  // a [K,H,W] source is a [K,3,H,W] frame tensor whose channel stride is 0
  if (!frame_extent_fits(dtype == CT3_MASK_F32 ? CT3_FRAMES_F32 : CT3_FRAMES_U8, K, H, W, stride_k, 0, stride_h, stride_w))
    return fail(CT3_EINVAL, "stride extent overflows int64%s");
  if ((int64_t)out_h * out_w > INT32_MAX) return fail(CT3_EINVAL, "output plane too large%s");
  CK(launch_prepare_masks(src, dtype == CT3_MASK_F32, K, H, W, stride_k, stride_h, stride_w, out_h, out_w, out,
                          (cudaStream_t)stream), "prepare_masks");
  return 0;
}

// ---- fp32 rows -> split operands of the GEMM engine ----------------------------------------------------------------
int ct3_split_rows(const float* x, int rows, int K, int Kpad, void* x_split, ct3_stream_t stream) {
  if (!x || !x_split || rows < 1 || K < 1 || Kpad < K || (Kpad % 64)) return fail(CT3_EINVAL, "bad split_rows argument%s");
  CK(launch_split_rows(x, rows, K, Kpad, 0, (__nv_bfloat16*)x_split, 0, (cudaStream_t)stream), "split_rows");
  return 0;
}

int ct3_split_rows_fp16(const float* x, int rows, int K, int Kpad, void* x_split, ct3_stream_t stream) {
  if (!x || !x_split || rows < 1 || K < 1 || Kpad < K || (Kpad % 64)) return fail(CT3_EINVAL, "bad split_rows argument%s");
  CK(launch_split_rows(x, rows, K, Kpad, 0, (__nv_bfloat16*)x_split, 0, (cudaStream_t)stream, /*fp16*/ 1), "split_rows");
  return 0;
}

}  // extern "C"
