// render.cu -- the track visualiser (reference cotracker/utils/visualizer.py, draw_tracks_on_video) on device uint8
// frames [T,H,W,3], in place, in stream order.  Every frame comes out bit-identical to the reference's PIL drawing.
//
// Ownership: PIL draws shapes one after the other, so on every pixel the LAST shape that covers it wins.  Here every
// shape scatters its draw-order key into a per-pixel int32 buffer with atomicMax, and a resolve pass writes the colour
// of the winning key and resets the key to -1.  Launches do not grow with the number of tracks:
//   - points: one scatter + one resolve (key = track index i);
//   - trails with tracks_leave_trace == -1 (no blend): one scatter over every (frame t, step s, track i) with key
//     u*N + i, u = first(t) + s (steps are drawn in ascending s, tracks in ascending i within a step) + one resolve;
//   - trails with tracks_leave_trace > 0: per step s one scatter (key = i) and one resolve that also blends the whole
//     frame with what it held before the step, in float64, as the reference's add_weighted does.
//
// Footprints are Pillow's (ImageDraw.ellipse / ImageDraw.line), restated as arithmetic:
//   - ellipse with a bounding box of integer corners (c-r, c+r): Pillow walks one quarter of the curve in doubled
//     coordinates (a = b = 2r) from (a, 0) to (0, b), at each step to whichever of (x, y+2), (x-2, y+2), (x-2, y)
//     has the smallest |a^2 y^2 + b^2 x^2 - a^2 b^2| (ties keep the earlier candidate).  Row dy of the disc covers
//     |dx| <= hi[|dy|], row dy of the one-pixel outline covers lo[|dy|] <= |dx| <= hi[|dy|], with lo/hi the smallest and
//     largest x the walk visits on that row.  A filled ellipse of radius 0 draws nothing; its outline is one pixel.
//     The rows depend on r alone and are computed on the host (make_stencil).
//   - line of width <= 1: Bresenham including both endpoints; the point of step i along the major axis is
//     minor0 + s * floor((2 d_minor i + d_major) / (2 d_major)), so the part inside the frame is walked directly.
//   - wider line: ImagingDrawWideLine's quadrilateral (offsets from ROUND_UP / ROUND_DOWN of (w-1)/2 over the length,
//     in double) filled by Pillow's scanline polygon rule: per row, the float32 crossings (y - y0) * dx + x0 of the
//     non-horizontal edges (an edge ending on the row, unless it is the polygon's last row, counts twice), sorted and
//     filled in pairs from ROUND_UP(left) to ROUND_DOWN(right); horizontal edges are drawn as spans.  Every float
//     operation is an explicit _rn intrinsic, as Pillow's x86-64 build evaluates it (no contraction).
#include <math.h>

#include "../../include/ct3_b200.h"
#include "kernels.cuh"

namespace ct3 {
namespace {

constexpr int kThreads = 256;
constexpr float kCoordLimit = 1073741824.0f;   // 2^30: coordinates at or beyond it (or not finite) draw nothing

struct Stencil {
  int r;
  int16_t lo[kRenderMaxRadius + 1], hi[kRenderMaxRadius + 1];
};

// Pillow's quarter-ellipse walk for a = b = 2r (see the header comment)
void make_stencil(int r, Stencil* st) {
  st->r = r;
  for (int i = 0; i <= r; ++i) st->lo[i] = INT16_MAX, st->hi[i] = -1;
  const int64_t a = 2 * r, a2 = a * a, a2b2 = a2 * a2;
  auto delta = [&](int64_t x, int64_t y) { const int64_t d = a2 * y * y + a2 * x * x - a2b2; return d < 0 ? -d : d; };
  int64_t cx = a, cy = 0;
  for (;;) {
    const int row = (int)(cy / 2), col = (int)(cx / 2);
    if (col < st->lo[row]) st->lo[row] = (int16_t)col;
    if (col > st->hi[row]) st->hi[row] = (int16_t)col;
    if (cx == 0 && cy == a) break;
    int64_t nx = cx, ny = cy + 2, nd = delta(nx, ny);
    if (nx > 1) {
      int64_t d = delta(cx - 2, cy + 2);
      if (nd > d) nx = cx - 2, ny = cy + 2, nd = d;
      d = delta(cx - 2, cy);
      if (nd > d) nx = cx - 2, ny = cy;
    }
    cx = nx, cy = ny;
  }
}

// reference: tracks.long() (truncation toward zero); false when the coordinate is not drawable
__device__ __forceinline__ bool trunc_coord(float v, int* out) {
  if (!(fabsf(v) < kCoordLimit)) return false;   // also false for NaN
  *out = (int)v;                                   // cvt.rzi
  return true;
}
__device__ __forceinline__ bool trunc_coord(double v, int* out) {
  if (!(fabs(v) < (double)kCoordLimit)) return false;
  *out = (int)v;
  return true;
}

__device__ __forceinline__ void put(int* keys, int H, int W, int x, int y, int key) {
  if ((unsigned)x < (unsigned)W && (unsigned)y < (unsigned)H) atomicMax(keys + ((int64_t)y * W + x), key);
}
__device__ __forceinline__ void span(int* keys, int H, int W, int xa, int y, int xb, int key) {
  if ((unsigned)y >= (unsigned)H) return;
  if (xa > xb) { const int t = xa; xa = xb; xb = t; }   // Pillow's hline swaps reversed ends
  if (xa < 0) xa = 0;
  if (xb > W - 1) xb = W - 1;
  int* row = keys + (int64_t)y * W;
  for (int x = xa; x <= xb; ++x) atomicMax(row + x, key);
}

// Pillow's ROUND_UP / ROUND_DOWN on float (f + 0.5F evaluated in float)
__device__ __forceinline__ int round_up_f(float f) {
  return f >= 0.0f ? (int)floorf(__fadd_rn(f, 0.5f)) : -(int)floorf(__fadd_rn(fabsf(f), 0.5f));
}
__device__ __forceinline__ int round_down_f(float f) {
  return f >= 0.0f ? (int)ceilf(__fsub_rn(f, 0.5f)) : -(int)ceilf(__fsub_rn(fabsf(f), 0.5f));
}
__device__ __forceinline__ int round_up_d(double f) {
  return f >= 0.0 ? (int)floor(f + 0.5) : -(int)floor(fabs(f) + 0.5);
}
__device__ __forceinline__ int round_down_d(double f) {
  return f >= 0.0 ? (int)ceil(f - 0.5) : -(int)ceil(fabs(f) - 0.5);
}

// width <= 1: Bresenham with both endpoints, walking only the steps whose major coordinate is inside the frame
__device__ void thin_line(int* keys, int H, int W, int x0, int y0, int x1, int y1, int key) {
  const int64_t dx = x1 >= x0 ? (int64_t)x1 - x0 : (int64_t)x0 - x1, dy = y1 >= y0 ? (int64_t)y1 - y0 : (int64_t)y0 - y1;
  const int xs = x1 >= x0 ? 1 : -1, ys = y1 >= y0 ? 1 : -1;
  const bool xmajor = dx > dy;
  const int64_t dmaj = xmajor ? dx : dy, dmin = xmajor ? dy : dx;
  const int m0 = xmajor ? x0 : y0, n0 = xmajor ? y0 : x0, ms = xmajor ? xs : ys, ns = xmajor ? ys : xs;
  const int M = xmajor ? W : H;
  // steps i in [0, dmaj] with 0 <= m0 + ms*i <= M-1
  int64_t ilo, ihi;
  if (ms > 0) ilo = -(int64_t)m0, ihi = (int64_t)M - 1 - m0;
  else ilo = (int64_t)m0 - (M - 1), ihi = m0;
  if (ilo < 0) ilo = 0;
  if (ihi > dmaj) ihi = dmaj;
  for (int64_t i = ilo; i <= ihi; ++i) {
    const int64_t k = dmaj == 0 ? 0 : (2 * dmin * i + dmaj) / (2 * dmaj);
    const int m = (int)(m0 + ms * i), n = (int)(n0 + ns * k);
    if (xmajor) put(keys, H, W, m, n, key);
    else put(keys, H, W, n, m, key);
  }
}

struct Edge { int x0, y0, xmin, xmax, ymin, ymax; float dx; };

__device__ __forceinline__ Edge make_edge(int x0, int y0, int x1, int y1) {
  Edge e;
  e.xmin = min(x0, x1), e.xmax = max(x0, x1), e.ymin = min(y0, y1), e.ymax = max(y0, y1);
  e.dx = y0 == y1 ? 0.0f : __fdiv_rn((float)((int64_t)x1 - x0), (float)((int64_t)y1 - y0));
  e.x0 = x0, e.y0 = y0;
  return e;
}

__device__ void wide_line(int* keys, int H, int W, int x0, int y0, int x1, int y1, int width, int key) {
  const int dx = x1 - x0, dy = y1 - y0;
  if (dx == 0 && dy == 0) { put(keys, H, W, x0, y0, key); return; }
  const double big = hypot((double)dx, (double)dy);
  const double small = (width - 1) / 2.0;
  const double rmax = round_up_d(small) / big, rmin = round_down_d(small) / big;
  const int dxmin = round_down_d(rmin * dy), dxmax = round_down_d(rmax * dy);
  const int dymin = round_down_d(rmin * dx), dymax = round_down_d(rmax * dx);
  const int vx[4] = {x0 - dxmin, x1 - dxmin, x1 + dxmax, x0 + dxmax};
  const int vy[4] = {y0 + dymax, y1 + dymax, y1 - dymin, y0 - dymin};
  // every loop below is unrolled over constant indices, so the edges and crossings stay in registers
  Edge e[4];
  int ylo = INT32_MAX, yhi = INT32_MIN;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    e[k] = make_edge(vx[k], vy[k], vx[(k + 1) & 3], vy[(k + 1) & 3]);
    ylo = min(ylo, e[k].ymin), yhi = max(yhi, e[k].ymax);
    if (e[k].ymin == e[k].ymax) span(keys, H, W, e[k].xmin, e[k].ymin, e[k].xmax, key);
  }
  const int ya = max(ylo, 0), yb = min(yhi, H - 1);
  for (int y = ya; y <= yb; ++y) {
    // edge k owns slots 2k (its crossing) and 2k+1 (the crossing again where the edge ends on this row); unused
    // slots hold +inf and sort to the end
    float xx[8];
    int j = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const bool on = e[k].ymin != e[k].ymax && y >= e[k].ymin && y <= e[k].ymax;
      const float x = __fadd_rn(__fmul_rn((float)(y - e[k].y0), e[k].dx), (float)e[k].x0);
      const bool twice = on && y == e[k].ymax && y < yhi;
      xx[2 * k] = on ? x : INFINITY;
      xx[2 * k + 1] = twice ? x : INFINITY;
      j += (on ? 1 : 0) + (twice ? 1 : 0);
    }
#pragma unroll
    for (int a = 0; a < 8; ++a)   // odd-even transposition sort of the 8 slots
#pragma unroll
      for (int b = a & 1; b + 1 < 8; b += 2) {
        const float lo = fminf(xx[b], xx[b + 1]), hi = fmaxf(xx[b], xx[b + 1]);
        xx[b] = lo, xx[b + 1] = hi;
      }
#pragma unroll
    for (int k = 1; k < 8; k += 2)
      if (k < j) span(keys, H, W, round_up_f(xx[k - 1]), y, round_down_f(xx[k]), key);
  }
}

// ---- frame preparation: F.pad(value=255) -> optional Grayscale + repeat -> .byte() -----------------------------
template <typename Tin>
__global__ void __launch_bounds__(kThreads) prepare_kernel(const Tin* __restrict__ src, int64_t st, int64_t sc,
                                                           int64_t sh, int64_t sw, int H, int W, int pad, int gray,
                                                           uint8_t* __restrict__ out) {
  const int Ho = H + 2 * pad, Wo = W + 2 * pad;
  const int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (p >= (int64_t)Ho * Wo) return;
  const int t = blockIdx.y;
  const int y = (int)(p / Wo) - pad, x = (int)(p % Wo) - pad;
  float v[3];
  if (y < 0 || y >= H || x < 0 || x >= W) {
    v[0] = v[1] = v[2] = 255.0f;
  } else {
    const Tin* f = src + (int64_t)t * st + (int64_t)y * sh + (int64_t)x * sw;
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = (float)f[c * sc];
  }
  uint8_t o[3];
  if (gray) {
    // torchvision rgb_to_grayscale: (0.2989 * r + 0.587 * g + 0.114 * b) in float32, one rounding per operation
    const float l = __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, v[0]), __fmul_rn(0.587f, v[1])), __fmul_rn(0.114f, v[2]));
    o[0] = o[1] = o[2] = (uint8_t)(int)l;   // .to(uint8) / .byte(): truncation
  } else {
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = (uint8_t)(int)v[c];
  }
  uint8_t* d = out + ((int64_t)t * Ho * Wo + p) * 3;
  d[0] = o[0], d[1] = o[1], d[2] = o[2];
}

// ---- points ------------------------------------------------------------------------------------------------------
// thread = (track i, footprint row); blockIdx.y = frame t
__global__ void __launch_bounds__(kThreads) points_scatter_kernel(const float* __restrict__ pts,
                                                                  const uint8_t* __restrict__ visible,
                                                                  const uint8_t* __restrict__ draw_mask, int N,
                                                                  Stencil st, int H, int W, int* __restrict__ keys) {
  const int rows = 2 * st.r + 1;
  const int64_t g = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (g >= (int64_t)N * rows) return;
  const int i = (int)(g / rows), dy = (int)(g % rows) - st.r;
  const int t = blockIdx.y;
  if (draw_mask && !draw_mask[i]) return;
  const float* q = pts + ((int64_t)t * N + i) * 2;
  int cx, cy;
  if (!trunc_coord(q[0], &cx) || !trunc_coord(q[1], &cy) || cx == 0 || cy == 0) return;
  const bool fill = visible ? visible[(int64_t)t * N + i] != 0 : true;
  if (fill && st.r == 0) return;   // Pillow draws nothing for a filled ellipse of zero size
  const int ady = dy < 0 ? -dy : dy;
  const int hi = st.hi[ady], lo = st.lo[ady];
  int* kf = keys + (int64_t)t * H * W;
  const int y = cy + dy;
  if (fill) {
    span(kf, H, W, cx - hi, y, cx + hi, i);
  } else {
    span(kf, H, W, cx - hi, y, cx - lo, i);
    if (lo > 0 || hi > 0) span(kf, H, W, cx + lo, y, cx + hi, i);
  }
}

// ---- trails ------------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ int first_index(int t, int trail) {
  return trail > 0 ? (t - trail > 0 ? t - trail : 0) : 0;
}

__device__ __forceinline__ bool seg_point(const float* pts, const double* diff, int S1, int N, int t, int u, int first,
                                          int i, int* x, int* y) {
  const float* q = pts + ((int64_t)u * N + i) * 2;
  int px, py;
  if (!trunc_coord(q[0], &px) || !trunc_coord(q[1], &py)) return false;
  if (!diff) { *x = px, *y = py; return true; }
  // compensate_for_camera_motion: int(track - diff[t, u]) in float64
  const double* d = diff + ((int64_t)t * S1 + (u - first)) * 2;
  return trunc_coord((double)px - d[0], x) && trunc_coord((double)py - d[1], y);
}

// thread = track i; blockIdx.y = frame t; blockIdx.z = step s - s0.  key = blend ? i : u*N + i
__global__ void __launch_bounds__(kThreads) trail_scatter_kernel(const float* __restrict__ pts,
                                                                 const uint8_t* __restrict__ draw_mask,
                                                                 const double* __restrict__ diff, int N, int H, int W,
                                                                 int t0, int trail, int S1, int s0, int linewidth,
                                                                 int* __restrict__ keys) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= N) return;
  const int t = t0 + blockIdx.y, s = s0 + blockIdx.z;
  const int first = first_index(t, trail);
  const int u = first + s;
  if (u + 1 > t) return;   // frame t draws steps s = 0 .. t - first - 1
  if (draw_mask && !draw_mask[i]) return;
  int xa, ya, xb, yb;
  if (!seg_point(pts, diff, S1, N, t, u, first, i, &xa, &ya) || xa == 0 || ya == 0) return;
  if (!seg_point(pts, diff, S1, N, t, u + 1, first, i, &xb, &yb)) return;
  const int key = trail > 0 ? i : u * N + i;
  int* kf = keys + (int64_t)t * H * W;
  if (linewidth <= 1) thin_line(kf, H, W, xa, ya, xb, yb, key);
  else wide_line(kf, H, W, xa, ya, xb, yb, linewidth, key);
}

// ---- resolve -----------------------------------------------------------------------------------------------------
// mode 0: points (colour row t), 1: unblended trails (key = u*N + i), 2: blended trail step s
__global__ void __launch_bounds__(kThreads) resolve_kernel(uint8_t* __restrict__ frames, int* __restrict__ keys,
                                                           const uint8_t* __restrict__ colors, int N, int64_t plane,
                                                           int t0, int mode, int trail, int s,
                                                           const double* __restrict__ alphas, int S) {
  const int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (p >= plane) return;
  const int t = t0 + blockIdx.y;
  const int64_t o = (int64_t)t * plane + p;
  int* kp = keys + o;
  const int k = *kp;
  uint8_t* px = frames + o * 3;
  if (mode != 2) {
    if (k < 0) return;
    const uint8_t* c = colors + ((mode == 0 ? (int64_t)t * N : 0) + k) * 3;
    px[0] = c[0], px[1] = c[1], px[2] = c[2];
    *kp = -1;
    return;
  }
  const int first = first_index(t, trail);
  if (first + s + 1 > t) return;   // no step s in this frame
  // add_weighted(drawn, a, original, 1 - a, 0): (drawn * a + original * (1 - a) + 0).astype(uint8), in float64
  const double a = alphas[((int64_t)t * S + s) * 2], b = alphas[((int64_t)t * S + s) * 2 + 1];
  const uint8_t* c = nullptr;
  if (k >= 0) { c = colors + ((int64_t)(first + s) * N + k) * 3; *kp = -1; }
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const double orig = (double)px[ch], drawn = c ? (double)c[ch] : orig;
    const double v = __dadd_rn(__dadd_rn(__dmul_rn(drawn, a), __dmul_rn(orig, b)), 0.0);
    px[ch] = (uint8_t)(int)v;
  }
}

// ---- optical-flow colours: flow_vis.flow_to_color(tracks - tracks[query_frame]) ---------------------------------
// Every operation is the float64 one numpy performs, as an explicit _rn intrinsic (no contraction); only atan2 is
// CUDA's (within 2 ulp of the correctly rounded value, as numpy's own SIMD and libm atan2 are not exact either).
constexpr int kWheel = 55;   // Middlebury colour wheel: RY 15, YG 6, GC 4, CB 11, BM 13, MR 6
struct ColorWheel { uint8_t c[kWheel][3]; };

// make_colorwheel(): floor(255 * i / n) is exact in integers for these sizes
ColorWheel make_colorwheel() {
  ColorWheel w;
  const int n[6] = {15, 6, 4, 11, 13, 6};
  // per segment: the channel held at 255, the channel that ramps, and whether it ramps up (floor(255*i/n)) or down
  const int full[6] = {0, 1, 1, 2, 2, 0}, ramp[6] = {1, 0, 2, 1, 0, 2}, up[6] = {1, 0, 1, 0, 1, 0};
  int k = 0;
  for (int s = 0; s < 6; ++s)
    for (int i = 0; i < n[s]; ++i, ++k) {
      w.c[k][0] = w.c[k][1] = w.c[k][2] = 0;
      const int r = 255 * i / n[s];
      w.c[k][full[s]] = 255;
      w.c[k][ramp[s]] = (uint8_t)(up[s] ? r : 255 - r);
    }
  return w;
}

// tracks.long() of one coordinate, kept where |x|, |y| < 2^30 so that squared norms of differences fit in int64:
// NaN counts as 0 and anything at or beyond +-2^30 (infinities included) as +-(2^30 - 1)
__device__ __forceinline__ int64_t flow_coord(float v) {
  if (v != v) return 0;
  if (!(fabsf(v) < kCoordLimit)) return v > 0.0f ? (1 << 30) - 1 : -((1 << 30) - 1);
  return (int64_t)(int)v;
}

__device__ __forceinline__ void flow_at(const float* __restrict__ pts, int N, int query_frame, int64_t e, int64_t* u,
                                        int64_t* v) {
  const int64_t i = e % N;
  const float* p = pts + e * 2;
  const float* q = pts + ((int64_t)query_frame * N + i) * 2;
  *u = flow_coord(p[0]) - flow_coord(q[0]);
  *v = flow_coord(p[1]) - flow_coord(q[1]);
}

// rad2max = max over all (t, n) of u*u + v*v in int64 (max of sqrt(float64(.)) is sqrt(float64(max)): both monotone).
// Grid-stride, one atomicMax per warp on a zeroed u64: the maximum does not depend on the order.
__global__ void __launch_bounds__(kThreads) flow_radmax_kernel(const float* __restrict__ pts, int N, int query_frame,
                                                               int64_t total, unsigned long long* __restrict__ rad2max) {
  unsigned long long m = 0;
  for (int64_t e = (int64_t)blockIdx.x * kThreads + threadIdx.x; e < total; e += (int64_t)gridDim.x * kThreads) {
    int64_t u, v;
    flow_at(pts, N, query_frame, e, &u, &v);
    const unsigned long long r2 = (unsigned long long)(u * u + v * v);
    m = r2 > m ? r2 : m;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long x = __shfl_xor_sync(0xffffffffu, m, o);
    m = x > m ? x : m;
  }
  if ((threadIdx.x & 31) == 0 && m > 0) atomicMax(rad2max, m);
}

// thread = entry (t, n): flow_uv_to_colors after the normalisation by rad_max + 1e-5
__global__ void __launch_bounds__(kThreads) flow_color_kernel(const float* __restrict__ pts, int N, int query_frame,
                                                              int64_t total,
                                                              const unsigned long long* __restrict__ rad2max,
                                                              ColorWheel wheel, uint8_t* __restrict__ colors) {
  const int64_t e = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (e >= total) return;
  int64_t iu, iv;
  flow_at(pts, N, query_frame, e, &iu, &iv);
  const double den = __dadd_rn(__dsqrt_rn(__ull2double_rn(*rad2max)), 1e-5);
  const double u = __ddiv_rn(__ll2double_rn(iu), den), v = __ddiv_rn(__ll2double_rn(iv), den);
  const double rad = __dsqrt_rn(__dadd_rn(__dmul_rn(u, u), __dmul_rn(v, v)));
  const double a = __ddiv_rn(atan2(-v, -u), 3.141592653589793);              // np.arctan2(-v, -u) / np.pi
  const double fk = __dmul_rn(__ddiv_rn(__dadd_rn(a, 1.0), 2.0), (double)(kWheel - 1));
  const int k0 = (int)floor(fk);
  const int k1 = k0 + 1 == kWheel ? 0 : k0 + 1;
  const double f = __dsub_rn(fk, (double)k0), g = __dsub_rn(1.0, f);
  // an atan2 a few ulp below -pi gives k0 = -1, which numpy's indexing reads as the last row
  const int r0 = k0 < 0 ? k0 + kWheel : k0;
  uint8_t* out = colors + e * 3;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const double c0 = __ddiv_rn((double)wheel.c[r0][ch], 255.0), c1 = __ddiv_rn((double)wheel.c[k1][ch], 255.0);
    double col = __dadd_rn(__dmul_rn(g, c0), __dmul_rn(f, c1));
    col = rad <= 1.0 ? __dsub_rn(1.0, __dmul_rn(rad, __dsub_rn(1.0, col))) : __dmul_rn(col, 0.75);
    out[ch] = (uint8_t)(int)floor(__dmul_rn(255.0, col));
  }
}

unsigned blocks(int64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

}  // namespace

cudaError_t launch_render_flow_colors(const float* pts, int T, int N, int query_frame, uint8_t* colors, void* workspace,
                                      cudaStream_t s) {
  const int64_t total = (int64_t)T * N;
  unsigned long long* rad2max = static_cast<unsigned long long*>(workspace);
  cudaError_t e = cudaMemsetAsync(rad2max, 0, sizeof(unsigned long long), s);
  if (e != cudaSuccess) return e;
  const unsigned nb = blocks(total);
  flow_radmax_kernel<<<nb < 1024 ? nb : 1024, kThreads, 0, s>>>(pts, N, query_frame, total, rad2max);
  flow_color_kernel<<<nb, kThreads, 0, s>>>(pts, N, query_frame, total, rad2max, make_colorwheel(), colors);
  return cudaGetLastError();
}

cudaError_t launch_render_prepare(const void* src, int dtype, int T, int H, int W, int64_t st, int64_t sc, int64_t sh,
                                  int64_t sw, int pad, int gray, uint8_t* out, cudaStream_t s) {
  const int64_t plane = (int64_t)(H + 2 * pad) * (W + 2 * pad);
  const dim3 grid(blocks(plane), T);
  if (dtype == CT3_FRAMES_U8)
    prepare_kernel<uint8_t><<<grid, kThreads, 0, s>>>(static_cast<const uint8_t*>(src), st, sc, sh, sw, H, W, pad, gray,
                                                      out);
  else
    prepare_kernel<float><<<grid, kThreads, 0, s>>>(static_cast<const float*>(src), st, sc, sh, sw, H, W, pad, gray,
                                                    out);
  return cudaGetLastError();
}

cudaError_t launch_render_tracks(uint8_t* frames, int T, int H, int W, const float* pts, const uint8_t* visible,
                                 const uint8_t* colors, const uint8_t* draw_mask, int N, int radius, int linewidth,
                                 int trail, int query_frame, const double* alphas, const double* diff, int* keys,
                                 cudaStream_t s) {
  const int64_t plane = (int64_t)H * W;
  cudaError_t e = cudaMemsetAsync(keys, 0xff, (size_t)T * plane * sizeof(int), s);   // every key -1
  if (e != cudaSuccess) return e;
  const int t0 = query_frame + 1;
  if (trail != 0 && t0 < T) {
    const int S = trail > 0 ? (trail < T - 1 ? trail : T - 1) : T - 1;   // most steps any frame draws
    const int nt = T - t0;
    if (trail < 0) {
      trail_scatter_kernel<<<dim3(blocks(N), nt, S), kThreads, 0, s>>>(pts, draw_mask, diff, N, H, W, t0, trail, S + 1,
                                                                       0, linewidth, keys);
      resolve_kernel<<<dim3(blocks(plane), nt), kThreads, 0, s>>>(frames, keys, colors, N, plane, t0, 1, trail, 0,
                                                                  nullptr, S);
    } else {
      for (int st = 0; st < S; ++st) {
        trail_scatter_kernel<<<dim3(blocks(N), nt, 1), kThreads, 0, s>>>(pts, draw_mask, diff, N, H, W, t0, trail,
                                                                         S + 1, st, linewidth, keys);
        resolve_kernel<<<dim3(blocks(plane), nt), kThreads, 0, s>>>(frames, keys, colors, N, plane, t0, 2, trail, st,
                                                                    alphas, S);
      }
    }
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  Stencil st;
  make_stencil(radius, &st);
  points_scatter_kernel<<<dim3(blocks((int64_t)N * (2 * radius + 1)), T), kThreads, 0, s>>>(pts, visible, draw_mask, N,
                                                                                           st, H, W, keys);
  resolve_kernel<<<dim3(blocks(plane), T), kThreads, 0, s>>>(frames, keys, colors, N, plane, 0, 0, trail, 0, nullptr,
                                                             1);
  return cudaGetLastError();
}

}  // namespace ct3
