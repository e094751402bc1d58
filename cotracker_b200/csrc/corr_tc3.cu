// corr_tc3.cu -- fused bilinear sampling + 4-D correlation, production kernel ("CorrBlock.sample" of the north star):
//
//   vol[(n,t,l)][k*49 + (a*7+b)] = < bilinear(F_l[t], cx/2^l + a-3, cy/2^l + b-3) , S_l[n, k, :] >
//   (get_correlation_feat + einsum, cotracker3_online.py:130-143, cotracker3_offline.py:144-156)
// NB the volume row is SUPPORT-MAJOR here (the reference and the other correlation kernels emit (a*7+b)*49 + k): a
// thread owns one support vector k, so its 49 values are one contiguous run of the row; corr_mlp.fc1 is multiplied with
// a copy of its weights whose columns are permuted the same way (api_loop.cu, Layout::corr_fc1_t).
//
// Correlate-then-interpolate like corr_tc2.cu (bilinear sampling is linear in the feature map, so the tensor cores
// correlate the RAW 8x8 texel patch around the track with the 49 support vectors and the epilogue blends the 64 raw
// correlations into the 49 sampled ones), but with the MMA TRANSPOSED: the support vectors are the M side and the
// texels the N side, so a thread of the epilogue owns ONE support vector k and sees all 64 raw correlations of a
// frame in its accumulator row.  Both blends (x, then y) become plain FMAs on the thread's own registers with
// warp-uniform weights: no shuffles, no exchange of texel rows between lanes.
//
//   pyramid  : ONE fp16 plane per level [T][H][W][128] (made once per update-loop call); texels are rounded to fp16
//              (2^-12 relative), the support vectors are exact to a split fp16 pair (prec.corr = 2, DESIGN.md section 2)
//   B tile   [128 texel rows x 64 ch] : rows f*64 + y*8 + x = the raw texels of 2 frames; each (frame, K-half) is ONE
//              4-D TMA box (64 ch x 8 x 8 x 1) landing in the 128B-swizzled K-major operand layout; ring of 3 K-half
//              slots (16 KiB), each freed as soon as the MMAs reading it have completed
//   A tiles  4 x [128 x 64 ch] : {hi, lo} plane x K-half of the 49 support vectors of (n,l) in rows 0..48 (rows 49..127
//              stay zero), built once per unit by 2 warps.  The hi and lo planes are CONCATENATED ALONG K:
//              D += S_hi[kh] . F[kh]^T  and  D += S_lo[kh] . F[kh]^T  accumulate into the same registers, so row k
//              holds the complete (S_hi + S_lo)[k] . F and the epilogue needs no exchange between warps.
//              (prec.corr = 1 skips the lo MMAs: single fp16 product.)
//   D        [64 x 128] fp32: one m64n128 wgmma accumulator of the MMA warpgroup (rows 0..48 live, columns = texels
//              f*64 + y*8 + x), stored to one of 2 accumulator tiles in shared memory (rows 0..48)
//   epilogue : 2 groups x 2 warps take tiles round-robin; thread = support vector k.
//              Per frame: 64 accumulator columns -> x-blend -> y-blend -> 49 sampled correlations ->
//              convert -> volume-row image in shared memory -> bulk shared->global copy of the whole 9.5 KiB row.
//              A border clamp only turns the tap indices into a clamped SHIFT of the interior pattern
//              (idx = clamp(a + d, 0, 7), d uniform per frame and axis), so every case -- interior, any border, far
//              outside -- runs the same register code through a warp-uniform switch on d; the per-sample weights
//              (exactly grid_sample's border-clamped taps, canonicalised to the shift pattern;
//              tests/test_host_logic.py brute-forces that this always works) are computed once per tile by the
//              otherwise idle lanes of the TMA warp.  The blend code exists ONCE (frame loop not unrolled): a fully
//              unrolled epilogue is hundreds of KB of SASS and thrashes the instruction cache.
//   schedule : persistent CTAs; a unit = (track n, level l) = T frames of one support operand.  A CTA's first unit is
//              blockIdx.x, the others come from a global counter (SMs differ in speed on this kernel).
//   L2       : texel boxes are loaded evict_last, volume rows stored evict_first (the 3.9 GB write stream would
//              otherwise push the pyramid, read ~100x, out of L2)
// Warps (12): 0,1 / 4,5 epilogue groups, 2 TMA issuer (+ tap tables), 3 idle, 6,7 support builders (6 also draws
// the units), 8..11 MMA warpgroup.
#include "gemm.cuh"
#include "kernels.cuh"

namespace ct3 {
namespace {

constexpr int TMA_WARP = 2;
constexpr int SB_WARP0 = 6;               // warps 6, 7 build the support operand
constexpr int MMA_WARP0 = 8;              // warps 8..11: the MMA warpgroup
constexpr int MMA_WARPS = 4;
constexpr int NGROUP = 2;                 // epilogue groups: warps {0,1}, {4,5}  (warp 3 idle)
constexpr int THREADS = 12 * 32;          // 168 registers per thread
constexpr int NSLOT = 3;                  // texel ring: slots of one K-half (64 channels) of a 2-frame tile
constexpr int A_SLOT = 16384;             // [128 texel rows x 128 B] fp16
constexpr int S_TILE = 16384;             // one (plane, K-half) of S: [128 rows x 128 B], rows 49..127 zero
constexpr int S_BYTES = 4 * S_TILE;       // tile index = plane * 2 + K-half
constexpr int NACC = 2;                   // accumulator tiles in shared memory: [64 rows][ACC_LD] fp32, rows 0..48 live
constexpr int ACC_LD = 128 + 4;
constexpr int ACC_BYTES = 64 * ACC_LD * 4;
constexpr int NPARAM = 8;                 // tap-table ring (a tile's slot is rewritten only after its epilogue read it)
constexpr int PRM_WORDS = 64;             // per tile: [frame 2][axis 2]{u[7], w[7]} = 56 floats, d[2][2] ints, flag
constexpr int ROW_BYTES_SPLIT = 2 * kVolPad * 2;   // 9728
constexpr int ROW_BYTES_H16 = kVolPad * 2;         // 4864
constexpr int IMG_GROUP = 2 * ROW_BYTES_SPLIT;
constexpr int OFF_A = 0;
constexpr int OFF_S = OFF_A + NSLOT * A_SLOT;
constexpr int OFF_IMG = OFF_S + S_BYTES;
constexpr int OFF_ACC = OFF_IMG + NGROUP * IMG_GROUP;
constexpr int OFF_PARAM = OFF_ACC + NACC * ACC_BYTES;
constexpr int OFF_BAR = OFF_PARAM + NPARAM * PRM_WORDS * 4;
constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
static_assert(SMEM_BYTES <= 232448, "shared memory budget");

struct Corr3Args {
  PyramidLayout lay;
  const float* support;        // [4][49, N, 128]
  const uint8_t* track_valid;  // [N] or null
  const float* coords;         // [T, N, 2]
  int T, N;
  uint16_t* vol;               // [N*T*4, 2*kVolPad] split bf16, or [N*T*4, kVolPad] fp16 (V16)
  int* unit_counter;           // zeroed before the launch: units beyond the first one per CTA are handed out dynamically
  FrameMap fm;                 // pyramid frame of (track, t): each box is one frame of the unit's own frame row
};
struct Corr3Maps {
  CUtensorMap m[kL];           // per level: fp16 dims (128, W, H, T_pyr), box (64, 8, 8, 1), 128B swizzle
};

__device__ __forceinline__ uint32_t sw128(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }
__host__ __device__ constexpr int clamp07(int v) { return v < 0 ? 0 : (v > 7 ? 7 : v); }

// origin of the 8-wide box holding every tap of the 7 border-clamped samples around c (size >= 8), and the shift of
// the tap pattern relative to the interior one (0 = interior)
__device__ __forceinline__ void box_origin8(float c, int size, int& origin, int& d) {
  const float cc = fminf(fmaxf(c, -16.f), (float)size + 16.f);
  const int base = (int)floorf(cc) - kR;
  origin = max(0, min(base, size - 8));
  d = max(-7, min(base - origin, 7));
}

// one border-clamped sample coordinate (exactly grid_sample(align_corners=True, padding_mode="border")) expressed in
// the shift pattern: value = u * box[clamp07(a + d)] + w * box[clamp07(a + d + 1)].  Returns false if the sample does
// not fit the pattern (never happens: brute-forced in tests/test_host_logic.py).
__device__ __forceinline__ bool tap_weights(float c, int a, int size, int origin, int d, float& u, float& w) {
  const float x = fminf(fmaxf(c + (float)(a - kR), 0.f), (float)(size - 1));
  const float xf = floorf(x);
  const int x0 = (int)xf;
  const float fr = x - xf;
  const int s0 = min(max(x0 - origin, 0), 7);
  const int s1 = (fr > 0.f) ? min(max(min(x0 + 1, size - 1) - origin, 0), 7) : s0;
  const int i0 = clamp07(a + d), i1 = clamp07(a + d + 1);
  if (s0 == i0 && (fr == 0.f || s1 == i1)) { u = 1.f - fr; w = fr; return true; }
  if (fr == 0.f && s0 == i1) { u = 0.f; w = 1.f; return true; }   // c + offset rounded up to the next integer in fp32
  u = 0.f; w = 0.f;
  return false;
}

// hx[y][a] = u[a] * v[y*8 + clamp07(a + D)] + w[a] * v[y*8 + clamp07(a + D + 1)]   for the 8 texel rows of a frame
template <int D>
__device__ __forceinline__ void xblend(const float (&v)[64], const float (&u)[7], const float (&w)[7], float (&hx)[8][7]) {
#pragma unroll
  for (int y = 0; y < 8; ++y)
#pragma unroll
    for (int a = 0; a < 7; ++a) hx[y][a] = u[a] * v[y * 8 + clamp07(a + D)] + w[a] * v[y * 8 + clamp07(a + D + 1)];
}
__device__ __forceinline__ void xblend_dispatch(int d, const float (&v)[64], const float (&u)[7], const float (&w)[7],
                                                float (&hx)[8][7]) {
  if (d == 0) { xblend<0>(v, u, w, hx); return; }   // interior tiles (the majority): a direct branch, no jump table
  switch (d) {   // warp-uniform
    case -7: xblend<-7>(v, u, w, hx); break;
    case -6: xblend<-6>(v, u, w, hx); break;
    case -5: xblend<-5>(v, u, w, hx); break;
    case -4: xblend<-4>(v, u, w, hx); break;
    case -3: xblend<-3>(v, u, w, hx); break;
    case -2: xblend<-2>(v, u, w, hx); break;
    case -1: xblend<-1>(v, u, w, hx); break;
    case 0: xblend<0>(v, u, w, hx); break;
    case 1: xblend<1>(v, u, w, hx); break;
    case 2: xblend<2>(v, u, w, hx); break;
    case 3: xblend<3>(v, u, w, hx); break;
    case 4: xblend<4>(v, u, w, hx); break;
    case 5: xblend<5>(v, u, w, hx); break;
    case 6: xblend<6>(v, u, w, hx); break;
    default: xblend<7>(v, u, w, hx); break;
  }
}
// out[a*7 + b] = uy[b] * hx[clamp07(b + D)][a] + wy[b] * hx[clamp07(b + D + 1)][a]
template <int D>
__device__ __forceinline__ void yblend(const float (&hx)[8][7], const float (&u)[7], const float (&w)[7], float (&out)[kP]) {
#pragma unroll
  for (int b = 0; b < 7; ++b)
#pragma unroll
    for (int a = 0; a < 7; ++a) out[a * 7 + b] = u[b] * hx[clamp07(b + D)][a] + w[b] * hx[clamp07(b + D + 1)][a];
}
__device__ __forceinline__ void yblend_dispatch(int d, const float (&hx)[8][7], const float (&u)[7], const float (&w)[7],
                                                float (&out)[kP]) {
  if (d == 0) { yblend<0>(hx, u, w, out); return; }
  switch (d) {
    case -7: yblend<-7>(hx, u, w, out); break;
    case -6: yblend<-6>(hx, u, w, out); break;
    case -5: yblend<-5>(hx, u, w, out); break;
    case -4: yblend<-4>(hx, u, w, out); break;
    case -3: yblend<-3>(hx, u, w, out); break;
    case -2: yblend<-2>(hx, u, w, out); break;
    case -1: yblend<-1>(hx, u, w, out); break;
    case 0: yblend<0>(hx, u, w, out); break;
    case 1: yblend<1>(hx, u, w, out); break;
    case 2: yblend<2>(hx, u, w, out); break;
    case 3: yblend<3>(hx, u, w, out); break;
    case 4: yblend<4>(hx, u, w, out); break;
    case 5: yblend<5>(hx, u, w, out); break;
    case 6: yblend<6>(hx, u, w, out); break;
    default: yblend<7>(hx, u, w, out); break;
  }
}

// Epilogue of one 2-frame tile for one thread = support vector k (accumulator row k).  The blend code exists ONCE (the
// frame loop is not unrolled; see the file header).
template <bool V16>
__device__ __forceinline__ void epilogue_tile(const float* acc_tile, int q, int lane, int grp, int nf,
                                              const float* prm, uint16_t* img, uint64_t* d_empty_bar, uint16_t* vrow) {
  constexpr int ROW_BYTES = V16 ? ROW_BYTES_H16 : ROW_BYTES_SPLIT;
  const int k = q * 32 + lane;                        // q in {0, 1}
  const bool live = k < kP;
  const int bar_id = 1 + grp;                         // named barrier of this group (64 threads)
  const float* arow = acc_tile + k * ACC_LD;         // rows >= 49 are never written and their results never stored
  const int* iprm = reinterpret_cast<const int*>(prm) + 56;
  if (iprm[4] == 0) asm volatile("trap;");   // a sample outside the shift pattern: impossible (see file header)
  if (k == 0) bulk_wait_read0();             // previous tile's row images have left shared memory ...
  asm volatile("bar.sync %0, 64;" ::"r"(bar_id) : "memory");   // ... before anyone overwrites them
#pragma unroll 1
  for (int f = 0; f < nf; ++f) {
    float hx[8][7];
    {
      float v[64];
      acc_row_ld<64>(arow + f * 64, v);
      float ux[7], wx[7];
#pragma unroll
      for (int a = 0; a < 7; ++a) { ux[a] = prm[(f * 2 + 0) * 14 + a]; wx[a] = prm[(f * 2 + 0) * 14 + 7 + a]; }
      xblend_dispatch(iprm[2 * f], v, ux, wx, hx);
    }
    float uy[7], wy[7];
#pragma unroll
    for (int b = 0; b < 7; ++b) { uy[b] = prm[(f * 2 + 1) * 14 + b]; wy[b] = prm[(f * 2 + 1) * 14 + 7 + b]; }
    const int dy = iprm[2 * f + 1];
    if (f == nf - 1) {
      // every accumulator read of this tile has completed and nothing below reads the tap table any more: releasing the
      // accumulator is also what eventually lets the TMA warp recycle the table slot
      __syncwarp();
      if (lane == 0) mbar_arrive(d_empty_bar);
    }
    float out[kP];
    yblend_dispatch(dy, hx, uy, wy, out);
    if (live) {
      // support-major volume row: element k*49 + i (i = a*7 + b), i.e. this thread's 49 values are CONTIGUOUS: one
      // 2-byte edge element (the first if the offset is odd, else the last) + 24 aligned 4-byte pairs per plane
      const bool odd = (k & 1) != 0;
      uint16_t* dst = img + f * (ROW_BYTES / 2) + k * kP;
      uint32_t* ph = reinterpret_cast<uint32_t*>(dst + (odd ? 1 : 0));
      if (V16) {
#pragma unroll
        for (int j = 0; j < 24; ++j) ph[j] = pack_h2(odd ? out[2 * j + 1] : out[2 * j], odd ? out[2 * j + 2] : out[2 * j + 1]);
        dst[odd ? 0 : 48] = __half_as_ushort(__float2half_rn(odd ? out[0] : out[48]));
      } else {
        uint32_t* pl = reinterpret_cast<uint32_t*>(dst + kVolPad + (odd ? 1 : 0));
#pragma unroll
        for (int j = 0; j < 24; ++j) {
          uint32_t hi, lo;
          split2(odd ? out[2 * j + 1] : out[2 * j], odd ? out[2 * j + 2] : out[2 * j + 1], hi, lo);
          ph[j] = hi;
          pl[j] = lo;
        }
        const bf16pair ed = split_bf16(odd ? out[0] : out[48]);
        dst[odd ? 0 : 48] = __bfloat16_as_ushort(ed.hi);
        dst[kVolPad + (odd ? 0 : 48)] = __bfloat16_as_ushort(ed.lo);
      }
    }
  }
  fence_proxy_async_smem();                   // image writes -> visible to the bulk-copy (async proxy) reads
  asm volatile("bar.sync %0, 64;" ::"r"(bar_id) : "memory");
  if (k == 0) {
#pragma unroll
    for (int t2 = 0; t2 < 2; ++t2)
      if (t2 < nf)
        bulk_store_s2g_hint(vrow + (int64_t)t2 * kL * (ROW_BYTES / 2), reinterpret_cast<uint8_t*>(img) + t2 * ROW_BYTES, ROW_BYTES,
                            l2_policy_evict_first());
    bulk_commit();
  }
}

template <bool V16, bool ONEPROD>
__global__ void __launch_bounds__(THREADS, 1)
corr_patch_t_kernel(const __grid_constant__ Corr3Args g, const __grid_constant__ Corr3Maps maps, int num_units) {
  constexpr int ROW_BYTES = V16 ? ROW_BYTES_H16 : ROW_BYTES_SPLIT;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* a_full = bars;                          // [NSLOT] TMA -> MMA         (count 1 + tx bytes)
  uint64_t* a_empty = bars + NSLOT;                 // [NSLOT] MMA -> TMA         (one arrive per MMA warp)
  uint64_t* d_full = bars + 2 * NSLOT;              // [NACC] MMA -> epilogue group  (one arrive per MMA warp)
  uint64_t* d_empty = bars + 2 * NSLOT + NACC;      // [NACC] epilogue group -> MMA  (count 2)
  uint64_t* s_full = bars + 2 * NSLOT + 2 * NACC;       // builders -> MMA, per unit  (count 2)
  uint64_t* s_empty = bars + 2 * NSLOT + 2 * NACC + 1;  // MMA -> builders, per unit  (one arrive per MMA warp)
  float* acc_base = reinterpret_cast<float*>(smem + OFF_ACC);
  // Unit queue.  A unit = (track n, level l) = T frames of one support operand; SMs differ by up to 10 % in speed on
  // this kernel (distance to the L2 slices), so only the first unit of a CTA is static (blockIdx.x) and the others
  // come from a global counter.  The first builder warp -- the role that runs furthest ahead -- draws the numbers and
  // publishes them here in order; every other role reads entry ui when it gets there (an entry is rewritten 8 units
  // later, no role lags that far).  -1 ends every role's loop.
  volatile int* unit_q = reinterpret_cast<volatile int*>(bars + 2 * NSLOT + 2 * NACC + 2);   // [8]
  volatile int* unit_tail = unit_q + 8;                                    // number of published entries
  auto unit_at = [&](uint32_t ui) -> int {
    uint32_t spins = 0;
    while (*unit_tail <= (int)ui) { if (++spins > (1u << 28)) asm volatile("trap;"); }
    __threadfence_block();
    return unit_q[ui & 7];
  };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_unit = (g.T + 1) / 2;

  // one-time: zero S (rows 49..127 of every tile stay zero forever) and the row images (K padding stays zero)
  for (int i = threadIdx.x; i < S_BYTES / 16; i += THREADS) reinterpret_cast<uint4*>(smem + OFF_S)[i] = make_uint4(0, 0, 0, 0);
  for (int i = threadIdx.x; i < NGROUP * IMG_GROUP / 16; i += THREADS) reinterpret_cast<uint4*>(smem + OFF_IMG)[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async_smem();
  if (threadIdx.x == 0) {
    for (int i = 0; i < NSLOT; ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], MMA_WARPS);
    }
    for (int i = 0; i < NACC; ++i) {
      mbar_init(&d_full[i], MMA_WARPS);
      mbar_init(&d_empty[i], 2);
    }
    mbar_init(s_full, 2);
    mbar_init(s_empty, MMA_WARPS);
    unit_q[0] = (int)blockIdx.x < num_units ? (int)blockIdx.x : -1;
    *unit_tail = 1;
    fence_barrier_init();
    for (int l = 0; l < kL; ++l) tma_prefetch_desc(&maps.m[l]);
  }
  __syncthreads();

  if (warp == TMA_WARP) {
    // ================================================================== TMA issuer + tap tables (whole warp)
    uint32_t it = 0, hc = 0;   // tile / K-half slot counters
    // the 67 MB pyramid is read ~100x (6.7 GB of texel boxes per launch) while 3.9 GB of volume rows stream out: keep
    // the texels in L2 (evict_last) and let the volume rows go first (evict_first in the epilogue's bulk copies)
    const uint64_t keep = l2_policy_evict_last();
    // lane -> (frame, axis, a) of the tap this lane evaluates for every tile
    const int pf = lane / 14, pax = (lane % 14) / 7, pa = lane % 7;
    for (uint32_t ui = 0;; ++ui) {
      const int u = unit_at(ui);
      if (u < 0) break;
      const int n = u / kL, l = u % kL;
      const int H = g.lay.h[l], W = g.lay.w[l];
      const float inv = 1.0f / (float)(1 << l);
      const int32_t* frow = frame_row(g.fm, n, g.T);
      for (int t0 = 0; t0 < g.T; t0 += 32) {
        const int tl = min(t0 + lane, g.T - 1);
        const float2 c = __ldg(reinterpret_cast<const float2*>(g.coords + ((int64_t)tl * g.N + n) * 2));
        const int cnt = min(32, g.T - t0);
        for (int k = 0; k < cnt; k += 2, ++it) {
          const int k1 = min(k + 1, 31);
          const float cx0 = __shfl_sync(0xffffffffu, c.x, k) * inv, cy0 = __shfl_sync(0xffffffffu, c.y, k) * inv;
          const float cx1 = __shfl_sync(0xffffffffu, c.x, k1) * inv, cy1 = __shfl_sync(0xffffffffu, c.y, k1) * inv;
          int bx0, by0, bx1, by1, dx0, dy0, dx1, dy1;
          box_origin8(cx0, W, bx0, dx0);
          box_origin8(cy0, H, by0, dy0);
          box_origin8(cx1, W, bx1, dx1);
          box_origin8(cy1, H, by1, dy1);
          // The first K-half slot of this tile doubles as the gate of the table slot: slot it % 8 was last used by
          // tile it - 8; the ring slot waited for here was freed by MMAs of tile it - 2, which were issued after
          // they had the accumulator that tile it - 4's epilogue had released after reading its table.
          mbar_wait_spin(&a_empty[hc % NSLOT], ((hc / NSLOT) & 1u) ^ 1u);
          {
            float* prm = reinterpret_cast<float*>(smem + OFF_PARAM) + (it % NPARAM) * PRM_WORDS;
            bool ok = true;
            if (lane < 28) {
              const float cc = pf ? (pax ? cy1 : cx1) : (pax ? cy0 : cx0);
              const int size = pax ? H : W;
              const int org = pf ? (pax ? by1 : bx1) : (pax ? by0 : bx0);
              const int dd = pf ? (pax ? dy1 : dx1) : (pax ? dy0 : dx0);
              float uu, ww;
              ok = tap_weights(cc, pa, size, org, dd, uu, ww);
              prm[(pf * 2 + pax) * 14 + pa] = uu;
              prm[(pf * 2 + pax) * 14 + 7 + pa] = ww;
            }
            const bool all_ok = __all_sync(0xffffffffu, ok);
            if (lane == 0) {
              int* ip = reinterpret_cast<int*>(prm) + 56;
              ip[0] = dx0; ip[1] = dy0; ip[2] = dx1; ip[3] = dy1;
              ip[4] = all_ok ? 1 : 0;
            }
          }
          __syncwarp();   // table stores of all lanes precede the arrive below (-> a_full -> d_full -> epilogue)
          if (elect_one()) {
            const int nf = (k + 1 < cnt) ? 2 : 1;
#pragma unroll
            for (int kh = 0; kh < 2; ++kh) {
              const uint32_t h = hc + kh;
              const int sl = h % NSLOT;
              if (kh == 1) mbar_wait_spin(&a_empty[sl], ((h / NSLOT) & 1u) ^ 1u);
              mbar_arrive_expect_tx(&a_full[sl], (uint32_t)(nf * (A_SLOT / 2)));
              uint8_t* dst = smem + OFF_A + sl * A_SLOT;
              tma_load_4d_hint(dst, &maps.m[l], kh * 64, bx0, by0, map_frame(frow, t0 + k), &a_full[sl], keep);
              if (nf == 2)
                tma_load_4d_hint(dst + 8192, &maps.m[l], kh * 64, bx1, by1, map_frame(frow, t0 + k + 1), &a_full[sl], keep);
            }
          }
          hc += 2;        // every lane tracks the slot counter (the table gate above is a warp-wide wait)
          __syncwarp();
        }
      }
    }
  } else if (warp >= MMA_WARP0) {
    // ================================================================== MMA warpgroup
    uint32_t it = 0, ui = 0, hc = 0;
    const uint32_t s_base = smem_u32(smem + OFF_S);
    for (;; ++ui) {
      if (unit_at(ui) < 0) break;
      mbar_wait(s_full, ui & 1u);
      for (int tp = 0; tp < tiles_per_unit; ++tp, ++it) {
        const int acc = it % NACC;
        float d[64];   // D[support k][texel]: rows 0..63 of S (49 live) x the 128 texels of the tile
#pragma unroll
        for (int kh = 0; kh < 2; ++kh, ++hc) {
          const int sl = hc % NSLOT;
          mbar_wait(&a_full[sl], (hc / NSLOT) & 1u);
          if (kh == 0) mbar_wait(&d_empty[acc], ((it / NACC) & 1u) ^ 1u);
          wgmma_fence();
          const uint32_t f_base = smem_u32(smem + OFF_A + sl * A_SLOT);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            // D[support k][texel] += S_lo[k] . F^T + S_hi[k] . F^T over this K-half (hi and lo concatenated along K)
            const uint64_t df = gmma_desc_sw128(f_base + j * 32);
            if (!ONEPROD)
              wgmma_tile<128, true>(d, gmma_desc_sw128(s_base + (uint32_t)((2 + kh) * S_TILE + j * 32)), df, (kh | j) != 0 ? 1u : 0u);
            wgmma_tile<128, true>(d, gmma_desc_sw128(s_base + (uint32_t)(kh * S_TILE + j * 32)), df,
                                  (!ONEPROD || (kh | j) != 0) ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait0(d);
          __syncwarp();
          if (lane == 0) mbar_arrive(&a_empty[sl]);
        }
        acc_store<128>(d, acc_base + acc * (ACC_BYTES / 4), ACC_LD, kP);
        __syncwarp();
        if (lane == 0) mbar_arrive(&d_full[acc]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(s_empty);       // this warp's MMAs of the unit have all completed
    }
  } else if (warp == SB_WARP0 || warp == SB_WARP0 + 1) {
    // ================================================================== support builders (A operand, once per unit)
    const int sb = warp - SB_WARP0;
    const int atom = lane >> 4, chunk = (lane & 15) >> 1, half = lane & 1;  // where this lane's 4 channels live
    uint8_t* s0 = smem + OFF_S;
    uint32_t ui = 0;
    for (;; ++ui) {
      if (sb == 0 && ui > 0) {           // draw the next unit and publish it
        int nu = 0;
        if (lane == 0) {
          nu = (int)gridDim.x + atomicAdd(g.unit_counter, 1);
          if (nu >= num_units) nu = -1;
          unit_q[ui & 7] = nu;
          __threadfence_block();
          *unit_tail = (int)ui + 1;
        }
      }
      const int u = unit_at(ui);
      if (u < 0) break;
      const int n = u / kL, l = u % kL;
      const bool valid = g.track_valid == nullptr || g.track_valid[n] != 0;
      float4 rows[25];
#pragma unroll
      for (int j = 0; j < 25; ++j) {
        const int p = sb + 2 * j;
        rows[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p < kP && valid)
          rows[j] = __ldg(reinterpret_cast<const float4*>(g.support + ((int64_t)l * kP * g.N + (int64_t)p * g.N + n) * kD) + lane);
      }
      if (ui > 0) mbar_wait(s_empty, (ui - 1) & 1u);   // MMAs of the previous unit have retired
#pragma unroll
      for (int j = 0; j < 25; ++j) {
        const int p = sb + 2 * j;
        if (p < kP) {
          uint32_t h0, l0, h1, l1;
          split2_h(rows[j].x, rows[j].y, h0, l0);
          split2_h(rows[j].z, rows[j].w, h1, l1);
          const uint32_t off = (uint32_t)(atom * S_TILE) + sw128(p, chunk) + (uint32_t)(half * 8);   // K-half = atom
          *reinterpret_cast<uint2*>(s0 + off) = make_uint2(h0, h1);                 // hi plane tiles 0, 1
          *reinterpret_cast<uint2*>(s0 + 2 * S_TILE + off) = make_uint2(l0, l1);    // lo plane tiles 2, 3
        }
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(s_full);
    }
  } else if ((warp & 3) < 2) {
    // ================================================================== epilogue: warps {0,1}, {4,5}
    const int grp = warp >> 2;                 // tiles with it % NGROUP == grp
    const int q = warp & 3;                    // rows 32q .. 32q+31 of the accumulator tile
    uint16_t* img = reinterpret_cast<uint16_t*>(smem + OFF_IMG + grp * IMG_GROUP);
    const float* prm_base = reinterpret_cast<const float*>(smem + OFF_PARAM);
    uint32_t it = 0;
    for (uint32_t ui = 0;; ++ui) {
      const int u = unit_at(ui);
      if (u < 0) break;
      const int n = u / kL, l = u % kL;
      for (int tp = 0; tp < tiles_per_unit; ++tp, ++it) {
        if ((int)(it % NGROUP) != grp) continue;
        const int acc = it % NACC;
        mbar_wait(&d_full[acc], (it / NACC) & 1u);
        const float* prm = prm_base + (it % NPARAM) * PRM_WORDS;
        const int nf = (2 * tp + 1 < g.T) ? 2 : 1;
        uint16_t* vrow = g.vol + (((int64_t)n * g.T + 2 * tp) * kL + l) * (ROW_BYTES / 2);
        epilogue_tile<V16>(acc_base + acc * (ACC_BYTES / 4), q, lane, grp, nf, prm, img, &d_empty[acc], vrow);
      }
    }
    if (q == 0 && lane == 0) bulk_wait0();     // outstanding volume-row copies of this group
  }
}

template <bool V16, bool ONEPROD>
cudaError_t launch_variant(const Corr3Args& g, const Corr3Maps& maps, int num_units, int num_sms, cudaStream_t s) {
  static DeviceOnce attr;
  cudaError_t e = once_per_device(attr, [&] {
    return cudaFuncSetAttribute(corr_patch_t_kernel<V16, ONEPROD>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  });
  if (e != cudaSuccess) return e;
  const int grid = num_units < num_sms ? num_units : num_sms;
  corr_patch_t_kernel<V16, ONEPROD><<<grid, THREADS, SMEM_BYTES, s>>>(g, maps, num_units);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_corr_patch_t(const __nv_bfloat16* pyr_half, int H4, int W4, const float* support,
                                const uint8_t* track_valid, const float* coords, int T, int N, int count,
                                __nv_bfloat16* vol, int vol16, int one_product, int num_sms, cudaStream_t s, int T_pyr,
                                const FrameMap& fm) {
  Corr3Args g;
  g.lay = pyramid_layout(T_pyr, H4, W4);
  g.support = support;
  g.track_valid = track_valid;
  g.coords = coords;
  g.T = T;
  g.N = N;
  g.vol = reinterpret_cast<uint16_t*>(vol);
  g.fm = fm;
  // every level of the pyramid workspace has room for two 16-bit planes (launch_split_pyramid); this kernel's single
  // fp16 plane uses the first half, so the unit counter can live right behind level 0's plane
  const size_t plane0 = (size_t)T_pyr * g.lay.h[0] * g.lay.w[0] * kD * 2;
  g.unit_counter = reinterpret_cast<int*>(reinterpret_cast<uintptr_t>(pyr_half) + ((plane0 + 15) & ~(size_t)15));
  cudaError_t e0 = cudaMemsetAsync(g.unit_counter, 0, sizeof(int), s);
  if (e0 != cudaSuccess) return e0;
  Corr3Maps maps;
  for (int l = 0; l < kL; ++l) {
    const uint64_t W = (uint64_t)g.lay.w[l], H = (uint64_t)g.lay.h[l];
    if (W < 8 || H < 8) return cudaErrorInvalidValue;
    const uint64_t dims[4] = {(uint64_t)kD, W, H, (uint64_t)T_pyr};
    const uint64_t strides[3] = {(uint64_t)kD * 2, W * kD * 2, H * W * kD * 2};
    const uint32_t box[4] = {64, 8, 8, 1};
    if (!encode_tensor_map(&maps.m[l], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, pyr_half + 2 * g.lay.off[l], dims, strides,
                           box, CU_TENSOR_MAP_SWIZZLE_128B))
      return cudaErrorInvalidValue;
  }
  const int num_units = count * kL;
  if (one_product)
    return vol16 ? launch_variant<true, true>(g, maps, num_units, num_sms, s)
                 : launch_variant<false, true>(g, maps, num_units, num_sms, s);
  return vol16 ? launch_variant<true, false>(g, maps, num_units, num_sms, s)
               : launch_variant<false, false>(g, maps, num_units, num_sms, s);
}

}  // namespace ct3
