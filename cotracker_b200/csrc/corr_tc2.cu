// corr_tc2.cu -- the split-bf16 (prec.corr = 3) kernel of the correlate-then-interpolate form of the fused sampling +
// 4-D correlation (every pyramid level at least 8x8 texels; corr_tc3.cu runs prec.corr 1 and 2, corr_tc.cu covers
// smaller maps, corr.cu is the fp32 SIMT check).
//
//   vol[(n,t,l)][(a*7+b)*49 + k] = < bilinear(F_l[t], cx/2^l + a-3, cy/2^l + b-3) , S_l[n, k, :] >
//   (get_correlation_feat + einsum, cotracker3_online.py:130-143, cotracker3_offline.py:144-156)
//
// Bilinear sampling is linear in the feature map, so the 49 sampled vectors never have to exist:
//   < sum_j w_j F[p_j] , S_k >  =  sum_j w_j < F[p_j] , S_k >.
// The tensor cores correlate the RAW 8x8 texel patch around the track with the 49 support vectors, and the
// epilogue blends the 64 raw correlations into the 49 sampled ones (separable, border clamp per sample exactly as
// grid_sample(padding_mode="border") does).  What this removes from the per-frame shared-memory budget of
// corr_tc.cu: the fp32 patch reads of the samplers, the split-bf16 A-tile writes, and the output staging image.
//
//   pyramid : a split-bf16 copy [level][plane hi|lo][T][H][W][128] made once per update-loop call
//   A tile  [128 x 128] : rows f*64 + y*8 + x = the raw texels of 2 frames; each (frame, plane, K-half) is ONE 4-D
//             TMA box (64 ch x 8 x 8 x 1) landing directly in the 128B-swizzled K-major operand layout; the 64 KiB ring
//             is split between the two groups (each owns the slots of its own tiles), each slot freed as soon as the
//             MMAs reading it have completed
//   B tile  [128 x 128] : rows 0..63 hi plane / 64..127 lo plane of the 49 support vectors of (n,l) (rows 49..63
//             of each plane zero), built once per unit by 2 warps
//   D       [128 x 128] : fp32 wgmma accumulators of the group that owns the tile: A_hi x [S_hi ; S_lo] (N=128, A_hi
//             fetched once for both products) and A_lo x S_hi (N=64 into columns 0..63); columns k and 64+k are added
//             in registers and the [128 x 64] sum goes to the group's accumulator tile in shared memory
//   epilogue (2 groups x 4 warps = 2 warpgroups, alternating tiles; each runs the MMAs of its own tiles) ->
//             x-blend by warp shuffles inside each 8-texel row -> y-blend: interior tiles entirely in registers (next
//             texel row = 8 lanes up, texel row 4 crosses the warp boundary through a 3 KiB exchange buffer); tiles
//             with a border clamp through a shared [row][a][k] buffer and a per-row tap table -> one thread per
//             volume row -> split-bf16 byte image of the two 9728-byte volume rows (reusing the blend buffer, K
//             padding zero) -> one bulk shared->global copy (TMA engine) per 9728-byte volume row
// Warps: 0 TMA issuer, 1 idle, 2..3 support builders, 4..11 the two MMA + epilogue groups.
// Diagnostics: -DCT3_TRACE records a clock64 timeline of CTA 0 (8 events per tile) and prints it after the 3rd launch.
#include <cstdio>
#include "gemm.cuh"
#include "kernels.cuh"

namespace ct3 {
namespace {

constexpr int TMA_WARP = 0;               // warp 1 idle
constexpr int SB_WARP0 = 2;               // 2 support-builder warps
constexpr int EPI_WARP0 = 4;              // warps 4..7 group 0, 8..11 group 1: each a warpgroup, MMA (wgmma) + epilogue
constexpr int THREADS = 12 * 32;
// Precision (products per correlation FLOP; DESIGN.md section 2): texels split bf16 hi|lo, support split bf16,
// A_hi x [S_hi;S_lo] + A_lo x S_hi (rel. err ~2^-17).
constexpr int A_PLANE = 16384;            // one 16-bit plane of a slot: [128 rows x 128 B]
constexpr int A_RING = 65536;             // ring bytes: 2 slots of hi|lo
constexpr int A_SLOT = 2 * A_PLANE;       // one K-half (64 channels) of a 2-frame tile
constexpr int NSLOT = A_RING / A_SLOT;
// Tiles alternate between the two MMA + epilogue groups, and each group owns half of the ring: K-half kh of tile it
// goes to slot (it & 1) * NSLOT/2 + u % (NSLOT/2), u = (it >> 1) * 2 + kh, in phase u / (NSLOT/2).  A slot is then only
// ever consumed by one group, in order, so a parity wait can never alias a phase two completions ahead.
__device__ __forceinline__ void ring_slot(uint32_t it, int kh, int& sl, uint32_t& parity) {
  constexpr uint32_t SPG = NSLOT / 2;
  const uint32_t u = (it >> 1) * 2u + (uint32_t)kh;
  sl = (int)((it & 1u) * SPG + u % SPG);
  parity = (u / SPG) & 1u;
}
constexpr int BAR_STRIDE = 4;             // barrier words per ring array in the barrier block (>= NSLOT)
constexpr int S_HALF = 2 * 8192;          // one K-half of S: [hi rows 0..63 | lo rows 64..127] x 128 B = one N=128 operand
constexpr int S_BYTES = 2 * S_HALF;       // 32 KiB
constexpr int H_A = 52;                   // floats per (texel row, a): 49 + pad, keeps every vector 16-byte aligned
constexpr int H_ROW = 7 * H_A;            // floats per texel row
constexpr int H_FRAME = 8 * H_ROW;        // floats: x-blended correlations [row 8][a 7][k 52] of one frame
constexpr int H_GROUP = 2 * H_FRAME * 4;  // bytes per epilogue group (2 frames)
constexpr int ROW_BYTES_SPLIT = 2 * kVolPad * 2;   // 9728: one volume row image [hi | lo] (split bf16)
constexpr int ROW_BYTES_H16 = kVolPad * 2;         // 4864: one volume row image, single fp16 plane
static_assert(2 * ROW_BYTES_SPLIT <= H_GROUP, "the output image of a tile reuses the blend buffer");
constexpr int ACC_LD = 64 + 4;            // per group: accumulator tile [128 rows][ACC_LD] fp32 (MMA registers -> row per thread)
constexpr int ACC_BYTES = 128 * ACC_LD * 4;
constexpr int NPARAM = 8;                 // parameter ring: a tile's slot may only be rewritten after its epilogue read it
constexpr int OFF_A = 0;
constexpr int OFF_S = OFF_A + A_RING;
constexpr int OFF_H = OFF_S + S_BYTES;
constexpr int OFF_TAB = OFF_H + 2 * H_GROUP;     // [group 2][frame 2][b 8] x {wy, row0*H_ROW, row1*H_ROW, -}
constexpr int XCH_GROUP = 2 * 7 * H_A * 4;       // texel row 4 of both frames: [frame][a][k], register y-blend path
constexpr int OFF_XCH = OFF_TAB + 2 * 2 * 8 * 16;
constexpr int OFF_PARAM = OFF_XCH + 2 * XCH_GROUP;   // [slot NPARAM][frame 2] x {cx, cy, box_x, box_y}
constexpr int OFF_ACC = OFF_PARAM + NPARAM * 2 * 16;
constexpr int OFF_BAR = OFF_ACC + 2 * ACC_BYTES;
constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
static_assert(SMEM_BYTES <= 232448, "shared memory budget");

struct Corr2Args {
  PyramidLayout lay;
  const float* support;        // [4][49, N, 128]
  const uint8_t* track_valid;  // [N] or null
  const float* coords;         // [T, N, 2]
  int T, N;
  int T_pyr;                   // frames of the pyramid copy (plane stride of the TMA map's dim 3)
  uint16_t* vol;               // [N*T*4, 2*kVolPad] split bf16, or [N*T*4, kVolPad] fp16 (V16)
  long long* trace;            // CT3_TRACE builds: [256 tiles][8 events] clock64 of CTA 0
  FrameMap fm;                 // pyramid frame of (track, t): each box is one frame of the unit's own frame row
};
#ifdef CT3_TRACE
#define TRACE(tile, ev) do { if (blockIdx.x == 0 && (tile) < 256) g.trace[(tile) * 8 + (ev)] = clock64(); } while (0)
#else
#define TRACE(tile, ev) do { } while (0)
#endif
struct Corr2Maps {
  CUtensorMap m[kL];           // per level: 16-bit dims (128, W, H, planes*T_pyr), box (64, 8, 8, 1), 128B swizzle
};

__device__ __forceinline__ uint32_t sw128(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }

// origin of the 8-wide box holding every tap of the 7 border-clamped samples around c (size >= 8)
__device__ __forceinline__ int box_origin8(float c, int size) {
  const float cc = fminf(fmaxf(c, -16.f), (float)size + 16.f);
  return max(0, min((int)floorf(cc) - kR, size - 8));
}

// one border-clamped sample coordinate -> (tap0, tap1) relative to the box origin and the weight of tap1.
// A zero weight folds tap1 onto tap0, which also absorbs the fp32 case c + offset rounding up to an integer.
__device__ __forceinline__ void tap_pair(float c, int off, int size, int origin, int& s0, int& s1, float& w) {
  const float x = fminf(fmaxf(c + (float)off, 0.f), (float)(size - 1));
  const float xf = floorf(x);
  const int x0 = (int)xf;
  w = x - xf;
  s0 = min(max(x0 - origin, 0), 7);
  s1 = (w > 0.f) ? min(max(min(x0 + 1, size - 1) - origin, 0), 7) : s0;
}

template <bool V16>
__global__ void __launch_bounds__(THREADS, 1)
corr_patch_tc_kernel(const __grid_constant__ Corr2Args g, const __grid_constant__ Corr2Maps maps, int num_units) {
  constexpr int ROW_BYTES = V16 ? ROW_BYTES_H16 : ROW_BYTES_SPLIT;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* a_full = bars;                  // [NSLOT] TMA -> MMA         (count 1 + tx bytes)
  uint64_t* a_empty = bars + BAR_STRIDE;    // [NSLOT] MMA -> TMA         (one arrive per warp of the consuming group)
  uint64_t* s_full = bars + 2 * BAR_STRIDE;      // builders -> MMA, per unit  (count 2)
  uint64_t* s_empty = bars + 2 * BAR_STRIDE + 1; // MMA -> builders, per unit  (one arrive per warp of both groups)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_unit = (g.T + 1) / 2;

  // one-time: zero S (rows 49..63 stay zero forever)
  for (int i = threadIdx.x; i < S_BYTES / 16; i += THREADS) reinterpret_cast<uint4*>(smem + OFF_S)[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async_smem();
  if (threadIdx.x == 0) {
    for (int i = 0; i < NSLOT; ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], 4);
    }
    mbar_init(s_full, 2);
    mbar_init(s_empty, 8);
    fence_barrier_init();
    for (int l = 0; l < kL; ++l) tma_prefetch_desc(&maps.m[l]);
  }
  __syncthreads();

  if (warp == TMA_WARP) {
    // ================================================================== TMA issuer (whole warp walks, lane 0 issues)
    uint32_t it = 0;   // tile counter
    for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
      const int n = u / kL, l = u % kL;
      const int H = g.lay.h[l], W = g.lay.w[l];
      const float inv = 1.0f / (float)(1 << l);
      const int32_t* frow = frame_row(g.fm, n, g.T);
      for (int t0 = 0; t0 < g.T; t0 += 32) {
        // coordinates of up to 32 frames in one round trip (lane = frame), then broadcast per tile
        const int tl = min(t0 + lane, g.T - 1);
        const float2 c = __ldg(reinterpret_cast<const float2*>(g.coords + ((int64_t)tl * g.N + n) * 2));
        const int cnt = min(32, g.T - t0);
        for (int k = 0; k < cnt; k += 2, ++it) {
          const int k1 = min(k + 1, 31);
          const float cx0 = __shfl_sync(0xffffffffu, c.x, k) * inv, cy0 = __shfl_sync(0xffffffffu, c.y, k) * inv;
          const float cx1 = __shfl_sync(0xffffffffu, c.x, k1) * inv, cy1 = __shfl_sync(0xffffffffu, c.y, k1) * inv;
          if (elect_one()) {
            const int nf = (k + 1 < cnt) ? 2 : 1;
            const int bx0 = box_origin8(cx0, W), by0 = box_origin8(cy0, H);
            const int bx1 = box_origin8(cx1, W), by1 = box_origin8(cy1, H);
#pragma unroll
            for (int kh = 0; kh < 2; ++kh) {
              int sl;
              uint32_t par;
              ring_slot(it, kh, sl, par);
              if (kh == 0) TRACE(it, 0);
              mbar_wait_spin(&a_empty[sl], par ^ 1u);
              if (kh == 0) TRACE(it, 1);
              if (kh == 0) {   // the tile's parameters become visible to the epilogue through a_full
                float4* prm = reinterpret_cast<float4*>(smem + OFF_PARAM + (it % NPARAM) * 32);
                prm[0] = make_float4(cx0, cy0, __int_as_float(bx0), __int_as_float(by0));
                prm[1] = make_float4(cx1, cy1, __int_as_float(bx1), __int_as_float(by1));
              }
              mbar_arrive_expect_tx(&a_full[sl], (uint32_t)(nf * (A_SLOT / 2)));
              uint8_t* dst = smem + OFF_A + sl * A_SLOT;
#pragma unroll
              for (int f = 0; f < 2; ++f) {
                if (f < nf) {
                  const int bx = f ? bx1 : bx0, by = f ? by1 : by0;
#pragma unroll
                  for (int pl = 0; pl < 2; ++pl)
                    tma_load_4d(dst + pl * A_PLANE + f * 8192, &maps.m[l], kh * 64, bx, by,
                                pl * g.T_pyr + map_frame(frow, t0 + k + f), &a_full[sl]);
                }
              }
            }
          }
        }
        __syncwarp();
      }
    }
  } else if (warp >= SB_WARP0 && warp < EPI_WARP0) {
    // ================================================================== support builders (B operand, once per unit)
    const int sb = warp - SB_WARP0;
    const int atom = lane >> 4, chunk = (lane & 15) >> 1, half = lane & 1;  // where this lane's 4 channels live
    uint8_t* s_hi = smem + OFF_S;
    uint32_t ui = 0;
    for (int u = blockIdx.x; u < num_units; u += gridDim.x, ++ui) {
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
          split2(rows[j].x, rows[j].y, h0, l0);
          split2(rows[j].z, rows[j].w, h1, l1);
          const uint32_t off = (uint32_t)(atom * S_HALF) + sw128(p, chunk) + (uint32_t)(half * 8);
          *reinterpret_cast<uint2*>(s_hi + off) = make_uint2(h0, h1);          // rows 0..63 of the K-half: hi plane
          *reinterpret_cast<uint2*>(s_hi + 8192 + off) = make_uint2(l0, l1);   // rows 64..127: lo plane
        }
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(s_full);
    }
  } else if (warp >= EPI_WARP0) {
    // ================================================================== MMA + epilogue groups
    const int grp = (warp - EPI_WARP0) >> 2;   // tiles with (it & 1) == grp
    const int q = warp & 3;                    // row quarter
    const int r = q * 32 + lane;               // D row = f*64 + y*8 + x; also this thread's index in the group
    const int f = r >> 6, py = (r >> 3) & 7, px = r & 7;
    const int a = min(px, 6);                  // x-offset index this lane blends (lane px == 7 only feeds others)
    float* hbuf = reinterpret_cast<float*>(smem + OFF_H + grp * H_GROUP);
    uint8_t* img = smem + OFF_H + grp * H_GROUP;     // output image of the tile, reuses hbuf once it has been read
    float4* tab = reinterpret_cast<float4*>(smem + OFF_TAB + grp * 256);
    float4* xch = reinterpret_cast<float4*>(smem + OFF_XCH + grp * XCH_GROUP);
    float4* hrow = reinterpret_cast<float4*>(hbuf + f * H_FRAME + py * H_ROW + a * H_A);
    float* acc_tile = reinterpret_cast<float*>(smem + OFF_ACC + grp * ACC_BYTES);
    const uint32_t s_base = smem_u32(smem + OFF_S);
    const int bar_id = 1 + grp;
    // volume row owned by this thread when the y-blend runs ...
    //   in registers (interior tiles): lane (texel row b = py < 7, a = px < 7) of frame f -> rho = a*7 + b
    const bool own_fast = px < 7 && py < 7;
    const int rho_fast = px * 7 + py;
    const int idle_fast = f * 15 + (py < 7 ? py : 7 + px);   // 0..29 among the 30 threads without a row
    //   through shared memory (tiles touching a border): thread r < 98 -> frame r / 49, rho = r % 49
    const bool own_gen = r < 2 * kP;
    const int yf = r >= kP ? 1 : 0;
    const int rho_gen = r - yf * kP;
    const int ya = rho_gen / 7, yb = rho_gen - ya * 7;
    uint32_t it = 0, ui = 0;
    for (int u = blockIdx.x; u < num_units; u += gridDim.x, ++ui) {
      const int n = u / kL, l = u % kL;
      const int H = g.lay.h[l], W = g.lay.w[l];
      mbar_wait(s_full, ui & 1u);
      for (int tp = 0; tp < tiles_per_unit; ++tp, ++it) {
        if ((int)(it & 1u) != grp) continue;
        {
          // D[texel row][k] over both K-halves: A x [S_hi ; S_lo] as ONE N=128 MMA (columns 0..63 += A_hi S_hi,
          // 64..127 += A_hi S_lo), then A_lo x S_hi (N=64) on columns 0..63; the halves are added in registers, so
          // the tile handed to the epilogue is [128 rows][64 columns]
          float d0[64], d1[64];
#pragma unroll
          for (int kh = 0; kh < 2; ++kh) {
            int sl;
            uint32_t par;
            ring_slot(it, kh, sl, par);
            mbar_wait(&a_full[sl], par);
            if (kh == 0) TRACE(it, 2);
            wgmma_fence();
            const uint32_t a_base = smem_u32(smem + OFF_A + sl * A_SLOT);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const uint64_t ds = gmma_desc_sw128(s_base + (uint32_t)(kh * S_HALF + j * 32));
              const uint32_t first = (kh | j) != 0 ? 1u : 0u;
              wgmma_tile<128, false>(d0, gmma_desc_sw128(a_base + j * 32), ds, first);
              wgmma_tile<128, false>(d1, gmma_desc_sw128(a_base + 8192 + j * 32), ds, first);
              wgmma_m64n64_bf16_head(d0, gmma_desc_sw128(a_base + A_PLANE + j * 32), ds, 1u);
              wgmma_m64n64_bf16_head(d1, gmma_desc_sw128(a_base + A_PLANE + 8192 + j * 32), ds, 1u);
            }
            wgmma_commit();
            wgmma_wait0(d0);
            wgmma_wait0(d1);
            __syncwarp();
            if (lane == 0) mbar_arrive(&a_empty[sl]);   // this K-half may be refilled
          }
          float o0[32], o1[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            o0[i] = d0[i] + d0[i + 32];
            o1[i] = d1[i] + d1[i + 32];
          }
          asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");   // the previous tile's rows have been read
          acc_store<64>(o0, acc_tile, ACC_LD);
          acc_store<64>(o1, acc_tile + 64 * ACC_LD, ACC_LD);
          asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
        }
        if (r == 0) TRACE(it, 5);
        const float4* prms = reinterpret_cast<const float4*>(smem + OFF_PARAM + (it % NPARAM) * 32);
        const float4 prm = prms[f];
        int sx0, sx1;
        float wx;
        tap_pair(prm.x, a - kR, W, __float_as_int(prm.z), sx0, sx1, wx);
        const float ux = 1.f - wx;
        const int src0 = (lane & 24) | sx0, src1 = (lane & 24) | sx1;
        // y taps of sample row b = lane & 7 of frame (lane >> 3) & 1, evaluated by lanes 0..6 / 8..14 of every warp.
        // Interior tile (both frames): sample row b blends texel rows b and b+1 of the box -> y-blend in registers.
        float wy_l;
        int r0_l, r1_l;
        {
          const float4 pq = prms[(lane >> 3) & 1];
          const int b = lane & 7;
          tap_pair(pq.y, min(b, 6) - kR, H, __float_as_int(pq.w), r0_l, r1_l, wy_l);
        }
        const bool ok_l = (lane & 7) == 7 || (r0_l == (lane & 7) && r1_l == (lane & 7) + (wy_l > 0.f ? 1 : 0));
        const bool fast = (__ballot_sync(0xffffffffu, ok_l) & 0xffffu) == 0xffffu;
        const float wy = __shfl_sync(0xffffffffu, wy_l, f * 8 + min(py, 6));   // this lane's row weight (fast path)
        // ---- x-blend: h[k] = (1-wx) D[(row, x0), k] + wx D[(row, x1), k]  for (texel row py, sample column a)
        float h[H_A];
        // h[k] = (A_hi + A_lo) S_hi + A_hi S_lo, 16 columns at a time
#pragma unroll
        for (int c4 = 0; c4 < 4; ++c4) {
          float v[16];
          acc_row_ld<16>(acc_tile + r * ACC_LD + 16 * c4, v);
#pragma unroll
          for (int j = 0; j < 16; ++j)
            if (16 * c4 + j < H_A) h[16 * c4 + j] = (16 * c4 + j < kP) ? v[j] : 0.f;
        }
        if (r == 0) TRACE(it, 6);
#pragma unroll
        for (int k = 0; k < kP; ++k) {
          const float v0 = __shfl_sync(0xffffffffu, h[k], src0), v1 = __shfl_sync(0xffffffffu, h[k], src1);
          h[k] = ux * v0 + wx * v1;
        }
        bool own;
        int ff, rho;
        if (fast) {
          // ---- y-blend in registers: the next texel row is 8 lanes up; texel row 4 (first row of the odd warp)
          // reaches the even warp's last row through a small exchange buffer
          if ((q & 1) && lane < 7) {
#pragma unroll
            for (int k4 = 0; k4 < H_A / 4; ++k4)
              xch[(f * 7 + lane) * (H_A / 4) + k4] = make_float4(h[4 * k4], h[4 * k4 + 1], h[4 * k4 + 2], h[4 * k4 + 3]);
          }
          if (r == 0) bulk_wait_read0();           // previous tile's image has left shared memory
          asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
          const bool edge = !(q & 1) && (lane >> 3) == 3 && px < 7;   // texel row 3: its lower neighbour is row 4
          const float uy = 1.f - wy;
#pragma unroll
          for (int k4 = 0; k4 < H_A / 4; ++k4) {
            float4 dn;
            dn.x = __shfl_down_sync(0xffffffffu, h[4 * k4 + 0], 8);
            dn.y = __shfl_down_sync(0xffffffffu, h[4 * k4 + 1], 8);
            dn.z = __shfl_down_sync(0xffffffffu, h[4 * k4 + 2], 8);
            dn.w = __shfl_down_sync(0xffffffffu, h[4 * k4 + 3], 8);
            if (edge) dn = xch[(f * 7 + px) * (H_A / 4) + k4];
            h[4 * k4 + 0] = uy * h[4 * k4 + 0] + wy * dn.x;
            h[4 * k4 + 1] = uy * h[4 * k4 + 1] + wy * dn.y;
            h[4 * k4 + 2] = uy * h[4 * k4 + 2] + wy * dn.z;
            h[4 * k4 + 3] = uy * h[4 * k4 + 3] + wy * dn.w;
          }
          own = own_fast;
          ff = f;
          rho = rho_fast;
        } else {
          // ---- y-blend through shared memory (any border clamp): [texel row][a][k] buffer + per-row tap table
          if (r == 0) bulk_wait_read0();
          asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");   // image of the previous tile is gone
          if (px < 7) {
#pragma unroll
            for (int k4 = 0; k4 < H_A / 4; ++k4) hrow[k4] = make_float4(h[4 * k4], h[4 * k4 + 1], h[4 * k4 + 2], h[4 * k4 + 3]);
          }
          if (q == 0 && lane < 16 && (lane & 7) < 7)   // one writer per (frame lane >> 3, sample row b = lane & 7)
            tab[(lane >> 3) * 8 + (lane & 7)] = make_float4(wy_l, __int_as_float(r0_l * H_ROW), __int_as_float(r1_l * H_ROW), 0.f);
          asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
          if (own_gen) {
            const float4 tb = tab[yf * 8 + yb];
            const float4* h0 = reinterpret_cast<const float4*>(hbuf + yf * H_FRAME + ya * H_A + __float_as_int(tb.y));
            const float4* h1 = reinterpret_cast<const float4*>(hbuf + yf * H_FRAME + ya * H_A + __float_as_int(tb.z));
            const float wyg = tb.x, uyg = 1.f - tb.x;
#pragma unroll
            for (int k4 = 0; k4 < H_A / 4; ++k4) {
              const float4 p0 = h0[k4], p1 = h1[k4];
              h[4 * k4 + 0] = uyg * p0.x + wyg * p1.x;
              h[4 * k4 + 1] = uyg * p0.y + wyg * p1.y;
              h[4 * k4 + 2] = uyg * p0.z + wyg * p1.z;
              h[4 * k4 + 3] = uyg * p0.w + wyg * p1.w;
            }
          }
          asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");   // h fully read: the image may overwrite it
          own = own_gen;
          ff = yf;
          rho = rho_gen;
        }
        // ---- byte image of the tile's two volume rows: [hi(2432) | lo(2432)] split bf16 each, or one fp16 plane (V16)
        if (own) {
          // 49 elements per plane at element offset rho*49: one 2-byte edge element (the first if that offset is odd,
          // else the last) + 24 aligned 4-byte pairs
          const bool odd = (rho & 1) != 0;
          uint16_t* dst_hi = reinterpret_cast<uint16_t*>(img + ff * ROW_BYTES) + rho * kP;
          uint32_t* ph = reinterpret_cast<uint32_t*>(dst_hi + (odd ? 1 : 0));
          if (V16) {
#pragma unroll
            for (int j = 0; j < 24; ++j) ph[j] = pack_h2(odd ? h[2 * j + 1] : h[2 * j], odd ? h[2 * j + 2] : h[2 * j + 1]);
            dst_hi[odd ? 0 : 48] = __half_as_ushort(__float2half_rn(odd ? h[0] : h[48]));
          } else {
            uint16_t* dst_lo = dst_hi + kVolPad;
            uint32_t* pl = reinterpret_cast<uint32_t*>(dst_lo + (odd ? 1 : 0));
#pragma unroll
            for (int j = 0; j < 24; ++j) {
              uint32_t hi, lo;
              split2(odd ? h[2 * j + 1] : h[2 * j], odd ? h[2 * j + 2] : h[2 * j + 1], hi, lo);
              ph[j] = hi;
              pl[j] = lo;
            }
            const bf16pair ed = split_bf16(odd ? h[0] : h[48]);
            dst_hi[odd ? 0 : 48] = __bfloat16_as_ushort(ed.hi);
            dst_lo[odd ? 0 : 48] = __bfloat16_as_ushort(ed.lo);
          }
        } else {
          // K padding (elements 2401..2431 of every plane of the image) = zero: one 2-byte element + 15 aligned pairs each
          for (int j = fast ? idle_fast : r - 2 * kP; j < (V16 ? 2 : 4) * 16; j += 128 - 2 * kP) {
            uint16_t* plane = reinterpret_cast<uint16_t*>(img) + (j >> 4) * kVolPad;
            const int w = j & 15;
            if (w == 0) plane[kVol] = 0;
            else *reinterpret_cast<uint32_t*>(plane + kVol - 1 + 2 * w) = 0u;
          }
        }
        fence_proxy_async_smem();                   // image writes -> visible to the bulk-copy (async proxy) reads
        asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
        // ---- copy-out: one bulk shared->global copy per volume row (9728 contiguous bytes), issued by one thread;
        // its shared-memory reads are awaited before the next tile of this group touches the buffer
        if (r == 0) {
#pragma unroll
          for (int t2 = 0; t2 < 2; ++t2) {
            const int t = 2 * tp + t2;
            if (t < g.T)
              bulk_store_s2g(g.vol + (((int64_t)n * g.T + t) * kL + l) * (ROW_BYTES / 2), img + t2 * ROW_BYTES, ROW_BYTES);
          }
          bulk_commit();
          TRACE(it, 7);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(s_empty);         // this warp's MMAs of the unit have all completed
    }
  }

  if (warp >= EPI_WARP0 && (threadIdx.x & 127) == 0) bulk_wait0();   // outstanding volume-row copies
}

// fp32 channels-last level -> [hi plane | lo plane] bf16, 4 channels per thread
__global__ void __launch_bounds__(256)
split_level_kernel(const float4* __restrict__ in, uint2* __restrict__ hi, uint2* __restrict__ lo, int64_t n4) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(in + i);
    uint32_t h0, l0, h1, l1;
    split2(v.x, v.y, h0, l0);
    split2(v.z, v.w, h1, l1);
    hi[i] = make_uint2(h0, h1);
    lo[i] = make_uint2(l0, l1);
  }
}

// fp32 channels-last level -> one fp16 plane (mode 1 / 2, read by corr_tc3.cu), 4 channels per thread
__global__ void __launch_bounds__(256)
half_level_kernel(const float4* __restrict__ in, uint2* __restrict__ out, int64_t n4) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(in + i);
    out[i] = make_uint2(pack_h2(v.x, v.y), pack_h2(v.z, v.w));
  }
}

template <bool V16>
cudaError_t launch_variant(const Corr2Args& g, const Corr2Maps& maps, int num_units, int num_sms, cudaStream_t s) {
  static DeviceOnce attr;
  cudaError_t e = once_per_device(attr, [&] {
    return cudaFuncSetAttribute(corr_patch_tc_kernel<V16>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  });
  if (e != cudaSuccess) return e;
  const int grid = num_units < num_sms ? num_units : num_sms;
  corr_patch_tc_kernel<V16><<<grid, THREADS, SMEM_BYTES, s>>>(g, maps, num_units);
  return cudaGetLastError();
}

}  // namespace

bool corr_patch_supported(int T, int H4, int W4) {
  const PyramidLayout lay = pyramid_layout(T, H4, W4);
  return lay.h[kL - 1] >= 8 && lay.w[kL - 1] >= 8;
}

cudaError_t launch_split_pyramid(const float* pyr, int T, int H4, int W4, __nv_bfloat16* pyr_split, int mode,
                                 cudaStream_t s) {
  const PyramidLayout lay = pyramid_layout(T, H4, W4);
  for (int l = 0; l < kL; ++l) {
    const int64_t n = (int64_t)T * lay.h[l] * lay.w[l] * kD;
    __nv_bfloat16* dst = pyr_split + 2 * lay.off[l];   // level l always starts at the same offset, whatever the mode
    const int64_t n4 = n / 4;
    const int grid = (int)((n4 + 255) / 256 < 132 * 16 ? (n4 + 255) / 256 : 132 * 16);
    if (mode == 3)
      split_level_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const float4*>(pyr + lay.off[l]),
                                              reinterpret_cast<uint2*>(dst), reinterpret_cast<uint2*>(dst + n), n4);
    else
      half_level_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const float4*>(pyr + lay.off[l]),
                                             reinterpret_cast<uint2*>(dst), n4);
  }
  return cudaGetLastError();
}

cudaError_t launch_corr_patch_tc(const __nv_bfloat16* pyr_split, int H4, int W4, const float* support,
                                 const uint8_t* track_valid, const float* coords, int T, int N, int count,
                                 __nv_bfloat16* vol_split, int vol16, int num_sms, cudaStream_t s, int T_pyr,
                                 const FrameMap& fm) {
  Corr2Args g;
  g.lay = pyramid_layout(T_pyr, H4, W4);
  g.support = support;
  g.track_valid = track_valid;
  g.coords = coords;
  g.T = T;
  g.N = N;
  g.T_pyr = T_pyr;
  g.vol = reinterpret_cast<uint16_t*>(vol_split);
  g.trace = nullptr;
  g.fm = fm;
#ifdef CT3_TRACE
  static long long* trace_buf = nullptr;
  if (!trace_buf) cudaMalloc(&trace_buf, 256 * 8 * sizeof(long long));
  g.trace = trace_buf;
#endif
  Corr2Maps maps;
  for (int l = 0; l < kL; ++l) {
    const uint64_t W = (uint64_t)g.lay.w[l], H = (uint64_t)g.lay.h[l];
    if (W < 8 || H < 8) return cudaErrorInvalidValue;
    const uint64_t dims[4] = {(uint64_t)kD, W, H, (uint64_t)(2 * T_pyr)};   // dim 3 = plane*T_pyr + frame
    const uint64_t strides[3] = {(uint64_t)kD * 2, W * kD * 2, H * W * kD * 2};
    const uint32_t box[4] = {64, 8, 8, 1};
    if (!encode_tensor_map(&maps.m[l], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, pyr_split + 2 * g.lay.off[l], dims, strides,
                           box, CU_TENSOR_MAP_SWIZZLE_128B))
      return cudaErrorInvalidValue;
  }
  const int num_units = count * kL;
  const cudaError_t le = vol16 ? launch_variant<true>(g, maps, num_units, num_sms, s)
                               : launch_variant<false>(g, maps, num_units, num_sms, s);
  if (le != cudaSuccess) return le;
#ifdef CT3_TRACE
  {
    static int calls = 0;
    if (++calls == 3) {
      cudaStreamSynchronize(s);
      static long long h[256 * 8];
      cudaMemcpy(h, trace_buf, sizeof(h), cudaMemcpyDeviceToHost);
      const char* nm[8] = {"tma_wait", "tma_go", "mma_afull", "mma_dempty", "mma_issued", "epi_dfull", "epi_dempty", "epi_end"};
      printf("tile");
      for (int e = 0; e < 8; ++e) printf(" %10s", nm[e]);
      printf("\n");
      for (int t = 32; t < 96; ++t) {
        printf("%4d", t);
        for (int e = 0; e < 8; ++e) printf(" %10lld", h[t * 8 + e] - h[32 * 8]);
        printf("\n");
      }
    }
  }
#endif
  return cudaGetLastError();
}

}  // namespace ct3
