// corr_tc.cu -- fused bilinear sampling + 4-D correlation on the Hopper tensor cores (the production path of
// launch_corr_sample; corr.cu keeps the exact-fp32 SIMT version the tests cross-check against).
//
//   vol[(n,t,l)][(a*7+b)*49 + (i*7+j)] = < bilinear(F_l[t], cx/2^l + a-3, cy/2^l + b-3) , S_l[n, i*7+j, :] >
//   (get_correlation_feat + einsum, cotracker3_online.py:130-143, cotracker3_offline.py:144-156)
//
// Persistent, warp-specialised; work unit = (track n, level l), tile = two frames of that unit:
//   patches : the 8x8-texel neighbourhood of a (t,n,l) is ONE 4-D TMA box load (128 ch x 8 x 8 x 1 frame = 32 KiB,
//             origin clamped into the map) from the channels-last pyramid into a 2-slot shared-memory ring; every
//             texel crosses L2->SM once (64 instead of 112 line reads per frame) and no warp waits on a gather
//   A tile  [128 x 128] : rows f*49 + a*7 + b (98 used) = the 49 sampled feature vectors of 2 frames, blended from
//             the staged patch (separable 4-tap, border clamp per sample) and stored split-bf16 in the
//             128B-swizzled K-major layout
//   B tile  [ 64 x 128] : the 49 support vectors of (n,l) (rows 49..63 zero), split-bf16, built once per unit
//   D       [128 x  64] : fp32, 3 wgmma per k16 step (lo*hi + hi*lo + hi*hi) by the epilogue warpgroup, handed to
//                         its row-per-thread epilogue through shared memory
//   epilogue            : accumulator row -> split-bf16 -> byte image of the complete 9728-byte volume rows
//                         ([hi(2432) | lo(2432)], K padding zero) -> fully coalesced 16-byte stores
// Warps: 0..13 samplers (warp w: frame w/7 of the tile, x-offset a = w%7), 14 idle, 15 TMA issuer, 16..19 MMA +
// epilogue warpgroup.  Neither the sampled features (10 GB/iteration in the reference) nor an fp32 volume
// ever touch HBM.
#include "gemm.cuh"
#include "kernels.cuh"

namespace ct3 {
namespace {

constexpr int PW = 14;                    // sampler warps
constexpr int TMA_WARP = 15;              // warp 14 idle
constexpr int EPI_WARP0 = 16;             // warps 16..19: one warpgroup, MMA (wgmma) + epilogue
constexpr int THREADS = 20 * 32;
constexpr int A_PART = 2 * 16384;         // one bf16 plane of A: 2 K-atoms x [128 rows x 128 B]
constexpr int A_BYTES = 2 * A_PART;       // hi + lo = 64 KiB
constexpr int S_PART = 2 * 8192;          // one plane of S: 2 K-atoms x [64 rows x 128 B]
constexpr int S_BYTES = 2 * S_PART;       // 32 KiB
constexpr int PATCH_BYTES = 8 * 8 * kD * 4;  // 32 KiB
constexpr int NPATCH = 2;
constexpr int ROW_BYTES = 2 * kVolPad * 2;   // 9728: one volume row image [hi | lo]
constexpr int STG_BYTES = 2 * ROW_BYTES;     // two frames per tile
constexpr int OFF_S = 0;
constexpr int OFF_A = OFF_S + S_BYTES;
constexpr int OFF_PATCH = OFF_A + A_BYTES;
constexpr int OFF_STG = OFF_PATCH + NPATCH * PATCH_BYTES;
constexpr int OFF_PARAM = OFF_STG + STG_BYTES;      // NPATCH x {cx, cy, box_x, box_y}
constexpr int ACC_LD = 64 + 4;            // accumulator tile [128 rows][ACC_LD] fp32 (MMA registers -> row per thread)
constexpr int OFF_ACC = OFF_PARAM + NPATCH * 16;
constexpr int OFF_BAR = OFF_ACC + 128 * ACC_LD * 4;
constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
static_assert(SMEM_BYTES <= 232448, "shared memory budget");

struct CorrTcArgs {
  const float* pyr;
  PyramidLayout lay;
  const float* support;        // [4][49, N, 128]
  const uint8_t* track_valid;  // [N] or null
  const float* coords;         // [T, N, 2]
  int T, N;
  __nv_bfloat16* vol;          // [N*T*4, 2*kVolPad]
  FrameMap fm;                 // pyramid frame of (track, t): the unit's patches all come from its own frame row
};
struct CorrMaps {
  CUtensorMap m[kL];           // per level: dims (128, W, H, T_pyr), box (128, min(W,8), min(H,8), 1), fp32, no swizzle
};

// byte offset of (row r, 16-byte chunk c) inside one [rows x 128 B] swizzle-128B K-atom
__device__ __forceinline__ uint32_t sw128(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }

// lane -> where its 4 channels [4*lane, 4*lane+4) live: K-atom, 16B chunk, 8-byte half
struct LanePos { int atom, chunk, half; };
__device__ __forceinline__ LanePos lane_pos(int lane) { return {lane >> 4, (lane & 15) >> 1, lane & 1}; }

__device__ __forceinline__ void store_split4(uint8_t* plane_hi, uint8_t* plane_lo, int atom_bytes, int row,
                                             LanePos lp, float4 v) {
  uint32_t h0, l0, h1, l1;
  split2(v.x, v.y, h0, l0);
  split2(v.z, v.w, h1, l1);
  const uint32_t off = (uint32_t)(lp.atom * atom_bytes) + sw128(row, lp.chunk) + (uint32_t)(lp.half * 8);
  *reinterpret_cast<uint2*>(plane_hi + off) = make_uint2(h0, h1);
  *reinterpret_cast<uint2*>(plane_lo + off) = make_uint2(l0, l1);
}

__device__ __forceinline__ float4 lerp4(float4 a, float4 b, float w) {
  const float u = 1.f - w;
  return make_float4(u * a.x + w * b.x, u * a.y + w * b.y, u * a.z + w * b.z, u * a.w + w * b.w);
}

// origin of the 8-wide box that contains every (clamped) tap of the 7 samples around c
__device__ __forceinline__ int box_origin(float c, int size) {
  const float cc = fminf(fmaxf(c, -16.f), (float)size + 16.f);
  const int o = (int)floorf(cc) - kR;
  return max(0, min(o, size - min(size, 8)));   // maps narrower than 8 texels: the box is the whole map
}

__global__ void __launch_bounds__(THREADS, 1)
corr_sample_tc_kernel(const __grid_constant__ CorrTcArgs g, const __grid_constant__ CorrMaps maps, int num_units) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* a_full = bars;          // samplers -> MMA            (count 14)
  uint64_t* a_empty = bars + 1;     // MMA -> samplers            (one arrive per MMA warp)
  uint64_t* s_full = bars + 2;      // samplers -> MMA, per unit  (count 14)
  uint64_t* s_empty = bars + 3;     // MMA -> samplers, per unit  (one arrive per MMA warp)
  uint64_t* p_full = bars + 4;      // [NPATCH] TMA -> samplers   (count 1 + tx bytes)
  uint64_t* p_empty = bars + 4 + NPATCH;   // [NPATCH] samplers -> TMA  (count 7)
  float* acc_tile = reinterpret_cast<float*>(smem + OFF_ACC);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_unit = (g.T + 1) / 2;

  // one-time: zero S (rows 49..63 stay zero forever) and the staging image (K padding stays zero)
  for (int i = threadIdx.x; i < S_BYTES / 16; i += THREADS) reinterpret_cast<uint4*>(smem + OFF_S)[i] = make_uint4(0, 0, 0, 0);
  for (int i = threadIdx.x; i < STG_BYTES / 16; i += THREADS) reinterpret_cast<uint4*>(smem + OFF_STG)[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async_smem();
  if (threadIdx.x == 0) {
    mbar_init(a_full, PW);
    mbar_init(a_empty, 4);
    mbar_init(s_full, PW);
    mbar_init(s_empty, 4);
    for (int i = 0; i < NPATCH; ++i) { mbar_init(&p_full[i], 1); mbar_init(&p_empty[i], 7); }
    fence_barrier_init();
    for (int l = 0; l < kL; ++l) tma_prefetch_desc(&maps.m[l]);
  }
  __syncthreads();

  if (warp < PW) {
    // ================================================================== samplers
    const LanePos lp = lane_pos(lane);
    const int f = warp / 7, a = warp % 7;  // frame of the tile / x-offset index owned by this warp
    uint32_t it = 0, ui = 0, fc = 0;       // tile / unit / frame counters of this CTA
    uint32_t aoff[7];                      // byte offsets of this lane's 8-byte slot in the 7 A rows it writes
#pragma unroll
    for (int b = 0; b < 7; ++b) aoff[b] = (uint32_t)(lp.atom * 16384) + sw128(f * kP + a * 7 + b, lp.chunk) + (uint32_t)(lp.half * 8);
    for (int u = blockIdx.x; u < num_units; u += gridDim.x, ++ui) {
      const int n = u / kL, l = u % kL;
      const int H = g.lay.h[l], W = g.lay.w[l];
      const int bw = min(W, 8), bh = min(H, 8);        // box extent (maps narrower than 8 texels: whole map)
      const int32_t* frow = frame_row(g.fm, n, g.T);
      // ---- support tile (B operand), once per unit
      if (ui > 0) mbar_wait(s_empty, (ui - 1) & 1u);   // MMAs of the previous unit have retired
      {
        const bool valid = g.track_valid == nullptr || g.track_valid[n] != 0;
        uint8_t* s_hi = smem + OFF_S;
        uint8_t* s_lo = smem + OFF_S + S_PART;
        for (int p = warp; p < kP; p += PW) {
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (valid) v = __ldg(reinterpret_cast<const float4*>(g.support + ((int64_t)l * kP * g.N + (int64_t)p * g.N + n) * kD) + lane);
          store_split4(s_hi, s_lo, 8192, p, lp, v);
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(s_full);
      }
      // ---- A tiles: two frames each, one (frame, x-offset) column of 7 samples per warp
      for (int tp = 0; tp < tiles_per_unit; ++tp, ++it) {
        const int t = 2 * tp + f;
        const int nf = (2 * tp + 1 < g.T) ? 2 : 1;     // frames in this tile
        float4 outv[7];
        if (t < g.T) {
          const uint32_t fr = fc + f;                  // frame sequence number -> ring slot
          const int slot = fr % NPATCH;
          mbar_wait(&p_full[slot], (fr / NPATCH) & 1u);
          const float4 prm = *reinterpret_cast<const float4*>(smem + OFF_PARAM + slot * 16);
          const float cx = prm.x, cy = prm.y;
          const int bx = __float_as_int(prm.z), by = __float_as_int(prm.w);
          const float* patch = reinterpret_cast<const float*>(smem + OFF_PATCH + slot * PATCH_BYTES) + lane * 4;
          const float x = fminf(fmaxf(cx + (float)(a - kR), 0.f), (float)(W - 1));
          const float xf = floorf(x);
          const int x0 = (int)xf, x1 = min(x0 + 1, W - 1);
          const float wx = x - xf;
          float wy[7];
          int y0[7], yl[8];   // yl[0] = y0 of sample 0, yl[k+1] = y1 of sample k: the (<= 8) distinct rows of the column
#pragma unroll
          for (int b = 0; b < 7; ++b) {
            const float y = fminf(fmaxf(cy + (float)(b - kR), 0.f), (float)(H - 1));
            const float yf = floorf(y);
            y0[b] = (int)yf;
            wy[b] = y - yf;
            if (b == 0) yl[0] = y0[0];
            yl[b + 1] = min(y0[b] + 1, H - 1);
          }
          // fast path (always, bar fp32 corner cases of floor(c + offset)): every tap of the column is in the box
          // and each sample's upper row is either the previous sample's lower row or (low-border clamp) row yl[0]
          bool fast = (x0 >= bx) && (x1 < bx + bw) && (yl[0] >= by) && (yl[7] < by + bh);
#pragma unroll
          for (int b = 1; b < 7; ++b) fast = fast && ((y0[b] == yl[b]) || (y0[b] == yl[0]));
          if (fast) {
            const float* pa = patch + (x0 - bx) * kD;
            const float* pb = patch + (x1 - bx) * kD;
            float4 hrow[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              const int ro = (yl[k] - by) * bw * kD;
              hrow[k] = lerp4(*reinterpret_cast<const float4*>(pa + ro), *reinterpret_cast<const float4*>(pb + ro), wx);
            }
#pragma unroll
            for (int b = 0; b < 7; ++b) {
              const bool same = (y0[b] == yl[b]);
              float4 h0;
              h0.x = same ? hrow[b].x : hrow[0].x; h0.y = same ? hrow[b].y : hrow[0].y;
              h0.z = same ? hrow[b].z : hrow[0].z; h0.w = same ? hrow[b].w : hrow[0].w;
              outv[b] = lerp4(h0, hrow[b + 1], wy[b]);
            }
          } else {
            const float* fm = g.pyr + g.lay.off[l] + (int64_t)map_frame(frow, t) * H * W * kD + lane * 4;
#pragma unroll
            for (int b = 0; b < 7; ++b) {
              const int y1 = yl[b + 1];
              const float4 h0 = lerp4(__ldg(reinterpret_cast<const float4*>(fm + ((int64_t)y0[b] * W + x0) * kD)),
                                      __ldg(reinterpret_cast<const float4*>(fm + ((int64_t)y0[b] * W + x1) * kD)), wx);
              const float4 h1 = lerp4(__ldg(reinterpret_cast<const float4*>(fm + ((int64_t)y1 * W + x0) * kD)),
                                      __ldg(reinterpret_cast<const float4*>(fm + ((int64_t)y1 * W + x1) * kD)), wx);
              outv[b] = lerp4(h0, h1, wy[b]);
            }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&p_empty[slot]);  // this warp is done reading the patch
        }
        fc += nf;
        mbar_wait(a_empty, (it & 1u) ^ 1u);            // MMAs of the previous tile have consumed A
        if (t < g.T) {
          uint8_t* a_hi = smem + OFF_A;
#pragma unroll
          for (int b = 0; b < 7; ++b) {
            uint32_t h0, l0, h1, l1;
            split2(outv[b].x, outv[b].y, h0, l0);
            split2(outv[b].z, outv[b].w, h1, l1);
            *reinterpret_cast<uint2*>(a_hi + aoff[b]) = make_uint2(h0, h1);
            *reinterpret_cast<uint2*>(a_hi + A_PART + aoff[b]) = make_uint2(l0, l1);
          }
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(a_full);
      }
    }
  } else if (warp == TMA_WARP) {
    // ================================================================== TMA issuer (whole warp walks, lane 0 issues)
    uint32_t fc = 0;
    for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
      const int n = u / kL, l = u % kL;
      const int H = g.lay.h[l], W = g.lay.w[l];
      const float inv = 1.0f / (float)(1 << l);
      const int32_t* frow = frame_row(g.fm, n, g.T);
      for (int t0 = 0; t0 < g.T; t0 += 32) {
        // coordinates of up to 32 frames in one round trip (lane = frame), then broadcast per frame
        const int tl = min(t0 + lane, g.T - 1);
        const float2 c = __ldg(reinterpret_cast<const float2*>(g.coords + ((int64_t)tl * g.N + n) * 2));
        const int cnt = min(32, g.T - t0);
        for (int k = 0; k < cnt; ++k, ++fc) {
          const float cx = __shfl_sync(0xffffffffu, c.x, k) * inv;
          const float cy = __shfl_sync(0xffffffffu, c.y, k) * inv;
          if (lane == 0) {
            const int slot = fc % NPATCH;
            mbar_wait(&p_empty[slot], ((fc / NPATCH) & 1u) ^ 1u);
            const int bx = box_origin(cx, W), by = box_origin(cy, H);
            *reinterpret_cast<float4*>(smem + OFF_PARAM + slot * 16) =
                make_float4(cx, cy, __int_as_float(bx), __int_as_float(by));
            mbar_arrive_expect_tx(&p_full[slot], (uint32_t)(min(W, 8) * min(H, 8) * kD * 4));
            tma_load_4d(smem + OFF_PATCH + slot * PATCH_BYTES, &maps.m[l], 0, bx, by, map_frame(frow, t0 + k),
                        &p_full[slot]);
          }
        }
        __syncwarp();
      }
    }
  } else if (warp >= EPI_WARP0) {
    // ================================================================== MMA (wgmma) + epilogue warpgroup
    const int q = warp & 3;              // row quarter
    const int r = q * 32 + lane;         // D row
    const int f = r >= kP ? 1 : 0;
    const int rho = r - f * kP;          // a*7+b
    const int et = threadIdx.x - EPI_WARP0 * 32;  // 0..127
    uint8_t* stg = smem + OFF_STG;
    const uint32_t s_base = smem_u32(smem + OFF_S);
    const uint32_t a_base = smem_u32(smem + OFF_A);
    uint32_t it = 0, ui = 0;
    for (int u = blockIdx.x; u < num_units; u += gridDim.x, ++ui) {
      const int n = u / kL, l = u % kL;
      mbar_wait(s_full, ui & 1u);
      for (int tp = 0; tp < tiles_per_unit; ++tp, ++it) {
        mbar_wait(a_full, it & 1u);
        float d0[32], d1[32];   // D rows 0..63 / 64..127 (samples) x 64 columns (support rows)
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
          const uint32_t ao = (uint32_t)((ks >> 2) * 16384 + (ks & 3) * 32);
          const uint32_t so = (uint32_t)((ks >> 2) * 8192 + (ks & 3) * 32);
          const uint64_t dsh = gmma_desc_sw128(s_base + so), dsl = gmma_desc_sw128(s_base + S_PART + so);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint32_t ah = (uint32_t)(h * 8192);   // rows 64..127 of the A atom
            const uint64_t dah = gmma_desc_sw128(a_base + ao + ah), dal = gmma_desc_sw128(a_base + A_PART + ao + ah);
            if (h == 0) {
              wgmma_tile<64, false>(d0, dal, dsh, ks != 0 ? 1u : 0u);
              wgmma_tile<64, false>(d0, dah, dsl, 1u);
              wgmma_tile<64, false>(d0, dah, dsh, 1u);
            } else {
              wgmma_tile<64, false>(d1, dal, dsh, ks != 0 ? 1u : 0u);
              wgmma_tile<64, false>(d1, dah, dsl, 1u);
              wgmma_tile<64, false>(d1, dah, dsh, 1u);
            }
          }
        }
        wgmma_commit();
        wgmma_wait0(d0);
        wgmma_wait0(d1);
        __syncwarp();
        if (lane == 0) mbar_arrive(a_empty);     // A may be rewritten by the samplers
        acc_store<64>(d0, acc_tile, ACC_LD);
        acc_store<64>(d1, acc_tile + 64 * ACC_LD, ACC_LD);
        asm volatile("bar.sync 1, 128;" ::: "memory");   // the whole tile is in shared memory
        const bool row_ok = r < 2 * kP && (2 * tp + f) < g.T;
        __nv_bfloat16* dst_hi = reinterpret_cast<__nv_bfloat16*>(stg + f * ROW_BYTES) + rho * kP;
        __nv_bfloat16* dst_lo = dst_hi + kVolPad;
        const float* arow = acc_tile + r * ACC_LD;
        // 49 bf16 per plane at element offset rho*49 of the row image: one 2-byte edge element (first column
        // if that offset is odd, else the last) + 24 aligned 4-byte pairs, in two loads of 32 columns
        const bool odd = (rho & 1) != 0;
        uint32_t* ph = reinterpret_cast<uint32_t*>(dst_hi + (odd ? 1 : 0));
        uint32_t* pl = reinterpret_cast<uint32_t*>(dst_lo + (odd ? 1 : 0));
        float v[32];
        acc_row_ld<32>(arow, v);                   // columns 0..31
        const float carry = v[31];
        if (row_ok) {
          if (odd) {
            const bf16pair e = split_bf16(v[0]);
            dst_hi[0] = e.hi;
            dst_lo[0] = e.lo;
          }
#pragma unroll
          for (int j = 0; j < 15; ++j) {
            uint32_t hi, lo;
            split2(odd ? v[2 * j + 1] : v[2 * j], odd ? v[2 * j + 2] : v[2 * j + 1], hi, lo);
            ph[j] = hi;
            pl[j] = lo;
          }
          if (!odd) {
            uint32_t hi, lo;
            split2(v[30], v[31], hi, lo);
            ph[15] = hi;
            pl[15] = lo;
          }
        }
        acc_row_ld<32>(arow + 32, v);              // columns 32..63 (32..48 used)
        if (row_ok) {
          if (odd) {
            uint32_t hi, lo;
            split2(carry, v[0], hi, lo);
            ph[15] = hi;
            pl[15] = lo;
          }
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            uint32_t hi, lo;
            split2(odd ? v[2 * k + 1] : v[2 * k], odd ? v[2 * k + 2] : v[2 * k + 1], hi, lo);
            ph[16 + k] = hi;
            pl[16 + k] = lo;
          }
          if (!odd) {
            const bf16pair e = split_bf16(v[16]);
            dst_hi[48] = e.hi;
            dst_lo[48] = e.lo;
          }
        }
        // all 128 epilogue threads: image complete -> coalesced copy-out of whole volume rows
        asm volatile("bar.sync 1, 128;" ::: "memory");
        for (int idx = et; idx < 2 * (ROW_BYTES / 16); idx += 128) {
          const int ff = idx / (ROW_BYTES / 16), w16 = idx % (ROW_BYTES / 16);
          const int t = 2 * tp + ff;
          if (t < g.T) {
            uint4* grow = reinterpret_cast<uint4*>(g.vol + (((int64_t)n * g.T + t) * kL + l) * (2 * kVolPad));
            grow[w16] = reinterpret_cast<const uint4*>(stg + ff * ROW_BYTES)[w16];
          }
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");   // image and accumulator tile may be overwritten by the next tile
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(s_empty);       // this warp's MMAs of the unit have all completed
    }
  }
}

}  // namespace

cudaError_t launch_corr_sample_tc(const float* pyr, int H4, int W4, const float* support,
                                  const uint8_t* track_valid, const float* coords, int T, int N, int count,
                                  __nv_bfloat16* vol_split, int num_sms, cudaStream_t s, int T_pyr,
                                  const FrameMap& fm) {
  CorrTcArgs g;
  g.pyr = pyr;
  g.lay = pyramid_layout(T_pyr, H4, W4);
  g.support = support;
  g.track_valid = track_valid;
  g.coords = coords;
  g.T = T;
  g.N = N;
  g.vol = vol_split;
  g.fm = fm;
  CorrMaps maps;
  for (int l = 0; l < kL; ++l) {
    const uint64_t W = (uint64_t)g.lay.w[l], H = (uint64_t)g.lay.h[l];
    const uint64_t dims[4] = {(uint64_t)kD, W, H, (uint64_t)T_pyr};
    const uint64_t strides[3] = {(uint64_t)kD * 4, W * kD * 4, H * W * kD * 4};
    const uint32_t box[4] = {(uint32_t)kD, (uint32_t)(W < 8 ? W : 8), (uint32_t)(H < 8 ? H : 8), 1};
    if (!encode_tensor_map(&maps.m[l], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, pyr + g.lay.off[l], dims, strides, box,
                           CU_TENSOR_MAP_SWIZZLE_NONE))
      return cudaErrorInvalidValue;
  }
  static DeviceOnce attr;
  {
    cudaError_t e = once_per_device(attr, [&] {
      return cudaFuncSetAttribute(corr_sample_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    });
    if (e != cudaSuccess) return e;
  }
  const int num_units = count * kL;
  const int grid = num_units < num_sms ? num_units : num_sms;
  corr_sample_tc_kernel<<<grid, THREADS, SMEM_BYTES, s>>>(g, maps, num_units);
  return cudaGetLastError();
}

}  // namespace ct3
