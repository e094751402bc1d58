// gemm.cu -- split-bf16x3 linear layers on the Hopper tensor cores (wgmma).
//
// Persistent warp-specialised kernel, one CTA per SM, four warpgroups:
//   warps 0..3  : MMA warpgroup   (wgmma m64n128k16 on both 64-row halves of the tile, 3 MMAs per k16 step:
//                                  lo*hi, hi*lo, hi*hi; fp32 accumulators in registers)
//   warp 4      : TMA producer    (cp.async.bulk.tensor, 128B-swizzled K-major tiles, ring of 2-4 stages); warps 5..7
//                                  only hand their registers to the MMA warpgroup (setmaxnreg)
//   warps 8..15 : epilogue        (bias / row-bias / GELU / residual -> fp32 and/or split-bf16 stores); two warps per
//                                  32-row quarter, so a tile drains in half the time of one warp per quarter
// The accumulator tile goes from the MMA registers to the epilogue through one fp32 tile in shared memory; the MMA
// warpgroup computes tile i+1 in registers while the epilogue drains tile i.  Tiles are 128 x 128; consecutive tile
// ids share the X (activation) tile so the big operand is read from HBM once and hit in L2 by the CTAs working on
// its other N-tiles.
//
// A second, deliberately simple SIMT kernel computes the same contraction from the same split operands
// (reconstructing hi+lo in fp32); tests use it to cross-check the tensor-core path on the GPU.
#include "gemm.cuh"

namespace ct3 {
namespace {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int TILE_A = BM * BK * 2;                    // 16 KiB (one 16-bit plane)
constexpr int TILE_B = BN * BK * 2;                    // 16 KiB
constexpr int MMA_WARPS = 4;                           // one warpgroup: warps 0..3
constexpr int TMA_WARP = 4;
constexpr int EPI_WARP0 = 8;                           // warps 5..7 of the producer warpgroup stay idle
constexpr int EPI_WARPS = 8;                           // two warps per 32-row quarter, each 64 columns
constexpr int CW = 16;                                 // epilogue chunk width (columns)
constexpr int STG_WORDS = 32 * CW;                     // per-warp transpose buffer (rotated rows: conflict-free both ways)
constexpr int MAX_STAGES = 4;
// Per products-per-FLOP variant: which operand planes a stage holds and how deep the ring is (at most 128 KiB).
//   3: A hi|lo, W hi|lo (64 KiB x 2)   2: A hi, W hi|lo (48 KiB x 2)   1: A hi, W hi (32 KiB x 4)
template <int NPROD>
struct Cfg {
  static constexpr int AP = NPROD >= 3 ? 2 : 1;
  static constexpr int BP = NPROD >= 2 ? 2 : 1;
  static constexpr int STAGE_BYTES = AP * TILE_A + BP * TILE_B;
  static constexpr int STAGES = NPROD >= 2 ? 2 : 4;
  static constexpr int OFF_B = AP * TILE_A;
};
constexpr int RING_BYTES = 2 * 65536;
static_assert(Cfg<1>::STAGES * Cfg<1>::STAGE_BYTES <= RING_BYTES && Cfg<2>::STAGES * Cfg<2>::STAGE_BYTES <= RING_BYTES &&
              Cfg<3>::STAGES * Cfg<3>::STAGE_BYTES <= RING_BYTES, "ring size");
constexpr int ACC_LD = BN + 4;                         // fp32 accumulator tile [BM][ACC_LD]
constexpr int OFF_ACC = RING_BYTES;
constexpr int OFF_STG = OFF_ACC + BM * ACC_LD * 4;
constexpr int OFF_BAR = OFF_STG + EPI_WARPS * STG_WORDS * 4;
constexpr int SMEM_BYTES = OFF_BAR + 256 /*barriers*/ + 1024 /*align slack*/;
static_assert(SMEM_BYTES <= 232448, "shared memory budget");
constexpr int THREADS = (EPI_WARP0 + EPI_WARPS) * 32;  // 4 warpgroups: 128 registers per thread at launch
// setmaxnreg moves registers from the producer warpgroup to the MMA warpgroup (2 x 64 fp32 accumulators per thread);
// the epilogue warpgroups keep the launch budget
constexpr int REG_TMA = 40, REG_MMA = 216, REG_EPI = 65536 / THREADS;
static_assert(128 * (REG_TMA + REG_MMA + 2 * REG_EPI) <= 65536, "register budget");

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == 1) return gelu_erf(x);
  if (act == 2) return gelu_tanh(x);
  return x;
}

// Epilogue of one 32-row x 16-column chunk by one warp.  Phase 1 (lane = row, read from the accumulator tile): bias /
// row-bias / activation, then the 16 output words of the row (16 fp32, or 8 packed-hi | 8 packed-lo bf16 pairs) go to
// a per-warp staging buffer whose rows are rotated by row/2 words (conflict-free for both access patterns without
// padding).  Phase 2 (lane = (row in a group of 8, 16-byte column group)): every warp instruction moves 8 rows x 64 B
// of global memory in whole 32-byte sectors.
__device__ __forceinline__ int stg_idx(int row, int word) { return row * CW + ((word + (row >> 1)) & (CW - 1)); }

__device__ __forceinline__ void epilogue_chunk(const GemmEpilogue& e, int M, int N, int row0, int col0, int lane,
                                               float (&v)[CW], uint32_t* stg) {
  const int row = row0 + lane;
  if (e.bias) {
    const float4* b4 = reinterpret_cast<const float4*>(e.bias + col0);
#pragma unroll
    for (int i = 0; i < CW / 4; ++i) {
      float4 b = __ldg(b4 + i);
      v[4 * i + 0] += b.x; v[4 * i + 1] += b.y; v[4 * i + 2] += b.z; v[4 * i + 3] += b.w;
    }
  }
  if (e.row_bias && row < M) {
    const int q = row / e.row_mod;
    const int brow = row - q * e.row_mod + (e.row_blk ? __ldg(e.row_blk + q) * e.row_mod : 0);
    const float4* b4 = reinterpret_cast<const float4*>(e.row_bias + (int64_t)brow * N + col0);
#pragma unroll
    for (int i = 0; i < CW / 4; ++i) {
      float4 b = __ldg(b4 + i);
      v[4 * i + 0] += b.x; v[4 * i + 1] += b.y; v[4 * i + 2] += b.z; v[4 * i + 3] += b.w;
    }
  }
  if (e.act != 0) {
#pragma unroll
    for (int i = 0; i < CW; ++i) v[i] = apply_act(v[i], e.act);
  }
  const int rsub = lane >> 2, q = lane & 3;   // phase-2 mapping: rows rsub + 8k, 16-byte group q of the 64-byte row
  if (e.out_f32) {
#pragma unroll
    for (int c = 0; c < CW; ++c) stg[stg_idx(lane, c)] = __float_as_uint(v[c]);
    __syncwarp();
    float* base = e.out_f32 + (int64_t)(row0 + rsub) * e.ld_f32 + col0 + 4 * q;
    const int64_t rstep = 8 * e.ld_f32;
    float4 x[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int r = 8 * k + rsub;
      x[k] = make_float4(__uint_as_float(stg[stg_idx(r, 4 * q + 0)]), __uint_as_float(stg[stg_idx(r, 4 * q + 1)]),
                         __uint_as_float(stg[stg_idx(r, 4 * q + 2)]), __uint_as_float(stg[stg_idx(r, 4 * q + 3)]));
    }
    if (e.residual) {
      float4 r4[4];
#pragma unroll
      for (int k = 0; k < 4; ++k)   // all residual rows in flight at once
        r4[k] = (row0 + 8 * k + rsub < M) ? *reinterpret_cast<const float4*>(base + k * rstep) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int k = 0; k < 4; ++k) { x[k].x += r4[k].x; x[k].y += r4[k].y; x[k].z += r4[k].z; x[k].w += r4[k].w; }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (row0 + 8 * k + rsub < M) *reinterpret_cast<float4*>(base + k * rstep) = x[k];
    __syncwarp();
  }
  if (e.out_split) {
#pragma unroll
    for (int i = 0; i < CW / 2; ++i) {
      uint32_t hi, lo;
      split2(v[2 * i], v[2 * i + 1], hi, lo);
      stg[stg_idx(lane, i)] = hi;              // words 0..7 : hi plane of this row (16 bf16)
      stg[stg_idx(lane, CW / 2 + i)] = lo;     // words 8..15: lo plane
    }
    __syncwarp();
    // output offset of this lane's row in 16-byte units (every offset is a multiple of 16 elements); one division
    // per chunk, then one 32-bit shuffle per stored row group
    uint32_t off16_lane = 0xffffffffu;
    if (row < M) {
      const int orow = row / e.row_group;
      off16_lane = (uint32_t)(((long long)orow * e.ld_split + (long long)(row % e.row_group) * N + col0) >> 3);
    }
    uint4* plane = reinterpret_cast<uint4*>(e.out_split + (q >= 2 ? e.lo_off : 0)) + (q & 1);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int r = 8 * k + rsub;
      const uint32_t o16 = __shfl_sync(0xffffffffu, off16_lane, r);
      const uint4 w4 = make_uint4(stg[stg_idx(r, 4 * q + 0)], stg[stg_idx(r, 4 * q + 1)], stg[stg_idx(r, 4 * q + 2)],
                                  stg[stg_idx(r, 4 * q + 3)]);
      if (o16 != 0xffffffffu) plane[o16] = w4;
    }
    __syncwarp();
  }
}

template <int NPROD>
__global__ void __launch_bounds__(THREADS, 1)
gemm_split3_tc_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, int M,
                      int N, int Kpad, int fp16, GemmEpilogue epi) {
  using C = Cfg<NPROD>;
  constexpr int STAGES = C::STAGES, STAGE_BYTES = C::STAGE_BYTES;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* empty_bar = full_bar + MAX_STAGES;
  uint64_t* tfull_bar = empty_bar + MAX_STAGES;   // accumulator tile written (MMA warps -> epilogue)
  uint64_t* tempty_bar = tfull_bar + 1;           // accumulator tile drained (epilogue -> MMA warps)
  float* acc_tile = reinterpret_cast<float*>(smem + OFF_ACC);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmW);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], MMA_WARPS);
    }
    mbar_init(tfull_bar, MMA_WARPS);
    mbar_init(tempty_bar, EPI_WARPS * 32);
    fence_barrier_init();
  }
  __syncthreads();

  const int num_mt = (M + BM - 1) / BM;
  const int num_nt = N / BN;
  const int num_tiles = num_mt * num_nt;
  const int num_kb = Kpad / BK;

  if (warp >= MMA_WARPS && warp < EPI_WARP0) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<REG_TMA>();
    if (warp == TMA_WARP && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int mt = tile / num_nt, nt = tile % num_nt;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
          uint8_t* s = smem + stage * STAGE_BYTES;
          tma_load_2d(s, &tmX, kb * BK, mt * BM, &full_bar[stage]);
          if (C::AP == 2) tma_load_2d(s + TILE_A, &tmX, Kpad + kb * BK, mt * BM, &full_bar[stage]);
          tma_load_2d(s + C::OFF_B, &tmW, kb * BK, nt * BN, &full_bar[stage]);
          if (C::BP == 2) tma_load_2d(s + C::OFF_B + TILE_B, &tmW, Kpad + kb * BK, nt * BN, &full_bar[stage]);
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else if (warp < MMA_WARPS) {
    // ------------------------------------------------------------------ MMA warpgroup
    setmaxnreg_inc<REG_MMA>();
    int stage = 0;
    uint32_t phase = 0, acc_phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      float d0[BN / 2], d1[BN / 2];
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);          // TMA bytes have landed
        wgmma_fence();
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
        if (fp16) mma_kblock<NPROD, BN, true>(d0, d1, sa, TILE_A, C::OFF_B, TILE_B, kb == 0);
        else mma_kblock<NPROD, BN, false>(d0, d1, sa, TILE_A, C::OFF_B, TILE_B, kb == 0);
        wgmma_commit();
        wgmma_wait0(d0);
        wgmma_wait0(d1);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);   // this warp's MMAs no longer read the slot
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      mbar_wait(tempty_bar, acc_phase ^ 1u);           // the epilogue has drained the previous tile
      acc_store<BN>(d0, acc_tile, ACC_LD);
      acc_store<BN>(d1, acc_tile + 64 * ACC_LD, ACC_LD);
      __syncwarp();
      if (lane == 0) mbar_arrive(tfull_bar);
      acc_phase ^= 1u;
    }
  } else {
    // ------------------------------------------------------------------ epilogue warps
    const int e = warp - EPI_WARP0;
    const int quarter = e & 3;                         // 32-row quarter of the tile
    constexpr int CH = BN / CW / (EPI_WARPS / 4);      // 16-column chunks per warp
    const int chunk0 = (e >> 2) * CH;
    uint32_t acc_phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int mt = tile / num_nt, nt = tile % num_nt;
      mbar_wait(tfull_bar, acc_phase);
      const int row0 = mt * BM + quarter * 32;
      uint32_t* stg = reinterpret_cast<uint32_t*>(smem + OFF_STG) + e * STG_WORDS;
      const float* arow = acc_tile + (quarter * 32 + lane) * ACC_LD;
#pragma unroll 1
      for (int chunk = chunk0; chunk < chunk0 + CH; ++chunk) {
        float v[CW];
        acc_row_ld<CW>(arow + chunk * CW, v);
        epilogue_chunk(epi, M, N, row0, nt * BN + chunk * CW, lane, v, stg);
      }
      mbar_arrive(tempty_bar);
      acc_phase ^= 1u;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Fused  q|k|v projection + per-track time attention  (Attention.forward inside the time AttnBlock,
// blocks.py:379-398, 426-432; cotracker.py:494-495):
//     att[row, h*48 .. h*48+47] = softmax( q_h k_h^T * 48^-1/2 ) v_h      over the T frames of the row's track.
// GEMM: X = LN(tokens) [M, 768 split] x Wqkv^T, the 1152 weight rows regrouped per head as [q_h(48) | k_h(48) | v_h(48)],
// so one 128 x 144 output tile holds everything head h needs for the tracks of a row tile.  Token rows are
// track-major (row = n*T + t): a tile starts at row mt*R with R = floor(128 / T) * T, i.e. it owns whole tracks
// (the MMA still multiplies 128 rows; the rows past R belong to the next tile and are ignored).
// With a per-track length table (ct3_loop_shape.group_T) track i attends over its first track_len[i] <= T frames only:
// the key loop ends there, so a track's result is that of a pass with T = track_len[i].  T > 128 is then allowed for
// tracks of at most 128 frames: R = T, one track per tile, and only its first 128 rows are computed.
// Three warpgroups: warps 0..3 MMA (wgmma m64n144k16 on both 64-row halves: 144 fp32 accumulators per thread),
// warps 4..7 producer (warp 4 issues the TMA loads), warps 8..11 epilogue (thread = row of the tile).  setmaxnreg moves
// registers from the producer warpgroup (40) to the other two (232 each) so that neither spills and the wgmmas are not
// serialised for lack of registers.  The accumulator tile is written to shared memory [row][q 48 | k 48 |
// v 48] fp32; each thread adds the bias to its row in place, keeping q in registers, and --
// after the group's named barrier -- runs exact fp32 online-softmax attention of its row against the T key rows of its
// track, then writes the 48 outputs as split bf16 straight into the out-projection's operand buffer.  The MMA
// warpgroup computes the next tile in registers meanwhile.
// The fp32 q|k|v tensor (4.6 KB per token) never reaches HBM and the separate attention launch disappears.
namespace qa {
constexpr int BNQ = 144;                               // q|k|v of one head
constexpr int TILE_BQ = BNQ * BK * 2;                  // 18432 B: the 144 weight rows, one plane
constexpr int STAGE = 2 * TILE_A + 2 * TILE_BQ;        // 69632 B
constexpr int NSTAGE = 2;
constexpr int QACC_LD = BNQ + 4;                        // floats per row of the accumulator tile (conflict-free float4)
constexpr int QOFF_ACC = NSTAGE * STAGE;
constexpr int OFF_BARQ = QOFF_ACC + BM * QACC_LD * 4;
constexpr int SMEM = OFF_BARQ + 256 + 1024;
constexpr int EPIW = 4;
constexpr int QEPI_WARP0 = 8;
constexpr int NTHREADS = 12 * 32;                      // 168 registers per thread at launch, rebalanced by setmaxnreg
constexpr int REG_PRODUCER = 40, REG_COMPUTE = 232;    // 128 x (40 + 232 + 232) <= 384 x 168
static_assert(128 * (REG_PRODUCER + 2 * REG_COMPUTE) <= NTHREADS * 168, "register budget");
static_assert(SMEM <= 232448, "shared memory budget");
}  // namespace qa

__global__ void __launch_bounds__(qa::NTHREADS, 1)
gemm_qkv_time_attn_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, int M,
                          int Kpad, int T, int R, const int32_t* __restrict__ track_len, float scale_log2e,
                          GemmEpilogue epi) {
  using namespace qa;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + OFF_BARQ);
  uint64_t* empty_bar = full_bar + NSTAGE;
  uint64_t* tfull_bar = empty_bar + NSTAGE;
  uint64_t* tempty_bar = tfull_bar + 1;
  float* acc = reinterpret_cast<float*>(smem + QOFF_ACC);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmW);
    for (int i = 0; i < NSTAGE; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], MMA_WARPS);
    }
    mbar_init(tfull_bar, MMA_WARPS);
    mbar_init(tempty_bar, EPIW * 32);
    fence_barrier_init();
  }
  __syncthreads();

  const int num_mt = (M + R - 1) / R;
  const int num_tiles = num_mt * kHeads;       // consecutive tiles = the 8 heads of one row tile (X stays in L2)
  const int num_kb = Kpad / BK;

  if (warp >= MMA_WARPS && warp < QEPI_WARP0) {
    setmaxnreg_dec<REG_PRODUCER>();
    if (warp == TMA_WARP && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int mt = tile / kHeads, h = tile % kHeads;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          mbar_arrive_expect_tx(&full_bar[stage], STAGE);
          uint8_t* s = smem + stage * STAGE;
          tma_load_2d(s, &tmX, kb * BK, mt * R, &full_bar[stage]);
          tma_load_2d(s + TILE_A, &tmX, Kpad + kb * BK, mt * R, &full_bar[stage]);
          tma_load_2d(s + 2 * TILE_A, &tmW, kb * BK, h * BNQ, &full_bar[stage]);
          tma_load_2d(s + 2 * TILE_A + TILE_BQ, &tmW, Kpad + kb * BK, h * BNQ, &full_bar[stage]);
          if (++stage == NSTAGE) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else if (warp < MMA_WARPS) {
    setmaxnreg_inc<REG_COMPUTE>();
    int stage = 0;
    uint32_t phase = 0, acc_phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      float d0[BNQ / 2], d1[BNQ / 2];
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        wgmma_fence();
        mma_kblock<3, BNQ, false>(d0, d1, smem_u32(smem + stage * STAGE), TILE_A, 2 * TILE_A, TILE_BQ, kb == 0);
        wgmma_commit();
        wgmma_wait0(d0);
        wgmma_wait0(d1);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
        if (++stage == NSTAGE) { stage = 0; phase ^= 1u; }
      }
      mbar_wait(tempty_bar, acc_phase ^ 1u);           // the epilogue is done with the previous tile's K/V
      acc_store<BNQ>(d0, acc, QACC_LD);
      acc_store<BNQ>(d1, acc + 64 * QACC_LD, QACC_LD);
      __syncwarp();
      if (lane == 0) mbar_arrive(tfull_bar);
      acc_phase ^= 1u;
    }
  } else {
    setmaxnreg_inc<REG_COMPUTE>();
    const int r = (warp - QEPI_WARP0) * 32 + lane;  // row of the tile
    const int tracks = R / T;
    const int jtrack = min(r / T, tracks - 1);     // rows past R are computed on a clamped track and never stored
    const float* kbase = acc + (int64_t)jtrack * T * QACC_LD + kDh;
    float* arow = acc + r * QACC_LD;
    uint32_t acc_phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int mt = tile / kHeads, h = tile % kHeads;
      mbar_wait(tfull_bar, acc_phase);
      acc_phase ^= 1u;
      float xq[kDh];
      // k, v + bias back into the tile in place, q (kept in registers for the attention) last
#pragma unroll
      for (int pi = 0; pi < 3; ++pi) {
        const int part = (pi + 1) % 3;   // 1 = k, 2 = v, 0 = q
        float x[kDh];
        const int col0 = kDh * part;
#pragma unroll
        for (int c = 0; c < kDh / 16; ++c) {
          float v[16];
          acc_row_ld<16>(arow + col0 + 16 * c, v);
          const float4* b4 = reinterpret_cast<const float4*>(epi.bias + h * BNQ + col0 + 16 * c);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float4 b = __ldg(b4 + i);
            x[16 * c + 4 * i + 0] = v[4 * i + 0] + b.x; x[16 * c + 4 * i + 1] = v[4 * i + 1] + b.y;
            x[16 * c + 4 * i + 2] = v[4 * i + 2] + b.z; x[16 * c + 4 * i + 3] = v[4 * i + 3] + b.w;
          }
        }
        if (part == 0) {
#pragma unroll
          for (int i = 0; i < kDh; ++i) xq[i] = x[i];
        } else {
          float4* dst = reinterpret_cast<float4*>(arow + col0);
#pragma unroll
          for (int i = 0; i < kDh / 4; ++i) dst[i] = make_float4(x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
        }
      }
      named_bar_sync(1, EPIW * 32);                  // K/V of this tile are final in shared memory
      {
        // the track's own length; a clamped track past M reads the last one (its rows are never stored).  Lengths
        // are at most min(T, 128) (gemm.cuh); the clamp keeps every key read inside this tile regardless
        const int Tk = track_len ? min(track_len[min(mt * tracks + jtrack, M / T - 1)], min(T, BM)) : T;
        float m = -INFINITY, l = 0.f;
        float o[kDh];
#pragma unroll
        for (int i = 0; i < kDh; ++i) o[i] = 0.f;
        for (int t0 = 0; t0 < Tk; t0 += 8) {
          float sc[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) sc[i] = 0.f;
#pragma unroll
          for (int d4 = 0; d4 < kDh / 4; ++d4) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float4 kk = *reinterpret_cast<const float4*>(kbase + min(t0 + i, Tk - 1) * QACC_LD + 4 * d4);
              sc[i] = fmaf(xq[4 * d4 + 0], kk.x, sc[i]);
              sc[i] = fmaf(xq[4 * d4 + 1], kk.y, sc[i]);
              sc[i] = fmaf(xq[4 * d4 + 2], kk.z, sc[i]);
              sc[i] = fmaf(xq[4 * d4 + 3], kk.w, sc[i]);
            }
          }
          float mnew = m;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            sc[i] = (t0 + i < Tk) ? sc[i] * scale_log2e : -INFINITY;
            mnew = fmaxf(mnew, sc[i]);
          }
          const float corr = exp2f(m - mnew);          // exp2(-inf) = 0 on the first chunk
          l *= corr;
#pragma unroll
          for (int i = 0; i < kDh; ++i) o[i] *= corr;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float pi = exp2f(sc[i] - mnew);      // 0 for the masked tail
            l += pi;
            const float* vr = kbase + min(t0 + i, Tk - 1) * QACC_LD + kDh;
#pragma unroll
            for (int d4 = 0; d4 < kDh / 4; ++d4) {
              const float4 vv = *reinterpret_cast<const float4*>(vr + 4 * d4);
              o[4 * d4 + 0] = fmaf(pi, vv.x, o[4 * d4 + 0]);
              o[4 * d4 + 1] = fmaf(pi, vv.y, o[4 * d4 + 1]);
              o[4 * d4 + 2] = fmaf(pi, vv.z, o[4 * d4 + 2]);
              o[4 * d4 + 3] = fmaf(pi, vv.w, o[4 * d4 + 3]);
            }
          }
          m = mnew;
        }
        mbar_arrive(tempty_bar);                     // this thread no longer reads the tile
        const int64_t grow = (int64_t)mt * R + r;
        if (r < R && grow < M) {
          const float inv = 1.0f / l;
          uint4* ph = reinterpret_cast<uint4*>(epi.out_split + grow * epi.ld_split + h * kDh);
          uint4* pl = reinterpret_cast<uint4*>(epi.out_split + grow * epi.ld_split + epi.lo_off + h * kDh);
#pragma unroll
          for (int i = 0; i < kDh / 8; ++i) {
            uint32_t hw[4], lw[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) split2(o[8 * i + 2 * j] * inv, o[8 * i + 2 * j + 1] * inv, hw[j], lw[j]);
            ph[i] = make_uint4(hw[0], hw[1], hw[2], hw[3]);
            pl[i] = make_uint4(lw[0], lw[1], lw[2], lw[3]);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// SIMT verification kernel: 64x64 tile, 256 threads, each 4x4 outputs; fp32 FMA on hi+lo.
__device__ __forceinline__ void epilogue_store1(const GemmEpilogue& e, int N, int row, int col, float v) {
  if (e.bias) v += e.bias[col];
  if (e.row_bias) {
    int64_t brow = row % e.row_mod;
    if (e.row_blk) brow += (int64_t)e.row_blk[row / e.row_mod] * e.row_mod;
    v += e.row_bias[brow * N + col];
  }
  v = apply_act(v, e.act);
  if (e.out_f32) {
    float* o = e.out_f32 + (int64_t)row * e.ld_f32 + col;
    if (e.residual) v += *o;
    *o = v;
  }
  if (e.out_split) {
    const int orow = row / e.row_group;
    const int ocol = (row % e.row_group) * N + col;
    bf16pair p = split_bf16(v);
    __nv_bfloat16* hp = e.out_split + (int64_t)orow * e.ld_split + ocol;
    hp[0] = p.hi;
    hp[e.lo_off] = p.lo;
  }
}

__global__ void __launch_bounds__(256)
gemm_split3_simt_kernel(const __nv_bfloat16* __restrict__ X, const __nv_bfloat16* __restrict__ W, int M, int N,
                        int Kpad, int64_t x_ld, int products, int fp16, GemmEpilogue epi) {
  __shared__ float As[16][64 + 1];
  __shared__ float Bs[16][64 + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  float acc[4][4] = {};
  const int64_t ld = 2 * (int64_t)Kpad;
  // the planes the tensor-core path multiplies: x_hi (+ x_lo when 3 products), w_hi (+ w_lo when >= 2 products)
  auto val = [fp16](const __nv_bfloat16* p) {
    return fp16 ? __half2float(*reinterpret_cast<const __half*>(p)) : __bfloat162float(*p);
  };
  for (int k0 = 0; k0 < Kpad; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      const int r = i >> 4, k = i & 15;
      const int gm = m0 + r, gn = n0 + r;
      float a = 0.f, b = 0.f;
      if (gm < M) a = val(X + gm * x_ld + k0 + k) + (products == 3 ? val(X + gm * x_ld + Kpad + k0 + k) : 0.f);
      if (gn < N) b = val(W + gn * ld + k0 + k) + (products >= 2 ? val(W + gn * ld + Kpad + k0 + k) : 0.f);
      As[k][r] = a;
      Bs[k][r] = b;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[k][ty * 4 + i]; b[i] = Bs[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      const int r = m0 + ty * 4 + i, c = n0 + tx * 4 + j;
      if (r < M && c < N) epilogue_store1(epi, N, r, c, acc[i][j]);
    }
}

// ------------------------------------------------------------------------------------------------
// host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static const EncodeTiledFn fn = [] {   // C++11 thread-safe one-time initialisation
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      return reinterpret_cast<EncodeTiledFn>(p);
    return (EncodeTiledFn) nullptr;
  }();
  return fn;
}

// 2-D bf16 tensor [rows, cols] row-major, box = 64 cols (128 B) x 128 rows, 128-byte swizzle, OOB -> 0
bool make_tmap(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows = 128) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return false;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 2};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

}  // namespace

bool encode_tensor_map(CUtensorMap* m, CUtensorMapDataType dtype, int rank, const void* base, const uint64_t* dims,
                       const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn || rank < 1 || rank > 5) return false;
  cuuint64_t d[5], st[5];
  cuuint32_t b[5], es[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) st[i] = strides_bytes[i];
  return fn(m, dtype, (cuuint32_t)rank, const_cast<void*>(base), d, st, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

namespace {

template <int NPROD>
cudaError_t launch_tc(const GemmProblem& p, const CUtensorMap& tmX, const CUtensorMap& tmW, int num_mt, int num_sms,
                      cudaStream_t stream) {
  static DeviceOnce attr;
  cudaError_t e = once_per_device(attr, [&] {
    return cudaFuncSetAttribute(gemm_split3_tc_kernel<NPROD>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  });
  if (e != cudaSuccess) return e;
  const int num_tiles = num_mt * (p.N / BN);
  const int grid = num_tiles < num_sms ? num_tiles : num_sms;
  gemm_split3_tc_kernel<NPROD><<<grid, THREADS, SMEM_BYTES, stream>>>(tmX, tmW, p.M, p.N, p.Kpad, p.fp16, p.epi);
  return cudaGetLastError();
}

}  // namespace

bool qkv_time_attn_supported(int T) { return T >= 1 && T <= BM; }

int gemm_qkv_time_attn_launch(const __nv_bfloat16* x_split, const __nv_bfloat16* w_heads, const float* bias_heads,
                              int M, int Kpad, int T, const int32_t* track_len, __nv_bfloat16* att_split,
                              int64_t ld_split, int lo_off, float scale, int num_sms, cudaStream_t stream,
                              const char** err) {
  *err = nullptr;
  if (M <= 0 || Kpad <= 0 || (Kpad % BK) != 0 || T < 1 || (!track_len && !qkv_time_attn_supported(T)) ||
      (M % T) != 0) {
    *err = "qkv_time_attn: need M > 0, M % T == 0, 1 <= T <= 128 (any T with track lengths), Kpad % 64 == 0";
    return (int)cudaErrorInvalidValue;
  }
  if (((reinterpret_cast<uintptr_t>(x_split) | reinterpret_cast<uintptr_t>(w_heads) |
        reinterpret_cast<uintptr_t>(att_split)) & 15) || (ld_split % 8) != 0 || (lo_off % 8) != 0) {
    *err = "qkv_time_attn: operands must be 16-byte aligned";
    return (int)cudaErrorInvalidValue;
  }
  const int R = T <= BM ? (BM / T) * T : T;
  CUtensorMap tmX, tmW;
  if (!make_tmap(&tmX, x_split, (uint64_t)M, 2ull * Kpad) ||
      !make_tmap(&tmW, w_heads, (uint64_t)(kHeads * qa::BNQ), 2ull * Kpad, (uint32_t)qa::BNQ)) {
    *err = "qkv_time_attn: cuTensorMapEncodeTiled failed";
    return (int)cudaErrorInvalidValue;
  }
  static DeviceOnce attr;
  cudaError_t e = once_per_device(attr, [&] {
    return cudaFuncSetAttribute(gemm_qkv_time_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, qa::SMEM);
  });
  if (e != cudaSuccess) { *err = "qkv_time_attn: cudaFuncSetAttribute failed"; return (int)e; }
  const int num_tiles = ((M + R - 1) / R) * kHeads;
  GemmEpilogue epi;
  epi.bias = bias_heads;
  epi.out_split = att_split;
  epi.ld_split = ld_split;
  epi.lo_off = lo_off;
  gemm_qkv_time_attn_kernel<<<num_tiles < num_sms ? num_tiles : num_sms, qa::NTHREADS, qa::SMEM, stream>>>(
      tmX, tmW, M, Kpad, T, R, track_len, scale * 1.44269504088896340736f, epi);
  return (int)cudaGetLastError();
}

const char* gemm_check(const GemmProblem& p) {
  if (p.M <= 0 || p.N <= 0 || p.Kpad <= 0 || (p.N % BN) != 0 || (p.Kpad % BK) != 0)
    return "gemm: need M>0, N % 128 == 0, Kpad % 64 == 0";
  if (p.products < 1 || p.products > 3 || p.fp16 < 0 || p.fp16 > 1) return "gemm: products in 1..3, fp16 in 0..1";
  const int64_t x_ld = p.x_ld ? p.x_ld : 2 * (int64_t)p.Kpad;
  if (x_ld < (p.products == 3 ? 2 : 1) * (int64_t)p.Kpad || (x_ld % 8) != 0)
    return "gemm: x_ld too small for the operand planes this product count reads";
  if ((reinterpret_cast<uintptr_t>(p.x_split) | reinterpret_cast<uintptr_t>(p.w_split)) & 15)
    return "gemm: operands must be 16-byte aligned";
  // The tensor-core epilogue reads bias / row bias and reads and writes the fp32 output as float4, and addresses the
  // split output in 16-byte units (epilogue_chunk): anything else would land in the wrong place without an error.
  const GemmEpilogue& e = p.epi;
  if (!e.out_f32 && !e.out_split) return "gemm: no output";
  if (e.row_mod < 1 || e.row_group < 1 || e.act < 0 || e.act > 2) return "gemm: need row_mod >= 1, row_group >= 1, act in 0..2";
  if (e.out_f32 && (e.ld_f32 < p.N || (e.ld_f32 % 4) != 0)) return "gemm: fp32 output pitch must be >= N and a multiple of 4";
  if (e.out_split) {
    const int64_t width = (int64_t)e.row_group * p.N;   // one plane of an output row
    if ((e.ld_split % 8) != 0 || (e.lo_off % 8) != 0) return "gemm: split output pitch and lo offset must be multiples of 8";
    if (e.lo_off < width || e.ld_split < e.lo_off + width) return "gemm: hi and lo planes of the split output overlap";
  }
  if ((reinterpret_cast<uintptr_t>(e.bias) | reinterpret_cast<uintptr_t>(e.row_bias) |
       reinterpret_cast<uintptr_t>(e.out_f32) | reinterpret_cast<uintptr_t>(e.out_split)) & 15)
    return "gemm: bias, row bias and outputs must be 16-byte aligned";
  return nullptr;
}

int gemm_launch(const GemmProblem& p, int impl, int num_sms, cudaStream_t stream, const char** err) {
  *err = gemm_check(p);
  if (*err) return (int)cudaErrorInvalidValue;
  const int64_t x_ld = p.x_ld ? p.x_ld : 2 * (int64_t)p.Kpad;
  if (impl == 1) {
    dim3 grid((p.N + 63) / 64, (p.M + 63) / 64);
    gemm_split3_simt_kernel<<<grid, 256, 0, stream>>>(p.x_split, p.w_split, p.M, p.N, p.Kpad, x_ld, p.products,
                                                      p.fp16, p.epi);
    return (int)cudaGetLastError();
  }
  const int num_mt = (p.M + BM - 1) / BM;
  CUtensorMap tmX, tmW;
  if (!make_tmap(&tmX, p.x_split, (uint64_t)p.M, (uint64_t)x_ld) ||
      !make_tmap(&tmW, p.w_split, (uint64_t)p.N, 2ull * p.Kpad)) {
    *err = "gemm: cuTensorMapEncodeTiled failed";
    return (int)cudaErrorInvalidValue;
  }
  cudaError_t e = p.products == 3 ? launch_tc<3>(p, tmX, tmW, num_mt, num_sms, stream)
                : p.products == 2 ? launch_tc<2>(p, tmX, tmW, num_mt, num_sms, stream)
                                  : launch_tc<1>(p, tmX, tmW, num_mt, num_sms, stream);
  return (int)e;
}

}  // namespace ct3
