// attention_p2v.cu -- point <- virtual cross attention on the Hopper tensor cores (wgmma):
//     out[n, t, h*48 ..] = softmax( q_h[n,t] . K_h[t]^T * 48^-1/2 ) V_h[t]          over the 64 virtual tokens of frame t
// (Attention.forward, blocks.py:379-398, called from CrossAttnBlock as space_point2virtual_blocks, cotracker.py:515-517).
// One CTA = one frame t x 128 consecutive tracks; per head:
//   0. ONE 3-D TMA box each brings the 128 query rows (48 fp32, rows T*ld apart in the track-major token layout), the 64
//      key rows and the 64 value rows of the head into shared memory; the loads of head h+1 are issued as soon as head
//      h's staging has been consumed, so they overlap its MMAs and softmax
//   1. conversion (a quarter warp per query row, conflict-free): fp32 -> split bf16 hi|lo planes written
//      as 128B-swizzled K-major operand tiles (q pre-multiplied by 48^-1/2 log2 e; head dim 48 zero-padded to the
//      64-element swizzle row); V_h is written TRANSPOSED ([48 dims x 64 keys], K = keys) as the B operand of the
//      second product
//   2. S = Q K^T : the CTA is one warpgroup; wgmma m64n64k16 on both 64-row halves, 3 k16 steps x 3 split products,
//      fp32 scores in registers (a query row's 64 scores are spread over the 4 lanes of a quad)
//   3. softmax per row in registers (max and sum over the quad by two shuffles, exp2), P normalised, split, written
//      over the Q tiles as the K-major A tile of the second product (64 keys = exactly one 128-byte row)
//   4. O = P V : wgmma m64n48k16 on both halves, 4 k16 steps x 3 split products -> registers -> split bf16 rows staged
//      in shared memory -> two 3-D TMA stores (hi plane, lo plane) into the out-projection's operand buffer
// A first version with one global load / store stream per thread (= per row, rows T*ld*4 bytes apart) was bound by the
// LSU request rate (252 us per call at N=6400, T=16; long_scoreboard 5.6 per issue); TMA moves whole rows instead.
// Two CTAs are resident per SM (113 KiB of shared memory each = the 228 KiB of the SM exactly).
// Grouped calls (AttnParams::gtile): every 128-track tile lies inside one group and reads that group's 64 key / value
// rows.  A TMA store clips only at the tensor-map bounds, so a group's last partial tile (unless it ends the track
// range) stores its valid rows with plain 16-byte stores instead: it never writes a row of the next group.
#include "gemm.cuh"
#include "kernels.cuh"

namespace ct3 {
namespace {

constexpr int PV_THREADS = 128;
constexpr int PV_STQ = 128 * kDh * 4;    // fp32 staging of the query rows: 24 KiB
constexpr int PV_STK = 64 * kDh * 4;     // fp32 staging of the key (value) rows: 12 KiB
constexpr int PV_TILE_Q = 128 * 128;     // [128 rows x 128 B] one plane of Q / P
constexpr int PV_TILE_K = 64 * 128;      // [64 keys x 128 B] one plane of K; V^T planes (48 x 128 B) are padded to the same
constexpr int PV_OFF_SQ = 0;
constexpr int PV_OFF_SK = PV_OFF_SQ + PV_STQ;
constexpr int PV_OFF_SV = PV_OFF_SK + PV_STK;
constexpr int PV_OFF_Q = PV_OFF_SV + PV_STK;             // 49152: hi | lo; reused for P and for the output rows
constexpr int PV_OFF_K = PV_OFF_Q + 2 * PV_TILE_Q;       // hi | lo
constexpr int PV_OFF_V = PV_OFF_K + 2 * PV_TILE_K;       // hi | lo
constexpr int PV_OFF_BAR = PV_OFF_V + kDh * 128;         // in the unused tail (rows 48..63) of the V^T hi plane
constexpr int PV_OFF_END = PV_OFF_V + 2 * PV_TILE_K;     // 114688
constexpr int PV_SMEM = PV_OFF_END + 1024;               // 2 x (PV_SMEM + 1 KiB driver reserve) = 228 KiB exactly
constexpr uint32_t PV_LOAD_BYTES = PV_STQ + 2 * PV_STK;
static_assert(2 * (PV_SMEM + 1024) <= 233472, "two CTAs per SM");
static_assert(128 * kDh * 2 <= PV_TILE_Q, "one plane of output rows fits one Q/P tile");
static_assert(kDh == 48 && kV == 64, "chunk arithmetic below");

struct P2vMaps { CUtensorMap q, kv, out; };

__device__ __forceinline__ uint32_t swz(int r, int c16) { return (uint32_t)(r * 128 + ((c16 ^ (r & 7)) << 4)); }

__global__ void __launch_bounds__(PV_THREADS, 2)
attn_p2v_tc_kernel(const __grid_constant__ P2vMaps maps, AttnParams p, int tiles_per_seq) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint64_t* bar_ld = reinterpret_cast<uint64_t*>(smem + PV_OFF_BAR);
  const int r = threadIdx.x, warp = r >> 5, lane = r & 31;
  const int t = blockIdx.x / tiles_per_seq, tile = blockIdx.x % tiles_per_seq;
  int n0 = tile * 128, kv0 = 0, n_end = p.Lq;   // tracks [n0, n_end) of this tile's group; its keys start at token kv0
  if (p.gtile) {
    const int g = p.gtile[2 * tile];
    n0 = p.gtile[2 * tile + 1];
    kv0 = g * kV;
    n_end = p.goff[g + 1];
  }
  const bool tma_store = n0 + 128 <= n_end || n_end == p.Lq;

  // zero the operand tiles once (V^T rows are fully rewritten per head, the K padding columns 48..63 never are)
  for (int i = r; i < (PV_OFF_END - PV_OFF_Q) / 16; i += PV_THREADS)
    reinterpret_cast<uint4*>(smem + PV_OFF_Q)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();   // the barriers live inside the zeroed range
  if (r == 0) {
    tma_prefetch_desc(&maps.q);
    tma_prefetch_desc(&maps.kv);
    tma_prefetch_desc(&maps.out);
    mbar_init(bar_ld, 1);
    fence_barrier_init();
  }
  __syncthreads();
  const float qscale = p.scale * 1.44269504088896340736f;
  // wgmma fragment rows of this thread: half hh, rows 64hh + rq and 64hh + rq + 8; columns 8j + cq, 8j + cq + 1
  const int rq = 16 * warp + (lane >> 2), cq = 2 * (lane & 3);
  const uint32_t sQ = smem_u32(smem + PV_OFF_Q), sK = smem_u32(smem + PV_OFF_K), sV = smem_u32(smem + PV_OFF_V);
  // key / value conversion: this thread's key and the first of its six 4-float chunks (rotated by the lane so that the
  // 192-byte staging rows are read, and the transposed V rows written, without bank conflicts)
  const int kv_key = (warp & 1) * 32 + lane, kv_c0 = (warp >> 1) * 6 + lane;

  auto issue_loads = [&](int h) {   // one thread
    mbar_arrive_expect_tx(bar_ld, PV_LOAD_BYTES);
    tma_load_3d(smem + PV_OFF_SQ, &maps.q, p.q_col + h * kDh, t, n0, bar_ld);
    tma_load_3d(smem + PV_OFF_SK, &maps.kv, p.k_col + h * kDh, t, kv0, bar_ld);
    tma_load_3d(smem + PV_OFF_SV, &maps.kv, p.v_col + h * kDh, t, kv0, bar_ld);
  };
  if (r == 0) issue_loads(0);

  for (int h = 0; h < kHeads; ++h) {
    const uint32_t ph = (uint32_t)(h & 1);
    mbar_wait(bar_ld, ph);
    // ---- 1. staging -> split operand tiles
    {
      // Q: 8 lanes per row, lane slot s < 6 converts the row's 16-byte chunk s (8 channels), slots 6 and 7 re-zero the
      // head-dim padding chunks (P lived there): a quarter warp writes one row = 8 distinct swizzle positions
      const float4* sq = reinterpret_cast<const float4*>(smem + PV_OFF_SQ);
      const int slot = r & 7;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int row = j * 16 + (r >> 3);
        uint4 qh = make_uint4(0, 0, 0, 0), ql = make_uint4(0, 0, 0, 0);
        if (slot < 6) {
          const float4 a = sq[row * 12 + 2 * slot], b = sq[row * 12 + 2 * slot + 1];
          split2(a.x * qscale, a.y * qscale, qh.x, ql.x);
          split2(a.z * qscale, a.w * qscale, qh.y, ql.y);
          split2(b.x * qscale, b.y * qscale, qh.z, ql.z);
          split2(b.z * qscale, b.w * qscale, qh.w, ql.w);
        }
        *reinterpret_cast<uint4*>(smem + PV_OFF_Q + swz(row, slot)) = qh;
        *reinterpret_cast<uint4*>(smem + PV_OFF_Q + PV_TILE_Q + swz(row, slot)) = ql;
      }
      const float4* sk = reinterpret_cast<const float4*>(smem + PV_OFF_SK) + kv_key * 12;
      const float4* sv = reinterpret_cast<const float4*>(smem + PV_OFF_SV) + kv_key * 12;
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        const int c = (kv_c0 + j) % 12;
        const float4 a = sk[c];
        uint32_t h0, l0, h1, l1;
        split2(a.x, a.y, h0, l0);
        split2(a.z, a.w, h1, l1);
        const uint32_t off = swz(kv_key, c >> 1) + (uint32_t)((c & 1) * 8);
        *reinterpret_cast<uint2*>(smem + PV_OFF_K + off) = make_uint2(h0, h1);
        *reinterpret_cast<uint2*>(smem + PV_OFF_K + PV_TILE_K + off) = make_uint2(l0, l1);
        // V^T: element (dim d, key) at row d, 16-byte chunk key / 8, position key % 8
        const float4 b = sv[c];
        const float vals[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int d = 4 * c + i;
          const bf16pair sp = split_bf16(vals[i]);
          const uint32_t vo = swz(d, kv_key >> 3) + (uint32_t)((kv_key & 7) * 2);
          *reinterpret_cast<__nv_bfloat16*>(smem + PV_OFF_V + vo) = sp.hi;
          *reinterpret_cast<__nv_bfloat16*>(smem + PV_OFF_V + PV_TILE_K + vo) = sp.lo;
        }
      }
    }
    fence_proxy_async_smem();
    __syncthreads();                               // tiles complete; staging consumed
    if (r == 0 && h + 1 < kHeads) issue_loads(h + 1);   // next head's rows arrive while this head computes
    // ---- 2. S = Q K^T (both 64-row halves; q already carries the softmax scale and log2 e)
    float s0[32], s1[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kDh / 16; ++kk) {
      const uint32_t ko = kk * 32;
      const uint64_t kh = gmma_desc_sw128(sK + ko), kl = gmma_desc_sw128(sK + PV_TILE_K + ko);
      const uint32_t first = kk != 0 ? 1u : 0u;
      wgmma_tile<64, false>(s0, gmma_desc_sw128(sQ + PV_TILE_Q + ko), kh, first);
      wgmma_tile<64, false>(s0, gmma_desc_sw128(sQ + ko), kl, 1u);
      wgmma_tile<64, false>(s0, gmma_desc_sw128(sQ + ko), kh, 1u);
      wgmma_tile<64, false>(s1, gmma_desc_sw128(sQ + 8192 + PV_TILE_Q + ko), kh, first);
      wgmma_tile<64, false>(s1, gmma_desc_sw128(sQ + 8192 + ko), kl, 1u);
      wgmma_tile<64, false>(s1, gmma_desc_sw128(sQ + 8192 + ko), kh, 1u);
    }
    wgmma_commit();
    wgmma_wait0(s0);
    wgmma_wait0(s1);
    __syncthreads();                               // every warp's MMAs have read the Q tiles: P may overwrite them
    // ---- 3. softmax of each row (4 lanes of a quad x 16 scores) -> normalised P (split) over the Q tiles
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float (&sc)[32] = hh ? s1 : s0;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {             // fragment elements 4j + 2rr + {0,1}: row 64hh + rq + 8rr
        float m = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j) m = fmaxf(m, fmaxf(sc[4 * j + 2 * rr], sc[4 * j + 2 * rr + 1]));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        float l = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          sc[4 * j + 2 * rr] = exp2f(sc[4 * j + 2 * rr] - m);
          sc[4 * j + 2 * rr + 1] = exp2f(sc[4 * j + 2 * rr + 1] - m);
          l += sc[4 * j + 2 * rr] + sc[4 * j + 2 * rr + 1];
        }
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const float inv = 1.0f / l;
        const int row = 64 * hh + rq + 8 * rr;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          uint32_t ph, pl;
          split2(sc[4 * j + 2 * rr] * inv, sc[4 * j + 2 * rr + 1] * inv, ph, pl);
          const uint32_t off = swz(row, j) + (uint32_t)(cq * 2);
          *reinterpret_cast<uint32_t*>(smem + PV_OFF_Q + off) = ph;
          *reinterpret_cast<uint32_t*>(smem + PV_OFF_Q + PV_TILE_Q + off) = pl;
        }
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
    // ---- 4. O = P V
    float o0[24], o1[24];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint32_t ko = kk * 32;
      const uint64_t vh = gmma_desc_sw128(sV + ko), vl = gmma_desc_sw128(sV + PV_TILE_K + ko);
      const uint32_t first = kk != 0 ? 1u : 0u;
      wgmma_tile<48, false>(o0, gmma_desc_sw128(sQ + PV_TILE_Q + ko), vh, first);
      wgmma_tile<48, false>(o0, gmma_desc_sw128(sQ + ko), vl, 1u);
      wgmma_tile<48, false>(o0, gmma_desc_sw128(sQ + ko), vh, 1u);
      wgmma_tile<48, false>(o1, gmma_desc_sw128(sQ + 8192 + PV_TILE_Q + ko), vh, first);
      wgmma_tile<48, false>(o1, gmma_desc_sw128(sQ + 8192 + ko), vl, 1u);
      wgmma_tile<48, false>(o1, gmma_desc_sw128(sQ + 8192 + ko), vh, 1u);
    }
    wgmma_commit();
    wgmma_wait0(o0);
    wgmma_wait0(o1);
    __syncthreads();                               // the P tiles are dead: stage the 128 x 48 output rows there
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const float (&oc)[24] = hh ? o1 : o0;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int row = 64 * hh + rq + 8 * rr;
#pragma unroll
        for (int j = 0; j < 6; ++j) {
          uint32_t oh, ol;
          split2(oc[4 * j + 2 * rr], oc[4 * j + 2 * rr + 1], oh, ol);
          const int off = row * (kDh * 2) + (8 * j + cq) * 2;   // dense 96-byte rows: hi plane | lo plane
          *reinterpret_cast<uint32_t*>(smem + PV_OFF_Q + off) = oh;
          *reinterpret_cast<uint32_t*>(smem + PV_OFF_Q + PV_TILE_Q + off) = ol;
        }
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
    if (tma_store) {
      if (r == 0) {
        tma_store_3d(&maps.out, h * kDh, t, n0, smem + PV_OFF_Q);
        tma_store_3d(&maps.out, p.lo_off + h * kDh, t, n0, smem + PV_OFF_Q + PV_TILE_Q);
        bulk_commit();
        bulk_wait_read0();    // the stores have read the rows: the next head may rewrite the Q tiles
      }
    } else {
      // rows [n0, n_end) only: 2 planes x 6 chunks of 16 bytes per 96-byte row
      for (int i = r; i < (n_end - n0) * 12; i += PV_THREADS) {
        const int row = i / 12, plane = (i % 12) / 6, c = i % 6;
        const uint4 v = *reinterpret_cast<const uint4*>(smem + PV_OFF_Q + plane * PV_TILE_Q + row * (kDh * 2) + c * 16);
        __nv_bfloat16* dst = p.out + ((int64_t)t * p.q_seq_stride + (int64_t)(n0 + row) * p.q_tok_stride) * p.out_ld +
                             plane * p.lo_off + h * kDh + c * 8;
        *reinterpret_cast<uint4*>(dst) = v;
      }
    }
    __syncthreads();
  }
  if (r == 0) bulk_wait0();
}

}  // namespace

bool attention_p2v_supported(const AttnParams& p) {
  return (p.gtile ? p.Lk >= kV && p.Lk % kV == 0 : p.Lk == kV) && p.Lq >= 1 && (p.q_ld % 4) == 0 && (p.kv_ld % 4) == 0 && (p.q_col % 4) == 0 && (p.k_col % 4) == 0 &&
         (p.v_col % 4) == 0 && (p.out_ld % 8) == 0 && (p.lo_off % 8) == 0 &&
         ((reinterpret_cast<uintptr_t>(p.q) | reinterpret_cast<uintptr_t>(p.kv) | reinterpret_cast<uintptr_t>(p.out)) & 15) == 0;
}

cudaError_t launch_attention_p2v(const AttnParams& p, cudaStream_t s) {
  if (!attention_p2v_supported(p)) return cudaErrorInvalidValue;
  P2vMaps maps;
  {
    // row of (sequence s, token i) = s*seq_stride + i*tok_stride: 3-D tensors (columns, sequence, token)
    const uint64_t qd[3] = {(uint64_t)p.q_ld, (uint64_t)p.num_seq, (uint64_t)p.Lq};
    const uint64_t qs[2] = {(uint64_t)p.q_seq_stride * p.q_ld * 4, (uint64_t)p.q_tok_stride * p.q_ld * 4};
    const uint32_t qb[3] = {(uint32_t)kDh, 1, 128};
    const uint64_t kd[3] = {(uint64_t)p.kv_ld, (uint64_t)p.num_seq, (uint64_t)p.Lk};
    const uint64_t ks[2] = {(uint64_t)p.k_seq_stride * p.kv_ld * 4, (uint64_t)p.k_tok_stride * p.kv_ld * 4};
    const uint32_t kb[3] = {(uint32_t)kDh, 1, 64};
    const uint64_t od[3] = {(uint64_t)p.out_ld, (uint64_t)p.num_seq, (uint64_t)p.Lq};
    const uint64_t os[2] = {(uint64_t)p.q_seq_stride * p.out_ld * 2, (uint64_t)p.q_tok_stride * p.out_ld * 2};
    const uint32_t ob[3] = {(uint32_t)kDh, 1, 128};
    if (!encode_tensor_map(&maps.q, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, p.q, qd, qs, qb, CU_TENSOR_MAP_SWIZZLE_NONE) ||
        !encode_tensor_map(&maps.kv, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, p.kv, kd, ks, kb, CU_TENSOR_MAP_SWIZZLE_NONE) ||
        !encode_tensor_map(&maps.out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, p.out, od, os, ob, CU_TENSOR_MAP_SWIZZLE_NONE))
      return cudaErrorInvalidValue;
  }
  static DeviceOnce attr;
  cudaError_t e = once_per_device(attr, [&] {
    return cudaFuncSetAttribute(attn_p2v_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PV_SMEM);
  });
  if (e != cudaSuccess) return e;
  const int tiles = p.gtile ? p.tiles : (p.Lq + 127) / 128;
  attn_p2v_tc_kernel<<<p.num_seq * tiles, PV_THREADS, PV_SMEM, s>>>(maps, p, tiles);
  return cudaGetLastError();
}

}  // namespace ct3
