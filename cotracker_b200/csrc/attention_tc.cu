// attention_tc.cu -- tensor-core attention core (production path; attention.cu keeps the exact-fp32 SIMT version
// used by the tests as an on-GPU cross-check).
//
//   out = softmax(q k^T * 48^-1/2) v      (Attention.forward, blocks.py:391-397), 8 heads x 48
//
// Flash-style: one warp owns a 16-query tile; keys stream through shared memory in chunks of KB; scores and
// P*V run on the tensor cores as m16n8k16 bf16 MMAs with every operand split hi+lo (3 MMAs per product:
// lo*hi + hi*lo + hi*hi, fp32 accumulate) -- the same 2^-17 product precision as the wgmma linear layers;
// max / exp / sum are fp32 on the accumulator fragments (online softmax).  Attention is ~2 % of a block's
// FLOPs and its tiles are 16 x 48: warp-level mma.sync is the right granularity here (a 64-row wgmma tile
// would idle 7/8 of the array for the T=16 time attention), the 128-wide contractions live in gemm.cu.
//
// Modes:  PER_WARP  = each warp has its own (sequence, head, q-tile) and its own K/V smem slice (time attention)
//         shared    = the 4 warps of a CTA share one (sequence, head) K/V chunk (space attention)
//         split-K   = the key range is split over gridDim.z CTAs that emit (m, l, O) partials (virtual <- point:
//                     64 queries x N keys), merged by attention_combine_kernel.
// Grouped calls (AttnParams::gl) run the shared mode over (group, frame) sequences of different lengths in one launch;
// each entry has its own split-K count, so every group's chunk ranges and combine order are those of a standalone call.
#include "kernels.cuh"

namespace ct3 {
namespace {

constexpr int WARPS = 4;
constexpr int KPAD = 56;  // bf16 row stride of K tiles: 112 B -> conflict-free fragment loads

__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int KB, bool PER_WARP>
__global__ void __launch_bounds__(WARPS * 32, 4)
attention_tc_kernel(AttnParams p, int q_tiles, int num_splits, int qtw, float* part_ml, float* part_o) {
  constexpr int VPAD = KB + 8;  // bf16 row stride of V^T tiles
  constexpr int SLICE = 2 * KB * KPAD + 2 * kDh * VPAD;  // bf16 elements per K/V staging slice
  extern __shared__ __align__(16) uint8_t att_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t4 = lane & 3;

  // ---- work item
  int s, h, qt, split = 0;
  bool active = true;
  if (PER_WARP) {
    const long long item = (long long)blockIdx.x * WARPS + warp;
    const long long items = (long long)p.num_seq * kHeads * q_tiles;
    active = item < items;
    const long long it = active ? item : 0;
    qt = (int)(it % q_tiles);
    h = (int)((it / q_tiles) % kHeads);
    s = (int)(it / ((long long)q_tiles * kHeads));
  } else {
    s = blockIdx.x;
    h = blockIdx.y % kHeads;
    const int qb = blockIdx.y / kHeads;
    qt = (qb * WARPS + warp) * qtw;   // first of the qtw query tiles this warp walks (single-chunk K/V only)
    split = blockIdx.z;
  }
  const SeqRows sr = seq_rows(p, s);   // PER_WARP (time attention) is never grouped
  const int Lq = sr.Lq, Lk = sr.Lk;
  const int nsp = p.gl ? (p.gsplit ? p.gsplit[sr.e] : 1) : num_splits;
  if (!PER_WARP) {
    q_tiles = (Lq + 15) / 16;
    // grouped: CTAs past this sequence's queries or split count (CTA-uniform, before any barrier)
    if (split >= nsp || (int)(blockIdx.y / kHeads) * WARPS * qtw >= q_tiles) return;
  }
  const int qt_first = qt;
  const bool item_ok = active;
  __nv_bfloat16* slice = reinterpret_cast<__nv_bfloat16*>(att_smem) + (PER_WARP ? warp * SLICE : 0);
  __nv_bfloat16* Kh = slice;
  __nv_bfloat16* Kl = Kh + KB * KPAD;
  __nv_bfloat16* Vh = Kl + KB * KPAD;   // V^T [48][VPAD]
  __nv_bfloat16* Vl = Vh + kDh * VPAD;

  // key range of this CTA (split-K) in units of chunks
  const int chunks = (Lk + KB - 1) / KB;
  const int c_per = (chunks + nsp - 1) / nsp;
  const int c_begin = split * c_per, c_end = min(chunks, c_begin + c_per);

  // K/V are staged once when they fit one chunk; the warp then walks qtw query tiles against them
  for (int ti = 0; ti < qtw; ++ti) {
  qt = qt_first + ti;
  active = item_ok && qt < q_tiles;
  if (qt >= q_tiles) qt = q_tiles - 1;
  const bool stage_now = (ti == 0) || (c_end - c_begin > 1);
  // ---- Q fragments (rows g and g+8 of the tile), split hi/lo
  const int q_row0 = qt * 16 + g, q_row1 = q_row0 + 8;
  uint32_t qh[3][4], ql[3][4];
  {
    const int r0 = min(q_row0, Lq - 1), r1 = min(q_row1, Lq - 1);
    const float* qp0 = p.q + (sr.q0 + (int64_t)r0 * p.q_tok_stride) * p.q_ld + p.q_col + h * kDh;
    const float* qp1 = p.q + (sr.q0 + (int64_t)r1 * p.q_tok_stride) * p.q_ld + p.q_col + h * kDh;
#pragma unroll
    for (int ks = 0; ks < 3; ++ks) {
      const float2 a0 = __ldg(reinterpret_cast<const float2*>(qp0 + 16 * ks + 2 * t4));
      const float2 a1 = __ldg(reinterpret_cast<const float2*>(qp1 + 16 * ks + 2 * t4));
      const float2 a2 = __ldg(reinterpret_cast<const float2*>(qp0 + 16 * ks + 8 + 2 * t4));
      const float2 a3 = __ldg(reinterpret_cast<const float2*>(qp1 + 16 * ks + 8 + 2 * t4));
      split2(a0.x, a0.y, qh[ks][0], ql[ks][0]);
      split2(a1.x, a1.y, qh[ks][1], ql[ks][1]);
      split2(a2.x, a2.y, qh[ks][2], ql[ks][2]);
      split2(a3.x, a3.y, qh[ks][3], ql[ks][3]);
    }
  }

  float o[6][4];
#pragma unroll
  for (int nd = 0; nd < 6; ++nd) o[nd][0] = o[nd][1] = o[nd][2] = o[nd][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  for (int c = c_begin; c < c_end; ++c) {
    const int kc0 = c * KB;
    // ---- stage K (row-major) and V^T, split hi/lo; zero-fill past Lk
    if (stage_now) {
      const int nthr = PER_WARP ? 32 : WARPS * 32;
      const int tid = PER_WARP ? lane : threadIdx.x;
      // one work item = 4 channels of two adjacent keys: K rows get 8-byte stores, V^T gets 4-byte stores of
      // (key j, key j+1) pairs instead of 2-byte scatters
      for (int idx = tid; idx < (KB / 2) * (kDh / 4); idx += nthr) {
        const int j = 2 * (idx / (kDh / 4)), d4 = idx % (kDh / 4);
        float4 k0 = make_float4(0.f, 0.f, 0.f, 0.f), k1 = k0, v0 = k0, v1 = k0;
        if (kc0 + j < Lk) {
          const float* base = p.kv + (sr.k0 + (int64_t)(kc0 + j) * p.k_tok_stride) * p.kv_ld + h * kDh;
          k0 = __ldg(reinterpret_cast<const float4*>(base + p.k_col) + d4);
          v0 = __ldg(reinterpret_cast<const float4*>(base + p.v_col) + d4);
        }
        if (kc0 + j + 1 < Lk) {
          const float* base = p.kv + (sr.k0 + (int64_t)(kc0 + j + 1) * p.k_tok_stride) * p.kv_ld + h * kDh;
          k1 = __ldg(reinterpret_cast<const float4*>(base + p.k_col) + d4);
          v1 = __ldg(reinterpret_cast<const float4*>(base + p.v_col) + d4);
        }
        uint32_t h0, l0_, h1, l1_;
        split2(k0.x, k0.y, h0, l0_);
        split2(k0.z, k0.w, h1, l1_);
        *reinterpret_cast<uint2*>(Kh + j * KPAD + 4 * d4) = make_uint2(h0, h1);
        *reinterpret_cast<uint2*>(Kl + j * KPAD + 4 * d4) = make_uint2(l0_, l1_);
        split2(k1.x, k1.y, h0, l0_);
        split2(k1.z, k1.w, h1, l1_);
        *reinterpret_cast<uint2*>(Kh + (j + 1) * KPAD + 4 * d4) = make_uint2(h0, h1);
        *reinterpret_cast<uint2*>(Kl + (j + 1) * KPAD + 4 * d4) = make_uint2(l0_, l1_);
        const float va[4] = {v0.x, v0.y, v0.z, v0.w}, vb[4] = {v1.x, v1.y, v1.z, v1.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          uint32_t vh, vl;
          split2(va[i], vb[i], vh, vl);   // (key j | key j+1) of channel 4*d4+i
          *reinterpret_cast<uint32_t*>(Vh + (4 * d4 + i) * VPAD + j) = vh;
          *reinterpret_cast<uint32_t*>(Vl + (4 * d4 + i) * VPAD + j) = vl;
        }
      }
    }
    if (stage_now) { if (PER_WARP) __syncwarp(); else __syncthreads(); }

    // ---- S = Q K^T  (16 x KB per warp)
    float sc[KB / 8][4];
#pragma unroll
    for (int nt = 0; nt < KB / 8; ++nt) sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 3; ++ks) {
#pragma unroll
      for (int nt = 0; nt < KB / 8; ++nt) {
        const int off = (nt * 8 + g) * KPAD + 16 * ks + 2 * t4;
        const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(Kh + off), bh1 = *reinterpret_cast<const uint32_t*>(Kh + off + 8);
        const uint32_t bl0 = *reinterpret_cast<const uint32_t*>(Kl + off), bl1 = *reinterpret_cast<const uint32_t*>(Kl + off + 8);
        mma16816(sc[nt], ql[ks], bh0, bh1);
        mma16816(sc[nt], qh[ks], bl0, bl1);
        mma16816(sc[nt], qh[ks], bh0, bh1);
      }
    }
    // ---- online softmax on the fragments (rows g: c0,c1 ; g+8: c2,c3)
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < KB / 8; ++nt) {
      const int key = kc0 + nt * 8 + 2 * t4;
      const bool v0 = key < Lk, v1 = key + 1 < Lk;
      sc[nt][0] = v0 ? sc[nt][0] * p.scale : -INFINITY;
      sc[nt][1] = v1 ? sc[nt][1] * p.scale : -INFINITY;
      sc[nt][2] = v0 ? sc[nt][2] * p.scale : -INFINITY;
      sc[nt][3] = v1 ? sc[nt][3] * p.scale : -INFINITY;
      mx0 = fmaxf(mx0, fmaxf(sc[nt][0], sc[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(sc[nt][2], sc[nt][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);   // finite: every chunk holds >= 1 valid key
    const float cr0 = expf(m0 - mn0), cr1 = expf(m1 - mn1);
    m0 = mn0; m1 = mn1;
    l0 *= cr0; l1 *= cr1;
#pragma unroll
    for (int nd = 0; nd < 6; ++nd) { o[nd][0] *= cr0; o[nd][1] *= cr0; o[nd][2] *= cr1; o[nd][3] *= cr1; }
#pragma unroll
    for (int nt = 0; nt < KB / 8; ++nt) {
      sc[nt][0] = expf(sc[nt][0] - mn0); sc[nt][1] = expf(sc[nt][1] - mn0);
      sc[nt][2] = expf(sc[nt][2] - mn1); sc[nt][3] = expf(sc[nt][3] - mn1);
      l0 += sc[nt][0] + sc[nt][1];
      l1 += sc[nt][2] + sc[nt][3];
    }
    // ---- O += P V   (P from the score fragments: two n8 tiles make one k16 A fragment)
#pragma unroll
    for (int j = 0; j < KB / 16; ++j) {
      uint32_t ph[4], pl[4];
      split2(sc[2 * j][0], sc[2 * j][1], ph[0], pl[0]);
      split2(sc[2 * j][2], sc[2 * j][3], ph[1], pl[1]);
      split2(sc[2 * j + 1][0], sc[2 * j + 1][1], ph[2], pl[2]);
      split2(sc[2 * j + 1][2], sc[2 * j + 1][3], ph[3], pl[3]);
#pragma unroll
      for (int nd = 0; nd < 6; ++nd) {
        const int off = (nd * 8 + g) * VPAD + 16 * j + 2 * t4;
        const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(Vh + off), bh1 = *reinterpret_cast<const uint32_t*>(Vh + off + 8);
        const uint32_t bl0 = *reinterpret_cast<const uint32_t*>(Vl + off), bl1 = *reinterpret_cast<const uint32_t*>(Vl + off + 8);
        mma16816(o[nd], pl, bh0, bh1);
        mma16816(o[nd], ph, bl0, bl1);
        mma16816(o[nd], ph, bh0, bh1);
      }
    }
    if (c_end - c_begin > 1) { if (PER_WARP) __syncwarp(); else __syncthreads(); }   // smem is restaged next chunk
  }

  // ---- finish: row sums across the quad, normalise, store
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  if (!active) continue;
  if (nsp > 1) {
    // partials: item = (slot * frames + frame) * heads + h, rows indexed by query
    const int64_t item = (((p.gl ? p.gslot[sr.e] : 0) + (int64_t)split) * (p.gl ? p.frames : p.num_seq) + sr.t) * kHeads + h;
    float* pml = part_ml + item * p.Lq * 2;
    float* po = part_o + item * p.Lq * kDh;
    if (q_row0 < Lq) {
      if (t4 == 0) { pml[q_row0 * 2] = m0; pml[q_row0 * 2 + 1] = l0; }
#pragma unroll
      for (int nd = 0; nd < 6; ++nd) *reinterpret_cast<float2*>(po + (int64_t)q_row0 * kDh + nd * 8 + 2 * t4) = make_float2(o[nd][0], o[nd][1]);
    }
    if (q_row1 < Lq) {
      if (t4 == 0) { pml[q_row1 * 2] = m1; pml[q_row1 * 2 + 1] = l1; }
#pragma unroll
      for (int nd = 0; nd < 6; ++nd) *reinterpret_cast<float2*>(po + (int64_t)q_row1 * kDh + nd * 8 + 2 * t4) = make_float2(o[nd][2], o[nd][3]);
    }
    continue;
  }
  const float i0 = 1.0f / l0, i1 = 1.0f / l1;
  if (q_row0 < Lq) {
    __nv_bfloat16* orow = p.out + (sr.q0 + (int64_t)q_row0 * p.q_tok_stride) * p.out_ld + h * kDh;
#pragma unroll
    for (int nd = 0; nd < 6; ++nd) {
      uint32_t hi, lo;
      split2(o[nd][0] * i0, o[nd][1] * i0, hi, lo);
      *reinterpret_cast<uint32_t*>(orow + nd * 8 + 2 * t4) = hi;
      *reinterpret_cast<uint32_t*>(orow + p.lo_off + nd * 8 + 2 * t4) = lo;
    }
  }
  if (q_row1 < Lq) {
    __nv_bfloat16* orow = p.out + (sr.q0 + (int64_t)q_row1 * p.q_tok_stride) * p.out_ld + h * kDh;
#pragma unroll
    for (int nd = 0; nd < 6; ++nd) {
      uint32_t hi, lo;
      split2(o[nd][2] * i1, o[nd][3] * i1, hi, lo);
      *reinterpret_cast<uint32_t*>(orow + nd * 8 + 2 * t4) = hi;
      *reinterpret_cast<uint32_t*>(orow + p.lo_off + nd * 8 + 2 * t4) = lo;
    }
  }
  }  // ti
}

// merge split-K partials: one warp per (s, h, query); lanes over the 48 output channels
__global__ void __launch_bounds__(128)
attention_combine_kernel(AttnParams p, int num_splits, const float* __restrict__ part_ml, const float* __restrict__ part_o) {
  const int64_t w = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int64_t total = (int64_t)p.num_seq * kHeads * p.Lq;
  if (w >= total) return;
  const int qi = (int)(w % p.Lq);
  const int h = (int)((w / p.Lq) % kHeads);
  const int s = (int)(w / ((int64_t)p.Lq * kHeads));
  const SeqRows sr = seq_rows(p, s);
  const int nsp = p.gl ? (p.gsplit ? p.gsplit[sr.e] : 1) : num_splits;
  if (nsp <= 1 || qi >= sr.Lq) return;   // grouped: this entry wrote its output directly
  const int64_t slot0 = p.gl ? p.gslot[sr.e] : 0, frames = p.gl ? p.frames : p.num_seq;
  float m = -INFINITY;
  for (int k = 0; k < nsp; ++k) {
    const int64_t item = ((slot0 + k) * frames + sr.t) * kHeads + h;
    m = fmaxf(m, part_ml[(item * p.Lq + qi) * 2]);
  }
  float l = 0.f, a0 = 0.f, a1 = 0.f;
  for (int k = 0; k < nsp; ++k) {
    const int64_t item = ((slot0 + k) * frames + sr.t) * kHeads + h;
    const float mk = part_ml[(item * p.Lq + qi) * 2], lk = part_ml[(item * p.Lq + qi) * 2 + 1];
    const float wgt = (mk == -INFINITY) ? 0.f : expf(mk - m);
    l += wgt * lk;
    const float* po = part_o + (item * p.Lq + qi) * kDh;
    a0 += wgt * po[lane];
    if (lane < kDh - 32) a1 += wgt * po[32 + lane];
  }
  const float inv = 1.0f / l;
  __nv_bfloat16* orow = p.out + (sr.q0 + (int64_t)qi * p.q_tok_stride) * p.out_ld + h * kDh;
  const bf16pair x = split_bf16(a0 * inv);
  orow[lane] = x.hi;
  orow[p.lo_off + lane] = x.lo;
  if (lane < kDh - 32) {
    const bf16pair y = split_bf16(a1 * inv);
    orow[32 + lane] = y.hi;
    orow[p.lo_off + 32 + lane] = y.lo;
  }
}

template <int KB, bool PER_WARP>
cudaError_t launch_variant(const AttnParams& p, int num_splits, int qtw, float* part_ml, float* part_o, cudaStream_t s) {
  constexpr int VPAD = KB + 8;
  constexpr int SLICE_BYTES = (2 * KB * KPAD + 2 * kDh * VPAD) * 2;
  const int smem = SLICE_BYTES * (PER_WARP ? WARPS : 1);
  const int q_tiles = (p.Lq + 15) / 16;
  static DeviceOnce attr;
  if (smem > 48 * 1024) {
    cudaError_t e = once_per_device(attr, [&] {
      return cudaFuncSetAttribute(attention_tc_kernel<KB, PER_WARP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    });
    if (e != cudaSuccess) return e;
  }
  if (PER_WARP) {
    const long long items = (long long)p.num_seq * kHeads * q_tiles;
    const long long blocks = (items + WARPS - 1) / WARPS;
    if (blocks > 0x7fffffffLL) return cudaErrorInvalidValue;
    attention_tc_kernel<KB, true><<<(unsigned)blocks, WARPS * 32, smem, s>>>(p, q_tiles, 1, 1, nullptr, nullptr);
  } else {
    const int qblocks = (q_tiles + WARPS * qtw - 1) / (WARPS * qtw);
    dim3 grid(p.num_seq, kHeads * qblocks, num_splits);
    if (grid.y > 65535 || grid.z > 65535) return cudaErrorInvalidValue;
    attention_tc_kernel<KB, false><<<grid, WARPS * 32, smem, s>>>(p, q_tiles, num_splits, qtw, part_ml, part_o);
  }
  return cudaGetLastError();
}

}  // namespace

size_t attention_partial_bytes(int num_seq, int Lq, int max_splits) {
  return (size_t)num_seq * kHeads * max_splits * Lq * (kDh + 2) * sizeof(float);
}

// split-K when the query side alone cannot fill the machine
int attention_tc_splits(int num_seq, int Lq, int Lk, int num_sms) {
  const int q_tiles = (Lq + 15) / 16;
  const int ctas = num_seq * kHeads * ((q_tiles + WARPS - 1) / WARPS);
  const int chunks = (Lk + 63) / 64;
  int splits = 1;
  if (ctas < 2 * num_sms && chunks >= 8) {
    // split-K so that the grid fills whole waves of the 4-CTA/SM occupancy: minimise waves x chunks-per-split
    const int slots = 4 * num_sms;
    long long best = -1;
    const int smax = kAttnMaxSplits < chunks / 2 ? kAttnMaxSplits : chunks / 2;
    for (int sp = 1; sp <= smax; ++sp) {
      const long long waves = ((long long)ctas * sp + slots - 1) / slots;
      const long long cost = waves * ((chunks + sp - 1) / sp);
      if (best < 0 || cost < best) { best = cost; splits = sp; }
    }
  }
  return splits;
}

// per_warp: sequences are short and independent (time attention); otherwise the CTA shares K/V.
// part: scratch of attention_partial_bytes(num_seq, Lq, kAttnMaxSplits) bytes or null (then no split-K).
cudaError_t launch_attention_tc(const AttnParams& p, bool per_warp, float* part, int num_sms, cudaStream_t s) {
  if (p.num_seq <= 0 || p.Lq <= 0 || p.Lk <= 0) return cudaSuccess;
  if (per_warp) {
    if (p.Lk <= 16) return launch_variant<16, true>(p, 1, 1, nullptr, nullptr, s);
    if (p.Lk <= 32) return launch_variant<32, true>(p, 1, 1, nullptr, nullptr, s);
    return launch_variant<64, true>(p, 1, 1, nullptr, nullptr, s);
  }
  const int q_tiles = (p.Lq + 15) / 16;
  const int chunks = (p.Lk + 63) / 64;
  int splits = 1, slots = 1;
  if (p.gl) {   // grouped: the caller chose every entry's count with attention_tc_splits
    if (p.split_max > 1) {
      if (!part || !p.gsplit || !p.gslot) return cudaErrorInvalidValue;
      splits = p.split_max;
      slots = p.split_slots;
    }
  } else if (part != nullptr) {
    splits = slots = attention_tc_splits(p.num_seq, p.Lq, p.Lk, num_sms);
  }
  if (splits == 1) {
    // K/V of one chunk are staged once per CTA: amortise the conversion over several query tiles per warp while
    // still leaving >= 4 CTAs per SM
    int qtw = 1;
    if (chunks == 1) while (qtw < 8 && (long long)p.num_seq * kHeads * ((q_tiles + WARPS * 2 * qtw - 1) / (WARPS * 2 * qtw)) >= 4LL * num_sms) qtw *= 2;
    return launch_variant<64, false>(p, 1, qtw, nullptr, nullptr, s);
  }
  float* part_ml = part;
  float* part_o = part + (size_t)slots * (p.gl ? p.frames : p.num_seq) * kHeads * p.Lq * 2;
  cudaError_t e = launch_variant<64, false>(p, splits, 1, part_ml, part_o, s);
  if (e != cudaSuccess) return e;
  const int64_t rows = (int64_t)p.num_seq * kHeads * p.Lq;
  attention_combine_kernel<<<(unsigned)((rows + 3) / 4), 128, 0, s>>>(p, splits, part_ml, part_o);
  return cudaGetLastError();
}

}  // namespace ct3
