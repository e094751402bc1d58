// attention.cu -- multi-head attention core  softmax(q k^T * 48^-1/2) v  (Attention.forward, blocks.py:379-398)
// for the four attention patterns of EfficientUpdateFormer (cotracker.py:493-523), expressed through one
// strided-row kernel:
//     time    : sequence = track,  Lq = Lk = T            rows  s*T + i
//     v <- p  : sequence = frame,  Lq = 64, Lk = N        q rows i*T + s (virtual), k rows j*T + s (points)
//     v self  : sequence = frame,  Lq = Lk = 64
//     p <- v  : sequence = frame,  Lq = N,  Lk = 64
// In a grouped call the space patterns run per (group, frame) sequence over that group's rows (seq_rows).
// One physical token layout (track-major) serves both orders: the reference's two permute().contiguous()
// copies per space block (cotracker.py:504,520) disappear into the row strides.
// Attention proper is ~2 % of the block FLOPs (SURVEY.md 8a); it runs exact fp32 flash-style (online softmax)
// on CUDA cores; the projections around it are the tensor-core GEMMs.
#include "kernels.cuh"

namespace ct3 {
namespace {

constexpr int WARPS = 8;
constexpr int KC = 64;         // keys per shared-memory chunk
constexpr int KLD = kDh + 1;   // 49: conflict-free for lane = key and lane = channel access

template <int RQ>
__global__ void __launch_bounds__(WARPS * 32)
attention_kernel(AttnParams p) {
  __shared__ float Ks[KC * KLD];
  __shared__ float Vs[KC * KLD];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y, s = blockIdx.x;
  const SeqRows sr = seq_rows(p, s);
  const int Lq = sr.Lq, Lk = sr.Lk;
  if ((int)blockIdx.z * WARPS * RQ >= Lq) return;   // grouped: this sequence is shorter than the longest one
  const int q0 = (blockIdx.z * WARPS + warp) * RQ;

  float q[RQ][kDh];
  float m[RQ], l[RQ], o0[RQ], o1[RQ];
#pragma unroll
  for (int r = 0; r < RQ; ++r) {
    const int qi = min(q0 + r, Lq - 1);
    const float4* qp = reinterpret_cast<const float4*>(
        p.q + (sr.q0 + (int64_t)qi * p.q_tok_stride) * p.q_ld + p.q_col + h * kDh);
#pragma unroll
    for (int d4 = 0; d4 < kDh / 4; ++d4) {
      const float4 v = __ldg(qp + d4);
      q[r][4 * d4 + 0] = v.x; q[r][4 * d4 + 1] = v.y; q[r][4 * d4 + 2] = v.z; q[r][4 * d4 + 3] = v.w;
    }
    m[r] = -INFINITY; l[r] = 0.f; o0[r] = 0.f; o1[r] = 0.f;
  }

  for (int kc0 = 0; kc0 < Lk; kc0 += KC) {
    // stage K and V rows of this chunk (zero-filled past Lk)
    for (int idx = threadIdx.x; idx < KC * (kDh / 4); idx += WARPS * 32) {
      const int j = idx / (kDh / 4), d4 = idx % (kDh / 4);
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (kc0 + j < Lk) {
        const float* base = p.kv + (sr.k0 + (int64_t)(kc0 + j) * p.k_tok_stride) * p.kv_ld + h * kDh;
        kv = __ldg(reinterpret_cast<const float4*>(base + p.k_col) + d4);
        vv = __ldg(reinterpret_cast<const float4*>(base + p.v_col) + d4);
      }
      float* kd = Ks + j * KLD + 4 * d4;
      float* vd = Vs + j * KLD + 4 * d4;
      kd[0] = kv.x; kd[1] = kv.y; kd[2] = kv.z; kd[3] = kv.w;
      vd[0] = vv.x; vd[1] = vv.y; vd[2] = vv.z; vd[3] = vv.w;
    }
    __syncthreads();
#pragma unroll 1
    for (int sub = 0; sub < KC / 32; ++sub) {
      if (kc0 + sub * 32 >= Lk) break;  // warp-uniform
      const int j = sub * 32 + lane;
      const bool valid = kc0 + j < Lk;
      float sc[RQ];
#pragma unroll
      for (int r = 0; r < RQ; ++r) sc[r] = 0.f;
      const float* kr = Ks + j * KLD;
#pragma unroll
      for (int d = 0; d < kDh; ++d) {
        const float kd = kr[d];
#pragma unroll
        for (int r = 0; r < RQ; ++r) sc[r] = fmaf(q[r][d], kd, sc[r]);
      }
      float pr[RQ];
#pragma unroll
      for (int r = 0; r < RQ; ++r) {
        const float sv = valid ? sc[r] * p.scale : -INFINITY;
        const float mnew = fmaxf(m[r], warp_max(sv));   // finite: at least one valid key in this sub-chunk
        pr[r] = valid ? expf(sv - mnew) : 0.f;
        const float corr = expf(m[r] - mnew);           // exp(-inf) = 0 on the first chunk
        l[r] = l[r] * corr + warp_sum(pr[r]);
        o0[r] *= corr;
        o1[r] *= corr;
        m[r] = mnew;
      }
      const float* vb = Vs + (sub * 32) * KLD;
#pragma unroll 8
      for (int jj = 0; jj < 32; ++jj) {
        const float v0 = vb[jj * KLD + lane];
        const float v1 = lane < kDh - 32 ? vb[jj * KLD + 32 + lane] : 0.f;
#pragma unroll
        for (int r = 0; r < RQ; ++r) {
          const float pj = __shfl_sync(0xffffffffu, pr[r], jj);
          o0[r] = fmaf(pj, v0, o0[r]);
          o1[r] = fmaf(pj, v1, o1[r]);
        }
      }
    }
    __syncthreads();
  }

#pragma unroll
  for (int r = 0; r < RQ; ++r) {
    const int qi = q0 + r;
    if (qi >= Lq) continue;
    const float inv = 1.0f / l[r];
    __nv_bfloat16* orow = p.out + (sr.q0 + (int64_t)qi * p.q_tok_stride) * p.out_ld + h * kDh;
    const bf16pair a = split_bf16(o0[r] * inv);
    orow[lane] = a.hi;
    orow[p.lo_off + lane] = a.lo;
    if (lane < kDh - 32) {
      const bf16pair b = split_bf16(o1[r] * inv);
      orow[32 + lane] = b.hi;
      orow[p.lo_off + 32 + lane] = b.lo;
    }
  }
}

}  // namespace

cudaError_t launch_attention(const AttnParams& p, cudaStream_t s) {
  if (p.num_seq <= 0 || p.Lq <= 0 || p.Lk <= 0) return cudaSuccess;
  constexpr int RQ = 2;
  dim3 grid(p.num_seq, kHeads, (p.Lq + WARPS * RQ - 1) / (WARPS * RQ));
  if (grid.z > 65535) return cudaErrorInvalidValue;
  attention_kernel<RQ><<<grid, WARPS * 32, 0, s>>>(p);
  return cudaGetLastError();
}

}  // namespace ct3
