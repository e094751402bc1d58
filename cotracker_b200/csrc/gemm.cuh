// gemm.cuh -- interface of the split-bf16x3 linear-layer engine.
//
//   Y[M, N] = epilogue( X[M, K] * W[N, K]^T )      (nn.Linear; blocks.py:61-67, :375-377, cotracker.py:409-412)
//
// Operands are stored "split": X_split[M, 2*Kpad] = [hi(Kpad) | lo(Kpad)] bf16 with x = hi + lo,
// likewise W_split[N, 2*Kpad].  The tensor cores accumulate hi*hi + lo*hi + hi*lo in fp32 (registers),
// i.e. all first-order terms of the fp32 product (rel. error ~2^-17 per product, vs 2^-11 for TF32).
#pragma once
#include "common.cuh"

namespace ct3 {

struct GemmEpilogue {
  const float* bias = nullptr;      // [N]
  const float* row_bias = nullptr;  // [row_mod, N]; row r adds row_bias[(r % row_mod)]   (time-embedding fold)
  int row_mod = 1;
  // [M / row_mod] or null: row r adds row_bias[row_blk[r / row_mod] * row_mod + r % row_mod] instead (one bias block of
  // row_mod rows per track: the time embedding of the track's group, ct3_loop_shape.group_T)
  const int32_t* row_blk = nullptr;
  int act = 0;                      // 0 none | 1 GELU(erf) | 2 GELU(tanh)
  // fp32 output (optional): out_f32[r*ld_f32 + c] = v   or  += v  when residual
  float* out_f32 = nullptr;
  int64_t ld_f32 = 0;
  int residual = 0;
  // split bf16 output (optional): orow = r / row_group, ocol = (r % row_group) * N + c
  //   hi -> out_split[orow*ld_split + ocol],  lo -> out_split[orow*ld_split + lo_off + ocol]
  __nv_bfloat16* out_split = nullptr;
  int64_t ld_split = 0;
  int lo_off = 0;
  int row_group = 1;
};

struct GemmProblem {
  const __nv_bfloat16* x_split;  // [M, x_ld]: hi plane at column 0, lo plane (if any) at column Kpad
  const __nv_bfloat16* w_split;  // [N, 2*Kpad]
  int M, N, Kpad;                // N % 128 == 0, Kpad % 64 == 0
  // Tensor-core products per FLOP (precision switch, DESIGN.md section 2):
  //   3 : hi*hi + lo*hi + hi*lo   (both operands split; rel. error ~2^-17 bf16 / ~2^-22 fp16)
  //   2 : x_hi*w_hi + x_hi*w_lo   (activation rounded to its hi plane, weights exact to the split)
  //   1 : x_hi*w_hi
  int products = 3;
  int fp16 = 0;                  // operand planes hold IEEE fp16 (11-bit significand) instead of bf16 (8-bit)
  int64_t x_ld = 0;              // row pitch of x in elements; 0 = 2*Kpad.  Kpad for a single-plane (hi only) operand
  GemmEpilogue epi;
};

// cuTensorMapEncodeTiled through the runtime's driver entry point (no libcuda link dependency).
// dims/box innermost first; strides_bytes has rank-1 entries (innermost stride is the element size).
bool encode_tensor_map(CUtensorMap* m, CUtensorMapDataType dtype, int rank, const void* base, const uint64_t* dims,
                       const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle);

// The argument checks of gemm_launch: null if p can run, else what is wrong with it (shapes, pitches, overlapping
// hi/lo planes, alignment).
const char* gemm_check(const GemmProblem& p);
// 0 = wgmma path, 1 = SIMT verification path.  Returns cudaError_t as int (0 = ok); a problem gemm_check rejects
// returns cudaErrorInvalidValue with *err set, before any launch.
int gemm_launch(const GemmProblem& p, int impl, int num_sms, cudaStream_t stream, const char** err);

// Fused q|k|v projection + per-track time attention (gemm.cu, gemm_qkv_time_attn_kernel).
//   x_split [M, 2*Kpad] (LayerNorm output, rows track-major n*T + t, M % T == 0), w_heads [8*144, 2*Kpad] with the
//   rows of head h = [q_h | k_h | v_h], bias_heads [8*144] likewise; att_split[row*ld_split + h*48 + c] (hi) and
//   + lo_off (lo) = softmax(q k^T scale) v.   T <= 128.
//   track_len [M / T] or null: track i attends over its first track_len[i] frames only (every row of it, its padded
//   rows too).  With it T may exceed 128 when every track_len is <= 128: each track is then a tile of its own and only
//   its first 128 rows are written.  The kernel clamps a length to min(T, 128) so that no key is read outside its tile.
bool qkv_time_attn_supported(int T);
int gemm_qkv_time_attn_launch(const __nv_bfloat16* x_split, const __nv_bfloat16* w_heads, const float* bias_heads,
                              int M, int Kpad, int T, const int32_t* track_len, __nv_bfloat16* att_split,
                              int64_t ld_split, int lo_off, float scale, int num_sms, cudaStream_t stream,
                              const char** err);

}  // namespace ct3
