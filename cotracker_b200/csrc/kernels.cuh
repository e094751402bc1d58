// kernels.cuh -- launchers of the non-GEMM kernels of the update loop (definitions in *.cu).
#pragma once
#include "../../include/ct3_b200.h"
#include "common.cuh"

namespace ct3 {

// ---- prep.cu : per-clip preparation -------------------------------------------------------------
struct PyramidLayout {
  int64_t off[kL];  // float offset of each level inside the pyramid buffer
  int h[kL], w[kL];
  int64_t total;
};
PyramidLayout pyramid_layout(int T, int H4, int W4);
cudaError_t launch_prepare_pyramid(const float* fmaps, int T, int H4, int W4, float* pyr, cudaStream_t s);
cudaError_t launch_sample_support(const float* pyr, int T, int H4, int W4, const int32_t* qframes,
                                  const float* qcoords, int N, const uint8_t* acc_mask, float* support,
                                  cudaStream_t s);

// pools levels 1..3 from an already normalised channels-last level 0 living in `pyr`
cudaError_t launch_pyramid_pools(int T, int H4, int W4, float* pyr, cudaStream_t s);

// ---- ingest.cu : raw frames -> encoder input ------------------------------------------------------
// src [T,3,H,W] (element strides st, sc, sh, sw; dtype CT3_FRAMES_U8 | CT3_FRAMES_F32) -> out [T,3,oh,ow] fp32 contiguous
// = 2 * (bilinear(align_corners=True) / 255) - 1, bit-identical to the ATen expression (see ingest.cu)
cudaError_t launch_prepare_frames(const void* src, int dtype, int T, int H, int W, int64_t st, int64_t sc, int64_t sh,
                                  int64_t sw, int oh, int ow, float* out, cudaStream_t s);

// ---- finish.cu : the predictor's tail (arguments validated by ct3_finish_tracks) --------------------
// forward (+ optional backward, reversed-clip time) tracks [B,T,N,2] / visibility probabilities [B,T,N], queries
// [B,N,3] -> tracks [B,T,n_keep,2] fp32 and visibility [B,T,n_keep] uint8 (0 | 1), bit-identical to the ATen sequence
cudaError_t launch_finish_tracks(const float* fwd_tracks, const float* fwd_vis, const float* bwd_tracks,
                                 const float* bwd_vis, const float* queries, int B, int T, int N, int n_keep,
                                 float threshold, float scale_x, float scale_y, float* tracks, uint8_t* visibility,
                                 cudaStream_t s);

// ---- online.cu : per-window state of K streams (arguments validated by ct3_online_window_*) -------------------
// streams: the device copy of the K entries; max_elems: the largest per-stream element count (S * n or (ind + T) * n)
cudaError_t launch_online_window_begin(const ct3_online_stream* streams, int K, int64_t max_elems, int S, int step,
                                       float inv_stride, const int32_t* qframes, const float* qcoords, int N,
                                       uint8_t* valid, uint8_t* entering, int32_t* rel, float* coords_init,
                                       float* vis_init, float* conf_init, cudaStream_t s);
cudaError_t launch_online_window_end(const ct3_online_stream* streams, int K, int64_t max_elems, float stride,
                                     const float* coords, const float* vis, const float* conf, int N, float threshold,
                                     cudaStream_t s);

// ---- render.cu : the track visualiser on uint8 frames [T,H,W,3] (arguments validated by ct3_render_*) ----------
constexpr int kRenderMaxRadius = 255;   // largest point radius (int(linewidth * 2)) the footprint table holds
cudaError_t launch_render_prepare(const void* src, int dtype, int T, int H, int W, int64_t st, int64_t sc, int64_t sh,
                                  int64_t sw, int pad, int gray, uint8_t* out, cudaStream_t s);
// keys: T*H*W int32 scratch, any content on entry, all -1 on return
cudaError_t launch_render_tracks(uint8_t* frames, int T, int H, int W, const float* pts, const uint8_t* visible,
                                 const uint8_t* colors, const uint8_t* draw_mask, int N, int radius, int linewidth,
                                 int trail, int query_frame, const double* alphas, const double* diff, int* keys,
                                 cudaStream_t s);
// pts [T,N,2] fp32 -> colors [T,N,3] uint8 (flow_vis colours of the flow from query_frame); workspace: one u64
cudaError_t launch_render_flow_colors(const float* pts, int T, int N, int query_frame, uint8_t* colors, void* workspace,
                                      cudaStream_t s);

// ---- enc_tail.cu : conv2 -> InstanceNorm -> ReLU -> conv3 of the encoder on the GEMM engine --------
cudaError_t launch_im2col3x3_split(const float* in, int T, int C, int H, int W, int Kpad, __nv_bfloat16* out,
                                   cudaStream_t s);
// scratch: instnorm_scratch_bytes(T, C) bytes (fp64 partial sums of the two-stage reduction)
size_t instnorm_scratch_bytes(int T, int C);
cudaError_t launch_instnorm_stats(const float* y, int T, int HW, int C, float eps, float* stats, void* scratch,
                                  cudaStream_t s);
cudaError_t launch_instnorm_relu_split(const float* y, const float* stats, int64_t rows, int HW, int C,
                                       __nv_bfloat16* out, cudaStream_t s);
cudaError_t launch_l2norm_rows(const float* in, int64_t rows, float* out, cudaStream_t s);
cudaError_t launch_upsample_concat(const float* const src[4], const int c[4], const int h[4], const int w[4], int T,
                                   int H, int W, float* out, cudaStream_t s);

// ---- enc_front.cu : the CNN encoder's convolutions, channels-last, on the tensor cores --------------------
// conv1 7x7/2 pad 3 (3 -> 64), fp32 SIMT: frames [T,3,H,W] -> out [T,Ho,Wo,64] NHWC (+ bias)
cudaError_t launch_conv_stem(const float* frames, const float* w, const float* bias, int T, int H, int W, float* out,
                             cudaStream_t s);
// 3x3 stride-1 pad-1 implicit-GEMM convolution: x_split [T*H*W, 2*C] (hi C | lo C), w_split [Cout, 2*9*C] packed by
// launch_pack_conv (tap-major K), out fp32 NHWC [T,H,W,Cout] (+ bias).  C, Cout multiples of 64.
cudaError_t launch_conv3x3_tc(const __nv_bfloat16* x_split, const __nv_bfloat16* w_split, const float* bias, int T,
                              int H, int W, int C, int Cout, float* out, int num_sms, cudaStream_t s);
// [Cout, Cin, taps] fp32 -> split [Cout_pad, 2*taps*Cp] with K = tap*Cp + c, zero padded
cudaError_t launch_pack_conv(const float* w, int Cout, int Cin, int taps, int Cp, int Cout_pad, __nv_bfloat16* out,
                             cudaStream_t s);
// stride-2 gather (taps 9: 3x3 pad 1; taps 1: 1x1) of a split NHWC activation into GEMM rows [T*Ho*Wo, 2*taps*C]
cudaError_t launch_gather_s2(const __nv_bfloat16* x_split, int T, int H, int W, int C, int taps, __nv_bfloat16* out,
                             cudaStream_t s);
// InstanceNorm + ReLU (+ residual: mode 1 x fp32; mode 2 x = 1x1/2 conv output normalised with stats_d) on NHWC rows
cudaError_t launch_norm_act(const float* y, const float* stats, const float* x, const float* stats_d, int mode,
                            int64_t rows, int HW, int C, float* out_f32, __nv_bfloat16* out_split, cudaStream_t s);
// bilinear (align_corners) resize of 4 NHWC fp32 sources (c channels used, cs channel stride) + concat -> split [rows, 2*Cp]
cudaError_t launch_upsample_concat_split(const float* const src[4], const int c[4], const int cs[4], const int h[4],
                                         const int w[4], int T, int Cp, int H, int W, __nv_bfloat16* out, cudaStream_t s);

// ---- corr.cu : correlation sampling ---------------------------------------------------------------
// Frame map of a ct3_update_loop pass: at time step t, track n of group g reads pyramid frame frames[g*T + t] (an index
// into the T_pyr frames of the pyramid).  frames == nullptr: frame t.  goff: [G+1] first track of every group (nullptr
// when G == 1).  Every correlation kernel works on units of ONE track, so the lookup is per (track, t): no tile or TMA
// box ever spans two tracks' frames.  n0: the global index of the launch's first track (a track slab of
// ct3_loop_shape.slab_tracks); the group lookup is by global track.
struct FrameMap {
  const int32_t* frames = nullptr;
  const int32_t* goff = nullptr;
  int G = 1;
  int n0 = 0;
};
// the T-entry frame row of track n of the launch (nullptr: identity)
__device__ __forceinline__ const int32_t* frame_row(const FrameMap& m, int n, int T) {
  if (!m.frames) return nullptr;
  int g = 0;
  if (m.goff) {   // largest g with goff[g] <= n0 + n
    n += m.n0;
    int hi = m.G - 1;
    while (g < hi) {
      const int mid = (g + hi + 1) >> 1;
      if (__ldg(m.goff + mid) <= n) g = mid; else hi = mid - 1;
    }
  }
  return m.frames + (int64_t)g * T;
}
__device__ __forceinline__ int map_frame(const int32_t* row, int t) { return row ? __ldg(row + t) : t; }

// vol_split [N*T*4, 2*kVolPad] bf16, row (n*T+t)*4+level; pyr holds T_pyr frames (T_pyr = T and fm = {} unless a frame
// map is given)
// impl: 0 tensor cores (correlate-then-interpolate when pyr_split is given and every level is >= 8x8: corr_tc3.cu for
//         modes 2 / 1, corr_tc2.cu for mode 3; else corr_tc.cu),
//       1 exact-fp32 SIMT, 2 corr_tc.cu always
// mode / vol16 apply to the correlate-then-interpolate path only (corr_uses_patch_kernel): products per correlation
// FLOP (3|2|1; pyr_split must have been made with the same mode) and a single-fp16-plane volume [N*T*4, kVolPad]
// instead of the split one; the other kernels always compute in fp32 / bf16x3 and write the split volume.
// Track range: the launch covers tracks [n0, n0 + count) of the N-track state and support (N stays their pitch) and
// writes their volume rows from row 0 of vol_split (a track slab of a ct3_update_loop pass; n0 = 0, count = N: all).
// The dispatcher moves support / track_valid / coords to track n0 and sets fm.n0; the kernels below it see `count`
// tracks at pitch N.
bool corr_uses_patch_kernel(int impl, bool have_pyr_split, int T, int H4, int W4);
cudaError_t launch_corr_sample(const float* pyr, const __nv_bfloat16* pyr_split, int H4, int W4, const float* support,
                               const uint8_t* track_valid, const float* coords, int T, int N, int n0, int count,
                               __nv_bfloat16* vol_split, int impl, int mode, int vol16, int num_sms, cudaStream_t s,
                               int T_pyr, const FrameMap& fm);

cudaError_t launch_corr_sample_tc(const float* pyr, int H4, int W4, const float* support,
                                  const uint8_t* track_valid, const float* coords, int T, int N, int count,
                                  __nv_bfloat16* vol_split, int num_sms, cudaStream_t s, int T_pyr, const FrameMap& fm);

// corr_tc2.cu: correlate-then-interpolate on a split-bf16 copy of the pyramid (mode 3)
//   pyr_split: per level at bf16 offset 2*off[l]: [plane hi|lo][T][H][W][128]   (same bytes as the fp32 pyramid)
bool corr_patch_supported(int T, int H4, int W4);
//   mode 3: [plane hi|lo][T][H][W][128] bf16;  mode 1/2: one fp16 plane [T][H][W][128] at the same level offset
cudaError_t launch_split_pyramid(const float* pyr, int T, int H4, int W4, __nv_bfloat16* pyr_split, int mode,
                                 cudaStream_t s);
cudaError_t launch_corr_patch_tc(const __nv_bfloat16* pyr_split, int H4, int W4, const float* support,
                                 const uint8_t* track_valid, const float* coords, int T, int N, int count,
                                 __nv_bfloat16* vol_split, int vol16, int num_sms, cudaStream_t s, int T_pyr,
                                 const FrameMap& fm);

// corr_tc3.cu: the production kernel -- same algorithm with the MMA transposed (supports = M side), one fp16 texel
// plane (pyr_split made with mode 1 or 2), supports split fp16 (mode 2) or one fp16 plane (one_product, mode 1)
cudaError_t launch_corr_patch_t(const __nv_bfloat16* pyr_half, int H4, int W4, const float* support,
                                const uint8_t* track_valid, const float* coords, int T, int N, int count,
                                __nv_bfloat16* vol, int vol16, int one_product, int num_sms, cudaStream_t s, int T_pyr,
                                const FrameMap& fm);

// ---- tokens.cu : elementwise / row-wise pieces of the transformer ---------------------------------
cudaError_t launch_layernorm_split(const float* x, int rows, const float* gamma, const float* beta, float eps,
                                   __nv_bfloat16* out_split, cudaStream_t s);
// the X rows of tracks [n0, n0 + count) of the [T, N] state into x_split from row 0; track_len [N] or null: track n's
// forward relative motion ends at its own last frame track_len[n] - 1 (ct3_loop_shape.group_T)
cudaError_t launch_build_x_small(const float* coords, const float* vis, const float* conf, int T, int N, int n0,
                                 int count, const int32_t* track_len, __nv_bfloat16* x_split, cudaStream_t s);
// one copy of the kV virtual tokens per group: rows (N + kV*g + i)*T + t, g < G
cudaError_t launch_init_virtual(float* tokens, const float* virt, int T, int N, int G, cudaStream_t s);
// host int32 array -> device, stream-ordered (kernel arguments carry the values: src may be freed on return)
cudaError_t launch_upload_i32(int32_t* dst, const int32_t* src_host, int n, cudaStream_t s);
// delta_out == nullptr: in-place state update; else write delta [N,T,4] and leave the state alone
cudaError_t launch_heads(const float* tokens, const float* w4, const float* b4, float* coords, float* vis,
                         float* conf, float* delta_out, int T, int N, cudaStream_t s);
cudaError_t launch_row_bias(const float* time_emb, const float* w_in, int T, float* out, cudaStream_t s);
// fp32 [rows,K] -> split [rows, 2*Kpad]; perm_x: apply the X column permutation (x_src_col)
// fp16 != 0: the planes hold IEEE fp16 (hi = fp16(x), lo = fp16(x - hi)) instead of bf16
cudaError_t launch_split_rows(const float* x, int rows, int K, int Kpad, int perm_x, __nv_bfloat16* out,
                              int64_t dst_row_off, cudaStream_t s, int fp16 = 0);

// ---- attention.cu -------------------------------------------------------------------------------
struct AttnParams {
  const float* q;  int64_t q_ld;  int q_col;
  const float* kv; int64_t kv_ld; int k_col, v_col;
  __nv_bfloat16* out; int64_t out_ld; int lo_off;
  int num_seq, Lq, Lk;
  int64_t q_seq_stride, q_tok_stride;  // q/out row = s*q_seq_stride + i*q_tok_stride
  int64_t k_seq_stride, k_tok_stride;  // k/v row  = s*k_seq_stride + j*k_tok_stride
  float scale;
  // Grouped space attention (ct3_loop_shape.G > 1): the tracks form contiguous groups, each with its own kV virtual
  // tokens.  gl == nullptr: one group, rows as above.  Otherwise sequence s = (entry s / frames, frame s % frames),
  // entry e covers group gl[e], and Lq / Lk are upper bounds.  A side with grp_stride != 0 is virtual (group g starts
  // at row g * grp_stride, kV tokens); a side with grp_stride == 0 holds points (group g = tracks [goff[g], goff[g+1])).
  const int32_t* gl;
  const int32_t* goff;     // [G+1] first track of every group
  const int32_t* gsplit;   // attention_tc.cu: [entries] split-K count (null: 1)
  const int32_t* gslot;    //                  [entries] first partial slot of a split entry
  int frames, split_max, split_slots;   // split_max: largest gsplit entry; split_slots: sum of gsplit over split entries
  int64_t q_grp_stride, k_grp_stride;
  // attention_p2v.cu: [tiles] (group, first track) of each 128-track tile; Lq = all tracks, Lk = kV * groups
  const int32_t* gtile;
  int tiles;
  // Ungrouped calls only: [num_seq] key counts or null (all Lk).  Sequence s attends over its first seq_len[s] <= Lk
  // keys; every one of its Lq queries is computed (time attention of a pass with ct3_loop_shape.group_T).
  const int32_t* seq_len;
};
// rows and lengths of sequence s (grouped or not)
struct SeqRows { int64_t q0, k0; int Lq, Lk, e, t; };
__device__ __forceinline__ SeqRows seq_rows(const AttnParams& p, int s) {
  SeqRows r;
  if (!p.gl) {
    r.q0 = (int64_t)s * p.q_seq_stride; r.k0 = (int64_t)s * p.k_seq_stride;
    r.Lq = p.Lq; r.Lk = p.seq_len ? p.seq_len[s] : p.Lk; r.e = 0; r.t = s;
    return r;
  }
  r.e = s / p.frames;
  r.t = s - r.e * p.frames;
  const int g = p.gl[r.e], n0 = p.goff[g], n = p.goff[g + 1] - n0;
  r.q0 = (int64_t)r.t * p.q_seq_stride + (p.q_grp_stride ? (int64_t)g * p.q_grp_stride : (int64_t)n0 * p.q_tok_stride);
  r.k0 = (int64_t)r.t * p.k_seq_stride + (p.k_grp_stride ? (int64_t)g * p.k_grp_stride : (int64_t)n0 * p.k_tok_stride);
  r.Lq = p.q_grp_stride ? kV : n;
  r.Lk = p.k_grp_stride ? kV : n;
  return r;
}
cudaError_t launch_attention(const AttnParams& p, cudaStream_t s);   // exact-fp32 SIMT (verification)


// ---- attention_tc.cu : tensor-core (mma.sync split-bf16x3) production path ------------------------
constexpr int kAttnMaxSplits = 32;
size_t attention_partial_bytes(int num_seq, int Lq, int max_splits);
// split-K count launch_attention_tc chooses for an ungrouped shared-K/V launch of this shape
int attention_tc_splits(int num_seq, int Lq, int Lk, int num_sms);
cudaError_t launch_attention_tc(const AttnParams& p, bool per_warp, float* part, int num_sms, cudaStream_t s);

// ---- attention_p2v.cu : point <- virtual cross attention (Lk == 64 keys) on wgmma --------------------------------------
bool attention_p2v_supported(const AttnParams& p);
cudaError_t launch_attention_p2v(const AttnParams& p, cudaStream_t s);

}  // namespace ct3
