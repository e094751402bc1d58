/*
 * ct3_b200.h -- C ABI of libct3_b200.so: the CoTracker3 iterative update loop
 * (correlation sampling + correlation MLP + EfficientUpdateFormer + delta heads)
 * as hand-written sm_90a CUDA.
 *
 * This is the drop-in boundary for the reference's inference hot path
 * (citations are file:line inside facebookresearch/co-tracker):
 *   cotracker/models/core/cotracker/cotracker3_offline.py:139-216   (offline loop body)
 *   cotracker/models/core/cotracker/cotracker3_online.py:187-263    (forward_window loop body)
 * and the per-clip preparation either side of it
 *   cotracker3_offline.py:92-127  (L2-normalise, avg-pool pyramid, support sampling).
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless the
 *     name ends in _host; the caller (PyTorch) owns every allocation, the library
 *     never allocates persistent device memory (scratch = caller workspace);
 *   - every entry point returns 0 on success, a negative CT3_E* code otherwise,
 *     never throws / exits; ct3_last_error() returns a thread-local message;
 *   - all work is enqueued on the given cudaStream_t and is asynchronous w.r.t.
 *     the host; the update loop has no batch dimension (cotracker3_offline.py:135,141): a batch of clips is
 *     more query groups of one ct3_update_loop pass with a frame map, each reading its own frames of one pyramid.
 *
 * Symbols (all extern "C"):  see the declarations below; tests/test_host_logic.py checks
 * that the built library exports each of them.
 */
#ifndef CT3_B200_H_
#define CT3_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* ct3_stream_t; /* == cudaStream_t */

enum {
  CT3_OK = 0,
  CT3_EINVAL = -1,   /* bad argument (shape, null pointer, alignment)          */
  CT3_ECUDA = -2,    /* a CUDA runtime/driver call failed (see ct3_last_error) */
  CT3_ENOSPC = -3    /* workspace / packed buffer too small                    */
};

/* Model constants fixed by the reference architecture
 * (cotracker3_online.py:43-92, cotracker.py:392-462). */
enum {
  CT3_LATENT = 128,     /* feature channels D                                  */
  CT3_LEVELS = 4,       /* corr_levels                                         */
  CT3_RADIUS = 3,       /* corr_radius -> 7x7 = 49 samples                     */
  CT3_P = 49,
  CT3_VOL = 2401,       /* 49*49 correlation volume per (t,n,level)            */
  CT3_VOL_PAD = 2432,   /* padded to a multiple of 64 for the tensor-core GEMM */
  CT3_HID = 384,        /* transformer width C                                 */
  CT3_HEADS = 8,
  CT3_DHEAD = 48,
  CT3_VIRT = 64,        /* virtual tracks                                      */
  CT3_XDIM = 1110,      /* transformer input width                             */
  CT3_XDIM_PAD = 1152,
  CT3_DEPTH = 3         /* time_depth == space_depth                           */
};

/* Order of the fp32 tensors handed to ct3_pack_weights (names are the
 * state-dict keys of the reference, SURVEY.md Appendix B).  Per transformer
 * layer i in [0,3) the block tensors follow in the order listed by
 * ct3_weight_name(). */
int ct3_num_weight_tensors(void);                 /* how many pointers ct3_pack_weights expects     */
const char* ct3_weight_name(int index);           /* state-dict key of tensor #index (NULL if OOR)  */

int ct3_version(void);
const char* ct3_last_error(void);

/* Debug/verification options ("gemm", "corr", "attn": 0 = tensor-core path (default),
 * 1 = SIMT fp32 verification kernel used by the tests to cross-check; "corr" = 2 forces the
 * sample-then-correlate tensor-core kernel that otherwise only serves pyramids with a level below 8x8).
 * "fuse" (time blocks, T <= 128): 1 = q|k|v projection and time attention in one kernel (default), 0 = separate
 * projection and attention kernels, which T > 128 always runs and the tests use as the cross-check. */
int ct3_set_option(const char* name, int value);
int ct3_get_option(const char* name, int* value);
/* Precision switches of the correlation branch ("prec.corr", "prec.fc1": tensor-core products per FLOP, 3 | 2 | 1;
 * DESIGN.md section 2).  Options and the live profiler are per HOST THREAD (thread_local), values are range-checked.
 * ct3_precision_info reports what actually runs for a (T, H4, W4) problem under the calling thread's options:
 * products of the 49x128x49 correlation contraction (cotracker3_offline.py:148-156), of corr_mlp.fc1
 * (blocks.py:61), and the bytes per element of the correlation volume (4 = split bf16 hi|lo, 2 = one fp16 plane). */
int ct3_precision_info(int T, int H4, int W4, int* corr_products, int* fc1_products, int* volume_bytes_per_element);
/* 1 when ct3_corr_sample / the update loop emit volume rows support-major (element k*49 + (a*7+b): corr_tc3.cu, the
 * default kernel) instead of the reference's sample-major (a*7+b)*49 + k (cotracker3_offline.py:148-156); the matching
 * column permutation of corr_mlp.fc1 is applied at pack time, so this only matters to callers of the stage API. */
int ct3_volume_is_support_major(int T, int H4, int W4, int* flag);

/* ---- one-time weight packing ------------------------------------------------
 * Replaces the nn.Module parameter storage read by cotracker3_online.py:73-92.
 * Splits every Linear weight into bf16 hi/lo planes ([out, 2*Kpad], K padded to
 * a multiple of 64), concatenates to_q|to_kv for self-attention blocks, permutes
 * the input_transform columns to the X layout documented in DESIGN.md. */
int ct3_packed_weights_bytes(size_t* out_bytes);
int ct3_pack_weights(const float* const* tensors_host_array_of_device_ptrs, int n_tensors,
                     void* packed, size_t packed_bytes, ct3_stream_t stream);

/* ---- raw frames -> encoder input -------------------------------------------
 * ct3_prepare_frames: the predictors' resize + normalisation (predictor.py:60-64, cotracker3_offline.py:63) in one
 * kernel.  src: T frames [T,3,H,W] of element type `dtype` (CT3_FRAMES_*) at arbitrary int64 ELEMENT strides
 * (stride_t, stride_c, stride_h, stride_w), so a channels-last [T,H,W,3] decoder buffer is read in place.
 * out: [T,3,out_h,out_w] fp32 contiguous, bit-identical to
 *     2 * (F.interpolate(src.float(), (out_h, out_w), mode="bilinear", align_corners=True) / 255) - 1
 * as PyTorch evaluates it on the GPU.  Null pointers, T/H/W/out_h/out_w < 1, an unknown dtype or a stride extent
 * (sum of |stride| * (size - 1), in bytes) or output size beyond int64, or an output plane out_h * out_w above
 * INT32_MAX pixels return CT3_EINVAL before any launch. */
enum { CT3_FRAMES_U8 = 0, CT3_FRAMES_F32 = 1 };
int ct3_prepare_frames(const void* src, int dtype, int T, int H, int W, int64_t stride_t, int64_t stride_c,
                       int64_t stride_h, int64_t stride_w, int out_h, int out_w, float* out, ct3_stream_t stream);

/* ---- the predictor's tail ---------------------------------------------------
 * ct3_finish_tracks: what CoTrackerPredictor does with the model's output (predictor.py:161-209), for B clips in one
 * kernel.  fwd_tracks [B,T,N,2] fp32 at model resolution and fwd_vis [B,T,N] fp32 visibility probabilities of the
 * forward pass; bwd_tracks / bwd_vis: the same of the pass on the clip played backwards, in reversed-clip time (frame
 * T-1-t is read for frame t), or both NULL; queries [B,N,3] fp32 (t, x, y) at model resolution.  Output element
 * (b, t, i), i < n_keep (the N - n_keep trailing tracks, the support grid, are dropped):
 *   the backward pass where (float)t < queries[b,i,0] and it is given, the forward pass elsewhere;
 *   visibility = probability > threshold;
 *   at t == (int64)queries[b,i,0] the track is the query point and visible (a query frame outside [0,T) pins nothing);
 *   tracks * (scale_x, scale_y), one fp32 multiply each.
 * tracks [B,T,n_keep,2] fp32, visibility [B,T,n_keep] uint8 (0 | 1), both contiguous and distinct from the inputs;
 * bit-identical to the torch expression.  Null pointers, one of the backward pair without the other, B/T/N < 1, n_keep
 * outside [1,N], track pointers not 8-byte aligned or more than 2^31 * 256 elements return CT3_EINVAL before any
 * launch. */
int ct3_finish_tracks(const float* fwd_tracks, const float* fwd_vis, const float* bwd_tracks, const float* bwd_vis,
                      const float* queries, int B, int T, int N, int n_keep, float threshold, float scale_x,
                      float scale_y, float* tracks, uint8_t* visibility, ct3_stream_t stream);

/* ---- streaming windows (cotracker3_online.py:457-541, predictor.py:276-309) ------------------------------------
 * One update-loop pass of the online model advances K streams by one window each.  Stream k holds tracks
 * [first, first + n) of the pass (streams follow each other: first_0 = 0, first_{k+1} = first_k + n_k, sum n_k = N),
 * its window starts at frame `ind` of the stream, its chunk has T real frames (window frames T..S-1 are padding) and
 * its window is pyramid frames [frame0, frame0 + S) of the pass.  Its history (coords * stride at model resolution,
 * visibility and confidence logits) has `len` frames written, `cap` frames allocated.  With ring = 0, frame f, track j
 * is at row f (element f * n + j) and len <= cap.  With ring = 1 the history is a ring: frame f is at row f mod cap,
 * len may exceed cap and only the last cap frames written, [len - cap, len), are held; a stream then runs in memory
 * that does not grow with its length.  window_end's output covers stream frames [out_first, ind + T).
 * `streams_host` is a HOST array of K entries; the library copies it into `workspace` (at least
 * K * sizeof(ct3_online_stream) bytes, 16-byte aligned) on `stream`, so the host array may be reused on return.
 * An entry whose fields after scale_y are zero is a plain history with an output of every frame. */
typedef struct {
  float* coords;          /* history [cap, n, 2] fp32                                                           */
  float* vis;             /* history [cap, n] fp32                                                              */
  float* conf;            /* history [cap, n] fp32                                                              */
  int64_t cap;            /* frames the history buffers hold                                                    */
  int64_t len;            /* history frames written before the window                                           */
  float* tracks;          /* window_end: predictor output [ind + T - out_first, n_keep, 2] fp32, or NULL         */
  uint8_t* visibility;    /* window_end: predictor output [ind + T - out_first, n_keep] uint8 (0 | 1)            */
  int32_t ind, T, n, first, frame0;
  int32_t n_keep;         /* window_end: the first n_keep tracks are output (the trailing support grid is dropped) */
  float scale_x, scale_y; /* window_end: output tracks = history * (scale_x, scale_y), one fp32 multiply each     */
  int64_t out_first;      /* window_end: the first stream frame of the output (0: every frame so far)           */
  int32_t ring;           /* 0: frame f at history row f; 1: frame f at row f mod cap                          */
  int32_t pad;            /* keeps the struct a multiple of 8 bytes; set to 0                                    */
} ct3_online_stream;
/* ct3_online_window_begin: the per-window state the update loop starts from, bit-identical to the torch expressions
 * (qf = qframes[i], the query frame in stream time; overlap = S - step):
 *   valid[i] = qf < ind + S;   entering[i] = left <= qf < ind + S with left = 0 at ind == 0, else ind + step;
 *   rel[i] = clamp(qf - ind, 0, S - 1) + frame0 (the frame sample_support reads the query's features from);
 *   for t in [0, S): where ind > 0 and qf < ind + overlap, the warm start from the history frame
 *   r = ind + min(t, overlap - 1): coords_init[t,i] = coords[r,j] * (1 / stride), vis_init / conf_init = vis / conf
 *   [r,j]; elsewhere coords_init[t,i] = qcoords[i], vis_init = conf_init = 0.
 * qframes [N] int32, qcoords [N,2] fp32 (feature-grid units); valid, entering [N] uint8, rel [N] int32,
 * coords_init [S,N,2], vis_init, conf_init [S,N] fp32.  Null pointers, K outside [1, 65535], S < 2, step outside
 * [1, S), stride < 1, a stream whose tracks do not tile [0, N) in order, T outside [1, S], ind < 0 or ind + S > 2^30,
 * frame0 + S > T_pyr, or (ind > 0) a null history or len < ind + overlap return CT3_EINVAL, a small workspace
 * CT3_ENOSPC, before any launch.  So do, with ring = 0, cap < len; with ring = 1, cap < S, ring outside {0, 1}, or
 * (ind > 0) an overlap frame the ring no longer holds (ind < len - cap).  Query frames beyond +-2^30 compare as
 * +-2^30. */
int ct3_online_window_begin(const ct3_online_stream* streams_host, int K, int S, int step, int stride, int T_pyr,
                            const int32_t* qframes, const float* qcoords, int N, uint8_t* valid, uint8_t* entering,
                            int32_t* rel, float* coords_init, float* vis_init, float* conf_init, void* workspace,
                            size_t workspace_bytes, ct3_stream_t stream);
/* ct3_online_window_end: the loop's result into the histories and the predictor's output, bit-identical to
 *   history[ind + t, j] = (coords[t, first + j] * stride, vis[...], conf[...])   for t < T  (frames ind + T.. untouched)
 *   tracks[f - out_first, j] = history_coords[f, j] * (scale_x, scale_y),
 *   visibility[f - out_first, j] = sigmoid(history_vis[f, j]) * sigmoid(history_conf[f, j]) > threshold
 *     for out_first <= f < ind + T, j < n_keep
 * with sigmoid(x) = 1 / (1 + expf(-x)) in fp32, as torch.sigmoid evaluates it, and history frames addressed through
 * the ring when ring = 1.  coords [S,N,2], vis, conf [S,N] fp32: the update loop's state (feature-grid units, logits).
 * The work is O((ind + T - out_first) * n) per stream with an output and O(T * n) without.  The same argument checks
 * as window_begin (without T_pyr and the overlap), plus len < ind, a stream with `tracks` whose visibility is NULL,
 * n_keep is outside [1, n] or out_first is outside [0, ind + T), and with ring = 0 cap < ind + T.  With ring = 1 also
 * (`tracks` set) an output frame before the window that the ring no longer holds (out_first < min(ind, len - cap)),
 * or an output longer than the ring (ind + T - out_first > cap: a frame the launch reads would share its row with one
 * it writes). */
int ct3_online_window_end(const ct3_online_stream* streams_host, int K, int S, int stride, const float* coords,
                          const float* vis, const float* conf, int N, float threshold, void* workspace,
                          size_t workspace_bytes, ct3_stream_t stream);

/* ---- track visualiser (reference cotracker/utils/visualizer.py) ---------------
 * Frames are uint8 [T,H,W,3] contiguous on the device, drawn in place; every result is bit-identical to the reference's
 * PIL drawing (footprint rules: render.cu).  T <= 65535.
 *
 * ct3_render_prepare: visualize()'s F.pad(video, (pad,)*4, value=255), optional transforms.Grayscale() repeated to 3
 * channels (float32 arithmetic, no contraction) and .byte() (truncation) in one kernel.  src: T frames [T,3,H,W] of
 * element type `dtype` (CT3_FRAMES_*) at any int64 element strides.  out: [T, H+2*pad, W+2*pad, 3] uint8.
 * Null pointers, T/H/W < 1, pad < 0, grayscale not 0|1, an unknown dtype, a stride extent beyond int64 bytes or an
 * output plane above INT32_MAX pixels return CT3_EINVAL before any launch. */
int ct3_render_prepare(const void* src, int dtype, int T, int H, int W, int64_t stride_t, int64_t stride_c,
                       int64_t stride_h, int64_t stride_w, int pad, int grayscale, uint8_t* out, ct3_stream_t stream);
/* Scratch of ct3_render_tracks: one int32 draw-order key per pixel.  CT3_EINVAL unless T, H, W, N >= 1, trail >= -1,
 * H*W <= INT32_MAX and T*N <= INT32_MAX. */
int ct3_render_workspace_bytes(int T, int H, int W, int N, int trail, size_t* out_bytes);
/* ct3_render_tracks: draw_tracks_on_video's trails and points (visualizer.py:238-288) on `frames`.
 *   pts        [T,N,2] fp32 (x, y) frame pixel coordinates, truncated toward zero as tracks.long() does; a point is
 *              drawn when both truncated coordinates are non-zero.  Coordinates that are not finite or whose magnitude
 *              is at least 2^30 draw nothing.
 *   visible    [T,N] uint8 or NULL (all visible): a visible point is a filled disc, a hidden one its outline only
 *   colors     [T,N,3] uint8: colour of track i at frame t (trail segments use the colour of their start frame)
 *   draw_mask  [N] uint8 or NULL: only tracks with a non-zero entry are drawn (compensate_for_camera_motion)
 *   radius     point radius int(linewidth * 2), 0..255;  linewidth: trail line width, >= 0
 *   trail      tracks_leave_trace: 0 no trails; -1 every earlier step, unblended; > 0 the last `trail` steps, each
 *              step blended with the frame it was drawn on.  Trails are drawn on frames query_frame+1 .. T-1.
 *              With S = min(trail, T-1) (T-1 for -1) steps at most per frame and first(t) = max(0, t - trail) (0 for
 *              -1), step s of frame t is the segment from frame first(t)+s to first(t)+s+1.
 *   alphas     [T,S,2] fp64 (a, 1-a) with a = (s/L)**2, L = t - first(t) + 1; required when trail > 0
 *   diff       [T,S+1,2] fp64 or NULL: camera-motion offset of frame first(t)+j in the window of frame t; segment
 *              endpoints become int(int(track) - diff)
 * Invalid arguments return CT3_EINVAL (a too small workspace CT3_ENOSPC) before any launch. */
int ct3_render_tracks(uint8_t* frames, int T, int H, int W, const float* pts, const uint8_t* visible,
                      const uint8_t* colors, const uint8_t* draw_mask, int N, int radius, int linewidth, int trail,
                      int query_frame, const double* alphas, const double* diff, void* workspace,
                      size_t workspace_bytes, ct3_stream_t stream);
/* Scratch of ct3_render_flow_colors (one u64).  CT3_EINVAL unless T, N >= 1 and T*N <= INT32_MAX. */
int ct3_render_flow_workspace_bytes(int T, int N, size_t* out_bytes);
/* ct3_render_flow_colors: the colours of mode="optical_flow" (visualizer.py:191-194),
 *     flow_vis.flow_to_color(tracks - tracks[query_frame]) with tracks = pts.long(),
 * the Middlebury colour code normalised by the largest flow magnitude over all T*N entries, into `colors` [T,N,3]
 * uint8 in the layout ct3_render_tracks reads.  pts [T,N,2] fp32 as ct3_render_tracks takes it, truncated toward zero.
 * Every float64 operation is numpy's, correctly rounded and uncontracted, except atan2, which is CUDA's (within 2 ulp
 * of the correctly rounded value); an entry whose colour depends on atan2's last bits may differ by 1 from a CPU's.
 * The result is exact for points whose truncated coordinates have magnitude below 2^30; beyond that a coordinate
 * counts as +-(2^30 - 1) and NaN as 0, so every result is defined and deterministic.  The maximum is reduced on the
 * device, in stream order, without host synchronisation.  Null pointers, T or N < 1, T*N > INT32_MAX, query_frame
 * outside [0, T) or a too small workspace return CT3_EINVAL before any launch. */
int ct3_render_flow_colors(const float* pts, int T, int N, int query_frame, uint8_t* colors, void* workspace,
                           size_t workspace_bytes, ct3_stream_t stream);

/* ---- per-clip preparation ---------------------------------------------------
 * ct3_prepare_pyramid: cotracker3_offline.py:92-117 (L2-normalise over channels,
 * 3x avg_pool2d(2,2)).  in: fnet output [T,128,H4,W4] fp32 channel-planar.
 * out: pyr = 4 levels, channels-last [T,Hl,Wl,128] fp32, concatenated; level
 * offsets (in floats) are returned by ct3_pyramid_layout. */
int ct3_pyramid_layout(int T, int H4, int W4, int64_t level_off[4], int level_h[4], int level_w[4],
                       int64_t* total_floats);
int ct3_prepare_pyramid(const float* fmaps, int T, int H4, int W4, float* pyr, ct3_stream_t stream);

/* ct3_sample_support: get_track_feat / sample_features5d
 * (cotracker3_online.py:113-128, model_utils.py:293-323) for all 4 levels.
 * queried_frames [N] int32 (already relative to the window, clamped into [0,T-1]),
 * queried_coords [N,2] fp32 in stride-4 feature units (x,y).
 * support out: [4][49,N,128] fp32 (the reference's [B,49,N,C] layout per level).
 * If accumulate_mask != NULL ([N] uint8) the sampled features are ADDED to
 * `support` where mask!=0 and nothing is written elsewhere (online accumulation,
 * cotracker3_online.py:433-434); otherwise they overwrite. */
int ct3_sample_support(const float* pyr, int T, int H4, int W4, const int32_t* queried_frames,
                       const float* queried_coords, int N, const uint8_t* accumulate_mask,
                       float* support, ct3_stream_t stream);

/* ---- encoder tail (SURVEY.md 8(f) rank 1, partially): conv2 3x3 (416->256) -> InstanceNorm -> ReLU ->
 * conv3 1x1 (256->128) (BasicEncoder.forward tail, blocks.py:215-218) + L2-normalise + pyramid
 * (cotracker3_offline.py:92-117) on the GEMM engine.  cat: [T,416,H4,W4] fp32 channel-planar = the concatenated,
 * bilinearly resized stage outputs (blocks.py:210-215).  Output = the same channels-last pyramid as
 * ct3_prepare_pyramid.  Weights: conv2.weight [256,416,3,3], conv2.bias, conv3.weight [128,256,1,1], conv3.bias. */
/* bilinear (align_corners=True) resize of the 4 stage outputs [T,Cs,Hs,Ws] (fp32, planar) to H x W and channel concat
 * -> out [T, sum Cs, H, W] (blocks.py:202-215); src/channels/heights/widths are HOST arrays of 4 entries. */
int ct3_upsample_concat(const float* const* src, const int* channels, const int* heights, const int* widths, int T,
                        int H, int W, float* out, ct3_stream_t stream);
int ct3_enc_tail_packed_bytes(size_t* out_bytes);
int ct3_enc_tail_pack(const float* conv2_w, const float* conv2_b, const float* conv3_w, const float* conv3_b,
                      void* packed, size_t packed_bytes, ct3_stream_t stream);
int ct3_enc_tail_workspace_bytes(int T, int H4, int W4, size_t* out_bytes);
int ct3_enc_tail(const void* packed, const float* cat, int T, int H4, int W4, float* pyr, void* workspace,
                 size_t workspace_bytes, ct3_stream_t stream);

/* ---- the hot loop -----------------------------------------------------------
 * One update-loop pass is described by a ct3_loop_shape.
 *   groups       : the N tracks form G contiguous groups of group_sizes[0..G-1] tracks.  Each group has its own 64
 *                  virtual tokens and the space attention stays inside its group; the groups share every other launch
 *                  (correlation, corr_mlp, GEMMs, LayerNorms, time attention, heads).
 *   frame map    : with T_pyr >= 1, at time step t group g reads pyramid frame group_frames[g*T + t], an index into
 *                  the T_pyr frames of `pyr` (ct3_pyramid_layout(T_pyr, H4, W4)).  A group tracking the clip played
 *                  backwards uses T-1-t; a padded window of the sliding-window model uses clamped indices.  Only
 *                  correlation sampling reads frames: time attention, the time embedding, tokens and heads work on the
 *                  group's own time axis.  With T_pyr = 0 step t reads frame t of a T-frame pyramid.
 *   track slabs  : with slab_tracks >= 1 the stages that are independent per row (correlation, corr_mlp, token
 *                  assembly, input_transform, the time blocks, the LayerNorm + projections of the point side of both
 *                  cross blocks, out-projections and MLP halves) run on slabs of slab_tracks whole tracks (the 64*G
 *                  virtual tracks in slabs of their own), so their scratch is sized by slab_tracks*T rows; the space
 *                  attentions still see every track of a group in one launch.  Full-size per point row: the fp32 token
 *                  (1536 B) and the point side of the space attentions (3072 B), 4608 B against 65,024 B without slabs
 *                  (DESIGN.md §4.4.5).  Supported up to (N + 64*G)*T <= 2^21 token rows: every element offset of a
 *                  full-size buffer then stays below 2^31.
 * Contract (default options, same device): group g's coords/vis/conf are BIT-IDENTICAL to a pass over that group's
 * tracks alone (G = 1, no slabs) on a pyramid holding frames group_frames[g][0..T) in that order (without a map: the
 * same pyramid), whatever the other groups are; and BIT-IDENTICAL for every slab_tracks: slab_tracks >= N is the
 * launch sequence and workspace of slab_tracks = 0.
 *   group lengths: with group_T set, group g is a clip of group_T[g] steps padded to the pass's T.  Its steps
 *                  [group_T[g], T) are padding: computed, with unspecified state.  Its time attention runs over its own
 *                  steps only, its relative-motion posenc ends at its own last step, its time embedding is time_emb[g]
 *                  and its space attention splits K as a pass of group_T[g] steps does.  Map its padded steps to real
 *                  frames of its clip (e.g. the last one) in group_frames.  NULL is the launch sequence without the field.
 * Contract with group_T: group g's coords/vis/conf at steps t < group_T[g] are BIT-IDENTICAL to a pass over that group
 * alone with T = group_T[g], time embedding time_emb[g][0..group_T[g]) and frames group_frames[g][0..group_T[g]), with
 * or without slabs.  A group of at most 128 steps takes the fused time attention whenever a pass of its own length
 * would, also in a pass with T > 128.
 * group_sizes, group_frames and group_T are HOST arrays and may be freed when the call returns: the device-side group
 * table, frame map and per-track lengths live in the workspace and are filled in stream order (the library still
 * allocates nothing).
 * Options: the default kernels and the exact-fp32 verification kernels ("gemm" / "corr" / "attn" = 1) support G > 1
 * and group_T, as does "fuse" = 0. */
typedef struct ct3_loop_shape {
  int T, N;                       /* loop time steps, tracks (both >= 1)                                              */
  int H4, W4;                     /* level-0 feature map; 0, 0 = transformer only (ct3_updateformer sizing)           */
  int G;                          /* track groups, 1 <= G <= N                                                        */
  const int32_t* group_sizes;     /* HOST [G], each >= 1, sum N; NULL allowed only for G == 1                         */
  int T_pyr;                      /* 0: no frame map, step t reads frame t of a T-frame pyramid;
                                     >= 1: a frame map into T_pyr frames is given                                     */
  const int32_t* group_frames;    /* HOST [G*T] indices into [0, T_pyr) iff T_pyr >= 1, else NULL                     */
  int slab_tracks;                /* 0: no slabs; >= 1: track slabs, and then (N + 64 G) T <= 2^21                    */
  const int32_t* group_T;         /* HOST [G] group lengths, each in [1, T], or NULL: every group has length T (102)  */
} ct3_loop_shape;

/* ct3_workspace_bytes: scratch needed by ct3_update_loop for `shape` (it includes the split-bf16 copy of the T_pyr
 * (0: T) frame pyramid the correlation kernel reads through TMA, sized once per call).  Only the numeric fields are
 * needed, so a pass can be sized before its arrays exist; the arrays are validated when given.  Grows by 64*T virtual
 * token rows per group; non-decreasing in slab_tracks.  H4 = W4 = 0 (with T_pyr = slab_tracks = 0) sizes
 * ct3_updateformer. */
int ct3_workspace_bytes(const ct3_loop_shape* shape, size_t* out_bytes);

/* ct3_update_loop: `iters` refinement iterations of the pass `shape`, in place on the state.
 *   packed   : ct3_pack_weights output
 *   pyr      : ct3_prepare_pyramid output (T frames of the window; T_pyr frames with a frame map)
 *   support  : [4][49,N,128] fp32; track_valid (may be NULL) [N] uint8 zeroes the
 *              support of not-yet-queried tracks (cotracker3_online.py:493-496)
 *   coords   : [T,N,2] fp32 stride-4 feature units, in/out
 *   vis,conf : [T,N] fp32 logits, in/out
 *   time_emb : [T,1110] fp32 (buffer already interpolated to T,
 *              cotracker3_online.py:145-156); with group_T [G,T,1110], group g's
 *              interpolated to group_T[g] in rows [0, group_T[g])
 *   workspace: ct3_workspace_bytes(shape) bytes, 256-byte aligned
 * On return coords/vis/conf hold the state after the last iteration (the caller
 * multiplies coords by the stride and applies sigmoid, cotracker3_offline.py:213-216).
 * Every field of the shape is validated: a null pointer or shape, T or N < 1, G outside [1, N], a group size < 1, sizes
 * not summing to N, a null group_sizes with G > 1, T_pyr < 0, a frame map without T_pyr >= 1 or T_pyr >= 1 without
 * one, a frame index outside [0, T_pyr), slab_tracks < 0, more than 2^21 token rows with slabs, a group_T entry outside
 * [1, T] (ct3_workspace_bytes checks it too, and sizes the per-group tables when it is set), iters < 0, a bad
 * pyramid shape or a misaligned workspace return CT3_EINVAL, and a workspace smaller than the query CT3_ENOSPC, before
 * anything is enqueued. */
int ct3_update_loop(const void* packed, const float* pyr, const float* support, const uint8_t* track_valid,
                    float* coords, float* vis, float* conf, const float* time_emb, int iters,
                    const ct3_loop_shape* shape, void* workspace, size_t workspace_bytes, ct3_stream_t stream);

/* ---- live profiler (bench.py roofline): CUDA events around every launch of the library, summed per
 * kernel category: 0 corr_sample, 1 gemm (wgmma), 2 attention, 3 layernorm, 4 misc.
 * ct3_profile_enable(1) clears and starts recording; ct3_profile_read synchronises and sums. */
int ct3_profile_enable(int on);
int ct3_profile_read(double ms[7], int launches[7], double* gemm_flops);

/* ---- stage-level entry points (used by the parity tests and profiles) ------- */

/* Correlation sampling alone (get_correlation_feat + einsum,
 * cotracker3_online.py:130-143, cotracker3_offline.py:144-156) for all levels:
 * vol_split [N*T*4, 2*2432] bf16: row ((n*T+t)*4+level), hi plane cols [0,2432),
 * lo plane cols [2432,4864); value = hi+lo, cols 2401..2431 are zero. */
/* scratch: ct3_pyramid_layout's total * 4 bytes (256-byte aligned) for the split-bf16 pyramid copy of the
 * correlate-then-interpolate kernel (used when every level is >= 8x8 texels); NULL selects the
 * sample-then-correlate kernel.  With prec.corr < 3 the copy is ONE fp16 plane per level (the first half of each
 * level's region); the default kernel keeps its 4-byte work counter behind level 0's plane, zeroed by the call. */
int ct3_corr_sample(const float* pyr, int H4, int W4, const float* support,
                    const uint8_t* track_valid, const float* coords, int T, int N,
                    void* vol_split, void* scratch, size_t scratch_bytes, ct3_stream_t stream);

/* The first half of one ct3_update_loop iteration, from the state to the point tokens, run by the loop's own code
 * under the calling thread's "gemm" / "corr" / "prec.*" options: correlation sampling (the split pyramid copy when the
 * correlate-then-interpolate kernel runs), corr_mlp (cotracker3_offline.py:142-160) into X, vis / conf / posenc
 * (:162-188), and input_transform with the time embedding folded in as a per-frame bias (:196, cotracker.py:486).
 * Arguments as ct3_update_loop; coords / vis / conf are only read.  Outputs, each optional (NULL = not copied), written
 * in stream order:
 *   vol_out    : the correlation volume with ct3_corr_sample's layout and bytes: [N*T*4, 2*2432] split bf16, or one
 *                fp16 plane [N*T*4, 2432] when ct3_precision_info reports 2 bytes per element; rows support-major when
 *                ct3_volume_is_support_major says so
 *   x_out      : X [N*T, 2*1152] split 16-bit rows (bf16 hi cols 0..1151 | lo cols 1152..2303), row n*T + t, in the
 *                device column order (DESIGN.md: correlation embeddings 0..1023, vis 1024, conf 1025, posenc
 *                1026..1109, zero 1110..1151), WITHOUT the time embedding
 *   tokens_out : the point tokens fp32 [N*T, 384], row n*T + t
 * workspace: ct3_workspace_bytes of the shape {T, N, H4, W4, G = 1} bytes, 256-byte aligned.  Invalid arguments return
 * CT3_EINVAL and a too small workspace CT3_ENOSPC, with ct3_update_loop's checks and messages, before any launch. */
int ct3_loop_tokens(const void* packed, const float* pyr, int H4, int W4, const float* support,
                    const uint8_t* track_valid, const float* coords, const float* vis, const float* conf,
                    const float* time_emb, int T, int N, void* vol_out, void* x_out, float* tokens_out,
                    void* workspace, size_t workspace_bytes, ct3_stream_t stream);

/* Generic split-bf16x3 linear layer  Y = act(X W^T + b)  (nn.Linear, blocks.py:61-67)
 *   x_split [M, 2*Kpad] bf16 (hi|lo), w_split [Nout, 2*Kpad] bf16, bias [Nout] fp32 or NULL
 *   act: 0 none, 1 GELU(erf), 2 GELU(tanh);  y fp32 [M, Nout] */
int ct3_linear(const void* x_split, const void* w_split, const float* bias, int M, int Nout,
               int Kpad, int act, float* y, ct3_stream_t stream);

/* Same with the precision switches of the GEMM engine: `products` tensor-core products per FLOP (3: split x split,
 * 2: x_hi x (w_hi + w_lo), 1: x_hi x w_hi) on bf16 (fp16 = 0) or IEEE-fp16 (fp16 = 1) planes. */
int ct3_linear_prec(const void* x_split, const void* w_split, const float* bias, int M, int Nout,
                    int Kpad, int act, int products, int fp16, float* y, ct3_stream_t stream);

/* The whole epilogue of the GEMM engine, as the update loop and the encoder use it (ct3_linear and ct3_linear_prec are
 * this call with x_ld = 0, no row bias, y of pitch Nout and no split output), under the thread's "gemm" option:
 *   v[r, c] = act( sum_k x[r, k] w[c, k] + bias[c] + row_bias[(r % row_mod) * Nout + c] )
 *   x_split   [M, x_ld] 16-bit planes: hi at column 0, lo at column Kpad (read when products == 3); x_ld = 0 means
 *             2*Kpad, Kpad a single hi plane (products 1 | 2)
 *   w_split   [Nout, 2*Kpad];  bias [Nout] and row_bias [row_mod, Nout] fp32 or NULL
 *   y         fp32 or NULL:  y[r*ld_y + c] = v, or += v when residual = 1
 *   y_split   16-bit or NULL: output row o = r / row_group holds rows o*row_group .. of v side by side,
 *             hi at y_split[o*ld_split + (r % row_group)*Nout + c], lo lo_off elements further (hi + lo = v)
 * Outputs are written on the M (split: ceil(M / row_group)) rows and the Nout (split: row_group*Nout) columns they own,
 * nothing else.  CT3_EINVAL before any launch: null x / w, no output, M < 1, Nout % 128, Kpad % 64, act outside
 * 0..2, products outside 1..3, fp16 outside 0..1, x_ld below the planes read or not a multiple of 8, row_mod or
 * row_group < 1 (also when unused), residual without y, ld_y < Nout or not a multiple of 4, ld_split or lo_off not a
 * multiple of 8, hi and lo planes that overlap (lo_off < row_group*Nout or ld_split < lo_off + row_group*Nout), and
 * x, w, bias, row_bias, y or y_split not 16-byte aligned. */
int ct3_linear_ex(const void* x_split, int64_t x_ld, const void* w_split, const float* bias, int M, int Nout,
                  int Kpad, int products, int fp16, int act, const float* row_bias, int row_mod, float* y,
                  int64_t ld_y, int residual, void* y_split, int64_t ld_split, int lo_off, int row_group,
                  ct3_stream_t stream);

/* LayerNorm over rows of 384 (blocks.py:411,416; the norm_context of the cross blocks, cotracker.py:549) into split
 * bf16 rows [rows, 768] (hi cols 0..383 | lo cols 384..767), the kernel the transformer body runs:
 *   out = (x - mean) / sqrt(var + eps) * gamma + beta     (gamma = beta = NULL: no affine)
 * x [rows, 384] fp32.  Null x / out, only one of gamma and beta, rows < 1, eps negative or not finite, or a pointer
 * that is not 16-byte aligned return CT3_EINVAL before any launch. */
int ct3_layernorm(const float* x, int rows, const float* gamma, const float* beta, float eps, void* out_split,
                  ct3_stream_t stream);

/* q|k|v projection and per-track attention of time block `depth` (0..2) of the transformer body, routed as the body
 * routes it under the thread's options: the fused kernel when "fuse" = 1, "gemm" = 0, "attn" != 1 and T <= 128,
 * otherwise the q|k|v GEMM into fp32 and the time-attention kernel.
 *   x_split   [rows, 768] split bf16: the LayerNorm output of the block's token rows, track-major (row n*T + t)
 *   out_split [rows, 768] split bf16 (hi cols 0..383 | lo 384..767): softmax(q k^T / sqrt(48)) v per track and head;
 *             no other row is written
 *   workspace ct3_time_block_attention_workspace_bytes(T, rows) bytes, 256-byte aligned
 * Null pointers, depth outside 0..2, T < 1, rows < 1, rows % T != 0, packed / x_split / out_split not 16-byte aligned
 * return CT3_EINVAL and a too small workspace CT3_ENOSPC, before any launch. */
int ct3_time_block_attention_workspace_bytes(int T, int rows, size_t* out_bytes);
int ct3_time_block_attention(const void* packed, int depth, const void* x_split, int T, int rows, void* out_split,
                             void* workspace, size_t workspace_bytes, ct3_stream_t stream);

/* fp32 [rows, K] -> split bf16 [rows, 2*Kpad] (zero padded); _fp16: the planes hold IEEE fp16 instead */
int ct3_split_rows(const float* x, int rows, int K, int Kpad, void* x_split, ct3_stream_t stream);
int ct3_split_rows_fp16(const float* x, int rows, int K, int Kpad, void* x_split, ct3_stream_t stream);

/* One EfficientUpdateFormer forward (cotracker.py:483-531) on an explicit token
 * input x [N, T, 1110] fp32 (time embedding already added, reference column order);
 * delta out [N, T, 4] fp32.  The tracks form G groups as in ct3_loop_shape; a NULL group_sizes_host means G = 1;
 * workspace: ct3_workspace_bytes of the shape {T, N, 0, 0, G}.  Checks and messages as ct3_update_loop. */
int ct3_updateformer(const void* packed, const float* x, int T, int N, const int32_t* group_sizes_host, int G,
                     float* delta, void* workspace, size_t workspace_bytes, ct3_stream_t stream);

/* One attention core  out = softmax(q k^T * 48^-1/2) v  per head (8 x 48; Attention.forward, blocks.py:391-397) of
 * the transformer body, chosen and launched exactly as ct3_updateformer does it under the calling thread's
 * "attn" option (time attention always takes the unfused path that T > 128 takes in the body).
 * Every buffer holds the body's (N + 64*G)*T token rows: point n at row n*T + t, virtual token i of group g at row
 * (N + 64*g + i)*T + t.
 *   kind CT3_ATTN_TIME                : per track (all N + 64*G of them) over its T frames; q = kv = fused q|k|v rows
 *                                       [rows, 1152] (q cols 0.., k 384.., v 768..)
 *        CT3_ATTN_VIRTUAL_FROM_POINT  : per (group, frame), the group's 64 virtual queries over its points;
 *                                       q [rows, 384], kv = k|v [rows, 768]
 *        CT3_ATTN_VIRTUAL_SELF        : per (group, frame), 64 virtual tokens over themselves; q, kv [rows, 1152]
 *        CT3_ATTN_POINT_FROM_VIRTUAL  : per (group, frame), the group's points over its 64 virtual tokens;
 *                                       q [rows, 384], kv [rows, 768]
 *   q, kv          : fp32 device buffers (may alias), 16-byte aligned; only the rows the kind reads are read
 *   out_split      : bf16 [rows, 768] (hi cols 0..383 | lo cols 384..767); the query rows of the kind are written,
 *                    no other row
 *   group_sizes_host, G : the track groups of ct3_loop_shape, sum = N, not NULL
 *   workspace      : ct3_attention_workspace_bytes(T, N, G) bytes, 256-byte aligned (split-K partials, group table)
 * Null pointers, an unknown kind, bad T/N/groups, misalignment return CT3_EINVAL and a too small workspace
 * CT3_ENOSPC, before any launch. */
enum { CT3_ATTN_TIME = 0, CT3_ATTN_VIRTUAL_FROM_POINT = 1, CT3_ATTN_VIRTUAL_SELF = 2, CT3_ATTN_POINT_FROM_VIRTUAL = 3 };
int ct3_attention_workspace_bytes(int T, int N, int G, size_t* out_bytes);
int ct3_attention(int kind, const float* q, const float* kv, int T, int N, const int32_t* group_sizes_host, int G,
                  void* out_split, void* workspace, size_t workspace_bytes, ct3_stream_t stream);

/* ---- the whole CNN encoder (BasicEncoder.forward, blocks.py:190-219; normalise + pyramid,
 * cotracker3_offline.py:92-117) on the tensor-core engine, channels-last ------------------------------------
 * frames [T,3,H,W] fp32 already scaled to [-1,1] (cotracker3_offline.py:63) -> pyr (ct3_pyramid_layout(T, H/4, W/4)).
 * conv1 7x7/2 runs as fp32 SIMT, every other convolution as split-bf16x3 wgmma GEMMs (3x3 stride-1: implicit GEMM
 * over TMA-shifted NHWC boxes; strided ones: gather + GEMM); InstanceNorm statistics in fp64.
 * Weight tensors in the order of ct3_encoder_weight_name() (state-dict keys below `fnet.`). */
int ct3_encoder_num_weight_tensors(void);
const char* ct3_encoder_weight_name(int index);
int ct3_encoder_packed_bytes(size_t* out_bytes);
int ct3_encoder_pack(const float* const* tensors_host_array_of_device_ptrs, int n_tensors, void* packed,
                     size_t packed_bytes, ct3_stream_t stream);
int ct3_encoder_workspace_bytes(int T, int H, int W, size_t* out_bytes);
int ct3_encoder(const void* packed, const float* frames, int T, int H, int W, float* pyr, void* workspace,
                size_t workspace_bytes, ct3_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* CT3_B200_H_ */
