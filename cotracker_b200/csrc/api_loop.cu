// api_loop.cu -- the update loop of the C ABI (see include/ct3_b200.h): weight packing, workspace carving and the
// launch sequence of one refinement iteration (cotracker3_offline.py:139-216, cotracker.py:483-531), whole or in
// track slabs (ct3_loop_shape.slab_tracks, DESIGN.md §4.4.5).
#include <math.h>

#include <string>
#include <vector>

#include "abi.cuh"

using namespace ct3;

namespace {

// ------------------------------------------------------------------------------------------------
// packed-weights layout
struct Block {
  Lin qkv_h;  // time blocks only: q|k|v regrouped per head, rows h*144 + [q_h(48) | k_h(48) | v_h(48)] (fused attention)
  Lin q;    // self-attention blocks: fused q|k|v (N = 1152); cross blocks: to_q (N = 384)
  Lin kv;   // cross blocks only: to_kv (N = 768)
  Lin out, fc1, fc2;
  size_t ctx_g = 0, ctx_b = 0;  // cross blocks: norm_context weight / bias (fp32 [384])
  bool cross = false;
};
struct Layout {
  Lin corr_fc1, corr_fc2, in_tr;
  Lin corr_fc1_h;   // corr_mlp.fc1 once more as split fp16 planes (prec.fc1 = 1 | 2); shares corr_fc1's bias
  Lin corr_fc1_t, corr_fc1_th;   // the same two with the columns in corr_tc3.cu's support-major volume order
  Block time[kDepth], vself[kDepth], p2v[kDepth], v2p[kDepth];
  size_t heads_w = 0, heads_b = 0, virt = 0, win_f32 = 0;
  size_t total = 0;
};

void place_block(Block& b, bool cross, size_t& off, bool time = false) {
  b.cross = cross;
  if (time) place_lin(b.qkv_h, 3 * kC, kC, off);
  if (cross) {
    b.ctx_g = off; off = align_up(off + kC * sizeof(float));
    b.ctx_b = off; off = align_up(off + kC * sizeof(float));
    place_lin(b.q, kC, kC, off);
    place_lin(b.kv, 2 * kC, kC, off);
  } else {
    place_lin(b.q, 3 * kC, kC, off);
  }
  place_lin(b.out, kC, kC, off);
  place_lin(b.fc1, kMlpHid, kC, off);
  place_lin(b.fc2, kC, kMlpHid, off);
}
const Layout& layout() {
  static const Layout L0 = [] {   // C++11 thread-safe one-time initialisation
    Layout L;
    size_t off = 0;
    place_lin(L.corr_fc1, kCorrHid, kVol, off);
    place_lin(L.corr_fc1_h, kCorrHid, kVol, off);
    place_lin(L.corr_fc1_t, kCorrHid, kVol, off);
    place_lin(L.corr_fc1_th, kCorrHid, kVol, off);
    place_lin(L.corr_fc2, kCorrOut, kCorrHid, off);
    place_lin(L.in_tr, kC, kX, off);
    L.win_f32 = off; off = align_up(off + (size_t)kC * kX * sizeof(float));
    L.virt = off;    off = align_up(off + (size_t)kV * kC * sizeof(float));
    L.heads_w = off; off = align_up(off + 4 * kC * sizeof(float));
    L.heads_b = off; off = align_up(off + 4 * sizeof(float));
    for (int i = 0; i < kDepth; ++i) {
      place_block(L.time[i], false, off, /*time*/ true);
      place_block(L.vself[i], false, off);
      place_block(L.p2v[i], true, off);
      place_block(L.v2p[i], true, off);
    }
    L.total = off;
    return L;
  }();
  return L0;
}

// ------------------------------------------------------------------------------------------------
// weight tensor order expected by ct3_pack_weights
const std::vector<std::string>& weight_names() {
  static const std::vector<std::string> names0 = [] {
    std::vector<std::string> names;
    const char* head[] = {"corr_mlp.fc1.weight", "corr_mlp.fc1.bias", "corr_mlp.fc2.weight", "corr_mlp.fc2.bias",
                          "updateformer.input_transform.weight", "updateformer.input_transform.bias",
                          "updateformer.virual_tracks", "updateformer.flow_head.weight", "updateformer.flow_head.bias",
                          "updateformer.vis_conf_head.weight", "updateformer.vis_conf_head.bias"};
    for (const char* h : head) names.push_back(h);
    const char* self_t[] = {"attn.to_q.weight", "attn.to_q.bias", "attn.to_kv.weight", "attn.to_kv.bias",
                            "attn.to_out.weight", "attn.to_out.bias", "mlp.fc1.weight", "mlp.fc1.bias",
                            "mlp.fc2.weight", "mlp.fc2.bias"};
    const char* cross_t[] = {"norm_context.weight", "norm_context.bias", "cross_attn.to_q.weight",
                             "cross_attn.to_q.bias", "cross_attn.to_kv.weight", "cross_attn.to_kv.bias",
                             "cross_attn.to_out.weight", "cross_attn.to_out.bias", "mlp.fc1.weight", "mlp.fc1.bias",
                             "mlp.fc2.weight", "mlp.fc2.bias"};
    for (int i = 0; i < kDepth; ++i) {
      const std::string idx = std::to_string(i) + ".";
      for (const char* t : self_t) names.push_back("updateformer.time_blocks." + idx + t);
      for (const char* t : self_t) names.push_back("updateformer.space_virtual_blocks." + idx + t);
      for (const char* t : cross_t) names.push_back("updateformer.space_point2virtual_blocks." + idx + t);
      for (const char* t : cross_t) names.push_back("updateformer.space_virtual2point_blocks." + idx + t);
    }
    return names;
  }();
  return names0;
}

// ------------------------------------------------------------------------------------------------
// workspace.  Without track slabs (slab == N) every buffer covers all rows.  With them (slab_tracks < N) the scratch
// of the row-independent stages (vol, h1, xs, hmid, and the first S = slab*T rows of ln / att / qkv) holds one slab
// of rows; ln / att keep the virtual rows full-size behind it; qkv is also the full-size space-attention operand of
// the point rows (virtual<-point k|v [N*T, 768], then point<-virtual q [N*T, 384] followed by its split output
// [N*T, 2*384]), which is never live at the same time as a time block's q|k|v.
struct Workspace {
  __nv_bfloat16* vol;     // [S*4, 2*2432]
  __nv_bfloat16* h1;      // [S*4, 2*384]
  __nv_bfloat16* xs;      // [S, 2*1152]
  float* tokens;          // [(N+64)*T, 384]
  __nv_bfloat16* ln;      // [S + 64*T, 2*384]  (virtual rows from row S)
  __nv_bfloat16* att;     // [S + 64*T, 2*384]  (virtual rows from row S)
  float* qkv;             // [(N+64)*T, 1152]; slabbed: max(S*1152, N*T*768)   (also point q / point kv / p<-v output)
  float* vqkv;            // [64*T, 1152]       (virtual q / kv / qkv)
  __nv_bfloat16* hmid;    // [S + 64*T, 2*1536]; slabbed: [S, 2*1536]
  float* row_bias;        // [T, 384]; with group_T [G*T, 384] (group g's time embedding in rows g*T ..)
  float* att_part;        // split-K partials of the virtual<-point attention
  __nv_bfloat16* pyr_split;  // split-bf16 copy of the pyramid (corr_tc2.cu); null when H4 == 0
  int32_t* groups;        // device group table of a grouped call (GroupPlan); null when G == 1
  int32_t* frames;        // device frame map [G, T] of a pass with T_pyr >= 1; null without one
  int32_t* track_len;     // [N + 64 G] length of every point and virtual track's group; null without group_T
  int32_t* track_group;   // [N] group of every point track (its row-bias block); null without group_T
  int slab;               // tracks per slab; N: no slabs
  size_t total;
  bool slabbed() const { return slab_rows < point_rows; }
  int64_t slab_rows = 0, point_rows = 0;   // S and N*T
};
// split-K slots of the virtual<-point partials: a group of n tracks splits at most min(32, ceil(n/64)/2) ways
// (attention_tc_splits), so G groups of N tracks in all need at most (N + 63 G)/128 slots beyond one group's 32
int partial_slots(int N, int G) {
  if (G == 1) return kAttnMaxSplits;
  const int64_t s = kAttnMaxSplits + ((int64_t)N + 63LL * G) / 128;
  return (int)(s < (int64_t)kAttnMaxSplits * G ? s : (int64_t)kAttnMaxSplits * G);
}
// int32 entries of the group table: offsets [G+1] | all [G] | split [G] | slot [G] | small [G] | tiles [2 * max tiles]
int64_t group_table_ints(int N, int G) { return (int64_t)5 * G + 1 + 2 * ((int64_t)N / 128 + G); }
// A pass runs its space attentions through a group table when it has several groups or group lengths (group_T): each
// group's split-K count is then its own, from its own length
bool grouped(const ct3_loop_shape& s) { return s.G > 1 || s.group_T; }

// The workspace of pass s (a null base only measures): the split pyramid copy is sized by the T_pyr (0: T) frames the
// correlation reads, room for the [G, T] frame map iff T_pyr >= 1, slab_tracks 0 or >= N: no slabs
Workspace carve(void* base, const ct3_loop_shape& s) {
  Workspace w;
  const int T = s.T, N = s.N, G = s.G, H4 = s.H4, W4 = s.W4, T_pyr = s.T_pyr > 0 ? s.T_pyr : s.T;
  w.slab = s.slab_tracks > 0 && s.slab_tracks < N ? s.slab_tracks : N;
  const size_t R = (size_t)(N + (size_t)kV * G) * T, Rp = (size_t)N * T, Rv = (size_t)kV * G * T;
  const size_t S = (size_t)w.slab * T, Mc = S * kL;
  w.slab_rows = (int64_t)S;
  w.point_rows = (int64_t)Rp;
  const bool sl = w.slabbed();
  Carver c(base);
  w.vol = (__nv_bfloat16*)c.take(Mc * 2 * kVolPad * 2);
  w.h1 = (__nv_bfloat16*)c.take(Mc * 2 * kCorrHid * 2);
  w.xs = (__nv_bfloat16*)c.take(S * 2 * kXPad * 2);
  w.tokens = (float*)c.take(R * kC * 4);
  w.ln = (__nv_bfloat16*)c.take((S + Rv) * 2 * kC * 2);
  w.att = (__nv_bfloat16*)c.take((S + Rv) * 2 * kC * 2);
  w.qkv = (float*)c.take(sl ? (S * 3 > Rp * 2 ? S * 3 : Rp * 2) * kC * 4 : R * 3 * kC * 4);
  w.vqkv = (float*)c.take(Rv * 3 * kC * 4);
  w.hmid = (__nv_bfloat16*)c.take((sl ? S : R) * 2 * kMlpHid * 2);
  w.row_bias = (float*)c.take((size_t)(s.group_T ? G : 1) * T * kC * 4);
  w.att_part = (float*)c.take(attention_partial_bytes(T, kV, partial_slots(N, G)));
  w.pyr_split = nullptr;
  if (H4 > 0 && W4 > 0 && corr_patch_supported(T_pyr, H4, W4))
    w.pyr_split = (__nv_bfloat16*)c.take((size_t)pyramid_layout(T_pyr, H4, W4).total * 4);
  w.groups = grouped(s) ? (int32_t*)c.take((size_t)group_table_ints(N, G) * 4) : nullptr;
  w.frames = s.T_pyr > 0 ? (int32_t*)c.take((size_t)G * T * 4) : nullptr;
  w.track_len = s.group_T ? (int32_t*)c.take(((size_t)N + (size_t)kV * G) * 4) : nullptr;
  w.track_group = s.group_T ? (int32_t*)c.take((size_t)N * 4) : nullptr;
  w.total = c.off;
  return w;
}

// ------------------------------------------------------------------------------------------------
struct Runner {
  const uint8_t* pk;
  const Layout& L;
  cudaStream_t s;
  int impl;

  int gemm(const char* what, const __nv_bfloat16* x, const Lin& lin, int M, const GemmEpilogue& e, int products = 3,
           int fp16 = 0, int64_t x_ld = 0) {
    GemmProblem p;
    p.products = products;
    p.fp16 = fp16;
    p.x_ld = x_ld;
    p.x_split = x;
    p.w_split = reinterpret_cast<const __nv_bfloat16*>(pk + lin.w);
    p.M = M;
    p.N = lin.N;
    p.Kpad = lin.Kpad;
    p.epi = e;
    if (!p.epi.bias) p.epi.bias = reinterpret_cast<const float*>(pk + lin.b);
    if (M == 0) return 0;
    ProfScope ps(s, CAT_GEMM, 2.0 * (double)M * lin.N * lin.K);
    return run_gemm(p, impl, s, what);
  }
  static GemmEpilogue to_f32(float* out, int ld, bool residual) {
    GemmEpilogue e;
    e.out_f32 = out; e.ld_f32 = ld; e.residual = residual ? 1 : 0;
    return e;
  }
  static GemmEpilogue to_split(__nv_bfloat16* out, int ld, int lo_off, int act) {
    GemmEpilogue e;
    e.out_split = out; e.ld_split = ld; e.lo_off = lo_off; e.act = act;
    return e;
  }
};

// a kernel launch returning cudaError_t, inside a profiler scope of category cat
#define RUNC(cat, call)                                        \
  do {                                                         \
    cudaError_t e__;                                           \
    { ProfScope ps__(R.s, cat); e__ = (cudaError_t)(call); }   \
    if (e__ != cudaSuccess) return fail_cuda(e__, #call);      \
  } while (0)
// a linear layer through R.gemm; the call's text names the layer in the error message
#define GEMM(...)                                                              \
  do {                                                                         \
    if (int rc__ = R.gemm("gemm(" #__VA_ARGS__ ")", __VA_ARGS__)) return rc__; \
  } while (0)

int run_attention(Runner& R, const Workspace& W, const AttnParams& a, bool per_warp) {
  if (g_opt_attn == 1) return (int)launch_attention(a, R.s);
  // point <- virtual (64 keys per frame, thousands of queries): wgmma kernel with TMA row staging (attention_p2v.cu)
  if (!per_warp && a.Lq > kV && attention_p2v_supported(a)) return (int)launch_attention_p2v(a, R.s);
  return (int)launch_attention_tc(a, per_warp, W.att_part, num_sms(), R.s);
}

// One attention of a transformer block: q at column 0 of q, k / v at columns k_col / v_col of kv, the result as split
// rows of `out` (pitch 2*kC).  Space attention (tracks == 0): one sequence per frame t < T of Lq queries over Lk keys,
// token i at row i*T + t.  Time attention: one sequence per track (`tracks` of them) over its T frames, rows n*T + t.
AttnParams attn_params(const float* q, int q_ld, const float* kv, int kv_ld, int k_col, int v_col, __nv_bfloat16* out,
                       int Lq, int Lk, int T, int tracks = 0) {
  AttnParams a{};
  a.q = q; a.q_ld = q_ld; a.q_col = 0;
  a.kv = kv; a.kv_ld = kv_ld; a.k_col = k_col; a.v_col = v_col;
  a.out = out; a.out_ld = 2 * kC; a.lo_off = kC;
  a.num_seq = tracks ? tracks : T; a.Lq = Lq; a.Lk = Lk;
  a.q_seq_stride = a.k_seq_stride = tracks ? T : 1;
  a.q_tok_stride = a.k_tok_stride = tracks ? 1 : T;
  a.scale = 1.0f / sqrtf((float)kDh);
  return a;
}

// Track groups of a pass (ct3_loop_shape.G): G contiguous track ranges, each with its own kV virtual tokens at rows
// (N + kV*g + i)*T + t.  G == 1 is one group (no table; every kernel indexes as it always did).
// For G > 1 the host builds the table below, uploads it into the workspace in stream order, and each space attention
// runs over (group, frame) sequences, choosing per group what a standalone call on that group's tracks would.
struct GroupPlan {
  int G = 1, max_n = 0;
  const int32_t *off = nullptr, *all = nullptr, *split = nullptr, *slot = nullptr, *small = nullptr, *tile = nullptr;
  int n_small = 0, n_tiles = 0, split_max = 1, split_slots = 0;
  // group lengths (ct3_loop_shape.group_T): every point and virtual track's length, on the device and on the host
  const int32_t *track_len = nullptr, *track_len_host = nullptr;
};

// group_T: null, or the G group lengths; a table is built whenever G > 1 or group_T is given (grouped())
int plan_groups(GroupPlan& gp, const int32_t* sizes, int G, int T, int N, const int32_t* group_T, int32_t* dev,
                cudaStream_t s) {
  gp.G = G;
  if (G == 1 && !group_T) return 0;
  std::vector<int32_t> h((size_t)group_table_ints(N, G), 0);
  int32_t* off = h.data();
  int32_t *all = off + G + 1, *split = all + G, *slot = split + G, *small = slot + G, *tile = small + G;
  const int nsm = num_sms();
  for (int g = 0; g < G; ++g) {
    const int n = sizes ? sizes[g] : N;
    off[g + 1] = off[g] + n;
    if (n > gp.max_n) gp.max_n = n;
    all[g] = g;
    // virtual <- point: the split-K count of a standalone call (T, or group_T[g], sequences of kV queries over n keys)
    split[g] = attention_tc_splits(group_T ? group_T[g] : T, kV, n, nsm);
    if (split[g] > 1) {
      slot[g] = gp.split_slots;
      gp.split_slots += split[g];
      if (split[g] > gp.split_max) gp.split_max = split[g];
    }
    // point <- virtual: a standalone call runs more than kV tracks on the wgmma kernel, fewer on mma.sync (run_attention)
    if (n > kV) {
      for (int n0 = off[g]; n0 < off[g + 1]; n0 += 128, ++gp.n_tiles) {
        tile[2 * gp.n_tiles] = g;
        tile[2 * gp.n_tiles + 1] = n0;
      }
    } else {
      small[gp.n_small++] = g;
    }
  }
  if (gp.split_slots > partial_slots(N, G)) return fail(CT3_EINVAL, "split-K partials exceed the workspace%s");
  CK(launch_upload_i32(dev, h.data(), (int)h.size(), s), "upload group table");
  gp.off = dev;
  gp.all = dev + (all - off);
  gp.split = dev + (split - off);
  gp.slot = dev + (slot - off);
  gp.small = dev + (small - off);
  gp.tile = dev + (tile - off);
  return 0;
}

// One space attention of a block (cotracker.py:510-517) over every group.  `a` describes it for one group of N tracks
// (sequence = frame); q_pts / k_pts tell which side holds the point tokens.
int space_attention(Runner& R, const Workspace& W, const GroupPlan& gp, AttnParams a, bool q_pts, bool k_pts) {
  if (!gp.off) return run_attention(R, W, a, false);
  const int T = a.num_seq, n_all = a.Lq;
  a.goff = gp.off;
  a.frames = T;
  a.q_grp_stride = q_pts ? 0 : (int64_t)kV * a.q_tok_stride;
  a.k_grp_stride = k_pts ? 0 : (int64_t)kV * a.k_tok_stride;
  a.Lq = q_pts ? gp.max_n : kV;
  a.Lk = k_pts ? gp.max_n : kV;
  AttnParams b = a;
  b.gl = gp.all;
  b.num_seq = T * gp.G;
  if (g_opt_attn == 1) return (int)launch_attention(b, R.s);
  if (!q_pts) {   // virtual <- point (split-K per group) and virtual self attention
    if (k_pts) { b.gsplit = gp.split; b.gslot = gp.slot; b.split_max = gp.split_max; b.split_slots = gp.split_slots; }
    return (int)launch_attention_tc(b, false, W.att_part, num_sms(), R.s);
  }
  // point <- virtual
  if (gp.n_small > 0) {
    b.gl = gp.small;
    b.num_seq = T * gp.n_small;
    b.Lq = kV;
    if (int rc = (int)launch_attention_tc(b, false, W.att_part, num_sms(), R.s)) return rc;
  }
  if (gp.n_tiles > 0) {
    AttnParams c = a;
    c.gtile = gp.tile;
    c.tiles = gp.n_tiles;
    c.Lq = n_all;
    c.Lk = kV * gp.G;
    return (int)launch_attention_p2v(c, R.s);
  }
  return 0;
}

// q|k|v projection and the per-track T x T attention of time block b on the LayerNorm output x [rows, 2*kC] (rows
// n*T + t) into att (split rows of pitch 2*kC).  With fuse = 1 on the product kernels (gemm 0, attn != 1) and T <= 128
// both run in ONE kernel, so fp32 q|k|v never reaches HBM; otherwise the b.q GEMM writes q|k|v to W.qkv [rows, 3*kC]
// and the per-warp attention kernel reads it.
// len / len_host: null, or the length of each of the rows / T tracks (ct3_loop_shape.group_T) on the device and the
// host: a track attends over its own frames only.  A track takes the kernel a pass of its own length would take: with
// T > 128 and fusion on, the runs of tracks of at most 128 frames take the fused kernel (one track per tile, rows
// t < 128) and the other runs the unfused one, each track once.  The fused kernel leaves rows [128, T) of a short
// track, all of them padding, unwritten: they are zeroed so that every padded row stays finite.
int time_attention(Runner& R, const Workspace& W, const Block& b, const __nv_bfloat16* x, __nv_bfloat16* att,
                   int rows, int T, const int32_t* len = nullptr, const int32_t* len_host = nullptr) {
  const bool fuse = g_opt[OPT_FUSE] == 1 && R.impl == 0 && g_opt_attn != 1;
  // The fused kernel reads keys [0, len) of a track from its 128-row tile: with T > 128 only tracks whose len_host
  // entry is at most 128 may reach it, which the run split below guarantees (qkv_time_attn_supported).
  auto fused = [&](int track0, int tracks) -> int {   // tracks [track0, track0 + tracks) of the rows
    ProfScope ps(R.s, CAT_QKVA, 0.0);
    const char* gerr = nullptr;
    const int64_t r0 = (int64_t)track0 * T;
    const int rc = gemm_qkv_time_attn_launch(
        x + r0 * 2 * kC, reinterpret_cast<const __nv_bfloat16*>(R.pk + b.qkv_h.w),
        reinterpret_cast<const float*>(R.pk + b.qkv_h.b), tracks * T, kC, T, len ? len + track0 : nullptr,
        att + r0 * 2 * kC, 2 * kC, kC, 1.0f / sqrtf((float)kDh), num_sms(), R.s, &gerr);
    return rc ? fail_launch(rc, "fused qkv + time attention", gerr) : 0;
  };
  auto unfused = [&](int track0, int tracks) -> int {
    const int64_t r0 = (int64_t)track0 * T;
    GEMM(x + r0 * 2 * kC, b.q, tracks * T, Runner::to_f32(W.qkv, 3 * kC, false));
    AttnParams a = attn_params(W.qkv, 3 * kC, W.qkv, 3 * kC, kC, 2 * kC, att + r0 * 2 * kC, T, T, T, tracks);
    a.seq_len = len ? len + track0 : nullptr;
    RUNC(CAT_ATTN, run_attention(R, W, a, true));
    return 0;
  };
  if (fuse && qkv_time_attn_supported(T)) return fused(0, rows / T);
  if (!fuse || !len_host) return unfused(0, rows / T);
  for (int i = 0, n = rows / T; i < n;) {
    const bool short_run = qkv_time_attn_supported(len_host[i]);
    int j = i + 1;
    while (j < n && qkv_time_attn_supported(len_host[j]) == short_run) ++j;
    if (short_run) {
      if (int rc = fused(i, j - i)) return rc;
      const size_t row_bytes = 2 * kC * sizeof(__nv_bfloat16);
      CK(cudaMemset2DAsync(att + ((int64_t)i * T + 128) * 2 * kC, (size_t)T * row_bytes, 0,
                           (size_t)(T - 128) * row_bytes, (size_t)(j - i), R.s),
         "zero padded time-attention rows");
    } else if (int rc = unfused(i, j - i)) {
      return rc;
    }
    i = j;
  }
  return 0;
}

// Row `row` of the token buffer in the scratch of the row-independent stages (ln, att, hmid, the time block's qkv):
// the same row without slabs, relative to the slab's first row with them.
int64_t scratch_row(const Workspace& W, int64_t row, int64_t slab_row0) { return W.slabbed() ? row - slab_row0 : row; }

// The track ranges [n, n + count) the row-independent stages run on, for tracks [n_begin, n_end) of the N point and
// kV*G virtual tracks: without slabs the whole range in one piece, so every launch is the unslabbed one; with them,
// pieces of at most W.slab tracks that never mix point and virtual tracks.  f(n, count) returns 0 or an error code.
template <class F>
int for_slabs(const Workspace& W, int N, int n_begin, int n_end, F&& f) {
  if (!W.slabbed()) return f(n_begin, n_end - n_begin);
  for (int n = n_begin; n < n_end;) {
    const int stop = n < N && n_end > N ? N : n_end;
    const int count = stop - n < W.slab ? stop - n : W.slab;
    if (int rc = f(n, count)) return rc;
    n += count;
  }
  return 0;
}

// x += to_out(attn(...)); x += mlp(LN(x))   for the rows [row0, row0+rows) of the token buffer, which lie in the slab
// whose first row is slab_row0
int mlp_half(Runner& R, const Workspace& W, const Block& b, int64_t row0, int rows, int64_t slab_row0) {
  float* x = W.tokens + row0 * kC;
  const int64_t s = scratch_row(W, row0, slab_row0);
  __nv_bfloat16* ln = W.ln + s * 2 * kC;
  __nv_bfloat16* hm = W.hmid + s * 2 * kMlpHid;
  RUNC(CAT_LN, launch_layernorm_split(x, rows, nullptr, nullptr, 1e-6f, ln, R.s));
  GEMM(ln, b.fc1, rows, Runner::to_split(hm, 2 * kMlpHid, kMlpHid, /*tanh*/ 2));
  GEMM(hm, b.fc2, rows, Runner::to_f32(x, kC, true));
  return 0;
}

// EfficientUpdateFormer body on W.tokens (point rows already hold input_transform output) -- cotracker.py:486-524.
// With track slabs (DESIGN.md §4.4.5) the row-independent stages run slab by slab (for_slabs); the space attentions
// always see every track of a group in one launch.
int transformer_body(Runner& R, const Workspace& W, int T, int N, const GroupPlan& gp) {
  const Layout& L = R.L;
  const int NV = kV * gp.G, Rp = N * T, Rv = NV * T;
  const uint8_t* pk = R.pk;
  RUNC(CAT_MISC, launch_init_virtual(W.tokens, reinterpret_cast<const float*>(pk + L.virt), T, N, gp.G, R.s));
  float* vtok = W.tokens + (int64_t)Rp * kC;
  __nv_bfloat16* ln_v = W.ln + W.slab_rows * 2 * kC;
  __nv_bfloat16* att_v = W.att + W.slab_rows * 2 * kC;
  // point<-virtual's q and output: with slabs both full-size in W.qkv, behind each other
  float* q_p = W.qkv;
  __nv_bfloat16* att_p = W.slabbed() ? reinterpret_cast<__nv_bfloat16*>(W.qkv + (int64_t)Rp * kC) : W.att;
  // LayerNorm (optionally with the context gamma / beta) of point tracks [n, n + count) into the slab scratch, then
  // the GEMM `lin` of those rows into out (pitch ld) at their own rows
  auto ln_gemm_points = [&](const Block& b, bool ctx, const Lin& lin, float* out, int ld) {
    return for_slabs(W, N, 0, N, [&](int n, int count) -> int {
      const int64_t r0 = (int64_t)n * T;
      __nv_bfloat16* ln = W.ln + scratch_row(W, r0, r0) * 2 * kC;
      RUNC(CAT_LN, launch_layernorm_split(W.tokens + r0 * kC, count * T,
                                          ctx ? reinterpret_cast<const float*>(pk + b.ctx_g) : nullptr,
                                          ctx ? reinterpret_cast<const float*>(pk + b.ctx_b) : nullptr,
                                          ctx ? 1e-5f : 1e-6f, ln, R.s));
      GEMM(ln, lin, count * T, Runner::to_f32(out + r0 * ld, ld, false));
      return 0;
    });
  };
  // the MLP half of tracks [n_begin, n_end), slab by slab
  auto mlp_tracks = [&](const Block& b, int n_begin, int n_end) {
    return for_slabs(W, N, n_begin, n_end, [&](int n, int count) -> int {
      return mlp_half(R, W, b, (int64_t)n * T, count * T, (int64_t)n * T);
    });
  };

  for (int i = 0; i < kDepth; ++i) {
    {  // ---- time block over every token row (points + virtual): sequence = track (cotracker.py:494-495)
      const Block& b = L.time[i];
      if (int rc = for_slabs(W, N, 0, N + NV, [&](int n, int count) -> int {
            const int64_t r0 = (int64_t)n * T;
            const int rows = count * T;
            const int64_t s0 = scratch_row(W, r0, r0);
            float* x = W.tokens + r0 * kC;
            RUNC(CAT_LN, launch_layernorm_split(x, rows, nullptr, nullptr, 1e-6f, W.ln + s0 * 2 * kC, R.s));
            if (int rc = time_attention(R, W, b, W.ln + s0 * 2 * kC, W.att + s0 * 2 * kC, rows, T,
                                        gp.track_len ? gp.track_len + n : nullptr,
                                        gp.track_len_host ? gp.track_len_host + n : nullptr))
              return rc;
            GEMM(W.att + s0 * 2 * kC, b.out, rows, Runner::to_f32(x, kC, true));
            return mlp_half(R, W, b, r0, rows, r0);
          }))
        return rc;
    }
    {  // ---- virtual <- point cross attention (cotracker.py:510-512): x = virtual, context = points
      const Block& b = L.v2p[i];
      RUNC(CAT_LN, launch_layernorm_split(vtok, Rv, nullptr, nullptr, 1e-6f, ln_v, R.s));
      GEMM(ln_v, b.q, Rv, Runner::to_f32(W.vqkv, kC, false));
      if (int rc = ln_gemm_points(b, true, b.kv, W.qkv, 2 * kC)) return rc;
      RUNC(CAT_ATTN, space_attention(R, W, gp, attn_params(W.vqkv, kC, W.qkv, 2 * kC, 0, kC, att_v, kV, N, T), false,
                                     true));
      GEMM(att_v, b.out, Rv, Runner::to_f32(vtok, kC, true));
      if (int rc = mlp_tracks(b, N, N + NV)) return rc;
    }
    {  // ---- virtual self attention (cotracker.py:514): sequence = frame over the 64 virtual tokens
      const Block& b = L.vself[i];
      RUNC(CAT_LN, launch_layernorm_split(vtok, Rv, nullptr, nullptr, 1e-6f, ln_v, R.s));
      GEMM(ln_v, b.q, Rv, Runner::to_f32(W.vqkv, 3 * kC, false));
      RUNC(CAT_ATTN, space_attention(R, W, gp, attn_params(W.vqkv, 3 * kC, W.vqkv, 3 * kC, kC, 2 * kC, att_v, kV, kV,
                                                           T), false, false));
      GEMM(att_v, b.out, Rv, Runner::to_f32(vtok, kC, true));
      if (int rc = mlp_tracks(b, N, N + NV)) return rc;
    }
    {  // ---- point <- virtual cross attention (cotracker.py:515-517): x = points, context = virtual
      const Block& b = L.p2v[i];
      if (int rc = ln_gemm_points(b, false, b.q, q_p, kC)) return rc;
      RUNC(CAT_LN, launch_layernorm_split(vtok, Rv, reinterpret_cast<const float*>(pk + b.ctx_g),
                                 reinterpret_cast<const float*>(pk + b.ctx_b), 1e-5f, ln_v, R.s));
      GEMM(ln_v, b.kv, Rv, Runner::to_f32(W.vqkv, 2 * kC, false));
      RUNC(CAT_ATTN, space_attention(R, W, gp, attn_params(q_p, kC, W.vqkv, 2 * kC, 0, kC, att_p, N, kV, T), true,
                                     false));
      if (int rc = for_slabs(W, N, 0, N, [&](int n, int count) -> int {
            const int64_t r0 = (int64_t)n * T;
            GEMM(att_p + r0 * 2 * kC, b.out, count * T, Runner::to_f32(W.tokens + r0 * kC, kC, true));
            return mlp_half(R, W, b, r0, count * T, r0);
          }))
        return rc;
    }
  }
  return 0;
}

// effective precision of the correlation branch for this thread's options: the single-plane / fewer-product modes
// exist in the correlate-then-interpolate kernels only (corr_tc3.cu, corr_tc2.cu), so whenever another correlation
// kernel runs the branch computes split x split
struct Prec {
  int corr, fc1; bool patch;
  bool vol16() const { return fc1 < 3; }
  bool support_major() const { return patch && corr != 3; }   // corr_tc3.cu writes k*49 + i
};
Prec effective_prec(bool have_pyr_split, int T, int H4, int W4) {
  Prec p;
  p.patch = corr_uses_patch_kernel(g_opt_corr, have_pyr_split, T, H4, W4);
  p.corr = p.patch ? g_opt[OPT_PREC_CORR] : 3;
  p.fc1 = p.patch ? g_opt[OPT_PREC_FC1] : 3;
  return p;
}

// input_transform of the X rows in W.xs into the point tokens of tracks [n0, n0 + count), with the per-frame bias
// row_bias [T, kC] when given (a track's rows start at a multiple of T, so row % T is the frame); with W.track_group
// (group_T) track n adds block track_group[n] of row_bias [G*T, kC], its group's time embedding
int input_transform(Runner& R, const Workspace& W, int T, int n0, int count, const float* row_bias) {
  GemmEpilogue e = Runner::to_f32(W.tokens + (int64_t)n0 * T * kC, kC, false);
  if (row_bias) { e.row_bias = row_bias; e.row_mod = T; }
  if (row_bias && W.track_group) e.row_blk = W.track_group + n0;
  GEMM(W.xs, R.L.in_tr, count * T, e);
  return 0;
}

// point_tokens for the tracks [n0, n0 + count) of the N-track state, from row 0 of the stage's scratch
int point_tokens_slab(Runner& R, const Workspace& W, const Prec& pr, const float* pyr, const __nv_bfloat16* pyr_split,
                      int H4, int W4, const float* support, const uint8_t* track_valid, const float* coords,
                      const float* vis, const float* conf, int T, int N, int T_pyr, const FrameMap& fm, int n0,
                      int count) {
  const Layout& L = R.L;
  const int Mc = count * T * kL;
  // (i)+(ii) sampling + 4-D correlation, all levels -> split volume
  RUNC(CAT_CORR, launch_corr_sample(pyr, pyr_split, H4, W4, support, track_valid, coords, T, N, n0, count, W.vol,
                                    g_opt_corr, pr.corr, pr.vol16() ? 1 : 0, num_sms(), R.s, T_pyr, fm));
  // (iii) corr_mlp: 2401 -> 384 (GELU erf) -> 256, written straight into X columns [256*l, 256*l+256)
  if (pr.vol16()) {   // single fp16 volume plane x split fp16 weights: 2 (or 1) tensor-core products per FLOP
    GEMM(W.vol, pr.support_major() ? L.corr_fc1_th : L.corr_fc1_h, Mc,
         Runner::to_split(W.h1, 2 * kCorrHid, kCorrHid, /*erf*/ 1), pr.fc1, /*fp16*/ 1, kVolPad);
  } else {
    GEMM(W.vol, pr.support_major() ? L.corr_fc1_t : L.corr_fc1, Mc,
         Runner::to_split(W.h1, 2 * kCorrHid, kCorrHid, /*erf*/ 1));
  }
  {
    GemmEpilogue e = Runner::to_split(W.xs, 2 * kXPad, kXPad, 0);
    e.row_group = kL;
    GEMM(W.h1, L.corr_fc2, Mc, e);
  }
  // vis, conf, posenc(rel. motion), zero pad -> X columns [1024,1152)
  RUNC(CAT_MISC, launch_build_x_small(coords, vis, conf, T, N, n0, count, W.track_len, W.xs, R.s));
  // (iv) input_transform (+ folded time embedding) -> point tokens
  return input_transform(R, W, T, n0, count, W.row_bias);
}

// The first half of one update-loop iteration, from the state to the point tokens: the correlation volume (W.vol),
// corr_mlp into the correlation columns of X and build_x_small into the rest (W.xs), then input_transform with the
// time-embedding fold W.row_bias into the point rows of W.tokens.  Reads coords / vis / conf, writes none of them.
// pyr_split: the split pyramid when the patch kernel runs (pr.patch), else null.  With track slabs each slab of
// tracks [n0, n0 + count) runs the whole stage through the slab scratch into its own rows of W.tokens.
int point_tokens(Runner& R, const Workspace& W, const Prec& pr, const float* pyr, const __nv_bfloat16* pyr_split,
                 int H4, int W4, const float* support, const uint8_t* track_valid, const float* coords,
                 const float* vis, const float* conf, int T, int N, int T_pyr, const FrameMap& fm) {
  return for_slabs(W, N, 0, N, [&](int n0, int count) -> int {
    return point_tokens_slab(R, W, pr, pyr, pyr_split, H4, W4, support, track_valid, coords, vis, conf, T, N, T_pyr,
                             fm, n0, count);
  });
}


// The steps update_loop and updateformer share once the point tokens are in W.tokens: the transformer body, then the
// heads: the state update of coords / vis / conf, or with delta != nullptr the raw deltas [N,T,4] instead.
int transform_and_heads(Runner& R, const Workspace& W, int T, int N, const GroupPlan& gp, float* coords, float* vis,
                        float* conf, float* delta) {
  const Layout& L = R.L;
  if (int rc = transformer_body(R, W, T, N, gp)) return rc;
  RUNC(CAT_MISC, launch_heads(W.tokens, reinterpret_cast<const float*>(R.pk + L.heads_w),
                              reinterpret_cast<const float*>(R.pk + L.heads_b), coords, vis, conf, delta, T, N, R.s));
  return 0;
}

int check_TN(int T, int N, int G = 1) {
  if (T < 1 || N < 1) return fail(CT3_EINVAL, "T and N must be >= 1%s");
  if (G < 1 || G > N) return fail(CT3_EINVAL, "G must be in [1, N]%s");
  if (((int64_t)N + (int64_t)kV * G) * T * 3 * kC >= (int64_t)1 << 40) return fail(CT3_EINVAL, "problem too large%s");
  return 0;
}

// The supported size of a pass in track slabs: at most 2^21 token rows (N + 64 G)*T.  Track slabs make problems
// reachable whose full-size buffers (tokens, the point rows' space-attention operands, up to 768 elements per row)
// no longer fit a full workspace; at this bound every element offset into them stays below 2^31, so no index
// arithmetic on the slabbed path can overflow 32 bits.  The slab-sized stages run the kernels of a full-workspace
// call on slab_tracks*T rows.
constexpr int64_t kSlabbedMaxRows = (int64_t)1 << 21;

// What a shape is checked for: the size query (host arrays checked when given; the pyramid unless H4 = W4 = 0 without
// a frame map or slabs, the transformer alone), a loop run (arrays and pyramid required) or ct3_updateformer (arrays
// required, no pyramid).
enum class Use { kSize, kLoop, kFormer };

int check_shape(const ct3_loop_shape* sh, Use use) {
  if (!sh) return fail(CT3_EINVAL, "null shape%s");
  const ct3_loop_shape& s = *sh;
  if (int rc = check_TN(s.T, s.N, s.G)) return rc;
  if (s.group_T)
    for (int g = 0; g < s.G; ++g)
      if (s.group_T[g] < 1 || s.group_T[g] > s.T) return fail(CT3_EINVAL, "every group_T entry must be in [1, T]%s");
  if (s.group_sizes) {
    int64_t sum = 0;
    for (int g = 0; g < s.G; ++g) {
      if (s.group_sizes[g] < 1) return fail(CT3_EINVAL, "every group size must be >= 1%s");
      sum += s.group_sizes[g];
    }
    if (sum != s.N) return fail(CT3_EINVAL, "group sizes must sum to N%s");
  } else if (use != Use::kSize && s.G > 1) {
    return fail(CT3_EINVAL, "null group_sizes with G > 1%s");
  }
  if (s.slab_tracks < 0) return fail(CT3_EINVAL, "slab_tracks must be >= 0%s");
  if (s.slab_tracks > 0 && ((int64_t)s.N + (int64_t)kV * s.G) * s.T > kSlabbedMaxRows)
    return fail(CT3_EINVAL, "problem too large for track slabs: (N + 64 G) * T must be <= 2^21%s");
  if (s.T_pyr < 0 || (s.T_pyr == 0 && s.group_frames))
    return fail(CT3_EINVAL, "T_pyr must be >= 1 with a frame map and 0 without one%s");
  if (s.T_pyr > 0) {
    if (s.group_frames) {
      for (int64_t i = 0; i < (int64_t)s.G * s.T; ++i)
        if (s.group_frames[i] < 0 || s.group_frames[i] >= s.T_pyr)
          return fail(CT3_EINVAL, "frame index outside [0, T_pyr)%s");
    } else if (use != Use::kSize) {
      return fail(CT3_EINVAL, "null group_frames with T_pyr >= 1%s");
    }
  }
  const bool former = s.H4 == 0 && s.W4 == 0 && s.T_pyr == 0 && s.slab_tracks == 0;
  if (use == Use::kFormer || (use == Use::kSize && former)) return 0;
  const int T_pyr = s.T_pyr > 0 ? s.T_pyr : s.T;   // a step's frame index stays within int32
  if ((int64_t)T_pyr * s.T >= (int64_t)1 << 31) return fail(CT3_EINVAL, "problem too large%s");
  return check_pyramid(T_pyr, s.H4, s.W4);
}

int update_loop(const void* packed, const float* pyr, const float* support, const uint8_t* track_valid, float* coords,
                float* vis, float* conf, const float* time_emb, int iters, const ct3_loop_shape* shape,
                void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (!packed || !pyr || !support || !coords || !vis || !conf || !time_emb || !workspace)
    return fail(CT3_EINVAL, "null argument%s");
  if (int rc = check_shape(shape, Use::kLoop)) return rc;
  if (iters < 0) return fail(CT3_EINVAL, "iters must be >= 0%s");
  if (int rc = check_aligned(workspace, "workspace")) return rc;
  const ct3_loop_shape& s = *shape;
  const int T = s.T, N = s.N, G = s.G, H4 = s.H4, W4 = s.W4, T_pyr = s.T_pyr > 0 ? s.T_pyr : s.T;
  const Workspace W = carve(workspace, s);
  if (int rc = check_space(workspace_bytes, W.total, "workspace")) return rc;
  const Layout& L = layout();
  Runner R{reinterpret_cast<const uint8_t*>(packed), L, stream, g_opt_gemm};
  GroupPlan gp;
  if (int rc = plan_groups(gp, s.group_sizes, G, T, N, s.group_T, W.groups, R.s)) return rc;
  std::vector<int32_t> track_len;   // group lengths: every track's, points then virtual tracks, and each point's group
  if (s.group_T) {
    track_len.resize((size_t)N + (size_t)kV * G);
    std::vector<int32_t> track_group((size_t)N);
    for (int g = 0, n0 = 0; g < G; ++g) {
      const int n = s.group_sizes ? s.group_sizes[g] : N;
      for (int i = 0; i < n; ++i) { track_len[n0 + i] = s.group_T[g]; track_group[n0 + i] = g; }
      for (int i = 0; i < kV; ++i) track_len[(size_t)N + (size_t)kV * g + i] = s.group_T[g];
      n0 += n;
    }
    CK(launch_upload_i32(W.track_len, track_len.data(), (int)track_len.size(), R.s), "upload track lengths");
    CK(launch_upload_i32(W.track_group, track_group.data(), N, R.s), "upload track groups");
    gp.track_len = W.track_len;
    gp.track_len_host = track_len.data();
  }
  FrameMap fm;
  if (s.T_pyr > 0) {   // the frame map reaches the device like the group table: in stream order, through kernel args
    CK(launch_upload_i32(W.frames, s.group_frames, G * T, R.s), "upload frame map");
    fm.frames = W.frames;
    fm.goff = G > 1 ? gp.off : nullptr;
    fm.G = G;
  }
  // split-bf16 copy of the pyramid: the TMA source of the correlation kernel, made once per call
  const Prec pr = effective_prec(W.pyr_split != nullptr, T_pyr, H4, W4);
  const __nv_bfloat16* pyr_split = (pr.patch && iters > 0) ? W.pyr_split : nullptr;
  if (pyr_split) RUNC(CAT_MISC, launch_split_pyramid(pyr, T_pyr, H4, W4, W.pyr_split, pr.corr, R.s));

  // W_in * time_emb[t]: x + time_emb is folded into a per-frame bias of input_transform (cotracker3_offline.py:196);
  // with group_T one [T, kC] block per group.  Each row is computed alone, so a block holds the bits a pass of the
  // group's own length computes
  RUNC(CAT_MISC, launch_row_bias(time_emb, reinterpret_cast<const float*>(R.pk + L.win_f32), s.group_T ? G * T : T,
                                 W.row_bias, R.s));

  for (int it = 0; it < iters; ++it) {
    // (i)-(iv) correlation, corr_mlp, X, input_transform -> point tokens
    if (int rc = point_tokens(R, W, pr, pyr, pyr_split, H4, W4, support, track_valid, coords, vis, conf, T, N, T_pyr,
                              fm))
      return rc;
    // transformer; (v) heads + state update
    if (int rc = transform_and_heads(R, W, T, N, gp, coords, vis, conf, nullptr)) return rc;
  }
  return 0;
}

// ct3_loop_tokens: the pyramid split, the time-embedding fold and point_tokens exactly as one update_loop iteration
// runs them (G = 1, no frame map), then copies of the volume, X and the point tokens.  Checks as update_loop.
int loop_tokens(const void* packed, const float* pyr, int H4, int W4, const float* support,
                const uint8_t* track_valid, const float* coords, const float* vis, const float* conf,
                const float* time_emb, int T, int N, void* vol_out, void* x_out, float* tokens_out, void* workspace,
                size_t workspace_bytes, cudaStream_t stream) {
  if (!packed || !pyr || !support || !coords || !vis || !conf || !time_emb || !workspace)
    return fail(CT3_EINVAL, "null argument%s");
  const ct3_loop_shape shape{T, N, H4, W4, 1, nullptr, 0, nullptr, 0, nullptr};
  if (int rc = check_shape(&shape, Use::kLoop)) return rc;
  if (int rc = check_aligned(workspace, "workspace")) return rc;
  const Workspace W = carve(workspace, shape);
  if (int rc = check_space(workspace_bytes, W.total, "workspace")) return rc;
  const Layout& L = layout();
  Runner R{reinterpret_cast<const uint8_t*>(packed), L, stream, g_opt_gemm};
  const Prec pr = effective_prec(W.pyr_split != nullptr, T, H4, W4);
  const __nv_bfloat16* pyr_split = pr.patch ? W.pyr_split : nullptr;
  if (pyr_split) RUNC(CAT_MISC, launch_split_pyramid(pyr, T, H4, W4, W.pyr_split, pr.corr, R.s));
  RUNC(CAT_MISC, launch_row_bias(time_emb, reinterpret_cast<const float*>(R.pk + L.win_f32), T, W.row_bias, R.s));
  if (int rc = point_tokens(R, W, pr, pyr, pyr_split, H4, W4, support, track_valid, coords, vis, conf, T, N, T,
                            FrameMap{}))
    return rc;
  const size_t Rp = (size_t)N * T;
  // the volume as ct3_corr_sample writes it: [Rp*4, 2*kVolPad] split bf16, or one fp16 plane [Rp*4, kVolPad]
  if (vol_out) CK(cudaMemcpyAsync(vol_out, W.vol, Rp * kL * kVolPad * (pr.vol16() ? 2 : 4), cudaMemcpyDeviceToDevice,
                                  R.s), "copy volume");
  if (x_out) CK(cudaMemcpyAsync(x_out, W.xs, Rp * 2 * kXPad * 2, cudaMemcpyDeviceToDevice, R.s), "copy X");
  if (tokens_out) CK(cudaMemcpyAsync(tokens_out, W.tokens, Rp * kC * 4, cudaMemcpyDeviceToDevice, R.s), "copy tokens");
  return 0;
}

int updateformer(const void* packed, const float* x, int T, int N, const int32_t* sizes, int G, float* delta,
                 void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (!packed || !x || !delta || !workspace) return fail(CT3_EINVAL, "null argument%s");
  const ct3_loop_shape shape{T, N, 0, 0, G, sizes, 0, nullptr, 0, nullptr};
  if (int rc = check_shape(&shape, Use::kFormer)) return rc;
  if (int rc = check_aligned(workspace, "workspace")) return rc;
  const Workspace W = carve(workspace, shape);
  if (int rc = check_space(workspace_bytes, W.total, "workspace")) return rc;
  Runner R{reinterpret_cast<const uint8_t*>(packed), layout(), stream, g_opt_gemm};
  GroupPlan gp;
  if (int rc = plan_groups(gp, sizes, G, T, N, nullptr, W.groups, R.s)) return rc;
  RUNC(CAT_MISC, launch_split_rows(x, N * T, kX, kXPad, /*perm_x*/ 1, W.xs, 0, R.s));
  if (int rc = input_transform(R, W, T, 0, N, nullptr)) return rc;
  return transform_and_heads(R, W, T, N, gp, nullptr, nullptr, nullptr, delta);
}

// ct3_attention: the split-K partials and the group table, the attention parts of carve()
Workspace carve_attention(void* base, int T, int N, int G) {
  Workspace w{};
  Carver c(base);
  w.att_part = (float*)c.take(attention_partial_bytes(T, kV, partial_slots(N, G)));
  w.groups = G > 1 ? (int32_t*)c.take((size_t)group_table_ints(N, G) * 4) : nullptr;
  w.total = c.off;
  return w;
}

// One attention of transformer_body on caller buffers of (N + kV*G)*T token rows, dispatched as the body does
int attention_stage(int kind, const float* q, const float* kv, int T, int N, const int32_t* sizes, int G, void* out,
                    void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (!q || !kv || !out || !workspace) return fail(CT3_EINVAL, "null argument%s");
  if (kind < CT3_ATTN_TIME || kind > CT3_ATTN_POINT_FROM_VIRTUAL) return fail(CT3_EINVAL, "unknown attention kind%s");
  const ct3_loop_shape shape{T, N, 0, 0, G, sizes, 0, nullptr, 0, nullptr};
  if (int rc = check_shape(&shape, Use::kFormer)) return rc;
  if (!sizes) return fail(CT3_EINVAL, "null group_sizes_host%s");
  if (((uintptr_t)q | (uintptr_t)kv | (uintptr_t)out) & 15) return fail(CT3_EINVAL, "q, kv and out must be 16-byte aligned%s");
  if (int rc = check_aligned(workspace, "workspace")) return rc;
  const Workspace W = carve_attention(workspace, T, N, G);
  if (int rc = check_space(workspace_bytes, W.total, "workspace")) return rc;
  Runner R{nullptr, layout(), stream, g_opt_gemm};
  const int64_t Rp = (int64_t)N * T;
  __nv_bfloat16* att = reinterpret_cast<__nv_bfloat16*>(out);
  if (kind == CT3_ATTN_TIME) {   // the unfused path of the time block: every track, points and virtual
    RUNC(CAT_ATTN, run_attention(R, W, attn_params(q, 3 * kC, kv, 3 * kC, kC, 2 * kC, att, T, T, T, N + kV * G), true));
    return 0;
  }
  GroupPlan gp;
  if (int rc = plan_groups(gp, sizes, G, T, N, nullptr, W.groups, R.s)) return rc;
  __nv_bfloat16* att_v = att + Rp * 2 * kC;
  if (kind == CT3_ATTN_VIRTUAL_FROM_POINT)
    RUNC(CAT_ATTN, space_attention(R, W, gp, attn_params(q + Rp * kC, kC, kv, 2 * kC, 0, kC, att_v, kV, N, T), false,
                                   true));
  else if (kind == CT3_ATTN_VIRTUAL_SELF)
    RUNC(CAT_ATTN, space_attention(R, W, gp, attn_params(q + Rp * 3 * kC, 3 * kC, kv + Rp * 3 * kC, 3 * kC, kC, 2 * kC,
                                                         att_v, kV, kV, T), false, false));
  else
    RUNC(CAT_ATTN, space_attention(R, W, gp, attn_params(q, kC, kv + Rp * 2 * kC, 2 * kC, 0, kC, att, N, kV, T), true,
                                   false));
  return 0;
}

// ct3_time_block_attention: the fp32 q|k|v of the unfused route, the only scratch time_attention reads
Workspace carve_time_block(void* base, int rows) {
  Workspace w{};
  Carver c(base);
  w.qkv = (float*)c.take((size_t)rows * 3 * kC * 4);
  w.total = c.off;
  return w;
}

int check_time_block(int T, int rows) {
  if (T < 1 || rows < 1 || rows % T) return fail(CT3_EINVAL, "need T >= 1, rows >= 1 and rows %% T == 0%s");
  return 0;
}

// q|k|v projection and attention of time block `depth` on caller buffers, routed as transformer_body routes it
int time_block_stage(const void* packed, int depth, const void* x_split, int T, int rows, void* out_split,
                     void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (!packed || !x_split || !out_split || !workspace) return fail(CT3_EINVAL, "null argument%s");
  if (depth < 0 || depth >= kDepth) return fail(CT3_EINVAL, "depth must be in [0, 3)%s");
  if (int rc = check_time_block(T, rows)) return rc;
  if (((uintptr_t)packed | (uintptr_t)x_split | (uintptr_t)out_split) & 15)
    return fail(CT3_EINVAL, "packed, x_split and out_split must be 16-byte aligned%s");
  if (int rc = check_aligned(workspace, "workspace")) return rc;
  const Workspace W = carve_time_block(workspace, rows);
  if (int rc = check_space(workspace_bytes, W.total, "workspace")) return rc;
  Runner R{reinterpret_cast<const uint8_t*>(packed), layout(), stream, g_opt_gemm};
  return time_attention(R, W, R.L.time[depth], reinterpret_cast<const __nv_bfloat16*>(x_split),
                        reinterpret_cast<__nv_bfloat16*>(out_split), rows, T);
}

}  // namespace

// ================================================================================================
extern "C" {

int ct3_volume_is_support_major(int T, int H4, int W4, int* flag) {
  if (!flag) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = check_pyramid(T, H4, W4)) return rc;
  *flag = effective_prec(true, T, H4, W4).support_major() ? 1 : 0;
  return 0;
}

int ct3_precision_info(int T, int H4, int W4, int* corr_products, int* fc1_products, int* volume_bytes_per_element) {
  if (int rc = check_pyramid(T, H4, W4)) return rc;
  const Prec pr = effective_prec(true, T, H4, W4);
  if (corr_products) *corr_products = pr.corr;
  if (fc1_products) *fc1_products = pr.fc1;
  if (volume_bytes_per_element) *volume_bytes_per_element = pr.vol16() ? 2 : 4;
  return 0;
}

int ct3_num_weight_tensors(void) { return (int)weight_names().size(); }
const char* ct3_weight_name(int index) {
  const auto& n = weight_names();
  if (index < 0 || index >= (int)n.size()) return nullptr;
  return n[index].c_str();
}

int ct3_packed_weights_bytes(size_t* out_bytes) {
  if (!out_bytes) return fail(CT3_EINVAL, "null out_bytes%s");
  *out_bytes = layout().total;
  return 0;
}

int ct3_pack_weights(const float* const* t, int n_tensors, void* packed, size_t packed_bytes, ct3_stream_t stream) {
  const Layout& L = layout();
  if (!t || !packed) return fail(CT3_EINVAL, "null argument%s");
  if (n_tensors != (int)weight_names().size()) return fail(CT3_EINVAL, "wrong number of weight tensors%s");
  if (int rc = check_space(packed_bytes, L.total, "packed buffer")) return rc;
  for (int i = 0; i < n_tensors; ++i)
    if (!t[i]) return fail(CT3_EINVAL, "null weight tensor: %s", weight_names()[i].c_str());
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* pk = reinterpret_cast<uint8_t*>(packed);
  CK(cudaMemsetAsync(pk, 0, L.total, s), "memset packed");
  auto put_lin = [&](const Lin& l, const float* w, const float* b, int rows, int row_off, int perm,
                     int fp16 = 0) -> cudaError_t {
    cudaError_t e = launch_split_rows(w, rows, l.K, l.Kpad, perm, reinterpret_cast<__nv_bfloat16*>(pk + l.w), row_off, s, fp16);
    if (e != cudaSuccess) return e;
    return cudaMemcpyAsync(pk + l.b + (size_t)row_off * 4, b, (size_t)rows * 4, cudaMemcpyDeviceToDevice, s);
  };
  auto put_f32 = [&](size_t off, const float* src, size_t count) {
    return cudaMemcpyAsync(pk + off, src, count * 4, cudaMemcpyDeviceToDevice, s);
  };
  int k = 0;
  CK(put_lin(L.corr_fc1, t[k], t[k + 1], kCorrHid, 0, 0), "pack corr_fc1");
  CK(put_lin(L.corr_fc1_h, t[k], t[k + 1], kCorrHid, 0, 0, /*fp16*/ 1), "pack corr_fc1 (fp16 planes)");
  CK(put_lin(L.corr_fc1_t, t[k], t[k + 1], kCorrHid, 0, /*volume transpose*/ 2), "pack corr_fc1 (support-major)");
  CK(put_lin(L.corr_fc1_th, t[k], t[k + 1], kCorrHid, 0, 2, /*fp16*/ 1), "pack corr_fc1 (support-major, fp16)"); k += 2;
  CK(put_lin(L.corr_fc2, t[k], t[k + 1], kCorrOut, 0, 0), "pack corr_fc2"); k += 2;
  CK(put_lin(L.in_tr, t[k], t[k + 1], kC, 0, /*perm_x*/ 1), "pack input_transform");
  CK(put_f32(L.win_f32, t[k], (size_t)kC * kX), "pack input_transform fp32"); k += 2;
  CK(put_f32(L.virt, t[k], (size_t)kV * kC), "pack virtual tracks"); k += 1;
  CK(put_f32(L.heads_w, t[k], 2 * kC), "pack flow_head.w");
  CK(put_f32(L.heads_b, t[k + 1], 2), "pack flow_head.b"); k += 2;
  CK(put_f32(L.heads_w + 2 * kC * 4, t[k], 2 * kC), "pack vis_conf_head.w");
  CK(put_f32(L.heads_b + 2 * 4, t[k + 1], 2), "pack vis_conf_head.b"); k += 2;
  auto put_self = [&](const Block& b) -> cudaError_t {
    cudaError_t e;
    if ((e = put_lin(b.q, t[k], t[k + 1], kC, 0, 0)) != cudaSuccess) return e;            // to_q  -> rows [0,384)
    if ((e = put_lin(b.q, t[k + 2], t[k + 3], 2 * kC, kC, 0)) != cudaSuccess) return e;   // to_kv -> rows [384,1152)
    if (b.qkv_h.N != 0) {   // per-head regrouping for the fused projection + time attention kernel
      for (int h = 0; h < kHeads; ++h) {
        const size_t wo = (size_t)h * kDh * kC;
        if ((e = put_lin(b.qkv_h, t[k] + wo, t[k + 1] + h * kDh, kDh, h * 3 * kDh, 0)) != cudaSuccess) return e;                         // q_h
        if ((e = put_lin(b.qkv_h, t[k + 2] + wo, t[k + 3] + h * kDh, kDh, h * 3 * kDh + kDh, 0)) != cudaSuccess) return e;               // k_h
        if ((e = put_lin(b.qkv_h, t[k + 2] + (size_t)kC * kC + wo, t[k + 3] + kC + h * kDh, kDh, h * 3 * kDh + 2 * kDh, 0)) != cudaSuccess) return e;   // v_h
      }
    }
    if ((e = put_lin(b.out, t[k + 4], t[k + 5], kC, 0, 0)) != cudaSuccess) return e;
    if ((e = put_lin(b.fc1, t[k + 6], t[k + 7], kMlpHid, 0, 0)) != cudaSuccess) return e;
    if ((e = put_lin(b.fc2, t[k + 8], t[k + 9], kC, 0, 0)) != cudaSuccess) return e;
    k += 10;
    return cudaSuccess;
  };
  auto put_cross = [&](const Block& b) -> cudaError_t {
    cudaError_t e;
    if ((e = put_f32(b.ctx_g, t[k], kC)) != cudaSuccess) return e;
    if ((e = put_f32(b.ctx_b, t[k + 1], kC)) != cudaSuccess) return e;
    if ((e = put_lin(b.q, t[k + 2], t[k + 3], kC, 0, 0)) != cudaSuccess) return e;
    if ((e = put_lin(b.kv, t[k + 4], t[k + 5], 2 * kC, 0, 0)) != cudaSuccess) return e;
    if ((e = put_lin(b.out, t[k + 6], t[k + 7], kC, 0, 0)) != cudaSuccess) return e;
    if ((e = put_lin(b.fc1, t[k + 8], t[k + 9], kMlpHid, 0, 0)) != cudaSuccess) return e;
    if ((e = put_lin(b.fc2, t[k + 10], t[k + 11], kC, 0, 0)) != cudaSuccess) return e;
    k += 12;
    return cudaSuccess;
  };
  for (int i = 0; i < kDepth; ++i) {
    CK(put_self(L.time[i]), "pack time block");
    CK(put_self(L.vself[i]), "pack virtual block");
    CK(put_cross(L.p2v[i]), "pack point2virtual block");
    CK(put_cross(L.v2p[i]), "pack virtual2point block");
  }
  return 0;
}

int ct3_workspace_bytes(const ct3_loop_shape* shape, size_t* out_bytes) {
  if (!out_bytes) return fail(CT3_EINVAL, "null out_bytes%s");
  if (int rc = check_shape(shape, Use::kSize)) return rc;
  *out_bytes = carve(nullptr, *shape).total;
  return 0;
}

int ct3_corr_sample(const float* pyr, int H4, int W4, const float* support, const uint8_t* track_valid,
                    const float* coords, int T, int N, void* vol_split, void* scratch, size_t scratch_bytes,
                    ct3_stream_t stream) {
  if (!pyr || !support || !coords || !vol_split) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = check_TN(T, N)) return rc;
  if (int rc = check_pyramid(T, H4, W4)) return rc;
  const __nv_bfloat16* pyr_split = nullptr;
  const Prec pr = effective_prec(scratch != nullptr, T, H4, W4);
  if (pr.patch) {
    if (int rc = check_aligned(scratch, "scratch")) return rc;
    if (int rc = check_space(scratch_bytes, (size_t)pyramid_layout(T, H4, W4).total * 4, "scratch")) return rc;
    CK(launch_split_pyramid(pyr, T, H4, W4, (__nv_bfloat16*)scratch, pr.corr, (cudaStream_t)stream), "split_pyramid");
    pyr_split = (const __nv_bfloat16*)scratch;
  }
  CK(launch_corr_sample(pyr, pyr_split, H4, W4, support, track_valid, coords, T, N, 0, N, (__nv_bfloat16*)vol_split,
                        g_opt_corr, pr.corr, pr.vol16() ? 1 : 0, num_sms(), (cudaStream_t)stream, T, FrameMap{}),
     "corr_sample");
  return 0;
}

int ct3_linear(const void* x_split, const void* w_split, const float* bias, int M, int Nout, int Kpad, int act,
               float* y, ct3_stream_t stream) {
  return ct3_linear_ex(x_split, 0, w_split, bias, M, Nout, Kpad, 3, 0, act, nullptr, 1, y, Nout, 0, nullptr, 0, 0, 1,
                       stream);
}

int ct3_linear_prec(const void* x_split, const void* w_split, const float* bias, int M, int Nout, int Kpad, int act,
                    int products, int fp16, float* y, ct3_stream_t stream) {
  return ct3_linear_ex(x_split, 0, w_split, bias, M, Nout, Kpad, products, fp16, act, nullptr, 1, y, Nout, 0, nullptr,
                       0, 0, 1, stream);
}

int ct3_linear_ex(const void* x_split, int64_t x_ld, const void* w_split, const float* bias, int M, int Nout, int Kpad,
                  int products, int fp16, int act, const float* row_bias, int row_mod, float* y, int64_t ld_y,
                  int residual, void* y_split, int64_t ld_split, int lo_off, int row_group, ct3_stream_t stream) {
  if (!x_split || !w_split) return fail(CT3_EINVAL, "null argument%s");
  if (residual != 0 && (residual != 1 || !y)) return fail(CT3_EINVAL, "ct3_linear: residual is 0, or 1 with y%s");
  GemmProblem p = linear_problem(x_split, w_split, bias, M, Nout, Kpad, y);
  p.x_ld = x_ld;
  p.products = products;
  p.fp16 = fp16;
  p.epi.act = act;
  p.epi.row_bias = row_bias;
  p.epi.row_mod = row_mod;
  p.epi.ld_f32 = ld_y;
  p.epi.residual = residual;
  p.epi.out_split = static_cast<__nv_bfloat16*>(y_split);
  p.epi.ld_split = ld_split;
  p.epi.lo_off = lo_off;
  p.epi.row_group = row_group;
  return run_gemm(p, g_opt_gemm, (cudaStream_t)stream, "ct3_linear");
}

int ct3_time_block_attention_workspace_bytes(int T, int rows, size_t* out_bytes) {
  if (!out_bytes) return fail(CT3_EINVAL, "null out_bytes%s");
  if (int rc = check_time_block(T, rows)) return rc;
  *out_bytes = carve_time_block(nullptr, rows).total;
  return 0;
}

int ct3_time_block_attention(const void* packed, int depth, const void* x_split, int T, int rows, void* out_split,
                             void* workspace, size_t workspace_bytes, ct3_stream_t stream) {
  return time_block_stage(packed, depth, x_split, T, rows, out_split, workspace, workspace_bytes, (cudaStream_t)stream);
}

int ct3_layernorm(const float* x, int rows, const float* gamma, const float* beta, float eps, void* out_split,
                  ct3_stream_t stream) {
  if (!x || !out_split) return fail(CT3_EINVAL, "null argument%s");
  if ((gamma == nullptr) != (beta == nullptr)) return fail(CT3_EINVAL, "gamma and beta must be given together%s");
  if (rows < 1) return fail(CT3_EINVAL, "rows must be >= 1%s");
  if (!(eps >= 0.f && eps <= 1e30f)) return fail(CT3_EINVAL, "eps must be finite and >= 0%s");
  if (((uintptr_t)x | (uintptr_t)gamma | (uintptr_t)beta | (uintptr_t)out_split) & 15)
    return fail(CT3_EINVAL, "x, gamma, beta and out_split must be 16-byte aligned%s");
  CK(launch_layernorm_split(x, rows, gamma, beta, eps, static_cast<__nv_bfloat16*>(out_split), (cudaStream_t)stream),
     "layernorm");
  return 0;
}

int ct3_update_loop(const void* packed, const float* pyr, const float* support, const uint8_t* track_valid,
                    float* coords, float* vis, float* conf, const float* time_emb, int iters,
                    const ct3_loop_shape* shape, void* workspace, size_t workspace_bytes, ct3_stream_t stream) {
  return update_loop(packed, pyr, support, track_valid, coords, vis, conf, time_emb, iters, shape, workspace,
                     workspace_bytes, (cudaStream_t)stream);
}

int ct3_loop_tokens(const void* packed, const float* pyr, int H4, int W4, const float* support,
                    const uint8_t* track_valid, const float* coords, const float* vis, const float* conf,
                    const float* time_emb, int T, int N, void* vol_out, void* x_out, float* tokens_out,
                    void* workspace, size_t workspace_bytes, ct3_stream_t stream) {
  return loop_tokens(packed, pyr, H4, W4, support, track_valid, coords, vis, conf, time_emb, T, N, vol_out, x_out,
                     tokens_out, workspace, workspace_bytes, (cudaStream_t)stream);
}

int ct3_updateformer(const void* packed, const float* x, int T, int N, const int32_t* group_sizes_host, int G,
                     float* delta, void* workspace, size_t workspace_bytes, ct3_stream_t stream) {
  return updateformer(packed, x, T, N, group_sizes_host, G, delta, workspace, workspace_bytes, (cudaStream_t)stream);
}

int ct3_attention_workspace_bytes(int T, int N, int G, size_t* out_bytes) {
  if (!out_bytes) return fail(CT3_EINVAL, "null out_bytes%s");
  if (int rc = check_TN(T, N, G)) return rc;
  *out_bytes = carve_attention(nullptr, T, N, G).total;
  return 0;
}

int ct3_attention(int kind, const float* q, const float* kv, int T, int N, const int32_t* group_sizes_host, int G,
                  void* out_split, void* workspace, size_t workspace_bytes, ct3_stream_t stream) {
  return attention_stage(kind, q, kv, T, N, group_sizes_host, G, out_split, workspace, workspace_bytes,
                         (cudaStream_t)stream);
}

}  // extern "C"
