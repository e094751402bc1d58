// api.cu -- C ABI of libct3_b200.so (see include/ct3_b200.h): weight packing, workspace carving and the
// launch sequence of one refinement iteration (cotracker3_offline.py:139-216, cotracker.py:483-531).
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <string>
#include <vector>

#include "../../include/ct3_b200.h"
#include "gemm.cuh"
#include "kernels.cuh"

using namespace ct3;

namespace {

thread_local char g_err[512] = "";
// Options and the profiler are PER HOST THREAD (thread_local): a thread that drives its own GPU/stream never sees
// another thread's verification switches or profile records.
struct OptDef { const char* name; int lo, hi; };
enum { OPT_GEMM = 0, OPT_CORR, OPT_ATTN, OPT_PREC_CORR, OPT_PREC_FC1, OPT_FUSE, OPT_COUNT };
constexpr int kDefPrecCorr = 2, kDefPrecFc1 = 3;   // DESIGN.md section 2
constexpr OptDef kOptDefs[OPT_COUNT] = {
    {"gemm", 0, 1},   // 0 wgmma, 1 SIMT verification
    {"corr", 0, 3},   // 0 wgmma correlate-then-interpolate (corr_tc3.cu / corr_tc2.cu), 1 exact-fp32 SIMT, 2 corr_tc.cu,
                      // 3 correlate-then-interpolate with corr_tc2.cu for every precision mode (A/B)
    {"attn", 0, 2},   // 0 tensor-core kernels (wgmma point<-virtual, mma.sync elsewhere), 1 exact-fp32 SIMT verification,
                      // 2 = mma.sync for point<-virtual too (A/B against attention_p2v.cu)
    // tensor-core products per FLOP of a GEMM group (DESIGN.md section 2): 3 = split x split (hi*hi + lo*hi + hi*lo),
    // 2 = fp16 activation plane x split fp16 weights, 1 = single fp16 product.  Only the correlation branch has the
    // switch: SURVEY 7.3 measured that every transformer GEMM breaks the 1e-3 px budget with fewer than 3 products.
    {"prec.corr", 1, 3},   // the 49x128x49 correlation contraction (corr_tc2.cu)
    {"prec.fc1", 1, 3},    // corr_mlp.fc1 (K = 2401): 1|2 also make the correlation volume a single fp16 plane
    // 0: separate LayerNorm / projection / attention kernels; 1: q|k|v projection + time attention in one kernel
    // (gemm_qkv_time_attn_kernel); 2: additionally every LayerNorm folded into the GEMMs around it (no LN kernels)
    {"fuse", 0, 2},
};
thread_local int g_opt[OPT_COUNT] = {0, 0, 0, kDefPrecCorr, kDefPrecFc1, 1};   // fuse = 2 measured slower (DESIGN.md 4.6)
#define g_opt_gemm g_opt[OPT_GEMM]
#define g_opt_corr g_opt[OPT_CORR]
#define g_opt_attn g_opt[OPT_ATTN]

int fail(int code, const char* fmt, const char* detail = "") {
  snprintf(g_err, sizeof(g_err), fmt, detail);
  return code;
}
int fail_cuda(cudaError_t e, const char* where) {
  snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
  return CT3_ECUDA;
}
#define CK(call, where)                                  \
  do {                                                   \
    cudaError_t e__ = (call);                            \
    if (e__ != cudaSuccess) return fail_cuda(e__, where); \
  } while (0)

int num_sms() {   // of the CURRENT device (one process may drive several GPUs)
  static std::atomic<int> cache[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev >= 0 && dev < 64) {
    const int c = cache[dev].load(std::memory_order_relaxed);
    if (c > 0) return c;
  }
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  if (dev >= 0 && dev < 64) cache[dev].store(n, std::memory_order_relaxed);
  return n;
}


// ------------------------------------------------------------------------------------------------
// optional live profiler: CUDA events around every launch, summed per kernel category (bench.py roofline)
enum { CAT_CORR = 0, CAT_GEMM = 1, CAT_ATTN = 2, CAT_LN = 3, CAT_MISC = 4, CAT_ENC = 5, CAT_QKVA = 6, CAT_COUNT = 7 };
struct ProfRec { int cat; cudaEvent_t a, b; double flops; int launches; };
thread_local bool g_prof_on = false;
thread_local std::vector<ProfRec> g_prof;
struct ProfScope {
  cudaStream_t s; int cat; double flops; int launches; cudaEvent_t a = nullptr, b = nullptr;
  ProfScope(cudaStream_t s_, int cat_, double flops_ = 0.0, int launches_ = 1)
      : s(s_), cat(cat_), flops(flops_), launches(launches_) {
    if (g_prof_on && cat_ >= 0) { cudaEventCreate(&a); cudaEventCreate(&b); cudaEventRecord(a, s); }
  }
  ~ProfScope() {
    if (a) { cudaEventRecord(b, s); g_prof.push_back({cat, a, b, flops, launches}); }
  }
};

size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// ------------------------------------------------------------------------------------------------
// packed-weights layout
struct Lin {
  size_t w = 0, b = 0;  // byte offsets: split weights [N, 2*Kpad] bf16 ; bias [N] fp32
  size_t ws = 0;        // fp32 [N]: sum_k W[n][k], the correction vector of a LayerNorm folded into this layer
  int N = 0, K = 0, Kpad = 0;
};
struct Block {
  Lin qkv_h;  // time blocks only: q|k|v regrouped per head, rows h*144 + [q_h(48) | k_h(48) | v_h(48)] (fused attention)
  Lin q;    // self-attention blocks: fused q|k|v (N = 1152); cross blocks: to_q (N = 384)
  Lin kv;   // cross blocks only: to_kv (N = 768)
  Lin kv_f; // cross blocks only: to_kv with the affine norm_context folded in (W diag(gamma), b + W beta)
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
  size_t scratch = 0;   // pack-time scratch: one folded to_kv weight [768, 384] + bias [768] in fp32
  size_t total = 0;
};

int pad64(int k) { return (k + 63) / 64 * 64; }

void place_lin(Lin& l, int N, int K, size_t& off) {
  l.N = N;
  l.K = K;
  l.Kpad = pad64(K);
  l.w = off;
  off = align_up(off + (size_t)N * 2 * l.Kpad * sizeof(__nv_bfloat16));
  l.b = off;
  off = align_up(off + (size_t)N * sizeof(float));
  l.ws = off;
  off = align_up(off + (size_t)N * sizeof(float));
}
void place_block(Block& b, bool cross, size_t& off, bool time = false) {
  b.cross = cross;
  if (time) place_lin(b.qkv_h, 3 * kC, kC, off);
  if (cross) {
    b.ctx_g = off; off = align_up(off + kC * sizeof(float));
    b.ctx_b = off; off = align_up(off + kC * sizeof(float));
    place_lin(b.q, kC, kC, off);
    place_lin(b.kv, 2 * kC, kC, off);
    place_lin(b.kv_f, 2 * kC, kC, off);
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
    L.scratch = off;
    off = align_up(off + (size_t)2 * kC * kC * sizeof(float) + (size_t)2 * kC * sizeof(float));
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
// workspace
struct Workspace {
  __nv_bfloat16* vol;     // [N*T*4, 2*2432]
  __nv_bfloat16* h1;      // [N*T*4, 2*384]
  __nv_bfloat16* xs;      // [N*T, 2*1152]
  float* tokens;          // [(N+64)*T, 384]
  __nv_bfloat16* traw;    // [(N+64)*T, 2*384]  the token rows once more as a split operand (LayerNorm fold)
  float* tstat;           // [(N+64)*T, 24, 2]  partial (sum, sum of squares) of every token row
  __nv_bfloat16* ln;      // [(N+64)*T, 2*384]
  __nv_bfloat16* att;     // [(N+64)*T, 2*384]
  float* qkv;             // [(N+64)*T, 1152]   (also point q [N*T,384] / point kv [N*T,768])
  float* vqkv;            // [64*T, 1152]       (virtual q / kv / qkv)
  __nv_bfloat16* hmid;    // [(N+64)*T, 2*1536]
  float* row_bias;        // [T, 384]
  float* att_part;        // split-K partials of the virtual<-point attention
  __nv_bfloat16* pyr_split;  // split-bf16 copy of the pyramid (corr_tc2.cu); null when H4 == 0
  int32_t* groups;        // device group table of a grouped call (GroupPlan); null when G == 1
  int32_t* frames;        // device frame map [G, T] of ct3_update_loop_frames; null without one
  size_t total;
};
// split-K slots of the virtual<-point partials: a group of n tracks splits at most min(32, ceil(n/64)/2) ways
// (attention_tc_splits), so G groups of N tracks in all need at most (N + 63 G)/128 slots beyond one group's 32
int partial_slots(int N, int G) {
  if (G == 1) return kAttnMaxSplits;
  const int64_t s = kAttnMaxSplits + ((int64_t)N + 63LL * G) / 128;
  return (int)(s < (int64_t)kAttnMaxSplits * G ? s : (int64_t)kAttnMaxSplits * G);
}
// int32 entries of the group table: offsets [G+1] | all [G] | split [G] | slot [G] | small [G] | tiles [2 * max tiles]
int64_t group_table_ints(int N, int G) { return G == 1 ? 0 : (int64_t)5 * G + 1 + 2 * ((int64_t)N / 128 + G); }

// T_pyr: frames of the pyramid the correlation reads (sizes the split copy; 0 = T); frames: room for a [G, T] frame map
Workspace carve(void* base, int T, int N, int H4 = 0, int W4 = 0, int G = 1, int T_pyr = 0, bool frames = false) {
  Workspace w;
  if (T_pyr == 0) T_pyr = T;
  const size_t R = (size_t)(N + (size_t)kV * G) * T, Rp = (size_t)N * T, Rv = (size_t)kV * G * T, Mc = Rp * kL;
  uint8_t* p = reinterpret_cast<uint8_t*>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) { uint8_t* r = p + off; off = align_up(off + bytes, 1024); return r; };
  w.vol = (__nv_bfloat16*)take(Mc * 2 * kVolPad * 2);
  w.h1 = (__nv_bfloat16*)take(Mc * 2 * kCorrHid * 2);
  w.xs = (__nv_bfloat16*)take(Rp * 2 * kXPad * 2);
  w.tokens = (float*)take(R * kC * 4);
  w.traw = (__nv_bfloat16*)take(R * 2 * kC * 2);
  w.tstat = (float*)take(R * kLnParts * 2 * 4);
  w.ln = (__nv_bfloat16*)take(R * 2 * kC * 2);
  w.att = (__nv_bfloat16*)take(R * 2 * kC * 2);
  w.qkv = (float*)take(R * 3 * kC * 4);
  w.vqkv = (float*)take(Rv * 3 * kC * 4);
  w.hmid = (__nv_bfloat16*)take(R * 2 * kMlpHid * 2);
  w.row_bias = (float*)take((size_t)T * kC * 4);
  w.att_part = (float*)take(attention_partial_bytes(T, kV, partial_slots(N, G)));
  w.pyr_split = nullptr;
  if (H4 > 0 && W4 > 0 && corr_patch_supported(T_pyr, H4, W4))
    w.pyr_split = (__nv_bfloat16*)take((size_t)pyramid_layout(T_pyr, H4, W4).total * 4);
  w.groups = G > 1 ? (int32_t*)take((size_t)group_table_ints(N, G) * 4) : nullptr;
  w.frames = frames ? (int32_t*)take((size_t)G * T * 4) : nullptr;
  w.total = off;
  return w;
}

// ------------------------------------------------------------------------------------------------
struct Runner {
  const uint8_t* pk;
  const Layout& L;
  cudaStream_t s;
  int impl;
  const char* gerr = nullptr;

  int gemm(const __nv_bfloat16* x, const Lin& lin, int M, const GemmEpilogue& e, int products = 3, int fp16 = 0,
           int64_t x_ld = 0) {
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
    return gemm_launch(p, impl, num_sms(), s, &gerr);
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

#define RUNC(cat, call)                                                                  \
  do {                                                                                   \
    int rc__;                                                                            \
    { ProfScope ps__(R.s, cat); rc__ = (int)(call); }                                    \
    if (rc__ != 0) {                                                                     \
      snprintf(g_err, sizeof(g_err), "%s failed: %s (%s)", #call,                        \
               cudaGetErrorString((cudaError_t)rc__), R.gerr ? R.gerr : "");             \
      return CT3_ECUDA;                                                                  \
    }                                                                                    \
  } while (0)

int run_attention(Runner& R, const Workspace& W, const AttnParams& a, bool per_warp) {
  if (g_opt_attn == 1) return (int)launch_attention(a, R.s);
  // point <- virtual (64 keys per frame, thousands of queries): wgmma kernel with TMA row staging (attention_p2v.cu)
  if (g_opt_attn == 0 && !per_warp && a.Lq > kV && attention_p2v_supported(a)) return (int)launch_attention_p2v(a, R.s);
  return (int)launch_attention_tc(a, per_warp, W.att_part, num_sms(), R.s);
}

// Track groups of a grouped call (ct3_update_loop_groups): G contiguous track ranges, each with its own kV virtual
// tokens at rows (N + kV*g + i)*T + t.  G == 1 is the plain call (no table; every kernel indexes as it always did).
// For G > 1 the host builds the table below, uploads it into the workspace in stream order, and each space attention
// runs over (group, frame) sequences, choosing per group what a standalone call on that group's tracks would.
struct GroupPlan {
  int G = 1, max_n = 0;
  const int32_t *off = nullptr, *all = nullptr, *split = nullptr, *slot = nullptr, *small = nullptr, *tile = nullptr;
  int n_small = 0, n_tiles = 0, split_max = 1, split_slots = 0;
};

int plan_groups(GroupPlan& gp, const int32_t* sizes, int G, int T, int N, int32_t* dev, cudaStream_t s) {
  gp.G = G;
  if (G == 1) return 0;
  std::vector<int32_t> h((size_t)group_table_ints(N, G), 0);
  int32_t* off = h.data();
  int32_t *all = off + G + 1, *split = all + G, *slot = split + G, *small = slot + G, *tile = small + G;
  const int nsm = num_sms();
  for (int g = 0; g < G; ++g) {
    const int n = sizes[g];
    off[g + 1] = off[g] + n;
    if (n > gp.max_n) gp.max_n = n;
    all[g] = g;
    // virtual <- point: the split-K count of a standalone call (T sequences of kV queries over n keys)
    split[g] = attention_tc_splits(T, kV, n, nsm);
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
  if (gp.G == 1) return run_attention(R, W, a, false);
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

// x += to_out(attn(...)); x += mlp(LN(x))   for the rows [row0, row0+rows) of the token buffer
int mlp_half(Runner& R, const Workspace& W, const Block& b, int64_t row0, int rows) {
  float* x = W.tokens + row0 * kC;
  __nv_bfloat16* ln = W.ln + row0 * 2 * kC;
  __nv_bfloat16* hm = W.hmid + row0 * 2 * kMlpHid;
  RUNC(CAT_LN, launch_layernorm_split(x, rows, nullptr, nullptr, 1e-6f, ln, R.s));
  RUNC(-1, R.gemm(ln, b.fc1, rows, Runner::to_split(hm, 2 * kMlpHid, kMlpHid, /*tanh*/ 2)));
  RUNC(-1, R.gemm(hm, b.fc2, rows, Runner::to_f32(x, kC, true)));
  return 0;
}

// EfficientUpdateFormer body on W.tokens (point rows already hold input_transform output) -- cotracker.py:486-524
int transformer_body(Runner& R, const Workspace& W, int T, int N, const GroupPlan& gp) {
  const Layout& L = R.L;
  const int Rp = N * T, Rv = kV * gp.G * T, Rall = Rp + Rv;
  const float scale = 1.0f / sqrtf((float)kDh);
  const uint8_t* pk = R.pk;
  RUNC(CAT_MISC, launch_init_virtual(W.tokens, reinterpret_cast<const float*>(pk + L.virt), T, N, gp.G, R.s));
  float* vtok = W.tokens + (int64_t)Rp * kC;
  __nv_bfloat16* ln_p = W.ln;
  __nv_bfloat16* ln_v = W.ln + (int64_t)Rp * 2 * kC;
  __nv_bfloat16* att_p = W.att;
  __nv_bfloat16* att_v = W.att + (int64_t)Rp * 2 * kC;

  for (int i = 0; i < kDepth; ++i) {
    {  // ---- time block over every token row (points + virtual): sequence = track (cotracker.py:494-495)
      const Block& b = L.time[i];
      RUNC(CAT_LN, launch_layernorm_split(W.tokens, Rall, nullptr, nullptr, 1e-6f, W.ln, R.s));
      if (g_opt[OPT_FUSE] >= 1 && R.impl == 0 && g_opt_attn != 1 && qkv_time_attn_supported(T)) {
        // q|k|v projection and the per-track T x T attention in ONE kernel: fp32 q|k|v never reaches HBM
        ProfScope ps(R.s, CAT_QKVA, 0.0);
        int rc = gemm_qkv_time_attn_launch(W.ln, reinterpret_cast<const __nv_bfloat16*>(pk + b.qkv_h.w),
                                           reinterpret_cast<const float*>(pk + b.qkv_h.b), Rall, kC, T, W.att, 2 * kC,
                                           kC, scale, nullptr, nullptr, 0.f, num_sms(), R.s, &R.gerr);
        if (rc != 0) {
          snprintf(g_err, sizeof(g_err), "fused qkv + time attention failed: %s (%s)",
                   cudaGetErrorString((cudaError_t)rc), R.gerr ? R.gerr : "");
          return CT3_ECUDA;
        }
      } else {
        RUNC(-1, R.gemm(W.ln, b.q, Rall, Runner::to_f32(W.qkv, 3 * kC, false)));
        AttnParams a{};
        a.q = W.qkv; a.q_ld = 3 * kC; a.q_col = 0;
        a.kv = W.qkv; a.kv_ld = 3 * kC; a.k_col = kC; a.v_col = 2 * kC;
        a.out = W.att; a.out_ld = 2 * kC; a.lo_off = kC;
        a.num_seq = N + kV * gp.G; a.Lq = T; a.Lk = T;
        a.q_seq_stride = T; a.q_tok_stride = 1; a.k_seq_stride = T; a.k_tok_stride = 1;
        a.scale = scale;
        RUNC(CAT_ATTN, run_attention(R, W, a, true));
      }
      RUNC(-1, R.gemm(W.att, b.out, Rall, Runner::to_f32(W.tokens, kC, true)));
      if (int rc = mlp_half(R, W, b, 0, Rall)) return rc;
    }
    {  // ---- virtual <- point cross attention (cotracker.py:510-512): x = virtual, context = points
      const Block& b = L.v2p[i];
      RUNC(CAT_LN, launch_layernorm_split(vtok, Rv, nullptr, nullptr, 1e-6f, ln_v, R.s));
      RUNC(CAT_LN, launch_layernorm_split(W.tokens, Rp, reinterpret_cast<const float*>(pk + b.ctx_g),
                                 reinterpret_cast<const float*>(pk + b.ctx_b), 1e-5f, ln_p, R.s));
      RUNC(-1, R.gemm(ln_v, b.q, Rv, Runner::to_f32(W.vqkv, kC, false)));
      RUNC(-1, R.gemm(ln_p, b.kv, Rp, Runner::to_f32(W.qkv, 2 * kC, false)));
      AttnParams a{};
      a.q = W.vqkv; a.q_ld = kC; a.q_col = 0;
      a.kv = W.qkv; a.kv_ld = 2 * kC; a.k_col = 0; a.v_col = kC;
      a.out = att_v; a.out_ld = 2 * kC; a.lo_off = kC;
      a.num_seq = T; a.Lq = kV; a.Lk = N;
      a.q_seq_stride = 1; a.q_tok_stride = T; a.k_seq_stride = 1; a.k_tok_stride = T;
      a.scale = scale;
      RUNC(CAT_ATTN, space_attention(R, W, gp, a, false, true));
      RUNC(-1, R.gemm(att_v, b.out, Rv, Runner::to_f32(vtok, kC, true)));
      if (int rc = mlp_half(R, W, b, Rp, Rv)) return rc;
    }
    {  // ---- virtual self attention (cotracker.py:514): sequence = frame over the 64 virtual tokens
      const Block& b = L.vself[i];
      RUNC(CAT_LN, launch_layernorm_split(vtok, Rv, nullptr, nullptr, 1e-6f, ln_v, R.s));
      RUNC(-1, R.gemm(ln_v, b.q, Rv, Runner::to_f32(W.vqkv, 3 * kC, false)));
      AttnParams a{};
      a.q = W.vqkv; a.q_ld = 3 * kC; a.q_col = 0;
      a.kv = W.vqkv; a.kv_ld = 3 * kC; a.k_col = kC; a.v_col = 2 * kC;
      a.out = att_v; a.out_ld = 2 * kC; a.lo_off = kC;
      a.num_seq = T; a.Lq = kV; a.Lk = kV;
      a.q_seq_stride = 1; a.q_tok_stride = T; a.k_seq_stride = 1; a.k_tok_stride = T;
      a.scale = scale;
      RUNC(CAT_ATTN, space_attention(R, W, gp, a, false, false));
      RUNC(-1, R.gemm(att_v, b.out, Rv, Runner::to_f32(vtok, kC, true)));
      if (int rc = mlp_half(R, W, b, Rp, Rv)) return rc;
    }
    {  // ---- point <- virtual cross attention (cotracker.py:515-517): x = points, context = virtual
      const Block& b = L.p2v[i];
      RUNC(CAT_LN, launch_layernorm_split(W.tokens, Rp, nullptr, nullptr, 1e-6f, ln_p, R.s));
      RUNC(CAT_LN, launch_layernorm_split(vtok, Rv, reinterpret_cast<const float*>(pk + b.ctx_g),
                                 reinterpret_cast<const float*>(pk + b.ctx_b), 1e-5f, ln_v, R.s));
      RUNC(-1, R.gemm(ln_p, b.q, Rp, Runner::to_f32(W.qkv, kC, false)));
      RUNC(-1, R.gemm(ln_v, b.kv, Rv, Runner::to_f32(W.vqkv, 2 * kC, false)));
      AttnParams a{};
      a.q = W.qkv; a.q_ld = kC; a.q_col = 0;
      a.kv = W.vqkv; a.kv_ld = 2 * kC; a.k_col = 0; a.v_col = kC;
      a.out = att_p; a.out_ld = 2 * kC; a.lo_off = kC;
      a.num_seq = T; a.Lq = N; a.Lk = kV;
      a.q_seq_stride = 1; a.q_tok_stride = T; a.k_seq_stride = 1; a.k_tok_stride = T;
      a.scale = scale;
      RUNC(CAT_ATTN, space_attention(R, W, gp, a, true, false));
      RUNC(-1, R.gemm(att_p, b.out, Rp, Runner::to_f32(W.tokens, kC, true)));
      if (int rc = mlp_half(R, W, b, 0, Rp)) return rc;
    }
  }
  return 0;
}

// effective precision of the correlation branch for this thread's options: the single-plane / fewer-product modes
// exist in corr_tc2.cu only, so whenever another correlation kernel runs the branch computes split x split
struct Prec {
  int corr, fc1; bool patch;
  bool vol16() const { return fc1 < 3; }
  bool support_major() const { return patch && corr != 3 && g_opt_corr == 0; }   // corr_tc3.cu writes k*49 + i
};
Prec effective_prec(bool have_pyr_split, int T, int H4, int W4) {
  Prec p;
  p.patch = corr_uses_patch_kernel(g_opt_corr, have_pyr_split, T, H4, W4);
  p.corr = p.patch ? g_opt[OPT_PREC_CORR] : 3;
  p.fc1 = p.patch ? g_opt[OPT_PREC_FC1] : 3;
  return p;
}

// LayerNorm-folded variant of transformer_body (option fuse = 2, tensor-core kernels, T <= 128): no LayerNorm kernel
// runs.  Every GEMM that writes token rows (input_transform, to_out, mlp.fc2) also emits them as a split-bf16 operand
// plus partial row statistics (GemmEpilogue::raw_split / stat_part); every GEMM that consumes LN(x) multiplies the
// RAW rows and applies  rstd * (W.x - mean * wsum) + b  in its epilogue; the affine norm_context of the cross blocks
// (cotracker.py:539-540) is folded into to_kv's weights and bias at pack time (Block::kv_f).
bool fold_enabled(const Runner& R, int T) {
  return g_opt[OPT_FUSE] == 2 && R.impl == 0 && g_opt_attn != 1 && qkv_time_attn_supported(T);
}

int transformer_body_fold(Runner& R, const Workspace& W, int T, int N) {
  const Layout& L = R.L;
  const int Rp = N * T, Rv = kV * T, Rall = Rp + Rv;
  const float scale = 1.0f / sqrtf((float)kDh);
  const uint8_t* pk = R.pk;
  RUNC(CAT_MISC, launch_init_virtual(W.tokens, reinterpret_cast<const float*>(pk + L.virt), T, N, 1, R.s));
  float* vtok = W.tokens + (int64_t)Rp * kC;
  __nv_bfloat16* raw_p = W.traw;
  __nv_bfloat16* raw_v = W.traw + (int64_t)Rp * 2 * kC;
  float* st_p = W.tstat;
  float* st_v = W.tstat + (int64_t)Rp * kLnParts * 2;
  __nv_bfloat16* att_p = W.att;
  __nv_bfloat16* att_v = W.att + (int64_t)Rp * 2 * kC;
  RUNC(CAT_LN, launch_rowstats_split(vtok, Rv, raw_v, st_v, R.s));
  auto ln = [&](GemmEpilogue e, const float* part, const Lin& lin, float eps) {
    e.ln_part = part; e.ln_wsum = reinterpret_cast<const float*>(pk + lin.ws); e.ln_eps = eps;
    return e;
  };
  auto prod = [&](GemmEpilogue e, __nv_bfloat16* raw, float* stat) { e.raw_split = raw; e.stat_part = stat; return e; };
  // x += mlp(LN(x)) on rows [row0, row0 + rows)
  auto mlp = [&](const Block& b, int64_t row0, int rows) -> int {
    float* x = W.tokens + row0 * kC;
    __nv_bfloat16* raw = W.traw + row0 * 2 * kC;
    float* st = W.tstat + row0 * kLnParts * 2;
    __nv_bfloat16* hm = W.hmid + row0 * 2 * kMlpHid;
    RUNC(-1, R.gemm(raw, b.fc1, rows, ln(Runner::to_split(hm, 2 * kMlpHid, kMlpHid, /*tanh*/ 2), st, b.fc1, 1e-6f)));
    RUNC(-1, R.gemm(hm, b.fc2, rows, prod(Runner::to_f32(x, kC, true), raw, st)));
    return 0;
  };
  auto attention = [&](const float* q, int q_ld, const float* kv, int kv_ld, int k_col, int v_col, __nv_bfloat16* out,
                       int Lq, int Lk) -> int {
    AttnParams a{};
    a.q = q; a.q_ld = q_ld; a.q_col = 0;
    a.kv = kv; a.kv_ld = kv_ld; a.k_col = k_col; a.v_col = v_col;
    a.out = out; a.out_ld = 2 * kC; a.lo_off = kC;
    a.num_seq = T; a.Lq = Lq; a.Lk = Lk;
    a.q_seq_stride = 1; a.q_tok_stride = T; a.k_seq_stride = 1; a.k_tok_stride = T;
    a.scale = scale;
    RUNC(CAT_ATTN, run_attention(R, W, a, false));
    return 0;
  };
  for (int i = 0; i < kDepth; ++i) {
    {  // ---- time block (cotracker.py:494-495)
      const Block& b = L.time[i];
      {
        ProfScope ps(R.s, CAT_QKVA, 0.0);
        int rc = gemm_qkv_time_attn_launch(W.traw, reinterpret_cast<const __nv_bfloat16*>(pk + b.qkv_h.w),
                                           reinterpret_cast<const float*>(pk + b.qkv_h.b), Rall, kC, T, W.att, 2 * kC,
                                           kC, scale, W.tstat, reinterpret_cast<const float*>(pk + b.qkv_h.ws), 1e-6f,
                                           num_sms(), R.s, &R.gerr);
        if (rc != 0) {
          snprintf(g_err, sizeof(g_err), "fused qkv + time attention failed: %s (%s)",
                   cudaGetErrorString((cudaError_t)rc), R.gerr ? R.gerr : "");
          return CT3_ECUDA;
        }
      }
      RUNC(-1, R.gemm(W.att, b.out, Rall, prod(Runner::to_f32(W.tokens, kC, true), W.traw, W.tstat)));
      if (int rc = mlp(b, 0, Rall)) return rc;
    }
    {  // ---- virtual <- point cross attention (cotracker.py:510-512)
      const Block& b = L.v2p[i];
      RUNC(-1, R.gemm(raw_v, b.q, Rv, ln(Runner::to_f32(W.vqkv, kC, false), st_v, b.q, 1e-6f)));
      RUNC(-1, R.gemm(raw_p, b.kv_f, Rp, ln(Runner::to_f32(W.qkv, 2 * kC, false), st_p, b.kv_f, 1e-5f)));
      if (int rc = attention(W.vqkv, kC, W.qkv, 2 * kC, 0, kC, att_v, kV, N)) return rc;
      RUNC(-1, R.gemm(att_v, b.out, Rv, prod(Runner::to_f32(vtok, kC, true), raw_v, st_v)));
      if (int rc = mlp(b, Rp, Rv)) return rc;
    }
    {  // ---- virtual self attention (cotracker.py:514)
      const Block& b = L.vself[i];
      RUNC(-1, R.gemm(raw_v, b.q, Rv, ln(Runner::to_f32(W.vqkv, 3 * kC, false), st_v, b.q, 1e-6f)));
      if (int rc = attention(W.vqkv, 3 * kC, W.vqkv, 3 * kC, kC, 2 * kC, att_v, kV, kV)) return rc;
      RUNC(-1, R.gemm(att_v, b.out, Rv, prod(Runner::to_f32(vtok, kC, true), raw_v, st_v)));
      if (int rc = mlp(b, Rp, Rv)) return rc;
    }
    {  // ---- point <- virtual cross attention (cotracker.py:515-517)
      const Block& b = L.p2v[i];
      RUNC(-1, R.gemm(raw_p, b.q, Rp, ln(Runner::to_f32(W.qkv, kC, false), st_p, b.q, 1e-6f)));
      RUNC(-1, R.gemm(raw_v, b.kv_f, Rv, ln(Runner::to_f32(W.vqkv, 2 * kC, false), st_v, b.kv_f, 1e-5f)));
      if (int rc = attention(W.qkv, kC, W.vqkv, 2 * kC, 0, kC, att_p, N, kV)) return rc;
      RUNC(-1, R.gemm(att_p, b.out, Rp, prod(Runner::to_f32(W.tokens, kC, true), raw_p, st_p)));
      if (int rc = mlp(b, 0, Rp)) return rc;
    }
  }
  return 0;
}

int check_TN(int T, int N, int G = 1) {
  if (T < 1 || N < 1) return fail(CT3_EINVAL, "T and N must be >= 1%s");
  if (G < 1 || G > N) return fail(CT3_EINVAL, "G must be in [1, N]%s");
  if (((int64_t)N + (int64_t)kV * G) * T * 3 * kC >= (int64_t)1 << 40) return fail(CT3_EINVAL, "problem too large%s");
  return 0;
}

// group arguments of the grouped entry points; N < 0: the sizes define N (ct3_updateformer_groups)
int check_groups(const int32_t* sizes, int G, int N, int* total) {
  if (!sizes) return fail(CT3_EINVAL, "null group_sizes_host%s");
  if (G < 1) return fail(CT3_EINVAL, "G must be >= 1%s");
  int64_t sum = 0;
  for (int g = 0; g < G; ++g) {
    if (sizes[g] < 1) return fail(CT3_EINVAL, "every group size must be >= 1%s");
    sum += sizes[g];
  }
  if (sum > (int64_t)1 << 30) return fail(CT3_EINVAL, "problem too large%s");
  if (N >= 0 && sum != N) return fail(CT3_EINVAL, "group sizes must sum to N%s");
  if (G > 1 && (g_opt[OPT_FUSE] == 2 || g_opt_attn == 2))
    return fail(CT3_EUNSUPPORTED, "grouped calls do not support fuse = 2 or attn = 2%s");
  *total = (int)sum;
  return 0;
}

// frames: host frame map [G, T] into the T_pyr pyramid frames, or null (frame t, T_pyr == T)
int update_loop(const void* packed, const float* pyr, int H4, int W4, const float* support, const uint8_t* track_valid,
                float* coords, float* vis, float* conf, const float* time_emb, int T, int N, const int32_t* sizes,
                int G, int iters, void* workspace, size_t workspace_bytes, cudaStream_t stream, int T_pyr,
                const int32_t* frames);

// frame-map arguments of ct3_update_loop_frames / ct3_workspace_bytes_frames (frames == nullptr: not checked here)
int check_frames(const int32_t* frames, int G, int T, int T_pyr) {
  if (T_pyr < 1) return fail(CT3_EINVAL, "T_pyr must be >= 1%s");
  if ((int64_t)T_pyr * T >= (int64_t)1 << 31 || (int64_t)G * T >= (int64_t)1 << 31)
    return fail(CT3_EINVAL, "problem too large%s");
  if (!frames) return 0;
  for (int64_t i = 0; i < (int64_t)G * T; ++i)
    if (frames[i] < 0 || frames[i] >= T_pyr) return fail(CT3_EINVAL, "frame index outside [0, T_pyr)%s");
  return 0;
}
int updateformer(const void* packed, const float* x, int T, int N, const int32_t* sizes, int G, float* delta,
                 void* workspace, size_t workspace_bytes, cudaStream_t stream);

}  // namespace

// ================================================================================================
extern "C" {

int ct3_version(void) { return 100; }
const char* ct3_last_error(void) { return g_err; }

int ct3_set_option(const char* name, int value) {
  if (!name) return fail(CT3_EINVAL, "null option name%s");
  for (int i = 0; i < OPT_COUNT; ++i)
    if (!strcmp(name, kOptDefs[i].name)) {
      if (value < kOptDefs[i].lo || value > kOptDefs[i].hi) return fail(CT3_EINVAL, "option value out of range: %s", name);
      g_opt[i] = value;
      return 0;
    }
  return fail(CT3_EINVAL, "unknown option %s", name);
}
int ct3_get_option(const char* name, int* value) {
  if (!name || !value) return fail(CT3_EINVAL, "null argument%s");
  for (int i = 0; i < OPT_COUNT; ++i)
    if (!strcmp(name, kOptDefs[i].name)) { *value = g_opt[i]; return 0; }
  return fail(CT3_EINVAL, "unknown option %s", name);
}

int ct3_volume_is_support_major(int T, int H4, int W4, int* flag) {
  if (!flag) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = ct3_pyramid_layout(T, H4, W4, nullptr, nullptr, nullptr, nullptr)) return rc;
  *flag = effective_prec(true, T, H4, W4).support_major() ? 1 : 0;
  return 0;
}

int ct3_precision_info(int T, int H4, int W4, int* corr_products, int* fc1_products, int* volume_bytes_per_element) {
  if (int rc = ct3_pyramid_layout(T, H4, W4, nullptr, nullptr, nullptr, nullptr)) return rc;
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
  if (packed_bytes < L.total) return fail(CT3_ENOSPC, "packed buffer too small%s");
  for (int i = 0; i < n_tensors; ++i)
    if (!t[i]) return fail(CT3_EINVAL, "null weight tensor: %s", weight_names()[i].c_str());
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* pk = reinterpret_cast<uint8_t*>(packed);
  CK(cudaMemsetAsync(pk, 0, L.total, s), "memset packed");
  auto put_lin = [&](const Lin& l, const float* w, const float* b, int rows, int row_off, int perm,
                     int fp16 = 0) -> cudaError_t {
    cudaError_t e = launch_split_rows(w, rows, l.K, l.Kpad, perm, reinterpret_cast<__nv_bfloat16*>(pk + l.w), row_off, s, fp16);
    if (e != cudaSuccess) return e;
    e = launch_rowsum(w, rows, l.K, reinterpret_cast<float*>(pk + l.ws) + row_off, s);
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
    {   // to_kv(norm_context(x)) with the affine part folded into the layer (stream-ordered reuse of the scratch)
      float* w2 = reinterpret_cast<float*>(pk + L.scratch);
      float* b2 = w2 + (size_t)2 * kC * kC;
      if ((e = launch_affine_fold(t[k + 4], t[k + 5], t[k], t[k + 1], 2 * kC, kC, w2, b2, s)) != cudaSuccess) return e;
      if ((e = put_lin(b.kv_f, w2, b2, 2 * kC, 0, 0)) != cudaSuccess) return e;
    }
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

int ct3_pyramid_layout(int T, int H4, int W4, int64_t level_off[4], int level_h[4], int level_w[4],
                       int64_t* total_floats) {
  if (T < 1 || H4 < 1 || W4 < 1) return fail(CT3_EINVAL, "bad pyramid shape%s");
  const PyramidLayout p = pyramid_layout(T, H4, W4);
  for (int l = 0; l < kL; ++l) {
    if (p.h[l] < 1 || p.w[l] < 1) return fail(CT3_EINVAL, "feature map too small for 4 pyramid levels%s");
    if (level_off) level_off[l] = p.off[l];
    if (level_h) level_h[l] = p.h[l];
    if (level_w) level_w[l] = p.w[l];
  }
  if (total_floats) *total_floats = p.total;
  return 0;
}

int ct3_prepare_pyramid(const float* fmaps, int T, int H4, int W4, float* pyr, ct3_stream_t stream) {
  if (!fmaps || !pyr) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = ct3_pyramid_layout(T, H4, W4, nullptr, nullptr, nullptr, nullptr)) return rc;
  CK(launch_prepare_pyramid(fmaps, T, H4, W4, pyr, (cudaStream_t)stream), "prepare_pyramid");
  return 0;
}

// every source offset sum |stride| * index of a [T,3,H,W] frame tensor must fit in int64, in bytes
static bool frame_extent_fits(int dtype, int T, int H, int W, int64_t stride_t, int64_t stride_c, int64_t stride_h,
                              int64_t stride_w) {
  const int64_t sizes[4] = {T, 3, H, W}, strides[4] = {stride_t, stride_c, stride_h, stride_w};
  const int64_t esize = dtype == CT3_FRAMES_U8 ? 1 : 4;
  int64_t extent = 0;
  for (int i = 0; i < 4; ++i) {
    if (strides[i] == INT64_MIN) return false;
    const int64_t a = strides[i] < 0 ? -strides[i] : strides[i], m = sizes[i] - 1;
    if (m > 0 && a > (INT64_MAX - extent) / m) return false;
    extent += a * m;
  }
  return extent <= INT64_MAX / esize;
}

int ct3_prepare_frames(const void* src, int dtype, int T, int H, int W, int64_t stride_t, int64_t stride_c,
                       int64_t stride_h, int64_t stride_w, int out_h, int out_w, float* out, ct3_stream_t stream) {
  if (!src || !out) return fail(CT3_EINVAL, "null argument%s");
  if (T < 1 || H < 1 || W < 1 || out_h < 1 || out_w < 1) return fail(CT3_EINVAL, "T, H, W, out_h and out_w must be >= 1%s");
  if (dtype != CT3_FRAMES_U8 && dtype != CT3_FRAMES_F32) return fail(CT3_EINVAL, "unknown frame dtype%s");
  if (!frame_extent_fits(dtype, T, H, W, stride_t, stride_c, stride_h, stride_w))
    return fail(CT3_EINVAL, "stride extent overflows int64%s");
  // the kernel indexes the pixels of one output plane with int
  if ((int64_t)out_h * out_w > INT32_MAX) return fail(CT3_EINVAL, "output plane too large%s");
  if ((int64_t)out_h * out_w > INT64_MAX / 12 / T) return fail(CT3_EINVAL, "output too large%s");
  CK(launch_prepare_frames(src, dtype, T, H, W, stride_t, stride_c, stride_h, stride_w, out_h, out_w, out,
                           (cudaStream_t)stream), "prepare_frames");
  return 0;
}

// ---- track visualiser (render.cu) ------------------------------------------------------------------------------
int ct3_render_prepare(const void* src, int dtype, int T, int H, int W, int64_t stride_t, int64_t stride_c,
                       int64_t stride_h, int64_t stride_w, int pad, int grayscale, uint8_t* out, ct3_stream_t stream) {
  if (!src || !out) return fail(CT3_EINVAL, "null argument%s");
  if (T < 1 || H < 1 || W < 1) return fail(CT3_EINVAL, "T, H and W must be >= 1%s");
  if (T > 65535) return fail(CT3_EINVAL, "T must be <= 65535%s");
  if (pad < 0) return fail(CT3_EINVAL, "pad must be >= 0%s");
  if (grayscale != 0 && grayscale != 1) return fail(CT3_EINVAL, "grayscale must be 0 or 1%s");
  if (dtype != CT3_FRAMES_U8 && dtype != CT3_FRAMES_F32) return fail(CT3_EINVAL, "unknown frame dtype%s");
  if (!frame_extent_fits(dtype, T, H, W, stride_t, stride_c, stride_h, stride_w))
    return fail(CT3_EINVAL, "stride extent overflows int64%s");
  const int64_t ho = (int64_t)H + 2 * (int64_t)pad, wo = (int64_t)W + 2 * (int64_t)pad;
  if (ho > INT32_MAX || wo > INT32_MAX || ho * wo > INT32_MAX) return fail(CT3_EINVAL, "output plane too large%s");
  CK(launch_render_prepare(src, dtype, T, H, W, stride_t, stride_c, stride_h, stride_w, pad, grayscale, out,
                           (cudaStream_t)stream), "render_prepare");
  return 0;
}

int ct3_render_workspace_bytes(int T, int H, int W, int N, int trail, size_t* out_bytes) {
  if (!out_bytes) return fail(CT3_EINVAL, "null argument%s");
  if (T < 1 || H < 1 || W < 1 || N < 1) return fail(CT3_EINVAL, "T, H, W and N must be >= 1%s");
  if (T > 65535) return fail(CT3_EINVAL, "T must be <= 65535%s");
  if (trail < -1) return fail(CT3_EINVAL, "trail must be >= -1%s");
  if ((int64_t)H * W > INT32_MAX) return fail(CT3_EINVAL, "frame plane too large%s");
  if ((int64_t)T * N > INT32_MAX) return fail(CT3_EINVAL, "T * N too large%s");   // draw-order keys u * N + i
  *out_bytes = align_up((size_t)T * H * W * sizeof(int32_t));
  return 0;
}

int ct3_render_tracks(uint8_t* frames, int T, int H, int W, const float* pts, const uint8_t* visible,
                      const uint8_t* colors, const uint8_t* draw_mask, int N, int radius, int linewidth, int trail,
                      int query_frame, const double* alphas, const double* diff, void* workspace,
                      size_t workspace_bytes, ct3_stream_t stream) {
  if (!frames || !pts || !colors || !workspace) return fail(CT3_EINVAL, "null argument%s");
  size_t need = 0;
  if (int rc = ct3_render_workspace_bytes(T, H, W, N, trail, &need)) return rc;
  if (radius < 0 || radius > kRenderMaxRadius) return fail(CT3_EINVAL, "radius must be in [0, 255]%s");
  if (linewidth < 0) return fail(CT3_EINVAL, "linewidth must be >= 0%s");
  if (query_frame < 0 || query_frame >= T) return fail(CT3_EINVAL, "query_frame must be in [0, T)%s");
  if (trail > 0 && !alphas) return fail(CT3_EINVAL, "trail > 0 needs the blend weights (alphas)%s");
  if (workspace_bytes < need) return fail(CT3_ENOSPC, "workspace too small%s");
  CK(launch_render_tracks(frames, T, H, W, pts, visible, colors, draw_mask, N, radius, linewidth, trail, query_frame,
                          alphas, diff, static_cast<int*>(workspace), (cudaStream_t)stream),
     "render_tracks");
  return 0;
}

int ct3_render_flow_workspace_bytes(int T, int N, size_t* out_bytes) {
  if (!out_bytes) return fail(CT3_EINVAL, "null argument%s");
  if (T < 1 || N < 1) return fail(CT3_EINVAL, "T and N must be >= 1%s");
  if ((int64_t)T * N > INT32_MAX) return fail(CT3_EINVAL, "T * N too large%s");
  *out_bytes = align_up(sizeof(unsigned long long));
  return 0;
}

int ct3_render_flow_colors(const float* pts, int T, int N, int query_frame, uint8_t* colors, void* workspace,
                           size_t workspace_bytes, ct3_stream_t stream) {
  if (!pts || !colors || !workspace) return fail(CT3_EINVAL, "null argument%s");
  size_t need = 0;
  if (int rc = ct3_render_flow_workspace_bytes(T, N, &need)) return rc;
  if (query_frame < 0 || query_frame >= T) return fail(CT3_EINVAL, "query_frame must be in [0, T)%s");
  if (workspace_bytes < need) return fail(CT3_EINVAL, "workspace too small%s");
  CK(launch_render_flow_colors(pts, T, N, query_frame, colors, workspace, (cudaStream_t)stream), "render_flow_colors");
  return 0;
}

int ct3_sample_support(const float* pyr, int T, int H4, int W4, const int32_t* queried_frames,
                       const float* queried_coords, int N, const uint8_t* accumulate_mask, float* support,
                       ct3_stream_t stream) {
  if (!pyr || !queried_frames || !queried_coords || !support) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = ct3_pyramid_layout(T, H4, W4, nullptr, nullptr, nullptr, nullptr)) return rc;
  if (N < 1) return fail(CT3_EINVAL, "N must be >= 1%s");
  CK(launch_sample_support(pyr, T, H4, W4, queried_frames, queried_coords, N, accumulate_mask, support,
                           (cudaStream_t)stream), "sample_support");
  return 0;
}

int ct3_profile_enable(int on) {
  for (auto& r : g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  g_prof.clear();
  g_prof_on = on != 0;
  return 0;
}
// ms[7], launches[7], gemm_flops (plain linear layers only; category 6 = the fused q|k|v + time-attention kernel): sums since ct3_profile_enable(1); synchronises the recorded events
int ct3_profile_read(double* ms, int* launches, double* gemm_flops) {
  if (!ms || !launches || !gemm_flops) return fail(CT3_EINVAL, "null argument%s");
  for (int i = 0; i < CAT_COUNT; ++i) { ms[i] = 0.0; launches[i] = 0; }
  *gemm_flops = 0.0;
  for (auto& r : g_prof) {
    CK(cudaEventSynchronize(r.b), "profile sync");
    float t = 0.f;
    CK(cudaEventElapsedTime(&t, r.a, r.b), "profile elapsed");
    ms[r.cat] += t;
    launches[r.cat] += r.launches;
    if (r.cat == CAT_GEMM) *gemm_flops += r.flops;
  }
  return 0;
}

int ct3_workspace_bytes(int T, int N, int H4, int W4, size_t* out_bytes) {
  return ct3_workspace_bytes_groups(T, N, 1, H4, W4, out_bytes);
}

int ct3_workspace_bytes_groups(int T, int N, int G, int H4, int W4, size_t* out_bytes) {
  if (!out_bytes) return fail(CT3_EINVAL, "null out_bytes%s");
  if (int rc = check_TN(T, N, G)) return rc;
  if ((H4 != 0 || W4 != 0))
    if (int rc = ct3_pyramid_layout(T, H4, W4, nullptr, nullptr, nullptr, nullptr)) return rc;
  *out_bytes = carve(nullptr, T, N, H4, W4, G).total;
  return 0;
}

int ct3_corr_sample(const float* pyr, int H4, int W4, const float* support, const uint8_t* track_valid,
                    const float* coords, int T, int N, void* vol_split, void* scratch, size_t scratch_bytes,
                    ct3_stream_t stream) {
  if (!pyr || !support || !coords || !vol_split) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = check_TN(T, N)) return rc;
  if (int rc = ct3_pyramid_layout(T, H4, W4, nullptr, nullptr, nullptr, nullptr)) return rc;
  const __nv_bfloat16* pyr_split = nullptr;
  const Prec pr = effective_prec(scratch != nullptr, T, H4, W4);
  if (pr.patch) {
    if ((uintptr_t)scratch & 255) return fail(CT3_EINVAL, "scratch must be 256-byte aligned%s");
    if (scratch_bytes < (size_t)pyramid_layout(T, H4, W4).total * 4) return fail(CT3_ENOSPC, "scratch too small%s");
    CK(launch_split_pyramid(pyr, T, H4, W4, (__nv_bfloat16*)scratch, pr.corr, (cudaStream_t)stream), "split_pyramid");
    pyr_split = (const __nv_bfloat16*)scratch;
  }
  CK(launch_corr_sample(pyr, pyr_split, H4, W4, support, track_valid, coords, T, N, (__nv_bfloat16*)vol_split,
                        g_opt_corr, pr.corr, pr.vol16() ? 1 : 0, num_sms(), (cudaStream_t)stream, T, FrameMap{}),
     "corr_sample");
  return 0;
}

int ct3_split_rows(const float* x, int rows, int K, int Kpad, void* x_split, ct3_stream_t stream) {
  if (!x || !x_split || rows < 1 || K < 1 || Kpad < K || (Kpad % 64)) return fail(CT3_EINVAL, "bad split_rows argument%s");
  CK(launch_split_rows(x, rows, K, Kpad, 0, (__nv_bfloat16*)x_split, 0, (cudaStream_t)stream), "split_rows");
  return 0;
}

int ct3_split_rows_fp16(const float* x, int rows, int K, int Kpad, void* x_split, ct3_stream_t stream) {
  if (!x || !x_split || rows < 1 || K < 1 || Kpad < K || (Kpad % 64)) return fail(CT3_EINVAL, "bad split_rows argument%s");
  CK(launch_split_rows(x, rows, K, Kpad, 0, (__nv_bfloat16*)x_split, 0, (cudaStream_t)stream, /*fp16*/ 1), "split_rows");
  return 0;
}

int ct3_linear(const void* x_split, const void* w_split, const float* bias, int M, int Nout, int Kpad, int act,
               float* y, ct3_stream_t stream) {
  return ct3_linear_prec(x_split, w_split, bias, M, Nout, Kpad, act, 3, 0, y, stream);
}

int ct3_linear_prec(const void* x_split, const void* w_split, const float* bias, int M, int Nout, int Kpad, int act,
                    int products, int fp16, float* y, ct3_stream_t stream) {
  if (!x_split || !w_split || !y) return fail(CT3_EINVAL, "null argument%s");
  if (M < 1 || Nout < 1 || (Nout % 128) || Kpad < 64 || (Kpad % 64) || act < 0 || act > 2)
    return fail(CT3_EINVAL, "ct3_linear: need M>=1, Nout %% 128 == 0, Kpad %% 64 == 0, act in 0..2%s");
  if (products < 1 || products > 3 || fp16 < 0 || fp16 > 1)
    return fail(CT3_EINVAL, "ct3_linear_prec: products in 1..3, fp16 in 0..1%s");
  GemmProblem p;
  p.products = products;
  p.fp16 = fp16;
  p.x_split = (const __nv_bfloat16*)x_split;
  p.w_split = (const __nv_bfloat16*)w_split;
  p.M = M; p.N = Nout; p.Kpad = Kpad;
  p.epi.bias = bias;
  p.epi.act = act;
  p.epi.out_f32 = y;
  p.epi.ld_f32 = Nout;
  const char* gerr = nullptr;
  int rc = gemm_launch(p, g_opt_gemm, num_sms(), (cudaStream_t)stream, &gerr);
  if (rc != 0) {
    snprintf(g_err, sizeof(g_err), "ct3_linear: %s (%s)", cudaGetErrorString((cudaError_t)rc), gerr ? gerr : "");
    return CT3_ECUDA;
  }
  return 0;
}

int ct3_update_loop(const void* packed, const float* pyr, int H4, int W4, const float* support,
                    const uint8_t* track_valid, float* coords, float* vis, float* conf, const float* time_emb,
                    int T, int N, int iters, void* workspace, size_t workspace_bytes, ct3_stream_t stream) {
  const int32_t one = N;
  return update_loop(packed, pyr, H4, W4, support, track_valid, coords, vis, conf, time_emb, T, N, &one, 1, iters,
                     workspace, workspace_bytes, (cudaStream_t)stream, T, nullptr);
}

int ct3_update_loop_groups(const void* packed, const float* pyr, int H4, int W4, const float* support,
                           const uint8_t* track_valid, float* coords, float* vis, float* conf, const float* time_emb,
                           int T, int N, int iters, void* workspace, size_t workspace_bytes, ct3_stream_t stream,
                           const int32_t* group_sizes_host, int G) {
  return update_loop(packed, pyr, H4, W4, support, track_valid, coords, vis, conf, time_emb, T, N, group_sizes_host, G,
                     iters, workspace, workspace_bytes, (cudaStream_t)stream, T, nullptr);
}

int ct3_workspace_bytes_frames(int T, int T_pyr, int N, int G, int H4, int W4, size_t* out_bytes) {
  if (!out_bytes) return fail(CT3_EINVAL, "null out_bytes%s");
  if (int rc = check_TN(T, N, G)) return rc;
  if (int rc = check_frames(nullptr, G, T, T_pyr)) return rc;
  if (int rc = ct3_pyramid_layout(T_pyr, H4, W4, nullptr, nullptr, nullptr, nullptr)) return rc;
  *out_bytes = carve(nullptr, T, N, H4, W4, G, T_pyr, true).total;
  return 0;
}

int ct3_update_loop_frames(const void* packed, const float* pyr, int T_pyr, int H4, int W4, const float* support,
                           const uint8_t* track_valid, float* coords, float* vis, float* conf, const float* time_emb,
                           int T, int N, int iters, void* workspace, size_t workspace_bytes, ct3_stream_t stream,
                           const int32_t* group_sizes_host, int G, const int32_t* group_frames_host) {
  if (!group_frames_host) return fail(CT3_EINVAL, "null group_frames_host%s");
  return update_loop(packed, pyr, H4, W4, support, track_valid, coords, vis, conf, time_emb, T, N, group_sizes_host, G,
                     iters, workspace, workspace_bytes, (cudaStream_t)stream, T_pyr, group_frames_host);
}

int ct3_updateformer(const void* packed, const float* x, int T, int N, float* delta, void* workspace,
                     size_t workspace_bytes, ct3_stream_t stream) {
  const int32_t one = N;
  return updateformer(packed, x, T, N, &one, 1, delta, workspace, workspace_bytes, (cudaStream_t)stream);
}

int ct3_updateformer_groups(const void* packed, const float* x, int T, const int32_t* group_sizes_host, int G,
                            float* delta, void* workspace, size_t workspace_bytes, ct3_stream_t stream) {
  return updateformer(packed, x, T, -1, group_sizes_host, G, delta, workspace, workspace_bytes, (cudaStream_t)stream);
}

}  // extern "C"

namespace {

int update_loop(const void* packed, const float* pyr, int H4, int W4, const float* support, const uint8_t* track_valid,
                float* coords, float* vis, float* conf, const float* time_emb, int T, int N, const int32_t* sizes,
                int G, int iters, void* workspace, size_t workspace_bytes, cudaStream_t stream, int T_pyr,
                const int32_t* frames) {
  if (!packed || !pyr || !support || !coords || !vis || !conf || !time_emb || !workspace)
    return fail(CT3_EINVAL, "null argument%s");
  if (int rc = check_TN(T, N)) return rc;
  int total = 0;
  if (int rc = check_groups(sizes, G, N, &total)) return rc;
  if (int rc = check_TN(T, N, G)) return rc;
  if (iters < 0) return fail(CT3_EINVAL, "iters must be >= 0%s");
  if (int rc = check_frames(frames, G, T, T_pyr)) return rc;
  if (int rc = ct3_pyramid_layout(T_pyr, H4, W4, nullptr, nullptr, nullptr, nullptr)) return rc;
  if ((uintptr_t)workspace & 255) return fail(CT3_EINVAL, "workspace must be 256-byte aligned%s");
  const Workspace W = carve(workspace, T, N, H4, W4, G, T_pyr, frames != nullptr);
  if (workspace_bytes < W.total) return fail(CT3_ENOSPC, "workspace too small%s");
  const Layout& L = layout();
  Runner R{reinterpret_cast<const uint8_t*>(packed), L, stream, g_opt_gemm};
  const uint8_t* pk = R.pk;
  GroupPlan gp;
  if (int rc = plan_groups(gp, sizes, G, T, N, W.groups, R.s)) return rc;
  FrameMap fm;
  if (frames) {   // the frame map reaches the device like the group table: in stream order, through kernel arguments
    CK(launch_upload_i32(W.frames, frames, G * T, R.s), "upload frame map");
    fm.frames = W.frames;
    fm.goff = G > 1 ? gp.off : nullptr;
    fm.G = G;
  }
  const int Rp = N * T, Mc = Rp * kL;
  // split-bf16 copy of the pyramid: the TMA source of the correlation kernel, made once per call
  const Prec pr = effective_prec(W.pyr_split != nullptr, T_pyr, H4, W4);
  const __nv_bfloat16* pyr_split = (pr.patch && iters > 0) ? W.pyr_split : nullptr;
  if (pyr_split) RUNC(CAT_MISC, launch_split_pyramid(pyr, T_pyr, H4, W4, W.pyr_split, pr.corr, R.s));

  // W_in * time_emb[t]: x + time_emb is folded into a per-frame bias of input_transform (cotracker3_offline.py:196)
  RUNC(CAT_MISC, launch_row_bias(time_emb, reinterpret_cast<const float*>(pk + L.win_f32), T, W.row_bias, R.s));

  for (int it = 0; it < iters; ++it) {
    // (i)+(ii) sampling + 4-D correlation, all levels -> split volume
    RUNC(CAT_CORR, launch_corr_sample(pyr, pyr_split, H4, W4, support, track_valid, coords, T, N, W.vol, g_opt_corr,
                                      pr.corr, pr.vol16() ? 1 : 0, num_sms(), R.s, T_pyr, fm));
    // (iii) corr_mlp: 2401 -> 384 (GELU erf) -> 256, written straight into X columns [256*l, 256*l+256)
    if (pr.vol16()) {   // single fp16 volume plane x split fp16 weights: 2 (or 1) tensor-core products per FLOP
      RUNC(-1, R.gemm(W.vol, pr.support_major() ? L.corr_fc1_th : L.corr_fc1_h, Mc,
                      Runner::to_split(W.h1, 2 * kCorrHid, kCorrHid, /*erf*/ 1), pr.fc1, /*fp16*/ 1, kVolPad));
    } else {
      RUNC(-1, R.gemm(W.vol, pr.support_major() ? L.corr_fc1_t : L.corr_fc1, Mc,
                      Runner::to_split(W.h1, 2 * kCorrHid, kCorrHid, /*erf*/ 1)));
    }
    {
      GemmEpilogue e = Runner::to_split(W.xs, 2 * kXPad, kXPad, 0);
      e.row_group = kL;
      RUNC(-1, R.gemm(W.h1, L.corr_fc2, Mc, e));
    }
    // vis, conf, posenc(rel. motion), zero pad -> X columns [1024,1152)
    RUNC(CAT_MISC, launch_build_x_small(coords, vis, conf, T, N, W.xs, R.s));
    // input_transform (+ folded time embedding) -> point tokens
    {
      GemmEpilogue e = Runner::to_f32(W.tokens, kC, false);
      e.row_bias = W.row_bias;
      e.row_mod = T;
      if (fold_enabled(R, T)) { e.raw_split = W.traw; e.stat_part = W.tstat; }
      RUNC(-1, R.gemm(W.xs, L.in_tr, Rp, e));
    }
    if (int rc = fold_enabled(R, T) ? transformer_body_fold(R, W, T, N) : transformer_body(R, W, T, N, gp)) return rc;
    // (v) heads + state update
    RUNC(CAT_MISC, launch_heads(W.tokens, reinterpret_cast<const float*>(pk + L.heads_w),
                     reinterpret_cast<const float*>(pk + L.heads_b), coords, vis, conf, nullptr, T, N, R.s));
  }
  return 0;
}

int updateformer(const void* packed, const float* x, int T, int N, const int32_t* sizes, int G, float* delta,
                 void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (!packed || !x || !delta || !workspace) return fail(CT3_EINVAL, "null argument%s");
  if (N >= 0)
    if (int rc = check_TN(T, N)) return rc;
  int total = 0;
  if (int rc = check_groups(sizes, G, N, &total)) return rc;
  N = total;
  if (int rc = check_TN(T, N, G)) return rc;
  if ((uintptr_t)workspace & 255) return fail(CT3_EINVAL, "workspace must be 256-byte aligned%s");
  const Workspace W = carve(workspace, T, N, 0, 0, G);
  if (workspace_bytes < W.total) return fail(CT3_ENOSPC, "workspace too small%s");
  const Layout& L = layout();
  Runner R{reinterpret_cast<const uint8_t*>(packed), L, stream, g_opt_gemm};
  const int Rp = N * T;
  GroupPlan gp;
  if (int rc = plan_groups(gp, sizes, G, T, N, W.groups, R.s)) return rc;
  RUNC(CAT_MISC, launch_split_rows(x, Rp, kX, kXPad, /*perm_x*/ 1, W.xs, 0, R.s));
  {
    GemmEpilogue e = Runner::to_f32(W.tokens, kC, false);
    if (fold_enabled(R, T)) { e.raw_split = W.traw; e.stat_part = W.tstat; }
    RUNC(-1, R.gemm(W.xs, L.in_tr, Rp, e));
  }
  if (int rc = fold_enabled(R, T) ? transformer_body_fold(R, W, T, N) : transformer_body(R, W, T, N, gp)) return rc;
  RUNC(CAT_MISC, launch_heads(W.tokens, reinterpret_cast<const float*>(R.pk + L.heads_w),
                   reinterpret_cast<const float*>(R.pk + L.heads_b), nullptr, nullptr, nullptr, delta, T, N, R.s));
  return 0;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// encoder tail (conv2 -> InstanceNorm -> ReLU -> conv3 -> L2-normalise -> pyramid), see enc_tail.cu
namespace {
constexpr int kEncCin = 416, kEncMid = 256, kEncK = kEncCin * 9;
struct EncLayout { Lin conv2, conv3; size_t total; };
const EncLayout& enc_layout() {
  static const EncLayout E0 = [] {
    EncLayout E;
    size_t off = 0;
    place_lin(E.conv2, kEncMid, kEncK, off);
    place_lin(E.conv3, kD, kEncMid, off);
    E.total = off;
    return E;
  }();
  return E0;
}
struct EncWs { __nv_bfloat16* a; float* y; __nv_bfloat16* ys; float* stats; void* stat_scratch; size_t total; int tc; };
EncWs enc_carve(void* base, int T, int H4, int W4) {
  EncWs w;
  w.tc = T < 16 ? T : 16;                         // frames per chunk: bounds the im2col operand to ~3 GB
  const size_t Mc = (size_t)w.tc * H4 * W4;
  uint8_t* p = reinterpret_cast<uint8_t*>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) { uint8_t* r = p + off; off = align_up(off + bytes, 1024); return r; };
  w.a = (__nv_bfloat16*)take(Mc * 2 * pad64(kEncK) * 2);
  w.y = (float*)take(Mc * kEncMid * 4);
  w.ys = (__nv_bfloat16*)take(Mc * 2 * kEncMid * 2);
  w.stats = (float*)take((size_t)w.tc * kEncMid * 2 * 4);
  w.stat_scratch = take(instnorm_scratch_bytes(w.tc, kEncMid));
  w.total = off;
  return w;
}
}  // namespace

extern "C" {

int ct3_enc_tail_packed_bytes(size_t* out_bytes) {
  if (!out_bytes) return fail(CT3_EINVAL, "null out_bytes%s");
  *out_bytes = enc_layout().total;
  return 0;
}

int ct3_enc_tail_pack(const float* conv2_w, const float* conv2_b, const float* conv3_w, const float* conv3_b,
                      void* packed, size_t packed_bytes, ct3_stream_t stream) {
  const EncLayout& E = enc_layout();
  if (!conv2_w || !conv2_b || !conv3_w || !conv3_b || !packed) return fail(CT3_EINVAL, "null argument%s");
  if (packed_bytes < E.total) return fail(CT3_ENOSPC, "packed buffer too small%s");
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* pk = reinterpret_cast<uint8_t*>(packed);
  CK(cudaMemsetAsync(pk, 0, E.total, s), "memset enc packed");
  CK(launch_split_rows(conv2_w, kEncMid, kEncK, E.conv2.Kpad, 0, reinterpret_cast<__nv_bfloat16*>(pk + E.conv2.w), 0, s), "pack conv2");
  CK(cudaMemcpyAsync(pk + E.conv2.b, conv2_b, kEncMid * 4, cudaMemcpyDeviceToDevice, s), "pack conv2 bias");
  CK(launch_split_rows(conv3_w, kD, kEncMid, E.conv3.Kpad, 0, reinterpret_cast<__nv_bfloat16*>(pk + E.conv3.w), 0, s), "pack conv3");
  CK(cudaMemcpyAsync(pk + E.conv3.b, conv3_b, kD * 4, cudaMemcpyDeviceToDevice, s), "pack conv3 bias");
  return 0;
}

int ct3_upsample_concat(const float* const* src, const int* channels, const int* heights, const int* widths, int T,
                        int H, int W, float* out, ct3_stream_t stream) {
  if (!src || !channels || !heights || !widths || !out) return fail(CT3_EINVAL, "null argument%s");
  int ctot = 0;
  for (int k = 0; k < 4; ++k) {
    if (!src[k] || channels[k] < 1 || heights[k] < 1 || widths[k] < 1) return fail(CT3_EINVAL, "bad stage tensor%s");
    ctot += channels[k];
  }
  if (T < 1 || H < 1 || W < 1) return fail(CT3_EINVAL, "bad output shape%s");
  CK(launch_upsample_concat(src, channels, heights, widths, T, H, W, out, (cudaStream_t)stream), "upsample_concat");
  return 0;
}

int ct3_enc_tail_workspace_bytes(int T, int H4, int W4, size_t* out_bytes) {
  if (!out_bytes) return fail(CT3_EINVAL, "null out_bytes%s");
  if (int rc = ct3_pyramid_layout(T, H4, W4, nullptr, nullptr, nullptr, nullptr)) return rc;
  *out_bytes = enc_carve(nullptr, T, H4, W4).total;
  return 0;
}

int ct3_enc_tail(const void* packed, const float* cat, int T, int H4, int W4, float* pyr, void* workspace,
                 size_t workspace_bytes, ct3_stream_t stream) {
  if (!packed || !cat || !pyr || !workspace) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = ct3_pyramid_layout(T, H4, W4, nullptr, nullptr, nullptr, nullptr)) return rc;
  if ((uintptr_t)workspace & 255) return fail(CT3_EINVAL, "workspace must be 256-byte aligned%s");
  const EncWs W = enc_carve(workspace, T, H4, W4);
  if (workspace_bytes < W.total) return fail(CT3_ENOSPC, "workspace too small%s");
  const EncLayout& E = enc_layout();
  const uint8_t* pk = reinterpret_cast<const uint8_t*>(packed);
  cudaStream_t s = (cudaStream_t)stream;
  const int HW = H4 * W4;
  const PyramidLayout lay = pyramid_layout(T, H4, W4);
  for (int t0 = 0; t0 < T; t0 += W.tc) {
    const int tc = (T - t0) < W.tc ? (T - t0) : W.tc;
    const int Mc = tc * HW;
    const float* in = cat + (int64_t)t0 * kEncCin * HW;
    float* f0 = pyr + lay.off[0] + (int64_t)t0 * HW * kD;   // conv3 rows (t,y,x) are the channels-last texels
    CK(launch_im2col3x3_split(in, tc, kEncCin, H4, W4, E.conv2.Kpad, W.a, s), "im2col conv2");
    const char* gerr = nullptr;
    GemmProblem p;
    p.x_split = W.a;
    p.w_split = reinterpret_cast<const __nv_bfloat16*>(pk + E.conv2.w);
    p.M = Mc; p.N = kEncMid; p.Kpad = E.conv2.Kpad;
    p.epi.bias = reinterpret_cast<const float*>(pk + E.conv2.b);
    p.epi.out_f32 = W.y; p.epi.ld_f32 = kEncMid;
    int rc = gemm_launch(p, g_opt_gemm, num_sms(), s, &gerr);
    if (rc != 0) { snprintf(g_err, sizeof(g_err), "enc conv2 gemm: %s (%s)", cudaGetErrorString((cudaError_t)rc), gerr ? gerr : ""); return CT3_ECUDA; }
    CK(launch_instnorm_stats(W.y, tc, HW, kEncMid, 1e-5f, W.stats, W.stat_scratch, s), "instnorm stats");
    CK(launch_instnorm_relu_split(W.y, W.stats, (int64_t)Mc, HW, kEncMid, W.ys, s), "instnorm relu split");
    GemmProblem q;
    q.x_split = W.ys;
    q.w_split = reinterpret_cast<const __nv_bfloat16*>(pk + E.conv3.w);
    q.M = Mc; q.N = kD; q.Kpad = E.conv3.Kpad;
    q.epi.bias = reinterpret_cast<const float*>(pk + E.conv3.b);
    q.epi.out_f32 = f0; q.epi.ld_f32 = kD;
    rc = gemm_launch(q, g_opt_gemm, num_sms(), s, &gerr);
    if (rc != 0) { snprintf(g_err, sizeof(g_err), "enc conv3 gemm: %s (%s)", cudaGetErrorString((cudaError_t)rc), gerr ? gerr : ""); return CT3_ECUDA; }
    CK(launch_l2norm_rows(f0, (int64_t)Mc, f0, s), "l2norm rows");
  }
  CK(launch_pyramid_pools(T, H4, W4, pyr, s), "pyramid pools");
  return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// Whole CNN encoder (BasicEncoder.forward, blocks.py:190-219) + L2-normalise + pyramid on the tensor-core engine,
// channels-last end to end (enc_front.cu + the GEMM engine); see ct3_encoder in include/ct3_b200.h.
namespace {

struct ConvW { size_t w = 0, b = 0; int cout = 0, cin = 0, taps = 0, cp = 0, cout_pad = 0; };
struct EncFull {
  size_t stem_w = 0, stem_b = 0;
  ConvW unit[4][2][2];   // [stage][unit][conv1|conv2]
  ConvW down[4];         // stage 1..3: 1x1 stride-2 shortcut of unit 0
  ConvW conv2;           // 3x3 416 -> 256 on the 448-channel padded concat
  Lin conv3;             // 1x1 256 -> 128 (linear-layer layout)
  size_t total = 0;
};
constexpr int kStageC[4] = {64, 96, 128, 128};      // real channels per stage
constexpr int kStageCp[4] = {64, 128, 128, 128};    // carried (padded) channels per stage
constexpr int kCatC = 416, kCatCp = 448;

void place_conv(ConvW& c, int cout, int cin, int taps, int cp, int cout_pad, size_t& off) {
  c.cout = cout; c.cin = cin; c.taps = taps; c.cp = cp; c.cout_pad = cout_pad;
  c.w = off;
  off = align_up(off + (size_t)cout_pad * 2 * taps * cp * sizeof(__nv_bfloat16));
  c.b = off;
  off = align_up(off + (size_t)cout_pad * sizeof(float));
}
const EncFull& enc_full() {
  static const EncFull E0 = [] {
    EncFull E;
    size_t off = 0;
    E.stem_w = off; off = align_up(off + (size_t)64 * 3 * 49 * 4);
    E.stem_b = off; off = align_up(off + 64 * 4);
    for (int s = 0; s < 4; ++s) {
      const int cin = s == 0 ? 64 : kStageC[s - 1], cin_p = s == 0 ? 64 : kStageCp[s - 1];
      place_conv(E.unit[s][0][0], kStageC[s], cin, 9, cin_p, kStageCp[s], off);
      place_conv(E.unit[s][0][1], kStageC[s], kStageC[s], 9, kStageCp[s], kStageCp[s], off);
      place_conv(E.unit[s][1][0], kStageC[s], kStageC[s], 9, kStageCp[s], kStageCp[s], off);
      place_conv(E.unit[s][1][1], kStageC[s], kStageC[s], 9, kStageCp[s], kStageCp[s], off);
      if (s > 0) place_conv(E.down[s], kStageC[s], cin, 1, cin_p, kStageCp[s], off);
    }
    place_conv(E.conv2, kEncMid, kCatC, 9, kCatCp, kEncMid, off);
    place_lin(E.conv3, kD, kEncMid, off);
    E.total = off;
    return E;
  }();
  return E0;
}
const std::vector<std::string>& enc_weight_names() {
  static const std::vector<std::string> names0 = [] {
    std::vector<std::string> n = {"conv1.weight", "conv1.bias"};
    for (int s = 1; s <= 4; ++s) {
      for (int u = 0; u < 2; ++u)
        for (int c = 1; c <= 2; ++c) {
          const std::string p = "layer" + std::to_string(s) + "." + std::to_string(u) + ".conv" + std::to_string(c);
          n.push_back(p + ".weight");
          n.push_back(p + ".bias");
        }
      if (s > 1) {
        n.push_back("layer" + std::to_string(s) + ".0.downsample.0.weight");
        n.push_back("layer" + std::to_string(s) + ".0.downsample.0.bias");
      }
    }
    for (const char* k : {"conv2.weight", "conv2.bias", "conv3.weight", "conv3.bias"}) n.push_back(k);
    return n;
  }();
  return names0;
}

inline int half_up(int v) { return (v - 1) / 2 + 1; }   // output size of a stride-2 conv (3x3 pad 1 or 1x1)
struct EncGeom { int h[4], w[4]; int H4, W4; };
EncGeom enc_geom(int H, int W) {
  EncGeom g;
  g.h[0] = half_up(H); g.w[0] = half_up(W);            // conv1 7x7/2 pad 3: floor((H-1)/2)+1
  for (int s = 1; s < 4; ++s) { g.h[s] = half_up(g.h[s - 1]); g.w[s] = half_up(g.w[s - 1]); }
  g.H4 = H / 4; g.W4 = W / 4;
  return g;
}
struct EncFullWs {
  float *fy, *fyd, *fx[4], *stats, *stats_d;
  void* stat_scratch;
  __nv_bfloat16 *sx, *sy, *gat, *gat_d, *cat;
  size_t total; int tc;
};
EncFullWs enc_full_carve(void* base, int T, int H, int W) {
  EncFullWs w;
  w.tc = T < 16 ? T : 16;
  const EncGeom g = enc_geom(H, W);
  size_t P[4];
  for (int s = 0; s < 4; ++s) P[s] = (size_t)w.tc * g.h[s] * g.w[s];
  const size_t P4 = (size_t)w.tc * g.H4 * g.W4;
  auto mx = [](size_t a, size_t b) { return a > b ? a : b; };
  size_t fy = P4 * kEncMid, sact = P4 * 2 * kEncMid, gat = 0, gat_d = 0, fyd = 0;
  for (int s = 0; s < 4; ++s) {
    fy = mx(fy, P[s] * kStageCp[s]);
    sact = mx(sact, P[s] * 2 * kStageCp[s]);
    if (s > 0) {
      gat = mx(gat, P[s] * 2 * 9 * kStageCp[s - 1]);
      gat_d = mx(gat_d, P[s] * 2 * kStageCp[s - 1]);
      fyd = mx(fyd, P[s] * kStageCp[s]);
    }
  }
  uint8_t* p = reinterpret_cast<uint8_t*>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) { uint8_t* r = p + off; off = align_up(off + bytes, 1024); return r; };
  w.fy = (float*)take(fy * 4);
  w.fyd = (float*)take(fyd * 4);
  for (int s = 0; s < 4; ++s) w.fx[s] = (float*)take(P[s] * kStageCp[s] * 4);
  w.sx = (__nv_bfloat16*)take(sact * 2);
  w.sy = (__nv_bfloat16*)take(sact * 2);
  w.gat = (__nv_bfloat16*)take(gat * 2);
  w.gat_d = (__nv_bfloat16*)take(gat_d * 2);
  w.cat = (__nv_bfloat16*)take(P4 * 2 * kCatCp * 2);
  w.stats = (float*)take((size_t)w.tc * 256 * 2 * 4);
  w.stats_d = (float*)take((size_t)w.tc * 256 * 2 * 4);
  w.stat_scratch = take(instnorm_scratch_bytes(w.tc, 256));
  w.total = off;
  return w;
}

}  // namespace

extern "C" {

int ct3_encoder_num_weight_tensors(void) { return (int)enc_weight_names().size(); }
const char* ct3_encoder_weight_name(int index) {
  const auto& n = enc_weight_names();
  if (index < 0 || index >= (int)n.size()) return nullptr;
  return n[index].c_str();
}
int ct3_encoder_packed_bytes(size_t* out_bytes) {
  if (!out_bytes) return fail(CT3_EINVAL, "null out_bytes%s");
  *out_bytes = enc_full().total;
  return 0;
}

int ct3_encoder_pack(const float* const* t, int n_tensors, void* packed, size_t packed_bytes, ct3_stream_t stream) {
  const EncFull& E = enc_full();
  if (!t || !packed) return fail(CT3_EINVAL, "null argument%s");
  if (n_tensors != (int)enc_weight_names().size()) return fail(CT3_EINVAL, "wrong number of encoder weight tensors%s");
  if (packed_bytes < E.total) return fail(CT3_ENOSPC, "packed buffer too small%s");
  for (int i = 0; i < n_tensors; ++i)
    if (!t[i]) return fail(CT3_EINVAL, "null weight tensor: %s", enc_weight_names()[i].c_str());
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* pk = reinterpret_cast<uint8_t*>(packed);
  CK(cudaMemsetAsync(pk, 0, E.total, s), "memset encoder packed");
  int k = 0;
  CK(cudaMemcpyAsync(pk + E.stem_w, t[k], (size_t)64 * 3 * 49 * 4, cudaMemcpyDeviceToDevice, s), "pack conv1");
  CK(cudaMemcpyAsync(pk + E.stem_b, t[k + 1], 64 * 4, cudaMemcpyDeviceToDevice, s), "pack conv1 bias");
  k += 2;
  auto put = [&](const ConvW& c, const float* w, const float* b) -> cudaError_t {
    cudaError_t e = launch_pack_conv(w, c.cout, c.cin, c.taps, c.cp, c.cout_pad, reinterpret_cast<__nv_bfloat16*>(pk + c.w), s);
    if (e != cudaSuccess) return e;
    return cudaMemcpyAsync(pk + c.b, b, (size_t)c.cout * 4, cudaMemcpyDeviceToDevice, s);   // padded bias rows stay zero
  };
  for (int st = 0; st < 4; ++st) {
    for (int u = 0; u < 2; ++u)
      for (int c = 0; c < 2; ++c) { CK(put(E.unit[st][u][c], t[k], t[k + 1]), "pack residual conv"); k += 2; }
    if (st > 0) { CK(put(E.down[st], t[k], t[k + 1]), "pack downsample conv"); k += 2; }
  }
  CK(put(E.conv2, t[k], t[k + 1]), "pack conv2"); k += 2;
  CK(launch_split_rows(t[k], kD, kEncMid, E.conv3.Kpad, 0, reinterpret_cast<__nv_bfloat16*>(pk + E.conv3.w), 0, s), "pack conv3");
  CK(cudaMemcpyAsync(pk + E.conv3.b, t[k + 1], kD * 4, cudaMemcpyDeviceToDevice, s), "pack conv3 bias");
  return 0;
}

int ct3_encoder_workspace_bytes(int T, int H, int W, size_t* out_bytes) {
  if (!out_bytes) return fail(CT3_EINVAL, "null out_bytes%s");
  if (T < 1 || H < 16 || W < 16) return fail(CT3_EINVAL, "encoder: need T >= 1 and H, W >= 16%s");
  if (int rc = ct3_pyramid_layout(T, H / 4, W / 4, nullptr, nullptr, nullptr, nullptr)) return rc;
  *out_bytes = enc_full_carve(nullptr, T, H, W).total;
  return 0;
}

int ct3_encoder(const void* packed, const float* frames, int T, int H, int W, float* pyr, void* workspace,
                size_t workspace_bytes, ct3_stream_t stream) {
  if (!packed || !frames || !pyr || !workspace) return fail(CT3_EINVAL, "null argument%s");
  if (T < 1 || H < 16 || W < 16) return fail(CT3_EINVAL, "encoder: need T >= 1 and H, W >= 16%s");
  const EncGeom g = enc_geom(H, W);
  if (int rc = ct3_pyramid_layout(T, g.H4, g.W4, nullptr, nullptr, nullptr, nullptr)) return rc;
  if ((uintptr_t)workspace & 255) return fail(CT3_EINVAL, "workspace must be 256-byte aligned%s");
  const EncFullWs Wk = enc_full_carve(workspace, T, H, W);
  if (workspace_bytes < Wk.total) return fail(CT3_ENOSPC, "workspace too small%s");
  const EncFull& E = enc_full();
  const uint8_t* pk = reinterpret_cast<const uint8_t*>(packed);
  cudaStream_t s = (cudaStream_t)stream;
  const PyramidLayout lay = pyramid_layout(T, g.H4, g.W4);
  const int nsm = num_sms();
  auto W16 = [&](const ConvW& c) { return reinterpret_cast<const __nv_bfloat16*>(pk + c.w); };
  auto B32 = [&](const ConvW& c) { return reinterpret_cast<const float*>(pk + c.b); };
  // y = GEMM(gathered rows, conv weights): the stride-2 convolutions
  auto gemm_rows = [&](const __nv_bfloat16* rows, const ConvW& c, int64_t M, float* y) -> int {
    GemmProblem p;
    p.x_split = rows;
    p.w_split = W16(c);
    p.M = (int)M; p.N = c.cout_pad; p.Kpad = c.taps * c.cp;
    p.epi.bias = B32(c);
    p.epi.out_f32 = y; p.epi.ld_f32 = c.cout_pad;
    const char* gerr = nullptr;
    int rc = gemm_launch(p, g_opt_gemm, nsm, s, &gerr);
    if (rc != 0) { snprintf(g_err, sizeof(g_err), "encoder gemm: %s (%s)", cudaGetErrorString((cudaError_t)rc), gerr ? gerr : ""); return CT3_ECUDA; }
    return 0;
  };
  const int chunks = (T + Wk.tc - 1) / Wk.tc;
  ProfScope ps_all(s, CAT_ENC, 0.0, chunks * 90 + 3);   // kernels launched per 16-frame chunk + the 3 pyramid pools
  for (int t0 = 0; t0 < T; t0 += Wk.tc) {
    const int tc = (T - t0) < Wk.tc ? (T - t0) : Wk.tc;
    // ---- stem: conv1 7x7/2 -> IN -> ReLU
    int h = g.h[0], w = g.w[0], C = 64;
    int64_t rows = (int64_t)tc * h * w;
    CK(launch_conv_stem(frames + (int64_t)t0 * 3 * H * W, reinterpret_cast<const float*>(pk + E.stem_w),
                        reinterpret_cast<const float*>(pk + E.stem_b), tc, H, W, Wk.fy, s), "conv1");
    CK(launch_instnorm_stats(Wk.fy, tc, h * w, C, 1e-5f, Wk.stats, Wk.stat_scratch, s), "stem stats");
    CK(launch_norm_act(Wk.fy, Wk.stats, nullptr, nullptr, 0, rows, h * w, C, Wk.fx[0], Wk.sx, s), "stem norm");
    // ---- four stages of two residual units
    for (int st = 0; st < 4; ++st) {
      float* X = Wk.fx[st];
      const int Cp = kStageCp[st];
      if (st > 0) {
        // unit 0 of a strided stage: y = conv3x3/2(x); x' = IN(conv1x1/2(x)); out = relu(x' + relu(IN(conv3x3(relu(IN(y))))))
        const int Cin = kStageCp[st - 1];
        const int ho = g.h[st], wo = g.w[st];
        const int64_t orows = (int64_t)tc * ho * wo;
        CK(launch_gather_s2(Wk.sx, tc, h, w, Cin, 9, Wk.gat, s), "gather 3x3/2");
        CK(launch_gather_s2(Wk.sx, tc, h, w, Cin, 1, Wk.gat_d, s), "gather 1x1/2");
        if (int rc = gemm_rows(Wk.gat, E.unit[st][0][0], orows, Wk.fy)) return rc;
        CK(launch_instnorm_stats(Wk.fy, tc, ho * wo, Cp, 1e-5f, Wk.stats, Wk.stat_scratch, s), "stats");
        CK(launch_norm_act(Wk.fy, Wk.stats, nullptr, nullptr, 0, orows, ho * wo, Cp, nullptr, Wk.sy, s), "norm");
        CK(launch_conv3x3_tc(Wk.sy, W16(E.unit[st][0][1]), B32(E.unit[st][0][1]), tc, ho, wo, Cp, Cp, Wk.fy, nsm, s), "conv");
        CK(launch_instnorm_stats(Wk.fy, tc, ho * wo, Cp, 1e-5f, Wk.stats, Wk.stat_scratch, s), "stats");
        if (int rc = gemm_rows(Wk.gat_d, E.down[st], orows, Wk.fyd)) return rc;
        CK(launch_instnorm_stats(Wk.fyd, tc, ho * wo, Cp, 1e-5f, Wk.stats_d, Wk.stat_scratch, s), "stats");
        CK(launch_norm_act(Wk.fy, Wk.stats, Wk.fyd, Wk.stats_d, 2, orows, ho * wo, Cp, X, Wk.sx, s), "norm");
        h = ho; w = wo; rows = orows;
      }
      for (int u = (st > 0 ? 1 : 0); u < 2; ++u) {
        // stride-1 unit: out = relu(x + relu(IN(conv(relu(IN(conv(x)))))))
        CK(launch_conv3x3_tc(Wk.sx, W16(E.unit[st][u][0]), B32(E.unit[st][u][0]), tc, h, w, Cp, Cp, Wk.fy, nsm, s), "conv");
        CK(launch_instnorm_stats(Wk.fy, tc, h * w, Cp, 1e-5f, Wk.stats, Wk.stat_scratch, s), "stats");
        CK(launch_norm_act(Wk.fy, Wk.stats, nullptr, nullptr, 0, rows, h * w, Cp, nullptr, Wk.sy, s), "norm");
        CK(launch_conv3x3_tc(Wk.sy, W16(E.unit[st][u][1]), B32(E.unit[st][u][1]), tc, h, w, Cp, Cp, Wk.fy, nsm, s), "conv");
        CK(launch_instnorm_stats(Wk.fy, tc, h * w, Cp, 1e-5f, Wk.stats, Wk.stat_scratch, s), "stats");
        CK(launch_norm_act(Wk.fy, Wk.stats, X, nullptr, 1, rows, h * w, Cp, X, Wk.sx, s), "norm");
      }
    }
    // ---- resize + concat -> conv2 3x3 -> IN -> ReLU -> conv3 1x1 -> L2-normalise (rows = level-0 texels)
    const int HW4 = g.H4 * g.W4;
    const int64_t Mc = (int64_t)tc * HW4;
    const float* srcs[4] = {Wk.fx[0], Wk.fx[1], Wk.fx[2], Wk.fx[3]};
    CK(launch_upsample_concat_split(srcs, kStageC, kStageCp, g.h, g.w, tc, kCatCp, g.H4, g.W4, Wk.cat, s), "upsample concat");
    CK(launch_conv3x3_tc(Wk.cat, W16(E.conv2), B32(E.conv2), tc, g.H4, g.W4, kCatCp, kEncMid, Wk.fy, nsm, s), "conv2");
    CK(launch_instnorm_stats(Wk.fy, tc, HW4, kEncMid, 1e-5f, Wk.stats, Wk.stat_scratch, s), "instnorm stats");
    CK(launch_instnorm_relu_split(Wk.fy, Wk.stats, Mc, HW4, kEncMid, Wk.sy, s), "instnorm relu split");
    float* f0 = pyr + lay.off[0] + (int64_t)t0 * HW4 * kD;
    {
      GemmProblem q;
      q.x_split = Wk.sy;
      q.w_split = reinterpret_cast<const __nv_bfloat16*>(pk + E.conv3.w);
      q.M = (int)Mc; q.N = kD; q.Kpad = E.conv3.Kpad;
      q.epi.bias = reinterpret_cast<const float*>(pk + E.conv3.b);
      q.epi.out_f32 = f0; q.epi.ld_f32 = kD;
      const char* gerr = nullptr;
      int rc = gemm_launch(q, g_opt_gemm, nsm, s, &gerr);
      if (rc != 0) { snprintf(g_err, sizeof(g_err), "encoder conv3 gemm: %s (%s)", cudaGetErrorString((cudaError_t)rc), gerr ? gerr : ""); return CT3_ECUDA; }
    }
    CK(launch_l2norm_rows(f0, Mc, f0, s), "l2norm rows");
  }
  CK(launch_pyramid_pools(T, g.H4, g.W4, pyr, s), "pyramid pools");
  return 0;
}

}  // extern "C"
