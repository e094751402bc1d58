// api_encoder.cu -- the encoder entry points of the C ABI (see include/ct3_b200.h): the encoder tail on the GEMM engine
// (ct3_enc_tail*) and the whole CNN encoder (ct3_encoder*), both ending in the L2-normalised 4-level pyramid.
#include <string>
#include <vector>

#include "abi.cuh"

using namespace ct3;

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
  Carver c(base);
  w.a = (__nv_bfloat16*)c.take(Mc * 2 * pad64(kEncK) * 2);
  w.y = (float*)c.take(Mc * kEncMid * 4);
  w.ys = (__nv_bfloat16*)c.take(Mc * 2 * kEncMid * 2);
  w.stats = (float*)c.take((size_t)w.tc * kEncMid * 2 * 4);
  w.stat_scratch = c.take(instnorm_scratch_bytes(w.tc, kEncMid));
  w.total = c.off;
  return w;
}

// The end of both encoders for frames [t0, t0+tc) of T: conv3 (1x1, 256 -> 128) of the split rows ys straight into
// level 0 of the pyramid (its rows (t,y,x) are the channels-last texels), L2-normalised; after the last chunk, the
// pools of levels 1..3.
// A trace sink (ct3_encoder_trace) takes a copy of conv3's output between the GEMM and the in-place L2 norm.
struct EncTrace;
int trace_put(EncTrace* tr, const void* src, size_t bytes, cudaStream_t s);

int pyramid_tail(const uint8_t* pk, const Lin& conv3, const __nv_bfloat16* ys, int T, int t0, int tc, int H4, int W4,
                 float* pyr, cudaStream_t s, EncTrace* tr = nullptr) {
  const int64_t Mc = (int64_t)tc * H4 * W4;
  float* f0 = pyr + pyramid_layout(T, H4, W4).off[0] + (int64_t)t0 * H4 * W4 * kD;
  if (int rc = run_gemm(linear_problem(ys, pk + conv3.w, pk + conv3.b, Mc, kD, conv3.Kpad, f0), g_opt_gemm, s,
                        "encoder conv3 gemm"))
    return rc;
  if (tr)
    if (int rc = trace_put(tr, f0, (size_t)Mc * kD * 4, s)) return rc;
  CK(launch_l2norm_rows(f0, Mc, f0, s), "l2norm rows");
  if (t0 + tc == T) CK(launch_pyramid_pools(T, H4, W4, pyr, s), "pyramid pools");
  return 0;
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
  if (int rc = check_space(packed_bytes, E.total, "packed buffer")) return rc;
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
  if (int rc = check_pyramid(T, H4, W4)) return rc;
  *out_bytes = enc_carve(nullptr, T, H4, W4).total;
  return 0;
}

int ct3_enc_tail(const void* packed, const float* cat, int T, int H4, int W4, float* pyr, void* workspace,
                 size_t workspace_bytes, ct3_stream_t stream) {
  if (!packed || !cat || !pyr || !workspace) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = check_pyramid(T, H4, W4)) return rc;
  if (int rc = check_aligned(workspace, "workspace")) return rc;
  const EncWs W = enc_carve(workspace, T, H4, W4);
  if (int rc = check_space(workspace_bytes, W.total, "workspace")) return rc;
  const EncLayout& E = enc_layout();
  const uint8_t* pk = reinterpret_cast<const uint8_t*>(packed);
  cudaStream_t s = (cudaStream_t)stream;
  const int HW = H4 * W4;
  for (int t0 = 0; t0 < T; t0 += W.tc) {
    const int tc = (T - t0) < W.tc ? (T - t0) : W.tc;
    const int Mc = tc * HW;
    CK(launch_im2col3x3_split(cat + (int64_t)t0 * kEncCin * HW, tc, kEncCin, H4, W4, E.conv2.Kpad, W.a, s),
       "im2col conv2");
    if (int rc = run_gemm(linear_problem(W.a, pk + E.conv2.w, pk + E.conv2.b, Mc, kEncMid, E.conv2.Kpad, W.y),
                          g_opt_gemm, s, "enc conv2 gemm"))
      return rc;
    CK(launch_instnorm_stats(W.y, tc, HW, kEncMid, 1e-5f, W.stats, W.stat_scratch, s), "instnorm stats");
    CK(launch_instnorm_relu_split(W.y, W.stats, (int64_t)Mc, HW, kEncMid, W.ys, s), "instnorm relu split");
    if (int rc = pyramid_tail(pk, E.conv3, W.ys, T, t0, tc, H4, W4, pyr, s)) return rc;
  }
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
  Carver c(base);
  w.fy = (float*)c.take(fy * 4);
  w.fyd = (float*)c.take(fyd * 4);
  for (int s = 0; s < 4; ++s) w.fx[s] = (float*)c.take(P[s] * kStageCp[s] * 4);
  w.sx = (__nv_bfloat16*)c.take(sact * 2);
  w.sy = (__nv_bfloat16*)c.take(sact * 2);
  w.gat = (__nv_bfloat16*)c.take(gat * 2);
  w.gat_d = (__nv_bfloat16*)c.take(gat_d * 2);
  w.cat = (__nv_bfloat16*)c.take(P4 * 2 * kCatCp * 2);
  w.stats = (float*)c.take((size_t)w.tc * 256 * 2 * 4);
  w.stats_d = (float*)c.take((size_t)w.tc * 256 * 2 * 4);
  w.stat_scratch = c.take(instnorm_scratch_bytes(w.tc, 256));
  w.total = c.off;
  return w;
}


// ct3_encoder / ct3_encoder_workspace_bytes: T >= 1, H, W >= 16 and a 4-level pyramid at H/4 x W/4, which makes the
// smallest frame 32 x 32 (include/ct3_b200.h)
int check_encoder_shape(int T, int H, int W) {
  if (T < 1 || H < 16 || W < 16) return fail(CT3_EINVAL, "encoder: need T >= 1 and H, W >= 16%s");
  return check_pyramid(T, H / 4, W / 4);
}

// ---- ct3_encoder_trace: the links of one chunk, each 256-byte aligned in the caller's buffer, in launch order
struct EncTrace {
  uint8_t* base = nullptr;
  size_t off[CT3_ENCODER_TRACE_LINKS] = {}, bytes[CT3_ENCODER_TRACE_LINKS] = {};
  int n = 0;   // links copied so far
};
// fills tr.off / tr.bytes for T (<= 16) frames of H x W; returns the total bytes
size_t trace_layout(EncTrace& tr, int T, int H, int W) {
  const EncGeom g = enc_geom(H, W);
  int n = 0;
  size_t off = 0;
  auto link = [&](int64_t rows, int C, int esz) {
    tr.off[n] = off;
    tr.bytes[n] = (size_t)rows * C * esz;
    off = align_up(off + tr.bytes[n]);
    ++n;
  };
  auto unit1 = [&](int64_t rows, int Cp) {   // a stride-1 residual unit
    link(rows, Cp, 4); link(T, 2 * Cp, 4); link(rows, 2 * Cp, 2);
    link(rows, Cp, 4); link(T, 2 * Cp, 4); link(rows, Cp, 4); link(rows, 2 * Cp, 2);
  };
  int64_t rows = (int64_t)T * g.h[0] * g.w[0];
  link(rows, 64, 4); link(T, 2 * 64, 4); link(rows, 64, 4); link(rows, 2 * 64, 2);
  for (int st = 0; st < 4; ++st) {
    const int Cp = kStageCp[st];
    rows = (int64_t)T * g.h[st] * g.w[st];
    if (st > 0) {
      const int Cin = kStageCp[st - 1];
      link(rows, 2 * 9 * Cin, 2); link(rows, 2 * Cin, 2);
      link(rows, Cp, 4); link(T, 2 * Cp, 4); link(rows, 2 * Cp, 2);
      link(rows, Cp, 4); link(T, 2 * Cp, 4);
      link(rows, Cp, 4); link(T, 2 * Cp, 4);
      link(rows, Cp, 4); link(rows, 2 * Cp, 2);
    }
    for (int u = (st > 0 ? 1 : 0); u < 2; ++u) unit1(rows, Cp);
  }
  const int64_t rows4 = (int64_t)T * g.H4 * g.W4;
  link(rows4, 2 * kCatCp, 2); link(rows4, kEncMid, 4); link(T, 2 * kEncMid, 4); link(rows4, 2 * kEncMid, 2);
  link(rows4, kD, 4);
  return off;
}

// the next link of the trace: its size must be the layout's
int trace_put(EncTrace* tr, const void* src, size_t bytes, cudaStream_t s) {
  if (tr->n >= CT3_ENCODER_TRACE_LINKS || bytes != tr->bytes[tr->n])
    return fail(CT3_EINVAL, "encoder trace: links out of step with the layout%s");
  CK(cudaMemcpyAsync(tr->base + tr->off[tr->n], src, bytes, cudaMemcpyDeviceToDevice, s), "encoder trace copy");
  ++tr->n;
  return 0;
}

// ct3_encoder with an optional trace sink: tr == nullptr launches exactly what ct3_encoder launches; otherwise each
// link's output is also copied into the trace buffer (trace_layout's order) right after the launch that writes it.
int encoder_run(const void* packed, const float* frames, int T, int H, int W, float* pyr, void* workspace,
                size_t workspace_bytes, cudaStream_t s, EncTrace* tr) {
  if (!packed || !frames || !pyr || !workspace) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = check_encoder_shape(T, H, W)) return rc;
  const EncGeom g = enc_geom(H, W);
  if (int rc = check_aligned(workspace, "workspace")) return rc;
  const EncFullWs Wk = enc_full_carve(workspace, T, H, W);
  if (int rc = check_space(workspace_bytes, Wk.total, "workspace")) return rc;
  const EncFull& E = enc_full();
  const uint8_t* pk = reinterpret_cast<const uint8_t*>(packed);
  const int nsm = num_sms();
  auto W16 = [&](const ConvW& c) { return reinterpret_cast<const __nv_bfloat16*>(pk + c.w); };
  auto B32 = [&](const ConvW& c) { return reinterpret_cast<const float*>(pk + c.b); };
  // y = GEMM(gathered rows, conv weights): the stride-2 convolutions
  auto gemm_rows = [&](const __nv_bfloat16* rows, const ConvW& c, int64_t M, float* y) {
    return run_gemm(linear_problem(rows, W16(c), B32(c), M, c.cout_pad, c.taps * c.cp, y), g_opt_gemm, s,
                    "encoder gemm");
  };
  // TAP(p, rows, C, element bytes): the trace copy of the [rows, C] output p of the launch just made
#define TAP(p, rows, C, esz) \
  if (tr)                    \
    if (int rc = trace_put(tr, p, (size_t)(rows) * (C) * (esz), s)) return rc
  const int chunks = (T + Wk.tc - 1) / Wk.tc;
  ProfScope ps_all(s, CAT_ENC, 0.0, chunks * 90 + 3);   // kernels launched per 16-frame chunk + the 3 pyramid pools
  for (int t0 = 0; t0 < T; t0 += Wk.tc) {
    const int tc = (T - t0) < Wk.tc ? (T - t0) : Wk.tc;
    // ---- stem: conv1 7x7/2 -> IN -> ReLU
    int h = g.h[0], w = g.w[0], C = 64;
    int64_t rows = (int64_t)tc * h * w;
    CK(launch_conv_stem(frames + (int64_t)t0 * 3 * H * W, reinterpret_cast<const float*>(pk + E.stem_w),
                        reinterpret_cast<const float*>(pk + E.stem_b), tc, H, W, Wk.fy, s), "conv1");
    TAP(Wk.fy, rows, C, 4);
    CK(launch_instnorm_stats(Wk.fy, tc, h * w, C, 1e-5f, Wk.stats, Wk.stat_scratch, s), "stem stats");
    TAP(Wk.stats, tc, 2 * C, 4);
    CK(launch_norm_act(Wk.fy, Wk.stats, nullptr, nullptr, 0, rows, h * w, C, Wk.fx[0], Wk.sx, s), "stem norm");
    TAP(Wk.fx[0], rows, C, 4);
    TAP(Wk.sx, rows, 2 * C, 2);
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
        TAP(Wk.gat, orows, 2 * 9 * Cin, 2);
        CK(launch_gather_s2(Wk.sx, tc, h, w, Cin, 1, Wk.gat_d, s), "gather 1x1/2");
        TAP(Wk.gat_d, orows, 2 * Cin, 2);
        if (int rc = gemm_rows(Wk.gat, E.unit[st][0][0], orows, Wk.fy)) return rc;
        TAP(Wk.fy, orows, Cp, 4);
        CK(launch_instnorm_stats(Wk.fy, tc, ho * wo, Cp, 1e-5f, Wk.stats, Wk.stat_scratch, s), "stats");
        TAP(Wk.stats, tc, 2 * Cp, 4);
        CK(launch_norm_act(Wk.fy, Wk.stats, nullptr, nullptr, 0, orows, ho * wo, Cp, nullptr, Wk.sy, s), "norm");
        TAP(Wk.sy, orows, 2 * Cp, 2);
        CK(launch_conv3x3_tc(Wk.sy, W16(E.unit[st][0][1]), B32(E.unit[st][0][1]), tc, ho, wo, Cp, Cp, Wk.fy, nsm, s), "conv");
        TAP(Wk.fy, orows, Cp, 4);
        CK(launch_instnorm_stats(Wk.fy, tc, ho * wo, Cp, 1e-5f, Wk.stats, Wk.stat_scratch, s), "stats");
        TAP(Wk.stats, tc, 2 * Cp, 4);
        if (int rc = gemm_rows(Wk.gat_d, E.down[st], orows, Wk.fyd)) return rc;
        TAP(Wk.fyd, orows, Cp, 4);
        CK(launch_instnorm_stats(Wk.fyd, tc, ho * wo, Cp, 1e-5f, Wk.stats_d, Wk.stat_scratch, s), "stats");
        TAP(Wk.stats_d, tc, 2 * Cp, 4);
        CK(launch_norm_act(Wk.fy, Wk.stats, Wk.fyd, Wk.stats_d, 2, orows, ho * wo, Cp, X, Wk.sx, s), "norm");
        TAP(X, orows, Cp, 4);
        TAP(Wk.sx, orows, 2 * Cp, 2);
        h = ho; w = wo; rows = orows;
      }
      for (int u = (st > 0 ? 1 : 0); u < 2; ++u) {
        // stride-1 unit: out = relu(x + relu(IN(conv(relu(IN(conv(x)))))))
        CK(launch_conv3x3_tc(Wk.sx, W16(E.unit[st][u][0]), B32(E.unit[st][u][0]), tc, h, w, Cp, Cp, Wk.fy, nsm, s), "conv");
        TAP(Wk.fy, rows, Cp, 4);
        CK(launch_instnorm_stats(Wk.fy, tc, h * w, Cp, 1e-5f, Wk.stats, Wk.stat_scratch, s), "stats");
        TAP(Wk.stats, tc, 2 * Cp, 4);
        CK(launch_norm_act(Wk.fy, Wk.stats, nullptr, nullptr, 0, rows, h * w, Cp, nullptr, Wk.sy, s), "norm");
        TAP(Wk.sy, rows, 2 * Cp, 2);
        CK(launch_conv3x3_tc(Wk.sy, W16(E.unit[st][u][1]), B32(E.unit[st][u][1]), tc, h, w, Cp, Cp, Wk.fy, nsm, s), "conv");
        TAP(Wk.fy, rows, Cp, 4);
        CK(launch_instnorm_stats(Wk.fy, tc, h * w, Cp, 1e-5f, Wk.stats, Wk.stat_scratch, s), "stats");
        TAP(Wk.stats, tc, 2 * Cp, 4);
        CK(launch_norm_act(Wk.fy, Wk.stats, X, nullptr, 1, rows, h * w, Cp, X, Wk.sx, s), "norm");
        TAP(X, rows, Cp, 4);
        TAP(Wk.sx, rows, 2 * Cp, 2);
      }
    }
    // ---- resize + concat -> conv2 3x3 -> IN -> ReLU -> conv3 1x1 -> L2-normalise (rows = level-0 texels)
    const int HW4 = g.H4 * g.W4;
    const float* srcs[4] = {Wk.fx[0], Wk.fx[1], Wk.fx[2], Wk.fx[3]};
    const int64_t rows4 = (int64_t)tc * HW4;
    CK(launch_upsample_concat_split(srcs, kStageC, kStageCp, g.h, g.w, tc, kCatCp, g.H4, g.W4, Wk.cat, s), "upsample concat");
    TAP(Wk.cat, rows4, 2 * kCatCp, 2);
    CK(launch_conv3x3_tc(Wk.cat, W16(E.conv2), B32(E.conv2), tc, g.H4, g.W4, kCatCp, kEncMid, Wk.fy, nsm, s), "conv2");
    TAP(Wk.fy, rows4, kEncMid, 4);
    CK(launch_instnorm_stats(Wk.fy, tc, HW4, kEncMid, 1e-5f, Wk.stats, Wk.stat_scratch, s), "instnorm stats");
    TAP(Wk.stats, tc, 2 * kEncMid, 4);
    CK(launch_instnorm_relu_split(Wk.fy, Wk.stats, rows4, HW4, kEncMid, Wk.sy, s), "instnorm relu split");
    TAP(Wk.sy, rows4, 2 * kEncMid, 2);
    if (int rc = pyramid_tail(pk, E.conv3, Wk.sy, T, t0, tc, g.H4, g.W4, pyr, s, tr)) return rc;
  }
#undef TAP
  return 0;
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
  if (int rc = check_space(packed_bytes, E.total, "packed buffer")) return rc;
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
  if (int rc = check_encoder_shape(T, H, W)) return rc;
  *out_bytes = enc_full_carve(nullptr, T, H, W).total;
  return 0;
}

int ct3_encoder(const void* packed, const float* frames, int T, int H, int W, float* pyr, void* workspace,
                size_t workspace_bytes, ct3_stream_t stream) {
  return encoder_run(packed, frames, T, H, W, pyr, workspace, workspace_bytes, (cudaStream_t)stream, nullptr);
}

int ct3_encoder_trace_layout(int T, int H, int W, int64_t* offsets, int64_t* bytes, size_t* total_bytes) {
  if (!total_bytes) return fail(CT3_EINVAL, "null total_bytes%s");
  if (int rc = check_encoder_shape(T, H, W)) return rc;
  if (T > 16) return fail(CT3_EINVAL, "encoder trace: one chunk, T <= 16%s");
  EncTrace tr;
  *total_bytes = trace_layout(tr, T, H, W);
  for (int i = 0; i < CT3_ENCODER_TRACE_LINKS; ++i) {
    if (offsets) offsets[i] = (int64_t)tr.off[i];
    if (bytes) bytes[i] = (int64_t)tr.bytes[i];
  }
  return 0;
}

int ct3_encoder_trace(const void* packed, const float* frames, int T, int H, int W, float* pyr, void* trace,
                      size_t trace_bytes, void* workspace, size_t workspace_bytes, ct3_stream_t stream) {
  if (!trace) return fail(CT3_EINVAL, "null argument%s");
  if (int rc = check_encoder_shape(T, H, W)) return rc;
  if (T > 16) return fail(CT3_EINVAL, "encoder trace: one chunk, T <= 16%s");
  if (int rc = check_aligned(trace, "trace")) return rc;
  EncTrace tr;
  tr.base = reinterpret_cast<uint8_t*>(trace);
  if (int rc = check_space(trace_bytes, trace_layout(tr, T, H, W), "trace buffer")) return rc;
  if (int rc = encoder_run(packed, frames, T, H, W, pyr, workspace, workspace_bytes, (cudaStream_t)stream, &tr))
    return rc;
  return tr.n == CT3_ENCODER_TRACE_LINKS ? 0 : fail(CT3_EINVAL, "encoder trace: links out of step with the layout%s");
}

}  // extern "C"
