// abi.cuh -- host-side pieces shared by the translation units of the C ABI (api.cu, api_loop.cu, api_encoder.cu):
// the error state, the per-thread options, the profiler, workspace carving and GEMM launches.  Host code only.
#pragma once
#include <stdint.h>

#include "../../include/ct3_b200.h"
#include "gemm.cuh"
#include "kernels.cuh"

namespace ct3 {

// ---- errors: every entry point returns a CT3_E* code and leaves its message in the thread's g_err (ct3_last_error)
extern thread_local char g_err[512];
int fail(int code, const char* fmt, const char* detail = "");
int fail_cuda(cudaError_t e, const char* where);
// rc: a launcher's cudaError_t as int; detail: its error string (may be null) -> "what: error (detail)", CT3_ECUDA
int fail_launch(int rc, const char* what, const char* detail);
#define CK(call, where)                                  \
  do {                                                   \
    cudaError_t e__ = (call);                            \
    if (e__ != cudaSuccess) return fail_cuda(e__, where); \
  } while (0)

// ---- per-thread options (ct3_set_option; names, ranges and defaults in api.cu)
enum { OPT_GEMM = 0, OPT_CORR, OPT_ATTN, OPT_PREC_CORR, OPT_PREC_FC1, OPT_FUSE, OPT_COUNT };
extern thread_local int g_opt[OPT_COUNT];
#define g_opt_gemm g_opt[OPT_GEMM]
#define g_opt_corr g_opt[OPT_CORR]
#define g_opt_attn g_opt[OPT_ATTN]

// ---- optional live profiler: CUDA events around launches, summed per kernel category (ct3_profile_read)
enum { CAT_CORR = 0, CAT_GEMM = 1, CAT_ATTN = 2, CAT_LN = 3, CAT_MISC = 4, CAT_ENC = 5, CAT_QKVA = 6, CAT_COUNT = 7 };
// records the work enqueued on s during its lifetime under category cat (cat < 0: nothing)
struct ProfScope {
  cudaStream_t s; int cat; double flops; int launches; cudaEvent_t a = nullptr, b = nullptr;
  ProfScope(cudaStream_t s_, int cat_, double flops_ = 0.0, int launches_ = 1);
  ~ProfScope();
};

int num_sms();   // of the CURRENT device (one process may drive several GPUs)
inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }
inline int pad64(int k) { return (k + 63) / 64 * 64; }

// ---- packed weights: a linear layer at byte offsets of the caller's packed buffer
struct Lin {
  size_t w = 0, b = 0;  // byte offsets: split weights [N, 2*Kpad] bf16 ; bias [N] fp32
  int N = 0, K = 0, Kpad = 0;
};
inline void place_lin(Lin& l, int N, int K, size_t& off) {
  l.N = N;
  l.K = K;
  l.Kpad = pad64(K);
  l.w = off;
  off = align_up(off + (size_t)N * 2 * l.Kpad * sizeof(__nv_bfloat16));
  l.b = off;
  off = align_up(off + (size_t)N * sizeof(float));
}

// ---- argument checks
// the shape check of every entry point that takes a pyramid of T frames of H4 x W4
inline int check_pyramid(int T, int H4, int W4) { return ct3_pyramid_layout(T, H4, W4, nullptr, nullptr, nullptr, nullptr); }
inline int check_aligned(const void* p, const char* name) {
  return ((uintptr_t)p & 255) ? fail(CT3_EINVAL, "%s must be 256-byte aligned", name) : 0;
}
inline int check_space(size_t have, size_t need, const char* name) {
  return have < need ? fail(CT3_ENOSPC, "%s too small", name) : 0;
}

// ---- caller workspaces: consecutive buffers, each 1024-byte aligned; a null base only measures (off = total bytes)
struct Carver {
  uint8_t* base;
  size_t off = 0;
  explicit Carver(void* b) : base(reinterpret_cast<uint8_t*>(b)) {}
  void* take(size_t bytes) {
    uint8_t* r = base + off;
    off = align_up(off + bytes, 1024);
    return r;
  }
};

// ---- GEMM engine
// a plain linear layer y[M, N] = x_split w_split^T + bias, fp32 rows of pitch N
GemmProblem linear_problem(const void* x_split, const void* w_split, const void* bias, int64_t M, int N, int Kpad,
                           float* y);
// launches p on engine impl (0 wgmma, 1 SIMT); a problem gemm_check rejects becomes CT3_EINVAL with "what: reason"
// before any launch, a failed launch CT3_ECUDA with "what: error (detail)"
int run_gemm(const GemmProblem& p, int impl, cudaStream_t s, const char* what);

}  // namespace ct3
