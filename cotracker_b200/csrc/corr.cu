// corr.cu -- fused bilinear sampling + 4-D correlation ("CorrBlock.sample" of the north star):
//   get_correlation_feat (cotracker3_online.py:130-143, F.grid_sample align_corners=True, padding "border")
//   + einsum("btnhwc,bnijc->btnhwij") (cotracker3_offline.py:154-156), all 4 pyramid levels in one launch.
//
//   vol[(n,t,l)][(a*7+b)*49 + (i*7+j)] = < bilinear(F_l[t], cx/2^l + a-3, cy/2^l + b-3) , S_l[n, i*7+j, :] >
//
// The 10 GB/iteration `corr_feat` tensor of the reference is never materialised: the 49 sampled feature
// vectors of a (t,n,level) live in shared memory only.  Output is written directly in the split-bf16 layout
// the correlation-MLP GEMM consumes (row (n*T+t)*4+level, 2432-padded hi plane | lo plane).
#include "kernels.cuh"

namespace ct3 {
namespace {

constexpr int kLd = kD + 4;  // smem row stride (floats): keeps float4 alignment, rotates banks

struct CorrArgs {
  const float* pyr;
  PyramidLayout lay;
  const float* support;        // [4][49, N, 128]
  const uint8_t* track_valid;  // [N] or null
  const float* coords;         // [T, N, 2]
  int T, N;
  __nv_bfloat16* vol;          // [N*T*4, 2*kVolPad]
  FrameMap fm;                 // pyramid frame of (track, t)
};

// v1: SIMT fp32.  block = (track n, level l), loops over frames.  256 threads.
//   phase 1: 8 warps build A[49][128] (one warp = one sample at a time, lane = 4 channels, 4 coalesced taps)
//   phase 2: 13x13 threads each own a 4x4 tile of the 49x49 output, K=128 from shared memory
__global__ void __launch_bounds__(256)
corr_sample_simt_kernel(CorrArgs g) {
  extern __shared__ float sm[];
  float* S = sm;                 // [52][kLd] (rows 49..51 zero)
  float* A = sm + 52 * kLd;      // [52][kLd]
  const int n = blockIdx.x, l = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int H = g.lay.h[l], W = g.lay.w[l];
  const bool valid = g.track_valid == nullptr || g.track_valid[n] != 0;

  for (int i = tid; i < 52 * (kD / 4); i += 256) {
    const int p = i / (kD / 4), c4 = i % (kD / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p < kP && valid)
      v = reinterpret_cast<const float4*>(g.support + ((int64_t)l * kP * g.N + (int64_t)p * g.N + n) * kD)[c4];
    reinterpret_cast<float4*>(S + p * kLd)[c4] = v;
    if (p >= kP) reinterpret_cast<float4*>(A + p * kLd)[c4] = make_float4(0.f, 0.f, 0.f, 0.f);
  }

  const float inv = 1.0f / (float)(1 << l);
  const int ti = tid / 13, tj = tid % 13;  // output tile (rows ti*4.., cols tj*4..) for tid < 169
  const int32_t* frow = frame_row(g.fm, n, g.T);

  for (int t = 0; t < g.T; ++t) {
    const float cx = g.coords[((int64_t)t * g.N + n) * 2 + 0] * inv;
    const float cy = g.coords[((int64_t)t * g.N + n) * 2 + 1] * inv;
    const float* fm = g.pyr + g.lay.off[l] + (int64_t)map_frame(frow, t) * H * W * kD;
    for (int p = warp; p < kP; p += 8) {
      const int a = p / 7, b = p % 7;
      const float x = fminf(fmaxf(cx + (float)(a - kR), 0.f), (float)(W - 1));
      const float y = fminf(fmaxf(cy + (float)(b - kR), 0.f), (float)(H - 1));
      const float xf = floorf(x), yf = floorf(y);
      const int x0 = (int)xf, y0 = (int)yf;
      const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
      const float wx = x - xf, wy = y - yf;
      const float4 v00 = reinterpret_cast<const float4*>(fm + ((int64_t)y0 * W + x0) * kD)[lane];
      const float4 v01 = reinterpret_cast<const float4*>(fm + ((int64_t)y0 * W + x1) * kD)[lane];
      const float4 v10 = reinterpret_cast<const float4*>(fm + ((int64_t)y1 * W + x0) * kD)[lane];
      const float4 v11 = reinterpret_cast<const float4*>(fm + ((int64_t)y1 * W + x1) * kD)[lane];
      float4 o;
      o.x = (1.f - wy) * ((1.f - wx) * v00.x + wx * v01.x) + wy * ((1.f - wx) * v10.x + wx * v11.x);
      o.y = (1.f - wy) * ((1.f - wx) * v00.y + wx * v01.y) + wy * ((1.f - wx) * v10.y + wx * v11.y);
      o.z = (1.f - wy) * ((1.f - wx) * v00.z + wx * v01.z) + wy * ((1.f - wx) * v10.z + wx * v11.z);
      o.w = (1.f - wy) * ((1.f - wx) * v00.w + wx * v01.w) + wy * ((1.f - wx) * v10.w + wx * v11.w);
      reinterpret_cast<float4*>(A + p * kLd)[lane] = o;
    }
    __syncthreads();

    __nv_bfloat16* row = g.vol + (((int64_t)n * g.T + t) * kL + l) * (2 * kVolPad);
    if (tid < 169) {
      float acc[4][4] = {};
      const float* ap = A + (ti * 4) * kLd;
      const float* sp = S + (tj * 4) * kLd;
#pragma unroll 4
      for (int k = 0; k < kD; k += 4) {
        float4 av[4], sv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          av[i] = *reinterpret_cast<const float4*>(ap + i * kLd + k);
          sv[i] = *reinterpret_cast<const float4*>(sp + i * kLd + k);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            acc[i][j] = fmaf(av[i].x, sv[j].x, acc[i][j]);
            acc[i][j] = fmaf(av[i].y, sv[j].y, acc[i][j]);
            acc[i][j] = fmaf(av[i].z, sv[j].z, acc[i][j]);
            acc[i][j] = fmaf(av[i].w, sv[j].w, acc[i][j]);
          }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int pa = ti * 4 + i;
        if (pa >= kP) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int ps = tj * 4 + j;
          if (ps >= kP) continue;
          const bf16pair v = split_bf16(acc[i][j]);
          row[pa * kP + ps] = v.hi;
          row[kVolPad + pa * kP + ps] = v.lo;
        }
      }
    } else if (tid < 169 + (kVolPad - kVol)) {
      const int c = kVol + (tid - 169);  // zero the K padding of both planes
      row[c] = __float2bfloat16_rn(0.f);
      row[kVolPad + c] = __float2bfloat16_rn(0.f);
    }
    __syncthreads();
  }
}

}  // namespace

bool corr_uses_patch_kernel(int impl, bool have_pyr_split, int T, int H4, int W4) {
  return impl == 0 && have_pyr_split && corr_patch_supported(T, H4, W4);
}

cudaError_t launch_corr_sample(const float* pyr, const __nv_bfloat16* pyr_split, int H4, int W4, const float* support,
                               const uint8_t* track_valid, const float* coords, int T, int N, int n0, int count,
                               __nv_bfloat16* vol_split, int impl, int mode, int vol16, int num_sms, cudaStream_t s,
                               int T_pyr, const FrameMap& fm_all) {
  // track n of the launch is track n0 + n of the state: support [4][49, N, 128], track_valid [N] and coords [T, N, 2]
  // keep pitch N, so moving their base to track n0 is the whole change for the kernels
  support += (int64_t)n0 * kD;
  if (track_valid) track_valid += n0;
  coords += (int64_t)n0 * 2;
  FrameMap fm = fm_all;
  fm.n0 = n0;
  if (corr_uses_patch_kernel(impl, pyr_split != nullptr, T_pyr, H4, W4)) {
    if (mode != 3)
      return launch_corr_patch_t(pyr_split, H4, W4, support, track_valid, coords, T, N, count, vol_split, vol16,
                                 mode == 1, num_sms, s, T_pyr, fm);
    return launch_corr_patch_tc(pyr_split, H4, W4, support, track_valid, coords, T, N, count, vol_split, vol16, num_sms,
                                s, T_pyr, fm);
  }
  if (vol16) return cudaErrorInvalidValue;   // only the patch kernel writes the single-plane volume
  if (impl != 1)
    return launch_corr_sample_tc(pyr, H4, W4, support, track_valid, coords, T, N, count, vol_split, num_sms, s, T_pyr,
                                 fm);
  CorrArgs g;  // impl 1: exact-fp32 SIMT verification kernel
  g.pyr = pyr;
  g.lay = pyramid_layout(T_pyr, H4, W4);
  g.support = support;
  g.track_valid = track_valid;
  g.coords = coords;
  g.T = T;
  g.N = N;
  g.vol = vol_split;
  g.fm = fm;
  const int smem = 2 * 52 * kLd * (int)sizeof(float);  // 54.9 KB
  static DeviceOnce attr;
  {
    cudaError_t e = once_per_device(attr, [&] {
      return cudaFuncSetAttribute(corr_sample_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    });
    if (e != cudaSuccess) return e;
  }
  dim3 grid(count, kL);
  corr_sample_simt_kernel<<<grid, 256, smem, s>>>(g);
  return cudaGetLastError();
}

}  // namespace ct3
