// enc_tail.cu -- the dominant tail of the CNN encoder (SURVEY.md 8(f) rank 1; reference blocks.py:215-218 and
// cotracker3_offline.py:92-117) on the split-bf16x3 tensor-core engine:
//     cat[T,416,H,W] -> conv2 3x3 (416->256) -> InstanceNorm -> ReLU -> conv3 1x1 (256->128) -> L2-normalise -> pyramid
// conv2 is 45 % and conv3 1.5 % of the encoder FLOPs.  The 3x3 convolution is an explicit im2col (written directly in
// the split-bf16 operand layout, K = c*9 + ky*3 + kx = the natural flattening of the [256,416,3,3] weight) followed
// by the cta_group::2 GEMM; both GEMM outputs are NHWC, i.e. row m = (t,y,x), so conv3's output rows ARE the
// channels-last level-0 texels and the planar->channels-last transpose of prepare_pyramid disappears.
#include "kernels.cuh"

namespace ct3 {
namespace {

// block: 32 consecutive x of one (t,y) x 64 consecutive k.  Read coalesced along x, write coalesced along k.
__global__ void __launch_bounds__(256)
im2col3x3_split_kernel(const float* __restrict__ in, int T, int C, int H, int W, int Kpad,
                       __nv_bfloat16* __restrict__ out) {
  __shared__ float tile[64][33];
  const int x0 = blockIdx.x * 32, k0 = blockIdx.y * 64;
  const int ty = blockIdx.z;   // t*H + y
  const int t = ty / H, y = ty % H;
  const int K = C * 9;
  {
    const int xi = threadIdx.x & 31;
    const int x = x0 + xi;
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      const int kk = p * 8 + (threadIdx.x >> 5);
      const int k = k0 + kk;
      float v = 0.f;
      if (k < K && x < W) {
        const int c = k / 9, r = k % 9;
        const int yy = y + r / 3 - 1, xx = x + r % 3 - 1;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = in[(((int64_t)t * C + c) * H + yy) * W + xx];
      }
      tile[kk][xi] = v;
    }
  }
  __syncthreads();
  {
    const int m = threadIdx.x >> 3, kq = threadIdx.x & 7;   // 32 rows x 8 groups of 8 k
    const int x = x0 + m;
    if (x < W) {
      uint32_t hi[4], lo[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) split2(tile[kq * 8 + 2 * i][m], tile[kq * 8 + 2 * i + 1][m], hi[i], lo[i]);
      __nv_bfloat16* row = out + ((int64_t)ty * W + x) * (2 * (int64_t)Kpad) + k0 + kq * 8;
      *reinterpret_cast<uint4*>(row) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
      *reinterpret_cast<uint4*>(row + Kpad) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    }
  }
}

// per (t, channel) mean / rstd over the HW rows of an NHWC fp32 tensor [T*HW, C], fp64 accumulation, deterministic:
// stage 1: block (32-channel group, t, split) sums its share of the rows (8 row lanes x rows strided by 8 * splits)
// into part[t][split][c][2]; stage 2: one thread per (t, c) adds the splits in order.  (A single block per (t, 32
// channels) left 32 blocks for the whole GPU on the 64-channel stages: 5.5 ms per step.)
constexpr int kStatSplits = 32;
__global__ void __launch_bounds__(256)
instnorm_partial_kernel(const float* __restrict__ y, int HW, int C, double* __restrict__ part /*[T,splits,C,2]*/) {
  const int t = blockIdx.y, sp = blockIdx.z, c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int r0 = threadIdx.x >> 5;   // 8 row lanes
  double s = 0.0, ss = 0.0;
  const float* base = y + (int64_t)t * HW * C + c;
  for (int r = sp * 8 + r0; r < HW; r += 8 * kStatSplits) {
    const float v = base[(int64_t)r * C];
    s += v;
    ss += (double)v * v;
  }
  __shared__ double sh[2][8][32];
  sh[0][r0][threadIdx.x & 31] = s;
  sh[1][r0][threadIdx.x & 31] = ss;
  __syncthreads();
  if (r0 == 0) {
    for (int i = 1; i < 8; ++i) { s += sh[0][i][threadIdx.x & 31]; ss += sh[1][i][threadIdx.x & 31]; }
    double* o = part + (((int64_t)t * kStatSplits + sp) * C + c) * 2;
    o[0] = s;
    o[1] = ss;
  }
}
__global__ void instnorm_finish_kernel(const double* __restrict__ part, int T, int HW, int C, float eps,
                                       float* __restrict__ stats /*[T,C,2]*/) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T * C) return;
  const int t = i / C, c = i % C;
  double s = 0.0, ss = 0.0;
  for (int sp = 0; sp < kStatSplits; ++sp) {
    const double* p = part + (((int64_t)t * kStatSplits + sp) * C + c) * 2;
    s += p[0];
    ss += p[1];
  }
  const double mean = s / HW;
  const double var = fmax(ss / HW - mean * mean, 0.0);
  stats[(int64_t)i * 2 + 0] = (float)mean;
  stats[(int64_t)i * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
}

// relu((y - mean) * rstd) -> split [rows, 2*C]; one thread = 4 channels of one row
__global__ void instnorm_relu_split_kernel(const float* __restrict__ y, const float* __restrict__ stats, int64_t rows,
                                           int HW, int C, __nv_bfloat16* __restrict__ out) {
  const int64_t total = rows * (C / 4);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % (C / 4));
    const int64_t r = i / (C / 4);
    const int t = (int)(r / HW);
    const float4 v = reinterpret_cast<const float4*>(y)[i];
    const float4* st = reinterpret_cast<const float4*>(stats + ((int64_t)t * C + c4 * 4) * 2);
    const float4 s0 = st[0], s1 = st[1];   // (mean0, rstd0, mean1, rstd1), (mean2, rstd2, mean3, rstd3)
    const float a = fmaxf((v.x - s0.x) * s0.y, 0.f), b = fmaxf((v.y - s0.z) * s0.w, 0.f);
    const float c = fmaxf((v.z - s1.x) * s1.y, 0.f), d = fmaxf((v.w - s1.z) * s1.w, 0.f);
    uint32_t h0, l0, h1, l1;
    split2(a, b, h0, l0);
    split2(c, d, h1, l1);
    __nv_bfloat16* o = out + r * (2 * (int64_t)C) + c4 * 4;
    *reinterpret_cast<uint2*>(o) = make_uint2(h0, h1);
    *reinterpret_cast<uint2*>(o + C) = make_uint2(l0, l1);
  }
}

// x / sqrt(max(sum_c x^2, 1e-12)) per row of 128 (cotracker3_offline.py:92-98); one warp per row, in -> out
__global__ void __launch_bounds__(256)
l2norm_rows_kernel(const float* __restrict__ in, int64_t rows, float* __restrict__ out) {
  const int64_t row = blockIdx.x * 8LL + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float4 v = reinterpret_cast<const float4*>(in + row * kD)[lane];
  const float ss = warp_sum(v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w);
  const float d = sqrtf(fmaxf(ss, 1e-12f));
  reinterpret_cast<float4*>(out + row * kD)[lane] = make_float4(v.x / d, v.y / d, v.z / d, v.w / d);
}

// bilinear (align_corners=True) resize of 4 stage outputs [T,Cs,Hs,Ws] to (H,W) + channel concat -> [T,416,H,W]
// (BasicEncoder._bilinear_intepolate + torch.cat, blocks.py:202-215).  One thread = one output pixel of one channel.
struct UpArgs {
  const float* src[4];
  int c[4], h[4], w[4], coff[4];
};
__global__ void upsample_concat_kernel(UpArgs a, int T, int Ctot, int H, int W, float* __restrict__ out) {
  const int64_t total = (int64_t)T * Ctot * H * W;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    int64_t r = i / W;
    const int y = (int)(r % H);
    r /= H;
    const int cc = (int)(r % Ctot);
    const int t = (int)(r / Ctot);
    int s = 0;
#pragma unroll
    for (int k = 1; k < 4; ++k) s = (cc >= a.coff[k]) ? k : s;
    const int c = cc - a.coff[s], hs = a.h[s], ws = a.w[s];
    const float* p = a.src[s] + ((int64_t)t * a.c[s] + c) * hs * ws;
    float v;
    if (hs == H && ws == W) {
      v = p[(int64_t)y * ws + x];
    } else {
      // area_pixel_compute_source_index(align_corners): src = dst * (in - 1) / (out - 1)
      const float sy = H > 1 ? (float)(hs - 1) / (float)(H - 1) : 0.f, sx = W > 1 ? (float)(ws - 1) / (float)(W - 1) : 0.f;
      const float fy = sy * (float)y, fx = sx * (float)x;
      const int y0 = (int)fy, x0 = (int)fx;
      const int y1 = min(y0 + 1, hs - 1), x1 = min(x0 + 1, ws - 1);
      const float ly = fy - (float)y0, lx = fx - (float)x0;
      const float v00 = p[(int64_t)y0 * ws + x0], v01 = p[(int64_t)y0 * ws + x1];
      const float v10 = p[(int64_t)y1 * ws + x0], v11 = p[(int64_t)y1 * ws + x1];
      v = (1.f - ly) * ((1.f - lx) * v00 + lx * v01) + ly * ((1.f - lx) * v10 + lx * v11);
    }
    out[i] = v;
  }
}

}  // namespace

cudaError_t launch_upsample_concat(const float* const src[4], const int c[4], const int h[4], const int w[4], int T,
                                   int H, int W, float* out, cudaStream_t s) {
  UpArgs a;
  int off = 0;
  for (int k = 0; k < 4; ++k) { a.src[k] = src[k]; a.c[k] = c[k]; a.h[k] = h[k]; a.w[k] = w[k]; a.coff[k] = off; off += c[k]; }
  const int64_t total = (int64_t)T * off * H * W;
  const int blocks = (int)((total + 255) / 256 > 132 * 64 ? 132 * 64 : (total + 255) / 256);
  upsample_concat_kernel<<<blocks, 256, 0, s>>>(a, T, off, H, W, out);
  return cudaGetLastError();
}

cudaError_t launch_im2col3x3_split(const float* in, int T, int C, int H, int W, int Kpad, __nv_bfloat16* out,
                                   cudaStream_t s) {
  dim3 grid((W + 31) / 32, Kpad / 64, T * H);
  if (grid.z > 65535) return cudaErrorInvalidValue;
  im2col3x3_split_kernel<<<grid, 256, 0, s>>>(in, T, C, H, W, Kpad, out);
  return cudaGetLastError();
}
size_t instnorm_scratch_bytes(int T, int C) { return (size_t)T * kStatSplits * C * 2 * sizeof(double); }
cudaError_t launch_instnorm_stats(const float* y, int T, int HW, int C, float eps, float* stats, void* scratch,
                                  cudaStream_t s) {
  dim3 grid(C / 32, T, kStatSplits);
  instnorm_partial_kernel<<<grid, 256, 0, s>>>(y, HW, C, reinterpret_cast<double*>(scratch));
  instnorm_finish_kernel<<<(T * C + 255) / 256, 256, 0, s>>>(reinterpret_cast<const double*>(scratch), T, HW, C, eps, stats);
  return cudaGetLastError();
}
cudaError_t launch_instnorm_relu_split(const float* y, const float* stats, int64_t rows, int HW, int C,
                                       __nv_bfloat16* out, cudaStream_t s) {
  const int64_t total = rows * (C / 4);
  const int blocks = (int)((total + 255) / 256 > 132 * 32 ? 132 * 32 : (total + 255) / 256);
  instnorm_relu_split_kernel<<<blocks, 256, 0, s>>>(y, stats, rows, HW, C, out);
  return cudaGetLastError();
}
cudaError_t launch_l2norm_rows(const float* in, int64_t rows, float* out, cudaStream_t s) {
  l2norm_rows_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(in, rows, out);
  return cudaGetLastError();
}

}  // namespace ct3
