// enc_front.cu -- the CNN encoder (BasicEncoder, reference blocks.py:141-219) on the split-bf16x3 tensor-core engine,
// channels-last throughout (SURVEY.md 8(f) rank 1):
//
//   conv1 7x7/2 (3->64)            : direct fp32 SIMT kernel (K = 147 is too thin for the tensor cores; 0.9 GFLOP/frame)
//   every 3x3 stride-1 convolution : conv3x3_tc_kernel -- IMPLICIT GEMM on wgmma: the A tile of filter tap (ky,kx) is a
//                                    4-D TMA box of the NHWC activation shifted by (kx-1, ky-1); out-of-bounds texels
//                                    arrive as zeros, which IS the convolution's zero padding.  No im2col buffer exists
//                                    (the explicit one of the previous encoder tail was 2.9 GB per 16 frames).
//   3x3/2 and 1x1/2 convolutions   : a gather into the GEMM operand layout + the linear-layer GEMM (gemm.cu); they are
//                                    1/4-resolution and 7 % of the FLOPs
//   InstanceNorm / ReLU / residual : row-wise kernels on the NHWC fp32 conv output that emit the split-bf16 operand of
//                                    the next convolution (InstanceNorm needs whole-image statistics, so it cannot
//                                    live in the producing epilogue)
//   resize + concat                : bilinear (align_corners) resize of the 4 stage outputs written directly as the
//                                    split-bf16 NHWC operand [T*H4*W4, 2*448] of conv2 (416 channels, zero padded)
//
// Activations between convolutions: fp32 NHWC [T,H,W,C] (conv outputs, residual stream) and split bf16
// [T*H*W, 2*C] = [hi C | lo C] per pixel (conv inputs).  Stage 2 carries its 96 channels padded to 128 (zero
// weights / zero bias keep the padding exactly zero through InstanceNorm and ReLU).
#include "gemm.cuh"
#include "kernels.cuh"

namespace ct3 {
namespace {

// ------------------------------------------------------------------------------------------------
// conv1: 7x7 stride 2 pad 3, 3 -> 64 channels, fp32.  Block = 8 x 32 output pixels, thread = 1 pixel x 64 channels
// (accumulators in registers), input patch + weights in shared memory.
constexpr int ST_TW = 32, ST_TH = 8, ST_C = 64;
constexpr int ST_PW = 2 * ST_TW + 5, ST_PH = 2 * ST_TH + 5;   // 69 x 21 input patch
__global__ void __launch_bounds__(256)
conv_stem_kernel(const float* __restrict__ in /*[T,3,H,W]*/, const float* __restrict__ w /*[64,3,7,7]*/,
                 const float* __restrict__ bias, int H, int W, int Ho, int Wo, float* __restrict__ out /*[T,Ho,Wo,64]*/) {
  __shared__ float patch[ST_PH][ST_PW + 1];          // one input channel at a time (static shared memory <= 48 KiB)
  __shared__ __align__(16) float ws[49][ST_C];      // [tap][cout] of that channel
  const int t = blockIdx.z, oy0 = blockIdx.y * ST_TH, ox0 = blockIdx.x * ST_TW;
  const int iy0 = 2 * oy0 - 3, ix0 = 2 * ox0 - 3;
  const int py = threadIdx.x >> 5, px = threadIdx.x & 31;
  float acc[ST_C];
#pragma unroll
  for (int i = 0; i < ST_C; ++i) acc[i] = 0.f;
#pragma unroll 1
  for (int c = 0; c < 3; ++c) {
    __syncthreads();
    for (int i = threadIdx.x; i < 49 * ST_C; i += 256) {
      const int co = i / 49, tap = i % 49;             // global layout [co][ci][ky][kx]
      ws[tap][co] = w[(co * 3 + c) * 49 + tap];
    }
    for (int i = threadIdx.x; i < ST_PH * ST_PW; i += 256) {
      const int r = i / ST_PW, x = i % ST_PW;
      const int iy = iy0 + r, ix = ix0 + x;
      float v = 0.f;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = in[(((int64_t)t * 3 + c) * H + iy) * W + ix];
      patch[r][x] = v;
    }
    __syncthreads();
#pragma unroll 1
    for (int ky = 0; ky < 7; ++ky)
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        const float v = patch[2 * py + ky][2 * px + kx];
        const float4* wr = reinterpret_cast<const float4*>(ws[ky * 7 + kx]);
#pragma unroll
        for (int j = 0; j < ST_C / 4; ++j) {
          const float4 w4 = wr[j];
          acc[4 * j + 0] = fmaf(v, w4.x, acc[4 * j + 0]);
          acc[4 * j + 1] = fmaf(v, w4.y, acc[4 * j + 1]);
          acc[4 * j + 2] = fmaf(v, w4.z, acc[4 * j + 2]);
          acc[4 * j + 3] = fmaf(v, w4.w, acc[4 * j + 3]);
        }
      }
  }
  const int oy = oy0 + py, ox = ox0 + px;
  if (oy < Ho && ox < Wo) {
    float4* o = reinterpret_cast<float4*>(out + (((int64_t)t * Ho + oy) * Wo + ox) * ST_C);
#pragma unroll
    for (int j = 0; j < ST_C / 4; ++j) {
      const float4 b = __ldg(reinterpret_cast<const float4*>(bias) + j);
      o[j] = make_float4(acc[4 * j] + b.x, acc[4 * j + 1] + b.y, acc[4 * j + 2] + b.z, acc[4 * j + 3] + b.w);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// 3x3 stride-1 pad-1 convolution as an implicit GEMM:  Y[(t,y,x), co] = sum_{ky,kx,c} X[t, y+ky-1, x+kx-1, c] W[co, ky, kx, c]
//   A tile (128 pixels = th rows x tw columns of one frame, 64 channels of one tap) = ONE 4-D TMA box per bf16 plane
//   B tile (BN output channels x 64 channels of one tap) from the packed weights [Cout, 2 * 9*C]  (K index = tap*C + c)
//   warps 0..3 MMA warpgroup (wgmma, 3 MMAs per k16: split x split), warp 4 TMA producer, warps 5..8 epilogue (bias,
//   fp32 NHWC stores); the accumulator tile goes from the MMA registers to the epilogue through shared memory
constexpr int CBM = 128, CBK = 64;
constexpr int CTILE_A = CBM * CBK * 2;       // 16 KiB per plane
constexpr int CMMA_WARPS = 4, CTMA_WARP = 4, CEPI_WARP0 = 5;
constexpr int CEPI_WARPS = 4;
constexpr int CTHREADS = (CMMA_WARPS + 1 + CEPI_WARPS) * 32;
template <int BN> struct ConvCfg {
  static constexpr int TILE_B = BN * CBK * 2;
  static constexpr int STAGE = 2 * CTILE_A + 2 * TILE_B;          // 64 KiB (BN 128) / 48 KiB (BN 64)
  static constexpr int STAGES = BN == 128 ? 2 : 3;
  static constexpr int ACC_LD = BN + 4;
  static constexpr int OFF_ACC = STAGES * STAGE;
  static constexpr int OFF_BAR = OFF_ACC + CBM * ACC_LD * 4;
  static constexpr int SMEM = OFF_BAR + 256 + 1024;
  static_assert(SMEM <= 232448, "shared memory budget");
};
struct ConvGeom {
  int T, H, W, C, Cout;      // C, Cout multiples of 64; Cout % BN == 0
  int tw, th;                // tile = th rows x tw columns, tw * th == 128
  int tiles_x, tiles_y;
};

template <int BN>
__global__ void __launch_bounds__(CTHREADS, 1)
conv3x3_tc_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, ConvGeom g,
                  const float* __restrict__ bias, float* __restrict__ out) {
  using C = ConvCfg<BN>;
  constexpr int STAGES = C::STAGES;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* tfull_bar = empty_bar + STAGES;
  uint64_t* tempty_bar = tfull_bar + 1;
  float* acc_tile = reinterpret_cast<float*>(smem + C::OFF_ACC);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmW);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], CMMA_WARPS);
    }
    mbar_init(tfull_bar, CMMA_WARPS);
    mbar_init(tempty_bar, CEPI_WARPS);
    fence_barrier_init();
  }
  __syncthreads();

  const int num_nt = g.Cout / BN;
  const int tiles_per_frame = g.tiles_x * g.tiles_y;
  const int num_tiles = g.T * tiles_per_frame * num_nt;     // consecutive tiles: the N-tiles of one pixel tile
  const int cblocks = g.C / CBK;
  const int num_kb = 9 * cblocks;
  const int Kp = 9 * g.C;

  if (warp == CTMA_WARP) {
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int nt = tile % num_nt, pt = tile / num_nt;
        const int t = pt / tiles_per_frame, r = pt % tiles_per_frame;
        const int y0 = (r / g.tiles_x) * g.th, x0 = (r % g.tiles_x) * g.tw;
        for (int kb = 0; kb < num_kb; ++kb) {
          const int tap = kb / cblocks, cb = kb % cblocks;
          const int ky = tap / 3, kx = tap % 3;
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)C::STAGE);
          uint8_t* s = smem + stage * C::STAGE;
          tma_load_4d(s, &tmX, cb * CBK, x0 + kx - 1, y0 + ky - 1, t, &full_bar[stage]);
          tma_load_4d(s + CTILE_A, &tmX, g.C + cb * CBK, x0 + kx - 1, y0 + ky - 1, t, &full_bar[stage]);
          tma_load_2d(s + 2 * CTILE_A, &tmW, tap * g.C + cb * CBK, nt * BN, &full_bar[stage]);
          tma_load_2d(s + 2 * CTILE_A + C::TILE_B, &tmW, Kp + tap * g.C + cb * CBK, nt * BN, &full_bar[stage]);
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else if (warp < CMMA_WARPS) {
    int stage = 0;
    uint32_t phase = 0, acc_phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      float d0[BN / 2], d1[BN / 2];
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        wgmma_fence();
        mma_kblock<3, BN, false>(d0, d1, smem_u32(smem + stage * C::STAGE), CTILE_A, 2 * CTILE_A, C::TILE_B, kb == 0);
        wgmma_commit();
        wgmma_wait0(d0);
        wgmma_wait0(d1);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      mbar_wait(tempty_bar, acc_phase ^ 1u);
      acc_store<BN>(d0, acc_tile, C::ACC_LD);
      acc_store<BN>(d1, acc_tile + 64 * C::ACC_LD, C::ACC_LD);
      __syncwarp();
      if (lane == 0) mbar_arrive(tfull_bar);
      acc_phase ^= 1u;
    }
  } else {
    // epilogue: 4 warps = 4 row quarters; thread = one pixel, 16 channels per chunk
    const int r = (warp - CEPI_WARP0) * 32 + lane;     // tile row = pixel (dy, dx)
    const int dy = r / g.tw, dx = r % g.tw;
    const float* arow = acc_tile + r * C::ACC_LD;
    uint32_t acc_phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int nt = tile % num_nt, pt = tile / num_nt;
      const int t = pt / tiles_per_frame, rr = pt % tiles_per_frame;
      const int y = (rr / g.tiles_x) * g.th + dy, x = (rr % g.tiles_x) * g.tw + dx;
      const bool valid = y < g.H && x < g.W;
      float* orow = out + (((int64_t)t * g.H + y) * g.W + x) * g.Cout + nt * BN;
      mbar_wait(tfull_bar, acc_phase);
#pragma unroll
      for (int c = 0; c < BN / 16; ++c) {
        const int col = c * 16;
        float v[16];
        acc_row_ld<16>(arow + col, v);
        if (valid) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float4 b = __ldg(reinterpret_cast<const float4*>(bias + nt * BN + col) + j);
            reinterpret_cast<float4*>(orow + col)[j] =
                make_float4(v[4 * j] + b.x, v[4 * j + 1] + b.y, v[4 * j + 2] + b.z, v[4 * j + 3] + b.w);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(tempty_bar);
      acc_phase ^= 1u;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// conv weight [Cout, Cin, kh, kw] fp32 -> split [Cout_pad, 2*Kp], K index = (ky*kw + kx) * Cp + c  (tap-major,
// channels padded to Cp; rows >= Cout and channels >= Cin are zero)
__global__ void pack_conv_kernel(const float* __restrict__ w, int Cout, int Cin, int taps, int Cp, int Cout_pad,
                                 __nv_bfloat16* __restrict__ out) {
  const int Kp = taps * Cp;
  const int64_t total = (int64_t)Cout_pad * Kp;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % Kp), co = (int)(i / Kp);
    const int tap = k / Cp, c = k % Cp;
    float v = 0.f;
    if (co < Cout && c < Cin) v = w[((int64_t)co * Cin + c) * taps + tap];
    const bf16pair p = split_bf16(v);
    out[(int64_t)co * 2 * Kp + k] = p.hi;
    out[(int64_t)co * 2 * Kp + Kp + k] = p.lo;
  }
}

// stride-2 gather of a split NHWC activation [T,H,W,2*C] into GEMM operand rows [T*Ho*Wo, 2*taps*C]
// (taps = 9: 3x3 pad 1; taps = 1: 1x1), 8 channels (16 bytes) per thread, zero outside the image
__global__ void gather_s2_kernel(const uint4* __restrict__ in, int T, int H, int W, int C, int taps, int Ho, int Wo,
                                 uint4* __restrict__ out) {
  const int c8n = C / 8;
  const int64_t total = (int64_t)T * Ho * Wo * taps * c8n * 2;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i;
    const int c8 = (int)(r % c8n); r /= c8n;
    const int tap = (int)(r % taps); r /= taps;
    const int plane = (int)(r % 2); r /= 2;
    const int ox = (int)(r % Wo); r /= Wo;
    const int oy = (int)(r % Ho);
    const int t = (int)(r / Ho);
    const int iy = taps == 9 ? 2 * oy + tap / 3 - 1 : 2 * oy, ix = taps == 9 ? 2 * ox + tap % 3 - 1 : 2 * ox;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = in[(((int64_t)t * H + iy) * W + ix) * (2 * c8n) + plane * c8n + c8];
    out[(((int64_t)t * Ho + oy) * Wo + ox) * (2 * taps * c8n) + plane * taps * c8n + tap * c8n + c8] = v;
  }
}

// z = relu((y - mean) * rstd) [+ residual terms], 4 channels per thread; writes fp32 and/or split.
//   mode 0: z = relu(IN(y))                                   (after conv1 of a unit, after the stem)
//   mode 1: z = relu(x + relu(IN(y)))                         (end of a stride-1 unit; x fp32 NHWC)
//   mode 2: z = relu(IN_d(yd) + relu(IN(y)))                  (end of a stride-2 unit; yd = 1x1/2 conv output)
__global__ void norm_act_kernel(const float* __restrict__ y, const float* __restrict__ stats, const float* __restrict__ x,
                                const float* __restrict__ stats_d, int mode, int64_t rows, int HW, int C,
                                float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_split) {
  const int64_t total = rows * (C / 4);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % (C / 4));
    const int64_t r = i / (C / 4);
    const int t = (int)(r / HW);
    const float4 v = reinterpret_cast<const float4*>(y)[i];
    const float4* st = reinterpret_cast<const float4*>(stats + ((int64_t)t * C + c4 * 4) * 2);
    const float4 s0 = st[0], s1 = st[1];
    float a = fmaxf((v.x - s0.x) * s0.y, 0.f), b = fmaxf((v.y - s0.z) * s0.w, 0.f);
    float c = fmaxf((v.z - s1.x) * s1.y, 0.f), d = fmaxf((v.w - s1.z) * s1.w, 0.f);
    if (mode != 0) {
      float4 xv = reinterpret_cast<const float4*>(x)[i];
      if (mode == 2) {
        const float4* sd = reinterpret_cast<const float4*>(stats_d + ((int64_t)t * C + c4 * 4) * 2);
        const float4 d0 = sd[0], d1 = sd[1];
        xv = make_float4((xv.x - d0.x) * d0.y, (xv.y - d0.z) * d0.w, (xv.z - d1.x) * d1.y, (xv.w - d1.z) * d1.w);
      }
      a = fmaxf(xv.x + a, 0.f); b = fmaxf(xv.y + b, 0.f); c = fmaxf(xv.z + c, 0.f); d = fmaxf(xv.w + d, 0.f);
    }
    if (out_f32) reinterpret_cast<float4*>(out_f32)[i] = make_float4(a, b, c, d);
    if (out_split) {
      uint32_t h0, l0, h1, l1;
      split2(a, b, h0, l0);
      split2(c, d, h1, l1);
      __nv_bfloat16* o = out_split + r * (2 * (int64_t)C) + c4 * 4;
      *reinterpret_cast<uint2*>(o) = make_uint2(h0, h1);
      *reinterpret_cast<uint2*>(o + C) = make_uint2(l0, l1);
    }
  }
}

// bilinear (align_corners=True) resize of the four NHWC stage outputs to (H,W) + channel concat, written as the
// split operand of conv2: out[(t,y,x)][c] hi, [Cp + c] lo, c in [0, 416) real, [416, Cp) zero
// (BasicEncoder._bilinear_intepolate + torch.cat, blocks.py:202-215).  Thread = 4 channels of one output pixel.
struct UpArgsN {
  const float* src[4];
  int c[4], cs[4], h[4], w[4], coff[4];   // c: channels used, cs: channel stride of the source (padded)
};
__global__ void upsample_concat_split_kernel(UpArgsN a, int T, int Ctot, int Cp, int H, int W,
                                             __nv_bfloat16* __restrict__ out) {
  const int c4n = Cp / 4;
  const int64_t total = (int64_t)T * H * W * c4n;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % c4n);
    int64_t r = i / c4n;                     // pixel row (t, y, x)
    const int x = (int)(r % W);
    const int y = (int)((r / W) % H);
    const int t = (int)(r / ((int64_t)W * H));
    const int cc = c4 * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (cc < Ctot) {
      int s = 0;
#pragma unroll
      for (int k = 1; k < 4; ++k) s = (cc >= a.coff[k]) ? k : s;
      const int c = cc - a.coff[s], hs = a.h[s], ws = a.w[s], cs = a.cs[s];
      const float* p = a.src[s] + (int64_t)t * hs * ws * cs + c;
      if (hs == H && ws == W) {
        v = *reinterpret_cast<const float4*>(p + ((int64_t)y * ws + x) * cs);
      } else {
        const float sy = H > 1 ? (float)(hs - 1) / (float)(H - 1) : 0.f, sx = W > 1 ? (float)(ws - 1) / (float)(W - 1) : 0.f;
        const float fy = sy * (float)y, fx = sx * (float)x;
        const int y0 = (int)fy, x0 = (int)fx;
        const int y1 = min(y0 + 1, hs - 1), x1 = min(x0 + 1, ws - 1);
        const float ly = fy - (float)y0, lx = fx - (float)x0;
        const float4 v00 = *reinterpret_cast<const float4*>(p + ((int64_t)y0 * ws + x0) * cs);
        const float4 v01 = *reinterpret_cast<const float4*>(p + ((int64_t)y0 * ws + x1) * cs);
        const float4 v10 = *reinterpret_cast<const float4*>(p + ((int64_t)y1 * ws + x0) * cs);
        const float4 v11 = *reinterpret_cast<const float4*>(p + ((int64_t)y1 * ws + x1) * cs);
        v.x = (1.f - ly) * ((1.f - lx) * v00.x + lx * v01.x) + ly * ((1.f - lx) * v10.x + lx * v11.x);
        v.y = (1.f - ly) * ((1.f - lx) * v00.y + lx * v01.y) + ly * ((1.f - lx) * v10.y + lx * v11.y);
        v.z = (1.f - ly) * ((1.f - lx) * v00.z + lx * v01.z) + ly * ((1.f - lx) * v10.z + lx * v11.z);
        v.w = (1.f - ly) * ((1.f - lx) * v00.w + lx * v01.w) + ly * ((1.f - lx) * v10.w + lx * v11.w);
      }
    }
    uint32_t h0, l0, h1, l1;
    split2(v.x, v.y, h0, l0);
    split2(v.z, v.w, h1, l1);
    __nv_bfloat16* o = out + r * (2 * (int64_t)Cp) + cc;
    *reinterpret_cast<uint2*>(o) = make_uint2(h0, h1);
    *reinterpret_cast<uint2*>(o + Cp) = make_uint2(l0, l1);
  }
}

inline int grid_cap(int64_t total, int block, int per_sm) {
  int64_t b = (total + block - 1) / block;
  const int64_t cap = 132LL * per_sm;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

template <int BN>
cudaError_t launch_conv_variant(const CUtensorMap& tmX, const CUtensorMap& tmW, const ConvGeom& g, const float* bias,
                                float* out, int num_sms, cudaStream_t s) {
  using C = ConvCfg<BN>;
  static DeviceOnce attr;
  cudaError_t e = once_per_device(attr, [&] {
    return cudaFuncSetAttribute(conv3x3_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM);
  });
  if (e != cudaSuccess) return e;
  const int64_t tiles = (int64_t)g.T * g.tiles_x * g.tiles_y * (g.Cout / BN);
  const int grid = (int)(tiles < num_sms ? tiles : num_sms);
  conv3x3_tc_kernel<BN><<<grid, CTHREADS, C::SMEM, s>>>(tmX, tmW, g, bias, out);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_conv_stem(const float* frames, const float* w, const float* bias, int T, int H, int W, float* out,
                             cudaStream_t s) {
  const int Ho = (H + 2 * 3 - 7) / 2 + 1, Wo = (W + 2 * 3 - 7) / 2 + 1;
  dim3 grid((Wo + ST_TW - 1) / ST_TW, (Ho + ST_TH - 1) / ST_TH, T);
  conv_stem_kernel<<<grid, 256, 0, s>>>(frames, w, bias, H, W, Ho, Wo, out);
  return cudaGetLastError();
}

// tile shape (tw x th = 128) wasting the fewest MMA rows on a H x W image
static void pick_tile(int H, int W, int& tw, int& th) {
  int64_t best = -1;
  for (int w = 128; w >= 8; w >>= 1) {
    const int h = 128 / w;
    const int64_t cover = (int64_t)((W + w - 1) / w) * w * ((H + h - 1) / h) * h;
    if (best < 0 || cover < best) { best = cover; tw = w; th = h; }
  }
}

cudaError_t launch_conv3x3_tc(const __nv_bfloat16* x_split, const __nv_bfloat16* w_split, const float* bias, int T,
                              int H, int W, int C, int Cout, float* out, int num_sms, cudaStream_t s) {
  if (T < 1 || H < 1 || W < 1 || C < 64 || (C % 64) || Cout < 64 || (Cout % 64)) return cudaErrorInvalidValue;
  ConvGeom g;
  g.T = T; g.H = H; g.W = W; g.C = C; g.Cout = Cout;
  pick_tile(H, W, g.tw, g.th);
  g.tiles_x = (W + g.tw - 1) / g.tw;
  g.tiles_y = (H + g.th - 1) / g.th;
  const int BN = (Cout % 128 == 0) ? 128 : 64;
  CUtensorMap tmX, tmW;
  {
    const uint64_t dims[4] = {(uint64_t)(2 * C), (uint64_t)W, (uint64_t)H, (uint64_t)T};
    const uint64_t strides[3] = {(uint64_t)2 * C * 2, (uint64_t)W * 2 * C * 2, (uint64_t)H * W * 2 * C * 2};
    const uint32_t box[4] = {64, (uint32_t)g.tw, (uint32_t)g.th, 1};
    if (!encode_tensor_map(&tmX, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, x_split, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))
      return cudaErrorInvalidValue;
    const uint64_t wd[2] = {(uint64_t)(2 * 9 * C), (uint64_t)Cout};
    const uint64_t ws[1] = {(uint64_t)(2 * 9 * C) * 2};
    const uint32_t wb[2] = {64, (uint32_t)BN};
    if (!encode_tensor_map(&tmW, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, w_split, wd, ws, wb, CU_TENSOR_MAP_SWIZZLE_128B))
      return cudaErrorInvalidValue;
  }
  return BN == 128 ? launch_conv_variant<128>(tmX, tmW, g, bias, out, num_sms, s)
                   : launch_conv_variant<64>(tmX, tmW, g, bias, out, num_sms, s);
}

cudaError_t launch_pack_conv(const float* w, int Cout, int Cin, int taps, int Cp, int Cout_pad, __nv_bfloat16* out,
                             cudaStream_t s) {
  pack_conv_kernel<<<grid_cap((int64_t)Cout_pad * taps * Cp, 256, 8), 256, 0, s>>>(w, Cout, Cin, taps, Cp, Cout_pad, out);
  return cudaGetLastError();
}

cudaError_t launch_gather_s2(const __nv_bfloat16* x_split, int T, int H, int W, int C, int taps, __nv_bfloat16* out,
                             cudaStream_t s) {
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;   // 3x3 pad 1 stride 2 and 1x1 stride 2 agree
  const int64_t total = (int64_t)T * Ho * Wo * taps * (C / 8) * 2;
  gather_s2_kernel<<<grid_cap(total, 256, 16), 256, 0, s>>>(reinterpret_cast<const uint4*>(x_split), T, H, W, C, taps, Ho, Wo,
                                                           reinterpret_cast<uint4*>(out));
  return cudaGetLastError();
}

cudaError_t launch_norm_act(const float* y, const float* stats, const float* x, const float* stats_d, int mode,
                            int64_t rows, int HW, int C, float* out_f32, __nv_bfloat16* out_split, cudaStream_t s) {
  norm_act_kernel<<<grid_cap(rows * (C / 4), 256, 16), 256, 0, s>>>(y, stats, x, stats_d, mode, rows, HW, C, out_f32, out_split);
  return cudaGetLastError();
}

cudaError_t launch_upsample_concat_split(const float* const src[4], const int c[4], const int cs[4], const int h[4],
                                         const int w[4], int T, int Cp, int H, int W, __nv_bfloat16* out, cudaStream_t s) {
  UpArgsN a;
  int off = 0;
  for (int k = 0; k < 4; ++k) {
    a.src[k] = src[k]; a.c[k] = c[k]; a.cs[k] = cs[k]; a.h[k] = h[k]; a.w[k] = w[k]; a.coff[k] = off;
    off += c[k];
  }
  upsample_concat_split_kernel<<<grid_cap((int64_t)T * H * W * (Cp / 4), 256, 32), 256, 0, s>>>(a, T, off, Cp, H, W, out);
  return cudaGetLastError();
}

}  // namespace ct3
