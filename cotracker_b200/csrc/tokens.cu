// tokens.cu -- the row-wise / elementwise pieces of one update iteration that are not GEMMs:
//   LayerNorm (blocks.py:411,416; cotracker.py:539-540,549), positional encoding of relative motion
//   (posenc, cotracker3_online.py:19-39; cotracker3_offline.py:164-188), virtual-token init
//   (cotracker.py:486-488), delta heads + state update (cotracker.py:526-529; cotracker3_offline.py:204-211),
//   the time-embedding fold W_in * time_emb[t] and fp32 -> split-bf16 conversion.
// Token rows are track-major: row = n*T + t for point tokens, (N+i)*T + t for virtual token i.
#include "kernels.cuh"

namespace ct3 {
namespace {

// one warp per row of 384; output split [rows, 768]
__global__ void __launch_bounds__(256)
layernorm_split_kernel(const float* __restrict__ x, int rows, const float* __restrict__ gamma,
                       const float* __restrict__ beta, float eps, __nv_bfloat16* __restrict__ out) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float4* xr = reinterpret_cast<const float4*>(x + (int64_t)row * kC);
  float4 v[3];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    v[i] = xr[lane + 32 * i];
    s += v[i].x + v[i].y + v[i].z + v[i].w;
  }
  const float mean = warp_sum(s) * (1.0f / kC);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
    ss += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w;
  }
  const float rstd = rsqrtf(warp_sum(ss) * (1.0f / kC) + eps);
  __nv_bfloat16* o = out + (int64_t)row * (2 * kC);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int c = (lane + 32 * i) * 4;
    float y0 = v[i].x * rstd, y1 = v[i].y * rstd, y2 = v[i].z * rstd, y3 = v[i].w * rstd;
    if (gamma) {
      const float4 gm = *reinterpret_cast<const float4*>(gamma + c);
      const float4 bt = *reinterpret_cast<const float4*>(beta + c);
      y0 = y0 * gm.x + bt.x; y1 = y1 * gm.y + bt.y; y2 = y2 * gm.z + bt.z; y3 = y3 * gm.w + bt.w;
    }
    uint32_t h0, l0, h1, l1;
    split2(y0, y1, h0, l0);
    split2(y2, y3, h1, l1);
    *reinterpret_cast<uint2*>(o + c) = make_uint2(h0, h1);
    *reinterpret_cast<uint2*>(o + kC + c) = make_uint2(l0, l1);
  }
}

// block = one (n,t) row, 128 threads = X columns 1024..1151: [vis, conf, posenc(84), zero pad(42)]
__global__ void __launch_bounds__(128)
build_x_small_kernel(const float* __restrict__ coords, const float* __restrict__ vis, const float* __restrict__ conf,
                     int T, int N, const int32_t* __restrict__ track_len, __nv_bfloat16* __restrict__ xs) {
  const int row = blockIdx.x;  // n*T + t
  const int n = row / T, t = row % T;
  const int Tn = track_len ? track_len[n] : T;   // the track's own length: its last real frame gets the zero pad
  const int c = threadIdx.x;
  float val = 0.f;
  if (c == 0) {
    val = vis[(int64_t)t * N + n];
  } else if (c == 1) {
    val = conf[(int64_t)t * N + n];
  } else if (c < 2 + 84) {
    const int e = c - 2;
    int comp, k;   // comp: 0 fwd.x 1 fwd.y 2 bwd.x 3 bwd.y ; k: -1 raw, else frequency index
    bool shift = false;
    if (e < 4) { comp = e; k = -1; }
    else if (e < 44) { comp = (e - 4) & 3; k = (e - 4) >> 2; }
    else { comp = (e - 44) & 3; k = (e - 44) >> 2; shift = true; }
    const int axis = comp & 1;
    const bool fwd = comp < 2;
    float u = 0.f;
    const float here = coords[((int64_t)t * N + n) * 2 + axis];
    if (fwd) {
      if (t + 1 < Tn) u = here - coords[((int64_t)(t + 1) * N + n) * 2 + axis];
    } else {
      if (t > 0) u = here - coords[((int64_t)(t - 1) * N + n) * 2 + axis];
    }
    u = u / (axis == 0 ? 128.0f : 96.0f);  // model_resolution / stride, fixed (cotracker3_offline.py:173-181)
    if (k < 0) {
      val = u;
    } else {
      float xb = u * (float)(1 << k);
      if (shift) xb = xb + 1.57079632679489662f;
      val = sinf(xb);
    }
  }
  const bf16pair p = split_bf16(val);
  __nv_bfloat16* o = xs + (int64_t)row * (2 * kXPad) + 1024 + c;
  o[0] = p.hi;
  o[kXPad] = p.lo;
}

__global__ void init_virtual_kernel(float* __restrict__ tokens, const float* __restrict__ virt, int T, int N, int G) {
  // tokens[(N + kV*g + i)*T + t][:] = virt[i][:]
  const int64_t total = (int64_t)kV * G * T * (kC / 4);
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(idx % (kC / 4));
    const int64_t r = idx / (kC / 4);  // (kV*g + i)*T + t
    const int i = (int)((r / T) % kV);
    reinterpret_cast<float4*>(tokens + ((int64_t)N * T + r) * kC)[c4] =
        reinterpret_cast<const float4*>(virt + (int64_t)i * kC)[c4];
  }
}

// one warp per point-token row: 4 dot products of length 384
__global__ void __launch_bounds__(256)
heads_kernel(const float* __restrict__ tokens, const float* __restrict__ w4, const float* __restrict__ b4,
             float* __restrict__ coords, float* __restrict__ vis, float* __restrict__ conf,
             float* __restrict__ delta_out, int T, int N) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= N * T) return;
  const float4* xr = reinterpret_cast<const float4*>(tokens + (int64_t)row * kC);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float4 x = xr[lane + 32 * i];
#pragma unroll
    for (int o = 0; o < 4; ++o) {
      const float4 w = reinterpret_cast<const float4*>(w4 + o * kC)[lane + 32 * i];
      acc[o] += x.x * w.x + x.y * w.y + x.z * w.z + x.w * w.w;
    }
  }
#pragma unroll
  for (int o = 0; o < 4; ++o) acc[o] = warp_sum(acc[o]) + b4[o];
  if (lane == 0) {
    const int n = row / T, t = row % T;
    if (delta_out) {
      *reinterpret_cast<float4*>(delta_out + (int64_t)row * 4) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    } else {
      const int64_t s = (int64_t)t * N + n;
      coords[2 * s + 0] += acc[0];
      coords[2 * s + 1] += acc[1];
      vis[s] += acc[2];
      conf[s] += acc[3];
    }
  }
}

// out[t][c] = sum_k time_emb[t][k] * w_in[c][k]   (reference column order on both sides); one warp per output
__global__ void __launch_bounds__(256)
row_bias_kernel(const float* __restrict__ te, const float* __restrict__ w, int T, float* __restrict__ out) {
  const int o = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (o >= T * kC) return;
  const int t = o / kC, c = o % kC;
  float acc = 0.f;
  for (int k = lane; k < kX; k += 32) acc = fmaf(te[(int64_t)t * kX + k], w[(int64_t)c * kX + k], acc);
  acc = warp_sum(acc);
  if (lane == 0) out[o] = acc;
}

__global__ void split_rows_kernel(const float* __restrict__ x, int rows, int K, int Kpad, int perm_x, int fp16,
                                  __nv_bfloat16* __restrict__ out, int64_t dst_row_off) {
  const int64_t total = (int64_t)rows * Kpad;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % Kpad);
    const int64_t r = idx / Kpad;
    // perm_x: 1 = X column permutation, 2 = correlation-volume transpose (dst k*49 + i <- src i*49 + k)
    const int sc = perm_x == 1 ? x_src_col(c) : (perm_x == 2 ? (c < kVol ? (c % kP) * kP + c / kP : -1) : (c < K ? c : -1));
    const float v = sc >= 0 ? x[r * K + sc] : 0.f;
    __nv_bfloat16* o = out + (dst_row_off + r) * (2 * (int64_t)Kpad) + c;
    if (fp16) {
      const __half hi = __float2half_rn(v), lo = __float2half_rn(v - __half2float(hi));
      reinterpret_cast<__half*>(o)[0] = hi;
      reinterpret_cast<__half*>(o)[Kpad] = lo;
    } else {
      const bf16pair p = split_bf16(v);
      o[0] = p.hi;
      o[Kpad] = p.lo;
    }
  }
}

// a chunk of a host int32 table passed by value (kernel arguments stay below 4 KiB)
constexpr int kI32Chunk = 960;
struct I32Chunk { int32_t v[kI32Chunk]; };
__global__ void upload_i32_kernel(int32_t* __restrict__ dst, const I32Chunk c, int n) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = c.v[i];
}

inline int grid_for(int64_t total, int block) {
  int64_t b = (total + block - 1) / block;
  const int64_t cap = 132 * 32;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

cudaError_t launch_layernorm_split(const float* x, int rows, const float* gamma, const float* beta, float eps,
                                   __nv_bfloat16* out_split, cudaStream_t s) {
  if (rows <= 0) return cudaSuccess;
  layernorm_split_kernel<<<(rows + 7) / 8, 256, 0, s>>>(x, rows, gamma, beta, eps, out_split);
  return cudaGetLastError();
}
cudaError_t launch_build_x_small(const float* coords, const float* vis, const float* conf, int T, int N, int n0,
                                 int count, const int32_t* track_len, __nv_bfloat16* x_split, cudaStream_t s) {
  // the kernel's track n is track n0 + n of the [T, N] state: same pitch, base moved to track n0
  build_x_small_kernel<<<count * T, 128, 0, s>>>(coords + (int64_t)n0 * 2, vis + n0, conf + n0, T, N,
                                                 track_len ? track_len + n0 : nullptr, x_split);
  return cudaGetLastError();
}
cudaError_t launch_init_virtual(float* tokens, const float* virt, int T, int N, int G, cudaStream_t s) {
  init_virtual_kernel<<<grid_for((int64_t)kV * G * T * (kC / 4), 256), 256, 0, s>>>(tokens, virt, T, N, G);
  return cudaGetLastError();
}
cudaError_t launch_upload_i32(int32_t* dst, const int32_t* src_host, int n, cudaStream_t s) {
  for (int i0 = 0; i0 < n; i0 += kI32Chunk) {
    I32Chunk c;
    const int m = n - i0 < kI32Chunk ? n - i0 : kI32Chunk;
    for (int i = 0; i < m; ++i) c.v[i] = src_host[i0 + i];
    upload_i32_kernel<<<1, 256, 0, s>>>(dst + i0, c, m);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}
cudaError_t launch_heads(const float* tokens, const float* w4, const float* b4, float* coords, float* vis,
                         float* conf, float* delta_out, int T, int N, cudaStream_t s) {
  heads_kernel<<<(N * T + 7) / 8, 256, 0, s>>>(tokens, w4, b4, coords, vis, conf, delta_out, T, N);
  return cudaGetLastError();
}
cudaError_t launch_row_bias(const float* time_emb, const float* w_in, int T, float* out, cudaStream_t s) {
  row_bias_kernel<<<(T * kC + 7) / 8, 256, 0, s>>>(time_emb, w_in, T, out);
  return cudaGetLastError();
}
cudaError_t launch_split_rows(const float* x, int rows, int K, int Kpad, int perm_x, __nv_bfloat16* out,
                              int64_t dst_row_off, cudaStream_t s, int fp16) {
  if (rows <= 0) return cudaSuccess;
  split_rows_kernel<<<grid_for((int64_t)rows * Kpad, 256), 256, 0, s>>>(x, rows, K, Kpad, perm_x, fp16, out, dst_row_off);
  return cudaGetLastError();
}

}  // namespace ct3
