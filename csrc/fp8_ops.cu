// FP8 (E4M3 / E5M2) producers for the fp8 wgmma GEMMs of `precision: amp_fp8` on sm_90a.
//
// The recipe is per-tensor scaling (photon_b200/train/fp8.py is the numerics oracle): activations and weights are cast to
// E4M3, gradients flowing backward to E5M2; every cast multiplies by the tensor role's scale and saturates; the GEMM epilogue
// multiplies by 1/(scale_a * scale_b). Nothing here makes an extra pass over an activation just to quantise it:
//
//   * ln_fwd_q8_kernel        LayerNorm (or, RMS instance, RMSNorm) forward whose ONLY output is the E4M3 tensor the next GEMM
//                             (and the wgrad) reads
//   * colsum_quant_kernel     bias-gradient column sums and the E5M2 copy of dY for dgrad / wgrad from the same read of dY
//   * (csrc/gemm_tcgen05.cu)  EPI_GELU_GRAD_Q8 writes gelu(z) as E4M3 from the up-projection's epilogue
//   * seg_amax / seg_quant    the four weight matrices of every block, E4M3 with CURRENT scaling, from the bf16 shadow
//   * update_scales_kernel    delayed scaling for activations / gradients: amax history ring -> next scale, all on device
//
// Scales, inverse scales and running amax values live in device arrays indexed by "role" so a whole training step stays
// CUDA-graph capturable (no host round trip to pick a scale). Replaces what the reference would reach through Composer's
// amp_fp8 -> TransformerEngine (ref: scripts/centralised_training.sh:91, commented out there).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <stdexcept>
#include <string>

#include "fp8_ops.h"
#include "fp8_round.cuh"
#include "launch.h"
#include "ptx.cuh"

namespace pb {

namespace {

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffff, v, o);
  return v;
}

// ------------------------------------------------------------------ LayerNorm / RMSNorm forward -> E4M3 (one warp per row)
// RMS: no mean (not written, may be null) and no beta, as in csrc/fused_ops.cu's ln_fwd_kernel.
template <int LN_NCH, bool RMS>
__global__ void __launch_bounds__(256) ln_fwd_q8_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma,
                                                         const float* __restrict__ beta, uint8_t* __restrict__ y8,
                                                         float* __restrict__ mean, float* __restrict__ rstd, long long T, int d,
                                                         float eps, const float* __restrict__ scale, float* __restrict__ amax) {
  __shared__ float smax[8];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long row = (long long)blockIdx.x * 8 + w;
  const float s = __ldg(scale);
  float am = 0.f;
  if (row < T) {
    const uint4* xr = reinterpret_cast<const uint4*>(x + row * d);
    uint4 buf[LN_NCH];
    float sum = 0.f;
#pragma unroll
    for (int c = 0; c < LN_NCH; ++c) {
      const int e = c * 256 + lane * 8;
      if (e < d) {
        buf[c] = xr[c * 32 + lane];
        float f[8];
        unpack8f(buf[c], f);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          if constexpr (RMS) sum += f[k] * f[k];
          else sum += f[k];
        }
      }
    }
    float mu = 0.f, var = warp_sum_f(sum) / d;   // var: mean(x^2) for RMS, otherwise mean(x) until the second pass
    if constexpr (!RMS) {
      mu = var;
      float ss = 0.f;
#pragma unroll
      for (int c = 0; c < LN_NCH; ++c) {
        const int e = c * 256 + lane * 8;
        if (e < d) {
          float f[8];
          unpack8f(buf[c], f);
#pragma unroll
          for (int k = 0; k < 8; ++k) ss += (f[k] - mu) * (f[k] - mu);
        }
      }
      var = warp_sum_f(ss) / d;
    }
    const float rs = rsqrtf(var + eps);
    if (lane == 0) {
      if constexpr (!RMS) mean[row] = mu;
      rstd[row] = rs;
    }
    uint2* yr = reinterpret_cast<uint2*>(y8 + row * d);
#pragma unroll
    for (int c = 0; c < LN_NCH; ++c) {
      const int e = c * 256 + lane * 8;
      if (e < d) {
        float f[8];
        unpack8f(buf[c], f);
        const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + e)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + e + 4));
        const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        if constexpr (RMS) {
#pragma unroll
          for (int k = 0; k < 8; ++k) f[k] = f[k] * rs * g[k];
        } else {
          float4 b0 = make_float4(0, 0, 0, 0), b1 = b0;
          if (beta) b0 = __ldg(reinterpret_cast<const float4*>(beta + e)), b1 = __ldg(reinterpret_cast<const float4*>(beta + e + 4));
          const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
          for (int k = 0; k < 8; ++k) f[k] = (f[k] - mu) * rs * g[k] + b[k];
        }
        am = amax8(f, am);
        yr[c * 32 + lane] = quant8<0>(f, s);
      }
    }
  }
  am = warp_max_f(am);
  if (lane == 0) smax[w] = am;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = smax[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) m = fmaxf(m, smax[i]);
    if (m > 0.f) atomic_max_pos_f32(amax, m);
  }
}

// ------------------------------------------------------------------ column sums (bias gradient) + fp8 copy in one read of dY
// Block = 8 warps x 256 columns; grid.y strips of rows. out_sum may be null (pure quantise), y8 may be null (pure column sum).
template <int FMT>
__global__ void __launch_bounds__(256) colsum_quant_kernel(const __nv_bfloat16* __restrict__ dy, long long ld, float* __restrict__ out_sum,
                                                            uint8_t* __restrict__ y8, long long ld8, const float* __restrict__ scale,
                                                            float* __restrict__ amax, long long T, int d, int rows_per_block) {
  __shared__ float ssum[8][256];
  __shared__ float smax[8];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int col = blockIdx.x * 256 + lane * 8;
  const long long r0 = (long long)blockIdx.y * rows_per_block;
  const long long r1 = r0 + rows_per_block < T ? r0 + rows_per_block : T;
  const float s = y8 ? __ldg(scale) : 1.0f;
  float as[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  float am = 0.f;
  if (col < d) {
    long long r = r0 + w;
    for (; r + 24 < r1; r += 32) {   // 4 independent 16-byte loads per thread in flight
      uint4 q[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) q[u] = *reinterpret_cast<const uint4*>(dy + (r + 8 * u) * ld + col);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float g[8];
        unpack8f(q[u], g);
#pragma unroll
        for (int k = 0; k < 8; ++k) as[k] += g[k];
        if (y8) {
          am = amax8(g, am);
          *reinterpret_cast<uint2*>(y8 + (r + 8 * u) * ld8 + col) = quant8<FMT>(g, s);
        }
      }
    }
    for (; r < r1; r += 8) {
      float g[8];
      unpack8f(*reinterpret_cast<const uint4*>(dy + r * ld + col), g);
#pragma unroll
      for (int k = 0; k < 8; ++k) as[k] += g[k];
      if (y8) {
        am = amax8(g, am);
        *reinterpret_cast<uint2*>(y8 + r * ld8 + col) = quant8<FMT>(g, s);
      }
    }
  }
  if (out_sum) {
#pragma unroll
    for (int k = 0; k < 8; ++k) ssum[w][lane * 8 + k] = as[k];
  }
  am = warp_max_f(am);
  if (lane == 0) smax[w] = am;
  __syncthreads();
  const int c = threadIdx.x;
  if (out_sum && blockIdx.x * 256 + c < d) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += ssum[i][c];
    atomicAdd(out_sum + blockIdx.x * 256 + c, t);
  }
  if (y8 && amax && threadIdx.x == 0) {
    float m = smax[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) m = fmaxf(m, smax[i]);
    if (m > 0.f) atomic_max_pos_f32(amax, m);
  }
}

// ------------------------------------------------------------------ weights: per-tensor CURRENT scaling from the bf16 shadow
// seg[i] = {offset, numel} (elements, multiples of 8) into the flat planes; role0 + i indexes scale / scale_inv / amax.
__global__ void __launch_bounds__(256) seg_amax_kernel(const __nv_bfloat16* __restrict__ src, const long long* __restrict__ seg,
                                                        float* __restrict__ amax) {
  __shared__ float smax[8];
  const long long off = seg[2 * blockIdx.y], n8 = seg[2 * blockIdx.y + 1] / 8;
  const uint4* p = reinterpret_cast<const uint4*>(src + off);
  float am = 0.f;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n8; i += gridDim.x * 256ll) {
    float f[8];
    unpack8f(p[i], f);
    am = amax8(f, am);
  }
  am = warp_max_f(am);
  if ((threadIdx.x & 31) == 0) smax[threadIdx.x >> 5] = am;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = smax[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) m = fmaxf(m, smax[i]);
    if (m > 0.f) atomic_max_pos_f32(amax + blockIdx.y, m);
  }
}
__global__ void __launch_bounds__(256) seg_quant_kernel(const __nv_bfloat16* __restrict__ src, uint8_t* __restrict__ dst,
                                                         const long long* __restrict__ seg, const float* __restrict__ amax,
                                                         float* __restrict__ scale, float* __restrict__ scale_inv, float fmax) {
  const long long off = seg[2 * blockIdx.y], n8 = seg[2 * blockIdx.y + 1] / 8;
  const float a = amax[blockIdx.y];
  const float s = weight_scale(a, fmax);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    scale[blockIdx.y] = s;
    scale_inv[blockIdx.y] = inv_scale(s);
  }
  const uint4* p = reinterpret_cast<const uint4*>(src + off);
  uint2* q = reinterpret_cast<uint2*>(dst + off);
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n8; i += gridDim.x * 256ll) {
    float f[8];
    unpack8f(p[i], f);
    q[i] = quant8<0>(f, s);
  }
}

// ------------------------------------------------------------------ delayed scaling: amax history -> next scale (one thread per role)
__global__ void update_scales_kernel(float* __restrict__ scale, float* __restrict__ scale_inv, float* __restrict__ amax,
                                     float* __restrict__ hist, const float* __restrict__ fmax, int* __restrict__ pos, int n, int H,
                                     float margin_mult) {
  const int slot = *pos % H;
  __syncthreads();
  for (int r = threadIdx.x; r < n; r += blockDim.x) {
    const float a = amax[r];
    amax[r] = 0.f;
    hist[(long long)r * H + slot] = a;
    float m = 0.f;
    for (int i = 0; i < H; ++i) m = fmaxf(m, hist[(long long)r * H + i]);
    if (m > 0.f && m < 3.0e38f) {   // no observation yet (or a non-finite one): keep the scale
      const float s = scale_of(fmax[r], m * margin_mult);
      scale[r] = s;
      scale_inv[r] = inv_scale(s);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) *pos = *pos + 1;
}

template <bool RMS>
void norm_fwd_q8(const void* x, const float* gamma, const float* beta, void* y8, float* mean, float* rstd, long long T, int d, float eps,
                 const float* scale, float* amax, cudaStream_t st) {
  const char* name = RMS ? "rmsnorm_fwd_q8" : "layernorm_fwd_q8";
  if (d % 8 || d > 16 * 256) throw std::runtime_error(std::string(name) + ": d must be a multiple of 8 and <= 4096");
  with_ln_chunks((d + 255) / 256, [&](auto N) {
    ln_fwd_q8_kernel<N, RMS><<<int((T + 7) / 8), 256, 0, st>>>((const __nv_bfloat16*)x, gamma, beta, (uint8_t*)y8, mean, rstd, T, d, eps,
                                                               scale, amax);
  });
  launched(name);
}

}  // namespace

void layernorm_fwd_q8(const void* x, const float* gamma, const float* beta, void* y8, float* mean, float* rstd, long long T, int d,
                      float eps, const float* scale, float* amax, cudaStream_t st) {
  norm_fwd_q8<false>(x, gamma, beta, y8, mean, rstd, T, d, eps, scale, amax, st);
}
void rmsnorm_fwd_q8(const void* x, const float* gamma, void* y8, float* rstd, long long T, int d, float eps, const float* scale, float* amax,
                    cudaStream_t st) {
  norm_fwd_q8<true>(x, gamma, nullptr, y8, nullptr, rstd, T, d, eps, scale, amax, st);
}

void colsum_quant(const void* dy, long long ld, float* out_sum, void* y8, long long ld8, int fmt, const float* scale, float* amax,
                  long long T, int d, cudaStream_t st) {
  if (d % 8) throw std::runtime_error("colsum_quant: the row length must be a multiple of 8");
  const int col_blocks = (d + 255) / 256;
  int strips = (132 * 4 + col_blocks - 1) / col_blocks;
  if (strips > T) strips = int(T);
  const int rows_per = int((T + strips - 1) / strips);
  dim3 grid(col_blocks, int((T + rows_per - 1) / rows_per));
  if (fmt == 0)
    colsum_quant_kernel<0><<<grid, 256, 0, st>>>((const __nv_bfloat16*)dy, ld, out_sum, (uint8_t*)y8, ld8, scale, amax, T, d, rows_per);
  else
    colsum_quant_kernel<1><<<grid, 256, 0, st>>>((const __nv_bfloat16*)dy, ld, out_sum, (uint8_t*)y8, ld8, scale, amax, T, d, rows_per);
  launched("colsum_quant");
}

void quantize_segments(const void* src_bf16, void* dst8, const long long* seg_dev, int n_seg, float* scale, float* scale_inv, float* amax,
                       cudaStream_t st) {
  if (n_seg <= 0) return;
  cudaError_t e = cudaMemsetAsync(amax, 0, sizeof(float) * n_seg, st);
  if (e != cudaSuccess) throw std::runtime_error(std::string("quantize_segments memset: ") + cudaGetErrorString(e));
  int bx = (132 * 8 + n_seg - 1) / n_seg;
  if (bx < 1) bx = 1;
  if (bx > 64) bx = 64;
  seg_amax_kernel<<<dim3(bx, n_seg), 256, 0, st>>>((const __nv_bfloat16*)src_bf16, seg_dev, amax);
  launched("seg_amax");
  seg_quant_kernel<<<dim3(bx, n_seg), 256, 0, st>>>((const __nv_bfloat16*)src_bf16, (uint8_t*)dst8, seg_dev, amax, scale, scale_inv, 448.0f);
  launched("seg_quant");
}

void update_scales(float* scale, float* scale_inv, float* amax, float* hist, const float* fmax, int* pos, int n, int H, float margin_mult,
                   cudaStream_t st) {
  if (n <= 0) return;
  update_scales_kernel<<<1, 256, 0, st>>>(scale, scale_inv, amax, hist, fmax, pos, n, H, margin_mult);
  launched("update_scales");
}

}  // namespace pb
