// Host API of the fp8 producers (see fp8_ops.cu): quantising LayerNorm, column-sum + quantise, weight quantisation with
// current scaling, delayed-scaling bookkeeping. Scales / amax values are device scalars.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pb {

// y8[T,d] = e4m3(layernorm(x) * *scale); *amax = max(*amax, max|layernorm(x)|); mean / rstd saved for the backward
void layernorm_fwd_q8(const void* x, const float* gamma, const float* beta, void* y8, float* mean, float* rstd, long long T, int d,
                      float eps, const float* scale, float* amax, cudaStream_t st);
// the same for RMSNorm (no beta, no mean): y8 = e4m3(x * rstd * gamma * *scale)
void rmsnorm_fwd_q8(const void* x, const float* gamma, void* y8, float* rstd, long long T, int d, float eps, const float* scale, float* amax,
                    cudaStream_t st);
// out_sum[j] += sum_t dy[t,j] (may be null);  y8[t,j] = fp8(dy[t,j] * *scale) (may be null), fmt 0 = E4M3, 1 = E5M2
void colsum_quant(const void* dy, long long ld, float* out_sum, void* y8, long long ld8, int fmt, const float* scale, float* amax,
                  long long T, int d, cudaStream_t st);
// n_seg tensors (seg_dev[2i] = element offset, seg_dev[2i+1] = numel) of a flat bf16 plane -> E4M3 at the same offsets of dst8,
// scale[i] = 448 / amax_i computed here (current scaling); scale / scale_inv / amax point at the first of the n_seg roles
void quantize_segments(const void* src_bf16, void* dst8, const long long* seg_dev, int n_seg, float* scale, float* scale_inv, float* amax,
                       cudaStream_t st);
// delayed scaling for n roles: push amax into the history ring (length H, position *pos), scale = fmax / (max(history) * margin_mult)
void update_scales(float* scale, float* scale_inv, float* amax, float* hist, const float* fmax, int* pos, int n, int H, float margin_mult,
                   cudaStream_t st);

}  // namespace pb
