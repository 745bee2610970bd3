// Host API of the wgmma flash-attention kernels (see attention_tcgen05.cu).
#pragma once
#include <cuda_runtime.h>

namespace pb {

// qkv: bf16 [B, S, (H + 2*Hkv)*dh] (fused projection output: H q heads, Hkv k heads, Hkv v heads; query head h uses kv head
// h / (H / Hkv), Hkv = H is multi-head attention); out: bf16 [B, S, H*dh]; lse: fp32 [B, H, S]
// alibi_slopes: optional fp32 [H] (score += slope_h * (key - query)), nullptr = off
// doc_start: optional int32 [B*S] (doc_bounds_launch), causal only: query q sees key k iff doc_start[q] <= k <= q; nullptr = off
// window: sliding window, causal only: query q sees key k iff q - window <= k <= q (window + 1 keys, intersected with the
// document mask); -1 = off
void attention_fwd_launch(const void* qkv, void* out, float* lse, int B, int S, int H, int Hkv, int dh, float scale, bool causal,
                          cudaStream_t st, const float* alibi_slopes = nullptr, const int* doc_start = nullptr, int window = -1);
// dqkv: bf16 shaped like qkv (dK / dV of a kv head summed over its query heads); delta: fp32 scratch [B,H,S]; dq_acc: fp32 scratch [B*S, H*dh],
// owned by the caller (zeroed here on st, then read by the last kernel on st). doc_start / doc_end: both or neither. lse, delta
// and doc_start must be 16-byte aligned. window: as in the forward
void attention_bwd_launch(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv, float* delta, float* dq_acc,
                          int B, int S, int H, int Hkv, int dh, float scale, bool causal, int num_sms, cudaStream_t st,
                          const float* alibi_slopes = nullptr, const int* doc_start = nullptr, const int* doc_end = nullptr,
                          int window = -1);
// sequence_id int64 [B, S] -> doc_start / doc_end int32 [B*S]: first / last row (within the sequence) of each row's document,
// documents being maximal runs of equal ids
void doc_bounds_launch(const long long* sequence_id, int* doc_start, int* doc_end, int B, int S, cudaStream_t st);
// in-place rotary embedding on the q and k heads of qkv [T, (H + 2*Hkv)*dh] (rotate-half); inverse = transposed rotation
void rope_launch(void* qkv, const float* cosT, const float* sinT, long long T, int S, int H, int Hkv, int dh, bool inverse,
                 cudaStream_t st);

}  // namespace pb
