// Kernels of the KV-cached greedy decoder (sm_90a): one query row per sequence and step.
//
// KV cache layout (one layer): k and v are each bf16 [B_max, Hkv, S_max, dh], row-major, so the keys of one (sequence, kv head)
// are S_max contiguous rows of dh elements. Hkv is the kv head count: H for multi-head attention, fewer with grouped-query
// attention, where query head h reads kv head h / (H / Hkv). The fused qkv rows are [(H + 2*Hkv)*dh]: q heads, k heads, v heads.
// The decoder keeps all layers in one tensor [L, 2, B_max, Hkv, S_max, dh]
// (index 0 = k, 1 = v). Position p of sequence b holds the key / value of token p; positions >= the sequence length are
// never read.
//
// Per-sequence state lives in device memory so that one launch serves a ragged batch and a captured CUDA graph stays valid
// as the sequences grow: pos[b] (int32) is the position of the token being processed this step, i.e. the number of cached
// positions before it is appended; attention covers keys 0..pos[b].
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pb {

enum SkinnyEpi : int {
  SKINNY_PLAIN = 0,      // Y = X W^T (+ bias)
  SKINNY_RESIDUAL = 1,   // Y = X W^T (+ bias) + R
  SKINNY_GELU = 2,       // Y = gelu_exact(X W^T (+ bias))  (the formula of the training epilogue)
  SKINNY_SILU = 3,       // Y = silu(X W^T (+ bias))  (the formula of the training epilogue)
  SKINNY_MUL = 4,        // Y = (X W^T (+ bias)) * R  (R: the multiplier, passed where the residual goes)
};

struct SkinnyArgs {
  const void* X = nullptr;   // [M, K] bf16, row stride ldx
  const void* W = nullptr;   // [N, K] bf16, row stride ldw
  void* Y = nullptr;         // [M, N] bf16, row stride ldy
  const float* bias = nullptr;
  const void* R = nullptr;   // residual (SKINNY_RESIDUAL) or multiplier (SKINNY_MUL) [M, N] bf16, row stride ldr
  long long ldx = 0, ldw = 0, ldy = 0, ldr = 0;
  int M = 0, N = 0, K = 0;
  int epi = SKINNY_PLAIN;
  int num_sms = 132;
};

// Number of K splits the launch uses for this shape (1 = no fp32 partials needed).
int skinny_gemm_splits(int M, int N, int K, int num_sms);
// Y[M,N] = epilogue(X[M,K] W[N,K]^T) for 1 <= M <= 64. `partials` is fp32 scratch of splits * M * N elements (unused when
// skinny_gemm_splits() == 1); the split partials are summed in split order, so the result is bitwise reproducible.
void skinny_gemm_launch(const SkinnyArgs& a, float* partials, cudaStream_t st);

// Number of KV chunks (one CTA each per sequence and kv head) for a cache of s_max positions.
int decode_attention_splits(int s_max);
// out[b, h*dh:(h+1)*dh] = softmax(q k^T * scale + alibi) v over keys 0..pos[b] of the cache (window >= 0: keys
// max(0, pos[b] - window)..pos[b], the sliding window; -1 = off).
// q: row b at q + b*ldq (head h at +h*dh); partial_o: fp32 [B, H, splits, dh]; partial_ml: fp32 [B, H, splits, 2].
void decode_attention_launch(const void* q, long long ldq, const void* kc, const void* vc, const int* pos, void* out, long long ldo,
                             float* partial_o, float* partial_ml, int B, int H, int Hkv, int dh, int s_max, float scale,
                             const float* alibi_slopes, cudaStream_t st, int window = -1);

// For each row b of the fused qkv [B, (H + 2*Hkv)*dh]: rotate q and k (rotate-half tables cos / sin [>= s_max, dh/2], nullptr = no RoPE)
// at position pos[b] (q in place), and write k, v into the cache at position pos[b] of slot slot[b] (slot == nullptr: slot b).
void decode_append_launch(void* qkv, long long ldqkv, const int* pos, void* kc, void* vc, const float* cosT, const float* sinT, int B,
                          int H, int Hkv, int dh, int s_max, const int* slot, cudaStream_t st);

// Several query rows per cache slot (log-likelihood scoring). tiles: int32 [n_tiles, 4] on the device, each
// (slot, first_row, n_rows <= 64, first_pos): query rows first_row .. first_row + n_rows - 1 of qkv [n_q, (H + 2*Hkv)*dh] (q, after
// RoPE) sit at positions first_pos + i of that slot, and row i attends to keys 0 .. first_pos + i of the slot:
//   out[first_row + i, h*dh:(h+1)*dh] = softmax(q k^T * scale + alibi) v.
// window >= 0 (sliding window) starts row i's keys at max(0, first_pos + i - window); -1 = off.
// Rows outside every tile are not written. The keys of all tile rows must already be in the cache (decode_append first).
// qkv and out rows must be 16-byte aligned (TMA); d_head 64 or 128.
void cache_attention_launch(const void* qkv, long long ldq, long long n_q, const void* kc, const void* vc, const int* tiles, int n_tiles,
                            void* out, long long ldo, int B_max, int H, int Hkv, int dh, int s_max, float scale,
                            const float* alibi_slopes, cudaStream_t st, int window = -1);

// h[b,:] = wte[ids[b],:] + wpe[pos[b],:] (wpe may be nullptr)
void embed_pos_launch(const int* ids, const int* pos, const void* wte, const void* wpe, void* out, int B, int d, int V, cudaStream_t st);

// ids[b] = argmax_v logits[b, v] (lowest index on ties); pos[b] += 1 when pos != nullptr
void argmax_advance_launch(const void* logits, long long ldl, int B, int V, int* ids, int* pos, cudaStream_t st);

}  // namespace pb
