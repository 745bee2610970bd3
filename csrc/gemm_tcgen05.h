// Host API of the wgmma GEMM family (see gemm_tcgen05.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pb {

enum Epilogue : int {
  EPI_BF16 = 0,       // D = bf16(acc*alpha + bias)
  EPI_RESIDUAL = 1,   // D = bf16(acc*alpha + bias + aux)
  EPI_GELU_DUAL = 2,  // D2 = bf16(z = acc*alpha + bias);  D = bf16(gelu(z))
  EPI_DGELU = 3,      // D = bf16((acc*alpha + bias) * gelu'(aux))
  EPI_F32 = 4,        // D (fp32) = acc*alpha   or  D += acc*alpha   (accumulate, red.global.add)
  // every other epilogue stores by TMA: D, D2 and D8 need 16-byte aligned base addresses and row strides
  EPI_GELU_GRAD = 5,  // z = acc*alpha + bias;  D = bf16(gelu(z));  D2 = bf16(gelu'(z))  — the backward then needs no erf/exp
  EPI_MUL = 6,        // D = bf16((acc*alpha + bias) * aux)
  EPI_GELU_GRAD_Q8 = 7,  // fp8 operands only: z = acc*alpha + bias;  D8 = e4m3(gelu(z) * *out_scale) (+ amax);  D2 = bf16(gelu'(z))
  EPI_SILU_GRAD = 8,  // z = acc*alpha + bias;  D = bf16(silu(z));  D2 = bf16(silu'(z))  — EPI_GELU_GRAD with SiLU
  // v = acc*alpha + bias;  D = bf16(v * aux);  D2 = bf16(v * aux2) — the gated FFN: forward up projection (aux = act(g),
  // aux2 = act'(g): D = act(g)*u, D2 = u*act'(g)) and its dgrad (aux = act(g), aux2 = u*act'(g): D = du, D2 = dg). aux and aux2
  // are read through the read-only data path, so D / D2 must not overlap them (no in-place update).
  EPI_MUL2 = 9,
};

struct GemmArgs {
  const void* A = nullptr;  // bf16: K-major [M,K] (lda = row stride) or MN-major [K,M]
  const void* B = nullptr;  // bf16: K-major [N,K] or MN-major [K,N]
  void* D = nullptr;        // [M,N] bf16 (fp32 for EPI_F32), ldd = row stride in elements
  void* D2 = nullptr;       // second output (EPI_GELU_DUAL / EPI_GELU_GRAD), bf16 [M,N]
  const float* bias = nullptr;
  const void* aux = nullptr;  // bf16 [M,N]
  const void* aux2 = nullptr; // bf16 [M,N], second multiplier (EPI_MUL2)
  int M = 0, N = 0, K = 0;
  long long lda = 0, ldb = 0, ldd = 0, ldd2 = 0, ld_aux = 0, ld_aux2 = 0;
  int a_mn = 0, b_mn = 0;
  int epi = EPI_BF16;
  int accumulate = 0;
  float alpha = 1.0f;
  int num_sms = 0;
  int cluster = 0;   // 0 = auto (2-CTA clusters with B multicast when >= 2 M tiles), 1 or 2 to force
  // ---- fp8 operands (wgmma e4m3 / e5m2, K-major only): A and B hold 1-byte elements, lda / ldb count elements (= bytes)
  int fp8 = 0;
  int a_fmt = 0, b_fmt = 0;           // 0 = E4M3, 1 = E5M2
  const float* sinv_a = nullptr;      // device scalars: 1 / quantisation scale of A and of B (multiplied into alpha)
  const float* sinv_b = nullptr;
  void* D8 = nullptr;                 // EPI_GELU_GRAD_Q8: E4M3 output [M,N], ldd8 = row stride in bytes
  long long ldd8 = 0;
  const float* out_scale = nullptr;   // device scalar: quantisation scale applied to the E4M3 output
  float* out_amax = nullptr;          // device scalar: running max |output| before scaling (bit pattern of a non-negative float)
};

void gemm_launch(const GemmArgs& g, cudaStream_t stream);
// [R, C] bytes (row stride ld) -> [C, R] contiguous: an MN-major fp8 operand made K-major
void transpose_u8(const void* src, long long ld, void* dst, int R, int C, cudaStream_t stream);

// ---- block-scaled MXFP8 (gemm_mxfp8.cu): E4M3 elements + one E8M0 scale per 32 K-elements of every row, scales applied per 32-K group to the wgmma partial sums
// x [R,K] bf16 -> q8 [R,K] E4M3, sf [K/128][rblk][512] scale atoms (rblk >= ceil(R/128); rows beyond R must be pre-zeroed)
void mx_quantize(const void* x_bf16, long long ld, void* q8, void* sf, long long R, int K, int rblk, cudaStream_t st);
// D[M,N] bf16 = (A.*SFA)[M,K] (B.*SFB)[N,K]^T (+ bias); sfa [K/128][ceil(M/128)][512], sfb [K/128][2*ceil(N/256)][512]
void gemm_mxfp8_launch(const void* A, const void* B, void* D, const void* sfa, const void* sfb, const float* bias, int M, int N, int K,
                       long long ldd, int num_sms, cudaStream_t stream);

CUtensorMap make_tmap_2d(const void* ptr, int elem_bytes, bool is_float32, uint64_t inner, uint64_t outer,
                         uint64_t ld_bytes, uint32_t box_inner, uint32_t box_outer, bool swizzle_128b = true);

}  // namespace pb
