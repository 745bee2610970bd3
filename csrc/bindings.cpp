// Python bindings (torch extension `photon_b200._C`) for the sm_90a kernels in this directory.
// Tensors are passed as torch::Tensor; every op runs on the current CUDA stream of the tensor's device.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda_runtime.h>
#include <pybind11/pybind11.h>
#include <torch/extension.h>

#include <atomic>
#include <cmath>
#include <cstdlib>
#include <limits>
#include <string>
#include <type_traits>
#include <vector>

#include "comm.h"
#include "fp8_ops.h"
#include "fused_ops.h"
#include "gemm_tcgen05.h"
#include "attention_tcgen05.h"
#include "decode.h"
#include "launch.h"

namespace py = pybind11;
using torch::Tensor;

namespace pb {
std::atomic<long long> g_launches{0};
}

namespace {

inline cudaStream_t stream_of(const Tensor& t) { return at::cuda::getCurrentCUDAStream(t.device().index()).stream(); }

inline void check_cuda(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
}
inline void check_bf16(const Tensor& t, const char* name) {
  check_cuda(t, name);
  TORCH_CHECK(t.scalar_type() == at::kBFloat16, name, " must be bfloat16");
}
inline void check_f32(const Tensor& t, const char* name) {
  check_cuda(t, name);
  TORCH_CHECK(t.scalar_type() == at::kFloat, name, " must be float32");
}
template <class T = void>
T* opt_ptr(const c10::optional<Tensor>& t) {
  if (!t.has_value()) return nullptr;
  if constexpr (std::is_void_v<T>) return t->data_ptr();
  else return t->data_ptr<T>();
}
inline int num_sms() { return at::cuda::getCurrentDeviceProperties()->multiProcessorCount; }
// The fused memory-bound kernels read and write rows as `bytes`-wide vectors (16: uint4 / float4, 8: four fp8 bytes as uint2):
// the base pointer and, for a 2-D operand, the row stride must be multiples of that width. Checked before any launch, since a
// misaligned vector access faults the device instead of raising.
inline void check_vec(const Tensor& t, const char* op, const char* name, int bytes = 16) {
  TORCH_CHECK((reinterpret_cast<uintptr_t>(t.data_ptr()) % bytes) == 0, op, ": ", name, " must start on a ", bytes, "-byte boundary");
  TORCH_CHECK(t.dim() < 2 || (t.stride(0) * t.element_size()) % bytes == 0, op, ": the row stride of ", name, " must be a multiple of ",
              bytes, " bytes");
}
inline void check_numel(const Tensor& t, int64_t n, const char* op, const char* name) {
  TORCH_CHECK(t.numel() == n, op, ": ", name, " must have ", n, " elements, not ", t.numel());
}

#define CUDA_OK(expr)                                                                        \
  do {                                                                                       \
    cudaError_t e__ = (expr);                                                                \
    TORCH_CHECK(e__ == cudaSuccess, #expr " failed: ", cudaGetErrorString(e__));             \
  } while (0)

// ---------------------------------------------------------------------------------- GEMM
// fp8 operands (1-byte tensors: torch.uint8 or float8 storage)
inline bool is_byte(const Tensor& t) {
  return t.scalar_type() == at::kByte || t.scalar_type() == at::kFloat8_e4m3fn || t.scalar_type() == at::kFloat8_e5m2;
}
// a: [M,K] (a_mn=0) or [K,M] (a_mn=1);  b: [N,K] (b_mn=0) or [K,N] (b_mn=1);  d: [M,N]. The checks and arguments gemm and
// gemm_fp8 share; the caller checks the operand dtypes and holds the device guard.
pb::GemmArgs gemm_args(const Tensor& a, const Tensor& b, Tensor& d, int a_mn, int b_mn, int epi, const c10::optional<Tensor>& bias,
                       const c10::optional<Tensor>& aux, const c10::optional<Tensor>& d2, bool accumulate, double alpha, int cluster,
                       const c10::optional<Tensor>& aux2 = c10::nullopt) {
  check_cuda(d, "d");
  TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && d.dim() == 2, "gemm operands must be 2-D");
  TORCH_CHECK(a.stride(1) == 1 && b.stride(1) == 1 && d.stride(1) == 1, "gemm operands must have unit inner stride");
  pb::GemmArgs g;
  g.M = int(a_mn ? a.size(1) : a.size(0));
  g.K = int(a_mn ? a.size(0) : a.size(1));
  g.N = int(b_mn ? b.size(1) : b.size(0));
  TORCH_CHECK((b_mn ? b.size(0) : b.size(1)) == g.K, "gemm: K mismatch between a and b");
  TORCH_CHECK(d.size(0) == g.M && d.size(1) == g.N, "gemm: output shape mismatch");
  g.A = a.data_ptr(), g.B = b.data_ptr(), g.D = d.data_ptr();
  g.lda = a.stride(0), g.ldb = b.stride(0), g.ldd = d.stride(0);
  g.a_mn = a_mn, g.b_mn = b_mn, g.epi = epi, g.accumulate = accumulate ? 1 : 0, g.alpha = float(alpha);
  if (epi == pb::EPI_F32) {
    TORCH_CHECK(d.scalar_type() == at::kFloat, "EPI_F32 needs a float32 output");
  } else {
    TORCH_CHECK(d.scalar_type() == at::kBFloat16, "bf16 epilogues need a bfloat16 output");
  }
  if (bias.has_value()) {
    check_f32(*bias, "bias");
    TORCH_CHECK(bias->numel() == g.N, "bias length must equal N");
    g.bias = bias->data_ptr<float>();
  }
  if (aux.has_value()) {
    check_bf16(*aux, "aux");
    TORCH_CHECK(aux->size(0) == g.M && aux->size(1) == g.N && aux->stride(1) == 1, "aux must be [M,N]");
    g.aux = aux->data_ptr(), g.ld_aux = aux->stride(0);
  }
  if (aux2.has_value()) {
    check_bf16(*aux2, "aux2");
    TORCH_CHECK(aux2->size(0) == g.M && aux2->size(1) == g.N && aux2->stride(1) == 1, "aux2 must be [M,N]");
    g.aux2 = aux2->data_ptr(), g.ld_aux2 = aux2->stride(0);
  }
  if (d2.has_value()) {
    check_bf16(*d2, "d2");
    TORCH_CHECK(d2->size(0) == g.M && d2->size(1) == g.N && d2->stride(1) == 1, "d2 must be [M,N]");
    g.D2 = d2->data_ptr(), g.ldd2 = d2->stride(0);
  }
  g.num_sms = num_sms();
  g.cluster = cluster;
  return g;
}
void gemm(const Tensor& a, const Tensor& b, Tensor& d, int a_mn, int b_mn, int epi, const c10::optional<Tensor>& bias,
          const c10::optional<Tensor>& aux, c10::optional<Tensor> d2, bool accumulate, double alpha, int cluster,
          const c10::optional<Tensor>& aux2) {
  check_bf16(a, "a");
  check_bf16(b, "b");
  c10::cuda::CUDAGuard guard(a.device());
  pb::gemm_launch(gemm_args(a, b, d, a_mn, b_mn, epi, bias, aux, d2, accumulate, alpha, cluster, aux2), stream_of(a));
}
// `meta` = float32 [3, n_roles] = (scale, scale_inv, amax) rows
void gemm_fp8(const Tensor& a, const Tensor& b, Tensor& d, int a_mn, int b_mn, int epi, int a_fmt, int b_fmt, const Tensor& meta, int role_a,
              int role_b, const c10::optional<Tensor>& bias, const c10::optional<Tensor>& aux, c10::optional<Tensor> d2, bool accumulate,
              double alpha, int cluster, c10::optional<Tensor> d8, int role_out) {
  check_cuda(a, "a");
  check_cuda(b, "b");
  TORCH_CHECK(is_byte(a) && is_byte(b), "gemm_fp8 operands must be 1-byte tensors");
  check_f32(meta, "meta");
  TORCH_CHECK(meta.dim() == 2 && meta.size(0) == 3 && meta.is_contiguous(), "meta must be contiguous float32 [3, n_roles]");
  const int64_t nr = meta.size(1);
  TORCH_CHECK(role_a >= 0 && role_a < nr && role_b >= 0 && role_b < nr, "role index out of range");
  c10::cuda::CUDAGuard guard(a.device());
  pb::GemmArgs g = gemm_args(a, b, d, a_mn, b_mn, epi, bias, aux, d2, accumulate, alpha, cluster);
  g.fp8 = 1, g.a_fmt = a_fmt, g.b_fmt = b_fmt;
  const float* m = meta.data_ptr<float>();
  g.sinv_a = m + nr + role_a, g.sinv_b = m + nr + role_b;
  if (d8.has_value()) {
    TORCH_CHECK(is_byte(*d8) && d8->size(0) == g.M && d8->size(1) == g.N && d8->stride(1) == 1, "d8 must be a 1-byte [M,N] tensor");
    TORCH_CHECK(role_out >= 0 && role_out < nr, "role_out out of range");
    g.D8 = d8->data_ptr(), g.ldd8 = d8->stride(0);
    g.out_scale = m + role_out;
    g.out_amax = const_cast<float*>(m) + 2 * nr + role_out;
  }
  // wgmma reads 8-bit operands K-major only: an MN-major operand is transposed into scratch first
  Tensor at_, bt_;
  if (a_mn) {
    at_ = torch::empty({g.M, g.K}, a.options().dtype(at::kByte));
    pb::transpose_u8(a.data_ptr(), a.stride(0), at_.data_ptr(), g.K, g.M, stream_of(a));
    g.A = at_.data_ptr(), g.lda = g.K, g.a_mn = 0;
  }
  if (b_mn) {
    bt_ = torch::empty({g.N, g.K}, b.options().dtype(at::kByte));
    pb::transpose_u8(b.data_ptr(), b.stride(0), bt_.data_ptr(), g.K, g.N, stream_of(a));
    g.B = bt_.data_ptr(), g.ldb = g.K, g.b_mn = 0;
  }
  pb::gemm_launch(g, stream_of(a));
}
// block-scaled MXFP8: quantise a bf16 matrix (rows padded to `rblk` 128-row blocks in the scale array) / multiply
std::vector<Tensor> mx_quantize(const Tensor& x, int64_t rblk) {
  check_bf16(x, "x");
  TORCH_CHECK(x.dim() == 2 && x.stride(1) == 1 && x.size(1) % 128 == 0, "mx_quantize expects [R,K] with K a multiple of 128");
  const int64_t R = x.size(0), K = x.size(1);
  if (rblk <= 0) rblk = (R + 127) / 128;
  TORCH_CHECK(rblk * 128 >= R, "rblk too small");
  c10::cuda::CUDAGuard guard(x.device());
  auto q = torch::empty({R, K}, x.options().dtype(at::kByte));
  auto sf = torch::zeros({K / 128, rblk, 512}, x.options().dtype(at::kByte));
  pb::mx_quantize(x.data_ptr(), x.stride(0), q.data_ptr(), sf.data_ptr(), R, int(K), int(rblk), stream_of(x));
  return {q, sf};
}
void gemm_mxfp8(const Tensor& a8, const Tensor& b8, Tensor& d, const Tensor& sfa, const Tensor& sfb, const c10::optional<Tensor>& bias) {
  TORCH_CHECK(is_byte(a8) && is_byte(b8) && a8.is_contiguous() && b8.is_contiguous(), "gemm_mxfp8 operands must be contiguous 1-byte matrices");
  check_bf16(d, "d");
  const int M = int(a8.size(0)), K = int(a8.size(1)), N = int(b8.size(0));
  TORCH_CHECK(b8.size(1) == K && d.size(0) == M && d.size(1) == N && d.stride(1) == 1, "gemm_mxfp8: shape mismatch");
  TORCH_CHECK(sfa.is_contiguous() && sfa.numel() == int64_t(K / 128) * ((M + 127) / 128) * 512, "sfa must be [K/128][ceil(M/128)][512]");
  TORCH_CHECK(sfb.is_contiguous() && sfb.numel() == int64_t(K / 128) * (2 * ((N + 255) / 256)) * 512, "sfb must be [K/128][2*ceil(N/256)][512]");
  if (bias.has_value()) check_f32(*bias, "bias");
  c10::cuda::CUDAGuard guard(a8.device());
  pb::gemm_mxfp8_launch(a8.data_ptr(), b8.data_ptr(), d.data_ptr(), sfa.data_ptr(), sfb.data_ptr(), opt_ptr<float>(bias), M, N, K,
                        d.stride(0), num_sms(), stream_of(a8));
}
// the checks of layernorm_fwd_q8 / rmsnorm_fwd_q8 (`mean` is null for RMSNorm); returns meta's role count
int64_t check_norm_fwd_q8(const char* op, const Tensor& x, const Tensor& gamma, const c10::optional<Tensor>& beta, const Tensor& y8,
                          const Tensor* mean, const Tensor& rstd, const Tensor& meta, int role) {
  check_bf16(x, "x");
  check_f32(gamma, "gamma");
  check_f32(meta, "meta");
  TORCH_CHECK(x.is_contiguous() && y8.is_contiguous() && is_byte(y8) && y8.numel() == x.numel(), op, ": y8 must be a contiguous 1-byte tensor shaped like x");
  const int64_t nr = meta.size(1);
  TORCH_CHECK(meta.dim() == 2 && meta.size(0) == 3 && role >= 0 && role < nr, "bad meta / role");
  const int d = int(x.size(-1));
  const int64_t T = x.numel() / d;
  if (mean) check_f32(*mean, "mean");
  check_f32(rstd, "rstd");
  check_numel(gamma, d, op, "gamma");
  if (mean) check_numel(*mean, T, op, "mean");
  check_numel(rstd, T, op, "rstd");
  check_vec(x, op, "x");
  check_vec(gamma, op, "gamma");
  check_vec(y8, op, "y8", 8);
  if (beta.has_value()) {
    check_f32(*beta, "beta");
    check_numel(*beta, d, op, "beta");
    check_vec(*beta, op, "beta");
  }
  return nr;
}
void layernorm_fwd_q8(const Tensor& x, const Tensor& gamma, const c10::optional<Tensor>& beta, Tensor& y8, Tensor& mean, Tensor& rstd,
                      double eps, Tensor& meta, int role) {
  const int64_t nr = check_norm_fwd_q8("layernorm_fwd_q8", x, gamma, beta, y8, &mean, rstd, meta, role);
  const int d = int(x.size(-1));
  c10::cuda::CUDAGuard guard(x.device());
  float* m = meta.data_ptr<float>();
  pb::layernorm_fwd_q8(x.data_ptr(), gamma.data_ptr<float>(), opt_ptr<float>(beta), y8.data_ptr(),
                       mean.data_ptr<float>(), rstd.data_ptr<float>(), x.numel() / d, d, float(eps), m + role, m + 2 * nr + role, stream_of(x));
}
void rmsnorm_fwd_q8(const Tensor& x, const Tensor& gamma, Tensor& y8, Tensor& rstd, double eps, Tensor& meta, int role) {
  const int64_t nr = check_norm_fwd_q8("rmsnorm_fwd_q8", x, gamma, c10::nullopt, y8, nullptr, rstd, meta, role);
  const int d = int(x.size(-1));
  c10::cuda::CUDAGuard guard(x.device());
  float* m = meta.data_ptr<float>();
  pb::rmsnorm_fwd_q8(x.data_ptr(), gamma.data_ptr<float>(), y8.data_ptr(), rstd.data_ptr<float>(), x.numel() / d, d, float(eps), m + role,
                     m + 2 * nr + role, stream_of(x));
}
// out_sum[j] += sum_t dy[t,j] and / or y8 = fp8(dy * scale[role]) with amax[role] updated — one read of dy
void colsum_quant(const Tensor& dy, c10::optional<Tensor> out_sum, c10::optional<Tensor> y8, int fmt, c10::optional<Tensor> meta, int role) {
  check_bf16(dy, "dy");
  TORCH_CHECK(dy.dim() == 2 && dy.stride(1) == 1, "colsum_quant expects [T,N] with unit inner stride");
  check_vec(dy, "colsum_quant", "dy");
  if (y8.has_value()) check_vec(*y8, "colsum_quant", "y8", 8);
  if (out_sum.has_value()) {
    check_f32(*out_sum, "out_sum");
    check_numel(*out_sum, dy.size(1), "colsum_quant", "out_sum");
  }
  c10::cuda::CUDAGuard guard(dy.device());
  const float* scale = nullptr;
  float* amax = nullptr;
  void* y = nullptr;
  long long ld8 = 0;
  if (y8.has_value()) {
    TORCH_CHECK(meta.has_value(), "quantising needs the meta tensor");
    check_f32(*meta, "meta");
    const int64_t nr = meta->size(1);
    TORCH_CHECK(meta->dim() == 2 && meta->size(0) == 3 && role >= 0 && role < nr, "bad meta / role");
    TORCH_CHECK(is_byte(*y8) && y8->dim() == 2 && y8->size(0) == dy.size(0) && y8->size(1) == dy.size(1) && y8->stride(1) == 1 &&
                    y8->stride(0) % 8 == 0, "y8 must be a 1-byte [T,N] tensor");
    scale = meta->data_ptr<float>() + role;
    amax = meta->data_ptr<float>() + 2 * nr + role;
    y = y8->data_ptr(), ld8 = y8->stride(0);
  }
  pb::colsum_quant(dy.data_ptr(), dy.stride(0), opt_ptr<float>(out_sum), y, ld8, fmt, scale, amax,
                   dy.size(0), int(dy.size(1)), stream_of(dy));
}
void fp8_quantize_segments(const Tensor& src, Tensor& dst8, const Tensor& seg, Tensor& meta, int role0) {
  check_bf16(src, "src");
  check_cuda(seg, "seg");
  check_f32(meta, "meta");
  TORCH_CHECK(seg.scalar_type() == at::kLong && seg.dim() == 2 && seg.size(1) == 2 && seg.is_contiguous(), "seg must be int64 [n,2] on the device");
  TORCH_CHECK(is_byte(dst8) && dst8.numel() >= src.numel(), "dst8 must be a 1-byte tensor at least as long as src");
  const int64_t nr = meta.size(1);
  const int n = int(seg.size(0));
  TORCH_CHECK(role0 >= 0 && role0 + n <= nr, "roles out of range");
  c10::cuda::CUDAGuard guard(src.device());
  float* m = meta.data_ptr<float>();
  pb::quantize_segments(src.data_ptr(), dst8.data_ptr(), reinterpret_cast<const long long*>(seg.data_ptr<int64_t>()), n, m + role0,
                        m + nr + role0, m + 2 * nr + role0, stream_of(src));
}
void fp8_update_scales(Tensor& meta, Tensor& hist, const Tensor& fmax, Tensor& pos, int n, double margin_mult) {
  check_f32(meta, "meta");
  check_f32(hist, "hist");
  check_f32(fmax, "fmax");
  TORCH_CHECK(pos.scalar_type() == at::kInt && pos.is_cuda(), "pos must be an int32 device tensor");
  const int64_t nr = meta.size(1);
  TORCH_CHECK(n <= nr && hist.dim() == 2 && hist.size(0) >= n && fmax.numel() >= n && hist.is_contiguous(), "bad history / fmax shapes");
  c10::cuda::CUDAGuard guard(meta.device());
  float* m = meta.data_ptr<float>();
  pb::update_scales(m, m + nr, m + 2 * nr, hist.data_ptr<float>(), fmax.data_ptr<float>(), pos.data_ptr<int>(), n, int(hist.size(1)),
                    float(margin_mult), stream_of(meta));
}

// ---------------------------------------------------------------------------------- attention
// n_kv_heads = -1 means multi-head attention: as many kv heads as query heads
inline int kv_heads(int n_heads, int n_kv_heads) { return n_kv_heads == -1 ? n_heads : n_kv_heads; }
// head counts of a fused qkv row of `width` elements: H q heads, then Hkv k heads and Hkv v heads of d_head each; returns d_head
int64_t check_qkv_heads(int64_t width, int n_heads, int n_kv_heads, const char* what) {
  TORCH_CHECK(n_heads > 0 && n_kv_heads > 0 && n_heads % n_kv_heads == 0, what, ": n_kv_heads = ", n_kv_heads,
              " must be positive and divide n_heads = ", n_heads);
  const int64_t units = int64_t(n_heads) + 2 * int64_t(n_kv_heads);
  TORCH_CHECK(width % units == 0, what, ": a qkv row of ", width, " elements is not (n_heads + 2 * n_kv_heads) = ", units,
              " heads of equal size");
  return width / units;
}
// shapes shared by the forward and the backward: qkv [B,S,(H+2*Hkv)*dh]; o-like tensors [B,S,H*dh]; row statistics fp32 [B,H,S]
void check_attention_args(const Tensor& qkv, const Tensor& out, const Tensor& lse, int n_heads, int n_kv_heads, bool causal,
                          const c10::optional<Tensor>& alibi_slopes) {
  TORCH_CHECK(qkv.dim() == 3 && qkv.is_contiguous(), "qkv must be contiguous [B,S,(n_heads+2*n_kv_heads)*d_head]");
  const int64_t B = qkv.size(0), S = qkv.size(1), d = check_qkv_heads(qkv.size(2), n_heads, n_kv_heads, "attention") * n_heads;
  TORCH_CHECK(out.is_contiguous() && out.sizes() == at::IntArrayRef({B, S, d}), "out must be contiguous [B,S,d]");
  TORCH_CHECK(lse.is_contiguous() && lse.sizes() == at::IntArrayRef({B, int64_t(n_heads), S}), "lse must be contiguous float32 [B,H,S]");
  if (alibi_slopes.has_value()) {
    TORCH_CHECK(causal, "attention: ALiBi slopes are only supported with the causal mask");
    check_f32(*alibi_slopes, "alibi_slopes");
    TORCH_CHECK(alibi_slopes->numel() == n_heads && alibi_slopes->is_contiguous(), "alibi_slopes must be contiguous with n_heads elements");
  }
}
// document-mask bounds (doc_bounds): int32 [B*S] on the device of qkv, contiguous; the mask is a refinement of the causal one
void check_doc_bound(const c10::optional<Tensor>& t, const char* name, const Tensor& qkv) {
  if (!t.has_value()) return;
  check_cuda(*t, name);
  TORCH_CHECK(t->scalar_type() == at::kInt, name, " must be int32");
  TORCH_CHECK(t->device() == qkv.device(), name, " must be on the device of qkv");
  TORCH_CHECK(t->is_contiguous() && t->numel() == qkv.size(0) * qkv.size(1), name, " must be contiguous int32 with B*S elements");
}
void check_doc_args(const Tensor& qkv, bool causal, const c10::optional<Tensor>& doc_start, const c10::optional<Tensor>& doc_end) {
  TORCH_CHECK(!doc_end.has_value() || doc_start.has_value(), "attention: doc_end without doc_start");
  TORCH_CHECK(!doc_start.has_value() || causal, "attention: the document mask is only supported with the causal mask");
  check_doc_bound(doc_start, "doc_start", qkv);
  check_doc_bound(doc_end, "doc_end", qkv);
}
// sliding window: -1 = off, otherwise query q sees keys q - window .. q; only with the causal mask
void check_window(int window, bool causal, const char* op) {
  TORCH_CHECK(window >= -1, op, ": sliding window ", window, " must be -1 (off) or >= 0");
  TORCH_CHECK(window == -1 || causal, op, ": a sliding window is only supported with the causal mask");
}
void attention_fwd(const Tensor& qkv, Tensor& out, Tensor& lse, int n_heads, double scale, bool causal,
                   const c10::optional<Tensor>& alibi_slopes, const c10::optional<Tensor>& doc_start, int n_kv_heads, int window) {
  check_bf16(qkv, "qkv");
  check_bf16(out, "out");
  check_f32(lse, "lse");
  n_kv_heads = kv_heads(n_heads, n_kv_heads);
  check_attention_args(qkv, out, lse, n_heads, n_kv_heads, causal, alibi_slopes);
  check_doc_args(qkv, causal, doc_start, c10::nullopt);
  check_window(window, causal, "attention_fwd");
  c10::cuda::CUDAGuard guard(qkv.device());
  const int B = int(qkv.size(0)), S = int(qkv.size(1)), dh = int(qkv.size(2) / (n_heads + 2 * n_kv_heads));
  pb::attention_fwd_launch(qkv.data_ptr(), out.data_ptr(), lse.data_ptr<float>(), B, S, n_heads, n_kv_heads, dh, float(scale), causal,
                           stream_of(qkv), opt_ptr<float>(alibi_slopes), opt_ptr<int>(doc_start), window);
}
void attention_bwd(const Tensor& qkv, const Tensor& out, const Tensor& dout, const Tensor& lse, Tensor& dqkv, Tensor& delta,
                   int n_heads, double scale, bool causal, const c10::optional<Tensor>& alibi_slopes,
                   const c10::optional<Tensor>& doc_start, const c10::optional<Tensor>& doc_end, int n_kv_heads, int window) {
  check_bf16(qkv, "qkv");
  check_bf16(out, "out");
  check_bf16(dout, "dout");
  check_bf16(dqkv, "dqkv");
  check_f32(lse, "lse");
  check_f32(delta, "delta");
  n_kv_heads = kv_heads(n_heads, n_kv_heads);
  check_attention_args(qkv, out, lse, n_heads, n_kv_heads, causal, alibi_slopes);
  check_doc_args(qkv, causal, doc_start, doc_end);
  TORCH_CHECK(doc_start.has_value() == doc_end.has_value(), "attention_bwd: doc_start needs doc_end");
  check_window(window, causal, "attention_bwd");
  TORCH_CHECK(dout.is_contiguous() && dout.sizes() == out.sizes(), "dout must be contiguous [B,S,d]");
  TORCH_CHECK(delta.is_contiguous() && delta.sizes() == lse.sizes(), "delta must be contiguous float32 [B,H,S]");
  TORCH_CHECK(dqkv.is_contiguous() && dqkv.sizes() == qkv.sizes(), "dqkv must be contiguous and shaped like qkv");
  c10::cuda::CUDAGuard guard(qkv.device());
  const int B = int(qkv.size(0)), S = int(qkv.size(1)), dh = int(qkv.size(2) / (n_heads + 2 * n_kv_heads)), d = n_heads * dh;
  // the fp32 dQ accumulator comes from the caching allocator on this stream: eagerly it is recycled in stream order, under
  // CUDA-graph capture it comes from the graph's private pool and lives as long as the graph
  Tensor dq_acc = at::empty({(int64_t)B * S, d}, qkv.options().dtype(at::kFloat));
  pb::attention_bwd_launch(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr<float>(), dqkv.data_ptr(), delta.data_ptr<float>(),
                           dq_acc.data_ptr<float>(), B, S, n_heads, n_kv_heads, dh, float(scale), causal, num_sms(), stream_of(qkv),
                           opt_ptr<float>(alibi_slopes), opt_ptr<int>(doc_start), opt_ptr<int>(doc_end), window);
}
// sequence_id int64 [B,S] -> doc_start / doc_end int32 [B*S] (first / last row of each row's document)
void doc_bounds(const Tensor& sequence_id, Tensor& doc_start, Tensor& doc_end) {
  check_cuda(sequence_id, "sequence_id");
  TORCH_CHECK(sequence_id.scalar_type() == at::kLong && sequence_id.dim() == 2 && sequence_id.is_contiguous(),
              "sequence_id must be contiguous int64 [B,S]");
  const int64_t B = sequence_id.size(0), S = sequence_id.size(1);
  for (const Tensor* t : {&doc_start, &doc_end}) {
    check_cuda(*t, "doc bounds");
    TORCH_CHECK(t->scalar_type() == at::kInt && t->is_contiguous() && t->numel() == B * S && t->device() == sequence_id.device(),
                "doc_start / doc_end must be contiguous int32 with B*S elements on the device of sequence_id");
  }
  c10::cuda::CUDAGuard guard(sequence_id.device());
  if (B == 0 || S == 0) return;
  pb::doc_bounds_launch(reinterpret_cast<const long long*>(sequence_id.data_ptr<int64_t>()), doc_start.data_ptr<int>(),
                        doc_end.data_ptr<int>(), int(B), int(S), stream_of(sequence_id));
}
void rope(Tensor& qkv, const Tensor& cos_t, const Tensor& sin_t, int n_heads, bool inverse, int n_kv_heads) {
  check_bf16(qkv, "qkv");
  check_f32(cos_t, "cos");
  check_f32(sin_t, "sin");
  TORCH_CHECK(qkv.dim() == 3 && qkv.is_contiguous(), "qkv must be contiguous [B,S,(n_heads+2*n_kv_heads)*d_head]");
  n_kv_heads = kv_heads(n_heads, n_kv_heads);
  const int dh = int(check_qkv_heads(qkv.size(2), n_heads, n_kv_heads, "rope"));
  c10::cuda::CUDAGuard guard(qkv.device());
  const int S = int(qkv.size(1));
  TORCH_CHECK(cos_t.is_contiguous() && sin_t.is_contiguous() && cos_t.size(0) >= S && cos_t.size(1) == dh / 2, "cos/sin must be [>=S, dh/2]");
  pb::rope_launch(qkv.data_ptr(), cos_t.data_ptr<float>(), sin_t.data_ptr<float>(), (long long)qkv.size(0) * S, S, n_heads, n_kv_heads, dh, inverse,
                  stream_of(qkv));
}

// ---------------------------------------------------------------------------------- decoding
inline void check_i32(const Tensor& t, const char* name) {
  check_cuda(t, name);
  TORCH_CHECK(t.scalar_type() == at::kInt && t.is_contiguous(), name, " must be contiguous int32");
}
// one layer of the k / v cache, [B_max, Hkv, S_max, dh], with Hkv the resolved n_kv_heads, which divides n_heads
void check_kv_cache(const Tensor& kc, const Tensor& vc, int n_heads, int n_kv_heads, const char* op) {
  check_bf16(kc, "k_cache");
  check_bf16(vc, "v_cache");
  TORCH_CHECK(kc.dim() == 4 && kc.is_contiguous() && vc.sizes() == kc.sizes() && vc.is_contiguous(), "k/v cache must be contiguous [B_max, Hkv, S_max, dh]");
  TORCH_CHECK(n_heads > 0 && n_kv_heads > 0 && kc.size(1) == n_kv_heads && n_heads % n_kv_heads == 0, op,
              ": cache heads must equal n_kv_heads and n_kv_heads divide n_heads");
}
// y[M,N] = epilogue(x[M,K] w[N,K]^T), 1 <= M <= 64
void skinny_gemm(const Tensor& x, const Tensor& w, Tensor& y, const c10::optional<Tensor>& bias, const c10::optional<Tensor>& residual,
                 int epi) {
  check_bf16(x, "x");
  check_bf16(w, "w");
  check_bf16(y, "y");
  TORCH_CHECK(x.dim() == 2 && w.dim() == 2 && y.dim() == 2, "skinny_gemm operands must be 2-D");
  TORCH_CHECK(x.stride(1) == 1 && w.stride(1) == 1 && y.stride(1) == 1, "skinny_gemm operands must have unit inner stride");
  TORCH_CHECK(x.size(1) == w.size(1), "skinny_gemm: K mismatch between x and w");
  TORCH_CHECK(y.size(0) == x.size(0) && y.size(1) == w.size(0), "skinny_gemm: output must be [M, N]");
  TORCH_CHECK(x.size(0) >= 1 && x.size(0) <= 64, "skinny_gemm: 1 <= M <= 64 rows");
  TORCH_CHECK(x.size(1) > 0 && x.size(1) % 8 == 0 && w.size(0) > 0, "skinny_gemm: K must be a positive multiple of 8 and N positive");
  check_vec(x, "skinny_gemm", "x");
  check_vec(w, "skinny_gemm", "w");
  TORCH_CHECK(epi >= pb::SKINNY_PLAIN && epi <= pb::SKINNY_MUL, "skinny_gemm: unknown epilogue");
  c10::cuda::CUDAGuard guard(x.device());
  pb::SkinnyArgs a;
  a.X = x.data_ptr(), a.W = w.data_ptr(), a.Y = y.data_ptr();
  a.ldx = x.stride(0), a.ldw = w.stride(0), a.ldy = y.stride(0);
  a.M = int(x.size(0)), a.N = int(w.size(0)), a.K = int(x.size(1));
  a.epi = epi;
  if (bias.has_value()) {
    check_f32(*bias, "bias");
    TORCH_CHECK(bias->numel() == a.N && bias->is_contiguous(), "bias must be contiguous with N elements");
    a.bias = bias->data_ptr<float>();
  }
  if (epi == pb::SKINNY_RESIDUAL || epi == pb::SKINNY_MUL) {
    TORCH_CHECK(residual.has_value(), "the residual and multiply epilogues need the residual / multiplier");
    check_bf16(*residual, "residual");
    TORCH_CHECK(residual->dim() == 2 && residual->size(0) == a.M && residual->size(1) == a.N && residual->stride(1) == 1,
                "residual must be [M, N]");
    a.R = residual->data_ptr(), a.ldr = residual->stride(0);
  }
  a.num_sms = num_sms();
  const int splits = pb::skinny_gemm_splits(a.M, a.N, a.K, a.num_sms);
  Tensor part;
  if (splits > 1) part = torch::empty({(long long)splits * a.M * a.N}, x.options().dtype(at::kFloat));
  pb::skinny_gemm_launch(a, splits > 1 ? part.data_ptr<float>() : nullptr, stream_of(x));
}
// kc / vc: one layer of the cache, [B_max, Hkv, S_max, dh]; q: rows of [B, >= H*dh] (the q heads of the fused qkv)
void decode_attention(const Tensor& q, const Tensor& kc, const Tensor& vc, const Tensor& pos, Tensor& out, int n_heads, double scale,
                      const c10::optional<Tensor>& alibi_slopes, int n_kv_heads, int window) {
  check_bf16(q, "q");
  check_bf16(out, "out");
  check_i32(pos, "pos");
  n_kv_heads = kv_heads(n_heads, n_kv_heads);
  check_kv_cache(kc, vc, n_heads, n_kv_heads, "decode_attention");
  const int B = int(q.size(0)), Hkv = int(kc.size(1)), H = n_heads, S = int(kc.size(2)), dh = int(kc.size(3));
  TORCH_CHECK(dh == 64 || dh == 128, "decode_attention: d_head must be 64 or 128");
  TORCH_CHECK(B <= kc.size(0) && pos.numel() >= B, "decode_attention: batch larger than the cache or the position vector");
  TORCH_CHECK(q.dim() == 2 && q.stride(1) == 1 && q.size(1) >= H * dh, "q must be [B, >= H*dh] with unit inner stride");
  TORCH_CHECK(out.dim() == 2 && out.size(0) == B && out.size(1) == H * dh && out.stride(1) == 1, "out must be [B, H*dh]");
  if (alibi_slopes.has_value()) {
    check_f32(*alibi_slopes, "alibi_slopes");
    TORCH_CHECK(alibi_slopes->numel() == n_heads, "alibi_slopes must have n_heads elements");
  }
  check_window(window, true, "decode_attention");
  c10::cuda::CUDAGuard guard(q.device());
  const int splits = pb::decode_attention_splits(S);
  Tensor po = torch::empty({(long long)B * H * splits * dh}, q.options().dtype(at::kFloat));
  Tensor pml = torch::empty({(long long)B * H * splits * 2}, q.options().dtype(at::kFloat));
  pb::decode_attention_launch(q.data_ptr(), q.stride(0), kc.data_ptr(), vc.data_ptr(), pos.data_ptr<int>(), out.data_ptr(), out.stride(0),
                              po.data_ptr<float>(), pml.data_ptr<float>(), B, H, Hkv, dh, S, float(scale), opt_ptr<float>(alibi_slopes),
                              stream_of(q), window);
}
void decode_append(Tensor& qkv, const Tensor& pos, Tensor& kc, Tensor& vc, const c10::optional<Tensor>& cos_t,
                   const c10::optional<Tensor>& sin_t, int n_heads, const c10::optional<Tensor>& slot, int n_kv_heads) {
  check_bf16(qkv, "qkv");
  check_i32(pos, "pos");
  n_kv_heads = kv_heads(n_heads, n_kv_heads);
  check_kv_cache(kc, vc, n_heads, n_kv_heads, "decode_append");
  const int B = int(qkv.size(0)), Hkv = int(kc.size(1)), H = n_heads, S = int(kc.size(2)), dh = int(kc.size(3));
  TORCH_CHECK(qkv.dim() == 2 && qkv.size(1) == (H + 2 * Hkv) * dh && qkv.stride(1) == 1, "qkv must be [B, (n_heads+2*n_kv_heads)*d_head]");
  check_vec(qkv, "decode_append", "qkv");
  TORCH_CHECK(pos.numel() >= B, "decode_append: position vector shorter than the batch");
  if (slot.has_value()) {
    check_i32(*slot, "slot");
    TORCH_CHECK(slot->numel() >= B, "decode_append: slot vector shorter than the batch");
  } else {
    TORCH_CHECK(B <= kc.size(0), "decode_append: batch larger than the cache");
  }
  TORCH_CHECK(cos_t.has_value() == sin_t.has_value(), "decode_append: pass both RoPE tables or neither");
  if (cos_t.has_value()) {
    check_f32(*cos_t, "cos");
    check_f32(*sin_t, "sin");
    TORCH_CHECK(cos_t->is_contiguous() && sin_t->is_contiguous() && cos_t->size(0) >= S && cos_t->size(1) == dh / 2,
                "cos/sin must be [>= S_max, dh/2]");
  }
  c10::cuda::CUDAGuard guard(qkv.device());
  pb::decode_append_launch(qkv.data_ptr(), qkv.stride(0), pos.data_ptr<int>(), kc.data_ptr(), vc.data_ptr(), opt_ptr<float>(cos_t),
                           opt_ptr<float>(sin_t), B, H, Hkv, dh, S, opt_ptr<int>(slot), stream_of(qkv));
}
// query rows of qkv [N, (H+2*Hkv)*dh] in tiles (int32 [T, 4]: slot, first_row, n_rows <= 64, first_pos) against one cache layer
void cache_attention(const Tensor& qkv, const Tensor& kc, const Tensor& vc, const Tensor& tiles, Tensor& out, int n_heads, double scale,
                     const c10::optional<Tensor>& alibi_slopes, int n_kv_heads, int window) {
  check_bf16(qkv, "qkv");
  check_bf16(out, "out");
  check_i32(tiles, "tiles");
  n_kv_heads = kv_heads(n_heads, n_kv_heads);
  check_kv_cache(kc, vc, n_heads, n_kv_heads, "cache_attention");
  const int Bm = int(kc.size(0)), Hkv = int(kc.size(1)), H = n_heads, S = int(kc.size(2)), dh = int(kc.size(3));
  TORCH_CHECK(dh == 64 || dh == 128, "cache_attention: d_head must be 64 or 128");
  TORCH_CHECK(qkv.dim() == 2 && qkv.size(1) == (H + 2 * Hkv) * dh && qkv.stride(1) == 1,
              "qkv must be [N, (n_heads+2*n_kv_heads)*d_head] with unit inner stride");
  check_vec(qkv, "cache_attention", "qkv");
  TORCH_CHECK(out.dim() == 2 && out.size(0) == qkv.size(0) && out.size(1) == H * dh && out.stride(1) == 1, "out must be [N, H*dh]");
  check_vec(out, "cache_attention", "out");
  TORCH_CHECK(tiles.dim() == 2 && tiles.size(1) == 4, "tiles must be int32 [T, 4] (slot, first_row, n_rows, first_pos)");
  if (alibi_slopes.has_value()) {
    check_f32(*alibi_slopes, "alibi_slopes");
    TORCH_CHECK(alibi_slopes->numel() == n_heads, "alibi_slopes must have n_heads elements");
  }
  check_window(window, true, "cache_attention");
  c10::cuda::CUDAGuard guard(qkv.device());
  pb::cache_attention_launch(qkv.data_ptr(), qkv.stride(0), qkv.size(0), kc.data_ptr(), vc.data_ptr(), tiles.data_ptr<int>(),
                             int(tiles.size(0)), out.data_ptr(), out.stride(0), Bm, H, Hkv, dh, S, float(scale), opt_ptr<float>(alibi_slopes),
                             stream_of(qkv), window);
}
void embed_pos(const Tensor& ids, const Tensor& pos, const Tensor& wte, const c10::optional<Tensor>& wpe, Tensor& out) {
  check_i32(ids, "ids");
  check_i32(pos, "pos");
  check_bf16(wte, "wte");
  check_bf16(out, "out");
  const int B = int(out.size(0)), d = int(wte.size(1));
  TORCH_CHECK(out.dim() == 2 && out.size(1) == d && out.is_contiguous() && d % 8 == 0, "out must be contiguous [B, d], d % 8 == 0");
  TORCH_CHECK(ids.numel() >= B && pos.numel() >= B, "ids / pos shorter than the batch");
  if (wpe.has_value()) {
    check_bf16(*wpe, "wpe");
    TORCH_CHECK(wpe->size(1) == d && wpe->is_contiguous(), "wpe must be contiguous [S, d]");
  }
  c10::cuda::CUDAGuard guard(ids.device());
  pb::embed_pos_launch(ids.data_ptr<int>(), pos.data_ptr<int>(), wte.data_ptr(), opt_ptr(wpe), out.data_ptr(), B, d, int(wte.size(0)),
                       stream_of(ids));
}
void argmax_advance(const Tensor& logits, Tensor& ids, c10::optional<Tensor> pos) {
  check_bf16(logits, "logits");
  check_i32(ids, "ids");
  TORCH_CHECK(logits.dim() == 2 && logits.stride(1) == 1, "logits must be [B, V] with unit inner stride");
  const int B = int(logits.size(0));
  TORCH_CHECK(ids.numel() >= B, "ids shorter than the batch");
  if (pos.has_value()) {
    check_i32(*pos, "pos");
    TORCH_CHECK(pos->numel() >= B, "pos shorter than the batch");
  }
  c10::cuda::CUDAGuard guard(logits.device());
  pb::argmax_advance_launch(logits.data_ptr(), logits.stride(0), B, int(logits.size(1)), ids.data_ptr<int>(), opt_ptr<int>(pos),
                            stream_of(logits));
}

// ---------------------------------------------------------------------------------- fused ops
void embed_fwd(const Tensor& ids, const Tensor& wte, const c10::optional<Tensor>& wpe, Tensor& out, int S) {
  check_cuda(ids, "ids");
  TORCH_CHECK(ids.scalar_type() == at::kLong && ids.is_contiguous(), "ids must be contiguous int64");
  check_bf16(wte, "wte");
  check_bf16(out, "out");
  TORCH_CHECK(wte.dim() == 2 && wte.is_contiguous() && wte.size(1) % 8 == 0, "embed_fwd: wte must be contiguous [V,d], d % 8 == 0");
  const int d = int(wte.size(1));
  TORCH_CHECK(out.is_contiguous() && out.numel() == ids.numel() * d, "embed_fwd: out must be contiguous [T,d]");
  TORCH_CHECK(S > 0, "embed_fwd: seq_len must be positive");
  check_vec(wte, "embed_fwd", "wte");
  check_vec(out, "embed_fwd", "out");
  if (wpe.has_value()) {
    check_bf16(*wpe, "wpe");
    TORCH_CHECK(wpe->dim() == 2 && wpe->size(1) == d && wpe->size(0) >= S && wpe->is_contiguous(), "embed_fwd: wpe must be contiguous [>=S,d]");
    check_vec(*wpe, "embed_fwd", "wpe");
  }
  c10::cuda::CUDAGuard guard(ids.device());
  pb::embed_fwd(ids.data_ptr<int64_t>(), wte.data_ptr(), opt_ptr(wpe), out.data_ptr(), ids.numel(), S, d, int(wte.size(0)), stream_of(ids));
}
// dwte / dwpe: either may be None (a frozen embedding); the kernel of a missing one is not launched
void embed_bwd(const Tensor& ids, const Tensor& dh, c10::optional<Tensor> dwte, c10::optional<Tensor> dwpe, int S) {
  check_cuda(ids, "ids");
  TORCH_CHECK(ids.scalar_type() == at::kLong && ids.is_contiguous(), "ids must be contiguous int64");
  check_bf16(dh, "dh");
  TORCH_CHECK(dh.dim() == 2 && dh.is_contiguous() && dh.size(0) == ids.numel() && dh.size(1) % 8 == 0, "dh must be contiguous [T,d], d % 8 == 0");
  TORCH_CHECK(S > 0 && ids.numel() % S == 0, "the token count must be a multiple of seq_len");
  check_vec(dh, "embed_bwd", "dh");
  const int d = int(dh.size(1));
  if (dwte.has_value()) {
    check_f32(*dwte, "dwte");
    TORCH_CHECK(dwte->dim() == 2 && dwte->size(1) == d && dwte->is_contiguous(), "dwte must be contiguous [V,d]");
    check_vec(*dwte, "embed_bwd", "dwte");
  }
  if (dwpe.has_value()) {
    check_f32(*dwpe, "dwpe");
    TORCH_CHECK(dwpe->dim() == 2 && dwpe->size(1) == d && dwpe->size(0) >= S && dwpe->is_contiguous(), "dwpe must be contiguous [>=S,d]");
    check_vec(*dwpe, "embed_bwd", "dwpe");
  }
  c10::cuda::CUDAGuard guard(ids.device());
  pb::embed_bwd(ids.data_ptr<int64_t>(), dh.data_ptr(), opt_ptr<float>(dwte), opt_ptr<float>(dwpe), ids.numel(), S, d,
                dwte.has_value() ? int(dwte->size(0)) : 0, stream_of(ids));
}
// dst[C,R] = src[R,C]^T for a 1-byte matrix (row stride ld): the K-major copy of an fp8 operand that is stored MN-major
void transpose_u8(const Tensor& src, Tensor& dst) {
  TORCH_CHECK(is_byte(src) && is_byte(dst) && src.dim() == 2 && dst.dim() == 2 && src.stride(1) == 1 && dst.is_contiguous(),
              "transpose_u8 expects 1-byte 2-D tensors with unit inner stride");
  TORCH_CHECK(dst.size(0) == src.size(1) && dst.size(1) == src.size(0), "dst must be [C,R] for src [R,C]");
  c10::cuda::CUDAGuard guard(src.device());
  pb::transpose_u8(src.data_ptr(), src.stride(0), dst.data_ptr(), int(src.size(0)), int(src.size(1)), stream_of(src));
}
// gamma / beta: fp32 [d]; mean / rstd: fp32 [T] with T = x.numel() / d; y / dx / dres shaped like x. `mean` is null for RMSNorm.
void check_layernorm(const char* op, const Tensor& x, const Tensor& gamma, const c10::optional<Tensor>& beta, const Tensor* mean,
                     const Tensor& rstd) {
  check_bf16(x, "x");
  check_f32(gamma, "gamma");
  if (mean) check_f32(*mean, "mean");
  check_f32(rstd, "rstd");
  TORCH_CHECK(x.dim() >= 1 && x.is_contiguous(), op, ": x must be contiguous");
  const int64_t d = x.size(-1);
  TORCH_CHECK(d > 0, op, ": empty rows");
  const int64_t T = x.numel() / d;
  check_numel(gamma, d, op, "gamma");
  if (mean) check_numel(*mean, T, op, "mean");
  check_numel(rstd, T, op, "rstd");
  TORCH_CHECK(gamma.is_contiguous() && (!mean || mean->is_contiguous()) && rstd.is_contiguous(), op,
              ": gamma, mean and rstd must be contiguous");
  check_vec(x, op, "x");
  check_vec(gamma, op, "gamma");
  if (beta.has_value()) {
    check_f32(*beta, "beta");
    check_numel(*beta, d, op, "beta");
    TORCH_CHECK(beta->is_contiguous(), op, ": beta must be contiguous");
    check_vec(*beta, op, "beta");
  }
}
void check_like_x(const char* op, const Tensor& t, const Tensor& x, const char* name) {
  check_bf16(t, name);
  TORCH_CHECK(t.is_contiguous() && t.numel() == x.numel() && t.size(-1) == x.size(-1), op, ": ", name, " must be contiguous and shaped like x");
  check_vec(t, op, name);
}
void layernorm_fwd(const Tensor& x, const Tensor& gamma, const c10::optional<Tensor>& beta, Tensor& y, Tensor& mean, Tensor& rstd,
                   double eps) {
  check_layernorm("layernorm_fwd", x, gamma, beta, &mean, rstd);
  check_like_x("layernorm_fwd", y, x, "y");
  c10::cuda::CUDAGuard guard(x.device());
  const int d = int(x.size(-1));
  pb::layernorm_fwd(x.data_ptr(), gamma.data_ptr<float>(), opt_ptr<float>(beta), y.data_ptr(),
                    mean.data_ptr<float>(), rstd.data_ptr<float>(), x.numel() / d, d, float(eps), stream_of(x));
}
void layernorm_bwd(const Tensor& dy, const Tensor& x, const Tensor& gamma, const Tensor& mean, const Tensor& rstd,
                   const c10::optional<Tensor>& dres, Tensor& dx, c10::optional<Tensor> dgamma, c10::optional<Tensor> dbeta) {
  check_layernorm("layernorm_bwd", x, gamma, c10::nullopt, &mean, rstd);
  check_like_x("layernorm_bwd", dy, x, "dy");
  check_like_x("layernorm_bwd", dx, x, "dx");
  if (dres.has_value()) check_like_x("layernorm_bwd", *dres, x, "dres");
  const int d = int(x.size(-1));
  for (const auto* t : {&dgamma, &dbeta}) {
    if (!t->has_value()) continue;
    check_f32(**t, "dgamma / dbeta");
    check_numel(**t, d, "layernorm_bwd", "dgamma / dbeta");
    TORCH_CHECK((*t)->is_contiguous(), "layernorm_bwd: dgamma / dbeta must be contiguous");
  }
  c10::cuda::CUDAGuard guard(x.device());
  pb::layernorm_bwd(dy.data_ptr(), x.data_ptr(), gamma.data_ptr<float>(), mean.data_ptr<float>(), rstd.data_ptr<float>(), opt_ptr(dres),
                    dx.data_ptr(), opt_ptr<float>(dgamma), opt_ptr<float>(dbeta), x.numel() / d, d, stream_of(x));
}
void rmsnorm_fwd(const Tensor& x, const Tensor& gamma, Tensor& y, Tensor& rstd, double eps) {
  check_layernorm("rmsnorm_fwd", x, gamma, c10::nullopt, nullptr, rstd);
  check_like_x("rmsnorm_fwd", y, x, "y");
  c10::cuda::CUDAGuard guard(x.device());
  const int d = int(x.size(-1));
  pb::rmsnorm_fwd(x.data_ptr(), gamma.data_ptr<float>(), y.data_ptr(), rstd.data_ptr<float>(), x.numel() / d, d, float(eps), stream_of(x));
}
void rmsnorm_bwd(const Tensor& dy, const Tensor& x, const Tensor& gamma, const Tensor& rstd, const c10::optional<Tensor>& dres, Tensor& dx,
                 c10::optional<Tensor> dgamma) {
  check_layernorm("rmsnorm_bwd", x, gamma, c10::nullopt, nullptr, rstd);
  check_like_x("rmsnorm_bwd", dy, x, "dy");
  check_like_x("rmsnorm_bwd", dx, x, "dx");
  if (dres.has_value()) check_like_x("rmsnorm_bwd", *dres, x, "dres");
  const int d = int(x.size(-1));
  if (dgamma.has_value()) {
    check_f32(*dgamma, "dgamma");
    check_numel(*dgamma, d, "rmsnorm_bwd", "dgamma");
    TORCH_CHECK(dgamma->is_contiguous(), "rmsnorm_bwd: dgamma must be contiguous");
  }
  c10::cuda::CUDAGuard guard(x.device());
  pb::rmsnorm_bwd(dy.data_ptr(), x.data_ptr(), gamma.data_ptr<float>(), rstd.data_ptr<float>(), opt_ptr(dres), dx.data_ptr(),
                  opt_ptr<float>(dgamma), x.numel() / d, d, stream_of(x));
}
void col_sum(const Tensor& dy, Tensor& out) {
  check_bf16(dy, "dy");
  check_f32(out, "out");
  TORCH_CHECK(dy.dim() == 2 && dy.stride(1) == 1, "col_sum expects [T,N] with unit inner stride");
  TORCH_CHECK(dy.size(1) % 8 == 0, "col_sum: the row length must be a multiple of 8");
  TORCH_CHECK(out.is_contiguous(), "col_sum: out must be contiguous");
  check_numel(out, dy.size(1), "col_sum", "out");
  check_vec(dy, "col_sum", "dy");
  c10::cuda::CUDAGuard guard(dy.device());
  pb::col_reduce(dy.data_ptr(), dy.stride(0), nullptr, nullptr, nullptr, out.data_ptr<float>(), nullptr, dy.size(0), int(dy.size(1)),
                 stream_of(dy));
}
void cross_entropy(Tensor& logits, const Tensor& targets, double grad_scale, bool write_grad, Tensor& stats,
                   c10::optional<Tensor> row_lse, const c10::optional<Tensor>& unigram_logp, double head_scale, double head_cap) {
  check_bf16(logits, "logits");
  TORCH_CHECK(logits.dim() == 2 && logits.stride(1) == 1, "logits must be [rows,V]");
  TORCH_CHECK(targets.scalar_type() == at::kLong && targets.is_contiguous(), "targets must be contiguous int64");
  TORCH_CHECK(targets.numel() == logits.size(0), "cross_entropy: one target per row of logits");
  TORCH_CHECK(stats.scalar_type() == at::kDouble && stats.numel() >= 4, "stats must be float64[>=4]");
  check_cuda(targets, "targets");
  check_cuda(stats, "stats");
  check_vec(logits, "cross_entropy", "logits");
  if (row_lse.has_value()) {
    check_f32(*row_lse, "row_lse");
    TORCH_CHECK(row_lse->is_contiguous() && row_lse->numel() >= logits.size(0), "cross_entropy: row_lse must be contiguous [>=rows]");
  }
  if (unigram_logp.has_value()) {
    check_f32(*unigram_logp, "unigram_logp");
    TORCH_CHECK(unigram_logp->is_contiguous() && unigram_logp->numel() >= logits.size(1), "cross_entropy: unigram_logp must be contiguous [>=V]");
  }
  TORCH_CHECK(head_scale > 0 && std::isfinite(head_scale), "cross_entropy: the logit scale must be positive and finite");
  TORCH_CHECK(head_cap >= 0 && std::isfinite(head_cap), "cross_entropy: the logit cap must be 0 (none) or positive and finite");
  c10::cuda::CUDAGuard guard(logits.device());
  pb::cross_entropy(logits.data_ptr(), logits.stride(0), targets.data_ptr<int64_t>(), logits.size(0), int(logits.size(1)), float(grad_scale),
                    write_grad, stats.data_ptr<double>(), opt_ptr<float>(row_lse), opt_ptr<float>(unigram_logp), float(head_scale),
                    float(head_cap), stream_of(logits));
}
// any length: the kernel reads float4s and then the last numel % 4 elements
void flat_l2_norm(const Tensor& x, Tensor& scratch_f64, Tensor& out_f32) {
  check_f32(x, "x");
  TORCH_CHECK(x.is_contiguous(), "flat_l2_norm: x must be contiguous");
  check_vec(x, "flat_l2_norm", "x");
  c10::cuda::CUDAGuard guard(x.device());
  cudaStream_t st = stream_of(x);
  CUDA_OK(cudaMemsetAsync(scratch_f64.data_ptr(), 0, sizeof(double), st));
  pb::flat_sqnorm(x.data_ptr<float>(), x.numel(), scratch_f64.data_ptr<double>(), st);
  pb::sqrt_finalize(scratch_f64.data_ptr<double>(), out_f32.data_ptr<float>(), st);
}
void axpby(Tensor& acc, const Tensor& x, double a, double b) {
  check_f32(acc, "acc");
  check_f32(x, "x");
  TORCH_CHECK(acc.numel() == x.numel() && acc.numel() % 4 == 0, "axpby: sizes must match and be multiples of 4");
  c10::cuda::CUDAGuard guard(acc.device());
  pb::axpby(acc.data_ptr<float>(), x.data_ptr<float>(), float(a), float(b), acc.numel(), stream_of(acc));
}
void cast_bf16(const Tensor& src, Tensor& dst) {
  check_f32(src, "src");
  check_bf16(dst, "dst");
  TORCH_CHECK(src.numel() == dst.numel() && src.numel() % 4 == 0, "cast: sizes must match and be multiples of 4");
  c10::cuda::CUDAGuard guard(src.device());
  pb::cast_fp32_to_bf16(src.data_ptr<float>(), dst.data_ptr(), src.numel(), stream_of(src));
}
void fused_optimizer(Tensor& p, const Tensor& g, Tensor& m, Tensor& v, c10::optional<Tensor> shadow, int kind, bool first_step, double lr,
                     double beta1, double beta2, double eps, double decay, double clip, double step_size, double inv_sqrt_bc2,
                     const c10::optional<Tensor>& grad_mult, double wd) {
  check_f32(p, "p");
  check_f32(g, "g");
  TORCH_CHECK(p.numel() % 4 == 0, "flat buffers must be multiples of 4 elements");
  // every plane the kernel touches is read / written as float4 (the shadow as 4 bf16) at the same index as p
  std::vector<std::pair<const Tensor*, const char*>> planes{{&p, "p"}, {&g, "g"}};
  if (kind != 2) planes.push_back({&m, "m"}), planes.push_back({&v, "v"});   // SGD keeps no moments
  for (auto& [t, name] : planes) {
    if (t != &p) check_f32(*t, name);
    TORCH_CHECK(t->is_contiguous(), "fused_optimizer: ", name, " must be contiguous");
    check_numel(*t, p.numel(), "fused_optimizer", name);
    check_vec(*t, "fused_optimizer", name);
  }
  if (shadow.has_value()) {
    check_bf16(*shadow, "shadow");
    TORCH_CHECK(shadow->is_contiguous(), "fused_optimizer: shadow must be contiguous");
    check_numel(*shadow, p.numel(), "fused_optimizer", "shadow");
    check_vec(*shadow, "fused_optimizer", "shadow", 8);
  }
  if (grad_mult.has_value()) check_f32(*grad_mult, "grad_mult");
  c10::cuda::CUDAGuard guard(p.device());
  pb::OptimHyper h;
  h.kind = kind, h.first_step = first_step ? 1 : 0;
  h.lr = float(lr), h.beta1 = float(beta1), h.beta2 = float(beta2), h.eps = float(eps), h.decay = float(decay), h.wd = float(wd);
  h.clip = std::isfinite(clip) ? float(clip) : std::numeric_limits<float>::infinity();
  h.step_size = float(step_size), h.inv_sqrt_bc2 = float(inv_sqrt_bc2);
  pb::fused_optimizer(p.data_ptr<float>(), g.data_ptr<float>(), kind != 2 ? m.data_ptr<float>() : nullptr, kind != 2 ? v.data_ptr<float>() : nullptr,
                      opt_ptr(shadow), p.numel(), h, opt_ptr<float>(grad_mult), stream_of(p));
}

// ---------------------------------------------------------------------------------- symmetric arena (CUDA IPC)
int64_t ipc_alloc(int64_t nbytes, int device) {
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  void* p = nullptr;
  CUDA_OK(cudaMalloc(&p, size_t(nbytes)));
  CUDA_OK(cudaMemset(p, 0, size_t(nbytes)));
  return reinterpret_cast<int64_t>(p);
}
py::bytes ipc_get_handle(int64_t ptr) {
  cudaIpcMemHandle_t h;
  CUDA_OK(cudaIpcGetMemHandle(&h, reinterpret_cast<void*>(ptr)));
  return py::bytes(reinterpret_cast<const char*>(&h), sizeof(h));
}
int64_t ipc_open_handle(const std::string& handle, int device) {
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  TORCH_CHECK(handle.size() == sizeof(cudaIpcMemHandle_t), "bad IPC handle size");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle.data(), sizeof(h));
  void* p = nullptr;
  CUDA_OK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  return reinterpret_cast<int64_t>(p);
}
void ipc_close(int64_t ptr) { CUDA_OK(cudaIpcCloseMemHandle(reinterpret_cast<void*>(ptr))); }
void ipc_free(int64_t ptr) { CUDA_OK(cudaFree(reinterpret_cast<void*>(ptr))); }
bool enable_peer_access(int device, int peer) {
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  int can = 0;
  CUDA_OK(cudaDeviceCanAccessPeer(&can, device, peer));
  if (!can) return false;
  cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) {
    cudaGetLastError();
    return true;
  }
  CUDA_OK(e);
  return true;
}
Tensor tensor_from_ptr(int64_t ptr, int64_t numel, const std::string& dtype, int device) {
  auto dt = dtype == "float32" ? at::kFloat : dtype == "bfloat16" ? at::kBFloat16 : dtype == "int32" ? at::kInt
          : dtype == "float64" ? at::kDouble : at::kByte;
  auto opts = torch::TensorOptions().dtype(dt).device(torch::kCUDA, device);
  return torch::from_blob(reinterpret_cast<void*>(ptr), {numel}, [](void*) {}, opts);
}

std::atomic<long long> g_comm_timeout_ms{120000};   // bound on every cross-GPU spin inside the NVLink kernels (0 = forever)

pb::CommCtl make_ctl(const std::vector<int64_t>& ctl_ptrs, int rank) {
  TORCH_CHECK(ctl_ptrs.size() >= 1 && ctl_ptrs.size() <= pb::MAX_PEERS, "1..8 peers supported");
  pb::CommCtl c{};
  c.n = int(ctl_ptrs.size());
  c.rank = rank;
  c.timeout_ns = static_cast<unsigned long long>(g_comm_timeout_ms.load()) * 1000000ull;
  for (int i = 0; i < c.n; ++i) c.ctl[i] = reinterpret_cast<uint32_t*>(ctl_ptrs[i]);
  return c;
}

void fed_round(const std::vector<int64_t>& ctl_ptrs, int rank, int device, int64_t epoch, const std::vector<int64_t>& acc_ptrs,
               const std::vector<int64_t>& xg_ptrs, const std::vector<int64_t>& xs_ptrs, int64_t m_ptr, int64_t v_ptr, int64_t lo, int64_t hi, int64_t total,
               int kind, double avg_scale, double lr, double mu, double eta, double beta1, double beta2, double tau, int64_t round_t,
               bool sign_compat, int64_t acc_mc, int64_t xg_mc, const c10::optional<Tensor>& seg_bounds, c10::optional<Tensor> seg_sums,
               double wsum, bool zero_seg_sums) {
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  pb::CommCtl c = make_ctl(ctl_ptrs, rank);
  pb::FedRoundArgs a{};
  for (int i = 0; i < c.n; ++i) {
    a.acc[i] = reinterpret_cast<const float*>(acc_ptrs[i]);
    a.xg[i] = reinterpret_cast<float*>(xg_ptrs[i]);
    a.xs[i] = xs_ptrs.empty() ? nullptr : reinterpret_cast<void*>(xs_ptrs[i]);
  }
  a.x = a.xg[rank];
  a.m = reinterpret_cast<float*>(m_ptr);
  a.v = reinterpret_cast<float*>(v_ptr);
  a.lo = lo, a.hi = hi, a.total = total, a.kind = kind, a.avg_scale = float(avg_scale), a.lr = float(lr), a.mu = float(mu);
  a.eta = float(eta), a.beta1 = float(beta1), a.beta2 = float(beta2), a.tau = float(tau);
  const double t = double(round_t < 1 ? 1 : round_t);
  a.inv_bc1 = float(1.0 / (1.0 - std::pow(beta1, t)));
  a.inv_bc2 = float(1.0 / (1.0 - std::pow(beta2, t)));
  a.sign = sign_compat ? 1.0f : -1.0f;
  a.acc_mc = reinterpret_cast<const float*>(acc_mc);   // NVLS multicast addresses (0 = P2P loops)
  a.xg_mc = reinterpret_cast<float*>(xg_mc);
  a.publish_wsum = wsum >= 0.0 ? 1 : 0;        // negative = the page was filled by set_wsum before (legacy callers)
  a.wsum = float(wsum >= 0.0 ? wsum : 0.0);
  a.zero_seg_sums = zero_seg_sums ? 1 : 0;
  {
    static const int walk = [] { const char* e = std::getenv("PB_ROUND_WALK"); return e ? std::atoi(e) : 0; }();
    a.walk = walk;
  }
  if (seg_bounds.has_value() && seg_sums.has_value()) {
    TORCH_CHECK(seg_bounds->is_cuda() && seg_bounds->scalar_type() == at::kLong && seg_bounds->is_contiguous() && seg_bounds->numel() >= 2,
                "seg_bounds must be a contiguous int64 device tensor with n_seg + 1 entries");
    a.n_seg = int(seg_bounds->numel()) - 1;
    TORCH_CHECK(seg_sums->is_cuda() && seg_sums->scalar_type() == at::kDouble && seg_sums->is_contiguous() && seg_sums->numel() == 5 * a.n_seg,
                "seg_sums must be a contiguous float64 device tensor [5, n_seg]");
    a.seg_bounds = reinterpret_cast<const long long*>(seg_bounds->data_ptr<int64_t>());
    a.seg_sums = seg_sums->data_ptr<double>();
  }
  pb::fed_round_launch(a, c, uint32_t(epoch), num_sms(), at::cuda::getCurrentCUDAStream(device).stream());
}
// ZeRO-3: accumulate the mean over ranks of slice `rank` of the unit's staging planes into `dst` (see comm.cu)
void zero3_reduce(const std::vector<int64_t>& ctl_ptrs, int rank, int device, int64_t epoch, const std::vector<int64_t>& stage_ptrs,
                  int64_t stage_mc, c10::optional<Tensor> dst, int64_t per) {
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  pb::CommCtl c = make_ctl(ctl_ptrs, rank);
  pb::ShardReduceArgs a{};
  TORCH_CHECK(per % 4 == 0 && per >= 0, "slice length must be a multiple of 4");
  if (per > 0) {
    TORCH_CHECK(dst.has_value() && dst->scalar_type() == at::kFloat && dst->numel() >= per && dst->is_contiguous(), "dst: fp32, >= per");
    TORCH_CHECK(int(stage_ptrs.size()) == c.n, "one staging plane per rank");
    for (int i = 0; i < c.n; ++i) a.stage[i] = reinterpret_cast<const float*>(stage_ptrs[i]);
    a.dst = dst->data_ptr<float>();
  }
  a.stage_mc = reinterpret_cast<const float*>(stage_mc);
  a.per = per;
  a.scale = 1.0f / float(c.n);
  pb::zero3_reduce_launch(a, c, uint32_t(epoch), num_sms(), at::cuda::getCurrentCUDAStream(device).stream());
}
// ZeRO-3 under amp_fp8: global amax exchange + E4M3 quantisation of this rank's pieces of every block weight matrix (see comm.cu)
void zero3_fp8_requant(const std::vector<int64_t>& ctl_ptrs, int rank, int device, int64_t epoch, const Tensor& w16, Tensor& w8,
                       const Tensor& pieces, Tensor& amax_local, const std::vector<int64_t>& amax_ptrs, Tensor& meta, const Tensor& roles) {
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  pb::CommCtl c = make_ctl(ctl_ptrs, rank);
  check_bf16(w16, "w16");
  check_f32(amax_local, "amax_local");
  check_f32(meta, "meta");
  check_cuda(pieces, "pieces");
  check_cuda(roles, "roles");
  TORCH_CHECK(is_byte(w8) && w8.numel() == w16.numel() && w8.is_contiguous() && w16.is_contiguous(), "w8: a 1-byte shard as long as w16");
  TORCH_CHECK(pieces.scalar_type() == at::kLong && pieces.dim() == 2 && pieces.size(1) == 3 && pieces.is_contiguous(),
              "pieces must be int64 [n,3] (shard offset, numel, weight slot) on the device");
  TORCH_CHECK(roles.scalar_type() == at::kInt && roles.dim() == 1 && roles.is_contiguous(), "roles must be int32 [n_weights]");
  TORCH_CHECK(amax_local.numel() == roles.numel() && amax_local.is_contiguous(), "amax_local: one fp32 per weight");
  TORCH_CHECK(meta.dim() == 2 && meta.size(0) == 3 && meta.is_contiguous(), "meta must be fp32 [3, n_roles]");
  TORCH_CHECK(int(amax_ptrs.size()) == c.n, "one amax plane per rank");
  pb::Zero3RequantArgs a{};
  a.w16 = w16.data_ptr(), a.w8 = static_cast<uint8_t*>(w8.data_ptr());
  a.pieces = reinterpret_cast<const long long*>(pieces.data_ptr<int64_t>()), a.n_pieces = int(pieces.size(0));
  a.n_w = int(roles.numel()), a.amax_local = amax_local.data_ptr<float>();
  for (int i = 0; i < c.n; ++i) a.amax[i] = reinterpret_cast<float*>(amax_ptrs[i]);
  a.meta = meta.data_ptr<float>(), a.n_roles = meta.size(1), a.roles = roles.data_ptr<int>();
  a.fmax = 448.0f;
  pb::zero3_fp8_requant_launch(a, c, uint32_t(epoch), num_sms(), at::cuda::getCurrentCUDAStream(device).stream());
}

// device-to-device copy between (possibly peer-mapped) raw addresses on the current stream: the copy engines pull a parameter
// slice from its owner over NVLink without occupying an SM
void memcpy_async(int64_t dst, int64_t src, int64_t nbytes, int device) {
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  cudaError_t e = cudaMemcpyAsync(reinterpret_cast<void*>(dst), reinterpret_cast<const void*>(src), size_t(nbytes), cudaMemcpyDefault,
                                  at::cuda::getCurrentCUDAStream(device).stream());
  TORCH_CHECK(e == cudaSuccess, "memcpy_async: ", cudaGetErrorString(e));
}

void ddp_allreduce(const std::vector<int64_t>& ctl_ptrs, int rank, int device, int64_t epoch, const std::vector<int64_t>& buf_ptrs, int64_t lo,
                   int64_t hi, c10::optional<Tensor> out_norm, int64_t buf_mc) {
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  pb::CommCtl c = make_ctl(ctl_ptrs, rank);
  pb::AllReduceArgs a{};
  for (int i = 0; i < c.n; ++i) a.buf[i] = reinterpret_cast<float*>(buf_ptrs[i]);
  a.lo = lo, a.hi = hi;
  a.buf_mc = reinterpret_cast<float*>(buf_mc);
  pb::ddp_allreduce_launch(a, c, uint32_t(epoch), opt_ptr<float>(out_norm), num_sms(), at::cuda::getCurrentCUDAStream(device).stream());
}
void ddp_zero_step(const std::vector<int64_t>& ctl_ptrs, int rank, int device, int64_t epoch, const std::vector<int64_t>& grad_ptrs,
                   const std::vector<int64_t>& param_ptrs, const std::vector<int64_t>& shadow_ptrs, Tensor m, Tensor v, int64_t lo, int64_t hi,
                   int64_t kind, bool first_step, double lr, double beta1, double beta2, double eps, double decay, double clip,
                   double step_size, double inv_sqrt_bc2, double max_norm, double grad_mult, c10::optional<Tensor> out_norm,
                   int64_t grads_mc, int64_t params_mc, int64_t shadow_mc, double wd) {
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  pb::CommCtl c = make_ctl(ctl_ptrs, rank);
  pb::ZeroStepArgs a{};
  for (int i = 0; i < c.n; ++i) {
    a.grads[i] = reinterpret_cast<float*>(grad_ptrs[i]);
    a.params[i] = reinterpret_cast<float*>(param_ptrs[i]);
    a.shadow[i] = shadow_ptrs.empty() ? nullptr : reinterpret_cast<void*>(shadow_ptrs[i]);
  }
  TORCH_CHECK(m.numel() == hi - lo && v.numel() == hi - lo, "ddp_zero_step: moment shards must have hi - lo elements");
  a.m = m.data_ptr<float>(), a.v = v.data_ptr<float>();
  a.lo = lo, a.hi = hi;
  a.h.kind = int(kind), a.h.first_step = first_step ? 1 : 0;
  a.h.lr = float(lr), a.h.beta1 = float(beta1), a.h.beta2 = float(beta2), a.h.eps = float(eps), a.h.decay = float(decay), a.h.wd = float(wd);
  a.h.clip = float(clip), a.h.step_size = float(step_size), a.h.inv_sqrt_bc2 = float(inv_sqrt_bc2);
  a.max_norm = float(max_norm), a.grad_mult = float(grad_mult);
  a.grads_mc = reinterpret_cast<const float*>(grads_mc);
  a.params_mc = reinterpret_cast<float*>(params_mc);
  a.shadow_mc = shadow_ptrs.empty() ? nullptr : reinterpret_cast<void*>(shadow_mc);
  pb::ddp_zero_step_launch(a, c, uint32_t(epoch), opt_ptr<float>(out_norm), num_sms(), at::cuda::getCurrentCUDAStream(device).stream());
}
void set_wsum(int64_t ctl_ptr, int device, double w, bool zero_sums) {
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  pb::set_wsum(reinterpret_cast<uint32_t*>(ctl_ptr), float(w), zero_sums, at::cuda::getCurrentCUDAStream(device).stream());
}

long long launch_count() { return pb::g_launches.load(); }
void reset_launch_count() { pb::g_launches = 0; }
void add_launch_count(long long n) { pb::g_launches += n; }  // launches replayed from a CUDA graph

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "photon_b200 sm_90a kernels (wgmma/TMA GEMM + attention, fused norm/loss/optimizer, NVLink collectives)";
  m.def("gemm", &gemm, py::arg("a"), py::arg("b"), py::arg("d"), py::arg("a_mn") = 0, py::arg("b_mn") = 0, py::arg("epi") = 0,
        py::arg("bias") = py::none(), py::arg("aux") = py::none(), py::arg("d2") = py::none(), py::arg("accumulate") = false,
        py::arg("alpha") = 1.0, py::arg("cluster") = 0, py::arg("aux2") = py::none());
  m.def("gemm_fp8", &gemm_fp8, py::arg("a"), py::arg("b"), py::arg("d"), py::arg("a_mn"), py::arg("b_mn"), py::arg("epi"), py::arg("a_fmt"),
        py::arg("b_fmt"), py::arg("meta"), py::arg("role_a"), py::arg("role_b"), py::arg("bias") = py::none(), py::arg("aux") = py::none(),
        py::arg("d2") = py::none(), py::arg("accumulate") = false, py::arg("alpha") = 1.0, py::arg("cluster") = 0,
        py::arg("d8") = py::none(), py::arg("role_out") = -1);
  m.def("layernorm_fwd_q8", &layernorm_fwd_q8);
  m.def("rmsnorm_fwd_q8", &rmsnorm_fwd_q8);
  m.def("mx_quantize", &mx_quantize, py::arg("x"), py::arg("rblk") = 0);
  m.def("gemm_mxfp8", &gemm_mxfp8, py::arg("a8"), py::arg("b8"), py::arg("d"), py::arg("sfa"), py::arg("sfb"), py::arg("bias") = py::none());
  m.def("colsum_quant", &colsum_quant, py::arg("dy"), py::arg("out_sum") = py::none(), py::arg("y8") = py::none(), py::arg("fmt") = 1,
        py::arg("meta") = py::none(), py::arg("role") = -1);
  m.def("fp8_quantize_segments", &fp8_quantize_segments);
  m.def("fp8_update_scales", &fp8_update_scales);
  m.def("attention_fwd", &attention_fwd, py::arg("qkv"), py::arg("out"), py::arg("lse"), py::arg("n_heads"), py::arg("scale"),
        py::arg("causal"), py::arg("alibi_slopes") = py::none(), py::arg("doc_start") = py::none(), py::arg("n_kv_heads") = -1,
        py::arg("window") = -1);
  m.def("attention_bwd", &attention_bwd, py::arg("qkv"), py::arg("out"), py::arg("dout"), py::arg("lse"), py::arg("dqkv"), py::arg("delta"),
        py::arg("n_heads"), py::arg("scale"), py::arg("causal"), py::arg("alibi_slopes") = py::none(), py::arg("doc_start") = py::none(),
        py::arg("doc_end") = py::none(), py::arg("n_kv_heads") = -1, py::arg("window") = -1);
  m.def("doc_bounds", &doc_bounds, py::arg("sequence_id"), py::arg("doc_start"), py::arg("doc_end"));
  m.def("rope", &rope, py::arg("qkv"), py::arg("cos"), py::arg("sin"), py::arg("n_heads"), py::arg("inverse"), py::arg("n_kv_heads") = -1);
  m.def("embed_fwd", &embed_fwd);
  m.def("skinny_gemm", &skinny_gemm, py::arg("x"), py::arg("w"), py::arg("y"), py::arg("bias") = py::none(), py::arg("residual") = py::none(),
        py::arg("epi") = 0);
  m.def("decode_attention", &decode_attention, py::arg("q"), py::arg("k_cache"), py::arg("v_cache"), py::arg("pos"), py::arg("out"),
        py::arg("n_heads"), py::arg("scale"), py::arg("alibi_slopes") = py::none(), py::arg("n_kv_heads") = -1, py::arg("window") = -1);
  m.def("decode_append", &decode_append, py::arg("qkv"), py::arg("pos"), py::arg("k_cache"), py::arg("v_cache"), py::arg("cos") = py::none(),
        py::arg("sin") = py::none(), py::arg("n_heads") = 1, py::arg("slot") = py::none(), py::arg("n_kv_heads") = -1);
  m.def("cache_attention", &cache_attention, py::arg("qkv"), py::arg("k_cache"), py::arg("v_cache"), py::arg("tiles"), py::arg("out"),
        py::arg("n_heads"), py::arg("scale"), py::arg("alibi_slopes") = py::none(), py::arg("n_kv_heads") = -1, py::arg("window") = -1);
  m.def("embed_pos", &embed_pos, py::arg("ids"), py::arg("pos"), py::arg("wte"), py::arg("wpe"), py::arg("out"));
  m.def("argmax_advance", &argmax_advance, py::arg("logits"), py::arg("ids"), py::arg("pos") = py::none());
  m.def("embed_bwd", &embed_bwd);
  m.def("transpose_u8", &transpose_u8);
  m.def("layernorm_fwd", &layernorm_fwd);
  m.def("layernorm_bwd", &layernorm_bwd);
  m.def("rmsnorm_fwd", &rmsnorm_fwd);
  m.def("rmsnorm_bwd", &rmsnorm_bwd);
  m.def("col_sum", &col_sum);
  m.def("cross_entropy", &cross_entropy);
  m.def("flat_l2_norm", &flat_l2_norm);
  m.def("axpby", &axpby);
  m.def("cast_bf16", &cast_bf16);
  // wd: ADOPT's coupled weight decay (decouple: false), after the other scalars so that calls without it keep their meaning
  m.def("fused_optimizer", &fused_optimizer, py::arg("p"), py::arg("g"), py::arg("m"), py::arg("v"), py::arg("shadow"), py::arg("kind"),
        py::arg("first_step"), py::arg("lr"), py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("decay"), py::arg("clip"),
        py::arg("step_size"), py::arg("inv_sqrt_bc2"), py::arg("grad_mult"), py::arg("wd") = 0.0);
  m.def("ipc_alloc", &ipc_alloc);
  m.def("ipc_get_handle", &ipc_get_handle);
  m.def("ipc_open_handle", &ipc_open_handle);
  m.def("ipc_close", &ipc_close);
  m.def("ipc_free", &ipc_free);
  m.def("enable_peer_access", &enable_peer_access);
  m.def("tensor_from_ptr", &tensor_from_ptr);
  m.def("fed_round", &fed_round, py::arg("ctl_ptrs"), py::arg("rank"), py::arg("device"), py::arg("epoch"), py::arg("acc_ptrs"),
        py::arg("xg_ptrs"), py::arg("xs_ptrs"), py::arg("m_ptr"), py::arg("v_ptr"), py::arg("lo"), py::arg("hi"), py::arg("total"),
        py::arg("kind"), py::arg("avg_scale"), py::arg("lr"), py::arg("mu"), py::arg("eta"), py::arg("beta1"), py::arg("beta2"),
        py::arg("tau"), py::arg("round_t"), py::arg("sign_compat"), py::arg("acc_mc") = 0, py::arg("xg_mc") = 0,
        py::arg("seg_bounds") = py::none(), py::arg("seg_sums") = py::none(), py::arg("wsum") = -1.0, py::arg("zero_seg_sums") = false);
  m.def("set_comm_timeout_ms", [](long long ms) { g_comm_timeout_ms = ms < 0 ? 0 : ms; });
  m.def("comm_timeout_ms", []() { return g_comm_timeout_ms.load(); });
  m.def("ctl_status_word_offset", &pb::ctl_status_word_offset);
  m.def("ddp_allreduce", &ddp_allreduce, py::arg("ctl_ptrs"), py::arg("rank"), py::arg("device"), py::arg("epoch"), py::arg("buf_ptrs"),
        py::arg("lo"), py::arg("hi"), py::arg("out_norm") = py::none(), py::arg("buf_mc") = 0);
  m.def("zero3_reduce", &zero3_reduce, py::arg("ctl_ptrs"), py::arg("rank"), py::arg("device"), py::arg("epoch"), py::arg("stage_ptrs"),
        py::arg("stage_mc"), py::arg("dst"), py::arg("per"));
  m.def("zero3_fp8_requant", &zero3_fp8_requant, py::arg("ctl_ptrs"), py::arg("rank"), py::arg("device"), py::arg("epoch"), py::arg("w16"),
        py::arg("w8"), py::arg("pieces"), py::arg("amax_local"), py::arg("amax_ptrs"), py::arg("meta"), py::arg("roles"));
  m.def("memcpy_async", &memcpy_async);
  m.def("ddp_zero_step", &ddp_zero_step, py::arg("ctl_ptrs"), py::arg("rank"), py::arg("device"), py::arg("epoch"), py::arg("grad_ptrs"),
        py::arg("param_ptrs"), py::arg("shadow_ptrs"), py::arg("m"), py::arg("v"), py::arg("lo"), py::arg("hi"), py::arg("kind"),
        py::arg("first_step"), py::arg("lr"), py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("decay"), py::arg("clip"),
        py::arg("step_size"), py::arg("inv_sqrt_bc2"), py::arg("max_norm"), py::arg("grad_mult"), py::arg("out_norm") = py::none(),
        py::arg("grads_mc") = 0, py::arg("params_mc") = 0, py::arg("shadow_mc") = 0, py::arg("wd") = 0.0);
  m.def("set_wsum", &set_wsum);
  m.def("ctl_sums_word_offset", &pb::ctl_sums_word_offset);
  m.def("launch_count", &launch_count);
  m.def("reset_launch_count", &reset_launch_count);
  m.def("add_launch_count", &add_launch_count);
  m.attr("CTL_WORDS") = pb::CTL_WORDS;
  m.attr("EPI_BF16") = int(pb::EPI_BF16);
  m.attr("EPI_RESIDUAL") = int(pb::EPI_RESIDUAL);
  m.attr("EPI_GELU_DUAL") = int(pb::EPI_GELU_DUAL);
  m.attr("EPI_DGELU") = int(pb::EPI_DGELU);
  m.attr("EPI_F32") = int(pb::EPI_F32);
  m.attr("EPI_GELU_GRAD") = int(pb::EPI_GELU_GRAD);
  m.attr("EPI_MUL") = int(pb::EPI_MUL);
  m.attr("EPI_GELU_GRAD_Q8") = int(pb::EPI_GELU_GRAD_Q8);
  m.attr("EPI_SILU_GRAD") = int(pb::EPI_SILU_GRAD);
  m.attr("EPI_MUL2") = int(pb::EPI_MUL2);
  m.attr("SKINNY_PLAIN") = int(pb::SKINNY_PLAIN);
  m.attr("SKINNY_RESIDUAL") = int(pb::SKINNY_RESIDUAL);
  m.attr("SKINNY_GELU") = int(pb::SKINNY_GELU);
  m.attr("SKINNY_SILU") = int(pb::SKINNY_SILU);
  m.attr("SKINNY_MUL") = int(pb::SKINNY_MUL);
}
