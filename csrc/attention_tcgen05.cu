// Causal flash attention for sm_90a on wgmma tensor cores, accumulators in registers.
//
// The fused QKV projection output is [B*S, (H + 2*HKV)*DH]: H query heads, then HKV key heads, then HKV value heads. With
// grouped-query attention (HKV < H) query head h uses kv head h / G, G = H / HKV; HKV = H is multi-head attention.
//
// Forward (attn_fwd_kernel<DH>): one CTA = one (batch, query head, 128-query tile), three warpgroups.
//   warpgroup 0 : TMA producer (one thread) — Q once, then a 2-stage ring of K / V tiles of the head's kv head straight out of
//                 the fused QKV buffer (no head split / transpose copies); gives its registers away (setmaxnreg)
//   warpgroups 1, 2: 64 query rows each — S = Q K^T (wgmma, both operands from shared memory, K-major), online softmax in
//                 registers (log2 domain, quad shuffles for the row max), O += P V with P taken from REGISTERS as the A operand
//                 (the S accumulator layout converts to the A fragment layout in place) and V consumed MN-major as stored.
//
// Backward (attn_bwd_kernel<DH>): one CTA = one (batch, kv head, 128-key tile) holding K_j, V_j in shared memory; warpgroups 1, 2
// own 64 key rows each and walk the query steps (128 rows at d_head 64, 64 at d_head 128; causal: those that see the key
// tile) of each of the G query heads of the group in turn, so dK / dV of the whole group accumulate in registers (no
// atomics). The producer brings each step's Q, dO and their lse / delta rows. S^T = K Q^T and dP^T = V dO^T (shared-memory
// operands), P^T and dS^T in registers, dV += P^T dO and dK += dS^T Q with the register A operand; dS^T is also written to a
// double-buffered shared-memory tile, where it reads as an MN-major dS for dQ = dS K (each warpgroup one 64 x 64 block); each
// warp's dQ rows leave through shared memory and a TMA reduce-add into an fp32 accumulator that a last kernel converts to bf16.
//
// Replaces flash-attn 2.x (mma.sync/cp.async) the reference calls through llm-foundry (SURVEY §2.5 K4).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <type_traits>

#include "attention_tcgen05.h"
#include "gemm_tcgen05.h"
#include "launch.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace pb {

namespace {

constexpr int BQ = 128, BKV = 128;
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

// ======================================================================================= forward
template <int DH>
struct FwdCfg {
  static constexpr int CH = DH / 64;              // 64-column (128-byte) swizzle chunks per tile
  static constexpr int TILE = 128 * 128 * CH;     // bytes of one [128 x DH] bf16 tile
  static constexpr int SMEM = TILE * 5 + 256 + 1024;   // Q, K[2], V[2], barriers
  static_assert(SMEM <= 232448, "smem budget");
};

template <int DH>
__device__ __forceinline__ void wgmma_pv(float (&o)[DH / 2], const uint32_t (&a)[4], uint64_t db) {
  if constexpr (DH == 64) wgmma_bf16_rs_n64<1>(o, a, db, 1u);
  else wgmma_bf16_rs_n128<1>(o, a, db, 1u);
}

// BOUND: every query row q has a lower bound lo(q) on its keys, and query q sees key k iff lo(q) <= k <= q (causal only).
// lo(q) = max(doc_start[q], q - window): doc_start [B*S] (optional, the document mask) holds the first row of each row's
// document (rows of one sequence); window is the sliding-window size (>= S when off). lo is non-decreasing along a sequence,
// so key tiles that end before lo of the tile's first row are never loaded.
// GQA: HKV < H (grouped-query attention); false compiles the multi-head kernel (HKV == H, the kv head is the query head).
template <int DH, bool ALIBI, bool BOUND, bool GQA>
__global__ void __launch_bounds__(384, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQKV, __nv_bfloat16* __restrict__ out, float* __restrict__ lse, int S, int H,
                float scale, int causal, const float* __restrict__ alibi_slopes, const int* __restrict__ doc_start, int HKV, int window) {
  using C = FwdCfg<DH>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + C::TILE;                     // [2]
  uint8_t* sV = sK + 2 * C::TILE;                 // [2]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * C::TILE);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;                    // [2]
  uint64_t* k_empty = bars + 3;                   // [2]
  uint64_t* v_full = bars + 5;                    // [2]
  uint64_t* v_empty = bars + 7;                   // [2]

  const int n_qt = S / BQ;
  const int qt = n_qt - 1 - int(blockIdx.x);      // heaviest (causal) tiles first
  const int bh = blockIdx.y, b = bh / H, h = bh - b * H;
  const int d_model = H * DH;
  // the kv head's K / V columns; the multi-head instances keep the multi-head expressions (and so the multi-head code)
  const int k_col = GQA ? d_model + h / (H / HKV) * DH : d_model + h * DH;
  const int v_col = GQA ? k_col + HKV * DH : 2 * d_model + h * DH;
  const int n_kv = causal ? qt + 1 : S / BKV;
  const auto lo_of = [&](int q) { return max(doc_start ? doc_start[b * S + q] : 0, q - window); };
  const int j0 = BOUND ? lo_of(qt * BQ) / BKV : 0;   // first key tile any row of this query tile sees
  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmQKV);
    mbar_init(q_full, 1);
    for (int s2 = 0; s2 < 2; ++s2) {
      mbar_init(&k_full[s2], 1);
      mbar_init(&k_empty[s2], 8);   // one arrival per consumer warp
      mbar_init(&v_full[s2], 1);
      mbar_init(&v_empty[s2], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      mbar_expect_tx(q_full, C::TILE);
#pragma unroll
      for (int c = 0; c < C::CH; ++c) tma_load_2d(sQ + c * 16384, &tmQKV, q_full, h * DH + c * 64, b * S + qt * BQ);
      for (int j = j0; j < n_kv; ++j) {
        const int n = j - j0, st = n & 1;
        const uint32_t ph = ((n >> 1) & 1) ^ 1;
        mbar_wait(&k_empty[st], ph);
        mbar_expect_tx(&k_full[st], C::TILE);
#pragma unroll
        for (int c = 0; c < C::CH; ++c)
          tma_load_2d(sK + st * C::TILE + c * 16384, &tmQKV, &k_full[st], k_col + c * 64, b * S + j * BKV);
        mbar_wait(&v_empty[st], ph);
        mbar_expect_tx(&v_full[st], C::TILE);
#pragma unroll
        for (int c = 0; c < C::CH; ++c)
          tma_load_2d(sV + st * C::TILE + c * 16384, &tmQKV, &v_full[st], v_col + c * 64, b * S + j * BKV);
      }
    }
    return;
  }
  // -------------------------------------------------------------------- softmax / MMA warpgroups (64 query rows each)
  regs_alloc<232>();
  const int cw = wg - 1;
  const int wq = (threadIdx.x >> 5) & 3;
  const int g = lane >> 2, t4 = lane & 3;
  const int qrow0 = qt * BQ + cw * 64 + wq * 16 + g;   // this thread's query rows: qrow0, qrow0 + 8
  const float sc = scale * LOG2E;
  const float slope2 = ALIBI ? alibi_slopes[h] * LOG2E : 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
  float sacc[64];
  // BOUND: first visible key of this thread's two rows, and of the tile's last row (the largest): key tiles starting at or
  // after the latter need no mask below the diagonal
  int dstart[2] = {0, 0}, dstart_last = 0;
  if (BOUND) {
    dstart[0] = lo_of(qrow0), dstart[1] = lo_of(qrow0 + 8);
    dstart_last = lo_of(qt * BQ + BQ - 1);
  }
  mbar_wait(q_full, 0);
  for (int j = j0; j < n_kv; ++j) {
    const int n = j - j0, st = n & 1;
    const uint32_t ph = (n >> 1) & 1;
    mbar_wait(&k_full[st], ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DH / 16; ++kk) {
      const int c = kk >> 2, off = (kk & 3) * 32;
      const uint64_t qd = desc_add(desc_sw128(sQ + c * 16384 + cw * 8192, 16), off);
      const uint64_t kd = desc_add(desc_sw128(sK + st * C::TILE + c * 16384, 16), off);
      wgmma_bf16_ss_n128<0, 0>(sacc, qd, kd, kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sacc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&k_empty[st]);
    // scaled (log2-domain) scores, causal mask on the diagonal tile, ALiBi bias slope * (key - query)
    const bool diag = causal && j == qt;
    const bool dmask = BOUND && j * BKV < dstart_last;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j8 = 0; j8 < 16; ++j8) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hh = e >> 1;
        const int key = j * BKV + 8 * j8 + 2 * t4 + (e & 1);
        const int q = qrow0 + 8 * hh;
        float x = sacc[4 * j8 + e] * sc;
        if (ALIBI) x = fmaf(slope2, float(key - q), x);
        if (diag && key > q) x = -INFINITY;
        if (dmask && key < dstart[hh]) x = -INFINITY;
        sacc[4 * j8 + e] = x;
        mx[hh] = fmaxf(mx[hh], x);
      }
    }
    float alpha[2];
    [[maybe_unused]] float msub[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffff, mx[hh], 1));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffff, mx[hh], 2));
      const float m_new = fmaxf(m[hh], mx[hh]);
      if constexpr (BOUND) {
        // a row can meet a tile with no visible key before its first one (m_new = -inf); subtracting 0 there keeps
        // exp2(-inf - -inf) = NaN out of alpha and P (both become 0, and l, O are still 0)
        msub[hh] = m_new == -INFINITY ? 0.f : m_new;
        alpha[hh] = exp2f(m[hh] - msub[hh]);
      } else {
        alpha[hh] = exp2f(m[hh] - m_new);   // 0 on the first tile (m = -inf)
      }
      m[hh] = m_new;
      l[hh] *= alpha[hh];
    }
    uint32_t pa[8][4];
#pragma unroll
    for (int j8 = 0; j8 < 16; ++j8) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pv = exp2f(sacc[4 * j8 + e] - (BOUND ? msub[e >> 1] : m[e >> 1]));
        sacc[4 * j8 + e] = pv;
        l[e >> 1] += pv;
      }
    }
#pragma unroll
    for (int kc = 0; kc < 8; ++kc) {
      // accumulator columns 16 kc .. 16 kc + 15 are the A fragment of k-step kc
      pa[kc][0] = pack_bf16(sacc[8 * kc + 0], sacc[8 * kc + 1]);
      pa[kc][1] = pack_bf16(sacc[8 * kc + 2], sacc[8 * kc + 3]);
      pa[kc][2] = pack_bf16(sacc[8 * kc + 4], sacc[8 * kc + 5]);
      pa[kc][3] = pack_bf16(sacc[8 * kc + 6], sacc[8 * kc + 7]);
    }
#pragma unroll
    for (int i = 0; i < DH / 8; ++i) {
      o[4 * i] *= alpha[0], o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1], o[4 * i + 3] *= alpha[1];
    }
    mbar_wait(&v_full[st], ph);
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < 8; ++kc)
      wgmma_pv<DH>(o, pa[kc], desc_add(desc_sw128(sV + st * C::TILE, 16384), kc * 2048));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&v_empty[st]);
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l[hh] += __shfl_xor_sync(0xffffffff, l[hh], 1);
    l[hh] += __shfl_xor_sync(0xffffffff, l[hh], 2);
    const float inv_l = 1.0f / l[hh];
    const int q = qrow0 + 8 * hh;
    __nv_bfloat16* orow = out + (long long)(b * S + q) * d_model + h * DH;
#pragma unroll
    for (int i = 0; i < DH / 8; ++i)
      *reinterpret_cast<uint32_t*>(orow + 8 * i + 2 * t4) = pack_bf16(o[4 * i + 2 * hh] * inv_l, o[4 * i + 2 * hh + 1] * inv_l);
    if (t4 == 0) lse[((long long)b * H + h) * S + q] = m[hh] * LN2 + __logf(l[hh]);
  }
}

// ======================================================================================= backward
// delta[b,h,q] = sum_d dO * O   (row-wise; feeds dS = P * (dP - delta)).  One thread per 8 contiguous elements (16-byte
// loads), DH/8 adjacent lanes form one (row, head) group and reduce with shuffles; the delta store is scattered but tiny.
__global__ void __launch_bounds__(256) attn_bwd_delta_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ dout,
                                                              float* __restrict__ delta, int S, int H, int DH, long long rows) {
  const int gl = DH / 8;                                  // lanes per (row, head): 8 for d_head 64, 16 for 128
  const long long n8 = rows * H * gl;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(o) + i);
    const uint4 g = __ldg(reinterpret_cast<const uint4*>(dout) + i);
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, gw[4] = {g.x, g.y, g.z, g.w};
    float acc = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 fa = unpack_bf16(aw[t]), fg = unpack_bf16(gw[t]);
      acc += fa.x * fg.x + fa.y * fg.y;
    }
    for (int off = gl >> 1; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffff, acc, off);
    if ((i % gl) == 0) {
      const long long rh = i / gl, r = rh / H;
      const int h = int(rh - r * H);
      const long long bb = r / S, sq = r - bb * S;
      delta[(bb * H + h) * S + sq] = acc;
    }
  }
}

// dq_acc (fp32, [B*S, H*DH]) * scale -> bf16 into the q columns of dqkv (rows of width w)
__global__ void attn_bwd_dq_convert_kernel(const float* __restrict__ dq_acc, __nv_bfloat16* __restrict__ dqkv, long long rows, int d, int w,
                                           float scale) {
  const long long n4 = rows * d / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(dq_acc)[i];
    const long long e = i * 4, r = e / d, c = e % d;
    uint2 o;
    o.x = pack_bf16(v.x * scale, v.y * scale), o.y = pack_bf16(v.z * scale, v.w * scale);
    *reinterpret_cast<uint2*>(dqkv + r * w + c) = o;
  }
}

// d_head 64 walks 128-query steps: S^T and dP^T are m64n128 (64 + 64 fp32 per thread) next to dV and dK (32 + 32), inside the
// 240-register consumer budget (setmaxnreg 240 / 24). d_head 128 doubles dV and dK, so it keeps 64-query steps.
template <int DH>
struct BwdCfg {
  static constexpr int CH = DH / 64;                        // 64-column swizzle chunks per tile
  static constexpr int BQS = DH == 64 ? 128 : 64;           // query rows per step
  static constexpr int KT = 128 * 128 * CH;                 // [128 x DH] bf16 (K, V)
  static constexpr int QC = BQS * 128;                      // one 64-column chunk of a [BQS x DH] bf16 tile (Q, dO)
  static constexpr int QT = QC * CH;
  static constexpr int DS = 128 * BQS * 2;                  // dS^T: [128 keys][BQS queries] bf16, 64 queries per swizzle chunk
  static constexpr int DQW = 16 * 64 * 4;                   // one consumer warp's dQ staging: [16 rows][64 columns] fp32
  static constexpr int RS = 3 * BQS * 4;                    // the step's lse, delta (fp32) and doc_start (int) rows
  static constexpr int SMEM = 2 * KT + 4 * QT + 2 * DS + 8 * DQW + 2 * RS + 256 + 1024;
  static_assert(SMEM <= 232448, "smem budget");
};

template <int DH>
__device__ __forceinline__ void wgmma_acc_rs(float (&d)[DH / 2], const uint32_t (&a)[4], uint64_t db) {
  if constexpr (DH == 64) wgmma_bf16_rs_n64<1>(d, a, db, 1u);
  else wgmma_bf16_rs_n128<1>(d, a, db, 1u);
}

// S^T / dP^T of one step: [64 keys x N queries], both operands K-major
template <int N>
__device__ __forceinline__ void wgmma_ss_kmajor(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (N == 128) wgmma_bf16_ss_n128<0, 0>(d, da, db, scale_d);
  else wgmma_bf16_ss_n64<0, 0>(d, da, db, scale_d);
}

// BOUND: as in the forward, read from the key's side: key k is seen by queries k .. hi(k), hi(k) = min(doc_end[k], k + window),
// with doc_end [B*S] (present iff doc_start is) the last row of each row's document, so the query walk of a key tile stops at
// the step holding hi of its last key. GQA: as in the forward.
template <int DH, bool ALIBI, bool BOUND, bool GQA>
__global__ void __launch_bounds__(384, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmKV, const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmDO,
                const __grid_constant__ CUtensorMap tmDQ, const float* __restrict__ lse, const float* __restrict__ delta,
                __nv_bfloat16* __restrict__ dqkv, int S, int H, float scale, int causal, const float* __restrict__ alibi_slopes,
                const int* __restrict__ doc_start, const int* __restrict__ doc_end, int HKV, int window) {
  using C = BwdCfg<DH>;
  constexpr int BQS = C::BQS;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;
  uint8_t* sV = sK + C::KT;
  uint8_t* sQ = sV + C::KT;              // [2]
  uint8_t* sDO = sQ + 2 * C::QT;         // [2]
  uint8_t* sDS = sDO + 2 * C::QT;        // [2]
  uint8_t* sDQ = sDS + 2 * C::DS;        // [8 consumer warps]
  uint8_t* sRS = sDQ + 8 * C::DQW;       // [2] lse, delta, doc_start of the Q / dO stage's rows
  uint64_t* bars = reinterpret_cast<uint64_t*>(sRS + 2 * C::RS);
  uint64_t* kv_full = bars;
  uint64_t* q_full = bars + 1;           // [2] Q_i + dO_i + their row statistics
  uint64_t* q_empty = bars + 3;          // [2]

  const int jt = int(gridDim.x) - 1 - int(blockIdx.x);   // causal: small key tiles see the most query tiles - start them first
  const int hkv = GQA ? HKV : H;                          // the multi-head instances keep the multi-head expressions
  const int bk = blockIdx.y, b = bk / hkv, hk = bk - b * hkv;
  const int G = GQA ? H / hkv : 1, h0 = hk * G;           // query heads h0 .. h0 + G - 1 read this kv head
  const int d_model = H * DH;
  const int k_col = d_model + hk * DH, v_col = GQA ? k_col + HKV * DH : 2 * d_model + hk * DH;
  const int i0 = causal ? jt * (128 / BQS) : 0;            // query steps of BQS rows
  const int n_q = BOUND ? min(doc_end ? doc_end[b * S + jt * 128 + 127] : S - 1, jt * 128 + 127 + window) / BQS + 1 : S / BQS;
  const bool doc = BOUND && doc_start != nullptr;
  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmKV);
    prefetch_tmap(&tmQ);
    prefetch_tmap(&tmDO);
    prefetch_tmap(&tmDQ);
    mbar_init(kv_full, 1);
    for (int s2 = 0; s2 < 2; ++s2) {
      mbar_init(&q_full[s2], 1);
      mbar_init(&q_empty[s2], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    regs_dealloc<24>();
    if (threadIdx.x == 0) {
      mbar_expect_tx(kv_full, 2 * C::KT);
#pragma unroll
      for (int c = 0; c < C::CH; ++c) {
        tma_load_2d(sK + c * 16384, &tmKV, kv_full, k_col + c * 64, b * S + jt * 128);
        tma_load_2d(sV + c * 16384, &tmKV, kv_full, v_col + c * 64, b * S + jt * 128);
      }
      for (int h = h0; h < h0 + G; ++h) {
        for (int i = i0; i < n_q; ++i) {
          const int n = (h - h0) * (n_q - i0) + i - i0, st = n & 1;   // (query head, query step) items in walk order
          mbar_wait(&q_empty[st], ((n >> 1) & 1) ^ 1);
          mbar_expect_tx(&q_full[st], 2 * C::QT + (doc ? 3 : 2) * BQS * 4);
#pragma unroll
          for (int c = 0; c < C::CH; ++c) {
            tma_load_2d(sQ + st * C::QT + c * C::QC, &tmQ, &q_full[st], h * DH + c * 64, b * S + i * BQS);
            tma_load_2d(sDO + st * C::QT + c * C::QC, &tmDO, &q_full[st], h * DH + c * 64, b * S + i * BQS);
          }
          const long long row = ((long long)b * H + h) * S + i * BQS;
          uint8_t* rs_st = sRS + st * C::RS;
          bulk_load(rs_st, lse + row, BQS * 4, &q_full[st]);
          bulk_load(rs_st + BQS * 4, delta + row, BQS * 4, &q_full[st]);
          if (doc) bulk_load(rs_st + 2 * BQS * 4, doc_start + (long long)b * S + i * BQS, BQS * 4, &q_full[st]);
        }
      }
    }
    return;
  }
  regs_alloc<240>();
  const int cw = wg - 1;
  const int wq = (threadIdx.x >> 5) & 3;
  const int g = lane >> 2, t4 = lane & 3;
  const int kl0 = cw * 64 + wq * 16 + g;          // this thread's key rows inside the tile: kl0, kl0 + 8
  const int key0 = jt * 128 + kl0;
  const float sc = scale * LOG2E;
  // the multi-head instances read their head's slope here, where the multi-head kernel always has
  const float slope2_mh = ALIBI && !GQA ? alibi_slopes[h0] * LOG2E : 0.f;
  float dv[DH / 2], dk[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) dv[i] = 0.f, dk[i] = 0.f;
  mbar_wait(kv_full, 0);
  // the query steps of each query head of the group in turn (one head for the multi-head instances)
  for (int h = h0; h < h0 + G; ++h) {
    const float slope2 = !GQA ? slope2_mh : ALIBI ? alibi_slopes[h] * LOG2E : 0.f;
    for (int i = i0; i < n_q; ++i) {
      const int n = (h - h0) * (n_q - i0) + i - i0, st = n & 1;   // walk position, as in the producer
      const int q0 = i * BQS;
      uint8_t* q_st = sQ + st * C::QT;
      uint8_t* do_st = sDO + st * C::QT;
      uint8_t* ds_st = sDS + st * C::DS;
      float s[BQS / 2], dp[BQS / 2];
      mbar_wait(&q_full[st], (n >> 1) & 1);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < DH / 16; ++kk) {   // S^T = K Q^T
        const int c = kk >> 2, off = (kk & 3) * 32;
        wgmma_ss_kmajor<BQS>(s, desc_add(desc_sw128(sK + c * 16384 + cw * 8192, 16), off), desc_add(desc_sw128(q_st + c * C::QC, 16), off),
                             kk > 0 ? 1u : 0u);
      }
#pragma unroll
      for (int kk = 0; kk < DH / 16; ++kk) {   // dP^T = V dO^T
        const int c = kk >> 2, off = (kk & 3) * 32;
        wgmma_ss_kmajor<BQS>(dp, desc_add(desc_sw128(sV + c * 16384 + cw * 8192, 16), off), desc_add(desc_sw128(do_st + c * C::QC, 16), off),
                             kk > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(s);
      wgmma_fence_regs(dp);
      // P^T = exp(S^T * scale + alibi - lse[q]) (masked where query < key, which only the step overlapping the key tile has),
      // dS^T = P^T * (dP^T - delta[q])
      const bool diag = causal && i < i0 + 128 / BQS;   // the steps that overlap the key tile
      const uint32_t rs = smem_u32(sRS + st * C::RS) + 8 * t4;   // this thread's query columns in the staged rows
      uint32_t pa[BQS / 16][4], da[BQS / 16][4];
#pragma unroll
      for (int j8 = 0; j8 < BQS / 8; ++j8) {
        const int qa = q0 + 8 * j8 + 2 * t4;
        const float2 L = ld_shared_f32x2(rs + 32 * j8);
        const float2 D = ld_shared_f32x2(rs + BQS * 4 + 32 * j8);
        const int2 DS = doc ? ld_shared_s32x2(rs + 2 * BQS * 4 + 32 * j8) : make_int2(0, 0);
        float pv[4], dsv[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int q = qa + (e & 1), key = key0 + 8 * (e >> 1);
          float x = fmaf(s[4 * j8 + e], sc, -((e & 1) ? L.y : L.x) * LOG2E);
          if (ALIBI) x = fmaf(slope2, float(key - q), x);
          float pr = exp2f(x);
          if (diag && q < key) pr = 0.f;
          if (BOUND && max((e & 1) ? DS.y : DS.x, q - window) > key) pr = 0.f;
          pv[e] = pr;
          dsv[e] = pr * (dp[4 * j8 + e] - ((e & 1) ? D.y : D.x));
          // a masked query (another document, or past the key's window) may carry a non-finite delta (its own keys' fault):
          // keep it out of dK
          if (BOUND && pr == 0.f) dsv[e] = 0.f;
        }
        // accumulator columns 16 kc .. 16 kc + 15 (queries) are the A fragment of k-step kc
        const int kc = j8 >> 1, hi = (j8 & 1) * 2;
        pa[kc][hi] = pack_bf16(pv[0], pv[1]);
        pa[kc][hi + 1] = pack_bf16(pv[2], pv[3]);
        da[kc][hi] = pack_bf16(dsv[0], dsv[1]);
        da[kc][hi + 1] = pack_bf16(dsv[2], dsv[3]);
      }
      wgmma_fence();
#pragma unroll
      for (int kc = 0; kc < BQS / 16; ++kc) {   // dV += P^T dO, dK += dS^T Q (B operands MN-major: 16 query rows per k-step)
        wgmma_acc_rs<DH>(dv, pa[kc], desc_add(desc_sw128(do_st, C::QC), kc * 2048));
        wgmma_acc_rs<DH>(dk, da[kc], desc_add(desc_sw128(q_st, C::QC), kc * 2048));
      }
      wgmma_commit();
      // dS^T -> this step's buffer (row = key, 64 queries = 128 bytes per chunk, 128-byte swizzle)
#pragma unroll
      for (int j8 = 0; j8 < BQS / 8; ++j8) {
        const int kc = j8 >> 1, hi = (j8 & 1) * 2;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int kl = kl0 + 8 * hh;
          *reinterpret_cast<uint32_t*>(ds_st + (j8 >> 3) * 16384 + kl * 128 + (((j8 & 7) ^ (kl & 7)) << 4) + 4 * t4) = da[kc][hi + hh];
        }
      }
      fence_proxy_async_smem();
      // the dQ MMAs read both warpgroups' key rows of dS^T. The buffer was last read by the dQ MMAs two steps back, which each
      // warpgroup waited for before it reached the previous step's barrier, so this is the step's only cross-warpgroup barrier.
      named_bar_sync(1, 256);
      // dQ = dS K for this warpgroup's 64 x 64 block: A = dS (MN-major: queries contiguous), B = K (MN-major)
      float dq[32];
      wgmma_fence();
#pragma unroll
      for (int kc = 0; kc < 8; ++kc) {
        wgmma_bf16_ss_n64<1, 1>(dq, desc_add(desc_sw128(ds_st + (DH == 64 ? cw * 16384 : 0), 16384), kc * 2048),
                                desc_add(desc_sw128(sK + (DH == 128 ? cw * 16384 : 0), 16384), kc * 2048), kc > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();   // dV and dK are done with the Q / dO stage
      wgmma_fence_regs(dv);
      wgmma_fence_regs(dk);
      __syncwarp();
      if (lane == 0) mbar_arrive(&q_empty[st]);
      wgmma_wait<0>();
      wgmma_fence_regs(dq);
      // dQ -> this warp's staging -> one bulk reduce-add per 32-column box into dq_acc; only the staging's previous read by
      // the bulk copy is waited for, not its global write. The warp's tile is 16 rows of the warpgroup's 64 x 64 block (d_head
      // 64: its 64 queries of the step; d_head 128: its half of the head dimension), staged as two [16 rows][32 fp32] boxes in
      // the 128-byte swizzle of the reduce-add tensor map.
      uint8_t* sDQw = sDQ + (cw * 4 + wq) * C::DQW;
      if (lane == 0) tma_wait_read<0>();
      __syncwarp();
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int r = g + 8 * hh, unit = (2 * (j & 3) + (t4 >> 1)) ^ g;   // r & 7 == g
          *reinterpret_cast<float2*>(sDQw + (j >> 2) * 2048 + r * 128 + (unit << 4) + 8 * (t4 & 1)) =
              make_float2(dq[4 * j + 2 * hh], dq[4 * j + 2 * hh + 1]);
        }
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
        const int row = b * S + q0 + (DH == 64 ? cw * 64 : 0) + wq * 16, col = h * DH + (DH == 128 ? cw * 64 : 0);
        tma_reduce_add_2d(&tmDQ, sDQw, col, row);
        tma_reduce_add_2d(&tmDQ, sDQw + 2048, col + 32, row);
        tma_commit();
      }
    }
  }
  // dK (x scale), dV of the kv head (summed over its query heads) -> bf16 -> dqkv
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    __nv_bfloat16* krow = dqkv + (long long)(b * S + key0 + 8 * hh) * (GQA ? d_model + 2 * HKV * DH : 3 * d_model) + k_col;
    __nv_bfloat16* vrow = krow + (GQA ? HKV * DH : d_model);
#pragma unroll
    for (int j = 0; j < DH / 8; ++j) {
      *reinterpret_cast<uint32_t*>(krow + 8 * j + 2 * t4) = pack_bf16(dk[4 * j + 2 * hh] * scale, dk[4 * j + 2 * hh + 1] * scale);
      *reinterpret_cast<uint32_t*>(vrow + 8 * j + 2 * t4) = pack_bf16(dv[4 * j + 2 * hh], dv[4 * j + 2 * hh + 1]);
    }
  }
  if (lane == 0) tma_wait_read<0>();   // the staging stays in place until the last reduce-add has read it
}

// ======================================================================================= document bounds
// One CTA per sequence: documents are maximal runs of equal ids. Each thread takes a contiguous chunk of rows, finds the
// last document start and the first document end in it, and a block-wide max- / min-scan over the chunks carries them across.
constexpr int DOC_THREADS = 1024;
__global__ void __launch_bounds__(DOC_THREADS) doc_bounds_kernel(const long long* __restrict__ ids, int* __restrict__ doc_start,
                                                                 int* __restrict__ doc_end, int S) {
  const long long* row = ids + (long long)blockIdx.x * S;
  int* ds = doc_start + (long long)blockIdx.x * S;
  int* de = doc_end + (long long)blockIdx.x * S;
  const int per = (S + DOC_THREADS - 1) / DOC_THREADS;
  const int lo = min(S, int(threadIdx.x) * per), hi = min(S, lo + per);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auto starts = [&](int s) { return s == 0 || row[s] != row[s - 1]; };
  auto ends = [&](int s) { return s == S - 1 || row[s] != row[s + 1]; };
  int last_start = -1, first_end = S;   // none in this chunk
  for (int s = lo; s < hi; ++s)
    if (starts(s)) last_start = s;
  for (int s = hi - 1; s >= lo; --s)
    if (ends(s)) first_end = s;
  // inclusive scans inside the warp: max of starts from the left, min of ends from the right
  int inc_start = last_start, inc_end = first_end;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int a = __shfl_up_sync(0xffffffff, inc_start, o), z = __shfl_down_sync(0xffffffff, inc_end, o);
    if (lane >= o) inc_start = max(inc_start, a);
    if (lane + o < 32) inc_end = min(inc_end, z);
  }
  __shared__ int warp_start[DOC_THREADS / 32], warp_end[DOC_THREADS / 32];
  if (lane == 31) warp_start[warp] = inc_start;
  if (lane == 0) warp_end[warp] = inc_end;
  __syncthreads();
  // exclusive: what the chunks before (after) this one contribute
  int carry_start = __shfl_up_sync(0xffffffff, inc_start, 1), carry_end = __shfl_down_sync(0xffffffff, inc_end, 1);
  if (lane == 0) carry_start = -1;
  if (lane == 31) carry_end = S;
  for (int w = 0; w < warp; ++w) carry_start = max(carry_start, warp_start[w]);
  for (int w = warp + 1; w < DOC_THREADS / 32; ++w) carry_end = min(carry_end, warp_end[w]);
  for (int s = lo; s < hi; ++s) {
    if (starts(s)) carry_start = s;
    ds[s] = carry_start;
  }
  for (int s = hi - 1; s >= lo; --s) {
    if (ends(s)) carry_end = s;
    de[s] = carry_end;
  }
}

}  // namespace

// a window that leaves some query a key it cannot see (window < S - 1) runs the bounded instances; a wider one is plain
// causal attention and runs the causal instances. The kernels take the window as >= S when it is off.
static bool window_binds(int window, int S) { return window >= 0 && window < S - 1; }

void attention_fwd_launch(const void* qkv, void* out, float* lse, int B, int S, int H, int Hkv, int dh, float scale, bool causal,
                          cudaStream_t st, const float* alibi_slopes, const int* doc_start, int window) {
  if (S % 128) throw std::runtime_error("photon_b200 attention: sequence length must be a multiple of 128");
  if (dh != 64 && dh != 128) throw std::runtime_error("photon_b200 attention: d_head must be 64 or 128");
  if (window >= 0 && !causal) throw std::runtime_error("photon_b200 attention: a sliding window needs the causal mask");
  const bool win = window_binds(window, S);
  const uint64_t w = uint64_t(H + 2 * Hkv) * dh;   // fused qkv row width
  CUtensorMap tm = make_tmap_2d(qkv, 2, false, w, uint64_t(B) * S, w * 2, 64, 128);
  const dim3 grid(S / 128, B * H);
  with_bools([&](auto gqa, auto alibi, auto wide, auto doc) {
    constexpr int DHV = wide ? 128 : 64;
    auto kern = attn_fwd_kernel<DHV, alibi, doc, gqa>;
    opt_in_smem(kern, FwdCfg<DHV>::SMEM);
    kern<<<grid, 384, FwdCfg<DHV>::SMEM, st>>>(tm, (__nv_bfloat16*)out, lse, S, H, scale, causal ? 1 : 0, alibi_slopes, doc_start, Hkv,
                                               win ? window : S);
  }, Hkv != H, alibi_slopes != nullptr, dh == 128, doc_start != nullptr || win);
  launched("attention fwd");
}

void attention_bwd_launch(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv, float* delta, float* dq_acc,
                          int B, int S, int H, int Hkv, int dh, float scale, bool causal, int num_sms, cudaStream_t st, const float* alibi_slopes,
                          const int* doc_start, const int* doc_end, int window) {
  if (S % 128) throw std::runtime_error("photon_b200 attention: sequence length must be a multiple of 128");
  if (dh != 64 && dh != 128) throw std::runtime_error("photon_b200 attention backward: d_head must be 64 or 128");
  if (window >= 0 && !causal) throw std::runtime_error("photon_b200 attention backward: a sliding window needs the causal mask");
  const bool win = window_binds(window, S);
  const int sms = num_sms > 0 ? num_sms : 132;
  const int d = H * dh;
  const uint64_t w = uint64_t(H + 2 * Hkv) * dh;   // fused qkv row width
  const long long rows = (long long)B * S;
  // the kernel bulk-copies lse / delta / doc_start rows of 64 or 128 entries: 16-byte aligned base addresses keep them aligned
  for (const void* p : {(const void*)lse, (const void*)delta, (const void*)doc_start})
    if (reinterpret_cast<uintptr_t>(p) & 15) throw std::runtime_error("photon_b200 attention backward: lse, delta and doc_start must be 16-byte aligned");
  cudaMemsetAsync(dq_acc, 0, size_t(rows) * d * sizeof(float), st);
  {
    const long long n8 = rows * H * (dh / 8);
    const int blocks = int(std::min<long long>((n8 + 255) / 256, sms * 16));
    attn_bwd_delta_kernel<<<blocks, 256, 0, st>>>((const __nv_bfloat16*)out, (const __nv_bfloat16*)dout, delta, S, H, dh, rows);
    launched("attention bwd delta");
  }
  CUtensorMap tmKV = make_tmap_2d(qkv, 2, false, w, uint64_t(rows), w * 2, 64, 128);
  CUtensorMap tmDQ = make_tmap_2d(dq_acc, 4, true, uint64_t(d), uint64_t(rows), uint64_t(d) * 4, 32, 16);   // one warp's 16 x 32 box
  const dim3 grid(S / 128, B * Hkv);
  with_bools([&](auto gqa, auto alibi, auto wide, auto doc) {
    constexpr int DHV = wide ? 128 : 64;
    using C = BwdCfg<DHV>;
    CUtensorMap tmQ = make_tmap_2d(qkv, 2, false, w, uint64_t(rows), w * 2, 64, C::BQS);
    CUtensorMap tmDO = make_tmap_2d(dout, 2, false, uint64_t(d), uint64_t(rows), uint64_t(d) * 2, 64, C::BQS);
    auto kern = attn_bwd_kernel<DHV, alibi, doc, gqa>;
    opt_in_smem(kern, C::SMEM);
    kern<<<grid, 384, C::SMEM, st>>>(tmKV, tmQ, tmDO, tmDQ, lse, delta, (__nv_bfloat16*)dqkv, S, H, scale, causal ? 1 : 0, alibi_slopes,
                                     doc_start, doc_end, Hkv, win ? window : S);
  }, Hkv != H, alibi_slopes != nullptr, dh == 128, doc_start != nullptr || win);
  launched("attention bwd");
  attn_bwd_dq_convert_kernel<<<sms * 8, 256, 0, st>>>(dq_acc, (__nv_bfloat16*)dqkv, rows, d, int(w), scale);
  launched("attention bwd dq convert");
}

void doc_bounds_launch(const long long* sequence_id, int* doc_start, int* doc_end, int B, int S, cudaStream_t st) {
  doc_bounds_kernel<<<B, DOC_THREADS, 0, st>>>(sequence_id, doc_start, doc_end, S);
  launched("doc_bounds");
}

// ---------------------------------------------------------------------------------------------- RoPE
// In-place rotary embedding (rotate-half / GPT-NeoX convention) on the H q heads and the Hkv k heads of a fused qkv buffer
// [T, (H + 2*Hkv)*dh] bf16 (the k heads follow the q heads, so together they are H + Hkv consecutive heads of each row);
// cos / sin: fp32 [S, dh/2]. inverse = 1 applies the transposed rotation (gradients of q, k).
namespace {
__global__ void __launch_bounds__(256) rope_kernel(__nv_bfloat16* __restrict__ qkv, const float* __restrict__ cosT, const float* __restrict__ sinT,
                                                   long long T, int S, int H, int Hkv, int dh, int inverse) {
  const int half = dh / 2, groups = half / 8;                 // 8 pairs (16 bytes of each half) per thread
  const int nh = H + Hkv;                                     // rotated heads per row: q heads, then k heads
  const long long n = T * nh * groups;                        // (token, head, group)
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int g = int(i % groups);
    const long long r = i / groups;
    const int h = int(r % nh);
    const long long t = r / nh;
    const int pos = int(t % S);
    __nv_bfloat16* base = qkv + t * ((long long)(H + 2 * Hkv) * dh) + (long long)h * dh + g * 8;
    const uint4 a = *reinterpret_cast<const uint4*>(base);
    const uint4 b = *reinterpret_cast<const uint4*>(base + half);
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
    uint32_t oa[4], ob[4];
    const float* c = cosT + (long long)pos * half + g * 8;
    const float* sn = sinT + (long long)pos * half + g * 8;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 x1 = unpack_bf16(aw[k]), x2 = unpack_bf16(bw[k]);
      const float c0 = c[2 * k], c1 = c[2 * k + 1];
      const float s0 = inverse ? -sn[2 * k] : sn[2 * k], s1 = inverse ? -sn[2 * k + 1] : sn[2 * k + 1];
      oa[k] = pack_bf16(x1.x * c0 - x2.x * s0, x1.y * c1 - x2.y * s1);
      ob[k] = pack_bf16(x2.x * c0 + x1.x * s0, x2.y * c1 + x1.y * s1);
    }
    *reinterpret_cast<uint4*>(base) = make_uint4(oa[0], oa[1], oa[2], oa[3]);
    *reinterpret_cast<uint4*>(base + half) = make_uint4(ob[0], ob[1], ob[2], ob[3]);
  }
}
}  // namespace

void rope_launch(void* qkv, const float* cosT, const float* sinT, long long T, int S, int H, int Hkv, int dh, bool inverse,
                 cudaStream_t st) {
  if (dh % 16) throw std::runtime_error("photon_b200 rope: d_head must be a multiple of 16");
  const long long n = T * (H + Hkv) * (dh / 16);
  const int blocks = int(std::min<long long>((n + 255) / 256, 132 * 16));
  rope_kernel<<<blocks, 256, 0, st>>>((__nv_bfloat16*)qkv, cosT, sinT, T, S, H, Hkv, dh, inverse ? 1 : 0);
  launched("rope");
}

}  // namespace pb
