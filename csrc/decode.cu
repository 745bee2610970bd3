// Kernels of the KV-cached greedy decoder for sm_90a (layouts and contracts in decode.h).
//
//   * skinny GEMM  Y[M,N] = X[M,K] W[N,K]^T for M <= 64 rows: a decode step is bound by streaming the weights, so the
//     weight rows fill the wgmma M side (m64) and the few activation rows are the N side (n8 / n16 / n32 / n64, "swap AB").
//     One producer thread streams 64 x 64 weight tiles and the matching activation tile by TMA through a 6-stage mbarrier
//     ring; one warpgroup issues the wgmmas. Every CTA owns 64 output columns and one K range; when the column tiles alone
//     cannot fill the GPU, K is split and the fp32 partials are summed in split order by a second kernel (no float atomics,
//     so the result does not depend on scheduling).
//   * decode attention: one query per (sequence, head) against the cache, split over 256-key chunks (flash-decoding); one CTA
//     serves the query heads of one kv head (grouped-query attention), so each cached row it loads is scored / weighed for
//     all of them; the chunk results (unnormalised o, running max, sum) of every query head are combined in chunk order.
//   * cache attention (scoring): tiles of up to 64 consecutive query rows of one cache slot against the slot's keys on wgmma,
//     with the causal mask at each row's own position.
//   * append (RoPE at each row's own position + cache write into the row's slot), embedding at per-row positions, argmax +
//     position advance.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <stdexcept>
#include <string>

#include "decode.h"
#include "gemm_tcgen05.h"
#include "launch.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace pb {

namespace {

constexpr float LOG2E = 1.4426950408889634f;

// ------------------------------------------------------------------------------------------- skinny GEMM
constexpr int SK_BN = 64;                  // weight rows (output columns) per CTA = wgmma M
constexpr int SK_BK = 64;                  // K elements per stage: 128 bytes per row, one 128B-swizzle atom row
constexpr int SK_STAGES = 6;
constexpr int SK_W_STAGE = SK_BN * 128;    // 8 KiB
constexpr int SK_THREADS = 160;            // warps 0-3: MMA + epilogue (one warpgroup); warp 4: TMA producer

template <int NB>
constexpr int sk_smem_bytes() { return SK_STAGES * (SK_W_STAGE + NB * 128) + 2 * SK_STAGES * 8 + 1024; }

struct SkParams {
  const float* bias;
  const __nv_bfloat16* R;
  long long ldr;
  __nv_bfloat16* Y;
  long long ldy;
  float* part;          // [splits, M, N] fp32 when splits > 1
  int M, N, K, kb_per_split, splits;
};

template <int EPI>
__device__ __forceinline__ float sk_finish(float v, const SkParams& p, int m, int n) {
  if (p.bias) v += __ldg(p.bias + n);
  if (EPI == SKINNY_RESIDUAL) v += __bfloat162float(p.R[(long long)m * p.ldr + n]);
  if (EPI == SKINNY_GELU) v = gelu_exact(v);
  if (EPI == SKINNY_SILU) v *= silu_sigmoid(v);
  if (EPI == SKINNY_MUL) v *= __bfloat162float(p.R[(long long)m * p.ldr + n]);
  return v;
}

template <int NB>
__device__ __forceinline__ void sk_mma(float (&acc)[NB / 2], uint64_t wd, uint64_t xd, uint32_t accum) {
  if constexpr (NB == 8) wgmma_bf16_ss_n8<0, 0>(acc, wd, xd, accum);
  else if constexpr (NB == 16) wgmma_bf16_ss_n16<0, 0>(acc, wd, xd, accum);
  else if constexpr (NB == 32) wgmma_bf16_ss_n32<0, 0>(acc, wd, xd, accum);
  else wgmma_bf16_ss_n64<0, 0>(acc, wd, xd, accum);
}

template <int NB, int EPI>
__global__ void __launch_bounds__(SK_THREADS)
skinny_gemm_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX, const SkParams p) {
  constexpr int X_STAGE = NB * 128;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sW = smem;
  uint8_t* sX = sW + SK_STAGES * SK_W_STAGE;
  uint64_t* full = reinterpret_cast<uint64_t*>(sX + SK_STAGES * X_STAGE);
  uint64_t* empty = full + SK_STAGES;

  const int n_blk = blockIdx.x, sp = blockIdx.y;
  const int num_kb = (p.K + SK_BK - 1) / SK_BK;
  const int kb0 = sp * p.kb_per_split, kb1 = min(num_kb, kb0 + p.kb_per_split);
  if (threadIdx.x == 0) {
    for (int s = 0; s < SK_STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4);   // one arrival per MMA warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (threadIdx.x >= 128) {
    // ------------------------------------------------------------ TMA producer (one thread)
    if (threadIdx.x == 128) {
      prefetch_tmap(&tmW);
      prefetch_tmap(&tmX);
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&empty[stage], phase ^ 1);
        mbar_expect_tx(&full[stage], SK_W_STAGE + X_STAGE);
        tma_load_2d(sW + stage * SK_W_STAGE, &tmW, &full[stage], kb * SK_BK, n_blk * SK_BN);
        tma_load_2d(sX + stage * X_STAGE, &tmX, &full[stage], kb * SK_BK, 0);   // rows >= M arrive as zeros
        if (++stage == SK_STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------- MMA warpgroup: D[64 weight rows, NB activation rows]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc[NB / 2];
#pragma unroll
  for (int i = 0; i < NB / 2; ++i) acc[i] = 0.f;
  int stage = 0, prev = -1;
  uint32_t phase = 0;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&full[stage], phase);
    const uint64_t wd = desc_sw128(sW + stage * SK_W_STAGE, 16);
    const uint64_t xd = desc_sw128(sX + stage * X_STAGE, 16);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) sk_mma<NB>(acc, desc_add(wd, k * 32), desc_add(xd, k * 32), (kb > kb0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();   // the previous stage's MMAs retired: release its shared memory
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
    prev = stage;
    if (++stage == SK_STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
  // accumulator (m64nNB): acc[4j + e] = weight row 16*warp + lane/4 + 8*(e/2), activation row 8j + 2*(lane%4) + e%2
#pragma unroll
  for (int j = 0; j < NB / 8; ++j) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int n = n_blk * SK_BN + warp * 16 + (lane >> 2) + 8 * (e >> 1);
      const int m = 8 * j + 2 * (lane & 3) + (e & 1);
      if (m >= p.M || n >= p.N) continue;
      const float v = acc[4 * j + e];
      if (p.splits > 1) p.part[((long long)sp * p.M + m) * p.N + n] = v;
      else p.Y[(long long)m * p.ldy + n] = __float2bfloat16_rn(sk_finish<EPI>(v, p, m, n));
    }
  }
}

// the split partials of one output element, summed in split order, then the epilogue
template <int EPI>
__global__ void __launch_bounds__(256) skinny_reduce_kernel(const SkParams p) {
  const long long total = (long long)p.M * p.N, plane = total;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int m = int(i / p.N), n = int(i % p.N);
    float v = 0.f;
    for (int s = 0; s < p.splits; ++s) v += p.part[s * plane + i];
    p.Y[(long long)m * p.ldy + n] = __float2bfloat16_rn(sk_finish<EPI>(v, p, m, n));
  }
}

template <int NB, int EPI>
void skinny_launch_inst(const CUtensorMap& tw, const CUtensorMap& tx, const SkParams& p, int tiles, cudaStream_t st) {
  auto kern = skinny_gemm_kernel<NB, EPI>;
  opt_in_smem(kern, sk_smem_bytes<NB>());
  kern<<<dim3(tiles, p.splits), SK_THREADS, sk_smem_bytes<NB>(), st>>>(tw, tx, p);
  launched("skinny gemm");
  if (p.splits > 1) {
    const long long total = (long long)p.M * p.N;
    const int blocks = int(std::min<long long>((total + 255) / 256, 132 * 8));
    skinny_reduce_kernel<EPI><<<blocks, 256, 0, st>>>(p);
    launched("skinny gemm split reduce");
  }
}

template <int EPI>
void skinny_launch_nb(const CUtensorMap& tw, const SkinnyArgs& a, const SkParams& p, int tiles, cudaStream_t st) {
  const int nb = a.M <= 8 ? 8 : a.M <= 16 ? 16 : a.M <= 32 ? 32 : 64;
  // activation tile: all M rows (box of nb rows; rows past M are filled with zeros by the TMA unit)
  const CUtensorMap tx = make_tmap_2d(a.X, 2, false, a.K, a.M, a.ldx * 2, SK_BK, nb);
  if (nb == 8) skinny_launch_inst<8, EPI>(tw, tx, p, tiles, st);
  else if (nb == 16) skinny_launch_inst<16, EPI>(tw, tx, p, tiles, st);
  else if (nb == 32) skinny_launch_inst<32, EPI>(tw, tx, p, tiles, st);
  else skinny_launch_inst<64, EPI>(tw, tx, p, tiles, st);
}

// ------------------------------------------------------------------------------------------- decode attention
constexpr int DA_CHUNK = 256;   // keys per CTA
constexpr int DA_THREADS = 128;

__device__ __forceinline__ float da_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffff, v, o);
  return v;
}

// One CTA = one (chunk, kv head, sequence). The G = H / HKV query heads of the kv head are taken NG at a time: each pass loads
// the chunk's key rows once and scores them against the pass's NG queries, then its value rows once for the NG weighted sums
// (G <= NG: every cached row of the chunk is read once). Per query head the arithmetic is that of one head alone.
// WIN: sliding window, the query sees keys lo .. pos[b] with lo = max(0, pos[b] - window); chunks wholly below lo return at
// once, and the chunk holding lo masks the keys below it.
template <int DH, bool ALIBI, int NG, bool WIN>
__global__ void __launch_bounds__(DA_THREADS)
decode_attn_kernel(const __nv_bfloat16* __restrict__ q, long long ldq, const __nv_bfloat16* __restrict__ kc,
                   const __nv_bfloat16* __restrict__ vc, const int* __restrict__ pos, float* __restrict__ po, float* __restrict__ pml,
                   int H, int HKV, int s_max, int n_split, float sc, const float* __restrict__ slopes, int window) {
  __shared__ float qs[NG][DH];
  __shared__ float ps[NG][DA_CHUNK];
  __shared__ float red[2][NG][4];
  __shared__ float os[4][NG][DH];
  const int s = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int len = pos[b] + 1;
  const int j0 = s * DA_CHUNK, j1 = min(len, j0 + DA_CHUNK);
  if (j0 >= j1) return;   // chunk past the sequence: the combine kernel reads only the chunks below pos[b] + 1
  const int lo = WIN ? max(0, pos[b] - window) : 0;
  if (WIN && j1 <= lo) return;   // chunk below the window: the combine kernel reads only the chunks from lo on
  const int G = H / HKV;
  const long long head = (long long)(b * HKV + hk) * s_max * DH;
  constexpr int PER = DH / 32;
  for (int h0 = hk * G; h0 < (hk + 1) * G; h0 += NG) {
    const int ng = min(NG, (hk + 1) * G - h0);   // query heads h0 .. h0 + ng - 1 in this pass
    for (int i = tid; i < NG * DH; i += DA_THREADS) {
      const int g = i / DH, e = i - g * DH;
      qs[g][e] = g < ng ? __bfloat162float(q[b * ldq + (h0 + g) * DH + e]) * sc : 0.f;
    }
    __syncthreads();
    float slope2[NG];
#pragma unroll
    for (int g = 0; g < NG; ++g) slope2[g] = ALIBI && g < ng ? slopes[h0 + g] * LOG2E : 0.f;
    // scores (log2 domain): one key per thread and pass, 16-byte loads of the key row, q broadcast from shared memory
    float mx[NG];
#pragma unroll
    for (int g = 0; g < NG; ++g) mx[g] = -INFINITY;
    for (int jj = tid; jj < DA_CHUNK; jj += DA_THREADS) {
      const int j = j0 + jj;
      float x[NG];
#pragma unroll
      for (int g = 0; g < NG; ++g) x[g] = -INFINITY;
      if (j < j1 && (!WIN || j >= lo)) {
        const uint4* kr = reinterpret_cast<const uint4*>(kc + head + (long long)j * DH);
        float acc[NG];
#pragma unroll
        for (int g = 0; g < NG; ++g) acc[g] = 0.f;
        // one head: the whole row in flight; several: a 16-byte piece at a time (their queries' registers would spill)
#pragma unroll(NG == 1 ? DH / 8 : 1)
        for (int c = 0; c < DH / 8; ++c) {
          const uint4 u = kr[c];
          const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            const float2 f = unpack_bf16(w[t]);
#pragma unroll
            for (int g = 0; g < NG; ++g) {
              acc[g] = fmaf(qs[g][c * 8 + 2 * t], f.x, acc[g]);
              acc[g] = fmaf(qs[g][c * 8 + 2 * t + 1], f.y, acc[g]);
            }
          }
        }
#pragma unroll
        for (int g = 0; g < NG; ++g) {
          x[g] = acc[g];
          if (ALIBI) x[g] = fmaf(slope2[g], float(j - (len - 1)), x[g]);   // slope * (key - query)
        }
      }
#pragma unroll
      for (int g = 0; g < NG; ++g) {
        ps[g][jj] = x[g];
        mx[g] = fmaxf(mx[g], x[g]);
      }
    }
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      mx[g] = warp_max_f(mx[g]);
      if (lane == 0) red[0][g][warp] = mx[g];
    }
    __syncthreads();
    float m[NG], l[NG];
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      m[g] = fmaxf(fmaxf(red[0][g][0], red[0][g][1]), fmaxf(red[0][g][2], red[0][g][3]));
      l[g] = 0.f;
    }
    for (int jj = tid; jj < DA_CHUNK; jj += DA_THREADS) {
#pragma unroll
      for (int g = 0; g < NG; ++g) {
        const float pv = (j0 + jj < j1 && (!WIN || j0 + jj >= lo)) ? exp2f(ps[g][jj] - m[g]) : 0.f;
        ps[g][jj] = pv;
        l[g] += pv;
      }
    }
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      l[g] = da_warp_sum(l[g]);
      if (lane == 0) red[1][g][warp] = l[g];
    }
    __syncthreads();
    // P.V: warp w takes keys w, w+4, ...; each lane owns DH/32 consecutive output dims (coalesced value rows)
    float o[NG][PER];
#pragma unroll
    for (int g = 0; g < NG; ++g)
#pragma unroll
      for (int i = 0; i < PER; ++i) o[g][i] = 0.f;
    for (int jj = (WIN ? max(lo - j0, 0) : 0) + warp; jj < j1 - j0; jj += 4) {
      const __nv_bfloat16* vr = vc + head + (long long)(j0 + jj) * DH + lane * PER;
      float f[PER];
      if constexpr (PER == 2) {
        const float2 f0 = unpack_bf16(*reinterpret_cast<const uint32_t*>(vr));
        f[0] = f0.x, f[1] = f0.y;
      } else {
        const uint2 u = *reinterpret_cast<const uint2*>(vr);
        const float2 f0 = unpack_bf16(u.x), f1 = unpack_bf16(u.y);
        f[0] = f0.x, f[1] = f0.y, f[2] = f1.x, f[3] = f1.y;
      }
#pragma unroll
      for (int g = 0; g < NG; ++g) {
        const float pv = ps[g][jj];
#pragma unroll
        for (int i = 0; i < PER; ++i) o[g][i] = fmaf(pv, f[i], o[g][i]);
      }
    }
#pragma unroll
    for (int g = 0; g < NG; ++g)
#pragma unroll
      for (int i = 0; i < PER; ++i) os[warp][g][lane * PER + i] = o[g][i];
    __syncthreads();
    for (int i = tid; i < ng * DH; i += DA_THREADS) {
      const int g = i / DH, e = i - g * DH;
      const long long slot = (long long)(b * H + h0 + g) * n_split + s;
      po[slot * DH + e] = ((os[0][g][e] + os[1][g][e]) + os[2][g][e]) + os[3][g][e];
    }
    if (tid < ng) {
      const long long slot = (long long)(b * H + h0 + tid) * n_split + s;
      pml[2 * slot] = fmaxf(fmaxf(red[0][tid][0], red[0][tid][1]), fmaxf(red[0][tid][2], red[0][tid][3]));
      pml[2 * slot + 1] = ((red[1][tid][0] + red[1][tid][1]) + red[1][tid][2]) + red[1][tid][3];
    }
    __syncthreads();   // the next pass reuses the shared buffers
  }
}

template <int DH, bool WIN>
__global__ void __launch_bounds__(DH) decode_combine_kernel(const float* __restrict__ po, const float* __restrict__ pml,
                                                            const int* __restrict__ pos, __nv_bfloat16* __restrict__ out, long long ldo,
                                                            int H, int n_split, int window) {
  const int h = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
  const int used = (pos[b] + 1 + DA_CHUNK - 1) / DA_CHUNK;
  const int first = WIN ? max(0, pos[b] - window) / DA_CHUNK : 0;   // the chunk holding the window's first key
  const long long slot0 = (long long)(b * H + h) * n_split;
  float M = -INFINITY;
  for (int s = first; s < used; ++s) M = fmaxf(M, pml[2 * (slot0 + s)]);
  float L = 0.f, o = 0.f;
  for (int s = first; s < used; ++s) {
    const float w = exp2f(pml[2 * (slot0 + s)] - M);
    L = fmaf(w, pml[2 * (slot0 + s) + 1], L);
    o = fmaf(w, po[(slot0 + s) * DH + t], o);
  }
  out[b * ldo + h * DH + t] = __float2bfloat16_rn(o / L);
}

// ------------------------------------------------------------------------------------------- cache attention
// One CTA = one (tile, head): up to 64 query rows of one cache slot, at consecutive positions, against that slot's keys.
// Warps 0-3 (one warpgroup) own the 64 rows: S = Q K^T on wgmma (both operands in shared memory, K-major), online softmax in
// registers (log2 domain), O += P V with P as the register A operand and V read MN-major as the cache stores it. Warp 4 is
// the TMA producer: Q once from the fused qkv, then 128-key K / V tiles of the head's kv head through a 2-stage ring from the
// cache viewed as [B_max * HKV * S_max, dh] rows. Every row is reduced by one thread quad in a fixed order: no atomics, bitwise repeatable.
constexpr int CA_BQ = 64, CA_BKV = 128;
constexpr int CA_THREADS = 160;

template <int DH>
struct CaCfg {
  static constexpr int CH = DH / 64;                // 64-column (128-byte) swizzle chunks per row
  static constexpr int Q_BYTES = CA_BQ * 128 * CH;  // [64 x DH] bf16: CH chunks of 8 KiB
  static constexpr int KV_BYTES = CA_BKV * 128 * CH;  // [128 x DH] bf16: CH chunks of 16 KiB
  static constexpr int SMEM = Q_BYTES + 4 * KV_BYTES + 9 * 8 + 1024;   // Q, K[2], V[2], barriers, 1 KiB alignment slack
  static_assert(SMEM <= 232448, "smem budget");
};

// WIN: sliding window, the row at position p sees keys max(0, p - window) .. p; the key-tile walk starts at the tile holding
// the first row's first key.
template <int DH, bool ALIBI, bool WIN>
__global__ void __launch_bounds__(CA_THREADS)
cache_attn_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                  const int4* __restrict__ tiles, __nv_bfloat16* __restrict__ out, long long ldo, long long n_q, int H, int HKV, int s_max,
                  float sc,
                  const float* __restrict__ slopes, int window) {
  using C = CaCfg<DH>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + C::Q_BYTES;        // [2]
  uint8_t* sV = sK + 2 * C::KV_BYTES;   // [2]
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sV + 2 * C::KV_BYTES);
  uint64_t* k_full = q_full + 1;        // [2]
  uint64_t* k_empty = q_full + 3;       // [2]
  uint64_t* v_full = q_full + 5;        // [2]
  uint64_t* v_empty = q_full + 7;       // [2]

  const int4 tile = tiles[blockIdx.x];  // (slot, first_row, n_rows, first_pos)
  const int h = blockIdx.y;
  const int n_kv = (tile.w + tile.z - 1) / CA_BKV + 1;   // key tiles up to the last row's position
  const int j0 = WIN ? max(0, tile.w - window) / CA_BKV : 0;
  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&k_empty[s], 4);   // one arrival per MMA warp
      mbar_init(&v_full[s], 1);
      mbar_init(&v_empty[s], 4);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (threadIdx.x >= 128) {
    // ------------------------------------------------------------ TMA producer (one thread)
    if (threadIdx.x == 128) {
      prefetch_tmap(&tmQ);
      prefetch_tmap(&tmK);
      prefetch_tmap(&tmV);
      const int kv_row0 = (tile.x * HKV + h / (H / HKV)) * s_max;
      mbar_expect_tx(q_full, C::Q_BYTES);   // rows past the last qkv row arrive as zeros
#pragma unroll
      for (int c = 0; c < C::CH; ++c) tma_load_2d(sQ + c * 8192, &tmQ, q_full, h * DH + c * 64, tile.y);
      for (int j = j0; j < n_kv; ++j) {
        const int st = (j - j0) & 1;
        const uint32_t ph = (((j - j0) >> 1) & 1) ^ 1;
        mbar_wait(&k_empty[st], ph);
        mbar_expect_tx(&k_full[st], C::KV_BYTES);
#pragma unroll
        for (int c = 0; c < C::CH; ++c) tma_load_2d(sK + st * C::KV_BYTES + c * 16384, &tmK, &k_full[st], c * 64, kv_row0 + j * CA_BKV);
        mbar_wait(&v_empty[st], ph);
        mbar_expect_tx(&v_full[st], C::KV_BYTES);
#pragma unroll
        for (int c = 0; c < C::CH; ++c) tma_load_2d(sV + st * C::KV_BYTES + c * 16384, &tmV, &v_full[st], c * 64, kv_row0 + j * CA_BKV);
      }
    }
    return;
  }

  // -------------------------------------------------------------- MMA warpgroup: 64 query rows x 128 keys per step
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t4 = lane & 3;
  const int r0 = warp * 16 + (lane >> 2);   // this thread's tile rows r0, r0 + 8 (accumulator layout of m64nN)
  const float slope2 = ALIBI ? slopes[h] * LOG2E : 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
  float s[64];
  mbar_wait(q_full, 0);
  for (int j = j0; j < n_kv; ++j) {
    const int st = (j - j0) & 1;
    const uint32_t ph = ((j - j0) >> 1) & 1;
    mbar_wait(&k_full[st], ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DH / 16; ++kk) {
      const int c = kk >> 2, off = (kk & 3) * 32;
      wgmma_bf16_ss_n128<0, 0>(s, desc_add(desc_sw128(sQ + c * 8192, 16), off),
                               desc_add(desc_sw128(sK + st * C::KV_BYTES + c * 16384, 16), off), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    __syncwarp();
    if (lane == 0) mbar_arrive(&k_empty[st]);
    // row r (position first_pos + r) sees keys 0 .. first_pos + r; key 0 is always visible, so m is finite after tile 0.
    // WIN: keys from first_pos + r - window on; a row can meet a tile with none of them (guarded below)
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j8 = 0; j8 < 16; ++j8) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hh = e >> 1;
        const int key = j * CA_BKV + 8 * j8 + 2 * t4 + (e & 1);
        const int qpos = tile.w + r0 + 8 * hh;
        float x = s[4 * j8 + e] * sc;
        if (ALIBI) x = fmaf(slope2, float(key - qpos), x);
        if (key > qpos) x = -INFINITY;
        if (WIN && key < qpos - window) x = -INFINITY;
        s[4 * j8 + e] = x;
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
      if constexpr (WIN) {
        // no visible key yet (m_new = -inf): subtracting 0 keeps exp2(-inf - -inf) = NaN out of alpha and P
        msub[hh] = m_new == -INFINITY ? 0.f : m_new;
        alpha[hh] = exp2f(m[hh] - msub[hh]);
      } else {
        alpha[hh] = exp2f(m[hh] - m_new);
      }
      m[hh] = m_new;
      l[hh] *= alpha[hh];
    }
    // P in bf16 as the A fragments of the 8 k-steps of P V (accumulator columns 16k .. 16k+15 = k-step k)
    uint32_t pa[8][4];
#pragma unroll
    for (int kc = 0; kc < 8; ++kc) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float p0 = exp2f(s[8 * kc + 2 * q] - (WIN ? msub[q & 1] : m[q & 1]));
        const float p1 = exp2f(s[8 * kc + 2 * q + 1] - (WIN ? msub[q & 1] : m[q & 1]));
        l[q & 1] += p0 + p1;
        pa[kc][q] = pack_bf16(p0, p1);
      }
    }
#pragma unroll
    for (int i = 0; i < DH / 8; ++i) {
      o[4 * i] *= alpha[0], o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1], o[4 * i + 3] *= alpha[1];
    }
    mbar_wait(&v_full[st], ph);
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < 8; ++kc) {
      const uint64_t vd = desc_add(desc_sw128(sV + st * C::KV_BYTES, 16384), kc * 2048);
      if constexpr (DH == 64) wgmma_bf16_rs_n64<1>(o, pa[kc], vd, 1u);
      else wgmma_bf16_rs_n128<1>(o, pa[kc], vd, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&v_empty[st]);
  }
  // only the rows of the tile are written
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int r = r0 + 8 * hh;
    l[hh] += __shfl_xor_sync(0xffffffff, l[hh], 1);
    l[hh] += __shfl_xor_sync(0xffffffff, l[hh], 2);
    if (r >= tile.z || tile.y + r >= n_q) continue;
    const float inv_l = 1.0f / l[hh];
    __nv_bfloat16* orow = out + (long long)(tile.y + r) * ldo + h * DH;
#pragma unroll
    for (int i = 0; i < DH / 8; ++i)
      *reinterpret_cast<uint32_t*>(orow + 8 * i + 2 * t4) = pack_bf16(o[4 * i + 2 * hh] * inv_l, o[4 * i + 2 * hh + 1] * inv_l);
  }
}

// ------------------------------------------------------------------------------------------- append / embed / argmax
__global__ void __launch_bounds__(128) decode_append_kernel(__nv_bfloat16* __restrict__ qkv, long long ld, const int* __restrict__ pos,
                                                            const int* __restrict__ slot, __nv_bfloat16* __restrict__ kc,
                                                            __nv_bfloat16* __restrict__ vc, const float* __restrict__ cosT,
                                                            const float* __restrict__ sinT, int H, int HKV, int dh, int s_max) {
  const int b = blockIdx.x, p = pos[b];
  const int sb = slot ? slot[b] : b;   // the cache slot this row writes
  const int d = H * dh, kvd = HKV * dh, half = dh / 2, groups = half / 8, vec = dh / 8;
  __nv_bfloat16* row = qkv + b * ld;
  const long long cache_row = ((long long)sb * HKV) * s_max + p;   // + h * s_max: row of kv head h
  if (cosT != nullptr) {
    // rotate-half RoPE at position p, the arithmetic of rope_kernel: the H q heads in place, the HKV k heads (which follow
    // them in the row) straight into the cache
    for (int i = threadIdx.x; i < (H + HKV) * groups; i += blockDim.x) {
      const int g = i % groups, h = i / groups;
      __nv_bfloat16* src = row + h * dh + g * 8;
      const uint4 a = *reinterpret_cast<const uint4*>(src);
      const uint4 bb = *reinterpret_cast<const uint4*>(src + half);
      const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {bb.x, bb.y, bb.z, bb.w};
      uint32_t oa[4], ob[4];
      const float* c = cosT + (long long)p * half + g * 8;
      const float* sn = sinT + (long long)p * half + g * 8;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 x1 = unpack_bf16(aw[k]), x2 = unpack_bf16(bw[k]);
        const float c0 = c[2 * k], c1 = c[2 * k + 1], s0 = sn[2 * k], s1 = sn[2 * k + 1];
        oa[k] = pack_bf16(x1.x * c0 - x2.x * s0, x1.y * c1 - x2.y * s1);
        ob[k] = pack_bf16(x2.x * c0 + x1.x * s0, x2.y * c1 + x1.y * s1);
      }
      __nv_bfloat16* dst = h < H ? src : kc + (cache_row + (long long)(h - H) * s_max) * dh + g * 8;
      *reinterpret_cast<uint4*>(dst) = make_uint4(oa[0], oa[1], oa[2], oa[3]);
      *reinterpret_cast<uint4*>(dst + half) = make_uint4(ob[0], ob[1], ob[2], ob[3]);
    }
  } else {
    for (int i = threadIdx.x; i < HKV * vec; i += blockDim.x) {
      const int h = i / vec, c = i % vec;
      *reinterpret_cast<uint4*>(kc + (cache_row + (long long)h * s_max) * dh + c * 8) =
          *reinterpret_cast<const uint4*>(row + d + h * dh + c * 8);
    }
  }
  for (int i = threadIdx.x; i < HKV * vec; i += blockDim.x) {
    const int h = i / vec, c = i % vec;
    *reinterpret_cast<uint4*>(vc + (cache_row + (long long)h * s_max) * dh + c * 8) =
        *reinterpret_cast<const uint4*>(row + d + kvd + h * dh + c * 8);
  }
}

__global__ void __launch_bounds__(128) embed_pos_kernel(const int* __restrict__ ids, const int* __restrict__ pos,
                                                        const __nv_bfloat16* __restrict__ wte, const __nv_bfloat16* __restrict__ wpe,
                                                        __nv_bfloat16* __restrict__ out, int d, int V) {
  const int b = blockIdx.x;
  int id = ids[b];
  id = id < 0 ? 0 : (id >= V ? V - 1 : id);
  const uint4* a = reinterpret_cast<const uint4*>(wte + (long long)id * d);
  const uint4* e = wpe ? reinterpret_cast<const uint4*>(wpe + (long long)pos[b] * d) : nullptr;
  uint4* o = reinterpret_cast<uint4*>(out + (long long)b * d);
  for (int i = threadIdx.x; i < d / 8; i += blockDim.x) {
    uint4 u = a[i];
    if (e) {
      const uint4 w = e[i];
      const uint32_t x[4] = {u.x, u.y, u.z, u.w}, y[4] = {w.x, w.y, w.z, w.w};
      uint32_t r[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = unpack_bf16(x[k]), g = unpack_bf16(y[k]);
        r[k] = pack_bf16(f.x + g.x, f.y + g.y);
      }
      u = make_uint4(r[0], r[1], r[2], r[3]);
    }
    o[i] = u;
  }
}

__device__ __forceinline__ void argmax_pick(float& best, int& idx, float ob, int oi) {
  if (ob > best || (ob == best && oi < idx)) best = ob, idx = oi;
}

__global__ void __launch_bounds__(1024) argmax_advance_kernel(const __nv_bfloat16* __restrict__ logits, long long ldl, int V,
                                                              int* __restrict__ ids, int* __restrict__ pos) {
  __shared__ float sb[32];
  __shared__ int si[32];
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float best = -INFINITY;
  int idx = 0x7fffffff;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    const float x = __bfloat162float(logits[b * ldl + v]);
    if (x > best) best = x, idx = v;   // ascending v: the first maximum of this thread's slice
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) argmax_pick(best, idx, __shfl_xor_sync(0xffffffff, best, o), __shfl_xor_sync(0xffffffff, idx, o));
  if (lane == 0) sb[warp] = best, si[warp] = idx;
  __syncthreads();
  if (warp == 0) {
    const int nw = blockDim.x >> 5;
    best = lane < nw ? sb[lane] : -INFINITY;
    idx = lane < nw ? si[lane] : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) argmax_pick(best, idx, __shfl_xor_sync(0xffffffff, best, o), __shfl_xor_sync(0xffffffff, idx, o));
    if (lane == 0) {
      ids[b] = idx == 0x7fffffff ? 0 : idx;
      if (pos) pos[b] += 1;
    }
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------- host
int skinny_gemm_splits(int M, int N, int K, int num_sms) {
  (void)M;
  const int tiles = (N + SK_BN - 1) / SK_BN;
  const int num_kb = (K + SK_BK - 1) / SK_BK;
  // aim for two resident CTAs per SM, keep >= 2 k-blocks per split
  int s = (2 * num_sms + tiles - 1) / tiles;
  const int max_s = num_kb / 2 > 1 ? num_kb / 2 : 1;
  if (s > max_s) s = max_s;
  if (s < 1) s = 1;
  const int per = (num_kb + s - 1) / s;
  return (num_kb + per - 1) / per;   // no empty tail split
}

void skinny_gemm_launch(const SkinnyArgs& a, float* partials, cudaStream_t st) {
  const int splits = skinny_gemm_splits(a.M, a.N, a.K, a.num_sms);
  if (splits > 1 && !partials) throw std::runtime_error("photon_b200 skinny gemm: split-K needs the fp32 partial buffer");
  SkParams p{};
  p.bias = a.bias;
  p.R = reinterpret_cast<const __nv_bfloat16*>(a.R), p.ldr = a.ldr;
  p.Y = reinterpret_cast<__nv_bfloat16*>(a.Y), p.ldy = a.ldy;
  p.part = partials;
  p.M = a.M, p.N = a.N, p.K = a.K, p.splits = splits;
  const int num_kb = (a.K + SK_BK - 1) / SK_BK;
  p.kb_per_split = (num_kb + splits - 1) / splits;
  const int tiles = (a.N + SK_BN - 1) / SK_BN;
  const CUtensorMap tw = make_tmap_2d(a.W, 2, false, a.K, a.N, a.ldw * 2, SK_BK, SK_BN);
  if (a.epi == SKINNY_PLAIN) skinny_launch_nb<SKINNY_PLAIN>(tw, a, p, tiles, st);
  else if (a.epi == SKINNY_RESIDUAL) skinny_launch_nb<SKINNY_RESIDUAL>(tw, a, p, tiles, st);
  else if (a.epi == SKINNY_GELU) skinny_launch_nb<SKINNY_GELU>(tw, a, p, tiles, st);
  else if (a.epi == SKINNY_SILU) skinny_launch_nb<SKINNY_SILU>(tw, a, p, tiles, st);
  else if (a.epi == SKINNY_MUL) skinny_launch_nb<SKINNY_MUL>(tw, a, p, tiles, st);
  else throw std::runtime_error("photon_b200 skinny gemm: unknown epilogue");
}

int decode_attention_splits(int s_max) { return (s_max + DA_CHUNK - 1) / DA_CHUNK; }

void decode_attention_launch(const void* q, long long ldq, const void* kc, const void* vc, const int* pos, void* out, long long ldo,
                             float* partial_o, float* partial_ml, int B, int H, int Hkv, int dh, int s_max, float scale,
                             const float* alibi_slopes, cudaStream_t st, int window) {
  if (B < 1) return;
  const int n_split = decode_attention_splits(s_max);
  const dim3 grid(n_split, Hkv, B);
  const int G = H / Hkv;
  const auto* qq = (const __nv_bfloat16*)q;
  const auto* kk = (const __nv_bfloat16*)kc;
  const auto* vv = (const __nv_bfloat16*)vc;
  const float sc = scale * LOG2E;
  with_bools([&](auto alibi, auto wide, auto win) {
    constexpr int D = wide ? 128 : 64;
    // the G query heads of a kv head are scored NG at a time
    const auto attn = [&](auto NG) {
      decode_attn_kernel<D, alibi, NG, win><<<grid, DA_THREADS, 0, st>>>(qq, ldq, kk, vv, pos, partial_o, partial_ml, H, Hkv, s_max, n_split,
                                                                        sc, alibi_slopes, window);
    };
    if (G == 1) attn(std::integral_constant<int, 1>{});
    else if (G == 2) attn(std::integral_constant<int, 2>{});
    else if (G <= 4) attn(std::integral_constant<int, 4>{});
    else attn(std::integral_constant<int, 8>{});
    launched("decode attention");
    decode_combine_kernel<D, win><<<dim3(H, B), D, 0, st>>>(partial_o, partial_ml, pos, (__nv_bfloat16*)out, ldo, H, n_split, window);
    launched("decode attention combine");
  }, alibi_slopes != nullptr, dh == 128, window >= 0 && window < s_max - 1);   // a wider window sees every cached key
}

void decode_append_launch(void* qkv, long long ldqkv, const int* pos, void* kc, void* vc, const float* cosT, const float* sinT, int B,
                          int H, int Hkv, int dh, int s_max, const int* slot, cudaStream_t st) {
  if (B < 1) return;
  if (dh % 16) throw std::runtime_error("photon_b200 decode append: d_head must be a multiple of 16");
  decode_append_kernel<<<B, 128, 0, st>>>((__nv_bfloat16*)qkv, ldqkv, pos, slot, (__nv_bfloat16*)kc, (__nv_bfloat16*)vc, cosT, sinT, H,
                                          Hkv, dh, s_max);
  launched("decode append");
}

void cache_attention_launch(const void* qkv, long long ldq, long long n_q, const void* kc, const void* vc, const int* tiles, int n_tiles,
                            void* out, long long ldo, int B_max, int H, int Hkv, int dh, int s_max, float scale,
                            const float* alibi_slopes, cudaStream_t st, int window) {
  if (n_tiles < 1 || n_q < 1) return;
  const long long kv_rows = (long long)B_max * Hkv * s_max;
  if (kv_rows >= (1LL << 31)) throw std::runtime_error("photon_b200 cache attention: the cache has more than 2^31 rows per layer");
  const CUtensorMap tq = make_tmap_2d(qkv, 2, false, uint64_t(H + 2 * Hkv) * dh, uint64_t(n_q), uint64_t(ldq) * 2, 64, CA_BQ);
  const CUtensorMap tk = make_tmap_2d(kc, 2, false, dh, kv_rows, uint64_t(dh) * 2, 64, CA_BKV);
  const CUtensorMap tv = make_tmap_2d(vc, 2, false, dh, kv_rows, uint64_t(dh) * 2, 64, CA_BKV);
  const dim3 grid(n_tiles, H);
  const auto* tt = reinterpret_cast<const int4*>(tiles);
  const float sc = scale * LOG2E;
  with_bools([&](auto alibi, auto wide, auto win) {
    constexpr int D = wide ? 128 : 64;
    auto kern = cache_attn_kernel<D, alibi, win>;
    opt_in_smem(kern, CaCfg<D>::SMEM);
    kern<<<grid, CA_THREADS, CaCfg<D>::SMEM, st>>>(tq, tk, tv, tt, (__nv_bfloat16*)out, ldo, n_q, H, Hkv, s_max, sc, alibi_slopes, window);
  }, alibi_slopes != nullptr, dh == 128, window >= 0 && window < s_max - 1);   // a wider window sees every cached key
  launched("cache attention");
}

void embed_pos_launch(const int* ids, const int* pos, const void* wte, const void* wpe, void* out, int B, int d, int V, cudaStream_t st) {
  if (B < 1) return;
  embed_pos_kernel<<<B, 128, 0, st>>>(ids, pos, (const __nv_bfloat16*)wte, (const __nv_bfloat16*)wpe, (__nv_bfloat16*)out, d, V);
  launched("embed_pos");
}

void argmax_advance_launch(const void* logits, long long ldl, int B, int V, int* ids, int* pos, cudaStream_t st) {
  if (B < 1) return;
  argmax_advance_kernel<<<B, 1024, 0, st>>>((const __nv_bfloat16*)logits, ldl, V, ids, pos);
  launched("argmax");
}

}  // namespace pb
