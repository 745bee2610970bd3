// Persistent, warp-specialised GEMM for sm_90a:  D[M,N] = A[M,K] * B[N,K]^T  (+ fused epilogue)
//
//   * operands staged global->shared by TMA (cp.async.bulk.tensor, 128B swizzle), 4-stage mbarrier ring filled by one
//     producer thread (its warpgroup hands its registers to the MMA warpgroups with setmaxnreg)
//   * two MMA warpgroups, 64 rows of the 128 x 256 tile each: wgmma.mma_async (bf16: m64n256k16, fp8: m64n256k32) with the
//     fp32 accumulators in registers; a stage is released as soon as the next stage's MMAs are issued (wait_group 1)
//   * epilogue: bias / residual / GELU / SiLU / dGELU / gating multipliers / fp8 re-quantisation in registers, then stmatrix
//     into a per-warpgroup 128B-swizzled staging buffer and TMA stores (cp.async.bulk.tensor) that drain while the next tile's
//     mainloop runs; fp32 outputs (weight gradients, split-K partials) go straight from registers, accumulated by red.global.add
//   * bf16 operands may be K-major ([rows,K] row-major) or MN-major ([K,rows] row-major) so forward, dgrad (B = W as stored)
//     and wgrad (A = dY^T, B = X^T as stored) need no transposes; wgmma reads 8-bit operands K-major only, so an MN-major fp8
//     operand is transposed into scratch first (transpose_u8)
//   * cluster 2: two CTAs on M-adjacent tiles share the B tile - each loads half of it and TMA multicasts it to both
//
// Replaces the cuBLASLt calls the reference reaches through torch (SURVEY §2.5 K3,K5-K8,K10).
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdlib>
#include <stdexcept>
#include <string>

#include "gemm_tcgen05.h"
#include "launch.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace pb {

namespace {

constexpr int BM = 128, BN = 256;
// A stage holds 128 BYTES of K per row for either operand type: 64 bf16 (4 k-steps of 16) or 128 fp8 (4 k-steps of 32),
// so the shared-memory plan, the TMA box bytes and the descriptor arithmetic are the same for both.
constexpr int ROW_BYTES = 128;
constexpr int A_STAGE = BM * ROW_BYTES;   // 16 KiB
constexpr int B_STAGE = BN * ROW_BYTES;   // 32 KiB
constexpr int STAGE_BYTES = A_STAGE + B_STAGE;
constexpr int STAGES = 4;
// epilogue staging: per MMA warpgroup two 8 KiB slots, each one TMA store box of 64 rows x 128 bytes
constexpr int EPI_SLOT = 64 * 128;
constexpr int EPI_WG_BYTES = 2 * EPI_SLOT;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 2 * EPI_WG_BYTES + 256 + 1024;
static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KiB dynamic shared memory of sm_90");
constexpr int NUM_THREADS = 384;   // warpgroup 0: TMA producer (one thread); warpgroups 1, 2: MMA + epilogue

struct Params {
  int M, N, K;
  int tiles_m, tiles_n, m_fastest;
  const float* bias;            // [N] fp32 or nullptr
  const __nv_bfloat16* aux;     // residual (EPI_RESIDUAL) or pre-activation z (EPI_DGELU) or multiplier (EPI_MUL, EPI_MUL2)
  long long ld_aux;             // row stride of aux, elements
  union {                       // (a union: the parameter block of the other epilogues keeps its size and offsets)
    float* d;                   // EPI_F32 output (the other outputs are written through their tensor maps)
    const __nv_bfloat16* aux2;  // EPI_MUL2: the second multiplier
  };
  long long ldd;                // row stride of d or aux2, elements
  int accumulate;               // EPI_F32: reduce-add into D instead of overwrite
  float alpha;                  // scale applied to the accumulator before the epilogue
  int splits, kb_per_split;     // split-K (EPI_F32 + accumulate): work item = (tile, k-range)
  // fp8 operands: element formats (0 = E4M3, 1 = E5M2) and the per-tensor de-scales, read from device memory
  // (delayed scaling keeps them on the device so the whole step stays CUDA-graph capturable)
  int a_fmt, b_fmt;
  const float* sinv_a;
  const float* sinv_b;
  // EPI_GELU_GRAD_Q8: the activation leaves as E4M3 (scaled by *out_scale, amax recorded) for the next fp8 GEMM
  const float* out_scale;
  float* out_amax;
};

__device__ __forceinline__ uint16_t pack_e4m3x2(float a, float b) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(b), "f"(a));   // first source -> upper byte
  return r;
}

// CL = 1: one CTA per 128x256 tile.
// CL = 2: a cluster of two CTAs computes two M-adjacent 128x256 tiles that share their B tile: each CTA loads 128 of the 256
//         B rows and multicasts them into both CTAs' shared memory, halving the L2 -> SM traffic of B. A stage may only be
//         refilled when the MMA warpgroups of BOTH CTAs released it, so every consumer warp arrives on both empty barriers.
//
// Outputs other than fp32 leave through TMA: tmD is D (bf16) or, for EPI_GELU_GRAD_Q8, the E4M3 output D8; tmD2 is D2. Their dims
// are the logical [M, N], so the TMA clips the M and N tails.
template <int A_MN, int B_MN, int EPI, int CL, int F8>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmD,
            const __grid_constant__ CUtensorMap tmD2, const Params p) {
  constexpr int BK = F8 ? 128 : 64;            // K elements per stage (128 bytes per row)
  constexpr int MNC = F8 ? 128 : 64;           // MN elements in one 128-byte row of an MN-major tile
  constexpr int CHUNK = BK * ROW_BYTES;        // bytes of one MN-major chunk: BK k-rows of 128 bytes
  constexpr bool TWO_OUT = EPI == EPI_GELU_DUAL || EPI == EPI_GELU_GRAD || EPI == EPI_GELU_GRAD_Q8 || EPI == EPI_SILU_GRAD ||
                          EPI == EPI_MUL2;
  constexpr bool AUX = EPI == EPI_RESIDUAL || EPI == EPI_DGELU || EPI == EPI_MUL || EPI == EPI_MUL2;
  static_assert(!F8 || (!A_MN && !B_MN), "8-bit wgmma operands are K-major");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = sA + STAGES * A_STAGE;
  uint8_t* sE = sB + STAGES * B_STAGE;         // epilogue staging, EPI_WG_BYTES per MMA warpgroup (1024-byte aligned)
  uint64_t* full = reinterpret_cast<uint64_t*>(sE + 2 * EPI_WG_BYTES);
  uint64_t* empty = full + STAGES;

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  const uint32_t crank = (CL > 1) ? cluster_ctarank() : 0;
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    if (EPI != EPI_F32) prefetch_tmap(&tmD);
    if (TWO_OUT) prefetch_tmap(&tmD2);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8 * CL);   // one arrival per MMA warp of every CTA that reads the stage
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (CL > 1) cluster_sync_all();   // peer barriers initialised before any multicast / remote arrive

  // work decomposition: units of CL M-adjacent tiles; every CTA of a cluster walks the same unit sequence
  const int tiles_mu = (p.tiles_m + CL - 1) / CL;
  const int num_tiles = tiles_mu * p.tiles_n;
  const int num_kb = (p.K + BK - 1) / BK;
  const int num_work = num_tiles * p.splits;
  const int w0 = blockIdx.x / CL, wstride = gridDim.x / CL;

  if (wg == 0) {
    // ======================= TMA producer (one thread) =======================
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int w = w0; w < num_work; w += wstride) {
        const int tile = w % num_tiles, sp = w / num_tiles;
        const int m_blk = (p.m_fastest ? tile % tiles_mu : tile / p.tiles_n) * CL + crank;
        const int n_blk = p.m_fastest ? tile / tiles_mu : tile % p.tiles_n;
        const int kb0 = sp * p.kb_per_split, kb1 = min(num_kb, kb0 + p.kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], STAGE_BYTES);
          uint8_t* a_dst = sA + stage * A_STAGE;
          uint8_t* b_dst = sB + stage * B_STAGE;
          if (A_MN) {
#pragma unroll
            for (int j = 0; j < BM / MNC; ++j) tma_load_2d(a_dst + j * CHUNK, &tmA, &full[stage], m_blk * BM + j * MNC, kb * BK);
          } else {
            tma_load_2d(a_dst, &tmA, &full[stage], kb * BK, m_blk * BM);
          }
          if (CL == 1) {
            if (B_MN) {
#pragma unroll
              for (int j = 0; j < BN / MNC; ++j) tma_load_2d(b_dst + j * CHUNK, &tmB, &full[stage], n_blk * BN + j * MNC, kb * BK);
            } else {
              tma_load_2d(b_dst, &tmB, &full[stage], kb * BK, n_blk * BN);
            }
          } else {
            // this CTA's half of B lands in both CTAs and completes bytes on both CTAs' full barrier of this stage
            if (B_MN) {
#pragma unroll
              for (int j = 0; j < BN / 2 / MNC; ++j) {
                const int c = crank * (BN / 2 / MNC) + j;
                tma_load_2d_mc(b_dst + c * CHUNK, &tmB, &full[stage], n_blk * BN + c * MNC, kb * BK, 0x3);
              }
            } else {
              tma_load_2d_mc(b_dst + crank * (BN / 2) * ROW_BYTES, &tmB, &full[stage], kb * BK, n_blk * BN + crank * (BN / 2), 0x3);
            }
          }
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ======================= MMA + epilogue (warpgroups 1, 2: rows 64 * (wg - 1) .. of the tile) =======================
    regs_alloc<232>();
    const int cw = wg - 1;                       // which 64-row half of the tile
    const int wq = (threadIdx.x >> 5) & 3;       // warp inside the warpgroup: 16 rows each
    const int g = lane >> 2, t4 = lane & 3;
    float alpha = p.alpha;
    if (F8) alpha *= (p.sinv_a ? __ldg(p.sinv_a) : 1.0f) * (p.sinv_b ? __ldg(p.sinv_b) : 1.0f);
    const float q8_scale = (EPI == EPI_GELU_GRAD_Q8 && p.out_scale) ? __ldg(p.out_scale) : 1.0f;
    float q8_amax = 0.f;
    uint32_t pass_ctr = 0;   // epilogue passes so far: which staging slot a one-box pass uses
    int stage = 0;
    uint32_t phase = 0;
    float acc[128];
    for (int w = w0; w < num_work; w += wstride) {
      const int tile = w % num_tiles, sp = w / num_tiles;
      const int m_blk = (p.m_fastest ? tile % tiles_mu : tile / p.tiles_n) * CL + crank;
      const int n_blk = p.m_fastest ? tile / tiles_mu : tile % p.tiles_n;
      const int kb0 = sp * p.kb_per_split, kb1 = min(num_kb, kb0 + p.kb_per_split);
      const int row0 = m_blk * BM + cw * 64;   // first output row of this warpgroup
      if (AUX) {
        // pull this tile's aux into L2 while the mainloop runs: the warp's 16 rows x 512 bytes = 64 lines, two per lane
#pragma unroll
        for (int i = lane; i < 64; i += 32) {
          const int r = row0 + wq * 16 + (i >> 2), c = n_blk * BN + (i & 3) * 64;
          if (r < p.M && c < p.N) prefetch_l2(p.aux + (long long)r * p.ld_aux + c);
          if (EPI == EPI_MUL2 && r < p.M && c < p.N) prefetch_l2(p.aux2 + (long long)r * p.ldd + c);
        }
      }
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint8_t* a_st = sA + stage * A_STAGE;
        const uint8_t* b_st = sB + stage * B_STAGE;
        // this warpgroup's 64 A rows: K-major -> 64 rows further; MN-major -> the cw-th 64-wide chunk (bf16 only)
        const uint64_t ad = A_MN ? desc_sw128(a_st + cw * CHUNK, CHUNK) : desc_sw128(a_st + cw * 64 * ROW_BYTES, 16);
        const uint64_t bd = B_MN ? desc_sw128(b_st, CHUNK) : desc_sw128(b_st, 16);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          // k-step inside the stage: 16 k-rows of 128 B (MN-major) or 32 bytes of K (K-major)
          const uint64_t adk = desc_add(ad, A_MN ? k * 16 * ROW_BYTES : k * 32);
          const uint64_t bdk = desc_add(bd, B_MN ? k * 16 * ROW_BYTES : k * 32);
          const uint32_t accum = (kb > kb0 || k > 0) ? 1u : 0u;
          if (F8) wgmma_f8_n256(acc, adk, bdk, accum, p.a_fmt, p.b_fmt);
          else wgmma_bf16_ss_n256<A_MN, B_MN>(acc, adk, bdk, accum);
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous stage's MMAs retired: release its shared memory
        if (prev >= 0 && lane == 0) {
          if (CL > 1) {
            mbar_arrive_remote(&empty[prev], 0);
            mbar_arrive_remote(&empty[prev], 1);
          } else {
            mbar_arrive(&empty[prev]);
          }
        }
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev >= 0 && lane == 0) {
        if (CL > 1) {
          mbar_arrive_remote(&empty[prev], 0);
          mbar_arrive_remote(&empty[prev], 1);
        } else {
          mbar_arrive(&empty[prev]);
        }
      }
      if (kb1 <= kb0) continue;
      if (row0 >= p.M) continue;              // the empty half of an M tail, or the idle CTA of a cluster on an odd tile count
      if (EPI == EPI_F32) {
        // ---------------------------------------------------------------- fp32 epilogue, straight from the registers
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long row = (long long)row0 + wq * 16 + g + 8 * h;
          if (row >= p.M) continue;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const int col = n_blk * BN + 8 * j + 2 * t4;
            if (col >= p.N) continue;   // N % 8 == 0: col + 1 < N as well
            const float v0 = acc[4 * j + 2 * h] * alpha, v1 = acc[4 * j + 2 * h + 1] * alpha;
            float* dst = p.d + row * p.ldd + col;
            if (p.accumulate || p.splits > 1) {
              red_add_f32x2(dst, v0, v1);
            } else {
              *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
            }
          }
        }
        continue;
      }
      // ---------------------------------------------------------------- bf16 / E4M3 epilogue through shared memory
      // A pass converts CPP columns of the warpgroup's 64 x 256 slice into the staging slots and stores them by TMA:
      //   * two outputs, 64 columns: D2's box in slot 0, D's in slot 1;
      //   * one output read with aux, 64 columns: one box, in the slot the previous pass did not use (the aux loads of a wider
      //     pass would not fit the register budget);
      //   * EPI_MUL2 (two outputs read with two multipliers): as two outputs, with the pass's aux loaded at its start (holding
      //     the next pass's two multipliers through the stores does not fit the register budget);
      //   * one output, 128 columns: two boxes, one per slot.
      // Only the issuing thread waits for its earlier stores to have been read out of the slots, so the writes to global memory
      // drain under the next pass and the next tile's mainloop.
      constexpr int CPP = (TWO_OUT || AUX) ? 64 : 128;
      constexpr int JP = CPP / 8;                 // 8-column accumulator groups per pass
      constexpr bool ONE_SLOT = !TWO_OUT && CPP == 64;
      uint8_t* stg = sE + cw * EPI_WG_BYTES;
      const uint32_t stg_u32 = smem_u32(stg);
      // aux of one pass (bf16 pairs; 0 outside [M, N]): the next pass's are loaded before this pass's barriers and stores
      uint32_t ax[JP][2], ax2[JP][2];
      const auto load_aux = [&](int q) {
#pragma unroll
        for (int jj = 0; jj < JP; ++jj)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const long long row = (long long)row0 + wq * 16 + g + 8 * h;
            const int col = n_blk * BN + q * CPP + 8 * jj + 2 * t4;
            ax[jj][h] = (col < p.N && row < p.M) ? __ldg(reinterpret_cast<const uint32_t*>(p.aux + row * p.ld_aux + col)) : 0u;
            if (EPI == EPI_MUL2)
              ax2[jj][h] = (col < p.N && row < p.M) ? __ldg(reinterpret_cast<const uint32_t*>(p.aux2 + row * p.ldd + col)) : 0u;
          }
      };
      if (AUX && EPI != EPI_MUL2) load_aux(0);
#pragma unroll
      for (int q = 0; q < BN / CPP; ++q) {
        const int cq = n_blk * BN + q * CPP;      // first output column of the pass
        if (cq >= p.N) break;
        if (EPI == EPI_MUL2) load_aux(q);
        const uint32_t slot = ONE_SLOT ? (pass_ctr++ & 1) * EPI_SLOT : 0;
        const auto slots_free = [&] {             // the previous boxes in the slots this pass writes have been read out
          if ((threadIdx.x & 127) == 0) {
            if (ONE_SLOT) tma_wait_read<1>();
            else tma_wait_read<0>();
          }
          named_bar_sync(1 + cw, 128);
        };
        uint32_t o1[JP][2], o2[JP][2];            // packed outputs: D and D2
        // one stmatrix.x4 covers the warp's 16 rows x 16 columns (groups jj, jj + 1): lane l addresses row l % 8 of matrix l / 8,
        // matrices ordered (rows 0-7, jj), (rows 8-15, jj), (rows 0-7, jj + 1), (rows 8-15, jj + 1). 128B swizzle: the 16-byte
        // chunk c of row r sits at chunk c ^ (r % 8).
        const auto stage_pair = [&](int jj) {
          const int r = wq * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
          const int cg = jj + (lane >> 4);        // 8-column group inside the pass
          const uint32_t off = r * 128 + (((cg & 7) ^ (r & 7)) << 4);
          if (TWO_OUT) {
            stmatrix_x4(stg_u32 + off, o2[jj][0], o2[jj][1], o2[jj + 1][0], o2[jj + 1][1]);
            if (EPI != EPI_GELU_GRAD_Q8) stmatrix_x4(stg_u32 + EPI_SLOT + off, o1[jj][0], o1[jj][1], o1[jj + 1][0], o1[jj + 1][1]);
          } else {
            stmatrix_x4(stg_u32 + slot + (cg >> 3) * EPI_SLOT + off, o1[jj][0], o1[jj][1], o1[jj + 1][0], o1[jj + 1][1]);
          }
        };
        // Q8 stages its outputs as they are made (the E4M3 bytes in slot 1, unswizzled: 64 rows of 64 bytes): holding a whole
        // pass for later does not fit the register budget
        if (EPI == EPI_GELU_GRAD_Q8) slots_free();
#pragma unroll
        for (int jj = 0; jj < JP; ++jj) {
          const int j = q * JP + jj;
          const int col = cq + 8 * jj + 2 * t4;
          const bool col_ok = col < p.N;          // N % 8 == 0: col + 1 < N as well
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const long long row = (long long)row0 + wq * 16 + g + 8 * h;
            const bool in = col_ok && row < p.M;  // elements outside [M, N] are computed but clipped by the TMA store
            float v0 = acc[4 * j + 2 * h] * alpha, v1 = acc[4 * j + 2 * h + 1] * alpha;
            if (p.bias != nullptr && col_ok) {
              const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
              v0 += b.x, v1 += b.y;
            }
            if (AUX) {
              const float2 f = unpack_bf16(ax[jj][h]);
              if (EPI == EPI_RESIDUAL) {
                v0 += f.x, v1 += f.y;
              } else if (EPI == EPI_MUL) {
                v0 *= f.x, v1 *= f.y;
              } else if (EPI == EPI_MUL2) {
                const float2 f2 = unpack_bf16(ax2[jj][h]);
                o2[jj][h] = pack_bf16(v0 * f2.x, v1 * f2.y);
                v0 *= f.x, v1 *= f.y;
              } else {
                v0 *= gelu_grad(f.x), v1 *= gelu_grad(f.y);
              }
            }
            if (EPI == EPI_GELU_DUAL) {
              o2[jj][h] = pack_bf16(v0, v1);   // z (pre-activation)
              v0 = gelu_exact(v0), v1 = gelu_exact(v1);
            } else if (EPI == EPI_GELU_GRAD || EPI == EPI_GELU_GRAD_Q8) {
              // gelu and its derivative share the CDF / PDF evaluation; the derivative replaces the pre-activation as the
              // tensor saved for backward, so the dgrad epilogue is a plain multiply
              float c0, pd0, c1, pd1;
              gelu_cdf_pdf(v0, c0, pd0);
              gelu_cdf_pdf(v1, c1, pd1);
              o2[jj][h] = pack_bf16(fmaf(v0, pd0, c0), fmaf(v1, pd1, c1));
              v0 *= c0, v1 *= c1;
              if (EPI == EPI_GELU_GRAD_Q8) {
                if (in) q8_amax = fmaxf(q8_amax, fmaxf(fabsf(v0), fabsf(v1)));
                st_shared_u16(stg_u32 + EPI_SLOT + (wq * 16 + g + 8 * h) * 64 + 8 * jj + 2 * t4, pack_e4m3x2(v0 * q8_scale, v1 * q8_scale));
                continue;
              }
            } else if (EPI == EPI_SILU_GRAD) {
              // silu and its derivative share the sigmoid (one exp); the derivative is saved as EPI_GELU_GRAD saves gelu'
              const float s0 = silu_sigmoid(v0), s1 = silu_sigmoid(v1);
              o2[jj][h] = pack_bf16(silu_grad_from(v0, s0), silu_grad_from(v1, s1));
              v0 *= s0, v1 *= s1;
            }
            o1[jj][h] = pack_bf16(v0, v1);
          }
          if (EPI == EPI_GELU_GRAD_Q8 && (jj & 1)) stage_pair(jj - 1);
        }
        if (AUX && EPI != EPI_MUL2 && q + 1 < BN / CPP) load_aux(q + 1);
        if (EPI != EPI_GELU_GRAD_Q8) {
          slots_free();
#pragma unroll
          for (int jj = 0; jj < JP; jj += 2) stage_pair(jj);
        }
        fence_proxy_async_smem();   // the generic-proxy writes become visible to the TMA (async proxy) reads
        named_bar_sync(1 + cw, 128);
        if ((threadIdx.x & 127) == 0) {
          if (TWO_OUT) {
            tma_store_2d(&tmD2, stg, cq, row0);
            tma_store_2d(&tmD, stg + EPI_SLOT, cq, row0);
          } else {
            tma_store_2d(&tmD, stg + slot, cq, row0);
            if (CPP == 128 && cq + 64 < p.N) tma_store_2d(&tmD, stg + EPI_SLOT, cq + 64, row0);
          }
          tma_commit();
        }
      }
    }
    if (EPI != EPI_F32 && (threadIdx.x & 127) == 0) tma_wait_all<0>();   // the last stores complete before the CTA exits
    if (EPI == EPI_GELU_GRAD_Q8 && p.out_amax) {
      q8_amax = warp_max_f(q8_amax);
      if (lane == 0 && q8_amax > 0.f) atomic_max_pos_f32(p.out_amax, q8_amax);
    }
  }
  if (CL > 1) cluster_sync_all();   // nobody leaves while the peer may still multicast into it or arrive on its barriers
}

// [R, C] bytes (row stride ld) -> [C, R] contiguous: makes an MN-major fp8 operand K-major for wgmma
__global__ void __launch_bounds__(256) transpose_u8_kernel(const uint8_t* __restrict__ src, long long ld, uint8_t* __restrict__ dst, int R, int C) {
  __shared__ uint8_t t[64][65];
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  for (int i = threadIdx.x; i < 64 * 64; i += 256) {
    const int r = i >> 6, c = i & 63;
    t[r][c] = (r0 + r < R && c0 + c < C) ? src[(long long)(r0 + r) * ld + c0 + c] : 0;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 64 * 64; i += 256) {
    const int c = i >> 6, r = i & 63;
    if (r0 + r < R && c0 + c < C) dst[(long long)(c0 + c) * R + r0 + r] = t[r][c];
  }
}

// Same for 64-aligned shapes and 16-byte aligned rows: 16-byte loads and stores, each thread gathers one 16-byte piece of an
// output row from a column of the shared tile
__global__ void __launch_bounds__(256) transpose_u8_v16_kernel(const uint8_t* __restrict__ src, long long ld, uint8_t* __restrict__ dst, int R) {
  __shared__ __align__(16) uint8_t t[64][80];
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  const int tr = threadIdx.x >> 2, tc = (threadIdx.x & 3) * 16;
  *reinterpret_cast<uint4*>(&t[tr][tc]) = __ldg(reinterpret_cast<const uint4*>(src + (long long)(r0 + tr) * ld + c0 + tc));
  __syncthreads();
  uint32_t w[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int r = tc + 4 * q;
    w[q] = uint32_t(t[r][tr]) | (uint32_t(t[r + 1][tr]) << 8) | (uint32_t(t[r + 2][tr]) << 16) | (uint32_t(t[r + 3][tr]) << 24);
  }
  *reinterpret_cast<uint4*>(dst + (long long)(c0 + tr) * R + r0 + tc) = make_uint4(w[0], w[1], w[2], w[3]);
}

// ------------------------------------------------------------------------------------------ host
using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                              const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                              CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn get_encode() {
  static EncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p)
      throw std::runtime_error("photon_b200: cuTensorMapEncodeTiled not available from the driver");
    fn = reinterpret_cast<EncodeFn>(p);
  }
  return fn;
}

}  // namespace

CUtensorMap make_tmap_2d(const void* ptr, int elem_bytes, bool is_float32, uint64_t inner, uint64_t outer,
                         uint64_t ld_bytes, uint32_t box_inner, uint32_t box_outer, bool swizzle_128b) {
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (ld_bytes & 15))
    throw std::runtime_error("photon_b200 TMA: base pointer and row stride must be 16-byte aligned");
  CUtensorMap m;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMapDataType dt = is_float32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                      : (elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8);
  CUresult r = get_encode()(&m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            swizzle_128b ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("photon_b200: cuTensorMapEncodeTiled failed, code " + std::to_string(int(r)));
  return m;
}

template <int A_MN, int B_MN, int EPI, int CL, int F8>
static void launch_cl(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& td, const CUtensorMap& td2, const Params& p, int grid,
                      cudaStream_t stream) {
  auto kern = gemm_kernel<A_MN, B_MN, EPI, CL, F8>;
  opt_in_smem(kern, SMEM_BYTES);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(NUM_THREADS);
  cfg.dynamicSmemBytes = SMEM_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kern, ta, tb, td, td2, p);
  launched("gemm");
}

template <int A_MN, int B_MN, int EPI, int F8>
static void launch_inst(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& td, const CUtensorMap& td2, const Params& p, int grid,
                        int cluster, cudaStream_t stream) {
  if (cluster == 2) launch_cl<A_MN, B_MN, EPI, 2, F8>(ta, tb, td, td2, p, grid, stream);
  else launch_cl<A_MN, B_MN, EPI, 1, F8>(ta, tb, td, td2, p, grid, stream);
}

void transpose_u8(const void* src, long long ld, void* dst, int R, int C, cudaStream_t stream) {
  const dim3 grid((C + 63) / 64, (R + 63) / 64);
  if (R % 64 == 0 && C % 64 == 0 && ld % 16 == 0 && !(reinterpret_cast<uintptr_t>(src) & 15) && !(reinterpret_cast<uintptr_t>(dst) & 15))
    transpose_u8_v16_kernel<<<grid, 256, 0, stream>>>((const uint8_t*)src, ld, (uint8_t*)dst, R);
  else
    transpose_u8_kernel<<<grid, 256, 0, stream>>>((const uint8_t*)src, ld, (uint8_t*)dst, R, C);
  launched("transpose_u8");
}

// Operands are bf16 or, with g.fp8, 8-bit floats (E4M3 / E5M2 chosen per operand, fp32 accumulate, per-tensor de-scales
// applied in the epilogue). Everything else — pipeline, tile shape, epilogues — is shared.
void gemm_launch(const GemmArgs& g, cudaStream_t stream) {
  if (g.M <= 0 || g.N <= 0 || g.K <= 0) return;
  if (g.N % 8) throw std::runtime_error("photon_b200 gemm: N must be a multiple of 8");
  if (g.fp8 && (g.a_mn || g.b_mn)) throw std::runtime_error("photon_b200 gemm: fp8 operands must be K-major (transpose_u8 first)");
  const bool f32 = g.epi == EPI_F32;
  const int eb = g.fp8 ? 1 : 2;                 // operand element bytes
  const int BKE = ROW_BYTES / eb;               // K elements per stage
  const int MNC = ROW_BYTES / eb;               // MN elements per 128-byte row of an MN-major tile
  // 2-CTA clusters (B tile multicast to both) whenever there are >= 2 M tiles
  const int cluster = (g.cluster > 0 ? g.cluster : ((g.M + BM - 1) / BM >= 2 ? 2 : 1));
  // A: K-major -> dims {K, M}, box {128 B of K, 128 rows};  MN-major -> dims {M, K}, box {128 B of M, BKE k-rows}
  CUtensorMap ta = g.a_mn ? make_tmap_2d(g.A, eb, false, g.M, g.K, g.lda * eb, MNC, BKE)
                          : make_tmap_2d(g.A, eb, false, g.K, g.M, g.lda * eb, BKE, BM);
  CUtensorMap tb = g.b_mn ? make_tmap_2d(g.B, eb, false, g.N, g.K, g.ldb * eb, MNC, BKE)
                          : make_tmap_2d(g.B, eb, false, g.K, g.N, g.ldb * eb, BKE, BN / cluster);
  const bool two_out = g.epi == EPI_GELU_DUAL || g.epi == EPI_GELU_GRAD || g.epi == EPI_GELU_GRAD_Q8 || g.epi == EPI_SILU_GRAD ||
                       g.epi == EPI_MUL2;
  if (two_out && !g.D2) throw std::runtime_error("photon_b200 gemm: the two-output epilogues need the second output");
  const auto aligned16 = [](const void* ptr, long long ld_bytes) { return !(reinterpret_cast<uintptr_t>(ptr) & 15) && !(ld_bytes % 16); };
  // the TMA store writes whole 16-byte pieces of a row, so the E4M3 output also needs N % 16 == 0 (bf16 rows: N % 8 == 0)
  if (g.epi == EPI_GELU_GRAD_Q8 && (!g.fp8 || !g.D8 || !aligned16(g.D8, g.ldd8) || g.N % 16))
    throw std::runtime_error("photon_b200 gemm: the fp8-output epilogue needs fp8 operands, a 16-byte aligned fp8 output and row stride, and N % 16 == 0");
  if ((g.epi == EPI_RESIDUAL || g.epi == EPI_DGELU || g.epi == EPI_MUL || g.epi == EPI_MUL2) &&
      (!g.aux || (g.ld_aux % 8) || (reinterpret_cast<uintptr_t>(g.aux) & 15)))
    throw std::runtime_error("photon_b200 gemm: aux operand missing or not 16-byte aligned");
  if (g.epi == EPI_MUL2 && (!g.aux2 || (g.ld_aux2 % 8) || (reinterpret_cast<uintptr_t>(g.aux2) & 15)))
    throw std::runtime_error("photon_b200 gemm: aux2 operand missing or not 16-byte aligned");
  if (g.bias && (reinterpret_cast<uintptr_t>(g.bias) & 15)) throw std::runtime_error("photon_b200 gemm: bias must be 16-byte aligned");
  if (g.epi != EPI_GELU_GRAD_Q8 && ((reinterpret_cast<uintptr_t>(g.D) & 15) || (g.ldd % 8)))
    throw std::runtime_error("photon_b200 gemm: output must be 16-byte aligned");
  if (two_out && !aligned16(g.D2, g.ldd2 * 2))
    throw std::runtime_error("photon_b200 gemm: the second output and its row stride must be 16-byte aligned");
  // output tensor maps: dims = the logical [M, N] (the TMA clips the tails), one box = 64 rows x 64 columns
  CUtensorMap td = ta, td2 = ta;   // ta stands in for the maps an epilogue does not use
  if (g.epi == EPI_GELU_GRAD_Q8) td = make_tmap_2d(g.D8, 1, false, g.N, g.M, g.ldd8, 64, 64, false);
  else if (!f32) td = make_tmap_2d(g.D, 2, false, g.N, g.M, g.ldd * 2, 64, 64);
  if (two_out) td2 = make_tmap_2d(g.D2, 2, false, g.N, g.M, g.ldd2 * 2, 64, 64);
  Params p{};
  p.M = g.M, p.N = g.N, p.K = g.K;
  p.tiles_m = (g.M + BM - 1) / BM;
  p.tiles_n = (g.N + BN - 1) / BN;
  // keep the larger operand streaming once: iterate the other dimension fastest
  p.m_fastest = (double(g.N) > double(g.M)) ? 1 : 0;
  p.bias = g.bias;
  p.aux = reinterpret_cast<const __nv_bfloat16*>(g.aux);
  p.ld_aux = g.ld_aux;
  p.d = reinterpret_cast<float*>(g.D), p.ldd = g.ldd;
  if (g.epi == EPI_MUL2) p.aux2 = reinterpret_cast<const __nv_bfloat16*>(g.aux2), p.ldd = g.ld_aux2;
  p.accumulate = g.accumulate;
  p.alpha = g.alpha;
  p.a_fmt = g.a_fmt, p.b_fmt = g.b_fmt, p.sinv_a = g.sinv_a, p.sinv_b = g.sinv_b;
  p.out_scale = g.out_scale, p.out_amax = g.out_amax;
  int sms = g.num_sms;
  if (sms <= 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  const int tiles = p.tiles_m * p.tiles_n;
  const int num_kb = (g.K + BKE - 1) / BKE;
  p.splits = 1;
  if (f32 && g.accumulate && tiles < sms && num_kb >= 16) {
    // few output tiles, long K (weight gradients): split K across CTAs, partials meet in the fp32
    // gradient bucket through red.global.add. Aim for ~2 waves, >= 8 k-blocks per split.
    int s = (2 * sms + tiles / 2) / tiles;
    if (s > num_kb / 8) s = num_kb / 8;
    if (s < 1) s = 1;
    p.splits = s;
    if (const char* e = std::getenv("PB_GEMM_SPLITS")) {  // tuning knob (scripts/bench_kernels.py sweeps it)
      const int v = std::atoi(e);
      if (v >= 1 && v <= num_kb) p.splits = v;
    }
  }
  p.kb_per_split = (num_kb + p.splits - 1) / p.splits;
  p.splits = (num_kb + p.kb_per_split - 1) / p.kb_per_split;  // drop empty tails
  const int work_units = ((p.tiles_m + cluster - 1) / cluster) * p.tiles_n * p.splits;
  int grid = work_units * cluster < sms ? work_units * cluster : (sms / cluster) * cluster;

#define PB_CASE(AM, BMJ, E, F)                                              \
  if (g.a_mn == AM && g.b_mn == BMJ && g.epi == E && int(g.fp8) == F) {     \
    launch_inst<AM, BMJ, E, F>(ta, tb, td, td2, p, grid, cluster, stream);  \
    return;                                                                 \
  }
  PB_CASE(0, 0, EPI_BF16, 0)
  PB_CASE(0, 0, EPI_RESIDUAL, 0)
  PB_CASE(0, 0, EPI_GELU_DUAL, 0)
  PB_CASE(0, 0, EPI_F32, 0)
  PB_CASE(0, 1, EPI_BF16, 0)
  PB_CASE(0, 1, EPI_DGELU, 0)
  PB_CASE(0, 1, EPI_MUL, 0)
  PB_CASE(0, 0, EPI_GELU_GRAD, 0)
  PB_CASE(0, 1, EPI_F32, 0)
  PB_CASE(1, 1, EPI_F32, 0)
  PB_CASE(1, 1, EPI_BF16, 0)
  PB_CASE(1, 0, EPI_F32, 0)
  PB_CASE(1, 0, EPI_BF16, 0)
  // gated / SiLU feed-forward blocks: activation + derivative, the two-multiplier forward and dgrad, the accumulating dgrad
  PB_CASE(0, 0, EPI_SILU_GRAD, 0)
  PB_CASE(0, 0, EPI_MUL2, 0)
  PB_CASE(0, 1, EPI_MUL2, 0)
  PB_CASE(0, 1, EPI_RESIDUAL, 0)
  // fp8 operands (K-major; the bindings transpose MN-major ones): forward, dgrad and wgrad epilogues
  PB_CASE(0, 0, EPI_BF16, 1)
  PB_CASE(0, 0, EPI_RESIDUAL, 1)
  PB_CASE(0, 0, EPI_GELU_GRAD, 1)
  PB_CASE(0, 0, EPI_GELU_GRAD_Q8, 1)
  PB_CASE(0, 0, EPI_F32, 1)
  PB_CASE(0, 0, EPI_MUL, 1)
#undef PB_CASE
  throw std::runtime_error("photon_b200 gemm: unsupported (a_major, b_major, epilogue, operand type) combination");
}

}  // namespace pb
