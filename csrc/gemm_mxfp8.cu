// Block-scaled FP8 GEMM for sm_90a:  D[M,N] = (A .* SFA)[M,K] * (B .* SFB)[N,K]^T (+ bias), bf16 out
//
//   OCP MXFP8: E4M3 elements, one E8M0 scale per 32 consecutive K elements of every row of A and of B. Hopper's tensor cores
//   take no scale operands, so every 32-K group is one wgmma.m64n128k32 into a partial accumulator, which is then multiplied by
//   scale_a(row) * scale_b(column) of that group and added to the running fp32 sum in registers.
//
//   * A / B tiles: TMA (128-byte swizzle) into a 4-stage mbarrier ring, 128 K-elements per stage, as in gemm_tcgen05.cu;
//   * scale factors: stored in global memory as per (128 rows x 128 K) block a 512-byte atom [32][4][4]: byte
//     (r % 32) * 16 + (r / 32) * 4 + (k / 32) holds the scale of row r, K-group k/32 — so a stage's scales are ONE contiguous
//     bulk copy per operand (cp.async.bulk, counted on the same mbarrier as the tiles);
//   * two MMA warpgroups (64 rows of the 128 x 128 tile each), epilogue from registers: bias -> bf16 -> global.
//
// mx_quantize_kernel produces both the E4M3 data and the scale atoms from a bf16 matrix in one pass (scale = 2^(floor(log2 amax) - 8)).
// North-star item "block-scaled fp8 for the GEMMs"; numerics oracle: de-quantise and multiply in fp32 (tests/test_fp8_gpu.py).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <stdexcept>
#include <string>

#include "gemm_tcgen05.h"
#include "launch.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace pb {

namespace {

constexpr int BM = 128, BN = 128, BK = 128;             // BK in elements = bytes
constexpr int A_STAGE = BM * 128, B_STAGE = BN * 128;    // 16 KiB each
constexpr int SF_BYTES = 512;                            // one 128-row scale atom per operand and stage
constexpr int STAGE_BYTES = A_STAGE + B_STAGE + 2 * SF_BYTES;
constexpr int STAGES = 4;
constexpr int SMEM_BYTES = STAGES * (A_STAGE + B_STAGE) + STAGES * 2 * SF_BYTES + 256 + 1024;
constexpr int NUM_THREADS = 384;   // warpgroup 0: TMA producer (one thread); warpgroups 1, 2: MMA + epilogue

struct MxParams {
  int M, N, K, tiles_m, tiles_n, mblk128, nblk128;
  const uint8_t* sfa;   // [K/128][ceil(M/128)][512]
  const uint8_t* sfb;   // [K/128][ceil(N/128) padded to even][512]
  const float* bias;
  __nv_bfloat16* d;
  long long ldd;
};

__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// E8M0 -> fp32: 2^(e - 127); e = 0 is 2^-127 (a denormal)
__device__ __forceinline__ float e8m0(uint32_t e) { return e ? __uint_as_float(e << 23) : __uint_as_float(0x00400000u); }

__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_mx_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const MxParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = sA + STAGES * A_STAGE;
  uint8_t* sSFA = sB + STAGES * B_STAGE;
  uint8_t* sSFB = sSFA + STAGES * SF_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(sSFB + STAGES * SF_BYTES);
  uint64_t* empty = full + STAGES;

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);   // one arrival per MMA warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int num_tiles = p.tiles_m * p.tiles_n;
  const int num_kb = (p.K + BK - 1) / BK;

  if (wg == 0) {
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int m_blk = t % p.tiles_m, n_blk = t / p.tiles_m;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], STAGE_BYTES);
          tma_load_2d(sA + stage * A_STAGE, &tmA, &full[stage], kb * BK, m_blk * BM);
          tma_load_2d(sB + stage * B_STAGE, &tmB, &full[stage], kb * BK, n_blk * BN);
          bulk_load(sSFA + stage * SF_BYTES, p.sfa + ((long long)kb * p.mblk128 + m_blk) * 512, SF_BYTES, &full[stage]);
          bulk_load(sSFB + stage * SF_BYTES, p.sfb + ((long long)kb * p.nblk128 + n_blk) * 512, SF_BYTES, &full[stage]);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    regs_alloc<232>();
    const int cw = wg - 1;
    const int wq = (threadIdx.x >> 5) & 3;
    const int g = lane >> 2, t4 = lane & 3;
    const int r0 = cw * 64 + wq * 16 + g;        // this thread's rows inside the tile: r0, r0 + 8
    int stage = 0;
    uint32_t phase = 0;
    float acc[64], part[64];
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const int m_blk = t % p.tiles_m, n_blk = t / p.tiles_m;
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint64_t ad = desc_sw128(sA + stage * A_STAGE + cw * 64 * 128, 16);
        const uint64_t bd = desc_sw128(sB + stage * B_STAGE, 16);
        const uint8_t* sfa = sSFA + stage * SF_BYTES;
        const uint8_t* sfb = sSFB + stage * SF_BYTES;
#pragma unroll 1
        for (int kg = 0; kg < 4; ++kg) {
          wgmma_fence();
          wgmma_e4m3_e4m3_n128(part, desc_add(ad, kg * 32), desc_add(bd, kg * 32), 0u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_regs(part);
          const float sa0 = e8m0(sfa[(r0 % 32) * 16 + (r0 / 32) * 4 + kg]);
          const float sa1 = e8m0(sfa[((r0 + 8) % 32) * 16 + ((r0 + 8) / 32) * 4 + kg]);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int c = 8 * j + 2 * t4;
            const float sb0 = e8m0(sfb[(c % 32) * 16 + (c / 32) * 4 + kg]);
            const float sb1 = e8m0(sfb[((c + 1) % 32) * 16 + ((c + 1) / 32) * 4 + kg]);
            acc[4 * j] = fmaf(part[4 * j], sa0 * sb0, acc[4 * j]);
            acc[4 * j + 1] = fmaf(part[4 * j + 1], sa0 * sb1, acc[4 * j + 1]);
            acc[4 * j + 2] = fmaf(part[4 * j + 2], sa1 * sb0, acc[4 * j + 2]);
            acc[4 * j + 3] = fmaf(part[4 * j + 3], sa1 * sb1, acc[4 * j + 3]);
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[stage]);
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long row = (long long)m_blk * BM + r0 + 8 * h;
        if (row >= p.M) continue;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = n_blk * BN + 8 * j + 2 * t4;
          if (col >= p.N) continue;
          float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
          if (p.bias != nullptr) v0 += __ldg(p.bias + col), v1 += __ldg(p.bias + col + 1);
          *reinterpret_cast<uint32_t*>(p.d + row * p.ldd + col) = pack_bf16(v0, v1);
        }
      }
    }
  }
}

// bf16 [R, K] (row stride ld) -> E4M3 [R, K] + E8M0 scale atoms [K/128][ceil(R/128) (padded to rblk)][512]; one thread = 8 elements,
// four neighbouring threads = one 32-element scale block.
__global__ void __launch_bounds__(256) mx_quantize_kernel(const __nv_bfloat16* __restrict__ x, long long ld, uint8_t* __restrict__ q,
                                                          uint8_t* __restrict__ sf, long long R, int K, int rblk) {
  const long long groups_per_row = K / 8;
  const long long total = R * groups_per_row;
  for (long long g = blockIdx.x * 256ll + threadIdx.x; g < ((total + 3) & ~3ll); g += gridDim.x * 256ll) {
    const bool ok = g < total;
    const long long r = ok ? g / groups_per_row : 0;
    const int k8 = ok ? int(g % groups_per_row) : 0;
    float f[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (ok) {
      const uint4 u = *reinterpret_cast<const uint4*>(x + r * ld + k8 * 8);
      const float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y), c = unpack_bf16(u.z), d = unpack_bf16(u.w);
      f[0] = a.x, f[1] = a.y, f[2] = b.x, f[3] = b.y, f[4] = c.x, f[5] = c.y, f[6] = d.x, f[7] = d.y;
    }
    float am = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) am = fmaxf(am, fabsf(f[i]));
    am = fmaxf(am, __shfl_xor_sync(0xffffffff, am, 1));
    am = fmaxf(am, __shfl_xor_sync(0xffffffff, am, 2));
    // OCP MX: shared exponent = floor(log2(amax)) - emax(E4M3 = 8); stored biased by 127; amax = 0 -> smallest scale
    int e = am > 0.f ? (int((__float_as_uint(am) >> 23) & 0xFF) - 127 - 8) : -127;
    e = e < -127 ? -127 : (e > 127 ? 127 : e);
    const float inv = __uint_as_float(uint32_t(127 - e) << 23);   // 2^-e (e in [-127, 127] -> exponent field 0..254; 0 -> denormal 0 handled below)
    const float s = (127 - e) == 0 ? 0.f : inv;
    if (ok) {
      uint2 o;
      o.x = pack_e4m3x4(f[0] * s, f[1] * s, f[2] * s, f[3] * s);
      o.y = pack_e4m3x4(f[4] * s, f[5] * s, f[6] * s, f[7] * s);
      *reinterpret_cast<uint2*>(q + r * (long long)K + k8 * 8) = o;
      if ((k8 & 3) == 0) {
        const int kg = k8 / 4;                   // 32-element group index along K
        const long long blk = (long long)(kg / 4) * rblk + r / 128;
        const int rr = int(r % 128);
        sf[blk * 512 + (rr % 32) * 16 + (rr / 32) * 4 + (kg % 4)] = uint8_t(e + 127);
      }
    }
  }
}

}  // namespace

void mx_quantize(const void* x_bf16, long long ld, void* q8, void* sf, long long R, int K, int rblk, cudaStream_t st) {
  if (K % 128) throw std::runtime_error("mx_quantize: K must be a multiple of 128");
  const long long groups = R * (K / 8);
  long long blocks = (groups + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  mx_quantize_kernel<<<int(blocks), 256, 0, st>>>((const __nv_bfloat16*)x_bf16, ld, (uint8_t*)q8, (uint8_t*)sf, R, K, rblk);
  launched("mx_quantize");
}

void gemm_mxfp8_launch(const void* A, const void* B, void* D, const void* sfa, const void* sfb, const float* bias, int M, int N, int K,
                       long long ldd, int num_sms, cudaStream_t stream) {
  if (K % 128 || N % 8) throw std::runtime_error("gemm_mxfp8: K must be a multiple of 128 and N of 8");
  CUtensorMap ta = make_tmap_2d(A, 1, false, K, M, K, BK, BM);
  CUtensorMap tb = make_tmap_2d(B, 1, false, K, N, K, BK, BN);
  MxParams p{};
  p.M = M, p.N = N, p.K = K;
  p.tiles_m = (M + BM - 1) / BM, p.tiles_n = (N + BN - 1) / BN;
  p.mblk128 = p.tiles_m, p.nblk128 = 2 * ((N + 255) / 256);
  p.sfa = reinterpret_cast<const uint8_t*>(sfa), p.sfb = reinterpret_cast<const uint8_t*>(sfb), p.bias = bias;
  p.d = reinterpret_cast<__nv_bfloat16*>(D), p.ldd = ldd;
  opt_in_smem(gemm_mx_kernel, SMEM_BYTES);
  int sms = num_sms > 0 ? num_sms : 132;
  const int tiles = p.tiles_m * p.tiles_n;
  gemm_mx_kernel<<<tiles < sms ? tiles : sms, NUM_THREADS, SMEM_BYTES, stream>>>(ta, tb, p);
  launched("gemm_mxfp8");
}

}  // namespace pb
