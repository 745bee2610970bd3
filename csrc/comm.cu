// In-kernel NVLink collectives fused with their adjacent compute (no NCCL on these paths):
//
//   fed_round_kernel   R1+R2 of a federated round (SURVEY §2.5 (c)): every GPU owns 1/n of the flat
//                      parameter index space; it pulls that slice of every peer's weighted client sum
//                      with P2P loads, forms the pseudo-gradient, applies the server optimizer
//                      (FedAvg / Nesterov / FedMom / FedAdam / FedYogi) on its shard of (x, m, v) in
//                      registers, accumulates the L2-norm by-products, and pushes the new fp32 values
//                      AND their bf16 cast straight into every peer's parameter planes with P2P stores.
//   ddp_allreduce_kernel  N1: one-pass reduce-scatter + all-gather of the flat gradient bucket over peer
//                      pointers, fused with the mean (1/n) and the squared-norm partials for clipping.
//   zero3_reduce_kernel   ZeRO-3 reduce-scatter of one unit's gradient into the owner's shard.
//   zero3_fp8_requant_kernel  ZeRO-3 under amp_fp8: global per-tensor amax exchange + E4M3 quantisation of the weight shards.
//
// Cross-GPU ordering uses epoch-valued flags in each rank's control page (st.release.sys /
// ld.acquire.sys); all CTAs are co-resident (grid <= #SMs) so in-kernel spinning is deadlock-free.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <stdexcept>
#include <string>

#include "comm.h"
#include "fp8_round.cuh"
#include "launch.h"
#include "optim_dev.cuh"
#include "ptx.cuh"

namespace pb {

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffff, v, o);
  return v;
}

// Control page layout (uint32 words) inside every rank's arena:
//   [0,8)   start flags (slot r written by rank r)      [8,16)  end flags
//   [16]    local "go" flag (block 0 -> other blocks)   [17]    local done-block counter   [24,32) mid-kernel flags
//   [32,34) float wsum (this rank's sum of client weights)   [64..) double sq_parts[8], double sums[8]
constexpr int CP_START = 0, CP_END = 8, CP_GO = 16, CP_DONE = 17, CP_GO2 = 18, CP_ABORT = 19, CP_STATUS = 20, CP_MID = 24, CP_WSUM = 32,
              CP_SQPARTS = 64, CP_SUMS = 96;

__device__ __forceinline__ unsigned long long now_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// spin until *flag >= epoch; false when `timeout_ns` (0 = wait forever) expires first
__device__ __forceinline__ bool wait_flag_sys(const uint32_t* flag, uint32_t epoch, unsigned long long timeout_ns) {
  if (ld_acquire_sys(flag) >= epoch) return true;
  const unsigned long long t0 = now_ns();
  unsigned spins = 0;
  while (ld_acquire_sys(flag) < epoch) {
    if (timeout_ns && (++spins & 1023u) == 0 && now_ns() - t0 > timeout_ns) return false;
  }
  return true;
}

// Start-of-kernel rendezvous of all ranks. Returns false on EVERY block of this rank when a peer did not show up within
// c.timeout_ns: nothing has been touched yet, the kernel returns immediately (a clean abort), the missing peers are
// recorded as a sticky bit mask in this rank's control page (CP_STATUS) for the host watchdog, and CP_ABORT holds the epoch.
// A dead rank therefore turns into an aborted round on the survivors instead of an endless spin.
__device__ __forceinline__ bool grid_peer_barrier_start(const CommCtl& c, uint32_t epoch, const float* publish_wsum = nullptr,
                                                        double* zero_buf = nullptr, int zero_n = 0) {
  uint32_t* mine = c.ctl[c.rank];
  __shared__ uint32_t s_abort;
  if (blockIdx.x == 0) {
    if (threadIdx.x == 0) s_abort = 0;
    // work that must be ordered before the grid starts / before peers read this rank's page: zero the per-tensor accumulators,
    // publish this rank's client-weight sum (saves two tiny launches per round)
    for (int i = threadIdx.x; i < zero_n; i += blockDim.x) zero_buf[i] = 0.0;
    __syncthreads();
    if (threadIdx.x < c.n) {
      if (publish_wsum) mine[CP_WSUM] = __float_as_uint(*publish_wsum);   // released by the flag store below (same thread)
      st_release_sys(c.ctl[threadIdx.x] + CP_START + c.rank, epoch);                 // tell peer t "rank is here"
      if (!wait_flag_sys(mine + CP_START + threadIdx.x, epoch, c.timeout_ns)) {       // wait for peer t
        atomicOr(mine + CP_STATUS, 1u << threadIdx.x);
        atomicOr(&s_abort, 1u);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      if (s_abort) mine[CP_ABORT] = epoch;
      __threadfence();
      asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(mine + CP_GO), "r"(epoch) : "memory");
    }
    __syncthreads();
    return s_abort == 0;
  }
  if (threadIdx.x == 0) {
    uint32_t v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(mine + CP_GO) : "memory");
    } while (v < epoch);
    s_abort = (*reinterpret_cast<volatile uint32_t*>(mine + CP_ABORT) == epoch) ? 1u : 0u;
  }
  __syncthreads();
  return s_abort == 0;
}

// returns true in the LAST block to finish (after all blocks' peer stores were fenced)
__device__ __forceinline__ bool grid_done(const CommCtl& c) {
  __shared__ int last;
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint32_t prev = atomicAdd(c.ctl[c.rank] + CP_DONE, 1u);
    last = (prev == gridDim.x - 1);
    if (last) c.ctl[c.rank][CP_DONE] = 0;
  }
  __syncthreads();
  return last != 0;
}

__device__ __forceinline__ void peer_barrier_end(const CommCtl& c, uint32_t epoch) {
  uint32_t* mine = c.ctl[c.rank];
  __threadfence_system();
  if (threadIdx.x < c.n) {
    st_release_sys(c.ctl[threadIdx.x] + CP_END + c.rank, epoch);
    // a peer that vanished INSIDE the kernel cannot be waited for: record it (bit 8+t = "left mid-kernel") and leave
    if (!wait_flag_sys(mine + CP_END + threadIdx.x, epoch, c.timeout_ns)) atomicOr(mine + CP_STATUS, 0x100u << threadIdx.x);
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------ R1 + R2
// Work decomposition: the shard is cut into UNITS of 256 floats (64 float4 = two coalesced 512-byte warp accesses); every
// warp owns a CONTIGUOUS run of units. Tensor boundaries of the flat layout are multiples of 256 floats, so a unit never
// straddles two tensors and a warp walks the tensor table monotonically: the five squared-norm partials (pseudo-gradient,
// fedavg result, new model, momentum, second momentum) are kept per tensor in registers and flushed with one warp reduction
// + five fp64 atomics when the warp crosses into the next tensor — the reference's `server/layer/{i}/l2_norm_*` metrics
// (ref: photon/strategy/fedadam.py:333-381) come out of the same single pass as the update itself.
constexpr int UNIT4 = 64;   // float4 per unit

__global__ void __launch_bounds__(512) fed_round_kernel(const FedRoundArgs a, const CommCtl c, const uint32_t epoch) {
  if (!grid_peer_barrier_start(c, epoch, a.publish_wsum ? &a.wsum : nullptr, a.zero_seg_sums ? a.seg_sums : nullptr,
                               a.zero_seg_sums && a.seg_sums ? 5 * a.n_seg : 0))
    return;

  // total client weight = sum over ranks (each rank published its own before the launch)
  float wtot = 0.f;
  for (int p = 0; p < c.n; ++p) wtot += __uint_as_float(ld_acquire_sys(c.ctl[p] + CP_WSUM));
  const bool skip = !(wtot > 0.f);  // no successful client anywhere -> keep the model (ignore_failed_rounds)
  const float inv = skip ? 0.f : a.avg_scale / wtot;

  const int lane = threadIdx.x & 31;
  float s_pg = 0.f, s_a = 0.f, s_x = 0.f, s_m = 0.f, s_v = 0.f;   // Σpg², Σa², Σx², Σm², Σv² of the tensor the warp is in
  __nv_bfloat16* xs_mine = reinterpret_cast<__nv_bfloat16*>(a.xs[c.rank]);
  const bool local_only = (c.n == 1);

  auto load_acc = [&](long long i) -> float4 {
    if (local_only) return __ldcs(reinterpret_cast<const float4*>(a.acc[0]) + i);     // plain streaming load: nobody else wrote it
    if (a.acc_mc) return mm_ld_reduce_add_f4(reinterpret_cast<const float4*>(a.acc_mc) + i);   // NVLS: the switch adds the N planes
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
    for (int p = 0; p < c.n; ++p) {  // fixed order -> bitwise reproducible across runs
      const float4 t = ld_peer_f4(reinterpret_cast<const float4*>(a.acc[p]) + i);
      acc.x += t.x, acc.y += t.y, acc.z += t.z, acc.w += t.w;
    }
    return acc;
  };
  // one float4 of the shard: pseudo-gradient, server optimizer, norm partials, broadcast (fp32 to all, bf16 locally)
  auto process = [&](long long i, float4 acc, float4 X, float4 Mv, float4 Vv) {
      float av[4] = {acc.x * inv, acc.y * inv, acc.z * inv, acc.w * inv};
      float xv[4] = {X.x, X.y, X.z, X.w};
      float mv[4] = {Mv.x, Mv.y, Mv.z, Mv.w}, vv[4] = {Vv.x, Vv.y, Vv.z, Vv.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float pg = xv[k] - av[k];
        s_pg += pg * pg;
        s_a += av[k] * av[k];
        switch (a.kind) {
          case 0:  // FedAvg
            xv[k] -= a.lr * pg;
            break;
          case 1:  // Nesterov (torch SGD form)
            mv[k] = a.mu * mv[k] + pg;
            xv[k] -= a.lr * (pg + a.mu * mv[k]);
            break;
          case 2: {  // FedMom
            const float vn = xv[k] - a.lr * pg;
            xv[k] = (1.f + a.mu) * vn - a.mu * mv[k];
            mv[k] = vn;
            break;
          }
          default: {  // 3 FedAdam, 4 FedYogi
            mv[k] = a.beta1 * mv[k] + (1.f - a.beta1) * pg;
            const float g2 = pg * pg;
            if (a.kind == 3) {
              vv[k] = a.beta2 * vv[k] + (1.f - a.beta2) * g2;
            } else {
              const float d = g2 - vv[k];
              vv[k] += (1.f - a.beta2) * g2 * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
            }
            const float step = a.eta * (mv[k] * a.inv_bc1) / (sqrtf(vv[k] * a.inv_bc2) + a.tau);
            xv[k] += a.sign * step;
            break;
          }
        }
        s_x += xv[k] * xv[k];
        s_m += mv[k] * mv[k];
        s_v += vv[k] * vv[k];
      }
      if (a.kind >= 1) reinterpret_cast<float4*>(a.m)[i] = make_float4(mv[0], mv[1], mv[2], mv[3]);
      if (a.kind >= 3) reinterpret_cast<float4*>(a.v)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
      // R2 (a): push the updated fp32 slice into every rank's global plane over NVLink
      const float4 nx = make_float4(xv[0], xv[1], xv[2], xv[3]);
      if (local_only) {
        reinterpret_cast<float4*>(a.xg[0])[i] = nx;
      } else if (a.xg_mc) {    // NVLS: one multicast store lands in every rank's global plane
        mm_st_f4(reinterpret_cast<float4*>(a.xg_mc) + i, nx);
      } else {
#pragma unroll 1
        for (int p = 0; p < c.n; ++p) st_peer_f4(reinterpret_cast<float4*>(a.xg[p]) + i, nx);
      }
      // R2 (b) for the OWN shard: the bf16 compute copy straight from registers (no second pass over this slice)
      if (xs_mine) {
        uint2 o;
        o.x = pack_bf16(xv[0], xv[1]), o.y = pack_bf16(xv[2], xv[3]);
        reinterpret_cast<uint2*>(xs_mine)[i] = o;
      }
  };
  int seg = 0;
  auto flush = [&]() {
    const float t0 = warp_sum(s_pg), t1 = warp_sum(s_a), t2 = warp_sum(s_x), t3 = warp_sum(s_m), t4 = warp_sum(s_v);
    if (lane == 0 && a.seg_sums) {
      double* d = a.seg_sums + seg;
      if (t0 != 0.f) atomicAdd(d, double(t0));
      if (t1 != 0.f) atomicAdd(d + a.n_seg, double(t1));
      if (t2 != 0.f) atomicAdd(d + 2 * a.n_seg, double(t2));
      if (t3 != 0.f) atomicAdd(d + 3 * a.n_seg, double(t3));
      if (t4 != 0.f) atomicAdd(d + 4 * a.n_seg, double(t4));
    }
    s_pg = s_a = s_x = s_m = s_v = 0.f;
  };
  if (!skip) {
    const long long u_lo = a.lo / (4 * UNIT4), u_hi = (a.hi + 4 * UNIT4 - 1) / (4 * UNIT4);   // shard bounds are unit-aligned
    // two walks over the units (a.walk, PB_ROUND_WALK): 0 = grid-stride, 1 = every BLOCK owns a contiguous run with its warps on
    // neighbouring unit pairs (a dense ~32 KiB window per block). Both keep every warp monotonic in the unit space, which is what
    // the per-tensor bookkeeping needs.
    const long long W = blockDim.x >> 5;
    long long ub, ue, ustep;
    if (a.walk == 0) {
      // grid-stride over unit PAIRS: at any moment the whole grid streams one dense window (2 KiB per warp, ~2.4 MiB per trip);
      // every warp still walks the unit space monotonically
      ub = u_lo + 2 * ((long long)blockIdx.x * W + (threadIdx.x >> 5));
      ue = u_hi;
      ustep = 2 * W * gridDim.x;
    } else {
      long long per = (u_hi - u_lo + gridDim.x - 1) / gridDim.x;
      per = (per + 1) & ~1ll;                                      // even: pairs never straddle two blocks
      const long long bb = u_lo + blockIdx.x * per;
      ue = (bb + per < u_hi) ? bb + per : u_hi;
      ub = bb + 2 * (threadIdx.x >> 5);
      ustep = 2 * W;
    }
    const long long hi4 = a.hi / 4;
    if (ub < ue && a.seg_bounds) {   // binary search: first tensor whose end is beyond this warp's first unit
      int l = 0, r = a.n_seg - 1;
      while (l < r) {
        const int mid = (l + r) >> 1;
        if (a.seg_bounds[mid + 1] > ub) r = mid;
        else l = mid + 1;
      }
      seg = l;
    }
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long u = ub; u < ue; u += ustep) {   // two units per trip: four 16-byte loads per plane per thread in flight
      float4 A[4], X[4], M[4], V[4];
      long long idx[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        idx[k] = (u + (k >> 1)) * UNIT4 + (k & 1) * 32 + lane;
        const bool ok = (u + (k >> 1)) < ue && idx[k] < hi4;
        if (!ok) idx[k] = -1;
        A[k] = ok ? load_acc(idx[k]) : z4;
        X[k] = ok ? reinterpret_cast<const float4*>(a.x)[idx[k]] : z4;
        M[k] = (ok && a.kind >= 1) ? reinterpret_cast<const float4*>(a.m)[idx[k]] : z4;
        V[k] = (ok && a.kind >= 3) ? reinterpret_cast<const float4*>(a.v)[idx[k]] : z4;
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if ((k & 1) == 0 && a.seg_bounds && (u + (k >> 1)) < ue) {   // entering a unit: did the warp cross into the next tensor?
          const long long unit = u + (k >> 1);
          if (unit >= a.seg_bounds[seg + 1]) {
            flush();
            while (seg + 1 < a.n_seg && unit >= a.seg_bounds[seg + 1]) ++seg;
          }
        }
        if (idx[k] >= 0) process(idx[k], A[k], X[k], M[k], V[k]);
      }
    }
    flush();
  }
  // every rank's slice has landed everywhere once the end barrier completes; the last block runs it and then
  // releases the whole grid into R2 (b) for the slices OWNED BY PEERS: the bf16 compute copy is cast LOCALLY from the received
  // fp32 plane (halves the NVLink bytes of the broadcast compared with also pushing the bf16 copy to 7 peers)
  uint32_t* mine = c.ctl[c.rank];
  if (grid_done(c)) {
    peer_barrier_end(c, epoch);
    if (threadIdx.x == 0) {
      __threadfence();
      asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(mine + CP_GO2), "r"(epoch) : "memory");
    }
  }
  if (xs_mine != nullptr && !skip && !local_only) {
    if (threadIdx.x == 0) {
      uint32_t v;
      do {
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(mine + CP_GO2) : "memory");
      } while (v < epoch);
    }
    __syncthreads();
    const float4* src = reinterpret_cast<const float4*>(a.xg[c.rank]);
    const long long lo4 = a.lo / 4, n_own = a.hi / 4 - lo4, n_rest = a.total / 4 - n_own;
    for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < n_rest; j += (long long)gridDim.x * blockDim.x) {
      const long long i = j < lo4 ? j : j + n_own;   // skip the own shard
      const float4 v = ld_peer_f4(src + i);  // written by peers during this launch: bypass the non-coherent path
      uint2 o;
      o.x = pack_bf16(v.x, v.y), o.y = pack_bf16(v.z, v.w);
      reinterpret_cast<uint2*>(xs_mine)[i] = o;
    }
  }
}

// ------------------------------------------------------------------------------------------ N1
__global__ void __launch_bounds__(512) ddp_allreduce_kernel(const AllReduceArgs a, const CommCtl c, const uint32_t epoch) {
  if (!grid_peer_barrier_start(c, epoch)) return;
  const float inv = 1.0f / c.n;
  float sq = 0.f;
  const long long lo4 = a.lo / 4, hi4 = a.hi / 4;
  for (long long i = lo4 + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < hi4; i += (long long)gridDim.x * blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a.buf_mc) {
      acc = mm_ld_reduce_add_f4(reinterpret_cast<const float4*>(a.buf_mc) + i);
    } else {
#pragma unroll 1
      for (int p = 0; p < c.n; ++p) {
        const float4 t = ld_peer_f4(reinterpret_cast<const float4*>(a.buf[p]) + i);
        acc.x += t.x, acc.y += t.y, acc.z += t.z, acc.w += t.w;
      }
    }
    acc.x *= inv, acc.y *= inv, acc.z *= inv, acc.w *= inv;
    sq += acc.x * acc.x + acc.y * acc.y + acc.z * acc.z + acc.w * acc.w;
    if (a.buf_mc) {
      mm_st_f4(reinterpret_cast<float4*>(a.buf_mc) + i, acc);
    } else {
#pragma unroll 1
      for (int p = 0; p < c.n; ++p) st_peer_f4(reinterpret_cast<float4*>(a.buf[p]) + i, acc);
    }
  }
  __shared__ float red[16];
  sq = warp_sum(sq);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sq;
  __syncthreads();
  double* sums = reinterpret_cast<double*>(c.ctl[c.rank] + CP_SUMS);
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) t += red[w];
    atomicAdd(sums + 7, double(t));
  }
  if (grid_done(c)) {
    if (threadIdx.x < c.n) {  // publish this shard's squared norm to every rank
      const double mine = *reinterpret_cast<volatile double*>(sums + 7);
      double* dst = reinterpret_cast<double*>(c.ctl[threadIdx.x] + CP_SQPARTS) + c.rank;
      asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(dst), "d"(mine) : "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) sums[7] = 0.0;
    peer_barrier_end(c, epoch);
  }
}

// ------------------------------------------------------------------------------------------ ZeRO-3 gradient reduce-scatter
// One UNIT (a transformer block, or the embeddings + final norm) of the flat gradient: every rank has just written the unit's
// gradient of its own microbatch into its staging plane (n slices of `per` floats); rank r owns slice r and accumulates the
// mean over ranks into its persistent fp32 gradient shard. Start barrier: every rank's staging plane is complete; end barrier:
// every rank has finished reading, so the plane may be overwritten by the next unit of the same parity.
__global__ void __launch_bounds__(512) zero3_reduce_kernel(const ShardReduceArgs a, const CommCtl c, const uint32_t epoch) {
  if (!grid_peer_barrier_start(c, epoch)) return;
  const long long off4 = (long long)c.rank * (a.per / 4), n4 = a.per / 4;
  float4* dst = reinterpret_cast<float4*>(a.dst);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a.stage_mc) {
      acc = mm_ld_reduce_add_f4(reinterpret_cast<const float4*>(a.stage_mc) + off4 + i);
    } else if (c.n == 1) {
      acc = reinterpret_cast<const float4*>(a.stage[0])[i];
    } else {
#pragma unroll 1
      for (int p = 0; p < c.n; ++p) {
        const float4 t = ld_peer_f4(reinterpret_cast<const float4*>(a.stage[p]) + off4 + i);
        acc.x += t.x, acc.y += t.y, acc.z += t.z, acc.w += t.w;
      }
    }
    float4 d = dst[i];
    d.x = fmaf(acc.x, a.scale, d.x), d.y = fmaf(acc.y, a.scale, d.y), d.z = fmaf(acc.z, a.scale, d.z), d.w = fmaf(acc.w, a.scale, d.w);
    dst[i] = d;
  }
  if (grid_done(c)) peer_barrier_end(c, epoch);
}

// ------------------------------------------------------------------------------------------ ZeRO-3 E4M3 weight shards
// Launched once per parameter version, after every rank has written its new bf16 shard. Phase 1: the partial amax of every block
// weight matrix over this rank's pieces of it; the last block publishes this rank's amax vector into row `rank` of every peer's
// amax plane. Mid barrier. Phase 2: global amax = max over the rows (order independent: every rank gets the same value), scale
// exactly as seg_quant_kernel computes it, the weight-role columns of meta, and this rank's pieces quantised into its E4M3 shard
// with the shared rounding code. End barrier: every rank's E4M3 shard is complete before anybody pulls from it.
__global__ void __launch_bounds__(512) zero3_fp8_requant_kernel(const Zero3RequantArgs a, const CommCtl c, const uint32_t epoch) {
  if (!grid_peer_barrier_start(c, epoch)) return;
  uint32_t* mine = c.ctl[c.rank];
  extern __shared__ float s_scale[];   // [n_w]
  __shared__ float smax[16];
  const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x, nthr = (long long)gridDim.x * blockDim.x;
  const __nv_bfloat16* w16 = static_cast<const __nv_bfloat16*>(a.w16);
  // ---- phase 1: partial amax per weight over this rank's pieces
  for (int p = 0; p < a.n_pieces; ++p) {
    const long long off = a.pieces[3 * p], n8 = a.pieces[3 * p + 1] / 8;
    const uint4* src = reinterpret_cast<const uint4*>(w16 + off);
    float am = 0.f;
    for (long long i = tid; i < n8; i += nthr) {
      float f[8];
      unpack8f(src[i], f);
      am = amax8(f, am);
    }
    am = warp_max_f(am);
    if ((threadIdx.x & 31) == 0) smax[threadIdx.x >> 5] = am;
    __syncthreads();
    if (threadIdx.x == 0) {
      float m = smax[0];
      for (int w = 1; w < (blockDim.x >> 5); ++w) m = fmaxf(m, smax[w]);
      if (m > 0.f) atomic_max_pos_f32(a.amax_local + a.pieces[3 * p + 2], m);
    }
    __syncthreads();
  }
  // ---- publish (last block), mid barrier, release the grid
  if (grid_done(c)) {
    for (int j = threadIdx.x; j < a.n_w; j += blockDim.x) {
      const float v = *reinterpret_cast<volatile float*>(a.amax_local + j);
      for (int p = 0; p < c.n; ++p) {
        float* dst = a.amax[p] + (long long)c.rank * a.n_w + j;
        asm volatile("st.relaxed.sys.global.f32 [%0], %1;" ::"l"(dst), "f"(v) : "memory");
      }
      a.amax_local[j] = 0.f;   // ready for the next version
    }
    __syncthreads();
    __threadfence_system();
    if (threadIdx.x < c.n) {
      st_release_sys(c.ctl[threadIdx.x] + CP_MID + c.rank, epoch);
      if (!wait_flag_sys(mine + CP_MID + threadIdx.x, epoch, c.timeout_ns)) atomicOr(mine + CP_STATUS, 0x100u << threadIdx.x);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(mine + CP_GO2), "r"(epoch) : "memory");
    }
  }
  if (threadIdx.x == 0) {
    uint32_t v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(mine + CP_GO2) : "memory");
    } while (v < epoch);
  }
  __syncthreads();
  // ---- phase 2: global amax -> scale (every weight: each rank computes with all of them), then this rank's pieces
  const float* rows = a.amax[c.rank];
  for (int j = threadIdx.x; j < a.n_w; j += blockDim.x) {
    float m = 0.f;
    for (int p = 0; p < c.n; ++p) {
      float x;
      asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(x) : "l"(rows + (long long)p * a.n_w + j) : "memory");
      m = fmaxf(m, x);
    }
    const float s = weight_scale(m, a.fmax);
    s_scale[j] = s;
    if (blockIdx.x == 0) {
      const long long r = a.roles[j];
      a.meta[r] = s;
      a.meta[a.n_roles + r] = inv_scale(s);
      a.meta[2 * a.n_roles + r] = m;
    }
  }
  __syncthreads();
  for (int p = 0; p < a.n_pieces; ++p) {
    const long long off = a.pieces[3 * p], n8 = a.pieces[3 * p + 1] / 8;
    const float s = s_scale[a.pieces[3 * p + 2]];
    const uint4* src = reinterpret_cast<const uint4*>(w16 + off);
    uint2* dst = reinterpret_cast<uint2*>(a.w8 + off);
    for (long long i = tid; i < n8; i += nthr) {
      float f[8];
      unpack8f(src[i], f);
      dst[i] = quant8<0>(f, s);
    }
  }
  if (grid_done(c)) peer_barrier_end(c, epoch);
}

// ------------------------------------------------------------------------------------------ N1 + K11 + K12
// Phase 1: every rank sums its shard of all gradient planes over NVLink (mean folded in), keeps the result in its own
// plane and publishes the shard's squared norm to every rank. Mid barrier. Phase 2: clip coefficient from the global norm,
// local optimizer on the shard of (p, m, v), new fp32 masters and bf16 casts pushed into every rank's planes.
__global__ void __launch_bounds__(512) ddp_zero_step_kernel(const ZeroStepArgs a, const CommCtl c, const uint32_t epoch, float* out_norm) {
  if (!grid_peer_barrier_start(c, epoch)) return;
  uint32_t* mine = c.ctl[c.rank];
  const float inv = a.grad_mult / c.n;
  float sq = 0.f;
  const long long lo4 = a.lo / 4, hi4 = a.hi / 4;
  float* gmine = a.grads[c.rank];
  for (long long i = lo4 + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < hi4; i += (long long)gridDim.x * blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a.grads_mc) {
      acc = mm_ld_reduce_add_f4(reinterpret_cast<const float4*>(a.grads_mc) + i);
    } else {
#pragma unroll 1
      for (int p = 0; p < c.n; ++p) {
        const float4 t = ld_peer_f4(reinterpret_cast<const float4*>(a.grads[p]) + i);
        acc.x += t.x, acc.y += t.y, acc.z += t.z, acc.w += t.w;
      }
    }
    acc.x *= inv, acc.y *= inv, acc.z *= inv, acc.w *= inv;
    sq += acc.x * acc.x + acc.y * acc.y + acc.z * acc.z + acc.w * acc.w;
    reinterpret_cast<float4*>(gmine)[i] = acc;   // re-read by the same thread in phase 2
  }
  __shared__ float red[16];
  __shared__ float s_coef;
  sq = warp_sum(sq);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sq;
  __syncthreads();
  double* sums = reinterpret_cast<double*>(mine + CP_SUMS);
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) t += red[w];
    atomicAdd(sums + 7, double(t));
  }
  if (grid_done(c)) {   // last block: publish the shard norm to every rank, cross-GPU barrier, release the grid
    if (threadIdx.x < c.n) {
      const double part = *reinterpret_cast<volatile double*>(sums + 7);
      double* dst = reinterpret_cast<double*>(c.ctl[threadIdx.x] + CP_SQPARTS) + c.rank;
      asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(dst), "d"(part) : "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) sums[7] = 0.0;
    __threadfence_system();
    if (threadIdx.x < c.n) {
      st_release_sys(c.ctl[threadIdx.x] + CP_MID + c.rank, epoch);
      if (!wait_flag_sys(mine + CP_MID + threadIdx.x, epoch, c.timeout_ns)) atomicOr(mine + CP_STATUS, 0x100u << threadIdx.x);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(mine + CP_GO2), "r"(epoch) : "memory");
    }
  }
  if (threadIdx.x == 0) {
    uint32_t v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(mine + CP_GO2) : "memory");
    } while (v < epoch);
    const double* parts = reinterpret_cast<const double*>(mine + CP_SQPARTS);
    double t = 0.0;
    for (int p = 0; p < c.n; ++p) {
      double x;
      asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(x) : "l"(parts + p) : "memory");
      t += x;
    }
    const float norm = float(sqrt(t));
    s_coef = a.max_norm > 0.f ? fminf(1.0f, a.max_norm / (norm + 1e-6f)) : 1.0f;
    if (blockIdx.x == 0 && out_norm) *out_norm = norm;
  }
  __syncthreads();
  const float coef = s_coef;
  // ---- phase 2: optimizer on the shard, broadcast of the new masters + bf16 casts
  for (long long i = lo4 + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < hi4; i += (long long)gridDim.x * blockDim.x) {
    const float4 G = reinterpret_cast<const float4*>(gmine)[i];
    const float4 P = reinterpret_cast<const float4*>(a.params[c.rank])[i];
    float pp[4] = {P.x, P.y, P.z, P.w};
    const float gg[4] = {G.x * coef, G.y * coef, G.z * coef, G.w * coef};
    float mm[4] = {0.f, 0.f, 0.f, 0.f}, vv[4] = {0.f, 0.f, 0.f, 0.f};
    const long long li = i - lo4;   // moments are shard-local
    if (a.h.kind != 2) {
      const float4 Mv = reinterpret_cast<const float4*>(a.m)[li];
      const float4 Vv = reinterpret_cast<const float4*>(a.v)[li];
      mm[0] = Mv.x, mm[1] = Mv.y, mm[2] = Mv.z, mm[3] = Mv.w;
      vv[0] = Vv.x, vv[1] = Vv.y, vv[2] = Vv.z, vv[3] = Vv.w;
    }
    optim_update4(pp, gg, mm, vv, a.h);
    if (a.h.kind != 2) {
      reinterpret_cast<float4*>(a.m)[li] = make_float4(mm[0], mm[1], mm[2], mm[3]);
      reinterpret_cast<float4*>(a.v)[li] = make_float4(vv[0], vv[1], vv[2], vv[3]);
    }
    const float4 np = make_float4(pp[0], pp[1], pp[2], pp[3]);
    uint2 nb;
    nb.x = pack_bf16(pp[0], pp[1]), nb.y = pack_bf16(pp[2], pp[3]);
    if (a.params_mc) {
      mm_st_f4(reinterpret_cast<float4*>(a.params_mc) + i, np);
      if (a.shadow_mc) mm_st_u2(reinterpret_cast<uint2*>(a.shadow_mc) + i, nb);
    } else {
#pragma unroll 1
      for (int p = 0; p < c.n; ++p) {
        st_peer_f4(reinterpret_cast<float4*>(a.params[p]) + i, np);
        if (a.shadow[p]) st_peer_u2(reinterpret_cast<uint2*>(a.shadow[p]) + i, nb);
      }
    }
  }
  if (grid_done(c)) peer_barrier_end(c, epoch);
}

__global__ void allreduce_norm_finalize_kernel(const uint32_t* ctl, int n, float* out_norm) {
  const double* parts = reinterpret_cast<const double*>(ctl + CP_SQPARTS);
  double t = 0.0;
  for (int p = 0; p < n; ++p) t += parts[p];
  *out_norm = float(sqrt(t));
}

__global__ void set_wsum_kernel(uint32_t* ctl, float w, int zero_sums) {
  ctl[CP_WSUM] = __float_as_uint(w);
  if (zero_sums) {
    double* s = reinterpret_cast<double*>(ctl + CP_SUMS);
    for (int i = 0; i < 7; ++i) s[i] = 0.0;
  }
}

}  // namespace

static int sm_count(int num_sms) {   // one CTA per SM (co-residency is what makes the in-kernel spins deadlock-free)
  if (num_sms > 0) return num_sms;
  int dev = 0, n = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 132;
}

int ctl_sums_word_offset() { return CP_SUMS; }
int ctl_status_word_offset() { return CP_STATUS; }

void fed_round_launch(const FedRoundArgs& a, const CommCtl& c, uint32_t epoch, int num_sms, cudaStream_t st) {
  if ((a.lo % 256) || (a.hi % 4)) throw std::runtime_error("fed_round: the shard must start on a 256-element boundary and end on a multiple of 4");
  fed_round_kernel<<<sm_count(num_sms), 512, 0, st>>>(a, c, epoch);
  launched("fed_round");
}
void ddp_allreduce_launch(const AllReduceArgs& a, const CommCtl& c, uint32_t epoch, float* out_norm, int num_sms, cudaStream_t st) {
  if ((a.lo % 4) || (a.hi % 4)) throw std::runtime_error("ddp_allreduce: shard bounds must be multiples of 4");
  ddp_allreduce_kernel<<<sm_count(num_sms), 512, 0, st>>>(a, c, epoch);
  launched("ddp_allreduce");
  if (out_norm) {
    allreduce_norm_finalize_kernel<<<1, 1, 0, st>>>(c.ctl[c.rank], c.n, out_norm);
    launched("allreduce_norm_finalize");
  }
}
void ddp_zero_step_launch(const ZeroStepArgs& a, const CommCtl& c, uint32_t epoch, float* out_norm, int num_sms, cudaStream_t st) {
  if ((a.lo % 4) || (a.hi % 4)) throw std::runtime_error("ddp_zero_step: shard bounds must be multiples of 4");
  ddp_zero_step_kernel<<<sm_count(num_sms), 512, 0, st>>>(a, c, epoch, out_norm);
  launched("ddp_zero_step");
}
void zero3_reduce_launch(const ShardReduceArgs& a, const CommCtl& c, uint32_t epoch, int num_sms, cudaStream_t st) {
  // a pure barrier (per == 0) needs one block; the reduction is bandwidth bound well below a full grid
  const int grid = a.per == 0 ? 1 : sm_count(num_sms);
  zero3_reduce_kernel<<<grid, 512, 0, st>>>(a, c, epoch);
  launched("zero3_reduce");
}
void zero3_fp8_requant_launch(const Zero3RequantArgs& a, const CommCtl& c, uint32_t epoch, int num_sms, cudaStream_t st) {
  if (a.n_w <= 0 || a.n_w > 12288) throw std::runtime_error("zero3_fp8_requant: 1..12288 weight matrices (one fp32 scale each in shared memory)");
  zero3_fp8_requant_kernel<<<sm_count(num_sms), 512, sizeof(float) * a.n_w, st>>>(a, c, epoch);
  launched("zero3_fp8_requant");
}

void set_wsum(uint32_t* ctl, float w, bool zero_sums, cudaStream_t st) {
  set_wsum_kernel<<<1, 1, 0, st>>>(ctl, w, zero_sums ? 1 : 0);
  launched("set_wsum");
}

}  // namespace pb
