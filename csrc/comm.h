// Host API of the fused NVLink collectives (see comm.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "fused_ops.h"

namespace pb {

constexpr int MAX_PEERS = 8;
constexpr int CTL_WORDS = 256;  // control page size in uint32 words (1 KiB)

struct CommCtl {
  uint32_t* ctl[MAX_PEERS];  // control page of every rank (peer-mapped)
  int n;
  int rank;
  unsigned long long timeout_ns;  // bound on every cross-GPU spin (0 = wait forever); see CP_STATUS / CP_ABORT in comm.cu
};

struct FedRoundArgs {
  const float* acc[MAX_PEERS];  // per-rank unnormalised weighted sum of its clients' params (full length)
  float* xg[MAX_PEERS];         // per-rank fp32 global/master plane (broadcast target); xg[rank] == x
  void* xs[MAX_PEERS];          // per-rank bf16 compute copy (may be null)
  float* x;                     // local server copy (only [lo,hi) is read/updated)
  float* m;
  float* v;
  long long lo, hi;             // this rank's shard, multiples of 4
  long long total;              // full flat length (local bf16 cast phase)
  int kind;                     // 0 fedavg, 1 nesterov, 2 fedmom, 3 fedadam, 4 fedyogi
  float avg_scale;              // scaling_fn(K)
  float lr, mu;                 // fedavg / nesterov / fedmom
  float eta, beta1, beta2, tau, inv_bc1, inv_bc2, sign;  // adam / yogi (sign=-1 descent, +1 reference compat)
  const float* acc_mc;          // NVLS: multicast address of the acc planes (in-switch reduction), or nullptr
  float* xg_mc;                 // NVLS: multicast address of the fp32 global planes (one store reaches every GPU), or nullptr
  // per-tensor squared-norm by-products: seg_bounds[0..n_seg] = tensor boundaries in units of 256 floats (ascending, the last
  // entry >= total/256), seg_sums = double[5][n_seg] (pg, fedavg result, model, momentum, second momentum); both may be null
  const long long* seg_bounds;
  int n_seg;
  double* seg_sums;
  float wsum;                   // this rank's sum of client weights, published to its control page by the kernel when publish_wsum
  int publish_wsum;
  int zero_seg_sums;            // zero seg_sums inside the kernel (first launch of a round)
  int walk;                     // 0 = grid-stride over unit pairs, 1 = block-contiguous runs (tuning knob PB_ROUND_WALK)
};

struct AllReduceArgs {
  float* buf[MAX_PEERS];
  long long lo, hi;
  float* buf_mc;                // NVLS multicast address of the gradient planes, or nullptr
};

// N1 + K11 + K12 in one launch (ZeRO-style): reduce-scatter of the gradient planes, global-norm clipping, the local
// optimizer on this rank's shard of (p, m, v), all-gather of the new fp32 masters and their bf16 cast.
struct ZeroStepArgs {
  float* grads[MAX_PEERS];      // per-rank flat gradient plane (full length)
  float* params[MAX_PEERS];     // per-rank fp32 master plane (full length)
  void* shadow[MAX_PEERS];      // per-rank bf16 compute copy (full length; may be null)
  float* m;                     // this rank's moment shards (length hi - lo)
  float* v;
  long long lo, hi;             // this rank's shard, multiples of 4
  OptimHyper h;
  float max_norm;               // <= 0: no clipping
  float grad_mult;              // 1 / loss scale
  const float* grads_mc;        // NVLS multicast addresses (nullptr = P2P loops)
  float* params_mc;
  void* shadow_mc;
};

// ZeRO-3 (full parameter sharding): reduce-scatter of ONE unit's gradient staging planes into the owner's gradient shard.
struct ShardReduceArgs {
  const float* stage[MAX_PEERS];  // per-rank staging plane of the unit: n slices of `per` floats (slice r belongs to rank r)
  const float* stage_mc;          // NVLS multicast address of the staging planes, or nullptr
  float* dst;                     // this rank's slice of the persistent fp32 gradient shard (per floats), accumulated into
  long long per;                  // slice length, multiple of 4 (0 = barrier only)
  float scale;                    // 1 / n (mean over ranks)
};
void zero3_reduce_launch(const ShardReduceArgs& a, const CommCtl& c, uint32_t epoch, int num_sms, cudaStream_t st);

// ZeRO-3 under amp_fp8: the E4M3 copy of every block weight matrix, quantised once per parameter version by the owners of its
// pieces with the tensor's GLOBAL amax (per-tensor current scaling, the same bytes the unsharded engine produces).
struct Zero3RequantArgs {
  const void* w16;                // this rank's bf16 shard
  uint8_t* w8;                    // this rank's E4M3 shard (same element offsets)
  const long long* pieces;        // [n_pieces][3]: shard offset, numel (both multiples of 8), weight slot
  int n_pieces;
  int n_w;                        // number of weight matrices (slots)
  float* amax_local;              // [n_w] this rank's partial amax; zero between launches (the kernel leaves it zeroed)
  float* amax[MAX_PEERS];         // every rank's amax plane [world][n_w]: row r is written by rank r
  float* meta;                    // the engine's fp8 scaling state [3][n_roles]: scale, 1/scale, amax
  long long n_roles;
  const int* roles;               // [n_w] weight slot -> role column of meta
  float fmax;                     // largest finite E4M3 value
};
void zero3_fp8_requant_launch(const Zero3RequantArgs& a, const CommCtl& c, uint32_t epoch, int num_sms, cudaStream_t st);

void ddp_zero_step_launch(const ZeroStepArgs& a, const CommCtl& c, uint32_t epoch, float* out_norm, int num_sms, cudaStream_t st);
void fed_round_launch(const FedRoundArgs& a, const CommCtl& c, uint32_t epoch, int num_sms, cudaStream_t st);
void ddp_allreduce_launch(const AllReduceArgs& a, const CommCtl& c, uint32_t epoch, float* out_norm, int num_sms, cudaStream_t st);
void set_wsum(uint32_t* ctl, float w, bool zero_sums, cudaStream_t st);
int ctl_sums_word_offset();
int ctl_status_word_offset();   // sticky word: bit t = peer t missed a start barrier, bit 8+t = peer t vanished mid-kernel

}  // namespace pb
