// The bf16 -> fp8 rounding helpers shared by every kernel that must produce the SAME bytes for the same values: the weight
// quantisation of the unsharded engine (fp8_ops.cu, seg_quant_kernel) and the once-per-version requantisation of the ZeRO-3
// weight shards (comm.cu, zero3_fp8_requant_kernel). One definition, so the two cannot drift apart. (The positive-float
// atomic max they both use is atomic_max_pos_f32 in ptx.cuh.)
#pragma once
#include <stdint.h>

#include "ptx.cuh"

namespace pb {

__device__ __forceinline__ void unpack8f(const uint4& u, float (&f)[8]) {
  float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y), c = unpack_bf16(u.z), d = unpack_bf16(u.w);
  f[0] = a.x, f[1] = a.y, f[2] = b.x, f[3] = b.y, f[4] = c.x, f[5] = c.y, f[6] = d.x, f[7] = d.y;
}
template <int FMT>
__device__ __forceinline__ uint2 quant8(const float (&f)[8], float s) {
  uint2 o;
  if (FMT == 0) {
    o.x = pack_e4m3x4(f[0] * s, f[1] * s, f[2] * s, f[3] * s);
    o.y = pack_e4m3x4(f[4] * s, f[5] * s, f[6] * s, f[7] * s);
  } else {
    o.x = pack_e5m2x4(f[0] * s, f[1] * s, f[2] * s, f[3] * s);
    o.y = pack_e5m2x4(f[4] * s, f[5] * s, f[6] * s, f[7] * s);
  }
  return o;
}
__device__ __forceinline__ float amax8(const float (&f)[8], float m) {
#pragma unroll
  for (int k = 0; k < 8; ++k) m = fmaxf(m, fabsf(f[k]));
  return m;
}
// Scales are the recipe's quotients rounded to nearest (photon_b200/train/fp8.py): the build's --use_fast_math would otherwise
// turn these divisions into approximate reciprocals, a few ulp away from fmax / amax and from the exact inverse of the scale.
__device__ __forceinline__ float scale_of(float fmax, float amax) { return __fdiv_rn(fmax, amax); }
__device__ __forceinline__ float inv_scale(float s) { return __frcp_rn(s); }
// per-tensor current scaling: the E4M3 scale of a weight from its amax (1 when the tensor is all zeros or not finite)
__device__ __forceinline__ float weight_scale(float amax, float fmax) { return (amax > 0.f && amax < 3.0e38f) ? scale_of(fmax, amax) : 1.0f; }

}  // namespace pb
