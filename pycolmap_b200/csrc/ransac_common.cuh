// ransac_common.cuh -- device pieces shared by the RANSAC kernels of the two-view verifier (verify.cu) and of the
// absolute pose estimator (abs_pose.cu): counter-based sampling, warp reductions and the three-way outcome of the
// division-free fp32 inlier test.  The dynamic trial bound (ComputeNumTrials, U:optim/ransac.h) is
// geom::compute_num_trials.
#pragma once
#include <cstdint>

namespace b2m {

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

__device__ __forceinline__ double shfl_d(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }
__device__ __forceinline__ double warp_sum_d(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Outcome of `residual <= thr` evaluated as lhs <= rhs = thr * denominator in fp32: bit 0 = clearly an inlier,
// bit 1 = borderline (within 1 % of the threshold, or not finite) -- the caller re-evaluates those in fp64, so a
// decision equals the fp64 one as long as the fp32 rounding of lhs and rhs stays inside the 1 % band (see the
// limits at verify.cu inlier_f32).  STRICT comparisons: lhs == rhs == 0 (both underflowed) or == inf (both overflowed) is
// neither clearly in nor clearly out, like any NaN.
__device__ __forceinline__ int classify_f32(float lhs, float rhs) {
  const int in = lhs < 0.99f * rhs ? 1 : 0;
  const int out = lhs > 1.01f * rhs ? 1 : 0;
  return in | ((in | out) ^ 1) << 1;
}

}  // namespace b2m
