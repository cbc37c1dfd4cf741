// match_guided_kernel.cu -- K1g: guided matching.  The wgmma int8 GEMM of K1 with an epilogue that
// first zeroes every dot product whose keypoint pair violates the two-view geometry of the image pair
// (float32, as upstream) and then runs the exact running top-2 / ratio / distance logic.
//
// Semantics: U:feature/sift.cc MatchGuidedSiftFeaturesCPU (COLMAP 3.9.1), SURVEY.md section 8 row G1,
// reached from R:pipeline/match_features.h:97-100 (SiftMatchingOptions.guided_matching):
//   CALIBRATED / UNCALIBRATED geometry -> squared Sampson error of F,  PLANAR / PANORAMIC /
//   PLANAR_OR_PANORAMIC -> squared forward transfer error of H; entries with error > max_error^2 get
//   dist = 0; then FindBestMatchesBruteForce; the result replaces TwoViewGeometry::inlier_matches.
// The float32 filter is written with non-fused single operations in the same order as the oracle
// (oracle/oracle_match.c orc_match_guided, compiled with -ffp-contract=off) so that the match indices
// are bit-identical.  Work unit = (pair, direction, 128-row strip); only pairs flagged by the decision
// kernel do any work, so the simple non-persistent pipeline of match_kernel.cu is reused (in 128-column halves,
// which leaves registers for the per-element test beside the accumulators).
#include "match_kernel.cuh"
#include "ptx.cuh"

namespace b2m {

namespace {

constexpr int kDim = 128;
constexpr int kTileM = 128;    // rows per CTA: two consumer warpgroups of 64 rows
constexpr int kTileN = 256;
constexpr int kStages = 4;
constexpr int kBytesA = kTileM * kDim;
constexpr int kBytesB = kTileN * kDim;
constexpr int kConsumerWarps = 8;
constexpr int kThreads = (kConsumerWarps + 1) * 32;   // + TMA producer warp

struct __align__(8) Barriers {
  uint64_t full_a;
  uint64_t full_b[kStages];
  uint64_t empty_b[kStages];
};

constexpr int kKpBytes = 2 * kTileN * 16;  // two buffers of 256 per-column float4 (the column's share of the residual)
constexpr size_t kSmemBytes = 1024 + kBytesA + kStages * kBytesB + kKpBytes + sizeof(Barriers);

__device__ __forceinline__ void merge_top2(uint32_t& a1, uint32_t& a2, uint32_t b1, uint32_t b2) {
  const uint32_t lo = min(a1, b1);
  a1 = max(a1, b1);
  a2 = max(max(a2, b2), lo);
}

// The geometric test of a matrix element, split into a per-row part, a per-column part and a per-element rest.
// kind 0: F, squared Sampson error r = num^2 / den <= thr; kind 1: H, squared forward transfer error.  Every float
// operation is rounded separately and in the order of orc_match_guided (oracle/oracle_match.c), so the decisions are
// bit-identical; what moves is WHERE an operand is computed:
//   num = x2 * Fx0 + y2 * Fx1 + Fx2,  den = ((Fx0^2 + Fx1^2) + Ft0^2) + Ft1^2,  Fx = F (x1, y1, 1),  Ft = F^T (x2, y2, 1)
// Fx depends on the image-1 keypoint only, Ft on the image-2 keypoint only.  Rows of the tile are image 1 in
// direction 0 and image 2 in direction 1, so one side is a per-thread constant and the other is staged per column
// (one float4 per column, computed once per tile by one thread instead of once per element by 128):
//   mode 0 (F, dir 0): row (Fx0, Fx1, Fx2, Fx0^2 + Fx1^2)      column (x2, y2, Ft0^2, Ft1^2)
//   mode 1 (F, dir 1): row (x2, y2, Ft0^2, Ft1^2)              column (Fx0, Fx1, Fx2, Fx0^2 + Fx1^2)
//   mode 2 (H): u = (H x1)_x / w, v = (H x1)_y / w belong to image 1, (x2, y2) to image 2; r = (u - x2)^2 + (v - y2)^2
//               (the sign of a correctly rounded difference does not change its square)
__device__ __forceinline__ float4 side_image1(int kind, const float* M, float x1, float y1) {
  if (kind == 0) {
    const float Fx0 = __fadd_rn(__fadd_rn(__fmul_rn(M[0], x1), __fmul_rn(M[1], y1)), M[2]);
    const float Fx1 = __fadd_rn(__fadd_rn(__fmul_rn(M[3], x1), __fmul_rn(M[4], y1)), M[5]);
    const float Fx2 = __fadd_rn(__fadd_rn(__fmul_rn(M[6], x1), __fmul_rn(M[7], y1)), M[8]);
    return make_float4(Fx0, Fx1, Fx2, __fadd_rn(__fmul_rn(Fx0, Fx0), __fmul_rn(Fx1, Fx1)));
  }
  const float w = __fadd_rn(__fadd_rn(__fmul_rn(M[6], x1), __fmul_rn(M[7], y1)), M[8]);
  const float u = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(M[0], x1), __fmul_rn(M[1], y1)), M[2]), w);
  const float v = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(M[3], x1), __fmul_rn(M[4], y1)), M[5]), w);
  return make_float4(u, v, 0.f, 0.f);
}
__device__ __forceinline__ float4 side_image2(int kind, const float* M, float x2, float y2) {
  if (kind == 0) {
    const float Ft0 = __fadd_rn(__fadd_rn(__fmul_rn(M[0], x2), __fmul_rn(M[3], y2)), M[6]);
    const float Ft1 = __fadd_rn(__fadd_rn(__fmul_rn(M[1], x2), __fmul_rn(M[4], y2)), M[7]);
    return make_float4(x2, y2, __fmul_rn(Ft0, Ft0), __fmul_rn(Ft1, Ft1));
  }
  return make_float4(x2, y2, 0.f, 0.f);
}

// `fl(a / den) <= thr` without the division.  thr_next = the next float above thr (thr > 0).
//   a > RU(den * thr_next) >= den * thr_next > den * thr_mid  =>  the quotient rounds above thr          (reject)
//   a < RD(den * thr)      <= den * thr                       =>  the quotient is below thr, rounds <= thr (accept)
// and only in the sliver between the two (relative width 2^-23), or with zero / infinite / NaN operands, the exact
// decision: the quotient rounds to a float <= thr iff a / den < thr_mid (the midpoint of thr and thr_next), or
// == thr_mid and the tie goes to thr (even mantissa); (double) den * thr_mid is exact (24 x 25 significand bits).
__device__ __noinline__ bool sampson_sliver(float a, float den, float thr, double thr_mid, bool thr_even) {
  if (!(den > 0.0f) || !(a < __int_as_float(0x7f800000)) || !(den < __int_as_float(0x7f800000)))
    return __fdiv_rn(a, den) <= thr;   // the literal expression (never on real data)
  const double lhs = static_cast<double>(a), rhs = static_cast<double>(den) * thr_mid;
  return lhs < rhs || (lhs == rhs && thr_even);
}

// One 128-column half of a tile: mask the dot products of the thread's two rows by the geometric test and update
// their tile-local top-2 keys.  Column 8 j + 2 q + e of the half is acc[4 j + 2 i + e] for row i; its side of the
// residual is cols[8 j + 2 q + e].  An element whose Sampson test falls in the sliver between the two bounds takes the
// exact decision at once (rare).
template <int MODE>
__device__ __forceinline__ void scan_half(const uint32_t (&acc)[64], const float4* cols, int q, int col0, const float4 (&r)[2],
                                          float thr, float thr_next, double thr_mid, bool thr_even, uint32_t (&k1)[2],
                                          uint32_t (&k2)[2]) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int col = 8 * j + 2 * q + e;
      const float4 c = cols[col];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        bool ok;
        if (MODE == 2) {
          const float du = __fsub_rn(r[i].x, c.x), dv = __fsub_rn(r[i].y, c.y);
          ok = __fadd_rn(__fmul_rn(du, du), __fmul_rn(dv, dv)) <= thr;
        } else {
          float num, den;
          if (MODE == 0) {
            num = __fadd_rn(__fadd_rn(__fmul_rn(c.x, r[i].x), __fmul_rn(c.y, r[i].y)), r[i].z);
            den = __fadd_rn(__fadd_rn(r[i].w, c.z), c.w);
          } else {
            num = __fadd_rn(__fadd_rn(__fmul_rn(r[i].x, c.x), __fmul_rn(r[i].y, c.y)), c.z);
            den = __fadd_rn(__fadd_rn(c.w, r[i].z), r[i].w);
          }
          const float a = __fmul_rn(num, num);
          // ok = a < RD(den * thr); decided = ok | a > RU(den * thr_next) (ordered compares: a NaN stays undecided)
          ok = a < __fmul_rd(den, thr);
          if (!ok && !(a > __fmul_ru(den, thr_next))) ok = sampson_sliver(a, den, thr, thr_mid, thr_even);
        }
        const uint32_t d = ok ? acc[4 * j + 2 * i + e] : 0u;
        const uint32_t key = d * 256u + static_cast<uint32_t>(255 - (col0 + col));
        const uint32_t lo = min(k1[i], key);
        k1[i] = max(k1[i], key);
        k2[i] = max(k2[i], lo);
      }
    }
  }
}

}  // namespace

__global__ void __launch_bounds__(kThreads, 1)
b2m_k1_guided_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmap_a, const MatchParams p,
                     const GuidedParams g) {
  const int pair = blockIdx.z;
  const int gkind = g.kind[pair];
  if (gkind < 0) return;  // pair not eligible for guided matching (uniform exit)
  const int dir = g.only_dir >= 0 ? g.only_dir : blockIdx.y;
  const int strip = blockIdx.x;
  const int ia = p.pairs[2 * pair + dir];
  const int ib = p.pairs[2 * pair + (dir ^ 1)];
  // gathered launch: the rows are the matched columns of the row direction, ranked ascending, their descriptors in the
  // pair's slice of the scratch (tmap_a); row r is feature gath_cols[r] of image `ia`
  const bool gathered = g.gath_cnt != nullptr;
  const int nA = gathered ? g.gath_cnt[pair] : p.img_nfeat[ia];
  const int nB = p.img_nfeat[ib];
  if (strip * kTileM >= nA) return;
  const int rowA = (gathered ? pair * p.mstride : p.img_row0[ia]) + strip * kTileM;
  const int rowB = p.img_row0[ib];
  const int n_tiles = (nB + kTileN - 1) / kTileN;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smA = smem;
  uint8_t* smB = smem + kBytesA;
  float4* kp_s = reinterpret_cast<float4*>(smem + kBytesA + kStages * kBytesB);
  Barriers* bars = reinterpret_cast<Barriers*>(smem + kBytesA + kStages * kBytesB + kKpBytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == kConsumerWarps && lane == 0) {
    tma_prefetch_desc(&tmap);
    tma_prefetch_desc(&tmap_a);
    mbar_init(&bars->full_a, 1);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&bars->full_b[s], 1);
      mbar_init(&bars->empty_b[s], kConsumerWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ===== TMA producer =====
    if (lane == 0 && n_tiles > 0) {
      mbar_arrive_expect_tx(&bars->full_a, kBytesA);
      tma_load_2d(smA, &tmap_a, &bars->full_a, 0, rowA);
      uint32_t stage = 0, phase = 0;
      for (int t = 0; t < n_tiles; ++t) {
        mbar_wait(&bars->empty_b[stage], phase ^ 1);
        mbar_arrive_expect_tx(&bars->full_b[stage], kBytesB);
        uint8_t* dst = smB + stage * kBytesB;
        tma_load_2d(dst, &tmap, &bars->full_b[stage], 0, rowB + t * kTileN);
        tma_load_2d(dst + kBytesA, &tmap, &bars->full_b[stage], 0, rowB + t * kTileN + 128);
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else {
    // ===== consumers: MMA, geometric mask, then exact running top-2 of the thread's two rows =====
    const int wg = warp >> 2;
    const int q = lane & 3;
    const int row0 = strip * kTileM + wg * 64 + (warp & 3) * 16 + (lane >> 2);   // rows row0 and row0 + 8
    float M[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) M[k] = g.model[pair * 9 + k];
    const float thr = g.max_residual;
    const float thr_next = __int_as_float(__float_as_int(thr) + 1);   // thr > 0: the next float above
    const double thr_mid = 0.5 * (static_cast<double>(thr) + static_cast<double>(thr_next));
    const bool thr_even = (__float_as_int(thr) & 1) == 0;
    const float2* kcol = g.kpts + p.img_row0[ib];
    // image 1 is pairs[2 * pair], image 2 is pairs[2 * pair + 1]: in direction 1 the rows are image 2
    const int mode = gkind == 0 ? dir : 2;
    float4 rc[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = row0 + 8 * i;
      const float2 kr = (row < nA) ? g.kpts[p.img_row0[ia] + (gathered ? g.gath_cols[static_cast<int64_t>(pair) * p.mstride + row] : row)]
                                   : make_float2(0.f, 0.f);
      rc[i] = (dir == 0) ? side_image1(gkind, M, kr.x, kr.y) : side_image2(gkind, M, kr.x, kr.y);
    }
    int32_t best_d[2] = {0, 0}, best_c[2] = {-1, -1}, second_d[2] = {0, 0};
    uint32_t acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0u;
    if (n_tiles > 0) mbar_wait(&bars->full_a, 0);
    const uint32_t a_addr = smem_u32(smA + wg * 64 * kDim);
    uint32_t stage = 0, phase = 0;
    for (int t = 0; t < n_tiles; ++t) {
      // stage the column side of this tile's 256 columns (one per thread), double-buffered by tile parity
      float4* kb = kp_s + (t & 1) * kTileN;
      for (int c = threadIdx.x; c < kTileN; c += kConsumerWarps * 32) {
        const int j = t * kTileN + c;
        const float2 kc = (j < nB) ? kcol[j] : make_float2(0.f, 0.f);
        kb[c] = (dir == 0) ? side_image2(gkind, M, kc.x, kc.y) : side_image1(gkind, M, kc.x, kc.y);
      }
      asm volatile("bar.sync 1, %0;" ::"r"(kConsumerWarps * 32) : "memory");
      mbar_wait(&bars->full_b[stage], phase);
      uint32_t k1[2] = {0, 0}, k2[2] = {0, 0};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        wgmma_tile_u8(acc, a_addr, smem_u32(smB + stage * kBytesB + h * (kBytesB / 2)));
        if (h == 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&bars->empty_b[stage]);   // the MMAs reading this stage have completed
        }
        const float4* cols = kb + 128 * h;
        if (mode == 0) scan_half<0>(acc, cols, q, 128 * h, rc, thr, thr_next, thr_mid, thr_even, k1, k2);
        else if (mode == 1) scan_half<1>(acc, cols, q, 128 * h, rc, thr, thr_next, thr_mid, thr_even, k1, k2);
        else scan_half<2>(acc, cols, q, 128 * h, rc, thr, thr_next, thr_mid, thr_even, k1, k2);
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        // the four lanes of a quad hold the four column residues of the same row (keys are unique inside a tile)
#pragma unroll
        for (int o = 1; o < 4; o <<= 1)
          merge_top2(k1[i], k2[i], __shfl_xor_sync(0xffffffffu, k1[i], o), __shfl_xor_sync(0xffffffffu, k2[i], o));
        const int32_t d1 = static_cast<int32_t>(k1[i] >> 8);
        const int32_t d2 = static_cast<int32_t>(k2[i] >> 8);
        if (d1 > best_d[i]) {
          second_d[i] = max(best_d[i], d2);
          best_d[i] = d1;
          best_c[i] = t * kTileN + (255 - static_cast<int32_t>(k1[i] & 255u));
        } else {
          second_d[i] = max(second_d[i], d1);
        }
      }
      if (++stage == kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    if (q < 2) {  // lane q of the quad writes row row0 + 8 q
      const int32_t bd = q ? best_d[1] : best_d[0], sd = q ? second_d[1] : second_d[0], bc = q ? best_c[1] : best_c[0];
      int32_t out = -1;
      if (bd > 0) {
        const float a = __ldg(p.acos_lut + min(bd, 262144));
        if (!(a > p.max_distance)) {
          const float b = __ldg(p.acos_lut + min(sd, 262144));
          if (!(a >= __fmul_rn(p.max_ratio, b))) out = bc;
        }
      }
      p.mbuf[(static_cast<int64_t>(pair) * 2 + dir) * p.mstride + row0 + 8 * q] = out;
    }
  }
}

cudaError_t launch_k1_guided(const CUtensorMap& tmap, const MatchParams& p, const GuidedParams& g, int n_pairs,
                             int max_strips, int n_dirs, cudaStream_t stream) {
  // function attributes are per device: several contexts on different GPUs may live in one process
  static bool attr_set[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
  if (!attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(b2m_k1_guided_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(kSmemBytes));
    if (e != cudaSuccess) return e;
    attr_set[dev] = true;
  }
  dim3 grid(max_strips, n_dirs, n_pairs);
  GuidedParams gq = g;
  gq.gath_cnt = nullptr;
  gq.gath_cols = nullptr;
  gq.only_dir = -1;
  b2m_k1_guided_kernel<<<grid, kThreads, kSmemBytes, stream>>>(tmap, tmap, p, gq);
  return cudaGetLastError();
}

// FindBestMatchesBruteForce keeps (i, m12[i]) iff m21[m12[i]] == i: the column direction is consulted at the matched
// columns only (the argument of launch_k1_filter_gather; here the masked matrix is the same for both directions, so it
// carries over unchanged).  Three launches: rows of image 1 against all of image 2; gather; the gathered rows of image
// 2 against all of image 1.  CTAs of the last launch beyond a pair's gathered rows exit at once.
cudaError_t launch_k1_guided_gather(const CUtensorMap& tmap, const CUtensorMap& tmap_gath, const MatchParams& p,
                                    const GuidedParams& g, const uint8_t* desc, int n_pairs, int max_strips,
                                    const GatherScratch& gs, cudaStream_t stream) {
  static bool attr_set[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
  if (!attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(b2m_k1_guided_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(kSmemBytes));
    if (e != cudaSuccess) return e;
    attr_set[dev] = true;
  }
  if (n_pairs <= 0) return cudaSuccess;
  dim3 grid(max_strips, 1, n_pairs);
  GuidedParams g0 = g;
  g0.gath_cnt = nullptr;
  g0.gath_cols = nullptr;
  g0.only_dir = 0;
  b2m_k1_guided_kernel<<<grid, kThreads, kSmemBytes, stream>>>(tmap, tmap, p, g0);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  e = launch_gather_matched_columns(p, desc, n_pairs, gs, g.kind, stream);
  if (e != cudaSuccess) return e;
  GuidedParams g1 = g;
  g1.gath_cnt = gs.cnt;
  g1.gath_cols = gs.cols;
  g1.only_dir = 1;
  b2m_k1_guided_kernel<<<grid, kThreads, kSmemBytes, stream>>>(tmap, tmap_gath, p, g1);
  return cudaGetLastError();
}

}  // namespace b2m
