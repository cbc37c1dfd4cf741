// match_kernel.cu -- K1: fused all-pairs uint8 descriptor GEMM (wgmma.mma_async u8, TMA-staged
// operands, accumulators in registers) + per-row top-2 / lowest-index arg-max / acos-LUT ratio &
// distance tests, and the cross-check + ordered compaction kernel.  The N x M distance matrix
// never leaves the SM.
//
// Semantics follow U:feature/sift.cc (COLMAP 3.9.1) ComputeSiftDistanceMatrix /
// FindBestMatchesOneWayBruteForce / FindBestMatchesBruteForce, reached from
// R:pipeline/match_features.h:45-48 (SURVEY.md section 8 rows M1-M3).
#include "match_kernel.cuh"
#include "ptx.cuh"

namespace b2m {

namespace {

constexpr int kDim = 128;            // descriptor bytes == K of the GEMM
constexpr int kTileM = 128;          // rows of A per CTA: two consumer warpgroups of 64 rows
constexpr int kTileN = 256;          // columns of B per MMA tile
constexpr int kStages = 4;           // B-tile ring depth
constexpr int kBytesA = kTileM * kDim;        // 16 KiB
constexpr int kBytesB = kTileN * kDim;        // 32 KiB
constexpr int kConsumerWarps = 8;             // warpgroups 0 and 1: MMA + epilogue
constexpr int kThreads = (kConsumerWarps + 1) * 32;  // + TMA producer warp

struct __align__(8) Barriers {
  uint64_t full_a;
  uint64_t full_b[kStages];
  uint64_t empty_b[kStages];
};

constexpr size_t kSmemBytes = 1024 /*align slack*/ + kBytesA + kStages * kBytesB + sizeof(Barriers);

// Merge two tile-local (largest, second-largest) key pairs.  Keys are unique inside a tile.
__device__ __forceinline__ void merge_top2(uint32_t& a1, uint32_t& a2, uint32_t b1, uint32_t b2) {
  const uint32_t lo = min(a1, b1);
  a1 = max(a1, b1);
  a2 = max(max(a2, b2), lo);
}

}  // namespace

__global__ void __launch_bounds__(kThreads, 1)
b2m_k1_match_kernel(const __grid_constant__ CUtensorMap tmap, const MatchParams p) {
  const int pair = blockIdx.z;
  const int dir = blockIdx.y;
  const int strip = blockIdx.x;
  const int ia = p.pairs[2 * pair + dir];
  const int ib = p.pairs[2 * pair + (dir ^ 1)];
  const int nA = p.img_nfeat[ia];
  const int nB = p.img_nfeat[ib];
  if (strip * kTileM >= nA) return;  // uniform exit before any barrier
  const int rowA = p.img_row0[ia] + strip * kTileM;
  const int rowB = p.img_row0[ib];
  const int n_tiles = (nB + kTileN - 1) / kTileN;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smA = smem;
  uint8_t* smB = smem + kBytesA;
  Barriers* bars = reinterpret_cast<Barriers*>(smem + kBytesA + kStages * kBytesB);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == kConsumerWarps && lane == 0) {
    tma_prefetch_desc(&tmap);
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
      tma_load_2d(smA, &tmap, &bars->full_a, 0, rowA);
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
    // ===== consumers: warpgroup wg multiplies rows 64 wg .. 64 wg + 63 with each 128-column half of every tile; each
    // thread keeps the running top-2 of its two rows (16 w + l / 4 and + 8) over its 64 columns of the tile
    const int wg = warp >> 2;
    const int q = lane & 3;
    const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    int32_t best_d[2] = {0, 0}, best_c[2] = {-1, -1}, second_d[2] = {0, 0};
    uint32_t acc[64];   // one 128-column half of a tile at a time
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0u;
    if (n_tiles > 0) mbar_wait(&bars->full_a, 0);
    const uint32_t a_addr = smem_u32(smA + wg * 64 * kDim);
    uint32_t stage = 0, phase = 0;
    for (int t = 0; t < n_tiles; ++t) {
      mbar_wait(&bars->full_b[stage], phase);
      uint32_t k1[2] = {0, 0}, k2[2] = {0, 0};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        wgmma_tile_u8(acc, a_addr, smem_u32(smB + stage * kBytesB + h * (kBytesB / 2)));
        if (h == 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&bars->empty_b[stage]);   // the MMAs reading this stage have completed
        }
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int j = 0; j < 16; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              // key = dot * 256 + (255 - local column): max picks the largest dot, lowest column
              const uint32_t key =
                  (acc[4 * j + 2 * i + e] << 8) | static_cast<uint32_t>(255 - (128 * h + 8 * j + 2 * q + e));
              const uint32_t lo = min(k1[i], key);
              k1[i] = max(k1[i], key);
              k2[i] = max(k2[i], lo);
            }
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        // the four lanes of a quad hold the four column residues of the same row
#pragma unroll
        for (int o = 1; o < 4; o <<= 1)
          merge_top2(k1[i], k2[i], __shfl_xor_sync(0xffffffffu, k1[i], o), __shfl_xor_sync(0xffffffffu, k2[i], o));
        const int32_t d1 = static_cast<int32_t>(k1[i] >> 8);
        const int32_t d2 = static_cast<int32_t>(k2[i] >> 8);
        if (d1 > best_d[i]) {  // strict: an equal dot in a later tile never displaces an earlier column
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
    if (q < 2) {  // lane q of the quad writes row q
      const int32_t bd = q ? best_d[1] : best_d[0], sd = q ? second_d[1] : second_d[0], bc = q ? best_c[1] : best_c[0];
      int32_t out = -1;
      if (bd > 0) {
        const float a = __ldg(p.acos_lut + min(bd, 262144));
        if (!(a > p.max_distance)) {
          const float b = __ldg(p.acos_lut + min(sd, 262144));
          if (!(a >= __fmul_rn(p.max_ratio, b))) out = bc;
        }
      }
      p.mbuf[(static_cast<int64_t>(pair) * 2 + dir) * p.mstride + strip * kTileM + row0 + 8 * q] = out;
    }
  }
}

// Cross-check + ordered compaction.  One CTA per pair.  FindBestMatchesBruteForce tail
// (U:feature/sift.cc): keep (i1, m12[i1]) iff m12[i1] != -1 and (no cross-check or
// m21[m12[i1]] == i1); output sorted by i1.
__global__ void __launch_bounds__(256) b2m_crosscheck_compact_kernel(const CompactParams p) {
  const int pair = blockIdx.x;
  const int i1 = p.pairs[2 * pair];
  const int n1 = p.img_nfeat[i1];
  const int32_t* m12 = p.mbuf + (static_cast<int64_t>(pair) * 2) * p.mstride;
  const int32_t* m21 = m12 + p.mstride;
  // gathered column direction: m21 holds one entry per MATCHED column, at the column's rank
  const int32_t* rank = p.colrank ? p.colrank + static_cast<int64_t>(pair) * p.mstride : nullptr;
  auto mutual = [&](int i, int j) { return m21[rank ? rank[j] : j] == i; };
  __shared__ int s_warp[8];
  __shared__ int s_base;
  __shared__ unsigned long long s_off;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (p.enable && p.enable[pair] < 0) {  // guided pass: this pair keeps its verified inliers
    if (threadIdx.x == 0) {
      p.pair_off[pair] = 0;
      p.pair_cnt[pair] = -1;
    }
    return;
  }

  if (p.cand_cnt && p.cand_cnt[2 * pair] == 0) {  // most pairs of an exhaustive batch: nothing matched
    if (threadIdx.x == 0) {
      p.pair_off[pair] = static_cast<int64_t>(atomicAdd(p.cursor, 0ull));
      p.pair_cnt[pair] = 0;
    }
    return;
  }

  // pass 1: count
  int cnt = 0;
  for (int i = threadIdx.x; i < n1; i += 256) {
    const int j = m12[i];
    cnt += (j >= 0 && (!p.cross_check || mutual(i, j))) ? 1 : 0;
  }
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) s_warp[warp] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int total = 0;
    for (int w = 0; w < 8; ++w) total += s_warp[w];
    s_off = atomicAdd(p.cursor, static_cast<unsigned long long>(total));
    p.pair_off[pair] = static_cast<int64_t>(s_off);
    p.pair_cnt[pair] = total;
    s_base = 0;
    s_warp[0] = total;
  }
  __syncthreads();
  if (s_warp[0] == 0) return;   // uniform: nothing to write
  __syncthreads();              // s_warp is reused by the ordered write
  uint2* out = p.arena + s_off;

  // pass 2: ordered write
  for (int i0 = 0; i0 < n1; i0 += 256) {
    const int i = i0 + threadIdx.x;
    int j = -1;
    bool keep = false;
    if (i < n1) {
      j = m12[i];
      keep = (j >= 0 && (!p.cross_check || mutual(i, j)));
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    const int wpre = __popc(ballot & ((1u << lane) - 1u));
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    int base = s_base;
    for (int w = 0; w < warp; ++w) base += s_warp[w];
    if (keep) {
      out[base + wpre] = make_uint2(static_cast<unsigned>(i), static_cast<unsigned>(j));
      if (p.pts) {  // matched pixel coordinates for the verifier (keypoints are float32, exact in double)
        const float2 a = p.kpts[p.img_row0[i1] + i];
        const float2 b = p.kpts[p.img_row0[p.pairs[2 * pair + 1]] + j];
        p.pts[s_off + base + wpre] = make_double4(a.x, a.y, b.x, b.y);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int total = 0;
      for (int w = 0; w < 8; ++w) total += s_warp[w];
      s_base += total;
    }
    __syncthreads();
  }
}

cudaError_t launch_k1_match(const CUtensorMap& tmap, const MatchParams& p, int n_pairs, int max_strips, int n_dirs,
                            cudaStream_t stream) {
  // function attributes are per device: several contexts on different GPUs may live in one process
  static bool attr_set[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
  if (!attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(b2m_k1_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(kSmemBytes));
    if (e != cudaSuccess) return e;
    attr_set[dev] = true;
  }
  dim3 grid(max_strips, n_dirs, n_pairs);
  b2m_k1_match_kernel<<<grid, kThreads, kSmemBytes, stream>>>(tmap, p);
  return cudaGetLastError();
}

cudaError_t launch_crosscheck_compact(const CompactParams& p, int n_pairs, cudaStream_t stream) {
  b2m_crosscheck_compact_kernel<<<n_pairs, 256, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace b2m
