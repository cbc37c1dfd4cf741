// match_filter_kernel.cu -- K1: persistent wgmma int8 GEMM with a *filter* epilogue, plus the exact
// resolve kernel.
//
// Grid = one CTA per SM, persistent: every CTA walks a static list of work units (image pair, direction,
// 256-row block of the "row" image A, 128-row half of that block).
//   * Two consumer warpgroups each issue wgmma.mma_async m64n128k32 (u8 x u8 -> s32) for their 64 rows of
//     the unit against each half of every 256-column tile of image B (four k-steps per half), accumulators in
//     registers.  Halves rather than one m64n256 keep the 64 accumulators and the 32 slot maxima of a thread
//     within the register budget of 288 threads per SM without spills.
//   * One producer warp streams B through a 4-stage ring of 32 KiB tiles (TMA, SWIZZLE_128B) and the A
//     strips through two buffers, so the pipeline runs straight across unit boundaries; barriers are set up
//     once per launch.
//   * While one warpgroup folds its accumulators the other one can use the tensor cores.
//
// Filter: instead of an exact running top-2 (4 ALU ops per accumulator) each row keeps 64 "slot maxima".
// Thread lane l of a quad (q = l % 4) holds the columns 8 j + 2 q + e (j = 0..31, e = 0, 1) of its rows; its
// slot r = 2 (j % 8) + e collects the four columns j = r / 2 + 8 c, c = 0..3, of every tile:
//     slot(16 q + r) = max over columns 256 t + 64 c + 8 (r >> 1) + 2 q + (r & 1)     (c = 0..3, all tiles t)
// At the end of the row
//     best = max over slots (exact);   S1 = second largest slot maximum (multiset), which is a LOWER
//     bound of the true second-best (= max(S1, second largest element inside the winning slot)).
// acos is monotone, so a row failing `acos(best) <= max_distance`, or failing the ratio test already
// against S1, is rejected exactly.  The survivors ("candidates": essentially the true matches) are
// resolved exactly by b2m_k1_resolve_kernel: it recomputes the n2/64 dot products of the winning slot
// with dp4a (all columns if several slots share the maximum), finds the lowest-index arg-max and the
// hidden second-best, and applies the float32 test of FindBestMatchesOneWayBruteForce.  The match
// indices are bit-identical to the exact kernel (match_kernel.cu) and to the CPU oracle.
//
// Semantics: U:feature/sift.cc (COLMAP 3.9.1), SURVEY.md section 8 rows M1-M3.
#include <cstdio>
#include "match_kernel.cuh"
#include "ptx.cuh"

namespace b2m {

namespace {

constexpr int kDim = 128;
constexpr int kTileM = 128;                        // rows per work unit: two consumer warpgroups of 64 rows
constexpr int kRowsPerItem = 256;                  // rows of A per work item (two units) == kRowPad
constexpr int kTileN = 256;                        // columns per B tile (the N of one wgmma)
constexpr int kStages = 4;                         // B-tile ring depth
constexpr int kABufs = 2;                          // A strips double-buffered across work units
constexpr int kBytesA = kTileM * kDim;             // 16 KiB per strip
constexpr int kBytesB = kTileN * kDim;             // 32 KiB per B tile
constexpr int kConsumerWarps = 8;
constexpr int kOwnSlots = 16;                      // slot maxima per row kept in one thread's registers
constexpr int kSlots = kOwnSlots * 4;              // 64 slot maxima per row (four lanes of a quad)
constexpr int kThreads = (kConsumerWarps + 1) * 32;  // + TMA producer warp
static_assert(kRowsPerItem == kRowPad && kTileN == kRowPad, "images are padded to whole items / column tiles");

struct __align__(8) Barriers {
  uint64_t full_a[kABufs];
  uint64_t empty_a[kABufs];
  uint64_t full_b[kStages];
  uint64_t empty_b[kStages];
};

constexpr size_t kSmemBytes = 1024 + kABufs * kBytesA + kStages * kBytesB + sizeof(Barriers);

// A work unit and the data every warp role derives from its index (pure function of `w` and `half`).
struct Item {
  int pair, dir, nA, nB, rowA, rowB, n_tiles, row0;  // row0: first row (inside image A) of this unit
  bool valid;
};
__device__ __forceinline__ Item decode_item(const MatchParams& p, int w, int half) {
  Item it;
  if (p.item_list) {
    // gathered column direction: rows = the gathered block of the pair (scratch tensor map), columns = image a
    it.pair = p.item_list[2 * w];
    const int cb = p.item_list[2 * w + 1];
    it.dir = 0;
    const int ib = p.pairs[2 * it.pair];
    it.nA = p.gath_cnt[it.pair];
    it.nB = p.img_nfeat[ib];
    it.valid = cb * kRowsPerItem < it.nA;
    it.row0 = cb * kRowsPerItem + half * kTileM;
    it.rowA = it.pair * p.mstride + it.row0;
    it.rowB = p.img_row0[ib];
    it.n_tiles = (it.nB + kTileN - 1) / kTileN;
    return it;
  }
  const int cb = w % p.blocks_per_image;
  const int pd = w / p.blocks_per_image;
  it.dir = pd % p.n_dirs;
  it.pair = pd / p.n_dirs;
  const int ia = p.pairs[2 * it.pair + it.dir];
  const int ib = p.pairs[2 * it.pair + (it.dir ^ 1)];
  it.nA = p.img_nfeat[ia];
  it.nB = p.img_nfeat[ib];
  // same answer for both halves of an item; an empty image B still yields a unit (n_tiles == 0)
  // so that its rows are written as "no match"
  it.valid = cb * kRowsPerItem < it.nA;
  it.row0 = cb * kRowsPerItem + half * kTileM;
  it.rowA = p.img_row0[ia] + it.row0;
  it.rowB = p.img_row0[ib];
  it.n_tiles = (it.nB + kTileN - 1) / kTileN;
  return it;
}

}  // namespace

__global__ void __launch_bounds__(kThreads, 1)
b2m_k1_filter_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmap_a,
                     const MatchParams p) {
  // tmap: the resident descriptor set (column tiles; row strips too unless the rows are gathered), tmap_a: the row
  // strips (== tmap except for the gathered column direction, where it covers the gather scratch)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smA = smem;                                     // [kABufs][16 KiB]
  uint8_t* smB = smem + kABufs * kBytesA;                  // [kStages][32 KiB]
  Barriers* bars = reinterpret_cast<Barriers*>(smB + kStages * kBytesB);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // gathered column direction: the work list was built on the device, so was its length
  const int n_units = 2 * (p.item_list ? __ldg(p.n_items_ptr) : p.n_items);

  if (warp == kConsumerWarps && lane == 0) {
    tma_prefetch_desc(&tmap);
    tma_prefetch_desc(&tmap_a);
    for (int s = 0; s < kABufs; ++s) {
      mbar_init(&bars->full_a[s], 1);
      mbar_init(&bars->empty_a[s], kConsumerWarps);
    }
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&bars->full_b[s], 1);
      mbar_init(&bars->empty_b[s], kConsumerWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ===== TMA producer (one lane) =====
    if (lane == 0) {
      uint32_t stage = 0, phase = 0, n_done = 0;
      for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
        const Item it = decode_item(p, u >> 1, u & 1);
        if (!it.valid || it.n_tiles == 0) continue;
        const uint32_t ab = n_done & 1, aph = (n_done >> 1) & 1;
        ++n_done;
        mbar_wait(&bars->empty_a[ab], aph ^ 1);  // the MMAs of the unit that used this A buffer completed
        mbar_arrive_expect_tx(&bars->full_a[ab], kBytesA);
        tma_load_2d(smA + ab * kBytesA, &tmap_a, &bars->full_a[ab], 0, it.rowA);
        for (int t = 0; t < it.n_tiles; ++t) {
          mbar_wait(&bars->empty_b[stage], phase ^ 1);
          mbar_arrive_expect_tx(&bars->full_b[stage], kBytesB);
          uint8_t* dst = smB + stage * kBytesB;
          tma_load_2d(dst, &tmap, &bars->full_b[stage], 0, it.rowB + t * kTileN);
          tma_load_2d(dst + kBytesA, &tmap, &bars->full_b[stage], 0, it.rowB + t * kTileN + 128);
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===== consumers: MMA + filter epilogue =====
    const int wg = warp >> 2;
    const int q = lane & 3;
    const int row_in_unit = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // rows row_in_unit and row_in_unit + 8
    uint32_t acc[64];   // one 128-column half of a tile at a time: the slot maxima stay in registers beside it
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0u;
    uint32_t stage = 0, phase = 0, n_done = 0;
    for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
      const Item it = decode_item(p, u >> 1, u & 1);
      if (!it.valid) continue;
      uint32_t S[2][kOwnSlots];   // slot maxima of the thread's two rows
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int r = 0; r < kOwnSlots; ++r) S[i][r] = 0u;
      if (it.n_tiles > 0) {
        const uint32_t ab = n_done & 1, aph = (n_done >> 1) & 1;
        ++n_done;
        mbar_wait(&bars->full_a[ab], aph);
        const uint32_t a_addr = smem_u32(smA + ab * kBytesA + wg * 64 * kDim);
#pragma unroll 1
        for (int t = 0; t < it.n_tiles; ++t) {
          mbar_wait(&bars->full_b[stage], phase);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            wgmma_tile_u8(acc, a_addr, smem_u32(smB + stage * kBytesB + h * (kBytesB / 2)));
            if (h == 1) {
              __syncwarp();
              if (lane == 0) mbar_arrive(&bars->empty_b[stage]);   // the MMAs reading this stage have completed
            }
            // column 128 h + 8 j + 2 q + e (acc[4 j + 2 i + e], j < 16) = 64 c + 8 (r >> 1) + 2 q + (r & 1) with
            // c = 2 h + j / 8, r = 2 (j % 8) + e
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
              for (int r = 0; r < kOwnSlots; ++r) {
                const int a0 = 4 * (r >> 1) + 2 * i + (r & 1);
                S[i][r] = max(S[i][r], max(acc[a0], acc[a0 + 32]));
              }
          }
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
        if (lane == 0) mbar_arrive(&bars->empty_a[ab]);
      }
      // (largest, second largest) over the 64 slot maxima of each row, multiset semantics, lowest slot id on ties:
      // the thread's 16 slots first, then the four lanes of the quad (slot ids 16 q + r)
      uint32_t best[2], s1[2];
      int sstar[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        best[i] = 0u;
        s1[i] = 0u;
        sstar[i] = 0;
#pragma unroll
        for (int r = 0; r < kOwnSlots; ++r) {
          const uint32_t v = S[i][r];
          if (v > best[i]) {
            s1[i] = best[i];
            best[i] = v;
            sstar[i] = 16 * q + r;
          } else {
            s1[i] = max(s1[i], v);
          }
        }
#pragma unroll
        for (int o = 1; o < 4; o <<= 1) {
          const uint32_t ob = __shfl_xor_sync(0xffffffffu, best[i], o);
          const uint32_t os = __shfl_xor_sync(0xffffffffu, s1[i], o);
          const int oslot = __shfl_xor_sync(0xffffffffu, sstar[i], o);
          const uint32_t ns = max(max(s1[i], os), min(best[i], ob));
          if (ob > best[i] || (ob == best[i] && oslot < sstar[i])) {
            best[i] = ob;
            sstar[i] = oslot;
          }
          s1[i] = ns;
        }
      }
      if (q < 2) {   // lane q of the quad decides row row_in_unit + 8 q
        const uint32_t b = q ? best[1] : best[0], s = q ? s1[1] : s1[0];
        const int slot = q ? sstar[1] : sstar[0];
        const float fa = __ldg(p.acos_lut + min(b, 262144u));
        const float fb = __ldg(p.acos_lut + min(s, 262144u));
        int32_t out = -1;
        if (b > 0u && !(fa > p.max_distance) && !(fa >= __fmul_rn(p.max_ratio, fb)))
          out = -2 - slot;  // candidate: resolve exactly
        const int64_t base = (static_cast<int64_t>(it.pair) * 2 + it.dir) * p.mstride;
        const int row = it.row0 + row_in_unit + 8 * q;
        p.mbuf[base + row] = out;
        if (out != -1 && row < it.nA) {
          p.aux[base + row] = make_uint2(b, s);
          const int k = atomicAdd(p.cand_cnt + it.pair * 2 + it.dir, 1);
          p.cand_rows[base + k] = row | (slot << 24);  // winning slot travels with the row
        }
      }
    }
  }
}

// Exact resolution of the candidate rows of one (pair, direction).
// Slot s = 16 q + r holds the columns j = 256 t + 64 c + 8 (r >> 1) + 2 q + (r & 1), c = 0..3, t = 0, 1, ... (slot_col
// below).
// Candidates are bucketed by winning slot (counting sort in shared memory) so that the n2/64 columns
// of a slot are staged in shared memory ONCE and reused by every candidate of the bucket (a warp per
// candidate, dp4a, oracle scan order per lane, multiset-aware merge across lanes).  Rows whose
// maximum is shared by several slots, and images with more than 16384 features, take the generic
// path that scans global memory.
namespace {

constexpr int kSlotColsMax = 256;      // columns of one slot staged in shared memory (images up to 16384 features)
constexpr int kResolveParts = 4;       // CTAs per (pair, direction); 1/2/4/8 measured within 1.5 % of each other
constexpr int kSlotRowStride = 144;    // bytes; 128-byte descriptors padded so that LDS.128 is conflict-free

// `it`-th column (ascending) of a slot: four columns in every 256-column tile
__device__ __forceinline__ int slot_col(int slot, int it) {
  return 256 * (it >> 2) + 64 * (it & 3) + 8 * ((slot & 15) >> 1) + 2 * (slot >> 4) + (slot & 1);
}

__device__ __forceinline__ uint32_t dot128(const uint32_t (&a)[32], const uint4* bp) {
  uint32_t d = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const uint4 v = bp[q];
    d = __dp4a(a[4 * q], v.x, d);
    d = __dp4a(a[4 * q + 1], v.y, d);
    d = __dp4a(a[4 * q + 2], v.z, d);
    d = __dp4a(a[4 * q + 3], v.w, d);
  }
  return d;
}

__device__ __forceinline__ void scan_update(uint32_t d, int j, uint32_t& bd, uint32_t& sd, int& bj) {
  if (d > bd) {
    sd = bd;
    bd = d;
    bj = j;
  } else if (d > sd) {
    sd = d;
  }
}

// merge the per-lane scans and take the exact accept decision (lane 0 writes)
__device__ __forceinline__ void finish_candidate(const MatchParams& p, int64_t out_index, uint32_t bd, uint32_t sd,
                                                 int bj, uint32_t best_f, uint32_t s1, bool multi, int lane) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const uint32_t obd = __shfl_xor_sync(0xffffffffu, bd, o);
    const uint32_t osd = __shfl_xor_sync(0xffffffffu, sd, o);
    const int obj = __shfl_xor_sync(0xffffffffu, bj, o);
    const uint32_t nsd = max(max(sd, osd), min(bd, obd));
    if (obd > bd || (obd == bd && obj >= 0 && (bj < 0 || obj < bj))) {
      bd = obd;
      bj = obj;
    }
    sd = nsd;
  }
  if (lane == 0) {
    const uint32_t second = multi ? sd : max(sd, s1);
    int32_t out = -1;
    if (bd > 0u && bd == best_f) {
      const float fa = __ldg(p.acos_lut + min(bd, 262144u));
      if (!(fa > p.max_distance)) {
        const float fb = __ldg(p.acos_lut + min(second, 262144u));
        if (!(fa >= __fmul_rn(p.max_ratio, fb))) out = bj;
      }
    }
    p.mbuf[out_index] = out;
  }
}

}  // namespace

// dir_only < 0: grid = 2 x n_pairs x kResolveParts, both directions; 0 / 1: grid = n_pairs x kResolveParts, that
// direction only.  With p.gath_desc the rows of direction 1 are the pair's GATHERED descriptors (of image b) and its
// columns are image a (launch_k1_filter_gather).
__global__ void __launch_bounds__(256) b2m_k1_resolve_kernel(const MatchParams p, const uint8_t* __restrict__ desc,
                                                             const int dir_only) {
  // kResolveParts CTAs share the candidates of one (pair, direction): part k takes the slots == k mod
  // kResolveParts (and the rows == k mod kResolveParts of the unstaged candidates), which cuts the
  // serial chain "stage a slot, score its candidates" of a true-match pair by that factor.
  const int part = blockIdx.x % kResolveParts;
  const int pd = blockIdx.x / kResolveParts;
  const int pair = dir_only < 0 ? pd >> 1 : pd;
  const int dir = dir_only < 0 ? pd & 1 : dir_only;
  const int n_cand = p.cand_cnt[pair * 2 + dir];
  if (n_cand == 0) return;
  const bool gathered = dir == 1 && p.gath_desc != nullptr;
  const int ia = p.pairs[2 * pair + dir];
  const int ib = gathered ? p.pairs[2 * pair] : p.pairs[2 * pair + (dir ^ 1)];
  const int nB = p.img_nfeat[ib];
  const int nB_pad = (nB + kRowPad - 1) / kRowPad * kRowPad;
  const uint8_t* A = gathered ? p.gath_desc + static_cast<int64_t>(pair) * p.mstride * kDim
                              : desc + static_cast<int64_t>(p.img_row0[ia]) * kDim;
  const uint8_t* Bm = desc + static_cast<int64_t>(p.img_row0[ib]) * kDim;
  const int64_t base = (static_cast<int64_t>(pair) * 2 + dir) * p.mstride;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_items = nB_pad / kSlots;
  const bool staged = n_items <= kSlotColsMax;

  __shared__ int s_start[kSlots + 1];
  __shared__ int s_fill[kSlots];
  __shared__ __align__(16) uint8_t s_cols[kSlotColsMax * kSlotRowStride];

  // candidate entry = row | slot << 24 (written by the selector warp); a candidate whose maximum is shared
  // by several slots, or any candidate of an image too large for the staging buffer, is "unstaged"
  auto bucket_of = [&](int entry) {
    const uint2 ax = p.aux[base + (entry & 0xFFFFFF)];
    return (ax.x == ax.y || !staged) ? kSlots : (entry >> 24);
  };

  // ---- counting sort of this part's staged candidates by slot
  for (int b = threadIdx.x; b < kSlots; b += 256) s_fill[b] = 0;
  __syncthreads();
  for (int c = threadIdx.x; c < n_cand; c += 256) {
    const int bucket = bucket_of(p.cand_rows[base + c]);
    if (bucket < kSlots) atomicAdd(&s_fill[bucket], 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int b = 0; b < kSlots; ++b) {  // same offsets in every part: the parts write disjoint ranges
      s_start[b] = acc;
      acc += s_fill[b];
      s_fill[b] = 0;
    }
    s_start[kSlots] = acc;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < n_cand; c += 256) {
    const int entry = p.cand_rows[base + c];
    const int bucket = bucket_of(entry);
    if (bucket < kSlots && bucket % kResolveParts == part)
      p.cand_sorted[base + s_start[bucket] + atomicAdd(&s_fill[bucket], 1)] = entry & 0xFFFFFF;
  }
  __syncthreads();

  // ---- staged slots of this part
  for (int b = part; b < kSlots; b += kResolveParts) {
    const int c0 = s_start[b], c1 = s_start[b + 1];
    if (c0 == c1) continue;  // uniform
    __syncthreads();  // previous slot's readers are done with s_cols
    for (int q = threadIdx.x; q < n_items * 8; q += 256) {
      const int it = q >> 3, seg = q & 7;
      const int j = slot_col(b, it);
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(Bm + static_cast<int64_t>(j) * kDim) + seg);
      *reinterpret_cast<uint4*>(s_cols + it * kSlotRowStride + seg * 16) = v;
    }
    __syncthreads();
    for (int c = c0 + warp; c < c1; c += 8) {
      const int row = p.cand_sorted[base + c];
      const uint2 ax = p.aux[base + row];
      uint32_t a[32];
      const uint4* ap = reinterpret_cast<const uint4*>(A + static_cast<int64_t>(row) * kDim);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const uint4 v = __ldg(ap + q);
        a[4 * q] = v.x; a[4 * q + 1] = v.y; a[4 * q + 2] = v.z; a[4 * q + 3] = v.w;
      }
      uint32_t bd = 0, sd = 0;
      int bj = -1;
      for (int it = lane; it < n_items; it += 32) {
        const int j = slot_col(b, it);
        const uint32_t d = dot128(a, reinterpret_cast<const uint4*>(s_cols + it * kSlotRowStride));
        scan_update(d, j, bd, sd, bj);
      }
      finish_candidate(p, base + row, bd, sd, bj, ax.x, ax.y, false, lane);
    }
  }

  // ---- unstaged candidates of this part: scan global memory (whole row if several slots share the maximum)
  for (int c = warp; c < n_cand; c += 8) {
    const int entry = p.cand_rows[base + c];
    const int row = entry & 0xFFFFFF;
    if (row % kResolveParts != part) continue;  // uniform in the warp
    const uint2 ax = p.aux[base + row];
    const bool multi = (ax.x == ax.y);
    if (!multi && staged) continue;
    const int slot = entry >> 24;
    uint32_t a[32];
    const uint4* ap = reinterpret_cast<const uint4*>(A + static_cast<int64_t>(row) * kDim);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const uint4 v = __ldg(ap + q);
      a[4 * q] = v.x; a[4 * q + 1] = v.y; a[4 * q + 2] = v.z; a[4 * q + 3] = v.w;
    }
    uint32_t bd = 0, sd = 0;
    int bj = -1;
    const int n_scan = multi ? nB_pad : n_items;
    for (int it = lane; it < n_scan; it += 32) {
      const int j = multi ? it : slot_col(slot, it);
      const uint32_t d = dot128(a, reinterpret_cast<const uint4*>(Bm + static_cast<int64_t>(j) * kDim));
      scan_update(d, j, bd, sd, bj);
    }
    finish_candidate(p, base + row, bd, sd, bj, ax.x, ax.y, multi, lane);
  }
}

cudaError_t launch_k1_filter(const CUtensorMap& tmap, const MatchParams& p_in,
                             const uint8_t* desc, int n_pairs, int max_strips, int n_dirs, int num_sms,
                             cudaStream_t stream, cudaEvent_t after_filter) {
  // function attributes are per device: several contexts on different GPUs may live in one process
  static bool attr_set[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
  if (!attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(b2m_k1_filter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(kSmemBytes));
    if (e != cudaSuccess) return e;
    attr_set[dev] = true;
  }
  MatchParams p = p_in;
  cudaError_t e = cudaMemsetAsync(p.cand_cnt, 0, sizeof(int32_t) * 2 * n_pairs, stream);
  if (e != cudaSuccess) return e;
  // rows never visited by a work item (dir 1 without cross-check is simply not produced)
  p.n_dirs = n_dirs;
  p.blocks_per_image = (max_strips * kTileM + kRowsPerItem - 1) / kRowsPerItem;
  p.n_items = n_pairs * n_dirs * p.blocks_per_image;
  const int ctas = 2 * p.n_items < num_sms ? 2 * p.n_items : num_sms;
  if (ctas > 0) {
    b2m_k1_filter_kernel<<<ctas, kThreads, kSmemBytes, stream>>>(tmap, tmap, p);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  if (after_filter) {
    e = cudaEventRecord(after_filter, stream);  // the roofline times the GEMM kernel alone
    if (e != cudaSuccess) return e;
  }
  b2m_k1_resolve_kernel<<<2 * n_pairs * kResolveParts, 256, 0, stream>>>(p, desc, -1);
  return cudaGetLastError();
}

namespace {
// live pair -> (b, a): the column direction becomes the row direction of the swapped pair; dead pair -> dummy
__global__ void b2m_k1_select_dir1_kernel(const int32_t* __restrict__ pairs, const int32_t* __restrict__ cand_cnt,
                                          int n_pairs, int dummy, int32_t* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_pairs) return;
  const bool live = cand_cnt[2 * k] > 0;
  out[2 * k] = live ? pairs[2 * k + 1] : dummy;
  out[2 * k + 1] = live ? pairs[2 * k] : dummy;
}

__global__ void b2m_compare_matches_kernel(const uint2* __restrict__ arena_a, const int64_t* __restrict__ off_a,
                                           const int32_t* __restrict__ cnt_a, const uint2* __restrict__ arena_b,
                                           const int64_t* __restrict__ off_b, const int32_t* __restrict__ cnt_b,
                                           int32_t* mismatch) {
  const int pair = blockIdx.x;
  const int n = cnt_a[pair];
  if (n != cnt_b[pair]) {
    if (threadIdx.x == 0) atomicOr(mismatch, 1);
    return;
  }
  const uint2* a = arena_a + off_a[pair];
  const uint2* b = arena_b + off_b[pair];
  bool bad = false;
  for (int i = threadIdx.x; i < n; i += blockDim.x) bad = bad || a[i].x != b[i].x || a[i].y != b[i].y;
  if (bad) atomicOr(mismatch, 2);
}
}  // namespace

cudaError_t launch_k1_filter_skip(const CUtensorMap& tmap, const MatchParams& p_in, const uint8_t* desc, int n_pairs,
                                  int max_strips, int num_sms, int32_t* pairs_scratch, int dummy_image,
                                  cudaStream_t stream, cudaEvent_t after_filter) {
  static bool attr_set[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
  if (!attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(b2m_k1_filter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(kSmemBytes));
    if (e != cudaSuccess) return e;
    attr_set[dev] = true;
  }
  if (n_pairs <= 0) return cudaSuccess;
  MatchParams p = p_in;
  cudaError_t e = cudaMemsetAsync(p.cand_cnt, 0, sizeof(int32_t) * 2 * n_pairs, stream);
  if (e != cudaSuccess) return e;
  p.n_dirs = 1;
  p.blocks_per_image = (max_strips * kTileM + kRowsPerItem - 1) / kRowsPerItem;
  p.n_items = n_pairs * p.blocks_per_image;
  const int ctas = 2 * p.n_items < num_sms ? 2 * p.n_items : num_sms;
  if (ctas > 0) {
    // 1. row direction of every pair
    b2m_k1_filter_kernel<<<ctas, kThreads, kSmemBytes, stream>>>(tmap, tmap, p);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    // 2. live pairs swapped, dead pairs -> dummy image (0 features: every work item invalid)
    b2m_k1_select_dir1_kernel<<<(n_pairs + 255) / 256, 256, 0, stream>>>(p.pairs, p.cand_cnt, n_pairs, dummy_image,
                                                                       pairs_scratch);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    // 3. column direction of the live pairs = row direction of the swapped pairs, written to the
    //    direction-1 halves: every index in the kernel is (pair * 2 + dir) * mstride (+ row) with dir = 0
    MatchParams q = p;
    q.pairs = pairs_scratch;
    q.mbuf = p.mbuf + p.mstride;
    q.aux = p.aux + p.mstride;
    q.cand_cnt = p.cand_cnt + 1;
    q.cand_rows = p.cand_rows + p.mstride;
    q.cand_sorted = p.cand_sorted + p.mstride;
    b2m_k1_filter_kernel<<<ctas, kThreads, kSmemBytes, stream>>>(tmap, tmap, q);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  if (after_filter) {
    e = cudaEventRecord(after_filter, stream);
    if (e != cudaSuccess) return e;
  }
  // 4. exact resolution of both directions (original pair list and base pointers)
  b2m_k1_resolve_kernel<<<2 * n_pairs * kResolveParts, 256, 0, stream>>>(p, desc, -1);
  return cudaGetLastError();
}

namespace {
// Gathered column direction, step 3 (see match_kernel.cuh): one CTA per pair.  The distinct columns some row of image
// a matched (m12 >= 0 after the exact resolve) are ranked ascending; rank, column list, gathered descriptors (padded
// with zero rows to a multiple of 256) and one work item per 256 gathered rows are written.
constexpr int kGatherMaxWords = 1024;  // columns / 32: images up to 32768 features (SiftMatchingOptions.max_num_matches)
__global__ void __launch_bounds__(256) b2m_k1_gather_kernel(const MatchParams p, const uint8_t* __restrict__ desc,
                                                            uint8_t* __restrict__ gdesc, int32_t* __restrict__ colrank,
                                                            int32_t* __restrict__ cols, int32_t* __restrict__ gcnt,
                                                            int32_t* __restrict__ items, int32_t* __restrict__ n_items,
                                                            const int32_t* __restrict__ enable) {
  const int pair = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __shared__ uint32_t s_bits[kGatherMaxWords];
  __shared__ int s_pref[kGatherMaxWords];
  __shared__ int s_warp[8], s_total, s_item0;
  // no candidate, hence no match: the column direction is never consulted (K1); guided matching: pair not eligible
  if (enable ? enable[pair] < 0 : p.cand_cnt[2 * pair] == 0) {
    if (tid == 0) gcnt[pair] = 0;
    return;
  }
  const int ia = p.pairs[2 * pair], ib = p.pairs[2 * pair + 1];
  const int nA = p.img_nfeat[ia], nB = p.img_nfeat[ib];
  const int n_words = (nB + 31) >> 5;
  const int64_t base = static_cast<int64_t>(pair) * p.mstride;
  const int32_t* m12 = p.mbuf + 2 * base;
  for (int w = tid; w < n_words; w += 256) s_bits[w] = 0u;
  __syncthreads();
  for (int i = tid; i < nA; i += 256) {
    const int j = m12[i];
    if (j >= 0) atomicOr(&s_bits[j >> 5], 1u << (j & 31));
  }
  __syncthreads();
  // exclusive prefix of the per-word popcounts (each thread owns a contiguous run of words)
  const int per = (n_words + 255) / 256;
  const int w0 = min(n_words, tid * per), w1 = min(n_words, w0 + per);
  int local = 0;
  for (int w = w0; w < w1; ++w) local += __popc(s_bits[w]);
  int incl = local;
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (tid == 0) {
    int acc = 0;
    for (int k = 0; k < 8; ++k) {
      const int v = s_warp[k];
      s_warp[k] = acc;
      acc += v;
    }
    s_total = acc;
    const int n_blocks = (acc + kRowPad - 1) / kRowPad;
    s_item0 = n_blocks > 0 ? atomicAdd(n_items, n_blocks) : 0;
    gcnt[pair] = acc;
  }
  __syncthreads();
  {
    int run = s_warp[warp] + incl - local;
    for (int w = w0; w < w1; ++w) {
      s_pref[w] = run;
      run += __popc(s_bits[w]);
    }
  }
  __syncthreads();
  const int nc = s_total;
  const int nc_pad = (nc + kRowPad - 1) / kRowPad * kRowPad;
  for (int t = tid; t < nc_pad / kRowPad; t += 256) {
    items[2 * (s_item0 + t)] = pair;
    items[2 * (s_item0 + t) + 1] = t;
  }
  for (int w = tid; w < n_words; w += 256) {
    uint32_t bits = s_bits[w];
    int r = s_pref[w];
    while (bits) {
      const int b = __ffs(bits) - 1;
      bits &= bits - 1;
      const int j = (w << 5) + b;
      colrank[base + j] = r;
      cols[base + r] = j;
      ++r;
    }
  }
  __syncthreads();   // cols[] of this CTA are visible to its own threads after the barrier (same block: global writes + __syncthreads)
  const uint4* src0 = reinterpret_cast<const uint4*>(desc + static_cast<int64_t>(p.img_row0[ib]) * kDim);
  uint4* dst0 = reinterpret_cast<uint4*>(gdesc + base * kDim);
  for (int q = tid; q < nc_pad * 8; q += 256) {
    const int r = q >> 3, seg = q & 7;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (r < nc) v = __ldg(src0 + static_cast<int64_t>(cols[base + r]) * 8 + seg);
    dst0[static_cast<int64_t>(r) * 8 + seg] = v;
  }
}
}  // namespace

// One phase of the gathered schedule (see match_kernel.cuh).  Phases of a batch must be enqueued in order 0, 1, 2, 3 on
// streams ordered by events; splitting them lets the scheduler run phase 1 (ALU kernels that need little of an SM)
// next to the previous batch's RANSAC kernels instead of in front of them.
//   0: row-direction GEMM over all pairs        1: its exact resolve (m12) + gather of the matched columns
//   2: GEMM over the gathered work list          3: exact resolve of the gathered direction
cudaError_t launch_k1_gather_phase(int phase, const CUtensorMap& tmap, const CUtensorMap& tmap_gath, const MatchParams& p_in,
                                   const uint8_t* desc, int n_pairs, int max_strips, int num_sms, const GatherScratch& g,
                                   cudaStream_t stream) {
  static bool attr_set[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
  if (!attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(b2m_k1_filter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(kSmemBytes));
    if (e != cudaSuccess) return e;
    attr_set[dev] = true;
  }
  if (n_pairs <= 0) return cudaSuccess;
  MatchParams p = p_in;
  p.n_dirs = 1;
  p.blocks_per_image = (max_strips * kTileM + kRowsPerItem - 1) / kRowsPerItem;
  p.n_items = n_pairs * p.blocks_per_image;
  p.item_list = nullptr;
  p.gath_desc = nullptr;
  const int ctas = 2 * p.n_items < num_sms ? 2 * p.n_items : num_sms;
  if (ctas <= 0) return cudaSuccess;
  cudaError_t e = cudaSuccess;
  switch (phase) {
    case 0:
      e = cudaMemsetAsync(p.cand_cnt, 0, sizeof(int32_t) * 2 * n_pairs, stream);
      if (e != cudaSuccess) return e;
      e = cudaMemsetAsync(g.n_items, 0, sizeof(int32_t), stream);
      if (e != cudaSuccess) return e;
      b2m_k1_filter_kernel<<<ctas, kThreads, kSmemBytes, stream>>>(tmap, tmap, p);
      break;
    case 1:
      b2m_k1_resolve_kernel<<<n_pairs * kResolveParts, 256, 0, stream>>>(p, desc, 0);
      b2m_k1_gather_kernel<<<n_pairs, 256, 0, stream>>>(p, desc, g.desc, g.colrank, g.cols, g.cnt, g.items, g.n_items, nullptr);
      break;
    case 2: {
      // rows = gathered descriptors, columns = image a; outputs go to the direction-1 halves (every index in the
      // kernel is (pair * 2 + dir) * mstride + row with dir = 0)
      MatchParams q = p;
      q.mbuf = p.mbuf + p.mstride;
      q.aux = p.aux + p.mstride;
      q.cand_cnt = p.cand_cnt + 1;
      q.cand_rows = p.cand_rows + p.mstride;
      q.cand_sorted = p.cand_sorted + p.mstride;
      q.item_list = g.items;
      q.n_items_ptr = g.n_items;
      q.gath_cnt = g.cnt;
      b2m_k1_filter_kernel<<<num_sms, kThreads, kSmemBytes, stream>>>(tmap, tmap_gath, q);
      break;
    }
    default:
      p.gath_desc = g.desc;   // original base pointers: the kernel adds the direction itself
      b2m_k1_resolve_kernel<<<n_pairs * kResolveParts, 256, 0, stream>>>(p, desc, 1);
      break;
  }
  return cudaGetLastError();
}

cudaError_t launch_gather_matched_columns(const MatchParams& p, const uint8_t* desc, int n_pairs, const GatherScratch& g,
                                          const int32_t* enable, cudaStream_t stream) {
  if (n_pairs <= 0) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(g.n_items, 0, sizeof(int32_t), stream);
  if (e != cudaSuccess) return e;
  b2m_k1_gather_kernel<<<n_pairs, 256, 0, stream>>>(p, desc, g.desc, g.colrank, g.cols, g.cnt, g.items, g.n_items, enable);
  return cudaGetLastError();
}

cudaError_t launch_k1_filter_gather(const CUtensorMap& tmap, const CUtensorMap& tmap_gath, const MatchParams& p_in,
                                    const uint8_t* desc, int n_pairs, int max_strips, int num_sms, const GatherScratch& g,
                                    cudaStream_t stream, cudaEvent_t after_filter) {
  for (int phase = 0; phase < 4; ++phase) {
    cudaError_t e = launch_k1_gather_phase(phase, tmap, tmap_gath, p_in, desc, n_pairs, max_strips, num_sms, g, stream);
    if (e != cudaSuccess) return e;
    if (phase == 2 && after_filter) {
      e = cudaEventRecord(after_filter, stream);
      if (e != cudaSuccess) return e;
    }
  }
  return cudaSuccess;
}

cudaError_t launch_compare_matches(const uint2* arena_a, const int64_t* off_a, const int32_t* cnt_a, const uint2* arena_b,
                                   const int64_t* off_b, const int32_t* cnt_b, int n_pairs, int32_t* mismatch,
                                   cudaStream_t stream) {
  if (n_pairs <= 0) return cudaSuccess;
  b2m_compare_matches_kernel<<<n_pairs, 256, 0, stream>>>(arena_a, off_a, cnt_a, arena_b, off_b, cnt_b, mismatch);
  return cudaGetLastError();
}

}  // namespace b2m
