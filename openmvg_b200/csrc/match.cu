// match.cu — exhaustive putative matching of 128-D uint8 SIFT descriptors on sm_90a.
//
// Replaces (reference, $OPENMVG/src/openMVG):
//   matching_image_collection/Matcher_Regions.cpp:32-107   pair loop (BRUTE_FORCE_L2)
//   matching/regions_matcher.hpp:162-207                   MatchDistanceRatio
//   matching/matcher_brute_force.hpp:100-200               2-NN scan (L2<uint8_t>, metric.hpp:55-93)
//   matching/matching_filters.hpp:38-60                    NNdistanceRatio
//
// Design (DESIGN.md §MATCH):
//   |q - b|^2 = |q|^2 + |b|^2 - 2 q.b.   q.b for a 128-query x 256-database tile is ONE dense
//   u8 x u8 -> s32 contraction with K = 128: four wgmma.mma_async (M64 N256 K32) per warpgroup fed by TMA
//   (128-byte rows, SWIZZLE_128B), accumulators in registers.
//   Epilogue (2 warpgroups): key = 512*dot + ckey[b], ckey[b] = -256*|b|^2 + (b / G)  — one IMAD gives
//   ((2 q.b - |b|^2) << 8) | group(b); the running MAX of the key over a 32-column chunk is one
//   max per element, and a top-2 over chunk maxima costs 3 ops per 32 elements.  The kernel thus
//   emits, per query, the exact best key (=> exact d1 and the 32..G-row group holding the nearest
//   neighbour) and the best key of any OTHER chunk (=> an upper bound ub2 >= d2 that is exact
//   whenever the second neighbour lies outside the best chunk).  A finalize kernel re-scans the one
//   group exactly (dp4a) only for queries that can still pass the ratio test with ub2, recovers
//   (i1, d2) exactly, applies  float(d1) < fratio*float(d2)  and compacts in ascending query order.
//   All integer arithmetic is exact, so the output is bit-identical to the reference.
#include "common.cuh"
#include <cub/device/device_radix_sort.cuh>

#include <cuda.h>
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <climits>
#include <cstring>
#include <memory>
#include <vector>

namespace omvg {

constexpr int TILE_Q = 128;      // queries per work unit: two consumer warpgroups of WG_ROWS
constexpr int TILE_DB = 256;     // wgmma N (database rows per tile)
constexpr int WG_ROWS = 64;      // wgmma M (queries per consumer warpgroup)
constexpr int ROW_PAD = 256;     // every image starts at a multiple of this many arena rows
constexpr int A_STAGES = 2, B_STAGES = 4;
constexpr int A_BYTES = TILE_Q * OMVG_DESC_LEN;                 // 16 KB
constexpr int B_BYTES = TILE_DB * OMVG_DESC_LEN;                // 32 KB
constexpr int CK_BYTES = TILE_DB * 4;                           //  1 KB of packed keys
constexpr int MATCH_THREADS = 384;  // warpgroup 0: TMA producer; warpgroups 1, 2: MMA + epilogue for query rows 0-63 / 64-127
constexpr int KEY_MIN = INT_MIN;

struct Unit { uint32_t q_row, db_row, n_db_tiles, out_off; };   // one (pair, 128-query tile); n_db_tiles = tiles | (rows per group / 32) << 20
constexpr uint32_t UNIT_TILES_MASK = 0xFFFFFu;

// --------------------------------------------------------------------------------- prep kernel
// norm[r] = |row r|^2 ; ckey[r] = -256*norm + (local_row / G) for real rows, INT_MIN for padding.
__global__ void prep_rows_kernel(const uint8_t *__restrict__ desc, const uint32_t *__restrict__ img_row0,
                                 const uint32_t *__restrict__ img_count, const uint32_t *__restrict__ img_group,
                                 const uint32_t *__restrict__ row_img, int32_t *__restrict__ norm,
                                 int32_t *__restrict__ ckey, uint32_t total_rows) {
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 3;   // 8 threads per row, 16 B each
  const uint32_t sub = threadIdx.x & 7;
  if (gw >= total_rows) return;
  const uint4 v = reinterpret_cast<const uint4 *>(desc + (size_t)gw * OMVG_DESC_LEN)[sub];
  uint32_t s = __dp4a(v.x, v.x, 0u); s = __dp4a(v.y, v.y, s); s = __dp4a(v.z, v.z, s); s = __dp4a(v.w, v.w, s);
  s += __shfl_xor_sync(0xffffffffu, s, 1); s += __shfl_xor_sync(0xffffffffu, s, 2); s += __shfl_xor_sync(0xffffffffu, s, 4);
  if (sub == 0) {
    const uint32_t img = row_img[gw >> 8];                      // ROW_PAD == 256 rows per slot
    const uint32_t local = gw - img_row0[img];
    norm[gw] = (int32_t)s;
    ckey[gw] = local < img_count[img] ? (int32_t)(-(int32_t)(s << 8) + (int32_t)(local / img_group[img])) : KEY_MIN;
  }
}

constexpr int DIG_LEN = 32;
constexpr int DG_BYTES = TILE_DB * DIG_LEN;                      //  8 KB of digits per database tile
constexpr int ACONST_BYTES = WG_ROWS * DIG_LEN;                  //  2 KB
constexpr int DIG_PAD = -128 * 2 - 128 * 255 * 30;               // -979456: all 32 digits = -128
constexpr int DIG_VMIN = -979328, DIG_VMAX = 971676;             // v = d0 + 255 M, d0 in [-128, 126], M in [-3840, 3810]
constexpr int DIG_SPREAD_MAX = DIG_VMAX - DIG_VMIN;              // 1 951 004 (in units of h)
// per-image min / max of h = ceil(|row|^2 / 2) over the real rows (one block per image)
__global__ void prep_minmax_kernel(const int32_t *__restrict__ norm, const uint32_t *__restrict__ img_row0,
                                   const uint32_t *__restrict__ img_count, int2 *__restrict__ out) {
  __shared__ int smin[8], smax[8];
  const uint32_t img = blockIdx.x, r0 = img_row0[img], n = img_count[img];
  int lo = INT_MAX, hi = INT_MIN;
  for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) { const int h = (norm[r0 + r] + 1) >> 1; lo = min(lo, h); hi = max(hi, h); }
  #pragma unroll
  for (int off = 16; off > 0; off >>= 1) { lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, off)); hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, off)); }
  if ((threadIdx.x & 31) == 0) { smin[threadIdx.x >> 5] = lo; smax[threadIdx.x >> 5] = hi; }
  __syncthreads();
  if (threadIdx.x == 0) { for (int w = 1; w < (int)(blockDim.x >> 5); ++w) { lo = min(lo, smin[w]); hi = max(hi, smax[w]); } out[img] = make_int2(lo, hi); }
}

// digits of v = c0 - h for real rows, all -128 for padding rows.  Byte 0 and byte 16 have weight 1, the others 255.
__global__ void prep_digits_kernel(const int32_t *__restrict__ norm, const uint32_t *__restrict__ img_row0,
                                   const uint32_t *__restrict__ img_count, const uint32_t *__restrict__ row_img,
                                   const int32_t *__restrict__ img_c0, uint4 *__restrict__ dig, uint32_t total_rows) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= total_rows) return;
  const uint32_t img = row_img[r >> 8], local = r - img_row0[img];
  uint32_t w[8];
  if (local < img_count[img]) {
    const int v = img_c0[img] - ((norm[r] + 1) >> 1);
    int M = (v + 128) / 255; if ((v + 128) - M * 255 < 0) --M;                // floor division
    const int d0 = v - 255 * M;                                               // [-128, 126]
    int qd = M / 30; if (M - qd * 30 < 0) --qd;
    const int rem = M - qd * 30;                                              // [0, 29]
    #pragma unroll
    for (int i = 0; i < 8; ++i) {
      uint32_t word = 0;
      #pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int pos = 4 * i + b;
        int d;
        if (pos == 0) d = d0; else if (pos == 16) d = 0;
        else { const int k = pos < 16 ? pos - 1 : pos - 2; d = qd + (k < rem ? 1 : 0); }
        word |= (uint32_t)(d & 255) << (8 * b);
      }
      w[i] = word;
    }
  } else {
    #pragma unroll
    for (int i = 0; i < 8; ++i) w[i] = 0x80808080u;
  }
  dig[2 * (size_t)r] = make_uint4(w[0], w[1], w[2], w[3]);
  dig[2 * (size_t)r + 1] = make_uint4(w[4], w[5], w[6], w[7]);
}

// --------------------------------------------------------------------------------- wgmma kernel
// One persistent CTA per SM walks the (pair, 128-query tile) units.  Warpgroup 0 (one thread) streams the query tile
// and the 256-row database tiles into shared memory with TMA; warpgroups 1 and 2 each own 64 of the 128 queries and
// multiply them with every database tile (wgmma m64n256k32 from shared memory), so a database tile is loaded once for
// both.  The 64 x 256 accumulator of a tile stays in registers (128 per thread) and the epilogue works on it there;
// while one warpgroup runs its epilogue the other one's MMAs keep the tensor cores busy.
//
// DIG = false (key arithmetic, any uint8 descriptors): key = 512 * dot + ckey[column] per accumulator, the packed keys
// of the tile ride with it in shared memory.
// DIG = true (fifth K-slice): the per-column constant rides in the MMA instead: a fifth K=32 slice multiplies a
// CONSTANT A tile (weights 1, 255 x 15, 1, 255 x 15 in every row) with 32 signed "digits" per database row (u8 x s8)
// so that the accumulator is   acc = q.b - h(b) + c0(image),  h = ceil(|b|^2 / 2).  The epilogue is then a pure
// running max and ONE key per 32-column chunk, key = 256 * max + group.  What is lost is the parity of |b|^2:
// 2 q.b - |b|^2 = 2 acc - 2 c0 + p, p in {0, 1}; the finalize kernel works with the two-sided bound and falls back to
// an exact scan of the whole database image in the (rare) cases where the one unit matters — see
// match_finalize_kernel<true>.  Padding rows carry the most negative digit vector (DIG_PAD), strictly below every
// real column, and zero descriptors.  Digit range: v = c0 - h must lie in [DIG_VMIN, DIG_VMAX]; omvg_match_prepare
// picks c0 per image and uses this variant only if every image fits (|b|^2 spread <= 3.9 M inside an image: always
// true for SIFT, whose |b|^2 is ~2.6e5).
//
// Per query the kernel emits the best chunk key k1 (exact d1 and the group holding the nearest neighbour) and the
// best key of any OTHER 32-column chunk k2 (an upper bound of d2).
template <bool DIG> __host__ __device__ constexpr int stage_bytes() { return B_BYTES + (DIG ? DG_BYTES : CK_BYTES); }   // multiples of 1 KB
template <bool DIG> constexpr int match_smem_bytes() {
  return 1024 /*align slack*/ + A_STAGES * A_BYTES + B_STAGES * stage_bytes<DIG>() + ACONST_BYTES + 256 /*barriers*/;
}

__device__ __forceinline__ void top2_update(int key, int &k1, int &k2) {
  k2 = max(k2, min(k1, key));
  k1 = max(k1, key);
}

template <bool DIG>
__global__ void __launch_bounds__(MATCH_THREADS, 1)
match_wgmma_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmap_dig,
                   const int32_t *__restrict__ ckey, const Unit *__restrict__ units, uint32_t n_units,
                   int2 *__restrict__ k12) {
  constexpr int STAGE = stage_bytes<DIG>();
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t *a_smem = smem;                                        // [A_STAGES][16 KB]
  uint8_t *b_smem = smem + A_STAGES * A_BYTES;                   // [B_STAGES][32 KB descriptors + 8 KB digits | 1 KB keys]
  uint8_t *aconst = b_smem + B_STAGES * STAGE;                   // [64][32 B] constant weights of the fifth slice
  uint64_t *bars = reinterpret_cast<uint64_t *>(aconst + ACONST_BYTES);
  uint64_t *full_a = bars, *empty_a = bars + A_STAGES, *full_b = bars + 2 * A_STAGES, *empty_b = full_b + B_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr uint32_t CONSUMER_WARPS = (MATCH_THREADS - 128) / 32;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap); if (DIG) prefetch_tmap(&tmap_dig);
    for (int i = 0; i < A_STAGES; ++i) { mbar_init(&full_a[i], 1); mbar_init(&empty_a[i], CONSUMER_WARPS); }
    for (int i = 0; i < B_STAGES; ++i) { mbar_init(&full_b[i], 1); mbar_init(&empty_b[i], CONSUMER_WARPS); }
    fence_barrier_init();
  }
  if (DIG) {   // both 16-byte halves of every row are {1, 255 x 15}, so the swizzle cannot matter
    for (int i = threadIdx.x; i < ACONST_BYTES / 16; i += blockDim.x)
      reinterpret_cast<uint4 *>(aconst)[i] = make_uint4(0xFFFFFF01u, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu);
    fence_proxy_async();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================================================================== TMA producer
    if (threadIdx.x == 0) {
      uint32_t g = 0, ul = 0;
      for (uint32_t u = blockIdx.x; u < n_units; u += gridDim.x, ++ul) {
        const Unit un = units[u];
        const uint32_t as = ul % A_STAGES, n_tiles = un.n_db_tiles & UNIT_TILES_MASK;
        mbar_wait(&empty_a[as], ((ul / A_STAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(&full_a[as], A_BYTES);
        tma_load_2d(a_smem + as * A_BYTES, &tmap, 0, (int)un.q_row, &full_a[as]);
        for (uint32_t t = 0; t < n_tiles; ++t, ++g) {
          const uint32_t st = g % B_STAGES;
          mbar_wait(&empty_b[st], ((g / B_STAGES) & 1) ^ 1);
          mbar_arrive_expect_tx(&full_b[st], STAGE);
          uint8_t *dst = b_smem + st * STAGE;
          const uint32_t row = un.db_row + t * TILE_DB;
          tma_load_2d(dst, &tmap, 0, (int)row, &full_b[st]);
          tma_load_2d(dst + A_BYTES, &tmap, 0, (int)(row + 128), &full_b[st]);
          if (DIG) tma_load_2d(dst + B_BYTES, &tmap_dig, 0, (int)row, &full_b[st]);
          else bulk_load_1d(dst + B_BYTES, ckey + row, CK_BYTES, &full_b[st]);
        }
      }
    }
    return;
  }

  // ======================================================================= MMA + epilogue (warpgroups 1 and 2)
  const uint32_t wg = (warp >> 2) - 1;                   // query rows [64 wg, 64 wg + 64) of the unit
  const uint32_t row_lo = wg * WG_ROWS + (warp & 3) * 16 + (lane >> 2);   // accumulator rows of this thread: row_lo, row_lo + 8
  const uint32_t col = 2 * (lane & 3);                   // + 8 j (+ 1): accumulator columns of this thread
  const uint64_t ac_desc = make_kmajor_sw32_desc(smem_u32(aconst));
  int32_t d[128];
  #pragma unroll
  for (int i = 0; i < 128; ++i) d[i] = 0;
  uint32_t g = 0, ul = 0;
  for (uint32_t u = blockIdx.x; u < n_units; u += gridDim.x, ++ul) {
    const Unit un = units[u];
    const uint32_t as = ul % A_STAGES, n_tiles = un.n_db_tiles & UNIT_TILES_MASK, gdiv = (un.n_db_tiles >> 20) & 0x7FFu;
    mbar_wait(&full_a[as], (ul / A_STAGES) & 1);
    const uint32_t a_addr = smem_u32(a_smem + as * A_BYTES + wg * WG_ROWS * OMVG_DESC_LEN);
    int k1lo = KEY_MIN, k2lo = KEY_MIN, k1hi = KEY_MIN, k2hi = KEY_MIN;
    for (uint32_t t = 0; t < n_tiles; ++t, ++g) {
      const uint32_t st = g % B_STAGES;
      mbar_wait(&full_b[st], (g / B_STAGES) & 1);
      const uint32_t b_addr = smem_u32(b_smem + st * STAGE);
      wgmma_fence(d);
      #pragma unroll
      for (int k = 0; k < OMVG_DESC_LEN / 32; ++k)
        wgmma_m64n256k32<false>(d, make_kmajor_sw128_desc(a_addr + k * 32), make_kmajor_sw128_desc(b_addr + k * 32), k > 0);
      if (DIG) wgmma_m64n256k32<true>(d, ac_desc, make_kmajor_sw32_desc(b_addr + B_BYTES), 1);
      wgmma_commit();
      wgmma_wait_all(d);
      if (DIG) {                                         // the tile is in registers: hand the stage back to the producer
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_b[st]);
      }
      const int2 *ck = reinterpret_cast<const int2 *>(b_smem + st * STAGE + B_BYTES);
      #pragma unroll
      for (int c = 0; c < TILE_DB / 32; ++c) {           // 32-column chunk c = accumulator columns 8 j, j in [4 c, 4 c + 4)
        int lo = KEY_MIN, hi = KEY_MIN;
        #pragma unroll
        for (int j = 4 * c; j < 4 * c + 4; ++j) {
          if (DIG) {
            lo = max(lo, max(d[4 * j + 0], d[4 * j + 1]));
            hi = max(hi, max(d[4 * j + 2], d[4 * j + 3]));
          } else {
            const int2 kk = ck[(8 * j + col) >> 1];
            lo = max(lo, max(d[4 * j + 0] * 512 + kk.x, d[4 * j + 1] * 512 + kk.y));
            hi = max(hi, max(d[4 * j + 2] * 512 + kk.x, d[4 * j + 3] * 512 + kk.y));
          }
        }
        // the four threads of a quad hold the same two rows: reduce the chunk maximum over them
        lo = max(lo, __shfl_xor_sync(0xffffffffu, lo, 1)); hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, 1));
        lo = max(lo, __shfl_xor_sync(0xffffffffu, lo, 2)); hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, 2));
        if (DIG) {
          const uint32_t chunk = t * 8 + c;
          const int gid = (int)(gdiv <= 1 ? chunk : chunk / gdiv);
          lo = lo * 256 + gid; hi = hi * 256 + gid;
        }
        top2_update(lo, k1lo, k2lo);
        top2_update(hi, k1hi, k2hi);
      }
      if (!DIG) {                                        // the packed keys have been read
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_b[st]);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_a[as]);
    if ((lane & 3) == 0) {
      k12[(size_t)un.out_off + row_lo] = make_int2(k1lo, k2lo);
      k12[(size_t)un.out_off + row_lo + 8] = make_int2(k1hi, k2hi);
    }
  }
}

// --------------------------------------------------------------------------------- finalize
struct PairInfo { uint32_t db_row0, db_count, db_group, q_row0, q_count; uint32_t unit0; uint64_t out_off; int32_t db_c0; int32_t pad_; };

// expand the per-pair table into the (pair, 128-query tile) work units on the device (one block per pair)
__global__ void expand_units_kernel(const PairInfo *__restrict__ pairs, Unit *__restrict__ units) {
  const PairInfo P = pairs[blockIdx.x];
  const uint32_t qt = (P.q_count + TILE_Q - 1) / TILE_Q, dt = (P.db_count + TILE_DB - 1) / TILE_DB;
  for (uint32_t t = threadIdx.x; t < qt; t += blockDim.x)
    units[P.unit0 + t] = Unit{P.q_row0 + t * TILE_Q, P.db_row0, dt | ((P.db_group / 32) << 20), (uint32_t)(P.out_off + t * TILE_Q)};
}

// exact top-2 of one query inside rows [r0, r1) of the database; whole warp cooperates.
__device__ __forceinline__ void warp_rescan(const uint8_t *__restrict__ desc, const int32_t *__restrict__ norm,
                                            uint32_t q_row, uint32_t r0, uint32_t r1, uint32_t db_row0,
                                            int lane, int &bd1, uint32_t &bi1, int &bd2) {
  const uint32_t qword = reinterpret_cast<const uint32_t *>(desc + (size_t)q_row * OMVG_DESC_LEN)[lane];
  const int qn = norm[q_row];
  int d1 = INT_MAX, d2 = INT_MAX; uint32_t i1 = 0xffffffffu;
  for (uint32_t base = r0; base < r1; base += 32) {              // uniform trip count for the shuffles
    const uint32_t r = base + lane;
    const bool ok = r < r1;
    const uint4 *rp = reinterpret_cast<const uint4 *>(desc + (size_t)(ok ? r : r0) * OMVG_DESC_LEN);
    uint32_t dot = 0;
    #pragma unroll
    for (int k = 0; k < 8; ++k) {
      const uint4 v = rp[k];
      dot = __dp4a(v.x, __shfl_sync(0xffffffffu, qword, 4 * k + 0), dot);
      dot = __dp4a(v.y, __shfl_sync(0xffffffffu, qword, 4 * k + 1), dot);
      dot = __dp4a(v.z, __shfl_sync(0xffffffffu, qword, 4 * k + 2), dot);
      dot = __dp4a(v.w, __shfl_sync(0xffffffffu, qword, 4 * k + 3), dot);
    }
    if (ok) {
      const int d = qn + norm[r] - 2 * (int)dot;
      if (d < d1) { d2 = d1; d1 = d; i1 = r - db_row0; } else if (d < d2) d2 = d;
    }
  }
  #pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const int od1 = __shfl_xor_sync(0xffffffffu, d1, off), od2 = __shfl_xor_sync(0xffffffffu, d2, off);
    const uint32_t oi1 = __shfl_xor_sync(0xffffffffu, i1, off);
    if (od1 < d1 || (od1 == d1 && oi1 < i1)) { d2 = min(od2, d1); d1 = od1; i1 = oi1; }
    else d2 = min(d2, od1);
  }
  bd1 = d1; bi1 = i1; bd2 = d2;
}

constexpr int FIN_THREADS = 256;
// DIG = false: keys of match_wgmma_kernel<false> (exact d1, exact bound ub2).
// DIG = true : keys of match_wgmma_kernel<true>.  A = key >> 8 is the chunk maximum of acc = q.b - h + c0, so the best column
// of that chunk has distance  D - 1 or D,  D = |q|^2 - 2 A + 2 c0  (parity of |b|^2 unknown).  Then
//   * A1 > A2: the nearest neighbour lies in the chunk (group) of A1 — every other column has acc <= A2 <= A1 - 1, i.e.
//     distance >= D1 + 1; its exact distance and index come from the group re-scan as before.
//   * A1 == A2: two chunks tie to within the parity -> exact scan of the whole database image for this query.
//   * the best column outside the group bounds d2 from above by D2 and the truth is D2 - 1 or D2; if the ratio test
//     gives the same answer for both, that is the answer, otherwise -> exact scan of the whole image.
//   * candidates are pre-filtered with the weakest case (d1 >= D1 - 1, d2 <= D2); float() and the multiplication by a
//     non-negative constant are monotone, so nothing that could pass is dropped.
// Chunks that hold only padding have A == DIG_PAD (never reached by a real column): "no second chunk".
template <bool DIG>
__global__ void __launch_bounds__(FIN_THREADS)
match_finalize_kernel(const uint8_t *__restrict__ desc, const int32_t *__restrict__ norm,
                      const PairInfo *__restrict__ pairs, int2 *__restrict__ k12, uint32_t *__restrict__ counts,
                      float fratio) {
  __shared__ uint32_t warp_tot[FIN_THREADS / 32];
  __shared__ uint32_t running;
  const PairInfo P = pairs[blockIdx.x];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) running = 0;
  __syncthreads();
  int2 *io = k12 + P.out_off;
  for (uint32_t q0 = 0; q0 < P.q_count; q0 += FIN_THREADS) {
    const uint32_t q = q0 + threadIdx.x;
    const bool valid = q < P.q_count;
    int ub2 = 0, lo2 = 0; uint32_t g1 = 0; bool cand = false, full = false;
    if (valid) {
      const int2 K = io[q];
      const int qn = norm[P.q_row0 + q];
      g1 = (uint32_t)(K.x & 255);
      if (!DIG) {
        const int d1 = qn - (K.x >> 8);
        ub2 = (K.y == KEY_MIN) ? INT_MAX : qn - (K.y >> 8);
        lo2 = ub2;
        cand = __int2float_rn(d1) < __fmul_rn(fratio, __int2float_rn(ub2));
      } else {
        const int A1 = K.x >> 8, A2 = K.y >> 8;
        const int D1 = qn - 2 * A1 + 2 * P.db_c0;
        const bool none2 = A2 <= DIG_PAD;
        ub2 = none2 ? INT_MAX : qn - 2 * A2 + 2 * P.db_c0;
        lo2 = none2 ? INT_MAX : ub2 - 1;
        cand = __int2float_rn(max(D1 - 1, 0)) < __fmul_rn(fratio, __int2float_rn(ub2));
        full = cand && !none2 && A1 == A2;
      }
    }
    bool keep = false; uint32_t idx = 0;
    uint32_t m = __ballot_sync(0xffffffffu, cand && !full);
    while (m) {
      const int src = __ffs(m) - 1; m &= m - 1;
      const uint32_t qq = __shfl_sync(0xffffffffu, q, src);
      const uint32_t gg = __shfl_sync(0xffffffffu, g1, src);
      const uint32_t r0 = P.db_row0 + gg * P.db_group;
      const uint32_t r1 = min(r0 + P.db_group, P.db_row0 + P.db_count);
      int bd1, bd2; uint32_t bi1;
      warp_rescan(desc, norm, P.q_row0 + qq, r0, r1, P.db_row0, lane, bd1, bi1, bd2);
      if (lane == src) {
        const bool k_hi = __int2float_rn(bd1) < __fmul_rn(fratio, __int2float_rn(min(ub2, bd2)));   // matching_filters.hpp:57
        const bool k_lo = __int2float_rn(bd1) < __fmul_rn(fratio, __int2float_rn(min(lo2, bd2)));
        if (k_hi == k_lo) keep = k_hi; else full = true;
        idx = bi1;
      }
    }
    if (DIG) {                                          // exact scan of the whole database image (rare)
      m = __ballot_sync(0xffffffffu, full);
      while (m) {
        const int src = __ffs(m) - 1; m &= m - 1;
        const uint32_t qq = __shfl_sync(0xffffffffu, q, src);
        int bd1, bd2; uint32_t bi1;
        warp_rescan(desc, norm, P.q_row0 + qq, P.db_row0, P.db_row0 + P.db_count, P.db_row0, lane, bd1, bi1, bd2);
        if (lane == src) { keep = __int2float_rn(bd1) < __fmul_rn(fratio, __int2float_rn(bd2)); idx = bi1; }
      }
    }
    // ordered compaction (ascending q): block exclusive scan of keep
    const uint32_t bal = __ballot_sync(0xffffffffu, keep);
    const uint32_t in_warp = __popc(bal & ((1u << lane) - 1));
    if (lane == 0) warp_tot[warp] = __popc(bal);
    __syncthreads();                                   // all reads of io[q0..] done, warp totals visible
    uint32_t before = running;
    for (int w = 0; w < warp; ++w) before += warp_tot[w];
    if (keep) reinterpret_cast<uint2 *>(io)[before + in_warp] = make_uint2(idx, q);
    __syncthreads();
    if (threadIdx.x == 0) { uint32_t t = 0; for (int w = 0; w < FIN_THREADS / 32; ++w) t += warp_tot[w]; running += t; }
    __syncthreads();
  }
  if (threadIdx.x == 0) counts[blockIdx.x] = running;
}

// exclusive scan of per-pair counts of one batch, offset by *total_io (running total over batches)
__global__ void scan_counts_kernel(const uint32_t *__restrict__ counts, uint32_t n, uint64_t *__restrict__ offsets,
                                   uint64_t *__restrict__ total_io) {
  __shared__ uint64_t wsum[32];
  __shared__ uint64_t carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = *total_io;
  __syncthreads();
  for (uint32_t base = 0; base < n; base += blockDim.x) {
    const uint32_t i = base + threadIdx.x;
    uint64_t v = i < n ? counts[i] : 0, x = v;
    #pragma unroll
    for (int off = 1; off < 32; off <<= 1) { const uint64_t y = __shfl_up_sync(0xffffffffu, x, off); if (lane >= off) x += y; }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    uint64_t pre = carry;
    for (int w = 0; w < warp; ++w) pre += wsum[w];
    if (i < n) offsets[i] = pre + x - v;
    __syncthreads();
    if (threadIdx.x == 0) { uint64_t t = 0; for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += wsum[w]; carry += t; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { offsets[n] = carry; *total_io = carry; }
}

__global__ void compact_kernel(const int2 *__restrict__ k12, const PairInfo *__restrict__ pairs,
                               const uint32_t *__restrict__ counts, const uint64_t *__restrict__ offsets,
                               uint2 *__restrict__ out) {
  const uint32_t p = blockIdx.x, n = counts[p];
  const uint2 *src = reinterpret_cast<const uint2 *>(k12 + pairs[p].out_off);
  uint2 *dst = out + offsets[p];
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}

// --------------------------------------------------------------------------------- SIMT validation
// Exact 2-NN by brute force with dp4a; one block per query.  Tests only.
__global__ void __launch_bounds__(128)
top2_simt_kernel(const uint8_t *__restrict__ desc, const int32_t *__restrict__ norm, uint32_t db_row0,
                 uint32_t db_count, uint32_t q_row0, int32_t *__restrict__ od1, uint32_t *__restrict__ oi1,
                 int32_t *__restrict__ od2) {
  __shared__ uint32_t qs[32];
  __shared__ int sd1[128], sd2[128]; __shared__ uint32_t si1[128];
  const uint32_t q = blockIdx.x;
  if (threadIdx.x < 32) qs[threadIdx.x] = reinterpret_cast<const uint32_t *>(desc + (size_t)(q_row0 + q) * OMVG_DESC_LEN)[threadIdx.x];
  __syncthreads();
  const int qn = norm[q_row0 + q];
  int d1 = INT_MAX, d2 = INT_MAX; uint32_t i1 = 0xffffffffu;
  for (uint32_t r = threadIdx.x; r < db_count; r += blockDim.x) {
    const uint4 *rp = reinterpret_cast<const uint4 *>(desc + (size_t)(db_row0 + r) * OMVG_DESC_LEN);
    uint32_t dot = 0;
    #pragma unroll
    for (int k = 0; k < 8; ++k) { const uint4 v = rp[k];
      dot = __dp4a(v.x, qs[4 * k], dot); dot = __dp4a(v.y, qs[4 * k + 1], dot);
      dot = __dp4a(v.z, qs[4 * k + 2], dot); dot = __dp4a(v.w, qs[4 * k + 3], dot); }
    const int d = qn + norm[db_row0 + r] - 2 * (int)dot;
    if (d < d1) { d2 = d1; d1 = d; i1 = r; } else if (d < d2) d2 = d;
  }
  sd1[threadIdx.x] = d1; sd2[threadIdx.x] = d2; si1[threadIdx.x] = i1;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int t = 1; t < 128; ++t) {
      const int a1 = sd1[t], a2 = sd2[t]; const uint32_t ai = si1[t];
      if (a1 < d1 || (a1 == d1 && ai < i1)) { d2 = min(a2, d1); d1 = a1; i1 = ai; } else d2 = min(d2, a1);
    }
    od1[q] = d1; oi1[q] = i1; od2[q] = d2;
  }
}

__global__ void decode_k12_kernel(const int2 *__restrict__ k12, const int32_t *__restrict__ norm, uint32_t q_row0,
                                  uint32_t n, int32_t *d1, uint32_t *g1, int32_t *ub2) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const int2 K = k12[q]; const int qn = norm[q_row0 + q];
  d1[q] = qn - (K.x >> 8); g1[q] = (uint32_t)(K.x & 255);
  ub2[q] = (K.y == KEY_MIN) ? INT_MAX : qn - (K.y >> 8);
}


// ================================================================================= cascade hashing (M9 / N2)
// openMVG's default matcher for scalar descriptors (matching/cascade_hasher.hpp, Cascade_Hashing_Matcher_Regions.cpp):
// 128-bit sign code + 6 x 10-bit bucket ids per descriptor, candidates = union of the query's 6 buckets in the
// database image, first 10 by (Hamming, insertion order), exact L2 on those, top-2 by (distance, id), ratio test.
// Everything after the hashing is exact integer work; the hashing is a float mat-vec whose summation order is
// fixed here (k ascending, separate multiply and add); the CPU checker used by the tests mirrors it.
constexpr int CH_GROUPS = 6, CH_BITS = 10, CH_NB = 1 << CH_BITS, CH_OUT = OMVG_DESC_LEN + CH_GROUPS * CH_BITS, CH_TOP = 10;
constexpr int CH_HASH_THREADS = 192, CH_HASH_ROWS = 16;

// integer column sums of one image (exact): the float means are formed on the host from them
__global__ void cascade_colsum_kernel(const uint8_t *__restrict__ desc, const uint32_t *__restrict__ img_row0, const uint32_t *__restrict__ img_count,
                                      unsigned long long *__restrict__ sums) {
  const uint32_t img = blockIdx.x, k = threadIdx.x;
  const uint8_t *base = desc + (size_t)img_row0[img] * OMVG_DESC_LEN;
  unsigned long long s = 0;
  for (uint32_t r = 0; r < img_count[img]; ++r) s += base[(size_t)r * OMVG_DESC_LEN + k];
  sums[(size_t)img * OMVG_DESC_LEN + k] = s;
}

// code bit j = (P_j . (d - zm) > 0), bucket id of group g = 10 such signs of S_g, MSB first (cascade_hasher.hpp:203-232)
__global__ void __launch_bounds__(CH_HASH_THREADS) cascade_hash_kernel(const uint8_t *__restrict__ desc, uint32_t total_rows, const float *__restrict__ zm,
                                                                       const float *__restrict__ proj /*[188][128]: primary then secondary*/,
                                                                       uint4 *__restrict__ code, uint4 *__restrict__ bid) {
  __shared__ float sd[CH_HASH_ROWS][OMVG_DESC_LEN];
  __shared__ uint32_t sbid[CH_HASH_ROWS][8];
  __shared__ uint32_t scode[CH_HASH_ROWS][4];
  const uint32_t row0 = blockIdx.x * CH_HASH_ROWS, t = threadIdx.x;
  for (uint32_t idx = t; idx < CH_HASH_ROWS * OMVG_DESC_LEN; idx += CH_HASH_THREADS) {
    const uint32_t r = idx >> 7, k = idx & 127;
    sd[r][k] = row0 + r < total_rows ? __fsub_rn((float)desc[(size_t)(row0 + r) * OMVG_DESC_LEN + k], zm[k]) : 0.0f;
  }
  if (t < CH_HASH_ROWS * 8) sbid[t >> 3][t & 7] = 0;
  __syncthreads();
  if (t < CH_OUT) {
    const float *pr = proj + (size_t)t * OMVG_DESC_LEN;
    float acc[CH_HASH_ROWS];
    #pragma unroll
    for (int r = 0; r < CH_HASH_ROWS; ++r) acc[r] = 0.0f;
    for (int k = 0; k < OMVG_DESC_LEN; ++k) {
      const float pv = pr[k];
      #pragma unroll
      for (int r = 0; r < CH_HASH_ROWS; ++r) acc[r] = __fadd_rn(acc[r], __fmul_rn(pv, sd[r][k]));
    }
    #pragma unroll
    for (int r = 0; r < CH_HASH_ROWS; ++r) {
      const bool bit = acc[r] > 0.0f;
      if (t < OMVG_DESC_LEN) { const uint32_t w = __ballot_sync(0xffffffffu, bit); if ((t & 31) == 0) scode[r][t >> 5] = w; }
      else if (bit) { const int u = t - OMVG_DESC_LEN, g = u / CH_BITS, b = u % CH_BITS; atomicOr(&sbid[r][g], 1u << (CH_BITS - 1 - b)); }
    }
  }
  __syncthreads();
  if (t < CH_HASH_ROWS && row0 + t < total_rows) {
    code[row0 + t] = make_uint4(scode[t][0], scode[t][1], scode[t][2], scode[t][3]);
    bid[row0 + t] = make_uint4(sbid[t][0] | (sbid[t][1] << 16), sbid[t][2] | (sbid[t][3] << 16), sbid[t][4] | (sbid[t][5] << 16), 0u);
  }
}

// sort keys (segment = image*6 + group | bucket | local id) for the bucket tables
__global__ void cascade_keys_kernel(const uint4 *__restrict__ bid, const uint32_t *__restrict__ img_row0, const uint32_t *__restrict__ img_count,
                                    const uint32_t *__restrict__ img_real0, uint32_t n_images, unsigned long long *__restrict__ keys) {
  const uint32_t img = blockIdx.y;
  for (uint32_t local = blockIdx.x * blockDim.x + threadIdx.x; local < img_count[img]; local += gridDim.x * blockDim.x) {
    const uint4 b = bid[img_row0[img] + local];
    const uint32_t ids[6] = {b.x & 0xffffu, b.x >> 16, b.y & 0xffffu, b.y >> 16, b.z & 0xffffu, b.z >> 16};
    #pragma unroll
    for (int g = 0; g < CH_GROUPS; ++g)
      keys[(size_t)CH_GROUPS * (img_real0[img] + local) + g] = ((unsigned long long)(img * CH_GROUPS + g) << 34) | ((unsigned long long)ids[g] << 24) | local;
  }
}
// bucket starts from the sorted keys (bucket index = key >> 24, dense: segment * 1024 + bucket id) and item ids
__global__ void cascade_starts_kernel(const unsigned long long *__restrict__ keys, uint64_t n, uint32_t n_buckets, uint32_t *__restrict__ start, uint32_t *__restrict__ items) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t > n) return;
  const long long lo = t == 0 ? -1 : (long long)(keys[t - 1] >> 24), hi = t == n ? (long long)n_buckets : (long long)(keys[t] >> 24);
  for (long long k = lo + 1; k <= hi; ++k) start[k] = (uint32_t)t;
  if (t < n) items[t] = (uint32_t)(keys[t] & 0xffffffull);
}

// one warp per query (4 queries per warp); writes out[out_off + q].x = matched database id or -1
__global__ void __launch_bounds__(256) cascade_query_kernel(const uint8_t *__restrict__ desc, const int32_t *__restrict__ norm, const uint4 *__restrict__ code,
                                                            const uint4 *__restrict__ bid, const uint32_t *__restrict__ bstart, const uint32_t *__restrict__ bitems,
                                                            const PairInfo *__restrict__ pairs, int2 *__restrict__ out, float fratio) {
  const PairInfo P = pairs[blockIdx.y];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int qq = 0; qq < 4; ++qq) {
    const uint32_t q = blockIdx.x * 32 + warp * 4 + qq;
    if (q >= P.q_count) return;
    const uint32_t qrow = P.q_row0 + q;
    const uint4 qc = code[qrow], qb4 = bid[qrow];
    const uint32_t qb[6] = {qb4.x & 0xffffu, qb4.x >> 16, qb4.y & 0xffffu, qb4.y >> 16, qb4.z & 0xffffu, qb4.z >> 16};
    uint32_t s[6], len[6], tot = 0;
    #pragma unroll
    for (int g = 0; g < CH_GROUPS; ++g) { const uint32_t b = (P.db_group * CH_GROUPS + g) * CH_NB + qb[g]; s[g] = bstart[b]; len[g] = bstart[b + 1] - s[g]; tot += len[g]; }
    int result = -1;
    if (tot > 2) {                                              // "not at least NN candidates" counts duplicates (:301-304)
      // first CH_TOP unique candidates by (Hamming, position in the concatenated bucket lists): CH_TOP selection rounds
      // over the (short) lists; a candidate is a duplicate iff it already sat in the query's bucket of an earlier group
      uint32_t last = 0, my_sel = 0; int nsel = 0;
      if (tot <= 128) {
        // common case: every candidate's (Hamming, position | id) key is formed ONCE into 4 registers per lane, then
        // CH_TOP rounds of warp-min pick the winners (the streaming form below re-reads the lists every round)
        unsigned long long kk[4];
        #pragma unroll
        for (int i = 0; i < 4; ++i) {
          kk[i] = 0xffffffffffffffffull;
          uint32_t pp = lane + 32 * i;
          if (pp < tot) {
            const uint32_t pos = pp; int g = 0; uint32_t sg = 0;
            bool found = false;
            #pragma unroll
            for (int g2 = 0; g2 < CH_GROUPS; ++g2) if (!found) { if (pp < len[g2]) { g = g2; sg = s[g2]; found = true; } else pp -= len[g2]; }
            const uint32_t id = bitems[sg + pp], row = P.db_row0 + id;
            const uint4 cb = bid[row];
            const uint32_t cbv[6] = {cb.x & 0xffffu, cb.x >> 16, cb.y & 0xffffu, cb.y >> 16, cb.z & 0xffffu, cb.z >> 16};
            bool dup = false;
            #pragma unroll
            for (int g2 = 0; g2 < CH_GROUPS; ++g2) if (g2 < g && cbv[g2] == qb[g2]) dup = true;
            if (!dup) {
              const uint4 cc = code[row];
              const uint32_t ham = __popc(cc.x ^ qc.x) + __popc(cc.y ^ qc.y) + __popc(cc.z ^ qc.z) + __popc(cc.w ^ qc.w);
              kk[i] = ((unsigned long long)((ham << 24) | pos) << 32) | id;
            }
          }
        }
        for (int r = 0; r < CH_TOP; ++r) {
          unsigned long long m = min(min(kk[0], kk[1]), min(kk[2], kk[3]));
          #pragma unroll
          for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
          if (m == 0xffffffffffffffffull) break;
          #pragma unroll
          for (int i = 0; i < 4; ++i) if (kk[i] == m) kk[i] = 0xffffffffffffffffull;
          if (lane == r) my_sel = (uint32_t)(m & 0xffffffffull);
          ++nsel;
        }
      } else
      for (int r = 0; r < CH_TOP; ++r) {
        uint32_t best = 0xffffffffu, base = 0;
        #pragma unroll
        for (int g = 0; g < CH_GROUPS; ++g) {
          for (uint32_t off0 = 0; off0 < len[g]; off0 += 32) {
            const uint32_t off = off0 + lane;
            if (off < len[g]) {
              const uint32_t row = P.db_row0 + bitems[s[g] + off];
              const uint4 cb = bid[row];
              const uint32_t cbv[6] = {cb.x & 0xffffu, cb.x >> 16, cb.y & 0xffffu, cb.y >> 16, cb.z & 0xffffu, cb.z >> 16};
              bool dup = false;
              #pragma unroll
              for (int g2 = 0; g2 < CH_GROUPS; ++g2) if (g2 < g && cbv[g2] == qb[g2]) dup = true;
              if (!dup) {
                const uint4 cc = code[row];
                const uint32_t ham = __popc(cc.x ^ qc.x) + __popc(cc.y ^ qc.y) + __popc(cc.z ^ qc.z) + __popc(cc.w ^ qc.w);
                const uint32_t key = ((ham << 24) | (base + off)) + 1u;
                if (key > last && key < best) best = key;
              }
            }
          }
          base += len[g];
        }
        #pragma unroll
        for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
        if (best == 0xffffffffu) break;
        last = best;
        uint32_t pos = (best - 1u) & 0xffffffu, id = 0; bool found = false;
        #pragma unroll
        for (int g = 0; g < CH_GROUPS; ++g) if (!found) { if (pos < len[g]) { id = bitems[s[g] + pos]; found = true; } else pos -= len[g]; }
        if (lane == r) my_sel = id;
        ++nsel;
      }
      if (nsel >= 2) {
        // exact L2 of the selected candidates: d = |q|^2 + |c|^2 - 2 q.c  (integers)
        const uint32_t qv = reinterpret_cast<const uint32_t *>(desc + (size_t)qrow * OMVG_DESC_LEN)[lane];
        const int qn = norm[qrow];
        unsigned long long mine = 0xffffffffffffffffull;
        for (int r = 0; r < nsel; ++r) {
          const uint32_t id = __shfl_sync(0xffffffffu, my_sel, r), row = P.db_row0 + id;
          uint32_t dot = __dp4a(qv, reinterpret_cast<const uint32_t *>(desc + (size_t)row * OMVG_DESC_LEN)[lane], 0u);
          #pragma unroll
          for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
          const int d = qn + norm[row] - 2 * (int)dot;
          if (lane == r) mine = ((unsigned long long)(uint32_t)d << 32) | id;
        }
        // top-2 of (distance, id) in lexicographic order (std::partial_sort of pair<dist,int>, :352-355)
        unsigned long long b1 = mine;
        #pragma unroll
        for (int o = 16; o > 0; o >>= 1) b1 = min(b1, __shfl_xor_sync(0xffffffffu, b1, o));
        unsigned long long b2 = mine == b1 ? 0xffffffffffffffffull : mine;
        #pragma unroll
        for (int o = 16; o > 0; o >>= 1) b2 = min(b2, __shfl_xor_sync(0xffffffffu, b2, o));
        const int d1 = (int)(b1 >> 32), d2 = (int)(b2 >> 32);
        if (__int2float_rn(d1) < __fmul_rn(fratio, __int2float_rn(d2))) result = (int)(uint32_t)(b1 & 0xffffffffull);   // matching_filters.hpp:57
      }
    }
    if (lane == 0) out[P.out_off + q].x = result;
  }
}

// ordered compaction of one pair's results: (database id, query id) for the kept queries, ascending query
__global__ void __launch_bounds__(FIN_THREADS) cascade_compact_kernel(const PairInfo *__restrict__ pairs, int2 *__restrict__ k12, uint32_t *__restrict__ counts) {
  __shared__ uint32_t warp_tot[FIN_THREADS / 32];
  __shared__ uint32_t running;
  const PairInfo P = pairs[blockIdx.x];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) running = 0;
  __syncthreads();
  int2 *io = k12 + P.out_off;
  for (uint32_t q0 = 0; q0 < P.q_count; q0 += FIN_THREADS) {
    const uint32_t q = q0 + threadIdx.x;
    const int v = q < P.q_count ? io[q].x : -1;
    const bool keep = v >= 0;
    const uint32_t bal = __ballot_sync(0xffffffffu, keep);
    const uint32_t in_warp = __popc(bal & ((1u << lane) - 1));
    if (lane == 0) warp_tot[warp] = __popc(bal);
    __syncthreads();
    uint32_t before = running;
    for (int w = 0; w < warp; ++w) before += warp_tot[w];
    if (keep) reinterpret_cast<uint2 *>(io)[before + in_warp] = make_uint2((uint32_t)v, q);
    __syncthreads();
    if (threadIdx.x == 0) { uint32_t t = 0; for (int w = 0; w < FIN_THREADS / 32; ++w) t += warp_tot[w]; running += t; }
    __syncthreads();
  }
  if (threadIdx.x == 0) counts[blockIdx.x] = running;
}

// ================================================================================= guided matching
// geometry_aware::GuidedMatching (robust_estimation/guided_matching.hpp:28-68 and 178-227) for a list of pairs: every
// feature i of image I is tested against every feature j of image J with the pair's model, in ascending j.  One block
// per (pair, 128 features of I), one thread per i; J's positions stream through shared memory in ascending j, so each
// thread runs the reference's sequential loop for its i and needs no merge.  PairInfo's q_* fields describe I (the
// side that is iterated) and db_* fields describe J.
//   error: EpipolarDistanceError (solver_fundamental_kernel.cpp:157-166) or AsymmetricError (solver_homography_kernel.hpp
//     :59-63).  The per-i sub-expressions (F x and |F x|^2_{0,1}, or the projected point of H x) are hoisted; the
//     reference evaluates exactly these, so every operation below is the reference's, explicitly rounded (this file
//     allows FMA contraction).  Built for x86-64-v3, the reference forms each row of M [x; 1] with one FMA, whose
//     operand order differs between the two errors (DESIGN §3.9); the per-j part and the norms have none.
//   DESC: distanceRatio<double>::update with the exact integer L2 of the two descriptors (|a|^2 + |b|^2 - 2 a.b, dp4a),
//     kept iff a second distance exists and bd < ratio * sbd in double.  !DESC: the lowest j of minimal error.
// out[out_off + i].x = j of the match or -1.
constexpr int GM_THREADS = 128, GM_CHUNK = 512;
struct GuidedModel { double M[9]; double thr; };

template <int MODEL, bool DESC>
__global__ void __launch_bounds__(GM_THREADS)
guided_match_kernel(const double2 *__restrict__ pos, const uint8_t *__restrict__ desc, const int32_t *__restrict__ norm,
                    const PairInfo *__restrict__ pairs, const GuidedModel *__restrict__ models, int2 *__restrict__ out,
                    double ratio) {
  __shared__ double2 sj[GM_CHUNK];
  const PairInfo P = pairs[blockIdx.y];
  if (blockIdx.x * GM_THREADS >= P.q_count) return;               // uniform over the block
  const uint32_t i = blockIdx.x * GM_THREADS + threadIdx.x;
  const bool active = i < P.q_count;
  const double *M = models[blockIdx.y].M;
  const double thr = models[blockIdx.y].thr;
  const double2 x = pos[P.q_row0 + (active ? i : 0)];
  double a0, a1, a2 = 0.0, n = 0.0;
  if (MODEL == OMVG_GUIDED_EPIPOLAR) {                           // F x: fma(F_k1, y, F_k0 x) + F_k2
    a0 = __dadd_rn(__fma_rn(M[1], x.y, __dmul_rn(M[0], x.x)), M[2]);
    a1 = __dadd_rn(__fma_rn(M[4], x.y, __dmul_rn(M[3], x.x)), M[5]);
    a2 = __dadd_rn(__fma_rn(M[7], x.y, __dmul_rn(M[6], x.x)), M[8]);
    n = __dadd_rn(__dmul_rn(a0, a0), __dmul_rn(a1, a1));
  } else {                                                         // H x: fma(H_k0, x, H_k1 y) + H_k2
    const double p0 = __dadd_rn(__fma_rn(M[0], x.x, __dmul_rn(M[1], x.y)), M[2]);
    const double p1 = __dadd_rn(__fma_rn(M[3], x.x, __dmul_rn(M[4], x.y)), M[5]);
    const double p2 = __dadd_rn(__fma_rn(M[6], x.x, __dmul_rn(M[7], x.y)), M[8]);
    a0 = __ddiv_rn(p0, p2); a1 = __ddiv_rn(p1, p2);
  }
  uint4 qd[8];
  int qn = 0;
  if (DESC) {
    const uint4 *qp = reinterpret_cast<const uint4 *>(desc + (size_t)(P.q_row0 + (active ? i : 0)) * OMVG_DESC_LEN);
    #pragma unroll
    for (int k = 0; k < 8; ++k) qd[k] = qp[k];
    qn = norm[P.q_row0 + (active ? i : 0)];
  }
  int bd = INT_MAX, sbd = INT_MAX;                                 // integer distances < 2^23: INT_MAX = "none yet"
  double emin = DBL_MAX;
  uint32_t idx = 0;
  for (uint32_t j0 = 0; j0 < P.db_count; j0 += GM_CHUNK) {
    const uint32_t nj = min((uint32_t)GM_CHUNK, P.db_count - j0);
    __syncthreads();
    for (uint32_t t = threadIdx.x; t < nj; t += GM_THREADS) sj[t] = pos[P.db_row0 + j0 + t];
    __syncthreads();
    if (!active) continue;
    for (uint32_t t = 0; t < nj; ++t) {
      const double2 y = sj[t];
      double err;
      if (MODEL == OMVG_GUIDED_EPIPOLAR) {
        const double dt = __dadd_rn(__dadd_rn(__dmul_rn(a0, y.x), __dmul_rn(a1, y.y)), a2);
        err = __ddiv_rn(__dmul_rn(dt, dt), n);
      } else {
        const double dx = __dsub_rn(y.x, a0), dy = __dsub_rn(y.y, a1);
        err = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
      }
      if (!(err < thr)) continue;
      if (DESC) {
        const uint32_t r = P.db_row0 + j0 + t;
        const uint4 *rp = reinterpret_cast<const uint4 *>(desc + (size_t)r * OMVG_DESC_LEN);
        uint32_t dot = 0;
        #pragma unroll
        for (int k = 0; k < 8; ++k) {
          const uint4 v = rp[k];
          dot = __dp4a(v.x, qd[k].x, dot); dot = __dp4a(v.y, qd[k].y, dot);
          dot = __dp4a(v.z, qd[k].z, dot); dot = __dp4a(v.w, qd[k].w, dot);
        }
        const int d = qn + norm[r] - 2 * (int)dot;
        if (d < bd) { idx = j0 + t; sbd = bd; bd = d; } else if (d < sbd) sbd = d;   // guided_matching.hpp:86-102
      } else if (err < emin) { emin = err; idx = j0 + t; }
    }
  }
  if (!active) return;
  const bool keep = DESC ? sbd != INT_MAX && __int2double_rn(bd) < __dmul_rn(ratio, __int2double_rn(sbd))   // :105-112
                         : emin < thr;
  out[P.out_off + i].x = keep ? (int)idx : -1;
}

// ordered compaction of one pair's guided results: (i, j) for the matched i, ascending i
__global__ void __launch_bounds__(FIN_THREADS) guided_compact_kernel(const PairInfo *__restrict__ pairs, int2 *__restrict__ k12, uint32_t *__restrict__ counts) {
  __shared__ uint32_t warp_tot[FIN_THREADS / 32];
  __shared__ uint32_t running;
  const PairInfo P = pairs[blockIdx.x];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) running = 0;
  __syncthreads();
  int2 *io = k12 + P.out_off;
  for (uint32_t q0 = 0; q0 < P.q_count; q0 += FIN_THREADS) {
    const uint32_t q = q0 + threadIdx.x;
    const int v = q < P.q_count ? io[q].x : -1;
    const bool keep = v >= 0;
    const uint32_t bal = __ballot_sync(0xffffffffu, keep);
    const uint32_t in_warp = __popc(bal & ((1u << lane) - 1));
    if (lane == 0) warp_tot[warp] = __popc(bal);
    __syncthreads();
    uint32_t before = running;
    for (int w = 0; w < warp; ++w) before += warp_tot[w];
    if (keep) reinterpret_cast<uint2 *>(io)[before + in_warp] = make_uint2(q, (uint32_t)v);
    __syncthreads();
    if (threadIdx.x == 0) { uint32_t t = 0; for (int w = 0; w < FIN_THREADS / 32; ++w) t += warp_tot[w]; running += t; }
    __syncthreads();
  }
  if (threadIdx.x == 0) counts[blockIdx.x] = running;
}

}  // namespace omvg

// ===================================================================================== host side
using namespace omvg;

namespace omvg {
template <typename T> using Buf = DevBuf<T, CudaAlloc>;   // the arena goes back to the driver with its image set

// everything tied to one image set (omvg_match_set_images): dropping it is a reset
struct ImageSet {
  uint32_t n_images = 0, total_rows = 0;
  std::vector<uint32_t> counts, row0, group;
  Buf<uint8_t> d_desc; Buf<int32_t> d_norm, d_ckey;
  Buf<uint32_t> d_img_row0, d_img_count, d_img_group, d_row_img;
  bool prepared = false;
  CUtensorMap tmap, tmap_dig;
  // fifth-slice kernel (match_wgmma_kernel<true>): 32 signed digits per arena row, per-image offset c0, eligibility
  Buf<uint4> d_dig; Buf<int32_t> d_img_c0; Buf<int2> d_hmm; std::vector<int32_t> c0; bool use_dig = false;
  // cascade hashing state (omvg_match_cascade_prepare)
  Buf<uint4> d_code, d_bid; Buf<uint32_t> d_bstart, d_bitems; Buf<float> d_proj, d_zm;
  bool cascade_ready = false; std::vector<float> h_zm;
  // guided matching (omvg_match_upload_positions / omvg_match_guided_run): one double2 per arena row
  Buf<double2> d_pos; std::vector<uint8_t> has_pos;
  bool loaded() const { return d_desc.p != nullptr; }
};
}  // namespace omvg

struct omvg_match_ctx {
  int device = 0, n_sms = 0;
  cudaStream_t stream = nullptr;
  ImageSet img;
  // run state
  Buf<int2> d_k12;
  Buf<Unit> d_units;
  Buf<PairInfo> d_pairs; Buf<uint32_t> d_counts;
  Buf<uint64_t> d_offsets;   // n_pairs + 1 (global)
  Buf<uint64_t> d_total;
  Buf<uint2> d_out;
  Buf<GuidedModel> d_models;
  uint64_t n_pairs_last = 0, total_last = 0; bool have_result = false;
  DevBuf<uint64_t, PinnedAlloc> h_offsets; DevBuf<uint2, PinnedAlloc> h_ij;
  uint64_t launches = 0;
  double tc_ms = 0; uint64_t tc_launches = 0; std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;
  std::vector<cudaEvent_t> ev_pool;
  size_t k12_budget_bytes = size_t(2) << 30;
};

namespace {

typedef CUresult (*encode_tiled_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int make_tmap(ImageSet &s) {
  void *fn = nullptr; cudaDriverEntryPointQueryResult qres;
  OMVG_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (!fn || qres != cudaDriverEntryPointSuccess) return fail(OMVG_E_CUDA, "cuTensorMapEncodeTiled not available");
  const cuuint64_t dims[2] = {OMVG_DESC_LEN, s.total_rows};
  const cuuint64_t strides[1] = {OMVG_DESC_LEN};
  const cuuint32_t box[2] = {OMVG_DESC_LEN, 128};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = ((encode_tiled_fn)fn)(&s.tmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, s.d_desc.p, dims, strides, box, estr,
                                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(OMVG_E_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  const cuuint64_t ddims[2] = {DIG_LEN, s.total_rows};
  const cuuint64_t dstrides[1] = {DIG_LEN};
  const cuuint32_t dbox[2] = {DIG_LEN, TILE_DB};
  const CUresult r2 = ((encode_tiled_fn)fn)(&s.tmap_dig, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, s.d_dig.p, ddims, dstrides, dbox, estr,
                                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_32B,
                                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r2 != CUDA_SUCCESS) return fail(OMVG_E_CUDA, "cuTensorMapEncodeTiled (digits) failed (%d)", (int)r2);
  return OMVG_OK;
}

int drain_timers(omvg_match_ctx *c) {
  for (auto &pr : c->pending) {
    float ms = 0; OMVG_CUDA(cudaEventSynchronize(pr.second)); OMVG_CUDA(cudaEventElapsedTime(&ms, pr.first, pr.second));
    c->tc_ms += ms; c->ev_pool.push_back(pr.first); c->ev_pool.push_back(pr.second);
  }
  c->pending.clear(); return OMVG_OK;
}
cudaEvent_t get_event(omvg_match_ctx *c) {
  if (!c->ev_pool.empty()) { cudaEvent_t e = c->ev_pool.back(); c->ev_pool.pop_back(); return e; }
  cudaEvent_t e; cudaEventCreate(&e); return e;
}

// a matcher kernel between two events: omvg_match_kernel_time reports the sum of these intervals
template <typename... P, typename... A>
int timed_launch(omvg_match_ctx *c, void (*k)(P...), dim3 grid, dim3 block, size_t smem, A &&...args) {
  const cudaEvent_t e0 = get_event(c), e1 = get_event(c);
  OMVG_CUDA(cudaEventRecord(e0, c->stream));
  if (const int rc = launch(c, k, grid, block, smem, std::forward<A>(args)...)) return rc;
  OMVG_CUDA(cudaEventRecord(e1, c->stream));
  c->pending.emplace_back(e0, e1); c->tc_launches++; return OMVG_OK;
}

// a new CSR result over n_pairs pairs: offsets[0] = 0, running total 0
int begin_result(omvg_match_ctx *c, uint64_t n_pairs) {
  if (const int rc = c->d_offsets.reserve(n_pairs + 1)) return rc;
  OMVG_CUDA(cudaMemsetAsync(c->d_total.p, 0, sizeof(uint64_t), c->stream));
  OMVG_CUDA(cudaMemsetAsync(c->d_offsets.p, 0, sizeof(uint64_t), c->stream));
  c->total_last = 0; c->n_pairs_last = n_pairs; c->have_result = false;
  return OMVG_OK;
}

// the per-pair counts of batch [p0, p0 + nb) are in d_counts and each pair's rows sit compacted at the start of its
// d_k12 segment: scan the counts into the global offsets and append the rows to d_out
int gather_batch(omvg_match_ctx *c, uint32_t nb, uint64_t p0) {
  int rc;
  if ((rc = launch(c, scan_counts_kernel, 1, 1024, 0, c->d_counts.p, nb, c->d_offsets.p + p0, c->d_total.p))) return rc;
  // size the global output buffer: needs the running total (one small sync per batch)
  uint64_t total = 0;
  OMVG_CUDA(cudaMemcpyAsync(&total, c->d_total.p, sizeof total, cudaMemcpyDeviceToHost, c->stream));
  OMVG_CUDA(cudaStreamSynchronize(c->stream));
  if (total > c->d_out.n) {
    Buf<uint2> n;
    if ((rc = n.alloc(std::max<size_t>(total, c->d_out.n * 2 + 1024)))) return rc;
    if (c->d_out.p && c->total_last) OMVG_CUDA(cudaMemcpyAsync(n.p, c->d_out.p, c->total_last * sizeof(uint2), cudaMemcpyDeviceToDevice, c->stream));
    OMVG_CUDA(cudaStreamSynchronize(c->stream));
    c->d_out = std::move(n);
  }
  if ((rc = launch(c, compact_kernel, nb, 128, 0, c->d_k12.p, c->d_pairs.p, c->d_counts.p, c->d_offsets.p + p0, c->d_out.p))) return rc;
  c->total_last = total;
  return OMVG_OK;
}

// What a pair costs the d_k12 budget (int2 rows): it joins a batch that has used `used` while used + need fits the
// budget, and the batch has then used used + use.
struct Cost { size_t need, use; };

// The pair loop of omvg_match_run, _cascade_run and _guided_run.  The pairs are cut into batches of at most `cap` pairs
// within the d_k12 budget (a batch takes at least one pair).  fill(p, P) fills the PairInfo of pair p, whose out_off is
// set, and returns the d_k12 rows it takes.  launches(p0, nb, rows, max q_count) runs the path's kernels on the
// uploaded table of batch [p0, p0 + nb): they leave the per-pair counts in d_counts and each pair's rows compacted at
// the start of its d_k12 segment.
template <typename CostF, typename FillF, typename LaunchF>
int run_pairs(omvg_match_ctx *c, const uint32_t *pair_i, const uint32_t *pair_j, uint64_t n_pairs, uint64_t cap,
              CostF cost, FillF fill, LaunchF launches) {
  for (uint64_t p = 0; p < n_pairs; ++p)
    if (pair_i[p] >= c->img.n_images || pair_j[p] >= c->img.n_images) return fail(OMVG_E_ARG, "pair %llu out of range", (unsigned long long)p);
  int rc;
  if ((rc = begin_result(c, n_pairs))) return rc;
  const size_t budget = c->k12_budget_bytes / sizeof(int2);
  std::vector<PairInfo> pinfo;
  for (uint64_t p0 = 0, p1; p0 < n_pairs; p0 = p1) {
    pinfo.clear(); size_t used = 0, rows = 0; uint32_t maxq = 0;
    for (p1 = p0; p1 < n_pairs && p1 - p0 < cap; ++p1) {
      const Cost k = cost(p1);
      if (p1 > p0 && used + k.need > budget) break;
      used += k.use;
      PairInfo P{}; P.out_off = rows; rows += fill(p1, P);
      maxq = std::max(maxq, P.q_count); pinfo.push_back(P);
    }
    if (rows > 0xffffffffull) return fail(OMVG_E_ARG, "batch too large");
    const uint32_t nb = (uint32_t)(p1 - p0);
    if ((rc = c->d_k12.reserve(std::max<size_t>(rows, 1))) || (rc = c->d_pairs.reserve(nb)) || (rc = c->d_counts.reserve(nb))) return rc;
    OMVG_CUDA(cudaMemcpyAsync(c->d_pairs.p, pinfo.data(), nb * sizeof(PairInfo), cudaMemcpyHostToDevice, c->stream));
    if ((rc = launches(p0, nb, rows, maxq)) || (rc = gather_batch(c, nb, p0))) return rc;
  }
  c->have_result = true; return OMVG_OK;
}

// one image's descriptors into the arena
int upload_desc(omvg_match_ctx *c, uint32_t image, const void *desc, cudaMemcpyKind kind) {
  if (!c) return fail(OMVG_E_ARG, "bad image %u", image);
  ImageSet &im = c->img;
  if (!im.loaded()) return fail(OMVG_E_STATE, "set_images first");
  if (image >= im.n_images || (!desc && im.counts[image])) return fail(OMVG_E_ARG, "bad image %u", image);
  OMVG_CUDA(cudaSetDevice(c->device));
  if (im.counts[image])
    OMVG_CUDA(cudaMemcpyAsync(im.d_desc.p + (size_t)im.row0[image] * OMVG_DESC_LEN, desc, (size_t)im.counts[image] * OMVG_DESC_LEN, kind, c->stream));
  im.prepared = false; im.cascade_ready = false; return OMVG_OK;
}

}  // namespace

extern "C" {

int omvg_version(void) { return 100; }
const char *omvg_last_error(void) { return last_error().c_str(); }
int omvg_device_count(void) {
  int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  int ok = 0; for (int d = 0; d < n; ++d) { cudaDeviceProp p; if (cudaGetDeviceProperties(&p, d) == cudaSuccess && p.major == 9 && p.minor == 0) ++ok; }
  return ok;
}

int omvg_match_create(omvg_match_ctx **out, int device) {
  if (!out) return fail(OMVG_E_ARG, "null ctx");
  int n_sms = 0;
  if (const int rc = check_device(device, &n_sms)) return rc;
  OMVG_CUDA(cudaSetDevice(device));
  std::unique_ptr<omvg_match_ctx, int (*)(omvg_match_ctx *)> c(new omvg_match_ctx, omvg_match_destroy);
  c->device = device; c->n_sms = n_sms;
  OMVG_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  OMVG_CUDA(cudaFuncSetAttribute(match_wgmma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, match_smem_bytes<false>()));
  OMVG_CUDA(cudaFuncSetAttribute(match_wgmma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, match_smem_bytes<true>()));
  if (const int rc = c->d_total.alloc(1)) return rc;
  if (const char *e = getenv("OMVG_MATCH_K12_MB")) c->k12_budget_bytes = size_t(atol(e)) << 20;
  *out = c.release(); return OMVG_OK;
}

int omvg_match_destroy(omvg_match_ctx *c) {
  if (!c) return OMVG_OK;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  drain_timers(c); for (auto e : c->ev_pool) cudaEventDestroy(e);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c; return OMVG_OK;                               // the buffers release themselves
}

// On failure the context is left without an image set: every call that needs one returns OMVG_E_STATE.
int omvg_match_set_images(omvg_match_ctx *c, uint32_t n_images, const uint32_t *counts) {
  if (!c || (!counts && n_images)) return fail(OMVG_E_ARG, "bad arguments");
  OMVG_CUDA(cudaSetDevice(c->device));
  OMVG_CUDA(cudaStreamSynchronize(c->stream));
  c->img = ImageSet(); c->have_result = false;            // the old set is released before the new one is allocated
  ImageSet s;
  s.n_images = n_images; s.counts.assign(counts, counts + n_images); s.row0.resize(n_images); s.group.resize(n_images);
  uint64_t rows = 0; std::vector<uint32_t> row_img;
  for (uint32_t k = 0; k < n_images; ++k) {
    s.row0[k] = (uint32_t)rows;
    const uint32_t padded = (counts[k] + ROW_PAD - 1) / ROW_PAD * ROW_PAD;
    s.group[k] = 32 * std::max<uint32_t>(1, (counts[k] + 8191) / 8192);      // rows/group <= 256 groups
    for (uint32_t r = 0; r < padded / ROW_PAD; ++r) row_img.push_back(k);
    rows += padded;
    if (rows + 2 * ROW_PAD > 0xffffffffull) return fail(OMVG_E_ARG, "collection too large (%llu rows)", (unsigned long long)rows);
  }
  rows += ROW_PAD;                                      // tail slot: TMA boxes never leave the arena
  row_img.push_back(n_images ? n_images - 1 : 0);
  s.total_rows = (uint32_t)rows;
  const size_t ni = std::max(1u, n_images);
  int rc;
  if ((rc = s.d_desc.alloc(rows * OMVG_DESC_LEN)) || (rc = s.d_norm.alloc(rows)) || (rc = s.d_ckey.alloc(rows)) ||
      (rc = s.d_dig.alloc(rows * DIG_LEN / sizeof(uint4))) || (rc = s.d_img_c0.alloc(ni)) || (rc = s.d_hmm.alloc(ni)) ||
      (rc = s.d_img_row0.alloc(ni)) || (rc = s.d_img_count.alloc(ni)) || (rc = s.d_img_group.alloc(ni)) ||
      (rc = s.d_row_img.alloc(row_img.size())))
    return rc;
  OMVG_CUDA(cudaMemsetAsync(s.d_desc.p, 0, rows * OMVG_DESC_LEN, c->stream));
  if (n_images) {
    OMVG_CUDA(cudaMemcpyAsync(s.d_img_row0.p, s.row0.data(), n_images * 4, cudaMemcpyHostToDevice, c->stream));
    OMVG_CUDA(cudaMemcpyAsync(s.d_img_count.p, s.counts.data(), n_images * 4, cudaMemcpyHostToDevice, c->stream));
    OMVG_CUDA(cudaMemcpyAsync(s.d_img_group.p, s.group.data(), n_images * 4, cudaMemcpyHostToDevice, c->stream));
  }
  OMVG_CUDA(cudaMemcpyAsync(s.d_row_img.p, row_img.data(), row_img.size() * 4, cudaMemcpyHostToDevice, c->stream));
  OMVG_CUDA(cudaStreamSynchronize(c->stream));
  if ((rc = make_tmap(s))) return rc;
  c->img = std::move(s); return OMVG_OK;
}

int omvg_match_upload_host(omvg_match_ctx *c, uint32_t image, const uint8_t *desc) {
  return upload_desc(c, image, desc, cudaMemcpyHostToDevice);
}

int omvg_match_upload_device(omvg_match_ctx *c, uint32_t image, const void *desc_dev) {
  return upload_desc(c, image, desc_dev, cudaMemcpyDeviceToDevice);
}

int omvg_match_upload_device_packed(omvg_match_ctx *c, const void *desc_dev) {
  if (!c || !desc_dev) return fail(OMVG_E_ARG, "bad arguments");
  if (!c->img.loaded()) return fail(OMVG_E_STATE, "set_images first");
  size_t off = 0;
  for (uint32_t k = 0; k < c->img.n_images; ++k) {
    const int rc = omvg_match_upload_device(c, k, static_cast<const uint8_t *>(desc_dev) + off);
    if (rc) return rc;
    off += (size_t)c->img.counts[k] * OMVG_DESC_LEN;
  }
  return OMVG_OK;
}

int omvg_match_prepare(omvg_match_ctx *c) {
  if (!c || !c->img.loaded()) return fail(OMVG_E_STATE, "set_images first");
  ImageSet &im = c->img;
  OMVG_CUDA(cudaSetDevice(c->device));
  const uint32_t threads = 256, rows_per_block = threads / 8;
  int rc;
  if ((rc = launch(c, prep_rows_kernel, (im.total_rows + rows_per_block - 1) / rows_per_block, threads, 0,
                   im.d_desc.p, im.d_img_row0.p, im.d_img_count.p, im.d_img_group.p, im.d_row_img.p, im.d_norm.p, im.d_ckey.p, im.total_rows)))
    return rc;
  // fifth-slice kernel: per-image range of h = ceil(|b|^2 / 2) -> offset c0 and eligibility (one small read-back)
  im.c0.assign(im.n_images, 0); im.use_dig = false;
  const bool force_tc4 = getenv("OMVG_MATCH_TC4") != nullptr;         // A/B: the key-arithmetic variant
  if (im.n_images && !force_tc4) {
    if ((rc = launch(c, prep_minmax_kernel, im.n_images, 256, 0, im.d_norm.p, im.d_img_row0.p, im.d_img_count.p, im.d_hmm.p))) return rc;
    std::vector<int2> hmm(im.n_images);
    OMVG_CUDA(cudaMemcpyAsync(hmm.data(), im.d_hmm.p, im.n_images * sizeof(int2), cudaMemcpyDeviceToHost, c->stream));
    OMVG_CUDA(cudaStreamSynchronize(c->stream));
    bool ok = true;
    for (uint32_t k = 0; k < im.n_images; ++k) {
      if (!im.counts[k]) continue;
      if ((long long)hmm[k].y - hmm[k].x > DIG_SPREAD_MAX || im.group[k] / 32 >= 2048) { ok = false; break; }
      im.c0[k] = std::max(0, hmm[k].y + DIG_VMIN);                           // v = c0 - h in [DIG_VMIN, DIG_VMAX]
    }
    if (ok) {
      OMVG_CUDA(cudaMemcpyAsync(im.d_img_c0.p, im.c0.data(), im.n_images * 4, cudaMemcpyHostToDevice, c->stream));
      if ((rc = launch(c, prep_digits_kernel, (im.total_rows + 255) / 256, 256, 0, im.d_norm.p, im.d_img_row0.p, im.d_img_count.p,
                       im.d_row_img.p, im.d_img_c0.p, im.d_dig.p, im.total_rows)))
        return rc;
      OMVG_CUDA(cudaStreamSynchronize(c->stream));                            // im.c0 (host vector) is read by the copy above
      im.use_dig = true;
    }
  }
  im.prepared = true; im.cascade_ready = false; return OMVG_OK;
}

int omvg_match_run(omvg_match_ctx *c, const uint32_t *pair_i, const uint32_t *pair_j, uint64_t n_pairs, float dist_ratio) {
  if (!c || ((!pair_i || !pair_j) && n_pairs)) return fail(OMVG_E_ARG, "bad arguments");
  if (!c->img.prepared) return fail(OMVG_E_STATE, "omvg_match_prepare must follow the uploads");
  if (!(dist_ratio >= 0.f)) return fail(OMVG_E_ARG, "dist_ratio must be >= 0");
  OMVG_CUDA(cudaSetDevice(c->device));
  const ImageSet &im = c->img;
  const float fratio = dist_ratio * dist_ratio;                   // numeric.h:56 Square<float>, regions_matcher.hpp:196
  // a batch is charged for every pair's padded queries, inactive pairs included
  auto cost = [&](uint64_t p) { const size_t need = size_t((im.counts[pair_j[p]] + TILE_Q - 1) / TILE_Q) * TILE_Q; return Cost{need, need}; };
  auto fill = [&](uint64_t p, PairInfo &P) -> size_t {
    const uint32_t I = pair_i[p], J = pair_j[p];
    P.db_row0 = im.row0[I]; P.db_count = im.counts[I]; P.db_group = im.group[I]; P.db_c0 = im.c0[I];
    P.q_row0 = im.row0[J]; P.q_count = im.counts[J];
    // Matcher_Regions.cpp:65-69,85-90 (empty regions) and matcher_brute_force.hpp:108-113 (NN > rows)
    if (P.db_count < 2) P.q_count = 0;
    if (!P.q_count) return 0;
    P.unit0 = (uint32_t)(P.out_off / TILE_Q);                     // one work unit per 128 queries
    return size_t((P.q_count + TILE_Q - 1) / TILE_Q) * TILE_Q;
  };
  auto launches = [&](uint64_t, uint32_t nb, size_t rows, uint32_t) {
    const size_t n_units = rows / TILE_Q;
    int rc;
    if (n_units) {
      if ((rc = c->d_units.reserve(n_units)) || (rc = launch(c, expand_units_kernel, nb, 64, 0, c->d_pairs.p, c->d_units.p))) return rc;
      const uint32_t grid = (uint32_t)std::min<size_t>(n_units, (size_t)c->n_sms);
      if ((rc = im.use_dig ? timed_launch(c, match_wgmma_kernel<true>, grid, MATCH_THREADS, match_smem_bytes<true>(), im.tmap, im.tmap_dig, im.d_ckey.p, c->d_units.p, (uint32_t)n_units, c->d_k12.p)
                           : timed_launch(c, match_wgmma_kernel<false>, grid, MATCH_THREADS, match_smem_bytes<false>(), im.tmap, im.tmap_dig, im.d_ckey.p, c->d_units.p, (uint32_t)n_units, c->d_k12.p)))
        return rc;
    }
    return launch(c, im.use_dig ? match_finalize_kernel<true> : match_finalize_kernel<false>, nb, FIN_THREADS, 0,
                  im.d_desc.p, im.d_norm.p, c->d_pairs.p, c->d_k12.p, c->d_counts.p, fratio);
  };
  return run_pairs(c, pair_i, pair_j, n_pairs, 1u << 20, cost, fill, launches);
}

int omvg_match_sync(omvg_match_ctx *c) {
  if (!c) return fail(OMVG_E_ARG, "null ctx");
  OMVG_CUDA(cudaSetDevice(c->device)); OMVG_CUDA(cudaStreamSynchronize(c->stream));
  return drain_timers(c);
}

int omvg_match_fetch(omvg_match_ctx *c, const uint64_t **offsets, const uint32_t **ij, uint64_t *n_matches) {
  if (!c || !offsets || !ij || !n_matches) return fail(OMVG_E_ARG, "bad arguments");
  if (!c->have_result) return fail(OMVG_E_STATE, "no result: call omvg_match_run");
  OMVG_CUDA(cudaSetDevice(c->device));
  const size_t no = c->n_pairs_last + 1, nm = c->total_last;
  int rc;
  if ((rc = c->h_offsets.reserve(no)) || (rc = c->h_ij.reserve(std::max<size_t>(nm, 1)))) return rc;
  OMVG_CUDA(cudaMemcpyAsync(c->h_offsets.p, c->d_offsets.p, no * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
  if (c->n_pairs_last == 0) { OMVG_CUDA(cudaStreamSynchronize(c->stream)); c->h_offsets.p[0] = 0; }
  if (nm) OMVG_CUDA(cudaMemcpyAsync(c->h_ij.p, c->d_out.p, nm * sizeof(uint2), cudaMemcpyDeviceToHost, c->stream));
  OMVG_CUDA(cudaStreamSynchronize(c->stream));
  drain_timers(c);
  *offsets = c->h_offsets.p; *ij = reinterpret_cast<const uint32_t *>(c->h_ij.p); *n_matches = nm;
  return OMVG_OK;
}

uint64_t omvg_match_launch_count(const omvg_match_ctx *c) { return c ? c->launches : 0; }
int omvg_match_kernel_variant(const omvg_match_ctx *c) { return (!c || !c->img.prepared) ? 0 : (c->img.use_dig ? 5 : 4); }

int omvg_match_kernel_time(omvg_match_ctx *c, double *ms, uint64_t *launches, int reset) {
  if (!c) return fail(OMVG_E_ARG, "null ctx");
  OMVG_CUDA(cudaSetDevice(c->device)); OMVG_CUDA(cudaStreamSynchronize(c->stream));
  const int rc = drain_timers(c); if (rc) return rc;
  if (ms) *ms = c->tc_ms; if (launches) *launches = c->tc_launches;
  if (reset) { c->tc_ms = 0; c->tc_launches = 0; }
  return OMVG_OK;
}

// ---- cascade hashing ---------------------------------------------------------------------------------------
// Hash every image (zero-mean vector over the USED images, Cascade_Hashing_Matcher_Regions.cpp:78-105), build the
// 6 x 1024 bucket tables of every image with one radix sort.  Needs omvg_match_prepare (row norms).
int omvg_match_cascade_prepare(omvg_match_ctx *c, const float *primary, const float *secondary, const uint8_t *used) {
  if (!c || !primary || !secondary) return fail(OMVG_E_ARG, "bad arguments");
  if (!c->img.prepared) return fail(OMVG_E_STATE, "omvg_match_prepare must come first");
  ImageSet &im = c->img;
  OMVG_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->stream;
  const uint32_t ni = im.n_images;
  for (uint32_t k = 0; k < ni; ++k) if (im.counts[k] >= (1u << 24)) return fail(OMVG_E_UNSUPPORTED, "image %u has more than 2^24 descriptors", k);
  im.cascade_ready = false;
  int rc;
  // zero-mean descriptor: exact integer column sums on the device, the two float reductions on the host
  // (float(sum)/float(n) per image; sequential float sum over the used images, / n_used: cascade_hasher.hpp:166-176)
  std::vector<unsigned long long> sums((size_t)ni * OMVG_DESC_LEN);
  {
    Buf<unsigned long long> d_sums;
    if ((rc = d_sums.alloc(std::max<size_t>(1, ni) * OMVG_DESC_LEN))) return rc;
    if (ni) {
      if ((rc = launch(c, cascade_colsum_kernel, ni, OMVG_DESC_LEN, 0, im.d_desc.p, im.d_img_row0.p, im.d_img_count.p, d_sums.p))) return rc;
      OMVG_CUDA(cudaMemcpyAsync(sums.data(), d_sums.p, sums.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    }
    OMVG_CUDA(cudaStreamSynchronize(st));
  }
  im.h_zm.assign(OMVG_DESC_LEN, 0.0f);
  uint32_t n_used = 0; for (uint32_t k = 0; k < ni; ++k) if (!used || used[k]) ++n_used;
  for (int col = 0; col < OMVG_DESC_LEN; ++col) {
    float acc = 0.0f;
    for (uint32_t k = 0; k < ni; ++k) { if (used && !used[k]) continue;
      const float m = im.counts[k] ? (float)sums[(size_t)k * OMVG_DESC_LEN + col] / (float)im.counts[k] : 0.0f; acc = acc + m; }
    im.h_zm[col] = n_used ? acc / (float)n_used : 0.0f;
  }
  if ((rc = im.d_proj.reserve((size_t)CH_OUT * OMVG_DESC_LEN)) || (rc = im.d_zm.reserve(OMVG_DESC_LEN))) return rc;
  OMVG_CUDA(cudaMemcpyAsync(im.d_proj.p, primary, (size_t)OMVG_DESC_LEN * OMVG_DESC_LEN * sizeof(float), cudaMemcpyHostToDevice, st));
  OMVG_CUDA(cudaMemcpyAsync(im.d_proj.p + (size_t)OMVG_DESC_LEN * OMVG_DESC_LEN, secondary, (size_t)CH_GROUPS * CH_BITS * OMVG_DESC_LEN * sizeof(float), cudaMemcpyHostToDevice, st));
  OMVG_CUDA(cudaMemcpyAsync(im.d_zm.p, im.h_zm.data(), OMVG_DESC_LEN * sizeof(float), cudaMemcpyHostToDevice, st));
  if ((rc = im.d_code.reserve(im.total_rows)) || (rc = im.d_bid.reserve(im.total_rows))) return rc;
  if ((rc = launch(c, cascade_hash_kernel, (im.total_rows + CH_HASH_ROWS - 1) / CH_HASH_ROWS, CH_HASH_THREADS, 0,
                   im.d_desc.p, im.total_rows, im.d_zm.p, im.d_proj.p, im.d_code.p, im.d_bid.p)))
    return rc;
  // bucket tables
  std::vector<uint32_t> real0(ni + 1, 0); for (uint32_t k = 0; k < ni; ++k) real0[k + 1] = real0[k] + im.counts[k];
  const uint64_t n_real = real0[ni], n_keys = n_real * CH_GROUPS; const uint32_t n_buckets = ni * CH_GROUPS * CH_NB;
  if (n_keys >= (1ull << 31)) return fail(OMVG_E_UNSUPPORTED, "collection too large for the bucket tables (%llu keys; CUB radix sort takes int counts)", (unsigned long long)n_keys);
  Buf<uint32_t> d_real0; Buf<unsigned long long> d_keys, d_keys2; Buf<uint8_t> d_tmp;
  if ((rc = im.d_bstart.alloc((size_t)n_buckets + 1)) || (rc = im.d_bitems.alloc(std::max<uint64_t>(1, n_keys))) ||
      (rc = d_real0.alloc(ni + 1)) || (rc = d_keys.alloc(std::max<uint64_t>(1, n_keys))) || (rc = d_keys2.alloc(std::max<uint64_t>(1, n_keys))))
    return rc;
  OMVG_CUDA(cudaMemcpyAsync(d_real0.p, real0.data(), (ni + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  if (n_keys) {
    if ((rc = launch(c, cascade_keys_kernel, dim3(32, ni), 256, 0, im.d_bid.p, im.d_img_row0.p, im.d_img_count.p, d_real0.p, ni, d_keys.p))) return rc;
    int seg_bits = 1; while ((1ull << seg_bits) < (unsigned long long)ni * CH_GROUPS) ++seg_bits;
    size_t tb = 0; OMVG_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, d_keys.p, d_keys2.p, (int)n_keys, 0, 34 + seg_bits, st));
    if ((rc = d_tmp.alloc(tb))) return rc;
    OMVG_CUDA(cub::DeviceRadixSort::SortKeys(d_tmp.p, tb, d_keys.p, d_keys2.p, (int)n_keys, 0, 34 + seg_bits, st));
    c->launches++;                                                            // the sort counts as one launch
  }
  if ((rc = launch(c, cascade_starts_kernel, (unsigned)((n_keys + 256) / 256), 256, 0, d_keys2.p, n_keys, n_buckets, im.d_bstart.p, im.d_bitems.p))) return rc;
  OMVG_CUDA(cudaStreamSynchronize(st));
  im.cascade_ready = true; return OMVG_OK;
}

// Cascade_Hashing_Matcher_Regions.cpp:110-189 for a list of pairs (I = database, J = queries).  The result is read
// with omvg_match_fetch: CSR rows of (i, j) in ascending j (the caller sorts by (i, j) as IndMatch::getDeduplicated does).
int omvg_match_cascade_run(omvg_match_ctx *c, const uint32_t *pair_i, const uint32_t *pair_j, uint64_t n_pairs, float dist_ratio) {
  if (!c || ((!pair_i || !pair_j) && n_pairs)) return fail(OMVG_E_ARG, "bad arguments");
  if (!c->img.cascade_ready) return fail(OMVG_E_STATE, "omvg_match_cascade_prepare first");
  if (!(dist_ratio >= 0.f)) return fail(OMVG_E_ARG, "dist_ratio must be >= 0");
  OMVG_CUDA(cudaSetDevice(c->device));
  const ImageSet &im = c->img;
  const float fratio = dist_ratio * dist_ratio;
  // a pair needs room for all of J's queries but takes none for an empty database image (:120-124)
  auto cost = [&](uint64_t p) { const uint32_t nq = im.counts[pair_j[p]]; return Cost{nq, im.counts[pair_i[p]] ? nq : 0}; };
  auto fill = [&](uint64_t p, PairInfo &P) -> size_t {
    const uint32_t I = pair_i[p], J = pair_j[p];
    P.db_row0 = im.row0[I]; P.db_count = im.counts[I]; P.db_group = I; P.q_row0 = im.row0[J];
    P.q_count = P.db_count ? im.counts[J] : 0;
    return P.q_count;
  };
  auto launches = [&](uint64_t, uint32_t nb, size_t, uint32_t maxq) {
    int rc;
    if (maxq && (rc = timed_launch(c, cascade_query_kernel, dim3((maxq + 31) / 32, nb), 256, 0, im.d_desc.p, im.d_norm.p, im.d_code.p, im.d_bid.p,
                                   im.d_bstart.p, im.d_bitems.p, c->d_pairs.p, c->d_k12.p, fratio)))
      return rc;
    return launch(c, cascade_compact_kernel, nb, FIN_THREADS, 0, c->d_pairs.p, c->d_k12.p, c->d_counts.p);
  };
  return run_pairs(c, pair_i, pair_j, n_pairs, 65535, cost, fill, launches);
}

// ---- guided matching ---------------------------------------------------------------------------------------
int omvg_match_upload_positions(omvg_match_ctx *c, uint32_t image, const double *xy) {
  if (!c) return fail(OMVG_E_ARG, "null ctx");
  ImageSet &im = c->img;
  if (!im.loaded()) return fail(OMVG_E_STATE, "set_images first");
  if (image >= im.n_images || (!xy && im.counts[image])) return fail(OMVG_E_ARG, "bad image %u", image);
  OMVG_CUDA(cudaSetDevice(c->device));
  if (!im.d_pos.p) {
    if (const int rc = im.d_pos.alloc(im.total_rows)) return rc;
    im.has_pos.assign(im.n_images, 0);
  }
  if (im.counts[image])
    OMVG_CUDA(cudaMemcpyAsync(im.d_pos.p + im.row0[image], xy, (size_t)im.counts[image] * sizeof(double2), cudaMemcpyHostToDevice, c->stream));
  im.has_pos[image] = 1;
  return OMVG_OK;
}

// GuidedMatching for pairs (I = pair_i[p], J = pair_j[p]); fetch with omvg_match_fetch: rows of (i, j), ascending i.
int omvg_match_guided_run(omvg_match_ctx *c, int32_t error_model, const uint32_t *pair_i, const uint32_t *pair_j, uint64_t n_pairs,
                          const double *models, const double *thresholds, double dist_ratio) {
  if (!c || ((!pair_i || !pair_j || !models || !thresholds) && n_pairs)) return fail(OMVG_E_ARG, "bad arguments");
  if (error_model != OMVG_GUIDED_EPIPOLAR && error_model != OMVG_GUIDED_TRANSFER) return fail(OMVG_E_ARG, "unknown error model %d", error_model);
  if (std::isnan(dist_ratio)) return fail(OMVG_E_ARG, "dist_ratio is NaN");
  if (!c->img.prepared) return fail(OMVG_E_STATE, "omvg_match_prepare must follow the uploads");
  const ImageSet &im = c->img;
  for (uint64_t p = 0; p < n_pairs; ++p) {
    if (pair_i[p] >= im.n_images || pair_j[p] >= im.n_images) return fail(OMVG_E_ARG, "pair %llu out of range", (unsigned long long)p);
    if (im.has_pos.empty() || !im.has_pos[pair_i[p]] || !im.has_pos[pair_j[p]]) return fail(OMVG_E_STATE, "pair %llu: an image has no positions", (unsigned long long)p);
    bool finite = std::isfinite(thresholds[p]);
    for (int k = 0; k < 9; ++k) finite = finite && std::isfinite(models[9 * p + k]);
    if (!finite) return fail(OMVG_E_ARG, "pair %llu: non-finite model or threshold", (unsigned long long)p);
  }
  OMVG_CUDA(cudaSetDevice(c->device));
  const bool desc = dist_ratio >= 0.0;
  auto kernel = error_model == OMVG_GUIDED_EPIPOLAR ? (desc ? guided_match_kernel<OMVG_GUIDED_EPIPOLAR, true> : guided_match_kernel<OMVG_GUIDED_EPIPOLAR, false>)
                                                    : (desc ? guided_match_kernel<OMVG_GUIDED_TRANSFER, true> : guided_match_kernel<OMVG_GUIDED_TRANSFER, false>);
  // I's features are the queries
  auto cost = [&](uint64_t p) { const size_t nq = im.counts[pair_i[p]]; return Cost{nq, nq}; };
  auto fill = [&](uint64_t p, PairInfo &P) -> size_t {
    const uint32_t I = pair_i[p], J = pair_j[p];
    P.q_row0 = im.row0[I]; P.q_count = im.counts[I]; P.db_row0 = im.row0[J]; P.db_count = im.counts[J];
    return P.q_count;
  };
  std::vector<GuidedModel> gm;
  auto launches = [&](uint64_t p0, uint32_t nb, size_t, uint32_t maxq) {
    gm.resize(nb);
    for (uint32_t b = 0; b < nb; ++b) { for (int k = 0; k < 9; ++k) gm[b].M[k] = models[9 * (p0 + b) + k]; gm[b].thr = thresholds[p0 + b]; }
    int rc;
    if ((rc = c->d_models.reserve(nb))) return rc;
    OMVG_CUDA(cudaMemcpyAsync(c->d_models.p, gm.data(), nb * sizeof(GuidedModel), cudaMemcpyHostToDevice, c->stream));
    if (maxq && (rc = timed_launch(c, kernel, dim3((maxq + GM_THREADS - 1) / GM_THREADS, nb), GM_THREADS, 0, im.d_pos.p, im.d_desc.p, im.d_norm.p,
                                   c->d_pairs.p, c->d_models.p, c->d_k12.p, dist_ratio)))
      return rc;
    return launch(c, guided_compact_kernel, nb, FIN_THREADS, 0, c->d_pairs.p, c->d_k12.p, c->d_counts.p);
  };
  return run_pairs(c, pair_i, pair_j, n_pairs, 65535, cost, fill, launches);
}

// Validation aid (tests only): hash codes [count][4], bucket ids [count][6] and the zero-mean vector [128].
int omvg_match_cascade_debug_hash(omvg_match_ctx *c, uint32_t image, uint32_t *codes, uint16_t *bids, float *zero_mean) {
  if (!c) return fail(OMVG_E_ARG, "bad arguments");
  const ImageSet &im = c->img;
  if (!im.cascade_ready) return fail(OMVG_E_STATE, "omvg_match_cascade_prepare first");
  if (image >= im.n_images) return fail(OMVG_E_ARG, "bad arguments");
  OMVG_CUDA(cudaSetDevice(c->device));
  const uint32_t n = im.counts[image];
  std::vector<uint4> hc(n), hb(n);
  if (n) { OMVG_CUDA(cudaMemcpyAsync(hc.data(), im.d_code.p + im.row0[image], n * sizeof(uint4), cudaMemcpyDeviceToHost, c->stream));
           OMVG_CUDA(cudaMemcpyAsync(hb.data(), im.d_bid.p + im.row0[image], n * sizeof(uint4), cudaMemcpyDeviceToHost, c->stream)); }
  OMVG_CUDA(cudaStreamSynchronize(c->stream));
  for (uint32_t r = 0; r < n; ++r) {
    if (codes) { codes[4 * r] = hc[r].x; codes[4 * r + 1] = hc[r].y; codes[4 * r + 2] = hc[r].z; codes[4 * r + 3] = hc[r].w; }
    if (bids) { bids[6 * r] = hb[r].x & 0xffff; bids[6 * r + 1] = hb[r].x >> 16; bids[6 * r + 2] = hb[r].y & 0xffff; bids[6 * r + 3] = hb[r].y >> 16; bids[6 * r + 4] = hb[r].z & 0xffff; bids[6 * r + 5] = hb[r].z >> 16; }
  }
  if (zero_mean) for (int k = 0; k < OMVG_DESC_LEN; ++k) zero_mean[k] = im.h_zm[k];
  return OMVG_OK;
}

int omvg_match_debug_top2_simt(omvg_match_ctx *c, uint32_t I, uint32_t J, int32_t *d1, uint32_t *i1, int32_t *d2) {
  if (!c) return fail(OMVG_E_ARG, "bad image");
  const ImageSet &im = c->img;
  if (!im.prepared) return fail(OMVG_E_STATE, "prepare first");
  if (I >= im.n_images || J >= im.n_images) return fail(OMVG_E_ARG, "bad image");
  OMVG_CUDA(cudaSetDevice(c->device));
  const uint32_t nq = im.counts[J];
  if (nq == 0 || im.counts[I] < 2) return fail(OMVG_E_ARG, "need >=2 database rows and >=1 query");
  Buf<int32_t> dd1, dd2; Buf<uint32_t> di1;
  int rc;
  if ((rc = dd1.alloc(nq)) || (rc = dd2.alloc(nq)) || (rc = di1.alloc(nq)) ||
      (rc = launch(c, top2_simt_kernel, nq, 128, 0, im.d_desc.p, im.d_norm.p, im.row0[I], im.counts[I], im.row0[J], dd1.p, di1.p, dd2.p)))
    return rc;
  OMVG_CUDA(cudaMemcpyAsync(d1, dd1.p, nq * 4, cudaMemcpyDeviceToHost, c->stream));
  OMVG_CUDA(cudaMemcpyAsync(i1, di1.p, nq * 4, cudaMemcpyDeviceToHost, c->stream));
  OMVG_CUDA(cudaMemcpyAsync(d2, dd2.p, nq * 4, cudaMemcpyDeviceToHost, c->stream));
  OMVG_CUDA(cudaStreamSynchronize(c->stream));
  return OMVG_OK;
}

int omvg_match_debug_top2_tc(omvg_match_ctx *c, uint32_t I, uint32_t J, int32_t *d1, uint32_t *g1, int32_t *ub2) {
  if (!c) return fail(OMVG_E_ARG, "bad image");
  const ImageSet &im = c->img;
  if (!im.prepared) return fail(OMVG_E_STATE, "prepare first");
  if (I >= im.n_images || J >= im.n_images) return fail(OMVG_E_ARG, "bad image");
  OMVG_CUDA(cudaSetDevice(c->device));
  const uint32_t nq = im.counts[J], ndb = im.counts[I];
  if (nq == 0 || ndb < 2) return fail(OMVG_E_ARG, "need >=2 database rows and >=1 query");
  const uint32_t qt = (nq + TILE_Q - 1) / TILE_Q, dt = (ndb + TILE_DB - 1) / TILE_DB;
  std::vector<Unit> units;
  for (uint32_t t = 0; t < qt; ++t) units.push_back(Unit{im.row0[J] + t * TILE_Q, im.row0[I], dt, t * TILE_Q});
  int rc;
  if ((rc = c->d_k12.reserve(size_t(qt) * TILE_Q)) || (rc = c->d_units.reserve(units.size()))) return rc;
  OMVG_CUDA(cudaMemcpyAsync(c->d_units.p, units.data(), units.size() * sizeof(Unit), cudaMemcpyHostToDevice, c->stream));
  Buf<int32_t> dd1, dd2; Buf<uint32_t> dg1;
  if ((rc = launch(c, match_wgmma_kernel<false>, std::min<uint32_t>(qt, c->n_sms), MATCH_THREADS, match_smem_bytes<false>(),
                   im.tmap, im.tmap_dig, im.d_ckey.p, c->d_units.p, qt, c->d_k12.p)) ||
      (rc = dd1.alloc(nq)) || (rc = dd2.alloc(nq)) || (rc = dg1.alloc(nq)) ||
      (rc = launch(c, decode_k12_kernel, (nq + 255) / 256, 256, 0, c->d_k12.p, im.d_norm.p, im.row0[J], nq, dd1.p, dg1.p, dd2.p)))
    return rc;
  OMVG_CUDA(cudaMemcpyAsync(d1, dd1.p, nq * 4, cudaMemcpyDeviceToHost, c->stream));
  OMVG_CUDA(cudaMemcpyAsync(g1, dg1.p, nq * 4, cudaMemcpyDeviceToHost, c->stream));
  OMVG_CUDA(cudaMemcpyAsync(ub2, dd2.p, nq * 4, cudaMemcpyDeviceToHost, c->stream));
  OMVG_CUDA(cudaStreamSynchronize(c->stream));
  c->have_result = false;
  return OMVG_OK;
}

}  // extern "C"
