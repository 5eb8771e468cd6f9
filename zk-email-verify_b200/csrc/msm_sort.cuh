// Index arithmetic of the two-level bucket sort of the signed digits (msm.cu).  Written so that it also compiles as
// plain C++ (tests/test_sort_emulation.py checks it on the CPU against a Python counting sort).
//
// A bucket index splits into a partition (the high bits) and a fine bin (the low `fine_bits` bits).
//   coarse pass : each block counts its digits per partition (mat1, partition-major: [part][block]); one exclusive
//                 scan of mat1 gives every block its write position in every partition, and the block writes its
//                 digits partition by partition into a staging array (entry word + fine bin).
//   fine pass   : a partition's run of the staging array is cut into tiles of `tile` digits.  Each tile counts its
//                 digits per fine bin into mat2, laid out [part][fine bin][tile of the part], so that one exclusive
//                 scan of mat2 gives every tile its write position in every bucket, in bucket order; the tile then
//                 writes its entries there.  hist / offsets follow from the scanned mat2 without a bucket histogram.
// Both scatters sort their block's digits by bin in shared memory first and then store them run by run.  A block's
// count in a bin is the difference of consecutive cells of the scanned matrix, and sort_tile_part finds the bin of a
// position in the block's sorted digits.
#pragma once
#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#define ZKE_SORT_HD __host__ __device__ __forceinline__
#else
#define ZKE_SORT_HD inline
#endif

namespace zke {
namespace dev {

ZKE_SORT_HD uint32_t sort_parts(uint32_t n_buckets, int fine_bits) { return (n_buckets + (1u << fine_bits) - 1) >> fine_bits; }

// the partition owning fine-pass tile w: the largest p with tile_base[p] <= w.  tile_base is the exclusive scan of the
// partitions' tile counts (tile_base[0] = 0, tile_base[n_parts] = total tiles > w); empty partitions own no tile.
ZKE_SORT_HD uint32_t sort_tile_part(const uint32_t* tile_base, uint32_t n_parts, uint32_t w) {
    uint32_t lo = 0, hi = n_parts;      // tile_base[lo] <= w < tile_base[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (tile_base[mid] <= w) lo = mid; else hi = mid;
    }
    return lo;
}

// cell of (fine bin f, tile t) of the partition whose tiles start at tile_base_p and number tiles_p
ZKE_SORT_HD size_t sort_cell(uint32_t tile_base_p, uint32_t tiles_p, uint32_t f, uint32_t t, int fine_bits) {
    return ((size_t)tile_base_p << fine_bits) + (size_t)f * tiles_p + t;
}

// offset of bucket b in the sorted entries (b == n_buckets: the total).  coarse_off: scanned mat1 (n_parts x
// coarse_blocks, plus the total); fine_off: scanned mat2.  A bucket of an empty partition starts where the partition does.
ZKE_SORT_HD uint32_t sort_bucket_offset(uint32_t b, uint32_t n_buckets, int fine_bits, const uint32_t* coarse_off,
                                        uint32_t coarse_blocks, const uint32_t* tile_base, const uint32_t* fine_off) {
    const uint32_t n_parts = sort_parts(n_buckets, fine_bits);
    if (b >= n_buckets) return coarse_off[(size_t)n_parts * coarse_blocks];
    const uint32_t p = b >> fine_bits, f = b & ((1u << fine_bits) - 1);
    const uint32_t tb = tile_base[p], tiles_p = tile_base[p + 1] - tb;
    return tiles_p ? fine_off[sort_cell(tb, tiles_p, f, 0, fine_bits)] : coarse_off[(size_t)p * coarse_blocks];
}

}  // namespace dev
}  // namespace zke
