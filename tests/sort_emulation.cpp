// CPU harness for the two-level bucket sort of msm.cu (see tests/test_sort_emulation.py): the five passes of
// DigitSort::run (coarse count, coarse scatter, partition tile counts, fine count, fine scatter) and the hist / offsets
// kernel, block by block and in order, on the index arithmetic of msm_sort.cuh.  The scatter passes stage a block's
// digits sorted by bin and store them run by run, as the kernels do in shared memory.
#include "msm_sort.cuh"
#include <algorithm>
#include <vector>
using namespace zke::dev;

static std::vector<uint32_t> exclusive_scan(const std::vector<uint32_t>& in) {   // with the total appended
    std::vector<uint32_t> out(in.size() + 1, 0);
    for (size_t i = 0; i < in.size(); ++i) out[i + 1] = out[i] + in[i];
    return out;
}

// one block of a scatter pass: items (bin[i], payload i) are sorted by bin into a local array, whose start of bin f
// comes from the block's counts (off[cell(f) + 1] - off[cell(f)], the next cell in scan order), and local position i
// is stored at off[cell(f)] + (i - local start of f), f found by sort_tile_part as the kernels find it
template <class Cell, class Store>
static void staged_scatter(uint32_t n_bins, Cell cell, const std::vector<uint32_t>& off, const std::vector<uint32_t>& bins, Store store) {
    std::vector<uint32_t> base(n_bins + 1, 0), goff(n_bins);
    for (uint32_t f = 0; f < n_bins; ++f) { goff[f] = off[cell(f)]; base[f + 1] = base[f] + off[cell(f) + 1] - off[cell(f)]; }
    std::vector<uint32_t> cur(base.begin(), base.end() - 1), local(bins.size());
    for (uint32_t i = 0; i < bins.size(); ++i) local[cur[bins[i]]++] = i;
    for (uint32_t i = 0; i < base[n_bins]; ++i) {
        const uint32_t f = sort_tile_part(base.data(), n_bins, i);
        store(goff[f] + (i - base[f]), local[i]);
    }
}

extern "C" {
// digits k = 0 .. n-1 of coarse block block[k] (non-decreasing, < n_blocks): bucket[k] < n_buckets, entry word word[k].
// hist, offsets: n_buckets + 1 words; entries: n words.  Returns the number of fine-pass tiles.
uint32_t sort_digits(const uint32_t* bucket, const uint32_t* word, const uint32_t* block, uint32_t n, uint32_t n_blocks,
                     uint32_t n_buckets, int fine_bits, uint32_t tile, uint32_t* hist, uint32_t* offsets, uint32_t* entries) {
    const uint32_t n_parts = sort_parts(n_buckets, fine_bits), F = 1u << fine_bits;
    std::vector<uint32_t> coarse((size_t)n_parts * n_blocks, 0);
    for (uint32_t k = 0; k < n; ++k) coarse[(size_t)(bucket[k] >> fine_bits) * n_blocks + block[k]]++;
    const std::vector<uint32_t> coarse_off = exclusive_scan(coarse);
    std::vector<uint32_t> stage(n), stage_fine(n);
    for (uint32_t k0 = 0, k1; k0 < n; k0 = k1) {
        const uint32_t blk = block[k0];
        for (k1 = k0; k1 < n && block[k1] == blk; ++k1) {}
        std::vector<uint32_t> bins;
        for (uint32_t k = k0; k < k1; ++k) bins.push_back(bucket[k] >> fine_bits);
        staged_scatter(n_parts, [&](uint32_t p) { return (size_t)p * n_blocks + blk; }, coarse_off, bins, [&](uint32_t g, uint32_t i) {
            stage[g] = word[k0 + i];
            stage_fine[g] = bucket[k0 + i] & (F - 1);
        });
    }
    std::vector<uint32_t> part_tiles(n_parts);
    for (uint32_t p = 0; p < n_parts; ++p) {
        const uint32_t cnt = coarse_off[(size_t)(p + 1) * n_blocks] - coarse_off[(size_t)p * n_blocks];
        part_tiles[p] = (cnt + tile - 1) / tile;
    }
    const std::vector<uint32_t> tile_base = exclusive_scan(part_tiles);
    const uint32_t fine_blocks = n / tile + n_parts;
    std::vector<uint32_t> fine((size_t)fine_blocks * F, 0xdeadbeef);
    auto tile_range = [&](uint32_t w, uint32_t& p, uint32_t& tb, uint32_t& tiles_p, uint32_t& t, uint32_t& beg, uint32_t& end) {
        p = sort_tile_part(tile_base.data(), n_parts, w);
        tb = tile_base[p]; tiles_p = tile_base[p + 1] - tb; t = w - tb;
        beg = coarse_off[(size_t)p * n_blocks] + t * tile;
        end = std::min(coarse_off[(size_t)(p + 1) * n_blocks], beg + tile);
    };
    for (uint32_t w = 0; w < fine_blocks; ++w) {
        if (w >= tile_base[n_parts]) { for (uint32_t f = 0; f < F; ++f) fine[(size_t)w * F + f] = 0; continue; }
        uint32_t p, tb, tiles_p, t, beg, end;
        tile_range(w, p, tb, tiles_p, t, beg, end);
        std::vector<uint32_t> bins(F, 0);
        for (uint32_t k = beg; k < end; ++k) bins[stage_fine[k]]++;
        for (uint32_t f = 0; f < F; ++f) fine[sort_cell(tb, tiles_p, f, t, fine_bits)] = bins[f];
    }
    const std::vector<uint32_t> fine_off = exclusive_scan(fine);
    for (uint32_t w = 0; w < tile_base[n_parts]; ++w) {
        uint32_t p, tb, tiles_p, t, beg, end;
        tile_range(w, p, tb, tiles_p, t, beg, end);
        std::vector<uint32_t> bins(stage_fine.begin() + beg, stage_fine.begin() + end);
        staged_scatter(F, [&](uint32_t f) { return sort_cell(tb, tiles_p, f, t, fine_bits); }, fine_off, bins,
                       [&](uint32_t g, uint32_t i) { entries[g] = stage[beg + i]; });
    }
    for (uint32_t b = 0; b <= n_buckets; ++b) {
        const uint32_t o = sort_bucket_offset(b, n_buckets, fine_bits, coarse_off.data(), n_blocks, tile_base.data(), fine_off.data());
        offsets[b] = o;
        hist[b] = b < n_buckets ? sort_bucket_offset(b + 1, n_buckets, fine_bits, coarse_off.data(), n_blocks, tile_base.data(), fine_off.data()) - o : 0;
    }
    return tile_base[n_parts];
}
}
