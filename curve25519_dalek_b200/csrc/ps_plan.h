// ps_plan.h -- the host plan of a segmented fold (the point sum of point_ops.cu, the scalar Sum / Product of scalars.cu).
// A level cuts segments (m + 1 offsets) into chunks of at most `chunk` consecutive items that never cross a segment
// boundary.  The chunks tile the items in order, so chunk c covers items [start[c], start[c+1]); segment j owns
// chunks [base[j], base[j+1]) (none when it is empty).  The next level's segments are the chunks' partial sums:
// its offsets are this level's base.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <vector>

// The segments' offsets (m + 1 values, m > 0) start at 0, do not decrease and end below 2^31
static inline bool ps_offsets_ok(const uint64_t *offsets, size_t m)
{
    if (offsets[0] != 0) return false;
    for (size_t j = 0; j < m; j++)
        if (offsets[j] > offsets[j + 1]) return false;
    return offsets[m] < (1ull << 31);
}

struct PsLevel {
    std::vector<uint32_t> start;    // nchunks + 1
    std::vector<uint32_t> base;     // m + 1
    uint32_t max_len = 0;           // the longest chunk
    uint32_t max_per_seg = 0;       // the most chunks of one segment
};

template <typename Off>
static inline void ps_plan_level(PsLevel &L, const Off *offsets, size_t m, uint32_t chunk)
{
    L.start.clear(); L.base.clear(); L.max_len = 0; L.max_per_seg = 0;
    L.base.reserve(m + 1);
    for (size_t j = 0; j < m; j++) {
        L.base.push_back((uint32_t)L.start.size());
        const uint64_t lo = (uint64_t)offsets[j], hi = (uint64_t)offsets[j + 1];
        uint32_t k = 0;
        for (uint64_t c = lo; c < hi; c += chunk, k++) {
            L.start.push_back((uint32_t)c);
            L.max_len = std::max(L.max_len, (uint32_t)std::min<uint64_t>(chunk, hi - c));
        }
        L.max_per_seg = std::max(L.max_per_seg, k);
    }
    L.base.push_back((uint32_t)L.start.size());
    L.start.push_back(m ? (uint32_t)offsets[m] : 0u);
}

// Pieces of whole chunks of a level with at most `piece` items each (piece >= chunk): cuts[k] .. cuts[k+1] are the
// chunks of piece k.
static inline void ps_pieces(std::vector<uint32_t> &cuts, const std::vector<uint32_t> &start, uint32_t piece)
{
    cuts.assign(1, 0);
    const uint32_t nchunks = (uint32_t)start.size() - 1;
    for (uint32_t c = 0; c < nchunks; c++)
        if (start[c + 1] - start[cuts.back()] > piece) cuts.push_back(c);
    if (cuts.back() != nchunks) cuts.push_back(nchunks);
}
