/*
 * aln_levels.hpp -- host-side helpers of the level-synchronous Hirschberg recursion (aln_core.cuh) shared by the batch
 * runtime (csrc/b200aln.cu) and the lane emulation (tests/emu/emu_aln.cpp): the expansion of run starts (aln_runs) into
 * operations / a CIGAR string.  The capacity of the sub-problem lists is in aln_layout.cuh.
 */
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../aln_core.cuh"

namespace b200aln {

/* run starts (start << 2 | op) + total operation count -> one operation per position (edlib's EDLIB_EDOP_* codes) */
inline void aln_expand_runs(const uint32_t* runs, int32_t n_runs, int32_t n_ops, std::vector<uint8_t>& out) {
    out.resize((size_t)n_ops);
    for (int32_t k = 0; k < n_runs; ++k) {
        const int32_t b = (int32_t)(runs[k] >> 2), e = k + 1 < n_runs ? (int32_t)(runs[k + 1] >> 2) : n_ops;
        for (int32_t x = b; x < e; ++x) out[(size_t)x] = (uint8_t)(runs[k] & 3u);
    }
}
/* edlibAlignmentToCigar(..., EDLIB_CIGAR_STANDARD) (edlib.cpp:1482-1520): match and mismatch are both 'M', a query
 * character alone is 'I', a target character alone is 'D' */
inline std::string aln_runs_to_cigar(const uint32_t* runs, int32_t n_runs, int32_t n_ops) {
    static const char letter[4] = {'M', 'I', 'D', 'M'};
    std::string out;
    int32_t k = 0;
    while (k < n_runs) {
        const char c = letter[runs[k] & 3u];
        const int32_t b = (int32_t)(runs[k] >> 2);
        int32_t e = k + 1;
        while (e < n_runs && letter[runs[e] & 3u] == c) ++e;
        const int32_t end = e < n_runs ? (int32_t)(runs[e] >> 2) : n_ops;
        out += std::to_string(end - b);
        out += c;
        k = e;
    }
    return out;
}

} // namespace b200aln
