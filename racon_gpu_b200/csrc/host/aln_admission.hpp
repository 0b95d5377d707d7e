/*
 * aln_admission.hpp -- the aligner batch's admission rule: how many device bytes one staged alignment costs, and whether
 * a batch with a given memory budget takes one more.  The batch runtime (csrc/b200aln.cu: b200aln_batch_add_overlap and
 * the columnar adds) applies it to every overlap it stages; the overlap driver's planner (host/overlap_units.hpp) applies
 * it to whole contigs and window ranges before any batch exists, so that each unit it plans is one the batch takes.
 * Host code only (g++ builds it too, for tests/emu).
 */
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>

#include "../../../include/b200aln.h"
#include "../aln_layout.cuh"
#include "../layer_cut.cuh"

namespace b200aln {

struct AlnJob { /* one alignment of the batch */
    int64_t q_off, t_off; /* into the sequence arena */
    int64_t ops_off;      /* into the operations arena (n + m bytes) */
    int32_t n, m;
    int32_t q_first, t_begin; /* where the segments start in read / contig coordinates (breaking points only) */
};
struct AlnResult {
    int32_t score, status, n_runs, n_ops;
    int64_t runs_off;  /* into the runs arena (words)  */
    int64_t cigar_off; /* into the text arena (bytes)  */
    int32_t cigar_len; /* without the terminating 0    */
    int32_t bp_count;  /* breaking points ((t, q) pairs) */
    int64_t bp_off;    /* into the breaking-point arena (pairs) */
};

constexpr int WARPS_PER_BLOCK = 2;
constexpr size_t ALN_MAX_JOBS = 0x7FFFFF00; /* alignments per batch */

inline int64_t slot_bytes_for(int32_t max_len) {
    size_t total = 0;
    AlnSlot s;
    aln_slot_bind(s, nullptr, max_len, &total);
    return (int64_t)total;
}
inline int32_t round_len(int32_t len) { /* slots are re-made only when the longest sequence outgrows them */
    int32_t r = 16384;
    while (r < len + 1 && r < (1 << 30)) r <<= 1;
    return r;
}
/* device bytes one alignment needs besides the slots: sequences, operations, run starts, its share of the lists */
inline int64_t var_bytes_for(int32_t n, int32_t m) {
    const int64_t len = (int64_t)n + m;
    return 8 * len + 80 + (int64_t)sizeof(AlnJob) + (int64_t)sizeof(AlnResult) +
           (2 * aln_open_capacity(n, m) + aln_leaf_capacity(n, m)) * (int64_t)sizeof(AlnRect);
}
/* device bytes the layer cut adds per overlap: the quality arena (it mirrors the whole sequence arena, so that a layer's
 * qualities sit at its bases' offset), and per window it touches its item, place and record */
inline int64_t cut_bytes_for(bool layer_cut, int32_t n, int32_t m, int64_t n_win) {
    return layer_cut ? (int64_t)n + m + (2 * (int64_t)sizeof(CutLayer) + 8) * n_win : 0;
}

/* what the alignments staged in one batch hold of its budget */
struct AlnLoad {
    int64_t var_bytes = 0; /* device bytes besides the slots */
    int32_t max_len = 0;   /* the longest sequence */
    size_t n_jobs = 0;
};

/* One more n x m alignment starting at t_begin on its contig, into a batch holding `load` (window_length > 0: its
 * breaking points are formed; layer_cut: its layers are cut too).  The slots get what the alignments leave, and at least
 * one block of them, sized for the longest sequence, must remain.  Returns B200ALN_SUCCESS with `load` advanced,
 * B200ALN_EXCEEDED_MAX_LENGTH when the pair fits no batch of this budget next to what is staged, or
 * B200ALN_EXCEEDED_MAX_ALIGNMENTS when the batch is full.  A set of alignments is taken in any order or in none: every
 * term grows with the set. */
inline int32_t aln_admit(AlnLoad& load, int64_t budget, int32_t window_length, bool layer_cut, int32_t n, int32_t m,
                         int32_t t_begin) {
    if ((int64_t)n + m >= ((int64_t)1 << 30)) return B200ALN_EXCEEDED_MAX_LENGTH; /* run starts are 30-bit */
    const int64_t n_win = aln_window_count(t_begin, m, window_length);
    const int64_t vb = var_bytes_for(n, m) + 16 * n_win + cut_bytes_for(layer_cut, n, m, n_win);
    const int32_t new_max = std::max(load.max_len, std::max(n, m));
    const int64_t min_slots = WARPS_PER_BLOCK * slot_bytes_for(round_len(new_max));
    if (vb + min_slots > budget) return B200ALN_EXCEEDED_MAX_LENGTH;
    if (load.var_bytes + vb + min_slots > budget || load.n_jobs >= ALN_MAX_JOBS) return B200ALN_EXCEEDED_MAX_ALIGNMENTS;
    load.var_bytes += vb;
    load.max_len = new_max;
    ++load.n_jobs;
    return B200ALN_SUCCESS;
}

} // namespace b200aln
