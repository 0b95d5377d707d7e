/*
 * aln_layout.cuh -- the overlap aligner's shapes and sizes (aln_core.cuh): edit operation codes, which sub-problems are
 * leaves, the sub-problem record, a resident warp's workspace (slot) and how many windows an alignment touches.  Kept
 * apart from the kernels' code so that host code -- the batch's admission rule (host/aln_admission.hpp) and the overlap
 * driver's planner -- can size a batch without compiling the kernels' device functions again.
 */
#pragma once
#include "poa_simt.cuh"

namespace b200aln {

enum : uint8_t { OP_MATCH = 0, OP_INSERT = 1, OP_DELETE = 2, OP_MISMATCH = 3, OP_NONE = 0xFF }; /* edlib.h EDLIB_EDOP_* */

#if POA_DEVICE
#define ALN_HD __host__ __device__ __forceinline__
#else
#define ALN_HD static inline
#endif

constexpr int64_t ALN_LEAF_DATA_LIMIT = 1024 * 1024; /* edlib.cpp:1157 */

/* edlib.cpp:1135-1157: is this sub-problem traced back directly? */
ALN_HD bool aln_is_leaf(int32_t n, int32_t m) {
    if (n == 0 || m == 0) return true;
    const int64_t blocks = (n + 63) / 64;
    return (2 * 8 + 4) * blocks * (int64_t)m + 2 * 4 * (int64_t)m < ALN_LEAF_DATA_LIMIT;
}

/* Open sub-problems by shape: 0 = at most one 32-block stripe of rows (one warp is all they can use), 1 = tall (several
 * stripes), 2 = huge (at least four stripes and so many cells that ONE of them on one warp would outlast a whole level of
 * ordinary ones: these always go to teams of warps) */
enum { ALN_SHORT = 0, ALN_TALL = 1, ALN_HUGE = 2, ALN_CLASSES = 3 };
ALN_HD int aln_shape(int32_t n, int32_t m) {
    if (n <= 64 * 32) return ALN_SHORT;
    return (n >= 4 * 64 * 32 && (int64_t)n * m >= (int64_t)32 << 20) ? ALN_HUGE : ALN_TALL;
}

/* one open sub-problem: rows [r0, r0 + n) of the query, columns [c0, c0 + m) of the target */
struct AlnRect {
    int32_t aln;
    int32_t r0, n, c0, m;
    int32_t top;  /* bit 0: the whole alignment (its optimum is reported as the edit distance); bit 1: `best` is a guess */
    int32_t best; /* the sub-problem's optimum (children of a split know theirs exactly), a guess to be verified, or -1 */
};
enum { ALN_TOP = 1, ALN_GUESS = 2 };
constexpr int32_t ALN_INF = 1 << 28; /* a distance no path has */
struct AlnSplit { /* result of one Hirschberg step */
    int32_t r;      /* split query index relative to the rect, -1 .. n-1; -2: inconsistent */
    int32_t ls, rs; /* optima of the upper-left and lower-right sub-problems */
    int32_t best;
};

/* the open list of the next level, the leaf list, and where an overflow of either is reported */
struct AlnLists {
    AlnRect* open[ALN_CLASSES]; /* the next level's open sub-problems by shape (aln_shape) */
    int32_t* n_open;            /* [ALN_CLASSES] adjacent counters */
    int32_t cap_open;           /* of each list */
    AlnRect* leaves;
    int32_t* n_leaves;
    int32_t cap_leaves;
    int32_t* overflow;
};

/* one leaf record: the vertical deltas of a 64-row block after a column (+1 bits, -1 bits) */
struct alignas(16) RecPM {
    uint64_t p, m;
};

/* per resident warp workspace */
struct AlnSlot {
    uint32_t* hbuf; /* [hrow words]     horizontal deltas of the row between two stripes, 2 bits a column (1 = +1, 2 = -1);
                       the row's last word is the anchor (the value under the stripe at the next strip's first column) */
    int32_t hrow_words;
    uint8_t* tcode; /* [max_len + 192]  the pass's target as codes 0..3 = ACGT, 4 = other; 64 bytes of padding in front */
    int32_t* Lc;    /* [max_len + 2]    last column of the forward pass:  Lc[i] = D(q[0..i), left half)              */
    int32_t* Rr;    /* [max_len + 2]    last column of the backward pass: Rr[i] = D(q[n-i..n), right half)          */
    RecPM* PM;      /* [leaf entries]   leaf records in wavefront order, see leaf_entry()                            */
    int32_t* S;     /* [leaf entries]   score under the block's last row                                             */
    int32_t* pre;   /* [4 max_len + 8]  target / query characters before every run (aln_breaking_points)            */
};
ALN_HD int64_t aln_hrow_words(int32_t max_len) { return (int64_t)max_len / 16 + 8; } /* one hand-over row */
ALN_HD int64_t aln_leaf_entries(int32_t max_len) { return ALN_LEAF_DATA_LIMIT / 20 + 31 * (int64_t)((max_len + 63) / 64) + 64; }
ALN_HD void aln_slot_bind(AlnSlot& s, uint8_t* base, int32_t max_len, size_t* total_out) {
    size_t o = 0;
    const size_t E = (size_t)aln_leaf_entries(max_len);
#define ALN_CARVE(field, type, count)                                  \
    do {                                                               \
        o = (o + 255) / 256 * 256;                                     \
        s.field = base ? reinterpret_cast<type*>(base + o) : nullptr;  \
        o += sizeof(type) * (size_t)(count);                           \
    } while (0)
    ALN_CARVE(hbuf, uint32_t, (size_t)aln_hrow_words(max_len));
    s.hrow_words = (int32_t)aln_hrow_words(max_len);
    ALN_CARVE(tcode, uint8_t, (size_t)max_len + 192);
    ALN_CARVE(Lc, int32_t, (size_t)max_len + 2);
    ALN_CARVE(Rr, int32_t, (size_t)max_len + 2);
    ALN_CARVE(PM, RecPM, E);
    ALN_CARVE(S, int32_t, E);
    ALN_CARVE(pre, int32_t, 4 * (size_t)max_len + 8);
#undef ALN_CARVE
    o = (o + 255) / 256 * 256;
    if (total_out) *total_out = o;
}

/* How many sub-problems one n x m alignment can have open at one level / leave as leaves in total.  A split halves the
 * columns and partitions the rows, so level d holds <= min(2^d, data / 2^d / 1 MB + 1) open sub-problems (each open one
 * carries >= 1 MB of leaf data, edlib.cpp:1155-1157); every open sub-problem has two children. */
ALN_HD int64_t aln_open_capacity(int32_t n, int32_t m) {
    const int64_t data = 20 * (int64_t)((n + 63) / 64) * m + 8 * (int64_t)m;
    return 2 * (data / ALN_LEAF_DATA_LIMIT + 1) + 2;
}
ALN_HD int64_t aln_leaf_capacity(int32_t n, int32_t m) { return 4 * aln_open_capacity(n, m) + 2; }

/* how many windows of length window_length the target segment [t_begin, t_begin + m) touches (racon overlap.cpp:229-235) */
ALN_HD int32_t aln_window_count(int32_t t_begin, int32_t m, int32_t window_length) {
    if (m <= 0 || window_length <= 0) return 0;
    return (t_begin + m - 1) / window_length - t_begin / window_length + 1;
}

} // namespace b200aln
