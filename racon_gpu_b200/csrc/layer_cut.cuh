/*
 * layer_cut.cuh -- racon's window layers cut on the device from the breaking points (src/polisher.cpp:403-457).
 *
 * Written once for two flavours, like aln_core.cuh: nvcc (the product: one thread per item, device atomics) and g++
 * (tests/emu: plain loops, so the CPU suite checks the same code against racon's windows).  Four phases over a batch:
 *   1. filter   one item per (overlap k, breaking-point pair j): racon's length filter, its quality filter and
 *               add_layer's empty-span check; a kept item becomes its record and is counted in its window;
 *   2. scan     exclusive prefix sum of the per-window counts;
 *   3. scatter  every kept item takes a free place of its window's range (in any order);
 *   4. place    every record moves to its rank among its window's items by item index -- overlap first, then j, which
 *               is racon's add order -- so the grouping is stable whatever order phase 3 ran in.
 */
#pragma once
#include <stdint.h>

#include "poa_simt.cuh"

#if defined(__CUDACC__)
#define CUT_FN __device__ __forceinline__
#define CUT_ATOMIC_ADD(p, v) atomicAdd((p), (v))
#else
#define CUT_FN static inline
#define CUT_ATOMIC_ADD(p, v) cut_host_add((p), (v))
static inline int32_t cut_host_add(int32_t* p, int32_t v) {
    const int32_t old = *p;
    *p = old + v;
    return old;
}
#endif

namespace b200aln {

/* one kept layer: what Window::add_layer receives (include/b200aln.h: b200aln_layer, same layout) */
struct CutLayer {
    int64_t q_off;      /* first base in the batch's query arena (device); its quality sits at the same offset */
    int32_t window;     /* contig window id: first_window + t / w */
    int32_t length;     /* q_{j+1} - q_j */
    int32_t begin, end; /* span in window coordinates: t_j - start, t_{j+1} - start - 1 */
    int32_t has_quality;
    int32_t overlap;    /* the overlap's index in the batch */
};

/* one overlap of the batch as the cut sees it */
struct CutOverlap {
    int64_t q_off;        /* its read segment in the query arena */
    int64_t bp_off;       /* its breaking points in the breaking-point arena (pairs) */
    int64_t item_off;     /* its first item: exclusive prefix sum of (breaking points / 2) in overlap order */
    int64_t first_window; /* id_to_first_window_id[t_id] */
    int32_t q_first;      /* where the segment starts in the strand-adjusted read */
    int32_t has_quality;
};

struct CutArgs {
    const CutOverlap* ov;
    int32_t n_overlaps;
    int64_t n_items;
    const uint32_t* bp;   /* (t, q) words */
    const uint8_t* qual;  /* parallel to the query arena */
    int32_t window_length;
    double quality_threshold;
    int64_t win_lo;       /* counts / offsets cover windows [win_lo, win_lo + n_win) */
    int64_t n_win;
    CutLayer* items;      /* [n_items] window -1: dropped */
    int32_t* counts;      /* [n_win] kept layers per window */
    int64_t* win_off;     /* [n_win + 1] exclusive prefix sum of counts */
    int32_t* fill;        /* [n_win] phase 3's cursors */
    int64_t* slots;       /* [kept] item index per place of a window's range, phase 3 order */
    CutLayer* out;        /* [kept] records grouped by window, racon's add order inside */
};

/* the overlap an item belongs to: last k with item_off[k] <= p (overlaps without items share an offset) */
CUT_FN int32_t cut_overlap_of(const CutArgs& a, int64_t p) {
    int32_t lo = 0, hi = a.n_overlaps - 1;
    while (lo < hi) {
        const int32_t mid = (lo + hi + 1) >> 1;
        if (a.ov[mid].item_off <= p) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

/* phase 1 for item p */
CUT_FN void cut_filter(const CutArgs& a, int64_t p) {
    const int32_t k = cut_overlap_of(a, p);
    const CutOverlap o = a.ov[k];
    const int64_t j = p - o.item_off;
    const uint32_t* w0 = a.bp + 2 * (o.bp_off + 2 * j);
    const uint32_t t0 = w0[0], q0 = w0[1], t1 = w0[2], q1 = w0[3];
    CutLayer r;
    r.q_off = o.q_off + (int64_t)(q0 - (uint32_t)o.q_first);
    r.window = -1;
    r.length = (int32_t)(q1 - q0);
    const uint32_t w = (uint32_t)a.window_length;
    const uint32_t start = (t0 / w) * w;
    r.begin = (int32_t)(t0 - start);
    r.end = (int32_t)(t1 - start - 1);
    r.has_quality = o.has_quality;
    r.overlap = k;
    /* polisher.cpp:411: the difference is uint32, compared as a double with 0.02 * window_length_ */
    bool keep = (double)(q1 - q0) >= 0.02 * (double)w;
    if (keep && o.has_quality) {
        /* polisher.cpp:419-425: a running double sum of (quality - 33), exact for any read below 2^53 / 94 bases, so an
         * integer sum converted once is the same number; then one division and racon's "<" */
        const uint8_t* q = a.qual + r.q_off;
        int64_t sum = 0;
        for (int32_t i = 0; i < r.length; ++i) sum += (int64_t)((uint32_t)q[i] - 33u);
        keep = !((double)sum / (double)(q1 - q0) < a.quality_threshold);
    }
    keep = keep && r.begin != r.end; /* Window::add_layer ignores an empty span (window.cpp:45-47) */
    if (keep) {
        r.window = (int32_t)(o.first_window + (int64_t)(t0 / w));
        CUT_ATOMIC_ADD(a.counts + (r.window - a.win_lo), 1);
    }
    a.items[p] = r;
}

/* phase 2: exclusive prefix sum of the per-window counts in one block of nt threads, in three steps with a barrier
 * between them.  Each thread sums a contiguous chunk of ceil(n_win / nt) windows into part[t]; thread 0 scans the
 * chunk sums and writes the total to win_off[n_win]; then each thread writes its chunk's offsets. */
CUT_FN void cut_scan_sum(const CutArgs& a, uint32_t t, uint32_t nt, int64_t* part) {
    const int64_t chunk = (a.n_win + (nt - 1)) / nt;
    const int64_t lo0 = (int64_t)t * chunk;
    const int64_t lo = lo0 < a.n_win ? lo0 : a.n_win, hi = lo + chunk < a.n_win ? lo + chunk : a.n_win;
    int64_t sum = 0;
    for (int64_t i = lo; i < hi; ++i) sum += a.counts[i];
    part[t] = sum;
}
CUT_FN void cut_scan_parts(const CutArgs& a, uint32_t nt, int64_t* part) {
    int64_t run = 0;
    for (int i = 0; i < (int)nt; ++i) {
        const int64_t v = part[i];
        part[i] = run;
        run += v;
    }
    a.win_off[a.n_win] = run;
}
CUT_FN void cut_scan_write(const CutArgs& a, uint32_t t, uint32_t nt, const int64_t* part) {
    const int64_t chunk = (a.n_win + (nt - 1)) / nt;
    const int64_t lo0 = (int64_t)t * chunk;
    const int64_t lo = lo0 < a.n_win ? lo0 : a.n_win, hi = lo + chunk < a.n_win ? lo + chunk : a.n_win;
    int64_t run = part[t];
    for (int64_t i = lo; i < hi; ++i) {
        a.win_off[i] = run;
        run += a.counts[i];
    }
}

/* phase 3 for item p */
CUT_FN void cut_scatter(const CutArgs& a, int64_t p) {
    const int32_t win = a.items[p].window;
    if (win < 0) return;
    const int64_t lw = win - a.win_lo;
    const int32_t s = CUT_ATOMIC_ADD(a.fill + lw, 1);
    a.slots[a.win_off[lw] + s] = p;
}

/* phase 4 for place i of the kept range */
CUT_FN void cut_place(const CutArgs& a, int64_t i) {
    const int64_t p = a.slots[i];
    const CutLayer r = a.items[p];
    const int64_t lw = r.window - a.win_lo;
    const int64_t lo = a.win_off[lw], hi = a.win_off[lw + 1];
    int64_t rank = 0;
    for (int64_t x = lo; x < hi; ++x) rank += a.slots[x] < p ? 1 : 0;
    a.out[lo + rank] = r;
}

} // namespace b200aln
