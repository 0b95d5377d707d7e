/*
 * emu_cut.cpp -- host build of the device layer cut (racon_gpu_b200/csrc/layer_cut.cuh; TEST INFRASTRUCTURE).
 *
 * Runs the four phases exactly as b200aln.cu launches them, one loop per launch; phase 2 (the scan) runs its three
 * steps for 1024 emulated threads, as the one block of aln_cut_scan_kernel does; phase 3 (the scatter, whose order on
 * the device is whatever the atomics make it) visits the items in a seeded random order, so the tests see that the
 * final grouping does not depend on it.  Never linked into the product library.
 */
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <random>
#include <vector>

#include "../../racon_gpu_b200/csrc/layer_cut.cuh"

using namespace b200aln;

extern "C" {

int32_t emu_cut_layer_bytes(void) { return (int32_t)sizeof(CutLayer); }

/* phase 2 as aln_cut_scan_kernel runs it: one block of 1024 threads, a barrier between the steps */
static void run_scan(const CutArgs& a) {
    const uint32_t nt = 1024;
    std::vector<int64_t> part(nt);
    for (uint32_t t = 0; t < nt; ++t) cut_scan_sum(a, t, nt, part.data());
    cut_scan_parts(a, nt, part.data());
    for (uint32_t t = 0; t < nt; ++t) cut_scan_write(a, t, nt, part.data());
}

/* phase 2 alone: win_off[n_win + 1] from counts[n_win] */
void emu_cut_scan(const int32_t* counts, int64_t n_win, int64_t* win_off) {
    CutArgs a{};
    a.counts = const_cast<int32_t*>(counts);
    a.n_win = n_win;
    a.win_off = win_off;
    run_scan(a);
}

/* n overlaps: q_off into `qual`'s arena, bp_off (pairs) into bp, bp_count (pairs), first_window, q_first, has_quality.
 * Writes up to the number of items records to out and n_win counts; returns the number of kept layers. */
int64_t emu_layer_cut(int32_t n, const int64_t* q_off, const int64_t* bp_off, const int32_t* bp_count,
                      const int64_t* first_window, const int32_t* q_first, const uint8_t* has_quality, const uint32_t* bp,
                      const uint8_t* qual, int32_t window_length, double quality_threshold, int64_t win_lo, int64_t n_win,
                      uint64_t seed, CutLayer* out, int32_t* counts) {
    std::vector<CutOverlap> ov((size_t)n);
    int64_t n_items = 0;
    for (int32_t k = 0; k < n; ++k) {
        ov[(size_t)k] = CutOverlap{q_off[k], bp_off[k], n_items, first_window[k], q_first[k], has_quality[k]};
        n_items += bp_count[k] / 2;
    }
    std::vector<CutLayer> items((size_t)n_items);
    std::vector<int32_t> fill((size_t)n_win, 0);
    std::vector<int64_t> win_off((size_t)n_win + 1, 0), slots((size_t)n_items);
    std::fill(counts, counts + n_win, 0);
    CutArgs a;
    a.ov = ov.data();
    a.n_overlaps = n;
    a.n_items = n_items;
    a.bp = bp;
    a.qual = qual;
    a.window_length = window_length;
    a.quality_threshold = quality_threshold;
    a.win_lo = win_lo;
    a.n_win = n_win;
    a.items = items.data();
    a.counts = counts;
    a.win_off = win_off.data();
    a.fill = fill.data();
    a.slots = slots.data();
    a.out = out;
    for (int64_t p = 0; p < n_items; ++p) cut_filter(a, p);
    run_scan(a);
    std::vector<int64_t> order((size_t)n_items);
    std::iota(order.begin(), order.end(), 0);
    std::mt19937_64 rng(seed);
    std::shuffle(order.begin(), order.end(), rng);
    for (int64_t p : order) cut_scatter(a, p);
    const int64_t kept = win_off[(size_t)n_win];
    for (int64_t i = 0; i < kept; ++i) cut_place(a, i);
    return kept;
}

} // extern "C"
