/*
 * overlap_units.hpp -- the work units of the overlap driver (overlap_polisher.cpp), planned from the input columns before
 * any batch exists.
 *
 * A unit is a run of consecutive windows together with every overlap that can give them a layer, in racon's order; one
 * aligner batch takes it whole.  A window only receives layers from overlaps on its own contig, and an overlap's breaking
 * points fall only in windows t_begin / w .. (t_end - 1) / w (aln_window_count), so a unit owning windows [wa, wb) of a
 * contig takes the contig's overlaps whose window span meets [wa, wb).  The cut orders each window's records by (overlap
 * index in the batch, breaking point), so a subsequence of racon's order keeps each window's order, and the alignment of
 * a pair does not depend on the rest of its batch: each owned window gets the records of a whole-contig round.
 *
 * Whole contigs are packed greedily in contig order, as many as the batch takes (rounds of whole contigs).  With
 * splitting, a contig that does not fit one batch alone becomes consecutive window ranges, each as long as fits; an
 * overlap crossing a boundary is aligned in every unit it meets.  A window whose overlaps alone do not fit, or a pair
 * that fits no batch of the budget, is reported as unfit_contig.  Units depend on the input, the window length and the
 * budget only.  The admission is the aligner batch's own (aln_admission.hpp).  Host code only (tests/emu builds it).
 */
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../../include/b200poa.h"
#include "aln_admission.hpp"
#include "overlap_polisher.hpp"

namespace racon_b200 {

struct OverlapUnit {
    int64_t contig;         /* its first contig */
    int64_t win_lo, win_hi; /* the windows it owns: [win_lo, win_hi), ids of the per-window outputs */
    int64_t ov_lo, ov_hi;   /* its overlaps: OverlapPlan::overlaps[ov_lo .. ov_hi), in racon's order */
    bool split;             /* one of several units of one contig */
};

struct OverlapPlan {
    std::vector<int64_t> first_window; /* [n_contigs + 1] id_to_first_window_id (polisher.cpp:384-398) */
    std::vector<OverlapUnit> units;    /* in window order */
    std::vector<int64_t> overlaps;     /* overlap indices of every unit, one run per unit */
    int64_t split_contigs = 0;         /* contigs polished in more than one unit */
    int64_t repeat_overlaps = 0;       /* alignments done more than once because of the splits */
    int64_t unfit_contig = -1;
};

/* The units of `in` for windows of length w and aligner batches of `budget` bytes, split (when `split`) at window
 * boundaries.  Returns B200POA_SUCCESS, B200POA_INVALID_ARGUMENT (inconsistent input), or B200POA_GENERIC_ERROR with
 * plan.unfit_contig set. */
inline int32_t plan_overlap_units(const OverlapInput& in, int32_t w, int64_t budget, bool split, OverlapPlan& plan) {
    plan = OverlapPlan{};
    if (w <= 0 || in.n_contigs < 0 || in.n_overlaps < 0 || !in.t_off) return B200POA_INVALID_ARGUMENT;
    if (in.n_overlaps > 0 && (!in.t_id || !in.t_begin || !in.t_end || !in.q_off || !in.q_first))
        return B200POA_INVALID_ARGUMENT;
    std::vector<int64_t>& fw = plan.first_window;
    fw.assign((size_t)in.n_contigs + 1, 0);
    for (int64_t c = 0; c < in.n_contigs; ++c) {
        const int64_t len = in.t_off[c + 1] - in.t_off[c];
        if (len < 0 || len >= ((int64_t)1 << 31)) return B200POA_INVALID_ARGUMENT;
        fw[(size_t)c + 1] = fw[(size_t)c] + (len + w - 1) / w;
    }
    /* the overlaps stably partitioned by t_id keep racon's order inside a contig */
    std::vector<int64_t> ov_begin((size_t)in.n_contigs + 1, 0), order((size_t)in.n_overlaps);
    for (int64_t k = 0; k < in.n_overlaps; ++k) {
        const int32_t c = in.t_id[k];
        if (c < 0 || c >= in.n_contigs || in.t_begin[k] < 0 || in.t_end[k] < in.t_begin[k] ||
            in.t_end[k] > in.t_off[c + 1] - in.t_off[c] || in.q_first[k] < 0 || in.q_off[k + 1] < in.q_off[k] ||
            in.q_off[k + 1] - in.q_off[k] >= ((int64_t)1 << 31))
            return B200POA_INVALID_ARGUMENT;
        ++ov_begin[(size_t)c + 1];
    }
    for (int64_t c = 0; c < in.n_contigs; ++c) ov_begin[(size_t)c + 1] += ov_begin[(size_t)c];
    {
        std::vector<int64_t> fill(ov_begin.begin(), ov_begin.end() - 1);
        for (int64_t k = 0; k < in.n_overlaps; ++k) order[(size_t)fill[(size_t)in.t_id[k]]++] = k;
    }
    /* overlap k into a batch holding `load`: the driver's aligner batches cut layers */
    auto admit = [&](b200aln::AlnLoad& load, int64_t k) {
        return b200aln::aln_admit(load, budget, w, true, (int32_t)(in.q_off[k + 1] - in.q_off[k]),
                                  in.t_end[k] - in.t_begin[k], in.t_begin[k]) == B200ALN_SUCCESS;
    };
    auto admit_contig = [&](b200aln::AlnLoad& load, int64_t c) {
        for (int64_t i = ov_begin[(size_t)c]; i < ov_begin[(size_t)c + 1]; ++i)
            if (!admit(load, order[(size_t)i])) return false;
        return true;
    };

    b200aln::AlnLoad load;
    int64_t first = -1, last = -1; /* the contigs with overlaps of the open round */
    auto close_round = [&]() {
        if (first < 0) return;
        plan.units.push_back(OverlapUnit{first, fw[(size_t)first], fw[(size_t)last + 1], ov_begin[(size_t)first],
                                         ov_begin[(size_t)last + 1], false});
        first = last = -1;
        load = b200aln::AlnLoad{};
    };
    for (int64_t c = 0; c < in.n_contigs; ++c) {
        if (ov_begin[(size_t)c] == ov_begin[(size_t)c + 1]) continue; /* no overlaps: no unit, the backbones stay */
        b200aln::AlnLoad with = load;
        if (!admit_contig(with, c)) {
            close_round(); /* contig c goes to the next unit */
            with = b200aln::AlnLoad{};
            if (!admit_contig(with, c)) {
                if (!split) {
                    plan.unfit_contig = c;
                    return B200POA_GENERIC_ERROR;
                }
                /* contig c alone does not fit: consecutive window ranges, each with the overlaps whose span meets it */
                const int64_t n_win = fw[(size_t)c + 1] - fw[(size_t)c], n_ov = ov_begin[(size_t)c + 1] - ov_begin[(size_t)c];
                if (n_win == 0) { /* an empty contig has no window to split at */
                    plan.unfit_contig = c;
                    return B200POA_GENERIC_ERROR;
                }
                std::vector<int64_t> lo((size_t)n_ov), hi((size_t)n_ov), by_lo_off((size_t)n_win + 1, 0), by_lo((size_t)n_ov);
                for (int64_t i = 0; i < n_ov; ++i) { /* racon's rank i of the contig's overlaps */
                    const int64_t k = order[(size_t)(ov_begin[(size_t)c] + i)];
                    const int64_t last_col = std::max<int64_t>(in.t_begin[k], (int64_t)in.t_end[k] - 1);
                    lo[(size_t)i] = std::min<int64_t>(in.t_begin[k] / w, n_win - 1);
                    hi[(size_t)i] = std::min<int64_t>(last_col / w, n_win - 1);
                    ++by_lo_off[(size_t)lo[(size_t)i] + 1];
                }
                for (int64_t x = 0; x < n_win; ++x) by_lo_off[(size_t)x + 1] += by_lo_off[(size_t)x];
                {
                    std::vector<int64_t> fill(by_lo_off.begin(), by_lo_off.end() - 1);
                    for (int64_t i = 0; i < n_ov; ++i) by_lo[(size_t)fill[(size_t)lo[(size_t)i]]++] = i;
                }
                std::vector<int64_t> members; /* ranks of the open unit's overlaps */
                int64_t wa = 0;
                b200aln::AlnLoad unit_load;
                const size_t units_before = plan.units.size();
                auto emit = [&](int64_t wb) {
                    std::sort(members.begin(), members.end());
                    const int64_t ov_lo = (int64_t)plan.overlaps.size();
                    for (int64_t i : members) plan.overlaps.push_back(order[(size_t)(ov_begin[(size_t)c] + i)]);
                    plan.units.push_back(OverlapUnit{c, fw[(size_t)c] + wa, fw[(size_t)c] + wb, ov_lo,
                                                     (int64_t)plan.overlaps.size(), true});
                };
                for (int64_t wb = 0; wb < n_win; ++wb) { /* window wb joins the open unit [wa, wb) */
                    b200aln::AlnLoad grown = unit_load;
                    bool ok = true;
                    for (int64_t x = by_lo_off[(size_t)wb]; x < by_lo_off[(size_t)wb + 1] && ok; ++x)
                        ok = admit(grown, order[(size_t)(ov_begin[(size_t)c] + by_lo[(size_t)x])]);
                    if (!ok) {
                        if (wb == wa) { /* the overlaps of window wa alone do not fit */
                            plan.unfit_contig = c;
                            return B200POA_GENERIC_ERROR;
                        }
                        emit(wb);
                        /* the next unit starts with the overlaps that cross into window wb */
                        std::vector<int64_t> crossing;
                        grown = b200aln::AlnLoad{};
                        for (int64_t i : members)
                            if (hi[(size_t)i] >= wb) {
                                crossing.push_back(i);
                                admit(grown, order[(size_t)(ov_begin[(size_t)c] + i)]);
                            }
                        members.swap(crossing);
                        wa = wb;
                        ok = true;
                        for (int64_t x = by_lo_off[(size_t)wb]; x < by_lo_off[(size_t)wb + 1] && ok; ++x)
                            ok = admit(grown, order[(size_t)(ov_begin[(size_t)c] + by_lo[(size_t)x])]);
                        if (!ok) {
                            plan.unfit_contig = c;
                            return B200POA_GENERIC_ERROR;
                        }
                    }
                    for (int64_t x = by_lo_off[(size_t)wb]; x < by_lo_off[(size_t)wb + 1]; ++x)
                        members.push_back(by_lo[(size_t)x]);
                    unit_load = grown;
                }
                emit(n_win);
                int64_t taken = 0;
                for (size_t u = units_before; u < plan.units.size(); ++u)
                    taken += plan.units[u].ov_hi - plan.units[u].ov_lo;
                ++plan.split_contigs;
                plan.repeat_overlaps += taken - n_ov;
                continue;
            }
        }
        load = with;
        if (first < 0) first = c;
        last = c;
    }
    close_round();
    /* whole-contig units take a run of the partition as it is; split units hold their own copies */
    if (plan.split_contigs == 0) plan.overlaps = std::move(order);
    else {
        std::vector<int64_t> all;
        all.reserve(plan.overlaps.size() + (size_t)in.n_overlaps);
        for (OverlapUnit& u : plan.units) {
            const int64_t lo = (int64_t)all.size();
            if (u.split) all.insert(all.end(), plan.overlaps.begin() + u.ov_lo, plan.overlaps.begin() + u.ov_hi);
            else all.insert(all.end(), order.begin() + u.ov_lo, order.begin() + u.ov_hi);
            u.ov_hi = lo + (u.ov_hi - u.ov_lo);
            u.ov_lo = lo;
        }
        plan.overlaps.swap(all);
    }
    return B200POA_SUCCESS;
}

} // namespace racon_b200
