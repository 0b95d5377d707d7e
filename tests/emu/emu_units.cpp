/*
 * emu_units.cpp -- host build of the overlap driver's planner (racon_gpu_b200/csrc/host/overlap_units.hpp) and of the
 * aligner batch's admission rule it shares with b200aln.cu (host/aln_admission.hpp; TEST INFRASTRUCTURE).
 * Never linked into the product library.
 */
#include <cstdint>
#include <cstring>

#include "../../racon_gpu_b200/csrc/host/overlap_units.hpp"

extern "C" {

/* aln_admit on a load passed in and out as {var_bytes, max_len, n_jobs} */
int32_t emu_admit(int64_t* load, int64_t budget, int32_t window_length, int32_t layer_cut, int32_t n, int32_t m,
                  int32_t t_begin) {
    b200aln::AlnLoad l;
    l.var_bytes = load[0];
    l.max_len = (int32_t)load[1];
    l.n_jobs = (size_t)load[2];
    const int32_t st = b200aln::aln_admit(l, budget, window_length, layer_cut != 0, n, m, t_begin);
    load[0] = l.var_bytes;
    load[1] = l.max_len;
    load[2] = (int64_t)l.n_jobs;
    return st;
}

/* plan_overlap_units over the columns the planner reads.  units: [units_cap][6] (contig, win_lo, win_hi, ov_lo, ov_hi,
 * split); overlaps: [ov_cap]; stats: split_contigs, repeat_overlaps, unfit_contig, number of units, number of overlaps.
 * Returns the planner's status, or -100 when a capacity is too small. */
int32_t emu_plan_units(int64_t n_contigs, const int64_t* t_off, int64_t n_overlaps, const int32_t* t_id,
                       const int32_t* t_begin, const int32_t* t_end, const int64_t* q_off, const int32_t* q_first,
                       int32_t window_length, int64_t budget, int32_t split, int64_t* units, int64_t units_cap,
                       int64_t* overlaps, int64_t ov_cap, int64_t* stats) {
    const racon_b200::OverlapInput in{n_contigs, nullptr, t_off, nullptr, n_overlaps, t_id, t_begin, t_end,
                                      nullptr, q_off, nullptr, nullptr, q_first};
    racon_b200::OverlapPlan plan;
    const int32_t st = racon_b200::plan_overlap_units(in, window_length, budget, split != 0, plan);
    stats[0] = plan.split_contigs;
    stats[1] = plan.repeat_overlaps;
    stats[2] = plan.unfit_contig;
    stats[3] = (int64_t)plan.units.size();
    stats[4] = (int64_t)plan.overlaps.size();
    if (st != B200POA_SUCCESS) return st;
    if ((int64_t)plan.units.size() > units_cap || (int64_t)plan.overlaps.size() > ov_cap) return -100;
    for (size_t i = 0; i < plan.units.size(); ++i) {
        const racon_b200::OverlapUnit& u = plan.units[i];
        const int64_t row[6] = {u.contig, u.win_lo, u.win_hi, u.ov_lo, u.ov_hi, u.split ? 1 : 0};
        std::memcpy(units + 6 * i, row, sizeof(row));
    }
    if (!plan.overlaps.empty()) std::memcpy(overlaps, plan.overlaps.data(), plan.overlaps.size() * sizeof(int64_t));
    return st;
}

} // extern "C"
