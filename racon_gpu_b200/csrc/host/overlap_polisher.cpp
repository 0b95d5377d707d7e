/* overlap_polisher.cpp -- see overlap_polisher.hpp and include/b200poa.h (b200poa_polish_overlaps[_ex|_multi]). */
#include "overlap_polisher.hpp"

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <thread>
#include <vector>

#include "../cuda_buffers.hpp"
#include "b200aln.h"
#include "b200poa.h"
#include "overlap_units.hpp"

namespace racon_b200 {

namespace {

/* everything one worker owns on its device; released on every return */
struct Resources {
    int32_t device = 0;
    b200aln_batch* aligner = nullptr;
    std::vector<b200poa_batch*> poa; /* tier 1's batches, then the second tier's */
    std::vector<cudaStream_t> streams;
    ~Resources() {
        b200buf::DeviceGuard g(device);
        for (b200poa_batch* b : poa) b200poa_batch_destroy(b); /* waits for its stream */
        for (cudaStream_t s : streams) cudaStreamDestroy(s);
        b200aln_batch_destroy(aligner);
    }
};

/* the counters of OverlapPolishOutput one worker adds up */
struct Counters {
    int64_t n_rounds = 0, h2d_bytes = 0, d2h_bytes = 0;
    int64_t tier2_windows = 0, tier2_polished = 0, tier2_batches = 0, exported_windows = 0, exported_bytes = 0;
};

/* what the workers share: the input, the plan, the per-window outputs (each unit writes only the rows of the windows it
 * owns), the exports by unit, the cursor over the units and the first error */
struct Shared {
    const OverlapInput& in;
    const OverlapPolishOptions& opt;
    const OverlapPlan& plan;
    const std::vector<int64_t>& win_off; /* every window's bytes in the contig arena */
    OverlapPolishOutput& out;
    std::vector<OverlapExport>* exports; /* [units] with export_layers, else null */
    b200poa_config cfg;                  /* tier 1: racon's limits */
    int32_t deep_size_cap, deep_seqs_cap;
    bool exact_tier2 = false;            /* with a device list: tier-2 outcomes of each window alone (polish_unit) */
    std::atomic<int64_t> next{0};
    std::atomic<int32_t> error{B200POA_SUCCESS};
    Shared(const OverlapInput& i, const OverlapPolishOptions& o, const OverlapPlan& p, const std::vector<int64_t>& wo,
           OverlapPolishOutput& ou)
        : in(i), opt(o), plan(p), win_off(wo), out(ou), exports(nullptr) {}
    void fail(int32_t st) { /* the first error wins */
        int32_t expected = B200POA_SUCCESS;
        error.compare_exchange_strong(expected, st);
    }
};

/* window gw as its backbone, unpolished (racon's CPU path or window.cpp:68-71 takes it from there) */
void backbone(const Shared& s, int64_t gw, int32_t status) {
    const int64_t a = s.win_off[(size_t)gw], b = s.win_off[(size_t)gw + 1];
    std::memcpy(s.out.cons_out + (size_t)gw * (size_t)s.out.stride, s.in.t_bases + a,
                (size_t)std::min<int64_t>(b - a, s.out.stride));
    s.out.cons_len[gw] = (int32_t)(b - a);
    s.out.polished[gw] = 0;
    s.out.status[gw] = status;
}

/* One device's share of the work: an aligner batch, the POA batches of both tiers and their streams, on the host thread
 * that runs it.  It claims units from the shared cursor until none is left or some worker has failed. */
class Worker {
public:
    Worker(Shared& s, int32_t device, size_t mem, int64_t aligner_budget)
        : s_(s), mem_(mem), aligner_budget_(aligner_budget) {
        r_.device = device;
    }
    Counters c;

    /* eager: create the batches before the first unit is claimed (the only worker); else with the first unit, so that a
     * worker left without a unit allocates nothing */
    void run(bool eager) {
        b200buf::DeviceGuard guard(r_.device);
        bool ready = eager;
        int32_t st = eager ? init() : B200POA_SUCCESS;
        while (st == B200POA_SUCCESS && s_.error.load() == B200POA_SUCCESS) {
            const int64_t u = s_.next.fetch_add(1);
            if (u >= (int64_t)s_.plan.units.size()) break;
            if (!ready) {
                st = init();
                ready = true;
                if (st != B200POA_SUCCESS) break;
            }
            st = polish_unit(u);
        }
        if (st != B200POA_SUCCESS) s_.fail(st);
    }

private:
    Shared& s_;
    size_t mem_;
    int64_t aligner_budget_;
    Resources r_;
    b200poa_config deep_cfg_{};
    b200poa_batch* deep_ = nullptr; /* owned by r_.poa once created */

    int32_t init() {
        const OverlapPolishOptions& opt = s_.opt;
        if (b200aln_batch_create(r_.device, nullptr, aligner_budget_, 0, &r_.aligner) != B200ALN_SUCCESS ||
            b200aln_batch_set_window_length(r_.aligner, opt.window_length, 1) != B200ALN_SUCCESS ||
            b200aln_batch_set_layer_cut(r_.aligner, opt.quality_threshold) != B200ALN_SUCCESS)
            return B200POA_CUDA_ERROR;
        for (int32_t i = 0; i < opt.poa_batches; ++i) {
            cudaStream_t st = nullptr;
            if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) return B200POA_CUDA_ERROR;
            r_.streams.push_back(st);
            b200poa_batch* b = nullptr;
            const int32_t rc = b200poa_batch_create(r_.device, st, mem_, B200POA_OUTPUT_CONSENSUS, &s_.cfg, (int16_t)opt.gap,
                                                    (int16_t)opt.mismatch, (int16_t)opt.match, &b);
            if (rc != B200POA_SUCCESS) return rc;
            r_.poa.push_back(b);
            b200poa_batch_set_option(b, B200POA_OPT_DOWNLOAD_COVERAGE, 0); /* the trim span comes from the device */
        }
        deep_cfg_ = s_.cfg;
        return B200POA_SUCCESS;
    }

    /* the second tier's size for windows whose longest sequence is `longest`: a multiple of 512 less one, within the cap */
    int32_t deep_size(int32_t longest) const {
        return std::min(std::max(1023, (longest + 1 + 511) / 512 * 512 - 1), s_.deep_size_cap);
    }

    /* the second tier's batch re-made with these limits (the one kept so far is released first).  B200POA_SUCCESS,
     * B200POA_INVALID_ARGUMENT when no batch with them fits the device's limits or the memory share, or an error. */
    int32_t make_deep(int32_t n_seqs, int32_t size) {
        const OverlapPolishOptions& opt = s_.opt;
        if (deep_) {
            b200poa_batch_destroy(deep_); /* waits for its stream */
            r_.poa.pop_back();
            deep_ = nullptr;
        } else if (r_.streams.size() == (size_t)opt.poa_batches) {
            cudaStream_t st = nullptr;
            if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) return B200POA_CUDA_ERROR;
            r_.streams.push_back(st);
        }
        b200poa_config_default(&deep_cfg_, size, n_seqs, 256, opt.banded ? B200POA_STATIC_BAND : B200POA_FULL_BAND);
        deep_cfg_.max_nodes_per_graph = std::min(deep_cfg_.max_nodes_per_graph, 32768); /* the engine's 16-bit node ids */
        const int32_t st = b200poa_batch_create(r_.device, r_.streams.back(), mem_, B200POA_OUTPUT_CONSENSUS, &deep_cfg_,
                                                (int16_t)opt.gap, (int16_t)opt.mismatch, (int16_t)opt.match, &deep_);
        if (st != B200POA_SUCCESS) {
            deep_ = nullptr;
            return st;
        }
        r_.poa.push_back(deep_);
        b200poa_batch_set_option(deep_, B200POA_OPT_DOWNLOAD_COVERAGE, 0);
        ++c.tier2_batches;
        return B200POA_SUCCESS;
    }

    /* Without a device list: one batch, sized for the deepest window and the longest sequence a round gives it so far.
     * B200POA_SUCCESS, B200POA_INVALID_ARGUMENT when no batch within the device's limits takes these windows (they then
     * stay with tier 1, as without the second tier), or an error. */
    int32_t ensure_deep(int32_t n_seqs, int32_t longest) {
        int32_t size = deep_size(longest);
        if (deep_ && deep_cfg_.max_sequences_per_poa >= n_seqs && deep_cfg_.max_sequence_size >= size) return B200POA_SUCCESS;
        if (deep_) { /* a round needs larger limits: the new batch keeps the old ones too */
            n_seqs = std::max(n_seqs, deep_cfg_.max_sequences_per_poa);
            size = std::max(size, deep_cfg_.max_sequence_size);
        }
        return make_deep(n_seqs, size);
    }

    /* Unit u: align its overlaps, cut their layers, polish the windows it owns in both tiers, export what is left.  The
     * aligner batch stays as it is until the last POA batch has returned its results. */
    int32_t polish_unit(int64_t u_index) {
        const OverlapInput& in = s_.in;
        const OverlapPolishOptions& opt = s_.opt;
        const OverlapUnit& u = s_.plan.units[(size_t)u_index];
        const std::vector<int64_t>& first_window = s_.plan.first_window;
        const std::vector<int64_t>& win_off = s_.win_off;
        OverlapPolishOutput& out = s_.out;

        b200aln_batch_reset(r_.aligner);
        for (int64_t i = u.ov_lo; i < u.ov_hi; ++i) { /* overlap k with its layer-cut inputs */
            const int64_t k = s_.plan.overlaps[(size_t)i];
            const int32_t ct = in.t_id[k];
            const int64_t q_off2[2] = {in.q_off[k], in.q_off[k + 1]};
            const int64_t t_off2[2] = {in.t_off[ct] + in.t_begin[k], in.t_off[ct] + in.t_end[k]};
            const int64_t fw = first_window[(size_t)ct];
            const int32_t tl = (int32_t)(in.t_off[ct + 1] - in.t_off[ct]);
            const uint8_t hq = in.has_quality && in.q_qual ? in.has_quality[k] : 0;
            const b200aln_layer_inputs li = {&fw, &tl, in.q_qual, &hq};
            int64_t added = 0;
            const int32_t st = b200aln_batch_add_overlaps_ex(r_.aligner, 1, in.q_bases, q_off2, in.t_bases, t_off2,
                                                             in.q_first + k, in.t_begin + k, &li, &added);
            if (st == B200ALN_EXCEEDED_MAX_ALIGNMENTS || st == B200ALN_EXCEEDED_MAX_LENGTH || (st == B200ALN_SUCCESS && added != 1))
                return B200POA_GENERIC_ERROR; /* the plan admitted it: never */
            if (st != B200ALN_SUCCESS) return B200POA_INVALID_ARGUMENT;
        }
        ++c.n_rounds;
        if (b200aln_batch_align_all(r_.aligner) != B200ALN_SUCCESS || b200aln_batch_sync(r_.aligner) != B200ALN_SUCCESS)
            return B200POA_CUDA_ERROR;
        for (int32_t k = 0, n = b200aln_batch_num_alignments(r_.aligner); k < n; ++k) {
            int32_t st = B200ALN_GENERIC_ERROR;
            b200aln_batch_get_alignment(r_.aligner, k, nullptr, nullptr, nullptr, nullptr, &st);
            if (st != B200ALN_SUCCESS) return B200POA_GENERIC_ERROR; /* racon exits when edlib fails (overlap.cpp:215-220) */
        }
        const b200aln_layer* layers = nullptr;
        const int32_t* count = nullptr;
        int64_t n_layers = 0, win_lo = 0, n_win = 0;
        if (b200aln_batch_get_layers(r_.aligner, &layers, &n_layers, &win_lo, &n_win, &count) != B200ALN_SUCCESS)
            return B200POA_GENERIC_ERROR;
        b200aln_batch_info ai;
        b200aln_batch_get_info(r_.aligner, &ai);
        c.h2d_bytes += ai.h2d_bytes;
        c.d2h_bytes += ai.d2h_bytes;
        /* the cut covers the whole contigs of the unit; the unit polishes, exports and writes the windows it owns only */
        const int64_t own_lo = std::max<int64_t>(u.win_lo - win_lo, 0), own_hi = std::min<int64_t>(u.win_hi - win_lo, n_win);

        /* which tier takes each window: the second one those with at least 3 sequences that tier 1 cannot take whole
         * (sizes from the records already on the host), within its caps; tier 1 every other one */
        const b200poa_config& cfg = s_.cfg;
        std::vector<int64_t> tier1, tier2;
        std::vector<int32_t> tier2_size, tier2_seqs; /* per tier-2 window: its own size (deep_size) and sequences */
        if (opt.deep_windows) {
            int32_t deepest = 0, longest = 0;
            int64_t l = 0;
            for (int64_t lw = 0; lw < own_lo; ++lw) l += count[lw];
            for (int64_t lw = own_lo; lw < own_hi; ++lw) {
                const int64_t gw = win_lo + lw;
                const int32_t nseq = 1 + count[lw];
                int32_t len = (int32_t)(win_off[(size_t)gw + 1] - win_off[(size_t)gw]);
                for (const int64_t l1 = l + count[lw]; l < l1; ++l) len = std::max(len, layers[l].length);
                const bool whole = nseq <= cfg.max_sequences_per_poa && len <= cfg.max_sequence_size;
                if (nseq >= 3 && !whole && nseq <= s_.deep_seqs_cap && len <= s_.deep_size_cap) {
                    tier2.push_back(lw);
                    tier2_size.push_back(deep_size(len));
                    tier2_seqs.push_back(nseq);
                    deepest = std::max(deepest, nseq);
                    longest = std::max(longest, len);
                }
            }
            if (!tier2.empty() && !s_.exact_tier2) {
                const int32_t st = ensure_deep(deepest, longest);
                if (st == B200POA_INVALID_ARGUMENT) tier2.clear();
                else if (st != B200POA_SUCCESS) return st;
            }
        }
        for (int64_t lw = own_lo, j = 0; lw < own_hi; ++lw) {
            if (j < (int64_t)tier2.size() && tier2[(size_t)j] == lw) ++j;
            else tier1.push_back(lw);
        }
        if (!s_.exact_tier2) c.tier2_windows += (int64_t)tier2.size();

        /* the POA batches take their tier's windows in order (cudapolisher.cpp:254-276), as runs of consecutive windows,
         * until none is left */
        auto drain = [&](const std::vector<int64_t>& todo, b200poa_batch* const* batches, int32_t n_batches,
                         const b200poa_config& bc, bool second) -> int32_t {
            const size_t per_batch = opt.max_windows_per_batch > 0 ? (size_t)opt.max_windows_per_batch : todo.size();
            std::vector<std::vector<int64_t>> fed((size_t)n_batches);
            std::vector<std::vector<int32_t>> seqs_added((size_t)n_batches);
            size_t pos = 0;
            while (pos < todo.size()) {
                std::vector<int32_t> launched;
                for (int32_t p = 0; p < n_batches && pos < todo.size(); ++p) {
                    b200poa_batch* b = batches[p];
                    b200poa_batch_reset(b);
                    std::vector<int64_t>& ids = fed[(size_t)p];
                    std::vector<int32_t>& added = seqs_added[(size_t)p];
                    ids.clear();
                    while (pos < todo.size() && ids.size() < per_batch) {
                        size_t e = pos + 1;
                        while (e < todo.size() && todo[e] == todo[e - 1] + 1 && e - pos < per_batch - ids.size()) ++e;
                        added.resize(ids.size() + (e - pos));
                        int64_t n_added = 0;
                        const int32_t st = b200poa_batch_add_windows_from_aligner(
                            b, r_.aligner, todo[pos], todo[pos] + (int64_t)(e - pos), win_off.data() + win_lo, in.t_bases,
                            in.t_qual, &n_added, added.data() + ids.size());
                        if (st != B200POA_SUCCESS) return st;
                        for (int64_t k = 0; k < n_added; ++k) ids.push_back(todo[pos + (size_t)k]);
                        pos += (size_t)n_added;
                        if ((size_t)n_added < e - (pos - (size_t)n_added)) break; /* the batch is full */
                    }
                    if (ids.empty()) return B200POA_EXCEEDED_MAXIMUM_SEQUENCE_SIZE; /* one window outgrows an empty batch */
                    const int32_t st = b200poa_batch_generate(b);
                    if (st != B200POA_SUCCESS) return st;
                    launched.push_back(p);
                }
                for (const int32_t p : launched) {
                    b200poa_batch* b = batches[p];
                    const uint8_t* cons = nullptr;
                    const uint16_t* cov = nullptr;
                    const int32_t *len = nullptr, *st = nullptr, *off = nullptr, *tr = nullptr;
                    const int32_t rc = b200poa_batch_get_consensus(b, &cons, &cov, &len, &st, &off, &tr);
                    if (rc != B200POA_SUCCESS) return rc;
                    b200poa_batch_info bi;
                    b200poa_batch_get_info(b, &bi);
                    c.h2d_bytes += bi.h2d_bytes;
                    c.d2h_bytes += bi.d2h_bytes;
                    const std::vector<int64_t>& ids = fed[(size_t)p];
                    /* cuda_polisher.cpp: the per-window results of b200poa_polisher_polish */
                    for (size_t i = 0; i < ids.size(); ++i) {
                        const int64_t lw = ids[i], gw = win_lo + lw;
                        const int64_t nseq = 1 + count[lw];
                        const bool dropped = seqs_added[(size_t)p][i] != nseq - 1;
                        if (nseq < 3 || st[i] != B200POA_SUCCESS || dropped) {
                            int32_t sv = st[i];
                            if (sv == B200POA_SUCCESS && nseq >= 3)
                                sv = nseq - 1 > bc.max_sequences_per_poa ? B200POA_EXCEEDED_MAXIMUM_SEQUENCES_PER_POA
                                                                         : B200POA_EXCEEDED_MAXIMUM_SEQUENCE_SIZE;
                            backbone(s_, gw, sv);
                            continue;
                        }
                        int32_t begin = 0, end = len[i] - 1;
                        if (opt.tgs && opt.trim) { /* window.cpp:118-139, evaluated on the device */
                            const int32_t tb = tr[i] & 0xFFFF, te = tr[i] >> 16;
                            if (tb < te) {
                                begin = tb;
                                end = te;
                            }
                        }
                        const int32_t n = end - begin + 1;
                        std::memcpy(out.cons_out + (size_t)gw * (size_t)out.stride, cons + off[i] + begin,
                                    (size_t)std::min(n, out.stride));
                        out.cons_len[gw] = n;
                        out.polished[gw] = 1;
                        out.status[gw] = B200POA_SUCCESS;
                        if (second) ++c.tier2_polished;
                    }
                }
            }
            return B200POA_SUCCESS;
        };
        int32_t st = drain(tier1, r_.poa.data(), opt.poa_batches, cfg, false);
        if (st != B200POA_SUCCESS) return st;
        if (!s_.exact_tier2) {
            if (!tier2.empty()) st = drain(tier2, &deep_, 1, deep_cfg_, true);
            if (st != B200POA_SUCCESS) return st;
        } else if (!tier2.empty()) {
            /* With a device list a window's outcome must not depend on the batch a worker kept from its earlier units:
             * the batch's size sets the graph's node cap (3 or 4 x size), the consensus cap (2 x size) and the score
             * cells' width.  A window the engine polishes within some limits gets the same consensus within any larger
             * ones, so each window climbs the sizes from its own (deep_size) in steps of 512, starting at the kept
             * batch's size when that is larger, until it is polished, fails for a reason no size changes, or no larger
             * batch can be created.  It ends polished exactly when the largest batch the memory share allows polishes
             * it, and unpolished with that attempt's status otherwise.  Windows no batch can take go to tier 1, as
             * without the second tier. */
            std::vector<size_t> pending(tier2.size());
            std::vector<uint8_t> ran(tier2.size(), 0);
            for (size_t i = 0; i < tier2.size(); ++i) pending[i] = i;
            int32_t size = *std::min_element(tier2_size.begin(), tier2_size.end());
            if (deep_) size = std::max(size, deep_cfg_.max_sequence_size);
            while (!pending.empty()) {
                std::vector<int64_t> run;
                int32_t seqs = 0;
                for (size_t i : pending)
                    if (tier2_size[i] <= size) {
                        run.push_back(tier2[i]);
                        seqs = std::max(seqs, tier2_seqs[i]);
                    }
                if (!run.empty()) {
                    if (!deep_ || deep_cfg_.max_sequence_size != size || deep_cfg_.max_sequences_per_poa < seqs) {
                        st = make_deep(std::max(seqs, deep_ ? deep_cfg_.max_sequences_per_poa : 0), size);
                        if (st == B200POA_INVALID_ARGUMENT) break; /* nor any larger one */
                        if (st != B200POA_SUCCESS) return st;
                    }
                    st = drain(run, &deep_, 1, deep_cfg_, true);
                    if (st != B200POA_SUCCESS) return st;
                    std::vector<size_t> left;
                    for (size_t i : pending) {
                        if (tier2_size[i] > size) {
                            left.push_back(i);
                            continue;
                        }
                        ran[i] = 1;
                        const int64_t gw = win_lo + tier2[i];
                        const int32_t sv = out.status[gw];
                        const bool size_bound = sv == B200POA_NODE_COUNT_EXCEEDED_MAXIMUM_GRAPH_SIZE ||
                                                sv == B200POA_EDGE_COUNT_EXCEEDED_MAXIMUM_GRAPH_SIZE ||
                                                sv == B200POA_SEQ_LEN_EXCEEDED_MAXIMUM_NODES_PER_WINDOW ||
                                                sv == B200POA_SCORE_RANGE_EXCEEDED || sv == B200POA_GENERIC_ERROR;
                        if (!out.polished[gw] && size_bound) left.push_back(i);
                    }
                    pending.swap(left);
                }
                if (size >= s_.deep_size_cap || pending.empty()) break;
                size = std::min(size + 512, s_.deep_size_cap);
            }
            std::vector<int64_t> leftover;
            for (size_t i = 0; i < tier2.size(); ++i) {
                if (ran[i]) ++c.tier2_windows;
                else leftover.push_back(tier2[i]);
            }
            if (!leftover.empty()) st = drain(leftover, r_.poa.data(), opt.poa_batches, cfg, false);
            if (st != B200POA_SUCCESS) return st;
        }

        /* the windows left unpolished that racon's CPU pass would still polish (window.cpp:68-71 leaves those with
         * fewer than 3 sequences as they are): their layers from the device, their backbones from the contigs */
        if (!s_.exports) return B200POA_SUCCESS;
        std::vector<int64_t> ids;
        for (int64_t lw = own_lo; lw < own_hi; ++lw)
            if (1 + count[lw] >= 3 && !out.polished[win_lo + lw]) ids.push_back(lw);
        if (ids.empty()) return B200POA_SUCCESS;
        b200aln_export ex;
        if (b200aln_batch_export_layers(r_.aligner, (int64_t)ids.size(), ids.data(), &ex) != B200ALN_SUCCESS)
            return B200POA_CUDA_ERROR;
        c.h2d_bytes += ex.h2d_bytes;
        c.d2h_bytes += ex.d2h_bytes;
        c.exported_bytes += ex.d2h_bytes;
        c.exported_windows += (int64_t)ids.size();
        OverlapExport& e = (*s_.exports)[(size_t)u_index];
        auto push = [&](const uint8_t* bases, const int8_t* wts, int64_t n, uint8_t has_w, int32_t bg, int32_t en) {
            e.bases.insert(e.bases.end(), bases, bases + n);
            e.weights.insert(e.weights.end(), wts, wts + n);
            e.has_weights.push_back(has_w);
            e.begins.push_back(bg);
            e.ends.push_back(en);
            e.seq_off.push_back(e.seq_off.back() + n);
        };
        std::vector<int8_t> bb_w;
        for (size_t i = 0; i < ids.size(); ++i) {
            const int64_t gw = win_lo + ids[i], a = win_off[(size_t)gw], n = win_off[(size_t)gw + 1] - a;
            bb_w.resize((size_t)n);
            for (int64_t k = 0; k < n; ++k) bb_w[(size_t)k] = in.t_qual ? (int8_t)((int32_t)in.t_qual[a + k] - 33) : 0;
            e.window_ids.push_back(gw);
            push(in.t_bases + a, bb_w.data(), n, 1, 0, 0); /* window.cpp:35-37 */
            for (int64_t l = ex.win_layer_off[i]; l < ex.win_layer_off[i + 1]; ++l) {
                const b200aln_layer& L = ex.layers[l];
                push(ex.bases + ex.seq_off[l], ex.weights + ex.seq_off[l], ex.seq_off[l + 1] - ex.seq_off[l],
                     L.has_quality ? 1 : 0, L.begin, L.end);
            }
            e.win_seq_off.push_back((int64_t)e.has_weights.size());
        }
        return B200POA_SUCCESS;
    }
};

/* src appended to dst, offsets shifted */
void append_export(OverlapExport& dst, const OverlapExport& src) {
    const int64_t seq0 = (int64_t)dst.has_weights.size(), byte0 = (int64_t)dst.bases.size();
    dst.window_ids.insert(dst.window_ids.end(), src.window_ids.begin(), src.window_ids.end());
    for (size_t i = 1; i < src.win_seq_off.size(); ++i) dst.win_seq_off.push_back(seq0 + src.win_seq_off[i]);
    for (size_t i = 1; i < src.seq_off.size(); ++i) dst.seq_off.push_back(byte0 + src.seq_off[i]);
    dst.bases.insert(dst.bases.end(), src.bases.begin(), src.bases.end());
    dst.weights.insert(dst.weights.end(), src.weights.begin(), src.weights.end());
    dst.has_weights.insert(dst.has_weights.end(), src.has_weights.begin(), src.has_weights.end());
    dst.begins.insert(dst.begins.end(), src.begins.begin(), src.begins.end());
    dst.ends.insert(dst.ends.end(), src.ends.begin(), src.ends.end());
}

/* The whole job on workers on `devices` (one per entry; a device listed twice runs two), the units split at window
 * boundaries when `split`. */
int32_t run(const OverlapInput& in, const OverlapPolishOptions& opt, const std::vector<int32_t>& devices, bool split,
            OverlapPolishOutput& out) {
    out.n_rounds = out.h2d_bytes = out.d2h_bytes = 0;
    out.tier2_windows = out.tier2_polished = out.tier2_batches = out.exported_windows = out.exported_bytes = 0;
    out.split_contigs = out.repeat_overlaps = 0;
    out.unfit_contig = -1;
    const int32_t w = opt.window_length;
    if (w <= 0 || opt.poa_batches <= 0 || in.n_contigs < 0 || in.n_overlaps < 0 || !in.t_off || !out.cons_out ||
        !out.cons_len || !out.polished || !out.status || out.stride <= 0 || devices.empty())
        return B200POA_INVALID_ARGUMENT;
    if (in.n_overlaps > 0 && (!in.t_id || !in.t_begin || !in.t_end || !in.q_bases || !in.q_off || !in.q_first))
        return B200POA_INVALID_ARGUMENT;

    /* memory: free bytes read once per device before any worker allocates, a share per POA batch, one for the aligner
     * batch and one for the second tier of every worker on it */
    std::map<int32_t, int32_t> per_device;
    for (int32_t d : devices) ++per_device[d];
    std::map<int32_t, size_t> mem_of;
    for (const auto& dn : per_device) {
        size_t mem = opt.mem_per_poa_batch;
        if (mem == 0) {
            b200buf::DeviceGuard guard(dn.first);
            size_t free_b = 0, total = 0;
            if (cudaMemGetInfo(&free_b, &total) != cudaSuccess) return B200POA_CUDA_ERROR;
            mem = (size_t)(0.9 * (double)free_b / ((double)dn.second * (opt.poa_batches + 1 + (opt.deep_windows ? 1 : 0))));
        }
        mem_of[dn.first] = mem;
    }
    if (split) { /* with a device list every worker gets the smallest share: which unit it takes cannot matter */
        size_t least = SIZE_MAX;
        for (const auto& dm : mem_of) least = std::min(least, dm.second);
        for (auto& dm : mem_of) dm.second = least;
    }
    int64_t budget = INT64_MAX; /* the plan holds for the smallest aligner batch */
    for (const auto& dm : mem_of) budget = std::min<int64_t>(budget, opt.aligner_mem > 0 ? opt.aligner_mem : (int64_t)dm.second);

    OverlapPlan plan;
    const int32_t pst = plan_overlap_units(in, w, budget, split, plan);
    out.unfit_contig = plan.unfit_contig;
    if (pst != B200POA_SUCCESS) return pst;
    out.split_contigs = plan.split_contigs;
    out.repeat_overlaps = plan.repeat_overlaps;

    /* every window's bytes in the contig arena: the windows of one contig are consecutive and the next contig starts
     * where the last window ends; every window starts as its backbone */
    const int64_t n_windows = plan.first_window.back();
    std::vector<int64_t> win_off((size_t)n_windows + 1, 0);
    for (int64_t c = 0, wi = 0; c < in.n_contigs; ++c) {
        const int64_t len = in.t_off[c + 1] - in.t_off[c];
        for (int64_t j = 0; j < len; j += w, ++wi) win_off[(size_t)wi] = in.t_off[c] + j;
        win_off[(size_t)plan.first_window[(size_t)c + 1]] = in.t_off[c + 1];
    }
    Shared s(in, opt, plan, win_off, out);
    for (int64_t gw = 0; gw < n_windows; ++gw) backbone(s, gw, B200POA_SUCCESS);
    std::vector<OverlapExport> exports;
    if (opt.export_layers && out.exported) {
        exports.resize(plan.units.size());
        s.exports = &exports;
    }
    b200poa_config_default(&s.cfg, 1023, 200, 256, opt.banded ? B200POA_STATIC_BAND : B200POA_FULL_BAND); /* cudabatch.cpp:56-59 */
    s.deep_size_cap = opt.deep_max_sequence_size > 0 ? std::min(opt.deep_max_sequence_size, 16380) : 16380;
    s.deep_seqs_cap = opt.deep_max_sequences_per_poa > 0 ? std::min(opt.deep_max_sequences_per_poa, 65535) : 65535;
    s.exact_tier2 = split;

    std::vector<std::unique_ptr<Worker>> workers;
    for (int32_t d : devices) {
        const size_t mem = mem_of[d];
        workers.emplace_back(new Worker(s, d, mem, opt.aligner_mem > 0 ? opt.aligner_mem : (int64_t)mem));
    }
    if (workers.size() == 1) {
        workers[0]->run(true);
    } else {
        std::vector<std::thread> threads;
        try {
            for (auto& wk : workers) threads.emplace_back([&s, p = wk.get()] {
                try {
                    p->run(false);
                } catch (...) {
                    s.fail(B200POA_GENERIC_ERROR);
                }
            });
        } catch (...) {
            s.fail(B200POA_GENERIC_ERROR);
        }
        for (std::thread& t : threads) t.join();
    }
    for (const auto& wk : workers) {
        const Counters& c = wk->c;
        out.n_rounds += c.n_rounds;
        out.h2d_bytes += c.h2d_bytes;
        out.d2h_bytes += c.d2h_bytes;
        out.tier2_windows += c.tier2_windows;
        out.tier2_polished += c.tier2_polished;
        out.tier2_batches += c.tier2_batches;
        out.exported_windows += c.exported_windows;
        out.exported_bytes += c.exported_bytes;
    }
    workers.clear(); /* every batch released before the call returns */
    const int32_t st = s.error.load();
    if (st != B200POA_SUCCESS) return st;
    /* the exports in ascending window id: the units' order */
    for (const OverlapExport& e : exports) append_export(*out.exported, e);
    return B200POA_SUCCESS;
}

} // namespace

int64_t overlap_window_count(const OverlapInput& in, int32_t w) {
    int64_t n = 0;
    for (int64_t c = 0; c < in.n_contigs; ++c) n += (in.t_off[c + 1] - in.t_off[c] + w - 1) / w;
    return n;
}

int32_t polish_overlaps(const OverlapInput& in, const OverlapPolishOptions& opt, OverlapPolishOutput& out) {
    return run(in, opt, {opt.device}, false, out);
}

int32_t polish_overlaps(const OverlapInput& in, const OverlapPolishOptions& opt, const std::vector<int32_t>& devices,
                        OverlapPolishOutput& out) {
    out.unfit_contig = -1;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n < 1) {
        cudaGetLastError();
        return B200POA_CUDA_ERROR;
    }
    std::vector<int32_t> d = devices;
    if (d.empty())
        for (int32_t i = 0; i < n; ++i) d.push_back(i);
    for (int32_t x : d)
        if (x < 0 || x >= n) return B200POA_INVALID_ARGUMENT; /* before anything is allocated */
    return run(in, opt, d, true, out);
}

} // namespace racon_b200

namespace {

racon_b200::OverlapPolishOptions options_from(const b200poa_overlap_options* o) {
    racon_b200::OverlapPolishOptions opt;
    opt.device = o->device_id;
    opt.poa_batches = o->poa_batches;
    opt.mem_per_poa_batch = o->mem_per_poa_batch;
    opt.aligner_mem = o->aligner_mem;
    opt.window_length = o->window_length;
    opt.quality_threshold = o->quality_threshold;
    opt.banded = o->banded;
    opt.match = o->match;
    opt.mismatch = o->mismatch;
    opt.gap = o->gap;
    opt.tgs = o->tgs != 0;
    opt.trim = o->trim != 0;
    opt.max_windows_per_batch = o->max_windows_per_batch;
    return opt;
}

template <class T>
T* copy_out(const std::vector<T>& v) { /* malloc'd, so that b200poa_free_export can release it from C */
    T* p = static_cast<T*>(std::malloc(std::max<size_t>(v.size(), 1) * sizeof(T)));
    if (p && !v.empty()) std::memcpy(p, v.data(), v.size() * sizeof(T));
    return p;
}

} // namespace

extern "C" int32_t b200poa_polish_overlaps(const b200poa_overlap_options* o, int64_t n_contigs, const uint8_t* t_bases,
                                           const int64_t* t_off, const uint8_t* t_qual, int64_t n_overlaps,
                                           const int32_t* t_id, const int32_t* t_begin, const int32_t* t_end,
                                           const uint8_t* q_bases, const int64_t* q_off, const uint8_t* q_qual,
                                           const uint8_t* has_quality, const int32_t* q_first, uint8_t* cons_out,
                                           int32_t stride, int32_t* cons_len, uint8_t* polished, int32_t* status_out,
                                           int64_t* n_rounds, int64_t* h2d_bytes, int64_t* d2h_bytes,
                                           int64_t* unfit_contig) {
    if (!o) return B200POA_INVALID_ARGUMENT;
    const racon_b200::OverlapPolishOptions opt = options_from(o);
    const racon_b200::OverlapInput in{n_contigs, t_bases, t_off, t_qual, n_overlaps, t_id, t_begin, t_end,
                                      q_bases, q_off, q_qual, has_quality, q_first};
    racon_b200::OverlapPolishOutput out{cons_out, stride, cons_len, polished, status_out};
    const int32_t st = racon_b200::polish_overlaps(in, opt, out);
    if (n_rounds) *n_rounds = out.n_rounds;
    if (h2d_bytes) *h2d_bytes = out.h2d_bytes;
    if (d2h_bytes) *d2h_bytes = out.d2h_bytes;
    if (unfit_contig) *unfit_contig = out.unfit_contig;
    return st;
}

namespace {

/* _ex and _multi: devices null = the one of opt->device_id, unsplit */
int32_t polish_overlaps_ex(const b200poa_overlap_options* o, b200poa_overlap_ex* ex, const std::vector<int32_t>* devices,
                           const racon_b200::OverlapInput& in, racon_b200::OverlapPolishOutput& out, int64_t* n_rounds,
                           int64_t* h2d_bytes, int64_t* d2h_bytes, int64_t* unfit_contig) {
    racon_b200::OverlapPolishOptions opt = options_from(o);
    racon_b200::OverlapExport exported;
    if (ex) {
        ex->exported = b200poa_overlap_export{};
        ex->tier2_windows = ex->tier2_polished = ex->tier2_batches = ex->exported_windows = ex->exported_bytes = 0;
        if (ex->deep_max_sequence_size < 0 || ex->deep_max_sequences_per_poa < 0) return B200POA_INVALID_ARGUMENT;
        opt.deep_windows = ex->deep_windows != 0;
        opt.export_layers = ex->export_layers != 0;
        opt.deep_max_sequence_size = ex->deep_max_sequence_size;
        opt.deep_max_sequences_per_poa = ex->deep_max_sequences_per_poa;
        out.exported = &exported;
    }
    int32_t st = devices ? racon_b200::polish_overlaps(in, opt, *devices, out) : racon_b200::polish_overlaps(in, opt, out);
    if (n_rounds) *n_rounds = out.n_rounds;
    if (h2d_bytes) *h2d_bytes = out.h2d_bytes;
    if (d2h_bytes) *d2h_bytes = out.d2h_bytes;
    if (unfit_contig) *unfit_contig = out.unfit_contig;
    if (!ex) return st;
    ex->tier2_windows = out.tier2_windows;
    ex->tier2_polished = out.tier2_polished;
    ex->tier2_batches = out.tier2_batches;
    ex->exported_windows = out.exported_windows;
    ex->exported_bytes = out.exported_bytes;
    if (st == B200POA_SUCCESS && opt.export_layers) {
        b200poa_overlap_export& e = ex->exported;
        e.n_windows = (int64_t)exported.window_ids.size();
        e.n_sequences = (int64_t)exported.has_weights.size();
        e.window_ids = copy_out(exported.window_ids);
        e.win_seq_off = copy_out(exported.win_seq_off);
        e.seq_off = copy_out(exported.seq_off);
        e.bases = copy_out(exported.bases);
        e.weights = copy_out(exported.weights);
        e.has_weights = copy_out(exported.has_weights);
        e.begins = copy_out(exported.begins);
        e.ends = copy_out(exported.ends);
        if (!e.window_ids || !e.win_seq_off || !e.seq_off || !e.bases || !e.weights || !e.has_weights || !e.begins ||
            !e.ends) {
            b200poa_free_export(&e);
            st = B200POA_GENERIC_ERROR;
        }
    }
    return st;
}

} // namespace

extern "C" int32_t b200poa_polish_overlaps_ex(const b200poa_overlap_options* o, b200poa_overlap_ex* ex, int64_t n_contigs,
                                              const uint8_t* t_bases, const int64_t* t_off, const uint8_t* t_qual,
                                              int64_t n_overlaps, const int32_t* t_id, const int32_t* t_begin,
                                              const int32_t* t_end, const uint8_t* q_bases, const int64_t* q_off,
                                              const uint8_t* q_qual, const uint8_t* has_quality, const int32_t* q_first,
                                              uint8_t* cons_out, int32_t stride, int32_t* cons_len, uint8_t* polished,
                                              int32_t* status_out, int64_t* n_rounds, int64_t* h2d_bytes,
                                              int64_t* d2h_bytes, int64_t* unfit_contig) {
    if (!o || !ex) return B200POA_INVALID_ARGUMENT;
    const racon_b200::OverlapInput in{n_contigs, t_bases, t_off, t_qual, n_overlaps, t_id, t_begin, t_end,
                                      q_bases, q_off, q_qual, has_quality, q_first};
    racon_b200::OverlapPolishOutput out{cons_out, stride, cons_len, polished, status_out};
    return polish_overlaps_ex(o, ex, nullptr, in, out, n_rounds, h2d_bytes, d2h_bytes, unfit_contig);
}

extern "C" int32_t b200poa_polish_overlaps_multi(const b200poa_overlap_options* o, b200poa_overlap_ex* ex,
                                                 int32_t n_devices, const int32_t* device_ids, int64_t n_contigs,
                                                 const uint8_t* t_bases, const int64_t* t_off, const uint8_t* t_qual,
                                                 int64_t n_overlaps, const int32_t* t_id, const int32_t* t_begin,
                                                 const int32_t* t_end, const uint8_t* q_bases, const int64_t* q_off,
                                                 const uint8_t* q_qual, const uint8_t* has_quality,
                                                 const int32_t* q_first, uint8_t* cons_out, int32_t stride,
                                                 int32_t* cons_len, uint8_t* polished, int32_t* status_out,
                                                 int64_t* n_rounds, int64_t* h2d_bytes, int64_t* d2h_bytes,
                                                 int64_t* unfit_contig, int64_t* split_contigs, int64_t* repeat_overlaps) {
    if (unfit_contig) *unfit_contig = -1;
    if (!o || n_devices < 0 || (n_devices > 0 && !device_ids)) return B200POA_INVALID_ARGUMENT;
    const std::vector<int32_t> devices(device_ids, device_ids + n_devices);
    const racon_b200::OverlapInput in{n_contigs, t_bases, t_off, t_qual, n_overlaps, t_id, t_begin, t_end,
                                      q_bases, q_off, q_qual, has_quality, q_first};
    racon_b200::OverlapPolishOutput out{cons_out, stride, cons_len, polished, status_out};
    const int32_t st = polish_overlaps_ex(o, ex, &devices, in, out, n_rounds, h2d_bytes, d2h_bytes, unfit_contig);
    if (split_contigs) *split_contigs = out.split_contigs;
    if (repeat_overlaps) *repeat_overlaps = out.repeat_overlaps;
    return st;
}

extern "C" void b200poa_free_export(b200poa_overlap_export* e) {
    if (!e) return;
    std::free(e->window_ids);
    std::free(e->win_seq_off);
    std::free(e->seq_off);
    std::free(e->bases);
    std::free(e->weights);
    std::free(e->has_weights);
    std::free(e->begins);
    std::free(e->ends);
    *e = b200poa_overlap_export{};
}
