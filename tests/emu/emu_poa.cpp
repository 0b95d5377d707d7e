/*
 * emu_poa.cpp -- lock-step CPU emulation of the one-window-per-warp engine (TEST INFRASTRUCTURE).
 *
 * Compiles racon_gpu_b200/csrc/poa_core.cuh in its host flavour (poa_simt.cuh: POA_LANES loops over
 * 32 lanes, collectives are plain loops) together with a scalar twin of the CUDA DP fill that
 * produces the identical skewed int16 band matrix.  The CPU test-suite runs it against the oracle
 * so that every graph phase of the kernel (row program, traceback, parallel add_alignment,
 * per-root topological sort, consensus) and the band definition are checked without a GPU.
 * Never linked into the product library.
 */
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <atomic>
#include <vector>

/* Traceback reach report: per window, how often the traceback took each of its paths (tests/emu_lib.py names the
 * fields, tests/tb_cases.py reads them).  traceback() and traceback_i32() count through POA_TB_REACH; the twin check
 * after every traceback (ScalarFill::traceback_twin) counts the rest. */
enum TbReach {
    TB_tracebacks = 0, /* tracebacks run (every adaptive try)                                              */
    TB_tile_loads,     /* tiles loaded                                                                     */
    TB_reanchors,      /* tiles re-anchored at the current cell because a step's data was not in the tile   */
    TB_global_npred,   /* steps read from global memory: more than 32 in-edges                              */
    TB_global_pred_cap,/* ... <= 32 in-edges, but CSR entries past TB_PRED_CAP                              */
    TB_global_far,     /* ... a predecessor more than TB_ROWS - 1 rows back after the re-anchor             */
    TB_common_steps,   /* steps of a row with one in-edge whose source is in the tile                      */
    TB_tile_steps,     /* other steps resolved in the tile                                                 */
    TB_neg_chunk_steps,/* tile steps that read a NEG-filled chunk (out of the row's band)                  */
    TB_band_hits,      /* adaptive band: tiles anchored within TB_EDGE_MARGIN of a band edge               */
    TB_row0_tail32,    /* tracebacks with a row-0 tail of 32 or more horizontal moves                      */
    TB_row0_tail64,    /* ... of 64 or more                                                                */
    TB_vrun32,         /* tracebacks with a run of 32 or more vertical moves                               */
    TB_count_mod0,     /* tracebacks whose entry count is 0 mod 32                                         */
    TB_count_mod1,     /* ... 1 mod 32                                                                     */
    TB_count_mod31,    /* ... 31 mod 32                                                                    */
    TB_i32_reads,      /* tracebacks on 32-bit cells (traceback_i32)                                       */
    TB_partial_reads,  /* tracebacks against a subgraph (partial-span layer)                               */
    TB_twin_mismatches,/* tracebacks whose alignment differs from the scalar twin's                        */
    TB_FIELDS
};
thread_local int32_t* tb_reach_now = nullptr; /* the window the calling thread works on, or nullptr */
#define POA_TB_REACH(field) (tb_reach_now ? (void)(tb_reach_now[TB_##field] += 1) : (void)0)
#define POA_TB_REACH_IF(cond, field) ((cond) ? POA_TB_REACH(field) : (void)0)
#define POA_TB_TWIN(fill, ...) (fill).traceback_twin(__VA_ARGS__)
#define POA_ALN_DIGEST 1 /* WindowView::aln_digest / aln_count: set for every window below */

/* Graph reach report: per window, how often add_alignment, the sorts, the subgraph and the consensus took each of their
 * paths (tests/emu_lib.py names the fields, tests/graph_cases.py reads them).  poa_core.cuh counts through
 * POA_GRAPH_REACH; the twins (GraphTwin below) count the rest. */
enum GraphReach {
    GR_new_nodes32 = 0, /* reads that add 32 or more new nodes                                           */
    GR_new_nodes64,     /* ... 64 or more                                                                 */
    GR_run_cross32,     /* new unaligned nodes whose run's root walk crosses a 32-position boundary       */
    GR_join1,           /* a new node joins a clique of 1 node (GR_join1 + k: of k + 1 nodes, up to 7)    */
    GR_join7 = GR_join1 + 6,
    GR_clique_mate,     /* read positions resolved to an existing aligned node of the same letter         */
    GR_edge_bumped,     /* edges whose weight a read added to                                              */
    GR_edge_created,    /* edges created                                                                   */
    GR_edge_same_root,  /* ... inside one root of the per-root sort (the root is marked dirty)             */
    GR_edge_cross_root, /* ... across two roots                                                            */
    GR_du_all,          /* groups of add_alignment_edges with all POA_ADD_DU walks of lane 0 active        */
    GR_walk_over32,     /* in-edge walks of more than 32 edges                                             */
    GR_read_len1,       /* reads of one base (they bump no coverage)                                       */
    GR_const_weights,   /* reads whose bases all weigh one constant                                        */
    GR_base_weights,    /* reads with per-base weights                                                     */
    GR_weight0,         /* reads of constant weight 0, and bases of weight 0                               */
    GR_dirty_over32,    /* sorts with more than 32 dirty multi-node roots (more than one batch of DFS)      */
    GR_sub_serial,      /* subgraphs ordered by mark_subgraph_serial because the graph exceeds sroot_cap   */
    GR_sweep_iter2,     /* chunks of the subgraph sweep that took 2 or more iterations                     */
    GR_sweep_iter3,     /* ... 3 or more                                                                   */
    GR_straddle,        /* chunks whose lower edge cuts a clique                                           */
    GR_straddle8,       /* ... a clique of KA + 1 nodes                                                    */
    GR_sub_begin0,      /* partial-span reads whose span begins at backbone node 0                         */
    GR_sub_end_last,    /* ... ends at the last backbone node                                              */
    GR_tie_in_block,    /* consensus: tied in-edges resolved literally, predecessor in the same 32-rank block */
    GR_tie_pre_block,   /* ... predecessor before the block                                                */
    GR_tie_equal_pred,  /* ... equal weight and equal predecessor score: '<=' picks the later edge         */
    GR_block_max_tie,   /* blocks whose maximum score is held by two or more nodes                         */
    GR_max_tie_across,  /* blocks whose maximum equals the running maximum of the earlier blocks           */
    GR_topsort_twins,   /* per-root sorts checked against topsort_serial                                   */
    GR_sub_twins,       /* warp-sweep subgraphs checked against mark_subgraph_serial                       */
    GR_cons_twins,      /* consensus_scores_full checked against spoa's literal loop                       */
    GR_twin_mismatches, /* twin checks that found a difference                                             */
    GR_FIELDS
};
/* the first twin check of a window that found a difference: kind (0 sort, 1 subgraph, 2 consensus), read (processing
 * position; the consensus: -1), index (rank, member position or node; -1: the count or max_id), the twin's value, the
 * engine's value */
constexpr int GR_MISMATCH_INTS = 5;
thread_local int32_t* graph_reach_now = nullptr; /* the window the calling thread works on, or nullptr */
#define POA_GRAPH_REACH(field) (graph_reach_now ? (void)(graph_reach_now[GR_##field] += 1) : (void)0)
#define POA_GRAPH_REACH_IF(cond, field) ((cond) ? POA_GRAPH_REACH(field) : (void)0)
#define POA_GRAPH_REACH_AT(field, k) (graph_reach_now ? (void)(graph_reach_now[GR_##field + (k)] += 1) : (void)0)
#define POA_GRAPH_TWIN(what, ...) graph_twin_##what(__VA_ARGS__)
#define POA_GRAPH_DIGEST 1 /* WindowView::graph_digest ..., WindowOut::cons_digest / cons_rounds: set below */
namespace b200poa {
struct Slot;
struct Params;
struct WinState;
}
static void graph_twin_topsort(const b200poa::Slot& s, const b200poa::Params& p, const b200poa::WinState& st, int32_t r);
static void graph_twin_subgraph(const b200poa::Slot& s, const b200poa::Params& p, const b200poa::WinState& st,
                                int32_t r, int32_t begin, int32_t end, int32_t n, int32_t cap);
static void graph_twin_consensus(const b200poa::Slot& s, int32_t N, int32_t max_id);
static void graph_twin_sweep_chunk(const b200poa::Slot& s, int32_t hi);
static void graph_twin_sweep_step();

#include "../../racon_gpu_b200/csrc/poa_core.cuh"

using namespace b200poa;

/* Twins of the graph phases.  Each runs on shadow copies of the arrays it writes (the graph itself is only read), so
 * that it cannot change what the engine does next. */
struct GraphTwin {
    int32_t* reach = nullptr;    /* this window's report (GR_FIELDS) */
    int32_t* mismatch = nullptr; /* this window's first mismatch (GR_MISMATCH_INTS), or nullptr */
    int32_t sweep_steps = 0;
    std::vector<uint8_t> marks, check;
    std::vector<uint16_t> stack, node_at, rank_of, sub_at, sub_rank;
    std::vector<uint32_t> row_meta, roff;
    std::vector<int32_t> c_score, c_pred;

    void size(const Params& p) {
        const size_t MN = (size_t)p.max_nodes, ME = (size_t)p.max_edges;
        marks.resize(MN);
        check.resize(MN);
        stack.resize(ME + (KA + 2) * MN);
        node_at.resize(MN);
        rank_of.resize(MN);
        sub_at.resize(MN);
        sub_rank.resize(MN);
        row_meta.resize(MN);
        roff.resize(MN + 1);
        c_score.resize(MN);
        c_pred.resize(MN);
    }
    Slot shadow(const Slot& s) {
        Slot t = s;
        t.marks = marks.data();
        t.check = check.data();
        t.stack = stack.data();
        t.node_at = node_at.data();
        t.rank_of = rank_of.data();
        t.sub_at = sub_at.data();
        t.sub_rank = sub_rank.data();
        t.row_meta = row_meta.data();
        t.roff = roff.data();
        t.c_score = c_score.data();
        t.c_pred = c_pred.data();
        return t;
    }
    void report(int32_t kind, int32_t r, int32_t idx, int32_t twin, int32_t eng) {
        reach[GR_twin_mismatches] += 1;
        if (mismatch && mismatch[0] < 0) {
            const int32_t m[GR_MISMATCH_INTS] = {kind, r, idx, twin, eng};
            std::copy(m, m + GR_MISMATCH_INTS, mismatch);
        }
    }
};
thread_local GraphTwin* graph_twin_now = nullptr;

/* after every per-root sort: topsort_serial must give the same rank order */
static void graph_twin_topsort(const Slot& s, const Params& p, const WinState& st, int32_t r) {
    GraphTwin* g = graph_twin_now;
    if (!g || p.serial_topsort) return;
    g->reach[GR_topsort_twins] += 1;
    const Slot t = g->shadow(s);
    WinState ts = st;
    topsort_serial(t, p, ts);
    for (int32_t k = 0; k < st.n_nodes; ++k)
        if (t.node_at[k] != s.node_at[k]) {
            g->report(0, r, k, t.node_at[k], s.node_at[k]);
            return;
        }
}

/* after every warp-sweep subgraph: mark_subgraph_serial must give the same members in the same order */
static void graph_twin_subgraph(const Slot& s, const Params& p, const WinState& st, int32_t r, int32_t begin,
                                int32_t end, int32_t n, int32_t cap) {
    GraphTwin* g = graph_twin_now;
    if (!g || p.serial_topsort || st.n_nodes > cap) return; /* the engine ran the serial order itself */
    g->reach[GR_sub_twins] += 1;
    const Slot t = g->shadow(s);
    WinState ts = st;
    const int32_t tn = mark_subgraph_serial(t, p, ts, begin, end);
    if (tn != n) {
        g->report(1, r, -1, tn, n);
        return;
    }
    for (int32_t k = 0; k < n; ++k)
        if (t.sub_at[k] != s.sub_at[k]) {
            g->report(1, r, k, t.sub_at[k], s.sub_at[k]);
            return;
        }
}

/* after consensus_scores_full: spoa's literal loop (graph.cpp:494-518, scores and predecessors -1 everywhere to start,
 * "scores[max_score_id] < scores[id]") must give the same scores, predecessors and max_id */
static void graph_twin_consensus(const Slot& s, int32_t N, int32_t max_id) {
    GraphTwin* g = graph_twin_now;
    if (!g) return;
    g->reach[GR_cons_twins] += 1;
    const Slot t = g->shadow(s);
    std::fill(g->c_score.begin(), g->c_score.begin() + N, -1);
    std::fill(g->c_pred.begin(), g->c_pred.begin() + N, -1);
    for (int32_t k = 0; k < N; ++k) t.node_at[k] = s.node_at[k];
    int32_t tmax = 0, unused = 0;
    consensus_scores_from(t, N, 0, false, tmax, unused, true);
    for (int32_t v = 0; v < N; ++v) {
        if (t.c_score[v] != s.c_score[v]) {
            g->report(2, -1, v, t.c_score[v], s.c_score[v]);
            return;
        }
        if (t.c_pred[v] != s.c_pred[v]) {
            g->report(2, -1, v, t.c_pred[v], s.c_pred[v]);
            return;
        }
    }
    if (tmax != max_id) g->report(2, -1, -1, tmax, max_id);
}

/* the subgraph sweep: a chunk [hi - 31, hi] begins (does its lower edge cut a clique?), one iteration of a chunk ran */
static void graph_twin_sweep_chunk(const Slot& s, int32_t hi) {
    GraphTwin* g = graph_twin_now;
    if (!g) return;
    g->sweep_steps = 0;
    const int32_t lo = hi - 31;
    if (lo < 1) return;
    const int32_t a = s.node_at[lo], b = s.node_at[lo - 1];
    for (int32_t q = 0; q < s.aln_cnt[a]; ++q)
        if (s.aln[a * KA + q] == b) {
            g->reach[GR_straddle] += 1;
            if (s.aln_cnt[a] == KA) g->reach[GR_straddle8] += 1;
        }
}
static void graph_twin_sweep_step() {
    GraphTwin* g = graph_twin_now;
    if (!g) return;
    ++g->sweep_steps;
    if (g->sweep_steps == 2) g->reach[GR_sweep_iter2] += 1;
    if (g->sweep_steps == 3) g->reach[GR_sweep_iter3] += 1;
}

namespace {

/* Scalar twin of the traceback (traceback() and traceback_i32()): spoa's priority -- diagonal over the in-edges in
 * order, then vertical over the in-edges in order, then horizontal -- walked one cell at a time on the same slot
 * matrix, re-reading every cell; no tile, no lanes, no output buffer.  Entries leftmost first; false if the band holds
 * no consistent path. */
struct ScalarTraceback {
    static bool walk(const Slot& s, const Params& p, const ReadGeom& g, const uint8_t* read, int32_t end_row,
                     const uint16_t* row_node, bool cells32, std::vector<int16_t>& node, std::vector<int16_t>& pos) {
        const int32_t* S32 = reinterpret_cast<const int32_t*>(s.S);
        const auto cell = [&](int32_t row, int32_t bs, int32_t col) -> int32_t {
            return cells32 ? cell32(S32, p.stride, g.bw, row, bs, col) : score_at_bs(s, p, g, row, bs, col);
        };
        const int32_t mg = p.match - p.gap, xg = p.mismatch - p.gap;
        node.clear();
        pos.clear();
        int32_t i = end_row, j = g.len;
        while (!(i == 0 && j == 0)) {
            int32_t ni = i, nj = j;
            if (i == 0) {
                nj = j - 1;
            } else {
                const uint32_t rec = s.row_rec[i];
                const int32_t np = rec_npred(rec), bs = rec_bs(rec), po = (int32_t)s.row_poff[i];
                const int32_t cur = cell(i, bs, j);
                const int32_t prof = (j > 0 && rec_code(rec) == (int32_t)read[j - 1]) ? mg : xg;
                bool found = false;
                for (int32_t k = 0; k < np && !found && j > 0; ++k) {
                    const uint32_t pe = s.row_pred[po + k];
                    if (cell((int32_t)(pe & 0xFFFFu), (int32_t)(pe >> 16), j - 1) + prof == cur) {
                        ni = (int32_t)(pe & 0xFFFFu);
                        nj = j - 1;
                        found = true;
                    }
                }
                for (int32_t k = 0; k < np && !found; ++k) {
                    const uint32_t pe = s.row_pred[po + k];
                    if (cell((int32_t)(pe & 0xFFFFu), (int32_t)(pe >> 16), j) + p.gap == cur) {
                        ni = (int32_t)(pe & 0xFFFFu);
                        found = true;
                    }
                }
                if (!found) {
                    if (j > 0 && cell(i, bs, j - 1) == cur) nj = j - 1;
                    else return false;
                }
            }
            node.push_back((int16_t)(i == ni ? -1 : (int32_t)row_node[i - 1]));
            pos.push_back((int16_t)(j == nj ? -1 : j - 1));
            i = ni;
            j = nj;
        }
        std::reverse(node.begin(), node.end());
        std::reverse(pos.begin(), pos.end());
        return true;
    }
};

/* the first traceback of a window that differs from its twin: read (processing position), try, entry index, the twin's
 * entry (node, pos), the engine's entry, the twin's and the engine's entry counts (-1: lost; entry -2: none) */
constexpr int TB_MISMATCH_INTS = 9;

/* Reach report: per window, which paths of the CUDA fill its reads would take (tests/fill_cases.py names the fields). */
enum Reach {
    R_VARIANT = 0,                  /* [FILL_VARIANTS] reads per fill_variant() (int16 cells) */
    R_CELLS32 = R_VARIANT + FILL_VARIANTS, /* fills on 32-bit cells (fill_rows_i32) */
    R_GENERAL_ROWS,                 /* rows flagged for the general path (pred_needs_general_path) */
    R_FAR_PREDS,                    /* predecessors older than the ring */
    R_JUMP_PREDS,                   /* predecessors whose band starts more than RING_PAD_BACK columns before the row's */
    R_MAX_NPRED,                    /* largest predecessor count of a row */
    R_ROWS_OVER32,                  /* rows with more than 32 predecessors */
    R_DYN_ROWS,                     /* rows whose letter needs the on-demand profile row */
    R_DYN_BUILDS,                   /* times that row is (re)built: the letter changed since the last such row */
    R_RETRIES,                      /* adaptive retries (a read filled again) */
    R_RETRIES_FULL,                 /* ... that reached the full matrix */
    R_MAX_LEN,                      /* longest read filled */
    R_FIELDS
};

/* Scalar twin of poa_fill.cuh: same cell definition, same NEG clamp, same band. */
struct ScalarFill {
    int64_t cells = 0;
    int32_t* reach = nullptr; /* this window's report, or nullptr */
    const uint8_t* last_read = nullptr;
    int32_t* tb_reach = nullptr;    /* this window's traceback report (TB_FIELDS), or nullptr */
    int32_t* tb_mismatch = nullptr; /* this window's first twin mismatch (TB_MISMATCH_INTS), or nullptr */
    const uint8_t* tb_last_read = nullptr;
    int32_t tb_try = 0;
    std::vector<int16_t> twin_node, twin_pos;

    /* POA_TB_TWIN: after every traceback of process_window(), walk the twin on the same matrix and compare */
    void traceback_twin(const Slot& s, const Params& p, const WinState& st, const ReadGeom& g, int32_t r,
                        const uint8_t* read, int32_t end_row, int32_t tb, const uint16_t* row_node, bool cells32,
                        bool partial) {
        tb_try = read == tb_last_read ? tb_try + 1 : 0;
        tb_last_read = read;
        const int32_t cap = p.max_nodes + p.max_len + 2;
        const bool lost = st.status == ST_TRACEBACK_LOST;
        const int32_t n = lost ? -1 : cap - tb;
        const bool twin_ok = ScalarTraceback::walk(s, p, g, read, end_row, row_node, cells32, twin_node, twin_pos);
        const int32_t tn = twin_ok ? (int32_t)twin_node.size() : -1;
        int32_t k = 0; /* first differing entry */
        while (k < n && k < tn && twin_node[(size_t)k] == s.tb_node[tb + k] && twin_pos[(size_t)k] == s.tb_pos[tb + k]) ++k;
        const bool same = tn == n && k == std::max(n, 0);
        if (tb_reach) {
            int32_t* t = tb_reach;
            t[TB_tracebacks] += 1;
            if (!same) t[TB_twin_mismatches] += 1;
            if (partial) t[TB_partial_reads] += 1;
            if (n >= 0) {
                t[TB_count_mod0] += n % 32 == 0;
                t[TB_count_mod1] += n % 32 == 1;
                t[TB_count_mod31] += n % 32 == 31;
                int32_t run = 0, longest = 0;
                for (int32_t e = tb; e < cap; ++e) {
                    run = (s.tb_pos[e] == -1 && s.tb_node[e] != -1) ? run + 1 : 0;
                    longest = std::max(longest, run);
                }
                t[TB_vrun32] += longest >= 32;
            }
        }
        if (!same && tb_mismatch && tb_mismatch[0] < 0) {
            const int32_t m[TB_MISMATCH_INTS] = {r, tb_try, k, k < tn ? twin_node[(size_t)k] : -2, k < tn ? twin_pos[(size_t)k] : -2,
                                                 k < n ? s.tb_node[tb + k] : -2, k < n ? s.tb_pos[tb + k] : -2, tn, n};
            std::copy(m, m + TB_MISMATCH_INTS, tb_mismatch);
        }
    }

    int32_t operator()(const Slot& s, const Params& p, WinState& st, const ReadGeom& g,
                       const uint8_t* read) {
        const int32_t N = g.n_rows;
        (void)st;
        const int32_t mg = p.match - p.gap, xg = p.mismatch - p.gap;
        if (reach) {
            reach[R_VARIANT + fill_variant(g)] += 1;
            if (read == last_read) {
                reach[R_RETRIES] += 1;
                if (!g.banded) reach[R_RETRIES_FULL] += 1;
            }
            if (g.len > reach[R_MAX_LEN]) reach[R_MAX_LEN] = g.len;
            int32_t dyn_code = -1;
            for (int32_t i = 1; i <= N; ++i) {
                const uint32_t rec = s.row_rec[i];
                const int32_t np = rec_npred(rec), po = (int32_t)s.row_poff[i];
                if (rec_far(rec)) reach[R_GENERAL_ROWS] += 1;
                if (np > reach[R_MAX_NPRED]) reach[R_MAX_NPRED] = np;
                if (np > 32) reach[R_ROWS_OVER32] += 1;
                if (rec_prow(rec) == 4) {
                    reach[R_DYN_ROWS] += 1;
                    if (rec_code(rec) != dyn_code) reach[R_DYN_BUILDS] += 1;
                    dyn_code = rec_code(rec);
                }
                for (int32_t k = 0; k < np; ++k) {
                    const uint32_t pe = s.row_pred[po + k];
                    const int32_t pr = (int32_t)(pe & 0xFFFFu), pbs = (int32_t)(pe >> 16);
                    if (i - pr >= p.ring_rows) reach[R_FAR_PREDS] += 1;
                    if (rec_bs(rec) - pbs > RING_PAD_BACK) reach[R_JUMP_PREDS] += 1;
                }
            }
        }
        last_read = read;
        for (int32_t c = 0; c < g.bw; ++c) s.S[c] = 0; /* row 0: H = j*gap  =>  S = 0 */
        int32_t best = NEG, end_row = 0;
        for (int32_t i = 1; i <= N; ++i) {
            const uint32_t rec = s.row_rec[i];
            const uint8_t code = (uint8_t)rec_code(rec);
            const int32_t np = rec_npred(rec);
            const int32_t po = (int32_t)s.row_poff[i];
            const int32_t bs = rec_bs(rec);
            int16_t* row = s.S + (size_t)i * p.stride;
            int32_t left = NEG;
            for (int32_t o = 0; o < g.bw; ++o) {
                const int32_t c = bs + o;
                const int32_t prof = (c >= 1 && c <= g.len && read[c - 1] == code) ? mg : xg;
                int32_t t = NEG;
                for (int32_t k = 0; k < np; ++k) {
                    const int32_t pr = (int32_t)(s.row_pred[po + k] & 0xFFFFu);
                    const int32_t d = score_at(s, p, g, pr, c - 1) + prof;
                    const int32_t v = score_at(s, p, g, pr, c) + p.gap;
                    if (d > t) t = d;
                    if (v > t) t = v;
                }
                if (left > t) t = left;
                if (t < NEG) t = NEG;
                row[o] = (int16_t)t;
                left = t;
            }
            cells += g.bw;
            if (rec_sink(rec)) {
                const int32_t v = score_at(s, p, g, i, g.len);
                if (v > best) {
                    best = v;
                    end_row = i;
                }
            }
        }
        return end_row;
    }
};

} // namespace

extern "C" {

/* Flat batch in ADD order + order[] (processing permutation), like poa_oracle_polish_windows.
 * Outputs the UNTRIMMED consensus, coverage and the per-window status.  rank_out (nullable):
 * n_windows x max_nodes final rank_to_node order, n_nodes_out (nullable) node counts.  emu_polish_windows_tb and
 * emu_polish_windows (below) are the same without the graph's, and without the traceback's, outputs. */
void emu_polish_windows_graph(int64_t n_windows, const int64_t* win_seq_off, const int64_t* seq_off,
                        const uint8_t* bases, const int8_t* weights, const uint8_t* has_weights,
                        const int32_t* begins, const int32_t* ends, const int32_t* order, int32_t m, int32_t x, int32_t gap,
                        int32_t max_nodes, int32_t max_edges, int32_t max_len, int32_t band_width,
                        int32_t serial_topsort, int32_t n_threads, uint8_t* cons_out,
                        uint16_t* cov_out, int32_t stride_out, int32_t* cons_len, int32_t* status,
                        int32_t* rank_out, int32_t* n_nodes_out, int64_t* cells_out, int32_t* trim_out,
                        /* MSA (all nullable): compact arena of msa_cap bytes + per-window offset / columns / status */
                        uint8_t* msa_out, int64_t msa_cap, int64_t* msa_off, int32_t* msa_cols, int32_t* msa_status,
                        /* ring_rows: the score-row ring of the GPU launch to compare with (the row program's far-predecessor
                         * flags depend on it).  Per sequence (window by window, processing order; nullable): the sum of
                         * fill_digest() over its fills and their number.  Per window (nullable): R_FIELDS reach counters. */
                        int32_t ring_rows, unsigned long long* digest_out, int32_t* fill_count_out, int32_t* reach_out,
                        /* Per sequence (nullable): aln_digest() of the alignment added to the graph and its entry
                         * count.  Per window (nullable): TB_FIELDS traceback reach counters, and the first traceback
                         * that differs from the scalar twin (TB_MISMATCH_INTS, read -1: none). */
                        unsigned long long* aln_digest_out, int32_t* aln_count_out, int32_t* tb_reach_out,
                        int32_t* tb_mismatch_out,
                        /* Per sequence (nullable): graph_digest() after it was added and sorted, the graph's node and
                         * edge counts, and for partial-span reads sub_digest() and the member count.  Per window
                         * (nullable): cons_digest() after the full scoring pass and after branch completion, the rounds
                         * of branch completion, GR_FIELDS graph reach counters and the first twin check that found a
                         * difference (GR_MISMATCH_INTS, kind -1: none). */
                        unsigned long long* graph_digest_out, int32_t* graph_nodes_out, int32_t* graph_edges_out,
                        unsigned long long* sub_digest_out, int32_t* sub_count_out, unsigned long long* cons_digest_out,
                        int32_t* cons_rounds_out, int32_t* graph_reach_out, int32_t* graph_mismatch_out) {
    Params p;
    p.max_nodes = max_nodes;
    p.max_edges = poa_edge_capacity(max_nodes); /* the engine derives the edge pool from the node capacity */
    (void)max_edges;
    p.max_len = max_len;
    const int32_t colsP = (max_len + 1 + 7) & ~7;
    p.adaptive = band_width < 0 ? 1 : 0; /* band_width < 0: adaptive band starting at -band_width */
    if (band_width < 0) band_width = -band_width;
    p.band_width = band_width;
    p.stride = (!p.adaptive && band_width > 0 && band_width < colsP) ? band_width : colsP;
    p.max_cons = stride_out;
    p.match = m;
    p.mismatch = x;
    p.gap = gap;
    p.force_cells32 = (serial_topsort & 2) ? 1 : 0; /* bit 1 of the flag: every read through the 32-bit path */
    p.wide_cells = (p.force_cells32 || !score_range_ok(p, p.max_nodes, p.max_len)) ? 1 : 0;
    p.serial_topsort = serial_topsort & 1;
    p.skip_consensus = 0;
    p.ring_rows = ring_rows;
    p.ring_stride = p.stride;
    Slot probe;
    size_t slot_bytes = 0;
    slot_bind(probe, nullptr, p, &slot_bytes);

    std::atomic<int64_t> cursor{0};
    std::atomic<int64_t> total_cells{0};
    unsigned long long msa_cursor = 0;
    if (msa_out) n_threads = 1; /* the host flavour of the bump allocator is not atomic */
    auto worker = [&]() {
        std::vector<uint8_t> slab(slot_bytes + 512);
        Slot s;
        slot_bind(s, reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(slab.data()) + 255) & ~uintptr_t(255)), p, nullptr);
        std::vector<uint8_t> wbases;
        std::vector<int8_t> wweights;
        std::vector<int64_t> woff, wwoff;
        std::vector<int32_t> wlen;
        std::vector<int32_t> wbeg, wend;
        ScalarFill fill;
        std::vector<uint8_t> tb_mem(TB_SCRATCH_BYTES + 64);
        TbScratch tbs;
        tb_bind(tbs, reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tb_mem.data()) + 15) & ~uintptr_t(15)));
        GraphTwin twin;
        twin.size(p);
        std::vector<int32_t> gr_scratch(GR_FIELDS);
        for (;;) {
            const int64_t w = cursor.fetch_add(1);
            if (w >= n_windows) break;
            const int64_t s0 = win_seq_off[w];
            const int32_t n = (int32_t)(win_seq_off[w + 1] - s0);
            wbases.clear();
            wweights.clear();
            woff.clear();
            wlen.clear();
            wwoff.clear();
            wbeg.clear();
            wend.clear();
            const uint32_t L0 = (uint32_t)(seq_off[s0 + order[s0] + 1] - seq_off[s0 + order[s0]]);
            const uint32_t offset = (uint32_t)(0.01 * L0); /* window.cpp:87 */
            bool too_long = false;
            for (int32_t k = 0; k < n; ++k) {
                const int64_t sq = s0 + order[s0 + k];
                const int64_t a = seq_off[sq], b = seq_off[sq + 1];
                if (b - a > max_len) too_long = true;
                woff.push_back((int64_t)wbases.size());
                wlen.push_back((int32_t)(b - a));
                wbases.insert(wbases.end(), bases + a, bases + b);
                if (has_weights[sq]) { /* explicit weights live in the compact arena ... */
                    wwoff.push_back((int64_t)wweights.size());
                    wweights.insert(wweights.end(), weights + a, weights + b);
                } else {
                    wwoff.push_back(-1 - 1); /* ... a sequence without quality weighs 1 per base and ships none */
                }
                /* window.cpp:92-93: full-span test (the product's host library applies the same rule) */
                const bool full = k == 0 || !begins ||
                                  ((uint32_t)begins[sq] < offset && (uint32_t)ends[sq] > L0 - offset);
                wbeg.push_back(full ? -1 : begins[sq]);
                wend.push_back(full ? -1 : ends[sq]);
            }
            if (too_long) {
                cons_len[w] = 0;
                status[w] = ST_EXCEEDED_MAX_SEQ_SIZE;
                if (msa_out) {
                    msa_off[w] = 0;
                    msa_cols[w] = 0;
                    msa_status[w] = ST_EXCEEDED_MAX_SEQ_SIZE;
                }
                continue;
            }
            WindowView wv;
            wv.n_seqs = n;
            wv.bases = wbases.data();
            wv.weights = wweights.data();
            wv.seq_off = woff.data();
            wv.seq_len = wlen.data();
            wv.w_off = wwoff.data();
            wv.seq_begin = wbeg.data();
            wv.seq_end = wend.data();
            std::vector<uint16_t> wpath(msa_out ? wbases.size() + 1 : 0);
            wv.path = msa_out ? wpath.data() : nullptr;
            std::vector<unsigned long long> wdigest((size_t)n, 0);
            std::vector<int32_t> wcount((size_t)n, 0);
            wv.fill_digest = wdigest.data();
            wv.fill_count = wcount.data();
            int32_t* reach = reach_out ? reach_out + w * R_FIELDS : nullptr;
            if (reach)
                for (int32_t k = 0; k < R_FIELDS; ++k) reach[k] = 0;
            fill.reach = reach;
            fill.last_read = nullptr;
            std::vector<unsigned long long> waln((size_t)n, 0);
            std::vector<int32_t> walncnt((size_t)n, 0);
            wv.aln_digest = waln.data();
            wv.aln_count = walncnt.data();
            std::vector<int32_t> tb_scratch(tb_reach_out ? 0 : TB_FIELDS);
            fill.tb_reach = tb_reach_out ? tb_reach_out + w * TB_FIELDS : tb_scratch.data();
            for (int32_t k = 0; k < TB_FIELDS; ++k) fill.tb_reach[k] = 0;
            tb_reach_now = fill.tb_reach;
            fill.tb_mismatch = tb_mismatch_out ? tb_mismatch_out + w * TB_MISMATCH_INTS : nullptr;
            if (fill.tb_mismatch)
                for (int32_t k = 0; k < TB_MISMATCH_INTS; ++k) fill.tb_mismatch[k] = -1;
            fill.tb_last_read = nullptr;
            std::vector<unsigned long long> wgraph((size_t)n, 0), wsub((size_t)n, 0);
            std::vector<int32_t> wnodes((size_t)n, 0), wedges((size_t)n, 0), wsubcnt((size_t)n, 0);
            wv.graph_digest = wgraph.data();
            wv.graph_nodes = wnodes.data();
            wv.graph_edges = wedges.data();
            wv.sub_digest = wsub.data();
            wv.sub_count = wsubcnt.data();
            unsigned long long wcons[2] = {0, 0};
            int32_t wrounds = 0;
            twin.reach = graph_reach_out ? graph_reach_out + w * GR_FIELDS : gr_scratch.data();
            for (int32_t k = 0; k < GR_FIELDS; ++k) twin.reach[k] = 0;
            twin.mismatch = graph_mismatch_out ? graph_mismatch_out + w * GR_MISMATCH_INTS : nullptr;
            if (twin.mismatch)
                for (int32_t k = 0; k < GR_MISMATCH_INTS; ++k) twin.mismatch[k] = -1;
            graph_reach_now = twin.reach;
            graph_twin_now = &twin;
            /* process_window writes its node count nowhere; recover it from the slot afterwards */
            uint32_t cursor = 0;
            int32_t off = 0, trim = 0;
            WindowOut out;
            out.cons = cons_out + w * (int64_t)stride_out; /* this window's row is its own arena */
            out.cov = cov_out + w * (int64_t)stride_out;
            out.cursor = &cursor;
            out.len = &cons_len[w];
            out.status = &status[w];
            out.off = &off;
            out.trim = &trim;
            out.trim_nseq = n;
            out.cons_digest = wcons;
            out.cons_rounds = &wrounds;
            long long moff = 0;
            int32_t mcols = 0, mst = 0;
            const int32_t n_final = process_window(s, p, wv, fill, tbs, out);
            tb_reach_now = nullptr;
            graph_reach_now = nullptr;
            graph_twin_now = nullptr;
            for (int32_t k = 0; k < n; ++k) {
                if (graph_digest_out) graph_digest_out[s0 + k] = wgraph[(size_t)k];
                if (graph_nodes_out) graph_nodes_out[s0 + k] = wnodes[(size_t)k];
                if (graph_edges_out) graph_edges_out[s0 + k] = wedges[(size_t)k];
                if (sub_digest_out) sub_digest_out[s0 + k] = wsub[(size_t)k];
                if (sub_count_out) sub_count_out[s0 + k] = wsubcnt[(size_t)k];
            }
            if (cons_digest_out) {
                cons_digest_out[2 * w] = wcons[0];
                cons_digest_out[2 * w + 1] = wcons[1];
            }
            if (cons_rounds_out) cons_rounds_out[w] = wrounds;
            if (aln_digest_out)
                for (int32_t k = 0; k < n; ++k) aln_digest_out[s0 + k] = waln[(size_t)k];
            if (aln_count_out)
                for (int32_t k = 0; k < n; ++k) aln_count_out[s0 + k] = walncnt[(size_t)k];
            if (digest_out)
                for (int32_t k = 0; k < n; ++k) digest_out[s0 + k] = wdigest[(size_t)k];
            if (fill_count_out)
                for (int32_t k = 0; k < n; ++k) fill_count_out[s0 + k] = wcount[(size_t)k];
            if (reach) { /* fills that did not go through the int16 twin ran on 32-bit cells */
                int32_t fills = 0, fills16 = 0;
                for (int32_t k = 0; k < n; ++k) fills += wcount[(size_t)k];
                for (int32_t v = 0; v < FILL_VARIANTS; ++v) fills16 += reach[R_VARIANT + v];
                reach[R_CELLS32] = fills - fills16;
            }
            if (msa_out) {
                MsaOut mo;
                mo.arena = msa_out;
                mo.cursor = &msa_cursor;
                mo.cap = (unsigned long long)msa_cap;
                mo.off = &moff;
                mo.cols = &mcols;
                mo.status = &mst;
                window_msa(s, p, n_final, status[w], wv, mo);
            }
            if (trim_out) trim_out[w] = trim;
            if (msa_out) {
                msa_off[w] = moff;
                msa_cols[w] = mcols;
                msa_status[w] = mst;
            }
            if (rank_out || n_nodes_out) {
                /* n_nodes = 1 + max rank_of over nodes is not stored; count nodes via root != unset:
                 * simplest is to re-derive from node_at being a permutation of [0, N). */
                int32_t N = 0;
                /* nodes are dense ids [0,N): N is the first id whose code was never written; the
                 * slab is reused, so instead track through cov/aln arrays is unreliable -> use the
                 * exported helper below. */
                (void)N;
            }
        }
        total_cells += fill.cells;
    };
    if (n_threads <= 1) {
        worker();
    } else {
        std::vector<std::thread> th;
        for (int32_t t = 0; t < n_threads; ++t) th.emplace_back(worker);
        for (auto& t : th) t.join();
    }
    if (cells_out) *cells_out = total_cells.load();
    (void)rank_out;
    (void)n_nodes_out;
}

void emu_polish_windows_tb(int64_t n_windows, const int64_t* win_seq_off, const int64_t* seq_off,
                           const uint8_t* bases, const int8_t* weights, const uint8_t* has_weights,
                           const int32_t* begins, const int32_t* ends, const int32_t* order, int32_t m, int32_t x,
                           int32_t gap, int32_t max_nodes, int32_t max_edges, int32_t max_len, int32_t band_width,
                           int32_t serial_topsort, int32_t n_threads, uint8_t* cons_out, uint16_t* cov_out,
                           int32_t stride_out, int32_t* cons_len, int32_t* status, int32_t* rank_out,
                           int32_t* n_nodes_out, int64_t* cells_out, int32_t* trim_out, uint8_t* msa_out,
                           int64_t msa_cap, int64_t* msa_off, int32_t* msa_cols, int32_t* msa_status, int32_t ring_rows,
                           unsigned long long* digest_out, int32_t* fill_count_out, int32_t* reach_out,
                           unsigned long long* aln_digest_out, int32_t* aln_count_out, int32_t* tb_reach_out,
                           int32_t* tb_mismatch_out) {
    emu_polish_windows_graph(n_windows, win_seq_off, seq_off, bases, weights, has_weights, begins, ends, order, m, x,
                             gap, max_nodes, max_edges, max_len, band_width, serial_topsort, n_threads, cons_out,
                             cov_out, stride_out, cons_len, status, rank_out, n_nodes_out, cells_out, trim_out, msa_out,
                             msa_cap, msa_off, msa_cols, msa_status, ring_rows, digest_out, fill_count_out, reach_out,
                             aln_digest_out, aln_count_out, tb_reach_out, tb_mismatch_out, nullptr, nullptr, nullptr,
                             nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
}

void emu_polish_windows(int64_t n_windows, const int64_t* win_seq_off, const int64_t* seq_off,
                        const uint8_t* bases, const int8_t* weights, const uint8_t* has_weights,
                        const int32_t* begins, const int32_t* ends, const int32_t* order, int32_t m, int32_t x, int32_t gap,
                        int32_t max_nodes, int32_t max_edges, int32_t max_len, int32_t band_width,
                        int32_t serial_topsort, int32_t n_threads, uint8_t* cons_out,
                        uint16_t* cov_out, int32_t stride_out, int32_t* cons_len, int32_t* status,
                        int32_t* rank_out, int32_t* n_nodes_out, int64_t* cells_out, int32_t* trim_out,
                        uint8_t* msa_out, int64_t msa_cap, int64_t* msa_off, int32_t* msa_cols, int32_t* msa_status,
                        int32_t ring_rows, unsigned long long* digest_out, int32_t* fill_count_out, int32_t* reach_out) {
    emu_polish_windows_tb(n_windows, win_seq_off, seq_off, bases, weights, has_weights, begins, ends, order, m, x, gap,
                          max_nodes, max_edges, max_len, band_width, serial_topsort, n_threads, cons_out, cov_out,
                          stride_out, cons_len, status, rank_out, n_nodes_out, cells_out, trim_out, msa_out, msa_cap,
                          msa_off, msa_cols, msa_status, ring_rows, digest_out, fill_count_out, reach_out, nullptr,
                          nullptr, nullptr, nullptr);
}

} // extern "C"
