/*
 * poa_core.cuh -- one-window-per-warp partial order alignment consensus (graph phases).
 *
 * Replaces, for racon's consensus path, what the reference runs in
 *   vendor/GenomeWorks/cudapoa/src/cudapoa_kernels.cuh:74-434   (generatePOAKernel)
 *   vendor/GenomeWorks/cudapoa/src/cudapoa_add_alignment.cuh:66-287
 *   vendor/GenomeWorks/cudapoa/src/cudapoa_topsort.cuh:101-195
 *   vendor/GenomeWorks/cudapoa/src/cudapoa_generate_consensus.cuh:35-354
 * but with the SEMANTICS of racon's CPU path (spoa), which is the parity target:
 *   vendor/spoa/src/sisd_alignment_engine.cpp:260-435, vendor/spoa/src/graph.cpp:94-589.
 *
 * Design (not a port): everything a window needs lives in a compact per-warp workspace
 * ("slot") -- nodes are SoA arrays of u8/u16, in-edges are a pooled linked list kept in insertion
 * order (spoa's in_edges_ order decides every tie-break), aligned-node cliques are <= KA inline ids.
 * cudapoa's fixed 50-edge / 50-aligned strides (cudapoa_structs.cuh:24-27) are gone, so a slot is
 * ~100 KB + the score band instead of 2-2.6 MB + 2-6 MB, and slots are per RESIDENT WARP, not per
 * window in the batch.
 *
 * The serial lane-0 phases of the reference are re-formulated as warp-parallel phases:
 *   - add_alignment: every read position is resolved independently (a path visits each aligned
 *     clique once), new node / edge ids come from warp prefix sums, each node receives at most one
 *     new in-edge per read so list order is preserved;
 *   - topological sort: spoa's DFS order is decomposed by ROOT (root[v] = smallest id whose
 *     ancestor-closure contains v).  root[] is fixed when a node is created, DFS_i for different
 *     roots are independent, so 32 roots are sorted concurrently and concatenated by a prefix sum.
 *     The plain serial DFS is kept (topsort_serial) as the in-kernel cross-check for tests.
 *   - traceback: the path is walked through a shared-memory tile of the score matrix loaded by one round
 *     of asynchronous copies; rows with one in-edge take a warp-uniform scalar step, rows with several are
 *     rated by different lanes and decided by one warp-min;
 *   - consensus: heaviest-bundle scores 32 ranks at a time (parallel gather, in-register resolve).
 * Every phase is bound by the latency of dependent loads to HBM (a window's graph does not stay in L2 with
 * 3552 windows in flight), so the loops are shaped to keep many independent loads in flight and to place
 * loads before stores (a load behind a store to the workspace cannot be hoisted by the compiler).
 *
 * Score cells are int16 in the "skewed" domain S[i][j] = H[i][j] - j*gap so that the horizontal
 * recurrence H[i][j-1]+gap becomes a pure prefix max:
 *   S[i][j] = max( max_p S[p][j-1] + (s(i,j) - gap), max_p S[p][j] + gap, S[i][j-1] ).
 * The DP fill itself is in poa_fill.cuh (CUDA); tests/emu has its scalar twin for the CPU tests.
 */
#pragma once
#include "poa_simt.cuh"

/* Test build (-DPOA_FILL_DIGEST=1, racon_gpu_b200/variants/libb200poa_digest.so and tests/emu): every DP fill is hashed
 * (fill_digest) so that the CUDA fill can be compared cell for cell with its scalar twin.  The product never has it. */
#ifndef POA_FILL_DIGEST
#define POA_FILL_DIGEST 0
#endif
/* Test build (-DPOA_ALN_DIGEST=1, the same library and tests/emu): the alignment every read adds to the graph is hashed
 * (aln_digest) so that the traceback can be compared read for read with its scalar twin and with spoa.  A define of its
 * own: a caller that fills only the fill-digest fields of WindowView stays correct. */
#ifndef POA_ALN_DIGEST
#define POA_ALN_DIGEST 0
#endif
/* Test build (-DPOA_GRAPH_DIGEST=1, the same library and tests/emu): the graph after every read (graph_digest), the
 * subgraph a partial-span read is aligned to (sub_digest) and the consensus scores before and after branch completion
 * (cons_digest) are hashed, so that add_alignment, the sorts, the subgraph and the heaviest bundle can be compared read
 * for read with the emulation and with spoa.  A define of its own, like POA_ALN_DIGEST. */
#ifndef POA_GRAPH_DIGEST
#define POA_GRAPH_DIGEST 0
#endif

/* Hooks of the emulation (tests/emu): POA_TB_REACH(field) counts a path of the traceback, POA_TB_REACH_IF(cond, field)
 * counts it when cond holds, and POA_TB_TWIN(fill, ...) checks every traceback against a scalar twin walk.  Elsewhere
 * they expand to nothing (cond is not evaluated): no kernel, the digest build included, contains them. */
#ifndef POA_TB_REACH
#define POA_TB_REACH(field) ((void)0)
#endif
#ifndef POA_TB_REACH_IF
#define POA_TB_REACH_IF(cond, field) ((void)0)
#endif
#ifndef POA_TB_TWIN
#define POA_TB_TWIN(fill, ...) ((void)0)
#endif
/* The same for the graph phases: POA_GRAPH_REACH(field) / POA_GRAPH_REACH_IF(cond, field) count a path of
 * add_alignment, the sorts, the subgraph or the consensus, and POA_GRAPH_TWIN(what, ...) checks the sort, the subgraph
 * and the consensus scores against their serial twins.  Elsewhere nothing. */
#ifndef POA_GRAPH_REACH
#define POA_GRAPH_REACH(field) ((void)0)
#endif
#ifndef POA_GRAPH_REACH_IF
#define POA_GRAPH_REACH_IF(cond, field) ((void)0)
#endif
#ifndef POA_GRAPH_REACH_AT /* the k-th of the counters that start at field */
#define POA_GRAPH_REACH_AT(field, k) ((void)0)
#endif
#ifndef POA_GRAPH_TWIN
#define POA_GRAPH_TWIN(what, ...) ((void)0)
#endif

namespace b200poa {

POA_FN void poa_atomic_add(uint32_t* p, uint32_t v) {
#if POA_DEVICE
    atomicAdd(p, v);
#else
    *p += v;
#endif
}

#ifndef POA_TS_U
#define POA_TS_U 4
#endif
constexpr int TS_U = POA_TS_U; /* nodes per lane per step in the node-parallel passes of the sort */
constexpr int KA = 7;                  /* max aligned nodes per node (clique size - 1) */
constexpr uint16_t NONE16 = 0xFFFFu;
constexpr int NEG = -30000;            /* "minus infinity" for int16 cells; see DESIGN.md */
constexpr int LANE_CELLS = 8;          /* int16 cells per lane per chunk (one 128-bit vector) */
constexpr int CHUNK = 32 * LANE_CELLS; /* 256 columns per warp pass */

/* status codes mirror claraparabricks::genomeworks::cudapoa::StatusType (cudapoa.hpp:32-45) */
enum Status : int32_t {
    ST_SUCCESS = 0,
    ST_EXCEEDED_MAX_POAS = 1,
    ST_EXCEEDED_MAX_SEQ_SIZE = 2,
    ST_EXCEEDED_MAX_SEQS_PER_POA = 3,
    ST_NODE_COUNT_EXCEEDED = 4,
    ST_EDGE_COUNT_EXCEEDED = 5,
    ST_EXCEEDED_ADAPTIVE_BAND = 6,
    ST_SEQ_LEN_EXCEEDED_MAX_NODES = 7,
    ST_LOOP_COUNT_EXCEEDED = 8,
    ST_OUTPUT_UNAVAILABLE = 9,
    ST_GENERIC_ERROR = 10,
    /* extensions (never returned by cudapoa) */
    ST_ALIGNED_COUNT_EXCEEDED = 11,  /* clique larger than KA+1 */
    ST_SCORE_RANGE_EXCEEDED = 12,    /* int16 cells cannot hold this alignment */
    ST_TRACEBACK_LOST = 13           /* band did not contain a consistent path */
};

struct Params {
    int32_t max_nodes;   /* MN : node capacity of a slot            */
    int32_t max_edges;   /* ME : edge pool capacity == poa_edge_capacity(max_nodes): the phases derive it from max_nodes
                            instead of keeping one more warp-uniform value alive (poa_simt.cuh) */
    int32_t max_len;     /* longest sequence accepted               */
    int32_t stride;      /* int16 cells per score row (multiple of 8) */
    int32_t band_width;  /* 0 = full band, else W (multiple of 8)   */
    int32_t max_cons;    /* row stride of the consensus / coverage outputs */
    int32_t match, mismatch, gap;
    int32_t serial_topsort; /* tests: use the serial DFS instead of the per-root sort */
    int32_t ring_rows;      /* fill: rows in the shared-memory score ring (power of two) */
    int32_t ring_stride;    /* fill: int16 cells per ring row */
    int32_t wide_cells;     /* the score region of a slot is sized for int32 cells: a read whose alignment does not fit
                               int16 (score_range_ok) is filled and traced with 32-bit cells -- the switch spoa makes,
                               simd_alignment_engine.cpp:668-673; cudapoa instantiates int32 per batch, batch.cu:114-138 */
    int32_t force_cells32;  /* tests: every read takes the 32-bit path */
    int32_t skip_consensus; /* the output mask has no OutputType::consensus (MSA only, cudapoa_kernels.cuh:198-216) */
    int32_t adaptive;       /* band_width is only the FIRST try of a read: a traceback that comes close to the band's
                               edge re-aligns the read with twice the width (cudapoa's retry protocol,
                               cudapoa_kernels.cuh:257-303, cudapoa_nw_adaptive_banded.cuh:265-281, 462-480) */
};

#if POA_DEVICE
#define POA_HD __host__ __device__ __forceinline__
#else
#define POA_HD static inline
#endif
POA_HD int32_t poa_edge_capacity(int32_t max_nodes) { return 6 * max_nodes < 65000 ? 6 * max_nodes : 65000; }

/* Per resident warp workspace.  All pointers are into one device slab (see slot_bytes()). */
struct Slot {
    /* graph */
    uint8_t* code;      /* [MN] node letter                                  */
    uint16_t* nin;      /* [MN] in-degree                                    */
    uint16_t* nout;     /* [MN] out-degree (only == 0 is ever asked)         */
    uint16_t* in_head;  /* [MN] first in-edge (pool index) or NONE16         */
    uint16_t* in_tail;  /* [MN] last in-edge                                 */
    uint16_t* cov;      /* [MN] number of sequences through the node         */
    uint8_t* aln_cnt;   /* [MN] number of aligned nodes                      */
    uint16_t* aln;      /* [MN*KA] aligned node ids in insertion order       */
    uint16_t* root;     /* [MN] topological-sort root of the node            */
    uint16_t* lpos;     /* [MN] position of the node inside its root's DFS order */
    uint16_t* rank_of;  /* [MN] node -> rank                                 */
    uint16_t* node_at;  /* [MN] rank -> node                                 */
    uint16_t* sub_at;   /* [MN] partial-span layers: subgraph rank -> node     */
    uint16_t* sub_rank; /* [MN] node -> subgraph rank, NONE16 = not a member   */
    uint16_t* e_src;    /* [ME] */
    uint16_t* e_dst;    /* [ME] */
    uint16_t* e_next;   /* [ME] next in-edge of e_dst, insertion order       */
    int32_t* e_w;       /* [ME] total weight                                 */
    uint8_t* e_ord;     /* [ME] position of the edge in its target's in-edge list (fixed at creation) */
    /* per-read "row program": the graph linearised in rank order (row = rank + 1) */
    uint32_t* row_meta; /* [MN] by RANK: letter | sink << 8 | in-degree << 16 of the node at that rank.  Written where the
                           ranks are (topological sort, backbone init), read by the row program: no gather through node_at */
    uint32_t* row_rec;  /* [MN+1] packed row record, see rec_make()                */
    uint32_t* row_poff; /* [MN+2] offset of the row's predecessor list       */
    uint32_t* row_pred; /* [ME+MN] predecessor ROW index (0 = virtual row) | its band start << 16, in in-edge order */
    uint32_t* row_pfill; /* [ME+MN] the same list pre-digested for the fill, see pfill_make() */
    /* scores */
    int16_t* S;         /* [(MN+1)*stride]                                   */
    /* traceback output, written back to front */
    int16_t* tb_node;   /* [MN+ML+2] */
    int16_t* tb_pos;    /* [MN+ML+2] */
    int32_t* asg;       /* [ML+1] node assigned to each read position        */
    /* topological sort scratch */
    uint32_t* cnt;      /* [MN+1] nodes per root                             */
    uint32_t* roff;     /* [MN+1] output offset per root / stack offset      */
    uint32_t* need;     /* [MN+1] stack need per root                        */
    uint8_t* dirty;     /* [MN+1] root needs its DFS redone after this read   */
    uint8_t* marks;     /* [MN] */
    uint8_t* check;     /* [MN] */
    uint16_t* stack;    /* [ME+2*MN*? ] see slot layout                      */
    /* consensus scratch */
    int32_t* c_score;   /* [MN] */
    int32_t* c_pred;    /* [MN] */
};

struct SlotLayout {
    size_t off[40];
    size_t total;
};

/* One definition of the slab carve-up, used by host allocation, the kernel and the emulation. */
POA_FN size_t poa_align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

#if POA_DEVICE
__host__ __device__ __forceinline__
#else
static inline
#endif
void slot_bind(Slot& s, uint8_t* base, const Params& p, size_t* total_out) {
    const size_t MN = (size_t)p.max_nodes, ME = (size_t)p.max_edges, ML = (size_t)p.max_len;
    size_t o = 0;
#define POA_CARVE(field, type, count)                                  \
    do {                                                               \
        o = (o + 15) / 16 * 16;                                        \
        s.field = base ? reinterpret_cast<type*>(base + o) : nullptr;  \
        o += sizeof(type) * (size_t)(count);                           \
    } while (0)
    POA_CARVE(code, uint8_t, MN);
    POA_CARVE(nin, uint16_t, MN);
    POA_CARVE(nout, uint16_t, MN);
    POA_CARVE(in_head, uint16_t, MN);
    POA_CARVE(in_tail, uint16_t, MN);
    POA_CARVE(cov, uint16_t, MN);
    POA_CARVE(aln_cnt, uint8_t, MN);
    POA_CARVE(aln, uint16_t, MN * KA);
    POA_CARVE(root, uint16_t, MN);
    POA_CARVE(lpos, uint16_t, MN);
    POA_CARVE(rank_of, uint16_t, MN);
    POA_CARVE(node_at, uint16_t, MN);
    POA_CARVE(sub_at, uint16_t, MN);
    POA_CARVE(sub_rank, uint16_t, MN);
    POA_CARVE(e_src, uint16_t, ME);
    POA_CARVE(e_dst, uint16_t, ME);
    POA_CARVE(e_next, uint16_t, ME);
    POA_CARVE(e_w, int32_t, ME);
    POA_CARVE(e_ord, uint8_t, ME);
    POA_CARVE(row_meta, uint32_t, MN);
    POA_CARVE(row_rec, uint32_t, MN + 1 + 128); /* +128: the fill prefetches 32-row blocks up to three blocks past the end */
    POA_CARVE(row_poff, uint32_t, MN + 2);
    POA_CARVE(row_pred, uint32_t, ME + MN + 96);
    POA_CARVE(row_pfill, uint32_t, ME + MN + 96); /* +96: the fill prefetches 32-entry blocks past the end */
    POA_CARVE(tb_node, int16_t, MN + ML + 2);
    POA_CARVE(tb_pos, int16_t, MN + ML + 2);
    POA_CARVE(asg, int32_t, ML + 1);
    POA_CARVE(cnt, uint32_t, MN + 1);
    POA_CARVE(roff, uint32_t, MN + 1);
    POA_CARVE(need, uint32_t, MN + 1);
    POA_CARVE(dirty, uint8_t, MN + 1);
    POA_CARVE(marks, uint8_t, MN);
    POA_CARVE(check, uint8_t, MN);
    POA_CARVE(stack, uint16_t, ME + (KA + 2) * MN);
    POA_CARVE(c_score, int32_t, MN);
    POA_CARVE(c_pred, int32_t, MN);
    o = (o + 255) / 256 * 256;
    s.S = base ? reinterpret_cast<int16_t*>(base + o) : nullptr;
    o += (p.wide_cells ? sizeof(int32_t) : sizeof(int16_t)) * (MN + 1) * (size_t)p.stride;
    o = (o + 255) / 256 * 256;
#undef POA_CARVE
    if (total_out) *total_out = o;
}

/* One window as the kernel sees it: sequences already in processing order. */
struct WindowView {
    int32_t n_seqs;
    const uint8_t* bases;    /* batch arena */
    const int8_t* weights;   /* compact arena: only sequences whose weights are not one constant live here */
    const int64_t* seq_off;  /* [n_seqs] start of each sequence in the bases arena, in PROCESSING order (the arena itself may hold
                                the sequences in any order: a pinned host arena is uploaded as it is, add order) */
    const int32_t* seq_len;  /* [n_seqs] their lengths */
    const int64_t* w_off;    /* [n_seqs] >= 0: offset of the sequence's weights in `weights`; < 0: every base weighs
                                -1 - w_off (racon: no quality string => 1, window.cpp:105-107; the '!' dummy quality of
                                a FASTA target => 0, polisher.cpp:171,392-395) -- such sequences ship no weight bytes */
    const int32_t* seq_begin; /* [n_seqs] layer span on the backbone, or -1 when the layer spans the window */
    const int32_t* seq_end;   /* (window.cpp:87,92-93 decides which; the host applies that rule)           */
    uint16_t* path;           /* MSA output only (else nullptr): arena parallel to `bases` (same seq_off) receiving the node
                                 every base of every sequence was assigned to -- the sequence's path through the graph,
                                 which spoa re-derives from edge labels (Node::successor, graph.cpp:31-43) and cudapoa
                                 from per-edge sequence lists (outgoing_edges_coverage, cudapoa_add_alignment.cuh:245-262) */
#if POA_FILL_DIGEST
    unsigned long long* fill_digest; /* [n_seqs] test build only: sum of fill_digest() over every fill of the sequence */
    int32_t* fill_count;             /* [n_seqs] fills of the sequence (adaptive retries included) */
#endif
#if POA_ALN_DIGEST
    unsigned long long* aln_digest;  /* [n_seqs] test build only: aln_digest() of the alignment added to the graph
                                        (last adaptive try) */
    int32_t* aln_count;              /* [n_seqs] its entries */
#endif
#if POA_GRAPH_DIGEST
    unsigned long long* graph_digest; /* [n_seqs] test build only: graph_digest() after sequence r was added and sorted
                                         (r = 0: the backbone); 0 once the window stopped on a status */
    int32_t* graph_nodes;             /* [n_seqs] nodes and edges of that graph */
    int32_t* graph_edges;
    unsigned long long* sub_digest;   /* [n_seqs] partial-span reads: sub_digest() of the subgraph's member order */
    int32_t* sub_count;               /* [n_seqs] its members */
#endif
};

/* Where a window's result goes: consensus and coverage are appended to compact arenas (one bump allocation per
 * window, 16-element granules), the per-window tables say where.  The coverage trim of window.cpp:118-139 is
 * evaluated here too, so that a caller that only wants the trimmed consensus never downloads the coverage. */
struct WindowOut {
    uint8_t* cons;     /* compact consensus arena                          */
    uint16_t* cov;     /* compact coverage arena, same offsets             */
    uint32_t* cursor;  /* elements used so far in both arenas              */
    int32_t* len;      /* this window's slots in the per-window tables ... */
    int32_t* status;
    int32_t* off;      /* ... offset of its consensus in the arenas        */
    int32_t* trim;     /* ... first (low 16 bits) and last (high 16 bits, signed) index whose coverage is
                          >= (trim_nseq - 1) / 2; first > last: no such base */
    int32_t trim_nseq; /* sequences the trim threshold counts (window.cpp:121: sequences_.size()) */
#if POA_GRAPH_DIGEST
    unsigned long long* cons_digest; /* [2] test build only: cons_digest() after consensus_scores_full() and after the
                                        last round of branch completion (generate_consensus writes them) */
    int32_t* cons_rounds;            /* rounds of branch completion */
#endif
};

/* OutputType::msa: a window's rows are bump-allocated in a compact arena like its consensus (n_seqs rows of `cols`
 * bytes).  Kept apart from WindowOut: process_window() never sees it, the caller runs generate_msa() afterwards. */
struct MsaOut {
    uint8_t* arena;
    unsigned long long* cursor; /* bytes used so far */
    unsigned long long cap;     /* arena capacity (the host admits windows by their worst case, this is the backstop) */
    long long* off;             /* this window's slots in the per-window tables: where its rows start ... */
    int32_t* cols;              /* ... their length ... */
    int32_t* status;            /* ... and the status of its MSA */
};

POA_FN uint32_t poa_bump(uint32_t* cursor, uint32_t n) {
#if POA_DEVICE
    return atomicAdd(cursor, n);
#else
    const uint32_t o = *cursor;
    *cursor += n;
    return o;
#endif
}
POA_FN unsigned long long poa_bump64(unsigned long long* cursor, unsigned long long n) {
#if POA_DEVICE
    return atomicAdd(cursor, n);
#else
    const unsigned long long o = *cursor;
    *cursor += n;
    return o;
#endif
}
POA_FN int poa_fls(unsigned m) { /* index of highest set bit, m != 0 */
#if POA_DEVICE
    return 31 - __clz((int)m);
#else
    return 31 - __builtin_clz(m);
#endif
}

/* Mutable per-window state (warp-uniform scalars). */
struct WinState {
    int32_t n_nodes;
    int32_t n_edges;
    int32_t status;
    int32_t n_columns; /* aligned cliques (a node without aligned mates counts as one): no path visits more nodes */
    int32_t band_hit;  /* traceback: the path came within TB_EDGE_MARGIN columns of a band edge that is not a matrix edge */
};

/* After a phase function has updated the state through its reference (local memory, which the compiler must assume
 * lane-dependent), pass the scalars through poa_uniform() so that the caller's control flow stays provably uniform. */
POA_FN void winstate_uniform(WinState& st) {
    st.n_nodes = poa_uniform(st.n_nodes);
    st.n_edges = poa_uniform(st.n_edges);
    st.status = poa_uniform(st.status);
    st.n_columns = poa_uniform(st.n_columns);
    st.band_hit = poa_uniform(st.band_hit);
}

/* optional per-phase cycle counters (diagnostics: B200POA_PHASE_TIMERS=1), device flavour only */
enum Phase { PH_PROGRAM = 0, PH_FILL, PH_TRACEBACK, PH_ADD, PH_TOPSORT, PH_CONSENSUS, PH_OTHER, PH_COUNT };
struct PhaseTimer {
    unsigned long long* acc; /* [PH_COUNT] global accumulators, or nullptr */
    long long t;
    POA_FN void start() {
#if POA_DEVICE
        if (acc) t = clock64();
#endif
    }
    POA_FN void lap(int ph) {
#if POA_DEVICE
        if (acc) {
            const long long n = clock64();
            if ((threadIdx.x & 31u) == 0u) atomicAdd(&acc[ph], (unsigned long long)(n - t));
            t = n;
        }
#else
        (void)ph;
#endif
    }
};

/* Sub-phase cycle counters: compiled in only for experiments (scripts/build_variant.sh ... -DB200POA_SUBTIMERS=1),
 * read back with b200poa_debug_subtimers(). */
#if POA_DEVICE && defined(B200POA_SUBTIMERS)
__device__ unsigned long long g_subtimers[32];
#define POA_SUB_BEGIN() long long _sub_t = clock64()
#define POA_SUB_LAP(k)                                                                          \
    do {                                                                                        \
        const long long _n = clock64();                                                         \
        if ((threadIdx.x & 31u) == 0u) atomicAdd(&g_subtimers[k], (unsigned long long)(_n - _sub_t)); \
        _sub_t = _n;                                                                            \
    } while (0)
#else
#define POA_SUB_BEGIN() ((void)0)
#define POA_SUB_LAP(k) ((void)0)
#endif

/* row_meta entry: letter | sink << 8 | in-degree << 16 */
POA_FN uint32_t meta_make(int32_t code, bool sink, int32_t nin) {
    return (uint32_t)code | (sink ? 0x100u : 0u) | ((uint32_t)nin << 16);
}

/* ------------------------------------------------------------------------------------------
 * Phase 0: backbone chain  (graph.cpp:274-292 add_sequence + :177-185; window.cpp:73-76)
 * ---------------------------------------------------------------------------------------- */
POA_FN_NOINLINE void init_backbone(const Slot& s_ref, const Params p_ref, WinState& st, const uint8_t* seq,
                          const int8_t* w, int32_t wconst, int32_t len) {
    const Slot s = s_ref;     /* local copies: no reloads of the descriptor after every store */
    const Params p = p_ref;
    len = poa_uniform(len);
    wconst = poa_uniform(wconst);
    if (len > p.max_nodes || len - 1 > p.max_edges) {
        st.status = ST_SEQ_LEN_EXCEEDED_MAX_NODES;
        return;
    }
    for (int32_t base = 0; base < len; base += 32) {
        POA_LANES(l) {
            const int32_t k = base + l;
            if (k >= len) continue;
            s.code[k] = seq[k];
            s.nin[k] = (k > 0) ? 1 : 0;
            s.nout[k] = (k + 1 < len) ? 1 : 0;
            s.in_head[k] = (k > 0) ? (uint16_t)(k - 1) : NONE16;
            s.in_tail[k] = s.in_head[k];
            s.cov[k] = (len >= 2) ? 1 : 0; /* Node::coverage counts edge labels (graph.cpp:44-58) */
            s.aln_cnt[k] = 0;
            s.root[k] = (uint16_t)k;
            s.lpos[k] = 0;
            s.cnt[k] = 1;
            s.need[k] = 0;
            s.dirty[k] = 0;
            s.rank_of[k] = (uint16_t)k;
            s.node_at[k] = (uint16_t)k;
            s.row_meta[k] = meta_make(seq[k], k + 1 >= len, k > 0 ? 1 : 0);
            if (k > 0) { /* edge k-1 : (k-1) -> k */
                s.e_src[k - 1] = (uint16_t)(k - 1);
                s.e_dst[k - 1] = (uint16_t)k;
                s.e_next[k - 1] = NONE16;
                s.e_w[k - 1] = w ? (int32_t)w[k - 1] + (int32_t)w[k] : 2 * wconst;
                s.e_ord[k - 1] = 0;
            }
        }
    }
    POA_SYNC();
    st.n_nodes = len;
    st.n_edges = len - 1;
    st.n_columns = len;
}

/* ------------------------------------------------------------------------------------------
 * Phase 1: row program.  Linearise the graph in rank order for the DP fill and traceback.
 *   row r+1  <->  node_at[r];  predecessor rows in in-edge order; a node without in-edges gets the
 *   single virtual predecessor row 0 (sisd_alignment_engine.cpp:289-290).
 * Band: static, centred on the (0,0)-(N,len) diagonal like cudapoa_nw_banded.cuh:35-55, but
 * snapped to 8-cell lanes so a row shift is a whole-lane shift.
 * ---------------------------------------------------------------------------------------- */
/* Packed row record (one u32 per row, read 32 rows at a time by the fill and distributed by
 * shuffle):  code[0:8) | sink[8] | profile row[9:12) | pred0-is-previous-row[12] | npred[13:21) |
 * band start / 8 [21:32). */
POA_FN uint32_t rec_make(int32_t code, bool sink, int32_t prow, int32_t npred, int32_t bs) {
    return (uint32_t)code | (sink ? 0x100u : 0u) | ((uint32_t)prow << 9) |
           ((uint32_t)npred << 13) | ((uint32_t)(bs >> 3) << 21);
}
POA_FN int32_t rec_code(uint32_t r) { return (int32_t)(r & 0xFFu); }
POA_FN bool rec_far(uint32_t r) { return (r & 0x1000u) != 0; }
POA_FN void poa_atomic_or(uint32_t* p, uint32_t v) {
#if POA_DEVICE
    atomicOr(p, v);
#else
    *p |= v;
#endif
}
POA_FN bool rec_sink(uint32_t r) { return (r & 0x100u) != 0; }
POA_FN int32_t rec_prow(uint32_t r) { return (int32_t)((r >> 9) & 7u); }
POA_FN int32_t rec_npred(uint32_t r) { return (int32_t)((r >> 13) & 0xFFu); }
POA_FN int32_t rec_bs(uint32_t r) { return (int32_t)(r >> 21) << 3; }
POA_FN int32_t prof_row_of(int32_t code) { /* A,C,G,T -> 0..3, anything else -> 4 (profile row built on demand) */
    switch (code) {
        case 'A': return 0;
        case 'C': return 1;
        case 'G': return 2;
        case 'T': return 3;
        default: return 4;
    }
}

/* Predecessor entry as the fill consumes it:  far[0] | band start/8 [1:12) | delta[12:32) (signed), with
 * delta = (ring slot of the predecessor row) * ring_row_bytes - band_start * 2, so that the shared-memory
 * address of the predecessor cell under column c is  ring_base + c*2 + delta  (one add per predecessor). */
/* Every ring row carries RING_PAD_FRONT cells before and RING_PAD_BACK cells after its band cells, all NEG:
 * the fill reads a predecessor row at a small forward shift (its band starts at or before ours) and one cell
 * to the left, and lands in the pads instead of testing the band limits. */
constexpr int RING_PAD_FRONT = 8;
constexpr int RING_PAD_BACK = 24;
POA_FN uint32_t pfill_make(int32_t row, int32_t pr, int32_t bsp, int32_t ring_rows, int32_t ring_stride) {
    const int32_t far = (row - pr >= ring_rows) ? 1 : 0;
    const int32_t delta = (pr & (ring_rows - 1)) * ring_stride * 2 + RING_PAD_FRONT * 2 - bsp * 2;
    return (uint32_t)far | ((uint32_t)(bsp >> 3) << 1) | ((uint32_t)delta << 12);
}
/* a row takes the fill's general path (record bit 12) if a predecessor is older than the ring or its band
 * starts more than the back pad before the row's own */
POA_FN bool pred_needs_general_path(int32_t row, int32_t bs_row, int32_t pr, int32_t bsp, int32_t ring_rows) {
    return row - pr >= ring_rows || bs_row - bsp > RING_PAD_BACK;
}

struct ReadGeom {
    int32_t len;    /* read length                                    */
    int32_t colsP;  /* (len+1) rounded up to a multiple of 8          */
    int32_t bw;     /* cells per row actually computed (multiple of 8) */
    int32_t banded; /* 1 if bw < colsP                                 */
    int32_t n_rows; /* graph rows of this alignment (whole graph, or the subgraph of a partial-span layer) */
    uint32_t step;  /* band centre advance per row, 16.16 fixed point: (len << 16) / n_rows */
};

POA_FN ReadGeom read_geometry(const Params& p, int32_t len, int32_t n_rows, int32_t band_width) {
    ReadGeom g;
    (void)p;
    g.len = len;
    g.n_rows = n_rows;
    g.colsP = (len + 1 + 7) & ~7;
    g.banded = (band_width > 0 && g.colsP > band_width) ? 1 : 0;
    g.bw = g.banded ? band_width : g.colsP;
    g.step = ((uint32_t)len << 16) / (uint32_t)(n_rows > 0 ? n_rows : 1); /* len < 2^15 by the config limits */
    return g;
}

/* Which DP fill a read on int16 cells takes (poa_fill.cuh, CudaFill); a read on 32-bit cells always runs fill_rows_i32.
 * One rule for the kernel and the emulation, which reports per window how many reads took each variant. */
enum FillVariant : int32_t {
    FILL_WIDE1 = 0,      /* full band, colsP <= 256: fill_rows_wide<1> ... */
    FILL_WIDE2,          /* ... <= 512 */
    FILL_WIDE3,          /* ... <= 768 */
    FILL_WIDE4,          /* ... <= 1024: fill_rows_wide<4> */
    FILL_CHUNKED_FULL,   /* full band over more than 1024 columns: fill_rows<false>, 256-column chunk passes */
    FILL_FULLW,          /* static band of exactly 256 columns: fill_rows<true> */
    FILL_CHUNKED_BANDED, /* any other band width: fill_rows<false> */
    FILL_VARIANTS
};
/* The rule, written once: calls visitor.run<variant>() for the variant of a read.  CudaFill runs the fill itself
 * through it (the same branches as a plain if-chain, so the kernel's code does not depend on this indirection). */
#if POA_DEVICE
#pragma nv_exec_check_disable
#endif
template <class Visitor>
POA_HD int32_t fill_dispatch(const ReadGeom& g, Visitor& v) {
    if (g.banded) return (g.bw == CHUNK) ? v.template run<FILL_FULLW>() : v.template run<FILL_CHUNKED_BANDED>();
    if (g.colsP <= 256) return v.template run<FILL_WIDE1>();
    if (g.colsP <= 512) return v.template run<FILL_WIDE2>();
    if (g.colsP <= 768) return v.template run<FILL_WIDE3>();
    if (g.colsP <= 1024) return v.template run<FILL_WIDE4>();
    return v.template run<FILL_CHUNKED_FULL>();
}
struct FillVariantOf {
    template <int32_t V>
    POA_HD int32_t run() { return V; }
};
POA_HD int32_t fill_variant(const ReadGeom& g) {
    FillVariantOf v;
    return fill_dispatch(g, v);
}

/* Copies of the geometry / parameters a phase function received by reference (i.e. through local memory, which
 * the compiler must treat as lane-dependent), laundered through poa_uniform(): see poa_simt.cuh. */
POA_FN ReadGeom geom_uniform(const ReadGeom& r) {
    ReadGeom g;
    g.len = poa_uniform(r.len);
    g.colsP = poa_uniform(r.colsP);
    g.bw = poa_uniform(r.bw);
    g.banded = poa_uniform(r.banded);
    g.n_rows = poa_uniform(r.n_rows);
    g.step = (uint32_t)poa_uniform((int32_t)r.step); /* < 2^31: len < 2^15 */
    return g;
}
/* Static band: centred on the (0,0)-(n_rows,len) diagonal.  One division per read (ReadGeom::step), a multiply per
 * row: every phase recomputes a row's band start with this function instead of loading it. */
POA_FN int32_t band_start(const ReadGeom& g, int32_t row, int32_t n_rows) {
    (void)n_rows; /* == g.n_rows */
    if (!g.banded) return 0;
    const int32_t center = (int32_t)(((uint32_t)row * g.step) >> 16); /* row <= n_rows: row * step <= len << 16 < 2^31 */
    int32_t bs = center - g.bw / 2;
    if (bs > g.colsP - g.bw) bs = g.colsP - g.bw;
    if (bs < 0) bs = 0;
    return bs & ~7;
}

#ifndef POA_PB_U
#define POA_PB_U 4
#endif
constexpr int PB_U = POA_PB_U; /* edges per lane per step in the edge-parallel pass of the row program */
POA_FN_NOINLINE void build_program(const Slot& s_ref, const Params p_ref, WinState& st, const ReadGeom g_ref) {
    const Slot s = s_ref;     /* local copies: no reloads of the descriptor after every store */
    const Params p = p_ref;
    const ReadGeom g = geom_uniform(g_ref);
    POA_SUB_BEGIN();
    const int32_t N = poa_uniform(st.n_nodes), E = poa_uniform(st.n_edges);
    /* pass A, node-parallel, 64 rows per step: row records and CSR offsets (row r+1 <-> node_at[r]) */
    int32_t run = 0; /* running predecessor offset (uniform) */
    POA_LANE0 { s.row_rec[0] = 0; }
    PerLane<int> wide;
    POA_LANES(l) { wide[l] = 0; }
    for (int32_t base = 0; base < N; base += 64) {
        PerLane<int> c0, c1, z0, z1;
        POA_LANES(l) { /* letter, in-degree and sink flag by rank: one coalesced load per row (row_meta) */
            const int32_t r0 = base + 2 * l, r1 = r0 + 1;
            const uint32_t m0 = r0 < N ? s.row_meta[r0] : 0u, m1 = r1 < N ? s.row_meta[r1] : 0u;
            const int32_t d0 = (int32_t)(m0 >> 16), d1 = (int32_t)(m1 >> 16);
            const int32_t k0 = (int32_t)(m0 & 0xFFu), k1 = (int32_t)(m1 & 0xFFu);
            const bool s0 = (m0 & 0x100u) != 0, s1 = (m1 & 0x100u) != 0;
            c0[l] = r0 < N ? (d0 ? d0 : 1) : 0;
            c1[l] = r1 < N ? (d1 ? d1 : 1) : 0;
            z0[l] = (r0 < N && d0 == 0) ? 1 : 0; /* no in-edge: the virtual predecessor row 0 */
            z1[l] = (r1 < N && d1 == 0) ? 1 : 0;
            if (c0[l] > 255 || c1[l] > 255) wide[l] = 1;
            if (r0 < N) s.row_rec[r0 + 1] = rec_make(k0, s0, prof_row_of(k0), c0[l] & 0xFF, band_start(g, r0 + 1, N));
            if (r1 < N) s.row_rec[r1 + 1] = rec_make(k1, s1, prof_row_of(k1), c1[l] & 0xFF, band_start(g, r1 + 1, N));
        }
        PerLane<int> off;
        POA_LANES(l) { off[l] = c0[l] + c1[l]; }
        const int32_t tot = warp_exscan(off);
        POA_LANES(l) {
            const int32_t r0 = base + 2 * l, r1 = r0 + 1;
            const int32_t o0 = run + off[l], o1 = o0 + c0[l];
            if (r0 < N) {
                s.row_poff[r0 + 1] = (uint32_t)o0;
                if (z0[l]) { /* virtual predecessor row 0 (sisd_alignment_engine.cpp:289-290) */
                    s.row_pred[o0] = 0;
                    s.row_pfill[o0] = pfill_make(r0 + 1, 0, 0, p.ring_rows, p.ring_stride);
                    if (pred_needs_general_path(r0 + 1, band_start(g, r0 + 1, N), 0, 0, p.ring_rows)) s.row_rec[r0 + 1] |= 0x1000u;
                }
            }
            if (r1 < N) {
                s.row_poff[r1 + 1] = (uint32_t)o1;
                if (z1[l]) {
                    s.row_pred[o1] = 0;
                    s.row_pfill[o1] = pfill_make(r1 + 1, 0, 0, p.ring_rows, p.ring_stride);
                    if (pred_needs_general_path(r1 + 1, band_start(g, r1 + 1, N), 0, 0, p.ring_rows)) s.row_rec[r1 + 1] |= 0x1000u;
                }
            }
        }
        run += tot;
    }
    POA_LANE0 { s.row_poff[N + 1] = (uint32_t)run; }
    if (warp_ballot(wide)) st.status = ST_EDGE_COUNT_EXCEEDED; /* in-degree > 255 does not fit the record */
    POA_SYNC();
    POA_SUB_LAP(0);
    /* pass B, edge-parallel, 128 edges per step: every edge drops its source row into its slot of the
     * target's predecessor list (slot = e_ord, the edge's position in the in-edge list, fixed when the
     * edge was created) -- no linked-list walking, three dependent loads per edge. */
    for (int32_t base = 0; base < E; base += 32 * PB_U) {
        POA_LANES(l) {
            int32_t d[PB_U], u[PB_U], q[PB_U], rd[PB_U], ru[PB_U], o[PB_U];
            bool ok[PB_U];
#pragma unroll
            for (int32_t k = 0; k < PB_U; ++k) { /* level 1: the edge itself (independent loads) */
                const int32_t e = base + 32 * k + l;
                ok[k] = e < E;
                d[k] = ok[k] ? (int32_t)s.e_dst[e] : 0;
                u[k] = ok[k] ? (int32_t)s.e_src[e] : 0;
                q[k] = ok[k] ? (int32_t)s.e_ord[e] : 0;
            }
#pragma unroll
            for (int32_t k = 0; k < PB_U; ++k) { /* level 2: ranks */
                rd[k] = s.rank_of[d[k]] + 1;
                ru[k] = s.rank_of[u[k]] + 1;
            }
#pragma unroll
            for (int32_t k = 0; k < PB_U; ++k) o[k] = (int32_t)s.row_poff[rd[k]] + q[k]; /* level 3: slot */
#pragma unroll
            for (int32_t k = 0; k < PB_U; ++k) {
                if (!ok[k]) continue;
                const int32_t pbs = band_start(g, ru[k], N);
                s.row_pred[o[k]] = (uint32_t)ru[k] | ((uint32_t)pbs << 16);
                s.row_pfill[o[k]] = pfill_make(rd[k], ru[k], pbs, p.ring_rows, p.ring_stride);
                if (pred_needs_general_path(rd[k], band_start(g, rd[k], N), ru[k], pbs, p.ring_rows))
                    poa_atomic_or(&s.row_rec[rd[k]], 0x1000u); /* rare */
            }
        }
    }
    POA_SUB_LAP(1);
    POA_SYNC();
}

/* ------------------------------------------------------------------------------------------
 * Partial-span layers (window.cpp:96-103): the read is aligned to the SUBGRAPH of nodes from which the
 * backbone node `end` can be reached backwards without passing a node with id < begin
 * (graph.cpp:592-615 extract_subgraph_nodes), in the topological order spoa computes for that
 * subgraph (graph.cpp:617-673: nodes relabelled in increasing id, in-edges and aligned lists filtered,
 * then Graph::topological_sort).  Relabelling is monotone, so that order is spoa's DFS run on the
 * original ids restricted to the members.  Serial on lane 0: only layers that do not span the window
 * take this path, and the member set is a fraction of the graph.
 * Outputs: sub_at[0..n_sub), sub_rank[] (NONE16 for non-members), roff[v] != 0 iff v has a successor inside the
 * subgraph.  Returns n_sub.
 * ---------------------------------------------------------------------------------------- */
POA_FN_NOINLINE int32_t mark_subgraph_serial(const Slot& s_ref, const Params p_ref, WinState& st, int32_t begin, int32_t end) {
    const Slot s = s_ref;
    const Params p = p_ref;
    const int32_t N = poa_uniform(st.n_nodes);
    begin = poa_uniform(begin);
    end = poa_uniform(end);
    for (int32_t base = 0; base < N; base += 32) {
        POA_LANES(l) {
            if (base + l < N) {
                s.sub_rank[base + l] = NONE16;
                s.marks[base + l] = 0; /* 1 = member (then DFS marks 0/1/2 live in check[]) */
                s.roff[base + l] = 0;
            }
        }
    }
    POA_SYNC();
    int32_t n_sub = 0;
    POA_LANE0 {
        /* membership: graph.cpp:592-615 */
        int32_t sp = 0;
        s.stack[sp++] = (uint16_t)end;
        while (sp != 0) {
            const int32_t id = s.stack[--sp];
            if (s.marks[id] == 0 && id >= begin) {
                for (uint16_t e = s.in_head[id]; e != NONE16; e = s.e_next[e]) s.stack[sp++] = s.e_src[e];
                for (int32_t q = 0; q < s.aln_cnt[id]; ++q) s.stack[sp++] = s.aln[id * KA + q];
                s.marks[id] = 1;
            }
        }
        /* order: graph.cpp:294-354 on the members (c_pred[]: 0 unmarked / 1 temporary / 2 permanent,
         * c_score[]: check_aligned flag; both arrays are free during the alignment of a read) */
        for (int32_t i = 0; i < N; ++i) {
            s.c_pred[i] = 0;
            s.c_score[i] = 1;
        }
        int32_t out = 0;
        for (int32_t i = 0; i < N; ++i) {
            if (!s.marks[i] || s.c_pred[i] != 0) continue;
            sp = 0;
            s.stack[sp++] = (uint16_t)i;
            while (sp != 0) {
                const int32_t id = s.stack[sp - 1];
                bool valid = true;
                if (s.c_pred[id] != 2) {
                    for (uint16_t e = s.in_head[id]; e != NONE16; e = s.e_next[e]) {
                        const int32_t u = s.e_src[e];
                        if (s.marks[u] && s.c_pred[u] != 2) {
                            s.stack[sp++] = (uint16_t)u;
                            valid = false;
                        }
                    }
                    const int32_t na = s.aln_cnt[id];
                    if (s.c_score[id]) {
                        for (int32_t q = 0; q < na; ++q) {
                            const int32_t a = s.aln[id * KA + q];
                            if (s.marks[a] && s.c_pred[a] != 2) {
                                s.stack[sp++] = (uint16_t)a;
                                s.c_score[a] = 0;
                                valid = false;
                            }
                        }
                    }
                    if (valid) {
                        s.c_pred[id] = 2;
                        if (s.c_score[id]) {
                            s.sub_at[out] = (uint16_t)id;
                            s.sub_rank[id] = (uint16_t)out;
                            ++out;
                            for (int32_t q = 0; q < na; ++q) {
                                const int32_t a = s.aln[id * KA + q];
                                if (!s.marks[a]) continue; /* aligned list filtered to members (graph.cpp:660-666) */
                                s.sub_at[out] = (uint16_t)a;
                                s.sub_rank[a] = (uint16_t)out;
                                ++out;
                            }
                        }
                    } else {
                        s.c_pred[id] = 1;
                    }
                }
                if (valid) --sp;
            }
        }
        /* out-degree inside the subgraph (a member without member successors is a sink of the alignment) */
        for (int32_t r = 0; r < out; ++r) {
            const int32_t v = s.sub_at[r];
            for (uint16_t e = s.in_head[v]; e != NONE16; e = s.e_next[e])
                if (s.marks[s.e_src[e]]) s.roff[s.e_src[e]] += 1;
        }
        n_sub = out;
    }
    POA_SYNC();
    n_sub = warp_bcast0(n_sub);
    (void)p;
    return n_sub;
}

/* The same subgraph and the same order, computed by the whole warp.
 *   Members.  v is a member iff `end` can be reached from it through edges and aligned-node links without leaving the
 *   ids >= begin, and spoa's DFS started at member i emits exactly the members whose first such reachable id (in id
 *   order) is i: sroot(v) = min id reachable from v.  Both come out of ONE sweep over the full graph's ranks from
 *   `end` downwards: a node passes its sroot to the sources of its in-edges (lower ranks) and to its aligned nodes
 *   (the ranks next to it: a clique is emitted as one run, topological_sort graph.cpp:294-354).  32 ranks at a time,
 *   iterated until nothing changes; consecutive chunks overlap by a clique's length so that a clique cut by a chunk
 *   boundary is settled as a whole.  sroot lives in shared memory (the tile scratch, idle between two alignments).
 *   Order.  rank(v) = (members with a smaller sroot) + (position of v in the DFS of its sroot restricted to that
 *   sroot's members): the per-root decomposition of topsort_roots(), run from scratch with every root "dirty".
 * Scratch that is free while a read is being prepared: the score matrix (counters, marks), stack, c_score/c_pred. */
POA_FN_NOINLINE void subgraph_members(const Slot& s_ref, int32_t N, int32_t begin, int32_t end, uint16_t* sroot) {
    const Slot s = s_ref;
    N = poa_uniform(N);
    begin = poa_uniform(begin);
    end = poa_uniform(end);
    uint32_t* const t_cnt = reinterpret_cast<uint32_t*>(s.S); /* [N] members per sroot */
    uint32_t* const t_need = t_cnt + N;                       /* [N] DFS stack bound per sroot */
    for (int32_t base = 0; base < N; base += 32) {
        POA_LANES(l) {
            const int32_t v = base + l;
            if (v < N) {
                s.sub_rank[v] = NONE16;
                s.roff[v] = 0;
                sroot[v] = NONE16;
                t_cnt[v] = 0;
                t_need[v] = 0;
            }
        }
    }
    POA_SYNC();
    POA_LANE0 { sroot[end] = (uint16_t)end; }
    int32_t r_top = (int32_t)s.rank_of[end] + KA;
    if (r_top > N - 1) r_top = N - 1;
    r_top = poa_uniform(r_top);
    POA_SYNC();
    /* ---- members and their sroot ---- */
    for (int32_t hi = r_top; hi >= 0; hi -= 32 - (KA + 1)) {
        POA_GRAPH_TWIN(sweep_chunk, s, hi);
        /* the chunk's topology, read once: up to four in-edge sources and the aligned nodes of every lane's node, packed
         * two ids per register (a longer in-edge list is walked in memory each time its node has something to pass on) */
        PerLane<int> vv, n_src, passed, s01, s23, m01, m23, m45, m6;
        POA_LANES(l) {
            const int32_t r = hi - l;
            int32_t v = r >= 0 ? (int32_t)s.node_at[r] : -1;
            if (v < begin) v = -1; /* backbone before `begin`: not a member, passes nothing on */
            vv[l] = v;
            passed[l] = 0x10000; /* the sroot this lane has last passed on (none yet) */
            uint32_t sp[4] = {NONE16, NONE16, NONE16, NONE16};
            uint32_t mt[8] = {NONE16, NONE16, NONE16, NONE16, NONE16, NONE16, NONE16, NONE16};
            int32_t n = 0;
            if (v >= 0) {
                for (uint16_t e = s.in_head[v]; e != NONE16;) {
                    const uint16_t nx = s.e_next[e];
                    const uint32_t u = s.e_src[e];
                    if (n < 4) sp[n] = u;
                    ++n;
                    e = nx;
                }
                const int32_t na = s.aln_cnt[v];
#pragma unroll
                for (int32_t q = 0; q < KA; ++q)
                    if (q < na) mt[q] = s.aln[v * KA + q];
            }
            n_src[l] = n;
            s01[l] = (int32_t)(sp[0] | (sp[1] << 16));
            s23[l] = (int32_t)(sp[2] | (sp[3] << 16));
            m01[l] = (int32_t)(mt[0] | (mt[1] << 16));
            m23[l] = (int32_t)(mt[2] | (mt[3] << 16));
            m45[l] = (int32_t)(mt[4] | (mt[5] << 16));
            m6[l] = (int32_t)mt[6];
        }
        /* pass sroots on until nothing moves.  Two lanes may write one target in the same step and the larger value
         * may land last: a lane counts its value as passed on only once every target is seen to hold it (or less). */
        for (;;) {
            PerLane<int> ch;
            POA_LANES(l) {
                ch[l] = 0;
                const int32_t v = vv[l];
                if (v < 0) continue;
                const int32_t x = sroot[v];
                if (x == NONE16 || x >= passed[l]) continue;
                const uint32_t tg[11] = {(uint32_t)s01[l] & 0xFFFFu, (uint32_t)s01[l] >> 16, (uint32_t)s23[l] & 0xFFFFu,
                                         (uint32_t)s23[l] >> 16,     (uint32_t)m01[l] & 0xFFFFu, (uint32_t)m01[l] >> 16,
                                         (uint32_t)m23[l] & 0xFFFFu, (uint32_t)m23[l] >> 16,     (uint32_t)m45[l] & 0xFFFFu,
                                         (uint32_t)m45[l] >> 16,     (uint32_t)m6[l] & 0xFFFFu};
                int32_t moved = 0;
#pragma unroll
                for (int32_t k = 0; k < 11; ++k) {
                    const int32_t u = (int32_t)tg[k];
                    const int32_t nx = x < u ? x : u;
                    if (u != NONE16 && u >= begin && (int32_t)sroot[u] > nx) {
                        sroot[u] = (uint16_t)nx;
                        moved = 1;
                    }
                }
                if (n_src[l] > 4) { /* rare: the rest of a long in-edge list */
                    int32_t k = 0;
                    for (uint16_t e = s.in_head[v]; e != NONE16; e = s.e_next[e], ++k) {
                        if (k < 4) continue;
                        const int32_t u = s.e_src[e];
                        const int32_t nx = x < u ? x : u;
                        if (u >= begin && (int32_t)sroot[u] > nx) {
                            sroot[u] = (uint16_t)nx;
                            moved = 1;
                        }
                    }
                }
                if (moved) ch[l] = 1; /* look again: the stores are checked in the next step */
                else passed[l] = x;   /* every target already holds it */
            }
            POA_SYNC();
            POA_GRAPH_TWIN(sweep_step);
            if (!warp_ballot(ch)) break;
        }
        if (hi < 32) break; /* this chunk reached rank 0 */
    }
}

/* second half of mark_subgraph(): the order of the members (functions of their own: see poa_simt.cuh on function size) */
POA_FN_NOINLINE int32_t subgraph_order(const Slot& s_ref, int32_t N, const uint16_t* sroot) {
    const Slot s = s_ref;
    N = poa_uniform(N);
    uint32_t* const t_cnt = reinterpret_cast<uint32_t*>(s.S); /* [N] members per sroot */
    uint32_t* const t_need = t_cnt + N;                       /* [N] DFS stack bound per sroot */
    uint32_t* const t_off = t_need + N;                       /* [N] first rank of the sroot's members */
    uint16_t* const t_lpos = reinterpret_cast<uint16_t*>(t_off + N); /* [N] position inside the sroot's DFS */
    uint8_t* const t_marks = reinterpret_cast<uint8_t*>(t_lpos + N); /* [N] DFS marks */
    uint8_t* const t_check = t_marks + N;                            /* [N] check_aligned flags */
    /* ---- 1. members: DFS flags, members and stack bound per sroot ---- */
    for (int32_t base = 0; base < N; base += 32 * TS_U) {
        POA_LANES(l) {
            int32_t r[TS_U], nn[TS_U];
#pragma unroll
            for (int32_t u = 0; u < TS_U; ++u) {
                const int32_t v = base + 32 * u + l;
                r[u] = v < N ? (int32_t)sroot[v] : (int32_t)NONE16;
                nn[u] = (v < N && r[u] != NONE16) ? (int32_t)s.nin[v] + (int32_t)s.aln_cnt[v] + 1 : 0;
            }
#pragma unroll
            for (int32_t u = 0; u < TS_U; ++u) {
                const int32_t v = base + 32 * u + l;
                if (v < N && r[u] != NONE16) {
                    t_marks[v] = 0;
                    t_check[v] = 1;
                    poa_atomic_add(&t_cnt[r[u]], 1u);
                    poa_atomic_add(&t_need[r[u]], (uint32_t)nn[u]);
                }
            }
        }
    }
    POA_SYNC();
    /* ---- 2a. offsets per sroot, work list of the sroots with more than one member ---- */
    int32_t out_run = 0, stk_run = 0, n_work = 0;
    for (int32_t base = 0; base < N; base += 64) {
        PerLane<int> ca, cb, na, nb, wa, wb;
        POA_LANES(l) {
            const int32_t i0 = base + 2 * l, i1 = i0 + 1;
            ca[l] = (i0 < N) ? (int)t_cnt[i0] : 0;
            cb[l] = (i1 < N) ? (int)t_cnt[i1] : 0;
            wa[l] = ca[l] > 1 ? 1 : 0;
            wb[l] = cb[l] > 1 ? 1 : 0;
            na[l] = wa[l] ? (int)t_need[i0] + 1 : 0;
            nb[l] = wb[l] ? (int)t_need[i1] + 1 : 0;
            if (ca[l] == 1) t_lpos[i0] = 0;
            if (cb[l] == 1) t_lpos[i1] = 0;
        }
        PerLane<int> oo, so, wo;
        POA_LANES(l) {
            oo[l] = ca[l] + cb[l];
            so[l] = na[l] + nb[l];
            wo[l] = wa[l] + wb[l];
        }
        const int32_t ctot = warp_exscan(oo);
        const int32_t stot = warp_exscan(so);
        const int32_t wtot = warp_exscan(wo);
        POA_LANES(l) {
            const int32_t i0 = base + 2 * l, i1 = i0 + 1;
            if (i0 < N) t_off[i0] = (uint32_t)(out_run + oo[l]);
            if (i1 < N) t_off[i1] = (uint32_t)(out_run + oo[l] + ca[l]);
            if (wa[l]) {
                s.c_score[n_work + wo[l]] = i0;
                s.c_pred[n_work + wo[l]] = stk_run + so[l];
            }
            if (wb[l]) {
                s.c_score[n_work + wo[l] + wa[l]] = i1;
                s.c_pred[n_work + wo[l] + wa[l]] = stk_run + so[l] + na[l];
            }
        }
        out_run += ctot;
        stk_run += stot;
        n_work += wtot;
    }
    POA_SYNC();
    /* ---- 2b. spoa's DFS inside each sroot (graph.cpp:294-354 on the members), 32 sroots at a time ---- */
    for (int32_t base = 0; base < n_work; base += 32) {
        POA_LANES(l) {
            if (base + l >= n_work) continue;
            const int32_t i = s.c_score[base + l];
            uint16_t* stk = s.stack + s.c_pred[base + l];
            int32_t sp = 0, out = 0;
            stk[sp++] = (uint16_t)i;
            while (sp != 0) {
                const int32_t id = stk[sp - 1];
                bool valid = true;
                if (t_marks[id] != 2) {
                    for (uint16_t e = s.in_head[id]; e != NONE16;) {
                        const uint16_t nx = s.e_next[e];
                        const int32_t u = s.e_src[e];
                        if ((int32_t)sroot[u] == i && t_marks[u] != 2) {
                            stk[sp++] = (uint16_t)u;
                            valid = false;
                        }
                        e = nx;
                    }
                    const int32_t na = s.aln_cnt[id];
                    if (t_check[id]) {
                        for (int32_t q = 0; q < na; ++q) {
                            const int32_t a = s.aln[id * KA + q];
                            if ((int32_t)sroot[a] == i && t_marks[a] != 2) { /* member clique mates share the sroot */
                                stk[sp++] = (uint16_t)a;
                                t_check[a] = 0;
                                valid = false;
                            }
                        }
                    }
                    if (valid) {
                        t_marks[id] = 2;
                        if (t_check[id]) {
                            t_lpos[id] = (uint16_t)out++;
                            for (int32_t q = 0; q < na; ++q) {
                                const int32_t a = s.aln[id * KA + q];
                                if ((int32_t)sroot[a] != i) continue; /* aligned list filtered to members (graph.cpp:660-666) */
                                t_lpos[a] = (uint16_t)out++;
                            }
                        }
                    } else {
                        t_marks[id] = 1;
                    }
                }
                if (valid) --sp;
            }
        }
    }
    POA_SYNC();
    /* ---- 3. subgraph ranks; out-degree inside the subgraph (a member without member successors is a sink) ---- */
    for (int32_t base = 0; base < N; base += 32) {
        POA_LANES(l) {
            const int32_t v = base + l;
            if (v >= N) continue;
            const int32_t x = sroot[v];
            if (x == NONE16) continue;
            const int32_t r = (int32_t)t_off[x] + (int32_t)t_lpos[v];
            s.sub_rank[v] = (uint16_t)r;
            s.sub_at[r] = (uint16_t)v;
            for (uint16_t e = s.in_head[v]; e != NONE16; e = s.e_next[e]) {
                const int32_t u = s.e_src[e];
                if (sroot[u] != NONE16) s.roff[u] = 1u; /* only "has a member successor" is ever asked; an atomic inside a
                                                           lane-divergent loop would also cost the module its uniformity proof */
            }
        }
    }
    POA_SYNC();
    return out_run;
}

POA_FN int32_t mark_subgraph(const Slot& s, const Params& p, WinState& st, int32_t begin, int32_t end, uint16_t* sroot,
                             int32_t sroot_cap) {
    const int32_t N = poa_uniform(st.n_nodes);
    POA_GRAPH_REACH_IF(!p.serial_topsort && N > sroot_cap, sub_serial);
    if (p.serial_topsort || N > sroot_cap) return mark_subgraph_serial(s, p, st, begin, end);
    subgraph_members(s, N, begin, end, sroot);
    return subgraph_order(s, N, sroot);
}

/* Row program of a subgraph alignment: rows follow sub_at[], predecessor lists keep only member
 * sources (in in-edge order), a row without member sources gets the virtual predecessor row 0. */
POA_FN_NOINLINE void build_program_sub(const Slot& s_ref, const Params p_ref, WinState& st, const ReadGeom g_ref) {
    const Slot s = s_ref;
    const Params p = p_ref;
    const ReadGeom g = geom_uniform(g_ref);
    const int32_t N = g.n_rows;
    int32_t run = 0;
    POA_LANE0 { s.row_rec[0] = 0; }
    PerLane<int> wide;
    POA_LANES(l) { wide[l] = 0; }
    for (int32_t base = 0; base < N; base += 32) {
        PerLane<int> c;
        POA_LANES(l) {
            const int32_t r = base + l;
            c[l] = 0;
            if (r < N) {
                const int32_t v = s.sub_at[r];
                int32_t d = 0;
                for (uint16_t e = s.in_head[v]; e != NONE16; e = s.e_next[e])
                    if (s.sub_rank[s.e_src[e]] != NONE16) ++d;
                c[l] = d ? d : 1;
            }
        }
        PerLane<int> off = c;
        const int32_t tot = warp_exscan(off);
        POA_LANES(l) {
            const int32_t r = base + l;
            if (r >= N) continue;
            const int32_t v = s.sub_at[r];
            const int32_t o = run + off[l];
            s.row_poff[r + 1] = (uint32_t)o;
            int32_t k = 0;
            bool far = false;
            for (uint16_t e = s.in_head[v]; e != NONE16; e = s.e_next[e]) {
                const int32_t sr = s.sub_rank[s.e_src[e]];
                if (sr == NONE16) continue;
                const int32_t pr = sr + 1;
                const int32_t pbs = band_start(g, pr, N);
                s.row_pred[o + k] = (uint32_t)pr | ((uint32_t)pbs << 16);
                s.row_pfill[o + k] = pfill_make(r + 1, pr, pbs, p.ring_rows, p.ring_stride);
                if (pred_needs_general_path(r + 1, band_start(g, r + 1, N), pr, pbs, p.ring_rows)) far = true;
                ++k;
            }
            if (k == 0) {
                s.row_pred[o] = 0;
                s.row_pfill[o] = pfill_make(r + 1, 0, 0, p.ring_rows, p.ring_stride);
                if (pred_needs_general_path(r + 1, band_start(g, r + 1, N), 0, 0, p.ring_rows)) far = true;
            }
            if (c[l] > 255) wide[l] = 1;
            const int32_t code = s.code[v];
            s.row_rec[r + 1] = rec_make(code, s.roff[v] == 0, prof_row_of(code), c[l] & 0xFF, band_start(g, r + 1, N)) |
                               (far ? 0x1000u : 0u);
        }
        run += tot;
    }
    POA_LANE0 { s.row_poff[N + 1] = (uint32_t)run; }
    if (warp_ballot(wide)) st.status = ST_EDGE_COUNT_EXCEEDED;
    POA_SYNC();
}

/* Score accessor used by the traceback (and by the scalar fill): cells outside the row's band
 * read as NEG (cudapoa_nw_banded.cuh:103-116 does the same with min_score_value). */
POA_FN int32_t score_at(const Slot& s, const Params& p, const ReadGeom& g, int32_t row, int32_t col) {
    if (col < 0) return NEG;
    const int32_t bs = rec_bs(s.row_rec[row]);
    const int32_t o = col - bs;
    if (o < 0 || o >= g.bw) return NEG;
    return s.S[(size_t)row * p.stride + o];
}

/* score accessor when the row's band start is already known (row_pred carries it) */
POA_FN int32_t score_at_bs(const Slot& s, const Params& p, const ReadGeom& g, int32_t row, int32_t bs, int32_t col) {
    if (col < 0) return NEG;
    const int32_t o = col - bs;
    if (o < 0 || o >= g.bw) return NEG;
    return s.S[(size_t)row * p.stride + o];
}

/* ------------------------------------------------------------------------------------------
 * 32-bit cells: the fallback for alignments that do not fit int16 (score_range_ok), i.e. where spoa switches its
 * SIMD engine to int32 (simd_alignment_engine.cpp:668-673).  Same recurrence, same row program, same band, same
 * skewed domain S = H - j*gap, one cell per lane per pass, predecessor rows read back from the score matrix (no
 * shared-memory ring), and a plain serial walk for the traceback: a correct path for rare, very large windows, not a
 * fast one.  The matrix overlays the int16 score region (Params::wide_cells: sized for it).
 * ---------------------------------------------------------------------------------------- */
constexpr int32_t NEG32 = -(1 << 29);

POA_FN int32_t cell32(const int32_t* S32, int32_t stride, int32_t bw, int32_t row, int32_t bs, int32_t col) {
    if (col < 0) return NEG32;
    const int32_t o = col - bs;
    if (o < 0 || o >= bw) return NEG32;
    return S32[(size_t)row * stride + o];
}

POA_FN_NOINLINE int32_t fill_rows_i32(const Slot& s_ref, const Params p, const ReadGeom g, const uint8_t* read) {
    const Slot s = s_ref;
    int32_t* const S32 = reinterpret_cast<int32_t*>(s.S);
    const int32_t N = g.n_rows, bw = g.bw, stride = p.stride;
    const int32_t mg = p.match - p.gap, xg = p.mismatch - p.gap;
    for (int32_t o0 = 0; o0 < bw; o0 += 32) {
        POA_LANES(l) {
            if (o0 + l < bw) S32[o0 + l] = 0; /* row 0: H = j*gap  =>  S = 0 */
        }
    }
    POA_SYNC();
    int32_t best = NEG32 - 1, end_row = 0;
    for (int32_t i = 1; i <= N; ++i) {
        const uint32_t rec = s.row_rec[i];
        const int32_t code = rec_code(rec), np = rec_npred(rec), bs = rec_bs(rec);
        const int32_t po = (int32_t)s.row_poff[i];
        int32_t carry = NEG32;
        for (int32_t o0 = 0; o0 < bw; o0 += 32) {
            PerLane<int> x;
            POA_LANES(l) {
                const int32_t o = o0 + l, c = bs + o;
                int32_t t = NEG32;
                if (o < bw) {
                    const int32_t prof = (c >= 1 && c <= g.len && (int32_t)read[c - 1] == code) ? mg : xg;
                    for (int32_t k = 0; k < np; ++k) {
                        const uint32_t pe = s.row_pred[po + k];
                        const int32_t pr = (int32_t)(pe & 0xFFFFu), pbs = (int32_t)(pe >> 16);
                        const int32_t d = cell32(S32, stride, bw, pr, pbs, c - 1) + prof;
                        const int32_t v = cell32(S32, stride, bw, pr, pbs, c) + p.gap;
                        if (d > t) t = d;
                        if (v > t) t = v;
                    }
                }
                x[l] = t;
            }
            warp_incl_max(x);
            POA_LANES(l) {
                const int32_t o = o0 + l;
                int32_t t = x[l] > carry ? x[l] : carry;
                if (t < NEG32) t = NEG32;
                x[l] = t;
                if (o < bw) S32[(size_t)i * stride + o] = t;
            }
            carry = poa_uniform(warp_get(x, 31));
        }
        POA_SYNC(); /* row i is visible to every lane before it is read as a predecessor */
        if (rec_sink(rec)) {
            const int32_t v = cell32(S32, stride, bw, i, bs, g.len);
            if (v > best) {
                best = v;
                end_row = i;
            }
        }
    }
    return end_row;
}

/* spoa's traceback priority (sisd_alignment_engine.cpp:366-424) on the int32 matrix: serial on lane 0. */
POA_FN_NOINLINE int32_t traceback_i32(const Slot& s_ref, const Params p, WinState& st, const ReadGeom g, int32_t end_row,
                                      const uint8_t* read, const uint16_t* row_node) {
    const Slot s = s_ref;
    const int32_t* const S32 = reinterpret_cast<const int32_t*>(s.S);
    const int32_t cap = p.max_nodes + p.max_len + 2, stride = p.stride, bw = g.bw;
    const int32_t mg = p.match - p.gap, xg = p.mismatch - p.gap;
    int32_t w = cap, lost = 0;
    POA_TB_REACH(i32_reads);
    POA_LANE0 {
        int32_t i = end_row, j = g.len;
        while (!(i == 0 && j == 0) && !lost) {
            if (w <= 0) {
                lost = 1;
                break;
            }
            int32_t ni = i, nj = j;
            if (i == 0) {
                nj = j - 1; /* row 0: only horizontal moves are left */
            } else {
                const uint32_t rec = s.row_rec[i];
                const int32_t np = rec_npred(rec), bs = rec_bs(rec), po = (int32_t)s.row_poff[i];
                const int32_t cur = cell32(S32, stride, bw, i, bs, j);
                const int32_t prof = (j > 0 && rec_code(rec) == (int32_t)read[j - 1]) ? mg : xg;
                bool found = false;
                for (int32_t k = 0; k < np && !found && j > 0; ++k) { /* diagonal, in-edges in order */
                    const uint32_t pe = s.row_pred[po + k];
                    if (cell32(S32, stride, bw, (int32_t)(pe & 0xFFFFu), (int32_t)(pe >> 16), j - 1) + prof == cur) {
                        ni = (int32_t)(pe & 0xFFFFu);
                        nj = j - 1;
                        found = true;
                    }
                }
                for (int32_t k = 0; k < np && !found; ++k) { /* vertical, in-edges in order */
                    const uint32_t pe = s.row_pred[po + k];
                    if (cell32(S32, stride, bw, (int32_t)(pe & 0xFFFFu), (int32_t)(pe >> 16), j) + p.gap == cur) {
                        ni = (int32_t)(pe & 0xFFFFu);
                        found = true;
                    }
                }
                if (!found) {
                    if (j > 0 && cell32(S32, stride, bw, i, bs, j - 1) == cur) nj = j - 1; /* horizontal */
                    else lost = 1;
                }
            }
            if (lost) break;
            --w;
            s.tb_node[w] = (int16_t)((i == ni) ? -1 : (int32_t)row_node[i - 1]);
            s.tb_pos[w] = (int16_t)((j == nj) ? -1 : j - 1);
            i = ni;
            j = nj;
        }
    }
    POA_SYNC();
    w = warp_bcast0(w);
    if (warp_bcast0(lost)) {
        st.status = ST_TRACEBACK_LOST;
        return cap;
    }
    return w;
}

/* ------------------------------------------------------------------------------------------
 * Phase 3: traceback  (sisd_alignment_engine.cpp:340-431)
 *   priority: diagonal over in-edges in order, vertical over in-edges in order, horizontal.
 *
 *   The score matrix lives in HBM and a step needs 3 dependent reads of it (row record ->
 *   predecessor list -> cells), ~600 steps per read: done naively that is ~2000 serial
 *   round-trips to memory per read.  Instead the path is followed through a TILE: the TB_ROWS rows
 *   below the current cell x TB_COLS columns left of it are fetched in ONE round of independent
 *   asynchronous copies (lane l fetches rows i-l, i-l-32: record, CSR offset, 16-byte score chunks) into
 *   on-chip scratch (shared memory on the device), and ~30 steps are then resolved from the tile.
 *   Predecessors of a step are tested by different lanes and the first match (spoa's priority) is
 *   taken by ballot.  The current cell value is carried along, never re-read.
 *   A step whose data is not in the tile (predecessor > 31 rows back, in-degree > 32) falls back
 *   to reading global memory directly.
 *   Output: tb_node/tb_pos filled back to front; returns the index of the first (leftmost) entry.
 * ---------------------------------------------------------------------------------------- */
#ifndef POA_TB_RPL
#define POA_TB_RPL 2
#endif
#ifndef POA_TB_CHUNKS
#define POA_TB_CHUNKS 4
#endif
constexpr int TB_RPL = POA_TB_RPL;       /* tile rows loaded per lane */
constexpr int TB_ROWS = 32 * TB_RPL;     /* tile rows */
constexpr int TB_CHUNKS = POA_TB_CHUNKS; /* tile columns in 8-cell chunks */
constexpr int TB_COLS = TB_CHUNKS * 8;
constexpr int TB_PRED_CAP = 192 * TB_RPL; /* predecessor entries a tile can hold */
constexpr int TB_EDGE_MARGIN = 24;        /* adaptive band: a tile anchored this close to a band edge asks for a wider band */

struct TbScratch {           /* device: shared memory (the fill's ring area); emulation: heap */
    int16_t* cells;          /* [TB_ROWS * TB_COLS]  row (r_hi - k) at k*TB_COLS, column c at c - c_lo */
    uint32_t* rec;           /* [TB_ROWS]   row records                                 */
    uint32_t* poff;          /* [TB_ROWS+1] poff[k] = CSR offset of row (r_hi - k); poff[TB_ROWS] unused */
    uint32_t* pred;          /* [TB_PRED_CAP] predecessor entries of the rows, per row at poff - pred_base */
    uint16_t* node;          /* [TB_ROWS]   node id of row (r_hi - k)                   */
    uint8_t* readc;          /* [TB_COLS + 8] read base under column c at c - c_lo (column c <-> read[c-1]) */
};
/* also the capacity mark_subgraph gets for its root array (process_window) and part of the launch's shared memory: it
 * sets the graph size above which partial-span layers take the lane-0 path (DESIGN §4) */
constexpr int TB_SCRATCH_BYTES = TB_ROWS * TB_COLS * 2 + TB_ROWS * 4 + (TB_ROWS + 1) * 4 + TB_PRED_CAP * 4 + TB_ROWS * 2 + TB_COLS + 8 + 28 +
                                 TB_ROWS * 4 + 32 * 4 + 4 + 16;

constexpr int TB_OFF_REC = TB_ROWS * TB_COLS * 2;          /* byte offsets of the parts, see tb_bind() */
constexpr int TB_OFF_POFF = TB_OFF_REC + TB_ROWS * 4;
constexpr int TB_OFF_PRED = TB_OFF_POFF + (TB_ROWS + 1) * 4;
constexpr int TB_OFF_NODE = TB_OFF_PRED + TB_PRED_CAP * 4;
constexpr int TB_OFF_READC = TB_OFF_NODE + TB_ROWS * 2;
constexpr int TB_OFF_INFO = (TB_OFF_READC + TB_COLS + 8 + 3) & ~3; /* [TB_ROWS] u32: node id | predecessor tile row | letter */
constexpr int TB_OFF_OUT = TB_OFF_INFO + TB_ROWS * 4;              /* [32] u32: buffered alignment entries */

struct alignas(16) Vec16 { /* 8 int16 cells moved as one 128-bit access */
    uint32_t x, y, z, w;
};
POA_FN void copy8(int16_t* dst, const int16_t* src) { *reinterpret_cast<Vec16*>(dst) = *reinterpret_cast<const Vec16*>(src); }
POA_FN void fill8(int16_t* dst, int32_t v) {
    const uint32_t pk = ((uint32_t)v & 0xFFFFu) | ((uint32_t)v << 16);
    Vec16 q;
    q.x = q.y = q.z = q.w = pk;
    *reinterpret_cast<Vec16*>(dst) = q;
}

/* Reads of the tile on the serial path: real shared-memory loads on the device (the tile pointers are
 * generic; a generic load pays the address-space resolution on every step of the dependent chain). */
#if POA_DEVICE
/* The tile lives at a fixed offset of the block's dynamic shared memory (the kernel binds TbScratch there) and is read
 * with plain loads from the __shared__ array: the compiler then knows the address space (LDS, no generic resolution)
 * AND that a load from a warp-uniform address yields a warp-uniform value -- an inline-asm ld.shared would hide both,
 * and every step of the walk would have to launder what it read (poa_simt.cuh). */
constexpr uint32_t POA_TB_SMEM_OFFSET = 32;
extern __shared__ __align__(16) unsigned char poa_smem[];
typedef uint32_t tile_addr; /* byte offset into poa_smem */
POA_FN tile_addr tile_base(void*) { return POA_TB_SMEM_OFFSET; }
POA_FN uint32_t tile_u32(tile_addr a, int32_t i) { return *reinterpret_cast<const uint32_t*>(poa_smem + a + 4u * (uint32_t)i); }
POA_FN int32_t tile_s16(tile_addr a, int32_t i) { return *reinterpret_cast<const int16_t*>(poa_smem + a + 2u * (uint32_t)i); }
POA_FN uint32_t tile_u16(tile_addr a, int32_t i) { return *reinterpret_cast<const uint16_t*>(poa_smem + a + 2u * (uint32_t)i); }
POA_FN uint32_t tile_u8(tile_addr a, int32_t i) { return poa_smem[a + (uint32_t)i]; }
POA_FN uint32_t tile_sa(tile_addr a) { return (uint32_t)__cvta_generic_to_shared(poa_smem) + a; } /* shared-window address */
/* asynchronous global -> shared copies used by the tile load (LDGSTS: no register staging, all in flight);
 * destinations are shared-window addresses, like every other access to the tile.  The copies carry no L2 cache hint:
 * for sm_90a, ptxas 12.9 turns the hinted form into LDGSTS instructions whose shared-address base and memory descriptor
 * are uniform registers nothing writes, and the kernel dies with an illegal instruction at the first tile load
 * (tests/test_codegen.py checks every LDGSTS descriptor is written). */
POA_FN void tile_copy16(tile_addr a, int32_t byte_off, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(tile_sa(a) + (uint32_t)byte_off), "l"(src) : "memory");
}
POA_FN void tile_copy4(tile_addr a, int32_t i, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(tile_sa(a) + 4u * (uint32_t)i), "l"(src) : "memory");
}
POA_FN void tile_copy_wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }
POA_FN void tile_st_u32(tile_addr a, int32_t i, uint32_t v) { *reinterpret_cast<uint32_t*>(poa_smem + a + 4u * (uint32_t)i) = v; }
POA_FN void tile_st_u16(tile_addr a, int32_t i, uint32_t v) { *reinterpret_cast<uint16_t*>(poa_smem + a + 2u * (uint32_t)i) = (uint16_t)v; }
POA_FN void tile_st_u8(tile_addr a, int32_t i, uint32_t v) { poa_smem[a + (uint32_t)i] = (unsigned char)v; }
POA_FN void tile_fill8(tile_addr a, int32_t byte_off, int32_t v) { /* 8 int16 cells */
    const uint32_t pk = ((uint32_t)v & 0xFFFFu) | ((uint32_t)v << 16);
    *reinterpret_cast<uint4*>(poa_smem + a + (uint32_t)byte_off) = make_uint4(pk, pk, pk, pk);
}
#else
typedef uint8_t* tile_addr;
POA_FN tile_addr tile_base(void* p) { return reinterpret_cast<uint8_t*>(p); }
POA_FN void tile_copy16(tile_addr a, int32_t byte_off, const void* src) { *reinterpret_cast<Vec16*>(a + byte_off) = *reinterpret_cast<const Vec16*>(src); }
POA_FN void tile_copy4(tile_addr a, int32_t i, const void* src) { reinterpret_cast<uint32_t*>(a)[i] = *reinterpret_cast<const uint32_t*>(src); }
POA_FN void tile_copy_wait() {}
POA_FN void tile_st_u32(tile_addr a, int32_t i, uint32_t v) { reinterpret_cast<uint32_t*>(a)[i] = v; }
POA_FN void tile_st_u16(tile_addr a, int32_t i, uint32_t v) { reinterpret_cast<uint16_t*>(a)[i] = (uint16_t)v; }
POA_FN void tile_st_u8(tile_addr a, int32_t i, uint32_t v) { a[i] = (uint8_t)v; }
POA_FN void tile_fill8(tile_addr a, int32_t byte_off, int32_t v) { fill8(reinterpret_cast<int16_t*>(a + byte_off), v); }
POA_FN uint32_t tile_u32(tile_addr a, int32_t i) { return reinterpret_cast<const uint32_t*>(a)[i]; }
POA_FN int32_t tile_s16(tile_addr a, int32_t i) { return reinterpret_cast<const int16_t*>(a)[i]; }
POA_FN uint32_t tile_u16(tile_addr a, int32_t i) { return reinterpret_cast<const uint16_t*>(a)[i]; }
POA_FN uint32_t tile_u8(tile_addr a, int32_t i) { return a[i]; }
#endif

/* Reach report of the emulation (POA_TB_REACH_IF): does the step at (i, j) read a tile chunk the load filled with NEG,
 * i.e. a cell of row i at j - 1 or of a predecessor at j or j - 1 outside that row's band?  (Band starts and the tile's
 * chunks are 8-aligned: a chunk lies wholly inside its row's band or wholly outside.) */
POA_FN bool tb_out_of_band(const ReadGeom& g, int32_t row, int32_t col) {
    const int32_t o = col - band_start(g, row, g.n_rows);
    return g.banded && col >= 0 && (o < 0 || o >= g.bw);
}
POA_FN bool tb_step_reads_neg_chunk(const ReadGeom& g, const uint32_t* row_poff, const uint32_t* row_pred, int32_t i,
                                    int32_t j, int32_t np) {
    bool neg = j > 0 && tb_out_of_band(g, i, j - 1);
    for (int32_t k = 0; k < np; ++k) {
        const int32_t pi = (int32_t)(row_pred[row_poff[i] + k] & 0xFFFFu);
        neg = neg || tb_out_of_band(g, pi, j) || (j > 0 && tb_out_of_band(g, pi, j - 1));
    }
    return neg;
}

POA_FN void tb_bind(TbScratch& t, uint8_t* base) {
    t.cells = reinterpret_cast<int16_t*>(base);
    base += TB_ROWS * TB_COLS * 2;
    t.rec = reinterpret_cast<uint32_t*>(base);
    base += TB_ROWS * 4;
    t.poff = reinterpret_cast<uint32_t*>(base);
    base += (TB_ROWS + 1) * 4;
    t.pred = reinterpret_cast<uint32_t*>(base);
    base += TB_PRED_CAP * 4;
    t.node = reinterpret_cast<uint16_t*>(base);
    base += TB_ROWS * 2;
    t.readc = base;
}

POA_FN_NOINLINE int32_t traceback(const Slot& s, const Params p, WinState& st, const ReadGeom g,
                         const uint8_t* read, int32_t end_row, const TbScratch& t, const uint16_t* row_node) {
    /* everything the loop touches is copied into locals first: `s`, `t`, `p`, `g` are references into
     * memory, and after each store the compiler would otherwise reload every pointer it needs */
    const Params pu = p;
    const int32_t cap = pu.max_nodes + pu.max_len + 2;
    end_row = poa_uniform(end_row);
    int16_t* const tb_node = s.tb_node;
    int16_t* const tb_pos = s.tb_pos;
    const uint32_t* const row_rec = s.row_rec;
    const uint32_t* const row_poff = s.row_poff;
    const uint32_t* const row_pred = s.row_pred;
    const uint16_t* const node_at = row_node; /* rank -> node of THIS alignment's rows (graph or subgraph) */
    const int16_t* const S = s.S;
    const ReadGeom gg = geom_uniform(g);
    const int32_t stride = pu.stride, gap = pu.gap, bw = gg.bw, rlen = gg.len;
    /* the tile is addressed from ONE base (shared-window address on the device); its parts sit at constant offsets */
    const tile_addr A_cells = tile_base(t.cells);
    const tile_addr A_rec = A_cells + TB_OFF_REC, A_poff = A_cells + TB_OFF_POFF, A_pred = A_cells + TB_OFF_PRED,
                    A_node = A_cells + TB_OFF_NODE, A_readc = A_cells + TB_OFF_READC, A_info = A_cells + TB_OFF_INFO,
                    A_out = A_cells + TB_OFF_OUT;
    POA_SUB_BEGIN();
    int32_t w = cap; /* write cursor (uniform) */
    int32_t i = end_row, j = rlen; /* both laundered above */
    const int32_t mg = pu.match - gap, xg = pu.mismatch - gap;
    int32_t cur = poa_uniform(score_at(s, p, g, i, j)); /* read through generic pointers: launder once */
    /* tile state (uniform) */
    int32_t r_hi = -1, r_lo = 0, c_lo = 0, c_hi = -1, pred_base = 0, pred_n = 0;
    /* alignment entries (node | read position) are collected in the tile and written out 32 at a time, coalesced:
     * entry b of the buffer belongs to index w + nb - 1 - b */
    int32_t nb = 0;
#define POA_TB_FLUSH()                                                                  \
    do {                                                                                \
        POA_SYNC();                                                                     \
        POA_LANES(l) {                                                                  \
            if (l < nb) {                                                               \
                const uint32_t e = tile_u32(A_out, l);                                  \
                tb_node[w + nb - 1 - l] = (int16_t)(e & 0xFFFFu);                       \
                tb_pos[w + nb - 1 - l] = (int16_t)(e >> 16);                            \
            }                                                                           \
        }                                                                               \
        POA_SYNC();                                                                     \
        nb = 0;                                                                         \
    } while (0)
    int32_t lost = 0; /* the band did not contain a consistent path: decided by a vote at the end of the step, so that
                         the function is never left from lane-dependent control flow (poa_simt.cuh) */
    while (!(i == 0 && j == 0)) {
        if (w <= 32) { /* every step consumes one entry: a path longer than nodes + read length is lost */
            st.status = ST_TRACEBACK_LOST;
            return cap;
        }
        if (i == 0) { /* first row: S[0][*] == 0, only horizontal moves are left */
            POA_TB_REACH_IF(j >= 32, row0_tail32);
            POA_TB_REACH_IF(j >= 64, row0_tail64);
            POA_TB_FLUSH();
            for (int32_t b = 0; b < j; b += 32) {
                POA_LANES(l) {
                    const int32_t jj = j - b - l;
                    if (jj >= 1 && w - 1 - b - l >= 0) {
                        tb_node[w - 1 - b - l] = -1;
                        tb_pos[w - 1 - b - l] = (int16_t)(jj - 1);
                    }
                }
            }
            w -= j;
            j = 0;
            if (w < 0) {
                st.status = ST_TRACEBACK_LOST;
                return cap;
            }
            break;
        }
        /* ---- make sure row i and columns j-1..j are in the tile ---- */
        bool reloaded = false;
        if (i > r_hi || i < r_lo || j > c_hi || (j > 0 && j - 1 < c_lo)) {
            POA_SUB_LAP(11);
            POA_TB_REACH(tile_loads);
            r_hi = i;
            r_lo = i - (TB_ROWS - 1) < 0 ? 0 : i - (TB_ROWS - 1);
            c_hi = j;
            c_lo = ((j + 1 - TB_COLS) < 0 ? 0 : (j + 1 - TB_COLS + 7)) & ~7; /* 8-aligned, covers j */
            if (gg.banded && pu.adaptive) { /* adaptive band: is the path (sampled once per tile) about to leave the band? */
                const int32_t bs_i = band_start(gg, i, gg.n_rows);
                if ((bs_i > 0 && j - bs_i < TB_EDGE_MARGIN) || (bs_i + bw < gg.colsP && bs_i + bw - 1 - j < TB_EDGE_MARGIN)) {
                    st.band_hit = 1;
                    POA_TB_REACH(band_hits);
                }
            }
            POA_SYNC();
            /* ONE round of independent loads.  The band start of a row is recomputed (same formula as the
             * row program) instead of read from its record, so the score chunks -- the loads that go to HBM --
             * depend on nothing; they are asynchronous global->shared copies, no registers in between.  Only
             * the predecessor entries need a second, short level (two CSR offsets, cache-resident). */
            const int32_t lo_row = r_lo < 1 ? 1 : r_lo;
            const int32_t p_lo = (int32_t)row_poff[lo_row];                           /* uniform loads (i >= 1 here) */
            const int32_t p_hi = (int32_t)row_poff[r_hi] + rec_npred(row_rec[r_hi]);
            POA_LANES(l) {
#pragma unroll
                for (int32_t rr = 0; rr < TB_RPL; ++rr) {
                    const int32_t k = l + 32 * rr;
                    const int32_t row = r_hi - k;
                    if (row < r_lo) continue;
                    const int32_t bs = band_start(gg, row, gg.n_rows);
#pragma unroll
                    for (int32_t q = 0; q < TB_CHUNKS; ++q) {
                        const int32_t o = c_lo + 8 * q - bs; /* 8-aligned both: whole chunk in the band or out */
                        const int32_t dst = (k * TB_COLS + 8 * q) * 2; /* byte offset in the tile */
                        if (o >= 0 && o + 8 <= bw) tile_copy16(A_cells, dst, S + (size_t)row * stride + o);
                        else tile_fill8(A_cells, dst, NEG);
                    }
                    if (row >= 1) {
                        tile_copy4(A_rec, k, row_rec + row);
                        tile_copy4(A_poff, k, row_poff + row);
                    } else {
                        tile_st_u32(A_rec, k, 0u);
                        tile_st_u32(A_poff, k, 0u);
                    }
                }
            }
            /* CSR entries of rows r_lo..r_hi are contiguous: [poff(r_lo'), poff(r_hi) + np(r_hi)) */
            pred_base = p_lo;
            pred_n = p_hi - p_lo;
            if (pred_n > TB_PRED_CAP) pred_n = TB_PRED_CAP; /* rows beyond the cap fall back to global */
            POA_LANES(l) {
                for (int32_t e = l; e < pred_n; e += 32) tile_copy4(A_pred, e, row_pred + pred_base + e);
            }
            /* the two items that pass through registers (a 2-byte node id per row, the read bases under the tile) come
             * last: their round trip overlaps the asynchronous copies already in flight instead of delaying them */
            POA_LANES(l) {
                uint32_t nd[TB_RPL];
#pragma unroll
                for (int32_t rr = 0; rr < TB_RPL; ++rr) {
                    const int32_t row = r_hi - (l + 32 * rr);
                    nd[rr] = row >= 1 ? (uint32_t)node_at[row - 1] : 0u; /* rows below r_lo are never read */
                }
                uint32_t rb[(TB_COLS + 31) / 32];
#pragma unroll
                for (int32_t u = 0; u < (TB_COLS + 31) / 32; ++u) {
                    const int32_t c = c_lo + l + 32 * u;
                    rb[u] = (c >= 1 && c <= rlen) ? (uint32_t)read[c - 1] : 0u;
                }
#pragma unroll
                for (int32_t rr = 0; rr < TB_RPL; ++rr) tile_st_u16(A_node, l + 32 * rr, nd[rr]);
#pragma unroll
                for (int32_t u = 0; u < (TB_COLS + 31) / 32; ++u)
                    if (l + 32 * u < TB_COLS) tile_st_u8(A_readc, l + 32 * u, rb[u]);
            }
            tile_copy_wait();
            POA_SYNC();
            /* digest for the serial walk: a row with ONE in-edge whose source is in the tile takes the short step */
            POA_LANES(l) {
#pragma unroll
                for (int32_t rr = 0; rr < TB_RPL; ++rr) {
                    const int32_t k = l + 32 * rr;
                    const int32_t row = r_hi - k;
                    if (row < r_lo) continue;
                    const uint32_t rc = tile_u32(A_rec, k);
                    const int32_t q = (int32_t)tile_u32(A_poff, k) - pred_base;
                    uint32_t tp = 0xFFu;
                    if (row >= 1 && rec_npred(rc) == 1 && q < pred_n) {
                        const int32_t pi = (int32_t)(tile_u32(A_pred, q) & 0xFFFFu);
                        if (pi >= r_lo) tp = (uint32_t)(r_hi - pi);
                    }
                    tile_st_u32(A_info, k, (tile_u16(A_node, k) << 16) | (tp << 8) | (uint32_t)rec_code(rc));
                }
            }
            POA_SYNC();
            POA_SUB_LAP(12);
            reloaded = true;
        }
        /* ---- one step at (i, j) ---- */
        int32_t ni = i, nj = j, ncur = cur;
        const int32_t ti = r_hi - i; /* tile row index of row i */
        const uint32_t info = tile_u32(A_info, ti);
        const int32_t tp = (int32_t)((info >> 8) & 0xFFu);
        uint32_t node_i = info >> 16;
        if (tp != 0xFF) {
            /* the common row (one in-edge, source in the tile): warp-uniform scalar code on four tile reads */
            POA_TB_REACH(common_steps);
            POA_TB_REACH_IF(tb_step_reads_neg_chunk(gg, row_poff, row_pred, i, j, 1), neg_chunk_steps);
            const int32_t x = j - c_lo; /* >= 1 unless j == 0 */
            const int32_t cb = tp * TB_COLS + x;
            const int32_t vv = tile_s16(A_cells, cb);
            const int32_t vd = tile_s16(A_cells, j > 0 ? cb - 1 : cb);
            const int32_t vh = tile_s16(A_cells, j > 0 ? ti * TB_COLS + x - 1 : cb);
            const int32_t prof = (j > 0 && (int32_t)(info & 0xFFu) == (int32_t)tile_u8(A_readc, x)) ? mg : xg;
            if (j > 0 && vd + prof == cur) {
                ni = r_hi - tp;
                nj = j - 1;
                ncur = cur - prof;
            } else if (vv + gap == cur) {
                ni = r_hi - tp;
                ncur = cur - gap;
            } else if (j > 0 && vh == cur) {
                nj = j - 1;
            } else {
                lost = 1;
            }
        } else {
        const uint32_t rec = tile_u32(A_rec, ti);
        const int32_t np = rec_npred(rec);
        const int32_t po = (int32_t)tile_u32(A_poff, ti);
        const int32_t prof = (j > 0 && rec_code(rec) == (int32_t)tile_u8(A_readc, j - c_lo)) ? mg : xg;
        bool in_tile = poa_uniform_pred((np <= 32) && (po - pred_base + np <= pred_n));
        int32_t found = 0;
        if (in_tile) {
            /* every lane rates its predecessor; ONE warp-min picks spoa's choice:
             *   0 = predecessor below the tile, 1+l = diagonal via in-edge l, 64+l = vertical via in-edge l */
            PerLane<int> key, pr;
            POA_LANES(l) {
                key[l] = 255;
                pr[l] = 0;
                if (l < np) {
                    const int32_t pi = (int32_t)(tile_u32(A_pred, po - pred_base + l) & 0xFFFFu);
                    pr[l] = pi;
                    if (pi < r_lo) {
                        key[l] = 0;
                    } else {
                        const int32_t cb = (r_hi - pi) * TB_COLS - c_lo + j;
                        if (tile_s16(A_cells, cb) + gap == cur) key[l] = 64 + l;
                        if (j > 0 && tile_s16(A_cells, cb - 1) + prof == cur) key[l] = 1 + l;
                    }
                }
            }
            const int32_t best = warp_min(key);
            if (best == 0) {
                in_tile = false;
            } else if (best < 64) {
                ni = warp_get(pr, best - 1);
                nj = j - 1;
                ncur = cur - prof;
                found = 1;
            } else if (best < 128) {
                ni = warp_get(pr, best - 64);
                nj = j;
                ncur = cur - gap;
                found = 1;
            } else if (poa_uniform_pred(j > 0 && tile_s16(A_cells, ti * TB_COLS + (j - 1 - c_lo)) == cur)) {
                nj = j - 1;
                found = 1;
            } else {
                lost = 1;
                found = 1;
            }
        }
        if (in_tile) {
            POA_TB_REACH(tile_steps);
            POA_TB_REACH_IF(tb_step_reads_neg_chunk(gg, row_poff, row_pred, i, j, np), neg_chunk_steps);
        }
        if (!in_tile) {
            if (!reloaded) { /* a predecessor fell off the tile: re-anchor the tile at (i, j) and retry */
                POA_TB_REACH(reanchors);
                r_hi = -1;
                continue;
            }
            /* even a tile anchored here does not hold the step: read global memory directly */
            POA_TB_REACH_IF(np > 32, global_npred);
            POA_TB_REACH_IF(np <= 32 && po - pred_base + np > pred_n, global_pred_cap);
            POA_TB_REACH_IF(np <= 32 && po - pred_base + np <= pred_n, global_far);
            const int32_t gpo = (int32_t)row_poff[i];
            for (int pass = 0; pass < 2 && !found; ++pass) { /* pass 0: diagonal, pass 1: vertical */
                for (int32_t b = 0; b < np && !found; b += 32) {
                    PerLane<int> hit, pr;
                    POA_LANES(l) {
                        hit[l] = 0;
                        pr[l] = 0;
                        if (b + l < np) {
                            const uint32_t pe = row_pred[gpo + b + l];
                            const int32_t pi = (int32_t)(pe & 0xFFFFu);
                            const int32_t pbs = (int32_t)(pe >> 16);
                            pr[l] = pi;
                            hit[l] = pass == 0 ? ((j > 0) && (score_at_bs(s, p, g, pi, pbs, j - 1) + prof == cur))
                                               : (score_at_bs(s, p, g, pi, pbs, j) + gap == cur);
                        }
                    }
                    const unsigned m = warp_ballot(hit);
                    if (m) {
                        ni = warp_get(pr, poa_ffs(m));
                        nj = pass == 0 ? j - 1 : j;
                        ncur = pass == 0 ? cur - prof : cur - gap;
                        found = 1;
                    }
                }
            }
            if (!found) {
                if (j > 0 && score_at_bs(s, p, g, i, rec_bs(rec), j - 1) == cur) {
                    nj = j - 1;
                } else {
                    lost = 1;
                }
            }
        }
        ni = poa_uniform(ni); /* decided through shuffles in the general step: launder (the common step reads only
                                 warp-uniform tile words, which the compiler proves uniform on its own) */
        nj = poa_uniform(nj);
        } /* general step */
        if (poa_uniform_pred(lost != 0)) {
            st.status = ST_TRACEBACK_LOST;
            return cap;
        }
        --w;
        tile_st_u32(A_out, nb, ((i == ni) ? 0xFFFFu : node_i) | ((uint32_t)((j == nj) ? 0xFFFF : (j - 1)) << 16));
        ++nb;
        if (nb == 32) POA_TB_FLUSH();
        i = ni;
        j = nj;
        cur = ncur;
    }
    POA_TB_FLUSH();
#undef POA_TB_FLUSH
    POA_SYNC();
    return w;
}

/* ------------------------------------------------------------------------------------------
 * Phase 4: add the alignment to the graph  (graph.cpp:155-272, 94-116)
 * ---------------------------------------------------------------------------------------- */
POA_FN_NOINLINE void add_alignment_edges(const Slot& s_ref, const Params p_ref, WinState& st, const int8_t* wt,
                                         int32_t wconst, int32_t len);

POA_FN_NOINLINE void add_alignment(const Slot& s_ref, const Params p_ref, WinState& st, const uint8_t* read,
                          const int8_t* wt, int32_t wconst, int32_t len, int32_t tb_begin) {
    const Slot s = s_ref;     /* local copies: no reloads of the descriptor after every store */
    const Params p = p_ref;
    const int32_t cap = p.max_nodes + p.max_len + 2;
    len = poa_uniform(len);
    tb_begin = poa_uniform(tb_begin);
    wconst = poa_uniform(wconst);
    POA_SUB_BEGIN();
    const int32_t N0 = poa_uniform(st.n_nodes);

    /* (a) resolve every read position: existing node, or a new node (unaligned / aligned to x).
     *     asg[pos] >= 0 : existing node;  -1 : new, unaligned;  -2-x : new, aligned to node x.
     *     Two alignment entries per lane per step: their dependent loads overlap. */
    for (int32_t base = tb_begin; base < cap; base += 64) {
        POA_LANES(l) {
            const int32_t k0 = base + l, k1 = base + 32 + l;
            const int32_t pos0 = k0 < cap ? (int32_t)s.tb_pos[k0] : -1, pos1 = k1 < cap ? (int32_t)s.tb_pos[k1] : -1;
            const int32_t x0 = k0 < cap ? (int32_t)s.tb_node[k0] : -1, x1 = k1 < cap ? (int32_t)s.tb_node[k1] : -1;
            const uint8_t let0 = pos0 >= 0 ? read[pos0] : (uint8_t)0, let1 = pos1 >= 0 ? read[pos1] : (uint8_t)0;
            const uint8_t cx0 = x0 >= 0 ? s.code[x0] : (uint8_t)0, cx1 = x1 >= 0 ? s.code[x1] : (uint8_t)0;
            for (int32_t u = 0; u < 2; ++u) {
                const int32_t pos = u ? pos1 : pos0, x = u ? x1 : x0;
                const uint8_t letter = u ? let1 : let0, cx = u ? cx1 : cx0;
                if (pos < 0) continue;
                int32_t a;
                if (x < 0) {
                    a = -1;
                } else if (cx == letter) {
                    a = x;
                } else {
                    a = -2 - x;
                    const int32_t na = s.aln_cnt[x];
                    for (int32_t q = 0; q < na; ++q) {
                        const int32_t y = s.aln[x * KA + q];
                        if (s.code[y] == letter) {
                            a = y;
                            break;
                        }
                    }
                    POA_GRAPH_REACH_IF(a >= 0, clique_mate);
                }
                s.asg[pos] = a;
            }
        }
    }
    POA_SYNC();

    POA_SUB_LAP(2);
    /* (b) create the new nodes; ids follow read order exactly like the serial add_node calls. */
    int32_t n_new = 0;
    int32_t fail = 0;
    int32_t n_cols = poa_uniform(st.n_columns);
    for (int32_t base = 0; base < len; base += 32) {
        PerLane<int> isnew;
        POA_LANES(l) {
            const int32_t pos = base + l;
            isnew[l] = (pos < len && s.asg[pos] < 0) ? 1 : 0;
        }
        PerLane<int> off = isnew;
        const int32_t tot = warp_exscan(off);
        {   /* a new node that is aligned to nothing opens a new column of the graph */
            PerLane<int> opens;
            POA_LANES(l) { opens[l] = (isnew[l] && s.asg[base + l] == -1) ? 1 : 0; }
            n_cols += poa_popc(warp_ballot(opens));
        }
        if (N0 + n_new + tot > p.max_nodes) {
            fail = ST_NODE_COUNT_EXCEEDED;
            break;
        }
        PerLane<int> bad;
        POA_LANES(l) {
            bad[l] = 0;
            const int32_t pos = base + l;
            if (pos >= len || !isnew[l]) continue;
            const int32_t v = N0 + n_new + off[l];
            const int32_t a = s.asg[pos];
            s.code[v] = read[pos];
            s.nin[v] = 0;
            s.nout[v] = 0;
            s.in_head[v] = NONE16;
            s.in_tail[v] = NONE16;
            s.cov[v] = 0;
            s.aln_cnt[v] = 0;
            s.cnt[v] = 0;   /* v may become a root itself */
            s.need[v] = 0;
            s.dirty[v] = 0;
            s.lpos[v] = 0;
            s.root[v] = NONE16; /* resolved in (c) */
            if (a <= -2) {      /* graph.cpp:226-237: join x's clique */
                const int32_t x = -2 - a;
                const int32_t na = s.aln_cnt[x];
                if (na + 1 > KA) {
                    bad[l] = 1;
                } else {
                    POA_GRAPH_REACH_AT(join1, na);
                    for (int32_t q = 0; q < na; ++q) {
                        const int32_t y = s.aln[x * KA + q];
                        s.aln[v * KA + q] = (uint16_t)y;
                        s.aln[y * KA + s.aln_cnt[y]] = (uint16_t)v;
                        s.aln_cnt[y] = (uint8_t)(s.aln_cnt[y] + 1);
                    }
                    s.aln[v * KA + na] = (uint16_t)x;
                    s.aln_cnt[v] = (uint8_t)(na + 1);
                    s.aln[x * KA + na] = (uint16_t)v;
                    s.aln_cnt[x] = (uint8_t)(na + 1);
                    s.root[v] = s.root[x];
                }
            }
            s.asg[pos] = v | 0x40000000; /* mark "new" until (c) is done */
        }
        if (warp_ballot(bad)) {
            fail = ST_ALIGNED_COUNT_EXCEEDED;
            break;
        }
        n_new += tot;
    }
    POA_SYNC();
    if (fail) {
        st.status = fail;
        return;
    }
    POA_GRAPH_REACH_IF(n_new >= 32, new_nodes32);
    POA_GRAPH_REACH_IF(n_new >= 64, new_nodes64);

    POA_SUB_LAP(3);
    /* (c) roots of new unaligned nodes: root[v] = min(v, root[next node on the read path]); a run
     *     of consecutive new unaligned nodes all see the node that ends the run. */
    for (int32_t base = 0; base < len; base += 32) {
        POA_LANES(l) {
            const int32_t pos = base + l;
            if (pos >= len) continue;
            const int32_t a = s.asg[pos];
            if (!(a & 0x40000000)) continue;
            const int32_t v = a & 0x3FFFFFFF;
            if (s.root[v] != NONE16) continue; /* aligned new node: root copied from its clique */
            int32_t q = pos + 1;
            int32_t r = v;
            while (q < len) {
                const int32_t b = s.asg[q];
                const int32_t u = b & 0x3FFFFFFF;
                if ((b & 0x40000000) && s.root[u] == NONE16) { /* still inside the run */
                    ++q;
                    continue;
                }
                /* u is an old node, or a new aligned node whose root is already final */
                if ((int32_t)s.root[u] < r) r = s.root[u];
                break;
            }
            POA_GRAPH_REACH_IF((q >> 5) != (pos >> 5), run_cross32);
            s.roff[v] = (uint32_t)r; /* stage: root[] of run members is still NONE16 for the others */
        }
    }
    POA_SYNC();
    for (int32_t base = 0; base < len; base += 32) {
        POA_LANES(l) {
            const int32_t pos = base + l;
            if (pos >= len) continue;
            const int32_t a = s.asg[pos];
            if (!(a & 0x40000000)) continue;
            const int32_t v = a & 0x3FFFFFFF;
            if (s.root[v] == NONE16) s.root[v] = (uint16_t)s.roff[v];
            s.asg[pos] = v;
            /* bookkeeping of the per-root topological sort: one more member, DFS must be redone */
            poa_atomic_add(&s.cnt[s.root[v]], 1u);
            s.dirty[s.root[v]] = 1;
        }
    }
    POA_SYNC();
    st.n_nodes = N0 + n_new;
    st.n_columns = n_cols;

    POA_SUB_LAP(4);
    add_alignment_edges(s_ref, p_ref, st, wt, wconst, len);
}

/* (d) edges prev -> cur for consecutive read positions (graph.cpp:248-259, 94-116), and
 * (e) coverage: every node on the read's path carries this sequence's label.
 * A function of its own: ptxas proves the warp-uniformity of a function's control flow only while the function stays
 * small enough (see poa_simt.cuh); the node and the edge stage together were not. */
POA_FN_NOINLINE void add_alignment_edges(const Slot& s_ref, const Params p_ref, WinState& st, const int8_t* wt,
                                         int32_t wconst, int32_t len) {
    const Slot s = s_ref;
    const Params p = p_ref;
    len = poa_uniform(len);
    wconst = poa_uniform(wconst);
    int32_t fail = 0;
    POA_SUB_BEGIN();
    int32_t n_edges = poa_uniform(st.n_edges);
    /* DU read positions per lane per step (pos, pos + 32, ...): the walk over a node's in-edge list is a chain of
     * dependent loads to HBM; the DU walks of a lane are interleaved so that their round trips overlap.  New edge
     * ids follow read order (position = base + 32 u + lane: u-major), computed from ballots. */
#ifndef POA_ADD_DU
#define POA_ADD_DU 4
#endif
    constexpr int DU = POA_ADD_DU;
    POA_GRAPH_REACH_IF(len == 1, read_len1);
    POA_GRAPH_REACH_IF(wt == nullptr, const_weights);
    POA_GRAPH_REACH_IF(wt != nullptr, base_weights);
    POA_GRAPH_REACH_IF(wt == nullptr && wconst == 0, weight0);
    for (int32_t base = 0; base < len; base += 32 * DU) {
        POA_GRAPH_REACH_IF(base + 32 * (DU - 1) < len, du_all);
        PerLane<int> hit[DU], need[DU];
        POA_LANES(l) {
            int32_t cur[DU], prev[DU], f[DU];
            uint16_t e[DU];
#pragma unroll
            for (int32_t u = 0; u < DU; ++u) {
                const int32_t pos = base + 32 * u + l;
                const bool in = pos < len;
                cur[u] = in ? s.asg[pos] : 0;
                prev[u] = (in && pos > 0) ? s.asg[pos - 1] : -1;
                f[u] = -1;
            }
            int32_t cv[DU];
#pragma unroll
            for (int32_t u = 0; u < DU; ++u) { /* loads before the stores, see below */
                const int32_t pos = base + 32 * u + l;
                const bool in = pos < len;
                cv[u] = (in && len >= 2) ? (int32_t)s.cov[cur[u]] : 0;
                e[u] = (in && pos > 0) ? s.in_head[cur[u]] : NONE16;
            }
#pragma unroll
            for (int32_t u = 0; u < DU; ++u)
                if (base + 32 * u + l < len && len >= 2) s.cov[cur[u]] = (uint16_t)(cv[u] + 1);
            for (;;) {
                bool any = false;
#pragma unroll
                for (int32_t u = 0; u < DU; ++u) any = any || e[u] != NONE16;
                if (!any) break;
                int32_t src[DU];
                uint16_t nx[DU];
#pragma unroll
                for (int32_t u = 0; u < DU; ++u) {
                    src[u] = e[u] != NONE16 ? (int32_t)s.e_src[e[u]] : -2;
                    nx[u] = e[u] != NONE16 ? s.e_next[e[u]] : NONE16;
                }
#pragma unroll
                for (int32_t u = 0; u < DU; ++u) {
                    if (src[u] == prev[u]) {
                        f[u] = e[u];
                        e[u] = NONE16;
                    } else {
                        e[u] = nx[u];
                    }
                }
            }
#pragma unroll
            for (int32_t u = 0; u < DU; ++u) {
                const int32_t pos = base + 32 * u + l;
                hit[u][l] = f[u];
                need[u][l] = (pos < len && pos > 0 && f[u] < 0) ? 1 : 0;
                POA_GRAPH_REACH_IF(pos < len && pos > 0 && (f[u] >= 0 ? s.e_ord[f[u]] >= 32 : s.nin[cur[u]] > 32),
                                   walk_over32);
            }
        }
        unsigned nmask[DU];
        int32_t first[DU], tot = 0;
#pragma unroll
        for (int32_t u = 0; u < DU; ++u) {
            nmask[u] = warp_ballot(need[u]);
            first[u] = tot;
            tot += poa_popc(nmask[u]);
        }
        if (n_edges + tot > poa_edge_capacity(p.max_nodes)) {
            fail = ST_EDGE_COUNT_EXCEEDED;
            break;
        }
        POA_LANES(l) {
            /* all loads of the DU positions first (their addresses do not depend on each other), then all the
             * stores: a load placed after a store to the same workspace could not be moved up by the compiler and
             * would cost a round trip of its own */
            int32_t cur[DU], prev[DU], w[DU], old_w[DU], nin_c[DU], tail_c[DU], nout_p[DU], root_c[DU], root_p[DU];
            bool act[DU];
#pragma unroll
            for (int32_t u = 0; u < DU; ++u) {
                const int32_t pos = base + 32 * u + l;
                act[u] = pos < len && pos != 0;
                cur[u] = act[u] ? s.asg[pos] : 0;
                prev[u] = act[u] ? s.asg[pos - 1] : 0;
                w[u] = act[u] ? (wt ? (int32_t)wt[pos - 1] + (int32_t)wt[pos] : 2 * wconst) : 0;
            }
#pragma unroll
            for (int32_t u = 0; u < DU; ++u) {
                const bool is_new = act[u] && hit[u][l] < 0;
                old_w[u] = (act[u] && !is_new) ? s.e_w[hit[u][l]] : 0;
                nin_c[u] = is_new ? (int32_t)s.nin[cur[u]] : 0;
                tail_c[u] = is_new ? (int32_t)s.in_tail[cur[u]] : 0;
                nout_p[u] = is_new ? (int32_t)s.nout[prev[u]] : 0;
                root_c[u] = is_new ? (int32_t)s.root[cur[u]] : 0;
                root_p[u] = is_new ? (int32_t)s.root[prev[u]] : 1;
            }
#pragma unroll
            for (int32_t u = 0; u < DU; ++u) {
                if (!act[u]) continue;
                const int32_t h = hit[u][l];
                POA_GRAPH_REACH_IF(wt != nullptr && wt[base + 32 * u + l] == 0, weight0);
                if (h >= 0) {
                    POA_GRAPH_REACH(edge_bumped);
                    s.e_w[h] = old_w[u] + w[u];
                } else {
                    POA_GRAPH_REACH(edge_created);
                    POA_GRAPH_REACH_IF(root_p[u] == root_c[u], edge_same_root);
                    POA_GRAPH_REACH_IF(root_p[u] != root_c[u], edge_cross_root);
                    const int32_t e = n_edges + first[u] + poa_popc(nmask[u] & ((1u << l) - 1u));
                    s.e_src[e] = (uint16_t)prev[u];
                    s.e_dst[e] = (uint16_t)cur[u];
                    s.e_next[e] = NONE16;
                    s.e_w[e] = w[u];
                    s.e_ord[e] = (uint8_t)(nin_c[u] < 255 ? nin_c[u] : 255);
                    if (tail_c[u] == NONE16) s.in_head[cur[u]] = (uint16_t)e;
                    else s.e_next[tail_c[u]] = (uint16_t)e;
                    s.in_tail[cur[u]] = (uint16_t)e;
                    s.nin[cur[u]] = (uint16_t)(nin_c[u] + 1);
                    s.nout[prev[u]] = (uint16_t)(nout_p[u] + 1);
                    if (root_p[u] == root_c[u]) s.dirty[root_c[u]] = 1;
                }
            }
        }
        n_edges += tot;
    }
    POA_SYNC();
    if (fail) {
        st.status = fail;
        return;
    }
    POA_SUB_LAP(5);
    st.n_edges = n_edges;
}

/* ------------------------------------------------------------------------------------------
 * Phase 5a: serial topological sort, the literal restatement of graph.cpp:294-354.
 * Kept for the test-suite (Params::serial_topsort) as the cross-check of the per-root sort.
 * ---------------------------------------------------------------------------------------- */
POA_FN_NOINLINE void topsort_serial(const Slot& s_ref, const Params p_ref, WinState& st) {
    const Slot s = s_ref;     /* local copies: no reloads of the descriptor after every store */
    const Params p = p_ref;
    const int32_t N = poa_uniform(st.n_nodes);
    for (int32_t base = 0; base < N; base += 32) {
        POA_LANES(l) {
            if (base + l < N) {
                s.marks[base + l] = 0;
                s.check[base + l] = 1;
            }
        }
    }
    POA_SYNC();
    POA_LANE0 {
        int32_t out = 0, sp = 0;
        for (int32_t i = 0; i < N; ++i) {
            if (s.marks[i] != 0) continue;
            s.stack[sp++] = (uint16_t)i;
            while (sp != 0) {
                const int32_t id = s.stack[sp - 1];
                bool valid = true;
                if (s.marks[id] != 2) {
                    for (uint16_t e = s.in_head[id]; e != NONE16; e = s.e_next[e]) {
                        const int32_t u = s.e_src[e];
                        if (s.marks[u] != 2) {
                            s.stack[sp++] = (uint16_t)u;
                            valid = false;
                        }
                    }
                    const int32_t na = s.aln_cnt[id];
                    if (s.check[id]) {
                        for (int32_t q = 0; q < na; ++q) {
                            const int32_t a = s.aln[id * KA + q];
                            if (s.marks[a] != 2) {
                                s.stack[sp++] = (uint16_t)a;
                                s.check[a] = 0;
                                valid = false;
                            }
                        }
                    }
                    if (valid) {
                        s.marks[id] = 2;
                        if (s.check[id]) {
                            s.node_at[out++] = (uint16_t)id;
                            for (int32_t q = 0; q < na; ++q) s.node_at[out++] = s.aln[id * KA + q];
                        }
                    } else {
                        s.marks[id] = 1;
                    }
                }
                if (valid) --sp;
            }
        }
    }
    POA_SYNC();
    for (int32_t base = 0; base < N; base += 32) {
        POA_LANES(l) {
            if (base + l < N) {
                const int32_t v = s.node_at[base + l];
                s.rank_of[v] = (uint16_t)(base + l);
                s.row_meta[base + l] = meta_make(s.code[v], s.nout[v] == 0, s.nin[v]);
            }
        }
    }
    POA_SYNC();
    (void)p;
}

/* ------------------------------------------------------------------------------------------
 * Phase 5b: per-root, incremental topological sort.
 *   spoa's outer loop visits ids in increasing order; the DFS started at i emits exactly the
 *   not-yet-emitted members of i's ancestor closure (in-edges + aligned cliques), i.e. the nodes
 *   with root[v] == i, and it only needs to know WHICH other nodes are already emitted
 *   (root[u] < i), not their order.  Hence rank(v) = (number of nodes with a smaller root) +
 *   (position of v inside DFS_root), and DFS_i only changes when root i gains a node or an
 *   internal edge -- add_alignment marks exactly those roots dirty.  Per read:
 *     1. nodes of dirty roots: reset DFS marks, accumulate the root's stack bound;
 *     2. prefix-sum the member counts over root ids and compact the dirty multi-node roots into a
 *        work list; then, 32 work items at a time, re-run spoa's DFS restricted to the root's own
 *        members and store each member's position (lpos);
 *     3. every node: rank = offset[root] + lpos.
 * ---------------------------------------------------------------------------------------- */
POA_FN_NOINLINE void topsort_roots(const Slot& s_ref, const Params p_ref, WinState& st) {
    const Slot s = s_ref;     /* local copies: no reloads of the descriptor after every store */
    const Params p = p_ref;
    POA_SUB_BEGIN();
    const int32_t N = poa_uniform(st.n_nodes);
    /* 1. members of dirty roots: reset DFS marks, accumulate the root's stack bound.  Four nodes per lane
     *    per step so that the dependent loads (root -> dirty -> in-degree) of all four are in flight together. */
    for (int32_t base = 0; base < N; base += 32 * TS_U) {
        POA_LANES(l) {
            int32_t r[TS_U], nn[TS_U];
            bool d[TS_U];
#pragma unroll
            for (int32_t u = 0; u < TS_U; ++u) {
                const int32_t v = base + 32 * u + l;
                r[u] = v < N ? (int32_t)s.root[v] : 0;
                nn[u] = v < N ? (int32_t)s.nin[v] + (int32_t)s.aln_cnt[v] + 1 : 0;
            }
#pragma unroll
            for (int32_t u = 0; u < TS_U; ++u) d[u] = (base + 32 * u + l < N) && s.dirty[r[u]];
#pragma unroll
            for (int32_t u = 0; u < TS_U; ++u) {
                const int32_t v = base + 32 * u + l;
                if (d[u]) {
                    s.marks[v] = 0;
                    s.check[v] = 1;
                    poa_atomic_add(&s.need[r[u]], (uint32_t)nn[u]);
                }
            }
        }
    }
    POA_SYNC();
    POA_SUB_LAP(6);
    /* 2a. offsets: prefix-sum the member counts over root ids (two ids per lane per step); collect the
     *     dirty multi-node roots into a compact work list (so that the DFS below keeps all lanes busy);
     *     need[] is consumed and zeroed for the next read. */
    int32_t out_run = 0, stk_run = 0, n_work = 0;
    for (int32_t base = 0; base < N; base += 64) {
        PerLane<int> ca, cb, na, nb, wa, wb;
        POA_LANES(l) {
            const int32_t i0 = base + 2 * l, i1 = i0 + 1;
            ca[l] = (i0 < N) ? (int)s.cnt[i0] : 0;
            cb[l] = (i1 < N) ? (int)s.cnt[i1] : 0;
            const int da = (i0 < N && ca[l] > 0) ? (int)s.dirty[i0] : 0;
            const int db = (i1 < N && cb[l] > 0) ? (int)s.dirty[i1] : 0;
            wa[l] = (da && ca[l] > 1) ? 1 : 0;
            wb[l] = (db && cb[l] > 1) ? 1 : 0;
            na[l] = wa[l] ? (int)s.need[i0] + 1 : 0;
            nb[l] = wb[l] ? (int)s.need[i1] + 1 : 0;
            if (da) {
                s.dirty[i0] = 0;
                s.need[i0] = 0;
                if (ca[l] == 1) s.lpos[i0] = 0;
            }
            if (db) {
                s.dirty[i1] = 0;
                s.need[i1] = 0;
                if (cb[l] == 1) s.lpos[i1] = 0;
            }
        }
        PerLane<int> oo, so, wo;
        POA_LANES(l) {
            oo[l] = ca[l] + cb[l];
            so[l] = na[l] + nb[l];
            wo[l] = wa[l] + wb[l];
        }
        const int32_t ctot = warp_exscan(oo);
        const int32_t stot = warp_exscan(so);
        const int32_t wtot = warp_exscan(wo);
        POA_LANES(l) {
            const int32_t i0 = base + 2 * l, i1 = i0 + 1;
            if (i0 < N) s.roff[i0] = (uint32_t)(out_run + oo[l]);
            if (i1 < N) s.roff[i1] = (uint32_t)(out_run + oo[l] + ca[l]);
            if (wa[l]) { /* work item: root id and where its DFS stack lives (c_score/c_pred are free here) */
                s.c_score[n_work + wo[l]] = i0;
                s.c_pred[n_work + wo[l]] = stk_run + so[l];
            }
            if (wb[l]) {
                s.c_score[n_work + wo[l] + wa[l]] = i1;
                s.c_pred[n_work + wo[l] + wa[l]] = stk_run + so[l] + na[l];
            }
        }
        out_run += ctot;
        stk_run += stot;
        n_work += wtot;
    }
    POA_SYNC();
    POA_SUB_LAP(7);
    POA_GRAPH_REACH_IF(n_work > 32, dirty_over32);
    /* 2b. spoa's DFS restricted to the members of each dirty root, 32 roots at a time */
    for (int32_t base = 0; base < n_work; base += 32) {
        POA_LANES(l) {
            if (base + l >= n_work) continue;
            const int32_t i = s.c_score[base + l];
            uint16_t* stk = s.stack + s.c_pred[base + l];
            int32_t sp = 0, out = 0;
            stk[sp++] = (uint16_t)i;
            while (sp != 0) {
                const int32_t id = stk[sp - 1];
                bool valid = true;
                if (s.marks[id] != 2) {
                    for (uint16_t e = s.in_head[id]; e != NONE16;) {
                        const uint16_t nx = s.e_next[e]; /* next link requested with the source, not after the stores below */
                        const int32_t u = s.e_src[e];
                        if ((int32_t)s.root[u] == i && s.marks[u] != 2) {
                            stk[sp++] = (uint16_t)u;
                            valid = false;
                        }
                        e = nx;
                    }
                    const int32_t na = s.aln_cnt[id];
                    if (s.check[id]) {
                        for (int32_t q = 0; q < na; ++q) {
                            const int32_t a = s.aln[id * KA + q];
                            if (s.marks[a] != 2) { /* clique mates always share the root */
                                stk[sp++] = (uint16_t)a;
                                s.check[a] = 0;
                                valid = false;
                            }
                        }
                    }
                    if (valid) {
                        s.marks[id] = 2;
                        if (s.check[id]) {
                            s.lpos[id] = (uint16_t)out++;
                            for (int32_t q = 0; q < na; ++q) s.lpos[s.aln[id * KA + q]] = (uint16_t)out++;
                        }
                    } else {
                        s.marks[id] = 1;
                    }
                }
                if (valid) --sp;
            }
        }
    }
    POA_SYNC();
    POA_SUB_LAP(8);
    /* 3. ranks (four nodes per lane per step, loads staged by dependency level).  The row program of the NEXT read wants,
     *    in rank order, each node's letter, in-degree and whether it is a sink: they are read here, where nodes are
     *    visited in id order (coalesced), and written by rank -- instead of gathered through node_at later. */
    for (int32_t base = 0; base < N; base += 32 * TS_U) {
        POA_LANES(l) {
            int32_t q[TS_U], lp[TS_U], r[TS_U];
            uint32_t meta[TS_U];
#pragma unroll
            for (int32_t k = 0; k < TS_U; ++k) {
                const int32_t v = base + 32 * k + l;
                q[k] = v < N ? (int32_t)s.root[v] : 0;
                lp[k] = v < N ? (int32_t)s.lpos[v] : 0;
                meta[k] = v < N ? meta_make(s.code[v], s.nout[v] == 0, s.nin[v]) : 0u;
            }
#pragma unroll
            for (int32_t k = 0; k < TS_U; ++k) r[k] = (int32_t)s.roff[q[k]] + lp[k];
#pragma unroll
            for (int32_t k = 0; k < TS_U; ++k) {
                const int32_t v = base + 32 * k + l;
                if (v < N) {
                    s.rank_of[v] = (uint16_t)r[k];
                    s.node_at[r[k]] = (uint16_t)v;
                    s.row_meta[r[k]] = meta[k];
                }
            }
        }
    }
    POA_SYNC();
    (void)p;
    POA_SUB_LAP(9);
}

/* ------------------------------------------------------------------------------------------
 * Consensus: heaviest bundle  (graph.cpp:494-542 traverse_heaviest_bundle, :544-589
 * branch_completion) and coverage (graph.cpp:447-453).  Writes the consensus FORWARD.
 * ---------------------------------------------------------------------------------------- */
POA_FN void consensus_scores_from(const Slot& s, int32_t N, int32_t first_rank, bool skip_dead,
                                  int32_t& max_id, int32_t& max_score, bool strict_init) {
    /* serial over ranks (lane 0) -- scores of predecessors must be final */
    for (int32_t r = first_rank; r < N; ++r) {
        const int32_t id = s.node_at[r];
        int32_t sc = -1, pd = -1;
        for (uint16_t e = s.in_head[id]; e != NONE16; e = s.e_next[e]) {
            const int32_t u = s.e_src[e];
            if (skip_dead && s.c_score[u] == -1) continue;
            const int32_t w = s.e_w[e];
            if (sc < w || (sc == w && s.c_score[pd] <= s.c_score[u])) {
                sc = w;
                pd = u;
            }
        }
        if (pd != -1) sc += s.c_score[pd];
        s.c_score[id] = sc;
        s.c_pred[id] = pd;
        if (strict_init) {
            if (s.c_score[max_id] < sc) max_id = id;
        } else if (max_score < sc) {
            max_score = sc;
            max_id = id;
        }
    }
}

/* The first, full scoring pass (graph.cpp:494-518), 32 ranks at a time.
 *   gather  (parallel): lane l walks the in-edges of the node at rank r0+l and finds its heaviest in-edge.  Only a
 *           TIE between equal weights needs predecessor scores to be decided (graph.cpp:505-509); the score of
 *           a predecessor ranked before this block is final and fetched here.
 *   resolve (serial over the 32 lanes, but on registers): score = weight + score[pred]; a predecessor inside
 *           the block is read from its lane by shuffle.  Tied nodes redo the literal walk against memory.
 * max_id follows the serial rule "first strictly larger score wins" (scores[max_score_id] < scores[id]). */
POA_FN void consensus_scores_full(const Slot& s, int32_t N, int32_t& max_id_out) {
    int32_t max_id = 0, max_sc = -1; /* scores[] starts at -1 everywhere */
    for (int32_t r0 = 0; r0 < N; r0 += 32) {
        PerLane<int> id, w, pd, prank, pre, tie, score;
        POA_LANES(l) {
            const int32_t r = r0 + l;
            id[l] = 0;
            w[l] = -1;
            pd[l] = -1;
            prank[l] = -1;
            pre[l] = 0;
            tie[l] = 0;
            score[l] = -1;
            if (r < N) {
                const int32_t v = s.node_at[r];
                id[l] = v;
                int32_t sc = -1, best = -1, t = 0;
                for (uint16_t e = s.in_head[v]; e != NONE16; e = s.e_next[e]) {
                    const int32_t ww = s.e_w[e];
                    if (sc < ww) {
                        sc = ww;
                        best = s.e_src[e];
                        t = 0;
                    } else if (sc == ww) {
                        t = 1;
                    }
                }
                w[l] = sc;
                pd[l] = best;
                tie[l] = t;
                if (best >= 0) {
                    const int32_t pr = s.rank_of[best];
                    prank[l] = pr;
                    if (pr < r0) pre[l] = s.c_score[best];
                }
            }
        }
        const int32_t cnt = N - r0 < 32 ? N - r0 : 32;
        const unsigned ties = warp_ballot(tie);
        for (int32_t k = 0; k < cnt; ++k) {
            if ((ties >> k) & 1u) { /* rare: the literal rule, predecessor scores from memory */
                POA_SYNC();
                POA_LANES(l) {
                    if (l != k) continue;
                    const int32_t v = id[l];
                    int32_t sc = -1, best = -1;
                    for (uint16_t e = s.in_head[v]; e != NONE16; e = s.e_next[e]) {
                        const int32_t u = s.e_src[e];
                        const int32_t ww = s.e_w[e];
                        if (sc < ww || (sc == ww && s.c_score[best] <= s.c_score[u])) {
                            POA_GRAPH_REACH_IF(sc == ww && s.c_score[best] == s.c_score[u], tie_equal_pred);
                            sc = ww;
                            best = u;
                        }
                    }
                    POA_GRAPH_REACH_IF(best != -1 && (int32_t)s.rank_of[best] >= r0, tie_in_block);
                    POA_GRAPH_REACH_IF(best != -1 && (int32_t)s.rank_of[best] < r0, tie_pre_block);
                    if (best != -1) sc += s.c_score[best];
                    score[l] = sc;
                    s.c_score[v] = sc;
                    s.c_pred[v] = best;
                }
                POA_SYNC();
                continue;
            }
            const int32_t pk = warp_get(prank, k);
            const int32_t from_lane = warp_get(score, pk >= r0 ? pk - r0 : 0);
            POA_LANES(l) {
                if (l != k) continue;
                int32_t sc = w[l];
                if (pd[l] != -1) sc += (pk >= r0) ? from_lane : pre[l];
                score[l] = sc;
                s.c_score[id[l]] = sc;
                s.c_pred[id[l]] = pd[l];
            }
        }
        POA_SYNC(); /* this block's scores are in memory before the next block gathers */
        PerLane<int> sv;
        POA_LANES(l) { sv[l] = l < cnt ? score[l] : -2; }
        const int32_t m = warp_max(sv);
        if (m > max_sc) {
            PerLane<int> is;
            POA_LANES(l) { is[l] = (l < cnt && score[l] == m) ? 1 : 0; }
            POA_GRAPH_REACH_IF(poa_popc(warp_ballot(is)) > 1, block_max_tie);
            max_id = warp_get(id, poa_ffs(warp_ballot(is)));
            max_sc = m;
        } else {
            POA_GRAPH_REACH_IF(m == max_sc, max_tie_across);
        }
    }
    max_id_out = max_id;
}

#if POA_GRAPH_DIGEST
POA_FN_NOINLINE unsigned long long cons_digest(const Slot& s_ref, int32_t N, int32_t max_id);
#endif

POA_FN_NOINLINE void generate_consensus(const Slot& s_ref, const Params p_ref, WinState& st, const WindowOut& out_ref) {
    const Slot s = s_ref;     /* local copies: no reloads of the descriptor after every store */
    const Params p = p_ref;
    WindowOut out = out_ref;
    out.trim_nseq = poa_uniform(out.trim_nseq);
    const int32_t N = poa_uniform(st.n_nodes);
    const int32_t n_edges_total = poa_uniform(st.n_edges);
    POA_SUB_BEGIN();
    int32_t n = 0;
    int32_t max_id_full = 0;
    consensus_scores_full(s, N, max_id_full);
    POA_GRAPH_TWIN(consensus, s, N, max_id_full);
#if POA_GRAPH_DIGEST
    int32_t max_id_last = 0, rounds = 0;
    {
        const unsigned long long d = cons_digest(s, N, max_id_full);
        POA_LANE0 { out.cons_digest[0] = d; }
        POA_SYNC();
    }
#endif
    POA_LANE0 {
        int32_t max_id = max_id_full;
        POA_SUB_LAP(13);
        int32_t guard = N + 1;
        while (s.nout[max_id] != 0 && guard-- > 0) { /* graph.cpp:520-530 */
#if POA_GRAPH_DIGEST
            ++rounds;
#endif
            const int32_t node_id = max_id;
            const int32_t rank = s.rank_of[node_id];
            /* invalidate the other sources of every out-neighbour (graph.cpp:547-554) */
            for (int32_t e = 0; e < n_edges_total; ++e) {
                if (s.e_src[e] != node_id) continue;
                const int32_t d = s.e_dst[e];
                for (uint16_t f = s.in_head[d]; f != NONE16; f = s.e_next[f])
                    if (s.e_src[f] != node_id) s.c_score[s.e_src[f]] = -1;
            }
            int32_t ms = 0;
            max_id = 0;
            consensus_scores_from(s, N, rank + 1, true, max_id, ms, false);
        }
        POA_SUB_LAP(14);
#if POA_GRAPH_DIGEST
        max_id_last = max_id;
#endif
        /* backtrack into the stack as scratch (path reversed); emitted forward below */
        int32_t v = max_id;
        while (s.c_pred[v] != -1 && n < N) {
            s.stack[n++] = (uint16_t)v;
            v = s.c_pred[v];
        }
        s.stack[n++] = (uint16_t)v;
    }
    POA_SYNC();
    n = warp_bcast0(n);
#if POA_GRAPH_DIGEST
    {
        const unsigned long long d = cons_digest(s, N, warp_bcast0(max_id_last));
        rounds = warp_bcast0(rounds);
        POA_LANE0 {
            out.cons_digest[1] = d;
            *out.cons_rounds = rounds;
        }
        POA_SYNC();
    }
#endif
    if (n > p.max_cons) {
        st.status = ST_GENERIC_ERROR;
        return;
    }
    /* one bump allocation in the compact output arenas (16-element granules keep every window 16-byte aligned) */
    int32_t off = 0;
    POA_LANE0 { off = (int32_t)poa_bump(out.cursor, ((uint32_t)n + 15u) & ~15u); }
    off = warp_bcast0(off);
    /* emit forward, 32 bases per step, and find the span racon's TGS trim keeps (window.cpp:118-139) */
    const int32_t avg = (out.trim_nseq - 1) / 2;
    int32_t first = n, last = -1;
    for (int32_t base = 0; base < n; base += 32) {
        PerLane<int> ok;
        POA_LANES(l) {
            const int32_t k = base + l;
            ok[l] = 0;
            if (k < n) {
                const int32_t id = s.stack[n - 1 - k];
                int32_t c = s.cov[id];
                const int32_t na = s.aln_cnt[id];
                for (int32_t q = 0; q < na; ++q) c += s.cov[s.aln[id * KA + q]];
                out.cons[off + k] = s.code[id];
                out.cov[off + k] = (uint16_t)c;
                ok[l] = c >= avg ? 1 : 0;
            }
        }
        const unsigned m = warp_ballot(ok);
        if (m) {
            if (first == n) first = base + poa_ffs(m);
            last = base + poa_fls(m);
        }
    }
    POA_SUB_LAP(15);
    POA_LANE0 {
        *out.len = n;
        *out.off = off;
        *out.trim = (int32_t)(((uint32_t)(last & 0xFFFF) << 16) | (uint32_t)(first & 0xFFFF)); /* last < 0 reads back as -1 */
    }
    POA_SYNC();
}

/* ------------------------------------------------------------------------------------------
 * Multiple sequence alignment  (spoa: graph.cpp:373-427 generate_multiple_sequence_alignment; cudapoa:
 * cudapoa_generate_msa.cuh:35-233 getNodeIDToMSAPosDevice / generateMSADevice / generateMSAKernel, one thread per
 * sequence walking labelled out-edges).  Here a sequence's path is simply the node each of its bases was assigned to
 * (add_alignment's asg[], kept in WindowView::path), so a row is one parallel scatter.
 * ---------------------------------------------------------------------------------------- */
/* after add_alignment: asg[pos] is the node of read position pos (identity: the backbone chain, node k = base k) */
POA_FN_NOINLINE void record_path(const int32_t* asg, uint16_t* path, int32_t len, int32_t identity) {
    len = poa_uniform(len);
    identity = poa_uniform(identity);
    for (int32_t base = 0; base < len; base += 32) {
        POA_LANES(l) {
            const int32_t pos = base + l;
            if (pos < len) path[pos] = (uint16_t)(identity ? pos : asg[pos]);
        }
    }
    POA_SYNC();
}

POA_FN void poa_store16_dash(uint8_t* dst) { /* 16 '-' at a 16-byte aligned address */
#if POA_DEVICE
    *reinterpret_cast<uint4*>(dst) = make_uint4(0x2D2D2D2Du, 0x2D2D2D2Du, 0x2D2D2D2Du, 0x2D2D2D2Du);
#else
    for (int k = 0; k < 16; ++k) dst[k] = (uint8_t)'-';
#endif
}

POA_FN_NOINLINE void generate_msa(const Slot& s_ref, const Params p_ref, int32_t n_nodes, const WindowView& wv_ref,
                                  const MsaOut& out_ref) {
    const Slot s = s_ref;
    const Params p = p_ref;
    const WindowView wv = wv_ref;
    const MsaOut out = out_ref;
    const int32_t N = poa_uniform(n_nodes);
    const int32_t n_seqs = poa_uniform(wv.n_seqs);
    /* 1. column of every node (graph.cpp:373-389): a node and its aligned nodes share a column, columns follow the
     *    topological order, and the sort emits a clique as one run of ranks (graph.cpp:334-341) -- so rank r opens a
     *    column iff no clique mate ranks before it, and column(r) = (#openers among ranks <= r) - 1.  c_score[] is free. */
    int32_t run = 0;
    for (int32_t base = 0; base < N; base += 32) {
        PerLane<int> opens, node;
        POA_LANES(l) {
            const int32_t r = base + l;
            opens[l] = 0;
            node[l] = 0;
            if (r < N) {
                const int32_t v = s.node_at[r];
                node[l] = v;
                int32_t first = r;
                const int32_t na = s.aln_cnt[v];
                for (int32_t q = 0; q < na; ++q) {
                    const int32_t rr = s.rank_of[s.aln[v * KA + q]];
                    if (rr < first) first = rr;
                }
                opens[l] = first == r ? 1 : 0;
            }
        }
        PerLane<int> before = opens;
        const int32_t tot = warp_exscan(before);
        POA_LANES(l) {
            if (base + l < N) s.c_score[node[l]] = run + before[l] + opens[l] - 1;
        }
        run += tot;
    }
    POA_SYNC();
    const int32_t cols = run;
    if (cols >= p.max_cons) { /* cudapoa_generate_msa.cuh:203-208: the MSA does not fit max_consensus_size */
        POA_LANE0 {
            *out.status = ST_EXCEEDED_MAX_SEQ_SIZE;
            *out.cols = 0;
            *out.off = 0;
        }
        POA_SYNC();
        return;
    }
    /* 2. one bump allocation for the window's rows (16-byte granules) */
    const unsigned long long bytes = ((unsigned long long)n_seqs * (unsigned long long)cols + 15ull) & ~15ull;
    int32_t lo = 0, hi = 0;
    POA_LANE0 {
        const unsigned long long o = poa_bump64(out.cursor, bytes);
        lo = (int32_t)(o & 0xFFFFFFFFull);
        hi = (int32_t)(o >> 32);
    }
    const unsigned long long off = ((unsigned long long)(uint32_t)warp_bcast0(hi) << 32) | (unsigned long long)(uint32_t)warp_bcast0(lo);
    if (poa_uniform_pred(off + bytes > out.cap)) { /* cap arrives through a reference: laundered (poa_simt.cuh) */
        POA_LANE0 {
            *out.status = ST_GENERIC_ERROR;
            *out.cols = 0;
            *out.off = 0;
        }
        POA_SYNC();
        return;
    }
    uint8_t* rows = out.arena + off;
    /* 3. gaps everywhere (graph.cpp:401), then every base into its node's column (:404-410) */
    for (unsigned long long o = 0; o < bytes; o += 32 * 16) {
        POA_LANES(l) {
            const unsigned long long q = o + (unsigned long long)l * 16ull;
            if (q < bytes) poa_store16_dash(rows + q);
        }
    }
    POA_SYNC();
    POA_FENCE();
    for (int32_t r = 0; r < n_seqs; ++r) {
        const int64_t so = wv.seq_off[r];
        const int32_t len = poa_uniform(wv.seq_len[r]);
        uint8_t* row = rows + (size_t)r * (size_t)cols;
        for (int32_t base = 0; base < len; base += 64) {
            POA_LANES(l) {
                const int32_t p0 = base + l, p1 = base + 32 + l;
                const int32_t v0 = p0 < len ? (int32_t)wv.path[so + p0] : 0, v1 = p1 < len ? (int32_t)wv.path[so + p1] : 0;
                const uint8_t b0 = p0 < len ? wv.bases[so + p0] : (uint8_t)0, b1 = p1 < len ? wv.bases[so + p1] : (uint8_t)0;
                const int32_t c0 = s.c_score[v0], c1 = s.c_score[v1];
                if (p0 < len) row[c0] = b0;
                if (p1 < len) row[c1] = b1;
            }
        }
    }
    POA_SYNC();
    POA_LANE0 {
        *out.status = ST_SUCCESS;
        *out.cols = cols;
        *out.off = (long long)off;
    }
    POA_SYNC();
}

/* ------------------------------------------------------------------------------------------
 * int16 safety: every real cell of the skewed matrix must stay far from NEG and from +32767.
 * In the skewed domain S = H - j*gap a horizontal step costs 0, a diagonal step costs (s - gap), a vertical step
 * costs gap, and the value of a real cell is the score of SOME path from (0,0): it visits at most `n_columns`
 * graph nodes (a path crosses every aligned clique at most once) and makes at most min(len, n_columns) diagonal
 * steps.  Hence
 *     S >= n_columns * min(gap, match - gap, mismatch - gap, 0)
 *     S <= min(len, n_columns) * max(match - gap, mismatch - gap, 0) + n_columns * max(gap, 0)
 * for banded and full-band fills alike.  Inside these limits no cell is ever clamped and the int16 matrix equals
 * spoa's, whichever width spoa itself picks (its own rule, simd_alignment_engine.cpp:668-673, is the cruder
 * max|score| * (nodes + len + 17) < 32767; cudapoa picks the width statically, cudapoa_limits.hpp:34-53).
 * Outside them the window reports ST_SCORE_RANGE_EXCEEDED.
 * ---------------------------------------------------------------------------------------- */
POA_HD bool score_range_ok(const Params& p, int32_t n_columns, int32_t len) {
    const int32_t mg = p.match - p.gap, xg = p.mismatch - p.gap; /* the fill keeps them as int8 */
    if (mg < -128 || mg > 127 || xg < -128 || xg > 127 || p.gap < -128 || p.gap > 127) return false;
    int32_t lo_step = p.gap < 0 ? p.gap : 0;
    if (mg < lo_step) lo_step = mg;
    if (xg < lo_step) lo_step = xg;
    int32_t hi_diag = mg > xg ? mg : xg;
    if (hi_diag < 0) hi_diag = 0;
    const int64_t lo = (int64_t)lo_step * n_columns;
    const int64_t hi = (int64_t)hi_diag * (len < n_columns ? len : n_columns) + (p.gap > 0 ? (int64_t)p.gap * n_columns : 0);
    return lo > NEG + 512 && hi < 32000;
}

#if POA_FILL_DIGEST || POA_ALN_DIGEST || POA_GRAPH_DIGEST
POA_FN unsigned long long digest_mix64(unsigned long long x) { /* splitmix64's finaliser */
    x ^= x >> 30;
    x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27;
    x *= 0x94d049bb133111ebull;
    x ^= x >> 31;
    return x;
}
POA_FN unsigned long long digest_warp_sum(const PerLane<unsigned long long>& acc) {
#if POA_DEVICE
    unsigned long long t = acc[0];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) t += __shfl_xor_sync(0xffffffffu, t, d);
    return t;
#else
    unsigned long long t = 0;
    for (int l = 0; l < 32; ++l) t += acc[l];
    return t;
#endif
}
#endif
#if POA_FILL_DIGEST
/* Hash of the score rows the fill of one read just wrote: the wrapping sum, over the real cells (rows 1..n_rows, columns
 * [band start, band start + bw) within [0, len]), of mix64(row, column, value).  A sum does not depend on the order in
 * which lanes visit cells.  Cells past the read are not specified by the fill's contract and are not hashed. */
POA_FN_NOINLINE unsigned long long fill_digest(const Slot& s_ref, const Params p, const ReadGeom g_ref, int32_t cells32) {
    const Slot s = s_ref;
    const ReadGeom g = geom_uniform(g_ref);
    const int32_t* const S32 = reinterpret_cast<const int32_t*>(s.S);
    PerLane<unsigned long long> acc;
    POA_LANES(l) { acc[l] = 0; }
    for (int32_t i = 1; i <= g.n_rows; ++i) {
        const int32_t bs = rec_bs(s.row_rec[i]);
        const size_t row = (size_t)i * (size_t)p.stride;
        POA_LANES(l) {
            for (int32_t o = l; o < g.bw && bs + o <= g.len; o += 32) {
                const int32_t v = cells32 ? S32[row + o] : (int32_t)s.S[row + o];
                const unsigned long long key = (unsigned long long)(uint32_t)v | ((unsigned long long)(bs + o) << 32) |
                                               ((unsigned long long)i << 48);
                acc[l] += digest_mix64(key + 0x9e3779b97f4a7c15ull);
            }
        }
    }
    return digest_warp_sum(acc);
}
#endif
#if POA_ALN_DIGEST
/* Hash of the alignment the traceback left in tb_node/tb_pos[tb, cap): the wrapping sum over entries k (k = 0 is the
 * leftmost) of mix64(k << 32 | (uint16)pos << 16 | (uint16)node), -1 included.  The oracle hashes spoa's alignments the
 * same way (poa_oracle_alignment_digests). */
POA_FN_NOINLINE unsigned long long aln_digest(const Slot& s_ref, const Params p, int32_t tb) {
    const Slot s = s_ref;
    const int32_t cap = p.max_nodes + p.max_len + 2;
    PerLane<unsigned long long> acc;
    POA_LANES(l) {
        acc[l] = 0;
        for (int32_t e = tb + l; e < cap; e += 32) {
            const unsigned long long key = (unsigned long long)(uint16_t)s.tb_node[e] |
                                           ((unsigned long long)(uint16_t)s.tb_pos[e] << 16) |
                                           ((unsigned long long)(uint32_t)(e - tb) << 32);
            acc[l] += digest_mix64(key + 0x9e3779b97f4a7c15ull);
        }
    }
    return digest_warp_sum(acc);
}
#endif
#if POA_GRAPH_DIGEST
/* Hash of the graph: the wrapping sum over nodes v of
 *   mix64(v | letter << 16 | rank << 24 | coverage << 40),
 *   for the aligned id at list position q:  mix64(v | q << 16 | id << 24 | 1 << 56),
 *   for the in-edge at list position k:     mix64(mix64(v | k << 16 | source << 32 | 2 << 56) + (uint32)weight).
 * Node ids, letters, the rank order, coverage, the order of every clique and in-edge list and every weight.  The oracle
 * hashes spoa's graph the same way (poa_oracle_graph_digests). */
POA_FN_NOINLINE unsigned long long graph_digest(const Slot& s_ref, int32_t N) {
    const Slot s = s_ref;
    N = poa_uniform(N);
    constexpr unsigned long long K = 0x9e3779b97f4a7c15ull;
    PerLane<unsigned long long> acc;
    POA_LANES(l) {
        acc[l] = 0;
        for (int32_t v = l; v < N; v += 32) {
            acc[l] += digest_mix64(((unsigned long long)v | ((unsigned long long)s.code[v] << 16) |
                                    ((unsigned long long)s.rank_of[v] << 24) | ((unsigned long long)s.cov[v] << 40)) + K);
            const int32_t na = s.aln_cnt[v];
            for (int32_t q = 0; q < na; ++q)
                acc[l] += digest_mix64(((unsigned long long)v | ((unsigned long long)q << 16) |
                                        ((unsigned long long)s.aln[v * KA + q] << 24) | (1ull << 56)) + K);
            int32_t k = 0;
            for (uint16_t e = s.in_head[v]; e != NONE16; e = s.e_next[e], ++k) {
                const unsigned long long h = digest_mix64(((unsigned long long)v | ((unsigned long long)k << 16) |
                                                           ((unsigned long long)s.e_src[e] << 32) | (2ull << 56)) + K);
                acc[l] += digest_mix64(h + (unsigned long long)(uint32_t)s.e_w[e]);
            }
        }
    }
    return digest_warp_sum(acc);
}
/* Hash of a subgraph's member order: the wrapping sum over k < n of mix64(k << 32 | sub_at[k] | 3 << 56). */
POA_FN_NOINLINE unsigned long long sub_digest(const Slot& s_ref, int32_t n) {
    const Slot s = s_ref;
    n = poa_uniform(n);
    PerLane<unsigned long long> acc;
    POA_LANES(l) {
        acc[l] = 0;
        for (int32_t k = l; k < n; k += 32)
            acc[l] += digest_mix64(((unsigned long long)s.sub_at[k] | ((unsigned long long)k << 32) | (3ull << 56)) +
                                   0x9e3779b97f4a7c15ull);
    }
    return digest_warp_sum(acc);
}
/* Hash of the consensus scores: the wrapping sum over nodes v of mix64(mix64(v | 4 << 56) + ((uint32)c_score[v] |
 * (uint32)c_pred[v] << 32)), plus mix64(max_id | 5 << 56). */
POA_FN_NOINLINE unsigned long long cons_digest(const Slot& s_ref, int32_t N, int32_t max_id) {
    const Slot s = s_ref;
    N = poa_uniform(N);
    max_id = poa_uniform(max_id);
    constexpr unsigned long long K = 0x9e3779b97f4a7c15ull;
    PerLane<unsigned long long> acc;
    POA_LANES(l) {
        acc[l] = l == 0 ? digest_mix64(((unsigned long long)(uint32_t)max_id | (5ull << 56)) + K) : 0ull;
        for (int32_t v = l; v < N; v += 32)
            acc[l] += digest_mix64(digest_mix64(((unsigned long long)v | (4ull << 56)) + K) +
                                   ((unsigned long long)(uint32_t)s.c_score[v] |
                                    ((unsigned long long)(uint32_t)s.c_pred[v] << 32)));
    }
    return digest_warp_sum(acc);
}
/* after the backbone (r = 0) or after read r was added and sorted */
POA_FN void record_graph_digest(const Slot& s, const WinState& st, const WindowView& wv, int32_t r) {
    const unsigned long long d = graph_digest(s, st.n_nodes);
    POA_LANE0 {
        wv.graph_digest[r] = d;
        wv.graph_nodes[r] = st.n_nodes;
        wv.graph_edges[r] = st.n_edges;
    }
    POA_SYNC();
}
#endif

/* ------------------------------------------------------------------------------------------
 * One window, start to finish  (racon::Window::generate_consensus, src/window.cpp:65-116, for
 * full-span layers; the caller trims).  Fill is the DP-fill functor:
 *     int32_t operator()(slot, params, state, geom, read) -> end row (0 = none)
 * ---------------------------------------------------------------------------------------- */
template <class Fill>
POA_FN int32_t process_window(const Slot& s, const Params& p, const WindowView& wv, Fill& fill, const TbScratch& tbs,
                              const WindowOut& out, PhaseTimer tm = PhaseTimer{nullptr, 0}) {
    WinState st;
    st.n_nodes = 0;
    st.n_edges = 0;
    st.n_columns = 0;
    st.band_hit = 0;
    st.status = ST_SUCCESS;
    const int32_t len0 = wv.seq_len[0];
    tm.start();
    {
        const int64_t wo = wv.w_off[0];
        init_backbone(s, p, st, wv.bases + wv.seq_off[0], wo >= 0 ? wv.weights + wo : nullptr, wo >= 0 ? 0 : (int32_t)(-1 - wo), len0);
        winstate_uniform(st);
        if (wv.path && st.status == ST_SUCCESS) record_path(s.asg, wv.path + wv.seq_off[0], len0, 1);
#if POA_GRAPH_DIGEST
        if (st.status == ST_SUCCESS) record_graph_digest(s, st, wv, 0);
#endif
    }
    for (int32_t r = 1; r < wv.n_seqs && st.status == ST_SUCCESS; ++r) {
        const uint8_t* read = wv.bases + wv.seq_off[r];
        const int64_t wo = wv.w_off[r];
        const int8_t* wt = wo >= 0 ? wv.weights + wo : nullptr;
        const int32_t wconst = wo >= 0 ? 0 : (int32_t)(-1 - wo);
        const int32_t len = wv.seq_len[r];
        /* int16 cells whenever the alignment provably fits them; else 32-bit cells if the batch was sized for them */
        const bool cells32 = p.force_cells32 != 0 || !score_range_ok(p, st.n_columns, len);
        if (cells32 && !p.wide_cells) {
            st.status = ST_SCORE_RANGE_EXCEEDED;
            break;
        }
        /* window.cpp:92-103: a layer that does not span the window is aligned to a subgraph */
        const int32_t sp_begin = wv.seq_begin ? wv.seq_begin[r] : -1;
        const int32_t sp_end = wv.seq_end ? wv.seq_end[r] : -1;
        const bool partial = sp_begin >= 0;
        int32_t n_rows = st.n_nodes;
        if (partial) {
            if (sp_end >= len0 || sp_begin >= sp_end) { /* racon's add_layer guarantees begin < end <= backbone */
                st.status = ST_GENERIC_ERROR;
                break;
            }
            n_rows = poa_uniform(mark_subgraph(s, p, st, sp_begin, sp_end, reinterpret_cast<uint16_t*>(tbs.cells), TB_SCRATCH_BYTES / 2));
            POA_GRAPH_REACH_IF(sp_begin == 0, sub_begin0);
            POA_GRAPH_REACH_IF(sp_end == len0 - 1, sub_end_last);
            POA_GRAPH_TWIN(subgraph, s, p, st, r, sp_begin, sp_end, n_rows, TB_SCRATCH_BYTES / 2);
#if POA_GRAPH_DIGEST
            {
                const unsigned long long d = sub_digest(s, n_rows);
                POA_LANE0 {
                    wv.sub_digest[r] = d;
                    wv.sub_count[r] = n_rows;
                }
                POA_SYNC();
            }
#endif
        }
        /* static band: one try.  Adaptive band: the configured width is the first try; a traceback that comes close to
         * a band edge (or loses the path) re-aligns this read with twice the width, up to the full matrix. */
        int32_t band_w = p.band_width;
        int32_t tb = 0;
        for (;;) {
            const ReadGeom g = read_geometry(p, len, n_rows, band_w);
            tm.lap(PH_OTHER);
            if (partial) build_program_sub(s, p, st, g);
            else build_program(s, p, st, g);
            winstate_uniform(st);
            POA_FENCE();
            tm.lap(PH_PROGRAM);
            if (st.status != ST_SUCCESS) break;
            const int32_t end_row = poa_uniform(cells32 ? fill_rows_i32(s, p, g, read) : fill(s, p, st, g, read));
            POA_FENCE(); /* the score rows must be in place before the traceback's asynchronous copies read them */
#if POA_FILL_DIGEST
            {
                const unsigned long long d = fill_digest(s, p, g, cells32 ? 1 : 0);
                POA_LANE0 {
                    wv.fill_digest[r] += d;
                    wv.fill_count[r] += 1;
                }
                POA_SYNC();
            }
#endif
            tm.lap(PH_FILL);
            st.band_hit = 0;
            if (end_row <= 0) {
                st.status = ST_TRACEBACK_LOST;
            } else {
                tb = poa_uniform(cells32 ? traceback_i32(s, p, st, g, end_row, read, partial ? s.sub_at : s.node_at)
                                         : traceback(s, p, st, g, read, end_row, tbs, partial ? s.sub_at : s.node_at));
                winstate_uniform(st);
                POA_FENCE();
                tm.lap(PH_TRACEBACK);
                POA_TB_TWIN(fill, s, p, st, g, r, read, end_row, tb, partial ? s.sub_at : s.node_at, cells32, partial);
            }
            if (p.adaptive && g.banded && (st.band_hit || st.status == ST_TRACEBACK_LOST)) {
                st.status = ST_SUCCESS;
                band_w *= 2;
                continue;
            }
            break;
        }
        if (st.status != ST_SUCCESS) break;
#if POA_ALN_DIGEST
        {
            const unsigned long long d = aln_digest(s, p, tb);
            POA_LANE0 {
                wv.aln_digest[r] = d;
                wv.aln_count[r] = p.max_nodes + p.max_len + 2 - tb;
            }
            POA_SYNC();
        }
#endif
        add_alignment(s, p, st, read, wt, wconst, len, tb);
        winstate_uniform(st);
        POA_FENCE();
        tm.lap(PH_ADD);
        if (st.status != ST_SUCCESS) break;
        if (wv.path) record_path(s.asg, wv.path + wv.seq_off[r], len, 0);
        if (p.serial_topsort) topsort_serial(s, p, st);
        else topsort_roots(s, p, st);
        winstate_uniform(st);
        POA_FENCE();
        tm.lap(PH_TOPSORT);
        POA_GRAPH_TWIN(topsort, s, p, st, r);
#if POA_GRAPH_DIGEST
        record_graph_digest(s, st, wv, r);
#endif
    }
    if (st.status == ST_SUCCESS && !p.skip_consensus) {
        generate_consensus(s, p, st, out);
        winstate_uniform(st);
    }
    tm.lap(PH_CONSENSUS);
    POA_LANE0 {
        if (st.status != ST_SUCCESS || p.skip_consensus) {
            *out.len = 0;
            *out.off = 0;
            *out.trim = (int32_t)0xFFFF0000u; /* first 0, last -1 */
        }
        *out.status = st.status;
    }
    POA_SYNC();
    return st.status == ST_SUCCESS ? st.n_nodes : -1; /* the graph stays in the slot: generate_msa() may follow */
}

/* The MSA of the window process_window() just finished (n_nodes = its return value, status = what it reported);
 * runs after the consensus because the column table takes over the consensus' score array. */
POA_FN void window_msa(const Slot& s, const Params& p, int32_t n_nodes, int32_t status, const WindowView& wv, const MsaOut& mo) {
    if (n_nodes >= 0) {
        generate_msa(s, p, n_nodes, wv, mo);
    } else {
        POA_LANE0 {
            *mo.status = status;
            *mo.cols = 0;
            *mo.off = 0;
        }
        POA_SYNC();
    }
}

} // namespace b200poa
