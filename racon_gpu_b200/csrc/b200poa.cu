/*
 * b200poa.cu -- C ABI (include/b200poa.h) + batch runtime + the POA kernel launch.
 *
 * Batch runtime = what vendor/GenomeWorks/cudapoa/src/cudapoa_batch.cuh:62-646 and
 * allocate_block.hpp:53-479 do in the reference, re-designed:
 *   - device memory is split into (a) per-RESIDENT-WARP workspaces ("slots": graph + score band)
 *     and (b) the batch's columnar input arena and compact outputs.  The reference sizes the batch
 *     by score-matrix memory per window (allocate_block.hpp:81-83: ~20-35k windows per 180 GB);
 *     here a batch is limited only by its arena, because a slot is reused by every window the warp
 *     pulls from the work queue;
 *   - one persistent launch per batch: grid = resident warps, each warp pops windows from an
 *     atomic cursor over a longest-first work list (depth/length-divergent windows, SURVEY.md 7);
 *   - H2D is 4 contiguous async copies of exactly the staged bytes, D2H copies exactly
 *     poa_count rows (the reference copies max_poas full rows, cudapoa_batch.cuh:213-222).
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <new>
#include <numeric>
#include <vector>

#include "../../include/b200poa.h"
#include "poa_core.cuh"
#include "poa_fill.cuh"
#include "cuda_buffers.hpp"

using namespace b200poa;
using namespace b200buf;

/* ------------------------------------------------------------------------------------------ */
/* kernel                                                                                      */
/* ------------------------------------------------------------------------------------------ */
struct KernelArgs {
    Params p;
    uint8_t* slab;       /* n_slots * slot_bytes */
    size_t slot_bytes;
    int32_t n_windows;
    const int32_t* work; /* window ids, most expensive first */
    int32_t* cursor;     /* [0] atomic work cursor, [1] elements used in the output arenas (both zeroed before launch) */
    const uint8_t* bases;
    const int8_t* weights;      /* compact: sequences with non-constant weights only */
    const int64_t* seq_off;     /* [n_seqs] start in the bases arena, processing order */
    const int32_t* seq_len;     /* [n_seqs] */
    const int64_t* w_off;       /* [n_seqs] offset into weights, or -1 - constant */
    const int32_t* win_seq_off; /* [n_windows+1] */
    const int32_t* win_flags;   /* per window: pre-set status (!= 0 => skip) */
    const int32_t* win_trim_nseq; /* per window: sequences counted by the trim threshold */
    const int32_t* seq_begin;   /* [n_seqs] layer span (-1 = spans the window)  */
    const int32_t* seq_end;     /* [n_seqs] */
    uint8_t* out_cons;          /* compact arenas, see WindowOut */
    uint16_t* out_cov;
    int32_t* out_len;
    int32_t* out_status;
    int32_t* out_off;
    int32_t* out_trim;
    /* multiple sequence alignment (output mask has B200POA_OUTPUT_MSA; else all null) */
    uint16_t* path;               /* [arena] node of every base, parallel to `bases` */
    uint8_t* out_msa;             /* compact MSA arena */
    unsigned long long* msa_cursor;
    unsigned long long msa_cap;
    long long* out_msa_off;
    int32_t* out_msa_cols;
    int32_t* out_msa_status;
    int32_t prof_stride; /* bytes per profile row        */
    int32_t ring_stride; /* int16 cells per ring row     */
    int32_t ring_rows;   /* power of two                 */
    unsigned long long* phase_cycles; /* diagnostics: [PH_COUNT] or nullptr */
#if POA_FILL_DIGEST
    unsigned long long* fill_digest; /* [staged sequences] see b200poa_debug_fill_digest */
    int32_t* fill_count;
#endif
#if POA_ALN_DIGEST
    unsigned long long* aln_digest;  /* [staged sequences] see b200poa_debug_aln_digest */
    int32_t* aln_count;
#endif
#if POA_GRAPH_DIGEST
    unsigned long long* graph_digest; /* [staged sequences] see b200poa_debug_graph_digest */
    int32_t* graph_nodes;
    int32_t* graph_edges;
    unsigned long long* sub_digest;
    int32_t* sub_count;
    unsigned long long* cons_digest;  /* [2 x staged windows] */
    int32_t* cons_rounds;             /* [staged windows] */
#endif
};

#ifndef POA_MIN_BLOCKS_PER_SM
#define POA_MIN_BLOCKS_PER_SM 20 /* 20 warps/SM => <= 96 registers per thread; on an H100 (400 W) 54k banded windows/s vs 49k at 24 and 53k at 16 */
#endif
__global__ void __launch_bounds__(32, POA_MIN_BLOCKS_PER_SM) poa_window_kernel(const KernelArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    /* The workspace descriptor is pure arithmetic on kernel parameters (constant bank): the
     * compiler rematerialises the few pointers a phase needs instead of pinning 33 of them. */
    Slot s;
    slot_bind(s, a.slab + (size_t)blockIdx.x * a.slot_bytes, a.p, nullptr);
    CudaFill fill;
    fill.smem_sa = (uint32_t)__cvta_generic_to_shared(smem_raw);
    fill.prof_stride = a.prof_stride;
    fill.ring_stride = a.ring_stride;
    fill.ring_mask = a.ring_rows - 1;
    /* the traceback tile overlays the query profile and the score-row ring: the fill rebuilds both per read */
    TbScratch tbs;
    tb_bind(tbs, smem_raw + 32);
    const int lane = threadIdx.x & 31;
    for (;;) {
        int32_t t = 0;
        if (lane == 0) t = atomicAdd(a.cursor, 1);
        t = warp_bcast0(t); /* through redux.sync: the work loop is provably warp-uniform (poa_simt.cuh) */
        if (t >= a.n_windows) break;
        const int32_t w = a.work[t];
        if (a.win_flags[w] != 0) {
            if (lane == 0) {
                a.out_len[w] = 0;
                a.out_off[w] = 0;
                a.out_trim[w] = (int32_t)0xFFFF0000u;
                a.out_status[w] = a.win_flags[w];
                if (a.out_msa) {
                    a.out_msa_off[w] = 0;
                    a.out_msa_cols[w] = 0;
                    a.out_msa_status[w] = a.win_flags[w];
                }
            }
            __syncwarp(); /* explicit reconvergence before the back edge: without it ptxas assumes a diverged loop head
                             and gives EVERY collective of the kernel a BRA.DIV slow path (poa_simt.cuh) */
            continue;
        }
        WindowView wv;
        const int32_t s0 = a.win_seq_off[w];
        wv.n_seqs = a.win_seq_off[w + 1] - s0;
        wv.bases = a.bases;
        wv.weights = a.weights;
        wv.seq_off = a.seq_off + s0;
        wv.seq_len = a.seq_len + s0;
        wv.w_off = a.w_off + s0;
        wv.seq_begin = a.seq_begin + s0;
        wv.seq_end = a.seq_end + s0;
        wv.path = a.path;
#if POA_FILL_DIGEST
        wv.fill_digest = a.fill_digest + s0;
        wv.fill_count = a.fill_count + s0;
#endif
#if POA_ALN_DIGEST
        wv.aln_digest = a.aln_digest + s0;
        wv.aln_count = a.aln_count + s0;
#endif
#if POA_GRAPH_DIGEST
        wv.graph_digest = a.graph_digest + s0;
        wv.graph_nodes = a.graph_nodes + s0;
        wv.graph_edges = a.graph_edges + s0;
        wv.sub_digest = a.sub_digest + s0;
        wv.sub_count = a.sub_count + s0;
#endif
        WindowOut out;
        out.cons = a.out_cons;
        out.cov = a.out_cov;
        out.cursor = reinterpret_cast<uint32_t*>(a.cursor + 1);
        out.len = a.out_len + w;
        out.status = a.out_status + w;
        out.off = a.out_off + w;
        out.trim = a.out_trim + w;
        out.trim_nseq = a.win_trim_nseq[w];
#if POA_GRAPH_DIGEST
        out.cons_digest = a.cons_digest + 2 * (size_t)w;
        out.cons_rounds = a.cons_rounds + w;
#endif
        const int32_t n_nodes = poa_uniform(process_window(s, a.p, wv, fill, tbs, out, PhaseTimer{a.phase_cycles, 0}));
        if (a.out_msa) { /* B200POA_OUTPUT_MSA */
            MsaOut mo;
            mo.arena = a.out_msa;
            mo.cursor = a.msa_cursor;
            mo.cap = a.msa_cap;
            mo.off = a.out_msa_off + w;
            mo.cols = a.out_msa_cols + w;
            mo.status = a.out_msa_status + w;
            window_msa(s, a.p, n_nodes, poa_uniform(a.out_status[w]), wv, mo);
        }
    }
}

/* ------------------------------------------------------------------------------------------ */
/* batch object                                                                                */
/* ------------------------------------------------------------------------------------------ */
#define CU_TRY(expr)                                                                         \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            std::fprintf(stderr, "[b200poa] CUDA error %s at %s:%d: %s\n", #expr, __FILE__,  \
                         __LINE__, cudaGetErrorString(_e));                                  \
            return B200POA_CUDA_ERROR;                                                       \
        }                                                                                    \
    } while (0)

namespace {
std::atomic<int32_t> g_batches{0};
} // namespace

/* Every buffer is a member that frees itself (cuda_buffers.hpp); the destructor waits for the batch's stream first. */
struct b200poa_batch {
    ~b200poa_batch() { cudaStreamSynchronize(stream); }
    int32_t id = 0;
    int32_t device = 0;
    cudaStream_t stream = nullptr;
    int32_t output_mask = 0;
    b200poa_config cfg{};
    Params p{};
    /* capacity */
    int32_t max_poas = 0;
    int64_t max_seqs = 0;
    int64_t arena_cap = 0;
    int32_t n_slots = 0;
    size_t slot_bytes = 0;
    int32_t smem_bytes = 0;
    int32_t prof_stride = 0;
    int32_t ring_stride = 0;
    int32_t ring_rows = 0;
    int32_t blocks_per_sm = 0;
    int32_t sm_count = 0;
    int32_t max_len_staged = 0;
    size_t device_bytes = 0;
    /* staged inputs (pinned host -> device); in direct mode bases and weights go up from the caller's arena instead */
    Mirror<uint8_t> bases;
    Mirror<int8_t> weights;
    Mirror<int64_t> seq_off, w_off;
    Mirror<int32_t> seq_len, seq_begin, seq_end;
    Mirror<int32_t> win_seq_off, win_flags, win_trim_nseq, work;
    /* outputs (device -> pinned host) */
    Mirror<int32_t> cursor; /* [2] work cursor, elements used in the output arenas */
    Mirror<uint8_t> cons;
    Mirror<uint16_t> cov;
    Mirror<int32_t> len, status, out_off, trim;
    DevBuf slab;
    DevBuf phase; /* B200POA_PHASE_TIMERS diagnostics */
    /* multiple sequence alignment (output mask has B200POA_OUTPUT_MSA) */
    DevBuf path;                        /* [arena_cap] node of every base */
    DevBuf msa;                         /* [msa_cap] compact rows */
    Mirror<unsigned long long> msa_cursor;
    Mirror<long long> msa_off;
    Mirror<int32_t> msa_cols, msa_status;
    PinnedBuf h_msa;                    /* grown on demand to the bytes a launch used */
    PinnedBuf h_msa_rows;               /* int32 per window: sequences staged = rows of its MSA */
#if POA_FILL_DIGEST
    DevBuf fill_digest, fill_count; /* [max_seqs] per staged sequence, see b200poa_debug_fill_digest */
#endif
#if POA_ALN_DIGEST
    DevBuf aln_digest, aln_count; /* [max_seqs] see b200poa_debug_aln_digest */
#endif
#if POA_GRAPH_DIGEST
    DevBuf graph_digest, graph_nodes, graph_edges, sub_digest, sub_count; /* [max_seqs] see b200poa_debug_graph_digest */
    DevBuf cons_digest, cons_rounds;                                      /* [2 x max_poas], [max_poas] */
#endif
    size_t msa_cap = 0;
    size_t msa_bound = 0;                  /* worst-case MSA bytes of the windows staged so far */
    bool msa_fetched = false;
    /* fill state */
    int32_t poa_count = 0;
    int64_t seq_count = 0;
    int64_t base_count = 0;
    int64_t weight_count = 0;  /* bytes in the compact weights arena */
    /* direct mode (b200poa_batch_add_windows_pinned): the batch's device arena mirrors the byte range [ext_lo, ext_hi)
     * of the caller's pinned host arena -- uploaded straight from there, no staging copy on the host */
    const uint8_t* ext_bases = nullptr;
    const int8_t* ext_weights = nullptr;
    int64_t ext_lo = 0, ext_hi = 0;
    bool ext_any_weights = false;
    int64_t out_elems = 0;     /* elements the last downloaded launch used in the output arenas */
    bool results_fetched = false;
    int32_t download_coverage = 1; /* B200POA_OPT_DOWNLOAD_COVERAGE */
    int32_t trim_counts_staged = 0; /* B200POA_OPT_TRIM_COUNTS_STAGED */
    int64_t h2d_bytes = 0, d2h_bytes = 0; /* PCIe bytes of the last generate / get_consensus */
    std::vector<int64_t> cost; /* per window work estimate for the longest-first work list */
    int64_t launches = 0;
    bool uploaded = false;
};

/* Shared memory geometry of a launch whose longest staged read has `max_len` bases: profile rows, score-row ring.
 * Full-band rows are laid out for fill_rows_wide (lane l owns 8*NV consecutive columns): profile and ring rows are
 * padded to a multiple of 256 columns. */
struct SmemGeometry {
    int32_t prof_stride, ring_stride, ring_rows, smem_bytes;
};
static SmemGeometry smem_geometry(const Params& p, int32_t max_len) {
    SmemGeometry g;
    const int32_t colsP = (max_len + 1 + 7) & ~7;
    const bool banded = !p.adaptive && p.band_width > 0 && p.band_width < colsP;
    /* fill_rows_wide (full-band rows, and reads shorter than the band in banded batches) gives lane l the columns
     * [l*8*NV, (l+1)*8*NV): lanes past the read still load -- never store -- profile bytes and ring cells up to
     * column 256*NV.  Rows are therefore sized by the longest read only, and the allocation ends with enough slack
     * for the loads of the last row. */
    g.prof_stride = banded ? std::max(colsP, 256) : colsP;
    const int32_t row_cells = banded ? std::max(p.band_width, 256) : colsP;
    /* in a banded batch the reads shorter than the band take fill_rows_wide too: a band of 384 columns runs reads of up
     * to 384 columns with NV = 2, whose lanes load up to column 512 of the last ring row */
    const int32_t slack_cells = 256 * ((row_cells + 255) / 256) - row_cells;
    g.ring_stride = row_cells + RING_PAD_FRONT + RING_PAD_BACK;
    int32_t ring_bytes = 4096;
    {   /* at least 8 ring rows: a predecessor more than 7 ranks back is rare (0.6%), more than 3 is not (19%) */
        const int32_t need8 = 8 * g.ring_stride * (int32_t)sizeof(int16_t);
        if (need8 > ring_bytes && need8 <= 20480) ring_bytes = need8;
    }
    if (const char* env = std::getenv("B200POA_RING_BYTES")) ring_bytes = std::atoi(env);
    int32_t rows = 2;
    while (rows < 32 && rows * 2 * g.ring_stride * (int32_t)sizeof(int16_t) <= ring_bytes) rows *= 2;
    g.ring_rows = rows;
    g.smem_bytes = 32 + std::max(((PROF_ROWS * g.prof_stride + 15) & ~15) +
                                     (g.ring_rows * g.ring_stride + slack_cells) * (int32_t)sizeof(int16_t),
                                 (int32_t)TB_SCRATCH_BYTES);
    return g;
}

/* One sequence as the staging code sees it. */
struct StagedSeq {
    const char* seq;
    const int8_t* w;   /* nullptr: no quality string (weight 1 per base) */
    int32_t len, bg, en;
    int64_t host_off;  /* direct mode: offset of the sequence in the caller's pinned arena */
    int64_t wmode;     /* direct mode: precomputed weight mode (-1 - constant, or >= 0: explicit weights); else INT64_MIN */
};
constexpr int64_t WMODE_UNKNOWN = INT64_MIN;

/* Stage one window whose sequences are given in processing order through a getter.
 * DIRECT = false: bases (and non-constant weights) are copied into the batch's own pinned staging arena.
 * DIRECT = true : nothing is copied; the tables point into the caller's pinned arena, whose byte range
 *                 [ext_lo, ext_hi) is uploaded as it is (sequences in add order; the tables carry the processing order). */
template <bool DIRECT, class Get>
static int32_t stage_window(b200poa_batch* b, int32_t n, Get get, int32_t* per_seq_status, int32_t* n_added_out,
                            int64_t win_lo = 0, int64_t win_hi = 0) {
    /* cudapoa_batch.cuh:108-148: the whole group must fit or the batch reports "full" */
    if (b->poa_count >= b->max_poas) return B200POA_EXCEEDED_MAXIMUM_POAS;
    int64_t bytes = 0;
    int32_t n_ok = 0;
    for (int32_t i = 0; i < n; ++i) {
        StagedSeq q;
        get(i, q);
        if (q.len <= b->cfg.max_sequence_size && n_ok < b->cfg.max_sequences_per_poa) {
            if (q.len <= 0) return B200POA_INVALID_ARGUMENT;
            if (q.w && q.wmode == WMODE_UNKNOWN) /* validate BEFORE anything is staged (cudapoa_batch.cuh:533-537 throws) */
                for (int32_t k = 0; k < q.len; ++k)
                    if (q.w[k] < 0) return B200POA_INVALID_ARGUMENT;
            bytes += q.len;
            ++n_ok;
        }
    }
    /* MSA output: n rows of at most min(max_consensus_size, sum of lengths) columns (every base adds at most one node;
     * longer alignments fail with exceeded_maximum_sequence_size, cudapoa_generate_msa.cuh:203-208): the batch is
     * "full" when the worst case of its windows would not fit the MSA arena (cudapoa_batch.cuh:122-125's back-pressure) */
    size_t msa_need = 0;
    if (b->output_mask & B200POA_OUTPUT_MSA) {
        msa_need = ((size_t)n_ok * (size_t)std::min<int64_t>(bytes, b->cfg.max_consensus_size) + 15) & ~(size_t)15;
        if (b->msa_bound + msa_need > b->msa_cap) return B200POA_EXCEEDED_MAXIMUM_POAS;
    }
    if (DIRECT) { /* the device arena mirrors the contiguous host range of the windows staged so far */
        const int64_t lo = b->poa_count == 0 ? win_lo : b->ext_lo;
        if (win_lo < lo || win_hi - lo > b->arena_cap || b->seq_count + n_ok > b->max_seqs) return B200POA_EXCEEDED_MAXIMUM_POAS;
    } else if (b->base_count + bytes > b->arena_cap || b->seq_count + n_ok > b->max_seqs) {
        return B200POA_EXCEEDED_MAXIMUM_POAS;
    }
    if (DIRECT) {
        if (b->poa_count == 0) b->ext_lo = win_lo;
        b->ext_hi = win_hi;
        b->base_count = b->ext_hi - b->ext_lo;
    }

    int32_t flag = 0, added = 0;
    int64_t cost = 0;
    int32_t bb_len = 0;
    bool backbone_rejected = false;
    for (int32_t i = 0; i < n; ++i) {
        StagedSeq q;
        get(i, q);
        const int32_t len = q.len, bg = q.bg, en = q.en;
        int32_t st = B200POA_SUCCESS;
        if (len > b->cfg.max_sequence_size) st = B200POA_EXCEEDED_MAXIMUM_SEQUENCE_SIZE; /* cudapoa_batch.cuh:501-504 */
        else if (added >= b->cfg.max_sequences_per_poa) st = B200POA_EXCEEDED_MAXIMUM_SEQUENCES_PER_POA; /* :513-516 */
        if (i == 0 && st != B200POA_SUCCESS) backbone_rejected = true;
        /* a window whose backbone was rejected stages nothing: no layer may take the backbone's place */
        if (backbone_rejected && st == B200POA_SUCCESS) st = B200POA_EXCEEDED_MAXIMUM_SEQUENCE_SIZE;
        if (per_seq_status) per_seq_status[i] = st;
        if (st != B200POA_SUCCESS) continue;
        int32_t sp_b = -1, sp_e = -1; /* -1: the layer spans the window */
        if (added == 0) {
            bb_len = len;
        } else if (!(bg == -1 && en == -1)) {
            /* window.cpp:87,92-93: does the layer span the whole window?  If not it is aligned to the
             * subgraph between its begin and end backbone positions (window.cpp:96-103). */
            const uint32_t L = (uint32_t)bb_len;
            const uint32_t offset = (uint32_t)(0.01 * L);
            if (!((uint32_t)bg < offset && (uint32_t)en > L - offset)) {
                sp_b = bg;
                sp_e = en;
                if (bg < 0 || en >= bb_len || bg >= en) flag = B200POA_INVALID_ARGUMENT; /* window.cpp:55-59 rejects it */
            }
        }
        b->seq_begin.h()[b->seq_count] = sp_b;
        b->seq_end.h()[b->seq_count] = sp_e;
        if (len > b->max_len_staged) b->max_len_staged = len;
        /* weights: a sequence whose bases all weigh the same (no quality string => 1, cudapoa_batch.cuh:525-530;
         * the '!' dummy quality of a FASTA target => 0) ships only that constant */
        int64_t wo = -1 - 1;
        if (DIRECT) {
            b->seq_off.h()[b->seq_count] = q.host_off - b->ext_lo;
            if (q.w) {
                wo = q.wmode;
                if (wo >= 0) { /* explicit weights: the weights arena mirrors the same host range */
                    wo = q.host_off - b->ext_lo;
                    b->ext_any_weights = true;
                }
            }
        } else {
            b->seq_off.h()[b->seq_count] = b->base_count;
            std::memcpy(b->bases.h() + b->base_count, q.seq, (size_t)len);
            if (q.w) {
                bool constant = true;
                for (int32_t k = 1; k < len && constant; ++k) constant = q.w[k] == q.w[0];
                if (constant) {
                    wo = -1 - (int64_t)q.w[0];
                } else {
                    wo = b->weight_count;
                    std::memcpy(b->weights.h() + b->weight_count, q.w, (size_t)len);
                    b->weight_count += len;
                }
            }
            b->base_count += len;
        }
        b->w_off.h()[b->seq_count] = wo;
        b->seq_len.h()[b->seq_count] = len;
        b->seq_count += 1;
        cost += (int64_t)len * (bb_len + (int64_t)added * (bb_len / 8 + 1));
        ++added;
    }
    if (backbone_rejected) flag = B200POA_EXCEEDED_MAXIMUM_SEQUENCE_SIZE; /* the kernel skips the window and reports why */
    b->win_flags.h()[b->poa_count] = flag;
    b->win_trim_nseq.h()[b->poa_count] = b->trim_counts_staged ? added : n; /* window.cpp:121 counts every sequence */
    if (b->h_msa_rows.p) reinterpret_cast<int32_t*>(b->h_msa_rows.p)[b->poa_count] = added;
    b->msa_bound += msa_need;
    b->poa_count += 1;
    b->win_seq_off.h()[b->poa_count] = (int32_t)b->seq_count;
    b->cost.push_back(cost);
    b->uploaded = false;
    if (n_added_out) *n_added_out = added > 0 ? added - 1 : 0;
    return B200POA_SUCCESS;
}

static int32_t alloc_batch_memory(b200poa_batch* b) {
    const Params& p = b->p;
    const size_t MP = (size_t)b->max_poas, MS = (size_t)b->max_seqs, AC = (size_t)b->arena_cap;
    CU_TRY(b->slab.need((size_t)b->n_slots * b->slot_bytes, false));
    if (const char* env = std::getenv("B200POA_SLAB_FILL")) /* debugging: the engine must not depend on what a slot held before */
        CU_TRY(cudaMemset(b->slab.p, std::atoi(env), (size_t)b->n_slots * b->slot_bytes));
    CU_TRY(b->bases.alloc(AC));
    CU_TRY(b->weights.alloc(AC));
    CU_TRY(b->seq_off.alloc(MS + 1));
    CU_TRY(b->w_off.alloc(MS + 1));
    CU_TRY(b->seq_len.alloc(MS + 1));
    CU_TRY(b->seq_begin.alloc(MS + 1));
    CU_TRY(b->seq_end.alloc(MS + 1));
    CU_TRY(b->win_seq_off.alloc(MP + 1));
    CU_TRY(b->win_flags.alloc(MP));
    CU_TRY(b->win_trim_nseq.alloc(MP));
    CU_TRY(b->work.alloc(MP));
    CU_TRY(b->cursor.alloc(2));
    CU_TRY(b->cons.alloc(MP * (size_t)p.max_cons));
    CU_TRY(b->cov.alloc(MP * (size_t)p.max_cons));
    CU_TRY(b->len.alloc(MP));
    CU_TRY(b->status.alloc(MP));
    CU_TRY(b->out_off.alloc(MP));
    CU_TRY(b->trim.alloc(MP));
    if (std::getenv("B200POA_PHASE_TIMERS")) {
        CU_TRY(b->phase.need(PH_COUNT * sizeof(unsigned long long), false));
        CU_TRY(cudaMemset(b->phase.p, 0, PH_COUNT * sizeof(unsigned long long)));
    }
    /* an estimate: of the per-sequence and per-window tables it counts 8 of 28 B a sequence and 16 of 32 B a window */
    b->device_bytes = (size_t)b->n_slots * b->slot_bytes + 2 * AC + (MS + 1) * 8 + MP * (16 + 3 * (size_t)p.max_cons);
    if (b->output_mask & B200POA_OUTPUT_MSA) {
        CU_TRY(b->path.need(AC * sizeof(uint16_t), false));
        CU_TRY(b->msa.need(b->msa_cap, false));
        CU_TRY(b->msa_cursor.alloc(1));
        CU_TRY(b->msa_off.alloc(MP));
        CU_TRY(b->msa_cols.alloc(MP));
        CU_TRY(b->msa_status.alloc(MP));
        if (!b->h_msa_rows.reserve(MP * sizeof(int32_t))) return B200POA_CUDA_ERROR;
        b->device_bytes += AC * sizeof(uint16_t) + b->msa_cap + MP * 16;
    }
#if POA_FILL_DIGEST
    CU_TRY(b->fill_digest.need((MS + 1) * sizeof(unsigned long long), false));
    CU_TRY(b->fill_count.need((MS + 1) * sizeof(int32_t), false));
#endif
#if POA_ALN_DIGEST
    CU_TRY(b->aln_digest.need((MS + 1) * sizeof(unsigned long long), false));
    CU_TRY(b->aln_count.need((MS + 1) * sizeof(int32_t), false));
#endif
#if POA_GRAPH_DIGEST
    CU_TRY(b->graph_digest.need((MS + 1) * sizeof(unsigned long long), false));
    CU_TRY(b->graph_nodes.need((MS + 1) * sizeof(int32_t), false));
    CU_TRY(b->graph_edges.need((MS + 1) * sizeof(int32_t), false));
    CU_TRY(b->sub_digest.need((MS + 1) * sizeof(unsigned long long), false));
    CU_TRY(b->sub_count.need((MS + 1) * sizeof(int32_t), false));
    CU_TRY(b->cons_digest.need(2 * (MP + 1) * sizeof(unsigned long long), false));
    CU_TRY(b->cons_rounds.need((MP + 1) * sizeof(int32_t), false));
#endif
    return B200POA_SUCCESS;
}

/* shared body of b200poa_batch_add_windows (staged) and b200poa_batch_add_windows_pinned (direct) */
template <bool DIRECT>
static int32_t add_windows_impl(b200poa_batch* b, int64_t n_windows, int64_t first, const int64_t* win_seq_off,
                                const int64_t* seq_off, const uint8_t* bases, const int8_t* weights,
                                const uint8_t* has_weights, const int64_t* weight_mode, const int32_t* begins,
                                const int32_t* ends, int64_t* n_added, int32_t* seqs_added) {
    if (!b || !n_added) return B200POA_INVALID_ARGUMENT;
    *n_added = 0;
    if (DIRECT ? (b->poa_count > 0 && (b->ext_bases != bases || b->ext_weights != weights)) : b->ext_bases != nullptr)
        return B200POA_INVALID_ARGUMENT; /* a batch is either staged or direct (one arena) until its next reset */
    std::vector<uint32_t> rank;
    for (int64_t w = first; w < n_windows; ++w) {
        const int64_t s0 = win_seq_off[w];
        const int32_t n = (int32_t)(win_seq_off[w + 1] - s0);
        /* src/window.cpp:78-85 == src/cuda/cudabatch.cpp:96-104 (see b200poa_layer_order) */
        rank.resize((size_t)n);
        for (int32_t i = 0; i < n; ++i) rank[(size_t)i] = (uint32_t)i;
        if (n > 1)
            std::sort(rank.begin() + 1, rank.end(),
                      [&](uint32_t lhs, uint32_t rhs) { return begins[s0 + lhs] < begins[s0 + rhs]; });
        auto get = [&](int32_t i, StagedSeq& q) {
            const int64_t s = s0 + rank[(size_t)i];
            q.seq = reinterpret_cast<const char*>(bases + seq_off[s]);
            q.w = has_weights[s] ? weights + seq_off[s] : nullptr;
            q.len = (int32_t)(seq_off[s + 1] - seq_off[s]);
            q.bg = begins[s];
            q.en = ends[s];
            q.host_off = seq_off[s];
            q.wmode = (DIRECT && weight_mode) ? weight_mode[s] : WMODE_UNKNOWN;
        };
        int32_t added = 0;
        const int32_t st = stage_window<DIRECT>(b, n, get, nullptr, &added, seq_off[s0], seq_off[win_seq_off[w + 1]]);
        if (st == B200POA_EXCEEDED_MAXIMUM_POAS) break;
        if (st != B200POA_SUCCESS) return st;
        if (DIRECT) {
            b->ext_bases = bases;
            b->ext_weights = weights;
        }
        if (seqs_added) seqs_added[*n_added] = added;
        ++*n_added;
    }
    return B200POA_SUCCESS;
}

extern "C" {

int32_t b200poa_init(void) { return B200POA_SUCCESS; } /* cudapoa.cpp:29-35: nothing to set up */

const char* b200poa_status_string(int32_t st) {
    switch (st) {
        case B200POA_SUCCESS: return "success";
        case B200POA_EXCEEDED_MAXIMUM_POAS: return "exceeded_maximum_poas";
        case B200POA_EXCEEDED_MAXIMUM_SEQUENCE_SIZE: return "exceeded_maximum_sequence_size";
        case B200POA_EXCEEDED_MAXIMUM_SEQUENCES_PER_POA: return "exceeded_maximum_sequences_per_poa";
        case B200POA_NODE_COUNT_EXCEEDED_MAXIMUM_GRAPH_SIZE: return "node_count_exceeded_maximum_graph_size";
        case B200POA_EDGE_COUNT_EXCEEDED_MAXIMUM_GRAPH_SIZE: return "edge_count_exceeded_maximum_graph_size";
        case B200POA_EXCEEDED_ADAPTIVE_BANDED_MATRIX_SIZE: return "exceeded_adaptive_banded_matrix_size";
        case B200POA_SEQ_LEN_EXCEEDED_MAXIMUM_NODES_PER_WINDOW: return "seq_len_exceeded_maximum_nodes_per_window";
        case B200POA_LOOP_COUNT_EXCEEDED_UPPER_BOUND: return "loop_count_exceeded_upper_bound";
        case B200POA_OUTPUT_TYPE_UNAVAILABLE: return "output_type_unavailable";
        case B200POA_GENERIC_ERROR: return "generic_error";
        case B200POA_ALIGNED_COUNT_EXCEEDED: return "aligned_count_exceeded";
        case B200POA_SCORE_RANGE_EXCEEDED: return "score_range_exceeded";
        case B200POA_TRACEBACK_LOST: return "traceback_lost";
        case B200POA_PARTIAL_SPAN_UNSUPPORTED: return "partial_span_unsupported";
        case B200POA_INVALID_ARGUMENT: return "invalid_argument";
        case B200POA_CUDA_ERROR: return "cuda_error";
        default: return "unknown";
    }
}

void b200poa_config_default(b200poa_config* cfg, int32_t max_seq_sz, int32_t max_seq_per_poa,
                            int32_t band_width, int32_t band_mode) {
    /* batch.cu:34-71 */
    cfg->max_sequence_size = max_seq_sz;
    cfg->max_consensus_size = 2 * max_seq_sz;
    cfg->alignment_band_width = (band_width + 127) / 128 * 128;
    cfg->max_sequences_per_poa = max_seq_per_poa;
    cfg->band_mode = band_mode;
    const int32_t mult = (band_mode == B200POA_FULL_BAND) ? 3 : 4;
    cfg->max_nodes_per_graph = (mult * max_seq_sz + 3) / 4 * 4;
}

void b200poa_layer_order(int32_t n, const int32_t* begins, int32_t* rank_out) {
    /* src/window.cpp:78-85 == src/cuda/cudabatch.cpp:96-104: libstdc++ std::sort is not stable, so
     * the SAME call on the SAME initial vector is what reproduces racon's processing order. */
    std::vector<uint32_t> rank;
    rank.reserve(static_cast<size_t>(n));
    for (int32_t i = 0; i < n; ++i) rank.emplace_back(static_cast<uint32_t>(i));
    if (n > 1)
        std::sort(rank.begin() + 1, rank.end(),
                  [&](uint32_t lhs, uint32_t rhs) { return begins[lhs] < begins[rhs]; });
    for (int32_t i = 0; i < n; ++i) rank_out[i] = static_cast<int32_t>(rank[static_cast<size_t>(i)]);
}

int32_t b200poa_batch_create(int32_t device_id, void* stream, size_t max_gpu_mem, int32_t output_mask,
                             const b200poa_config* cfg, int16_t gap_score, int16_t mismatch_score,
                             int16_t match_score, b200poa_batch** out) {
    if (!out || !cfg) return B200POA_INVALID_ARGUMENT;
    *out = nullptr;
    /* batch.cu:64-66,93-98 argument checks */
    if (cfg->max_sequence_size <= 0 || cfg->max_sequences_per_poa <= 0 || cfg->alignment_band_width < 0 ||
        cfg->max_nodes_per_graph < cfg->max_sequence_size || cfg->max_consensus_size < cfg->max_sequence_size ||
        cfg->max_nodes_per_graph > 32768 || cfg->max_sequence_size > 16380 ||
        (cfg->band_mode != B200POA_FULL_BAND && cfg->band_mode != B200POA_STATIC_BAND &&
         cfg->band_mode != B200POA_ADAPTIVE_BAND))
        return B200POA_INVALID_ARGUMENT;
    if (max_gpu_mem == 0) return B200POA_INVALID_ARGUMENT; /* Test_CudapoaBatch.cu: zero memory throws */
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device_id < 0 || device_id >= ndev) return B200POA_CUDA_ERROR;

    DeviceGuard guard(device_id);
    std::unique_ptr<b200poa_batch> b(new (std::nothrow) b200poa_batch()); /* freed on every early return */
    if (!b) return B200POA_GENERIC_ERROR;
    b->id = g_batches++;
    b->device = device_id;
    b->stream = static_cast<cudaStream_t>(stream);
    b->output_mask = output_mask;
    b->cfg = *cfg;

    Params& p = b->p;
    p.max_nodes = cfg->max_nodes_per_graph;
    p.max_edges = poa_edge_capacity(cfg->max_nodes_per_graph);
    p.max_len = cfg->max_sequence_size;
    const int32_t colsP = (p.max_len + 1 + 7) & ~7;
    p.band_width = (cfg->band_mode != B200POA_FULL_BAND) ? ((cfg->alignment_band_width + 7) & ~7) : 0;
    p.adaptive = cfg->band_mode == B200POA_ADAPTIVE_BAND ? 1 : 0;
    /* score rows: the band in static mode; whole rows in full and adaptive mode (a retry may widen up to the matrix) */
    p.stride = (!p.adaptive && p.band_width > 0 && p.band_width < colsP) ? p.band_width : colsP;
    p.max_cons = cfg->max_consensus_size;
    p.match = match_score;
    p.mismatch = mismatch_score;
    p.gap = gap_score;
    p.serial_topsort = std::getenv("B200POA_SERIAL_TOPSORT") ? 1 : 0;
    p.force_cells32 = std::getenv("B200POA_FORCE_CELLS32") ? 1 : 0; /* tests only */
    /* 32-bit score cells (SURVEY 8f-3): the slots are sized for them only when a read within this batch's limits could
     * overflow int16 (worst case: a path through max_nodes columns), which racon's scorings and limits never do */
    p.wide_cells = (p.force_cells32 || !score_range_ok(p, p.max_nodes, p.max_len)) ? 1 : 0;
    p.ring_rows = 8;
    p.ring_stride = p.stride;
    if (p.max_nodes > 65000) return B200POA_INVALID_ARGUMENT;

    Slot probe;
    slot_bind(probe, nullptr, p, &b->slot_bytes);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device_id) != cudaSuccess) return B200POA_CUDA_ERROR;
    b->sm_count = prop.multiProcessorCount;
    /* worst-case shared memory (longest admissible read) must be launchable; the attribute is per function and per
     * device, so it is raised to the device's opt-in limit once and never lowered by a later, smaller batch */
    const SmemGeometry worst = smem_geometry(p, p.max_len);
    if (worst.smem_bytes > (int32_t)prop.sharedMemPerBlockOptin) {
        std::fprintf(stderr, "[b200poa] batch %d: max_sequence_size %d needs %d B of shared memory per block (device limit %zu)\n",
                     b->id, p.max_len, worst.smem_bytes, (size_t)prop.sharedMemPerBlockOptin);
        return B200POA_INVALID_ARGUMENT;
    }
    if (cudaFuncSetAttribute(poa_window_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)prop.sharedMemPerBlockOptin) != cudaSuccess) return B200POA_CUDA_ERROR;
    /* slots are sized for the best occupancy a launch can reach (short reads => small profile) */
    int blocks_per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, poa_window_kernel, 32, 4096) != cudaSuccess) return B200POA_CUDA_ERROR;
    if (const char* env = std::getenv("B200POA_BLOCKS_PER_SM")) {
        int v = std::atoi(env);
        if (v > 0 && v < blocks_per_sm) blocks_per_sm = v;
    }
    if (blocks_per_sm < 1) return B200POA_INVALID_ARGUMENT;
    b->blocks_per_sm = blocks_per_sm;
    int64_t want_slots = (int64_t)blocks_per_sm * prop.multiProcessorCount;

    /* memory plan: at most half of the budget for slots, the rest for the arena + outputs */
    int64_t slots_by_mem = (int64_t)((max_gpu_mem / 2) / b->slot_bytes);
    if (slots_by_mem < 1) {
        std::fprintf(stderr, "[b200poa] batch %d: %.2f GB is not enough for one window workspace (%.2f MB)\n",
                     b->id, max_gpu_mem / 1073741824.0, b->slot_bytes / 1048576.0);
        return B200POA_INVALID_ARGUMENT;
    }
    b->n_slots = (int32_t)std::min(want_slots, slots_by_mem);
    size_t rest = max_gpu_mem - (size_t)b->n_slots * b->slot_bytes;
    const bool want_msa = (output_mask & B200POA_OUTPUT_MSA) != 0;
    if (want_msa) { /* the MSA arena: a quarter of what the slots leave, at most 4 GiB (B200POA_MSA_ARENA_MB overrides);
                       never less than one worst-case window */
        size_t cap_msa = std::min<size_t>(rest / 4, (size_t)4 << 30);
        if (const char* env = std::getenv("B200POA_MSA_ARENA_MB")) cap_msa = (size_t)std::atoll(env) << 20;
        const size_t one = ((size_t)cfg->max_sequences_per_poa * (size_t)cfg->max_consensus_size + 15) & ~(size_t)15;
        if (cap_msa < one) cap_msa = one;
        if (cap_msa >= rest) return B200POA_INVALID_ARGUMENT;
        b->msa_cap = cap_msa;
        rest -= cap_msa;
    }
    /* staging is pinned host memory too: keep it bounded (B200POA_MAX_STAGING_MB, default 3 GiB) */
    size_t cap = 3ull << 30;
    if (const char* env = std::getenv("B200POA_MAX_STAGING_MB")) cap = (size_t)std::atoll(env) << 20;
    if (rest > cap) rest = cap;
    /* per window: outputs 3*max_cons + ~64 B tables; per base: 2 B; per sequence: 8 B */
    const size_t out_per_win = (size_t)p.max_cons * 3 + 64;
    int64_t max_poas = (int64_t)(rest / 4 / out_per_win);
    if (max_poas < 1) max_poas = 1;
    if (max_poas > (1 << 22)) max_poas = 1 << 22;
    b->max_poas = (int32_t)max_poas;
    size_t arena = (rest - (size_t)max_poas * out_per_win) / (want_msa ? 4 : 2); /* bases + weights (+ the 16-bit path arena) */
    arena = arena / 10 * 9; /* 10% of the arena budget goes to the sequence offset table */
    if (arena < (size_t)p.max_len * 4) arena = (size_t)p.max_len * 4;
    b->arena_cap = (int64_t)arena;
    b->max_seqs = std::max<int64_t>((int64_t)(arena / 10 / 8), 1024) + max_poas;

    const int32_t ast = alloc_batch_memory(b.get());
    if (ast != B200POA_SUCCESS) return ast;
    b->seq_off.h()[0] = 0;
    b->win_seq_off.h()[0] = 0;
    b->cost.reserve((size_t)b->max_poas);
    *out = b.release();
    return B200POA_SUCCESS;
}

int32_t b200poa_batch_add_group(b200poa_batch* b, const b200poa_entry* entries, int32_t n, int32_t* per_seq_status) {
    if (!b || !entries || n <= 0) return B200POA_INVALID_ARGUMENT;
    if (b->ext_bases) return B200POA_INVALID_ARGUMENT; /* a batch is either staged or direct until its next reset */
    auto get = [&](int32_t i, StagedSeq& q) {
        q.seq = entries[i].seq;
        q.w = entries[i].weights;
        q.len = entries[i].length;
        q.bg = entries[i].begin;
        q.en = entries[i].end;
        q.host_off = 0;
        q.wmode = WMODE_UNKNOWN;
    };
    return stage_window<false>(b, n, get, per_seq_status, nullptr);
}

int32_t b200poa_batch_add_windows(b200poa_batch* b, int64_t n_windows, int64_t first,
                                  const int64_t* win_seq_off, const int64_t* seq_off,
                                  const uint8_t* bases, const int8_t* weights,
                                  const uint8_t* has_weights, const int32_t* begins,
                                  const int32_t* ends, int64_t* n_added, int32_t* seqs_added) {
    return add_windows_impl<false>(b, n_windows, first, win_seq_off, seq_off, bases, weights, has_weights, nullptr, begins,
                                   ends, n_added, seqs_added);
}

int32_t b200poa_batch_add_windows_pinned(b200poa_batch* b, int64_t n_windows, int64_t first,
                                         const int64_t* win_seq_off, const int64_t* seq_off,
                                         const uint8_t* bases, const int8_t* weights,
                                         const uint8_t* has_weights, const int64_t* weight_mode,
                                         const int32_t* begins, const int32_t* ends, int64_t* n_added,
                                         int32_t* seqs_added) {
    if (!weight_mode) return B200POA_INVALID_ARGUMENT;
    return add_windows_impl<true>(b, n_windows, first, win_seq_off, seq_off, bases, weights, has_weights, weight_mode, begins,
                                  ends, n_added, seqs_added);
}

void b200poa_weight_modes(int64_t n_sequences, const int64_t* seq_off, const int8_t* weights, const uint8_t* has_weights,
                          int64_t* weight_mode) {
    for (int64_t s = 0; s < n_sequences; ++s) {
        if (!has_weights[s]) {
            weight_mode[s] = -1 - 1; /* no quality string: weight 1 (window.cpp:105-107) */
            continue;
        }
        const int8_t* w = weights + seq_off[s];
        const int64_t len = seq_off[s + 1] - seq_off[s];
        bool constant = true;
        for (int64_t k = 1; k < len && constant; ++k) constant = w[k] == w[0];
        weight_mode[s] = (constant && len > 0) ? -1 - (int64_t)w[0] : 0;
    }
}

int32_t b200poa_batch_total_poas(const b200poa_batch* b) { return b ? b->poa_count : 0; }
int32_t b200poa_batch_id(const b200poa_batch* b) { return b ? b->id : -1; }

int32_t b200poa_batch_upload(b200poa_batch* b) {
    if (!b) return B200POA_INVALID_ARGUMENT;
    if (b->poa_count == 0) return B200POA_SUCCESS;
    DeviceGuard g(b->device);
    /* longest-first work list */
    std::iota(b->work.h(), b->work.h() + b->poa_count, 0);
    std::stable_sort(b->work.h(), b->work.h() + b->poa_count,
                     [&](int32_t x, int32_t y) { return b->cost[(size_t)x] > b->cost[(size_t)y]; });
    const size_t W = (size_t)b->poa_count, S = (size_t)b->seq_count;
    int64_t weight_bytes = b->weight_count;
    if (b->ext_bases) { /* direct mode: the caller's pinned arena range goes up as it is */
        CU_TRY(cudaMemcpyAsync(b->bases.d(), b->ext_bases + b->ext_lo, (size_t)b->base_count, cudaMemcpyHostToDevice, b->stream));
        weight_bytes = b->ext_any_weights ? b->base_count : 0;
        if (weight_bytes > 0)
            CU_TRY(cudaMemcpyAsync(b->weights.d(), b->ext_weights + b->ext_lo, (size_t)weight_bytes, cudaMemcpyHostToDevice, b->stream));
    } else {
        CU_TRY(b->bases.upload((size_t)b->base_count, b->stream));
        if (weight_bytes > 0) /* only sequences with non-constant weights carry bytes */
            CU_TRY(b->weights.upload((size_t)weight_bytes, b->stream));
    }
    CU_TRY(b->seq_off.upload(S, b->stream));
    CU_TRY(b->seq_len.upload(S, b->stream));
    CU_TRY(b->w_off.upload(S, b->stream));
    CU_TRY(b->seq_begin.upload(S, b->stream));
    CU_TRY(b->seq_end.upload(S, b->stream));
    CU_TRY(b->win_seq_off.upload(W + 1, b->stream));
    CU_TRY(b->win_flags.upload(W, b->stream));
    CU_TRY(b->win_trim_nseq.upload(W, b->stream));
    CU_TRY(b->work.upload(W, b->stream));
    b->h2d_bytes = b->base_count + weight_bytes + (int64_t)(S * 28 + (W + 1) * 4 + W * 12);
    b->uploaded = true;
    return B200POA_SUCCESS;
}

int32_t b200poa_batch_launch(b200poa_batch* b) {
    if (!b) return B200POA_INVALID_ARGUMENT;
    if (b->poa_count == 0) return B200POA_SUCCESS;
    if (!b->uploaded) return B200POA_INVALID_ARGUMENT;
    DeviceGuard g(b->device);
    CU_TRY(cudaMemsetAsync(b->cursor.d(), 0, 2 * sizeof(int32_t), b->stream));
    if (b->msa_cursor.d()) CU_TRY(cudaMemsetAsync(b->msa_cursor.d(), 0, sizeof(unsigned long long), b->stream));
    KernelArgs a;
    a.p = b->p;
    a.slab = static_cast<uint8_t*>(b->slab.p);
    a.slot_bytes = b->slot_bytes;
    a.n_windows = b->poa_count;
    a.work = b->work.d();
    a.cursor = b->cursor.d();
    a.bases = b->bases.d();
    a.weights = b->weights.d();
    a.seq_off = b->seq_off.d();
    a.seq_len = b->seq_len.d();
    a.w_off = b->w_off.d();
    a.win_seq_off = b->win_seq_off.d();
    a.win_flags = b->win_flags.d();
    a.win_trim_nseq = b->win_trim_nseq.d();
    a.seq_begin = b->seq_begin.d();
    a.seq_end = b->seq_end.d();
    a.out_cons = b->cons.d();
    a.out_cov = b->cov.d();
    a.out_len = b->len.d();
    a.out_status = b->status.d();
    a.out_off = b->out_off.d();
    a.out_trim = b->trim.d();
    a.path = static_cast<uint16_t*>(b->path.p);
    a.out_msa = static_cast<uint8_t*>(b->msa.p);
    a.msa_cursor = b->msa_cursor.d();
    a.msa_cap = (unsigned long long)b->msa_cap;
    a.out_msa_off = b->msa_off.d();
    a.out_msa_cols = b->msa_cols.d();
    a.out_msa_status = b->msa_status.d();
    a.p.skip_consensus = (b->output_mask & B200POA_OUTPUT_CONSENSUS) ? 0 : 1;
    /* shared memory geometry follows the longest read actually staged */
    const SmemGeometry sg = smem_geometry(b->p, b->max_len_staged);
    b->prof_stride = sg.prof_stride;
    b->ring_stride = sg.ring_stride;
    b->ring_rows = sg.ring_rows;
    b->smem_bytes = sg.smem_bytes;
    int occ = 0;
    CU_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, poa_window_kernel, 32, (size_t)b->smem_bytes));
    if (occ < 1) return B200POA_INVALID_ARGUMENT;
    b->blocks_per_sm = occ;
    a.prof_stride = b->prof_stride;
    a.ring_stride = b->ring_stride;
    a.ring_rows = b->ring_rows;
    a.p.ring_rows = b->ring_rows;
    a.p.ring_stride = b->ring_stride;
    a.phase_cycles = static_cast<unsigned long long*>(b->phase.p);
#if POA_FILL_DIGEST
    CU_TRY(cudaMemsetAsync(b->fill_digest.p, 0, (size_t)b->seq_count * sizeof(unsigned long long), b->stream));
    CU_TRY(cudaMemsetAsync(b->fill_count.p, 0, (size_t)b->seq_count * sizeof(int32_t), b->stream));
    a.fill_digest = static_cast<unsigned long long*>(b->fill_digest.p);
    a.fill_count = static_cast<int32_t*>(b->fill_count.p);
#endif
#if POA_ALN_DIGEST
    CU_TRY(cudaMemsetAsync(b->aln_digest.p, 0, (size_t)b->seq_count * sizeof(unsigned long long), b->stream));
    CU_TRY(cudaMemsetAsync(b->aln_count.p, 0, (size_t)b->seq_count * sizeof(int32_t), b->stream));
    a.aln_digest = static_cast<unsigned long long*>(b->aln_digest.p);
    a.aln_count = static_cast<int32_t*>(b->aln_count.p);
#endif
#if POA_GRAPH_DIGEST
    {
        const size_t ns = (size_t)b->seq_count, nw = (size_t)b->poa_count;
        CU_TRY(cudaMemsetAsync(b->graph_digest.p, 0, ns * sizeof(unsigned long long), b->stream));
        CU_TRY(cudaMemsetAsync(b->graph_nodes.p, 0, ns * sizeof(int32_t), b->stream));
        CU_TRY(cudaMemsetAsync(b->graph_edges.p, 0, ns * sizeof(int32_t), b->stream));
        CU_TRY(cudaMemsetAsync(b->sub_digest.p, 0, ns * sizeof(unsigned long long), b->stream));
        CU_TRY(cudaMemsetAsync(b->sub_count.p, 0, ns * sizeof(int32_t), b->stream));
        CU_TRY(cudaMemsetAsync(b->cons_digest.p, 0, 2 * nw * sizeof(unsigned long long), b->stream));
        CU_TRY(cudaMemsetAsync(b->cons_rounds.p, 0, nw * sizeof(int32_t), b->stream));
    }
    a.graph_digest = static_cast<unsigned long long*>(b->graph_digest.p);
    a.graph_nodes = static_cast<int32_t*>(b->graph_nodes.p);
    a.graph_edges = static_cast<int32_t*>(b->graph_edges.p);
    a.sub_digest = static_cast<unsigned long long*>(b->sub_digest.p);
    a.sub_count = static_cast<int32_t*>(b->sub_count.p);
    a.cons_digest = static_cast<unsigned long long*>(b->cons_digest.p);
    a.cons_rounds = static_cast<int32_t*>(b->cons_rounds.p);
#endif
    /* persistent grid: one warp per resident slot */
    const int grid = std::max(1, std::min(std::min(b->n_slots, occ * b->sm_count), b->poa_count));
    poa_window_kernel<<<grid, 32, (size_t)b->smem_bytes, b->stream>>>(a);
    CU_TRY(cudaGetLastError());
    b->launches += 1;
    b->results_fetched = false;
    b->msa_fetched = false;
    return B200POA_SUCCESS;
}

/* D2H, first half: the per-window tables (length, status, arena offset, trim span) and the arena fill level.  The
 * compact consensus (and coverage) bytes follow in b200poa_batch_get_consensus, once the fill level is known: exactly
 * sum(len) bytes cross PCIe instead of poa_count full rows (the reference copies max_poas full rows,
 * cudapoa_batch.cuh:213-222). */
int32_t b200poa_batch_download(b200poa_batch* b) {
    if (!b) return B200POA_INVALID_ARGUMENT;
    if (b->poa_count == 0) return B200POA_SUCCESS;
    DeviceGuard g(b->device);
    const size_t W = (size_t)b->poa_count;
    CU_TRY(b->len.download(W, b->stream));
    CU_TRY(b->status.download(W, b->stream));
    CU_TRY(b->out_off.download(W, b->stream));
    CU_TRY(b->trim.download(W, b->stream));
    CU_TRY(b->cursor.download(2, b->stream));
    if (b->msa.p) { /* the MSA tables; the rows follow in b200poa_batch_get_msa once the fill level is known */
        CU_TRY(b->msa_off.download(W, b->stream));
        CU_TRY(b->msa_cols.download(W, b->stream));
        CU_TRY(b->msa_status.download(W, b->stream));
        CU_TRY(b->msa_cursor.download(1, b->stream));
    }
    return B200POA_SUCCESS;
}

int32_t b200poa_batch_generate(b200poa_batch* b) {
    int32_t st = b200poa_batch_upload(b);
    if (st != B200POA_SUCCESS) return st;
    st = b200poa_batch_launch(b);
    if (st != B200POA_SUCCESS) return st;
    return b200poa_batch_download(b);
}

int32_t b200poa_batch_get_consensus(b200poa_batch* b, const uint8_t** cons, const uint16_t** cov,
                                    const int32_t** lens, const int32_t** status, const int32_t** offsets,
                                    const int32_t** trim) {
    if (!b) return B200POA_INVALID_ARGUMENT;
    if (!(b->output_mask & B200POA_OUTPUT_CONSENSUS)) return B200POA_OUTPUT_TYPE_UNAVAILABLE; /* cudapoa_batch.cuh:205-209 */
    DeviceGuard g(b->device);
    CU_TRY(cudaStreamSynchronize(b->stream));
    if (b->poa_count > 0 && !b->results_fetched) { /* D2H, second half: the used part of the compact arenas */
        const size_t used = (size_t)(uint32_t)b->cursor.h()[1];
        b->out_elems = (int64_t)used;
        if (used > 0) {
            CU_TRY(b->cons.download(used, b->stream));
            if (b->download_coverage) CU_TRY(b->cov.download(used, b->stream));
            CU_TRY(cudaStreamSynchronize(b->stream));
        }
        b->d2h_bytes = (int64_t)b->poa_count * 16 + 8 + (int64_t)used * (b->download_coverage ? 3 : 1);
        b->results_fetched = true;
    }
    if (cons) *cons = b->cons.h();
    if (cov) *cov = b->download_coverage ? b->cov.h() : nullptr;
    if (lens) *lens = b->len.h();
    if (status) *status = b->status.h();
    if (offsets) *offsets = b->out_off.h();
    if (trim) *trim = b->trim.h();
    return B200POA_SUCCESS;
}

int32_t b200poa_batch_get_msa(b200poa_batch* b, const uint8_t** msa, const int64_t** offsets, const int32_t** n_rows,
                              const int32_t** n_cols, const int32_t** status) {
    if (!b) return B200POA_INVALID_ARGUMENT;
    if (!(b->output_mask & B200POA_OUTPUT_MSA)) return B200POA_OUTPUT_TYPE_UNAVAILABLE; /* cudapoa_batch.cuh:263-267 */
    DeviceGuard g(b->device);
    CU_TRY(cudaStreamSynchronize(b->stream));
    if (b->poa_count > 0 && !b->msa_fetched) { /* exactly the bytes the launch used (the reference copies
                                                  max_poas x max_sequences_per_poa x max_consensus_size, :271-275) */
        const size_t used = (size_t)*b->msa_cursor.h();
        if (!b->h_msa.reserve(used)) return B200POA_CUDA_ERROR;
        if (used > 0) {
            CU_TRY(cudaMemcpyAsync(b->h_msa.p, b->msa.p, used, cudaMemcpyDeviceToHost, b->stream));
            CU_TRY(cudaStreamSynchronize(b->stream));
        }
        b->d2h_bytes += (int64_t)used + (int64_t)b->poa_count * 16 + 8;
        b->msa_fetched = true;
    }
    static_assert(sizeof(long long) == sizeof(int64_t), "offset table type");
    if (msa) *msa = b->h_msa.p;
    if (offsets) *offsets = reinterpret_cast<const int64_t*>(b->msa_off.h());
    if (n_rows) *n_rows = reinterpret_cast<const int32_t*>(b->h_msa_rows.p);
    if (n_cols) *n_cols = b->msa_cols.h();
    if (status) *status = b->msa_status.h();
    return B200POA_SUCCESS;
}

int32_t b200poa_batch_set_option(b200poa_batch* b, int32_t option, int64_t value) {
    if (!b) return B200POA_INVALID_ARGUMENT;
    switch (option) {
        case B200POA_OPT_DOWNLOAD_COVERAGE: b->download_coverage = value != 0; return B200POA_SUCCESS;
        case B200POA_OPT_TRIM_COUNTS_STAGED:
            if (b->poa_count != 0) return B200POA_INVALID_ARGUMENT; /* decided per window at staging */
            b->trim_counts_staged = value != 0;
            return B200POA_SUCCESS;
        default: return B200POA_INVALID_ARGUMENT;
    }
}

int32_t b200poa_batch_reset(b200poa_batch* b) {
    if (!b) return B200POA_INVALID_ARGUMENT;
    b->poa_count = 0;
    b->seq_count = 0;
    b->base_count = 0;
    b->weight_count = 0;
    b->ext_bases = nullptr;
    b->ext_weights = nullptr;
    b->ext_lo = b->ext_hi = 0;
    b->ext_any_weights = false;
    b->cost.clear();
    b->uploaded = false;
    b->results_fetched = false;
    b->msa_fetched = false;
    b->msa_bound = 0;
    b->max_len_staged = 0;
    return B200POA_SUCCESS;
}

void b200poa_batch_destroy(b200poa_batch* b) {
    if (!b) return;
    DeviceGuard g(b->device);
    delete b;
}

int32_t b200poa_batch_phase_cycles(b200poa_batch* b, uint64_t* out, int32_t n) {
    /* diagnostics (B200POA_PHASE_TIMERS=1): cycles per phase summed over warps since creation */
    if (!b || !out || !b->phase.p) return B200POA_OUTPUT_TYPE_UNAVAILABLE;
    unsigned long long h[PH_COUNT];
    DeviceGuard g(b->device);
    CU_TRY(cudaStreamSynchronize(b->stream));
    CU_TRY(cudaMemcpy(h, b->phase.p, sizeof(h), cudaMemcpyDeviceToHost));
    for (int32_t i = 0; i < n && i < PH_COUNT; ++i) out[i] = h[i];
    return B200POA_SUCCESS;
}

int32_t b200poa_batch_get_info(const b200poa_batch* b, b200poa_batch_info* info) {
    if (!b || !info) return B200POA_INVALID_ARGUMENT;
    info->n_slots = b->n_slots;
    info->max_poas = b->max_poas;
    info->arena_capacity = b->arena_cap;
    info->slot_bytes = (int64_t)b->slot_bytes;
    info->device_bytes = (int64_t)b->device_bytes;
    info->staged_bases = b->base_count;
    info->kernel_launches = b->launches;
    info->smem_bytes = b->smem_bytes;
    info->blocks_per_sm = b->blocks_per_sm;
    info->h2d_bytes = b->h2d_bytes;
    info->d2h_bytes = b->d2h_bytes;
    return B200POA_SUCCESS;
}

} // extern "C"

#if POA_FILL_DIGEST
/* test build only (not part of include/b200poa.h): after the last launch, per staged sequence (staging order: windows in
 * add order, each window's sequences in processing order) the sum of the digests of its DP fills and their number, and
 * the score-row ring the launch used.  Synchronises. */
extern "C" int32_t b200poa_debug_fill_digest(b200poa_batch* b, uint64_t* digest, int32_t* count, int64_t n,
                                             int32_t* ring_rows, int32_t* ring_stride) {
    if (!b || !digest || !count || n < b->seq_count) return B200POA_INVALID_ARGUMENT;
    DeviceGuard g(b->device);
    CU_TRY(cudaStreamSynchronize(b->stream));
    CU_TRY(cudaMemcpy(digest, b->fill_digest.p, (size_t)b->seq_count * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    CU_TRY(cudaMemcpy(count, b->fill_count.p, (size_t)b->seq_count * sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (ring_rows) *ring_rows = b->ring_rows;
    if (ring_stride) *ring_stride = b->ring_stride;
    return B200POA_SUCCESS;
}
#endif
#if POA_ALN_DIGEST
/* test build only: after the last launch, per staged sequence (same order as b200poa_debug_fill_digest) aln_digest() of
 * the alignment added to the graph and its entry count; 0 and 0 for backbones and for reads never added.  Synchronises. */
extern "C" int32_t b200poa_debug_aln_digest(b200poa_batch* b, uint64_t* digest, int32_t* count, int64_t n) {
    if (!b || !digest || !count || n < b->seq_count) return B200POA_INVALID_ARGUMENT;
    DeviceGuard g(b->device);
    CU_TRY(cudaStreamSynchronize(b->stream));
    CU_TRY(cudaMemcpy(digest, b->aln_digest.p, (size_t)b->seq_count * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    CU_TRY(cudaMemcpy(count, b->aln_count.p, (size_t)b->seq_count * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return B200POA_SUCCESS;
}
#endif
#if POA_GRAPH_DIGEST
/* test build only: after the last launch, per staged sequence (same order as b200poa_debug_fill_digest) graph_digest()
 * of the graph after the sequence was added and sorted with its node and edge counts (0 once its window stopped on a
 * status), and for partial-span reads sub_digest() of the subgraph's member order with its member count (else 0 and 0);
 * per staged window (add order) cons_digest() after the full scoring pass and after the last round of branch
 * completion, and the number of rounds (0 where no consensus was generated).  Synchronises. */
extern "C" int32_t b200poa_debug_graph_digest(b200poa_batch* b, uint64_t* graph_digest, int32_t* graph_nodes,
                                              int32_t* graph_edges, uint64_t* sub_digest, int32_t* sub_count, int64_t n,
                                              uint64_t* cons_digest, int32_t* cons_rounds, int64_t n_windows) {
    if (!b || !graph_digest || !graph_nodes || !graph_edges || !sub_digest || !sub_count || !cons_digest ||
        !cons_rounds || n < b->seq_count || n_windows < b->poa_count)
        return B200POA_INVALID_ARGUMENT;
    DeviceGuard g(b->device);
    CU_TRY(cudaStreamSynchronize(b->stream));
    const size_t ns = (size_t)b->seq_count, nw = (size_t)b->poa_count;
    CU_TRY(cudaMemcpy(graph_digest, b->graph_digest.p, ns * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    CU_TRY(cudaMemcpy(graph_nodes, b->graph_nodes.p, ns * sizeof(int32_t), cudaMemcpyDeviceToHost));
    CU_TRY(cudaMemcpy(graph_edges, b->graph_edges.p, ns * sizeof(int32_t), cudaMemcpyDeviceToHost));
    CU_TRY(cudaMemcpy(sub_digest, b->sub_digest.p, ns * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    CU_TRY(cudaMemcpy(sub_count, b->sub_count.p, ns * sizeof(int32_t), cudaMemcpyDeviceToHost));
    CU_TRY(cudaMemcpy(cons_digest, b->cons_digest.p, 2 * nw * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    CU_TRY(cudaMemcpy(cons_rounds, b->cons_rounds.p, nw * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return B200POA_SUCCESS;
}
#endif

#if defined(B200POA_SUBTIMERS)
/* experiments only (not part of include/b200poa.h): sub-phase cycle counters since the last call */
extern "C" int32_t b200poa_debug_subtimers(unsigned long long* out32) {
    if (cudaMemcpyFromSymbol(out32, b200poa::g_subtimers, sizeof(unsigned long long) * 32) != cudaSuccess) return 1;
    unsigned long long zero[32] = {0};
    return cudaMemcpyToSymbol(b200poa::g_subtimers, zero, sizeof(zero)) != cudaSuccess;
}
#endif
