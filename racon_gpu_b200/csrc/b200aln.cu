/*
 * b200aln.cu -- C ABI (include/b200aln.h) + batch runtime + kernel launches of the overlap aligner (aln_core.cuh).
 *
 * Replaces what racon's CUDABatchAligner reaches through cudaaligner's Aligner (src/cuda/cudaaligner.cpp:50-98 ->
 * vendor/GenomeWorks/cudaaligner/src/aligner_global*.cpp, hirschberg_myers_gpu.cu), with the results of racon's CPU
 * path (edlib, src/overlap.cpp:205-224).  Runtime design:
 *   - per-RESIDENT-WARP workspaces ("slots": two distance columns, the stripe hand-over row, 1 MB of leaf records),
 *     reused by every sub-problem the warp takes from the level's list; persistent grids, one atomic cursor per launch;
 *   - per-resident-BLOCK team workspaces (hand-over rows, code rows, the two middle columns) for sub-problems that a team
 *     of warps takes (aln_split_team_kernel);
 *   - the Hirschberg recursion is level-synchronous over the whole batch and its lists live on the device: per level at
 *     most one team launch and one one-warp launch (huge sub-problems of a saturated level: teams on a side stream) and
 *     one 12-byte read-back (how many sub-problems of each shape the next level has);
 *   - results leave the device compact: CIGAR text and / or breaking points formed on the device and bump-allocated into
 *     arenas, a 48-byte record per alignment -- not (n + m) bytes per alignment; run starts only when somebody asks;
 *   - with a layer cut set, racon's window layers are cut from the breaking points on the device (layer_cut.cuh) and only
 *     their 32-byte records come back; the layer bytes stay in the query arena for a POA batch to gather;
 *   - uploads come from the batch's pinned staging copy or straight from the caller's page-locked columnar buffers (view);
 *   - a pool (b200aln_aligner_*) runs several such batches per device on every device, one host thread each.
 * Nothing here falls back to a CPU aligner; a CUDA failure is a status, not a different code path.
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "../../include/b200aln.h"
#include "aln_core.cuh"
#include "cuda_buffers.hpp"
#include "host/aln_admission.hpp"
#include "host/aln_levels.hpp"
#include "layer_cut.cuh"

using namespace b200aln;
using namespace b200buf;

static_assert(sizeof(CutLayer) == sizeof(b200aln_layer) && offsetof(CutLayer, window) == offsetof(b200aln_layer, window) &&
                  offsetof(CutLayer, overlap) == offsetof(b200aln_layer, overlap),
              "the layer records leave the device as they are");

namespace {

enum { /* int32 words of the device counter block */
    CT_CURSOR = 0,      /* [128] one work cursor per launch                                  */
    CT_NOPEN = 128,     /* [32][4] sub-problems open at level k by shape (3 adjacent words + pad) */
    CT_NLEAVES = 256,
    CT_OVERFLOW = 257,
    CT_RUNS = 258,      /* u64: entries used in the runs arena                               */
    CT_CELLS = 260,     /* u64: distance-matrix cells computed                               */
    CT_TEXT = 262,      /* u64: bytes used in the CIGAR text arena                           */
    CT_BP = 264,        /* u64: (t, q) pairs reserved in the breaking-point arena            */
    CT_WORDS = 268,
    MAX_LEVELS = 31
};

struct AlnKernelArgs {
    uint8_t* slab;
    size_t slot_bytes;
    uint8_t* team_slab; /* n_team_blocks * team_slot_bytes */
    size_t team_slot_bytes;
    int32_t max_len;
    const uint8_t* seq;
    const AlnJob* jobs;
    uint8_t* ops;
    AlnResult* res;
    int32_t* counters;
#if ALN_SPLIT_DIGEST
    AlnSplitRec* log; /* [log_cap] one record per split attempt (b200aln_debug_split_log) */
    int32_t* log_count; /* records appended; more than log_cap: the log overflowed */
    int32_t log_cap;
#endif
#if ALN_LEAF_DIGEST
    AlnLeafRec* leaf_log;    /* [leaf_log_cap] one record per leaf (b200aln_debug_leaf_log) */
    int32_t* leaf_log_count; /* records appended; more than leaf_log_cap: the log overflowed */
    int32_t leaf_log_cap;
#endif
};

/* what one split launch works through: up to three lists of a level, one after the other (largest shapes first) */
struct AlnWork {
    const AlnRect* list[ALN_CLASSES];
    int32_t n[ALN_CLASSES];
    int32_t total;
#if ALN_SPLIT_DIGEST
    int32_t level, path; /* for the split log */
#endif
};
__device__ __forceinline__ AlnRect work_item(const AlnWork& w, int32_t k) {
    if (k < w.n[0]) return w.list[0][k];
    k -= w.n[0];
    if (k < w.n[1]) return w.list[1][k];
    return w.list[2][k - w.n[1]];
}
#ifndef ALN_MIN_BLOCKS
#define ALN_MIN_BLOCKS 16 /* 32 warps per SM => at most 64 registers per thread */
#endif

__device__ __forceinline__ void bind_slot(const AlnKernelArgs& a, AlnSlot& s) {
    const size_t slot = (size_t)blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
    aln_slot_bind(s, a.slab + slot * a.slot_bytes, a.max_len, nullptr);
}
__device__ __forceinline__ void bind_eq(EqTab& eq, uint64_t* tab) {
    eq.sa = (uint32_t)__cvta_generic_to_shared(tab + (threadIdx.x >> 5) * ALN_EQ_WORDS);
}
__device__ __forceinline__ int32_t take_work(int32_t* cursor) {
    int32_t t = 0;
    if ((threadIdx.x & 31u) == 0u) t = atomicAdd(cursor, 1);
    return __shfl_sync(0xffffffffu, t, 0);
}

#if ALN_SPLIT_DIGEST
/* test build: appends the record of one split attempt; whole warp (the hashes), lane 0 holds `sp` */
__device__ __noinline__ void log_split(const AlnKernelArgs& a, const AlnRect& r, int32_t band, int32_t attempt, int32_t level,
                                       int32_t path, int32_t flags, const AlnSplit& sp, const int32_t* Lc, const int32_t* Rr) {
    const unsigned long long lh = aln_col_digest(Lc, r.n), rh = aln_col_digest(Rr, r.n);
    if ((threadIdx.x & 31u) == 0u) {
        const int32_t k = atomicAdd(a.log_count, 1);
        if (k < a.log_cap) {
            AlnSplitRec x;
            x.aln = r.aln;
            x.r0 = r.r0;
            x.c0 = r.c0;
            x.n = r.n;
            x.m = r.m;
            x.band = band;
            x.attempt = attempt;
            x.level = level;
            x.path = path;
            x.flags = flags;
            x.r = sp.r;
            x.ls = sp.ls;
            x.rs = sp.rs;
            x.best = sp.best;
            x.pad[0] = x.pad[1] = 0;
            x.lc_hash = lh;
            x.rr_hash = rh;
            a.log[k] = x;
        }
    }
    __syncwarp();
}
#endif

/* one Hirschberg level: every open sub-problem is split, its children are filed for the next level or as leaves */
__global__ void __launch_bounds__(32 * WARPS_PER_BLOCK, ALN_MIN_BLOCKS) aln_split_kernel(const AlnKernelArgs a, const AlnWork work,
                                                                                        const AlnLists next, int32_t* cursor) {
    __shared__ uint64_t eq_tab[WARPS_PER_BLOCK * ALN_EQ_WORDS];
    AlnSlot s;
    bind_slot(a, s);
    EqTab eq;
    bind_eq(eq, eq_tab);
    for (;;) {
        const int32_t k = take_work(cursor);
        if (k >= work.total) break;
        const AlnRect r = work_item(work, k);
        const AlnJob job = a.jobs[r.aln];
        AlnSplit sp;
        int64_t cells = aln_split(s, eq, a.seq + job.q_off + r.r0, a.seq + job.t_off + r.c0, r.n, r.m, aln_band_of(r.best), &sp);
#if ALN_SPLIT_DIGEST
        log_split(a, r, aln_band_of(r.best), 0, work.level, work.path, 0, sp, s.Lc, s.Rr);
#endif
        if (r.top & ALN_GUESS) { /* the host's guess was too small? then nothing of that pass can be trusted: no band */
            const int32_t found = __shfl_sync(0xffffffffu, sp.best, 0);
            if (found > r.best) {
                cells += aln_split(s, eq, a.seq + job.q_off + r.r0, a.seq + job.t_off + r.c0, r.n, r.m, -1, &sp);
#if ALN_SPLIT_DIGEST
                log_split(a, r, -1, 1, work.level, work.path, 0, sp, s.Lc, s.Rr);
#endif
            }
        }
        if ((threadIdx.x & 31u) == 0u) {
            if (r.top & ALN_TOP) a.res[r.aln].score = sp.best;
            AlnRect ul, lr;
            if (aln_children(r, sp, ul, lr)) {
                aln_push(next, ul);
                aln_push(next, lr);
            } else {
                a.res[r.aln].status = B200ALN_GENERIC_ERROR;
            }
            atomicAdd(reinterpret_cast<unsigned long long*>(a.counters + CT_CELLS), (unsigned long long)cells);
        }
        __syncwarp();
    }
}

/* The same for TALL sub-problems when a level has too few of them to fill the device one warp each: a block per
 * sub-problem, a team of ALN_TEAM warps on the forward pass and another on the backward pass at the same time, the
 * stripes of a pass pipelined through the team (aln_core.cuh: Teams).  Block workspace: 2 x ALN_TEAM hand-over rows, two
 * code rows, the two middle columns. */
#ifndef ALN_TEAM_WAVES
#define ALN_TEAM_WAVES 4 /* teams while a level's tall sub-problems fit this many waves of team blocks */
#endif
struct TeamSlot {
    uint32_t* hrow[2];
    uint8_t* tcode[2];
    int32_t *Lc, *Rr;
};
__host__ __device__ inline void team_slot_bind(TeamSlot& t, uint8_t* base, int32_t max_len, size_t* total_out) {
    size_t o = 0;
    auto carve = [&](size_t bytes) {
        o = (o + 255) / 256 * 256;
        uint8_t* p = base ? base + o : nullptr;
        o += bytes;
        return p;
    };
    const size_t hrow = (size_t)aln_hrow_words(max_len);
    for (int k = 0; k < 2; ++k) t.hrow[k] = reinterpret_cast<uint32_t*>(carve(sizeof(uint32_t) * hrow * ALN_TEAM));
    for (int k = 0; k < 2; ++k) t.tcode[k] = carve((size_t)max_len + 192);
    t.Lc = reinterpret_cast<int32_t*>(carve(sizeof(int32_t) * ((size_t)max_len + 2)));
    t.Rr = reinterpret_cast<int32_t*>(carve(sizeof(int32_t) * ((size_t)max_len + 2)));
    o = (o + 255) / 256 * 256;
    if (total_out) *total_out = o;
}
__global__ void __launch_bounds__(64 * ALN_TEAM, 1024 / (64 * ALN_TEAM)) aln_split_team_kernel(const AlnKernelArgs a, const AlnWork work,
                                                                                                  const AlnLists next, int32_t* cursor) {
    __shared__ uint64_t eq_tab[2 * ALN_TEAM * ALN_EQ_WORDS];
    __shared__ unsigned long long prog[2 * ALN_TEAM];
    __shared__ int32_t s_k, s_redo;
#if ALN_SPLIT_DIGEST
    __shared__ int32_t s_timed_out;
    if (threadIdx.x == 0) s_timed_out = 0;
#endif
    TeamSlot ts;
    team_slot_bind(ts, a.team_slab + (size_t)blockIdx.x * a.team_slot_bytes, a.max_len, nullptr);
    const int warp = (int)(threadIdx.x >> 5), side = warp / ALN_TEAM; /* side 0: forward pass, side 1: backward pass */
    EqTab eq;
    bind_eq(eq, eq_tab);
    TeamCtx team;
    team.w = warp % ALN_TEAM;
    team.n = ALN_TEAM;
    team.bar_id = 1 + side;
    team.prog_sa = (uint32_t)__cvta_generic_to_shared(prog + side * ALN_TEAM);
#if ALN_SPLIT_DIGEST
    team.timed_out = &s_timed_out;
#endif
    const int32_t hrow_words = (int32_t)aln_hrow_words(a.max_len);
    for (;;) {
        if (threadIdx.x == 0) s_k = atomicAdd(cursor, 1);
        __syncthreads();
        const int32_t k = s_k;
        if (k >= work.total) break;
        const AlnRect r = work_item(work, k);
        const AlnJob job = a.jobs[r.aln];
        const uint8_t* q = a.seq + job.q_off + r.r0;
        const uint8_t* t = a.seq + job.t_off + r.c0;
        const int32_t lh = r.m / 2, rh = r.m - lh; /* edlib.cpp:1216-1217 */
        AlnSplit sp;
        for (int attempt = 0; attempt < 2; ++attempt) {
            /* banded first when the sub-problem's optimum is known or guessed; a guess that proves too small: once more, whole */
            const int32_t band = attempt == 0 ? aln_band_of(r.best) : -1;
            int64_t cells;
            if (side == 0)
                cells = myers_pass<true>(SeqView{q, 1}, r.n, SeqView{t, 1}, lh, band, team, ts.hrow[0], hrow_words, ts.tcode[0], eq, ts.Lc,
                                         nullptr, nullptr);
            else
                cells = myers_pass<true>(SeqView{q + (r.n - 1), -1}, r.n, SeqView{t + (r.m - 1), -1}, rh, band, team, ts.hrow[1],
                                         hrow_words, ts.tcode[1], eq, ts.Rr, nullptr, nullptr);
            if ((threadIdx.x & 31u) == 0u && cells)
                atomicAdd(reinterpret_cast<unsigned long long*>(a.counters + CT_CELLS), (unsigned long long)cells);
            __threadfence_block();
            __syncthreads(); /* both middle columns are complete */
            if (warp == 0) {
                aln_split_rule(ts.Lc, ts.Rr, r.n, r.m, &sp);
                if ((threadIdx.x & 31u) == 0u) s_redo = (attempt == 0 && (r.top & ALN_GUESS) && sp.best > r.best) ? 1 : 0;
#if ALN_SPLIT_DIGEST
                log_split(a, r, band, attempt, work.level, work.path, s_timed_out ? ALN_REC_TIMEOUT : 0, sp, ts.Lc, ts.Rr);
                if ((threadIdx.x & 31u) == 0u) s_timed_out = 0; /* before the next attempt's passes (the barrier below) */
#endif
            }
            __syncthreads();
            if (!s_redo) break;
        }
        if (warp == 0 && (threadIdx.x & 31u) == 0u) {
            if (r.top & ALN_TOP) a.res[r.aln].score = sp.best;
            AlnRect ul, lr;
            if (aln_children(r, sp, ul, lr)) {
                aln_push(next, ul);
                aln_push(next, lr);
            } else {
                a.res[r.aln].status = B200ALN_GENERIC_ERROR;
            }
        }
        __syncthreads(); /* the columns and s_k are free again */
    }
}

/* all leaves of all levels: the matrix as block records, the walk back, operations into the alignment's region */
__global__ void __launch_bounds__(32 * WARPS_PER_BLOCK, ALN_MIN_BLOCKS) aln_leaf_kernel(const AlnKernelArgs a, const AlnRect* leaves,
                                                                        int32_t n_leaves, int32_t* cursor) {
    __shared__ uint64_t eq_tab[WARPS_PER_BLOCK * ALN_EQ_WORDS];
    AlnSlot s;
    bind_slot(a, s);
    EqTab eq;
    bind_eq(eq, eq_tab);
    for (;;) {
        const int32_t k = take_work(cursor);
        if (k >= n_leaves) break;
        const AlnRect r = leaves[k];
        const AlnJob job = a.jobs[r.aln];
#if ALN_LEAF_DIGEST
        AlnLeafRec lr;
#endif
        const int64_t cells = aln_leaf(s, eq, a.seq + job.q_off + r.r0, a.seq + job.t_off + r.c0, r.n, r.m,
                                       (r.top & ALN_GUESS) ? -1 : aln_band_of(r.best), a.ops + job.ops_off + r.r0 + r.c0,
                                       (r.top & ALN_TOP) ? &a.res[r.aln].score : nullptr
#if ALN_LEAF_DIGEST
                                       , &lr
#endif
        );
        if ((threadIdx.x & 31u) == 0u)
            atomicAdd(reinterpret_cast<unsigned long long*>(a.counters + CT_CELLS), (unsigned long long)cells);
#if ALN_LEAF_DIGEST
        if ((threadIdx.x & 31u) == 0u) { /* lane 0 holds the record */
            lr.aln = r.aln;
            lr.r0 = r.r0;
            lr.c0 = r.c0;
            lr.top = r.top;
            const int32_t at = atomicAdd(a.leaf_log_count, 1);
            if (at < a.leaf_log_cap) a.leaf_log[at] = lr;
        }
#endif
        __syncwarp();
    }
}

/* operations -> run starts -> CIGAR text and / or breaking points, all bump-allocated into compact arenas */
struct AlnOutArgs {
    uint32_t* runs;
    unsigned long long runs_cap;
    uint8_t* text; /* null: no CIGAR text wanted */
    unsigned long long text_cap;
    uint32_t* bp;  /* null / window_length 0: no breaking points wanted */
    unsigned long long bp_cap; /* pairs */
    int32_t window_length;
};
__global__ void __launch_bounds__(32 * WARPS_PER_BLOCK) aln_cigar_kernel(const AlnKernelArgs a, int32_t n_alignments,
                                                                         const AlnOutArgs o, int32_t* cursor) {
    const bool lane0 = (threadIdx.x & 31u) == 0u;
    AlnSlot s;
    bind_slot(a, s);
    for (;;) {
        const int32_t k = take_work(cursor);
        if (k >= n_alignments) break;
        const AlnJob job = a.jobs[k];
        const uint8_t* ops = a.ops + job.ops_off;
        int32_t n_ops = 0;
        const int32_t n_runs = aln_runs(ops, job.n + job.m, nullptr, n_ops);
        unsigned long long off = 0;
        if (lane0) off = atomicAdd(reinterpret_cast<unsigned long long*>(a.counters + CT_RUNS), (unsigned long long)n_runs);
        off = __shfl_sync(0xffffffffu, off, 0);
        bool ok = off + (unsigned long long)n_runs <= o.runs_cap;
        AlnResult r = a.res[k]; /* score and status were written by the split / leaf kernels */
        if (ok) {
            aln_runs(ops, job.n + job.m, o.runs + off, n_ops);
            r.n_runs = n_runs;
            r.n_ops = n_ops;
            r.runs_off = (int64_t)off;
        }
        if (ok && o.text) {
            const int32_t bytes = aln_cigar_text(o.runs + off, n_runs, n_ops, nullptr);
            unsigned long long toff = 0;
            if (lane0) toff = atomicAdd(reinterpret_cast<unsigned long long*>(a.counters + CT_TEXT), (unsigned long long)bytes + 1ull);
            toff = __shfl_sync(0xffffffffu, toff, 0);
            ok = toff + (unsigned long long)bytes + 1ull <= o.text_cap;
            if (ok) {
                aln_cigar_text(o.runs + off, n_runs, n_ops, o.text + toff);
                if (lane0) o.text[toff + (unsigned long long)bytes] = 0;
                r.cigar_off = (int64_t)toff;
                r.cigar_len = bytes;
            }
        }
        if (ok && o.bp && o.window_length > 0) {
            const int32_t n_win = aln_window_count(job.t_begin, job.m, o.window_length);
            unsigned long long boff = 0;
            if (lane0) boff = atomicAdd(reinterpret_cast<unsigned long long*>(a.counters + CT_BP), 2ull * (unsigned long long)n_win);
            boff = __shfl_sync(0xffffffffu, boff, 0);
            ok = boff + 2ull * (unsigned long long)n_win <= o.bp_cap;
            if (ok) {
                r.bp_count = aln_breaking_points(o.runs + off, n_runs, n_ops, job.q_first, job.t_begin, job.m, o.window_length,
                                                 s.pre, o.bp + 2ull * boff);
                r.bp_off = (int64_t)boff;
            }
        }
        if (lane0) {
            if (!ok) r.status = B200ALN_GENERIC_ERROR;
            a.res[k] = r;
        }
        __syncwarp();
    }
}

/* racon's window layers from the breaking points (layer_cut.cuh); one thread per item / window / place */
__global__ void aln_cut_filter_kernel(const CutArgs a) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < a.n_items; p += (int64_t)gridDim.x * blockDim.x)
        cut_filter(a, p);
}
/* exclusive prefix sum of the per-window counts, one block: each thread sums a contiguous chunk, the chunk sums are
 * scanned in shared memory, then each thread writes its chunk's offsets */
__global__ void __launch_bounds__(1024) aln_cut_scan_kernel(const CutArgs a) {
    __shared__ int64_t part[1024];
    cut_scan_sum(a, threadIdx.x, 1024, part);
    __syncthreads();
    if (threadIdx.x == 0) cut_scan_parts(a, 1024, part);
    __syncthreads();
    cut_scan_write(a, threadIdx.x, 1024, part);
}
__global__ void aln_cut_scatter_kernel(const CutArgs a) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < a.n_items; p += (int64_t)gridDim.x * blockDim.x)
        cut_scatter(a, p);
}
__global__ void aln_cut_place_kernel(const CutArgs a, const int64_t* n_kept) {
    const int64_t n = *n_kept;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        cut_place(a, i);
}
/* b200aln_batch_export_layers: one warp per exported layer (layer_cut.cuh cut_export_layer) */
__global__ void __launch_bounds__(256) aln_layer_export_kernel(const ExportArgs a) {
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int32_t lane = (int32_t)(threadIdx.x & 31u);
    for (int64_t k = warp; k < a.n_jobs; k += n_warps) cut_export_layer(a, k, lane, 32);
}

} // namespace

/* ------------------------------------------------------------------------------------------ */
/* host side                                                                                   */
/* ------------------------------------------------------------------------------------------ */

struct b200aln_batch {
    int32_t device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t side = nullptr; /* huge sub-problems run on teams beside a saturated level's one-warp grid */
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    bool own_stream = false;
    int64_t budget = 0;
    int32_t sm_count = 0, blocks_per_sm = 0;

    /* host staging */
    PinnedBuf h_seq;
    /* view mode (b200aln_batch_add_overlaps_view): the caller's columnar buffers are uploaded as they are */
    const uint8_t* view_q = nullptr;
    const uint8_t* view_t = nullptr;
    int64_t view_q_bytes = 0, view_t_bytes = 0;
    std::vector<AlnJob> jobs;
    int64_t ops_bytes = 0;
    int64_t cap_open = 0, cap_leaves = 0; /* list capacities the staged alignments need */
    AlnLoad load; /* what the staged alignments hold of the budget (host/aln_admission.hpp) */

    /* device */
    DevBuf d_slab, d_team_slab, d_seq, d_jobs, d_ops, d_res, d_runs, d_text, d_bp, d_list[ALN_CLASSES][2], d_leaves, d_counters;
    int32_t n_slots = 0, slot_max_len = 0, n_team_blocks = 0, team_blocks_per_sm = 0;
    size_t slot_bytes = 0, team_slot_bytes = 0;

    /* results */
    std::vector<AlnResult> res;
    PinnedBuf h_runs, h_text, h_bp;
    int32_t band_guess_permille = -1; /* -1: learn from the previous align_all; 0: never guess; > 0: fixed */
    int32_t learnt_permille = 0;
    int32_t window_length = 0; /* > 0: breaking points are formed on the device */
    bool skip_cigars = false;  /* the CIGAR text is neither formed nor downloaded */
    int64_t n_windows = 0;     /* windows the staged overlaps touch */
    std::vector<int64_t> bp_off_tab;
    std::vector<int32_t> bp_cnt_tab;
    /* layer cut (b200aln_batch_set_layer_cut): per staged overlap its contig's first window, the contig's length and
     * whether the read has qualities; the qualities lie parallel to the query bytes (staged in h_qual, or the view's) */
    bool layer_cut = false;
    double quality_threshold = 0.0;
    std::vector<int64_t> cut_first_window;
    std::vector<int32_t> cut_t_length;
    std::vector<uint8_t> cut_has_q;
    PinnedBuf h_qual;
    const uint8_t* view_qual = nullptr;
    DevBuf d_qual, d_cut_ov, d_cut_items, d_cut_counts, d_cut_off, d_cut_slots, d_cut_out;
    PinnedBuf h_layers, h_win_count;
    int64_t n_layers = 0, cut_win_lo = 0, cut_n_win = 0;
    /* b200aln_batch_export_layers: its records, offsets and the downloaded bytes (bases, then weights) */
    DevBuf d_export, d_export_jobs;
    PinnedBuf h_export;
    std::vector<CutLayer> export_records;
    std::vector<int64_t> export_win_off, export_seq_off;
    unsigned long long n_runs_total = 0;
    bool runs_on_host = false; /* the run starts are fetched only when a caller asks for operations */
    std::vector<int64_t> t_off; /* per alignment, for b200aln_batch_get_cigars */
    std::vector<int32_t> t_len, t_ed, t_st;
    PinnedBuf h_counters; /* CT_WORDS int32 */
    bool aligned = false, synced = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    b200aln_batch_info info{};
#if ALN_SPLIT_DIGEST
    DevBuf d_log; /* count, then the records of the last align_all (b200aln_debug_split_log) */
    int32_t log_cap = 0;
#endif
#if ALN_LEAF_DIGEST
    DevBuf d_leaf_log; /* count, then the records of the last align_all (b200aln_debug_leaf_log) */
    int32_t leaf_log_cap = 0;
#endif
};

namespace {

#define ALN_CU(call)                               \
    do {                                           \
        cudaError_t e_ = (call);                   \
        if (e_ != cudaSuccess) {                   \
            cudaGetLastError();                    \
            return B200ALN_CUDA_ERROR;             \
        }                                          \
    } while (0)

int32_t ensure_slots(b200aln_batch* b) {
    const int32_t want_len = round_len(b->load.max_len);
    if (b->n_slots > 0 && want_len <= b->slot_max_len) return B200ALN_SUCCESS;
    const int64_t sb = slot_bytes_for(want_len);
    const int64_t resident = (int64_t)b->sm_count * b->blocks_per_sm * WARPS_PER_BLOCK;
    int64_t avail = b->budget - b->load.var_bytes;
    /* team workspaces (tall sub-problems of thin levels) take at most a quarter of what is left; none is fine too:
     * tall sub-problems then run one warp each */
    size_t tsb = 0;
    TeamSlot ts;
    team_slot_bind(ts, nullptr, want_len, &tsb);
    int64_t nt = std::min<int64_t>((int64_t)b->sm_count * b->team_blocks_per_sm, (avail / 4) / (int64_t)tsb);
    if (avail - nt * (int64_t)tsb < WARPS_PER_BLOCK * sb) nt = 0;
    avail -= nt * (int64_t)tsb;
    int64_t n = std::min<int64_t>(resident, avail / sb);
    n -= n % WARPS_PER_BLOCK;
    if (n < WARPS_PER_BLOCK) return B200ALN_EXCEEDED_MAX_LENGTH;
    ALN_CU(b->d_slab.need((size_t)(n * sb), false));
    if (nt > 0) ALN_CU(b->d_team_slab.need((size_t)(nt * (int64_t)tsb), false));
    b->n_slots = (int32_t)n;
    b->slot_bytes = (size_t)sb;
    b->n_team_blocks = (int32_t)nt;
    b->team_slot_bytes = tsb;
    b->slot_max_len = want_len;
    return B200ALN_SUCCESS;
}

/* After the CIGAR kernel, with the per-alignment records on the host: racon's window layers from the breaking points
 * (layer_cut.cuh), grouped by window in racon's add order, and their download -- the per-window counts, then exactly
 * the kept records.  One synchronisation (the number of kept layers). */
int32_t run_layer_cut(b200aln_batch* b, bool with_qual) {
    const size_t n_aln = b->jobs.size();
    const int32_t w = b->window_length;
    std::vector<CutOverlap> ov(n_aln);
    int64_t n_items = 0, win_lo = INT64_MAX, win_hi = 0;
    for (size_t k = 0; k < n_aln; ++k) {
        const AlnResult& r = b->res[k];
        const AlnJob& j = b->jobs[k];
        CutOverlap& o = ov[k];
        o.q_off = j.q_off;
        o.bp_off = r.bp_off;
        o.item_off = n_items;
        o.first_window = b->cut_first_window[k];
        o.q_first = j.q_first;
        o.has_quality = with_qual ? b->cut_has_q[k] : 0;
        if (r.status == 0 && r.bp_count > 0) n_items += r.bp_count / 2; /* a failed alignment cuts nothing */
        win_lo = std::min(win_lo, o.first_window);
        win_hi = std::max(win_hi, o.first_window + (b->cut_t_length[k] + w - 1) / w);
    }
    if (win_hi <= win_lo) win_lo = win_hi = 0;
    b->cut_win_lo = win_lo;
    b->cut_n_win = win_hi - win_lo;
    b->n_layers = 0;
    cudaStream_t s = b->stream;
    const size_t nw = (size_t)b->cut_n_win;
    ALN_CU(b->d_cut_ov.need(sizeof(CutOverlap) * n_aln + 64));
    ALN_CU(b->d_cut_items.need(sizeof(CutLayer) * (size_t)n_items + 64));
    ALN_CU(b->d_cut_out.need(sizeof(CutLayer) * (size_t)n_items + 64));
    ALN_CU(b->d_cut_slots.need(sizeof(int64_t) * (size_t)n_items + 64));
    ALN_CU(b->d_cut_counts.need(2 * sizeof(int32_t) * nw + 64)); /* counts, then phase 3's cursors */
    ALN_CU(b->d_cut_off.need(sizeof(int64_t) * (nw + 1)));
    if (!b->h_win_count.reserve(sizeof(int32_t) * nw + 64) || !b->h_layers.reserve(sizeof(CutLayer) * (size_t)n_items + 64))
        return B200ALN_GENERIC_ERROR;
    CutArgs a;
    a.ov = static_cast<const CutOverlap*>(b->d_cut_ov.p);
    a.n_overlaps = (int32_t)n_aln;
    a.n_items = n_items;
    a.bp = static_cast<const uint32_t*>(b->d_bp.p);
    a.qual = static_cast<const uint8_t*>(b->d_qual.p);
    a.window_length = w;
    a.quality_threshold = b->quality_threshold;
    a.win_lo = win_lo;
    a.n_win = (int64_t)nw;
    a.items = static_cast<CutLayer*>(b->d_cut_items.p);
    a.counts = static_cast<int32_t*>(b->d_cut_counts.p);
    a.fill = a.counts + nw;
    a.win_off = static_cast<int64_t*>(b->d_cut_off.p);
    a.slots = static_cast<int64_t*>(b->d_cut_slots.p);
    a.out = static_cast<CutLayer*>(b->d_cut_out.p);
    ALN_CU(cudaMemcpyAsync(b->d_cut_ov.p, ov.data(), sizeof(CutOverlap) * n_aln, cudaMemcpyHostToDevice, s));
    ALN_CU(cudaMemsetAsync(b->d_cut_counts.p, 0, 2 * sizeof(int32_t) * nw + 64, s));
    const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((n_items + 255) / 256, (int64_t)b->sm_count * 8));
    if (n_items > 0) aln_cut_filter_kernel<<<grid, 256, 0, s>>>(a);
    aln_cut_scan_kernel<<<1, 1024, 0, s>>>(a);
    if (n_items > 0) {
        aln_cut_scatter_kernel<<<grid, 256, 0, s>>>(a);
        aln_cut_place_kernel<<<grid, 256, 0, s>>>(a, a.win_off + nw);
    }
    ALN_CU(cudaGetLastError());
    b->info.kernel_launches += n_items > 0 ? 4 : 1;
    int64_t* kept = reinterpret_cast<int64_t*>(b->h_win_count.p + ((sizeof(int32_t) * nw + 7) & ~(size_t)7)); /* after the counts */
    ALN_CU(cudaMemcpyAsync(kept, a.win_off + nw, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    if (nw) ALN_CU(cudaMemcpyAsync(b->h_win_count.p, a.counts, sizeof(int32_t) * nw, cudaMemcpyDeviceToHost, s));
    ALN_CU(cudaStreamSynchronize(s));
    if (*kept < 0 || *kept > n_items) return B200ALN_GENERIC_ERROR;
    b->n_layers = *kept;
    if (b->n_layers)
        ALN_CU(cudaMemcpyAsync(b->h_layers.p, a.out, sizeof(CutLayer) * (size_t)b->n_layers, cudaMemcpyDeviceToHost, s));
    b->info.h2d_bytes += (int64_t)(sizeof(CutOverlap) * n_aln);
    b->info.d2h_bytes += (int64_t)(sizeof(int64_t) + sizeof(int32_t) * nw + sizeof(CutLayer) * (size_t)b->n_layers);
    return B200ALN_SUCCESS;
}

} // namespace

extern "C" {

int32_t b200aln_init(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) {
        cudaGetLastError();
        return B200ALN_CUDA_ERROR;
    }
    return B200ALN_SUCCESS;
}

const char* b200aln_status_string(int32_t st) {
    switch (st) {
        case B200ALN_SUCCESS: return "success";
        case B200ALN_UNINITIALIZED: return "uninitialized";
        case B200ALN_EXCEEDED_MAX_ALIGNMENTS: return "exceeded_max_alignments";
        case B200ALN_EXCEEDED_MAX_LENGTH: return "exceeded_max_length";
        case B200ALN_EXCEEDED_MAX_ALIGNMENT_DIFFERENCE: return "exceeded_max_alignment_difference";
        case B200ALN_GENERIC_ERROR: return "generic_error";
        case B200ALN_INVALID_ARGUMENT: return "invalid_argument";
        case B200ALN_CUDA_ERROR: return "cuda_error";
        default: return "unknown";
    }
}

void b200aln_batch_destroy(b200aln_batch* b) {
    if (!b) return;
    cudaSetDevice(b->device);
    /* both streams are idle before the members' destructors free the buffers they used */
    if (b->stream) cudaStreamSynchronize(b->stream);
    if (b->side) cudaStreamSynchronize(b->side);
    if (b->ev_fork) cudaEventDestroy(b->ev_fork);
    if (b->ev_join) cudaEventDestroy(b->ev_join);
    if (b->side) cudaStreamDestroy(b->side);
    if (b->ev0) cudaEventDestroy(b->ev0);
    if (b->ev1) cudaEventDestroy(b->ev1);
    if (b->own_stream && b->stream) cudaStreamDestroy(b->stream);
    delete b;
    cudaGetLastError();
}

int32_t b200aln_batch_create(int32_t device_id, void* stream, int64_t max_gpu_mem, int32_t max_bandwidth,
                             b200aln_batch** out) {
    (void)max_bandwidth; /* cudaaligner's band can cost optimality; this engine's bands cannot (b200aln.h) */
    if (!out) return B200ALN_INVALID_ARGUMENT;
    *out = nullptr;
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess) {
        cudaGetLastError();
        return B200ALN_CUDA_ERROR;
    }
    if (device_id < 0 || device_id >= n_dev) return B200ALN_INVALID_ARGUMENT;
    b200aln_batch* b = new (std::nothrow) b200aln_batch();
    if (!b) return B200ALN_GENERIC_ERROR;
    b->device = device_id;
    int32_t st = B200ALN_SUCCESS;
    do {
        if (cudaSetDevice(device_id) != cudaSuccess) { st = B200ALN_CUDA_ERROR; break; }
        size_t free_b = 0, total_b = 0;
        if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) { st = B200ALN_CUDA_ERROR; break; }
        b->budget = max_gpu_mem > 0 ? max_gpu_mem : (int64_t)((double)free_b * 0.9);
        if (b->budget < ((int64_t)4 << 20)) { st = B200ALN_INVALID_ARGUMENT; break; }
        if (stream) {
            b->stream = static_cast<cudaStream_t>(stream);
        } else {
            if (cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking) != cudaSuccess) { st = B200ALN_CUDA_ERROR; break; }
            b->own_stream = true;
        }
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, device_id) != cudaSuccess) { st = B200ALN_CUDA_ERROR; break; }
        b->sm_count = prop.multiProcessorCount;
        int bps_split = 0, bps_leaf = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps_split, aln_split_kernel, 32 * WARPS_PER_BLOCK, 0) != cudaSuccess ||
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps_leaf, aln_leaf_kernel, 32 * WARPS_PER_BLOCK, 0) != cudaSuccess) {
            st = B200ALN_CUDA_ERROR;
            break;
        }
        b->blocks_per_sm = std::max(1, std::min(bps_split, bps_leaf));
        int bps_team = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps_team, aln_split_team_kernel, 64 * ALN_TEAM, 0) != cudaSuccess) {
            st = B200ALN_CUDA_ERROR;
            break;
        }
        b->team_blocks_per_sm = std::max(0, bps_team);
        if (!b->h_counters.reserve(CT_WORDS * sizeof(int32_t)) ||
            cudaEventCreate(&b->ev0) != cudaSuccess || cudaEventCreate(&b->ev1) != cudaSuccess ||
            cudaStreamCreateWithFlags(&b->side, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreateWithFlags(&b->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&b->ev_join, cudaEventDisableTiming) != cudaSuccess) {
            st = B200ALN_CUDA_ERROR;
            break;
        }
        b->info.device_id = device_id;
    } while (0);
    if (st != B200ALN_SUCCESS) {
        cudaGetLastError();
        b200aln_batch_destroy(b);
        return st;
    }
    *out = b;
    return B200ALN_SUCCESS;
}

int32_t b200aln_batch_set_window_length(b200aln_batch* b, int32_t window_length, int32_t skip_cigars) {
    if (!b || window_length < 0) return B200ALN_INVALID_ARGUMENT;
    if (!b->jobs.empty()) return B200ALN_GENERIC_ERROR; /* staged overlaps were budgeted for the old setting */
    if (window_length == 0 && skip_cigars) return B200ALN_INVALID_ARGUMENT; /* nothing would come back */
    b->window_length = window_length;
    b->skip_cigars = skip_cigars != 0;
    return B200ALN_SUCCESS;
}

int32_t b200aln_batch_add_alignment(b200aln_batch* b, const char* query, int32_t n, const char* target, int32_t m) {
    return b200aln_batch_add_overlap(b, query, n, target, m, 0, 0);
}

/* the layer cut's inputs of one overlap are admissible (b200aln_layer_inputs) */
static bool cut_inputs_ok(int32_t m, int32_t t_begin, int64_t first_window, int32_t t_length) {
    return first_window >= 0 && first_window < ((int64_t)1 << 31) - ((int64_t)t_length + 1) && (int64_t)t_begin + m <= t_length;
}

/* add_overlap with the layer cut's inputs (qual: nullable, parallel to the query) */
static int32_t add_one(b200aln_batch* b, const char* query, int32_t n, const char* target, int32_t m, int32_t q_first,
                       int32_t t_begin, const uint8_t* qual, int64_t first_window, int32_t t_length) {
    if (!b || n < 0 || m < 0 || (n > 0 && !query) || (m > 0 && !target) || q_first < 0 || t_begin < 0)
        return B200ALN_INVALID_ARGUMENT;
    if ((int64_t)t_begin + m >= ((int64_t)1 << 31) || (int64_t)q_first + n >= ((int64_t)1 << 31)) return B200ALN_INVALID_ARGUMENT;
    if (b->layer_cut && !cut_inputs_ok(m, t_begin, first_window, t_length)) return B200ALN_INVALID_ARGUMENT;
    if (b->aligned || b->view_q) return B200ALN_GENERIC_ERROR; /* reset() first, like a cudaaligner batch after align_all */
    AlnLoad load = b->load;
    const int32_t adm = aln_admit(load, b->budget, b->window_length, b->layer_cut, n, m, t_begin);
    if (adm != B200ALN_SUCCESS) return adm;
    if (b->h_seq.used + (size_t)n + (size_t)m > b->h_seq.cap) cudaSetDevice(b->device); /* the staging buffer grows: page-lock it in this batch's context */
    if (!b->h_seq.reserve(b->h_seq.used + (size_t)n + (size_t)m)) return B200ALN_GENERIC_ERROR;
    if (b->layer_cut) { /* the qualities take the query's offsets in a buffer of their own */
        if (b->h_seq.used + (size_t)n + (size_t)m > b->h_qual.cap) cudaSetDevice(b->device);
        if (!b->h_qual.reserve(b->h_seq.used + (size_t)n + (size_t)m)) return B200ALN_GENERIC_ERROR;
        if (qual && n) std::memcpy(b->h_qual.p + b->h_seq.used, qual, (size_t)n);
        else if (n) std::memset(b->h_qual.p + b->h_seq.used, 0, (size_t)n);
        if (m) std::memset(b->h_qual.p + b->h_seq.used + n, 0, (size_t)m); /* the target's place: never read */
        b->h_qual.used = b->h_seq.used + (size_t)n + (size_t)m;
        b->cut_first_window.push_back(first_window);
        b->cut_t_length.push_back(t_length);
        b->cut_has_q.push_back(qual ? 1 : 0);
    }
    AlnJob j;
    j.q_off = (int64_t)b->h_seq.used;
    if (n) std::memcpy(b->h_seq.p + b->h_seq.used, query, (size_t)n);
    b->h_seq.used += (size_t)n;
    j.t_off = (int64_t)b->h_seq.used;
    if (m) std::memcpy(b->h_seq.p + b->h_seq.used, target, (size_t)m);
    b->h_seq.used += (size_t)m;
    j.ops_off = b->ops_bytes;
    j.n = n;
    j.m = m;
    j.q_first = q_first;
    j.t_begin = t_begin;
    b->n_windows += aln_window_count(t_begin, m, b->window_length);
    b->ops_bytes += (int64_t)n + m;
    b->cap_open += aln_open_capacity(n, m);
    b->cap_leaves += aln_leaf_capacity(n, m);
    b->load = load;
    b->jobs.push_back(j);
    return B200ALN_SUCCESS;
}

int32_t b200aln_batch_add_overlap(b200aln_batch* b, const char* query, int32_t n, const char* target, int32_t m,
                                  int32_t q_first, int32_t t_begin) {
    return add_one(b, query, n, target, m, q_first, t_begin, nullptr, 0, t_begin + m);
}

int32_t b200aln_batch_set_layer_cut(b200aln_batch* b, double quality_threshold) {
    if (!b || !(quality_threshold == quality_threshold)) return B200ALN_INVALID_ARGUMENT;
    if (!b->jobs.empty() || b->aligned) return B200ALN_GENERIC_ERROR; /* staged overlaps were budgeted without it */
    if (b->window_length <= 0) return B200ALN_GENERIC_ERROR;          /* b200aln_batch_set_window_length first */
    b->layer_cut = true;
    b->quality_threshold = quality_threshold;
    return B200ALN_SUCCESS;
}

int32_t b200aln_batch_num_alignments(const b200aln_batch* b) { return b ? (int32_t)b->jobs.size() : 0; }

int32_t b200aln_batch_align_all(b200aln_batch* b) {
    if (!b) return B200ALN_INVALID_ARGUMENT;
    if (b->aligned) return B200ALN_SUCCESS;
    const int32_t n_aln = (int32_t)b->jobs.size();
    b->info.levels = 0;
    b->info.kernel_launches = 0;
    b->info.n_open = b->info.n_leaves = b->info.cells = 0;
    b->info.h2d_bytes = b->info.d2h_bytes = 0;
    b->info.kernel_ms = 0.f;
    b->res.assign((size_t)n_aln, AlnResult{0, 0, 0, 0, 0, 0, 0, 0, 0});
    b->h_bp.used = 0;
    b->runs_on_host = false;
    b->n_runs_total = 0;
    b->h_text.used = 0;
    if (n_aln == 0) {
        b->aligned = b->synced = true;
        return B200ALN_SUCCESS;
    }
    ALN_CU(cudaSetDevice(b->device));
    int32_t st = ensure_slots(b);
    if (st != B200ALN_SUCCESS) return st;
    b->info.n_slots = b->n_slots;
    b->info.n_team_blocks = b->n_team_blocks;

    /* the first level, classified on the host: largest first, so the persistent grid starts with the long ones */
    std::vector<AlnRect> first[ALN_CLASSES], leaves0;
    /* the guessed distance per 1000 characters of the longer sequence: fixed by the caller, or learnt from this batch's
     * previous align_all (1.25 x the rate 90 % of its alignments stayed under); none for a batch that has seen nothing yet */
    const int32_t rate_permille = b->band_guess_permille >= 0 ? b->band_guess_permille : b->learnt_permille;
    for (int32_t k = 0; k < n_aln; ++k) {
        const AlnJob& j = b->jobs[(size_t)k];
        if (j.n == 0 && j.m == 0) continue;
        /* a top sub-problem's optimum is unknown: the host guesses (b200aln_batch_set_band_guess), the kernels verify */
        const bool leaf = aln_is_leaf(j.n, j.m);
        int32_t guess = -1;
        if (!leaf && rate_permille > 0)
            guess = (int32_t)std::min<int64_t>(((int64_t)std::max(j.n, j.m) * rate_permille + 999) / 1000 + 32, (int64_t)1 << 29);
        (leaf ? leaves0 : first[aln_shape(j.n, j.m)]).push_back(AlnRect{k, 0, j.n, 0, j.m, guess >= 0 ? (ALN_TOP | ALN_GUESS) : ALN_TOP, guess});
    }
    const auto larger = [](const AlnRect& x, const AlnRect& y) { return (int64_t)x.n * x.m > (int64_t)y.n * y.m; };
    size_t first_total = 0, first_max = 0;
    for (int c = 0; c < ALN_CLASSES; ++c) {
        std::stable_sort(first[c].begin(), first[c].end(), larger);
        first_total += first[c].size();
        first_max = std::max(first_max, first[c].size());
    }
    const int64_t cap_open = std::max<int64_t>(b->cap_open, (int64_t)first_max) + 16;
    const int64_t cap_leaves = std::max<int64_t>(b->cap_leaves, (int64_t)leaves0.size()) + 16;
    if (cap_open >= 0x7FFFFFFF || cap_leaves >= 0x7FFFFFFF) return B200ALN_EXCEEDED_MAX_ALIGNMENTS;

    const size_t seq_bytes = b->view_q ? (size_t)(b->view_q_bytes + b->view_t_bytes) : b->h_seq.used;
    ALN_CU(b->d_seq.need(seq_bytes + 64));
    ALN_CU(b->d_jobs.need(sizeof(AlnJob) * (size_t)n_aln));
    ALN_CU(b->d_ops.need((size_t)b->ops_bytes + 64));
    ALN_CU(b->d_res.need(sizeof(AlnResult) * (size_t)n_aln));
    ALN_CU(b->d_runs.need(sizeof(uint32_t) * ((size_t)b->ops_bytes + 64)));
    const unsigned long long text_cap = 2ull * (unsigned long long)b->ops_bytes + (unsigned long long)n_aln + 64; /* "1M1I..." at worst */
    ALN_CU(b->d_text.need((size_t)text_cap));
    const bool want_bp = b->window_length > 0;
    const unsigned long long bp_cap = 2ull * (unsigned long long)b->n_windows + 16; /* (t, q) pairs */
    if (want_bp) ALN_CU(b->d_bp.need((size_t)bp_cap * 8));
    for (int c = 0; c < ALN_CLASSES; ++c) {
        ALN_CU(b->d_list[c][0].need(sizeof(AlnRect) * (size_t)cap_open));
        ALN_CU(b->d_list[c][1].need(sizeof(AlnRect) * (size_t)cap_open));
    }
    ALN_CU(b->d_leaves.need(sizeof(AlnRect) * (size_t)cap_leaves));
    ALN_CU(b->d_counters.need(sizeof(int32_t) * CT_WORDS));
#if ALN_SPLIT_DIGEST
    /* a split per open sub-problem (fewer than the leaves) and a redo per alignment at most */
    b->log_cap = (int32_t)std::min<int64_t>(cap_leaves + n_aln + 64, 0x7FFFFFF);
    ALN_CU(b->d_log.need(sizeof(AlnSplitRec) * ((size_t)b->log_cap + 1)));
    ALN_CU(cudaMemsetAsync(b->d_log.p, 0, sizeof(AlnSplitRec), b->stream));
#endif
#if ALN_LEAF_DIGEST
    /* a record per leaf: the leaf list's capacity (more leaves would have overflowed the list itself) */
    b->leaf_log_cap = (int32_t)std::min<int64_t>(cap_leaves, 0x7FFFFFF);
    ALN_CU(b->d_leaf_log.need(sizeof(AlnLeafRec) * ((size_t)b->leaf_log_cap + 1)));
    ALN_CU(cudaMemsetAsync(b->d_leaf_log.p, 0, sizeof(AlnLeafRec), b->stream));
#endif

    cudaStream_t s = b->stream;
    int32_t* ct = static_cast<int32_t*>(b->d_counters.p);
    int32_t* hc = reinterpret_cast<int32_t*>(b->h_counters.p);
    std::memset(hc, 0, sizeof(int32_t) * CT_WORDS);
    for (int c = 0; c < ALN_CLASSES; ++c) hc[CT_NOPEN + c] = (int32_t)first[c].size();
    hc[CT_NLEAVES] = (int32_t)leaves0.size();
    ALN_CU(cudaMemcpyAsync(ct, hc, sizeof(int32_t) * CT_WORDS, cudaMemcpyHostToDevice, s));
    if (b->view_q) { /* straight from the caller's buffers (page-locked ones upload at full PCIe speed) */
        if (b->view_q_bytes)
            ALN_CU(cudaMemcpyAsync(b->d_seq.p, b->view_q, (size_t)b->view_q_bytes, cudaMemcpyHostToDevice, s));
        if (b->view_t_bytes)
            ALN_CU(cudaMemcpyAsync(static_cast<uint8_t*>(b->d_seq.p) + b->view_q_bytes, b->view_t, (size_t)b->view_t_bytes,
                                   cudaMemcpyHostToDevice, s));
    } else {
        ALN_CU(cudaMemcpyAsync(b->d_seq.p, b->h_seq.p, b->h_seq.used, cudaMemcpyHostToDevice, s));
    }
    size_t qual_bytes = 0; /* the layer cut's qualities, at the query bytes' offsets; none when no read has any */
    if (b->layer_cut && std::find(b->cut_has_q.begin(), b->cut_has_q.end(), 1) != b->cut_has_q.end()) {
        const uint8_t* src = b->view_q ? b->view_qual : b->h_qual.p;
        qual_bytes = b->view_q ? (size_t)b->view_q_bytes : b->h_qual.used;
        ALN_CU(b->d_qual.need(seq_bytes + 64));
        if (src && qual_bytes) ALN_CU(cudaMemcpyAsync(b->d_qual.p, src, qual_bytes, cudaMemcpyHostToDevice, s));
    }
    ALN_CU(cudaMemcpyAsync(b->d_jobs.p, b->jobs.data(), sizeof(AlnJob) * (size_t)n_aln, cudaMemcpyHostToDevice, s));
    for (int c = 0; c < ALN_CLASSES; ++c)
        if (!first[c].empty())
            ALN_CU(cudaMemcpyAsync(b->d_list[c][0].p, first[c].data(), sizeof(AlnRect) * first[c].size(), cudaMemcpyHostToDevice, s));
    if (!leaves0.empty())
        ALN_CU(cudaMemcpyAsync(b->d_leaves.p, leaves0.data(), sizeof(AlnRect) * leaves0.size(), cudaMemcpyHostToDevice, s));
    ALN_CU(cudaMemsetAsync(b->d_ops.p, 0xFF, (size_t)b->ops_bytes + 64, s));
    ALN_CU(cudaMemsetAsync(b->d_res.p, 0, sizeof(AlnResult) * (size_t)n_aln, s));
    /* the pageable vectors above (jobs, first, leaves0) must not be touched before the copies were issued from them:
     * cudaMemcpyAsync from pageable memory stages them before returning */
    b->info.h2d_bytes = (int64_t)(seq_bytes + qual_bytes + sizeof(AlnJob) * (size_t)n_aln + sizeof(AlnRect) * (first_total + leaves0.size()) +
                                  sizeof(int32_t) * CT_WORDS);

    AlnKernelArgs a;
    a.slab = static_cast<uint8_t*>(b->d_slab.p);
    a.slot_bytes = b->slot_bytes;
    a.team_slab = static_cast<uint8_t*>(b->d_team_slab.p);
    a.team_slot_bytes = b->team_slot_bytes;
    a.max_len = b->slot_max_len;
    a.seq = static_cast<const uint8_t*>(b->d_seq.p);
    a.jobs = static_cast<const AlnJob*>(b->d_jobs.p);
    a.ops = static_cast<uint8_t*>(b->d_ops.p);
    a.res = static_cast<AlnResult*>(b->d_res.p);
    a.counters = ct;
#if ALN_SPLIT_DIGEST
    a.log_count = static_cast<int32_t*>(b->d_log.p);
    a.log = static_cast<AlnSplitRec*>(b->d_log.p) + 1;
    a.log_cap = b->log_cap;
#endif
#if ALN_LEAF_DIGEST
    a.leaf_log_count = static_cast<int32_t*>(b->d_leaf_log.p);
    a.leaf_log = static_cast<AlnLeafRec*>(b->d_leaf_log.p) + 1;
    a.leaf_log_cap = b->leaf_log_cap;
#endif
    const int32_t max_blocks = b->n_slots / WARPS_PER_BLOCK;
    auto grid_for = [&](int64_t items) {
        return (unsigned)std::max<int64_t>(1, std::min<int64_t>(max_blocks, (items + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK));
    };

    ALN_CU(cudaEventRecord(b->ev0, s));
    int32_t n_open[ALN_CLASSES];
    for (int c = 0; c < ALN_CLASSES; ++c) n_open[c] = (int32_t)first[c].size();
    int32_t level = 0, launch = 0;
    b->info.team_launches = 0;
    while (n_open[ALN_SHORT] + n_open[ALN_TALL] + n_open[ALN_HUGE] > 0) {
        if (level + 1 >= MAX_LEVELS || launch + 4 >= 128) return B200ALN_GENERIC_ERROR;
        int32_t* ct_next = ct + CT_NOPEN + 4 * (level + 1);
        AlnLists next;
        for (int c = 0; c < ALN_CLASSES; ++c) next.open[c] = static_cast<AlnRect*>(b->d_list[c][(level + 1) & 1].p);
        next.n_open = ct_next;
        next.cap_open = (int32_t)cap_open;
        next.leaves = static_cast<AlnRect*>(b->d_leaves.p);
        next.n_leaves = ct + CT_NLEAVES;
        next.cap_leaves = (int32_t)cap_leaves;
        next.overflow = ct + CT_OVERFLOW;
        /* Thin level (its longest sub-problem bounds its time): a team of warps per tall or huge sub-problem, the
         * one-stripe ones one warp each.  Saturated level (enough sub-problems to fill the device one warp each): the huge
         * ones -- any of which would outlast the rest of the level on one warp -- still go to teams, on a side stream
         * beside the one-warp grid that does everything else. */
        const auto work_of = [&](bool huge, bool tall, bool shrt) {
            AlnWork w;
            const bool take[ALN_CLASSES] = {shrt, tall, huge};
            int slot = 0;
            w.total = 0;
            for (int c = ALN_CLASSES - 1; c >= 0; --c) { /* huge, tall, short */
                w.list[slot] = static_cast<const AlnRect*>(b->d_list[c][level & 1].p);
                w.n[slot] = take[c] ? n_open[c] : 0;
                w.total += w.n[slot];
                ++slot;
            }
#if ALN_SPLIT_DIGEST
            w.level = level;
            w.path = ALN_PATH_WARP;
#endif
            return w;
        };
        const auto team = [&](const AlnWork& w_in, cudaStream_t on) {
            AlnWork w = w_in;
#if ALN_SPLIT_DIGEST
            w.path = on == b->side ? ALN_PATH_SIDE : ALN_PATH_TEAM;
#endif
            if (w.total == 0) return;
            aln_split_team_kernel<<<(unsigned)std::min(w.total, b->n_team_blocks), 64 * ALN_TEAM, 0, on>>>(
                a, w, next, ct + CT_CURSOR + launch);
            ++launch;
            ++b->info.team_launches;
        };
        const auto solo = [&](const AlnWork& w) {
            if (w.total == 0) return;
            aln_split_kernel<<<grid_for(w.total), 32 * WARPS_PER_BLOCK, 0, s>>>(a, w, next, ct + CT_CURSOR + launch);
            ++launch;
        };
        const bool teams = b->n_team_blocks > 0;
        const bool thin = teams && (int64_t)n_open[ALN_TALL] + n_open[ALN_HUGE] <= (int64_t)ALN_TEAM_WAVES * b->n_team_blocks;
        bool forked = false;
        if (!teams) {
            solo(work_of(true, true, true));
        } else if (thin) {
            team(work_of(true, true, false), s);
            solo(work_of(false, false, true));
        } else {
            if (n_open[ALN_HUGE] > 0) {
                ALN_CU(cudaEventRecord(b->ev_fork, s));
                ALN_CU(cudaStreamWaitEvent(b->side, b->ev_fork, 0));
                team(work_of(true, false, false), b->side);
                ALN_CU(cudaEventRecord(b->ev_join, b->side));
                forked = true;
            }
            solo(work_of(false, true, true));
        }
        ALN_CU(cudaGetLastError());
        if (forked) ALN_CU(cudaStreamWaitEvent(s, b->ev_join, 0));
        b->info.n_open += (int64_t)n_open[0] + n_open[1] + n_open[2];
        ALN_CU(cudaMemcpyAsync(hc + CT_NOPEN + 4 * (level + 1), ct_next, ALN_CLASSES * sizeof(int32_t),
                               cudaMemcpyDeviceToHost, s));
        ALN_CU(cudaStreamSynchronize(s));
        for (int c = 0; c < ALN_CLASSES; ++c)
            n_open[c] = std::min<int32_t>(hc[CT_NOPEN + 4 * (level + 1) + c], (int32_t)cap_open);
        ++level;
    }
    b->info.levels = level;
    ALN_CU(cudaMemcpyAsync(hc + CT_NLEAVES, ct + CT_NLEAVES, 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    ALN_CU(cudaStreamSynchronize(s));
    if (hc[CT_OVERFLOW]) return B200ALN_GENERIC_ERROR;
    const int32_t n_leaves = hc[CT_NLEAVES];
    b->info.n_leaves = n_leaves;
    if (n_leaves > 0) {
        aln_leaf_kernel<<<grid_for(n_leaves), 32 * WARPS_PER_BLOCK, 0, s>>>(a, static_cast<const AlnRect*>(b->d_leaves.p),
                                                                            n_leaves, ct + CT_CURSOR + launch);
        ALN_CU(cudaGetLastError());
        ++launch;
    }
    AlnOutArgs oa;
    oa.runs = static_cast<uint32_t*>(b->d_runs.p);
    oa.runs_cap = (unsigned long long)b->ops_bytes + 64;
    oa.text = b->skip_cigars ? nullptr : static_cast<uint8_t*>(b->d_text.p);
    oa.text_cap = text_cap;
    oa.bp = want_bp ? static_cast<uint32_t*>(b->d_bp.p) : nullptr;
    oa.bp_cap = bp_cap;
    oa.window_length = b->window_length;
    aln_cigar_kernel<<<grid_for(n_aln), 32 * WARPS_PER_BLOCK, 0, s>>>(a, n_aln, oa, ct + CT_CURSOR + launch);
    ALN_CU(cudaGetLastError());
    ++launch;
    ALN_CU(cudaEventRecord(b->ev1, s));
    b->info.kernel_launches = launch;
    /* compact results: the per-alignment records and the counters now, then exactly the CIGAR bytes produced; the run
     * starts stay on the device until a caller asks for operations (b200aln_batch_get_alignment / _get_ops) */
    ALN_CU(cudaMemcpyAsync(b->res.data(), b->d_res.p, sizeof(AlnResult) * (size_t)n_aln, cudaMemcpyDeviceToHost, s));
    ALN_CU(cudaMemcpyAsync(hc + CT_RUNS, ct + CT_RUNS, 10 * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    ALN_CU(cudaStreamSynchronize(s));
    if (b->layer_cut) {
        st = run_layer_cut(b, qual_bytes > 0);
        if (st != B200ALN_SUCCESS) return st;
    }
    unsigned long long n_runs_total = 0, cells = 0, text_total = 0;
    std::memcpy(&n_runs_total, hc + CT_RUNS, 8);
    std::memcpy(&cells, hc + CT_CELLS, 8);
    std::memcpy(&text_total, hc + CT_TEXT, 8);
    b->info.cells = (int64_t)cells;
    b->n_runs_total = std::min<unsigned long long>(n_runs_total, (unsigned long long)b->ops_bytes + 64);
    text_total = std::min<unsigned long long>(text_total, text_cap);
    if (!b->h_text.reserve((size_t)text_total + 64)) return B200ALN_GENERIC_ERROR;
    b->h_text.used = (size_t)text_total;
    if (text_total)
        ALN_CU(cudaMemcpyAsync(b->h_text.p, b->d_text.p, (size_t)text_total, cudaMemcpyDeviceToHost, s));
    unsigned long long bp_total = 0;
    std::memcpy(&bp_total, hc + CT_BP, 8);
    /* with a layer cut the breaking points stay on the device: only the layer records come back */
    bp_total = want_bp && !b->layer_cut ? std::min<unsigned long long>(bp_total, bp_cap) : 0;
    if (!b->h_bp.reserve((size_t)bp_total * 8 + 64)) return B200ALN_GENERIC_ERROR;
    b->h_bp.used = (size_t)bp_total * 8;
    if (bp_total) ALN_CU(cudaMemcpyAsync(b->h_bp.p, b->d_bp.p, (size_t)bp_total * 8, cudaMemcpyDeviceToHost, s));
    b->info.d2h_bytes += (int64_t)(sizeof(AlnResult) * (size_t)n_aln + (size_t)text_total + (size_t)bp_total * 8 +
                                  sizeof(int32_t) * (size_t)(level + 12));
    b->aligned = true;
    b->synced = false;
    return B200ALN_SUCCESS;
}

int32_t b200aln_batch_sync(b200aln_batch* b) {
    if (!b) return B200ALN_INVALID_ARGUMENT;
    if (!b->aligned) return B200ALN_UNINITIALIZED;
    if (b->synced) return B200ALN_SUCCESS;
    ALN_CU(cudaSetDevice(b->device));
    ALN_CU(cudaStreamSynchronize(b->stream));
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, b->ev0, b->ev1) == cudaSuccess) b->info.kernel_ms = ms;
    else cudaGetLastError();
    const size_t n_aln = b->jobs.size();
    b->t_off.resize(n_aln);
    b->t_len.resize(n_aln);
    b->t_ed.resize(n_aln);
    b->t_st.resize(n_aln);
    b->bp_off_tab.resize(n_aln);
    b->bp_cnt_tab.resize(n_aln);
    for (size_t k = 0; k < n_aln; ++k) {
        const AlnResult& r = b->res[k];
        const bool bp_ok = b->window_length > 0 && r.status == 0 && r.bp_off >= 0 && r.bp_count >= 0 &&
                           (b->layer_cut || (size_t)(r.bp_off + r.bp_count) * 8 <= b->h_bp.used);
        b->bp_off_tab[k] = bp_ok ? r.bp_off : 0;
        b->bp_cnt_tab[k] = bp_ok ? r.bp_count : 0;
        const bool ok = r.status == 0 && (b->skip_cigars ? (b->window_length == 0 || bp_ok) :
                        (r.cigar_off >= 0 && r.cigar_len >= 0 &&
                         (size_t)(r.cigar_off + r.cigar_len) < b->h_text.used)); /* its terminating 0 included */
        b->t_off[k] = ok && !b->skip_cigars ? r.cigar_off : 0;
        b->t_len[k] = ok && !b->skip_cigars ? r.cigar_len : 0;
        b->t_ed[k] = r.score;
        b->t_st[k] = ok ? B200ALN_SUCCESS : (r.status ? r.status : B200ALN_GENERIC_ERROR);
    }
    if (n_aln >= 8) { /* what the next align_all of this batch will guess (verified on the device, so only speed is at stake) */
        std::vector<int32_t> rates;
        rates.reserve(n_aln);
        for (size_t k = 0; k < n_aln; ++k) {
            const int32_t len = std::max(b->jobs[k].n, b->jobs[k].m);
            if (len > 0 && b->t_st[k] == B200ALN_SUCCESS) rates.push_back((int32_t)(((int64_t)b->res[k].score * 1000 + len - 1) / len));
        }
        if (rates.size() >= 8) {
            const size_t p90 = rates.size() * 9 / 10;
            std::nth_element(rates.begin(), rates.begin() + (std::ptrdiff_t)p90, rates.end());
            b->learnt_permille = std::min(1000, rates[p90] * 5 / 4 + 1);
        }
    }
    b->synced = true;
    return B200ALN_SUCCESS;
}

int32_t b200aln_batch_set_band_guess(b200aln_batch* b, int32_t permille) {
    if (!b || permille < -1 || permille > 1000) return B200ALN_INVALID_ARGUMENT;
    b->band_guess_permille = permille;
    return B200ALN_SUCCESS;
}

int32_t b200aln_batch_get_breaking_points(const b200aln_batch* b, const uint32_t** points, const int64_t** off,
                                          const int32_t** count) {
    if (!b) return B200ALN_INVALID_ARGUMENT;
    if (!b->aligned || !b->synced) return B200ALN_UNINITIALIZED;
    if (b->window_length <= 0) return B200ALN_GENERIC_ERROR; /* b200aln_batch_set_window_length first */
    if (b->layer_cut) return B200ALN_GENERIC_ERROR;          /* they stayed on the device (b200aln_batch_get_layers) */
    if (points) *points = reinterpret_cast<const uint32_t*>(b->h_bp.p);
    if (off) *off = b->bp_off_tab.data();
    if (count) *count = b->bp_cnt_tab.data();
    return B200ALN_SUCCESS;
}

int32_t b200aln_batch_get_layers(const b200aln_batch* b, const b200aln_layer** layers, int64_t* n_layers,
                                 int64_t* first_window, int64_t* n_windows, const int32_t** window_count) {
    if (!b) return B200ALN_INVALID_ARGUMENT;
    if (!b->aligned || !b->synced) return B200ALN_UNINITIALIZED;
    if (!b->layer_cut) return B200ALN_GENERIC_ERROR; /* b200aln_batch_set_layer_cut first */
    if (layers) *layers = reinterpret_cast<const b200aln_layer*>(b->h_layers.p);
    if (n_layers) *n_layers = b->n_layers;
    if (first_window) *first_window = b->cut_win_lo;
    if (n_windows) *n_windows = b->cut_n_win;
    if (window_count) *window_count = reinterpret_cast<const int32_t*>(b->h_win_count.p);
    return B200ALN_SUCCESS;
}

int32_t b200aln_batch_export_layers(b200aln_batch* b, int64_t n, const int64_t* windows, b200aln_export* out) {
    if (!b || n < 0 || (n > 0 && !windows) || !out) return B200ALN_INVALID_ARGUMENT;
    if (!b->aligned || !b->synced) return B200ALN_UNINITIALIZED;
    if (!b->layer_cut) return B200ALN_GENERIC_ERROR;
    const CutLayer* rec = reinterpret_cast<const CutLayer*>(b->h_layers.p);
    std::vector<ExportJob> jobs;
    std::vector<int64_t> picked;
    const int64_t total = cut_export_plan(rec, reinterpret_cast<const int32_t*>(b->h_win_count.p), b->cut_n_win, windows,
                                          n, jobs, picked, b->export_win_off);
    if (total < 0) return B200ALN_INVALID_ARGUMENT;
    b->export_records.clear();
    b->export_seq_off.assign(1, 0);
    for (size_t i = 0; i < jobs.size(); ++i) {
        b->export_records.push_back(rec[picked[i]]);
        b->export_seq_off.push_back(jobs[i].dst + jobs[i].len);
    }
    if (total > 0) { /* nothing exported: no launch, no copy */
        cudaSetDevice(b->device);
        cudaStream_t s = b->stream;
        ALN_CU(b->d_export_jobs.need(sizeof(ExportJob) * jobs.size()));
        ALN_CU(b->d_export.need((size_t)(2 * total)));
        if (!b->h_export.reserve((size_t)(2 * total))) return B200ALN_GENERIC_ERROR;
        ALN_CU(cudaMemcpyAsync(b->d_export_jobs.p, jobs.data(), sizeof(ExportJob) * jobs.size(), cudaMemcpyHostToDevice, s));
        ExportArgs a;
        a.jobs = static_cast<const ExportJob*>(b->d_export_jobs.p);
        a.n_jobs = (int64_t)jobs.size();
        a.total = total;
        a.bases = static_cast<const uint8_t*>(b->d_seq.p);
        a.qual = static_cast<const uint8_t*>(b->d_qual.p);
        a.out = static_cast<uint8_t*>(b->d_export.p);
        const unsigned grid = (unsigned)std::min<int64_t>((a.n_jobs + 7) / 8, (int64_t)b->sm_count * 16);
        aln_layer_export_kernel<<<grid, 256, 0, s>>>(a);
        ALN_CU(cudaGetLastError());
        ALN_CU(cudaMemcpyAsync(b->h_export.p, b->d_export.p, (size_t)(2 * total), cudaMemcpyDeviceToHost, s));
        ALN_CU(cudaStreamSynchronize(s)); /* also what makes the pageable job table safe to free */
    }
    out->n_layers = (int64_t)b->export_records.size();
    out->layers = reinterpret_cast<const b200aln_layer*>(b->export_records.data());
    out->win_layer_off = b->export_win_off.data();
    out->seq_off = b->export_seq_off.data();
    out->bases = total > 0 ? b->h_export.p : nullptr;
    out->weights = total > 0 ? reinterpret_cast<const int8_t*>(b->h_export.p + total) : nullptr;
    out->h2d_bytes = total > 0 ? (int64_t)(sizeof(ExportJob) * jobs.size()) : 0;
    out->d2h_bytes = 2 * total;
    return B200ALN_SUCCESS;
}

int32_t b200aln_batch_device_arena(const b200aln_batch* b, int32_t* device, const uint8_t** bases,
                                   const uint8_t** qualities) {
    if (!b) return B200ALN_INVALID_ARGUMENT;
    if (!b->aligned) return B200ALN_UNINITIALIZED;
    if (device) *device = b->device;
    if (bases) *bases = static_cast<const uint8_t*>(b->d_seq.p);
    if (qualities) *qualities = static_cast<const uint8_t*>(b->d_qual.p);
    return B200ALN_SUCCESS;
}

int32_t b200aln_batch_get_cigars(const b200aln_batch* b, const char** text, const int64_t** off, const int32_t** len,
                                 const int32_t** edit_distance, const int32_t** status) {
    if (!b) return B200ALN_INVALID_ARGUMENT;
    if (!b->aligned || !b->synced) return B200ALN_UNINITIALIZED;
    if (b->skip_cigars) return B200ALN_GENERIC_ERROR; /* the batch was told not to form them */
    if (text) *text = reinterpret_cast<const char*>(b->h_text.p);
    if (off) *off = b->t_off.data();
    if (len) *len = b->t_len.data();
    if (edit_distance) *edit_distance = b->t_ed.data();
    if (status) *status = b->t_st.data();
    return B200ALN_SUCCESS;
}

int32_t b200aln_batch_add_alignments(b200aln_batch* b, int64_t n, const uint8_t* q_bases, const int64_t* q_off,
                                     const uint8_t* t_bases, const int64_t* t_off, int64_t* n_added) {
    return b200aln_batch_add_overlaps(b, n, q_bases, q_off, t_bases, t_off, nullptr, nullptr, n_added);
}

/* overlap k's layer-cut inputs (li nullable: contig of its own, 0-based, no qualities) */
static void layer_inputs_of(const b200aln_layer_inputs* li, const int64_t* q_off, int64_t k, int32_t t_begin, int32_t m,
                            const uint8_t** qual, int64_t* first_window, int32_t* t_length) {
    *first_window = li && li->first_window ? li->first_window[k] : 0;
    *t_length = li && li->t_length ? li->t_length[k] : t_begin + m;
    *qual = li && li->q_quality && li->has_quality && li->has_quality[k] ? li->q_quality + q_off[k] : nullptr;
}

int32_t b200aln_batch_add_overlaps(b200aln_batch* b, int64_t n, const uint8_t* q_bases, const int64_t* q_off,
                                   const uint8_t* t_bases, const int64_t* t_off, const int32_t* q_first,
                                   const int32_t* t_begin, int64_t* n_added) {
    return b200aln_batch_add_overlaps_ex(b, n, q_bases, q_off, t_bases, t_off, q_first, t_begin, nullptr, n_added);
}

int32_t b200aln_batch_add_overlaps_ex(b200aln_batch* b, int64_t n, const uint8_t* q_bases, const int64_t* q_off,
                                      const uint8_t* t_bases, const int64_t* t_off, const int32_t* q_first,
                                      const int32_t* t_begin, const b200aln_layer_inputs* li, int64_t* n_added) {
    if (n_added) *n_added = 0;
    if (!b || n < 0 || (n > 0 && (!q_bases || !q_off || !t_bases || !t_off))) return B200ALN_INVALID_ARGUMENT;
    int64_t k = 0;
    int32_t st = B200ALN_SUCCESS;
    for (; k < n; ++k) {
        const int32_t nn = (int32_t)(q_off[k + 1] - q_off[k]), mm = (int32_t)(t_off[k + 1] - t_off[k]);
        const int32_t tb = t_begin ? t_begin[k] : 0;
        const uint8_t* qual = nullptr;
        int64_t fw = 0;
        int32_t tl = 0;
        layer_inputs_of(li, q_off, k, tb, mm, &qual, &fw, &tl);
        st = add_one(b, reinterpret_cast<const char*>(q_bases + q_off[k]), nn, reinterpret_cast<const char*>(t_bases + t_off[k]),
                     mm, q_first ? q_first[k] : 0, tb, qual, fw, tl);
        if (st != B200ALN_SUCCESS) break;
    }
    if (n_added) *n_added = k;
    if (st == B200ALN_EXCEEDED_MAX_ALIGNMENTS && k > 0) return B200ALN_SUCCESS; /* full: align, reset, go on from k */
    return st;
}

int32_t b200aln_batch_add_overlaps_view(b200aln_batch* b, int64_t n, const uint8_t* q_bases, const int64_t* q_off,
                                        const uint8_t* t_bases, const int64_t* t_off, const int32_t* q_first,
                                        const int32_t* t_begin, int64_t* n_added) {
    return b200aln_batch_add_overlaps_view_ex(b, n, q_bases, q_off, t_bases, t_off, q_first, t_begin, nullptr, n_added);
}

int32_t b200aln_batch_add_overlaps_view_ex(b200aln_batch* b, int64_t n, const uint8_t* q_bases, const int64_t* q_off,
                                           const uint8_t* t_bases, const int64_t* t_off, const int32_t* q_first,
                                           const int32_t* t_begin, const b200aln_layer_inputs* li, int64_t* n_added) {
    if (n_added) *n_added = 0;
    if (!b || n < 0 || (n > 0 && (!q_bases || !q_off || !t_bases || !t_off))) return B200ALN_INVALID_ARGUMENT;
    if (b->aligned || !b->jobs.empty()) return B200ALN_GENERIC_ERROR; /* an empty batch only: one view per fill */
    if (n == 0) return B200ALN_SUCCESS;
    int64_t k = 0;
    int32_t st = B200ALN_SUCCESS;
    for (; k < n; ++k) { /* the same admission as add_overlap, without the copy */
        const int64_t nn = q_off[k + 1] - q_off[k], mm = t_off[k + 1] - t_off[k];
        const int32_t qf = q_first ? q_first[k] : 0, tb = t_begin ? t_begin[k] : 0;
        if (nn < 0 || mm < 0 || qf < 0 || tb < 0 || (int64_t)tb + mm >= ((int64_t)1 << 31) || (int64_t)qf + nn >= ((int64_t)1 << 31)) {
            st = B200ALN_INVALID_ARGUMENT;
            break;
        }
        if (nn + mm >= ((int64_t)1 << 30)) { st = B200ALN_EXCEEDED_MAX_LENGTH; break; }
        const int32_t ni = (int32_t)nn, mi = (int32_t)mm;
        const uint8_t* qual = nullptr;
        int64_t fw = 0;
        int32_t tl = 0;
        layer_inputs_of(li, q_off, k, tb, mi, &qual, &fw, &tl);
        if (b->layer_cut && !cut_inputs_ok(mi, tb, fw, tl)) { st = B200ALN_INVALID_ARGUMENT; break; }
        st = aln_admit(b->load, b->budget, b->window_length, b->layer_cut, ni, mi, tb);
        if (st != B200ALN_SUCCESS) break;
        if (b->layer_cut) {
            b->cut_first_window.push_back(fw);
            b->cut_t_length.push_back(tl);
            b->cut_has_q.push_back(qual ? 1 : 0);
        }
        AlnJob j;
        j.q_off = q_off[k] - q_off[0];
        j.t_off = t_off[k] - t_off[0]; /* + the query bytes, once their total is known */
        j.ops_off = b->ops_bytes;
        j.n = ni;
        j.m = mi;
        j.q_first = qf;
        j.t_begin = tb;
        b->n_windows += aln_window_count(tb, mi, b->window_length);
        b->ops_bytes += nn + mm;
        b->cap_open += aln_open_capacity(ni, mi);
        b->cap_leaves += aln_leaf_capacity(ni, mi);
        b->jobs.push_back(j);
    }
    if (k > 0) {
        b->view_q = q_bases + q_off[0];
        b->view_t = t_bases + t_off[0];
        b->view_q_bytes = q_off[k] - q_off[0];
        b->view_t_bytes = t_off[k] - t_off[0];
        /* the view's qualities: the same byte range of the caller's quality column (read only for has_quality overlaps) */
        b->view_qual = b->layer_cut && li && li->q_quality ? li->q_quality + q_off[0] : nullptr;
        for (AlnJob& j : b->jobs) j.t_off += b->view_q_bytes;
    }
    if (n_added) *n_added = k;
    if (st == B200ALN_EXCEEDED_MAX_ALIGNMENTS && k > 0) return B200ALN_SUCCESS;
    return st;
}

int32_t b200aln_host_register(const void* p, int64_t bytes) {
    if (!p || bytes <= 0) return B200ALN_INVALID_ARGUMENT;
    if (cudaHostRegister(const_cast<void*>(p), (size_t)bytes, cudaHostRegisterPortable) != cudaSuccess) {
        cudaGetLastError();
        return B200ALN_CUDA_ERROR;
    }
    return B200ALN_SUCCESS;
}
int32_t b200aln_host_unregister(const void* p) {
    if (!p) return B200ALN_INVALID_ARGUMENT;
    if (cudaHostUnregister(const_cast<void*>(p)) != cudaSuccess) {
        cudaGetLastError();
        return B200ALN_CUDA_ERROR;
    }
    return B200ALN_SUCCESS;
}

/* the run starts of the last align_all, fetched on first use */
static int32_t fetch_runs(const b200aln_batch* cb) {
    b200aln_batch* b = const_cast<b200aln_batch*>(cb);
    if (b->runs_on_host) return B200ALN_SUCCESS;
    ALN_CU(cudaSetDevice(b->device));
    b->h_runs.used = 0;
    if (!b->h_runs.reserve((size_t)b->n_runs_total * sizeof(uint32_t) + 64)) return B200ALN_GENERIC_ERROR;
    if (b->n_runs_total) {
        ALN_CU(cudaMemcpyAsync(b->h_runs.p, b->d_runs.p, (size_t)b->n_runs_total * sizeof(uint32_t), cudaMemcpyDeviceToHost, b->stream));
        ALN_CU(cudaStreamSynchronize(b->stream));
    }
    b->h_runs.used = (size_t)b->n_runs_total * sizeof(uint32_t);
    b->info.d2h_bytes += (int64_t)b->h_runs.used;
    b->runs_on_host = true;
    return B200ALN_SUCCESS;
}

int32_t b200aln_batch_get_alignment(const b200aln_batch* b, int32_t index, const uint32_t** runs, int32_t* n_runs,
                                    int32_t* n_ops, int32_t* edit_distance, int32_t* status) {
    if (!b || index < 0 || (size_t)index >= b->jobs.size()) return B200ALN_INVALID_ARGUMENT;
    if (!b->aligned || !b->synced) return B200ALN_UNINITIALIZED;
    if (runs) {
        const int32_t fs = fetch_runs(b);
        if (fs != B200ALN_SUCCESS) return fs;
    }
    const AlnResult& r = b->res[(size_t)index];
    const bool ok = r.status == 0 && r.runs_off >= 0 && (!runs ||
                    (size_t)(r.runs_off + r.n_runs) * sizeof(uint32_t) <= b->h_runs.used);
    if (runs) *runs = ok ? reinterpret_cast<const uint32_t*>(b->h_runs.p) + r.runs_off : nullptr;
    if (n_runs) *n_runs = ok ? r.n_runs : 0;
    if (n_ops) *n_ops = ok ? r.n_ops : 0;
    if (edit_distance) *edit_distance = r.score;
    if (status) *status = ok ? B200ALN_SUCCESS : (r.status ? r.status : B200ALN_GENERIC_ERROR);
    return B200ALN_SUCCESS;
}

int64_t b200aln_batch_get_cigar(const b200aln_batch* b, int32_t index, char* out, int64_t cap) {
    if (!b || index < 0 || (size_t)index >= b->jobs.size()) return -(int64_t)B200ALN_INVALID_ARGUMENT;
    if (!b->aligned || !b->synced) return -(int64_t)B200ALN_UNINITIALIZED;
    if (b->skip_cigars) return -(int64_t)B200ALN_GENERIC_ERROR;
    if (b->t_st[(size_t)index] != B200ALN_SUCCESS) return -(int64_t)b->t_st[(size_t)index];
    const int64_t len = b->t_len[(size_t)index];
    if (out && cap > 0) {
        const size_t k = (size_t)std::min<int64_t>(len, cap - 1);
        std::memcpy(out, b->h_text.p + b->t_off[(size_t)index], k);
        out[k] = 0;
    }
    return len;
}

int64_t b200aln_batch_get_ops(const b200aln_batch* b, int32_t index, uint8_t* out, int64_t cap) {
    const uint32_t* runs = nullptr;
    int32_t n_runs = 0, n_ops = 0, st = 0;
    const int32_t rc = b200aln_batch_get_alignment(b, index, &runs, &n_runs, &n_ops, nullptr, &st);
    if (rc != B200ALN_SUCCESS) return -(int64_t)rc;
    if (st != B200ALN_SUCCESS) return -(int64_t)st;
    if (out && cap > 0) {
        std::vector<uint8_t> ops;
        aln_expand_runs(runs, n_runs, n_ops, ops);
        std::memcpy(out, ops.data(), (size_t)std::min<int64_t>(cap, n_ops));
    }
    return n_ops;
}

int32_t b200aln_batch_reset(b200aln_batch* b) {
    if (!b) return B200ALN_INVALID_ARGUMENT;
    cudaSetDevice(b->device);
    if (b->aligned && !b->synced) cudaStreamSynchronize(b->stream);
    cudaGetLastError();
    b->jobs.clear();
    b->h_seq.used = 0;
    b->view_q = b->view_t = nullptr;
    b->view_q_bytes = b->view_t_bytes = 0;
    b->view_qual = nullptr;
    b->h_qual.used = 0;
    b->cut_first_window.clear();
    b->cut_t_length.clear();
    b->cut_has_q.clear();
    b->n_layers = b->cut_win_lo = b->cut_n_win = 0;
    b->export_records.clear();
    b->export_win_off.clear();
    b->export_seq_off.clear();
    b->ops_bytes = 0;
    b->n_windows = 0;
    b->h_bp.used = 0;
    b->cap_open = b->cap_leaves = 0;
    b->load = AlnLoad{};
    b->res.clear();
    b->h_runs.used = 0;
    b->h_text.used = 0;
    b->runs_on_host = false;
    b->n_runs_total = 0;
    b->aligned = b->synced = false;
    return B200ALN_SUCCESS;
}

int32_t b200aln_batch_get_info(const b200aln_batch* b, b200aln_batch_info* info) {
    if (!b || !info) return B200ALN_INVALID_ARGUMENT;
    *info = b->info;
    return B200ALN_SUCCESS;
}

int32_t b200aln_align_pairs(int32_t device_id, int64_t max_gpu_mem, int64_t n, const uint8_t* q_bases,
                            const int64_t* q_off, const uint8_t* t_bases, const int64_t* t_off, int32_t* edit_distance,
                            char* cigars, int64_t cigar_cap, int64_t* cigar_off, b200aln_batch_info* info) {
    if (n < 0 || (n > 0 && (!q_bases || !q_off || !t_bases || !t_off || !cigar_off))) return B200ALN_INVALID_ARGUMENT;
    b200aln_batch* b = nullptr;
    int32_t st = b200aln_batch_create(device_id, nullptr, max_gpu_mem, 0, &b);
    if (st != B200ALN_SUCCESS) return st;
    b200aln_batch_info total{};
    total.device_id = device_id;
    int64_t done = 0, used = 0;
    bool too_small = false;
    if (n > 0) cigar_off[0] = 0;
    while (done < n && st == B200ALN_SUCCESS) {
        int64_t k = done;
        for (; k < n; ++k) {
            const int32_t rc = b200aln_batch_add_alignment(b, reinterpret_cast<const char*>(q_bases + q_off[k]),
                                                           (int32_t)(q_off[k + 1] - q_off[k]),
                                                           reinterpret_cast<const char*>(t_bases + t_off[k]),
                                                           (int32_t)(t_off[k + 1] - t_off[k]));
            if (rc == B200ALN_EXCEEDED_MAX_ALIGNMENTS && k > done) break;
            if (rc != B200ALN_SUCCESS) { st = rc == B200ALN_EXCEEDED_MAX_ALIGNMENTS ? B200ALN_EXCEEDED_MAX_LENGTH : rc; break; }
        }
        if (st != B200ALN_SUCCESS) break;
        st = b200aln_batch_align_all(b);
        if (st == B200ALN_SUCCESS) st = b200aln_batch_sync(b);
        if (st != B200ALN_SUCCESS) break;
        for (int64_t i = done; i < k; ++i) {
            int32_t ed = 0, ast = 0;
            b200aln_batch_get_alignment(b, (int32_t)(i - done), nullptr, nullptr, nullptr, &ed, &ast);
            if (ast != B200ALN_SUCCESS) { st = ast; break; }
            if (edit_distance) edit_distance[i] = ed;
            const int64_t room = too_small ? 0 : cigar_cap - used;
            const int64_t len = b200aln_batch_get_cigar(b, (int32_t)(i - done), room > 0 ? cigars + used : nullptr, room);
            if (len < 0) { st = (int32_t)-len; break; }
            if (len + 1 > room) too_small = true;
            used += len + 1;
            cigar_off[i + 1] = used;
        }
        b200aln_batch_info bi;
        b200aln_batch_get_info(b, &bi);
        total.n_slots = bi.n_slots;
        total.n_team_blocks = bi.n_team_blocks;
        total.team_launches += bi.team_launches;
        total.levels = std::max(total.levels, bi.levels);
        total.kernel_launches += bi.kernel_launches;
        total.n_open += bi.n_open;
        total.n_leaves += bi.n_leaves;
        total.cells += bi.cells;
        total.h2d_bytes += bi.h2d_bytes;
        total.d2h_bytes += bi.d2h_bytes;
        total.kernel_ms += bi.kernel_ms;
        b200aln_batch_reset(b);
        done = k;
    }
    b200aln_batch_destroy(b);
    if (info) *info = total;
    if (st == B200ALN_SUCCESS && too_small) return B200ALN_EXCEEDED_MAX_LENGTH;
    return st;
}

/* ------------------------------------------------------------------------------------------ */
/* aligner pool: the GPU section of CUDAPolisher::find_overlap_breaking_points (cudapolisher.cpp:74-214) -- several
 * batches per device, several devices, one host thread per batch filling, aligning and emptying it -- over columnar
 * segments.  While one batch's kernels run, the other batches' threads stage, upload and copy results out.         */
/* ------------------------------------------------------------------------------------------ */
struct b200aln_aligner {
    std::vector<b200aln_batch*> batches;
};

void b200aln_aligner_destroy(b200aln_aligner* h) {
    if (!h) return;
    for (b200aln_batch* b : h->batches) b200aln_batch_destroy(b);
    delete h;
}

int32_t b200aln_aligner_create(int32_t n_devices, const int32_t* device_ids, int32_t batches_per_device,
                               int64_t max_gpu_mem_per_batch, b200aln_aligner** out) {
    if (!out) return B200ALN_INVALID_ARGUMENT;
    *out = nullptr;
    if (n_devices <= 0 || !device_ids || batches_per_device <= 0 || batches_per_device > 16) return B200ALN_INVALID_ARGUMENT;
    b200aln_aligner* h = new (std::nothrow) b200aln_aligner();
    if (!h) return B200ALN_GENERIC_ERROR;
    for (int32_t d = 0; d < n_devices; ++d) {
        int64_t per_batch = max_gpu_mem_per_batch;
        if (per_batch <= 0) { /* like racon: 90 % of the device's free memory, split between its batches (cudapolisher.cpp:118-123) */
            size_t free_b = 0, total_b = 0;
            if (cudaSetDevice(device_ids[d]) != cudaSuccess || cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) {
                cudaGetLastError();
                b200aln_aligner_destroy(h);
                return B200ALN_CUDA_ERROR;
            }
            int32_t same = 0; /* the same device may be listed more than once */
            for (int32_t e = 0; e < n_devices; ++e) same += device_ids[e] == device_ids[d];
            per_batch = (int64_t)((double)free_b * 0.9) / ((int64_t)batches_per_device * same);
        }
        for (int32_t k = 0; k < batches_per_device; ++k) {
            b200aln_batch* b = nullptr;
            const int32_t st = b200aln_batch_create(device_ids[d], nullptr, per_batch, 0, &b);
            if (st != B200ALN_SUCCESS) {
                b200aln_aligner_destroy(h);
                return st;
            }
            h->batches.push_back(b);
        }
    }
    *out = h;
    return B200ALN_SUCCESS;
}

int32_t b200aln_aligner_num_batches(const b200aln_aligner* h) { return h ? (int32_t)h->batches.size() : 0; }

int32_t b200aln_aligner_align(b200aln_aligner* h, int64_t n, const uint8_t* q_bases, const int64_t* q_off,
                              const uint8_t* t_bases, const int64_t* t_off, int32_t* edit_distance, char* cigars,
                              int64_t cigar_cap, int64_t* cigar_off, int32_t* cigar_len, int64_t* cigar_bytes,
                              b200aln_batch_info* info) {
    if (cigar_bytes) *cigar_bytes = 0;
    if (!h || h->batches.empty() || n < 0) return B200ALN_INVALID_ARGUMENT;
    if (n > 0 && (!q_bases || !q_off || !t_bases || !t_off || !cigar_off || !cigar_len || (cigar_cap > 0 && !cigars)))
        return B200ALN_INVALID_ARGUMENT;
    const int32_t workers = (int32_t)h->batches.size();
    /* chunks: large enough that a batch's levels fill the device (a thin level is bound by its longest sub-problem, not by
     * throughput), small enough that the batches take turns: about 1.5e11 matrix cells (10 ms of kernels) or more each */
    double cells = 0;
    for (int64_t k = 0; k < n; ++k) cells += (double)(q_off[k + 1] - q_off[k]) * (double)(t_off[k + 1] - t_off[k]);
    const int64_t n_chunks = std::max<int64_t>(1, std::min<int64_t>(4 * (int64_t)workers, (int64_t)(cells / 1.5e11)));
    const int64_t chunk = std::max<int64_t>(1, (n + n_chunks - 1) / n_chunks);
    std::atomic<int64_t> next{0}, used{0};
    std::atomic<int32_t> first_error{B200ALN_SUCCESS};
    std::vector<b200aln_batch_info> infos((size_t)workers);
    auto work = [&](int32_t w) {
        b200aln_batch* b = h->batches[(size_t)w];
        b200aln_batch_info acc{};
        b200aln_batch_get_info(b, &acc);
        acc.levels = acc.kernel_launches = acc.team_launches = 0;
        acc.n_open = acc.n_leaves = acc.cells = acc.h2d_bytes = acc.d2h_bytes = 0;
        acc.kernel_ms = 0.f;
        b200aln_batch_reset(b);
        for (;;) {
            if (first_error.load() != B200ALN_SUCCESS) break;
            const int64_t start = next.fetch_add(chunk);
            if (start >= n) break;
            const int64_t end = std::min(n, start + chunk);
            int64_t pos = start;
            while (pos < end) {
                int64_t added = 0;
                int32_t st = b200aln_batch_add_overlaps_view(b, end - pos, q_bases, q_off + pos, t_bases, t_off + pos, nullptr, nullptr, &added);
                if (st == B200ALN_SUCCESS) st = b200aln_batch_align_all(b);
                if (st == B200ALN_SUCCESS) st = b200aln_batch_sync(b);
                const char* text = nullptr;
                const int64_t* off = nullptr;
                const int32_t *len = nullptr, *ed = nullptr, *ast = nullptr;
                if (st == B200ALN_SUCCESS) st = b200aln_batch_get_cigars(b, &text, &off, &len, &ed, &ast);
                if (st == B200ALN_SUCCESS) {
                    /* one reservation and one copy per batch: the batch's text arena as it is; strings end with a 0 */
                    const int64_t bytes = (int64_t)b->h_text.used;
                    const int64_t base = used.fetch_add(bytes);
                    const bool fits = base + bytes <= cigar_cap;
                    if (fits && bytes) std::memcpy(cigars + base, text, (size_t)bytes);
                    for (int64_t k = 0; k < added; ++k) {
                        if (ast[k] != B200ALN_SUCCESS) st = ast[k];
                        if (edit_distance) edit_distance[pos + k] = ed[k];
                        cigar_off[pos + k] = fits ? base + off[k] : -1;
                        cigar_len[pos + k] = len[k];
                    }
                }
                b200aln_batch_info bi;
                b200aln_batch_get_info(b, &bi);
                acc.levels = std::max(acc.levels, bi.levels);
                acc.kernel_launches += bi.kernel_launches;
                acc.team_launches += bi.team_launches;
                acc.n_open += bi.n_open;
                acc.n_leaves += bi.n_leaves;
                acc.cells += bi.cells;
                acc.h2d_bytes += bi.h2d_bytes;
                acc.d2h_bytes += bi.d2h_bytes;
                acc.kernel_ms += bi.kernel_ms;
                b200aln_batch_reset(b);
                if (st != B200ALN_SUCCESS) {
                    int32_t expect = B200ALN_SUCCESS;
                    first_error.compare_exchange_strong(expect, st);
                    break;
                }
                pos += added;
            }
        }
        infos[(size_t)w] = acc;
    };
    std::vector<std::thread> threads;
    for (int32_t w = 1; w < workers; ++w) threads.emplace_back(work, w);
    work(0);
    for (std::thread& t : threads) t.join();
    if (info) {
        b200aln_batch_info total = infos[0];
        for (int32_t w = 1; w < workers; ++w) {
            const b200aln_batch_info& x = infos[(size_t)w];
            total.levels = std::max(total.levels, x.levels);
            total.kernel_launches += x.kernel_launches;
            total.team_launches += x.team_launches;
            total.n_open += x.n_open;
            total.n_leaves += x.n_leaves;
            total.cells += x.cells;
            total.h2d_bytes += x.h2d_bytes;
            total.d2h_bytes += x.d2h_bytes;
            total.kernel_ms += x.kernel_ms; /* launches of different batches overlap: a sum of device times, not a span */
        }
        *info = total;
    }
    if (cigar_bytes) *cigar_bytes = used.load();
    const int32_t st = first_error.load();
    if (st != B200ALN_SUCCESS) return st;
    return used.load() > cigar_cap ? B200ALN_EXCEEDED_MAX_LENGTH : B200ALN_SUCCESS;
}

} // extern "C"

#if ALN_SPLIT_DIGEST
/* test build only (not part of include/b200aln.h): the split log of the last align_all, one AlnSplitRec per split
 * attempt in the order the kernels appended them.  *count = records appended; *rec_bytes = sizeof(AlnSplitRec).  Copies
 * min(count, cap) records to out (nullable).  B200ALN_GENERIC_ERROR when the log overflowed (count > its capacity: the
 * records beyond it are lost).  Synchronises. */
extern "C" int32_t b200aln_debug_split_log(b200aln_batch* b, void* out, int64_t cap, int64_t* count, int32_t* rec_bytes) {
    if (!b || !count) return B200ALN_INVALID_ARGUMENT;
    if (rec_bytes) *rec_bytes = (int32_t)sizeof(AlnSplitRec);
    *count = 0;
    if (!b->aligned || !b->d_log.p) return B200ALN_UNINITIALIZED;
    ALN_CU(cudaSetDevice(b->device));
    ALN_CU(cudaStreamSynchronize(b->stream));
    int32_t n = 0;
    ALN_CU(cudaMemcpy(&n, b->d_log.p, sizeof(int32_t), cudaMemcpyDeviceToHost));
    *count = n;
    const int64_t k = std::min<int64_t>(std::min<int64_t>(n, b->log_cap), cap);
    if (out && k > 0)
        ALN_CU(cudaMemcpy(out, static_cast<AlnSplitRec*>(b->d_log.p) + 1, sizeof(AlnSplitRec) * (size_t)k, cudaMemcpyDeviceToHost));
    return n > b->log_cap ? B200ALN_GENERIC_ERROR : B200ALN_SUCCESS;
}
#endif

#if ALN_LEAF_DIGEST
/* test build only (not part of include/b200aln.h): the leaf log of the last align_all, one AlnLeafRec per leaf in the
 * order the leaf kernel appended them.  Same contract as b200aln_debug_split_log. */
extern "C" int32_t b200aln_debug_leaf_log(b200aln_batch* b, void* out, int64_t cap, int64_t* count, int32_t* rec_bytes) {
    if (!b || !count) return B200ALN_INVALID_ARGUMENT;
    if (rec_bytes) *rec_bytes = (int32_t)sizeof(AlnLeafRec);
    *count = 0;
    if (!b->aligned || !b->d_leaf_log.p) return B200ALN_UNINITIALIZED;
    ALN_CU(cudaSetDevice(b->device));
    ALN_CU(cudaStreamSynchronize(b->stream));
    int32_t n = 0;
    ALN_CU(cudaMemcpy(&n, b->d_leaf_log.p, sizeof(int32_t), cudaMemcpyDeviceToHost));
    *count = n;
    const int64_t k = std::min<int64_t>(std::min<int64_t>(n, b->leaf_log_cap), cap);
    if (out && k > 0)
        ALN_CU(cudaMemcpy(out, static_cast<AlnLeafRec*>(b->d_leaf_log.p) + 1, sizeof(AlnLeafRec) * (size_t)k, cudaMemcpyDeviceToHost));
    return n > b->leaf_log_cap ? B200ALN_GENERIC_ERROR : B200ALN_SUCCESS;
}
#endif
