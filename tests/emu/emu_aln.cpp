/*
 * emu_aln.cpp -- lock-step CPU emulation of the overlap aligner (TEST INFRASTRUCTURE).
 *
 * Compiles racon_gpu_b200/csrc/aln_core.cuh in its host flavour (poa_simt.cuh: POA_LANES loops over 32 lanes, shuffles
 * are plain loops) and drives it level by level exactly like the batch runtime (csrc/b200aln.cu) does on the device --
 * aln_push files the children, the leaf list is traced back at the end, aln_runs forms the runs -- so that the wavefront
 * bit-vector passes, the split rule, the leaf records, the traceback and the run formation are checked against the
 * oracle / the unmodified edlib without a GPU.  Never linked into the product library.
 */
#include <atomic>
#include <cstdarg>
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <random>
#include <string>
#include <thread>
#include <vector>

#include "../../racon_gpu_b200/csrc/host/aln_levels.hpp"

using namespace b200aln;

/* ------------------------------------------------------------------------------------------
 * Teams on threads (built with ALN_EMU_TEAMS=1, aln_core.cuh: Teams).  One AlnEmuTeam per pass direction, like one
 * half of aln_split_team_kernel's block: ALN_TEAM threads ("warps"), the ring of ALN_TEAM hand-over rows, ALN_TEAM
 * progress words.  Progress words and hand-over rows persist from pass to pass, as on the device, so a pass that skipped
 * its reset would read the previous pass's state.  The protocol checker:
 *   - every hand-over word has a shadow tag (pass, stripe) of its last writer; a load must find the stripe it names,
 *     written in the current pass (catches reads before the write, stale words, and words overwritten too early);
 *   - every warp keeps the target of its last team_wait; a load of a word those columns do not cover fails, whatever the
 *     schedule (the wait contract).
 * team_wait yields at random (seeded per warp) and gives up after a timeout instead of hanging.
 * ---------------------------------------------------------------------------------------- */
namespace b200aln {
struct AlnEmuTeam {
    int32_t n = ALN_TEAM;
    const uint32_t* hbuf = nullptr;
    int64_t words = 0, hrow_words = 0;
    std::unique_ptr<std::atomic<uint64_t>[]> tag; /* (pass + 1) << 32 | stripe; 0: never written */
    std::atomic<uint64_t> prog[ALN_TEAM];
    int64_t pass = 0;
    double timeout_s = 20.0;
    std::chrono::steady_clock::time_point t0;
    /* barrier */
    std::mutex mu;
    std::condition_variable cv;
    int32_t arrived = 0;
    int64_t generation = 0;
    /* per warp (written by its own thread only) */
    int32_t wait_stripe[ALN_TEAM], wait_cols[ALN_TEAM];
    std::mt19937_64 rng[ALN_TEAM];
    /* what the pass ran */
    std::atomic<int32_t> stripes{0}, left_matrix{0}, anchors{0}, other{0}, waits{0};
    /* failures: the first message is kept */
    std::atomic<int32_t> failures{0}, timeouts{0};
    std::string first;

    void fail(const char* fmt, ...) __attribute__((format(printf, 2, 3)));
};
void AlnEmuTeam::fail(const char* fmt, ...) {
    failures.fetch_add(1);
    std::lock_guard<std::mutex> g(mu);
    if (!first.empty()) return;
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    first = buf;
}
static bool emu_timed_out(AlnEmuTeam* e) {
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - e->t0).count() > e->timeout_s;
}
static void emu_jitter(AlnEmuTeam* e, int32_t w, int one_in) {
    const uint64_t x = e->rng[w]();
    if (x % (uint64_t)one_in) return;
    if ((x >> 20) & 1) std::this_thread::yield();
    else std::this_thread::sleep_for(std::chrono::microseconds((x >> 24) % 40));
}
void aln_emu_barrier(AlnEmuTeam* e, int32_t w) {
    emu_jitter(e, w, 2);
    std::unique_lock<std::mutex> g(e->mu);
    const int64_t gen = e->generation;
    if (++e->arrived == e->n) {
        e->arrived = 0;
        ++e->generation;
        e->cv.notify_all();
        return;
    }
    while (e->generation == gen) {
        if (e->cv.wait_for(g, std::chrono::milliseconds(100)) == std::cv_status::timeout && emu_timed_out(e)) {
            e->timeouts.fetch_add(1);
            return;
        }
    }
}
void aln_emu_publish(AlnEmuTeam* e, int32_t w, int32_t stripe, int32_t cols_done) {
    emu_jitter(e, w, 16);
    e->prog[w].store(((uint64_t)(uint32_t)stripe << 32) | (uint32_t)cols_done, std::memory_order_release);
}
void aln_emu_wait(AlnEmuTeam* e, int32_t w, int32_t stripe, int32_t cols_needed) {
    const uint64_t target = ((uint64_t)(uint32_t)stripe << 32) | (uint32_t)cols_needed;
    emu_jitter(e, w, 4);
    e->waits.fetch_add(1, std::memory_order_relaxed);
    for (uint64_t polls = 0; e->prog[stripe % e->n].load(std::memory_order_acquire) < target; ++polls) {
        std::this_thread::yield();
        if ((polls & 1023) == 1023 && emu_timed_out(e)) {
            e->timeouts.fetch_add(1);
            e->fail("pass %lld warp %d: team_wait for stripe %d, %d columns timed out", (long long)e->pass, w, stripe, cols_needed);
            break;
        }
    }
    e->wait_stripe[w] = stripe;
    e->wait_cols[w] = cols_needed;
}
void aln_emu_hrow_store(AlnEmuTeam* e, int32_t w, const uint32_t* p, int32_t stripe) {
    const int64_t k = p - e->hbuf;
    if (k < 0 || k >= e->words) {
        e->fail("pass %lld warp %d stripe %d: store outside the hand-over rows (word %lld)", (long long)e->pass, w, stripe, (long long)k);
        return;
    }
    e->tag[k].store(((uint64_t)(e->pass + 1) << 32) | (uint32_t)stripe, std::memory_order_relaxed);
}
void aln_emu_hrow_load(AlnEmuTeam* e, int32_t w, const uint32_t* p, int32_t stripe, int32_t cols_needed) {
    const int64_t k = p - e->hbuf;
    if (k < 0 || k >= e->words) {
        e->fail("pass %lld warp %d stripe %d: load outside the hand-over rows (word %lld)", (long long)e->pass, w, stripe + 1, (long long)k);
        return;
    }
    const bool anchor = k % e->hrow_words == e->hrow_words - 1;
    if (anchor) e->anchors.fetch_add(1, std::memory_order_relaxed);
    const uint64_t t = e->tag[k].load(std::memory_order_relaxed);
    const uint64_t want = ((uint64_t)(e->pass + 1) << 32) | (uint32_t)stripe;
    if (t != want)
        e->fail("pass %lld warp %d stripe %d: %s (ring row %lld word %lld) holds pass %lld stripe %d, expected stripe %d of this pass",
                (long long)e->pass, w, stripe + 1, anchor ? "the anchor" : "a hand-over word", (long long)(k / e->hrow_words),
                (long long)(k % e->hrow_words), (long long)(t >> 32) - 1, t ? (int32_t)(uint32_t)t : -1, stripe);
    if (e->n > 1 && (e->wait_stripe[w] != stripe || e->wait_cols[w] < cols_needed))
        e->fail("pass %lld warp %d stripe %d: loads %s (word %lld) that needs %d columns of stripe %d, but its last team_wait "
                "was for %d columns of stripe %d",
                (long long)e->pass, w, stripe + 1, anchor ? "the anchor" : "a hand-over word", (long long)(k % e->hrow_words),
                cols_needed, stripe, e->wait_cols[w], e->wait_stripe[w]);
}
void aln_emu_stripe(AlnEmuTeam* e, int32_t w, int32_t stripe, int32_t c_lo, int32_t c_hi, bool has_other) {
    (void)w; (void)stripe;
    e->stripes.fetch_add(1, std::memory_order_relaxed);
    if (c_lo > c_hi) e->left_matrix.fetch_add(1, std::memory_order_relaxed);
    if (has_other) e->other.fetch_add(1, std::memory_order_relaxed);
}
} // namespace b200aln

/* the workspace of one emulated team block: like TeamSlot (csrc/b200aln.cu), for sequences up to max_len */
struct EmuTeamBlock {
    int32_t max_len, hrow_words;
    std::vector<uint32_t> hrow[2];
    std::vector<uint8_t> tcode[2];
    std::vector<int32_t> Lc, Rr;
    AlnEmuTeam team[2];
    int64_t passes = 0;
    explicit EmuTeamBlock(int32_t len) : max_len(len), hrow_words((int32_t)aln_hrow_words(len)) {
        for (int k = 0; k < 2; ++k) {
            hrow[k].assign((size_t)hrow_words * ALN_TEAM, 0xDEADBEEFu); /* never-written words: garbage, tag 0 */
            tcode[k].assign((size_t)len + 192, 0);
            AlnEmuTeam& e = team[k];
            e.hbuf = hrow[k].data();
            e.hrow_words = hrow_words;
            e.words = (int64_t)hrow_words * ALN_TEAM;
            e.tag.reset(new std::atomic<uint64_t>[(size_t)e.words]);
            for (int64_t i = 0; i < e.words; ++i) e.tag[i].store(0);
            for (int w = 0; w < ALN_TEAM; ++w) e.prog[w].store(0);
        }
        Lc.assign((size_t)len + 2, 0);
        Rr.assign((size_t)len + 2, 0);
    }
    /* both passes of one attempt, 2 x ALN_TEAM threads like aln_split_team_kernel's block */
    void passes_of(const uint8_t* q, int32_t n, const uint8_t* t, int32_t m, int32_t band, uint64_t seed) {
        const int32_t lh = m / 2, rh = m - lh;
        for (int k = 0; k < 2; ++k) {
            AlnEmuTeam& e = team[k];
            e.pass = passes;
            e.t0 = std::chrono::steady_clock::now();
            for (int w = 0; w < ALN_TEAM; ++w) {
                e.wait_stripe[w] = e.wait_cols[w] = -1;
                e.rng[w].seed(seed * 0x9E3779B97F4A7C15ull + (uint64_t)(2 * passes + k) * 131 + (uint64_t)w);
            }
        }
        ++passes;
        std::vector<std::thread> th;
        for (int side = 0; side < 2; ++side) {
            for (int w = 0; w < ALN_TEAM; ++w) {
                th.emplace_back([=]() {
                    EqTab eq;
                    TeamCtx c{w, ALN_TEAM, 1 + side, 0};
                    c.emu = &team[side];
                    if (side == 0)
                        myers_pass<true>(SeqView{q, 1}, n, SeqView{t, 1}, lh, band, c, hrow[0].data(), hrow_words, tcode[0].data(), eq,
                                         Lc.data(), nullptr, nullptr);
                    else
                        myers_pass<true>(SeqView{q + (n - 1), -1}, n, SeqView{t + (m - 1), -1}, rh, band, c, hrow[1].data(),
                                         hrow_words, tcode[1].data(), eq, Rr.data(), nullptr, nullptr);
                });
            }
        }
        for (std::thread& x : th) x.join();
    }
};

static AlnSplitRec split_record(const AlnRect& r, int32_t band, int32_t attempt, int32_t level, int32_t path, const AlnSplit& sp,
                                const int32_t* Lc, const int32_t* Rr) {
    AlnSplitRec x;
    std::memset(&x, 0, sizeof x);
    x.aln = r.aln;
    x.r0 = r.r0;
    x.c0 = r.c0;
    x.n = r.n;
    x.m = r.m;
    x.band = band;
    x.attempt = attempt;
    x.level = level;
    x.path = path;
    x.r = sp.r;
    x.ls = sp.ls;
    x.rs = sp.rs;
    x.best = sp.best;
    x.lc_hash = aln_col_digest(Lc, r.n);
    x.rr_hash = aln_col_digest(Rr, r.n);
    return x;
}

extern "C" {

int32_t emu_split_rec_bytes(void) { return (int32_t)sizeof(AlnSplitRec); }

/* One Hirschberg step of an n x m sub-problem the way a split kernel runs it: mode 0 on one warp (aln_split_kernel),
 * mode 1 on a team block of 2 x ALN_TEAM threads (aln_split_team_kernel), then the split rule and the same redo rule:
 * best < 0 runs without a band; guess != 0 marks best as the host's guess, and a pass whose optimum proves larger is
 * redone without a band.  Per attempt a: Lc[a (n + 1) + i], Rr[a (n + 1) + i] (i = 0..n), split[4 a ..] = r, ls, rs,
 * best, band_out[a] = the band myers_pass got.  Team mode: stats[7] (nullable) = stripes run, stripes whose strip left the
 * matrix, anchor loads, stripes of a target with letters outside ACGT, team_waits, protocol failures, timeouts, summed
 * over the attempts of both teams; msg (nullable) the first failure.  Returns the number of attempts. */
int32_t emu_split(const uint8_t* q, int32_t n, const uint8_t* t, int32_t m, int32_t best, int32_t guess, int32_t mode, uint64_t seed,
                  int32_t* Lc, int32_t* Rr, int32_t* split, int32_t* band_out, int64_t* stats, char* msg, int32_t msg_cap) {
    const int32_t max_len = (n > m ? n : m) + 1;
    std::unique_ptr<EmuTeamBlock> blk;
    std::vector<uint8_t> slab;
    AlnSlot s;
    EqTab eq;
    if (mode == 1) {
        blk.reset(new EmuTeamBlock(max_len));
    } else {
        size_t slot_bytes = 0;
        aln_slot_bind(s, nullptr, max_len, &slot_bytes);
        slab.resize(slot_bytes + 512);
        aln_slot_bind(s, reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(slab.data()) + 255) & ~uintptr_t(255)), max_len, nullptr);
    }
    int32_t attempts = 0;
    for (int32_t attempt = 0; attempt < 2; ++attempt) {
        const int32_t band = attempt == 0 ? aln_band_of(best) : -1;
        AlnSplit sp;
        const int32_t *lc, *rr;
        if (mode == 1) {
            blk->passes_of(q, n, t, m, band, seed);
            aln_split_rule(blk->Lc.data(), blk->Rr.data(), n, m, &sp);
            lc = blk->Lc.data();
            rr = blk->Rr.data();
        } else {
            aln_split(s, eq, q, t, n, m, band, &sp);
            lc = s.Lc;
            rr = s.Rr;
        }
        std::memcpy(Lc + (size_t)attempt * (n + 1), lc, sizeof(int32_t) * ((size_t)n + 1));
        std::memcpy(Rr + (size_t)attempt * (n + 1), rr, sizeof(int32_t) * ((size_t)n + 1));
        split[4 * attempt] = sp.r;
        split[4 * attempt + 1] = sp.ls;
        split[4 * attempt + 2] = sp.rs;
        split[4 * attempt + 3] = sp.best;
        band_out[attempt] = band;
        attempts = attempt + 1;
        if (!(guess && sp.best > best)) break;
    }
    if (mode == 1) {
        if (stats) {
            for (int k = 0; k < 7; ++k) stats[k] = 0;
            for (const AlnEmuTeam& e : blk->team) {
                stats[0] += e.stripes;
                stats[1] += e.left_matrix;
                stats[2] += e.anchors;
                stats[3] += e.other;
                stats[4] += e.waits;
                stats[5] += e.failures;
                stats[6] += e.timeouts;
            }
        }
        if (msg && msg_cap > 0) {
            const std::string& f = !blk->team[0].first.empty() ? blk->team[0].first : blk->team[1].first;
            std::snprintf(msg, (size_t)msg_cap, "%s%s", f.empty() ? "" : (blk->team[0].first.empty() ? "backward pass: " : "forward pass: "),
                          f.c_str());
        }
    }
    return attempts;
}

int32_t emu_leaf_rec_bytes(void) { return (int32_t)sizeof(AlnLeafRec); }

/* aln_ops_digest of len bytes (the hash the leaf records carry) */
uint64_t emu_ops_digest(const uint8_t* ops, int32_t len) { return aln_ops_digest(ops, len); }

/* a slab for one slot of sequences up to max_len, 256-byte aligned like the device's */
static uint8_t* emu_slot(std::vector<uint8_t>& slab, AlnSlot& s, int32_t max_len, size_t* bytes) {
    size_t slot_bytes = 0;
    aln_slot_bind(s, nullptr, max_len, &slot_bytes);
    slab.assign(slot_bytes + 512, 0);
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(slab.data()) + 255) & ~uintptr_t(255));
    aln_slot_bind(s, base, max_len, nullptr);
    if (bytes) *bytes = slot_bytes;
    return base;
}

/* One leaf the way aln_leaf_kernel runs it, in a slot whose whole workspace (hand-over row, code row, columns, leaf
 * records, scores, pre) first holds: poison 0 zeros, 1 0xFF bytes, 2 0xA5 bytes, 3 seeded random bytes, 4 seeded random
 * bytes and then the leftovers of the leaf (pq, pn, pt, pm) run in it with band pband.  ops_out: the leaf's (n + m)-byte
 * region, holes OP_NONE; *rec its record (aln, r0, c0, top 0).  Returns the cells the pass computed. */
int64_t emu_leaf(const uint8_t* q, int32_t n, const uint8_t* t, int32_t m, int32_t band, int32_t poison, uint64_t seed,
                 const uint8_t* pq, int32_t pn, const uint8_t* pt, int32_t pm, int32_t pband, uint8_t* ops_out, AlnLeafRec* rec) {
    int32_t max_len = (n > m ? n : m) + 1;
    if (poison == 4 && (pn > pm ? pn : pm) + 1 > max_len) max_len = (pn > pm ? pn : pm) + 1;
    std::vector<uint8_t> slab;
    AlnSlot s;
    EqTab eq;
    size_t bytes = 0;
    uint8_t* base = emu_slot(slab, s, max_len, &bytes);
    if (poison == 0 || poison == 1 || poison == 2) {
        std::memset(base, poison == 0 ? 0x00 : poison == 1 ? 0xFF : 0xA5, bytes);
    } else {
        std::mt19937_64 rng(seed);
        for (size_t k = 0; k < bytes; ++k) base[k] = (uint8_t)(rng() >> 56);
    }
    if (poison == 4) {
        std::vector<uint8_t> other((size_t)pn + (size_t)pm + 1, OP_NONE);
        AlnLeafRec x;
        aln_leaf(s, eq, pq, pt, pn, pm, pband, other.data(), nullptr, &x);
    }
    std::memset(ops_out, OP_NONE, (size_t)n + (size_t)m);
    std::memset(rec, 0, sizeof *rec);
    const int64_t cells = aln_leaf(s, eq, q, t, n, m, band, ops_out, nullptr, rec);
    rec->aln = rec->r0 = rec->c0 = rec->top = 0;
    return cells;
}

/* Aligns one pair; ops_out must hold n + m bytes.  Returns the number of operations (holes removed); -1 inconsistent
 * split, -2 list overflow, -3 the runs do not spell the operations.  *score the edit distance; *levels (nullable) the
 * depth of the recursion; *n_leaves likewise; cigar_out (nullable, cigar_cap bytes) the CIGAR formed from the runs;
 * bp_out (nullable, 4 words per window of the target segment) the breaking points for window_length;
 * guess (< 0: none) a guessed bound on the edit distance: the top sub-problem runs banded and is redone without a band when
 * its optimum turns out larger (what the kernels do with the host's guess).  log (nullable, log_cap records): one record
 * per split attempt like the device's split log (b200aln_debug_split_log), alignment index aln_index, path one warp;
 * *log_count = records written (more than log_cap: the rest were dropped).  leaf_log (nullable, leaf_cap records): one
 * record per leaf like the device's leaf log (b200aln_debug_leaf_log); *leaf_count = leaves. */
int64_t emu_align(const uint8_t* q, int32_t n, const uint8_t* t, int32_t m, uint8_t* ops_out, int32_t* score,
                  int32_t* levels, int32_t* n_leaves, char* cigar_out, int64_t cigar_cap, int32_t q_first, int32_t t_begin,
                  int32_t window_length, uint32_t* bp_out, int32_t* bp_count, int32_t guess, int32_t aln_index,
                  AlnSplitRec* log, int64_t log_cap, int64_t* log_count, AlnLeafRec* leaf_log, int64_t leaf_cap,
                  int64_t* leaf_count) {
    const int32_t max_len = (n > m ? n : m) + 1;
    size_t slot_bytes = 0;
    AlnSlot s;
    EqTab eq;
    aln_slot_bind(s, nullptr, max_len, &slot_bytes);
    std::vector<uint8_t> slab(slot_bytes + 512);
    aln_slot_bind(s, reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(slab.data()) + 255) & ~uintptr_t(255)), max_len, nullptr);
    std::vector<uint8_t> ops((size_t)n + (size_t)m, OP_NONE);
    const int32_t cap_open = (int32_t)aln_open_capacity(n, m), cap_leaves = (int32_t)aln_leaf_capacity(n, m);
    std::vector<AlnRect> level[ALN_CLASSES], next[ALN_CLASSES], leaves((size_t)cap_leaves);
    int32_t n_level[ALN_CLASSES] = {0, 0, 0}, n_next[ALN_CLASSES] = {0, 0, 0}, n_leaf = 0, overflow = 0, depth = 0;
    AlnLists first, L;
    for (int c = 0; c < ALN_CLASSES; ++c) {
        level[c].resize((size_t)cap_open);
        next[c].resize((size_t)cap_open);
    }
    auto bind = [&](AlnLists& x, std::vector<AlnRect>* lists, int32_t* counts) {
        for (int c = 0; c < ALN_CLASSES; ++c) x.open[c] = lists[c].data();
        x.n_open = counts;
        x.cap_open = cap_open;
        x.leaves = leaves.data();
        x.n_leaves = &n_leaf;
        x.cap_leaves = cap_leaves;
        x.overflow = &overflow;
    };
    bind(first, level, n_level);
    aln_push(first, AlnRect{aln_index, 0, n, 0, m, guess >= 0 ? (ALN_TOP | ALN_GUESS) : ALN_TOP, guess >= 0 ? guess : -1});
    int64_t n_log = 0;
    const auto log_split = [&](const AlnRect& r, int32_t band, int32_t attempt, const AlnSplit& sp) {
        if (log && n_log < log_cap) log[n_log] = split_record(r, band, attempt, depth, ALN_PATH_WARP, sp, s.Lc, s.Rr);
        ++n_log;
    };
    while (n_level[0] + n_level[1] + n_level[2] > 0) {
        n_next[0] = n_next[1] = n_next[2] = 0;
        bind(L, next, n_next);
        for (int c = 0; c < ALN_CLASSES; ++c) { /* the emulation runs tall and huge sub-problems on one warp as well */
            for (int32_t k = 0; k < n_level[c]; ++k) {
                const AlnRect r = level[c][(size_t)k];
                AlnSplit sp;
                aln_split(s, eq, q + r.r0, t + r.c0, r.n, r.m, aln_band_of(r.best), &sp);
                log_split(r, aln_band_of(r.best), 0, sp);
                if ((r.top & ALN_GUESS) && sp.best > r.best) { /* the guess was too small: nothing of that pass can be trusted */
                    aln_split(s, eq, q + r.r0, t + r.c0, r.n, r.m, -1, &sp);
                    log_split(r, -1, 1, sp);
                }
                if (r.top & ALN_TOP) *score = sp.best;
                AlnRect ul, lr;
                if (!aln_children(r, sp, ul, lr)) return -1;
                aln_push(L, ul);
                aln_push(L, lr);
            }
        }
        for (int c = 0; c < ALN_CLASSES; ++c) {
            level[c].swap(next[c]);
            n_level[c] = n_next[c];
        }
        ++depth;
    }
    if (overflow) return -2;
    for (int32_t k = 0; k < n_leaf; ++k) {
        const AlnRect r = leaves[(size_t)k];
        AlnLeafRec x;
        aln_leaf(s, eq, q + r.r0, t + r.c0, r.n, r.m, (r.top & ALN_GUESS) ? -1 : aln_band_of(r.best), ops.data() + r.r0 + r.c0,
                 (r.top & ALN_TOP) ? score : nullptr, &x);
        x.aln = r.aln;
        x.r0 = r.r0;
        x.c0 = r.c0;
        x.top = r.top;
        if (leaf_log && k < leaf_cap) leaf_log[k] = x;
    }
    if (leaf_count) *leaf_count = n_leaf;
    int64_t k = 0;
    for (uint8_t op : ops)
        if (op != OP_NONE) ops_out[k++] = op;
    /* the runs must spell the same operations */
    int32_t n_ops = -1;
    const int32_t n_runs = aln_runs(ops.data(), n + m, nullptr, n_ops);
    std::vector<uint32_t> runs((size_t)n_runs + 1);
    if (aln_runs(ops.data(), n + m, runs.data(), n_ops) != n_runs || n_ops != k) return -3;
    std::vector<uint8_t> spelled;
    aln_expand_runs(runs.data(), n_runs, n_ops, spelled);
    if (spelled.size() != (size_t)k || (k > 0 && std::memcmp(spelled.data(), ops_out, (size_t)k) != 0)) return -3;
    if (cigar_out) { /* the engine's own text (aln_cigar_text) must equal the host-side spelling of the runs */
        const std::string c = aln_runs_to_cigar(runs.data(), n_runs, n_ops);
        const int32_t bytes = aln_cigar_text(runs.data(), n_runs, n_ops, nullptr);
        if ((int64_t)bytes + 1 > cigar_cap || bytes != (int32_t)c.size()) return -3;
        if (aln_cigar_text(runs.data(), n_runs, n_ops, reinterpret_cast<uint8_t*>(cigar_out)) != bytes) return -3;
        cigar_out[bytes] = 0;
        if (c != cigar_out) return -3;
    }
    if (bp_out && window_length > 0) { /* breaking points from the same run starts */
        std::vector<int32_t> pre(2 * ((size_t)n_runs + 1) + 2);
        *bp_count = aln_breaking_points(runs.data(), n_runs, n_ops, q_first, t_begin, m, window_length, pre.data(), bp_out);
    }
    if (log_count) *log_count = n_log;
    if (levels) *levels = depth;
    if (n_leaves) *n_leaves = n_leaf;
    return k;
}

} // extern "C"
