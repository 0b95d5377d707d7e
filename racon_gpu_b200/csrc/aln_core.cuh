/*
 * aln_core.cuh -- batched global (Needleman-Wunsch, unit cost) alignment of overlaps with path, a warp or a team of
 * warps per sub-problem, written against poa_simt.cuh (CUDA flavour = the product, lane emulation = tests/emu).
 *
 * Replaces, for racon's overlap alignment step (src/cuda/cudapolisher.cpp:74-214, src/cuda/cudaaligner.cpp:50-98), what
 * the reference runs in vendor/GenomeWorks/cudaaligner (Aligner::align_all: Myers / Hirschberg-Myers kernels) -- but
 * with the RESULT of racon's CPU path, which is the parity target: the alignment edlib returns
 * (src/overlap.cpp:205-224; vendor/edlib/edlib/src/edlib.cpp).  Which optimal alignment that is follows from rules on
 * the plain distance matrix D (oracle/aln_oracle.c restates and pins them):
 *   - a sub-problem (n query x m target characters) is trivial (n == 0 or m == 0), traced back directly when
 *     20 * ceil(n / 64) * m + 8 * m < 2^20 (edlib.cpp:1155-1157), or split by Hirschberg at lh = m / 2 otherwise;
 *   - traceback: first possible move of up (query character alone), left (target character alone), diagonal
 *     (edlib.cpp:983-1093);
 *   - split: first query index r = 0..n-2 with L[r] + R[r+1] == optimum, else r = -1, else r = n-1 (:1282-1308).
 *
 * Design (not a port of either library):
 *   - the recursion is LEVEL-SYNCHRONOUS over the whole batch: the lists of open sub-problems live on the device, a
 *     level's launches resolve every open sub-problem (a forward and a backward bit-vector pass to the middle column, then
 *     the split rule) and file the two children by shape -- short / tall / huge, aln_shape -- into the next level's lists
 *     or the leaf list (aln_push); the host only reads a counter per shape and level.  One warp per sub-problem where a
 *     level fills the device that way; a TEAM of warps (forward and backward pass at once, stripes pipelined) per tall
 *     sub-problem where the level is thin, and per huge one always.  ONE launch then traces back all leaves of all
 *     levels, one more turns every alignment's operations into run starts, CIGAR text and (on request) racon's
 *     breaking points;
 *   - bit-vector passes (Myers 1999 / Hyyro 2003 block recurrence, 64 rows per word) run as a WAVEFRONT across the
 *     warp: lane l owns block l of a 32-block stripe (2048 rows) and works on column (step - l); the 2-bit horizontal
 *     delta of its last row travels to lane l + 1 in one shuffle per step, the column's character code comes from a code
 *     row, its match mask from the lane's shared-memory table; 16 steps to a group (immediates instead of bookkeeping).
 *     Taller sub-problems take several stripes; the last lane's deltas go to the next stripe packed 16 columns to a word;
 *   - bands only where they are exact: a sub-problem whose optimum is known (every child of a split) runs the diagonal
 *     strip that holds all values up to it, the top level a guessed strip that the split rule's result verifies; what a
 *     strip leaves out is overestimated, never underestimated, so the choice rules above see the same values (myers_pass);
 *   - a leaf stores (Pv, Mv, bottom score) per block and column -- 20 bytes, the record edlib keeps, which is why the
 *     1 MB rule bounds a leaf's workspace -- in wavefront order (coalesced), and any cell's value is
 *     bottom - popc(Pv & below) + popc(Mv & below): the traceback rates the 32 cells of the diagonal in front of the walk
 *     at once and emits whole runs of diagonal moves;
 *   - edit operations go to ops[r0 + c0 ...] of the alignment's (n + m)-byte region: sub-problems never overlap there,
 *     holes stay 0xFF and are dropped when the run starts are formed.
 */
#pragma once
#include "aln_layout.cuh"
#include "poa_simt.cuh"

namespace b200aln {
using b200poa::PerLane;
using b200poa::poa_ffs;
using b200poa::poa_uniform;
using b200poa::poa_uniform_pred;
using b200poa::warp_ballot;
using b200poa::warp_bcast0;
using b200poa::warp_exscan;
using b200poa::warp_get;
using b200poa::warp_min;
using b200poa::warp_shift_up1;

/* The match masks of a lane's block, one 64-bit word per character code, looked up once per column: shared memory on
 * the device (one LDS instead of a chain of selects; [5][32] words per warp), a plain array in the emulation. */
#define ALN_EQ_WORDS (5 * 32)
#ifndef ALN_STEP_UNROLL
#define ALN_STEP_UNROLL 16 /* 1, 2, 4, 8 or 16 */
#endif
struct EqTab {
#if POA_DEVICE
    uint32_t sa; /* shared-memory address of this warp's table */
#else
    uint64_t v[ALN_EQ_WORDS];
#endif
};
POA_FN void eq_store(EqTab& t, int code, int lane, uint64_t x) {
#if POA_DEVICE
    asm volatile("st.shared.u64 [%0], %1;" ::"r"(t.sa + (uint32_t)(code * 32 + lane) * 8u), "l"(x) : "memory");
#else
    t.v[code * 32 + lane] = x;
#endif
}
POA_FN uint64_t eq_load(const EqTab& t, int code, int lane) {
#if POA_DEVICE
    uint64_t x;
    asm volatile("ld.shared.u64 %0, [%1];" : "=l"(x) : "r"(t.sa + (uint32_t)(code * 32 + lane) * 8u) : "memory");
    return x;
#else
    return t.v[code * 32 + lane];
#endif
}

POA_FN int32_t aln_take(int32_t* counter) { /* called by ONE lane */
#if POA_DEVICE
    return atomicAdd(counter, 1);
#else
    return (*counter)++;
#endif
}
/* files a sub-problem: empty ones vanish, leaves (edlib.cpp:1135-1157) go to the leaf list, the rest stays open.  ONE lane. */
POA_FN void aln_push(const AlnLists& L, const AlnRect r) {
    if (r.n == 0 && r.m == 0) return;
    const bool leaf = aln_is_leaf(r.n, r.m);
    const int shape = aln_shape(r.n, r.m);
    const int32_t k = aln_take(leaf ? L.n_leaves : L.n_open + shape);
    if (k < (leaf ? L.cap_leaves : L.cap_open)) (leaf ? L.leaves : L.open[shape])[k] = r;
    else *L.overflow = 1;
}
/* upper-left and lower-right sub-problems of `r` split at query index sr (relative, -1 .. n-1), edlib.cpp:1321-1333 */
POA_FN bool aln_children(const AlnRect r, const AlnSplit sp, AlnRect& ul, AlnRect& lr) {
    const int32_t sr = sp.r;
    if (sr < -1 || sr > r.n - 1) return false;
    const int32_t lh = r.m / 2, uh = sr + 1;
    ul = AlnRect{r.aln, r.r0, uh, r.c0, lh, 0, sp.ls}; /* the children's optima are the two terms of the parent's */
    lr = AlnRect{r.aln, r.r0 + uh, r.n - uh, r.c0 + lh, r.m - lh, 0, sp.rs};
    return true;
}
/* The band a pass may confine itself to when nothing above `best` matters: cells with |i - j| <= best hold every value
 * <= best exactly (Ukkonen); two more diagonals so that the traceback's neighbours of path cells are computed cells. */
POA_FN int32_t aln_band_of(int32_t best) { return best < 0 ? -1 : best + 2; }

/* a sequence read forwards (step +1) or backwards (step -1): element k = p[k * step] */
struct SeqView {
    const uint8_t* p;
    int32_t step;
};
POA_FN uint8_t seq_at(const SeqView s, int32_t k) { return s.p[(int64_t)k * s.step]; }

/* a byte of the slot / the sequence arena (global memory, written earlier by this warp: a coherent load) */
POA_FN int glb_u8(const uint8_t* p) {
#if POA_DEVICE
    unsigned v;
    asm volatile("ld.global.u8 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return (int)v;
#else
    return (int)*p;
#endif
}
POA_FN int aln_popc64(uint64_t x) {
#if POA_DEVICE
    return __popcll(x);
#else
    return __builtin_popcountll(x);
#endif
}
POA_FN int aln_code(uint8_t c) { /* A C G T -> 0..3, anything else -> 4 */
    return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : 4;
}

/* where the record of (block b, column j) of a leaf with B blocks and `cols` columns lives: stripes of 32 blocks one
 * after the other, inside a stripe in wavefront order (step = j + lane, nb lanes per step) */
POA_FN int64_t leaf_entry(int32_t b, int32_t j, int32_t B, int32_t cols) {
    const int32_t s0 = b & ~31, l = b & 31;
    const int32_t nb = B - s0 < 32 ? B - s0 : 32;
    return (int64_t)s0 * (cols + 31) + (int64_t)(j + l) * nb + l;
}

/* ------------------------------------------------------------------------------------------
 * Teams.  A tall sub-problem is many stripes; stripe s + 1 needs, column by column, the horizontal deltas stripe s leaves
 * under its last row.  One warp runs the stripes one after the other (n = 1).  A TEAM of n warps of one block runs them
 * as a pipeline: warp w takes stripes w, w + n, ...; a stripe's last lane packs its deltas 16 columns to a word into the
 * stripe's hand-over row (global memory, row s mod n) and publishes its progress -- (stripe << 32 | columns done), one
 * word of shared memory per warp -- every 32 columns; the next stripe's warp polls that word before it fetches the row's
 * next word, 16 columns ahead of their use.  Producers never wait, so the pipeline cannot deadlock.
 *
 * Test builds.  ALN_EMU_TEAMS (host flavour, tests/emu only): a team's warps are threads and the primitives below call
 * the emulation's hooks (aln_emu_*): atomic progress words, a mutex / condition-variable barrier, and a protocol checker
 * -- every hand-over word carries a shadow tag (pass, stripe) of its writer, and every load names the stripe that must
 * have written it and the columns the consumer's last team_wait must cover.  ALN_SPLIT_DIGEST (device test build): a
 * team_wait gives up after ALN_WAIT_POLLS polls and flags it, so that a protocol error is a failed record, not a hung
 * block.  Neither changes the product's code: the extra arguments are ignored there.
 * ---------------------------------------------------------------------------------------- */
#ifndef ALN_TEAM
#define ALN_TEAM 4 /* warps per team (aln_split_team_kernel runs two teams: the forward and the backward pass) */
#endif
#ifndef ALN_EMU_TEAMS
#define ALN_EMU_TEAMS 0
#endif
#ifndef ALN_SPLIT_DIGEST
#define ALN_SPLIT_DIGEST 0
#endif
#ifndef ALN_LEAF_DIGEST
#define ALN_LEAF_DIGEST 0
#endif
#if ALN_EMU_TEAMS && POA_DEVICE
#error "ALN_EMU_TEAMS is the host emulation's"
#endif
#if ALN_EMU_TEAMS
struct AlnEmuTeam; /* tests/emu/emu_aln.cpp */
void aln_emu_barrier(AlnEmuTeam* e, int32_t w);
void aln_emu_publish(AlnEmuTeam* e, int32_t w, int32_t stripe, int32_t cols_done);
void aln_emu_wait(AlnEmuTeam* e, int32_t w, int32_t stripe, int32_t cols_needed);
void aln_emu_hrow_store(AlnEmuTeam* e, int32_t w, const uint32_t* p, int32_t stripe);
void aln_emu_hrow_load(AlnEmuTeam* e, int32_t w, const uint32_t* p, int32_t stripe, int32_t cols_needed);
void aln_emu_stripe(AlnEmuTeam* e, int32_t w, int32_t stripe, int32_t c_lo, int32_t c_hi, bool has_other);
#endif
#if ALN_SPLIT_DIGEST && !defined(ALN_WAIT_POLLS)
#define ALN_WAIT_POLLS (1u << 24)
#endif
struct TeamCtx {
    int32_t w, n;     /* this warp's place in its team, warps in the team (1: a warp on its own) */
    int32_t bar_id;   /* the team's named barrier (device, n > 1) */
    uint32_t prog_sa; /* shared-memory address of the team's n progress words (device, n > 1) */
#if ALN_EMU_TEAMS
    AlnEmuTeam* emu = nullptr; /* the emulated team (null: a warp on its own, nothing to check) */
#endif
#if ALN_SPLIT_DIGEST
    int32_t* timed_out = nullptr; /* set when a team_wait gave up */
#endif
};
POA_FN void team_barrier(const TeamCtx c) {
#if POA_DEVICE
    if (c.n > 1) { /* literal barrier numbers: a register id would make ptxas reserve all sixteen */
        if (c.bar_id == 1) asm volatile("bar.sync 1, %0;" ::"r"(c.n * 32) : "memory");
        else asm volatile("bar.sync 2, %0;" ::"r"(c.n * 32) : "memory");
    } else {
        __syncwarp();
    }
#elif ALN_EMU_TEAMS
    if (c.emu && c.n > 1) aln_emu_barrier(c.emu, c.w);
#else
    (void)c;
#endif
}
POA_FN void team_publish(const TeamCtx c, int32_t stripe, int32_t cols_done) { /* ONE lane, after its row stores */
#if POA_DEVICE
    __threadfence_block();
    const unsigned long long v = ((unsigned long long)(uint32_t)stripe << 32) | (uint32_t)cols_done;
    asm volatile("st.volatile.shared.u64 [%0], %1;" ::"r"(c.prog_sa + 8u * (uint32_t)c.w), "l"(v) : "memory");
#elif ALN_EMU_TEAMS
    if (c.emu) aln_emu_publish(c.emu, c.w, stripe, cols_done);
#else
    (void)c; (void)stripe; (void)cols_done;
#endif
}
POA_FN void team_wait(const TeamCtx c, int32_t stripe, int32_t cols_needed) { /* whole warp: until `stripe` got that far */
#if POA_DEVICE
    const unsigned long long target = ((unsigned long long)(uint32_t)stripe << 32) | (uint32_t)cols_needed;
    const uint32_t sa = c.prog_sa + 8u * (uint32_t)(stripe % c.n);
    unsigned long long v;
#if ALN_SPLIT_DIGEST
    uint32_t polls = 0;
#endif
    do {
        asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(v) : "r"(sa) : "memory");
#if ALN_SPLIT_DIGEST
        if (++polls >= ALN_WAIT_POLLS) {
            *c.timed_out = 1;
            break;
        }
#endif
    } while (v < target);
    __threadfence_block();
#elif ALN_EMU_TEAMS
    if (c.emu) aln_emu_wait(c.emu, c.w, stripe, cols_needed);
#else
    (void)c; (void)stripe; (void)cols_needed;
#endif
}
/* A word of a hand-over row: written by another warp of the block moments ago, so not through a stale L1 line.
 * `stripe`: the stripe that must have written it in this pass; `cols_needed`: the columns the consumer's last team_wait
 * must cover for the word to be complete (emulated teams check both). */
POA_FN uint32_t hrow_load(const uint32_t* p, const TeamCtx c, int32_t stripe, int32_t cols_needed) {
#if POA_DEVICE
    (void)c; (void)stripe; (void)cols_needed;
    uint32_t v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
#else
#if ALN_EMU_TEAMS
    if (c.emu) aln_emu_hrow_load(c.emu, c.w, p, stripe, cols_needed);
#else
    (void)c; (void)stripe; (void)cols_needed;
#endif
    return *p;
#endif
}
/* the columns the stripe above must have run for word k of its hand-over row to be complete: 16 k .. 16 k + 15, or up
 * to its last column p_hi */
POA_FN int32_t hrow_word_cols(int32_t k, int32_t p_hi) { return 16 * k + 16 < p_hi + 1 ? 16 * k + 16 : p_hi + 1; }
/* a word of a hand-over row (or its anchor) written by `stripe`; ONE lane */
POA_FN void hrow_store(uint32_t* p, uint32_t v, const TeamCtx c, int32_t stripe) {
#if ALN_EMU_TEAMS
    if (c.emu) aln_emu_hrow_store(c.emu, c.w, p, stripe);
#else
    (void)c; (void)stripe;
#endif
    *p = v;
}

/* The step's shifts on the FMA pipe.  LOP3 / IADD3 / SHF all issue on the ALU pipe (one warp instruction per two cycles
 * per scheduler) and the step is bound by it; integer multiply-add issues on the other pipe.  (x << 1) | bit is
 * x * 2 + bit (bit 0 of x * 2 is clear), x >> 31 is the high word of x * 2: written as mad / mul.hi in PTX so that the
 * compiler cannot strength-reduce them back into shifts and adds. */
POA_FN uint64_t shl1_or_bit(uint64_t x, uint32_t bit) {
#if POA_DEVICE
    const uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    uint32_t nlo, carry, nhi; /* three multiply-adds; a wide one is turned back into LEA + LEA.HI.X (ALU pipe) */
    asm("mad.lo.u32 %0, %1, 2, %2;" : "=r"(nlo) : "r"(lo), "r"(bit));
    asm("mul.hi.u32 %0, %1, 2;" : "=r"(carry) : "r"(lo));
    asm("mad.lo.u32 %0, %1, 2, %2;" : "=r"(nhi) : "r"(hi), "r"(carry));
    return ((uint64_t)nhi << 32) | nlo;
#else
    return (x << 1) | bit;
#endif
}
POA_FN int top_bit(uint64_t x) { /* bit 63 */
#if POA_DEVICE
    uint32_t r;
    asm("mul.hi.u32 %0, %1, 2;" : "=r"(r) : "r"((uint32_t)(x >> 32)));
    return (int)r;
#else
    return (int)(x >> 63);
#endif
}
POA_FN int twice_plus(int a, int b) { /* 2 a + b */
#if POA_DEVICE
    int r;
    asm("mad.lo.s32 %0, %1, 2, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
#else
    return 2 * a + b;
#endif
}

/* a character that is none of ACGT equals only itself (edlib's alphabet is the set of bytes seen): rare */
POA_FN uint64_t eq_other(const SeqView q, int32_t row0, int32_t cnt, int tc) {
    uint64_t Eq = 0;
    for (int32_t k = 0; k < cnt; ++k)
        if ((int)seq_at(q, row0 + k) == tc) Eq |= (uint64_t)1 << k;
    return Eq;
}

/*
 * One bit-vector pass: the distance matrix of q[0..n) against t[0..cols), boundary D[i][0] = i, D[0][j] = j.
 *   out_col (nullable): receives the last column, out_col[i] = D[i][cols], i = 0..n
 *   PM / S  (nullable): receive the record of every (block, column), leaf_entry() order
 * Returns the number of matrix cells this warp computed (its stripes' rows x the columns they ran).
 * Myers' block recurrence in Hyyro's formulation (64 rows per word): with Pv/Mv the +1/-1 vertical deltas of the previous
 * column, Eq the rows whose character equals the column's and hin the horizontal delta entering from above,
 *   Xv = Eq | Mv;  Eq |= (hin < 0);  Xh = (((Eq & Pv) + Pv) ^ Pv) | Eq;  Ph = Mv | ~(Xh | Pv);  Mh = Pv & Xh;
 *   hout = bit63(Ph) - bit63(Mh);  Ph = Ph << 1 | (hin > 0);  Mh = Mh << 1 | (hin < 0);
 *   Pv' = Mh | ~(Xv | Ph);  Mv' = Ph & Xv.
 * Wavefront: lane l owns block s0 + l and works on column (step - l); what crosses lanes is the 2-bit delta code
 * (1 = +1, 2 = -1) of the block's last row, one shuffle per step -- the only thing on the step's dependency chain.
 * The column's character code comes straight from the slot's code row (loaded one step ahead), its match mask from the
 * lane's shared-memory table.
 * Band (band >= 0: the caller only needs values <= band - 2 to be exact, and anything larger to stay larger): a cell
 * (i, j) with D <= band has |i - j| <= band, so the stripe of rows (R0, R1] only runs the columns R0 - band .. R1 + band - 1
 * -- for a Hirschberg half that is a diagonal strip instead of the whole rectangle.  What it does not compute it
 * OVERESTIMATES: it starts at its first column with all vertical deltas + 1 under the value the stripe above had there
 * (the "anchor", handed over with the deltas), takes + 1 for every entering delta beyond the stripe above's last column,
 * and reports ALN_INF for rows whose strip ends before the last column.  Overestimates never win a minimum against the
 * exact values of the cells a path of cost <= band - 2 runs through, all of which are computed (edlib's own band rests on
 * the same argument, edlib.cpp:540-760).
 */
template <bool TEAM>
POA_FN_NOINLINE int64_t myers_pass(const SeqView q, int32_t n, const SeqView t, int32_t cols, int32_t band, const TeamCtx team_in,
                                uint32_t* hbuf, int32_t hrow_words, uint8_t* tcode_base, const EqTab eq_in, int32_t* out_col,
                                RecPM* PM, int32_t* S) {
    n = poa_uniform(n);
    cols = poa_uniform(cols);
    band = poa_uniform(band);
    EqTab eq = eq_in; /* by value: a reference would live in local memory and be re-read every step */
    const TeamCtx team = TEAM ? team_in : TeamCtx{0, 1, 0, 0}; /* TEAM = false: the team code folds away */
    const int32_t B = (n + 63) / 64;
    uint8_t* tcode = tcode_base + 64; /* tcode[-64 .. cols + 63] may be read (by lanes whose column is out of range) */
    if (TEAM && team.n > 1) {
        POA_LANE0 { team_publish(team, 0, 0); } /* progress words of the previous pass are void */
    }
    /* every warp of a team looks at the whole target once (does it hold a character that is none of ACGT?) and writes
     * its share of the code row */
    bool has_other = false;
    for (int32_t base = -64; base < cols + 64; base += 32) {
        PerLane<int> other;
        POA_LANES(l) {
            const int32_t c = base + l;
            const int code = (c >= 0 && c < cols) ? aln_code(seq_at(t, c)) : 0;
            other[l] = code == 4;
            if (((base + 64) >> 5) % team.n == team.w) tcode[c] = (uint8_t)code;
        }
        if (warp_ballot(other)) has_other = true;
    }
    if (out_col && team.w == 0) {
        POA_LANE0 { out_col[0] = cols; }
    }
    POA_SYNC();
    POA_FENCE();
    if (TEAM) team_barrier(team);
    const int32_t n_stripes = (B + 31) / 32;
    int64_t cells_done = 0;
    for (int32_t sidx = team.w; sidx < n_stripes; sidx += team.n) {
        const int32_t s0 = 32 * sidx;
        const int32_t nb = B - s0 < 32 ? B - s0 : 32;
        const bool more = s0 + 32 < B; /* another stripe follows: the last lane's horizontal deltas are kept */
        const bool lower = s0 > 0;     /* lane 0 enters with the deltas the stripe above left behind */
        const bool piped = TEAM && lower && team.n > 1;
        const uint32_t* row_in = hbuf + (int64_t)((sidx + team.n - 1) % team.n) * hrow_words;
        uint32_t* row_out = hbuf + (int64_t)(sidx % team.n) * hrow_words;
        /* the columns this stripe runs, the last one the stripe above ran, the first one the stripe below will run */
        const int32_t R0 = 64 * s0, R1 = 64 * (s0 + nb) < n ? 64 * (s0 + nb) : n;
        const int32_t c_lo = band < 0 || R0 - band < 0 ? 0 : R0 - band;
        const int32_t c_hi = band < 0 || R1 + band - 1 > cols - 1 ? cols - 1 : R1 + band - 1;
        const int32_t p_hi = band < 0 || R0 + band - 1 > cols - 1 ? cols - 1 : R0 + band - 1;
        const int32_t a_col = (band < 0 || R1 - band <= 0) ? -1 : R1 - band - 1; /* the anchor column for the stripe below */
#if ALN_EMU_TEAMS
        if (team.emu) aln_emu_stripe(team.emu, team.w, sidx, c_lo, c_hi, has_other); /* what the emulated pass ran */
#endif
        if (c_lo > c_hi) { /* the strip has left the matrix: no row from here on reaches the last column */
            if (out_col) {
                for (int32_t r = R0 + 1; r <= R1; r += 32) {
                    POA_LANES(l) {
                        if (r + l <= R1) out_col[r + l] = ALN_INF;
                    }
                }
            }
            continue;
        }
        cells_done += (int64_t)(R1 - R0) * (c_hi - c_lo + 1);
        const int32_t step_first = c_lo & ~15;
        const int32_t w_last_in = p_hi >> 4; /* words of the row above this index were never written: every delta + 1 */
        uint32_t hword = 0x55555555u, hword_next = 0x55555555u; /* stripe 0: D[0][j] = j, every delta + 1 */
        int32_t base_top = lower ? R0 : 0; /* D[R0][c_lo]: the left border's R0 when the strip starts at column 0 */
        if (piped) team_wait(team, sidx - 1, step_first + 32 < p_hi + 1 ? step_first + 32 : p_hi + 1);
        if (lower) {
            const int32_t k0 = step_first >> 4;
            if (k0 <= w_last_in) hword = hrow_load(row_in + k0, team, sidx - 1, hrow_word_cols(k0, p_hi));
            if (k0 + 1 <= w_last_in) hword_next = hrow_load(row_in + k0 + 1, team, sidx - 1, hrow_word_cols(k0 + 1, p_hi));
            if (c_lo > 0) base_top = (int32_t)hrow_load(row_in + (hrow_words - 1), team, sidx - 1, c_lo); /* at column c_lo - 1 */
        }
        PerLane<uint64_t> Pv, Mv;
        PerLane<int> bot, link, tc_next, hacc;
        POA_LANES(l) {
            const int32_t b = s0 + l;
            uint64_t e0 = 0, e1 = 0, e2 = 0, e3 = 0;
            if (l < nb) {
                const int32_t row0 = 64 * b;
                const int32_t cnt = n - row0 < 64 ? n - row0 : 64;
                for (int32_t k = 0; k < cnt; ++k) {
                    const int c = aln_code(seq_at(q, row0 + k));
                    const uint64_t bit = (uint64_t)1 << k;
                    if (c == 0) e0 |= bit;
                    else if (c == 1) e1 |= bit;
                    else if (c == 2) e2 |= bit;
                    else if (c == 3) e3 |= bit;
                }
            }
            eq_store(eq, 0, l, e0);
            eq_store(eq, 1, l, e1);
            eq_store(eq, 2, l, e2);
            eq_store(eq, 3, l, e3);
            eq_store(eq, 4, l, 0);
            Pv[l] = ~(uint64_t)0;
            Mv[l] = 0;
            bot[l] = base_top + 64 * (l + 1); /* all vertical deltas + 1 under the stripe's top at its first column */
            link[l] = 0;
            tc_next[l] = glb_u8(tcode + (step_first - l));
            hacc[l] = 0;
        }
        POA_SYNC();
        const int32_t steps = c_hi + nb; /* the last lane's last column is step c_hi + nb - 1 */
        /* One step of the wavefront.  OTHER = 0 leaves out the cold path for characters that are none of ACGT (a pass
         * whose target holds none -- the rule -- runs the unrolled loop below without carrying that code 16 times). */
#define ALN_STEP(OTHER)                                                                                                  \
    {                                                                                                                    \
        const int h0 = (int)((hword >> ((step & 15) * 2)) & 3u);                                                         \
        PerLane<int> in;                                                                                                 \
        warp_shift_up1(link, in); /* in[l] = the delta code lane l - 1 produced in the previous step */                  \
        POA_LANES(l) {                                                                                                   \
            const int32_t c = step - l;                                                                                  \
            const int code = tc_next[l];                                                                                 \
            const int hcode = l == 0 ? h0 : in[l];                                                                       \
            tc_next[l] = glb_u8(tcode + (c + 1)); /* next step's column, a step ahead of its use */                      \
            if (l < nb && (uint32_t)(c - c_lo) <= (uint32_t)(c_hi - c_lo)) { /* lane l works on column c */                 \
                uint64_t Eq;                                                                                             \
                if (!(OTHER) || code < 4) Eq = eq_load(eq, code, l);                                                     \
                else Eq = eq_other(q, 64 * (s0 + l), n - 64 * (s0 + l) < 64 ? n - 64 * (s0 + l) : 64, (int)seq_at(t, c)); \
                const uint64_t pv = Pv[l], mv = Mv[l];                                                                   \
                const uint32_t pos = (uint32_t)(hcode & 1), neg = (uint32_t)(hcode >> 1); /* hcode <= 2 */               \
                const uint64_t Xv = Eq | mv;                                                                             \
                const uint64_t Eh = Eq | (uint64_t)neg;                                                                  \
                const uint64_t Xh = (((Eh & pv) + pv) ^ pv) | Eh;                                                        \
                uint64_t Ph = mv | ~(Xh | pv);                                                                           \
                uint64_t Mh = pv & Xh;                                                                                   \
                const int ph63 = top_bit(Ph), mh63 = top_bit(Mh);                                                        \
                Ph = shl1_or_bit(Ph, pos);                                                                               \
                Mh = shl1_or_bit(Mh, neg);                                                                               \
                const uint64_t npv = Mh | ~(Xv | Ph);                                                                    \
                const uint64_t nmv = Ph & Xv;                                                                            \
                Pv[l] = npv;                                                                                             \
                Mv[l] = nmv;                                                                                             \
                bot[l] = bot[l] + ph63 - mh63;                                                                           \
                const int out = twice_plus(mh63, ph63); /* 1 = +1, 2 = -1 */                                             \
                if (PM) {                                                                                                \
                    const int64_t e = (int64_t)s0 * (cols + 31) + (int64_t)step * nb + l;                                \
                    PM[e] = RecPM{npv, nmv};                                                                             \
                    S[e] = bot[l];                                                                                       \
                }                                                                                                        \
                if (more && l == 31) { /* 16 columns to a word; this row's reader is at least 16 columns behind */       \
                    hacc[l] |= out << ((c & 15) * 2);                                                                    \
                    if (c == a_col) hrow_store(row_out + (hrow_words - 1), (uint32_t)bot[l], team, sidx); /* anchor */   \
                    if ((c & 15) == 15 || c == c_hi) {                                                                   \
                        /* beyond the strip's last column every delta counts + 1 */                                      \
                        if (c == c_hi && (c & 15) != 15) hacc[l] |= (int)(0x55555555u << (((c & 15) + 1) * 2));          \
                        hrow_store(row_out + (c >> 4), (uint32_t)hacc[l], team, sidx);                                   \
                        hacc[l] = 0;                                                                                     \
                        if (TEAM && team.n > 1 && ((c & 31) == 31 || c == c_hi)) team_publish(team, sidx, c + 1);        \
                    }                                                                                                    \
                }                                                                                                        \
                link[l] = out;                                                                                           \
            }                                                                                                            \
        }                                                                                                                \
    }
        /* ALN_STEP_UNROLL steps to a group (a divisor of 16): inside a group the entering delta's bit position and the
         * code row's offsets are immediates and the once-in-16-steps bookkeeping costs nothing; the steps a group runs
         * past `steps` find every lane's column out of range */
        for (int32_t step0 = step_first; step0 < steps; step0 += ALN_STEP_UNROLL) {
            if ((step0 & 15) == 0 && step0 > step_first) { /* the next 16 entering deltas; their successor word a word ahead */
                hword = hword_next;
                hword_next = 0x55555555u;
                if (lower && (step0 >> 4) + 1 <= w_last_in) {
                    if (piped) team_wait(team, sidx - 1, p_hi + 1 < step0 + 32 ? p_hi + 1 : step0 + 32);
                    hword_next = hrow_load(row_in + (step0 >> 4) + 1, team, sidx - 1, hrow_word_cols((step0 >> 4) + 1, p_hi));
                }
            }
            if (!has_other) {
#pragma unroll
                for (int32_t u = 0; u < ALN_STEP_UNROLL; ++u) {
                    const int32_t step = step0 + u;
                    ALN_STEP(0)
                }
            } else {
                for (int32_t u = 0; u < ALN_STEP_UNROLL; ++u) {
                    const int32_t step = step0 + u;
                    ALN_STEP(1)
                }
            }
        }
#undef ALN_STEP
        if (out_col && c_hi < cols - 1) { /* the strip ends before the last column: nothing cheap enough ends in these rows */
            for (int32_t r = R0 + 1; r <= R1; r += 32) {
                POA_LANES(l) {
                    if (r + l <= R1) out_col[r + l] = ALN_INF;
                }
            }
        } else if (out_col) { /* the last column, row by row: D = (score above the block) + running sum of the vertical deltas */
            POA_LANES(l) {
                if (l < nb) {
                    const int32_t row0 = 64 * (s0 + l);
                    const int32_t cnt = n - row0 < 64 ? n - row0 : 64;
                    const uint64_t pv = Pv[l], mv = Mv[l];
                    int run = bot[l] - aln_popc64(pv) + aln_popc64(mv);
                    for (int32_t k = 0; k < cnt; ++k) {
                        run += (int)((pv >> k) & 1u) - (int)((mv >> k) & 1u);
                        out_col[row0 + k + 1] = run;
                    }
                }
            }
        }
        POA_SYNC();
        POA_FENCE(); /* hbuf / out_col written by one lane are read by others next; the Eq table is rebuilt */
    }
    return cells_done;
}

/* ------------------------------------------------------------------------------------------
 * One Hirschberg step (edlib.cpp:1198-1344)
 * ---------------------------------------------------------------------------------------- */
/* the split rule on the two middle columns: Lc[i] = D(q[0..i), left half), Rr[i] = D(q[n-i..n), right half) */
POA_FN_NOINLINE void aln_split_rule(const int32_t* Lc, const int32_t* Rr, int32_t n, int32_t m, AlnSplit* out) {
    n = poa_uniform(n);
    m = poa_uniform(m);
    const int32_t lh = m / 2, rh = m - lh; /* edlib.cpp:1216-1217 */
    /* the optimum of the sub-problem is the smallest left + right sum over all crossing points of the middle */
    PerLane<int> acc;
    POA_LANES(l) { acc[l] = 0x7FFFFFFF; }
    for (int32_t base = 0; base <= n - 2; base += 32) {
        POA_LANES(l) {
            const int32_t idx = base + l;
            if (idx <= n - 2) {
                const int v = Lc[idx + 1] + Rr[n - idx - 1];
                if (v < acc[l]) acc[l] = v;
            }
        }
    }
    int32_t best = warp_min(acc);
    const int32_t top_sum = poa_uniform(lh + Rr[n]);    /* r = -1: the left half is all deletions  (:1292-1299) */
    const int32_t bot_sum = poa_uniform(Lc[n] + rh);    /* r = n-1: the right half is all deletions (:1300-1308) */
    if (top_sum < best) best = top_sum;
    if (bot_sum < best) best = bot_sum;
    int32_t r = -2;
    for (int32_t base = 0; base <= n - 2 && r == -2; base += 32) { /* first index wins (:1282-1290) */
        PerLane<int> hit;
        POA_LANES(l) {
            const int32_t idx = base + l;
            hit[l] = (idx <= n - 2 && Lc[idx + 1] + Rr[n - idx - 1] == best) ? 1 : 0;
        }
        const unsigned mask = warp_ballot(hit);
        if (mask) r = base + poa_ffs(mask);
    }
    int32_t ls = 0, rs = 0;
    if (r >= 0) {
        ls = poa_uniform(Lc[r + 1]);
        rs = poa_uniform(Rr[n - r - 1]);
    } else if (top_sum == best) {
        r = -1;
        ls = lh;
        rs = best - lh;
    } else if (bot_sum == best) {
        r = n - 1;
        rs = rh;
        ls = best - rh;
    }
    POA_LANE0 {
        out->r = r;
        out->ls = ls;
        out->rs = rs;
        out->best = best;
    }
    POA_SYNC();
}

POA_FN_NOINLINE int64_t aln_split(const AlnSlot& s_ref, EqTab& eq, const uint8_t* q, const uint8_t* t, int32_t n, int32_t m,
                                  int32_t band, AlnSplit* out) {
    const AlnSlot s = s_ref;
    n = poa_uniform(n);
    m = poa_uniform(m);
    const int32_t lh = m / 2, rh = m - lh;
    int64_t cells = myers_pass<false>(SeqView{q, 1}, n, SeqView{t, 1}, lh, band, TeamCtx{0, 1, 0, 0}, s.hbuf, s.hrow_words, s.tcode, eq,
                                      s.Lc, nullptr, nullptr);
    cells += myers_pass<false>(SeqView{q + (n - 1), -1}, n, SeqView{t + (m - 1), -1}, rh, band, TeamCtx{0, 1, 0, 0}, s.hbuf,
                               s.hrow_words, s.tcode, eq, s.Rr, nullptr, nullptr);
    aln_split_rule(s.Lc, s.Rr, n, m, out);
    return cells;
}

#if ALN_SPLIT_DIGEST || ALN_LEAF_DIGEST || !POA_DEVICE
/* Test builds: one record per split attempt (b200aln_debug_split_log on the device, the batch emulation in tests/emu),
 * so that every Hirschberg step -- both middle columns, the split -- can be compared between the two. */
enum { ALN_PATH_WARP = 0, ALN_PATH_TEAM = 1, ALN_PATH_SIDE = 2 }; /* one warp; a team in a thin level; a team on the side stream */
enum { ALN_REC_TIMEOUT = 1 };                                      /* flags: a team_wait gave up */
struct AlnSplitRec {
    int32_t aln, r0, c0, n, m;
    int32_t band;    /* what myers_pass got: -1 none */
    int32_t attempt; /* 0, or 1: redone without a band after a guess that proved too small */
    int32_t level, path, flags;
    int32_t r, ls, rs, best;
    int32_t pad[2];
    unsigned long long lc_hash, rr_hash; /* aln_col_digest of Lc[0..n] and Rr[0..n] */
};
POA_FN unsigned long long aln_mix64(unsigned long long x) { /* splitmix64's finaliser */
    x ^= x >> 30;
    x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27;
    x *= 0x94d049bb133111ebull;
    x ^= x >> 31;
    return x;
}
POA_FN unsigned long long aln_warp_sum64(const PerLane<unsigned long long>& acc) { /* wrapping; every lane gets it */
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
/* Hash of a middle column: the wrapping sum over rows i = 0..n of mix64(i, col[i]), independent of the order lanes visit
 * the rows in.  Whole warp. */
POA_FN_NOINLINE unsigned long long aln_col_digest(const int32_t* col, int32_t n) {
    n = poa_uniform(n);
    PerLane<unsigned long long> acc;
    POA_LANES(l) { acc[l] = 0; }
    for (int32_t base = 0; base <= n; base += 32) {
        POA_LANES(l) {
            const int32_t i = base + l;
            if (i <= n) acc[l] += aln_mix64((((unsigned long long)(uint32_t)i << 32) | (uint32_t)col[i]) + 0x9e3779b97f4a7c15ull);
        }
    }
    return aln_warp_sum64(acc);
}
#endif

#if ALN_LEAF_DIGEST || !POA_DEVICE
/* Test builds: one record per leaf (b200aln_debug_leaf_log on the device, the batch emulation and emu_leaf in tests/emu),
 * so that every walk -- its operations, its end score and the paths it took -- can be compared between the two and held
 * against the plain matrix.  aln_leaf fills it through an optional pointer; the counters exist only in these builds. */
#define ALN_LEAF_REC 1
struct AlnLeafRec {
    int32_t aln, r0, c0, n, m;
    int32_t band;  /* what myers_pass got: -1 none */
    int32_t top;   /* the rect's flags (ALN_TOP, ALN_GUESS) */
    int32_t score; /* D at the leaf's last cell as the walk reads it from the records; n + m when n or m is 0 */
    int32_t diag_rounds, diag_ops, matches; /* rounds that moved diagonally, their moves, the matches among them */
    int32_t up_rounds, left_rounds;
    int32_t full_runs;                      /* rounds whose whole diagonal of 32 cells moved diagonally (~dm == 0) */
    int32_t reload_block, reload_col;       /* window reloads: the walk entered the block above / moved > 24 columns */
    int32_t border_lanes;                   /* cells rated on the left border (jw - l == 0) */
    int32_t tail, tail_kind;                /* moves along a border after the walk: 1 insertions, 2 deletions, 0 none */
    int32_t pad;
    long long cells;                        /* what myers_pass returned */
    unsigned long long ops_hash;            /* aln_ops_digest of the leaf's (n + m)-byte region, holes included */
};
/* Hash of an operations region: the wrapping sum over positions p of mix64(p << 8 | op), holes (OP_NONE) included,
 * independent of the order lanes visit the positions in.  Whole warp. */
POA_FN_NOINLINE unsigned long long aln_ops_digest(const uint8_t* ops, int32_t len) {
    len = poa_uniform(len);
    PerLane<unsigned long long> acc;
    POA_LANES(l) { acc[l] = 0; }
    for (int32_t base = 0; base < len; base += 32) {
        POA_LANES(l) {
            const int32_t p = base + l;
            if (p < len) acc[l] += aln_mix64((((unsigned long long)(uint32_t)p << 8) | (uint32_t)glb_u8(ops + p)) + 0x9e3779b97f4a7c15ull);
        }
    }
    return aln_warp_sum64(acc);
}
/* the walk's record is complete: hash its region, hand it over; whole warp */
POA_FN void aln_leaf_finish(AlnLeafRec* rec, AlnLeafRec& lr, const uint8_t* ops, int32_t len) {
    POA_FENCE(); /* the region was written by every lane */
    lr.ops_hash = aln_ops_digest(ops, len);
    POA_LANE0 { *rec = lr; }
    POA_SYNC();
}
#define ALN_LEAF_COUNT(stmt) stmt
#else
#define ALN_LEAF_REC 0
#define ALN_LEAF_COUNT(stmt)
#endif

/* ------------------------------------------------------------------------------------------
 * A leaf: store the whole matrix as block records, walk back from the last cell (edlib.cpp:909-1126)
 * ---------------------------------------------------------------------------------------- */
POA_FN uint64_t warp_get64(const PerLane<uint64_t>& x, int src) {
#if POA_DEVICE
    return __shfl_sync(0xffffffffu, x.v, src);
#else
    return x.v[src];
#endif
}
POA_FN uint64_t aln_below(int32_t k) { return k == 63 ? (uint64_t)0 : (~(uint64_t)0 << (k + 1)); } /* rows under row k */
POA_FN int aln_bit(uint64_t x, int32_t k) { return (int)((x >> k) & 1u); }

/* The records of block b for the 32 columns jw, jw-1, .. jw-31 (lane l holds column c = jw - l AND its left neighbour
 * c - 1): one round of strided loads instead of a dependent round trip per traceback step */
struct LeafWindow {
    PerLane<uint64_t> P, M, Pn, Mn; /* column c, column c - 1 */
    PerLane<int> S, Sn;
};
POA_FN void leaf_window_load(const AlnSlot& s, LeafWindow& w, int32_t b, int32_t jw, int32_t B, int32_t cols) {
    POA_LANES(l) {
        const int32_t c = jw - l;
        uint64_t p = 0, m = 0, pn = 0, mn = 0;
        int sc = 0, scn = 0;
        if (c >= 0) {
            const int64_t e = leaf_entry(b, c, B, cols);
            const RecPM r = s.PM[e];
            p = r.p;
            m = r.m;
            sc = s.S[e];
        }
        if (c >= 1) {
            const int64_t e = leaf_entry(b, c - 1, B, cols);
            const RecPM r = s.PM[e];
            pn = r.p;
            mn = r.m;
            scn = s.S[e];
        }
        w.P[l] = p;
        w.M[l] = m;
        w.S[l] = sc;
        w.Pn[l] = pn;
        w.Mn[l] = mn;
        w.Sn[l] = scn;
    }
}

/*
 * ops: the (n + m)-byte region of this sub-problem, filled from its END backwards (holes stay OP_NONE in front).
 * Cell (i, j) stands for D[i + 1][j + 1].  Any cell's value follows from its block's record alone -- bottom score minus the
 * +1 deltas under the row plus the -1 deltas under it -- so the move edlib takes AT a cell (first possible of up, left,
 * diagonal; edlib.cpp:983-1093) does not depend on how the walk got there.  The warp therefore looks at the 32 cells of
 * the DIAGONAL through the current one at once: lane d rates cell (i - d, j - d) from the records of its column and the
 * column to the left (with k = row mod 64:  cell = S - popc(P & below k) + popc(M & below k);  up = cell - bit_k(P) +
 * bit_k(M);  left and diagonal the same from the neighbour column), one ballot gives the length of the run of diagonal
 * moves in front of the walk, and the whole run -- matches and mismatches -- is written in one coalesced store.  Up and
 * left moves take a round each.  A new window of records is loaded every 25 columns or when the walk enters the block
 * above.
 * Test builds (ALN_LEAF_REC): rec (nullable) receives the leaf's AlnLeafRec -- every field but aln, r0, c0 and top.
 */
POA_FN_NOINLINE int64_t aln_leaf(const AlnSlot& s_ref, EqTab& eq, const uint8_t* q, const uint8_t* t, int32_t n, int32_t m,
                                 int32_t band, uint8_t* ops, int32_t* score_out
#if ALN_LEAF_REC
                                 , AlnLeafRec* rec = nullptr
#endif
) {
    const AlnSlot s = s_ref;
    n = poa_uniform(n);
    m = poa_uniform(m);
#if ALN_LEAF_REC
    AlnLeafRec lr{};
    lr.n = n;
    lr.m = m;
    lr.band = band;
#endif
    if (n == 0 || m == 0) { /* edlib.cpp:1135-1142 */
        const int32_t len = n + m;
        const uint8_t op = n == 0 ? OP_DELETE : OP_INSERT;
        for (int32_t base = 0; base < len; base += 32) {
            POA_LANES(l) {
                if (base + l < len) ops[base + l] = op;
            }
        }
        if (score_out) {
            POA_LANE0 { *score_out = len; }
        }
        POA_SYNC();
#if ALN_LEAF_REC
        if (rec) {
            lr.score = len;
            lr.tail = len;
            lr.tail_kind = len == 0 ? 0 : n == 0 ? 2 : 1;
            aln_leaf_finish(rec, lr, ops, len);
        }
#endif
        return 0;
    }
    const int64_t cells = myers_pass<false>(SeqView{q, 1}, n, SeqView{t, 1}, m, band, TeamCtx{0, 1, 0, 0}, s.hbuf, s.hrow_words, s.tcode,
                                            eq, nullptr, s.PM, s.S);
    const int32_t B = (n + 63) / 64;
    LeafWindow win;
    int32_t i = n - 1, j = m - 1;
    int32_t jw = j, wb = i >> 6; /* the window: columns jw .. jw - 31 of block wb */
    leaf_window_load(s, win, wb, jw, B, m);
    if (score_out) {
        POA_LANE0 {
            const int32_t k = i & 63;
            *score_out = win.S[0] - aln_popc64(win.P[0] & aln_below(k)) + aln_popc64(win.M[0] & aln_below(k));
        }
    }
#if ALN_LEAF_REC
    POA_LANE0 { lr.score = win.S[0] - aln_popc64(win.P[0] & aln_below(i & 63)) + aln_popc64(win.M[0] & aln_below(i & 63)); }
#endif
    int32_t w = n + m; /* next write position + 1 */
    while (i >= 0 && j >= 0) {
        if ((i >> 6) != wb || jw - j > 24) { /* the walk left the window, or fewer than 7 cells of its diagonal are in it */
            ALN_LEAF_COUNT(if ((i >> 6) != wb) ++lr.reload_block; else ++lr.reload_col;)
            wb = i >> 6;
            jw = j;
            leaf_window_load(s, win, wb, jw, B, m);
        }
        const int32_t off = jw - j, k = i & 63;
        PerLane<int> is_diag, is_up, is_match;
#if ALN_LEAF_REC
        PerLane<int> on_border;
#endif
        POA_LANES(l) {
            const int32_t d = l - off, kk = k - d; /* lane l rates cell (i - d, j - d): row kk of the block, column jw - l */
            int diag = 0, up = 0, match = 0;
            ALN_LEAF_COUNT(on_border[l] = 0;)
            if (d >= 0 && kk >= 0 && jw - l >= 0) {
                const uint64_t under = aln_below(kk);
                const int32_t cell = win.S[l] - aln_popc64(win.P[l] & under) + aln_popc64(win.M[l] & under);
                const int32_t u = cell - aln_bit(win.P[l], kk) + aln_bit(win.M[l], kk);
                int32_t lf, ul;
                if (jw - l > 0) {
                    lf = win.Sn[l] - aln_popc64(win.Pn[l] & under) + aln_popc64(win.Mn[l] & under);
                    ul = lf - aln_bit(win.Pn[l], kk) + aln_bit(win.Mn[l], kk);
                } else { /* the left border: D[r + 1][0] = r + 1 */
                    lf = (i - d) + 1;
                    ul = i - d;
                    ALN_LEAF_COUNT(on_border[l] = 1;)
                }
                if (u + 1 == cell) up = 1;                 /* up: the query character stands alone (edlib.cpp:983-1013) */
                else if (lf + 1 != cell) diag = 1;          /* not left (:1015-1044) either: diagonal (:1046-1093)        */
                match = ul == cell;
            }
            is_diag[l] = diag;
            is_up[l] = up;
            is_match[l] = match;
        }
        const unsigned dm = warp_ballot(is_diag) >> off; /* bit d: the cell d steps down the diagonal moves diagonally */
        const int32_t run = ~dm == 0u ? 32 : poa_ffs(~dm);
        ALN_LEAF_COUNT(lr.border_lanes += b200poa::poa_popc(warp_ballot(on_border));)
        if (run > 0) {
            POA_LANES(l) {
                const int32_t d = l - off;
                if (d >= 0 && d < run) ops[w - 1 - d] = is_match[l] ? OP_MATCH : OP_MISMATCH;
            }
#if ALN_LEAF_REC
            ++lr.diag_rounds;
            lr.diag_ops += run;
            lr.full_runs += run == 32 ? 1 : 0;
            lr.matches += b200poa::poa_popc((warp_ballot(is_match) >> off) & (run == 32 ? ~0u : (1u << run) - 1u));
#endif
            w -= run;
            i -= run;
            j -= run;
        } else {
            const bool up = ((warp_ballot(is_up) >> off) & 1u) != 0u;
            --w;
            POA_LANE0 { ops[w] = up ? OP_INSERT : OP_DELETE; }
            ALN_LEAF_COUNT(if (up) ++lr.up_rounds; else ++lr.left_rounds;)
            if (up) --i;
            else --j;
        }
    }
    /* along the left border (insertions) or the top border (deletions) */
    const int32_t rest = (i >= 0 ? i : j) + 1;
    const uint8_t rop = i >= 0 ? OP_INSERT : OP_DELETE;
    for (int32_t base = 0; base < rest; base += 32) {
        POA_LANES(l) {
            if (base + l < rest) ops[w - rest + base + l] = rop;
        }
    }
    POA_SYNC();
#if ALN_LEAF_REC
    if (rec) {
        lr.tail = rest;
        lr.tail_kind = rest == 0 ? 0 : i >= 0 ? 1 : 2;
        lr.cells = cells;
        aln_leaf_finish(rec, lr, ops, n + m);
    }
#endif
    return cells;
}

/* ------------------------------------------------------------------------------------------
 * Operations -> runs (what a CIGAR is made of).  ops: an alignment's (n + m)-byte region with holes; a run start is a
 * position whose operation differs from the previous (non-hole) one.  Writes start_index << 2 | op for every run start
 * to runs[] (nullable: count only) and returns the number of runs; *n_ops = operations in total (the end of the last
 * run).  The host takes differences (Alignment::convert_to_cigar merges match / mismatch runs into 'M' like
 * edlibAlignmentToCigar(EDLIB_CIGAR_STANDARD), edlib.cpp:1482-1520).
 * ---------------------------------------------------------------------------------------- */
POA_FN int aln_fls(unsigned x) { /* index of the highest set bit, x != 0 */
#if POA_DEVICE
    return 31 - __clz((int)x);
#else
    return 31 - __builtin_clz(x);
#endif
}
POA_FN_NOINLINE int32_t aln_runs(const uint8_t* ops, int32_t len, uint32_t* runs, int32_t& n_ops_out) {
    len = poa_uniform(len);
    int32_t n_runs = 0, n_valid = 0, carry = 4; /* carry: the last operation seen, 4 = none yet */
    for (int32_t base = 0; base < len; base += 32) {
        PerLane<int> cls, b0, b1, ok;
        POA_LANES(l) {
            const int32_t idx = base + l;
            const int op = idx < len ? (int)ops[idx] : (int)OP_NONE;
            cls[l] = op;
            ok[l] = op != (int)OP_NONE;
            b0[l] = ok[l] && (op & 1);
            b1[l] = ok[l] && (op & 2);
        }
        const unsigned valid = warp_ballot(ok), m0 = warp_ballot(b0), m1 = warp_ballot(b1);
        if (valid == 0) continue;
        PerLane<int> start;
        POA_LANES(l) {
            const unsigned under = valid & ((1u << l) - 1u);
            int prev = carry;
            if (under) {
                const int p = aln_fls(under);
                prev = (int)((m0 >> p) & 1u) | (int)(((m1 >> p) & 1u) << 1);
            }
            start[l] = ok[l] && prev != cls[l];
        }
        const unsigned sm = warp_ballot(start);
        if (runs) {
            POA_LANES(l) {
                if (start[l]) {
                    const unsigned under = (1u << l) - 1u;
                    runs[n_runs + b200poa::poa_popc(sm & under)] =
                        ((uint32_t)(n_valid + b200poa::poa_popc(valid & under)) << 2) | (uint32_t)cls[l];
                }
            }
        }
        n_runs += b200poa::poa_popc(sm);
        n_valid += b200poa::poa_popc(valid);
        const int p = aln_fls(valid);
        carry = (int)((m0 >> p) & 1u) | (int)(((m1 >> p) & 1u) << 1);
    }
    n_ops_out = n_valid;
    POA_SYNC();
    POA_FENCE(); /* the run starts are read by other lanes next (aln_cigar_text) */
    return n_runs;
}

/* ------------------------------------------------------------------------------------------
 * Run starts -> CIGAR text, on the device: edlibAlignmentToCigar(EDLIB_CIGAR_STANDARD) (edlib.cpp:1482-1520) spells
 * match and mismatch 'M', a query character alone 'I', a target character alone 'D', each maximal run as <length><letter>.
 * Returns the number of bytes (no terminator); out nullable (count only).  32 run starts per round: a start whose
 * letter differs from its predecessor's closes the run opened before it; lengths come from the neighbouring start.
 * ---------------------------------------------------------------------------------------- */
POA_FN void warp_gather(const PerLane<int>& x, const PerLane<int>& src, PerLane<int>& out) {
#if POA_DEVICE
    out.v = __shfl_sync(0xffffffffu, x.v, src.v);
#else
    for (int l = 0; l < 32; ++l) out.v[l] = x.v[src.v[l]];
#endif
}
POA_FN int aln_ndigits(int32_t v) {
    int d = 1;
    for (int32_t p = 10; d < 10 && v >= p; p *= 10) ++d;
    return d;
}
POA_FN void aln_write_run(uint8_t* out, int32_t len, int nd, int cls) {
    for (int k = nd - 1; k >= 0; --k) {
        out[k] = (uint8_t)('0' + len % 10);
        len /= 10;
    }
    out[nd] = cls == 1 ? (uint8_t)'I' : cls == 2 ? (uint8_t)'D' : (uint8_t)'M';
}
POA_FN_NOINLINE int32_t aln_cigar_text(const uint32_t* runs, int32_t n_runs, int32_t n_ops, uint8_t* out) {
    n_runs = poa_uniform(n_runs);
    n_ops = poa_uniform(n_ops);
    int32_t bytes = 0, open_start = 0, open_cls = -1; /* the letter run that is open: where it starts, its class */
    for (int32_t base = 0; base < n_runs; base += 32) {
        PerLane<int> st, cl, prevc, flag, src, pst, pcl, nb;
        POA_LANES(l) {
            const int32_t k = base + l;
            const uint32_t r = k < n_runs ? runs[k] : 0u;
            const int c = (int)(r & 3u);
            st[l] = (int)(r >> 2);
            cl[l] = k < n_runs ? (c == 1 ? 1 : c == 2 ? 2 : 0) : 3;
        }
        warp_shift_up1(cl, prevc);
        POA_LANES(l) { flag[l] = cl[l] != 3 && cl[l] != (l == 0 ? open_cls : prevc[l]); }
        const unsigned mask = warp_ballot(flag);
        if (mask == 0) continue;
        POA_LANES(l) {
            const unsigned under = mask & ((1u << l) - 1u);
            src[l] = under ? aln_fls(under) : l;
        }
        warp_gather(st, src, pst);
        warp_gather(cl, src, pcl);
        PerLane<int> len, cls;
        POA_LANES(l) {
            const unsigned under = mask & ((1u << l) - 1u);
            const int32_t s0 = under ? pst[l] : open_start;
            cls[l] = under ? pcl[l] : open_cls;
            len[l] = st[l] - s0;
            nb[l] = (flag[l] && cls[l] >= 0) ? aln_ndigits(len[l]) + 1 : 0;
        }
        PerLane<int> off = nb;
        const int32_t total = warp_exscan(off);
        if (out) {
            POA_LANES(l) {
                if (nb[l]) aln_write_run(out + bytes + off[l], len[l], nb[l] - 1, cls[l]);
            }
        }
        bytes += total;
        const int p = aln_fls(mask);
        open_start = warp_get(st, p);
        open_cls = warp_get(cl, p);
    }
    if (open_cls >= 0) {
        const int32_t len = n_ops - open_start;
        const int nd = aln_ndigits(len);
        if (out) {
            POA_LANE0 { aln_write_run(out + bytes, len, nd, open_cls); }
        }
        bytes += nd + 1;
    }
    POA_SYNC();
    return bytes;
}

/* ------------------------------------------------------------------------------------------
 * Run starts -> breaking points (racon::Overlap::find_breaking_points_from_cigar, src/overlap.cpp:226-290): the
 * consumer of the CIGAR, evaluated where the alignment already is.  Windows are the stretches of target coordinates
 * between consecutive multiples of window_length (:229-235); a window that contains at least one match / mismatch
 * column emits its first one as (t, q) and its last one as (t + 1, q + 1) (:248-263).
 * Pass 1 (32 runs a round): target and query characters consumed before every run -> pre[] (two words a run, plus the
 * totals).  Pass 2 (32 windows a round, a lane each): binary search for the runs around the window's two ends, a short
 * walk over the runs that consume no target or are deletions; kept windows are written in order (ballot + prefix).
 * out: (t, q) pairs, capacity 4 words per window; returns the number of pairs.
 * ---------------------------------------------------------------------------------------- */
POA_FN_NOINLINE int32_t aln_breaking_points(const uint32_t* runs, int32_t n_runs, int32_t n_ops, int32_t q_first, int32_t t_begin,
                                            int32_t m, int32_t window_length, int32_t* pre, uint32_t* out) {
    n_runs = poa_uniform(n_runs);
    n_ops = poa_uniform(n_ops);
    /* pass 1: pre[2k] = target characters before run k, pre[2k + 1] = query characters before run k; k = n_runs: totals */
    int32_t t_run = 0, q_run = 0;
    for (int32_t base = 0; base < n_runs; base += 32) {
        PerLane<int> tl, ql;
        POA_LANES(l) {
            const int32_t k = base + l;
            int tlen = 0, qlen = 0;
            if (k < n_runs) {
                const uint32_t r = runs[k];
                const int32_t len = (k + 1 < n_runs ? (int32_t)(runs[k + 1] >> 2) : n_ops) - (int32_t)(r >> 2);
                const int op = (int)(r & 3u);
                tlen = op == OP_INSERT ? 0 : len;
                qlen = op == OP_DELETE ? 0 : len;
            }
            tl[l] = tlen;
            ql[l] = qlen;
        }
        PerLane<int> to = tl, qo = ql;
        const int32_t tsum = warp_exscan(to), qsum = warp_exscan(qo);
        POA_LANES(l) {
            const int32_t k = base + l;
            if (k < n_runs) {
                pre[2 * k] = t_run + to[l];
                pre[2 * k + 1] = q_run + qo[l];
            }
        }
        t_run += tsum;
        q_run += qsum;
    }
    POA_LANE0 {
        pre[2 * n_runs] = t_run;
        pre[2 * n_runs + 1] = q_run;
    }
    POA_SYNC();
    POA_FENCE();
    /* pass 2 */
    const int32_t n_win = aln_window_count(t_begin, m, window_length);
    const int32_t first_mult = (t_begin / window_length + 1) * window_length; /* smallest multiple > t_begin */
    int32_t n_out = 0;
    for (int32_t base = 0; base < n_win; base += 32) {
        PerLane<int> keep, ft, fq, lt, lq;
        POA_LANES(l) {
            const int32_t j = base + l;
            keep[l] = 0;
            ft[l] = fq[l] = lt[l] = lq[l] = 0;
            if (j < n_win) {
                /* the window's target range, relative to the segment: [lo, hi] */
                const int32_t lo = j == 0 ? 0 : first_mult + (j - 1) * window_length - t_begin;
                const int32_t hi = (j == n_win - 1 ? t_begin + m : first_mult + j * window_length) - 1 - t_begin;
                /* first run whose target span ends beyond lo: smallest k with pre[2(k + 1)] > lo */
                int32_t a = 0, b = n_runs;
                while (a < b) {
                    const int32_t mid = (a + b) >> 1;
                    if (pre[2 * (mid + 1)] > lo) b = mid;
                    else a = mid + 1;
                }
                int32_t k = a;
                while (k < n_runs && pre[2 * k] <= hi) { /* forward to the first match / mismatch run inside the window */
                    const int op = (int)(runs[k] & 3u);
                    if (op == OP_MATCH || op == OP_MISMATCH) {
                        const int32_t t = pre[2 * k] > lo ? pre[2 * k] : lo;
                        ft[l] = t_begin + t;
                        fq[l] = q_first + pre[2 * k + 1] + (t - pre[2 * k]);
                        keep[l] = 1;
                        break;
                    }
                    ++k;
                }
                if (keep[l]) {
                    /* last run that starts at or before hi: largest k with pre[2k] <= hi */
                    a = 0;
                    b = n_runs - 1;
                    while (a < b) {
                        const int32_t mid = (a + b + 1) >> 1;
                        if (pre[2 * mid] <= hi) a = mid;
                        else b = mid - 1;
                    }
                    k = a;
                    for (;;) { /* backward to the last match / mismatch run (one exists: the first one at the latest) */
                        const int op = (int)(runs[k] & 3u);
                        if (op == OP_MATCH || op == OP_MISMATCH) {
                            const int32_t last = pre[2 * (k + 1)] - 1 < hi ? pre[2 * (k + 1)] - 1 : hi;
                            lt[l] = t_begin + last + 1;
                            lq[l] = q_first + pre[2 * k + 1] + (last - pre[2 * k]) + 1;
                            break;
                        }
                        --k;
                    }
                }
            }
        }
        const unsigned mask = warp_ballot(keep);
        POA_LANES(l) {
            if (keep[l]) {
                uint32_t* o = out + 4 * (n_out + b200poa::poa_popc(mask & ((1u << l) - 1u)));
                o[0] = (uint32_t)ft[l];
                o[1] = (uint32_t)fq[l];
                o[2] = (uint32_t)lt[l];
                o[3] = (uint32_t)lq[l];
            }
        }
        n_out += b200poa::poa_popc(mask);
    }
    POA_SYNC();
    return 2 * n_out;
}

} // namespace b200aln
