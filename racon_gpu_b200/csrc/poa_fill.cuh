/*
 * poa_fill.cuh -- the DP fill: banded / full Needleman-Wunsch of one read against the DAG, one warp
 * per window, hand-written for sm_90a (H100).
 *
 * Replaces vendor/GenomeWorks/cudapoa/src/cudapoa_nw.cuh:150-473 and cudapoa_nw_banded.cuh:172-482
 * (fill part) with spoa's recurrence (vendor/spoa/src/sisd_alignment_engine.cpp:283-338).
 *
 * Mapping
 *   - a row is processed in chunks of 256 columns: 32 lanes x 8 int16 cells, one 128-bit vector
 *     per lane (the reference uses 4 cells per lane and 64-bit loads, cudapoa_nw.cuh:82-99);
 *   - cells are packed two per 32-bit register and updated with the native packed instructions
 *     VIADDMNMX.S16x2 (__viaddmax_s16x2: max(a+b, c), one issue slot per two cells and
 *     predecessor term) and VIMNMX3.S16x2;
 *   - the matrix is kept in the skewed domain S = H - j*gap, which turns the horizontal dependency
 *     H[i][j-1]+gap into a plain prefix max: 14 packed ops inside the lane + a 5-step warp scan,
 *     instead of the reference's iterate-until-stable loop (cudapoa_nw.cuh:272-317);
 *   - the graph is consumed as two register-resident streams: packed 32-bit row records and the
 *     CSR predecessor list.  Each is fetched 32 entries at a time by one coalesced load (one entry
 *     per lane), double-buffered, and handed out by a shuffle -- the row loop issues no dependent
 *     global load for its own metadata;
 *   - predecessor rows are read from a shared-memory ring holding the last R score rows
 *     (predecessors are almost always within a few ranks, SURVEY.md App. D); an older predecessor
 *     is first copied from global/L2 into a spare shared row.  Every row is also written once to
 *     HBM for the traceback (that write is the algorithmic traffic);
 *   - shared memory is addressed with 32-bit shared-window addresses (ld/st.shared via PTX), which
 *     keeps the per-predecessor address arithmetic to one IMAD;
 *   - the band is snapped to multiples of 8 columns, so a predecessor row with a different band
 *     start is the same 128-bit load at a lane-shifted address; cells outside a band read NEG;
 *   - match/mismatch terms come from a per-read profile in shared memory (one LDS.128 per lane per
 *     row), built once per read for A,C,G,T,N (+ one on-demand slot for any other letter).
 *
 * Must produce exactly the matrix the scalar twin in tests/emu/emu_poa.cpp (ScalarFill) produces.
 */
#pragma once
#include "poa_core.cuh"

namespace b200poa {

#if POA_DEVICE

constexpr int PROF_ROWS = 5; /* A C G T + one on-demand row for any other letter (N, IUPAC, ...) */

__device__ __forceinline__ uint32_t pack2(int lo, int hi) {
    return ((uint32_t)lo & 0xFFFFu) | ((uint32_t)hi << 16);
}
/* shared memory through 32-bit shared-window addresses */
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, uint4 v) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint2 lds64(uint32_t addr) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t prmt_sext(uint32_t a, uint32_t sel) {
    uint32_t d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(0u), "r"(sel));
    return d;
}
__device__ __forceinline__ void sts8(uint32_t addr, int v) {
    asm volatile("st.shared.u8 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void sts16(uint32_t addr, int v) {
    asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

/*
 * Shared memory of one block (one warp), in int16 cells:
 *   [0, 8)                                  eight NEG cells: where out-of-band lanes point their loads
 *   [8, 16)                                 eight zero cells: profile of lanes beyond the band
 *   [16, 16 + PROF_ROWS*prof_stride/2)      profile rows, ONE BYTE per column (s - gap fits int8), widened
 *                                           to int16 pairs with two sign-replicating PRMTs per 4 cells
 *   [.., + ring_rows*ring_stride)           ring of score rows (an older predecessor is staged in the slot the
 *                                           current row will take: that slot holds a row out of reach); every row is
 *                                           RING_PAD_FRONT NEG cells | band cells | RING_PAD_BACK NEG cells
 */
struct FillArgs { /* everything the row loop needs, and nothing else (keeps its register set small) */
    int16_t* S;
    const uint32_t* row_rec;
    const uint32_t* row_pred;  /* rank | band start: only read for predecessors older than the ring */
    const uint32_t* row_pfill; /* the stream the row loop consumes */
    const uint8_t* read;
    uint32_t smem_sa;
    int32_t stride;      /* cells per global score row */
    int32_t prof_stride;
    int32_t ring_stride;
    int32_t ring_mask;
    int32_t N, len, colsP, bw;
    int32_t mg, xg, gap;
};

/* A load that stays where it is written: the row loop prefetches its record stream a block ahead, and the compiler would
 * otherwise sink the load to just before its first use (one register less, one full memory latency more per block). */
__device__ __forceinline__ uint32_t ldg_pinned(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
/* rare (after a row with more than 32 predecessors): restart the predecessor stream at entry `at`.  A call on purpose:
 * as a predicated load inside the re-alignment it shared a scoreboard with the prefetch of the next 32 entries, and the
 * first shuffle of every re-aligned row waited for that prefetch to land. */
__device__ __noinline__ uint2 fill_restart_pred_stream(const uint32_t* row_pfill, int at) {
    const int lane = threadIdx.x & 31;
    return make_uint2(row_pfill[at + lane], row_pfill[at + 32 + lane]);
}

/* rare: predecessor older than the ring -> copy its row from global memory into the spare row */
__device__ __noinline__ void fill_stage_far_row(const int16_t* src, uint32_t far_sa, int bw) {
    const int lane8 = (threadIdx.x & 31) * 8;
    __syncwarp();
#pragma unroll 1
    for (int o = lane8; o < bw; o += CHUNK)
        sts128(far_sa + (uint32_t)o * 2u, *reinterpret_cast<const uint4*>(src + o));
    __syncwarp();
}

__device__ __noinline__ void fill_build_dyn_prof_row(uint32_t row_sa, int c, const uint8_t* read, int len,
                                                     int colsP, int mg, int xg) {
    const int lane = threadIdx.x & 31;
    __syncwarp();
#pragma unroll 1
    for (int col = lane; col < colsP; col += 32) {
        int v = xg;
        if (col >= 1 && col <= len && (int)read[col - 1] == c) v = mg;
        sts8(row_sa + (uint32_t)col, v);
    }
    __syncwarp();
}

/* The row loop.  Deliberately NOT inlined into the window loop: compiled on its own, its loop
 * invariants stay in registers instead of being rematerialised around every use.
 * FULLW = the row is exactly one 256-column chunk with all 32 lanes active (static band 256 on reads
 * longer than the band: the headline configuration) -- no chunk loop, no lane masking, no carry. */
template <bool FULLW>
__device__ __noinline__ int32_t fill_rows(const FillArgs fa) {
    int lane; /* read once through volatile asm so that it is kept, not re-derived from S2R per use */
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));
    const int N = fa.N;
    const int mg = fa.mg, xg = fa.xg;
    const uint32_t NEG2 = pack2(NEG, NEG);
    const uint32_t G2 = pack2(fa.gap, fa.gap);
    const int bw = fa.bw;
    const int nchunks = FULLW ? 1 : (bw + CHUNK - 1) / CHUNK;
    const size_t stride = (size_t)fa.stride;
    int16_t* const S = fa.S;
    const uint32_t* const row_rec = fa.row_rec;
    const uint32_t* const row_pred = fa.row_pred;
    const uint32_t* const row_pfill = fa.row_pfill;
    const uint8_t* const read = fa.read;
    const int ring_mask = fa.ring_mask;
    const int R = ring_mask + 1;
    const int prof_stride = fa.prof_stride;
    const uint32_t neg_sa = fa.smem_sa;
    const uint32_t zero_sa = fa.smem_sa + 16u;
    const uint32_t prof_sa = fa.smem_sa + 32u;
    const uint32_t ring_sa = prof_sa + (((uint32_t)(PROF_ROWS * prof_stride) + 15u) & ~15u); /* profile: 1 byte per column */
    const uint32_t ring_row_bytes = (uint32_t)fa.ring_stride * 2u;
    const int lane8 = lane * 8;
    int dyn_code = -1; /* letter currently held by the on-demand profile row */

    __syncwarp();
    if (lane < 8) sts16(neg_sa + (uint32_t)lane * 2u, NEG);
    else if (lane < 16) sts16(neg_sa + (uint32_t)lane * 2u, 0);
#pragma unroll 1
    for (int col = lane; col < fa.colsP; col += 32) { /* the four fixed profile rows in one pass */
        const int ch = (col >= 1 && col <= fa.len) ? (int)read[col - 1] : -1;
        sts8(prof_sa + (uint32_t)(0 * prof_stride + col), ch == 'A' ? mg : xg);
        sts8(prof_sa + (uint32_t)(1 * prof_stride + col), ch == 'C' ? mg : xg);
        sts8(prof_sa + (uint32_t)(2 * prof_stride + col), ch == 'G' ? mg : xg);
        sts8(prof_sa + (uint32_t)(3 * prof_stride + col), ch == 'T' ? mg : xg);
    }
    /* NEG pads of every ring row (the traceback tile overlays this memory between two fills) */
#pragma unroll 1
    for (int idx = lane; idx < R * (1 + RING_PAD_BACK / 8); idx += 32) {
        const int row = idx / (1 + RING_PAD_BACK / 8), part = idx % (1 + RING_PAD_BACK / 8);
        /* the back pad follows THIS read's band cells (ring rows are sized for the widest band of the batch) */
        const uint32_t cell = part == 0 ? 0u : (uint32_t)(RING_PAD_FRONT + bw + 8 * (part - 1));
        sts128(ring_sa + (uint32_t)row * ring_row_bytes + cell * 2u, make_uint4(NEG2, NEG2, NEG2, NEG2));
    }
    /* row 0: H[0][j] = j*gap  =>  S = 0 (global copy for the traceback, ring slot 0 for the fill) */
#pragma unroll 1
    for (int o = lane8; o < bw; o += CHUNK) {
        *reinterpret_cast<uint4*>(S + o) = make_uint4(0u, 0u, 0u, 0u);
        sts128(ring_sa + (uint32_t)(RING_PAD_FRONT + o) * 2u, make_uint4(0u, 0u, 0u, 0u));
    }
    /* register-resident streams: lane l holds entry (base + l); the next 32 are prefetched.
     * predA always starts at or before the current row's first entry and is re-aligned (two shuffles)
     * whenever a row's entries would run past it, so a row with <= 32 predecessors reads them all
     * from predA with a single shuffle each. */
    uint32_t recA = row_rec[lane];
    int pbase = 0; /* row_pfill index held by lane 0 of predA */
    uint32_t predA = row_pfill[lane];
    uint32_t predB = row_pfill[32 + lane];
    __syncwarp();

    int best = NEG, end_row = 0;
    int po = 0; /* running offset into row_pfill (CSR is contiguous in row order) */
    int16_t* Srow = S; /* global score row of the current graph row */
    /* rows in blocks of 32: the record stream is shifted once per block, not tested once per row */
    int i = 1;
#pragma unroll 1
    for (int blk_end = 31; i <= N; blk_end += 32) {
    const int i_end = blk_end < N ? blk_end : N;
    const uint32_t recN = ldg_pinned(row_rec + blk_end + 1 + lane); /* the next block's records, in flight during this one */
#pragma unroll 1
    for (; i <= i_end; ++i) {
        const uint32_t rec = __shfl_sync(0xffffffffu, recA, i & 31);
        const int np = rec_npred(rec);
        const int bs = rec_bs(rec);
        const int prow = rec_prow(rec);
        if (__any_sync(0xffffffffu, prow == 4)) { /* the vote makes the branch provably warp-uniform, see poa_uniform() */
            const int code = rec_code(rec);
            if (dyn_code != code) {
                fill_build_dyn_prof_row(prof_sa + (uint32_t)(4 * prof_stride), code, read, fa.len, fa.colsP, mg, xg);
                dyn_code = code;
            }
        }
        const uint32_t prof_row_sa = prof_sa + (uint32_t)(prow * prof_stride + bs + lane8);
        Srow += stride;
        const uint32_t ring_row_sa = ring_sa + RING_PAD_FRONT * 2u + (uint32_t)(i & ring_mask) * ring_row_bytes;
        uint32_t carry = NEG2; /* S[i][last column of the previous chunk], both halves */
        int rel = po - pbase;  /* lane of predA holding this row's first entry */
        if (rel + np > 32) {   /* re-align the stream so that predA starts at this row (uniform, ~1 row in 18) */
            if (rel > 32) { /* a row with > 32 entries jumped past predB */
                const uint2 t = fill_restart_pred_stream(row_pfill, po);
                predA = t.x;
                predB = t.y;
            } else {
                const int src = (lane + rel) & 31;
                const uint32_t xa = __shfl_sync(0xffffffffu, predA, src);
                const uint32_t xb = __shfl_sync(0xffffffffu, predB, src);
                predA = (lane + rel < 32) ? xa : xb;
                predB = row_pfill[po + 32 + lane];
            }
            pbase = po;
            rel = 0;
        }

#pragma unroll 1
        for (int k = 0; k < nchunks; ++k) {
            const int o0 = FULLW ? lane8 : k * CHUNK + lane8; /* offset of this lane's cells in the row */
            const bool active = FULLW ? true : (o0 < bw);
            const int c0 = bs + o0;                            /* first column of this lane */
            const uint2 Pb = lds64(active ? prof_row_sa + (uint32_t)(FULLW ? 0 : k * CHUNK) : zero_sa); /* 8 int8 */
            uint4 P; /* widen to 8 int16: byte b -> (b, sign(b)) */
            P.x = prmt_sext(Pb.x, 0x9180u); /* PTX prmt: selector bit 3 replicates the byte's sign */
            P.y = prmt_sext(Pb.x, 0xB3A2u); /* (__byte_perm() only honours 3 selector bits) */
            P.z = prmt_sext(Pb.y, 0x9180u);
            P.w = prmt_sext(Pb.y, 0xB3A2u);
            uint32_t a0 = NEG2, a1 = NEG2, a2 = NEG2, a3 = NEG2;
            /* per-chunk constants of the band tests: an inactive lane can never be "in band" */
            const unsigned lim_v = active ? (unsigned)(bw - 8) : 0u; /* off <= lim_v; inactive lanes have off >= bw > 0 */
            const unsigned lim_l = active ? (unsigned)bw : 0u;       /* off - 1 < lim_l */
            const uint32_t c0_sa = ring_sa + (uint32_t)c0 * 2u;

/* one predecessor term: V = its 8 cells under this lane, leftw = its cell under column c0-1 */
#define POA_FILL_ACCUMULATE()                                                                              \
    do {                                                                                                   \
        const uint4 V = lds128((unsigned)off <= lim_v ? cell_sa : neg_sa);                                 \
        const uint32_t leftw = lds_u16((unsigned)(off - 1) < lim_l ? cell_sa - 2u : neg_sa);               \
        POA_FILL_TERM();                                                                                   \
    } while (0)
#define POA_FILL_TERM()                                                                                    \
    do {                                                                                                   \
        const uint32_t d0 = __byte_perm(leftw, V.x, 0x5410); /* (left cell, first cell): one PRMT */       \
        const uint32_t d1 = __funnelshift_l(V.x, V.y, 16);                                                 \
        const uint32_t d2 = __funnelshift_l(V.y, V.z, 16);                                                 \
        const uint32_t d3 = __funnelshift_l(V.z, V.w, 16);                                                 \
        a0 = __viaddmax_s16x2(d0, P.x, a0);                                                                \
        a1 = __viaddmax_s16x2(d1, P.y, a1);                                                                \
        a2 = __viaddmax_s16x2(d2, P.z, a2);                                                                \
        a3 = __viaddmax_s16x2(d3, P.w, a3);                                                                \
        a0 = __viaddmax_s16x2(V.x, G2, a0);                                                                \
        a1 = __viaddmax_s16x2(V.y, G2, a1);                                                                \
        a2 = __viaddmax_s16x2(V.z, G2, a2);                                                                \
        a3 = __viaddmax_s16x2(V.w, G2, a3);                                                                \
    } while (0)

            if (FULLW && !rec_far(rec) && np <= 32) {
                /* the common row of the banded configuration: every predecessor is in the ring, its band starts
                 * 0..RING_PAD_BACK columns before ours, its stream entry is in predA.  Whatever falls outside the
                 * predecessor's band lands in the row's NEG pads: no tests at all. */
                {   /* every row has at least one predecessor (a node without in-edges has the virtual row 0): the first
                     * one initialises the accumulators */
                    const uint32_t pe = __shfl_sync(0xffffffffu, predA, rel);
                    const uint32_t cell_sa = c0_sa + (uint32_t)((int)pe >> 12);
                    const uint4 V = lds128(cell_sa);
                    const uint32_t leftw = lds_u16(cell_sa - 2u);
                    POA_FILL_TERM();
                }
#pragma unroll 1
                for (int q = 1; q < np; ++q) {
                    const uint32_t pe = __shfl_sync(0xffffffffu, predA, rel + q);
                    const uint32_t cell_sa = c0_sa + (uint32_t)((int)pe >> 12);
                    const uint4 V = lds128(cell_sa);
                    const uint32_t leftw = lds_u16(cell_sa - 2u);
                    POA_FILL_TERM();
                }
            } else if (!rec_far(rec) && np <= 32) {
                /* every predecessor is in the ring and its stream entry is in predA
                 * (out-of-band loads are redirected to the NEG cells: no branches, no predicates) */
#pragma unroll 1
                for (int q = 0; q < np; ++q) {
                    const uint32_t pe = __shfl_sync(0xffffffffu, predA, rel + q);
                    const int off = c0 - (int)((pe & 0xFFEu) << 2); /* offset of column c0 in the predecessor row */
                    const uint32_t cell_sa = c0_sa + (uint32_t)((int)pe >> 12);
                    POA_FILL_ACCUMULATE();
                }
            } else {
#pragma unroll 1
                for (int q = 0; q < np; ++q) {
                    uint32_t pe;
                    if (rel + q < 32) pe = __shfl_sync(0xffffffffu, predA, rel + q);
                    else pe = row_pfill[po + q]; /* in-degree > 32: straight from memory */
                    const int off = c0 - (int)((pe & 0xFFEu) << 2);
                    uint32_t cell_sa = c0_sa + (uint32_t)((int)pe >> 12);
                    if (__any_sync(0xffffffffu, (pe & 1u) != 0)) { /* predecessor older than the ring */
                        const int pr = (int)(row_pred[po + q] & 0xFFFFu);
                        if (FULLW) {
                            /* staged in the ring slot row i itself will take at the end of the row: it holds row i - R,
                             * which no predecessor within the ring's reach can be */
                            fill_stage_far_row(S + (size_t)pr * stride, ring_row_sa, bw);
                            cell_sa = ring_row_sa + (uint32_t)off * 2u;
                        } else {
                            /* several chunks per row: the row's own slot already holds the finished chunks, so the
                             * predecessor's cells come straight from the score matrix (L2/HBM; rare) */
                            const int16_t* src = S + (size_t)pr * stride;
                            uint4 V = make_uint4(NEG2, NEG2, NEG2, NEG2);
                            if ((unsigned)off <= lim_v) V = *reinterpret_cast<const uint4*>(src + off);
                            const uint32_t leftw = (unsigned)(off - 1) < lim_l ? (uint32_t)(uint16_t)src[off - 1] : (uint32_t)(uint16_t)NEG;
                            POA_FILL_TERM();
                            continue;
                        }
                    }
                    POA_FILL_ACCUMULATE();
                }
            }
#undef POA_FILL_ACCUMULATE
#undef POA_FILL_TERM

            /* horizontal: inclusive prefix max over the 8 cells of the lane ... */
            a0 = __vmaxs2(a0, __byte_perm(a0, NEG2, 0x1054));
            a1 = __vmaxs2(a1, __byte_perm(a1, NEG2, 0x1054));
            a2 = __vmaxs2(a2, __byte_perm(a2, NEG2, 0x1054));
            a3 = __vmaxs2(a3, __byte_perm(a3, NEG2, 0x1054));
            a1 = __vmaxs2(a1, __byte_perm(a0, a0, 0x3232));
            a2 = __vmaxs2(a2, __byte_perm(a1, a1, 0x3232));
            a3 = __vmaxs2(a3, __byte_perm(a2, a2, 0x3232));
            /* ... then across lanes (packed, both halves equal) */
            uint32_t tt = __byte_perm(a3, a3, 0x3232);
            if (!FULLW && nchunks > 1) tt = __vmaxs2(tt, lane == 0 ? carry : NEG2);
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) /* lanes below d get their own value back from SHFL.UP: max is a no-op */
                tt = __vmaxs2(tt, __shfl_up_sync(0xffffffffu, tt, d));
            uint32_t excl = __shfl_up_sync(0xffffffffu, tt, 1);
            excl = lane == 0 ? carry : excl;
            a0 = __vimax3_s16x2(a0, excl, NEG2);
            a1 = __vimax3_s16x2(a1, excl, NEG2);
            a2 = __vimax3_s16x2(a2, excl, NEG2);
            a3 = __vimax3_s16x2(a3, excl, NEG2);
            if (!FULLW && nchunks > 1) {
                carry = __shfl_sync(0xffffffffu, tt, 31);
                carry = __vmaxs2(carry, NEG2);
            }

            if (active) {
                const uint4 out = make_uint4(a0, a1, a2, a3);
                __stcs(reinterpret_cast<uint4*>(Srow + o0), out); /* streaming: written once, read once by the traceback; keep L2 for the graph */
                sts128(ring_row_sa + (uint32_t)o0 * 2u, out);
            }

            if (rec_sink(rec)) { /* sink row: candidate end cell at column len */
                const int eo = fa.len - bs - (FULLW ? 0 : k * CHUNK);
                if (eo >= 0 && eo < CHUNK && eo + (FULLW ? 0 : k * CHUNK) < bw) {
                    const int e8 = eo & 7;
                    uint32_t w = (e8 < 2) ? a0 : (e8 < 4) ? a1 : (e8 < 6) ? a2 : a3;
                    int val = (e8 & 1) ? ((int)w >> 16) : (int)(int16_t)(w & 0xFFFFu);
                    val = __shfl_sync(0xffffffffu, val, eo >> 3);
                    if (val > best) {
                        best = val;
                        end_row = i;
                    }
                }
            }
        }
        po += np;
        __syncwarp(); /* row i (ring + global) is visible to every lane before it is read */
    }
    recA = recN;
    }
    return end_row;
}


/* ------------------------------------------------------------------------------------------------
 * Full-band rows (every row starts at column 0): ONE pass per row, whatever the read length.
 * Lane l owns the 8*NV consecutive columns [l*8*NV, (l+1)*8*NV) -- NV 128-bit vectors -- so a row costs one
 * record decode, one profile load, one in-lane scan over 4*NV packed registers and ONE 5-step warp scan,
 * instead of NV (and, for reads just over a multiple of 256 columns, NV+1) complete chunk passes.  The only cell a
 * lane needs from another lane is the one left of its first column (the diagonal operand); inside the lane the
 * diagonal operand of vector v is carried over from the last cell of vector v-1.  Lanes (and vectors) beyond the
 * read compute on stale shared memory and are never stored: a prefix max only flows left to right.
 * All rows have band start 0, so a predecessor is the same lane-private columns of another ring row: no band
 * tests, no lane shifts.  Must produce exactly the matrix ScalarFill (tests/emu/emu_poa.cpp) produces.
 * ---------------------------------------------------------------------------------------------- */
template <int NV>
__device__ __noinline__ int32_t fill_rows_wide(const FillArgs fa) {
    int lane;
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));
    const int N = fa.N;
    const uint32_t NEG2 = pack2(NEG, NEG);
    const uint32_t G2 = pack2(fa.gap, fa.gap);
    const int bw = fa.bw;
    const size_t stride = (size_t)fa.stride;
    int16_t* const S = fa.S;
    const uint32_t* const row_rec = fa.row_rec;
    const uint32_t* const row_pfill = fa.row_pfill;
    const int ring_mask = fa.ring_mask;
    const int R = ring_mask + 1;
    const int prof_stride = fa.prof_stride;
    const uint32_t prof_sa = fa.smem_sa + 32u;
    const uint32_t ring_sa = prof_sa + (((uint32_t)(PROF_ROWS * prof_stride) + 15u) & ~15u);
    const uint32_t ring_row_bytes = (uint32_t)fa.ring_stride * 2u;
    const int col0 = lane * (8 * NV);                   /* first column of this lane */
    const uint32_t c0_sa = ring_sa + (uint32_t)col0 * 2u;
    const int ring_cols = fa.ring_stride - RING_PAD_FRONT; /* cells a ring row can take after its front pad */
    int dyn_code = -1;

    __syncwarp();
    {   /* the four fixed profile rows in one pass; columns beyond the read (up to the lanes' full width) score xg */
        const int pw = prof_stride;
#pragma unroll 1
        for (int col = lane; col < pw; col += 32) {
            const int ch = (col >= 1 && col <= fa.len) ? (int)fa.read[col - 1] : -1;
            sts8(prof_sa + (uint32_t)(0 * prof_stride + col), ch == 'A' ? fa.mg : fa.xg);
            sts8(prof_sa + (uint32_t)(1 * prof_stride + col), ch == 'C' ? fa.mg : fa.xg);
            sts8(prof_sa + (uint32_t)(2 * prof_stride + col), ch == 'G' ? fa.mg : fa.xg);
            sts8(prof_sa + (uint32_t)(3 * prof_stride + col), ch == 'T' ? fa.mg : fa.xg);
        }
    }
    /* NEG front pad of every ring row (the cell left of column 0) */
    if (lane < R) sts128(ring_sa + (uint32_t)lane * ring_row_bytes, make_uint4(NEG2, NEG2, NEG2, NEG2));
    /* row 0: S = 0 */
#pragma unroll
    for (int v = 0; v < NV; ++v) {
        const int c = col0 + 8 * v;
        if (c < bw) *reinterpret_cast<uint4*>(S + c) = make_uint4(0u, 0u, 0u, 0u);
        if (c + 8 <= ring_cols) sts128(c0_sa + RING_PAD_FRONT * 2u + 16u * v, make_uint4(0u, 0u, 0u, 0u));
    }
    uint32_t recA = row_rec[lane];
    int pbase = 0;
    uint32_t predA = row_pfill[lane];
    uint32_t predB = row_pfill[32 + lane];
    __syncwarp();

    int best = NEG, end_row = 0;
    int po = 0;
    int16_t* Srow = S;
    const int end_lane = fa.len / (8 * NV), end_cell = fa.len % (8 * NV); /* where column len lives */
    /* rows in blocks of 32: the record stream is shifted once per block, not tested once per row */
    int i = 1;
#pragma unroll 1
    for (int blk_end = 31; i <= N; blk_end += 32) {
    const int i_end = blk_end < N ? blk_end : N;
    const uint32_t recN = ldg_pinned(row_rec + blk_end + 1 + lane); /* the next block's records, in flight during this one */
#pragma unroll 1
    for (; i <= i_end; ++i) {
        const uint32_t rec = __shfl_sync(0xffffffffu, recA, i & 31);
        const int np = rec_npred(rec);
        const int prow = rec_prow(rec);
        if (__any_sync(0xffffffffu, prow == 4)) { /* the vote makes the branch provably warp-uniform, see poa_uniform() */
            const int code = rec_code(rec);
            if (dyn_code != code) {
                fill_build_dyn_prof_row(prof_sa + (uint32_t)(4 * prof_stride), code, fa.read, fa.len, prof_stride, fa.mg, fa.xg);
                dyn_code = code;
            }
        }
        Srow += stride;
        int rel = po - pbase;
        if (rel + np > 32) {
            if (rel > 32) { /* a row with > 32 entries jumped past predB */
                const uint2 t = fill_restart_pred_stream(row_pfill, po);
                predA = t.x;
                predB = t.y;
            } else {
                const int src = (lane + rel) & 31;
                const uint32_t xa = __shfl_sync(0xffffffffu, predA, src);
                const uint32_t xb = __shfl_sync(0xffffffffu, predB, src);
                predA = (lane + rel < 32) ? xa : xb;
                predB = row_pfill[po + 32 + lane];
            }
            pbase = po;
            rel = 0;
        }
        /* profile: 8*NV int8 under this lane's columns, widened to int16 pairs */
        uint32_t P[4 * NV];
        {
            const uint32_t psa = prof_sa + (uint32_t)(prow * prof_stride + col0);
#pragma unroll
            for (int v = 0; v < NV; ++v) {
                const uint2 Pb = lds64(psa + 8u * v);
                P[4 * v + 0] = prmt_sext(Pb.x, 0x9180u);
                P[4 * v + 1] = prmt_sext(Pb.x, 0xB3A2u);
                P[4 * v + 2] = prmt_sext(Pb.y, 0x9180u);
                P[4 * v + 3] = prmt_sext(Pb.y, 0xB3A2u);
            }
        }
        uint32_t a[4 * NV];
#pragma unroll
        for (int k = 0; k < 4 * NV; ++k) a[k] = NEG2;

#define POA_WIDE_TERM(cell_sa)                                                                         \
    do {                                                                                               \
        uint32_t left = lds_u16((cell_sa) - 2u) << 16;                                                 \
        _Pragma("unroll") for (int v = 0; v < NV; ++v) {                                               \
            const uint4 V = lds128((cell_sa) + 16u * v);                                               \
            const uint32_t d0 = __funnelshift_l(left, V.x, 16);                                        \
            const uint32_t d1 = __funnelshift_l(V.x, V.y, 16);                                         \
            const uint32_t d2 = __funnelshift_l(V.y, V.z, 16);                                         \
            const uint32_t d3 = __funnelshift_l(V.z, V.w, 16);                                         \
            a[4 * v + 0] = __viaddmax_s16x2(d0, P[4 * v + 0], a[4 * v + 0]);                           \
            a[4 * v + 1] = __viaddmax_s16x2(d1, P[4 * v + 1], a[4 * v + 1]);                           \
            a[4 * v + 2] = __viaddmax_s16x2(d2, P[4 * v + 2], a[4 * v + 2]);                           \
            a[4 * v + 3] = __viaddmax_s16x2(d3, P[4 * v + 3], a[4 * v + 3]);                           \
            a[4 * v + 0] = __viaddmax_s16x2(V.x, G2, a[4 * v + 0]);                                    \
            a[4 * v + 1] = __viaddmax_s16x2(V.y, G2, a[4 * v + 1]);                                    \
            a[4 * v + 2] = __viaddmax_s16x2(V.z, G2, a[4 * v + 2]);                                    \
            a[4 * v + 3] = __viaddmax_s16x2(V.w, G2, a[4 * v + 3]);                                    \
            left = V.w;                                                                                \
        }                                                                                              \
    } while (0)

        if (!rec_far(rec) && np <= 32) {
#pragma unroll 1
            for (int q = 0; q < np; ++q) {
                const uint32_t pe = __shfl_sync(0xffffffffu, predA, rel + q);
                const uint32_t cell_sa = c0_sa + (uint32_t)((int)pe >> 12);
                POA_WIDE_TERM(cell_sa);
            }
        } else {
#pragma unroll 1
            for (int q = 0; q < np; ++q) {
                uint32_t pe;
                if (rel + q < 32) pe = __shfl_sync(0xffffffffu, predA, rel + q);
                else pe = row_pfill[po + q];
                uint32_t cell_sa = c0_sa + (uint32_t)((int)pe >> 12);
                if (__any_sync(0xffffffffu, (pe & 1u) != 0)) { /* predecessor older than the ring: stage its row in the spare slot */
                    const int pr = (int)(fa.row_pred[po + q] & 0xFFFFu);
                    /* staged in the ring slot this row takes at its end (it holds row i - R, out of the ring's reach) */
                    const uint32_t own_sa = ring_sa + RING_PAD_FRONT * 2u + (uint32_t)(i & ring_mask) * ring_row_bytes;
                    fill_stage_far_row(S + (size_t)pr * stride, own_sa, bw);
                    cell_sa = own_sa + (uint32_t)col0 * 2u;
                }
                POA_WIDE_TERM(cell_sa);
            }
        }
#undef POA_WIDE_TERM

        /* inclusive prefix max over the lane's 8*NV cells: inside each register, then register to register */
        a[0] = __vmaxs2(a[0], __byte_perm(a[0], NEG2, 0x1054));
#pragma unroll
        for (int k = 1; k < 4 * NV; ++k)
            a[k] = __vimax3_s16x2(a[k], __byte_perm(a[k], NEG2, 0x1054), __byte_perm(a[k - 1], a[k - 1], 0x3232));
        /* ... then across lanes */
        uint32_t tt = __byte_perm(a[4 * NV - 1], a[4 * NV - 1], 0x3232);
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) tt = __vmaxs2(tt, __shfl_up_sync(0xffffffffu, tt, d));
        uint32_t excl = __shfl_up_sync(0xffffffffu, tt, 1);
        excl = lane == 0 ? NEG2 : excl;
#pragma unroll
        for (int k = 0; k < 4 * NV; ++k) a[k] = __vimax3_s16x2(a[k], excl, NEG2);

        const uint32_t ring_row_sa = c0_sa + RING_PAD_FRONT * 2u + (uint32_t)(i & ring_mask) * ring_row_bytes;
#pragma unroll
        for (int v = 0; v < NV; ++v) {
            const uint4 out = make_uint4(a[4 * v], a[4 * v + 1], a[4 * v + 2], a[4 * v + 3]);
            if (col0 + 8 * v < bw) __stcs(reinterpret_cast<uint4*>(Srow + col0 + 8 * v), out);
            if (col0 + 8 * v + 8 <= ring_cols) sts128(ring_row_sa + 16u * v, out); /* rows are as long as the longest read */
        }
        if (rec_sink(rec)) { /* candidate end cell at column len */
            uint32_t w = a[0];
#pragma unroll
            for (int k = 1; k < 4 * NV; ++k)
                if ((end_cell >> 1) == k) w = a[k];
            int val = (end_cell & 1) ? ((int)w >> 16) : (int)(int16_t)(w & 0xFFFFu);
            val = __shfl_sync(0xffffffffu, val, end_lane);
            if (val > best) {
                best = val;
                end_row = i;
            }
        }
        po += np;
        __syncwarp();
    }
    recA = recN;
    }
    return end_row;
}

struct CudaFill {
    uint32_t smem_sa;    /* shared-window address of the block's dynamic shared memory */
    int32_t prof_stride;
    int32_t ring_stride; /* cells per ring row (>= widest band of the batch) */
    int32_t ring_mask;   /* ring_rows - 1 (power of two) */

    __device__ __forceinline__ int32_t operator()(const Slot& s, const Params& p, WinState& st, const ReadGeom& g,
                                                  const uint8_t* read) {
        FillArgs fa;
        fa.S = s.S;
        fa.row_rec = s.row_rec;
        fa.row_pred = s.row_pred;
        fa.row_pfill = s.row_pfill;
        fa.read = read;
        fa.smem_sa = smem_sa;
        fa.stride = p.stride;
        fa.prof_stride = prof_stride;
        fa.ring_stride = ring_stride;
        fa.ring_mask = ring_mask;
        fa.N = g.n_rows;
        fa.len = g.len;
        fa.colsP = g.colsP;
        fa.bw = g.bw;
        fa.mg = p.match - p.gap;
        fa.xg = p.mismatch - p.gap;
        fa.gap = p.gap;
        Run run{fa};
        return fill_dispatch(g, run); /* fill_variant()'s rule */
    }
    struct Run {
        const FillArgs& fa;
        template <int32_t V>
        __device__ __forceinline__ int32_t run() {
            if (V == FILL_FULLW) return fill_rows<true>(fa);
            if (V == FILL_WIDE1) return fill_rows_wide<1>(fa);
            if (V == FILL_WIDE2) return fill_rows_wide<2>(fa);
            if (V == FILL_WIDE3) return fill_rows_wide<3>(fa);
            if (V == FILL_WIDE4) return fill_rows_wide<4>(fa);
            return fill_rows<false>(fa); /* FILL_CHUNKED_BANDED (other band widths), FILL_CHUNKED_FULL (256-column passes) */
        }
    };
};

#endif /* POA_DEVICE */

} // namespace b200poa
