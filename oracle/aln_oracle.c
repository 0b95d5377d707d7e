/*
 * aln_oracle.c -- CPU restatement of the overlap alignment of racon's CPU path (TEST INFRASTRUCTURE ONLY).
 *
 * racon aligns every overlap with edlib (src/overlap.cpp:205-224: edlibAlign(q, t, {k = -1, EDLIB_MODE_NW,
 * EDLIB_TASK_PATH}) + edlibAlignmentToCigar(EDLIB_CIGAR_STANDARD)).  edlib (vendor/edlib/edlib/src/edlib.cpp, pinned in
 * the reference tree) is a bit-vector implementation; WHICH of the many optimal alignments it returns is decided by two
 * rules that can be stated on the plain edit-distance matrix D (D[i][j] = distance of q[0..i) and t[0..j)):
 *
 *   obtainAlignment (edlib.cpp:1128-1176): a sub-problem (n query x m target characters, known optimum `best`) is
 *     - trivial when n == 0 (m deletions) or m == 0 (n insertions)                                        (:1135-1142)
 *     - traced back directly when (2*8 + 4) * ceil(n / 64) * m + 2*4 * m < 2^20 bytes                        (:1155-1157)
 *     - split by Hirschberg otherwise                                                                   (:1172-1175)
 *   obtainAlignmentTraceback (:909-1126): from the last cell, at every cell take the FIRST possible move of
 *     up (query character alone: EDLIB_EDOP_INSERT) if D[i-1][j] + 1 == D[i][j]                         (:983-1013)
 *     left (target character alone: EDLIB_EDOP_DELETE) if D[i][j-1] + 1 == D[i][j]                      (:1015-1044)
 *     diagonal (MATCH if D[i-1][j-1] == D[i][j] else MISMATCH)                                          (:1046-1093)
 *     and once a border is reached run along it                                                 (:987-991,1021-1027,1052-1065)
 *   obtainAlignmentHirschberg (:1198-1344): split the target at lh = m / 2; with L[r] = distance of q[0..r] and t[0..lh)
 *     and R[r] = distance of q[r..n) and t[lh..m), take the FIRST query index r = 0 .. n-2 with L[r] + R[r+1] == best
 *     (:1282-1290); failing that the border cases r = -1 (lh + R[0], :1292-1299), then r = n-1 (L[n-1] + (m - lh),
 *     :1300-1308); recurse on (q[0..r], t[0..lh), L) and (q[r+1..n), t[lh..m), R)                       (:1321-1333).
 * The band edlib computes in (Ukkonen, k = best) never changes these choices: every value a rule compares is <= best,
 * and inside the band such values are exact (cells outside it are > best).
 *
 * Pinned: tests/test_aligner.py holds this restatement against the UNMODIFIED edlib compiled into oracle/_ref
 * (ref_edlib_nw) on thousands of random pairs around every threshold and on the real lambda-phage overlaps of the
 * reference's test data.  Only tests/, smoke() and bench.py's CPU legs may load it.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { OP_MATCH = 0, OP_INSERT = 1, OP_DELETE = 2, OP_MISMATCH = 3 }; /* edlib.h EDLIB_EDOP_* */

typedef struct {
    uint8_t* ops;
    int64_t n, cap;
    int overflow;
} opbuf;

static void emit(opbuf* o, uint8_t op, int64_t count) {
    for (int64_t k = 0; k < count; ++k) {
        if (o->n < o->cap) o->ops[o->n] = op;
        else o->overflow = 1;
        o->n++;
    }
}

/* last column of the distance matrix of q[0..n) (step sq: +1 forward, -1 backward from q) against t[0..m) (step st):
 * col[i] = D[i][m], i = 0..n.  Exported: the tests hold the engine's Hirschberg middle columns against it. */
void aln_oracle_last_column(const char* q, int32_t n, int sq, const char* t, int32_t m, int st, int32_t* col) {
    for (int32_t i = 0; i <= n; ++i) col[i] = i;
    for (int32_t j = 1; j <= m; ++j) {
        const char tc = t[(int64_t)(j - 1) * st];
        int32_t diag = col[0];
        col[0] = j;
        for (int32_t i = 1; i <= n; ++i) {
            const int32_t up = col[i - 1] + 1, left = col[i] + 1, dg = diag + (q[(int64_t)(i - 1) * sq] == tc ? 0 : 1);
            diag = col[i];
            int32_t v = up < left ? up : left;
            if (dg < v) v = dg;
            col[i] = v;
        }
    }
}

/* edlib.cpp:909-1126 on the full matrix of a small sub-problem */
static void traceback(const char* q, int32_t n, const char* t, int32_t m, opbuf* out) {
    int32_t* D = (int32_t*)malloc(sizeof(int32_t) * (size_t)(n + 1) * (size_t)(m + 1));
    const size_t W = (size_t)m + 1;
    for (int32_t j = 0; j <= m; ++j) D[j] = j;
    for (int32_t i = 1; i <= n; ++i) {
        D[i * W] = i;
        for (int32_t j = 1; j <= m; ++j) {
            int32_t v = D[(i - 1) * W + j] + 1;
            const int32_t l = D[i * W + j - 1] + 1, d = D[(i - 1) * W + j - 1] + (q[i - 1] == t[j - 1] ? 0 : 1);
            if (l < v) v = l;
            if (d < v) v = d;
            D[i * W + j] = v;
        }
    }
    /* back to front, reversed at the end like edlib.cpp:1123 */
    uint8_t* rev = (uint8_t*)malloc((size_t)n + (size_t)m + 1);
    int64_t k = 0;
    int32_t i = n, j = m;
    while (i > 0 || j > 0) {
        if (i == 0) {
            rev[k++] = OP_DELETE;
            --j;
        } else if (j == 0) {
            rev[k++] = OP_INSERT;
            --i;
        } else {
            const int32_t cur = D[i * W + j];
            if (D[(i - 1) * W + j] + 1 == cur) {
                rev[k++] = OP_INSERT;
                --i;
            } else if (D[i * W + j - 1] + 1 == cur) {
                rev[k++] = OP_DELETE;
                --j;
            } else {
                rev[k++] = D[(i - 1) * W + j - 1] == cur ? OP_MATCH : OP_MISMATCH;
                --i;
                --j;
            }
        }
    }
    while (k > 0) emit(out, rev[--k], 1);
    free(rev);
    free(D);
}

static int align_rec(const char* q, int32_t n, const char* t, int32_t m, int32_t best, opbuf* out) {
    if (n == 0 || m == 0) { /* edlib.cpp:1135-1142 */
        emit(out, n == 0 ? OP_DELETE : OP_INSERT, (int64_t)n + m);
        return 0;
    }
    const int64_t blocks = (n + 63) / 64;
    const int64_t data = (2 * 8 + 4) * blocks * m + 2 * 4 * (int64_t)m; /* edlib.cpp:1155-1156 */
    if (data < 1024 * 1024) {
        traceback(q, n, t, m, out);
        return 0;
    }
    const int32_t lh = m / 2, rh = m - lh; /* edlib.cpp:1216-1217 */
    int32_t* L = (int32_t*)malloc(sizeof(int32_t) * (size_t)(n + 1));
    int32_t* Rr = (int32_t*)malloc(sizeof(int32_t) * (size_t)(n + 1));
    aln_oracle_last_column(q, n, 1, t, lh, 1, L);                      /* L[i]  = D(q[0..i), t[0..lh))                */
    aln_oracle_last_column(q + n - 1, n, -1, t + m - 1, rh, -1, Rr);   /* Rr[i] = D(q[n-i..n), t[lh..m))              */
    int32_t r = -2, ls = 0, rs = 0;
    for (int32_t idx = 0; idx <= n - 2; ++idx) { /* edlib.cpp:1282-1290: scoresLeft[idx] + scoresRight[idx + 1] */
        if (L[idx + 1] + Rr[n - idx - 1] == best) {
            r = idx;
            ls = L[idx + 1];
            rs = Rr[n - idx - 1];
            break;
        }
    }
    if (r == -2 && lh + Rr[n] == best) { /* :1292-1299 */
        r = -1;
        ls = lh;
        rs = Rr[n];
    }
    if (r == -2 && L[n] + rh == best) { /* :1300-1308 */
        r = n - 1;
        ls = L[n];
        rs = rh;
    }
    free(L);
    free(Rr);
    if (r == -2) return 1; /* edlib.cpp:1313-1317: best is not the optimum */
    const int32_t ul = r + 1;
    if (align_rec(q, ul, t, lh, ls, out)) return 1;
    return align_rec(q + ul, n - ul, t + lh, rh, rs, out);
}

/* The edit operations edlibAlign(q, t, NW, PATH) returns (left to right); *score = the edit distance.
 * Returns their number, or -1 (empty input, ops buffer too small, inconsistency). */
int64_t aln_oracle_nw(const char* q, int32_t n, const char* t, int32_t m, uint8_t* ops, int64_t cap, int32_t* score) {
    if (n <= 0 || m <= 0) return -1;
    int32_t* col = (int32_t*)malloc(sizeof(int32_t) * (size_t)(n + 1));
    aln_oracle_last_column(q, n, 1, t, m, 1, col);
    const int32_t best = col[n];
    free(col);
    if (score) *score = best;
    opbuf o = {ops, 0, cap, 0};
    if (align_rec(q, n, t, m, best, &o) || o.overflow) return -1;
    return o.n;
}

/* edlibAlignmentToCigar(..., EDLIB_CIGAR_STANDARD) (edlib.cpp:262-316): run lengths of M (match or mismatch), I, D.
 * Returns the string length (without NUL), or -1 if cap is too small. */
int64_t aln_oracle_cigar(const uint8_t* ops, int64_t n_ops, char* out, int64_t cap) {
    static const char letter[4] = {'M', 'I', 'D', 'M'};
    int64_t w = 0;
    for (int64_t i = 0; i < n_ops;) {
        int64_t j = i;
        while (j < n_ops && letter[ops[j]] == letter[ops[i]]) ++j;
        char tmp[24];
        int len = 0;
        for (int64_t v = j - i; v > 0; v /= 10) tmp[len++] = (char)('0' + v % 10);
        if (w + len + 2 > cap) return -1;
        while (len > 0) out[w++] = tmp[--len];
        out[w++] = letter[ops[i]];
        i = j;
    }
    if (w + 1 > cap) return -1;
    out[w] = 0;
    return w;
}

/*
 * Breaking points of an overlap from its alignment (racon::Overlap::find_breaking_points_from_cigar,
 * src/overlap.cpp:226-290), restated on edit operations instead of CIGAR text (M and X both advance query and target and
 * count as "match" there, :245; I advances the query, :268; D the target, :271).
 *   window ends (:229-235): every multiple i of window_length with t_begin < i < t_end gives i - 1, then t_end - 1;
 *   q_ptr starts at q_first - 1 with q_first = strand ? q_length - q_end : q_begin (:241), t_ptr at t_begin - 1 (:242);
 *   a window that saw at least one M/X emits its first one as (t, q) and its last one as (t + 1, q + 1) when the target
 *   position reaches the window's end, on an M/X or a D (:252-263, :274-283).
 * out receives (t, q) pairs, 2 per emitted window; returns the number of pairs, -1 if cap is too small.
 */
int64_t aln_oracle_breaking_points(const uint8_t* ops, int64_t n_ops, int32_t q_first, int32_t t_begin, int32_t t_end,
                                   int32_t window_length, uint32_t* out, int64_t cap) {
    int64_t n_out = 0;
    int64_t next_end = -1; /* the current window's end */
    int64_t i_mult = ((int64_t)t_begin / window_length + 1) * (int64_t)window_length; /* smallest multiple > t_begin */
    next_end = i_mult < t_end ? i_mult - 1 : (int64_t)t_end - 1;
    int found = 0;
    int64_t q_ptr = (int64_t)q_first - 1, t_ptr = (int64_t)t_begin - 1;
    uint32_t first_t = 0, first_q = 0, last_t = 0, last_q = 0;
    for (int64_t k = 0; k < n_ops; ++k) {
        const uint8_t op = ops[k];
        int target_moved = 0;
        if (op == OP_MATCH || op == OP_MISMATCH) {
            ++q_ptr;
            ++t_ptr;
            if (!found) {
                found = 1;
                first_t = (uint32_t)t_ptr;
                first_q = (uint32_t)q_ptr;
            }
            last_t = (uint32_t)(t_ptr + 1);
            last_q = (uint32_t)(q_ptr + 1);
            target_moved = 1;
        } else if (op == OP_INSERT) {
            ++q_ptr;
        } else {
            ++t_ptr;
            target_moved = 1;
        }
        if (target_moved && t_ptr == next_end) {
            if (found) {
                if (n_out + 2 > cap) return -1;
                out[2 * n_out] = first_t;
                out[2 * n_out + 1] = first_q;
                out[2 * n_out + 2] = last_t;
                out[2 * n_out + 3] = last_q;
                n_out += 2;
            }
            found = 0;
            if (next_end == (int64_t)t_end - 1) break;
            i_mult += window_length;
            next_end = i_mult < t_end ? i_mult - 1 : (int64_t)t_end - 1;
        }
    }
    return n_out;
}
