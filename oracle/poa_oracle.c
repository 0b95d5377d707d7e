/*
 * poa_oracle.c -- CPU restatement of racon's spoa consensus path.  TEST INFRASTRUCTURE ONLY:
 * see poa_oracle.h for the list of allowed callers and the parity pins.
 *
 * Every function names the reference lines it restates (paths relative to the reference repository).
 * The scalar engine (sisd_alignment_engine.cpp) is the readable twin of the AVX2 engine racon
 * actually runs (simd_alignment_engine.cpp:700-1045); the two are checked equal through
 * oracle/_ref in tests/test_oracle.py.
 */
#include "poa_oracle.h"

#include <limits.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    int32_t* v;
    int32_t n, cap;
} ivec;

static void iv_push(ivec* a, int32_t x) {
    if (a->n == a->cap) {
        a->cap = a->cap ? a->cap * 2 : 4;
        a->v = (int32_t*)realloc(a->v, sizeof(int32_t) * (size_t)a->cap);
    }
    a->v[a->n++] = x;
}
static void iv_free(ivec* a) {
    free(a->v);
    a->v = NULL;
    a->n = a->cap = 0;
}

typedef struct {
    int32_t src, dst;
    int64_t weight; /* spoa::Edge::total_weight_ */
    ivec labels;    /* spoa::Edge::sequence_labels_ */
} edge_t;

typedef struct {
    char letter;  /* decoder_[code_] : comparisons in spoa are on the decoded char */
    ivec in;      /* edge indices, insertion order (spoa::Node::in_edges_) */
    ivec out;     /* edge indices, insertion order (spoa::Node::out_edges_) */
    ivec aligned; /* node ids, insertion order (spoa::Node::aligned_nodes_ids_) */
} node_t;

struct poa_graph {
    node_t* nodes;
    int32_t nn, ncap;
    edge_t* edges;
    int32_t ne, ecap;
    int32_t num_sequences;
    ivec rank_to_node;
    ivec begin_nodes; /* spoa::Graph::sequences_begin_nodes_ids_ */
};

poa_graph* poa_graph_create(void) { return (poa_graph*)calloc(1, sizeof(poa_graph)); }

void poa_graph_destroy(poa_graph* g) {
    if (!g) return;
    for (int32_t i = 0; i < g->nn; ++i) {
        iv_free(&g->nodes[i].in);
        iv_free(&g->nodes[i].out);
        iv_free(&g->nodes[i].aligned);
    }
    for (int32_t i = 0; i < g->ne; ++i) iv_free(&g->edges[i].labels);
    free(g->nodes);
    free(g->edges);
    iv_free(&g->rank_to_node);
    iv_free(&g->begin_nodes);
    free(g);
}

int32_t poa_graph_num_nodes(const poa_graph* g) { return g->nn; }
int32_t poa_graph_num_edges(const poa_graph* g) { return g->ne; }
void poa_graph_rank_to_node(const poa_graph* g, int32_t* out) {
    memcpy(out, g->rank_to_node.v, sizeof(int32_t) * (size_t)g->rank_to_node.n);
}

/* graph.cpp:88-92 Graph::add_node */
static int32_t add_node(poa_graph* g, char letter) {
    if (g->nn == g->ncap) {
        g->ncap = g->ncap ? g->ncap * 2 : 1024;
        g->nodes = (node_t*)realloc(g->nodes, sizeof(node_t) * (size_t)g->ncap);
    }
    memset(&g->nodes[g->nn], 0, sizeof(node_t));
    g->nodes[g->nn].letter = letter;
    return g->nn++;
}

/* graph.cpp:94-116 Graph::add_edge: bump an existing (begin,end) edge or create one that is
 * appended to begin.out_edges_ and end.in_edges_. */
static void add_edge_labelled(poa_graph* g, int32_t begin, int32_t end, int64_t weight) {
    node_t* b = &g->nodes[begin];
    for (int32_t k = 0; k < b->out.n; ++k) {
        edge_t* e = &g->edges[b->out.v[k]];
        if (e->dst == end) {
            iv_push(&e->labels, g->num_sequences);
            e->weight += weight;
            return;
        }
    }
    if (g->ne == g->ecap) {
        g->ecap = g->ecap ? g->ecap * 2 : 2048;
        g->edges = (edge_t*)realloc(g->edges, sizeof(edge_t) * (size_t)g->ecap);
    }
    edge_t* e = &g->edges[g->ne];
    memset(e, 0, sizeof(*e));
    e->src = begin;
    e->dst = end;
    e->weight = weight;
    iv_push(&e->labels, g->num_sequences);
    iv_push(&g->nodes[begin].out, g->ne);
    iv_push(&g->nodes[end].in, g->ne);
    g->ne++;
}

/* graph.cpp:274-292 Graph::add_sequence: chain of new nodes for seq[begin,end) */
static int32_t add_sequence(poa_graph* g, const char* seq, const uint32_t* w, int32_t begin,
                            int32_t end) {
    if (begin == end) return -1;
    int32_t first = add_node(g, seq[begin]);
    for (int32_t i = begin + 1; i < end; ++i) {
        int32_t id = add_node(g, seq[i]);
        add_edge_labelled(g, id - 1, id, (int64_t)w[i - 1] + w[i]);
    }
    return first;
}

/* graph.cpp:294-354 Graph::topological_sort: iterative DFS, aligned nodes emitted as a group */
static void topological_sort(poa_graph* g) {
    int32_t n = g->nn;
    g->rank_to_node.n = 0;
    uint8_t* marks = (uint8_t*)calloc((size_t)n + 1, 1);
    uint8_t* check = (uint8_t*)malloc((size_t)n + 1);
    memset(check, 1, (size_t)n + 1);
    ivec stack = {0};
    for (int32_t i = 0; i < n; ++i) {
        if (marks[i] != 0) continue;
        iv_push(&stack, i);
        while (stack.n != 0) {
            int32_t id = stack.v[stack.n - 1];
            int valid = 1;
            if (marks[id] != 2) {
                const node_t* nd = &g->nodes[id];
                for (int32_t k = 0; k < nd->in.n; ++k) {
                    int32_t s = g->edges[nd->in.v[k]].src;
                    if (marks[s] != 2) {
                        iv_push(&stack, s);
                        valid = 0;
                    }
                }
                if (check[id]) {
                    for (int32_t k = 0; k < nd->aligned.n; ++k) {
                        int32_t a = nd->aligned.v[k];
                        if (marks[a] != 2) {
                            iv_push(&stack, a);
                            check[a] = 0;
                            valid = 0;
                        }
                    }
                }
                if (valid) {
                    marks[id] = 2;
                    if (check[id]) {
                        iv_push(&g->rank_to_node, id);
                        for (int32_t k = 0; k < nd->aligned.n; ++k)
                            iv_push(&g->rank_to_node, nd->aligned.v[k]);
                    }
                } else {
                    marks[id] = 1;
                }
            }
            if (valid) stack.n--;
        }
    }
    iv_free(&stack);
    free(marks);
    free(check);
}

/* graph.cpp:155-272 Graph::add_alignment (weights overload) */
void poa_graph_add_alignment(poa_graph* g, const poa_pair* aln, int32_t n_aln, const char* seq,
                             int32_t len, const uint32_t* w) {
    if (len == 0) return;
    if (n_aln == 0) { /* graph.cpp:177-185 */
        iv_push(&g->begin_nodes, add_sequence(g, seq, w, 0, len));
        ++g->num_sequences;
        topological_sort(g);
        return;
    }
    int32_t first_valid = -1, last_valid = -1; /* graph.cpp:187-192 valid_seq_ids */
    for (int32_t i = 0; i < n_aln; ++i) {
        if (aln[i].pos != -1) {
            if (first_valid == -1) first_valid = aln[i].pos;
            last_valid = aln[i].pos;
        }
    }
    int32_t tmp = g->nn;
    int32_t begin_node = add_sequence(g, seq, w, 0, first_valid);
    int32_t head = (tmp == g->nn) ? -1 : g->nn - 1;
    int32_t tail = add_sequence(g, seq, w, last_valid + 1, len);
    int32_t new_id = -1;
    int64_t prev_w = (head == -1) ? 0 : (int64_t)w[first_valid - 1];

    for (int32_t i = 0; i < n_aln; ++i) {
        if (aln[i].pos == -1) continue;
        char letter = seq[aln[i].pos];
        int32_t an = aln[i].node;
        if (an == -1) {
            new_id = add_node(g, letter);
        } else if (g->nodes[an].letter == letter) {
            new_id = an;
        } else {
            int32_t aligned_to = -1;
            for (int32_t k = 0; k < g->nodes[an].aligned.n; ++k) {
                int32_t a = g->nodes[an].aligned.v[k];
                if (g->nodes[a].letter == letter) {
                    aligned_to = a;
                    break;
                }
            }
            if (aligned_to == -1) { /* graph.cpp:226-237 */
                new_id = add_node(g, letter);
                int32_t na = g->nodes[an].aligned.n;
                for (int32_t k = 0; k < na; ++k) {
                    int32_t a = g->nodes[an].aligned.v[k];
                    iv_push(&g->nodes[new_id].aligned, a);
                    iv_push(&g->nodes[a].aligned, new_id);
                }
                iv_push(&g->nodes[new_id].aligned, an);
                iv_push(&g->nodes[an].aligned, new_id);
            } else {
                new_id = aligned_to;
            }
        }
        if (begin_node == -1) begin_node = new_id; /* graph.cpp:244-246 */
        if (head != -1) add_edge_labelled(g, head, new_id, prev_w + (int64_t)w[aln[i].pos]);
        head = new_id;
        prev_w = (int64_t)w[aln[i].pos];
    }
    if (tail != -1) add_edge_labelled(g, head, tail, prev_w + (int64_t)w[last_valid + 1]);
    ++g->num_sequences;
    iv_push(&g->begin_nodes, begin_node); /* graph.cpp:269 */
    topological_sort(g);
}

/* sisd_alignment_engine.cpp:94-241 (initialize, kNW/kLinear) + 260-435 (linear) */
int32_t poa_align_nw(const poa_graph* g, const char* seq, int32_t len, int32_t m, int32_t x,
                     int32_t gap, poa_pair** out) {
    *out = NULL;
    if (g->nn == 0 || len == 0) return 0; /* sisd:247-249 */
    const int32_t W = len + 1, Hh = g->nn + 1;
    const int32_t NEG = INT_MIN + 1024;
    int32_t* H = (int32_t*)malloc(sizeof(int32_t) * (size_t)W * (size_t)Hh);
    int32_t* rank = (int32_t*)malloc(sizeof(int32_t) * (size_t)g->nn);
    const int32_t* r2n = g->rank_to_node.v;
    for (int32_t i = 0; i < g->nn; ++i) rank[r2n[i]] = i;

    /* sisd:158-160,186-209 : first row j*g, first column g + max over predecessors */
    H[0] = 0;
    for (int32_t j = 1; j < W; ++j) H[j] = j * gap;
    for (int32_t i = 1; i < Hh; ++i) {
        const node_t* nd = &g->nodes[r2n[i - 1]];
        int32_t pen = nd->in.n == 0 ? 0 : NEG;
        for (int32_t k = 0; k < nd->in.n; ++k) {
            int32_t pi = rank[g->edges[nd->in.v[k]].src] + 1;
            if (H[(size_t)pi * W] > pen) pen = H[(size_t)pi * W];
        }
        H[(size_t)i * W] = pen + gap;
    }

    int32_t max_score = NEG, max_i = -1, max_j = -1;
    for (int32_t r = 0; r < g->nn; ++r) { /* sisd:283-338 */
        const node_t* nd = &g->nodes[r2n[r]];
        const int32_t i = r + 1;
        int32_t* row = &H[(size_t)i * W];
        int32_t pi = nd->in.n == 0 ? 0 : rank[g->edges[nd->in.v[0]].src] + 1;
        const int32_t* prow = &H[(size_t)pi * W];
        for (int32_t j = 1; j < W; ++j) {
            int32_t d = prow[j - 1] + (nd->letter == seq[j - 1] ? m : x);
            int32_t v = prow[j] + gap;
            row[j] = d > v ? d : v;
        }
        for (int32_t p = 1; p < nd->in.n; ++p) {
            pi = rank[g->edges[nd->in.v[p]].src] + 1;
            prow = &H[(size_t)pi * W];
            for (int32_t j = 1; j < W; ++j) {
                int32_t d = prow[j - 1] + (nd->letter == seq[j - 1] ? m : x);
                int32_t v = prow[j] + gap;
                int32_t b = d > v ? d : v;
                if (b > row[j]) row[j] = b;
            }
        }
        for (int32_t j = 1; j < W; ++j) {
            int32_t h = row[j - 1] + gap;
            if (h > row[j]) row[j] = h;
        }
        if (nd->out.n == 0 && max_score < row[W - 1]) { /* sisd:329-331 */
            max_score = row[W - 1];
            max_i = i;
            max_j = W - 1;
        }
    }

    /* backtrack, sisd:340-431 */
    poa_pair* rev = (poa_pair*)malloc(sizeof(poa_pair) * (size_t)(W + Hh));
    int32_t n = 0;
    int32_t i = max_i, j = max_j, prev_i = 0, prev_j = 0;
    while (!(i == 0 && j == 0)) {
        const int32_t Hij = H[(size_t)i * W + j];
        int found = 0;
        if (i != 0 && j != 0) {
            const node_t* nd = &g->nodes[r2n[i - 1]];
            int32_t mc = (nd->letter == seq[j - 1]) ? m : x;
            int32_t np = nd->in.n == 0 ? 1 : nd->in.n;
            for (int32_t p = 0; p < np && !found; ++p) {
                int32_t pi = nd->in.n == 0 ? 0 : rank[g->edges[nd->in.v[p]].src] + 1;
                if (Hij == H[(size_t)pi * W + (j - 1)] + mc) {
                    prev_i = pi;
                    prev_j = j - 1;
                    found = 1;
                }
            }
        }
        if (!found && i != 0) {
            const node_t* nd = &g->nodes[r2n[i - 1]];
            int32_t np = nd->in.n == 0 ? 1 : nd->in.n;
            for (int32_t p = 0; p < np && !found; ++p) {
                int32_t pi = nd->in.n == 0 ? 0 : rank[g->edges[nd->in.v[p]].src] + 1;
                if (Hij == H[(size_t)pi * W + j] + gap) {
                    prev_i = pi;
                    prev_j = j;
                    found = 1;
                }
            }
        }
        if (!found && j != 0 && Hij == H[(size_t)i * W + j - 1] + gap) {
            prev_i = i;
            prev_j = j - 1;
            found = 1;
        }
        if (!found) { /* cannot happen for a consistent matrix */
            fprintf(stderr, "[poa_oracle] traceback lost at (%d,%d)\n", i, j);
            abort();
        }
        rev[n].node = (i == prev_i) ? -1 : r2n[i - 1];
        rev[n].pos = (j == prev_j) ? -1 : j - 1;
        ++n;
        i = prev_i;
        j = prev_j;
    }
    poa_pair* fwd = (poa_pair*)malloc(sizeof(poa_pair) * (size_t)(n ? n : 1));
    for (int32_t k = 0; k < n; ++k) fwd[k] = rev[n - 1 - k];
    free(rev);
    free(H);
    free(rank);
    *out = fwd;
    return n;
}

/* graph.cpp:44-58 Node::coverage : distinct sequence labels over in- and out-edges */
static uint32_t node_coverage(const poa_graph* g, int32_t id, uint8_t* seen) {
    const node_t* nd = &g->nodes[id];
    uint32_t c = 0;
    memset(seen, 0, (size_t)g->num_sequences + 1);
    for (int pass = 0; pass < 2; ++pass) {
        const ivec* lst = pass == 0 ? &nd->in : &nd->out;
        for (int32_t k = 0; k < lst->n; ++k) {
            const edge_t* e = &g->edges[lst->v[k]];
            for (int32_t l = 0; l < e->labels.n; ++l) {
                if (!seen[e->labels.v[l]]) {
                    seen[e->labels.v[l]] = 1;
                    ++c;
                }
            }
        }
    }
    return c;
}

/* graph.cpp:544-589 Graph::branch_completion */
static int32_t branch_completion(const poa_graph* g, int64_t* scores, int32_t* pred, int32_t rank) {
    const int32_t* r2n = g->rank_to_node.v;
    int32_t node_id = r2n[rank];
    const node_t* nd = &g->nodes[node_id];
    for (int32_t k = 0; k < nd->out.n; ++k) {
        const node_t* dst = &g->nodes[g->edges[nd->out.v[k]].dst];
        for (int32_t q = 0; q < dst->in.n; ++q) {
            int32_t s = g->edges[dst->in.v[q]].src;
            if (s != node_id) scores[s] = -1;
        }
    }
    int64_t max_score = 0;
    int32_t max_id = 0;
    for (int32_t i = rank + 1; i < g->nn; ++i) {
        int32_t id = r2n[i];
        scores[id] = -1;
        pred[id] = -1;
        const node_t* cur = &g->nodes[id];
        for (int32_t k = 0; k < cur->in.n; ++k) {
            const edge_t* e = &g->edges[cur->in.v[k]];
            if (scores[e->src] == -1) continue;
            if (scores[id] < e->weight ||
                (scores[id] == e->weight && scores[pred[id]] <= scores[e->src])) {
                scores[id] = e->weight;
                pred[id] = e->src;
            }
        }
        if (pred[id] != -1) scores[id] += scores[pred[id]];
        if (max_score < scores[id]) {
            max_score = scores[id];
            max_id = id;
        }
    }
    return max_id;
}

static uint64_t consensus_digest(const poa_graph* g, const int64_t* scores, const int32_t* pred, int32_t max_id,
                                 int64_t* overflow);

/* graph.cpp:440-457 generate_consensus(dst, verbose=false) + 494-542 traverse_heaviest_bundle.  cons_digest (nullable,
 * 2 values): consensus_digest() after the first loop and after the last branch_completion; rounds: how many
 * branch_completion ran; overflow: scores that do not fit 32 bits. */
static int32_t graph_consensus(poa_graph* g, char** cons, uint32_t** cov, uint64_t* cons_digest, int32_t* rounds,
                               int64_t* overflow);
int32_t poa_graph_consensus(poa_graph* g, char** cons, uint32_t** cov) {
    return graph_consensus(g, cons, cov, NULL, NULL, NULL);
}
static int32_t graph_consensus(poa_graph* g, char** cons, uint32_t** cov, uint64_t* cons_digest, int32_t* rounds,
                               int64_t* overflow) {
    const int32_t n = g->nn;
    const int32_t* r2n = g->rank_to_node.v;
    int32_t* pred = (int32_t*)malloc(sizeof(int32_t) * (size_t)(n + 1));
    int64_t* scores = (int64_t*)malloc(sizeof(int64_t) * (size_t)(n + 1));
    for (int32_t i = 0; i < n; ++i) {
        pred[i] = -1;
        scores[i] = -1;
    }
    int32_t max_id = 0;
    for (int32_t r = 0; r < n; ++r) {
        int32_t id = r2n[r];
        const node_t* nd = &g->nodes[id];
        for (int32_t k = 0; k < nd->in.n; ++k) {
            const edge_t* e = &g->edges[nd->in.v[k]];
            if (scores[id] < e->weight ||
                (scores[id] == e->weight && scores[pred[id]] <= scores[e->src])) {
                scores[id] = e->weight;
                pred[id] = e->src;
            }
        }
        if (pred[id] != -1) scores[id] += scores[pred[id]];
        if (scores[max_id] < scores[id]) max_id = id;
    }
    if (cons_digest) cons_digest[0] = consensus_digest(g, scores, pred, max_id, overflow);
    if (rounds) *rounds = 0;
    if (g->nodes[max_id].out.n != 0) {
        int32_t* n2r = (int32_t*)malloc(sizeof(int32_t) * (size_t)n);
        for (int32_t i = 0; i < n; ++i) n2r[r2n[i]] = i;
        while (g->nodes[max_id].out.n != 0) {
            max_id = branch_completion(g, scores, pred, n2r[max_id]);
            if (rounds) ++*rounds;
        }
        free(n2r);
    }
    if (cons_digest) cons_digest[1] = consensus_digest(g, scores, pred, max_id, overflow);
    int32_t* path = (int32_t*)malloc(sizeof(int32_t) * (size_t)(n + 1));
    int32_t len = 0;
    while (pred[max_id] != -1) {
        path[len++] = max_id;
        max_id = pred[max_id];
    }
    path[len++] = max_id;
    *cons = (char*)malloc((size_t)len + 1);
    *cov = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)len);
    uint8_t* seen = (uint8_t*)malloc((size_t)g->num_sequences + 1);
    for (int32_t k = 0; k < len; ++k) {
        int32_t id = path[len - 1 - k];
        (*cons)[k] = g->nodes[id].letter;
        uint32_t c = node_coverage(g, id, seen);
        for (int32_t a = 0; a < g->nodes[id].aligned.n; ++a)
            c += node_coverage(g, g->nodes[id].aligned.v[a], seen);
        (*cov)[k] = c;
    }
    (*cons)[len] = 0;
    free(seen);
    free(path);
    free(pred);
    free(scores);
    return len;
}

/* graph.cpp:592-673 extract_subgraph_nodes + subgraph.  mapping (size g->nn) maps subgraph id ->
 * graph id (graph.cpp:675-683 update_alignment). */
static poa_graph* subgraph(const poa_graph* g, int32_t begin, int32_t end, int32_t* mapping) {
    const int32_t n = g->nn;
    uint8_t* is_sub = (uint8_t*)calloc((size_t)n + 1, 1);
    ivec stack = {0};
    iv_push(&stack, end);
    while (stack.n) {
        int32_t id = stack.v[--stack.n];
        if (!is_sub[id] && id >= begin) {
            const node_t* nd = &g->nodes[id];
            for (int32_t k = 0; k < nd->in.n; ++k) iv_push(&stack, g->edges[nd->in.v[k]].src);
            for (int32_t k = 0; k < nd->aligned.n; ++k) iv_push(&stack, nd->aligned.v[k]);
            is_sub[id] = 1;
        }
    }
    iv_free(&stack);
    poa_graph* s = poa_graph_create();
    s->num_sequences = g->num_sequences;
    int32_t* g2s = (int32_t*)malloc(sizeof(int32_t) * (size_t)(n + 1));
    for (int32_t i = 0; i < n; ++i) {
        mapping[i] = -1;
        g2s[i] = -1;
    }
    for (int32_t i = 0; i < n; ++i) {
        if (!is_sub[i]) continue;
        int32_t sid = add_node(s, g->nodes[i].letter);
        g2s[i] = sid;
        mapping[sid] = i;
    }
    for (int32_t i = 0; i < n; ++i) {
        if (!is_sub[i]) continue;
        const node_t* nd = &g->nodes[i];
        for (int32_t k = 0; k < nd->in.n; ++k) {
            const edge_t* e = &g->edges[nd->in.v[k]];
            if (g2s[e->src] == -1) continue;
            add_edge_labelled(s, g2s[e->src], g2s[i], e->weight);
        }
        for (int32_t k = 0; k < nd->aligned.n; ++k) {
            if (g2s[nd->aligned.v[k]] == -1) continue;
            iv_push(&s->nodes[g2s[i]].aligned, g2s[nd->aligned.v[k]]);
        }
    }
    topological_sort(s);
    free(g2s);
    free(is_sub);
    return s;
}

/* Hash of one alignment, the way the engine's test build hashes the one it adds to the graph (poa_core.cuh
 * aln_digest): the wrapping sum over pairs k (k = 0 leftmost) of mix64(k << 32 | pos << 16 | node), node and pos as
 * int16 (-1 included), with splitmix64's finaliser as mix64. */
static uint64_t digest_mix64(uint64_t x) {
    x ^= x >> 30;
    x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27;
    x *= 0x94d049bb133111ebull;
    x ^= x >> 31;
    return x;
}
static uint64_t alignment_digest(const poa_pair* aln, int32_t n) {
    uint64_t t = 0;
    for (int32_t k = 0; k < n; ++k) {
        const uint64_t key = (uint64_t)(uint16_t)(int16_t)aln[k].node | ((uint64_t)(uint16_t)(int16_t)aln[k].pos << 16) |
                             ((uint64_t)(uint32_t)k << 32);
        t += digest_mix64(key + 0x9e3779b97f4a7c15ull);
    }
    return t;
}

/* The engine stores a weight or a score as int32 (poa_core.cuh Slot::e_w, c_score) where spoa keeps int64: the hashes
 * below take the low 32 bits, as the engine's wrapping sums would hold them, and count every value that does not fit
 * (so that a truncation shows up as a failure instead of as a silent agreement). */
static uint32_t low32(int64_t v, int64_t* overflow) {
    if (overflow && (v > INT32_MAX || v < INT32_MIN)) ++*overflow;
    return (uint32_t)(uint64_t)v;
}

/* Hash of the graph, the way the engine's test build hashes its own (poa_core.cuh graph_digest): the wrapping sum over
 * nodes v of mix64(v | letter << 16 | rank << 24 | coverage << 40) (coverage as Node::coverage counts it, by labels),
 * for the aligned id at list position q mix64(v | q << 16 | id << 24 | 1 << 56), and for the in-edge at list position
 * k mix64(mix64(v | k << 16 | source << 32 | 2 << 56) + weight), the weight's low 32 bits. */
static uint64_t graph_digest(const poa_graph* g, int64_t* overflow) {
    const uint64_t K = 0x9e3779b97f4a7c15ull;
    int32_t* rank = (int32_t*)malloc(sizeof(int32_t) * (size_t)(g->nn + 1));
    uint8_t* seen = (uint8_t*)malloc((size_t)g->num_sequences + 1);
    for (int32_t r = 0; r < g->rank_to_node.n; ++r) rank[g->rank_to_node.v[r]] = r;
    uint64_t t = 0;
    for (int32_t v = 0; v < g->nn; ++v) {
        const node_t* nd = &g->nodes[v];
        t += digest_mix64(((uint64_t)v | ((uint64_t)(uint8_t)nd->letter << 16) | ((uint64_t)(uint16_t)rank[v] << 24) |
                           ((uint64_t)(uint16_t)node_coverage(g, v, seen) << 40)) + K);
        for (int32_t q = 0; q < nd->aligned.n; ++q)
            t += digest_mix64(((uint64_t)v | ((uint64_t)q << 16) | ((uint64_t)nd->aligned.v[q] << 24) | (1ull << 56)) + K);
        for (int32_t k = 0; k < nd->in.n; ++k) {
            const edge_t* e = &g->edges[nd->in.v[k]];
            const uint64_t h = digest_mix64(((uint64_t)v | ((uint64_t)k << 16) | ((uint64_t)e->src << 32) | (2ull << 56)) + K);
            t += digest_mix64(h + low32(e->weight, overflow));
        }
    }
    free(seen);
    free(rank);
    return t;
}

/* Hash of a subgraph's member order as graph ids (poa_core.cuh sub_digest): sum over k of mix64(k << 32 | id | 3 << 56) */
static uint64_t subgraph_digest(const poa_graph* s, const int32_t* mapping) {
    uint64_t t = 0;
    for (int32_t k = 0; k < s->rank_to_node.n; ++k)
        t += digest_mix64(((uint64_t)(uint16_t)mapping[s->rank_to_node.v[k]] | ((uint64_t)k << 32) | (3ull << 56)) +
                          0x9e3779b97f4a7c15ull);
    return t;
}

/* Hash of the consensus scores (poa_core.cuh cons_digest): sum over nodes v of mix64(mix64(v | 4 << 56) + (score |
 * pred << 32)), both as their low 32 bits, plus mix64(max_id | 5 << 56) */
static uint64_t consensus_digest(const poa_graph* g, const int64_t* scores, const int32_t* pred, int32_t max_id,
                                 int64_t* overflow) {
    const uint64_t K = 0x9e3779b97f4a7c15ull;
    uint64_t t = digest_mix64(((uint64_t)(uint32_t)max_id | (5ull << 56)) + K);
    for (int32_t v = 0; v < g->nn; ++v)
        t += digest_mix64(digest_mix64(((uint64_t)v | (4ull << 56)) + K) +
                          ((uint64_t)low32(scores[v], overflow) | ((uint64_t)(uint32_t)pred[v] << 32)));
    return t;
}

/* per sequence of a window: what poa_oracle_graph_digests reports (all nullable) */
typedef struct {
    uint64_t* graph_digest;
    int32_t* graph_nodes;
    int32_t* graph_edges;
    uint64_t* sub_digest;
    int32_t* sub_count;
    int64_t* overflow;
} graph_trace;

/* window.cpp:73-116: the graph of one window -- backbone, then every layer aligned (whole graph or subgraph) and added.
 * aln_digest / aln_count (nullable, n_seqs each): per sequence the digest and length of the alignment that was added
 * (graph ids; 0 and 0 for the backbone).  gt (nullable): per sequence the graph after it was added, and the subgraph a
 * partial-span read was aligned to. */
static poa_graph* window_graph(int32_t n_seqs, const char* const* seqs, const int32_t* lens,
                               const int8_t* const* weights, const int32_t* begins, const int32_t* ends,
                               int32_t m, int32_t x, int32_t gap, int64_t* stats, uint64_t* aln_digest,
                               int32_t* aln_count, const graph_trace* gt) {
    int32_t maxlen = 0;
    for (int32_t i = 0; i < n_seqs; ++i)
        if (lens[i] > maxlen) maxlen = lens[i];
    uint32_t* w = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)(maxlen + 1));

    poa_graph* g = poa_graph_create();
    if (aln_digest) aln_digest[0] = 0;
    if (aln_count) aln_count[0] = 0;
    for (int32_t k = 0; k < lens[0]; ++k) w[k] = weights[0] ? (uint32_t)weights[0][k] : 1u;
    poa_graph_add_alignment(g, NULL, 0, seqs[0], lens[0], w); /* window.cpp:73-76 */
    if (gt) {
        gt->graph_digest[0] = graph_digest(g, gt->overflow);
        gt->graph_nodes[0] = g->nn;
        gt->graph_edges[0] = g->ne;
        gt->sub_digest[0] = 0;
        gt->sub_count[0] = 0;
    }

    const uint32_t L = (uint32_t)lens[0];
    const uint32_t offset = (uint32_t)(0.01 * L); /* window.cpp:87 */
    for (int32_t i = 1; i < n_seqs; ++i) {
        poa_pair* aln = NULL;
        int32_t n_aln;
        if (gt) {
            gt->sub_digest[i] = 0;
            gt->sub_count[i] = 0;
        }
        if (!begins || ((uint32_t)begins[i] < offset && (uint32_t)ends[i] > L - offset)) { /* window.cpp:92-95 */
            if (stats) {
                stats[2] += (int64_t)g->nn * (lens[i] + 1);
                stats[4] += (int64_t)g->nn * (lens[i] + 1 < 256 ? lens[i] + 1 : 256);
            }
            n_aln = poa_align_nw(g, seqs[i], lens[i], m, x, gap, &aln);
        } else { /* window.cpp:96-103 */
            int32_t* mapping = (int32_t*)malloc(sizeof(int32_t) * (size_t)(g->nn + 1));
            poa_graph* s = subgraph(g, begins[i], ends[i], mapping);
            if (gt) {
                gt->sub_digest[i] = subgraph_digest(s, mapping);
                gt->sub_count[i] = s->nn;
            }
            if (stats) {
                stats[2] += (int64_t)s->nn * (lens[i] + 1);
                stats[4] += (int64_t)s->nn * (lens[i] + 1 < 256 ? lens[i] + 1 : 256);
            }
            n_aln = poa_align_nw(s, seqs[i], lens[i], m, x, gap, &aln);
            for (int32_t k = 0; k < n_aln; ++k)
                if (aln[k].node != -1) aln[k].node = mapping[aln[k].node];
            poa_graph_destroy(s);
            free(mapping);
        }
        if (aln_digest) aln_digest[i] = alignment_digest(aln, n_aln);
        if (aln_count) aln_count[i] = n_aln;
        for (int32_t k = 0; k < lens[i]; ++k) w[k] = weights[i] ? (uint32_t)weights[i][k] : 1u;
        poa_graph_add_alignment(g, aln, n_aln, seqs[i], lens[i], w);
        free(aln);
        if (stats) stats[3] += 1;
        if (gt) {
            gt->graph_digest[i] = graph_digest(g, gt->overflow);
            gt->graph_nodes[i] = g->nn;
            gt->graph_edges[i] = g->ne;
        }
    }
    free(w);
    return g;
}

/* window.cpp:65-142 Window::generate_consensus */
int32_t poa_oracle_window_consensus(int32_t n_seqs, const char* const* seqs, const int32_t* lens,
                                    const int8_t* const* weights, const int32_t* begins,
                                    const int32_t* ends, int32_t tgs, int32_t trim, int32_t m,
                                    int32_t x, int32_t gap, char* cons_out, uint32_t* cov_out,
                                    int32_t max_out, int32_t* polished, int64_t* stats) {
    if (stats) stats[0] = stats[1] = stats[2] = stats[3] = stats[4] = stats[5] = 0;
    if (n_seqs < 3) { /* window.cpp:68-71 */
        if (polished) *polished = 0;
        if (lens[0] > max_out) return -1;
        memcpy(cons_out, seqs[0], (size_t)lens[0]);
        if (cov_out) memset(cov_out, 0, sizeof(uint32_t) * (size_t)lens[0]);
        return lens[0];
    }
    poa_graph* g = window_graph(n_seqs, seqs, lens, weights, begins, ends, m, x, gap, stats, NULL, NULL, NULL);

    char* cons = NULL;
    uint32_t* cov = NULL;
    int32_t clen = poa_graph_consensus(g, &cons, &cov);
    if (stats) {
        stats[0] = g->nn;
        stats[1] = g->ne;
    }
    int32_t b = 0, e = clen - 1;
    if (tgs && trim) { /* window.cpp:118-139 */
        uint32_t avg = (uint32_t)(n_seqs - 1) / 2;
        for (; b < clen; ++b)
            if (cov[b] >= avg) break;
        for (; e >= 0; --e)
            if (cov[e] >= avg) break;
        if (b >= e) { /* chimeric warning: keep the untrimmed consensus */
            b = 0;
            e = clen - 1;
        }
    }
    int32_t out_len = e - b + 1;
    int32_t ret = out_len;
    if (out_len > max_out) {
        ret = -1;
    } else {
        memcpy(cons_out, cons + b, (size_t)out_len);
        if (cov_out) memcpy(cov_out, cov + b, sizeof(uint32_t) * (size_t)out_len);
    }
    if (polished) *polished = 1;
    free(cons);
    free(cov);
    poa_graph_destroy(g);
    return ret;
}

/* ------------------------------------------------------------------------------------------
 * Multiple sequence alignment  (graph.cpp:373-389 initialize_multiple_sequence_alignment,
 * :391-427 generate_multiple_sequence_alignment with include_consensus = false, Node::successor :31-43).
 * This is what the reference's own MSA test holds cudapoa's Batch::get_msa against
 * (vendor/GenomeWorks/cudapoa/tests/Test_CudapoaGenerateMSA2.cu:62-79,117-128).
 * Returns the number of rows (= sequences); *rows_out is ONE malloc'ed block of n_rows x *msa_len bytes.
 * ---------------------------------------------------------------------------------------- */
int32_t poa_graph_msa(const poa_graph* g, char** rows_out, int32_t* msa_len) {
    int32_t* msa_id = (int32_t*)malloc(sizeof(int32_t) * (size_t)(g->nn + 1));
    int32_t n_cols = 0;
    for (int32_t i = 0; i < g->nn; ++i) { /* graph.cpp:379-386: a node and its aligned nodes share one column */
        int32_t id = g->rank_to_node.v[i];
        msa_id[id] = n_cols;
        for (int32_t j = 0; j < g->nodes[id].aligned.n; ++j) msa_id[g->rank_to_node.v[++i]] = n_cols;
        ++n_cols;
    }
    char* rows = (char*)malloc((size_t)g->num_sequences * (size_t)n_cols + 1);
    memset(rows, '-', (size_t)g->num_sequences * (size_t)n_cols);
    for (int32_t i = 0; i < g->num_sequences; ++i) { /* graph.cpp:400-414 */
        char* row = rows + (size_t)i * (size_t)n_cols;
        int32_t id = g->begin_nodes.v[i];
        for (;;) {
            row[msa_id[id]] = g->nodes[id].letter;
            int32_t next = -1; /* Node::successor: first out-edge that carries this sequence's label */
            for (int32_t k = 0; k < g->nodes[id].out.n && next < 0; ++k) {
                const edge_t* e = &g->edges[g->nodes[id].out.v[k]];
                for (int32_t q = 0; q < e->labels.n; ++q)
                    if (e->labels.v[q] == i) {
                        next = e->dst;
                        break;
                    }
            }
            if (next < 0) break;
            id = next;
        }
    }
    free(msa_id);
    *rows_out = rows;
    *msa_len = n_cols;
    return g->num_sequences;
}

/* The MSA of one window whose graph is built like window.cpp:73-116 builds it (sequences in processing order; a
 * cudapoa-style group is the special case "every layer spans the window": begins/ends NULL). */
int32_t poa_oracle_window_msa(int32_t n_seqs, const char* const* seqs, const int32_t* lens,
                              const int8_t* const* weights, const int32_t* begins, const int32_t* ends,
                              int32_t m, int32_t x, int32_t gap, char** rows_out, int32_t* msa_len) {
    if (!ends) begins = NULL;
    poa_graph* g = window_graph(n_seqs, seqs, lens, weights, begins, ends, m, x, gap, NULL, NULL, NULL, NULL);
    int32_t n = poa_graph_msa(g, rows_out, msa_len);
    poa_graph_destroy(g);
    return n;
}

void poa_oracle_free(void* p) { free(p); }

/* ------------------------------------------------------------------------------------------
 * Flat-batch runner: same role as racon::Polisher::polish (src/polisher.cpp:486-548): one task
 * per window, here with a shared cursor over pthreads.
 * ---------------------------------------------------------------------------------------- */
#include <pthread.h>

typedef struct {
    int64_t n_windows;
    const int64_t* win_seq_off;
    const int64_t* seq_off;
    const uint8_t* bases;
    const int8_t* weights;
    const uint8_t* has_weights;
    const int32_t* begins;
    const int32_t* ends;
    const int32_t* order;
    int32_t tgs, trim, m, x, gap;
    char* cons_out;
    uint16_t* cov_out;
    int32_t stride;
    int32_t* cons_len;
    uint8_t* polished;
    int64_t* stats;
    uint64_t* aln_digest; /* set: the job digests alignments (poa_oracle_alignment_digests) instead of polishing */
    int32_t* aln_count;
    graph_trace graph;    /* graph.graph_digest set: the job digests graphs (poa_oracle_graph_digests) */
    uint64_t* cons_digest;
    int32_t* cons_rounds;
    int64_t* overflow;    /* [n_windows] */
    int32_t* max_indegree; /* [n_windows] */
    int64_t cursor;
    pthread_mutex_t mu;
} batch_job;

static void* batch_worker(void* arg) {
    batch_job* job = (batch_job*)arg;
    int32_t cap = 0;
    const char** seqs = NULL;
    int32_t* lens = NULL;
    const int8_t** wts = NULL;
    int32_t *bg = NULL, *en = NULL;
    uint32_t* cov = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)job->stride);
    for (;;) {
        pthread_mutex_lock(&job->mu);
        int64_t w = job->cursor++;
        pthread_mutex_unlock(&job->mu);
        if (w >= job->n_windows) break;
        int64_t s0 = job->win_seq_off[w];
        int32_t n = (int32_t)(job->win_seq_off[w + 1] - s0);
        if (n > cap) {
            cap = n;
            seqs = (const char**)realloc((void*)seqs, sizeof(char*) * (size_t)cap);
            lens = (int32_t*)realloc(lens, sizeof(int32_t) * (size_t)cap);
            wts = (const int8_t**)realloc((void*)wts, sizeof(int8_t*) * (size_t)cap);
            bg = (int32_t*)realloc(bg, sizeof(int32_t) * (size_t)cap);
            en = (int32_t*)realloc(en, sizeof(int32_t) * (size_t)cap);
        }
        for (int32_t k = 0; k < n; ++k) {
            int64_t s = s0 + job->order[s0 + k];
            seqs[k] = (const char*)(job->bases + job->seq_off[s]);
            lens[k] = (int32_t)(job->seq_off[s + 1] - job->seq_off[s]);
            wts[k] = job->has_weights[s] ? job->weights + job->seq_off[s] : NULL;
            bg[k] = job->begins[s];
            en[k] = job->ends[s];
        }
        if (job->aln_digest) {
            poa_graph_destroy(window_graph(n, seqs, lens, wts, bg, en, job->m, job->x, job->gap, NULL,
                                           job->aln_digest + s0, job->aln_count + s0, NULL));
            continue;
        }
        if (job->graph.graph_digest) {
            int64_t* of = job->overflow + w;
            *of = 0;
            const graph_trace gt = {job->graph.graph_digest + s0, job->graph.graph_nodes + s0,
                                    job->graph.graph_edges + s0, job->graph.sub_digest + s0, job->graph.sub_count + s0,
                                    of};
            poa_graph* g = window_graph(n, seqs, lens, wts, bg, en, job->m, job->x, job->gap, NULL, NULL, NULL, &gt);
            int32_t deg = 0;
            for (int32_t v = 0; v < g->nn; ++v)
                if (g->nodes[v].in.n > deg) deg = g->nodes[v].in.n;
            job->max_indegree[w] = deg;
            char* cons = NULL;
            uint32_t* ccov = NULL;
            graph_consensus(g, &cons, &ccov, job->cons_digest + 2 * w, job->cons_rounds + w, of);
            free(cons);
            free(ccov);
            poa_graph_destroy(g);
            continue;
        }
        int32_t pol = 0;
        int32_t len = poa_oracle_window_consensus(
            n, seqs, lens, wts, bg, en, job->tgs, job->trim, job->m, job->x, job->gap,
            job->cons_out + w * (int64_t)job->stride, cov, job->stride, &pol,
            job->stats ? job->stats + 6 * w : NULL);
        job->cons_len[w] = len;
        job->polished[w] = (uint8_t)pol;
        if (job->cov_out && len > 0)
            for (int32_t k = 0; k < len; ++k)
                job->cov_out[w * (int64_t)job->stride + k] = (uint16_t)cov[k];
    }
    free(cov);
    free((void*)seqs);
    free(lens);
    free((void*)wts);
    free(bg);
    free(en);
    return NULL;
}

static void run_batch_job(batch_job* job, int32_t n_threads) {
    pthread_mutex_init(&job->mu, NULL);
    if (n_threads <= 1) {
        batch_worker(job);
    } else {
        pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)n_threads);
        for (int32_t t = 0; t < n_threads; ++t) pthread_create(&th[t], NULL, batch_worker, job);
        for (int32_t t = 0; t < n_threads; ++t) pthread_join(th[t], NULL);
        free(th);
    }
    pthread_mutex_destroy(&job->mu);
}

void poa_oracle_alignment_digests(int64_t n_windows, const int64_t* win_seq_off, const int64_t* seq_off,
                                  const uint8_t* bases, const int8_t* weights, const uint8_t* has_weights,
                                  const int32_t* begins, const int32_t* ends, const int32_t* order, int32_t m,
                                  int32_t x, int32_t gap, int32_t n_threads, uint64_t* aln_digest, int32_t* aln_count) {
    batch_job job;
    memset(&job, 0, sizeof(job));
    job.n_windows = n_windows;
    job.win_seq_off = win_seq_off;
    job.seq_off = seq_off;
    job.bases = bases;
    job.weights = weights;
    job.has_weights = has_weights;
    job.begins = begins;
    job.ends = ends;
    job.order = order;
    job.m = m;
    job.x = x;
    job.gap = gap;
    job.aln_digest = aln_digest;
    job.aln_count = aln_count;
    run_batch_job(&job, n_threads);
}

void poa_oracle_graph_digests(int64_t n_windows, const int64_t* win_seq_off, const int64_t* seq_off,
                              const uint8_t* bases, const int8_t* weights, const uint8_t* has_weights,
                              const int32_t* begins, const int32_t* ends, const int32_t* order, int32_t m, int32_t x,
                              int32_t gap, int32_t n_threads, uint64_t* graph_digest, int32_t* graph_nodes,
                              int32_t* graph_edges, uint64_t* sub_digest, int32_t* sub_count, uint64_t* cons_digest,
                              int32_t* cons_rounds, int64_t* overflow, int32_t* max_indegree) {
    batch_job job;
    memset(&job, 0, sizeof(job));
    job.n_windows = n_windows;
    job.win_seq_off = win_seq_off;
    job.seq_off = seq_off;
    job.bases = bases;
    job.weights = weights;
    job.has_weights = has_weights;
    job.begins = begins;
    job.ends = ends;
    job.order = order;
    job.m = m;
    job.x = x;
    job.gap = gap;
    job.graph.graph_digest = graph_digest;
    job.graph.graph_nodes = graph_nodes;
    job.graph.graph_edges = graph_edges;
    job.graph.sub_digest = sub_digest;
    job.graph.sub_count = sub_count;
    job.cons_digest = cons_digest;
    job.cons_rounds = cons_rounds;
    job.overflow = overflow;
    job.max_indegree = max_indegree;
    run_batch_job(&job, n_threads);
}

void poa_oracle_polish_windows(int64_t n_windows, const int64_t* win_seq_off, const int64_t* seq_off,
                               const uint8_t* bases, const int8_t* weights,
                               const uint8_t* has_weights, const int32_t* begins,
                               const int32_t* ends, const int32_t* order, int32_t tgs, int32_t trim,
                               int32_t m, int32_t x, int32_t gap, int32_t n_threads, char* cons_out,
                               uint16_t* cov_out, int32_t stride, int32_t* cons_len,
                               uint8_t* polished, int64_t* stats) {
    batch_job job;
    memset(&job, 0, sizeof(job));
    job.n_windows = n_windows;
    job.win_seq_off = win_seq_off;
    job.seq_off = seq_off;
    job.bases = bases;
    job.weights = weights;
    job.has_weights = has_weights;
    job.begins = begins;
    job.ends = ends;
    job.order = order;
    job.tgs = tgs;
    job.trim = trim;
    job.m = m;
    job.x = x;
    job.gap = gap;
    job.cons_out = cons_out;
    job.cov_out = cov_out;
    job.stride = stride;
    job.cons_len = cons_len;
    job.polished = polished;
    job.stats = stats;
    run_batch_job(&job, n_threads);
}

/* ------------------------------------------------------------------------------------------------
 * Edit distance of two long strings (the metric of racon's end-to-end goldens, test/racon_test.cpp:
 * 16-25 uses edlib's global alignment distance): Ukkonen's band with a doubling threshold, O(n*k).
 * Test helper for the stitched-contig checks.
 * ---------------------------------------------------------------------------------------------- */
int64_t poa_oracle_edit_distance(const char* a, int64_t la, const char* b, int64_t lb) {
    if (la < lb) {
        const char* t = a; a = b; b = t;
        int64_t tl = la; la = lb; lb = tl;
    }
    /* la >= lb; rows over a, columns over b */
    for (int64_t k = 64;; k *= 2) {
        if (k > la) k = la;
        const int64_t W = 2 * k + 1, INF = 1 << 30;
        int64_t* prev = (int64_t*)malloc(sizeof(int64_t) * (size_t)(W + 2));
        int64_t* cur = (int64_t*)malloc(sizeof(int64_t) * (size_t)(W + 2));
        /* cell (i, j) lives at index j - i + k + 1, diagonals -k..k around the main diagonal shifted by 0 */
        for (int64_t d = 0; d < W + 2; ++d) prev[d] = INF;
        for (int64_t j = 0; j <= lb && j <= k; ++j) prev[j + k + 1] = j;
        for (int64_t i = 1; i <= la; ++i) {
            for (int64_t d = 0; d < W + 2; ++d) cur[d] = INF;
            int64_t jlo = i - k < 0 ? 0 : i - k, jhi = i + k > lb ? lb : i + k;
            for (int64_t j = jlo; j <= jhi; ++j) {
                const int64_t d = j - i + k + 1;
                int64_t v = INF;
                if (j == 0) v = i;
                else {
                    const int64_t sub = prev[d] + (a[i - 1] != b[j - 1]);  /* (i-1, j-1): same diagonal */
                    const int64_t del = prev[d + 1] + 1;                     /* (i-1, j) */
                    const int64_t ins = cur[d - 1] + 1;                      /* (i, j-1) */
                    v = sub < del ? sub : del;
                    if (ins < v) v = ins;
                }
                cur[d] = v;
            }
            int64_t* t = prev; prev = cur; cur = t;
        }
        int64_t res = INF;
        if (lb - la + k + 1 >= 1 && lb - la + k + 1 <= W) res = prev[lb - la + k + 1];
        free(prev);
        free(cur);
        if (res <= k || k >= la) return res;
    }
}
