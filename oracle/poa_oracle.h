/*
 * poa_oracle.h -- CPU restatement of racon's spoa consensus path (TEST INFRASTRUCTURE ONLY).
 *
 * This is the parity oracle for the GPU POA engine.  It restates, in plain C, the
 * reference algorithm that racon's CPU polisher runs per window:
 *   racon::Window::generate_consensus            src/window.cpp:65-142
 *   spoa::SisdAlignmentEngine::linear (NW)       vendor/spoa/src/sisd_alignment_engine.cpp:94-241,260-435
 *   spoa::Graph::add_alignment / add_edge        vendor/spoa/src/graph.cpp:94-116,155-292
 *   spoa::Graph::topological_sort                vendor/spoa/src/graph.cpp:294-354
 *   spoa::Graph::generate_consensus & friends    vendor/spoa/src/graph.cpp:44-58,440-589
 *   spoa::Graph::subgraph / update_alignment     vendor/spoa/src/graph.cpp:592-683
 *   spoa::Graph::generate_multiple_sequence_alignment  vendor/spoa/src/graph.cpp:373-427
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * may load this library.  The product (racon_gpu_b200/) never links, imports or calls it.
 *
 * Parity pin: checked against (a) the spoa GlobalConsensus / GlobalConsensusWithQualities
 * golden strings (vendor/spoa/test/spoa_test.cpp:220-238,283-301; fixtures in tests/golden/)
 * and (b) the real reference compiled from its sources into oracle/_ref (see
 * oracle/Makefile) on thousands of seeded windows (tests/test_oracle.py).
 */
#ifndef POA_ORACLE_H
#define POA_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct poa_graph poa_graph;

typedef struct {
    int32_t node; /* graph node id or -1 */
    int32_t pos;  /* read position or -1  */
} poa_pair;

poa_graph* poa_graph_create(void);
void poa_graph_destroy(poa_graph* g);
int32_t poa_graph_num_nodes(const poa_graph* g);
int32_t poa_graph_num_edges(const poa_graph* g);
/* rank_to_node order after the last topological sort; out must hold num_nodes entries */
void poa_graph_rank_to_node(const poa_graph* g, int32_t* out);

/* Global (NW) linear-gap alignment of seq against the graph.  Returns the number of pairs
 * written into *out (malloc'ed, caller frees), in left-to-right order. */
int32_t poa_align_nw(const poa_graph* g, const char* seq, int32_t len, int32_t m, int32_t x,
                     int32_t gap, poa_pair** out);

/* weights[i] is the per-base weight (quality - 33, or 1). */
void poa_graph_add_alignment(poa_graph* g, const poa_pair* aln, int32_t n_aln, const char* seq,
                             int32_t len, const uint32_t* weights);

/* Heaviest-bundle consensus; *cons (not NUL terminated) and *cov are malloc'ed. Returns length. */
int32_t poa_graph_consensus(poa_graph* g, char** cons, uint32_t** cov);

/*
 * Window-level oracle == racon::Window::generate_consensus.
 *   seqs[0] is the backbone; seqs[1..n) are the layers ALREADY in processing order
 *   (the order window.cpp:84-85's std::sort produces).
 *   weights[i] may be NULL => weight 1 for every base (window.cpp:105-107).
 *   begins/ends: layer span on the backbone (ignored for i == 0).
 *   tgs != 0 && trim != 0 enables the coverage trim (window.cpp:118-139).
 * Outputs: cons_out must hold max_out bytes, cov_out (nullable) max_out uint32 (coverage of the
 * UNTRIMMED consensus is trimmed alongside).  Returns consensus length, or -1 if max_out too small.
 * *polished receives window.cpp's return value; *stats (nullable, 6 x int64) receives
 * {final node count, final edge count, sum over reads of rows x (len+1) DP cells, #reads aligned,
 *  sum over reads of rows x min(len+1, 256) (the cells of a 256-column band), 0}.
 */
int32_t poa_oracle_window_consensus(int32_t n_seqs, const char* const* seqs, const int32_t* lens,
                                    const int8_t* const* weights, const int32_t* begins,
                                    const int32_t* ends, int32_t tgs, int32_t trim, int32_t m,
                                    int32_t x, int32_t gap, char* cons_out, uint32_t* cov_out,
                                    int32_t max_out, int32_t* polished, int64_t* stats);

/*
 * Flat-batch runner (same layout as oracle/ref_driver.cpp:ref_polish_windows): window w owns
 * sequences [win_seq_off[w], win_seq_off[w+1]) given in ADD order; order[s] (same indexing) is the
 * local index of the sequence processed at that step (order[win_seq_off[w]] == 0), i.e. the
 * permutation window.cpp:78-85 computes.  n_threads pthreads share a window cursor.
 * cons_out: n_windows rows of `stride` bytes; cov_out nullable (n_windows x stride uint16).
 * stats nullable: n_windows x 6 int64 (see poa_oracle_window_consensus).
 */
void poa_oracle_polish_windows(int64_t n_windows, const int64_t* win_seq_off, const int64_t* seq_off,
                               const uint8_t* bases, const int8_t* weights,
                               const uint8_t* has_weights, const int32_t* begins,
                               const int32_t* ends, const int32_t* order, int32_t tgs, int32_t trim,
                               int32_t m, int32_t x, int32_t gap, int32_t n_threads, char* cons_out,
                               uint16_t* cov_out, int32_t stride, int32_t* cons_len,
                               uint8_t* polished, int64_t* stats);

/* The alignments spoa adds to each window's graph, same flat layout and processing order as
 * poa_oracle_polish_windows: per sequence (ADD-order index of its window's first sequence + processing position) the
 * wrapping sum over pairs k (k = 0 leftmost) of mix64(k << 32 | (uint16)pos << 16 | (uint16)node) with graph node ids
 * (a subgraph alignment mapped back, graph.cpp:675-683) and the number of pairs; 0 and 0 for the backbone. */
void poa_oracle_alignment_digests(int64_t n_windows, const int64_t* win_seq_off, const int64_t* seq_off,
                                  const uint8_t* bases, const int8_t* weights, const uint8_t* has_weights,
                                  const int32_t* begins, const int32_t* ends, const int32_t* order, int32_t m,
                                  int32_t x, int32_t gap, int32_t n_threads, uint64_t* aln_digest, int32_t* aln_count);

/* spoa's graph of each window, hashed the way the engine's test build hashes its own (poa_core.cuh graph_digest,
 * sub_digest, cons_digest); same flat layout and processing order as poa_oracle_alignment_digests.  Per sequence: the
 * graph after it was added (the backbone: after the chain) with its node and edge counts, and for a partial-span read
 * the member order of the subgraph it was aligned to (graph ids) with the member count (else 0 and 0).  Per window:
 * the consensus scores after traverse_heaviest_bundle's first loop and after the last branch_completion (2 values),
 * the number of branch_completion rounds, how many weights or scores did not fit 32 bits (the engine keeps them as
 * int32; the hashes take the low 32 bits), and the largest in-degree of the final graph. */
void poa_oracle_graph_digests(int64_t n_windows, const int64_t* win_seq_off, const int64_t* seq_off,
                              const uint8_t* bases, const int8_t* weights, const uint8_t* has_weights,
                              const int32_t* begins, const int32_t* ends, const int32_t* order, int32_t m, int32_t x,
                              int32_t gap, int32_t n_threads, uint64_t* graph_digest, int32_t* graph_nodes,
                              int32_t* graph_edges, uint64_t* sub_digest, int32_t* sub_count, uint64_t* cons_digest,
                              int32_t* cons_rounds, int64_t* overflow, int32_t* max_indegree);

/* spoa::Graph::generate_multiple_sequence_alignment(dst, false)  (graph.cpp:373-427): one row per sequence in the
 * order they were added, '-' where the sequence has no base in a column.  *rows_out is one malloc'ed block of
 * n_rows x *msa_len bytes (free with poa_oracle_free); returns n_rows. */
int32_t poa_graph_msa(const poa_graph* g, char** rows_out, int32_t* msa_len);
/* The same for a window built like racon builds it (sequences in processing order; begins/ends NULL: every layer
 * spans the window, i.e. a plain cudapoa group). */
int32_t poa_oracle_window_msa(int32_t n_seqs, const char* const* seqs, const int32_t* lens,
                              const int8_t* const* weights, const int32_t* begins, const int32_t* ends,
                              int32_t m, int32_t x, int32_t gap, char** rows_out, int32_t* msa_len);
void poa_oracle_free(void* p);

/* Global edit distance of two long strings (banded, doubling threshold); test helper for the stitched-contig
 * goldens of test/racon_test.cpp:88-130,176-196. */
int64_t poa_oracle_edit_distance(const char* a, int64_t la, const char* b, int64_t lb);

#ifdef __cplusplus
}
#endif
#endif
