/*
 * b200poa.h -- C ABI of the H100-native (sm_90a) batched POA consensus engine.
 *
 * This is the drop-in boundary for racon's CUDA polishing path.  Each entry point replaces one
 * member of the C++ interface racon binds today (paths relative to the racon-gpu repository):
 *
 *   b200poa_init                 <- cudapoa::Init()                         vendor/GenomeWorks/cudapoa/include/claraparabricks/genomeworks/cudapoa/cudapoa.hpp:56
 *   b200poa_config_default       <- BatchConfig::BatchConfig(max_seq_sz, max_seq_per_poa, band_width, banding)
 *                                                                           .../cudapoa/batch.hpp:57-80, cudapoa/src/batch.cu:34-71
 *   b200poa_batch_create         <- create_batch(device, stream, max_gpu_mem, output_mask, config, gap, mismatch, match)
 *                                                                           .../cudapoa/batch.hpp:174-181
 *   b200poa_batch_add_group      <- Batch::add_poa_group(per_seq_status, group)   .../cudapoa/batch.hpp:104-105
 *   b200poa_batch_total_poas     <- Batch::get_total_poas()                 .../cudapoa/batch.hpp:110
 *   b200poa_batch_generate       <- Batch::generate_poa()                   .../cudapoa/batch.hpp:113
 *   b200poa_batch_get_consensus  <- Batch::get_consensus(consensus, coverage, output_status)  .../cudapoa/batch.hpp:125-127
 *   b200poa_batch_get_msa        <- Batch::get_msa(msa, output_status)      .../cudapoa/batch.hpp:141-142
 *   b200poa_batch_id             <- Batch::batch_id()                       .../cudapoa/batch.hpp:155
 *   b200poa_batch_reset          <- Batch::reset()                          .../cudapoa/batch.hpp:158
 *   b200poa_batch_destroy        <- Batch::~Batch()
 *   b200poa_layer_order          <- the std::sort in CUDABatchProcessor::addWindow   src/cuda/cudabatch.cpp:96-104
 *                                   (same call as Window::generate_consensus, src/window.cpp:78-85)
 *   b200poa_batch_add_windows    <- the addWindow loop of CUDAPolisher::polish's fill_next_batch
 *                                   src/cuda/cudapolisher.cpp:254-276, over a columnar window arena
 *   b200poa_batch_add_windows_from_aligner <- the same loop over windows whose layers an aligner batch cut on the
 *                                   device (Polisher::initialize's layer loop, src/polisher.cpp:403-457)
 *   b200poa_polish_overlaps      <- Polisher::initialize's window loop + CUDAPolisher::polish for one device,
 *                                   src/polisher.cpp:384-457, src/cuda/cudapolisher.cpp:216-345
 *   b200poa_polish_overlaps_ex   <- the same, plus the windows racon's GPU limits leave to its CPU pass
 *                                   (cudapolisher.cpp:354-383): polished on the device, or handed back
 *   b200poa_polish_overlaps_multi <- the same on every device, contigs too large for one aligner batch split
 *
 * Plain C types only: no C++ objects, no exceptions, no torch types cross this boundary.
 * Status codes are the values of cudapoa::StatusType (cudapoa.hpp:32-45) plus three extensions.
 *
 * Semantics differ from the reference GPU path in one deliberate way: results equal racon's CPU
 * (spoa) path -- spoa's topological order, strict ">" consensus tie-breaks, spoa coverage -- which
 * the reference GPU path does not reproduce (test/racon_test.cpp:311-312 vs :106-107).
 */
#ifndef B200POA_H
#define B200POA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* cudapoa::StatusType values (cudapoa.hpp:32-45) */
enum {
    B200POA_SUCCESS = 0,
    B200POA_EXCEEDED_MAXIMUM_POAS = 1,              /* batch full: launch what you have */
    B200POA_EXCEEDED_MAXIMUM_SEQUENCE_SIZE = 2,     /* per-entry, soft: entry skipped */
    B200POA_EXCEEDED_MAXIMUM_SEQUENCES_PER_POA = 3, /* per-entry, soft: entry skipped */
    B200POA_NODE_COUNT_EXCEEDED_MAXIMUM_GRAPH_SIZE = 4,
    B200POA_EDGE_COUNT_EXCEEDED_MAXIMUM_GRAPH_SIZE = 5,
    B200POA_EXCEEDED_ADAPTIVE_BANDED_MATRIX_SIZE = 6,
    B200POA_SEQ_LEN_EXCEEDED_MAXIMUM_NODES_PER_WINDOW = 7,
    B200POA_LOOP_COUNT_EXCEEDED_UPPER_BOUND = 8,
    B200POA_OUTPUT_TYPE_UNAVAILABLE = 9,
    B200POA_GENERIC_ERROR = 10,
    /* extensions */
    B200POA_ALIGNED_COUNT_EXCEEDED = 11, /* more than 8 mutually aligned nodes in one column */
    B200POA_SCORE_RANGE_EXCEEDED = 12,   /* alignment does not fit int16 cells */
    B200POA_TRACEBACK_LOST = 13,         /* static band did not contain a consistent path */
    B200POA_PARTIAL_SPAN_UNSUPPORTED = 14, /* reserved (partial-span layers are aligned on the device since r01) */
    B200POA_INVALID_ARGUMENT = 15,       /* what the C++ API reports by throwing std::invalid_argument */
    B200POA_CUDA_ERROR = 16              /* what the C++ API reports by aborting in GW_CU_CHECK_ERR */
};

/* cudapoa::BandMode (cudapoa.hpp:47-53).  adaptive_band is not selectable from racon (cudabatch.cpp:59); here it
 * means: align with alignment_band_width first and re-align a read with twice the width whenever its traceback comes
 * close to the band's edge (cudapoa's retry protocol, cudapoa_kernels.cuh:257-303), up to the full matrix. */
enum { B200POA_FULL_BAND = 0, B200POA_STATIC_BAND = 1, B200POA_ADAPTIVE_BAND = 2 };

/* cudapoa::OutputType (cudapoa.hpp:59-63); racon asks for consensus only (cudabatch.cpp:64) */
enum { B200POA_OUTPUT_CONSENSUS = 0x1, B200POA_OUTPUT_MSA = 0x2 };

/* cudapoa::BatchConfig (batch.hpp:57-80).  Fill with b200poa_config_default. */
typedef struct b200poa_config {
    int32_t max_sequence_size;     /* racon: 1023 (cudabatch.cpp:56) */
    int32_t max_consensus_size;    /* 2 * max_sequence_size */
    int32_t max_nodes_per_graph;   /* 3x (full band) / 4x (static band) max_sequence_size */
    int32_t alignment_band_width;  /* racon: 256 */
    int32_t max_sequences_per_poa; /* racon: 200 (cudapolisher.cpp:226) */
    int32_t band_mode;             /* B200POA_FULL_BAND | B200POA_STATIC_BAND | B200POA_ADAPTIVE_BAND */
} b200poa_config;

/* cudapoa::Entry (batch.hpp:45-53) + the layer span racon's Window knows (window.hpp:73) */
typedef struct b200poa_entry {
    const char* seq;       /* borrowed for the duration of the call */
    const int8_t* weights; /* per-base weight (PHRED-33); NULL => 1 per base */
    int32_t length;
    int32_t begin;         /* layer span on the backbone; ignored for entry 0 */
    int32_t end;           /* (begin,end) = (0, backbone_len-1) or (-1,-1) => spans the window */
} b200poa_entry;

typedef struct b200poa_batch b200poa_batch;

int32_t b200poa_init(void);

void b200poa_config_default(b200poa_config* cfg, int32_t max_seq_sz, int32_t max_seq_per_poa,
                            int32_t band_width, int32_t band_mode);

/* stream: a cudaStream_t owned by the caller (cudabatch.cpp:54,74).  max_gpu_mem: device bytes the
 * batch may use (cudapolisher.cpp:233-238 passes 0.9*free/batches). */
int32_t b200poa_batch_create(int32_t device_id, void* stream, size_t max_gpu_mem, int32_t output_mask,
                             const b200poa_config* cfg, int16_t gap_score, int16_t mismatch_score,
                             int16_t match_score, b200poa_batch** out);

/* entries[0] is the backbone, entries[1..n) the layers ALREADY in processing order.
 * per_seq_status (nullable) receives n codes.  Returns B200POA_EXCEEDED_MAXIMUM_POAS when the batch
 * is full (nothing added). */
int32_t b200poa_batch_add_group(b200poa_batch* b, const b200poa_entry* entries, int32_t n,
                                int32_t* per_seq_status);

/* The order racon processes a window's sequences in (rank_out[0] == 0): src/window.cpp:78-85. */
void b200poa_layer_order(int32_t n, const int32_t* begins, int32_t* rank_out);

/*
 * Columnar fast path: add windows [first, n_windows) of a flat arena (layout documented in
 * racon_gpu_b200/windows.py) until the batch is full.  Sequences are in ADD order; the processing
 * order is derived inside with b200poa_layer_order.  *n_added receives the number of windows
 * accepted; seqs_added (nullable, one per accepted window) the number of layers actually staged
 * (cudabatch.cpp:134-153's seqs_added_per_window_).
 */
int32_t b200poa_batch_add_windows(b200poa_batch* b, int64_t n_windows, int64_t first,
                                  const int64_t* win_seq_off, const int64_t* seq_off,
                                  const uint8_t* bases, const int8_t* weights,
                                  const uint8_t* has_weights, const int32_t* begins,
                                  const int32_t* ends, int64_t* n_added, int32_t* seqs_added);

/*
 * Zero-staging variant of b200poa_batch_add_windows for a columnar arena that lives in PINNED host memory (what
 * b200poa_arena_finalize produces): nothing is copied on the host; the batch records the byte range of the arena its
 * windows span and b200poa_batch_generate uploads that range as it is (sequences in add order, the per-sequence tables
 * carry the processing order).  `weight_mode[s]` (b200poa_weight_modes) says per sequence whether its weights are one
 * constant (-1 - constant: nothing to ship) or explicit (>= 0: the weights arena range is uploaded too).  The arena
 * must stay alive and unchanged until the batch's results have been fetched; windows must be added in arena order,
 * and a batch is either staged or pinned between two resets.
 */
int32_t b200poa_batch_add_windows_pinned(b200poa_batch* b, int64_t n_windows, int64_t first,
                                         const int64_t* win_seq_off, const int64_t* seq_off,
                                         const uint8_t* bases, const int8_t* weights,
                                         const uint8_t* has_weights, const int64_t* weight_mode,
                                         const int32_t* begins, const int32_t* ends, int64_t* n_added,
                                         int32_t* seqs_added);
/*
 * Windows whose layers an aligner batch cut on the device (b200aln_batch_set_layer_cut): the rest of the addWindow loop
 * of CUDAPolisher::polish (src/cuda/cudapolisher.cpp:254-276) after racon's own layer loop (src/polisher.cpp:403-457).
 * Window w of the aligner's window range (b200aln_batch_get_layers: first_window + w) is its backbone -- host bytes
 * bb_bases[bb_off[w] .. bb_off[w + 1]) and their qualities bb_qual (same offsets; NULL: a FASTA target, whose '!' dummy
 * quality weighs 0) -- and the aligner's records of that window in add order; the processing order is
 * b200poa_layer_order over their begins.  Adds windows first, first + 1, .. last - 1 of the range until the batch is full
 * (*n_added, seqs_added as for b200poa_batch_add_windows).  The layer bytes and their weights (quality - 33, or 1 for
 * a read without qualities) are gathered from the aligner's device arena into this batch's by a kernel in
 * b200poa_batch_upload: none of them crosses PCIe.  The batch must be on the aligner batch's device, and the aligner
 * batch must stay alive and unreset until this batch's results have been fetched; between two resets a batch gathers
 * from one aligner batch and takes no direct-mode windows.
 */
struct b200aln_batch; /* include/b200aln.h */
int32_t b200poa_batch_add_windows_from_aligner(b200poa_batch* b, const struct b200aln_batch* a, int64_t first,
                                               int64_t last, const int64_t* bb_off, const uint8_t* bb_bases, const uint8_t* bb_qual,
                                               int64_t* n_added, int32_t* seqs_added);

/*
 * Whole job from aligned overlaps on one device (racon_b200::polish_overlaps, racon_gpu_b200/csrc/host/): the loop at the
 * end of Polisher::initialize (src/polisher.cpp:384-457) and the GPU section of CUDAPolisher::polish
 * (src/cuda/cudapolisher.cpp:216-345), in rounds of whole contigs -- one aligner batch (b200aln_batch_set_layer_cut)
 * and `poa_batches` POA batches fed from it with b200poa_batch_add_windows_from_aligner.
 * Contig c: t_bases[t_off[c] .. t_off[c + 1]), qualities at the same offsets of t_qual (NULL: FASTA contigs).  Overlap
 * k, in racon's order after its filtering: contig t_id[k], segment [t_begin[k], t_end[k]), the strand-adjusted read
 * segment q_bases[q_off[k] .. q_off[k + 1]) starting at q_first[k] in the strand-adjusted read, its qualities at the same
 * offsets of q_qual where has_quality[k] (reverse_quality() for '-').  Outputs per window, contig by contig
 * (id_to_first_window_id order): those of b200poa_polisher_polish.  *n_rounds: aligner rounds; h2d / d2h_bytes: PCIe
 * bytes of every batch.  A contig whose overlaps do not fit one aligner batch (aligner_mem) is not split:
 * B200POA_GENERIC_ERROR with *unfit_contig = its index (-1 otherwise).  b200poa_polish_overlaps_multi runs the same on
 * several devices and splits such a contig.
 */
typedef struct b200poa_overlap_options {
    int32_t device_id;
    int32_t poa_batches;           /* racon -c */
    size_t mem_per_poa_batch;      /* 0: 0.9 * free / (poa_batches + 1) */
    int64_t aligner_mem;           /* 0: mem_per_poa_batch */
    int32_t window_length;         /* racon -w */
    double quality_threshold;      /* racon -q */
    int32_t banded;                /* racon -b */
    int32_t match, mismatch, gap;
    int32_t tgs, trim;
    int32_t max_windows_per_batch; /* 0: fill each POA batch */
} b200poa_overlap_options;
int32_t b200poa_polish_overlaps(const b200poa_overlap_options* opt, int64_t n_contigs, const uint8_t* t_bases,
                                const int64_t* t_off, const uint8_t* t_qual, int64_t n_overlaps, const int32_t* t_id,
                                const int32_t* t_begin, const int32_t* t_end, const uint8_t* q_bases,
                                const int64_t* q_off, const uint8_t* q_qual, const uint8_t* has_quality,
                                const int32_t* q_first, uint8_t* cons_out, int32_t stride, int32_t* cons_len,
                                uint8_t* polished, int32_t* status_out, int64_t* n_rounds, int64_t* h2d_bytes,
                                int64_t* d2h_bytes, int64_t* unfit_contig);

/*
 * b200poa_polish_overlaps with the windows racon's GPU limits leave unpolished taken care of (racon_b200::polish_overlaps,
 * overlap_polisher.hpp).  Same arguments and outputs, plus `ex`:
 *   deep_windows   != 0: a second tier of POA batches polishes on the device the windows the first one (racon's limits:
 *                  1023 bases per sequence, 200 sequences per window) cannot take whole -- with at least 3 sequences,
 *                  at most deep_max_sequences_per_poa sequences (0: 65535) and none longer than deep_max_sequence_size
 *                  (0: 16380).  Their consensus is spoa's over all their layers, as on racon's CPU path.  0: the outputs
 *                  of b200poa_polish_overlaps.
 *   export_layers  != 0: every window still unpolished with at least 3 sequences comes back in `exported`, in the
 *                  layout of b200poa_polisher_polish's arguments (racon_gpu_b200/windows.py): per window its backbone
 *                  (weights quality - 33, 0 for a FASTA contig; span (0, 0)) and then its layers in racon's add order
 *                  (weights quality - 33, or 1 with has_weights 0 for a read without qualities).  window_ids[i] is the
 *                  window's index in the per-window outputs.  The library allocates the arrays; release them with
 *                  b200poa_free_export (also after a failed call).  Racon's CPU pass, or b200poa_polisher_* with large
 *                  limits, polishes them (cudapolisher.cpp:354-383).
 * Counters (out): tier2_windows given to the second tier, tier2_polished of them polished there, tier2_batches
 * second-tier batches created (re-created when a later round needs larger limits), exported_windows, exported_bytes
 * (device -> host bytes of the export, included in *d2h_bytes).
 */
typedef struct b200poa_overlap_export {
    int64_t n_windows, n_sequences;
    int64_t* window_ids;  /* [n_windows] */
    int64_t* win_seq_off; /* [n_windows + 1] */
    int64_t* seq_off;     /* [n_sequences + 1] */
    uint8_t* bases;       /* [seq_off[n_sequences]] */
    int8_t* weights;      /* [seq_off[n_sequences]] */
    uint8_t* has_weights; /* [n_sequences] */
    int32_t* begins;      /* [n_sequences] */
    int32_t* ends;        /* [n_sequences] */
} b200poa_overlap_export;
typedef struct b200poa_overlap_ex {
    int32_t deep_windows;
    int32_t export_layers;
    int32_t deep_max_sequence_size;
    int32_t deep_max_sequences_per_poa;
    b200poa_overlap_export exported;
    int64_t tier2_windows, tier2_polished, tier2_batches;
    int64_t exported_windows, exported_bytes;
} b200poa_overlap_ex;
int32_t b200poa_polish_overlaps_ex(const b200poa_overlap_options* opt, b200poa_overlap_ex* ex, int64_t n_contigs,
                                   const uint8_t* t_bases, const int64_t* t_off, const uint8_t* t_qual,
                                   int64_t n_overlaps, const int32_t* t_id, const int32_t* t_begin, const int32_t* t_end,
                                   const uint8_t* q_bases, const int64_t* q_off, const uint8_t* q_qual,
                                   const uint8_t* has_quality, const int32_t* q_first, uint8_t* cons_out, int32_t stride,
                                   int32_t* cons_len, uint8_t* polished, int32_t* status_out, int64_t* n_rounds,
                                   int64_t* h2d_bytes, int64_t* d2h_bytes, int64_t* unfit_contig);
/* frees the arrays of an export and zeroes it */
void b200poa_free_export(b200poa_overlap_export* e);

/*
 * b200poa_polish_overlaps_ex on several devices, with contigs too large for one aligner batch split at window boundaries
 * (racon_b200::polish_overlaps with a device list, overlap_polisher.hpp).  One worker -- an aligner batch, `poa_batches`
 * POA batches and, with deep_windows, a second-tier batch, on a host thread of its own -- per entry of device_ids; a
 * device listed twice runs two workers.  n_devices == 0: one worker on every visible device.  opt->device_id is ignored.
 * mem_per_poa_batch 0: 0.9 * the device's free memory / (workers on it * (poa_batches + 1 + deep_windows)), read once per
 * device before any worker allocates.
 * The work is planned up front in units: runs of whole contigs, as b200poa_polish_overlaps's rounds, and for a contig
 * whose overlaps do not fit one aligner batch alone, consecutive window ranges, each with the overlaps whose window span
 * meets it (in racon's order), each as long as fits.  Every window gets the same layers in the same order as in a
 * whole-contig round.  Every worker gets the smallest device's memory share, and with aligner_mem 0 every unit is
 * planned for it.  A second-tier window is polished exactly when the largest second-tier batch that share allows
 * polishes it (it climbs the sizes from its own in steps of 512), so the outputs and the export (byte for byte,
 * ascending window id) do not depend on the number of workers, which worker ran which unit, or where a contig was
 * split.  They equal b200poa_polish_overlaps_ex's, except that a window its round-sized second tier leaves unpolished
 * for a graph or consensus limit may be polished here.
 * ex: nullable (both options off).  *n_rounds: units; *split_contigs: contigs polished in more than one unit;
 * *repeat_overlaps: alignments done more than once because of the splits (an overlap crossing a unit boundary is aligned
 * in every unit it meets).  B200POA_INVALID_ARGUMENT for a device id out of range, before anything is allocated;
 * B200POA_GENERIC_ERROR with *unfit_contig set when the overlaps of one window alone do not fit one aligner batch.
 */
int32_t b200poa_polish_overlaps_multi(const b200poa_overlap_options* opt, b200poa_overlap_ex* ex, int32_t n_devices,
                                      const int32_t* device_ids, int64_t n_contigs, const uint8_t* t_bases,
                                      const int64_t* t_off, const uint8_t* t_qual, int64_t n_overlaps, const int32_t* t_id,
                                      const int32_t* t_begin, const int32_t* t_end, const uint8_t* q_bases,
                                      const int64_t* q_off, const uint8_t* q_qual, const uint8_t* has_quality,
                                      const int32_t* q_first, uint8_t* cons_out, int32_t stride, int32_t* cons_len,
                                      uint8_t* polished, int32_t* status_out, int64_t* n_rounds, int64_t* h2d_bytes,
                                      int64_t* d2h_bytes, int64_t* unfit_contig, int64_t* split_contigs,
                                      int64_t* repeat_overlaps);

void b200poa_weight_modes(int64_t n_sequences, const int64_t* seq_off, const int8_t* weights,
                          const uint8_t* has_weights, int64_t* weight_mode);

int32_t b200poa_batch_total_poas(const b200poa_batch* b);

/* Asynchronous on the batch's stream: H2D of the staged arena, the POA kernel, D2H of the results. */
int32_t b200poa_batch_generate(b200poa_batch* b);

/* The three stages of b200poa_batch_generate, separately (benchmarks time the kernel alone with
 * inputs already resident in HBM). All asynchronous on the batch's stream. */
int32_t b200poa_batch_upload(b200poa_batch* b);
int32_t b200poa_batch_launch(b200poa_batch* b);
int32_t b200poa_batch_download(b200poa_batch* b);

/*
 * Synchronises the stream and completes the download.  Window i's UNTRIMMED consensus is the lens[i] bytes at
 * cons + offsets[i], its per-base coverage the lens[i] values at cov + offsets[i] (compact arenas: exactly
 * sum(lens) elements crossed PCIe), status[i] its StatusType.  trim[i] packs the span racon's TGS coverage trim
 * keeps (src/window.cpp:118-139, threshold (n_seqs - 1) / 2), evaluated on the device: first = trim & 0xFFFF,
 * last = trim >> 16 (arithmetic; first >= last means "keep the whole consensus", window.cpp:134-137).
 * Pointers are into batch-owned pinned host memory, valid until reset/destroy.  *cov is NULL when the batch was
 * told not to download coverage (B200POA_OPT_DOWNLOAD_COVERAGE = 0).
 */
int32_t b200poa_batch_get_consensus(b200poa_batch* b, const uint8_t** cons, const uint16_t** cov,
                                    const int32_t** lens, const int32_t** status, const int32_t** offsets,
                                    const int32_t** trim);

/*
 * Batch::get_msa (batch.hpp:141-142, cudapoa_batch.cuh:260-313): synchronises and completes the download of the
 * multiple sequence alignments (the batch must have been created with B200POA_OUTPUT_MSA in its output mask, else
 * B200POA_OUTPUT_TYPE_UNAVAILABLE).  Window i's alignment is n_rows[i] rows of n_cols[i] bytes, back to back at
 * msa + offsets[i]; row k belongs to the k-th sequence STAGED for the window (entry order of b200poa_batch_add_group;
 * processing order for the columnar adds), '-' where the sequence has no base in a column.  Rows and columns are those
 * of spoa::Graph::generate_multiple_sequence_alignment (vendor/spoa/src/graph.cpp:373-427), which is what the
 * reference's own test compares cudapoa with (cudapoa/tests/Test_CudapoaGenerateMSA2.cu:117-128).  status[i] is the
 * window's StatusType; an alignment of max_consensus_size columns or more reports
 * B200POA_EXCEEDED_MAXIMUM_SEQUENCE_SIZE like the reference (cudapoa_generate_msa.cuh:203-208) and has n_cols 0.
 * Only the bytes the launch produced cross PCIe (the reference copies max_poas x max_sequences_per_poa x
 * max_consensus_size).  Pointers are into batch-owned pinned host memory, valid until the next generate / reset.
 */
int32_t b200poa_batch_get_msa(b200poa_batch* b, const uint8_t** msa, const int64_t** offsets, const int32_t** n_rows,
                              const int32_t** n_cols, const int32_t** status);

/* Batch options (extensions).  DOWNLOAD_COVERAGE (default 1): 0 = callers that only need the trimmed consensus skip
 * two thirds of the D2H bytes.  TRIM_COUNTS_STAGED (default 0, set before adding windows): 1 = the trim threshold
 * counts the sequences actually staged, which is what the reference GPU adapter does when it truncates a deep
 * window (src/cuda/cudabatch.cpp:134-153, 232-233); 0 = every sequence of the window like the CPU path. */
enum { B200POA_OPT_DOWNLOAD_COVERAGE = 1, B200POA_OPT_TRIM_COUNTS_STAGED = 2 };
int32_t b200poa_batch_set_option(b200poa_batch* b, int32_t option, int64_t value);

int32_t b200poa_batch_id(const b200poa_batch* b);
int32_t b200poa_batch_reset(b200poa_batch* b);
void b200poa_batch_destroy(b200poa_batch* b);

/* introspection used by benchmarks and tests */
typedef struct b200poa_batch_info {
    int32_t n_slots;          /* resident warps = windows in flight on the device */
    int32_t max_poas;         /* window capacity of the batch */
    int64_t arena_capacity;   /* bases capacity */
    int64_t slot_bytes;       /* device bytes per slot */
    int64_t device_bytes;     /* total device allocation */
    int64_t staged_bases;     /* bases currently staged */
    int64_t kernel_launches;  /* kernels launched since creation */
    int32_t smem_bytes;       /* dynamic shared memory per block */
    int32_t blocks_per_sm;    /* occupancy the launch was sized for */
    int64_t h2d_bytes;        /* bytes the last upload moved host -> device */
    int64_t d2h_bytes;        /* bytes the last download + get_consensus moved device -> host */
} b200poa_batch_info;
int32_t b200poa_batch_get_info(const b200poa_batch* b, b200poa_batch_info* info);

/* diagnostics: with B200POA_PHASE_TIMERS=1 in the environment at batch creation, the kernel sums
 * clock64() cycles per phase {program, fill, traceback, add_alignment, topsort, consensus, other}. */
int32_t b200poa_batch_phase_cycles(b200poa_batch* b, uint64_t* out, int32_t n);

const char* b200poa_status_string(int32_t status);

/*
 * Whole-job entry: racon's GPU window scheduler (CUDAPolisher::polish, src/cuda/cudapolisher.cpp:
 * 216-345) over a columnar window arena with HOST buffers: `batches_per_device` batch processors
 * per device (racon -c), one host thread each, a shared window cursor, pinned staging, H2D, the POA
 * kernel, D2H and racon's coverage trim (src/window.cpp:118-139).
 *   device_ids NULL / n_devices 0 => every visible device.
 *   mem_per_batch 0 => 0.9 * free / batches_per_device (cudapolisher.cpp:233-236).
 *   cons_out: n_windows rows of `stride` bytes; cons_len[w] the (trimmed) length; polished[w] is
 *   racon's per-window bool.  false => the row holds the window's BACKBONE (window.cpp:68-71 for < 3
 *   sequences; also when status_out[w] != success or layers were dropped by the batch limits) and the
 *   caller's CPU path may still polish it, as racon does for the reference's failures (cudapolisher.cpp:354-383).
 */
int32_t b200poa_polish_windows(int64_t n_windows, const int64_t* win_seq_off, const int64_t* seq_off,
                               const uint8_t* bases, const int8_t* weights, const uint8_t* has_weights,
                               const int32_t* begins, const int32_t* ends, int32_t tgs, int32_t trim,
                               int32_t match, int32_t mismatch, int32_t gap, int32_t banded,
                               int32_t n_devices, const int32_t* device_ids, int32_t batches_per_device,
                               size_t mem_per_batch, int32_t max_windows_per_round, uint8_t* cons_out,
                               int32_t stride, int32_t* cons_len, uint8_t* polished, int32_t* status_out,
                               int64_t* kernel_launches);

/* Persistent form of b200poa_polish_windows: the batch processors (device workspaces, pinned
 * staging, streams) are created once -- as CUDAPolisher::polish does per run,
 * src/cuda/cudapolisher.cpp:226-240 -- and reused by every polish call.  h2d_bytes / d2h_bytes
 * (nullable) receive the bytes copied across PCIe by the call. */
typedef struct b200poa_polisher b200poa_polisher;
int32_t b200poa_polisher_create(int32_t n_devices, const int32_t* device_ids, int32_t batches_per_device,
                                size_t mem_per_batch, int32_t banded, int32_t match, int32_t mismatch,
                                int32_t gap, b200poa_polisher** out);
int32_t b200poa_polisher_polish(b200poa_polisher* h, int64_t n_windows, const int64_t* win_seq_off,
                                const int64_t* seq_off, const uint8_t* bases, const int8_t* weights,
                                const uint8_t* has_weights, const int32_t* begins, const int32_t* ends,
                                int32_t tgs, int32_t trim, int32_t max_windows_per_round, uint8_t* cons_out,
                                int32_t stride, int32_t* cons_len, uint8_t* polished, int32_t* status_out,
                                int64_t* kernel_launches, int64_t* h2d_bytes, int64_t* d2h_bytes);
void b200poa_polisher_destroy(b200poa_polisher* h);

/* b200poa_polisher_create with every knob: zero fields mean racon's values (cudabatch.cpp:56-59:
 * BatchConfig(1023, 200, 256, mode)).  accept_truncated = 0 (default): a window whose layers were dropped by
 * max_sequence_size / max_sequences_per_poa comes back UNPOLISHED (its backbone, polished = 0, status =
 * the exceeded limit) so that results never silently differ from racon's CPU path; accept_truncated = 1: what the
 * reference GPU adapter does (src/cuda/cudabatch.cpp:134-153, 232-233) -- polish with the layers that fitted, trim
 * threshold = staged layers / 2, report polished = 1. */
typedef struct b200poa_polisher_options {
    int32_t n_devices;
    const int32_t* device_ids;
    int32_t batches_per_device;
    size_t mem_per_batch;
    int32_t banded;                /* 0 full band, 1 static band (racon -b), 2 adaptive band */
    int32_t match, mismatch, gap;
    int32_t max_sequence_size;
    int32_t max_sequences_per_poa;
    int32_t band_width;
    int32_t accept_truncated;
} b200poa_polisher_options;
int32_t b200poa_polisher_create_ex(const b200poa_polisher_options* opt, b200poa_polisher** out);

/* Pack the rows of a [n_rows x stride] byte matrix (row i valid up to lens[i]) back to back into `flat`
 * (capacity >= sum(lens)); offsets[i] (n_rows + 1 entries) receives where row i starts.  Host utility for the final
 * consensus gather (only sum(len) bytes travel).  Returns the number of bytes written. */
int64_t b200poa_compact_rows(const uint8_t* rows, int64_t n_rows, int64_t stride, const int32_t* lens, uint8_t* flat,
                             int64_t* offsets);

/* ---- columnar window construction (SURVEY.md 8(f)-2) ------------------------------------------------
 * Replaces the per-window objects racon builds in Polisher::initialize (src/polisher.cpp:384-457 with
 * createWindow / Window::add_layer, src/window.cpp:15-63) by ONE arena in the layout b200poa_polisher_polish
 * consumes.  Same argument checks as the reference (which exits; here: -1 / INVALID_ARGUMENT), layers of
 * different windows may arrive interleaved, layers of one window keep their add order.  Sequence and quality
 * pointers are borrowed until b200poa_arena_finalize copies them (quality -> weight = char - 33,
 * graph.cpp:138-147; nullptr quality -> weight 1, :124-129).  Building is host-only; finalize additionally page-locks
 * the arena when a CUDA device is present, so that b200poa_polisher_polish_arena uploads batches straight from it
 * (b200poa_batch_add_windows_pinned: no per-batch staging copy). */
typedef struct b200poa_arena b200poa_arena;
b200poa_arena* b200poa_arena_create(void);
int64_t b200poa_arena_add_window(b200poa_arena* a, const char* backbone, uint32_t backbone_length,
                                 const char* quality, uint32_t quality_length); /* window index or -1 */
int32_t b200poa_arena_add_layer(b200poa_arena* a, int64_t window, const char* sequence, uint32_t sequence_length,
                                const char* quality, uint32_t quality_length, uint32_t begin, uint32_t end);
/* the same calls for windows that already exist as columns (layout of b200poa_polisher_polish) */
int32_t b200poa_arena_append_columns(b200poa_arena* a, int64_t n_windows, const int64_t* win_seq_off,
                                     const int64_t* seq_off, const uint8_t* bases, const int8_t* weights,
                                     const uint8_t* has_weights, const int32_t* begins, const int32_t* ends);
int32_t b200poa_arena_finalize(b200poa_arena* a);
/* after finalize: pointers stay valid until destroy */
int32_t b200poa_arena_view(const b200poa_arena* a, int64_t* n_windows, int64_t* n_sequences,
                           const int64_t** win_seq_off, const int64_t** seq_off, const uint8_t** bases,
                           const int8_t** weights, const uint8_t** has_weights, const int32_t** begins,
                           const int32_t** ends);
/* b200poa_polisher_polish over a finalized arena (same outputs) */
int32_t b200poa_polisher_polish_arena(b200poa_polisher* h, const b200poa_arena* a, int32_t tgs, int32_t trim,
                                      int32_t max_windows_per_round, uint8_t* cons_out, int32_t stride,
                                      int32_t* cons_len, uint8_t* polished, int32_t* status_out,
                                      int64_t* kernel_launches, int64_t* h2d_bytes, int64_t* d2h_bytes);
void b200poa_arena_destroy(b200poa_arena* a);

/* The same job driven through the C++ class API that mirrors racon's (racon_b200::createWindow /
 * Window::add_layer / CUDABatchProcessor / polish_windows, racon_gpu_b200/csrc/host/): the path a
 * racon maintainer's code takes.  Same arguments as b200poa_polish_windows. */
int32_t b200poa_polish_windows_via_adapter(int64_t n_windows, const int64_t* win_seq_off,
                                           const int64_t* seq_off, const uint8_t* bases,
                                           const int8_t* weights, const uint8_t* has_weights,
                                           const int32_t* begins, const int32_t* ends, int32_t tgs,
                                           int32_t trim, int32_t match, int32_t mismatch, int32_t gap,
                                           int32_t banded, int32_t n_devices, const int32_t* device_ids,
                                           int32_t batches_per_device, size_t mem_per_batch,
                                           int32_t max_windows_per_round, uint8_t* cons_out, int32_t stride,
                                           int32_t* cons_len, uint8_t* polished);

#ifdef __cplusplus
}
#endif
#endif /* B200POA_H */
