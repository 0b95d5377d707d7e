/*
 * overlap_polisher.hpp -- polish contigs from aligned overlaps on the device without the host window arena:
 * the loop at the end of racon's Polisher::initialize (src/polisher.cpp:400-457) and the GPU section of
 * CUDAPolisher::polish (src/cuda/cudapolisher.cpp:216-345), on one device or on several.
 *
 * The work runs in UNITS (overlap_units.hpp), planned from the input before any batch exists: runs of whole contigs, and
 * with a device list, window ranges of a contig too large for one aligner batch.  A window only receives layers from
 * overlaps on its own contig, so a unit is a run of windows together with every overlap whose window span meets it, in
 * racon's order.  One aligner batch per unit aligns them, forms the breaking points and cuts the layers on the device
 * (b200aln_batch_set_layer_cut); the device's POA batches then gather the layers of the windows the unit owns from the
 * aligner's arena (b200poa_batch_add_windows_from_aligner), and only then is the aligner batch reset.  Without a device
 * list a contig whose overlaps do not fit one aligner batch is reported (unfit_contig), never split.
 *
 * Each WORKER -- one per entry of the device list, so a device listed twice runs two -- owns an aligner batch,
 * `poa_batches` POA batches, an optional second-tier batch and their streams, on a host thread of its own.  Workers
 * claim units from one cursor and write the rows of the windows they own directly; the export is merged in unit order,
 * which is ascending window id.  Units depend on the input and the aligner budget only; every worker gets the smallest
 * device's memory share; and each second-tier window climbs the batch sizes from its own until it is polished or no
 * larger batch fits that share (polish_unit), so the outputs do not depend on how many workers ran the units, which
 * one took which unit, or where a contig was split.
 *
 * The POA batches have racon's GPU limits (1023 bases per sequence, 200 sequences per window, cudabatch.cpp:56-59).  With
 * deep_windows, a second tier takes the windows they cannot take whole -- more than 200 sequences, or one longer than
 * 1023 bases -- in one more POA batch per worker sized from the unit's records (b200aln_batch_get_layers): its
 * max_sequences_per_poa the deepest such window's sequence count, its max_sequence_size their longest sequence rounded
 * up to a multiple of 512 less one.  That batch lives across units and is re-created only when a unit needs larger
 * limits (with a device list: also when a window climbs to a larger size).  With export_layers, every window still unpolished after both tiers that has at least 3 sequences comes back
 * as a host window arena (b200aln_batch_export_layers: one kernel and one D2H of exactly its layers' bytes), so that
 * racon's CPU pass can redo it as it does for the windows its GPU path fails (cudapolisher.cpp:354-383).
 * Parsing, overlap filtering (remove_invalid_overlaps), the CPU redo of unpolished windows and stitching stay in racon.
 */
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

namespace racon_b200 {

struct OverlapPolishOptions {
    int32_t device = 0;               /* the device without a device list */
    int32_t poa_batches = 1;          /* racon -c: POA batches of a worker */
    size_t mem_per_poa_batch = 0;     /* 0 = 0.9 * free / (workers on the device * (poa_batches + 1 + deep_windows)) */
    int64_t aligner_mem = 0;          /* 0 = the same share as one POA batch */
    int32_t window_length = 500;      /* racon -w */
    double quality_threshold = 10.0;  /* racon -q */
    int32_t banded = 0;               /* racon -b */
    int32_t match = 3, mismatch = -5, gap = -4;
    bool tgs = true, trim = true;     /* window type kTGS and racon's --no-trimming left off */
    int32_t max_windows_per_batch = 0; /* 0 = fill each POA batch */
    bool deep_windows = false;         /* the second tier of POA batches (above); off: racon's limits only */
    bool export_layers = false;        /* hand back the windows left unpolished (OverlapPolishOutput::exported) */
    int32_t deep_max_sequence_size = 0;     /* tier-2 cap on a window's longest sequence; 0 = 16380 (the engine's) */
    int32_t deep_max_sequences_per_poa = 0; /* tier-2 cap on a window's sequences; 0 = 65535 (16-bit coverage) */
};

/* Windows handed back, in the host window arena's layout (window_arena.hpp, racon_gpu_b200/windows.py): per window its
 * backbone (the contig's bases, weights quality - 33, or 0 for a FASTA contig's '!' dummy quality; span (0, 0)), then
 * its layers in racon's add order.  window_ids[i]: the window's index in the outputs (contig by contig). */
struct OverlapExport {
    std::vector<int64_t> window_ids;
    std::vector<int64_t> win_seq_off{0}, seq_off{0};
    std::vector<uint8_t> bases, has_weights;
    std::vector<int8_t> weights;
    std::vector<int32_t> begins, ends;
};

/* Columnar inputs.  Contig c: t_bases[t_off[c] .. t_off[c + 1]), its qualities at the same offsets of t_qual (NULL:
 * FASTA contigs, racon's '!' dummy quality).  Overlap k (racon's order, after its filtering): contig t_id[k], contig
 * segment [t_begin[k], t_end[k]), the strand-adjusted read segment q_bases[q_off[k] .. q_off[k + 1]) starting at
 * q_first[k] in the strand-adjusted read, its qualities at the same offsets of q_qual where has_quality[k] != 0
 * (reverse_quality() for '-' overlaps). */
struct OverlapInput {
    int64_t n_contigs;
    const uint8_t* t_bases;
    const int64_t* t_off;
    const uint8_t* t_qual;
    int64_t n_overlaps;
    const int32_t* t_id;
    const int32_t* t_begin;
    const int32_t* t_end;
    const uint8_t* q_bases;
    const int64_t* q_off;
    const uint8_t* q_qual;
    const uint8_t* has_quality;
    const int32_t* q_first;
};

/* Per window of every contig (racon's window order: contig by contig, id_to_first_window_id): the same outputs as
 * b200poa_polisher_polish -- cons_out rows of `stride` bytes, cons_len, polished (false: the backbone, for racon's CPU
 * path), status. */
struct OverlapPolishOutput {
    uint8_t* cons_out;
    int32_t stride;
    int32_t* cons_len;
    uint8_t* polished;
    int32_t* status;
    int64_t n_rounds = 0;                 /* units */
    int64_t h2d_bytes = 0, d2h_bytes = 0; /* aligner and POA batches together */
    int64_t unfit_contig = -1;            /* a contig whose overlaps do not fit one aligner batch */
    int64_t tier2_windows = 0;            /* windows given to the second tier */
    int64_t tier2_polished = 0;           /* of them: polished there */
    int64_t tier2_batches = 0;            /* second-tier batches created (the first, and each re-creation) */
    int64_t exported_windows = 0;         /* windows appended to *exported */
    int64_t exported_bytes = 0;           /* bytes their export moved device -> host (bases and weights) */
    OverlapExport* exported = nullptr;    /* with export_layers: where the exported windows are appended */
    int64_t split_contigs = 0;            /* contigs polished in more than one unit */
    int64_t repeat_overlaps = 0;          /* alignments done more than once because of the splits */
};

/* The number of windows of the input (sum over contigs of ceil(length / window_length)). */
int64_t overlap_window_count(const OverlapInput& in, int32_t window_length);

/* On opt.device, in units of whole contigs.  Returns a b200poa status: B200POA_SUCCESS, B200POA_INVALID_ARGUMENT,
 * B200POA_CUDA_ERROR, or B200POA_GENERIC_ERROR with out.unfit_contig set when a contig's overlaps do not fit one aligner
 * batch. */
int32_t polish_overlaps(const OverlapInput& in, const OverlapPolishOptions& opt, OverlapPolishOutput& out);

/* On one worker per entry of `devices` (empty: every visible device; opt.device is not used), a contig too large for
 * one aligner batch split at window boundaries.  With aligner_mem 0 every unit is planned for the smallest worker's
 * share.  B200POA_INVALID_ARGUMENT for a device id out of range, before anything is allocated; B200POA_GENERIC_ERROR
 * with out.unfit_contig set when the overlaps of one window alone do not fit one aligner batch. */
int32_t polish_overlaps(const OverlapInput& in, const OverlapPolishOptions& opt, const std::vector<int32_t>& devices,
                        OverlapPolishOutput& out);

} // namespace racon_b200
