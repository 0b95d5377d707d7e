/* cuda_batch.cpp -- see cuda_batch.hpp.  Mirrors src/cuda/cudabatch.cpp. */
#include "cuda_batch.hpp"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <stdexcept>
#include <string>

#include "../cuda_buffers.hpp"

namespace racon_b200 {

using namespace b200poa_cpp;

std::atomic<uint32_t> CUDABatchProcessor::batches;

std::unique_ptr<CUDABatchProcessor> createCUDABatch(uint32_t max_window_depth, uint32_t device, size_t avail_mem,
                                                    int8_t gap, int8_t mismatch, int8_t match,
                                                    bool cuda_banded_alignment, bool trim) {
    return std::unique_ptr<CUDABatchProcessor>(new CUDABatchProcessor(max_window_depth, device, avail_mem, gap,
                                                                      mismatch, match, cuda_banded_alignment, trim));
}

CUDABatchProcessor::CUDABatchProcessor(uint32_t max_window_depth, uint32_t device, size_t avail_mem, int8_t gap,
                                       int8_t mismatch, int8_t match, bool cuda_banded_alignment, bool trim)
    : device_(device), trim_(trim) {
    bid_ = CUDABatchProcessor::batches++;
    b200buf::DeviceGuard guard(static_cast<int>(device));
    cudaStream_t s = nullptr;
    if (cudaStreamCreate(&s) != cudaSuccess) /* cudabatch.cpp:54 */
        throw std::runtime_error("[racon_b200::CUDABatchProcessor] cudaStreamCreate failed");
    stream_ = s;
    /* cudabatch.cpp:56-68 */
    BatchConfig batch_config(1023, static_cast<int32_t>(max_window_depth), 256,
                             cuda_banded_alignment ? BandMode::static_band : BandMode::full_band);
    cudapoa_batch_ = create_batch(static_cast<int32_t>(device), stream_, avail_mem, OutputType::consensus,
                                  batch_config, gap, mismatch, match);
}

CUDABatchProcessor::~CUDABatchProcessor() {
    cudapoa_batch_.reset();
    b200buf::DeviceGuard guard(static_cast<int>(device_));
    cudaStreamDestroy(static_cast<cudaStream_t>(stream_)); /* cudabatch.cpp:74 */
}

void CUDABatchProcessor::convertPhredQualityToWeights(const char* qual, uint32_t qual_length,
                                                      std::vector<int8_t>& weights) {
    weights.clear(); /* cudabatch.cpp:182-191 */
    for (uint32_t i = 0; i < qual_length; i++) weights.push_back(static_cast<uint8_t>(qual[i]) - 33);
}

bool CUDABatchProcessor::addWindow(std::shared_ptr<Window> window) {
    const uint32_t num_seqs = static_cast<uint32_t>(window->sequences_.size());
    if (num_seqs < 3) { /* window.cpp:68-71 / cudabatch.cpp:218-227: backbone, status false; never staged */
        windows_.push_back(window);
        staged_index_.push_back(-1);
        seqs_added_per_window_.push_back(0);
        dropped_layers_.push_back(false);
        return true;
    }
    Group poa_group;
    std::vector<std::vector<int8_t>> all_read_weights(num_seqs, std::vector<int8_t>());

    /* cudabatch.cpp:96-104: processing order = the same std::sort call as window.cpp:78-85 */
    std::vector<uint32_t> rank;
    rank.reserve(num_seqs);
    for (uint32_t i = 0; i < num_seqs; ++i) rank.emplace_back(i);
    std::sort(rank.begin() + 1, rank.end(), [&](uint32_t lhs, uint32_t rhs) {
        return window->positions_[lhs].first < window->positions_[rhs].first; });

    for (uint32_t j = 0; j < num_seqs; j++) {
        const uint32_t i = rank.at(j);
        const auto& seq = window->sequences_.at(i);
        const auto& qualities = window->qualities_.at(i);
        Entry e;
        e.seq = seq.first;
        e.length = static_cast<int32_t>(seq.second);
        if (qualities.first == nullptr) {
            e.weights = nullptr; /* window.cpp:105-107: no quality => weight 1 */
        } else {
            convertPhredQualityToWeights(qualities.first, qualities.second, all_read_weights[i]);
            e.weights = all_read_weights[i].data();
        }
        e.begin = static_cast<int32_t>(window->positions_[i].first);
        e.end = static_cast<int32_t>(window->positions_[i].second);
        poa_group.push_back(e);
    }

    std::vector<StatusType> entry_status;
    const StatusType status = cudapoa_batch_->add_poa_group(entry_status, poa_group);
    if (status != StatusType::success) return false; /* batch full (cudabatch.cpp:129-132) */
    windows_.push_back(window);
    staged_index_.push_back(staged_++);

    int32_t seq_added = 0;
    bool dropped = false;
    for (uint32_t i = 1; i < entry_status.size(); i++) { /* cudabatch.cpp:134-153 */
        if (entry_status[i] == StatusType::exceeded_maximum_sequence_size ||
            entry_status[i] == StatusType::exceeded_maximum_sequences_per_poa) {
            dropped = true;
            continue;
        } else if (entry_status[i] != StatusType::success) {
            throw std::runtime_error("Could not add sequence to POA in batch " + std::to_string(cudapoa_batch_->batch_id()));
        }
        seq_added++;
    }
    if (!entry_status.empty() && entry_status[0] != StatusType::success) dropped = true;
    seqs_added_per_window_.push_back(static_cast<uint32_t>(seq_added));
    dropped_layers_.push_back(dropped);
    return true;
}

bool CUDABatchProcessor::hasWindows() const { return !windows_.empty(); }

void CUDABatchProcessor::generatePOA() { cudapoa_batch_->generate_poa(); }

void CUDABatchProcessor::getConsensus() {
    std::vector<std::string> consensuses;
    std::vector<std::vector<uint16_t>> coverages;
    std::vector<StatusType> output_status;
    if (staged_ > 0) cudapoa_batch_->get_consensus(consensuses, coverages, output_status);

    for (uint32_t i = 0; i < windows_.size(); i++) {
        auto window = windows_.at(i);
        const int32_t k = staged_index_[i];
        if (k < 0) { /* fewer than 3 sequences: backbone, "failed" (window.cpp:68-71) */
            window->consensus_ = std::string(window->sequences_.front().first, window->sequences_.front().second);
            window_consensus_status_.emplace_back(false);
            continue;
        }
        if (output_status.at(k) != StatusType::success || dropped_layers_[i]) {
            /* left to the caller's CPU polisher (cudabatch.cpp:209-213); until then the window reads as its
             * backbone, so a caller without a CPU path stitches unpolished sequence, never a hole */
            window->consensus_ = std::string(window->sequences_.front().first, window->sequences_.front().second);
            window_consensus_status_.emplace_back(false);
            continue;
        }
        window->consensus_ = consensuses[k];
        if (window->type_ == WindowType::kTGS && trim_) { /* window.cpp:118-139 */
            const uint32_t average_coverage = (static_cast<uint32_t>(window->sequences_.size()) - 1) / 2;
            const std::vector<uint16_t>& cov = coverages[k];
            int32_t begin = 0, end = static_cast<int32_t>(window->consensus_.size()) - 1;
            for (; begin < static_cast<int32_t>(window->consensus_.size()); ++begin)
                if (cov[begin] >= average_coverage) break;
            for (; end >= 0; --end)
                if (cov[end] >= average_coverage) break;
            if (begin >= end) {
                std::fprintf(stderr, "[racon_b200::CUDABatchProcessor] warning: contig %lu might be chimeric in window %u!\n",
                             static_cast<unsigned long>(window->id_), window->rank_);
            } else {
                window->consensus_ = window->consensus_.substr(begin, end - begin + 1);
            }
        }
        window_consensus_status_.emplace_back(true);
    }
}

const std::vector<bool>& CUDABatchProcessor::generateConsensus() {
    if (staged_ > 0) generatePOA();
    getConsensus();
    return window_consensus_status_;
}

void CUDABatchProcessor::reset() {
    windows_.clear();
    staged_index_.clear();
    window_consensus_status_.clear();
    seqs_added_per_window_.clear();
    dropped_layers_.clear();
    staged_ = 0;
    cudapoa_batch_->reset();
}

} // namespace racon_b200
