/* cuda_polisher.cpp -- see cuda_polisher.hpp and include/b200poa.h (b200poa_polish_windows). */
#include "cuda_polisher.hpp"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <new>
#include <stdexcept>
#include <chrono>
#include <cstdlib>
#include <string>
#include <thread>

#include "../cuda_buffers.hpp"
#include "b200poa.h"
#include "cuda_batch.hpp"
#include "window_arena.hpp"

namespace racon_b200 {

static std::vector<int32_t> resolve_devices(const std::vector<int32_t>& want) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n < 1)
        throw std::runtime_error("[racon_b200] no CUDA device visible (this engine has no CPU fallback)");
    std::vector<int32_t> d = want;
    if (d.empty())
        for (int i = 0; i < n; ++i) d.push_back(i);
    for (int32_t x : d)
        if (x < 0 || x >= n) throw std::invalid_argument("[racon_b200] invalid device id");
    return d;
}

static size_t batch_memory(int32_t device, uint32_t batches, size_t requested) {
    if (requested) return requested;
    size_t free_b = 0, total = 0;
    b200buf::DeviceGuard guard(device);
    cudaMemGetInfo(&free_b, &total);
    return static_cast<size_t>(0.9 * static_cast<double>(free_b) / batches); /* cudapolisher.cpp:233-236 */
}

std::vector<bool> polish_windows(std::vector<std::shared_ptr<Window>>& windows, const PolishOptions& opt) {
    const std::vector<int32_t> devices = resolve_devices(opt.devices);
    const uint32_t nb = std::max<uint32_t>(opt.cudapoa_batches, 1);
    std::vector<std::unique_ptr<CUDABatchProcessor>> processors;
    for (int32_t dev : devices) {
        const size_t mem = batch_memory(dev, nb, opt.mem_per_batch);
        for (uint32_t b = 0; b < nb; ++b)
            processors.emplace_back(createCUDABatch(opt.max_depth_per_window, static_cast<uint32_t>(dev), mem, opt.gap,
                                                    opt.mismatch, opt.match, opt.cuda_banded_alignment, opt.trim));
    }
    std::vector<bool> status(windows.size(), false);
    std::mutex mutex_windows;
    uint32_t next_window_index = 0;

    /* cudapolisher.cpp:254-276 */
    auto fill_next_batch = [&](CUDABatchProcessor* batch) -> std::pair<uint32_t, uint32_t> {
        batch->reset();
        std::lock_guard<std::mutex> guard(mutex_windows);
        const uint32_t initial_count = next_window_index;
        const uint32_t count = static_cast<uint32_t>(windows.size());
        while (next_window_index < count) {
            if (opt.max_windows_per_round && next_window_index - initial_count >= opt.max_windows_per_round) break;
            if (batch->addWindow(windows.at(next_window_index))) next_window_index++;
            else break;
        }
        return {initial_count, next_window_index};
    };
    /* cudapolisher.cpp:286-333 */
    auto process_batch = [&](CUDABatchProcessor* batch) {
        while (true) {
            const std::pair<uint32_t, uint32_t> range = fill_next_batch(batch);
            if (!batch->hasWindows()) break;
            const std::vector<bool>& results = batch->generateConsensus();
            if (results.size() != (range.second - range.first))
                throw std::runtime_error("Windows processed doesn't match range of windows passed to batch");
            std::lock_guard<std::mutex> guard(mutex_windows);
            for (uint32_t i = 0; i < results.size(); i++) status.at(range.first + i) = results.at(i);
        }
    };
    std::vector<std::thread> threads; /* cudapolisher.cpp:336-350 (thread_pool_->submit per processor) */
    std::vector<std::string> errors(processors.size());
    for (size_t t = 0; t < processors.size(); ++t)
        threads.emplace_back([&, t]() {
            try {
                process_batch(processors[t].get());
            } catch (const std::exception& e) {
                errors[t] = e.what();
            }
        });
    for (auto& t : threads) t.join();
    for (const auto& e : errors)
        if (!e.empty()) throw std::runtime_error(e);
    return status;
}

} // namespace racon_b200

/* ------------------------------------------------------------------------------------------------
 * Columnar entry point: the same scheduler over a flat window arena, without materialising
 * racon_b200::Window objects.  Each batch thread claims a chunk of windows under the mutex, packs it
 * into its pinned staging OUTSIDE the mutex, runs the batch and writes trimmed results.
 * ---------------------------------------------------------------------------------------------- */
namespace {

struct FlatProc {
    int32_t device = 0;
    cudaStream_t stream = nullptr;
    b200poa_batch* batch = nullptr;
};

} // namespace

struct b200poa_polisher {
    std::vector<FlatProc> procs;
    int32_t banded = 0;
    int32_t accept_truncated = 0;
    int32_t max_sequences_per_poa = 200;
};

extern "C" void b200poa_polisher_destroy(b200poa_polisher* h) {
    if (!h) return;
    for (auto& p : h->procs) {
        cudaSetDevice(p.device);
        if (p.batch) b200poa_batch_destroy(p.batch);
        if (p.stream) cudaStreamDestroy(p.stream);
    }
    delete h;
}

extern "C" int32_t b200poa_polisher_create_ex(const b200poa_polisher_options* opt, b200poa_polisher** out) {
    using namespace racon_b200;
    if (!out || !opt) return B200POA_INVALID_ARGUMENT;
    *out = nullptr;
    std::vector<int32_t> devices;
    try {
        std::vector<int32_t> want;
        for (int32_t i = 0; i < opt->n_devices; ++i) want.push_back(opt->device_ids[i]);
        devices = resolve_devices(want);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "%s\n", e.what());
        return B200POA_CUDA_ERROR;
    }
    const uint32_t nb = static_cast<uint32_t>(std::max(opt->batches_per_device, 1));
    b200poa_polisher* h = new b200poa_polisher();
    h->banded = opt->banded;
    h->accept_truncated = opt->accept_truncated;
    int32_t rc = B200POA_SUCCESS;
    b200poa_config cfg; /* cudabatch.cpp:56-59: BatchConfig(1023, max_depth 200, 256, band mode) unless overridden */
    b200poa_config_default(&cfg, opt->max_sequence_size > 0 ? opt->max_sequence_size : 1023,
                           opt->max_sequences_per_poa > 0 ? opt->max_sequences_per_poa : 200,
                           opt->band_width > 0 ? opt->band_width : 256,
                           opt->banded == 2 ? B200POA_ADAPTIVE_BAND : opt->banded ? B200POA_STATIC_BAND : B200POA_FULL_BAND);
    h->max_sequences_per_poa = cfg.max_sequences_per_poa;
    for (int32_t dev : devices) {
        const size_t mem = batch_memory(dev, nb, opt->mem_per_batch);
        for (uint32_t k = 0; k < nb && rc == B200POA_SUCCESS; ++k) {
            FlatProc p;
            p.device = dev;
            cudaSetDevice(dev);
            if (cudaStreamCreate(&p.stream) != cudaSuccess) rc = B200POA_CUDA_ERROR;
            else rc = b200poa_batch_create(dev, p.stream, mem, B200POA_OUTPUT_CONSENSUS, &cfg, static_cast<int16_t>(opt->gap),
                                           static_cast<int16_t>(opt->mismatch), static_cast<int16_t>(opt->match), &p.batch);
            if (rc == B200POA_SUCCESS) {
                /* the polisher only needs the trimmed consensus: the trim span comes from the device, the coverage stays there */
                b200poa_batch_set_option(p.batch, B200POA_OPT_DOWNLOAD_COVERAGE, 0);
                b200poa_batch_set_option(p.batch, B200POA_OPT_TRIM_COUNTS_STAGED, opt->accept_truncated ? 1 : 0);
            }
            h->procs.push_back(p);
        }
    }
    if (rc != B200POA_SUCCESS) {
        b200poa_polisher_destroy(h);
        return rc;
    }
    *out = h;
    return B200POA_SUCCESS;
}

extern "C" int32_t b200poa_polisher_create(int32_t n_devices, const int32_t* device_ids, int32_t batches_per_device,
                                           size_t mem_per_batch, int32_t banded, int32_t match, int32_t mismatch,
                                           int32_t gap, b200poa_polisher** out) {
    b200poa_polisher_options opt;
    std::memset(&opt, 0, sizeof(opt));
    opt.n_devices = n_devices;
    opt.device_ids = device_ids;
    opt.batches_per_device = batches_per_device;
    opt.mem_per_batch = mem_per_batch;
    opt.banded = banded;
    opt.match = match;
    opt.mismatch = mismatch;
    opt.gap = gap;
    return b200poa_polisher_create_ex(&opt, out);
}

/* pinned_weight_mode != nullptr: the arrays are a page-locked arena (b200poa_arena_finalize) -> zero-staging batches */
static int32_t polisher_polish_impl(b200poa_polisher* h, int64_t n_windows, const int64_t* win_seq_off,
                                    const int64_t* seq_off, const uint8_t* bases, const int8_t* weights,
                                    const uint8_t* has_weights, const int64_t* pinned_weight_mode, const int32_t* begins,
                                    const int32_t* ends, int32_t tgs, int32_t trim, int32_t max_windows_per_round,
                                    uint8_t* cons_out, int32_t stride, int32_t* cons_len, uint8_t* polished,
                                    int32_t* status_out, int64_t* kernel_launches, int64_t* h2d_bytes, int64_t* d2h_bytes) {
    if (!h || n_windows < 0 || !win_seq_off || !seq_off || !cons_out || !cons_len || !polished) return B200POA_INVALID_ARGUMENT;
    std::vector<FlatProc>& procs = h->procs;
    std::mutex mu;
    int64_t cursor = 0;
    int64_t launches = 0, up_bytes = 0, down_bytes = 0;
    const int64_t chunk = max_windows_per_round > 0
                              ? max_windows_per_round
                              : std::max<int64_t>(256, (n_windows + (int64_t)procs.size() * 4 - 1) / ((int64_t)procs.size() * 4));
    const int64_t n_procs = static_cast<int64_t>(procs.size());
    auto worker = [&](FlatProc* p, int64_t index) -> int32_t {
        cudaSetDevice(p->device);
        int64_t lo = 0, hi = 0; /* claimed but not yet processed windows */
        std::vector<int32_t> seqs_added;
        /* The processors share the GPU: while one of them downloads, trims and stages, the kernels of the others
         * must keep it full.  Their first rounds are therefore of different sizes (1/P, 2/P, ... of a round), which
         * starts the first kernel early and keeps the processors out of step from then on. */
        bool first_claim = true;
        const bool timers = std::getenv("B200POA_E2E_TIMERS") != nullptr; /* diagnostics: where a round's wall time goes */
        double t_stage = 0, t_gpu = 0, t_post = 0;
        int rounds = 0;
        auto now = []() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
        const double t_begin = now();
        for (;;) {
            if (lo == hi) {
                std::lock_guard<std::mutex> g(mu);
                const int64_t want = first_claim ? std::max<int64_t>(1, chunk * (index + 1) / n_procs) : chunk;
                first_claim = false;
                lo = cursor;
                hi = std::min<int64_t>(n_windows, lo + want);
                cursor = hi;
            }
            if (lo == hi) {
                if (timers)
                    std::fprintf(stderr, "[b200poa e2e] proc %lld: %d rounds, stage %.1f ms, upload+kernel+download %.1f ms, trim/copy-out %.1f ms, total %.1f ms\n",
                                 (long long)index, rounds, 1e3 * t_stage, 1e3 * t_gpu, 1e3 * t_post, 1e3 * (now() - t_begin));
                return B200POA_SUCCESS;
            }
            const double t0 = now();
            b200poa_batch_reset(p->batch);
            int64_t first = lo, n_added = 0;
            seqs_added.resize(static_cast<size_t>(hi - lo));
            /* stage [lo, hi) but stop at the first window that does not fit */
            int32_t st = pinned_weight_mode
                             ? b200poa_batch_add_windows_pinned(p->batch, hi, first, win_seq_off, seq_off, bases, weights,
                                                                has_weights, pinned_weight_mode, begins, ends, &n_added,
                                                                seqs_added.data())
                             : b200poa_batch_add_windows(p->batch, hi, first, win_seq_off, seq_off, bases, weights, has_weights,
                                                         begins, ends, &n_added, seqs_added.data());
            if (st != B200POA_SUCCESS) return st;
            if (n_added == 0) return B200POA_EXCEEDED_MAXIMUM_POAS; /* a single window larger than the batch */
            const double t1 = now();
            st = b200poa_batch_generate(p->batch);
            if (st != B200POA_SUCCESS) return st;
            const uint8_t* c; const int32_t* l; const int32_t* s; const int32_t* off; const int32_t* tr;
            st = b200poa_batch_get_consensus(p->batch, &c, nullptr, &l, &s, &off, &tr);
            if (st != B200POA_SUCCESS) return st;
            const double t2 = now();
            b200poa_batch_info info;
            b200poa_batch_get_info(p->batch, &info);
            for (int64_t i = 0; i < n_added; ++i) {
                const int64_t w = first + i;
                const int64_t nseq = win_seq_off[w + 1] - win_seq_off[w];
                uint8_t* dst = cons_out + static_cast<size_t>(w) * static_cast<size_t>(stride);
                if (status_out) status_out[w] = s[i];
                const bool dropped = seqs_added[static_cast<size_t>(i)] != nseq - 1; /* layers cut by the batch limits */
                if (nseq < 3 || s[i] != B200POA_SUCCESS || (dropped && !h->accept_truncated)) {
                    /* window.cpp:68-71 (< 3 sequences), a kernel status, or -- unless the caller accepts the reference
                     * GPU adapter's depth truncation (cudabatch.cpp:134-153) -- dropped layers: the window comes back
                     * as its backbone with polished = 0, never as a hole; the caller's CPU path may still polish it */
                    const int64_t a = seq_off[win_seq_off[w]], b = seq_off[win_seq_off[w] + 1];
                    std::memcpy(dst, bases + a, static_cast<size_t>(std::min<int64_t>(b - a, stride)));
                    cons_len[w] = static_cast<int32_t>(b - a);
                    polished[w] = 0;
                    if (status_out && s[i] == B200POA_SUCCESS && nseq >= 3)
                        status_out[w] = nseq - 1 > h->max_sequences_per_poa ? B200POA_EXCEEDED_MAXIMUM_SEQUENCES_PER_POA
                                                                             : B200POA_EXCEEDED_MAXIMUM_SEQUENCE_SIZE;
                    continue;
                }
                int32_t begin = 0, end = l[i] - 1;
                if (tgs && trim) { /* window.cpp:118-139, evaluated on the device (WindowOut::trim) */
                    const int32_t tb = tr[i] & 0xFFFF, te = tr[i] >> 16;
                    if (tb < te) {
                        begin = tb;
                        end = te;
                    }
                }
                const int32_t n = end - begin + 1;
                std::memcpy(dst, c + off[i] + begin, static_cast<size_t>(std::min(n, stride)));
                cons_len[w] = n;
                polished[w] = 1;
            }
            {
                std::lock_guard<std::mutex> g(mu);
                launches += 1;
                up_bytes += info.h2d_bytes;
                down_bytes += info.d2h_bytes;
            }
            lo = first + n_added;
            t_stage += t1 - t0;
            t_gpu += t2 - t1;
            t_post += now() - t2;
            ++rounds;
        }
    };
    std::vector<int32_t> results(procs.size(), B200POA_SUCCESS);
    std::vector<std::thread> th;
    for (size_t t = 0; t < procs.size(); ++t) th.emplace_back([&, t]() { results[t] = worker(&procs[t], (int64_t)t); });
    for (auto& t : th) t.join();
    int32_t rc = B200POA_SUCCESS;
    for (int32_t r : results)
        if (r != B200POA_SUCCESS) rc = r;
    if (kernel_launches) *kernel_launches = launches;
    if (h2d_bytes) *h2d_bytes = up_bytes;
    if (d2h_bytes) *d2h_bytes = down_bytes;
    return rc;
}

extern "C" int32_t b200poa_polisher_polish(b200poa_polisher* h, int64_t n_windows, const int64_t* win_seq_off,
                                           const int64_t* seq_off, const uint8_t* bases, const int8_t* weights,
                                           const uint8_t* has_weights, const int32_t* begins, const int32_t* ends,
                                           int32_t tgs, int32_t trim, int32_t max_windows_per_round, uint8_t* cons_out,
                                           int32_t stride, int32_t* cons_len, uint8_t* polished, int32_t* status_out,
                                           int64_t* kernel_launches, int64_t* h2d_bytes, int64_t* d2h_bytes) {
    return polisher_polish_impl(h, n_windows, win_seq_off, seq_off, bases, weights, has_weights, nullptr, begins, ends, tgs,
                                trim, max_windows_per_round, cons_out, stride, cons_len, polished, status_out,
                                kernel_launches, h2d_bytes, d2h_bytes);
}

extern "C" int32_t b200poa_polish_windows(int64_t n_windows, const int64_t* win_seq_off, const int64_t* seq_off,
                                          const uint8_t* bases, const int8_t* weights, const uint8_t* has_weights,
                                          const int32_t* begins, const int32_t* ends, int32_t tgs, int32_t trim,
                                          int32_t match, int32_t mismatch, int32_t gap, int32_t banded,
                                          int32_t n_devices, const int32_t* device_ids, int32_t batches_per_device,
                                          size_t mem_per_batch, int32_t max_windows_per_round, uint8_t* cons_out,
                                          int32_t stride, int32_t* cons_len, uint8_t* polished, int32_t* status_out,
                                          int64_t* kernel_launches) {
    b200poa_polisher* h = nullptr;
    int32_t rc = b200poa_polisher_create(n_devices, device_ids, batches_per_device, mem_per_batch, banded, match, mismatch, gap, &h);
    if (rc != B200POA_SUCCESS) return rc;
    rc = b200poa_polisher_polish(h, n_windows, win_seq_off, seq_off, bases, weights, has_weights, begins, ends, tgs, trim,
                                 max_windows_per_round, cons_out, stride, cons_len, polished, status_out, kernel_launches,
                                 nullptr, nullptr);
    b200poa_polisher_destroy(h);
    return rc;
}

/* ------------------------------------------------------------------------------------------------
 * Same job through the class API a racon maintainer would use: racon_b200::createWindow / add_layer
 * (== racon::createWindow / Window::add_layer), then polish_windows (== CUDAPolisher::polish's GPU
 * section) driving racon_b200::CUDABatchProcessor::addWindow / generateConsensus.  Qualities are
 * passed as PHRED+33 strings exactly as racon holds them (polisher.cpp:392-395, 430-441).
 * ---------------------------------------------------------------------------------------------- */
extern "C" int32_t b200poa_polish_windows_via_adapter(int64_t n_windows, const int64_t* win_seq_off,
                                                      const int64_t* seq_off, const uint8_t* bases,
                                                      const int8_t* weights, const uint8_t* has_weights,
                                                      const int32_t* begins, const int32_t* ends, int32_t tgs,
                                                      int32_t trim, int32_t match, int32_t mismatch, int32_t gap,
                                                      int32_t banded, int32_t n_devices, const int32_t* device_ids,
                                                      int32_t batches_per_device, size_t mem_per_batch,
                                                      int32_t max_windows_per_round, uint8_t* cons_out, int32_t stride,
                                                      int32_t* cons_len, uint8_t* polished) {
    using namespace racon_b200;
    try {
        const int64_t n_bases = seq_off[win_seq_off[n_windows]];
        std::string quality(static_cast<size_t>(n_bases), '!');
        for (int64_t i = 0; i < n_bases; ++i) quality[static_cast<size_t>(i)] = static_cast<char>(weights[i] + 33);
        std::vector<std::shared_ptr<Window>> windows;
        windows.reserve(static_cast<size_t>(n_windows));
        for (int64_t w = 0; w < n_windows; ++w) {
            const int64_t s0 = win_seq_off[w], s1 = win_seq_off[w + 1];
            const uint32_t bl = static_cast<uint32_t>(seq_off[s0 + 1] - seq_off[s0]);
            auto win = createWindow(static_cast<uint64_t>(w), 0, tgs ? WindowType::kTGS : WindowType::kNGS,
                                    reinterpret_cast<const char*>(bases + seq_off[s0]), bl, quality.data() + seq_off[s0], bl);
            if (!win) return B200POA_INVALID_ARGUMENT;
            for (int64_t s = s0 + 1; s < s1; ++s) {
                const uint32_t len = static_cast<uint32_t>(seq_off[s + 1] - seq_off[s]);
                if (!win->add_layer(reinterpret_cast<const char*>(bases + seq_off[s]), len,
                                    has_weights[s] ? quality.data() + seq_off[s] : nullptr, has_weights[s] ? len : 0,
                                    static_cast<uint32_t>(begins[s]), static_cast<uint32_t>(ends[s])))
                    return B200POA_INVALID_ARGUMENT;
            }
            windows.push_back(win);
        }
        PolishOptions opt;
        for (int32_t i = 0; i < n_devices; ++i) opt.devices.push_back(device_ids[i]);
        opt.cudapoa_batches = static_cast<uint32_t>(std::max(batches_per_device, 1));
        opt.cuda_banded_alignment = banded != 0;
        opt.match = static_cast<int8_t>(match);
        opt.mismatch = static_cast<int8_t>(mismatch);
        opt.gap = static_cast<int8_t>(gap);
        opt.trim = trim != 0;
        opt.mem_per_batch = mem_per_batch;
        opt.max_windows_per_round = static_cast<uint32_t>(std::max(max_windows_per_round, 0));
        const std::vector<bool> st = polish_windows(windows, opt);
        for (int64_t w = 0; w < n_windows; ++w) {
            const std::string& c = windows[static_cast<size_t>(w)]->consensus();
            std::memcpy(cons_out + static_cast<size_t>(w) * static_cast<size_t>(stride), c.data(),
                        std::min<size_t>(c.size(), static_cast<size_t>(stride)));
            cons_len[w] = static_cast<int32_t>(c.size());
            polished[w] = st[static_cast<size_t>(w)] ? 1 : 0;
        }
    } catch (const std::invalid_argument& e) {
        std::fprintf(stderr, "[b200poa] %s\n", e.what());
        return B200POA_INVALID_ARGUMENT;
    } catch (const std::exception& e) {
        std::fprintf(stderr, "[b200poa] %s\n", e.what());
        return B200POA_GENERIC_ERROR;
    }
    return B200POA_SUCCESS;
}


/* ---- columnar window construction: C ABI over racon_b200::WindowArena (window_arena.hpp) ---- */
struct b200poa_arena {
    racon_b200::WindowArena arena;
    std::vector<int64_t> weight_mode; /* per sequence, b200poa_weight_modes */
    std::vector<std::string> quality_store; /* b200poa_arena_append_columns: quality strings kept alive until finalize */
    bool pinned = false;              /* bases/weights are page-locked (cudaHostRegister) */
};

extern "C" b200poa_arena* b200poa_arena_create(void) { return new (std::nothrow) b200poa_arena(); }

extern "C" int64_t b200poa_arena_add_window(b200poa_arena* a, const char* backbone, uint32_t backbone_length,
                                            const char* quality, uint32_t quality_length) {
    if (!a || !backbone || !quality) return -1; /* racon always gives the backbone a quality ('!' for FASTA targets) */
    return a->arena.add_window(backbone, backbone_length, quality, quality_length);
}

extern "C" int32_t b200poa_arena_add_layer(b200poa_arena* a, int64_t window, const char* sequence,
                                           uint32_t sequence_length, const char* quality, uint32_t quality_length,
                                           uint32_t begin, uint32_t end) {
    if (!a || (!sequence && sequence_length != 0)) return B200POA_INVALID_ARGUMENT;
    return a->arena.add_layer(window, sequence, sequence_length, quality, quality_length, begin, end)
               ? B200POA_SUCCESS
               : B200POA_INVALID_ARGUMENT;
}

/* Convenience for callers that already hold their windows as columns (tests, bench): the same add_window / add_layer
 * calls as above, one per sequence, qualities rebuilt as PHRED+33 characters from the weights. */
extern "C" int32_t b200poa_arena_append_columns(b200poa_arena* a, int64_t n_windows, const int64_t* win_seq_off,
                                                const int64_t* seq_off, const uint8_t* bases, const int8_t* weights,
                                                const uint8_t* has_weights, const int32_t* begins, const int32_t* ends) {
    if (!a || a->arena.finalized()) return B200POA_INVALID_ARGUMENT;
    a->quality_store.emplace_back();
    std::string& q = a->quality_store.back(); /* add_* borrow the pointers until finalize */
    q.resize(static_cast<size_t>(seq_off[win_seq_off[n_windows]]));
    for (size_t i = 0; i < q.size(); ++i) q[i] = static_cast<char>(weights[i] + 33);
    for (int64_t w = 0; w < n_windows; ++w) {
        const int64_t s0 = win_seq_off[w], s1 = win_seq_off[w + 1];
        const uint32_t bl = static_cast<uint32_t>(seq_off[s0 + 1] - seq_off[s0]);
        const int64_t id = a->arena.add_window(reinterpret_cast<const char*>(bases + seq_off[s0]), bl, q.data() + seq_off[s0], bl);
        if (id < 0) return B200POA_INVALID_ARGUMENT;
        for (int64_t s = s0 + 1; s < s1; ++s) {
            const uint32_t len = static_cast<uint32_t>(seq_off[s + 1] - seq_off[s]);
            if (!a->arena.add_layer(id, reinterpret_cast<const char*>(bases + seq_off[s]), len,
                                    has_weights[s] ? q.data() + seq_off[s] : nullptr, has_weights[s] ? len : 0,
                                    static_cast<uint32_t>(begins[s]), static_cast<uint32_t>(ends[s])))
                return B200POA_INVALID_ARGUMENT;
        }
    }
    return B200POA_SUCCESS;
}

extern "C" int32_t b200poa_arena_finalize(b200poa_arena* a) {
    if (!a) return B200POA_INVALID_ARGUMENT;
    if (a->arena.finalized()) return B200POA_SUCCESS;
    a->arena.finalize();
    a->quality_store.clear();
    const racon_b200::WindowArena& w = a->arena;
    a->weight_mode.assign(static_cast<size_t>(w.n_sequences()), 0);
    b200poa_weight_modes(w.n_sequences(), w.seq_off().data(), w.weights().data(), w.has_weights().data(), a->weight_mode.data());
    /* page-lock the arena where a CUDA device exists: batches then upload straight from it.  Without a device (or if
     * the driver refuses) the arena stays pageable and polishing goes through the staging copy. */
    int ndev = 0;
    if (!w.bases().empty() && cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0) {
        const bool ok_b = cudaHostRegister(const_cast<uint8_t*>(w.bases().data()), w.bases().size(), cudaHostRegisterPortable) == cudaSuccess;
        const bool ok_w = ok_b && cudaHostRegister(const_cast<int8_t*>(w.weights().data()), w.weights().size(), cudaHostRegisterPortable) == cudaSuccess;
        if (ok_b && !ok_w) cudaHostUnregister(const_cast<uint8_t*>(w.bases().data()));
        a->pinned = ok_b && ok_w;
        if (!a->pinned) cudaGetLastError(); /* not an error of the caller's */
    } else {
        cudaGetLastError();
    }
    return B200POA_SUCCESS;
}

extern "C" int32_t b200poa_arena_view(const b200poa_arena* a, int64_t* n_windows, int64_t* n_sequences,
                                      const int64_t** win_seq_off, const int64_t** seq_off, const uint8_t** bases,
                                      const int8_t** weights, const uint8_t** has_weights, const int32_t** begins,
                                      const int32_t** ends) {
    if (!a || !a->arena.finalized()) return B200POA_INVALID_ARGUMENT;
    const racon_b200::WindowArena& w = a->arena;
    if (n_windows) *n_windows = w.n_windows();
    if (n_sequences) *n_sequences = w.n_sequences();
    if (win_seq_off) *win_seq_off = w.win_seq_off().data();
    if (seq_off) *seq_off = w.seq_off().data();
    if (bases) *bases = w.bases().data();
    if (weights) *weights = w.weights().data();
    if (has_weights) *has_weights = w.has_weights().data();
    if (begins) *begins = w.begins().data();
    if (ends) *ends = w.ends().data();
    return B200POA_SUCCESS;
}

extern "C" int32_t b200poa_polisher_polish_arena(b200poa_polisher* h, const b200poa_arena* a, int32_t tgs, int32_t trim,
                                                 int32_t max_windows_per_round, uint8_t* cons_out, int32_t stride,
                                                 int32_t* cons_len, uint8_t* polished, int32_t* status_out,
                                                 int64_t* kernel_launches, int64_t* h2d_bytes, int64_t* d2h_bytes) {
    if (!a || !a->arena.finalized()) return B200POA_INVALID_ARGUMENT;
    const racon_b200::WindowArena& w = a->arena;
    return polisher_polish_impl(h, w.n_windows(), w.win_seq_off().data(), w.seq_off().data(), w.bases().data(),
                                w.weights().data(), w.has_weights().data(), a->pinned ? a->weight_mode.data() : nullptr,
                                w.begins().data(), w.ends().data(), tgs, trim, max_windows_per_round, cons_out, stride,
                                cons_len, polished, status_out, kernel_launches, h2d_bytes, d2h_bytes);
}

extern "C" void b200poa_arena_destroy(b200poa_arena* a) {
    if (a && a->pinned) {
        cudaHostUnregister(const_cast<uint8_t*>(a->arena.bases().data()));
        cudaHostUnregister(const_cast<int8_t*>(a->arena.weights().data()));
    }
    delete a;
}

extern "C" int64_t b200poa_compact_rows(const uint8_t* rows, int64_t n_rows, int64_t stride, const int32_t* lens,
                                        uint8_t* flat, int64_t* offsets) {
    int64_t o = 0;
    for (int64_t i = 0; i < n_rows; ++i) {
        if (offsets) offsets[i] = o;
        const int64_t n = std::min<int64_t>(lens[i], stride);
        std::memcpy(flat + o, rows + i * stride, static_cast<size_t>(n));
        o += n;
    }
    if (offsets) offsets[n_rows] = o;
    return o;
}
