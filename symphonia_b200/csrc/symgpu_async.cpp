// Asynchronous, thread-safe MP3 entry points: symgpu_mp3_submit / symgpu_mp3_submit_quantized / symgpu_mp3_wait
// (include/symgpu.h, SURVEY.md §8b "proposed exports").
//
// The reference's decoders are one object per stream, one decode() call per packet (codecs/audio.rs:251-298), made by
// the registry (registry.rs:260-269); a server runs hundreds of them on as many threads.  One launch per packet wastes
// the GPU (a kernel sized for every SM, for one frame), so the context gathers what the decoders of all threads have submitted into
// ONE batch: a frame is copied into pinned staging memory under a mutex (submit), and the first thread that waits for a
// ticket of the oldest unfinished batch closes it and runs it for everybody (wait) -- group commit: while that batch is
// on the device the other threads keep submitting into the next one.  Batches run in order, so the frames of a stream are
// synthesised in submission order; a stream appears at most once per batch (a second frame of the same stream closes the
// batch), which is what makes every slot a one-frame run of its stream.
#include <cuda_runtime.h>

#include <condition_variable>
#include <cstring>
#include <deque>
#include <memory>
#include <mutex>
#include <new>
#include <unordered_set>
#include <vector>

#include "ctx.h"

using namespace symgpu;
using namespace symgpu_detail;

namespace {

constexpr uint32_t kBatchCap = 2048; // frames per batch: 2048 x 18.7 KB = 38 MB of pinned staging

enum class BatchState { Open, Running, Done };

struct Batch {
    uint64_t seq = 0;
    BatchState state = BatchState::Open;
    bool closed = false; // no more frames (full, or a stream came back for a second frame)
    symgpu_status status = SYMGPU_OK;
    uint32_t n = 0, collected = 0;
    symgpu_mp3_gc* units = nullptr; // pinned [cap][4]
    float* spectra = nullptr;       // pinned [cap][2304]
    float* pcm = nullptr;           // pinned [cap][2304]
    std::vector<symgpu_mp3_run> runs;
    std::unordered_set<uint32_t> streams;
    ~Batch() {
        if (units) cudaFreeHost(units);
        if (spectra) cudaFreeHost(spectra);
        if (pcm) cudaFreeHost(pcm);
    }
};

} // namespace

struct symgpu_async_mp3 {
    std::mutex m;
    std::condition_variable cv;
    std::deque<std::unique_ptr<Batch>> live; // oldest first; back() is the open batch
    std::vector<std::unique_ptr<Batch>> pool; // collected batches, staging reused
    uint64_t next_seq = 1;
    uint64_t batches_run = 0, frames_run = 0;
};

void symgpu_async_mp3_destroy(symgpu_async_mp3* a) { delete a; }

namespace {

symgpu_async_mp3* state_of(symgpu_ctx* ctx) {
    // created under the context's async mutex by the first submit
    static std::mutex create_m;
    std::lock_guard<std::mutex> g(create_m);
    if (!ctx->async_mp3) ctx->async_mp3 = new (std::nothrow) symgpu_async_mp3();
    return ctx->async_mp3;
}

Batch* open_batch(symgpu_ctx* ctx, symgpu_async_mp3* a) { // a->m held
    if (!a->live.empty() && !a->live.back()->closed && a->live.back()->state == BatchState::Open) return a->live.back().get();
    std::unique_ptr<Batch> b;
    if (!a->pool.empty()) {
        b = std::move(a->pool.back());
        a->pool.pop_back();
    } else {
        b.reset(new (std::nothrow) Batch());
        if (!b) return nullptr;
        DeviceGuard guard(ctx->device);
        if (cudaMallocHost(&b->units, (size_t)kBatchCap * 4 * sizeof(symgpu_mp3_gc)) != cudaSuccess ||
            cudaMallocHost(&b->spectra, (size_t)kBatchCap * SYMGPU_MP3_FRAME_FLOATS * sizeof(float)) != cudaSuccess ||
            cudaMallocHost(&b->pcm, (size_t)kBatchCap * SYMGPU_MP3_FRAME_FLOATS * sizeof(float)) != cudaSuccess)
            return nullptr;
    }
    b->seq = a->next_seq++;
    b->state = BatchState::Open;
    b->closed = false;
    b->status = SYMGPU_OK;
    b->n = b->collected = 0;
    b->runs.clear();
    b->streams.clear();
    a->live.push_back(std::move(b));
    return a->live.back().get();
}

symgpu_status submit_impl(symgpu_ctx* ctx, uint32_t stream, const symgpu_mp3_gc* units, const float* spectra, const int16_t* quant,
                          uint8_t gpf, uint8_t channels, symgpu_ticket* ticket) {
    if (!ctx || !units || (!spectra == !quant) || !ticket) return SYMGPU_ERR_ARG;
    if (stream >= ctx->n_mp3_streams) return SYMGPU_ERR_LIMIT;
    symgpu_mp3_run run{};
    run.stream = stream;
    run.first_frame = 0;
    run.n_frames = 1;
    run.granules_per_frame = gpf;
    run.channels = channels;
    // a malformed frame is refused here, alone: inside a batch it would fail every frame of the launch
    const symgpu_status chk = symgpu_mp3_units_check(units, &run, 1, 1);
    if (chk != SYMGPU_OK) return chk;
    // the Huffman stage's values become +-POW43[|q|] before the lock is taken (read_huffman_samples' table lookup,
    // requantize.rs:128, :144, which the reference does on the CPU as well)
    float expanded[SYMGPU_MP3_FRAME_FLOATS];
    if (quant) {
        const float* pow43 = mp3_tables_host().pow43;
        for (int i = 0; i < SYMGPU_MP3_FRAME_FLOATS; ++i) {
            const int q = quant[i];
            const int mag = q < 0 ? -q : q;
            if (mag > 8206) return SYMGPU_ERR_DECODE;
            expanded[i] = q < 0 ? -pow43[mag] : pow43[mag];
        }
        spectra = expanded;
    }
    symgpu_async_mp3* a = state_of(ctx);
    if (!a) return SYMGPU_ERR_LIMIT;
    std::unique_lock<std::mutex> lk(a->m);
    Batch* b = open_batch(ctx, a);
    if (!b) return SYMGPU_ERR_LIMIT;
    if (b->streams.count(stream)) { // the stream's previous frame is still in this batch: it goes first, in its own launch
        b->closed = true;
        b = open_batch(ctx, a);
        if (!b) return SYMGPU_ERR_LIMIT;
    }
    const uint32_t slot = b->n++;
    std::memcpy(b->units + (size_t)slot * 4, units, 4 * sizeof(symgpu_mp3_gc));
    std::memcpy(b->spectra + (size_t)slot * SYMGPU_MP3_FRAME_FLOATS, spectra, SYMGPU_MP3_FRAME_FLOATS * sizeof(float));
    run.first_frame = slot;
    b->runs.push_back(run);
    b->streams.insert(stream);
    if (b->n == kBatchCap) b->closed = true;
    ticket->batch = b->seq;
    ticket->slot = slot;
    ticket->reserved = 0;
    return SYMGPU_OK;
}

} // namespace

extern "C" {

symgpu_status symgpu_mp3_submit(symgpu_ctx* ctx, uint32_t stream, const symgpu_mp3_gc* units, const float* spectra,
                                uint8_t granules_per_frame, uint8_t channels, symgpu_ticket* ticket) {
    try {
        return submit_impl(ctx, stream, units, spectra, nullptr, granules_per_frame, channels, ticket);
    } catch (...) { // no C++ exception crosses the ABI
        return SYMGPU_ERR_LIMIT;
    }
}

symgpu_status symgpu_mp3_submit_quantized(symgpu_ctx* ctx, uint32_t stream, const symgpu_mp3_gc* units, const int16_t* quant,
                                          uint8_t granules_per_frame, uint8_t channels, symgpu_ticket* ticket) {
    try {
        return submit_impl(ctx, stream, units, nullptr, quant, granules_per_frame, channels, ticket);
    } catch (...) {
        return SYMGPU_ERR_LIMIT;
    }
}

static symgpu_status wait_impl(symgpu_ctx* ctx, symgpu_ticket ticket, float* pcm) {
    if (!ctx || !pcm || !ctx->async_mp3) return SYMGPU_ERR_ARG;
    symgpu_async_mp3* a = ctx->async_mp3;
    std::unique_lock<std::mutex> lk(a->m);
    for (;;) {
        Batch* b = nullptr;
        for (auto& p : a->live)
            if (p->seq == ticket.batch) b = p.get();
        if (!b || ticket.slot >= b->n) return SYMGPU_ERR_ARG; // unknown or already collected ticket
        if (b->state == BatchState::Done) {
            const symgpu_status st = b->status;
            if (st == SYMGPU_OK) std::memcpy(pcm, b->pcm + (size_t)ticket.slot * SYMGPU_MP3_FRAME_FLOATS, SYMGPU_MP3_FRAME_FLOATS * sizeof(float));
            if (++b->collected == b->n) { // every ticket of the batch has been redeemed: its staging goes back to the pool
                for (auto it = a->live.begin(); it != a->live.end(); ++it)
                    if (it->get() == b) {
                        a->pool.push_back(std::move(*it));
                        a->live.erase(it);
                        break;
                    }
            }
            return st;
        }
        // Batches run in order: only the oldest unfinished one may start, and only if nothing is on the device.
        Batch* oldest = nullptr;
        bool running = false;
        for (auto& p : a->live) {
            if (p->state == BatchState::Running) running = true;
            if (!oldest && p->state != BatchState::Done) oldest = p.get();
        }
        if (!running && oldest && oldest->state == BatchState::Open && oldest->seq <= b->seq) {
            Batch* run = oldest; // lead: close it and run it for every thread that has a frame in it
            run->closed = true;
            run->state = BatchState::Running;
            lk.unlock();
            const symgpu_status st = symgpu_mp3_synth_host(ctx, run->units, run->spectra, run->runs.data(), (uint32_t)run->runs.size(), run->n, run->pcm);
            lk.lock();
            run->status = st;
            run->state = BatchState::Done;
            a->batches_run += 1;
            a->frames_run += run->n;
            a->cv.notify_all();
            continue;
        }
        a->cv.wait(lk);
    }
}

symgpu_status symgpu_mp3_wait(symgpu_ctx* ctx, symgpu_ticket ticket, float* pcm) {
    try {
        return wait_impl(ctx, ticket, pcm);
    } catch (...) {
        return SYMGPU_ERR_LIMIT;
    }
}

void symgpu_mp3_async_stats(const symgpu_ctx* ctx, uint64_t* batches, uint64_t* frames) {
    uint64_t b = 0, f = 0;
    if (ctx && ctx->async_mp3) {
        std::lock_guard<std::mutex> g(ctx->async_mp3->m);
        b = ctx->async_mp3->batches_run;
        f = ctx->async_mp3->frames_run;
    }
    if (batches) *batches = b;
    if (frames) *frames = f;
}

} // extern "C"
