// Asynchronous, thread-safe entry points: symgpu_{mp3,aac,mpa12,vorbis}_submit, symgpu_mp3_submit_quantized and the matching
// _wait calls (include/symgpu.h, SURVEY.md §8b "proposed exports").
//
// The reference's decoders are one object per stream, one decode() call per packet (codecs/audio.rs:251-298), made by
// the registry (registry.rs:260-269); a server runs hundreds of them on as many threads.  One launch per packet wastes
// the GPU (a kernel sized for every SM, for one frame), so the context gathers what the decoders of all threads have submitted into
// ONE batch: a frame is copied into pinned staging memory under a mutex (submit), and the first thread that waits for a
// ticket of the oldest unfinished batch closes it and runs it for everybody (wait) -- group commit: while that batch is
// on the device the other threads keep submitting into the next one.  Batches run in order, so the frames of a stream are
// synthesised in submission order; a stream appears at most once per batch (a second frame of the same stream closes the
// batch), which is what makes every slot a one-frame run of its stream.
//
// Every codec has a queue of its own (Layer I and Layer II too: a launch takes one time-slot count), and the queues differ
// only in what a slot holds and in the host entry point that runs a closed batch.  Leaders of different queues take the
// context's launch lock around that call: they share the device staging buffer, the plan caches and the CUDA stream.
#include <cuda_runtime.h>

#include <algorithm>
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

constexpr uint32_t kBatchCap = 2048;                // slots per batch: 2048 MP3 frames x 18.7 KB = 38 MB of pinned staging
constexpr size_t kBatchBytes = size_t(64) << 20;    // pinned staging per batch at most: a 4096-float Vorbis row is 64 KB a slot
constexpr int kQueues = SYMGPU_CODEC_VORBIS + 1;    // one per symgpu_codec

enum class BatchState { Open, Running, Done };

// What the codec's run record of a slot needs besides the slot itself.
struct SlotInfo {
    uint32_t stream;
    uint32_t dst_row;    // floats per channel of the caller's PCM buffer (Vorbis: the packet's own slot)
    uint8_t channels;
    uint8_t granules;    // MP3 only
};

struct Batch {
    uint64_t seq = 0;
    BatchState state = BatchState::Open;
    bool closed = false; // no more frames (full, or a stream came back for a second frame)
    symgpu_status status = SYMGPU_OK;
    uint32_t n = 0, collected = 0, cap = 0;
    uint32_t row = 0;                       // floats per channel of an output slot (and of a Vorbis residue slot)
    size_t bytes[3] = {0, 0, 0};            // bytes per slot of the codec's input arrays
    size_t offset[3] = {0, 0, 0};           // where array k starts in `in`
    unsigned char* in = nullptr;            // pinned: the input arrays, [cap][bytes[k]] each
    float* out = nullptr;                   // pinned [cap][2][row]
    size_t in_cap = 0, out_cap = 0;
    std::vector<SlotInfo> slots;
    std::vector<symgpu_aac_tns> tns;        // AAC: the filters of the batch; units' tns_first point into it
    std::unordered_set<uint32_t> streams;
    unsigned char* at(int k, uint32_t slot) { return in + offset[k] + (size_t)slot * bytes[k]; }
    ~Batch() {
        if (in) cudaFreeHost(in);
        if (out) cudaFreeHost(out);
    }
};

struct Queue {
    std::mutex m;
    std::condition_variable cv;
    std::deque<std::unique_ptr<Batch>> live; // oldest first; back() is the open batch
    std::vector<std::unique_ptr<Batch>> pool; // collected batches, staging reused
    uint64_t next_seq = 1;
    uint64_t batches_run = 0, frames_run = 0;
};

} // namespace

struct symgpu_async {
    Queue q[kQueues];
};

symgpu_async* symgpu_async_create() { return new (std::nothrow) symgpu_async(); }
void symgpu_async_destroy(symgpu_async* a) { delete a; }

namespace {

// Bytes per slot of each input array, in the order the codec's host entry point takes them.
void slot_layout(int codec, uint32_t row, size_t bytes[3]) {
    bytes[0] = bytes[1] = bytes[2] = 0;
    switch (codec) {
        case SYMGPU_CODEC_MP3: // units [2][2], spectra [2][2][576]
            bytes[0] = 4 * sizeof(symgpu_mp3_gc), bytes[1] = SYMGPU_MP3_FRAME_FLOATS * sizeof(float);
            break;
        case SYMGPU_CODEC_MP1: bytes[0] = 2 * 32 * 12 * sizeof(float); break; // subbands [2][32][12]
        case SYMGPU_CODEC_MP2: bytes[0] = 2 * 32 * 36 * sizeof(float); break; // subbands [2][32][36]
        case SYMGPU_CODEC_AAC: // units [2], coeffs [2][1024]
            bytes[0] = 2 * sizeof(symgpu_aac_unit), bytes[1] = 2 * 1024 * sizeof(float);
            break;
        case SYMGPU_CODEC_VORBIS: // unit, floor_y [2][65], residue [2][row]
            bytes[0] = sizeof(symgpu_vorbis_unit), bytes[1] = 2 * 65 * sizeof(uint16_t), bytes[2] = 2 * (size_t)row * sizeof(float);
            break;
    }
}

Batch* open_batch(symgpu_ctx* ctx, Queue& q, int codec, uint32_t row) { // q.m held
    if (!q.live.empty() && !q.live.back()->closed && q.live.back()->state == BatchState::Open) return q.live.back().get();
    std::unique_ptr<Batch> b;
    if (!q.pool.empty()) {
        b = std::move(q.pool.back());
        q.pool.pop_back();
    } else {
        b.reset(new (std::nothrow) Batch());
        if (!b) return nullptr;
    }
    slot_layout(codec, row, b->bytes);
    const size_t out_bytes = 2 * (size_t)row * sizeof(float);
    const size_t per_slot = b->bytes[0] + b->bytes[1] + b->bytes[2] + out_bytes;
    b->cap = (uint32_t)std::max<size_t>(1, std::min<size_t>(kBatchCap, kBatchBytes / per_slot));
    size_t in_bytes = 0;
    for (int k = 0; k < 3; ++k) {
        b->offset[k] = in_bytes;
        in_bytes += ((size_t)b->cap * b->bytes[k] + 255) & ~(size_t)255;
    }
    {
        DeviceGuard guard(ctx->device);
        if (b->in_cap < in_bytes) { // a pooled batch of a shorter Vorbis row, or a new one
            if (b->in) cudaFreeHost(b->in);
            b->in = nullptr, b->in_cap = 0;
            if (cudaMallocHost(&b->in, in_bytes) != cudaSuccess) return nullptr;
            b->in_cap = in_bytes;
        }
        if (b->out_cap < (size_t)b->cap * out_bytes) {
            if (b->out) cudaFreeHost(b->out);
            b->out = nullptr, b->out_cap = 0;
            if (cudaMallocHost(&b->out, (size_t)b->cap * out_bytes) != cudaSuccess) return nullptr;
            b->out_cap = (size_t)b->cap * out_bytes;
        }
    }
    b->row = row;
    b->seq = q.next_seq++;
    b->state = BatchState::Open;
    b->closed = false;
    b->status = SYMGPU_OK;
    b->n = b->collected = 0;
    b->slots.clear();
    b->tns.clear();
    b->streams.clear();
    q.live.push_back(std::move(b));
    return q.live.back().get();
}

// Takes a slot of the open batch of `codec` for one frame of `stream` and lets `fill` copy the frame into it.  `row`: the
// output row a new batch gets; `need`: the least row this frame fits (Vorbis: its stream's blocksize_1 / 2).
template <typename Fill>
symgpu_status enqueue(symgpu_ctx* ctx, int codec, uint32_t row, uint32_t need, const SlotInfo& info, symgpu_ticket* ticket, Fill&& fill) {
    Queue& q = ctx->async->q[codec];
    std::unique_lock<std::mutex> lk(q.m);
    Batch* b = open_batch(ctx, q, codec, row);
    if (!b) return SYMGPU_ERR_LIMIT;
    // the stream's previous frame is still in this batch: it goes first, in its own launch.  A Vorbis slot configured after the
    // batch was opened may need longer rows: the batch closes too.
    if (b->streams.count(info.stream) || b->row < need) {
        b->closed = true;
        b = open_batch(ctx, q, codec, row);
        if (!b) return SYMGPU_ERR_LIMIT;
    }
    const uint32_t slot = b->n++;
    fill(*b, slot);
    b->slots.push_back(info);
    b->streams.insert(info.stream);
    if (b->n == b->cap) b->closed = true;
    ticket->batch = b->seq;
    ticket->slot = slot;
    ticket->reserved = (uint32_t)codec;
    return SYMGPU_OK;
}

// Runs a closed batch through the codec's host entry point: every slot is a one-frame run of its stream.
symgpu_status launch(symgpu_ctx* ctx, int codec, Batch& b) {
    std::lock_guard<std::mutex> g(ctx->launch_m);
    const uint32_t n = b.n;
    switch (codec) {
        case SYMGPU_CODEC_MP3: {
            std::vector<symgpu_mp3_run> runs(n);
            for (uint32_t i = 0; i < n; ++i) runs[i] = symgpu_mp3_run{b.slots[i].stream, i, 1, b.slots[i].granules, b.slots[i].channels, 0};
            return symgpu_mp3_synth_host(ctx, reinterpret_cast<const symgpu_mp3_gc*>(b.at(0, 0)), reinterpret_cast<const float*>(b.at(1, 0)),
                                         runs.data(), n, n, b.out);
        }
        case SYMGPU_CODEC_MP1:
        case SYMGPU_CODEC_MP2: {
            std::vector<symgpu_mpa12_run> runs(n);
            for (uint32_t i = 0; i < n; ++i) runs[i] = symgpu_mpa12_run{b.slots[i].stream, i, 1, b.slots[i].channels, {0, 0, 0}};
            return symgpu_mpa12_synth_host(ctx, reinterpret_cast<const float*>(b.at(0, 0)), runs.data(), n, n,
                                           codec == SYMGPU_CODEC_MP1 ? 12u : 36u, b.out);
        }
        case SYMGPU_CODEC_AAC: {
            std::vector<symgpu_aac_run> runs(n);
            for (uint32_t i = 0; i < n; ++i) runs[i] = symgpu_aac_run{b.slots[i].stream, i, 1, b.slots[i].channels, {0, 0, 0}};
            return symgpu_aac_synth_host(ctx, reinterpret_cast<const symgpu_aac_unit*>(b.at(0, 0)), b.tns.empty() ? nullptr : b.tns.data(),
                                         (uint32_t)b.tns.size(), reinterpret_cast<const float*>(b.at(1, 0)), runs.data(), n, n, b.out);
        }
        case SYMGPU_CODEC_VORBIS: {
            std::vector<symgpu_vorbis_run> runs(n);
            for (uint32_t i = 0; i < n; ++i) runs[i] = symgpu_vorbis_run{b.slots[i].stream, i, 1, 0};
            return symgpu_vorbis_synth_host(ctx, reinterpret_cast<const symgpu_vorbis_unit*>(b.at(0, 0)),
                                            reinterpret_cast<const uint16_t*>(b.at(1, 0)), reinterpret_cast<const float*>(b.at(2, 0)),
                                            runs.data(), n, n, b.row, b.out);
        }
    }
    return SYMGPU_ERR_ARG;
}

symgpu_status wait_impl(symgpu_ctx* ctx, int codec, symgpu_ticket ticket, float* pcm) {
    if (!ctx || !pcm || !ctx->async || ticket.reserved != (uint32_t)codec) return SYMGPU_ERR_ARG;
    Queue& q = ctx->async->q[codec];
    std::unique_lock<std::mutex> lk(q.m);
    for (;;) {
        Batch* b = nullptr;
        for (auto& p : q.live)
            if (p->seq == ticket.batch) b = p.get();
        if (!b || ticket.slot >= b->n) return SYMGPU_ERR_ARG; // unknown or already collected ticket
        if (b->state == BatchState::Done) {
            const symgpu_status st = b->status;
            if (st == SYMGPU_OK) {
                const uint32_t dst_row = b->slots[ticket.slot].dst_row, k = std::min(dst_row, b->row);
                for (int ch = 0; ch < 2; ++ch) {
                    float* dst = pcm + (size_t)ch * dst_row;
                    std::memcpy(dst, b->out + ((size_t)ticket.slot * 2 + ch) * b->row, k * sizeof(float));
                    if (dst_row > k) std::memset(dst + k, 0, (dst_row - k) * sizeof(float));
                }
            }
            if (++b->collected == b->n) { // every ticket of the batch has been redeemed: its staging goes back to the pool
                for (auto it = q.live.begin(); it != q.live.end(); ++it)
                    if (it->get() == b) {
                        q.pool.push_back(std::move(*it));
                        q.live.erase(it);
                        break;
                    }
            }
            return st;
        }
        // Batches run in order: only the oldest unfinished one may start, and only if nothing of this queue is on the device.
        Batch* oldest = nullptr;
        bool running = false;
        for (auto& p : q.live) {
            if (p->state == BatchState::Running) running = true;
            if (!oldest && p->state != BatchState::Done) oldest = p.get();
        }
        if (!running && oldest && oldest->state == BatchState::Open && oldest->seq <= b->seq) {
            Batch* run = oldest; // lead: close it and run it for every thread that has a frame in it
            run->closed = true;
            run->state = BatchState::Running;
            lk.unlock();
            symgpu_status st;
            try {
                st = launch(ctx, codec, *run);
            } catch (...) {
                st = SYMGPU_ERR_LIMIT;
            }
            lk.lock();
            run->status = st;
            run->state = BatchState::Done;
            q.batches_run += 1;
            q.frames_run += run->n;
            q.cv.notify_all();
            continue;
        }
        q.cv.wait(lk);
    }
}

symgpu_status mp3_submit_impl(symgpu_ctx* ctx, uint32_t stream, const symgpu_mp3_gc* units, const float* spectra, const int16_t* quant,
                              uint8_t gpf, uint8_t channels, symgpu_ticket* ticket) {
    if (!ctx || !units || (!spectra == !quant) || !ticket || !ctx->async) return SYMGPU_ERR_ARG;
    if (stream >= ctx->n_mp3_streams) return SYMGPU_ERR_LIMIT;
    const symgpu_mp3_run run{stream, 0, 1, gpf, channels, 0};
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
    return enqueue(ctx, SYMGPU_CODEC_MP3, 1152, 1152, SlotInfo{stream, 1152, channels, gpf}, ticket, [&](Batch& b, uint32_t slot) {
        std::memcpy(b.at(0, slot), units, 4 * sizeof(symgpu_mp3_gc));
        std::memcpy(b.at(1, slot), spectra, SYMGPU_MP3_FRAME_FLOATS * sizeof(float));
    });
}

symgpu_status aac_submit_impl(symgpu_ctx* ctx, uint32_t stream, const symgpu_aac_unit* units, const symgpu_aac_tns* tns, uint32_t n_tns,
                              const float* coeffs, uint8_t channels, symgpu_ticket* ticket) {
    if (!ctx || !units || !coeffs || !ticket || (n_tns && !tns) || !ctx->async) return SYMGPU_ERR_ARG;
    const uint8_t n_ch = channels ? channels : 2;
    if (n_ch > 2) return SYMGPU_ERR_ARG;
    if (stream >= ctx->n_aac_streams) return SYMGPU_ERR_LIMIT;
    const symgpu_status chk = symgpu_aac_units_check(units, tns, n_tns, 1);
    if (chk != SYMGPU_OK) return chk;
    return enqueue(ctx, SYMGPU_CODEC_AAC, 1024, 1024, SlotInfo{stream, 1024, n_ch, 0}, ticket, [&](Batch& b, uint32_t slot) {
        // the filters each unit names move to the end of the batch's list, and tns_first with them
        symgpu_aac_unit u[2];
        std::memcpy(u, units, sizeof u);
        for (symgpu_aac_unit& x : u) {
            if (!x.n_tns) continue;
            const uint32_t first = x.tns_first;
            x.tns_first = (uint32_t)b.tns.size();
            b.tns.insert(b.tns.end(), tns + first, tns + first + x.n_tns);
        }
        std::memcpy(b.at(0, slot), u, sizeof u);
        std::memcpy(b.at(1, slot), coeffs, 2 * 1024 * sizeof(float));
    });
}

symgpu_status mpa12_submit_impl(symgpu_ctx* ctx, uint32_t stream, const float* subbands, uint32_t n_slots, uint8_t channels,
                                symgpu_ticket* ticket) {
    if (!ctx || !subbands || !ticket || !ctx->async || (n_slots != 12 && n_slots != 36) || channels < 1 || channels > 2) return SYMGPU_ERR_ARG;
    if (stream >= ctx->n_mp3_streams) return SYMGPU_ERR_LIMIT;
    const int codec = n_slots == 12 ? SYMGPU_CODEC_MP1 : SYMGPU_CODEC_MP2;
    return enqueue(ctx, codec, 1152, 1152, SlotInfo{stream, 1152, channels, 0}, ticket, [&](Batch& b, uint32_t slot) {
        std::memcpy(b.at(0, slot), subbands, 2 * 32 * (size_t)n_slots * sizeof(float));
    });
}

symgpu_status vorbis_submit_impl(symgpu_ctx* ctx, uint32_t stream, const symgpu_vorbis_unit* unit, const uint16_t* floor_y,
                                 const float* residue, uint32_t slot, symgpu_ticket* ticket) {
    if (!ctx || !unit || !floor_y || !residue || !ticket || !ctx->async) return SYMGPU_ERR_ARG;
    if (stream >= ctx->vorbis_slot_floors.size()) return SYMGPU_ERR_LIMIT;
    const symgpu_vorbis_stream cfg = ctx->h_vorbis_streams[stream];
    if (cfg.bs1_exp == 0) return SYMGPU_ERR_ARG; // the slot was never configured
    const uint32_t need = (1u << cfg.bs1_exp) >> 1;
    if (slot < need) return SYMGPU_ERR_ARG;
    // what the kernel would otherwise read as "true" or as another slot's floor setup
    if (unit->block_flag > 1 || unit->prev_block_flag > 1) return SYMGPU_ERR_DECODE;
    const uint32_t base = stream * SYMGPU_VORBIS_SLOT_FLOORS, n_floors = ctx->vorbis_slot_floors[stream];
    for (int ch = 0; ch < 2; ++ch) {
        if (unit->do_not_decode[ch] > 1) return SYMGPU_ERR_DECODE;
        const uint32_t f = unit->floor[ch];
        if (f != 0xffff && (ch >= cfg.channels || f < base || f >= base + n_floors)) return SYMGPU_ERR_DECODE;
    }
    const uint32_t row = std::max(ctx->vorbis_row.load(), need);
    return enqueue(ctx, SYMGPU_CODEC_VORBIS, row, need, SlotInfo{stream, slot, cfg.channels, 0}, ticket, [&](Batch& b, uint32_t s) {
        std::memcpy(b.at(0, s), unit, sizeof *unit);
        std::memcpy(b.at(1, s), floor_y, 2 * 65 * sizeof(uint16_t));
        float* r = reinterpret_cast<float*>(b.at(2, s));
        const uint32_t k = std::min(slot, b.row); // >= need: the stream's samples all fit
        for (int ch = 0; ch < 2; ++ch) {
            std::memcpy(r + (size_t)ch * b.row, residue + (size_t)ch * slot, k * sizeof(float));
            if (b.row > k) std::memset(r + (size_t)ch * b.row + k, 0, (b.row - k) * sizeof(float));
        }
    });
}

} // namespace

extern "C" {

// No C++ exception crosses the ABI: what a submission or wait throws (allocation) becomes SYMGPU_ERR_LIMIT.
#define SYMGPU_NOTHROW(call)          \
    try {                             \
        return call;                  \
    } catch (...) {                   \
        return SYMGPU_ERR_LIMIT;      \
    }

symgpu_status symgpu_mp3_submit(symgpu_ctx* ctx, uint32_t stream, const symgpu_mp3_gc* units, const float* spectra,
                                uint8_t granules_per_frame, uint8_t channels, symgpu_ticket* ticket) {
    SYMGPU_NOTHROW(mp3_submit_impl(ctx, stream, units, spectra, nullptr, granules_per_frame, channels, ticket))
}

symgpu_status symgpu_mp3_submit_quantized(symgpu_ctx* ctx, uint32_t stream, const symgpu_mp3_gc* units, const int16_t* quant,
                                          uint8_t granules_per_frame, uint8_t channels, symgpu_ticket* ticket) {
    SYMGPU_NOTHROW(mp3_submit_impl(ctx, stream, units, nullptr, quant, granules_per_frame, channels, ticket))
}

symgpu_status symgpu_mp3_wait(symgpu_ctx* ctx, symgpu_ticket ticket, float* pcm) { SYMGPU_NOTHROW(wait_impl(ctx, SYMGPU_CODEC_MP3, ticket, pcm)) }

symgpu_status symgpu_aac_submit(symgpu_ctx* ctx, uint32_t stream, const symgpu_aac_unit* units, const symgpu_aac_tns* tns,
                                uint32_t n_tns, const float* coeffs, uint8_t channels, symgpu_ticket* ticket) {
    SYMGPU_NOTHROW(aac_submit_impl(ctx, stream, units, tns, n_tns, coeffs, channels, ticket))
}

symgpu_status symgpu_aac_wait(symgpu_ctx* ctx, symgpu_ticket ticket, float* pcm) { SYMGPU_NOTHROW(wait_impl(ctx, SYMGPU_CODEC_AAC, ticket, pcm)) }

symgpu_status symgpu_mpa12_submit(symgpu_ctx* ctx, uint32_t stream, const float* subbands, uint32_t n_slots, uint8_t channels,
                                  symgpu_ticket* ticket) {
    SYMGPU_NOTHROW(mpa12_submit_impl(ctx, stream, subbands, n_slots, channels, ticket))
}

symgpu_status symgpu_mpa12_wait(symgpu_ctx* ctx, symgpu_ticket ticket, float* pcm) {
    // a Layer I ticket comes from the Layer I queue, a Layer II ticket from the Layer II queue
    const int codec = ticket.reserved == SYMGPU_CODEC_MP1 ? SYMGPU_CODEC_MP1 : SYMGPU_CODEC_MP2;
    SYMGPU_NOTHROW(wait_impl(ctx, codec, ticket, pcm))
}

symgpu_status symgpu_vorbis_submit(symgpu_ctx* ctx, uint32_t stream, const symgpu_vorbis_unit* unit, const uint16_t* floor_y,
                                   const float* residue, uint32_t slot, symgpu_ticket* ticket) {
    SYMGPU_NOTHROW(vorbis_submit_impl(ctx, stream, unit, floor_y, residue, slot, ticket))
}

symgpu_status symgpu_vorbis_wait(symgpu_ctx* ctx, symgpu_ticket ticket, float* pcm) { SYMGPU_NOTHROW(wait_impl(ctx, SYMGPU_CODEC_VORBIS, ticket, pcm)) }

symgpu_status symgpu_async_stats(const symgpu_ctx* ctx, int codec, uint64_t* batches, uint64_t* frames) {
    if (!ctx || codec < 0 || codec >= kQueues) return SYMGPU_ERR_ARG;
    uint64_t b = 0, f = 0;
    if (ctx->async) {
        Queue& q = ctx->async->q[codec];
        std::lock_guard<std::mutex> g(q.m);
        b = q.batches_run;
        f = q.frames_run;
    }
    if (batches) *batches = b;
    if (frames) *frames = f;
    return SYMGPU_OK;
}

void symgpu_mp3_async_stats(const symgpu_ctx* ctx, uint64_t* batches, uint64_t* frames) {
    if (symgpu_async_stats(ctx, SYMGPU_CODEC_MP3, batches, frames) != SYMGPU_OK) {
        if (batches) *batches = 0;
        if (frames) *frames = 0;
    }
}

} // extern "C"
