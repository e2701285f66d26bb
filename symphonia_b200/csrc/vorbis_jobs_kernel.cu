// Vorbis jobs built on the device from the tables of symgpu_ogg_index_dev (DESIGN §5b / §5f, include/symgpu.h): the headers
// decode.ogg_vorbis_index chooses, the packets' bytes gathered, and every audio packet's symgpu_vorbis_job with the reader's
// leading discard and page end trim.  The per-file and per-packet rules are functions of include/symgpu/packetizer.hpp that
// tests/cpp/ogg_vorbis_jobs_driver.cpp also runs on the CPU (vorbis_stream_heads, vorbis_is_audio, vorbis_packet_exp,
// vorbis_packet_time, ogg_run_start, ogg_packet_end_trim).  What a host walk does packet after packet is done here by scans:
//   symgpu_vorbis_heads_dev  1. vorbis_heads_kernel, one thread per file: the stream's end and its headers;
//                            2. vorbis_audio_kernel, one thread per packet: is it an audio packet;
//                            3. vorbis_rank_scan_kernel, one block: audio packets and bytes before each packet;
//                            4. vorbis_heads_total_kernel, one thread per file: its audio packets and bytes.
//   symgpu_ogg_gather_dev    ogg_gather_kernel, one warp per packet named.
//   symgpu_vorbis_jobs_dev   1. vorbis_job_gather_kernel, one warp per packet: bytes gathered, job slot, block exponent;
//                            2. vorbis_job_scan_kernel, one block: previous block exponent, duration, discard, runs of equal
//                               page sequence and the prefix sums of duration and discard;
//                            3. vorbis_job_trim_kernel, one thread per job: the run's start and the packet's end trim.
#include <cuda_runtime.h>

#include "../../include/symgpu/packetizer.hpp"
#include "batch_call.h"
#include "ogg_device.cuh"

namespace {

using namespace symgpu::packet;
using symgpu_detail::Carver;
using namespace symgpu_detail::ogg_dev;

constexpr uint32_t kNoFile = 0xffffffffu;

__device__ inline VorbisStreamHeads stream_heads(const symgpu_vorbis_file_heads& h) {
    return VorbisStreamHeads{h.n_stream, h.status ? h.n_stream : h.setup};
}

template <class T, class Op>
__device__ inline T warp_inclusive(T v, Op op) {
    const uint32_t lane = threadIdx.x & 31;
    for (int o = 1; o < 32; o *= 2) {
        const T u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= uint32_t(o)) v = op(u, v);
    }
    return v;
}

// Inclusive scan of v over a block of 1024 threads with `carry` (every thread's equal) in front; carry becomes the new total.
template <class T, class Op>
__device__ inline T block_inclusive(T v, Op op, T& carry, T* buf) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T s = warp_inclusive(v, op);
    if (lane == 31) buf[warp] = s;
    __syncthreads();
    if (warp == 0) buf[lane] = warp_inclusive(buf[lane], op);
    __syncthreads();
    s = op(carry, warp ? op(buf[warp - 1], s) : s);
    carry = op(carry, buf[31]);
    __syncthreads();
    return s;
}

struct Add {
    template <class T>
    __device__ T operator()(T a, T b) const { return a + b; }
};
struct Max {
    __device__ uint32_t operator()(uint32_t a, uint32_t b) const { return a > b ? a : b; }
};

// ---- heads --------------------------------------------------------------------------------------------------------------

__global__ void vorbis_heads_kernel(const uint8_t* __restrict__ data, const symgpu_file_range* __restrict__ files, uint32_t n_files,
                                    const symgpu_ogg_packet* __restrict__ packets, uint64_t n_packets, const symgpu_piece* __restrict__ pieces,
                                    const symgpu_ogg_file_index* __restrict__ index, symgpu_vorbis_file_heads* heads) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_files) return;
    const symgpu_ogg_file_index ix = index[i];
    symgpu_vorbis_file_heads h{};
    if (ix.n_packets == 0 || !tables_ok(ix, n_packets)) {
        h.status = SYMGPU_VORBIS_NO_PACKETS;
    } else {
        const symgpu_ogg_packet* pk = packets + ix.first_packet;
        const VorbisStreamHeads s = vorbis_stream_heads(data + files[i].offset, pk, ix.n_packets, pieces + ix.first_piece);
        h.n_stream = s.n_stream, h.ident_len = uint32_t(pk[0].len);
        if (s.setup == s.n_stream) h.status = SYMGPU_VORBIS_NO_SETUP;
        else h.setup = s.setup, h.setup_len = uint32_t(pk[s.setup].len);
    }
    heads[i] = h;
}

// ranks[p].audio, and the packet's length in byte_at for the scan that follows.
__global__ void vorbis_audio_kernel(const uint8_t* __restrict__ data, const symgpu_file_range* __restrict__ files, uint32_t n_files,
                                    const symgpu_ogg_packet* __restrict__ packets, uint64_t n_packets, const symgpu_piece* __restrict__ pieces,
                                    const symgpu_ogg_file_index* __restrict__ index, const symgpu_vorbis_file_heads* __restrict__ heads,
                                    symgpu_vorbis_packet_rank* ranks) {
    for (uint64_t p = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; p < n_packets; p += uint64_t(gridDim.x) * blockDim.x) {
        const uint32_t f = file_of_packet(index, n_files, p);
        const symgpu_ogg_file_index ix = index[f];
        const symgpu_vorbis_file_heads h = heads[f];
        bool audio = false;
        if (h.status == 0 && p >= ix.first_packet && p - ix.first_packet < ix.n_packets)
            audio = vorbis_is_audio(data + files[f].offset, packets + ix.first_packet, pieces + ix.first_piece, stream_heads(h),
                                    uint32_t(p - ix.first_packet));
        symgpu_vorbis_packet_rank r{};
        r.byte_at = audio ? packets[p].len : 0, r.audio = audio;
        ranks[p] = r;
    }
}

// Exclusive sums of audio packets and their bytes over the whole table, in one block of 1024 threads.
__global__ void __launch_bounds__(1024) vorbis_rank_scan_kernel(symgpu_vorbis_packet_rank* ranks, uint64_t n_packets) {
    __shared__ uint64_t buf[32];
    uint64_t carry_n = 0, carry_b = 0;
    for (uint64_t base = 0; base < n_packets; base += 1024) {
        const uint64_t p = base + threadIdx.x;
        const uint64_t a = p < n_packets ? ranks[p].audio : 0, b = p < n_packets ? ranks[p].byte_at : 0;
        const uint64_t sa = block_inclusive(a, Add{}, carry_n, buf), sb = block_inclusive(b, Add{}, carry_b, buf);
        if (p < n_packets) ranks[p].rank = sa - a, ranks[p].byte_at = sb - b;
    }
}

__global__ void vorbis_heads_total_kernel(const symgpu_ogg_packet* __restrict__ packets, const symgpu_ogg_file_index* __restrict__ index,
                                          uint32_t n_files, const symgpu_vorbis_packet_rank* __restrict__ ranks, symgpu_vorbis_file_heads* heads) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_files || heads[i].status) return;
    const symgpu_ogg_file_index ix = index[i];
    const uint64_t first = ix.first_packet, last = first + ix.n_packets - 1;
    const symgpu_vorbis_packet_rank a = ranks[first], z = ranks[last];
    heads[i].n_audio = uint32_t(z.rank + z.audio - a.rank);
    heads[i].audio_bytes = z.byte_at + (z.audio ? packets[last].len : 0) - a.byte_at;
}

// ---- gathers --------------------------------------------------------------------------------------------------------------

__global__ void ogg_gather_kernel(const uint8_t* __restrict__ data, const symgpu_file_range* __restrict__ files, uint32_t n_files,
                                  const symgpu_ogg_packet* __restrict__ packets, const symgpu_piece* __restrict__ pieces,
                                  const symgpu_ogg_file_index* __restrict__ index, const symgpu_ogg_packet_ref* __restrict__ refs, uint64_t n_refs,
                                  uint8_t* out, uint64_t out_cap) {
    const uint64_t warps = uint64_t(gridDim.x) * (blockDim.x / 32);
    for (uint64_t r = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) / 32; r < n_refs; r += warps) {
        const symgpu_ogg_packet_ref ref = refs[r];
        if (ref.file >= n_files) continue;
        const symgpu_ogg_file_index ix = index[ref.file];
        if (ref.packet >= ix.n_packets || (ix.status & SYMGPU_OGG_NOT_WRITTEN)) continue;
        const symgpu_ogg_packet pk = packets[ix.first_packet + ref.packet];
        if (ref.dst > out_cap || pk.len > out_cap - ref.dst) continue;
        warp_copy_packet(out + ref.dst, data + files[ref.file].offset, pieces + ix.first_piece + pk.first_piece, pk.n_pieces);
    }
}

// ---- jobs -----------------------------------------------------------------------------------------------------------------

struct JobScratch {
    uint32_t* first;     // the file's first job; kNoFile: no packet filled the slot
    uint32_t* count;     // the file's number of jobs
    uint8_t* exp;        // vorbis_packet_exp
    uint32_t* seq;       // page_sequence
    uint64_t* absgp;     // page_absgp
    uint32_t* dur;
    uint32_t* discard;
    uint32_t* run;       // run of equal page_sequence (a run never crosses files)
    int64_t* dur_sum;    // inclusive prefix sums over the job table
    int64_t* discard_sum;
    uint32_t* run_head;  // per run: its first job
};

__global__ void vorbis_job_gather_kernel(const uint8_t* __restrict__ data, const symgpu_file_range* __restrict__ files, uint32_t n_files,
                                         const symgpu_ogg_packet* __restrict__ packets, uint64_t n_packets,
                                         const symgpu_piece* __restrict__ pieces, const symgpu_ogg_file_index* __restrict__ index,
                                         const symgpu_vorbis_packet_rank* __restrict__ ranks, const symgpu_vorbis_file_jobs* __restrict__ fjobs,
                                         uint8_t* out, symgpu_vorbis_job* jobs, JobScratch s) {
    const uint64_t warps = uint64_t(gridDim.x) * (blockDim.x / 32);
    for (uint64_t p = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) / 32; p < n_packets; p += warps) {
        const symgpu_vorbis_packet_rank rk = ranks[p];
        if (!rk.audio) continue;
        const uint32_t f = file_of_packet(index, n_files, p);
        const symgpu_ogg_file_index ix = index[f];
        const symgpu_vorbis_file_jobs fj = fjobs[f];
        if (!fj.n_modes || p < ix.first_packet || p - ix.first_packet >= ix.n_packets) continue;
        const symgpu_vorbis_packet_rank base = ranks[ix.first_packet];
        const uint64_t jr = rk.rank - base.rank, off = rk.byte_at - base.byte_at;
        const symgpu_ogg_packet pk = packets[p];
        if (jr >= fj.n_jobs || off > fj.n_bytes || pk.len > fj.n_bytes - off) continue;
        const uint8_t* d = data + files[f].offset;
        const symgpu_piece* pc = pieces + ix.first_piece + pk.first_piece;
        warp_copy_packet(out + fj.byte_at + off, d, pc, pk.n_pieces);
        if ((threadIdx.x & 31) == 0) {
            const uint64_t j = fj.first_job + jr;
            uint8_t head[2] = {0, 0};
            const uint32_t got = ogg_packet_head(d, pc, pk.n_pieces, head, 2);
            s.first[j] = fj.first_job, s.count[j] = fj.n_jobs;
            s.exp[j] = vorbis_packet_exp(head, got, fj.n_modes, fj.long_block_mask, fj.bs0_exp, fj.bs1_exp);
            s.seq[j] = pk.page_sequence, s.absgp[j] = pk.page_absgp;
            jobs[j] = symgpu_vorbis_job{fj.byte_at + off, uint32_t(pk.len), 0, 0, 0};
        }
    }
}

// In job order, with carries from tile to tile: the nearest earlier job of the same file with a block (a max-scan of "job
// index + 1 where the exponent is non-zero", shifted by one), the packet's duration and discard, run heads (a job that starts
// its file or whose page_sequence differs from the job before) and their running count, and the prefix sums of duration and
// discard.
__global__ void __launch_bounds__(1024) vorbis_job_scan_kernel(uint32_t n_jobs, JobScratch s) {
    __shared__ uint64_t buf64[32];
    __shared__ uint32_t buf32[32];
    uint32_t carry_prev = 0, carry_runs = 0;
    uint64_t carry_dur = 0, carry_disc = 0;
    for (uint32_t base = 0; base < n_jobs; base += 1024) {
        const uint32_t j = base + threadIdx.x;
        const bool valid = j < n_jobs;
        const uint32_t first = valid ? s.first[j] : kNoFile;
        const bool own = first != kNoFile;
        const uint8_t e = own ? s.exp[j] : 0;
        // job j - 1 (if it has a block) as the candidate previous block of job j
        const uint32_t key = valid && j > 0 && s.first[j - 1] != kNoFile && s.exp[j - 1] ? j : 0;
        const uint32_t prev = block_inclusive(key, Max{}, carry_prev, buf32);   // latest job < j with a block, plus 1
        const uint8_t prev_exp = own && prev && prev - 1 >= first ? s.exp[prev - 1] : 0;
        uint64_t dur = 0, disc = 0;
        vorbis_packet_time(prev_exp, e, dur, disc);
        const uint32_t head = valid && (!own || j == first || s.seq[j] != s.seq[j - 1]);
        const uint32_t runs = block_inclusive(head, Add{}, carry_runs, buf32);
        const uint64_t sd = block_inclusive(valid ? dur : 0, Add{}, carry_dur, buf64);
        const uint64_t sc = block_inclusive(valid ? disc : 0, Add{}, carry_disc, buf64);
        if (valid) {
            s.dur[j] = uint32_t(dur), s.discard[j] = uint32_t(disc), s.run[j] = runs - 1;
            s.dur_sum[j] = int64_t(sd), s.discard_sum[j] = int64_t(sc);
            if (head) s.run_head[runs - 1] = j;
        }
    }
}

__global__ void vorbis_job_trim_kernel(uint32_t n_jobs, JobScratch s, symgpu_vorbis_job* jobs) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_jobs || s.first[j] == kNoFile) return;
    const uint32_t first = s.first[j], last = first + s.count[j];
    const uint32_t r = s.run[j], h = s.run_head[r], n_runs = s.run[n_jobs - 1] + 1;
    const uint32_t next_head = r + 1 < n_runs ? s.run_head[r + 1] : n_jobs;
    const int64_t dur_before = h ? s.dur_sum[h - 1] : 0, disc_before = h ? s.discard_sum[h - 1] : 0;
    const int64_t tot = s.dur_sum[next_head - 1] - dur_before, disc = s.discard_sum[next_head - 1] - disc_before;
    const int64_t end = int64_t(s.absgp[h]);
    const bool have_prev = h > first;
    const uint32_t ph = have_prev ? s.run_head[r - 1] : h;
    const int64_t start = ogg_run_start(have_prev, s.seq[ph], int64_t(s.absgp[ph]), s.seq[h], h == first && next_head == last, tot, disc, end);
    jobs[j].discard = s.discard[j];
    jobs[j].trim_end = ogg_packet_end_trim(start + (s.dur_sum[j] - dur_before), end, s.dur[j], s.discard[j]);
}

}  // namespace

using namespace symgpu_detail;

extern "C" symgpu_status symgpu_vorbis_heads_dev(symgpu_ctx* ctx, const uint8_t* data, size_t n_bytes, const symgpu_file_range* files, size_t n_files,
                                                 const symgpu_ogg_packet* packets, size_t n_packets, const symgpu_piece* pieces,
                                                 const symgpu_ogg_file_index* index, symgpu_vorbis_file_heads* heads, symgpu_vorbis_packet_rank* ranks) {
    if (!ctx || (n_files && (!index || !heads)) || (n_packets && (!packets || !pieces || !ranks))) return SYMGPU_ERR_ARG;
    symgpu_status e = check_files(data, n_bytes, files, n_files);
    if (e != SYMGPU_OK || n_files == 0) return e;
    DeviceGuard guard(ctx->device);
    Carver c;
    const size_t at_files = c.take(n_files * sizeof(symgpu_file_range));
    if ((e = ensure_stage(ctx, c.at)) != SYMGPU_OK) return e;
    auto* d_files = reinterpret_cast<symgpu_file_range*>(static_cast<char*>(ctx->d_stage) + at_files);
    cudaStream_t st = ctx->stream;
    CU(ctx, cudaMemcpyAsync(d_files, files, n_files * sizeof(symgpu_file_range), cudaMemcpyHostToDevice, st));
    const uint32_t nf = uint32_t(n_files);
    vorbis_heads_kernel<<<(nf + 127) / 128, 128, 0, st>>>(data, d_files, nf, packets, n_packets, pieces, index, heads);
    CU(ctx, cudaGetLastError());
    vorbis_audio_kernel<<<blocks_for(n_packets, 256), 256, 0, st>>>(data, d_files, nf, packets, n_packets, pieces, index, heads, ranks);
    CU(ctx, cudaGetLastError());
    vorbis_rank_scan_kernel<<<1, 1024, 0, st>>>(ranks, n_packets);
    CU(ctx, cudaGetLastError());
    vorbis_heads_total_kernel<<<(nf + 127) / 128, 128, 0, st>>>(packets, index, nf, ranks, heads);
    CU(ctx, cudaGetLastError());
    ctx->launches += 4;
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_ogg_gather_dev(symgpu_ctx* ctx, const uint8_t* data, size_t n_bytes, const symgpu_file_range* files, size_t n_files,
                                               const symgpu_ogg_packet* packets, const symgpu_piece* pieces, const symgpu_ogg_file_index* index,
                                               const symgpu_ogg_packet_ref* refs, size_t n_refs, uint8_t* out, size_t out_cap) {
    if (!ctx || (n_files && !index) || (n_refs && (!refs || !packets || !pieces)) || (out_cap && !out)) return SYMGPU_ERR_ARG;
    symgpu_status e = check_files(data, n_bytes, files, n_files);
    if (e != SYMGPU_OK || n_files == 0 || n_refs == 0) return e;
    DeviceGuard guard(ctx->device);
    Carver c;
    const size_t at_files = c.take(n_files * sizeof(symgpu_file_range)), at_refs = c.take(n_refs * sizeof(symgpu_ogg_packet_ref));
    if ((e = ensure_stage(ctx, c.at)) != SYMGPU_OK) return e;
    char* stage = static_cast<char*>(ctx->d_stage);
    auto* d_files = reinterpret_cast<symgpu_file_range*>(stage + at_files);
    auto* d_refs = reinterpret_cast<symgpu_ogg_packet_ref*>(stage + at_refs);
    cudaStream_t st = ctx->stream;
    CU(ctx, cudaMemcpyAsync(d_files, files, n_files * sizeof(symgpu_file_range), cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemcpyAsync(d_refs, refs, n_refs * sizeof(symgpu_ogg_packet_ref), cudaMemcpyHostToDevice, st));
    ogg_gather_kernel<<<blocks_for(n_refs * 32, 256), 256, 0, st>>>(data, d_files, uint32_t(n_files), packets, pieces, index, d_refs, n_refs, out, out_cap);
    CU(ctx, cudaGetLastError());
    ++ctx->launches;
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_vorbis_jobs_dev(symgpu_ctx* ctx, const uint8_t* data, size_t n_bytes, const symgpu_file_range* files, size_t n_files,
                                                const symgpu_ogg_packet* packets, size_t n_packets, const symgpu_piece* pieces,
                                                const symgpu_ogg_file_index* index, const symgpu_vorbis_packet_rank* ranks,
                                                const symgpu_vorbis_file_jobs* file_jobs, uint8_t* out, size_t out_cap, symgpu_vorbis_job* jobs,
                                                size_t n_jobs) {
    if (!ctx || (n_files && (!index || !file_jobs)) || (n_packets && (!packets || !pieces || !ranks)) || (out_cap && !out) || (n_jobs && !jobs))
        return SYMGPU_ERR_ARG;
    symgpu_status e = check_files(data, n_bytes, files, n_files);
    if (e != SYMGPU_OK) return e;
    if (n_jobs >= kNoFile) return SYMGPU_ERR_LIMIT;
    for (size_t i = 0; i < n_files; ++i) {
        const symgpu_vorbis_file_jobs& f = file_jobs[i];
        if (!f.n_modes) continue;
        if (f.n_modes > 64 || f.bs0_exp < 6 || f.bs0_exp > f.bs1_exp || f.bs1_exp > 13 || f.first_job > n_jobs || f.n_jobs > n_jobs - f.first_job ||
            f.byte_at > out_cap || f.n_bytes > out_cap - f.byte_at)
            return SYMGPU_ERR_ARG;
    }
    if (n_files == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    Carver c;
    const size_t at_files = c.take(n_files * sizeof(symgpu_file_range)), at_fjobs = c.take(n_files * sizeof(symgpu_vorbis_file_jobs));
    const size_t at_first = c.take(n_jobs * 4), at_count = c.take(n_jobs * 4), at_exp = c.take(n_jobs), at_seq = c.take(n_jobs * 4);
    const size_t at_gp = c.take(n_jobs * 8), at_dur = c.take(n_jobs * 4), at_disc = c.take(n_jobs * 4), at_run = c.take(n_jobs * 4);
    const size_t at_dsum = c.take(n_jobs * 8), at_csum = c.take(n_jobs * 8), at_head = c.take(n_jobs * 4);
    if ((e = ensure_stage(ctx, c.at)) != SYMGPU_OK) return e;
    char* stage = static_cast<char*>(ctx->d_stage);
    auto* d_files = reinterpret_cast<symgpu_file_range*>(stage + at_files);
    auto* d_fjobs = reinterpret_cast<symgpu_vorbis_file_jobs*>(stage + at_fjobs);
    const JobScratch s{reinterpret_cast<uint32_t*>(stage + at_first), reinterpret_cast<uint32_t*>(stage + at_count), reinterpret_cast<uint8_t*>(stage + at_exp),
                       reinterpret_cast<uint32_t*>(stage + at_seq), reinterpret_cast<uint64_t*>(stage + at_gp), reinterpret_cast<uint32_t*>(stage + at_dur),
                       reinterpret_cast<uint32_t*>(stage + at_disc), reinterpret_cast<uint32_t*>(stage + at_run), reinterpret_cast<int64_t*>(stage + at_dsum),
                       reinterpret_cast<int64_t*>(stage + at_csum), reinterpret_cast<uint32_t*>(stage + at_head)};
    cudaStream_t st = ctx->stream;
    CU(ctx, cudaMemcpyAsync(d_files, files, n_files * sizeof(symgpu_file_range), cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemcpyAsync(d_fjobs, file_jobs, n_files * sizeof(symgpu_vorbis_file_jobs), cudaMemcpyHostToDevice, st));
    if (n_jobs) {
        CU(ctx, cudaMemsetAsync(s.first, 0xff, n_jobs * 4, st));
        CU(ctx, cudaMemsetAsync(jobs, 0, n_jobs * sizeof(symgpu_vorbis_job), st));
    }
    const uint32_t nj = uint32_t(n_jobs);
    vorbis_job_gather_kernel<<<blocks_for(uint64_t(n_packets) * 32, 256), 256, 0, st>>>(data, d_files, uint32_t(n_files), packets, n_packets, pieces,
                                                                                       index, ranks, d_fjobs, out, jobs, s);
    CU(ctx, cudaGetLastError());
    vorbis_job_scan_kernel<<<1, 1024, 0, st>>>(nj, s);
    CU(ctx, cudaGetLastError());
    vorbis_job_trim_kernel<<<blocks_for(nj, 256), 256, 0, st>>>(nj, s, jobs);
    CU(ctx, cudaGetLastError());
    ctx->launches += 3;
    return SYMGPU_OK;
}
