// CAF files holding ALAC indexed on the device, many resident files per call (include/symgpu.h "CAF indexed on the device";
// DESIGN §5b).  The chunk rules are packetizer.hpp's caf_open and caf_varint, the very functions of the host index.
//
//   caf_open_kernel        one thread per file: the chunk walk and the magic cookie -> the file's info record
//   scans                  per file: table bytes and integer counts -> where each file's table bytes and integers start
//   caf_flag_kernel        one thread per table byte: 1 where a byte ends an integer (top bit clear)
//   scan                   the flags -> each integer's number
//   caf_integer_kernel     one thread per table byte that ends an integer: the integer from its at most 9 bytes
//   scan by file           sizes -> each packet's offset from the file's data start
//   caf_fit_kernel         one thread per integer: whether the packet lies whole in the file (a prefix of each file's packets)
//   scan                   packets kept per file -> first_packet
//   caf_write_kernel       one thread per integer: the kept packets and their jobs
#include <cuda_runtime.h>

#include <cub/device/device_scan.cuh>

#include "batch_call.h"
#include "caf_records.h"

using namespace symgpu_detail;
using namespace symgpu::packet;

namespace {

constexpr unsigned long long kSizeClamp = 1ull << 33;  // any size above 2^32 - 1 ends the packets; clamped, the offsets cannot wrap

__global__ void __launch_bounds__(128) caf_open_kernel(const uint8_t* __restrict__ data, const symgpu_file_range* __restrict__ files, uint32_t n_files,
                                                       symgpu_caf_info* __restrict__ infos) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_files) return;
    const symgpu_file_range f = files[i];
    CafAlac a;
    const Status s = caf_open(data + f.offset, f.len, a);
    infos[i] = caf_info_record(a, s);
}

// per file: its table bytes and integers, with a trailing zero so that the exclusive scans end with the totals
__global__ void __launch_bounds__(256) caf_extent_kernel(const symgpu_caf_info* __restrict__ infos, uint32_t n_files, unsigned long long* __restrict__ tbytes,
                                                         unsigned long long* __restrict__ tints) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n_files) return;
    const bool ok = i < n_files && infos[i].open == SYMGPU_OK;
    tbytes[i] = ok ? infos[i].table_bytes : 0;
    tints[i] = ok ? infos[i].table_packets : 0;
}

// the file holding table byte t: the last file whose tables start at or before t (files without table bytes share their start
// with the next file, so the last one is the one that holds t)
__device__ __forceinline__ uint32_t file_of(const unsigned long long* tbase, uint32_t n_files, unsigned long long t) {
    uint32_t lo = 0, hi = n_files;  // tbase[lo] <= t < tbase[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (tbase[mid] <= t) lo = mid;
        else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(256) caf_flag_kernel(const uint8_t* __restrict__ data, const symgpu_file_range* __restrict__ files, uint32_t n_files,
                                                       const symgpu_caf_info* __restrict__ infos, const unsigned long long* __restrict__ tbase,
                                                       unsigned long long n_table, uint32_t* __restrict__ flags) {
    const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_table) return;
    const uint32_t f = file_of(tbase, n_files, t);
    flags[t] = data[files[f].offset + infos[f].table_at + (t - tbase[f])] & 0x80 ? 0u : 1u;
}

__global__ void __launch_bounds__(256) caf_integer_kernel(const uint8_t* __restrict__ data, const symgpu_file_range* __restrict__ files, uint32_t n_files,
                                                          const symgpu_caf_info* __restrict__ infos, const unsigned long long* __restrict__ tbase,
                                                          unsigned long long n_table, const uint32_t* __restrict__ flags, const uint32_t* __restrict__ number,
                                                          unsigned long long* __restrict__ sizes, uint32_t* __restrict__ keys) {
    const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_table || !flags[t]) return;
    const uint32_t f = file_of(tbase, n_files, t);
    const uint8_t* table = data + files[f].offset + infos[f].table_at;
    const unsigned long long local = t - tbase[f];
    unsigned long long first = local;
    while (first > 0 && local - first < 8 && (table[first - 1] & 0x80)) --first;  // caf_open saw at most 9 bytes per integer
    uint64_t at = first, v = 0;
    caf_varint(table, local + 1, at, v);
    const uint32_t q = number[t];
    sizes[q] = v < kSizeClamp ? v : kSizeClamp;
    keys[q] = f;
}

__global__ void __launch_bounds__(256) caf_fit_kernel(const symgpu_file_range* __restrict__ files, const symgpu_caf_info* __restrict__ infos,
                                                      uint32_t n_ints, const unsigned long long* __restrict__ sizes, const uint32_t* __restrict__ keys,
                                                      const unsigned long long* __restrict__ offs, unsigned long long* __restrict__ kept) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n_ints) return;
    const uint32_t f = keys[q];
    if (caf_packet_fits(infos[f].data_start, offs[q], sizes[q], files[f].len)) atomicAdd(&kept[f], 1ull);
}

__global__ void __launch_bounds__(256) caf_write_kernel(const symgpu_file_range* __restrict__ files, symgpu_caf_info* __restrict__ infos, uint32_t n_files,
                                                        uint32_t n_ints, const unsigned long long* __restrict__ ibase, const unsigned long long* __restrict__ sizes,
                                                        const uint32_t* __restrict__ keys, const unsigned long long* __restrict__ offs,
                                                        const unsigned long long* __restrict__ kept, const unsigned long long* __restrict__ first,
                                                        uint64_t* __restrict__ first_packet, symgpu_caf_packet* __restrict__ packets, symgpu_alac_job* __restrict__ jobs,
                                                        unsigned long long cap) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < n_files) {  // the per-file records ride along with the first threads
        infos[q].n_packets = kept[q];
        first_packet[q] = first[q];
    }
    if (q >= n_ints) return;
    const uint32_t f = keys[q];
    const unsigned long long k = q - ibase[f];
    if (k >= kept[f] || first[f] + k >= cap) return;
    const symgpu_caf_info& info = infos[f];
    const uint64_t offset = info.data_start + offs[q];
    if (packets) packets[first[f] + k] = symgpu_caf_packet{offset, uint32_t(sizes[q]), info.frames_per_packet};
    if (jobs) jobs[first[f] + k] = symgpu_alac_job{files[f].offset + offset, uint32_t(sizes[q]), f, info.frame_length, 0};
}

symgpu_status check_files(const symgpu_ctx* ctx, const uint8_t* data, size_t n_bytes, const symgpu_file_range* files, size_t n_files) {
    if (!ctx || (n_bytes && !data) || (n_files && !files)) return SYMGPU_ERR_ARG;
    if (n_files > SYMGPU_CAF_MAX_FILES) return SYMGPU_ERR_LIMIT;
    for (size_t i = 0; i < n_files; ++i) {
        if (files[i].offset > n_bytes || files[i].len > n_bytes - files[i].offset) return SYMGPU_ERR_ARG;
        if (files[i].len >= (1ull << 32)) return SYMGPU_ERR_LIMIT;
    }
    return SYMGPU_OK;
}

// the per-file scratch: the file ranges, then the extents and their scans
struct FileScratch {
    size_t files, tbytes, tints, tbase, ibase, kept, first, total;
};
FileScratch file_layout(size_t n_files) {
    FileScratch s;
    Carver c;
    s.files = c.take(n_files * sizeof(symgpu_file_range));
    s.tbytes = c.take((n_files + 1) * 8);
    s.tints = c.take((n_files + 1) * 8);
    s.tbase = c.take((n_files + 1) * 8);
    s.ibase = c.take((n_files + 1) * 8);
    s.kept = c.take((n_files + 1) * 8);
    s.first = c.take((n_files + 1) * 8);
    s.total = c.at;
    return s;
}

}  // namespace

extern "C" symgpu_status symgpu_caf_open_dev(symgpu_ctx* ctx, const uint8_t* data, size_t n_bytes, const symgpu_file_range* files, size_t n_files,
                                             symgpu_caf_info* infos) {
    symgpu_status e = check_files(ctx, data, n_bytes, files, n_files);
    if (e != SYMGPU_OK) return e;
    if (n_files && !infos) return SYMGPU_ERR_ARG;
    if (n_files == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    const FileScratch s = file_layout(n_files);
    e = ensure_stage(ctx, s.total);
    if (e != SYMGPU_OK) return e;
    auto* d_files = reinterpret_cast<symgpu_file_range*>(static_cast<char*>(ctx->d_stage) + s.files);
    CU(ctx, cudaMemcpyAsync(d_files, files, n_files * sizeof(symgpu_file_range), cudaMemcpyHostToDevice, ctx->stream));
    caf_open_kernel<<<(uint32_t(n_files) + 127) / 128, 128, 0, ctx->stream>>>(data, d_files, uint32_t(n_files), infos);
    CU(ctx, cudaGetLastError());
    CU(ctx, cudaStreamSynchronize(ctx->stream));  // the host ranges are staged through a buffer the next call may reuse
    ctx->launches += 1;
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_caf_packets_dev(symgpu_ctx* ctx, const uint8_t* data, size_t n_bytes, const symgpu_file_range* files, size_t n_files,
                                                symgpu_caf_info* infos, uint64_t* first_packet, symgpu_caf_packet* packets, symgpu_alac_job* jobs,
                                                size_t cap_packets) {
    symgpu_status e = check_files(ctx, data, n_bytes, files, n_files);
    if (e != SYMGPU_OK) return e;
    if (n_files && (!infos || !first_packet)) return SYMGPU_ERR_ARG;
    if (n_files == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    const uint32_t nf = uint32_t(n_files);
    cudaStream_t st = ctx->stream;
    // phase 1: the extents, their scans and the two totals (the one host wait)
    size_t t_ext = 0;
    CU(ctx, cub::DeviceScan::ExclusiveSum(nullptr, t_ext, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, int(nf + 1), st));
    FileScratch fs = file_layout(n_files);
    Carver c0{fs.total};
    const size_t o_temp0 = c0.take(t_ext);
    const size_t o_totals = c0.take(16);
    e = ensure_stage(ctx, c0.at);
    if (e != SYMGPU_OK) return e;
    char* stage = static_cast<char*>(ctx->d_stage);
    auto P = [&](size_t o) { return reinterpret_cast<unsigned long long*>(stage + o); };
    CU(ctx, cudaMemcpyAsync(stage + fs.files, files, n_files * sizeof(symgpu_file_range), cudaMemcpyHostToDevice, st));
    caf_extent_kernel<<<(nf + 1 + 255) / 256, 256, 0, st>>>(infos, nf, P(fs.tbytes), P(fs.tints));
    CU(ctx, cudaGetLastError());
    size_t tb = t_ext;
    CU(ctx, cub::DeviceScan::ExclusiveSum(stage + o_temp0, tb, P(fs.tbytes), P(fs.tbase), int(nf + 1), st));
    tb = t_ext;
    CU(ctx, cub::DeviceScan::ExclusiveSum(stage + o_temp0, tb, P(fs.tints), P(fs.ibase), int(nf + 1), st));
    CU(ctx, cudaMemcpyAsync(P(o_totals), P(fs.tbase) + nf, 8, cudaMemcpyDeviceToDevice, st));
    CU(ctx, cudaMemcpyAsync(P(o_totals) + 1, P(fs.ibase) + nf, 8, cudaMemcpyDeviceToDevice, st));
    unsigned long long totals[2];
    CU(ctx, cudaMemcpyAsync(totals, P(o_totals), 16, cudaMemcpyDeviceToHost, st));
    CU(ctx, cudaStreamSynchronize(st));
    ctx->launches += 5;
    const unsigned long long n_table = totals[0], n_ints = totals[1];
    if (n_table >= 0xffffffffull || n_ints >= 0xffffffffull) return SYMGPU_ERR_LIMIT;
    // phase 2: the tables
    size_t t_flags = 0, t_key = 0, t_kept = 0;
    CU(ctx, cub::DeviceScan::ExclusiveSum(nullptr, t_flags, (const uint32_t*)nullptr, (uint32_t*)nullptr, int(n_table), st));
    CU(ctx, cub::DeviceScan::ExclusiveSumByKey(nullptr, t_key, (const uint32_t*)nullptr, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                               int(n_ints), cuda::std::equal_to<>(), st));
    CU(ctx, cub::DeviceScan::ExclusiveSum(nullptr, t_kept, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, int(nf + 1), st));
    size_t t_max = t_flags > t_key ? t_flags : t_key;
    t_max = t_max > t_kept ? t_max : t_kept;
    Carver c{c0.at};
    const size_t o_flags = c.take(n_table * 4), o_number = c.take(n_table * 4), o_sizes = c.take(n_ints * 8), o_keys = c.take(n_ints * 4),
                 o_offs = c.take(n_ints * 8), o_temp = c.take(t_max);
    e = ensure_stage_keep(ctx, c.at, c0.at);
    if (e != SYMGPU_OK) return e;
    stage = static_cast<char*>(ctx->d_stage);
    const auto* d_files = reinterpret_cast<const symgpu_file_range*>(stage + fs.files);
    auto* flags = reinterpret_cast<uint32_t*>(stage + o_flags);
    auto* number = reinterpret_cast<uint32_t*>(stage + o_number);
    auto* keys = reinterpret_cast<uint32_t*>(stage + o_keys);
    CU(ctx, cudaMemsetAsync(P(fs.kept), 0, (n_files + 1) * 8, st));
    if (n_table) {
        const unsigned grid = unsigned((n_table + 255) / 256);
        caf_flag_kernel<<<grid, 256, 0, st>>>(data, d_files, nf, infos, P(fs.tbase), n_table, flags);
        CU(ctx, cudaGetLastError());
        size_t tt = t_max;
        CU(ctx, cub::DeviceScan::ExclusiveSum(stage + o_temp, tt, flags, number, int(n_table), st));
        caf_integer_kernel<<<grid, 256, 0, st>>>(data, d_files, nf, infos, P(fs.tbase), n_table, flags, number, P(o_sizes), keys);
        CU(ctx, cudaGetLastError());
    }
    const unsigned grid_i = unsigned((n_ints > n_files ? n_ints : n_files) + 255) / 256;
    if (n_ints) {
        size_t tt = t_max;
        CU(ctx, cub::DeviceScan::ExclusiveSumByKey(stage + o_temp, tt, keys, P(o_sizes), P(o_offs), int(n_ints), cuda::std::equal_to<>(), st));
        caf_fit_kernel<<<unsigned((n_ints + 255) / 256), 256, 0, st>>>(d_files, infos, uint32_t(n_ints), P(o_sizes), keys, P(o_offs), P(fs.kept));
        CU(ctx, cudaGetLastError());
    }
    size_t tt = t_max;
    CU(ctx, cub::DeviceScan::ExclusiveSum(stage + o_temp, tt, P(fs.kept), P(fs.first), int(nf + 1), st));
    caf_write_kernel<<<grid_i, 256, 0, st>>>(d_files, infos, nf, uint32_t(n_ints), P(fs.ibase), P(o_sizes), keys, P(o_offs), P(fs.kept), P(fs.first),
                                             first_packet, packets, jobs, cap_packets);
    CU(ctx, cudaGetLastError());
    ctx->launches += 10;
    return SYMGPU_OK;
}

static_assert(sizeof(symgpu_caf_info) == 96, "record size is ABI");
