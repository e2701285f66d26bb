// Device side of the MP3 entropy front-end (SURVEY §8f N1; parity in tests/test_mp3_entropy_gpu.py).
//
// One thread decodes one granule-channel with the very functions the CPU front-end runs (mp3_entropy.h), from the
// compacted main-data stream and the job table symgpu_mp3_entropy_plan builds from side information alone.  For 8192
// frames that is 32 768 independent decoders of ~300 symbols each: latency-bound serial work per thread, hidden by
// having every resident thread slot of the GPU busy.  What crosses PCIe is the compressed main data plus 64 bytes per
// job (~0.64 KB per frame) instead of 4.6 KB of quantised spectrum, and units + spectra are born in HBM where the
// synthesis kernel reads them.
#include <cuda_runtime.h>

#include <mutex>
#include <vector>

#include "ctx.h"
#include "mp3_entropy.h"
#include "pack_kernel.h"

using namespace symgpu_detail;
using symgpu::mp3e::GcJob;
using symgpu::mp3e::HuffSet;

namespace {

__global__ void __launch_bounds__(128) mp3_entropy_kernel(const uint8_t* __restrict__ md, const GcJob* __restrict__ jobs, uint32_t n_jobs, HuffSet hs,
                                                          symgpu_mp3_gc* __restrict__ units, int16_t* __restrict__ quant, uint32_t* __restrict__ failed) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_jobs) return;
    const GcJob j = jobs[k];
    if (symgpu::mp3e::decode_gc_job(j, md, hs, units + j.out_index, quant + size_t(j.out_index) * 576)) atomicOr(failed + (j.out_index >> 2), 1u);
}

// The flat Huffman tables, uploaded once per device.
struct DeviceLut {
    std::mutex mu;
    uint32_t* d[64] = {};
};
DeviceLut g_lut;

}  // namespace

cudaError_t symgpu::device_huffset(int device, HuffSet& out) {
    if (device < 0 || device >= 64) return cudaErrorInvalidDevice;
    size_t words = 0;
    const HuffSet& host = symgpu::mp3_huffset_host(&words);
    std::lock_guard<std::mutex> lock(g_lut.mu);
    if (!g_lut.d[device]) {
        uint32_t* p = nullptr;
        cudaError_t e = cudaMalloc(&p, words * sizeof(uint32_t));
        if (e != cudaSuccess) return e;
        e = cudaMemcpy(p, host.lut, words * sizeof(uint32_t), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) return cudaFree(p), e;
        g_lut.d[device] = p;
    }
    out = host;
    out.lut = g_lut.d[device];
    return cudaSuccess;
}

extern "C" symgpu_status symgpu_mp3_entropy_dev(symgpu_ctx* ctx, const uint8_t* d_md, size_t md_len, const symgpu_mp3_gc_job* d_jobs, size_t n_jobs,
                                                symgpu_mp3_gc* d_units, int16_t* d_quant, uint32_t* d_failed) {
    if (!ctx || (n_jobs && (!d_jobs || !d_units || !d_quant || !d_failed)) || (!d_md && md_len) || n_jobs > 0xffffffffull) return SYMGPU_ERR_ARG;
    if (n_jobs == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    HuffSet hs;
    CU(ctx, symgpu::device_huffset(ctx->device, hs));
    const unsigned block = 128, grid = unsigned((n_jobs + block - 1) / block);
    mp3_entropy_kernel<<<grid, block, 0, ctx->stream>>>(d_md, reinterpret_cast<const GcJob*>(d_jobs), uint32_t(n_jobs), hs, d_units, d_quant, d_failed);
    ctx->launches += 1;
    CU(ctx, cudaGetLastError());
    return SYMGPU_OK;
}

// File bytes in host memory -> planar f32 PCM in host memory, entropy decode and synthesis both on the device.
extern "C" symgpu_status symgpu_mp3_decode_files_host(symgpu_ctx* ctx, const symgpu_mp3_file* files, uint32_t n_files, float* pcm, size_t pcm_frames_cap,
                                                      uint32_t* good_per_file, uint32_t* frame_of, uint32_t* n_rounds) {
    if (!ctx || !files || !n_files || !pcm || !good_per_file || !frame_of) return SYMGPU_ERR_ARG;
    DeviceGuard guard(ctx->device);
    size_t total_packets = 0, total_bytes = 0;
    for (uint32_t f = 0; f < n_files; ++f) {
        if (!files[f].data || (files[f].n_packets && !files[f].packets) || files[f].stream >= ctx->n_mp3_streams) return SYMGPU_ERR_ARG;
        total_packets += files[f].n_packets;
        for (size_t i = 0; i < files[f].n_packets; ++i) total_bytes += files[f].packets[i].size;
    }
    if (total_packets > pcm_frames_cap) return SYMGPU_ERR_LIMIT;
    std::vector<uint8_t> md(total_bytes + 8), bad(total_packets, 0);
    std::vector<GcJob> jobs(total_packets * 4);
    std::vector<symgpu_mp3_run> runs(n_files);
    std::vector<uint32_t> failed(total_packets + 1);
    uint32_t rounds = 0;
    size_t n_frames = 0, md_len = 0;
    for (;;) {
        ++rounds;
        n_frames = md_len = 0;
        size_t packet_base = 0;
        bool again = false;
        for (uint32_t f = 0; f < n_files; ++f) {
            size_t len = 0, good = 0;
            symgpu_mp3_frame_info info{};
            const symgpu_status s = symgpu_mp3_entropy_plan(files[f].data, files[f].n, files[f].packets, files[f].n_packets, bad.data() + packet_base,
                                                            md.data() + md_len, md.size() - md_len, &len, reinterpret_cast<symgpu_mp3_gc_job*>(jobs.data() + n_frames * 4),
                                                            frame_of + n_frames, &good, &info);
            if (s != SYMGPU_OK) return s;
            for (size_t k = n_frames * 4; k < (n_frames + good) * 4; ++k) jobs[k].seg_begin += md_len, jobs[k].out_index += uint32_t(n_frames * 4);
            // a joint-stereo pair must share its window sequence (stereo.rs:503-505): the reference refuses such a frame after
            // reading it; it is left out here (deviation: a first granule the reference had already synthesised is lost with it)
            for (size_t g = 0; g < good; ++g)
                for (int gr = 0; gr < 2; ++gr) {
                    const GcJob &a = jobs[(n_frames + g) * 4 + gr * 2], &b = jobs[(n_frames + g) * 4 + gr * 2 + 1];
                    if (a.kind == symgpu::mp3e::kJobMute || b.kind == symgpu::mp3e::kJobMute) continue;
                    if (!(a.unit_flags & (SYMGPU_MP3_F_MID_SIDE | SYMGPU_MP3_F_INTENSITY))) continue;
                    if (a.side.block_type != b.side.block_type || (a.side.block_type == SYMGPU_MP3_SHORT && a.side.mixed != b.side.mixed))
                        bad[packet_base + frame_of[n_frames + g]] = 2, again = true;
                }
            runs[f] = symgpu_mp3_run{files[f].stream, uint32_t(n_frames), uint32_t(good), info.granules, info.channels, 0};
            good_per_file[f] = uint32_t(good);
            n_frames += good, md_len += len, packet_base += files[f].n_packets;
        }
        if (again) continue;
        if (n_frames == 0) break;
        const size_t unit_bytes = n_frames * 4 * sizeof(symgpu_mp3_gc), quant_bytes = n_frames * 4 * 576 * sizeof(int16_t), spec_bytes = 2 * quant_bytes;
        const size_t md_pad = (md_len + 255) & ~size_t(255), job_bytes = n_frames * 4 * sizeof(GcJob), fail_bytes = (n_frames * 4 + 255) & ~size_t(255);
        const symgpu_status st = ensure_stage(ctx, spec_bytes * 2 + quant_bytes + unit_bytes + md_pad + job_bytes + fail_bytes);
        if (st != SYMGPU_OK) return st;
        char* base = static_cast<char*>(ctx->d_stage);
        float* d_spec = reinterpret_cast<float*>(base);
        float* d_pcm = reinterpret_cast<float*>(base + spec_bytes);
        int16_t* d_quant = reinterpret_cast<int16_t*>(base + 2 * spec_bytes);
        symgpu_mp3_gc* d_units = reinterpret_cast<symgpu_mp3_gc*>(base + 2 * spec_bytes + quant_bytes);
        uint8_t* d_md = reinterpret_cast<uint8_t*>(base + 2 * spec_bytes + quant_bytes + unit_bytes);
        GcJob* d_jobs = reinterpret_cast<GcJob*>(d_md + md_pad);
        uint32_t* d_failed = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(d_jobs) + job_bytes);
        CU(ctx, cudaMemcpyAsync(d_md, md.data(), md_len, cudaMemcpyHostToDevice, ctx->stream));
        CU(ctx, cudaMemcpyAsync(d_jobs, jobs.data(), job_bytes, cudaMemcpyHostToDevice, ctx->stream));
        CU(ctx, cudaMemsetAsync(d_failed, 0, n_frames * sizeof(uint32_t), ctx->stream));
        symgpu_status s = symgpu_mp3_entropy_dev(ctx, d_md, md_len, reinterpret_cast<const symgpu_mp3_gc_job*>(d_jobs), n_frames * 4, d_units, d_quant, d_failed);
        if (s != SYMGPU_OK) return s;
        CU(ctx, cudaMemcpyAsync(failed.data(), d_failed, n_frames * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
        CU(ctx, cudaStreamSynchronize(ctx->stream));
        // the first failure of each file is certain; the frames behind it were planned with a reservoir the reference empties
        packet_base = 0;
        size_t frame_base = 0;
        for (uint32_t f = 0; f < n_files; ++f) {
            for (size_t g = 0; g < good_per_file[f]; ++g)
                if (failed[frame_base + g]) {
                    bad[packet_base + frame_of[frame_base + g]] = 1, again = true;
                    break;
                }
            frame_base += good_per_file[f], packet_base += files[f].n_packets;
        }
        if (again) continue;
        bool partial = false;
        for (uint32_t f = 0; f < n_files; ++f) partial |= good_per_file[f] && (runs[f].granules_per_frame == 1 || runs[f].channels == 1);
        if (partial) CU(ctx, cudaMemsetAsync(d_pcm, 0, spec_bytes, ctx->stream));
        ctx->launches += 1;
        CU(ctx, symgpu::dequant_launch(d_quant, d_spec, n_frames * SYMGPU_MP3_FRAME_FLOATS, ctx->d_mp3_tab->pow43, ctx->stream));
        std::vector<symgpu_mp3_run> live;
        for (uint32_t f = 0; f < n_files; ++f)
            if (good_per_file[f]) live.push_back(runs[f]);
        s = symgpu_mp3_synth_dev(ctx, d_units, d_spec, live.data(), uint32_t(live.size()), uint32_t(n_frames), d_pcm);
        if (s != SYMGPU_OK) return s;
        CU(ctx, cudaMemcpyAsync(pcm, d_pcm, spec_bytes, cudaMemcpyDeviceToHost, ctx->stream));
        CU(ctx, cudaStreamSynchronize(ctx->stream));
        break;
    }
    if (n_rounds) *n_rounds = rounds;
    return SYMGPU_OK;
}
