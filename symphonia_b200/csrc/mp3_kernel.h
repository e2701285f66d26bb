// Host <-> kernel interface of the fused MP3 synthesis kernel (mp3_kernel.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/symgpu.h"
#include "tables.h"

namespace symgpu {

// Granules per tile and warps per CTA.  One persistent CTA of 16 warps per SM (4 per scheduler: 5
// would cap the kernel at 96 registers because registers are partitioned per scheduler).  A CTA walks a
// CHAIN of consecutive tiles of the same stream and carries overlap + polyphase history from one tile
// to the next through shared memory, so only the first tile of a chain that starts inside a run pays
// the 2-granule halo.  Short runs (a few frames per stream, the serving shape) are packed several to a
// group, so that all 16 warps have a granule job.  16 granule jobs in the hybrid phase; 288 time slots
// x 2 channels = 576 DCT jobs for 512 threads; 288 slots = 18 per warp in the window phase.  Shared
// memory: 432 XT rows (114 KB) + the TMA stage of 16 granules (74 KB) + carry (8 KB) + scratch.
#ifndef SYMGPU_MP3_T
#define SYMGPU_MP3_T 16
#define SYMGPU_MP3_NW 16
#endif
constexpr int kMp3TileGranules = SYMGPU_MP3_T;
constexpr int kMp3Warps = SYMGPU_MP3_NW;

// kTileLoadState / kTileStoreState: the tile starts / ends a run and exchanges state with HBM.
// kTileCarryIn / kTileCarryOut: the tile continues / is continued by the neighbouring tile of the same
// CTA's chain and exchanges state through shared memory.  A tile with neither input flag recomputes a
// 2-granule halo (and then holds at most kMp3TileGranules granules with NW >= n + 2).
// kTileGroupEnd: the CTA processes its chain in GROUPS of consecutive tiles (pieces of possibly different
// streams) that together hold at most kMp3Warps granule jobs and kMp3GroupRegions XT regions; the flag marks
// a group's last tile.  kTileCarryIn only on a group's first tile, kTileCarryOut only on its last.
enum : uint8_t { kTileLoadState = 1, kTileStoreState = 2, kTileCarryIn = 4, kTileCarryOut = 8, kTileGroupEnd = 16 };
constexpr int kMp3GroupTiles = 8;    // pieces per group
constexpr int kMp3GroupRegions = 24; // XT regions per group: one history region + one per granule, per piece

// One step of a CTA's work: `n_granules` consecutive granules of one stream.  Built on the host from
// the caller's runs (symgpu.cpp: build_plan).
struct Mp3Tile {
    uint32_t first_frame; // batch frame index holding the tile's first granule
    uint32_t stream;      // per-stream state slot
    uint16_t first_gr;    // granule-in-frame of the tile's first granule
    uint16_t n_granules;  // 1..kMp3TileGranules
    uint8_t gpf;          // granules per frame: 2 (MPEG-1) or 1 (MPEG-2 / 2.5)
    uint8_t n_ch;         // 1 or 2
    uint8_t flags;        // kTileLoadState | kTileStoreState
    uint8_t pad;
};
static_assert(sizeof(Mp3Tile) == 16, "Mp3Tile is 16 bytes");

// Persistent per-stream state in HBM: what Layer3.overlap and Layer3.synthesis hold in the
// reference (layer3/mod.rs:254-259, synthesis.rs:145-154), in feed-forward form: instead of the
// 16x64 v_vec FIFO we keep the last 15 DCT-32 output vectors (both channels interleaved), from
// which every FIFO entry the next 15 slots can read is a copy or a negation.
struct Mp3StreamState {
    float overlap[2][32][18];
    float2 dhist[15][32];
};

struct Mp3Args {
    const symgpu_mp3_gc* units;
    const float* spectra;
    float* pcm;
    const uint32_t* cta_first; // [n_ctas + 1]: CTA b walks tiles cta_first[b] .. cta_first[b + 1] - 1 in order
    const Mp3Tile* tiles;
    int n_tiles;
    int n_ctas;
    int multi_tile_groups;     // some group of the plan holds more than one tile (see kTileGroupEnd)
    Mp3StreamState* states; // [n_streams][2] double-buffered, see gen
    uint32_t* gen;          // [n_streams] state generation; buffer (gen & 1) is current
    unsigned* done;         // retired-CTA counter (self-resetting)
    const Mp3Tables* tab;
};

// MPEG Layer I / II polyphase synthesis (mpa12_synth_kernel): tiles are whole frames of one stream, `n_granules`
// counts frames; per-stream state = Mp3StreamState.dhist (the overlap part is unused).
struct Mpa12Args {
    const float* subbands;     // [n_frames][2][32][n_slots]: samples[ch][n_slots * sb + s] of the layer decoders
    float* pcm;                // [n_frames][2][1152], the first 32 * n_slots samples of a plane are written
    const uint32_t* cta_first;
    const Mp3Tile* tiles;
    int n_tiles;
    int n_ctas;
    int n_slots;               // 12 (Layer I) or 36 (Layer II)
    Mp3StreamState* states;
    uint32_t* gen;
    unsigned* done;
    const Mp3Tables* tab;
};
cudaError_t mpa12_launch(const Mpa12Args& a, cudaStream_t stream);
int mpa12_tile_frames(int n_slots); // frames per tile

cudaError_t mp3_upload_const(const Mp3Tables& t, cudaStream_t stream);
cudaError_t mp3_launch(const Mp3Args& a, cudaStream_t stream);
int mp3_tile_granules();
int mp3_halo_tile_granules(); // limit for a tile that recomputes its halo (two warps go to the halo granules)
int mp3_cta_warps();           // warps per CTA = granule jobs per group
// Persistent grid size of the kernel on the current device (SM count x resident CTAs), <= 0 on error.
int mp3_grid_size(cudaError_t* err);

// ---- second-generation Layer III kernel (mp3_kernel_v2.cu): warp-autonomous, channel pairs in float2 ----
// A warp owns a SHARE of the batch's granules (a list of Mp3Tile segments, walked in order); share s runs on
// warp s / grid of CTA s % grid.  Tile flags: kTileLoadState (the segment starts its run: state from HBM),
// kTileStoreState (it ends its run: state to HBM), kTileCarryIn / kTileCarryOut (the segment continues / is
// continued by the neighbouring segment of the same share: the state simply stays in the warp); a segment with
// neither input flag recomputes a 2-granule halo.
#ifndef SYMGPU_MP3_V2_NW
#define SYMGPU_MP3_V2_NW 12
#endif
constexpr int kMp3V2Warps = SYMGPU_MP3_V2_NW;
struct Mp3V2Args {
    const symgpu_mp3_gc* units;
    const float* spectra;
    float* pcm;
    const uint32_t* first; // [n_shares + 1]: share s walks tiles first[s] .. first[s + 1] - 1 in order
    const Mp3Tile* tiles;
    int n_tiles;
    int n_shares;
    Mp3StreamState* states; // [n_streams][2] double-buffered, see gen
    uint32_t* gen;          // [n_streams] state generation; buffer (gen & 1) is current
    unsigned* done;         // retired-CTA counter (self-resetting)
    const Mp3Tables* tab;
};
cudaError_t mp3v2_upload_const(const Mp3Tables& t, cudaStream_t stream);
cudaError_t mp3v2_launch(const Mp3V2Args& a, int n_ctas, cudaStream_t stream, bool short_runs);
int mp3v2_cta_warps();
int mp3v2_ctas_per_sm();
bool mp3v2_set_variant(int nw, int mode); // experiments: warps per CTA, variant bits (mp3_kernel_v2.cu)
int mp3v2_sm_count(cudaError_t* err); // SMs of the current device (= CTAs of a full launch), <= 0 on error

} // namespace symgpu
