// ORACLE (test infrastructure, NOT product code): CPU restatement of the reference's conversions FROM an i32 sample, which is what
// copy_to_slice_interleaved::<S> applies to the FLAC decoder's AudioBuffer<i32> (samples scaled to 32 bits).
//
//   FromSample<i32> for u8, i16, i24, i32, f32   symphonia-core/src/audio/conv.rs:516-531
//   Rust `>>` on i32 is arithmetic, on u32 logical; `as` between integer types truncates; `as f32` from f64 rounds to nearest even.
//
// PARITY PINNING: tests/test_flac_convert.py replays the reference's own assertions (conv.rs:709-711 u8, :924-926 i16,
// :967-969 i24: i32::MAX -> MAX, 0 -> MID, i32::MIN -> MIN; :1096-1098 f32: -> 2147483647 / 2147483648 as f32, 0, -1).
//
// Kept apart from oracle_conv.cpp (the conversions from f32), which stays as it is.
#include <cstddef>
#include <cstdint>

#include "../include/symgpu.h"

extern "C" {

uint8_t oracle_conv_i32_u8(int32_t s) { return (uint8_t)(((uint32_t)s + 0x80000000u) >> 24); }
int16_t oracle_conv_i32_s16(int32_t s) { return (int16_t)(s >> 16); }
int32_t oracle_conv_i32_s24(int32_t s) { return s >> 8; }
float oracle_conv_i32_f32(int32_t s) { return (float)((double)s / 2147483648.0); }

// n samples of `in` as `format` (SYMGPU_FMT_*) into `out`; s24 in an int32 as oracle_pcm_pack stores it.  1 for an unknown format.
int oracle_conv_i32_pack(const int32_t* in, size_t n, int format, void* out) {
    for (size_t i = 0; i < n; ++i) {
        switch (format) {
        case SYMGPU_FMT_F32: static_cast<float*>(out)[i] = oracle_conv_i32_f32(in[i]); break;
        case SYMGPU_FMT_S16: static_cast<int16_t*>(out)[i] = oracle_conv_i32_s16(in[i]); break;
        case SYMGPU_FMT_S24: static_cast<int32_t*>(out)[i] = oracle_conv_i32_s24(in[i]); break;
        case SYMGPU_FMT_S32: static_cast<int32_t*>(out)[i] = in[i]; break;
        case SYMGPU_FMT_U8: static_cast<uint8_t*>(out)[i] = oracle_conv_i32_u8(in[i]); break;
        default: return 1;
        }
    }
    return 0;
}
}
