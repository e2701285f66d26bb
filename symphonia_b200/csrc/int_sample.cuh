// The caller's sample format from a decoder's 32-bit-scaled integer sample, shared by the FLAC and ALAC interleaving kernels.
#pragma once
#include <cstdint>

#include "../../include/symgpu.h"

// The reference's FromSample<i32> (symphonia-core/src/audio/conv.rs:516-531) applied to the decoder's 32-bit-scaled sample: what
// copy_to_slice_interleaved::<S> makes of the FLAC decoder's AudioBuffer<i32>.  Every conversion is exact; f32 is the double
// quotient rounded once.
template <int Format>
struct FlacSample;
template <>
struct FlacSample<SYMGPU_FMT_S32> {
    using type = int32_t;
    static __device__ __forceinline__ type from(int32_t s) { return s; }
};
template <>
struct FlacSample<SYMGPU_FMT_S24> {
    using type = int32_t;  // an s24 sample in an int32, as the f32 output stage stores it
    static __device__ __forceinline__ type from(int32_t s) { return s >> 8; }
};
template <>
struct FlacSample<SYMGPU_FMT_S16> {
    using type = int16_t;
    static __device__ __forceinline__ type from(int32_t s) { return int16_t(s >> 16); }
};
template <>
struct FlacSample<SYMGPU_FMT_U8> {
    using type = uint8_t;
    static __device__ __forceinline__ type from(int32_t s) { return uint8_t((uint32_t(s) + 0x80000000u) >> 24); }
};
template <>
struct FlacSample<SYMGPU_FMT_F32> {
    using type = float;
    static __device__ __forceinline__ type from(int32_t s) { return __double2float_rn(double(s) / 2147483648.0); }
};
