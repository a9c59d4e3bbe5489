// Element functions of IQArray.convert_to (IQArray.py:127-200): numpy's integer wrap-around and C's float -> int truncation.
// convert.cu converts whole captures with them; subexport.cu converts the I column to uint8 on the fly.
#pragma once
#include "common.cuh"

// numpy astype(float32 -> small int) is a C cast: on x86-64 cvttss2si to int32 (INT_MIN for NaN / out of range), low bits kept
__device__ __forceinline__ int32_t c_cast_i32(float v) {
    if (!(fabsf(v) < 2147483648.0f)) return (int32_t)0x80000000;
    return __float2int_rz(v);
}

template <typename S, typename D>
__device__ __forceinline__ D conv_one(S x);

// ---- from uint8 (IQArray.py:131-143)
template <> __device__ __forceinline__ int8_t conv_one<uint8_t, int8_t>(uint8_t x) { return (int8_t)(uint8_t)(x - 128u); }
template <> __device__ __forceinline__ int16_t conv_one<uint8_t, int16_t>(uint8_t x) { return (int16_t)(uint16_t)(((int)x - 128) << 8); }
template <> __device__ __forceinline__ uint16_t conv_one<uint8_t, uint16_t>(uint8_t x) { return (uint16_t)((unsigned)x << 8); }
template <> __device__ __forceinline__ float conv_one<uint8_t, float>(uint8_t x) { return __fadd_rn(__fmul_rn((float)x, 0.0078125f), -1.0f); }
// ---- from int8 (:145-153)
template <> __device__ __forceinline__ uint8_t conv_one<int8_t, uint8_t>(int8_t x) { return (uint8_t)((int)x + 128); }
template <> __device__ __forceinline__ int16_t conv_one<int8_t, int16_t>(int8_t x) { return (int16_t)(uint16_t)((int)x << 8); }
template <> __device__ __forceinline__ uint16_t conv_one<int8_t, uint16_t>(int8_t x) { return (uint16_t)(((int)x + 128) << 8); }
template <> __device__ __forceinline__ float conv_one<int8_t, float>(int8_t x) { return __fmul_rn((float)x, 0.0078125f); }
// ---- from uint16 (:155-170)
template <> __device__ __forceinline__ int8_t conv_one<uint16_t, int8_t>(uint16_t x) { return (int8_t)(((int16_t)(uint16_t)(x - 32768u)) >> 8); }
template <> __device__ __forceinline__ uint8_t conv_one<uint16_t, uint8_t>(uint16_t x) { return (uint8_t)(x >> 8); }
template <> __device__ __forceinline__ int16_t conv_one<uint16_t, int16_t>(uint16_t x) { return (int16_t)(uint16_t)(x - 32768u); }
template <> __device__ __forceinline__ float conv_one<uint16_t, float>(uint16_t x) { return __fadd_rn(__fmul_rn((float)x, 3.0517578125e-05f), -1.0f); }
// ---- from int16 (:172-183)
template <> __device__ __forceinline__ int8_t conv_one<int16_t, int8_t>(int16_t x) { return (int8_t)(x >> 8); }
template <> __device__ __forceinline__ uint8_t conv_one<int16_t, uint8_t>(int16_t x) { return (uint8_t)(((uint16_t)((int)x + 32768)) >> 8); }
template <> __device__ __forceinline__ uint16_t conv_one<int16_t, uint16_t>(int16_t x) { return (uint16_t)((int)x + 32768); }
template <> __device__ __forceinline__ float conv_one<int16_t, float>(int16_t x) { return __fmul_rn((float)x, 3.0517578125e-05f); }
// ---- from float32 (:185-200)
template <> __device__ __forceinline__ int8_t conv_one<float, int8_t>(float x) { return (int8_t)c_cast_i32(__fmul_rn(x, 127.0f)); }
template <> __device__ __forceinline__ uint8_t conv_one<float, uint8_t>(float x) { return (uint8_t)c_cast_i32(__fmul_rn(__fadd_rn(x, 1.0f), 127.0f)); }
template <> __device__ __forceinline__ int16_t conv_one<float, int16_t>(float x) { return (int16_t)c_cast_i32(__fmul_rn(x, 32767.0f)); }
template <> __device__ __forceinline__ uint16_t conv_one<float, uint16_t>(float x) { return (uint16_t)c_cast_i32(__fmul_rn(__fadd_rn(x, 1.0f), 32767.0f)); }
