// 16-bit storage types of the activations: fp16, and bf16 (fp32's exponent range: the VAE decoder's path for weights
// whose activations overflow fp16).  Conversions to / from fp32 are overloaded on the storage type, so one kernel
// template serves both; the fp16 instantiations compile to the same conversions the fp16-only kernels used.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace omg {

template <typename T>
struct Pair;
template <>
struct Pair<__half> {
    using type = __half2;
};
template <>
struct Pair<__nv_bfloat16> {
    using type = __nv_bfloat162;
};
template <typename T>
using pair_t = typename Pair<T>::type;

__device__ __forceinline__ float to_f32(__half x) { return __half2float(x); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 x) { return __bfloat162float(x); }
__device__ __forceinline__ float2 to_f32x2(__half2 x) { return __half22float2(x); }
// bf16 -> fp32 is exact (the high half of the fp32 word): plain integer ops, which the compiler can rematerialise
// instead of keeping converted copies live (cuda_bf16's conversion is inline asm)
__device__ __forceinline__ float2 to_f32x2(__nv_bfloat162 x) {
    const uint32_t u = *reinterpret_cast<const uint32_t*>(&x);
    return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}

// round-to-nearest-even pair (a, b) in the storage type T
template <typename T>
__device__ __forceinline__ pair_t<T> from_f32x2(float a, float b);
template <>
__device__ __forceinline__ __half2 from_f32x2<__half>(float a, float b) { return __floats2half2_rn(a, b); }
template <>
__device__ __forceinline__ __nv_bfloat162 from_f32x2<__nv_bfloat16>(float a, float b) { return __floats2bfloat162_rn(a, b); }

}  // namespace omg
