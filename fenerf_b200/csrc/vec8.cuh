// Eight consecutive stream elements (fp16 or fp32) as one vector load / store: the backward's streams.  Internal.
#pragma once
#include <cuda_fp16.h>

namespace fn {

template <typename T> struct Vec8;
template <> struct Vec8<__half> {
    __align__(16) __half v[8];
    __device__ __forceinline__ void set(int i, float x) { v[i] = __float2half_rn(x); }
    __device__ __forceinline__ float get(int i) const { return __half2float(v[i]); }
    __device__ __forceinline__ void load(const __half* p) { *reinterpret_cast<uint4*>(v) = *reinterpret_cast<const uint4*>(p); }
    __device__ __forceinline__ void store(__half* p) const { *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(v); }
};
template <> struct Vec8<float> {
    __align__(16) float v[8];
    __device__ __forceinline__ void set(int i, float x) { v[i] = x; }
    __device__ __forceinline__ float get(int i) const { return v[i]; }
    __device__ __forceinline__ void load(const float* p) {
        reinterpret_cast<float4*>(v)[0] = reinterpret_cast<const float4*>(p)[0];
        reinterpret_cast<float4*>(v)[1] = reinterpret_cast<const float4*>(p)[1];
    }
    __device__ __forceinline__ void store(float* p) const {
        reinterpret_cast<float4*>(p)[0] = reinterpret_cast<const float4*>(v)[0];
        reinterpret_cast<float4*>(p)[1] = reinterpret_cast<const float4*>(v)[1];
    }
};

}  // namespace fn
