// rsb_dtype.cuh -- the 16-bit element types the reader kernels and their GEMM are instantiated for: __half (fp16, the
// default) and __nv_bfloat16 (bf16, the reference's reader dtype).  Every conversion to the element type rounds to
// nearest even, as torch does when it writes a half or bfloat16 tensor from its fp32 arithmetic.
#ifndef RSB_DTYPE_CUH_
#define RSB_DTYPE_CUH_

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace rsbdt {

template <typename T> struct pair_of;
template <> struct pair_of<__half> { using type = __half2; };
template <> struct pair_of<__nv_bfloat16> { using type = __nv_bfloat162; };
template <typename T> using pair_t = typename pair_of<T>::type;

__device__ __forceinline__ float to_f(__half x) { return __half2float(x); }
__device__ __forceinline__ float to_f(__nv_bfloat16 x) { return __bfloat162float(x); }
__device__ __forceinline__ float2 to_f2(__half2 x) { return __half22float2(x); }
__device__ __forceinline__ float2 to_f2(__nv_bfloat162 x) { return __bfloat1622float2(x); }

template <typename T> __device__ __forceinline__ T from_f(float x);
template <> __device__ __forceinline__ __half from_f<__half>(float x) { return __float2half_rn(x); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }

template <typename T> __device__ __forceinline__ pair_t<T> from_f2(float lo, float hi);
template <> __device__ __forceinline__ __half2 from_f2<__half>(float lo, float hi) { return __floats2half2_rn(lo, hi); }
template <> __device__ __forceinline__ __nv_bfloat162 from_f2<__nv_bfloat16>(float lo, float hi) {
    return __floats2bfloat162_rn(lo, hi);
}

// the bits of the pair (lo, hi) rounded to T, as a 32-bit mma / store operand
template <typename T> __device__ __forceinline__ uint32_t pair_bits(float lo, float hi) {
    const pair_t<T> h = from_f2<T>(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}

}  // namespace rsbdt
#endif
