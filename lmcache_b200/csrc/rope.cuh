// rope.cuh -- the rotation arithmetic of the rope shift (rope.cu), shared with the mover's fused gather-and-turn
// (mover.cu, b200kv_pack_chunks_rope): one definition, so a key turned while it is packed holds exactly the bits the
// shift gives when it turns the packed row.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200kv {

template <class E> __device__ __forceinline__ float to_f(E v);
template <> __device__ __forceinline__ float to_f<__nv_bfloat16_raw>(__nv_bfloat16_raw v) {
    return __uint_as_float((uint32_t)v.x << 16);
}
template <> __device__ __forceinline__ float to_f<__half_raw>(__half_raw v) { return __half2float(__half(v)); }
template <class E> __device__ __forceinline__ E from_f(float f);
template <> __device__ __forceinline__ __nv_bfloat16_raw from_f<__nv_bfloat16_raw>(float f) {
    return __nv_bfloat16_raw(__float2bfloat16_rn(f));
}
template <> __device__ __forceinline__ __half_raw from_f<__half_raw>(float f) { return __half_raw(__float2half_rn(f)); }

// (a, b) <- (a cos - b sin, b cos + a sin), in fp32, rounded once to E
template <class E>
__device__ __forceinline__ void rotate(E& a, E& b, float2 t) {
    const float x = to_f(a), y = to_f(b);
    a = from_f<E>(fmaf(x, t.x, -y * t.y));
    b = from_f<E>(fmaf(y, t.x, x * t.y));
}

// The gather side turns one element at a time out of an unchanged source: channel c (relative to the rotary offset, in
// [0, 2 half)) pairs with rope_partner(c), and the element keeps its own half of rotate()'s result.
__device__ __forceinline__ int rope_partner(int c, int half, bool neox) {
    return neox ? (c < half ? c + half : c - half) : (c ^ 1);
}

template <class E>
__device__ __forceinline__ E rope_turn_one(E own, E partner, int c, const float2* t, int half, bool neox) {
    const bool first = neox ? c < half : (c & 1) == 0;           // own is the pair's a
    const int j = neox ? (first ? c : c - half) : c >> 1;
    E a = first ? own : partner, b = first ? partner : own;
    rotate(a, b, __ldg(t + j));
    return first ? a : b;
}

// Turns v, channels c0 .. c0 + N - 1 of one key row whose channel 0 is at `row` (read for the partners; never written),
// by the table row t.  N > 1: 16 bytes, wholly inside or outside [offset, offset + 2 half), with offset and the
// pairing 16-byte aligned (the caller's launch rule), so neox partners are one aligned vector half a rotary range
// away and gptj partners lie in v itself.
template <class E, int N>
__device__ __forceinline__ void rope_turn_vec(E* v, const E* row, int c0, const float2* t, int half, int offset,
                                              bool neox) {
    const int c = c0 - offset;
    if (c < 0 || c >= 2 * half) return;
    E p[N];
    if (N == 1) {
        p[0] = row[offset + rope_partner(c, half, neox)];
    } else if (neox) {
        union { uint4 q; E e[N]; } u;
        u.q = *reinterpret_cast<const uint4*>(row + offset + rope_partner(c, half, true));
#pragma unroll
        for (int k = 0; k < N; ++k) p[k] = u.e[k];
    } else {
#pragma unroll
        for (int k = 0; k < N; ++k) p[k] = v[k ^ 1];
    }
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] = rope_turn_one(v[k], p[k], c + k, t, half, neox);
}

}  // namespace b200kv
