// jsgpu_scan.cuh — the library's device prefix scans: a warp scan and a CTA scan that continues from a carry, over any T made
// of 32-bit words and any associative op (op(a, b): a, then b) with identity id.
#pragma once
#include <cstdint>
#include <cstring>

template <typename T, typename F>
__device__ __forceinline__ T js_shfl_words(T x, F f)       // f (a shuffle) applied to each 32-bit word of x
{
    static_assert(sizeof(T) % 4 == 0, "shuffled as 32-bit words");
    uint32_t w[sizeof(T) / 4];
    memcpy(w, &x, sizeof(T));
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 4); i++) w[i] = f(w[i]);
    memcpy(&x, w, sizeof(T));
    return x;
}

// Over lanes 0 .. W-1 (W a power of two; the whole warp calls): returns the exclusive prefix of v, id in lane 0, and sets
// `inc` to the inclusive one.
template <int W = 32, typename T, typename Op>
__device__ __forceinline__ T js_warp_scan(T v, T id, Op op, T& inc)
{
    const uint32_t lane = threadIdx.x & 31;
    inc = v;
#pragma unroll
    for (int d = 1; d < W; d <<= 1) {
        const T o = js_shfl_words(inc, [d](uint32_t x) { return __shfl_up_sync(0xffffffffu, x, d); });
        if (lane >= (uint32_t)d) inc = op(o, inc);
    }
    const T ex = js_shfl_words(inc, [](uint32_t x) { return __shfl_up_sync(0xffffffffu, x, 1); });
    return lane ? ex : id;
}
__device__ __forceinline__ uint32_t js_add(uint32_t a, uint32_t b) { return a + b; }

// Over a CTA of NT threads, after `carry` (the same in every thread): returns carry op (the values of the threads before
// this one) and advances `carry` by the whole CTA's.  s_w: NT / 32 elements of shared memory (NT / 32 + 1 above 16 warps),
// free again at the next call.  Up to 16 warps, every thread combines the warp totals itself, which takes no barrier after
// that of the totals.  With more, 32 serial steps in every thread would cost more than a barrier: warp 0 scans the totals
// for all.
template <int NT, typename T, typename Op>
__device__ __forceinline__ T js_block_scan(T v, T id, Op op, T& carry, T* s_w)
{
    constexpr uint32_t NW = NT / 32;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T inc, before = carry;
    const T ex = js_warp_scan(v, id, op, inc);
    __syncthreads();                                          // the previous call is done with s_w
    if (lane == 31) s_w[warp] = inc;
    __syncthreads();
    if constexpr (NW <= 16) {
#pragma unroll
        for (uint32_t k = 0; k < NW; k++) {
            const T w = s_w[k];
            if (k < warp) before = op(before, w);
            carry = op(carry, w);
        }
    } else {
        if (warp == 0) {                                      // s_w[w] becomes carry op the warps before w, s_w[NW] the new carry
            const T wex = js_warp_scan<NW>(lane < NW ? s_w[lane] : id, id, op, inc);
            __syncwarp();
            if (lane < NW) s_w[lane] = op(carry, wex);
            if (lane == NW - 1) s_w[NW] = op(carry, inc);
        }
        __syncthreads();
        before = s_w[warp];
        carry = s_w[NW];
    }
    return op(before, ex);
}
