// devsim.cu -- test-only device build of ac_core.cuh: the rANS encoder step the kernels run (rans_put), swept over
// every (freq, quotient) pair it can meet and compared with integer division.  Not part of the product library.
//
// Why two states per pair cover all 2^47 pairs (x, f) with x < f << 16:
//   rans_put's quotient estimate is  F2I.RZ( I2F.RZ(x) * c ),  c = rcp(f) * 0.99999952 > 0 fixed by f.  Each of the three
//   operations is monotone non-decreasing in x, so the estimate is.  The true quotient is constant on a bucket
//   [q f, q f + f).  If the step is right at x = q f the estimate there is >= q - 1, and if it is right at
//   x = q f + f - 1 the estimate there is <= q (an estimate of q + 1 or more, or q - 2 or less, survives the single
//   fix-up and yields a wrong state); by monotonicity the estimate is q - 1 or q on the whole bucket, which the fix-up
//   makes exact.  So "right at both ends of every bucket" is "right everywhere": 2 * 65535 * 65535 = 8.6e9 steps.
//   The states below 2^16 (q f < 2^16) cannot occur in a stream; they are swept all the same.
//   The push branch (the state sheds its low halfword first) does not touch the division: it is run on the states
//   (x << 16) | h for the x < 2^16 of the sweep, into a two-halfword row per thread, at both values of the row index.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../lmcache_b200/csrc/ac_core.cuh"

namespace {

using namespace b200kv;

constexpr int kThreads = 256;
constexpr int kQBlocks = 65536 / kThreads;    // blockIdx.x * 256 + threadIdx.x = q (q = 0 idles)
constexpr int kFRows = 264;                   // blockIdx.y strides over f

struct Tally {
    unsigned long long steps, bad, fixups, pushes, first;   // first: smallest (f << 18 | q << 2 | which) that went wrong
};

// the estimate alone, as rans_put forms it: only to COUNT the fix-ups (rans_put does not report them)
__device__ __forceinline__ uint32_t estimate(uint32_t x, uint32_t f) {
    float rc;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(__uint2float_rn(f)));
    return __float2uint_rz(__uint2float_rz(x) * (rc * 0.99999952316284179688f));
}

// one step from state x; which: 0 / 1 the ends of the bucket, 2 / 3 the same behind a push.  Returns got != want.
__device__ __forceinline__ bool one(uint32_t f, uint32_t q, uint32_t which, uint16_t* row, uint32_t* got, uint32_t* want,
                                    uint32_t* xin) {
    const uint32_t r = (which & 1u) ? f - 1u : 0u;
    const uint32_t start = (which & 1u) ? 65536u - f : (q * 40503u) % (65537u - f);     // start + f <= 65536
    uint32_t x = q * f + r;
    const uint32_t h = (q * 2654435761u + f) >> 16;
    int32_t nk = (which & 2u) ? -(int32_t)(q & 1u) : 0;
    const int32_t nk0 = nk;
    if (which & 2u) { x = (x << 16) | h; row[0] = 0xdeadu; row[1] = 0xbeefu; }
    *xin = x;
    rans_put(x, nk, row + 2, start, f);
    *got = x;
    *want = (q << 16) + r + start;
    bool bad = x != *want;
    if (which & 2u) {
        // halfword number k lands at row_end + 2 nk - 2 bytes: row[1] for nk = 0, row[0] for nk = -1; the other stays
        const volatile uint16_t* v = row;
        const uint32_t at = nk0 == 0 ? 1u : 0u;
        bad = bad || nk != nk0 - 1 || v[at] != (uint16_t)h || v[1u - at] != (at ? 0xdeadu : 0xbeefu);
    } else {
        bad = bad || nk != 0;
    }
    return bad;
}

__global__ void __launch_bounds__(kThreads) sweep_kernel(uint16_t* scratch, Tally* tally) {
    const uint32_t q = blockIdx.x * kThreads + threadIdx.x;
    uint16_t* row = scratch + 2ull * ((unsigned long long)blockIdx.y * 65536ull + q);
    unsigned long long steps = 0, bad = 0, fix = 0, pushes = 0, first = ~0ull;
    if (q != 0u) {
        for (uint32_t f = 1u + blockIdx.y; f < 65536u; f += gridDim.y) {
            const bool small = q * f + f - 1u < 65536u;
            for (uint32_t which = 0; which < (small ? 4u : 2u); ++which) {
                uint32_t got, want, xin;
                const bool b = one(f, q, which, row, &got, &want, &xin);
                ++steps;
                pushes += which >> 1;
                if (which < 2u) fix += estimate(xin, f) != q ? 1u : 0u;
                if (b) {
                    ++bad;
                    const unsigned long long key = ((unsigned long long)f << 18) | ((unsigned long long)q << 2) | which;
                    first = key < first ? key : first;
                }
            }
        }
    }
    // one atomic per warp and counter
    for (int o = 16; o > 0; o >>= 1) {
        steps += __shfl_down_sync(0xffffffffu, steps, o);
        bad += __shfl_down_sync(0xffffffffu, bad, o);
        fix += __shfl_down_sync(0xffffffffu, fix, o);
        pushes += __shfl_down_sync(0xffffffffu, pushes, o);
        const unsigned long long other = __shfl_down_sync(0xffffffffu, first, o);
        first = other < first ? other : first;
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&tally->steps, steps);
        atomicAdd(&tally->bad, bad);
        atomicAdd(&tally->fixups, fix);
        atomicAdd(&tally->pushes, pushes);
        atomicMin(&tally->first, first);
    }
}

// the first wrong step again, alone, to report its states
__global__ void replay_kernel(uint16_t* scratch, unsigned long long key, uint32_t* out) {
    uint32_t got, want, xin;
    one((uint32_t)(key >> 18), (uint32_t)(key >> 2) & 0xffffu, (uint32_t)key & 3u, scratch, &got, &want, &xin);
    out[0] = xin; out[1] = got; out[2] = want;
    out[3] = estimate(((uint32_t)key & 2u) ? xin >> 16 : xin, (uint32_t)(key >> 18));
}

}  // namespace

// out[0] steps run, [1] wrong steps, [2] steps of the plain sweep that took the fix-up, [3] steps behind a push,
// [4..9] the first wrong step: f, q, which (0 x = q f, 1 x = q f + f - 1, 2 / 3 the same behind a push), x, state got,
// state wanted, [10] its quotient estimate, [11] kernel time in microseconds (CUDA events).  Returns a cudaError_t.
extern "C" int devsim_rans_sweep(unsigned long long* out) {
    uint16_t* scratch = nullptr;
    Tally* tally = nullptr;
    uint32_t* rep = nullptr;
    cudaError_t e = cudaMalloc(&scratch, 2ull * 2ull * 65536ull * kFRows);
    if (e == cudaSuccess) e = cudaMalloc(&tally, sizeof(Tally));
    if (e == cudaSuccess) e = cudaMalloc(&rep, 4 * sizeof(uint32_t));
    Tally h = {0, 0, 0, 0, ~0ull};
    uint32_t hr[4] = {0, 0, 0, 0};
    float ms = 0.f;
    if (e == cudaSuccess) e = cudaMemcpy(tally, &h, sizeof(h), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        cudaEvent_t a, b;
        cudaEventCreate(&a);
        cudaEventCreate(&b);
        cudaEventRecord(a);
        sweep_kernel<<<dim3(kQBlocks, kFRows), kThreads>>>(scratch, tally);
        cudaEventRecord(b);
        e = cudaDeviceSynchronize();
        if (e == cudaSuccess) cudaEventElapsedTime(&ms, a, b);
        cudaEventDestroy(a);
        cudaEventDestroy(b);
    }
    if (e == cudaSuccess) e = cudaMemcpy(&h, tally, sizeof(h), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && h.bad != 0) {
        replay_kernel<<<1, 1>>>(scratch, h.first, rep);
        e = cudaDeviceSynchronize();
        if (e == cudaSuccess) e = cudaMemcpy(hr, rep, sizeof(hr), cudaMemcpyDeviceToHost);
    }
    cudaFree(scratch);
    cudaFree(tally);
    cudaFree(rep);
    if (e != cudaSuccess) return (int)e;
    out[0] = h.steps; out[1] = h.bad; out[2] = h.fixups; out[3] = h.pushes;
    out[4] = h.first >> 18; out[5] = (h.first >> 2) & 0xffffu; out[6] = h.first & 3u;
    out[7] = hr[0]; out[8] = hr[1]; out[9] = hr[2]; out[10] = hr[3];
    out[11] = (unsigned long long)(ms * 1000.f);
    return 0;
}
