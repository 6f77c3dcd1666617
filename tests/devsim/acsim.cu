// acsim.cu -- test-only device build of ac_core.cuh's arithmetic coder (container version 1): the steps the kernels
// run (enc_symbol2 / enc_finish2 / dec_init2 / dec_symbol2) on given CDF rows and symbols with their per-step state, a
// clamp harness (a row of a few words between guard words, all in one allocation) and a decoder sweep.  Not part of the
// product library; tests/test_gpu_ac_edges.py loads it through ac_edges.build_acsim().
#include <cuda_runtime.h>
#include <stdint.h>

#include <initializer_list>
#include <utility>

#include "../../lmcache_b200/csrc/ac_core.cuh"

using namespace b200kv;

namespace {

// per-step encoder state (x, rng, lo, m, w) after every enc_symbol2 and after enc_finish2 (entry g)
__global__ void ac_encode_kernel(const uint16_t* cdf, const uint8_t* sym, int g, int n, uint32_t* steps, uint32_t* rows,
                                 uint32_t cap, uint32_t* lens) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint16_t* c = cdf + 33 * j;
    uint32_t* row = rows + (size_t)j * cap;
    uint32_t* o = steps + (size_t)j * (g + 1) * 5;
    EncState2 st;
    st.init();
    for (int i = 0; i < g; ++i) {
        const uint32_t s = sym[(size_t)j * g + i];
        const uint32_t lo = c[s], hi = s >= 31u ? 0x10000u : c[s + 1];
        enc_symbol2(st, lo, hi - lo, row, cap);
        o[5 * i] = st.x; o[5 * i + 1] = st.rng; o[5 * i + 2] = st.lo; o[5 * i + 3] = st.m; o[5 * i + 4] = st.w;
    }
    lens[j] = enc_finish2(st, row, cap);
    o[5 * g] = st.x; o[5 * g + 1] = st.rng; o[5 * g + 2] = st.lo; o[5 * g + 3] = st.m; o[5 * g + 4] = st.w;
}

struct GlobalWords {   // aligned big-endian words from global memory, as decode_kernel's WordSrc hands them out
    const uint32_t* p;
    __device__ uint32_t next_be() { return __byte_perm(*p++, 0u, 0x0123); }
};

// dec_init2 + dec_symbol2<NSTEPS> over stream j, which starts `start[j]` bytes into the word buffer; per symbol
// (span, off, pos, symbol, key) as they were when the symbol was decoded
template <int NSTEPS>
__global__ void ac_decode_kernel(const uint16_t* cdf, const uint32_t* words, const uint32_t* start, int g, int n,
                                 uint32_t* steps) {
    __shared__ uint32_t tab[64][33];
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    uint32_t* e = tab[threadIdx.x];
    for (int i = 0; i < 33; ++i) e[i] = dec_table_entry((uint32_t)i, cdf[33 * j + i]);
    GlobalWords src{words + (start[j] >> 2)};
    DecState2 st;
    dec_init2(st, src, start[j] & 3u);
    uint32_t* o = steps + (size_t)j * g * 5;
    for (int i = 0; i < g; ++i) {
        o[5 * i] = st.span; o[5 * i + 1] = st.off; o[5 * i + 2] = st.pos;
        o[5 * i + 4] = dec_key_approx(st.off, st.span);
        o[5 * i + 3] = dec_symbol2<NSTEPS>(st, src, e, i == g - 1) >> 2;
    }
}

// a row of `cap` words with `guard` words on both sides, all in one allocation: the stream is longer than the row
__global__ void ac_clamp_kernel(const uint16_t* c, const uint8_t* sym, int g, uint32_t cap, uint32_t guard, uint32_t* buf,
                                uint32_t* res) {
    uint32_t* row = buf + guard;
    EncState2 st;
    st.init();
    for (int i = 0; i < g; ++i) {
        const uint32_t s = sym[i];
        const uint32_t lo = c[s], hi = s >= 31u ? 0x10000u : c[s + 1];
        enc_symbol2(st, lo, hi - lo, row, cap);
    }
    res[0] = enc_finish2(st, row, cap);
    res[1] = st.w;
}

struct NoSrc {
    __device__ uint32_t next_be() { return 0u; }
};

// one (row, span) pair per thread: for every symbol s of the row (c[s + 1] > c[s]) the offsets plo(s) - 1, plo(s),
// plo(s) + 1, phi(s) - 2, phi(s) - 1, phi(s) (those in [0, span)): dec_symbol2 against the exact 64-bit rule, the key's
// count (key >> 16) against the exact count ((off + 1) 2^16 - 1) / span, and whether the search's guess was exact
template <int NSTEPS>
__global__ void ac_sweep_kernel(const uint16_t* cdf, int nrows, const uint32_t* spans, int nspans,
                                unsigned long long* tally) {
    __shared__ uint32_t tab[64][33];
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nrows * nspans) return;
    const int rw = t / nspans;
    const uint32_t span = spans[t % nspans];
    uint32_t* e = tab[threadIdx.x];
    for (int i = 0; i < 33; ++i) e[i] = dec_table_entry((uint32_t)i, cdf[33 * rw + i]);
    const unsigned long long S = span ? (unsigned long long)span : (1ull << 32);
    constexpr uint32_t kTop = (1u << NSTEPS) - 1u;
    unsigned long long checks = 0, wrong = 0, slow = 0, kerr[4] = {0, 0, 0, 0};
    for (uint32_t s = 0; s <= kTop && s < 31u; ++s) {
        const uint32_t c0 = e[s] >> 16, c1 = e[s + 1] >> 16;
        if (c1 <= c0) continue;
        const unsigned long long plo = (S * c0) >> 16, phi = (S * c1) >> 16;
        const long long cand[6] = {(long long)plo - 1, (long long)plo, (long long)plo + 1, (long long)phi - 2,
                                   (long long)phi - 1, (long long)phi};
        for (int k = 0; k < 6; ++k) {
            if (cand[k] < 0 || (unsigned long long)cand[k] >= S) continue;
            const uint32_t off = (uint32_t)cand[k];
            uint32_t want = 0;
            for (uint32_t q = 1; q <= kTop; ++q) if (((S * (e[q] >> 16)) >> 16) <= off) want = q;
            if (want > kTop || (NSTEPS == 4 && want > 14u)) continue;        // 16-bin planes never code symbols 15..
            DecState2 st;
            st.x = 0u; st.span = span; st.off = off; st.cur = st.nxt = 0u; st.pos = 0u;
            NoSrc src;
            const uint32_t key = dec_key_approx(off, span);
            uint32_t guess = 0;
            for (uint32_t q = 1; q <= kTop; ++q) if (e[q] <= key) guess = q;
            const uint32_t got = dec_symbol2<NSTEPS>(st, src, e, true) >> 2;
            const unsigned long long cnt = (((unsigned long long)off + 1ull) * 65536ull - 1ull) / S;
            const long long d = (long long)(key >> 16) - (long long)cnt;
            ++checks;
            wrong += got != want ? 1u : 0u;
            slow += guess != want || (NSTEPS == 5 && guess == 31u) ? 1u : 0u;
            kerr[d <= -2 ? 0 : d >= 2 ? 3 : d < 0 ? 1 : 2] += d == 0 ? 0u : 1u;
        }
    }
    atomicAdd(&tally[0], checks);
    atomicAdd(&tally[1], wrong);
    atomicAdd(&tally[2], slow);
    for (int k = 0; k < 4; ++k) atomicAdd(&tally[3 + k], kerr[k]);
}

template <class F>
int with_device(const std::initializer_list<std::pair<void**, size_t>>& bufs, F&& body) {
    cudaError_t e = cudaSuccess;
    for (auto& b : bufs) if (e == cudaSuccess) e = cudaMalloc(b.first, b.second);
    if (e == cudaSuccess) e = body();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    for (auto& b : bufs) cudaFree(*b.first);
    return (int)e;
}

}  // namespace

// n streams of g symbols each (sym uint8 [n, g]) under cdf uint16 [n, 33]: steps uint32 [n, g + 1, 5], rows uint32
// [n, cap], lens uint32 [n].  Returns a cudaError_t.
extern "C" int devsim_ac_encode(const uint16_t* cdf, const uint8_t* sym, int g, int n, uint32_t cap, uint32_t* steps,
                                uint32_t* rows, uint32_t* lens) {
    uint16_t* dc = nullptr; uint8_t* ds = nullptr; uint32_t *dst = nullptr, *dr = nullptr, *dl = nullptr;
    const size_t ns = (size_t)n * (g + 1) * 5 * 4, nr = (size_t)n * cap * 4;
    return with_device({{(void**)&dc, (size_t)n * 66}, {(void**)&ds, (size_t)n * g + 1}, {(void**)&dst, ns},
                        {(void**)&dr, nr}, {(void**)&dl, (size_t)n * 4}}, [&]() {
        cudaMemcpy(dc, cdf, (size_t)n * 66, cudaMemcpyHostToDevice);
        cudaMemcpy(ds, sym, (size_t)n * g, cudaMemcpyHostToDevice);
        cudaMemset(dr, 0, nr);
        ac_encode_kernel<<<(n + 63) / 64, 64>>>(dc, ds, g, n, dst, dr, cap, dl);
        cudaError_t e = cudaDeviceSynchronize();
        if (e == cudaSuccess) e = cudaMemcpy(steps, dst, ns, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(rows, dr, nr, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(lens, dl, (size_t)n * 4, cudaMemcpyDeviceToHost);
        return e;
    });
}

// n streams of g symbols in `bytes` (nbytes, a multiple of 4 with at least 16 bytes after the last stream), stream j
// starting at byte start[j]: steps uint32 [n, g, 5] = (span, off, pos, symbol, key) per symbol.  nsteps: 4 or 5.
extern "C" int devsim_ac_decode(const uint16_t* cdf, const uint8_t* bytes, int64_t nbytes, const uint32_t* start, int g,
                                int n, int nsteps, uint32_t* steps) {
    uint16_t* dc = nullptr; uint32_t *dw = nullptr, *dsrt = nullptr, *dst = nullptr;
    const size_t ns = (size_t)n * g * 5 * 4;
    return with_device({{(void**)&dc, (size_t)n * 66}, {(void**)&dw, (size_t)nbytes}, {(void**)&dsrt, (size_t)n * 4},
                        {(void**)&dst, ns}}, [&]() {
        cudaMemcpy(dc, cdf, (size_t)n * 66, cudaMemcpyHostToDevice);
        cudaMemcpy(dw, bytes, (size_t)nbytes, cudaMemcpyHostToDevice);
        cudaMemcpy(dsrt, start, (size_t)n * 4, cudaMemcpyHostToDevice);
        if (nsteps == 4) ac_decode_kernel<4><<<(n + 63) / 64, 64>>>(dc, dw, dsrt, g, n, dst);
        else ac_decode_kernel<5><<<(n + 63) / 64, 64>>>(dc, dw, dsrt, g, n, dst);
        cudaError_t e = cudaDeviceSynchronize();
        if (e == cudaSuccess) e = cudaMemcpy(steps, dst, ns, cudaMemcpyDeviceToHost);
        return e;
    });
}

// one stream of g symbols into a row of `cap` words between `guard` guard words on each side (buf: cap + 2 guard words,
// in and out: the guard words are whatever the caller put there).  res[0] = enc_finish2's length, res[1] = st.w.
extern "C" int devsim_ac_clamp(const uint16_t* cdf, const uint8_t* sym, int g, uint32_t cap, uint32_t guard,
                               uint32_t* buf, uint32_t* res) {
    uint16_t* dc = nullptr; uint8_t* ds = nullptr; uint32_t *db = nullptr, *dres = nullptr;
    const size_t nb = (size_t)(cap + 2 * guard) * 4;
    return with_device({{(void**)&dc, 66}, {(void**)&ds, (size_t)g + 1}, {(void**)&db, nb}, {(void**)&dres, 8}}, [&]() {
        cudaMemcpy(dc, cdf, 66, cudaMemcpyHostToDevice);
        cudaMemcpy(ds, sym, (size_t)g, cudaMemcpyHostToDevice);
        cudaMemcpy(db, buf, nb, cudaMemcpyHostToDevice);
        ac_clamp_kernel<<<1, 1>>>(dc, ds, g, cap, guard, db, dres);
        cudaError_t e = cudaDeviceSynchronize();
        if (e == cudaSuccess) e = cudaMemcpy(buf, db, nb, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(res, dres, 8, cudaMemcpyDeviceToHost);
        return e;
    });
}

// every CDF row (cdf uint16 [nrows, 33]) at every span (0 = 2^32): tally[0] offsets checked, [1] wrong symbols, [2] offsets
// where the search's guess was not the symbol (the slow path ran), [3..6] key counts off by <= -2, -1, +1, >= +2
extern "C" int devsim_ac_sweep(const uint16_t* cdf, int nrows, const uint32_t* spans, int nspans, int nsteps,
                               unsigned long long* tally) {
    uint16_t* dc = nullptr; uint32_t* dsp = nullptr; unsigned long long* dt = nullptr;
    const int n = nrows * nspans;
    return with_device({{(void**)&dc, (size_t)nrows * 66}, {(void**)&dsp, (size_t)nspans * 4}, {(void**)&dt, 7 * 8}}, [&]() {
        cudaMemcpy(dc, cdf, (size_t)nrows * 66, cudaMemcpyHostToDevice);
        cudaMemcpy(dsp, spans, (size_t)nspans * 4, cudaMemcpyHostToDevice);
        cudaMemset(dt, 0, 7 * 8);
        if (nsteps == 4) ac_sweep_kernel<4><<<(n + 63) / 64, 64>>>(dc, nrows, dsp, nspans, dt);
        else ac_sweep_kernel<5><<<(n + 63) / 64, 64>>>(dc, nrows, dsp, nspans, dt);
        cudaError_t e = cudaDeviceSynchronize();
        if (e == cudaSuccess) e = cudaMemcpy(tally, dt, 7 * 8, cudaMemcpyDeviceToHost);
        return e;
    });
}
