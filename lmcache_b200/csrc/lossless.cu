// lossless.cu -- the lossless KV container (B2KV versions 5 and 6): encode / decode kernels and their C-ABI entry points.
//
// Every 16-bit element u is split as v = rotl16(u, 1): sym = v >> 8 (bf16: the 8 exponent bits; fp16: the 5 exponent bits
// and the top 3 mantissa bits), raw = v & 0xff (sign and the rest of the mantissa).  The raw bytes are stored verbatim; the
// symbols of each (plane, channel) are rANS-coded (32-bit state, 16-bit renormalisation, 12-bit probabilities) against
// one frequency row per plane.  A one-byte element (FP8, uint8) is its own symbol and has no raw byte.  include/b200kv.h
// states the format; tests/lossless_ref.py (16-bit) and tests/lossless8_ref.py (one-byte) are its numpy statements.
// The kernels that touch elements take the element size as a template parameter EB (2 or 1); LlEnc / LlDec.rawb is the
// raw bytes per element, EB - 1.
//
// Thread mapping, as in codec.cu: one stream = one (plane, channel) = one thread; a CTA owns CT consecutive channels of
// one plane of one chunk, so a warp reads 64 contiguous bytes per token and writes 32 contiguous raw bytes.
//   encode: ll_hist_kernel (per-(chunk, plane) histogram) -> ll_norm_kernel (frequency rows) -> ll_encode_kernel (raw
//           bytes in place, rANS into a worst-case scratch row) -> ll_scan_kernel (tile offsets, header, sizes_out) ->
//           ll_compact_kernel (streams into the payload).  The KV is read twice: once for the histogram, once to code.
//   layer-wise encode (b200kv_lossless_encode_layers_plan / _layers / _finish): the same kernels over the planes of a
//           range of layers (a plane-range remap, the identity for the whole container), with the raw rows staged in
//           the workspace -> ll_scan_kernel (the call's segment bytes per chunk) -> ll_place_kernel (the arena rule,
//           segment rows) -> ll_raw_copy_kernel + ll_compact_kernel (raw rows and streams into the arena) ... and at
//           the end ll_finish_kernel (headers into the fixed images, sizes_out).
//   decode: ll_tile_sum_kernel -> ll_scan_kernel (stream offsets from the lengths section; the plan) ->
//           ll_decode_kernel (once for every layer, or once per range of layers: b200kv_lossless_decode_layers).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <type_traits>

#include "ac_core.cuh"
#include "common.cuh"

namespace b200kv {
namespace {

constexpr int kCT = 128;                 // streams (threads) per CTA
constexpr int kScale = 12;               // probability precision: M = 4096
constexpr uint32_t kM = 1u << kScale;
constexpr int kSyms = 256;
constexpr int kMaxTokens = 4096;         // tokens per container (u16 stream lengths)
constexpr int kSlice = 128;              // tokens per histogram CTA
constexpr int kFreqRowBytes = 2 * kSyms;

// fixed sections of a container of P planes of C channels and t tokens with rawb raw bytes per element (1 for 16-bit
// elements, 0 for one-byte ones); max_stream: the longest stream the encoder can produce (4 state bytes + <= ceil(3t/4)
// + 1 renormalisation halfwords), max_total: the worst-case container
struct LlLayout {
    int64_t off_freq, off_lens, off_raw, off_payload, max_stream, max_total;
};
__host__ __device__ __forceinline__ int64_t ll_max_words(int t) { return (3 * (int64_t)t + 3) / 4 + 1; }
__host__ __device__ __forceinline__ LlLayout ll_layout(int P, int64_t C, int t, int rawb) {
    LlLayout lo;
    lo.off_freq = B200KV_HEADER_BYTES;
    lo.off_lens = lo.off_freq + (int64_t)P * kFreqRowBytes;
    lo.off_raw = align16(lo.off_lens + 2 * (int64_t)P * C);
    lo.off_payload = align16(lo.off_raw + (int64_t)P * t * C * rawb);
    lo.max_stream = 4 + 2 * ll_max_words(t);
    lo.max_total = align16(lo.off_payload + (int64_t)P * C * lo.max_stream);
    return lo;
}

struct LlEnc {
    PlaneTable pt;                       // source planes (maxq unused)
    int64_t sT, sH, tok_begin;
    const int64_t* slot_map;
    int32_t L, H, D, C, NP, dtype;       // NP = planes: 2L, or L for a latent KV
    int32_t rawb;                        // raw bytes per element: 1 (16-bit elements) or 0 (one-byte elements)
    int32_t n_chunks, chunk_tokens, last_chunk_tokens, tpp, ntiles, rw;   // rw: halfwords per scratch row
    uint8_t* out;                        // containers (the layer-wise encode: fixed images [0, off_raw))
    int64_t out_stride;
    uint64_t* sizes_out;
    // The launch codes the planes of layers [lb, lb + nl), npc per chunk: local plane pl < nl is plane lb + pl, the
    // others L + lb + pl - nl (ll_plane; the identity for lb = 0, nl = L).  Scratch rows are indexed by local plane.
    int32_t lb, nl, npc;
    int32_t layers_left;                 // layers not yet encoded after this call (arena reserve, ll_place_kernel)
    uint32_t* hist;                      // [n][npc][256] symbol counts
    uint32_t* err;                       // [n] bit 0: a stream outgrew the bound; bit 16: the chunk did not fit the arena
    uint32_t* tab;                       // [n][npc][256] (start << 16) | freq
    unsigned long long* tile;            // [n][ntiles] stream bytes per tile, then exclusive prefix
    uint32_t* state;                     // [n][npc][C] final coder states
    uint16_t* scratch;                   // [n][npc][C][rw] renormalisation halfwords, the last one pushed first
    uint8_t* raw;                        // raw rows of (chunk j, local plane pl): raw + j * raw_stride + pl * t * C
                                         // (16-bit elements only)
    int64_t raw_stride;
    // b200kv_lossless_encode_layers only (arena NULL otherwise): raw rows and streams go to a device arena
    uint8_t* arena;
    int64_t arena_bytes;
    unsigned long long* chunk_base;      // [n] arena offset of chunk j's segment of this call, ~0 = chunk failed
    unsigned long long* cursor;          // first free arena byte (device-held across calls)
    unsigned int* fail_from;             // first failed chunk (n_chunks: none); every later chunk fails too
    unsigned long long* totals;          // [n] bytes of chunk j's segment of this call
    unsigned long long* ptotal;          // [n] stream bytes of every call so far (the header's payload_bytes)
    int64_t* seg;                        // [n][NP][3] segment rows (b200kv_lossless_encode_layers_plan)
};
static_assert(sizeof(LlEnc) < kMaxParamBytes, "LlEnc must stay under 4 KB of kernel parameters");

struct LlDecChunk {
    const uint8_t* base;
    int64_t dst_tok;
    int64_t payload_bytes;               // total_bytes - off_payload, from the caller: every stream must lie inside
    int32_t t;
    // head window (b200kv_lossless_decode_plan_heads; the whole container otherwise): container channels [cw0, cw1) are
    // decoded into destination channel c + dshift; they lie in tiles [ct0, ct0 + ntw) of every plane
    int32_t ct0, ntw, cw0, cw1, dshift;
};

struct LlDec {
    PlaneTable pt;                       // destination planes (maxq unused)
    int64_t sT, sH;
    const int64_t* slot_map;
    int32_t L, H, D, C, NP, tpp, ntiles, dtype, version, n_chunks;   // H, C: the containers' (src_H with windows)
    int32_t rawb;                        // raw bytes per element: 1 (16-bit elements) or 0 (one-byte elements)
    int32_t wtpp;                        // tiles launched per plane: the largest window's ntw (tpp without windows)
    int32_t lb, nl;                      // the launch decodes layers [lb, lb + nl): blockIdx.y < nl keys, then values
    const LlDecChunk* chunks;
    unsigned long long* tile;            // [n][ntiles]
    uint32_t* status;                    // [n] or NULL
};
static_assert(sizeof(LlDec) < kMaxParamBytes, "LlDec must stay under 4 KB of kernel parameters");

// What b200kv_lossless_decode_plan decided, kept in the caller's b200kv_lossless_decode_plan_t: the decode kernel's
// parameter block (its chunk descriptors and tile offsets live in the workspace).
constexpr uint32_t kLlPlanMagic = 0x4e4c504cu;   // "LPLN"
struct LlPlan {
    uint32_t magic, pad;
    LlDec P;
};
static_assert(sizeof(LlPlan) <= sizeof(b200kv_lossless_decode_plan_t), "b200kv_lossless_decode_plan_t too small");

// What b200kv_lossless_encode_layers_plan decided, kept in the caller's b200kv_lossless_encode_plan_t: the kernels'
// parameter block (its counters live in the workspace), the layers encoded so far and the most one call may take.
constexpr uint32_t kLlEncPlanMagic = 0x4c50454cu;   // "LEPL"
struct LlEncPlan {
    uint32_t magic;
    int32_t max_layers;
    LayerSet done;
    LlEnc P;
};
static_assert(sizeof(LlEncPlan) <= sizeof(b200kv_lossless_encode_plan_t), "b200kv_lossless_encode_plan_t too small");

__device__ __forceinline__ int ll_chunk_t(const LlEnc& P, int j) {
    return j == P.n_chunks - 1 ? P.last_chunk_tokens : P.chunk_tokens;
}

// container plane of the launch's local plane (LlEnc.lb / nl)
__device__ __forceinline__ int ll_plane(const LlEnc& P, int pl) {
    return pl < P.nl ? P.lb + pl : P.L + P.lb + (pl - P.nl);
}

// bytes of the raw part of a chunk's segment in the layer-wise encode: the call's raw rows, and -- in the call that
// holds the last plane -- the container's zero bytes between the raw section and off_payload, then 16-byte aligned
__device__ __forceinline__ int64_t ll_seg_raw(const LlEnc& P, int t, const LlLayout& lo) {
    int64_t r = (int64_t)P.npc * t * P.C * P.rawb;
    if (P.lb + P.nl == P.L) r += lo.off_payload - lo.off_raw - (int64_t)P.NP * t * P.C * P.rawb;
    return align16(r);
}

// header of chunk j with `payload` stream bytes
__device__ __forceinline__ void ll_put_header(const LlEnc& P, int j, unsigned long long payload, uint32_t status) {
    const int t = ll_chunk_t(P, j);
    const LlLayout lo = ll_layout(P.NP, P.C, t, P.rawb);
    b200kv_header hd;
    memset(&hd, 0, sizeof(hd));
    hd.magic = B200KV_MAGIC;
    hd.version = P.NP == P.L ? 6u : 5u;
    hd.L = (uint32_t)P.L; hd.H = (uint32_t)P.H; hd.D = (uint32_t)P.D;
    hd.ntokens = (uint32_t)t;
    hd.ngroups = 1u;
    hd.max_dtype = (uint32_t)P.dtype;
    hd.payload_bytes = payload;
    hd.total_bytes = (uint64_t)lo.off_payload + payload;
    hd.status = status;
    if (hd.total_bytes > (uint64_t)P.out_stride && P.arena == nullptr) hd.status |= 2u;   // cannot happen within the bound
    *reinterpret_cast<b200kv_header*>(P.out + (int64_t)j * P.out_stride) = hd;
    P.sizes_out[j] = hd.status ? 0ull : hd.total_bytes;
}

__device__ __forceinline__ uint32_t rotl1(uint32_t u) { return ((u << 1) | (u >> 15)) & 0xffffu; }
__device__ __forceinline__ uint32_t rotr1(uint32_t v) { return ((v >> 1) | (v << 15)) & 0xffffu; }

// element type of EB bytes, and the coded form of an element u: 16-bit v = rotl16(u, 1) (symbol v >> 8, raw byte
// v & 0xff); a one-byte element is its own symbol (v = u << 8, no raw byte)
template <int EB> using ll_elem_t = typename std::conditional<EB == 2, uint16_t, uint8_t>::type;
template <int EB>
__device__ __forceinline__ uint32_t ll_code(uint32_t u) { return EB == 2 ? rotl1(u) : u << 8; }

// exclusive prefix of v over a CTA of NT threads, and the CTA's total (every thread must call it)
template <int NT, class T>
__device__ __forceinline__ T cta_excl_scan(T v, T* s_w, T* total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    T inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) s_w[w] = inc;
    __syncthreads();
    T base = 0, tot = 0;
#pragma unroll
    for (int i = 0; i < NT / 32; ++i) {
        const T x = s_w[i];
        if (i < w) base += x;
        tot += x;
    }
    __syncthreads();
    *total = tot;
    return base + inc - v;
}

// ------------------------------------------------------------------------------------------ encode
// 1) symbol histogram of one (chunk, plane, channel tile, slice of kSlice tokens): warp-private bins in shared memory,
//    lanes with equal symbols aggregated (__match_any_sync), then one global add per nonzero bin
template <bool PAGED, int EB>
__global__ void __launch_bounds__(kCT) ll_hist_kernel(LlEnc P) {
    __shared__ uint32_t s_h[kCT / 32][kSyms];
    const int j = blockIdx.z, pl = blockIdx.y, p = ll_plane(P, pl);
    const int tile = blockIdx.x % P.tpp, slice = blockIdx.x / P.tpp;
    const int t = ll_chunk_t(P, j);
    const int i0 = slice * kSlice;
    if (i0 >= t) return;
    const int i1 = min(t, i0 + kSlice);
    for (int i = threadIdx.x; i < (kCT / 32) * kSyms; i += kCT) (&s_h[0][0])[i] = 0u;
    __syncthreads();
    const int c = tile * kCT + threadIdx.x;
    const bool on = c < P.C;
    const int h = on ? c / P.D : 0, d = on ? c - h * P.D : 0;
    const ll_elem_t<EB>* base = reinterpret_cast<const ll_elem_t<EB>*>(P.pt.p[p]) + (int64_t)h * P.sH + d;
    const int64_t tok0 = P.tok_begin + (int64_t)j * P.chunk_tokens;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = i0; i < i1; i += 4) {
        uint32_t u[4];
#pragma unroll
        for (int k = 0; k < 4; ++k)
            u[k] = on && i + k < i1 ? __ldg(base + tok_row<PAGED>(P.slot_map, tok0 + i + k) * P.sT) : 0u;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t sym = on && i + k < i1 ? ll_code<EB>(u[k]) >> 8 : 0x100u;   // 0x100: no symbol
            const uint32_t peers = __match_any_sync(0xffffffffu, sym);
            if (sym < 0x100u && lane == __ffs(peers) - 1) atomicAdd(&s_h[w][sym], (uint32_t)__popc(peers));
        }
    }
    __syncthreads();
    uint32_t* g = P.hist + ((int64_t)j * P.npc + pl) * kSyms;
    for (int s = threadIdx.x; s < kSyms; s += kCT) {
        uint32_t v = 0u;
#pragma unroll
        for (int k = 0; k < kCT / 32; ++k) v += s_h[k][s];
        if (v) atomicAdd(g + s, v);
    }
}

// 2) frequency row of one (chunk, plane), one thread per symbol (the normalisation of include/b200kv.h):
//    K = symbols that occur, N = C * t;  f_s = n_s ? 1 + floor(n_s * (4096 - K) / N) : 0;  the symbol with the largest
//    count (the smallest such symbol on ties) gets 4096 - sum(f) more.
__global__ void __launch_bounds__(kSyms) ll_norm_kernel(LlEnc P) {
    __shared__ uint32_t s_w[kSyms / 32];
    __shared__ unsigned long long s_k[kSyms / 32];
    const int j = blockIdx.y, pl = blockIdx.x, p = ll_plane(P, pl), s = threadIdx.x;
    const int t = ll_chunk_t(P, j);
    const int64_t row = (int64_t)j * P.npc + pl;
    const uint32_t n = P.hist[row * kSyms + s];
    const uint32_t K = (uint32_t)__syncthreads_count(n != 0u);
    const uint64_t N = (uint64_t)P.C * (uint64_t)t;
    uint32_t f = n ? 1u + (uint32_t)(((uint64_t)n * (kM - K)) / N) : 0u;
    uint32_t F;
    cta_excl_scan<kSyms>(f, s_w, &F);
    // argmax of (count, -symbol)
    unsigned long long key = n ? ((unsigned long long)n << 8) | (unsigned long long)(255 - s) : 0ull;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long y = __shfl_xor_sync(0xffffffffu, key, o);
        key = y > key ? y : key;
    }
    if ((threadIdx.x & 31) == 0) s_k[threadIdx.x >> 5] = key;
    __syncthreads();
    unsigned long long best = 0ull;
#pragma unroll
    for (int k = 0; k < kSyms / 32; ++k) best = s_k[k] > best ? s_k[k] : best;
    if (s == 255 - (int)(best & 0xffull)) f += kM - F;
    uint32_t tot;
    const uint32_t start = cta_excl_scan<kSyms>(f, s_w, &tot);
    P.tab[row * kSyms + s] = (start << 16) | f;
    uint8_t* cont = P.out + (int64_t)j * P.out_stride;
    reinterpret_cast<uint16_t*>(cont + B200KV_HEADER_BYTES + (int64_t)p * kFreqRowBytes)[s] = (uint16_t)f;
}

// 3) one thread per (chunk, plane, channel): raw bytes to their place in the container, symbols rANS-coded from the last
//    token to the first (so that the decoder runs forward) into the stream's scratch row.  Encoder step with M = 4096:
//      if (x >> 20) >= f: push x & 0xffff, x >>= 16;   x = ((x / f) << 12) + (x mod f) + start
//    The bound is compared as x >> 20 against f, not x against f << 20: a single-symbol plane has f = 4096, and 4096 << 20
//    does not fit 32 bits.  With f = 4096 the step leaves x unchanged and pushes nothing.  Plain integer division.
//    One-byte elements have no raw bytes.
template <bool PAGED, int EB>
__global__ void __launch_bounds__(kCT) ll_encode_kernel(LlEnc P) {
    __shared__ uint32_t s_tab[kSyms];
    __shared__ unsigned long long s_w[kCT / 32];
    const int j = blockIdx.z, pl = blockIdx.y, p = ll_plane(P, pl), tile = blockIdx.x;
    const int t = ll_chunk_t(P, j);
    const int64_t row = (int64_t)j * P.npc + pl;
    for (int s = threadIdx.x; s < kSyms; s += kCT) s_tab[s] = P.tab[row * kSyms + s];
    __syncthreads();
    const int c = tile * kCT + threadIdx.x;
    const bool on = c < P.C;
    const LlLayout lo = ll_layout(P.NP, P.C, t, P.rawb);
    uint8_t* cont = P.out + (int64_t)j * P.out_stride;
    uint32_t x = kRansLow;
    int32_t k = 0;
    if (on) {
        const int h = c / P.D, d = c - h * P.D;
        const ll_elem_t<EB>* base = reinterpret_cast<const ll_elem_t<EB>*>(P.pt.p[p]) + (int64_t)h * P.sH + d;
        const int64_t tok0 = P.tok_begin + (int64_t)j * P.chunk_tokens;
        uint8_t* raw = P.raw + (int64_t)j * P.raw_stride + (int64_t)pl * t * P.C + c;
        uint16_t* srow = P.scratch + (row * P.C + c) * P.rw;
        const int rw = P.rw;
        uint32_t nxt = __ldg(base + tok_row<PAGED>(P.slot_map, tok0 + t - 1) * P.sT);
        for (int i = t - 1; i >= 0; --i) {
            const uint32_t u = nxt;
            if (i > 0) nxt = __ldg(base + tok_row<PAGED>(P.slot_map, tok0 + i - 1) * P.sT);
            const uint32_t v = ll_code<EB>(u);
            if (EB == 2) raw[(int64_t)i * P.C] = (uint8_t)v;
            const uint32_t e = s_tab[v >> 8];
            const uint32_t f = e & 0xffffu;
            if ((x >> 20) >= f) {
                if (k < rw) srow[rw - 1 - k] = (uint16_t)x;
                ++k;
                x >>= 16;
            }
            x = ((x / f) << kScale) + (x % f) + (e >> 16);
        }
        if (k > ll_max_words(t)) atomicOr(&P.err[j], 1u);
        reinterpret_cast<uint16_t*>(cont + lo.off_lens)[(int64_t)p * P.C + c] = (uint16_t)min(4 + 2 * k, 0xffff);
        P.state[row * P.C + c] = x;
    }
    unsigned long long tot;
    cta_excl_scan<kCT, unsigned long long>(on ? 4ull + 2ull * (unsigned long long)k : 0ull, s_w, &tot);
    if (threadIdx.x == 0) P.tile[(int64_t)j * P.ntiles + (int64_t)pl * P.tpp + tile] = tot;
}

// exclusive prefix of one chunk's tile values in place; returns the chunk's total to thread 0
__device__ unsigned long long ll_scan_tiles(unsigned long long* v, int n) {
    __shared__ unsigned long long s_w[32];
    unsigned long long carry = 0ull;
    for (int b = 0; b < n; b += blockDim.x) {
        const int i = b + threadIdx.x;
        const unsigned long long x = i < n ? v[i] : 0ull;
        const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
        unsigned long long inc = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += y;
        }
        if (lane == 31) s_w[w] = inc;
        __syncthreads();
        unsigned long long base = 0ull, tot = 0ull;
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) {
            if (k < w) base += s_w[k];
            tot += s_w[k];
        }
        if (i < n) v[i] = carry + base + inc - x;
        carry += tot;
        __syncthreads();
    }
    return carry;
}

// 4a) per chunk: tile offsets, then the header and sizes_out[j] (0 when the chunk's status is nonzero), and zeros in the
//     two alignment gaps (after the lengths, after the raw rows) instead of whatever the output buffer held.  In the
//     layer-wise encode: the bytes of the chunk's segment of this call instead (the raw part, then the streams).
__global__ void __launch_bounds__(1024) ll_enc_scan_kernel(LlEnc P) {
    const int j = blockIdx.x;
    const unsigned long long payload = ll_scan_tiles(P.tile + (int64_t)j * P.ntiles, P.ntiles);
    if (threadIdx.x != 0) return;
    const int t = ll_chunk_t(P, j);
    const LlLayout lo = ll_layout(P.NP, P.C, t, P.rawb);
    if (P.arena != nullptr) {
        P.totals[j] = (unsigned long long)ll_seg_raw(P, t, lo) + payload;
        return;
    }
    ll_put_header(P, j, payload, P.err[j]);
    uint8_t* cont = P.out + (int64_t)j * P.out_stride;
    for (int64_t b = lo.off_lens + 2 * (int64_t)P.NP * P.C; b < lo.off_raw; ++b) cont[b] = 0u;
    for (int64_t b = lo.off_raw + (int64_t)P.NP * t * P.C * P.rawb; b < lo.off_payload; ++b) cont[b] = 0u;
}

// 4b) streams into the payload (the layer-wise encode: into the chunk's segment, after its raw part), a warp per 32
//     streams: [LE32 state][halfwords in decode order]
__global__ void __launch_bounds__(kCT) ll_compact_kernel(LlEnc P) {
    __shared__ uint32_t s_w[kCT / 32];
    const int j = blockIdx.z, pl = blockIdx.y, p = ll_plane(P, pl), tile = blockIdx.x;
    if (P.err[j]) return;                                // an overflowed stream, or no room in the arena
    const int t = ll_chunk_t(P, j);
    const LlLayout lo = ll_layout(P.NP, P.C, t, P.rawb);
    uint8_t* cont = P.out + (int64_t)j * P.out_stride;
    uint8_t* base = P.arena != nullptr ? P.arena + P.chunk_base[j] + ll_seg_raw(P, t, lo) : cont + lo.off_payload;
    const int64_t row = (int64_t)j * P.npc + pl;
    const int c = tile * kCT + threadIdx.x;
    const bool on = c < P.C;
    const uint32_t len = on ? reinterpret_cast<const uint16_t*>(cont + lo.off_lens)[(int64_t)p * P.C + c] : 0u;
    uint32_t tot;
    const uint32_t ex = cta_excl_scan<kCT>(len, s_w, &tot);
    const unsigned long long off = P.tile[(int64_t)j * P.ntiles + (int64_t)pl * P.tpp + tile] + ex;
    const uint32_t st = on ? P.state[row * P.C + c] : 0u;
    const int lane = threadIdx.x & 31;
    const int cw = tile * kCT + (threadIdx.x & ~31);
    for (int src = 0; src < 32; ++src) {
        const uint32_t sl = __shfl_sync(0xffffffffu, len, src);
        const unsigned long long so = __shfl_sync(0xffffffffu, off, src);
        const uint32_t sx = __shfl_sync(0xffffffffu, st, src);
        if (sl == 0u) continue;
        const uint32_t nh = sl >> 1, k = nh - 2;
        const uint16_t* r = P.scratch + (row * P.C + cw + src) * P.rw + (P.rw - k) - 2;
        uint16_t* dst = reinterpret_cast<uint16_t*>(base + so);
        for (uint32_t q = lane; q < nh; q += 32)
            dst[q] = q == 0 ? (uint16_t)sx : q == 1 ? (uint16_t)(sx >> 16) : r[q];
    }
}

// ------------------------------------------------------------------------------------------ layer-wise encode
// After ll_enc_scan_kernel: each chunk's segment of this call gets room in the arena by the arena rule (arena_place,
// common.cuh), the stream bytes of the chunks placed are added to their payload totals, and every plane of the call gets
// its segment row (arena offset of its raw rows, arena offset of its streams, stream bytes).  One CTA.
__global__ void __launch_bounds__(1024) ll_place_kernel(LlEnc P) {
    const int tid = threadIdx.x;
    arena_place(P.n_chunks, P.totals, P.layers_left, P.nl, P.arena_bytes, P.cursor, P.fail_from, P.chunk_base, P.err);
    for (int j = tid; j < P.n_chunks; j += 1024)
        if (P.chunk_base[j] != ~0ull) {
            const int t = ll_chunk_t(P, j);
            P.ptotal[j] += P.totals[j] - (unsigned long long)ll_seg_raw(P, t, ll_layout(P.NP, P.C, t, P.rawb));
        }
    for (int k = tid; k < P.n_chunks * P.npc; k += 1024) {
        const int j = k / P.npc, pl = k - j * P.npc;
        const int t = ll_chunk_t(P, j);
        const unsigned long long raw = (unsigned long long)ll_seg_raw(P, t, ll_layout(P.NP, P.C, t, P.rawb));
        const unsigned long long* tb = P.tile + (int64_t)j * P.ntiles;
        const unsigned long long off = tb[pl * P.tpp];
        const unsigned long long end = pl + 1 < P.npc ? tb[(pl + 1) * P.tpp] : P.totals[j] - raw;
        const unsigned long long cb = P.chunk_base[j];
        int64_t* row = P.seg + ((int64_t)j * P.NP + ll_plane(P, pl)) * 3;
        row[0] = cb == ~0ull ? -1 : (int64_t)(cb + (unsigned long long)pl * t * P.C * P.rawb);
        row[1] = cb == ~0ull ? -1 : (int64_t)(cb + raw + off);
        row[2] = (int64_t)(end - off);
    }
}

// The raw part of each placed chunk's segment: the call's staged raw rows, then zeros up to the segment's streams (the
// container's gap before off_payload, when the call holds the last plane, and the alignment).  16 bytes per thread.
__global__ void __launch_bounds__(256) ll_raw_copy_kernel(LlEnc P) {
    const int j = blockIdx.y;
    if (P.err[j]) return;
    const int t = ll_chunk_t(P, j);
    const int64_t nraw = (int64_t)P.npc * t * P.C * P.rawb, nseg = ll_seg_raw(P, t, ll_layout(P.NP, P.C, t, P.rawb));
    const uint8_t* src = P.raw + (int64_t)j * P.raw_stride;
    uint8_t* dst = P.arena + P.chunk_base[j];
    for (int64_t b = 16 * ((int64_t)blockIdx.x * blockDim.x + threadIdx.x); b < nseg; b += 16 * (int64_t)gridDim.x * blockDim.x) {
        uint4 v;
        if (b + 16 <= nraw) {
            v = __ldg(reinterpret_cast<const uint4*>(src + b));
        } else {
            uint8_t x[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) x[i] = b + i < nraw ? src[b + i] : (uint8_t)0;
            memcpy(&v, x, 16);
        }
        *reinterpret_cast<uint4*>(dst + b) = v;
    }
}

__global__ void ll_encl_init_kernel(LlEnc P) {
    *P.cursor = 0ull;
    *P.fail_from = (unsigned)P.n_chunks;
}

// headers into the fixed images from the payload of every call; sizes_out 0 for a chunk with a nonzero status
__global__ void ll_finish_kernel(LlEnc P) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < P.n_chunks) ll_put_header(P, j, P.ptotal[j], P.err[j]);
}

// ------------------------------------------------------------------------------------------ decode
// stream bytes per tile, from the lengths section: one warp per tile
__global__ void __launch_bounds__(128) ll_tile_sum_kernel(LlDec P) {
    const int j = blockIdx.y;
    const int tl = blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (tl >= P.ntiles) return;
    const int p = tl / P.tpp, c0 = (tl - p * P.tpp) * kCT;
    const uint16_t* lens = reinterpret_cast<const uint16_t*>(P.chunks[j].base + B200KV_HEADER_BYTES +
                                                             (int64_t)P.NP * kFreqRowBytes) + (int64_t)p * P.C;
    unsigned long long s = 0ull;
    for (int c = c0 + lane; c < min(P.C, c0 + kCT); c += 32) s += lens[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) P.tile[(int64_t)j * P.ntiles + tl] = s;
}

__global__ void __launch_bounds__(1024) ll_dec_scan_kernel(LlDec P) {
    ll_scan_tiles(P.tile + (int64_t)blockIdx.x * P.ntiles, P.ntiles);
}

// One CTA per (chunk, plane, tile of CT channels): the plane's frequency row becomes a 4096-entry slot -> symbol table and
// (start, freq) pairs in shared memory; each thread decodes its stream forward, recombines every symbol with its raw
// byte and stores the element through the destination descriptor.  Decoder step:
//   slot = x & 4095;  s = sym(slot);  x = f(s) * (x >> 12) + slot - start(s);  if x < 2^16: x = (x << 16) | next LE16
// and after the last token x == 2^16 with every halfword of the stream consumed.  Reads stay inside the stream's own
// bytes, and the stream inside the payload, whatever the lengths and frequency rows say.
// A launch covers the planes of layers [lb, lb + nl) only (b200kv_lossless_decode_layers): it reads the header, those
// planes' frequency rows, the lengths section (through the tile offsets the plan computed from it), those planes' raw
// rows and those planes' streams, and nothing else of the container.
// With a head window (b200kv_lossless_decode_plan_heads) CTA x of a plane is tile ct0 + x of the container, and CTAs
// past the window's ntw leave.  Every thread of a tile still reads its length and joins the scan, because a stream's
// offset depends on the lengths before it in the tile, but only the channels [cw0, cw1) decode, into destination
// channel c + dshift, and only they can set status bits: a damaged stream outside the window is never read.
template <bool PAGED, int EB>
__global__ void __launch_bounds__(kCT) ll_decode_kernel(LlDec P) {
    __shared__ uint32_t s_ent[kSyms];
    __shared__ uint8_t s_sym[kM];
    __shared__ uint32_t s_w[kCT / 32];
    const int j = blockIdx.z;
    const int p = (int)blockIdx.y < P.nl ? P.lb + (int)blockIdx.y : P.L + P.lb + ((int)blockIdx.y - P.nl);
    const LlDecChunk dc = P.chunks[j];
    if ((int)blockIdx.x >= dc.ntw) return;
    const int tile = dc.ct0 + (int)blockIdx.x;
    const int t = dc.t;
    const LlLayout lo = ll_layout(P.NP, P.C, t, P.rawb);
    uint32_t bad = 0u;
    if (threadIdx.x == 0) {
        const b200kv_header* hd = reinterpret_cast<const b200kv_header*>(dc.base);
        if (hd->magic != B200KV_MAGIC || hd->version != (uint32_t)P.version || hd->L != (uint32_t)P.L ||
            hd->H != (uint32_t)P.H || hd->D != (uint32_t)P.D || hd->ntokens != (uint32_t)t ||
            hd->max_dtype != (uint32_t)P.dtype)
            bad |= 4u;
    }
    // frequency row: two symbols per thread
    const uint16_t* frow = reinterpret_cast<const uint16_t*>(dc.base + B200KV_HEADER_BYTES + (int64_t)p * kFreqRowBytes);
    const uint32_t f0 = frow[2 * threadIdx.x], f1 = frow[2 * threadIdx.x + 1];
    uint32_t ftot;
    const uint32_t st0 = cta_excl_scan<kCT>(f0 + f1, s_w, &ftot);
    if (ftot != kM) {                                   // damaged frequency row: nothing of this plane is decoded
        if (threadIdx.x == 0 && P.status != nullptr) atomicOr(&P.status[j], bad | 1u);
        return;
    }
    s_ent[2 * threadIdx.x] = (st0 << 16) | f0;
    s_ent[2 * threadIdx.x + 1] = ((st0 + f0) << 16) | f1;
    __syncthreads();
    for (int slot = threadIdx.x; slot < (int)kM; slot += kCT) {
        int s = 0;                                      // the last symbol whose start <= slot: it has f >= 1
#pragma unroll
        for (int step = kSyms / 2; step > 0; step >>= 1)
            if ((s_ent[s + step] >> 16) <= (uint32_t)slot) s += step;
        s_sym[slot] = (uint8_t)s;
    }
    __syncthreads();
    const int c = tile * kCT + threadIdx.x;
    const bool on = c < P.C;
    const uint32_t len = on ? reinterpret_cast<const uint16_t*>(dc.base + lo.off_lens)[(int64_t)p * P.C + c] : 0u;
    uint32_t tot;
    const uint32_t ex = cta_excl_scan<kCT>(len, s_w, &tot);
    if (on && c >= dc.cw0 && c < dc.cw1) {
        const unsigned long long off = P.tile[(int64_t)j * P.ntiles + (int64_t)p * P.tpp + tile] + ex;
        if (off + len > (unsigned long long)dc.payload_bytes) {
            bad |= 2u;
        } else if (len < 4u || ((len | off) & 1u)) {     // a damaged odd length before this stream makes its start odd
            bad |= 1u;
        } else {
            const uint16_t* sp = reinterpret_cast<const uint16_t*>(dc.base + lo.off_payload + off);
            uint32_t x = (uint32_t)sp[0] | ((uint32_t)sp[1] << 16);
            const uint16_t* wp = sp + 2;
            const uint32_t nw = (len - 4u) >> 1;
            uint32_t k = 0u;
            const int oc = c + dc.dshift;                // destination channel
            const int h = oc / P.D, d = oc - h * P.D;
            ll_elem_t<EB>* dst = reinterpret_cast<ll_elem_t<EB>*>(const_cast<uint16_t*>(P.pt.p[p])) + (int64_t)h * P.sH + d;
            const uint8_t* raw = dc.base + lo.off_raw + (int64_t)p * t * P.C + c;
#pragma unroll 4
            for (int i = 0; i < t; ++i) {
                const uint32_t rb = EB == 2 ? raw[(int64_t)i * P.C] : 0u;
                const uint32_t slot = x & (kM - 1u);
                const uint32_t sym = s_sym[slot];
                const uint32_t e = s_ent[sym];
                x = (e & 0xffffu) * (x >> kScale) + slot - (e >> 16);
                if (x < kRansLow) {
                    const uint32_t hw = k < nw ? (uint32_t)wp[k] : 0u;
                    ++k;
                    x = (x << 16) | hw;
                }
                dst[tok_row<PAGED>(P.slot_map, dc.dst_tok + i) * P.sT] =
                    EB == 2 ? (ll_elem_t<EB>)rotr1((sym << 8) | rb) : (ll_elem_t<EB>)sym;
            }
            if (x != kRansLow || k != nw) bad |= 1u;
        }
    }
    if (bad != 0u && P.status != nullptr) atomicOr(&P.status[j], bad);
}

// The header fields a stream-offset computation trusts, checked before anything past the header is read: a lossless
// version, a shape the calls accept, and -- for the device form -- fixed sections that fit total_bytes and `limit`.
__host__ __device__ __forceinline__ bool ll_offsets_header_ok(const b200kv_header& hd, int64_t limit, LlLayout* lo,
                                                              int* NP) {
    if (hd.magic != B200KV_MAGIC || (hd.version != 5u && hd.version != 6u) || hd.L == 0u ||
        hd.L > (uint32_t)(B200KV_MAX_PLANES / 2) || hd.H == 0u || hd.D == 0u ||
        (uint64_t)hd.H * hd.D >= (1ull << 24) || hd.ntokens == 0u || hd.ntokens > (uint32_t)kMaxTokens)
        return false;
    int rawb;                                           // the element dtype decides the raw section
    if (hd.max_dtype == B200KV_DT_BF16 || hd.max_dtype == B200KV_DT_FP16) rawb = 1;
    else if (hd.max_dtype == B200KV_DT_U8 || hd.max_dtype == B200KV_DT_FP8_E4M3 || hd.max_dtype == B200KV_DT_FP8_E5M2)
        rawb = 0;
    else return false;
    *NP = hd.version == 6u ? (int)hd.L : 2 * (int)hd.L;
    *lo = ll_layout(*NP, (int64_t)hd.H * hd.D, (int)hd.ntokens, rawb);
    return (uint64_t)lo->off_payload <= hd.total_bytes && lo->off_payload <= limit;
}

// Stream offsets of lossless containers in device memory (b200kv_lossless_plane_offsets_device): one CTA of 32 warps
// per container, one warp per plane at a time, summing the plane's u16 lengths.  out row j: [off_payload, end of plane
// 0's streams, ..., end of plane P-1 = total_bytes], zeros after it; or -1 in entry 0 when the header is not that of a
// lossless container whose fixed sections fit total_bytes and the row stride (nothing past the header is read then), or
// the lengths do not add up to total_bytes.
__global__ void __launch_bounds__(1024) ll_plane_offsets_kernel(const uint8_t* base, int64_t stride, int64_t* out) {
    __shared__ unsigned long long s_sum[B200KV_MAX_PLANES];
    const uint8_t* c = base + (int64_t)blockIdx.x * stride;
    int64_t* o = out + (int64_t)blockIdx.x * (B200KV_MAX_PLANES + 1);
    const b200kv_header hd = *reinterpret_cast<const b200kv_header*>(c);
    LlLayout lo;
    int NP;
    if (!ll_offsets_header_ok(hd, stride, &lo, &NP)) {
        if (threadIdx.x == 0) o[0] = -1;
        return;
    }
    const int64_t C = (int64_t)hd.H * hd.D;
    const uint16_t* lens = reinterpret_cast<const uint16_t*>(c + lo.off_lens);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int p = NP + 1 + (int)threadIdx.x; p <= B200KV_MAX_PLANES; p += blockDim.x) o[p] = 0;   // the row past P + 1
    for (int p = warp; p < NP; p += blockDim.x >> 5) {
        const uint16_t* row = lens + p * C;
        unsigned long long sum = 0ull;
        for (int64_t i = lane; i < C; i += 32) sum += row[i];
#pragma unroll
        for (int k = 16; k > 0; k >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, k);
        if (lane == 0) s_sum[p] = sum;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t off = lo.off_payload;
        o[0] = off;
        for (int p = 0; p < NP; ++p) {
            off += (int64_t)s_sum[p];
            o[p + 1] = off;
        }
        if (off != (int64_t)hd.total_bytes) o[0] = -1;
    }
}

// ------------------------------------------------------------------------------------------ host side
// launch KERNEL<paged, element bytes> of an LlEnc / LlDec parameter block P (kCT threads per CTA)
#define LL_LAUNCH_ELEM(KERNEL, GRID, P, STREAM)                                                                        \
    do {                                                                                                               \
        if ((P).slot_map != nullptr) {                                                                                 \
            if ((P).rawb) KERNEL<true, 2><<<(GRID), kCT, 0, (STREAM)>>>(P);                                            \
            else KERNEL<true, 1><<<(GRID), kCT, 0, (STREAM)>>>(P);                                                     \
        } else {                                                                                                       \
            if ((P).rawb) KERNEL<false, 2><<<(GRID), kCT, 0, (STREAM)>>>(P);                                           \
            else KERNEL<false, 1><<<(GRID), kCT, 0, (STREAM)>>>(P);                                                    \
        }                                                                                                              \
    } while (0)

int fill_planes(const b200kv_kv_desc* kv, PlaneTable* pt) {
    float bins[B200KV_MAX_PLANES];
    for (int i = 0; i < B200KV_MAX_PLANES; ++i) bins[i] = 32.0f;   // no quantiser here; keeps the table valid
    return make_plane_table(kv, bins, bins, pt);
}

struct LlEncWs { size_t hist, err, tab, tile, state, scratch, total; };
LlEncWs ll_enc_ws(int64_t n, int64_t NP, int64_t C, int chunk_tokens, int64_t* rw_out) {
    const int64_t tpp = (C + kCT - 1) / kCT;
    const int64_t rw = (ll_max_words(chunk_tokens) + 1) & ~(int64_t)1;
    LlEncWs w;
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o = (o + bytes + 255) & ~(size_t)255; return at; };
    w.hist = take(sizeof(uint32_t) * n * NP * kSyms);
    w.err = take(sizeof(uint32_t) * n);
    w.tab = take(sizeof(uint32_t) * n * NP * kSyms);
    w.tile = take(sizeof(unsigned long long) * n * NP * tpp);
    w.state = take(sizeof(uint32_t) * n * NP * C);
    w.scratch = take(sizeof(uint16_t) * n * NP * C * rw);
    w.total = o;
    if (rw_out) *rw_out = rw;
    return w;
}

// b200kv_lossless_encode_layers_plan's workspace: the state that lives across calls (error words, payload totals,
// chunk bases, cursor + fail_from, segment bytes), then one call's scratch for npc = planes of at most max_layers
// layers: histograms, tables, tile totals, coder states, scratch rows, and the call's raw rows, staged.
struct LlEnclWs { size_t err, ptotal, cbase, state, totals, hist, tab, tile, cstate, scratch, raw, total; int64_t rw, raw_stride; };
LlEnclWs ll_encl_ws(int64_t n, int64_t npc, int64_t C, int chunk_tokens) {
    const int64_t tpp = (C + kCT - 1) / kCT;
    LlEnclWs w;
    w.rw = (ll_max_words(chunk_tokens) + 1) & ~(int64_t)1;
    w.raw_stride = align16(npc * chunk_tokens * C);
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o = (o + bytes + 255) & ~(size_t)255; return at; };
    w.err = take(sizeof(uint32_t) * n);
    w.ptotal = take(sizeof(unsigned long long) * n);
    w.cbase = take(sizeof(unsigned long long) * n);
    w.state = take(16);
    w.totals = take(sizeof(unsigned long long) * n);
    w.hist = take(sizeof(uint32_t) * n * npc * kSyms);
    w.tab = take(sizeof(uint32_t) * n * npc * kSyms);
    w.tile = take(sizeof(unsigned long long) * n * npc * tpp);
    w.cstate = take(sizeof(uint32_t) * n * npc * C);
    w.scratch = take(sizeof(uint16_t) * n * npc * C * w.rw);
    w.raw = take((size_t)(n * w.raw_stride));
    w.total = o;
    return w;
}

size_t ll_dec_ws(int64_t n, int64_t NP, int64_t C, size_t* off_tile) {
    const int64_t tpp = (C + kCT - 1) / kCT;
    *off_tile = ((size_t)sizeof(LlDecChunk) * n + 255) & ~(size_t)255;
    return *off_tile + sizeof(unsigned long long) * n * NP * tpp;
}

bool shape_ok(int32_t L, int32_t H, int32_t D, int32_t t) {
    return L > 0 && 2 * (int64_t)L <= B200KV_MAX_PLANES && H > 0 && D > 0 && (int64_t)H * D < (1ll << 24) && t > 0 &&
           t <= kMaxTokens;
}

}  // namespace
}  // namespace b200kv

using namespace b200kv;

extern "C" {

int b200kv_lossless_layout(int32_t L, int32_t H, int32_t D, int32_t ntokens, int32_t latent,
                           b200kv_lossless_layout_t* out) {
    return b200kv_lossless_layout_dt(L, H, D, ntokens, latent, B200KV_DT_BF16, out);
}

int b200kv_lossless_layout_dt(int32_t L, int32_t H, int32_t D, int32_t ntokens, int32_t latent, int32_t dtype,
                              b200kv_lossless_layout_t* out) {
    B2_REQUIRE(out != nullptr, "out is NULL");
    B2_REQUIRE(shape_ok(L, H, D, ntokens), "bad shape (L <= 128, H * D < 2^24, 1 <= ntokens <= 4096)");
    B2_REQUIRE(dtype_bytes(dtype) != 0, "dtype must be one of B200KV_DT_*");
    const LlLayout lo = ll_layout(latent ? L : 2 * L, (int64_t)H * D, ntokens, dtype_bytes(dtype) - 1);
    out->off_freq = lo.off_freq;
    out->off_lens = lo.off_lens;
    out->off_raw = lo.off_raw;
    out->off_payload = lo.off_payload;
    out->fixed_bytes = lo.off_payload;
    out->max_stream_bytes = lo.max_stream;
    out->max_total_bytes = lo.max_total;
    return 0;
}

int64_t b200kv_lossless_workspace_bytes(int32_t L, int32_t H, int32_t D, int32_t chunk_tokens, int32_t n_chunks,
                                        int32_t latent, int32_t decode) {
    if (!shape_ok(L, H, D, chunk_tokens) || n_chunks <= 0) return -2;
    const int64_t NP = latent ? L : 2 * (int64_t)L, C = (int64_t)H * D;
    if (decode) {
        size_t off;
        return (int64_t)ll_dec_ws(n_chunks, NP, C, &off);
    }
    return (int64_t)ll_enc_ws(n_chunks, NP, C, chunk_tokens, nullptr).total;
}

int b200kv_lossless_encode(const b200kv_kv_desc* kv, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                           int32_t last_chunk_tokens, void* out, int64_t out_stride, uint64_t* sizes_out,
                           void* workspace, int64_t workspace_bytes, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    LlEnc P;
    if (int rc = fill_planes(kv, &P.pt)) return rc;
    B2_REQUIRE(shape_ok(kv->L, kv->H, kv->D, chunk_tokens), "bad shape (H * D < 2^24, 1 <= chunk_tokens <= 4096)");
    B2_REQUIRE(n_chunks > 0 && n_chunks <= 65535, "n_chunks must be in [1, 65535]");
    B2_REQUIRE(last_chunk_tokens > 0 && last_chunk_tokens <= chunk_tokens, "last_chunk_tokens out of range");
    B2_REQUIRE(out != nullptr && (reinterpret_cast<uintptr_t>(out) & 15) == 0 && (out_stride & 15) == 0,
               "out / out_stride must be 16-byte aligned");
    B2_REQUIRE(sizes_out != nullptr, "sizes_out is NULL");
    B2_REQUIRE(tok_begin >= 0, "tok_begin must be >= 0");
    P.NP = kv_ppl(kv) * kv->L;
    P.L = kv->L; P.H = kv->H; P.D = kv->D; P.C = kv->H * kv->D; P.dtype = kv_dtype(kv);
    P.rawb = kv_elem_bytes(kv) - 1;
    const LlLayout lo = ll_layout(P.NP, P.C, chunk_tokens, P.rawb);
    B2_REQUIRE(out_stride >= lo.max_total, "out_stride smaller than the worst-case container (b200kv_lossless_layout)");
    P.sT = kv->sT; P.sH = kv->sH; P.tok_begin = tok_begin;
    P.slot_map = kv->slot_map;
    P.n_chunks = n_chunks; P.chunk_tokens = chunk_tokens; P.last_chunk_tokens = last_chunk_tokens;
    P.tpp = (P.C + kCT - 1) / kCT;
    P.ntiles = P.NP * P.tpp;
    int64_t rw;
    const LlEncWs w = ll_enc_ws(n_chunks, P.NP, P.C, chunk_tokens, &rw);
    B2_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)w.total, "workspace too small");
    P.rw = (int32_t)rw;
    P.out = static_cast<uint8_t*>(out);
    P.out_stride = out_stride;
    P.sizes_out = sizes_out;
    P.lb = 0; P.nl = P.L; P.npc = P.NP; P.layers_left = 0;        // every plane: the remap is the identity
    P.raw = P.out + lo.off_raw;                                   // raw rows in place (off_raw does not depend on t)
    P.raw_stride = out_stride;
    P.arena = nullptr; P.arena_bytes = 0; P.chunk_base = nullptr; P.cursor = nullptr; P.fail_from = nullptr;
    P.totals = nullptr; P.ptotal = nullptr; P.seg = nullptr;
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    P.hist = reinterpret_cast<uint32_t*>(ws + w.hist);
    P.err = reinterpret_cast<uint32_t*>(ws + w.err);
    P.tab = reinterpret_cast<uint32_t*>(ws + w.tab);
    P.tile = reinterpret_cast<unsigned long long*>(ws + w.tile);
    P.state = reinterpret_cast<uint32_t*>(ws + w.state);
    P.scratch = reinterpret_cast<uint16_t*>(ws + w.scratch);
    B2_CHECK_CUDA(cudaMemsetAsync(ws, 0, w.tab, stream));        // histograms and error words
    const unsigned nslices = (unsigned)((chunk_tokens + kSlice - 1) / kSlice);
    const dim3 ghist((unsigned)P.tpp * nslices, (unsigned)P.NP, (unsigned)n_chunks);
    const dim3 gtile((unsigned)P.tpp, (unsigned)P.NP, (unsigned)n_chunks);
    LL_LAUNCH_ELEM(ll_hist_kernel, ghist, P, stream);
    B2_CHECK_CUDA(cudaGetLastError());
    ll_norm_kernel<<<dim3((unsigned)P.NP, (unsigned)n_chunks), kSyms, 0, stream>>>(P);
    B2_CHECK_CUDA(cudaGetLastError());
    LL_LAUNCH_ELEM(ll_encode_kernel, gtile, P, stream);
    B2_CHECK_CUDA(cudaGetLastError());
    ll_enc_scan_kernel<<<(unsigned)n_chunks, 1024, 0, stream>>>(P);
    B2_CHECK_CUDA(cudaGetLastError());
    ll_compact_kernel<<<gtile, kCT, 0, stream>>>(P);
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int b200kv_lossless_plane_offsets(const void* container, int64_t nbytes, int64_t* out, int32_t n_out) {
    B2_REQUIRE(container != nullptr && out != nullptr && nbytes >= (int64_t)sizeof(b200kv_header), "bad arguments");
    b200kv_header hd;
    memcpy(&hd, container, sizeof(hd));
    LlLayout lo;
    int NP;
    B2_REQUIRE(ll_offsets_header_ok(hd, INT64_MAX, &lo, &NP),
               "not a version-5 or version-6 container of a possible shape, or total_bytes shorter than its fixed sections");
    B2_REQUIRE(n_out >= NP + 1, "out must hold P + 1 offsets (P = 2L, or L for version 6)");
    B2_REQUIRE(nbytes >= lo.off_raw, "buffer shorter than the header, frequency rows and lengths");
    const int64_t C = (int64_t)hd.H * hd.D;
    const uint16_t* lens = reinterpret_cast<const uint16_t*>(static_cast<const uint8_t*>(container) + lo.off_lens);
    int64_t o = lo.off_payload;
    out[0] = o;
    for (int p = 0; p < NP; ++p) {
        for (int64_t c = 0; c < C; ++c) o += lens[p * C + c];
        out[p + 1] = o;
    }
    return o == (int64_t)hd.total_bytes ? 0 : 1;
}

int b200kv_lossless_plane_offsets_device(const void* containers, int64_t stride, int32_t n, int64_t* out, void* stream) {
    B2_REQUIRE(containers != nullptr && out != nullptr && n > 0 && stride >= (int64_t)sizeof(b200kv_header) &&
               (stride & 15) == 0 && (reinterpret_cast<uintptr_t>(containers) & 15) == 0, "bad arguments");
    ll_plane_offsets_kernel<<<(unsigned)n, 1024, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint8_t*>(containers), stride, out);
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// b200kv_lossless_decode_plan and b200kv_lossless_decode_plan_heads: src_head0 == NULL decodes every container whole
// (src_H = dst->H)
static int ll_decode_plan_impl(const void* containers, int64_t containers_bytes, const int64_t* offsets,
                               const int64_t* total_bytes, const int32_t* ntokens, const int64_t* dst_tok,
                               int32_t n_chunks, int32_t max_dtype, const b200kv_kv_desc* dst, uint32_t* status_out,
                               void* workspace, int64_t workspace_bytes, b200kv_lossless_decode_plan_t* plan_out,
                               cudaStream_t stream, int32_t src_H, const int32_t* src_head0, const int32_t* dst_head0,
                               const int32_t* n_heads) {
    B2_REQUIRE(plan_out != nullptr, "plan is NULL");
    LlPlan* plan = reinterpret_cast<LlPlan*>(plan_out);
    plan->magic = 0u;
    LlDec& P = plan->P;
    if (int rc = fill_planes(dst, &P.pt)) return rc;
    B2_REQUIRE(containers && offsets && total_bytes && ntokens && dst_tok && n_chunks > 0 && n_chunks <= 65535,
               "bad chunk arrays");
    B2_REQUIRE(dtype_bytes(max_dtype) != 0, "bad max_dtype");
    B2_REQUIRE(kv_dtype(dst) == max_dtype,
               "the destination's dtype is not the stored one: a lossless container is decoded into its own dtype only");
    B2_REQUIRE(shape_ok(dst->L, dst->H, dst->D, 1), "bad destination shape");
    if (src_head0 == nullptr) src_H = dst->H;
    std::vector<HeadWindow> win;
    if (int rc = plan_head_windows(n_chunks, dst_tok, kv_ppl(dst) == 1, dst->H, dst->D, src_H, src_head0, dst_head0,
                                   n_heads, kCT, &win, &P.wtpp))
        return rc;
    P.NP = kv_ppl(dst) * dst->L;
    P.L = dst->L; P.H = src_H; P.D = dst->D; P.C = src_H * dst->D;
    P.dtype = max_dtype;
    P.rawb = dtype_bytes(max_dtype) - 1;
    P.version = kv_ppl(dst) == 1 ? 6 : 5;
    P.sT = dst->sT; P.sH = dst->sH;
    P.slot_map = dst->slot_map;
    P.n_chunks = n_chunks;
    P.tpp = (P.C + kCT - 1) / kCT;
    P.ntiles = P.NP * P.tpp;
    for (int j = 0; j < n_chunks; ++j) {
        B2_REQUIRE(ntokens[j] > 0 && ntokens[j] <= kMaxTokens, "ntokens must be in [1, 4096]");
        B2_REQUIRE((offsets[j] & 15) == 0, "container offsets must be 16-byte aligned");
        const LlLayout lj = ll_layout(P.NP, P.C, ntokens[j], P.rawb);
        B2_REQUIRE(total_bytes[j] >= lj.off_payload, "container shorter than its fixed sections (truncated or corrupt)");
        B2_REQUIRE(offsets[j] >= 0 && offsets[j] + total_bytes[j] + B200KV_READ_SLACK <= containers_bytes,
                   "containers buffer must extend B200KV_READ_SLACK bytes past the end of every container");
    }
    size_t off_tile;
    const size_t need = ll_dec_ws(n_chunks, P.NP, P.C, &off_tile);
    B2_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)need, "workspace too small");
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    {   // chunk descriptors: small pageable -> device copy (staged by the driver before the call returns)
        LlDecChunk* hc = static_cast<LlDecChunk*>(malloc(sizeof(LlDecChunk) * (size_t)n_chunks));
        B2_REQUIRE(hc != nullptr, "out of host memory");
        for (int j = 0; j < n_chunks; ++j) {
            hc[j].base = static_cast<const uint8_t*>(containers) + offsets[j];
            hc[j].dst_tok = dst_tok[j];
            hc[j].payload_bytes = total_bytes[j] - ll_layout(P.NP, P.C, ntokens[j], P.rawb).off_payload;
            hc[j].t = ntokens[j];
            const HeadWindow& w = win[(size_t)j];
            hc[j].ct0 = w.ct0;
            hc[j].ntw = w.ntw;
            hc[j].cw0 = w.cw0;
            hc[j].cw1 = w.cw1;
            hc[j].dshift = w.dshift;
        }
        cudaError_t e = cudaMemcpyAsync(ws, hc, sizeof(LlDecChunk) * (size_t)n_chunks, cudaMemcpyHostToDevice, stream);
        free(hc);
        B2_CHECK_CUDA(e);
    }
    P.chunks = reinterpret_cast<const LlDecChunk*>(ws);
    P.tile = reinterpret_cast<unsigned long long*>(ws + off_tile);
    P.status = status_out;
    if (status_out) B2_CHECK_CUDA(cudaMemsetAsync(status_out, 0, sizeof(uint32_t) * (size_t)n_chunks, stream));
    ll_tile_sum_kernel<<<dim3((unsigned)((P.ntiles + 3) / 4), (unsigned)n_chunks), 128, 0, stream>>>(P);
    B2_CHECK_CUDA(cudaGetLastError());
    ll_dec_scan_kernel<<<(unsigned)n_chunks, 1024, 0, stream>>>(P);
    B2_CHECK_CUDA(cudaGetLastError());
    plan->magic = kLlPlanMagic;
    return 0;
}

int b200kv_lossless_decode_plan(const void* containers, int64_t containers_bytes, const int64_t* offsets,
                                const int64_t* total_bytes, const int32_t* ntokens, const int64_t* dst_tok,
                                int32_t n_chunks, int32_t max_dtype, const b200kv_kv_desc* dst, uint32_t* status_out,
                                void* workspace, int64_t workspace_bytes, b200kv_lossless_decode_plan_t* plan_out,
                                void* stream) {
    return ll_decode_plan_impl(containers, containers_bytes, offsets, total_bytes, ntokens, dst_tok, n_chunks, max_dtype,
                               dst, status_out, workspace, workspace_bytes, plan_out, static_cast<cudaStream_t>(stream), 0,
                               nullptr, nullptr, nullptr);
}

int b200kv_lossless_decode_plan_heads(const void* containers, int64_t containers_bytes, const int64_t* offsets,
                                      const int64_t* total_bytes, const int32_t* ntokens, const int64_t* dst_tok,
                                      int32_t n_chunks, int32_t max_dtype, const b200kv_kv_desc* dst,
                                      uint32_t* status_out, void* workspace, int64_t workspace_bytes,
                                      b200kv_lossless_decode_plan_t* plan_out, void* stream, int32_t src_H,
                                      const int32_t* src_head0, const int32_t* dst_head0, const int32_t* n_heads) {
    if (plan_out != nullptr) reinterpret_cast<LlPlan*>(plan_out)->magic = 0u;
    B2_REQUIRE(src_head0 != nullptr, "head window arrays are NULL");
    return ll_decode_plan_impl(containers, containers_bytes, offsets, total_bytes, ntokens, dst_tok, n_chunks, max_dtype,
                               dst, status_out, workspace, workspace_bytes, plan_out, static_cast<cudaStream_t>(stream),
                               src_H, src_head0, dst_head0, n_heads);
}

int b200kv_lossless_decode_layers(const b200kv_lossless_decode_plan_t* plan_in, int32_t layer_begin, int32_t layer_end,
                                  void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B2_REQUIRE(plan_in != nullptr, "plan is NULL");
    const LlPlan* plan = reinterpret_cast<const LlPlan*>(plan_in);
    B2_REQUIRE(plan->magic == kLlPlanMagic, "not a plan made by b200kv_lossless_decode_plan");
    LlDec P = plan->P;
    B2_REQUIRE(layer_begin >= 0 && layer_begin < layer_end && layer_end <= P.L, "layer range out of range");
    P.lb = layer_begin;
    P.nl = layer_end - layer_begin;
    const int ppl = P.NP / P.L;
    const dim3 g((unsigned)P.wtpp, (unsigned)(ppl * P.nl), (unsigned)P.n_chunks);
    LL_LAUNCH_ELEM(ll_decode_kernel, g, P, stream);
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int b200kv_lossless_decode(const void* containers, int64_t containers_bytes, const int64_t* offsets,
                           const int64_t* total_bytes, const int32_t* ntokens, const int64_t* dst_tok, int32_t n_chunks,
                           int32_t max_dtype, const b200kv_kv_desc* dst, uint32_t* status_out, void* workspace,
                           int64_t workspace_bytes, void* stream) {
    b200kv_lossless_decode_plan_t plan;
    if (int rc = b200kv_lossless_decode_plan(containers, containers_bytes, offsets, total_bytes, ntokens, dst_tok,
                                             n_chunks, max_dtype, dst, status_out, workspace, workspace_bytes, &plan,
                                             stream))
        return rc;
    return b200kv_lossless_decode_layers(&plan, 0, dst->L, stream);
}

int64_t b200kv_lossless_encode_layers_workspace_bytes(int32_t L, int32_t H, int32_t D, int32_t chunk_tokens,
                                                      int32_t n_chunks, int32_t latent, int32_t max_layers) {
    if (!shape_ok(L, H, D, chunk_tokens) || n_chunks <= 0 || n_chunks > 65535 || max_layers <= 0 || max_layers > L)
        return -2;
    return (int64_t)ll_encl_ws(n_chunks, (latent ? 1 : 2) * (int64_t)max_layers, (int64_t)H * D, chunk_tokens).total;
}

int b200kv_lossless_encode_layers_plan(const b200kv_kv_desc* kv, int64_t tok_begin, int32_t n_chunks,
                                       int32_t chunk_tokens, int32_t last_chunk_tokens, void* arena, int64_t arena_bytes,
                                       void* fixed_out, int64_t fixed_stride, int64_t* seg_sizes_out,
                                       uint64_t* sizes_out, int32_t max_layers, void* workspace, int64_t workspace_bytes,
                                       b200kv_lossless_encode_plan_t* plan_out, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B2_REQUIRE(plan_out != nullptr, "plan is NULL");
    LlEncPlan* plan = reinterpret_cast<LlEncPlan*>(plan_out);
    plan->magic = 0u;
    LlEnc& P = plan->P;
    if (int rc = fill_planes(kv, &P.pt)) return rc;
    B2_REQUIRE(shape_ok(kv->L, kv->H, kv->D, chunk_tokens), "bad shape (H * D < 2^24, 1 <= chunk_tokens <= 4096)");
    B2_REQUIRE(n_chunks > 0 && n_chunks <= 65535, "n_chunks must be in [1, 65535]");
    B2_REQUIRE(last_chunk_tokens > 0 && last_chunk_tokens <= chunk_tokens, "last_chunk_tokens out of range");
    B2_REQUIRE(tok_begin >= 0, "tok_begin must be >= 0");
    B2_REQUIRE(max_layers > 0 && max_layers <= kv->L, "max_layers out of range");
    B2_REQUIRE(seg_sizes_out != nullptr && sizes_out != nullptr, "seg_sizes_out / sizes_out is NULL");
    B2_REQUIRE(arena != nullptr && (reinterpret_cast<uintptr_t>(arena) & 15) == 0 && arena_bytes >= 0,
               "arena must be 16-byte aligned, arena_bytes >= 0");
    B2_REQUIRE(fixed_out != nullptr && (reinterpret_cast<uintptr_t>(fixed_out) & 15) == 0 && (fixed_stride & 15) == 0,
               "fixed_out / fixed_stride must be 16-byte aligned");
    P.NP = kv_ppl(kv) * kv->L;
    P.L = kv->L; P.H = kv->H; P.D = kv->D; P.C = kv->H * kv->D; P.dtype = kv_dtype(kv);
    P.rawb = kv_elem_bytes(kv) - 1;
    const LlLayout lo = ll_layout(P.NP, P.C, chunk_tokens, P.rawb);
    B2_REQUIRE(fixed_stride >= lo.off_raw, "fixed_stride smaller than the fixed image [0, off_raw) (b200kv_lossless_layout)");
    P.sT = kv->sT; P.sH = kv->sH; P.tok_begin = tok_begin;
    P.slot_map = kv->slot_map;
    P.n_chunks = n_chunks; P.chunk_tokens = chunk_tokens; P.last_chunk_tokens = last_chunk_tokens;
    P.tpp = (P.C + kCT - 1) / kCT;
    const LlEnclWs w = ll_encl_ws(n_chunks, (int64_t)kv_ppl(kv) * max_layers, P.C, chunk_tokens);
    B2_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)w.total, "workspace too small");
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    P.rw = (int32_t)w.rw;
    P.out = static_cast<uint8_t*>(fixed_out);
    P.out_stride = fixed_stride;
    P.sizes_out = sizes_out;
    P.err = reinterpret_cast<uint32_t*>(ws + w.err);
    P.ptotal = reinterpret_cast<unsigned long long*>(ws + w.ptotal);
    P.chunk_base = reinterpret_cast<unsigned long long*>(ws + w.cbase);
    P.cursor = reinterpret_cast<unsigned long long*>(ws + w.state);
    P.fail_from = reinterpret_cast<unsigned int*>(ws + w.state + 8);
    P.totals = reinterpret_cast<unsigned long long*>(ws + w.totals);
    P.hist = reinterpret_cast<uint32_t*>(ws + w.hist);
    P.tab = reinterpret_cast<uint32_t*>(ws + w.tab);
    P.tile = reinterpret_cast<unsigned long long*>(ws + w.tile);
    P.state = reinterpret_cast<uint32_t*>(ws + w.cstate);
    P.scratch = reinterpret_cast<uint16_t*>(ws + w.scratch);
    P.raw = ws + w.raw;
    P.raw_stride = w.raw_stride;
    P.arena = static_cast<uint8_t*>(arena);
    P.arena_bytes = arena_bytes;
    P.seg = seg_sizes_out;
    P.lb = 0; P.nl = 0; P.npc = 0; P.ntiles = 0; P.layers_left = 0;    // per call
    // error words, totals, cursor; the fixed images too, so that their gap before off_raw is zero
    B2_CHECK_CUDA(cudaMemsetAsync(ws, 0, w.hist, stream));
    B2_CHECK_CUDA(cudaMemsetAsync(fixed_out, 0, (size_t)fixed_stride * n_chunks, stream));
    ll_encl_init_kernel<<<1, 1, 0, stream>>>(P);
    B2_CHECK_CUDA(cudaGetLastError());
    plan->max_layers = max_layers;
    plan->done = LayerSet::range(0, 0);
    plan->magic = kLlEncPlanMagic;
    return 0;
}

int b200kv_lossless_encode_layers(b200kv_lossless_encode_plan_t* plan_in, int32_t layer_begin, int32_t layer_end,
                                  void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B2_REQUIRE(plan_in != nullptr, "plan is NULL");
    LlEncPlan* plan = reinterpret_cast<LlEncPlan*>(plan_in);
    B2_REQUIRE(plan->magic == kLlEncPlanMagic, "not a plan made by b200kv_lossless_encode_layers_plan");
    LlEnc P = plan->P;
    B2_REQUIRE(layer_begin >= 0 && layer_begin < layer_end && layer_end <= P.L, "layer range out of range");
    B2_REQUIRE(layer_end - layer_begin <= plan->max_layers, "more layers than the plan's workspace holds");
    const LayerSet bits = LayerSet::range(layer_begin, layer_end);
    B2_REQUIRE(!plan->done.intersects(bits), "a layer of the range was encoded before");
    P.lb = layer_begin;
    P.nl = layer_end - layer_begin;
    P.npc = (P.NP / P.L) * P.nl;
    P.ntiles = P.npc * P.tpp;
    P.layers_left = P.L - plan->done.count() - bits.count();
    const int n = P.n_chunks;
    B2_CHECK_CUDA(cudaMemsetAsync(P.hist, 0, sizeof(uint32_t) * (size_t)n * P.npc * kSyms, stream));
    const unsigned nslices = (unsigned)((P.chunk_tokens + kSlice - 1) / kSlice);
    const dim3 ghist((unsigned)P.tpp * nslices, (unsigned)P.npc, (unsigned)n);
    const dim3 gtile((unsigned)P.tpp, (unsigned)P.npc, (unsigned)n);
    LL_LAUNCH_ELEM(ll_hist_kernel, ghist, P, stream);
    ll_norm_kernel<<<dim3((unsigned)P.npc, (unsigned)n), kSyms, 0, stream>>>(P);
    LL_LAUNCH_ELEM(ll_encode_kernel, gtile, P, stream);
    ll_enc_scan_kernel<<<(unsigned)n, 1024, 0, stream>>>(P);
    ll_place_kernel<<<1, 1024, 0, stream>>>(P);
    if (P.rawb) {   // one-byte elements have no raw rows, and their segments no raw part
        // ~16 KB of raw rows per CTA pass; at most 64 CTAs per chunk
        const int64_t raw_bytes = align16((int64_t)P.npc * P.chunk_tokens * P.C) + 16;
        const unsigned rx = (unsigned)std::min<int64_t>(64, (raw_bytes + 16 * 256 * 4 - 1) / (16 * 256 * 4));
        ll_raw_copy_kernel<<<dim3(rx, (unsigned)n), 256, 0, stream>>>(P);
    }
    ll_compact_kernel<<<gtile, kCT, 0, stream>>>(P);
    B2_CHECK_CUDA(cudaGetLastError());
    plan->done.add(bits);
    return 0;
}

int b200kv_lossless_encode_layers_finish(const b200kv_lossless_encode_plan_t* plan_in, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B2_REQUIRE(plan_in != nullptr, "plan is NULL");
    const LlEncPlan* plan = reinterpret_cast<const LlEncPlan*>(plan_in);
    B2_REQUIRE(plan->magic == kLlEncPlanMagic, "not a plan made by b200kv_lossless_encode_layers_plan");
    const LlEnc& P = plan->P;
    B2_REQUIRE(plan->done == LayerSet::range(0, P.L), "a layer was never encoded");
    ll_finish_kernel<<<(P.n_chunks + 127) / 128, 128, 0, stream>>>(P);
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // extern "C"
