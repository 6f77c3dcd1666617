// codec.cu -- CacheGen encode / decode kernels for sm_90a and their C-ABI entry points.
//
// Replaces (reference paths relative to the LMCache v0.1.2 tree):
//   encode: lmcache/storage_backend/serde/cachegen_encoder.py:266-325 (encode_function) incl. the three
//           torchac_cuda calls, collect_bytes and the pickle container (cachegen_basics.py:131-136)
//   decode: lmcache/storage_backend/serde/cachegen_decoder.py:52-106,143-202
//
// Three container versions share these kernels (include/b200kv.h): 1 = arithmetic coder, 2 = rANS, both with the
// reference's CDF tensor as a section; 3 (default) = rANS streams that carry their own symbol histogram, from which the
// decoder rebuilds the CDF (ac_core.cuh: stream header; DESIGN.md 3.9).
//
// Thread mapping: one entropy-coder stream = one (plane nl, channel c) = one thread; a CTA owns a
// tile of CT consecutive channels of one plane (and one <=256-token group).  Global KV reads/writes are
// then naturally coalesced along the channel dimension (a warp touches 64 contiguous bytes per token)
// and the tile's byte streams are contiguous in the container.  The coder writes each stream to a temp
// row in global memory; stream compaction (collect_bytes in the reference) is a separate scan + gather
// pass (enc_scan_kernel, compact_kernel) that stages a tile's byte range in shared memory and writes it
// with 16-byte stores, so no CTA ever waits on another one.  DESIGN.md section 3 has the per-kernel story.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "ac_core.cuh"
#include "common.cuh"

namespace b200kv {

constexpr int CT = 128;            // streams (threads) per tile
constexpr int SPW = 6;             // 5-bit symbols packed per 32-bit word in shared memory
constexpr int SYMW = 43;           // words per symbol row: ceil(256 / 6); odd -> conflict-free columns
constexpr int PAIRW = 33;          // split mode: words per CDF-pair row (32 symbols + cdf[32]); odd
constexpr int TEMPW_FUSED = 40;    // words per stream in the tile's temp rows: an own-CDF stream of <= 256 symbols
                                   //   costs <= 1267.9 ideal bits under the rounded CDF (width >= n*65504/256 - 0.02)
                                   //   + < 0.001 bits of truncation + 2 termination bits = 1269.95 bits -> 159 bytes,
                                   //   40 words (DESIGN.md 3.2; tests/ac_edges.py own_bound_bits)
constexpr int TEMPW_SPLIT = 132;   // foreign CDF (chunk > 256 tokens): <= 16 bits / symbol + termination; 16-byte rows
constexpr int TEMPW_FUSED_RANS = 48;   // rANS, own-CDF streams: <= 95 renormalisation halfwords for ANY symbol order
                                       //   (ideal <= 1268.5 bits, < 1 bit of overshoot per step; DESIGN.md 3.7); the 32-bit
                                       //   final state goes to its own array.  Split mode: <= 1 halfword per symbol = 128 words
constexpr int CODER_AC = 0, CODER_RANS = 1;   // payload coder; B2KV container version = coder + 1 ...
constexpr int CODER_RANS_COMPACT = 2;         // ... 3 = rANS payload + compact side information (ac_core.cuh, make_layout)
constexpr int kHdrRowWords = 8;               // version 3: header words 2..8 of a long stream header, in front of the rANS part
constexpr int TEMPW_FUSED_RANS_HDR = TEMPW_FUSED_RANS + kHdrRowWords;

struct EncParams {
    PlaneTable pt;
    int64_t sT, sH, tok_begin;
    const int64_t* slot_map;         // paged KV: token i of the call lives in row slot_map[i] of every plane; NULL = row i
    int32_t L, H, D, C, dtype;
    int32_t n_chunks, chunk_tokens, last_chunk_tokens, tpp;   // tpp = tiles per plane
    int32_t tiles_full, tempw;                                 // tiles per full chunk; words per temp row
    int32_t stage_bytes;                                       // compact_kernel: bytes of shared-memory stage per CTA
    int32_t coder;                                             // CODER_AC | CODER_RANS (the payload coder)
    int32_t compact;                                           // 1 = container version 3 (histogram in the stream, u8 half-lengths)
    int32_t ppl;                                               // planes per layer: 2 (K, V) or 1 (latent KV, version 4)
    uint8_t* out;
    int64_t out_stride;
    uint64_t* sizes_out;
    uint32_t* temp;                  // [n_tiles][CT][tempw] coder output before compaction
    uint32_t* rstate;                // rANS: [n_tiles][CT] final coder states (the first 4 bytes of every stream); version 3:
                                     //   [n_tiles][CT] records of 4 words {header word 0, header word 1, state, header bytes}
    uint32_t* tile_tot;              // [n_chunks][tiles_full] bytes per tile, then exclusive prefix (in place)
    unsigned long long* totals;      // [n_chunks] payload bytes
    unsigned int* err;               // [n_chunks]
    // encode_kernel<FUSED = true> (persistent): the next work item to claim, and per (chunk, launch plane) the number of
    // absmax items done; both zero at launch
    unsigned int* ticket;
    unsigned int* ready;             // [n_chunks][ppl * nlay]
    int32_t vec;                     // every plane's rows allow 128-bit loads (absmax)
    int32_t lb, nlay;                // this launch codes layers [lb, lb + nlay): planes lb.. and L + lb.. (all: 0, L)
    // b200kv_encode_layers only (NULL / 0 otherwise): the payload goes to a device arena instead of out + j * out_stride
    uint8_t* arena;
    int64_t arena_bytes;
    unsigned long long* chunk_base;  // [n_chunks] arena offset of chunk j's bytes of this call, ~0 = chunk failed
    unsigned long long* cursor;      // first free arena byte (device-held across calls)
    unsigned int* fail_from;         // first failed chunk (n_chunks: none); every later chunk fails too
    unsigned long long* ptotal;      // [n_chunks] payload bytes of every call so far
    int64_t* seg;                    // [n_chunks][2L][2] (arena offset, bytes) per plane; mapped host memory
    int32_t layers_left;             // layers not yet encoded after this call (arena reserve, place_kernel)
};
static_assert(sizeof(EncParams) < kMaxParamBytes, "EncParams must stay under 4 KB of kernel parameters");

// plane of the launch's local plane index: K planes lb.., then V planes L + lb.. (the identity when lb = 0, nlay = L).
// A latent KV (ppl = 1) has local < nlay throughout: planes lb..
__device__ __forceinline__ int launch_plane(const EncParams& P, int local) {
    return local + (local < P.nlay ? P.lb : P.L - P.nlay + P.lb);
}

// section offsets of a container of this call (encode and decode parameter blocks alike)
template <class Prm>
__device__ __forceinline__ Layout layout_of(const Prm& P, int t) {
    return make_layout(P.L, P.C, t, P.compact, P.ppl);
}

// stream lengths section: int32 bytes (versions 1, 2) or u8 bytes / 2 (version 3: header + rANS stream, even, <= 230 bytes)
__device__ __forceinline__ uint32_t load_len(const uint8_t* sec, int64_t idx, bool compact) {
    return compact ? 2u * (uint32_t)sec[idx] : (uint32_t)reinterpret_cast<const int32_t*>(sec)[idx];
}
__device__ __forceinline__ void store_len(uint8_t* sec, int64_t idx, uint32_t len, bool compact) {
    if (compact) sec[idx] = (uint8_t)(len >> 1);
    else reinterpret_cast<int32_t*>(sec)[idx] = (int32_t)len;
}

// Version 3: build the stream's header (ac_core.cuh) -- which symbols occur and how often.  The bytes are assembled in
// a register, a word at a time: words 0 and 1 (mask + the first counts: all there is for streams with few symbols) are
// returned and go to the tile's side array (one coalesced 16-byte record per stream, next to the rANS state), words 2..8
// -- streams with many symbols only -- go to the front of the stream's temp row.  Returns the header length (even,
// <= kHdrMax).  cnt[i] is 0 for i >= nb by construction.
__device__ __forceinline__ uint32_t build_stream_header(const uint32_t (&cnt)[32], uint32_t mask, uint32_t wany, int nb,
                                                        uint32_t* rowfront, uint32_t& w0, uint32_t& w1) {
    // mask: bit i <=> cnt[i] != 0; wany: the OR of the masks of the warp's lanes (a symbol nobody uses costs one test)
    const uint32_t top = 0x80000000u >> __clz((int)mask);        // the last set bit: its count is implied
    const uint32_t st = mask & ~top;                             // symbols whose count is stored
    const uint32_t mb = (uint32_t)hdr_mask_bytes(nb);
    w0 = 0u;
    w1 = 0u;
    uint32_t widx = 0u, acc = mask, sh = 8u * mb;                // sh = 8 * bytes held in acc
    auto flush = [&]() {
        if (widx == 0u) w0 = acc;
        else if (widx == 1u) w1 = acc;
        else rowfront[widx - 2u] = acc;
        ++widx;
        acc = 0u;
        sh = 0u;
    };
    if (sh == 32u) flush();
#pragma unroll
    for (int i = 0; i < 32; ++i) {
        if (i < nb && ((wany >> i) & 1u) && ((st >> i) & 1u)) {
            acc |= cnt[i] << sh;
            sh += 8u;
            if (sh == 32u) flush();
        }
    }
    uint32_t hlen = mb + (uint32_t)__popc(st);
    hlen += hlen & 1u;
    if (sh != 0u) flush();
    return hlen;
}

// the mask of a stream header at p (2-byte aligned), restricted to the plane's nb symbols
__device__ __forceinline__ uint32_t read_header_mask(const uint8_t* p, int nb) {
    uint32_t m = *reinterpret_cast<const uint16_t*>(p);
    if (nb > 16) m |= (uint32_t)*reinterpret_cast<const uint16_t*>(p + 2) << 16;
    if (nb <= 8) m &= 0xffu;
    return nb >= 32 ? m : m & ((1u << nb) - 1u);
}

__device__ __forceinline__ int chunk_tokens_of(const EncParams& P, int j) {
    return j == P.n_chunks - 1 ? P.last_chunk_tokens : P.chunk_tokens;
}

// ------------------------------------------------------------------------------------------ absmax
// max1 = amax(|x|, channels) per (plane, token), kept in the input half dtype
// (cachegen_encoder.py:54-55).  |x| ordering == integer ordering of (bits & 0x7fff); a NaN in the row
// wins (pattern above inf), like torch.amax.  One warp per row, 128-bit loads when alignment allows.
// Chunks of <= 256 tokens do not launch absmax_kernel: the persistent encode_kernel<FUSED = true> computes the maxima
// itself, as work items ordered ahead of the tiles that read them (encode_kernel).  A separate kernel cannot hide this
// HBM-bound pass under the instruction-bound coder: round 2 tried it on a second stream (128-thread blocks with <= 32
// registers) with no gain -- both coder kernels fill the SM's shared memory with their own CTAs (7 x 32.5 KB, 12 x 18.6
// KB incl. the 1 KB the system reserves per CTA), so not even a block without shared memory finds room.  Chunks of more
// than 256 tokens still launch it: their chunk-wide CDF (cdf_kernel) needs every maximum of the chunk first.
//
// The bits of |x| of one row (C channels at row, head pitch sH) reduced to their maximum over the warp.
template <bool VEC>
__device__ __forceinline__ uint32_t row_absmax(const EncParams& P, const uint16_t* row, int lane) {
    uint32_t m = 0;
    if (VEC) {
        const int vec_per_head = P.D >> 3;
        const int nvec = P.H * vec_per_head;
        // batches of 4 loads per lane, all in flight before the first is used (a slot past the row reads as 0)
        constexpr int B = 4;
        for (int v0 = lane; v0 < nvec; v0 += 32 * B) {
            uint4 q[B];
#pragma unroll
            for (int b = 0; b < B; ++b) {
                const int v = v0 + 32 * b;
                const int h = v / vec_per_head, dv = v - h * vec_per_head;
                q[b] = v < nvec ? __ldg(reinterpret_cast<const uint4*>(row + (int64_t)h * P.sH + dv * 8)) : make_uint4(0, 0, 0, 0);
            }
#pragma unroll
            for (int b = 0; b < B; ++b) {
                const uint32_t w[4] = {q[b].x, q[b].y, q[b].z, q[b].w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint32_t a = w[k] & 0x7fff7fffu;
                    m = max(m, max(a & 0xffffu, a >> 16));
                }
            }
        }
    } else {
        for (int c = lane; c < P.C; c += 32) {
            const int h = c / P.D, d = c - h * P.D;
            m = max(m, (uint32_t)(__ldg(row + (int64_t)h * P.sH + d) & 0x7fffu));
        }
    }
    return __reduce_max_sync(0xffffffffu, m);
}

template <bool VEC, bool PAGED>
__global__ void __launch_bounds__(256) absmax_kernel(EncParams P, int64_t total_tokens) {
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t nrows = (int64_t)P.ppl * P.nlay * total_tokens;
    if (warp >= nrows) return;
    const int nl = launch_plane(P, (int)(warp / total_tokens));
    const int64_t T = warp % total_tokens;
    const uint16_t* row = P.pt.p[nl] + tok_row<PAGED>(P.slot_map, P.tok_begin + T) * P.sT;
    const uint32_t m = row_absmax<VEC>(P, row, lane);
    if (lane == 0) {
        const int j = (int)(T / P.chunk_tokens);
        const int tj = chunk_tokens_of(P, j);
        const Layout lo = layout_of(P, tj);
        uint16_t* maxes = reinterpret_cast<uint16_t*>(P.out + (int64_t)j * P.out_stride + lo.off_maxes);
        maxes[(int64_t)nl * tj + (T - (int64_t)j * P.chunk_tokens)] = (uint16_t)m;
    }
}

// ------------------------------------------------------------------------------------------ helpers
// block-wide exclusive scan of one uint32 per thread (CT threads); returns exclusive prefix, total in *total
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* s_warp, uint32_t* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t n = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += n;
    }
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    uint32_t base = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < CT / 32; ++w) {
        const uint32_t s = s_warp[w];
        if (w < wid) base += s;
        tot += s;
    }
    *total = tot;
    return base + inc - v;
}

// tile -> (chunk j, group g, plane nl, channel tile ct); tiles of a chunk are ordered (g, nl, ct), which is the
// order of the streams in the container payload.  Returns false for tiles beyond the (ragged) last chunk.
// A launch over layers [lb, lb + nlay) has tiles_full = ppl * nlay * tpp tiles per chunk (one group: v3 / v4 only); its
// tile_in_chunk counts the launch's tiles, and the local plane maps to the real one with one select (launch_plane).
struct TileId { int j, g, nl, ct, t, tok0, gt, tile_in_chunk; };
__device__ __forceinline__ bool decode_tile(const EncParams& P, uint32_t tile, TileId* id) {
    const uint32_t per_group = (uint32_t)P.ppl * P.nlay * P.tpp;
    const uint32_t j = tile / (uint32_t)P.tiles_full;
    const uint32_t rem = tile - j * (uint32_t)P.tiles_full;
    id->j = (int)j;
    id->tile_in_chunk = (int)rem;
    id->t = chunk_tokens_of(P, (int)j);
    id->g = (int)(rem / per_group);
    if (id->g * kGroup >= id->t) return false;
    const uint32_t rem2 = rem - (uint32_t)id->g * per_group;
    const int local = (int)(rem2 / P.tpp);
    id->ct = (int)(rem2 - (uint32_t)local * P.tpp);
    id->nl = launch_plane(P, local);
    id->tok0 = id->g * kGroup;
    id->gt = min(kGroup, id->t - id->tok0);
    return true;
}

// Walk one stream's gt tokens in register double-buffered batches of BT loads (the loads of batch b+1 are in flight
// while batch b is consumed) and hand every quantised symbol to `f(symbol)`, in token order.  Used where symbols are
// consumed on the fly (chunk-wide histogram, coding against a chunk-wide CDF).
template <int DT, bool PAGED, int BT, class F>
__device__ __forceinline__ void for_each_symbol(const uint16_t* cbase, const int64_t* slot_map, int64_t tokabs, int64_t s1,
                                                int gt, const float* fac, float maxq, F&& f) {
    const int nbatch = (gt + BT - 1) / BT;
    uint16_t xa[BT], xb[BT];
    auto load = [&](uint16_t (&x)[BT], int b) {
        const int tk = b * BT;
#pragma unroll
        for (int k = 0; k < BT; ++k)
            x[k] = tk + k < gt ? __ldg(cbase + tok_row<PAGED>(slot_map, tokabs + tk + k) * s1) : (uint16_t)0;
    };
    auto use = [&](const uint16_t (&x)[BT], int b) {
        const int tk = b * BT;
        uint32_t q[BT];
#pragma unroll
        for (int k = 0; k < BT; ++k) q[k] = quant_symbol(half_to_float(x[k], DT), fac[min(tk + k, kGroup - 1)], maxq);
#pragma unroll
        for (int k = 0; k < BT; ++k)
            if (tk + k < gt) f(q[k]);
    };
    load(xa, 0);
    for (int b = 0; b < nbatch; b += 2) {
        if (b + 1 < nbatch) load(xb, b + 1);
        use(xa, b);
        if (b + 1 < nbatch) {
            if (b + 2 < nbatch) load(xa, b + 2);
            use(xb, b + 1);
        }
    }
}

// Same walk from the last token to the first (rANS codes a stream back to front so that the decoder runs forwards).
template <int DT, bool PAGED, int BT, class F>
__device__ __forceinline__ void for_each_symbol_rev(const uint16_t* cbase, const int64_t* slot_map, int64_t tokabs, int64_t s1,
                                                    int gt, const float* fac, float maxq, F&& f) {
    const int nbatch = (gt + BT - 1) / BT;
    uint16_t xa[BT], xb[BT];
    auto load = [&](uint16_t (&x)[BT], int b) {
        const int tk = b * BT;
#pragma unroll
        for (int k = 0; k < BT; ++k)
            x[k] = tk + k < gt ? __ldg(cbase + tok_row<PAGED>(slot_map, tokabs + tk + k) * s1) : (uint16_t)0;
    };
    auto use = [&](const uint16_t (&x)[BT], int b) {
        const int tk = b * BT;
        uint32_t q[BT];
#pragma unroll
        for (int k = 0; k < BT; ++k) q[k] = quant_symbol(half_to_float(x[k], DT), fac[min(tk + k, kGroup - 1)], maxq);
#pragma unroll
        for (int k = BT - 1; k >= 0; --k)
            if (tk + k < gt) f(q[k]);
    };
    load(xa, nbatch - 1);
    for (int b = nbatch - 1; b >= 0; b -= 2) {
        if (b >= 1) load(xb, b - 1);
        use(xa, b);
        if (b >= 1) {
            if (b >= 2) load(xa, b - 2);
            use(xb, b - 1);
        }
    }
}

// The rANS encoder step the kernels below run, rans_put, lives in ac_core.cuh, where the test-only device build
// (tests/devsim) can reach it.

// ------------------------------------------------------------------------------------------ encode
// One tile = CT consecutive channels of one plane and one <= 256-token group; one thread = one coder stream.
// FUSED (chunk <= 256 tokens): quantise -> 5-bit symbols in shared memory + thread-private histogram -> CDF (the
//   33-entry rows are contiguous in smem and in the container: one coalesced copy) -> arithmetic coding.  The kernel is
//   persistent and also computes the maxima the tiles read (absmax_item).
// !FUSED (chunk > 256 tokens): the chunk-wide CDF was produced by cdf_kernel; one tile codes one group, quantising
//   on the fly.
// Coder output goes to the tile's temp rows in global memory (sparse 32-bit stores, merged in L2); stream lengths go to
// the container; the tile's byte total goes to tile_tot.  Compaction into the contiguous payload (collect_bytes in the
// reference) is done by scan_kernel + compact_kernel afterwards.
//
// Persistent schedule (FUSED): a unit is one (chunk j, launch plane); its work is kAbsItems absmax items (kAbsRows token
// rows each, over all C channels) and tpp tiles.  Tickets are claimed with one atomicAdd each and come in steps of
// kAbsItems + tpp: step s holds the absmax items of unit s, then the tiles of unit s - kAbsLead.  A tile waits until its
// unit's ready counter shows every absmax item done.
// Measured on the H100 (DESIGN.md 3.2): 8 rows and a lead of 16 units beat 4 rows and leads of 8, 24 and 32.
constexpr int kAbsRows = 8;                   // token rows per absmax item: 2 per warp
constexpr int kAbsItems = kGroup / kAbsRows;  // absmax items per unit (a ragged chunk's unused items only count as done)
constexpr int kAbsLead = 16;                  // units by which a unit's absmax items run ahead of its tiles

// The maxima of token rows [item * kAbsRows, +kAbsRows) of one unit, written to the container's maxes section exactly as
// absmax_kernel writes them; then the unit's ready counter goes up by one.  Uses no shared memory.  An item does not get
// faster with more bytes in flight: 8 loads per lane measured the same, bulk copies into shared-memory slots slower
// (DESIGN.md 3.2).
template <bool PAGED>
__device__ __forceinline__ void absmax_item(const EncParams& P, int unit, int item) {
    const int nloc = P.ppl * P.nlay;
    const int j = unit / nloc;
    const int nl = launch_plane(P, unit - j * nloc);
    const int tj = chunk_tokens_of(P, j);
    const Layout lo = layout_of(P, tj);
    uint16_t* maxes = reinterpret_cast<uint16_t*>(P.out + (int64_t)j * P.out_stride + lo.off_maxes) + (int64_t)nl * tj;
    const int64_t tok0 = P.tok_begin + (int64_t)j * P.chunk_tokens;
    const int lane = threadIdx.x & 31;
    const int r0 = item * kAbsRows, r1 = min(tj, (item + 1) * kAbsRows);
    for (int r = r0 + (threadIdx.x >> 5); r < r1; r += CT / 32) {
        const uint16_t* row = P.pt.p[nl] + tok_row<PAGED>(P.slot_map, tok0 + r) * P.sT;
        const uint32_t m = P.vec ? row_absmax<true>(P, row, lane) : row_absmax<false>(P, row, lane);
        if (lane == 0) {
            maxes[r] = (uint16_t)m;
            __threadfence();
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(P.ready + unit) : "memory");
}

template <bool FUSED, int DT, bool PAGED, int CODER, class TileOf>
__device__ __forceinline__ void encode_tile(const EncParams& P, TileOf tile_of, uint32_t* smem, uint32_t* s_warp) {
    // FUSED : symbol rows u32[CT][SYMW] | cdf rows u16[CT][33] (also the histogram) | fac[256] (later fl32(n/t)[257])
    // !FUSED: pair rows u32[CT][33]                                                 | fac[256]
    constexpr int ROWS_W = FUSED ? CT * SYMW : 0;
    constexpr int TAB_W = FUSED ? (CT * kLp * 2 + 3) / 4 : CT * PAIRW;
    uint32_t* rows = smem;
    uint32_t* tab = smem + ROWS_W;
    float* fac = reinterpret_cast<float*>(smem + ((ROWS_W + TAB_W + 3) & ~3));

    const int tid = threadIdx.x;
    TileId id;
    const uint32_t tile = tile_of();
    if (!decode_tile(P, tile, &id)) return;
    const int NL = P.ppl * P.L;
    const int j = id.j, nl = id.nl, ct = id.ct, t = id.t, gt = id.gt;
    const int c = ct * CT + tid;
    const bool active = c < P.C;
    const int ncols = min(CT, P.C - ct * CT);

    uint8_t* cont = P.out + (int64_t)j * P.out_stride;
    const Layout lo = layout_of(P, t);
    const uint16_t* maxes = reinterpret_cast<const uint16_t*>(cont + lo.off_maxes) + (int64_t)nl * t + id.tok0;
    const float maxq = P.pt.maxq[nl];
    const int64_t s1 = P.sT;
    if (FUSED) {
        // Wait for the unit's kAbsItems absmax items.  Why this wait always ends, whatever order the hardware launches or
        // schedules CTAs in: tickets are handed out in increasing order, one atomicAdd each, and a CTA claims a ticket
        // only while it is running and only after finishing its previous item.  The absmax items of this tile's unit
        // hold smaller tickets (step u against step u + kAbsLead), so each of them was claimed before this tile was, by
        // a CTA that is resident now or has finished.  An absmax item waits on nothing, so each one completes.  No work
        // item waits on a later ticket: there is no cycle, and nothing spins on work that is not yet running.
        if (tid == 0) {
            const unsigned int* rd = P.ready + tile / (uint32_t)P.tpp;
            uint32_t ns = 32u;
            for (;;) {
                uint32_t v;
                asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(rd) : "memory");
                if (v >= (uint32_t)kAbsItems) break;
                __nanosleep(ns);
                ns = min(2u * ns, 1024u);
            }
        }
        __syncthreads();
    }
    // FUSED: "safe" factors (an infinite factor becomes NaN: same symbols, and pass 1 can skip the range check).  The
    // maxima of this launch are read past L1 (__ldcg): L1 is not coherent with the other SMs' writes.
    for (int i = tid; i < gt; i += CT)
        fac[i] = FUSED ? quant_factor_safe(maxq, half_to_float(__ldcg(maxes + i), DT))
                       : quant_factor(maxq, half_to_float(maxes[i], DT));
    if (FUSED) for (int i = gt + tid; i < kGroup + 8; i += CT) fac[i] = 0.0f;      // padded slots of the last batch

    const int h = active ? c / P.D : 0;
    // first token of this tile in the call's token numbering; cbase = this stream's channel in row 0 of the plane
    const int64_t tokabs = P.tok_begin + (int64_t)j * P.chunk_tokens + id.tok0;
    const uint16_t* cbase = P.pt.p[nl] + (int64_t)h * P.sH + (active ? c - h * P.D : 0);
    const uint16_t* src = cbase + (PAGED ? 0 : tokabs * P.sT);          // !PAGED: token tk is at src + tk * sT
    uint32_t* trow = P.temp + ((int64_t)tile * CT + tid) * P.tempw;
    uint32_t cap = (uint32_t)P.tempw;
    // keep the row pointer and the capacity as plain register values: otherwise every flush re-derives the address
    // from (tile, tid, tempw, base) with six extra instructions
    asm volatile("" : "+l"(trow), "+r"(cap));
    uint32_t len = 0u, hlen = 0u;

    if (FUSED) {
        uint32_t* myrow = rows + tid * SYMW;
        uint16_t* cdfr = reinterpret_cast<uint16_t*>(tab);
        uint16_t* crow = cdfr + tid * kLp;
        uint16_t* hist = crow;
#pragma unroll
        for (int i = 0; i < kLp; ++i) crow[i] = 0;
        // No L2 prefetch of the tile's rows: its unit's absmax items read them shortly before, and a prefetch burst
        // per tile made the encode slower (DESIGN.md 3.2).
        __syncthreads();   // fac ready
        if (active) {
            // ---- pass 1: batches of 12 tokens (two packed words), register double-buffered: the loads of batch b+1
            // are in flight while batch b is quantised, so a warp never sits out a full L2 round trip per batch.
            // Slots past the group's end (last word / last batch) read as x = 0 with factor 0 and are quantised like
            // the rest; their known symbol is taken out of the histogram afterwards, and pass 2 never reads them.
            constexpr int NB = 2, BT = NB * SPW;
            const int nbatch = (gt + BT - 1) / BT;
            uint16_t xa[BT], xb[BT];
            const uint32_t s1u = (uint32_t)s1;
            const uint32_t two = 2u * (uint32_t)min(P.n_chunks, 1);      // 2, but opaque to the compiler
            auto load = [&](uint16_t (&x)[BT], int b) {
                const int tk = b * BT;
                if constexpr (PAGED) {
                    const int64_t* sm = P.slot_map + tokabs + tk;
#pragma unroll
                    for (int k = 0; k < BT; ++k) x[k] = tk + k < gt ? __ldg(cbase + __ldg(sm + k) * s1) : (uint16_t)0;
                } else {
                    // token tk + k is one row further than token tk + k - 1: ONE IMAD.WIDE.U32 per address (row
                    // pitch x 2, the 2 from a register ptxas cannot fold, added to the previous address) instead of the
                    // 64-bit add chains the compiler builds from the pointer arithmetic (fewer than
                    // half the instructions per load).  The chain of twelve is off the critical path: the batch is a prefetch.
                    const uint16_t* q = src + (int64_t)tk * s1;
                    if (tk + BT <= gt) {
#pragma unroll
                        for (int k = 0; k < BT; ++k) {
                            x[k] = __ldg(q);
                            asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(q) : "r"(s1u), "r"(two));
                        }
                    } else {
#pragma unroll
                        for (int k = 0; k < BT; ++k) {
                            x[k] = tk + k < gt ? __ldg(q) : (uint16_t)0;
                            asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(q) : "r"(s1u), "r"(two));
                        }
                    }
                }
            };
            auto quantise = [&](const uint16_t (&x)[BT], int b) {
                const int tk = b * BT;
                // all symbols of the batch first (independent chains), then the histogram read-modify-writes: those
                // may alias each other, so interleaving them with the arithmetic would serialise the whole batch
                uint32_t q[BT];
#pragma unroll
                for (int k = 0; k < BT; ++k) q[k] = quant_symbol_nc(half_to_float(x[k], DT), fac[tk + k], maxq);
#pragma unroll
                for (int half = 0; half < NB; ++half) {
                    if (tk + half * SPW < gt) {
                        uint32_t word = 0u;
#pragma unroll
                        for (int k = 0; k < SPW; ++k) {
                            hist[q[half * SPW + k]] += 1;               // symbols are <= 30 by construction
                            word |= q[half * SPW + k] << (5 * k);
                        }
                        myrow[b * NB + half] = word;
                    }
                }
            };
            load(xa, 0);
            for (int b = 0; b < nbatch; b += 2) {
                if (b + 1 < nbatch) load(xb, b + 1);
                quantise(xa, b);
                if (b + 1 < nbatch) {
                    if (b + 2 < nbatch) load(xa, b + 2);
                    quantise(xb, b + 1);
                }
            }
            const int pad = (gt + SPW - 1) / SPW * SPW - gt;            // padded slots in the last word
            if (pad) hist[quant_symbol(0.0f, 0.0f, maxq)] -= (uint16_t)pad;
        }
        __syncthreads();   // every thread is done with fac: reuse it as the fl32(n / t) table
        {
            const float tf = (float)t;
            for (int n = tid; n <= t; n += CT) fac[n] = fdiv((float)n, tf);
        }
        __syncthreads();
        if (active) {
            // ---- CDF from the thread's own histogram, written over it (counts -> registers first)
            uint32_t cnt[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) cnt[i] = hist[i];
            // symbols no lane of the warp uses are skipped (their cdf entries follow from the previous one)
            uint32_t mask = 0u;
#pragma unroll
            for (int i = 0; i < 32; ++i) mask |= (cnt[i] != 0u ? 1u : 0u) << i;
            const uint32_t wany = __reduce_or_sync(__activemask(), mask);
            CdfAccum2 acc;
            acc.init();
#pragma unroll
            for (uint32_t i = 0; i < 32u; ++i) {
                crow[i] = (uint16_t)acc.value(i);
                if ((wany >> i) & 1u) acc.absorb(fac[cnt[i]]);
            }
            crow[32] = (uint16_t)acc.value(32u);
            // version 3 keeps the histogram instead of the CDF row (the CDF is a function of it): the stream's header
            if (P.compact) {
                uint32_t w0, w1;
                hlen = build_stream_header(cnt, mask, wany, 2 * ((int)maxq + 1), trow, w0, w1);
                reinterpret_cast<uint2*>(P.rstate)[((int64_t)tile_of() * CT + tid) * 2] = make_uint2(w0, w1);
            }
        }
        __syncthreads();
        if (!P.compact) {   // the tile's 33-entry rows are contiguous in smem and in the container: straight coalesced copy
            uint16_t* dstc = reinterpret_cast<uint16_t*>(cont + lo.off_cdf) + ((int64_t)nl * P.C + ct * CT) * kLp;
            for (int e = tid; e < ncols * kLp; e += CT) dstc[e] = cdfr[e];
        }
        // ---- pass 2: entropy-code the stream
        if (active && CODER == CODER_RANS) {
            // rANS: last token first; halfwords land at a descending pointer, so the row's tail is the stream in
            // decode order.  Row capacity (96 halfwords) cannot be exceeded (DESIGN.md 3.7): no clamp, no flag.
            uint32_t x = kRansLow;
            const uint16_t* const wend = reinterpret_cast<const uint16_t*>(trow) + 2 * P.tempw;     // the row's end
            int32_t nk = 0;                                                // minus the number of halfwords pushed
            const char* const cb = reinterpret_cast<const char*>(crow);
            // symbol s -> byte offset 2 s of its CDF entry: ((word >> 5 k) & 31) * 2 as one shift + one mask
            auto code = [&](uint32_t word, int k) {
                const uint32_t o = (k == 0 ? word << 1 : word >> (5 * k - 1)) & 62u;     // s <= 30: entry s + 1 is real
                const uint32_t c_lo = *reinterpret_cast<const uint16_t*>(cb + o);
                const uint32_t c_hi = *reinterpret_cast<const uint16_t*>(cb + o + 2);
                rans_put(x, nk, wend, c_lo, c_hi - c_lo);
            };
            int w = (gt - 1) / SPW;
            {
                const uint32_t word = myrow[w];
                for (int k = gt - 1 - w * SPW; k >= 0; --k) code(word, k);
            }
            for (--w; w >= 0; --w) {
                const uint32_t word = myrow[w];
#pragma unroll
                for (int k = SPW - 1; k >= 0; --k) code(word, k);
            }
            if (P.compact) reinterpret_cast<uint2*>(P.rstate)[((int64_t)tile_of() * CT + tid) * 2 + 1] = make_uint2(x, hlen);
            else P.rstate[(int64_t)tile_of() * CT + tid] = x;
            len = hlen + 4u - 2u * (uint32_t)nk;
        } else if (active) {
            EncState2 st;
            st.init();
            int tk = 0;
            for (int w = 0; tk < gt; ++w) {
                const uint32_t word = myrow[w];
                if (tk + SPW <= gt) {
#pragma unroll
                    for (int k = 0; k < SPW; ++k) {
                        const uint32_t sidx = (word >> (5 * k)) & 31u;       // <= 30: crow[sidx + 1] is a real entry
                        const uint32_t c_lo = crow[sidx];
                        enc_symbol2(st, c_lo, (uint32_t)crow[sidx + 1u] - c_lo, trow, cap);
                    }
                    tk += SPW;
                } else {
                    for (int k = 0; tk < gt; ++k, ++tk) {
                        const uint32_t sidx = (word >> (5 * k)) & 31u;
                        const uint32_t c_lo = crow[sidx];
                        enc_symbol2(st, c_lo, (uint32_t)crow[sidx + 1u] - c_lo, trow, cap);
                    }
                }
            }
            len = enc_finish2(st, trow, cap);
            if (st.w > cap) atomicOr(&P.err[j], 1u);   // size bound violated (cannot happen; stores were clamped)
        }
    } else {
        // CDF of the whole chunk was written by cdf_kernel: load it and build the (c_lo | width << 16) rows
        uint32_t* prow = tab + tid * PAIRW;
        const uint16_t* cdf_src =
            reinterpret_cast<const uint16_t*>(cont + lo.off_cdf) + ((int64_t)nl * P.C + ct * CT) * kLp;
        for (int e = tid; e < ncols * kLp; e += CT) tab[e] = cdf_src[e];
        __syncthreads();   // also: fac ready
        if (active) {
            uint32_t cv[kLp];
#pragma unroll
            for (int i = 0; i < kLp; ++i) cv[i] = prow[i] & 0xffffu;
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                const uint32_t hi = (i == 31) ? 0x10000u : cv[i + 1];
                prow[i] = cv[i] | ((hi - cv[i]) << 16);
            }
            if (CODER == CODER_RANS) {
                // at most one halfword per symbol: the 264-halfword row cannot overflow
                uint32_t x = kRansLow;
                const uint16_t* const wend = reinterpret_cast<const uint16_t*>(trow) + 2 * TEMPW_SPLIT;
                int32_t nk = 0;
                for_each_symbol_rev<DT, PAGED, 4>(cbase, P.slot_map, tokabs, s1, gt, fac, maxq, [&](uint32_t q) {
                    const uint32_t pr = prow[q];
                    rans_put(x, nk, wend, pr & 0xffffu, pr >> 16);
                });
                P.rstate[(int64_t)tile_of() * CT + tid] = x;
                len = 4u - 2u * (uint32_t)nk;
            } else {
                EncState2 st;
                st.init();
                for_each_symbol<DT, PAGED, 4>(cbase, P.slot_map, tokabs, s1, gt, fac, maxq, [&](uint32_t q) {
                    const uint32_t pr = prow[q];
                    enc_symbol2(st, pr & 0xffffu, pr >> 16, trow, cap);
                });
                len = enc_finish2(st, trow, cap);
                if (st.w > cap) atomicOr(&P.err[j], 1u);
            }
        }
    }

    // ---- stream lengths to the container, tile total for the compaction scan
    if (active) store_len(cont + lo.off_lengths, ((int64_t)id.g * NL + nl) * P.C + c, len, P.compact != 0);
    uint32_t tile_total;
    (void)block_excl_scan(len, s_warp, &tile_total);
    if (tid == 0) P.tile_tot[(int64_t)j * P.tiles_full + id.tile_in_chunk] = tile_total;
}

// FUSED: persistent, occupancy x SM count CTAs claiming tickets (see above); !FUSED: one tile per CTA
template <bool FUSED, int DT, bool PAGED, int CODER>
__global__ void __launch_bounds__(CT, FUSED ? 7 : 4) encode_kernel(EncParams P) {
    // 128-byte aligned base (also in cdf_kernel and decode_kernel): the shared-memory layout the kernels were measured with
    extern __shared__ __align__(128) uint32_t smem[];
    __shared__ uint32_t s_warp[CT / 32];
    if constexpr (!FUSED) {
        encode_tile<false, DT, PAGED, CODER>(P, [] { return (uint32_t)blockIdx.x; }, smem, s_warp);
    } else {
        // thread 0 claims the ticket and names the work in s_work: a tile, an absmax item (kWorkAbsmax | unit *
        // kAbsItems + item), a ticket without work, or the end.  Nothing of the schedule stays live in registers across
        // an item, and the tile body reads its index back from s_work where it needs it late, so it keeps the registers
        // it had as a kernel of its own.
        constexpr uint32_t kWorkDone = 0xffffffffu, kWorkNone = 0xfffffffeu, kWorkAbsmax = 0x80000000u;
        __shared__ uint32_t s_work;
        for (;;) {
            __syncthreads();   // the previous item is done with shared memory and s_work
            if (threadIdx.x == 0) {
                const uint32_t units = (uint32_t)P.n_chunks * (uint32_t)(P.ppl * P.nlay);
                const uint32_t step = (uint32_t)(kAbsItems + P.tpp);
                const uint32_t k = atomicAdd(P.ticket, 1u);
                const uint32_t s = k / step, r = k - s * step;
                uint32_t w = kWorkNone;
                if (s >= units + kAbsLead) w = kWorkDone;
                else if (r < (uint32_t)kAbsItems) { if (s < units) w = kWorkAbsmax | (s * kAbsItems + r); }
                else if (s >= (uint32_t)kAbsLead) w = (s - kAbsLead) * (uint32_t)P.tpp + (r - kAbsItems);
                s_work = w;
            }
            __syncthreads();
            const uint32_t w = s_work;
            if (w == kWorkDone) break;
            if (w == kWorkNone) continue;
            if (w & kWorkAbsmax) {
                const uint32_t a = w & ~kWorkAbsmax;
                absmax_item<PAGED>(P, (int)(a / kAbsItems), (int)(a % kAbsItems));
            } else {
                encode_tile<true, DT, PAGED, CODER>(P, [] { return *static_cast<volatile uint32_t*>(&s_work); }, smem, s_warp);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------ cdf (chunks > 256 tokens)
template <int DT, bool PAGED>
__global__ void __launch_bounds__(CT) cdf_kernel(EncParams P) {
    extern __shared__ __align__(128) uint32_t smem[];
    uint32_t* cnts = smem;                                        // CT * PAIRW counters
    float* fac = reinterpret_cast<float*>(cnts + CT * PAIRW);     // kGroup
    const int tid = threadIdx.x;
    const int NL = P.ppl * P.L;
    const uint32_t per_chunk = (uint32_t)NL * P.tpp;
    const uint32_t j = blockIdx.x / per_chunk;
    const uint32_t rem = blockIdx.x - j * per_chunk;
    const int nl = (int)(rem / P.tpp);
    const int ct = (int)(rem - (uint32_t)nl * P.tpp);
    const int t = chunk_tokens_of(P, (int)j);
    const int c = ct * CT + tid;
    const bool active = c < P.C;
    const int ncols = min(CT, P.C - ct * CT);
    uint8_t* cont = P.out + (int64_t)j * P.out_stride;
    const Layout lo = layout_of(P, t);
    const uint16_t* maxes = reinterpret_cast<const uint16_t*>(cont + lo.off_maxes) + (int64_t)nl * t;
    const float maxq = P.pt.maxq[nl];
    uint32_t* prow = cnts + tid * PAIRW;
#pragma unroll
    for (int i = 0; i < PAIRW; ++i) prow[i] = 0u;
    const int h = active ? c / P.D : 0;
    const int64_t tokabs = P.tok_begin + (int64_t)j * P.chunk_tokens;
    const uint16_t* cbase = P.pt.p[nl] + (int64_t)h * P.sH + (active ? c - h * P.D : 0);
    for (int tok0 = 0; tok0 < t; tok0 += kGroup) {
        const int gt = min(kGroup, t - tok0);
        __syncthreads();
        for (int i = tid; i < gt; i += CT) fac[i] = quant_factor(maxq, half_to_float(maxes[tok0 + i], DT));
        __syncthreads();
        if (active)
            for_each_symbol<DT, PAGED, 12>(cbase, P.slot_map, tokabs + tok0, P.sT, gt, fac, maxq,
                                           [&](uint32_t q) { prow[q] += 1u; });
    }
    if (active) {   // counts -> CDF values, written back over the counter row
        uint32_t cnt[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) cnt[i] = prow[i];
        CdfAccum acc;
        acc.init(t);
#pragma unroll
        for (uint32_t i = 0; i < 32u; ++i) prow[i] = acc.next(i, cnt[i]);
        prow[32] = acc.next(32u, 0u);
    }
    __syncthreads();
    uint16_t* dstc = reinterpret_cast<uint16_t*>(cont + lo.off_cdf) + ((int64_t)nl * P.C + ct * CT) * kLp;
    for (int e = tid; e < ncols * kLp; e += CT) dstc[e] = (uint16_t)cnts[e];   // rows are PAIRW == kLp words: e maps 1:1
}

// ------------------------------------------------------------------------------------------ compaction
// exclusive prefix over a chunk's tile totals (in place) + the chunk's payload size; one CTA per chunk
__global__ void __launch_bounds__(1024) enc_scan_kernel(EncParams P) {
    __shared__ unsigned long long s_w[32];
    __shared__ unsigned long long s_carry;
    const int j = blockIdx.x;
    const int t = chunk_tokens_of(P, j);
    const int ntiles = ((t + kGroup - 1) / kGroup) * P.ppl * P.nlay * P.tpp;
    uint32_t* tb = P.tile_tot + (int64_t)j * P.tiles_full;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0ull;
    __syncthreads();
    for (int base = 0; base < ntiles; base += 1024) {
        const int i = base + threadIdx.x;
        const unsigned long long v = i < ntiles ? tb[i] : 0ull;
        unsigned long long inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            unsigned long long n = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += n;
        }
        if (lane == 31) s_w[wid] = inc;
        __syncthreads();
        unsigned long long wbase = 0ull, tot = 0ull;
        for (int w = 0; w < 32; ++w) {
            const unsigned long long s = s_w[w];
            if (w < wid) wbase += s;
            tot += s;
        }
        const unsigned long long carry = s_carry;
        const unsigned long long excl = carry + wbase + inc - v;
        if (i < ntiles) {
            if (excl + v >= (1ull << 32)) atomicOr(&P.err[j], 8u);     // payload offsets are 32-bit per chunk
            tb[i] = (uint32_t)excl;
        }
        __syncthreads();
        if (threadIdx.x == 0) s_carry = carry + tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) P.totals[j] = s_carry;
}

// one stream: temp row (MSB-first native words, 16-byte aligned) -> len bytes at d.  16-byte loads, all of a row's loads
// (ten at a time for the long split-mode rows) in flight before the first use -- a word-at-a-time loop left one load in
// flight per thread and the kernel waiting on L2/DRAM latency.
__device__ __forceinline__ void copy_row(uint8_t* d, const uint32_t* srcw, uint32_t len, bool short_row) {
    auto put_word = [&](uint32_t w, uint32_t v) {
        const uint32_t nb = min(4u, len - 4u * w);
#pragma unroll
        for (uint32_t b = 0; b < 4u; ++b)
            if (b < nb) d[4u * w + b] = (uint8_t)(v >> (24u - 8u * b));
    };
    auto put_vec = [&](uint32_t qq, const uint4& v) {
        put_word(4u * qq, v.x);
        if (16u * qq + 4u < len) put_word(4u * qq + 1u, v.y);
        if (16u * qq + 8u < len) put_word(4u * qq + 2u, v.z);
        if (16u * qq + 12u < len) put_word(4u * qq + 3u, v.w);
    };
    constexpr int NV = TEMPW_FUSED / 4;
    static_assert(TEMPW_SPLIT % 4 == 0 && TEMPW_FUSED % 4 == 0, "temp rows must be 16-byte multiples");
    if (short_row) {                                       // fused mode: the whole row is <= NV vectors
        uint4 v[NV];
#pragma unroll
        for (int q = 0; q < NV; ++q)
            if (16u * q < len) v[q] = __ldg(reinterpret_cast<const uint4*>(srcw) + q);
#pragma unroll
        for (int q = 0; q < NV; ++q)
            if (16u * q < len) put_vec((uint32_t)q, v[q]);
    } else {                                               // split mode: rows up to 33 vectors, four in flight
        constexpr int NL = 4;
        for (uint32_t q0 = 0; 16u * q0 < len; q0 += NL) {
            uint4 v[NL];
#pragma unroll
            for (int q = 0; q < NL; ++q)
                if (16u * (q0 + q) < len) v[q] = __ldg(reinterpret_cast<const uint4*>(srcw) + q0 + q);
#pragma unroll
            for (int q = 0; q < NL; ++q)
                if (16u * (q0 + q) < len) put_vec(q0 + q, v[q]);
        }
    }
}

// rANS stream: the 32-bit final state (little-endian), then the tail of the temp row -- `nb` bytes of halfwords that the
// coder stored at descending addresses, already in decode order.  d is 2-byte aligned (every stream length is even).
// 16-byte loads, four in flight; typical streams (a few dozen bytes) take one round.
__device__ __forceinline__ void copy_row_rans(uint8_t* d, const uint32_t* row, uint32_t rowbytes, uint32_t nb, uint32_t state) {
    uint16_t* dh = reinterpret_cast<uint16_t*>(d);
    dh[0] = (uint16_t)state;
    dh[1] = (uint16_t)(state >> 16);
    const uint32_t h0 = (rowbytes - nb) >> 1;                  // first halfword of the stream inside the row
    const uint32_t hend = rowbytes >> 1;
    constexpr int NLV = 4;
    for (uint32_t q0 = h0 >> 3; 8u * q0 < hend; q0 += NLV) {
        uint4 v[NLV];
#pragma unroll
        for (int q = 0; q < NLV; ++q)
            if (8u * (q0 + q) < hend) v[q] = __ldg(reinterpret_cast<const uint4*>(row) + q0 + q);
#pragma unroll
        for (int q = 0; q < NLV; ++q) {
            if (8u * (q0 + q) < hend) {
                const uint32_t w[4] = {v[q].x, v[q].y, v[q].z, v[q].w};
#pragma unroll
                for (uint32_t i = 0; i < 8u; ++i) {
                    const uint32_t hw = 8u * (q0 + q) + i;
                    if (hw >= h0) dh[2u + hw - h0] = (uint16_t)(w[i >> 1] >> (16u * (i & 1u)));
                }
            }
        }
    }
}

// move each tile's streams from its temp rows to their final, contiguous place in the payload
// (collect_bytes, cachegen_encoder.py:225-238).  Each thread copies its own stream into a shared-memory image of the
// tile's byte range (placed at the destination's 16-byte phase), then the CTA writes that range with 16-byte vector
// stores: the payload is written as full sectors no matter how short the individual streams are.
__global__ void __launch_bounds__(CT, 12) compact_kernel(EncParams P) {
    extern __shared__ __align__(16) uint8_t stage[];      // 16 + CT * tempw * 4 bytes
    __shared__ uint32_t s_warp[CT / 32];
    const int tid = threadIdx.x;
    TileId id;
    if (!decode_tile(P, blockIdx.x, &id)) return;
    const int NL = P.ppl * P.L;
    const int c = id.ct * CT + tid;
    uint8_t* cont = P.out + (int64_t)id.j * P.out_stride;
    const Layout lo = layout_of(P, id.t);
    const bool rans = P.coder == CODER_RANS;
    const uint32_t rowbytes = (uint32_t)P.tempw * 4u;
    // no stream is longer than its temp row (+ the state, + header words 0 and 1, which live in the side array)
    const uint32_t len = c < P.C ? min(load_len(cont + lo.off_lengths, ((int64_t)id.g * NL + id.nl) * P.C + c, P.compact != 0),
                                       rowbytes + (rans ? 4u : 0u) + (P.compact ? 8u : 0u)) : 0u;
    uint32_t tile_total;
    const uint32_t my_off = block_excl_scan(len, s_warp, &tile_total);
    const uint64_t base = P.tile_tot[(int64_t)id.j * P.tiles_full + id.tile_in_chunk];
    uint8_t* dst;
    if (P.chunk_base) {                                  // arena: place_kernel gave the chunk room, or marked it failed
        const unsigned long long cb = P.chunk_base[id.j];
        if (cb == ~0ull) return;
        dst = P.arena + cb + base;
    } else {
        const int64_t room = P.out_stride - lo.off_payload;
        if ((int64_t)(base + tile_total) > room) {      // never write past the slot the caller gave us
            if (tid == 0) atomicOr(&P.err[id.j], 4u);
            return;
        }
        dst = cont + lo.off_payload + base;
    }
    const uint32_t phase = (uint32_t)(reinterpret_cast<uintptr_t>(dst) & 15u);
    // the image of the tile's byte range must fit the shared-memory stage the launch provided; a tile coded against a
    // foreign CDF may (rarely) exceed it, then every thread writes its own stream straight to the payload
    const bool staged = phase + tile_total <= (uint32_t)P.stage_bytes;
    if (len && rans) {
        const uint32_t* srcw = P.temp + ((int64_t)blockIdx.x * CT + tid) * P.tempw;
        uint32_t state, hl = 0u;
        const uint32_t* tail = srcw;                               // the row's rANS part (halfwords right-aligned in it)
        uint32_t tailbytes = rowbytes;
        if (P.compact) {
            // version 3: header words 0, 1, the state and the header length come from the tile's side array (one coalesced
            // 16-byte load), header words 2..8 -- long headers only -- from the front of the row
            const uint4 rec = __ldg(reinterpret_cast<const uint4*>(P.rstate) + (int64_t)blockIdx.x * CT + tid);
            state = rec.z;
            hl = min(min(rec.w, (uint32_t)kHdrMax), max(len, 4u) - 4u);
            uint32_t hw[9] = {rec.x, rec.y, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
            if (hl > 8u) {
                const uint4 a = __ldg(reinterpret_cast<const uint4*>(srcw)), b = __ldg(reinterpret_cast<const uint4*>(srcw) + 1);
                hw[2] = a.x; hw[3] = a.y; hw[4] = a.z; hw[5] = a.w; hw[6] = b.x; hw[7] = b.y; hw[8] = b.z;
            }
            uint16_t* dh = reinterpret_cast<uint16_t*>(staged ? stage + phase + my_off : dst + my_off);
#pragma unroll
            for (uint32_t k = 0; k < kHdrMax / 2; ++k)
                if (2u * k < hl) dh[k] = (uint16_t)(hw[k >> 1] >> (16u * (k & 1u)));
            tail = srcw + kHdrRowWords;
            tailbytes = rowbytes - 4u * kHdrRowWords;
        } else {
            state = P.rstate[(int64_t)blockIdx.x * CT + tid];
        }
        if (staged) copy_row_rans(stage + phase + my_off + hl, tail, tailbytes, max(len, 4u + hl) - 4u - hl, state);
        else copy_row_rans(dst + my_off + hl, tail, tailbytes, max(len, 4u + hl) - 4u - hl, state);
    } else if (len) {
        const uint32_t* srcw = P.temp + ((int64_t)blockIdx.x * CT + tid) * P.tempw;
        // two instantiations, so that the staged one compiles to shared-memory stores and not to generic ones
        if (staged) {
            copy_row(stage + phase + my_off, srcw, len, P.tempw == TEMPW_FUSED);
        } else {                                             // rare: plain word loop, keeps the kernel's registers low
            uint8_t* d = dst + my_off;
            for (uint32_t w = 0; 4u * w < len; ++w) {
                const uint32_t v = __ldg(srcw + w);
                for (uint32_t b = 0; b < 4u && 4u * w + b < len; ++b) d[4u * w + b] = (uint8_t)(v >> (24u - 8u * b));
            }
        }
    }
    if (!staged) return;                                     // uniform per CTA
    __syncthreads();
    // [phase, phase + tile_total) of `stage` -> dst - phase + same offsets; vector body, byte head / tail
    const uint32_t lo_b = phase, hi_b = phase + tile_total;
    const uint32_t body0 = min(hi_b, (lo_b + 15u) & ~15u), body1 = max(body0, hi_b & ~15u);
    uint8_t* dbase = dst - phase;
    for (uint32_t i = lo_b + tid; i < body0; i += CT) dbase[i] = stage[i];
    for (uint32_t i = body0 + 16u * tid; i < body1; i += 16u * CT)
        *reinterpret_cast<uint4*>(dbase + i) = *reinterpret_cast<const uint4*>(stage + i);
    for (uint32_t i = body1 + tid; i < hi_b; i += CT) dbase[i] = stage[i];
}

// ------------------------------------------------------------------------------------------ arena placement
// b200kv_encode_layers: after enc_scan_kernel, give each chunk's bytes of this call (its K planes, then its V planes)
// room in the arena by the arena rule (arena_place, common.cuh), then one (offset, bytes) row per plane.  One CTA: a few
// hundred chunks at most, and it runs once per call.
__global__ void __launch_bounds__(1024) place_kernel(EncParams P) {
    const int tid = threadIdx.x;
    arena_place(P.n_chunks, P.totals, P.layers_left, P.nlay, P.arena_bytes, P.cursor, P.fail_from, P.chunk_base, P.err);
    for (int i = tid; i < P.n_chunks; i += 1024)
        if (P.chunk_base[i] != ~0ull) P.ptotal[i] += P.totals[i];
    const int NLc = P.ppl * P.nlay;
    for (int k = tid; k < P.n_chunks * NLc; k += 1024) {
        const int j = k / NLc, pl = k - j * NLc;
        const uint32_t* tb = P.tile_tot + (int64_t)j * P.tiles_full;
        const unsigned long long off = tb[pl * P.tpp];
        const unsigned long long end = pl + 1 < NLc ? (unsigned long long)tb[(pl + 1) * P.tpp] : P.totals[j];
        const unsigned long long cb = P.chunk_base[j];       // written above by this CTA
        int64_t* row = P.seg + ((int64_t)j * P.ppl * P.L + launch_plane(P, pl)) * 2;
        row[0] = cb == ~0ull ? -1 : (int64_t)(cb + off);
        row[1] = (int64_t)(end - off);
    }
}

__global__ void encl_init_kernel(EncParams P) {
    *P.cursor = 0ull;
    *P.fail_from = (unsigned)P.n_chunks;
}

// ------------------------------------------------------------------------------------------ finalize
__global__ void finalize_kernel(EncParams P) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= P.n_chunks) return;
    const int t = chunk_tokens_of(P, j);
    const Layout lo = layout_of(P, t);
    b200kv_header* hd = reinterpret_cast<b200kv_header*>(P.out + (int64_t)j * P.out_stride);
    hd->magic = B200KV_MAGIC;
    // 1: arithmetic coder, 2: rANS, 3: rANS + compact sections, 4: version 3 with one plane per layer (latent KV)
    hd->version = P.compact ? (P.ppl == 1 ? 4u : 3u) : (uint32_t)P.coder + 1u;
    hd->L = P.L; hd->H = P.H; hd->D = P.D;
    hd->ntokens = t;
    hd->ngroups = lo.ngroups;
    hd->max_dtype = P.dtype;
    hd->payload_bytes = P.totals[j];
    hd->total_bytes = (uint64_t)lo.off_payload + P.totals[j];
    hd->status = P.err[j];
    hd->reserved[0] = hd->reserved[1] = hd->reserved[2] = 0u;
    if (P.sizes_out) P.sizes_out[j] = hd->status ? 0ull : hd->total_bytes;     // 0 = this chunk failed (see header.status)
    {
        // the padding in front of the maxima, the lengths and the payload (< 16 bytes each) is zero, not whatever the
        // output buffer held before: a container's bytes are a function of the KV alone, and no stale device memory
        // travels with it to a tier
        uint8_t* c = reinterpret_cast<uint8_t*>(hd);
        const int64_t NL = (int64_t)P.ppl * P.L;
        const int64_t ends[3] = {lo.off_cdf + (P.compact ? NL : NL * P.C * kLp * 2), lo.off_maxes + NL * t * 2,
                                 lo.off_lengths + (int64_t)lo.ngroups * NL * P.C * (P.compact ? 1 : 4)};
        const int64_t starts[3] = {lo.off_maxes, lo.off_lengths, lo.off_payload};
        for (int k = 0; k < 3; ++k)
            for (int64_t b = ends[k]; b < starts[k]; ++b) c[b] = 0u;
    }
    if (P.compact) {                               // counts per stream of every plane: makes the container self-describing
        uint8_t* nbmap = reinterpret_cast<uint8_t*>(hd) + lo.off_cdf;
        const int NL = P.ppl * P.L;
        for (int nl = 0; nl < (int)align16(NL); ++nl) nbmap[nl] = nl < NL ? (uint8_t)(2 * ((int)P.pt.maxq[nl] + 1)) : (uint8_t)0;
    }
}

// ------------------------------------------------------------------------------------------ decode
struct DecChunk {
    const uint8_t* base;
    int64_t dst_tok;
    int32_t t, ngroups;
    uint32_t payload_bytes;      // from the (host-validated) header: stream offsets are clamped to it
    // head window (b200kv_decode_plan_heads; the whole container otherwise): container channels [cw0, cw1) are decoded
    // into destination channel c + dshift; they lie in tiles [ct0, ct0 + ntw) of every plane
    int32_t ct0, ntw, cw0, cw1, dshift;
};

// The decode's parameter block lives in the caller's b200kv_decode_plan_t (256 words), so it carries the destination's
// plane table inline only up to kInlinePlanes planes (L <= 64).  A deeper model's full table goes to the plan's
// workspace and the kernel reads it from there (decode_kernel<..., GT = true>): one uniform load per CTA, per plane.
constexpr int kInlinePlanes = 128;
struct DecParams {
    PlaneTableT<kInlinePlanes> pt;   // destination planes; maxq = C_l = bins // 2 - 1 (2L <= kInlinePlanes)
    const PlaneTable* gpt;           // device copy of the whole table when 2L > kInlinePlanes; NULL otherwise
    int64_t sT, sH;
    const int64_t* slot_map;     // paged destination: token i lives in row slot_map[i]; NULL = row i
    int32_t L, H, D, C, out_dtype, max_dtype, n_chunks, tpp, tiles_max;   // H, C: the containers' (src_H with windows)
    int32_t compact;             // containers are version 3 (or 4)
    int32_t ppl;                 // planes per layer: 2 (K, V) or 1 (latent KV, version 4)
    int32_t version;             // the header version the coder (and the destination's planes) name: status bit 2 if not
    int32_t lb, nlay;            // decode_kernel: this launch decodes layers [lb, lb + nlay), i.e. planes lb.. and L + lb..
    int32_t wtpp;                // decode_kernel: tiles launched per plane = the largest window's ntw (tpp without windows)
    const DecChunk* chunks;      // device
    unsigned long long* tile_base;   // [n_chunks][tiles_max]: tile sums, then exclusive prefix
    uint32_t* status;            // [n_chunks] or NULL: bit 0 = a rANS stream did not return to its initial state,
                                 //   bit 1 = stream offsets beyond the payload (corrupt lengths section)
};
static_assert(sizeof(DecParams) < kMaxParamBytes, "DecParams must stay under 4 KB of kernel parameters");

// plane nl's destination pointer and quantiser constant: inline (GT = false) or from the device copy (GT = true)
template <bool GT>
__device__ __forceinline__ const uint16_t* dec_plane(const DecParams& P, int nl) {
    if constexpr (GT) return P.gpt->p[nl];
    else return P.pt.p[nl];
}
template <bool GT>
__device__ __forceinline__ float dec_maxq(const DecParams& P, int nl) {
    if constexpr (GT) return P.gpt->maxq[nl];
    else return P.pt.maxq[nl];
}

// tile sums of the stream lengths: one warp per tile
__global__ void __launch_bounds__(128) tile_sum_kernel(DecParams P) {
    const int j = blockIdx.y;
    const int tile = blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const DecChunk dc = P.chunks[j];
    // the header is part of the fixed sections: a container of another version than the call's coder (e.g. version 3
    // handed to a latent destination) is flagged, so the caller drops the chunk as a miss
    if (blockIdx.x == 0 && threadIdx.x == 0 && P.status != nullptr &&
        reinterpret_cast<const uint32_t*>(dc.base)[1] != (uint32_t)P.version)
        atomicOr(&P.status[j], 4u);
    const int NL = P.ppl * P.L;
    const int ntiles = dc.ngroups * NL * P.tpp;
    if (tile >= ntiles) return;
    const int plane_row = tile / P.tpp;          // g * NL + nl
    const int ct = tile - plane_row * P.tpp;
    const Layout lo = layout_of(P, dc.t);
    const int c0 = ct * CT, c1 = min(P.C, c0 + CT);
    uint32_t s = 0;
    for (int c = c0 + lane; c < c1; c += 32) s += load_len(dc.base + lo.off_lengths, (int64_t)plane_row * P.C + c, P.compact != 0);
    s = __reduce_add_sync(0xffffffffu, s);
    if (lane == 0) P.tile_base[(int64_t)j * P.tiles_max + tile] = s;
}

// exclusive prefix over a chunk's tile sums (in place); one CTA per chunk
__global__ void __launch_bounds__(1024) tile_scan_kernel(DecParams P) {
    __shared__ unsigned long long s_w[32];
    __shared__ unsigned long long s_carry;
    const int j = blockIdx.x;
    const DecChunk dc = P.chunks[j];
    const int ntiles = dc.ngroups * P.ppl * P.L * P.tpp;
    unsigned long long* tb = P.tile_base + (int64_t)j * P.tiles_max;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0ull;
    __syncthreads();
    for (int base = 0; base < ntiles; base += 1024) {
        const int i = base + threadIdx.x;
        const unsigned long long v = i < ntiles ? tb[i] : 0ull;
        unsigned long long inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            unsigned long long n = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += n;
        }
        if (lane == 31) s_w[wid] = inc;
        __syncthreads();
        unsigned long long wbase = 0ull, tot = 0ull;
        for (int w = 0; w < 32; ++w) {
            const unsigned long long s = s_w[w];
            if (w < wid) wbase += s;
            tot += s;
        }
        const unsigned long long carry = s_carry;
        if (i < ntiles) tb[i] = carry + wbase + inc - v;
        __syncthreads();
        if (threadIdx.x == 0) s_carry = carry + tot;
        __syncthreads();
    }
}

// Plane boundaries of version-3 / version-4 containers in device memory (b200kv_plane_offsets_device): one CTA of 32
// warps per container, one warp per plane at a time, 16-byte loads (the sum is a handful of independent loads per lane,
// not a chain of byte loads: it runs on the store worker's copy stream, in front of the wave's device->host copies).  out
// row j: [off_payload, end of plane 0, ..., end of plane P-1 = total_bytes] (P = 2L, or L for version 4), or -1 in entry 0
// when the container is neither or its half-lengths do not add up to total_bytes.
__global__ void __launch_bounds__(1024) plane_offsets_kernel(const uint8_t* base, int64_t stride, int64_t* out) {
    __shared__ uint32_t s_sum[B200KV_MAX_PLANES];
    const uint8_t* c = base + (int64_t)blockIdx.x * stride;
    int64_t* o = out + (int64_t)blockIdx.x * (B200KV_MAX_PLANES + 1);
    const uint32_t* hw = reinterpret_cast<const uint32_t*>(c);
    const uint32_t version = hw[1], L = hw[2], H = hw[3], D = hw[4], t = hw[5];
    const uint64_t total = *reinterpret_cast<const uint64_t*>(c + 40);
    // the header alone decides whether the fixed sections lie inside the container and inside this row: nothing past the
    // header is read before that is known (the lengths section alone is 2L * C bytes, so C <= stride bounds the layout)
    const uint64_t C64 = (uint64_t)H * D;
    if (hw[0] != B200KV_MAGIC || (version != 3u && version != 4u) || L == 0u || 2u * L > (uint32_t)B200KV_MAX_PLANES ||
        H == 0u || D == 0u || t == 0u || t > (uint32_t)kGroup || C64 > (uint64_t)stride || C64 >= (1ull << 31)) {
        if (threadIdx.x == 0) o[0] = -1;
        return;
    }
    const int ppl = version == 4u ? 1 : 2;
    const int NL = ppl * (int)L;
    const int64_t C = (int64_t)C64;
    const Layout lo = make_layout((int)L, (int)C, (int)t, 1, ppl);
    if ((uint64_t)lo.off_payload > total || lo.off_payload > stride) {
        if (threadIdx.x == 0) o[0] = -1;
        return;
    }
    const uint8_t* half = c + lo.off_lengths;                  // 16-byte aligned (container and section)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int p = NL + 1 + (int)threadIdx.x; p <= B200KV_MAX_PLANES; p += blockDim.x) o[p] = 0;   // the row past P + 1
    for (int p = warp; p < NL; p += blockDim.x >> 5) {
        const uint8_t* row = half + p * C;
        uint32_t sum = 0;
        if ((C & 15) == 0) {
            const uint4* v = reinterpret_cast<const uint4*>(row);
#pragma unroll 4
            for (int64_t i = lane; i < C / 16; i += 32) {
                const uint4 q = v[i];
                sum = __dp4a(q.x, 0x01010101u, sum);
                sum = __dp4a(q.y, 0x01010101u, sum);
                sum = __dp4a(q.z, 0x01010101u, sum);
                sum = __dp4a(q.w, 0x01010101u, sum);
            }
        } else {
            for (int64_t i = lane; i < C; i += 32) sum += row[i];
        }
        sum = __reduce_add_sync(0xffffffffu, sum);
        if (lane == 0) s_sum[p] = sum;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t off = lo.off_payload;
        o[0] = off;
        for (int p = 0; p < NL; ++p) {
            off += 2 * (int64_t)s_sum[p];
            o[p + 1] = off;
        }
        if (off != (int64_t)total) o[0] = -1;
    }
}

// Aligned big-endian word reader over the stream's bytes in global memory with a one-word look-ahead: the
// load for word i+1 is issued when word i is consumed, so its L2/L1 latency overlaps ~8+ symbols of decoding.
// Each lane walks its own stream; a 32-byte sector serves 8 consecutive refills from L1.
struct WordSrc {
    const uint32_t* base;   // the container, as words
    uint32_t idx;        // next word to load: a 32-bit index keeps the refill to one IMAD.WIDE + one add
    uint32_t ahead;
    __device__ __forceinline__ void prime() { ahead = __ldg(base + idx); ++idx; }
    __device__ __forceinline__ uint32_t next_be() {
        const uint32_t w = ahead;
        ahead = __ldg(base + idx);
        ++idx;
        return __byte_perm(w, 0u, 0x0123);
    }
};
// Both readers may run past the end of their stream (a decoder consumes at most 18 bits (arithmetic coder) / one
// halfword (rANS) per symbol, whatever the bytes say): at most B200KV_READ_SLACK bytes past the stream's start, which
// b200kv_decode_chunks checks against the size of the caller's buffer.  A corrupt lengths section therefore cannot make
// a kernel read outside that buffer: stream starts are clamped to the payload, reads are bounded from there.
//
// Bytes read past the end of a stream never reach an output or a status bit (version 2 / 3 streams, rANS), so the
// bytes of the next plane need not have arrived when a plane is decoded (a layer-major upload, b200kv_decode_layers):
//   - rANS loop (rans_decode_stream): the init loads 3 words and every window move one more, but a halfword enters the
//     state only through the PRMT of a renormalisation, and the decoder renormalises exactly where the encoder pushed
//     (same state sequence), i.e. it consumes exactly the stream's halfwords.  Look-ahead words are loaded, never used.
//   - v3 header, byte reader (all_short): the load at cb + popc(mask below i) happens for every symbol the warp uses,
//     but the value is kept only for a set, non-last bit of the lane's own mask: an index < the number of stored
//     counts, inside the header.  The mask itself is cut to hdr_mask_bytes(nb) bytes.
//   - v3 header, register reader: words are loaded while 4k < header length; next_byte() hands out the count bytes
//     only, all of them inside the header (the funnel shift may carry later bytes in the same register, unread).
//   - status: bit 1 comes from the lengths section (fixed sections) and payload_bytes, bit 0 from the final state.
//   - arithmetic coder (version 1): the decoder does shift bits past the end of its stream into `off`, but none of them
//     can change a symbol: termination emits the final bit and its pending run, which leave every continuation of the
//     stream inside the final interval, so every decision `plo <= off < phi` holds whatever follows (tests/ac_edges.py,
//     tests/test_gpu_ac_edges.py decode with 0x00 / 0xFF after the planes).  Status comes from the lengths section only.
// The layer-major upload of lmcache_b200/pipeline.py splits version-3 containers only.

// rANS: aligned little-endian words off a running pointer; the look-ahead lives in the decoder state (RansDec::nxt)
struct LeWordSrc {
    const uint32_t* p;
    __device__ __forceinline__ uint32_t next_le() { return __ldg(p++); }
};

__device__ __forceinline__ uint16_t out_half(float v, int dt) {
    // hardware RNE converts (NaN payloads are canonicalised; every finite / inf value matches torch's cast)
    return dt ? __half_as_ushort(__float2half_rn(v)) : __bfloat16_as_ushort(__float2bfloat16_rn(v));
}
// typed store of the converted value (the 16-bit result goes straight from F2FP to STG.U16)
template <int OUT_DT>
__device__ __forceinline__ void store_half(uint16_t* p, float v) {
    if constexpr (OUT_DT) *reinterpret_cast<__half*>(p) = __float2half_rn(v);
    else *reinterpret_cast<__nv_bfloat16*>(p) = __float2bfloat16_rn(v);
}

// value = lut * row_max (one rounded multiply, cachegen_decoder.py:31-35), converted RNE and stored as 16 bits
// (F2FP + STG.U16, no register merge in between)
template <int OUT_DT>
__device__ __forceinline__ void store_dequant(uint16_t* base, uint32_t off, float lutv, float row_max, uint32_t two) {
    const float v = __fmul_rn(lutv, row_max);
    // address = base + 2 * off as ONE IMAD.WIDE (`two` = 2, opaque to ptxas, keeps it off the ALU pipe); the converted value stays in the low half of a 32-bit register
    // (F2FP.PACK_AB with a zero upper half) and STG.U16 stores that half: no 16-bit register shuffling
    if constexpr (OUT_DT)
        asm volatile("{\n\t.reg .b64 ad;\n\t.reg .b32 r;\n\t.reg .b16 lo, hi;\n\t"
                     "mad.wide.u32 ad, %1, %3, %0;\n\t"
                     "cvt.rn.f16x2.f32 r, 0f00000000, %2;\n\t"
                     "mov.b32 {lo, hi}, r;\n\t"
                     "st.global.b16 [ad], lo;\n\t}" ::"l"(base), "r"(off), "f"(v), "r"(two) : "memory");
    else
        asm volatile("{\n\t.reg .b64 ad;\n\t.reg .b32 r;\n\t.reg .b16 lo, hi;\n\t"
                     "mad.wide.u32 ad, %1, %3, %0;\n\t"
                     "cvt.rn.bf16x2.f32 r, 0f00000000, %2;\n\t"
                     "mov.b32 {lo, hi}, r;\n\t"
                     "st.global.b16 [ad], lo;\n\t}" ::"l"(base), "r"(off), "f"(v), "r"(two) : "memory");
}

// per-thread decode loop: one stream, gt symbols, straight to the destination layout.
// PAGED: dst is the stream's channel in row 0 of the plane and `slots` points at the group's first slot-map entry.
template <int OUT_DT, int NSTEPS, bool PAGED>
__device__ __forceinline__ void decode_stream(const uint8_t* cont, uint32_t my_off, const uint32_t* erow,
                                              const float* lut, const float* mx, uint16_t* dst, uint32_t sT, int gt,
                                              const int64_t* slots) {
    const uint32_t skip = my_off & 3u;            // containers are 16-byte aligned
    WordSrc src{reinterpret_cast<const uint32_t*>(cont), my_off >> 2, 0u};
    src.prime();
    DecState2 st;
    dec_init2(st, src, skip);
    uint16_t* d = dst;                                      // running pointer: one 64-bit add per token
    // dec_symbol2 returns 4 * symbol = the byte offset into the fp32 LUT
    auto lut_at = [&](uint32_t s4) { return *reinterpret_cast<const float*>(reinterpret_cast<const char*>(lut) + s4); };
    if constexpr (PAGED) {
        for (int i = 0; i < gt - 1; ++i)
            store_half<OUT_DT>(dst + __ldg(slots + i) * (int64_t)sT,
                               dequant_value(lut_at(dec_symbol2<NSTEPS>(st, src, erow, false)), mx[i]));
        store_half<OUT_DT>(dst + __ldg(slots + gt - 1) * (int64_t)sT,
                           dequant_value(lut_at(dec_symbol2<NSTEPS>(st, src, erow, true)), mx[gt - 1]));
    } else {
        for (int i = 0; i < gt - 1; ++i, d += sT)
            store_half<OUT_DT>(d, dequant_value(lut_at(dec_symbol2<NSTEPS>(st, src, erow, false)), mx[i]));
        store_half<OUT_DT>(d, dequant_value(lut_at(dec_symbol2<NSTEPS>(st, src, erow, true)), mx[gt - 1]));
    }
}

// one lower-bound step through a stream's table whose entries are PITCH bytes apart: a += ROWS entries iff the entry ROWS
// further is <= key.  The add is an IMAD with an opaque multiplier (FMA pipe; see rans_decode_stream).
template <uint32_t ROWS, uint32_t PITCH>
__device__ __forceinline__ void rans_search_step(uint32_t& a, uint32_t key, uint32_t one) {
    uint32_t ev;
    asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(ev) : "r"(a), "n"(ROWS * PITCH));
    asm("{\n\t.reg .pred p;\n\tsetp.le.u32 p, %1, %2;\n\t@p mad.lo.u32 %0, %3, %4, %0;\n\t}"
        : "+r"(a) : "r"(ev), "r"(key), "r"(one), "n"(ROWS * PITCH));
}

// rANS decode loop (container version 2): one stream, gt symbols, straight to the destination layout.
// Per symbol: key = (x << 16) | 0xffff; lower-bound search over the stream's packed table pk[i] = (cdf[i] << 16) | freq(i)
// -- the two top levels sit in registers, the rest are LDS off a running shared-memory address --; the winning entry
// carries start and freq, so the state update is one multiply-add; at most one 16-bit renormalisation (a PRMT out of the
// two-word window, a predicated aligned load when the window moves on).  Returns the final state (2^16 when intact).
template <int OUT_DT, int NSTEPS, bool PAGED, bool TR>
__device__ __forceinline__ uint32_t rans_decode_stream(const uint8_t* cont, uint32_t my_off, const uint32_t* pk,
                                                       const float* lut, const float* mx, uint16_t* dst, uint32_t sT, int gt,
                                                       const int64_t* slots, uint32_t one) {
    // stream words are addressed as container base + 32-bit word index: the address of the next word is one IMAD.WIDE
    // (FMA pipe, not predicated), only the load and the index increment are predicated
    const uint32_t* const wbase = reinterpret_cast<const uint32_t*>(cont);
    uint32_t idx = my_off >> 2;
    struct Src {
        const uint32_t* b; uint32_t& i;
        __device__ __forceinline__ uint32_t next_le() { return __ldg(b + i++); }
    } src{wbase, idx};
    RansDec st;
    rans_dec_init(st, src, (my_off >> 1) & 1u);
    constexpr uint32_t H = 1u << (NSTEPS - 1);
    // `pk` points at this stream's entry 0.  Two table layouts (decode_kernel builds either):
    //   TR = false  rows of 33 words per stream (odd pitch: lanes that read the SAME entry never collide; lanes that read
    //               different entries sometimes do -- 2.7 extra wavefronts per warp-symbol at 0.6 bits/symbol, 7.4 at 4.1)
    //   TR = true   transposed, entry i of every stream in one 512-byte row: a lane never leaves its own bank.  A 16-symbol
    //               table (NSTEPS = 4) fills rows 0..15 only, and rows 16..31 hold the LUT replicated down the columns
    //               (row 16 + s = lut[s] in every column): the LUT value sits a constant 16 rows past the winning entry,
    //               so it costs no address arithmetic.  A 32-symbol table computes lut_a + 4 * symbol from the
    //               entry's address: two more instructions per symbol.
    // 16-symbol planes always take the transposed table with the LUT replica (decode_kernel); for 32-symbol planes the
    // host picks by the containers' measured bits per symbol (b200kv_decode_chunks).
    constexpr bool kRep = TR && NSTEPS == 4;
    constexpr uint32_t kPitch = TR ? CT * 4u : 4u;
    constexpr uint32_t kIdx = TR ? CT : 1u;
    const uint32_t a0 = (uint32_t)__cvta_generic_to_shared(pk);
    const uint32_t a0h = a0 + kPitch * H;
    const uint32_t r_mid = pk[kIdx * H], r_lo = pk[kIdx * (H / 2)], r_hi = pk[kIdx * (H + H / 2)];
    const uint32_t lut_a = (uint32_t)__cvta_generic_to_shared(lut);            // TR: lut[s] = lut_a + ((a - a0) >> 7)
    const uint32_t lut_rel = lut_a - a0;                                       // !TR: lut[s] = a + lut_rel
    uint32_t off = 0u;                                                         // element offset of the current token row
    // Two integer pipes share this loop's work: IMAD (FMA pipe) and ISETP / SEL / PRMT / LOP3 (ALU pipe), each one warp
    // instruction per 2 cycles.  Some additions are written as IMADs whose multiplier ptxas cannot fold (`one` is 1 but
    // comes from a kernel parameter), which pins them to the FMA pipe; the 16-bit shifts are PRMTs (ALU pipe) and the
    // warp-uniform token offset a plain add (uniform datapath).  That split measured fastest on the H100 (DESIGN.md 3.4):
    // with the shifts as IMADs too, the FMA pipe ran 66 of a 4-symbol trip's 151 instructions and bound the loop.
    const uint32_t mone = 0u - one, two = one + one, c25 = one << 25;
    auto step = [&](float row_max, int i) {
        uint32_t key, xh;
        asm("prmt.b32 %0, %1, %2, 0x1054;" : "=r"(key) : "r"(st.x), "r"(mone));         // (x << 16) | 0xffff
        asm("prmt.b32 %0, %1, 0, 0x4432;" : "=r"(xh) : "r"(st.x));                      // x >> 16
        const bool p1 = r_mid <= key;
        uint32_t a = p1 ? a0h : a0;
        const uint32_t m = p1 ? r_hi : r_lo;
        asm("{\n\t.reg .pred p;\n\tsetp.le.u32 p, %1, %2;\n\t@p mad.lo.u32 %0, %3, %4, %0;\n\t}"
            : "+r"(a) : "r"(m), "r"(key), "r"(one), "n"(kPitch * (H / 2)));
        if constexpr (H >= 16) rans_search_step<4, kPitch>(a, key, one);         // entries H/4 .. 1 further on
        rans_search_step<2, kPitch>(a, key, one);
        rans_search_step<1, kPitch>(a, key, one);
        uint32_t e, la;
        float lv;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(e) : "r"(a));
        if constexpr (kRep) {
            asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(lv) : "r"(a), "n"(16u * CT * 4u));   // the LUT replica
        } else {
            if constexpr (TR) asm("mad.hi.u32 %0, %1, %2, %3;" : "=r"(la) : "r"(a - a0), "r"(c25), "r"(lut_a));   // lut_a + 4 * symbol
            else la = a + lut_rel;
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(lv) : "r"(la));
        }
        // x = freq * (x >> 16) + slot - start
        uint32_t dl;
        asm("prmt.b32 %0, %1, 0, 0x4432;" : "=r"(dl) : "r"(key - e));                 // (key - e) >> 16
        st.x = (e & 0xffffu) * xh + dl;
        // renormalisation, branch-free (a warp takes this path on most symbols, so a branch would run for all lanes
        // anyway): p = x < 2^16 -> pull the next halfword out of the window; q = p and the window's upper half was
        // taken -> the window moves on (cur = nxt, nxt = next aligned word)
        const uint32_t* const wad = wbase + idx;
        asm volatile(
            "{\n\t.reg .pred p, q;\n\t"
            "setp.lt.u32 p, %0, 65536;\n\t"
            "setp.eq.and.u32 q, %3, 0x1076, p;\n\t"
            "@p prmt.b32 %0, %0, %1, %3;\n\t"
            "@p mad.lo.u32 %3, %3, %7, 0x20ca;\n\t"     // 0x1054 <-> 0x1076: sel = 0x20ca - sel
            "@q mov.b32 %1, %2;\n\t"
            "@q ld.global.nc.u32 %2, [%5];\n\t"
            "@q mad.lo.u32 %4, %6, %6, %4;\n\t"         // idx += 1
            "}"
            : "+r"(st.x), "+r"(st.cur), "+r"(st.nxt), "+r"(st.sel), "+r"(idx)
            : "l"(wad), "r"(one), "r"(mone));
        if constexpr (PAGED) {
            store_dequant<OUT_DT>(dst + __ldg(slots + i) * (int64_t)sT, 0u, lv, row_max, two);
        } else {
            store_dequant<OUT_DT>(dst, off, lv, row_max, two);
            off += sT;
        }
    };
    int i = 0;
#pragma unroll 1
    for (; i + 4 <= gt; i += 4) {                                               // 4 symbols per trip: the body is ~150
        const float4 m4 = *reinterpret_cast<const float4*>(mx + i);            // instructions, it must stay in the
        step(m4.x, i); step(m4.y, i + 1); step(m4.z, i + 2); step(m4.w, i + 3);   // instruction cache next to its twin
    }
#pragma unroll 1
    for (; i < gt; ++i) step(mx[i], i);
    return st.x;
}

// One tile = CT streams of one (chunk, group, plane).  Only the per-stream tables (33 words per stream, built from the
// 66-byte CDF rows which are contiguous in the container: one coalesced read), the row maxima and a 32-entry
// dequantisation LUT live in shared memory (~18 KB per CTA), so many CTAs stay resident and hide the serial latency of
// each stream's coder.  Symbols are dequantised and stored straight into the destination layout (no uint8 / fp32
// intermediates in HBM).  CODER selects the payload format (container version 1: arithmetic coder, 2: rANS).
template <int OUT_DT, bool PAGED, int CODER, bool TR, bool GT>
__global__ void __launch_bounds__(CT, 12) decode_kernel(DecParams P) {
    extern __shared__ __align__(128) uint32_t smem[];
    uint32_t* tab = smem;                                                            // CT * 33 words (rows of 33, odd)
    float* mx = reinterpret_cast<float*>(smem + CT * kLp);                           // kGroup
    float* lut = mx + kGroup;                                                        // 32
    __shared__ uint32_t s_warp[CT / 32];

    const int tid = threadIdx.x;
    const int j = blockIdx.y;
    const DecChunk dc = P.chunks[j];
    const int NL = P.ppl * P.L;
    const int per_group = NL * P.tpp;
    // blockIdx.x walks the launch's tiles of each group: K planes lb.., then V planes L + lb.. (a latent KV: planes lb..
    // only), and in each plane the wtpp tiles from the chunk's window tile ct0 on (those past the window's ntw leave);
    // `tile` is the tile's index among all of the chunk's tiles (tile_base).  Without windows ct0 = 0 and ntw = wtpp = tpp.
    const int launch_group = P.ppl * P.nlay * P.wtpp;
    const int g = blockIdx.x / launch_group;
    if (g >= dc.ngroups) return;
    const int kt = blockIdx.x - g * launch_group;
    const int kp = kt / P.wtpp;
    const int wt = kt - kp * P.wtpp;
    if (wt >= dc.ntw) return;
    const int nl = kp + (kp < P.nlay ? P.lb : P.L - P.nlay + P.lb);
    const int ct = dc.ct0 + wt;
    const int tile = g * per_group + nl * P.tpp + ct;
    const int tok0 = g * kGroup;
    const int gt = min(kGroup, dc.t - tok0);
    const int c = ct * CT + tid;
    // every stream of the tile takes part in the scan of its lengths; only those in the window are decoded
    const bool in_c = c < P.C;
    const bool active = c >= dc.cw0 && c < dc.cw1;
    const int ncols = min(CT, P.C - ct * CT);
    const Layout lo = layout_of(P, dc.t);

    const uint32_t len = in_c ? load_len(dc.base + lo.off_lengths, ((int64_t)g * NL + nl) * P.C + c, P.compact != 0) : 0u;
    uint32_t tile_total;
    const uint32_t my_rel = block_excl_scan(len, s_warp, &tile_total);
    // the stream's byte offset inside the container; a corrupt lengths section cannot push it outside the payload
    const unsigned long long want = P.tile_base[(int64_t)j * P.tiles_max + tile] + my_rel;
    const bool beyond = want + len > (unsigned long long)dc.payload_bytes;
    const uint32_t my_off = (uint32_t)lo.off_payload + (uint32_t)min(want, (unsigned long long)dc.payload_bytes);

    // stage the per-stream tables (one contiguous run of ncols * 33 halfwords in the container), row maxima, LUT
    const uint16_t* cdf_src = reinterpret_cast<const uint16_t*>(dc.base + lo.off_cdf) + ((int64_t)nl * P.C + ct * CT) * kLp;
    const uint16_t* maxes = reinterpret_cast<const uint16_t*>(dc.base + lo.off_maxes) + (int64_t)nl * dc.t + tok0;
    const float cq = dec_maxq<GT>(P, nl);
    // the rANS table layout of this plane (rans_decode_stream): 16-symbol planes always transposed, 32-symbol ones as
    // the host chose
    const bool trl = CODER == CODER_RANS && (TR || cq <= 7.0f);
    bool built = false;
    uint32_t hl = 0u;                        // version 3: bytes of stream header in front of the rANS state
    if constexpr (CODER == CODER_RANS) {
        if (P.compact) {
            // Container version 3: the stream starts with its symbol histogram; the CDF is a function of it (CdfAccum,
            // the same arithmetic as the encoder), so every thread rebuilds its own table -- row-major or transposed,
            // both conflict-free for thread-private writes.  fl32(n / t) comes from a table that borrows the row-maxima
            // area (mx[0..255] + lut[0] = 257 floats) until the table is built.
            float* pn = mx;
            const float tf = (float)dc.t;
            for (int n = tid; n <= kGroup; n += CT) pn[n] = fdiv((float)n, tf);
            __syncthreads();
            // the stream's header: mask of the symbols that occur, then their counts (the last one is implied).
            // Two readers, chosen per warp: when most lanes' headers are short (<= 8 bytes: few symbols per stream, the
            // streams themselves are short and neighbours share cache lines) each count is one byte load at a position
            // that depends on the mask alone -- branch-free; when a quarter of the lanes or more have long headers, the
            // header is pulled into registers with aligned word loads, only as many as it is long, and consumed a byte
            // at a time (scattered byte loads would cost a cache-line access each): byte loads alone are slower at high
            // entropy, registers alone at low entropy (measured, whole kernel, at 0.6 / 4.1 payload bits per symbol).
            const int nb = 2 * ((int)cq + 1);
            const uint32_t mbytes = (uint32_t)hdr_mask_bytes(nb);
            const uint8_t* sp = dc.base + my_off;
            const uint32_t al = (uint32_t)(reinterpret_cast<uintptr_t>(sp) & 3u);          // 0 or 2
            const uint32_t* wp = reinterpret_cast<const uint32_t*>(sp - al);
            const uint32_t fs = 8u * al;
            uint32_t x_prev = __ldg(wp), x_next = __ldg(wp + 1);
            const uint32_t hb0 = __funnelshift_r(x_prev, x_next, fs);
            uint32_t mask = hb0;
            if (nb <= 8) mask &= 0xffu;
            else if (nb <= 16) mask &= 0xffffu;
            if (nb < 32) mask &= (1u << nb) - 1u;
            hl = hdr_len(mask, nb);
            const uint32_t top = 0x80000000u >> __clz((int)mask);               // the last set bit: its count is implied
            const bool all_short = __popc(__ballot_sync(0xffffffffu, active && hl > 8u)) < 8;
            const uint32_t wany = __reduce_or_sync(0xffffffffu, active ? mask : 0u);
            if (active) {
                uint32_t sum = 0u;
                uint32_t hb[9];
                uint32_t widx = mbytes >> 2, inw = mbytes & 3u, cur = 0u;        // register reader: word, byte in word
                const uint8_t* const cb = sp + mbytes;
                if (!all_short) {
                    hb[0] = hb0;
#pragma unroll
                    for (int k = 1; k < 9; ++k) {
                        hb[k] = 0u;
                        if ((uint32_t)(4 * k) < hl && (k < 5 || nb > 16)) {      // 16-symbol planes: <= 18 bytes
                            x_prev = x_next;
                            x_next = __ldg(wp + k + 1);
                            hb[k] = __funnelshift_r(x_prev, x_next, fs);
                        }
                    }
                    cur = (widx == 0u ? hb[0] : hb[1]) >> (8u * inw);
                }
                auto next_byte = [&]() -> uint32_t {
                    const uint32_t v = cur & 255u;
                    cur >>= 8;
                    if (++inw == 4u) {
                        inw = 0u;
                        ++widx;
                        cur = hb[1];
#pragma unroll
                        for (int k = 2; k < 9; ++k) cur = widx == (uint32_t)k ? hb[k] : cur;
                    }
                    return v;
                };
                auto count = [&](int i) -> uint32_t {                            // called once per i, ascending
                    if (i >= nb) return 0u;
                    const uint32_t bit = 1u << (i & 31);
                    uint32_t n = 0u;
                    if (all_short) {                                             // uniform per warp
                        const uint32_t below = i == 0 ? 0u : mask & (0xffffffffu >> (32 - (i & 31)));
                        const uint32_t v = __ldg(cb + __popc(below));
                        n = (mask & bit) ? v : 0u;
                        n = (top & bit) ? (uint32_t)dc.t - sum : n;
                        sum += n;
                    } else if (mask & bit) {
                        n = (top & bit) ? (uint32_t)dc.t - sum : next_byte();
                        sum += n;
                    }
                    return min(n, (uint32_t)kGroup);                             // a damaged header cannot index past pn[256]
                };
                CdfAccum2 acc;
                acc.init();
                uint32_t c0 = 0u;
                // every entry the symbol search can read (0..15 for <= 16 symbols, 0..31 otherwise), not only the nb the
                // plane uses: a plane of 4..14 or 18..30 symbols would otherwise search uninitialised shared memory.
                // Entries past nb are the reference's CDF there (no mass, one slot each), as in a version-2 CDF row.
                const int nsearch = cq <= 7.0f ? 16 : 32;
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                    if (i < nsearch) {
                        if ((wany >> i) & 1u) acc.absorb(pn[count(i)]);          // uniform per warp: symbols nobody uses
                        uint32_t c1 = acc.value((uint32_t)i + 1u);
                        if (i == 31) c1 = 0x10000u;                              // cdf[32] wraps to 0 in 16 bits and means 65536
                        const uint32_t e = rans_table_entry(c0, c1);
                        if (trl) tab[i * CT + tid] = e;
                        else tab[tid * kLp + i] = e;
                        c0 = c1;
                    }
                }
            }
            __syncthreads();                                                     // pn is dead: maxima and LUT take its place
            for (int i = tid; i < gt; i += CT) mx[i] = half_to_float(maxes[i], P.max_dtype);
            if (tid < 32) lut[tid] = dequant_lut((uint32_t)tid, cq);
            built = true;
        }
    }
    if (!built) {
        if (trl) {
            // TRANSPOSED table: entry i of stream tid at tab[i * CT + tid], entry = (cdf[i] << 16) | freq(i).  Built in two
            // steps through a staging copy of the raw CDF rows that lives in the table's own upper half (bytes 8448..16895):
            // coalesced global -> staging; every thread turns ITS row (33 halfwords, stride 33: conflict-free) into column
            // entries 0..15 (bytes 0..8191, clear of the staging); entries 16..31 -- needed by 32-bin planes only -- go
            // through registers so that they may overwrite the staging once everybody has read it.
            uint16_t* stg = reinterpret_cast<uint16_t*>(smem) + (CT * kLp);            // second half of the CT*kLp words
            for (int e = tid; e < ncols * kLp; e += CT) stg[e] = __ldg(cdf_src + e);
            for (int i = tid; i < gt; i += CT) mx[i] = half_to_float(maxes[i], P.max_dtype);
            if (tid < 32) lut[tid] = dequant_lut((uint32_t)tid, cq);
            __syncthreads();
            const uint16_t* my = stg + tid * kLp;
            if (active) {
                uint32_t c0 = my[0];
    #pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const uint32_t c1 = my[i + 1];
                    tab[i * CT + tid] = rans_table_entry(c0, c1);
                    c0 = c1;
                }
            }
            if (cq > 7.0f) {                                                            // uniform per CTA
                uint32_t cv[17];
                if (active) {
    #pragma unroll
                    for (int i = 0; i < 16; ++i) cv[i] = my[16 + i];
                    cv[16] = 0x10000u;                                                   // cdf[32] is stored as 0 and means 65536
                }
                __syncthreads();
                if (active) {
    #pragma unroll
                    for (int i = 0; i < 16; ++i) tab[(16 + i) * CT + tid] = rans_table_entry(cv[i], cv[i + 1]);
                }
            }
        } else {
            for (int e = tid; e < ncols * kLp; e += CT) {
                const uint32_t i = (uint32_t)e % (uint32_t)kLp;
                const uint32_t c0 = __ldg(cdf_src + e);
                if constexpr (CODER == CODER_RANS) {
                    // (cdf[i] << 16) | freq(i); cdf[32] is stored as 0 and stands for 65536; entry 32 is never searched
                    const uint32_t c1 = i < 31u ? (uint32_t)__ldg(cdf_src + e + 1) : 0x10000u;
                    tab[e] = i < 32u ? rans_table_entry(c0, c1) : 0xFFFFFFFFu;
                } else {
                    tab[e] = dec_table_entry(i, c0);
                }
            }
            for (int i = tid; i < gt; i += CT) mx[i] = half_to_float(maxes[i], P.max_dtype);
            if (tid < 32) lut[tid] = dequant_lut((uint32_t)tid, cq);
        }
    }
    __syncthreads();

    if (!active) return;
    const uint32_t* erow = tab + tid * kLp;
    const int oc = c + dc.dshift;                          // destination channel
    const int h = oc / P.D;
    uint16_t* dst = const_cast<uint16_t*>(dec_plane<GT>(P, nl)) + (PAGED ? 0 : (dc.dst_tok + tok0) * P.sT) + (int64_t)h * P.sH +
                    (oc - h * P.D);
    const int64_t* slots = PAGED ? P.slot_map + dc.dst_tok + tok0 : nullptr;
    uint32_t bad = beyond ? 2u : 0u;
    if constexpr (CODER == CODER_RANS) {
        uint32_t xf;
        const uint32_t one = min((uint32_t)P.n_chunks, 1u);      // 1, but opaque to the compiler (see rans_decode_stream)
        const uint32_t* pk = trl ? tab + tid : tab + tid * kLp;
        if (cq <= 7.0f) {
            // the LUT replica in rows 16..31 of this thread's column, which only this thread reads (whatever the table
            // build staged there is dead after the barrier above)
#pragma unroll
            for (int s = 0; s < 16; ++s) tab[(16 + s) * CT + tid] = __float_as_uint(lut[s]);
            xf = rans_decode_stream<OUT_DT, 4, PAGED, true>(dc.base, my_off + hl, pk, lut, mx, dst, (uint32_t)P.sT, gt, slots, one);
        } else {
            xf = rans_decode_stream<OUT_DT, 5, PAGED, TR>(dc.base, my_off + hl, pk, lut, mx, dst, (uint32_t)P.sT, gt, slots, one);
        }
        bad |= xf != kRansLow ? 1u : 0u;
    } else {
        if (cq <= 7.0f) decode_stream<OUT_DT, 4, PAGED>(dc.base, my_off, erow, lut, mx, dst, (uint32_t)P.sT, gt, slots);   // <= 16 bins: symbols 0..14
        else decode_stream<OUT_DT, 5, PAGED>(dc.base, my_off, erow, lut, mx, dst, (uint32_t)P.sT, gt, slots);
    }
    if (bad != 0u && P.status != nullptr) atomicOr(&P.status[j], bad);
}

// ------------------------------------------------------------------------------------------ host side
int make_plane_table(const b200kv_kv_desc* kv, const float* key_bins, const float* value_bins, PlaneTable* out) {
    B2_REQUIRE(kv != nullptr, "kv descriptor is NULL");
    B2_REQUIRE(!kv_split(kv), B2_SPLIT_REFUSED);
    B2_REQUIRE(kv->L > 0 && 2 * kv->L <= B200KV_MAX_PLANES, "L out of range");
    B2_REQUIRE(kv->H > 0 && kv->D > 0, "H/D must be positive");
    const int es = kv_elem_bytes(kv);
    B2_REQUIRE(es != 0, "dtype must be one of B200KV_DT_*");
    B2_REQUIRE(kv->planes != nullptr || kv->base != nullptr, "no KV pointer");
    for (int kvi = 0; kvi < kv_ppl(kv); ++kvi)
        for (int l = 0; l < kv->L; ++l) {
            const int nl = kvi * kv->L + l;
            const uint16_t* p = reinterpret_cast<const uint16_t*>(
                kv->planes ? static_cast<const uint8_t*>(kv->planes[nl])
                           : static_cast<const uint8_t*>(kv->base) + (l * kv->sL + kvi * kv->sKV) * es);
            B2_REQUIRE(p != nullptr, "NULL plane pointer");
            out->p[nl] = p;
            const float bins = kvi ? value_bins[l] : key_bins[l];
            out->maxq[nl] = floorf(bins / 2.0f) - 1.0f;       // bins // 2 - 1  (cachegen_encoder.py:53)
            B2_REQUIRE(out->maxq[nl] >= 1.0f && out->maxq[nl] <= 15.0f, "bins must be in [4, 32]");
        }
    return 0;
}

static int tiles_per_plane(int C) { return (C + CT - 1) / CT; }

// The CacheGen codec quantises 16-bit elements: a one-byte KV (FP8) is refused here, before anything is enqueued, and
// stored by the lossless codec instead
static int cachegen_dtype_ok(const b200kv_kv_desc* kv) {
    B2_REQUIRE(kv != nullptr, "kv descriptor is NULL");
    B2_REQUIRE(!kv_split(kv), B2_SPLIT_REFUSED);
    B2_REQUIRE(kv_elem_bytes(kv) == 2,
               "CacheGen codes bf16 / fp16 KV only; one-byte (FP8) KV is stored by the lossless codec");
    return 0;
}

// ---- optional per-kernel timing (bench.py's roofline leg): events around each launch of the last call
enum { kProfAbsmax = 0, kProfCdf, kProfEncode, kProfFinalize, kProfTileSum, kProfTileScan, kProfDecode, kProfCount };
static bool g_prof_on = false;
static cudaEvent_t g_prof_ev[kProfCount][2];
static bool g_prof_have[kProfCount];
static bool g_prof_init = false;

struct ProfScope {
    int slot;
    cudaStream_t stream;
    ProfScope(int slot_, cudaStream_t s) : slot(slot_), stream(s) {
        if (!g_prof_on) return;
        if (!g_prof_init) {
            for (int i = 0; i < kProfCount; ++i) { cudaEventCreate(&g_prof_ev[i][0]); cudaEventCreate(&g_prof_ev[i][1]); }
            g_prof_init = true;
        }
        cudaEventRecord(g_prof_ev[slot][0], stream);
    }
    ~ProfScope() {
        if (!g_prof_on) return;
        cudaEventRecord(g_prof_ev[slot][1], stream);
        g_prof_have[slot] = true;
    }
};

static int enc_tempw(bool fused, int coder, bool compact = false) {
    if (compact) return TEMPW_FUSED_RANS_HDR;
    return fused ? (coder == CODER_RANS ? TEMPW_FUSED_RANS : TEMPW_FUSED) : TEMPW_SPLIT;
}

// Everything in front of off_state is zeroed by every call.  sync: encode_kernel<FUSED = true>'s ticket counter, then
// one ready counter per unit (n_units = chunks x planes)
static size_t enc_ws_layout(int64_t n_tiles_alloc, int n_chunks, int64_t n_units, int tempw, int coder, bool compact,
                            size_t* off_tot, size_t* off_totals, size_t* off_err, size_t* off_sync, size_t* off_state,
                            size_t* off_temp) {
    size_t o = 0;
    *off_tot = o;    o += (size_t)n_tiles_alloc * 4;  o = (o + 255) & ~(size_t)255;
    *off_totals = o; o += (size_t)n_chunks * 8;       o = (o + 255) & ~(size_t)255;
    *off_err = o;    o += (size_t)n_chunks * 4;       o = (o + 255) & ~(size_t)255;
    *off_sync = o;   o += (size_t)(1 + n_units) * 4;  o = (o + 255) & ~(size_t)255;
    *off_state = o;  o += coder == CODER_RANS ? (size_t)n_tiles_alloc * CT * (compact ? 16 : 4) : 0;  o = (o + 255) & ~(size_t)255;
    *off_temp = o;   o += (size_t)n_tiles_alloc * CT * (size_t)tempw * 4;
    return (o + 255) & ~(size_t)255;
}

// b200kv_encode_layers_plan's workspace: the state that lives across calls (err, running payload totals, chunk bases,
// cursor + fail_from), then one call's scratch -- tile totals, payload totals, coder states and temp rows for the tiles
// of at most max_layers layers, and encode_kernel's ticket and ready counters for the units (chunks x planes) of such a call.
struct EnclWs { size_t err, ptotal, cbase, state, tot, totals, sync, rstate, temp, bytes; };
static EnclWs encl_ws_layout(int n_chunks, int64_t call_tiles, int64_t call_units) {
    EnclWs w;
    size_t o = 0;
    auto take = [&](size_t* off, size_t n) { *off = o; o = (o + n + 255) & ~(size_t)255; };
    take(&w.err, (size_t)n_chunks * 4);
    take(&w.ptotal, (size_t)n_chunks * 8);
    take(&w.cbase, (size_t)n_chunks * 8);
    take(&w.state, 16);
    take(&w.tot, (size_t)call_tiles * 4);
    take(&w.totals, (size_t)n_chunks * 8);
    take(&w.sync, (size_t)(1 + call_units) * 4);
    take(&w.rstate, (size_t)call_tiles * CT * 16);
    take(&w.temp, (size_t)call_tiles * CT * TEMPW_FUSED_RANS_HDR * 4);
    w.bytes = o;
    return w;
}

// What b200kv_encode_layers_plan decided, kept in the caller's b200kv_encode_plan_t: the kernels' parameter block (its
// counters live in the workspace), the layers encoded so far and the most one call may take.
constexpr uint32_t kEncPlanMagic = 0x4e4c5045u;   // "EPLN"
struct EncPlan {
    uint32_t magic;
    int32_t max_layers;
    LayerSet done;           // the layers encoded so far
    EncParams P;
};
static_assert(sizeof(EncPlan) <= sizeof(b200kv_encode_plan_t), "b200kv_encode_plan_t too small");

constexpr size_t kSmemFused = (size_t)(((CT * SYMW + (CT * kLp * 2 + 3) / 4 + 3) & ~3) + kGroup + 8) * 4;
constexpr int kStageRans = 12 * 1024;   // compact_kernel's stage without an entropy hint (b200kv_encode_chunks)

// every plane's token rows can be read with 128-bit loads
static bool rows_vec(const EncParams& P) {
    bool vec = (P.D % 8 == 0) && (P.sT % 8 == 0) && (P.sH % 8 == 0);
    for (int nl = 0; nl < P.ppl * P.L && vec; ++nl) vec = (reinterpret_cast<uintptr_t>(P.pt.p[nl]) & 15) == 0;
    return vec;
}

// absmax over the rows of the launch's planes (P.lb, P.nlay) and tokens [0, total_tokens) of the call (chunks > 256
// tokens; shorter chunks have encode_kernel compute their maxima)
static int launch_absmax(const EncParams& P, int64_t total_tokens, cudaStream_t stream) {
    const bool vec = P.vec != 0;
    const bool paged = P.slot_map != nullptr;
    const int64_t rows = (int64_t)P.ppl * P.nlay * total_tokens;
    const int64_t blocks = (rows + 7) / 8;
    B2_REQUIRE(blocks < (1ll << 31), "too many rows in one call");
    if (vec && !paged) absmax_kernel<true, false><<<(unsigned)blocks, 256, 0, stream>>>(P, total_tokens);
    else if (vec) absmax_kernel<true, true><<<(unsigned)blocks, 256, 0, stream>>>(P, total_tokens);
    else if (!paged) absmax_kernel<false, false><<<(unsigned)blocks, 256, 0, stream>>>(P, total_tokens);
    else absmax_kernel<false, true><<<(unsigned)blocks, 256, 0, stream>>>(P, total_tokens);
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// The persistent encode_kernel<FUSED = true>: as many CTAs as fit on the device at once (the occupancy is asked once per
// instantiation), never more than there are tickets.  P.ticket and P.ready must be zero.
template <int DT, bool PAGED, int CODER>
static int launch_encode_fused(const EncParams& P, cudaStream_t stream) {
    static int occ = 0;
    auto kern = encode_kernel<true, DT, PAGED, CODER>;
    B2_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemFused));
    if (occ == 0) {
        int n = 0;
        B2_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, CT, kSmemFused));
        B2_REQUIRE(n > 0, "encode_kernel does not fit on this device");
        occ = n;
    }
    int dev = 0, sms = 0;
    B2_CHECK_CUDA(cudaGetDevice(&dev));
    B2_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int64_t tickets = ((int64_t)P.n_chunks * P.ppl * P.nlay + kAbsLead) * (kAbsItems + P.tpp);
    B2_REQUIRE(tickets < (1ll << 31) - 2, "too many work items in one call");
    const int64_t grid = std::min<int64_t>((int64_t)occ * sms, tickets);
    kern<<<(unsigned)grid, CT, kSmemFused, stream>>>(P);
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// chunk descriptors, tile bases, and -- for more than kInlinePlanes planes (NP) only -- the device copy of the plane table
static size_t dec_ws_layout(int64_t tiles_max, int n_chunks, int NP, size_t* off_tb, size_t* off_pt) {
    size_t o = ((size_t)n_chunks * sizeof(DecChunk) + 255) & ~(size_t)255;
    *off_tb = o;
    o += (size_t)n_chunks * (size_t)tiles_max * 8;
    o = (o + 255) & ~(size_t)255;
    *off_pt = o;
    if (NP > kInlinePlanes) o = (o + sizeof(PlaneTable) + 255) & ~(size_t)255;
    return o;
}

// What b200kv_decode_plan decided, kept in the caller's b200kv_decode_plan_t: the decode kernel's parameter block (its
// chunk descriptors and tile bases live in the workspace) and the kernel variant.
constexpr uint32_t kPlanMagic = 0x4e4c5044u;   // "DPLN"
struct DecPlan {
    uint32_t magic;
    int32_t coder;           // CODER_AC | CODER_RANS
    int32_t transposed;      // rANS table layout
    int32_t gmax;            // groups of the longest chunk
    DecParams P;
};
static_assert(sizeof(DecPlan) <= sizeof(b200kv_decode_plan_t), "b200kv_decode_plan_t too small");

}  // namespace b200kv

using namespace b200kv;

extern "C" {

int b200kv_container_layout(int32_t L, int32_t H, int32_t D, int32_t ntokens, b200kv_layout* out) {
    return b200kv_container_layout_v(L, H, D, ntokens, CODER_RANS, out);
}

int b200kv_container_layout_v(int32_t L, int32_t H, int32_t D, int32_t ntokens, int32_t coder, b200kv_layout* out) {
    B2_REQUIRE(out != nullptr && L > 0 && H > 0 && D > 0 && ntokens > 0, "bad shape");
    const int ppl = (coder & B200KV_KV_LATENT) ? 1 : 2;
    coder &= ~B200KV_KV_LATENT;
    B2_REQUIRE(coder >= CODER_AC && coder <= CODER_RANS_COMPACT, "unknown coder");
    const int compact = coder == CODER_RANS_COMPACT ? 1 : 0;
    B2_REQUIRE(ppl == 2 || compact, "a latent KV (container version 4) is coded with B200KV_CODER_RANS_COMPACT only");
    B2_REQUIRE(!compact || ntokens <= kGroup, "the compact container holds chunks of at most 256 tokens");
    const Layout lo = make_layout(L, H * D, ntokens, compact, ppl);
    out->off_cdf = lo.off_cdf;
    out->off_maxes = lo.off_maxes;
    out->off_lengths = lo.off_lengths;
    out->off_payload = lo.off_payload;
    out->fixed_bytes = lo.off_payload;
    // per stream per group: <= 16 bits per symbol (CDF width >= 1/65536) + termination -- 2 flush bits + pad for the
    // arithmetic coder, the 32-bit final state for rANS
    const int64_t streams = (int64_t)ppl * L * H * D;
    out->max_total_bytes = align16(lo.off_payload + streams * (2 * (int64_t)ntokens + 4 * (int64_t)lo.ngroups +
                                                              (compact ? kHdrMax : 0)) + 16);
    return 0;
}

int b200kv_plane_offsets(const void* container, int64_t nbytes, int64_t* out, int32_t n_out) {
    B2_REQUIRE(container != nullptr && out != nullptr && nbytes >= (int64_t)sizeof(b200kv_header), "bad arguments");
    b200kv_header hd;
    memcpy(&hd, container, sizeof(hd));
    B2_REQUIRE(hd.magic == B200KV_MAGIC && (hd.version == 3 || hd.version == 4), "not a version-3 or version-4 container");
    B2_REQUIRE(hd.L > 0 && 2 * (int64_t)hd.L <= B200KV_MAX_PLANES && hd.H > 0 && hd.D > 0 && hd.ntokens > 0 &&
               hd.ntokens <= (uint32_t)kGroup, "impossible shape");
    const int ppl = hd.version == 4 ? 1 : 2;
    const int NL = ppl * (int)hd.L;
    const int64_t C = (int64_t)hd.H * hd.D;
    B2_REQUIRE(n_out >= NL + 1, "out must hold P + 1 offsets (P = 2L, or L for version 4)");
    const Layout lo = make_layout((int)hd.L, (int)C, (int)hd.ntokens, 1, ppl);
    B2_REQUIRE(nbytes >= lo.off_payload, "buffer shorter than the fixed sections");
    const uint8_t* half = static_cast<const uint8_t*>(container) + lo.off_lengths;
    int64_t o = lo.off_payload;
    out[0] = o;
    for (int p = 0; p < NL; ++p) {
        uint32_t sum = 0;                          // <= 4096 * 255 per plane at the largest shapes: no overflow
        for (int64_t c = 0; c < C; ++c) sum += half[p * C + c];
        o += 2 * (int64_t)sum;
        out[p + 1] = o;
    }
    return o == (int64_t)hd.total_bytes ? 0 : 1;
}

int b200kv_plane_offsets_device(const void* containers, int64_t stride, int32_t n, int64_t* out, void* stream) {
    B2_REQUIRE(containers != nullptr && out != nullptr && n > 0 && stride >= (int64_t)sizeof(b200kv_header) &&
               (stride & 15) == 0 && (reinterpret_cast<uintptr_t>(containers) & 15) == 0, "bad arguments");
    plane_offsets_kernel<<<(unsigned)n, 1024, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const uint8_t*>(containers),
                                                                                      stride, out);
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int64_t b200kv_encode_workspace_bytes(int32_t L, int32_t H, int32_t D, int32_t chunk_tokens, int32_t n_chunks,
                                      int32_t coder) {
    if (L <= 0 || H <= 0 || D <= 0 || chunk_tokens <= 0 || n_chunks <= 0) return -2;
    const int ppl = (coder & B200KV_KV_LATENT) ? 1 : 2;
    coder &= 0xff;
    const bool compact = coder == CODER_RANS_COMPACT;          // same kernels; rows hold the stream header too
    if (compact) coder = CODER_RANS;
    if (coder != CODER_AC && coder != CODER_RANS) return -2;
    if (compact && chunk_tokens > kGroup) return -2;
    if (ppl == 1 && !compact) return -2;
    const int64_t G = (chunk_tokens + kGroup - 1) / kGroup;
    const int64_t n_tiles = (int64_t)n_chunks * G * ppl * L * tiles_per_plane(H * D);
    size_t a, b, c, d, e, f;
    return (int64_t)enc_ws_layout(n_tiles, n_chunks, (int64_t)n_chunks * ppl * L, enc_tempw(chunk_tokens <= kGroup, coder, compact),
                                  coder, compact, &a, &b, &c, &d, &e, &f);
}

int64_t b200kv_decode_workspace_bytes(int32_t L, int32_t H, int32_t D, int32_t chunk_tokens, int32_t n_chunks) {
    if (L <= 0 || H <= 0 || D <= 0 || chunk_tokens <= 0 || n_chunks <= 0) return -2;
    const int64_t G = (chunk_tokens + kGroup - 1) / kGroup;
    const int64_t tiles_max = G * 2 * L * tiles_per_plane(H * D);     // 2L planes: also enough for a latent KV's L
    size_t a, b;
    return (int64_t)dec_ws_layout(tiles_max, n_chunks, 2 * L, &a, &b);
}

int b200kv_encode_chunks(const b200kv_kv_desc* kv, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                         int32_t last_chunk_tokens, const float* key_bins, const float* value_bins, int32_t coder,
                         void* out, int64_t out_stride, uint64_t* sizes_out, void* workspace, int64_t workspace_bytes,
                         void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    EncParams P;
    B2_REQUIRE(key_bins && value_bins, "bins are NULL");
    if (int rc = cachegen_dtype_ok(kv)) return rc;
    const bool hint_mid = (coder & B200KV_ENCODE_HINT_MID_ENTROPY) != 0;
    coder &= 0xff;
    B2_REQUIRE(coder >= CODER_AC && coder <= CODER_RANS_COMPACT, "coder must be one of B200KV_CODER_*");
    P.compact = coder == CODER_RANS_COMPACT ? 1 : 0;
    if (P.compact) coder = CODER_RANS;                          // version 3 = rANS payload + compact side information
    P.coder = coder;
    if (int rc = make_plane_table(kv, key_bins, value_bins, &P.pt)) return rc;
    P.ppl = kv_ppl(kv);
    B2_REQUIRE(P.ppl == 2 || P.compact, "a latent KV (B200KV_KV_LATENT) is coded with B200KV_CODER_RANS_COMPACT only");
    B2_REQUIRE(n_chunks > 0 && chunk_tokens > 0, "n_chunks / chunk_tokens must be positive");
    B2_REQUIRE(!P.compact || chunk_tokens <= kGroup, "the compact container (B200KV_CODER_RANS_COMPACT) holds chunks of at most 256 tokens");
    B2_REQUIRE(last_chunk_tokens > 0 && last_chunk_tokens <= chunk_tokens, "last_chunk_tokens out of range");
    B2_REQUIRE(out != nullptr && (reinterpret_cast<uintptr_t>(out) & 15) == 0 && (out_stride & 15) == 0,
               "out / out_stride must be 16-byte aligned");
    B2_REQUIRE(tok_begin >= 0, "tok_begin must be >= 0");
    P.sT = kv->sT; P.sH = kv->sH; P.tok_begin = tok_begin;
    P.slot_map = kv->slot_map;
    const bool paged = kv->slot_map != nullptr;
    P.L = kv->L; P.H = kv->H; P.D = kv->D; P.C = kv->H * kv->D; P.dtype = kv_dtype(kv);
    P.n_chunks = n_chunks; P.chunk_tokens = chunk_tokens; P.last_chunk_tokens = last_chunk_tokens;
    P.tpp = tiles_per_plane(P.C);
    P.out = static_cast<uint8_t*>(out);
    P.out_stride = out_stride;
    P.sizes_out = sizes_out;
    P.lb = 0; P.nlay = P.L;
    P.arena = nullptr; P.arena_bytes = 0; P.chunk_base = nullptr; P.cursor = nullptr; P.fail_from = nullptr;
    P.ptotal = nullptr; P.seg = nullptr; P.layers_left = 0;
    const Layout lo = make_layout(P.L, P.C, chunk_tokens, P.compact, P.ppl);
    B2_REQUIRE(out_stride >= lo.off_payload + 16, "out_stride smaller than the fixed container sections");

    const int64_t G = lo.ngroups;
    const int64_t per_group = (int64_t)P.ppl * P.L * P.tpp;
    const int64_t tiles_full = G * per_group;
    const int64_t n_tiles = (int64_t)n_chunks * tiles_full;     // tiles beyond a ragged last chunk exit at once
    const bool fused = chunk_tokens <= kGroup;
    P.tiles_full = (int32_t)tiles_full;
    P.tempw = enc_tempw(fused, coder, P.compact != 0);
    size_t off_tot, off_totals, off_err, off_sync, off_state, off_temp;
    const size_t need = enc_ws_layout(n_tiles, n_chunks, (int64_t)n_chunks * P.ppl * P.L, P.tempw, coder, P.compact != 0, &off_tot,
                                      &off_totals, &off_err, &off_sync, &off_state, &off_temp);
    B2_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)need, "workspace too small");
    B2_REQUIRE(n_tiles < (1ll << 31) && tiles_full < (1ll << 31), "too many tiles in one call");
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    P.tile_tot = reinterpret_cast<uint32_t*>(ws + off_tot);
    P.totals = reinterpret_cast<unsigned long long*>(ws + off_totals);
    P.err = reinterpret_cast<unsigned int*>(ws + off_err);
    P.temp = reinterpret_cast<uint32_t*>(ws + off_temp);
    P.rstate = reinterpret_cast<uint32_t*>(ws + off_state);
    P.ticket = reinterpret_cast<unsigned int*>(ws + off_sync);
    P.ready = P.ticket + 1;
    P.vec = rows_vec(P) ? 1 : 0;
    B2_CHECK_CUDA(cudaMemsetAsync(ws, 0, off_state, stream));    // counters only; states and temp rows need no init

    // 1) per-(plane, token) absmax -> maxes sections: a kernel of its own for chunks > 256 tokens, inside encode_kernel
    //    for the others
    const int64_t total_tokens = (int64_t)(n_chunks - 1) * chunk_tokens + last_chunk_tokens;
    for (int i = 0; i <= kProfFinalize; ++i) g_prof_have[i] = false;
    if (!fused) {
        ProfScope prof(kProfAbsmax, stream);
        if (int rc = launch_absmax(P, total_tokens, stream)) return rc;
    }
    // 2) encode (streams -> temp rows, lengths, tile totals)
    const size_t smem_split = (size_t)(((CT * PAIRW + 3) & ~3) + kGroup + 4) * 4;
    const size_t smem_cdf = (size_t)(CT * PAIRW + kGroup) * 4;
#define B2_LAUNCH_ENC1(FUSED, DT, PAGED, CODER, SMEM)                                                      \
    do {                                                                                                   \
        B2_CHECK_CUDA(cudaFuncSetAttribute(encode_kernel<FUSED, DT, PAGED, CODER>,                         \
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(SMEM)));     \
        encode_kernel<FUSED, DT, PAGED, CODER><<<(unsigned)n_tiles, CT, (SMEM), stream>>>(P);              \
    } while (0)
#define B2_LAUNCH_ENC(FUSED, DT, PAGED, SMEM)                                                              \
    do {                                                                                                   \
        if (coder == CODER_RANS) B2_LAUNCH_ENC1(FUSED, DT, PAGED, CODER_RANS, SMEM);                       \
        else B2_LAUNCH_ENC1(FUSED, DT, PAGED, CODER_AC, SMEM);                                             \
    } while (0)
#define B2_LAUNCH_ENC2(FUSED, SMEM)                                                                        \
    do {                                                                                                   \
        if (P.dtype == B200KV_DT_BF16) { if (paged) B2_LAUNCH_ENC(FUSED, 0, true, SMEM); else B2_LAUNCH_ENC(FUSED, 0, false, SMEM); } \
        else { if (paged) B2_LAUNCH_ENC(FUSED, 1, true, SMEM); else B2_LAUNCH_ENC(FUSED, 1, false, SMEM); } \
    } while (0)
    if (fused) {
        ProfScope prof(kProfEncode, stream);
        int rc;
        if (P.dtype == B200KV_DT_BF16) {
            if (paged) rc = coder == CODER_RANS ? launch_encode_fused<0, true, CODER_RANS>(P, stream) : launch_encode_fused<0, true, CODER_AC>(P, stream);
            else rc = coder == CODER_RANS ? launch_encode_fused<0, false, CODER_RANS>(P, stream) : launch_encode_fused<0, false, CODER_AC>(P, stream);
        } else {
            if (paged) rc = coder == CODER_RANS ? launch_encode_fused<1, true, CODER_RANS>(P, stream) : launch_encode_fused<1, true, CODER_AC>(P, stream);
            else rc = coder == CODER_RANS ? launch_encode_fused<1, false, CODER_RANS>(P, stream) : launch_encode_fused<1, false, CODER_AC>(P, stream);
        }
        if (rc) return rc;
    } else {
        const unsigned cdf_blocks = (unsigned)((int64_t)n_chunks * per_group);
        {
            ProfScope prof(kProfCdf, stream);
            if (P.dtype == B200KV_DT_BF16) {
                if (paged) cdf_kernel<0, true><<<cdf_blocks, CT, smem_cdf, stream>>>(P);
                else cdf_kernel<0, false><<<cdf_blocks, CT, smem_cdf, stream>>>(P);
            } else {
                if (paged) cdf_kernel<1, true><<<cdf_blocks, CT, smem_cdf, stream>>>(P);
                else cdf_kernel<1, false><<<cdf_blocks, CT, smem_cdf, stream>>>(P);
            }
        }
        B2_CHECK_CUDA(cudaGetLastError());
        ProfScope prof(kProfEncode, stream);
        B2_LAUNCH_ENC2(false, smem_split);
    }
#undef B2_LAUNCH_ENC2
#undef B2_LAUNCH_ENC
#undef B2_LAUNCH_ENC1
    B2_CHECK_CUDA(cudaGetLastError());
    // 3) compaction (collect_bytes) + headers + sizes
    {
        ProfScope prof(kProfFinalize, stream);
        // stage = the fused mode's worst case (128 x 160 B + alignment phase); in split mode a tile can in principle
        // reach 128 x 528 B, but sizing the stage for that would leave 3 CTAs per SM for streams that are typically
        // a few dozen bytes long -- oversized tiles take the direct path inside the kernel
        P.stage_bytes = coder == CODER_RANS ? CT * (TEMPW_FUSED_RANS * 4 + 4) + 32 : CT * TEMPW_FUSED * 4 + 32;
        // The kernel waits on sparse row reads: more resident CTAs hide more of that latency.  Without an entropy hint a
        // tile's streams total a few KB, so a 12 KB stage (12 CTAs per SM instead of 9: measured faster) covers
        // them; the rare larger tile takes the kernel's direct path.
        if (coder == CODER_RANS && !hint_mid) P.stage_bytes = 12 * 1024;
        B2_CHECK_CUDA(cudaFuncSetAttribute(compact_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, P.stage_bytes));
        enc_scan_kernel<<<(unsigned)n_chunks, 1024, 0, stream>>>(P);
        compact_kernel<<<(unsigned)n_tiles, CT, (size_t)P.stage_bytes, stream>>>(P);
        finalize_kernel<<<(n_chunks + 127) / 128, 128, 0, stream>>>(P);
    }
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int64_t b200kv_encode_layers_workspace_bytes(int32_t L, int32_t H, int32_t D, int32_t chunk_tokens, int32_t n_chunks,
                                             int32_t max_layers) {
    if (L <= 0 || H <= 0 || D <= 0 || chunk_tokens <= 0 || chunk_tokens > kGroup || n_chunks <= 0 || max_layers <= 0 ||
        max_layers > L)
        return -2;
    return (int64_t)encl_ws_layout(n_chunks, (int64_t)n_chunks * 2 * max_layers * tiles_per_plane(H * D),
                                   (int64_t)n_chunks * 2 * max_layers).bytes;
}

int b200kv_encode_layers_plan(const b200kv_kv_desc* kv, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                              int32_t last_chunk_tokens, const float* key_bins, const float* value_bins, int32_t coder,
                              void* arena, int64_t arena_bytes, void* fixed_out, int64_t fixed_stride, int64_t* seg_sizes_out,
                              uint64_t* sizes_out, int32_t max_layers, void* workspace, int64_t workspace_bytes,
                              b200kv_encode_plan_t* plan_out, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B2_REQUIRE(plan_out != nullptr, "plan is NULL");
    EncPlan* plan = reinterpret_cast<EncPlan*>(plan_out);
    plan->magic = 0u;
    EncParams& P = plan->P;
    B2_REQUIRE(key_bins && value_bins, "bins are NULL");
    B2_REQUIRE((coder & 0xff) == CODER_RANS_COMPACT,
               "the layer-wise encode writes compact containers only (B200KV_CODER_RANS_COMPACT)");
    if (int rc = cachegen_dtype_ok(kv)) return rc;
    if (int rc = make_plane_table(kv, key_bins, value_bins, &P.pt)) return rc;
    P.ppl = kv_ppl(kv);
    B2_REQUIRE(n_chunks > 0 && chunk_tokens > 0, "n_chunks / chunk_tokens must be positive");
    B2_REQUIRE(chunk_tokens <= kGroup, "the compact container (B200KV_CODER_RANS_COMPACT) holds chunks of at most 256 tokens");
    B2_REQUIRE(last_chunk_tokens > 0 && last_chunk_tokens <= chunk_tokens, "last_chunk_tokens out of range");
    B2_REQUIRE(tok_begin >= 0, "tok_begin must be >= 0");
    B2_REQUIRE(max_layers > 0 && max_layers <= kv->L, "max_layers out of range");
    B2_REQUIRE(arena != nullptr && arena_bytes >= 0 && seg_sizes_out != nullptr && sizes_out != nullptr, "bad outputs");
    B2_REQUIRE(fixed_out != nullptr && (reinterpret_cast<uintptr_t>(fixed_out) & 15) == 0 && (fixed_stride & 15) == 0,
               "fixed_out / fixed_stride must be 16-byte aligned");
    P.sT = kv->sT; P.sH = kv->sH; P.tok_begin = tok_begin;
    P.slot_map = kv->slot_map;
    P.L = kv->L; P.H = kv->H; P.D = kv->D; P.C = kv->H * kv->D; P.dtype = kv_dtype(kv);
    P.n_chunks = n_chunks; P.chunk_tokens = chunk_tokens; P.last_chunk_tokens = last_chunk_tokens;
    P.tpp = tiles_per_plane(P.C);
    P.coder = CODER_RANS;
    P.compact = 1;
    P.tempw = TEMPW_FUSED_RANS_HDR;
    P.stage_bytes = kStageRans;
    const Layout lo = make_layout(P.L, P.C, chunk_tokens, 1, P.ppl);
    B2_REQUIRE(fixed_stride >= lo.off_payload, "fixed_stride smaller than the fixed container sections");
    P.out = static_cast<uint8_t*>(fixed_out);
    P.out_stride = fixed_stride;
    P.sizes_out = sizes_out;
    P.arena = static_cast<uint8_t*>(arena);
    P.arena_bytes = arena_bytes;
    P.seg = seg_sizes_out;
    const int64_t call_tiles = (int64_t)n_chunks * P.ppl * max_layers * P.tpp;
    B2_REQUIRE(call_tiles < (1ll << 31), "too many tiles in one call");
    const EnclWs w = encl_ws_layout(n_chunks, call_tiles, (int64_t)n_chunks * P.ppl * max_layers);
    B2_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)w.bytes, "workspace too small");
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    P.err = reinterpret_cast<unsigned int*>(ws + w.err);
    P.ptotal = reinterpret_cast<unsigned long long*>(ws + w.ptotal);
    P.chunk_base = reinterpret_cast<unsigned long long*>(ws + w.cbase);
    P.cursor = reinterpret_cast<unsigned long long*>(ws + w.state);
    P.fail_from = reinterpret_cast<unsigned int*>(ws + w.state + 8);
    P.tile_tot = reinterpret_cast<uint32_t*>(ws + w.tot);
    P.totals = reinterpret_cast<unsigned long long*>(ws + w.totals);
    P.rstate = reinterpret_cast<uint32_t*>(ws + w.rstate);
    P.temp = reinterpret_cast<uint32_t*>(ws + w.temp);
    P.ticket = reinterpret_cast<unsigned int*>(ws + w.sync);
    P.ready = P.ticket + 1;
    P.vec = rows_vec(P) ? 1 : 0;
    // counters; the fixed images too, so that their padding bytes are zero whatever the buffer held before
    B2_CHECK_CUDA(cudaMemsetAsync(ws, 0, w.tot, stream));
    B2_CHECK_CUDA(cudaMemsetAsync(fixed_out, 0, (size_t)fixed_stride * n_chunks, stream));
    encl_init_kernel<<<1, 1, 0, stream>>>(P);
    B2_CHECK_CUDA(cudaGetLastError());
    B2_CHECK_CUDA(cudaFuncSetAttribute(compact_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, P.stage_bytes));
    plan->max_layers = max_layers;
    plan->done = LayerSet::range(0, 0);
    plan->magic = kEncPlanMagic;
    return 0;
}

int b200kv_encode_layers(b200kv_encode_plan_t* plan_in, int32_t layer_begin, int32_t layer_end, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B2_REQUIRE(plan_in != nullptr, "plan is NULL");
    EncPlan* plan = reinterpret_cast<EncPlan*>(plan_in);
    B2_REQUIRE(plan->magic == kEncPlanMagic, "not a plan made by b200kv_encode_layers_plan");
    EncParams P = plan->P;
    B2_REQUIRE(layer_begin >= 0 && layer_begin < layer_end && layer_end <= P.L, "layer range out of range");
    B2_REQUIRE(layer_end - layer_begin <= plan->max_layers, "more layers than the plan's workspace holds");
    const LayerSet bits = LayerSet::range(layer_begin, layer_end);
    B2_REQUIRE(!plan->done.intersects(bits), "a layer of the range was encoded before");
    P.lb = layer_begin;
    P.nlay = layer_end - layer_begin;
    P.layers_left = P.L - plan->done.count() - bits.count();
    P.tiles_full = P.ppl * P.nlay * P.tpp;
    const int64_t n_tiles = (int64_t)P.n_chunks * P.tiles_full;
    // encode_kernel's ticket and ready counters start at zero (the maxima are computed inside it)
    B2_CHECK_CUDA(cudaMemsetAsync(P.ticket, 0, (size_t)(1 + (int64_t)P.n_chunks * P.ppl * P.nlay) * 4, stream));
    int rc;
    if (P.dtype == B200KV_DT_BF16) rc = P.slot_map ? launch_encode_fused<0, true, CODER_RANS>(P, stream) : launch_encode_fused<0, false, CODER_RANS>(P, stream);
    else rc = P.slot_map ? launch_encode_fused<1, true, CODER_RANS>(P, stream) : launch_encode_fused<1, false, CODER_RANS>(P, stream);
    if (rc) return rc;
    enc_scan_kernel<<<(unsigned)P.n_chunks, 1024, 0, stream>>>(P);
    place_kernel<<<1, 1024, 0, stream>>>(P);
    compact_kernel<<<(unsigned)n_tiles, CT, (size_t)P.stage_bytes, stream>>>(P);
    B2_CHECK_CUDA(cudaGetLastError());
    plan->done.add(bits);
    return 0;
}

int b200kv_encode_layers_finish(const b200kv_encode_plan_t* plan_in, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B2_REQUIRE(plan_in != nullptr, "plan is NULL");
    const EncPlan* plan = reinterpret_cast<const EncPlan*>(plan_in);
    B2_REQUIRE(plan->magic == kEncPlanMagic, "not a plan made by b200kv_encode_layers_plan");
    EncParams P = plan->P;
    B2_REQUIRE(plan->done == LayerSet::range(0, P.L), "a layer was never encoded");
    P.totals = P.ptotal;                   // headers carry the payload of every call
    finalize_kernel<<<(P.n_chunks + 127) / 128, 128, 0, stream>>>(P);
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// b200kv_decode_plan and b200kv_decode_plan_heads: src_head0 == NULL decodes every container whole (src_H = dst->H)
static int decode_plan_impl(const void* containers, int64_t containers_bytes, const int64_t* offsets,
                            const int64_t* total_bytes, const int32_t* ntokens, const int64_t* dst_tok, int32_t n_chunks,
                            int32_t max_dtype, int32_t coder, const b200kv_kv_desc* dst, const float* key_bins,
                            const float* value_bins, uint32_t* status_out, void* workspace, int64_t workspace_bytes,
                            b200kv_decode_plan_t* plan_out, cudaStream_t stream, int32_t src_H, const int32_t* src_head0,
                            const int32_t* dst_head0, const int32_t* n_heads) {
    B2_REQUIRE(plan_out != nullptr, "plan is NULL");
    DecPlan* plan = reinterpret_cast<DecPlan*>(plan_out);
    plan->magic = 0u;
    DecParams& P = plan->P;
    B2_REQUIRE(key_bins && value_bins, "bins are NULL");
    B2_REQUIRE(dst != nullptr, "destination descriptor is NULL");
    if (int rc = cachegen_dtype_ok(dst)) return rc;
    const bool latent = (coder & B200KV_KV_LATENT) != 0;
    coder &= ~B200KV_KV_LATENT;
    B2_REQUIRE(coder >= CODER_AC && coder <= CODER_RANS_COMPACT, "coder must be one of B200KV_CODER_*");
    B2_REQUIRE(!latent || coder == CODER_RANS_COMPACT, "B200KV_KV_LATENT names container version 4: rANS-compact only");
    B2_REQUIRE(latent == (kv_ppl(dst) == 1),
               latent ? "a version-4 (latent) container needs a latent destination (B200KV_KV_LATENT)"
                      : "a latent destination (B200KV_KV_LATENT) takes version-4 containers only");
    P.compact = coder == CODER_RANS_COMPACT ? 1 : 0;
    P.version = latent ? 4 : coder + 1;
    if (P.compact) coder = CODER_RANS;
    P.ppl = kv_ppl(dst);
    PlaneTable full;
    if (int rc = make_plane_table(dst, key_bins, value_bins, &full)) return rc;
    const int NP = P.ppl * dst->L;
    for (int nl = 0; nl < std::min(NP, kInlinePlanes); ++nl) {
        P.pt.p[nl] = full.p[nl];
        P.pt.maxq[nl] = full.maxq[nl];
    }
    P.gpt = nullptr;                         // set below, once every check has passed, when NP > kInlinePlanes
    B2_REQUIRE(containers && offsets && total_bytes && ntokens && dst_tok && n_chunks > 0, "bad chunk arrays");
    B2_REQUIRE(max_dtype == B200KV_DT_BF16 || max_dtype == B200KV_DT_FP16, "bad max_dtype");
    B2_REQUIRE(dst->sT > 0 && dst->sT < (1ll << 23), "destination token stride out of range");
    if (src_head0 == nullptr) src_H = dst->H;
    std::vector<HeadWindow> win;
    if (int rc = plan_head_windows(n_chunks, dst_tok, latent, dst->H, dst->D, src_H, src_head0, dst_head0, n_heads, CT,
                                   &win, &P.wtpp))
        return rc;
    P.sT = dst->sT; P.sH = dst->sH;
    P.slot_map = dst->slot_map;
    P.L = dst->L; P.H = src_H; P.D = dst->D; P.C = src_H * dst->D;
    P.out_dtype = kv_dtype(dst); P.max_dtype = max_dtype; P.n_chunks = n_chunks;
    P.tpp = tiles_per_plane(P.C);
    P.lb = 0; P.nlay = P.L;
    int tmax = 0;
    for (int j = 0; j < n_chunks; ++j) {
        B2_REQUIRE(ntokens[j] > 0, "ntokens must be positive");
        B2_REQUIRE(!P.compact || ntokens[j] <= kGroup, "a compact container holds at most 256 tokens");
        B2_REQUIRE((offsets[j] & 15) == 0, "container offsets must be 16-byte aligned");
        // the fixed sections are addressed from (L, H, D, ntokens); the buffer must hold them in full
        const Layout lj = make_layout(P.L, P.C, ntokens[j], P.compact, P.ppl);
        B2_REQUIRE(total_bytes[j] >= lj.off_payload && total_bytes[j] - lj.off_payload < (1ll << 32),
                   "container shorter than its fixed sections (truncated or corrupt)");
        B2_REQUIRE(offsets[j] >= 0 && offsets[j] + total_bytes[j] + B200KV_READ_SLACK <= containers_bytes,
                   "containers buffer must extend B200KV_READ_SLACK bytes past the end of every container");
        tmax = ntokens[j] > tmax ? ntokens[j] : tmax;
    }
    const int64_t Gmax = (tmax + kGroup - 1) / kGroup;
    const int64_t tiles_max = Gmax * NP * P.tpp;
    B2_REQUIRE(tiles_max < (1ll << 31) && n_chunks <= 65535, "too many tiles / chunks in one call");
    // table layout of the rANS decoder's 32-symbol planes (16-symbol planes always take the transposed table with its
    // LUT replica, decode_kernel): the conflict-free (transposed) one pays off above ~3.6 payload bits per symbol
    // (measured: row-major is faster at 0.6 bits, transposed at 4.1 bits); the containers say how
    // many bits they hold.  B200KV_DECODE_TABLE=rows|transposed overrides (measurement knob).
    bool transposed = false;
    {
        double bits = 0.0, syms = 0.0;
        for (int j = 0; j < n_chunks; ++j) {
            const Layout lj = make_layout(P.L, P.C, ntokens[j], P.compact, P.ppl);
            bits += 8.0 * (double)(total_bytes[j] - lj.off_payload);
            syms += (double)NP * (double)P.C * ntokens[j];
        }
        // a version-3 payload also carries the stream histograms: ~0.5 bits per symbol at that entropy
        transposed = bits > (P.compact ? 4.1 : 3.6) * syms && bits < 6.0 * syms;   // a slot bound instead of a size says nothing: rows
        if (const char* e = getenv("B200KV_DECODE_TABLE")) transposed = e[0] == 't';
    }
    P.tiles_max = (int32_t)tiles_max;
    size_t off_tb, off_pt;
    const size_t need = dec_ws_layout(tiles_max, n_chunks, NP, &off_tb, &off_pt);
    B2_REQUIRE(workspace != nullptr && workspace_bytes >= (int64_t)need, "workspace too small");
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    if (NP > kInlinePlanes) {           // the whole table, staged from pageable memory before the call returns
        B2_CHECK_CUDA(cudaMemcpyAsync(ws + off_pt, &full, sizeof(PlaneTable), cudaMemcpyHostToDevice, stream));
        P.gpt = reinterpret_cast<const PlaneTable*>(ws + off_pt);
    }
    // chunk descriptors: small pageable -> device copy (staged by the driver before the call returns)
    {
        DecChunk* hc = static_cast<DecChunk*>(malloc(sizeof(DecChunk) * (size_t)n_chunks));
        B2_REQUIRE(hc != nullptr, "out of host memory");
        for (int j = 0; j < n_chunks; ++j) {
            hc[j].base = static_cast<const uint8_t*>(containers) + offsets[j];
            hc[j].dst_tok = dst_tok[j];
            hc[j].t = ntokens[j];
            hc[j].ngroups = (ntokens[j] + kGroup - 1) / kGroup;
            const Layout lj = make_layout(P.L, P.C, ntokens[j], P.compact, P.ppl);
            hc[j].payload_bytes = (uint32_t)(total_bytes[j] - lj.off_payload);
            const HeadWindow& w = win[(size_t)j];
            hc[j].cw0 = w.cw0;
            hc[j].cw1 = w.cw1;
            hc[j].dshift = w.dshift;
            hc[j].ct0 = w.ct0;
            hc[j].ntw = w.ntw;
        }
        cudaError_t e = cudaMemcpyAsync(ws, hc, sizeof(DecChunk) * (size_t)n_chunks, cudaMemcpyHostToDevice, stream);
        free(hc);
        B2_CHECK_CUDA(e);
    }
    P.chunks = reinterpret_cast<const DecChunk*>(ws);
    P.tile_base = reinterpret_cast<unsigned long long*>(ws + off_tb);
    P.status = status_out;
    if (status_out) B2_CHECK_CUDA(cudaMemsetAsync(status_out, 0, sizeof(uint32_t) * (size_t)n_chunks, stream));

    dim3 gsum((unsigned)((tiles_max + 3) / 4), (unsigned)n_chunks);
    {
        ProfScope prof(kProfTileSum, stream);
        tile_sum_kernel<<<gsum, 128, 0, stream>>>(P);
    }
    B2_CHECK_CUDA(cudaGetLastError());
    {
        ProfScope prof(kProfTileScan, stream);
        tile_scan_kernel<<<(unsigned)n_chunks, 1024, 0, stream>>>(P);
    }
    B2_CHECK_CUDA(cudaGetLastError());
    plan->coder = coder;
    plan->transposed = transposed ? 1 : 0;
    plan->gmax = (int32_t)Gmax;
    plan->magic = kPlanMagic;
    return 0;
}

int b200kv_decode_plan(const void* containers, int64_t containers_bytes, const int64_t* offsets,
                       const int64_t* total_bytes, const int32_t* ntokens, const int64_t* dst_tok, int32_t n_chunks,
                       int32_t max_dtype, int32_t coder, const b200kv_kv_desc* dst, const float* key_bins,
                       const float* value_bins, uint32_t* status_out, void* workspace, int64_t workspace_bytes,
                       b200kv_decode_plan_t* plan_out, void* stream) {
    return decode_plan_impl(containers, containers_bytes, offsets, total_bytes, ntokens, dst_tok, n_chunks, max_dtype,
                            coder, dst, key_bins, value_bins, status_out, workspace, workspace_bytes, plan_out,
                            static_cast<cudaStream_t>(stream), 0, nullptr, nullptr, nullptr);
}

int b200kv_decode_plan_heads(const void* containers, int64_t containers_bytes, const int64_t* offsets,
                             const int64_t* total_bytes, const int32_t* ntokens, const int64_t* dst_tok, int32_t n_chunks,
                             int32_t max_dtype, int32_t coder, const b200kv_kv_desc* dst, const float* key_bins,
                             const float* value_bins, uint32_t* status_out, void* workspace, int64_t workspace_bytes,
                             b200kv_decode_plan_t* plan_out, void* stream, int32_t src_H, const int32_t* src_head0,
                             const int32_t* dst_head0, const int32_t* n_heads) {
    if (plan_out != nullptr) reinterpret_cast<DecPlan*>(plan_out)->magic = 0u;
    B2_REQUIRE(src_head0 != nullptr, "head window arrays are NULL");
    return decode_plan_impl(containers, containers_bytes, offsets, total_bytes, ntokens, dst_tok, n_chunks, max_dtype,
                            coder, dst, key_bins, value_bins, status_out, workspace, workspace_bytes, plan_out,
                            static_cast<cudaStream_t>(stream), src_H, src_head0, dst_head0, n_heads);
}

int b200kv_decode_layers(const b200kv_decode_plan_t* plan_in, int32_t layer_begin, int32_t layer_end, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B2_REQUIRE(plan_in != nullptr, "plan is NULL");
    const DecPlan* plan = reinterpret_cast<const DecPlan*>(plan_in);
    B2_REQUIRE(plan->magic == kPlanMagic, "not a plan made by b200kv_decode_plan");
    DecParams P = plan->P;
    B2_REQUIRE(layer_begin >= 0 && layer_begin < layer_end && layer_end <= P.L, "layer range out of range");
    P.lb = layer_begin;
    P.nlay = layer_end - layer_begin;
    const int coder = plan->coder;
    const bool transposed = plan->transposed != 0;
    const size_t smem = (size_t)(CT * kLp + kGroup + 32) * 4;
    dim3 grid((unsigned)((int64_t)plan->gmax * P.ppl * P.nlay * P.wtpp), (unsigned)P.n_chunks);
    ProfScope prof(kProfDecode, stream);
#define B2_LAUNCH_DEC2(DT, PAGED, CODER, TR, GT)                                                                       \
    do {                                                                                                               \
        B2_CHECK_CUDA(cudaFuncSetAttribute(decode_kernel<DT, PAGED, CODER, TR, GT>,                                    \
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                   \
        decode_kernel<DT, PAGED, CODER, TR, GT><<<grid, CT, smem, stream>>>(P);                                        \
    } while (0)
#define B2_LAUNCH_DEC1(DT, PAGED, CODER, TR)                                                                           \
    do {                                                                                                               \
        if (P.gpt != nullptr) B2_LAUNCH_DEC2(DT, PAGED, CODER, TR, true);                                              \
        else B2_LAUNCH_DEC2(DT, PAGED, CODER, TR, false);                                                              \
    } while (0)
#define B2_LAUNCH_DEC(DT, PAGED)                                                                                       \
    do {                                                                                                               \
        if (coder == CODER_RANS && transposed) B2_LAUNCH_DEC1(DT, PAGED, CODER_RANS, true);                            \
        else if (coder == CODER_RANS) B2_LAUNCH_DEC1(DT, PAGED, CODER_RANS, false);                                    \
        else B2_LAUNCH_DEC1(DT, PAGED, CODER_AC, false);                                                               \
    } while (0)
    if (P.out_dtype == B200KV_DT_BF16) { if (P.slot_map) B2_LAUNCH_DEC(0, true); else B2_LAUNCH_DEC(0, false); }
    else { if (P.slot_map) B2_LAUNCH_DEC(1, true); else B2_LAUNCH_DEC(1, false); }
#undef B2_LAUNCH_DEC
#undef B2_LAUNCH_DEC1
#undef B2_LAUNCH_DEC2
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int b200kv_decode_chunks(const void* containers, int64_t containers_bytes, const int64_t* offsets,
                         const int64_t* total_bytes, const int32_t* ntokens, const int64_t* dst_tok, int32_t n_chunks,
                         int32_t max_dtype,
                         int32_t coder, const b200kv_kv_desc* dst, const float* key_bins, const float* value_bins,
                         uint32_t* status_out, void* workspace, int64_t workspace_bytes, void* stream) {
    b200kv_decode_plan_t plan;
    if (int rc = b200kv_decode_plan(containers, containers_bytes, offsets, total_bytes, ntokens, dst_tok, n_chunks,
                                    max_dtype, coder, dst, key_bins, value_bins, status_out, workspace, workspace_bytes,
                                    &plan, stream))
        return rc;
    return b200kv_decode_layers(&plan, 0, dst->L, stream);
}

int b200kv_profile_enable(int32_t on) {
    g_prof_on = on != 0;
    for (int i = 0; i < kProfCount; ++i) g_prof_have[i] = false;
    return 0;
}

int b200kv_profile_last(float* ms, int32_t n) {
    B2_REQUIRE(ms != nullptr && n >= kProfCount, "need room for 7 floats");
    for (int i = 0; i < kProfCount; ++i) {
        ms[i] = -1.0f;
        if (g_prof_on && g_prof_have[i]) {
            B2_CHECK_CUDA(cudaEventSynchronize(g_prof_ev[i][1]));
            B2_CHECK_CUDA(cudaEventElapsedTime(&ms[i], g_prof_ev[i][0], g_prof_ev[i][1]));
        }
    }
    return kProfCount;
}

}  // extern "C"
