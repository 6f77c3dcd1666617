// mover.cu -- blob pack/unpack kernels and the GPU <-> pinned-host mover primitives.
//
// Replaces (reference paths relative to the LMCache v0.1.2 tree):
//   lmcache/cache_engine.py:98-118   _tuple_kv_to_blob    (3x torch.stack + permute)
//   lmcache/cache_engine.py:131-161  _slice_kv_at         (split + .contiguous() per chunk)
//   lmcache/cache_engine.py:362-368  retrieve-side torch.cat + _blob_to_tuple_kv
//   lmcache/storage_backend/local_backend.py:82-100,141-144  pageable .to("cpu") / .to("cuda") + device sync
// with ONE gather (store) / scatter (retrieve) pass between the engine's 2L KV tensors and the per-chunk
// blobs.  When the chunk buffer is pinned host memory mapped into the device address space, the same
// kernel is the device->host (or host->device) mover: the data crosses PCIe exactly once, as 16-byte
// coalesced accesses, with no intermediate device blob.
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include <vector>

#include "common.cuh"
#include "rope.cuh"

namespace b200kv {

struct PackParams {
    PlaneTable pt;
    int64_t sT, sH, tok_begin;
    const int64_t* slot_map;       // paged KV: token i lives in row slot_map[i]; NULL = row i
    int32_t L, H, D, n_chunks, chunk_tokens, last_chunk_tokens, hf_layout;
    int32_t ppl;                   // planes per layer: 2 (K, V) or 1 (latent KV: chunk blob [L, t, H*D])
    int32_t l0, nl;                // layers [l0, l0 + nl) move; a chunk holds only those, layer l0 first
    uint8_t* chunks;
    int64_t chunk_stride_bytes;
    uint8_t* const* table;         // TABLE: chunk j starts at table[j] (a device array) instead of chunks + j * stride
    // ROPE (b200kv_pack_chunks_rope): channels [rot_offset, rot_offset + 2 half) of the key planes of call token i turn
    // by table row seg_of_tok[i] of cs (-1: copied as they are); neox pairs (d, d + half), gptj (2d, 2d + 1)
    const int32_t* seg_of_tok;
    const float2* cs;
    int32_t half, rot_offset, neox;
};
static_assert(sizeof(PackParams) < kMaxParamBytes, "PackParams must stay under 4 KB of kernel parameters");

// One grid-stride loop over (chunk, plane, token, vector) units; VEC elements of type E per unit (one 16-byte vector,
// or one element).  vllm chunk layout [L,2,t,H,D]; huggingface [L,2,H,t,D]; a latent KV (ppl = 1) [L,t,H,D] -- of the
// nl layers of the range, whose local layer i is the KV's layer l0 + i.
// TABLE: the chunk pointers come from a device table the host never reads, so a vector instance checks each chunk's
// alignment itself and moves a misaligned chunk's vectors element by element (a layer slice is a multiple of 16 bytes
// whenever the vector path is taken, so the chunk pointer decides for all of its layers).
// ROPE (pack only, E a 16-bit float type, TABLE false): a key unit of a turned token turns its own VEC channels on the
// way, reading a neox partner vector from the same source row (rope_turn_vec); the launch rule takes the vector path
// only when no vector straddles the rotary range or its halves.
template <class E, int VEC, bool PACK, bool TABLE, bool ROPE = false>
__global__ void __launch_bounds__(256) pack_kernel(PackParams P) {
    using vec_t = typename std::conditional<VEC * sizeof(E) == 16, uint4, E>::type;
    const int NL = P.ppl * P.nl;
    const int vph = P.D / VEC;                 // vectors per head row
    const int64_t vpt = (int64_t)P.H * vph;    // vectors per token
    const int64_t per_chunk_full = (int64_t)NL * P.chunk_tokens * vpt;
    const int64_t total = (int64_t)(P.n_chunks - 1) * per_chunk_full + (int64_t)NL * P.last_chunk_tokens * vpt;
    for (int64_t u = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; u < total; u += (int64_t)gridDim.x * blockDim.x) {
        int64_t j = u / per_chunk_full;
        if (j >= P.n_chunks) j = P.n_chunks - 1;
        int64_t r = u - j * per_chunk_full;
        const int t = (j == P.n_chunks - 1) ? P.last_chunk_tokens : P.chunk_tokens;
        // r indexes [l][kv][tok][h][v] of the chunk (vllm order) -- map to plane kv*L + l0 + l
        const int64_t per_plane = (int64_t)t * vpt;
        const int lk = (int)(r / per_plane);       // l*ppl + kv, l local to the range
        r -= (int64_t)lk * per_plane;
        const int tok = (int)(r / vpt);
        r -= (int64_t)tok * vpt;
        const int h = (int)(r / vph);
        const int v = (int)(r - (int64_t)h * vph);
        const int l = P.l0 + (P.ppl == 2 ? lk >> 1 : lk), kv = P.ppl == 2 ? lk & 1 : 0;
        const E* plane = reinterpret_cast<const E*>(P.pt.p[kv * P.L + l]);
        int64_t row = P.tok_begin + j * P.chunk_tokens + tok;
        if (P.slot_map) row = __ldg(P.slot_map + row);       // consecutive threads share the token: broadcast, L1 hit
        const int64_t src_off = row * P.sT + (int64_t)h * P.sH + (int64_t)v * VEC;
        int64_t dst_off;   // in elements, inside the chunk
        if (P.hf_layout) dst_off = (((int64_t)lk * P.H + h) * t + tok) * P.D + (int64_t)v * VEC;
        else dst_off = (((int64_t)lk * t + tok) * P.H + h) * P.D + (int64_t)v * VEC;
        uint8_t* base;
        if (TABLE) base = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(P.table) + j));
        else base = P.chunks + j * P.chunk_stride_bytes;
        E* cptr = reinterpret_cast<E*>(base) + dst_off;
        if (TABLE && VEC > 1 && (reinterpret_cast<uintptr_t>(base) & 15) != 0) {
            E* kptr = const_cast<E*>(plane) + src_off;
#pragma unroll
            for (int e = 0; e < VEC; ++e) {
                if (PACK) cptr[e] = kptr[e];
                else kptr[e] = cptr[e];
            }
            continue;
        }
        if (ROPE && PACK) {
            union { vec_t q; E e[VEC]; } w;
            w.q = *reinterpret_cast<const vec_t*>(plane + src_off);
            const int seg = kv == 0 ? __ldg(P.seg_of_tok + j * P.chunk_tokens + tok) : -1;
            if (seg >= 0)
                rope_turn_vec<E, VEC>(w.e, plane + (src_off - (int64_t)v * VEC), v * VEC, P.cs + (int64_t)seg * P.half,
                                      P.half, P.rot_offset, P.neox != 0);
            *reinterpret_cast<vec_t*>(cptr) = w.q;
        } else if (PACK) {
            *reinterpret_cast<vec_t*>(cptr) = *reinterpret_cast<const vec_t*>(plane + src_off);
        } else {
            *reinterpret_cast<vec_t*>(const_cast<E*>(plane) + src_off) = *reinterpret_cast<const vec_t*>(cptr);
        }
    }
}

template <class E, bool TABLE>
static void launch_pack_kernel(bool pack, bool vec, unsigned blocks, const PackParams& P, cudaStream_t stream) {
    constexpr int V = 16 / sizeof(E);
    if (pack) {
        if (vec) pack_kernel<E, V, true, TABLE><<<blocks, 256, 0, stream>>>(P);
        else pack_kernel<E, 1, true, TABLE><<<blocks, 256, 0, stream>>>(P);
    } else {
        if (vec) pack_kernel<E, V, false, TABLE><<<blocks, 256, 0, stream>>>(P);
        else pack_kernel<E, 1, false, TABLE><<<blocks, 256, 0, stream>>>(P);
    }
}

template <class E>
static void launch_pack_rope_kernel(bool vec, unsigned blocks, const PackParams& P, cudaStream_t stream) {
    if (vec) pack_kernel<E, 16 / sizeof(E), true, false, true><<<blocks, 256, 0, stream>>>(P);
    else pack_kernel<E, 1, true, false, true><<<blocks, 256, 0, stream>>>(P);
}

// ---------------------------------------------------------------------------------------- split paged caches
// B200KV_KV_PAGED_SPLIT (vLLM's PagedAttention / xFormers layout): per layer a key block tensor [nb, H, D/x, bs, x] and a
// value block tensor [nb, H, D, bs] (x = 16 / es).  The chunk side is the vllm blob [nl, 2, t, H, D], as for rows.
//
// Work unit: one group of bs consecutive call tokens (slot-map indices [k*bs, k*bs + bs)) x one plane x hb heads.  A
// group whose tokens all lie in the moved range and in one chunk, and whose slots are b*bs + 0 .. bs-1, is a tile: the
// CTA moves it through shared memory (rows [hh][o][D] of `pitch` bytes), with coalesced accesses on both sides:
//   key:   the cache holds 16-byte vectors (x channels of one token) in [D/x][bs] order per head: a permutation of
//          vectors, read in cache order and written in chunk-row order;
//   value: the cache holds [D][bs] per head, a real transpose: vw-byte vectors along the tokens of one channel are
//          scattered into the rows, the rows leave as 16-byte vectors.
// Every other group (a call that starts mid-block, a scrambled slot map, ragged ends, a misaligned chunk) moves element
// by element in the same launch.
struct SplitParams {
    PlaneTable pt;                 // planes kv*L + l: layer l's key (kv 0) and value (kv 1) block tensors
    const int64_t* slot_map;
    uint8_t* chunks;
    int64_t chunk_stride_bytes;
    uint8_t* const* table;         // TABLE: chunk j starts at table[j]
    int64_t tok_begin, k0;         // first call token; first group
    int32_t n_groups, hb, nhb;     // groups; heads per unit; head blocks per group (H / hb)
    int32_t L, H, D, bs, n_chunks, chunk_tokens, last_chunk_tokens, l0, nl;
    int32_t vw;                    // bytes per value-side vector of the tile path (16 or 8); 0: element-wise only
    int32_t pitch;                 // shared-memory bytes per token row of one head: D * es + 16
    const int32_t* seg_of_tok;     // ROPE: as in PackParams, indexed by call token - tok_begin
    const float2* cs;
    int32_t half, rot_offset, neox;
};
static_assert(sizeof(SplitParams) < kMaxParamBytes, "SplitParams must stay under 4 KB of kernel parameters");

template <int W>
struct VecOf;
template <>
struct VecOf<16> { using T = uint4; };
template <>
struct VecOf<8> { using T = uint2; };

// value tile, cache side: W-byte vectors along the tokens of one channel <-> elements of the shared-memory rows
template <class E, int W, bool PACK>
__device__ __forceinline__ void split_value_tile(const SplitParams& P, E* cache, uint8_t* s) {
    using V = typename VecOf<W>::T;
    constexpr int VO = W / (int)sizeof(E);         // tokens per vector
    const int noc = P.bs / VO;                     // vectors per channel row of the cache
    const int nv = P.hb * P.D * noc;
    for (int i = threadIdx.x; i < nv; i += blockDim.x) {
        const int hh = i / (P.D * noc), r = i - hh * (P.D * noc);
        const int d = r / noc, oc = r - d * noc;
        E* srow = reinterpret_cast<E*>(s + (int64_t)(hh * P.bs + oc * VO) * P.pitch) + d;
        union { V v; E e[VO]; } u;
        if (PACK) {
            u.v = *reinterpret_cast<const V*>(cache + (int64_t)i * VO);
#pragma unroll
            for (int e = 0; e < VO; ++e) srow[(int64_t)e * P.pitch / (int)sizeof(E)] = u.e[e];
        } else {
#pragma unroll
            for (int e = 0; e < VO; ++e) u.e[e] = srow[(int64_t)e * P.pitch / (int)sizeof(E)];
            *reinterpret_cast<V*>(cache + (int64_t)i * VO) = u.v;
        }
    }
}

// ROPE (pack only, E a 16-bit float type, TABLE false): the tile path turns each key vector as it leaves the permuted
// shared-memory rows for the chunk (a neox partner is read from the same shared row), which takes a rotary range
// aligned to 16-byte vectors (the launch rule sends any other to the element-wise path); the element-wise path turns
// each key element it moves, reading its partner from the cache (a pack never writes the cache).
template <class E, bool PACK, bool TABLE, bool ROPE = false>
__global__ void __launch_bounds__(256) split_kernel(SplitParams P) {
    extern __shared__ __align__(16) uint8_t s_tile[];
    constexpr int X = 16 / (int)sizeof(E);         // elements per 16-byte vector: the key's x
    const int DX = P.D / X;
    const int64_t g_end = P.tok_begin + (int64_t)(P.n_chunks - 1) * P.chunk_tokens + P.last_chunk_tokens;
    const int64_t units = (int64_t)P.n_groups * 2 * P.nl * P.nhb;
    for (int64_t u = blockIdx.x; u < units; u += gridDim.x) {
        const int hbi = (int)(u % P.nhb);
        const int64_t r = u / P.nhb;
        const int64_t g0 = (P.k0 + r % P.n_groups) * P.bs;
        const int lk = (int)(r / P.n_groups);      // local layer * 2 + kv
        const int kv = lk & 1, h0 = hbi * P.hb;
        E* plane = const_cast<E*>(reinterpret_cast<const E*>(P.pt.p[kv * P.L + P.l0 + (lk >> 1)]));
        // tile test (uniform over the CTA until the slot check)
        bool tile = P.vw != 0 && g0 >= P.tok_begin && g0 + P.bs <= g_end;
        int64_t j = 0, blk = 0;
        int tok0 = 0, t = 0;
        uint8_t* base = nullptr;
        if (tile) {
            j = (g0 - P.tok_begin) / P.chunk_tokens;
            tok0 = (int)(g0 - P.tok_begin - j * P.chunk_tokens);
            t = j == P.n_chunks - 1 ? P.last_chunk_tokens : P.chunk_tokens;
            base = TABLE ? reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(P.table) + j))
                         : P.chunks + j * P.chunk_stride_bytes;
            tile = tok0 + P.bs <= t && (!TABLE || (reinterpret_cast<uintptr_t>(base) & 15) == 0);
        }
        if (tile) {
            const int64_t s0 = __ldg(P.slot_map + g0);
            blk = s0 / P.bs;
            bool ok = s0 % P.bs == 0;
            for (int o = threadIdx.x; o < P.bs; o += blockDim.x) ok = ok && __ldg(P.slot_map + g0 + o) == s0 + o;
            tile = __syncthreads_and(ok) != 0;
        }
        if (tile) {
            E* cache = plane + (blk * P.H + h0) * (int64_t)P.D * P.bs;     // heads h0 .. h0 + hb - 1: contiguous
            E* crow = reinterpret_cast<E*>(base) + (((int64_t)lk * t + tok0) * P.H + h0) * P.D;
            const int nv = P.hb * P.bs * DX;       // 16-byte vectors of the tile
            const int64_t HD = (int64_t)P.H * P.D;
            if (!PACK) {                           // chunk rows -> shared memory
                for (int i = threadIdx.x; i < nv; i += blockDim.x) {
                    const int o = i / (P.hb * DX), q = i - o * (P.hb * DX), hh = q / DX, dx = q - hh * DX;
                    *reinterpret_cast<uint4*>(s_tile + (int64_t)(hh * P.bs + o) * P.pitch + dx * 16) =
                        *reinterpret_cast<const uint4*>(crow + o * HD + (int64_t)hh * P.D + dx * X);
                }
                __syncthreads();
            }
            if (kv == 0) {                         // key: vector i of the cache = (hh, dx, o)
                for (int i = threadIdx.x; i < nv; i += blockDim.x) {
                    const int hh = i / (P.bs * DX), q = i - hh * (P.bs * DX), dx = q / P.bs, o = q - dx * P.bs;
                    uint4* sv = reinterpret_cast<uint4*>(s_tile + (int64_t)(hh * P.bs + o) * P.pitch + dx * 16);
                    uint4* cv = reinterpret_cast<uint4*>(cache + (int64_t)i * X);
                    if (PACK) *sv = *cv;
                    else *cv = *sv;
                }
            } else if (P.vw == 16) {
                split_value_tile<E, 16, PACK>(P, cache, s_tile);
            } else {
                split_value_tile<E, 8, PACK>(P, cache, s_tile);
            }
            if (PACK) {                            // shared memory -> chunk rows
                __syncthreads();
                for (int i = threadIdx.x; i < nv; i += blockDim.x) {
                    const int o = i / (P.hb * DX), q = i - o * (P.hb * DX), hh = q / DX, dx = q - hh * DX;
                    if (ROPE) {
                        const E* srow = reinterpret_cast<const E*>(s_tile + (int64_t)(hh * P.bs + o) * P.pitch);
                        union { uint4 q; E e[X]; } w;
                        w.q = *reinterpret_cast<const uint4*>(srow + dx * X);
                        const int seg = kv == 0 ? __ldg(P.seg_of_tok + (g0 + o - P.tok_begin)) : -1;
                        if (seg >= 0)
                            rope_turn_vec<E, X>(w.e, srow, dx * X, P.cs + (int64_t)seg * P.half, P.half, P.rot_offset,
                                                P.neox != 0);
                        *reinterpret_cast<uint4*>(crow + o * HD + (int64_t)hh * P.D + dx * X) = w.q;
                        continue;
                    }
                    *reinterpret_cast<uint4*>(crow + o * HD + (int64_t)hh * P.D + dx * X) =
                        *reinterpret_cast<const uint4*>(s_tile + (int64_t)(hh * P.bs + o) * P.pitch + dx * 16);
                }
            }
            __syncthreads();                       // the next unit reuses the shared rows
            continue;
        }
        // element-wise: every token of the group that the call moves, wherever its slot is
        const int ne = P.bs * P.hb * P.D;
        for (int i = threadIdx.x; i < ne; i += blockDim.x) {
            const int o = i / (P.hb * P.D), q = i - o * (P.hb * P.D), hh = q / P.D, d = q - hh * P.D;
            const int64_t g = g0 + o;
            if (g < P.tok_begin || g >= g_end) continue;
            const int64_t jj = (g - P.tok_begin) / P.chunk_tokens;
            const int tok = (int)(g - P.tok_begin - jj * P.chunk_tokens);
            const int tt = jj == P.n_chunks - 1 ? P.last_chunk_tokens : P.chunk_tokens;
            uint8_t* cb = TABLE ? reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(P.table) + jj))
                                : P.chunks + jj * P.chunk_stride_bytes;
            const int64_t s = __ldg(P.slot_map + g), b = s / P.bs, so = s - b * P.bs;
            const int h = h0 + hh;
            const int64_t coff = kv == 0 ? (((b * P.H + h) * DX + d / X) * P.bs + so) * X + d % X
                                         : ((b * P.H + h) * (int64_t)P.D + d) * P.bs + so;
            E* ce = reinterpret_cast<E*>(cb) + (((int64_t)lk * tt + tok) * P.H + h) * P.D + d;
            if (ROPE && PACK) {
                E e = plane[coff];
                const int c = d - P.rot_offset;
                const int seg = kv == 0 && c >= 0 && c < 2 * P.half ? __ldg(P.seg_of_tok + (g - P.tok_begin)) : -1;
                if (seg >= 0) {
                    const int pd = P.rot_offset + rope_partner(c, P.half, P.neox != 0);
                    const E p = plane[(((b * P.H + h) * DX + pd / X) * P.bs + so) * X + pd % X];
                    e = rope_turn_one(e, p, c, P.cs + (int64_t)seg * P.half, P.half, P.neox != 0);
                }
                *ce = e;
            } else if (PACK) {
                *ce = plane[coff];
            } else {
                plane[coff] = *ce;
            }
        }
    }
}

// b200kv_pack_chunks_rope's rotation: seg_of_tok per call token, the (cos, sin) table, the rotary channels and pairing
struct RopeArgs {
    const int32_t* seg_of_tok;
    const float* cos_sin;
    int32_t rotary_dim, offset, style;
    // 16-byte vectors can turn: no vector straddles the rotary range or (neox) its halves
    bool vec_ok(int ev) const { return offset % ev == 0 && (style == 0 ? (rotary_dim / 2) % ev : rotary_dim % ev) == 0; }
};

template <class P_t>
static void set_rope(P_t& P, const RopeArgs* rope) {
    P.seg_of_tok = rope ? rope->seg_of_tok : nullptr;
    P.cs = rope ? reinterpret_cast<const float2*>(rope->cos_sin) : nullptr;
    P.half = rope ? rope->rotary_dim / 2 : 0;
    P.rot_offset = rope ? rope->offset : 0;
    P.neox = rope ? rope->style == 0 : 0;
}

template <class E>
static int launch_split_rope_kernel(unsigned blocks, size_t smem, const SplitParams& P, cudaStream_t stream) {
    auto k = split_kernel<E, true, false, true>;
    if (smem > 48 * 1024) B2_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<blocks, 256, smem, stream>>>(P);
    return 0;
}

template <class E, bool TABLE>
static int launch_split_kernel(bool pack, unsigned blocks, size_t smem, const SplitParams& P, cudaStream_t stream) {
    auto k = pack ? split_kernel<E, true, TABLE> : split_kernel<E, false, TABLE>;
    if (smem > 48 * 1024) B2_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<blocks, 256, smem, stream>>>(P);
    return 0;
}

static int launch_split(bool pack, const b200kv_kv_desc* kv, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                        int32_t last_chunk_tokens, int32_t hf_layout, int32_t layer_begin, int32_t layer_end,
                        void* chunks, int64_t chunk_stride_bytes, void* const* table, cudaStream_t stream,
                        const RopeArgs* rope = nullptr) {
    B2_REQUIRE(kv->L > 0 && 2 * kv->L <= B200KV_MAX_PLANES, "bad kv descriptor");
    B2_REQUIRE(!(kv->dtype & B200KV_KV_LATENT), "a latent KV has no split layout (B200KV_KV_PAGED_SPLIT)");
    B2_REQUIRE(hf_layout == 0, "a split paged KV (B200KV_KV_PAGED_SPLIT) moves to and from vllm chunks only (hf_layout 0)");
    B2_REQUIRE(kv->slot_map != nullptr, "a split paged KV (B200KV_KV_PAGED_SPLIT) needs a slot_map");
    const int es = dtype_bytes(kv_split_dtype(kv));
    B2_REQUIRE(es != 0, "dtype must be one of B200KV_DT_*");
    B2_REQUIRE(kv->H > 0 && kv->D > 0 && kv->sT > 0, "H, D and the block size (sT) must be positive");
    B2_REQUIRE(kv->D % (16 / es) == 0, "a split paged KV needs D % x == 0 (x = 16 / element size)");
    B2_REQUIRE(tok_begin >= 0, "tok_begin must be >= 0");
    if (layer_end < 0) layer_end = kv->L;
    B2_REQUIRE(0 <= layer_begin && layer_begin < layer_end && layer_end <= kv->L, "bad layer range");
    B2_REQUIRE(n_chunks > 0 && chunk_tokens > 0 && last_chunk_tokens > 0 && last_chunk_tokens <= chunk_tokens,
               "bad chunking");
    B2_REQUIRE(table != nullptr || chunks != nullptr, "chunks is NULL");
    SplitParams P;
    b200kv_kv_desc rows = *kv;                 // the planes' pointers, read through the rows' table builder
    rows.dtype = kv_split_dtype(kv);
    float bins[B200KV_MAX_PLANES];
    for (int i = 0; i < B200KV_MAX_PLANES; ++i) bins[i] = 32.0f;
    if (int rc = make_plane_table(&rows, bins, bins, &P.pt)) return rc;
    P.l0 = layer_begin;
    P.nl = layer_end - layer_begin;
    const int64_t chunk_bytes = (int64_t)es * P.nl * 2 * chunk_tokens * kv->H * kv->D;
    B2_REQUIRE(table != nullptr || chunk_stride_bytes >= chunk_bytes || n_chunks == 1, "chunk_stride_bytes too small");
    P.slot_map = kv->slot_map;
    P.chunks = static_cast<uint8_t*>(chunks);
    P.chunk_stride_bytes = chunk_stride_bytes;
    P.table = reinterpret_cast<uint8_t* const*>(table);
    P.tok_begin = tok_begin;
    P.L = kv->L; P.H = kv->H; P.D = kv->D;
    B2_REQUIRE(kv->sT <= (1 << 20), "block size out of range");
    P.bs = (int32_t)kv->sT;
    P.n_chunks = n_chunks; P.chunk_tokens = chunk_tokens; P.last_chunk_tokens = last_chunk_tokens;
    const int64_t g_end = tok_begin + (int64_t)(n_chunks - 1) * chunk_tokens + last_chunk_tokens;
    P.k0 = tok_begin / P.bs;
    const int64_t n_groups = (g_end - 1) / P.bs - P.k0 + 1;
    B2_REQUIRE(n_groups < (1ll << 31), "too many tokens");
    P.n_groups = (int32_t)n_groups;
    // heads per unit: the most that keep a tile within 16 KB (at least one)
    const int64_t head_bytes = (int64_t)P.bs * P.D * es;
    P.hb = 1;
    for (int h = kv->H; h >= 1; --h)
        if (kv->H % h == 0 && h * head_bytes <= 16384) { P.hb = h; break; }
    P.nhb = kv->H / P.hb;
    P.pitch = P.D * es + 16;
    // the tile path: 16-byte aligned planes and chunks (a table's entries are checked by the kernel), a whole number of
    // 8- or 16-byte vectors per cache channel row, and a tile that fits in shared memory
    P.vw = (P.bs * es) % 16 == 0 ? 16 : (P.bs * es) % 8 == 0 ? 8 : 0;
    if (table == nullptr && (((reinterpret_cast<uintptr_t>(chunks) & 15) != 0) || chunk_stride_bytes % 16 != 0)) P.vw = 0;
    for (int kvi = 0; kvi < 2 && P.vw; ++kvi)
        for (int l = layer_begin; l < layer_end && P.vw; ++l)
            if ((reinterpret_cast<uintptr_t>(P.pt.p[kvi * P.L + l]) & 15) != 0) P.vw = 0;
    if (rope && !rope->vec_ok(16 / es)) P.vw = 0;     // the tile turns whole 16-byte vectors
    set_rope(P, rope);
    size_t smem = (size_t)P.hb * P.bs * P.pitch;
    if (smem > 200 * 1024) P.vw = 0;
    if (P.vw == 0) smem = 0;
    const int64_t units = n_groups * 2 * P.nl * P.nhb;
    int dev = 0, sms = 0;
    B2_CHECK_CUDA(cudaGetDevice(&dev));
    B2_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    int64_t blocks = std::min<int64_t>(units, (int64_t)sms * 8 * 4);
    if (blocks < 1) blocks = 1;
    int rc;
    if (rope) {
        if (kv_split_dtype(kv) == B200KV_DT_BF16) rc = launch_split_rope_kernel<__nv_bfloat16_raw>((unsigned)blocks, smem, P, stream);
        else rc = launch_split_rope_kernel<__half_raw>((unsigned)blocks, smem, P, stream);
    } else if (table != nullptr) {
        if (es == 2) rc = launch_split_kernel<uint16_t, true>(pack, (unsigned)blocks, smem, P, stream);
        else rc = launch_split_kernel<uint8_t, true>(pack, (unsigned)blocks, smem, P, stream);
    } else {
        if (es == 2) rc = launch_split_kernel<uint16_t, false>(pack, (unsigned)blocks, smem, P, stream);
        else rc = launch_split_kernel<uint8_t, false>(pack, (unsigned)blocks, smem, P, stream);
    }
    if (rc) return rc;
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// layer_end < 0: every layer.  table != NULL: chunk j starts at table[j] (chunks and chunk_stride_bytes unused).
// rope != NULL (pack, no table): b200kv_pack_chunks_rope, which has checked the rotation's arguments
static int launch_pack(bool pack, const b200kv_kv_desc* kv, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                       int32_t last_chunk_tokens, int32_t hf_layout, int32_t layer_begin, int32_t layer_end,
                       void* chunks, int64_t chunk_stride_bytes, void* const* table, cudaStream_t stream,
                       const RopeArgs* rope = nullptr) {
    PackParams P;
    B2_REQUIRE(kv != nullptr && kv->L > 0 && 2 * kv->L <= B200KV_MAX_PLANES, "bad kv descriptor");
    if (kv_split(kv))
        return launch_split(pack, kv, tok_begin, n_chunks, chunk_tokens, last_chunk_tokens, hf_layout, layer_begin,
                            layer_end, chunks, chunk_stride_bytes, table, stream, rope);
    if (layer_end < 0) layer_end = kv->L;
    B2_REQUIRE(0 <= layer_begin && layer_begin < layer_end && layer_end <= kv->L, "bad layer range");
    float bins[B200KV_MAX_PLANES];
    for (int i = 0; i < B200KV_MAX_PLANES; ++i) bins[i] = 32.0f;   // unused by pack/unpack; keeps the table valid
    if (int rc = make_plane_table(kv, bins, bins, &P.pt)) return rc;
    B2_REQUIRE(n_chunks > 0 && chunk_tokens > 0 && last_chunk_tokens > 0 && last_chunk_tokens <= chunk_tokens,
               "bad chunking");
    B2_REQUIRE(table != nullptr || chunks != nullptr, "chunks is NULL");
    P.ppl = kv_ppl(kv);
    P.l0 = layer_begin;
    P.nl = layer_end - layer_begin;
    const int es = kv_elem_bytes(kv);
    const int64_t chunk_bytes = (int64_t)es * P.nl * P.ppl * chunk_tokens * kv->H * kv->D;
    B2_REQUIRE(table != nullptr || chunk_stride_bytes >= chunk_bytes || n_chunks == 1, "chunk_stride_bytes too small");
    P.sT = kv->sT; P.sH = kv->sH; P.tok_begin = tok_begin;
    P.slot_map = kv->slot_map;
    P.L = kv->L; P.H = kv->H; P.D = kv->D;
    P.n_chunks = n_chunks; P.chunk_tokens = chunk_tokens; P.last_chunk_tokens = last_chunk_tokens;
    P.hf_layout = hf_layout;
    P.chunks = static_cast<uint8_t*>(chunks);
    P.chunk_stride_bytes = chunk_stride_bytes;
    P.table = reinterpret_cast<uint8_t* const*>(table);
    const int ev = 16 / es;                    // elements per 16-byte vector
    // a table's entries are checked by the kernel (they are in device memory)
    bool vec = (kv->D % ev == 0) && (kv->sT % ev == 0) && (kv->sH % ev == 0) &&
               (table != nullptr || (((reinterpret_cast<uintptr_t>(chunks) & 15) == 0) && (chunk_stride_bytes % 16 == 0)));
    for (int kvi = 0; kvi < P.ppl && vec; ++kvi)
        for (int l = layer_begin; l < layer_end && vec; ++l)
            vec = (reinterpret_cast<uintptr_t>(P.pt.p[kvi * P.L + l]) & 15) == 0;
    if (rope) vec = vec && rope->vec_ok(ev);
    set_rope(P, rope);
    const int V = vec ? ev : 1;
    const int64_t total = ((int64_t)(n_chunks - 1) * chunk_tokens + last_chunk_tokens) * P.ppl * P.nl * kv->H * (kv->D / V);
    int64_t blocks = (total + 255) / 256;
    int dev = 0, sms = 0;
    B2_CHECK_CUDA(cudaGetDevice(&dev));
    B2_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int64_t cap = (int64_t)sms * 8 * 4;   // a few waves of SMs x 8 CTAs; grid-stride covers the rest
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    if (rope) {
        if (kv_dtype(kv) == B200KV_DT_BF16) launch_pack_rope_kernel<__nv_bfloat16_raw>(vec, (unsigned)blocks, P, stream);
        else launch_pack_rope_kernel<__half_raw>(vec, (unsigned)blocks, P, stream);
    } else if (table != nullptr) {
        if (es == 2) launch_pack_kernel<uint16_t, true>(pack, vec, (unsigned)blocks, P, stream);
        else launch_pack_kernel<uint8_t, true>(pack, vec, (unsigned)blocks, P, stream);
    } else {
        if (es == 2) launch_pack_kernel<uint16_t, false>(pack, vec, (unsigned)blocks, P, stream);
        else launch_pack_kernel<uint8_t, false>(pack, vec, (unsigned)blocks, P, stream);
    }
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace b200kv

using namespace b200kv;

extern "C" {

int b200kv_pack_chunks(const b200kv_kv_desc* src, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                       int32_t last_chunk_tokens, int32_t hf_layout, void* chunks, int64_t chunk_stride_bytes,
                       void* stream) {
    return launch_pack(true, src, tok_begin, n_chunks, chunk_tokens, last_chunk_tokens, hf_layout, 0, -1, chunks,
                       chunk_stride_bytes, nullptr, static_cast<cudaStream_t>(stream));
}

int b200kv_pack_chunks_rope(const b200kv_kv_desc* src, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                            int32_t last_chunk_tokens, int32_t hf_layout, void* chunks, int64_t chunk_stride_bytes,
                            const int32_t* seg_of_tok, const float* cos_sin, int32_t rotary_dim, int32_t offset,
                            int32_t style, void* stream) {
    // b200kv_rope_shift's refusals; launch_pack makes b200kv_pack_chunks' own
    B2_REQUIRE(src != nullptr, "kv descriptor is NULL");
    B2_REQUIRE(cos_sin != nullptr, "cos_sin table is NULL");
    B2_REQUIRE(seg_of_tok != nullptr, "seg_of_tok is NULL");
    B2_REQUIRE(style == 0 || style == 1, "style must be 0 (neox) or 1 (gptj)");
    const int dt = kv_split(src) ? kv_split_dtype(src) : kv_dtype(src);
    B2_REQUIRE(dt == B200KV_DT_BF16 || dt == B200KV_DT_FP16,
               "the rope pack takes 16-bit keys only: rotating a one-byte (FP8) key would round it again");
    B2_REQUIRE(rotary_dim > 0 && rotary_dim % 2 == 0, "rotary_dim must be even and positive");
    B2_REQUIRE(offset >= 0 && (int64_t)offset + rotary_dim <= src->D, "offset + rotary_dim exceeds the head size D");
    const RopeArgs rope{seg_of_tok, cos_sin, rotary_dim, offset, style};
    return launch_pack(true, src, tok_begin, n_chunks, chunk_tokens, last_chunk_tokens, hf_layout, 0, -1, chunks,
                       chunk_stride_bytes, nullptr, static_cast<cudaStream_t>(stream), &rope);
}

int b200kv_unpack_chunks(const void* chunks, int64_t chunk_stride_bytes, int32_t n_chunks, int32_t chunk_tokens,
                         int32_t last_chunk_tokens, int32_t hf_layout, const b200kv_kv_desc* dst, int64_t tok_begin,
                         void* stream) {
    return launch_pack(false, dst, tok_begin, n_chunks, chunk_tokens, last_chunk_tokens, hf_layout, 0, -1,
                       const_cast<void*>(chunks), chunk_stride_bytes, nullptr, static_cast<cudaStream_t>(stream));
}

int b200kv_pack_chunks_layers(const b200kv_kv_desc* src, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                              int32_t last_chunk_tokens, int32_t hf_layout, int32_t layer_begin, int32_t layer_end,
                              void* const* chunk_ptrs, void* stream) {
    B2_REQUIRE(chunk_ptrs != nullptr, "chunk_ptrs is NULL");
    B2_REQUIRE(layer_end >= 0, "bad layer range");
    return launch_pack(true, src, tok_begin, n_chunks, chunk_tokens, last_chunk_tokens, hf_layout, layer_begin,
                       layer_end, nullptr, 0, chunk_ptrs, static_cast<cudaStream_t>(stream));
}

int b200kv_unpack_chunks_layers(const void* const* chunk_ptrs, int32_t n_chunks, int32_t chunk_tokens,
                                int32_t last_chunk_tokens, int32_t hf_layout, int32_t layer_begin, int32_t layer_end,
                                const b200kv_kv_desc* dst, int64_t tok_begin, void* stream) {
    B2_REQUIRE(chunk_ptrs != nullptr, "chunk_ptrs is NULL");
    B2_REQUIRE(layer_end >= 0, "bad layer range");
    return launch_pack(false, dst, tok_begin, n_chunks, chunk_tokens, last_chunk_tokens, hf_layout, layer_begin,
                       layer_end, nullptr, 0, const_cast<void* const*>(chunk_ptrs), static_cast<cudaStream_t>(stream));
}

int b200kv_pinned_alloc(void** host_ptr, int64_t bytes) {
    B2_REQUIRE(host_ptr != nullptr && bytes > 0, "bad pinned_alloc arguments");
    B2_CHECK_CUDA(cudaHostAlloc(host_ptr, (size_t)bytes, cudaHostAllocPortable | cudaHostAllocMapped));
    return 0;
}

int b200kv_pinned_free(void* host_ptr) {
    if (host_ptr) B2_CHECK_CUDA(cudaFreeHost(host_ptr));
    return 0;
}

int b200kv_host_device_ptr(void* host_ptr, void** device_ptr) {
    B2_REQUIRE(host_ptr != nullptr && device_ptr != nullptr, "NULL pointer");
    B2_CHECK_CUDA(cudaHostGetDevicePointer(device_ptr, host_ptr, 0));
    return 0;
}

int b200kv_copy_async(void* dst, const void* src, int64_t bytes, void* stream) {
    B2_REQUIRE(dst != nullptr && src != nullptr && bytes >= 0, "bad copy arguments");
    if (bytes == 0) return 0;
    B2_CHECK_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDefault, static_cast<cudaStream_t>(stream)));
    return 0;
}

int b200kv_copy2d_async(void* dst, int64_t dst_pitch, const void* src, int64_t src_pitch, int64_t row_bytes,
                        int64_t rows, void* stream) {
    B2_REQUIRE(dst != nullptr && src != nullptr && row_bytes >= 0 && rows >= 0, "bad copy2d arguments");
    if (row_bytes == 0 || rows == 0) return 0;
    B2_CHECK_CUDA(cudaMemcpy2DAsync(dst, (size_t)dst_pitch, src, (size_t)src_pitch, (size_t)row_bytes, (size_t)rows,
                                    cudaMemcpyDefault, static_cast<cudaStream_t>(stream)));
    return 0;
}

int b200kv_copy_batch_async(void* const* dsts, const void* const* srcs, const int64_t* sizes, int64_t n, void* stream) {
    B2_REQUIRE(n >= 0 && (n == 0 || (dsts != nullptr && srcs != nullptr && sizes != nullptr)), "bad batch copy arguments");
    std::vector<void*> d, s;
    std::vector<size_t> z;
    for (int64_t i = 0; i < n; ++i) {
        B2_REQUIRE(dsts[i] != nullptr && srcs[i] != nullptr && sizes[i] >= 0, "bad batch copy arguments");
        if (sizes[i] == 0) continue;
        d.push_back(dsts[i]);
        s.push_back(const_cast<void*>(srcs[i]));
        z.push_back((size_t)sizes[i]);
    }
    if (d.empty()) return 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // cudaMemcpyBatchAsync refuses the legacy default stream (NULL, e.g. torch's default stream) with "invalid argument":
    // there the copies go one call each
    if (st != nullptr && st != cudaStreamLegacy) {
        // one driver call for the whole batch: per-copy submission costs ~2 us of host time per copy, which is the copy
        // engine's time for a few hundred KB -- a layer of a layer-major upload is many copies of that size
        cudaMemcpyAttributes attr = {};
        attr.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
        attr.flags = cudaMemcpyFlagPreferOverlapWithCompute;
        size_t attr_idx = 0, fail_idx = 0;
        const cudaError_t e = cudaMemcpyBatchAsync(d.data(), s.data(), z.data(), d.size(), &attr, &attr_idx, 1, &fail_idx,
                                                   st);
        // a driver older than the runtime (CUDA < 12.8) answers cudaErrorCallRequiresNewerDriver, a device or stream that
        // cannot take the batch cudaErrorNotSupported: then the same copies, one call each
        if (e != cudaErrorNotSupported && e != cudaErrorCallRequiresNewerDriver) {
            B2_CHECK_CUDA(e);
            return 0;
        }
        (void)cudaGetLastError();
    }
    for (size_t i = 0; i < d.size(); ++i) B2_CHECK_CUDA(cudaMemcpyAsync(d[i], s[i], z[i], cudaMemcpyDefault, st));
    return 0;
}

int b200kv_stream_create(void** stream) {
    B2_REQUIRE(stream != nullptr, "NULL pointer");
    cudaStream_t s;
    B2_CHECK_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    *stream = s;
    return 0;
}
int b200kv_stream_destroy(void* stream) {
    if (stream) B2_CHECK_CUDA(cudaStreamDestroy(static_cast<cudaStream_t>(stream)));
    return 0;
}
int b200kv_stream_sync(void* stream) {
    B2_CHECK_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
    return 0;
}
int b200kv_event_create(void** event) {
    B2_REQUIRE(event != nullptr, "NULL pointer");
    cudaEvent_t e;
    B2_CHECK_CUDA(cudaEventCreate(&e));
    *event = e;
    return 0;
}
int b200kv_event_destroy(void* event) {
    if (event) B2_CHECK_CUDA(cudaEventDestroy(static_cast<cudaEvent_t>(event)));
    return 0;
}
int b200kv_event_record(void* event, void* stream) {
    B2_CHECK_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(event), static_cast<cudaStream_t>(stream)));
    return 0;
}
int b200kv_event_query(void* event) {
    cudaError_t e = cudaEventQuery(static_cast<cudaEvent_t>(event));
    if (e == cudaSuccess) return 0;
    if (e == cudaErrorNotReady) return 1;
    set_error(std::string("cudaEventQuery: ") + cudaGetErrorString(e));
    return -1;
}
int b200kv_event_sync(void* event) {
    B2_CHECK_CUDA(cudaEventSynchronize(static_cast<cudaEvent_t>(event)));
    return 0;
}
int b200kv_stream_wait_event(void* stream, void* event) {
    B2_CHECK_CUDA(cudaStreamWaitEvent(static_cast<cudaStream_t>(stream), static_cast<cudaEvent_t>(event), 0));
    return 0;
}
int b200kv_event_elapsed_ms(void* start, void* stop, float* ms) {
    B2_REQUIRE(ms != nullptr, "NULL pointer");
    B2_CHECK_CUDA(cudaEventElapsedTime(ms, static_cast<cudaEvent_t>(start), static_cast<cudaEvent_t>(stop)));
    return 0;
}

int b200kv_version(void) { return B200KV_VERSION; }

int b200kv_device_count(void) {
    int n = 0;
    B2_CHECK_CUDA(cudaGetDeviceCount(&n));
    return n;
}

}  // extern "C"

namespace b200kv {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
}  // namespace b200kv

extern "C" const char* b200kv_last_error(void) { return b200kv::g_last_error.c_str(); }
