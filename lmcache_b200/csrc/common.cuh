// common.cuh -- error plumbing and small device helpers shared by the libb200kv translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/b200kv.h"

namespace b200kv {

void set_error(const std::string& msg);   // thread-local last error (api.cu)

#define B2_CHECK_CUDA(expr)                                                                      \
    do {                                                                                         \
        cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess) {                                                                 \
            ::b200kv::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));             \
            return -1;                                                                           \
        }                                                                                        \
    } while (0)

#define B2_REQUIRE(cond, msg)                                                                    \
    do {                                                                                         \
        if (!(cond)) {                                                                           \
            ::b200kv::set_error(std::string("invalid argument: ") + (msg));                      \
            return -2;                                                                           \
        }                                                                                        \
    } while (0)

// Kernel-parameter copy of the per-plane base pointers and quantiser constants
// (plane nl = kv * L + l).  Lives in the constant bank; indexed dynamically.  3 KB at 256 planes: every parameter block
// that holds one stays under the classic 4 KB kernel-parameter limit (static_asserts next to each).
template <int N>
struct PlaneTableT {
    const uint16_t* p[N];                // first element of the plane; one-byte elements: read it as a uint8_t*
    float maxq[N];                       // bins // 2 - 1
};
using PlaneTable = PlaneTableT<B200KV_MAX_PLANES>;
constexpr size_t kMaxParamBytes = 4096;

// Planes per layer of a kv_desc (1 for a latent KV, B200KV_KV_LATENT) and its element dtype without the latent flag.
// The split flag (B200KV_KV_PAGED_SPLIT) is kept in kv_dtype on purpose: dtype_bytes of it is 0, so no entry point can
// read a split descriptor as rows; the mover, the only one that takes it, clears it with kv_split_dtype.
inline int kv_ppl(const b200kv_kv_desc* kv) { return (kv->dtype & B200KV_KV_LATENT) ? 1 : 2; }
inline int kv_dtype(const b200kv_kv_desc* kv) { return kv->dtype & ~B200KV_KV_LATENT; }
inline bool kv_split(const b200kv_kv_desc* kv) { return (kv->dtype & B200KV_KV_PAGED_SPLIT) != 0; }
inline int kv_split_dtype(const b200kv_kv_desc* kv) { return kv->dtype & ~B200KV_KV_PAGED_SPLIT; }
#define B2_SPLIT_REFUSED                                                                                             \
    "a split paged descriptor (B200KV_KV_PAGED_SPLIT) is taken by the pack / unpack calls only: stage it into a "  \
    "blob with b200kv_pack_chunks first"
// Bytes per element of a B200KV_DT_* code (without the latent flag), 0 for an unknown code.
inline int dtype_bytes(int dt) {
    return dt == B200KV_DT_BF16 || dt == B200KV_DT_FP16 ? 2
           : dt == B200KV_DT_U8 || dt == B200KV_DT_FP8_E4M3 || dt == B200KV_DT_FP8_E5M2 ? 1 : 0;
}
inline int kv_elem_bytes(const b200kv_kv_desc* kv) { return dtype_bytes(kv_dtype(kv)); }

// Fill a PlaneTable from a kv_desc + bins (planes kv * L + l; a latent KV's plane l takes key_bins[l]); returns 0 or <0
// with error set.  Takes every dtype of dtype_bytes: the CacheGen entry points refuse the one-byte ones themselves.
int make_plane_table(const b200kv_kv_desc* kv, const float* key_bins, const float* value_bins, PlaneTable* out);

// Row of a token inside its plane.  PAGED: the caller's slot mapping (vLLM's paged KV cache: row = block * block_size
// + offset); every lane of a warp asks for the same token, so the lookup is one broadcast load that hits L1.
template <bool PAGED>
__device__ __forceinline__ int64_t tok_row(const int64_t* slot_map, int64_t tok) {
    if constexpr (PAGED) return __ldg(slot_map + tok);
    else return tok;
}

// The head window of one container in a decode plan (b200kv_decode_plan_heads, b200kv_lossless_decode_plan_heads; the
// whole container otherwise): container channels [cw0, cw1) are decoded into destination channel c + dshift; they lie in
// tiles [ct0, ct0 + ntw) of CT channels of every plane.
struct HeadWindow {
    int32_t ct0, ntw, cw0, cw1, dshift;
};

// The head windows of a decode plan's n_chunks containers of src_H heads of D channels, and in *wtpp the largest ntw
// (the tiles a decode launches per plane).  With src_head0 != NULL, container j's heads [src_head0[j], src_head0[j] +
// n_heads[j]) land in the destination's heads from dst_head0[j] on.  Refused (nothing written): a latent destination
// (no heads to split), NULL window arrays, src_H out of range, an empty window, one outside the container's heads or
// the destination's dst_H heads, and two containers at one destination token that share a destination head.
// src_head0 == NULL: every container whole, [0, src_H * D) with no shift.  Returns 0, or -2 with the error set.
inline int plan_head_windows(int32_t n_chunks, const int64_t* dst_tok, bool latent, int32_t dst_H, int32_t D,
                             int32_t src_H, const int32_t* src_head0, const int32_t* dst_head0, const int32_t* n_heads,
                             int CT, std::vector<HeadWindow>* win, int32_t* wtpp) {
    const bool windows = src_head0 != nullptr;
    B2_REQUIRE(!windows || !latent, "head windows need a (K, V) destination: a latent KV has no heads to split");
    if (windows) {
        B2_REQUIRE(dst_head0 != nullptr && n_heads != nullptr, "head window arrays are NULL");
        B2_REQUIRE(src_H > 0 && (int64_t)src_H * D < (1ll << 24), "src_H out of range");
        for (int j = 0; j < n_chunks; ++j) {
            B2_REQUIRE(n_heads[j] >= 1, "a head window must hold at least one head");
            B2_REQUIRE(src_head0[j] >= 0 && src_head0[j] <= src_H - n_heads[j], "head window outside the container's heads");
            B2_REQUIRE(dst_head0[j] >= 0 && dst_head0[j] <= dst_H - n_heads[j],
                       "head window outside the destination's heads");
        }
        // containers that share a destination token must not share a destination head
        std::vector<int> ord((size_t)n_chunks);
        for (int j = 0; j < n_chunks; ++j) ord[(size_t)j] = j;
        std::sort(ord.begin(), ord.end(), [&](int a, int b) {
            return dst_tok[a] != dst_tok[b] ? dst_tok[a] < dst_tok[b] : dst_head0[a] < dst_head0[b];
        });
        for (size_t k = 1; k < ord.size(); ++k) {
            const int a = ord[k - 1], b = ord[k];
            B2_REQUIRE(dst_tok[a] != dst_tok[b] || dst_head0[a] + n_heads[a] <= dst_head0[b],
                       "head windows overlap at the same destination token");
        }
    }
    win->resize((size_t)n_chunks);
    int32_t wt = windows ? 1 : (int32_t)(((int64_t)src_H * D + CT - 1) / CT);
    for (int j = 0; j < n_chunks; ++j) {
        HeadWindow& w = (*win)[(size_t)j];
        w.cw0 = windows ? src_head0[j] * D : 0;
        w.cw1 = windows ? (src_head0[j] + n_heads[j]) * D : src_H * D;
        w.dshift = windows ? (dst_head0[j] - src_head0[j]) * D : 0;
        w.ct0 = w.cw0 / CT;
        w.ntw = (w.cw1 - 1) / CT - w.ct0 + 1;
        wt = std::max(wt, w.ntw);
    }
    *wtpp = wt;
    return 0;
}

// A set of layers [0, B200KV_MAX_PLANES / 2): bit l % 64 of word l / 64.  The layer-wise encode plans (CacheGen and
// lossless) record in one the layers encoded so far.
struct LayerSet {
    static constexpr int kWords = B200KV_MAX_PLANES / 2 / 64;
    uint64_t w[kWords];
    // layers [a, b), 0 <= a <= b <= kWords * 64
    static LayerSet range(int a, int b) {
        LayerSet s;
        for (int i = 0; i < kWords; ++i) {
            const int lo = a - 64 * i > 0 ? a - 64 * i : 0, hi = b - 64 * i < 64 ? b - 64 * i : 64;   // inside word i
            s.w[i] = lo >= hi ? 0ull : (hi - lo == 64 ? ~0ull : ((1ull << (hi - lo)) - 1ull) << lo);
        }
        return s;
    }
    bool intersects(const LayerSet& o) const {
        uint64_t x = 0ull;
        for (int i = 0; i < kWords; ++i) x |= w[i] & o.w[i];
        return x != 0ull;
    }
    bool operator==(const LayerSet& o) const {
        for (int i = 0; i < kWords; ++i)
            if (w[i] != o.w[i]) return false;
        return true;
    }
    void add(const LayerSet& o) {
        for (int i = 0; i < kWords; ++i) w[i] |= o.w[i];
    }
    int count() const {
        int n = 0;
        for (int i = 0; i < kWords; ++i) n += __builtin_popcountll(w[i]);
        return n;
    }
};
static_assert(LayerSet::kWords * 64 == B200KV_MAX_PLANES / 2, "one bit per layer");

// The arena rule of the layer-wise stores (place_kernel in codec.cu, ll_place_kernel in lossless.cu; its host
// statement is pipeline.arena_placement).  After a call's encode, chunk i's bytes of the call, seg_bytes[i], get room
// in the arena in chunk order from the device-held cursor, 16-byte aligned.  Chunk i fits iff every chunk before it
// fits and the arena still holds, after chunks 0..i of this call, the layers still to come for them at this call's size
// per layer (layers_left / nlay times this call's bytes of chunks 0..i): without that reserve the first calls would
// fill the arena with every chunk and a later call would find no room even for chunk 0.  The first chunk that does not
// fit is remembered (fail_from), so the chunks that fit are always a prefix, over this call and every later one.
// chunk_base[i] gets the arena offset, or ~0 with bit 16 OR-ed into err[i].  One CTA of 1024 threads, every thread
// calls it; on return chunk_base is visible to the whole CTA.
__device__ __forceinline__ void arena_place(int n_chunks, const unsigned long long* seg_bytes, int layers_left, int nlay,
                                            int64_t arena_bytes, unsigned long long* cursor, unsigned int* fail_from,
                                            unsigned long long* chunk_base, unsigned int* err) {
    __shared__ unsigned long long s_w[32];
    __shared__ unsigned long long s_carry, s_end;
    __shared__ unsigned int s_fail;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) {
        s_carry = s_end = *cursor;
        s_fail = *fail_from;
    }
    __syncthreads();
    const unsigned long long start = s_carry;
    for (int b0 = 0; b0 < n_chunks; b0 += 1024) {
        const int i = b0 + tid;
        const unsigned long long v = i < n_chunks ? (seg_bytes[i] + 15ull) & ~15ull : 0ull;
        unsigned long long inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long n = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += n;
        }
        if (lane == 31) s_w[wid] = inc;
        const unsigned int fail0 = s_fail;
        const unsigned long long carry = s_carry;
        __syncthreads();
        unsigned long long wbase = 0ull;
        for (int w = 0; w < wid; ++w) wbase += s_w[w];
        const unsigned long long end = carry + wbase + inc;
        if (i < n_chunks) {
            const unsigned long long reserve = (end - start) * (unsigned long long)layers_left / (unsigned)nlay;
            const bool fits = (unsigned)i < fail0 && end + reserve <= (unsigned long long)arena_bytes;
            chunk_base[i] = fits ? end - v : ~0ull;
            if (fits) {
                atomicMax(&s_end, end);
            } else {
                atomicOr(&err[i], 16u);
                atomicMin(&s_fail, (unsigned)i);
            }
        }
        __syncthreads();
        if (tid == 0) s_carry = s_end;
        __syncthreads();
    }
    if (tid == 0) {
        *cursor = s_carry;
        *fail_from = s_fail;
    }
}

}  // namespace b200kv
