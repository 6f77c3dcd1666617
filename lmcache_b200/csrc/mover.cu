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
};
static_assert(sizeof(PackParams) < kMaxParamBytes, "PackParams must stay under 4 KB of kernel parameters");

// One grid-stride loop over (chunk, plane, token, vector) units; VEC elements of type E per unit (one 16-byte vector,
// or one element).  vllm chunk layout [L,2,t,H,D]; huggingface [L,2,H,t,D]; a latent KV (ppl = 1) [L,t,H,D] -- of the
// nl layers of the range, whose local layer i is the KV's layer l0 + i.
// TABLE: the chunk pointers come from a device table the host never reads, so a vector instance checks each chunk's
// alignment itself and moves a misaligned chunk's vectors element by element (a layer slice is a multiple of 16 bytes
// whenever the vector path is taken, so the chunk pointer decides for all of its layers).
template <class E, int VEC, bool PACK, bool TABLE>
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
        if (PACK) *reinterpret_cast<vec_t*>(cptr) = *reinterpret_cast<const vec_t*>(plane + src_off);
        else *reinterpret_cast<vec_t*>(const_cast<E*>(plane) + src_off) = *reinterpret_cast<const vec_t*>(cptr);
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

// layer_end < 0: every layer.  table != NULL: chunk j starts at table[j] (chunks and chunk_stride_bytes unused).
static int launch_pack(bool pack, const b200kv_kv_desc* kv, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                       int32_t last_chunk_tokens, int32_t hf_layout, int32_t layer_begin, int32_t layer_end,
                       void* chunks, int64_t chunk_stride_bytes, void* const* table, cudaStream_t stream) {
    PackParams P;
    B2_REQUIRE(kv != nullptr && kv->L > 0 && 2 * kv->L <= B200KV_MAX_PLANES, "bad kv descriptor");
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
    const int V = vec ? ev : 1;
    const int64_t total = ((int64_t)(n_chunks - 1) * chunk_tokens + last_chunk_tokens) * P.ppl * P.nl * kv->H * (kv->D / V);
    int64_t blocks = (total + 255) / 256;
    int dev = 0, sms = 0;
    B2_CHECK_CUDA(cudaGetDevice(&dev));
    B2_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int64_t cap = (int64_t)sms * 8 * 4;   // a few waves of SMs x 8 CTAs; grid-stride covers the rest
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    if (table != nullptr) {
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
