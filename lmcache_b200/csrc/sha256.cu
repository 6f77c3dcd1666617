// sha256.cu -- chunked token-id prefix hash on the GPU.
//
// Replaces LMCacheEngine._hash / _chunk_tokens / _prefix_hash (lmcache/cache_engine.py:58-96):
//     h_i = sha256( ascii_hex(h_{i-1}) || bytes(tokens[i*cs:(i+1)*cs]) ).hexdigest(),   h_{-1} = ""
// which costs the reference one tokens.cpu() device->host sync per chunk.  Here the whole chain runs on the
// caller's stream and only the 32-byte digests cross to the host (one copy, no per-chunk sync).
//
// A SHA-256 chain is serial by construction (Merkle-Damgard: every 64-byte block needs the previous state, and
// chunk i's first block is the previous digest), so one chain is latency-bound: 64 rounds x ~4 dependent
// operations per block.  The work is therefore split by what depends on the chain:
//   1. sha256_expand_kernel -- every block that holds only token bytes / padding is state-independent.  The hex
//      prefix is exactly 64 bytes = one block, so the token bytes of a chunk always start on a block boundary and
//      all blocks after the prefix block qualify.  One thread per block expands the message schedule and stores
//      (W + K)[0..63] (256 B per block) in a scratch buffer.  Fully parallel, ~45 % of the total work.
//   2. sha256_chain_kernel -- one thread per sequence walks its chunks: expands the one prefix block itself, then
//      streams the precomputed (W + K) blocks through 64 fully unrolled rounds with register renaming.
//      Independent sequences (batched requests, RAG chunk mixes) occupy the other lanes / warps.
#include <cuda_runtime.h>

#include <mutex>
#include <stdint.h>
#include <stdlib.h>

#include "common.cuh"

namespace b200kv {

__constant__ uint32_t kK[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
    0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
    0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
    0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
    0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
    0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
    0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};

__device__ __forceinline__ uint32_t rotr(uint32_t x, int n) { return __funnelshift_r(x, x, n); }

struct ShaParams {
    const uint8_t* tokens;
    const int64_t* seq_offsets;   // device, n_seq + 1 token indices
    const int64_t* seq_block0;    // device, n_seq + 1: first scratch block of each sequence
    const int64_t* seq_chunk0;    // device, n_seq + 1: first digest slot of each sequence
    uint32_t* scratch;            // [n_blocks][64]  (W + K)
    uint8_t* digests;
    uint32_t* ready;              // or NULL: ready[slot] = epoch once digest `slot` is visible (system scope)
    uint32_t epoch;
    int64_t n_blocks;
    int32_t n_seq, elem_size, chunk_size;
    int32_t blocks_per_full_chunk;   // ceil((chunk_size * elem_size + 9) / 64): tail blocks (tokens + padding) of a full chunk
};

// expand 16 message words into (W + K)[64]
__device__ __forceinline__ void expand_store(uint32_t (&w)[64], uint32_t* dst) {
#pragma unroll
    for (int i = 16; i < 64; ++i) {
        const uint32_t s0 = rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3);
        const uint32_t s1 = rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
        w[i] = w[i - 16] + s0 + w[i - 7] + s1;
    }
#pragma unroll
    for (int i = 0; i < 64; i += 4) {
        uint4 v = make_uint4(w[i] + kK[i], w[i + 1] + kK[i + 1], w[i + 2] + kK[i + 2], w[i + 3] + kK[i + 3]);
        *reinterpret_cast<uint4*>(dst + i) = v;
    }
}

// One thread per state-independent block.  Block b of sequence s: chunk ci = b / bpc (all chunks of a sequence but
// the last are full), k = block index inside the chunk's token+padding tail.
__global__ void __launch_bounds__(128) sha256_expand_kernel(ShaParams P) {
    const int64_t gb = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (gb >= P.n_blocks) return;
    // find the sequence (few sequences: linear / binary search over seq_block0)
    int lo = 0, hi = P.n_seq;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (P.seq_block0[mid] <= gb) lo = mid; else hi = mid;
    }
    const int s = lo;
    const int64_t b = gb - P.seq_block0[s];
    const int64_t t0 = P.seq_offsets[s], t1 = P.seq_offsets[s + 1];
    const int64_t ci = b / P.blocks_per_full_chunk;
    const int64_t k = b - ci * P.blocks_per_full_chunk;
    const int64_t tb = t0 + ci * P.chunk_size;
    const int64_t cnt = (t1 - tb) < P.chunk_size ? (t1 - tb) : P.chunk_size;
    const uint32_t nbytes = (uint32_t)(cnt * P.elem_size);            // token bytes of this chunk
    const uint32_t plen = ci == 0 ? 0u : 64u;
    const uint64_t bits = (uint64_t)(plen + nbytes) * 8ull;
    const uint32_t ntail = (nbytes + 9u + 63u) / 64u;                  // blocks in this chunk's tail
    if (cnt <= 0 || (uint32_t)k >= ntail) return;                      // slack slot of a ragged last chunk
    const uint8_t* tok = P.tokens + tb * P.elem_size;
    const bool word_ok = (reinterpret_cast<uintptr_t>(tok) & 3u) == 0u;
    uint32_t w[64];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const uint32_t o = (uint32_t)k * 64u + 4u * i;                 // byte offset inside the tail
        if (word_ok && o + 4u <= nbytes) {
            w[i] = __byte_perm(__ldg(reinterpret_cast<const uint32_t*>(tok + o)), 0u, 0x0123);
        } else {
            uint32_t v = 0u;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const uint32_t p = o + q;
                uint32_t byte = 0u;
                if (p < nbytes) byte = tok[p];
                else if (p == nbytes) byte = 0x80u;
                else if (p >= ntail * 64u - 8u) byte = (uint32_t)(bits >> (8u * (ntail * 64u - 1u - p))) & 0xffu;
                v = (v << 8) | byte;
            }
            w[i] = v;
        }
    }
    expand_store(w, P.scratch + gb * 64);
}

// 64 rounds over precomputed (W + K); state in registers, variables renamed instead of rotated.
// One chain is one thread, so the chain is bound by the latency of e -> Sigma1 -> t1 -> e', not by pipe throughput: all
// of it stays on the integer ALU pipe (three-input IADD3s).  Moving additions or rotations to the FMA pipe (IMADs)
// lengthened that dependency chain and was slower (DESIGN.md 3.5).
#define B2_SHA_ROUND(a, b, c, d, e, f, g, h, wk)                                                          \
    {                                                                                                      \
        const uint32_t s1_ = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25);                                       \
        const uint32_t ch_ = ((e) & (f)) ^ (~(e) & (g));                                                   \
        const uint32_t s0_ = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22);                                       \
        const uint32_t mj_ = ((a) & (b)) ^ ((a) & (c)) ^ ((b) & (c));                                      \
        const uint32_t t1_ = (h) + s1_ + ch_ + (wk);                                                       \
        (d) += t1_;                                                                                        \
        (h) = t1_ + s0_ + mj_;                                                                             \
    }

// 64 rounds over a block's (W + K) held in registers
__device__ __forceinline__ void compress_regs(uint32_t (&st)[8], const uint4 (&q)[16]) {
    uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
    for (int i = 0; i < 16; i += 2) {
        const uint4 x = q[i], y = q[i + 1];
        B2_SHA_ROUND(a, b, c, d, e, f, g, h, x.x)
        B2_SHA_ROUND(h, a, b, c, d, e, f, g, x.y)
        B2_SHA_ROUND(g, h, a, b, c, d, e, f, x.z)
        B2_SHA_ROUND(f, g, h, a, b, c, d, e, x.w)
        B2_SHA_ROUND(e, f, g, h, a, b, c, d, y.x)
        B2_SHA_ROUND(d, e, f, g, h, a, b, c, y.y)
        B2_SHA_ROUND(c, d, e, f, g, h, a, b, y.z)
        B2_SHA_ROUND(b, c, d, e, f, g, h, a, y.w)
    }
    st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

// ... and over a block staged in shared memory: slot[i * 32] is this lane's i-th 16-byte group
__device__ __forceinline__ void compress_smem(uint32_t (&st)[8], const uint4* slot) {
    uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
    for (int i = 0; i < 16; i += 2) {
        const uint4 x = slot[i * 32], y = slot[(i + 1) * 32];
        B2_SHA_ROUND(a, b, c, d, e, f, g, h, x.x)
        B2_SHA_ROUND(h, a, b, c, d, e, f, g, x.y)
        B2_SHA_ROUND(g, h, a, b, c, d, e, f, x.z)
        B2_SHA_ROUND(f, g, h, a, b, c, d, e, x.w)
        B2_SHA_ROUND(e, f, g, h, a, b, c, d, y.x)
        B2_SHA_ROUND(d, e, f, g, h, a, b, c, y.y)
        B2_SHA_ROUND(c, d, e, f, g, h, a, b, y.z)
        B2_SHA_ROUND(b, c, d, e, f, g, h, a, y.w)
    }
    st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

constexpr int kShaStages = 3;

// One thread per sequence (chain).  The precomputed (W + K) blocks of a chunk are streamed through a three-stage ring in
// shared memory with per-thread cp.async groups: block k + 2 is in flight while block k is consumed, so the chain never
// waits for L2 / DRAM (an earlier version kept the next block in registers; the compiler sank those loads to the point where
// the registers became free, late in the loop body, and the chain waited for them).
// The ring is lane-interleaved at 16-byte granularity: a warp's LDS.128 of "its" i-th group is one conflict-free request.
__global__ void __launch_bounds__(32) sha256_chain_kernel(ShaParams P) {
    __shared__ __align__(16) uint4 ring[kShaStages][16][32];
    const int lane = threadIdx.x;
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= P.n_seq) return;
    const int64_t t0 = P.seq_offsets[s], t1 = P.seq_offsets[s + 1];
    int64_t slot = P.seq_chunk0[s];
    int64_t gb = P.seq_block0[s];
    uint32_t dig[8];
    bool first = true;
    const uint32_t ring_a = (uint32_t)__cvta_generic_to_shared(&ring[0][0][lane]);
    for (int64_t tb = t0; tb < t1; tb += P.chunk_size, ++slot) {
        const int64_t cnt = (t1 - tb) < P.chunk_size ? (t1 - tb) : P.chunk_size;
        const uint32_t ntail = ((uint32_t)(cnt * P.elem_size) + 9u + 63u) / 64u;
        const uint4* wk4 = reinterpret_cast<const uint4*>(P.scratch + gb * 64);
        // block k of this chunk -> ring stage k % 3, as one cp.async group (an empty group when k is past the end keeps
        // the group arithmetic uniform)
        auto issue = [&](uint32_t k) {
            if (k < ntail) {
                const uint4* src = wk4 + 16 * (size_t)k;
                const uint32_t dst = ring_a + (k % kShaStages) * (16u * 32u * 16u);
#pragma unroll
                for (int i = 0; i < 16; ++i)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + (uint32_t)i * 512u), "l"(src + i) : "memory");
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        };
        issue(0);
        issue(1);
        uint32_t st[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au,
                          0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
        if (!first) {
            // prefix block: the 64 hex characters of the previous digest, 8 per state word (its rounds cover the latency
            // of the first two token blocks)
            uint32_t w[64];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
#pragma unroll
                for (int hw = 0; hw < 2; ++hw) {
                    uint32_t v = 0u;
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const uint32_t nib = (dig[i] >> (28 - 4 * (4 * hw + q))) & 15u;
                        v = (v << 8) | (nib < 10u ? 0x30u + nib : 0x57u + nib);      // '0'..'9', 'a'..'f'
                    }
                    w[2 * i + hw] = v;
                }
            }
            // expand in registers: (W + K) as 16 uint4
#pragma unroll
            for (int i = 16; i < 64; ++i) {
                const uint32_t s0 = rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3);
                const uint32_t s1 = rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
                w[i] = w[i - 16] + s0 + w[i - 7] + s1;
            }
            uint4 q[16];
#pragma unroll
            for (int i = 0; i < 16; ++i)
                q[i] = make_uint4(w[4 * i] + kK[4 * i], w[4 * i + 1] + kK[4 * i + 1], w[4 * i + 2] + kK[4 * i + 2],
                                  w[4 * i + 3] + kK[4 * i + 3]);
            compress_regs(st, q);
        }
#pragma unroll 1
        for (uint32_t k = 0; k < ntail; ++k) {
            asm volatile("cp.async.wait_group 1;" ::: "memory");          // all but the newest group: block k has landed
            issue(k + 2);                                                  // into the stage block k - 1 has just left
            compress_smem(st, &ring[k % kShaStages][0][lane]);
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        gb += P.blocks_per_full_chunk;      // scratch blocks are laid out at a fixed stride per chunk
        // big-endian words, eight 4-byte stores (the buffer is usually mapped host memory: every store is a PCIe write)
        uint32_t* out = reinterpret_cast<uint32_t*>(P.digests + slot * 32);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            dig[i] = st[i];
            out[i] = __byte_perm(st[i], 0u, 0x0123);
        }
        if (P.ready != nullptr) {
            // a host thread polls this word and then reads the digest: make the digest visible system-wide first
            __threadfence_system();
            *reinterpret_cast<volatile uint32_t*>(P.ready + slot) = P.epoch;
        }
        first = false;
    }
}

}  // namespace b200kv

using namespace b200kv;

extern "C" int b200kv_sha256_chain(const void* tokens, int32_t elem_size, const int64_t* seq_offsets, int32_t n_seq,
                                   int32_t chunk_size, void* digests, void* stream_) {
    return b200kv_sha256_chain_ready(tokens, elem_size, seq_offsets, n_seq, chunk_size, digests, nullptr, 0u, stream_);
}

extern "C" int b200kv_sha256_chain_ready(const void* tokens, int32_t elem_size, const int64_t* seq_offsets, int32_t n_seq,
                                         int32_t chunk_size, void* digests, uint32_t* ready, uint32_t epoch,
                                         void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B2_REQUIRE(seq_offsets != nullptr && n_seq > 0, "bad sequence table");
    B2_REQUIRE(elem_size == 1 || elem_size == 2 || elem_size == 4 || elem_size == 8, "elem_size must be 1/2/4/8");
    B2_REQUIRE(chunk_size > 0, "chunk_size must be positive");
    B2_REQUIRE((int64_t)chunk_size * elem_size < (1ll << 28), "chunk too large");
    const int64_t bpc = ((int64_t)chunk_size * elem_size + 9 + 63) / 64;
    // host tables: per sequence, first scratch block and first digest slot (chunks at a fixed block stride)
    int64_t* tab = static_cast<int64_t*>(malloc(sizeof(int64_t) * 3 * (size_t)(n_seq + 1)));
    B2_REQUIRE(tab != nullptr, "out of host memory");
    int64_t* h_off = tab;
    int64_t* h_blk = tab + (n_seq + 1);
    int64_t* h_chk = tab + 2 * (n_seq + 1);
    int64_t nchunks = 0;
    for (int s = 0; s <= n_seq; ++s) {
        h_off[s] = seq_offsets[s];
        h_blk[s] = nchunks * bpc;
        h_chk[s] = nchunks;
        if (s < n_seq) {
            if (seq_offsets[s + 1] < seq_offsets[s]) {
                free(tab);
                B2_REQUIRE(false, "seq_offsets must be non-decreasing");
            }
            nchunks += (seq_offsets[s + 1] - seq_offsets[s] + chunk_size - 1) / chunk_size;
        }
    }
    if (nchunks == 0) { free(tab); return 0; }
    if (tokens == nullptr || digests == nullptr) {
        free(tab);
        B2_REQUIRE(false, "NULL tokens / digests");
    }
    const int64_t n_blocks = nchunks * bpc;
    const size_t tab_bytes = sizeof(int64_t) * 3 * (size_t)(n_seq + 1);
    const size_t tab_pad = (tab_bytes + 255) & ~(size_t)255;
    // Scratch comes from a grow-only per-device buffer owned by the library, not from cudaMallocAsync: the default memory
    // pool hands its memory back to the driver at every synchronisation point (release threshold 0), so a per-call pool
    // allocation turned into a real allocation -- milliseconds or more once the process has gigabytes of mapped page-locked
    // memory -- on the critical path of every store() and retrieve().  Calls are ordered through an event, so
    // two streams can share the buffer.
    static std::mutex mu;
    static uint8_t* g_buf[64] = {nullptr};
    static size_t g_cap[64] = {0};
    static cudaEvent_t g_ev[64] = {nullptr};
    int devi = 0;
    B2_CHECK_CUDA(cudaGetDevice(&devi));
    if (devi < 0 || devi >= 64) devi = 0;
    std::lock_guard<std::mutex> lk(mu);
    const size_t need = tab_pad + (size_t)n_blocks * 256;
    if (g_ev[devi] == nullptr) {
        cudaError_t ee = cudaEventCreateWithFlags(&g_ev[devi], cudaEventDisableTiming);
        if (ee != cudaSuccess) { free(tab); B2_CHECK_CUDA(ee); }
    } else {
        cudaError_t ee = g_cap[devi] < need ? cudaEventSynchronize(g_ev[devi]) : cudaStreamWaitEvent(stream, g_ev[devi], 0);
        if (ee != cudaSuccess) { free(tab); B2_CHECK_CUDA(ee); }
    }
    if (g_cap[devi] < need) {
        if (g_buf[devi]) cudaFree(g_buf[devi]);
        g_buf[devi] = nullptr;
        g_cap[devi] = 0;
        const size_t cap = need < ((size_t)1 << 20) ? ((size_t)1 << 20) : need * 2;
        cudaError_t ee = cudaMalloc(&g_buf[devi], cap);
        if (ee != cudaSuccess) { free(tab); B2_CHECK_CUDA(ee); }
        g_cap[devi] = cap;
    }
    uint8_t* dmem = g_buf[devi];
    cudaError_t e = cudaMemcpyAsync(dmem, tab, tab_bytes, cudaMemcpyHostToDevice, stream);   // pageable: staged before return
    free(tab);
    B2_CHECK_CUDA(e);
    ShaParams P;
    P.tokens = static_cast<const uint8_t*>(tokens);
    P.seq_offsets = reinterpret_cast<const int64_t*>(dmem);
    P.seq_block0 = P.seq_offsets + (n_seq + 1);
    P.seq_chunk0 = P.seq_offsets + 2 * (n_seq + 1);
    P.scratch = reinterpret_cast<uint32_t*>(dmem + tab_pad);
    P.digests = static_cast<uint8_t*>(digests);
    P.ready = ready;
    P.epoch = epoch;
    P.n_blocks = n_blocks;
    P.n_seq = n_seq; P.elem_size = elem_size; P.chunk_size = chunk_size;
    P.blocks_per_full_chunk = (int32_t)bpc;
    sha256_expand_kernel<<<(unsigned)((n_blocks + 127) / 128), 128, 0, stream>>>(P);
    e = cudaGetLastError();
    if (e == cudaSuccess) {
        sha256_chain_kernel<<<(unsigned)((n_seq + 31) / 32), 32, 0, stream>>>(P);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaEventRecord(g_ev[devi], stream);
    B2_CHECK_CUDA(e);
    return 0;
}
