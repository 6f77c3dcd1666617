// blend.cu -- the cache side of CacheBlend's selective recomputation: how far the model's fresh keys of a layer are from
// the cached key rows of that layer, and which tokens to recompute from there on.
//
// A reused document's KV at layers >= 1 was computed without attending to what now precedes it.  CacheBlend recomputes
// the share of the reused tokens whose cached KV deviates most from a fresh computation.  The model computes the fresh
// keys; these two kernels give the choice, identical on every tensor-parallel rank:
//
//   b200kv_blend_deviation: dev[i] = sum over (h, c) of (fresh - cached)^2 in fp32, for the key plane of one layer, in
//                      every layout a kv_desc carries.  The order of that sum depends on (H, D) only -- not on the
//                      layout, n, i, the alignment or the launch -- so the same rows give the same bits everywhere, and
//                      ranks that all-reduce their partial sums get the same totals.
//   b200kv_blend_select: the forced rows (cand == 0) in row order, then the k candidates of largest dev in row order;
//                      ties go to the lower row, NaN ranks as +inf.  A radix select on the keys' bit patterns in a
//                      fixed number of launches, with no host sync and no atomic whose order shows in the result.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "rope.cuh"     // to_f: the exact widening of a 16-bit element to fp32

namespace b200kv {

// ---------------------------------------------------------------------------------------------- deviation
struct BlendDevParams {
    const void* plane;             // the key plane of the layer (the latent plane of a latent KV)
    const int64_t* slot_map;       // NULL: row = view token
    const int64_t* tok;            // [n] view token of fresh row i
    const void* fresh;             // [n] rows of fresh_stride elements
    float* dev;                    // [n]
    int64_t n, fresh_stride, sT, sH;
    int32_t H, D, bs;              // bs: the split layout's block size
};

// Element offset of channel d (d % 8 == 0 when a vector is read there) of head h in cache row `row` of the key plane.
// SPLIT: key blocks [nb, H, D/8, bs, 8] (x = 8 for 16-bit elements); rows: row * sT + h * sH + d.
template <bool SPLIT>
__device__ __forceinline__ int64_t dev_key_off(const BlendDevParams& P, int64_t row, int h, int d) {
    if (SPLIT) {
        const int64_t b = row / P.bs, o = row - b * P.bs;
        return (((b * P.H + h) * (P.D / 8) + d / 8) * P.bs + o) * 8 + d % 8;
    }
    return row * P.sT + (int64_t)h * P.sH + d;
}

// Element `hi` (0: low half) of a 32-bit word holding two 16-bit elements
template <class E>
__device__ __forceinline__ E elem(uint32_t w, int hi) {
    E e;
    e.x = (unsigned short)(hi ? w >> 16 : w & 0xffffu);
    return e;
}

// The summation order, the same for every instantiation: channel c of the H*D of a row (c = h * D + d) belongs to lane
// (c / 8) % 32 of the row's warp; a lane adds its channels in ascending order, (f - k)^2 by one fma each; the 32 lane sums
// are folded by the xor butterfly 16, 8, 4, 2, 1 (every lane ends with the same bits, as a + b == b + a).  VEC reads the
// 8 channels of a group as one 16-byte vector (D % 8 == 0, aligned strides and pointers); otherwise element by element.
template <class E, bool VEC, bool SPLIT>
__global__ void __launch_bounds__(256) blend_dev_kernel(BlendDevParams P) {
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int C = P.H * P.D, ng = (C + 7) / 8;
    const E* plane = reinterpret_cast<const E*>(P.plane);
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < P.n; i += nw) {
        const int64_t t = __ldg(P.tok + i);
        const int64_t row = P.slot_map ? __ldg(P.slot_map + t) : t;
        const E* f = reinterpret_cast<const E*>(P.fresh) + i * P.fresh_stride;
        float acc = 0.0f;
        for (int g = lane; g < ng; g += 32) {
            const int c0 = g * 8;
            if (VEC) {
                const int h = c0 / P.D, d = c0 - h * P.D;
                const uint4 a = __ldg(reinterpret_cast<const uint4*>(f + c0));
                const uint4 b = __ldg(reinterpret_cast<const uint4*>(plane + dev_key_off<SPLIT>(P, row, h, d)));
                const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const float x = __fsub_rn(to_f(elem<E>(aw[k / 2], k & 1)), to_f(elem<E>(bw[k / 2], k & 1)));
                    acc = __fmaf_rn(x, x, acc);
                }
            } else {
                const int ce = min(c0 + 8, C);
                for (int c = c0; c < ce; ++c) {
                    const int h = c / P.D, d = c - h * P.D;
                    const float x = __fsub_rn(to_f(f[c]), to_f(plane[dev_key_off<SPLIT>(P, row, h, d)]));
                    acc = __fmaf_rn(x, x, acc);
                }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
        if (lane == 0) P.dev[i] = acc;
    }
}

template <class E>
static void launch_dev(bool vec, bool split, unsigned blocks, const BlendDevParams& P, cudaStream_t st) {
    if (vec) {
        if (split) blend_dev_kernel<E, true, true><<<blocks, 256, 0, st>>>(P);
        else blend_dev_kernel<E, true, false><<<blocks, 256, 0, st>>>(P);
    } else {
        if (split) blend_dev_kernel<E, false, true><<<blocks, 256, 0, st>>>(P);
        else blend_dev_kernel<E, false, false><<<blocks, 256, 0, st>>>(P);
    }
}

// ---------------------------------------------------------------------------------------------- select
// Every select kernel runs 256 threads.  The workspace holds the four 256-bin histograms of the radix passes, then one
// (forced, greater, equal) count per compaction CTA.
constexpr int kSelThreads = 256;
constexpr int kSelMaxCtas = 1024;
constexpr int64_t kSelPerCta = 1024;

static int sel_ctas(int64_t n) {
    return (int)std::max<int64_t>(1, std::min<int64_t>((n + kSelPerCta - 1) / kSelPerCta, kSelMaxCtas));
}

// The order of the selection as an unsigned key: larger dev, larger key.  NaN ranks as +inf, -0 ties with +0.
__device__ __forceinline__ uint32_t sel_key(float v) {
    uint32_t u = __float_as_uint(v);
    if (v != v) u = 0x7f800000u;
    if (u == 0x80000000u) u = 0u;
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Inclusive scan of v over the 256 threads of the CTA; *total gets the sum of all.  Every thread calls it.
__device__ __forceinline__ uint32_t cta_scan(uint32_t v, uint32_t* total) {
    __shared__ uint32_t s_w[kSelThreads / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += y;
    }
    if (lane == 31) s_w[wid] = v;
    __syncthreads();
    uint32_t base = 0, all = 0;
#pragma unroll
    for (int w = 0; w < kSelThreads / 32; ++w) {
        base += w < wid ? s_w[w] : 0u;
        all += s_w[w];
    }
    __syncthreads();
    *total = all;
    return base + v;
}

// The radix decisions of passes [0, passes), replayed by every CTA from the histograms (integer sums: the same bits in
// every CTA).  Pass p looks at key bits [24 - 8p, 32 - 8p) of the candidates whose higher bits equal `prefix`;
// krem counts the candidates still to take among them.  none: k or the candidates are 0, nothing is selected.
struct SelState {
    uint32_t prefix, mask, krem, none;
};

__device__ SelState sel_replay(const uint32_t* hist, int passes, int64_t k) {
    __shared__ SelState s;
    if (threadIdx.x == 0) {
        s.prefix = 0u;
        s.mask = 0u;
        s.krem = 0u;
        s.none = 0u;
    }
    __syncthreads();
    for (int p = 0; p < passes; ++p) {
        const int t = threadIdx.x, d = 255 - t;               // thread t holds digit 255 - t: scan from the top
        const uint32_t v = __ldcg(hist + p * 256 + d);
        uint32_t total;
        const uint32_t cum = cta_scan(v, &total);             // candidates with a digit >= d
        if (p == 0 && t == 0) {
            const uint32_t keff = k < (int64_t)total ? (uint32_t)k : total;
            s.krem = keff;
            s.none = keff == 0u ? 1u : 0u;
        }
        __syncthreads();
        const uint32_t krem = s.krem;
        const uint32_t none = s.none;
        __syncthreads();
        if (!none && cum >= krem && cum - v < krem) {         // exactly one digit holds the krem-th largest
            const int shift = 24 - 8 * p;
            s.prefix |= (uint32_t)d << shift;
            s.mask |= 0xffu << shift;
            s.krem = krem - (cum - v);
        }
        __syncthreads();
    }
    const SelState r = s;
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(kSelThreads) blend_hist_kernel(const float* dev, const uint8_t* cand, int64_t n,
                                                                 int64_t k, uint32_t* ws, int pass) {
    __shared__ uint32_t h[kSelThreads / 32][256];            // one histogram per warp: fewer same-address collisions
    const SelState s = sel_replay(ws, pass, k);
    if (pass > 0 && s.none) return;                           // uniform across the CTA
    const int wid = threadIdx.x >> 5, shift = 24 - 8 * pass;
    for (int w = 0; w < kSelThreads / 32; ++w) h[w][threadIdx.x] = 0u;
    __syncthreads();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        if (!__ldg(cand + i)) continue;
        const uint32_t key = sel_key(__ldg(dev + i));
        if ((key & s.mask) == s.prefix) atomicAdd(&h[wid][(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    uint32_t c = 0;
    for (int w = 0; w < kSelThreads / 32; ++w) c += h[w][threadIdx.x];
    if (c) atomicAdd(ws + pass * 256 + threadIdx.x, c);      // integer sums: the order does not show
}

// Flags of row i against the threshold key T of the select: forced, greater, equal
struct SelFlags {
    uint32_t f, g, e;
};
__device__ __forceinline__ SelFlags sel_flags(const float* dev, const uint8_t* cand, int64_t i, const SelState& s) {
    SelFlags r{0u, 0u, 0u};
    if (!__ldg(cand + i)) {
        r.f = 1u;
    } else if (!s.none) {
        const uint32_t key = sel_key(__ldg(dev + i));
        r.g = key > s.prefix;
        r.e = key == s.prefix;
    }
    return r;
}

// CTA c owns rows [c * per, min(n, (c + 1) * per)): its (forced, greater, equal) counts
__global__ void __launch_bounds__(kSelThreads) blend_count_kernel(const float* dev, const uint8_t* cand, int64_t n,
                                                                  int64_t k, int64_t per, uint32_t* ws) {
    const SelState s = sel_replay(ws, 4, k);
    const int64_t a = blockIdx.x * per, b = min(n, a + per);
    uint32_t f = 0, g = 0, e = 0;
    for (int64_t i = a + threadIdx.x; i < b; i += kSelThreads) {
        const SelFlags x = sel_flags(dev, cand, i, s);
        f += x.f;
        g += x.g;
        e += x.e;
    }
    __shared__ uint32_t s_c[3];
    if (threadIdx.x < 3) s_c[threadIdx.x] = 0u;
    __syncthreads();
    atomicAdd(&s_c[0], f);                                    // integer sums: the order does not show
    atomicAdd(&s_c[1], g);
    atomicAdd(&s_c[2], e);
    __syncthreads();
    if (threadIdx.x < 3) ws[4 * 256 + 4 * blockIdx.x + threadIdx.x] = s_c[threadIdx.x];
}

// Rows in order: forced row i at (forced rows before i); a candidate taken at n_forced + (greater rows before i) +
// min(equal rows before i, krem).  An equal row is taken while fewer than krem equal rows precede it.
__global__ void __launch_bounds__(kSelThreads) blend_write_kernel(const float* dev, const uint8_t* cand, int64_t n,
                                                                  int64_t k, int64_t per, const uint32_t* ws,
                                                                  int64_t* rows) {
    const SelState s = sel_replay(ws, 4, k);
    const uint32_t* cnt = ws + 4 * 256;
    uint32_t fb = 0, gb = 0, eb = 0, ft = 0;
    for (int j = threadIdx.x; j < (int)gridDim.x; j += kSelThreads) {
        const uint32_t* o = cnt + 4 * j;
        const uint32_t f = __ldcg(o), g = __ldcg(o + 1), e = __ldcg(o + 2);
        ft += f;
        if (j < (int)blockIdx.x) {
            fb += f;
            gb += g;
            eb += e;
        }
    }
    cta_scan(fb, &fb);
    cta_scan(gb, &gb);
    cta_scan(eb, &eb);
    cta_scan(ft, &ft);
    const int64_t a = blockIdx.x * per, b = min(n, a + per);
    for (int64_t base = a; base < b; base += kSelThreads) {
        const int64_t i = base + threadIdx.x;
        SelFlags x{0u, 0u, 0u};
        if (i < b) x = sel_flags(dev, cand, i, s);
        const uint32_t packed = x.f | (x.g << 10) | (x.e << 20);      // at most 256 each: 10-bit fields
        uint32_t tot;
        const uint32_t ex = cta_scan(packed, &tot) - packed;
        const uint32_t F = fb + (ex & 1023u), G = gb + ((ex >> 10) & 1023u), E = eb + (ex >> 20);
        if (x.f) rows[F] = i;
        if (x.g) rows[(int64_t)ft + G + min(E, s.krem)] = i;
        if (x.e && E < s.krem) rows[(int64_t)ft + G + E] = i;
        fb += tot & 1023u;
        gb += (tot >> 10) & 1023u;
        eb += tot >> 20;
    }
}

// ---------------------------------------------------------------------------------------------- segmented select
// b200kv_blend_select per segment [seg[s], seg[s+1]) of one array, in the same seven operations whatever n, B and the
// spread of the rows.  The rows are cut into CTAs as for the one-segment select, so a CTA's range may cross many segment
// boundaries.  Per segment the workspace holds four 256-bin histograms and the radix state after each pass; a launch
// settles the previous pass's decision of every segment its range overlaps (one warp per segment, every CTA that
// overlaps a segment writes the same values) instead of replaying the decisions of one global histogram.
//
// Workspace, in 32-bit words: hist [4][B][256] | state [4][B][4] (after passes 1..4: prefix, mask, krem, candidates) |
// out_start [B] | base [B][3] | per CTA [ctas][4] (forced, greater, equal rows of its last segment; that segment).
constexpr int kSegWords = 4 * 256 + 16 + 1 + 3;
constexpr int kSegSlots = 8;                                  // segments of a CTA counted in shared memory

struct SegSel {
    const float* dev;
    const uint8_t* cand;
    const int64_t* seg;
    const int64_t* k;
    int64_t n, per;
    int32_t B;
    uint32_t* ws;
    int64_t* rows;
};

__device__ __forceinline__ uint32_t* seg_hist(const SegSel& P, int pass, int s) {
    return P.ws + ((int64_t)pass * P.B + s) * 256;
}
__device__ __forceinline__ uint32_t* seg_state(const SegSel& P, int after, int s) {   // state after `after` passes
    return P.ws + (int64_t)1024 * P.B + ((int64_t)(after - 1) * P.B + s) * 4;
}
__device__ __forceinline__ uint32_t* seg_ostart(const SegSel& P, int s) { return P.ws + (int64_t)1040 * P.B + s; }
__device__ __forceinline__ uint32_t* seg_cta(const SegSel& P, int c) {
    return P.ws + (int64_t)kSegWords * P.B + 4 * (int64_t)c;
}

// The largest s in [lo, hi] with seg[s] <= i: the segment of row i (empty segments at i are skipped)
__device__ __forceinline__ int seg_of(const int64_t* seg, int lo, int hi, int64_t i) {
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(seg + mid) <= i) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// k of segment s against its candidates: the rows it selects
__device__ __forceinline__ uint32_t seg_keff(const SegSel& P, int s, uint32_t cand) {
    const int64_t k = __ldg(P.k + s);
    return k < (int64_t)cand ? (k > 0 ? (uint32_t)k : 0u) : cand;
}

// The rows of segment s in the output: its forced rows and min(k, candidates); 0 for an empty segment (never settled)
__device__ __forceinline__ uint32_t seg_size(const SegSel& P, int s) {
    const uint32_t len = (uint32_t)(__ldg(P.seg + s + 1) - __ldg(P.seg + s));
    if (len == 0u) return 0u;
    const uint32_t cand = __ldcg(seg_state(P, 4, s) + 3);
    return len - cand + seg_keff(P, s, cand);
}

// One warp: the decision of pass `pass` for segment s, from its histogram of that pass and its state before it (the
// integer sums of sel_replay, in the same order of digits): the state after it, written to the workspace and to *sh
// when given.  Lane l holds digits 255 - 8l - j, j < 8.
__device__ void seg_settle(const SegSel& P, int pass, int s, uint4* sh) {
    const int lane = threadIdx.x & 31;
    const uint32_t* h = seg_hist(P, pass, s);
    uint32_t v[8], sum = 0u;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        v[j] = __ldcg(h + 255 - 8 * lane - j);
        sum += v[j];
    }
    uint32_t inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    const uint32_t total = __shfl_sync(0xffffffffu, inc, 31);
    uint32_t prefix = 0u, mask = 0u, krem, cand;
    if (pass == 0) {
        cand = total;
        krem = seg_keff(P, s, cand);
    } else {
        const uint32_t* o = seg_state(P, pass, s);
        prefix = __ldcg(o);
        mask = __ldcg(o + 1);
        krem = __ldcg(o + 2);
        cand = __ldcg(o + 3);
    }
    const bool none = seg_keff(P, s, cand) == 0u;
    uint32_t found = 0u, d = 0u, kn = 0u;
    if (!none) {
        uint32_t cum = inc - sum;                            // candidates with a digit above this lane's
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            cum += v[j];
            if (cum >= krem && cum - v[j] < krem) {          // exactly one digit holds the krem-th largest
                found = 1u;
                d = 255u - 8u * lane - j;
                kn = krem - (cum - v[j]);
            }
        }
    }
    const uint32_t who = __ballot_sync(0xffffffffu, found);
    if (who) {
        const int src = __ffs(who) - 1;
        d = __shfl_sync(0xffffffffu, d, src);
        kn = __shfl_sync(0xffffffffu, kn, src);
        const int shift = 24 - 8 * pass;
        prefix |= d << shift;
        mask |= 0xffu << shift;
        krem = kn;
    }
    if (lane == 0) {
        const uint4 r = make_uint4(prefix, mask, krem, cand);
        uint32_t* o = seg_state(P, pass + 1, s);
        o[0] = r.x;
        o[1] = r.y;
        o[2] = r.z;
        o[3] = r.w;
        if (sh) *sh = r;
    }
}

// The CTA's rows [*a, *b) and the segments they cross, [*s0, *s1]; false for a CTA past the end
__device__ __forceinline__ bool seg_range(const SegSel& P, int64_t* a, int64_t* b, int* s0, int* s1) {
    *a = blockIdx.x * P.per;
    *b = min(P.n, *a + P.per);
    if (*a >= *b) return false;
    *s0 = seg_of(P.seg, 0, P.B - 1, *a);
    *s1 = seg_of(P.seg, *s0, P.B - 1, *b - 1);
    return true;
}

// Settle pass `pass` for the CTA's segments [s0, s1], one warp per segment; the first kSegSlots land in st[] too
__device__ __forceinline__ void seg_settle_all(const SegSel& P, int pass, int s0, int s1, uint4* st) {
    for (int s = s0 + (int)(threadIdx.x >> 5); s <= s1; s += kSelThreads / 32)
        seg_settle(P, pass, s, s - s0 < kSegSlots ? st + (s - s0) : nullptr);
    __syncthreads();
}

__device__ __forceinline__ uint4 seg_state_of(const SegSel& P, int s, int s0, const uint4* st) {
    if (s - s0 < kSegSlots) return st[s - s0];
    const uint32_t* o = seg_state(P, 4, s);
    return make_uint4(__ldcg(o), __ldcg(o + 1), __ldcg(o + 2), __ldcg(o + 3));
}

__global__ void __launch_bounds__(kSelThreads) blend_seg_hist_kernel(SegSel P, int pass) {
    __shared__ uint32_t h[kSegSlots][256];
    __shared__ uint4 st[kSegSlots];
    int64_t a, b;
    int s0, s1;
    if (!seg_range(P, &a, &b, &s0, &s1)) return;
    if (pass > 0) seg_settle_all(P, pass - 1, s0, s1, st);
    for (int j = 0; j < kSegSlots; ++j) h[j][threadIdx.x] = 0u;
    __syncthreads();
    const int shift = 24 - 8 * pass;
    for (int64_t i = a + threadIdx.x; i < b; i += kSelThreads) {
        if (!__ldg(P.cand + i)) continue;
        const int s = seg_of(P.seg, s0, s1, i);
        uint32_t prefix = 0u, mask = 0u;
        if (pass > 0) {
            uint4 x;
            if (s - s0 < kSegSlots) {
                x = st[s - s0];
            } else {
                const uint32_t* o = seg_state(P, pass, s);
                x = make_uint4(__ldcg(o), __ldcg(o + 1), 0u, __ldcg(o + 3));
            }
            if (seg_keff(P, s, x.w) == 0u) continue;          // nothing selected in s
            prefix = x.x;
            mask = x.y;
        }
        const uint32_t key = sel_key(__ldg(P.dev + i));
        if ((key & mask) != prefix) continue;
        const uint32_t d = (key >> shift) & 255u;
        if (s - s0 < kSegSlots) atomicAdd(&h[s - s0][d], 1u);
        else atomicAdd(seg_hist(P, pass, s) + d, 1u);        // integer sums: the order does not show
    }
    __syncthreads();
    for (int j = 0; j < kSegSlots && s0 + j <= s1; ++j) {
        const uint32_t c = h[j][threadIdx.x];
        if (c) atomicAdd(seg_hist(P, pass, s0 + j) + threadIdx.x, c);
    }
}

// Flags of row i of segment s (state x after the four passes) against the segment's threshold key
__device__ __forceinline__ SelFlags seg_flags(const SegSel& P, int64_t i, int s, const uint4& x) {
    SelFlags r{0u, 0u, 0u};
    if (!__ldg(P.cand + i)) {
        r.f = 1u;
    } else if (seg_keff(P, s, x.w) != 0u) {
        const uint32_t key = sel_key(__ldg(P.dev + i));
        r.g = key > x.x;
        r.e = key == x.x;
    }
    return r;
}

// Settles the last pass; CTA c records the (forced, greater, equal) rows of its last segment and that segment
__global__ void __launch_bounds__(kSelThreads) blend_seg_count_kernel(SegSel P) {
    __shared__ uint4 st[kSegSlots];
    __shared__ uint32_t s_c[3];
    int64_t a, b;
    int s0, s1;
    uint32_t* out = seg_cta(P, blockIdx.x);
    if (!seg_range(P, &a, &b, &s0, &s1)) {
        if (threadIdx.x < 4) out[threadIdx.x] = threadIdx.x == 3 ? 0xffffffffu : 0u;
        return;
    }
    seg_settle_all(P, 3, s0, s1, st);
    const uint4 x = seg_state_of(P, s1, s0, st);
    uint32_t f = 0, g = 0, e = 0;
    for (int64_t i = max(a, __ldg(P.seg + s1)) + threadIdx.x; i < b; i += kSelThreads) {
        const SelFlags y = seg_flags(P, i, s1, x);
        f += y.f;
        g += y.g;
        e += y.e;
    }
    if (threadIdx.x < 3) s_c[threadIdx.x] = 0u;
    __syncthreads();
    atomicAdd(&s_c[0], f);                                    // integer sums: the order does not show
    atomicAdd(&s_c[1], g);
    atomicAdd(&s_c[2], e);
    __syncthreads();
    if (threadIdx.x < 4) out[threadIdx.x] = threadIdx.x == 3 ? (uint32_t)s1 : s_c[threadIdx.x];
}

// Row i of segment s goes to out_start[s] + (forced rows of s before i) if forced; a candidate taken to out_start[s] +
// F_s + (greater rows of s before i) + min(equal rows of s before i, krem_s).  "Before i" counts the rows of s in
// earlier CTAs (the carry of the CTA's first segment) and in this CTA: a running inclusive scan of the flags minus its
// value at the segment's first row.
__global__ void __launch_bounds__(kSelThreads) blend_seg_write_kernel(SegSel P) {
    __shared__ uint4 st[kSegSlots];
    __shared__ uint32_t s_base[3][kSelThreads];
    int64_t a, b;
    int s0, s1;
    if (!seg_range(P, &a, &b, &s0, &s1)) return;
    for (int j = threadIdx.x; j < kSegSlots && s0 + j <= s1; j += kSelThreads) {
        const uint32_t* o = seg_state(P, 4, s0 + j);
        st[j] = make_uint4(__ldcg(o), __ldcg(o + 1), __ldcg(o + 2), __ldcg(o + 3));
    }
    // the rows of s0 in earlier CTAs
    uint32_t fc = 0, gc = 0, ec = 0;
    for (int j = threadIdx.x; j < (int)blockIdx.x; j += kSelThreads) {
        const uint32_t* o = seg_cta(P, j);
        if (__ldcg(o + 3) == (uint32_t)s0) {
            fc += __ldcg(o);
            gc += __ldcg(o + 1);
            ec += __ldcg(o + 2);
        }
    }
    cta_scan(fc, &fc);
    cta_scan(gc, &gc);
    cta_scan(ec, &ec);
    // the output rows of the segments before s0, then the output start of every segment of the CTA
    uint32_t o0 = 0;
    for (int s = threadIdx.x; s < s0; s += kSelThreads) o0 += seg_size(P, s);
    cta_scan(o0, &o0);
    for (int base = s0; base <= s1; base += kSelThreads) {
        const int s = base + threadIdx.x;
        const uint32_t sz = s <= s1 ? seg_size(P, s) : 0u;
        uint32_t tot;
        const uint32_t inc = cta_scan(sz, &tot);
        if (s <= s1) *seg_ostart(P, s) = o0 + inc - sz;     // the same value from every CTA that overlaps s
        o0 += tot;
    }
    __syncthreads();
    // running counts of the CTA's rows before the tile, and the base of the segment open at the tile's first row
    uint32_t fr = 0, gr = 0, er = 0;
    uint32_t fo = 0u - fc, go = 0u - gc, eo = 0u - ec;
    for (int64_t t0 = a; t0 < b; t0 += kSelThreads) {
        const int64_t i = t0 + threadIdx.x;
        SelFlags x{0u, 0u, 0u};
        int s = s0;
        int64_t start = 0;
        uint4 y = make_uint4(0u, 0u, 0u, 0u);
        if (i < b) {
            s = seg_of(P.seg, s0, s1, i);
            start = __ldg(P.seg + s);
            y = seg_state_of(P, s, s0, st);
            x = seg_flags(P, i, s, y);
        }
        const uint32_t packed = x.f | (x.g << 10) | (x.e << 20);      // at most 256 each: 10-bit fields
        uint32_t tot;
        const uint32_t ex = cta_scan(packed, &tot) - packed;
        const uint32_t F = fr + (ex & 1023u), G = gr + ((ex >> 10) & 1023u), E = er + (ex >> 20);
        if (i < b && start == i && i > a) {                   // s starts here: its base
            s_base[0][threadIdx.x] = F;
            s_base[1][threadIdx.x] = G;
            s_base[2][threadIdx.x] = E;
        }
        __syncthreads();
        if (i < b) {
            uint32_t bf = fo, bg = go, be = eo;
            if (start > t0) {
                const int o = (int)(start - t0);
                bf = s_base[0][o];
                bg = s_base[1][o];
                be = s_base[2][o];
            }
            const uint32_t Fs = F - bf, Gs = G - bg, Es = E - be;
            const int64_t os = __ldcg(seg_ostart(P, s));
            const uint32_t len = (uint32_t)(__ldg(P.seg + s + 1) - start);
            const int64_t ft = os + (len - y.w);              // forced rows of s: its rows less its candidates
            if (x.f) P.rows[os + Fs] = i;
            if (x.g) P.rows[ft + Gs + min(Es, y.z)] = i;
            if (x.e && Es < y.z) P.rows[ft + Gs + Es] = i;
        }
        // the segment open at the next tile's first row: still the open one, or one that started in this tile
        const int64_t nx = t0 + kSelThreads;
        if (nx < b) {
            const int64_t ns = __ldg(P.seg + seg_of(P.seg, s0, s1, nx));
            if (ns == nx) {                                   // it starts at the next tile: the counts so far
                fo = fr + (tot & 1023u);
                go = gr + ((tot >> 10) & 1023u);
                eo = er + (tot >> 20);
            } else if (ns > t0) {
                const int o = (int)(ns - t0);
                fo = s_base[0][o];
                go = s_base[1][o];
                eo = s_base[2][o];
            }
        }
        fr += tot & 1023u;
        gr += (tot >> 10) & 1023u;
        er += tot >> 20;
        __syncthreads();
    }
}

}  // namespace b200kv

using namespace b200kv;

extern "C" {

int b200kv_blend_deviation(const b200kv_kv_desc* kv, int32_t layer, int64_t n, const int64_t* tok, const void* fresh,
                           int64_t fresh_row_stride, float* dev, void* stream) {
    B2_REQUIRE(kv != nullptr, "kv descriptor is NULL");
    B2_REQUIRE(n >= 0, "n must be non-negative");
    B2_REQUIRE(n == 0 || (tok != nullptr && fresh != nullptr && dev != nullptr), "NULL pointer");
    B2_REQUIRE(kv->L > 0 && 2 * kv->L <= B200KV_MAX_PLANES, "L out of range");
    B2_REQUIRE(kv->H > 0 && kv->D > 0, "H/D must be positive");
    B2_REQUIRE(0 <= layer && layer < kv->L, "layer outside [0, L)");
    const bool split = kv_split(kv);
    const int dt = split ? kv_split_dtype(kv) : kv_dtype(kv);
    B2_REQUIRE(dt == B200KV_DT_BF16 || dt == B200KV_DT_FP16,
               "the blend deviation takes 16-bit keys only (the segment calls refuse FP8 KV)");
    const int64_t C = (int64_t)kv->H * kv->D;
    B2_REQUIRE(C < (1ll << 30), "H * D too large");
    B2_REQUIRE(fresh_row_stride >= C, "fresh row stride is smaller than H * D");
    if (split) {
        B2_REQUIRE(!(kv->dtype & B200KV_KV_LATENT), "a latent KV has no split layout");
        B2_REQUIRE(kv->slot_map != nullptr, "a split paged KV (B200KV_KV_PAGED_SPLIT) needs a slot_map");
        B2_REQUIRE(kv->D % 8 == 0, "a split paged KV needs D % x == 0");
        B2_REQUIRE(kv->sT > 0 && kv->sT <= (1 << 20), "block size out of range");
    }
    b200kv_kv_desc rows = *kv;                 // the planes' pointers, read through the rows' table builder
    rows.dtype = dt | (kv->dtype & B200KV_KV_LATENT);
    float bins[B200KV_MAX_PLANES];
    for (int i = 0; i < B200KV_MAX_PLANES; ++i) bins[i] = 32.0f;
    PlaneTable pt;
    if (int rc = make_plane_table(&rows, bins, bins, &pt)) return rc;
    if (n == 0) return 0;
    BlendDevParams P;
    P.plane = pt.p[layer];
    P.slot_map = kv->slot_map;
    P.tok = tok;
    P.fresh = fresh;
    P.dev = dev;
    P.n = n;
    P.fresh_stride = fresh_row_stride;
    P.sT = kv->sT;
    P.sH = kv->sH;
    P.H = kv->H;
    P.D = kv->D;
    P.bs = split ? (int32_t)kv->sT : 0;
    // 16-byte vectors: groups of 8 channels inside one head, every row start and the planes 16-byte aligned (the split
    // layout keeps 8 channels of a token together: its strides are always aligned)
    const bool vec = kv->D % 8 == 0 && fresh_row_stride % 8 == 0 && (reinterpret_cast<uintptr_t>(fresh) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(P.plane) & 15) == 0 &&
                     (split || (kv->sT % 8 == 0 && kv->sH % 8 == 0));
    int devi = 0, sms = 0;
    B2_CHECK_CUDA(cudaGetDevice(&devi));
    B2_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, devi));
    const int64_t blocks = std::max<int64_t>(1, std::min<int64_t>((n + 7) / 8, (int64_t)sms * 8));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (dt == B200KV_DT_BF16) launch_dev<__nv_bfloat16_raw>(vec, split, (unsigned)blocks, P, st);
    else launch_dev<__half_raw>(vec, split, (unsigned)blocks, P, st);
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int64_t b200kv_blend_select_workspace_bytes(int64_t n) {
    if (n < 0) return -2;
    return (int64_t)(4 * 256 + 4 * sel_ctas(n)) * (int64_t)sizeof(uint32_t);
}

int b200kv_blend_select(const float* dev, const uint8_t* cand, int64_t n, int64_t k, int64_t* rows, void* workspace,
                        int64_t workspace_bytes, void* stream) {
    B2_REQUIRE(n >= 0 && n < (1ll << 31), "n outside [0, 2^31)");
    B2_REQUIRE(k >= 0, "k must be non-negative");
    B2_REQUIRE(n == 0 || (dev != nullptr && cand != nullptr && rows != nullptr && workspace != nullptr),
               "NULL pointer");
    if (n == 0) return 0;
    B2_REQUIRE(workspace_bytes >= b200kv_blend_select_workspace_bytes(n), "workspace too small");
    B2_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 3) == 0, "workspace must be 4-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    uint32_t* ws = static_cast<uint32_t*>(workspace);
    const int ctas = sel_ctas(n);
    const int64_t per = (n + ctas - 1) / ctas;
    B2_CHECK_CUDA(cudaMemsetAsync(ws, 0, 4 * 256 * sizeof(uint32_t), st));
    for (int p = 0; p < 4; ++p) blend_hist_kernel<<<ctas, kSelThreads, 0, st>>>(dev, cand, n, k, ws, p);
    blend_count_kernel<<<ctas, kSelThreads, 0, st>>>(dev, cand, n, k, per, ws);
    blend_write_kernel<<<ctas, kSelThreads, 0, st>>>(dev, cand, n, k, per, ws, rows);
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int64_t b200kv_blend_select_batch_workspace_bytes(int64_t n, int64_t B) {
    if (n < 0 || B < 1 || B >= (1ll << 31)) return -2;
    return (B * kSegWords + 4 * (int64_t)sel_ctas(n)) * (int64_t)sizeof(uint32_t);
}

int b200kv_blend_select_batch(const float* dev, const uint8_t* cand, int64_t n, int64_t B, const int64_t* seg,
                              const int64_t* k, int64_t* rows, void* workspace, int64_t workspace_bytes,
                              void* stream) {
    B2_REQUIRE(n >= 0 && n < (1ll << 31), "n outside [0, 2^31)");
    B2_REQUIRE(B >= 1 && B < (1ll << 31), "B outside [1, 2^31)");
    B2_REQUIRE(n == 0 || (dev != nullptr && cand != nullptr && seg != nullptr && k != nullptr && rows != nullptr &&
                          workspace != nullptr),
               "NULL pointer");
    if (n == 0) return 0;
    B2_REQUIRE(workspace_bytes >= b200kv_blend_select_batch_workspace_bytes(n, B), "workspace too small");
    B2_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 3) == 0, "workspace must be 4-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int ctas = sel_ctas(n);
    SegSel P;
    P.dev = dev;
    P.cand = cand;
    P.seg = seg;
    P.k = k;
    P.n = n;
    P.per = (n + ctas - 1) / ctas;
    P.B = (int32_t)B;
    P.ws = static_cast<uint32_t*>(workspace);
    P.rows = rows;
    B2_CHECK_CUDA(cudaMemsetAsync(P.ws, 0, (size_t)B * 4 * 256 * sizeof(uint32_t), st));
    for (int p = 0; p < 4; ++p) blend_seg_hist_kernel<<<ctas, kSelThreads, 0, st>>>(P, p);
    blend_seg_count_kernel<<<ctas, kSelThreads, 0, st>>>(P);
    blend_seg_write_kernel<<<ctas, kSelThreads, 0, st>>>(P);
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // extern "C"
