// rope.cu -- rotary position shift of stored keys, for KV reused at another position than the one it was computed at.
//
// vLLM caches K after the rotary embedding: a document prefilled alone at positions 0..n-1 holds R(i)·k_i.  Placed at
// offset s it must hold R(s + i)·k_i = R(s)·(R(i)·k_i): every key row is rotated by s·θ_j, pair by pair.  V carries no
// position and is not touched.
//
//   b200kv_rope_table: cos / sin of s·inv_freq[j] for every segment shift s, the angle in fp64, range-reduced, then
//                      rounded once to fp32 (a shift of 65536 at inv_freq 1 is 6.6e4 rad: its fp32 product alone would be
//                      ~4e-3 rad off, far more than one bf16 ulp of the result).
//   b200kv_rope_shift: one launch rotates channels [offset, offset + rotary_dim) of the key rows of a token range, every
//                      layer and head, in any layout a kv_desc carries (rows, slot-mapped rows, the split key blocks).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "rope.cuh"     // to_f / from_f / rotate: the same arithmetic as the mover's b200kv_pack_chunks_rope

namespace b200kv {

struct RopeParams {
    PlaneTable pt;                 // key plane l = pt.p[l] (the latent plane of a latent KV)
    const int64_t* slot_map;       // NULL: row = token
    const int32_t* seg_of_tok;     // [ntok]: table row of token tok_begin + i, or -1
    const float2* cs;              // [n_seg][half]: (cos, sin)
    int64_t sT, sH, tok_begin, ntok;
    int32_t L, H, D, half, offset, bs;   // bs: the split layout's block size
};
static_assert(sizeof(RopeParams) < kMaxParamBytes, "RopeParams must stay under 4 KB of kernel parameters");

// Element offset of channel c (c % X == 0 when a vector is read there) of head h of the token in cache row `row`.
// SPLIT: key blocks [nb, H, D/X, bs, X]; rows: row * sT + h * sH + c.
template <int X, bool SPLIT>
__device__ __forceinline__ int64_t key_off(const RopeParams& P, int64_t row, int h, int c) {
    if (SPLIT) {
        const int64_t b = row / P.bs, o = row - b * P.bs;
        return (((b * P.H + h) * (P.D / X) + c / X) * P.bs + o) * X + c % X;
    }
    return row * P.sT + (int64_t)h * P.sH + c;
}

// One unit = NP rotation pairs of one (token, layer, head).  NEOX: pairs (j, j + half), a unit reads NP channels from
// each half (NP = 8: two 16-byte vectors).  GPT-J: pairs (2j, 2j + 1), a unit reads 2 NP channels (NP = 4: one vector).
// NP = 1: one pair, element by element (any alignment).  Rows: a unit's neighbours are the next pairs of the same row;
// SPLIT: the same pairs of the next token, which the split layout keeps 16 bytes further (coalesced either way).
template <class E, int NP, bool NEOX, bool SPLIT>
__global__ void __launch_bounds__(256) rope_shift_kernel(RopeParams P) {
    constexpr int X = 16 / (int)sizeof(E);
    const int upr = P.half / NP;                          // units per (token, layer, head)
    const int64_t per_tok = (int64_t)P.L * P.H * upr;
    const int64_t total = P.ntok * per_tok;
    for (int64_t u = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; u < total; u += (int64_t)gridDim.x * blockDim.x) {
        int64_t i, r;
        if (SPLIT) {
            r = u / P.ntok;
            i = u - r * P.ntok;
        } else {
            i = u / per_tok;
            r = u - i * per_tok;
        }
        const int seg = __ldg(P.seg_of_tok + i);
        if (seg < 0) continue;
        const int v = (int)(r % upr);                     // r = (l * H + h) * upr + v
        const int64_t lh = r / upr;
        const int h = (int)(lh % P.H), l = (int)(lh / P.H);
        const int64_t tok = P.tok_begin + i;
        const int64_t row = P.slot_map ? __ldg(P.slot_map + tok) : tok;
        E* plane = const_cast<E*>(reinterpret_cast<const E*>(P.pt.p[l]));
        const int j0 = v * NP;
        const float2* t = P.cs + (int64_t)seg * P.half + j0;
        if (NEOX) {
            E* pa = plane + key_off<X, SPLIT>(P, row, h, P.offset + j0);
            E* pb = plane + key_off<X, SPLIT>(P, row, h, P.offset + P.half + j0);
            if (NP == 1) {
                rotate(*pa, *pb, __ldg(t));
            } else {
                union { uint4 q; E e[8]; } a, b;
                a.q = *reinterpret_cast<const uint4*>(pa);
                b.q = *reinterpret_cast<const uint4*>(pb);
#pragma unroll
                for (int k = 0; k < NP; ++k) rotate(a.e[k], b.e[k], __ldg(t + k));
                *reinterpret_cast<uint4*>(pa) = a.q;
                *reinterpret_cast<uint4*>(pb) = b.q;
            }
        } else {
            if (NP == 1) {
                E* pa = plane + key_off<X, SPLIT>(P, row, h, P.offset + 2 * j0);
                E* pb = plane + key_off<X, SPLIT>(P, row, h, P.offset + 2 * j0 + 1);
                rotate(*pa, *pb, __ldg(t));
            } else {
                E* pa = plane + key_off<X, SPLIT>(P, row, h, P.offset + 2 * j0);
                union { uint4 q; E e[8]; } a;
                a.q = *reinterpret_cast<const uint4*>(pa);
#pragma unroll
                for (int k = 0; k < NP; ++k) rotate(a.e[2 * k], a.e[2 * k + 1], __ldg(t + k));
                *reinterpret_cast<uint4*>(pa) = a.q;
            }
        }
    }
}

template <class E, bool NEOX, bool SPLIT>
static void launch_rope(bool vec, unsigned blocks, const RopeParams& P, cudaStream_t stream) {
    if (vec) rope_shift_kernel<E, NEOX ? 8 : 4, NEOX, SPLIT><<<blocks, 256, 0, stream>>>(P);
    else rope_shift_kernel<E, 1, NEOX, SPLIT><<<blocks, 256, 0, stream>>>(P);
}

template <class E>
static void launch_rope_e(bool vec, bool neox, bool split, unsigned blocks, const RopeParams& P, cudaStream_t stream) {
    if (neox) {
        if (split) launch_rope<E, true, true>(vec, blocks, P, stream);
        else launch_rope<E, true, false>(vec, blocks, P, stream);
    } else {
        if (split) launch_rope<E, false, true>(vec, blocks, P, stream);
        else launch_rope<E, false, false>(vec, blocks, P, stream);
    }
}

// One thread per (segment, frequency): the angle s * inv_freq[j] in fp64 (exact to 2^-53 relative: a 31-bit shift times
// a 24-bit mantissa), reduced to [-pi, pi] by a two-part 2*pi (Cody-Waite), then sincos in fp64, rounded once to fp32.
__global__ void rope_table_kernel(const int64_t* shifts, int32_t n_seg, const float* inv_freq, int32_t half,
                                  float2* cos_sin) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_seg * half) return;
    const int s = i / half, j = i - s * half;
    const double a = (double)__ldg(shifts + s) * (double)__ldg(inv_freq + j);
    constexpr double kTwoPiHi = 6.28318530717958623200e+00;     // 2*pi rounded to double
    constexpr double kTwoPiLo = 2.44929359829470635445e-16;     // 2*pi - kTwoPiHi
    const double k = rint(a * 0.15915494309189533577);          // a / (2*pi), to the nearest turn
    const double red = fma(-k, kTwoPiLo, fma(-k, kTwoPiHi, a));
    double sn, cn;
    sincos(red, &sn, &cn);
    cos_sin[i] = make_float2((float)cn, (float)sn);
}

}  // namespace b200kv

using namespace b200kv;

extern "C" {

int b200kv_rope_table(const int64_t* shifts, int32_t n_seg, const float* inv_freq, int32_t rotary_dim, float* cos_sin,
                      void* stream) {
    B2_REQUIRE(shifts != nullptr && inv_freq != nullptr && cos_sin != nullptr, "NULL pointer");
    B2_REQUIRE(n_seg > 0, "n_seg must be positive");
    B2_REQUIRE(rotary_dim > 0 && rotary_dim % 2 == 0, "rotary_dim must be even and positive");
    const int half = rotary_dim / 2;
    B2_REQUIRE((int64_t)n_seg * half < (1ll << 31), "table too large");
    const int n = n_seg * half;
    rope_table_kernel<<<(n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        shifts, n_seg, inv_freq, half, reinterpret_cast<float2*>(cos_sin));
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int b200kv_rope_shift(const b200kv_kv_desc* kv, int64_t tok_begin, int64_t ntok, const int32_t* seg_of_tok,
                      const float* cos_sin, int32_t rotary_dim, int32_t offset, int32_t style, void* stream) {
    B2_REQUIRE(kv != nullptr, "kv descriptor is NULL");
    B2_REQUIRE(cos_sin != nullptr, "cos_sin table is NULL");
    B2_REQUIRE(ntok >= 0 && tok_begin >= 0, "bad token range");
    B2_REQUIRE(ntok == 0 || seg_of_tok != nullptr, "seg_of_tok is NULL");
    B2_REQUIRE(style == 0 || style == 1, "style must be 0 (neox) or 1 (gptj)");
    B2_REQUIRE(kv->L > 0 && 2 * kv->L <= B200KV_MAX_PLANES, "L out of range");
    B2_REQUIRE(kv->H > 0 && kv->D > 0, "H/D must be positive");
    const bool split = kv_split(kv);
    const int dt = split ? kv_split_dtype(kv) : kv_dtype(kv);
    B2_REQUIRE(dt == B200KV_DT_BF16 || dt == B200KV_DT_FP16,
               "the rope shift takes 16-bit keys only: rotating a one-byte (FP8) key would round it again");
    B2_REQUIRE(rotary_dim > 0 && rotary_dim % 2 == 0, "rotary_dim must be even and positive");
    B2_REQUIRE(offset >= 0 && (int64_t)offset + rotary_dim <= kv->D, "offset + rotary_dim exceeds the head size D");
    if (split) {
        B2_REQUIRE(!(kv->dtype & B200KV_KV_LATENT), "a latent KV has no split layout");
        B2_REQUIRE(kv->slot_map != nullptr, "a split paged KV (B200KV_KV_PAGED_SPLIT) needs a slot_map");
        B2_REQUIRE(kv->D % 8 == 0, "a split paged KV needs D % x == 0");
        B2_REQUIRE(kv->sT > 0 && kv->sT <= (1 << 20), "block size out of range");
    }
    RopeParams P;
    b200kv_kv_desc rows = *kv;                 // the planes' pointers, read through the rows' table builder
    rows.dtype = dt | (kv->dtype & B200KV_KV_LATENT);
    float bins[B200KV_MAX_PLANES];
    for (int i = 0; i < B200KV_MAX_PLANES; ++i) bins[i] = 32.0f;
    if (int rc = make_plane_table(&rows, bins, bins, &P.pt)) return rc;
    if (ntok == 0) return 0;
    P.slot_map = kv->slot_map;
    P.seg_of_tok = seg_of_tok;
    P.cs = reinterpret_cast<const float2*>(cos_sin);
    P.sT = kv->sT; P.sH = kv->sH; P.tok_begin = tok_begin; P.ntok = ntok;
    P.L = kv->L; P.H = kv->H; P.D = kv->D;
    P.half = rotary_dim / 2;
    P.offset = offset;
    P.bs = split ? (int32_t)kv->sT : 0;
    const bool neox = style == 0;
    // 16-byte vectors: neox takes 8 channels from each half, gptj 4 pairs; the channels, strides and planes must be
    // 16-byte aligned (the split layout keeps X = 8 channels of one token together: its strides are always aligned)
    bool vec = offset % 8 == 0 && (neox ? P.half % 8 == 0 : rotary_dim % 8 == 0) &&
               (split || (kv->sT % 8 == 0 && kv->sH % 8 == 0));
    for (int l = 0; l < kv->L && vec; ++l) vec = (reinterpret_cast<uintptr_t>(P.pt.p[l]) & 15) == 0;
    const int np = vec ? (neox ? 8 : 4) : 1;
    const int64_t total = ntok * kv->L * kv->H * (P.half / np);
    int dev = 0, sms = 0;
    B2_CHECK_CUDA(cudaGetDevice(&dev));
    B2_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    int64_t blocks = std::min<int64_t>((total + 255) / 256, (int64_t)sms * 8 * 4);
    if (blocks < 1) blocks = 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (dt == B200KV_DT_BF16) launch_rope_e<__nv_bfloat16_raw>(vec, neox, split, (unsigned)blocks, P, st);
    else launch_rope_e<__half_raw>(vec, neox, split, (unsigned)blocks, P, st);
    B2_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // extern "C"
