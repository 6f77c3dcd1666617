// ac_core.cuh -- arithmetic shared by every codec kernel: half conversions, the bit-exact
// CacheGen quantiser / dequantiser, the CDF normalisation and the arithmetic-coder state machines.
//
// Everything here is __host__ __device__ so that tests/hostsim can compile the *same* functions with
// g++ and check them against the oracle on the CPU (test infrastructure only; the product library
// only ever runs them inside CUDA kernels).
//
// Normative behaviour (reference file:line, relative to the LMCache v0.1.2 tree):
//   quantise    lmcache/storage_backend/serde/cachegen_encoder.py:40-61   fp32 div, mul, add each rounded
//   dequantise  lmcache/storage_backend/serde/cachegen_decoder.py:24-35   fp32 sub, div, mul each rounded
//   CDF         cachegen_encoder.py:95-126,185-196 (torch-CPU semantics: fp32 n/t, double cumsum)
//   coder       torchac lineage as called at cachegen_encoder.py:255-260 / cachegen_decoder.py:65-66
//               (32-bit low/high, 16-bit CDF, E1/E2/E3 renormalisation, MSB-first bit packing)
//
// Two coders live here, both producing exactly the bit-by-bit reference bitstream:
//   * EncState / DecState (enc_symbol, dec_symbol): a direct restatement with batched shifts
//       n = clz(low ^ high)                 E1/E2 shifts: the n leading bits agree and are emitted
//       m = clz(((~low | high) << 1) | 1)   E3 shifts: m more "pending" bits
//     kept as the readable baseline the host tests compare against;
//   * EncState2 / DecState2 (enc_symbol2, dec_symbol2): what the kernels run.  They track the ABSOLUTE
//     low (pending bits = carry resolution), so every shift of any kind is one funnel shift with one
//     count k = n + m, emission needs no pending counter, and the decoder finds the symbol with an
//     approximate reciprocal + a fixed-depth branch-free search that the exact interval products verify
//     (DESIGN.md sections 3.2 and 3.4).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B2_HD __host__ __device__ __forceinline__
#else
#define B2_HD inline
#endif

namespace b200kv {

constexpr int kLp = 33;       // CDF entries per stream
constexpr int kMaxSym = 31;   // Lp - 2
constexpr int kGroup = 256;   // tokens per coder group

// ---------------------------------------------------------------- bit helpers
B2_HD uint32_t f2u(float f) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    union { float f; uint32_t u; } v; v.f = f; return v.u;
#endif
}
B2_HD float u2f(uint32_t u) {
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    union { float f; uint32_t u; } v; v.u = u; return v.f;
#endif
}
B2_HD uint32_t clz32(uint32_t x) {  // x != 0
#if defined(__CUDA_ARCH__)
    return (uint32_t)__clz((int)x);
#else
    return (uint32_t)__builtin_clz(x);
#endif
}

// upper 32 bits of (hi:lo) << n, 0 <= n <= 31
B2_HD uint32_t funnel_l(uint32_t lo, uint32_t hi, uint32_t n) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(lo, hi, n);
#else
    return n ? ((hi << n) | (lo >> (32u - n))) : hi;
#endif
}
// lower 32 bits of (hi:lo) >> n, 0 <= n <= 31
B2_HD uint32_t funnel_r(uint32_t lo, uint32_t hi, uint32_t n) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, n);
#else
    return n ? ((lo >> n) | (hi << (32u - n))) : lo;
#endif
}
B2_HD uint32_t bswap32(uint32_t v) {
#if defined(__CUDA_ARCH__)
    return __byte_perm(v, 0u, 0x0123);
#else
    return __builtin_bswap32(v);
#endif
}

// position of the leading one (FLO / bfind); 0xFFFFFFFF for x == 0
B2_HD uint32_t bfind32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    uint32_t r;
    asm("bfind.u32 %0, %1;" : "=r"(r) : "r"(x));
    return r;
#else
    return x ? 31u - (uint32_t)__builtin_clz(x) : 0xFFFFFFFFu;
#endif
}

// (1 << p) - 1 for 0 <= p <= 31: one BMSK, no constant register
B2_HD uint32_t low_mask(uint32_t p) {
#if defined(__CUDA_ARCH__)
    uint32_t r;
    asm("bmsk.clamp.b32 %0, 0, %1;" : "=r"(r) : "r"(p));
    return r;
#else
    return (1u << p) - 1u;
#endif
}

// (x << n) | ones(n), 0 <= n <= 31 : one funnel shift with an all-ones low word
B2_HD uint32_t shl_fill1(uint32_t x, uint32_t n) { return funnel_l(0xFFFFFFFFu, x, n); }

// number of E3 ("straddle") steps for a normalised interval low = 0..., high = 1...:
// count of leading positions (from bit 30 down) where low has 1 and high has 0
B2_HD uint32_t e3_count(uint32_t low, uint32_t high) {
    const uint32_t x = ((~low) | high) & 0x7FFFFFFFu;        // one LOP3
#if defined(__CUDA_ARCH__)
    return 30u - (uint32_t)(31 - __clz((int)x));               // FLO of 0 is -1 -> 31
#else
    return x ? 30u - (31u - (uint32_t)__builtin_clz(x)) : 31u;
#endif
}

// fp32 ops that must not be contracted / reordered
B2_HD float fdiv(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fdiv_rn(a, b);
#else
    volatile float r = a / b; return r;
#endif
}
B2_HD float fmul(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    volatile float r = a * b; return r;
#endif
}
B2_HD float fadd(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    volatile float r = a + b; return r;
#endif
}
B2_HD float frint(float a) {   // round half to even
#if defined(__CUDA_ARCH__)
    return rintf(a);
#else
    return __builtin_nearbyintf(a);
#endif
}

// ---------------------------------------------------------------- half <-> float (bit patterns)
B2_HD float bf16_to_float(uint16_t h) { return u2f((uint32_t)h << 16); }

B2_HD uint16_t float_to_bf16(float f) {  // RNE, NaN stays NaN (matches torch .to(bfloat16))
    uint32_t u = f2u(f);
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x0040u);
    u += 0x7fffu + ((u >> 16) & 1u);
    return (uint16_t)(u >> 16);
}

B2_HD float fp16_to_float(uint16_t h) {
    uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
    uint32_t exp = (h >> 10) & 0x1fu;
    uint32_t man = h & 0x3ffu;
    if (exp == 0) {
        if (man == 0) return u2f(sign);
        // subnormal: value = man * 2^-24
        float v = (float)man * 5.9604644775390625e-08f;
        return u2f(f2u(v) | sign);
    }
    if (exp == 31) return u2f(sign | 0x7f800000u | (man << 13));
    return u2f(sign | ((exp + 112u) << 23) | (man << 13));
}

B2_HD uint16_t float_to_fp16(float f) {  // RNE with overflow to inf, subnormals, NaN kept (torch .to(float16))
    uint32_t u = f2u(f);
    uint32_t sign = (u >> 16) & 0x8000u;
    uint32_t a = u & 0x7fffffffu;
    if (a > 0x7f800000u) return (uint16_t)(sign | 0x7e00u | ((a >> 13) & 0x3ffu));  // NaN
    if (a >= 0x477ff000u) return (uint16_t)(sign | 0x7c00u);   // >= 65520 rounds to inf (also inf)
    if (a < 0x38800000u) {                                     // < 2^-14: subnormal or zero
        if (a < 0x33000000u) return (uint16_t)sign;            // < 2^-25 -> 0 (2^-25 itself ties to even = 0)
        // value = a_float ; result mantissa = rne(a_float * 2^24)
        uint32_t e = a >> 23;                    // biased exponent (102..112)
        uint32_t m = (a & 0x7fffffu) | 0x800000u;
        uint32_t shift = 126u - e;               // 14..24 : drop this many bits of the 24-bit mantissa
        uint32_t r = m >> shift;
        uint32_t rem = m & ((1u << shift) - 1u);
        uint32_t half = 1u << (shift - 1);
        if (rem > half || (rem == half && (r & 1u))) r++;
        return (uint16_t)(sign | r);
    }
    uint32_t r = a - 0x38000000u;                // rebias exponent (127 -> 15)
    uint32_t lsb = (r >> 13) & 1u;
    r += 0xfffu + lsb;
    return (uint16_t)(sign | (r >> 13));
}

B2_HD float half_to_float(uint16_t h, int dtype) { return dtype ? fp16_to_float(h) : bf16_to_float(h); }
B2_HD uint16_t float_to_half(float f, int dtype) { return dtype ? float_to_fp16(f) : float_to_bf16(f); }

// ---------------------------------------------------------------- quantise (a6) / dequantise (a11)
// factor = MAX / float(max_half)            (one fp32 division per (plane, token))
B2_HD float quant_factor(float maxq, float row_max) { return fdiv(maxq, row_max); }

// symbol = int8( round_half_even( x * factor + MAX ) ), NaN -> 0
B2_HD uint32_t quant_symbol(float x, float factor, float maxq) {
    const float v = fadd(fmul(x, factor), maxq);
#if defined(__CUDA_ARCH__)
    const uint32_t q = (uint32_t)__float2int_rn(v);       // round-half-even; NaN -> 0; +-inf saturate
#else
    const float r = frint(v);
    const uint32_t q = (r >= -1.0f && r <= 1000.0f) ? (uint32_t)(int)r : 0xffffffffu;
#endif
    // valid symbols are 0..2*MAX <= 30; NaN / +-inf rows give 0, as torch's float->int8 cast does on x86
    return q <= 30u ? q : 0u;
}

// The same symbol without the range check, for factors made by quant_factor_safe.  Why that is enough: rows whose
// maximum is finite and large enough give |x * f| <= MAX (1 + 2^-22), hence symbols 0..2 MAX; a NaN row maximum gives
// f = NaN and an infinite one f = 0, both of which already yield in-range symbols (F2I(NaN) = 0; finite x -> MAX,
// x = +-inf -> inf * 0 = NaN -> 0); the only factor that can leave the range is f = +inf (row maximum zero or so
// small that MAX / max overflows), where the checked quantiser returns 0 for every element (x != 0 -> +-inf ->
// saturated -> 0; x == 0 -> NaN -> 0) -- exactly what f = NaN produces.  So replacing an infinite factor by NaN keeps
// every symbol bit-identical and makes the check redundant.
B2_HD float quant_factor_safe(float maxq, float row_max) {
    const float f = fdiv(maxq, row_max);
    return (f2u(f) & 0x7fffffffu) == 0x7f800000u ? u2f(0x7fc00000u) : f;
}
B2_HD uint32_t quant_symbol_nc(float x, float factor, float maxq) {
#if defined(__CUDA_ARCH__)
    return (uint32_t)__float2int_rn(fadd(fmul(x, factor), maxq));
#else
    return quant_symbol(x, factor, maxq);
#endif
}

// LUT entry: (sym - C) / C ; value = lut * float(max_half)
B2_HD float dequant_lut(uint32_t sym, float cq) { return fdiv(fadd((float)sym, -cq), cq); }
B2_HD float dequant_value(float lut, float row_max) { return fmul(lut, row_max); }

// ---------------------------------------------------------------- CDF normalisation (a7)
// counts n[0..32] over t tokens -> cdf[0..32] as uint16 bit patterns (int16 tensor in the reference).
// Sequential state so a caller can stream it: feed counts in order.
struct CdfAccum {
    double cum;
    float prev;
    float tf;
    B2_HD void init(int t) { cum = 0.0; prev = 0.0f; tf = (float)t; }
    // returns cdf[i] for the i-th call (i = 0..32), then absorbs n_i
    B2_HD uint16_t next(uint32_t i, uint32_t n_i) { return next_p(i, fdiv((float)n_i, tf)); }
    // same, with p_i = fl32(n_i / t) supplied by the caller (e.g. from a per-tile table of n / t)
    B2_HD uint16_t next_p(uint32_t i, float p_i) {
        float r = frint(fmul(prev, 65504.0f));
        uint16_t v = (uint16_t)((uint32_t)(int)r + i);
        cum += (double)p_i;
        prev = (float)cum;
        return v;
    }
};

// The same arithmetic split into value() / absorb(): cdf[i] only changes when a count is absorbed, so a caller whose
// lanes share a loop (one stream per lane) can skip the symbols none of its lanes uses -- absorbing p = 0 leaves cum, its
// fp32 image and therefore rint(image * 65504) untouched.  value(i) == CdfAccum's i-th return value.
struct CdfAccum2 {
    double cum;
    uint32_t R;     // rint(fl32(cum) * 65504)
    B2_HD void init() { cum = 0.0; R = 0u; }
    B2_HD uint32_t value(uint32_t i) const { return (R + i) & 0xffffu; }
    B2_HD void absorb(float p_i) {
        cum += (double)p_i;
        R = (uint32_t)(int)frint(fmul((float)cum, 65504.0f));
    }
};

// ---------------------------------------------------------------- arithmetic encoder (a8)
struct EncState {
    uint32_t low, high, pending;
    uint64_t acc;   // bit accumulator, newest bits at the bottom
    uint32_t nb;    // valid bits in acc (< 32 between calls)
    B2_HD void init() { low = 0u; high = 0xFFFFFFFFu; pending = 0u; acc = 0ull; nb = 0u; }
};

// Sink concept: void put_word(uint32_t w)  -- w holds 32 stream bits, first bit in the MSB.
template <class Sink>
B2_HD void enc_put_bits(EncState& st, uint32_t v, uint32_t k, Sink& sink) {   // 0 <= k <= 32, v < 2^k
    st.acc = (st.acc << k) | (uint64_t)v;
    st.nb += k;
    if (st.nb >= 32u) {
        st.nb -= 32u;
        sink.put_word((uint32_t)(st.acc >> st.nb));
    }
}

template <class Sink>
B2_HD void enc_bit_and_pending(EncState& st, uint32_t bit, Sink& sink) {
    enc_put_bits(st, bit, 1u, sink);
    uint32_t p = st.pending;
    const uint32_t fill = bit ? 0u : 0xFFFFFFFFu;
    while (p) {
        uint32_t k = p < 32u ? p : 32u;
        enc_put_bits(st, k == 32u ? fill : (fill & ((1u << k) - 1u)), k, sink);
        p -= k;
    }
    st.pending = 0u;
}

// code one symbol whose CDF interval is [c_lo, c_lo + width), width >= 1, c_lo + width <= 65536
template <class Sink>
B2_HD void enc_symbol(EncState& st, uint32_t c_lo, uint32_t width, Sink& sink) {
    const uint32_t r = st.high - st.low;                       // span - 1
    const uint32_t c_hi = c_lo + width;
    const uint64_t plo = (uint64_t)r * c_lo + c_lo;            // span * c_lo
    const uint64_t phi = (uint64_t)r * c_hi + c_hi;            // span * c_hi
    uint32_t low = st.low + (uint32_t)(plo >> 16);
    uint32_t high = st.low - 1u + (uint32_t)(phi >> 16);
    // E1/E2: the n leading bits of low and high agree -> they are final
    const uint32_t n = clz32((low ^ high) | 1u);
    if (n) {
        const uint32_t top = low >> (32u - n);
        if (st.pending == 0u) {
            enc_put_bits(st, top, n, sink);
        } else {
            enc_bit_and_pending(st, top >> (n - 1u), sink);
            enc_put_bits(st, top & ((1u << (n - 1u)) - 1u), n - 1u, sink);
        }
        low <<= n;
        high = (high << n) | ((1u << n) - 1u);
    }
    // E3: while low = 01.., high = 10.. the interval straddles the midpoint
    const uint32_t m = clz32((((~low) | high) << 1) | 1u);
    st.pending += m;
    st.low = (low << m) & 0x7FFFFFFFu;
    st.high = (high << m) | 0x80000000u | ((1u << m) - 1u);
}

// ---- production encoder step: same bitstream as enc_symbol, organised for SIMT execution.
// The reference coder delays "pending" (E3) bits until the next agreed bit tells whether they are 01..1 or 10..0.
// That is carry resolution in disguise, so the production coder tracks the ABSOLUTE low instead:
//   x   = window of the absolute low = reference `low` with its MSB flipped while E3 bits are pending
//   rng = reference high - low
// With h = x + (phi - 1) (wrapping), x ^ h equals low ^ high and the E3 pattern below the MSB is unchanged, so the
// shift counts n (E1/E2) and m (E3) come out exactly as in the reference, and EVERY shift -- E1, E2 or E3 -- simply
// moves the MSB of x into the output: out = (out << k) | (x >> (32 - k)), x <<= k, k = n + m.  A pending run that
// resolves to 10..0 shows up as a carry out of x + plo, which is added to the output accumulator (the run 01..1 is
// sitting there and ripples).  No pending counter, no masks, no data-dependent emission branch; termination is
// x + 2^30 with the same carry rule, then the top two bits.
// The accumulator `lo` holds nb < 32 unflushed bits, right aligned, zero above -- except a carry that rippled
// through all nb of them, which then sits at bit nb and, at the next flush, lands one position above the 32-bit
// word being written: the (rare) signal to increment the words already in the row.
struct EncState2 {
    uint32_t x, rng;
    uint32_t lo;     // unflushed output bits
    uint32_t m;      // (number of them) - 32, i.e. -32..-1 between calls: "a word is full" is just m >= 0
    uint32_t w;      // words written to the row so far
    B2_HD void init() { x = 0u; rng = 0xFFFFFFFFu; lo = 0u; m = 0xFFFFFFE0u; w = 0u; }
    B2_HD uint32_t nbits() const { return m & 31u; }
};

// (x << n) with n taken as an unsigned 32-bit count: 0 for n >= 32 (PTX shl clamps; C++ would be undefined)
B2_HD uint32_t shl_clamp(uint32_t x, uint32_t n) {
#if defined(__CUDA_ARCH__)
    uint32_t r;
    asm("shl.b32 %0, %1, %2;" : "=r"(r) : "r"(x), "r"(n));
    return r;
#else
    return n >= 32u ? 0u : x << n;
#endif
}

// add `over` to the number formed by row words [0, w) (word 0 most significant): the carry left the accumulator.
// Only called with w >= 1 (a carry can only ripple into words that exist).
B2_HD void enc_ripple(uint32_t* row, uint32_t w, uint32_t capm1, uint32_t over) {
    do {
        --w;
        uint32_t* q = row + (w < capm1 ? w : capm1);
        const uint32_t v = *q + over;
        *q = v;
        over = v < over ? 1u : 0u;
    } while (over != 0u && w != 0u);
}

// append the top k bits of x (0 <= k <= 31) to the accumulator; flush one word when 32 are available
B2_HD void enc_append(EncState2& st, uint32_t x, uint32_t k, uint32_t* row, uint32_t capm1) {
    const uint32_t hi = funnel_l(st.lo, 0u, k);                 // bits pushed above 32 (incl. a rippled carry)
    const uint32_t lo = funnel_l(x, st.lo, k);
    const uint32_t m = st.m + k;                                // >= 0 (as int32) iff 32 bits are ready; then m = bits left
    const uint32_t word = funnel_r(lo, hi, m & 31u);            // meaningful only when flushing (funnel shifts wrap)
    uint32_t* dst = row + (st.w < capm1 ? st.w : capm1);
    const bool flush = (int32_t)m >= 0;
#if defined(__CUDA_ARCH__)
    // one predicated store: in a warp some lane flushes on nearly every symbol, so a branch here would run for all
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ge.s32 p, %0, 0;\n\t@p st.global.u32 [%1], %2;\n\t}"
                 :: "r"(m), "l"(dst), "r"(word) : "memory");
#else
    if (flush) *dst = word;
#endif
    // hi != 0 only when flushing (otherwise every accumulator bit, the carry bit included, stays inside lo); a bit
    // above the 32-bit word just written is a carry that rippled through all unflushed bits
    const uint32_t over = funnel_r(hi, 0u, m & 31u);
    if (over != 0u) enc_ripple(row, st.w, capm1, over);          // rare
    // flushed bits leave: keep the low m bits.  Without a flush m is "negative" = a huge unsigned count, the clamped
    // shift yields 0 and every bit stays (carry bit too)
    st.lo = lo & ~shl_clamp(0xFFFFFFFFu, m);
    st.w += flush ? 1u : 0u;
    st.m = m | 0xFFFFFFE0u;                                     // (m mod 32) - 32
}

// row: word-addressed output row with capacity `cap` words (stores are clamped to the last word so a
// violated size bound can never write outside the row; the bound itself is proven in DESIGN.md 3.2).
// Row words hold the stream MSB-first in NATIVE order (stream byte 4w+b = bits 31-8b.. of word w): whoever moves the
// row to its final place writes the bytes out (compact_kernel), so the coder spends no byte swap per symbol.
B2_HD void enc_symbol2(EncState2& st, uint32_t c_lo, uint32_t width, uint32_t* row, uint32_t cap) {
    const uint32_t r = st.rng;
    const uint32_t c_hi = c_lo + width;
    const uint32_t plo = (uint32_t)(((uint64_t)r * c_lo + c_lo) >> 16);
    const uint32_t phi = (uint32_t)(((uint64_t)r * c_hi + c_hi) >> 16);   // wraps to 0 when it is 2^32
    const uint32_t h = st.x + phi - 1u;
    uint32_t x;
#if defined(__CUDA_ARCH__)
    // carry out of x + plo: the pending run resolves to 10..0 -- add it to the accumulator
    asm("add.cc.u32 %0, %2, %3;\n\taddc.u32 %1, %4, 0;" : "=r"(x), "=r"(st.lo) : "r"(st.x), "r"(plo), "r"(st.lo));
#else
    x = st.x + plo;
    st.lo += x < plo ? 1u : 0u;
#endif
    // k = n + m in one go: p = position of the first differing bit (n = 31 - p agreed bits above it); below it the
    // E3 run continues while x has 1 and h has 0, so k = 30 - (position of the first bit below p with ~x | h)
    const uint32_t p = bfind32((x ^ h) | 1u);
    const uint32_t f = ((~x) | h) & low_mask(p);
    const uint32_t k = 30u - bfind32(f);                         // <= 18: the coded interval is >= 2^14 wide
    st.x = x << k;
    st.rng = shl_fill1(h, k) - st.x;
    enc_append(st, x, k, row, cap - 1u);
}

// terminate: the reference's final bit + pending run = the top two bits of x + 2^30 (with carry), zero padded to a
// byte; returns the stream's byte length
B2_HD uint32_t enc_finish2(EncState2& st, uint32_t* row, uint32_t cap) {
    const uint32_t capm1 = cap - 1u;
    const uint32_t x = st.x + 0x40000000u;
    st.lo += x < 0x40000000u ? 1u : 0u;
    enc_append(st, x, 2u, row, capm1);
    const uint32_t nb = st.nbits();
    const uint32_t over = st.lo >> nb;                          // a carry that rippled through the whole tail
    if (over) { if (st.w) enc_ripple(row, st.w, capm1, over); st.lo &= ~(0xFFFFFFFFu << nb); }
    const uint32_t full = st.w;
    if (nb) { row[st.w < capm1 ? st.w : capm1] = st.lo << (32u - nb); st.w++; }
    return 4u * full + ((nb + 7u) >> 3);
}

// terminate the stream; returns the number of trailing bits (0..31) still in st.acc (left to the caller
// to write, zero padded to a byte), after the final bit + pending bits were queued.
template <class Sink>
B2_HD uint32_t enc_finish(EncState& st, Sink& sink) {
    st.pending += 1u;
    enc_bit_and_pending(st, st.low < 0x40000000u ? 0u : 1u, sink);
    return st.nb;
}

// ---------------------------------------------------------------- arithmetic decoder (a10)
// Source concept: uint32_t next_word() -- next 32 stream bits (first bit in the MSB), zeros past the end.
struct DecState {
    uint32_t low, high, value;
    uint64_t res;   // bit reservoir, left aligned
    uint32_t rb;    // valid bits in res
};

template <class Src>
B2_HD void dec_refill(DecState& st, Src& src) {
    if (st.rb < 32u) {
        st.res |= (uint64_t)src.next_word() << (32u - st.rb);
        st.rb += 32u;
    }
}

template <class Src>
B2_HD uint32_t dec_take(DecState& st, uint32_t k, Src& src) {   // 1 <= k <= 32
    dec_refill(st, src);
    uint32_t v = (uint32_t)(st.res >> (64u - k));
    st.res <<= k;
    st.rb -= k;
    return v;
}

template <class Src>
B2_HD void dec_init(DecState& st, Src& src) {
    st.low = 0u; st.high = 0xFFFFFFFFu; st.res = 0ull; st.rb = 0u;
    st.value = dec_take(st, 32u, src);
}

// Decode one symbol.  cdf(i) returns the uint16 CDF entry i (0..31) of this stream.
// `last` suppresses the state update after the final symbol of the stream (reference: break at i == N-1).
template <class Src, class CdfFn>
B2_HD uint32_t dec_symbol(DecState& st, Src& src, CdfFn cdf, bool last) {
    const uint32_t r = st.high - st.low;
    const uint32_t off = st.value - st.low;
    uint32_t lo = 0u, hi = 32u;
    uint64_t plo = 0ull, phi = (uint64_t)r + 1ull;              // products at lo / hi  (cdf(32) := 65536)
#pragma unroll
    for (int it = 0; it < 5; ++it) {
        const uint32_t mid = (lo + hi) >> 1;
        const uint32_t c = cdf(mid);
        const uint64_t pm = ((uint64_t)r * c + c) >> 16;        // (span * cdf[mid]) >> 16
        if (pm <= (uint64_t)off) { lo = mid; plo = pm; } else { hi = mid; phi = pm; }
    }
    if (last) return lo;
    uint32_t low = st.low + (uint32_t)plo;
    uint32_t high = st.low - 1u + (uint32_t)phi;
    uint32_t value = st.value;
    const uint32_t n = clz32((low ^ high) | 1u);
    if (n) {
        value = (value << n) | dec_take(st, n, src);
        low <<= n;
        high = (high << n) | ((1u << n) - 1u);
    }
    const uint32_t m = clz32((((~low) | high) << 1) | 1u);
    if (m) {
        value = ((value << m) ^ 0x80000000u) | dec_take(st, m, src);
        low = (low << m) & 0x7FFFFFFFu;
        high = (high << m) | 0x80000000u | ((1u << m) - 1u);
    }
    st.low = low; st.high = high; st.value = value;
    return lo;
}

// ---- production decoder step: same symbols as dec_symbol, organised for SIMT execution.
//  * state is (low, rng, off) with off = value - low.  Both E1/E2 and E3 renormalisation steps then act on off as a
//    plain left shift that pulls in stream bits (the E3 "value -= 2^30" cancels against low's cleared MSB), so the
//    decoder never materialises `value` and needs no MSB flip.
//  * stream bits come from a two-word window (cur : nxt) with a bit position pos < 32: the next k <= 18 bits are
//    funnel_l(t, x, k) with t = funnel_l(nxt, cur, pos); a refill is `cur = nxt; nxt = next word; pos -= 32`.
//  * symbol search: fixed-depth and branch-free (warp lanes never diverge; a data-dependent walk was measured
//    2x slower because a warp pays for its longest lane), see dec_symbol2.
struct DecState2 {
    uint32_t x, span, off; // x: window of the absolute low (enc_symbol2); span = high - low + 1 (0 means 2^32)
    uint32_t cur, nxt;     // stream words (big-endian bit order), nxt is the look-ahead
    uint32_t pos;          // bits of `cur` already consumed (< 32 between symbols)
};

// Word source concept: uint32_t next_be() -- next 4 stream bytes as a big-endian word (aligned load + swap).
template <class Src>
B2_HD void dec_refill2(DecState2& st, Src& src) {
    if (st.pos >= 32u) {
        st.cur = st.nxt;
        st.nxt = src.next_be();
        st.pos -= 32u;
    }
}

// `skip` = number of leading bytes of the first aligned word that belong to the previous stream (0..3)
template <class Src>
B2_HD void dec_init2(DecState2& st, Src& src, uint32_t skip) {
    st.x = 0u; st.span = 0u;
    st.cur = src.next_be();
    st.nxt = src.next_be();
    st.pos = 8u * skip;
    st.off = funnel_l(st.nxt, st.cur, st.pos);        // first 32 stream bits (value, low = 0)
    st.pos += 32u;
    dec_refill2(st, src);
}

B2_HD uint32_t umulhi32(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}

// Search key ~ floor((value - low) * 2^32 / span): its top 16 bits are the reference's count
//   count = ((value - low + 1) * 2^16 - 1) / span
// to within +-1 (one MUFU.RCP instead of a 64-bit division; the low bits only break ties), so  e[i] <= key  with
// e[i] = cdf[i] << 16 is the count-domain compare cdf[i] <= count.  F2I.U32 saturates, NaN gives 0.
// `span` is a uint32 (0 stands for 2^32: the guess is then arbitrary and the exactness check repairs it).
B2_HD uint32_t dec_key_approx(uint32_t off, uint32_t span) {
#if defined(__CUDA_ARCH__)
    float rc;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(__uint2float_rn(span)));     // one MUFU.RCP; span > 2^30
    return __float2uint_rz(__uint2float_rn(off) * (rc * 4294967296.0f));
#else
    if (span == 0u) return 0u;
    const float q = ((float)off / (float)span) * 4294967296.0f;
    return q >= 4294967040.0f ? 0xFFFFFFFFu : (uint32_t)q;
#endif
}

// The decoder reads the stream's CDF as a table of 33 words  e[i] = cdf[i] << 16  (e[32] = 0xFFFFFFFF):
//   * compares in the count domain become  e[i] <= (count << 16 | 0xFFFF);
//   * (span * cdf[i]) >> 16  ==  umulhi(span, e[i])  for span < 2^32: one IMAD.HI, no 64-bit arithmetic.
B2_HD uint32_t dec_table_entry(uint32_t i, uint32_t cdf16) { return i < 32u ? (cdf16 << 16) : 0xFFFFFFFFu; }

// exact interval products for symbol s from the pre-shifted table, valid for every state (incl. span = 2^32)
B2_HD void dec_exact_products(const uint32_t* e, uint32_t r, uint32_t s, uint32_t* plo, uint32_t* phi) {
    const uint32_t c0 = e[s] >> 16;
    const uint32_t c1 = s >= 31u ? 0x10000u : (e[s + 1u] >> 16);
    *plo = (uint32_t)(((uint64_t)r * c0 + c0) >> 16);
    *phi = (uint32_t)(((uint64_t)r * c1 + c1) >> 16);          // 2^32 wraps to 0 (the reference's uint32 maths)
}

#if defined(__CUDACC__)
// one lower-bound step on a 32-bit shared-memory address: a += 4*STEP iff table[a/4 + STEP] <= key
template <int STEP>
__device__ __forceinline__ void dec_search_steps(uint32_t& a, uint32_t key) {
    uint32_t ev;
    asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(ev) : "r"(a), "n"(STEP * 4));
    a = ev <= key ? a + STEP * 4 : a;
    if constexpr (STEP > 1) dec_search_steps<STEP / 2>(a, key);
}
#endif

// Decode one symbol; returns 4 * symbol (the byte offset of its entry in a 32-bit table, which is what the table
// walk produces and what the caller's dequantisation LUT wants).  NSTEPS = 5 searches symbols 0..31, NSTEPS = 4
// symbols 0..15 (planes with <= 16 bins only ever code symbols 0..14).
//  1. s~ = max{ s : cdf[s] <= count~ } by a fixed-depth, branch-free lower-bound search in the count domain
//     (per step: one LDS off a running pointer, one compare, one predicated add).
//  2. plo = umulhi(span, e[s]), phi = umulhi(span, e[s+1]) -- needed for the state update anyway.  The symbol is exact
//     iff plo <= off < phi (the reference's rule cdf[s] <= count  <=>  (span*cdf[s])>>16 <= off), checked in wrapping
//     uint32 arithmetic as (off - plo) < (phi - plo).
//  3. count~ is within +-1 of count, so the check almost never fails; when it does (or when span = 2^32, where umulhi
//     cannot be used, or s = 31 whose upper bound is 2^16) a slow path recomputes the products with 64-bit arithmetic
//     and walks to the exact symbol.  The result is exact whatever the approximation did.
template <int NSTEPS, class Src>
B2_HD uint32_t dec_symbol2(DecState2& st, Src& src, const uint32_t* e, bool last) {
    const uint32_t span = st.span;                               // 0 when the interval is the whole 32-bit range
    const uint32_t r = span - 1u;
    const uint32_t off = st.off;
    const uint32_t cnt16 = dec_key_approx(off, span);
    constexpr uint32_t kTop = (1u << NSTEPS) - 1u;               // highest searchable symbol
#if defined(__CUDA_ARCH__)
    // the table lives in shared memory: walk it with a 32-bit shared address so that every step is
    // LDS [a + imm] / ISETP / select, and the symbol index falls out of the address
    const uint32_t a0 = (uint32_t)__cvta_generic_to_shared(e);
    uint32_t a = a0;
    dec_search_steps<(1 << (NSTEPS - 1))>(a, cnt16);
    uint32_t s4 = a - a0;                                        // 4 * symbol: the table walk yields a byte offset
    uint32_t e0, e1;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(e0) : "r"(a));
    asm volatile("ld.shared.u32 %0, [%1+4];" : "=r"(e1) : "r"(a));
#else
    const uint32_t* a = e;
#pragma unroll
    for (int step = 1 << (NSTEPS - 1); step > 0; step >>= 1) a = a[step] <= cnt16 ? a + step : a;
    uint32_t s4 = 4u * (uint32_t)(a - e);
    const uint32_t e0 = a[0], e1 = a[1];
#endif
    uint32_t plo = umulhi32(span, e0);
    uint32_t phi = umulhi32(span, e1);
    if ((uint32_t)(off - plo) >= (uint32_t)(phi - plo) || (NSTEPS == 5 && s4 == 124u)) {
        uint32_t s = s4 >> 2;
        dec_exact_products(e, r, s, &plo, &phi);
        while (off < plo && s > 0u) { --s; dec_exact_products(e, r, s, &plo, &phi); }
        while (s < kTop && (uint32_t)(off - plo) >= (uint32_t)(phi - plo)) { ++s; dec_exact_products(e, r, s, &plo, &phi); }
        s4 = 4u * s;
    }
    if (last) return s4;
    // renormalisation exactly as in enc_symbol2: all k = n + m shifts (E1/E2/E3) at once, on the absolute-low window
    const uint32_t x = st.x + plo;
    const uint32_t h = st.x + phi - 1u;
    const uint32_t p = bfind32((x ^ h) | 1u);
    const uint32_t f = ((~x) | h) & low_mask(p);
    const uint32_t k = 30u - bfind32(f);                         // <= 18 for 16-bit CDFs
    const uint32_t t = funnel_l(st.nxt, st.cur, st.pos);         // the next 32 unread stream bits
    st.off = funnel_l(t, off - plo, k);                          // ((off - plo) << k) | next k bits
    st.pos += k;
    st.x = x << k;
    st.span = (phi - plo) << k;                                  // (high - low + 1) << k; 2^32 wraps to 0
    dec_refill2(st, src);
    return s4;
}

// ---------------------------------------------------------------- rANS coder ("B2KV" container version 2)
// The arithmetic-coder bitstream is this build's own (the reference's coder lives in the absent torchac_cuda wheel;
// SURVEY.md 8c), so container version 2 carries a cheaper entropy coder over the SAME per-stream 16-bit CDF section,
// the same stream order and the same lengths section: range-ANS with a 32-bit state and 16-bit renormalisation.
//
// Normative stream format, one stream = one (plane, channel) over one group of g <= 256 tokens, CDF c[0..32]
// (c[32] := 65536), start(s) = c[s], freq(s) = c[s+1] - c[s] >= 1:
//   encoder   x = 2^16; for i = g-1 .. 0:  s = sym[i]; if (x >> 16) >= freq(s): push halfword (x & 0xffff), x >>= 16;
//             x = (x / freq(s)) << 16 | ... i.e.  x = ((x / f) << 16) + (x mod f) + start(s)
//   bytes     x as a little-endian uint32, then the pushed halfwords in REVERSE push order, each little-endian;
//             length = 4 + 2 * pushes (always even)
//   decoder   x = LE32(bytes[0..4)); for i = 0 .. g-1:  slot = x & 0xffff; s = max{ s : c[s] <= slot }; emit s;
//             x = freq(s) * (x >> 16) + slot - start(s); if x < 2^16: x = (x << 16) | next LE16
//             after the last symbol x == 2^16 again (a free integrity check of the stream).
// No carries, no pending bits, no bit counting: one multiply per decoded symbol, one division per encoded symbol,
// at most one 16-bit renormalisation step per symbol.  Cost: the 32-bit final state instead of the arithmetic
// coder's ~2 termination bits (+19 bits per stream on average, measured).
constexpr uint32_t kRansLow = 1u << 16;

// decoder table entry i (0..31): (c[i] << 16) | freq(i).  The search compares entries against (slot << 16) | 0xffff
// (c[i] <= slot  <=>  entry <= key, because freq <= 0xffff), and the winning entry carries start and freq.
B2_HD uint32_t rans_table_entry(uint32_t c_i, uint32_t c_next) { return (c_i << 16) | ((c_next - c_i) & 0xffffu); }

// x / f and x mod f for x < f << 16, 1 <= f < 2^16, by plain division: the host statement of the encoder step, for
// tests/hostsim only.  No kernel calls it or rans_enc_symbol, so neither has a device branch; the kernels run rans_put
// below, whose quotient is a biased reciprocal estimate plus one fix-up.
inline uint32_t rans_divmod(uint32_t x, uint32_t f, uint32_t* rem) {
    *rem = x % f;
    return x / f;
}

// Encoder step on the state alone; `emit(h)` receives the low halfword when the state must shrink first.
template <class Emit>
inline void rans_enc_symbol(uint32_t& x, uint32_t start, uint32_t freq, Emit&& emit) {
    const uint32_t xh = x >> 16;
    if (xh >= freq) { emit(x & 0xffffu); x = xh; }
    uint32_t r;
    const uint32_t q = rans_divmod(x, freq, &r);
    x = (q << 16) + r + start;
}

#if defined(__CUDACC__)
// rANS encoder step as the kernels run it (same arithmetic as rans_enc_symbol, laid out for issue slots):
//   * the state shrinks by one halfword when it must; halfword number k (counted downwards: nk = -k) lands at
//     row_end + 2 * nk - 2, so the row's tail holds the halfwords in decode order.  The address is one unpredicated
//     IMAD.WIDE, only the 16-bit store and the count are predicated;
//   * q = x / f by one reciprocal biased low and one fix-up.  The estimate is q or q - 1 for EVERY x < f << 16,
//     1 <= f < 2^16: tests/devsim runs this function on an H100 at both ends of every quotient bucket [q f, q f + f)
//     (the estimate is monotone in x, the quotient constant on a bucket), 8.6e9 steps, and compares with integer
//     division: no wrong state; the fix-up is taken at every x = q f and, for f > 1, at no x = q f + f - 1 (NVIDIA H100
//     80GB HBM3, 700 W limit; tests/test_gpu_rans_edges.py::test_rans_put_exhaustive_sweep);
//   * x' = (q << 16) + (x - q f) + start  ==  x + start + q * (65536 - f).
__device__ __forceinline__ void rans_put(uint32_t& x, int32_t& nk, const uint16_t* row_end, uint32_t start, uint32_t freq) {
    const uint32_t xh = x >> 16;
    asm volatile(
        "{\n\t.reg .pred p;\n\t.reg .b64 ad;\n\t"
        "setp.ge.u32 p, %2, %3;\n\t"
        "mad.wide.s32 ad, %1, 2, %4;\n\t"
        "@p st.global.u16 [ad+-2], %0;\n\t"
        "@p add.s32 %1, %1, -1;\n\t"
        "selp.b32 %0, %2, %0, p;\n\t"
        "}"
        : "+r"(x), "+r"(nk) : "r"(xh), "r"(freq), "l"(row_end) : "memory");
    float rc;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(__uint2float_rn(freq)));
    const uint32_t q = __float2uint_rz(__uint2float_rz(x) * (rc * 0.99999952316284179688f));   // floor(x / f) or one less
    // With m = 65536 - f:  a = q m + x;  x - q f = a - (q << 16);  x' = a + start, plus m when the estimate was one short.
    // Six integer instructions (m, a, r, compare, add, predicated add) where "negate f, r, compare, q + 1, select, x +
    // start, m, multiply-add" took eight (ncu, round 2).
    const uint32_t m = 65536u - freq;
    const uint32_t a = q * m + x;
    const uint32_t r = a - (q << 16);
    x = a + start;
    if (r >= freq) x += m;
}
#endif

// Decoder state: x plus a two-word window over the stream's halfwords (aligned 32-bit loads, one word of look-ahead).
// `sel` is the PRMT selector that builds (x << 16) | next halfword from (x, cur): 0x1054 takes cur's low half,
// 0x1076 its high half.
struct RansDec {
    uint32_t x, cur, nxt, sel;
};

B2_HD uint32_t prmt32(uint32_t a, uint32_t b, uint32_t sel) {
#if defined(__CUDA_ARCH__)
    return __byte_perm(a, b, sel);
#else
    const uint64_t v = ((uint64_t)b << 32) | a;
    uint32_t r = 0;
    for (int i = 0; i < 4; ++i) r |= (uint32_t)((v >> (8u * ((sel >> (4 * i)) & 7u))) & 0xffu) << (8 * i);
    return r;
#endif
}

// Word source concept: uint32_t next_le() -- next aligned 4 stream bytes as a little-endian word.
// `odd` = 1 when the stream starts at the upper halfword of its first aligned word.
template <class Src>
B2_HD void rans_dec_init(RansDec& st, Src& src, uint32_t odd) {
    const uint32_t w0 = src.next_le();
    const uint32_t w1 = src.next_le();
    st.x = funnel_r(w0, w1, 16u * odd);             // the 4 state bytes, wherever they start
    st.cur = w1;
    st.nxt = src.next_le();
    st.sel = 0x1054u + 0x22u * odd;
}

// pull one halfword into the state (x < 2^16 on entry)
template <class Src>
B2_HD void rans_dec_renorm(RansDec& st, Src& src) {
    if (st.x < kRansLow) {
        st.x = prmt32(st.x, st.cur, st.sel);
        const bool wrap = st.sel == 0x1076u;
        st.sel ^= 0x22u;
        if (wrap) { st.cur = st.nxt; st.nxt = src.next_le(); }
    }
}

// Decode one symbol from table pk[0..31] (rans_table_entry); NSTEPS = 5 searches symbols 0..31, NSTEPS = 4
// symbols 0..15.  Plain-C++ restatement used by the host tests; the kernels run the same arithmetic with the two top
// search levels held in registers (codec.cu, rans_decode_stream).
template <int NSTEPS, class Src>
B2_HD uint32_t rans_dec_symbol(RansDec& st, Src& src, const uint32_t* pk) {
    const uint32_t key = (st.x << 16) | 0xffffu;
    uint32_t s = 0;
#pragma unroll
    for (int step = 1 << (NSTEPS - 1); step > 0; step >>= 1) s = pk[s + step] <= key ? s + step : s;
    const uint32_t e = pk[s];
    st.x = (e & 0xffffu) * (st.x >> 16) + ((key - e) >> 16);
    rans_dec_renorm(st, src);
    return s;
}

// ---------------------------------------------------------------- container layout (host + device)
B2_HD int64_t align16(int64_t x) { return (x + 15) & ~(int64_t)15; }

struct Layout {
    int64_t off_cdf, off_maxes, off_lengths, off_payload;
    int32_t ngroups;
};

// Containers of version 1 / 2:  header | cdf i16[2L][C][33] | maxes | lengths i32[G][2L][C] | payload.
// Compact container, version 3 (chunks of <= 256 tokens, i.e. one group):
//   header | nb u8[2L] (pad to 16) | maxes | half-lengths u8[2L][C] | payload
// The per-stream CDF row is gone: the CDF is a function of the stream's symbol histogram and the token count (CdfAccum),
// and every stream carries that histogram in front of its rANS bytes (stream header, below); a stream's byte length
// (even, <= 230) is stored halved in one byte.  nb(plane) = 2 * (bins // 2) is the number of symbols a plane can emit.
// off_cdf is the first byte after the header in both layouts (the nb map in version 3).
// ppl: planes per layer, 2 (keys, values) or 1 (a latent KV: version 4 is the compact layout with L planes).
B2_HD Layout make_layout(int L, int C, int t, int compact = 0, int ppl = 2) {
    Layout lo;
    const int64_t NL = (int64_t)ppl * L;
    lo.ngroups = (t + kGroup - 1) / kGroup;
    lo.off_cdf = 64;
    if (compact) {
        lo.off_maxes = align16(lo.off_cdf + NL);
        lo.off_lengths = align16(lo.off_maxes + NL * t * 2);
        lo.off_payload = align16(lo.off_lengths + (int64_t)lo.ngroups * NL * C);
    } else {
        lo.off_maxes = align16(lo.off_cdf + NL * C * kLp * 2);
        lo.off_lengths = align16(lo.off_maxes + NL * t * 2);
        lo.off_payload = align16(lo.off_lengths + (int64_t)lo.ngroups * NL * C * 4);
    }
    return lo;
}

// ---------------------------------------------------------------- version-3 stream header
// stream = [mask: ceil(nb / 8) bytes, little-endian, bit s set <=> symbol s occurs]
//          [one count byte per set bit, ascending, EXCEPT the last set bit: its count is t - (sum of the others)]
//          [one zero byte if the header length is odd]  [LE32 rANS state] [LE16 renormalisation words ...]
// Counts that are stored are <= 255 (two or more symbols share <= 256 tokens); a lone symbol's count (up to 256) is
// implied.  Header length <= 4 + 31 + 1 = 36 bytes.
constexpr int kHdrMax = 36;
B2_HD int hdr_mask_bytes(int nb) { return (nb + 7) >> 3; }
B2_HD uint32_t hdr_len(uint32_t mask, int nb) {
#if defined(__CUDA_ARCH__)
    const uint32_t nz = (uint32_t)__popc(mask);
#else
    uint32_t nz = 0;
    for (uint32_t m = mask; m; m &= m - 1u) ++nz;
#endif
    const uint32_t h = (uint32_t)hdr_mask_bytes(nb) + (nz ? nz - 1u : 0u);
    return h + (h & 1u);
}
// Host-side restatement (tests): build the header of one stream from its counts; returns its length.
inline uint32_t hdr_write_host(uint8_t* dst, const uint32_t* cnt, int nb) {
    uint32_t mask = 0;
    for (int i = 0; i < nb; ++i) mask |= (cnt[i] ? 1u : 0u) << i;
    const int mb = hdr_mask_bytes(nb);
    for (int b = 0; b < mb; ++b) dst[b] = (uint8_t)(mask >> (8 * b));
    int last = -1;
    for (int i = 0; i < nb; ++i) if (cnt[i]) last = i;
    uint32_t pos = (uint32_t)mb;
    for (int i = 0; i < nb; ++i) if (cnt[i] && i != last) dst[pos++] = (uint8_t)cnt[i];
    if (pos & 1u) dst[pos++] = 0;
    return pos;
}

}  // namespace b200kv
