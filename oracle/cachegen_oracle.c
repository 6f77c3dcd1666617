/*
 * oracle/cachegen_oracle.c -- CPU restatement of the LMCache v0.1.2 CacheGen hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under lmcache_b200/ may import, link or call this
 * file; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs use it, and only as the checker / the timed CPU baseline.
 *
 * Each function cites the reference file:line (relative to the reference tree) it follows.
 *
 * Parity status
 *   quantise / dequantise / CDF / SHA-256 chain : PINNED against golden vectors generated
 *       from the reference's own functions (tests/golden/make_golden.py).
 *   arithmetic-coder bitstream                  : "parity unpinned" -- the coder lives in
 *       the un-vendored PyPI wheel `torchac_cuda >= 0.2.5` (setup.py:19), absent from
 *       the reference tree.  This file restates the published torchac-lineage algorithm
 *       (32-bit low/high, 16-bit CDF precision, E1/E2/E3 renormalisation with pending
 *       bits, MSB-first packing; SURVEY.md Appendix A.3/A.4) and anchors it on the
 *       reference call sites cachegen_encoder.py:241-262,301-316 and
 *       cachegen_decoder.py:52-66.
 *   rANS bitstream, version-3 stream framing    : this build's own wire format (container
 *       versions 2 and 3, include/b200kv.h), restated here independently of the kernels:
 *       same status as the arithmetic coder ("parity unpinned"), same anchors.  What a
 *       version-3 reader evaluates -- the CDF as a function of the stored histogram,
 *       oracle_cdf_from_counts -- IS pinned to the reference-made CDF goldens.
 *
 * Build: gcc -O2 -fopenmp -ffp-contract=off -fno-fast-math -shared -fPIC (oracle/Makefile).
 * -ffp-contract=off matters: the reference rounds the fp32 mul and add separately
 * (cachegen_encoder.py:57-59); an FMA flips symbols.
 */
#include <math.h>
#include <omp.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORACLE_LP 33          /* CDF entries per stream: int(bins.max()) + 1 = 33  (cachegen_encoder.py:287-289) */
#define ORACLE_MAXSYM 31      /* Lp - 2 */

/* ------------------------------------------------------------------ half <-> float */

static inline float bf16_to_f32(uint16_t h) {
    uint32_t u = (uint32_t)h << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
}

static inline uint16_t f32_to_bf16_rne(float f) { /* torch .to(bfloat16): round-nearest-even, NaN kept quiet */
    uint32_t u;
    memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x0040u);
    uint32_t lsb = (u >> 16) & 1u;
    u += 0x7fffu + lsb;
    return (uint16_t)(u >> 16);
}

static inline float fp16_to_f32(uint16_t h) {
    _Float16 x;
    memcpy(&x, &h, 2);
    return (float)x;
}

static inline uint16_t f32_to_fp16_rne(float f) {
    _Float16 x = (_Float16)f;
    uint16_t h;
    memcpy(&h, &x, 2);
    return h;
}

/* dtype: 0 = bfloat16, 1 = float16 */
static inline float half_to_f32(uint16_t h, int dtype) { return dtype ? fp16_to_f32(h) : bf16_to_f32(h); }
static inline uint16_t f32_to_half(float f, int dtype) { return dtype ? f32_to_fp16_rne(f) : f32_to_bf16_rne(f); }

/* ------------------------------------------------------------------ a6: quantise
 * Follows cachegen_encoder.py:40-61 (torch_quant_vectorized) on the K / V planes produced
 * by _split_kv (:76-91) and concatenated K-layers-then-V-layers (:284-285).
 *
 *   MAX  = bins // 2 - 1                       (fp32 tensor arithmetic)
 *   max1 = amax(|x|, dim=channel)              (kept in the input half dtype)
 *   f    = MAX / max1                          (fp32 true division)
 *   q    = round_half_even(x * f + MAX)        (fp32 mul, fp32 add, separately rounded)
 *   sym  = int8(q)                             (NaN -> 0, observed on torch CPU)
 *
 * x     : [L, 2, t, C] half, element strides given (channel stride 1)
 * sym   : [2L, t, C] int8, plane nl = kv * L + l
 * maxes : [2, L, t] half bits (maxes[0] = max_tensors_key, maxes[1] = max_tensors_value)
 */
void oracle_quantize(const uint16_t* x, int dtype, int L, int t, int C,
                     int64_t sL, int64_t sKV, int64_t sT,
                     const float* key_bins, const float* value_bins,
                     int8_t* sym, uint16_t* maxes) {
#pragma omp parallel for collapse(2) schedule(static)
    for (int kv = 0; kv < 2; ++kv) {
        for (int l = 0; l < L; ++l) {
            const float bins = kv ? value_bins[l] : key_bins[l];
            const float MAX = floorf(bins / 2.0f) - 1.0f;
            for (int tok = 0; tok < t; ++tok) {
                const uint16_t* row = x + l * sL + kv * sKV + (int64_t)tok * sT;
                /* amax(|x|): propagates NaN like torch.amax */
                float m = 0.0f;
                uint16_t mbits = 0;
                int isnan_row = 0;
                for (int c = 0; c < C; ++c) {
                    uint16_t a = row[c] & 0x7fffu;
                    float af = half_to_f32(a, dtype);
                    if (af != af) { isnan_row = 1; mbits = a; }
                    else if (!isnan_row && af > m) { m = af; mbits = a; }
                }
                maxes[((int64_t)kv * L + l) * t + tok] = mbits;
                const float mf = half_to_f32(mbits, dtype);
                const float f = MAX / mf;
                int8_t* out = sym + (((int64_t)kv * L + l) * t + tok) * C;
                for (int c = 0; c < C; ++c) {
                    float v = half_to_f32(row[c], dtype);
                    volatile float p = v * f;          /* separately rounded (no FMA) */
                    float q = nearbyintf(p + MAX);
                    out[c] = (q != q) ? 0 : (int8_t)(int)q;
                }
            }
        }
    }
}

/* ------------------------------------------------------------------ a7: CDF
 * In-tree spec of what torchac_cuda.calculate_cdf is meant to compute:
 *   compute_cdf.process_batch (cachegen_encoder.py:185-196):
 *       counts = one_hot(sym).sum(tokens) / ntokens      (fp32 true division, torch CPU)
 *       cdf_f  = cumsum(counts).roll(1); cdf_f[:,0] = 0  (torch CPU cumsum accumulates in
 *                                                          double and stores fp32 per step)
 *   _convert_to_int_and_normalize(cdf_f, True) (cachegen_encoder.py:95-126):
 *       cdf = int16( round_half_even( cdf_f * (2^16 - (Lp-1)) ) ) + arange(Lp)
 * Values >= 32768 wrap into the int16 bit pattern (coder reads them as uint16); entry 32
 * (= 65536) wraps to 0 and is never read (coder uses 0x10000 for max_symbol).
 *
 * sym : [NL, t, C] int8 ; cdf : [NL, C, 33] int16
 */
static void cdf_row(const uint32_t* n, int t, int16_t* o) {
    double cum = 0.0;
    float prev = 0.0f; /* cdf_f[i] = cumsum[i-1] */
    for (int i = 0; i < ORACLE_LP; ++i) {
        float scaled = prev * 65504.0f;             /* 2^16 - (Lp - 1) */
        float r = nearbyintf(scaled);
        o[i] = (int16_t)(uint16_t)((uint32_t)(int32_t)r + (uint32_t)i);
        float p = (float)n[i] / (float)t;
        cum += (double)p;
        prev = (float)cum;
    }
}

/* the histogram the CDF is computed from: counts [NL, C, 33] uint32 (entry 32 is always 0) */
void oracle_counts(const int8_t* sym, int NL, int t, int C, uint32_t* counts) {
#pragma omp parallel for schedule(static)
    for (int64_t s = 0; s < (int64_t)NL * C; ++s) {
        const int nl = (int)(s / C), c = (int)(s % C);
        uint32_t* n = counts + s * ORACLE_LP;
        memset(n, 0, sizeof(uint32_t) * ORACLE_LP);
        for (int tok = 0; tok < t; ++tok) {
            int v = sym[((int64_t)nl * t + tok) * C + c];
            if (v >= 0 && v < ORACLE_LP) n[v]++;
        }
    }
}

/* the CDF as a function of the histogram and the token count (what a version-3 container's reader evaluates) */
void oracle_cdf_from_counts(const uint32_t* counts, int64_t nstreams, int t, int16_t* cdf) {
#pragma omp parallel for schedule(static)
    for (int64_t s = 0; s < nstreams; ++s) cdf_row(counts + s * ORACLE_LP, t, cdf + s * ORACLE_LP);
}

/* ------------------------------------------------------------------ B2KV version 3: streams that carry their histogram
 * (this build's own wire format, include/b200kv.h; no reference counterpart -- the reference stores the CDF tensor).
 * stream = [mask: ceil(nb/8) bytes LE, bit s <=> counts[s] > 0] [count byte per set bit, ascending, except the last set
 *           bit (implied: t - sum of the others)] [zero byte if the header length is odd] [rANS stream]
 * counts : [NL, C, 33] uint32; nb : [NL] symbols per plane; rans_len : [NL, C] int32; rans : concatenated rANS streams.
 * Returns the packed payload size; half_len[s] = (header + rANS bytes) / 2. */
static int v3_header(const uint32_t* n, int nb, uint8_t* h) {
    uint32_t mask = 0;
    int last = -1, pos, mb = (nb + 7) / 8;
    for (int i = 0; i < nb; ++i) if (n[i]) { mask |= 1u << i; last = i; }
    for (int b = 0; b < mb; ++b) h[b] = (uint8_t)(mask >> (8 * b));
    pos = mb;
    for (int i = 0; i < nb; ++i) if (n[i] && i != last) h[pos++] = (uint8_t)n[i];
    if (pos & 1) h[pos++] = 0;
    return pos;
}

int64_t oracle_v3_pack(const uint32_t* counts, const int32_t* nb, int NL, int C, const int32_t* rans_len,
                       const uint8_t* rans, uint8_t* out, int64_t cap, uint8_t* half_len) {
    int64_t o = 0, r = 0;
    for (int64_t s = 0; s < (int64_t)NL * C; ++s) {
        uint8_t h[40];
        const int hl = v3_header(counts + s * ORACLE_LP, nb[s / C], h);
        const int64_t total = hl + rans_len[s];
        if (o + total > cap || (total & 1) || total / 2 > 255) return -1;
        memcpy(out + o, h, (size_t)hl);
        memcpy(out + o + hl, rans + r, (size_t)rans_len[s]);
        half_len[s] = (uint8_t)(total / 2);
        o += total;
        r += rans_len[s];
    }
    return o;
}

/* inverse; returns the number of rANS bytes written to `rans`, or -1 on a malformed header */
int64_t oracle_v3_unpack(const uint8_t* payload, int64_t n, const uint8_t* half_len, const int32_t* nb, int NL, int C,
                         int t, uint32_t* counts, int32_t* rans_len, uint8_t* rans) {
    int64_t o = 0, r = 0;
    for (int64_t s = 0; s < (int64_t)NL * C; ++s) {
        const int b = nb[s / C], mb = (b + 7) / 8;
        const int64_t total = 2 * (int64_t)half_len[s];
        uint32_t mask = 0, sum = 0, *c = counts + s * ORACLE_LP;
        int nz = 0, last = -1, pos = mb, hl;
        if (o + total > n || total < mb) return -1;
        for (int k = 0; k < mb; ++k) mask |= (uint32_t)payload[o + k] << (8 * k);
        if (b < 32) mask &= (1u << b) - 1u;
        memset(c, 0, sizeof(uint32_t) * ORACLE_LP);
        for (int i = 0; i < b; ++i) if (mask >> i & 1) { ++nz; last = i; }
        hl = mb + (nz ? nz - 1 : 0);
        hl += hl & 1;
        if (hl + 4 > total || nz == 0) return -1;
        for (int i = 0; i < b; ++i)
            if ((mask >> i & 1) && i != last) { c[i] = payload[o + pos++]; sum += c[i]; if (!c[i]) return -1; }
        if (sum >= (uint32_t)t) return -1;
        c[last] = (uint32_t)t - sum;
        rans_len[s] = (int32_t)(total - hl);
        memcpy(rans + r, payload + o + hl, (size_t)(total - hl));
        r += total - hl;
        o += total;
    }
    return o == n ? r : -1;
}

void oracle_cdf(const int8_t* sym, int NL, int t, int C, int16_t* cdf) {
#pragma omp parallel for schedule(static)
    for (int64_t s = 0; s < (int64_t)NL * C; ++s) {
        const int nl = (int)(s / C), c = (int)(s % C);
        uint32_t n[ORACLE_LP];
        memset(n, 0, sizeof n);
        for (int tok = 0; tok < t; ++tok) {
            int v = sym[((int64_t)nl * t + tok) * C + c];
            if (v >= 0 && v < ORACLE_LP) n[v]++;
        }
        cdf_row(n, t, cdf + s * ORACLE_LP);
    }
}

/* ------------------------------------------------------------------ a8: arithmetic encoder
 * torchac-lineage coder (SURVEY.md Appendix A.3); one independent stream per (nl, c) over
 * a group of g <= 256 consecutive tokens, coded in token order with the stream's static
 * CDF (cachegen_encoder.py:245-252).  Rows are then compacted in (nl, c) row-major order
 * (collect_bytes, cachegen_encoder.py:225-238).
 */
typedef struct {
    uint8_t* p;
    int64_t n, cap;
    uint8_t cache;
    int count;
} bitw_t;

static inline void bw_append(bitw_t* w, int bit) {
    w->cache = (uint8_t)((w->cache << 1) | (bit & 1));
    if (++w->count == 8) {
        if (w->n < w->cap) w->p[w->n] = w->cache;
        w->n++;
        w->count = 0;
        w->cache = 0;
    }
}

static inline void bw_bit_and_pending(bitw_t* w, int bit, uint64_t* pending) {
    bw_append(w, bit);
    while (*pending) { bw_append(w, !bit); (*pending)--; }
}

/* encode one stream; returns byte count (may exceed cap: caller checks) */
static int64_t ac_encode_stream(const uint16_t* cdf, const int8_t* sym, int64_t sym_stride, int g,
                                uint8_t* out, int64_t cap) {
    bitw_t w = {out, 0, cap, 0, 0};
    uint32_t low = 0, high = 0xFFFFFFFFu;
    uint64_t pending = 0;
    for (int i = 0; i < g; ++i) {
        const int s = sym[i * sym_stride];
        const uint64_t span = (uint64_t)high - (uint64_t)low + 1;
        const uint32_t c_lo = cdf[s];
        const uint32_t c_hi = (s == ORACLE_MAXSYM) ? 0x10000u : cdf[s + 1];
        high = (low - 1) + (uint32_t)((span * c_hi) >> 16);
        low = low + (uint32_t)((span * c_lo) >> 16);
        for (;;) {
            if (high < 0x80000000u) {
                bw_bit_and_pending(&w, 0, &pending);
                low <<= 1; high = (high << 1) | 1u;
            } else if (low >= 0x80000000u) {
                bw_bit_and_pending(&w, 1, &pending);
                low <<= 1; high = (high << 1) | 1u;
            } else if (low >= 0x40000000u && high < 0xC0000000u) {
                pending++;
                low = (low << 1) & 0x7FFFFFFFu;
                high = (high << 1) | 0x80000001u;
            } else break;
        }
    }
    pending++;
    bw_bit_and_pending(&w, (low < 0x40000000u) ? 0 : 1, &pending);
    while (w.count) bw_append(&w, 0);   /* zero-pad to a byte */
    return w.n;
}

/* Encode one token group.
 *   cdf     : [NL, C, 33] int16
 *   sym     : [NL, t_total, C] int8 ; the group is tokens [tok0, tok0 + g)
 *   out     : compact bytestream (capacity cap); lengths : [NL, C] int32
 * Returns total bytes N, or -1 if cap would be exceeded.
 */
int64_t oracle_encode_group(const int16_t* cdf, const int8_t* sym, int NL, int t_total, int tok0, int g,
                            int C, uint8_t* out, int64_t cap, int32_t* lengths) {
    const int64_t nstreams = (int64_t)NL * C;
    const int64_t rowcap = 2 * (int64_t)g + 8;          /* <= 16 bits / symbol + flush */
    uint8_t* stage = (uint8_t*)malloc((size_t)(nstreams * rowcap));
    if (!stage) return -2;
#pragma omp parallel for schedule(static)
    for (int64_t s = 0; s < nstreams; ++s) {
        const int nl = (int)(s / C), c = (int)(s % C);
        const int8_t* sp = sym + ((int64_t)nl * t_total + tok0) * C + c;
        lengths[s] = (int32_t)ac_encode_stream((const uint16_t*)(cdf + s * ORACLE_LP), sp, C, g,
                                               stage + s * rowcap, rowcap);
    }
    int64_t total = 0;
    for (int64_t s = 0; s < nstreams; ++s) total += lengths[s];
    if (total > cap) { free(stage); return -1; }
    int64_t off = 0;
    for (int64_t s = 0; s < nstreams; ++s) {           /* collect_bytes: row-major, no padding */
        memcpy(out + off, stage + s * rowcap, (size_t)lengths[s]);
        off += lengths[s];
    }
    free(stage);
    return total;
}

/* ------------------------------------------------------------------ a10: arithmetic decoder
 * SURVEY.md Appendix A.4; stream (nl,c) occupies [P - len, P) with P the inclusive prefix sum
 * of the flattened lengths (cachegen_decoder.py:52-66).  Bits past a stream's end read as 0.
 */
typedef struct {
    const uint8_t* p;
    int64_t n, pos;
    uint8_t cache;
    int bits;
} bitr_t;

static inline void br_get(bitr_t* r, uint32_t* value) {
    if (r->bits == 0) {
        if (r->pos == r->n) { *value <<= 1; return; }
        r->cache = r->p[r->pos++];
        r->bits = 8;
    }
    *value = (*value << 1) | ((r->cache >> (r->bits - 1)) & 1u);
    r->bits--;
}

static void ac_decode_stream(const uint16_t* cdf, const uint8_t* in, int64_t n, int g, uint8_t* out,
                             int64_t out_stride) {
    bitr_t r = {in, n, 0, 0, 0};
    uint32_t low = 0, high = 0xFFFFFFFFu, value = 0;
    for (int i = 0; i < 32; ++i) br_get(&r, &value);
    for (int i = 0; i < g; ++i) {
        const uint64_t span = (uint64_t)high - (uint64_t)low + 1;
        const uint16_t count = (uint16_t)((((uint64_t)value - (uint64_t)low + 1) * 0x10000u - 1) / span);
        int left = 0, right = ORACLE_MAXSYM + 1;
        while (left + 1 < right) {
            int m = (left + right) / 2;
            uint16_t v = cdf[m];
            if (v < count) left = m; else if (v > count) right = m; else { left = m; break; }
        }
        const int s = left;
        out[i * out_stride] = (uint8_t)s;
        if (i == g - 1) break;
        const uint32_t c_lo = cdf[s];
        const uint32_t c_hi = (s == ORACLE_MAXSYM) ? 0x10000u : cdf[s + 1];
        high = (low - 1) + (uint32_t)((span * c_hi) >> 16);
        low = low + (uint32_t)((span * c_lo) >> 16);
        for (;;) {
            if (low >= 0x80000000u || high < 0x80000000u) {
                low <<= 1; high = (high << 1) | 1u;
                br_get(&r, &value);
            } else if (low >= 0x40000000u && high < 0xC0000000u) {
                low = (low << 1) & 0x7FFFFFFFu;
                high = (high << 1) | 0x80000001u;
                value -= 0x40000000u;
                br_get(&r, &value);
            } else break;
        }
    }
}

/* out_sym : [NL, t_total, C] uint8, group written at tokens [tok0, tok0+g) */
void oracle_decode_group(const int16_t* cdf, const uint8_t* bytes, const int32_t* lengths, int NL,
                         int t_total, int tok0, int g, int C, uint8_t* out_sym) {
    const int64_t nstreams = (int64_t)NL * C;
    int64_t* start = (int64_t*)malloc(sizeof(int64_t) * (size_t)nstreams);
    int64_t acc = 0;
    for (int64_t s = 0; s < nstreams; ++s) { start[s] = acc; acc += lengths[s]; }
#pragma omp parallel for schedule(static)
    for (int64_t s = 0; s < nstreams; ++s) {
        const int nl = (int)(s / C), c = (int)(s % C);
        ac_decode_stream((const uint16_t*)(cdf + s * ORACLE_LP), bytes + start[s], lengths[s], g,
                         out_sym + ((int64_t)nl * t_total + tok0) * C + c, C);
    }
    free(start);
}

/* ------------------------------------------------------------------ a8/a10, container version 2: rANS
 * The coder of B2KV container version 2 (lmcache_b200/csrc/ac_core.cuh, "rANS coder"): same per-stream CDF, same
 * stream order (collect_bytes, cachegen_encoder.py:225-238), same lengths section and prefix-sum addressing
 * (cachegen_decoder.py:52-66) as the arithmetic coder above; only the bytes of a stream differ.  Like the arithmetic
 * coder's bitstream it is "parity unpinned" against the reference (torchac_cuda absent) -- it is this build's format,
 * restated here independently of the product code (plain division / modulo, a byte stack) as the checker.
 *   encoder: x = 2^16; for i = g-1..0: f = c[s+1]-c[s]; if (x >> 16) >= f: push16(x & 0xffff), x >>= 16;
 *            x = ((x / f) << 16) + (x % f) + c[s]
 *   stream : LE32(x), then the pushed halfwords in reverse push order (LE16 each)
 *   decoder: x = LE32; per symbol: slot = x & 0xffff; s = max{s: c[s] <= slot}; x = f*(x>>16) + slot - c[s];
 *            if x < 2^16: x = (x << 16) | next LE16
 */
static int64_t rans_encode_stream(const uint16_t* cdf, const int8_t* sym, int64_t sym_stride, int g,
                                  uint8_t* out, int64_t cap) {
    uint16_t stack[512];
    int k = 0;
    uint32_t x = 1u << 16;
    for (int i = g - 1; i >= 0; --i) {
        const int s = sym[i * sym_stride];
        const uint32_t c_lo = cdf[s];
        const uint32_t c_hi = (s == ORACLE_MAXSYM) ? 0x10000u : cdf[s + 1];
        const uint32_t f = c_hi - c_lo;
        if ((x >> 16) >= f) { if (k < 512) stack[k] = (uint16_t)(x & 0xffffu); k++; x >>= 16; }
        x = ((x / f) << 16) + (x % f) + c_lo;
    }
    const int64_t n = 4 + 2 * (int64_t)k;
    if (n <= cap && k <= 512) {
        out[0] = (uint8_t)x; out[1] = (uint8_t)(x >> 8); out[2] = (uint8_t)(x >> 16); out[3] = (uint8_t)(x >> 24);
        for (int j = 0; j < k; ++j) {
            const uint16_t h = stack[k - 1 - j];
            out[4 + 2 * j] = (uint8_t)h; out[5 + 2 * j] = (uint8_t)(h >> 8);
        }
    }
    return n;
}

/* returns the final state (2^16 for an intact stream) */
static uint32_t rans_decode_stream(const uint16_t* cdf, const uint8_t* in, int64_t n, int g, uint8_t* out,
                                   int64_t out_stride) {
    uint32_t x = 0;
    for (int i = 0; i < 4; ++i) x |= (uint32_t)(i < n ? in[i] : 0) << (8 * i);
    int64_t p = 4;
    for (int i = 0; i < g; ++i) {
        const uint32_t slot = x & 0xffffu;
        int s = 0;
        while (s < ORACLE_MAXSYM && (uint32_t)cdf[s + 1] <= slot && cdf[s + 1] != 0) s++;   /* cdf[32] wraps to 0 */
        out[i * out_stride] = (uint8_t)s;
        const uint32_t c_lo = cdf[s];
        const uint32_t c_hi = (s == ORACLE_MAXSYM) ? 0x10000u : cdf[s + 1];
        x = (c_hi - c_lo) * (x >> 16) + slot - c_lo;
        if (x < (1u << 16)) {
            const uint32_t h = (uint32_t)(p < n ? in[p] : 0) | ((uint32_t)(p + 1 < n ? in[p + 1] : 0) << 8);
            x = (x << 16) | h;
            p += 2;
        }
    }
    return x;
}

int64_t oracle_encode_group_rans(const int16_t* cdf, const int8_t* sym, int NL, int t_total, int tok0, int g,
                                 int C, uint8_t* out, int64_t cap, int32_t* lengths) {
    const int64_t nstreams = (int64_t)NL * C;
    const int64_t rowcap = 2 * (int64_t)g + 8;
    uint8_t* stage = (uint8_t*)malloc((size_t)(nstreams * rowcap));
    if (!stage) return -2;
#pragma omp parallel for schedule(static)
    for (int64_t s = 0; s < nstreams; ++s) {
        const int nl = (int)(s / C), c = (int)(s % C);
        const int8_t* sp = sym + ((int64_t)nl * t_total + tok0) * C + c;
        lengths[s] = (int32_t)rans_encode_stream((const uint16_t*)(cdf + s * ORACLE_LP), sp, C, g,
                                                 stage + s * rowcap, rowcap);
    }
    int64_t total = 0;
    for (int64_t s = 0; s < nstreams; ++s) total += lengths[s];
    if (total > cap) { free(stage); return -1; }
    int64_t off = 0;
    for (int64_t s = 0; s < nstreams; ++s) {
        memcpy(out + off, stage + s * rowcap, (size_t)lengths[s]);
        off += lengths[s];
    }
    free(stage);
    return total;
}

/* returns the number of streams whose final state is not 2^16 (0 for intact input) */
int64_t oracle_decode_group_rans(const int16_t* cdf, const uint8_t* bytes, const int32_t* lengths, int NL,
                                 int t_total, int tok0, int g, int C, uint8_t* out_sym) {
    const int64_t nstreams = (int64_t)NL * C;
    int64_t* start = (int64_t*)malloc(sizeof(int64_t) * (size_t)nstreams);
    int64_t acc = 0, bad = 0;
    for (int64_t s = 0; s < nstreams; ++s) { start[s] = acc; acc += lengths[s]; }
#pragma omp parallel for schedule(static) reduction(+ : bad)
    for (int64_t s = 0; s < nstreams; ++s) {
        const int nl = (int)(s / C), c = (int)(s % C);
        const uint32_t xf = rans_decode_stream((const uint16_t*)(cdf + s * ORACLE_LP), bytes + start[s], lengths[s], g,
                                               out_sym + ((int64_t)nl * t_total + tok0) * C + c, C);
        bad += xf != (1u << 16);
    }
    free(start);
    return bad;
}

/* ------------------------------------------------------------------ a11: dequantise + assemble
 * do_dequantize (cachegen_decoder.py:24-35): C_l = bins//2 - 1 ; x = ((q - C_l) / C_l) * max
 * with three separately rounded fp32 ops, then the blob is re-interleaved to [L,2,t,H,D] and
 * cast .to(bfloat16) (vllm) / .to(float16) (huggingface) (cachegen_decoder.py:182-200).
 *
 * sym   : [2L, t, C] uint8 ; maxes : [2, L, t] half bits of dtype `max_dtype`
 * out   : half bits of dtype `out_dtype`, element strides oL/oKV/oT (channel stride 1)
 */
void oracle_dequantize(const uint8_t* sym, const uint16_t* maxes, int max_dtype, int L, int t, int C,
                       const float* key_bins, const float* value_bins, int out_dtype, uint16_t* out,
                       int64_t oL, int64_t oKV, int64_t oT) {
#pragma omp parallel for collapse(2) schedule(static)
    for (int kv = 0; kv < 2; ++kv) {
        for (int l = 0; l < L; ++l) {
            const float bins = kv ? value_bins[l] : key_bins[l];
            const float Cq = floorf(bins / 2.0f) - 1.0f;
            for (int tok = 0; tok < t; ++tok) {
                const float m = half_to_f32(maxes[((int64_t)kv * L + l) * t + tok], max_dtype);
                const uint8_t* in = sym + (((int64_t)kv * L + l) * t + tok) * C;
                uint16_t* o = out + l * oL + kv * oKV + (int64_t)tok * oT;
                for (int c = 0; c < C; ++c) {
                    volatile float a = (float)in[c] - Cq;
                    volatile float b = a / Cq;
                    float v = b * m;
                    o[c] = f32_to_half(v, out_dtype);
                }
            }
        }
    }
}

/* ------------------------------------------------------------------ a1: SHA-256 prefix chain
 * LMCacheEngine._hash / _prefix_hash (cache_engine.py:58-96):
 *   h_i = sha256( ascii_hex(h_{i-1}) || bytes(tokens[i*cs:(i+1)*cs]) ).hexdigest(),  h_{-1} = ""
 * Token bytes are the tensor's native little-endian dtype.  The tail partial chunk is hashed.
 */
static const uint32_t K256[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
    0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
    0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
    0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
    0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
    0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
    0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};

static inline uint32_t rotr32(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }

static void sha256_block(uint32_t st[8], const uint8_t blk[64]) {
    uint32_t w[64];
    for (int i = 0; i < 16; ++i)
        w[i] = ((uint32_t)blk[4 * i] << 24) | ((uint32_t)blk[4 * i + 1] << 16) | ((uint32_t)blk[4 * i + 2] << 8) |
               blk[4 * i + 3];
    for (int i = 16; i < 64; ++i) {
        uint32_t s0 = rotr32(w[i - 15], 7) ^ rotr32(w[i - 15], 18) ^ (w[i - 15] >> 3);
        uint32_t s1 = rotr32(w[i - 2], 17) ^ rotr32(w[i - 2], 19) ^ (w[i - 2] >> 10);
        w[i] = w[i - 16] + s0 + w[i - 7] + s1;
    }
    uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
    for (int i = 0; i < 64; ++i) {
        uint32_t t1 = h + (rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25)) + ((e & f) ^ (~e & g)) + K256[i] + w[i];
        uint32_t t2 = (rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
        h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

static void sha256_two_part(const uint8_t* p1, size_t n1, const uint8_t* p2, size_t n2, uint8_t digest[32]) {
    uint32_t st[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    const size_t total = n1 + n2;
    uint8_t blk[64];
    size_t fill = 0;
    for (size_t i = 0; i < total; ++i) {
        blk[fill++] = (i < n1) ? p1[i] : p2[i - n1];
        if (fill == 64) { sha256_block(st, blk); fill = 0; }
    }
    blk[fill++] = 0x80;
    if (fill > 56) { while (fill < 64) blk[fill++] = 0; sha256_block(st, blk); fill = 0; }
    while (fill < 56) blk[fill++] = 0;
    uint64_t bits = (uint64_t)total * 8;
    for (int i = 0; i < 8; ++i) blk[56 + i] = (uint8_t)(bits >> (56 - 8 * i));
    sha256_block(st, blk);
    for (int i = 0; i < 8; ++i) {
        digest[4 * i] = (uint8_t)(st[i] >> 24); digest[4 * i + 1] = (uint8_t)(st[i] >> 16);
        digest[4 * i + 2] = (uint8_t)(st[i] >> 8); digest[4 * i + 3] = (uint8_t)st[i];
    }
}

/* tokens: raw little-endian token bytes (n_tokens * elem_size); digests: [n_chunks][32] raw.
 * Returns n_chunks = ceil(n_tokens / chunk_size). */
int oracle_sha256_chain(const uint8_t* tokens, int64_t n_tokens, int elem_size, int chunk_size, uint8_t* digests) {
    static const char hexd[] = "0123456789abcdef";
    uint8_t prefix[64];
    size_t plen = 0;
    int n = 0;
    for (int64_t i = 0; i < n_tokens; i += chunk_size, ++n) {
        int64_t cnt = n_tokens - i < chunk_size ? n_tokens - i : chunk_size;
        uint8_t* d = digests + 32 * (size_t)n;
        sha256_two_part(prefix, plen, tokens + i * elem_size, (size_t)cnt * elem_size, d);
        for (int k = 0; k < 32; ++k) { prefix[2 * k] = hexd[d[k] >> 4]; prefix[2 * k + 1] = hexd[d[k] & 15]; }
        plen = 64;
    }
    return n;
}

/* torchrun exports OMP_NUM_THREADS=1; the CPU baseline legs of bench.py ask for all host threads explicitly. */
int oracle_set_threads(int n) {
    if (n > 0) omp_set_num_threads(n);
    return omp_get_max_threads();
}

int oracle_version(void) { return 3; }
