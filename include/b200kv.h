/*
 * b200kv.h -- C ABI of libb200kv.so, the H100 (sm_90a) KV-cache store/load hot path.
 *
 * This is the drop-in boundary for ONE path of LMCache v0.1.2 (paths below are relative to the
 * reference tree): CacheGen encode / decode, the chunked token-id SHA-256 prefix hash, and the
 * GPU <-> pinned-host mover.  Each entry point names the reference interface it replaces.
 *
 * Conventions
 *   - every function is extern "C", returns int: 0 = ok, <0 = error (b200kv_last_error() gives the
 *     message for the calling thread).  No torch / pybind types: raw device/host pointers, sizes,
 *     element strides and a cudaStream_t passed as void*.
 *   - the caller owns every buffer.  Work is enqueued on `stream` and is asynchronous unless the
 *     function says otherwise.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails.
 *
 * KV layout: element (l, kv, tok, h, d) of the chunk/blob lives at
 *       base + (l*sL + kv*sKV + tok*sT + h*sH + d) * es bytes           (d is contiguous)
 *   or, when `planes` is non-NULL, at planes[kv*L + l] + (tok*sT + h*sH + d) * es bytes,
 *   es = the element size of kv->dtype: 2 for B200KV_DT_BF16 / _FP16, 1 for B200KV_DT_U8 / _FP8_E4M3 / _FP8_E5M2.
 *   vllm blob [L,2,T,H,D]: sL=2*T*H*D sKV=T*H*D sT=H*D sH=D ; huggingface [L,2,H,T,D]: sT=D sH=T*D.
 *   The planes form takes the 2L tensors of the engine's kv tuple as they are
 *   (replaces the stack/stack/stack/permute + split/.contiguous() copies of
 *   lmcache/cache_engine.py:98-118,131-161).
 */
#ifndef B200KV_H_
#define B200KV_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200KV_VERSION 4           /* ABI version; 2: b200kv_kv_desc.slot_map; 3: coder selection, decode status, total_bytes;
                                    * 4: compact container (B200KV_CODER_RANS_COMPACT), b200kv_container_layout_v,
                                    *    b200kv_sha256_chain_ready.  Added since without changing anything that
                                    *    existed (the number stays 4; a caller that needs them looks the symbols up,
                                    *    e.g. dlsym): b200kv_decode_plan / b200kv_decode_layers, b200kv_plane_offsets,
                                    *    b200kv_plane_offsets_device, b200kv_copy_batch_async,
                                    *    b200kv_encode_layers_workspace_bytes / b200kv_encode_layers_plan /
                                    *    b200kv_encode_layers / b200kv_encode_layers_finish, b200kv_decode_plan_heads,
                                    *    b200kv_lossless_layout / b200kv_lossless_workspace_bytes / b200kv_lossless_encode /
                                    *    b200kv_lossless_decode (container versions 5 and 6), b200kv_lossless_plane_offsets /
                                    *    b200kv_lossless_plane_offsets_device / b200kv_lossless_decode_plan /
                                    *    b200kv_lossless_decode_layers (b200kv_lossless_decode_plan_t),
                                    *    b200kv_lossless_decode_plan_heads,
                                    *    b200kv_lossless_encode_layers_workspace_bytes /
                                    *    b200kv_lossless_encode_layers_plan / b200kv_lossless_encode_layers /
                                    *    b200kv_lossless_encode_layers_finish (b200kv_lossless_encode_plan_t),
                                    *    b200kv_lm_open_begin / b200kv_lm_read_ranges / b200kv_lm_close_handles,
                                    *    b200kv_lm_server_num_handles, b200kv_pack_chunks_layers /
                                    *    b200kv_unpack_chunks_layers, b200kv_rope_table / b200kv_rope_shift.
                                    *    B200KV_MAX_PLANES went from 128 to 256 (models of up to 128 layers): the row
                                    *    width of b200kv_plane_offsets_device, B200KV_MAX_PLANES + 1, and the size of
                                    *    b200kv_encode_plan_t, 256 -> 512 words, changed with it; a caller takes them
                                    *    from this header.  b200kv_decode_plan_t keeps its 256 words. */
#define B200KV_CODER_AC 0          /* payload = torchac-lineage arithmetic coder; container version 1 */
#define B200KV_CODER_RANS 1        /* payload = rANS, 32-bit state / 16-bit renormalisation; container version 2 */
#define B200KV_CODER_RANS_COMPACT 2 /* rANS as in version 2, compact side information; container version 3 (chunks of
                                     * <= 256 tokens): the per-stream CDF row (66 B) is replaced by the symbol histogram it
                                     * is a function of, carried sparsely in front of the stream's rANS bytes (~5 B at the
                                     * headline entropy), the int32 stream length by one byte */
#define B200KV_CONTAINER_VERSION(coder) ((coder) + 1) /* "B2KV" wire container version (b200kv_header.version) */
#define B200KV_ENCODE_HINT_MID_ENTROPY 0x200  /* OR into `coder` of b200kv_encode_chunks: the caller expects more than ~1.2
                                               * payload bits per symbol (e.g. the previous call's sizes said so); the
                                               * compaction kernel then keeps its full-size shared-memory stage (tiles of
                                               * 10+ KB).  Output bytes are identical either way. */
#define B200KV_KV_LATENT 0x100  /* OR into b200kv_kv_desc.dtype: the KV holds ONE plane per layer (multi-head latent attention,
                                 * e.g. DeepSeek-V2/V3's [T, 576] latent vector), not a (K, V) pair.  Plane l of layer l is
                                 * planes[l], or base + (l*sL + tok*sT + h*sH + d) * es (sKV unused); it is coded with layer l's
                                 * KEY bins.  Such a descriptor reads and writes container version 4 = version 3 with L planes
                                 * instead of 2L (rANS-compact coder only; refused with coders 0 and 1).  OR it into `coder`
                                 * wherever a coder names a container: b200kv_container_layout_v, b200kv_encode_workspace_bytes
                                 * and the decode calls (coder B200KV_CODER_RANS_COMPACT | B200KV_KV_LATENT = version 4; a
                                 * decode whose coder and destination disagree on the flag is refused).  Added without
                                 * changing anything that existed: every entry point below that names "2L" means L for a latent
                                 * descriptor, and b200kv_decode_plan_heads refuses a latent destination. */
#define B200KV_KV_PAGED_SPLIT 0x400  /* OR into b200kv_kv_desc.dtype: a paged (K, V) cache in the split layout of vLLM's
                                      * PagedAttention / xFormers backend (PagedAttention.split_kv_cache), where a token's
                                      * row is not contiguous.  Added without changing anything that existed
                                      * (b200kv_version() stays 4).  planes[kv*L + l] are layer l's key and value block
                                      * tensors, slot_map is required (slot s: block b = s / bs, offset o = s % bs), sT
                                      * carries bs (block_size), sL / sKV / sH are unused.  With x = 16 / es (8 for 16-bit
                                      * elements, 16 for one-byte ones), element (h, d) of slot s is, in elements,
                                      *   key   [nb, H, D/x, bs, x]: planes[l]     + ((b*H + h)*(D/x) + d/x)*bs*x + o*x + d%x
                                      *   value [nb, H, D, bs]:      planes[L + l] + ((b*H + h)*D + d)*bs + o
                                      * Only the mover takes it: b200kv_pack_chunks / _unpack_chunks / _pack_chunks_layers /
                                      * _unpack_chunks_layers, vllm chunk layout (hf_layout 0), D % x == 0.  Every CacheGen and
                                      * lossless entry point refuses it (< 0, nothing enqueued): stage the KV into a blob with
                                      * b200kv_pack_chunks first.  Not combined with B200KV_KV_LATENT. */
#define B200KV_LP 33            /* CDF entries per stream (cachegen_encoder.py:287-289: int(bins.max()) + 1) */
#define B200KV_GROUP_TOKENS 256 /* CACHEGEN_GPU_MAX_TOKENS_PER_CHUNK (cachegen_basics.py:13) */
#define B200KV_MAX_PLANES 256   /* 2 * nlayers upper bound: models of up to 128 layers */
#define B200KV_DT_BF16 0
#define B200KV_DT_FP16 1
/* One-byte elements (FP8 KV caches): torch.uint8 (vLLM 0.6.x allocates its fp8 cache so), torch.float8_e4m3fn,
 * torch.float8_e5m2.  Added without changing anything that existed (b200kv_version() stays 4).  The mover and the
 * lossless codec take them; the CacheGen entry points (b200kv_encode_chunks, b200kv_encode_layers_plan,
 * b200kv_decode_chunks, b200kv_decode_plan, b200kv_decode_plan_heads) refuse them (< 0, nothing enqueued): their
 * quantiser would round values FP8 has already rounded. */
#define B200KV_DT_U8 2
#define B200KV_DT_FP8_E4M3 3
#define B200KV_DT_FP8_E5M2 4

#define B200KV_READ_SLACK 640   /* bytes that must be readable past the end of every container handed to the decoder */
#define B200KV_MAGIC 0x564B3242u /* "B2KV" little-endian */
#define B200KV_HEADER_BYTES 64

typedef struct b200kv_kv_desc {
    const void* base;          /* used when planes == NULL */
    const void* const* planes; /* HOST array of 2L device pointers, index kv*L + l; or NULL */
    int64_t sL, sKV, sT, sH;   /* element strides (sL/sKV ignored when planes != NULL) */
    int32_t L, H, D;           /* layers, kv heads, head size; channels C = H*D */
    int32_t dtype;             /* B200KV_DT_* of the KV elements */
    const int64_t* slot_map;   /* DEVICE array or NULL.  Paged KV (vLLM's slot_mapping, lmcache-vllm's
                                * lmcache_store_kv / lmcache_retrieve_kv, docs LLM_Engine.rst:91-109): token i of the call
                                * (tok_begin + i for encode, dst_tok[j] + i for decode) lives in row slot_map[i] of every
                                * plane, i.e. `tok` in the address formula above is replaced by slot_map[tok].  The codec
                                * and pack / unpack kernels gather / scatter through it, so the paged cache is read and
                                * written in place. */
} b200kv_kv_desc;

/* Wire container of one encoded chunk ("B2KV" v1 / v2 / v3).  All sections 16-byte aligned, little-endian.
 * Logical content == CacheGenGPUEncoderOutput (cachegen_basics.py:109-142):
 *   cdf [2L,C,33] int16 | max_tensors_key/value [2,L,t] half | per <=256-token group:
 *   bytestream_lengths [2L,C] int32 + bytestream (streams in (nl,c) row-major order, no padding).
 * Flat instead of pickled CUDA tensors so it can be produced on the device in one buffer and moved
 * with one async copy.
 * Versions 1 and 2 differ ONLY in the bytes of each stream inside `bytestream`: the reference's coder lives in the
 * un-vendored torchac_cuda wheel, so the bitstream is this build's own (SURVEY.md 8c).  v1 = 32-bit binary arithmetic
 * coder (torchac lineage, MSB-first bits); v2 = rANS over the same 16-bit CDFs: LE32 final state, then LE16
 * renormalisation words in decode order (normative description: lmcache_b200/csrc/ac_core.cuh).
 * Version 3 (one <= 256-token group per container) has no CDF section:
 *   header | nb u8[2L] (pad to 16) | maxes | half-lengths u8[2L][C] | bytestream
 * nb(plane) = 2 * (bins(plane) // 2) = the symbols a plane can emit (16 or 32 for the reference's bin tables).  Every
 * stream of the bytestream is  [mask: ceil(nb / 8) bytes LE, bit s set <=> symbol s occurs in the stream]
 *   [one count byte per set bit, ascending, except the LAST set bit, whose count is ntokens - (sum of the others)]
 *   [a zero byte if that makes the length even] [the version-2 rANS stream];  half-lengths[c] = bytes of all that / 2.
 * The CDF the reference keeps (cachegen_encoder.py:287-290) is a function of these counts n_s and t = ntokens:
 *   cdf[i] = int16(rint(fl32(sum_{k<i} fl32(n_k / t), accumulated in double) * 65504) + i)      (in-tree spec :95-126)
 * so CacheGenGPUEncoderOutput.from_bytes rebuilds the identical tensor, and the decoder evaluates it on the device.
 * Version 4 (B200KV_KV_LATENT: one plane per layer) is version 3 with P = L planes instead of 2L:
 *   header | nb u8[L] (pad to 16) | maxes [L, t] | half-lengths u8[L][C] | bytestream (streams in plane order)
 * header.L is the number of layers (= planes). */
typedef struct b200kv_header {
    uint32_t magic, version;
    uint32_t L, H, D;
    uint32_t ntokens, ngroups;
    uint32_t max_dtype;        /* dtype of the max tensors (== input dtype) */
    uint64_t payload_bytes;    /* all groups' bytestreams, concatenated in group order */
    uint64_t total_bytes;      /* header + sections + payload */
    uint32_t status;           /* 0 = ok; nonzero = encoder detected an internal overflow */
    uint32_t reserved[3];
} b200kv_header;

/* Section offsets of a container with the given shape (pure arithmetic, host side). */
typedef struct b200kv_layout {
    int64_t off_cdf, off_maxes, off_lengths, off_payload;
    int64_t fixed_bytes;       /* == off_payload */
    int64_t max_total_bytes;   /* worst case: payload at 2 bytes/symbol + flush */
} b200kv_layout;

int b200kv_version(void);
const char* b200kv_last_error(void);
/* number of CUDA devices visible, or <0 with an error: lets callers fail loudly up front */
int b200kv_device_count(void);

int b200kv_container_layout(int32_t L, int32_t H, int32_t D, int32_t ntokens, b200kv_layout* out);   /* versions 1, 2 */
/* Same for the container `coder` produces (B200KV_CODER_RANS_COMPACT: off_cdf is the nb map, there is no CDF section). */
int b200kv_container_layout_v(int32_t L, int32_t H, int32_t D, int32_t ntokens, int32_t coder, b200kv_layout* out);

/* Host side: where each plane's streams lie in a version-3 container in host memory (its fixed sections are read, nothing
 * else): out[0..2L], plane p (keys of layer p, then values of layer p - L) is bytes [out[p], out[p+1]) of the container,
 * out[0] = layout.off_payload.  Returns 0, 1 when the half-lengths do not add up to header.total_bytes (damaged), <0 for
 * anything that is not a version-3 container. */
int b200kv_plane_offsets(const void* container, int64_t nbytes, int64_t* out, int32_t n_out);
/* Same for n containers in DEVICE memory, container j at containers + j*stride (the encoder's output, before it leaves the
 * device): row j of out (DEVICE or mapped-host int64[n][B200KV_MAX_PLANES + 1]) gets the 2L + 1 offsets and zeros in the
 * rest of the row, or -1 in its
 * entry 0 for a container that is not version 3, whose header claims fixed sections longer than its total_bytes or than
 * `stride` (nothing past the header is read then), or whose half-lengths do not add up.  Asynchronous on `stream`. */
int b200kv_plane_offsets_device(const void* containers, int64_t stride, int32_t n, int64_t* out, void* stream);

/* Bytes of device scratch b200kv_encode_chunks / b200kv_decode_chunks need for a call. */
int64_t b200kv_encode_workspace_bytes(int32_t L, int32_t H, int32_t D, int32_t chunk_tokens, int32_t n_chunks,
                                      int32_t coder);
int64_t b200kv_decode_workspace_bytes(int32_t L, int32_t H, int32_t D, int32_t chunk_tokens, int32_t n_chunks);

/*
 * CacheGen encode.  Replaces, for n_chunks consecutive chunks in ONE call:
 *   torch_quant_vectorized x2            cachegen_encoder.py:40-61,282-285
 *   torchac_cuda.calculate_cdf x2        cachegen_encoder.py:287-290   (in-tree spec :95-126,185-196)
 *   torchac_cuda.encode_fast_new + collect_bytes per <=256-token group   :225-262,301-316
 *   CacheGenGPUEncoderOutput.to_bytes    cachegen_basics.py:131-136   (container written on device)
 * i.e. the body of CacheGenSerializer.to_bytes (cachegen_encoder.py:353-389).
 *
 * Chunk j covers tokens [tok_begin + j*chunk_tokens, ...) and holds chunk_tokens tokens except the
 * last one, which holds last_chunk_tokens (1..chunk_tokens).  Its container is written at
 * out + j*out_stride (device memory, out_stride >= layout.max_total_bytes or the call fails with
 * the header status set if the payload does not fit).  sizes_out[j] (device or mapped-host memory)
 * receives total_bytes of chunk j, or 0 when the chunk's header carries a nonzero status.
 * key_bins / value_bins: HOST float arrays of length L (make_key_bins / make_value_bins, :339-350).
 * coder: B200KV_CODER_* -- which entropy coder fills the bytestreams (and hence header.version).
 */
int b200kv_encode_chunks(const b200kv_kv_desc* kv, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                         int32_t last_chunk_tokens, const float* key_bins, const float* value_bins, int32_t coder,
                         void* out, int64_t out_stride, uint64_t* sizes_out, void* workspace, int64_t workspace_bytes,
                         void* stream);

/*
 * CacheGen decode.  Replaces, for n_chunks containers in ONE call:
 *   CacheGenGPUEncoderOutput.from_bytes  cachegen_basics.py:138-142   (parsed on the host by caller)
 *   decode_chunk cumsum + torchac_cuda.decode_fast_prefsum            cachegen_decoder.py:52-66
 *   decode_function_gpu / .float()                                     :70-106
 *   do_dequantize x2 + stack/reshape/permute/.to(bf16|fp16)            :24-35,177-200
 * i.e. the body of CacheGenDeserializer.from_bytes (:143-202).
 *
 * containers: DEVICE buffer; container j starts at containers + offsets[j] (HOST int64 array, 16-byte
 * aligned offsets).  Shapes are passed by the caller (it has parsed the headers): all chunks share
 * L/H/D; ntokens[j] (HOST int32 array) tokens each.  Chunk j's tokens are written to `dst` at token
 * index dst_tok[j] (HOST int64 array) using dst's strides; dst->dtype is the output dtype
 * (bf16 for vllm, fp16 for huggingface, cachegen_decoder.py:189-200) and max_dtype the dtype of the
 * stored max tensors.  total_bytes[j] (HOST int64 array) = header.total_bytes of container j and containers_bytes = the
 * size of the `containers` buffer; the call fails unless offsets[j] + total_bytes[j] + B200KV_READ_SLACK <=
 * containers_bytes for every j (the slack bytes may hold anything, e.g. the next container).  Given that, the kernels
 * never read outside the buffer whatever the lengths section says: stream starts are clamped to the payload and a
 * stream reads a bounded number of bytes from its start (a corrupt or truncated blob from a remote tier is a cache
 * miss, not an illegal address).
 * coder = header.version - 1 of the containers (one call, one coder).
 * status_out: NULL, or DEVICE / mapped-host uint32[n_chunks], zeroed by the call and then OR-ed with
 *   1 = a rANS stream did not return to its initial state (payload or CDF bytes damaged),
 *   2 = stream offsets beyond the payload (lengths section damaged); valid once the stream has run,
 *   4 = the container's header.version is not the one `coder` names (B200KV_CODER_RANS_COMPACT | B200KV_KV_LATENT: 4).
 *       The call cannot read the headers before it returns, so it trusts `coder`; a container of another version (e.g.
 *       version 3 into a latent destination) is decoded as if it were one and flagged here: treat it as a miss.
 */
int b200kv_decode_chunks(const void* containers, int64_t containers_bytes, const int64_t* offsets,
                         const int64_t* total_bytes, const int32_t* ntokens, const int64_t* dst_tok, int32_t n_chunks,
                         int32_t max_dtype,
                         int32_t coder, const b200kv_kv_desc* dst, const float* key_bins, const float* value_bins,
                         uint32_t* status_out, void* workspace, int64_t workspace_bytes, void* stream);

/*
 * The same decode in two steps, so that a caller can decode a layer as soon as its bytes have arrived (vLLM's
 * per-layer KV loading: wait_for_layer_load before each attention layer).  b200kv_decode_chunks == plan + layers(0, L).
 *
 * b200kv_decode_plan takes b200kv_decode_chunks' arguments and makes all of its checks, zeroes status_out, writes the
 * chunk descriptors into `workspace` and enqueues the stream-offset kernels (tile sums, tile scan).  Those read the
 * FIXED sections of every container only (header, nb map / CDF rows, maxes, lengths: [0, layout.off_payload)), so the
 * payload may still be on its way.  It records its decisions (the table layout among them) in *plan, caller-owned host
 * memory; the workspace, containers buffer, destination and status_out must stay valid until the last layers call
 * has run on the device.
 *
 * b200kv_decode_layers enqueues the decode of layers [layer_begin, layer_end): planes layer_begin.. (keys) and
 * L + layer_begin.. (values), 0 <= layer_begin < layer_end <= L, and ORs into the plan's status_out.  Any set of
 * calls that covers every layer once writes what b200kv_decode_chunks writes.  A call reads the fixed sections and
 * the payload bytes of its planes' streams; in a version 1, 2 or 3 container nothing past a stream's own bytes reaches
 * an output or a status bit, so the bytes of later planes may be unwritten (codec.cu explains why).  In a version 3
 * container (one group) the streams of plane p are the contiguous range that the half-lengths of planes < p and <= p
 * delimit; containers of several groups (versions 1 / 2 with more than 256 tokens) spread a plane over every group.
 */
typedef struct b200kv_decode_plan_t {
    uint64_t opaque[256];      /* the decode kernel's parameter block; for more than 64 layers its plane table is kept in
                                * the plan's workspace (b200kv_decode_workspace_bytes counts it) */
} b200kv_decode_plan_t;

int b200kv_decode_plan(const void* containers, int64_t containers_bytes, const int64_t* offsets,
                       const int64_t* total_bytes, const int32_t* ntokens, const int64_t* dst_tok, int32_t n_chunks,
                       int32_t max_dtype, int32_t coder, const b200kv_kv_desc* dst, const float* key_bins,
                       const float* value_bins, uint32_t* status_out, void* workspace, int64_t workspace_bytes,
                       b200kv_decode_plan_t* plan, void* stream);
int b200kv_decode_layers(const b200kv_decode_plan_t* plan, int32_t layer_begin, int32_t layer_end, void* stream);

/*
 * b200kv_decode_plan for a window of each container's KV heads: decoding the containers of another tensor-parallel
 * layout into this rank's heads.  Container j holds src_H heads (its header's L and D are dst's, its H is src_H; the
 * workspace is b200kv_decode_workspace_bytes(L, src_H, D, ...)).  Its heads [src_head0[j], src_head0[j] + n_heads[j])
 * are decoded into destination heads [dst_head0[j], dst_head0[j] + n_heads[j]) at token dst_tok[j]; every other
 * destination byte is left as it was.  The three arrays are HOST int32[n_chunks].  Containers may share a dst_tok when
 * their destination head ranges do not overlap (several source shards into one rank, in one call).  The values are
 * those of a whole decode: every (plane, channel) stream of a container is independent, and the stream offsets come from
 * the fixed sections.  Status bits come from the decoded streams only.  b200kv_decode_layers runs the plan as it runs
 * b200kv_decode_plan's.  Only the tiles of CT = 128 streams that meet a window are launched; a thread whose channel
 * lies outside the window writes nothing.  Containers of every version are accepted, those of several groups (versions
 * 1 / 2, more than 256 tokens) included.  Refused, writing nothing: n_heads[j] < 1, a window outside [0, src_H), a
 * destination range outside [0, dst->H), and overlapping destination ranges at one dst_tok.
 */
int b200kv_decode_plan_heads(const void* containers, int64_t containers_bytes, const int64_t* offsets,
                             const int64_t* total_bytes, const int32_t* ntokens, const int64_t* dst_tok, int32_t n_chunks,
                             int32_t max_dtype, int32_t coder, const b200kv_kv_desc* dst, const float* key_bins,
                             const float* value_bins, uint32_t* status_out, void* workspace, int64_t workspace_bytes,
                             b200kv_decode_plan_t* plan, void* stream, int32_t src_H, const int32_t* src_head0,
                             const int32_t* dst_head0, const int32_t* n_heads);

/*
 * The encode of b200kv_encode_chunks in three steps, so that a layer can be encoded as soon as the forward pass has
 * written it (vLLM's save_kv_layer after each attention layer, wait_for_save at the end).  Version-3 containers only
 * (coder B200KV_CODER_RANS_COMPACT, chunk_tokens <= 256).
 *
 * b200kv_encode_layers_plan takes b200kv_encode_chunks' KV arguments and makes its checks, zeroes the counters in
 * `workspace` and the n_chunks fixed-section images at fixed_out + j * fixed_stride (fixed_stride >= layout.off_payload),
 * and records its decisions in *plan (caller-owned host memory).  The KV is not read yet.  max_layers: the most layers
 * one b200kv_encode_layers call may take (the workspace holds one call's temp rows:
 * b200kv_encode_layers_workspace_bytes).
 *
 * b200kv_encode_layers enqueues, for layers [layer_begin, layer_end) -- planes layer_begin.. and L + layer_begin.. -- of
 * every chunk: the row maxima and the half-lengths into the chunk's fixed image, the entropy coding, and the compaction
 * of those planes' streams into the device arena (arena_bytes bytes).  The bytes of chunk j for the call (its K planes,
 * then its V planes) are placed 16-byte aligned at a device-held cursor, in (call, chunk) order.  A chunk whose bytes do
 * not fit fails, and so does every later chunk of the plan: the chunks that fit are always a prefix.  Row (j, p) of
 * seg_sizes_out (DEVICE or mapped-host int64[n_chunks][2L][2]) gets the arena offset (-1: chunk failed) and the size of
 * plane p of chunk j.  A chunk that fails in a later call than its first keeps the rows of the calls that had placed it
 * (those bytes stay in the arena, unused); the rows of the failing call and of every later one are -1.  Read the rows of
 * chunks whose sizes_out is nonzero only.  Each layer is encoded once; a layer range that was encoded before is an error.
 *
 * b200kv_encode_layers_finish writes each chunk's header into its fixed image and sizes_out[j] (total_bytes, or 0 when
 * the chunk failed: header.status bit 16 = did not fit the arena), and fails unless every layer was encoded.
 *
 * For every chunk that did not fail, fixed image [0, layout.off_payload) || the 2L planes in order (keys of layers
 * 0..L-1, then values) are byte for byte the container b200kv_encode_chunks writes.  The KV, the arena, the images, the
 * outputs and the workspace must stay valid until the finish step has run on the device.
 */
typedef struct b200kv_encode_plan_t {
    uint64_t opaque[512];      /* holds the encode kernels' parameter block and a 128-bit set of the layers encoded */
} b200kv_encode_plan_t;

int64_t b200kv_encode_layers_workspace_bytes(int32_t L, int32_t H, int32_t D, int32_t chunk_tokens, int32_t n_chunks,
                                             int32_t max_layers);
int b200kv_encode_layers_plan(const b200kv_kv_desc* kv, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                              int32_t last_chunk_tokens, const float* key_bins, const float* value_bins, int32_t coder,
                              void* arena, int64_t arena_bytes, void* fixed_out, int64_t fixed_stride, int64_t* seg_sizes_out,
                              uint64_t* sizes_out, int32_t max_layers, void* workspace, int64_t workspace_bytes,
                              b200kv_encode_plan_t* plan, void* stream);
int b200kv_encode_layers(b200kv_encode_plan_t* plan, int32_t layer_begin, int32_t layer_end, void* stream);
int b200kv_encode_layers_finish(const b200kv_encode_plan_t* plan, void* stream);

/*
 * Lossless container ("B2KV" versions 5 and 6).  Added without changing anything that existed: b200kv_version() stays 4,
 * and neither b200kv_container_layout_v nor the CacheGen decode calls know these versions.
 *
 * Version 5 holds a (K, V) KV of P = 2L planes (keys of layers 0..L-1, then values), version 6 a latent KV
 * (B200KV_KV_LATENT) of P = L planes.  header.max_dtype is the element dtype (B200KV_DT_*), ngroups = 1, reserved = 0,
 * 1 <= ntokens = t <= 4096; C = H * D channels.  Every 16-bit element u (bf16, fp16) is split, for both dtypes alike, as
 *     v = rotl16(u, 1),  sym = v >> 8,  raw = v & 0xff        (bf16: sym = the 8 exponent bits; fp16: the 5 exponent bits
 *                                                              and the 3 top mantissa bits), u = rotr16((sym << 8) | raw, 1)
 * A one-byte element (B200KV_DT_U8, _FP8_E4M3, _FP8_E5M2) is its own symbol, sym = the byte, and has no raw byte: the
 * raw section of such a container is empty (0 bytes, so off_payload == off_raw); everything else below is the same.
 * A build that predates the one-byte dtypes refuses such a container through its max_dtype check, and off_payload
 * follows from max_dtype, so a one-byte container is never read as a 16-bit one.
 * Sections, each starting 16-byte aligned, little-endian:
 *     header | freq u16[P][256] | lens u16[P][C] | raw u8[P][t][C] (16-bit elements only) | streams
 * freq[p]: the symbol histogram n_s of plane p (its t * C elements, N = t * C) normalised to M = 4096:
 *     K = #{s : n_s > 0};  f_s = 0 if n_s = 0, else 1 + floor(n_s * (4096 - K) / N)      (integer arithmetic)
 *     then the symbol with the largest n_s (the smallest symbol among equals) gets 4096 - sum(f) added.
 *   This is one pass with no loop: K <= 256 < 4096, every occurring symbol starts at 1, and the floors sum to at most
 *   4096 - K, so the remainder 4096 - sum(f) is >= 0 and adding it keeps every frequency >= 1; the row sums to 4096.
 *   start_s = f_0 + ... + f_{s-1}.
 * raw[p][i][c]: the raw byte of token i, channel c of plane p, stored verbatim.
 * streams: one rANS stream per (plane, channel) over the t symbols, in (plane, channel) order, back to back; lens[p][c]
 *   is its byte length, payload_bytes their sum, total_bytes = offset of the streams + payload_bytes.  The coder is the
 *   project's rANS (32-bit state, 16-bit renormalisation; lmcache_b200/csrc/ac_core.cuh) with 12-bit probabilities:
 *     encoder   x = 2^16; for i = t-1 .. 0:  s = sym[i]; if (x >> 20) >= f_s: push halfword (x & 0xffff), x >>= 16;
 *               x = ((x / f_s) << 12) + (x mod f_s) + start_s
 *     bytes     x as LE32, then the pushed halfwords in REVERSE push order (LE16 each); length = 4 + 2 * pushes, even
 *     decoder   x = LE32; for i = 0 .. t-1:  slot = x & 4095; s = the symbol with start_s <= slot < start_s + f_s;
 *               x = f_s * (x >> 12) + slot - start_s; if x < 2^16: x = (x << 16) | next LE16
 *               after the last symbol x == 2^16 again and every halfword has been read (the integrity check).
 *   The renormalisation bound is f << 20; it is tested as (x >> 20) >= f because a single-symbol plane has f = 4096 and
 *   4096 << 20 overflows 32 bits (such a plane's streams are the 4 bytes of x = 2^16 and nothing else).  A stream is at
 *   most 4 + 2 * ceil(3t / 4) + 2 bytes (12 bits per symbol), which fits u16 for t <= 4096; an encode whose stream
 *   exceeds it sets header.status bit 0 (sizes_out 0).  tests/lossless_ref.py is the numpy statement of all this for
 *   16-bit elements, tests/lossless8_ref.py for one-byte ones.
 */
typedef struct b200kv_lossless_layout_t {
    int64_t off_freq, off_lens, off_raw, off_payload;
    int64_t fixed_bytes;       /* == off_payload */
    int64_t max_stream_bytes;  /* 4 + 2 * ceil(3t / 4) + 2 */
    int64_t max_total_bytes;   /* align16(off_payload + P * C * max_stream_bytes): the out_stride an encode needs */
} b200kv_lossless_layout_t;

/* Section offsets of a version-5 (latent = 0) or version-6 (latent != 0) container of 16-bit elements; L <= 128,
 * 1 <= ntokens <= 4096. */
int b200kv_lossless_layout(int32_t L, int32_t H, int32_t D, int32_t ntokens, int32_t latent, b200kv_lossless_layout_t* out);
/* The same for elements of `dtype` (B200KV_DT_*, without the latent flag): for a one-byte dtype off_payload == off_raw
 * and max_total_bytes has no raw section.  A 16-bit layout bounds the one-byte layout of the same shape field by field. */
int b200kv_lossless_layout_dt(int32_t L, int32_t H, int32_t D, int32_t ntokens, int32_t latent, int32_t dtype,
                              b200kv_lossless_layout_t* out);
/* Bytes of device scratch one b200kv_lossless_encode (decode = 0) or b200kv_lossless_decode (decode != 0) call needs;
 * < 0 for a shape the calls refuse.  The encode's is dominated by a worst-case scratch row per stream.  The figure is
 * that of 16-bit elements and bounds the need of one-byte elements too (this and
 * b200kv_lossless_encode_layers_workspace_bytes take no dtype). */
int64_t b200kv_lossless_workspace_bytes(int32_t L, int32_t H, int32_t D, int32_t chunk_tokens, int32_t n_chunks,
                                        int32_t latent, int32_t decode);
/*
 * Lossless encode: the KV, chunking, out / out_stride / sizes_out and workspace arguments of b200kv_encode_chunks
 * (out_stride >= max_total_bytes of chunk_tokens; chunk_tokens <= 4096).  Version 6 when kv->dtype carries
 * B200KV_KV_LATENT, 5 otherwise.  The KV is read twice (histogram, then coding), in stream order.
 */
int b200kv_lossless_encode(const b200kv_kv_desc* kv, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                           int32_t last_chunk_tokens, void* out, int64_t out_stride, uint64_t* sizes_out,
                           void* workspace, int64_t workspace_bytes, void* stream);
/*
 * Lossless decode: b200kv_decode_chunks' container arguments (DEVICE containers at 16-byte aligned offsets[j],
 * total_bytes[j] = header.total_bytes, the buffer extending B200KV_READ_SLACK bytes past every container, ntokens[j],
 * dst_tok[j]) into the destination `dst`.  max_dtype = header.max_dtype, the stored element dtype: dst must have that
 * dtype (a lossless codec does not cast), else the call is refused.  The version decoded is 6 for a latent destination,
 * 5 otherwise.  Reads stay inside each container whatever its lengths and frequency rows say, and nothing is written
 * outside the destination rows of the call's tokens.  status_out: NULL, or DEVICE / mapped-host uint32[n_chunks], zeroed
 * by the call and then OR-ed with
 *   1 = a stream did not return to its initial state or did not use exactly its bytes, or a frequency row does not sum
 *       to 4096 (that plane is not written),
 *   2 = a stream that lies beyond the payload (lengths section damaged; that stream is not written),
 *   4 = the header is not the one the call names: another version than the destination's latent-ness says, or another
 *       L / H / D / ntokens / max_dtype.
 */
int b200kv_lossless_decode(const void* containers, int64_t containers_bytes, const int64_t* offsets,
                           const int64_t* total_bytes, const int32_t* ntokens, const int64_t* dst_tok, int32_t n_chunks,
                           int32_t max_dtype, const b200kv_kv_desc* dst, uint32_t* status_out, void* workspace,
                           int64_t workspace_bytes, void* stream);

/* Host side: where each plane's streams lie in a lossless container in host memory (the header and the lengths section
 * are read, nothing else; nbytes >= off_raw): out[0..P], the streams of plane p (keys of layer p, then values of layer
 * p - L; P = L for version 6) are bytes [out[p], out[p+1]) of the container, out[0] = off_payload (the header's
 * max_dtype decides it).  Plane p's raw rows are bytes [off_raw + p * t * C, off_raw + (p + 1) * t * C) for 16-bit
 * elements, none for one-byte ones: b200kv_lossless_layout_dt gives them.  Returns 0, 1 when the lengths do not
 * add up to header.total_bytes (damaged), <0 for anything that is not a lossless container of a possible shape. */
int b200kv_lossless_plane_offsets(const void* container, int64_t nbytes, int64_t* out, int32_t n_out);
/* Same for n containers in DEVICE memory at containers + j*stride, as b200kv_plane_offsets_device: row j of out (DEVICE or
 * mapped-host int64[n][B200KV_MAX_PLANES + 1]) gets the P + 1 offsets and zeros in the rest of the row, or -1 in its entry
 * 0 for a container that is not lossless, whose fixed sections do not fit its total_bytes or `stride` (nothing past the
 * header is read then), or whose lengths do not add up.  Asynchronous on `stream`. */
int b200kv_lossless_plane_offsets_device(const void* containers, int64_t stride, int32_t n, int64_t* out, void* stream);

/*
 * The lossless decode in two steps, as b200kv_decode_plan / b200kv_decode_layers for the CacheGen containers: a caller
 * decodes a layer as soon as its bytes have arrived.  b200kv_lossless_decode == plan + layers(0, L).
 *
 * b200kv_lossless_decode_plan takes b200kv_lossless_decode's arguments and makes all of its checks, zeroes status_out,
 * writes the chunk descriptors into `workspace` and enqueues the stream-offset kernels.  Those read [0, off_raw) of every
 * container only (header, frequency rows, lengths), so the raw rows and the streams may still be on their way.  The
 * workspace, containers buffer, destination and status_out must stay valid until the last layers call has run.
 *
 * b200kv_lossless_decode_layers enqueues the decode of layers [layer_begin, layer_end): planes layer_begin.. (keys) and
 * L + layer_begin.. (values), or planes layer_begin.. alone for version 6, 0 <= layer_begin < layer_end <= L.  A call
 * reads the header, its planes' frequency rows, the lengths, its planes' raw rows and its planes' streams; no byte of
 * another plane reaches an output or a status bit.  It writes the destination rows of its layers only and ORs into the
 * plan's status_out, so any set of calls that covers every layer once writes what b200kv_lossless_decode writes, status
 * bits included.
 */
typedef struct b200kv_lossless_decode_plan_t {
    uint64_t opaque[512];      /* the decode kernel's parameter block (its 3 KB plane table included) */
} b200kv_lossless_decode_plan_t;

int b200kv_lossless_decode_plan(const void* containers, int64_t containers_bytes, const int64_t* offsets,
                                const int64_t* total_bytes, const int32_t* ntokens, const int64_t* dst_tok,
                                int32_t n_chunks, int32_t max_dtype, const b200kv_kv_desc* dst, uint32_t* status_out,
                                void* workspace, int64_t workspace_bytes, b200kv_lossless_decode_plan_t* plan,
                                void* stream);
int b200kv_lossless_decode_layers(const b200kv_lossless_decode_plan_t* plan, int32_t layer_begin, int32_t layer_end,
                                  void* stream);

/*
 * b200kv_lossless_decode_plan for a window of each container's KV heads, as b200kv_decode_plan_heads is for
 * b200kv_decode_plan: decoding the lossless containers of another tensor-parallel layout into this rank's heads.
 * Container j holds src_H heads (its header's L and D are dst's, its H is src_H; the workspace is
 * b200kv_lossless_workspace_bytes(L, src_H, D, ..., decode = 1)).  Its heads [src_head0[j], src_head0[j] + n_heads[j])
 * are decoded into destination heads [dst_head0[j], dst_head0[j] + n_heads[j]) at token dst_tok[j]; every other
 * destination byte is left as it was.  The three arrays are HOST int32[n_chunks].  Containers may share a dst_tok when
 * their destination head ranges do not overlap.  The result is an ordinary plan: b200kv_lossless_decode_layers runs it.
 * The values are the bits the source layout stored: every (plane, channel) stream is independent, and the stream offsets
 * come from the lengths section, which the plan sums whole.  Only the tiles of 128 streams that meet a window are
 * launched; a thread whose channel lies outside its window reads its length only and writes nothing.  Status bits come
 * from the header, the frequency rows of the planes decoded and the streams decoded: a damaged stream outside the window
 * sets none (a damaged length before the window moves the window's offsets, and its streams then fail).  Refused,
 * writing nothing and leaving status_out alone: n_heads[j] < 1, a window outside [0, src_H), a destination range outside
 * [0, dst->H), overlapping destination ranges at one dst_tok, and a latent destination (version 6 has no heads).  As for
 * the whole decode, dst's dtype must be the stored one.
 */
int b200kv_lossless_decode_plan_heads(const void* containers, int64_t containers_bytes, const int64_t* offsets,
                                      const int64_t* total_bytes, const int32_t* ntokens, const int64_t* dst_tok,
                                      int32_t n_chunks, int32_t max_dtype, const b200kv_kv_desc* dst,
                                      uint32_t* status_out, void* workspace, int64_t workspace_bytes,
                                      b200kv_lossless_decode_plan_t* plan, void* stream, int32_t src_H,
                                      const int32_t* src_head0, const int32_t* dst_head0, const int32_t* n_heads);

/*
 * The lossless encode in three steps, as b200kv_encode_layers_plan / _layers / _finish for the CacheGen containers: a
 * layer is encoded as soon as the forward pass has written it.  Versions 5 and 6, chunk_tokens <= 4096.
 *
 * b200kv_lossless_encode_layers_plan takes b200kv_lossless_encode's KV and chunking arguments and makes its checks,
 * zeroes the error words, payload totals and the arena cursor in `workspace` and the n_chunks fixed images at
 * fixed_out + j * fixed_stride, and records its decisions in *plan (caller-owned host memory).  A fixed image is
 * [0, off_raw) of the container (header, frequency rows, lengths): fixed_stride >= off_raw, 16-byte aligned.  The KV is
 * not read yet.  max_layers: the most layers one b200kv_lossless_encode_layers call may take (the workspace holds one
 * call's scratch and raw rows: b200kv_lossless_encode_layers_workspace_bytes).  arena: DEVICE, 16-byte aligned.
 *
 * b200kv_lossless_encode_layers enqueues, for layers [layer_begin, layer_end) -- planes layer_begin.. and L +
 * layer_begin.., or planes layer_begin.. alone for version 6 -- of every chunk: the histograms and frequency rows
 * (into the fixed image), the coding (lengths into the fixed image), and one segment per chunk in the device arena of
 * arena_bytes bytes:
 *     [the call's planes' raw rows, t * C bytes each (none for one-byte elements), in plane order; in the call that
 *      holds the last plane followed by the container's zero bytes up to off_payload; zeros to a 16-byte boundary]
 *     [the call's planes' streams, in order]
 * Segments are placed by the rule of b200kv_encode_layers (16-byte aligned at a device-held cursor in (call, chunk)
 * order, with a reserve for the layers still to come; the chunks that fit are always a prefix).  Row (j, p) of
 * seg_sizes_out (DEVICE or mapped-host int64[n_chunks][P][3], P = 2L or L) gets (arena offset of plane p's raw rows,
 * arena offset of its streams, its stream bytes); the offsets are -1 for a chunk that failed, and a chunk that fails in a
 * later call than its first keeps the rows of the calls that had placed it, as in b200kv_encode_layers.  Read the rows of
 * chunks whose sizes_out is nonzero only.  Each layer is encoded once.
 *
 * b200kv_lossless_encode_layers_finish writes each chunk's header into its fixed image from the stream bytes of every
 * call, and sizes_out[j] (total_bytes, or 0 when header.status is nonzero: bit 16 = did not fit the arena, bit 0 = a
 * stream outgrew its bound), and fails unless every layer was encoded.
 *
 * For every chunk that did not fail, fixed image [0, off_raw) || for p = 0..P-1 the raw bytes at row (j, p)[0]
 * (t * C of them, 0 for one-byte elements; for p = P - 1 up to off_payload) || for p = 0..P-1 the row (j, p)[2] stream
 * bytes at row (j, p)[1]
 * is byte for byte the container b200kv_lossless_encode writes.  Every refusal returns < 0 and enqueues nothing: a layer
 * range out of bounds or encoded before, finish before every layer was encoded, a plan not made by
 * b200kv_lossless_encode_layers_plan, a misaligned arena or fixed image, a too small fixed stride or workspace, and the
 * shapes b200kv_lossless_encode refuses.  The KV, arena, images, outputs and workspace must stay valid until the finish
 * step has run on the device.
 */
typedef struct b200kv_lossless_encode_plan_t {
    uint64_t opaque[512];      /* the encode kernels' parameter block and a 128-bit set of the layers encoded */
} b200kv_lossless_encode_plan_t;

int64_t b200kv_lossless_encode_layers_workspace_bytes(int32_t L, int32_t H, int32_t D, int32_t chunk_tokens,
                                                      int32_t n_chunks, int32_t latent, int32_t max_layers);
int b200kv_lossless_encode_layers_plan(const b200kv_kv_desc* kv, int64_t tok_begin, int32_t n_chunks,
                                       int32_t chunk_tokens, int32_t last_chunk_tokens, void* arena, int64_t arena_bytes,
                                       void* fixed_out, int64_t fixed_stride, int64_t* seg_sizes_out,
                                       uint64_t* sizes_out, int32_t max_layers, void* workspace, int64_t workspace_bytes,
                                       b200kv_lossless_encode_plan_t* plan, void* stream);
int b200kv_lossless_encode_layers(b200kv_lossless_encode_plan_t* plan, int32_t layer_begin, int32_t layer_end,
                                  void* stream);
int b200kv_lossless_encode_layers_finish(const b200kv_lossless_encode_plan_t* plan, void* stream);

/*
 * Token-id prefix hash.  Replaces LMCacheEngine._chunk_tokens/_hash/_prefix_hash
 * (cache_engine.py:58-96): h_i = sha256(ascii_hex(h_{i-1}) || bytes(tokens[i*cs:(i+1)*cs])), h_{-1} = "".
 * n_seq independent sequences are hashed concurrently (one chain each).  tokens: DEVICE pointer to the
 * raw little-endian token ids (elem_size bytes each: 8 for int64, 4 for int32); sequence s covers
 * tokens [seq_offsets[s], seq_offsets[s+1]) (HOST int64 array of n_seq+1 entries).  digests: DEVICE
 * or mapped-host buffer, 32 raw bytes per chunk, sequences back to back, ceil(len/chunk_size) each.
 */
int b200kv_sha256_chain(const void* tokens, int32_t elem_size, const int64_t* seq_offsets, int32_t n_seq,
                        int32_t chunk_size, void* digests, void* stream);
/* Same, and digest k is announced as soon as it exists: ready[k] (DEVICE-visible uint32 array, one word per digest slot,
 * normally mapped host memory like `digests`; or NULL) is set to `epoch` after digest k has been made visible system-wide.
 * A chain is serial -- one 256-token chunk after another -- so a host thread that polls ready[] can look up and move the first
 * chunks while the later ones are still being hashed (LMCacheEngine.store / retrieve do).  The digests must be 4-byte
 * aligned. */
int b200kv_sha256_chain_ready(const void* tokens, int32_t elem_size, const int64_t* seq_offsets, int32_t n_seq,
                              int32_t chunk_size, void* digests, uint32_t* ready, uint32_t epoch, void* stream);

/*
 * Blob pack / unpack between a kv_desc (tuple-of-tensors or strided blob) and contiguous chunk blobs
 * [L,2,t,H,D] (vllm) / [L,2,H,t,D] (huggingface), t = chunk tokens.  Replaces _tuple_kv_to_blob +
 * _slice_kv_at (.contiguous() per chunk) and the retrieve-side torch.cat
 * (cache_engine.py:98-161,362-368) with one gather / scatter kernel.
 * `chunks` is DEVICE memory, or pinned host memory mapped into the device address space (then the kernel
 * itself is the GPU->host mover).  Chunk j starts at chunks + j*chunk_stride_bytes.
 * hf_layout != 0 selects the huggingface chunk layout.  Elements of every B200KV_DT_* move as they are (16-byte
 * vectors when D, the strides and the pointers allow it, element by element otherwise).
 */
int b200kv_pack_chunks(const b200kv_kv_desc* src, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                       int32_t last_chunk_tokens, int32_t hf_layout, void* chunks, int64_t chunk_stride_bytes,
                       void* stream);
int b200kv_unpack_chunks(const void* chunks, int64_t chunk_stride_bytes, int32_t n_chunks, int32_t chunk_tokens,
                         int32_t last_chunk_tokens, int32_t hf_layout, const b200kv_kv_desc* dst, int64_t tok_begin,
                         void* stream);
/* The same for the layers [layer_begin, layer_end) of every chunk, in one launch, wherever each chunk lives.
 * chunk_ptrs is a DEVICE array of n_chunks pointers (device or mapped pinned memory): chunk j's layer l lies at
 * chunk_ptrs[j] + (l - layer_begin) * slice_bytes(t_j), where a layer slice is [2,t,H,D] (vllm) / [2,H,t,D]
 * (huggingface) / [t,D] (latent KV) and t_j is chunk_tokens, or last_chunk_tokens for the last chunk.  One pointer thus
 * names the range inside a full chunk blob (blob_j + layer_begin * slice) or a staging area that holds only the range.
 * Planes of other layers are neither read nor written.  16-byte vectors where D, the strides, the planes and each
 * chunk pointer allow it (a chunk pointer that is not 16-byte aligned moves element by element).  < 0, with nothing
 * enqueued, for a NULL table, a range outside 0 <= layer_begin < layer_end <= L, or a bad chunking. */
int b200kv_pack_chunks_layers(const b200kv_kv_desc* src, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                              int32_t last_chunk_tokens, int32_t hf_layout, int32_t layer_begin, int32_t layer_end,
                              void* const* chunk_ptrs, void* stream);
int b200kv_unpack_chunks_layers(const void* const* chunk_ptrs, int32_t n_chunks, int32_t chunk_tokens,
                                int32_t last_chunk_tokens, int32_t hf_layout, int32_t layer_begin, int32_t layer_end,
                                const b200kv_kv_desc* dst, int64_t tok_begin, void* stream);

/*
 * Rotary position shift of stored keys (non-prefix reuse: a segment cached at positions 0..n-1 served at positions
 * s..s+n-1).  vLLM caches K after the rotary embedding, R(i)·k_i; at offset s attention needs R(s + i)·k_i =
 * R(s)·(R(i)·k_i).  Added without changing anything that existed (b200kv_version() stays 4).
 *
 * b200kv_rope_table fills cos_sin (DEVICE float [n_seg][rotary_dim/2][2]) with (cos, sin) of shifts[s] * inv_freq[j]:
 * shifts is a DEVICE int64 [n_seg], inv_freq a DEVICE float32 [rotary_dim/2] (any frequency-only rope scaling: plain
 * theta, Llama-3's, YaRN's frequencies).  The angle is computed in fp64 and range-reduced before sincos, then rounded
 * once to fp32.  < 0, nothing enqueued: NULL pointers, n_seg <= 0, an odd or non-positive rotary_dim.
 *
 * b200kv_rope_shift rotates in place, in one launch, channels [offset, offset + rotary_dim) of every head of the KEY
 * planes (kv = 0; the one plane of a B200KV_KV_LATENT descriptor) of tokens [tok_begin, tok_begin + ntok) of the view,
 * every layer.  Token tok_begin + i is rotated by table row seg_of_tok[i] (DEVICE int32 [ntok]); -1 leaves the row
 * alone, neither read nor written.  style 0 (neox) pairs channels (d, d + rotary_dim/2), style 1 (gptj) (2d, 2d + 1);
 * pair j turns by row (cos, sin)[j]: (a, b) <- (a cos - b sin, b cos + a sin), each element loaded, converted to fp32,
 * rotated and rounded once back to its dtype.  V planes, channels outside the rotary range and other tokens are not
 * touched.  Every layout a kv_desc carries: blobs (vllm, huggingface), tuples, latent views, slot-mapped rows and
 * B200KV_KV_PAGED_SPLIT key blocks.  16-byte vectors where offset, rotary_dim, the strides and the planes allow it.
 * < 0, nothing enqueued: a one-byte dtype (FP8 / U8: rotating would round values FP8 already rounded), an odd or
 * non-positive rotary_dim, offset < 0 or offset + rotary_dim > D, a NULL cos_sin, a NULL seg_of_tok with ntok > 0, a
 * style other than 0 and 1.  Table rows are not bounds-checked: seg_of_tok holds -1 or rows of cos_sin.
 */
int b200kv_rope_table(const int64_t* shifts, int32_t n_seg, const float* inv_freq, int32_t rotary_dim, float* cos_sin,
                      void* stream);
int b200kv_rope_shift(const b200kv_kv_desc* kv, int64_t tok_begin, int64_t ntok, const int32_t* seg_of_tok,
                      const float* cos_sin, int32_t rotary_dim, int32_t offset, int32_t style, void* stream);
/* b200kv_rope_shift restricted to the key planes of layers [layer_begin, layer_end): a layer-wise retrieve turns each
 * layer's keys as soon as that layer has landed.  b200kv_rope_shift is the range [0, L), and calls whose ranges cover
 * each layer once give its result bit for bit.  Plane pointers of other layers are never dereferenced, and the vector
 * path's alignment test looks at the range's planes only.  < 0, nothing enqueued: what b200kv_rope_shift refuses, and a
 * layer range that is empty or outside [0, L).  Added without changing anything that existed (b200kv_version() stays
 * 4). */
/* The unpack direction of b200kv_pack_chunks_rope, for a layer range: chunk j (chunk_ptrs[j], DEVICE, the chunk's
 * layer range as in b200kv_unpack_chunks_layers) holds chunk_ntok[j] tokens (DEVICE int32, 1 .. chunk_tokens) and
 * lands at view token dst_tok[j] (DEVICE int64); the rotary channels of its key planes turn by table row chunk_seg[j]
 * (DEVICE int32; -1: copied).  Chunks need not be contiguous in the view nor of one size: a layer-wise segment retrieve
 * writes one layer of every hit chunk of every segment in one launch.  Every destination b200kv_unpack_chunks_layers
 * takes (blobs, tuples, latent views, slot-mapped and block-strided rows, B200KV_KV_PAGED_SPLIT).  Each key element
 * reads its rotation partner from the chunk, with b200kv_rope_shift's arithmetic: the result is bit-identical to
 * b200kv_unpack_chunks_layers of each chunk followed by b200kv_rope_shift_layers.  A misaligned chunk pointer moves
 * element by element.  < 0, nothing enqueued: NULL arrays, what b200kv_rope_shift_layers refuses (one-byte dtypes, an
 * odd or non-positive rotary_dim, offset < 0 or offset + rotary_dim > D, a NULL cos_sin, a bad style or layer range)
 * and what b200kv_unpack_chunks_layers refuses.  The device arrays are not bounds-checked.  Added without changing
 * anything that existed (b200kv_version() stays 4). */
int b200kv_unpack_chunks_layers_rope(const void* const* chunk_ptrs, int32_t n_chunks, int32_t chunk_tokens,
                                     const int32_t* chunk_ntok, const int64_t* dst_tok, const int32_t* chunk_seg,
                                     int32_t hf_layout, int32_t layer_begin, int32_t layer_end,
                                     const b200kv_kv_desc* dst, const float* cos_sin, int32_t rotary_dim, int32_t offset,
                                     int32_t style, void* stream);
int b200kv_rope_shift_layers(const b200kv_kv_desc* kv, int32_t layer_begin, int32_t layer_end, int64_t tok_begin,
                             int64_t ntok, const int32_t* seg_of_tok, const float* cos_sin, int32_t rotary_dim,
                             int32_t offset, int32_t style, void* stream);
/* The pack direction of b200kv_unpack_chunks_layers_rope: chunk j takes chunk_ntok[j] tokens (DEVICE int32, 1 ..
 * chunk_tokens) from view token src_tok[j] (DEVICE int64) and writes layers [layer_begin, layer_end) of them to
 * chunk_ptrs[j] (DEVICE array; device or mapped pinned memory) in b200kv_pack_chunks_layers' chunk layout ([2,t,H,D],
 * [2,H,t,D] with hf_layout, [t,D] for a latent KV, per layer, t = chunk_ntok[j]); the rotary channels of its key
 * planes turn by table row chunk_seg[j] (DEVICE int32; -1: copied).  A layer-wise segment store stages one layer of
 * every segment in one launch, each turned back by -start.  Every source b200kv_pack_chunks_rope takes (blobs, tuples,
 * latent views, slot-mapped and block-strided rows, B200KV_KV_PAGED_SPLIT).  Each key element reads its rotation
 * partner from the source, which is never written, with b200kv_rope_shift's arithmetic: the result is bit-identical to
 * b200kv_pack_chunks_rope of the same tokens restricted to the range, and to b200kv_pack_chunks_layers followed by
 * b200kv_rope_shift_layers of the packed chunk.  V planes, other channels and other layers' planes are neither read
 * nor written.  A misaligned chunk pointer is written element by element.  < 0, nothing enqueued: NULL arrays, what
 * b200kv_rope_shift_layers refuses (one-byte dtypes, an odd or non-positive rotary_dim, offset < 0 or offset +
 * rotary_dim > D, a NULL cos_sin, a bad style or layer range) and what b200kv_pack_chunks_layers refuses.  The device
 * arrays are not bounds-checked.  Added without changing anything that existed (b200kv_version() stays 4). */
int b200kv_pack_chunks_layers_rope(const b200kv_kv_desc* src, int32_t n_chunks, int32_t chunk_tokens,
                                   const int32_t* chunk_ntok, const int64_t* src_tok, const int32_t* chunk_seg,
                                   int32_t hf_layout, int32_t layer_begin, int32_t layer_end,
                                   void* const* chunk_ptrs, const float* cos_sin, int32_t rotary_dim,
                                   int32_t offset, int32_t style, void* stream);
/* b200kv_pack_chunks with the keys turned on the way (a segment of a longer prompt stored as if prefilled alone: its
 * keys turned by -start): the same descriptors (blobs, tuples, latent views, slot-mapped and block-strided rows,
 * B200KV_KV_PAGED_SPLIT), chunk layouts and destinations (device or mapped pinned memory) as b200kv_pack_chunks, in one
 * launch.  Call token tok_begin + i has channels [offset, offset + rotary_dim) of its key planes (kv = 0; the plane of a
 * B200KV_KV_LATENT descriptor) turned by row seg_of_tok[i] (DEVICE int32, one per token packed) of cos_sin, with
 * b200kv_rope_shift's pairing and arithmetic; -1, V planes and every other channel are copied bit for bit.  The result
 * is bit-identical to b200kv_pack_chunks followed by b200kv_rope_shift of the packed rows; the source is only read.
 * < 0, nothing enqueued: what b200kv_rope_shift refuses (one-byte dtypes, an odd or non-positive rotary_dim, offset < 0
 * or offset + rotary_dim > D, NULL cos_sin or seg_of_tok, a style other than 0 and 1) and what b200kv_pack_chunks
 * refuses.  Added without changing anything that existed (b200kv_version() stays 4). */
int b200kv_pack_chunks_rope(const b200kv_kv_desc* src, int64_t tok_begin, int32_t n_chunks, int32_t chunk_tokens,
                            int32_t last_chunk_tokens, int32_t hf_layout, void* chunks, int64_t chunk_stride_bytes,
                            const int32_t* seg_of_tok, const float* cos_sin, int32_t rotary_dim, int32_t offset,
                            int32_t style, void* stream);

/*
 * CacheBlend's selective recomputation, the cache's side (lmcache_b200/csrc/blend.cu).  A reused document's KV at layers
 * >= 1 was computed without attending to the tokens now in front of it; the model recomputes the reused tokens whose
 * cached keys deviate most from fresh ones.  These calls measure the deviation and choose the tokens, identically on
 * every tensor-parallel rank.  Added without changing anything that existed (b200kv_version() stays 4).
 *
 * b200kv_blend_deviation: fresh (DEVICE, n rows of fresh_row_stride elements, the first H*D of each used) holds the
 * model's keys of one layer after the rotary embedding, in the cache's dtype; row i belongs to view token tok[i]
 * (DEVICE int64 [n], through slot_map as in every other entry point).  dev[i] (DEVICE float [n]) gets
 *     sum over h < H, d < D of (fresh[i][h*D + d] - key(layer, tok[i], h, d))^2
 * in fp32, over the key plane of `layer` only (kv = 0; the one plane of a B200KV_KV_LATENT descriptor, all D channels).
 * The summation order depends on (H, D) alone: channel c = h*D + d belongs to lane (c / 8) % 32, each lane accumulates
 * its channels in ascending c with one fma per element, and the 32 lane sums are folded by an xor butterfly (16, 8, 4,
 * 2, 1).  The same rows therefore give the same bits in every layout, at every n, row index, alignment and launch:
 * ranks that sum their heads' dev get one total.  Every descriptor b200kv_rope_shift takes: blobs (vllm, huggingface),
 * tuples, latent views, slot-mapped and block-strided rows, B200KV_KV_PAGED_SPLIT key blocks.  16-byte vectors when D,
 * the strides, fresh_row_stride and the pointers allow it, element by element otherwise.  < 0, nothing enqueued: a
 * one-byte dtype, NULL pointers with n > 0, a layer outside [0, L), fresh_row_stride < H*D.
 *
 * b200kv_blend_select: rows (DEVICE int64) gets every row i < n with cand[i] == 0 (DEVICE uint8 [n]) in ascending order,
 * then, in ascending order, the min(k, n_cand) candidate rows (cand != 0) of largest dev (DEVICE float [n]): n_forced +
 * min(k, n_cand) entries, a count the caller knows from cand.  Ties go to the lower row; NaN ranks as +inf (and -0 as
 * +0), so a damaged row is recomputed.  Seven operations on `stream` whatever n (a 4 KB memset, four radix-histogram
 * passes over the keys' bit patterns, a count pass and the compaction), no host sync, and no atomic whose order shows
 * in the result.  workspace: DEVICE, 4-byte aligned, b200kv_blend_select_workspace_bytes(n) bytes; n < 2^31.  < 0,
 * nothing enqueued: n or k negative, NULL pointers with n > 0, a small workspace.
 *
 * b200kv_blend_select_batch: b200kv_blend_select per segment of one array, for a prefill batch of B requests whose rows
 * are concatenated.  Segment s covers rows [seg[s], seg[s+1]) (DEVICE int64 [B+1]; seg[0] = 0, seg[B] = n, not
 * decreasing; empty segments are allowed) and selects k[s] (DEVICE int64 [B], >= 0) candidates.  rows gets one block
 * per segment, in segment order: the segment's forced rows in ascending order, then its min(k[s], candidates of s)
 * candidates of largest dev in ascending order, as global row indices.  Restricted to one segment the block is exactly
 * b200kv_blend_select of that slice plus seg[s]: ties to the lower row, NaN as +inf, -0 as +0.  The same seven
 * operations on `stream` whatever n, B and the spread of the rows over the segments (a memset of the histograms, four
 * radix passes, a count pass and the compaction), no host sync, and no atomic whose order shows in the result.  seg
 * and k are device data: their preconditions are the caller's, not checked.  workspace: DEVICE, 4-byte aligned,
 * b200kv_blend_select_batch_workspace_bytes(n, B) bytes = 4176 bytes per segment (four 256-bin histograms and the
 * radix state of each pass, the block's start and the segment's first-row counts) + 16 bytes per CTA of the row
 * split (at most 1024 CTAs).  < 0, nothing enqueued: n outside [0, 2^31), B outside [1, 2^31), NULL pointers with
 * n > 0, a small or misaligned workspace.
 */
int b200kv_blend_deviation(const b200kv_kv_desc* kv, int32_t layer, int64_t n, const int64_t* tok, const void* fresh,
                           int64_t fresh_row_stride, float* dev, void* stream);
int64_t b200kv_blend_select_workspace_bytes(int64_t n);
int b200kv_blend_select(const float* dev, const uint8_t* cand, int64_t n, int64_t k, int64_t* rows, void* workspace,
                        int64_t workspace_bytes, void* stream);
int64_t b200kv_blend_select_batch_workspace_bytes(int64_t n, int64_t B);
int b200kv_blend_select_batch(const float* dev, const uint8_t* cand, int64_t n, int64_t B, const int64_t* seg,
                              const int64_t* k, int64_t* rows, void* workspace, int64_t workspace_bytes,
                              void* stream);

/*
 * GPU <-> pinned-host mover.  Replaces LMCLocalBackend.put_blocking/put_nonblocking/get
 * (local_backend.py:82-100,128-144: pageable tensor.to("cpu") / .to("cuda") + torch.cuda.synchronize()).
 */
int b200kv_pinned_alloc(void** host_ptr, int64_t bytes);       /* cudaHostAlloc(portable|mapped) */
int b200kv_pinned_free(void* host_ptr);
int b200kv_host_device_ptr(void* host_ptr, void** device_ptr); /* device alias of a pinned allocation */
int b200kv_copy_async(void* dst, const void* src, int64_t bytes, void* stream);  /* cudaMemcpyDefault */
/* strided 2-D copy: `rows` rows of `row_bytes`, pitches in bytes (chunk slice of a [L,2,T,H,D] blob) */
int b200kv_copy2d_async(void* dst, int64_t dst_pitch, const void* src, int64_t src_pitch, int64_t row_bytes,
                        int64_t rows, void* stream);
/* n copies of sizes[i] bytes from srcs[i] to dsts[i] (HOST pointer arrays), in stream order as a batch: the copies of one
 * call may run in any order among themselves.  One cudaMemcpyBatchAsync where the driver has it (CUDA >= 12.8) and the
 * stream is not the legacy default stream (NULL), which that call refuses; one cudaMemcpyAsync per copy otherwise. */
int b200kv_copy_batch_async(void* const* dsts, const void* const* srcs, const int64_t* sizes, int64_t n, void* stream);
int b200kv_stream_create(void** stream);                       /* non-blocking side stream */
int b200kv_stream_destroy(void* stream);
int b200kv_stream_sync(void* stream);
int b200kv_event_create(void** event);
int b200kv_event_destroy(void* event);
int b200kv_event_record(void* event, void* stream);
int b200kv_event_query(void* event);                           /* 0 = complete, 1 = pending, <0 = error */
int b200kv_event_sync(void* event);
int b200kv_stream_wait_event(void* stream, void* event);
int b200kv_event_elapsed_ms(void* start, void* stop, float* ms);

/*
 * Per-kernel device timing of the most recent encode / decode call (CUDA events recorded on the call's
 * stream around each launch).  Not part of the reference surface: bench.py's roofline leg uses it so the
 * dominant kernel is timed live, outside any profiler.  Slots: 0 absmax, 1 cdf, 2 encode, 3 scan+compact+finalize,
 * 4 tile_sum, 5 tile_scan, 6 decode; -1 = not launched.  Not thread-safe; enable only while benchmarking.
 */
int b200kv_profile_enable(int32_t on);
int b200kv_profile_last(float* ms, int32_t n);

/*
 * lm:// remote tier, client and server (SURVEY 8f rank 2).  Host-only: no device work, usable without a GPU.
 * Wire-compatible with lmcache/protocol.py:4-70 (158-byte client header "ii150s", 8-byte server header "ii"), so either
 * side interoperates with the reference's Python client (storage_backend/connector/lm_connector.py:15-84) and server
 * (lmcache/server/__main__.py:29-104).  Payloads are sent from / received into caller memory in one pass (Python bytes,
 * a pinned slab, ...); a connection serialises whole request / response exchanges; the server's EXIST / GET are O(1)
 * hash lookups under a reader-writer lock (the reference scans list_keys()).  Keys are <= 150 bytes.
 */
int b200kv_lm_server_start(const char* host, int32_t port, void** server); /* port 0 = ephemeral; threads run until stop */
int32_t b200kv_lm_server_port(void* server);
int64_t b200kv_lm_server_num_keys(void* server);
int b200kv_lm_server_stop(void* server);
int b200kv_lm_connect(const char* host, int32_t port, void** conn);
int b200kv_lm_close(void* conn);
int b200kv_lm_put(void* conn, const char* key, const void* data, int64_t len);      /* connection.set(); no server ack */
int b200kv_lm_exists(void* conn, const char* key);                                  /* 1 present, 0 absent, <0 error */
/* GET / LIST in two calls, because the caller allocates the destination once the length is known:
 *   n = b200kv_lm_get_begin(conn, key)   payload length >= 0, -1 = miss, < -1 = error
 *   b200kv_lm_read(conn, dst, n)         payload into caller memory (must follow a successful begin, also for n = 0) */
int64_t b200kv_lm_get_begin(void* conn, const char* key);
int64_t b200kv_lm_list_begin(void* conn);                                           /* keys joined by '\n' */
int b200kv_lm_read(void* conn, void* dst, int64_t len);
/* Ranged reads of stored values (this project's servers only: send them after b200kv_lm_exists(conn, "b200kv-ranges-v1")
 * returned 1; the reference server answers 0, and it ignores an unknown command without a reply, so a client that sent
 * one would wait forever).  A handle holds the
 * value as it was at OPEN -- a later PUT of the key does not change what READ returns -- and lives until CLOSE or the
 * end of the connection; a server keeps at most 4096 per connection.
 *   n = b200kv_lm_open_begin(conn, key, prefix, &handle, &size)   n = min(prefix, size) bytes pending, -1 = miss or
 *                                                                    the handle cap, < -1 = error; then
 *   b200kv_lm_read(conn, dst, n)                                   the value's first n bytes into caller memory
 *   b200kv_lm_read_ranges(conn, m, handles, offsets, sizes, dst)   range i of handle i into dst[i]; sum of sizes < 2^31;
 *                                                                    0 = done, 1 = refused (unknown handle or a range
 *                                                                    out of bounds; nothing written), < 0 = error
 *   b200kv_lm_close_handles(conn, m, handles)                      unknown handles are ignored */
int64_t b200kv_lm_open_begin(void* conn, const char* key, int64_t prefix, uint32_t* handle, int64_t* size);
int b200kv_lm_read_ranges(void* conn, int32_t m, const uint32_t* handles, const uint64_t* offsets, const uint64_t* sizes,
                          void* const* dst);
int b200kv_lm_close_handles(void* conn, int32_t m, const uint32_t* handles);
int64_t b200kv_lm_server_num_handles(void* server);                                 /* open handles, all connections */

#ifdef __cplusplus
}
#endif
#endif /* B200KV_H_ */
