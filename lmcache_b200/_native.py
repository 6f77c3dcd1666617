"""ctypes binding of libb200kv.so (include/b200kv.h) -- the only door to the CUDA hot path.

There is deliberately no fallback: if the shared library is missing, or no CUDA device is
visible, every compute entry point raises.  `lib()` only needs the .so; `require_cuda()`
additionally needs a device.
"""
from __future__ import annotations

import ctypes
import os
import threading
from typing import Optional, Sequence

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200kv.so")

DT_BF16 = 0
DT_FP16 = 1
DT_U8 = 2           # one-byte elements: torch.uint8 (vLLM 0.6.x's fp8 cache), float8_e4m3fn, float8_e5m2
DT_FP8_E4M3 = 3
DT_FP8_E5M2 = 4
ONE_BYTE_DTYPES = (DT_U8, DT_FP8_E4M3, DT_FP8_E5M2)
CODER_AC = 0       # container version 1: arithmetic coder
CODER_RANS = 1     # container version 2: rANS
CODER_RANS_COMPACT = 2   # container version 3: rANS streams that carry their own histogram (no CDF section), one-byte lengths
ENCODE_HINT_MID_ENTROPY = 0x200    # B200KV_ENCODE_HINT_MID_ENTROPY
KV_LATENT = 0x100        # B200KV_KV_LATENT: OR-ed into KvDesc.dtype (one plane per layer) and into a coder (container version 4)
KV_PAGED_SPLIT = 0x400   # B200KV_KV_PAGED_SPLIT: OR-ed into KvDesc.dtype (vLLM's PagedAttention split cache; mover only)
CODER_LATENT = CODER_RANS_COMPACT | KV_LATENT   # the coder argument that names container version 4
CODER_LOSSLESS = 4       # names container version 5: lossless, (K, V) planes (not a b200kv_encode_chunks coder)
CODER_LOSSLESS_LATENT = CODER_LOSSLESS | KV_LATENT   # container version 6: lossless, one plane per layer
LOSSLESS_MAX_TOKENS = 4096   # tokens per lossless container
HDR_MAX = 36            # longest version-3 stream header (4 mask bytes + 31 counts + 1 pad)
CODERS = {"ac": CODER_AC, "rans": CODER_RANS, "rans_compact": CODER_RANS_COMPACT}
LP = 33
GROUP_TOKENS = 256
MAX_PLANES = 256         # B200KV_MAX_PLANES: 2L for models of up to 128 layers
MAGIC = 0x564B3242
HEADER_BYTES = 64
READ_SLACK = 640     # B200KV_READ_SLACK

c_i32, c_i64, c_vp, c_u64 = ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p, ctypes.c_uint64


class NativeError(RuntimeError):
    """Nonzero return code from libb200kv (message from b200kv_last_error())."""


class KvDesc(ctypes.Structure):
    """struct b200kv_kv_desc"""
    _fields_ = [
        ("base", c_vp),
        ("planes", ctypes.POINTER(c_vp)),
        ("sL", c_i64), ("sKV", c_i64), ("sT", c_i64), ("sH", c_i64),
        ("L", c_i32), ("H", c_i32), ("D", c_i32),
        ("dtype", c_i32),
        ("slot_map", c_vp),     # device int64[ntokens] or NULL (paged KV)
    ]


class Header(ctypes.Structure):
    """struct b200kv_header (64 bytes)"""
    _fields_ = [
        ("magic", ctypes.c_uint32), ("version", ctypes.c_uint32),
        ("L", ctypes.c_uint32), ("H", ctypes.c_uint32), ("D", ctypes.c_uint32),
        ("ntokens", ctypes.c_uint32), ("ngroups", ctypes.c_uint32),
        ("max_dtype", ctypes.c_uint32),
        ("payload_bytes", c_u64), ("total_bytes", c_u64),
        ("status", ctypes.c_uint32), ("reserved", ctypes.c_uint32 * 3),
    ]


class Layout(ctypes.Structure):
    """struct b200kv_layout"""
    _fields_ = [("off_cdf", c_i64), ("off_maxes", c_i64), ("off_lengths", c_i64), ("off_payload", c_i64),
                ("fixed_bytes", c_i64), ("max_total_bytes", c_i64)]


class LosslessLayout(ctypes.Structure):
    """struct b200kv_lossless_layout_t"""
    _fields_ = [("off_freq", c_i64), ("off_lens", c_i64), ("off_raw", c_i64), ("off_payload", c_i64),
                ("fixed_bytes", c_i64), ("max_stream_bytes", c_i64), ("max_total_bytes", c_i64)]


class DecodePlan(ctypes.Structure):
    """struct b200kv_decode_plan_t (opaque, filled by b200kv_decode_plan)"""
    _fields_ = [("opaque", ctypes.c_uint64 * 256)]


class EncodePlan(ctypes.Structure):
    """struct b200kv_encode_plan_t (opaque, filled by b200kv_encode_layers_plan)"""
    _fields_ = [("opaque", ctypes.c_uint64 * 512)]


class LosslessDecodePlan(ctypes.Structure):
    """struct b200kv_lossless_decode_plan_t (opaque, filled by b200kv_lossless_decode_plan)"""
    _fields_ = [("opaque", ctypes.c_uint64 * 512)]


class LosslessEncodePlan(ctypes.Structure):
    """struct b200kv_lossless_encode_plan_t (opaque, filled by b200kv_lossless_encode_layers_plan)"""
    _fields_ = [("opaque", ctypes.c_uint64 * 512)]


assert ctypes.sizeof(Header) == HEADER_BYTES

# name -> (restype, argtypes); every symbol include/b200kv.h declares
SIGNATURES = {
    "b200kv_version": (c_i32, []),
    "b200kv_last_error": (ctypes.c_char_p, []),
    "b200kv_device_count": (c_i32, []),
    "b200kv_container_layout": (c_i32, [c_i32, c_i32, c_i32, c_i32, ctypes.POINTER(Layout)]),
    "b200kv_container_layout_v": (c_i32, [c_i32, c_i32, c_i32, c_i32, c_i32, ctypes.POINTER(Layout)]),
    "b200kv_plane_offsets": (c_i32, [c_vp, c_i64, c_vp, c_i32]),
    "b200kv_plane_offsets_device": (c_i32, [c_vp, c_i64, c_i32, c_vp, c_vp]),
    "b200kv_encode_workspace_bytes": (c_i64, [c_i32, c_i32, c_i32, c_i32, c_i32, c_i32]),
    "b200kv_decode_workspace_bytes": (c_i64, [c_i32, c_i32, c_i32, c_i32, c_i32]),
    "b200kv_encode_chunks": (c_i32, [ctypes.POINTER(KvDesc), c_i64, c_i32, c_i32, c_i32, c_vp, c_vp, c_i32, c_vp, c_i64,
                                      c_vp, c_vp, c_i64, c_vp]),
    "b200kv_decode_chunks": (c_i32, [c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, ctypes.POINTER(KvDesc),
                                      c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]),
    "b200kv_decode_plan": (c_i32, [c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, ctypes.POINTER(KvDesc),
                                    c_vp, c_vp, c_vp, c_vp, c_i64, ctypes.POINTER(DecodePlan), c_vp]),
    "b200kv_decode_layers": (c_i32, [ctypes.POINTER(DecodePlan), c_i32, c_i32, c_vp]),
    "b200kv_decode_plan_heads": (c_i32, [c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, ctypes.POINTER(KvDesc),
                                          c_vp, c_vp, c_vp, c_vp, c_i64, ctypes.POINTER(DecodePlan), c_vp, c_i32, c_vp,
                                          c_vp, c_vp]),
    "b200kv_encode_layers_workspace_bytes": (c_i64, [c_i32, c_i32, c_i32, c_i32, c_i32, c_i32]),
    "b200kv_encode_layers_plan": (c_i32, [ctypes.POINTER(KvDesc), c_i64, c_i32, c_i32, c_i32, c_vp, c_vp, c_i32, c_vp,
                                          c_i64, c_vp, c_i64, c_vp, c_vp, c_i32, c_vp, c_i64, ctypes.POINTER(EncodePlan),
                                          c_vp]),
    "b200kv_encode_layers": (c_i32, [ctypes.POINTER(EncodePlan), c_i32, c_i32, c_vp]),
    "b200kv_encode_layers_finish": (c_i32, [ctypes.POINTER(EncodePlan), c_vp]),
    "b200kv_lossless_layout": (c_i32, [c_i32, c_i32, c_i32, c_i32, c_i32, ctypes.POINTER(LosslessLayout)]),
    "b200kv_lossless_layout_dt": (c_i32, [c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, ctypes.POINTER(LosslessLayout)]),
    "b200kv_lossless_workspace_bytes": (c_i64, [c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32]),
    "b200kv_lossless_encode": (c_i32, [ctypes.POINTER(KvDesc), c_i64, c_i32, c_i32, c_i32, c_vp, c_i64, c_vp, c_vp,
                                        c_i64, c_vp]),
    "b200kv_lossless_decode": (c_i32, [c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, ctypes.POINTER(KvDesc), c_vp,
                                        c_vp, c_i64, c_vp]),
    "b200kv_lossless_plane_offsets": (c_i32, [c_vp, c_i64, c_vp, c_i32]),
    "b200kv_lossless_plane_offsets_device": (c_i32, [c_vp, c_i64, c_i32, c_vp, c_vp]),
    "b200kv_lossless_decode_plan": (c_i32, [c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, ctypes.POINTER(KvDesc),
                                             c_vp, c_vp, c_i64, ctypes.POINTER(LosslessDecodePlan), c_vp]),
    "b200kv_lossless_decode_layers": (c_i32, [ctypes.POINTER(LosslessDecodePlan), c_i32, c_i32, c_vp]),
    "b200kv_lossless_decode_plan_heads": (c_i32, [c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32,
                                                   ctypes.POINTER(KvDesc), c_vp, c_vp, c_i64,
                                                   ctypes.POINTER(LosslessDecodePlan), c_vp, c_i32, c_vp, c_vp, c_vp]),
    "b200kv_lossless_encode_layers_workspace_bytes": (c_i64, [c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32]),
    "b200kv_lossless_encode_layers_plan": (c_i32, [ctypes.POINTER(KvDesc), c_i64, c_i32, c_i32, c_i32, c_vp, c_i64, c_vp,
                                                   c_i64, c_vp, c_vp, c_i32, c_vp, c_i64,
                                                   ctypes.POINTER(LosslessEncodePlan), c_vp]),
    "b200kv_lossless_encode_layers": (c_i32, [ctypes.POINTER(LosslessEncodePlan), c_i32, c_i32, c_vp]),
    "b200kv_lossless_encode_layers_finish": (c_i32, [ctypes.POINTER(LosslessEncodePlan), c_vp]),
    "b200kv_sha256_chain": (c_i32, [c_vp, c_i32, c_vp, c_i32, c_i32, c_vp, c_vp]),
    "b200kv_sha256_chain_ready": (c_i32, [c_vp, c_i32, c_vp, c_i32, c_i32, c_vp, c_vp, ctypes.c_uint32, c_vp]),
    "b200kv_pack_chunks": (c_i32, [ctypes.POINTER(KvDesc), c_i64, c_i32, c_i32, c_i32, c_i32, c_vp, c_i64, c_vp]),
    "b200kv_unpack_chunks": (c_i32, [c_vp, c_i64, c_i32, c_i32, c_i32, c_i32, ctypes.POINTER(KvDesc), c_i64, c_vp]),
    "b200kv_pack_chunks_layers": (c_i32, [ctypes.POINTER(KvDesc), c_i64, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp,
                                          c_vp]),
    "b200kv_unpack_chunks_layers": (c_i32, [c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, ctypes.POINTER(KvDesc),
                                            c_i64, c_vp]),
    "b200kv_rope_table": (c_i32, [c_vp, c_i32, c_vp, c_i32, c_vp, c_vp]),
    "b200kv_rope_shift": (c_i32, [ctypes.POINTER(KvDesc), c_i64, c_i64, c_vp, c_vp, c_i32, c_i32, c_i32, c_vp]),
    "b200kv_unpack_chunks_layers_rope": (c_i32, [c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_i32, c_i32, c_i32,
                                                 ctypes.POINTER(KvDesc), c_vp, c_i32, c_i32, c_i32, c_vp]),
    "b200kv_pack_chunks_layers_rope": (c_i32, [ctypes.POINTER(KvDesc), c_i32, c_i32, c_vp, c_vp, c_vp, c_i32, c_i32,
                                               c_i32, c_vp, c_vp, c_i32, c_i32, c_i32, c_vp]),
    "b200kv_rope_shift_layers": (c_i32, [ctypes.POINTER(KvDesc), c_i32, c_i32, c_i64, c_i64, c_vp, c_vp, c_i32, c_i32,
                                         c_i32, c_vp]),
    "b200kv_pack_chunks_rope": (c_i32, [ctypes.POINTER(KvDesc), c_i64, c_i32, c_i32, c_i32, c_i32, c_vp, c_i64, c_vp,
                                        c_vp, c_i32, c_i32, c_i32, c_vp]),
    "b200kv_blend_deviation": (c_i32, [ctypes.POINTER(KvDesc), c_i32, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "b200kv_blend_select_workspace_bytes": (c_i64, [c_i64]),
    "b200kv_blend_select": (c_i32, [c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_i64, c_vp]),
    "b200kv_blend_select_batch_workspace_bytes": (c_i64, [c_i64, c_i64]),
    "b200kv_blend_select_batch": (c_i32, [c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]),
    "b200kv_pinned_alloc":(c_i32, [ctypes.POINTER(c_vp), c_i64]),
    "b200kv_pinned_free": (c_i32, [c_vp]),
    "b200kv_host_device_ptr": (c_i32, [c_vp, ctypes.POINTER(c_vp)]),
    "b200kv_copy_async": (c_i32, [c_vp, c_vp, c_i64, c_vp]),
    "b200kv_copy2d_async": (c_i32, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i64, c_vp]),
    "b200kv_copy_batch_async": (c_i32, [c_vp, c_vp, c_vp, c_i64, c_vp]),
    "b200kv_stream_create": (c_i32, [ctypes.POINTER(c_vp)]),
    "b200kv_stream_destroy": (c_i32, [c_vp]),
    "b200kv_stream_sync": (c_i32, [c_vp]),
    "b200kv_event_create": (c_i32, [ctypes.POINTER(c_vp)]),
    "b200kv_event_destroy": (c_i32, [c_vp]),
    "b200kv_event_record": (c_i32, [c_vp, c_vp]),
    "b200kv_event_query": (c_i32, [c_vp]),
    "b200kv_event_sync": (c_i32, [c_vp]),
    "b200kv_stream_wait_event": (c_i32, [c_vp, c_vp]),
    "b200kv_event_elapsed_ms": (c_i32, [c_vp, c_vp, ctypes.POINTER(ctypes.c_float)]),
    "b200kv_profile_enable": (c_i32, [c_i32]),
    "b200kv_profile_last": (c_i32, [ctypes.POINTER(ctypes.c_float), c_i32]),
    "b200kv_lm_server_start": (c_i32, [ctypes.c_char_p, c_i32, ctypes.POINTER(c_vp)]),
    "b200kv_lm_server_port": (c_i32, [c_vp]),
    "b200kv_lm_server_num_keys": (c_i64, [c_vp]),
    "b200kv_lm_server_stop": (c_i32, [c_vp]),
    "b200kv_lm_connect": (c_i32, [ctypes.c_char_p, c_i32, ctypes.POINTER(c_vp)]),
    "b200kv_lm_close": (c_i32, [c_vp]),
    "b200kv_lm_put": (c_i32, [c_vp, ctypes.c_char_p, c_vp, c_i64]),
    "b200kv_lm_exists": (c_i32, [c_vp, ctypes.c_char_p]),
    "b200kv_lm_get_begin": (c_i64, [c_vp, ctypes.c_char_p]),
    "b200kv_lm_list_begin": (c_i64, [c_vp]),
    "b200kv_lm_read": (c_i32, [c_vp, c_vp, c_i64]),
    "b200kv_lm_open_begin": (c_i64, [c_vp, ctypes.c_char_p, c_i64, c_vp, c_vp]),
    "b200kv_lm_read_ranges": (c_i32, [c_vp, c_i32, c_vp, c_vp, c_vp, c_vp]),
    "b200kv_lm_close_handles": (c_i32, [c_vp, c_i32, c_vp]),
    "b200kv_lm_server_num_handles": (c_i64, [c_vp]),
}
PROFILE_SLOTS = ("absmax", "cdf", "encode", "compact", "tile_sum", "tile_scan", "decode")

_lib: Optional[ctypes.CDLL] = None
_lock = threading.Lock()


def lib() -> ctypes.CDLL:
    """Load libb200kv.so (built in-tree by __graft_entry__.build()).  Raises if absent."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise RuntimeError(
                        f"{LIB_PATH} is missing: the CUDA extension is not built "
                        f"(run `python -c 'import __graft_entry__ as g; g.build()'`). There is no CPU fallback.")
                L = ctypes.CDLL(LIB_PATH)
                for name, (res, args) in SIGNATURES.items():
                    fn = getattr(L, name)      # AttributeError if the .so lacks a declared symbol
                    fn.restype = res
                    fn.argtypes = args
                _lib = L
    return _lib


_pylib: Optional[ctypes.PyDLL] = None


def pylib() -> ctypes.PyDLL:
    """The library through ctypes.PyDLL, for b200kv_plane_offsets_device and b200kv_lossless_plane_offsets_device alone:
    the call keeps the GIL.  It is one kernel launch on the store worker; giving the GIL up and taking it back there costs
    the store more than the launch whenever the caller's thread is busy in Python (it spins on the hash chain's ready words
    while a store runs)."""
    global _pylib
    if _pylib is None:
        lib()
        with _lock:
            if _pylib is None:
                L = ctypes.PyDLL(LIB_PATH)
                for name in ("b200kv_plane_offsets_device", "b200kv_lossless_plane_offsets_device"):
                    res, args = SIGNATURES[name]
                    getattr(L, name).restype = res
                    getattr(L, name).argtypes = args
                _pylib = L
    return _pylib


def last_error() -> str:
    msg = lib().b200kv_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def check(rc: int, what: str = "") -> int:
    if rc < 0:
        raise NativeError(f"libb200kv {what} failed (rc={rc}): {last_error()}")
    return rc


_cuda_ok: Optional[bool] = None


def require_cuda() -> None:
    """Fail loudly when the hot path cannot run (no device / no driver)."""
    global _cuda_ok
    if _cuda_ok is None:
        n = lib().b200kv_device_count()
        _cuda_ok = n > 0
        if not _cuda_ok:
            _cuda_ok = None
            raise RuntimeError(f"lmcache_b200 needs a CUDA device (sm_90a); none usable: {last_error() or 'count=0'}. "
                               f"There is no CPU fallback.")


def container_layout(L: int, H: int, D: int, ntokens: int, coder: int = CODER_RANS) -> Layout:
    """Section offsets of the container `coder` produces (versions 1 and 2 share a layout; CODER_LATENT: version 4)."""
    lo = Layout()
    check(lib().b200kv_container_layout_v(L, H, D, ntokens, coder, ctypes.byref(lo)), "container_layout")
    return lo


def coder_of_version(version: int) -> int:
    """The coder argument that names a container version: version - 1 for versions 1 to 3, CODER_LATENT for 4; the
    lossless containers: CODER_LOSSLESS for 5, CODER_LOSSLESS_LATENT for 6."""
    if version == 4:
        return CODER_LATENT
    if version == 6:
        return CODER_LOSSLESS_LATENT
    return int(version) - 1


def planes_of(version: int, L: int) -> int:
    """Planes of a container: one per layer in versions 4 and 6 (a latent KV), a (K, V) pair per layer otherwise."""
    return L if version in (4, 6) else 2 * L


def lossless_layout(L: int, H: int, D: int, ntokens: int, latent: bool = False, dtype: int = DT_BF16) -> LosslessLayout:
    """Section offsets of a lossless container (version 5, or 6 for a latent KV) of elements of `dtype` (DT_*): a
    one-byte dtype has no raw section."""
    lo = LosslessLayout()
    check(lib().b200kv_lossless_layout_dt(L, H, D, ntokens, int(bool(latent)), int(dtype), ctypes.byref(lo)),
          "lossless_layout")
    return lo


def nb_map(key_bins, value_bins, L: int) -> list:
    """symbols a stream of every plane (keys then values) can emit = the nb map of a compact container: 2 * (bins // 2)"""
    return [2 * (int(b) // 2) for b in list(key_bins)[:L]] + [2 * (int(b) // 2) for b in list(value_bins)[:L]]


def float_array(vals: Sequence[float]):
    return (ctypes.c_float * len(vals))(*[float(v) for v in vals])


def i64_array(vals: Sequence[int]):
    return (c_i64 * len(vals))(*[int(v) for v in vals])


def i32_array(vals: Sequence[int]):
    return (c_i32 * len(vals))(*[int(v) for v in vals])
