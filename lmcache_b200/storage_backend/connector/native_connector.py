"""lm:// client on the native library (csrc/lmnet.cu): same wire protocol and the same RemoteConnector surface as
LMCServerConnector (lmcache/storage_backend/connector/lm_connector.py:15-84), but the socket work happens in C++
with the GIL released -- payloads are sent straight from the caller's buffer (Python bytes, a pinned slab) and
received straight into the bytearray handed back to the deserializer."""
import ctypes
import threading
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

from lmcache_b200 import _native as N
from lmcache_b200.protocol import MAX_KEY_LENGTH, RANGES_PROBE_KEY
from lmcache_b200.storage_backend.connector.base_connector import RemoteConnector


def _ptr_len(obj):
    """(address, length, keepalive) of a bytes-like object without copying when possible."""
    if isinstance(obj, bytes):
        return ctypes.cast(ctypes.c_char_p(obj), ctypes.c_void_p), len(obj), obj
    mv = memoryview(obj)
    if not mv.contiguous:
        b = mv.tobytes()
        return ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p), len(b), b
    mv = mv.cast("B")
    if mv.readonly:
        b = mv.tobytes()
        return ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p), len(b), b
    n = mv.nbytes
    if n == 0:
        return ctypes.c_void_p(0), 0, mv
    arr = (ctypes.c_char * n).from_buffer(mv)
    return ctypes.cast(arr, ctypes.c_void_p), n, (arr, mv)


class LMCNativeConnector(RemoteConnector):

    def __init__(self, host: str, port: int):
        self._lib = N.lib()
        h = ctypes.c_void_p()
        N.check(self._lib.b200kv_lm_connect(host.encode(), int(port), ctypes.byref(h)), "lm_connect")
        self._h = h
        self.lock = threading.Lock()      # begin + read of a GET form one exchange

    @staticmethod
    def _key(key: str) -> bytes:
        k = key.encode()
        assert len(k) <= MAX_KEY_LENGTH, f"Key length {len(k)} exceeds maximum {MAX_KEY_LENGTH}"
        return k

    def exists(self, key: str) -> bool:
        with self.lock:
            return self._h is not None and self._lib.b200kv_lm_exists(self._h, self._key(key)) == 1

    def set(self, key: str, obj) -> None:
        ptr, n, keep = _ptr_len(obj)
        with self.lock:
            N.check(self._lib.b200kv_lm_put(self._h, self._key(key), ptr, n), "lm_put")
        del keep

    def _read(self, n: int) -> Optional[bytearray]:
        buf = bytearray(n)
        dst = (ctypes.c_char * n).from_buffer(buf) if n else None
        rc = self._lib.b200kv_lm_read(self._h, ctypes.cast(dst, ctypes.c_void_p) if n else None, n)
        del dst
        return buf if rc == 0 else None

    def get(self, key: str) -> Optional[bytearray]:
        with self.lock:
            if self._h is None:
                return None
            n = self._lib.b200kv_lm_get_begin(self._h, self._key(key))
            if n < 0:
                return None
            return self._read(n)

    def get_into(self, key: str, dst_ptr: int, cap: int) -> Optional[int]:
        """GET straight into caller memory (e.g. a page-locked slab): returns the payload length, None on a miss.
        A payload larger than `cap` is drained and reported as a miss (the caller's bound was wrong)."""
        with self.lock:
            if self._h is None:
                return None
            n = self._lib.b200kv_lm_get_begin(self._h, self._key(key))
            if n < 0:
                return None
            if n > cap:
                self._read(n)
                return None
            rc = self._lib.b200kv_lm_read(self._h, ctypes.c_void_p(dst_ptr) if n else None, n)
            return n if rc == 0 else None

    # ---- ranged reads (lmcache_b200/protocol.py): only after supports_ranges() said the server has them
    def supports_ranges(self) -> bool:
        return self.exists(RANGES_PROBE_KEY)

    def open_into(self, key: str, prefix: int, alloc: Callable[[int], Tuple[int, object]]):
        """OPEN `key`: alloc(size) -> (address, obj) gives the memory its first min(prefix, size) bytes go to.  Returns
        (handle, size, prefix bytes received, obj), or None on a miss.  Raises when the exchange fails (the connection is
        then out of step) or alloc raises (the handle is closed first)."""
        handle, size = ctypes.c_uint32(), ctypes.c_int64()
        with self.lock:
            if self._h is None:
                raise N.NativeError("lm:// connection is closed")
            n = self._lib.b200kv_lm_open_begin(self._h, self._key(key), int(prefix), ctypes.byref(handle),
                                               ctypes.byref(size))
            if n == -1:
                return None
            N.check(n, "lm_open_begin")
            try:
                ptr, obj = alloc(int(size.value))
            except BaseException:
                self._read(n)
                self._lib.b200kv_lm_close_handles(self._h, 1, ctypes.byref(handle))
                raise
            N.check(self._lib.b200kv_lm_read(self._h, ctypes.c_void_p(ptr) if n else None, n), "lm_read")
        return int(handle.value), int(size.value), int(n), obj

    def read_ranges(self, handles: Sequence[int], offsets: Sequence[int], sizes: Sequence[int],
                    dst_ptrs: Sequence[int]) -> bool:
        """READ: range i (offset, size) of handles[i] straight into dst_ptrs[i].  The sizes add up to less than 2^31.
        True when done, False when the server refused it (nothing written); raises when the exchange fails."""
        h = np.ascontiguousarray(handles, dtype=np.uint32)
        o = np.ascontiguousarray(offsets, dtype=np.uint64)
        z = np.ascontiguousarray(sizes, dtype=np.uint64)
        d = np.ascontiguousarray(dst_ptrs, dtype=np.uint64)
        with self.lock:
            if self._h is None:
                raise N.NativeError("lm:// connection is closed")
            rc = N.check(self._lib.b200kv_lm_read_ranges(self._h, len(h), h.ctypes.data, o.ctypes.data, z.ctypes.data,
                                                         d.ctypes.data), "lm_read_ranges")
        return rc == 0

    def close_handles(self, handles: Sequence[int]) -> None:
        h = np.ascontiguousarray(handles, dtype=np.uint32)
        with self.lock:
            if self._h is None:
                raise N.NativeError("lm:// connection is closed")
            N.check(self._lib.b200kv_lm_close_handles(self._h, len(h), h.ctypes.data), "lm_close_handles")

    def list(self) -> List[str]:
        with self.lock:
            if self._h is None:
                return []
            n = self._lib.b200kv_lm_list_begin(self._h)
            if n < 0:
                return []
            data = self._read(n)
        return [] if not data else [k for k in bytes(data).decode().split("\n") if k]

    def close(self) -> None:
        with self.lock:
            if self._h is not None:
                self._lib.b200kv_lm_close(self._h)
                self._h = None
