"""lm:// client (lmcache/storage_backend/connector/lm_connector.py:15-84): blocking TCP, fixed headers
from lmcache_b200.protocol.  One lock covers a whole request/response exchange, so concurrent put / get
threads cannot interleave on the socket (the reference locks sends only, see its TODO:1)."""
import ctypes
import socket
import struct
import threading
from typing import Callable, List, Optional, Sequence, Tuple

from lmcache_b200.protocol import (MAX_REPLY, OPEN_META, RANGES_PROBE_KEY, READ_ENTRY, ClientMetaMessage, Constants,
                                   ServerMetaMessage)
from lmcache_b200.storage_backend.connector.base_connector import RemoteConnector


class LMCServerConnector(RemoteConnector):

    def __init__(self, host: str, port: int):
        self.sock = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
        self.sock.connect((host, port))
        self.lock = threading.Lock()

    def _recv_exact(self, n: int) -> Optional[bytearray]:
        buf = bytearray(n)
        view, got = memoryview(buf), 0
        while got < n:
            k = self.sock.recv_into(view[got:], n - got)
            if k == 0:
                return None
            got += k
        return buf

    def _request(self, command: int, key: str, payload=None) -> None:
        length = 0 if payload is None else len(payload)
        self.sock.sendall(ClientMetaMessage(command, key, length).serialize())
        if payload is not None:
            self.sock.sendall(payload)

    def exists(self, key: str) -> bool:
        with self.lock:
            self._request(Constants.CLIENT_EXIST, key)
            hdr = self._recv_exact(ServerMetaMessage.packlength())
        return hdr is not None and ServerMetaMessage.deserialize(bytes(hdr)).code == Constants.SERVER_SUCCESS

    def set(self, key: str, obj) -> None:
        with self.lock:
            self._request(Constants.CLIENT_PUT, key, obj)   # the server sends no ack for PUT (server/__main__.py:46-48)

    def get(self, key: str) -> Optional[bytes]:
        with self.lock:
            self._request(Constants.CLIENT_GET, key)
            hdr = self._recv_exact(ServerMetaMessage.packlength())
            if hdr is None:
                return None
            meta = ServerMetaMessage.deserialize(bytes(hdr))
            if meta.code != Constants.SERVER_SUCCESS:
                return None
            return self._recv_exact(meta.length)

    def get_into(self, key: str, dst_ptr: int, cap: int) -> Optional[int]:
        """GET straight into caller memory (e.g. a page-locked slab): returns the payload length, None on a miss.
        A payload larger than `cap` is drained and reported as a miss."""
        with self.lock:
            self._request(Constants.CLIENT_GET, key)
            hdr = self._recv_exact(ServerMetaMessage.packlength())
            if hdr is None:
                return None
            meta = ServerMetaMessage.deserialize(bytes(hdr))
            if meta.code != Constants.SERVER_SUCCESS:
                return None
            n = meta.length
            if n > cap:
                self._recv_exact(n)
                return None
            if n == 0:
                return 0
            view = memoryview((ctypes.c_char * n).from_address(dst_ptr)).cast("B")
            got = 0
            while got < n:
                k = self.sock.recv_into(view[got:], n - got)
                if k == 0:
                    return None
                got += k
            return n

    def _recv_to(self, ptr: int, n: int) -> None:
        if n == 0:
            return
        view = memoryview((ctypes.c_char * n).from_address(ptr)).cast("B")
        got = 0
        while got < n:
            k = self.sock.recv_into(view[got:], n - got)
            if k == 0:
                raise ConnectionError("lm:// connection closed")
            got += k

    def _reply(self) -> ServerMetaMessage:
        hdr = self._recv_exact(ServerMetaMessage.packlength())
        if hdr is None:
            raise ConnectionError("lm:// connection closed")
        return ServerMetaMessage.deserialize(bytes(hdr))

    # ---- ranged reads (lmcache_b200/protocol.py): only after supports_ranges() said the server has them
    def supports_ranges(self) -> bool:
        return self.exists(RANGES_PROBE_KEY)

    def open_into(self, key: str, prefix: int, alloc: Callable[[int], Tuple[int, object]]):
        """LMCNativeConnector.open_into: (handle, size, prefix bytes received, obj) or None on a miss"""
        with self.lock:
            self.sock.sendall(ClientMetaMessage(Constants.CLIENT_OPEN, key, int(prefix)).serialize())
            meta = self._reply()
            if meta.code != Constants.SERVER_SUCCESS:
                return None
            body = self._recv_exact(OPEN_META.size)
            if body is None or meta.length < OPEN_META.size:
                raise ConnectionError("lm:// OPEN reply malformed or cut short")
            handle, _, size = OPEN_META.unpack(bytes(body))
            n = meta.length - OPEN_META.size
            try:
                ptr, obj = alloc(size)
            except BaseException:
                self._recv_exact(n)
                self.sock.sendall(ClientMetaMessage(Constants.CLIENT_CLOSE, "", 4).serialize() + struct.pack("<I", handle))
                self._reply()
                raise
            self._recv_to(ptr, n)
        return handle, size, n, obj

    def read_ranges(self, handles: Sequence[int], offsets: Sequence[int], sizes: Sequence[int],
                    dst_ptrs: Sequence[int]) -> bool:
        sizes = [int(z) for z in sizes]
        assert sum(sizes) <= MAX_REPLY, "a READ reply must stay below 2^31 bytes: split the request"
        body = b"".join(READ_ENTRY.pack(int(h), 0, int(o), z) for h, o, z in zip(handles, offsets, sizes))
        with self.lock:
            self.sock.sendall(ClientMetaMessage(Constants.CLIENT_READ, "", len(body)).serialize() + body)
            meta = self._reply()
            if meta.code != Constants.SERVER_SUCCESS:
                return False
            if meta.length != sum(sizes):
                raise ConnectionError("lm:// READ reply length does not match the request")
            for p, z in zip(dst_ptrs, sizes):
                self._recv_to(int(p), z)
        return True

    def close_handles(self, handles: Sequence[int]) -> None:
        body = b"".join(struct.pack("<I", int(h)) for h in handles)
        with self.lock:
            self.sock.sendall(ClientMetaMessage(Constants.CLIENT_CLOSE, "", len(body)).serialize() + body)
            self._reply()

    def list(self) -> List[str]:
        with self.lock:
            self._request(Constants.CLIENT_LIST, "")
            hdr = self._recv_exact(ServerMetaMessage.packlength())
            if hdr is None:
                return []
            meta = ServerMetaMessage.deserialize(bytes(hdr))
            if meta.code != Constants.SERVER_SUCCESS or meta.length == 0:
                return []
            data = self._recv_exact(meta.length)
        return [] if data is None else [k for k in bytes(data).decode().split("\n") if k]

    def close(self) -> None:
        try:
            self.sock.close()
        except OSError:
            pass
