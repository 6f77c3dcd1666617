"""lm:// cache server: `python -m lmcache_b200.server <host> <port> [--python]`.
Default: the native server of libb200kv (csrc/lmnet.cu); `--python` runs the pure-Python one below.

Speaks the reference wire protocol (lmcache/protocol.py, lmcache/server/__main__.py:29-93): opaque bytes
in an in-memory dict, thread per client, no ack on PUT.  It never touches KV math; it exists so the
engine-over-socket configurations can be exercised on a box that does not have the reference tree.
EXIST is a dict lookup (the reference scans list_keys(), server/__main__.py:78-80).

Ranged reads (OPEN / READ / CLOSE, lmcache_b200/protocol.py) as the native server has them: a handle keeps the
bytearray the key held at OPEN -- a PUT replaces that object, never mutates it -- so READ serves that snapshot."""
import socket
import struct
import sys
import threading

from lmcache_b200.protocol import (MAX_HANDLES, MAX_REPLY, OPEN_META, RANGES_PROBE_KEY, READ_ENTRY, ClientMetaMessage,
                                   Constants, ServerMetaMessage)


class LMCacheServer:

    def __init__(self, host: str, port: int):
        self.store = {}
        self.lock = threading.Lock()
        self.sock = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
        self.sock.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
        self.sock.bind((host, port))
        self.sock.listen()
        self.handles_open = 0        # OPEN handles of every connection

    @staticmethod
    def _recv_exact(conn, n):
        buf = bytearray(n)
        view, got = memoryview(buf), 0
        while got < n:
            k = conn.recv_into(view[got:], n - got)
            if k == 0:
                return None
            got += k
        return buf

    def _count(self, d: int) -> None:
        with self.lock:
            self.handles_open += d

    def num_handles(self) -> int:
        with self.lock:
            return self.handles_open

    def _ranges(self, conn, meta, handles, nxt):
        """OPEN / READ / CLOSE; returns the next handle number, or None when the connection is lost"""
        fail = ServerMetaMessage(Constants.SERVER_FAIL, 0).serialize()
        if meta.command == Constants.CLIENT_OPEN:
            with self.lock:
                data = self.store.get(meta.key)
            if data is None or meta.length < 0 or len(handles) >= MAX_HANDLES:
                conn.sendall(fail)
                return nxt
            while nxt in handles or nxt == 0:
                nxt = (nxt + 1) & 0xffffffff
            handles[nxt] = data
            self._count(1)
            n = min(meta.length, len(data))
            conn.sendall(ServerMetaMessage(Constants.SERVER_SUCCESS, 16 + n).serialize() + OPEN_META.pack(nxt, 0, len(data)) +
                         bytes(memoryview(data)[:n]))
            return (nxt + 1) & 0xffffffff
        if meta.length < 0:
            return None
        body = self._recv_exact(conn, meta.length)
        if body is None:
            return None
        if meta.command == Constants.CLIENT_CLOSE:
            for (h,) in struct.iter_unpack("<I", body[:meta.length // 4 * 4]):
                if handles.pop(h, None) is not None:
                    self._count(-1)
            conn.sendall(ServerMetaMessage(Constants.SERVER_SUCCESS, 0).serialize())
            return nxt
        ranges, total = [], 0
        ok = meta.length % READ_ENTRY.size == 0
        for h, _, off, nb in (READ_ENTRY.iter_unpack(body) if ok else ()):
            data = handles.get(h)
            if data is None or off > len(data) or nb > len(data) - off or total + nb > MAX_REPLY:
                ok = False
                break
            ranges.append(memoryview(data)[off:off + nb])
            total += nb
        if not ok:
            conn.sendall(fail)
            return nxt
        conn.sendall(b"".join([ServerMetaMessage(Constants.SERVER_SUCCESS, total).serialize()] + ranges))
        return nxt

    def handle_client(self, conn):
        handles, nxt = {}, 1                 # this connection's snapshots
        try:
            while True:
                header = self._recv_exact(conn, ClientMetaMessage.packlength())
                if header is None:
                    break
                meta = ClientMetaMessage.deserialize(bytes(header))
                if meta.command == Constants.CLIENT_PUT:
                    data = self._recv_exact(conn, meta.length)
                    if data is None:
                        break
                    with self.lock:
                        self.store[meta.key] = data
                elif meta.command == Constants.CLIENT_GET:
                    with self.lock:
                        data = self.store.get(meta.key)
                    if data is None:
                        conn.sendall(ServerMetaMessage(Constants.SERVER_FAIL, 0).serialize())
                    else:
                        conn.sendall(ServerMetaMessage(Constants.SERVER_SUCCESS, len(data)).serialize())
                        conn.sendall(data)
                elif meta.command == Constants.CLIENT_EXIST:
                    with self.lock:
                        ok = meta.key in self.store or meta.key == RANGES_PROBE_KEY
                    conn.sendall(ServerMetaMessage(Constants.SERVER_SUCCESS if ok else Constants.SERVER_FAIL,
                                                   0).serialize())
                elif meta.command == Constants.CLIENT_LIST:
                    with self.lock:
                        data = "\n".join(self.store.keys()).encode()
                    conn.sendall(ServerMetaMessage(Constants.SERVER_SUCCESS, len(data)).serialize())
                    conn.sendall(data)
                elif meta.command in (Constants.CLIENT_OPEN, Constants.CLIENT_READ, Constants.CLIENT_CLOSE):
                    nxt = self._ranges(conn, meta, handles, nxt)
                    if nxt is None:
                        break
                else:
                    break
        finally:
            self._count(-len(handles))
            conn.close()

    def run(self):
        try:
            while True:
                conn, _ = self.sock.accept()
                threading.Thread(target=self.handle_client, args=(conn,), daemon=True).start()
        finally:
            self.sock.close()


def run_native(host: str, port: int) -> None:
    """The same server in C++ (csrc/lmnet.cu): thread per client, O(1) EXIST / GET under a reader-writer lock,
    payloads received into / sent from one buffer each.  Runs until the process is terminated."""
    import ctypes
    import signal
    import time

    from lmcache_b200 import _native as N
    lib = N.lib()
    h = ctypes.c_void_p()
    N.check(lib.b200kv_lm_server_start(host.encode(), port, ctypes.byref(h)), "lm_server_start")
    stop = []
    signal.signal(signal.SIGTERM, lambda *_: stop.append(1))
    try:
        while not stop:
            time.sleep(0.2)
    except KeyboardInterrupt:
        pass
    lib.b200kv_lm_server_stop(h)


def main():
    args = [a for a in sys.argv[1:] if a != "--python"]
    if len(args) not in (2, 3):
        print(f"Usage: {sys.argv[0]} <host> <port> [cpu] [--python]")
        sys.exit(1)
    if "--python" in sys.argv[1:]:
        LMCacheServer(args[0], int(args[1])).run()
    else:
        run_native(args[0], int(args[1]))


if __name__ == "__main__":
    main()
