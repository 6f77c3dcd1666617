"""Ranged reads on the lm:// wire (OPEN / READ / CLOSE behind the EXIST probe), against both of this project's servers
(native, csrc/lmnet.cu, and the pure-Python one), and the host side of the layer-major remote retrieve: the READ plan
(pipeline.ranged_read_plan) and the prefix-only container record.  Host-only: runs without a GPU."""
import ctypes
import socket
import threading
import time

import numpy as np
import pytest

import __graft_entry__ as ge

ge.build_cuda()
from lmcache_b200 import _native as N  # noqa: E402
from lmcache_b200.pipeline import READ_MAX_BYTES, layer_copy_ranges, ranged_read_plan, read_container  # noqa: E402
from lmcache_b200.protocol import (MAX_HANDLES, RANGES_PROBE_KEY, ClientMetaMessage, Constants,  # noqa: E402
                                   ServerMetaMessage)
from lmcache_b200.server.__main__ import LMCacheServer  # noqa: E402
from lmcache_b200.storage_backend.connector.lm_connector import LMCServerConnector  # noqa: E402
from lmcache_b200.storage_backend.connector.native_connector import LMCNativeConnector  # noqa: E402


class _Server:
    def __init__(self, kind):
        self.kind = kind
        if kind == "native":
            self.lib = N.lib()
            self.h = ctypes.c_void_p()
            N.check(self.lib.b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(self.h)))
            self.port = self.lib.b200kv_lm_server_port(self.h)
        else:
            self.srv = LMCacheServer("127.0.0.1", 0)
            self.port = self.srv.sock.getsockname()[1]
            threading.Thread(target=self.srv.run, daemon=True).start()

    def num_handles(self) -> int:
        return self.lib.b200kv_lm_server_num_handles(self.h) if self.kind == "native" else self.srv.num_handles()

    def stop(self):
        if self.kind == "native":
            N.check(self.lib.b200kv_lm_server_stop(self.h))
        else:
            self.srv.sock.close()


@pytest.fixture(params=["native", "python"])
def server(request):
    s = _Server(request.param)
    yield s
    s.stop()


@pytest.fixture(params=["native", "python"])
def client(request, server):
    c = (LMCNativeConnector if request.param == "native" else LMCServerConnector)("127.0.0.1", server.port)
    yield c
    c.close()


def _put(c, key, value):
    c.set(key, value)
    for _ in range(400):                 # PUT has no ack: the server may still be reading the payload
        got = c.get(key)
        if got is not None and bytes(got) == bytes(value):
            return
        time.sleep(0.005)
    raise AssertionError("PUT did not land")


def _wait_handles(server, want):
    for _ in range(400):
        if server.num_handles() == want:
            return True
        time.sleep(0.005)
    return False


class _Buf:
    """caller memory for open_into / read_ranges"""

    def __init__(self):
        self.bufs = []

    def alloc(self, size):
        b = ctypes.create_string_buffer(max(1, size))
        self.bufs.append(b)
        return ctypes.addressof(b), b


def test_probe_answers_on_both_servers(client):
    assert client.supports_ranges()
    assert client.exists(RANGES_PROBE_KEY) and client.get(RANGES_PROBE_KEY) is None     # a probe, not a stored key


def test_open_read_close_random(server, client):
    rng = np.random.default_rng(5)
    values = {f"k{i}": rng.integers(0, 256, n, dtype=np.uint8).tobytes() for i, n in enumerate([0, 1, 100, 4097, 300000])}
    for k, v in values.items():
        _put(client, k, v)
    mem = _Buf()
    opened = {}
    for k, v in values.items():
        for prefix in (0, 7, len(v), len(v) + 10):
            r = client.open_into(k, prefix, mem.alloc)
            assert r is not None
            handle, size, got, buf = r
            assert size == len(v) and got == min(prefix, len(v)) and buf.raw[:got] == v[:got]
            opened.setdefault(k, []).append((handle, buf))
    assert client.open_into("missing", 10, mem.alloc) is None
    assert server.num_handles() == sum(len(x) for x in opened.values())
    # many ranges per READ, zero-length ranges, ranges ending at the value's end
    hs, offs, sizes, dsts, want = [], [], [], [], []
    for k, v in values.items():
        h, buf = opened[k][0]
        n = len(v)
        for _ in range(50):
            a = int(rng.integers(0, n + 1))
            b = int(rng.integers(a, n + 1)) if rng.random() < 0.8 else n
            d = ctypes.create_string_buffer(max(1, b - a))
            mem.bufs.append(d)
            hs.append(h); offs.append(a); sizes.append(b - a); dsts.append(ctypes.addressof(d)); want.append((d, v[a:b]))
    assert client.read_ranges(hs, offs, sizes, dsts)
    for d, w in want:
        assert d.raw[:len(w)] == w
    assert client.read_ranges([], [], [], [])
    for k in values:
        client.close_handles([h for h, _ in opened[k]])
    assert server.num_handles() == 0
    assert client.read_ranges([hs[0]], [0], [0], [dsts[0]]) is False         # closed: unknown
    assert bytes(client.get("k4")) == values["k4"]


def test_refusals_keep_the_connection(server, client):
    _put(client, "v", b"0123456789")
    mem = _Buf()
    h, size, got, _ = client.open_into("v", 4, mem.alloc)
    d = ctypes.create_string_buffer(16)
    p = ctypes.addressof(d)
    assert not client.read_ranges([h + 1000], [0], [1], [p])                 # unknown handle
    assert not client.read_ranges([h], [5], [6], [p])                       # past the end
    assert not client.read_ranges([h], [11], [0], [p])                      # offset past the end
    assert not client.read_ranges([h, h], [0, 0], [2, 11], [p, p])          # one bad entry refuses the whole READ
    assert d.raw == b"\0" * 16                                               # ... and nothing was written
    assert bytes(client.get("v")) == b"0123456789"                          # still in step
    assert client.read_ranges([h], [10], [0], [p]) and client.read_ranges([h], [6], [4], [p]) and d.raw[:4] == b"6789"
    # another connection's handle is unknown there
    other = type(client)("127.0.0.1", server.port)
    assert not other.read_ranges([h], [0], [1], [p])
    assert bytes(other.get("v")) == b"0123456789"
    other.close()
    client.close_handles([h, 12345])                                         # unknown handles are ignored
    assert server.num_handles() == 0


def test_snapshot_survives_a_put(server, client):
    _put(client, "s", b"A" * 1000)
    mem = _Buf()
    h, size, _, _ = client.open_into("s", 0, mem.alloc)
    _put(client, "s", b"B" * 2000)
    d = ctypes.create_string_buffer(1000)
    assert client.read_ranges([h], [0], [1000], [ctypes.addressof(d)]) and d.raw == b"A" * 1000
    assert not client.read_ranges([h], [0], [1001], [ctypes.addressof(d)])  # the snapshot's size, not the new value's
    client.close_handles([h])


def test_handles_dropped_on_disconnect_and_capped(server):
    c = LMCNativeConnector("127.0.0.1", server.port)
    _put(c, "x", b"xyz")
    mem = _Buf()
    for _ in range(MAX_HANDLES):
        assert c.open_into("x", 1, mem.alloc) is not None
    assert c.open_into("x", 1, mem.alloc) is None                            # the cap holds
    assert bytes(c.get("x")) == b"xyz"
    assert server.num_handles() == MAX_HANDLES
    c.close()
    assert _wait_handles(server, 0)


def test_alloc_failure_closes_the_handle(server, client):
    _put(client, "y", b"abcdef")

    def boom(size):
        raise MemoryError("no room")
    with pytest.raises(MemoryError):
        client.open_into("y", 3, boom)
    assert server.num_handles() == 0 and bytes(client.get("y")) == b"abcdef"


class _ReferenceStub:
    """A server that speaks only the reference's four commands (lmcache/server/__main__.py): EXIST answers FAIL for a
    key it does not hold, and any other command is ignored -- no reply, and whatever body follows is read as the next
    header.  It records every command it receives."""

    def __init__(self):
        self.sock = socket.socket()
        self.sock.bind(("127.0.0.1", 0))
        self.sock.listen()
        self.port = self.sock.getsockname()[1]
        self.commands = []
        self.store = {}
        threading.Thread(target=self._run, daemon=True).start()

    def _run(self):
        while True:
            try:
                conn, _ = self.sock.accept()
            except OSError:
                return
            threading.Thread(target=self._serve, args=(conn,), daemon=True).start()

    def _serve(self, conn):
        n = ClientMetaMessage.packlength()
        try:
            while True:
                hdr = conn.recv(n, socket.MSG_WAITALL)
                if len(hdr) < n:
                    return
                m = ClientMetaMessage.deserialize(hdr)
                self.commands.append(m.command)
                if m.command == Constants.CLIENT_PUT:
                    self.store[m.key] = conn.recv(m.length, socket.MSG_WAITALL) if m.length else b""
                elif m.command == Constants.CLIENT_GET:
                    v = self.store.get(m.key)
                    conn.sendall(ServerMetaMessage(Constants.SERVER_FAIL if v is None else Constants.SERVER_SUCCESS,
                                                   0 if v is None else len(v)).serialize() + (v or b""))
                elif m.command == Constants.CLIENT_EXIST:
                    conn.sendall(ServerMetaMessage(Constants.SERVER_SUCCESS if m.key in self.store else
                                                   Constants.SERVER_FAIL, 0).serialize())
                elif m.command == Constants.CLIENT_LIST:
                    data = "\n".join(self.store).encode()
                    conn.sendall(ServerMetaMessage(Constants.SERVER_SUCCESS, len(data)).serialize() + data)
        finally:
            conn.close()

    def close(self):
        self.sock.close()


@pytest.mark.parametrize("kind", ["native", "python"])
def test_probe_is_false_on_the_reference_shape(kind):
    stub = _ReferenceStub()
    c = (LMCNativeConnector if kind == "native" else LMCServerConnector)("127.0.0.1", stub.port)
    try:
        c.set("a", b"1")
        assert not c.supports_ranges()
        assert bytes(c.get("a")) == b"1"
        assert max(stub.commands) <= Constants.CLIENT_LIST
    finally:
        c.close()
        stub.close()


# ---------------------------------------------------------------------------------------------- READ plan (pure)
def _containers(kind, L, H, D, ntok, rng):
    """(plane offsets, total bytes, raw rows or None, fixed-section bound) of containers of the given token counts:
    the section layout of the format, with random stream lengths"""
    latent = kind in ("v4", "v6")
    P = L if latent else 2 * L
    out = []
    for t in ntok:
        if kind in ("v3", "v4"):
            lo = N.container_layout(L, H, D, t, N.CODER_LATENT if latent else N.CODER_RANS_COMPACT)
            pay, raw = int(lo.off_payload), None
        else:
            lo = N.lossless_layout(L, H, D, t, latent)
            pay = int(lo.off_payload)
            raw = (int(lo.off_raw), t * H * D)
        o = np.concatenate([[pay], pay + np.cumsum(rng.integers(4 * H * D, 40 * H * D, P))]).astype(np.int64)
        out.append((o, int(o[-1]), raw))
    return out


@pytest.mark.parametrize("kind", ["v3", "v4", "v5", "v6"])
@pytest.mark.parametrize("k", [1, 3])
def test_read_plan_covers_every_container_once(kind, k):
    rng = np.random.default_rng(hash(kind) % 1000 + k)
    L, H, D = 5, 2, 16
    full = 256 if kind in ("v3", "v4") else 1024
    ntok = [full, full, full, full - 37]                 # a ragged tail
    cons = _containers(kind, L, H, D, ntok, rng)
    latent = kind in ("v4", "v6")
    if kind in ("v3", "v4"):
        prefix = int(N.container_layout(L, H, D, full, N.CODER_LATENT if latent else N.CODER_RANS_COMPACT).off_payload)
    else:
        prefix = int(N.lossless_layout(L, H, D, full, latent).off_raw)
    planes = [o for o, _, _ in cons]
    planes[1] = None                                     # a container uploaded whole (no plane offsets)
    nbytes = [t for _, t, _ in cons]
    raw = None if kind in ("v3", "v4") else [r for _, _, r in cons]
    fixed, start, size = layer_copy_ranges(planes, nbytes, L, 1 if latent else 2, raw)
    got = [min(prefix, t) for t in nbytes]
    got[1] = 100                                         # its prefix stops inside the fixed sections
    conn_of = [j % k for j in range(len(nbytes))]
    for max_bytes in (READ_MAX_BYTES, 5000):
        reads = ranged_read_plan(fixed, start, size, got, conn_of, k, max_bytes=max_bytes, max_ranges=7)
        cover = [np.zeros(t, np.int32) for t in nbytes]
        for j, g in enumerate(got):
            cover[j][:g] += 1
        for c in range(k):
            for layer in range(L):
                for e in reads[c][layer]:
                    assert len(e) <= 7 and e[:, 2].sum() <= max_bytes and (e[:, 2] > 0).all()
                    for j, off, nb in e.tolist():
                        assert conn_of[j] == c
                        cover[j][off:off + nb] += 1
                        if layer > 0:                    # a later layer's bytes are that layer's planes only
                            lo_ = start[layer][np.arange(start.shape[1]) % len(nbytes) == j]
                            hi_ = lo_ + size[layer][np.arange(start.shape[1]) % len(nbytes) == j]
                            assert ((lo_ <= off) & (off + nb <= hi_)).any()
        for j in range(len(nbytes)):
            assert (cover[j] == 1).all(), (kind, j)
        # whatever layer l's copy reads is in host memory once layers 0..l of every connection are done
        for layer in range(L):
            have = [np.zeros(t, bool) for t in nbytes]
            for j, g in enumerate(got):
                have[j][:g] = True
            for c in range(k):
                for lay in range(layer + 1):
                    for e in reads[c][lay]:
                        for j, off, nb in e.tolist():
                            have[j][off:off + nb] = True
            for col in range(start.shape[1]):
                j = col % len(nbytes)
                assert have[j][start[layer, col]:start[layer, col] + size[layer, col]].all()
            for j in range(len(nbytes)):
                assert have[j][:fixed[j]].all()


def test_read_plan_splits_below_2_31():
    n, L = 2, 1
    fixed = np.array([10, 10], np.int64)
    start = np.array([[10, 10, 3 << 30, 3 << 30]], np.int64)
    size = np.array([[3 << 30, 3 << 30, 1 << 30, 1 << 30]], np.int64)
    reads = ranged_read_plan(fixed, start, size, [10, 10], [0, 0], 1)
    tot = 0
    for e in reads[0][0]:
        assert e[:, 2].sum() <= READ_MAX_BYTES
        tot += int(e[:, 2].sum())
    assert tot == int(size.sum()) and len(reads[0][0]) >= 4


# ---------------------------------------------------------------------------------------------- prefix-only records
class _Blk:
    def __init__(self, data: bytes):
        self.buf = bytearray(data)
        self.freed = False

    def view(self):
        return memoryview(self.buf)

    def free(self):
        self.freed = True


def test_prefix_record_matches_the_whole_one():
    """A lossless and a CacheGen-layout container built from the format's sections: the record read from the fixed
    sections alone equals the one read from the whole container."""
    from lmcache_b200.codec import parse_header, parse_lossless_header, plane_offsets, lossless_plane_offsets

    class _Codec:
        def __init__(self, parse, offs):
            self.parse_header, self.plane_offsets = staticmethod(parse), staticmethod(offs)

        def accepts(self, hd, latent=False):
            return True
    rng = np.random.default_rng(9)
    L, H, D, t = 3, 2, 8, 200
    for kind in ("v3", "v5"):
        hd = N.Header()
        hd.magic, hd.version, hd.L, hd.H, hd.D, hd.ntokens, hd.max_dtype, hd.ngroups = \
            N.MAGIC, 3 if kind == "v3" else 5, L, H, D, t, N.DT_BF16, 1
        P, C = 2 * L, H * D
        if kind == "v3":
            lo = N.container_layout(L, H, D, t, N.CODER_RANS_COMPACT)
            half = rng.integers(2, 20, P * C).astype(np.uint8)
            fixed = bytearray(int(lo.off_payload))
            fixed[64:64 + P] = bytes([8] * P)
            fixed[int(lo.off_lengths):int(lo.off_lengths) + P * C] = half.tobytes()
            payload = 2 * int(half.astype(np.int64).sum())
            codec = _Codec(parse_header, plane_offsets)
        else:
            lo = N.lossless_layout(L, H, D, t, False)
            lens = rng.integers(4, 60, P * C).astype(np.uint16)
            fixed = bytearray(int(lo.off_payload))
            fixed[int(lo.off_lens):int(lo.off_lens) + 2 * P * C] = lens.tobytes()
            payload = int(lens.astype(np.int64).sum())
            codec = _Codec(parse_lossless_header, lossless_plane_offsets)
        hd.payload_bytes = payload
        hd.total_bytes = int(lo.off_payload) + payload
        fixed[:64] = bytes(hd)
        data = bytes(fixed) + rng.integers(0, 256, payload, dtype=np.uint8).tobytes()
        whole = read_container(codec, _Blk(data), len(data))
        if whole is None:
            pytest.skip("synthetic container not accepted by the header check")
        pre = int(lo.off_payload if kind == "v3" else lo.off_raw)
        part = read_container(codec, _Blk(data[:pre] + b"\0" * (len(data) - pre)), len(data), prefix=pre)
        assert part is not None and whole.planes is not None
        for f in ("nbytes", "ntokens", "L", "H", "D", "max_dtype", "coder"):
            assert getattr(part, f) == getattr(whole, f)
        assert np.array_equal(part.planes, whole.planes)
        short = read_container(codec, _Blk(data), len(data), prefix=70 if kind == "v3" else 64)
        assert short is not None and short.planes is None           # prefix inside the fixed sections: uploaded whole
