"""CPU: (1) the BASELINE configs[3] flow across processes -- a writer process, a reader process and one lm:// server
process -- at the level that needs no GPU: token ids -> SHA-256 chain -> engine key strings -> B2KV containers over the
wire -> header checks -> decode, with the CPU oracle standing in for the kernels on both sides;
(2) wire interoperability with the REFERENCE's own server and client (lmcache/server/__main__.py:29-104,
lmcache/storage_backend/connector/lm_connector.py:15-84), through the byte exchange of a session between the two
recorded by tests/golden/make_lm_wire.py (tests/golden/golden_lm_wire.npz)."""
import ctypes
import json
import os
import socket
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _wait_port(port, proc=None, tries=900):
    for _ in range(tries):
        try:
            socket.create_connection(("127.0.0.1", port), timeout=0.2).close()
            return True
        except OSError:
            if proc is not None and proc.poll() is not None:
                return False
            time.sleep(0.1)
    return False


WORKER = r'''
import os, sys, json
import numpy as np
sys.path.insert(0, {root!r})
import torch
from oracle import oracle as O
from lmcache_b200.codec import parse_header
from lmcache_b200.storage_backend.connector import CreateConnector
from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenGPUBytestream, CacheGenGPUEncoderOutput
from lmcache_b200.utils import CacheEngineKey
role, url, coder = sys.argv[1], sys.argv[2], int(sys.argv[3])
MODEL, L, H, D, T, cs = "lmsys/longchat-7b-16k", 3, 2, 16, 600, 256
tokens = np.random.default_rng(42).integers(0, 32000, T, dtype=np.int64)
bits = O.synth_kv_bits(L, T, H * D, seed=9)
kb, vb = O.make_bins(MODEL)
keys = [CacheEngineKey("vllm", MODEL, 2, 0, h).to_string() for h in O.sha256_chain(tokens, cs)]
conn = CreateConnector(url)
if role == "writer":
    for j, key in enumerate(keys):
        x = bits[:, :, j * cs:(j + 1) * cs]
        t = x.shape[2]
        enc = O.encode_chunk(x, O.DT_BF16, kb, vb, coder)
        mk = torch.from_numpy(enc["maxes"][0].view(np.int16)).view(torch.bfloat16).reshape(L, t, 1)
        mv = torch.from_numpy(enc["maxes"][1].view(np.int16)).view(torch.bfloat16).reshape(L, t, 1)
        raw = CacheGenGPUEncoderOutput([CacheGenGPUBytestream(torch.from_numpy(b), torch.from_numpy(ln), g) for b, ln, g in enc["groups"]],
                                       torch.from_numpy(enc["cdf"]), mk, mv, H, D, coder,
                                       torch.from_numpy(O.counts(enc["sym"]).astype(np.int32)), O.nb_map(kb, vb, L)).to_bytes()
        assert raw[4] == coder + 1
        conn.set(key, raw)
    assert conn.exists(keys[-1]) or True          # one round trip: the server has consumed the PUTs before it
    print(json.dumps({{"stored": len(keys)}}))
else:
    got, ok = 0, True
    for j, key in enumerate(keys + [CacheEngineKey("vllm", MODEL, 2, 0, "0" * 64).to_string()]):
        bs = conn.get(key)
        if bs is None:
            break
        hd = parse_header(bs)                     # structural checks of the flat container
        out = CacheGenGPUEncoderOutput.from_bytes(bytes(bs))
        enc = dict(cdf=out.cdf.numpy(), maxes=np.stack([out.max_tensors_key.view(torch.int16).numpy().view(np.uint16).reshape(L, -1),
                                                         out.max_tensors_value.view(torch.int16).numpy().view(np.uint16).reshape(L, -1)]),
                   groups=[(c.bytestream.numpy(), c.bytestream_lengths.numpy(), c.ntokens) for c in out.data_chunks], coder=out.coder)
        dec = O.decode_chunk(enc, O.DT_BF16, kb, vb, O.DT_BF16)
        x = bits[:, :, j * cs:(j + 1) * cs]
        want = O.decode_chunk(O.encode_chunk(x, O.DT_BF16, kb, vb, coder), O.DT_BF16, kb, vb, O.DT_BF16)
        ok = ok and hd.ntokens == x.shape[2] and np.array_equal(dec, want)
        got += 1
    print(json.dumps({{"hits": got, "ok": bool(ok)}}))
conn.close()
'''


@pytest.mark.parametrize("coder", [0, 1, 2])
@pytest.mark.parametrize("server_kind", ["native", "python"])
def test_c4_flow_two_processes_one_server(coder, server_kind, tmp_path):
    import json
    port = _free_port()
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    args = [sys.executable, "-m", "lmcache_b200.server", "127.0.0.1", str(port)] + (["--python"] if server_kind == "python" else [])
    srv = subprocess.Popen(args, env=env)
    try:
        assert _wait_port(port, srv)
        script = tmp_path / "worker.py"
        script.write_text(WORKER.format(root=ROOT))
        url = f"lm://127.0.0.1:{port}"
        w = subprocess.run([sys.executable, str(script), "writer", url, str(coder)], env=env, capture_output=True, text=True, timeout=300)
        assert w.returncode == 0, w.stderr[-2000:]
        assert json.loads(w.stdout.strip().splitlines()[-1]) == {"stored": 3}
        r = subprocess.run([sys.executable, str(script), "reader", url.replace("lm://", "lmn://"), str(coder)], env=env,
                           capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr[-2000:]
        assert json.loads(r.stdout.strip().splitlines()[-1]) == {"hits": 3, "ok": True}     # 2 full chunks + the 88-token tail, then a miss
    finally:
        srv.terminate()
        srv.wait()


def _recv_exact(s, n):
    buf = bytearray()
    while len(buf) < n:
        d = s.recv(min(n - len(buf), 1 << 20))
        if not d:
            break
        buf.extend(d)
    return bytes(buf)


def _wire():
    """the recorded session: calls (op, key, value or expected answer) and per call (client bytes, server bytes)"""
    z = np.load(os.path.join(HERE, "golden", "golden_lm_wire.npz"))
    calls = json.loads(z["calls"].tobytes().decode())
    return calls, [(z[f"c2s_{i}"].tobytes(), z[f"s2c_{i}"].tobytes()) for i in range(len(calls))]


class _RecordedServer:
    """plays the reference server's side of the recorded session to one connection: reads each request, which must be
    the reference client's bytes, and answers with the reference server's bytes"""

    def __init__(self, segs):
        self.sock = socket.create_server(("127.0.0.1", 0))
        self.port = self.sock.getsockname()[1]
        self.segs, self.done, self.errors = segs, 0, []
        self.thread = threading.Thread(target=self._run, daemon=True)
        self.thread.start()

    def _run(self):
        conn, _ = self.sock.accept()
        with conn:
            for i, (c2s, s2c) in enumerate(self.segs):
                got = _recv_exact(conn, len(c2s))
                if got != c2s:
                    self.errors.append(f"call {i}: request differs from the reference client's ({len(got)} B, first "
                                       f"difference at {next((k for k, (a, b) in enumerate(zip(got, c2s)) if a != b), min(len(got), len(c2s)))})")
                    return
                conn.sendall(s2c)
                self.done += 1

    def close(self):
        self.thread.join(timeout=30)
        self.sock.close()


@pytest.mark.parametrize("scheme", ["lm", "lmn"])
def test_our_clients_against_the_reference_server(scheme):
    """this package's two lm:// clients in the recorded session against the reference server's recorded answers: every
    request byte-identical to the reference client's, every answer read as the reference client read it"""
    from lmcache_b200.storage_backend.connector import CreateConnector
    calls, segs = _wire()
    srv = _RecordedServer(segs)
    try:
        c = CreateConnector(f"{scheme}://127.0.0.1:{srv.port}")
        seen = set()
        for call in calls:
            op, k = call["op"], call["key"]
            if op == "set":
                c.set(k, bytes([call["byte"]]) * call["size"])
            elif op == "exists":
                assert c.exists(k) == call["want"]
            elif op == "get":
                want = None if call["want"] is None else bytes([call["want"]["byte"]]) * call["want"]["size"]
                if want is None or k in seen:          # the second GET of a key goes through get_into
                    got = c.get(k)
                    assert (got is None) if want is None else bytes(got) == want
                else:
                    buf = np.zeros(len(want) + 64, np.uint8)
                    assert c.get_into(k, buf.ctypes.data, buf.size) == len(want) and buf[:len(want)].tobytes() == want
                    seen.add(k)
            else:
                assert sorted(c.list()) == sorted(call["want"])
        c.close()
    finally:
        srv.close()
    assert not srv.errors, srv.errors
    assert srv.done == len(segs)


def test_reference_client_against_our_native_server():
    """the reference client's recorded requests sent to csrc/lmnet.cu's server: every answer byte-identical to the
    reference server's (LIST: the same keys, in any order)"""
    import __graft_entry__ as ge
    ge.build_cuda()
    from lmcache_b200 import _native as N
    calls, segs = _wire()
    lib = N.lib()
    h = ctypes.c_void_p()
    N.check(lib.b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(h)))
    try:
        s = socket.create_connection(("127.0.0.1", lib.b200kv_lm_server_port(h)))
        for i, (call, (c2s, s2c)) in enumerate(zip(calls, segs)):
            s.sendall(c2s)
            got = _recv_exact(s, len(s2c))
            if call["op"] == "list":
                assert got[:8] == s2c[:8] and sorted(got[8:].split(b"\n")) == sorted(s2c[8:].split(b"\n")), i
            else:
                assert got == s2c, (i, call["op"])
        s.close()
        assert lib.b200kv_lm_server_num_keys(h) == 4
    finally:
        N.check(lib.b200kv_lm_server_stop(h))
